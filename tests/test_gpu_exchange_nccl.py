"""Two executors on two GPUs: the in-library NCCL exchange (b200_exchange_stage) under the distributed stage
driver, results compared with the CPU oracle on the GLOBAL tables.  Needs 2 GPUs; skipped on
a single-GPU box.  Covers the three exchange modes: hash repartition (every query), gather to the merge task
(every final stage) and broadcast of a join build side (q5 stage 1 -> stage 2), with inline (q1: a few hundred
bytes) and direct (q5 / q3: the lineitem shuffle) payloads and string columns."""
import multiprocessing as mp
import os

import pyarrow as pa
import pytest

from ballista_b200 import driver, tpch
from util import assert_tables_equal

pytestmark = pytest.mark.gpu


def _n_gpus():
    try:
        import subprocess
        out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True, timeout=20).stdout
        return sum(1 for ln in out.splitlines() if ln.startswith("GPU "))
    except Exception:
        return 0


def _worker(rank, world, nccl_id, case, q, window):
    try:
        import ballista_b200 as bb
        eng = bb.GpuExecutionEngine(rank, 0, rank, world)
        if window:
            eng.set_config("b200.exchange.window_bytes", str(window))
        eng.comm_init(nccl_id)
        name, tables, msf, parts, stages = case
        eng.tpch_load(tables, msf, rank, world, parts)
        stats = []
        res = driver.run_stages_distributed(eng, stages, f"{name}-dist", rank, world, on_stage=lambda s, m, st: stats.append((s, m, st)),
                                            fused=bool(window))
        stats.append((-1, -1, {"fused_exchanges": eng.counter("fused_exchanges"), "window": eng.counter("exchange_window_bytes")}))
        payload = None
        if rank == 0 and res is not None:
            sink = pa.BufferOutputStream()
            with pa.ipc.new_stream(sink, res.schema) as w:
                w.write_table(res)
            payload = sink.getvalue().to_pybytes()
        q.put((rank, "ok", payload, stats))
        eng.close()
    except Exception as ex:  # pragma: no cover
        import traceback
        q.put((rank, "error", traceback.format_exc(), None))


def _run_case(case, world=2, window=0):
    import ballista_b200 as bb
    ctx = mp.get_context("spawn")
    nccl_id = bb.GpuExecutionEngine.comm_unique_id()
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, nccl_id, case, q, window)) for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    for _ in range(world):
        rank, status, payload, stats = q.get(timeout=300)
        assert status == "ok", payload
        got[rank] = (payload, stats)
    for p in procs:
        p.join(timeout=60)
    table = pa.ipc.open_stream(got[0][0]).read_all() if got[0][0] else None
    return table, got[0][1]


def _oracle(oracle, oracle_lib, case):
    name, tables, msf, parts, stages = case
    for t, cols in tables.items():
        n = oracle_lib.lib().oracle_tpch_table_rows(t.encode(), msf)
        oracle.drop_table(t)
        np_ = 1 if n < 1000 else 2
        step = (n + np_ - 1) // np_
        for p in range(np_):
            oracle.tpch_generate(t, msf, p, min(n, p * step), min(n, (p + 1) * step), cols)
    return driver.run_stages(oracle, stages, f"{name}-o")


needs2 = pytest.mark.skipif(_n_gpus() < 2, reason="needs 2 GPUs")


@needs2
def test_q1_two_gpus(oracle, oracle_lib):
    case = ("q1", {"lineitem": tpch.Q1_COLUMNS}, 100, 2, tpch.q1(4))
    got, stats = _run_case(case)
    want = _oracle(oracle, oracle_lib, case)
    assert_tables_equal(got, want, sort=False)
    assert stats and all(st["sent_bytes"] < 16384 for s, _, st in stats if s >= 0)   # the inline path


@needs2
def test_q5_two_gpus(oracle, oracle_lib):
    case = ("q5", tpch.Q5_TABLES, 200, 2, tpch.q5(4))
    got, stats = _run_case(case)
    want = _oracle(oracle, oracle_lib, case)
    assert want.num_rows > 0
    assert_tables_equal(got, want, sort=False)
    assert any(st["sent_bytes"] > 16384 for s, _, st in stats if s >= 0)    # the lineitem shuffle took the direct path
    assert any(m == 2 for _, m, _ in stats)                                  # the broadcast build side


@needs2
@pytest.mark.parametrize("window", [256 << 20, 4096])
def test_q5_two_gpus_fused_shuffle(oracle, oracle_lib, window):
    """Writer + hash exchange as one collective (b200_stage_execute_exchange): the scatter kernel stores the rows of the
    fixed-width shuffles (lineitem, orders, supplier keys) straight into the owning executor's window over NVLink.  With a
    window too small for any exchange every executor falls back to the two-step path; same result either way."""
    case = ("q5f", tpch.Q5_TABLES, 200, 2, tpch.q5(4))
    got, stats = _run_case(case, window=window)
    want = _oracle(oracle, oracle_lib, case)
    assert want.num_rows > 0
    assert_tables_equal(got, want, sort=False)
    info = [st for s, _, st in stats if s == -1][0]
    assert info["window"] >= window
    assert any(st.get("fused") for s, _, st in stats if s >= 0)             # the driver took the collective entry point
    if window > 4096:
        assert info["fused_exchanges"] >= 3                                  # ... and the kernel wrote into the peers' windows
        assert any(st.get("fused") and st["sent_bytes"] > 16384 for s, _, st in stats if s >= 0)
    else:
        assert info["fused_exchanges"] == 0


@needs2
def test_q17_q12_two_gpus_fused_shuffle(oracle, oracle_lib):
    """Nullable / multi-task shapes through the fused shuffle: q12 and q17 at 2 map tasks per executor."""
    for name, tables in (("q12", tpch.Q12_TABLES), ("q17", tpch.Q17_TABLES)):
        msf = 100
        if name == "q17":
            for t, cols in tables.items():
                n = oracle_lib.lib().oracle_tpch_table_rows(t.encode(), msf)
                oracle.drop_table(t)
                oracle.tpch_generate(t, msf, 0, 0, n, cols)
            first = pa.Table.from_batches([oracle.export_table("part", 0)]).slice(0, 1).to_pylist()[0]
            stages = tpch.q17(4, first["p_brand"], first["p_container"])
        else:
            stages = tpch.q12(4)
        case = (name + "f", tables, msf, 2, stages)
        got, stats = _run_case(case, window=256 << 20)
        want = _oracle(oracle, oracle_lib, case)
        assert_tables_equal(got, want, sort=False, f64_rtol=1e-12)
        # q17 shuffles lineitem as (l_partkey, l_quantity, l_extendedprice): fixed width -> written into the peers' windows;
        # both of q12's shuffles carry a string column and take the two-step path
        assert ([st for s, _, st in stats if s == -1][0]["fused_exchanges"] >= 1) == (name == "q17")


@needs2
def test_q3_q12_q17_two_gpus(oracle, oracle_lib):
    seg = None
    for name, tables, mk in (("q12", tpch.Q12_TABLES, lambda: tpch.q12(4)), ("q17", tpch.Q17_TABLES, None), ("q3", tpch.Q3_TABLES, None)):
        msf = 100
        if name == "q17" or name == "q3":
            # parameters that exist in the generated data
            for t, cols in tables.items():
                n = oracle_lib.lib().oracle_tpch_table_rows(t.encode(), msf)
                oracle.drop_table(t)
                oracle.tpch_generate(t, msf, 0, 0, n, cols)
            if name == "q17":
                first = pa.Table.from_batches([oracle.export_table("part", 0)]).slice(0, 1).to_pylist()[0]
                stages = tpch.q17(4, first["p_brand"], first["p_container"])
            else:
                seg = pa.Table.from_batches([oracle.export_table("customer", 0)]).slice(0, 1).to_pylist()[0]["c_mktsegment"]
                stages = tpch.q3(4, seg)
        else:
            stages = mk()
        case = (name, tables, msf, 2, stages)
        got, _ = _run_case(case)
        want = _oracle(oracle, oracle_lib, case)
        if name == "q3":
            assert got.column("revenue").to_pylist() == want.column("revenue").to_pylist()
            assert_tables_equal(got, want, sort=True)
        else:
            assert_tables_equal(got, want, sort=False, f64_rtol=1e-12)
