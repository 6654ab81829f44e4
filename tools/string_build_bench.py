"""Device string builders (concat / || / concat_ws / CAST .. AS Utf8 writing into the launch's character arena) over TPC-H
lineitem.

  python tools/string_build_bench.py [--sf 10] [--steps 5] [--warmup 2]

lineitem is generated in HBM (tpch_generate).  Each case is one stage, ProjectionExec(expression) under an unpartitioned
shuffle writer, prepared once and executed `steps` times after `warmup` runs.  Reported per case: the median device time of
the stage's kernels (CUDA events, b200.metrics.kernel_timing), the median wall time, and bytes per second of device time,
counting the input bytes the expression reads (values, offsets and characters) plus the bytes of the result strings
(intermediate results, such as the cast inside `||`, are written to the arena too but not counted).  string_arena_retries
must stay 0: every case has a sound first arena.  The results of the last run are checked against a host computation on
a sample of rows.  Prints one JSON line with the card's name and power limit read in the same run."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from parquet_scan_bench import card  # noqa: E402


def cases(P):
    c = P.col
    return [
        ("CAST(l_orderkey AS Utf8) || '-' || l_shipmode", ["l_orderkey", "l_shipmode"],
         P.str_concat(P.cast(c("l_orderkey"), "utf8"), P.lit_utf8("-"), c("l_shipmode"))),
        ("concat_ws('|', l_returnflag, l_linestatus, l_shipmode)", ["l_returnflag", "l_linestatus", "l_shipmode"],
         P.fn("concat_ws", P.lit_utf8("|"), c("l_returnflag"), c("l_linestatus"), c("l_shipmode"))),
        ("CAST(l_extendedprice AS Utf8)", ["l_extendedprice"], P.cast(c("l_extendedprice"), "utf8")),
    ]


def host_value(S, row, label):
    if label.startswith("CAST(l_orderkey"):
        return S.str_concat(S.str_concat(str(row["l_orderkey"]), "-"), row["l_shipmode"])
    if label.startswith("concat_ws"):
        return S.concat_ws("|", row["l_returnflag"], row["l_linestatus"], row["l_shipmode"])
    return S.cast_decimal(S._unscaled(row["l_extendedprice"], 2), 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=float, default=10.0)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--parts", type=int, default=4)
    args = ap.parse_args()

    import pyarrow as pa
    import pyarrow.compute as pc
    import ballista_b200 as bb
    import string_build_cases as S
    from ballista_b200 import plan as P
    from ballista_b200 import tpch

    name, watts = card()
    eng = bb.GpuExecutionEngine(0)
    eng.set_config("b200.metrics.kernel_timing", "on")
    msf = int(round(args.sf * 1000))
    cols = ["l_orderkey", "l_shipmode", "l_returnflag", "l_linestatus", "l_extendedprice"]
    rows = eng.tpch_load({"lineitem": cols}, msf, parts=args.parts)["lineitem"]
    n_parts = eng.n_table_partitions("lineitem")
    # input bytes per column: fixed-width values, or Arrow offsets plus characters
    col_bytes = {}
    for cname in cols:
        b = 0
        for p in range(n_parts):
            a = eng.export_table("lineitem", p).column(cname)
            if pa.types.is_string(a.type):
                b += 4 * len(a) + pc.sum(pc.binary_length(a)).as_py()
            else:
                b += a.type.byte_width * len(a)
        col_bytes[cname] = b

    results = {}
    retries0 = eng.counter("string_arena_retries")
    ok = True
    for i, (label, used, e) in enumerate(cases(P)):
        job = f"sb{i}"
        st = P.Stage(1, P.shuffle_writer(P.project([(e, "r")], tpch.table_scan("lineitem", cols)), 1))
        qse = eng.create_query_stage_exec(job, 1, st.json(job))
        dev, wall = [], []
        out_bytes = 0
        for it in range(args.warmup + args.steps):
            eng.remove_job_data(job)
            eng.synchronize()
            eng.kernel_stats(reset=True)
            t0 = time.perf_counter()
            for p in range(n_parts):
                qse.execute_query_stage(p)
            eng.synchronize()
            t1 = time.perf_counter()
            ks = eng.kernel_stats(reset=True)
            if it >= args.warmup:
                wall.append((t1 - t0) * 1e3)
                dev.append(sum(v["ms"] for v in ks.values()))
        out_bytes = 0
        for p in range(n_parts):
            got = eng.partition_export(job, 1, p).column(0)
            out_bytes += pc.sum(pc.binary_length(got)).as_py() or 0
            src = eng.export_table("lineitem", p)
            for k in range(0, len(got), max(1, len(got) // 2000)):
                row = {cn: src.column(cn)[k].as_py() for cn in used}
                if got[k].as_py() != host_value(S, row, label):
                    ok = False
        qse.release()
        eng.remove_job_data(job)
        in_bytes = sum(col_bytes[cn] for cn in used)
        dev_ms, wall_ms = statistics.median(dev), statistics.median(wall)
        results[label] = {"rows": rows, "input_bytes": in_bytes, "result_bytes": out_bytes, "device_ms": dev_ms, "wall_ms": wall_ms,
                          "GBps_device": (in_bytes + out_bytes) / (dev_ms * 1e6) if dev_ms else None}
        sys.stderr.write(f"{label:60s} device {dev_ms:8.3f} ms  wall {wall_ms:8.3f} ms  "
                         f"{results[label]['GBps_device'] or 0:7.1f} GB/s (input + result bytes)\n")
    retries = eng.counter("string_arena_retries") - retries0
    eng.close()
    out = {"bench": "string_build", "sf": args.sf, "card": name, "power_limit_w": watts, "steps": args.steps, "warmup": args.warmup,
           "parity_sampled": ok, "string_arena_retries": retries, "cases": results}
    print(json.dumps(out))
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
