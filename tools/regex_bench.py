"""Device regex predicates (OP_REGEX: one thread per row walks the DFA) against the LIKE operation they replace.

  python tools/regex_bench.py [--sf 10] [--steps 5] [--warmup 2]

TPC-H lineitem.l_comment and part.p_name are generated in HBM (tpch_generate; the generator writes random lower-case
letters, so the patterns are chosen to hit that data).  Each case is one stage: FilterExec(predicate) under a partial
COUNT(*), prepared once and executed `steps` times after `warmup` runs.  Reported per case: the median device time of the
stage's kernels (CUDA events, b200.metrics.kernel_timing), the median wall time of the stage, the string bytes of the
column over the device time, and the rows kept.  Pairs that must agree (a regex and the LIKE it restates) are checked.
Prints one JSON line with the card's name and power limit read in the same run."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from parquet_scan_bench import card  # noqa: E402


def cases(P):
    lc, pn = P.col("l_comment"), P.col("p_name")
    return [
        ("l_comment ~ 'q.*z'", "lineitem", "l_comment", P.regex_match(lc, "q.*z")),
        ("l_comment LIKE '%q%z%'", "lineitem", "l_comment", P.like(lc, "%q%z%")),
        ("l_comment ~ '^[a-m]{3}(ab|cd)+'", "lineitem", "l_comment", P.regex_match(lc, "^[a-m]{3}(ab|cd)+")),
        ("p_name ILIKE '%GREEN%'", "part", "p_name", P.like(pn, "%GREEN%", case_insensitive=True)),
        ("p_name LIKE '%green%'", "part", "p_name", P.like(pn, "%green%")),
        ("p_name ~ '^[a-m]{3}(ab|cd)+'", "part", "p_name", P.regex_match(pn, "^[a-m]{3}(ab|cd)+")),
    ]


AGREE = [("l_comment ~ 'q.*z'", "l_comment LIKE '%q%z%'"), ("p_name ILIKE '%GREEN%'", "p_name LIKE '%green%'")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=float, default=10.0)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--parts", type=int, default=4)
    args = ap.parse_args()

    import pyarrow as pa
    import ballista_b200 as bb
    from ballista_b200 import plan as P

    name, watts = card()
    eng = bb.GpuExecutionEngine(0)
    eng.set_config("b200.metrics.kernel_timing", "on")
    msf = int(round(args.sf * 1000))
    rows = eng.tpch_load({"lineitem": ["l_comment"], "part": ["p_name"]}, msf, parts=args.parts)

    def run(table, col, pred, job, agg_fn):
        sch = [P.field(col, "utf8", False)]
        scan = P.scan(table, sch)
        node = P.aggregate("Partial", [], [agg_fn(P)], P.filter_(pred, scan) if pred is not None else scan)
        st = P.Stage(1, P.shuffle_writer(node, 1))
        qse = eng.create_query_stage_exec(job, 1, st.json(job))
        n_parts = eng.n_table_partitions(table)
        dev, wall, value = [], [], None
        for i in range(args.warmup + args.steps):
            eng.remove_job_data(job)
            eng.synchronize()
            eng.kernel_stats(reset=True)
            t0 = time.perf_counter()
            for p in range(n_parts):
                qse.execute_query_stage(p)
            eng.synchronize()
            t1 = time.perf_counter()
            ks = eng.kernel_stats(reset=True)
            if i >= args.warmup:
                wall.append((t1 - t0) * 1e3)
                dev.append(sum(v["ms"] for v in ks.values()))
            tbl = pa.Table.from_batches([eng.partition_export(job, 1, 0)])
            value = sum(v for v in tbl.column(0).to_pylist() if v is not None)
        qse.release()
        eng.remove_job_data(job)
        return value, statistics.median(dev) if dev else None, statistics.median(wall)

    col_bytes = {}
    for table, col in (("lineitem", "l_comment"), ("part", "p_name")):
        col_bytes[col], _, _ = run(table, col, None, f"bytes-{col}", lambda P, c=col: P.agg("sum", P.fn("octet_length", P.col(c)), "b"))
    results = {}
    for i, (label, table, col, pred) in enumerate(cases(P)):
        kept, dev_ms, wall_ms = run(table, col, pred, f"rx{i}", lambda P: P.agg("count", None, "n"))
        results[label] = {"rows": rows[table], "kept": kept, "string_bytes": col_bytes[col], "device_ms": dev_ms, "wall_ms": wall_ms,
                          "GBps_device": (col_bytes[col] / (dev_ms * 1e6)) if dev_ms else None}
        sys.stderr.write(f"{label:36s} kept {kept:>10}  device {dev_ms:8.3f} ms  wall {wall_ms:8.3f} ms  "
                         f"{results[label]['GBps_device'] or 0:7.1f} GB/s of string bytes\n")
    agree = all(results[a]["kept"] == results[b]["kept"] for a, b in AGREE)
    regex_compiles = eng.counter("regex_compiles")
    eng.close()
    out = {"bench": "regex", "sf": args.sf, "card": name, "power_limit_w": watts, "steps": args.steps, "warmup": args.warmup,
           "parity": agree, "regex_compiles": regex_compiles, "cases": results}
    print(json.dumps(out))
    if not agree:
        sys.exit(1)


if __name__ == "__main__":
    main()
