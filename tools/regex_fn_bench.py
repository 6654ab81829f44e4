"""Device regexp_count and regexp_replace (the count op and the replace builder over the span DFAs) on TPC-H l_comment.

  python tools/regex_fn_bench.py [--sf 10] [--steps 5] [--warmup 2]

lineitem.l_comment is generated in HBM (tpch_generate; the generator writes random lower-case letters, so the
patterns are chosen to hit that data).  Each case is one stage: a partial SUM over the function's result (the count, or the
octet_length of the replaced string, so every replaced byte is built), prepared once and executed `steps` times after
`warmup` runs.  Reported per case: the median device time of the stage's kernels (CUDA events, b200.metrics.kernel_timing),
the median wall time of the stage, the column's string bytes over the device time, and the summed value.  Prints one JSON
line with the card's name and power limit read in the same run."""
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
    lc, s = P.col("l_comment"), P.lit_utf8
    count = lambda *a: P.agg("sum", P.fn("regexp_count", lc, *a), "v")                                    # noqa: E731
    replaced = lambda *a: P.agg("sum", P.fn("octet_length", P.fn("regexp_replace", lc, *a)), "v")       # noqa: E731
    return [
        ("regexp_count(l_comment, 'e')", count(s("e"))),
        ("regexp_count(l_comment, '[a-f]+')", count(s("[a-f]+"))),
        ("regexp_count(l_comment, 'q.*z')", count(s("q.*z"))),
        ("regexp_replace(l_comment, 'e', 'E')", replaced(s("e"), s("E"))),
        ("regexp_replace(l_comment, 'e', 'E', 'g')", replaced(s("e"), s("E"), s("g"))),
        ("regexp_replace(l_comment, '[a-f]+', '-', 'g')", replaced(s("[a-f]+"), s("-"), s("g"))),
    ]


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
    rows = eng.tpch_load({"lineitem": ["l_comment"]}, msf, parts=args.parts)["lineitem"]

    def run(agg, job):
        scan = P.scan("lineitem", [P.field("l_comment", "utf8", False)])
        st = P.Stage(1, P.shuffle_writer(P.aggregate("Partial", [], [agg], scan), 1))
        qse = eng.create_query_stage_exec(job, 1, st.json(job))
        n_parts = eng.n_table_partitions("lineitem")
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

    col_bytes, _, _ = run(P.agg("sum", P.fn("octet_length", P.col("l_comment")), "b"), "bytes")
    results = {}
    for i, (label, agg) in enumerate(cases(P)):
        value, dev_ms, wall_ms = run(agg, f"rxfn{i}")
        results[label] = {"rows": rows, "value": value, "string_bytes": col_bytes, "device_ms": dev_ms, "wall_ms": wall_ms,
                          "GBps_device": (col_bytes / (dev_ms * 1e6)) if dev_ms else None}
        sys.stderr.write(f"{label:48s} value {value:>12}  device {dev_ms:8.3f} ms  wall {wall_ms:8.3f} ms  "
                         f"{results[label]['GBps_device'] or 0:7.1f} GB/s of string bytes\n")
    # without g only the first 'e' changes, and a one-byte replacement keeps every length
    sane = results["regexp_replace(l_comment, 'e', 'E')"]["value"] == col_bytes == results["regexp_replace(l_comment, 'e', 'E', 'g')"]["value"]
    eng.close()
    out = {"bench": "regex_fn", "sf": args.sf, "card": name, "power_limit_w": watts, "steps": args.steps, "warmup": args.warmup,
           "lengths_kept": sane, "cases": results}
    print(json.dumps(out))
    if not sane:
        sys.exit(1)


if __name__ == "__main__":
    main()
