"""Device time of first_value / last_value against a plain MIN of the same shape.

  python tools/first_last_bench.py [--sf 1 10] [--steps 5] [--warmup 1]

TPC-H lineitem (generated on the device) in one partition, one Single AggregateExec per plan, keyed on
(l_returnflag, l_linestatus) (4 groups: the register sink) and on l_orderkey (the global sink):
  last      last_value(l_shipmode ORDER BY l_shipdate, l_linenumber)     against   min   min(l_shipmode)
For each: the median over --steps runs of the device time, launches and algorithmic bytes of every pipeline_agg_*
kernel family (pass 1 and each first/last pass apart), and the step's wall time.  Prints one JSON line per scale factor
with the card's name and power limit; fails without a GPU."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=float, nargs="+", default=[1.0, 10.0])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()

    import ballista_b200 as bb
    from ballista_b200 import driver
    from ballista_b200 import plan as P
    c = P.col

    eng = bb.GpuExecutionEngine(0)
    name, watts = card()
    cols = ["l_orderkey", "l_linenumber", "l_shipdate", "l_shipmode", "l_returnflag", "l_linestatus"]
    sch = [P.field("l_orderkey", "i64", False), P.field("l_linenumber", "i32", False), P.field("l_shipdate", "date32", False),
           P.field("l_shipmode", "utf8", False), P.field("l_returnflag", "utf8", False), P.field("l_linestatus", "utf8", False)]
    ob = [P.sort_key(c("l_shipdate")), P.sort_key(c("l_linenumber"))]
    plans = {"last": [P.agg("last_value", c("l_shipmode"), "m", order_by=ob)], "min": [P.agg("min", c("l_shipmode"), "m")]}
    keys = {"reg": [(c("l_returnflag"), "rf"), (c("l_linestatus"), "ls")], "global": [(c("l_orderkey"), "ok")]}
    eng.set_config("b200.metrics.kernel_timing", "on")
    for sf in args.sf:
        msf = int(round(sf * 1000))
        rows = eng.tpch_table_rows("lineitem", msf)
        eng.drop_table("lineitem")
        eng.tpch_generate("lineitem", msf, 0, 0, rows, cols)
        out = {}
        for kname, kk in keys.items():
            for pname, aggs in plans.items():
                st = [P.Stage(1, P.shuffle_writer(P.aggregate("Single", kk, aggs, P.scan("lineitem", sch)), 1))]
                dev, wall, fams = [], [], {}
                for i in range(args.warmup + args.steps):
                    eng.kernel_stats(reset=True)
                    passes0 = eng.counter("first_last_passes")
                    t0 = time.perf_counter()
                    res = driver.run_stages(eng, st, f"flb-{sf}-{kname}-{pname}-{i}")
                    t1 = time.perf_counter()
                    ks = eng.kernel_stats()
                    if i >= args.warmup:
                        agg = {k: v for k, v in ks.items() if k.startswith("pipeline_agg") or k.startswith("pipeline_fused") or k.startswith("groupby")}
                        dev.append(sum(v["ms"] for v in agg.values()))
                        wall.append((t1 - t0) * 1e3)
                        for k, v in agg.items():
                            fams.setdefault(k, []).append(v)
                        passes = eng.counter("first_last_passes") - passes0
                out[f"{kname}/{pname}"] = {
                    "agg_kernel_ms": round(statistics.median(dev), 3), "step_ms": round(statistics.median(wall), 3), "groups": res.num_rows,
                    "first_last_passes": passes,
                    "families": {k: {"ms": round(statistics.median(x["ms"] for x in v), 3), "launches": v[0]["launches"], "bytes": v[0]["bytes"]}
                                 for k, v in sorted(fams.items())}}
        print(json.dumps({"bench": "first_last", "sf": sf, "rows": rows, "steps": args.steps, "gpu": name, "power_limit_w": watts,
                          "results": out}), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
