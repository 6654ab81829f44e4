"""Device time of bool / bit and regr_* aggregates against the MIN / MAX and CORR they are expected to cost like.

  python tools/regr_bool_bit_bench.py [--sf 10] [--steps 5] [--warmup 1]

TPC-H lineitem (generated on the device) in one partition, one Single AggregateExec per plan, keyed on
(l_returnflag, l_linestatus) (4 groups: the register sink) and on l_suppkey (the global sink):
  bitbool   bit_or(l_partkey), bool_and(l_quantity < 25)       against   minmax   max(l_partkey), min(l_quantity < 25)
  regr      all nine regr_*(l_extendedprice, l_quantity)       against   corr     corr(l_quantity, l_extendedprice)
For each: the median over --steps runs of the summed device time of the pipeline_agg_* kernel families (pass 2
included), and the step's wall time.  Prints one JSON line with the card's name and power limit."""
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

REGR = ["regr_slope", "regr_intercept", "regr_count", "regr_r2", "regr_avgx", "regr_avgy", "regr_sxx", "regr_syy", "regr_sxy"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=float, default=10.0)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()

    import ballista_b200 as bb
    from ballista_b200 import driver
    from ballista_b200 import plan as P
    c = P.col

    eng = bb.GpuExecutionEngine(0)
    msf = int(round(args.sf * 1000))
    rows = eng.tpch_table_rows("lineitem", msf)
    cols = ["l_partkey", "l_suppkey", "l_quantity", "l_extendedprice", "l_returnflag", "l_linestatus"]
    eng.tpch_generate("lineitem", msf, 0, 0, rows, cols)
    sch = [P.field("l_partkey", "i64", False), P.field("l_suppkey", "i64", False), P.field("l_quantity", P.dec(15, 2), False),
           P.field("l_extendedprice", P.dec(15, 2), False), P.field("l_returnflag", "utf8", False), P.field("l_linestatus", "utf8", False)]
    small = P.binop("<", c("l_quantity"), P.lit_dec(2500, 15, 2))
    plans = {
        "bitbool": [P.agg("bit_or", c("l_partkey"), "bo"), P.agg("bool_and", small, "ba")],
        "minmax": [P.agg("max", c("l_partkey"), "mx"), P.agg("min", small, "mn")],
        "regr": [P.agg(fn, c("l_extendedprice"), fn, arg2=c("l_quantity")) for fn in REGR],
        "corr": [P.agg("corr", c("l_quantity"), "cr", arg2=c("l_extendedprice"))],
    }
    keys = {"reg": [(c("l_returnflag"), "rf"), (c("l_linestatus"), "ls")], "global": [(c("l_suppkey"), "sk")]}
    eng.set_config("b200.metrics.kernel_timing", "on")
    out = {}
    for kname, kk in keys.items():
        for pname, aggs in plans.items():
            st = [P.Stage(1, P.shuffle_writer(P.aggregate("Single", kk, aggs, P.scan("lineitem", sch)), 1))]
            dev, wall, fams = [], [], None
            for i in range(args.warmup + args.steps):
                eng.kernel_stats(reset=True)
                t0 = time.perf_counter()
                res = driver.run_stages(eng, st, f"rbb-{kname}-{pname}-{i}")
                t1 = time.perf_counter()
                ks = eng.kernel_stats()
                if i >= args.warmup:
                    agg = {k: v for k, v in ks.items() if k.startswith("pipeline_agg") or k.startswith("pipeline_fused") or k.startswith("groupby")}
                    dev.append(sum(v["ms"] for v in agg.values()))
                    wall.append((t1 - t0) * 1e3)
                    fams = sorted(agg)
            out[f"{kname}/{pname}"] = {"agg_kernel_ms": round(statistics.median(dev), 3), "step_ms": round(statistics.median(wall), 3),
                                       "families": fams, "groups": res.num_rows}
    name, watts = card()
    print(json.dumps({"bench": "regr_bool_bit", "sf": args.sf, "rows": rows, "steps": args.steps, "gpu": name, "power_limit_w": watts,
                      "results": out}))
    eng.close()


if __name__ == "__main__":
    main()
