"""Device time of the math functions (DESIGN.md §6 (xviii)) in a projection, against abs of the same column (the cold-op
baseline).

  python tools/math_fn_bench.py [--sf 10] [--steps 5] [--warmup 1] [--fns sqrt exp ...]

TPC-H lineitem (generated on the device) in one partition.  Each plan projects one function over
CAST(l_extendedprice AS DOUBLE) (f64) or over CAST(l_extendedprice AS FLOAT) (f32).  For each: the median over --steps runs
of the pipeline kernels' device time, and GB/s of the input (the 16-byte Decimal128 column) plus the output (8 or 4 bytes a
row) over it.  Prints one JSON line with the card's name and power limit; fails without a GPU."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from parquet_scan_bench import card  # noqa: E402

FNS = ["abs", "sqrt", "cbrt", "exp", "ln", "log10", "sin", "cos", "tan", "atan", "tanh", "asinh", "degrees", "signum", "trunc",
       "power", "atan2", "log_base"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=float, default=10.0)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--fns", nargs="+", default=FNS)
    args = ap.parse_args()

    import ballista_b200 as bb
    from ballista_b200 import driver
    from ballista_b200 import plan as P
    c = P.col

    eng = bb.GpuExecutionEngine(0)
    name, watts = card()
    msf = int(round(args.sf * 1000))
    rows = eng.tpch_table_rows("lineitem", msf)
    eng.drop_table("lineitem")
    eng.tpch_generate("lineitem", msf, 0, 0, rows, ["l_extendedprice"])
    sch = [P.field("l_extendedprice", P.dec(15, 2), False)]
    eng.set_config("b200.metrics.kernel_timing", "on")
    out = {}
    for t in ("f64", "f32"):
        x = P.cast(c("l_extendedprice"), t)
        for fn in args.fns:
            if fn == "power" and t == "f32":
                continue
            if fn == "power":
                e = P.fn("power", x, P.lit_f64(0.5))
            elif fn == "atan2":
                e = P.fn("atan2", x, x)
            elif fn == "log_base":
                e = P.fn("log", x, x)
            elif fn == "trunc":
                e = P.fn("trunc", x, P.lit_i64(1))
            else:
                e = P.fn(fn, x)
            st = [P.Stage(1, P.shuffle_writer(P.project([(e, "r")], P.scan("lineitem", sch)), 1))]
            dev = []
            for i in range(args.warmup + args.steps):
                eng.kernel_stats(reset=True)
                res = driver.run_stages(eng, st, f"mfb-{t}-{fn}-{i}")
                ks = eng.kernel_stats()
                if i >= args.warmup:
                    dev.append(sum(v["ms"] for k, v in ks.items() if k.startswith("pipeline")))
            assert res.num_rows == rows
            ms = statistics.median(dev)
            nbytes = rows * (16 + (8 if t == "f64" else 4))
            out[f"{fn}/{t}"] = {"device_ms": round(ms, 3), "gb_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1)}
    print(json.dumps({"bench": "math_fn", "sf": args.sf, "rows": rows, "steps": args.steps, "gpu": name, "power_limit_w": watts,
                      "results": out}), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
