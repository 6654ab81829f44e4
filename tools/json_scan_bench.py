"""Device scan of TPC-H lineitem written as newline-delimited JSON (b200_engine_register_json).

  python tools/json_scan_bench.py [--sf 1] [--steps 3] [--warmup 1] [--no-parity]

lineitem comes from the oracle's generator and is written one object per line with every column's key, decimals as JSON
numbers and dates as "YYYY-MM-DD" strings (about twice the bytes of the .tbl file).  The file is registered twice, with q1's
columns and with all 16, and for each: the median wall time of register_json, the device time of each kernel family
(json_records, json_fields, json_convert, json_strings) and the file's GB/s over the summed device time.  The same file read
by pyarrow.json.read_json on every host core is reported beside it as an Arrow C++ stand-in for the host path (not
arrow-rs).  q1 on the scanned table is checked against the CPU oracle.  Prints one JSON line with the card's name and power
limit."""
import argparse
import os
import shutil
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402  (cpu_q1, tables_equal, usable_cpus)
from parquet_scan_bench import card  # noqa: E402

FAMILIES = ("json_records", "json_fields", "json_convert", "json_strings")


def ndjson_lines(t):
    """One JSON object per row of t, as a pyarrow string array (vectorised: no Python loop over rows)."""
    import pyarrow as pa
    import pyarrow.compute as pc
    parts = []
    for i, name in enumerate(t.column_names):
        c = t.column(i)
        if pa.types.is_string(c.type) or pa.types.is_date32(c.type):
            s = pc.cast(c, pa.string())
            s = pc.replace_substring(pc.replace_substring(s, "\\", "\\\\"), '"', '\\"')
            s = pc.binary_join_element_wise('"', s, '"', "")
        else:
            s = pc.cast(c, pa.string())
        parts.append(pc.binary_join_element_wise(("{" if i == 0 else ",") + '"' + name + '":', s, ""))
    return pc.binary_join_element_wise(*parts, "}\n", "")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=float, default=1.0)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--no-parity", action="store_true")
    args = ap.parse_args()

    import pyarrow as pa
    import pyarrow.json as pajson
    import ballista_b200 as bb
    import oracle_ffi
    from ballista_b200 import driver, tpch

    eng = bb.GpuExecutionEngine(0)
    msf = int(round(args.sf * 1000))
    rows = eng.tpch_table_rows("lineitem", msf)
    threads = bench.usable_cpus()
    oracle_ffi.build()
    o = oracle_ffi.OracleEngine()
    cols = [f["name"] for f in tpch.SCHEMAS["lineitem"]]
    schema = tpch.SCHEMAS["lineitem"]
    tmp = tempfile.mkdtemp(prefix="b200-json-scan-")
    path = os.path.join(tmp, "lineitem.json")
    out, results = {}, {}
    try:
        # written a slice at a time, so host memory holds one slice of the table
        step = 2_000_000
        with open(path, "wb") as fh:
            for r0 in range(0, rows, step):
                o.drop_table("lineitem")
                o.tpch_generate("lineitem", msf, 0, r0, min(rows, r0 + step), cols)
                t = pa.Table.from_batches([o.export_table("lineitem", 0)])
                fh.write("".join(ndjson_lines(t).to_pylist()).encode())
        o.drop_table("lineitem")
        size = os.path.getsize(path)
        print(f"written {size} bytes", file=sys.stderr, flush=True)
        # pyarrow's JSON reader does not turn strings into date32: the host reference keeps the dates as strings
        pa_schema = pa.schema([(f["name"], pa.decimal128(*f["type"]["dec"]) if isinstance(f["type"], dict) else
                                {"i64": pa.int64(), "i32": pa.int32(), "utf8": pa.string(), "date32": pa.string()}[f["type"]]) for f in schema])
        t0 = time.perf_counter()
        host = pajson.read_json(path, parse_options=pajson.ParseOptions(explicit_schema=pa_schema))
        host_s = time.perf_counter() - t0
        assert host.num_rows == rows
        del host
        eng.set_config("b200.metrics.kernel_timing", "on")
        for name, want in (("q1_columns", tpch.Q1_COLUMNS), ("all_16_columns", cols)):
            for _ in range(max(args.warmup, 1)):
                eng.drop_table("lineitem")
                eng.register_json("lineitem", 0, path, schema, columns=want)
            eng.synchronize()
            eng.kernel_stats(reset=True)
            wall = []
            for _ in range(args.steps):
                eng.drop_table("lineitem")
                t0 = time.perf_counter()
                eng.register_json("lineitem", 0, path, schema, columns=want)
                eng.synchronize()
                wall.append(time.perf_counter() - t0)
            ks = eng.kernel_stats(reset=True)
            fam = {k: {"ms": ks[k]["ms"] / args.steps, "algorithmic_gbs": (ks[k]["bytes"] / args.steps) / (ks[k]["ms"] / args.steps / 1e3) / 1e9}
                   for k in FAMILIES if k in ks and ks[k]["ms"] > 0}
            dev_ms = sum(v["ms"] for v in fam.values())
            out[name] = {"columns": len(want), "register_json_ms": 1e3 * statistics.median(wall), "device_ms": dev_ms,
                         "file_gbs_over_device_time": size / (dev_ms / 1e3) / 1e9 if dev_ms > 0 else 0.0, "families": fam}
            if name == "q1_columns":
                results[name] = driver.run_stages(eng, tpch.q1(1), "json-bench")
                eng.remove_job_data("json-bench")
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    o.close()
    parity = {"checked": False}
    if not args.no_parity:
        _, want = bench.cpu_q1(msf, 0, rows, threads, steps=1, warmup=0)
        want = pa.Table.from_batches([want])
        equal = all(bench.tables_equal(got, want) for got in results.values())
        parity = {"checked": True, "equal": equal, "what": f"q1 on the scanned table == CPU oracle q1 on the same {rows} generated rows, bit-exact"}
    name, watts = card()
    line = {
        "workload": f"device NDJSON scan of TPC-H lineitem, SF{args.sf:g} ({rows} rows, {size} bytes)",
        "steps": args.steps, "warmup": max(args.warmup, 1), "gpu": name, "power_limit_w": watts,
        "timing": "register_json: median host wall time (file in the page cache); kernels: CUDA events per kernel family",
        "scans": out,
        "host_reference": {"what": f"pyarrow.json.read_json {pa.__version__} on {threads} host threads: an Arrow C++ stand-in for the "
                                   "host path, not arrow-rs", "seconds": host_s, "file_gbs": size / host_s / 1e9},
        "parity_checked": bool(parity.get("checked") and parity.get("equal")), "parity": parity,
    }
    print(__import__("json").dumps(line), flush=True)
    eng.close()
    if parity.get("checked") and not parity.get("equal"):
        raise SystemExit(3)


if __name__ == "__main__":
    main()
