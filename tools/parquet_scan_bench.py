"""Device Parquet scan of TPC-H lineitem's q1 columns in several page encodings (b200_engine_register_parquet).

  python tools/parquet_scan_bench.py [--sf 10] [--steps 5] [--warmup 2] [--codec snappy|gzip|lz4|none] [--no-parity]

The columns come from the oracle's generator and are written by pyarrow, with --codec (default Snappy), into a temporary
directory in the encodings of FILES.  With gzip or lz4 each file also reports the GB/s of uncompressed page bytes its
decompression kernel (family parquet_gzip / parquet_lz4) writes.  Per file: warmed-up median wall time of the
registration, device time and achieved GB/s of the value decode (family parquet_decode_values; GB/s = (uncompressed page bytes read + decoded Arrow bytes written) / device
time), the other scan kernels' device time and pages per column.  Then q1 on each scanned table is checked against the
CPU oracle.  Prints one JSON line, with the card name and its power limit beside the numbers."""
import argparse
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402  (cpu_q1, tables_equal, usable_cpus, measured_hbm_peak)

# --codec -> (pyarrow write options, codec name in FILES' descriptions, decompression kernel family reported as GB/s).
# gzip is written at zlib's default level 6, which Hadoop's and Spark's GzipCodec use; pyarrow's own default, level 9, is
# about nine times slower to write (a minute per SF1 file).
CODECS = {"snappy": (dict(compression="snappy"), "Snappy", None),
          "gzip": (dict(compression="gzip", compression_level=6), "GZIP", "parquet_gzip"),
          "lz4": (dict(compression="lz4"), "LZ4_RAW", "parquet_lz4"),
          "none": (dict(compression="none"), "uncompressed", None)}

FILES = {
    "default": "pyarrow's defaults: dictionary pages (PLAIN once a dictionary grows too large), decimals as FIXED_LEN_BYTE_ARRAY, Snappy",
    "plain": "PLAIN pages, decimals as INT64, Snappy",
    "delta": "DELTA_BINARY_PACKED integers / dates / decimals (as INT64), DELTA_LENGTH_BYTE_ARRAY strings, Snappy",
}


def write_options(kind, schema):
    import pyarrow as pa
    if kind == "default":
        return {}
    if kind == "plain":
        return dict(use_dictionary=False, store_decimal_as_integer=True)
    enc = {f.name: "DELTA_LENGTH_BYTE_ARRAY" if pa.types.is_string(f.type) else "DELTA_BINARY_PACKED" for f in schema}
    return dict(use_dictionary=False, column_encoding=enc, store_decimal_as_integer=True)


def card(gpu_index=0):
    """(name, power limit in W) of the card, read-only queries; None where unavailable."""
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(gpu_index)
        name = pynvml.nvmlDeviceGetName(h)
        return (name.decode() if isinstance(name, bytes) else name), pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1000.0
    except Exception:
        pass
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", str(gpu_index)],
                           capture_output=True, text=True, timeout=10)
        name, watts = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return name, float(watts)
    except Exception:
        return None, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=float, default=10.0)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--codec", choices=sorted(CODECS), default="snappy")
    ap.add_argument("--no-parity", action="store_true")
    args = ap.parse_args()

    from concurrent.futures import ThreadPoolExecutor
    import pyarrow as pa
    import pyarrow.parquet as pq
    import ballista_b200 as bb
    import oracle_ffi
    from ballista_b200 import driver, tpch

    eng = bb.GpuExecutionEngine(0)
    msf = int(round(args.sf * 1000))
    rows = eng.tpch_table_rows("lineitem", msf)
    threads = bench.usable_cpus()
    oracle_ffi.build()
    o = oracle_ffi.OracleEngine()
    step = -(-rows // threads)
    with ThreadPoolExecutor(threads) as pool:
        list(pool.map(lambda p: o.tpch_generate("lineitem", msf, p, min(rows, p * step), min(rows, (p + 1) * step), tpch.Q1_COLUMNS), range(threads)))
    host = pa.Table.from_batches([o.export_table("lineitem", p) for p in range(threads)])
    eng.set_config("b200.metrics.kernel_timing", "on")
    peak, peak_src = bench.measured_hbm_peak()
    tmp = tempfile.mkdtemp(prefix="b200-parquet-scan-")
    out, results = {}, {}
    try:
        for kind in FILES:
            path = os.path.join(tmp, f"lineitem-{kind}.parquet")
            print(f"{kind}: writing with {args.codec}", file=sys.stderr, flush=True)
            pq.write_table(host, path, **CODECS[args.codec][0], **write_options(kind, host.schema))
            print(f"{kind}: written ({os.path.getsize(path)} bytes), timing register_parquet", file=sys.stderr, flush=True)
            md = pq.ParquetFile(path).metadata
            page_bytes = sum(md.row_group(g).column(c).total_uncompressed_size for g in range(md.num_row_groups) for c in range(md.num_columns))
            desc = bb.engine.parquet_describe(path)
            for _ in range(max(args.warmup, 1)):
                eng.drop_table("lineitem")
                eng.register_parquet("lineitem", 0, path, tpch.Q1_COLUMNS)
            eng.synchronize()
            eng.kernel_stats(reset=True)
            wall = []
            for _ in range(args.steps):
                eng.drop_table("lineitem")
                t0 = time.perf_counter()
                eng.register_parquet("lineitem", 0, path, tpch.Q1_COLUMNS)
                eng.synchronize()
                wall.append(time.perf_counter() - t0)
            ks = eng.kernel_stats(reset=True)
            dec = ks.get("parquet_decode_values", {"ms": 0.0, "bytes": 0})
            dec_ms = dec["ms"] / args.steps
            dec_bytes = page_bytes + dec["bytes"] / args.steps
            dec_gbs = dec_bytes / (dec_ms / 1e3) / 1e9 if dec_ms > 0 else 0.0
            results[kind] = driver.run_stages(eng, tpch.q1(1), f"pq-{kind}")
            eng.remove_job_data(f"pq-{kind}")
            out[kind] = {
                "what": FILES[kind].replace("Snappy", CODECS[args.codec][1]), "file_bytes": os.path.getsize(path), "uncompressed_page_bytes": page_bytes,
                "register_parquet_ms": 1e3 * statistics.median(wall),
                "decode_values_ms": dec_ms, "decode_values_gbs": dec_gbs, "decode_values_frac_of_hbm_peak": dec_gbs / peak,
                "other_kernels_ms": {k: v["ms"] / args.steps for k, v in sorted(ks.items())
                                     if k.startswith("parquet_") and k != "parquet_decode_values" and v["launches"]},
                "pages_per_column": {c["name"]: c["data_pages"] for c in desc["columns"]},
                "encodings": {c["name"]: c["encodings"] for c in desc["columns"]},
            }
            family = CODECS[args.codec][2]
            if family:
                dms = ks.get(family, {"ms": 0.0})["ms"] / args.steps
                out[kind]["decompress_ms"] = dms
                out[kind]["decompress_gbs"] = page_bytes / (dms / 1e3) / 1e9 if dms > 0 else 0.0
            os.remove(path)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    del host
    o.close()
    parity = {"checked": False}
    if not args.no_parity:
        try:
            os.sched_setaffinity(0, bench.START_AFFINITY)
        except Exception:
            pass
        _, want = bench.cpu_q1(msf, 0, rows, threads, steps=1, warmup=0)
        want = pa.Table.from_batches([want])
        bad = [k for k, got in results.items() if not bench.tables_equal(got, want)]
        parity = {"checked": True, "equal": not bad, "mismatch": bad,
                  "what": f"q1 on each scanned table == CPU oracle q1 on the same {rows} generated rows, bit-exact"}
    name, watts = card()
    line = {
        "workload": f"device Parquet scan of TPC-H lineitem's q1 columns, SF{args.sf:g} ({rows} rows), written by pyarrow {pa.__version__}"
                    + ("" if args.codec == "snappy" else " with " + ", ".join(f"{k}={v}" for k, v in CODECS[args.codec][0].items())),
        "steps": args.steps, "warmup": max(args.warmup, 1), "gpu": name, "power_limit_w": watts,
        "timing": "register_parquet: median host wall time (file in the page cache); kernels: CUDA events per kernel family",
        "gbs": "(uncompressed page bytes + decoded Arrow bytes) / parquet_decode_values device time",
        "hbm_peak_gbs": peak, "hbm_peak_source": peak_src, "files": out,
        "parity_checked": bool(parity.get("checked") and parity.get("equal")), "parity": parity,
    }
    print(__import__("json").dumps(line), flush=True)
    eng.close()
    if parity.get("checked") and not parity.get("equal"):
        raise SystemExit(3)


if __name__ == "__main__":
    main()
