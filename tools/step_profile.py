"""Device timeline of warm q1 steps (SF10 lineitem resident in HBM, the step of bench.py) under torch.profiler.

Writes OUT_DIR/step_profile.pt.trace.json (Chrome trace) and prints, per step: every kernel, copy and memset on the
engine stream with its duration and the idle gap before it, the CUDA runtime calls that block the host
(cudaStreamSynchronize / cudaEventSynchronize / synchronous cudaMemcpy) and the engine's launch and host-wait counters.
Usage: python tools/step_profile.py [OUT_DIR] [steps] [msf]"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import ballista_b200 as bb  # noqa: E402
from ballista_b200 import tpch  # noqa: E402

out_dir = sys.argv[1] if len(sys.argv) > 1 else "."
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
msf = int(sys.argv[3]) if len(sys.argv) > 3 else 10000
os.makedirs(out_dir, exist_ok=True)

dev = torch.device("cuda", 0)
torch.cuda.set_device(dev)
eng = bb.GpuExecutionEngine(0)
stream = torch.cuda.Stream(device=dev)
eng.set_stream(stream.cuda_stream)
n = eng.tpch_table_rows("lineitem", msf)
eng.tpch_generate("lineitem", msf, 0, 0, n, tpch.Q1_COLUMNS)
stages = tpch.q1(1)


def counters():
    c = {"kernel_launches": eng.kernel_launches()}
    try:
        c["host_syncs"] = eng.counter("host_syncs")
    except Exception:
        pass
    return c


def step(job):
    for st in stages:
        q = eng.create_query_stage_exec(job, st.stage_id, st.json(job))
        q.execute_query_stage(0)
        q.release()
    res = eng.partition_export(job, 3, 0)
    eng.remove_job_data(job)
    return res


for w in range(5):
    step(f"warm#{w}")
torch.cuda.synchronize(dev)

c0 = counters()
marks = []
acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
with torch.profiler.profile(activities=acts) as prof:
    for k in range(steps):
        with torch.profiler.record_function(f"step#{k}"):
            t0 = time.perf_counter()
            step(f"step#{k}")
            marks.append((time.perf_counter() - t0) * 1e3)
torch.cuda.synchronize(dev)
c1 = counters()
trace_path = os.path.join(out_dir, "step_profile.pt.trace.json")
prof.export_chrome_trace(trace_path)

with open(trace_path) as f:
    ev = json.load(f)["traceEvents"]
dev_ev = sorted((e for e in ev if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")), key=lambda e: e["ts"])
step_ev = sorted((e for e in ev if e.get("ph") == "X" and e.get("cat") == "user_annotation" and str(e.get("name", "")).startswith("step#")),
                 key=lambda e: e["ts"])
blocking = ("cudaStreamSynchronize", "cudaEventSynchronize", "cudaDeviceSynchronize", "cudaMemcpy")
rt_ev = [e for e in ev if e.get("ph") == "X" and e.get("cat") == "cuda_runtime"]

print(f"device: {torch.cuda.get_device_name(dev)}")
print(f"per step: kernel launches {(c1['kernel_launches'] - c0['kernel_launches']) / steps:.1f}" +
      (f", host waits {(c1['host_syncs'] - c0['host_syncs']) / steps:.1f}" if "host_syncs" in c1 else ""))
print("host wall ms per step (profiled): " + ", ".join(f"{m:.3f}" for m in marks))
for si, se in enumerate(step_ev):
    a, b = se["ts"], se["ts"] + se["dur"]
    # device work is attributed to the step whose host span launched it: take events that start inside [a, next step)
    nb = step_ev[si + 1]["ts"] if si + 1 < len(step_ev) else float("inf")
    ds = [e for e in dev_ev if a <= e["ts"] < nb]
    rs = [e for e in rt_ev if a <= e["ts"] < b]
    busy = sum(e["dur"] for e in ds)
    span = (ds[-1]["ts"] + ds[-1]["dur"] - ds[0]["ts"]) if ds else 0.0
    waits = [e for e in rs if e["name"] in blocking]
    launches = [e for e in rs if e["name"] in ("cudaLaunchKernel", "cudaLaunchKernelExC", "cuLaunchKernel", "cuLaunchKernelEx")]
    print(f"== step {si}: host {se['dur'] / 1e3:.3f} ms, device span {span / 1e3:.3f} ms, device busy {busy / 1e3:.3f} ms, "
          f"{len(ds)} device ops ({sum(1 for e in ds if e['cat'] == 'kernel')} kernels), {len(launches)} launch calls, "
          f"{len(waits)} blocking calls ({sum(e['dur'] for e in waits) / 1e3:.3f} ms)")
    rt_names = {}
    for e in rs:
        s = rt_names.setdefault(e["name"], [0, 0.0])
        s[0] += 1
        s[1] += e["dur"]
    print("   runtime calls: " + ", ".join(f"{k} x{v[0]} {v[1] / 1e3:.3f}ms" for k, v in sorted(rt_names.items(), key=lambda kv: -kv[1][1])))
    prev_end = None
    for e in ds:
        gap = (e["ts"] - prev_end) if prev_end is not None else 0.0
        print(f"   +{(e['ts'] - ds[0]['ts']) / 1e3:8.3f} ms gap {gap:7.1f} us  {e['dur']:8.1f} us  {e['cat']:10s} {e['name'][:110]}")
        prev_end = max(prev_end or 0.0, e["ts"] + e["dur"])
eng.close()
