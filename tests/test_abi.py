"""The C-ABI shared library loads (no GPU needed) and exports every symbol include/b200exec.h declares."""
import os
import re

import ballista_b200 as bb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    src = open(os.path.join(ROOT, "include", "b200exec.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    L = bb.engine.load_library()
    fns = header_functions()
    assert len(fns) >= 20
    missing = [f for f in fns if not hasattr(L, f)]
    assert not missing, missing


def test_python_binding_lists_the_same_symbols():
    assert sorted(bb.engine.EXPORTED_SYMBOLS) == header_functions()


def test_version_string():
    assert b"sm_90a" in bb.engine.load_library().b200_version()


def test_struct_layouts_match_header():
    import ctypes as C
    assert C.sizeof(bb.engine.ShuffleWritePartition) == 48   # 4*u64 + i64 + 2*i32
    assert C.sizeof(bb.engine.OperatorMetrics) == 48 + 6 * 8


def test_engine_requires_a_gpu_no_cpu_fallback():
    """Without a CUDA device the product must fail loudly instead of computing on the CPU."""
    import torch
    if torch.cuda.is_available():
        return
    try:
        bb.GpuExecutionEngine(0)
    except bb.B200Error as e:
        assert e.code == -4
    else:
        raise AssertionError("engine creation must fail without a GPU")


def test_header_is_plain_c_and_usable_without_python(tmp_path):
    """include/b200exec.h compiles as C99 with -Wall -Werror, and a C program linked against the library decodes a protobuf
    plan, types it and encodes a TaskStatus (host-only entry points: no GPU needed)."""
    import base64
    import ctypes as C
    import json
    import shutil
    import subprocess
    cc = shutil.which("gcc") or shutil.which("cc")
    assert cc, "no C compiler"
    lib_dir = os.path.dirname(bb.engine.LIB_PATH)
    exe = str(tmp_path / "c_consumer")
    subprocess.check_call([cc, "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "native", "c_consumer.c"), "-o", exe, "-L", lib_dir, "-lb200exec", f"-Wl,-rpath,{lib_dir}"])
    with open(os.path.join(ROOT, "tests", "golden", "proto_plans.json")) as fh:
        case = [c for c in json.load(fh)["cases"] if c["name"] == "q3/stage5"][0]
    plan = tmp_path / "plan.pb"
    plan.write_bytes(base64.b64decode(case["proto_b64"]))
    out = subprocess.run([exe, str(plan)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    kv = dict(tok.split("=", 1) for line in out.stdout.splitlines() for tok in line.split() if "=" in tok)
    assert "sm_90a" in out.stdout
    assert int(kv["sizeof_task_result"]) == C.sizeof(bb.engine.TaskResult)
    assert int(kv["sizeof_swp"]) == C.sizeof(bb.engine.ShuffleWritePartition) and int(kv["sizeof_metrics"]) == C.sizeof(bb.engine.OperatorMetrics)
    assert kv["has_job"] == "1" and int(kv["ir_bytes"]) > 100 and int(kv["typed_bytes"]) > 100
    assert kv["malformed_rc"] == "-1" and kv["status_rc"] == "0" and int(kv["status_len"]) > 20
