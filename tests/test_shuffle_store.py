"""CPU: the shuffle store (csrc/host/shuffle_store.hpp) keeps Ballista's executor-side shuffle rules -- task retry, piece
order, empty partitions, failed-task cleanup, stage / job removal, the partition count, one executor's snapshot and the
hand-over of exchanged partitions (tests/native/shuffle_store_check.cpp).  Built with plain g++: the store makes no CUDA
calls, so only the CUDA headers are needed."""
import os
import shutil
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cuda_include():
    nvcc = shutil.which("nvcc")
    home = os.path.dirname(os.path.dirname(nvcc)) if nvcc else os.environ.get("CUDA_HOME", "/usr/local/cuda")
    return os.path.join(home, "include")


def test_shuffle_store_rules(tmp_path):
    exe = str(tmp_path / "shuffle_store_check")
    subprocess.run(["g++", "-O2", "-std=c++17", "-I" + _cuda_include(),
                    os.path.join(ROOT, "tests", "native", "shuffle_store_check.cpp"), "-o", exe], check=True)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60).stdout
    assert "fails=0" in out, out
