import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def oracle_lib():
    import oracle_ffi
    oracle_ffi.build()
    return oracle_ffi


@pytest.fixture()
def oracle(oracle_lib):
    e = oracle_lib.OracleEngine()
    yield e
    e.close()


@pytest.fixture(scope="session")
def gpu_engine_session():
    import ballista_b200 as bb
    try:
        e = bb.GpuExecutionEngine(0)
    except bb.engine.B200Error as ex:
        # no CUDA device here: the engine has no CPU path, so the gpu-marked tests cannot run at all
        pytest.skip(f"no usable CUDA device: {ex}")
    yield e
    e.close()


@pytest.fixture()
def gpu(gpu_engine_session):
    # the engine remembers, per plan shape, which aggregate strategy the data needed last time; tests that assert which
    # kernel ran must not depend on what an earlier test fed the same plan
    gpu_engine_session.set_config("b200.agg.reset_hints", "1")
    return gpu_engine_session
