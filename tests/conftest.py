import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def _have_cuda():
    try:
        import ctypes
        lib = ctypes.CDLL("libcuda.so.1")
        n = ctypes.c_int(0)
        return lib.cuInit(0) == 0 and lib.cuDeviceGetCount(ctypes.byref(n)) == 0 and n.value > 0
    except Exception:
        return False


HAVE_CUDA = _have_cuda()


def pytest_collection_modifyitems(config, items):
    if HAVE_CUDA:
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def built():
    import __graft_entry__ as g
    g.build()
    return True


@pytest.fixture(scope="session")
def model():
    from lifelike_agility_and_play_b200.model.compile_model import load_model
    return load_model()


@pytest.fixture(scope="session")
def blob(model):
    from lifelike_agility_and_play_b200.model.compile_model import pack_model
    return pack_model(model)


@pytest.fixture(scope="session")
def small_mocap():
    from lifelike_agility_and_play_b200.mocap import synthetic_mocap
    return synthetic_mocap(6, seed=3, min_frames=380, max_frames=700)


@pytest.fixture(scope="session")
def oracle_lib(built):
    from oracle import oracle
    return oracle.load()


@pytest.fixture()
def make_oracle(oracle_lib, blob, small_mocap):
    from lifelike_agility_and_play_b200._capi import VecEngine
    made = []

    def _make(n, mocap=None, blob_=None, **cfg):
        e = VecEngine(oracle_lib, n, blob if blob_ is None else blob_, small_mocap if mocap is None else mocap, **cfg)
        made.append(e)
        return e
    yield _make
    for e in made:
        e.close()


@pytest.fixture()
def make_cuda(built, blob, small_mocap):
    from lifelike_agility_and_play_b200 import _capi as capi
    made = []

    def _make(n, mocap=None, blob_=None, **cfg):
        e = capi.VecEngine(capi.load_cuda_library(), n, blob if blob_ is None else blob_,
                           small_mocap if mocap is None else mocap, **cfg)
        made.append(e)
        return e
    yield _make
    for e in made:
        e.close()
