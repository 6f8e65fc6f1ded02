"""Model refresh without a GPU: the three C-ABI entries refuse null handles and arguments before touching a device, the Python wrappers
refuse wrong array counts, shapes, levels and sources with ValueError before calling the library, the pool-region statement
(policy_epmc.pool_regions, mirrored by llq_hier_policy_set_pool_model) on designed offset tables, and the pack kernel's registers."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from lifelike_agility_and_play_b200 import policy
from lifelike_agility_and_play_b200.policy_epmc import (EPMC_SHAPES, SEPMC_SHAPES, DeviceHierPolicy, DeviceOpponentPool, DeviceSepmcTrainPolicy,
                                                        pool_regions, random_weights, weight_blob)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LLQ_EINVAL = -1
RV = 101


@pytest.fixture(scope="module")
def lib(built):
    lib = C.CDLL(policy.POLICY_LIB_PATH)
    lib.llq_policy_last_error.restype = C.c_char_p
    lib.llq_hier_policy_last_error.restype = C.c_char_p
    return lib


def test_refresh_entries_are_exported(lib):
    for name in ("llq_policy_set_weights", "llq_hier_policy_set_weights", "llq_hier_policy_set_pool_model"):
        assert name in policy.POLICY_EXPORTS and hasattr(lib, name)


def test_entries_refuse_null_handles_and_arguments(lib):
    blob = np.zeros(policy.N_WEIGHTS, np.float32)
    bp, n = blob.ctypes.data_as(C.c_void_p), C.c_int64(blob.size)
    for on_device in (0, 1):
        assert lib.llq_policy_set_weights(None, bp, n, C.c_int32(on_device), None) == LLQ_EINVAL
        assert lib.llq_hier_policy_set_weights(None, bp, n, C.c_int32(on_device), None) == LLQ_EINVAL
        assert lib.llq_hier_policy_set_pool_model(None, C.c_int32(0), bp, n, C.c_int32(on_device), None) == LLQ_EINVAL
    assert b"null" in lib.llq_hier_policy_last_error() and b"null" in lib.llq_policy_last_error()


def _detached(cls, **attrs):
    """A wrapper object with no library handle: the Python checks run, the library is never reached (it is None)."""
    obj = cls.__new__(cls)
    obj.__dict__.update(dict(_h=None, lib=None, _lib=None, device=0), **attrs)
    return obj


def test_pmc_wrapper_refuses_wrong_arrays_and_sources():
    from test_policy import random_weights as pmc_weights
    pol = _detached(policy.DevicePolicy)
    w = pmc_weights(0)
    assert [a.shape for a in w] == [tuple(s) for s in policy.PMC_SHAPES]
    for bad in (w[:27], w + [w[0]], random_weights(False, 0), np.zeros(policy.N_WEIGHTS, np.float32)):
        with pytest.raises(ValueError, match="arrays"):
            pol.set_weights(bad)
    w2 = list(w)
    w2[10] = np.zeros((206, 256), np.float32)
    with pytest.raises(ValueError, match="array 10"):
        pol.set_weights(w2)
    for t in (torch.zeros(policy.N_WEIGHTS), torch.zeros(policy.N_WEIGHTS, dtype=torch.float64)):
        with pytest.raises(ValueError, match="CUDA"):
            pol.set_weights(t)


@pytest.mark.parametrize("cls", [DeviceHierPolicy, DeviceSepmcTrainPolicy])
def test_hierarchical_wrappers_refuse_wrong_level_count_and_shapes(cls):
    for strategic in ((False, True) if cls is DeviceHierPolicy else (True,)):
        shapes, other = (SEPMC_SHAPES, EPMC_SHAPES) if strategic else (EPMC_SHAPES, SEPMC_SHAPES)
        w = random_weights(strategic, 1)
        h = _detached(cls, strategic=strategic, n_weights=weight_blob(w)[0].size)
        with pytest.raises(ValueError, match="expected the %d arrays" % len(shapes)):
            h.set_weights(random_weights(not strategic, 1))                     # the other level
        with pytest.raises(ValueError, match="expected the %d arrays" % len(shapes)):
            h.set_weights(w[:-1])
        w2 = list(w)
        w2[60] = np.zeros((3, 3), np.float32)
        with pytest.raises(ValueError, match="array 60"):
            h.set_weights(w2)
        with pytest.raises(ValueError, match="CUDA"):
            h.set_weights(torch.from_numpy(weight_blob(w)[0]))
        assert len(other) != len(shapes)


def test_pool_wrapper_refuses_bad_slots_and_set_weights():
    models = [random_weights(True, k) for k in range(3)]
    blob, starts = weight_blob(models[0])
    pool = _detached(DeviceOpponentPool, strategic=True, n_models=3, n_weights=3 * blob.size,
                     regions=[(k * blob.size, (k + 1) * blob.size) for k in range(3)])
    for k in (-1, 3):
        with pytest.raises(ValueError, match="outside"):
            pool.set_model(k, models[0])
    with pytest.raises(ValueError, match="set_model"):
        pool.set_weights(models[0])
    with pytest.raises(ValueError, match="expected the 152 arrays"):
        pool.set_model(1, random_weights(False, 0))
    pool.regions = None
    with pytest.raises(ValueError, match="share arrays"):
        pool.set_model(1, models[0])


def _table(starts_per_model, size):
    """A pool's [K * 101] role table where model k's roles start at starts_per_model[k] + r * size."""
    return np.concatenate([s + size * np.arange(RV) for s in starts_per_model]).astype(np.int32)


def test_pool_regions_on_designed_tables():
    size, gap = 10, 4
    m = RV * size + gap                                                    # a model's region: its arrays plus an unlisted tail
    # contiguous, in order: region k = [k m, (k + 1) m), the last up to the end of the blob
    assert pool_regions(_table([0, m, 2 * m], size), 3, 3 * m) == [(0, m), (m, 2 * m), (2 * m, 3 * m)]
    assert pool_regions(_table([0], size), 1, m + 7) == [(0, m + 7)]
    # unordered: models stored in the blob in the order 2, 0, 1, with a prefix before the first
    assert pool_regions(_table([5 + m, 5 + 2 * m, 5], size), 3, 5 + 3 * m) == [(5 + m, 5 + 2 * m), (5 + 2 * m, 5 + 3 * m), (5, 5 + m)]
    # the smallest role offset is not role 0's
    off = _table([0, m], size)
    off[0], off[1] = off[1], off[0]
    assert pool_regions(off, 2, 2 * m) == [(0, m), (m, 2 * m)]
    # shared: model 1's role 7 is model 0's array -> model 1 starts inside model 0, whose arrays then leave its region
    off = _table([0, m], size)
    off[RV + 7] = 7 * size
    assert pool_regions(off, 2, 2 * m) is None
    # shared: two models on the same arrays (the same start)
    assert pool_regions(_table([0, 0], size), 2, m) is None
    # shared: model 0's last role points into model 1's arrays
    off = _table([0, m], size)
    off[RV - 1] = m + 3 * size
    assert pool_regions(off, 2, 2 * m) is None


def test_pack_kernel_registers_and_no_spills():
    """pmc_pack_kernel: no spills, few registers (a grid-stride copy)."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "lifelike_agility_and_play_b200", "csrc", "llq_policy.cu")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c", "-o", os.devnull, src],
                         capture_output=True, text=True, check=True).stderr
    blocks = [b for b in out.split("Compiling entry function")[1:] if "pmc_pack_kernel" in b.split("\n")[0]]
    assert len(blocks) == 1, out
    regs = int(re.search(r"Used (\d+) registers", blocks[0]).group(1))
    spills = [int(x) for x in re.findall(r"(\d+) bytes spill (?:stores|loads)", blocks[0])]
    assert regs <= 64 and spills == [0, 0], (regs, spills)
