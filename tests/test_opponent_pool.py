"""The opponent pool on the CPU: the statement of its cutoffs and bucketing (tests/opponent_pool_cases.py), the refusals of
llq_hier_policy_create_pool / _set_pool_probs that come before the device, and the resources of the two pool kernels."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import opponent_pool_cases as oc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LLQ_EINVAL = -1


def test_cutoffs_skip_zero_probabilities_and_end_at_2_32():
    t = oc.cutoffs([0.0, 0.25, 0.0, 0.75, 0.0])
    assert t.dtype == np.uint64 and int(t[-1]) == 1 << 32
    assert int(t[0]) == 0 and int(t[1]) == int(t[2]) == 1 << 30 and int(t[3]) == int(t[4]) == 1 << 32
    r = np.array([0, 1, (1 << 30) - 1, 1 << 30, (1 << 32) - 1], np.int64)
    assert oc.pick(r, t).tolist() == [1, 1, 1, 3, 3]                 # models 0, 2 and 4 are never drawn
    rng = np.random.default_rng(0)
    got = oc.pick(rng.integers(0, 1 << 32, 4096), t)
    assert set(got.tolist()) == {1, 3}
    assert oc.pick(np.array([(1 << 32) - 1]), oc.cutoffs([1.0])).tolist() == [0]


def test_cutoffs_use_the_sequential_sum():
    """np.sum adds 16 values pairwise and keeps the tiny ones; the sequential sum (the C entry's) loses each of them against 1."""
    p = np.array([1.0] + [2.0 ** -53] * 15)
    assert np.sum(p) != 1.0
    t = oc.cutoffs(p)
    assert all(int(x) == 1 << 32 for x in t)                          # cum_k / total = 1 for every k: models 1..15 are never drawn
    seq = np.floor(np.cumsum(p) / np.sum(p) * 2.0 ** 32).astype(np.uint64)
    assert int(seq[0]) != int(t[0])


def test_bucketing_pads_orders_and_bounds_the_grid():
    rng = np.random.default_rng(1)
    for n, K in ((1, 1), (45, 6), (300, 64), (1059, 7), (8, 3)):
        model = rng.integers(-1, K + 1, n).astype(np.int32)
        seg_cta, entries = oc.bucket(model, K)
        assert len(entries) == seg_cta[-1] * oc.KROWS and seg_cta[-1] <= (n + 7) // 8 + K
        for k in range(K):
            seg = entries[seg_cta[k] * 8:seg_cta[k + 1] * 8]
            rows = seg[seg >= 0]
            assert len(seg) % 8 == 0 and len(seg) - len(rows) < 8 and (seg[len(rows):] == -1).all()
            assert np.array_equal(rows, np.flatnonzero(model == k))     # ascending, every row of model k
        ctas = oc.cta_rows(model, K)
        assert len(ctas) == (n + 7) // 8 + K
        for k, rows in (c for c in ctas if c is not None):
            assert all(model[r] == k for r in rows if r >= 0)
    # K = 1: CTA b runs rows 8b .. 8b + 7, as llq_hier_policy_forward does
    n = 45
    ctas = oc.cta_rows(np.zeros(n, np.int32), 1)
    for b in range((n + 7) // 8):
        rows = np.arange(8 * b, 8 * b + 8)
        assert np.array_equal(ctas[b][1], np.where(rows < n, rows, -1)) and ctas[b][0] == 0
    assert ctas[-1] is None


def test_assign_draws_only_done_rows_and_records_every_row():
    t = oc.cutoffs([0.5, 0.5, 0.0])
    model = np.array([2, 0, 1, -1, 3, 1], np.int32)
    done = np.array([0, 1, 0, 0, 0, 1], np.uint8)
    m, rec = oc.assign(model, done, t, 3, 100, 7, 9)
    assert m[[0, 2, 3, 4]].tolist() == [2, 1, -1, 3] and set(m[[1, 5]].tolist()) <= {0, 1}
    assert rec.tolist() == [2.0, float(m[1]), 1.0, -1.0, -1.0, float(m[5])]
    m2, rec2 = oc.assign(model, None, t, 3, 100, 7, 9)
    assert np.array_equal(m2, model) and rec2.tolist() == [2.0, 0.0, 1.0, -1.0, -1.0, 1.0]


@pytest.fixture(scope="module")
def lib(built):
    from lifelike_agility_and_play_b200.policy import POLICY_LIB_PATH
    lib = C.CDLL(POLICY_LIB_PATH)
    lib.llq_hier_policy_last_error.restype = C.c_char_p
    return lib


def test_create_pool_and_set_probs_refusals_before_the_device(lib):
    blob, off = np.zeros(64, np.float32), np.zeros(101 * 3, np.int32)
    h = C.c_void_p()

    def create(b, nw, o, k, rows, out=True):
        return lib.llq_hier_policy_create_pool(b, C.c_int64(nw), o, C.c_int32(k), C.c_int32(rows), C.c_int32(0), C.byref(h) if out else None)
    bp, op = blob.ctypes.data_as(C.c_void_p), off.ctypes.data_as(C.c_void_p)
    assert create(None, 64, op, 3, 16) == LLQ_EINVAL
    assert create(bp, 64, None, 3, 16) == LLQ_EINVAL
    assert create(bp, 64, op, 3, 16, out=False) == LLQ_EINVAL
    for k in (0, -1, 65):
        assert create(bp, 64, op, k, 16) == LLQ_EINVAL and b"n_models" in lib.llq_hier_policy_last_error()
    for rows in (0, -8):
        assert create(bp, 64, op, 3, rows) == LLQ_EINVAL and b"max_rows" in lib.llq_hier_policy_last_error()
    for bad in (64, -1):
        o = off.copy()
        o[101 * 2 + 50] = bad                                          # model 2's role 50
        assert create(bp, 64, o.ctypes.data_as(C.c_void_p), 3, 16) == LLQ_EINVAL and b"outside" in lib.llq_hier_policy_last_error()
    p = np.ones(3)
    assert lib.llq_hier_policy_set_pool_probs(None, p.ctypes.data_as(C.c_void_p), C.c_int32(3)) == LLQ_EINVAL


def test_pool_kernels_fit_two_ctas_per_sm():
    """hier_pool_kernel and hier_pool_assign_kernel: at most 128 registers and no spills; the pool forward's shared memory is dynamic
    (Smem plus its 8 row ids), so two of its CTAs still fit on an SM."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "lifelike_agility_and_play_b200", "csrc", "llq_policy_hier.cu")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c", "-o", os.devnull, src],
                         capture_output=True, text=True, check=True).stderr
    found = {}
    for block in out.split("Compiling entry function")[1:]:
        m = re.search(r"(hier_pool_kernel|hier_pool_assign_kernel)E", block)
        if not m:
            continue
        regs = int(re.search(r"Used (\d+) registers", block).group(1))
        spills = [int(x) for x in re.findall(r"(\d+) bytes spill (?:stores|loads)", block)]
        smem = re.search(r"(\d+) bytes smem", block)
        found[m.group(1)] = (regs, spills, int(smem.group(1)) if smem else 0)
    assert sorted(found) == ["hier_pool_assign_kernel", "hier_pool_kernel"], out
    for name, (regs, spills, smem) in found.items():
        assert regs <= 128 and spills == [0, 0], (name, regs, spills)
    assert found["hier_pool_kernel"][2] == 0
    assert 2 * (103424 + 32 + 1024) <= 228 * 1024
