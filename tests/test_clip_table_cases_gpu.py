"""The PMC reset kernel's prioritized clip table and auto-reset draw at motion-library sizes (3,902 to C_MAX clips) against the
fp64 statement of tests/episode_cases.py, env by env and clip by clip, on the batches of tests/clip_table_cases.py; and the limit
llq_load_mocap puts on the table.

Bars as in tests/test_episode_cases_gpu.py: done, F_TIME, F_CLIP, F_EPISODE_ID, F_OB_ID and the counters exactly equal, F_AVG_REWARD
within 1 ulp and F_SAMPLE_PROB within 8 ulp of the statement, reward, reset rows and observations within KAPPA S + 2^-23 |ref|.  On the
exact table of the reset batches, the draws, F_SAMPLE_PROB and F_AVG_REWARD are exactly equal.

KAPPA = 64.  Largest error / S measured on an H100 80GB HBM3 at a 700 W power limit, one run: observation 2.96, reset observation
2.85, F_KIN_STATE 0.93, reset state and reset F_KIN_STATE 0.60, reward 0.25, reward_sum 0.10 (beyond its fp32 rounding);
F_SAMPLE_PROB at most 4 ulp.

Before the limit, tables above 3,902 clips were accepted by llq_load_mocap and then failed every reset-kernel launch (the table did not
fit in 48 kB of shared memory beside the kernel's static tables)."""
import re

import numpy as np
import pytest

import clip_table_cases as ct
import episode_cases as ec

pytestmark = pytest.mark.gpu


def _lib():
    from lifelike_agility_and_play_b200 import _capi as capi
    return capi.load_cuda_library()


@pytest.mark.parametrize("k", range(len(ct.CASES)))
def test_the_clip_table_matches_the_statement(k, built):
    io = "device2" if ct.CASES[k][0] == 4097 else "host"
    ratios = ec.run_case(_lib(), ct.case(k), io)
    print("case %d (n = %d, C = %d, %s): %s" % (k, ct.CASES[k][0], ct.CASES[k][1], io, ratios))


@pytest.mark.parametrize("C", ct.SIZES)
def test_resets_on_the_exact_table(C, built):
    print("C = %d: %s" % (C, ct.run_resets(_lib(), C)))


def _twins(C):
    """two handles on the same batch, each reset on the same table"""
    ctx, avg, ep, _, _ = ct.reset_batch(C)
    from lifelike_agility_and_play_b200 import _capi as capi
    es = [ec.make(_lib(), ctx, 1) for _ in range(2)]
    for e in es:
        e.set(capi.F_AVG_REWARD, avg); e.set(capi.F_EPISODE_ID, ep); e.reset()
    return ctx, es


def _load(e, C):
    """llq_load_mocap of C short clips on handle e: (return code, message)"""
    import ctypes
    mc, _ = ec.mocap(C, ct.FRAMES)
    frames = np.ascontiguousarray(mc.frames, np.float64)
    offs = np.ascontiguousarray(mc.offsets, np.int32)
    L = e.lib.lib
    rc = L.llq_load_mocap(e._h, frames.ctypes.data_as(ctypes.c_void_p), offs.ctypes.data_as(ctypes.c_void_p), C, float(mc.frame_dt))
    return rc, (L.llq_last_error() or b"").decode()


def test_the_largest_table_loads_and_one_more_clip_is_refused(built):
    """C_MAX + 1 clips are refused, naming C_MAX, before the handle's table is touched: its next steps are bit-identical to a twin
    that never saw the refused load.  The C_MAX batches above load, step and reset."""
    from lifelike_agility_and_play_b200 import _capi as capi
    ctx, (a, b) = _twins(3903)
    try:
        rc, msg = _load(a, ct.C_MAX + 1)
        assert rc == -1, (rc, msg)                      # LLQ_EINVAL
        m = re.search(r"at most (\d+) clips", msg)
        assert m, msg
        c_max = int(m.group(1))
        assert c_max == ct.C_MAX and c_max >= 26000, msg
        rng = np.random.default_rng(5)
        for _ in range(3):
            act = rng.uniform(-1, 1, (ctx["n"], 12)).astype(np.float32)
            oa, ra, da = a.step(act)
            ob, rb, db = b.step(act)
            assert np.array_equal(oa, ob) and np.array_equal(ra, rb) and np.array_equal(da, db)
            for f in (capi.F_STATE, capi.F_CLIP, capi.F_TIME, capi.F_SAMPLE_PROB, capi.F_AVG_REWARD):
                assert np.array_equal(a.get(f), b.get(f)), f
        rc, msg = _load(a, ct.C_MAX)
        assert rc == 0, msg
    finally:
        a.close(); b.close()
