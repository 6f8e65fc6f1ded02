"""The EPMC corridor generator of the reset kernel against the fp64 statement of tests/corridor_cases.py, env by env, on both reset
paths: a masked `llq_reset` of designed keys set through F_EPISODE_ID, and the auto-reset inside `llq_step` after designed
time-outs.

Exactly equal: F_NBOX, every box row below nbox, and the aux slots TARGET_X, TARGET_Y, INIT_POS_DIFF_LEN and LAST_POS_DIFF_LEN (the
kernel writes the target's double and its fabs, so no rounding is left to allow for).  The reset observation's target block is within
the EPMC pin's bar (tests/epmc_episode_cases.py: KAPPA S + 2^-23 |ref|).  Envs outside the mask, or not ended by the step, keep their
corridor and aux row.  Rows at or past nbox are stale and not read: a handle that built a 34-box corridor before its 10-box one
steps bit for bit like a twin that saw only the 10-box one."""
import numpy as np
import pytest

import corridor_cases as cc
import epmc_episode_cases as xc
from lifelike_agility_and_play_b200 import _capi as capi
from test_golden_epmc import terrain_gold

pytestmark = pytest.mark.gpu

SIZES = (1, 15, 16, 17, 33, 4097, 8192)          # 8192: the bench's batch; the others end the reset kernel in a partial block


def make(element, ranges, n, gid0, blob, **over):
    e = capi.VecEngine(capi.load_cuda_library(), n, blob, None, **cc.engine_config(element, ranges, gid0, **over))
    e.set_init_state(terrain_gold(element)["init_state"])
    e.reset()
    return e


def read(e):
    return (e.get(capi.F_BOXES).reshape(e.n, capi.MAX_BOXES, 6), e.get(capi.F_NBOX), e.get(capi.F_AUX), e.get(capi.F_STATE),
            e.get(capi.F_EPISODE_ID))


def check_rows(rows, got, ref, obs, what):
    boxes, nbox, aux, st, _ = got
    bad = np.flatnonzero(nbox[rows] != ref["nbox"])
    assert not len(bad), (what, "nbox", [(int(rows[i]), int(nbox[rows[i]]), int(ref["nbox"][i])) for i in bad[:6]])
    live = np.arange(capi.MAX_BOXES)[None, :] < ref["nbox"][:, None]
    diff = np.argwhere((boxes[rows] != ref["boxes"]).any(2) & live)
    assert not len(diff), (what, "box rows differ", len(diff), int((boxes[rows] != ref["boxes"])[live].sum()),
                           [(int(rows[i]), int(j), boxes[rows[i], j], ref["boxes"][i, j]) for i, j in diff[:4]])
    for s, v in ref["aux"].items():
        bad = np.flatnonzero(aux[rows, s] != v)
        assert not len(bad), (what, "aux", s, [(int(rows[i]), aux[rows[i], s], v[i]) for i in bad[:6]])
    # the target block of the reset observation: R^-1 (target - pos) normalised in xy, target_spd
    a = aux[rows]
    s64 = st[rows].astype(np.float64)
    ref_t, S = xc._sens(lambda em: dict(tail=(lambda t: em.add(t, np.abs(t)))(
        xc.target_block(s64, a[:, capi.AUX_TARGET_X], a[:, capi.AUX_TARGET_Y], a[:, capi.AUX_TARGET_SPD], em))), ("tail",))
    xc.ec._ratio(obs[rows, 913:916], ref_t["tail"], S["tail"], xc.KAPPA, what + " target block")


def check_kept(rows, got, before, what):
    for k, name in enumerate(("F_BOXES", "F_NBOX", "F_AUX", "F_STATE", "F_EPISODE_ID")):
        assert np.array_equal(got[k][rows], before[k][rows]), (what, name)


@pytest.mark.parametrize("ranges", list(cc.RANGES))
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("element", [1, 2, 3])
def test_masked_reset_matches_the_statement(element, n, ranges, built, blob):
    gid0 = cc.GID0[n % 2]
    ep, cats = cc.keys(element, ranges, n, gid0)
    e = make(element, ranges, n, gid0, blob)
    try:
        e.set(capi.F_EPISODE_ID, ep)
        before = read(e)
        mask = np.ones(n, bool)
        mask[len(cc.CATS) + 1::7] = False          # the designed envs reset; some of the others keep their row
        obs = e.reset(mask)
        got = read(e)
        rows = np.flatnonzero(mask)
        ref = cc.statement(element, cc.RANGES[ranges], cc.SEED, gid0 + rows, ep[rows])
        check_rows(rows, got, ref, obs, "masked reset")
        assert np.array_equal(got[4][rows], ep[rows] + 1)
        check_kept(np.flatnonzero(~mask), got, before, "masked reset")
    finally:
        e.close()


@pytest.mark.parametrize("ranges", list(cc.RANGES))
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("element", [1, 2, 3])
def test_auto_reset_matches_the_statement(element, n, ranges, built, blob):
    """max_steps 2: envs whose counter is 1 time out in the step and reset with the episode id they stepped with"""
    gid0 = cc.GID0[(n + 1) % 2]
    ep, cats = cc.keys(element, ranges, n, gid0)
    e = make(element, ranges, n, gid0, blob, auto_reset=1, max_steps=2)
    try:
        e.set(capi.F_EPISODE_ID, ep)
        timeout = np.ones(n, bool)
        timeout[len(cc.CATS) + 2::5] = False
        aux = e.get(capi.F_AUX)
        aux[:, capi.AUX_COUNTER] = timeout
        e.set(capi.F_AUX, aux)
        before = read(e)
        obs, _, done = e.step(np.zeros((n, 12), np.float32))
        done = done.astype(bool)
        assert done[timeout].all()
        got = read(e)
        rows = np.flatnonzero(done)
        ref = cc.statement(element, cc.RANGES[ranges], cc.SEED, gid0 + rows, ep[rows])
        check_rows(rows, got, ref, obs, "auto-reset")
        assert np.array_equal(got[4][rows], ep[rows] + 1)
        kept = np.flatnonzero(~done)
        for k in (0, 1, 4):
            assert np.array_equal(got[k][kept], before[k][kept])
    finally:
        e.close()


def _keys_with(element, gid, count, seed):
    """per global id, an episode id whose corridor has `count` objects"""
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 2 ** 40)
    cand = base + np.arange(64, dtype=np.int64)
    U = cc.draws(cc.SEED, np.repeat(gid, 64), np.tile(cand, len(gid)), 4)[:, 2].reshape(len(gid), 64)
    hit = cc.count_of(element, U) == count
    assert hit.any(1).all()
    return cand[np.argmax(hit, 1)]


@pytest.mark.parametrize("n", [33, 8192])
def test_stale_rows_past_nbox_are_not_read(n, built, blob):
    """handle A builds a 34-box cube corridor, then a 10-box one; twin B sees only the 10-box reset (same keys, same aux)"""
    gid0 = cc.GID0[1]
    gid = gid0 + np.arange(n)
    big, small = _keys_with(3, gid, 4, 1), _keys_with(3, gid, 1, 2)
    A, B = make(3, "shipped", n, gid0, blob, auto_reset=1), make(3, "shipped", n, gid0, blob, auto_reset=1)
    try:
        A.set(capi.F_EPISODE_ID, big)
        A.reset(np.ones(n, bool))
        assert (A.get(capi.F_NBOX) == 34).all()
        aux = B.get(capi.F_AUX)
        for e in (A, B):
            e.set(capi.F_AUX, aux)
            e.set(capi.F_EPISODE_ID, small)
        oA, oB = A.reset(np.ones(n, bool)), B.reset(np.ones(n, bool))
        bA, bB = (e.get(capi.F_BOXES).reshape(n, capi.MAX_BOXES, 6) for e in (A, B))
        assert (A.get(capi.F_NBOX) == 10).all() and (B.get(capi.F_NBOX) == 10).all()
        # F_BOXES reads rows past nbox as zero; on the device A's rows 10-33 still hold the cube sets of its 34-box corridor
        assert np.array_equal(bA, bB)
        assert np.array_equal(oA, oB)
        c0A, c0B = A.counters(), B.counters()
        rng = np.random.default_rng(n)
        for t in range(20):
            act = (0.3 * rng.standard_normal((n, 12))).astype(np.float32)
            (oA, rA, dA), (oB, rB, dB) = A.step(act), B.step(act)
            assert np.array_equal(oA, oB) and np.array_equal(rA, rB) and np.array_equal(dA, dB), t
        for f in (capi.F_STATE, capi.F_AUX, capi.F_NBOX, capi.F_EPISODE_ID, capi.F_WARMSTART, capi.F_FOOT_POS):
            assert np.array_equal(A.get(f), B.get(f), equal_nan=True), f
        assert np.array_equal(A.counters() - c0A, B.counters() - c0B)
    finally:
        A.close(); B.close()
