"""The fp64 statement of the EPMC corridor generator (tests/corridor_cases.py) against the reference's terrain goldens and the CPU
oracle, bit for bit, and the reach of its designed categories."""
import numpy as np
import pytest

import corridor_cases as cc
from lifelike_agility_and_play_b200 import _capi as capi
from test_golden_epmc import terrain_gold

# (element, ranges) of the designed batches
BATCHES = [(e, r) for e in (1, 2, 3) for r in cc.RANGES]


@pytest.mark.parametrize("element", [1, 2, 3])
def test_statement_reproduces_the_reference_goldens(element):
    """tests/golden/gen_golden_epmc_terrain_from_reference.py keys episode k of its single env with (seed, 0, k) on the shipped
    ranges; the reference's box rows are its double centres and half extents"""
    g = terrain_gold(element)
    eps = np.arange(len(g["nbox"]), dtype=np.int64)
    ref = cc.statement(element, cc.RANGES["shipped"], int(g["seed"]), np.zeros(len(eps), np.int64), eps)
    assert np.array_equal(ref["nbox"], g["nbox"])
    for k, nb in enumerate(g["nbox"]):
        rows, tgx = cc.corridor(element, cc.RANGES["shipped"], cc.draws(int(g["seed"]), 0, k)[0])
        assert np.array_equal(rows, g["boxes"][k][:nb]), (k, np.argwhere(rows != g["boxes"][k][:nb])[:6])
        assert np.array_equal(ref["boxes"][k], g["boxes"][k].astype(np.float32))
        assert tgx == g["reset_aux"][k][capi.AUX_TARGET_X] and g["reset_aux"][k][capi.AUX_TARGET_Y] == 0.0
        assert ref["aux"][capi.AUX_TARGET_X][k] == tgx


def run_reset(lib, element, ranges, n, gid0, ep, blob):
    """(boxes [n, MAX_BOXES, 6], nbox, aux) after a reset of every env of a fresh handle with episode ids ep"""
    e = capi.VecEngine(lib, n, blob, None, **cc.engine_config(element, ranges, gid0))
    try:
        e.set_init_state(terrain_gold(element)["init_state"])
        e.reset()
        e.set(capi.F_EPISODE_ID, ep)
        e.reset(np.ones(n, bool))
        return e.get(capi.F_BOXES).reshape(n, capi.MAX_BOXES, 6), e.get(capi.F_NBOX), e.get(capi.F_AUX)
    finally:
        e.close()


def check(got, ref, what):
    boxes, nbox, aux = got
    bad = np.flatnonzero(nbox != ref["nbox"])
    assert not len(bad), (what, "nbox", bad[:8])
    diff = np.argwhere(boxes != ref["boxes"])
    assert not len(diff), (what, "boxes", len(diff), [(tuple(int(x) for x in d), boxes[tuple(d)], ref["boxes"][tuple(d)]) for d in diff[:6]])
    for s, v in ref["aux"].items():
        bad = np.flatnonzero(aux[:, s] != v)
        assert not len(bad), (what, "aux", s, [(int(i), aux[i, s], v[i]) for i in bad[:6]])


@pytest.mark.parametrize("element,ranges", BATCHES)
@pytest.mark.parametrize("gid0", cc.GID0)
def test_oracle_matches_the_statement(element, ranges, gid0, oracle_lib, blob):
    """F_BOXES (zero past nbox on the oracle), F_NBOX and the corridor's aux slots exactly; episode ids e and e + 2^32 alike"""
    n = 17
    ep, cats = cc.keys(element, ranges, n, gid0)
    gid = gid0 + np.arange(n)
    ref = cc.statement(element, cc.RANGES[ranges], cc.SEED, gid, ep)
    check(run_reset(oracle_lib, element, ranges, n, gid0, ep, blob), ref, "oracle")
    flip = np.where(ep >= 2 ** 32, ep - 2 ** 32, ep + 2 ** 32)
    check(run_reset(oracle_lib, element, ranges, n, gid0, flip, blob), ref, "oracle, ids shifted by 2^32")


@pytest.mark.parametrize("element,ranges", BATCHES)
def test_every_category_is_reached(element, ranges):
    reached = set()
    for gid0 in cc.GID0:
        for n in (1, 17):
            ep, cats = cc.keys(element, ranges, n, gid0)
            gid = gid0 + np.arange(n)
            ok = cc.reaches(element, ranges, gid, ep, cats)
            assert ok.all(), [(int(i), cats[i]) for i in np.flatnonzero(~ok)]
            assert (ep >= 2 ** 32).any() and (ep < 2 ** 32).any() or n == 1
            reached |= set(cats)
            ref = cc.statement(element, cc.RANGES[ranges], cc.SEED, gid, ep)
            nb = {c: int(ref["nbox"][i]) for i, c in enumerate(cats)}
            assert nb["count_1"] == (4 if element < 3 else 10) and (n == 1 or nb["count_max"] == (20 if element < 3 else 34))
    want = set(cc.cats_of(element, ranges))
    assert want <= reached
    # the fp32-rounded bounds move a box value on every batch but element 1 and 3 with lo == hi (0.3 and 2.5 round to fp32
    # numbers whose walls round alike)
    assert ("f32_bound" in want) == (ranges != "equal" or element == 2)


def test_fp32_bounds_reach_the_box_values():
    """the default hole gap [0.25, 0.3]: the share of bar centres (z = 0.15 + g) that the fp32-rounded bounds move, on 2^14 keys"""
    U = cc.draws(cc.SEED, np.zeros(2 ** 14, np.int64), np.arange(2 ** 14, dtype=np.int64))
    g_d = 0.25 + U[:, 4] * (0.3 - 0.25)
    g_f = cc.f32(0.25) + U[:, 4] * (cc.f32(0.3) - cc.f32(0.25))
    share = np.mean(np.float32(0.15 + g_d) != np.float32(0.15 + g_f))
    assert 0.1 < share < 0.3, share


def test_dfma_and_unfused_draws_round_alike_in_fp32():
    """no key separates the kernel's contracted lo + u (hi - lo) from the statement's unfused form in fp32 (see corridor_cases)"""
    for lo, hi in ((0.02, 0.5), (0.05, 0.15), (0.25, 0.3), (0.1, 1.3), (0.1, 0.3)):
        assert cc.fma_search(lo, hi, count=2 ** 12) == 0, (lo, hi)
