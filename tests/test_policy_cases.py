"""The fp64 policy statements and the designed batches of tests/policy_cases.py, on the CPU: Philox against the Random123 known
answers, the statements against the fp32 numpy classes of the package, and every designed category reached with every row decisive."""
import numpy as np
import pytest

import policy_cases as pc
from lifelike_agility_and_play_b200.policy import PmcPolicy
from lifelike_agility_and_play_b200.policy_epmc import EpmcPolicy, SepmcPolicy, random_weights as hier_random_weights


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_matches_the_known_answers(ctr, key, want):
    assert tuple(int(x) for x in pc.philox4x32(*ctr, *key)) == want


def test_box_muller_uniforms_use_the_kernels_fp32_operations():
    """A draw of r.x >= 2^32 - 128 rounds to 1.0f and is clamped to 0.99999994f: eps stays finite and small, as on the device."""
    rows = np.arange(20000)
    eps = pc.pmc_eps(rows, 2 ** 40 + 3, 2 ** 32 + 7)
    assert np.isfinite(eps).all() and abs(eps.mean()) < 0.02 and abs(eps.std() - 1.0) < 0.02
    u = (np.float32(np.float32(2 ** 32 - 100) + np.float32(0.5)) * np.float32(2.0 ** -32))
    assert u == np.float32(1.0) and np.minimum(u, np.float32(0.99999994)) < 1.0


def _agree(got, ref, S, name, factor=64.0):
    err = np.abs(np.asarray(got, np.float64) - ref)
    bar = factor * S + 1e-6 * np.abs(ref) + 1e-7
    assert (err <= bar).all(), (name, float((err / bar).max()))


def test_pmc_statement_agrees_with_the_fp32_class():
    rng = np.random.default_rng(4)
    w = pc.pmc_random_weights(9)
    obs = (2.0 * rng.standard_normal((256, 207))).astype(np.float32)
    ref, S = pc.pmc_eval(w, obs)
    host = PmcPolicy(w)
    a, code = host.act(obs, return_code=True)
    dec = ref["gap"] > 4 * pc.KAPPA_PMC * S["gap"]
    assert dec.mean() > 0.9
    assert np.array_equal(code[dec], ref["code"][dec])
    _agree(a[dec], ref["mean"][dec], S["mean"][dec], "mean")
    _agree(host.value(obs), ref["value"], S["value"], "value")


@pytest.mark.parametrize("strategic", [False, True])
def test_hierarchical_statement_agrees_with_the_fp32_class(strategic):
    rng = np.random.default_rng(6)
    w = hier_random_weights(strategic, 2)
    n, ow, ssz = 96, (965 if strategic else 916), (128 if strategic else 64)
    obs = np.stack([pc._hier_row(rng, "random", ow) for _ in range(n)])
    state = pc.hier_random_state(rng, n, ssz)
    done = pc.DONE_BYTES[np.arange(n) % 4]
    ref, S, _ = pc.hier_eval(w, obs, state, done)
    mask = (done != 0).astype(np.float32)
    if strategic:
        a, st, ang, code = SepmcPolicy(w).act(obs, state, mask, return_aux=True)
        inside = np.abs(ref["heading_pre"]) < np.pi - 1e-4
        _agree(ang[inside], ref["heading"][inside], S["heading"][inside], "heading")
    else:
        a, st, code = EpmcPolicy(w).act(obs, state, mask, return_code=True)
    dec = ref["gap"] > 4 * pc.KAPPA_HIER * S["gap"]
    assert dec.mean() > 0.9
    assert np.array_equal(code[dec], ref["code"][dec])
    _agree(st, ref["state"], S["state"], "state")
    _agree(a[dec], ref["actions"][dec], S["actions"][dec], "actions")


def _all_reached(reached):
    missing = {k: (len(v) - sum(v), len(v)) for k, v in reached.items() if not all(v)}
    assert not missing, missing


def test_pmc_batch_reaches_every_category_and_every_row_is_decisive():
    w, obs, cats, info, ref, S = pc.pmc_case()
    assert obs.shape == (pc.PMC_N, 207) and obs.dtype == np.float32
    reached = pc.pmc_reaches(w, obs, cats, info, ref, S)
    assert set(reached) == {"random", "clip", "saturate", "tie_same_lane_lo", "tie_same_lane_hi", "tight", "tiny_std"}
    _all_reached(reached)
    ties = set(info["ties"])
    dec = ref["gap"] > 4 * pc.KAPPA_PMC * S["gap"]
    assert dec.all(), np.flatnonzero(~dec)
    # the designed ties are exact in the fp64 distances and resolve to the lowest column
    for i, (lo, mid, hi) in info["ties"].items():
        d = ref["dist"][i]
        assert d[lo] == d[mid] == d[hi] and ref["code"][i] == lo and np.all(d[:lo] > d[lo])
    assert len(ties) == 6 and w[1][0, pc.TINY_STD_COL] == np.float32(1e-9)
    assert np.isnan(pc.padded(obs[:3], 260, 207)[:, 207:]).all()


@pytest.mark.parametrize("strategic", [False, True])
def test_hierarchical_batch_reaches_every_category_and_every_row_is_decisive(strategic):
    w, obs, state, done, cats, info, ref, S = pc.hier_case(strategic)
    reached = pc.hier_reaches(w, obs, cats, info, ref, S)
    want = {"random", "border", "lidar_wrap", "tie_same_lane_lo", "tie_same_lane_hi", "tight"}
    if strategic:
        want |= {"slot%d" % k for k in range(29)} | {"heading_clip_high", "heading_clip_low", "heading_inside"}
    assert set(reached) == want
    _all_reached(reached)
    dec = ref["gap"] > 4 * pc.KAPPA_HIER * S["gap"]
    assert dec.all(), np.flatnonzero(~dec)
    for i, (lo, mid, hi) in info["ties"].items():
        lg = ref["logits"][i]
        assert lg[lo] == lg[mid] == lg[hi] and ref["code"][i] == lo and np.all(lg[:lo] < lg[lo])
    assert set(np.unique(done).tolist()) == {0, 1, 2, 255} and (np.abs(state) > 0).all(1).all()
