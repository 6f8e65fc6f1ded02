"""The fp64 EPMC episode statement and the designed batches of tests/epmc_episode_cases.py, on the CPU: the statement replays the
reference goldens, the oracle matches the statement on every designed env, every category is reached and every branch decisive.
Without these checks tests/test_epmc_episode_cases_gpu.py could pass vacuously."""
import numpy as np
import pytest

import epmc_episode_cases as xc
from lifelike_agility_and_play_b200 import _capi as capi
from test_golden_epmc import EPMC_CFG, GOLD, terrain_gold

EXACT = list(xc.EXACT_AUX)
CONT = [capi.AUX_TARGET_X, capi.AUX_TARGET_Y, capi.AUX_TARGET_SPD, capi.AUX_TARGET_ANGLE, capi.AUX_LAST_POS_DIFF_LEN,
        capi.AUX_TOTAL_SPD, capi.AUX_MAX_SPD, capi.AUX_PUSH_F, capi.AUX_PUSH_F + 1, capi.AUX_PUSH_F + 2]


def _golden_ctx(g, element):
    return dict(n=1, element=element, substeps=10, push=EPMC_CFG["push_enabled"], gid0=0, seed=int(g["seed"]), max_steps=int(g["max_steps"]),
                cmd_freq=(EPMC_CFG["cmd_freq_lo"], EPMC_CFG["cmd_freq_hi"]), target_spd=(EPMC_CFG["target_spd_lo"], EPMC_CFG["target_spd_hi"]), push_h=(EPMC_CFG["push_h_lo"], EPMC_CFG["push_h_hi"]),
                push_v=(EPMC_CFG["push_v_lo"], EPMC_CFG["push_v_hi"]), start_count=EPMC_CFG["push_start_count"],
                interval=EPMC_CFG["push_interval_steps"], duration=EPMC_CFG["push_duration_steps"])


@pytest.mark.parametrize("element", [0, 1, 2, 3])
def test_the_statement_replays_the_reference_golden(element):
    """Every step of the reference's own run (teleported steps excepted): the golden state before and after the step and the golden
    aux before it give the golden done and counters exactly, the reward and the continuous aux within 1e-6."""
    g = np.load(GOLD) if element == 0 else terrain_gold(element)
    ctx = _golden_ctx(g, element)
    tp = set(int(s) for s in g["tp_step"]) if "tp_step" in g.files else set()
    checked, reaches, redraws, pushes = 0, 0, 0, 0
    for t in range(len(g["episode"])):
        ep = int(g["episode"][t])
        first = t == 0 or g["episode"][t - 1] != ep
        if t in tp:
            continue
        st0 = g["reset_state"][ep] if first else g["state"][t - 1]
        aux0 = g["reset_aux"][ep] if first else g["aux"][t - 1]
        before = dict(state=st0[None], aux=aux0[None].copy(), episode=np.array([ep + 1]), obs=np.zeros((1, 916)),
                      actions=g["action"][t][None].astype(np.float64), reward_sum=np.zeros(1, np.float32))
        ref = xc.step_statement(ctx, before, g["state"][t][None])
        assert bool(ref["done"][0]) == bool(g["done"][t]), (element, t)
        assert np.array_equal(ref["aux"][0, EXACT], g["aux"][t][EXACT]), (element, t, ref["aux"][0, EXACT], g["aux"][t][EXACT])
        assert abs(ref["reward64"][0] - g["reward"][t]) <= 1e-6, (element, t, ref["reward64"][0], g["reward"][t])
        assert np.allclose(ref["aux"][0, CONT], g["aux"][t][CONT], rtol=1e-6, atol=1e-6), (element, t, ref["aux"][0, CONT] - g["aux"][t][CONT])
        checked += 1
        reaches += bool(ref["reach"][0]); redraws += bool(ref["redraw"][0]); pushes += int(ref["push_on"][0] > 0)
    print("element %d: %d steps, %d reach, %d redraws, %d pushed" % (element, checked, reaches, redraws, pushes))
    assert redraws > 1 and checked > 90


def test_the_reset_statement_replays_the_reference_golden():
    """The reset draws of the reference's own run: friction, cmd_vary_freq, the push draw, and the reset state's orientation."""
    g = np.load(GOLD)
    ctx = _golden_ctx(g, 0)
    ctx.update(friction=(EPMC_CFG["friction_lo"], EPMC_CFG["friction_hi"]), init_state=g["init_state"])
    acc = np.zeros(1)
    for ep in range(len(g["reset_aux"])):
        aux = np.zeros((1, capi.AUX_DIM)); aux[0, capi.AUX_YAW_ACCUM_DEG] = acc[0]
        ref = xc.reset_statement(ctx, np.array([0]), np.array([ep]), aux, np.array([8.0]))
        want = g["reset_aux"][ep]
        assert np.array_equal(ref["aux"][0, EXACT], want[EXACT]), (ep, ref["aux"][0, EXACT], want[EXACT])
        c = [capi.AUX_FOOT_FRICTION, capi.AUX_PUSH_F, capi.AUX_PUSH_F + 1, capi.AUX_PUSH_F + 2, capi.AUX_TARGET_X, capi.AUX_LAST_POS_DIFF_LEN]
        assert np.allclose(ref["aux"][0, c], want[c], rtol=1e-6, atol=1e-6), (ep, ref["aux"][0, c], want[c])
        q = ref["state"][0, 3:7] * np.sign(ref["state"][0, 3:7] @ g["reset_state"][ep][3:7])
        assert np.allclose(q, g["reset_state"][ep][3:7], atol=1e-6) and np.allclose(ref["state"][0, 0:3], g["reset_state"][ep][0:3])
        acc = ref["aux"][:, capi.AUX_YAW_ACCUM_DEG]


@pytest.mark.parametrize("k", range(len(xc.CASES)))
def test_the_oracle_matches_the_statement(k, oracle_lib):
    ratios = xc.run_case(oracle_lib, k, "host", oracle=True)
    print("case %d (n = %d, element %d): %s" % (k, xc.CASES[k][0], xc.CASES[k][1], ratios))


def test_the_designed_batches_reach_every_category(oracle_lib):
    """on the oracle's post-step states: every env reaches its category, every branch is decisive, every ray of the post pose is
    decisive; all categories, reward terms and batch edges occur"""
    seen, terms, eps = set(), set(), []
    for k in range(len(xc.CASES)):
        ctx, before, cats = xc.case(k)
        e = xc.make(oracle_lib, ctx, 0)
        xc.set_before(e, before)
        e.step(before["actions"])
        f = xc.readback(e)
        e.close()
        post = f["state"].astype(np.float64)
        ref = xc.step_statement(ctx, before, post)
        ok = xc.reaches(ctx, before, ref, cats, post)
        assert ok.all(), (k, [(int(i), cats[i]) for i in np.nonzero(~ok)[0][:8]])
        d = xc.decisive(ctx, ref, before, post)
        assert d.all(), (k, [(int(i), cats[i]) for i in np.nonzero(~d)[0][:8]])
        fin = np.isfinite(post).all(1)
        for i in np.nonzero(fin)[0]:
            bx = xc.pcs.corridor_boxes(f["boxes"][i, :f["nbox"][i]]) if f["nbox"][i] else xc.pcs.SLAB
            assert xc.pcs.rays_decisive(post[i, 0:3], xc.pcs.rot(post[i, 3:7]), bx).all(), (k, int(i), cats[i])
        seen |= set(cats)
        if ctx["element"]:
            live = ~ref["bad"]
            terms |= {xc.TERMS[int(np.argmax(np.abs(ref["terms"][i])))] for i in np.nonzero(live)[0]}
        if ctx["gid0"]:
            assert len(set((ctx["gid0"] + np.arange(ctx["n"])) >> 32)) == 2      # the gid's high word changes inside the batch
        eps.append(before["episode"])
    eps = np.concatenate(eps)
    assert (eps >= 2 ** 32).any() and (eps < 2 ** 32).any()
    every = set(xc.cats_of(0, 1)) | set(xc.cats_of(1, 1))
    assert every <= seen, every - seen
    assert terms == set(xc.TERMS), terms
    assert {c[0] for c in xc.CASES} == {1, 7, 8, 9, 15, 16, 17, 31, 32, 33, 4097} and {c[1] for c in xc.CASES} == {0, 1, 2, 3}
    assert {c[2] for c in xc.CASES} == {1, 10} and {c[3] for c in xc.CASES} == {0, 1}


def test_episode_ids_key_only_their_low_word():
    """e and e + 2^32 draw the same numbers in every stream: the engines put the episode's low word into the Philox counter"""
    u = xc.stream_uniforms(7, np.array([3, 3]), np.array([5, 5 + 2 ** 32]), 1, 0)
    assert np.array_equal(u[:, 0], u[:, 1])
