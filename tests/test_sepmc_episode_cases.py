"""The fp64 SEPMC episode statement and the designed pairs of tests/sepmc_episode_cases.py, on the CPU: the statement replays the
reference golden, the oracle matches the statement on every designed pair, every category is reached and every branch decisive.
Without these checks tests/test_sepmc_episode_cases_gpu.py could pass vacuously."""
import numpy as np
import pytest

import perception_cases as pcs
import sepmc_episode_cases as sc
from lifelike_agility_and_play_b200 import _capi as capi
from test_golden_sepmc import EXACT_AUX, GOLD, SEPMC_CFG, teleports

# the golden does not record the push force (its columns are zero): the push count and draws pin the schedule
CONT = [capi.AUX_FLAG_X, capi.AUX_FLAG_Y, capi.AUX_CONTROL_SPD, capi.AUX_TOTAL_SPD, capi.AUX_MAX_SPD, capi.AUX_FOOT_FRICTION]


def _golden_ctx(g):
    return dict(n=2, substeps=10, push=SEPMC_CFG["push_enabled"], gid0=0, seed=int(g["seed"]), max_steps=int(g["max_steps"]),
                friction=(SEPMC_CFG["friction_lo"], SEPMC_CFG["friction_hi"]), push_h=(SEPMC_CFG["push_h_lo"], SEPMC_CFG["push_h_hi"]),
                push_v=(SEPMC_CFG["push_v_lo"], SEPMC_CFG["push_v_hi"]), start_count=SEPMC_CFG["push_start_count"],
                interval=SEPMC_CFG["push_interval_steps"], duration=SEPMC_CFG["push_duration_steps"], init_state=g["init_state"])


def test_the_statement_replays_the_reference_golden():
    """Every step of the reference's own run, teleported steps from the teleported state.  The golden does not record the pose
    before the last sub-step, so the replay takes the touch from the observed switch (the robot without the flag touched it) and
    the tag from done without robot 0's fall or timeup; the rest is stated: done and the exact aux slots exactly, the reward within
    1e-7, the continuous aux within 1e-6."""
    g = np.load(GOLD)
    ctx = _golden_ctx(g)
    tp = teleports(g)
    switches, tags, pushes = 0, 0, 0
    for t in range(len(g["episode"])):
        ep = int(g["episode"][t])
        first = t == 0 or g["episode"][t - 1] != ep
        st0 = (g["reset_state"][ep] if first else g["state"][t - 1]).copy()
        for r, s in tp.get(t, []):
            st0[r] = s
        aux0 = (g["reset_aux"][ep] if first else g["aux"][t - 1]).copy()
        post = g["state"][t].astype(np.float64)
        before = dict(state=st0, aux=aux0, episode=np.array([ep + 1, ep + 1]), obs=np.zeros((2, capi.OBS_DIM_SEPMC)),
                      actions=g["action"][t].astype(np.float64), reward_sum=np.zeros(2, np.float32))
        sw = bool(g["aux"][t][0, capi.AUX_SWITCH_FLAG])
        holder = 0 if aux0[0, capi.AUX_WITH_FLAG] == 1 else 1
        touch = np.zeros(2, bool)
        touch[1 - holder] = sw
        lz, r22 = sc.ec.tilt(post[:1])
        fall0 = abs(lz[0]) > sc.LIMIT or r22[0] < 0.5
        tag = bool(g["done"][t]) and not fall0 and aux0[0, capi.AUX_COUNTER] + 1 < ctx["max_steps"]
        bx = pcs.arena_boxes(aux0[0, capi.AUX_FLAG_X], aux0[0, capi.AUX_FLAG_Y])
        geo = dict(touch=touch, tag=np.array([tag]), vis=np.array(pcs.visible(post[0], post[1], bx)))
        ref = sc.step_statement(ctx, before, post, geo)
        want = g["aux"][t]
        assert bool(ref["done"][0]) == bool(g["done"][t]), t
        assert np.array_equal(ref["aux"][:, EXACT_AUX], want[:, EXACT_AUX]), (t, ref["aux"][:, EXACT_AUX], want[:, EXACT_AUX])
        assert np.allclose(ref["reward64"], g["reward"][t], atol=1e-7), (t, ref["reward64"], g["reward"][t])
        assert np.allclose(ref["aux"][:, CONT], want[:, CONT], rtol=1e-6, atol=1e-6), (t, ref["aux"][:, CONT] - want[:, CONT])
        switches += sw; tags += tag; pushes += int(ref["push_on"][0] > 0)
    print("%d steps, %d switches, %d tags, %d pushed" % (len(g["episode"]), switches, tags, pushes))
    assert switches >= 2 and tags >= 1 and pushes > 0


def test_the_reset_statement_replays_the_reference_golden():
    """The 8 resets of the reference's own run: the draws of the pair, the chained yaw accumulator, the reset state, the
    observation row (prop, the rays and the SEPMC vectors)"""
    g = np.load(GOLD)
    ctx = _golden_ctx(g)
    acc = 0.0
    for ep in range(len(g["reset_aux"])):
        ref = sc.reset_statement(ctx, np.array([0]), np.array([ep]), np.array([acc]), np.zeros(2, bool))
        want = g["reset_aux"][ep]
        st = ref["state"]
        vis = pcs.visible(st[0], st[1], pcs.arena_boxes(*[f[0] for f in ref["flag_reset"]]))
        ref["aux"][:, capi.AUX_OPPO_VISIBLE] = vis
        assert np.array_equal(ref["aux"][:, EXACT_AUX], want[:, EXACT_AUX]), (ep, ref["aux"][:, EXACT_AUX], want[:, EXACT_AUX])
        c = [capi.AUX_FLAG_X, capi.AUX_FLAG_Y, capi.AUX_CONTROL_SPD, capi.AUX_FOOT_FRICTION]      # the golden has no yaw column:
        # the reset orientations below pin the accumulator's chain
        assert np.allclose(ref["aux"][:, c], want[:, c], rtol=1e-6, atol=1e-6), (ep, ref["aux"][:, c], want[:, c])
        q = st[:, 3:7] * np.sign(np.sum(st[:, 3:7] * g["reset_state"][ep][:, 3:7], 1))[:, None]
        assert np.allclose(q, g["reset_state"][ep][:, 3:7], atol=1e-6) and np.allclose(st[:, 0:3], g["reset_state"][ep][:, 0:3])
        obs = g["reset_obs"][ep].astype(np.float64)
        assert np.allclose(ref["obs"], obs[:, 0:135], atol=1e-6)
        V, _ = sc.perception(st, ref["aux"][:, capi.AUX_WITH_FLAG], *ref["flag_reset"], ref["aux"][:, capi.AUX_CONTROL_SPD], vis)
        assert np.allclose(V, obs[:, 135:], rtol=1e-6, atol=1e-5), (ep, np.argwhere(np.abs(V - obs[:, 135:]) > 1e-5)[:5])
        acc = ref["aux"][0, capi.AUX_YAW_ACCUM_DEG]


@pytest.mark.parametrize("k", range(len(sc.CASES)))
def test_the_oracle_matches_the_statement(k, oracle_lib):
    ratios = sc.run_case(oracle_lib, k, "host", oracle=True)
    print("case %d (n = %d): %s" % (k, sc.CASES[k][0], ratios))


def test_the_designed_batches_reach_every_category(oracle_lib):
    """on the oracle's post-step states: every pair reaches its category, every branch is decisive, every ray of the post poses is
    decisive; all categories and batch edges occur"""
    seen, eps = set(), []
    for k in range(len(sc.CASES)):
        ctx, before, cats = sc.case(k)
        e = sc.make(oracle_lib, ctx, 0)
        sc.xc.set_before(e, before)
        e.step(before["actions"])
        post = e.get(capi.F_STATE).astype(np.float64)
        e.close()
        geo = sc.geometry(ctx, before, post)
        ref = sc.step_statement(ctx, before, post, geo)
        ok = sc.reaches(ctx, before, ref, geo, cats, post)
        assert ok.all(), (k, [(int(p), cats[p]) for p in np.nonzero(~ok)[0][:8]])
        d = sc.decisive(ctx, ref, geo, before, post)
        assert d.all(), (k, [(int(p), cats[p]) for p in np.nonzero(~d)[0][:8]])
        fx, fy = ref["flag_step"]
        fin = np.repeat(np.isfinite(post).all(1).reshape(-1, 2).all(1), 2)     # the rows whose perception is compared
        for i in np.nonzero(fin)[0]:
            assert pcs.rays_decisive(post[i, 0:3], pcs.rot(post[i, 3:7]), pcs.arena_boxes(fx[i // 2], fy[i // 2])).all(), (k, int(i), cats[i // 2])
        seen |= set(cats)
        if ctx["gid0"]:
            assert len(set((ctx["gid0"] + np.arange(ctx["n"])) >> 32)) == 2      # the gid's high word changes inside the batch
        eps.append(before["episode"])
    eps = np.concatenate(eps)
    assert (eps >= 2 ** 32).any() and (eps < 2 ** 32).any()
    every = set(sc.cats_of(10, 1)) | set(sc.ID_CATS)
    assert every <= seen, every - seen
    assert {c[0] for c in sc.CASES} == {2, 8, 10, 16, 18, 32, 34, 162}
    assert {c[1] for c in sc.CASES} == {1, 10} and {c[2] for c in sc.CASES} == {0, 1}
    assert {c[3] for c in sc.CASES} == {0, 2 ** 32 - 4, 2 ** 32 - 5}
