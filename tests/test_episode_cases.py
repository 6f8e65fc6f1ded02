"""The fp64 episode statement and the designed batches of tests/episode_cases.py, on the CPU: the statement against the scipy
reference of test_envlogic_scipy.py, the oracle against the statement on every designed env, every category reached and every branch
decisive.  Without these checks tests/test_episode_cases_gpu.py could pass vacuously."""
import numpy as np
import pytest

import episode_cases as ec
from test_envlogic_scipy import ref_future, ref_mocap_state, ref_prop, ref_reward
from test_policy_cases import test_philox_matches_the_known_answers  # noqa: F401  (the draw's Philox is policy_cases.philox4x32)


def test_the_statement_agrees_with_the_scipy_reference(model):
    ctx, before, cats, _ = ec.case(5)
    st = before["state"].astype(np.float64)
    ref = ec.step_statement(ctx, before, st)
    frames, dt = ctx["frames"], ctx["mc"].frame_dt
    clip = before["clip"]
    for i in range(ctx["n"]):
        s = ctx["off"][clip[i]] + ref["frame_id"][i]
        f = min(max(ref["frac"][i], 0.0), 1.0)      # scipy's Slerp rejects the -1e-16 fractions of a time just below a frame boundary
        kin = ref_mocap_state(frames[s], frames[s + 1], f, dt)
        k = ref["kin"][i].copy()
        k[3:7] *= np.sign(np.dot(k[3:7], kin[3:7]))
        assert np.allclose(k, kin, rtol=0, atol=1e-9)
        if ref["bad"][i]:                             # a NaN state: the engine's `bad` rule (no counterpart in the reference)
            assert ref["reward64"][i] == 0.0 and ref["done"][i]
            continue
        r, angle = ref_reward(model, st[i], kin, w=ctx["weights"])
        assert abs(r - ref["reward64"][i]) < 1e-12 and abs(angle - ref["angle"][i]) < 1e-9
        assert np.allclose(ref["obs"][i, 66:99], ref_prop(st[i]), rtol=0, atol=1e-12)
        stored = ec.MocapTable(frames, ctx["mc"].offsets, dt, ctx["mc"].names)
        assert np.allclose(ref["obs"][i, 135:], ref_future(stored, clip[i], ref["frame_id"][i], f, st[i, 0:3], st[i, 3:7]), rtol=0, atol=1e-9)
    # the sequential clock of the reference's sub-step loop
    t = before["time"].copy()
    for _ in range(ctx["substeps"]):
        t = t + ctx["sim_dt"]
    assert np.array_equal(t, ref["time"])


@pytest.mark.parametrize("k", range(len(ec.CASES)))
def test_the_oracle_matches_the_statement(k, oracle_lib):
    ratios = ec.run_case(oracle_lib, k, "host", oracle=True)
    print("case %d (n = %d): %s" % (k, ec.CASES[k][0], ratios))


def test_the_designed_batches_reach_every_category():
    seen, terms, first, last, eps = set(), set(), False, False, []
    for k in range(len(ec.CASES)):
        ctx, before, cats, designed = ec.case(k)
        ref = ec.step_statement(ctx, before, before["state"].astype(np.float64))
        ok = ec.reaches(ctx, before, ref, cats)
        assert ok.all(), [(int(i), cats[i]) for i in np.nonzero(~ok)[0][:8]]
        seen |= set(cats)
        terms |= {ec.TERMS[int(np.argmax(ref["loss"][i]))] for i in range(ctx["n"])}      # each reward term dominant somewhere
        C = ctx["mc"].n_clips
        first |= any(j == 0 and s > 0 for j, s in designed.values())
        last |= any(j == C - 2 and s < 0 for j, s in designed.values())
        fin = np.nonzero(ref["done"])[0]
        # finishers of one clip in different CTAs of the step kernel (16 envs) and of the reset kernel (32 envs), env 0 and N - 1
        if ctx["n"] == 4097:
            tab = [i for i in ec._designated_indices(ctx["n"]) if ref["done"][i]]
            assert {0, 4096} <= set(tab) and len({i // 16 for i in tab}) >= 6 and len({i // 32 for i in tab}) >= 4
            clips = set(int(c) for c in before["clip"][fin])
            assert len(clips) < C                                      # clips without a finisher keep their value
        if ctx["gid0"]:
            gid = ctx["gid0"] + np.arange(ctx["n"])
            assert len(set(gid >> 32)) == 2                             # the high word of the counter changes inside the batch
        eps.append(before["episode"])
        # the fp32 addition of the reward to reward_sum rounds (the sum is not the exact fp64 one)
        assert (ref["reward_sum"].astype(np.float64) != before["reward_sum"].astype(np.float64) + ref["reward64"]).mean() > 0.5
    eps = np.concatenate(eps)
    assert (eps >= 2 ** 32).any() and (eps < 2 ** 32).any()                  # the counter's episode high word
    assert set(ec.CATS) <= seen, set(ec.CATS) - seen
    assert set(ec.TERMS) == terms, terms
    assert first and last
    assert {c[1] for c in ec.CASES} == {1, 6, 66, 127, 128, 129, 300} and {c[2] for c in ec.CASES} == {1, 10}
    assert {c[3] for c in ec.CASES} == {3.0, 2.5}


def test_every_branch_is_decisive():
    for k in range(len(ec.CASES)):
        ctx, before, cats, _ = ec.case(k)
        ref = ec.step_statement(ctx, before, before["state"].astype(np.float64))
        d = ec.decisive(ref)
        assert d.all(), [(int(i), cats[i]) for i in np.nonzero(~d)[0][:8]]
