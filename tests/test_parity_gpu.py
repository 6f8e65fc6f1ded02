"""T2/T3: CUDA engine vs CPU oracle through the C-ABI (the parity tests proper; run with -m gpu on an H100).

Tolerance (BASELINE.json north_star): 1e-4 relative.  "Relative" is taken per observation block (prop / future) and per
state block against the block's max-norm, floor 1 -- the reference's own observation consumer normalises per block.
Bullet's step is discontinuous at joint limits and at contact make/break; a step whose oracle decision margin
(LLQ_F_DECISION_MARGIN) is within rounding distance of such a branch may legitimately flip in fp32 and is excluded from
the tight bound (and counted)."""
import numpy as np
import pytest

from lifelike_agility_and_play_b200 import _capi as capi

pytestmark = pytest.mark.gpu

MU_A = np.array([.0124, -.011, -.0793, -.0125, -.0108, -.0806, .0402, -.0505, -.1956, -.0433, -.0515, -.2156], np.float32)
SIGMA_A = np.array([.0853, .1525, .1747, .0847, .1503, .1766, .1025, .2023, .3701, .1021, .2035, .426], np.float32)
TOL = 1e-4
MARGIN_OK = 2e-5      # rad / m: decisions closer than this to a branch are fp32-ambiguous


def blockrel(a, b):
    """max |a-b| / max(1, max|b|) per row."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.max(np.abs(a - b), axis=1) / np.maximum(1.0, np.max(np.abs(b), axis=1))


def teacher_force(gpu, cpu):
    gpu.set(capi.F_STATE, cpu.get(capi.F_STATE)); gpu.set(capi.F_WARMSTART, cpu.get(capi.F_WARMSTART))
    gpu.set(capi.F_OBS, cpu.get(capi.F_OBS)); gpu.set(capi.F_TIME, cpu.get(capi.F_TIME))
    gpu.set(capi.F_CLIP, cpu.get(capi.F_CLIP)); gpu.set(capi.F_REWARD_SUM, cpu.get(capi.F_REWARD_SUM))


def test_reset_parity(make_cuda, make_oracle):
    n = 1000           # deliberately not a multiple of 8 / 32
    gpu, cpu = make_cuda(n, seed=21), make_oracle(n, seed=21)
    og, oc = gpu.reset(), cpu.reset()
    assert np.array_equal(gpu.get(capi.F_CLIP), cpu.get(capi.F_CLIP))            # integer work: bit exact
    assert np.array_equal(gpu.get(capi.F_TIME), cpu.get(capi.F_TIME))            # fp64 Philox -> time: bit exact
    assert np.array_equal(gpu.get(capi.F_EPISODE_ID), cpu.get(capi.F_EPISODE_ID))
    assert blockrel(og[:, :99], oc[:, :99]).max() < TOL and blockrel(og[:, 135:], oc[:, 135:]).max() < TOL
    assert np.all(og[:, 99:135] == 0)
    assert blockrel(gpu.get(capi.F_STATE), cpu.get(capi.F_STATE)).max() < TOL
    # K2: after reset the three stacked props are identical
    assert np.array_equal(og[:, 0:33], og[:, 33:66]) and np.array_equal(og[:, 0:33], og[:, 66:99])
    # masked reset touches only the masked envs
    mask = np.zeros(n, np.uint8); mask[::7] = 1
    before = gpu.get(capi.F_TIME).copy()
    gpu.reset(mask); cpu.reset(mask)
    assert np.array_equal(gpu.get(capi.F_TIME), cpu.get(capi.F_TIME))
    assert np.array_equal(gpu.get(capi.F_TIME)[mask == 0], before[mask == 0])


def test_teacher_forced_step_parity(make_cuda, make_oracle):
    """T2: identical (state, action) into both engines, one full policy step (10 sub-steps) each, 2048 x 12 = 24.5k pairs
    by default (LLQ_PARITY_STEPS raises it; 50 steps = 1e5 pairs).  Requirements:
      * >= 99.9 % of ALL env-steps within 1e-4 relative (obs blocks, state, reward), done flags equal;
      * every env-step that exceeds 1e-4 sits within NEAR_BRANCH of a discontinuity of Bullet's step (joint-limit row
        appears/disappears, contact makes/breaks) according to the oracle's decision margin;
      * nothing outside the fp32-ambiguous band (margin > MARGIN_OK) deviates by more than 5e-3."""
    import os
    n, steps = 2048, int(os.environ.get("LLQ_PARITY_STEPS", 12))
    NEAR_BRANCH = 5e-4         # rad / m.  A weak filter (resting feet sit ~5e-4 m from the contact-breaking threshold, so ~60 % of all
                               # env-steps are this close to a branch); the strong statement is the <= 0.1 % share above
    gpu, cpu = make_cuda(n, seed=5), make_oracle(n, seed=5)
    gpu.reset(); cpu.reset()
    rng = np.random.default_rng(0)
    E, M, ER, DD = [], [], [], []
    for t in range(steps):
        a = np.clip(MU_A + SIGMA_A * rng.standard_normal((n, 12)).astype(np.float32), -1, 1).astype(np.float32)
        teacher_force(gpu, cpu)
        og, rg, dg = gpu.step(a)
        oc, rc, dc = cpu.step(a)
        assert np.array_equal(og[:, 99:135], oc[:, 99:135])                       # action history is copied, not computed
        E.append(np.maximum.reduce([blockrel(og[:, :99], oc[:, :99]), blockrel(og[:, 135:], oc[:, 135:]),
                                    blockrel(gpu.get(capi.F_STATE), cpu.get(capi.F_STATE))]))
        ER.append(np.abs(rg - rc) / np.maximum(1e-2, np.abs(rc)))
        M.append(cpu.get(capi.F_DECISION_MARGIN)); DD.append(dg != dc)
        # envs that finished are re-seeded identically on both sides so the sweep keeps covering fresh states
        m = dc.astype(np.uint8)
        if m.any():
            cpu.reset(m); gpu.reset(m)
    e, er, m, dd = np.concatenate(E), np.concatenate(ER), np.concatenate(M), np.concatenate(DD)
    bad = (e >= TOL) | (er >= TOL) | dd
    print("teacher-forced: %d env-steps; rel err percentiles 50/99/99.9/max = %.1e %.1e %.1e %.1e; reward max %.1e; "
          "%d above 1e-4 (margins %s); %.2f %% of env-steps have a margin below NEAR_BRANCH" % (e.size, np.percentile(e, 50), np.percentile(e, 99), np.percentile(e, 99.9), e.max(),
                                         er.max(), int(bad.sum()), ["%.1e" % x for x in m[bad][:8]], 100.0 * float((m < NEAR_BRANCH).mean())))
    assert bad.mean() <= 1e-3, "more than 0.1%% of env-steps deviate by > 1e-4: %d of %d" % (bad.sum(), bad.size)
    assert np.all(m[bad] < NEAR_BRANCH), "a deviation > 1e-4 occurred away from any branch of the step: margins %s" % m[bad]
    assert e[m > MARGIN_OK].max() < 5e-3
    cg, cc = gpu.counters(), cpu.counters()
    assert abs(int(cg[2]) - int(cc[2])) <= 0.002 * cc[2] + 3 and abs(int(cg[3]) - int(cc[3])) <= 0.02 * cc[3] + 3   # rows solved


def test_open_loop_drift_is_bounded(make_cuda, make_oracle):
    """T3: without teacher forcing the two trajectories separate chaotically; report the curve, bound the first steps."""
    n = 256
    gpu, cpu = make_cuda(n, seed=9), make_oracle(n, seed=9)
    gpu.reset(); cpu.reset()
    rng = np.random.default_rng(1)
    med = []
    alive = np.ones(n, bool)
    for t in range(25):
        a = (0.5 * SIGMA_A * rng.standard_normal((n, 12))).astype(np.float32)
        og, rg, dg = gpu.step(a); oc, rc, dc = cpu.step(a)
        alive &= ~(dg.astype(bool) | dc.astype(bool))
        if alive.sum() < 16:
            break
        med.append(float(np.median(blockrel(og[alive, :99], oc[alive, :99]))))
    print("open-loop median rel. prop error per step:", ["%.1e" % m for m in med])
    assert med[0] < TOL and med[min(4, len(med) - 1)] < 1e-2


def test_auto_reset_and_prioritized_table(make_cuda, make_oracle):
    n = 512
    gpu, cpu = make_cuda(n, seed=3, auto_reset=1), make_oracle(n, seed=3, auto_reset=1)
    gpu.reset(); cpu.reset()
    rng = np.random.default_rng(2)
    finished = 0
    for t in range(40):
        a = np.clip(MU_A + 2 * SIGMA_A * rng.standard_normal((n, 12)).astype(np.float32), -1, 1).astype(np.float32)
        teacher_force(gpu, cpu)
        gpu.set(capi.F_EPISODE_ID, cpu.get(capi.F_EPISODE_ID)); gpu.set(capi.F_AVG_REWARD, cpu.get(capi.F_AVG_REWARD))
        og, rg, dg = gpu.step(a); oc, rc, dc = cpu.step(a)
        margin = cpu.get(capi.F_DECISION_MARGIN)
        same = dg == dc
        assert same[margin > 2.5e-4].all()
        finished += int(dc.sum())
        if same.all():
            assert np.allclose(gpu.get(capi.F_AVG_REWARD), cpu.get(capi.F_AVG_REWARD), rtol=1e-4, atol=1e-6)
            assert np.allclose(gpu.get(capi.F_SAMPLE_PROB), cpu.get(capi.F_SAMPLE_PROB), rtol=1e-3, atol=1e-7)
            clip_eq = gpu.get(capi.F_CLIP) == cpu.get(capi.F_CLIP)
            assert clip_eq.mean() > 0.995       # a uniform draw can straddle a cdf edge that differs in the 7th digit
            rs = dc.astype(bool) & clip_eq
            if rs.any():   # freshly reset envs: time bit-exact, reset observation within tolerance
                assert np.array_equal(gpu.get(capi.F_TIME)[rs], cpu.get(capi.F_TIME)[rs])
                assert blockrel(og[rs][:, :99], oc[rs][:, :99]).max() < TOL
                assert np.all(og[rs][:, 99:135] == 0)
    assert finished > 0, "the sweep never finished an episode; the test is vacuous"


def test_shard_invariance_and_determinism(make_cuda):
    """RNG streams are keyed by the global env id, envs never interact: a [2048,4096) shard equals the second half of a
    4096-env engine bit for bit, and a re-run is bit-identical."""
    n = 4096
    full = make_cuda(n, seed=77, auto_reset=1)
    half = make_cuda(n // 2, seed=77, auto_reset=1, global_env_offset=n // 2)
    again = make_cuda(n, seed=77, auto_reset=1)
    o1, o2, o3 = full.reset(), half.reset(), again.reset()
    assert np.array_equal(o1[n // 2:], o2) and np.array_equal(o1, o3)
    rng = np.random.default_rng(4)
    for t in range(12):
        a = np.clip(MU_A + SIGMA_A * rng.standard_normal((n, 12)).astype(np.float32), -1, 1).astype(np.float32)
        r1, r2, r3 = full.step(a), half.step(a[n // 2:]), again.step(a)
        for x, y in zip(r1, r3):
            assert np.array_equal(x, y)
        # the prioritized-sampling table is per shard (one table per actor process in the reference), so only
        # compare until the first episode ends anywhere
        if not r1[2].any():
            for x, y in zip(r1, r2):
                assert np.array_equal(x[n // 2:], y)


def test_full_size_properties(make_cuda):
    """BASELINE config[1] size (4096 envs): size-independent properties of the rollout."""
    n = 4096
    eng = make_cuda(n, seed=1234, auto_reset=1)
    obs = eng.reset()
    rng = np.random.default_rng(5678)
    dones = 0
    prev = obs
    for t in range(60):
        a = np.clip(MU_A + SIGMA_A * rng.standard_normal((n, 12)).astype(np.float32), -1, 1).astype(np.float32)
        obs, rew, done = eng.step(a)
        assert np.all(np.isfinite(obs)) and np.all(np.isfinite(rew))
        assert np.all(rew >= 0) and np.all(rew <= 1.0 + 1e-6)                       # convex combination of exp(-x)
        alive = done == 0
        # history shift (PLE:282-290): prop blocks 0,1 are last step's blocks 1,2; same for the action history
        assert np.array_equal(obs[alive, 0:66], prev[alive, 33:99])
        assert np.array_equal(obs[alive, 99:123], prev[alive, 111:135])
        assert np.array_equal(obs[alive, 123:135], a[alive])
        # e_g is a unit vector
        assert np.allclose(np.linalg.norm(obs[:, 96:99], axis=1), 1.0, atol=1e-5)
        fresh = done == 1
        assert np.all(obs[fresh, 99:135] == 0) and np.array_equal(obs[fresh, 0:33], obs[fresh, 66:99])
        dones += int(done.sum())
        prev = obs
    assert dones > 0
    st = eng.get(capi.F_STATE)
    assert np.allclose(np.linalg.norm(st[:, 3:7], axis=1), 1.0, atol=1e-4)
    assert np.abs(st[:, 7:]).max() <= 100.0 + 1e-3
    c = eng.counters()
    assert c[0] == 60 * n and c[1] == dones and c[4] >= 120


@pytest.mark.parametrize("n", [1, 3, 9, 37])
def test_ragged_batch_sizes(n, make_cuda, make_oracle):
    """Edge sizes: fewer envs than a warp holds (8), than a CTA holds (32), odd counts -- the padded lanes of the last warp must
    neither write nor disturb the live ones (reset, masked reset of the last env, teacher-forced steps, auto-reset bookkeeping)."""
    gpu, cpu = make_cuda(n, seed=31, auto_reset=1), make_oracle(n, seed=31, auto_reset=1)
    og, oc = gpu.reset(), cpu.reset()
    assert og.shape == (n, 207) and np.array_equal(gpu.get(capi.F_CLIP), cpu.get(capi.F_CLIP))
    assert blockrel(og[:, :99], oc[:, :99]).max() < TOL and blockrel(og[:, 135:], oc[:, 135:]).max() < TOL
    mask = np.zeros(n, np.uint8); mask[-1] = 1
    gpu.reset(mask); cpu.reset(mask)
    assert np.array_equal(gpu.get(capi.F_TIME), cpu.get(capi.F_TIME))
    rng = np.random.default_rng(n)
    for t in range(4):
        a = np.clip(MU_A + SIGMA_A * rng.standard_normal((n, 12)).astype(np.float32), -1, 1).astype(np.float32)
        teacher_force(gpu, cpu)
        og, rg, dg = gpu.step(a)
        oc, rc, dc = cpu.step(a)
        near = cpu.get(capi.F_DECISION_MARGIN) < 2.5e-4
        assert np.array_equal(dg[~near], dc[~near])
        ok = (dc == 0) & (dg == 0) & ~near                      # finished envs were re-seeded by each side's own table
        e = np.maximum(blockrel(og[:, :99], oc[:, :99]), blockrel(og[:, 135:], oc[:, 135:]))
        assert np.all(e[ok] < TOL) and np.all(np.abs(rg - rc)[ok] < TOL)
    assert gpu.counters()[0] == 4 * n
