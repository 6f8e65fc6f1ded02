"""EPMC (PlayGroundEnv element 0): CUDA engine vs CPU oracle through the C-ABI (run with -m gpu)."""
import os

import numpy as np
import pytest

import perception_cases as pc
from lifelike_agility_and_play_b200 import _capi as capi
from test_golden_epmc import EPMC_CFG, GOLD
from test_parity_gpu import MU_A, SIGMA_A, TOL, blockrel

pytestmark = pytest.mark.gpu
CONT = [capi.AUX_TARGET_X, capi.AUX_TARGET_Y, capi.AUX_TARGET_SPD, capi.AUX_FOOT_FRICTION, capi.AUX_INIT_POS_DIFF_LEN]   # target, speed command, friction, initial distance


def _pair(n, blob, oracle_lib, seed, **over):
    cfg = dict(EPMC_CFG); cfg.update(over)
    g = np.load(GOLD)
    gpu = capi.VecEngine(capi.load_cuda_library(), n, blob, None, seed=seed, **cfg)
    cpu = capi.VecEngine(oracle_lib, n, blob, None, seed=seed, **cfg)
    for e in (gpu, cpu):
        e.set_init_state(g["init_state"])
    return gpu, cpu


def test_epmc_reset_parity(built, blob, oracle_lib):
    n = 500
    gpu, cpu = _pair(n, blob, oracle_lib, 31)
    for rep in range(3):          # yaw accumulates over resets (PGE:181-189 mutates the shared init-state dict)
        og, oc = gpu.reset(), cpu.reset()
        ag, ac = gpu.get(capi.F_AUX), cpu.get(capi.F_AUX)
        assert np.array_equal(ag[:, [0, 1, 9, 14, 15]], ac[:, [0, 1, 9, 14, 15]])                 # integer bookkeeping: exact
        assert np.allclose(ag, ac, rtol=1e-6, atol=1e-6)
        assert blockrel(og, oc).max() < TOL
        assert blockrel(gpu.get(capi.F_STATE), cpu.get(capi.F_STATE)).max() < TOL
    gpu.close(); cpu.close()


def _front_flips(og, oc, st, err_other):
    """Env-steps whose only deviation is a percep_front ray that is not decisive under the fp64 caster on the oracle's post-step
    pose (within 1e-4 m of the ground-plane branch): every other block within TOL, and every deviating front ray non-decisive."""
    fg, fc = og[:, 588:913].astype(np.float64), oc[:, 588:913].astype(np.float64)
    dev = np.abs(fg - fc) > TOL * np.maximum(1.0, np.abs(fc).max(1, keepdims=True))     # blockrel's normalisation, per value
    out = np.zeros(len(og), bool)
    for i in np.flatnonzero(dev.any(1) & (err_other < TOL)):
        s = st[i].astype(np.float64)
        dec = pc.rays_decisive(s[0:3], pc.rot(s[3:7]), pc.SLAB)[pc.N_DOWN + pc.N_1D:]
        out[i] = not dec[dev[i]].any()
    return out


def _sweep(gpu, cpu, n, steps, rng, front=None):
    E, M, DD, MU = [], [], [], []
    for t in range(steps):
        a = np.clip(MU_A + SIGMA_A * rng.standard_normal((n, 12)).astype(np.float32), -1, 1).astype(np.float32)
        for f in (capi.F_STATE, capi.F_WARMSTART, capi.F_OBS, capi.F_TIME, capi.F_AUX, capi.F_EPISODE_ID, capi.F_REWARD_SUM):
            gpu.set(f, cpu.get(f))
        og, rg, dg = gpu.step(a); oc, rc, dc = cpu.step(a)
        ag, ac = gpu.get(capi.F_AUX), cpu.get(capi.F_AUX)
        assert np.array_equal(ag[:, [0, 1, 9, 14, 15]], ac[:, [0, 1, 9, 14, 15]]), "counters / push schedule / draw indices"
        assert np.allclose(ag[:, [2, 3, 4, 5, 10, 11, 12, 13]], ac[:, [2, 3, 4, 5, 10, 11, 12, 13]], rtol=1e-6, atol=1e-5), "command / push draws"
        e = np.maximum.reduce([blockrel(og[:, :135], oc[:, :135]), blockrel(og[:, 135:], oc[:, 135:]),
                               blockrel(gpu.get(capi.F_STATE), cpu.get(capi.F_STATE)),
                               np.abs(rg - rc) / np.maximum(1e-4, np.abs(rc)) * 1e-1])
        if front is not None:
            other = np.maximum.reduce([blockrel(og[:, :135], oc[:, :135]), blockrel(og[:, 135:588], oc[:, 135:588]), blockrel(og[:, 913:], oc[:, 913:]),
                                       blockrel(gpu.get(capi.F_STATE), cpu.get(capi.F_STATE)), np.abs(rg - rc) / np.maximum(1e-4, np.abs(rc)) * 1e-1])
            front.append(_front_flips(og, oc, cpu.get(capi.F_STATE), other))
        E.append(e); M.append(cpu.get(capi.F_DECISION_MARGIN)); DD.append(dg != dc); MU.append(ac[:, 13].copy())
        m = dc.astype(np.uint8)
        if m.any():
            cpu.reset(m); gpu.reset(m)
    return np.concatenate(E), np.concatenate(M), np.concatenate(DD), np.concatenate(MU)


def test_epmc_substep_parity(built, blob, oracle_lib):
    """Teacher-forced at *sub-step* granularity (substeps = 1, so every 2 ms physics step starts from identical states),
    through the drop from z = 0.5, the landing impacts and the push windows, with the shipped friction range [0.4, 3.0].
    Bullet's 10-iteration Gauss-Seidel is not converged and, for friction coefficients well above 1, amplifies rounding
    differences (the same would hold between a float and a double build of Bullet itself); the bound on the fraction of
    deviating sub-steps is therefore looser than for PMC (ground x foot friction 0.45), and the deviating ones must be
    high-friction or near-branch cases."""
    n, steps = 1024, int(os.environ.get("LLQ_PARITY_SUBSTEPS", 140))
    gpu, cpu = _pair(n, blob, oracle_lib, 7, cmd_freq_lo=30, cmd_freq_hi=90, max_steps=400, substeps=1)
    gpu.reset(); cpu.reset()
    e, m, dd, mu = _sweep(gpu, cpu, n, steps, np.random.default_rng(3))
    bad = (e >= TOL) | dd
    print("EPMC sub-step teacher-forced: %d sub-steps; rel err 50/99/99.9/max = %.1e %.1e %.1e %.1e; %d above 1e-4; their mu %s margins %s" % (
        e.size, np.percentile(e, 50), np.percentile(e, 99), np.percentile(e, 99.9), e.max(), int(bad.sum()),
        ["%.2f" % x for x in mu[bad][:10]], ["%.0e" % x for x in m[bad][:10]]))
    assert bad.mean() <= 1e-3 and np.percentile(e, 99.9) < TOL
    assert e.max() < 5e-2
    gpu.close(); cpu.close()
    # the deviations come from iterating the (unconverged, for large friction non-contractive) Gauss-Seidel sweep: with a single
    # iteration the same sweep stays within 1e-3 everywhere and deviates > 1e-4 in < 0.03 % of the sub-steps
    # (measured: 1 / 3 / 10 / 30 iterations -> 21 / 53 / 65 / 139 deviating sub-steps of 143k, max 2.5e-4 / 6e-4 / 8e-3 / 0.45)
    gpu, cpu = _pair(n, blob, oracle_lib, 7, cmd_freq_lo=30, cmd_freq_hi=90, max_steps=400, substeps=1, solver_iters=1)
    gpu.reset(); cpu.reset()
    front = []
    e1, m1, dd1, mu1 = _sweep(gpu, cpu, n, steps, np.random.default_rng(3), front)
    # a percep_front ray grazing the ground plane may hit on one side and miss on the other: such an env-step is excused only when
    # nothing else deviates and every deviating front ray is within 1e-4 m of its branch (tests/perception_cases.py)
    front_flip = np.concatenate(front)
    print("  with solver_iters = 1: %d above 1e-4, max %.1e" % (int(((e1 >= TOL) & ~front_flip).sum()), e1[~front_flip].max()))
    assert ((e1 >= TOL) & ~front_flip).mean() <= 3e-4 and e1[~front_flip].max() < 1e-3 and front_flip.sum() <= 3
    gpu.close(); cpu.close()


def test_epmc_policy_step_parity_moderate_friction(built, blob, oracle_lib):
    """Full policy steps (10 sub-steps) with the friction range capped at 1.0: same criteria as the PMC test."""
    n, steps = 1024, int(os.environ.get("LLQ_PARITY_STEPS", 12))
    gpu, cpu = _pair(n, blob, oracle_lib, 7, cmd_freq_lo=3, cmd_freq_hi=9, max_steps=40, friction_hi=1.0)
    gpu.reset(); cpu.reset()
    e, m, dd, mu = _sweep(gpu, cpu, n, steps, np.random.default_rng(3))
    bad = (e >= TOL) | dd
    print("EPMC policy-step teacher-forced (mu <= 1): %d env-steps; rel err 50/99/99.9/max = %.1e %.1e %.1e %.1e; %d above 1e-4 (margins %s)" % (
        e.size, np.percentile(e, 50), np.percentile(e, 99), np.percentile(e, 99.9), e.max(), int(bad.sum()), ["%.1e" % x for x in m[bad][:8]]))
    # 0.20 % measured with every collision sphere of the robot live (llq_config.knee_contacts = 2; 25 of 12 288 env-steps, all but a
    # handful within 5e-4 rad / m of a joint-limit or contact branch of the step); the bar leaves room for one more such step
    assert bad.mean() <= 2.5e-3
    assert (bad & (m > 5e-4)).mean() <= 1e-3          # away from any branch of Bullet's step the 1e-4 bar holds for 99.9 %
    gpu.close(); cpu.close()


# ------------------------------------------------------------------------------------------------------------------------
# elements 1-3: corridor arenas (walls, hurdles / bars / cubes)
from test_golden_epmc import T_CONT, T_EXACT, terrain_cfg, terrain_gold  # noqa: E402


def _terrain_pair(element, n, blob, oracle_lib, seed, **over):
    g = terrain_gold(element)
    cfg = terrain_cfg(g); cfg.update(over)
    gpu = capi.VecEngine(capi.load_cuda_library(), n, blob, None, seed=seed, **cfg)
    cpu = capi.VecEngine(oracle_lib, n, blob, None, seed=seed, **cfg)
    for e in (gpu, cpu):
        e.set_init_state(g["init_state"])
    return gpu, cpu


@pytest.mark.parametrize("element", [1, 2, 3])
def test_epmc_terrain_reset_parity(element, built, blob, oracle_lib):
    n = 512
    gpu, cpu = _terrain_pair(element, n, blob, oracle_lib, 41)
    for rep in range(2):
        og, oc = gpu.reset(), cpu.reset()
        assert np.array_equal(gpu.get(capi.F_NBOX), cpu.get(capi.F_NBOX))
        assert np.allclose(gpu.get(capi.F_BOXES), cpu.get(capi.F_BOXES), rtol=1e-6, atol=1e-6)
        ag, ac = gpu.get(capi.F_AUX), cpu.get(capi.F_AUX)
        assert np.array_equal(ag[:, T_EXACT], ac[:, T_EXACT])
        assert np.allclose(ag[:, T_CONT], ac[:, T_CONT], rtol=1e-6, atol=1e-6)
        assert np.maximum(blockrel(og[:, :135], oc[:, :135]), blockrel(og[:, 135:], oc[:, 135:])).max() < TOL
    gpu.close(); cpu.close()


def _crowd_terrain(cpu, rng, n):
    """drop a share of the robots onto / next to their obstacles, the walls and the target"""
    st = cpu.get(capi.F_STATE); aux = cpu.get(capi.F_AUX)
    bx = cpu.get(capi.F_BOXES).reshape(n, 36, 6); nb = cpu.get(capi.F_NBOX)
    for i in rng.choice(n, size=n // 4, replace=False):
        kind = rng.integers(0, 4)
        j = rng.integers(2, nb[i])
        b = bx[i, j]
        if kind == 0:       # on top of / inside the footprint of an obstacle
            st[i, 0] = b[0] + rng.uniform(-0.3, 0.3); st[i, 1] = rng.uniform(-0.2, 0.2); st[i, 2] = 0.31 + (b[2] + b[5] if b[2] - b[5] < 0.05 else 0.0)
        elif kind == 1:     # at the near wall
            st[i, 1] = (bx[i, 0, 1] - bx[i, 0, 4]) - rng.uniform(0.05, 0.3)
        elif kind == 2:     # feet at an obstacle's front edge
            st[i, 0] = b[0] - b[3] - rng.uniform(0.15, 0.3); st[i, 1] = rng.uniform(-0.2, 0.2)
        else:               # next to the target
            st[i, 0] = aux[i, capi.AUX_TARGET_X] - rng.uniform(0.2, 0.8); st[i, 1] = rng.uniform(-0.2, 0.2); st[i, 2] = 0.35
    cpu.set(capi.F_STATE, st)


@pytest.mark.parametrize("element", [1, 2, 3])
def test_epmc_terrain_policy_step_parity(element, built, blob, oracle_lib):
    """Teacher-forced policy steps in the corridor arenas, friction capped at 1 (see the flat-arena test above for why)."""
    n, steps = 1024, int(os.environ.get("LLQ_PARITY_STEPS", 12))
    gpu, cpu = _terrain_pair(element, n, blob, oracle_lib, 7, max_steps=40, friction_hi=1.0, cmd_freq_lo=3, cmd_freq_hi=9)
    gpu.reset(); cpu.reset()
    rng = np.random.default_rng(3)
    E, DD, M, reach = [], [], [], 0
    for t in range(steps):
        if t % 3 == 1:
            _crowd_terrain(cpu, rng, n)
        a = np.clip(MU_A + SIGMA_A * rng.standard_normal((n, 12)).astype(np.float32), -1, 1).astype(np.float32)
        for f in (capi.F_STATE, capi.F_WARMSTART, capi.F_OBS, capi.F_TIME, capi.F_AUX, capi.F_EPISODE_ID, capi.F_REWARD_SUM):
            gpu.set(f, cpu.get(f))
        og, rg, dg = gpu.step(a); oc, rc, dc = cpu.step(a)
        ag, ac = gpu.get(capi.F_AUX), cpu.get(capi.F_AUX)
        assert np.array_equal(ag[:, T_EXACT], ac[:, T_EXACT])
        e = np.maximum.reduce([blockrel(og[:, :135], oc[:, :135]), blockrel(og[:, 135:460], oc[:, 135:460]), blockrel(og[:, 460:588], oc[:, 460:588]),
                               blockrel(og[:, 588:913], oc[:, 588:913]), blockrel(og[:, 913:], oc[:, 913:]),
                               blockrel(gpu.get(capi.F_STATE), cpu.get(capi.F_STATE)), np.abs(rg - rc) / (1 + np.abs(rc))])
        E.append(e); DD.append(dg != dc); M.append(cpu.get(capi.F_DECISION_MARGIN)); reach += int((rc > 0.2).sum())
        m = dc.astype(np.uint8)
        if m.any():
            cpu.reset(m); gpu.reset(m)
    e, dd, m = np.concatenate(E), np.concatenate(DD), np.concatenate(M)
    bad = (e >= TOL) | dd
    print("EPMC element %d teacher-forced: %d env-steps; rel err 50/99/99.9/max = %.1e %.1e %.1e %.1e; %d above 1e-4, %d of them with a decision margin "
          "above 5e-4; %d done mismatches; %d reaches" % (element, e.size, np.percentile(e, 50), np.percentile(e, 99), np.percentile(e, 99.9), e.max(),
                                                       int((e >= TOL).sum()), int((bad & (m > 5e-4)).sum()), int(dd.sum()), reach))
    # robots are repeatedly dropped INTO obstacles (_crowd_terrain): with every collision sphere and the auxiliary edge cylinders live, trunk /
    # hips / shanks start centimetres inside boxes, Bullet's penetration recovery throws them out at metres per second, spheres sit between a
    # box face and its edge cylinder (which of the two owns the manifold point is a branch of the step) and the unconverged Gauss-Seidel sweep
    # amplifies fp32 rounding.  Bars: 1.5 % of all env-steps may deviate, 0.4 % of those away from every branch.
    assert reach > 0 and bad.mean() <= 1.5e-2 and (bad & (m > 5e-4)).mean() <= 4e-3 and np.percentile(e, 99) < 3e-4
    gpu.close(); cpu.close()


@pytest.mark.parametrize("element", [1, 2, 3])
def test_cuda_replays_reference_epmc_terrain_golden(element, built, blob):
    """The reference-generated corridor files through the CUDA engine's own reset()/step() path, robot state teacher-forced."""
    g = terrain_gold(element)
    eng = capi.VecEngine(capi.load_cuda_library(), 1, blob, None, seed=int(g["seed"]), **terrain_cfg(g))
    eng.set_init_state(g["init_state"])
    tp = {int(s): st for s, st in zip(g["tp_step"], g["tp_state"])}
    step, worst, deviating = 0, 0.0, 0
    for ep in range(len(g["reset_obs"])):
        obs = eng.reset()
        nb = int(eng.get(capi.F_NBOX)[0])
        assert nb == int(g["nbox"][ep])
        assert np.allclose(eng.get(capi.F_BOXES)[0].reshape(36, 6)[:nb], g["boxes"][ep][:nb], rtol=1e-6, atol=1e-6)
        assert blockrel(obs, g["reset_obs"][ep][None]).max() < 1e-5
        t = 0
        while step < len(g["episode"]) and g["episode"][step] == ep:
            if t > 0 or step in tp:
                st = eng.get(capi.F_STATE); wm = eng.get(capi.F_WARMSTART)
                if t > 0:
                    st[0] = g["state"][step - 1]
                if step in tp:
                    st[0] = tp[step]; wm[0] = 0.0
                eng.set(capi.F_STATE, st); eng.set(capi.F_WARMSTART, wm)
            o, r, d = eng.step(g["action"][step][None])
            e_new = max(blockrel(o[:, 66:99], g["obs"][step][None, 66:99]).max(), blockrel(o[:, 135:460], g["obs"][step][None, 135:460]).max(),
                        blockrel(o[:, 460:588], g["obs"][step][None, 460:588]).max(), blockrel(o[:, 588:913], g["obs"][step][None, 588:913]).max(),
                        blockrel(o[:, 913:], g["obs"][step][None, 913:]).max())
            worst = max(worst, e_new)
            # a flailing or fallen robot (episode 0, feet wedged into boxes) sits on contact / joint-limit decision boundaries where a
            # single fp32 step may take the other branch: such steps are counted, not tolerated silently
            deviating += int(e_new >= 5e-3 or abs(r[0] - g["reward"][step]) >= 2e-4)
            assert bool(d[0]) == bool(g["done"][step]), ("done", step)
            aux = eng.get(capi.F_AUX)[0]
            assert np.array_equal(aux[T_EXACT], g["aux"][step][T_EXACT]), ("counters", step)
            assert np.allclose(aux[CONT], g["aux"][step][CONT], rtol=1e-5, atol=1e-6)
            step += 1; t += 1
    assert step == len(g["episode"])
    print("CUDA vs reference EPMC element %d golden (state teacher-forced): %d of %d steps deviate by more than 5e-3 (worst %.1e)" % (
        element, deviating, step, worst))
    assert deviating <= 0.06 * step
    eng.close()
