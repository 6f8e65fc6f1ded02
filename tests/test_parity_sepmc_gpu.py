"""SEPMC (ChaseTagGameEnv, empty arena): CUDA engine vs CPU oracle through the C-ABI, and the CUDA engine against the
reference-generated golden file (run with -m gpu).  Tolerance: 1e-4 relative (blockrel) on observations and state."""
import os

import numpy as np
import pytest

from lifelike_agility_and_play_b200 import _capi as capi
from test_golden_sepmc import CONT_AUX, EXACT_AUX, GOLD, SEG, SEPMC_CFG, align, relerr, teleports
from test_parity_gpu import MU_A, SIGMA_A, TOL, blockrel

pytestmark = pytest.mark.gpu
FLAG_SPD_MU = [capi.AUX_FLAG_X, capi.AUX_FLAG_Y, capi.AUX_CONTROL_SPD, capi.AUX_FOOT_FRICTION]
FIELDS = (capi.F_STATE, capi.F_WARMSTART, capi.F_OBS, capi.F_TIME, capi.F_AUX, capi.F_EPISODE_ID, capi.F_REWARD_SUM)


def _pair(n, blob, oracle_lib, seed, **over):
    cfg = dict(SEPMC_CFG); cfg.update(over)
    g = np.load(GOLD)
    gpu = capi.VecEngine(capi.load_cuda_library(), n, blob, None, seed=seed, **cfg)
    cpu = capi.VecEngine(oracle_lib, n, blob, None, seed=seed, **cfg)
    for e in (gpu, cpu):
        e.set_init_state(g["init_state"])
    return gpu, cpu


def seg_err(og, oc):
    """worst block-relative error over the observation entries, per robot"""
    return np.maximum.reduce([blockrel(og[:, a:b], oc[:, a:b]) for a, b in SEG.values()])


def test_sepmc_reset_parity(built, blob, oracle_lib):
    n = 512
    gpu, cpu = _pair(n, blob, oracle_lib, 31, max_steps=50)
    assert gpu.obs_dim == 965
    for rep in range(3):          # the pair's yaw accumulates over resets (CTG:209-215 mutates the shared init-state dict)
        og, oc = gpu.reset(), cpu.reset()
        ag, ac = gpu.get(capi.F_AUX), cpu.get(capi.F_AUX)
        assert np.array_equal(ag[:, EXACT_AUX], ac[:, EXACT_AUX])
        assert np.allclose(ag[:, CONT_AUX + [capi.AUX_YAW_ACCUM_DEG]], ac[:, CONT_AUX + [capi.AUX_YAW_ACCUM_DEG]], rtol=1e-6, atol=1e-6)
        assert seg_err(og, oc).max() < TOL
        assert blockrel(gpu.get(capi.F_STATE), cpu.get(capi.F_STATE)).max() < TOL
    gpu.close(); cpu.close()


def _crowd(cpu, rng, n):
    """move some pairs into the interesting situations: next to the flag, next to each other, at a wall"""
    st = cpu.get(capi.F_STATE); aux = cpu.get(capi.F_AUX)
    for p in rng.choice(n // 2, size=n // 8, replace=False):
        kind = rng.integers(0, 4)
        r = 2 * p + rng.integers(0, 2)
        if kind == 0:       # onto the flag
            st[r, 0:2] = aux[r, [capi.AUX_FLAG_X, capi.AUX_FLAG_Y]] + rng.uniform(-0.25, 0.25, 2)
        elif kind == 1:     # onto the partner
            st[r, 0:2] = st[r ^ 1, 0:2] + rng.uniform(-0.35, 0.35, 2)
        elif kind == 2:     # into a wall
            ax = rng.integers(0, 2)
            st[r, ax] = rng.choice([-1.0, 1.0]) * rng.uniform(2.2, 2.4)
        else:               # flag right in front of the head
            st[r, 0:2] = aux[r, [capi.AUX_FLAG_X, capi.AUX_FLAG_Y]] - 0.35 * np.array([1 - 2 * (st[r, 4] ** 2 + st[r, 5] ** 2), 2 * (st[r, 3] * st[r, 4] + st[r, 5] * st[r, 6])])
    cpu.set(capi.F_STATE, st)


def _sweep(gpu, cpu, n, steps, rng, crowd_every=3):
    E, M, DD = [], [], []
    ev = dict(switch=0, tag=0, invisible=0, wall=0)
    for t in range(steps):
        if crowd_every and t % crowd_every == 1:
            _crowd(cpu, rng, n)
        a = np.clip(MU_A + SIGMA_A * rng.standard_normal((n, 12)).astype(np.float32), -1, 1).astype(np.float32)
        for f in FIELDS:
            gpu.set(f, cpu.get(f))
        og, rg, dg = gpu.step(a); oc, rc, dc = cpu.step(a)
        ag, ac = gpu.get(capi.F_AUX), cpu.get(capi.F_AUX)
        m = cpu.get(capi.F_DECISION_MARGIN)
        # discrete outcomes (touch / tag / visibility / counters) must agree except right at a geometric threshold
        disc = np.any(ag[:, EXACT_AUX + [capi.AUX_FLAG_TOUCH]] != ac[:, EXACT_AUX + [capi.AUX_FLAG_TOUCH]], axis=1) | (dg != dc) | (np.abs(rg - rc) > 1e-6)
        e = np.maximum(seg_err(og, oc), blockrel(gpu.get(capi.F_STATE), cpu.get(capi.F_STATE)))
        assert np.allclose(ag[~disc][:, [2, 3, 4, 13]], ac[~disc][:, [2, 3, 4, 13]], rtol=1e-6, atol=1e-6), "flag position / speed command / friction"
        ok = ~disc & (e < TOL)
        assert np.allclose(ag[ok][:, [7, 8]], ac[ok][:, [7, 8]], rtol=1e-3, atol=1e-4), "speed statistics"
        E.append(e); M.append(m); DD.append(disc)
        ev["switch"] += int(ac[:, 6].sum()); ev["tag"] += int((np.abs(rc) > 0).sum() - ac[:, 6].sum()); ev["invisible"] += int((ac[:, 5] == 0).sum())
        st = cpu.get(capi.F_STATE)
        ev["wall"] += int((np.abs(st[:, 0:2]).max(1) > 2.2).sum())
        mk = dc.astype(np.uint8)
        if mk.any():
            cpu.reset(mk); gpu.reset(mk)
    return np.concatenate(E), np.concatenate(M), np.concatenate(DD), ev


def test_sepmc_policy_step_parity(built, blob, oracle_lib):
    """Teacher-forced full policy steps; pairs are regularly moved next to the flag / each other / the walls so that switches,
    tags, occlusions and wall contacts all occur.  Friction capped at 1 (see tests/test_parity_epmc_gpu.py for why)."""
    n, steps = 1024, int(os.environ.get("LLQ_PARITY_STEPS", 14))
    gpu, cpu = _pair(n, blob, oracle_lib, 7, max_steps=40, friction_hi=1.0, push_start_count=-30, push_interval_steps=120, push_duration_steps=40)
    gpu.reset(); cpu.reset()
    e, m, dd, ev = _sweep(gpu, cpu, n, steps, np.random.default_rng(3))
    bad = (e >= TOL) | dd
    print("SEPMC policy-step teacher-forced: %d robot-steps; rel err 50/99/99.9/max = %.1e %.1e %.1e %.1e; %d above 1e-4, %d discrete mismatches; events %s" % (
        e.size, np.percentile(e, 50), np.percentile(e, 99), np.percentile(e, 99.9), e.max(), int((e >= TOL).sum()), int(dd.sum()), ev))
    assert ev["switch"] > 0 and ev["tag"] > 0 and ev["invisible"] > 0 and ev["wall"] > 0
    assert bad.mean() <= 3e-3 and dd.mean() <= 1e-3
    gpu.close(); cpu.close()


def test_sepmc_substep_parity_shipped_friction(built, blob, oracle_lib):
    n, steps = 1024, int(os.environ.get("LLQ_PARITY_SUBSTEPS", 120))
    gpu, cpu = _pair(n, blob, oracle_lib, 9, max_steps=400, substeps=1, push_start_count=-30, push_interval_steps=120, push_duration_steps=40)
    gpu.reset(); cpu.reset()
    e, m, dd, ev = _sweep(gpu, cpu, n, steps, np.random.default_rng(5), crowd_every=40)
    bad = (e >= TOL) | dd
    print("SEPMC sub-step teacher-forced: %d sub-steps; rel err 50/99/99.9/max = %.1e %.1e %.1e %.1e; %d above 1e-4" % (
        e.size, np.percentile(e, 50), np.percentile(e, 99), np.percentile(e, 99.9), e.max(), int(bad.sum())))
    assert bad.mean() <= 2e-3 and np.percentile(e, 99.9) < 10 * TOL
    gpu.close(); cpu.close()


def test_cuda_replays_reference_sepmc_golden(built, blob):
    """The reference-generated file through the CUDA engine's own reset()/step() sampling path.  The robot states are
    teacher-forced from the file before every step (fp32 trajectories separate chaotically otherwise), everything else --
    reset draws, push schedule, flag / tag / visibility logic, counters -- runs open loop and must match exactly."""
    g = np.load(GOLD)
    eng = capi.VecEngine(capi.load_cuda_library(), 2, blob, None, seed=int(g["seed"]), max_steps=int(g["max_steps"]), **SEPMC_CFG)
    eng.set_init_state(g["init_state"])
    tp = teleports(g)
    step, worst, deviating = 0, 0.0, []
    for ep in range(len(g["reset_obs"])):
        obs = eng.reset()
        assert seg_err(obs, g["reset_obs"][ep]).max() < 1e-5, ("reset obs", ep)
        aux = eng.get(capi.F_AUX)
        assert np.array_equal(aux[:, EXACT_AUX], g["reset_aux"][ep][:, EXACT_AUX])
        assert np.allclose(aux[:, CONT_AUX], g["reset_aux"][ep][:, CONT_AUX], rtol=1e-5, atol=1e-6)
        t = 0
        while step < len(g["episode"]) and g["episode"][step] == ep:
            if t > 0 or step in tp:
                st = eng.get(capi.F_STATE); wm = eng.get(capi.F_WARMSTART)
                if t > 0:
                    st[:] = align(st, g["state"][step - 1])
                for r, s37 in tp.get(step, []):
                    st[r] = s37; wm[r] = 0.0
                eng.set(capi.F_STATE, st); eng.set(capi.F_WARMSTART, wm)
            o, r, d = eng.step(g["action"][step])
            # prop history entries older than this step were produced by the free-running fp32 engine: compare the new frame,
            # the perception and the game vectors
            new = np.r_[66:99, 123:965]
            e_new = blockrel(o[:, new], g["obs"][step][:, new]).max()
            worst = max(worst, e_new)
            # a step in which a joint sits within fp32 rounding of its stop (or a sphere within rounding of the contact threshold) may take
            # the other branch of Bullet's step than the fp64 reference run did: such steps are counted and bounded, not tolerated silently
            if e_new >= 5e-3:
                deviating.append((step, float(e_new)))
            assert np.allclose(r, g["reward"][step], atol=1e-6), ("reward", step, r, g["reward"][step])
            assert bool(d[0]) == bool(d[1]) == bool(g["done"][step]), ("done", step)
            aux = eng.get(capi.F_AUX)
            assert np.array_equal(aux[:, EXACT_AUX], g["aux"][step][:, EXACT_AUX]), ("discrete", step, aux[:, EXACT_AUX], g["aux"][step][:, EXACT_AUX])
            assert np.allclose(aux[:, FLAG_SPD_MU], g["aux"][step][:, FLAG_SPD_MU], rtol=1e-5, atol=1e-6), ("flag / speed / friction", step)
            step += 1; t += 1
    assert step == len(g["episode"])
    print("CUDA vs reference SEPMC golden (state teacher-forced): %d of %d steps deviate by more than 5e-3 %s; every reward / done / counter equal" % (
        len(deviating), step, deviating[:4]))
    assert len(deviating) <= 0.02 * step
    eng.close()
