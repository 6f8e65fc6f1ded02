"""Row f3: TLeague-format unrolls from a trajectory slab (parallel/unroll.py; distill_actor.py:164-167, pmc_net_data.py:7-16)
and the on-device actor loops that fill the slab (parallel/rollout.py)."""
import numpy as np
import pytest
import torch

from lifelike_agility_and_play_b200.parallel import (RECORD_SHAPES, RECORD_WIDTH, TRAJ_WIDTH, lambda_returns, slab_records,
                                                     slab_to_unrolls, unflatten_unroll)
from lifelike_agility_and_play_b200.parallel.trajectory import COL_ACTION, COL_DONE, COL_NEGLOGP, COL_REWARD, COL_VALUE


def _slab(T=9, N=5, seed=0):
    rng = np.random.default_rng(seed)
    s = rng.standard_normal((T, N, TRAJ_WIDTH)).astype(np.float32)
    s[:, :, COL_DONE] = (rng.random((T, N)) < 0.2).astype(np.float32)
    s[:, :, COL_REWARD] = rng.random((T, N)).astype(np.float32)
    return torch.from_numpy(s)


def test_lambda_returns_against_scalar_recursion():
    s = _slab()
    T, N, _ = s.shape
    gamma, lam = 0.95, 0.9
    boot = torch.from_numpy(np.random.default_rng(1).standard_normal(N).astype(np.float32))
    r, d, v = s[:, :, COL_REWARD], s[:, :, COL_DONE], s[:, :, COL_VALUE]
    got = lambda_returns(r, gamma * (1 - d), v, boot, lam).numpy()
    for i in range(N):                       # the forward view written out per env in float64 (pmc_net.py:213-224 semantics)
        R, Vn = float(boot[i]), float(boot[i])
        for t in range(T - 1, -1, -1):
            disc = gamma * (1.0 - float(d[t, i]))
            R = float(r[t, i]) + disc * ((1 - lam) * Vn + lam * R)
            Vn = float(v[t, i])
            assert abs(got[t, i] - R) < 1e-5
    # lam = 1 and no terminations: plain discounted sum + bootstrap
    r1 = torch.ones((4, 1)); z = torch.zeros((4, 1))
    out = lambda_returns(r1, 0.5 * torch.ones((4, 1)), z, torch.tensor([8.0]), 1.0)
    assert np.allclose(out[:, 0].numpy(), [1 + .5 * (1 + .5 * (1 + .5 * (1 + .5 * 8))), 1 + .5 * (1 + .5 * (1 + 4)), 1 + .5 * 5, 5.0])


def test_unroll_tuple_layout_round_trip():
    s = _slab(T=7, N=3, seed=4)
    infos = [[{"a": 1}], [], [{"b": 2}, {"c": 3}]]
    unrolls = slab_to_unrolls(s, "model:0001", infos=infos, gamma=0.95, lam=0.95)
    assert len(unrolls) == 3
    for i, (key, flat, inf, shapes) in enumerate(unrolls):
        assert key == "model:0001" and flat.dtype == np.float32 and flat.shape == (7 * RECORD_WIDTH,)
        assert shapes == RECORD_SHAPES and inf == infos[i]
        steps = unflatten_unroll(flat, shapes)
        assert len(steps) == 7
        for t, leaves in enumerate(steps):
            prop, prop_a, future, act, neglogp, disc, r, R, V, flat_p = leaves
            row = s[t, i].numpy()
            assert np.array_equal(np.concatenate([prop, prop_a, future]), row[:207])
            assert np.array_equal(act, row[COL_ACTION:COL_ACTION + 12])
            assert neglogp.shape == () and neglogp == row[COL_NEGLOGP]
            assert disc == np.float32(0.95) * (1 - row[COL_DONE]) and r[0] == row[COL_REWARD] and V[0] == row[COL_VALUE]
            assert flat_p.shape == (24,) and np.array_equal(flat_p[:12], act) and np.all(flat_p[12:] == -2.0)
        # the step that ends an episode does not bootstrap: R = r
        for t in range(7):
            if s[t, i, COL_DONE] == 1:
                assert abs(steps[t][7][0] - s[t, i, COL_REWARD].item()) < 1e-6
    rec = slab_records(s)
    assert rec.shape == (3, 7, RECORD_WIDTH)
    with pytest.raises(AssertionError):
        slab_records(s[:, :, :100])


@pytest.mark.gpu
def test_rollout_worker_records_are_aligned(built):
    """RolloutWorker (policy kernel -> fused step, slab rows written in place) against the same CUDA engine driven through
    the host API with the slab's own actions: record t must hold (obs_t, a_t, r_t, done_t), obs_{t+1} = what the step returned."""
    from lifelike_agility_and_play_b200 import _capi as capi
    from lifelike_agility_and_play_b200.model.compile_model import load_model_blob
    from lifelike_agility_and_play_b200.mocap import synthetic_mocap
    from lifelike_agility_and_play_b200.parallel import RolloutWorker
    from lifelike_agility_and_play_b200.policy import DevicePolicy, PmcPolicy
    from test_policy import random_weights
    n, T = 96, 6
    blob, mocap = load_model_blob(), synthetic_mocap(5, seed=2, min_frames=380, max_frames=420)
    w = random_weights(9); w[25] *= 0.05; w[27][:] = -2.0        # logstd_init (pmc_net_data.py:93)
    pol, host_pol = DevicePolicy(w, device=0), PmcPolicy(w)
    lib = capi.load_cuda_library()
    eng = capi.VecEngine(lib, n, blob, mocap, seed=21, device=0, auto_reset=1)
    chk = capi.VecEngine(lib, n, blob, mocap, seed=21, device=0, auto_reset=1)
    worker = RolloutWorker(eng, pol, T, "cuda:0", sample=True, seed=5)
    o0 = eng.reset()
    assert np.array_equal(o0, chk.reset())
    worker.start(o0)
    views, boots = [], []
    for u in range(2):
        for _ in range(T):
            worker.step()
        v = worker.finish_unroll()
        worker.wait()
        views.append(v.clone())                                        # the view itself is recycled after the next unroll
        boots.append(worker.bootstrap_value.clone())
    torch.cuda.synchronize()
    slab = torch.cat(views, 0).cpu().numpy()                       # [2T, N, 223]
    obs = o0
    n_close = 0
    for t in range(2 * T):
        assert np.array_equal(slab[t, :, :207], obs), "record %d does not hold the observation the action was computed from" % t
        a = slab[t, :, COL_ACTION:COL_ACTION + 12]
        a_ref, c_ref = host_pol.act(obs, return_code=True)
        nlp_ref = host_pol.neglogp(a, a_ref)                          # the recorded -log p belongs to the recorded (sampled) action
        close = np.abs(slab[t, :, COL_NEGLOGP] - nlp_ref) < 1e-2
        n_close += int(close.sum())                                   # a different VQ code only at fp32 distance ties (test_policy.py)
        assert np.abs(slab[t, :, COL_VALUE] - host_pol.value(obs)).max() < 1e-4 * (1 + np.abs(host_pol.value(obs)).max())
        obs, rew, done = chk.step(a)
        assert np.array_equal(rew, slab[t, :, COL_REWARD]) and np.array_equal(done.astype(np.float32), slab[t, :, COL_DONE])
    assert n_close >= 0.999 * 2 * T * n, (n_close, 2 * T * n)
    # bootstrap of slab 0 = V(obs_T) = the value recorded with the first step of slab 1; `obs` now holds the observation after the
    # last step = what slab 1's bootstrap was computed from
    assert np.abs(boots[0].cpu().numpy() - slab[T, :, COL_VALUE]).max() < 1e-5
    assert np.abs(boots[1].cpu().numpy() - host_pol.value(obs)).max() < 1e-4 * (1 + np.abs(host_pol.value(obs)).max())
    unrolls = slab_to_unrolls(torch.from_numpy(slab), "m", gamma=0.95, lam=0.95)
    assert len(unrolls) == n and unrolls[0][1].size == 2 * T * RECORD_WIDTH
    pol.close(); eng.close(); chk.close()


@pytest.mark.gpu
def test_workers_refuse_an_engine_without_auto_reset(built):
    """The workers step through the engine's auto-reset: an engine with auto_reset=0 is refused before anything is allocated."""
    from lifelike_agility_and_play_b200 import _capi as capi
    from lifelike_agility_and_play_b200.model.compile_model import load_model_blob
    from lifelike_agility_and_play_b200.mocap import synthetic_mocap
    from lifelike_agility_and_play_b200.parallel import HierRolloutWorker, RolloutWorker
    from lifelike_agility_and_play_b200.policy import DevicePolicy
    from lifelike_agility_and_play_b200.policy_epmc import DeviceHierPolicy, random_weights as hier_weights
    from test_policy import random_weights
    lib, blob = capi.load_cuda_library(), load_model_blob()
    pmc = capi.VecEngine(lib, 8, blob, synthetic_mocap(2, seed=2, min_frames=380, max_frames=420), seed=21, device=0, auto_reset=0)
    epmc = capi.VecEngine(lib, 8, blob, None, device=0, env_kind=capi.ENV_EPMC, auto_reset=0)
    pol, hpol = DevicePolicy(random_weights(9), device=0), DeviceHierPolicy(hier_weights(False, 0), device=0, train=True)
    with pytest.raises(ValueError, match="auto_reset=1"):
        RolloutWorker(pmc, pol, 4, "cuda:0")
    with pytest.raises(ValueError, match="auto_reset=1"):
        HierRolloutWorker(epmc, hpol, 4, "cuda:0")
    pol.close(); hpol.close(); pmc.close(); epmc.close()
