"""The opponent pool on the GPU (run with -m gpu on an H100): llq_hier_policy_forward_pool against llq_hier_policy_forward of each row's
model bit for bit, its draws against the statement of tests/opponent_pool_cases.py, and SepmcRolloutWorker with a pool against a
host-driven replay."""
import numpy as np
import pytest

import opponent_pool_cases as oc
import policy_cases as pc

pytestmark = pytest.mark.gpu

CANARY = 0x7FBADBAD
SEED = 0x1234_5678_9ABC
W = 984


def _canary(torch, shape, dtype=None):
    t = torch.full(shape, CANARY, dtype=torch.int32, device="cuda")
    return t if dtype is torch.int32 else t.view(torch.float32)


def _bits(t):
    import torch
    return t.view(torch.int32).cpu().numpy() if t.dtype == torch.float32 else t.cpu().numpy()


@pytest.fixture(scope="module")
def models(built):
    from lifelike_agility_and_play_b200.policy_epmc import random_weights
    return [random_weights(True, 100 + k) for k in range(64)]


def _inputs(n, seed):
    rng = np.random.default_rng(seed)
    obs = np.stack([pc._hier_row(rng, pc.HIER_CATS[i % 3], 965) for i in range(n)])
    return obs, pc.hier_random_state(rng, n, 128)


def _pool_run(torch, pool, obs, obs_ld, state, model, done, counter=0, gid0=0, rec_ld=3):
    """One forward_pool with canary outputs (8 rows past n); returns bits of (actions, codes, heading, state, model, record)."""
    n = len(model)
    t_obs = torch.from_numpy(pc.padded(obs, obs_ld, 965)).cuda()
    st = _canary(torch, (n + 8, 128))
    st[:n] = torch.from_numpy(state).cuda()
    act, codes, head = _canary(torch, (n + 8, 12)), _canary(torch, (n + 8,), torch.int32), _canary(torch, (n + 8,))
    rec = _canary(torch, ((n + 8) * rec_ld,))
    d_model = torch.from_numpy(np.asarray(model, np.int32)).cuda()
    t_done = None if done is None else torch.from_numpy(np.asarray(done, np.uint8)).cuda()
    pool.forward(t_obs.data_ptr(), obs_ld, n, None if t_done is None else t_done.data_ptr(), st.data_ptr(), act.data_ptr(), codes.data_ptr(),
                 head.data_ptr(), d_model.data_ptr(), rec.data_ptr(), rec_ld, SEED, counter, gid0)
    torch.cuda.synchronize()
    return [_bits(x) for x in (act, codes, head, st)] + [d_model.cpu().numpy(), _bits(rec)]


def _reference(torch, dets, obs, state, model, done):
    """llq_hier_policy_forward of every row's model (each model on all rows: a row does not depend on the other rows of its CTA)."""
    n = len(model)
    out = [np.full((n, 12), CANARY, np.int32), np.full(n, CANARY, np.int32), np.full(n, CANARY, np.int32), np.full((n, 128), CANARY, np.int32)]
    t_obs = torch.from_numpy(np.ascontiguousarray(obs)).cuda()
    t_done = torch.from_numpy(np.asarray(done, np.uint8)).cuda()
    for k in set(int(m) for m in model if 0 <= m < len(dets)):
        st = torch.from_numpy(np.ascontiguousarray(state)).cuda()
        act, codes, head = torch.zeros((n, 12), device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda"), torch.zeros(n, device="cuda")
        dets[k].forward(t_obs.data_ptr(), 965, n, t_done.data_ptr(), st.data_ptr(), act.data_ptr(), codes.data_ptr(), head.data_ptr())
        torch.cuda.synchronize()
        rows = np.flatnonzero(np.asarray(model) == k)
        for o, t in zip(out, (act, codes, head, st)):
            o[rows] = _bits(t)[rows]
    return out


def _compare(got, ref, model, K, rec_ld, n):
    act, codes, head, st, _, rec = got
    for name, g, r in zip(("actions", "codes", "heading", "state"), (act, codes, head, st), ref):
        assert np.array_equal(g[:n], r), (name, np.flatnonzero((g[:n] != r).reshape(n, -1).any(1))[:10])
        assert (g[n:] == CANARY).all(), (name, "rows past n written")
    m = np.asarray(model)
    want = np.where((m >= 0) & (m < K), m, -1).astype(np.float32).view(np.int32)
    assert np.array_equal(rec[:n * rec_ld:rec_ld], want), "record"
    owned = np.zeros(len(rec), bool)
    owned[:n * rec_ld:rec_ld] = True
    assert (rec[~owned] == CANARY).all(), "record written outside rows i * rec_ld"


def _designed_models(rng, sizes, absent):
    """Rows of model k in `sizes[k]` (interleaved at random), plus `absent` rows of out-of-range models (-1 and K)."""
    model = np.concatenate([np.full(s, k, np.int32) for k, s in enumerate(sizes)] + [np.array([-1, len(sizes), 1000][:absent], np.int32)])
    return model[rng.permutation(len(model))]


@pytest.mark.parametrize("case", ["segments", "one-row", "k1", "k64", "strided"])
def test_pool_forward_equals_each_rows_model_bit_for_bit(models, case):
    import torch
    from lifelike_agility_and_play_b200.policy_epmc import DeviceHierPolicy, DeviceOpponentPool
    rng = np.random.default_rng(["segments", "one-row", "k1", "k64", "strided"].index(case))
    obs_ld, K = 965, 6
    if case in ("segments", "strided"):
        model = _designed_models(rng, [0, 1, 7, 8, 9, 17], 3)      # 45 rows: segments of 0, 1, 7, 8, 9 and 17 rows, three absent models
        obs_ld = 2 * W if case == "strided" else 965
    elif case == "one-row":
        model = np.array([4], np.int32)
    elif case == "k1":
        K, model = 1, np.zeros(61, np.int32)
    else:
        K = 64
        model = rng.integers(0, 64, 300).astype(np.int32)
        model[model == 17] = 18                                        # model 17 absent
        model[:2] = [-1, 64]
    n = len(model)
    assert case != "segments" or n % 8
    obs, state = _inputs(n, 3)
    pool = DeviceOpponentPool(models[:K], device=0, max_rows=max(n, 64))
    dets = [DeviceHierPolicy(models[k], device=0) if k in set(model.tolist()) else None for k in range(K)]
    done = np.zeros(n, np.uint8)
    got = _pool_run(torch, pool, obs, obs_ld, state, model, done)
    ref = _reference(torch, dets, obs, state, model, done)
    out_of_range = (model < 0) | (model >= K)
    for r in ref[:3]:
        r[out_of_range] = CANARY                                       # a row of no segment is left untouched: outputs and state
    ref[3][out_of_range] = state.view(np.int32)[out_of_range]
    _compare(got, ref, model, K, 3, n)
    assert np.array_equal(got[4], model), "an undrawn row changed its model"
    pool.close()
    for d in dets:
        if d is not None:
            d.close()


def test_draws_match_the_statement_at_the_cutoff(models):
    """Cutoffs set to r_a + 1 for two rows with r_b = r_a + 1: row a draws model k, row b model k + 1 (k = 0 and k = 1)."""
    import torch
    from lifelike_agility_and_play_b200.policy_epmc import DeviceOpponentPool
    counter = 5
    ga, gb, ra = oc.adjacent_words(SEED, counter, 1 << 20, 1 << 17)
    assert oc.draw_words([gb], SEED, counter)[0] == ra + 1
    pool = DeviceOpponentPool(models[:3], device=0, max_rows=16)
    obs, state = _inputs(1, 5)
    A = 1 << 20
    for k, probs in ((0, [ra + 1, (1 << 32) - ra - 1 - A, A]), (1, [A, ra + 1 - A, (1 << 32) - ra - 1])):
        pool.set_probs(probs)
        t = oc.cutoffs(probs)
        assert int(t[k]) == ra + 1
        for g, want in ((ga, k), (gb, k + 1)):
            got = _pool_run(torch, pool, obs, 965, state, [2 - k], [1], counter, g)
            assert got[4][0] == want == oc.pick([oc.draw_words([g], SEED, counter)[0]], t)[0], (k, g, got[4][0])
    pool.close()


def test_draws_zero_probability_wipe_keep_and_record(models):
    import torch
    from lifelike_agility_and_play_b200.policy_epmc import DeviceHierPolicy, DeviceOpponentPool
    n, K = 4096, 3
    obs, state = _inputs(n, 9)
    pool = DeviceOpponentPool(models[:K], device=0, max_rows=n, probs=[0.5, 0.5, 0.0])
    t = oc.cutoffs([0.5, 0.5, 0.0])
    dets = [DeviceHierPolicy(models[k], device=0) for k in range(K)]
    rng = np.random.default_rng(4)
    model = rng.integers(0, K, n).astype(np.int32)
    drawn_any = set()
    for counter in range(4):
        done = (rng.random(n) < 0.5).astype(np.uint8)
        done[done != 0] = pc.DONE_BYTES[1 + rng.integers(0, 3, int(done.sum()))]
        want, rec = oc.assign(model, done, t, K, 77, SEED, counter)
        got = _pool_run(torch, pool, obs, 965, state, model, done, counter, 77, rec_ld=1)
        assert np.array_equal(got[4], want), np.flatnonzero(got[4] != want)[:10]
        assert np.array_equal(got[5][:n], rec.view(np.int32))
        drawn_any |= set(want[done != 0].tolist())
        ref = _reference(torch, dets, obs, state, want, done)          # drawn rows: done != 0, the reference wipes their state
        _compare(got, ref, want, K, 1, n)
        model = want
    assert drawn_any == {0, 1}, drawn_any                              # model 2 (p = 0) never drawn
    # no done flags: no draws, the record is written all the same
    got = _pool_run(torch, pool, obs, 965, state, model, None, 9, 77, rec_ld=1)
    assert np.array_equal(got[4], model) and np.array_equal(got[5][:n], model.astype(np.float32).view(np.int32))
    pool.close()
    for d in dets:
        d.close()


def test_pool_entry_points(models):
    import torch
    from lifelike_agility_and_play_b200.policy_epmc import DeviceHierPolicy, DeviceOpponentPool
    pool = DeviceOpponentPool(models[:2], device=0, max_rows=16)
    assert pool.n_models == 2 and pool.strategic and not pool.train and pool.state_dim == 128 and pool.obs_dim == 965
    obs, st, act = torch.zeros((17, W), device="cuda"), torch.zeros((17, 128), device="cuda"), torch.zeros((17, 12), device="cuda")
    m = torch.zeros(17, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError, match="forward_pool"):
        DeviceHierPolicy.forward(pool, obs.data_ptr(), 965, 8, None, st.data_ptr(), act.data_ptr())
    with pytest.raises(RuntimeError, match="max_rows"):
        pool.forward(obs.data_ptr(), 965, 17, None, st.data_ptr(), act.data_ptr(), None, None, m.data_ptr(), None, 1, 0, 0)
    with pytest.raises(RuntimeError, match="row stride"):
        pool.forward(obs.data_ptr(), 964, 8, None, st.data_ptr(), act.data_ptr(), None, None, m.data_ptr(), None, 1, 0, 0)
    det = DeviceHierPolicy(models[0], device=0)
    with pytest.raises(RuntimeError, match="not a pool handle"):
        DeviceOpponentPool.forward(det, obs.data_ptr(), 965, 8, None, st.data_ptr(), act.data_ptr(), None, None, m.data_ptr(), None, 1, 0, 0)
    for bad in ([1.0], [1.0, -0.1], [0.0, 0.0], [1.0, float("nan")], [1.0, float("inf")]):
        with pytest.raises(ValueError):
            pool.set_probs(bad)
    with pytest.raises(ValueError):
        DeviceOpponentPool.set_probs(det, [1.0])
    pool.close(); det.close()


def test_worker_with_a_pool_against_a_replay(models):
    """SepmcRolloutWorker against a pool of 3 with probabilities [0.5, 0.5, 0]: seat 1 of every row is SepmcPolicy(models[opponent]),
    the opponent column holds the statement's draw at every game start and stays constant within a game, model 2 never plays."""
    import torch
    from lifelike_agility_and_play_b200 import _capi as capi
    from lifelike_agility_and_play_b200.model.compile_model import load_model_blob
    from lifelike_agility_and_play_b200.parallel import SepmcRolloutWorker, sepmc_slab_records
    from lifelike_agility_and_play_b200.parallel.trajectory import SCOL_ACTION, SCOL_CODE, SCOL_DONE, SCOL_OPPONENT, SCOL_REWARD, SCOL_VALUE
    from lifelike_agility_and_play_b200.policy_epmc import DeviceOpponentPool, DeviceSepmcTrainPolicy, SepmcPolicy, random_weights
    from lifelike_agility_and_play_b200.sim_envs.playground_env import INIT_STATE_RUN_0
    import strategic_train_cases as sc
    P, T, seed, gid0 = 20, 5, 77, 1000
    n = 2 * P
    w = random_weights(True, 4)
    opp_w = [[a.copy() for a in models[k]] for k in range(3)]
    for x in [w] + opp_w:
        x[149] = (0.05 * x[149]).astype(np.float32)                    # small actions: the robots stay up for a while
    pol = DeviceSepmcTrainPolicy(w, device=0)
    pool = DeviceOpponentPool(opp_w, device=0, max_rows=P, probs=[0.5, 0.5, 0.0])
    host, host_opp = SepmcPolicy(w), [SepmcPolicy(x) for x in opp_w]
    cfg = dict(kp=50.0, kd=0.5, max_tau=16.0, ground_friction=1.0, max_steps=4, seed=5, friction_hi=1.0, env_kind=capi.ENV_SEPMC,
               auto_reset=1, global_env_offset=gid0)
    lib, blob = capi.load_cuda_library(), load_model_blob()
    eng, chk = capi.VecEngine(lib, n, blob, None, device=0, **cfg), capi.VecEngine(lib, n, blob, None, device=0, **cfg)
    for e in (eng, chk):
        e.set_init_state(INIT_STATE_RUN_0)
    small = DeviceOpponentPool(opp_w, device=0, max_rows=P - 1)
    with pytest.raises(ValueError, match="max_rows"):
        SepmcRolloutWorker(eng, pol, small, T, "cuda:0")
    small.close()
    worker = SepmcRolloutWorker(eng, pol, pool, T, "cuda:0", seed=seed)
    o0 = eng.reset()
    assert np.array_equal(o0, chk.reset())
    worker.start(o0)
    unrolls = []
    for _ in range(2):
        for _ in range(T):
            worker.step()
        u = worker.finish_unroll()
        worker.wait()
        unrolls.append([x.clone() for x in u])
    torch.cuda.synchronize()
    pair_gid = gid0 // 2 + np.arange(P)
    t_cut = oc.cutoffs([0.5, 0.5, 0.0])
    obs, mask, n_code, starts = o0, np.ones(P, np.float32), 0, 0
    s_opp, opp = np.zeros((P, 128), np.float32), np.full(P, -7, np.int64)
    for k, (slab_t, init, first, boot) in enumerate(unrolls):
        slab = slab_t.cpu().numpy()
        s_pol, s_val = init.cpu().numpy()[:, :128], init.cpu().numpy()[:, 128:]
        for t in range(T):
            calls = k * T + t
            assert np.array_equal(slab[t, :, :965], obs)
            rec_opp = slab[t, 0::2, SCOL_OPPONENT]
            new = mask != 0
            want = opp.copy()
            want[new] = oc.pick(oc.draw_words(pair_gid[new], seed, calls), t_cut)
            starts += int(new.sum())
            assert np.array_equal(rec_opp, want.astype(np.float32)), (k, t, rec_opp, want)
            opp = want
            assert (slab[t, 1::2, SCOL_OPPONENT] == 0).all()
            a = slab[t, :, SCOL_ACTION:SCOL_ACTION + 12]
            code = slab[t, :, SCOL_CODE].astype(np.int64)
            for m in np.unique(opp):
                rows = np.flatnonzero(opp == m)
                a1, s1, _, c1 = host_opp[m].act(obs[1::2][rows], s_opp[rows], mask[rows], return_aux=True)
                s_opp[rows] = s1
                same1 = c1 == code[1::2][rows]
                n_code += int(same1.sum())
                assert np.abs(a[1::2][rows][same1] - a1[same1]).max(initial=0) < 1e-4, "seat 1 is not its model's forward"
            eps_ref = sc.eps_of(pair_gid, seed, calls)
            a0, s_pol, h0, c0, nlp0 = host.act(obs[0::2], s_pol, mask, return_aux=True, eps=eps_ref, return_neglogp=True)
            same = c0 == code[0::2]
            n_code += int(same.sum())
            assert np.abs(a[0::2][same] - a0[same]).max(initial=0) < 1e-4
            v_h, s_val = host.value(obs[0::2], s_val, mask)
            assert np.abs(slab[t, 0::2, SCOL_VALUE] - v_h).max() < 1e-4 * (1 + np.abs(v_h).max())
            obs, rew, done = chk.step(a)
            assert np.array_equal(rew, slab[t, :, SCOL_REWARD]) and np.array_equal(done.astype(np.float32), slab[t, :, SCOL_DONE])
            mask = done[0::2].astype(np.float32)
        rec = sepmc_slab_records(slab_t, init, first, boot, with_opponent=True)
        assert list(rec)[-1] == "opponent" and rec["opponent"].dtype == torch.int64
        assert np.array_equal(rec["opponent"].cpu().numpy(), slab[:, 0::2, SCOL_OPPONENT].astype(np.int64))
    assert n_code >= 0.99 * 4 * T * P, (n_code, 4 * T * P)
    assert starts > P, "no game restarted inside the run: the redraws are not exercised"
    worker.set_opponent_probs([0.0, 1.0, 0.0])
    pol.close(); pool.close(); eng.close(); chk.close()
