"""The environmental level's training forward (llq_hier_policy_forward_rec) against the fp64 statement of tests/hier_train_cases.py row
by row, its batch edges, its recurrence, and the recurrent rollout worker against a host-driven replay (run with -m gpu on an H100).

Every row of the designed batch is decisive at both of its counters, so sampled codes must be exactly equal, and V, -log p, actions and
both state halves within kappa S + 2^-23 |ref| (kappa = KAPPA_HIER = 20).  The printed ratio is the largest (|err| - 2^-23 |ref|) / S
per output: the kappa the test needs.  Largest ratios measured on an H100 80GB HBM3 at a 700 W power limit: V 4.74, -log p 2.44,
actions 9.63, state 3.54.
"""
import numpy as np
import pytest

import hier_train_cases as hc
import policy_cases as pc

pytestmark = pytest.mark.gpu

CANARY = 0x7FBADBAD
RATIOS = {}


def _canary(torch, shape, dtype=None):
    t = torch.full(shape, CANARY, dtype=torch.int32, device="cuda")
    return t if dtype is torch.int32 else t.view(torch.float32)


def _bits(t):
    import torch
    return t.view(torch.int32).cpu().numpy() if t.dtype == torch.float32 else t.cpu().numpy()


def _check(name, got, ref, S):
    got = np.asarray(got, np.float64)
    err = np.abs(got - ref)
    slack = err - pc.U * np.abs(ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(slack > 0, slack / S, 0.0)
    RATIOS[name] = max(RATIOS.get(name, 0.0), float(np.nanmax(ratio)) if ratio.size else 0.0)
    bad = np.argwhere(~(err <= hc.KAPPA * S + pc.U * np.abs(ref)))
    assert len(bad) == 0, (name, [(tuple(int(j) for j in b), float(got[tuple(b)]), float(ref[tuple(b)]), float(S[tuple(b)])) for b in bad[:8]])


@pytest.fixture(scope="module")
def case(built):
    from lifelike_agility_and_play_b200.policy_epmc import DeviceHierPolicy
    w, obs, state, done, counters, info, evals = hc.train_case()
    dev = DeviceHierPolicy(w, device=0, train=True)
    yield w, obs, state, done, counters, info, evals, dev
    dev.close()
    print("training forward kappa needed: %s" % {k: "%.3g" % v for k, v in RATIOS.items()})


def _run(torch, dev, obs, obs_ld, out_ld, n, state, done, counter, gid0=hc.ROW_GID0):
    """One forward_rec on the first n rows with canary outputs (8 rows past n); returns (actions, codes, values, neglogp, state)."""
    t_obs = torch.from_numpy(pc.padded(obs[:n], obs_ld, 916)).cuda()
    st = _canary(torch, (n + 8, 128))
    st[:n] = torch.from_numpy(np.ascontiguousarray(state[:n])).cuda()
    t_done = None if done is None else torch.from_numpy(np.ascontiguousarray(done[:n])).cuda()
    act, codes = _canary(torch, (n + 8, 12)), _canary(torch, (n + 8,), torch.int32)
    val, nlp = _canary(torch, ((n + 8) * out_ld,)), _canary(torch, ((n + 8) * out_ld,))
    dev.forward_rec(t_obs.data_ptr(), obs_ld, n, t_done.data_ptr() if t_done is not None else None, st.data_ptr(), act.data_ptr(),
                    codes.data_ptr(), val.data_ptr(), nlp.data_ptr(), out_ld, hc.SEED, counter, gid0)
    torch.cuda.synchronize()
    return act, codes, val, nlp, st


def _compare(n, out_ld, ref, S, act, codes, val, nlp, st):
    got = codes.cpu().numpy()
    assert np.array_equal(got[:n], ref["code"][:n]), np.flatnonzero(got[:n] != ref["code"][:n])[:10]
    v, lp = val.cpu().numpy(), nlp.cpu().numpy()
    _check("value", v[:n * out_ld:out_ld], ref["value"][:n], S["value"][:n])
    _check("-log p", lp[:n * out_ld:out_ld], ref["neglogp"][:n], S["neglogp"][:n])
    _check("actions", act.cpu().numpy()[:n], ref["actions"][:n], S["actions"][:n])
    _check("state", st.cpu().numpy()[:n], ref["state"][:n], S["state"][:n])
    owned = np.zeros(len(v), bool)
    owned[:n * out_ld:out_ld] = True
    for name, t, keep in (("codes", codes, slice(n, None)), ("actions", act, slice(n, None)), ("state", st, slice(n, None))):
        assert (_bits(t)[keep] == CANARY).all(), (name, "rows past n written")
    for name, t in (("values", val), ("neglogp", nlp)):
        assert (_bits(t)[~owned] == CANARY).all(), (name, "written outside rows i * out_ld, i < n")


@pytest.mark.parametrize("lds", [(916, 1), (917, 3), (1024, 936)], ids=["916-1", "917-3", "1024-936"])
@pytest.mark.parametrize("n", [1, 7, 8, 9, 300, 1059])
def test_training_forward_matches_the_fp64_statement(case, n, lds):
    import torch
    w, obs, state, done, counters, info, evals, dev = case
    obs_ld, out_ld = lds
    for counter, (ref, S) in zip(counters, evals):
        _compare(n, out_ld, ref, S, *_run(torch, dev, obs, obs_ld, out_ld, n, state, done, counter))


def test_record_slab_and_shards(case):
    """forward_rec into the value / -log p columns of a [n, 936] slab whose observation is read in place: every other column and every
    row past n stays bit for bit; a shard launched on rows k.. with row_gid0 + k reproduces those rows bit for bit."""
    import torch
    from lifelike_agility_and_play_b200.parallel.trajectory import HCOL_NEGLOGP, HCOL_VALUE, HIER_TRAJ_WIDTH as W
    w, obs, state, done, counters, info, evals, dev = case
    n = hc.N
    init = np.full((n + 8, W), 0, np.int32)
    init[:] = CANARY
    init = init.view(np.float32)
    init[:n, :916] = obs
    runs = []
    for first in (0, 45, 64):
        slab = torch.from_numpy(init.copy()).cuda()
        st = torch.from_numpy(np.ascontiguousarray(state)).cuda()
        act, codes = _canary(torch, (n + 8, 12)), _canary(torch, (n + 8,), torch.int32)
        t_done = torch.from_numpy(done).cuda()
        row = slab.data_ptr() + first * W * 4
        dev.forward_rec(row, W, n - first, t_done.data_ptr() + first, st.data_ptr() + first * 512, act.data_ptr() + first * 48,
                        codes.data_ptr() + first * 4, row + HCOL_VALUE * 4, row + HCOL_NEGLOGP * 4, W, hc.SEED, counters[0], hc.ROW_GID0 + first)
        torch.cuda.synchronize()
        runs.append((first, [_bits(x) for x in (slab, act, codes, st)]))
    ref, S = evals[0]
    s0 = runs[0][1][0].view(np.float32)
    _check("value", s0[:n, HCOL_VALUE], ref["value"], S["value"])
    _check("-log p", s0[:n, HCOL_NEGLOGP], ref["neglogp"], S["neglogp"])
    written = np.zeros(init.shape, bool)
    written[:n, [HCOL_VALUE, HCOL_NEGLOGP]] = True
    assert np.array_equal(runs[0][1][0][~written], init.view(np.int32)[~written])
    for first, outs in runs[1:]:
        for name, a, b in zip(("slab", "actions", "codes", "state"), outs, runs[0][1]):
            assert np.array_equal(a[first:], b[first:]), (name, first)
        assert np.array_equal(outs[0][:first], init.view(np.int32)[:first])


@pytest.mark.parametrize("shift", [8, 1])
def test_rows_do_not_depend_on_their_place_in_the_batch(case, shift):
    import torch
    w, obs, state, done, counters, info, evals, dev = case
    n = hc.N
    out = []
    for s in (0, shift):
        o = np.concatenate([obs[n - s:], obs]) if s else obs
        st = np.concatenate([state[n - s:], state]) if s else state
        d = np.concatenate([done[n - s:], done]) if s else done
        r = _run(torch, dev, o, 916, 1, len(o), st, d, counters[1], hc.ROW_GID0 - s)
        out.append([_bits(x)[s:s + n] for x in r])
    for name, a, b in zip(("actions", "codes", "values", "neglogp", "state"), *out):
        assert np.array_equal(a, b), (name, shift, int((a != b).sum()))


def test_recurrence(case):
    """Four steps from a non-zero state of both LSTMs, done bytes 0, 1, 2 and 255 (every non-zero byte wipes both halves) and
    d_done = NULL on one step; each step's reference starts from the kernel's incoming state."""
    import torch
    w, obs, state, done, counters, info, evals, dev = case
    state0, obs_all, done_all, ctrs = hc.recurrence_case(w)
    n = len(state0)
    st_in = state0
    for step, (o, d, c) in enumerate(zip(obs_all, done_all, ctrs)):
        d_use = None if step == hc.NULL_DONE_STEP else d
        ref, S = hc.train_eval(hc.Trunks(w, o, st_in, d_use if d_use is not None else np.zeros(n, np.uint8)),
                               hc.uniforms(hc.ROW_GID0 + np.arange(n), hc.SEED, c))
        assert hc.decisive(ref, S).all(), "a recurrence row is not decisive from the kernel's state"
        act, codes, val, nlp, st = _run(torch, dev, o, 916, 1, n, st_in, d_use, c)
        _compare(n, 1, ref, S, act, codes, val, nlp, st)
        if step == 0:
            assert set(np.unique(d).tolist()) == {0, 1, 2, 255} and (np.abs(st_in[d != 0][:, :64]) > 0).any(1).all()
            assert (np.abs(st_in[d != 0][:, 64:]) > 0).any(1).all()
        st_in = st.cpu().numpy()[:n].copy()


def test_training_handle_entry_points(built):
    import torch
    from lifelike_agility_and_play_b200.policy_epmc import DeviceHierPolicy, random_weights
    with pytest.raises(RuntimeError, match="environmental level only"):
        DeviceHierPolicy(random_weights(True, 0), device=0, train=True)
    tr, det = DeviceHierPolicy(random_weights(False, 0), device=0, train=True), DeviceHierPolicy(random_weights(False, 0), device=0)
    assert tr.state_dim == 128 and det.state_dim == 64
    obs, st, act = torch.zeros((8, 916), device="cuda"), torch.zeros((8, 128), device="cuda"), torch.zeros((8, 12), device="cuda")
    with pytest.raises(RuntimeError, match="forward_rec"):
        tr.forward(obs.data_ptr(), 916, 8, None, st.data_ptr(), act.data_ptr())
    with pytest.raises(RuntimeError, match="not a training handle"):
        det.forward_rec(obs.data_ptr(), 916, 8, None, st.data_ptr(), act.data_ptr(), None, None, None, 1, 0, 0)
    tr.close(); det.close()


@pytest.mark.parametrize("element", [0, 3])
def test_worker_against_a_replay(built, element):
    """HierRolloutWorker (training forward -> fused step, slab rows written in place, two unrolls) against a second engine driven
    through the host API with the slab's own action columns."""
    import torch
    from lifelike_agility_and_play_b200 import _capi as capi
    from lifelike_agility_and_play_b200.model.compile_model import load_model_blob
    from lifelike_agility_and_play_b200.parallel import HierRolloutWorker, hier_slab_records
    from lifelike_agility_and_play_b200.parallel.trajectory import HCOL_ACTION, HCOL_CODE, HCOL_DONE, HCOL_NEGLOGP, HCOL_REWARD, HCOL_VALUE
    from lifelike_agility_and_play_b200.policy_epmc import DeviceHierPolicy, EpmcPolicy, random_weights
    from lifelike_agility_and_play_b200.sim_envs.playground_env import INIT_STATE_RUN_0
    n, T, seed, gid0 = 40, 5, 77, 1000
    w = random_weights(False, 4)
    w[99] = (0.05 * w[99]).astype(np.float32)                  # small actions: the robots stay up for a while
    pol, host = DeviceHierPolicy(w, device=0, train=True), EpmcPolicy(w)
    cfg = dict(kp=50.0, kd=0.5, max_tau=16.0, ground_friction=1.0, max_steps=7, seed=5, friction_hi=1.0, env_kind=capi.ENV_EPMC,
               element_id=element, cmd_freq_lo=25, cmd_freq_hi=40, auto_reset=1, global_env_offset=gid0)
    lib, blob = capi.load_cuda_library(), load_model_blob()
    eng, chk = capi.VecEngine(lib, n, blob, None, device=0, **cfg), capi.VecEngine(lib, n, blob, None, device=0, **cfg)
    for e in (eng, chk):
        e.set_init_state(INIT_STATE_RUN_0)
    worker = HierRolloutWorker(eng, pol, T, "cuda:0", seed=seed)
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
    obs, mask, n_code = o0, np.ones(n, np.float32), 0
    for k, (slab_t, init, first, boot) in enumerate(unrolls):
        slab = slab_t.cpu().numpy()
        init, first = init.cpu().numpy(), first.cpu().numpy()
        if k == 0:
            assert (init == 0).all() and (first == 1).all()
        else:
            assert np.array_equal(first.astype(np.float32), prev_slab[T - 1, :, HCOL_DONE])
            assert np.abs(init - np.concatenate([s_code, s_val], axis=1)).max() < 1e-4     # the host chain's state at the unroll boundary
            assert np.array_equal(boots_prev, slab[0, :, HCOL_VALUE].view(np.int32)), "bootstrap differs from the next forward's V"
        s_code, s_val = init[:, :64], init[:, 64:]               # the host chain restarts from the device's state
        for t in range(T):
            assert np.array_equal(slab[t, :, :916], obs), "record %d does not hold the observation the action was computed from" % t
            a = slab[t, :, HCOL_ACTION:HCOL_ACTION + 12]
            code = slab[t, :, HCOL_CODE].astype(np.int64)
            u = hc.uniforms(gid0 + np.arange(n), seed, k * T + t)
            a_h, s_code, c_h, nlp_h = host.act(obs, s_code, mask, return_code=True, uniforms=u, return_neglogp=True)
            v_h, s_val = host.value(obs, s_val, mask)
            same = c_h == code
            n_code += int(same.sum())
            assert np.abs(a[same] - a_h[same]).max(initial=0) < 1e-4, "the action is not the decoder's on the recorded code"
            assert np.abs(slab[t, same, HCOL_NEGLOGP] - nlp_h[same]).max(initial=0) < 1e-3
            assert np.abs(slab[t, :, HCOL_VALUE] - v_h).max() < 1e-4 * (1 + np.abs(v_h).max())
            obs, rew, done = chk.step(a)
            assert np.array_equal(rew, slab[t, :, HCOL_REWARD]) and np.array_equal(done.astype(np.float32), slab[t, :, HCOL_DONE])
            mask = done.astype(np.float32)
        rec = hier_slab_records(slab_t, unrolls[k][1], unrolls[k][2], unrolls[k][3])
        assert tuple(rec["A_Z"].shape) == (T, n) and np.array_equal(rec["M"][0].cpu().numpy(), first.astype(np.float32))
        assert np.array_equal(rec["M"][1:].cpu().numpy(), slab[:-1, :, HCOL_DONE])
        prev_slab, boots_prev = slab, boot.cpu().numpy().view(np.int32)
    assert n_code >= 0.99 * 2 * T * n, (n_code, 2 * T * n)
    assert (prev_slab[:, :, HCOL_DONE] == 1).any(), "no episode ended: the wipes are not exercised"
    pol.close(); eng.close(); chk.close()
