"""The strategic level's training forward (llq_hier_policy_forward_rec_strategic) against the fp64 statement of
tests/strategic_train_cases.py row by row, its batch edges, its recurrence, its refusals, and the chase-tag rollout worker against a
host-driven replay (run with -m gpu on an H100).

Every row of the designed batch is decisive at both of its counters, so codes must be exactly equal, and the raw heading, V, -log p,
actions and all three state parts within kappa S + 2^-23 |ref| (kappa = KAPPA_HIER = 20).  The printed ratio is the largest
(|err| - 2^-23 |ref|) / S per output: the kappa the test needs.
"""
import numpy as np
import pytest

import policy_cases as pc
import strategic_train_cases as sc

pytestmark = pytest.mark.gpu

CANARY = 0x7FBADBAD
RATIOS = {}
OUTS = ("heading", "values", "neglogp")


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
    bad = np.argwhere(~(err <= sc.KAPPA * S + pc.U * np.abs(ref)))
    assert len(bad) == 0, (name, [(tuple(int(j) for j in b), float(got[tuple(b)]), float(ref[tuple(b)]), float(S[tuple(b)])) for b in bad[:8]])


@pytest.fixture(scope="module")
def case(built):
    from lifelike_agility_and_play_b200.policy_epmc import DeviceSepmcTrainPolicy
    w, obs, state, done, counters, info, evals, mean_codes = sc.train_case()
    dev = DeviceSepmcTrainPolicy(w, device=0)
    yield w, obs, state, done, counters, info, evals, dev
    dev.close()
    print("strategic training forward kappa needed: %s" % {k: "%.3g" % v for k, v in RATIOS.items()})


def _run(torch, dev, obs, obs_ld, out_ld, n, state, done, counter, gid0=sc.ROW_GID0):
    """One forward_rec on the first n rows with canary outputs (8 rows past n); returns (actions, codes, heading, values, neglogp, state)."""
    t_obs = torch.from_numpy(pc.padded(obs[:n], obs_ld, 965)).cuda()
    st = _canary(torch, (n + 8, 192))
    st[:n] = torch.from_numpy(np.ascontiguousarray(state[:n])).cuda()
    t_done = None if done is None else torch.from_numpy(np.ascontiguousarray(done[:n])).cuda()
    act, codes = _canary(torch, (n + 8, 12)), _canary(torch, (n + 8,), torch.int32)
    hd, val, nlp = (_canary(torch, ((n + 8) * out_ld,)) for _ in range(3))
    dev.forward_rec(t_obs.data_ptr(), obs_ld, n, t_done.data_ptr() if t_done is not None else None, st.data_ptr(), act.data_ptr(),
                    codes.data_ptr(), hd.data_ptr(), val.data_ptr(), nlp.data_ptr(), out_ld, sc.SEED, counter, gid0)
    torch.cuda.synchronize()
    return act, codes, hd, val, nlp, st


def _compare(n, out_ld, ref, S, act, codes, hd, val, nlp, st):
    got = codes.cpu().numpy()
    assert np.array_equal(got[:n], ref["code"][:n]), np.flatnonzero(got[:n] != ref["code"][:n])[:10]
    for name, t, key in (("heading", hd, "heading"), ("value", val, "value"), ("-log p", nlp, "neglogp")):
        _check(name, t.cpu().numpy()[:n * out_ld:out_ld], ref[key][:n], S[key][:n])
    _check("actions", act.cpu().numpy()[:n], ref["actions"][:n], S["actions"][:n])
    s = st.cpu().numpy()[:n]
    for name, k in (("state heading", 0), ("state code", 64), ("state value", 128)):
        _check(name, s[:, k:k + 64], ref["state"][:n, k:k + 64], S["state"][:n, k:k + 64])
    owned = np.zeros(len(val), bool)
    owned[:n * out_ld:out_ld] = True
    for name, t in (("codes", codes), ("actions", act), ("state", st)):
        assert (_bits(t)[n:] == CANARY).all(), (name, "rows past n written")
    for name, t in zip(OUTS, (hd, val, nlp)):
        assert (_bits(t)[~owned] == CANARY).all(), (name, "written outside rows i * out_ld, i < n")


@pytest.mark.parametrize("lds", [(965, 1), (966, 3), (1968, 1968)], ids=["965-1", "966-3", "seat-1968"])
@pytest.mark.parametrize("n", [1, 7, 8, 9, 300, 1059])
def test_strategic_training_forward_matches_the_fp64_statement(case, n, lds):
    import torch
    w, obs, state, done, counters, info, evals, dev = case
    obs_ld, out_ld = lds
    for counter, (ref, S) in zip(counters, evals):
        _compare(n, out_ld, ref, S, *_run(torch, dev, obs, obs_ld, out_ld, n, state, done, counter))


def test_record_slab_and_shards(case):
    """forward_rec_strategic into the heading / value / -log p columns of a [n, 984] slab whose observation is read in place: every
    other column and every row past n stays bit for bit; a shard launched on rows k.. with row_gid0 + k reproduces those rows."""
    import torch
    from lifelike_agility_and_play_b200.parallel.trajectory import SCOL_HEADING, SCOL_NEGLOGP, SCOL_VALUE, SEPMC_TRAJ_WIDTH as W
    w, obs, state, done, counters, info, evals, dev = case
    n = sc.N
    init = np.full((n + 8, W), CANARY, np.int32).view(np.float32)
    init[:n, :965] = obs
    runs = []
    for first in (0, 45, 64):
        slab = torch.from_numpy(init.copy()).cuda()
        st = torch.from_numpy(np.ascontiguousarray(state)).cuda()
        act, codes = _canary(torch, (n + 8, 12)), _canary(torch, (n + 8,), torch.int32)
        t_done = torch.from_numpy(done).cuda()
        row = slab.data_ptr() + first * W * 4
        dev.forward_rec(row, W, n - first, t_done.data_ptr() + first, st.data_ptr() + first * 768, act.data_ptr() + first * 48,
                        codes.data_ptr() + first * 4, row + SCOL_HEADING * 4, row + SCOL_VALUE * 4, row + SCOL_NEGLOGP * 4, W, sc.SEED,
                        counters[0], sc.ROW_GID0 + first)
        torch.cuda.synchronize()
        runs.append((first, [_bits(x) for x in (slab, act, codes, st)]))
    ref, S = evals[0]
    s0 = runs[0][1][0].view(np.float32)
    _check("heading", s0[:n, SCOL_HEADING], ref["heading"], S["heading"])
    _check("value", s0[:n, SCOL_VALUE], ref["value"], S["value"])
    _check("-log p", s0[:n, SCOL_NEGLOGP], ref["neglogp"], S["neglogp"])
    written = np.zeros(init.shape, bool)
    written[:n, [SCOL_HEADING, SCOL_VALUE, SCOL_NEGLOGP]] = True
    assert np.array_equal(runs[0][1][0][~written], init.view(np.int32)[~written])
    for first, outs in runs[1:]:
        for name, a, b in zip(("slab", "actions", "codes", "state"), outs, runs[0][1]):
            assert np.array_equal(a[first:], b[first:]), (name, first)
        assert np.array_equal(outs[0][:first], init.view(np.int32)[:first])


@pytest.mark.parametrize("shift", [8, 1])
def test_rows_do_not_depend_on_their_place_in_the_batch(case, shift):
    import torch
    w, obs, state, done, counters, info, evals, dev = case
    n = sc.N
    out = []
    for s in (0, shift):
        o = np.concatenate([obs[n - s:], obs]) if s else obs
        st = np.concatenate([state[n - s:], state]) if s else state
        d = np.concatenate([done[n - s:], done]) if s else done
        r = _run(torch, dev, o, 965, 1, len(o), st, d, counters[1], sc.ROW_GID0 - s)
        out.append([_bits(x)[s:s + n] for x in r])
    for name, a, b in zip(("actions", "codes", "heading", "values", "neglogp", "state"), *out):
        assert np.array_equal(a, b), (name, shift, int((a != b).sum()))


def test_recurrence(case):
    """Four steps from a non-zero state of all three LSTMs, done bytes 0, 1, 2 and 255 (every non-zero byte wipes all three) and
    d_done = NULL on one step; each step's reference starts from the kernel's incoming state."""
    import torch
    w, obs, state, done, counters, info, evals, dev = case
    state0, obs_all, done_all, ctrs = sc.recurrence_case(w)
    n = len(state0)
    gid = sc.ROW_GID0 + np.arange(n)
    st_in = state0
    for step, (o, d, c) in enumerate(zip(obs_all, done_all, ctrs)):
        d_use = None if step == sc.NULL_DONE_STEP else d
        ref, S = sc.train_eval(sc.Trunks(w, o, st_in, d_use if d_use is not None else np.zeros(n, np.uint8)), gid, sc.SEED, c)
        assert sc.decisive(ref, S).all(), "a recurrence row is not decisive from the kernel's state"
        out = _run(torch, dev, o, 965, 1, n, st_in, d_use, c)
        _compare(n, 1, ref, S, *out)
        if step == 0:
            assert set(np.unique(d).tolist()) == {0, 1, 2, 255}
            for k in (0, 64, 128):
                assert (np.abs(st_in[d != 0][:, k:k + 64]) > 0).any(1).all()
        st_in = out[5].cpu().numpy()[:n].copy()


def test_strategic_training_handle_entry_points(built):
    import ctypes as C
    import torch
    from lifelike_agility_and_play_b200.policy_epmc import DeviceHierPolicy, DeviceSepmcTrainPolicy, random_weights
    with pytest.raises(RuntimeError, match="environmental level only"):
        DeviceHierPolicy(random_weights(True, 0), device=0, train=True)
    with pytest.raises(RuntimeError, match="llq_hier_policy_create_train_strategic"):
        DeviceHierPolicy(random_weights(True, 0), device=0, train=True)
    tr, det = DeviceSepmcTrainPolicy(random_weights(True, 0), device=0), DeviceHierPolicy(random_weights(True, 0), device=0)
    env_tr = DeviceHierPolicy(random_weights(False, 0), device=0, train=True)
    assert tr.state_dim == 192 and det.state_dim == 128
    obs, st, act = torch.zeros((8, 984), device="cuda"), torch.zeros((8, 192), device="cuda"), torch.zeros((8, 12), device="cuda")
    with pytest.raises(RuntimeError, match="forward_rec_strategic"):
        tr.forward(obs.data_ptr(), 965, 8, None, st.data_ptr(), act.data_ptr())
    with pytest.raises(RuntimeError, match="forward_rec_strategic"):
        DeviceHierPolicy.forward_rec(tr, obs.data_ptr(), 965, 8, None, st.data_ptr(), act.data_ptr(), None, None, None, 1, 0, 0)
    for other in (det, env_tr):
        with pytest.raises(RuntimeError, match="not a strategic training handle"):
            DeviceSepmcTrainPolicy.forward_rec(other, obs.data_ptr(), 965, 8, None, st.data_ptr(), act.data_ptr(), None, None, None, None, 1, 0, 0)
    with pytest.raises(RuntimeError, match="row stride"):
        tr.forward_rec(obs.data_ptr(), 964, 8, None, st.data_ptr(), act.data_ptr(), None, None, None, None, 1, 0, 0)
    # the table lengths are checked before anything reaches the device
    lib, h = tr.lib, C.c_void_p()
    blob, off = np.zeros(16, np.float32), np.zeros(101, np.int32)
    rc = lib.llq_hier_policy_create_train_strategic(blob.ctypes.data_as(C.c_void_p), C.c_int64(16), off.ctypes.data_as(C.c_void_p), C.c_int32(101),
                                                    off.ctypes.data_as(C.c_void_p), C.c_int32(45), C.c_int32(0), C.byref(h))
    assert rc != 0 and b"wrong length" in lib.llq_hier_policy_last_error()
    tr.close(); det.close(); env_tr.close()


def test_worker_against_a_replay(built):
    """SepmcRolloutWorker (training forward on seat 0, the frozen opponent's forward on seat 1, copies, fused step; two unrolls) against
    a second engine driven through the host API with the slab's own action columns."""
    import torch
    from lifelike_agility_and_play_b200 import _capi as capi
    from lifelike_agility_and_play_b200.model.compile_model import load_model_blob
    from lifelike_agility_and_play_b200.parallel import SepmcRolloutWorker, sepmc_slab_records
    from lifelike_agility_and_play_b200.parallel.trajectory import (SCOL_ACTION, SCOL_CODE, SCOL_DONE, SCOL_HEADING, SCOL_NEGLOGP, SCOL_REWARD,
                                                                    SCOL_VALUE)
    from lifelike_agility_and_play_b200.policy_epmc import DeviceHierPolicy, DeviceSepmcTrainPolicy, SepmcPolicy, random_weights
    from lifelike_agility_and_play_b200.sim_envs.playground_env import INIT_STATE_RUN_0
    P, T, seed, gid0 = 20, 5, 77, 1000
    n = 2 * P
    w, wo = random_weights(True, 4), random_weights(True, 5)
    for x in (w, wo):
        x[149] = (0.05 * x[149]).astype(np.float32)            # small actions: the robots stay up for a while
    pol, opp = DeviceSepmcTrainPolicy(w, device=0), DeviceHierPolicy(wo, device=0)
    host, host_opp = SepmcPolicy(w), SepmcPolicy(wo)
    cfg = dict(kp=50.0, kd=0.5, max_tau=16.0, ground_friction=1.0, max_steps=7, seed=5, friction_hi=1.0, env_kind=capi.ENV_SEPMC,
               auto_reset=1, global_env_offset=gid0)
    lib, blob = capi.load_cuda_library(), load_model_blob()
    eng, chk = capi.VecEngine(lib, n, blob, None, device=0, **cfg), capi.VecEngine(lib, n, blob, None, device=0, **cfg)
    for e in (eng, chk):
        e.set_init_state(INIT_STATE_RUN_0)
    with pytest.raises(ValueError):
        SepmcRolloutWorker(eng, opp, opp, T, "cuda:0")
    with pytest.raises(ValueError):
        SepmcRolloutWorker(eng, pol, pol, T, "cuda:0")
    worker = SepmcRolloutWorker(eng, pol, opp, T, "cuda:0", seed=seed)
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
    obs, mask, n_code = o0, np.ones(P, np.float32), 0
    s_opp = np.zeros((P, 128), np.float32)
    for k, (slab_t, init, first, boot) in enumerate(unrolls):
        slab = slab_t.cpu().numpy()
        init, first = init.cpu().numpy(), first.cpu().numpy()
        if k == 0:
            assert (init == 0).all() and (first == 1).all()
        else:
            assert np.array_equal(first.astype(np.float32), prev_slab[T - 1, 0::2, SCOL_DONE])
            assert np.abs(init - np.concatenate([s_pol, s_val], axis=1)).max() < 1e-4     # the host chain's state at the unroll boundary
            assert np.array_equal(boots_prev, slab[0, 0::2, SCOL_VALUE].view(np.int32)), "bootstrap differs from the next forward's V"
        s_pol, s_val = init[:, :128], init[:, 128:]              # the host chain restarts from the device's state
        for t in range(T):
            assert np.array_equal(slab[t, :, :965], obs), "record %d does not hold the observation the action was computed from" % t
            a = slab[t, :, SCOL_ACTION:SCOL_ACTION + 12]
            code = slab[t, :, SCOL_CODE].astype(np.int64)
            # seat 1: a replay of the opponent's deterministic forward
            a1, s_opp, _, c1 = host_opp.act(obs[1::2], s_opp, mask, return_aux=True)
            same1 = c1 == code[1::2]
            n_code += int(same1.sum())
            assert np.abs(a[1::2][same1] - a1[same1]).max(initial=0) < 1e-4, "seat 1 is not the opponent's forward"
            assert (slab[t, 1::2, [SCOL_VALUE, SCOL_NEGLOGP, SCOL_HEADING]] == 0).all()
            # seat 0: the decoder on the code of the recorded heading; -log p of the recorded heading; V of the value tower
            head = slab[t, 0::2, SCOL_HEADING]
            eps_ref = sc.eps_of(pair_gid, seed, k * T + t)
            a0, s_pol, h0, c0, nlp0 = host.act(obs[0::2], s_pol, mask, return_aux=True, eps=eps_ref, return_neglogp=True)
            assert np.abs(h0 - head).max() < 1e-4 * (1 + np.abs(head).max()), "recorded heading is not mean + exp(logstd) eps"
            same = c0 == code[0::2]
            n_code += int(same.sum())
            assert np.abs(a[0::2][same] - a0[same]).max(initial=0) < 1e-4, "the action is not the decoder's on the recorded heading's code"
            assert np.abs(slab[t, 0::2, SCOL_NEGLOGP] - nlp0).max() < 1e-4
            v_h, s_val = host.value(obs[0::2], s_val, mask)
            assert np.abs(slab[t, 0::2, SCOL_VALUE] - v_h).max() < 1e-4 * (1 + np.abs(v_h).max())
            obs, rew, done = chk.step(a)
            assert np.array_equal(rew, slab[t, :, SCOL_REWARD]) and np.array_equal(done.astype(np.float32), slab[t, :, SCOL_DONE])
            mask = done[0::2].astype(np.float32)
            assert np.array_equal(done[0::2], done[1::2])
        rec = sepmc_slab_records(slab_t, unrolls[k][1], unrolls[k][2], unrolls[k][3])
        assert tuple(rec["A_HLC"].shape) == (T, P) and np.array_equal(rec["M"][0].cpu().numpy(), first.astype(np.float32))
        assert np.array_equal(rec["M"][1:].cpu().numpy(), slab[:-1, 0::2, SCOL_DONE])
        prev_slab, boots_prev = slab, boot.cpu().numpy().view(np.int32)
    assert n_code >= 0.99 * 4 * T * P, (n_code, 4 * T * P)
    assert (prev_slab[:, :, SCOL_DONE] == 1).any(), "no game ended: the wipes are not exercised"
    pol.close(); opp.close(); eng.close(); chk.close()
