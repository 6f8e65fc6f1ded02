"""Model refresh on the GPU (run with -m gpu on an H100): a refreshed handle against fresh handles of the same weights bit for bit, at every
level and for both sources; the stream ordering of refreshes queued behind a sleeping stream with no synchronisation; pool slots; the
three rollout workers refreshed in the middle of an unroll against host-driven replays."""
import ctypes as C

import numpy as np
import pytest

import hier_train_cases as hc
import policy_cases as pc
import strategic_train_cases as sc

pytestmark = pytest.mark.gpu

SEED, COUNTER, GID0 = 0x1234_5678_9ABC, 7, 1000
SLEEP = int(3e8)                          # GPU cycles the stream sleeps before its first forward: every refresh call returns before it ends


def _bits(t):
    import torch
    return t.view(torch.int32).cpu().numpy() if t.dtype == torch.float32 else t.cpu().numpy()


def _pmc(seed):
    from test_policy import random_weights
    w = random_weights(seed)
    w[25] *= 0.05
    w[27][:] = -1.0
    return w


class _Pmc:
    """forward_rec with sampling of a DevicePolicy, every output (actions, codes, V, -log p)."""
    state_dim = 0

    def __init__(self, torch, n, seed):
        rng = np.random.default_rng(seed)
        self.torch, self.n = torch, n
        self.obs = torch.from_numpy(rng.standard_normal((n, 207)).astype(np.float32)).cuda()

    def make(self, w):
        from lifelike_agility_and_play_b200.policy import DevicePolicy
        return DevicePolicy(w, device=0)

    def run(self, pol, stream=None):
        torch, n = self.torch, self.n
        out = [torch.zeros((n, 12), device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda"), torch.zeros(n, device="cuda"),
               torch.zeros(n, device="cuda")]
        assert pol._lib.llq_policy_forward_rec(pol._h, self.obs.data_ptr(), 207, n, out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(),
                                               out[3].data_ptr(), 1, SEED, COUNTER, GID0, stream) == 0
        return out

    @staticmethod
    def blob(w):
        from lifelike_agility_and_play_b200.policy import pack_weights
        return pack_weights(w)


class _Hier:
    """One forward of a hierarchical handle (deterministic, environmental or strategic training) from fixed observations, states and
    done flags; every output (actions, codes, heading, V, -log p, state)."""

    def __init__(self, torch, kind, n, seed):
        self.torch, self.kind, self.n = torch, kind, n
        self.strategic = kind in ("sepmc", "sepmc_train")
        self.state_dim = {"epmc": 64, "epmc_train": 128, "sepmc": 128, "sepmc_train": 192}[kind]
        rng = np.random.default_rng(seed)
        ow = 965 if self.strategic else 916
        self.ow = ow
        self.obs = torch.from_numpy(np.stack([pc._hier_row(rng, pc.HIER_CATS[i % 3], ow) for i in range(n)])).cuda()
        self.state0 = torch.from_numpy(pc.hier_random_state(rng, n, self.state_dim)).cuda()
        done = np.zeros(n, np.uint8)
        done[rng.random(n) < 0.3] = 1
        self.done = torch.from_numpy(done).cuda()

    def weights(self, seed):
        from lifelike_agility_and_play_b200.policy_epmc import random_weights
        return random_weights(self.strategic, seed)

    def make(self, w):
        from lifelike_agility_and_play_b200.policy_epmc import DeviceHierPolicy, DeviceSepmcTrainPolicy
        if self.kind == "sepmc_train":
            return DeviceSepmcTrainPolicy(w, device=0)
        return DeviceHierPolicy(w, device=0, train=self.kind == "epmc_train")

    def run(self, pol, stream=None, state=None):
        torch, n = self.torch, self.n
        st = self.state0.clone() if state is None else state
        act, codes, head = torch.zeros((n, 12), device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda"), torch.zeros(n, device="cuda")
        val, nlp = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
        a = (self.obs.data_ptr(), self.ow, n, self.done.data_ptr(), st.data_ptr(), act.data_ptr(), codes.data_ptr())
        if self.kind in ("epmc", "sepmc"):
            pol.forward(*a, head.data_ptr(), stream=stream)
        elif self.kind == "epmc_train":
            pol.forward_rec(*a, val.data_ptr(), nlp.data_ptr(), 1, SEED, COUNTER, GID0, stream=stream)
        else:
            pol.forward_rec(*a, head.data_ptr(), val.data_ptr(), nlp.data_ptr(), 1, SEED, COUNTER, GID0, stream=stream)
        return [act, codes, head, val, nlp, st]

    @staticmethod
    def blob(w):
        from lifelike_agility_and_play_b200.policy_epmc import weight_blob
        return weight_blob(w)[0]


def _same(got, want, what):
    names = ("actions", "codes", "heading", "V", "-log p", "state")
    for name, g, r in zip(names, got, want):
        assert np.array_equal(_bits(g), _bits(r)), (what, name)


def _case(torch, kind):
    if kind == "pmc":
        case = _Pmc(torch, 300, 1)
        return case, [_pmc(s) for s in (11, 12, 13)]
    case = _Hier(torch, kind, 83, 2)
    return case, [case.weights(s) for s in (11, 12, 13)]


KINDS = ["pmc", "epmc", "epmc_train", "sepmc", "sepmc_train"]


@pytest.mark.parametrize("kind", KINDS)
def test_refresh_equals_a_fresh_handle_bit_for_bit(built, kind):
    """Create from A, forward, set_weights(B), forward, ...: every output equals that of a fresh handle of the same weights on the same
    observations, states, done flags, seed and counter; host and device sources, and a refresh to the weights the handle holds."""
    import torch
    case, (A, B, _) = _case(torch, kind)
    fresh = {"A": case.make(A), "B": case.make(B)}
    ref = {k: case.run(p) for k, p in fresh.items()}
    torch.cuda.synchronize()
    assert not np.array_equal(_bits(ref["A"][0]), _bits(ref["B"][0]))
    pol = case.make(A)
    blobs = {"A": torch.from_numpy(case.blob(A)).cuda(), "B": torch.from_numpy(case.blob(B)).cuda()}
    _same(case.run(pol), ref["A"], "created from A")
    for src, name in (("host", "A"), ("host", "B"), ("device", "B"), ("host", "A"), ("device", "A"), ("device", "B"), ("host", "B")):
        pol.set_weights({"A": A, "B": B}[name] if src == "host" else blobs[name])
        _same(case.run(pol), ref[name], "%s refresh to %s" % (src, name))
    torch.cuda.synchronize()
    if kind == "pmc":
        # the packed image against the host statement of the forward (a refreshed and a fresh handle share the packer)
        from lifelike_agility_and_play_b200.policy import PmcPolicy
        host = PmcPolicy(B)
        obs = case.obs.cpu().numpy()
        act = torch.zeros((case.n, 12), device="cuda")
        codes = torch.zeros(case.n, dtype=torch.int32, device="cuda")
        val = torch.zeros(case.n, device="cuda")
        pol.forward_ex(case.obs.data_ptr(), 207, case.n, act.data_ptr(), codes.data_ptr(), val.data_ptr(), None)
        torch.cuda.synchronize()
        a_h, c_h = host.act(obs, return_code=True)
        same = codes.cpu().numpy() == c_h
        assert same.mean() > 0.99 and np.abs(act.cpu().numpy()[same] - a_h[same]).max() < 1e-4
        assert np.abs(val.cpu().numpy() - host.value(obs)).max() < 1e-4 * (1 + np.abs(host.value(obs)).max())
    for p in list(fresh.values()) + [pol]:
        p.close()


def _raw_set(pol, kind, buf, on_device, stream):
    """The library entry itself, so that the caller's host buffer is one array overwritten after every call."""
    ptr = buf.data_ptr() if on_device else buf.ctypes.data
    if kind == "pmc":
        return pol._lib.llq_policy_set_weights(pol._h, C.c_void_p(ptr), C.c_int64(buf.size if not on_device else buf.numel()), C.c_int32(on_device),
                                               C.c_void_p(stream))
    n = buf.size if not on_device else buf.numel()
    return pol.lib.llq_hier_policy_set_weights(pol._h, C.c_void_p(ptr), C.c_int64(n), C.c_int32(on_device), C.c_void_p(stream))


@pytest.mark.parametrize("source", ["host", "device"])
@pytest.mark.parametrize("kind", ["pmc", "epmc_train", "sepmc_train"])
def test_refreshes_are_ordered_on_their_stream(built, kind, source):
    """One stream, no synchronisation: sleep, forward, refresh to B, forward, refresh to C, forward -> A, B, C.  The host buffer is
    overwritten as soon as each call returns; a refresh on another stream, or a staging buffer reused before its copy left it, fails."""
    import torch
    case, (A, B, Cw) = _case(torch, kind)
    refs = []
    for w in (A, B, Cw):
        p = case.make(w)
        refs.append(case.run(p))
        torch.cuda.synchronize()
        p.close()
    pol = case.make(A)
    blobs = [case.blob(w) for w in (B, Cw)]
    dev = [torch.from_numpy(b).cuda() for b in blobs]
    buf = np.empty_like(blobs[0])
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    outs = []
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP)
        outs.append(case.run(pol, stream=s.cuda_stream))
        for i in range(2):
            if source == "host":
                buf[:] = blobs[i]
                assert _raw_set(pol, kind, buf, 0, s.cuda_stream) == 0
                buf[:] = np.nan                                            # the caller reuses its array at once
            else:
                assert _raw_set(pol, kind, dev[i], 1, s.cuda_stream) == 0
            # the stream still sleeps after the first refresh (a second host refresh waits for the first copy, so not always after that)
            assert i or not s.query(), "the stream woke before the first refresh was queued: the ordering was not exercised"
            outs.append(case.run(pol, stream=s.cuda_stream))
    assert source == "host" or not s.query(), "the stream woke before the last call returned"
    s.synchronize()
    for i, (got, want) in enumerate(zip(outs, refs)):
        _same(got, want, "forward %d" % i)
    pol.close()


def test_entry_refusals_on_the_device(built):
    import torch
    from lifelike_agility_and_play_b200.policy import DevicePolicy
    from lifelike_agility_and_play_b200.policy_epmc import DeviceHierPolicy, DeviceOpponentPool, random_weights, weight_blob
    w = random_weights(True, 3)
    det, pool = DeviceHierPolicy(w, device=0), DeviceOpponentPool([w, w], device=0, max_rows=8)
    lib = det.lib
    blob = weight_blob(w)[0]
    n = C.c_int64(blob.size)
    hp, dp = C.c_void_p(blob.ctypes.data), torch.from_numpy(blob).cuda()
    assert lib.llq_hier_policy_set_weights(det._h, hp, C.c_int64(blob.size - 4), 0, None) == -1
    assert lib.llq_hier_policy_set_weights(det._h, hp, n, C.c_int32(2), None) == -1
    assert lib.llq_hier_policy_set_weights(det._h, hp, n, C.c_int32(1), None) == -1 and b"device memory" in lib.llq_hier_policy_last_error()
    assert lib.llq_hier_policy_set_weights(pool._h, hp, n, 0, None) == -1 and b"set_pool_model" in lib.llq_hier_policy_last_error()
    assert lib.llq_hier_policy_set_pool_model(det._h, 0, hp, n, 0, None) == -1 and b"not a pool" in lib.llq_hier_policy_last_error()
    for k in (-1, 2):
        assert lib.llq_hier_policy_set_pool_model(pool._h, C.c_int32(k), hp, n, 0, None) == -1
    assert lib.llq_hier_policy_set_pool_model(pool._h, 1, hp, C.c_int64(blob.size + 4), 0, None) == -1
    assert lib.llq_hier_policy_set_pool_model(pool._h, 1, C.c_void_p(dp.data_ptr()), n, 1, None) == 0
    with pytest.raises(ValueError, match="set_model"):
        pool.set_weights(w)
    with pytest.raises(ValueError):
        det.set_weights(dp[:-4].clone())
    pmc = DevicePolicy(_pmc(1), device=0)
    pb = np.zeros(358647, np.float32)
    assert pmc._lib.llq_policy_set_weights(pmc._h, C.c_void_p(pb.ctypes.data), C.c_int64(358647), C.c_int32(1), None) == -1
    assert pmc._lib.llq_policy_set_weights(pmc._h, C.c_void_p(pb.ctypes.data), C.c_int64(358646), C.c_int32(0), None) == -1
    torch.cuda.synchronize()
    det.close(); pool.close(); pmc.close()


def _pool_from_table(blob, off, K, rows):
    """A pool handle straight from a designed blob and offset table."""
    from lifelike_agility_and_play_b200.policy_epmc import DeviceOpponentPool, _HierHandle, _vp
    pool = DeviceOpponentPool.__new__(DeviceOpponentPool)
    _HierHandle.__init__(pool, "llq_hier_policy_create_pool", _vp(blob), C.c_int64(blob.size), _vp(off), C.c_int32(K), C.c_int32(rows), C.c_int32(0))
    return pool


def _pool_fwd(torch, pool, case, model, done=None, state=None):
    n = case.n
    st = case.state0.clone() if state is None else state.clone()
    act, codes, head = torch.zeros((n, 12), device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda"), torch.zeros(n, device="cuda")
    m = torch.from_numpy(np.asarray(model, np.int32)).cuda()
    d = None if done is None else torch.from_numpy(np.asarray(done, np.uint8)).cuda()
    assert pool.lib.llq_hier_policy_forward_pool(pool._h, C.c_void_p(case.obs.data_ptr()), C.c_int64(965), C.c_int32(n),
                                                 C.c_void_p(0 if d is None else d.data_ptr()), C.c_void_p(st.data_ptr()), C.c_void_p(act.data_ptr()),
                                                 C.c_void_p(codes.data_ptr()), C.c_void_p(head.data_ptr()), C.c_void_p(m.data_ptr()), None,
                                                 C.c_int64(1), C.c_uint64(SEED), C.c_uint64(COUNTER), C.c_int64(GID0), None) == 0
    torch.cuda.synchronize()
    return [_bits(x) for x in (act, codes, head, st)], m.cpu().numpy()


def _single(torch, case, w, done):
    """The deterministic forward of a single handle of w on all rows (with done flags `done`)."""
    p = case.make(w)
    d = torch.from_numpy(np.asarray(done, np.uint8)).cuda()
    st = case.state0.clone()
    act, codes, head = torch.zeros((case.n, 12), device="cuda"), torch.zeros(case.n, dtype=torch.int32, device="cuda"), torch.zeros(case.n, device="cuda")
    p.forward(case.obs.data_ptr(), 965, case.n, d.data_ptr(), st.data_ptr(), act.data_ptr(), codes.data_ptr(), head.data_ptr())
    torch.cuda.synchronize()
    p.close()
    return [_bits(x) for x in (act, codes, head, st)]


@pytest.mark.parametrize("source", ["host", "device"])
def test_pool_slot_refresh(built, source):
    """set_model(1, B) on a pool of 3: rows on models 0 and 2 are bit for bit as before, rows on model 1 equal a single B handle's forward
    with the state they carry (the game goes on); then model 2, at probability 0, is filled with C, given all the probability, and
    drawn by every row, whose forward is C's from a wiped state."""
    import torch
    from lifelike_agility_and_play_b200.policy_epmc import DeviceOpponentPool, weight_blob
    case = _Hier(torch, "sepmc", 83, 4)
    A = [case.weights(s) for s in (20, 21, 22)]
    B, Cw = case.weights(23), case.weights(24)
    src = (lambda w: w) if source == "host" else (lambda w: torch.from_numpy(weight_blob(w)[0]).cuda())
    pool = DeviceOpponentPool(A, device=0, max_rows=case.n, probs=[0.5, 0.5, 0.0])
    model = np.arange(case.n) % 3
    keep = np.zeros(case.n, np.uint8)
    before, _ = _pool_fwd(torch, pool, case, model)
    pool.set_model(1, src(B))
    after, m = _pool_fwd(torch, pool, case, model)
    assert np.array_equal(m, model)
    on1 = model == 1
    b_ref = _single(torch, case, B, keep)
    for name, x, y, r in zip(("actions", "codes", "heading", "state"), before, after, b_ref):
        assert np.array_equal(x[~on1], y[~on1]), ("rows on other models changed", name)
        assert np.array_equal(y[on1], r[on1]), ("rows on the refreshed model", name)
        assert not np.array_equal(x[on1], y[on1]) or name == "codes"
    pool.set_model(1, src(A[1]))                                      # back to the weights it was created with
    again, _ = _pool_fwd(torch, pool, case, model)
    for x, y in zip(before, again):
        assert np.array_equal(x, y)
    pool.set_model(2, src(Cw))
    pool.set_probs([0.0, 0.0, 1.0])
    done = np.ones(case.n, np.uint8)
    drawn, m = _pool_fwd(torch, pool, case, model, done)
    assert (m == 2).all()
    for x, r in zip(drawn, _single(torch, case, Cw, done)):
        assert np.array_equal(x, r)
    pool.close()


def test_pool_regions_in_the_library(built):
    """The regions of designed tables: models stored in the blob in the order 2, 0, 1 (unordered) with a prefix; a refresh of model 0
    lands in its region only.  A pool whose models share an array refuses set_pool_model."""
    import torch
    from lifelike_agility_and_play_b200.policy_epmc import hier_role_arrays, pool_regions, weight_blob
    case = _Hier(torch, "sepmc", 40, 5)
    W = [case.weights(s) for s in (30, 31, 32)]
    B = case.weights(33)
    blobs, starts = zip(*[weight_blob(w) for w in W])
    size = blobs[0].size
    order, pre = [2, 0, 1], 8
    base = {k: pre + order.index(k) * size for k in range(3)}
    blob = np.concatenate([np.zeros(pre, np.float32)] + [blobs[k] for k in order])
    roles = hier_role_arrays(True)
    off = np.concatenate([starts[k][roles] + base[k] for k in range(3)]).astype(np.int32)
    assert pool_regions(off, 3, blob.size) == [(base[k], base[k] + size) for k in range(3)]
    pool = _pool_from_table(blob, off, 3, case.n)
    model = np.arange(case.n) % 3
    before, _ = _pool_fwd(torch, pool, case, model)
    nb = weight_blob(B)[0]
    assert pool.lib.llq_hier_policy_set_pool_model(pool._h, 0, C.c_void_p(nb.ctypes.data), C.c_int64(nb.size), 0, None) == 0
    after, _ = _pool_fwd(torch, pool, case, model)
    ref = _single(torch, case, B, np.zeros(case.n, np.uint8))
    on0 = model == 0
    for x, y, r in zip(before, after, ref):
        assert np.array_equal(x[~on0], y[~on0]) and np.array_equal(y[on0], r[on0])
    pool.close()
    shared = off.copy()
    shared[101 + 5] = shared[5]                                      # model 1 uses model 0's array of role 5
    assert pool_regions(shared, 3, blob.size) is None
    pool = _pool_from_table(blob, shared, 3, case.n)
    for k in range(3):
        assert pool.lib.llq_hier_policy_set_pool_model(pool._h, k, C.c_void_p(nb.ctypes.data), C.c_int64(nb.size), 0, None) == -1
    assert b"share" in pool.lib.llq_hier_policy_last_error()
    pool.close()


# ------------------------------------------------------------------------------------------------------------------------ the workers
SWITCH = 3                                                           # update at step 3 of the first unroll: records 0..2 A, 3.. B


def _run_worker(torch, worker, o0, T, on_switch=None):
    worker.start(o0)
    unrolls = []
    for _ in range(2):
        for t in range(T):
            if on_switch is not None and len(unrolls) == 0 and t == SWITCH:
                on_switch(worker)
            worker.step()
        u = worker.finish_unroll()
        worker.wait()
        unrolls.append([x.clone() for x in (u if isinstance(u, tuple) else (u,))])
    torch.cuda.synchronize()
    return unrolls


def _keeps_state(torch, update):
    """on_switch: `update`(worker), checking that it leaves the state, masks and counters as they were."""
    def go(worker):
        worker.wait()
        torch.cuda.synchronize()
        keep = [x.clone() for x in (getattr(worker, "state", None), getattr(worker, "mask", None), getattr(worker, "opp_state", None)) if x is not None]
        calls, t = worker.calls, worker.t
        update(worker)
        worker.wait()
        torch.cuda.synchronize()
        now = [x for x in (getattr(worker, "state", None), getattr(worker, "mask", None), getattr(worker, "opp_state", None)) if x is not None]
        assert all(torch.equal(a, b) for a, b in zip(keep, now)) and (worker.calls, worker.t) == (calls, t), "the refresh touched the state"
    return go


def test_pmc_worker_refresh(built):
    """RolloutWorker with update_policy(B) at step 3: records 0..2 bit for bit those of a worker that never refreshes, and the replay with
    the host policy switched at step 3."""
    import torch
    from lifelike_agility_and_play_b200 import _capi as capi
    from lifelike_agility_and_play_b200.mocap import synthetic_mocap
    from lifelike_agility_and_play_b200.model.compile_model import load_model_blob
    from lifelike_agility_and_play_b200.parallel import RolloutWorker
    from lifelike_agility_and_play_b200.parallel.trajectory import COL_ACTION, COL_DONE, COL_NEGLOGP, COL_REWARD, COL_VALUE
    from lifelike_agility_and_play_b200.policy import DevicePolicy, PmcPolicy
    n, T = 96, 6
    A, B = _pmc(9), _pmc(10)
    A[27][:] = B[27][:] = -2.0
    blob, mocap = load_model_blob(), synthetic_mocap(5, seed=2, min_frames=380, max_frames=420)
    lib = capi.load_cuda_library()
    engs = [capi.VecEngine(lib, n, blob, mocap, seed=21, device=0, auto_reset=1) for _ in range(3)]
    pols = [DevicePolicy(A, device=0) for _ in range(2)]
    o0 = engs[0].reset()
    for e in engs[1:]:
        assert np.array_equal(o0, e.reset())
    got = _run_worker(torch, RolloutWorker(engs[0], pols[0], T, "cuda:0", seed=5), o0, T, _keeps_state(torch, lambda w: w.update_policy(B)))
    plain = _run_worker(torch, RolloutWorker(engs[1], pols[1], T, "cuda:0", seed=5), o0, T)
    assert np.array_equal(_bits(got[0][0][:SWITCH]), _bits(plain[0][0][:SWITCH]))
    assert not np.array_equal(_bits(got[0][0][SWITCH]), _bits(plain[0][0][SWITCH]))
    slab = torch.cat([u[0] for u in got], 0).cpu().numpy()
    chk, obs, n_close = engs[2], o0, 0
    for t in range(2 * T):
        host = PmcPolicy(A if t < SWITCH else B)
        assert np.array_equal(slab[t, :, :207], obs)
        a = slab[t, :, COL_ACTION:COL_ACTION + 12]
        mean = host.act(obs)
        n_close += int((np.abs(slab[t, :, COL_NEGLOGP] - host.neglogp(a, mean)) < 1e-2).sum())
        v = host.value(obs)
        assert np.abs(slab[t, :, COL_VALUE] - v).max() < 1e-4 * (1 + np.abs(v).max()), t
        obs, rew, done = chk.step(a)
        assert np.array_equal(rew, slab[t, :, COL_REWARD]) and np.array_equal(done.astype(np.float32), slab[t, :, COL_DONE])
    assert n_close >= 0.999 * 2 * T * n, (n_close, 2 * T * n)
    for x in pols + engs:
        x.close()


def test_epmc_worker_refresh(built):
    """HierRolloutWorker with update_policy(B as a device blob) at step 3: records 0..2 as a worker that never refreshes, the replay
    switched at step 3 carrying its LSTM states across the switch."""
    import torch
    from lifelike_agility_and_play_b200 import _capi as capi
    from lifelike_agility_and_play_b200.model.compile_model import load_model_blob
    from lifelike_agility_and_play_b200.parallel import HierRolloutWorker
    from lifelike_agility_and_play_b200.parallel.trajectory import HCOL_ACTION, HCOL_CODE, HCOL_DONE, HCOL_NEGLOGP, HCOL_REWARD, HCOL_VALUE
    from lifelike_agility_and_play_b200.policy_epmc import DeviceHierPolicy, EpmcPolicy, random_weights, weight_blob
    from lifelike_agility_and_play_b200.sim_envs.playground_env import INIT_STATE_RUN_0
    n, T, seed, gid0 = 40, 5, 77, 1000
    A, B = random_weights(False, 4), random_weights(False, 6)
    for w in (A, B):
        w[99] = (0.05 * w[99]).astype(np.float32)
    cfg = dict(kp=50.0, kd=0.5, max_tau=16.0, ground_friction=1.0, max_steps=7, seed=5, friction_hi=1.0, env_kind=capi.ENV_EPMC,
               element_id=3, cmd_freq_lo=25, cmd_freq_hi=40, auto_reset=1, global_env_offset=gid0)
    lib, blob = capi.load_cuda_library(), load_model_blob()
    engs = [capi.VecEngine(lib, n, blob, None, device=0, **cfg) for _ in range(3)]
    for e in engs:
        e.set_init_state(INIT_STATE_RUN_0)
    pols = [DeviceHierPolicy(A, device=0, train=True) for _ in range(2)]
    o0 = engs[0].reset()
    for e in engs[1:]:
        assert np.array_equal(o0, e.reset())
    b_dev = torch.from_numpy(weight_blob(B)[0]).cuda()
    got = _run_worker(torch, HierRolloutWorker(engs[0], pols[0], T, "cuda:0", seed=seed), o0, T,
                      _keeps_state(torch, lambda w: w.update_policy(b_dev)))
    plain = _run_worker(torch, HierRolloutWorker(engs[1], pols[1], T, "cuda:0", seed=seed), o0, T)
    assert np.array_equal(_bits(got[0][0][:SWITCH]), _bits(plain[0][0][:SWITCH]))
    chk, obs, mask, n_code = engs[2], o0, np.ones(n, np.float32), 0
    for k, (slab_t, init, first, boot) in enumerate(got):
        slab = slab_t.cpu().numpy()
        init = init.cpu().numpy()
        if k == 0:
            s_code, s_val = init[:, :64], init[:, 64:]              # the host chain runs through the switch with its own states
        else:
            assert np.abs(init - np.concatenate([s_code, s_val], axis=1)).max() < 1e-4
            s_code, s_val = init[:, :64], init[:, 64:]
        for t in range(T):
            host = EpmcPolicy(A if (k, t) < (0, SWITCH) else B)
            assert np.array_equal(slab[t, :, :916], obs)
            a = slab[t, :, HCOL_ACTION:HCOL_ACTION + 12]
            code = slab[t, :, HCOL_CODE].astype(np.int64)
            u = hc.uniforms(gid0 + np.arange(n), seed, k * T + t)
            a_h, s_code, c_h, nlp_h = host.act(obs, s_code, mask, return_code=True, uniforms=u, return_neglogp=True)
            v_h, s_val = host.value(obs, s_val, mask)
            same = c_h == code
            n_code += int(same.sum())
            assert np.abs(a[same] - a_h[same]).max(initial=0) < 1e-4, (k, t)
            assert np.abs(slab[t, same, HCOL_NEGLOGP] - nlp_h[same]).max(initial=0) < 1e-3, (k, t)
            assert np.abs(slab[t, :, HCOL_VALUE] - v_h).max() < 1e-4 * (1 + np.abs(v_h).max()), (k, t)
            obs, rew, done = chk.step(a)
            assert np.array_equal(rew, slab[t, :, HCOL_REWARD]) and np.array_equal(done.astype(np.float32), slab[t, :, HCOL_DONE])
            mask = done.astype(np.float32)
    assert n_code >= 0.99 * 2 * T * n, (n_code, 2 * T * n)
    for x in pols + engs:
        x.close()


@pytest.mark.parametrize("opponent", ["single", "pool"])
def test_sepmc_worker_refresh(built, opponent):
    """SepmcRolloutWorker with update_policy(B) and update_opponent at step 3 (the single opponent, or model 1 of a pool of 3):
    records 0..2 as a worker that never refreshes; the replay with both seats' host policies switched at step 3."""
    import torch
    from lifelike_agility_and_play_b200 import _capi as capi
    from lifelike_agility_and_play_b200.model.compile_model import load_model_blob
    from lifelike_agility_and_play_b200.parallel import SepmcRolloutWorker
    from lifelike_agility_and_play_b200.parallel.trajectory import (SCOL_ACTION, SCOL_CODE, SCOL_DONE, SCOL_HEADING, SCOL_NEGLOGP, SCOL_OPPONENT,
                                                                    SCOL_REWARD, SCOL_VALUE)
    from lifelike_agility_and_play_b200.policy_epmc import (DeviceHierPolicy, DeviceOpponentPool, DeviceSepmcTrainPolicy, SepmcPolicy, random_weights,
                                                            weight_blob)
    from lifelike_agility_and_play_b200.sim_envs.playground_env import INIT_STATE_RUN_0
    P, T, seed, gid0 = 20, 5, 77, 1000
    n, pool = 2 * P, opponent == "pool"
    A, B = random_weights(True, 4), random_weights(True, 7)
    opp_w = [random_weights(True, s) for s in (5, 8, 9)]               # pool models (the single opponent is the first)
    OB = random_weights(True, 10)                                     # the opponent's new weights
    for x in [A, B, OB] + opp_w:
        x[149] = (0.05 * x[149]).astype(np.float32)
    cfg = dict(kp=50.0, kd=0.5, max_tau=16.0, ground_friction=1.0, max_steps=7, seed=5, friction_hi=1.0, env_kind=capi.ENV_SEPMC,
               auto_reset=1, global_env_offset=gid0)
    lib, blob = capi.load_cuda_library(), load_model_blob()
    engs = [capi.VecEngine(lib, n, blob, None, device=0, **cfg) for _ in range(3)]
    for e in engs:
        e.set_init_state(INIT_STATE_RUN_0)

    def make_opp():
        return DeviceOpponentPool(opp_w, device=0, max_rows=P, probs=[0.25, 0.75, 0.0]) if pool else DeviceHierPolicy(opp_w[0], device=0)
    pols, opps = [DeviceSepmcTrainPolicy(A, device=0) for _ in range(2)], [make_opp() for _ in range(2)]
    o0 = engs[0].reset()
    for e in engs[1:]:
        assert np.array_equal(o0, e.reset())
    ob_dev = torch.from_numpy(weight_blob(OB)[0]).cuda()
    worker = SepmcRolloutWorker(engs[0], pols[0], opps[0], T, "cuda:0", seed=seed)
    with pytest.raises(ValueError):
        worker.update_opponent(OB, k=None if pool else 1)

    def update(w):
        w.update_policy(B)
        w.update_opponent(ob_dev, k=1 if pool else None)
    got = _run_worker(torch, worker, o0, T, _keeps_state(torch, update))
    plain = _run_worker(torch, SepmcRolloutWorker(engs[1], pols[1], opps[1], T, "cuda:0", seed=seed), o0, T)
    assert np.array_equal(_bits(got[0][0][:SWITCH]), _bits(plain[0][0][:SWITCH]))
    pair_gid = gid0 // 2 + np.arange(P)
    chk, obs, mask, n_code, n_new = engs[2], o0, np.ones(P, np.float32), 0, 0
    s_opp = np.zeros((P, 128), np.float32)
    for k, (slab_t, init, first, boot) in enumerate(got):
        slab = slab_t.cpu().numpy()
        init = init.cpu().numpy()
        if k == 1:
            assert np.abs(init - np.concatenate([s_pol, s_val], axis=1)).max() < 1e-4
        s_pol, s_val = init[:, :128], init[:, 128:]
        for t in range(T):
            new = (k, t) >= (0, SWITCH)
            host = SepmcPolicy(B if new else A)
            omodels = [OB if (new and (j == (1 if pool else 0))) else opp_w[j] for j in range(3)]
            assert np.array_equal(slab[t, :, :965], obs)
            a = slab[t, :, SCOL_ACTION:SCOL_ACTION + 12]
            code = slab[t, :, SCOL_CODE].astype(np.int64)
            opp = slab[t, 0::2, SCOL_OPPONENT].astype(np.int64) if pool else np.zeros(P, np.int64)
            if pool and new:
                n_new += int((opp == 1).sum())
            for m in np.unique(opp):
                rows = np.flatnonzero(opp == m)
                a1, s1, _, c1 = SepmcPolicy(omodels[m]).act(obs[1::2][rows], s_opp[rows], mask[rows], return_aux=True)
                s_opp[rows] = s1
                same1 = c1 == code[1::2][rows]
                n_code += int(same1.sum())
                assert np.abs(a[1::2][rows][same1] - a1[same1]).max(initial=0) < 1e-4, ("seat 1", k, t, m)
            eps = sc.eps_of(pair_gid, seed, k * T + t)
            a0, s_pol, h0, c0, nlp0 = host.act(obs[0::2], s_pol, mask, return_aux=True, eps=eps, return_neglogp=True)
            assert np.abs(h0 - slab[t, 0::2, SCOL_HEADING]).max() < 1e-4 * (1 + np.abs(h0).max()), (k, t)
            same = c0 == code[0::2]
            n_code += int(same.sum())
            assert np.abs(a[0::2][same] - a0[same]).max(initial=0) < 1e-4, (k, t)
            assert np.abs(slab[t, 0::2, SCOL_NEGLOGP] - nlp0).max() < 1e-4
            v_h, s_val = host.value(obs[0::2], s_val, mask)
            assert np.abs(slab[t, 0::2, SCOL_VALUE] - v_h).max() < 1e-4 * (1 + np.abs(v_h).max()), (k, t)
            obs, rew, done = chk.step(a)
            assert np.array_equal(rew, slab[t, :, SCOL_REWARD]) and np.array_equal(done.astype(np.float32), slab[t, :, SCOL_DONE])
            mask = done[0::2].astype(np.float32)
    assert n_code >= 0.99 * 4 * T * P, (n_code, 4 * T * P)
    assert not pool or n_new > 0, "no pair played the refreshed pool model"
    for x in pols + opps + engs:
        x.close()
