"""The policy kernels against the fp64 statements of tests/policy_cases.py, row by row with no exclusions (run with -m gpu on an H100).

Every row of the designed batches is decisive (its code clears the runner-up by more than 4 kappa S_gap) or is a designed exact tie,
so codes must be exactly equal (the lowest index on a tie), and every action, value, state, heading, sample and -log p must be within
kappa S + 2^-23 |ref| of the reference, S the error model's sensitivity of that output.  The printed ratio is the largest
(|err| - 2^-23 |ref|) / S over all outputs of a test: the kappa that test needs.

Around the numbers: outputs are allocated with extra rows (one tile: 32 PMC rows, 8 hierarchical rows) filled with a canary bit
pattern, which must come back bit for bit; the observation padding past column 207 / 916 / 965 is NaN.

Measured on an H100 80GB HBM3 at a 600 W power limit (largest error / S over the whole file):
  PMC            mean 88.2, value 6.69, sample 36.4, -log p 3.01          -> KAPPA_PMC = 400
  hierarchical   actions 2.08, state 4.73, heading 1.28 (recurrence: 2.01, 4.01, 1.28)   -> KAPPA_HIER = 20
The PMC ratio is large because the 3xTF32 layers truncate both operand splits (up to ~2^-20 per product, always towards zero);
plain TF32 or 2xTF32 layers are ~2^10 times further off and fail every PMC test of this file.  Placement is bit-identical for
a one-tile and for a one-row shift, on both kernels.
"""
import numpy as np
import pytest

import policy_cases as pc

pytestmark = pytest.mark.gpu

CANARY = 0x7FBADBAD            # a NaN bit pattern
SEED, COUNTER, GID0 = 2 ** 40 + 3, 2 ** 32 + 7, 3 * 10 ** 6 + 1
RATIOS = {}


def _canary(torch, shape, dtype=None):
    t = torch.full(shape, CANARY, dtype=torch.int32, device="cuda")
    return t if dtype is torch.int32 else t.view(torch.float32)


def _bits(t):
    import torch
    return t.view(torch.int32).cpu().numpy() if t.dtype == torch.float32 else t.cpu().numpy()


def _check(name, got, ref, S, kappa, key):
    got = np.asarray(got, np.float64)
    err = np.abs(got - ref)
    slack = err - pc.U * np.abs(ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(slack > 0, slack / S, 0.0)
    RATIOS[key] = max(RATIOS.get(key, 0.0), float(np.nanmax(ratio)) if ratio.size else 0.0)
    bad = np.argwhere(~(err <= kappa * S + pc.U * np.abs(ref)))
    assert len(bad) == 0, (name, [(tuple(int(j) for j in b), float(got[tuple(b)]), float(ref[tuple(b)]), float(S[tuple(b)])) for b in bad[:8]])


def _canary_intact(name, t, n):
    b = _bits(t)[n:]
    assert (b == CANARY).all(), (name, "rows past n written")


@pytest.fixture(scope="module")
def pmc(built):
    from lifelike_agility_and_play_b200.policy import DevicePolicy
    w, obs, cats, info, ref, S = pc.pmc_case()
    dev = DevicePolicy(w, device=0)
    yield w, obs, ref, S, dev
    dev.close()
    print("PMC kappa needed: %s" % {k: "%.3g" % v for k, v in RATIOS.items() if k.startswith("pmc")})


def _rec(dev, obs_ptr, ld, n, act, codes, values, nlp, out_ld, seed, counter, gid0):
    rc = dev._lib.llq_policy_forward_rec(dev._h, obs_ptr, ld, n, act, codes, values, nlp, out_ld, seed, counter, gid0, None)
    assert rc == 0, dev._lib.llq_policy_last_error()


@pytest.mark.parametrize("ld", [207, 223, 260])
@pytest.mark.parametrize("n", [1, 31, 32, 33, 4097])
def test_pmc_every_row_matches_the_fp64_statement(pmc, n, ld):
    """forward (mean, codes), forward_ex (+ value) and forward_rec (sampled, -log p, codes) on the first n designed rows."""
    import torch
    w, obs, ref, S, dev = pmc
    k = pc.KAPPA_PMC
    t_obs = torch.from_numpy(pc.padded(obs[:n], ld, 207)).cuda()
    sref, sS = pc.pmc_sample_eval(w, ref["mean"][:n], S["mean"][:n], GID0 + np.arange(n), SEED, COUNTER)
    for entry in ("forward", "forward_ex", "forward_rec"):
        act, codes, val, nlp = _canary(torch, (n + 32, 12)), _canary(torch, (n + 32,), torch.int32), _canary(torch, (n + 32,)), _canary(torch, (n + 32,))
        if entry == "forward":
            dev.forward(t_obs.data_ptr(), ld, n, act.data_ptr(), codes.data_ptr())
        elif entry == "forward_ex":
            dev.forward_ex(t_obs.data_ptr(), ld, n, act.data_ptr(), codes.data_ptr(), val.data_ptr(), None)
        else:
            _rec(dev, t_obs.data_ptr(), ld, n, act.data_ptr(), codes.data_ptr(), val.data_ptr(), nlp.data_ptr(), 1, SEED, COUNTER, GID0)
        torch.cuda.synchronize()
        got_code = codes.cpu().numpy()[:n]
        assert np.array_equal(got_code, ref["code"][:n]), (entry, np.flatnonzero(got_code != ref["code"][:n])[:10])
        a = act.cpu().numpy()[:n]
        if entry == "forward_rec":
            _check("sample", a, sref["sample"], sS["sample"], k, "pmc sample")
            _check("-log p", nlp.cpu().numpy()[:n], sref["neglogp"], sS["neglogp"], k, "pmc -log p")
            eps = (a.astype(np.float64) - ref["mean"][:n]) / np.exp(np.asarray(w[27], np.float64).reshape(-1))
            assert np.abs(eps - sref["eps"]).max() < 1e-3
        else:
            _check("mean", a, ref["mean"][:n], S["mean"][:n], k, "pmc mean")
        if entry != "forward":
            _check("value", val.cpu().numpy()[:n], ref["value"][:n], S["value"][:n], k, "pmc value")
        for name, t in (("actions", act), ("codes", codes), ("values", val), ("neglogp", nlp)):
            _canary_intact(entry + " " + name, t, n if (name != "values" or entry != "forward") and (name != "neglogp" or entry == "forward_rec") else 0)


def test_pmc_record_slab_and_shards(pmc):
    """forward_rec into the value / -log p columns of a [n, 223] record slab whose observation is read in place: every other
    column and every row past n stays bit for bit; a shard launched on rows k.. with row_gid0 + k reproduces those rows."""
    import torch
    from lifelike_agility_and_play_b200.parallel.trajectory import COL_NEGLOGP, COL_VALUE, TRAJ_WIDTH
    w, obs, ref, S, dev = pmc
    n, k = pc.PMC_N, pc.KAPPA_PMC
    init = np.full((n + 32, TRAJ_WIDTH), np.nan, np.float32).view(np.int32)
    init[:] = CANARY
    init = init.view(np.float32)
    init[:n, :207] = obs
    runs = []
    for first in (0, 45, 64):
        slab = torch.from_numpy(init.copy()).cuda()
        act = _canary(torch, (n + 32, 12))
        row = slab.data_ptr() + first * TRAJ_WIDTH * 4
        dev.forward_rec(row, TRAJ_WIDTH, n - first, act.data_ptr() + first * 48, row + COL_VALUE * 4, row + COL_NEGLOGP * 4, TRAJ_WIDTH,
                        seed=SEED, counter=COUNTER, row_gid0=GID0 + first)
        torch.cuda.synchronize()
        runs.append((first, slab.cpu().numpy(), act.cpu().numpy()))
    _, s0, a0 = runs[0]
    sref, sS = pc.pmc_sample_eval(w, ref["mean"], S["mean"], GID0 + np.arange(n), SEED, COUNTER)
    _check("sample", a0[:n], sref["sample"], sS["sample"], k, "pmc sample")
    _check("-log p", s0[:n, COL_NEGLOGP], sref["neglogp"], sS["neglogp"], k, "pmc -log p")
    _check("value", s0[:n, COL_VALUE], ref["value"], S["value"], k, "pmc value")
    written = np.zeros(init.shape, bool)
    written[:n, [COL_VALUE, COL_NEGLOGP]] = True
    assert np.array_equal(s0.view(np.int32)[~written], init.view(np.int32)[~written])
    assert (a0[n:].view(np.int32) == CANARY).all()
    for first, s, a in runs[1:]:
        assert np.array_equal(s.view(np.int32)[first:], s0.view(np.int32)[first:]), first
        assert np.array_equal(a.view(np.int32)[first:], a0.view(np.int32)[first:]), first
        assert (s.view(np.int32)[:first] == init.view(np.int32)[:first]).all() and (a[:first].view(np.int32) == CANARY).all()


@pytest.mark.parametrize("shift", [32, 1])
def test_pmc_rows_do_not_depend_on_their_place_in_the_batch(pmc, shift):
    import torch
    w, obs, ref, S, dev = pmc
    n = pc.PMC_N
    out = []
    for s in (0, shift):
        o = np.concatenate([obs[n - s:], obs]) if s else obs
        t_obs = torch.from_numpy(np.ascontiguousarray(o)).cuda()
        m = len(o)
        act, codes, val, nlp = (torch.zeros((m, 12), device="cuda"), torch.zeros(m, dtype=torch.int32, device="cuda"),
                                torch.zeros(m, device="cuda"), torch.zeros(m, device="cuda"))
        _rec(dev, t_obs.data_ptr(), 207, m, act.data_ptr(), codes.data_ptr(), val.data_ptr(), nlp.data_ptr(), 1, SEED, COUNTER, GID0 - s)
        mean = torch.zeros((m, 12), device="cuda")
        dev.forward(t_obs.data_ptr(), 207, m, mean.data_ptr(), None)
        torch.cuda.synchronize()
        out.append([_bits(x)[s:] for x in (act, codes, val, nlp, mean)])
    for name, a, b in zip(("sample", "code", "value", "-log p", "mean"), *out):
        assert np.array_equal(a, b), (name, shift, int((a != b).sum()))


# ------------------------------------------------------------------------------------------------------------ hierarchical
@pytest.fixture(scope="module", params=[False, True], ids=["epmc", "sepmc"])
def hier(request, built):
    from lifelike_agility_and_play_b200.policy_epmc import DeviceHierPolicy
    case = pc.hier_case(request.param)
    dev = DeviceHierPolicy(case[0], device=0)
    yield (request.param,) + case + (dev,)
    dev.close()
    print("hierarchical kappa needed: %s" % {k: "%.3g" % v for k, v in RATIOS.items() if k.startswith("hier")})


def _hier_run(torch, dev, obs, ld, n, state, done, with_codes=True, with_heading=True):
    ow, ssz = dev.obs_dim, dev.state_dim
    t_obs = torch.from_numpy(pc.padded(obs[:n], ld, ow)).cuda()
    st = _canary(torch, (n + 8, ssz))
    st[:n] = torch.from_numpy(np.ascontiguousarray(state[:n])).cuda()
    t_done = None if done is None else torch.from_numpy(np.ascontiguousarray(done[:n])).cuda()
    act, codes, head = _canary(torch, (n + 8, 12)), _canary(torch, (n + 8,), torch.int32), _canary(torch, (n + 8,))
    dev.forward(t_obs.data_ptr(), ld, n, t_done.data_ptr() if t_done is not None else None, st.data_ptr(), act.data_ptr(),
                codes.data_ptr() if with_codes else None, head.data_ptr() if (with_heading and dev.strategic) else None)
    torch.cuda.synchronize()
    return act, codes, head, st


def _hier_compare(strategic, n, ref, S, act, codes, head, st, with_codes=True, with_heading=True, key="hier"):
    k = pc.KAPPA_HIER
    if with_codes:
        got = codes.cpu().numpy()[:n]
        assert np.array_equal(got, ref["code"][:n]), np.flatnonzero(got != ref["code"][:n])[:10]
    _canary_intact("codes", codes, n if with_codes else 0)
    _check("actions", act.cpu().numpy()[:n], ref["actions"][:n], S["actions"][:n], k, key + " actions")
    _check("state", st.cpu().numpy()[:n], ref["state"][:n], S["state"][:n], k, key + " state")
    _canary_intact("actions", act, n)
    _canary_intact("state", st, n)
    if strategic and with_heading:
        _check("heading", head.cpu().numpy()[:n], ref["heading"][:n], S["heading"][:n], k, key + " heading")
    _canary_intact("heading", head, n if (strategic and with_heading) else 0)


@pytest.mark.parametrize("ld", ["ow", "ow+1", 1024])
@pytest.mark.parametrize("n", [1, 7, 8, 9, 300, 1059])
def test_hierarchical_every_row_matches_the_fp64_statement(hier, n, ld):
    import torch
    strategic, w, obs, state, done, cats, info, ref, S, dev = hier
    ld = {"ow": dev.obs_dim, "ow+1": dev.obs_dim + 1}.get(ld, ld)
    act, codes, head, st = _hier_run(torch, dev, obs, ld, n, state, done)
    _hier_compare(strategic, n, ref, S, act, codes, head, st)


@pytest.mark.parametrize("shift", [8, 1])
def test_hierarchical_rows_do_not_depend_on_their_place_in_the_batch(hier, shift):
    import torch
    strategic, w, obs, state, done, cats, info, ref, S, dev = hier
    n = pc.HIER_N
    out = []
    for s in (0, shift):
        o = np.concatenate([obs[n - s:], obs]) if s else obs
        st = np.concatenate([state[n - s:], state]) if s else state
        d = np.concatenate([done[n - s:], done]) if s else done
        r = _hier_run(torch, dev, o, dev.obs_dim, len(o), st, d)
        out.append([_bits(x)[s:s + n] for x in r])
    for name, a, b in zip(("actions", "codes", "heading", "state"), *out):
        if name == "heading" and not strategic:
            continue
        assert np.array_equal(a, b), (name, shift, int((a != b).sum()))


def test_hierarchical_recurrence(hier):
    """Four steps from a non-zero state with done bytes 0, 1, 2 and 255 (every non-zero byte wipes); d_done = NULL on one step and
    d_codes / d_heading = NULL on another; each step's reference starts from the kernel's incoming state."""
    import torch
    from lifelike_agility_and_play_b200.policy_epmc import DeviceHierPolicy
    strategic, w, obs, state, done, cats, info, ref, S, _ = hier
    w = pc.hier_recurrence_weights(w, strategic, info)
    dev = DeviceHierPolicy(w, device=0)
    state0, obs_all, done_all = pc.hier_recurrence_case(strategic, w)
    n = len(state0)
    st_in = state0
    for step, (o, d) in enumerate(zip(obs_all, done_all)):
        d_use = None if step == pc.NULL_DONE_STEP else d
        with_codes = step != 1
        r, Sr, _ = pc.hier_eval(w, o, st_in, d_use if d_use is not None else np.zeros(n, np.uint8))
        assert (r["gap"] > 4 * pc.KAPPA_HIER * Sr["gap"]).all(), "a recurrence row is not decisive from the kernel's state"
        act, codes, head, st = _hier_run(torch, dev, o, dev.obs_dim, n, st_in, d_use, with_codes=with_codes, with_heading=with_codes)
        _hier_compare(strategic, n, r, Sr, act, codes, head, st, with_codes=with_codes, with_heading=with_codes, key="hier recurrence")
        if step == 0:
            assert set(np.unique(d).tolist()) == {0, 1, 2, 255} and (np.abs(st_in[d != 0]) > 0).any(1).all()
        st_in = st.cpu().numpy()[:n].copy()
    dev.close()
