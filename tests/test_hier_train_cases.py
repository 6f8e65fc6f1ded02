"""The environmental level's training forward on the CPU: its fp64 statement (tests/hier_train_cases.py) against the fp32 host class
`EpmcPolicy` (value tower, sampled code from given uniforms, -log p), the designed batch, and the learner tensors of an unroll."""
import numpy as np
import pytest
import torch

import hier_train_cases as hc
import policy_cases as pc
from lifelike_agility_and_play_b200.parallel import hier_slab_records
from lifelike_agility_and_play_b200.parallel.trajectory import (HCOL_ACTION, HCOL_CODE, HCOL_DONE, HCOL_NEGLOGP, HCOL_REWARD, HCOL_VALUE,
                                                                HIER_TRAJ_WIDTH)
from lifelike_agility_and_play_b200.policy_epmc import EPMC_SHAPES, EpmcPolicy, hier_role_arrays


def _agree(got, ref, S, name, factor=64.0):
    err = np.abs(np.asarray(got, np.float64) - ref)
    bar = factor * S + 1e-6 * np.abs(ref) + 1e-7
    assert (err <= bar).all(), (name, float((err / bar).max()))


def test_value_tower_table_matches_the_shipped_shapes():
    roles = hier_role_arrays(False, value_tower=True)
    assert len(roles) == 45 and roles[0] == 2 and roles[-1] == 46
    shapes = [EPMC_SHAPES[i] for i in roles]
    assert shapes[0] == (135, 128) and shapes[26] == (3, 32) and shapes[28] == (120, 64) and shapes[30] == (64, 128)
    assert shapes[32] == (256, 256) and shapes[34] == (256, 128) and shapes[43] == (32, 1) and shapes[44] == (1,)
    with pytest.raises(ValueError):
        hier_role_arrays(True, value_tower=True)


def test_uniforms_are_formed_as_the_kernel_forms_them():
    """u = ((float)r + 0.5f) 2^-32 in fp32 from the Philox words (pinned to the Random123 known answers in test_policy_cases.py), and
    every r >= 2^32 - 128, which rounds to u = 1.0f, is clamped to 0.99999994f: g stays finite (16.6)."""
    gid = hc.ROW_GID0 + np.arange(5)
    r, u = hc.draws(gid, hc.SEED, hc.COUNTER_BASE)
    c = pc.philox4x32(gid[2] & 0xFFFFFFFF, 7, hc.COUNTER_BASE & 0xFFFFFFFF, hc.COUNTER_BASE >> 32, hc.SEED & 0xFFFFFFFF, hc.SEED >> 32)
    assert [int(x) for x in r[2, 28:32]] == [int(x) for x in c]
    f = np.float32
    assert u.dtype == np.float32 and u[2, 29] == (f(int(c[1])) + f(0.5)) * f(2.0 ** -32)
    edge = np.array([hc.CLAMP_R - 1, hc.CLAMP_R, 2 ** 32 - 1], np.uint64)
    ue = np.minimum((edge.astype(f) + f(0.5)) * f(2.0 ** -32), f(0.99999994))
    assert ue[0] < 1.0 and ue[1] == ue[2] == f(0.99999994)
    g = hc.gumbel(ue, pc.REF)
    assert np.isfinite(g).all() and 16.0 < g[1] < 17.0


def test_statement_agrees_with_the_fp32_class():
    rng = np.random.default_rng(6)
    w = hc.design_weights(3)
    n = 96
    obs = np.stack([pc._hier_row(rng, "random", 916) for _ in range(n)])
    state = pc.hier_random_state(rng, n, 128)
    done = pc.DONE_BYTES[np.arange(n) % 4]
    u = hc.uniforms(hc.ROW_GID0 + np.arange(n), hc.SEED, hc.COUNTER_BASE)
    ref, S = hc.train_eval(hc.Trunks(w, obs, state, done), u)
    mask = (done != 0).astype(np.float32)
    host = EpmcPolicy(w)
    a, st, code, nlp = host.act(obs, state[:, :64], mask, return_code=True, uniforms=u, return_neglogp=True)
    v, vst = host.value(obs, state[:, 64:], mask)
    dec = hc.decisive(ref, S)
    assert dec.mean() > 0.9
    assert np.array_equal(code[dec], ref["code"][dec])
    _agree(v, ref["value"], S["value"], "value")
    _agree(np.concatenate([st, vst], axis=1), ref["state"], S["state"], "state")
    _agree(a[dec], ref["actions"][dec], S["actions"][dec], "actions")
    # the fp32 class rounds its logits once more than the kernel's model does; 1e-4 relative covers that at |logit| ~ 100
    assert (np.abs(nlp[dec] - ref["neglogp"][dec]) <= 64 * S["neglogp"][dec] + 1e-4 * (1 + np.abs(ref["logits"][dec]).max(1))).all()


def test_designed_batch_reaches_every_category_and_every_row_is_decisive():
    w, obs, state, done, counters, info, evals = hc.train_case()
    assert obs.shape == (hc.N, 916) and state.shape == (hc.N, 128) and len(counters) == 2
    reached = hc.reaches(w, obs, state, done, counters, info, evals)
    missing = {k: (len(v) - sum(v), len(v)) for k, v in reached.items() if not any(v)}
    assert not missing, missing
    for ref, S in evals:
        assert hc.decisive(ref, S).all()
        assert np.isfinite(ref["neglogp"]).all() and (ref["neglogp"] >= 0).all()


def _hier_slab(T=9, N=5, seed=0):
    rng = np.random.default_rng(seed)
    s = rng.standard_normal((T, N, HIER_TRAJ_WIDTH)).astype(np.float32)
    s[:, :, HCOL_DONE] = (rng.random((T, N)) < 0.25).astype(np.float32)
    s[:, :, HCOL_REWARD] = rng.random((T, N)).astype(np.float32)
    s[:, :, HCOL_CODE] = rng.integers(0, 256, (T, N)).astype(np.float32)
    return torch.from_numpy(s)


def test_hier_slab_records():
    T, N = 9, 5
    s = _hier_slab(T, N)
    rng = np.random.default_rng(2)
    init = torch.from_numpy(rng.standard_normal((N, 128)).astype(np.float32))
    first = torch.tensor([1, 0, 1, 0, 0], dtype=torch.uint8)
    boot = torch.from_numpy(rng.standard_normal(N).astype(np.float32))
    rec = hier_slab_records(s, init, first, boot)
    shapes = {"prop": (99,), "prop_a": (36,), "percep_2d": (25, 13), "percep_1d": (128,), "percep_front": (25, 13), "target": (3,)}
    assert list(rec)[:6] == list(shapes)
    c = 0
    for name, sh in shapes.items():
        k = int(np.prod(sh))
        assert tuple(rec[name].shape) == (T, N) + sh
        assert np.array_equal(rec[name].reshape(T, N, k).numpy(), s[:, :, c:c + k].numpy())
        c += k
    assert c == HCOL_ACTION
    assert rec["A_Z"].dtype == torch.int64 and np.array_equal(rec["A_Z"].numpy(), s[:, :, HCOL_CODE].numpy().astype(np.int64))
    assert np.array_equal(rec["neglogp"].numpy(), s[:, :, HCOL_NEGLOGP].numpy()) and np.array_equal(rec["V"].numpy(), s[:, :, HCOL_VALUE].numpy())
    assert np.array_equal(rec["r"].numpy(), s[:, :, HCOL_REWARD].numpy())
    d = s[:, :, HCOL_DONE].numpy()
    assert np.allclose(rec["discount"].numpy(), 0.95 * (1 - d))
    assert np.array_equal(rec["M"][0].numpy(), first.numpy().astype(np.float32)) and np.array_equal(rec["M"][1:].numpy(), d[:-1])
    assert rec["S"] is init
    for i in range(N):                       # the lambda-return recursion written out per env in float64 (test_unroll.py)
        R, Vn = float(boot[i]), float(boot[i])
        for t in range(T - 1, -1, -1):
            disc = 0.95 * (1.0 - float(d[t, i]))
            R = float(s[t, i, HCOL_REWARD]) + disc * (0.05 * Vn + 0.95 * R)
            Vn = float(s[t, i, HCOL_VALUE])
            assert abs(rec["R"][t, i].item() - R) < 1e-5
    with pytest.raises(AssertionError):
        hier_slab_records(s[:, :, :900], init, first, boot)
