"""The strategic level's training forward on the CPU: its fp64 statement (tests/strategic_train_cases.py) against the fp32 host class
`SepmcPolicy` (value tower, heading sampled from given eps, -log p), the designed batch, the learner tensors of an unroll, and the
resources of the three kernel instances."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import policy_cases as pc
import strategic_train_cases as sc
from lifelike_agility_and_play_b200.parallel import sepmc_slab_records
from lifelike_agility_and_play_b200.parallel.trajectory import (SCOL_ACTION, SCOL_CODE, SCOL_DONE, SCOL_HEADING, SCOL_NEGLOGP, SCOL_REWARD,
                                                                SCOL_VALUE, SEPMC_TRAJ_WIDTH)
from lifelike_agility_and_play_b200.policy_epmc import SEPMC_SHAPES, SepmcPolicy, hier_role_arrays, strategic_train_role_arrays

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _agree(got, ref, S, name, factor=64.0):
    err = np.abs(np.asarray(got, np.float64) - ref)
    bar = factor * S + 1e-6 * np.abs(ref) + 1e-7
    assert (err <= bar).all(), (name, float((err / bar).max()))


def test_training_table_matches_the_shipped_shapes():
    roles = strategic_train_role_arrays()
    assert len(roles) == 50 and roles[0] == 2 and roles[48] == 50 and roles[49] == 96
    shapes = [SEPMC_SHAPES[i] for i in roles]
    assert shapes[0] == (135, 128) and shapes[26] == (88, 64) and shapes[28] == (64, 128)
    assert shapes[30] == (29, 64) and shapes[32] == (64, 64) and shapes[34] == (64, 128) and shapes[36] == (384, 256)
    assert shapes[38] == (256, 128) and shapes[47] == (32, 1) and shapes[48] == (1,) and shapes[49] == (1, 1)
    with pytest.raises(ValueError):
        hier_role_arrays(True, value_tower=True)


def test_draw_is_formed_as_the_kernel_forms_it():
    """u0 = ((float)r.x + 0.5f) 2^-32 and u1 = (float)r.y 2^-32 in fp32 from the Philox words of q = 64 (the numpy Philox is pinned to
    the Random123 known answers in test_policy_cases.py); r.x >= 2^32 - 128 is clamped to 0.99999994f, so eps stays finite."""
    gid = sc.ROW_GID0 + np.arange(5)
    rx, u0, u1, ang = sc.draws(gid, sc.SEED, sc.COUNTER_BASE)
    c = pc.philox4x32(gid[3] & 0xFFFFFFFF, 64, sc.COUNTER_BASE & 0xFFFFFFFF, sc.COUNTER_BASE >> 32, sc.SEED & 0xFFFFFFFF, sc.SEED >> 32)
    f = np.float32
    assert int(rx[3]) == int(c[0]) and u0.dtype == np.float32
    assert u0[3] == (f(int(c[0])) + f(0.5)) * f(2.0 ** -32) and u1[3] == f(int(c[1])) * f(2.0 ** -32)
    assert ang[3] == f(6.283185307179586) * u1[3]
    eps = sc.eps_of(gid, sc.SEED, sc.COUNTER_BASE)
    assert np.allclose(eps, np.sqrt(-2.0 * np.log(u0.astype(np.float64))) * np.cos(ang.astype(np.float64)))
    c1, i1 = sc.search_clamp_counter(sc.N, sc.COUNTER_BASE)
    rx, u0, _, _ = sc.draws(sc.ROW_GID0 + np.array([i1]), sc.SEED, c1)
    assert int(rx[0]) >= sc.CLAMP_R and u0[0] == f(0.99999994) and np.isfinite(sc.eps_of(sc.ROW_GID0 + np.array([i1]), sc.SEED, c1)).all()


def test_statement_agrees_with_the_fp32_class():
    rng = np.random.default_rng(6)
    w = sc.design_weights(3)
    n = 96
    obs = np.stack([pc._hier_row(rng, "random", 965) for _ in range(n)])
    state = pc.hier_random_state(rng, n, 192)
    done = pc.DONE_BYTES[np.arange(n) % 4]
    gid = sc.ROW_GID0 + np.arange(n)
    ref, S = sc.train_eval(sc.Trunks(w, obs, state, done), gid, sc.SEED, sc.COUNTER_BASE)
    mask = (done != 0).astype(np.float32)
    host = SepmcPolicy(w)
    a, st, head, code, nlp = host.act(obs, state[:, :128], mask, return_aux=True, eps=ref["eps"], return_neglogp=True)
    v, vst = host.value(obs, state[:, 128:], mask)
    dec = sc.decisive(ref, S)
    assert dec.mean() > 0.9
    assert np.array_equal(code[dec], ref["code"][dec])
    _agree(head, ref["heading"], S["heading"], "heading")
    _agree(nlp, ref["neglogp"], S["neglogp"], "-log p")
    _agree(v, ref["value"], S["value"], "value")
    _agree(np.concatenate([st, vst], axis=1)[dec], ref["state"][dec], S["state"][dec], "state")
    _agree(a[dec], ref["actions"][dec], S["actions"][dec], "actions")
    # without eps the class keeps its deterministic result: the clipped mean heading
    a0, st0, head0, code0 = host.act(obs, state[:, :128], mask, return_aux=True)
    assert np.allclose(head0, np.clip(ref["mu"], -np.pi, np.pi), atol=1e-4)


def test_designed_batch_reaches_every_category_and_every_row_is_decisive():
    w, obs, state, done, counters, info, evals, mean_codes = sc.train_case()
    assert obs.shape == (sc.N, 965) and state.shape == (sc.N, 192) and len(counters) == 2
    reached = sc.reaches(w, obs, state, done, counters, info, evals, mean_codes)
    missing = {k: (len(v) - sum(v), len(v)) for k, v in reached.items() if not any(v)}
    assert not missing, missing
    for ref, S in evals:
        assert sc.decisive(ref, S).all()
        assert np.isfinite(ref["neglogp"]).all() and np.isfinite(ref["heading"]).all()


def _sepmc_slab(T=9, P=5, seed=0):
    rng = np.random.default_rng(seed)
    s = rng.standard_normal((T, 2 * P, SEPMC_TRAJ_WIDTH)).astype(np.float32)
    d = (rng.random((T, P)) < 0.25).astype(np.float32)
    s[:, 0::2, SCOL_DONE] = d
    s[:, 1::2, SCOL_DONE] = d
    s[:, :, SCOL_REWARD] = rng.random((T, 2 * P)).astype(np.float32)
    s[:, :, SCOL_CODE] = rng.integers(0, 256, (T, 2 * P)).astype(np.float32)
    return torch.from_numpy(s)


def test_sepmc_slab_records():
    T, P = 9, 5
    s = _sepmc_slab(T, P)
    s0 = s[:, 0::2].numpy()
    rng = np.random.default_rng(2)
    init = torch.from_numpy(rng.standard_normal((P, 192)).astype(np.float32))
    first = torch.tensor([1, 0, 1, 0, 0], dtype=torch.uint8)
    boot = torch.from_numpy(rng.standard_normal(P).astype(np.float32))
    rec = sepmc_slab_records(s, init, first, boot)
    shapes = {"prop": (99,), "prop_a": (36,), "percept_2d": (25, 13), "percept_1d": (128,), "percept_front": (25, 13), "percept_vec": (5,),
              "oppo_info": (15,), "oppo_info_cheat": (15,), "flag_info": (7,), "flag_info_cheat": (7,), "with_flag": (2,), "control_spd": (1,)}
    assert list(rec) == list(shapes) + ["A_HLC", "A_Z", "neglogp", "discount", "r", "V", "R", "M", "S"]
    c = 0
    for name, sh in shapes.items():
        k = int(np.prod(sh))
        assert tuple(rec[name].shape) == (T, P) + sh
        assert np.array_equal(rec[name].reshape(T, P, k).numpy(), s0[:, :, c:c + k])
        c += k
    assert c == SCOL_ACTION
    assert np.array_equal(rec["A_HLC"].numpy(), s0[:, :, SCOL_HEADING])
    assert rec["A_Z"].dtype == torch.int64 and np.array_equal(rec["A_Z"].numpy(), s0[:, :, SCOL_CODE].astype(np.int64))
    assert np.array_equal(rec["neglogp"].numpy(), s0[:, :, SCOL_NEGLOGP]) and np.array_equal(rec["V"].numpy(), s0[:, :, SCOL_VALUE])
    assert np.array_equal(rec["r"].numpy(), s0[:, :, SCOL_REWARD])
    d = s0[:, :, SCOL_DONE]
    assert np.allclose(rec["discount"].numpy(), 0.95 * (1 - d))
    assert np.array_equal(rec["M"][0].numpy(), first.numpy().astype(np.float32)) and np.array_equal(rec["M"][1:].numpy(), d[:-1])
    assert rec["S"] is init
    for i in range(P):                       # the lambda-return recursion written out per pair in float64 (test_unroll.py)
        R, Vn = float(boot[i]), float(boot[i])
        for t in range(T - 1, -1, -1):
            disc = 0.95 * (1.0 - float(d[t, i]))
            R = float(s0[t, i, SCOL_REWARD]) + disc * (0.05 * Vn + 0.95 * R)
            Vn = float(s0[t, i, SCOL_VALUE])
            assert abs(rec["R"][t, i].item() - R) < 1e-5
    with pytest.raises(AssertionError):
        sepmc_slab_records(s[:, :, :936], init, first, boot)
    with pytest.raises(AssertionError):
        sepmc_slab_records(s[:, :9], init, first, boot)


def test_kernel_instances_fit_two_ctas_per_sm():
    """All three instances of hier_policy_kernel (deterministic, environmental training, strategic training): at most 128 registers
    and no spills, so two CTAs of 256 threads fit the 64 K register file; their shared memory is the dynamic `Smem` block
    (103 424 B, two per SM), with no static shared memory."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "lifelike_agility_and_play_b200", "csrc", "llq_policy_hier.cu")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c", "-o", os.devnull, src],
                         capture_output=True, text=True, check=True).stderr
    found = {}
    for block in out.split("Compiling entry function")[1:]:
        m = re.search(r"hier_policy_kernelILi(\d)E", block)
        if not m:
            continue
        regs = int(re.search(r"Used (\d+) registers", block).group(1))
        spills = [int(x) for x in re.findall(r"(\d+) bytes spill (?:stores|loads)", block)]
        smem = re.search(r"(\d+) bytes smem", block)
        found[int(m.group(1))] = (regs, spills, int(smem.group(1)) if smem else 0)
    assert sorted(found) == [0, 1, 2], out
    for mode, (regs, spills, smem) in found.items():
        assert regs <= 128 and spills == [0, 0] and smem == 0, (mode, regs, spills, smem)
