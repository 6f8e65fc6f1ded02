"""The perception rays of the EPMC and SEPMC observations against the fp64 caster of tests/perception_cases.py, on the oracle alone
(no GPU): the caster agrees with the pybullet shim's independent slab test, the oracle's observation on the designed poses matches
the caster ray by ray, the physics-off step leaves every pose where it was set, the batches reach every category, and the kernel's
candidate windows cover the rays' reach.  Without these checks tests/test_perception_cases_gpu.py could pass vacuously."""
import os
import re

import numpy as np
import pytest

import perception_cases as pc
from lifelike_agility_and_play_b200 import _capi as capi
from test_golden_epmc import EPMC_CFG, GOLD as EPMC_GOLD
from test_solver_cases import init_state, kind_cfg

SEED = 20261016
# one sub-step without forces: no solver iteration, no PD torque, no gravity, no push; with zero velocities the pose stays put
PHYSICS_OFF = dict(substeps=1, solver_iters=0, kp=0.0, kd=0.0, gravity_z=0.0, push_enabled=0, auto_reset=0)
N_CORRIDOR, N_FLAT, N_PAIRS = 45, 21, 23          # not multiples of 8 or 16: the last warp has padded rows
CASES = [("epmc", 0), ("epmc", 1), ("epmc", 2), ("epmc", 3), ("sepmc", 0)]


def config(kind, element):
    if kind == "sepmc":
        cfg = kind_cfg("sepmc")
    elif element == 0:
        cfg = dict(EPMC_CFG); cfg.update(max_steps=1000, friction_hi=1.0)
    else:
        cfg = kind_cfg("corridor", element)
    cfg.update(PHYSICS_OFF, seed=SEED)
    return cfg


def make(lib, kind, element, n):
    e = capi.VecEngine(lib, n, _blob(), None, **config(kind, element))
    e.set_init_state(init_state("sepmc") if kind == "sepmc" else (np.load(EPMC_GOLD)["init_state"] if element == 0 else init_state("corridor", element)))
    e.reset()
    return e


_BLOB = []


def _blob():
    if not _BLOB:
        from lifelike_agility_and_play_b200.model.compile_model import pack_model
        _BLOB.append(pack_model(pc.sc.MODEL))
    return _BLOB[0]


_BATCHES = {}


def designed(kind, element, oracle_lib):
    """(n, states, aux to set or None, categories, builder's visibility or None) of a case; deterministic, cached"""
    key = (kind, element)
    if key not in _BATCHES:
        rng = np.random.default_rng(SEED + 10 * element + (5 if kind == "sepmc" else 0))
        if kind == "sepmc":
            states, flags, cats, vis = pc.sepmc_batch(rng, N_PAIRS)
            n = len(states)
            e = make(oracle_lib, kind, element, n)
            aux = e.get(capi.F_AUX)
            e.close()
            aux[:, 2] = np.repeat(flags[:, 0], 2); aux[:, 3] = np.repeat(flags[:, 1], 2)
            _BATCHES[key] = (n, states, aux, cats, vis)
        elif element == 0:
            states, cats = pc.flat_batch(rng, N_FLAT)
            _BATCHES[key] = (N_FLAT, states, None, cats, None)
        else:
            e = make(oracle_lib, kind, element, N_CORRIDOR)
            boxes = e.get(capi.F_BOXES).reshape(N_CORRIDOR, capi.MAX_BOXES, 6).astype(np.float64)
            nbox = e.get(capi.F_NBOX)
            e.close()
            states, cats = pc.corridor_batch(rng, boxes, nbox, element)
            _BATCHES[key] = (N_CORRIDOR, states, None, cats, None)
    return _BATCHES[key]


def prepared(lib, kind, element, oracle_lib, src=None):
    """an engine over the designed batch, ready to step: the designed states (and SEPMC flags) set on the oracle's reset, or every
    per-env field copied from src"""
    n, states, aux, cats, _ = designed(kind, element, oracle_lib)
    e = make(lib, kind, element, n)
    if src is not None:
        for f in (capi.F_STATE, capi.F_WARMSTART, capi.F_OBS, capi.F_TIME, capi.F_AUX, capi.F_EPISODE_ID, capi.F_REWARD_SUM):
            e.set(f, src.get(f))
        return e
    e.set(capi.F_STATE, states); e.set(capi.F_WARMSTART, np.zeros((n, 32), np.float32))
    if aux is not None:
        e.set(capi.F_AUX, aux)
    return e


def step(e):
    """one step with zero actions: (obs, post-step state, post-step aux, boxes, nbox)"""
    obs = e.step(np.zeros((e.n, 12), np.float32))[0]
    return obs, e.get(capi.F_STATE), e.get(capi.F_AUX), e.get(capi.F_BOXES).reshape(e.n, capi.MAX_BOXES, 6).astype(np.float64), e.get(capi.F_NBOX)


def assert_pose_kept(st, designed_states, qtol=1e-7):
    """the physics is off: the pose after the step is the pose that was set"""
    assert np.array_equal(st[:, 0:3], designed_states[:, 0:3])
    q, q0 = st[:, 3:7].astype(np.float64), designed_states[:, 3:7].astype(np.float64)
    q *= np.sign(np.sum(q * q0, 1))[:, None]
    assert np.abs(q - q0).max() <= qtol, np.abs(q - q0).max()


def reference_rows(kind, st, aux, boxes, nbox):
    """caster values of obs 135.. and their sensitivity, per env, on the given (post-step) states"""
    n = len(st)
    V, S = [], []
    if kind == "sepmc":
        for p in range(n // 2):
            a, b = st[2 * p].astype(np.float64), st[2 * p + 1].astype(np.float64)
            vis = pc.visible(a, b, pc.arena_boxes(aux[2 * p, 2], aux[2 * p, 3]))
            for i, (s, o) in enumerate(((a, b), (b, a))):
                v, s_ = pc.sepmc_row(s, o, aux[2 * p + i], aux[2 * p + 1 - i], vis[i])
                V.append(v); S.append(s_)
    else:
        for i in range(n):
            bx = pc.corridor_boxes(boxes[i, :nbox[i]]) if nbox[i] > 0 else pc.SLAB
            v, s_ = pc.epmc_row(st[i], bx, aux[i])
            V.append(v); S.append(s_)
    return np.array(V), np.array(S)


def post_pose_decisive(kind, st, aux, boxes, nbox):
    ok = []
    for i in range(len(st)):
        s = st[i].astype(np.float64)
        bx = pc.arena_boxes(aux[i, 2], aux[i, 3]) if kind == "sepmc" else (pc.corridor_boxes(boxes[i, :nbox[i]]) if nbox[i] > 0 else pc.SLAB)
        ok.append(pc.rays_decisive(s[0:3], pc.rot(s[3:7]), bx))
    return np.array(ok)


ORACLE_A = 1e-5


@pytest.mark.parametrize("kind,element", CASES)
def test_the_oracle_matches_the_caster_ray_by_ray(kind, element, oracle_lib):
    e = prepared(oracle_lib, kind, element, oracle_lib)
    obs, st, aux, boxes, nbox = step(e)
    e.close()
    n, designed_states, _, _, vis = designed(kind, element, oracle_lib)
    assert_pose_kept(st, designed_states)
    if kind == "sepmc":
        assert not aux[:, 6].any(), "a flag switch moved the flag during the step"
        assert np.array_equal(aux[:, 5] != 0, vis), "oppo_visible"
    ref, S = reference_rows(kind, st, aux, boxes, nbox)
    got = obs[:, 135:].astype(np.float64)
    err = np.abs(got - ref)
    bar = ORACLE_A * np.maximum(1.0, np.abs(ref)) + 4 * S
    print("%s element %d: %d envs, max |oracle - caster| %.1e, largest S %.1e" % (kind, element, len(st), err.max(), S.max()))
    assert np.all(err <= bar), [(int(i), int(j) + 135, got[i, j], ref[i, j]) for i, j in np.argwhere(err > bar)[:10]]
    assert post_pose_decisive(kind, st, aux, boxes, nbox).all()


# ---------------------------------------------------------------------------------------------------------------- categories
@pytest.mark.parametrize("kind,element", CASES)
def test_the_designed_batches_reach_every_category(kind, element, oracle_lib):
    n, states, aux, cats, vis = designed(kind, element, oracle_lib)
    counts = {c: cats.count(c) for c in sorted(set(cats))}
    print("%s element %d: %d envs, categories %s" % (kind, element, n, counts))
    want = {0: pc.FLAT_CATS, 1: pc.CORRIDOR_CATS, 2: pc.CORRIDOR_CATS, 3: pc.CORRIDOR_CATS + ("high_mask",)}[element] if kind == "epmc" else pc.SEPMC_CATS
    assert set(want) <= set(cats), set(want) - set(cats)
    assert n % 8 != 0
    # every env reaches what its category is named for
    if kind == "sepmc":
        assert vis.any() and not vis.all(), "pairs on both sides of oppo_visible"
        missed = [(p, cats[p]) for p in range(n // 2) if not pc.reaches("sepmc", cats[p], states[2 * p], pc.arena_boxes(aux[2 * p, 2], aux[2 * p, 3]))]
    elif element == 0:
        missed = [(i, cats[i]) for i in range(n) if not pc.reaches("flat", cats[i], states[i], pc.SLAB)]
    else:
        bx = [pc.corridor_boxes(b) for b in _boxes(element, oracle_lib)]
        missed = [(i, cats[i]) for i in range(n) if not pc.reaches("corridor", cats[i], states[i], bx[i])]
    assert not missed, missed


_BOX_CACHE = {}


def _boxes(element, oracle_lib):
    if element not in _BOX_CACHE:
        e = make(oracle_lib, "epmc", element, N_CORRIDOR)
        b = e.get(capi.F_BOXES).reshape(N_CORRIDOR, capi.MAX_BOXES, 6).astype(np.float64)
        nb = e.get(capi.F_NBOX)
        e.close()
        _BOX_CACHE[element] = [b[i, :nb[i]] for i in range(N_CORRIDOR)]
    return _BOX_CACHE[element]


# ---------------------------------------------------------------------------------------------------------------- the shim
def _shim_client(boxes):
    from golden import pybullet_shim as shim
    c = shim.FakeBulletClient.__new__(shim.FakeBulletClient)
    c.bodies = []
    for b in boxes[1:]:                                  # the shim adds the ground slab itself
        body = shim._Body("static")
        body.box = (b[3:] - b[:3]) / 2
        body.ray_target = True
        body.state[0:3] = (b[3:] + b[:3]) / 2
        c.bodies.append(body)
    return c


@pytest.mark.parametrize("arena", ["sepmc", "corridor"])
def test_the_caster_agrees_with_the_shims_slab_test(arena, oracle_lib):
    """A few thousand random segments, many of them from inside a box or axis-parallel: same hit / miss, same first box, same
    fraction (to 1e-12) as pybullet_shim.FakeBulletClient.rayTestBatch."""
    rng = np.random.default_rng(5)
    sets = [pc.arena_boxes(0.7, -1.2)] if arena == "sepmc" else [pc.corridor_boxes(b) for b in _boxes(3, oracle_lib)[:4]]
    total = 0
    for boxes in sets:
        c = _shim_client(boxes)
        lo, hi = boxes[1:, :3].min(0) - 1, boxes[1:, 3:].max(0) + 1
        o = rng.uniform(lo, hi, (800, 3))
        e = o + rng.normal(0, 3, (800, 3))
        e[::4, 2] = o[::4, 2]                            # horizontal
        e[1::4, :2] = o[1::4, :2]                        # vertical
        o[2::8] = (boxes[1 + rng.integers(len(boxes) - 1, size=100), :3] + boxes[1 + rng.integers(len(boxes) - 1, size=100), 3:])[:100] / 2
        f, j, ax, inside = pc.cast(o, e, boxes)
        res = c.rayTestBatch(o, e)
        for k, r in enumerate(res):
            if r[0] == -1:
                assert f[k] < 0, (k, f[k])
            else:
                assert f[k] >= 0 and abs(f[k] - r[2]) <= 1e-12, (k, f[k], r[2])
                uid = r[0]
                assert (j[k] == 0) if uid == len(c.bodies) else (j[k] == uid + 1), (k, j[k], uid)
        total += len(o)
        assert (f >= 0).any() and (f < 0).any()
    print("%s: %d segments agree" % (arena, total))


# ---------------------------------------------------------------------------------------------------------------- windows
def _kernel_constants(pattern):
    src = open(os.path.join(os.path.dirname(pc.__file__), "..", "lifelike_agility_and_play_b200", "csrc", "llq_kernels.cuh")).read()
    return re.findall(pattern, src)


def test_the_candidate_windows_cover_the_rays_reach():
    """stage_corridor_masks keeps the boxes whose footprint lies within a window of the base: the down-ray grid's corner reaches
    hypot(1.2, 0.6) = 1.342 m from the base in any yaw, a front ray's end |(3, 0.25, 0.3)| = 3.025 m in any orientation.
    ray_boxlist's culling pad around the segment's bounds must not be negative (it would drop grazing boxes)."""
    grid = [float(x) for x in _kernel_constants(r"box_mask\(boxes, nb, k, px, py, pz, ([0-9.]+)f, false\);   // 2\.4 x 1\.2")]
    front = [float(x) for x in _kernel_constants(r"box_mask\(boxes, nb, k, px, py, pz, ([0-9.]+)f, false\);   // 3 m rays")]
    pads = [float(x) for x in _kernel_constants(r"fminf\(o\.x, ex\) - ([0-9.e+-]+)f")]
    assert len(grid) == len(front) == len(pads) == 1, (grid, front, pads)
    g = np.stack(np.meshgrid(pc.GX, pc.GY, indexing="ij"), -1).reshape(-1, 2)
    f = np.stack(np.meshgrid(pc.FY, pc.FZ, indexing="ij"), -1).reshape(-1, 2)
    grid_reach = np.linalg.norm(g, axis=1).max()
    front_reach = np.sqrt(9.0 + (f ** 2).sum(1)).max()
    print("grid reach %.4f m of a %.2f m window; front reach %.4f m of %.2f m; culling pad %g m" % (grid_reach, grid[0], front_reach, front[0], pads[0]))
    assert abs(grid_reach - pc.GRID_REACH) < 1e-12 and abs(front_reach - pc.FRONT_REACH) < 1e-12
    assert grid[0] >= grid_reach and front[0] >= front_reach and pads[0] >= 0
