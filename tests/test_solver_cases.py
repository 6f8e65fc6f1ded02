"""The designed single-sub-step states of tests/solver_cases.py, checked on the fp64 oracle alone (no GPU): every state takes exactly
the branches it was designed for, and the batches the GPU tests run reach every lane mapping of the step kernel's solver.  Without
these checks a change of the model, the caps or the pairing could make tests/test_solver_cases_gpu.py pass vacuously."""
import numpy as np
import pytest

import solver_cases as sc
from lifelike_agility_and_play_b200 import _capi as capi
from test_golden_epmc import terrain_cfg, terrain_gold
from test_golden_sepmc import SEPMC_CFG

SEED = 20261015


def kind_cfg(kind, element=1):
    """llq_config overrides of the three arenas for single-sub-step, teacher-forced runs (pushes off: they are drawn, not designed)"""
    base = dict(substeps=1, auto_reset=0)
    if kind == "pmc":
        return base
    if kind == "sepmc":
        cfg = dict(SEPMC_CFG); cfg.update(base, push_enabled=0, max_steps=1000, friction_hi=1.0)
        return cfg
    cfg = terrain_cfg(terrain_gold(element)); cfg.update(base, push_enabled=0, max_steps=1000, friction_hi=1.0)
    return cfg


def init_state(kind, element=1):
    if kind == "pmc":
        return None
    if kind == "sepmc":
        from test_golden_sepmc import GOLD
        return np.load(GOLD)["init_state"]
    return terrain_gold(element)["init_state"]


def make(lib, kind, n, blob, mocap, element=1, **over):
    cfg = kind_cfg(kind, element); cfg.update(seed=SEED); cfg.update(over)
    e = capi.VecEngine(lib, n, blob, mocap if kind == "pmc" else None, **cfg)
    if kind != "pmc":
        e.set_init_state(init_state(kind, element))
    e.reset()
    return e


def corridor_statics(eng, element):
    boxes = eng.get(capi.F_BOXES).reshape(eng.n, 36, 6).astype(np.float64)
    nbox = eng.get(capi.F_NBOX)
    aux = kind_cfg("corridor", element)["auxiliary_radius"]
    return boxes, nbox, (lambda i: sc.Statics(boxes=boxes[i, :nbox[i]], aux_r=aux, element=element))


def designed_batch(kind, oracle_lib, blob, mocap, element=1):
    """(states [N, 37] float32, per-env decisions) of the batch a kind's GPU test runs; deterministic"""
    rng = np.random.default_rng(SEED + {"pmc": 0, "sepmc": 1, "corridor": 10 + element}[kind])
    if kind == "corridor":
        eng = make(oracle_lib, kind, 40, blob, mocap, element)
        boxes, nbox, statics_of = corridor_statics(eng, element)
        eng.close()
        return sc.corridor_batch(rng, statics_of, boxes, nbox)
    return sc.ground_batch(rng, sc.Statics(walls=kind == "sepmc"), kind=2 if kind == "sepmc" else 0)


KINDS = [("pmc", 1), ("sepmc", 1), ("corridor", 1), ("corridor", 3)]


@pytest.mark.parametrize("kind,element", KINDS)
def test_designed_states_take_their_branches_on_the_oracle(kind, element, oracle_lib, blob, small_mocap):
    """Each designed state alone in a one-env oracle handle (SEPMC: a pair of two copies), one sub-step: the contact and limit rows
    solved and the rows dropped by the caps are exactly the designed ones, and no decision is within DELTA of its branch."""
    states, decs = designed_batch(kind, oracle_lib, blob, small_mocap, element)
    n = len(states)
    reached = sc.warp_cases([d["nc"] for d in decs], [d["nl"] for d in decs])[1]
    width = 2 if kind == "sepmc" else 1
    worst = np.inf
    for i in range(n):
        e = make(oracle_lib, kind, width, blob, small_mocap, element, global_env_offset=i if kind == "corridor" else 0)
        e.set(capi.F_STATE, np.repeat(states[i:i + 1], width, 0)); e.set(capi.F_WARMSTART, np.zeros((width, 32), np.float32))
        c0 = e.counters().copy()
        e.step(np.zeros((width, 12), np.float32))
        c = (e.counters() - c0) // width
        d = decs[i]
        want = (3 * min(d["nc"], sc.MAX_CON), min(d["nl"], sc.MAX_LIM), max(d["nc"] - sc.MAX_CON, 0) + max(d["nl"] - sc.MAX_LIM, 0))
        assert (c[2], c[3], c[5]) == want, (kind, i, d["nc"], d["nl"], c)
        m = float(e.get(capi.F_DECISION_MARGIN).min())
        worst = min(worst, m)
        assert m >= 0.999 * sc.DELTA_C, (kind, i, m)
        e.close()
    print("%s: %d designed states, smallest oracle decision margin %.1e; mapping cases of the batch: %s" % (kind, n, worst, sorted(reached)))


@pytest.mark.parametrize("kind,element", KINDS)
def test_designed_batches_reach_every_lane_mapping(kind, element, oracle_lib, blob, small_mocap):
    states, decs = designed_batch(kind, oracle_lib, blob, small_mocap, element)
    mapping, reached = sc.warp_cases([d["nc"] for d in decs], [d["nl"] for d in decs])
    print("%s: %d envs, cases reached: %s" % (kind, len(states), sorted(reached)))
    if kind == "corridor":
        assert reached & {"two_pass", "borrow", "borrow_empty"}, reached
        nz = np.concatenate([d["nz"] for d in decs])
        # box tops (|n.z| = 1) and faces (0), and edge-cylinder / box-edge normals on both sides of btPlaneSpace1's branch
        general = nz[(nz > 1e-6) & (nz < 1 - 1e-6)]
        assert (general > np.sqrt(0.5)).any() and (general < np.sqrt(0.5)).any() and (nz == 1).any() and (nz == 0).any(), general
    else:
        assert reached == set(sc.CASES), set(sc.CASES) - reached
    pens = np.concatenate([d["pen"] for d in decs])
    if kind != "corridor":
        # limit rows on both sides of the split-impulse threshold, some of them within 1 cm of it on the deep side
        assert (pens > sc.SPLIT_PEN).any() and (pens < sc.SPLIT_PEN - 0.005).any() and ((pens < sc.SPLIT_PEN) & (pens > -0.05)).any()


def test_the_mapping_follows_the_documented_rule():
    """warp_cases on hand-made counts: ties go to the lower slot, warp w pairs ranks w and 15 - w, unused slots copy env N - 1"""
    # CTA 0: 32 rows, two of 20, 7, 4 and eleven empty envs; CTA 1: eight of 19 rows and eight of 3; CTA 2: env 32 (17 rows, 9
    # limit rows) and its 15 copies
    nc = [8, 0, 2, 6, 6, 1] + [0] * 10 + [6] * 8 + [1] * 8 + [3]
    nl = [8, 0, 1, 2, 2, 1] + [0] * 10 + [1] * 8 + [0] * 8 + [9]
    m, reached = sc.warp_cases(nc, nl)
    assert m[0][2:] == (0, 15, 32, 0, "exact32")
    assert m[1][2:] == (3, 14, 20, 0, "borrow_empty") and m[2][2:] == (4, 13, 20, 0, "borrow_empty")
    assert m[3][2:] == (2, 12, 7, 0, "split16") and m[4][2:] == (5, 11, 4, 0, "split16") and m[7][2:] == (7, 8, 0, 0, "empty")
    assert [x[2:] for x in m[8:16]] == [(16 + w, 31 - w, 19, 3, "borrow") for w in range(8)]
    assert all(x[6] == "two_pass" and x[2] == x[3] == 32 for x in m[16:])
    assert reached == {"exact32", "borrow", "borrow_empty", "split16", "empty", "two_pass", "limit_cap", "shadow"}
    assert sc.lane_offset(m, 31) == 19 and sc.lane_offset(m, 16) == 0 and sc.lane_offset(m, 3) == 0 and sc.lane_offset(m, 32) == 0


# ---------------------------------------------------------------------------------------------------------------- corridor window
def _kernel_constant(fname, pattern):
    """a constant read from the step kernel's source, so that the window tests follow the kernel"""
    import os
    import re
    src = open(os.path.join(os.path.dirname(sc.__file__), "..", "lifelike_agility_and_play_b200", "csrc", fname)).read()
    found = re.findall(pattern, src)
    assert len(found) == 1, (fname, pattern, found)
    return float(found[0])


# boxes whose footprint lies within the window (m, per axis) of the base are contact candidates; the first kMaxCand of them are kept
KERNEL_WINDOW = _kernel_constant("llq_step16.cuh", r"box_mask\(bxs, E\.nbox\[env\], k, \(float\)px, \(float\)py, \(float\)pz, ([0-9.]+)f, false\)")
KERNEL_MAX_CAND = int(_kernel_constant("llq_kernels.cuh", r"kMaxCand = ([0-9]+);"))


def test_every_sphere_stays_inside_the_candidate_window():
    """Over the joint ranges (plus 0.04 rad past the stops) and any base orientation, a sphere's horizontal offset from the base, plus
    its radius, the contact breaking distance, the auxiliary cylinder radius and 0.06 m of travel in one step, fits in the window."""
    rng = np.random.default_rng(1)
    reach = 0.0
    for t in range(3000):
        q = rng.uniform(sc.LOWER - 0.04, sc.UPPER + 0.04)
        if t % 3 == 0:                         # legs stretched: extremes of every joint
            q = np.where(rng.random(12) < 0.5, sc.LOWER - 0.04, sc.UPPER + 0.04)
        off = sc.sphere_offsets(np.array([0, 0, 0, 1.0]), q)
        reach = max(reach, float(np.max(np.linalg.norm(off, axis=1) + sc.RADIUS)))      # any orientation turns this onto an axis
    need = reach + sc.BREAKING + 0.02 + 0.06
    print("farthest sphere surface from the base CoM: %.3f m; window needed %.3f m of %.2f" % (reach, need, KERNEL_WINDOW))
    assert need <= KERNEL_WINDOW


@pytest.mark.parametrize("element", [1, 2, 3])
def test_no_corridor_puts_more_boxes_in_reach_than_the_kernel_keeps(element, oracle_lib, blob):
    """Corridors from the reset (many seeds): at any base position in the corridor, the boxes whose footprint lies within the window
    number at most kMaxCand -- the kernel keeps the first kMaxCand candidates and would silently skip the rest."""
    worst = 0
    for seed in range(4):
        eng = make(oracle_lib, "corridor", 256, blob, None, element, seed=seed)
        boxes = eng.get(capi.F_BOXES).reshape(256, 36, 6).astype(np.float64); nbox = eng.get(capi.F_NBOX)
        eng.close()
        for i in range(256):
            b = boxes[i, :nbox[i]]
            lo_y, hi_y = b[0, 1] + b[0, 4], b[1, 1] - b[1, 4]        # between the inner faces of the two walls
            if lo_y > hi_y:
                lo_y, hi_y = hi_y, lo_y
            xs = np.arange(b[2:, 0].min() - 1.0, b[2:, 0].max() + 1.0, 0.02) if len(b) > 2 else np.zeros(1)
            ys = np.linspace(lo_y, hi_y, 9)
            X, Y = np.meshgrid(xs, ys)
            inx = np.abs(b[None, None, :, 0] - X[..., None]) <= b[None, None, :, 3] + KERNEL_WINDOW
            iny = np.abs(b[None, None, :, 1] - Y[..., None]) <= b[None, None, :, 4] + KERNEL_WINDOW
            worst = max(worst, int((inx & iny).sum(-1).max()))
    print("element %d: at most %d boxes within the window" % (element, worst))
    assert worst <= KERNEL_MAX_CAND
