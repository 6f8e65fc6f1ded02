"""The designed single-sub-step states of tests/solver_cases.py, checked on the fp64 oracle alone (no GPU): every state takes exactly
the branches it was designed for, and the batches the GPU tests run reach every lane mapping of the step kernel's solver.  Without
these checks a change of the model, the caps or the pairing could make tests/test_solver_cases_gpu.py pass vacuously."""
import numpy as np
import pytest

import solver_cases as sc
from lifelike_agility_and_play_b200 import _capi as capi
from test_golden_epmc import EPMC_CFG, GOLD as EPMC_GOLD, terrain_cfg, terrain_gold
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
    if kind == "epmc":                                 # the flat arena, element 0
        cfg = dict(EPMC_CFG); cfg.update(base, push_enabled=0, max_steps=1000, friction_hi=1.0)
        return cfg
    cfg = terrain_cfg(terrain_gold(element)); cfg.update(base, push_enabled=0, max_steps=1000, friction_hi=1.0)
    return cfg


def init_state(kind, element=1):
    if kind == "pmc":
        return None
    if kind == "sepmc":
        from test_golden_sepmc import GOLD
        return np.load(GOLD)["init_state"]
    if kind == "epmc":
        return np.load(EPMC_GOLD)["init_state"]
    return terrain_gold(element)["init_state"]


def make(lib, kind, n, blob, mocap, element=1, **over):
    cfg = kind_cfg(kind, element); cfg.update(seed=SEED); cfg.update(over)
    e = capi.VecEngine(lib, n, blob, mocap if kind == "pmc" else None, **cfg)
    if kind != "pmc":
        e.set_init_state(init_state(kind, element))
    e.reset()
    return e


def corridor_statics(eng, element, rule=2):
    boxes = eng.get(capi.F_BOXES).reshape(eng.n, 36, 6).astype(np.float64)
    nbox = eng.get(capi.F_NBOX)
    aux = kind_cfg("corridor", element)["auxiliary_radius"]
    return boxes, nbox, (lambda i: sc.Statics(boxes=boxes[i, :nbox[i]], aux_r=aux, element=element, rule=rule))


def designed_batch(kind, oracle_lib, blob, mocap, element=1, rule=2):
    """(states [N, 37] float32, per-env decisions) of the batch a kind's GPU test runs (rule = llq_config.knee_contacts);
    deterministic"""
    rng = np.random.default_rng(SEED + {"pmc": 0, "sepmc": 1, "epmc": 20, "corridor": 10 + element}[kind] + 100 * (2 - rule))
    if kind == "corridor":
        eng = make(oracle_lib, kind, 40, blob, mocap, element)
        boxes, nbox, statics_of = corridor_statics(eng, element, rule)
        eng.close()
        if rule != 2:
            return sc.legacy_batch(rng, statics_of, 40, rule, boxes=int(nbox.min()))
        return sc.corridor_batch(rng, statics_of, boxes, nbox, element)
    S = sc.Statics(walls=kind == "sepmc", rule=rule)
    if rule != 2:
        return sc.legacy_batch(rng, lambda i: S, 40, rule)
    return sc.ground_batch(rng, S, kind=2 if kind == "sepmc" else 0)


KINDS = [("pmc", 1), ("sepmc", 1), ("corridor", 1), ("corridor", 3), ("epmc", 0), ("corridor", 2)]
# the legacy contact sets (llq_config.knee_contacts 0: the feet, 1: feet and knee wheels, one contact per leg)
LEGACY = [(k, 1, r) for k in ("pmc", "sepmc", "corridor") for r in (0, 1)]


def oracle_one_by_one(oracle_lib, blob, mocap, kind, element, states, decs, **over):
    """Each designed state alone in a one-env oracle handle (SEPMC: a pair of two copies), one sub-step: the contact and limit rows
    solved and the rows dropped by the caps are exactly the designed ones, and no decision is within DELTA of its branch.  Returns
    the smallest oracle decision margin."""
    width = 2 if kind == "sepmc" else 1
    worst = np.inf
    for i in range(len(states)):
        e = make(oracle_lib, kind, width, blob, mocap, element, global_env_offset=i if kind == "corridor" else 0, **over)
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
    return worst


@pytest.mark.parametrize("kind,element", KINDS)
def test_designed_states_take_their_branches_on_the_oracle(kind, element, oracle_lib, blob, small_mocap):
    """Each designed state alone in a one-env oracle handle (SEPMC: a pair of two copies), one sub-step: the contact and limit rows
    solved and the rows dropped by the caps are exactly the designed ones, and no decision is within DELTA of its branch."""
    states, decs = designed_batch(kind, oracle_lib, blob, small_mocap, element)
    reached = sc.warp_cases([d["nc"] for d in decs], [d["nl"] for d in decs])[1]
    worst = oracle_one_by_one(oracle_lib, blob, small_mocap, kind, element, states, decs)
    print("%s element %d: %d designed states, smallest oracle decision margin %.1e; mapping cases of the batch: %s" % (
        kind, element, len(states), worst, sorted(reached)))


@pytest.mark.parametrize("kind,element", KINDS)
def test_designed_batches_reach_every_lane_mapping(kind, element, oracle_lib, blob, small_mocap):
    states, decs = designed_batch(kind, oracle_lib, blob, small_mocap, element)
    mapping, reached = sc.warp_cases([d["nc"] for d in decs], [d["nl"] for d in decs])
    print("%s element %d: %d envs, cases reached: %s" % (kind, element, len(states), sorted(reached)))
    if kind == "corridor" and element == 2:
        assert reached & {"two_pass", "borrow", "borrow_empty"}, reached
        nrm = np.concatenate([d["normal"] for d in decs]); kd = np.concatenate([d["kind"] for d in decs])
        cyl_nz = np.abs(nrm[kd == 2, 2])
        # bottom faces (n = -z), corners inside a bar, bottom-edge cylinders on both sides of btPlaneSpace1's branch, both cylinders
        assert (nrm[kd == 1, 2] == -1).any(), nrm[kd == 1]
        assert sum(d["inside"] for d in decs) > 0
        assert (cyl_nz > np.sqrt(0.5)).any() and (cyl_nz < np.sqrt(0.5)).any(), cyl_nz
        assert (nrm[kd == 2, 0] > 0).any() and (nrm[kd == 2, 0] < 0).any()
        # every bar robot also stands on the ground
        assert all(d["nc"] > d["n_off_ground"] for d in decs if d["n_off_ground"])
    elif kind == "corridor":
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


@pytest.mark.parametrize("kind,element,rule", LEGACY)
def test_legacy_contact_sets_take_their_branches_and_reach_every_category(kind, element, rule, oracle_lib, blob, small_mocap):
    """knee_contacts 0 and 1: every designed state takes its branches on the oracle (under rule 1 including which of a leg's foot and
    knee wheel is deeper, by at least DELTA_C), and the batch reaches the lane mappings 4-8 spheres allow and, per env, the
    categories of solver_cases.LEGACY_FEATURES: foot deeper, wheel deeper, wheel alone, a leg-order index other than the sphere-order
    one, a knee wheel within the breaking distance of a wall or box that neither engine collides, feet on walls and boxes."""
    states, decs = designed_batch(kind, oracle_lib, blob, small_mocap, element, rule)
    reached = sc.warp_cases([d["nc"] for d in decs], [d["nl"] for d in decs])[1]
    assert {"split16", "borrow", "borrow_empty", "empty"} <= reached, reached
    got = {}
    for i, d in enumerate(decs):
        assert d["nc"] <= 4 and (rule == 1 or d["ignored"] == 0)
        for f in sc.features(d):
            got.setdefault(f, []).append(i)
    want = set(sc.LEGACY_FEATURES[rule]) - (set() if kind != "pmc" else {"ignored", "off_ground"})
    assert want <= set(got), want - set(got)
    margin_r = min(d["margin_r"] for d in decs)
    worst = oracle_one_by_one(oracle_lib, blob, small_mocap, kind, element, states, decs, knee_contacts=rule)
    print("%s rule %d: %d envs, mapping cases %s; categories (envs): %s; smallest foot-vs-wheel margin %.1e, smallest oracle margin %.1e" % (
        kind, rule, len(states), sorted(reached), {f: len(v) for f, v in sorted(got.items())}, margin_r, worst))


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


# ---------------------------------------------------------------------------------------------------------------- pushes and clamps
DYN_KINDS = [("epmc", 0), ("sepmc", 1), ("corridor", 1)]
DYN_CASES = ("push_in", "push_redraw", "push_after", "pd_clamp", "vel_clamp", "vel_impulse")
PUSH_MIN = 10.0           # N: the least push the batches keep


def _pd_clamps(rng, st, kp, kd, max_tau):
    """PD target and torque clamps on an airborne state (float32 values changed in place, actions returned):
      - the thighs of legs 0 / 1 at q = -2.85 +- 0.05 (clear of both stops) with q + a below -3: the target clamp sets the target to
        -3, and the torque kp (-3 - q) - kd qd (qd within +-1 rad/s) stays inside +-max_tau -- a target clamp at +-pi would saturate it;
      - the knees of legs 2 / 3 within 0.03..0.06 rad of their upper stop with q + a above +3, and qd (about 15..25 rad/s) such that
        the torque kp (3 - q) - kd qd is 2..5 Nm inside +max_tau;
      - every hip torque past +max_tau (legs 0, 2) or -max_tau (legs 1, 3), with joint velocities of 5..15 rad/s against it, so that
        the joint damping that follows the clamp is not 0."""
    a = np.clip(0.3 * rng.standard_normal(12), -1, 1)
    q, qd = st[13:25], st[25:37]
    for k in range(2):
        j = 3 * k + 1
        q[j] = -2.85 + rng.uniform(-0.05, 0.05); qd[j] = rng.uniform(-1, 1)
        a[j] = -3.0 - q[j] - rng.uniform(0.3, 1.0)
    for k in (2, 3):
        j = 3 * k + 2
        q[j] = sc.UPPER[j] - rng.uniform(0.03, 0.06)
        qd[j] = (kp * (3.0 - float(np.float32(q[j]))) - max_tau + rng.uniform(2.0, 5.0)) / kd
        a[j] = 3.0 - q[j] + rng.uniform(0.3, 1.0)
    for k in range(4):
        s = 1.0 if k % 2 == 0 else -1.0
        qd[3 * k] = -s * rng.uniform(5.0, 15.0)
        a[3 * k] = s * (max_tau + 2.0 + kd * abs(qd[3 * k])) / kp + s * rng.uniform(0.0, 0.3)
    return a


def pd_categories(st, a, kp, kd, max_tau):
    """per joint: '+target' / '-target' (q + a beyond +-3 by 0.05, the torque from the clamped target inside +-max_tau by 0.5 Nm),
    '+tau' / '-tau' (the PD torque beyond +-max_tau by 1 Nm)"""
    q, qd = st[13:25].astype(np.float64), st[25:37].astype(np.float64)
    tg = np.clip(q + a, -3, 3)
    tau = kp * (tg - q) - kd * qd
    cat = np.full(12, "", object)
    inside = np.abs(tau) < max_tau - 0.5
    cat[(q + a > 3.05) & inside] = "+target"; cat[(q + a < -3.05) & inside] = "-target"
    cat[tau > max_tau + 1] = "+tau"; cat[tau < -max_tau - 1] = "-tau"
    return cat


VEL = np.r_[7:13, 25:37]    # the base (linear, angular) and joint velocities of a state row: each clamped to +-max_coord_vel


def crossings(before, after, vmax):
    """per env: velocity entries that start inside the bound by 1e-4 and that the sub-step carries beyond it by 1e-4 (after: the
    oracle's state with max_coord_vel at 1e9, no rows), and entries that start beyond it"""
    v0, v1 = np.abs(before[:, VEL].astype(np.float64)), np.abs(after[:, VEL])
    return ((v0 < vmax - 1e-4) & (v1 > vmax + 1e-4)).sum(1), (v0 > vmax).sum(1)


def dynamics_batch(kind, oracle_lib, blob, mocap, element):
    """Designed pairs of envs (SEPMC: the two robots of a pair), one case of DYN_CASES per pair, in turn: a push inside its window, on
    the window's first sub-step after an interval redraw, on the first sub-step after the window (airborne robots and robots on the
    ground alone, decisions as in the solver pin); the PD target and torque clamps (_pd_clamps); velocities within 3 m/s of
    +-max_coord_vel, some beyond it and some that the sub-step carries across it (airborne, see designed_dynamics); a robot falling at
    30..60 m/s onto the ground, whose contact impulse drives joint velocities into the bound.  Every state is checked against the
    statics of its own env (corridor: its own corridor, the robot on the corridor's centre line 8 m before its start).
    Returns (states, decisions, actions, case per env, the batch handle's llq_config); designed_dynamics adds the F_AUX schedule."""
    rng = np.random.default_rng(SEED + 50 + {"epmc": 0, "sepmc": 1, "corridor": 2}[kind])
    npair = 4 * len(DYN_CASES)
    eng = make(oracle_lib, kind, 2 * npair, blob, mocap, element)
    cfg = eng.cfg
    S = sc.Statics(walls=kind == "sepmc")
    statics_of = corridor_statics(eng, element)[2] if kind == "corridor" else (lambda i: S)
    eng.close()
    states, decs, acts, cases = [], [], [], []
    for p in range(npair):
        case = DYN_CASES[p % len(DYN_CASES)]
        for r in range(2):
            i = len(states)
            partner = kind == "sepmc" and r == 1 and case.startswith("push")      # the partner of a pushed SEPMC robot
            name = "light" if case == "vel_impulse" or (case.startswith("push") and r == 1 and not partner) else "air"
            for _ in range(200):
                st, d0 = sc.robot(rng, S, name)
                st = st.copy(); a = np.clip(0.3 * rng.standard_normal(12), -1, 1)
                if partner:
                    a = np.zeros(12)
                elif case == "pd_clamp":
                    a = _pd_clamps(rng, st, cfg.kp, cfg.kd, cfg.max_tau)
                    cat = pd_categories(st, a.astype(np.float32), cfg.kp, cfg.kd, cfg.max_tau)
                    if not ({"+target", "-target", "+tau", "-tau"} <= set(cat)):
                        continue
                elif case == "vel_clamp":
                    pick = rng.random(18) < 0.5
                    v = np.sign(rng.standard_normal(18)) * (cfg.max_coord_vel + rng.uniform(0.5, 3.0, 18))
                    st[VEL[pick]] = v[pick]
                elif case == "vel_impulse":
                    st[9] = -rng.uniform(30.0, 60.0)
                if kind == "corridor":
                    b = statics_of(i).boxes
                    st[0] -= 8.0; st[1] = 0.5 * (b[0, 1] + b[1, 1]) + rng.uniform(-0.05, 0.05)
                d = sc.decisions(st, statics_of(i))
                if sc.clear(d) and (d["nc"], d["nl"], d["n_off_ground"]) == (d0["nc"], d0["nl"], 0):
                    break
            else:
                raise RuntimeError("no %s state for env %d (%s)" % (case, i, kind))
            states.append(st); decs.append(d); acts.append(a); cases.append(case)
    return np.stack(states).astype(np.float32), decs, np.stack(acts).astype(np.float32), cases, cfg


def push_aux(eng, cases, rng_seed):
    """F_AUX of a fresh handle with the push schedule of each env's case (push count, the force of an EPMC push inside its window,
    the draw index); every other case starts far before its push window"""
    aux = eng.get(capi.F_AUX).copy()
    rng = np.random.default_rng(rng_seed)
    for i, c in enumerate(cases):
        aux[i, capi.AUX_PUSH_COUNT] = {"push_in": 5 + (i // 2) % 7, "push_redraw": PUSH_INTERVAL - 1, "push_after": PUSH_DURATION - 1}.get(c, -1000)
        h, th, v = rng.uniform(PUSH_MIN, 50.0), rng.uniform(-np.pi, np.pi), rng.uniform(0.0, 10.0)
        aux[i, capi.AUX_PUSH_F:capi.AUX_PUSH_F + 3] = (h * np.cos(th), h * np.sin(th), v)
        aux[i, capi.AUX_PUSH_DRAWS] = 1 + 2 * (i // 2)
    return aux


PUSH_INTERVAL, PUSH_DURATION = EPMC_CFG["push_interval_steps"], EPMC_CFG["push_duration_steps"]


def dyn_run(oracle_lib, blob, mocap, kind, element, states, aux, acts, warm=None, **over):
    """one oracle sub-step of the dynamics batch with pushes on; returns (state after, F_AUX after, warm start after)"""
    n = len(states)
    e = make(oracle_lib, kind, n, blob, mocap, element, **dict(dict(push_enabled=1), **over))
    e.set(capi.F_STATE, states); e.set(capi.F_WARMSTART, np.zeros((n, 32), np.float32) if warm is None else warm); e.set(capi.F_AUX, aux)
    e.step(acts)
    out = (e.get(capi.F_STATE).astype(np.float64), e.get(capi.F_AUX).copy(), e.get(capi.F_WARMSTART).copy())
    e.close()
    return out


def designed_dynamics(kind, oracle_lib, blob, mocap, element):
    """dynamics_batch with its F_AUX: the draw index of every drawn push moved on until each force drawn is at least PUSH_MIN; in
    the vel_clamp envs the four velocity entries inside the bound that change most in the sub-step are put half their change
    (v' - v, measured on the oracle with max_coord_vel at 1e9) inside it, so that v + a dt crosses it, a few times over as a depends
    on v.  Returns (states, decisions, F_AUX, actions, case per env, llq_config)."""
    states, decs, acts, cases, cfg = dynamics_batch(kind, oracle_lib, blob, mocap, element)
    n = len(states)
    e = make(oracle_lib, kind, n, blob, mocap, element, push_enabled=1)
    aux = push_aux(e, cases, SEED)
    e.close()
    vmax = cfg.max_coord_vel
    vc = np.flatnonzero(np.array(cases) == "vel_clamp")
    for _ in range(6):
        after = dyn_run(oracle_lib, blob, mocap, kind, element, states, aux, acts, max_coord_vel=1e9)[0]
        if (crossings(states[vc], after[vc], vmax)[0] > 0).all():
            break
        for i in vc:
            v0 = states[i, VEL].astype(np.float64)
            dv = after[i, VEL] - v0
            cand = [j for j in np.argsort(-np.abs(dv)) if abs(v0[j]) <= vmax and abs(dv[j]) > 1e-2][:4]
            for j in cand:
                states[i, VEL[j]] = np.sign(dv[j]) * (vmax - 0.5 * abs(dv[j]))
    else:
        raise RuntimeError("no velocity the sub-step carries across the bound")
    pushed = np.array([c.startswith("push") for c in cases])
    for _ in range(50):
        after = dyn_run(oracle_lib, blob, mocap, kind, element, states, aux, acts)[1]
        f = np.linalg.norm(after[:, capi.AUX_PUSH_F:capi.AUX_PUSH_F + 3], axis=1)
        weak = pushed & (f < PUSH_MIN)
        if kind == "sepmc":
            weak = np.repeat(weak.reshape(-1, 2).any(1), 2)
        if not weak.any():
            return states, decs, aux, acts, cases, cfg
        aux[weak, capi.AUX_PUSH_DRAWS] += 2 * n
    raise RuntimeError("no draw index gives pushes of PUSH_MIN")


DYN_BAR = 2e-5            # TOL1 at solver_iters 1 / 10: the visibility checks ask for 100x this
STATE_BLOCKS = {"pose": np.r_[0:7, 13:25], "base velocity": np.r_[7:13], "joint velocity": np.r_[25:37]}


def blockwise(a, b):
    """blockrel per state block (pose, base velocity, joint velocity): a 100 m/s velocity does not scale the pose comparison"""
    from test_parity_gpu import blockrel
    return {k: blockrel(a[:, ix], b[:, ix]) for k, ix in STATE_BLOCKS.items()}


@pytest.mark.parametrize("kind,element", DYN_KINDS)
def test_pushes_and_clamps_are_designed_and_visible(kind, element, oracle_lib, blob, small_mocap):
    """Every env of the dynamics batch takes its designed branches on the oracle (as in the solver pin), reaches its category (the PD
    clamps per joint; in every vel_clamp env an entry the sub-step carries across the bound and one beyond it) and is visible: the
    same step with the push off, or with max_tau / max_coord_vel at 1e9, moves the post-step state by at least 100x the GPU bar in
    some state block (a push after its window: not at all, and the same env one sub-step earlier in the window: by 100x)."""
    states, decs, aux, acts, cases, cfg = designed_dynamics(kind, oracle_lib, blob, small_mocap, element)
    cases = np.array(cases)
    # every state takes its designed branches on the oracle (a pair of copies for SEPMC, the env's own corridor)
    worst = oracle_one_by_one(oracle_lib, blob, small_mocap, kind, element, states, decs)
    assert all(d["n_off_ground"] == 0 for d in decs)
    for i in np.flatnonzero(cases == "pd_clamp"):
        assert {"+target", "-target", "+tau", "-tau"} <= set(pd_categories(states[i], acts[i], cfg.kp, cfg.kd, cfg.max_tau)), i
    ref, aux_after, _ = dyn_run(oracle_lib, blob, small_mocap, kind, element, states, aux, acts)
    def moved(other):
        return np.max(np.stack(list(blockwise(other, ref).values())), axis=0)
    off = dyn_run(oracle_lib, blob, small_mocap, kind, element, states, aux, acts, push_enabled=0)[0]
    inwin = aux.copy(); inwin[:, capi.AUX_PUSH_COUNT] = np.where(cases == "push_after", PUSH_DURATION - 2, aux[:, capi.AUX_PUSH_COUNT])
    earlier = dyn_run(oracle_lib, blob, small_mocap, kind, element, states, inwin, acts)[0]
    no_tau = dyn_run(oracle_lib, blob, small_mocap, kind, element, states, aux, acts, max_tau=1e9)[0]
    no_vel = dyn_run(oracle_lib, blob, small_mocap, kind, element, states, aux, acts, max_coord_vel=1e9)[0]
    vc = cases == "vel_clamp"
    cross, beyond = crossings(states[vc], no_vel[vc], cfg.max_coord_vel)
    assert (cross > 0).all() and (beyond > 0).all(), (cross, beyond)
    f = np.linalg.norm(aux_after[:, capi.AUX_PUSH_F:capi.AUX_PUSH_F + 3], axis=1)
    pushed = np.char.startswith(cases.astype(str), "push")
    assert np.all(f[pushed] >= PUSH_MIN), f[pushed]
    if kind == "sepmc":
        assert np.all(aux_after[0::2, capi.AUX_PUSH_DRAWS] == aux_after[1::2, capi.AUX_PUSH_DRAWS])
    vis = {}
    for c, m in (("push_in", moved(off)), ("push_redraw", moved(off)), ("push_after", moved(earlier)),
                 ("pd_clamp", moved(no_tau)), ("vel_clamp", moved(no_vel)), ("vel_impulse", moved(no_vel))):
        sel = cases == c
        vis[c] = float(m[sel].min())
        assert np.all(m[sel] >= 100 * DYN_BAR), (c, np.flatnonzero(sel & (m < 100 * DYN_BAR)), m[sel])
    assert np.array_equal(moved(off)[cases == "push_after"], np.zeros((cases == "push_after").sum()))
    print("%s: %d envs, smallest oracle decision margin %.1e; velocity entries carried across / starting beyond the bound per "
          "vel_clamp env >= %d / %d; smallest visibility per case (block-relative change): %s" % (
              kind, len(cases), worst, cross.min(), beyond.min(), ", ".join("%s %.1e" % kv for kv in vis.items())))
