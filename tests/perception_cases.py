"""Designed poses for the perception rays of the EPMC and SEPMC observations (host only, fp64 numpy).

The caster states the 778 rays of an observation row (obs 135-912) the way the oracle does (oracle/llq_oracle.cpp
epmc_drill_terrain / epmc_drill / sepmc_write_obs, PGE:374-447, CTG:598-638):
  percept_2d     25 x 13 rays straight down from z = 10 to z = -10 over the base-frame grid; value = hit z, 0 on a miss
  percept_1d     128 horizontal rays of 20 m from the base position, starting at the base yaw; a miss reports |pos|
  percept_front  25 x 13 rays of 3 m along body +x from body (0, y, z); a miss reports 3
against the ground slab (-100..100 x -100..100 x -10..0), the env's corridor boxes (EPMC elements 1-3, walls first) or the
SEPMC arena (four 1 cm walls, the 0.1 x 0.1 x 0.5 flag).  The closest hit wins, ties to the earlier box; a ray whose origin lies
strictly inside a box does not hit that box (Bullet's convex cast).  It also states the rest of the row: the EPMC target block
(obs 913-915) and the SEPMC vectors (obs 913-964) with the opponent's visibility.

A ray is decisive when its branch does not change with every box grown and shrunk by DELTA and the segment lengthened and shortened
by DELTA: hit or miss, the first box hit and its axis of entry, for every box whether the origin is inside it, and for a down ray
the set of footprints it lands in.  The branch is the box id, not the hit point: where two boxes share the hit plane (a hurdle's
side flush with a corridor wall) the ray is not decisive and its pose is not used.  DELTA = 1e-4 m is 25x the fp32 resolution of
a position at 50 m, the far end of a corridor.  The SEPMC visibility segments (root to root, head to the opponent's feet, wheels
and handles) must also be decisive with the flag grown and shrunk by DELTA_VIS = 1 cm: the flag blocks or clears each of them by
at least 1 cm, so that the engines' oppo_visible flags can be compared exactly.

The builder designs one base pose per env (joints at solver_cases.NOMINAL, zero velocities) in a named category and keeps it only
when every ray is decisive and the pose reaches what its category is named for (reaches(): the geometry a kernel shortcut depends
on, e.g. a down ray on a box that a 1.30 m window would drop, a flag-hitting line between 0.0700 m and the cull radius).
"""
import numpy as np

import solver_cases as sc
from helpers import link_kinematics, quat_to_matrix
from lifelike_agility_and_play_b200.model.compile_model import H_NPROXIES, H_OFF_PROXIES, PROXY, load_model_blob

DELTA = 1e-4
DELTA_VIS = 1e-2
S_EPS = 1e-5                       # m: origin / end moves for the sensitivity term of the bars
SLAB = np.array([[-100.0, -100.0, -10.0, 100.0, 100.0, 0.0]])
WALL_IN = 2.495
GX = np.array([-1.2 + a * (2.4 / 24.0) for a in range(24)] + [1.2])
GY = np.array([-0.6 + b * (1.2 / 12.0) for b in range(12)] + [0.6])
FY = np.array([-0.25 + a * (0.5 / 24.0) for a in range(24)] + [0.25])
FZ = np.array([-0.3 + b * (0.4 / 12.0) for b in range(12)] + [0.1])
GRID_REACH = float(np.hypot(1.2, 0.6))                 # 1.342 m: a grid corner's distance from the base
FRONT_REACH = float(np.sqrt(9.0 + 0.25 ** 2 + 0.3 ** 2))   # 3.025 m: a front ray's end from the base
N_DOWN, N_1D, N_FRONT = 325, 128, 325


def _proxies():
    b = load_model_blob()
    o, n = int(b[H_OFF_PROXIES]), int(b[H_NPROXIES])
    return np.asarray(b[o:o + n * PROXY], np.float64).reshape(n, PROXY)[:, :6]


PROXIES = _proxies()                                   # link, centre (link frame), radius, kind (0 foot 1 wheel 2 hip 3 corner 4 handle)
HEAD = int(np.flatnonzero(PROXIES[:, 5] == 4)[0])      # the front handle
TARGETS = np.flatnonzero(np.isin(PROXIES[:, 5], (0, 1, 4)))


# ---------------------------------------------------------------------------------------------------------------- boxes
def corridor_boxes(b):
    """[lo xyz, hi xyz] rows of the ground slab and an env's boxes (rows centre, half extents as F_BOXES holds them)"""
    b = np.asarray(b, np.float64).reshape(-1, 6)
    return np.concatenate([SLAB, np.concatenate([b[:, :3] - b[:, 3:], b[:, :3] + b[:, 3:]], 1)])


def arena_boxes(fx, fy):
    return np.array([SLAB[0], [-2.5, 2.495, 0, 2.5, 2.505, 2], [-2.5, -2.505, 0, 2.5, -2.495, 2], [2.495, -2.5, 0, 2.505, 2.5, 2],
                     [-2.505, -2.5, 0, -2.495, 2.5, 2], [fx - 0.05, fy - 0.05, 0, fx + 0.05, fy + 0.05, 0.5]], np.float64)


# ---------------------------------------------------------------------------------------------------------------- caster
def cast(o, e, boxes, grow=0.0):
    """Closest hit of the segments o -> e (R, 3) against boxes (B, 6) grown by `grow`.  Returns (fraction or -1, box, axis of entry,
    origin inside (R, B)); box and axis are -1 on a miss."""
    g = np.broadcast_to(np.asarray(grow, np.float64), (len(boxes),))[None, :, None]
    lo, hi = boxes[None, :, :3] - g, boxes[None, :, 3:] + g
    O, D = o[:, None, :], (e - o)[:, None, :]
    inside = np.all((O > lo) & (O < hi), axis=2)
    zero = D == 0.0
    with np.errstate(divide="ignore", invalid="ignore"):
        ta, tb = (lo - O) / D, (hi - O) / D
    tmin = np.where(zero, -np.inf, np.minimum(ta, tb))
    tmax = np.where(zero, np.inf, np.maximum(ta, tb))
    off = np.any(zero & ((O < lo) | (O > hi)), axis=2)
    t0, ax = tmin.max(2), tmin.argmax(2)
    t1 = np.minimum(1.0, tmax.min(2))
    hit = ~inside & ~off & (t0 > 0.0) & (t0 <= t1)
    t = np.where(hit, t0, np.inf)
    j = t.argmin(1)
    r = np.arange(len(o))
    h = np.isfinite(t[r, j])
    return np.where(h, t[r, j], -1.0), np.where(h, j, -1), np.where(h, ax[r, j], -1), inside


def pose_rays(pos, R):
    """(origins, ends) of the 778 rays of a base pose, in observation order"""
    pos = np.asarray(pos, np.float64)
    g = np.stack(np.meshgrid(GX, GY, indexing="ij"), -1).reshape(-1, 2)
    t = g[:, :1] * R[:, 0] + g[:, 1:] * R[:, 1] + pos
    down_o = np.stack([t[:, 0], t[:, 1], np.full(N_DOWN, 10.0)], 1)
    down_e = np.stack([t[:, 0], t[:, 1], np.full(N_DOWN, -10.0)], 1)
    yaw = np.arctan2(R[1, 0], R[0, 0])
    ang = yaw + 2.0 * np.pi * np.arange(N_1D) / 128.0
    h_o = np.tile(pos, (N_1D, 1))
    h_e = pos + 20.0 * np.stack([np.cos(ang), np.sin(ang), np.zeros(N_1D)], 1)
    f = np.stack(np.meshgrid(FY, FZ, indexing="ij"), -1).reshape(-1, 2)
    f_o = f[:, :1] * R[:, 1] + f[:, 1:] * R[:, 2] + pos
    f_e = f_o + 3.0 * R[:, 0]
    return np.concatenate([down_o, h_o, f_o]), np.concatenate([down_e, h_e, f_e])


def ray_values(o, e, boxes, pos):
    """observation values of the 778 rays (o, e from pose_rays) and the cast"""
    f, j, ax, inside = cast(o, e, boxes)
    L = np.linalg.norm(e - o, axis=1)
    v = np.where(f < 0, L, f * L)
    v[:N_DOWN] = np.where(f[:N_DOWN] < 0, 0.0, 10.0 - 20.0 * f[:N_DOWN])
    v[N_DOWN:N_DOWN + N_1D] = np.where(f[N_DOWN:N_DOWN + N_1D] < 0, np.linalg.norm(pos), v[N_DOWN:N_DOWN + N_1D])
    return v, (f, j, ax, inside)


def sensitivity(o, e, boxes, pos):
    """S per ray: the largest change of the value when the ray's origin and / or end move by S_EPS along an axis"""
    v0 = ray_values(o, e, boxes, pos)[0]
    S = np.zeros_like(v0)
    for ax in range(3):
        for s in (-S_EPS, S_EPS):
            u = np.zeros(3); u[ax] = s
            for mo, me in ((1, 1), (1, 0), (0, 1)):
                S = np.maximum(S, np.abs(ray_values(o + mo * u, e + me * u, boxes, pos + mo * u)[0] - v0))
    return S


def _branch(o, e, boxes, grow, down):
    f, j, ax, inside = cast(o, e, boxes, grow)
    fp = np.zeros_like(inside)
    if down.any():
        g = np.broadcast_to(np.asarray(grow, np.float64), (len(boxes),))[None, :, None]
        lo, hi = boxes[None, :, :2] - g, boxes[None, :, 3:5] + g
        fp = np.all((o[:, None, :2] >= lo) & (o[:, None, :2] <= hi), axis=2) & down[:, None]
    return f >= 0, j, ax, inside, fp


def decisive(o, e, boxes, delta=DELTA, down=None):
    """per segment: is its branch the same with every box grown / shrunk by delta (a number, or one per box) and the segment
    lengthened / shortened by DELTA"""
    down = np.zeros(len(o), bool) if down is None else down
    d = e - o
    u = d / np.linalg.norm(d, axis=1, keepdims=True)
    ref = _branch(o, e, boxes, 0.0, down)
    ok = np.ones(len(o), bool)
    delta = np.asarray(delta, np.float64)
    for g in (-1, 0, 1):
        for s in (-DELTA, 0.0, DELTA):
            if g == 0 and s == 0.0:
                continue
            b = _branch(o, e + s * u, boxes, g * delta, down)
            for x, y in zip(ref, b):
                ok &= (x == y).reshape(len(o), -1).all(1)
    return ok


def down_mask():
    m = np.zeros(N_DOWN + N_1D + N_FRONT, bool)
    m[:N_DOWN] = True
    return m


def rays_decisive(pos, R, boxes):
    o, e = pose_rays(pos, R)
    return decisive(o, e, boxes, down=down_mask())


# ---------------------------------------------------------------------------------------------------------------- rows
def rot(quat):
    return quat_to_matrix(quat)


def epmc_row(st, boxes, aux):
    """(values of obs 135-915, per-value sensitivity) of an EPMC env at state st, boxes (B, 6 lo/hi), F_AUX row aux"""
    st = np.asarray(st, np.float64)
    pos, R = st[0:3], rot(st[3:7])
    o, e = pose_rays(pos, R)
    v = ray_values(o, e, boxes, pos)[0]
    S = sensitivity(o, e, boxes, pos)
    d = R.T @ np.array([aux[2] - pos[0], aux[3] - pos[1], -pos[2]])
    n = np.hypot(d[0], d[1])
    tail = np.array([d[0] / n, d[1] / n, aux[4]])
    return np.concatenate([v, tail]), np.concatenate([S, np.zeros(3)])


def proxy_points(st):
    ks = link_kinematics(sc.MODEL, np.asarray(st, np.float64))
    return np.array([ks[int(p[0])]["p"] + ks[int(p[0])]["R"] @ p[1:4] for p in PROXIES])


def vis_segments(st_a, st_b):
    """(origins, ends) of the visibility segments of a pair: the root segment (robot 0 -> robot 1), then for each robot its head to
    the opponent's feet, wheels and handles"""
    pa, pb = proxy_points(st_a), proxy_points(st_b)
    o = [np.asarray(st_a[0:3], np.float64)] + [pa[HEAD]] * len(TARGETS) + [pb[HEAD]] * len(TARGETS)
    e = [np.asarray(st_b[0:3], np.float64)] + list(pb[TARGETS]) + list(pa[TARGETS])
    return np.array(o), np.array(e)


def visible(st_a, st_b, boxes):
    """oppo_visible of both robots (CTG:472-493): a clear root segment, or a clear segment from the robot's head to any of the
    opponent's feet, wheels and handles; and the bearing test against visible_angle = pi"""
    o, e = vis_segments(st_a, st_b)
    clear = cast(o, e, boxes)[0] < 0
    nt = len(TARGETS)
    out = []
    for i, (s, t) in enumerate(((st_a, st_b), (st_b, st_a))):
        vis = clear[0] or clear[1 + i * nt:1 + (i + 1) * nt].any()
        R = rot(s[3:7])
        yaw = np.arctan2(R[1, 0], R[0, 0])
        d = np.asarray(t[0:3], np.float64) - np.asarray(s[0:3], np.float64)
        cv = (np.cos(yaw) * d[0] + np.sin(yaw) * d[1]) / np.hypot(d[0], d[1])
        out.append(bool(vis and cv >= np.cos(np.pi)))
    return out


def sepmc_row(st, st_o, aux, aux_o, vis):
    """(values of obs 135-964, sensitivity) of SEPMC robot st with opponent st_o; aux rows give the flag, with_flag and the speed
    command; vis is this robot's oppo_visible"""
    st, st_o = np.asarray(st, np.float64), np.asarray(st_o, np.float64)
    fx, fy = aux[2], aux[3]
    boxes = arena_boxes(fx, fy)
    pos, R = st[0:3], rot(st[3:7])
    o, e = pose_rays(pos, R)
    v = ray_values(o, e, boxes, pos)[0]
    S = sensitivity(o, e, boxes, pos)
    yaw = np.arctan2(R[1, 0], R[0, 0])
    Ro = rot(st_o[3:7])
    yawo = np.arctan2(Ro[1, 0], Ro[0, 0])
    po = st_o[0:3]
    dl, vl, wl = R.T @ (po - pos), R.T @ st_o[7:10], R.T @ st_o[10:13]
    oppo = np.array([1.0 if vis else 0.0, *po, *dl, np.cos(yawo - yaw), np.sin(yawo - yaw), *vl, *wl])
    fl = R.T @ (np.array([fx, fy, 0.25]) - pos)
    flag = np.array([1.0, fx, fy, 0.25, *fl])
    tail = np.concatenate([[*pos, np.cos(yaw), np.sin(yaw)], oppo * (1.0 if vis else 0.0), oppo, flag, flag, [aux[1], aux_o[1], aux[4]]])
    return np.concatenate([v, tail]), np.concatenate([S, np.zeros(len(tail))])


# ---------------------------------------------------------------------------------------------------------------- poses
def state_of(pos, quat):
    st = np.zeros(37)
    st[0:3] = pos
    st[3:7] = np.asarray(quat) / np.linalg.norm(quat)
    st[13:25] = sc.NOMINAL
    return st.astype(np.float32)


def rpy_of(R):
    return np.arctan2(R[2, 1], R[2, 2]), -np.arcsin(np.clip(R[2, 0], -1, 1)), np.arctan2(R[1, 0], R[0, 0])


def align(u, t):
    """a rotation taking unit vector u onto unit vector t"""
    v, c = np.cross(u, t), float(u @ t)
    K = np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])
    return np.eye(3) + K + K @ K / (1.0 + c)


def _orientation(rng, mode):
    if mode == "level":
        return sc.quat_from_rpy(0.0, 0.0, rng.uniform(-np.pi, np.pi))
    if mode == "tilt":
        return sc.quat_from_rpy(rng.uniform(-0.4, 0.4), rng.uniform(-0.4, 0.4), rng.uniform(-np.pi, np.pi))
    if mode == "flip":                                 # upside down: R's third column points down
        return sc.quat_from_rpy(np.pi + rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3), rng.uniform(-np.pi, np.pi))
    if mode == "roll90":
        return sc.quat_from_rpy(rng.choice([-1, 1]) * np.pi / 2 + rng.uniform(-0.1, 0.1), rng.uniform(-0.3, 0.3), rng.uniform(-np.pi, np.pi))
    q = rng.standard_normal(4)                         # uniform over SO(3)
    return q / np.linalg.norm(q)


def _edge_pose(rng, reach_dir, face, axis, u):
    """orientation taking body vector reach_dir onto +axis (world), and the base coordinate along axis that puts its tip u inside face"""
    t = np.zeros(3); t[axis] = 1.0
    phi = rng.uniform(-0.2, 0.2)                       # any turn about the target axis keeps the reach
    K = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    R = (np.eye(3) + np.sin(phi) * K + (1 - np.cos(phi)) * K @ K) @ align(reach_dir / np.linalg.norm(reach_dir), t)
    return sc.quat_from_rpy(*rpy_of(R)), face - (np.linalg.norm(reach_dir) - u)


def corridor_pose(rng, cat, b):
    """(pos, quat) of category cat in a corridor with boxes b (centre, half extents; walls first)"""
    half_gap = b[0, 1] - b[0, 4]
    obs = b[2:]
    j = int(rng.integers(len(obs)))
    ob = obs[j]
    xmax = float((obs[:, 0] + obs[:, 3]).max())
    y = rng.uniform(-0.8, 0.8) * half_gap
    if cat in ("random", "flip", "roll90", "any"):
        pos = [rng.uniform(-0.5, xmax + 0.5), y, rng.uniform(0.05, 0.9)]
        return pos, _orientation(rng, {"random": "tilt"}.get(cat, cat))
    if cat == "in_box":
        return ob[:3] + rng.uniform(-0.8, 0.8, 3) * ob[3:], _orientation(rng, "any")
    if cat == "in_wall":
        w = b[int(rng.integers(2))]
        return [rng.uniform(-0.5, xmax + 0.5), w[1] + rng.uniform(-0.8, 0.8) * w[4], rng.uniform(0.1, 1.9)], _orientation(rng, "any")
    if cat in ("z_in", "z_out"):
        u = rng.uniform(2e-4, 1e-3) * (1 if cat == "z_in" else -1)
        lo, hi = ob[2] - ob[5], ob[2] + ob[5]
        z = hi - u if (lo < 0.01 or rng.random() < 0.5) else lo + u
        return [ob[0] - ob[3] - rng.uniform(0.3, 1.5), y, z], sc.quat_from_rpy(0.0, 0.0, rng.uniform(-0.5, 0.5))
    if cat in ("grid_edge_x", "grid_edge_y"):
        u = rng.uniform(1e-3, 5e-3)
        if cat == "grid_edge_x":                       # the corner (1.2, 0.6) swings out to GRID_REACH along +x
            quat, x = sc.quat_from_rpy(0.0, 0.0, -np.arctan2(0.6, 1.2)), ob[0] - ob[3] - (GRID_REACH - u)
            return [x, rng.uniform(-0.5, 0.5) * half_gap, rng.uniform(0.3, 0.6)], quat
        quat = sc.quat_from_rpy(0.0, 0.0, np.pi / 2 - np.arctan2(0.6, 1.2))     # ... along +y, into the wall on +y
        return [rng.uniform(-0.5, xmax + 0.5), half_gap - (GRID_REACH - u), rng.uniform(0.3, 0.6)], quat
    if cat in ("front_edge_x", "front_edge_y"):
        u = rng.uniform(1e-3, 5e-3)
        tip = np.array([3.0, 0.25, -0.3])              # the end of front ray (a = 24, b = 0)
        if cat == "front_edge_x":
            quat, x = _edge_pose(rng, tip, ob[0] - ob[3], 0, u)
            return [x, rng.uniform(-0.5, 0.5) * half_gap, ob[2] + rng.uniform(-0.5, 0.5) * ob[5]], quat
        # the +y wall's inner face, or in a corridor narrower than the rays the -y wall's outer face, approached from outside
        face = half_gap if 2 * half_gap > 3.2 else b[1, 1] - b[1, 4]
        quat, yy = _edge_pose(rng, tip, face, 1, u)
        return [rng.uniform(-0.5, xmax + 0.5), yy, rng.uniform(0.3, 1.5)], quat
    if cat in ("pad_before", "pad_after"):            # facing -x beyond the last obstacle: the front rays end at its back face
        u = rng.uniform(2e-4, 1e-3) * (1 if cat == "pad_after" else -1)
        last = obs[int(np.argmax(obs[:, 0] + obs[:, 3]))]
        return [last[0] + last[3] + 3.0 - u, y, last[2] + rng.uniform(0.0, 0.2)], sc.quat_from_rpy(0.0, 0.0, np.pi)
    if cat == "high_mask":                             # over boxes 32 and 33 (element 3 with four step sets)
        x = rng.uniform(b[32, 0] - 0.3, b[33, 0] + 0.3)
        return [x, rng.uniform(-0.3, 0.3) * half_gap, rng.uniform(0.3, 0.6)], sc.quat_from_rpy(0.0, 0.0, rng.uniform(-0.3, 0.3))
    if cat == "off_slab":
        return [100.0 - rng.uniform(0.1, 1.0), y, rng.uniform(0.2, 0.8)], _orientation(rng, "tilt")
    raise KeyError(cat)


CORRIDOR_CATS = ("random", "flip", "roll90", "in_box", "in_wall", "z_in", "z_out", "grid_edge_x", "grid_edge_y", "front_edge_x",
                 "front_edge_y", "pad_before", "pad_after", "off_slab")


def corridor_batch(rng, boxes, nbox, element, tries=300):
    """One designed state per env (its own corridor); returns (states float32, categories)"""
    states, cats = [], []
    k = 0
    for i in range(len(boxes)):
        b = np.asarray(boxes[i, :nbox[i]], np.float64)
        if element == 3 and nbox[i] >= 34 and cats.count("high_mask") < 3:
            cat = "high_mask"
        else:
            cat = CORRIDOR_CATS[k % len(CORRIDOR_CATS)]
            k += 1
        bx = corridor_boxes(b)
        for _ in range(tries):
            pos, quat = corridor_pose(rng, cat, b)
            st = state_of(pos, quat)
            if rays_decisive(st[0:3].astype(np.float64), rot(st[3:7]), bx).all() and reaches("corridor", cat, st, bx):
                break
        else:
            raise RuntimeError("no decisive pose for env %d (%s)" % (i, cat))
        states.append(st); cats.append(cat)
    return np.stack(states), cats


FLAT_CATS = ("pitched", "below", "any")


def flat_batch(rng, n, tries=300):
    """EPMC element 0 (the ground slab alone): pitched poses whose front rays cross z = 0, origins below z = 0, any orientation"""
    states, cats = [], []
    bx = SLAB.copy()
    for i in range(n):
        cat = FLAT_CATS[i % len(FLAT_CATS)]
        for _ in range(tries):
            xy = rng.uniform(-3, 3, 2)
            if cat == "pitched":
                pos, quat = [*xy, rng.uniform(0.1, 0.9)], sc.quat_from_rpy(rng.uniform(-0.3, 0.3), rng.uniform(0.1, 0.8), rng.uniform(-np.pi, np.pi))
            elif cat == "below":
                pos, quat = [*xy, rng.uniform(-0.3, -0.01)], _orientation(rng, "tilt")
            else:
                pos, quat = [*xy, rng.uniform(-0.2, 0.9)], _orientation(rng, "any")
            st = state_of(pos, quat)
            if rays_decisive(st[0:3].astype(np.float64), rot(st[3:7]), bx).all() and reaches("flat", cat, st, bx):
                break
        else:
            raise RuntimeError("no decisive flat pose (%s)" % cat)
        states.append(st); cats.append(cat)
    return np.stack(states), cats


# ---------------------------------------------------------------------------------------------------------------- SEPMC pairs
def _flag_clear(states, fx, fy, gap=0.05):
    """no proxy of either robot within gap of the flag box (a touch would move the flag during the step)"""
    box = arena_boxes(fx, fy)[5]
    for st in states:
        p = proxy_points(st)
        q = p - np.clip(p, box[:3], box[3:])
        if (np.linalg.norm(q, axis=1) - PROXIES[:, 4] < gap).any():
            return False
    return True


def sepmc_pose(rng, cat):
    """(pos, quat, flag xy or None) of robot 0 of a pair in category cat"""
    s = rng.choice([-1.0, 1.0])
    ax = int(rng.integers(2))

    def at(c, z):
        p = [rng.uniform(-2.0, 2.0), rng.uniform(-2.0, 2.0), z]
        p[ax] = s * c
        return p
    if cat == "inside":
        return [*rng.uniform(-2.3, 2.3, 2), rng.uniform(0.1, 1.5)], _orientation(rng, "any"), None
    if cat == "band":                                 # 2.49 < |x| < 2.495: the general path while inside the arena
        return at(rng.uniform(2.4902, 2.4948), rng.uniform(0.2, 1.0)), _orientation(rng, "tilt"), None
    if cat == "in_wall":                              # inside a wall, on the arena's side of its centre: the first 1-D ray runs
        c = rng.uniform(2.4952, 2.4996)               # along the wall, tilted outwards just enough to reach the crossing wall
        t = rng.choice([-1.0, 1.0])                   # before it leaves the wall's x (or y) range
        p = [0.0, 0.0, rng.uniform(0.2, 1.8)]
        p[ax], p[1 - ax] = s * c, t * rng.uniform(1.9, 2.3)
        alpha = rng.uniform(0.2, 0.8) * np.arctan((2.5 - c - 2e-4) / (WALL_IN - abs(p[1 - ax])))
        d = np.zeros(2); d[1 - ax] = t * np.cos(alpha); d[ax] = s * np.sin(alpha)
        return p, sc.quat_from_rpy(0.0, 0.0, np.arctan2(d[1], d[0])), None
    if cat == "in_wall_outer":                        # inside a wall, beyond its centre
        return at(rng.uniform(2.5002, 2.5048), rng.uniform(0.2, 1.8)), _orientation(rng, "tilt"), None
    if cat == "outside":
        return at(rng.uniform(2.6, 4.0), rng.uniform(0.2, 1.0)), _orientation(rng, "tilt"), None
    if cat == "below":                                # front-ray origins below the ground
        return [*rng.uniform(-2.0, 2.0, 2), rng.uniform(0.03, 0.2)], _orientation(rng, "level"), None
    if cat == "over_wall":                            # rays that pass over a wall top
        if rng.random() < 0.5:
            return [*rng.uniform(-2.2, 2.2, 2), rng.uniform(2.05, 2.6)], _orientation(rng, "tilt"), None
        p = at(rng.uniform(1.0, 2.2), rng.uniform(1.6, 1.95))
        yaw = (0.0 if ax == 0 else np.pi / 2) + (0.0 if s > 0 else np.pi) + rng.uniform(-0.5, 0.5)
        return p, sc.quat_from_rpy(rng.uniform(-0.2, 0.2), -rng.uniform(0.2, 0.6), yaw), None
    if cat == "flag_corner":                          # a front ray clips a flag corner by 0.25-0.4 mm, inside the cull radius
        pos = np.array([*rng.uniform(-1.5, 1.5, 2), rng.uniform(0.3, 0.4)])
        yaw = np.pi / 4 + rng.integers(4) * np.pi / 2 + rng.uniform(-0.03, 0.03)
        quat = sc.quat_from_rpy(0.0, 0.0, yaw)
        R = rot(quat)
        a, bb = int(rng.integers(25)), int(rng.integers(13))
        o = pos + FY[a] * R[:, 1] + FZ[bb] * R[:, 2]
        d, n = R[:2, 0], np.array([-R[1, 0], R[0, 0]])
        h = 0.05 * (abs(n[0]) + abs(n[1]))
        # the line passes the flag's centre at h - u in (0.0700, 0.0707) m: inside the kernel's cull radius sqrt(0.00501), outside
        # a radius of 0.07 m, with the corner clipped by more than DELTA along either axis
        F = o[:2] + rng.uniform(1.0, 2.5) * d + rng.choice([-1, 1]) * (h - rng.uniform(2.5e-4, 4e-4)) * n
        return pos, quat, F
    if cat == "flag_top":                             # rays that pass over the flag top
        pos = np.array([*rng.uniform(-1.5, 1.5, 2), rng.uniform(0.82, 1.2)])
        quat = _orientation(rng, "level")
        return pos, quat, pos[:2] + rng.uniform(1.0, 2.0) * rot(quat)[:2, 0]
    if cat == "grid_wall":                            # down-ray grid points inside a wall strip
        return at(rng.uniform(1.6, 2.4), rng.uniform(0.3, 0.6)), _orientation(rng, "level"), None
    if cat == "grid_flag":                            # ... and inside the flag footprint
        pos = np.array([*rng.uniform(-1.5, 1.5, 2), rng.uniform(0.6, 0.9)])
        quat = _orientation(rng, "level")
        R = rot(quat)
        return pos, quat, pos[:2] + R[:2, :2] @ np.array([rng.uniform(-1.0, 1.0), rng.uniform(-0.5, 0.5)])
    if cat == "off_slab":                             # grid points beyond the slab's edge
        p = at(100.0 - rng.uniform(0.1, 1.0), rng.uniform(0.2, 0.8))
        return p, _orientation(rng, "tilt"), None
    raise KeyError(cat)


SEPMC_CATS = ("inside", "band", "in_wall", "in_wall_outer", "outside", "below", "over_wall", "flag_corner", "flag_top", "grid_wall", "grid_flag", "off_slab")


def sepmc_batch(rng, n_pairs, tries=400):
    """n_pairs designed pairs: robot 0 in a category, robot 1 anywhere in the arena, the flag away from both robots unless the
    category places it.  Every ray of both robots is decisive and so is every visibility segment (by DELTA_VIS).  Returns
    (states [2 n_pairs, 37] float32, flags [n_pairs, 2], categories, oppo_visible [2 n_pairs])"""
    states, flags, cats, vis = [], [], [], []
    for p in range(n_pairs):
        cat = SEPMC_CATS[p % len(SEPMC_CATS)]
        for _ in range(tries):
            pos, quat, F = sepmc_pose(rng, cat)
            a = state_of(pos, quat)
            b = state_of([*rng.uniform(-2.2, 2.2, 2), rng.uniform(0.25, 0.6)], _orientation(rng, "tilt"))
            if F is None:
                F = rng.uniform(-2.0, 2.0, 2)
            F = np.asarray(F, np.float64)
            if np.abs(F).max() > 2.4 or not _flag_clear((a, b), *F):
                continue
            bx = arena_boxes(*F)
            if not reaches("sepmc", cat, a, bx):
                continue
            if not all(rays_decisive(s[0:3].astype(np.float64), rot(s[3:7]), bx).all() for s in (a, b)):
                continue
            o, e = vis_segments(a, b)
            if not decisive(o, e, bx, np.array([DELTA] * 5 + [DELTA_VIS])).all():
                continue
            break
        else:
            raise RuntimeError("no decisive pair (%s)" % cat)
        states += [a, b]; flags.append(F); cats.append(cat); vis += visible(a, b, bx)
    return np.stack(states), np.array(flags), cats, np.array(vis)


# ---------------------------------------------------------------------------------------------------------------- reach
SEPMC_INSIDE = 2.49                 # |x|, |y| below which the kernel takes ray_arena_inside
FLAG_CULL2 = 0.00501                # the kernel's flag cull radius squared


def _sepmc_inside_path(o):
    """rays (origins o in pose_rays order) that the kernel casts with ray_arena_inside: 1-D rays from a base with |x|, |y| < 2.49,
    front rays from such an origin above z = 0"""
    m = np.zeros(len(o), bool)
    a = (np.abs(o[:, 0]) < SEPMC_INSIDE) & (np.abs(o[:, 1]) < SEPMC_INSIDE)
    m[N_DOWN:N_DOWN + N_1D] = a[N_DOWN:N_DOWN + N_1D]
    m[N_DOWN + N_1D:] = a[N_DOWN + N_1D:] & (o[N_DOWN + N_1D:, 2] > 0)
    return m


def arena_inside(o, e, boxes):
    """ray_arena_inside's answer in fp64: the ground top when the ray goes down from above it, the first wall plane crossed (only
    its z range checked), the flag unless culled.  Valid only for origins inside the arena; used to show where it is not."""
    d = e - o
    best = np.full(len(o), -1.0)
    g = (d[:, 2] < 0) & (o[:, 2] > 0)
    with np.errstate(divide="ignore", invalid="ignore"):
        tg = -o[:, 2] / d[:, 2]
        tw = np.minimum(np.where(d[:, 0] != 0, (np.where(d[:, 0] > 0, WALL_IN, -WALL_IN) - o[:, 0]) / d[:, 0], 2.0),
                        np.where(d[:, 1] != 0, (np.where(d[:, 1] > 0, WALL_IN, -WALL_IN) - o[:, 1]) / d[:, 1], 2.0))
    best = np.where(g & (tg <= 1), tg, best)
    z = o[:, 2] + tw * d[:, 2]
    best = np.where((tw <= 1) & (z >= 0) & (z <= 2) & ((best < 0) | (tw < best)), tw, best)
    fx, fy = (boxes[5, 0] + boxes[5, 3]) / 2, (boxes[5, 1] + boxes[5, 4]) / 2
    cr = d[:, 0] * (fy - o[:, 1]) - d[:, 1] * (fx - o[:, 0])
    near = ~(cr * cr > FLAG_CULL2 * (d[:, 0] ** 2 + d[:, 1] ** 2))
    ff = cast(o, e, boxes[5:6])[0]
    return np.where(near & (ff >= 0) & ((best < 0) | (ff < best)), ff, best)


def reaches(kind, cat, st, boxes):
    """Does a designed pose reach what its category is named for?  kind 'corridor' (boxes: slab + the env's boxes, lo / hi rows),
    'flat' or 'sepmc' (robot 0 of the pair; boxes = arena_boxes).  Each check states the geometry a kernel shortcut depends on."""
    st = np.asarray(st, np.float64)
    pos, R = st[0:3], rot(st[3:7])
    o, e = pose_rays(pos, R)
    f, j, ax, inside = cast(o, e, boxes)
    dn, h1, fr = slice(0, N_DOWN), slice(N_DOWN, N_DOWN + N_1D), slice(N_DOWN + N_1D, None)
    if kind == "flat":
        if cat == "pitched":
            return bool(((o[fr, 2] > 0) & (e[fr, 2] < 0)).any())        # front rays cross the ground plane
        if cat == "below":
            return bool(pos[2] < 0 and (o[fr, 2] < 0).any())
        return True
    if kind == "corridor":
        c, hx = (boxes[:, :3] + boxes[:, 3:]) / 2, (boxes[:, 3:] - boxes[:, :3]) / 2

        def beyond(rays, w):           # a ray of `rays` hits a box (not the slab) that a window of w m around the base would drop
            jj = j[rays]
            k = jj[jj > 0]
            return bool(((np.abs(c[k, 0] - pos[0]) > hx[k, 0] + w) | (np.abs(c[k, 1] - pos[1]) > hx[k, 1] + w)).any())
        if cat == "random":
            return R[2, 2] > 0
        if cat == "flip":                                                # upside down
            return R[2, 2] < 0
        if cat == "roll90":                                              # the body's y axis nearly vertical
            return abs(R[2, 1]) > 0.9
        if cat == "in_box":
            return bool(inside[N_DOWN, 3:].any())                        # the base (the 1-D rays' origin) inside an obstacle
        if cat == "in_wall":
            return bool(inside[N_DOWN, 1:3].any())
        if cat in ("z_in", "z_out"):
            lo, hi = boxes[3:, 2], boxes[3:, 5]
            d = np.minimum(np.abs(pos[2] - lo), np.abs(pos[2] - hi))
            tall = boxes.copy(); tall[3:, 2] = -10.0; tall[3:, 5] = 10.0
            crossed = np.unique(cast(o[h1], e[h1], tall)[1]) - 3       # obstacles the 1-D rays reach when z is ignored
            crossed = crossed[crossed >= 0]
            within = (pos[2] > lo) & (pos[2] < hi)
            want = within if cat == "z_in" else ~within
            return bool((want[crossed] & (d[crossed] >= DELTA) & (d[crossed] <= 1e-3)).any())
        if cat.startswith("grid_edge"):
            return beyond(dn, 1.30)
        if cat.startswith("front_edge"):
            return beyond(fr, 3.00)
        if cat == "pad_after":                                           # a front ray hits within 1 mm of its end
            return bool((j[fr] > 0).any() and (f[fr][j[fr] > 0] > 1 - 1e-3 / 3).any())
        if cat == "pad_before":                                          # ... or ends within 1 mm before a box face
            u = (e - o) / np.linalg.norm(e - o, axis=1, keepdims=True)
            f2, j2 = cast(o[fr], e[fr] + 1e-3 * u[fr], boxes)[:2]
            return bool(((j[fr] != j2) & (j2 > 0)).any())
        if cat == "high_mask":                                           # down rays land on boxes 32 and 33 (the mask's high word)
            return bool((j[dn] - 1 >= 32).any())
        if cat == "off_slab":
            return bool((np.abs(o[dn, :2]) > 100).any())
        raise KeyError(cat)
    a = np.abs(pos[:2]).max()
    ins = _sepmc_inside_path(o)
    if cat == "inside":
        return a < SEPMC_INSIDE
    if cat == "band":
        return SEPMC_INSIDE < a < WALL_IN
    if cat == "in_wall":                      # inside a wall, on the arena's side of its centre, with a 1-D ray that the inside
        f_in = arena_inside(o[h1], e[h1], boxes)     # fast path would get wrong (its origin is not inside the arena)
        f_gen = f[h1]
        return bool(WALL_IN < a < 2.5 and ((np.sign(f_in) != np.sign(f_gen)) | (np.abs(f_in - f_gen) > 1e-6)).any())
    if cat == "in_wall_outer":
        return 2.5 < a < 2.505
    if cat == "outside":
        return 2.505 < a < 99
    if cat == "below":
        return bool((o[fr, 2] < 0).any())
    if cat == "over_wall":                   # an inside-path ray, not stopped by the flag, crosses the first wall plane above z = 2
        d = e - o
        with np.errstate(divide="ignore", invalid="ignore"):
            tw = np.minimum(np.where(d[:, 0] != 0, (np.sign(d[:, 0]) * WALL_IN - o[:, 0]) / d[:, 0], np.inf),
                            np.where(d[:, 1] != 0, (np.sign(d[:, 1]) * WALL_IN - o[:, 1]) / d[:, 1], np.inf))
        z = o[:, 2] + tw * d[:, 2]
        return bool((ins & (tw > 0) & (tw <= 1) & (z > 2 + DELTA) & (j != 5)).any())
    fx, fy = (boxes[5, 0] + boxes[5, 3]) / 2, (boxes[5, 1] + boxes[5, 4]) / 2
    if cat == "flag_corner":                                             # an inside-path ray hits the flag with its line at
        d = e - o                                                        # (0.0700, sqrt(0.00501)) m from the flag's centre
        cr = d[:, 0] * (fy - o[:, 1]) - d[:, 1] * (fx - o[:, 0])
        r2 = cr * cr / np.maximum(d[:, 0] ** 2 + d[:, 1] ** 2, 1e-30)   # inside-path rays are never vertical
        return bool((ins & (j == 5) & (r2 > 0.0049) & (r2 <= FLAG_CULL2)).any())
    if cat == "flag_top":                                                # a ray crosses the flag's footprint above its top
        tall = boxes.copy(); tall[5, 5] = 10.0
        return bool(((cast(o[N_DOWN:], e[N_DOWN:], tall)[1] == 5) & (j[N_DOWN:] != 5)).any())
    if cat == "grid_wall":
        return bool(((j[dn] >= 1) & (j[dn] <= 4)).any())
    if cat == "grid_flag":
        return bool((j[dn] == 5).any())
    if cat == "off_slab":
        return bool((np.abs(o[dn, :2]) > 100).any())
    raise KeyError(cat)
