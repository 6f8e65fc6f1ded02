"""Designed single-sub-step states for the step kernel's constraint solver (host only, fp64 numpy).

With llq_config.substeps = 1 every discrete decision of the step is taken on the pose handed in: contact make / break
(dist < contact_breaking), which static owns a sphere's manifold point, whether a joint limit row exists, and the -0.04 rad
split-impulse threshold of a limit row.  A state whose every such decision sits at least DELTA_C (m) / DELTA_Q (rad) away from its
branch cannot flip in fp32, so the CUDA step and the fp64 oracle solve the same rows and their results can be compared env by env
with no exclusions.

The builder places robots (joint angles past the stops included) on the ground, against the SEPMC arena walls and on / against the
boxes and edge cylinders of an EPMC corridor, keeps the states that clear every branch, and assembles batches whose CTAs of 16 envs
reach the solver's lane mappings (see warp_cases):
  split16     both envs of a warp have <= 16 rows, each on its own half-warp
  borrow      one env has more than 16 rows and takes lanes from its partner, whose rows start right after them
  borrow_empty  an env with 17..31 rows beside a partner without rows (its rows spill into the upper half-warp alone)
  two_pass    the pair has more than 32 rows: each env is solved on all 32 lanes in turn
  empty       neither env of the warp has a row
  exact32     an env with exactly 32 rows (8 contacts, 8 limit rows) paired with an empty one
  contact_cap an env with more than 8 contacts (the rest is dropped and counted in counter [5])
  limit_cap   an env with more than 8 violated joint limits
  shadow      the last CTA is partly filled and env N - 1, whose copies fill the unused slots, is the heaviest robot of that CTA
"""
import numpy as np

from helpers import link_kinematics
from lifelike_agility_and_play_b200.model.compile_model import contact_proxy_spheres, load_model

BREAKING = 0.02 * 0.025          # llq_config.contact_breaking (default)
WALL_IN = 2.495                  # inner faces of the SEPMC arena walls
SPLIT_PEN = -0.04                # split-impulse threshold of a joint-limit row
DELTA_C = 1e-3                   # m: least distance of a contact / owner decision from its branch
DELTA_Q = 5e-3                   # rad: least distance of a joint-limit / split-impulse decision from its branch
DELTA_N = 1e-3                   # least distance of a box / cylinder normal's |n.z| from 1/sqrt(2) (btPlaneSpace1's branch)
MAX_CON = MAX_LIM = 8            # LLQ_MAX_CONTACTS, LLQ_MAX_LIMIT_ROWS
EPB = 16                         # envs per CTA of the step kernel
CASES = ("split16", "borrow", "borrow_empty", "two_pass", "empty", "exact32", "contact_cap", "limit_cap", "shadow")

MODEL = load_model()
_LINKS = MODEL["links"]
_DOF_LINK = {l["dof_index"]: i for i, l in enumerate(_LINKS) if l["joint_type"] == "revolute"}
LOWER = np.array([_LINKS[_DOF_LINK[j]]["lower"] for j in range(12)])
UPPER = np.array([_LINKS[_DOF_LINK[j]]["upper"] for j in range(12)])
NOMINAL = np.array([-0.03, -0.78, 1.69] * 2 + [-0.03, -0.73, 1.57] * 2)


def _sphere_table():
    """(link, centre in the link frame, radius) of the 32 collision spheres, in the order both engines keep: 4 feet, then the proxies"""
    rows = []
    for i, ln in enumerate(_LINKS):
        for c in ln["collisions"]:
            if c["type"] == "sphere" and ln["name"].endswith("4"):
                rows.append((i, np.array(c["xyz"], np.float64), float(c["radius"])))
    rows += [(int(s[0]), np.array(s[1:4], np.float64), float(s[4])) for s in contact_proxy_spheres(MODEL)]
    return rows


SPHERES = _sphere_table()
RADIUS = np.array([s[2] for s in SPHERES])


def sphere_offsets(quat, q):
    """world sphere centres minus the base position, for base orientation quat (xyzw) and joint angles q"""
    st = np.zeros(37); st[3:7] = quat; st[13:25] = q
    ks = link_kinematics(MODEL, st)
    return np.array([ks[l]["p"] + ks[l]["R"] @ c for l, c, _ in SPHERES])


def quat_from_rpy(roll, pitch, yaw):
    cr, sr, cp, sp, cy, sy = np.cos(roll / 2), np.sin(roll / 2), np.cos(pitch / 2), np.sin(pitch / 2), np.cos(yaw / 2), np.sin(yaw / 2)
    return np.array([sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy])


# ---------------------------------------------------------------------------------------------------------------- statics
def _box_dist(cw, b):
    """clearance of sphere centres cw (n, 3) from box b (centre, half extents), the outward normal as the engines compute it, and --
    for a centre inside the box -- how much deeper the second-nearest face lies than the one it leaves through (inf outside)"""
    p = cw - b[:3]
    c = np.clip(p, -b[3:6], b[3:6])
    v = p - c
    ln = np.linalg.norm(v, axis=1)
    inside = ln == 0.0
    n = v / np.where(inside, 1.0, ln)[:, None]
    d = ln.copy()
    face_margin = np.full(len(cw), np.inf)
    if inside.any():                                   # centre inside: leave through the nearest face
        depth = np.concatenate([b[3:6] - p, b[3:6] + p], axis=1)[inside]
        f = np.argmin(depth, axis=1)
        d[inside] = -depth[np.arange(len(f)), f]
        nn = np.zeros((len(f), 3)); nn[np.arange(len(f)), f % 3] = np.where(f < 3, 1.0, -1.0)
        n[inside] = nn
        face_margin[inside] = np.diff(np.sort(depth, axis=1)[:, :2], axis=1)[:, 0]
    return d, n, face_margin


class Statics:
    """The static shapes a robot's spheres collide with: the ground, the SEPMC arena walls, the boxes of an EPMC corridor (walls
    first) with the two auxiliary edge cylinders of every box after the walls (tops of hurdles and cubes, bottoms of bars).
    rule = llq_config.knee_contacts: the spheres are the first 4 (0: feet), 8 (1: feet, knee wheels) or all 32 (2) rows of SPHERES;
    under rules 0 and 1 only the feet meet walls, boxes and cylinders."""

    def __init__(self, walls=False, boxes=None, aux_r=0.0, element=0, rule=2):
        self.walls = walls
        self.boxes = np.zeros((0, 6)) if boxes is None else np.asarray(boxes, np.float64).reshape(-1, 6)
        self.cyl = []
        if aux_r > 0:
            for b in self.boxes[2:]:
                for side in (-1, 1):
                    self.cyl.append((b[0] + side * b[3], b[1], b[2] + (-b[5] if element == 2 else b[5]), b[4], aux_r))
        self.element, self.rule = element, rule
        self.ns = {0: 4, 1: 8, 2: len(SPHERES)}[rule]
        self.radius = RADIUS[:self.ns]
        self.touch = np.arange(self.ns) < (self.ns if rule == 2 else 4)

    def shapes(self, cw):
        """per static: (clearance (n,), normal (n, 3), kind, inside-face margin (n,)) with kind 0 ground / plane, 1 box, 2 cylinder;
        the clearance from walls, boxes and cylinders is given for every sphere, including those the rule keeps from them"""
        R = self.radius
        none = np.full(len(cw), np.inf)
        out = [(cw[:, 2] - R, np.tile([0.0, 0.0, 1.0], (len(cw), 1)), 0, none)]
        if self.walls:
            for n in ((-1, 0, 0), (1, 0, 0), (0, -1, 0), (0, 1, 0)):
                n = np.array(n, np.float64)
                out.append((cw @ n + WALL_IN - R, np.tile(n, (len(cw), 1)), 0, none))
        for b in self.boxes:
            d, n, fm = _box_dist(cw, b)
            out.append((d - R, n, 1, fm))
        for x, y, z, hy, r in self.cyl:
            dx, dz = cw[:, 0] - x, cw[:, 2] - z
            ln = np.hypot(dx, dz)
            beside = np.abs(cw[:, 1] - y) > hy
            d = np.where(beside | (ln == 0), np.inf, ln - r - R)
            n = np.stack([dx, np.zeros_like(dx), dz], 1) / np.where(ln == 0, 1.0, ln)[:, None]
            out.append((d, n, 2, none))
        return out

    def off_ground(self, d):
        """clearances from a wall, box or cylinder as the rule sees them: inf for the spheres it keeps away"""
        return np.where(self.touch, d, np.inf)

    def clearance(self, cw):
        """(dist, second, normal, owner kind, owner index, inside-face margin, clearance from the nearest wall / box / cylinder
        ignoring the rule) per sphere: the owner is the first static with the smallest clearance (index 0 = the ground)"""
        sh = self.shapes(cw)
        D = np.stack([s[0] for s in sh])
        raw = D[1:].min(axis=0) if len(D) > 1 else np.full(len(cw), np.inf)
        D[1:] = np.where(self.touch, D[1:], np.inf)
        o = np.argmin(D, axis=0)
        idx = np.arange(cw.shape[0])
        dist = D[o, idx]
        D2 = D.copy(); D2[o, idx] = np.inf
        second = D2.min(axis=0)
        normal = np.stack([s[1] for s in sh])[o, idx]
        kind = np.array([s[2] for s in sh])[o]
        fm = np.stack([s[3] for s in sh])[o, idx]
        return dist, second, normal, kind, o, fm, raw


# ---------------------------------------------------------------------------------------------------------------- decisions
LEG_CASES = ("foot_deeper", "wheel_deeper", "wheel_alone", "foot_alone")


def decisions(state, statics):
    """Every discrete decision of one sub-step on `state` (fp64 arithmetic on the values as given): per sphere contact / owner /
    normal / the face a centre inside a box leaves through, per joint the limit row and its split-impulse side, and under rule 1 per
    leg which of foot and knee wheel keeps the leg's one contact.  Returns a dict with the counts the engines solve and the margins."""
    st = np.asarray(state, np.float64)
    cw = sphere_offsets(st[3:7], st[13:25])[:statics.ns] + st[0:3]
    dist, second, normal, kind, owner, face_m, raw = statics.clearance(cw)
    contact = dist < BREAKING
    m = np.abs(dist - BREAKING).min()
    close = second < BREAKING + DELTA_C
    if close.any():
        m = min(m, (second - dist)[close].min())
    inside = contact & (kind == 1) & (dist + statics.radius < 0)        # centre inside a box
    if inside.any():
        m = min(m, face_m[inside].min())
    legs, m_r = [None] * 4, np.inf
    if statics.rule == 1:                              # one contact per leg, the deeper of foot and wheel (the foot wins ties)
        for l in range(4):
            f, w = l, 4 + l
            if contact[f] and contact[w]:
                m_r = min(m_r, abs(dist[f] - dist[w]))
                legs[l] = "wheel_deeper" if dist[w] < dist[f] else "foot_deeper"
                contact[f if dist[w] < dist[f] else w] = False
            elif contact[w] or contact[f]:
                legs[l] = "wheel_alone" if contact[w] else "foot_alone"
    kept = np.flatnonzero(contact)
    general = contact & (kind != 0)                    # box / cylinder normals go through btPlaneSpace1's two branches
    nz = np.abs(normal[:, 2])
    m_n = np.abs(nz - np.sqrt(0.5))[general].min() if general.any() else np.inf
    q = st[13:25]
    pen = np.where(q - LOWER <= 0, q - LOWER, np.where(UPPER - q <= 0, UPPER - q, np.inf))
    viol = np.isfinite(pen)
    mq = min(np.abs(q - LOWER).min(), np.abs(UPPER - q).min())
    if viol.any():
        mq = min(mq, np.abs(pen[viol] - SPLIT_PEN).min())
    # a sphere the rule keeps from walls and boxes, within the breaking distance of one and clear of the ground, both by DELTA_C
    ignored = ~statics.touch & (raw < BREAKING - DELTA_C) & (cw[:, 2] - statics.radius >= BREAKING + DELTA_C)
    return dict(nc=int(contact.sum()), nl=int(viol.sum()), contact=contact, n_off_ground=int((contact & (owner != 0)).sum()), pen=pen[viol],
                margin_c=m, margin_q=mq, margin_n=m_n, margin_r=m_r, nz=nz[general], normal=normal[general], kind=kind[general],
                inside=int(inside.sum()), legs=legs, ignored=int(ignored.sum()),
                leg_order=bool(statics.rule == 1 and list(kept) != sorted(kept, key=lambda s: s % 4)))


def clear(dec):
    return dec["margin_c"] >= DELTA_C and dec["margin_q"] >= DELTA_Q and dec["margin_n"] >= DELTA_N and dec["margin_r"] >= DELTA_C


# ---------------------------------------------------------------------------------------------------------------- sampling
def _joint_angles(rng, family, n_viol):
    """12 joint angles: n_viol of them past a stop (by 0.005 .. 0.11 rad, clear of the split-impulse threshold), the rest inside"""
    if family == "stand":
        q = NOMINAL + 0.15 * rng.standard_normal(12)
    elif family == "fold":                             # legs along the trunk, knees folded: the robot lies on its belly
        q = np.tile([0.0, -1.57, 2.4], 4) + np.tile([0.3, 0.15, 0.1], 4) * rng.standard_normal(12)
    else:
        q = rng.uniform(LOWER, UPPER)
    q = np.clip(q, LOWER + DELTA_Q + 1e-3, UPPER - DELTA_Q - 1e-3)
    for j in rng.choice(12, size=n_viol, replace=False):
        pen = -rng.uniform(DELTA_Q + 1e-3, 0.11)
        if abs(pen - SPLIT_PEN) < DELTA_Q + 1e-3:
            pen = SPLIT_PEN - np.sign(pen - SPLIT_PEN + 1e-12) * (DELTA_Q + 2e-3)
        q[j] = LOWER[j] + pen if rng.random() < 0.5 else UPPER[j] - pen
    return q


def _place(rng, off, shape_fn, direction, k, ref, lo=-0.05):
    """Base position with the k-th closest sphere (k = 0: the closest one, clear) at a chosen clearance from one static
    (shape_fn: centres -> clearances): t = 0 puts the centre of the sphere that leads along -direction on the point ref, the robot is
    moved along direction by t in [lo, 0.6].  Every other decision is checked afterwards."""
    target = BREAKING - rng.uniform(DELTA_C + 5e-4, 0.012) if k > 0 else BREAKING + rng.uniform(DELTA_C + 5e-4, 0.05)
    kk = max(k, 1) - 1
    p0 = ref - np.min(off @ direction) * direction
    hi = 0.6

    def f(t):
        return np.sort(shape_fn(off + p0 + t * direction))[kk] - target
    if f(lo) > 0 or f(hi) < 0:
        return None
    for _ in range(40):
        mid = 0.5 * (lo + hi)
        lo, hi = (mid, hi) if f(mid) < 0 else (lo, mid)
    return p0 + hi * direction


def design(rng, statics, family="stand", n_viol=0, k_ground=0, target=None, tilt=0.15):
    """One designed state (float32 values) or None.  target: None (ground only), ('wall', k), ('top', box, k), ('face', box, k),
    ('cyl', index, k), ('under', bar, k), ('under_cyl', index, k); with '_any' appended to the name the k-th closest sphere is
    counted among all spheres, also those the contact rule keeps from walls and boxes."""
    q = _joint_angles(rng, family, n_viol).astype(np.float32).astype(np.float64)
    quat = quat_from_rpy(tilt * rng.standard_normal(), tilt * rng.standard_normal(), rng.uniform(-np.pi, np.pi))
    quat = (quat / np.linalg.norm(quat)).astype(np.float32).astype(np.float64)
    off = sphere_offsets(quat, q)[:statics.ns]
    R, ring = statics.radius, statics.off_ground
    if target is not None and target[0].endswith("_any"):   # place the k-th closest of all spheres, also those the rule keeps away
        target, ring = (target[0][:-4],) + tuple(target[1:]), (lambda d: d)
    ground = lambda c: c[:, 2] - R
    ez = np.array([0.0, 0.0, 1.0])
    p = np.zeros(3)
    if target is not None and target[0] == "top":
        b = statics.boxes[target[1]]
        p = np.array([b[0] + rng.uniform(-0.5, 0.5) * b[3], b[1] + rng.uniform(-0.5, 0.5) * b[4], b[2] + b[5]])   # a point of the top face
        box = lambda c: ring(_box_dist(c, b)[0] - R)
        p = _place(rng, off, box, ez, target[2], p)
    elif target is not None and target[0] in ("under", "under_cyl"):
        # on the ground below a bar, crouched until the k-th closest sphere meets the bar's bottom face (n = -z) or one of its
        # bottom-edge cylinders
        if target[0] == "under":
            b = statics.boxes[target[1]]
            xy = np.array([b[0] + rng.uniform(-0.3, 0.3), b[1] + rng.uniform(-0.5, 0.5) * b[4], 0.0])
            box = lambda c: ring(_box_dist(c, b)[0] - R)
        else:
            x, y, z, hy, r = statics.cyl[target[1]]
            xy = np.array([x + rng.uniform(-0.35, 0.35), y + rng.uniform(-0.5, 0.5) * hy, 0.0])
            box = lambda c: ring(np.where(np.abs(c[:, 1] - y) > hy, np.inf, np.hypot(c[:, 0] - x, c[:, 2] - z) - r - R))
        kb = target[2]
        tb = BREAKING - rng.uniform(DELTA_C + 5e-4, 0.006)
        tg = BREAKING - rng.uniform(DELTA_C + 5e-4, 0.006)
        crouch = np.tile([0.0, -1.0, 2.0], 4)

        def at(s):
            qs = np.clip(q + s * crouch, LOWER + DELTA_Q + 1e-3, UPPER - DELTA_Q - 1e-3).astype(np.float32).astype(np.float64)
            o = sphere_offsets(quat, qs)[:statics.ns]
            lift = tg - np.sort(ground(o + xy))[max(k_ground, 1) - 1]
            return qs, xy + lift * ez, np.sort(box(o + xy + lift * ez))[kb - 1] - tb
        lo_s, hi_s = 0.0, 0.7
        if at(lo_s)[2] > 0 or at(hi_s)[2] < 0:
            return None
        for _ in range(30):
            mid = 0.5 * (lo_s + hi_s)
            lo_s, hi_s = (mid, hi_s) if at(mid)[2] < 0 else (lo_s, mid)
        q, p, _ = at(hi_s)
    else:
        if target is not None and target[0] == "face":
            b = statics.boxes[target[1]]
            p = np.array([b[0] - b[3], b[1] + rng.uniform(-0.6, 0.6) * b[4], 0.0])                 # a point of the front face
        elif target is not None and target[0] == "cyl":
            x, y, z, hy, r = statics.cyl[target[1]]
            p = np.array([x, y + rng.uniform(-0.6, 0.6) * hy, z])
        elif target is not None and target[0] == "wall":
            p = np.array([WALL_IN, rng.uniform(-1.5, 1.5), 0.0])
        else:
            p = np.array([rng.uniform(-1, 1), rng.uniform(-1, 1), 0.0])
        if target is None or target[0] != "cyl":
            p = _place(rng, off, ground, ez, k_ground, p)
        if p is not None and target is not None:
            if target[0] == "wall":
                p = _place(rng, off, lambda c: ring(WALL_IN - c[:, 0] - R), np.array([-1.0, 0.0, 0.0]), target[1], p)
            elif target[0] == "face":
                box = lambda c: ring(_box_dist(c, b)[0] - R)
                p = _place(rng, off, box, np.array([-1.0, 0.0, 0.0]), target[2], p)
            else:
                phi = rng.uniform(0.15, np.pi - 0.15)
                if statics.element == 2:               # a bar's cylinders sit on its bottom edges: approach from below
                    phi = -phi
                d = np.array([np.cos(phi), 0.0, np.sin(phi)])
                cyl = lambda c: ring(np.where(np.abs(c[:, 1] - y) > hy, np.inf, np.hypot(c[:, 0] - x, c[:, 2] - z) - r - R))
                p = _place(rng, off, cyl, d, target[2], p, lo=0.0)
    if p is None:
        return None
    st = np.zeros(37)
    st[0:3] = p; st[3:7] = quat; st[13:25] = q
    st[7:10] = 0.3 * rng.standard_normal(3); st[10:13] = 0.5 * rng.standard_normal(3); st[25:37] = rng.standard_normal(12)
    st = st.astype(np.float32)
    dec = decisions(st, statics)
    return (st, dec) if clear(dec) else None


def sample(rng, statics, want, tries=4000, **kw):
    """a designed state whose (contacts, limit rows) satisfy want(nc, nl)"""
    for _ in range(tries):
        r = design(rng, statics, **{k: (v(rng) if callable(v) else v) for k, v in kw.items()})
        if r is not None and want(r[1]["nc"], r[1]["nl"]):
            return r
    raise RuntimeError("no designed state found for %s" % (kw,))


# the robots the batches are made of: (sampler arguments, predicate on (contacts, limit rows))
KINDS = {
    "air": (dict(family="stand", n_viol=0, k_ground=0), lambda c, l: c == 0 and l == 0),
    "light": (dict(family="stand", n_viol=lambda r: int(r.integers(0, 3)), k_ground=lambda r: int(r.integers(1, 5))),
              lambda c, l: 1 <= c and 3 * c + l <= 16),
    "heavy": (dict(family="fold", n_viol=lambda r: int(r.integers(2, 8)), k_ground=lambda r: int(r.integers(6, 9)), tilt=0.05),
              lambda c, l: 17 <= 3 * min(c, MAX_CON) + min(l, MAX_LIM) < 32),
    "mid": (dict(family="fold", n_viol=lambda r: int(r.integers(2, 6)), k_ground=lambda r: int(r.integers(5, 7)), tilt=0.05),
            lambda c, l: 17 <= 3 * c + l <= 20),
    "light12": (dict(family="stand", n_viol=lambda r: int(r.integers(0, 3)), k_ground=lambda r: int(r.integers(1, 4))),
                lambda c, l: 1 <= c and 3 * c + l <= 12),
    "exact32": (dict(family="fold", n_viol=8, k_ground=8, tilt=0.05), lambda c, l: c == 8 and l == 8),
    "ccap": (dict(family="fold", n_viol=lambda r: int(r.integers(0, 6)), k_ground=lambda r: int(r.integers(9, 13)), tilt=0.05),
             lambda c, l: c > MAX_CON),
    "lcap": (dict(family="random", n_viol=lambda r: int(r.integers(9, 13)), k_ground=lambda r: int(r.integers(0, 4)), tilt=0.3),
             lambda c, l: l > MAX_LIM),
}


def robot(rng, statics, name, **over):
    kw, want = KINDS[name]
    kw = dict(kw); kw.update(over)
    return sample(rng, statics, want, **kw)


# ---------------------------------------------------------------------------------------------------------------- lane mapping
def warp_cases(nc, nl):
    """The step kernel's pairing for one sub-step of a batch with raw per-env counts nc, nl: per CTA, per warp, the two envs and
    the case.  Rule (llq_step16.cuh): counts are capped (8 contacts, 8 limit rows); rank by 3 nc + nl descending, ties to the lower
    slot; warp w takes ranks w and EPB - 1 - w.  Unused slots of the last CTA are copies of env N - 1.
    Returns (list of (cta, warp, env_a, env_b, rows_a, rows_b, case), set of cases reached)."""
    nc, nl = np.asarray(nc), np.asarray(nl)
    n = len(nc)
    rows = 3 * np.minimum(nc, MAX_CON) + np.minimum(nl, MAX_LIM)
    out, reached = [], set()
    if (nc > MAX_CON).any():
        reached.add("contact_cap")
    if (nl > MAX_LIM).any():
        reached.add("limit_cap")
    for c in range((n + EPB - 1) // EPB):
        envs = [min(c * EPB + s, n - 1) for s in range(EPB)]
        key = [(-rows[e], s) for s, e in enumerate(envs)]
        order = sorted(range(EPB), key=lambda s: key[s])
        ragged = c * EPB + EPB > n
        if ragged and rows[n - 1] == max(rows[e] for e in envs) and rows[n - 1] > 0:
            reached.add("shadow")
        for w in range(EPB // 2):
            sa, sb = order[w], order[EPB - 1 - w]
            na, nb = int(rows[envs[sa]]), int(rows[envs[sb]])
            if na + nb == 0:
                case = "empty"
            elif na + nb > 32:
                case = "two_pass"
            elif na == 32 and nb == 0:
                case = "exact32"
            elif na <= 16 and nb <= 16:
                case = "split16"
            else:
                case = "borrow" if nb > 0 else "borrow_empty"
            reached.add(case)
            out.append((c, w, envs[sa], envs[sb], na, nb, case))
    return out, reached


def lane_offset(mapping, env):
    """First lane of env's rows, counted from the start of a half-warp: 0 for the lower env of a warp, for the upper env of a split-16
    warp (lanes 16 + r) and for both envs of a two-pass warp (the upper half-warp then receives the lower one's partial sums, and
    a + b = b + a); the partner's row count for the upper env of a borrow warp.  An env's impulse sums are the same tree of
    additions, hence bit-identical, wherever its offset is the same: padded sweep steps add 0 * delta, partner lanes add +0."""
    for c, w, ea, eb, na, nb, case in mapping:
        if ea == env or eb == env:
            return na if case == "borrow" and eb == env and ea != env else 0
    raise KeyError(env)


# ---------------------------------------------------------------------------------------------------------------- batches
def ground_batch(rng, statics, kind=0):
    """A batch whose CTAs reach every case of CASES on the ground (and, with statics.walls, against the arena walls):
      CTA 0  exact32 + 5 light + 10 airborne     -> exact32, split16 (light + air), empty (air + air)
      CTA 1  8 with 17..20 rows + 8 with <= 12      -> borrow (every pair <= 32 rows, the partner's rows start at lane nA)
      CTA 2  16 heavy, contact and limit overflow -> two_pass, contact_cap, limit_cap
      CTA 3  ragged: 6 airborne, 1 light, env N - 1 heavy (8 copies of it fill the CTA) -> shadow, two_pass, borrow_empty
    N = 56 (SEPMC counts robots in pairs).  kind 2 (SEPMC) also puts some robots against a wall."""
    walls = kind == 2
    def r(name):
        over = {}
        if walls and rng.random() < 0.4 and name != "air":
            over["target"] = ("wall", int(rng.integers(1, 4)))
        return robot(rng, statics, name, **over)
    plan = (["exact32"] + ["light"] * 5 + ["air"] * 10 + ["mid"] * 8 + ["light12"] * 8
            + ["heavy"] * 12 + ["ccap"] * 2 + ["lcap"] * 2 + ["air"] * 6 + ["light"] + ["heavy"])
    got = [r(p) for p in plan]
    return np.stack([g[0] for g in got]), [g[1] for g in got]


def corridor_batch(rng, statics_of, boxes, nbox, element=1):
    """EPMC corridor: env i is designed against its own corridor (statics_of(i)) -- on a box top, against a box face, on an edge
    cylinder, heavy on the ground between the boxes -- 2 CTAs and a ragged third.  Bars (element 2) have roles of their own, each a
    robot standing on the ground under a bar with its back touching it: a sphere at the bar's bottom face (n = -z), trunk corners
    (r = 0) whose centre is inside the bar, a sphere on one of its bottom-edge cylinders (the two sides in turn); and heavy robots on
    the ground between the bars."""
    n = boxes.shape[0]
    states, decs = [], []
    for i in range(n):
        S = statics_of(i)
        nb = int(nbox[i])
        role = i % (5 if element == 2 else 4)
        for _ in range(400):
            j = int(rng.integers(2, nb))
            want = None
            if element == 2:
                if role < 2:                           # role 1: a trunk corner's centre inside the bar
                    kw = dict(family="stand", n_viol=0, tilt=0.1, k_ground=int(rng.integers(1, 5)), target=("under", j, int(rng.integers(1, 3))))
                    want = (lambda d: d["inside"] == 0 and d["nc"] > d["n_off_ground"] and 1 in d["kind"]) if role == 0 else (lambda d: d["inside"] > 0 and d["nc"] > d["n_off_ground"])
                elif role < 4:                         # the two bottom-edge cylinders in turn
                    kw = dict(family="stand", n_viol=0, tilt=0.1, k_ground=int(rng.integers(1, 5)),
                              target=("under_cyl", 2 * (j - 2) + (i // 5 + role) % 2, int(rng.integers(1, 3))))
                    want = lambda d: d["nc"] > d["n_off_ground"] > 0 and 2 in d["kind"]
                else:
                    kw = dict(family="fold", n_viol=int(rng.integers(3, 8)), k_ground=int(rng.integers(6, 9)), tilt=0.05)
                    want = lambda d: 3 * min(d["nc"], MAX_CON) + min(d["nl"], MAX_LIM) > 16
            elif role == 0:
                kw = dict(family="stand", n_viol=int(rng.integers(0, 3)), target=("top", j, int(rng.integers(1, 5))))
            elif role == 1:
                kw = dict(family="stand", n_viol=int(rng.integers(0, 3)), k_ground=int(rng.integers(0, 4)), target=("face", j, int(rng.integers(1, 4))))
            elif role == 2:
                kw = dict(family="stand", n_viol=int(rng.integers(0, 2)), tilt=0.4, target=("cyl", 2 * (j - 2) + int(rng.integers(0, 2)), int(rng.integers(1, 3))))
            else:
                kw = dict(family="fold", n_viol=int(rng.integers(3, 8)), k_ground=int(rng.integers(6, 9)), tilt=0.05, target=("face", j, 1))
                want = lambda d: 3 * min(d["nc"], MAX_CON) + min(d["nl"], MAX_LIM) > 16
            res = design(rng, S, **kw)
            if res is not None and (want is None or want(res[1])):
                break
        else:
            raise RuntimeError("no corridor state for env %d (role %d)" % (i, role))
        states.append(res[0]); decs.append(res[1])
    return np.stack(states), decs


LEGACY_FEATURES = {0: ("ground", "off_ground"),
                   1: ("foot_deeper", "wheel_deeper", "wheel_alone", "leg_order", "ignored", "off_ground")}


def features(dec):
    """the legacy-set categories one designed state reaches"""
    f = {x for x in dec["legs"] if x is not None}
    if dec["leg_order"]:
        f.add("leg_order")
    if dec["ignored"]:
        f.add("ignored")
    if dec["n_off_ground"]:
        f.add("off_ground")
    if dec["nc"] > dec["n_off_ground"]:
        f.add("ground")
    return f


def legacy_batch(rng, statics_of, n, rule, boxes=0):
    """Rules 0 and 1 (feet; feet and knee wheels, one contact per leg): 3 CTAs, N = n (>= 40).  CTA 0: 6 light robots (<= 12 rows)
    beside 10 airborne ones -> split16, empty; CTA 1: 8 robots with 17..20 rows (4 contacts, >= 5 limit rows) beside 8 light ones ->
    borrow; CTA 2 (ragged): airborne robots and env N - 1 with 17..20 rows -> borrow_empty.  The light robots take the categories of
    LEGACY_FEATURES in turn (against the statics' walls or boxes where there are any: boxes > 2 is the corridor's box count)."""
    walls = statics_of(0).walls
    feats = [f for f in LEGACY_FEATURES[rule] if (walls or boxes > 2) or f not in ("ignored", "off_ground")]
    plan = (["light"] * 6 + ["air"] * 10 + ["mid"] * 8 + ["light"] * 8 + ["air"] * (n - 33) + ["mid"])
    states, decs, nl_ = [], [], 0
    for i, role in enumerate(plan):
        S = statics_of(i)
        want_f = feats[nl_ % len(feats)] if role == "light" else None
        nl_ += role == "light"
        for _ in range(6000):
            j = int(rng.integers(2, boxes)) if boxes > 2 else 0
            k = int(rng.integers(1, 4))
            target = None
            if want_f in ("ignored", "off_ground"):
                tail = "_any" if want_f == "ignored" else ""
                target = ("wall" + tail, k) if walls else (("face" + tail, j, k) if rng.random() < 0.7 else ("top", j, k))
            if role == "air":
                kw = dict(family="stand", n_viol=0, k_ground=0)
            elif role == "mid":
                kw = dict(family="stand", n_viol=int(rng.integers(5, 9)), k_ground=int(rng.integers(4, S.ns + 1)), tilt=0.1)
            else:
                kw = dict(family=("stand", "fold")[int(rng.integers(0, 2))], n_viol=int(rng.integers(0, 2)),
                          k_ground=int(rng.integers(0 if target else 1, min(7, S.ns + 1))), tilt=0.3, target=target)
            res = design(rng, S, **kw)
            if res is None:
                continue
            d = res[1]
            rows = 3 * d["nc"] + d["nl"]
            if role == "air" and d["nc"] == 0 and d["nl"] == 0:
                break
            if role == "mid" and 17 <= rows <= 20:
                break
            if role == "light" and 1 <= d["nc"] and rows <= 12 and want_f in features(d):
                break
        else:
            raise RuntimeError("no rule-%d state for env %d (%s, %s)" % (rule, i, role, want_f))
        states.append(res[0]); decs.append(d)
    return np.stack(states), decs
