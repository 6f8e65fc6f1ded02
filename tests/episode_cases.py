"""fp64 statement of the PMC episode logic and designed batches on which every branch of it is decisive (host only, numpy float64).

The statement covers what the learner is handed after one `llq_step` of the PMC engine: the mocap clock, the kinematic target, the
five-term tracking reward and `reward_sum`, the termination flags, the hurdle-plate hand-over, the prioritized clip table
(`F_AVG_REWARD`, `F_SAMPLE_PROB`), the clip / phase draw of an auto-reset and the reset row.  It is computed from the fields read back
after the step and the fields set before it, so it needs no dynamics: the batches run with the physics off (no PD torque, no gravity,
no solver iteration, no push) and with zero velocities, so every pose stays where it was set.

  clock     `time += sim_dt` once per sub-step, in sequence; the cursor is `floor(t / frame_dt)` of the time *before* the last
            increment (the one-sub-step lag of the reference), clamped to `nf - margin + 2`
  target    motion_lib's interpolation on the frames at the precision the engine stores them (positions fp64, quaternion and joints
            fp32)
  reward    the five terms of primitive_level_env with the feet of tests/helpers.foot_positions; `reward_sum` accumulates in fp32
  done      fall (`|left_z| > 1/sqrt 2` or `R22 < 0.5`), ended (`frame_id >= nf - margin - 1`), diff (`angle > 1` or `dp > 1`)
  plates    `ob_id` moves on while `time > apex + 0.5` (the plates of these batches are out of reach, so no plate is hit)
  table     the highest finished env index wins its clip; `avg[c] = float32 reward_sum / max_steps[c]`; `p = (1 - avg)^factor / sum`,
            `cdf = cumsum(p) / cumsum(p)[-1]`, both sums sequential
  draw      Philox4x32-10, counter (gid lo, gid hi, episode lo, episode hi), key (seed lo, seed hi), `u = (c + 0.5) / 2^32`; the clip is
            the first with `cdf > u1`, the phase `u2 * frame_dt * (nf - margin - 1)`

Error model.  `policy_cases.ErrorModel`: every input (the fp32 state read back, the stored mocap frames) is perturbed by one fp32
rounding, `x (1 + u r)`, every output by `u |y| r`, and the results of fp32 rotation algebra by an absolute `u` on unit quaternions
and rotation vectors and `u |v|` on rotated vectors; the largest deviation over R_DRAWS draws is the output's sensitivity S.  The
GPU bar is KAPPA S + 2^-23 |ref|.

Decisiveness.  Every continuous branch quantity (left_z, R22, angle, dp) clears its threshold by at least DELTA on the post-step
state.  The table is stated from the fp32 reward sums the engine keeps, so it is exact whatever the last bit of a reward.  Integer
branches (cursor, `ob_id`, the clip draw) are hit exactly; the designed cdf edges lie 1e-8 to 1e-6 from the draw (an edge closer
than that would move across the draw with one fp32 ulp of a reward sum, between the builder and the engine).
"""
import numpy as np
from scipy.spatial.transform import Rotation as R

import perception_cases as pcs

from lifelike_agility_and_play_b200.mocap import MocapTable, synthetic_mocap
from lifelike_agility_and_play_b200.model.compile_model import load_model, rpy_to_matrix
from policy_cases import ErrorModel, REF, U, philox4x32, R_DRAWS

# GPU bar factor: at least 4x the largest error / S measured on an H100 80GB HBM3 at a 400 W power limit: 8.8 (the observation;
# reset rows 2.9, kin 0.5, reward 0.6)
KAPPA = 64.0
DELTA = 1e-4
SEED = 20261017
POLICY_DT = 0.02
PHYSICS_OFF = dict(solver_iters=0, kp=0.0, kd=0.0, gravity_z=0.0, push_enabled=0)
TILT = 0.5                    # the mocap base is pitched by 0.5 rad, so R22 < 0.5 can be reached with angle < 1
PAD_FRAMES = 256              # the engine pads the frame table with copies of the last frame
PLATE_APEX = (0.3, 0.5, 0.7)  # plates of the clips c % 3 != 1 (the others have none), 10 km away unless a hit env is designed on them
PLATE_HALF = (0.01, 0.01, 1.0)  # a thin post: the proxy it meets first is the one nearest in the horizontal plane
BREAKING = 0.02 * 0.025       # contact_breaking of the default configuration
PROXY_KINDS = ("foot", "wheel", "hip", "corner")  # kinds 0..3 of the model's proxy table (4, the handles, serve SEPMC only)
LIMIT = 0.70710678118654752
W_DEFAULT = (0.3, 0.05, 0.1, 0.5, 0.05)

# batches: (n envs, n clips, sub-steps, prioritized_sample_factor, global_env_offset, reward weights)
CASES = [
    (1, 6, 10, 3.0, 0, W_DEFAULT),
    (15, 1, 10, 3.0, 0, W_DEFAULT),
    (16, 66, 10, 3.0, 0, (0.05, 0.05, 0.8, 0.05, 0.05)),
    (17, 127, 10, 2.5, 0, (0.05, 0.8, 0.05, 0.05, 0.05)),
    (31, 128, 1, 3.0, 0, W_DEFAULT),
    (33, 129, 10, 3.0, 2 ** 32 - 5, (0.05, 0.05, 0.05, 0.05, 0.8)),
    (4097, 300, 10, 3.0, 0, W_DEFAULT),
]

CLOCK_CATS = ("ended_below", "ended_at", "clamp", "boundary", "recip")
TERM_CATS = ("left_pos_in", "left_pos_out", "left_neg_in", "left_neg_out", "r22_in", "r22_out", "angle_in", "angle_out", "dp_in", "dp_out")
PLATE_CATS = ("ob_before", "ob_after", "ob_multi", "ob_last", "ob_none")
HIT_CATS = tuple("hit_%s_%s" % (k, side) for k in PROXY_KINDS for side in ("in", "out"))
NAN_CATS = ("nan_action", "nan_state")
OTHER_CATS = ("track", "jp", "finish")
CATS = CLOCK_CATS + TERM_CATS + PLATE_CATS + HIT_CATS + NAN_CATS + OTHER_CATS
FINISHING = ("ended_at", "clamp", "left_pos_in", "left_neg_in", "r22_in", "angle_in", "dp_in", "finish", "nan_state") + HIT_CATS[0::2]
TERMS = ("jp", "jv", "ee", "pose", "vel")


# ------------------------------------------------------------------------------------------------------------ mocap and geometry
def mocap(n_clips):
    """synthetic clips of 300..420 frames, the base pitched by TILT; with their plate table"""
    mc = synthetic_mocap(n_clips, seed=n_clips, min_frames=300, max_frames=420)
    f = mc.frames.copy()
    f[:, 3:7] = (R.from_quat(f[:, 3:7]) * R.from_euler("y", TILT)).as_quat()
    mc = MocapTable(f, mc.offsets, mc.frame_dt, mc.names)
    rows, offs = [], [0]
    for c in range(n_clips):
        if c % 3 != 1:
            rows += [[a, 1e4, 1e4, 0.0] for a in PLATE_APEX]
        offs.append(len(rows))
    return mc, (np.array(rows, np.float64).reshape(-1, 4), np.array(offs, np.int32))


def stored_frames(mc):
    """the frame table as the engine holds it: quaternion and joints in fp32, padded with the last frame"""
    f = mc.frames.copy()
    f[:, 3:] = f[:, 3:].astype(np.float32).astype(np.float64)
    return np.concatenate([f, np.repeat(f[-1:], PAD_FRAMES, 0)])


def margin(frame_dt):
    return int(np.ceil(POLICY_DT / frame_dt)) + int(1.0 / frame_dt) + 2


def max_steps(mc):
    m = margin(mc.frame_dt)
    return np.array([(mc.offsets[c + 1] - mc.offsets[c] - m) * mc.frame_dt / POLICY_DT for c in range(mc.n_clips)])


def quat_matrix(q):
    x, y, z, w = (q / np.linalg.norm(q, axis=-1, keepdims=True)).T
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], -1),
                     np.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], -1),
                     np.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1)], -2)


_MODEL = []


def model():
    if not _MODEL:
        _MODEL.append(load_model())
    return _MODEL[0]


def _rodrigues(axis, q):
    a = np.asarray(axis, np.float64)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    s, c = np.sin(q)[:, None, None], np.cos(q)[:, None, None]
    return np.eye(3) + s * K + (1 - c) * (K @ K)


def foot_positions(st):
    """[n, 4, 3] world CoM of the four link_*4 (tests/helpers.foot_positions, batched)"""
    links = model()["links"]
    Rb = quat_matrix(st[:, 3:7])
    Rl, pl = [None] * len(links), [None] * len(links)
    Rl[0] = Rb @ np.array(links[0]["R_in"]).T
    pl[0] = st[:, 0:3] - Rl[0] @ np.array(links[0]["inertial_xyz"])
    out = {}
    for i, l in enumerate(links):
        if i > 0:
            pi = l["parent_index"]
            pl[i] = pl[pi] + Rl[pi] @ np.array(l["joint_xyz"])
            Rq = _rodrigues(l["axis"], st[:, 13 + l["dof_index"]]) if l["joint_type"] == "revolute" else np.eye(3)
            Rl[i] = Rl[pi] @ rpy_to_matrix(l["joint_rpy"]) @ Rq
        out[l["name"]] = pl[i] + Rl[i] @ np.array(l["inertial_xyz"])
    return np.stack([out["link_%s4" % leg] for leg in ("FR", "FL", "HR", "HL")], 1)


# ------------------------------------------------------------------------------------------------------------ the statement
def clock(t0, substeps, sim_dt, frame_dt, nf, m):
    """(time after the step, cursor, fraction): the cursor samples the time before the last increment, then the clamp"""
    t = np.array(t0, np.float64)
    for s in range(substeps):
        if s == substeps - 1:
            fid = np.floor(t / frame_dt).astype(np.int64)
            frac = (t - fid * frame_dt) / frame_dt
            last = nf - m + 2
            over, under = fid > last, fid < 0
            fid = np.where(over, last, np.where(under, 0, fid)); frac = np.where(over | under, 0.0, frac)
        t = t + sim_dt
    return t, fid, frac


def mocap_state(frames, idx, frac, dt, em=REF):
    """motion_lib's interpolated state [n, 37] between frames idx and idx + 1 (global indices)"""
    fc, fn = em.rel(frames[idx]), em.rel(frames[idx + 1])
    frac = np.asarray(frac, np.float64)
    rc, rn = R.from_quat(fc[:, 3:7]), R.from_quat(fn[:, 3:7])
    out = np.zeros((len(idx), 37))
    out[:, 0:3] = fc[:, 0:3] + frac[:, None] * (fn[:, 0:3] - fc[:, 0:3])
    out[:, 3:7] = (rc * R.from_rotvec(frac[:, None] * (rc.inv() * rn).as_rotvec())).as_quat()
    out[:, 7:10] = (fn[:, 0:3] - fc[:, 0:3]) / dt
    rv = (rn * rc.inv()).as_rotvec()
    a = np.linalg.norm(rv, axis=1)[:, None]
    out[:, 10:13] = rv / (a + 1e-8) * a / dt
    out[:, 13:25] = fc[:, 7:] + frac[:, None] * (fn[:, 7:] - fc[:, 7:])
    out[:, 25:37] = (fn[:, 7:] - fc[:, 7:]) / dt
    # fp32 quaternion algebra: an absolute error of u on the unit quaternion and on the rotation vector of the velocity
    out[:, 3:7] = em.add(out[:, 3:7], 1.0)
    out[:, 10:13] = em.add(out[:, 10:13], 4.0 / dt)
    return out


def _rotated(v, em):
    """a vector rotated in fp32: an absolute error of u |v| on every component"""
    return em.add(v, np.linalg.norm(v, axis=1)[:, None])


def prop(st, em=REF):
    Rb = R.from_quat(st[:, 3:7])
    return np.concatenate([st[:, 13:25], st[:, 25:37], _rotated(Rb.inv().apply(st[:, 10:13]), em), _rotated(Rb.inv().apply(st[:, 7:10]), em),
                           em.add(Rb.as_matrix()[:, 2, :], 1.0)], 1)


def future(frames, start, frac, dt, base_pos, base_orn, em=REF):
    """[n, 72]: the four future targets (1/30, 1/15, 1/3, 1 s) relative to the base; start = global index of the cursor frame"""
    rb = R.from_quat(base_orn)
    out = []
    for tf in (1. / 30., 1. / 15., 1. / 3., 1.):
        t = dt * frac + tf
        fid = np.floor(t / dt).astype(np.int64)
        s = mocap_state(frames, start + fid, t / dt - fid, dt, em)
        rv = (rb.inv() * R.from_quat(s[:, 3:7])).as_rotvec()
        a = np.linalg.norm(rv, axis=1)[:, None]
        out += [_rotated(rb.inv().apply(s[:, 0:3] - base_pos), em), em.add(rv / (a + 1e-8) * a, 4.0), s[:, 13:25]]
    return np.concatenate(out, 1)


def tracking(dyn, kin, weights, em=REF):
    """(reward, per-term weighted loss [n, 5], angle, dp)"""
    w = np.array(weights, np.float64) / np.sum(weights)
    ep = em.add(np.sum((foot_positions(dyn) - foot_positions(kin)) ** 2, (1, 2)), 40 * U)
    a = np.linalg.norm((R.from_quat(kin[:, 3:7]) * R.from_quat(dyn[:, 3:7]).inv()).as_rotvec(), axis=1)
    a = em.add(a, 4.0)
    dp = np.sum((dyn[:, 0:3] - kin[:, 0:3]) ** 2, 1)
    r = np.stack([np.exp(-1.0 * np.sum((dyn[:, 13:25] - kin[:, 13:25]) ** 2, 1)), np.exp(-0.1 * np.sum((dyn[:, 25:37] - kin[:, 25:37]) ** 2, 1)),
                  np.exp(-40.0 * ep), np.exp(-20.0 * dp - 10.0 * a ** 2),
                  np.exp(-2.0 * np.sum((dyn[:, 7:10] - kin[:, 7:10]) ** 2, 1) - 0.2 * np.sum((dyn[:, 10:13] - kin[:, 10:13]) ** 2, 1))], 1)
    r = em.rel(r)
    return r @ w, w * (1 - r), a, dp


def tilt(st):
    """(left_z, R22) of the base orientation"""
    M = quat_matrix(st[:, 3:7])
    return M[:, 0, 2] * M[:, 1, 0] - M[:, 1, 2] * M[:, 0, 0], M[:, 2, 2]


def plate_clearance(ctx, before, st):
    """[n, proxies] distance of each detection proxy (feet, knee wheels, hips: spheres; trunk corners: points) from the env's active
    plate, minus the contact-breaking threshold; +inf where the clip has no plate or the plate is more than 10 m away"""
    n = len(st)
    kinds = np.flatnonzero(pcs.PROXIES[:, 5] <= 3)
    out = np.full((n, len(kinds)), np.inf)
    clip = before["clip"]
    for i in range(n):
        o, no = ctx["ob_off"][clip[i]], ctx["ob_off"][clip[i] + 1] - ctx["ob_off"][clip[i]]
        if no == 0 or not np.all(np.isfinite(st[i])):
            continue
        row = ctx["ob_table"][o + before["ob_id"][i]]
        if np.hypot(st[i, 0] - row[1], st[i, 1] - row[2]) > 10.0:
            continue
        w = pcs.proxy_points(st[i])[kinds] - np.array([row[1], row[2], 0.0])
        c, s_ = np.cos(row[3]), np.sin(row[3])
        b = np.stack([c * w[:, 0] + s_ * w[:, 1], -s_ * w[:, 0] + c * w[:, 1], w[:, 2]], 1)
        q = b - np.clip(b, -np.array(PLATE_HALF), np.array(PLATE_HALF))
        out[i] = np.linalg.norm(q, axis=1) - pcs.PROXIES[kinds, 4] - BREAKING
    return out


def step_statement(ctx, before, st, em=REF):
    """the outputs of one step from the fields set before it (`before`) and the post-step state `st` read back"""
    frames, off, nf, m, dt = ctx["frames"], ctx["off"], ctx["nf"], ctx["m"], ctx["mc"].frame_dt
    clip = before["clip"]
    time, fid, frac = clock(before["time"], ctx["substeps"], ctx["sim_dt"], dt, nf[clip], m)
    st = em.rel(np.asarray(st, np.float64))
    kin = mocap_state(frames, off[clip] + fid, frac, dt, em)
    rew, loss, angle, dp = tracking(st, kin, ctx["weights"], em)
    left_z, r22 = tilt(st)
    fall = (np.abs(left_z) > LIMIT) | (r22 < 0.5)
    ended = fid >= nf[clip] - m - 1
    diff = (angle > 1.0) | (dp > 1.0)
    clear = plate_clearance(ctx, before, st)
    ob_hit = (clear < 0).any(1)
    # a non-finite state or reward: `bad`, done with reward 0 (comparisons with NaN are false, so fall / diff / the hit stay off)
    bad = ~np.isfinite(st).all(1) | ~np.isfinite(rew)
    rew = np.where(bad, 0.0, rew)
    ob = before["ob_id"].copy()
    oo, no = ctx["ob_off"][clip], ctx["ob_off"][clip + 1] - ctx["ob_off"][clip]
    for i in range(len(ob)):
        while ob[i] < no[i] - 1 and time[i] > ctx["ob_table"][oo[i] + ob[i], 0] + 0.5:
            ob[i] += 1
    obs = np.concatenate([before["obs"][:, 33:99], prop(st, em), before["obs"][:, 111:135], before["actions"],
                          future(frames, off[clip] + fid, frac, dt, st[:, 0:3], st[:, 3:7], em)], 1)
    rs = (np.float32(1) * before["reward_sum"].astype(np.float32) + rew.astype(np.float32)).astype(np.float32)
    return dict(time=time, frame_id=fid, frac=frac, kin=kin, reward=em.add(rew, np.abs(rew)), loss=loss, angle=angle, dp=dp,
                left_z=left_z, r22=r22, fall=fall, ended=ended, diff=diff, clear=clear, ob_hit=ob_hit, bad=bad,
                done=fall | ended | diff | ob_hit | bad, ob_id=ob, obs=em.add(obs, np.abs(obs)), reward_sum=rs, reward64=rew)


def sensitivity(ctx, before, st, draws=R_DRAWS):
    """S of reward, kin, obs: the largest deviation from the reference over `draws` draws of the error model"""
    ref = step_statement(ctx, before, st)
    S = {k: np.zeros_like(ref[k]) for k in ("reward64", "kin", "obs")}
    for d in range(draws):
        got = step_statement(ctx, before, st, ErrorModel(SEED + d))
        S["reward64"] = np.maximum(S["reward64"], np.abs(got["reward"] - ref["reward64"]))
        for k in ("kin", "obs"):
            S[k] = np.maximum(S[k], np.abs(got[k] - ref[k]))
    return ref, S


def table(ctx, done, clip, rs, avg_old):
    """(avg, p, cdf, winner per clip) after the step's table update"""
    C = len(avg_old)
    win = np.full(C, -1)
    for e in np.nonzero(done)[0]:
        win[clip[e]] = max(win[clip[e]], e)
    avg = np.array(avg_old, np.float64)
    for c in np.nonzero(win >= 0)[0]:
        avg[c] = np.float64(rs[win[c]]) / ctx["max_steps"][c]
    w = np.power(1.0 - avg, ctx["factor"])
    p = w / np.cumsum(w)[-1]
    cdf = np.cumsum(p)
    return avg, p, cdf / cdf[-1], win


def uniforms(seed, gid, ep):
    gid, ep = np.asarray(gid, np.int64).astype(np.uint64), np.asarray(ep, np.int64).astype(np.uint64)
    M = np.uint64(0xFFFFFFFF)
    c = philox4x32(gid & M, gid >> np.uint64(32), ep & M, ep >> np.uint64(32), int(seed) & 0xFFFFFFFF, int(seed) >> 32)
    return (c[0].astype(np.float64) + 0.5) * (1.0 / 4294967296.0), (c[1].astype(np.float64) + 0.5) * (1.0 / 4294967296.0)


def draw(ctx, cdf, gid, ep):
    """(clip, t0, cursor, fraction) of the auto-reset of envs with global ids gid and episode ids ep"""
    u1, u2 = uniforms(ctx["seed"], gid, ep)
    above = cdf[None, :] > u1[:, None]
    clip = np.where(above.any(1), np.argmax(above, 1), len(cdf) - 1)
    nf, m, dt = ctx["nf"][clip], ctx["m"], ctx["mc"].frame_dt
    t0 = u2 * (dt * (nf - m - 1).astype(np.float64))
    fid = np.floor(t0 / dt).astype(np.int64)
    frac = (t0 - fid * dt) / dt
    return clip, t0, fid, frac, u1


def reset_statement(ctx, clip, fid, frac, em=REF):
    """(state [n, 37], observation row [n, 207]) of a reset at (clip, cursor, fraction)"""
    frames, start, dt = ctx["frames"], ctx["off"][clip] + fid, ctx["mc"].frame_dt
    st = mocap_state(frames, start, frac, dt, em)
    p = prop(st, em)
    obs = np.concatenate([p, p, p, np.zeros((len(st), 36)), future(frames, start, frac, dt, st[:, 0:3], st[:, 3:7], em)], 1)
    return st, obs


def reset_sensitivity(ctx, clip, fid, frac, draws=R_DRAWS):
    st, obs = reset_statement(ctx, clip, fid, frac)
    Ss, So = np.zeros_like(st), np.zeros_like(obs)
    for d in range(draws):
        em = ErrorModel(SEED + 100 + d)
        s2, o2 = reset_statement(ctx, clip, fid, frac, em)
        Ss = np.maximum(Ss, np.abs(em.add(s2, np.abs(s2)) - st)); So = np.maximum(So, np.abs(em.add(o2, np.abs(o2)) - obs))
    return st, obs, Ss, So


# ------------------------------------------------------------------------------------------------------------ designed batches
def context(case):
    n, n_clips, substeps, factor, gid0, weights = case
    mc, (ob_table, ob_off) = mocap(n_clips)
    nf = np.diff(mc.offsets).astype(np.int64)
    return dict(n=n, mc=mc, frames=stored_frames(mc), off=mc.offsets.astype(np.int64), nf=nf, m=margin(mc.frame_dt), substeps=substeps,
                sim_dt=1.0 / 500.0, factor=factor, gid0=gid0, weights=weights, seed=SEED + n, ob_table=ob_table, ob_off=ob_off,
                max_steps=max_steps(mc))


def engine_config(ctx, auto_reset):
    w = ctx["weights"]
    return dict(PHYSICS_OFF, substeps=ctx["substeps"], prioritized_sample_factor=ctx["factor"], global_env_offset=ctx["gid0"],
                seed=ctx["seed"], auto_reset=auto_reset, w_joint_pos=w[0], w_joint_vel=w[1], w_end_effector=w[2], w_root_pose=w[3],
                w_root_vel=w[4])


def _t0_for(ctx, rng, clip, fid_target):
    """a start time whose cursor lands on fid_target with a fraction well inside (0, 1)"""
    dt = ctx["mc"].frame_dt
    return (fid_target + rng.uniform(0.2, 0.8)) * dt - (ctx["substeps"] - 1) * ctx["sim_dt"]


def _search_t0(ctx, rng, clip, want):
    """a start time near a frame boundary whose sampled time t (the (substeps - 1)-th sum) satisfies want(t)"""
    dt, S1 = ctx["mc"].frame_dt, ctx["substeps"] - 1
    hi = ctx["nf"][clip] - ctx["m"] - 3
    for _ in range(2000):
        k = int(rng.integers(5, hi))
        t0 = k * dt - S1 * ctx["sim_dt"]
        for j in range(-64, 65):
            t = t0 + j * np.spacing(t0)
            ts = t
            for _ in range(S1):
                ts += ctx["sim_dt"]
            if want(ts, dt):
                return t
    raise RuntimeError("no start time found")


def _rotate(q, rot, world=False):
    r = R.from_quat(q)
    return ((rot * r) if world else (r * rot)).as_quat()


def _solve(f, target, lo, hi):
    for _ in range(80):
        mid = 0.5 * (lo + hi)
        if (f(mid) - target) * (f(lo) - target) > 0:
            lo = mid
        else:
            hi = mid
    return 0.5 * (lo + hi)


def _design_state(kin, cat, rng):
    """the post-step state of a category, from the kinematic target at the post-step clock; velocities zero"""
    st = kin.copy()
    st[7:13] = 0.0; st[25:37] = 0.0
    q = st[3:7]
    one = lambda qq: tilt(np.concatenate([np.zeros(3), qq])[None])
    side = rng.uniform(2, 8) * DELTA
    if cat.startswith("left"):
        sgn = 1.0 if "_pos_" in cat else -1.0
        tgt = sgn * (LIMIT + (side if cat.endswith("_in") else -side))
        q = _rotate(q, R.from_euler("y", -0.3))
        phi = _solve(lambda a: one(_rotate(q, R.from_euler("x", sgn * a)))[0][0], tgt, 0.0, 1.3)
        st[3:7] = _rotate(q, R.from_euler("x", sgn * phi))
    elif cat.startswith("r22"):
        tgt = 0.5 - side if cat.endswith("_in") else 0.5 + side
        th = _solve(lambda a: one(_rotate(q, R.from_euler("y", a)))[1][0], tgt, 0.0, 1.2)
        st[3:7] = _rotate(q, R.from_euler("y", th))
    elif cat.startswith("angle"):
        st[3:7] = _rotate(q, R.from_euler("z", 1.0 + side if cat.endswith("_in") else 1.0 - side), world=True)
    elif cat.startswith("dp"):
        d = np.sqrt(1.0 + side if cat.endswith("_in") else 1.0 - side)
        h = rng.uniform(0, 2 * np.pi)
        st[0] += d * np.cos(h); st[1] += d * np.sin(h)
    elif cat == "finish":
        st[0] += 2.0
    elif cat == "jp":
        st[13:25:3] += 0.35
    elif cat != "track":
        st[13:25] += rng.normal(0, 0.05, 12)
        st[0:3] += rng.normal(0, 0.03, 3)
    st[3:7] /= np.linalg.norm(st[3:7])
    return st.astype(np.float32)


def _place_plate(st, kind, side, rng):
    """(x, y) of a post that the first proxy of `kind` it meets touches by `side` DELTA-steps (in: inside the breaking threshold, out:
    just outside) while every other proxy stays at least 10 DELTA outside; None if no direction gives that"""
    rows = np.flatnonzero(pcs.PROXIES[:, 5] <= 3)
    P, r = pcs.proxy_points(st)[rows], pcs.PROXIES[rows, 4]
    kinds = pcs.PROXIES[rows, 5]
    half = np.array(PLATE_HALF)
    g = rng.uniform(2, 8) * DELTA * (-1.0 if side == "in" else 1.0)

    def clear(cx, cy):
        q = P - np.array([cx, cy, 0.0])
        return np.linalg.norm(q - np.clip(q, -half, half), axis=1) - r - BREAKING

    for a in rng.permutation(72) * (2 * np.pi / 72):
        u = np.array([np.cos(a), np.sin(a)])
        for j in np.flatnonzero(kinds == kind):
            lo, hi = 0.0, 1.0
            for _ in range(60):
                mid = 0.5 * (lo + hi)
                c = P[j, :2] + mid * u
                lo, hi = (mid, hi) if clear(*c)[j] < g else (lo, mid)
            c = P[j, :2] + 0.5 * (lo + hi) * u
            cl = clear(*c)
            others = np.delete(cl, j)
            if abs(cl[j] - g) < 1e-9 and (others >= 10 * DELTA).all():
                return c
    return None


def _designated_indices(n):
    """envs that finish on the table clips: env 0, env N - 1 and envs in different CTAs of the step kernel (16 envs per CTA) and of
    the reset kernel (32 per CTA)"""
    return sorted({i for i in (0, 1, 15, 16, 17, 31, 32, 33, 63, 64, 2048, 4095, n - 2, n - 1) if 0 <= i < n})


def build(case):
    """(ctx, before, categories): the designed fields of a batch; deterministic"""
    ctx = context(case)
    n, C = ctx["n"], ctx["mc"].n_clips
    rng = np.random.default_rng(SEED + n)
    fin_clips = [C // 2, min(C - 1, C // 2 + 1)] if C > 4 else list(range(C))          # the clips finishers use
    plate_clips = [c for c in range(C) if c % 3 != 1]
    # clips whose plates are moved next to a hit env: no other env uses them, so each such env owns one (clip, plate) slot
    cand = [c for c in plate_clips if c not in fin_clips and c not in (0, 1, C - 2, C - 1)]
    hit_clips = cand[::3] if C >= 30 else []
    slots = [(c, j) for c in hit_clips for j in range(len(PLATE_APEX))]
    plate_clips = [c for c in plate_clips if c not in hit_clips]
    free_clips = [c for c in range(C) if c not in hit_clips]
    ctx["ob_table"] = ctx["ob_table"].copy()
    cats = []
    tab = _designated_indices(n)
    for i in range(n):
        cat = "finish" if i in tab else CATS[(i * 7 + n) % len(CATS)]
        if (cat == "ob_none" and C == 1) or (cat in HIT_CATS and len(slots) <= sum(c in HIT_CATS for c in cats)):
            cat = "track"
        cats.append(cat)
    slot_of = {}
    clip = np.zeros(n, np.int64)
    t0 = np.zeros(n)
    ob0 = np.zeros(n, np.int64)
    dt = ctx["mc"].frame_dt
    for i, cat in enumerate(cats):
        if cat in HIT_CATS:
            slot_of[i] = slots[len(slot_of)]
            c, ob0[i] = slot_of[i]
        elif cat in FINISHING:
            c = fin_clips[(i // 3) % len(fin_clips)]
        elif cat.startswith("ob_") and cat != "ob_none":
            c = plate_clips[i % len(plate_clips)]
        elif cat == "ob_none":
            c = 1
        else:
            c = free_clips[int(rng.integers(len(free_clips)))]
        nf = ctx["nf"][c]
        clip[i] = c
        if cat == "ended_below":
            t0[i] = _t0_for(ctx, rng, c, nf - ctx["m"] - 2)
        elif cat == "ended_at":
            t0[i] = _t0_for(ctx, rng, c, nf - ctx["m"] - 1)
        elif cat == "clamp":
            t0[i] = _t0_for(ctx, rng, c, nf - ctx["m"] + 6)
        elif cat == "boundary":
            t0[i] = _search_t0(ctx, rng, c, lambda ts, dt: ts / dt == np.floor(ts / dt))
        elif cat == "recip":
            t0[i] = _search_t0(ctx, rng, c, lambda ts, dt: np.floor(ts / dt) != np.floor(ts * (1.0 / dt)))
        elif cat.startswith("ob_") and cat != "ob_none":
            apex = PLATE_APEX
            T = {"ob_before": apex[0] + 0.5 - rng.uniform(1e-9, 1e-6), "ob_after": apex[0] + 0.5 + rng.uniform(1e-9, 1e-6),
                 "ob_multi": apex[1] + 0.5 + rng.uniform(0.01, 0.1), "ob_last": apex[2] + 0.5 + rng.uniform(0.01, 0.1)}[cat]
            if cat == "ob_last":
                ob0[i] = len(apex) - 1
            t0[i] = _exact_end_time(ctx, T)
        else:
            t0[i] = _t0_for(ctx, rng, c, int(rng.integers(3, nf - ctx["m"] - 3)))
    time, fid, frac = clock(t0, ctx["substeps"], ctx["sim_dt"], dt, ctx["nf"][clip], ctx["m"])
    kin = mocap_state(ctx["frames"], ctx["off"][clip] + fid, frac, dt)
    st = np.stack([_design_state(kin[i], cats[i], rng) for i in range(n)])
    for i, (c, j) in slot_of.items():
        _, kind, side = cats[i].split("_")
        for _ in range(50):                   # a pose whose proxies leave a direction free: redraw the joint noise until one does
            xy = _place_plate(st[i].astype(np.float64), PROXY_KINDS.index(kind), side, rng)
            if xy is not None:
                break
            st[i] = _design_state(kin[i], cats[i], rng)
        else:
            raise RuntimeError("no plate placement for %s" % cats[i])
        ctx["ob_table"][ctx["ob_off"][c] + j, 1:3] = xy
    ep = np.where(rng.random(n) < 0.5, rng.integers(0, 1000, n), rng.integers(2 ** 32, 2 ** 40, n)).astype(np.int64)
    obs = rng.normal(0, 1, (n, 207)).astype(np.float32)
    actions = rng.uniform(-1, 1, (n, 12)).astype(np.float32)
    for i, cat in enumerate(cats):
        if cat == "nan_action":               # the PD target clamp maps NaN to its lower bound; the observation carries the NaN
            actions[i, rng.integers(12)] = np.nan
        elif cat == "nan_state":              # a NaN joint angle: the reward is NaN, the step turns `bad`
            st[i, 13 + rng.integers(12)] = np.nan
    before = dict(clip=clip, time=t0, ob_id=ob0, episode=ep, obs=obs, actions=actions, state=st,
                  reward_sum=np.zeros(n, np.float32), avg=rng.uniform(-0.2, 0.6, C))
    # reward_sum: fp32 values the step's reward does not add to exactly (avg = reward_sum / max_steps stays below 1)
    before["reward_sum"] = rng.uniform(0.0, 60.0, n).astype(np.float32)
    ref = step_statement(ctx, before, st.astype(np.float64))
    before["avg"], designed = design_edges(ctx, before, ref, rng)
    return ctx, before, cats, designed


def _exact_end_time(ctx, T):
    """a start time whose post-step time lands just below (or above) T, by at most 1e-6"""
    t0 = T - ctx["substeps"] * ctx["sim_dt"]
    for _ in range(4):
        t = t0
        for _ in range(ctx["substeps"]):
            t += ctx["sim_dt"]
        t0 += T - t
    return t0


def design_edges(ctx, before, ref, rng, n_inner=6):
    """F_AVG_REWARD to set before the step.  Clips without a finisher are free: a free pair (j, j + 1) is re-weighted so that cdf[j]
    lands 1e-8..1e-6 above or below the u1 of a finishing env -- the smallest u1 on the first edge, the largest on the last one, and
    up to n_inner others on the edge they fall next to.  Returns the table and {env: (edge clip j, side)}."""
    C = ctx["mc"].n_clips
    avg = before["avg"].copy()
    done = ref["done"]
    fin = np.nonzero(done)[0]
    if C < 4 or len(fin) < 2:
        return avg, {}
    u1, _ = uniforms(ctx["seed"], ctx["gid0"] + fin, before["episode"][fin])
    busy = set(int(c) for c in before["clip"][fin])
    f = ctx["factor"]
    order = [int(np.argmin(u1)), int(np.argmax(u1))] + [k for k in rng.permutation(len(fin)) if k not in (np.argmin(u1), np.argmax(u1))]
    plan, used = [], set()
    for r, k in enumerate(order):
        upd, _, cdf, _ = table(ctx, done, before["clip"], ref["reward_sum"], avg)
        j = 0 if r == 0 else (C - 2 if r == 1 else int(np.searchsorted(cdf, u1[k], side="right")))
        if j >= C - 1 or {j, j + 1} & (busy | used):
            continue
        side = 1.0 if r % 2 == 0 else -1.0
        t = u1[k] + side * 10 ** rng.uniform(-7.5, -6.2)
        w = np.power(1.0 - upd, f)
        P, pair = np.sum(w[:j]), w[j] + w[j + 1]
        Q = np.sum(w) - P - pair
        X = max(pair, 1.5 * max(P / t - P - Q, (t * (P + Q) - P) / (1 - t), 0.0))
        wj = t * (P + X + Q) - P
        avg[j], avg[j + 1] = 1.0 - wj ** (1.0 / f), 1.0 - (X - wj) ** (1.0 / f)
        used |= {j, j + 1}
        plan.append((int(fin[k]), j, side, u1[k], t))
        if len(plan) >= 2 + n_inner:
            break
    for _ in range(2):            # a rescaled pair moved the other edges: place them again, now with every pair's sum kept
        for e, j, side, u, t in plan:
            w = np.power(1.0 - table(ctx, done, before["clip"], ref["reward_sum"], avg)[0], f)
            P, X = np.sum(w[:j]), w[j] + w[j + 1]
            wj = t * np.sum(w) - P
            if 0.0 < wj < X:
                avg[j], avg[j + 1] = 1.0 - wj ** (1.0 / f), 1.0 - (X - wj) ** (1.0 / f)
    _, _, cdf, _ = table(ctx, done, before["clip"], ref["reward_sum"], avg)
    designed = {e: (j, side) for e, j, side, u, t in plan if 1e-8 <= side * (cdf[j] - u) <= 1e-6}
    return avg, designed


def reaches(ctx, before, ref, cat):
    """does each env reach its category on the post-step statement `ref`"""
    n = ctx["n"]
    m, nf = ctx["m"], ctx["nf"][before["clip"]]
    fid = ref["frame_id"]
    lz, r22 = ref["left_z"], ref["r22"]
    ok = np.zeros(n, bool)
    for i, c in enumerate(cat):
        ok[i] = {
            "ended_below": fid[i] == nf[i] - m - 2, "ended_at": fid[i] == nf[i] - m - 1,
            "clamp": fid[i] == nf[i] - m + 2 and ref["frac"][i] == 0.0,
            "boundary": True, "recip": True,
            "left_pos_in": lz[i] > LIMIT, "left_pos_out": LIMIT - 1e-3 < lz[i] < LIMIT, "left_neg_in": lz[i] < -LIMIT,
            "left_neg_out": -LIMIT < lz[i] < -LIMIT + 1e-3, "r22_in": r22[i] < 0.5, "r22_out": 0.5 < r22[i] < 0.501,
            "angle_in": 1.0 < ref["angle"][i] < 1.001, "angle_out": 0.999 < ref["angle"][i] < 1.0,
            "dp_in": 1.0 < ref["dp"][i] < 1.001, "dp_out": 0.999 < ref["dp"][i] < 1.0,
            "ob_before": ref["ob_id"][i] == 0 and ref["time"][i] > PLATE_APEX[0] + 0.5 - 1e-6,
            "ob_after": ref["ob_id"][i] == 1 and ref["time"][i] < PLATE_APEX[0] + 0.5 + 1e-6,
            "ob_multi": ref["ob_id"][i] == 2 and before["ob_id"][i] == 0, "ob_last": ref["ob_id"][i] == 2 and before["ob_id"][i] == 2,
            "ob_none": ctx["ob_off"][before["clip"][i] + 1] == ctx["ob_off"][before["clip"][i]],
            "track": ref["loss"][i, [0, 2, 3]].sum() < 1e-3, "jp": True, "finish": bool(ref["done"][i]),
            "nan_action": bool(np.isnan(before["actions"][i]).any()) and not ref["done"][i],
            "nan_state": bool(ref["bad"][i]) and ref["reward64"][i] == 0.0,
        }[c] if c not in HIT_CATS else _hit_reached(ref, i, c)
        if c in ("boundary", "recip"):
            t = before["time"][i]
            for _ in range(ctx["substeps"] - 1):
                t += ctx["sim_dt"]
            dt = ctx["mc"].frame_dt
            ok[i] = (t / dt == np.floor(t / dt)) if c == "boundary" else (np.floor(t / dt) != np.floor(t * (1.0 / dt)))
        if c in ("left_pos_out", "left_neg_out", "r22_out", "angle_out", "dp_out", "ended_below") and ref["done"][i]:
            ok[i] = False
    return ok


def _hit_reached(ref, i, cat):
    """the nearest proxy is of the category's kind, inside (or just outside) the threshold, and the only thing that ends the step"""
    _, kind, side = cat.split("_")
    rows = np.flatnonzero(pcs.PROXIES[:, 5] <= 3)
    cl = ref["clear"][i]
    j = int(np.argmin(cl))
    other = bool(ref["fall"][i] or ref["diff"][i] or ref["ended"][i] or ref["bad"][i])
    return pcs.PROXIES[rows[j], 5] == PROXY_KINDS.index(kind) and ((cl[j] < 0) == (side == "in")) and abs(cl[j]) < 1e-3 and not other


def decisive(ref):
    """every continuous branch quantity clears its threshold by DELTA (each proxy's plate clearance included)"""
    return ref["bad"] | ((np.abs(np.abs(ref["left_z"]) - LIMIT) >= DELTA) & (np.abs(ref["r22"] - 0.5) >= DELTA)
                         & (np.abs(ref["angle"] - 1.0) >= DELTA) & (np.abs(ref["dp"] - 1.0) >= DELTA) & (np.abs(ref["clear"]) >= DELTA).all(1))


_BUILT = {}


def case(k):
    if k not in _BUILT:
        _BUILT[k] = build(CASES[k])
    return _BUILT[k]


# ------------------------------------------------------------------------------------------------------------ running a batch
IO_PATHS = ("host", "pinned", "device1", "device2")    # device<r>: step_device into a slab with obs_ld > width and record mode r
_BLOB = []


def _blob():
    if not _BLOB:
        from lifelike_agility_and_play_b200.model.compile_model import pack_model
        _BLOB.append(pack_model(model()))
    return _BLOB[0]


def make(lib, ctx, auto_reset):
    from lifelike_agility_and_play_b200 import _capi as capi
    e = capi.VecEngine(lib, ctx["n"], _blob(), ctx["mc"], **engine_config(ctx, auto_reset))
    e.load_obstacles(ctx["ob_table"], ctx["ob_off"], PLATE_HALF)
    e.reset()
    return e


def set_before(e, before, table_too=True):
    from lifelike_agility_and_play_b200 import _capi as capi
    n = e.n
    for f, v in ((capi.F_STATE, before["state"]), (capi.F_WARMSTART, np.zeros((n, 32), np.float32)), (capi.F_CLIP, before["clip"]),
                 (capi.F_TIME, before["time"]), (capi.F_REWARD_SUM, before["reward_sum"]), (capi.F_EPISODE_ID, before["episode"]),
                 (capi.F_OB_ID, before["ob_id"]), (capi.F_OBS, before["obs"]), (capi.F_EPISODE_STEPS, np.zeros(n, np.int32))):
        e.set(f, v)
    if table_too:
        e.set(capi.F_AVG_REWARD, before["avg"])


class Slab:
    """step_device through a torch slab: two blocks of n rows of obs_ld = width + 16 floats and CANARY rows past each, so record
    mode 2 (trajectory columns in the row block before the observation's) has its rows; the canary rows must come back untouched"""
    CANARY = 3

    def __init__(self, e, record):
        import torch
        self.e, self.record, self.n, self.w = e, record, e.n, e.obs_dim
        self.ld = self.w + 16
        dev = torch.device("cuda", 0)
        self.rows = 2 * self.n + self.CANARY
        self.slab = torch.full((self.rows, self.ld), -7.0, device=dev)
        self.rew = torch.zeros(self.n + 1, device=dev); self.done = torch.zeros(self.n + 1, dtype=torch.uint8, device=dev)
        self.act = torch.zeros((self.n, 12), device=dev)
        e.set_option("record", record)

    def step(self, actions):
        import torch
        self.act.copy_(torch.from_numpy(actions))
        obs_block = self.slab[self.n:]
        self.e.step_device(self.act.data_ptr(), obs_block.data_ptr(), self.rew.data_ptr(), self.done.data_ptr(), obs_ld=self.ld)
        self.e.sync()
        s = self.slab.cpu().numpy()
        rec = s[self.n:2 * self.n] if self.record == 1 else s[:self.n]
        assert np.all(s[2 * self.n:] == -7.0), "canary rows past the batch were written"
        assert np.all(self.rew.cpu().numpy()[self.n:] == 0) and np.all(self.done.cpu().numpy()[self.n:] == 0)
        assert np.all(rec[:, self.w + 14:] == -7.0)
        if self.record == 2:
            assert np.all(s[:self.n, :self.w] == -7.0)
        else:
            assert np.all(s[:self.n] == -7.0), "record mode 1 wrote outside the observation's row block"
        obs = s[self.n:2 * self.n, :self.w]
        return obs, self.rew.cpu().numpy()[:self.n].copy(), self.done.cpu().numpy()[:self.n].copy(), rec[:, self.w:self.w + 14]


def step_io(e, actions, io, slab=None):
    """(obs, reward, done, record columns or None) of one step through an I/O path"""
    if io == "host":
        return e.step(actions) + (None,)
    if io == "pinned":
        a, o, r, d = e.pinned_io()
        a[...] = actions
        e.step_pinned(a, o, r, d)
        return o.copy(), r.copy(), d.copy(), None
    return slab.step(actions)


def readback(e):
    from lifelike_agility_and_play_b200 import _capi as capi
    return {k: e.get(f) for k, f in (("state", capi.F_STATE), ("kin", capi.F_KIN_STATE), ("time", capi.F_TIME), ("clip", capi.F_CLIP),
                                     ("episode", capi.F_EPISODE_ID), ("ob_id", capi.F_OB_ID), ("reward_sum", capi.F_REWARD_SUM),
                                     ("avg", capi.F_AVG_REWARD), ("prob", capi.F_SAMPLE_PROB), ("obs", capi.F_OBS))} | {"counters": e.counters()}


def _sign_fix(q, ref):
    return q * np.where(np.sum(q * ref, 1) < 0, -1.0, 1.0)[:, None]


def _ratio(got, ref, S, kappa, what, rows=None):
    """largest |got - ref| / S beyond the 2^-23 |ref| allowance; asserts the bar kappa S + 2^-23 |ref| element by element"""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    if rows is not None:
        got, ref, S = got[rows], ref[rows], S[rows]
    nan = np.isnan(ref)                    # NaN actions travel into the observation: NaN exactly where the statement has one
    assert np.array_equal(np.isnan(got), nan), (what, np.argwhere(np.isnan(got) != nan)[:6])
    got, ref, S = np.where(nan, 0.0, got), np.where(nan, 0.0, ref), np.where(nan, 0.0, S)
    err = np.abs(got - ref) - U * np.abs(ref)
    bad = err > kappa * S
    assert not bad.any(), (what, [(tuple(int(x) for x in ix), got[tuple(ix)], ref[tuple(ix)], S[tuple(ix)]) for ix in np.argwhere(bad)[:6]])
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err > 0, err / np.maximum(S, 1e-300), 0.0)
    return float(r.max()) if r.size else 0.0


def ulps(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a.view(np.int64) - b.view(np.int64))


def run_case(lib, k, io="host", kappa=KAPPA, oracle=False):
    """Run batch k through `lib` (CUDA engine or oracle) and compare every output with the statement.  Engine A (auto_reset 0)
    takes two steps, the second with the highest finisher of every clip taken back (the winner ping-pong buffers); engine B
    (auto_reset 1) takes the first step again and draws.  Returns the largest error / S ratios.

    oracle=True: the oracle keeps reward_sum in fp64 (the reference's python float), the engine in fp32.  Its rewards are held to
    5e-7 + 4 S, its reward sums and table to 1e-6 relative, and the draws of the designed-edge envs (which lie closer to an edge than that
    difference moves it) are not compared."""
    ctx, before, cats, designed = case(k)
    n = ctx["n"]
    ratios = {}
    A, B = make(lib, ctx, 0), make(lib, ctx, 1)
    try:
        slabs = [Slab(x, int(io[-1])) if io.startswith("device") else None for x in (A, B)]
        c0A, c0B = A.counters(), B.counters()
        set_before(A, before); set_before(B, before)
        oA, rA, dA, recA = step_io(A, before["actions"], io, slabs[0])
        fa = readback(A)
        oB, rB, dB, recB = step_io(B, before["actions"], io, slabs[1])
        fb = readback(B)
        # ---- engine A: the step statement on the state read back
        st = fa["state"].astype(np.float64)
        ref, S = sensitivity(ctx, before, st)
        assert decisive(ref).all(), [(int(i), cats[i]) for i in np.nonzero(~decisive(ref))[0][:6]]
        assert reaches(ctx, before, ref, cats).all()
        done = ref["done"]
        assert np.array_equal(dA.astype(bool), done), [(int(i), cats[i], int(dA[i])) for i in np.nonzero(dA.astype(bool) != done)[0][:8]]
        assert np.array_equal(fa["time"], ref["time"]) and np.array_equal(fa["ob_id"], ref["ob_id"])
        assert np.array_equal(fa["clip"], before["clip"]) and np.array_equal(fa["episode"], before["episode"])
        assert int(fa["counters"][1] - c0A[1]) == int(done.sum()) and int(fa["counters"][0] - c0A[0]) == n
        if oracle:
            # (the oracle interpolates the fp64 frames: 4 S covers the fp32 storage of the engine's)
            assert np.all(np.abs(rA - ref["reward64"]) <= 5e-7 + 4 * S["reward64"]), np.abs(rA - ref["reward64"]).max()
        else:
            ratios["reward"] = _ratio(rA, ref["reward64"], S["reward64"], kappa, "reward")
        # reward_sum: fp32 sum of the value set and the reward; within one fp32 rounding of the statement's sum on the engine's reward
        rs_own = (before["reward_sum"] + rA).astype(np.float32)
        assert oracle or np.array_equal(fa["reward_sum"], rs_own)
        ratios["reward_sum"] = _ratio(fa["reward_sum"], before["reward_sum"].astype(np.float64) + ref["reward64"], S["reward64"] + np.spacing(rs_own),
                                      kappa, "reward_sum")
        kin = fa["kin"].astype(np.float64); kin[:, 3:7] = _sign_fix(kin[:, 3:7], ref["kin"][:, 3:7])
        ratios["kin"] = _ratio(kin, ref["kin"], S["kin"], kappa, "F_KIN_STATE")
        # a `bad` env's new prop and future blocks are made of its NaN state; its reward (0), done, clock and copied blocks are checked
        ratios["obs"] = _ratio(oA, ref["obs"], S["obs"], kappa, "obs", rows=~ref["bad"])
        assert np.all(rA[ref["bad"]] == 0) and np.all(dA[ref["bad"]] == 1)
        assert np.array_equal(oA, fa["obs"], equal_nan=True)
        assert np.array_equal(oA[:, 0:66], before["obs"][:, 33:99]) and np.array_equal(oA[:, 99:123], before["obs"][:, 111:135])
        assert np.array_equal(oA[:, 123:135], before["actions"], equal_nan=True)
        # ---- the table, from the reward sums the engine kept (exact on both sides)
        avg, p, cdf, win = table(ctx, done, before["clip"], fa["reward_sum"], before["avg"])
        if oracle:
            assert np.allclose(fa["avg"], avg, rtol=1e-6, atol=0) and np.allclose(fa["prob"], p, rtol=1e-6, atol=0)
        else:
            assert ulps(fa["avg"], avg).max() <= 1, (fa["avg"], avg)
            assert ulps(fa["prob"], p).max() <= 8, ulps(fa["prob"], p).max()
            ratios["prob_ulps"] = int(ulps(fa["prob"], p).max())
        # ---- engine B: same step, then the auto-reset draws
        assert np.array_equal(rB, rA) and np.array_equal(dB, dA)
        assert np.array_equal(fb["avg"], fa["avg"]) and np.array_equal(fb["prob"], fa["prob"])
        keep = ~done
        for key in ("state", "kin", "time", "clip", "episode", "ob_id", "reward_sum"):
            assert np.array_equal(fb[key][keep], fa[key][keep]), key
        assert np.array_equal(oB[keep], oA[keep], equal_nan=True)
        assert int(fb["counters"][1] - c0B[1]) == int(done.sum()) and int(fb["counters"][0] - c0B[0]) == n
        fin = np.nonzero(done)[0]
        if len(fin):
            clip, t0, fid, frac, u1 = draw(ctx, cdf, ctx["gid0"] + fin, before["episode"][fin])
            for e_, (j, side) in designed.items():
                r = int(np.nonzero(fin == e_)[0][0])
                assert clip[r] == (j if side > 0 else j + 1) and 1e-9 <= abs(cdf[j] - u1[r]) <= 1e-6, (e_, j, side, clip[r], cdf[j] - u1[r])
            cmp = ~np.isin(fin, list(designed)) if oracle else np.ones(len(fin), bool)
            fin, clip, t0, fid, frac = fin[cmp], clip[cmp], t0[cmp], fid[cmp], frac[cmp]
            assert np.array_equal(fb["clip"][fin], clip), [(int(fin[i]), int(fb["clip"][fin][i]), int(clip[i])) for i in np.nonzero(fb["clip"][fin] != clip)[0][:6]]
            assert np.array_equal(fb["time"][fin], t0) and np.array_equal(fb["episode"][fin], before["episode"][fin] + 1)
            assert np.all(fb["ob_id"][fin] == 0) and np.all(fb["reward_sum"][fin] == 0)
            rst, robs, Ss, So = reset_sensitivity(ctx, clip, fid, frac)
            got = fb["state"][fin].astype(np.float64); got[:, 3:7] = _sign_fix(got[:, 3:7], rst[:, 3:7])
            ratios["reset_state"] = _ratio(got, rst, Ss, kappa, "reset state")
            got = fb["kin"][fin].astype(np.float64); got[:, 3:7] = _sign_fix(got[:, 3:7], rst[:, 3:7])
            ratios["reset_kin"] = _ratio(got, rst, Ss, kappa, "reset F_KIN_STATE")
            ratios["reset_obs"] = _ratio(oB[fin], robs, So, kappa, "reset obs")
            assert np.array_equal(oB[fin], fb["obs"][fin])
            assert np.all(oB[fin][:, 99:135] == 0) and np.array_equal(oB[fin][:, 0:33], oB[fin][:, 66:99])
        # ---- record columns: the finishing step's action, reward and done, also for envs that were reset in the same call
        for rec, rw, dn in ((recA, rA, dA), (recB, rB, dB)):
            if rec is not None:
                assert np.array_equal(rec[:, :12], before["actions"], equal_nan=True) and np.array_equal(rec[:, 12], rw)
                assert np.array_equal(rec[:, 13], dn.astype(np.float32))
        # ---- engine A, second step: the highest finisher of every clip is taken back, so a lower one must win the slot
        before2 = dict(before)
        st2 = before["state"].copy()
        back = [int(w) for w in win if w >= 0 and cats[w] == "finish"]
        for w in back:
            st2[w, 0] -= np.float32(2.0)
        before2["state"] = st2
        set_before(A, before2, table_too=False)
        o2, r2, d2, _ = step_io(A, before["actions"], io, slabs[0])
        f2 = readback(A)
        ref2 = step_statement(ctx, before2, f2["state"].astype(np.float64))
        assert np.array_equal(d2.astype(bool), ref2["done"])
        assert int(f2["counters"][1] - c0A[1]) == int(done.sum() + ref2["done"].sum()) and int(f2["counters"][0] - c0A[0]) == 2 * n
        assert not any(ref2["done"][w] for w in back)
        avg2, p2, _, win2 = table(ctx, ref2["done"], before["clip"], f2["reward_sum"], fa["avg"])
        if oracle:
            assert np.allclose(f2["avg"], avg2, rtol=1e-6, atol=0)
        else:
            assert ulps(f2["avg"], avg2).max() <= 1 and ulps(f2["prob"], p2).max() <= 8
        ratios["n_done"] = int(done.sum()); ratios["n_designed_edges"] = len(designed); ratios["n_taken_back"] = len(back)
        return ratios
    finally:
        A.close(); B.close()
