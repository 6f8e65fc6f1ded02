"""fp64 statement of the SEPMC episode logic (ChaseTagGameEnv, the empty arena) and designed pairs on which every branch of it is
decisive (host only, numpy float64).

Robots 2p and 2p + 1 are the two agents of pair p.  Like tests/epmc_episode_cases.py the statement is computed from the fields set
before the step (F_STATE, F_AUX, F_OBS, F_EPISODE_ID) and the state read back after it, so it states no dynamics: the batches run
with the physics and the damping off, zero angular and joint velocities and non-zero base linear velocities (pure translation).

  contacts  of the last sub-step, on the pose before it (CTG:426-456): post - v sim_dt (the start pose with one sub-step).  Flag
            touch: a hip or knee-wheel proxy of the robot within contact_breaking of the 0.1 x 0.1 x 0.5 flag box.  Tag: a hip or
            wheel proxy of ROBOT 0 within contact_breaking of any of robot 1's 22 proxies (feet, wheels, hips, the two handles, the
            eight trunk corners of radius 0).  LLQ_AUX_FLAG_TOUCH is the robot's touch
  visible   perception_cases.visible on the post poses, with the flag where it stood during the step (CTG:472-493)
  switch    when the robot without the flag touches it (CTG:573-581): with_flag swaps, switch_flag = 1, the flag is redrawn from
            stream 4, draw `flag_draws`, keyed by the pair's global id (robot 0's) and robot 0's episode: (-2 + 4 u0, -2 + 4 u1);
            flag_draws += 1 on both robots
  stats     spd = |v_xy| in fp32; total_spd and max_spd (strict >) in double; counter += 1
  done      shared by the pair: robot 0's fall (|left_z| > 1/sqrt 2 or R22 < 0.5), counter >= max_steps, tag, or `bad` (a
            non-finite post state) in either robot
  reward    (CTG:640-652, 412-419) +-1 on a switch and +-1 on a tag that ends the step, the sign from with_flag after the switch
            (+ for the holder); 0 on both robots of a `bad` step.  reward_sum in fp32
  push      the pair's schedule per sub-step (PR:56-87): count += 1; when count > 0, one draw on `count % interval == 0` (then
            count = 0), and inside the window robot r takes draw push_draws - 1 + r, then push_draws += 2.  Stream 2, keyed as
            the flag; the force (h cos 2 pi u0, h sin 2 pi u0, v) in fp32
  obs       prop / action history shift, the new prop, the action, then perception_cases.sepmc_row: the 778 rays, percept_vec,
            the opponent blocks masked by visibility, flag_info at the flag of the step (before a switch), with_flag after the
            switch as [own, partner], control_spd
  reset     (CTG:261-304, 204-230) stream 1, draws 0-2, keyed by the pair's id and robot 0's episode before the reset:
            fix_spd = 0.5 + 2.5 u0[0] (fp32), with_flag = floor(2 u0[1]) for robot 0, friction, both start positions, the pair's
            yaw accumulator fmod'ed twice (robot 0, then robot 1; read from robot 0), the flag (u2[1], u2[2]); push draw #0 taken
            (force 0, push_draws = 1); the init state yawed at z = 0.5; then the stale-touch switch: reset() runs _prepare_drill,
            which reads the previous episode's last LLQ_AUX_FLAG_TOUCH (a switch draws stream 4 index 0, flag_draws = 1).  Both
            robots get robot 0's episode + 1.  A masked reset of either robot resets the pair

Error model and bars as in tests/epmc_episode_cases.py (policy_cases.ErrorModel, S per output; the GPU bar KAPPA S + 2^-23 |ref|).
The perception columns (obs 135-964: rays and the SEPMC vectors) keep the perception pin's bar 1e-5 max(1, |ref|) + 4 S.

Decisiveness.  On the pose before the last sub-step every hip / wheel flag gap and every robot-0-body / robot-1-proxy gap clears
contact_breaking by DELTA (PUSH_CLEAR on pushed pairs, whose motion is not stated); robot 0's fall quantities clear their thresholds
by DELTA; every visibility segment clears or hits the flag by DELTA_VIS and the walls by DELTA; every ray of the post poses is
decisive; spd clears max_spd by DELTA.  A robot with a NaN joint angle stays 1 m from the flag and its partner: the engines
integrate it differently (the oracle stops the pair, the step kernel clamps its velocities to the bound), and its post state is
not stated beyond `bad`.
"""
import numpy as np

import episode_cases as ec
import epmc_episode_cases as xc
import perception_cases as pcs
from lifelike_agility_and_play_b200 import _capi as capi
from epmc_episode_cases import f32
from policy_cases import REF

# GPU bar factor, as for the PMC and EPMC pins
KAPPA = xc.KAPPA
DELTA = 1e-4
PUSH_CLEAR = 5e-2
SEED = 20261019
MAX_STEPS = 23
FRICTION = (0.4, 3.0)
PUSH_H, PUSH_V = (0.0, 4.73), (0.0, 0.97)       # small: a pushed robot (its motion is not stated) stays near its pose
PUSH_SCHEDULE = dict(push_start_count=-4, push_interval_steps=7, push_duration_steps=3)
SIM_DT = 1.0 / 500.0
BREAKING = ec.BREAKING
LIMIT = ec.LIMIT
KIND = pcs.PROXIES[:, 5].astype(int)
RAD = pcs.PROXIES[:, 4]
BODY = np.flatnonzero((KIND == 1) | (KIND == 2))         # hips and knee wheels: the "body" of CTG:427
KIND_NAMES = ("foot", "wheel", "hip", "corner", "handle")

# batches: (n robots, sub-steps, pushes on, global_env_offset).  A step CTA holds 16 envs and a tail warp 8.
CASES = [
    (2, 10, 1, 0),
    (8, 1, 1, 0),
    (10, 10, 0, 2 ** 32 - 4),
    (16, 1, 0, 0),
    (18, 10, 1, 2 ** 32 - 5),
    (32, 1, 1, 2 ** 32 - 4),
    (34, 10, 1, 2 ** 32 - 5),
    (162, 10, 1, 2 ** 32 - 5),
]
# The largest batch has 162 robots rather than thousands: the pairs are designed one by one on the host (about 0.3 s each with the
# retries), and 162 = 10 x 16 + 2 already leaves a padded last CTA and a part-filled tail warp.

TOUCH_CATS = ("touch_hip_in", "touch_hip_out", "touch_wheel_in", "touch_wheel_out", "touch_foot", "touch_holder", "touch_both")
MOVE_CATS = ("touch_pre_only", "touch_post_only")           # 10 sub-steps: in on the pose before the last one, out after it
TAG_CATS = tuple("tag_%s_%s" % (k, s) for k in KIND_NAMES for s in ("in", "out")) + ("tag_reverse", "tag_switch", "tag_timeup",
                                                                                       "tag_hold0", "tag_hold1")
TERM_CATS = ("left_pos_in", "left_pos_out", "left_neg_in", "left_neg_out", "r22_in", "r22_out", "fall1", "timeup_at", "timeup_before")
BAD_CATS = ("nan_action0", "nan_action1", "nan_joint0", "nan_joint1", "nan1_switch")      # nan1_switch: the oracle's bad reward
ID_CATS = ("ids_switch", "ids_push")                    # unequal episode ids in a pair: the first pairs of the batches of 17 pairs or more
VIS_CATS = ("vis_root", "vis_head", "vis_none", "vis_behind", "vis_stacked")
SPD_CATS = ("max_up", "max_keep")
PUSH_CATS = ("push_cross", "push_draw", "push_last", "push_off_first")
RESET_CATS = ("stale_switch", "stale_holder", "yaw0_below", "yaw0_above", "yaw1_below", "yaw1_above")
COMMON = TOUCH_CATS + TAG_CATS + TERM_CATS + BAD_CATS + VIS_CATS + SPD_CATS + RESET_CATS + ("plain",)


def cats_of(substeps, push):
    return COMMON + (MOVE_CATS if substeps > 1 else ()) + (PUSH_CATS if push else ())


def id_cats(push):
    return ID_CATS if push else ID_CATS[:1]


def rep(x):
    """a per-pair array onto both robots"""
    return np.repeat(np.asarray(x), 2, axis=0)


# ------------------------------------------------------------------------------------------------------------ geometry
def flag_gaps(p, fx, fy):
    """[22] distance of each proxy sphere to the flag box minus contact_breaking"""
    box = pcs.arena_boxes(fx, fy)[5]
    with np.errstate(invalid="ignore"):
        return np.linalg.norm(p - np.clip(p, box[:3], box[3:]), axis=1) - RAD - BREAKING


def tag_gaps(p0, p1):
    """[8, 22] robot 0's body proxies against robot 1's proxies, minus contact_breaking"""
    return np.linalg.norm(p0[BODY][:, None] - p1[None], axis=2) - RAD[BODY][:, None] - RAD[None] - BREAKING


def pair_geometry(sa, sb, fx, fy):
    """contact quantities of a pair at poses sa, sb (flag at fx, fy)"""
    pa, pb = pcs.proxy_points(sa), pcs.proxy_points(sb)
    ga, gb = flag_gaps(pa, fx, fy), flag_gaps(pb, fx, fy)
    tg = tag_gaps(pa, pb)
    rev = np.linalg.norm(pb[BODY][:, None] - pa[None], axis=2) - RAD[BODY][:, None] - RAD[None] - BREAKING
    with np.errstate(invalid="ignore"):
        return dict(flag=np.stack([ga, gb]), touch=np.array([(ga[BODY] < 0).any(), (gb[BODY] < 0).any()]), tag_gap=tg,
                    tag=bool((tg < 0).any()), rev=rev)


def pre_pose(ctx, before, post):
    """the pose before the last sub-step: the start pose with one sub-step, else post - v sim_dt (pure translation)"""
    if ctx["substeps"] == 1:
        return before["state"].astype(np.float64)
    pre = post.copy()
    pre[:, 0:3] -= post[:, 7:10] * SIM_DT
    return pre


def geometry(ctx, before, post):
    """contacts on the pose before the last sub-step, the same quantities on the post pose, visibility on the post pose"""
    n = len(post)
    pre = pre_pose(ctx, before, post)
    fx, fy = before["aux"][0::2, capi.AUX_FLAG_X], before["aux"][0::2, capi.AUX_FLAG_Y]
    G, Gp, vis, cv, vis_ok, root = [], [], np.zeros(n, bool), np.zeros(n), np.ones(n // 2, bool), np.zeros(n // 2, bool)
    for p in range(n // 2):
        a, b = 2 * p, 2 * p + 1
        G.append(pair_geometry(pre[a], pre[b], fx[p], fy[p]))
        Gp.append(pair_geometry(post[a], post[b], fx[p], fy[p]))
        if np.isfinite(post[a]).all() and np.isfinite(post[b]).all():
            bx = pcs.arena_boxes(fx[p], fy[p])
            vis[a:b + 1] = pcs.visible(post[a], post[b], bx)
            o, e = pcs.vis_segments(post[a], post[b])
            vis_ok[p] = pcs.decisive(o, e, bx, np.array([DELTA] * 5 + [pcs.DELTA_VIS])).all()
            root[p] = pcs.cast(o[:1], e[:1], bx)[0][0] < 0
            for i, (s, t) in enumerate(((post[a], post[b]), (post[b], post[a]))):
                R = pcs.rot(s[3:7])
                yaw = np.arctan2(R[1, 0], R[0, 0])
                d = t[0:3] - s[0:3]
                with np.errstate(invalid="ignore"):
                    cv[a + i] = (np.cos(yaw) * d[0] + np.sin(yaw) * d[1]) / np.hypot(d[0], d[1])
    touch = np.concatenate([g["touch"] for g in G])
    return dict(pre=G, post=Gp, touch=touch, tag=np.array([g["tag"] for g in G]), vis=vis, cv=cv, vis_ok=vis_ok, root=root)


# ------------------------------------------------------------------------------------------------------------ the statement
def pair_push(ctx, gidp, ep0, count, draws, force):
    """(count, draws [P], force [n, 3], sub-steps on [P], (count, on, fired) per sub-step) of the pairs' push schedule"""
    count, draws, force = count.copy(), draws.copy(), force.copy()
    on = np.zeros(len(count), np.int64)
    trace = []
    if not ctx["push"]:
        return count, draws, force, on, trace
    for _ in range(ctx["substeps"]):
        count += 1
        pos = count > 0
        fire = pos & (count % ctx["interval"] == 0)
        draws[fire] += 1
        count[fire] = 0
        o = pos & (count < ctx["duration"])
        idx = np.flatnonzero(o)
        for r in (0, 1):
            if len(idx):
                force[2 * idx + r] = xc.push_force(ctx, gidp[idx], ep0[idx], draws[idx] - 1 + r)
        draws[o] += 2
        on += o
        trace.append((count.copy(), o, fire))
    return count, draws, force, on, trace


def step_statement(ctx, before, st, geo, em=REF):
    """the outputs of one step from the fields set before it (`before`), the post-step state `st` read back and its contact and
    visibility geometry `geo` (decisive: computed once, on the unperturbed state)"""
    n = len(st)
    P = n // 2
    aux = before["aux"]
    gidp = ctx["gid0"] + 2 * np.arange(P)
    ep0 = before["episode"][0::2] - 1
    st = em.rel(np.asarray(st, np.float64))
    touch, tag = geo["touch"], geo["tag"]
    wf = aux[:, capi.AUX_WITH_FLAG].astype(np.int64)
    fd = aux[0::2, capi.AUX_FLAG_DRAWS].astype(np.int64)
    sw = ((wf[0::2] == 1) & touch[1::2]) | ((wf[1::2] == 1) & touch[0::2])
    fx, fy = aux[0::2, capi.AUX_FLAG_X].copy(), aux[0::2, capi.AUX_FLAG_Y].copy()
    nfx, nfy = fx.copy(), fy.copy()
    if sw.any():
        u = xc.stream_uniforms(ctx["seed"], gidp[sw], ep0[sw], 4, fd[sw])
        nfx[sw], nfy[sw] = -2.0 + 4.0 * u[0], -2.0 + 4.0 * u[1]
    nw = np.where(rep(sw), 1 - wf, wf)
    with np.errstate(invalid="ignore"):
        spd = em.rel(np.hypot(st[:, 7], st[:, 8]))
        total = aux[:, capi.AUX_TOTAL_SPD] + spd
        mx = np.where(spd > aux[:, capi.AUX_MAX_SPD], spd, aux[:, capi.AUX_MAX_SPD])
        counter = aux[:, capi.AUX_COUNTER].astype(np.int64) + 1
        left_z, r22 = ec.tilt(st)
        fall = (np.abs(left_z) > LIMIT) | (r22 < 0.5)
    bad_r = ~np.isfinite(st).all(1)
    bad = bad_r[0::2] | bad_r[1::2]
    timeup = counter[0::2] >= ctx["max_steps"]
    done = fall[0::2] | timeup | tag | bad
    s0 = np.where(nw[0::2] == 1, 1.0, -1.0)
    r0 = np.where(bad, 0.0, s0 * (sw.astype(np.float64) + (done & tag)))
    rew = np.stack([r0, -r0], 1).reshape(n)
    pc, pd, pf, pon, _ = pair_push(ctx, gidp, ep0, aux[0::2, capi.AUX_PUSH_COUNT].astype(np.int64),
                                   aux[0::2, capi.AUX_PUSH_DRAWS].astype(np.int64), aux[:, capi.AUX_PUSH_F:capi.AUX_PUSH_F + 3])
    new = aux.copy()
    new[:, capi.AUX_COUNTER] = counter; new[:, capi.AUX_WITH_FLAG] = nw
    new[:, capi.AUX_FLAG_X] = rep(nfx); new[:, capi.AUX_FLAG_Y] = rep(nfy)
    new[:, capi.AUX_OPPO_VISIBLE] = geo["vis"]; new[:, capi.AUX_SWITCH_FLAG] = rep(sw)
    new[:, capi.AUX_TOTAL_SPD] = total; new[:, capi.AUX_MAX_SPD] = mx
    new[:, capi.AUX_PUSH_COUNT] = rep(pc); new[:, capi.AUX_PUSH_DRAWS] = rep(pd); new[:, capi.AUX_PUSH_F:capi.AUX_PUSH_F + 3] = pf
    new[:, capi.AUX_FLAG_DRAWS] = rep(fd + sw); new[:, capi.AUX_FLAG_TOUCH] = touch
    obs = np.concatenate([before["obs"][:, 33:99], ec.prop(st, em), before["obs"][:, 111:135], before["actions"]], 1)
    rs = (before["reward_sum"].astype(np.float32) + rew.astype(np.float32)).astype(np.float32)
    foot = ec.foot_positions(st).reshape(n, 12)
    return dict(sw=sw, counter=counter, left_z=left_z, r22=r22, fall=fall, timeup=timeup, bad=bad, done=done, spd=spd, reward64=rew,
                reward=em.add(rew, np.abs(rew)), reward_sum=rs, aux=em.add(new, np.abs(new)), obs=em.add(obs, np.abs(obs)),
                foot=em.add(foot, np.abs(foot)), push_on=pon, flag_step=(fx, fy), with_flag=nw, max_before=aux[:, capi.AUX_MAX_SPD])


def sensitivity(ctx, before, st, geo):
    return xc._sens(lambda em: step_statement(ctx, before, st, geo, em), ("reward", "aux", "obs", "foot"))


_ROWS = {}


def perception(st, with_flag, fx, fy, ctrl, vis):
    """(values [n, 830], S) of obs 135-964 of the pairs at states st: with_flag [n], the flag of each pair [P], control_spd [n],
    oppo_visible [n]"""
    V, S = [], []
    for i in range(len(st)):
        j = i ^ 1
        key = (st[i].tobytes(), st[j].tobytes(), int(with_flag[i]), int(with_flag[j]), float(fx[i // 2]), float(fy[i // 2]),
               float(ctrl[i]), bool(vis[i]))
        if key not in _ROWS:
            a = np.array([0.0, with_flag[i], fx[i // 2], fy[i // 2], ctrl[i]])
            b = np.array([0.0, with_flag[j], fx[i // 2], fy[i // 2], ctrl[j]])
            _ROWS[key] = pcs.sepmc_row(st[i], st[j], a, b, vis[i])
        v, s = _ROWS[key]
        V.append(v); S.append(s)
    return np.array(V), np.array(S)


def reset_statement(ctx, gidp, ep0, acc, touch, em=REF):
    """(state [n, 37], aux [n, 18], observation row 0-134 [n, 135], the perception inputs) of resets of pairs gidp whose robot 0
    had episode id ep0 and yaw accumulator acc; touch [n] = LLQ_AUX_FLAG_TOUCH before the reset"""
    P = len(gidp)
    n = 2 * P
    u0, u1, u2 = (xc.stream_uniforms(ctx["seed"], gidp, ep0, 1, k) for k in range(3))
    fix = f32(0.5 + 2.5 * u0[0])
    wflag = np.floor(2.0 * u0[1]).astype(np.int64)
    lo, hi = f32(ctx["friction"][0]), f32(ctx["friction"][1])
    mu = lo + u0[2] * (hi - lo)
    px = np.stack([-2.0 + 4.0 * u0[3], -2.0 + 4.0 * u1[1]], 1).reshape(n)
    py = np.stack([-2.0 + 4.0 * u1[0], -2.0 + 4.0 * u1[2]], 1).reshape(n)
    ya = np.fmod(acc + 360.0 * u1[3], 360.0)
    yb = np.fmod(ya + 360.0 * u2[0], 360.0)
    yaw = np.stack([ya, yb], 1).reshape(n)
    fx, fy = -2.0 + 4.0 * u2[1], -2.0 + 4.0 * u2[2]
    wf = np.stack([wflag, 1 - wflag], 1).reshape(n)
    t = np.asarray(touch, bool)
    sw = ((wf[0::2] == 1) & t[1::2]) | ((wf[1::2] == 1) & t[0::2])
    nfx, nfy = fx.copy(), fy.copy()
    if sw.any():
        u = xc.stream_uniforms(ctx["seed"], gidp[sw], ep0[sw], 4, np.zeros(int(sw.sum()), np.int64))
        nfx[sw], nfy[sw] = -2.0 + 4.0 * u[0], -2.0 + 4.0 * u[1]
    nw = np.where(rep(sw), 1 - wf, wf)
    I0 = f32(ctx["init_state"])
    half = 0.5 * yaw * (np.pi / 180.0)
    q0 = I0[3:7] / np.linalg.norm(I0[3:7])
    qn = xc.qmul(np.repeat(q0[None], n, 0), np.stack([np.zeros(n), np.zeros(n), f32(np.sin(half)), f32(np.cos(half))], 1))
    st = np.repeat(I0[None], n, 0)
    st[:, 0], st[:, 1], st[:, 2] = px, py, 0.5
    st[:, 3:7] = em.add(qn, 1.0)
    new = np.zeros((n, capi.AUX_DIM))
    new[:, capi.AUX_WITH_FLAG] = nw; new[:, capi.AUX_FLAG_X] = rep(nfx); new[:, capi.AUX_FLAG_Y] = rep(nfy)
    new[:, capi.AUX_CONTROL_SPD] = rep(fix); new[:, capi.AUX_SWITCH_FLAG] = rep(sw)
    new[:, capi.AUX_PUSH_COUNT] = ctx["start_count"]; new[:, capi.AUX_FOOT_FRICTION] = rep(mu)
    new[:, capi.AUX_PUSH_DRAWS] = 1 if ctx["push"] else 0; new[:, capi.AUX_FLAG_DRAWS] = rep(sw)
    new[:, capi.AUX_YAW_ACCUM_DEG] = rep(yb); new[:, capi.AUX_FLAG_TOUCH] = t
    p = ec.prop(st, em)
    obs = np.concatenate([p, p, p, np.zeros((n, 36))], 1)
    foot = ec.foot_positions(st).reshape(n, 12)
    return dict(state=em.add(st, np.abs(st)), aux=em.add(new, np.abs(new)), obs=em.add(obs, np.abs(obs)), foot=em.add(foot, np.abs(foot)),
                sw=sw, flag_reset=(fx, fy), yaw_sums=(acc + 360.0 * u1[3], ya + 360.0 * u2[0]), wflag=wflag)


def reset_sensitivity(ctx, gidp, ep0, acc, touch):
    return xc._sens(lambda em: reset_statement(ctx, gidp, ep0, acc, touch, em), ("state", "aux", "obs", "foot"), seed=SEED + 100)


# ------------------------------------------------------------------------------------------------------------ designed batches
def init_state():
    from test_golden_sepmc import GOLD
    return np.load(GOLD)["init_state"].astype(np.float64)


def context(case):
    n, substeps, push, gid0 = case[:4]
    return dict(n=n, substeps=substeps, push=push, gid0=gid0, seed=SEED + n, max_steps=MAX_STEPS, friction=FRICTION, push_h=PUSH_H,
                push_v=PUSH_V, start_count=PUSH_SCHEDULE["push_start_count"], interval=PUSH_SCHEDULE["push_interval_steps"],
                duration=PUSH_SCHEDULE["push_duration_steps"], init_state=init_state(), T=substeps * SIM_DT)


def engine_config(ctx, auto_reset):
    from test_golden_sepmc import SEPMC_CFG
    cfg = dict(SEPMC_CFG)
    cfg.update(ec.PHYSICS_OFF, lin_damping=0.0, ang_damping=0.0, substeps=ctx["substeps"], push_enabled=ctx["push"], contact_breaking=BREAKING,
               global_env_offset=ctx["gid0"], seed=ctx["seed"], auto_reset=auto_reset, max_steps=ctx["max_steps"], friction_lo=FRICTION[0],
               friction_hi=FRICTION[1], push_h_lo=PUSH_H[0], push_h_hi=PUSH_H[1], push_v_lo=PUSH_V[0], push_v_hi=PUSH_V[1], **PUSH_SCHEDULE)
    return cfg


def make(lib, ctx, auto_reset):
    e = capi.VecEngine(lib, ctx["n"], ec._blob(), None, **engine_config(ctx, auto_reset))
    e.set_init_state(ctx["init_state"])
    e.reset()
    return e


def _robot(I0, x, y, yaw, z=None):
    s = f32(I0).copy()
    s[7:13] = 0.0; s[25:37] = 0.0
    s[0:3] = (x, y, I0[2] if z is None else z)
    s[3:7] = xc._yaw_quat(yaw, I0[3:7])
    s[3:7] /= np.linalg.norm(s[3:7])
    return s


def _proxy(s, i):
    return pcs.proxy_points(s)[i]


def _pick(rng, kind):
    return int(rng.choice(np.flatnonzero(KIND == kind)))


def _flag_at(rng, s, i, g):
    """a flag whose side face lies g + contact_breaking beyond proxy i of robot s, away from the robot"""
    p = _proxy(s, i)
    d = p[0:2] - s[0:2]
    a = int(np.argmax(np.abs(d)))
    c = p[0:2].copy()
    c[a] += np.sign(d[a]) * (0.05 + RAD[i] + BREAKING + g)
    c[1 - a] += rng.uniform(-0.03, 0.03)
    return c


def _place_against(rng, s_fixed, j, i, g, I0, yaw=None):
    """robot state whose proxy i sits g + contact_breaking outside proxy j of s_fixed, away from s_fixed's base"""
    p = _proxy(s_fixed, j)
    d = p - s_fixed[0:3]
    d /= np.linalg.norm(d)
    tgt = p + d * (RAD[i] + RAD[j] + BREAKING + g)
    s = _robot(I0, 0.0, 0.0, rng.uniform(-np.pi, np.pi) if yaw is None else yaw)
    s[0:3] += tgt - _proxy(s, i)
    return s


def _side(rng):
    return rng.uniform(2, 8) * DELTA


def _far_flag(rng, states, gap):
    for _ in range(200):
        F = rng.uniform(-2.0, 2.0, 2)
        if pcs._flag_clear(states, *F, gap=gap):
            return F
    raise RuntimeError("no clear flag position")


def _design(ctx, cat, rng, I0, ep):
    """(robot 0, robot 1 on the pose before the last sub-step, flag xy, extras: velocities, with_flag, counter, push count, NaN)
    of a pair in category cat whose robot 0 has episode id ep"""
    sub, ms = ctx["substeps"], ctx["max_steps"]
    x = dict(wf0=int(rng.integers(2)), counter=int(rng.integers(0, ms - 3)), v=[rng.uniform(0, 0.6) * np.array([np.cos(h), np.sin(h)])
                                                                               for h in rng.uniform(-np.pi, np.pi, 2)], push_count=-1000, nan=None)
    a = _robot(I0, *rng.uniform(-1.6, 1.6, 2), rng.uniform(-np.pi, np.pi))
    h = rng.uniform(-np.pi, np.pi)
    L = rng.uniform(0.8, 1.8)
    b = _robot(I0, np.clip(a[0] + L * np.cos(h), -2.1, 2.1), np.clip(a[1] + L * np.sin(h), -2.1, 2.1), rng.uniform(-np.pi, np.pi))
    F = None
    kind = {"hip": 2, "wheel": 1, "foot": 0}
    if cat in TOUCH_CATS + MOVE_CATS or cat in ("nan1_switch", "stale_switch", "stale_holder", "ids_switch"):
        r = int(rng.integers(2))
        k = cat.split("_")[1] if cat.startswith("touch_") and cat.split("_")[1] in kind else str(rng.choice(["hip", "wheel"]))
        g = -_side(rng) if cat.endswith("_in") or cat in ("touch_foot", "touch_holder", "touch_both", "touch_pre_only", "nan1_switch",
                                                         "stale_switch", "stale_holder", "ids_switch") else _side(rng)
        if cat == "nan1_switch":
            r = 0
        s = (a, b)[r]
        F = _flag_at(rng, s, _pick(rng, kind[k]), g)
        x["wf0"] = (1 if r == 1 else 0) if cat not in ("touch_holder", "stale_switch", "stale_holder") else (1 if r == 0 else 0)
        if cat in ("stale_switch", "stale_holder"):
            u = xc.stream_uniforms(ctx["seed"], [ctx["gid_pair"]], [ep], 1, 0)
            wnew = int(np.floor(2.0 * u[1][0]))                 # robot 0's with_flag in the new episode
            holder_new = 0 if wnew else 1
            r = 1 - holder_new if cat == "stale_switch" else holder_new
            s = (a, b)[r]
            F = _flag_at(rng, s, _pick(rng, kind[k]), g)
            x["wf0"] = 1 if r == 0 else 0                       # the toucher holds the flag in the step: no switch there
            x["counter"] = ms - 1
        if cat == "ids_switch":
            x["counter"] = ms - 1
        if cat == "touch_both":                                 # the partner's hip against the opposite face
            o = (b, a)[r]
            i = _pick(rng, 2)
            d = F - s[0:2]
            ax = int(np.argmax(np.abs(d)))
            tgt = np.array([F[0], F[1], _proxy(o, i)[2]])
            tgt[ax] += np.sign(d[ax]) * (0.05 + RAD[i] + BREAKING - _side(rng))
            tgt[1 - ax] += rng.uniform(-0.03, 0.03)
            o[0:2] += tgt[0:2] - _proxy(o, i)[0:2]
        if cat in MOVE_CATS:
            p = _proxy(s, 0)
            c = np.array([F[0], F[1]])
            away = (s[0:2] - c) / np.linalg.norm(s[0:2] - c)
            ax = int(np.argmax(np.abs(away)))
            dirv = np.zeros(2); dirv[ax] = np.sign(away[ax])
            step = abs(g) + rng.uniform(3e-4, 1e-3)
            x["v"][r] = dirv * step / SIM_DT * (1.0 if cat == "touch_pre_only" else -1.0)
            x["wf0"] = 1 if r == 1 else 0
        if cat == "nan1_switch":                                # at rest: the oracle stops integrating a pair with a bad robot
            x["nan"] = ("joint", 1)
            x["v"] = [np.zeros(2), np.zeros(2)]
    elif cat.startswith("tag_"):
        parts = cat.split("_")
        if parts[1] in KIND_NAMES:
            j = _pick(rng, KIND_NAMES.index(parts[1]))
            g = -_side(rng) if parts[2] == "in" else _side(rng)
        else:
            j, g = int(rng.integers(22)), -_side(rng)
        if parts[1] == "reverse":                               # robot 1's body against robot 0's foot
            b = _place_against(rng, a, _pick(rng, 0), int(rng.choice(BODY)), g, I0)
        else:
            a = _place_against(rng, b, j, int(rng.choice(BODY)), g, I0)
        if cat == "tag_switch":
            r = int(rng.integers(2))
            F = _flag_at(rng, (a, b)[r], _pick(rng, 2), -_side(rng))
            x["wf0"] = 1 if r == 1 else 0
        x["wf0"] = {"tag_hold0": 1, "tag_hold1": 0}.get(cat, x["wf0"])
        if cat == "tag_timeup":
            x["counter"] = ms - 1
    elif cat in TERM_CATS:
        if cat == "fall1":
            b = ec._design_state(b, "r22_in", rng).astype(np.float64)
        elif cat.startswith("timeup"):
            x["counter"] = ms - 1 if cat == "timeup_at" else ms - 2
        else:
            pos = a[0:3].copy()
            a = ec._design_state(a, cat, rng).astype(np.float64)
            a[0:3] = pos
        x["v"][0] = x["v"][0] * 0
    elif cat in BAD_CATS[:4]:
        r = int(cat[-1])
        x["nan"] = ("action" if "action" in cat else "joint", r)
        x["v"] = [np.zeros(2), np.zeros(2)]
    elif cat == "vis_head":
        L = rng.uniform(0.6, 1.2)
        a[0:2] = rng.uniform(-1.0, 1.0, 2)
        b[0:2] = a[0:2] + L * np.array([np.cos(h), np.sin(h)])
        F = a[0:2] + rng.uniform(0.35, 0.65) * (b[0:2] - a[0:2])
        x["v"] = [np.zeros(2), np.zeros(2)]
    elif cat == "vis_none":                                     # robot 1 beyond a wall
        ax, sgn = int(rng.integers(2)), rng.choice([-1.0, 1.0])
        b[ax] = sgn * rng.uniform(2.7, 3.3)
        b[1 - ax] = rng.uniform(-2.0, 2.0)
        x["v"] = [np.zeros(2), np.zeros(2)]
    elif cat == "vis_behind":
        R = pcs.rot(a[3:7])
        yaw = np.arctan2(R[1, 0], R[0, 0]) + np.pi - 1e-3 * rng.choice([-1.0, 1.0])
        b[0:2] = a[0:2] + rng.uniform(0.8, 1.5) * np.array([np.cos(yaw), np.sin(yaw)])
        x["v"] = [np.zeros(2), np.zeros(2)]
    elif cat == "vis_stacked":
        b[0:2] = a[0:2]
        b[2] = a[2] + rng.uniform(1.0, 1.4)
        x["v"] = [np.zeros(2), np.zeros(2)]
    elif cat in SPD_CATS:
        pass
    elif cat in PUSH_CATS + ("ids_push",):
        iv, du = ctx["interval"], ctx["duration"]
        x["push_count"] = {"push_cross": -(sub // 2), "push_draw": iv - int(rng.integers(1, min(sub, iv) + 1)),
                           "push_last": 0 if sub > 1 else du - 2, "push_off_first": 0 if sub > 1 else du - 1, "ids_push": -(sub // 2)}[cat]
        if cat == "ids_push":                                   # pushed in this step, then reset by the timeup
            x["counter"] = ms - 1
    elif cat in RESET_CATS:
        x["counter"] = ms - 1
    if F is None:
        F = _far_flag(rng, (a, b), PUSH_CLEAR if cat in PUSH_CATS + ("ids_push",) else 0.1)
    if x["nan"] and x["nan"][0] == "joint":                     # the NaN robot 1 m from the flag and 1.3 m from its partner
        r = x["nan"][1]
        s, o = (a, b) if r == 0 else (b, a)
        for _ in range(200):
            s[0:2] = rng.uniform(-2.2, 2.2, 2)
            if np.hypot(*(s[0:2] - o[0:2])) > 1.3 and np.hypot(*(s[0:2] - F)) > 1.0:
                break
    return a, b, F, x


def _pair_aux(rng, ctx, x, F, sts):
    A = np.zeros((2, capi.AUX_DIM))
    A[:, capi.AUX_COUNTER] = x["counter"]
    A[:, capi.AUX_WITH_FLAG] = (x["wf0"], 1 - x["wf0"])
    A[:, capi.AUX_FLAG_X], A[:, capi.AUX_FLAG_Y] = F
    A[:, capi.AUX_CONTROL_SPD] = f32(rng.uniform(0.5, 3.0, 2))
    A[:, capi.AUX_OPPO_VISIBLE] = rng.integers(0, 2, 2)
    A[:, capi.AUX_SWITCH_FLAG] = rng.integers(0, 2)
    A[:, capi.AUX_TOTAL_SPD] = rng.uniform(0.0, 2.0, 2) * max(x["counter"], 1)
    spd = [np.hypot(*f32(s[7:9])) for s in sts]
    A[:, capi.AUX_MAX_SPD] = [sp + (rng.uniform(0.05, 0.5) if rng.random() < 0.5 else -min(rng.uniform(0.05, 0.5), sp / 2)) if sp > 0.1
                             else rng.uniform(1.0, 2.0) for sp in spd]
    A[:, capi.AUX_PUSH_COUNT] = x["push_count"]
    A[:, capi.AUX_PUSH_F:capi.AUX_PUSH_F + 3] = f32(rng.uniform(-20, 20, (2, 3)))
    A[:, capi.AUX_FOOT_FRICTION] = rng.uniform(0.4, 3.0)
    A[:, capi.AUX_PUSH_DRAWS] = rng.integers(1, 9)
    A[:, capi.AUX_FLAG_DRAWS] = rng.integers(0, 9)
    A[:, capi.AUX_YAW_ACCUM_DEG] = rng.uniform(0, 360)
    A[:, capi.AUX_FLAG_TOUCH] = rng.integers(0, 2, 2)
    return A


def _predicted(ctx, before, rows):
    """the post state of the pair rows when nothing pushes them: start + v T"""
    st = before["state"][rows].astype(np.float64)
    st[:, 0:3] += st[:, 7:10] * ctx["T"]
    return st


def _pair_ok(ctx, cat, before, p, pushed):
    """the designed pair p is decisive (contacts on the pose before the last sub-step, rays and visibility on the predicted post
    pose) and reaches its category on the statement"""
    rows = np.array([2 * p, 2 * p + 1])
    sub = dict(state=before["state"][rows], aux=before["aux"][rows], episode=before["episode"][rows], obs=before["obs"][rows],
               actions=before["actions"][rows], reward_sum=before["reward_sum"][rows])
    post = _predicted(ctx, sub, [0, 1])
    c = dict(ctx, gid0=ctx["gid0"] + 2 * p)
    geo = geometry(c, sub, post)
    ref = step_statement(c, sub, post, geo)
    if not decisive(c, ref, geo, sub, post).all():
        return False
    fin = np.isfinite(post).all(1)
    fx, fy = sub["aux"][0, capi.AUX_FLAG_X], sub["aux"][0, capi.AUX_FLAG_Y]
    bx = pcs.arena_boxes(fx, fy)
    if fin.all() and not all(pcs.rays_decisive(s[0:3], pcs.rot(s[3:7]), bx).all() for s in post):
        return False
    if pushed:
        # a pushed robot moves by micrometres and turns by up to ~5e-5 rad: its rays stay decisive 3 mm and 1e-3 rad away
        offs = [np.array([x, y, z]) * 3e-3 for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)]
        turns = [ec.R.from_rotvec(np.eye(3)[ax] * sg * 1e-3).as_matrix() for ax in range(3) for sg in (-1, 1)]
        if not all(pcs.rays_decisive(s[0:3] + o, pcs.rot(s[3:7]), bx).all() for s in post for o in offs):
            return False
        if not all(pcs.rays_decisive(s[0:3], T @ pcs.rot(s[3:7]), bx).all() for s in post for T in turns):
            return False
    return bool(reaches(c, sub, ref, geo, [cat], post)[0])


def build(case):
    """(ctx, before, categories per pair): the designed fields of a batch; deterministic"""
    ctx = context(case)
    n, sub = ctx["n"], ctx["substeps"]
    P = n // 2
    rng = np.random.default_rng(SEED + 7 * n + sub + 3 * ctx["push"])
    cl = cats_of(sub, ctx["push"])
    cats = [cl[(p + n) % len(cl)] for p in range(P)]                  # every category once per len(cl) pairs
    if P >= 17:
        fix = id_cats(ctx["push"]) + ("nan1_switch", "nan_joint0", "nan_joint1")
        cats[:len(fix)] = fix
    I0 = ctx["init_state"]
    st = np.zeros((n, 37))
    aux = np.zeros((n, capi.AUX_DIM))
    ep = np.repeat(np.where(rng.random(P) < 0.5, rng.integers(1, 1000, P), rng.integers(2 ** 32 - 500, 2 ** 32 + 500, P)), 2).astype(np.int64)
    actions = rng.uniform(-1, 1, (n, 12)).astype(np.float32)
    obs = rng.normal(0, 1, (n, capi.OBS_DIM_SEPMC)).astype(np.float32)
    before = dict(state=st, aux=aux, episode=ep, obs=obs, actions=actions, reward_sum=rng.uniform(0.0, 3.0, n).astype(np.float32))
    for p, cat in enumerate(cats):
        rows = [2 * p, 2 * p + 1]
        if cat in ID_CATS:
            ep[2 * p + 1] = ep[2 * p] + int(rng.integers(1, 2 ** 20))
        for attempt in range(800):
            if attempt == 400 and cat not in ID_CATS + BAD_CATS:    # a rare pair the category cannot be placed for: a plain pair
                cat = cats[p] = "plain"                             # (the coverage test asserts every category elsewhere)
            c = dict(ctx, gid_pair=ctx["gid0"] + 2 * p)
            a, b, F, x = _design(c, cat, rng, I0, int(ep[2 * p]))
            for r, s in enumerate((a, b)):
                s[7:9] = x["v"][r]
                s[0:3] -= np.append(x["v"][r], 0.0) * (ctx["T"] - SIM_DT)       # designed on the pose before the last sub-step
            st[rows] = np.stack([a, b]).astype(np.float32)
            aux[rows] = _pair_aux(rng, ctx, x, F, st[rows])
            if cat in RESET_CATS[2:]:                           # the accumulator sum of robot r lands just below / above 360
                r = int(cat[3])
                u1 = xc.stream_uniforms(ctx["seed"], [c["gid_pair"]], [ep[2 * p]], 1, 1)[3][0]
                u2 = xc.stream_uniforms(ctx["seed"], [c["gid_pair"]], [ep[2 * p]], 1, 2)[0][0]
                dl = rng.uniform(1e-3, 1e-2) * (1 if cat.endswith("above") else -1)
                ya = 360.0 + dl - (360.0 * u2 if r == 1 else 0.0)
                aux[rows, capi.AUX_YAW_ACCUM_DEG] = np.mod(ya - 360.0 * u1, 360.0)
            actions[rows] = rng.uniform(-1, 1, (2, 12)).astype(np.float32)
            if x["nan"]:
                what, r = x["nan"]
                if what == "action":
                    actions[2 * p + r, rng.integers(12)] = np.nan
                else:
                    st[2 * p + r, 13 + rng.integers(12)] = np.nan
            if _pair_ok(ctx, cat, before, p, cat in PUSH_CATS + ("ids_push",)):
                break
        else:
            raise RuntimeError("no decisive pair %d (%s)" % (p, cat))
    return ctx, before, cats


def reaches(ctx, before, ref, geo, cats, post):
    """does each pair reach its category, on the statement `ref` of the post-step state `post` and its geometry `geo`"""
    P = len(cats)
    aux0 = before["aux"]
    wf = aux0[:, capi.AUX_WITH_FLAG].astype(int)
    gidp = ctx["gid0"] + 2 * np.arange(P)
    ep0 = before["episode"][0::2] - 1
    _, _, _, _, trace = pair_push(ctx, gidp, ep0, aux0[0::2, capi.AUX_PUSH_COUNT].astype(np.int64),
                                  aux0[0::2, capi.AUX_PUSH_DRAWS].astype(np.int64), aux0[:, capi.AUX_PUSH_F:capi.AUX_PUSH_F + 3])
    counts = np.array([t[0] for t in trace]).T if trace else np.zeros((P, 0))
    ons = np.array([t[1] for t in trace]).T if trace else np.zeros((P, 0), bool)
    fired = np.array([t[2] for t in trace]).T if trace else np.zeros((P, 0), bool)
    fin = np.isfinite(post).all(1)
    ok = np.zeros(P, bool)
    for p, c in enumerate(cats):
        a, b = 2 * p, 2 * p + 1
        G, Gp = geo["pre"][p], geo["post"][p]
        d, sw, tag = bool(ref["done"][p]), bool(ref["sw"][p]), bool(geo["tag"][p])
        tch = geo["touch"][a:b + 1]
        holder = 0 if wf[a] == 1 else 1
        nonh = 1 - holder
        with np.errstate(invalid="ignore"):
            kgap = {k: np.array([G["flag"][r][KIND == kk].min() for r in (0, 1)]) for k, kk in (("hip", 2), ("wheel", 1), ("foot", 0))}
            post_touch = np.array([(Gp["flag"][r][BODY] < 0).any() for r in (0, 1)])
            tk = {KIND_NAMES[kk]: G["tag_gap"][:, KIND == kk].min() for kk in range(5)}
        u = None
        if c.startswith("touch_") and c.split("_")[1] in ("hip", "wheel"):
            k, side = c.split("_")[1:]
            g = kgap[k][nonh]
            u = (sw and g < 0) if side == "in" else (not tch.any() and 0 < g < 1e-3)
        elif c == "touch_foot":
            u = not tch.any() and bool((kgap["foot"] < 0).any())
        elif c == "touch_holder":
            u = bool(tch[holder]) and not tch[nonh] and not sw
        elif c == "touch_both":
            u = bool(tch.all()) and sw
        elif c == "touch_pre_only":
            u = sw and not post_touch.any()
        elif c == "touch_post_only":
            u = not sw and not tch.any() and bool(post_touch.any())
        elif c.startswith("tag_") and c.split("_")[1] in KIND_NAMES:
            k, side = c.split("_")[1:]
            u = (tag and tk[k] < 0) if side == "in" else (not tag and 0 < tk[k] < 1e-3)
        elif c == "tag_reverse":
            u = not tag and bool((G["rev"][:, KIND == 0] < 0).any())
        elif c == "tag_switch":
            u = tag and sw and d
        elif c == "tag_timeup":
            u = tag and bool(ref["timeup"][p])
        elif c in ("tag_hold0", "tag_hold1"):
            u = tag and d and int(ref["with_flag"][a]) == (1 if c == "tag_hold0" else 0)
        elif c in ("left_pos_in", "left_neg_in"):
            u = (ref["left_z"][a] > LIMIT) if "pos" in c else (ref["left_z"][a] < -LIMIT)
        elif c in ("left_pos_out", "left_neg_out"):
            lz = ref["left_z"][a] * (1 if "pos" in c else -1)
            u = LIMIT - 1e-3 < lz < LIMIT and not d
        elif c == "r22_in":
            u = ref["r22"][a] < 0.5 and d
        elif c == "r22_out":
            u = 0.5 < ref["r22"][a] < 0.501 and not d
        elif c == "fall1":
            u = bool(ref["fall"][b]) and not d
        elif c == "timeup_at":
            u = bool(ref["timeup"][p]) and not (tag or ref["fall"][a] or ref["bad"][p])
        elif c == "timeup_before":
            u = not d and ref["counter"][a] == ctx["max_steps"] - 1
        elif c.startswith("nan_action"):
            u = bool(np.isnan(before["actions"][a + int(c[-1])]).any()) and not d
        elif c.startswith("nan_joint"):
            u = bool(ref["bad"][p]) and not fin[a + int(c[-1])] and fin[b - int(c[-1])]
        elif c == "nan1_switch":
            u = bool(ref["bad"][p]) and sw and not fin[b]
        elif c == "vis_root":
            u = bool(geo["root"][p]) and bool(geo["vis"][a] and geo["vis"][b])
        elif c == "vis_head":
            u = not geo["root"][p] and bool(geo["vis"][a] or geo["vis"][b])
        elif c == "vis_none":
            u = bool(fin[a] and fin[b]) and not (geo["vis"][a] or geo["vis"][b])
        elif c == "vis_behind":
            u = bool(geo["vis"][a]) and -1.0 < geo["cv"][a] < -np.cos(2e-3)
        elif c == "vis_stacked":
            u = post[a, 0] == post[b, 0] and post[a, 1] == post[b, 1] and not (geo["vis"][a] or geo["vis"][b])
        elif c == "max_up":
            u = ref["spd"][a] > ref["max_before"][a] and not d
        elif c == "max_keep":
            u = ref["spd"][a] < ref["max_before"][a] and not d
        elif c == "push_cross":
            u = counts.shape[1] > 0 and aux0[a, capi.AUX_PUSH_COUNT] <= 0 and bool((counts[p] > 0).any())
        elif c == "push_draw":
            u = bool(fired[p].any())
        elif c == "push_last":
            u = bool((ons[p] & (counts[p] == ctx["duration"] - 1)).any())
        elif c == "push_off_first":
            u = bool((~ons[p] & (counts[p] == ctx["duration"])).any())
        elif c in ("stale_switch", "stale_holder", "yaw0_below", "yaw0_above", "yaw1_below", "yaw1_above"):
            rs = reset_statement(ctx, gidp[p:p + 1], before["episode"][a:a + 1], aux0[a:a + 1, capi.AUX_YAW_ACCUM_DEG], tch)
            if c == "stale_switch":
                u = d and bool(rs["sw"][0]) and not sw
            elif c == "stale_holder":
                u = d and not rs["sw"][0] and bool(tch.any()) and not sw
            else:
                x = rs["yaw_sums"][int(c[3])][0]
                u = d and ((359.99 < x < 360.0 - 1e-3) if c.endswith("below") else (360.0 + 1e-3 < x < 360.01))
        elif c == "ids_switch":
            u = before["episode"][a] != before["episode"][b] and sw and d
        elif c == "ids_push":
            u = before["episode"][a] != before["episode"][b] and bool(ons[p].any()) and d
        elif c == "plain":
            u = not d
        ok[p] = bool(u)
    return ok


def decisive(ctx, ref, geo, before, post):
    """per pair: contact gaps clear contact_breaking by DELTA (PUSH_CLEAR if pushed), robot 0's fall quantities their thresholds,
    the visibility segments their boxes (finite pairs), spd the stored max_spd"""
    P = len(post) // 2
    ok = np.ones(P, bool)
    for p in range(P):
        m = PUSH_CLEAR if ref["push_on"][p] > 0 else DELTA
        G = geo["pre"][p]
        fin = np.isfinite(post[2 * p:2 * p + 2]).all(1)
        gaps = [G["flag"][r][BODY] for r in (0, 1) if fin[r]]
        if fin.all():
            gaps += [G["tag_gap"].ravel(), G["rev"].ravel()]
            ok[p] &= bool(geo["vis_ok"][p])
        g = np.concatenate(gaps) if gaps else np.zeros(0)
        ok[p] &= bool((np.abs(g) >= m).all())
        if fin[0]:
            ok[p] &= abs(abs(ref["left_z"][2 * p]) - LIMIT) >= DELTA and abs(ref["r22"][2 * p] - 0.5) >= DELTA
        for r in (0, 1):
            if fin[r] and ref["push_on"][p] == 0:
                ok[p] &= abs(ref["spd"][2 * p + r] - ref["max_before"][2 * p + r]) >= DELTA
    return ok


_BUILT = {}


def case(k):
    if k not in _BUILT:
        _BUILT[k] = build(CASES[k])
    return _BUILT[k]


# ------------------------------------------------------------------------------------------------------------ running a batch
EXACT_AUX = (capi.AUX_COUNTER, capi.AUX_WITH_FLAG, capi.AUX_OPPO_VISIBLE, capi.AUX_SWITCH_FLAG, capi.AUX_PUSH_COUNT, capi.AUX_PUSH_DRAWS,
             capi.AUX_FLAG_DRAWS, capi.AUX_FLAG_TOUCH)
CONT_AUX = tuple(c for c in range(capi.AUX_DIM) if c not in EXACT_AUX)


def readback(e):
    out = {k: e.get(f) for k, f in (("state", capi.F_STATE), ("aux", capi.F_AUX), ("episode", capi.F_EPISODE_ID), ("obs", capi.F_OBS),
                                     ("reward_sum", capi.F_REWARD_SUM), ("foot", capi.F_FOOT_POS))}
    out["counters"] = e.counters()
    return out


def _exact(got, ref, cols, rows, what, cats):
    wrong = [(int(rows[i]), cats[rows[i] // 2], int(c), got[i, c], ref[i, c]) for c in cols for i in np.nonzero(got[:, c] != ref[:, c])[0]]
    assert not wrong, (what, wrong[:8])


def _check_reset(ck, ctx, cats, pairs, got, obs, ep0, acc, touch, what):
    """the reset pairs `pairs`: state, aux, episode, observation row, feet against the reset statement"""
    rows = np.stack([2 * pairs, 2 * pairs + 1], 1).reshape(-1)
    gidp = ctx["gid0"] + 2 * pairs
    ref, S = reset_sensitivity(ctx, gidp, ep0, acc, touch)
    st = got["state"][rows].astype(np.float64)
    st[:, 3:7] = ec._sign_fix(st[:, 3:7], ref["state"][:, 3:7])
    ck.near(st, ref["state"], S["state"], what + " F_STATE")
    a = got["aux"][rows]
    # oppo_visible of the reset poses (drawn, not designed) is stated by the caster on the engine's own reset poses
    vis = np.zeros(len(rows), bool)
    for q in range(len(pairs)):
        vis[2 * q:2 * q + 2] = pcs.visible(st[2 * q], st[2 * q + 1], pcs.arena_boxes(ref["flag_reset"][0][q], ref["flag_reset"][1][q]))
    want = ref["aux"].copy()
    want[:, capi.AUX_OPPO_VISIBLE] = vis
    _exact(a, want, EXACT_AUX, rows, what, cats)
    ck.near(a[:, CONT_AUX], want[:, CONT_AUX], S["aux"][:, CONT_AUX], what + " aux")
    assert np.array_equal(got["episode"][rows], rep(ep0 + 1)) and np.all(got["reward_sum"][rows] == 0), (what, "episode")
    o = obs[rows].astype(np.float64)
    ck.near(o[:, 0:135], ref["obs"], S["obs"], what + " obs")
    assert np.array_equal(obs[rows], got["obs"][rows])
    V, SV = perception(st, want[:, capi.AUX_WITH_FLAG], *ref["flag_reset"], want[:, capi.AUX_CONTROL_SPD], vis)
    ck.rays(o[:, 135:], V, SV, what + " perception")
    ck.near(got["foot"][rows], ref["foot"], S["foot"], what + " F_FOOT_POS")


def run_case(lib, k, io="host", kappa=KAPPA, oracle=False):
    """Run batch k through `lib` (CUDA engine or oracle) and compare every output with the statement, robot by robot.  Engine A
    (auto_reset 0) takes the step; engine B (auto_reset 1) takes it again and resets the pairs it ends, then a masked reset of every
    third robot (its pair resets; some of them just auto-reset).  Returns the largest error / S ratios."""
    ctx, before, cats = case(k)
    n = ctx["n"]
    P = n // 2
    ck = xc.Check(kappa, oracle)
    A, B = make(lib, ctx, 0), make(lib, ctx, 1)
    try:
        slabs = [ec.Slab(x, int(io[-1])) if io.startswith("device") else None for x in (A, B)]
        c0A, c0B = A.counters(), B.counters()
        xc.set_before(A, before); xc.set_before(B, before)
        oA, rA, dA, recA = ec.step_io(A, before["actions"], io, slabs[0])
        fa = readback(A)
        oB, rB, dB, recB = ec.step_io(B, before["actions"], io, slabs[1])
        fb = readback(B)
        # ---- engine A: the step statement on the state read back
        post = fa["state"].astype(np.float64)
        geo = geometry(ctx, before, post)
        ref, S = sensitivity(ctx, before, post, geo)
        dec = decisive(ctx, ref, geo, before, post)
        assert dec.all(), [(int(p), cats[p]) for p in np.nonzero(~dec)[0][:6]]
        ok = reaches(ctx, before, ref, geo, cats, post)
        assert ok.all(), [(int(p), cats[p]) for p in np.nonzero(~ok)[0][:8]]
        done = rep(ref["done"])
        assert np.array_equal(dA.astype(bool), done), [(int(i), cats[i // 2], int(dA[i])) for i in np.nonzero(dA.astype(bool) != done)[0][:8]]
        assert int(fa["counters"][1] - c0A[1]) == int(done.sum()) and int(fa["counters"][0] - c0A[0]) == n
        fin = rep(np.isfinite(post).all(1).reshape(P, 2).all(1))        # pairs without a NaN robot
        a = fa["aux"]
        rows = np.arange(n)
        _exact(a[fin], ref["aux"][fin], EXACT_AUX, rows[fin], "aux", cats)
        _exact(a, ref["aux"], tuple(c for c in EXACT_AUX if c != capi.AUX_OPPO_VISIBLE), rows, "aux", cats)
        ck.near(a[:, CONT_AUX], ref["aux"][:, CONT_AUX], S["aux"][:, CONT_AUX], "aux")
        ck.near(rA, ref["reward64"], S["reward"], "reward")
        assert np.all(rA[rep(ref["bad"])] == 0)
        rs_own = (before["reward_sum"] + rA).astype(np.float32)
        assert oracle or np.array_equal(fa["reward_sum"], rs_own)
        ck.near(fa["reward_sum"], before["reward_sum"].astype(np.float64) + ref["reward64"], S["reward"] + np.spacing(rs_own), "reward_sum")
        assert np.array_equal(fa["episode"], before["episode"]) and np.array_equal(oA, fa["obs"], equal_nan=True)
        # a NaN robot's post state is not stated: its pair's observation rows and feet are left out; reward, done, counters and
        # the copied blocks are checked
        ck.near(oA[:, 0:135], ref["obs"], S["obs"], "obs", rows=fin)
        assert np.array_equal(oA[:, 0:66], before["obs"][:, 33:99]) and np.array_equal(oA[:, 99:123], before["obs"][:, 111:135])
        assert np.array_equal(oA[:, 123:135], before["actions"], equal_nan=True)
        fx, fy = ref["flag_step"]
        V, SV = perception(post[fin], ref["with_flag"][fin], fx[fin[0::2]], fy[fin[0::2]], before["aux"][fin, capi.AUX_CONTROL_SPD], geo["vis"][fin])
        ck.rays(oA[fin, 135:], V, SV, "perception")
        ck.near(fa["foot"], ref["foot"], S["foot"], "F_FOOT_POS", rows=fin)
        # ---- engine B: the same step, then the auto-reset of the pairs it ended
        assert np.array_equal(rB, rA) and np.array_equal(dB, dA)
        keep = ~done
        for key in ("state", "aux", "episode", "reward_sum", "foot"):
            assert np.array_equal(fb[key][keep], fa[key][keep], equal_nan=True), key
        assert np.array_equal(oB[keep], oA[keep], equal_nan=True)
        assert int(fb["counters"][1] - c0B[1]) == int(done.sum()) and int(fb["counters"][0] - c0B[0]) == n
        fin_p = np.nonzero(ref["done"])[0]
        if len(fin_p):
            _check_reset(ck, ctx, cats, fin_p, fb, oB, before["episode"][2 * fin_p] , ref["aux"][2 * fin_p, capi.AUX_YAW_ACCUM_DEG],
                         ref["aux"][np.stack([2 * fin_p, 2 * fin_p + 1], 1).reshape(-1), capi.AUX_FLAG_TOUCH],
                         "auto-reset")
        for rec, rw, dn in ((recA, rA, dA), (recB, rB, dB)):
            if rec is not None:
                assert np.array_equal(rec[:, :12], before["actions"], equal_nan=True) and np.array_equal(rec[:, 12], rw)
                assert np.array_equal(rec[:, 13], dn.astype(np.float32))
        # ---- engine B: a masked reset of every third robot: its pair resets, some of them reset by the step already
        mask = np.zeros(n, bool); mask[::3] = True
        o2 = B.reset(mask)
        f2 = readback(B)
        pairs = np.nonzero(mask.reshape(P, 2).any(1))[0]
        prow = np.stack([2 * pairs, 2 * pairs + 1], 1).reshape(-1)
        _check_reset(ck, ctx, cats, pairs, f2, o2, fb["episode"][2 * pairs], fb["aux"][2 * pairs, capi.AUX_YAW_ACCUM_DEG],
                     fb["aux"][prow, capi.AUX_FLAG_TOUCH], "masked reset")
        other = np.ones(n, bool); other[prow] = False
        for key in ("state", "aux", "episode", "reward_sum", "obs"):
            assert np.array_equal(f2[key][other], fb[key][other], equal_nan=True), key
        ck.ratios["n_done"] = int(done.sum())
        return ck.ratios
    finally:
        A.close(); B.close()
