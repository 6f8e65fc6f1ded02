"""fp64 statement of the EPMC episode logic (PlayGroundEnv, elements 0-3) and designed batches on which every branch of it is
decisive (host only, numpy float64).

The statement covers what the learner is handed after one `llq_step` of the EPMC engine and after an EPMC reset.  Like
tests/episode_cases.py it is computed from the fields set before the step (F_STATE, F_AUX, F_OBS, F_EPISODE_ID, the env's boxes)
and the state read back after it, so it states no dynamics: the batches run with the physics off (no PD torque, no gravity, no
solver iteration, no damping).  Base velocities are not zero, so the robots move during the step and the start pose and the post
pose differ.

  command   redrawn when `counter % cmd_freq == 0` (the counter before the increment, PGE:302-317): Philox stream 3, draw `cmd_draws`,
            keyed by (seed, global env id, episode - 1).  Element 0: the target 100 m from the START pose in direction 2 pi u0, and
            `last_pos_diff_len` recomputed; elements 1-3 keep their target and set `target_angle = atan2` from the start pose on every
            step.  `target_spd = lo + u1 (hi - lo)` with lo, hi rounded to fp32 (StepParams), the result held as a float
  done      counter += 1; fall (|left_z| > 1/sqrt 2 or R22 < 0.5), reach (`plen < 0.5` on the post pose), timeup
            (`counter >= max_steps`), bad (a non-finite state or reward: reward 0)
  reward    spd = |v . u| with u = (target - pos) / plen rounded to fp32; total_spd and max_spd (strict >) in double.  Element 0:
            exp(-|spd - target_spd|) exp(5 (cos yaw ux + sin yaw uy - 1)) / max_steps.  Elements 1-3 (PGE:504-539):
            reward_rot / max_steps * 0.2 - 0.1 (plen - last_len) / init_len, last_len := plen, plus exp(-|total_spd / counter -
            target_spd|) on reach (the incremented counter).  reward_sum in fp32
  push      per sub-step (PR:56-87): count += 1; when count > 0, a draw (stream 2, index push_draws) on `count % interval == 0`, after
            which count = 0; push_on = count < duration.  The force is (h cos 2 pi u0, h sin 2 pi u0, v) in fp32
  obs       prop / action history shift, the new prop, the action, the 778 perception rays of tests/perception_cases.py on the post
            pose and the env's boxes, and the target block R^-1 (target - pos) normalised in xy, target_spd
  reset     stream 1, draw 0 keyed by the episode id before the reset: friction u0, yaw accumulator fmod(acc + 360 u1, 360),
            cmd_freq = lo + floor(u2 (hi - lo)); the initial push draw; the init state with the yaw composed on the right (the
            half-angle sine and cosine rounded to fp32) at (0, 0, 0.5); target_spd kept from the previous episode (PGE:170-172);
            target x, last and init distance from the env's target (8 m on element 0; the corridor's, read back, on elements 1-3)

Both engines key the Philox counter with the episode's low 32 bits and 24 bits of the global env id's high word (the top byte is
the stream), so episode ids e and e + 2^32 draw the same numbers: the batches use ids on both sides of 2^32.

A robot on its target (plen = 0) has a non-finite direction u: its reward is NaN, so the step is `bad` (reward 0, done) and its
total_spd turns NaN.  Its target columns are R^-1 (0, 0, -z) normalised in xy, finite for the tilted base of that category.

Error model.  policy_cases.ErrorModel: the post-step state read back is perturbed by one fp32 rounding, the fp32 intermediates of the
kernel (spd, yaw, the exponents, the rotated target) and every output by `u |y|`; the largest deviation over R_DRAWS draws is the
output's sensitivity S.  The GPU bar is KAPPA S + 2^-23 |ref|; the perception rays keep the perception pin's bar.

Decisiveness.  Every continuous branch quantity (left_z, R22, plen, spd against max_spd) clears its threshold by DELTA on the post
state, by 1 cm where the robot moves during the step; the push envs stay 5 cm from every threshold.  Integer branches (the redraw,
timeup, the push schedule) are hit exactly; the reset's `u2 (hi - lo)` lies 1e-8 to 1e-6 from an integer on the designed envs.
"""
import numpy as np

import episode_cases as ec
import perception_cases as pcs
from lifelike_agility_and_play_b200 import _capi as capi
from policy_cases import ErrorModel, REF, philox4x32, R_DRAWS

# GPU bar factor, as for the PMC pin; the largest error / S measured on an H100 80GB HBM3 at a 700 W power limit is 18.8 (F_FOOT_POS,
# the kinematic chain's fp32 rounding beyond the one-rounding model), the others at most 8.3
KAPPA = 64.0
PERCEPTION_A = 1e-5
DELTA = 1e-4
MOVE = 1e-2                    # threshold clearance of a robot that moves during the step
PUSH_CLEAR = 5e-2              # ... and of a pushed one
SEED = 20261018
MAX_STEPS = 37
CMD_FREQ = (3, 11)
TARGET_SPD = (0.3, 2.7)        # not fp32 numbers: StepParams rounds them
FRICTION = (0.4, 3.0)
PUSH_H, PUSH_V = (0.0, 47.3), (0.0, 9.7)
PUSH_SCHEDULE = dict(push_start_count=-4, push_interval_steps=7, push_duration_steps=3)
LIMIT = ec.LIMIT
SIM_DT = 1.0 / 500.0

# batches: (n envs, element, sub-steps, pushes on, global_env_offset)
CASES = [
    (1, 0, 10, 1, 0),
    (7, 1, 10, 1, 0),
    (8, 2, 1, 1, 0),
    (9, 3, 10, 0, 0),
    (15, 0, 1, 1, 0),
    (16, 1, 10, 0, 0),
    (17, 2, 10, 1, 0),
    (31, 3, 1, 1, 0),
    (32, 0, 10, 0, 0),
    (33, 3, 10, 1, 2 ** 32 - 5),
    (4097, 0, 10, 1, 2 ** 32 - 5),
]

CMD_CATS = ("redraw0", "redraw_k", "redraw_f1", "noredraw")
REACH_CATS = ("reach_in", "reach_out", "reach_edge", "reach_cross", "reach_timeup", "reach_fall")
TIME_CATS = ("timeup_at", "timeup_before")
FALL_CATS = ("left_pos_in", "left_pos_out", "left_neg_in", "left_neg_out", "r22_in", "r22_out")
BAD_CATS = ("nan_action", "nan_joint", "on_target")
SPD_CATS = ("max_up", "max_keep")
PUSH_CATS = ("push_cross", "push_draw", "push_last", "push_off_first")
CORRIDOR_CATS = ("rot_dom", "dist_dom", "bonus_avg")
RESET_CATS = ("freq_below", "freq_above", "yaw_below", "yaw_above")
COMMON = CMD_CATS + REACH_CATS + TIME_CATS + FALL_CATS + BAD_CATS + SPD_CATS + ("plain",)
TERMS = ("rot", "dist", "bonus")


def cats_of(element, push):
    c = COMMON + (("post_pose",) + RESET_CATS if element == 0 else CORRIDOR_CATS)
    return c + (PUSH_CATS if push else ())


# ------------------------------------------------------------------------------------------------------------ Philox
def stream_uniforms(seed, gid, ep, stream, index):
    """[4, n] uniforms of stream_uniforms (csrc/llq_kernels.cuh, oracle): counter (gid lo, 24 bits of gid hi | stream << 24,
    episode lo, index), key (seed lo, seed hi)"""
    gid = np.asarray(gid, np.int64).astype(np.uint64)
    ep = np.asarray(ep, np.int64).astype(np.uint64)
    M = np.uint64(0xFFFFFFFF)
    c = philox4x32(gid & M, ((gid >> np.uint64(32)) & np.uint64(0xFFFFFF)) | np.uint64(stream << 24), ep & M,
                   np.asarray(index, np.int64).astype(np.uint64), int(seed) & 0xFFFFFFFF, int(seed) >> 32)
    return np.stack([(x.astype(np.float64) + 0.5) * (1.0 / 4294967296.0) for x in c])


def f32(x):
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)


def push_force(ctx, gid, ep, index):
    u = stream_uniforms(ctx["seed"], gid, ep, 2, index)
    lo, hi = f32(ctx["push_h"][0]), f32(ctx["push_h"][1])
    h = lo + u[1] * (hi - lo)
    a = 2.0 * np.pi * u[0]
    v = f32(ctx["push_v"][0]) + u[2] * (f32(ctx["push_v"][1]) - f32(ctx["push_v"][0]))
    return np.stack([f32(h * np.cos(a)), f32(h * np.sin(a)), f32(v)], 1)


def push_schedule(ctx, gid, ep, count, draws, force):
    """(count, draws, force, sub-steps on, (count, on) per sub-step) after the step's sub-steps"""
    count, draws, force = count.copy(), draws.copy(), force.copy()
    on = np.zeros(len(count), np.int64)
    trace = []
    if not ctx["push"]:
        return count, draws, force, on, trace
    for _ in range(ctx["substeps"]):
        count += 1
        pos = count > 0
        fire = pos & (count % ctx["interval"] == 0)
        if fire.any():
            force[fire] = push_force(ctx, gid[fire], ep[fire], draws[fire])
            draws[fire] += 1
            count[fire] = 0
        o = pos & (count < ctx["duration"])
        on += o
        trace.append((count.copy(), o))
    return count, draws, force, on, trace


# ------------------------------------------------------------------------------------------------------------ the statement
def yaw_of(st):
    M = ec.quat_matrix(st[:, 3:7])
    return np.arctan2(M[:, 1, 0], M[:, 0, 0]), M


def target_block(st, tx, ty, ts, em=REF):
    """obs 913-915: R^-1 (target - pos) normalised in xy, target_spd"""
    M = ec.quat_matrix(st[:, 3:7])
    d = np.einsum("nji,nj->ni", M, np.stack([f32(tx - st[:, 0]), f32(ty - st[:, 1]), f32(-st[:, 2])], 1))
    d = ec._rotated(d, em)
    n = np.hypot(d[:, 0], d[:, 1])
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.stack([d[:, 0] / n, d[:, 1] / n, ts], 1)


def step_statement(ctx, before, st, em=REF):
    """the outputs of one step from the fields set before it (`before`) and the post-step state `st` read back"""
    n = len(st)
    aux = before["aux"]
    gid = ctx["gid0"] + np.arange(n)
    ep = before["episode"] - 1
    st = em.rel(np.asarray(st, np.float64))
    start = before["state"][:, 0:3].astype(np.float64)
    counter = aux[:, capi.AUX_COUNTER].astype(np.int64)
    freq = aux[:, capi.AUX_CMD_FREQ].astype(np.int64)
    draws = aux[:, capi.AUX_CMD_DRAWS].astype(np.int64)
    tx, ty = aux[:, capi.AUX_TARGET_X].copy(), aux[:, capi.AUX_TARGET_Y].copy()
    ts, angle, last = aux[:, capi.AUX_TARGET_SPD].copy(), aux[:, capi.AUX_TARGET_ANGLE].copy(), aux[:, capi.AUX_LAST_POS_DIFF_LEN].copy()
    init = aux[:, capi.AUX_INIT_POS_DIFF_LEN] if ctx["element"] else np.ones(n)
    redraw = counter % freq == 0
    if redraw.any():
        u = stream_uniforms(ctx["seed"], gid[redraw], ep[redraw], 3, draws[redraw])
        if ctx["element"] == 0:
            a = 2.0 * np.pi * u[0]
            angle[redraw] = a
            tx[redraw] = start[redraw, 0] + np.cos(a) * 100.0
            ty[redraw] = start[redraw, 1] + np.sin(a) * 100.0
            last[redraw] = np.hypot(start[redraw, 0] - tx[redraw], start[redraw, 1] - ty[redraw])
        lo, hi = f32(ctx["target_spd"][0]), f32(ctx["target_spd"][1])
        ts[redraw] = f32(lo + u[1] * (hi - lo))
        draws = draws + redraw
    if ctx["element"]:
        angle = np.arctan2(ty - start[:, 1], tx - start[:, 0])
    counter = counter + 1
    dx, dy = tx - st[:, 0], ty - st[:, 1]
    plen = np.hypot(dx, dy)
    left_z, r22 = ec.tilt(st)
    fall = (np.abs(left_z) > LIMIT) | (r22 < 0.5)
    reach = plen < 0.5
    timeup = counter >= ctx["max_steps"]
    with np.errstate(invalid="ignore", divide="ignore"):
        ux, uy = f32(dx / plen), f32(dy / plen)
        spd = np.abs(st[:, 7] * ux + st[:, 8] * uy)
        spd = em.add(spd, np.abs(st[:, 7] * ux) + np.abs(st[:, 8] * uy))
        total = aux[:, capi.AUX_TOTAL_SPD] + spd
        mx = np.where(spd > aux[:, capi.AUX_MAX_SPD], spd, aux[:, capi.AUX_MAX_SPD])
        yaw, _ = yaw_of(st)
        yaw = em.add(yaw, 4.0)
        cy, sy = np.cos(yaw), np.sin(yaw)
        arg = em.add((cy * ux + sy * uy - 1.0) * 5.0, 10.0)
        rot = em.rel(np.exp(arg))
        if ctx["element"] == 0:
            vel = em.rel(np.exp(-np.abs(em.add(spd - ts, np.abs(ts)))))
            terms = np.stack([vel * rot / ctx["max_steps"], np.zeros(n), np.zeros(n)], 1)
        else:
            dist = f32((plen - last) / init)
            bonus = np.where(reach, em.rel(np.exp(-np.abs(em.add(f32(total / counter) - ts, np.abs(ts))))), 0.0)
            terms = np.stack([rot / ctx["max_steps"] * 0.2, -dist * 0.1, bonus], 1)
            last = plen
        rew = terms.sum(1)
        rew = em.add(rew, np.abs(terms).sum(1))
    bad = ~np.isfinite(st).all(1) | ~np.isfinite(rew)
    rew = np.where(bad, 0.0, rew)
    done = fall | reach | timeup | bad
    pc, pd, pf, pon, _ = push_schedule(ctx, gid, ep, aux[:, capi.AUX_PUSH_COUNT].astype(np.int64),
                                       aux[:, capi.AUX_PUSH_DRAWS].astype(np.int64), aux[:, capi.AUX_PUSH_F:capi.AUX_PUSH_F + 3])
    new = aux.copy()
    new[:, capi.AUX_COUNTER] = counter; new[:, capi.AUX_CMD_DRAWS] = draws
    new[:, capi.AUX_TARGET_X] = tx; new[:, capi.AUX_TARGET_Y] = ty; new[:, capi.AUX_TARGET_SPD] = ts
    new[:, capi.AUX_TARGET_ANGLE] = angle; new[:, capi.AUX_LAST_POS_DIFF_LEN] = last
    new[:, capi.AUX_TOTAL_SPD] = total; new[:, capi.AUX_MAX_SPD] = mx
    new[:, capi.AUX_PUSH_COUNT] = pc; new[:, capi.AUX_PUSH_DRAWS] = pd; new[:, capi.AUX_PUSH_F:capi.AUX_PUSH_F + 3] = pf
    obs = np.concatenate([before["obs"][:, 33:99], ec.prop(st, em), before["obs"][:, 111:135], before["actions"]], 1)
    tail = target_block(st, tx, ty, ts, em)
    rs = (before["reward_sum"].astype(np.float32) + rew.astype(np.float32)).astype(np.float32)
    foot = ec.foot_positions(st).reshape(n, 12)
    return dict(redraw=redraw, counter=counter, plen=plen, left_z=left_z, r22=r22, fall=fall, reach=reach, timeup=timeup, bad=bad,
                done=done, spd=spd, terms=terms, reward64=rew, reward=em.add(rew, np.abs(rew)), reward_sum=rs, aux=em.add(new, np.abs(new)),
                obs=em.add(obs, np.abs(obs)), tail=em.add(tail, np.abs(tail)), foot=em.add(foot, np.abs(foot)), push_on=pon,
                max_before=aux[:, capi.AUX_MAX_SPD])


def _sens(f, keys, draws=R_DRAWS, seed=SEED):
    ref = f(REF)
    S = {k: np.zeros_like(np.asarray(ref[k], np.float64)) for k in keys}
    for d in range(draws):
        got = f(ErrorModel(seed + d))
        for k in keys:
            with np.errstate(invalid="ignore"):
                S[k] = np.maximum(S[k], np.nan_to_num(np.abs(np.asarray(got[k], np.float64) - ref[k]), nan=0.0))
    return ref, S


def sensitivity(ctx, before, st):
    return _sens(lambda em: step_statement(ctx, before, st, em), ("reward", "aux", "obs", "tail", "foot"))


def perception(st, boxes, nbox, aux):
    """(values [n, 778], S) of obs 135-912 on the states st"""
    V, S = [], []
    for i in range(len(st)):
        bx = pcs.corridor_boxes(boxes[i, :nbox[i]]) if nbox[i] > 0 else pcs.SLAB
        v, s = pcs.epmc_row(np.asarray(st[i], np.float64), bx, aux[i])
        V.append(v[:778]); S.append(s[:778])
    return np.array(V), np.array(S)


def qmul(a, b):
    x1, y1, z1, w1 = a.T
    x2, y2, z2, w2 = b.T
    return np.stack([w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2, w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2,
                     w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2, w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2], 1)


def reset_draws(ctx, gid, ep, acc):
    """(friction, yaw accumulator, cmd_freq, push draws, push force) of resets of envs gid whose episode id is ep before the reset"""
    u = stream_uniforms(ctx["seed"], gid, ep, 1, 0)
    fr = f32(ctx["friction"][0]) + u[0] * (f32(ctx["friction"][1]) - f32(ctx["friction"][0]))
    yaw = np.fmod(acc + 360.0 * u[1], 360.0)
    lo, hi = ctx["cmd_freq"]
    freq = lo + np.floor(u[2] * (hi - lo))
    n = len(gid)
    if ctx["push"]:
        return fr, yaw, freq, np.ones(n), push_force(ctx, gid, ep, np.zeros(n, np.int64)), u
    return fr, yaw, freq, np.zeros(n), np.zeros((n, 3)), u


def reset_statement(ctx, gid, ep, aux, tgx, em=REF):
    """(state [n, 37], aux [n, 18], observation row without the rays [n, 135 + 3]) of resets; tgx = the new episode's target x"""
    n = len(gid)
    fr, yaw, freq, pdraws, pf, _ = reset_draws(ctx, gid, ep, aux[:, capi.AUX_YAW_ACCUM_DEG])
    I0 = f32(ctx["init_state"])
    half = 0.5 * yaw * (np.pi / 180.0)
    q0 = I0[3:7] / np.linalg.norm(I0[3:7])
    qn = qmul(np.repeat(q0[None], n, 0), np.stack([np.zeros(n), np.zeros(n), f32(np.sin(half)), f32(np.cos(half))], 1))
    st = np.repeat(I0[None], n, 0)
    st[:, 0:3] = (0.0, 0.0, 0.5)
    st[:, 3:7] = em.add(qn, 1.0)
    new = aux.copy()
    new[:, capi.AUX_COUNTER] = 0; new[:, capi.AUX_CMD_FREQ] = freq; new[:, capi.AUX_TARGET_X] = tgx; new[:, capi.AUX_TARGET_Y] = 0.0
    new[:, capi.AUX_LAST_POS_DIFF_LEN] = np.abs(tgx); new[:, capi.AUX_INIT_POS_DIFF_LEN] = np.abs(tgx)
    new[:, capi.AUX_TOTAL_SPD] = 0.0; new[:, capi.AUX_MAX_SPD] = 0.0
    new[:, capi.AUX_PUSH_COUNT] = ctx["start_count"]
    new[:, capi.AUX_PUSH_F:capi.AUX_PUSH_F + 3] = pf; new[:, capi.AUX_FOOT_FRICTION] = fr
    new[:, capi.AUX_PUSH_DRAWS] = pdraws; new[:, capi.AUX_CMD_DRAWS] = 0; new[:, capi.AUX_YAW_ACCUM_DEG] = yaw
    p = ec.prop(st, em)
    obs = np.concatenate([p, p, p, np.zeros((n, 36)), target_block(st, tgx, np.zeros(n), aux[:, capi.AUX_TARGET_SPD], em)], 1)
    foot = ec.foot_positions(st).reshape(n, 12)
    return dict(state=em.add(st, np.abs(st)), aux=em.add(new, np.abs(new)), obs=em.add(obs, np.abs(obs)), foot=em.add(foot, np.abs(foot)))


def reset_sensitivity(ctx, gid, ep, aux, tgx):
    return _sens(lambda em: reset_statement(ctx, gid, ep, aux, tgx, em), ("state", "aux", "obs", "foot"), seed=SEED + 100)


# ------------------------------------------------------------------------------------------------------------ designed batches
def init_state(element):
    from test_golden_epmc import GOLD, terrain_gold
    return (np.load(GOLD) if element == 0 else terrain_gold(element))["init_state"].astype(np.float64)


def context(case):
    n, element, substeps, push, gid0 = case
    return dict(n=n, element=element, substeps=substeps, push=push, gid0=gid0, seed=SEED + n, max_steps=MAX_STEPS,
                cmd_freq=CMD_FREQ, target_spd=TARGET_SPD, friction=FRICTION, push_h=PUSH_H, push_v=PUSH_V, start_count=PUSH_SCHEDULE["push_start_count"],
                interval=PUSH_SCHEDULE["push_interval_steps"], duration=PUSH_SCHEDULE["push_duration_steps"], init_state=init_state(element),
                T=substeps * SIM_DT)


def engine_config(ctx, auto_reset):
    from test_golden_epmc import EPMC_CFG, terrain_cfg, terrain_gold
    cfg = dict(EPMC_CFG) if ctx["element"] == 0 else terrain_cfg(terrain_gold(ctx["element"]))
    cfg.update(ec.PHYSICS_OFF, lin_damping=0.0, ang_damping=0.0, substeps=ctx["substeps"], push_enabled=ctx["push"],
               global_env_offset=ctx["gid0"], seed=ctx["seed"], auto_reset=auto_reset, max_steps=ctx["max_steps"],
               cmd_freq_lo=CMD_FREQ[0], cmd_freq_hi=CMD_FREQ[1], target_spd_lo=TARGET_SPD[0], target_spd_hi=TARGET_SPD[1],
               friction_lo=FRICTION[0], friction_hi=FRICTION[1], push_h_lo=PUSH_H[0], push_h_hi=PUSH_H[1], push_v_lo=PUSH_V[0],
               push_v_hi=PUSH_V[1], **PUSH_SCHEDULE)
    return cfg


_BLOB = []


def make(lib, ctx, auto_reset):
    if not _BLOB:
        from lifelike_agility_and_play_b200.model.compile_model import pack_model
        _BLOB.append(pack_model(ec.model()))
    e = capi.VecEngine(lib, ctx["n"], _BLOB[0], None, **engine_config(ctx, auto_reset))
    e.set_init_state(ctx["init_state"])
    e.reset()
    return e


def _yaw_quat(yaw, base):
    """the init orientation turned by yaw about world z"""
    return (ec.R.from_euler("z", yaw) * ec.R.from_quat(base)).as_quat()


def _search_episodes(ctx, gid, want, rng, start):
    """an episode id (before the reset) near `start` whose stream-1 draw satisfies want(u)"""
    for t in range(50):
        ep = (start if t < 5 else int(rng.integers(1, 2 ** 33))) + rng.integers(0, 2 ** 20) + np.arange(2 ** 18)
        u = stream_uniforms(ctx["seed"], np.full(len(ep), gid), ep, 1, 0)
        ok = np.flatnonzero(want(u))
        if len(ok):
            return int(ep[ok[0]])
    raise RuntimeError("no episode id found")


def _freq_edge(u, side):
    x = u[2] * (CMD_FREQ[1] - CMD_FREQ[0])
    d = x - np.round(x)
    return (side * d >= 1e-8) & (side * d <= 1e-6) & (np.round(x) > 0) & (np.round(x) < CMD_FREQ[1] - CMD_FREQ[0])


def build(case, boxes, nbox):
    """(ctx, before, categories): the designed fields of a batch; deterministic.  boxes / nbox: the env's corridor after the first
    reset (an input of the statement)"""
    ctx = context(case)
    n, el, T = ctx["n"], ctx["element"], ctx["T"]
    rng = np.random.default_rng(SEED + 7 * n + el)
    cl = cats_of(el, ctx["push"])
    cats = [cl[(i * 7 + n) % len(cl)] for i in range(n)]
    I0 = ctx["init_state"]
    st = np.repeat(f32(I0)[None], n, 0)
    st[:, 7:13] = 0.0; st[:, 25:37] = 0.0
    aux = np.zeros((n, capi.AUX_DIM))
    ep = np.where(rng.random(n) < 0.5, rng.integers(1, 1000, n), rng.integers(2 ** 32 - 500, 2 ** 32 + 500, n)).astype(np.int64)
    actions = rng.uniform(-1, 1, (n, 12)).astype(np.float32)
    obs = rng.normal(0, 1, (n, 916)).astype(np.float32)
    for i, cat in enumerate(cats):
        bx = boxes[i, :nbox[i]].astype(np.float64)
        for attempt in range(200):
            s, a = _design(ctx, cat, rng, bx, I0)
            s = s.astype(np.float32)
            if el and not _rays_ok(s, T, bx, cat in PUSH_CATS):
                continue
            break
        else:
            raise RuntimeError("no decisive pose for env %d (%s)" % (i, cat))
        st[i], aux[i] = s, a
        gid = ctx["gid0"] + i
        if cat in ("freq_below", "freq_above"):
            ep[i] = _search_episodes(ctx, gid, lambda u: _freq_edge(u, -1 if cat == "freq_below" else 1), rng, int(ep[i]))
        elif cat in ("yaw_below", "yaw_above"):
            u1 = stream_uniforms(ctx["seed"], [gid], [ep[i]], 1, 0)[1][0]
            dl = rng.uniform(1e-3, 1e-2)
            aux[i, capi.AUX_YAW_ACCUM_DEG] = 360.0 - 360.0 * u1 + (dl if cat == "yaw_above" else -dl)
        if cat == "nan_action":
            actions[i, rng.integers(12)] = np.nan
        elif cat == "nan_joint":
            st[i, 13 + rng.integers(12)] = np.nan
    before = dict(state=st, aux=aux, episode=ep, obs=obs, actions=actions, reward_sum=rng.uniform(0.0, 3.0, n).astype(np.float32))
    return ctx, before, cats


def _rays_ok(s, T, bx, pushed=False):
    """every ray decisive at the start and the predicted post pose; a pushed robot (it moves by millimetres) also 3 mm away"""
    p = s.astype(np.float64)
    b = pcs.corridor_boxes(bx)
    offs = [np.zeros(3), T * p[7:10]] + ([np.array([x, y, z]) * 3e-3 for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)] if pushed else [])
    return all(pcs.rays_decisive(p[0:3] + o, pcs.rot(p[3:7]), b).all() for o in offs)


def _design(ctx, cat, rng, bx, I0):
    """(state, aux) of one env before the step"""
    el, T, ms = ctx["element"], ctx["T"], ctx["max_steps"]
    s = f32(I0).copy()
    s[7:13] = 0.0; s[25:37] = 0.0
    yaw = rng.uniform(-np.pi, np.pi)
    if el:
        half = bx[0, 1] - bx[0, 4]
        xmax = float((bx[2:, 0] + bx[2:, 3]).max()) if len(bx) > 2 else 5.0
        x, y = rng.uniform(0.3, xmax), rng.uniform(-0.6, 0.6) * min(half, 1.5)
    else:
        x, y = rng.uniform(-3, 3, 2)
    s[0:3] = f32([x, y, rng.uniform(0.62, 0.9)])
    s[3:7] = _yaw_quat(yaw, I0[3:7])
    a = np.zeros(capi.AUX_DIM)
    freq = int(rng.integers(CMD_FREQ[0], CMD_FREQ[1]))
    counter = int(rng.integers(1, ms - 3))
    if counter % freq == 0:
        counter += 1
    a[capi.AUX_CMD_FREQ] = freq
    a[capi.AUX_CMD_DRAWS] = rng.integers(0, 20)
    a[capi.AUX_TARGET_SPD] = f32(rng.uniform(*TARGET_SPD))
    a[capi.AUX_TOTAL_SPD] = rng.uniform(0.0, 2.0) * max(counter, 1)
    a[capi.AUX_MAX_SPD] = rng.uniform(3.0, 4.0)                # above any speed of the batches unless a category sets it
    a[capi.AUX_PUSH_COUNT] = -1000                              # far from the window unless a push category sets it
    a[capi.AUX_PUSH_DRAWS] = rng.integers(1, 9)
    a[capi.AUX_PUSH_F:capi.AUX_PUSH_F + 3] = f32(rng.uniform(-20, 20, 3))
    a[capi.AUX_FOOT_FRICTION] = rng.uniform(0.4, 3.0)
    a[capi.AUX_YAW_ACCUM_DEG] = rng.uniform(0, 360)
    a[capi.AUX_TARGET_ANGLE] = rng.uniform(-3, 3)
    # a target 2..8 m away and a velocity of up to 1.5 m/s: plen stays far from 0.5
    h = rng.uniform(-np.pi, np.pi)
    dist = rng.uniform(2.0, 8.0)
    v = rng.uniform(0.0, 1.5) * np.array([np.cos(rng.uniform(-np.pi, np.pi)), np.sin(rng.uniform(-np.pi, np.pi))])
    # the angular velocity stays zero: the orientation does not change during the step
    to_target = np.array([np.cos(h), np.sin(h)])
    if cat in CMD_CATS or cat == "post_pose":
        if cat == "redraw0":
            counter = 0
        elif cat == "redraw_k":
            counter = freq * int(rng.integers(1, max(2, (ms - 2) // freq)))
        elif cat == "redraw_f1":
            freq = 1
        elif cat == "noredraw":
            counter = freq * int(rng.integers(1, max(2, (ms - 1) // freq))) - 1
        elif cat == "post_pose":
            counter = freq * int(rng.integers(0, max(1, (ms - 2) // freq)))
            v = rng.uniform(1.0 / T * MOVE * 1.5, 1.0 / T * MOVE * 3) * np.array([np.cos(h + 1), np.sin(h + 1)])
    elif cat in REACH_CATS or cat in ("on_target", "bonus_avg"):
        if cat == "reach_in":
            dist, v = 0.5 - rng.uniform(2, 8) * DELTA, v * 0
        elif cat == "reach_out":
            dist, v = 0.5 + rng.uniform(2, 8) * DELTA, v * 0
        elif cat == "reach_edge":                  # plen exactly 0.5 in double: the strict < is stated exactly
            dist, v, h = 0.5, v * 0, 0.0
            to_target = np.array([1.0, 0.0])
        elif cat in ("reach_cross", "bonus_avg"):
            a_, b_ = rng.uniform(1, 2) * MOVE, rng.uniform(1, 2) * MOVE
            dist = 0.5 + a_
            v = (a_ + b_) / T * to_target
        elif cat == "reach_timeup":
            dist, v, counter, freq = 0.5 - rng.uniform(2, 8) * DELTA, v * 0, ms - 1, ms + 3
        elif cat == "reach_fall":
            dist, v = 0.5 - rng.uniform(2, 8) * DELTA, v * 0
            s = ec._design_state(s, "r22_in", rng).astype(np.float64)
        elif cat == "on_target":
            dist, v = 0.0, v * 0
        if cat == "bonus_avg":
            counter = int(rng.integers(1, 4))
            a[capi.AUX_TOTAL_SPD] = rng.uniform(0.5, 2.0)
        if counter % freq == 0 and cat != "reach_timeup":
            counter += 1
    elif cat in TIME_CATS:
        counter = ms - 1 if cat == "timeup_at" else ms - 2
        freq = ms + 3
    elif cat in FALL_CATS:
        v = v * 0
        s = ec._design_state(s, cat, rng).astype(np.float64)
    elif cat in SPD_CATS:
        v = rng.uniform(0.5, 1.5) * np.array([np.cos(h + 0.4), np.sin(h + 0.4)])
        spd = abs(v @ to_target)           # the direction to the target does not change by more than 1e-3 rad during the step
        dist = rng.uniform(20.0, 40.0)
        a[capi.AUX_MAX_SPD] = spd - 0.05 if cat == "max_up" else spd + 0.05
    elif cat in CORRIDOR_CATS:
        if cat == "rot_dom":
            v = v * 0
            s[3:7] = _yaw_quat(h + rng.uniform(-0.2, 0.2), base=I0[3:7])
        elif cat == "dist_dom":
            v = rng.uniform(1.0, 2.0) * to_target
            s[3:7] = _yaw_quat(h + np.pi + rng.uniform(-0.3, 0.3), base=I0[3:7])
            a[capi.AUX_INIT_POS_DIFF_LEN] = rng.uniform(0.3, 1.0)
    elif cat in PUSH_CATS:
        v = v * 0
        dist = rng.uniform(3.0, 8.0)
        sub, iv, du = ctx["substeps"], ctx["interval"], ctx["duration"]
        pc = {"push_cross": -(sub // 2), "push_draw": iv - int(rng.integers(1, min(sub, iv) + 1)),
              "push_last": 0 if sub > 1 else du - 2, "push_off_first": 0 if sub > 1 else du - 1}[cat]
        a[capi.AUX_PUSH_COUNT] = pc
    elif cat in RESET_CATS:
        dist, v = 0.5 - rng.uniform(2, 8) * DELTA, v * 0
        if counter % freq == 0:
            counter += 1
    if el == 0 and cat in ("redraw0", "redraw_k", "redraw_f1", "post_pose") and not cat == "post_pose":
        v = v * 0 if rng.random() < 0.5 else v
    s[7:9] = v
    tgt = s[0:2] + dist * to_target
    a[capi.AUX_TARGET_X], a[capi.AUX_TARGET_Y] = (tgt[0], tgt[1]) if cat == "reach_edge" else (f32(tgt[0]), f32(tgt[1]))
    if cat == "on_target":
        s[3:7] = ec._design_state(s, "left_pos_out", rng).astype(np.float64)[3:7]      # tilted: R^-1 (0, 0, -z) has a direction
        a[capi.AUX_TARGET_X], a[capi.AUX_TARGET_Y] = f32(s[0]), f32(s[1])
    a[capi.AUX_COUNTER] = counter
    a[capi.AUX_CMD_FREQ] = freq
    last = np.hypot(s[0] - a[capi.AUX_TARGET_X], s[1] - a[capi.AUX_TARGET_Y])
    a[capi.AUX_LAST_POS_DIFF_LEN] = last + (rng.uniform(-1e-3, 1e-3) if cat == "rot_dom" else rng.uniform(-0.3, 0.3))
    if not a[capi.AUX_INIT_POS_DIFF_LEN]:
        a[capi.AUX_INIT_POS_DIFF_LEN] = rng.uniform(4.0, 12.0)
    s[3:7] /= np.linalg.norm(s[3:7])
    return s, a


def reaches(ctx, before, ref, cats, post):
    """does each env reach its category, on the statement `ref` of the post-step state `post`"""
    n = ctx["n"]
    aux0 = before["aux"]
    c0 = aux0[:, capi.AUX_COUNTER].astype(np.int64)
    fq = aux0[:, capi.AUX_CMD_FREQ].astype(np.int64)
    moved = np.hypot(*(post[:, 0:2] - before["state"][:, 0:2].astype(np.float64)).T)
    start_plen = np.hypot(aux0[:, capi.AUX_TARGET_X] - before["state"][:, 0], aux0[:, capi.AUX_TARGET_Y] - before["state"][:, 1])
    gid = ctx["gid0"] + np.arange(n)
    _, _, _, _, trace = push_schedule(ctx, gid, before["episode"] - 1, aux0[:, capi.AUX_PUSH_COUNT].astype(np.int64),
                                      aux0[:, capi.AUX_PUSH_DRAWS].astype(np.int64), aux0[:, capi.AUX_PUSH_F:capi.AUX_PUSH_F + 3])
    counts = np.array([t[0] for t in trace]).T if trace else np.zeros((n, 0))
    ons = np.array([t[1] for t in trace]).T if trace else np.zeros((n, 0), bool)
    others = ref["fall"] | ref["timeup"] | ref["bad"]
    ok = np.zeros(n, bool)
    for i, c in enumerate(cats):
        r = ref
        u = dict(
            redraw0=c0[i] == 0, redraw_k=r["redraw"][i] and c0[i] > 0 and fq[i] > 1, redraw_f1=fq[i] == 1,
            noredraw=(c0[i] + 1) % fq[i] == 0 and not r["redraw"][i],
            post_pose=r["redraw"][i] and moved[i] >= MOVE,
            reach_in=r["reach"][i] and moved[i] == 0 and not others[i], reach_edge=r["plen"][i] == 0.5 and not r["done"][i], reach_out=not r["reach"][i] and 0.5 < r["plen"][i] < 0.501 and moved[i] == 0,
            reach_cross=r["reach"][i] and start_plen[i] > 0.5 + MOVE and r["plen"][i] < 0.5 - MOVE and not others[i],
            reach_timeup=r["reach"][i] and r["timeup"][i], reach_fall=r["reach"][i] and r["fall"][i],
            timeup_at=r["timeup"][i] and not (r["reach"][i] or r["fall"][i] or r["bad"][i]), timeup_before=not r["done"][i] and r["counter"][i] == ctx["max_steps"] - 1,
            left_pos_in=r["left_z"][i] > LIMIT, left_pos_out=LIMIT - 1e-3 < r["left_z"][i] < LIMIT and not r["done"][i],
            left_neg_in=r["left_z"][i] < -LIMIT, left_neg_out=-LIMIT < r["left_z"][i] < -LIMIT + 1e-3 and not r["done"][i],
            r22_in=r["r22"][i] < 0.5, r22_out=0.5 < r["r22"][i] < 0.501 and not r["done"][i],
            nan_action=bool(np.isnan(before["actions"][i]).any()) and not r["done"][i],
            nan_joint=bool(r["bad"][i]) and not np.isfinite(post[i]).all(),
            on_target=bool(r["bad"][i]) and r["plen"][i] == 0.0 and np.isfinite(post[i]).all(),
            max_up=r["spd"][i] > r["max_before"][i] and not r["done"][i], max_keep=r["spd"][i] < r["max_before"][i] and not r["done"][i],
            plain=not r["done"][i],
            rot_dom=int(np.argmax(np.abs(r["terms"][i]))) == 0, dist_dom=int(np.argmax(np.abs(r["terms"][i]))) == 1,
            bonus_avg=r["reach"][i] and abs(r["terms"][i, 2] - np.exp(-abs(f32(r["aux"][i, capi.AUX_TOTAL_SPD] / (r["counter"][i] - 1)) - r["aux"][i, capi.AUX_TARGET_SPD]))) > 1e-3,
            push_cross=counts.shape[1] > 0 and aux0[i, capi.AUX_PUSH_COUNT] <= 0 and (counts[i] > 0).any(),
            push_draw=r["aux"][i, capi.AUX_PUSH_DRAWS] > aux0[i, capi.AUX_PUSH_DRAWS],
            push_last=bool((ons[i] & (counts[i] == ctx["duration"] - 1)).any()),
            push_off_first=bool((~ons[i] & (counts[i] == ctx["duration"])).any()),
            freq_below=r["done"][i], freq_above=r["done"][i], yaw_below=r["done"][i], yaw_above=r["done"][i],
        )[c]
        ok[i] = bool(u)
        if c in ("freq_below", "freq_above"):
            uu = stream_uniforms(ctx["seed"], [gid[i]], [before["episode"][i]], 1, 0)
            ok[i] &= bool(_freq_edge(uu, -1 if c == "freq_below" else 1)[0])
        if c in ("yaw_below", "yaw_above"):
            u1 = stream_uniforms(ctx["seed"], [gid[i]], [before["episode"][i]], 1, 0)[1][0]
            x = aux0[i, capi.AUX_YAW_ACCUM_DEG] + 360.0 * u1
            ok[i] &= (359.99 < x < 360.0 - 1e-3) if c == "yaw_below" else (360.0 + 1e-3 < x < 360.01)
    return ok


def decisive(ctx, ref, before, post):
    """every continuous branch quantity clears its threshold by DELTA, by MOVE where the robot moved, by PUSH_CLEAR where it was
    pushed; a `bad` env decides nothing else"""
    moved = np.hypot(*(post[:, 0:2] - before["state"][:, 0:2].astype(np.float64)).T) > 0
    m = np.where(ref["push_on"] > 0, PUSH_CLEAR, np.where(moved, MOVE, DELTA))
    with np.errstate(invalid="ignore"):
        ok = (np.abs(np.abs(ref["left_z"]) - LIMIT) >= DELTA) & (np.abs(ref["r22"] - 0.5) >= DELTA) & (np.abs(ref["plen"] - 0.5) >= m)
        ok &= np.abs(ref["spd"] - ref["max_before"]) >= DELTA
    return ref["bad"] | ok | ((ref["plen"] == 0.5) & (np.abs(np.abs(ref["left_z"]) - LIMIT) >= DELTA) & (np.abs(ref["r22"] - 0.5) >= DELTA))


_BUILT = {}


def case(k):
    """(ctx, before, categories) of batch k; the corridors are those of the oracle's first reset (the engines draw the same)"""
    if k not in _BUILT:
        from oracle import oracle
        ctx = context(CASES[k])
        e = make(oracle.load(), ctx, 0)
        boxes, nbox = e.get(capi.F_BOXES).reshape(ctx["n"], capi.MAX_BOXES, 6).astype(np.float64), e.get(capi.F_NBOX)
        e.close()
        _BUILT[k] = build(CASES[k], boxes, nbox)
    return _BUILT[k]


# ------------------------------------------------------------------------------------------------------------ running a batch
EXACT_AUX = (capi.AUX_COUNTER, capi.AUX_CMD_FREQ, capi.AUX_CMD_DRAWS, capi.AUX_PUSH_COUNT, capi.AUX_PUSH_DRAWS)
CONT_AUX = tuple(c for c in range(capi.AUX_DIM) if c not in EXACT_AUX)


def set_before(e, before):
    n = e.n
    for f, v in ((capi.F_STATE, before["state"]), (capi.F_WARMSTART, np.zeros((n, 32), np.float32)), (capi.F_AUX, before["aux"]),
                 (capi.F_EPISODE_ID, before["episode"]), (capi.F_OBS, before["obs"]), (capi.F_REWARD_SUM, before["reward_sum"]),
                 (capi.F_EPISODE_STEPS, np.zeros(n, np.int32))):
        e.set(f, v)


def readback(e):
    out = {k: e.get(f) for k, f in (("state", capi.F_STATE), ("aux", capi.F_AUX), ("episode", capi.F_EPISODE_ID), ("obs", capi.F_OBS),
                                     ("reward_sum", capi.F_REWARD_SUM), ("foot", capi.F_FOOT_POS), ("nbox", capi.F_NBOX))}
    out["boxes"] = e.get(capi.F_BOXES).reshape(e.n, capi.MAX_BOXES, 6).astype(np.float64)
    out["counters"] = e.counters()
    return out


class Check:
    """the bars: KAPPA S + 2^-23 |ref| on the CUDA engine (ratios kept), 1e-6 max(1, |ref|) + 4 S on the oracle (fp64 throughout);
    the perception rays A max(1, |ref|) + 4 S on both"""

    def __init__(self, kappa, oracle):
        self.kappa, self.oracle, self.ratios = kappa, oracle, {}

    def near(self, got, ref, S, what, rows=None):
        if self.oracle:
            got, ref, S = (np.asarray(x, np.float64) for x in (got, ref, S))
            if rows is not None:
                got, ref, S = got[rows], ref[rows], S[rows]
            nan = np.isnan(ref)
            assert np.array_equal(np.isnan(got), nan), (what, np.argwhere(np.isnan(got) != nan)[:6])
            err = np.abs(np.where(nan, 0.0, got - ref))
            bad = err > 1e-6 * np.maximum(1.0, np.abs(np.where(nan, 0.0, ref))) + 4 * S
            assert not bad.any(), (what, [(tuple(int(x) for x in ix), got[tuple(ix)], ref[tuple(ix)]) for ix in np.argwhere(bad)[:6]])
            return
        r = ec._ratio(got, ref, S, self.kappa, what, rows)
        self.ratios[what] = max(self.ratios.get(what, 0.0), r)

    def rays(self, got, ref, S, what):
        err = np.abs(np.asarray(got, np.float64) - ref)
        bar = PERCEPTION_A * np.maximum(1.0, np.abs(ref)) + 4 * S
        bad = np.argwhere(err > bar)
        assert len(bad) == 0, (what, [(int(i), int(j) + 135, got[i, j], ref[i, j], S[i, j]) for i, j in bad[:6]])
        self.ratios[what + " A"] = max(self.ratios.get(what + " A", 0.0), float(((err - 4 * S) / np.maximum(1.0, np.abs(ref))).max()))


def _check_reset(ck, ctx, cats, rows, got, obs, gid, ep, aux_in, what):
    """the reset rows `rows`: state, aux, episode, observation row, feet against the reset statement"""
    tgx = np.full(len(rows), 8.0) if ctx["element"] == 0 else got["aux"][rows, capi.AUX_TARGET_X]
    ref, S = reset_sensitivity(ctx, gid, ep, aux_in, tgx)
    st = got["state"][rows].astype(np.float64)
    st[:, 3:7] = ec._sign_fix(st[:, 3:7], ref["state"][:, 3:7])
    ck.near(st, ref["state"], S["state"], what + " F_STATE")
    a = got["aux"][rows]
    wrong = [(int(rows[i]), cats[rows[i]], int(c), a[i, c], ref["aux"][i, c]) for c in EXACT_AUX for i in np.nonzero(a[:, c] != ref["aux"][:, c])[0]]
    assert not wrong, (what, wrong[:8])
    ck.near(a[:, CONT_AUX], ref["aux"][:, CONT_AUX], S["aux"][:, CONT_AUX], what + " aux")
    assert np.array_equal(got["episode"][rows], ep + 1) and np.all(got["reward_sum"][rows] == 0)
    o = obs[rows].astype(np.float64)
    ck.near(o[:, np.r_[0:135, 913:916]], ref["obs"], S["obs"], what + " obs")
    assert np.array_equal(obs[rows], got["obs"][rows])
    V, SV = perception(ref["state"], got["boxes"][rows], got["nbox"][rows], a)
    ck.rays(o[:, 135:913], V, SV, what + " rays")
    ck.near(got["foot"][rows], ref["foot"], S["foot"], what + " F_FOOT_POS")


def run_case(lib, k, io="host", kappa=KAPPA, oracle=False):
    """Run batch k through `lib` (CUDA engine or oracle) and compare every output with the statement, env by env.  Engine A
    (auto_reset 0) takes the step; engine B (auto_reset 1) takes it again and resets the envs it ends, then a masked reset of
    every third env (some of them just auto-reset).  Returns the largest error / S ratios."""
    ctx, before, cats = case(k)
    n = ctx["n"]
    gid = ctx["gid0"] + np.arange(n)
    ck = Check(kappa, oracle)
    A, B = make(lib, ctx, 0), make(lib, ctx, 1)
    try:
        slabs = [ec.Slab(x, int(io[-1])) if io.startswith("device") else None for x in (A, B)]
        c0A, c0B = A.counters(), B.counters()
        set_before(A, before); set_before(B, before)
        oA, rA, dA, recA = ec.step_io(A, before["actions"], io, slabs[0])
        fa = readback(A)
        oB, rB, dB, recB = ec.step_io(B, before["actions"], io, slabs[1])
        fb = readback(B)
        # ---- engine A: the step statement on the state read back
        post = fa["state"].astype(np.float64)
        ref, S = sensitivity(ctx, before, post)
        assert decisive(ctx, ref, before, post).all(), [(int(i), cats[i]) for i in np.nonzero(~decisive(ctx, ref, before, post))[0][:6]]
        ok = reaches(ctx, before, ref, cats, post)
        assert ok.all(), [(int(i), cats[i]) for i in np.nonzero(~ok)[0][:8]]
        done = ref["done"]
        assert np.array_equal(dA.astype(bool), done), [(int(i), cats[i], int(dA[i])) for i in np.nonzero(dA.astype(bool) != done)[0][:8]]
        assert int(fa["counters"][1] - c0A[1]) == int(done.sum()) and int(fa["counters"][0] - c0A[0]) == n
        a = fa["aux"]
        wrong = [(int(i), cats[i], int(c), a[i, c], ref["aux"][i, c]) for c in EXACT_AUX for i in np.nonzero(a[:, c] != ref["aux"][:, c])[0]]
        assert not wrong, ("aux", wrong[:8])
        ck.near(a[:, CONT_AUX], ref["aux"][:, CONT_AUX], S["aux"][:, CONT_AUX], "aux")
        ck.near(rA, ref["reward64"], S["reward"], "reward")
        assert np.all(rA[ref["bad"]] == 0)
        rs_own = (before["reward_sum"] + rA).astype(np.float32)
        assert oracle or np.array_equal(fa["reward_sum"], rs_own)
        ck.near(fa["reward_sum"], before["reward_sum"].astype(np.float64) + ref["reward64"], S["reward"] + np.spacing(rs_own), "reward_sum")
        assert np.array_equal(fa["episode"], before["episode"]) and np.array_equal(oA, fa["obs"], equal_nan=True)
        # a NaN joint angle makes the post state NaN: its new prop, rays and feet are made of it; reward, done, counters and the
        # copied blocks are checked
        fin_st = np.isfinite(post).all(1)
        ck.near(oA[:, 0:135], ref["obs"], S["obs"], "obs", rows=fin_st)
        ck.near(oA[:, 913:916], ref["tail"], S["tail"], "target block", rows=fin_st)
        assert np.array_equal(oA[:, 0:66], before["obs"][:, 33:99]) and np.array_equal(oA[:, 99:123], before["obs"][:, 111:135])
        assert np.array_equal(oA[:, 123:135], before["actions"], equal_nan=True)
        V, SV = perception(post[fin_st], fa["boxes"][fin_st], fa["nbox"][fin_st], ref["aux"][fin_st])
        ck.rays(oA[fin_st, 135:913], V, SV, "rays")
        ck.near(fa["foot"], ref["foot"], S["foot"], "F_FOOT_POS", rows=fin_st)
        # ---- engine B: the same step, then the auto-reset of the envs it ended
        assert np.array_equal(rB, rA) and np.array_equal(dB, dA)
        keep = ~done
        for key in ("state", "aux", "episode", "reward_sum", "foot"):
            assert np.array_equal(fb[key][keep], fa[key][keep], equal_nan=True), key
        assert np.array_equal(oB[keep], oA[keep], equal_nan=True)
        assert int(fb["counters"][1] - c0B[1]) == int(done.sum()) and int(fb["counters"][0] - c0B[0]) == n
        fin = np.nonzero(done)[0]
        if len(fin):
            _check_reset(ck, ctx, cats, fin, fb, oB, gid[fin], before["episode"][fin], ref["aux"][fin], "auto-reset")
        # ---- record columns: the finishing step's action, reward and done, also for envs reset in the same call
        for rec, rw, dn in ((recA, rA, dA), (recB, rB, dB)):
            if rec is not None:
                assert np.array_equal(rec[:, :12], before["actions"], equal_nan=True) and np.array_equal(rec[:, 12], rw)
                assert np.array_equal(rec[:, 13], dn.astype(np.float32))
        # ---- engine B: a masked reset of every third env, some of them reset by the step already
        mask = np.zeros(n, bool); mask[::3] = True
        o2 = B.reset(mask)
        f2 = readback(B)
        rows = np.nonzero(mask)[0]
        _check_reset(ck, ctx, cats, rows, f2, o2, gid[rows], fb["episode"][rows], fb["aux"][rows], "masked reset")
        for key in ("state", "aux", "episode", "reward_sum", "obs"):
            assert np.array_equal(f2[key][~mask], fb[key][~mask], equal_nan=True), key
        ck.ratios["n_done"] = int(done.sum())
        return ck.ratios
    finally:
        A.close(); B.close()
