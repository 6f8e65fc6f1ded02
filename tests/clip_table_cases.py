"""Designed batches for the prioritized clip table and the auto-reset draw at motion-library sizes: thousands to tens of thousands
of clips (host only, numpy float64).  The statement is tests/episode_cases.py's (`table`, `uniforms`, `draw`, `reset_statement`);
this module only builds inputs at sizes that module's category builder cannot reach (its plate, clock and termination categories
need clips of 300 frames and more, which would take gigabytes at these clip counts).

The reset kernel holds the clip table (8 B per clip) in dynamic shared memory.  Without the opt-in it fits 3,902 clips beside the
kernel's 17,936 B of static tables (48 kB per block); with it, (232,448 - 17,936) / 8 = C_MAX on an H100.  The sizes straddle the
first limit and reach the second.

Step batches (`build`, run by episode_cases.run_case): every env either finishes (`finish`: displaced 2 m from its target, so dp > 1)
or tracks its target exactly (`track`).  The finishers use many different clips spread over the table, env 0 and env N - 1 share
one (the highest env wins it), and they sit in many different 32-env blocks of the reset kernel, so every block's rebuild of the
table is compared.  F_AVG_REWARD is set before the step so that the weights (1 - avg)^factor span more than 12 decades and include
zero-weight clips (avg = 1); episode_cases.design_edges then moves cdf edges 1e-8..1e-6 to either side of finishers' draws: the
first and the last interval, an edge just above clip 3,902 and one in the last 1 % of the table.

Reset batches (`reset_batch`): `llq_reset` (mode 1, no table update) on an exact table -- five positive weights, dyadics of 33
bits whose sums are exact in fp64, and zero weights elsewhere -- on which the cdf passes exactly through the u1 of designated envs and stays flat over zero-weight clips after
them: the first clip with cdf > u1 is the first positive clip past the flat run, the first with cdf >= u1 the edge clip itself.
Then `llq_reset_to` (mode 2) at clip ids 0, 3,902, 3,903 and C - 1.

Clips are margin + 3 .. margin + 40 frames long (the shortest `llq_load_mocap` accepts), so C_MAX clips take 0.6 GB as fp64.
"""
import numpy as np

import episode_cases as ec

C_MAX = 26814              # the largest table the engine accepts on an H100 (tests/test_clip_table_cases_gpu.py reads it back)
FRAME_DT = 1.0 / 120.0     # synthetic_mocap's
FRAMES = (ec.margin(FRAME_DT) + 3, ec.margin(FRAME_DT) + 40)
SIZES = (3902, 3903, 8192, C_MAX)

# step batches: (n envs, n clips, sub-steps, prioritized_sample_factor, global_env_offset, reward weights)
CASES = [
    (17, 3902, 10, 3.0, 0, ec.W_DEFAULT),
    (4097, 3902, 10, 3.0, 0, ec.W_DEFAULT),
    (1, 3903, 10, 3.0, 0, ec.W_DEFAULT),
    (4097, 3903, 10, 2.5, 0, ec.W_DEFAULT),
    (17, 8192, 10, 3.0, 2 ** 32 - 5, ec.W_DEFAULT),
    (4097, 8192, 10, 3.0, 0, ec.W_DEFAULT),
    (1, C_MAX, 10, 3.0, 0, ec.W_DEFAULT),
    (17, C_MAX, 10, 2.5, 0, ec.W_DEFAULT),
    (4097, C_MAX, 10, 3.0, 0, ec.W_DEFAULT),
]
ZERO_RUN = range(3898, 3908)   # zero-weight clips across the old limit


def edge_targets(C):
    """the designed inner edges: just above clip 3,902 and in the last 1 % of the table"""
    return ([3903] if C > 3906 else []) + [C - 2 - C // 200]


def build(case):
    """(ctx, before, categories, designed) of a step batch, the form episode_cases.run_case takes; deterministic"""
    ctx = ec.context(case, FRAMES)
    n, C = ctx["n"], ctx["mc"].n_clips
    rng = np.random.default_rng(ec.SEED + 31 * C + n)
    nfm = ctx["nf"] - ctx["m"]
    ms = ctx["max_steps"]
    fin = set(ec._designated_indices(n))
    if n > 32:
        fin |= {int(i) for i in np.flatnonzero(rng.random(n) < 0.5)}
    fin = sorted(fin)
    cats = ["finish" if i in fin else "track" for i in range(n)]
    clip = np.zeros(n, np.int64)
    # finishers on distinct clips with max_steps >= 4 (so avg = reward_sum / max_steps < 1), env N - 1 on env 0's clip; a lone env
    # on the last such clip
    targets = edge_targets(C)
    edge_pairs = {0, 1, C - 2, C - 1} | {c for j in targets for c in (j, j + 1)}          # kept free of finishers for design_edges
    long_ = np.array([c for c in np.flatnonzero(nfm >= 10) if c not in edge_pairs])
    clip[fin] = rng.choice(long_, len(fin), replace=False) if n > 1 else long_[-1]
    clip[n - 1] = clip[0]
    free = np.flatnonzero(nfm >= 5)
    track = [i for i in range(n) if i not in fin]
    clip[track] = free[rng.integers(len(free), size=len(track))]
    # the cursor inside the clip, at least 3 frames in (the time before the last sub-step stays positive) and not ended
    fid = np.array([int(rng.integers(3, nfm[c] - 1)) for c in clip])
    t0 = np.array([ec._t0_for(ctx, rng, c, f) for c, f in zip(clip, fid)])
    time, fid, frac = ec.clock(t0, ctx["substeps"], ctx["sim_dt"], ctx["mc"].frame_dt, ctx["nf"][clip], ctx["m"])
    kin = ec.mocap_state(ctx["frames"], ctx["off"][clip] + fid, frac, ctx["mc"].frame_dt)
    st = np.stack([ec._design_state(kin[i], cats[i], rng) for i in range(n)])
    ep = np.where(rng.random(n) < 0.5, rng.integers(0, 1000, n), rng.integers(2 ** 32, 2 ** 40, n)).astype(np.int64)
    rs = np.where(np.isin(np.arange(n), fin), rng.uniform(0.0, 0.5, n) * ms[clip], rng.uniform(0.0, 60.0, n)).astype(np.float32)
    avg = 1.0 - 10.0 ** rng.uniform(-5.0, 0.0, C)
    avg[::50] = 1.0
    avg[[c for c in ZERO_RUN if c < C]] = 1.0
    before = dict(clip=clip, time=t0, ob_id=np.zeros(n, np.int64), episode=ep, obs=rng.normal(0, 1, (n, 207)).astype(np.float32),
                  actions=rng.uniform(-1, 1, (n, 12)).astype(np.float32), state=st, reward_sum=rs, avg=avg)
    ref = ec.step_statement(ctx, before, st.astype(np.float64))
    before["avg"], designed = ec.design_edges(ctx, before, ref, rng, targets=targets)
    return ctx, before, cats, designed


_BUILT = {}


def case(k):
    if k not in _BUILT:
        _BUILT.clear()                      # one table of tens of thousands of clips at a time
        _BUILT[k] = build(CASES[k])
    return _BUILT[k]


# ------------------------------------------------------------------------------------------------------------ reset batches
def reset_batch(C, n=64):
    """(ctx, F_AVG_REWARD, F_EPISODE_ID, {env: edge clip}, (clip, time) of llq_reset_to): an exact table with factor 1 on which the
    cdf passes exactly through the u1 of envs 0, 31, 32 and N - 1, each edge followed by zero-weight clips"""
    ctx = ec.context((n, C, 10, 1.0, 0, ec.W_DEFAULT), FRAMES)
    rng = np.random.default_rng(ec.SEED + 7 * C + n)
    ep = rng.integers(0, 2 ** 40, n).astype(np.int64)
    tied = [0, 31, 32, n - 1]
    u1, _ = ec.uniforms(ctx["seed"], ctx["gid0"] + np.array(tied), ep[tied])
    order = np.argsort(u1)
    ends = [C // 8, min(3902, C - 400), min(4000, C - 200), C - 2 - C // 200]     # the edge clips, increasing, one per tied env by u1
    w = np.zeros(C)
    prev = 0.0
    edges = {}
    for r, k in enumerate(order):             # one clip per segment of the cdf: a dyadic of 33 bits, so every sum is exact
        w[ends[r]] = u1[k] - prev
        edges[tied[k]] = ends[r]
        prev = u1[k]
    w[C - 1] = 1.0 - prev
    avg = 1.0 - w                             # factor 1: the weight is 1 - avg, exact for these powers of two
    assert np.array_equal(1.0 - avg, w)
    rc = np.resize(np.array([c for c in (0, 3902, 3903, C - 1) if c < C]), n)
    nfm = ctx["nf"][rc] - ctx["m"] - 1
    rt = rng.uniform(0.0, 1.0, n) * ctx["mc"].frame_dt * nfm
    return ctx, avg, ep, edges, (rc, rt)


def reset_draw(ctx, avg, gid, ep):
    """the statement's draw on the table avg, as llq_reset (no table update) makes it"""
    _, _, cdf, _ = ec.table(ctx, np.zeros(0, bool), np.zeros(0, np.int64), np.zeros(0, np.float32), avg)
    return ec.draw(ctx, cdf, gid, ep), cdf


def run_resets(lib, C, kappa=ec.KAPPA, oracle=False):
    """llq_reset on the exact table (draws, F_SAMPLE_PROB, F_AVG_REWARD at full length, reset rows), then llq_reset_to at clip ids
    0, 3,902, 3,903 and C - 1, against the statement; returns the largest error / S ratios.  The engine's reset kernel derives the
    table from F_AVG_REWARD; the oracle draws from F_SAMPLE_PROB as the last step left it, so it is handed that as well."""
    from lifelike_agility_and_play_b200 import _capi as capi
    ctx, avg, ep, edges, (rc, rt) = reset_batch(C)
    n = ctx["n"]
    e = ec.make(lib, ctx, 1)
    try:
        e.set(capi.F_AVG_REWARD, avg)
        if oracle:
            e.set(capi.F_SAMPLE_PROB, 1.0 - avg)
        e.set(capi.F_EPISODE_ID, ep)
        obs = e.reset()
        f = ec.readback(e)
        (clip, t0, fid, frac, u1), cdf = reset_draw(ctx, avg, ctx["gid0"] + np.arange(n), ep)
        for env, j in edges.items():           # the tie: cdf[j] == u1 exactly, then zero-weight clips, then the drawn clip
            assert cdf[j] == u1[env] and clip[env] > j + 1 and np.all(cdf[j:clip[env]] == u1[env]), (env, j, clip[env])
        assert np.array_equal(f["clip"], clip), [(i, int(f["clip"][i]), int(clip[i])) for i in np.nonzero(f["clip"] != clip)[0][:6]]
        assert np.array_equal(f["time"], t0) and np.array_equal(f["episode"], ep + 1)
        assert np.array_equal(f["avg"], avg) and np.array_equal(f["prob"], 1.0 - avg)     # exact table: p = w exactly
        ratios = ec.reset_ratios(ctx, f["state"], f["kin"], obs, clip, fid, frac, kappa)
        obs = e.reset_to(rc.astype(np.int32), rt)
        f = ec.readback(e)
        assert np.array_equal(f["clip"], rc) and np.array_equal(f["time"], rt) and np.array_equal(f["episode"], ep + 1)
        fid = np.floor(rt / ctx["mc"].frame_dt).astype(np.int64)
        frac = (rt - fid * ctx["mc"].frame_dt) / ctx["mc"].frame_dt
        ratios.update({k + "_to": v for k, v in ec.reset_ratios(ctx, f["state"], f["kin"], obs, rc, fid, frac, kappa).items()})
        assert np.array_equal(f["avg"], avg) and np.array_equal(f["prob"], 1.0 - avg)
        return ratios
    finally:
        e.close()
