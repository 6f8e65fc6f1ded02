"""fp64 statement of the strategic level's training forward (llq_hier_policy_forward_rec_strategic, csrc/llq_policy_hier.cu) and a
designed batch on which every sampled heading's clip and every code is decisive (host only, numpy float64).

The statement adds to the hierarchical statement of tests/policy_cases.py (`Hier`, `ErrorModel`, the same building blocks):
  sample        eps = sqrt(-2 log u0) cos(2 pi u1), u0 = min((r.x + 1/2) 2^-32, 0.99999994) and u1 = r.y 2^-32 formed in fp32 exactly as
                the kernel forms them (2 pi u1 too), r from Philox4x32-10 with counter (low 32 bits of the global row, 64, counter lo,
                counter hi) and key (seed lo, seed hi); a = mu + exp(logstd) eps from the UNCLIPPED heading mean
  -log p        0.5 eps^2 + logstd + 0.5 log(2 pi)
  code          the code controller on (cos, sin) of clip(a, +-float(pi)) and the commanded speed, argmax code, decoder on that code
  value tower   arrays 2-50: prop 135 -> 128 | perception encoder (no target) 88 -> 64 -> 128 | game vector 29 -> 64 -> 64 -> 128,
                concatenated 384 -> 256, layer-norm LSTM (40-48) on its own state [c, h] (floats 128-191 of the row's 192), V = h W49 + b50
The error model perturbs the log, the square root, the cosine and the product of the draw, exp(logstd), the sum mu + e eps and the sum of
-log p.

Decisiveness.  A row is decisive when its code's logit clears the runner-up's by more than 4 kappa S_gap and its raw heading is more
than 4 kappa S_heading from both clip kinks +-float(pi).  The batch is launched at two counters (COUNTERS): at the first, found by
searching the counter, one row's u0 hits the clamp.  Rows that are not decisive at both counters get a new observation.
"""
import functools

import numpy as np

import policy_cases as pc
from lifelike_agility_and_play_b200.policy_epmc import hier_role_arrays, random_weights, strategic_train_role_arrays

KAPPA = pc.KAPPA_HIER
N = pc.HIER_N
SEED = (7 << 32) + 12345                     # non-zero high words: a dropped high word changes every draw
COUNTER_BASE = (3 << 32) + 17
ROW_GID0 = 2 ** 32 - 500                     # rows 500.. wrap to global ids 0.. in the low 32 bits of the Philox counter
CLAMP_R = 2 ** 32 - 128                      # r.x >= CLAMP_R: (float)r + 0.5f rounds to 2^32, u0 to 1.0f
Q_HEADING = 64
LOGSTD = np.log(0.6)                         # heading std 0.6: samples cross the clip kinks both ways, codes move with the sample
TRAIN_ARRAYS = strategic_train_role_arrays()
F = np.float32


def draws(global_rows, seed, counter):
    """(r.x, u0 fp32, u1 fp32, 2 pi u1 fp32) of the heading draw of each global row."""
    g = np.asarray(global_rows, np.int64).astype(np.uint64) & pc.M32
    c = pc.philox4x32(g, Q_HEADING, counter & 0xFFFFFFFF, counter >> 32, seed & 0xFFFFFFFF, seed >> 32)
    scale = F(2.3283064365386963e-10)
    u0 = np.minimum((c[0].astype(F) + F(0.5)) * scale, F(0.99999994))
    u1 = c[1].astype(F) * scale
    return c[0], u0, u1, F(6.283185307179586) * u1


def eps_of(global_rows, seed, counter, em=pc.REF):
    _, u0, _, ang = draws(global_rows, seed, counter)
    rad = em.rel(np.sqrt(em.rel(-2.0 * np.log(u0.astype(np.float64)))))
    return em.rel(rad * em.rel(np.cos(ang.astype(np.float64))))


def sample(mu, logstd, eps, em):
    """(raw heading a, -log p) of the Gaussian head."""
    e = em.rel(np.exp(logstd))
    a = em.add(mu + e * eps, np.abs(mu) + np.abs(e * eps))
    c = 0.5 * np.log(2.0 * np.pi)
    t = 0.5 * eps * eps
    return a, em.add(t + logstd + c, t + abs(logstd) + c)


def heading_trunk(net, obs, p, st, em):
    """(mu before the clip, new [c, h]) of the heading controller; st [n, 64] already wiped."""
    r = net.r
    pe = pc.fc(p, r[56], r[57], em, "relu")
    pcp = pc.fc(pc.perception(obs, r[58:82], em), r[82], r[83], em, "relu")
    ge = pc.fc(pc.fc(obs[:, pc.GAME_COLS], r[84], r[85], em, "relu"), r[86], r[87], em, "relu")
    e = pc.fc(np.concatenate([pe, pcp, ge], axis=1), r[88], r[89], em, "relu")
    c, h = pc.lstm_step(e, st[:, :32], st[:, 32:], r[90:99], em)
    return pc.fc(h, r[99], r[100], em)[:, 0], np.concatenate([c, h], axis=1)


def code_trunk(net, obs, p, ang, st, em):
    """(h, new [c, h]) of the code controller on the clipped heading `ang`; st [n, 64] already wiped."""
    r = net.r
    tgt = np.stack([em.rel(np.cos(ang)), em.rel(np.sin(ang)), obs[:, 964]], axis=1)
    pe = pc.fc(p, r[2], r[3], em, "relu")
    t = pc.fc(tgt, r[28], r[29], em, "relu")
    ce = pc.fc(np.concatenate([t, pc.perception(obs, r[4:28], em)], axis=1), r[30], r[31], em, "relu")
    e = pc.fc(np.concatenate([pe, ce], axis=1), r[32], r[33], em, "relu")
    c, h = pc.lstm_step(e, st[:, :32], st[:, 32:], r[34:43], em)
    return h, np.concatenate([c, h], axis=1)


def value_tower(wv, obs, p, st, em):
    """(V, new [c, h]) of the strategic value tower; st [n, 64] already wiped; wv = the 50 arrays of the training table."""
    v1 = pc.fc(p, wv[0], wv[1], em, "relu")
    v2 = pc.fc(pc.fc(pc.perception(obs, wv[2:26], em), wv[26], wv[27], em, "relu"), wv[28], wv[29], em, "relu")
    v3 = obs[:, pc.GAME_COLS]
    for k in range(3):
        v3 = pc.fc(v3, wv[30 + 2 * k], wv[31 + 2 * k], em, "relu")
    v4 = pc.fc(np.concatenate([v1, v2, v3], axis=1), wv[36], wv[37], em, "relu")
    c, h = pc.lstm_step(v4, st[:, :32], st[:, 32:], wv[38:47], em)
    return pc.fc(h, wv[47], wv[48], em)[:, 0], np.concatenate([c, h], axis=1)


class Trunks:
    """The counter-independent parts (heading mean, value tower) for the reference and R_DRAWS error-model draws."""

    def __init__(self, w, obs, state, done, draws_=pc.R_DRAWS):
        self.net = pc.Hier(w)
        self.wv = [np.asarray(w[i], np.float64) for i in TRAIN_ARRAYS]
        self.logstd = float(self.wv[49].reshape(-1)[0])
        self.obs = np.asarray(obs[:, :965], np.float64)
        keep = (np.asarray(done) == 0)[:, None] if done is not None else np.ones((len(obs), 1), bool)
        self.st = np.where(keep, np.asarray(state, np.float64), 0.0)
        self.runs = []
        for k in range(draws_ + 1):
            em = pc.REF if k == 0 else pc.ErrorModel(8000 + k)
            p = pc.normalise(self.obs[:, :135], self.net.r[0][0], self.net.r[1][0], em)
            mu, sh = heading_trunk(self.net, self.obs, p, self.st[:, 0:64], em)
            v, sv = value_tower(self.wv, self.obs, p, self.st[:, 128:192], em)
            self.runs.append(dict(p=p, mu=mu, sh=sh, value=v, sv=sv, em=em))

    def take(self, rows):
        out = object.__new__(Trunks)
        out.net, out.wv, out.logstd = self.net, self.wv, self.logstd
        out.obs, out.st = self.obs[rows], self.st[rows]
        out.runs = [dict({k: (v[rows] if isinstance(v, np.ndarray) else v) for k, v in r.items()}) for r in self.runs]
        return out


def train_eval(tr, global_rows, seed, counter):
    """Reference outputs (code, gap, logits, heading (raw), eps, neglogp, value, actions, state [n, 192]) and sensitivities S of the
    strategic training forward; the draws keep the reference's code, as the kernel does on a decisive row."""
    net = tr.net
    same = pc.same_columns(np.vstack([net.r[43], net.r[44][None]]))

    def run(k, em):
        rd = tr.runs[k]
        eps = eps_of(global_rows, seed, counter, em)
        a, nl = sample(rd["mu"], tr.logstd, eps, em)
        h, sc = code_trunk(net, tr.obs, rd["p"], np.clip(a, -pc.PI32, pc.PI32), tr.st[:, 64:128], em)
        return dict(p=rd["p"], eps=eps, heading=a, neglogp=nl, logits=net.logits(h, em), value=rd["value"],
                    state=np.concatenate([rd["sh"], sc, rd["sv"]], axis=1))
    r0 = run(0, pc.REF)
    code = r0["logits"].argmax(1)
    ref = dict(code=code, gap=pc.code_gap(r0["logits"], code, same, -1.0), actions=net.actions(r0["p"], code, pc.REF), mu=tr.runs[0]["mu"],
               **{k: r0[k] for k in ("eps", "heading", "neglogp", "logits", "value", "state")})
    S = {k: np.zeros_like(ref[k], np.float64) for k in ("gap", "heading", "neglogp", "value", "actions", "state")}
    for i in range(1, len(tr.runs)):
        em = pc.ErrorModel(9000 + i)
        g = run(i, em)
        got = dict(gap=pc.code_gap(g["logits"], code, same, -1.0), heading=g["heading"], neglogp=g["neglogp"], value=g["value"],
                   actions=net.actions(g["p"], code, em), state=g["state"])
        for k in S:
            S[k] = np.maximum(S[k], np.abs(got[k] - ref[k]))
    return ref, S


def mean_heading_codes(tr):
    """The argmax code each row would take with the clipped heading MEAN (the deterministic forward's), fp64 reference."""
    r0 = tr.runs[0]
    h, _ = code_trunk(tr.net, tr.obs, r0["p"], np.clip(r0["mu"], -pc.PI32, pc.PI32), tr.st[:, 64:128], pc.REF)
    return tr.net.logits(h, pc.REF).argmax(1)


def decisive(ref, S, margin=1.0):
    bar = 4.0 * KAPPA * margin
    kink = np.minimum(np.abs(ref["heading"] - pc.PI32), np.abs(ref["heading"] + pc.PI32))
    return (ref["gap"] > bar * S["gap"]) & (kink > bar * S["heading"])


def design_weights(seed):
    """Random weights of the shipped architecture with the heading mean spread past +-pi both ways, logits spread over many codes and the
    heading logstd at log 0.6."""
    rng = np.random.default_rng(seed)
    w = [a.copy() for a in random_weights(True, seed + 1)]
    roles = hier_role_arrays(True)
    obs = np.stack([pc._hier_row(rng, "random", 965) for _ in range(64)])
    st = pc.hier_random_state(rng, 64, 192)
    w[roles[99]] = (40.0 * w[roles[99]]).astype(np.float32)
    w[roles[100]] = np.zeros_like(w[roles[100]])
    tr = Trunks(w, obs, st, np.zeros(64, np.uint8), draws_=0)
    w[roles[100]] = np.array([-np.median(tr.runs[0]["mu"])], np.float32)
    h, _ = code_trunk(tr.net, tr.obs, tr.runs[0]["p"], np.zeros(64), tr.st[:, 64:128], pc.REF)
    w[roles[43]] = (4.0 * w[roles[43]]).astype(np.float32)
    w[roles[44]] = (-(h.mean(0) @ w[roles[43]]) + 0.1 * w[roles[44]]).astype(np.float32)
    w[96] = np.array([[LOGSTD]], np.float32)
    return w


def search_clamp_counter(n, start):
    """First counter >= start at which one of the rows ROW_GID0 + 0..n-1 draws r.x >= CLAMP_R (u0 on the clamp); (counter, row)."""
    gid = (ROW_GID0 + np.arange(n)).astype(np.uint64) & pc.M32
    step = 4096
    for c0 in range(start, start + 64 * step, step):
        cs = np.arange(c0, c0 + step, dtype=np.uint64)
        rx = pc.philox4x32(gid[None, :], Q_HEADING, (cs & pc.M32)[:, None], (cs >> np.uint64(32))[:, None], SEED & 0xFFFFFFFF, SEED >> 32)[0]
        hit = np.argwhere(rx >= CLAMP_R)
        if len(hit):
            k, i = hit[0]
            return int(cs[k]), int(i)
    raise AssertionError("no clamped draw found")


def build_train_case(seed=0, n=N):
    """(w, obs [n, 965], state [n, 192], done, counters, info): every row decisive at both counters; info names the clamp row."""
    rng = np.random.default_rng(seed + 31)
    w = design_weights(seed)
    cats = [pc.HIER_CATS[i % 3] for i in range(n)]
    obs = np.stack([pc._hier_row(rng, c, 965) for c in cats])
    state = pc.hier_random_state(rng, n, 192)
    done = pc.DONE_BYTES[rng.integers(0, 4, n)]
    done[:8] = [0, 1, 2, 255, 0, 0, 255, 2]
    gid = ROW_GID0 + np.arange(n)
    c1, i1 = search_clamp_counter(n, COUNTER_BASE)
    counters = (c1, COUNTER_BASE + 1)
    rows = np.arange(n)
    for _ in range(60):
        tr = Trunks(w, obs[rows], state[rows], done[rows])
        bad = set()
        for c in counters:
            ref, S = train_eval(tr, gid[rows], SEED, c)
            bad |= set(rows[~decisive(ref, S)].tolist())
        if not bad:
            if len(rows) == n:
                return w, obs, state, done, counters, dict(clamp=(c1, i1))
            rows = np.arange(n)                  # confirm on the whole batch
            continue
        rows = np.array(sorted(bad))
        for i in rows:
            obs[i] = pc._hier_row(rng, cats[i], 965)
    raise AssertionError("strategic training rows stay undecided")


def reaches(w, obs, state, done, counters, info, evals, mean_codes):
    """What the batch is designed to reach, each entry a list of per-row (or per-batch) flags of which one must hold."""
    c1, i1 = info["clamp"]
    gid = ROW_GID0 + np.arange(len(obs))
    out = {}
    for (ref, S) in evals:
        a = ref["heading"]
        out.setdefault("heading_inside", []).extend((np.abs(a) < pc.PI32).tolist())
        out.setdefault("heading_above_pi", []).extend((a > pc.PI32).tolist())
        out.setdefault("heading_below_-pi", []).extend((a < -pc.PI32).tolist())
        out.setdefault("mean_inside_sample_outside", []).extend(((np.abs(ref["mu"]) < pc.PI32) & (np.abs(a) > pc.PI32)).tolist())
        out.setdefault("|eps|>3", []).extend((np.abs(ref["eps"]) > 3.0).tolist())
        out.setdefault("code_differs_from_mean_heading_code", []).extend((ref["code"] != mean_codes).tolist())
        out.setdefault("code_equals_mean_heading_code", []).extend((ref["code"] == mean_codes).tolist())
    rx, u0, _, _ = draws(gid[i1:i1 + 1], SEED, c1)
    out["u0_clamped"] = [bool(int(rx[0]) >= CLAMP_R and u0[0] == F(0.99999994) and counters[0] == c1)]
    out["done_bytes_on_nonzero_states"] = [set(np.unique(done).tolist()) == {0, 1, 2, 255} and
                                           all(bool((np.abs(state[:, k:k + 64]) > 0).any(1).all()) for k in (0, 64, 128))]
    out["high_words"] = [SEED >> 32 != 0 and all(c >> 32 != 0 for c in counters)]
    out["row_gid_wraps"] = [bool(((gid >> 32) == 0).any() and ((gid >> 32) == 1).any())]
    return out


@functools.lru_cache(maxsize=None)
def train_case():
    """The designed batch with its reference and sensitivities at both counters and the mean-heading codes (built once per session)."""
    w, obs, state, done, counters, info = build_train_case()
    tr = Trunks(w, obs, state, done)
    gid = ROW_GID0 + np.arange(len(obs))
    evals = [train_eval(tr, gid, SEED, c) for c in counters]
    return w, obs, state, done, counters, info, evals, mean_heading_codes(tr)


RECUR_N, RECUR_STEPS, NULL_DONE_STEP = 300, 4, 2


def recurrence_case(w, seed=0, n=RECUR_N, steps=RECUR_STEPS):
    """Observations, done bytes and counters of `steps` recurrent steps from a non-zero state, every row decisive with a margin of 2
    along the fp64 chain (the GPU test feeds each step's reference the kernel's incoming state; the margin covers the difference)."""
    rng = np.random.default_rng(seed + 91)
    cats = [pc.HIER_CATS[i % 3] for i in range(n)]
    state = pc.hier_random_state(rng, n, 192)
    state0 = state.copy()
    gid = ROW_GID0 + np.arange(n)
    obs_all, done_all, ctr = [], [], []
    for s in range(steps):
        obs = np.stack([pc._hier_row(rng, c, 965) for c in cats])
        done = np.zeros(n, np.uint8) if s == NULL_DONE_STEP else pc.DONE_BYTES[(np.arange(n) + s) % 4]
        counter = COUNTER_BASE + 1000 + s
        rows = np.arange(n)
        for _ in range(60):
            ref, S = train_eval(Trunks(w, obs[rows], state[rows], done[rows]), gid[rows], SEED, counter)
            bad = rows[~decisive(ref, S, 2.0)]
            if not len(bad):
                if len(rows) == n:
                    break
                rows = np.arange(n)
                continue
            rows = bad
            for i in bad:
                obs[i] = pc._hier_row(rng, cats[i], 965)
        else:
            raise AssertionError("recurrence rows stay undecided")
        obs_all.append(obs)
        done_all.append(done)
        ctr.append(counter)
        state = ref["state"].astype(np.float32)
    return state0, obs_all, done_all, ctr
