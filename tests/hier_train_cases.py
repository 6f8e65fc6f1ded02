"""fp64 statement of the environmental level's training forward (llq_hier_policy_forward_rec, csrc/llq_policy_hier.cu) and a designed
batch on which every sampled code is decisive (host only, numpy float64).

The statement adds to the hierarchical statement of tests/policy_cases.py (`Hier`, `ErrorModel`, the same building blocks):
  value tower   arrays 2-46: v1 = relu(p W2 + b3) | ce = usr_cmd_encoder(4-31) -> v2 = relu(ce W32 + b33); v3 = relu([v1 | v2] W34 + b35);
                layer-norm LSTM(36-44) on its own state [c, h] (the second half of the row's 128 floats, wiped like the first); V = h W45 + b46
  sample        code = argmax_j (l_j + g_j), g = -log(-log u), u = min((r + 1/2) 2^-32, 0.99999994) formed in fp32 exactly as the
                kernel forms it, r from Philox4x32-10 with counter (low 32 bits of the global row, q, counter lo, counter hi) and key
                (seed lo, seed hi), q = 0..63 -> logits 4q..4q+3
  -log p        (m - l_code) + log sum_j exp(l_j - m), m the largest logit
  actions       the decoder on the SAMPLED code
The error model perturbs each log of g, the sum l + g, every exp, the sum and the log of -log p, and the two subtractions.

Decisiveness.  A row's sampled code is decisive when its l + g clears the runner-up's by more than 4 kappa S_gap.  The batch is
launched at two counters (COUNTERS): at the first, one row's winning column draws r >= 2^32 - 128 (u hits the clamp, g = 16.6);
at the second, one row's clamped column loses (without the clamp its g would be +inf and it would win).  Every row is decisive at
both counters; rows that are not get a new observation.
"""
import functools

import numpy as np

import policy_cases as pc
from lifelike_agility_and_play_b200.policy_epmc import hier_role_arrays, random_weights

KAPPA = pc.KAPPA_HIER
N = pc.HIER_N
SEED = (7 << 32) + 12345                     # non-zero high words: a dropped high word changes every draw
COUNTER_BASE = (3 << 32) + 17
ROW_GID0 = 2 ** 32 - 500                     # rows 500.. wrap to global ids 0.. in the low 32 bits of the Philox counter
CLAMP_R = 2 ** 32 - 128                      # r >= CLAMP_R: (float)r + 0.5f rounds to 2^32, u to 1.0f
LOGIT_GAIN = 16.0                            # logits spread by ~4 per row: rare codes (p < 1e-3), clamped columns that lose
OFFSET_GAIN = 400.0                          # one LSTM unit adds a row-wide offset of up to +-150 to every logit of the row
VALUE_ARRAYS = hier_role_arrays(False, value_tower=True)


def draws(global_rows, seed, counter):
    """r [n, 256] (uint64 holding uint32) and the fp32 u the kernel forms from it."""
    g = (np.asarray(global_rows, np.int64).astype(np.uint64) & pc.M32)[:, None]
    q = np.arange(64, dtype=np.uint64)[None, :]
    c = pc.philox4x32(g, q, counter & 0xFFFFFFFF, counter >> 32, seed & 0xFFFFFFFF, seed >> 32)
    r = np.stack(c, axis=2).reshape(len(g), 256)
    f = np.float32
    u = np.minimum((r.astype(f) + f(0.5)) * f(2.0 ** -32), f(0.99999994))
    return r, u


def uniforms(global_rows, seed, counter):
    return draws(global_rows, seed, counter)[1]


def gumbel(u, em):
    return em.rel(-np.log(em.rel(-np.log(np.asarray(u, np.float64)))))


def neglogp(lg, code, em):
    m = lg.max(1)
    s = em.rel(np.exp(em.add(lg - m[:, None], np.abs(lg - m[:, None]))))
    tot = em.add(s.sum(1), s.sum(1))
    a = em.add(m - lg[np.arange(len(code)), code], np.abs(m - lg[np.arange(len(code)), code]))
    ls = em.rel(np.log(tot))
    return em.add(a + ls, np.abs(a) + np.abs(ls))


def value_tower(wv, obs, p, state, done, em):
    """(V, new [c, h]) of the value tower; state [n, 64], wiped where done != 0."""
    keep = (np.asarray(done) == 0)[:, None] if done is not None else np.ones((len(obs), 1), bool)
    st = np.where(keep, np.asarray(state, np.float64), 0.0)
    v1 = pc.fc(p, wv[0], wv[1], em, "relu")
    t = pc.fc(obs[:, 913:916], wv[26], wv[27], em, "relu")
    ce = pc.fc(np.concatenate([t, pc.perception(obs, wv[2:26], em)], axis=1), wv[28], wv[29], em, "relu")
    v2 = pc.fc(ce, wv[30], wv[31], em, "relu")
    v3 = pc.fc(np.concatenate([v1, v2], axis=1), wv[32], wv[33], em, "relu")
    c, h = pc.lstm_step(v3, st[:, :32], st[:, 32:], wv[34:43], em)
    return pc.fc(h, wv[43], wv[44], em)[:, 0], np.concatenate([c, h], axis=1)


def _keys(lg, u, em):
    g = gumbel(u, em)
    return em.add(lg + g, np.abs(lg) + np.abs(g))


def _gap(keys, code):
    k = keys.copy()
    win = k[np.arange(len(code)), code].copy()
    k[np.arange(len(code)), code] = -np.inf
    return win - k.max(1)


class Trunks:
    """The parts before the noise (code trunk, logits, value tower) for the reference and R_DRAWS error-model draws."""

    def __init__(self, w, obs, state, done, draws_=pc.R_DRAWS):
        net = pc.Hier(w)
        wv = [np.asarray(w[i], np.float64) for i in VALUE_ARRAYS]
        obs64 = np.asarray(obs[:, :916], np.float64)
        self.runs = []
        for k in range(draws_ + 1):
            em = pc.REF if k == 0 else pc.ErrorModel(8000 + k)
            t = net.trunk(obs, state[:, :64], done, em)
            v, vs = value_tower(wv, obs64, t["p"], state[:, 64:], done, em)
            self.runs.append(dict(p=t["p"], logits=net.logits(t["h"], em), value=v, state=np.concatenate([t["state"], vs], axis=1), em=em))
        self.net = net

    def take(self, rows):
        out = object.__new__(Trunks)
        out.net = self.net
        out.runs = [dict({k: (v[rows] if isinstance(v, np.ndarray) else v) for k, v in r.items()}) for r in self.runs]
        return out

    def put(self, rows, other):
        for a, b in zip(self.runs, other.runs):
            for k, v in a.items():
                if isinstance(v, np.ndarray):
                    v[rows] = b[k]


def train_eval(trunks, u):
    """Reference outputs (code, keys, gap, logits, neglogp, value, actions, state) and sensitivities S of the training forward from
    the uniforms u [n, 256]; the draws keep the reference's code, as the kernel does on a decisive row."""
    r0 = trunks.runs[0]
    keys = _keys(r0["logits"], u, pc.REF)
    code = keys.argmax(1)
    ref = dict(code=code, keys=keys, logits=r0["logits"], gap=_gap(keys, code), neglogp=neglogp(r0["logits"], code, pc.REF), value=r0["value"],
               actions=trunks.net.actions(r0["p"], code, pc.REF), state=r0["state"])
    S = {k: np.zeros_like(ref[k], np.float64) for k in ("gap", "neglogp", "value", "actions", "state")}
    for i, rd in enumerate(trunks.runs[1:]):
        em = pc.ErrorModel(9000 + i)
        got = dict(gap=_gap(_keys(rd["logits"], u, em), code), neglogp=neglogp(rd["logits"], code, em), value=rd["value"],
                   actions=trunks.net.actions(rd["p"], code, em), state=rd["state"])
        for k in S:
            S[k] = np.maximum(S[k], np.abs(got[k] - ref[k]))
    return ref, S


def decisive(ref, S, margin=1.0):
    return ref["gap"] > 4.0 * KAPPA * margin * S["gap"]


def design_weights(seed):
    """Random weights of the shipped architecture with logits spread wide (LOGIT_GAIN) and a row-wide offset carried by one LSTM unit."""
    rng = np.random.default_rng(seed)
    w = [a.copy() for a in random_weights(False, seed + 1)]
    roles = hier_role_arrays(False)
    obs = np.stack([pc._hier_row(rng, "random", 916) for _ in range(64)])
    h = pc.Hier(w).trunk(obs, pc.hier_random_state(rng, 64, 64), np.zeros(64, np.uint8), pc.REF)["h"]
    W = LOGIT_GAIN * np.asarray(w[roles[43]], np.float64)
    k = int(np.argmax(h.std(0)))
    W[k] += OFFSET_GAIN
    w[roles[43]] = W.astype(np.float32)
    w[roles[44]] = (-(h.mean(0) @ W)).astype(np.float32)
    return w


def _search_counter(trunks, start, want_win, rows_ok):
    """First counter >= start at which a row of rows_ok has a clamped draw that wins (want_win) / loses decisively."""
    n = len(trunks.runs[0]["value"])
    gid = ROW_GID0 + np.arange(n)
    for counter in range(start, start + 20000):
        r, u = draws(gid, SEED, counter)
        hit_rows, hit_cols = np.nonzero(r >= CLAMP_R)
        for i, c in zip(hit_rows, hit_cols):
            if not rows_ok[i]:
                continue
            keys = _keys(trunks.runs[0]["logits"][i:i + 1], u[i:i + 1], pc.REF)[0]
            win = int(keys.argmax())
            if want_win and win == c:
                return counter, int(i), int(c)
            if not want_win and win != c and keys[win] - keys[c] > 1.0:
                return counter, int(i), int(c)
    raise AssertionError("no clamped draw found")


def build_train_case(seed=0, n=N):
    """(w, obs [n, 916], state [n, 128], done, counters, info): every row decisive at both counters; info names the clamp rows."""
    rng = np.random.default_rng(seed + 31)
    w = design_weights(seed)
    cats = [pc.HIER_CATS[i % 3] for i in range(n)]
    obs = np.stack([pc._hier_row(rng, c, 916) for c in cats])
    state = pc.hier_random_state(rng, n, 128)
    done = pc.DONE_BYTES[rng.integers(0, 4, n)]
    done[:8] = [0, 1, 2, 255, 0, 0, 255, 2]
    gid = ROW_GID0 + np.arange(n)
    tr = Trunks(w, obs, state, done)
    c1, i1, col1 = _search_counter(tr, COUNTER_BASE, True, np.ones(n, bool))
    ok = np.ones(n, bool)
    ok[i1] = False
    c2, i2, col2 = _search_counter(tr, c1 + 1, False, ok)
    counters = (c1, c2)
    protect = {i1, i2}
    for _ in range(60):
        bad = set()
        for c in counters:
            ref, S = train_eval(tr, uniforms(gid, SEED, c))
            bad |= set(np.flatnonzero(~decisive(ref, S)).tolist())
        assert not bad & protect, ("a clamp row is not decisive", bad & protect)
        if not bad:
            info = dict(clamp_win=(c1, i1, col1), clamp_lose=(c2, i2, col2))
            return w, obs, state, done, counters, info
        rows = np.array(sorted(bad))
        for i in rows:
            obs[i] = pc._hier_row(rng, cats[i], 916)
        tr.put(rows, Trunks(w, obs[rows], state[rows], done[rows]))
    raise AssertionError("training rows stay undecided")


def reaches(w, obs, state, done, counters, info, evals):
    """What the batch is designed to reach, each entry a list of per-row (or per-batch) flags of which one must hold."""
    (c1, i1, col1), (c2, i2, col2) = info["clamp_win"], info["clamp_lose"]
    gid = ROW_GID0 + np.arange(len(obs))
    out = {}
    for c, (ref, S) in zip(counters, evals):
        am = ref["logits"].argmax(1)
        out.setdefault("sampled_is_argmax", []).extend((ref["code"] == am).tolist())
        out.setdefault("sampled_is_not_argmax", []).extend((ref["code"] != am).tolist())
        out.setdefault("p_below_1e-3", []).extend((ref["neglogp"] > np.log(1000.0)).tolist())
        out.setdefault("offset_ge_100", []).extend((ref["logits"].min(1) >= 100.0).tolist())
        out.setdefault("offset_le_-100", []).extend((ref["logits"].max(1) <= -100.0).tolist())
        out.setdefault("first_lane_winner", []).extend((ref["code"] % 32 == 0).tolist())
        out.setdefault("last_lane_winner", []).extend((ref["code"] % 32 == 31).tolist())
    r1 = draws(gid[i1:i1 + 1], SEED, c1)[0][0]
    r2 = draws(gid[i2:i2 + 1], SEED, c2)[0][0]
    out["clamp_wins"] = [bool(r1[col1] >= CLAMP_R and evals[0][0]["code"][i1] == col1)]
    out["clamp_loses"] = [bool(r2[col2] >= CLAMP_R and evals[1][0]["code"][i2] != col2)]
    out["done_bytes_on_nonzero_states"] = [set(np.unique(done).tolist()) == {0, 1, 2, 255} and bool((np.abs(state) > 0).all())]
    out["high_words"] = [SEED >> 32 != 0 and all(c >> 32 != 0 for c in counters)]
    out["row_gid_wraps"] = [bool(((gid >> 32) == 0).any() and ((gid >> 32) == 1).any())]
    return out


@functools.lru_cache(maxsize=None)
def train_case():
    """The designed batch with its reference and sensitivities at both counters (built once per session)."""
    w, obs, state, done, counters, info = build_train_case()
    tr = Trunks(w, obs, state, done)
    gid = ROW_GID0 + np.arange(len(obs))
    evals = [train_eval(tr, uniforms(gid, SEED, c)) for c in counters]
    return w, obs, state, done, counters, info, evals


RECUR_N, RECUR_STEPS, NULL_DONE_STEP = 300, 4, 2


def recurrence_case(w, seed=0, n=RECUR_N, steps=RECUR_STEPS):
    """Observations, done bytes and counters of `steps` recurrent steps from a non-zero state, every row decisive with a margin of 2
    along the fp64 chain (the GPU test feeds each step's reference the kernel's incoming state; the margin covers the difference)."""
    rng = np.random.default_rng(seed + 91)
    cats = [pc.HIER_CATS[i % 3] for i in range(n)]
    state = pc.hier_random_state(rng, n, 128)
    state0 = state.copy()
    gid = ROW_GID0 + np.arange(n)
    obs_all, done_all, ctr = [], [], []
    for s in range(steps):
        obs = np.stack([pc._hier_row(rng, c, 916) for c in cats])
        done = np.zeros(n, np.uint8) if s == NULL_DONE_STEP else pc.DONE_BYTES[(np.arange(n) + s) % 4]
        counter = COUNTER_BASE + 1000 + s
        u = uniforms(gid, SEED, counter)
        tr = Trunks(w, obs, state, done)
        for _ in range(60):
            ref, S = train_eval(tr, u)
            bad = np.flatnonzero(~decisive(ref, S, 2.0))
            if not len(bad):
                break
            for i in bad:
                obs[i] = pc._hier_row(rng, cats[i], 916)
            tr.put(bad, Trunks(w, obs[bad], state[bad], done[bad]))
        else:
            raise AssertionError("recurrence rows stay undecided")
        obs_all.append(obs)
        done_all.append(done)
        ctr.append(counter)
        state = ref["state"].astype(np.float32)
    return state0, obs_all, done_all, ctr
