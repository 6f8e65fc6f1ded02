"""fp64 statements of the three policy nets and designed batches on which every code is decisive (host only, numpy float64).

The nets are the ones `pmc_policy_kernel` (csrc/llq_policy.cu) and `hier_policy_kernel` (csrc/llq_policy_hier.cu) evaluate, written
afresh in float64 with the kernels' documented conventions: running-mean normalisation with `+1e-8` on the std and a clip to +-5,
layer-norm LSTMs with forget bias 1 and LN epsilon 1e-12 and the state `[c, h]` (the heading LSTM first at the strategic level),
TF 'SAME' convolutions (the 25 x 13 maps padded 1 before and 2 after in the stride-2 layer), the 128-ray lidar with periodic padding
4, the 29-slot game vector 913-917 | 918-932 | 948-954 | 962-963, the heading clipped to +-float(pi) (the kernel's constant, 8.7e-8
above pi), the first index winning ties of the code argmin / argmax, Philox4x32-10 + Box-Muller noise keyed by the global row.

Error model.  Every statement takes an `ErrorModel`; off, it is the reference.  On, it perturbs the result of every operation group
by one fp32 rounding's worth, r ~ U[-1, 1] per element, u = 2^-23:
  dense / conv layers and sums:        y += u (|x| @ |W| + |b|) r
  transcendentals and products:        y *= 1 + u r
  layer norms:                         y += u ((|x| + |mean|) |gamma| / sigma + |beta|) r   (the relative rule on each of the two terms)
The largest deviation from the reference over R_DRAWS draws is the sensitivity S of every output.  The GPU bars are kappa * S + u |ref|.

Decisiveness.  A row's code is decisive when the fp64 gap between the winner and the nearest code with a different codebook column
(PMC, in squared distance) or logit column (hierarchical, in logits) exceeds 4 kappa S_gap, S_gap the error model's sensitivity of
that gap.  The builders keep only batches in which every row is decisive or is a designed exact tie; rows that are not are redrawn.
"""
import functools

import numpy as np

from lifelike_agility_and_play_b200.policy_epmc import hier_role_arrays, random_weights as hier_random_weights

U = 2.0 ** -23
R_DRAWS = 4
# GPU bar factors, one per kernel: at least 4x the largest error / S measured on an H100 80GB HBM3 at a 600 W power limit
# (tests/test_policy_cases_gpu.py lists the measurements).  PMC: 88.2 -> 400 (the 3xTF32 layers truncate their operand splits, a
# bias of up to ~2^-20 per product that the one-rounding model does not carry); hierarchical: 4.73 -> 20.
KAPPA_PMC = 400.0
KAPPA_HIER = 20.0
PI32 = float(np.float32(np.pi))          # the heading clip of hier_policy_kernel: 3.14159265358979f
GAME_COLS = np.r_[913:918, 918:933, 948:955, 962:964]
M32 = np.uint64(0xFFFFFFFF)


class ErrorModel:
    """seed None: the reference (no perturbation); otherwise one draw of the error model."""

    def __init__(self, seed=None):
        self.rng = None if seed is None else np.random.default_rng(seed)

    @property
    def on(self):
        return self.rng is not None

    def add(self, y, mag):
        return y if self.rng is None else y + U * mag * self.rng.uniform(-1.0, 1.0, np.shape(y))

    def rel(self, y):
        return y if self.rng is None else y * (1.0 + U * self.rng.uniform(-1.0, 1.0, np.shape(y)))


REF = ErrorModel()


def fc(x, W, b, em, act=None):
    y = x @ W if b is None else x @ W + b
    if em.on:
        y = em.add(y, np.abs(x) @ np.abs(W) + (0.0 if b is None else np.abs(b)))
    if act == "relu":
        return np.maximum(y, 0.0)
    if act == "tanh":
        return em.rel(np.tanh(y))
    return y


def fc_elementwise(x, W, b, em):
    """b + sum_k x[:, k] W[k] summed column by column in a fixed order: identical columns give identical results (a BLAS matmul
    may round two identical columns differently)."""
    y = np.broadcast_to(b, (x.shape[0], W.shape[1])).copy()
    for k in range(W.shape[0]):
        y += x[:, k, None] * W[k][None]
    return em.add(y, np.abs(x) @ np.abs(W) + np.abs(b)) if em.on else y


def normalise(obs, mean, std, em):
    d = std + 1e-8
    y = (obs - mean) / d
    if em.on:
        y = em.add(y, (np.abs(obs) + np.abs(mean)) / d)
    return np.clip(y, -5.0, 5.0)


def _f64(w):
    return [np.asarray(a, np.float64) for a in w]


# ------------------------------------------------------------------------------------------------------------------- PMC
PMC_SHAPES = [(1, 135), (1, 135), (1, 72), (1, 72), (207, 256), (256,), (256, 256), (256,), (256, 1), (1,), (207, 256), (256,), (256, 256),
              (256,), (256, 32), (32,), (32, 256), (135, 64), (64,), (32, 32), (32,), (96, 256), (256,), (256, 256), (256,), (256, 12), (12,),
              (1, 12)]


def pmc_random_weights(seed):
    rng = np.random.default_rng(seed)
    w = [(rng.standard_normal(s) / np.sqrt(s[0] if len(s) == 2 and s[0] > 1 else 1.0)).astype(np.float32) for s in PMC_SHAPES]
    w[1] = np.abs(w[1]) + 0.1
    w[3] = np.abs(w[3]) + 0.1
    w[27] = (0.3 * w[27] - 0.5).astype(np.float32)
    return w


def pmc_trunk(W, obs, em):
    """Normalised observation, value head and the VQ encoder's z (none of them depends on the codebook)."""
    p = normalise(obs[:, :135], W[0][0], W[1][0], em)
    f = normalise(obs[:, 135:207], W[2][0], W[3][0], em)
    x = np.concatenate([p, f], axis=1)
    v = fc(fc(fc(x, W[4], W[5], em, "tanh"), W[6], W[7], em, "tanh"), W[8], W[9], em)[:, 0]
    z = fc(fc(fc(x, W[10], W[11], em, "relu"), W[12], W[13], em, "relu"), W[14], W[15], em)
    return dict(p=p, x=x, value=v, z=z)


def pmc_distances(z, cb, em):
    """Squared distance of every row's z to every code, summed over k in order, element by element like the kernel."""
    d = np.zeros((z.shape[0], cb.shape[1]))
    for k in range(cb.shape[0]):
        t = z[:, k, None] - cb[k][None]
        d += t * t
    return em.add(d, d)


def pmc_mean(W, p, code, em):
    zq = W[16][:, code].T
    x = np.concatenate([fc(p, W[17], W[18], em, "relu"), fc(zq, W[19], W[20], em, "relu")], axis=1)
    x = fc(fc(x, W[21], W[22], em, "relu"), W[23], W[24], em, "relu")
    return fc(x, W[25], W[26], em)


def same_columns(cb):
    """same[i, j]: codebook (or logit) columns i and j are identical."""
    return np.all(cb[:, :, None] == cb[:, None, :], axis=0)


def code_gap(d, code, same, sign=1.0):
    """sign = 1: distances (argmin); -1: logits (argmax).  Gap to the nearest column that differs from the winner's."""
    v = sign * d
    masked = np.where(same[code], np.inf, v)
    return masked.min(1) - v[np.arange(len(code)), code]


def pmc_eval(w, obs, draws=R_DRAWS):
    """Reference outputs of the PMC net on fp32 `obs` [n, >=207] and their sensitivities S over `draws` error-model draws
    (the draws keep the reference's code, as the kernel does on a decisive row)."""
    W = _f64(w)
    obs = np.asarray(obs[:, :207], np.float64)
    same = same_columns(W[16])
    t = pmc_trunk(W, obs, REF)
    d = pmc_distances(t["z"], W[16], REF)
    code = np.argmin(d, axis=1)
    ref = dict(code=code, dist=d, z=t["z"], value=t["value"], gap=code_gap(d, code, same), mean=pmc_mean(W, t["p"], code, REF))
    S = {k: np.zeros_like(ref[k]) for k in ("z", "value", "gap", "mean")}
    for i in range(draws):
        em = ErrorModel(1000 + i)
        ti = pmc_trunk(W, obs, em)
        di = pmc_distances(ti["z"], W[16], em)
        got = dict(z=ti["z"], value=ti["value"], gap=code_gap(di, code, same), mean=pmc_mean(W, ti["p"], code, em))
        for k in S:
            S[k] = np.maximum(S[k], np.abs(got[k] - ref[k]))
    return ref, S


# --------------------------------------------------------------------------------------------- Philox4x32-10, Box-Muller
def philox4x32(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 of the kernel (csrc/llq_policy.cu) on uint32 values held in uint64 arrays."""
    c = [np.asarray(x, np.uint64) & M32 for x in (c0, c1, c2, c3)]
    k0, k1 = np.uint64(k0) & M32, np.uint64(k1) & M32
    c = np.broadcast_arrays(*c)
    c0, c1, c2, c3 = [x.copy() for x in c]
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c0
        p1 = np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & M32
        k0 = (k0 + np.uint64(0x9E3779B9)) & M32
        k1 = (k1 + np.uint64(0xBB67AE85)) & M32
    return c0, c1, c2, c3


def pmc_eps(global_rows, seed, counter, em=REF):
    """eps [n, 12] of row `global_rows` (= row_gid0 + row): counter (row, q, counter lo, counter hi), key (seed lo, seed hi); the
    uniforms with the kernel's fp32 operations, log / sqrt / sin / cos in fp64."""
    g = np.asarray(global_rows, np.int64).astype(np.uint64) & M32
    seed, counter = int(seed), int(counter)
    f = np.float32
    eps = np.zeros((len(g), 12))
    for q in range(3):
        r = philox4x32(g, q, counter & 0xFFFFFFFF, counter >> 32, seed & 0xFFFFFFFF, seed >> 32)
        rf = [x.astype(np.float32) for x in r]
        scale = f(2.3283064365386963e-10)
        u0, u1 = (rf[0] + f(0.5)) * scale, rf[1] * scale
        u2, u3 = (rf[2] + f(0.5)) * scale, rf[3] * scale
        pairs = []
        for ua, ub in ((u0, u1), (u2, u3)):
            ua = np.minimum(ua, f(0.99999994)).astype(np.float64)
            rad = em.rel(np.sqrt(em.rel(-2.0 * np.log(ua))))
            ang = (f(6.283185307179586) * ub).astype(np.float64)
            pairs.append((em.rel(rad * em.rel(np.cos(ang))), em.rel(rad * em.rel(np.sin(ang)))))
        eps[:, 4 * q], eps[:, 4 * q + 1] = pairs[0]
        eps[:, 4 * q + 2], eps[:, 4 * q + 3] = pairs[1]
    return eps


def pmc_sample(mean, logstd, eps, em=REF):
    """The sampled action mean + exp(logstd) eps and its -log p = 0.5 sum eps^2 + sum logstd + 6 log(2 pi)."""
    ls = np.asarray(logstd, np.float64).reshape(-1)
    e = em.rel(np.exp(ls))
    a = em.add(mean + e * eps, np.abs(mean) + np.abs(e * eps))
    terms = 0.5 * eps * eps + ls
    c = 6.0 * np.log(2.0 * np.pi)
    return a, em.add(c + terms.sum(1), c + np.abs(terms).sum(1))


def pmc_sample_eval(w, mean_ref, S_mean, global_rows, seed, counter, draws=R_DRAWS):
    """Reference sample / -log p and their sensitivities (the mean's own sensitivity S_mean enters as a bound)."""
    ls = np.asarray(w[27], np.float64).reshape(-1)
    eps = pmc_eps(global_rows, seed, counter)
    a, nl = pmc_sample(mean_ref, ls, eps)
    Sa, Snl = np.array(S_mean, np.float64), np.zeros_like(nl)
    for i in range(draws):
        em = ErrorModel(2000 + i)
        ai, nli = pmc_sample(mean_ref, ls, pmc_eps(global_rows, seed, counter, em), em)
        Sa = np.maximum(Sa, np.abs(ai - a) + S_mean)
        Snl = np.maximum(Snl, np.abs(nli - nl))
    return dict(eps=eps, sample=a, neglogp=nl), dict(sample=Sa, neglogp=Snl)


# --------------------------------------------------------------------------------------------------------- PMC batches
PMC_N = 4097
PMC_TIE_SAME_LANE_LO = (0, 33, 2000)       # winner copied to winner - 32 (same lane) and winner + 1
PMC_TIE_SAME_LANE_HI = (31, 1000, 4096)    # winner copied to winner - 1 and winner + 32 (same lane)
PMC_TIGHT = (1, 32, 3000, 4095)
PMC_CATS = ("random", "clip", "saturate")
TINY_STD_COL = 7                            # prop column with running std 1e-9


def _pmc_row(rng, cat, w):
    x = (2.0 * rng.standard_normal(207)).astype(np.float32)
    mean = np.concatenate([w[0][0], w[2][0]])
    std = np.concatenate([w[1][0], w[3][0]])
    if cat == "clip":                       # prop and future entries far past +-5 sigma
        k = rng.choice(207, 40, replace=False)
        k = np.concatenate([k, [3, 150]])
        x[k] = (mean[k] + np.sign(rng.standard_normal(len(k))) * rng.uniform(6.0, 60.0, len(k)) * std[k]).astype(np.float32)
    elif cat == "saturate":                 # every normalised value at +-5: the first tanh layer runs deep in saturation
        x[:] = (mean + np.sign(rng.standard_normal(207)) * 50.0 * std).astype(np.float32)
    x[TINY_STD_COL] = np.float32(mean[TINY_STD_COL] + np.sign(rng.standard_normal()) * rng.uniform(1e-3, 1.0))
    return x


def pmc_categories(n=PMC_N):
    cats = [PMC_CATS[(i * 7) % 3] if i % 5 else "random" for i in range(n)]
    for i in PMC_TIE_SAME_LANE_LO:
        cats[i] = "tie_same_lane_lo"
    for i in PMC_TIE_SAME_LANE_HI:
        cats[i] = "tie_same_lane_hi"
    for i in PMC_TIGHT:
        cats[i] = "tight"
    return cats


def _pmc_decisive(ref, S, kappa, rows=None):
    g, s = ref["gap"], S["gap"]
    ok = g > 4.0 * kappa * s
    return ok if rows is None else ok[rows]


def _tie_columns(c, same_lo):
    return (c - 32, c + 1) if same_lo else (c - 1, c + 32)


def _fit_designed_winners(code, ties_lo, ties_hi, tight, redraw):
    """Redraw designed rows until their winners are distinct and leave room for the tie columns; redraw(i) returns row i's new
    (decisive) code."""
    designed = list(ties_lo) + list(ties_hi) + list(tight)
    for _ in range(400):
        used, bad = set(), None
        for i in designed:
            if int(code[i]) in used:
                bad = i
                break
            used.add(int(code[i]))
        if bad is None:
            for rows, same_lo in ((ties_lo, True), (ties_hi, False)):
                for i in rows:
                    lo, hi = _tie_columns(int(code[i]), same_lo)
                    if bad is None and (lo < 0 or hi > 255 or {lo, hi} & used):
                        bad = i
                    used |= {lo, hi}
        if bad is None:
            return
        code[bad] = redraw(bad)
    raise AssertionError("no room for the designed codes")


def _pmc_redraw_one(rng, w, obs, i, kappa):
    while True:
        obs[i] = _pmc_row(rng, "random", w)
        r, s = pmc_eval(w, obs[i:i + 1])
        if r["gap"][0] > 4.0 * kappa * s["gap"][0]:
            return int(r["code"][0])


def build_pmc_case(seed=0, kappa=KAPPA_PMC, n=PMC_N):
    """Weights (fp32 list of 28 arrays) and observations [n, 207] fp32 with every row decisive or a designed exact tie.
    Returns (w, obs, cats, info) with info the designed columns."""
    rng = np.random.default_rng(seed)
    w = pmc_random_weights(seed + 1)
    w[1] = w[1].copy()
    w[1][0, TINY_STD_COL] = np.float32(1e-9)
    cats = pmc_categories(n)
    # a codebook on the encoder's output, as a trained one is: the nearest code is as near as the nearest other row
    zs = pmc_trunk(_f64(w), np.stack([_pmc_row(rng, PMC_CATS[k % 3], w) for k in range(256)]).astype(np.float64), REF)["z"]
    w[16] = (zs.T + 0.3 * rng.standard_normal((32, 256))).astype(np.float32)
    obs = np.stack([_pmc_row(rng, c, w) for c in cats])
    # 1. every row decisive on the random codebook
    for _ in range(30):
        ref, S = pmc_eval(w, obs)
        bad = np.flatnonzero(~_pmc_decisive(ref, S, kappa))
        if len(bad) == 0:
            break
        for i in bad:
            obs[i] = _pmc_row(rng, cats[i] if cats[i] in PMC_CATS else "random", w)
    else:
        raise AssertionError("PMC rows stay undecided")
    # 2. exact ties: a designed row's winner copied to a lower and a higher column
    cb = w[16].copy()
    code = ref["code"]
    _fit_designed_winners(code, PMC_TIE_SAME_LANE_LO, PMC_TIE_SAME_LANE_HI, PMC_TIGHT, lambda i: _pmc_redraw_one(rng, w, obs, i, kappa))
    ref, S = pmc_eval(w, obs)
    code = ref["code"]
    used = {int(code[i]) for i in PMC_TIE_SAME_LANE_LO + PMC_TIE_SAME_LANE_HI + PMC_TIGHT}
    info = dict(ties={}, tight={})
    for rows, same_lo in ((PMC_TIE_SAME_LANE_LO, True), (PMC_TIE_SAME_LANE_HI, False)):
        for i in rows:
            c = int(code[i])
            lo, hi = _tie_columns(c, same_lo)
            cb[:, lo] = cb[:, c]
            cb[:, hi] = cb[:, c]
            used |= {lo, hi}
            info["ties"][i] = (lo, c, hi)
    # 3. tight codes: two fresh columns around the row's fp64 z, gap between 4 kappa and 8 kappa S_gap
    W = _f64(w)
    z = ref["z"]
    Szs = [pmc_trunk(W, np.asarray(obs[list(PMC_TIGHT)], np.float64), ErrorModel(1000 + k))["z"] for k in range(R_DRAWS)]
    free = [c for c in range(256) if c not in used]
    rng.shuffle(free)
    place = {}
    for j, i in enumerate(PMC_TIGHT):
        a, b = sorted(free[2 * j:2 * j + 2])
        used |= {a, b}
        v1, v2 = rng.standard_normal(32), rng.standard_normal(32)
        v1 /= np.linalg.norm(v1)
        v2 /= np.linalg.norm(v2)
        rho = 0.3
        first = (a, b) if rng.uniform() < 0.5 else (b, a)            # the winner is the lower or the higher column
        cb[:, first[0]] = (z[i] + rho * v1).astype(np.float32)
        target = None
        for _ in range(6):
            cbf = cb.astype(np.float64)
            cols = list(first)
            d = pmc_distances(z[i:i + 1], cbf[:, cols], REF)[0]
            sg = max(abs((pmc_distances(Szs[k][j:j + 1], cbf[:, cols], ErrorModel(3000 + k))[0] @ [-1.0, 1.0]) - (d @ [-1.0, 1.0]))
                     for k in range(R_DRAWS))
            target = 6.0 * kappa * max(sg, 1e-12)
            r2 = np.sqrt(rho * rho + target)
            cb[:, first[1]] = (z[i] + r2 * v2).astype(np.float32)
        info["tight"][i] = first
        place[i] = (z[i], rho, v2)
    w[16] = cb
    # 4. every other row still decisive; redraw those that are not
    designed = set(PMC_TIE_SAME_LANE_LO + PMC_TIE_SAME_LANE_HI + PMC_TIGHT)
    for _ in range(30):
        ref, S = pmc_eval(w, obs)
        ok = _pmc_decisive(ref, S, kappa)
        bad = [i for i in np.flatnonzero(~ok) if i not in info["ties"]]
        assert not [i for i in bad if i in designed], ("designed rows undecided", bad)
        # the gap of a tight row from the whole batch's sensitivity: move its second code until the gap is 6 kappa S_gap
        moved = False
        for i, (zi, rho, v2) in place.items():
            ratio = ref["gap"][i] / S["gap"][i]
            if not 4.5 * kappa < ratio < 7.5 * kappa:
                w[16][:, info["tight"][i][1]] = (zi + np.sqrt(rho * rho + 6.0 * kappa * S["gap"][i]) * v2).astype(np.float32)
                moved = True
        if moved:
            continue
        if not bad:
            break
        for i in bad:
            obs[i] = _pmc_row(rng, cats[i] if cats[i] in PMC_CATS else "random", w)
    else:
        raise AssertionError("PMC rows stay undecided")
    return w, obs, cats, info


def pmc_reaches(w, obs, cats, info, ref, S, kappa=KAPPA_PMC):
    """Per category, the rows that reach what the category is named for."""
    W = _f64(w)
    x = pmc_trunk(W, np.asarray(obs, np.float64), REF)["x"]
    mean = np.concatenate([W[0][0], W[2][0]])
    std = np.concatenate([W[1][0], W[3][0]])
    raw = (np.asarray(obs[:, :207], np.float64) - mean) / (std + 1e-8)
    pre1 = x @ W[4] + W[5]
    out = {}
    for i, c in enumerate(cats):
        if c == "clip":
            ok = (np.abs(raw[i, :135]) > 5.5).any() and (np.abs(raw[i, 135:]) > 5.5).any()
        elif c == "saturate":
            ok = (np.abs(pre1[i]) > 3.0).mean() > 0.4 and (np.abs(x[i]) == 5.0).all()
        elif c.startswith("tie"):
            lo, mid, hi = info["ties"][i]
            d = ref["dist"][i]
            same_lane = (lo % 32 == mid % 32) if c == "tie_same_lane_lo" else (hi % 32 == mid % 32)
            ok = ref["code"][i] == lo and d[lo] == d[mid] == d[hi] and same_lane and ref["gap"][i] > 4 * kappa * S["gap"][i]
        elif c == "tight":
            ok = 4 * kappa * S["gap"][i] < ref["gap"][i] < 8 * kappa * S["gap"][i] and ref["code"][i] == info["tight"][i][0]
        else:
            ok = True
        out.setdefault(c, []).append(bool(ok))
    out["tiny_std"] = [bool((np.abs(raw[:, TINY_STD_COL]) > 5.0).all())]
    return out


# -------------------------------------------------------------------------------------------------- hierarchical nets
def _same_pad(n, k, s):
    out = -(-n // s)
    total = max((out - 1) * s + k - n, 0)
    return out, total // 2, total - total // 2


def conv_same_relu(x, Wc, b, stride, em):
    """x [B, H, W, C], Wc [kh, kw, C, O] (TF layout), 'SAME' padding, ReLU."""
    B, H, Wd, C = x.shape
    kh, kw, _, O = Wc.shape
    oh, pt, pb = _same_pad(H, kh, stride)
    ow, pl, pr = _same_pad(Wd, kw, stride)
    xp = np.pad(x, ((0, 0), (pt, pb), (pl, pr), (0, 0)))
    cols = np.concatenate([xp[:, i:i + (oh - 1) * stride + 1:stride, j:j + (ow - 1) * stride + 1:stride, :]
                           for i in range(kh) for j in range(kw)], axis=3).reshape(-1, kh * kw * C)      # taps in [kh][kw][C] order
    Wf = Wc.reshape(kh * kw * C, O)
    y = (cols @ Wf + b).reshape(B, oh, ow, O)
    if em.on:
        y = em.add(y, (np.abs(cols) @ np.abs(Wf) + np.abs(b)).reshape(B, oh, ow, O))
    return np.maximum(y, 0.0)


def enc2d(m, ws, em):
    e = m[..., None]
    e = conv_same_relu(e, ws[0], ws[1], 1, em)
    e = conv_same_relu(e, ws[2], ws[3], 2, em)
    e = conv_same_relu(e, ws[4], ws[5], 2, em)
    e = conv_same_relu(e, ws[6], ws[7], 1, em)
    return e.reshape(e.shape[0], -1)


def enc1d(r, ws, em, k=4):
    p = np.concatenate([r[:, -k:], r, r[:, :k]], axis=1)[:, None, :, None]       # periodic padding
    e = conv_same_relu(p, ws[0][None], ws[1], 1, em)[:, :, k:-k, :]
    e = conv_same_relu(e, ws[2][None], ws[3], 2, em)
    e = conv_same_relu(e, ws[4][None], ws[5], 2, em)
    e = conv_same_relu(e, ws[6][None], ws[7], 1, em)
    return e.reshape(e.shape[0], -1)


def perception(obs, ws, em):
    """[2-D map (28) | lidar (32) | front map (28)] of one usr_cmd_encoder."""
    return np.concatenate([enc2d(obs[:, 135:460].reshape(-1, 25, 13), ws[0:8], em), enc1d(obs[:, 460:588], ws[8:16], em),
                           enc2d(obs[:, 588:913].reshape(-1, 25, 13), ws[16:24], em)], axis=1)


def layer_norm(x, beta, gamma, em):
    m = x.mean(1, keepdims=True)
    inv = 1.0 / np.sqrt(((x - m) ** 2).mean(1, keepdims=True) + 1e-12)
    y = (x - m) * inv * gamma + beta
    return em.add(y, (np.abs(x) + np.abs(m)) * inv * np.abs(gamma) + np.abs(beta)) if em.on else y


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def lstm_step(x, c, h, ws, em):
    wx, wh, b, bx, gx, bh, gh, bc, gc = ws
    zx = layer_norm(fc(x, wx, None, em), bx, gx, em)
    zh = layer_norm(fc(h, wh, None, em), bh, gh, em)
    z = em.add(zx + zh + b, np.abs(zx) + np.abs(zh) + np.abs(b))
    gi, gf, go, gu = np.split(z, 4, axis=1)
    sf, si = em.rel(sigmoid(gf + 1.0)), em.rel(sigmoid(gi))                  # forget bias 1
    tu, so = em.rel(np.tanh(gu)), em.rel(sigmoid(go))
    c2 = em.add(sf * c + si * tu, np.abs(sf * c) + np.abs(si * tu))
    h2 = em.rel(so * em.rel(np.tanh(layer_norm(c2, bc, gc, em))))
    return c2, h2


class Hier:
    """fp64 view of an environmental- (102 arrays) or strategic-level (152 arrays) model, by the kernel's roles
    (include/llq_policy.h)."""

    def __init__(self, weights):
        self.strategic = len(weights) == 152
        self.r = [np.asarray(weights[i], np.float64) for i in hier_role_arrays(self.strategic)]
        self.ow = 965 if self.strategic else 916
        self.ssz = 128 if self.strategic else 64

    def trunk(self, obs, state, done, em):
        """Everything up to the code LSTM's h: (p, h, new state, heading before / after the clip)."""
        r = self.r
        obs = np.asarray(obs[:, :self.ow], np.float64)
        state = np.asarray(state, np.float64)
        keep = (np.asarray(done) == 0)[:, None] if done is not None else np.ones((len(obs), 1), bool)
        state = np.where(keep, state, 0.0)
        p = normalise(obs[:, :135], r[0][0], r[1][0], em)
        new_state, pre, ang = np.zeros_like(state), None, None
        st = 0
        if self.strategic:
            pe = fc(p, r[56], r[57], em, "relu")
            pc = fc(perception(obs, r[58:82], em), r[82], r[83], em, "relu")
            ge = fc(fc(obs[:, GAME_COLS], r[84], r[85], em, "relu"), r[86], r[87], em, "relu")
            e = fc(np.concatenate([pe, pc, ge], axis=1), r[88], r[89], em, "relu")
            c, h = lstm_step(e, state[:, 0:32], state[:, 32:64], r[90:99], em)
            new_state[:, 0:32], new_state[:, 32:64] = c, h
            pre = fc(h, r[99], r[100], em)[:, 0]
            ang = np.clip(pre, -PI32, PI32)
            tgt = np.stack([em.rel(np.cos(ang)), em.rel(np.sin(ang)), obs[:, 964]], axis=1)
            st = 64
        else:
            tgt = obs[:, 913:916]
        pe = fc(p, r[2], r[3], em, "relu")
        t = fc(tgt, r[28], r[29], em, "relu")
        ce = fc(np.concatenate([t, perception(obs, r[4:28], em)], axis=1), r[30], r[31], em, "relu")
        e = fc(np.concatenate([pe, ce], axis=1), r[32], r[33], em, "relu")
        c, h = lstm_step(e, state[:, st:st + 32], state[:, st + 32:st + 64], r[34:43], em)
        new_state[:, st:st + 32], new_state[:, st + 32:st + 64] = c, h
        return dict(p=p, h=h, state=new_state, heading_pre=pre, heading=ang)

    def logits(self, h, em):
        return fc_elementwise(h, self.r[43], self.r[44], em)

    def actions(self, p, code, em):
        r = self.r
        zq = r[45][:, code].T
        x = np.concatenate([fc(p, r[46], r[47], em, "relu"), fc(zq, r[48], r[49], em, "relu")], axis=1)
        x = fc(fc(x, r[50], r[51], em, "relu"), r[52], r[53], em, "relu")
        return fc(x, r[54], r[55], em)


def hier_eval(w, obs, state, done, draws=R_DRAWS, trunks=None):
    """Reference outputs of the hierarchical net (new state, logits, code, heading before / after the clip, actions) and their
    sensitivities; `trunks` (reference, draws) from an earlier call on the same rows skips the part before the logits."""
    net = Hier(w)
    if trunks is None:
        trunks = (net.trunk(obs, state, done, REF), [net.trunk(obs, state, done, ErrorModel(5000 + i)) for i in range(draws)])
    t, tds = trunks
    same = same_columns(np.vstack([net.r[43], net.r[44][None]]))
    lg = net.logits(t["h"], REF)
    code = np.argmax(lg, axis=1)
    ref = dict(code=code, logits=lg, gap=code_gap(lg, code, same, -1.0), actions=net.actions(t["p"], code, REF), state=t["state"])
    if net.strategic:
        ref["heading"], ref["heading_pre"] = t["heading"], t["heading_pre"]
    S = {k: np.zeros_like(v, np.float64) for k, v in ref.items() if k != "code"}
    for i, td in enumerate(tds):
        em = ErrorModel(6000 + i)
        lgi = net.logits(td["h"], em)
        got = dict(logits=lgi, gap=code_gap(lgi, code, same, -1.0), actions=net.actions(td["p"], code, em), state=td["state"])
        if net.strategic:
            got["heading"], got["heading_pre"] = td["heading"], td["heading_pre"]
        for k in S:
            S[k] = np.maximum(S[k], np.abs(got[k] - ref[k]))
    return ref, S, trunks


# ---------------------------------------------------------------------------------------------- hierarchical batches
HIER_N = 1059                               # 132 * 8 + 3
HIER_TIE_SAME_LANE_LO = (0, 9, 500)
HIER_TIE_SAME_LANE_HI = (7, 300, 1058)
HIER_TIGHT = (1, 8, 301, 1057)
HIER_CATS = ("random", "border", "lidar_wrap")


def _hier_row(rng, cat, ow):
    x = rng.standard_normal(ow).astype(np.float32)
    x[135:913] = np.abs(x[135:913]) * 0.7                  # heights and distances are non-negative
    if cat == "border":                                    # features on the first / last rows and columns of both maps
        for m0 in (135, 588):
            m = (0.1 * np.abs(rng.standard_normal((25, 13)))).astype(np.float32)
            m[0, :], m[-1, :] = rng.uniform(2.0, 4.0, 13), rng.uniform(2.0, 4.0, 13)
            m[:, 0], m[:, -1] = rng.uniform(2.0, 4.0, 25), rng.uniform(2.0, 4.0, 25)
            x[m0:m0 + 325] = m.reshape(-1)
    elif cat == "lidar_wrap":                              # distinct large values on rays 0, 1, 126, 127
        x[460:588] = 0.1 * np.abs(rng.standard_normal(128))
        x[460 + np.array([0, 1, 126, 127])] = rng.permutation([3.0, 4.0, 5.0, 6.0]) + rng.uniform(0.0, 0.5, 4)
    elif cat.startswith("slot"):                           # game-vector slot k singled out
        k = int(cat[4:])
        x[GAME_COLS] = 0.05 * rng.standard_normal(29)
        x[GAME_COLS[k]] = np.sign(rng.standard_normal()) * rng.uniform(3.0, 5.0)
    return x


def hier_categories(strategic, n=HIER_N):
    cats = [HIER_CATS[i % 3] for i in range(n)]
    if strategic:
        for k in range(29):
            cats[10 + 11 * k] = "slot%d" % k
    for i in HIER_TIE_SAME_LANE_LO:
        cats[i] = "tie_same_lane_lo"
    for i in HIER_TIE_SAME_LANE_HI:
        cats[i] = "tie_same_lane_hi"
    for i in HIER_TIGHT:
        cats[i] = "tight"
    return cats


def _row_cat(c):
    return c if (c in HIER_CATS or c.startswith("slot")) else "random"


def hier_random_state(rng, n, ssz):
    return (0.6 * rng.standard_normal((n, ssz))).astype(np.float32)


DONE_BYTES = np.array([0, 1, 2, 255], np.uint8)


def _redraw_until_decisive(w, obs, state, done, cats, rng, kappa, protect=(), margin=1.0, redraw_state=False):
    """Redraw the rows whose code is not decisive (gap > 4 kappa margin S_gap) until none is left; returns (ref, S, trunks)."""
    net = Hier(w)
    ref, S, tr = hier_eval(w, obs, state, done)
    merged = False
    for _ in range(60):
        bad = np.flatnonzero(~(ref["gap"] > 4.0 * kappa * margin * S["gap"]))
        assert not set(bad.tolist()) & set(protect), ("designed rows undecided", sorted(set(bad.tolist()) & set(protect)))
        if len(bad) == 0:
            if not merged:
                return ref, S, tr
            ref, S, tr = hier_eval(w, obs, state, done)          # confirm on the whole batch's draws
            merged = False
            continue
        merged = True
        for i in bad:
            obs[i] = _hier_row(rng, _row_cat(cats[i]), net.ow)
            if redraw_state:                # the incoming state can hold a row on one code
                state[i] = hier_random_state(rng, 1, net.ssz)[0]
        r2, S2, t2 = hier_eval(w, obs[bad], state[bad], done[bad])
        for k in ref:
            ref[k][bad] = r2[k]
        for k in S:
            S[k][bad] = S2[k]
        t0, td = tr
        for d_all, d_new in zip([t0] + td, [t2[0]] + t2[1]):
            for k, v in d_all.items():
                if v is not None:
                    v[bad] = d_new[k]
    raise AssertionError("hierarchical rows stay undecided: %s" % bad[:10])


def build_hier_case(strategic, seed=0, kappa=KAPPA_HIER, n=HIER_N):
    """Weights (fp32 list), observations [n, ow] fp32, a non-zero incoming state, done bytes in {0, 1, 2, 255}; every row
    decisive or a designed exact tie.  Returns (w, obs, state, done, cats, info)."""
    rng = np.random.default_rng(seed)
    w = [a.copy() for a in hier_random_weights(strategic, seed + 1)]
    roles = hier_role_arrays(strategic)
    if strategic:
        w[roles[99]] = (40.0 * w[roles[99]]).astype(np.float32)          # heading pushed past +-pi on some rows, both ways
        w[roles[100]] = np.zeros_like(w[roles[100]])
    ow, ssz = (965, 128) if strategic else (916, 64)
    cats = hier_categories(strategic, n)
    obs = np.stack([_hier_row(rng, _row_cat(c), ow) for c in cats])
    state = hier_random_state(rng, n, ssz)
    # random LSTM outputs share a large common part: centre the logits on it so that the rows spread over many codes
    h = Hier(w).trunk(obs[:64], state[:64], np.zeros(64, np.uint8), REF)["h"]
    w[roles[43]] = (4.0 * w[roles[43]]).astype(np.float32)
    if strategic:                          # the same for the heading: centred, then both clips are reached
        pre = Hier(w).trunk(obs[:64], state[:64], np.zeros(64, np.uint8), REF)["heading_pre"]
        w[roles[100]] = np.array([-np.median(pre)], np.float32)
    w[roles[44]] = (-(h.mean(0) @ w[roles[43]]) + 0.1 * w[roles[44]]).astype(np.float32)
    done = DONE_BYTES[rng.integers(0, 4, n)]
    done[:8] = [0, 1, 2, 255, 0, 0, 255, 2]
    ref, S, tr = _redraw_until_decisive(w, obs, state, done, cats, rng, kappa, redraw_state=True)
    Wl, bl = w[roles[43]].copy(), w[roles[44]].copy()
    code = ref["code"]
    designed = HIER_TIE_SAME_LANE_LO + HIER_TIE_SAME_LANE_HI + HIER_TIGHT

    def redraw(i):
        while True:
            obs[i] = _hier_row(rng, "random", ow)
            r, s, _ = hier_eval(w, obs[i:i + 1], state[i:i + 1], done[i:i + 1])
            if r["gap"][0] > 4.0 * kappa * s["gap"][0]:
                return int(r["code"][0])
    _fit_designed_winners(code, HIER_TIE_SAME_LANE_LO, HIER_TIE_SAME_LANE_HI, HIER_TIGHT, redraw)
    ref, S, tr = _redraw_until_decisive(w, obs, state, done, cats, rng, kappa, redraw_state=True)
    code = ref["code"]
    used = {int(code[i]) for i in designed}
    info = dict(ties={}, tight={})
    for rows, same_lo in ((HIER_TIE_SAME_LANE_LO, True), (HIER_TIE_SAME_LANE_HI, False)):
        for i in rows:
            c = int(code[i])
            lo, hi = _tie_columns(c, same_lo)
            Wl[:, lo] = Wl[:, c]; Wl[:, hi] = Wl[:, c]
            bl[lo] = bl[c]; bl[hi] = bl[c]
            used |= {lo, hi}
            info["ties"][i] = (lo, c, hi)
    free = [c for c in range(256) if c not in used]
    rng.shuffle(free)
    net_t0, net_td = tr
    hs = [net_t0["h"]] + [td["h"] for td in net_td]
    for j, i in enumerate(HIER_TIGHT):
        # a column pair: c2 copies the winner's weights with its bias lowered by 6 kappa S_gap (the row's winner stays c; a row with
        # another winner is not affected unless c is within that gap of its own winner)
        c, c2 = int(code[i]), int(free[j])
        used.add(c2)
        Wl[:, c2] = Wl[:, c]
        bl[c2] = np.float32(bl[c] - 1e-3)
        for _ in range(4):
            lg = [fc_elementwise(h[i:i + 1], Wl.astype(np.float64), bl.astype(np.float64), REF if k == 0 else ErrorModel(7000 + k))[0]
                  for k, h in enumerate(hs)]
            g = lg[0][c] - lg[0][c2]
            sg = max(abs((x[c] - x[c2]) - g) for x in lg[1:])
            bl[c2] = np.float32(bl[c] - 6.0 * kappa * sg)
        info["tight"][i] = (c, c2)
    w[roles[43]], w[roles[44]] = Wl, bl
    for _ in range(6):                     # the tight gaps against the whole batch's S_gap
        ref, S, tr = _redraw_until_decisive(w, obs, state, done, cats, rng, kappa, protect=designed, redraw_state=True)
        off = [i for i in HIER_TIGHT if not 4.5 * kappa < ref["gap"][i] / S["gap"][i] < 7.5 * kappa]
        if not off:
            return w, obs, state, done, cats, info
        for i in off:
            c, c2 = info["tight"][i]
            w[roles[44]][c2] = np.float32(w[roles[44]][c] - 6.0 * kappa * S["gap"][i])
    raise AssertionError("tight logits out of range")


def hier_reaches(w, obs, cats, info, ref, S, kappa=KAPPA_HIER):
    out = {}
    for i, c in enumerate(cats):
        if c == "border":
            ok = True
            for m0 in (135, 588):
                m = obs[i, m0:m0 + 325].reshape(25, 13)
                edge = np.concatenate([m[0], m[-1], m[:, 0], m[:, -1]])
                ok = ok and edge.min() >= 2.0 and m[1:-1, 1:-1].max() < 0.5
        elif c == "lidar_wrap":
            ray = obs[i, 460:588]
            wrap = ray[[0, 1, 126, 127]]
            ok = len(set(wrap.tolist())) == 4 and wrap.min() >= 3.0 and np.delete(ray, [0, 1, 126, 127]).max() < 1.0
        elif c.startswith("slot"):
            ok = int(np.argmax(np.abs(obs[i, GAME_COLS]))) == int(c[4:]) and np.abs(obs[i, GAME_COLS]).max() >= 3.0
        elif c.startswith("tie"):
            lo, mid, hi = info["ties"][i]
            lg = ref["logits"][i]
            same_lane = (lo % 32 == mid % 32) if c == "tie_same_lane_lo" else (hi % 32 == mid % 32)
            ok = ref["code"][i] == lo and lg[lo] == lg[mid] == lg[hi] and same_lane and ref["gap"][i] > 4 * kappa * S["gap"][i]
        elif c == "tight":
            ok = 4 * kappa * S["gap"][i] < ref["gap"][i] < 8 * kappa * S["gap"][i] and ref["code"][i] == info["tight"][i][0]
        else:
            ok = True
        out.setdefault(c, []).append(bool(ok))
    if "heading_pre" in ref:
        out["heading_clip_high"] = [bool((ref["heading_pre"] > PI32).any())]
        out["heading_clip_low"] = [bool((ref["heading_pre"] < -PI32).any())]
        out["heading_inside"] = [bool((np.abs(ref["heading_pre"]) < 3.0).any())]
    return out


NULL_DONE_STEP = 2                 # the recurrence step launched with d_done = NULL (no row wipes)


def hier_recurrence_weights(w, strategic, info):
    """The designed weights without the tight logit pairs (their partner bias lowered by 10): a row carried by its state onto a
    tight pair's winner could not be made decisive by redrawing its observation.  The exact ties stay."""
    w = [a.copy() for a in w]
    b = w[hier_role_arrays(strategic)[44]]
    for c, c2 in info["tight"].values():
        b[c2] = np.float32(b[c] - 10.0)
    return w


def hier_recurrence_case(strategic, w, seed=0, kappa=KAPPA_HIER, n=300, steps=4):
    """Observations and done bytes for `steps` recurrent steps from a non-zero state, every row decisive with a margin of 2 along
    the fp64 chain (the GPU test feeds the reference the kernel's incoming state; the margin covers the difference)."""
    rng = np.random.default_rng(seed + 77)
    net = Hier(w)
    cats = [HIER_CATS[i % 3] for i in range(n)]
    state = hier_random_state(rng, n, net.ssz)
    state0 = state.copy()
    obs_all, done_all = [], []
    for s in range(steps):
        obs = np.stack([_hier_row(rng, c, net.ow) for c in cats])
        done = np.zeros(n, np.uint8) if s == NULL_DONE_STEP else DONE_BYTES[(np.arange(n) + s) % 4]
        ref, S, _ = _redraw_until_decisive(w, obs, state, done, cats, rng, kappa, margin=2.0)
        obs_all.append(obs)
        done_all.append(done)
        state = ref["state"].astype(np.float32)
    return state0, obs_all, done_all


def padded(obs, ld, width):
    """[n, ld] fp32 rows: the observation in the first `width` columns, NaN in the rest (a kernel that reads them fails)."""
    out = np.full((obs.shape[0], ld), np.nan, np.float32)
    out[:, :width] = obs[:, :width]
    return out


@functools.lru_cache(maxsize=None)
def pmc_case():
    """The designed PMC batch with its reference and sensitivities (built once per session)."""
    w, obs, cats, info = build_pmc_case()
    ref, S = pmc_eval(w, obs)
    return w, obs, cats, info, ref, S


@functools.lru_cache(maxsize=None)
def hier_case(strategic):
    w, obs, state, done, cats, info = build_hier_case(strategic)
    ref, S, _ = hier_eval(w, obs, state, done)
    return w, obs, state, done, cats, info, ref, S
