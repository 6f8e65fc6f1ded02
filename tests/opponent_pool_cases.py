"""Statement of the opponent pool's assign step (llq_hier_policy_forward_pool, csrc/llq_policy_hier.cu hier_pool_assign_kernel): the
cutoffs of a probability vector, the per-row draw, the record, and the bucketing of rows by model into CTA segments."""
import numpy as np

import policy_cases as pc

KROWS = 8                     # rows per CTA of the policy kernels
Q_POOL = 65                   # Philox counter word 1 of the draw (0..63: Gumbel draws, 64: the heading)
TWO32 = 1 << 32


def cutoffs(probs):
    """t_k = floor(cum_k / cum_{K-1} 2^32) with cum_k the SEQUENTIAL fp64 sum p_0 + ... + p_k; t_{K-1} = 2^32 (uint64)."""
    p = [float(x) for x in probs]
    cum, s = [], 0.0
    for x in p:
        s += x
        cum.append(s)
    t = [int(np.floor(c / s * 4294967296.0)) for c in cum[:-1]] + [TWO32]
    return np.array(t, np.uint64)


def draw_words(gid, seed, counter):
    """r = word x of Philox4x32-10 at counter (low 32 bits of gid, 65, counter lo, counter hi), key (seed lo, seed hi)."""
    gid = np.asarray(gid, np.int64)
    c = pc.philox4x32(gid.astype(np.uint64) & np.uint64(0xFFFFFFFF), Q_POOL, counter & 0xFFFFFFFF, counter >> 32, seed & 0xFFFFFFFF, seed >> 32)
    return c[0].astype(np.int64)


def pick(r, t):
    """The smallest k with r < t_k."""
    r = np.asarray(r, np.int64)
    return np.array([int(np.flatnonzero(int(x) < t.astype(object))[0]) for x in r], np.int32)


def assign(model, done, t, n_models, row_gid0, seed, counter):
    """(model after the draws, record per row) of one call: rows with done != 0 draw (done None: no draws); the record is the model, or
    -1 outside [0, K)."""
    model = np.array(model, np.int32)
    if done is not None:
        d = np.flatnonzero(np.asarray(done) != 0)
        if len(d):
            model[d] = pick(draw_words(row_gid0 + d, seed, counter), t)
    rec = np.where((model >= 0) & (model < n_models), model, -1).astype(np.float32)
    return model, rec


def bucket(model, n_models):
    """(seg_cta [K + 1], entries [seg_cta[K] * 8]): model k's rows in ascending order from entry seg_cta[k] * 8, padded with -1 to a
    multiple of 8; rows outside [0, K) are in no segment."""
    model = np.asarray(model)
    seg_cta, entries = [0], []
    for k in range(n_models):
        rows = np.flatnonzero(model == k).tolist()
        rows += [-1] * ((-len(rows)) % KROWS)
        entries += rows
        seg_cta.append(seg_cta[-1] + len(rows) // KROWS)
    return np.array(seg_cta, np.int64), np.array(entries, np.int64)


def cta_rows(model, n_models):
    """For every CTA of the pool forward's grid of ceil(n / 8) + K: (model, its 8 row entries), or None past the last segment."""
    seg_cta, entries = bucket(model, n_models)
    grid = (len(model) + KROWS - 1) // KROWS + n_models
    out = []
    for b in range(grid):
        if b >= seg_cta[-1]:
            out.append(None)
            continue
        k = int(np.flatnonzero(seg_cta[:n_models] <= b)[-1])
        out.append((k, entries[b * KROWS:(b + 1) * KROWS]))
    return out


def adjacent_words(seed, counter, lo, n):
    """Two global rows g_a, g_b in [lo, lo + n) whose draw words are r_b = r_a + 1 (searched out; the numpy Philox is pinned to the
    Random123 known answers in test_policy_cases.py)."""
    g = lo + np.arange(n, dtype=np.int64)
    r = draw_words(g, seed, counter)
    o = np.argsort(r, kind="stable")
    d = np.flatnonzero(np.diff(r[o]) == 1)
    assert len(d), "no adjacent pair of draw words in the searched range"
    return int(g[o[d[0]]]), int(g[o[d[0] + 1]]), int(r[o[d[0]]])
