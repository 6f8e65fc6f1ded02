"""fp64 statement of the EPMC corridor generator (elements 1-3: walls with hurdles, bars or cubes) and designed batches of keys on
which every draw of it is decisive (host only, numpy float64 and Python floats).

The statement restates BSE's `_generate_random_width_walls` and `_create_hurdles` / `_create_holes` / `_create_cubes(easy)` driven by
the engine's terrain stream:

  draws     draw k is slot k & 3 of stream_uniforms(seed, global env id, episode id before the reset, 5, k >> 2);
            uniform(lo, hi) = lo + u (hi - lo) with double bounds, an unfused multiply and add (Python's); randint(lo, hi) =
            lo + floor(u (hi - lo))
  order     wall width, wall gap, object count; per object (hurdle) height and depth / (bar) depth and gap height / (cube set) the
            spacing; the target offset after pass 0 (+-1 m for elements 1 and 2, +-3 m for element 3); then pass 1
  boxes     the two walls (+y first), then the pass-0 objects, then the pass-1 objects; a row is the fp32 rounding of the double
            centre and of the half extents lx / 2, ly / 2, lz / 2
  aux       TARGET_X = the target x in double, TARGET_Y = 0, INIT_POS_DIFF_LEN = LAST_POS_DIFF_LEN = |TARGET_X| (the reset kernel
            writes fabs of the same double): all four exactly equal on every engine

The DFMA into which nvcc contracts `lo + u (hi - lo)` and the unfused form round alike whenever hi - lo is an integer below 2^20:
u = (x + 1/2) / 2^32 has at most 33 significant bits, so u (hi - lo) is exact.  That holds for the depths uniform(1, 3), the
target offsets uniform(-1, 1) and uniform(-3, 3), the cube spacing uniform(0, 1) and the wall gap ranges of every batch here, so
no draw of them separates the two forms, and the target x cannot.  For the wall width (0.48 wide on the shipped range), the hurdle
height (0.1) and the bar gap (0.05 on the default range) the two forms differ by one double ulp in some draws, but an fp32 box value
moves only when that double lies within an ulp of an fp32 rounding boundary (about 2^-29 of those draws): `fma_search` found none
over 2^18 keys on each of [0.02, 0.5], [0.05, 0.15], [0.25, 0.3], [0.1, 1.3] and [0.1, 0.3], so the batches hold no such category
and the kernel's contraction is left as it is.

Ids e and e + 2^32 draw alike (the key takes the episode's low 32 bits), as in the other EPMC streams.

Categories, each asserted per env on the statement (`reaches`):
  count_1, count_max   1 and 9 hurdles / bars (20 boxes), 1 and 4 cube sets (10 and 34 boxes)
  count_below/above    the count's u (hi - lo) 1e-9 to 1e-6 below / above an interior integer: a uniform of fewer than 53 bits, or
                       a randint with hi - lo + 1, flips it
  f32_bound            the fp32-rounded bounds give a different fp32 box value than the double bounds (every range on which some
                       draw does so)
The designed envs alternate episode ids below and above 2^32 (a single env takes one above), the other envs draw ids on both sides,
and the batches start at global id 0 or 2^32 - 5.
"""
import functools

import numpy as np

from epmc_episode_cases import stream_uniforms
from lifelike_agility_and_play_b200 import _capi as capi

SEED = 20261019
GID0 = (0, 2 ** 32 - 5)
MAX_DRAWS = 40                       # elements 1 and 2 with 9 objects: 2 + 1 + 2 * 9 * 2 + 1 (element 3: at most 12)
# terrain ranges (wall width, wall gap, hole gap) of the batches
RANGES = {
    "shipped": ((0.02, 0.5), (1.0, 20.0), (0.25, 0.25)),      # the generator's config (example_epmc_train.sh), tests/test_golden_epmc.py
    "default": ((0.02, 0.5), (1.0, 20.0), (0.25, 0.3)),       # llq_config's defaults: hole gap [0.25, 0.3] (BSE:372-373)
    "equal": ((0.3, 0.3), (2.5, 2.5), (0.3, 0.3)),            # lo == hi
    "odd": ((0.1, 1.3), (1.3, 7.3), (0.1, 0.3)),              # no bound is an fp32 number
}
CATS = ("count_1", "count_max", "count_below", "count_above", "f32_bound")


def f32(x):
    return float(np.float32(x))


def f32_bounds(ranges):
    return tuple((f32(lo), f32(hi)) for lo, hi in ranges)


def engine_config(element, ranges, gid0, **over):
    from test_golden_epmc import terrain_cfg, terrain_gold
    (wl, wh), (gl, gh), (hl, hh) = RANGES[ranges]
    cfg = terrain_cfg(terrain_gold(element))
    cfg.update(wall_width_lo=wl, wall_width_hi=wh, wall_gap_lo=gl, wall_gap_hi=gh, hole_gap_lo=hl, hole_gap_hi=hh,
               global_env_offset=gid0, seed=SEED, push_enabled=0)
    cfg.update(over)
    return cfg


# ------------------------------------------------------------------------------------------------------------ the statement
def draws(seed, gid, ep, count=MAX_DRAWS):
    """[n, count] terrain draws of the keys (gid, ep)"""
    gid, ep = np.atleast_1d(gid), np.atleast_1d(ep)
    return np.concatenate([stream_uniforms(seed, gid, ep, 5, j).T for j in range((count + 3) // 4)], 1)[:, :count]


def corridor(element, ranges, u):
    """(rows [nbox, 6] in double before the fp32 rounding, target x) of one env from its draws u (BSE:170-263, 308-500)"""
    it = iter(float(x) for x in u)

    def uniform(lo, hi):
        return lo + next(it) * (hi - lo)

    def randint(lo, hi):
        return lo + int(np.floor(next(it) * (hi - lo)))

    rows = []

    def box(cx, cy, cz, lx, ly, lz):
        rows.append((cx, cy, cz, lx / 2, ly / 2, lz / 2))

    (wl, wh), (gl, gh), (hl, hh) = ranges
    width = uniform(wl, wh)
    gap = uniform(gl, gh)
    box(5.0, gap / 2.0 + width / 2.0, 1.0, 200.0, width, 2.0)
    box(5.0, -(gap / 2.0 + width / 2.0), 1.0, 200.0, width, 2.0)
    cur = 0.0
    if element in (1, 2):
        n = randint(1, 10)
        for p in range(2):
            for _ in range(n):
                if element == 1:
                    h = uniform(0.05, 0.15)
                    d = uniform(1.0, 3.0)
                    box(cur + d / 2, 0.0, h / 2, 0.1, gap, h)
                else:
                    d = uniform(1.0, 3.0)
                    g = uniform(hl, hh)
                    box(cur + d / 2, 0.0, 0.3 / 2 + g, 0.1, gap, 0.3)
                cur += d + 0.1
            if p == 0:
                tgx = cur + uniform(-1.0, 1.0)
    else:
        ns = randint(1, 5)
        for p in range(2):
            for _ in range(ns):
                cur += uniform(0.0, 1.0)
                box(1.75 + cur, 0.0, 0.25 / 2, 0.5, gap, 0.25)
                box(1.0 + cur, 0.0, 0.1 / 2, 0.5, gap, 0.1)
                cur += 1.75 + 0.25
                box(cur + 0.5, 0.0, 0.25 / 2, 0.5, gap, 0.25)
                box(cur + 1.25, 0.0, 0.1 / 2, 0.5, gap, 0.1)
                cur += 3.0
            if p == 0:
                tgx = cur + uniform(-3.0, 3.0)
    return np.array(rows), tgx


def statement(element, ranges, seed, gid, ep):
    """the engine's view of resets of envs gid whose episode id before the reset is ep: boxes [n, MAX_BOXES, 6] float32 (zero
    past nbox), nbox [n], aux {slot: [n] double}; `ranges` are the (lo, hi) pairs of wall width, wall gap, hole gap"""
    U = draws(seed, gid, ep)
    n = len(U)
    boxes = np.zeros((n, capi.MAX_BOXES, 6), np.float32)
    nbox = np.zeros(n, np.int32)
    tgx = np.zeros(n)
    for i in range(n):
        rows, tgx[i] = corridor(element, ranges, U[i])
        nbox[i] = len(rows)
        boxes[i, :len(rows)] = rows.astype(np.float32)
    aux = {capi.AUX_TARGET_X: tgx, capi.AUX_TARGET_Y: np.zeros(n), capi.AUX_INIT_POS_DIFF_LEN: np.abs(tgx),
           capi.AUX_LAST_POS_DIFF_LEN: np.abs(tgx)}
    return dict(boxes=boxes, nbox=nbox, aux=aux)


# ------------------------------------------------------------------------------------------------------------ designed keys
def count_range(element):
    return 9 if element in (1, 2) else 4            # randint(1, 10) / randint(1, 5): u (hi - lo) with hi - lo = 9 / 4


def count_of(element, u2):
    return 1 + np.floor(u2 * count_range(element)).astype(np.int64)


def _edge(element, u2, side):
    x = u2 * count_range(element)
    k = np.round(x)
    d = side * (x - k)
    return (d >= 1e-9) & (d <= 1e-6) & (k > 0) & (k < count_range(element))


def _f32_differs(element, ranges, U):
    """[n] bool: the statement's boxes with the fp32-rounded bounds differ from those with the double bounds"""
    out = np.zeros(len(U), bool)
    for i in range(len(U)):
        a = corridor(element, RANGES[ranges], U[i])[0].astype(np.float32)
        b = corridor(element, f32_bounds(RANGES[ranges]), U[i])[0].astype(np.float32)
        out[i] = not np.array_equal(a, b)
    return out


def _want(element, ranges, cat, U):
    if cat == "count_1":
        return count_of(element, U[:, 2]) == 1
    if cat == "count_max":
        return count_of(element, U[:, 2]) == count_range(element)
    if cat in ("count_below", "count_above"):
        return _edge(element, U[:, 2], -1 if cat == "count_below" else 1)
    return _f32_differs(element, ranges, U)


def _search(element, ranges, cat, gid, high, rng):
    """an episode id (below 2^32, or from 2^32 up when `high`) whose draws reach `cat` for global id gid"""
    chunk = 2 ** 20 if cat in ("count_below", "count_above") else 256
    for _ in range(40):
        ep = int(rng.integers(1, 2 ** 31)) + np.arange(chunk, dtype=np.int64) + (2 ** 32 if high else 0)
        U = draws(SEED, np.full(chunk, gid), ep, 4 if cat != "f32_bound" else MAX_DRAWS)
        ok = np.flatnonzero(_want(element, ranges, cat, U))
        if len(ok):
            return int(ep[ok[0]])
    raise RuntimeError("no episode id reaches %s" % cat)


@functools.lru_cache(maxsize=None)
def cats_of(element, ranges):
    """the designed categories of a batch: f32_bound where 256 sample draws reach it (with lo == hi it is all or nothing)"""
    U = draws(SEED, np.zeros(256, np.int64), np.arange(256, dtype=np.int64))
    return CATS if _f32_differs(element, ranges, U).any() else CATS[:4]


@functools.lru_cache(maxsize=None)
def keys(element, ranges, n, gid0):
    """(episode ids before the reset [n], categories [n]): env i < len(cats) is designed for cats[i] (ids alternating below and
    above 2^32), the others draw random ids on both sides of 2^32"""
    rng = np.random.default_rng([element, n, gid0, len(ranges)])
    ep = np.where(rng.random(n) < 0.5, rng.integers(0, 2 ** 31, n), rng.integers(2 ** 32, 2 ** 32 + 2 ** 31, n)).astype(np.int64)
    cl = cats_of(element, ranges)
    cats = ["random"] * n
    for i in range(min(n, len(cl))):
        cats[i] = cl[i]
        ep[i] = _design(element, ranges, cl[i], gid0 + i, (i + (n == 1)) % 2 == 1)
    return ep, tuple(cats)


@functools.lru_cache(maxsize=None)
def _design(element, ranges, cat, gid, high):
    # the count categories do not depend on the ranges: one search serves all of them
    key_ranges = ranges if cat == "f32_bound" else "shipped"
    return _search(element, key_ranges, cat, gid, high, np.random.default_rng([element, gid % 2 ** 32, CATS.index(cat), high,
                                                                                 len(key_ranges)]))


def reaches(element, ranges, gid, ep, cats):
    """[n] bool: env i reaches cats[i] on the statement (random envs reach nothing in particular)"""
    U = draws(SEED, gid, ep)
    ok = np.ones(len(ep), bool)
    for i, c in enumerate(cats):
        if c != "random":
            ok[i] = bool(_want(element, ranges, c, U[i:i + 1])[0])
    return ok


def fma_search(lo, hi, gid=0, count=2 ** 20):
    """the number of draws among `count` keys whose DFMA lo + u (hi - lo) and unfused form round to different fp32 values of
    the quantity and of its half (exact rational arithmetic for the DFMA)"""
    from fractions import Fraction
    u = draws(SEED, np.full(count, gid), np.arange(count, dtype=np.int64), 1)[:, 0]
    w = hi - lo
    unf = lo + u * w
    near = np.flatnonzero(np.abs(np.float32(unf).astype(np.float64) - unf) > 0)      # all draws but exact fp32 values
    hits = 0
    for i in near:
        fus = float(Fraction(float(u[i])) * Fraction(w) + Fraction(lo))
        hits += f32(fus) != f32(unf[i]) or f32(fus / 2) != f32(unf[i] / 2)
    return hits
