"""The clip-table batches of tests/clip_table_cases.py on the CPU: the oracle against the fp64 statement at every table size, every
category reached.  Without these checks tests/test_clip_table_cases_gpu.py could pass vacuously."""
import numpy as np
import pytest

import clip_table_cases as ct
import episode_cases as ec


@pytest.mark.parametrize("k", range(len(ct.CASES)))
def test_the_oracle_matches_the_statement(k, oracle_lib):
    ratios = ec.run_case(oracle_lib, ct.case(k), "host", oracle=True)
    print("case %d (n = %d, C = %d): %s" % (k, ct.CASES[k][0], ct.CASES[k][1], ratios))


@pytest.mark.parametrize("C", ct.SIZES)
def test_the_oracle_resets_on_the_exact_table(C, oracle_lib):
    print("C = %d: %s" % (C, ct.run_resets(oracle_lib, C, oracle=True)))


def test_the_batches_reach_every_category():
    edges = set()
    for k, case in enumerate(ct.CASES):
        n, C = case[0], case[1]
        ctx, before, cats, designed = ct.case(k)
        ref = ec.step_statement(ctx, before, before["state"].astype(np.float64))
        assert ec.reaches(ctx, before, ref, cats).all() and ec.decisive(ref).all()
        done = ref["done"]
        assert np.array_equal(done, np.array([c == "finish" for c in cats]))
        avg, p, cdf, win = ec.table(ctx, done, before["clip"], ref["reward_sum"], before["avg"])
        # weights over more than 12 decades, zero-weight clips; clips without a finisher keep the value set before the step
        assert p.max() / p[p > 0].min() > 1e12 and (p == 0).sum() >= 10
        assert np.array_equal(avg[win < 0], before["avg"][win < 0]) and (win < 0).sum() >= C - n
        assert np.all(avg <= 1.0) and np.all(np.diff(cdf) >= 0)
        if n > 1:                          # env 0 and env N - 1 finish on one clip: the highest env wins it
            assert done[0] and done[n - 1] and before["clip"][0] == before["clip"][n - 1] and win[before["clip"][0]] == n - 1
        if n == 4097:                      # finishers of ~2000 different clips in every 32-env block of the reset kernel
            fin = np.nonzero(done)[0]
            assert len(set(before["clip"][fin])) >= 2000 and len({i // 32 for i in fin}) == (n + 31) // 32
            assert (before["clip"][fin] > 3902).sum() >= (100 if C > 3903 else 0)
        for j, side in designed.values():
            edges |= {("first" if j == 0 and side > 0 else "last" if j == C - 2 and side < 0 else "inner", j > 3902, j >= 0.99 * C)}
        # the draws the statement makes: searchsorted equals the first-clip-above rule it replaced, the C - 1 fallback included
        u = np.concatenate([ec.uniforms(ctx["seed"], ctx["gid0"] + np.arange(n), before["episode"])[0], [1.0 - 1e-17, 1.0]])
        above = cdf[None, :] > u[:, None]
        assert np.array_equal(np.minimum(np.searchsorted(cdf, u, side="right"), C - 1), np.where(above.any(1), np.argmax(above, 1), C - 1))
    kinds = {e[0] for e in edges}
    assert {"first", "last", "inner"} <= kinds
    assert any(e[0] == "inner" and e[1] for e in edges) and any(e[0] == "inner" and e[2] for e in edges)
    assert {c[1] for c in ct.CASES} == set(ct.SIZES) and {c[0] for c in ct.CASES} == {1, 17, 4097}


@pytest.mark.parametrize("C", ct.SIZES)
def test_the_exact_table_ties_the_draw(C):
    """the designed envs' u1 equals a cdf edge exactly; the statement draws past the zero-weight clips after it"""
    ctx, avg, ep, edges, (rc, rt) = ct.reset_batch(C)
    (clip, *_ , u1), cdf = ct.reset_draw(ctx, avg, ctx["gid0"] + np.arange(ctx["n"]), ep)
    assert len(edges) == 4 and any(j >= 0.99 * C for j in edges.values()) and (C < 8192 or any(j >= 3902 for j in edges.values()))
    for env, j in edges.items():
        assert cdf[j] == u1[env] and clip[env] > j + 1 and avg[clip[env]] < 1.0 and np.all(avg[j + 1:clip[env]] == 1.0)
    assert set(rc) == {c for c in (0, 3902, 3903, C - 1) if c < C}
