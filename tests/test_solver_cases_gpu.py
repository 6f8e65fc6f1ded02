"""The step kernel's constraint solver against the fp64 oracle, env by env with no exclusions (run with -m gpu on an H100).

The batches are tests/solver_cases.py's designed states: one sub-step (llq_config.substeps = 1) from a pose on which every discrete
decision -- contact make / break, owner static, joint-limit row, split-impulse side -- is at least 1 mm / 5 mrad from its branch, so
both engines solve the same rows and the projected Gauss-Seidel sweep with a fixed iteration count is a continuous function of the
input.  The CTAs reach every lane mapping of the solver (split 16, borrow, two-pass, empty pair, 32 rows beside an empty partner,
both caps, the copies of env N - 1 in a partly filled CTA), on the PMC ground, against the SEPMC arena walls and on the boxes and
edge cylinders of two EPMC corridors.

Bars (block-relative state error, and per-sphere normal impulse error over max(1, the env's largest impulse)) for solver_iters
0 / 1 / 10, per env: the smallest round number at least 4x the largest error measured on an H100 80GB HBM3 (700 W power limit).
  TOL1, every env whose contacts are all with the ground (the plane z = 0 is exact in both engines), in all four batches:
    iters 0   measured 2.0e-06  -> 1e-5   (dynamics + the application of the warm start)
    iters 1   measured 2.6e-06  -> 2e-5   (one sweep: no Gauss-Seidel amplification)
    iters 10  measured 2.7e-06  -> 2e-5   (the production setting)
  TOL1_FP32_STATICS, envs with a contact on an SEPMC arena wall or a corridor box / edge cylinder.  The kernel holds those positions in
  fp32 (the walls at 2.495f = 2.495 - 1.1e-7 m, a box at x = 5 m to within 2.4e-7 m); through the contact target -dist / dt (1.1e-7 m
  is 5.5e-5 m/s) and the normals of box edges a few mm from the sphere centre that offset, not the solver, sets these bars -- the
  ground-only envs of the same batches stay within TOL1:
    iters 0   measured 8.2e-06  -> 5e-5
    iters 1   measured 1.0e-04  -> 5e-4
    iters 10  measured 1.5e-04  -> 1e-3

The same bars hold the extensions of the pin, unchanged.  Largest error over the bar that applies, at any of solver_iters 0 / 1 / 10,
measured on an H100 80GB HBM3 (700 W power limit):
  EPMC flat arena (element 0)                                           0.21
  corridor element 2, the bars (bottom faces, corners inside, bottom-edge cylinders, ground and bar at once)   0.22
  knee_contacts 0 (feet): PMC 0.20, SEPMC 0.22, corridor element 1 0.24
  knee_contacts 1 (feet, knee wheels, one contact per leg): PMC 0.19, SEPMC 0.46 (9.1e-6 at iters 10 on the ground), corridor 0.17
  pushes and clamps, per state block: EPMC flat 0.17, SEPMC 0.24, corridor element 1 0.19
"""
import numpy as np
import pytest

import solver_cases as sc
from lifelike_agility_and_play_b200 import _capi as capi
from test_parity_gpu import blockrel
from test_solver_cases import DYN_KINDS, KINDS, LEGACY, blockwise, designed_batch, designed_dynamics, make

pytestmark = pytest.mark.gpu

TOL1 = {0: 1e-5, 1: 2e-5, 10: 2e-5}
TOL1_FP32_STATICS = {0: 5e-5, 1: 5e-4, 10: 1e-3}
LAM_FLOOR = 1e-6          # N s: impulses below this count as zero on both sides
FIELDS = {"pmc": (capi.F_STATE, capi.F_WARMSTART, capi.F_OBS, capi.F_TIME, capi.F_CLIP, capi.F_REWARD_SUM),
          "other": (capi.F_STATE, capi.F_WARMSTART, capi.F_OBS, capi.F_TIME, capi.F_AUX, capi.F_EPISODE_ID, capi.F_REWARD_SUM)}


def one_step(gpu, cpu, kind, states, warm, actions, aux=None):
    """teacher-forced sub-step from the designed states; returns (state err per env, impulse err per env, counters gpu, cpu)"""
    cpu.set(capi.F_STATE, states); cpu.set(capi.F_WARMSTART, warm)
    if aux is not None:
        cpu.set(capi.F_AUX, aux)
    for f in FIELDS["pmc" if kind == "pmc" else "other"]:
        gpu.set(f, cpu.get(f))
    g0, c0 = gpu.counters().copy(), cpu.counters().copy()
    gpu.step(actions); cpu.step(actions)
    e = blockrel(gpu.get(capi.F_STATE), cpu.get(capi.F_STATE))
    lg, lc = gpu.get(capi.F_WARMSTART).astype(np.float64), cpu.get(capi.F_WARMSTART).astype(np.float64)
    scale = np.maximum(np.abs(lc).max(1), 1e-30)
    el = np.abs(lg - lc).max(1) / np.maximum(scale, 1.0)
    big = np.maximum(np.abs(lg), np.abs(lc)) > LAM_FLOOR
    same_set = np.all(((lg != 0) == (lc != 0)) | ~big, axis=1)
    return e, el, same_set, gpu.counters() - g0, cpu.counters() - c0


def compare(kind, element, states, decs, blob, small_mocap, oracle_lib, actions=None, aux=None, blocks=False, **over):
    """every env of a designed batch, one sub-step on both engines at solver_iters 0 / 1 / 10, with and without a warm start: the
    rows solved and dropped are equal, so is the set of spheres with a normal impulse, and the state (blocks: each state block on its
    own) and the impulses are within the bars.  Returns the largest error per iteration count over the bar that applies."""
    n = len(states)
    rng = np.random.default_rng(7)
    warm_nz = rng.uniform(0.0, 3.0, (n, 32)).astype(np.float32)       # also on spheres without contact: both engines must drop it
    a = np.clip(0.3 * rng.standard_normal((n, 12)), -1, 1).astype(np.float32)
    actions = a if actions is None else actions
    off_ground = np.array([d["n_off_ground"] > 0 for d in decs])      # a wall, box or edge-cylinder contact: TOL1_FP32_STATICS
    print("  %d of %d envs touch a wall, box or edge cylinder" % (off_ground.sum(), n))
    ratio = {}
    for iters in (0, 1, 10):
        bar = np.where(off_ground, TOL1_FP32_STATICS[iters], TOL1[iters])
        worst = {True: 0.0, False: 0.0}
        ratio[iters] = 0.0
        for warm in (np.zeros((n, 32), np.float32), warm_nz):
            gpu = make(capi.load_cuda_library(), kind, n, blob, small_mocap, element, solver_iters=iters, **over)
            cpu = make(oracle_lib, kind, n, blob, small_mocap, element, solver_iters=iters, **over)
            e, el, same, cg, cc = one_step(gpu, cpu, kind, states, warm, actions, aux)
            if blocks:
                per = blockwise(gpu.get(capi.F_STATE), cpu.get(capi.F_STATE))
                e = np.max(np.stack(list(per.values())), axis=0)
            gpu.close(); cpu.close()
            for k in (True, False):
                if (off_ground == k).any():
                    worst[k] = max(worst[k], np.maximum(e, el)[off_ground == k].max())
            ratio[iters] = max(ratio[iters], float(np.max(np.maximum(e, el) / bar)))
            assert (cg[2], cg[3], cg[5]) == (cc[2], cc[3], cc[5]), ("rows solved / dropped", iters, cg[:6], cc[:6])
            assert same.all(), ("envs whose set of spheres with a normal impulse differs", np.flatnonzero(~same))
            assert np.all(e < bar), ("state", iters, np.flatnonzero(e >= bar), e.max())
            assert np.all(el < bar), ("impulse", iters, np.flatnonzero(el >= bar), el.max())
        print("  solver_iters %2d: max state / impulse err %.1e on the ground alone (bar %.0e), %.1e with a wall, box or cylinder (bar %.0e)" % (
            iters, worst[False], TOL1[iters], worst[True], TOL1_FP32_STATICS[iters]))
    return ratio


@pytest.mark.parametrize("kind,element", KINDS)
def test_designed_substeps_match_the_oracle_env_by_env(kind, element, built, blob, small_mocap, oracle_lib):
    states, decs = designed_batch(kind, oracle_lib, blob, small_mocap, element)
    mapping, reached = sc.warp_cases([d["nc"] for d in decs], [d["nl"] for d in decs])
    print("%s element %d: %d envs, mapping cases %s" % (kind, element, len(states), sorted(reached)))
    assert reached & {"two_pass", "borrow", "contact_cap", "limit_cap"}, "the batch reaches none of the solver's heavy paths"
    ratio = compare(kind, element, states, decs, blob, small_mocap, oracle_lib)
    print("  largest error over its bar: %s" % ratio)


@pytest.mark.parametrize("kind,element,rule", LEGACY)
def test_legacy_contact_sets_match_the_oracle_env_by_env(kind, element, rule, built, blob, small_mocap, oracle_lib):
    """knee_contacts 0 and 1: the feet alone, or feet and knee wheels with one contact per leg (the deeper one, in leg order)"""
    states, decs = designed_batch(kind, oracle_lib, blob, small_mocap, element, rule)
    print("%s element %d rule %d: %d envs, mapping cases %s" % (kind, element, rule, len(states),
                                                              sorted(sc.warp_cases([d["nc"] for d in decs], [d["nl"] for d in decs])[1])))
    ratio = compare(kind, element, states, decs, blob, small_mocap, oracle_lib, knee_contacts=rule)
    print("  largest error over its bar: %s" % ratio)


@pytest.mark.parametrize("kind,element", DYN_KINDS)
def test_pushes_and_clamps_match_the_oracle_env_by_env(kind, element, built, blob, small_mocap, oracle_lib):
    """pushes inside their window, on the first sub-step after a redraw and just after the window; the PD target and torque clamps;
    velocities at the +-max_coord_vel bound before and after the impulses -- compared per state block"""
    states, decs, aux, acts, cases, _ = designed_dynamics(kind, oracle_lib, blob, small_mocap, element)
    print("%s element %d: %d envs" % (kind, element, len(states)))
    ratio = compare(kind, element, states, decs, blob, small_mocap, oracle_lib, actions=acts, aux=aux, blocks=True, push_enabled=1)
    print("  largest error over its bar: %s" % ratio)


# ---------------------------------------------------------------------------------------------------------------- placement
def _placements(rng, blob, oracle_lib, small_mocap):
    """Two designed robots -- X (light: <= 16 rows) and H (heavy: 17..31 rows) -- each in four batches: among airborne robots (lifted
    1 m so they stay airborne for a whole policy step), beside a partner of the other weight, in a CTA of 16 heavy robots, and as
    env N - 1 of a batch of 20 (its copies fill the last CTA).  Returns {subject: [(name, states, index of the subject)]}."""
    S = sc.Statics()
    X, dx = sc.robot(rng, S, "light", n_viol=2, k_ground=2)
    H = sc.robot(rng, S, "heavy")[0]
    nx = 3 * dx["nc"] + dx["nl"]
    kw = dict(sc.KINDS["heavy"][0]); kw.update(n_viol=2, k_ground=6)
    P = sc.sample(rng, S, lambda c, l: 17 <= 3 * c + l <= 32 - nx, **kw)[0]           # a heavy partner that leaves X lanes to borrow
    air = np.stack([sc.robot(rng, S, "air")[0] for _ in range(19)]); air[:, 2] += 1.0
    heavy = np.stack([sc.robot(rng, S, "heavy")[0] for _ in range(15)])
    out = {}
    for name, s, other in (("X", X, P), ("H", H, X)):
        out[name] = [("among airborne", np.concatenate([s[None], air[:15]]), 0),
                     ("beside a partner", np.stack([s, other]), 0),      # the partner is env N - 1: its copies fill the CTA
                     ("all-heavy CTA", np.concatenate([heavy, s[None]]), 15),
                     ("env N-1 of a ragged batch", np.concatenate([air, s[None]]), 19)]
    return out


def _counts(states):
    d = [sc.decisions(s, sc.Statics()) for s in states]
    return [x["nc"] for x in d], [x["nl"] for x in d]


PLACEMENT_BAR = 1e-7       # 4x the largest difference measured on an H100 80GB HBM3 (700 W): 0 with 1 sub-step, 1.5e-08 with 10


@pytest.mark.parametrize("substeps", [1, 10])
def test_a_robots_result_does_not_depend_on_its_placement(substeps, built, blob, small_mocap, oracle_lib):
    """The pairing moves a robot's rows to other lanes, never to other arithmetic: wherever its rows start at the same lane of a
    half-warp (solver_cases.lane_offset) the outputs are bit-identical -- a padded sweep step adds 0 * delta and a partner's lane +0 to
    the sums; elsewhere only the addition order of the impulse sums differs.  With 10 sub-steps the pairing of later sub-steps depends
    on the partners' contacts: bit identity is asserted where every partner is airborne or a copy of the robot."""
    rng = np.random.default_rng(11)
    runs = _placements(rng, blob, oracle_lib, small_mocap)
    for subject, places in runs.items():
        outs = []
        for name, states, idx in places:
            n = len(states)
            gpu = make(capi.load_cuda_library(), "pmc", n, blob, small_mocap, substeps=substeps)
            cpu = make(oracle_lib, "pmc", n, blob, small_mocap, substeps=substeps)
            cpu.set(capi.F_STATE, states); cpu.set(capi.F_WARMSTART, np.zeros((n, 32), np.float32))
            for f in FIELDS["pmc"]:
                gpu.set(f, cpu.get(f))
            gpu.step(np.zeros((n, 12), np.float32))
            mapping = sc.warp_cases(*_counts(states))[0]
            case = [x[6] for x in mapping if idx in (x[2], x[3])][0]
            print("%s, %d sub-steps: %s -- first sub-step in a %s warp, rows from lane offset %d" % (
                subject, substeps, name, case, sc.lane_offset(mapping, idx)))
            outs.append((name, np.concatenate([gpu.get(capi.F_STATE)[idx], gpu.get(capi.F_WARMSTART)[idx]]), sc.lane_offset(mapping, idx)))
            gpu.close(); cpu.close()
        ref_name, ref, ref_off = outs[0]
        for name, out, off in outs[1:]:
            diff = float(np.max(np.abs(out.astype(np.float64) - ref) / np.maximum(1.0, np.abs(ref))))
            identical = off == ref_off and (substeps == 1 or name.startswith("env N-1"))
            print("%s, %d sub-steps: %s (lane offset %d) vs %s (%d): max rel diff %.1e%s" % (
                subject, substeps, name, off, ref_name, ref_off, diff, " (bit-identical expected)" if identical else ""))
            if identical:
                assert np.array_equal(out, ref), (subject, name, diff)
            else:
                assert diff < PLACEMENT_BAR, (subject, name, diff)
