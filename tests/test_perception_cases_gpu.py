"""The step kernel's perception rays against the fp64 caster, ray by ray with no exclusions (run with -m gpu on an H100).

The batches are tests/perception_cases.py's designed poses, stepped once with the physics off (one sub-step, no solver iteration,
no PD torque, no gravity, no push, zero velocities), so the observation is a function of the pose that was set, the env's boxes,
target and flag.  Every ray of every env is decisive: its branch (hit or miss, first box and face, origin inside a box, footprints
of a down ray) holds with every box grown and shrunk by 1e-4 m.  The categories reach the EPMC corridor's candidate windows at their
edge, the 64-bit box mask's high word (element 3 with 34 boxes), the culling pad of ray_boxlist, a base inside a box or a wall, the
1-D rays' z window, the slab's edge, and the SEPMC fast paths (ray_arena_inside and its wall-top check, the flag's cull radius, the
closed-form down ray and its off-slab fallback).  Batch sizes (21, 45, 46) leave padded rows in the last warp.

Bar per value: A * max(1, |ref|) + 4 S, S = the caster's largest change when the ray's origin and end move by 1e-5 m (the reach
of fp32 inputs on a decisive ray; grazing hits on 20 m rays make it large).  A is a round number at least 4x the largest error
beyond 4 S (the A each value needs) measured on an H100 80GB HBM3, over all five cases.  Every ray of every case is within 4 S
alone; the largest absolute ray errors are 1.2e-6 (element 0), 1.5e-4 (a grazing 20 m corridor ray, within its 4 S), 8.4e-6
(corridor front rays) and 5.8e-5 (SEPMC front rays).  The tails need 2.3e-7 (EPMC target direction) and 8.0e-7 (SEPMC vectors,
fp32 rounding of the opponent block) at a 400 W power limit; 5.4e-7 and 1.1e-6 on an earlier batch at 700 W:
  measured 1.1e-6  -> A = 1e-5
"""
import numpy as np
import pytest

from lifelike_agility_and_play_b200 import _capi as capi
from test_perception_cases import CASES, assert_pose_kept, designed, post_pose_decisive, prepared, reference_rows, step

pytestmark = pytest.mark.gpu

A = 1e-5


@pytest.mark.parametrize("kind,element", CASES)
def test_cuda_perception_matches_the_caster_ray_by_ray(kind, element, built, oracle_lib):
    n, states, _, cats, vis = designed(kind, element, oracle_lib)
    cpu = prepared(oracle_lib, kind, element, oracle_lib)
    gpu = prepared(capi.load_cuda_library(), kind, element, oracle_lib, src=cpu)
    obs, st, aux, boxes, nbox = step(gpu)
    aux_cpu = step(cpu)[2]
    gpu.close(); cpu.close()
    assert_pose_kept(st, states, qtol=2.5e-7)        # the kernel turns the quaternion into the inertial frame and back in fp32
    assert post_pose_decisive(kind, st, aux, boxes, nbox).all()
    if kind == "sepmc":
        assert not aux[:, capi.AUX_SWITCH_FLAG].any(), "a flag switch moved the flag during the step"
        # the flag blocks or clears every visibility segment by >= 1 cm: the flags are equal, and equal to the builder's
        assert np.array_equal(aux[:, capi.AUX_OPPO_VISIBLE], aux_cpu[:, capi.AUX_OPPO_VISIBLE]) and np.array_equal(aux[:, capi.AUX_OPPO_VISIBLE] != 0, vis), (aux[:, capi.AUX_OPPO_VISIBLE], aux_cpu[:, capi.AUX_OPPO_VISIBLE], vis)
    ref, S = reference_rows(kind, st, aux, boxes, nbox)
    got = obs[:, 135:].astype(np.float64)
    err = np.abs(got - ref)
    scale = np.maximum(1.0, np.abs(ref))
    need = (err - 4 * S) / scale                          # the smallest A each value needs
    blocks = {"down": slice(0, 325), "1-D": slice(325, 453), "front": slice(453, 778), "tail": slice(778, None)}
    print("%s element %d, %d envs: %s" % (kind, element, n, "; ".join(
        "%s max err %.1e (A needed %.1e)" % (k, err[:, s].max(), max(need[:, s].max(), 0.0)) for k, s in blocks.items())))
    bar = A * scale + 4 * S
    bad = np.argwhere(err > bar)
    assert len(bad) == 0, [(int(i), cats[i // 2 if kind == "sepmc" else i], int(j) + 135, got[i, j], ref[i, j], S[i, j]) for i, j in bad[:10]]
