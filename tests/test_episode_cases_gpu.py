"""The episode logic of the PMC step and reset kernels against the fp64 statement of tests/episode_cases.py, env by env, with no
env excluded: tracking reward, reward_sum, termination, the mocap clock, the hurdle-plate hand-over, the prioritized clip table and
the auto-reset draw, through every I/O path.

Exactly equal: done, F_TIME, F_CLIP, F_EPISODE_ID, F_OB_ID, the record columns and counters [0] and [1].  F_AVG_REWARD within 1 ulp
of the statement on the engine's own fp32 reward sums, F_SAMPLE_PROB within 8 ulp (device pow against libm).  Reward, reward_sum,
F_KIN_STATE, the observation and the reset rows within KAPPA S + 2^-23 |ref|.

KAPPA = 64.  Largest error / S measured on an H100 80GB HBM3 at a 400 W power limit, over two runs of these batches: observation 8.8,
reset observation 2.9, F_KIN_STATE 1.1, reset state and reset F_KIN_STATE 0.72, reward 0.64, reward_sum 0.07 (beyond its fp32
rounding); F_SAMPLE_PROB at most 3 ulp."""
import pytest

import episode_cases as ec

pytestmark = pytest.mark.gpu


# the I/O path of each batch: the 4097-env batch goes through record mode 2 (the trajectory columns one row block before the
# observation's), the two-CTA edge batches through the others; the edge-of-2^32 batch and the 4097 batch run every path below
CASE_IO = ("host", "pinned", "device1", "device2", "host", "device1", "device2")


@pytest.mark.parametrize("k", range(len(ec.CASES)))
def test_episode_logic_matches_the_statement(k, built):
    from lifelike_agility_and_play_b200 import _capi as capi
    ratios = ec.run_case(capi.load_cuda_library(), k, CASE_IO[k])
    print("case %d (n = %d, %s): %s" % (k, ec.CASES[k][0], CASE_IO[k], ratios))


@pytest.mark.parametrize("k,io", [(k, io) for k in (5, 6) for io in ec.IO_PATHS if io != CASE_IO[k]])
def test_every_io_path(k, io, built):
    """the 33-env batch (counter high word changing inside it) and the 4097-env batch through host, pinned and device memory,
    record modes 1 and 2"""
    from lifelike_agility_and_play_b200 import _capi as capi
    ratios = ec.run_case(capi.load_cuda_library(), k, io)
    print("case %d (%s): %s" % (k, io, ratios))
