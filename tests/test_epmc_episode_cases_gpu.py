"""The EPMC episode logic of the step and reset kernels against the fp64 statement of tests/epmc_episode_cases.py, env by env,
with no env excluded: commands, reach, timeup, fall, `bad`, the joystick and corridor rewards, the push schedule, the auto-reset
and masked-reset draws and rows, through every I/O path.

Exactly equal: done, the record columns, counters [0] and [1], F_EPISODE_ID, F_NBOX, and the aux counter, cmd_freq, cmd_draws,
push_count and push_draws.  Within KAPPA S + 2^-23 |ref|: reward, reward_sum, the other aux slots (target, target_spd,
target_angle, last_pos_diff_len, total_spd / max_spd, push force, friction, yaw accumulator), the observation's prop, action and
target columns, F_FOOT_POS, the reset rows and reset F_STATE.  The perception columns: 1e-5 max(1, |ref|) + 4 S (the perception
pin's bar).

KAPPA = 64 (epmc_episode_cases.KAPPA), the PMC pin's factor.  Largest error / S measured on an H100 80GB HBM3 at a 700 W power
limit, over every batch and I/O path: F_FOOT_POS 18.8, auto-reset F_FOOT_POS 4.5 and masked-reset 8.3, the observation 7.7,
reset observations 7.8 and 6.4, the target block 6.9, reward 2.6, aux 0.97, reset F_STATE 0.02, reward_sum 0.02 (beyond its fp32
rounding).  Every perception value is within 4 S alone."""
import pytest

import epmc_episode_cases as xc

pytestmark = pytest.mark.gpu

# the I/O path of each batch; the batches whose global ids cross 2^32 (33 and 4097 envs) run every path below
CASE_IO = ("host", "pinned", "device1", "device2", "host", "pinned", "device1", "device2", "host", "host", "device2")


@pytest.mark.parametrize("k", range(len(xc.CASES)))
def test_epmc_episode_logic_matches_the_statement(k, built):
    from lifelike_agility_and_play_b200 import _capi as capi
    ratios = xc.run_case(capi.load_cuda_library(), k, CASE_IO[k])
    print("case %d (n = %d, element %d, %s): %s" % (k, xc.CASES[k][0], xc.CASES[k][1], CASE_IO[k], ratios))


@pytest.mark.parametrize("k,io", [(k, io) for k in (9, 10) for io in xc.ec.IO_PATHS if io != CASE_IO[k]])
def test_every_io_path(k, io, built):
    """the 33- and 4097-env batches through host, pinned and device memory, record modes 1 and 2, canary rows past n"""
    from lifelike_agility_and_play_b200 import _capi as capi
    ratios = xc.run_case(capi.load_cuda_library(), k, io)
    print("case %d (%s): %s" % (k, io, ratios))
