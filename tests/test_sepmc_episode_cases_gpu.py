"""The SEPMC episode logic of the step and reset kernels against the fp64 statement of tests/sepmc_episode_cases.py, robot by robot
and pair by pair, with no pair excluded: flag touch and switch, tag, visibility, fall, timeup, `bad`, the rewards, the pair's push
stream, the auto-reset and masked-reset draws and rows, through every I/O path.

Exactly equal: done, the record columns, counters [0] and [1], F_EPISODE_ID, and the aux counter, with_flag, oppo_visible,
switch_flag, push_count, push_draws, flag_draws and flag_touch.  Within KAPPA S + 2^-23 |ref|: reward, reward_sum, the other aux
slots (flag xy, control_spd, total_spd / max_spd, push force, friction, yaw accumulator), the observation's prop and action
columns, F_FOOT_POS, the reset rows and reset F_STATE.  The perception columns (obs 135-964): 1e-5 max(1, |ref|) + 4 S (the
perception pin's bar).  A pair with a NaN joint angle is checked on done, reward, counters and the integer aux slots other than
oppo_visible; its post state is not stated.

KAPPA = 64 (sepmc_episode_cases.KAPPA), the PMC and EPMC pins' factor.  Largest error / S measured on an H100 80GB HBM3 at a 700 W
power limit, over every batch and I/O path: the observation 6.6, auto-reset observations 3.9, F_FOOT_POS 3.3, masked-reset
observations 3.2, masked-reset F_FOOT_POS 2.1, auto-reset F_FOOT_POS 1.8, reset F_STATE 0.006; aux, reward and reward_sum 0 (equal
to the statement's fp32 values).  Every perception value is within 4 S plus 1e-6 max(1, |ref|)."""
import pytest

import sepmc_episode_cases as sc

pytestmark = pytest.mark.gpu

# the I/O path of each batch; the 34- and 162-robot batches (global ids crossing 2^32) run every path below
CASE_IO = ("host", "pinned", "device1", "device2", "host", "pinned", "host", "device2")


@pytest.mark.parametrize("k", range(len(sc.CASES)))
def test_sepmc_episode_logic_matches_the_statement(k, built):
    from lifelike_agility_and_play_b200 import _capi as capi
    ratios = sc.run_case(capi.load_cuda_library(), k, CASE_IO[k])
    print("case %d (n = %d, %s): %s" % (k, sc.CASES[k][0], CASE_IO[k], ratios))


@pytest.mark.parametrize("k,io", [(k, io) for k in (6, 7) for io in sc.ec.IO_PATHS if io != CASE_IO[k]])
def test_every_io_path(k, io, built):
    """the 34- and 162-robot batches through host, pinned and device memory, record modes 1 and 2, canary rows past n"""
    from lifelike_agility_and_play_b200 import _capi as capi
    ratios = sc.run_case(capi.load_cuda_library(), k, io)
    print("case %d (%s): %s" % (k, io, ratios))
