"""A reset clears the contact warm start of every collision sphere, not only the feet: a new episode starts without the impulses
the previous one left on the knees, hips, shanks and trunk corners (the oracle clears all LLQ_MAX_SPHERES too)."""
import numpy as np
import pytest

from lifelike_agility_and_play_b200 import _capi as capi

pytestmark = pytest.mark.gpu
KINDS = ["pmc", "epmc0", "epmc3", "sepmc"]


def _engine(lib, kind, n, blob, mocap, **over):
    from lifelike_agility_and_play_b200.sim_envs.playground_env import INIT_STATE_RUN_0
    if kind == "pmc":
        return capi.VecEngine(lib, n, blob, mocap, seed=3, **over)
    cfg = dict(kp=50.0, kd=0.5, max_tau=16.0, max_steps=100, seed=3, **over)
    cfg.update(dict(env_kind=capi.ENV_SEPMC) if kind == "sepmc" else dict(env_kind=capi.ENV_EPMC, element_id=int(kind[-1])))
    eng = capi.VecEngine(lib, n, blob, None, **cfg)
    eng.set_init_state(INIT_STATE_RUN_0)
    return eng


@pytest.mark.parametrize("kind", KINDS)
def test_masked_reset_clears_all_warm_start_entries(built, blob, small_mocap, kind):
    n = 64
    eng = _engine(capi.load_cuda_library(), kind, n, blob, small_mocap)
    eng.reset()
    warm = (1.0 + np.arange(n * 32, dtype=np.float32)).reshape(n, 32)
    eng.set(capi.F_WARMSTART, warm)
    env = np.arange(n)
    mask = ((env // 2) % 2 == 0) if kind == "sepmc" else (env % 2 == 0)        # SEPMC: whole pairs
    eng.reset(mask.astype(np.uint8))
    got = eng.get(capi.F_WARMSTART)
    assert np.all(got[mask] == 0.0), np.nonzero(got[mask])
    assert np.array_equal(got[~mask].view(np.uint32), warm[~mask].view(np.uint32))
    eng.close()


def test_auto_reset_clears_the_non_foot_spheres_of_a_fallen_robot(built, blob, small_mocap, oracle_lib):
    """Robot 0 lies upside down on its trunk: its trunk corners touch the ground and it falls in the first step."""
    n = 8
    a = np.zeros((n, 12), np.float32)
    rows = {}
    for name, lib, auto in (("cuda", capi.load_cuda_library(), 1), ("oracle", oracle_lib, 1), ("oracle_no_reset", oracle_lib, 0)):
        eng = _engine(lib, "pmc", n, blob, small_mocap, auto_reset=auto)
        eng.reset()
        st = eng.get(capi.F_STATE)
        st[0, 2] = 0.05; st[0, 3:7] = [1.0, 0.0, 0.0, 0.0]; st[0, 7:13] = 0.0; st[0, 25:] = 0.0
        eng.set(capi.F_STATE, st)
        eng.set(capi.F_WARMSTART, np.zeros((n, 32), np.float32))
        _, _, done = eng.step(a)
        assert done[0] == 1
        rows[name] = eng.get(capi.F_WARMSTART)[0]
        eng.close()
    assert np.any(rows["oracle_no_reset"][4:] != 0.0)          # the pose does load non-foot spheres
    assert np.all(rows["cuda"] == 0.0), rows["cuda"]
    assert np.all(rows["oracle"] == 0.0)
