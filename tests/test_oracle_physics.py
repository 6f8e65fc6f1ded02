"""T0: analytic invariants of the oracle's dynamics (SURVEY 8c parity protocol).  These pin the oracle's
articulated-body algorithm to mechanics itself, since no Bullet golden vectors exist (parity unpinned)."""
import numpy as np
import pytest

from lifelike_agility_and_play_b200 import _capi as capi
from helpers import frictionless_model_blob, mechanics, random_state

FREE = dict(kp=0.0, kd=0.0, lin_damping=0.0, ang_damping=0.0, substeps=1)


def _run(eng, st, steps):
    eng.reset_to(0, 0.1)
    eng.set(capi.F_STATE, st[None].astype(np.float32))
    for _ in range(steps):
        eng.step(np.zeros((1, 12), np.float32))
    return eng.get(capi.F_STATE)[0].astype(np.float64)


def test_energy_and_momentum_conservation(model, make_oracle):
    blob0 = frictionless_model_blob(model)
    drift = []
    for dt in (0.002, 0.0005):
        eng = make_oracle(1, blob_=blob0, gravity_z=0.0, sim_dt=dt, **FREE)
        st = random_state(np.random.default_rng(0), vel_scale=0.3).astype(np.float32).astype(np.float64)
        m0 = mechanics(model, st)
        s1 = _run(eng, st, int(round(0.1 / dt)))
        m1 = mechanics(model, s1)
        assert eng.counters()[capi.CNT_LIMIT_ROWS] == 0, "state must stay inside the joint limits for this test"
        drift.append((abs(m1["KE"] - m0["KE"]) / m0["KE"], np.abs(m1["P"] - m0["P"]).max(), np.abs(m1["L"] - m0["L"]).max()))
    assert drift[0][0] < 2e-5 and drift[0][1] < 1e-4 and drift[0][2] < 3e-4
    # first-order integrator: errors shrink ~4x when dt shrinks 4x
    assert drift[1][1] < 0.4 * drift[0][1] and drift[1][2] < 0.4 * drift[0][2]


def test_free_fall_of_centre_of_mass(model, make_oracle):
    """With gravity and no contact the CoM accelerates at exactly g whatever the joints do."""
    blob0 = frictionless_model_blob(model)
    eng = make_oracle(1, blob_=blob0, sim_dt=0.001, **FREE)
    st = random_state(np.random.default_rng(1), z=50.0, vel_scale=0.3).astype(np.float32).astype(np.float64)
    m0 = mechanics(model, st)
    T = 100
    s1 = _run(eng, st, T)
    m1 = mechanics(model, s1)
    t = T * 0.001
    v_expected = m0["P"] / m0["mass"] + np.array([0, 0, -9.80665 * t])
    assert np.allclose(m1["P"] / m1["mass"], v_expected, atol=2e-4)


def test_static_stand_supports_weight(model, make_oracle):
    """Standing on four feet: at rest the summed normal impulses per sub-step equal m g dt."""
    eng = make_oracle(1, kp=100.0, kd=5.0, max_tau=30.0)
    eng.reset_to(0, 0.1)
    st = np.zeros(37, np.float32)
    st[2] = 0.34; st[6] = 1.0
    st[13:25] = np.array([-0.03, -0.78, 1.69] * 2 + [-0.03, -0.73, 1.57] * 2)
    eng.set(capi.F_STATE, st[None])
    nominal = st[13:25].copy()
    for _ in range(200):
        # the action is a residual on the *current* joint angles (PLE:199-200): servo back to the nominal pose
        q = eng.get(capi.F_STATE)[0, 13:25]
        eng.step((nominal - q)[None].astype(np.float32))
    w = eng.get(capi.F_WARMSTART)[0]
    s = eng.get(capi.F_STATE)[0]
    assert np.all(w[:4] > 0) and np.all(w[4:] == 0), "all four feet (spheres 0-3) should be loaded, nothing else"
    assert abs(w.sum() - 13.00021 * 9.80665 * 0.002) < 1e-4 * 13.00021 * 9.80665 * 0.002
    assert 0.25 < s[2] < 0.36 and np.abs(s[7:13]).max() < 1e-3 and np.abs(s[25:37]).max() < 1e-3


def test_velocity_clamp_keeps_dirty_states_finite(make_oracle):
    """SURVEY K10: resets can land on frames that violate joint limits with huge finite-difference velocities."""
    eng = make_oracle(1)
    eng.reset_to(0, 0.1)
    st = eng.get(capi.F_STATE)
    st[0, 13:25] += 3.0       # far outside the limits
    st[0, 25:37] = 700.0
    eng.set(capi.F_STATE, st)
    for _ in range(5):
        o, r, d = eng.step(np.zeros((1, 12), np.float32))
        assert np.all(np.isfinite(o)) and np.isfinite(r[0])
    assert np.abs(eng.get(capi.F_STATE)[0, 25:37]).max() <= 100.0 + 1e-3     # m_maxCoordinateVelocity


def test_contact_needs_proximity(make_oracle):
    """A foot further than the (relative) contact breaking threshold from the plane creates no rows."""
    eng = make_oracle(1, substeps=1)
    eng.reset_to(0, 0.1)
    st = eng.get(capi.F_STATE); st[0, 2] += 1.0
    eng.set(capi.F_STATE, st)
    c0 = eng.counters()[capi.CNT_CONTACT_ROWS]
    eng.step(np.zeros((1, 12), np.float32))
    assert eng.counters()[capi.CNT_CONTACT_ROWS] == c0
    assert np.all(eng.get(capi.F_WARMSTART) == 0)


def test_translation_invariance_of_the_tracking_env(oracle_lib, blob, small_mocap):
    """Domain property (flat infinite ground): shifting every mocap clip by (dx, dy) shifts the rollout and nothing else -- the
    body-frame observation, the reward and the termination of every step are unchanged.  World positions are carried in fp64
    on both engines precisely so that this holds tens of metres away from the origin (DESIGN.md 3)."""
    from lifelike_agility_and_play_b200._capi import VecEngine, F_STATE
    from lifelike_agility_and_play_b200.mocap import MocapTable
    shifted = MocapTable(small_mocap.frames.copy(), small_mocap.offsets, small_mocap.frame_dt, small_mocap.names)
    shifted.frames[:, 0] += 37.25; shifted.frames[:, 1] -= 12.5
    n = 24
    a = VecEngine(oracle_lib, n, blob, small_mocap, seed=8, auto_reset=1)
    b = VecEngine(oracle_lib, n, blob, shifted, seed=8, auto_reset=1)
    oa, ob = a.reset(), b.reset()
    assert np.abs(oa - ob).max() < 1e-6
    rng = np.random.default_rng(3)
    for t in range(40):
        act = (0.15 * rng.standard_normal((n, 12))).astype(np.float32)
        (oa, ra, da), (ob, rb, db) = a.step(act), b.step(act)
        assert np.array_equal(da, db)
        assert np.abs(oa - ob).max() < 2e-5 and np.abs(ra - rb).max() < 2e-6, (t, np.abs(oa - ob).max())
    sa, sb = a.get(F_STATE), b.get(F_STATE)
    assert np.abs(sb[:, 0] - sa[:, 0] - 37.25).max() < 1e-4 and np.abs(sb[:, 1] - sa[:, 1] + 12.5).max() < 1e-4
    assert np.abs(sa[:, 2:] - sb[:, 2:]).max() < 2e-5
    a.close(); b.close()
