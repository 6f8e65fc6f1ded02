"""The C-ABI boundary: exported symbols, loud failure without a GPU, call-order errors, gym surface."""
import ctypes
import os
import re

import numpy as np
import pytest

from lifelike_agility_and_play_b200 import _capi as capi
from conftest import HAVE_CUDA, ROOT


def _declared():
    txt = open(os.path.join(ROOT, "include", "llq.h")).read()
    return sorted(set(re.findall(r"\b(llq_\w+)\s*\(", txt)) - {"llq_config", "llq_engine"})


def test_both_libraries_export_every_declared_symbol(built):
    names = _declared()
    assert len(names) >= 17
    from oracle import oracle
    for path in (capi.CUDA_LIB_PATH, oracle.LIB_PATH):
        lib = ctypes.CDLL(path)
        for n in names:
            assert hasattr(lib, n), "%s does not export %s" % (path, n)


def test_field_ids_and_aux_slots_match_header():
    txt = open(os.path.join(ROOT, "include", "llq.h")).read()
    defs = re.findall(r"^#define LLQ_((?:F|AUX|CNT)_\w+)\s+(\d+)", txt, re.M)
    assert len(defs) >= 16 + 25 + 6
    for name, value in defs:
        assert getattr(capi, name) == int(value), name


def test_config_struct_matches_header(built, oracle_lib):
    cfg = oracle_lib.default_config()
    assert cfg.struct_size == ctypes.sizeof(capi.LlqConfig)
    cuda = capi.LlqLibrary(capi.CUDA_LIB_PATH)
    c2 = cuda.default_config()
    assert cuda.is_cuda and not oracle_lib.is_cuda and cuda.abi == oracle_lib.abi == 4
    for f, _ in capi.LlqConfig._fields_:
        assert getattr(cfg, f) == getattr(c2, f), f
    assert (cfg.substeps, cfg.solver_iters, cfg.kp, cfg.kd, cfg.max_tau) == (10, 10, 50.0, 0.5, 18.0)
    assert cfg.gravity_z == -9.80665 and cfg.sim_dt == 1 / 500.0


@pytest.mark.skipif(HAVE_CUDA, reason="needs a host without a GPU")
def test_cuda_engine_fails_loudly_without_gpu(built, blob, small_mocap):
    """No silent CPU fallback on the product path."""
    with pytest.raises(capi.LlqError) as ei:
        capi.VecEngine(capi.load_cuda_library(), 4, blob, small_mocap)
    assert ei.value.code == -3 and "CUDA" in str(ei.value)


def test_call_order_and_argument_errors(make_oracle, oracle_lib, blob, small_mocap):
    eng = make_oracle(2)
    with pytest.raises(capi.LlqError) as ei:
        eng.step(np.zeros((2, 12), np.float32))            # step before reset
    assert ei.value.code == -4
    eng.reset()
    with pytest.raises(ValueError):
        eng.step(np.zeros((3, 12), np.float32))
    with pytest.raises(capi.LlqError):
        eng.reset_to(99, 0.1)
    with pytest.raises(capi.LlqError):
        eng.reset_to(0, 1e9)
    with pytest.raises(capi.LlqError):
        capi.VecEngine(oracle_lib, 0, blob, small_mocap)
    with pytest.raises(capi.LlqError):
        capi.VecEngine(oracle_lib, 1, blob[:-3], small_mocap)


def test_state_roundtrip_and_counters(make_oracle):
    eng = make_oracle(5, seed=1)
    eng.reset()
    st = eng.get(capi.F_STATE)
    eng.set(capi.F_STATE, st)
    assert np.array_equal(eng.get(capi.F_STATE), st)
    o, r, d = eng.step(np.zeros((5, 12), np.float32))
    assert o.shape == (5, 207) and r.shape == (5,) and d.dtype == np.uint8
    assert eng.counters()[capi.CNT_ENV_STEPS] == 5
    assert np.all(eng.get(capi.F_EPISODE_STEPS) == 1)


def _tracking_cfg(mocap):
    return {'arena_id': 'LeggedRobotTracking', 'render': False, 'data_path': '', 'mocap': mocap, 'control_freq': 50.0,
            'prop_type': ['joint_pos', 'joint_vel', 'root_ang_vel_loc', 'root_lin_vel_loc', 'e_g'],
            'prioritized_sample_factor': 3.0, 'set_obstacle': False, 'kp': 50.0, 'kd': 0.5, 'max_tau': 18,
            'reward_weights': {'joint_pos': 0.3, 'joint_vel': 0.05, 'end_effector': 0.1, 'root_pose': 0.5, 'root_vel': 0.05}}


def _drive(env):
    """The loop of test_scripts/primitive_level/test_primitive_level_env.py:61-96, head-less, random policy."""
    ob_space, ac_space = env.observation_space, env.action_space
    obs = env.reset(inter_kwargs={})
    assert isinstance(obs, tuple) and list(obs[0].keys()) == ['prop', 'prop_a', 'future']
    assert [obs[0][k].shape for k in obs[0]] == [(99,), (36,), (72,)]
    rng = np.random.default_rng(0)
    n_done = 0
    for t in range(120):
        act = (0.1 * rng.standard_normal(12)).astype(np.float32)
        obs, rwd, done, info = env.step([act])
        assert isinstance(rwd, tuple) and isinstance(done, bool) and isinstance(info, dict)
        assert 0.0 <= rwd[0] <= 1.0 + 1e-6
        if done:
            n_done += 1
            obs = env.reset()
    return ob_space, ac_space, n_done


def test_gym_surface_on_oracle(monkeypatch, oracle_lib, small_mocap):
    """Host logic of the drop-in factories (CPE:21-64,143-147), exercised on the CPU by swapping the engine factory."""
    from lifelike_agility_and_play_b200.sim_envs import create_envs, primitive_level_env as ple
    monkeypatch.setattr(ple, "engine_factory", lambda n, blob, mocap, **cfg: capi.VecEngine(oracle_lib, n, blob, mocap, **{k: v for k, v in cfg.items() if k != "device"}))
    env = create_envs.create_tracking_game(**_tracking_cfg(small_mocap))
    ob, ac, _ = _drive(env)
    assert len(ob.spaces) == 1 and list(ob.spaces[0].spaces.keys()) == ['prop', 'prop_a', 'future']
    assert ob.spaces[0].spaces['prop'].shape == (99,) and ac.spaces[0].shape == (12,)
    env.close()
    env2 = create_envs.create_tracking_env(**_tracking_cfg(small_mocap))
    assert list(env2.observation_space.spaces.keys()) == ['prop', 'prop_a', 'future'] and env2.action_space.shape == (12,)
    env2.close()
    with pytest.raises(AssertionError):
        create_envs.create_tracking_game(**dict(_tracking_cfg(small_mocap), arena_id="nope"))          # CPE:22-25
    with pytest.raises(TypeError):
        create_envs.create_tracking_game(**dict(_tracking_cfg(small_mocap), prop_type=""))             # PLE:112-113
    with pytest.raises(TypeError):
        create_envs.create_chase_tag_game(arena_id="CTG")                                               # CTG:98-99: prop_type must be a list


EPMC_ENV_CONFIG = {
    'arena_id': 'Playground', 'render': False, 'control_freq': 50.0,
    'prop_type': ['joint_pos', 'joint_vel', 'root_ang_vel_loc', 'root_lin_vel_loc', 'e_g'],
    'kp': 50.0, 'kd': 0.5, 'max_tau': 16, 'max_steps': 30, 'obs_randomization': {},
    'env_randomize_config': {
        'element_id': 0, 'height_range': [0.0, 0.0], 'friction_range': [0.4, 3.0],
        'disturb_force_config': {'start_time': 0.5, 'interval_time': 1.0, 'duration_time': 0.2, 'horizontal_force': [0, 50], 'vertical_force': [0, 10]},
        'cmd_vary_freq_range': [9999, 10000], 'target_spd_range': [0.5, 3.0], 'auxiliary_radius': 0.02,
        'hole_config': {'min_gap_height': 0.25, 'max_gap_height': 0.25}},
}


def _drive_epmc(env):
    """The loop of test_scripts/environmental_level/test_environmental_level_env.py, head-less, random policy."""
    obs = env.reset(inter_kwargs={})
    assert list(obs[0].keys()) == ['prop', 'prop_a', 'percep_2d', 'percep_1d', 'percep_front', 'target']
    assert [obs[0][k].shape for k in obs[0]] == [(99,), (36,), (25, 13), (128,), (25, 13), (3,)]
    assert np.all(obs[0]['percep_2d'] == 0) and np.allclose(obs[0]['percep_1d'], 0.5)          # flat ground; |base_pos| = 0.5 (K8)
    rng = np.random.default_rng(0)
    dones = 0
    for t in range(70):
        obs, rwd, done, info = env.step([{'A_Z': 0, 'A_LLC': (0.1 * rng.standard_normal(12)).astype(np.float32)}])
        assert isinstance(done, bool) and 0.0 <= rwd[0] <= 1.0 / 30 + 1e-9
        assert abs(np.linalg.norm(obs[0]['target'][:2]) - 1.0) < 1e-5 and 0.5 <= obs[0]['target'][2] <= 3.0
        if done:
            assert set(info) >= {'ave_spd', 'max_spd'}
            dones += 1
            obs = env.reset()
    assert dones >= 2          # max_steps = 30


def test_epmc_gym_surface_on_oracle(monkeypatch, oracle_lib):
    from lifelike_agility_and_play_b200.sim_envs import create_envs, playground_env as pge
    monkeypatch.setattr(pge, "engine_factory", lambda n, blob, **cfg: capi.VecEngine(oracle_lib, n, blob, None, **{k: v for k, v in cfg.items() if k != "device"}))
    env = create_envs.create_playground_game(**EPMC_ENV_CONFIG)
    assert list(env.action_space.spaces[0].spaces.keys()) == ['A_Z', 'A_LLC']
    _drive_epmc(env)
    env.close()
    cfg = pge.epmc_engine_config(50.0, 50.0, 0.5, 16, 1000, EPMC_ENV_CONFIG['env_randomize_config'])
    assert (cfg['push_start_count'], cfg['push_interval_steps'], cfg['push_duration_steps'], cfg['substeps']) == (-250, 499, 100, 10)   # K7
    bad = dict(EPMC_ENV_CONFIG, env_randomize_config=dict(EPMC_ENV_CONFIG['env_randomize_config'], element_id=4))
    with pytest.raises(ValueError):
        create_envs.create_playground_game(**bad)                                                   # BSE:263
    for element in (1, 2, 3):           # corridor arenas: walls, hurdles / bars / cubes
        cfg = dict(EPMC_ENV_CONFIG, env_randomize_config=dict(EPMC_ENV_CONFIG['env_randomize_config'], element_id=element))
        env = create_envs.create_playground_game(**cfg)
        assert env.reward_type == 'average_speed'
        obs = env.reset(inter_kwargs={})
        nb = int(env.env._engine.get(capi.F_NBOX)[0])
        bx = env.env._engine.get(capi.F_BOXES)[0].reshape(36, 6)
        assert 4 <= nb <= 36 and np.all(bx[:2, 3] == 100.0) and bx[0, 1] == -bx[1, 1] > 0          # two 200 m walls, symmetric
        assert np.allclose(bx[2:nb, 4], bx[0, 1] - bx[0, 4], rtol=0, atol=1e-6)                     # obstacles span the corridor (seed from OS entropy)
        assert obs[0]['percep_1d'].max() < 20.0 + 1e-3 and abs(np.linalg.norm(obs[0]['target'][:2]) - 1.0) < 1e-5
        for t in range(5):
            obs, rwd, done, info = env.step([{'A_LLC': np.zeros(12, np.float32)}])
        assert np.isfinite(rwd[0])
        env.close()


SEPMC_ENV_CONFIG = {          # train_scripts/example_sepmc_train.sh:94-117 with a short episode
    'arena_id': 'CTG', 'render': False, 'control_freq': 50.0,
    'prop_type': ['joint_pos', 'joint_vel', 'root_ang_vel_loc', 'root_lin_vel_loc', 'e_g'],
    'kp': 50.0, 'kd': 0.5, 'max_tau': 16, 'max_steps': 25, 'obs_randomization': {},
    'env_randomize_config': {'friction_range': [0.4, 3.0],
                             'disturb_force_config': {'start_time': 0.5, 'interval_time': 1.0, 'duration_time': 0.2,
                                                      'horizontal_force': [0, 50], 'vertical_force': [0, 10]}},
    'element_config': {'rand_cube': False, 'hurdle': False, 'hole': False},
}


def _drive_sepmc(env):
    """The loop of test_scripts/strategic_level/test_strategic_level_env.py, head-less, random policies for both agents."""
    obs = env.reset()
    keys = ['prop', 'prop_a', 'percept_2d', 'percept_1d', 'percept_front', 'percept_vec', 'oppo_info', 'oppo_info_cheat', 'flag_info',
            'flag_info_cheat', 'with_flag', 'control_spd']
    assert len(obs) == 2 and all(list(o.keys()) == keys for o in obs)
    assert [obs[0][k].shape for k in keys] == [(99,), (36,), (25, 13), (128,), (25, 13), (5,), (15,), (15,), (7,), (7,), (2,), (1,)]
    assert obs[0]['with_flag'][0] + obs[1]['with_flag'][0] == 1 and obs[0]['with_flag'][0] == obs[1]['with_flag'][1]
    assert 0.5 <= obs[0]['control_spd'][0] <= 3.0 and obs[0]['control_spd'][0] == obs[1]['control_spd'][0]
    assert np.allclose(obs[0]['oppo_info_cheat'][1:4], obs[1]['percept_vec'][:3])              # the opponent's position
    assert 0.0 < obs[0]['percept_1d'].min() and obs[0]['percept_1d'].max() < 7.2                # every horizontal ray ends on a wall / the flag
    rng = np.random.default_rng(0)
    dones = 0
    for t in range(60):
        acts = [{'A_HLC': np.zeros(1), 'A_Z': 0, 'A_LLC': (0.1 * rng.standard_normal(12)).astype(np.float32)} for _ in range(2)]
        obs, rwd, done, info = env.step(acts)
        assert isinstance(done, bool) and len(rwd) == 2 and rwd[0] == -rwd[1] and rwd[0] in (-2.0, -1.0, 0.0, 1.0, 2.0)
        assert set(info) == {'avg_spd0', 'avg_spd1', 'max_spd0', 'max_spd1'}
        if done:
            dones += 1
            obs = env.reset()
    assert dones >= 2          # max_steps = 25
    assert len(env.with_flag) == 2 and len(env.target_pos) == 3


def test_sepmc_gym_surface_on_oracle(monkeypatch, oracle_lib):
    from lifelike_agility_and_play_b200.sim_envs import create_envs, chase_tag_game_env as ctg
    monkeypatch.setattr(ctg, "engine_factory", lambda n, blob, **cfg: capi.VecEngine(oracle_lib, n, blob, None, **{k: v for k, v in cfg.items() if k != "device"}))
    env = create_envs.create_chase_tag_game(**SEPMC_ENV_CONFIG)
    assert len(env.observation_space.spaces) == 2 and list(env.action_space.spaces[0].spaces.keys()) == ['A_HLC', 'A_Z', 'A_LLC']
    _drive_sepmc(env)
    env.close()
    cfg = ctg.sepmc_engine_config(50.0, 50.0, 0.5, 16, 1000, SEPMC_ENV_CONFIG['env_randomize_config'])
    assert (cfg['push_start_count'], cfg['push_interval_steps'], cfg['push_duration_steps'], cfg['substeps']) == (-250, 499, 100, 10)
    with pytest.raises(NotImplementedError):
        create_envs.create_chase_tag_game(**dict(SEPMC_ENV_CONFIG, element_config={'rand_cube': True}))
    env2 = create_envs.create_chase_tag_env(**SEPMC_ENV_CONFIG)                                   # CPE:157-161
    assert list(env2.observation_space.spaces.keys())[0] == 'prop' and env2.action_space.spaces['A_LLC'].shape == (12,)
    env2.close()


@pytest.mark.gpu
def test_sepmc_gym_surface_on_cuda():
    from lifelike_agility_and_play_b200.sim_envs import create_envs
    env = create_envs.create_chase_tag_game(**SEPMC_ENV_CONFIG)
    _drive_sepmc(env)
    env.close()


@pytest.mark.gpu
def test_epmc_gym_surface_on_cuda():
    from lifelike_agility_and_play_b200.sim_envs import create_envs
    env = create_envs.create_playground_game(**EPMC_ENV_CONFIG)
    _drive_epmc(env)
    env.close()


@pytest.mark.gpu
def test_gym_surface_on_cuda(small_mocap):
    from lifelike_agility_and_play_b200.sim_envs import create_envs
    env = create_envs.create_tracking_game(**_tracking_cfg(small_mocap))
    _drive(env)
    env.close()


def test_mocap_loader_roundtrip(tmp_path, small_mocap):
    """Reference on-disk format (ML:19-46): JSON per clip, sorted file order."""
    import json
    from lifelike_agility_and_play_b200.mocap import load_mocap
    for i in (2, 0, 1):
        with open(tmp_path / ("clip_%02d.txt" % i), "w") as f:
            json.dump({"FrameDuration": small_mocap.frame_dt, "LegOrder": ["FR", "FL", "HR", "HL"], "Frames": small_mocap.clip(i).tolist()}, f)
    (tmp_path / "notes.md").write_text("ignored")
    t = load_mocap(str(tmp_path))
    assert t.n_clips == 3 and t.names == ["clip_00.txt", "clip_01.txt", "clip_02.txt"]
    assert np.array_equal(t.clip(1), small_mocap.clip(1)) and t.margin() == 125
    rep = t.validation_report(lower=np.full(12, -5.0), upper=np.full(12, 5.0))
    assert rep[0]["limit_violations"] == 0 and rep[0]["quat_norm_err"] < 1e-9
    with pytest.raises(FileNotFoundError):
        load_mocap(str(tmp_path / "missing"))


def test_pinned_io_path_matches_plain_step(make_oracle):
    """LLQ_IO_PINNED entry (page-locked buffers, no staging copy) gives the same results as llq_step."""
    a, b = make_oracle(6, seed=4), make_oracle(6, seed=4)
    a.reset(); b.reset()
    act_p, obs_p, rew_p, done_p = b.pinned_io()
    rng = np.random.default_rng(1)
    for _ in range(3):
        act = (0.1 * rng.standard_normal((6, 12))).astype(np.float32)
        o, r, d = a.step(act)
        act_p[...] = act
        b.step_pinned(act_p, obs_p, rew_p, done_p)
        assert np.array_equal(o, obs_p) and np.array_equal(r, rew_p) and np.array_equal(d, done_p)


def test_shipped_pmc_train_config_with_obstacle(monkeypatch, oracle_lib):
    """train_scripts/example_pmc_train.sh:67-79 verbatim (set_obstacle True, obstacle_height left to the factory default 0.0)."""
    from lifelike_agility_and_play_b200.sim_envs import create_envs, primitive_level_env as ple
    from lifelike_agility_and_play_b200.mocap import synthetic_mocap, obstacle_table
    monkeypatch.setattr(ple, "engine_factory", lambda n, blob, mocap, **cfg: capi.VecEngine(oracle_lib, n, blob, mocap, **{k: v for k, v in cfg.items() if k != "device"}))
    mc = synthetic_mocap(3, seed=5, min_frames=400, max_frames=500)
    mc.frames[:, 2] += 0.25 * np.exp(-((np.arange(len(mc.frames)) % 400 - 200) / 20.0) ** 2)      # periodic jumps
    assert obstacle_table(mc)[1][-1] >= 3
    cfg = {'arena_id': 'LeggedRobotTracking', 'render': False, 'data_path': '', 'mocap': mc, 'control_freq': 50.0,
           'prop_type': ['joint_pos', 'joint_vel', 'root_ang_vel_loc', 'root_lin_vel_loc', 'e_g'],
           'prioritized_sample_factor': 3.0, 'set_obstacle': True, 'kp': 50.0, 'kd': 0.5, 'max_tau': 18,
           'reward_weights': {'joint_pos': 0.3, 'joint_vel': 0.05, 'end_effector': 0.1, 'root_pose': 0.5, 'root_vel': 0.05}}
    env = create_envs.create_tracking_game(**cfg)
    _drive(env)
    env.close()


@pytest.mark.gpu
def test_record_mode_writes_the_whole_trajectory_row(make_cuda):
    """llq_set_option("record", 1): the step kernel writes action | reward | done behind the observation of the slab row it is
    handed (SURVEY 8e: no column copies after the step); auto-reset rewrites only the observation part."""
    import torch
    n, ld = 96, 207 + 16
    eng = make_cuda(n, seed=4, auto_reset=1)
    eng.reset()
    eng.set_option("record", 1)
    dev = torch.device("cuda", 0)
    slab = torch.full((3, n, ld), -7.0, device=dev)
    rew = torch.zeros(n, device=dev); done = torch.zeros(n, dtype=torch.uint8, device=dev)
    rng = np.random.default_rng(0)
    for t in range(3):
        a = torch.from_numpy((0.4 * rng.standard_normal((n, 12))).astype(np.float32)).to(dev)
        eng.step_device(a.data_ptr(), slab[t].data_ptr(), rew.data_ptr(), done.data_ptr(), obs_ld=ld)
        eng.sync()
        row = slab[t].cpu().numpy()
        assert np.array_equal(row[:, 207:219], a.cpu().numpy())
        assert np.array_equal(row[:, 219], rew.cpu().numpy())
        assert np.array_equal(row[:, 220], done.cpu().numpy().astype(np.float32))
        assert np.all(row[:, 221:] == -7.0)                                  # neglogp | value belong to the policy kernel
        assert np.array_equal(row[:, :207], eng.get(capi.F_OBS))
    with pytest.raises(capi.LlqError):
        eng.step_device(a.data_ptr(), slab[0].data_ptr(), rew.data_ptr(), done.data_ptr(), obs_ld=207 + 8)


@pytest.mark.gpu
def test_two_handles_on_two_devices_in_one_process(built, blob, small_mocap):
    """llq.h: several handles (one per GPU) may coexist in one process -- the > 48 kB dynamic shared memory opt-in of the step
    kernel is a per-device function attribute and must be raised on each handle's device."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    engs = [capi.VecEngine(capi.load_cuda_library(), 64, blob, small_mocap, seed=8, device=d) for d in (0, 1)]
    a = (0.1 * np.random.default_rng(0).standard_normal((64, 12))).astype(np.float32)
    outs = []
    for e in engs:
        e.reset()
        outs.append(e.step(a))
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])
    for e in engs:
        e.close()


@pytest.mark.gpu
def test_reset_to_ignores_unvalidated_entries_of_masked_out_envs(make_cuda):
    """clip / time of envs whose mask is 0 are never used to index the mocap table; a stale clock past the clip end stays on the
    clip's last playable frame (the reference raises IndexError there)."""
    n = 40
    eng = make_cuda(n, seed=2)
    eng.reset()
    mask = np.zeros(n, np.uint8); mask[::2] = 1
    clip = np.where(mask == 1, 1, -12345).astype(np.int32)
    t = np.where(mask == 1, 0.25, 1e9)
    eng.reset_to(clip, t, mask=mask)
    assert np.all(eng.get(capi.F_CLIP)[mask == 1] == 1)
    with pytest.raises(capi.LlqError):
        eng.set(capi.F_TIME, np.full(n, -1.0))
    eng.set(capi.F_TIME, np.full(n, 1e4))                                    # far past every clip
    obs, rew, done = eng.step(np.zeros((n, 12), np.float32))
    assert np.all(done == 1) and np.all(np.isfinite(obs)) and np.all(np.isfinite(rew))
