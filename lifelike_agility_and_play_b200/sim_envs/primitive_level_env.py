"""Gym-style single-environment adaptor over the batched engine.

Mirrors ``PrimitiveLevelEnv`` (reference primitive_level_env/primitive_level_env.py:26-435): same constructor
keywords, ``observation_space`` / ``action_space``, ``reset()``, ``step(rl_action)``, ``close()``, same error for a
non-list ``prop_type`` (PLE:112-113).  The arithmetic runs in the CUDA engine through the C-ABI
(``llq_reset`` / ``llq_step``); this class only shapes buffers.

Documented deviations (DESIGN.md 9): the real-time ``time.sleep`` of PLE:241-244 is dropped; rendering /
video options are accepted and ignored; observations are float32 (the reference returns float64).
"""
from collections import OrderedDict

import numpy as np

from .. import _capi as capi
from .. import spaces
from ..mocap import load_mocap
from ..model.compile_model import load_model_blob

SHIPPED_PROP_TYPE = ['joint_pos', 'joint_vel', 'root_ang_vel_loc', 'root_lin_vel_loc', 'e_g']
_FULL_PROP_SIZE = {'joint_pos': 12, 'joint_vel': 12, 'root_lin_vel_loc': 3, 'root_ang_vel_loc': 3, 'e_g': 3}


def _default_engine_factory(n_envs, model_blob, mocap, **cfg):
    """Product path: the sm_90a engine, or a hard error (no CPU fallback)."""
    return capi.VecEngine(capi.load_cuda_library(), n_envs, model_blob, mocap, **cfg)


# tests swap this for the oracle to exercise the adaptor's host logic without a GPU
engine_factory = _default_engine_factory


def default_seed():
    """The reference draws from the unseeded global np.random, so every actor process differs; an engine constructed without a
    seed does the same (OS entropy), instead of every actor replaying the streams of seed 0."""
    import os
    return int.from_bytes(os.urandom(8), 'little') >> 1


class PrimitiveLevelEnv:
    metadata = {}

    def __init__(self, enable_render=False, control_freq=50.0, sim_freq=500.0, kp=50.0, kd=0.5,
                 foot_lateral_friction=0.5, max_tau=18, enable_gui=True, video_path=None, data_path="",
                 prop_type=None, stack_frame_num=3, prioritized_sample_factor=0.0, set_obstacle=False,
                 obstacle_height=0.2, reward_weights=None, seed=None, device=0, mocap=None):
        if video_path is not None:
            assert isinstance(video_path, str) and video_path.endswith('.mp4')       # PLE:53-55
        if not isinstance(prop_type, list):
            raise TypeError("Expected 'prop_type' to be a list.")                      # PLE:112-113
        for e in prop_type:
            if e not in _FULL_PROP_SIZE:
                raise KeyError(e)                                                      # PLE:110-111
        if list(prop_type) != SHIPPED_PROP_TYPE or stack_frame_num != 3:
            raise NotImplementedError("the engine implements the shipped prop_type %r with stack_frame_num=3"
                                      % (SHIPPED_PROP_TYPE,))
        if isinstance(max_tau, (list, tuple)):
            # LR:244 draws one value at construction; the per-episode re-draw of PLE:153 writes a dead attribute
            max_tau = float(np.random.uniform(*max_tau))
        self._policy_step = 1.0 / control_freq                                          # PLE:47
        self._time_step = 1.0 / sim_freq                                                # PLE:49
        self.num_env_steps = int(self._policy_step / self._time_step)                   # PLE:52
        w = reward_weights or {'joint_pos': 0.6, 'joint_vel': 0.05, 'end_effector': 0.1, 'root_pose': 0.15,
                               'root_vel': 0.1}                                         # PLE:352-363
        self._mocap = mocap if mocap is not None else load_mocap(data_path)             # PLE:129 -> ML:19-46
        self._engine = engine_factory(
            1, load_model_blob(), self._mocap, device=device, seed=default_seed() if seed is None else seed, substeps=self.num_env_steps,
            sim_dt=self._time_step, policy_dt=self._policy_step, kp=kp, kd=kd, max_tau=float(max_tau),
            foot_friction=foot_lateral_friction, prioritized_sample_factor=prioritized_sample_factor, auto_reset=0,
            w_joint_pos=w['joint_pos'], w_joint_vel=w['joint_vel'], w_end_effector=w['end_effector'],
            w_root_pose=w['root_pose'], w_root_vel=w['root_vel'])
        if set_obstacle:                                                                # PLE:141-142,173-193
            from ..mocap import obstacle_table
            tab, offs = obstacle_table(self._mocap)
            self._engine.load_obstacles(tab, offs, (0.025, 0.5, float(obstacle_height)))  # PLE:184
        prop_size = sum(_FULL_PROP_SIZE[e] for e in prop_type) * stack_frame_num
        self.observation_space = spaces.Dict(OrderedDict({                              # PLE:117-123
            'prop': spaces.Box(0, 0, shape=(prop_size,)),
            'prop_a': spaces.Box(0, 0, shape=(12 * stack_frame_num,)),
            'future': spaces.Box(0, 0, shape=(72,)),
        }))
        self.action_space = spaces.Box(0, 0, shape=(12,))                               # PLE:124
        self._prop_size = prop_size
        self.reward_sum = 0.0

    # -- helpers
    def _split(self, row):
        p = self._prop_size
        return OrderedDict({'prop': row[:p].copy(), 'prop_a': row[p:p + 36].copy(), 'future': row[p + 36:].copy()})

    @property
    def time(self):
        return float(self._engine.get(capi.F_TIME)[0])

    @property
    def sampled_data_idx(self):
        return int(self._engine.get(capi.F_CLIP)[0])

    # -- gym surface
    def reset(self):
        self.reward_sum = 0.0
        return self._split(self._engine.reset()[0])                                     # PLE:150-171

    def step(self, rl_action):
        action = np.asarray(rl_action, dtype=np.float32).reshape(1, 12)                 # PLE:198
        obs, reward, done = self._engine.step(action)                                   # PLE:195-245
        self.reward_sum += float(reward[0])
        return self._split(obs[0]), float(reward[0]), bool(done[0]), {}

    def close(self):
        if self._engine is not None:
            self._engine.close()
            self._engine = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
