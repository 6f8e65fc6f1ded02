"""Gym-style single-environment adaptor for the environmental-level (EPMC) playground env.

Mirrors ``PlayGroundEnv`` (reference max_game_elements/playground_env.py:57-539) : ``element_id`` 0 is the flat
"joystick" arena that the shipped training script selects (train_scripts/example_epmc_train.sh:100), 1-3 the corridor
arenas of ``BulletStatics`` (hurdles / "holes" = bars to pass under / cubes, bullet_static_entities.py:170-500).  Same
constructor keywords, observation / action spaces (PGE:129-150), ``reset(**kwargs)``, ``step(rl_action)`` (dict with
``A_LLC`` or a bare 12-vector, PGE:323), ``info`` keys on termination (PGE:345-357).  Only the feet collide with the
corridor's boxes (DESIGN.md 5): a bar does not stop the trunk, a hurdle does not stop a shank.
"""
from collections import OrderedDict

import numpy as np

from .. import _capi as capi
from .. import spaces
from ..model.compile_model import load_model_blob
from .primitive_level_env import SHIPPED_PROP_TYPE, _FULL_PROP_SIZE, default_seed

# LeggedRobot.get_init_states_info() (LR:115-117) -> utils/constants.py:103-116 STATES_INFO_12_RUN_0
INIT_STATE_RUN_0 = np.array(
    [0.0, 0.0, 0.3343530097022097,
     0.013840790797843786, 0.023505515131419717, -0.0003254560394373679, 0.9996278394216837,
     0.00809597744709567, -0.020893862693440735, -0.001824006727717542,
     0.0838167925768054, -0.00447012899185979, 0.04114855957667429,
     -0.02776715425087109, -0.7790427096234822, 1.687309016042587, -0.02761322597239251, -0.7777310768160954, 1.6837882482054838,
     -0.02776264511056588, -0.7333994876717276, 1.5669191826863689, -0.027617718742577027, -0.7319111056361625, 1.5631584243808343,
     -0.05228733284239881, -0.0686649273790696, 0.05668137846569721, -0.03640328999561543, -0.02286152438035316, 0.0029650694829541635,
     0.010717179495497164, -0.09457474021233203, 0.10883376594280847, 0.023988549884502025, -0.055563832783516176, 0.03375014202679161])


def _default_engine_factory(n_envs, model_blob, **cfg):
    return capi.VecEngine(capi.load_cuda_library(), n_envs, model_blob, None, **cfg)


engine_factory = _default_engine_factory      # tests swap this for the oracle


def epmc_engine_config(control_freq=50, kp=50.0, kd=1.0, max_tau=16, max_steps=1000, env_randomize_config=None):
    """llq_config fields for the EPMC env from the reference's kwargs (PGE:57-179, PR:7-54); the integer sub-step counts
    use the reference's own float floor divisions (PR:45-46,53: 0.2 // 0.002 = 100, 1.0 // 0.002 = 499, -0.5 // 0.002 = -250)."""
    erc = env_randomize_config
    time_step = 1.0 / 500.0                                                                  # PGE:85
    cfg = dict(env_kind=capi.ENV_EPMC, sim_dt=time_step, policy_dt=1.0 / control_freq, substeps=int((1.0 / control_freq) / time_step),
               kp=kp, kd=kd, max_tau=float(max_tau), ground_friction=1.0,                   # max_game_elements plane.urdf:5
               max_steps=int(max_steps), friction_lo=float(erc['friction_range'][0]), friction_hi=float(erc['friction_range'][1]),
               target_spd_lo=float(erc['target_spd_range'][0]), target_spd_hi=float(erc['target_spd_range'][1]))
    cfg.update(element_id=int(erc['element_id']), wall_width_lo=0.02, wall_width_hi=0.5, wall_gap_lo=1.0, wall_gap_hi=20.0)   # PGE:160-161,199
    cfg.update(auxiliary_radius=float(erc.get('auxiliary_radius') or 0.0))                  # PGE -> BulletStatics(auxiliary_radius=...), BSE:9-16
    hc = erc.get('hole_config') or {}
    cfg.update(hole_gap_lo=float(hc.get('min_gap_height', 0.25)), hole_gap_hi=float(hc.get('max_gap_height', 0.3)))    # BSE:372-373
    lo, hi = erc.get('cmd_vary_freq_range', [25, 200])                                        # PGE:170
    cfg.update(cmd_freq_lo=int(lo), cmd_freq_hi=int(hi))
    dfc = erc.get('disturb_force_config')
    if dfc is not None:
        d = dict(start_time=0., interval_time=5., duration_time=0.5, horizontal_force=20, vertical_force=5)
        d.update(dfc)
        assert d['duration_time'] <= d['interval_time']                                      # PR:35
        assert isinstance(d['horizontal_force'], list) and isinstance(d['vertical_force'], list)   # PR:91-92
        cfg.update(push_enabled=1, push_start_count=int(-d['start_time'] // time_step),
                   push_interval_steps=int(d['interval_time'] // time_step), push_duration_steps=int(d['duration_time'] // time_step),
                   push_h_lo=float(d['horizontal_force'][0]), push_h_hi=float(d['horizontal_force'][1]),
                   push_v_lo=float(d['vertical_force'][0]), push_v_hi=float(d['vertical_force'][1]))
    else:
        cfg.update(push_enabled=0)
    return cfg


class PlayGroundEnv:
    metadata = {}

    def __init__(self, enable_render=False, control_freq=50, kp=50.0, kd=1.0, max_tau=16, prop_type=None, stack_frame_num=3,
                 max_steps=1000, obs_randomization=None, env_randomize_config=None, seed=None, device=0):
        if not isinstance(prop_type, list):
            raise TypeError("Expected 'prop_type' to be a list.")                            # PGE:125-126
        for e in prop_type:
            if e not in _FULL_PROP_SIZE:
                raise KeyError(e)
        if list(prop_type) != SHIPPED_PROP_TYPE or stack_frame_num != 3:
            raise NotImplementedError("the engine implements the shipped prop_type with stack_frame_num=3")
        if env_randomize_config['element_id'] not in (0, 1, 2, 3):
            raise ValueError('Unknown element id.')                                           # BSE:263
        if any(k in (env_randomize_config.get('hole_config') or {}) for k in ('length', 'height', 'max_distance', 'min_distance')):
            raise NotImplementedError("only min/max_gap_height of hole_config are wired through")
        if obs_randomization:
            raise NotImplementedError("obs_randomization (episodic observation noise, PGE:174-179) is not built yet")
        if isinstance(max_tau, (list, tuple)):
            max_tau = float(np.random.uniform(*max_tau))                                     # LR:244 (PGE:236 writes a dead attribute)
        self._max_steps = max_steps
        seed = default_seed() if seed is None else seed
        self._engine = engine_factory(1, load_model_blob(), device=device, seed=seed, auto_reset=0,
                                      **epmc_engine_config(control_freq, kp, kd, max_tau, max_steps, env_randomize_config))
        self._engine.set_init_state(INIT_STATE_RUN_0)
        self.observation_space = spaces.Dict(OrderedDict({                                   # PGE:129-137
            'prop': spaces.Box(0, 0, shape=(99,)), 'prop_a': spaces.Box(0, 0, shape=(36,)),
            'percep_2d': spaces.Box(0, 0, shape=(25, 13)), 'percep_1d': spaces.Box(0, 0, shape=(128,)),
            'percep_front': spaces.Box(0, 0, shape=(25, 13)), 'target': spaces.Box(0, 0, shape=(3,)),
        }))
        self.action_space = spaces.Dict(OrderedDict({'A_Z': spaces.Discrete(256), 'A_LLC': spaces.Box(0, 0, shape=(12,))}))   # PGE:141-144
        self.reward_type = 'joystick' if env_randomize_config['element_id'] == 0 else 'average_speed'                      # PGE:201-204
        self.episodic_reward = OrderedDict({'reward_vel': 0.0, 'reward_rotation': 0.0, 'reward_dist': 0.0, 'reward_avg_spd': 0.0})

    @staticmethod
    def _split(row):
        return OrderedDict({'prop': row[0:99].copy(), 'prop_a': row[99:135].copy(), 'percep_2d': row[135:460].reshape(25, 13).copy(),
                            'percep_1d': row[460:588].copy(), 'percep_front': row[588:913].reshape(25, 13).copy(),
                            'target': row[913:916].copy()})

    def reset(self, **kwargs):
        self.episodic_reward = OrderedDict({'reward_vel': 0.0, 'reward_rotation': 0.0, 'reward_dist': 0.0, 'reward_avg_spd': 0.0})   # PGE:228
        obs = self._split(self._engine.reset()[0])                                           # PGE:196-249
        self._last_len = float(self._engine.get(capi.F_AUX)[0][capi.AUX_LAST_POS_DIFF_LEN])
        return obs

    def _episodic_terms(self, aux, reward, done):
        """The per-term sums the reference reports in `info` on termination (PGE:354-357, 498-501, 527-538), restated on the host from
        the step's post-state: the kernel returns the summed reward only."""
        st = self._engine.get(capi.F_STATE)[0].astype(np.float64)
        d = np.array([aux[capi.AUX_TARGET_X] - st[0], aux[capi.AUX_TARGET_Y] - st[1]])
        plen = float(np.linalg.norm(d))
        u = d / plen
        x, y, z, w = st[3:7] / np.linalg.norm(st[3:7])
        yaw = np.arctan2(2 * (x * y + z * w), 1 - 2 * (y * y + z * z))
        reward_rotation = float(np.exp((np.cos(yaw) * u[0] + np.sin(yaw) * u[1] - 1.0) * 5.0))
        if self.reward_type == 'joystick':
            spd = abs(st[7] * u[0] + st[8] * u[1])
            self.episodic_reward['reward_rotation'] += reward_rotation / float(self._max_steps)
            self.episodic_reward['reward_vel'] += float(np.exp(-abs(spd - aux[capi.AUX_TARGET_SPD]))) / float(self._max_steps)
        else:
            init_len = float(aux[capi.AUX_INIT_POS_DIFF_LEN])
            scaled_rot = reward_rotation / float(self._max_steps) * 0.1
            scaled_dist = -((plen - self._last_len) / init_len) * 0.1
            self._last_len = plen
            self.episodic_reward['reward_rotation'] += scaled_rot * 2.0
            self.episodic_reward['reward_dist'] += scaled_dist
            if done and plen < 0.5:
                self.episodic_reward['reward_avg_spd'] += float(reward) - (scaled_rot * 2.0 + scaled_dist)

    def step(self, rl_action):
        a = rl_action['A_LLC'] if isinstance(rl_action, dict) and 'A_LLC' in rl_action else rl_action    # PGE:323
        obs, reward, done = self._engine.step(np.asarray(a, dtype=np.float32).reshape(1, 12))
        info = {}
        aux = self._engine.get(capi.F_AUX)[0]
        self._episodic_terms(aux, reward[0], bool(done[0]))
        if done[0]:                                                                           # PGE:345-357
            info['ave_spd'] = float(aux[capi.AUX_TOTAL_SPD] / aux[capi.AUX_COUNTER])
            info['max_spd'] = float(aux[capi.AUX_MAX_SPD])
            for key in ('reward_vel', 'reward_rotation', 'reward_dist', 'reward_avg_spd'):
                info[key] = self.episodic_reward[key]
        return self._split(obs[0]), float(reward[0]), bool(done[0]), info

    def close(self):
        if self._engine is not None:
            self._engine.close()
            self._engine = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
