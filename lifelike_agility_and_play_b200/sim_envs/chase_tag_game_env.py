"""Gym-style adaptor for the strategic-level (SEPMC) chase-tag game: two robots, one flag, one walled 5 m x 5 m arena.

Mirrors ``ChaseTagGameEnv`` (reference max_game/chase_tag_game_env.py:21-652) for the shipped arena
(train_scripts/example_sepmc_train.sh:113-116: no random cubes, hurdle or holes): same constructor keywords, the Tuple of
two Dict observation / action spaces (CTG:101-138), ``reset(**kwargs)`` -> list of two OrderedDicts, ``step(rl_actions)``
with a list of two ``{'A_LLC': ...}`` dicts -> ``(obs, [r0, r1], done, info)`` with the speed statistics in ``info``
(CTG:402-407).  Arena elements (rand_cube / hurdle / hole: box terrain) raise ``NotImplementedError``.
"""
from collections import OrderedDict

import numpy as np

from .. import _capi as capi
from .. import spaces
from ..model.compile_model import load_model_blob
from .playground_env import INIT_STATE_RUN_0
from .primitive_level_env import SHIPPED_PROP_TYPE, _FULL_PROP_SIZE
from .primitive_level_env import default_seed


def _default_engine_factory(n_envs, model_blob, **cfg):
    return capi.VecEngine(capi.load_cuda_library(), n_envs, model_blob, None, **cfg)


engine_factory = _default_engine_factory      # tests swap this for the oracle

# observation entries in emission order (CTG:101-114)
OBS_LAYOUT = (('prop', 99, None), ('prop_a', 36, None), ('percept_2d', 325, (25, 13)), ('percept_1d', 128, None),
              ('percept_front', 325, (25, 13)), ('percept_vec', 5, None), ('oppo_info', 15, None), ('oppo_info_cheat', 15, None),
              ('flag_info', 7, None), ('flag_info_cheat', 7, None), ('with_flag', 2, None), ('control_spd', 1, None))


def sepmc_engine_config(control_freq=25.0, kp=50.0, kd=1.0, max_tau=16, max_steps=1000, env_randomize_config=None):
    """llq_config fields from the reference's kwargs (CTG:22-35, 51-56, 160-163; PR:7-54 with its float floor divisions)."""
    erc = env_randomize_config
    time_step = 1.0 / 500.0                                                                  # CTG:52
    cfg = dict(env_kind=capi.ENV_SEPMC, sim_dt=time_step, policy_dt=1.0 / control_freq, substeps=int((1.0 / control_freq) / time_step),
               kp=kp, kd=kd, max_tau=float(max_tau), ground_friction=1.0,                   # max_game/data/urdf/small_v3/plane.urdf:5
               max_steps=int(max_steps), friction_lo=float(erc['friction_range'][0]), friction_hi=float(erc['friction_range'][1]))
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


class ChaseTagGameEnv:
    metadata = {}

    def __init__(self, enable_render=False, control_freq=25.0, kp=50.0, kd=1.0, max_tau=16, terrain_perception=None, prop_type=None,
                 stack_frame_num=3, n_max=2, max_steps=1000, visible_angle=np.pi, obs_randomization=None, env_randomize_config=None,
                 element_config=None, seed=None, device=0):
        if not isinstance(prop_type, list):
            raise TypeError("Expected 'prop_type' to be a list.")                            # CTG:98-99
        for e in prop_type:
            if e not in _FULL_PROP_SIZE:
                raise KeyError(e)
        if list(prop_type) != SHIPPED_PROP_TYPE or stack_frame_num != 3 or n_max != 2 or visible_angle != np.pi:
            raise NotImplementedError("the engine implements the shipped prop_type, stack_frame_num=3, n_max=2, visible_angle=pi")
        if any((element_config or {}).get(k) for k in ('rand_cube', 'hurdle', 'hole')):
            raise NotImplementedError("chase-tag arena elements (rand_cube / hurdle / hole: box terrain) are not built yet; "
                                      "the shipped empty arena is")
        if obs_randomization:
            raise NotImplementedError("obs_randomization (episodic observation noise, CTG:198-202) is not built yet")
        if 'control_spd' in env_randomize_config:
            raise NotImplementedError("a fixed control_spd override (CTG:364) is not built yet")
        if isinstance(max_tau, (list, tuple)):
            max_tau = float(np.random.uniform(*max_tau))                                     # LR:244
        self.n_max = n_max
        self.max_steps = max_steps
        self._engine = engine_factory(2, load_model_blob(), device=device, seed=default_seed() if seed is None else seed, auto_reset=0,
                                      **sepmc_engine_config(control_freq, kp, kd, max_tau, max_steps, env_randomize_config))
        self._engine.set_init_state(INIT_STATE_RUN_0)
        dict_obs_space = OrderedDict((k, spaces.Box(0, 0, shape=shp if shp else (n,))) for k, n, shp in OBS_LAYOUT)
        self.observation_space = spaces.Tuple([spaces.Dict(dict_obs_space)] * n_max)         # CTG:115
        self.action_space = spaces.Tuple([spaces.Dict(OrderedDict({                          # CTG:131-136
            'A_HLC': spaces.Box(0, 0, shape=(1,)), 'A_Z': spaces.Discrete(256), 'A_LLC': spaces.Box(0, 0, shape=(12,))}))] * n_max)

    @staticmethod
    def _split(row):
        out, o = OrderedDict(), 0
        for k, n, shp in OBS_LAYOUT:
            v = row[o:o + n].copy()
            out[k] = v.reshape(shp) if shp else v
            o += n
        return out

    @property
    def with_flag(self):
        aux = self._engine.get(capi.F_AUX)
        return [bool(aux[0, capi.AUX_WITH_FLAG]), bool(aux[1, capi.AUX_WITH_FLAG])]

    @property
    def oppo_visible(self):
        aux = self._engine.get(capi.F_AUX)
        return np.array([bool(aux[0, capi.AUX_OPPO_VISIBLE]), bool(aux[1, capi.AUX_OPPO_VISIBLE])])

    @property
    def target_pos(self):
        aux = self._engine.get(capi.F_AUX)
        return [float(aux[0, capi.AUX_FLAG_X]), float(aux[0, capi.AUX_FLAG_Y]), 0.25]

    def reset(self, **kwargs):
        obs = self._engine.reset()                                                           # CTG:261-304
        return [self._split(obs[0]), self._split(obs[1])]

    def step(self, rl_actions):
        a = np.stack([np.asarray(x['A_LLC'], dtype=np.float32).reshape(12) for x in rl_actions])      # CTG:379
        obs, reward, done = self._engine.step(a)
        aux = self._engine.get(capi.F_AUX)
        spd = aux[:, capi.AUX_TOTAL_SPD] / aux[:, capi.AUX_COUNTER]
        info = {'avg_spd0': float(spd[0]), 'avg_spd1': float(spd[1]),                                  # CTG:402-407
                'max_spd0': float(aux[0, capi.AUX_MAX_SPD]), 'max_spd1': float(aux[1, capi.AUX_MAX_SPD])}
        return [self._split(obs[0]), self._split(obs[1])], [float(reward[0]), float(reward[1])], bool(done[0]), info

    def close(self):
        if self._engine is not None:
            self._engine.close()
            self._engine = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
