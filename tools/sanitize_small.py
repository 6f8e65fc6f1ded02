"""Small PMC + EPMC + obstacle run for compute-sanitizer (memcheck / racecheck / initcheck)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from lifelike_agility_and_play_b200 import _capi as capi
from lifelike_agility_and_play_b200.model.compile_model import load_model_blob
from lifelike_agility_and_play_b200.mocap import synthetic_mocap, obstacle_table
from lifelike_agility_and_play_b200.sim_envs.playground_env import INIT_STATE_RUN_0, epmc_engine_config

blob = load_model_blob()
mc = synthetic_mocap(4, seed=2, min_frames=400, max_frames=520)
mc.frames[:, 2] += 0.25 * np.exp(-((np.arange(len(mc.frames)) % 300 - 150) / 15.0) ** 2)
lib = capi.load_cuda_library()
rng = np.random.default_rng(0)
for n in (5, 70):
    e = capi.VecEngine(lib, n, blob, mc, seed=1, auto_reset=1)
    e.load_obstacles(*obstacle_table(mc), (0.025, 0.5, 0.2))
    e.reset()
    for t in range(12):
        e.step((0.4 * rng.standard_normal((n, 12))).astype(np.float32))
    e.reset(np.arange(n) % 2 == 0)
    e.close()
    erc = {'element_id': 0, 'friction_range': [0.4, 3.0], 'cmd_vary_freq_range': [3, 9], 'target_spd_range': [0.5, 3.0],
           'disturb_force_config': {'start_time': 0.02, 'interval_time': 0.1, 'duration_time': 0.05, 'horizontal_force': [0, 50], 'vertical_force': [0, 10]}}
    e = capi.VecEngine(lib, n, blob, None, seed=1, auto_reset=1, **epmc_engine_config(50.0, 50.0, 0.5, 16, 20, erc))
    e.set_init_state(INIT_STATE_RUN_0)
    e.reset()
    for t in range(25):
        e.step((0.4 * rng.standard_normal((n, 12))).astype(np.float32))
    e.close()
    # corridor arena (boxes, auxiliary edge cylinders, candidate staging) and the chase-tag pair game; large actions make robots fall
    # over: envs with more than 16 rows borrow their partner's lanes, CTAs full of them run the solver in two passes
    erc3 = dict(erc, element_id=3, auxiliary_radius=0.02)
    e = capi.VecEngine(lib, n, blob, None, seed=2, auto_reset=1, **epmc_engine_config(50.0, 50.0, 0.5, 16, 30, erc3))
    e.set_init_state(INIT_STATE_RUN_0)
    e.reset()
    for t in range(25):
        e.step((1.0 * rng.standard_normal((n, 12))).astype(np.float32))
    assert e.counters()[capi.CNT_DROPPED] == 0
    e.close()
    from lifelike_agility_and_play_b200.sim_envs.chase_tag_game_env import sepmc_engine_config
    n2 = n + (n & 1)
    e = capi.VecEngine(lib, n2, blob, None, seed=3, auto_reset=1, **sepmc_engine_config(50.0, 50.0, 0.5, 16, 30, {'friction_range': [0.4, 3.0], 'disturb_force_config': erc['disturb_force_config']}))
    e.set_init_state(INIT_STATE_RUN_0)
    e.reset()
    for t in range(25):
        e.step((1.0 * rng.standard_normal((n2, 12))).astype(np.float32))
    e.close()
# policy kernel (3xTF32 MMA layers, value head, sampling) on a ragged row count, rows read in place with a slab stride
import torch
from lifelike_agility_and_play_b200.policy import DevicePolicy
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from test_policy import random_weights
pol = DevicePolicy(random_weights(2), device=0)
for n in (1, 77):
    o = torch.randn((n, 223), device="cuda"); a = torch.zeros((n, 12), device="cuda"); v = torch.zeros((n,), device="cuda")
    p = torch.zeros((n,), device="cuda"); c = torch.zeros((n,), device="cuda", dtype=torch.int32)
    pol.forward(o.data_ptr(), 223, n, a.data_ptr(), c.data_ptr(), None)
    pol.forward_ex(o.data_ptr(), 223, n, a.data_ptr(), c.data_ptr(), v.data_ptr(), p.data_ptr(), 5, 9, None)
    torch.cuda.synchronize()
pol.close()
# environmental- / strategic-level policy kernel (convolutions, LSTM state in place, ragged row count, slab stride)
from lifelike_agility_and_play_b200.policy_epmc import DeviceHierPolicy, random_weights as hier_weights
for strategic in (False, True):
    hp = DeviceHierPolicy(hier_weights(strategic, 3), device=0)
    for n in (1, 37):
        ld = hp.obs_dim + 3
        o = torch.rand((n, ld), device="cuda"); a = torch.zeros((n, 12), device="cuda"); st = torch.zeros((n, hp.state_dim), device="cuda")
        d = (torch.rand((n,), device="cuda") < 0.5).to(torch.uint8); c = torch.zeros((n,), device="cuda", dtype=torch.int32); hd = torch.zeros((n,), device="cuda")
        hp.forward(o.data_ptr(), ld, n, d.data_ptr(), st.data_ptr(), a.data_ptr(), c.data_ptr(), hd.data_ptr() if strategic else None)
        hp.forward(o.data_ptr(), ld, n, None, st.data_ptr(), a.data_ptr(), None, None)
        torch.cuda.synchronize()
    hp.close()
print("sanitize run done")
