#!/usr/bin/env python
"""Behavioural pin of the strategic level (SURVEY rows a23-a26): both robots of every pair run the reference's shipped, Bullet-trained
strategic-level policy (data/models/strategic_level.model; host restatement lifelike_agility_and_play_b200/policy_epmc.py::SepmcPolicy,
mean heading + argmax code + mean action like test_scripts/strategic_level/test_strategic_level_env.py:96) in this repo's chase-tag
game with that script's configuration (friction 0.4-1.0, pushes on, shipped empty arena) and the games are counted by how they end:
tag (the chaser touches the runner), a fall, or time-up.

    python tools/statistical_pin_sepmc.py --stage DIR
    python tools/statistical_pin_sepmc.py --staged DIR --engine oracle --pairs 64 --steps 1000 --out profiles/...json
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from lifelike_agility_and_play_b200 import _capi as capi  # noqa: E402
from lifelike_agility_and_play_b200.model.compile_model import load_model_blob  # noqa: E402
from lifelike_agility_and_play_b200.policy_epmc import SepmcPolicy  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--engine", default="oracle", choices=["oracle", "cuda"])
    ap.add_argument("--pairs", type=int, default=32)
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--model", default="/root/reference/data/models/strategic_level.model")
    ap.add_argument("--stage", default="")
    ap.add_argument("--staged", default="")
    ap.add_argument("--push", type=int, default=1)
    ap.add_argument("--out", default="")
    ap.add_argument("--policy", default="host", choices=["host", "device"], help="numpy statement or csrc/llq_policy_hier.cu")
    a = ap.parse_args()
    if a.stage:
        from load_reference_model import load
        os.makedirs(a.stage, exist_ok=True)
        w = load(a.model).model
        np.savez(os.path.join(a.stage, "sepmc.npz"), **{"w%d" % i: np.asarray(x, np.float32) for i, x in enumerate(w)})
        print("staged", a.stage)
        return
    if a.staged:
        wz = np.load(os.path.join(a.staged, "sepmc.npz"))
        weights = [wz["w%d" % i] for i in range(152)]
    else:
        from load_reference_model import load
        weights = load(a.model).model
    pol = SepmcPolicy(weights)
    from lifelike_agility_and_play_b200.sim_envs.chase_tag_game_env import sepmc_engine_config
    from lifelike_agility_and_play_b200.sim_envs.playground_env import INIT_STATE_RUN_0
    erc = {'friction_range': [0.4, 1.0],
           'disturb_force_config': {'start_time': 0.5, 'interval_time': 1.0, 'duration_time': 0.2, 'horizontal_force': [0, 50],
                                    'vertical_force': [0, 10]} if a.push else None}
    cfg = sepmc_engine_config(50.0, 50.0, 0.5, 16, 1000, erc)
    if a.engine == "oracle":
        from oracle import oracle
        lib = oracle.load()
    else:
        lib = capi.load_cuda_library()
    n = 2 * a.pairs
    eng = capi.VecEngine(lib, n, load_model_blob(), None, seed=2026, auto_reset=0, **cfg)
    eng.set_init_state(INIT_STATE_RUN_0)
    obs = eng.reset()
    state, mask = pol.initial_state(n), np.ones(n, np.float32)
    dev = None
    if a.policy == "device":
        import torch
        from lifelike_agility_and_play_b200.policy_epmc import DeviceHierPolicy
        dev = DeviceHierPolicy(weights, device=0)
        t_state = torch.zeros((n, dev.state_dim), device="cuda"); t_act = torch.zeros((n, 12), device="cuda")
        t_code = torch.zeros((n,), device="cuda", dtype=torch.int32)
    alive = np.zeros(a.pairs, int)
    ends = {"tag": 0, "fall": 0, "timeup": 0}
    ep_len, tag_rew, speeds, gaps = [], [], [], []
    codes = np.zeros(256, int)
    for t in range(a.steps):
        if dev is not None:
            t_obs = torch.from_numpy(np.ascontiguousarray(obs, np.float32)).cuda(); t_done = torch.from_numpy(mask.astype(np.uint8)).cuda()
            dev.forward(t_obs.data_ptr(), obs.shape[1], n, t_done.data_ptr(), t_state.data_ptr(), t_act.data_ptr(), t_code.data_ptr())
            torch.cuda.synchronize()
            act, code = t_act.cpu().numpy(), t_code.cpu().numpy()
        else:
            act, state, ang, code = pol.act(obs, state, mask, return_aux=True)
        codes += np.bincount(code, minlength=256)
        mask[:] = 0
        obs, r, d = eng.step(act)
        alive += 1
        st = eng.get(capi.F_STATE).astype(np.float64)
        speeds.append(np.hypot(st[:, 7], st[:, 8]).mean())
        gaps.append(np.hypot(st[0::2, 0] - st[1::2, 0], st[0::2, 1] - st[1::2, 1]).mean())
        if d.any():
            aux = eng.get(capi.F_AUX)
            for p in np.flatnonzero(d[0::2]):
                fell = False
                for i in (2 * p, 2 * p + 1):
                    x, y, z, w = st[i, 3:7] / np.linalg.norm(st[i, 3:7])
                    r22 = 1 - 2 * (x * x + y * y)
                    left_z = 2 * (x * z + y * w) * 2 * (x * y + z * w) - 2 * (y * z - x * w) * (1 - 2 * (y * y + z * z))
                    fell = fell or r22 < 0.5 or abs(left_z) > 0.7071
                cause = "fall" if fell else ("timeup" if aux[2 * p, capi.AUX_COUNTER] >= cfg["max_steps"] else "tag")
                ends[cause] += 1
                ep_len.append(int(alive[p]))
                if cause == "tag":
                    tag_rew.append(float(r[2 * p]))
                alive[p] = 0
            obs_r = eng.reset(d.astype(np.uint8))
            obs = np.where(d[:, None] != 0, obs_r, obs)
            mask = d.astype(np.float32)
    tot = max(1, sum(ends.values()))
    rep = {"engine": a.engine, "pairs": a.pairs, "steps": a.steps, "games_finished": int(sum(ends.values())), "ended_by": ends,
           "tag_frac": ends["tag"] / tot, "fall_frac": ends["fall"] / tot, "median_game_steps": float(np.median(ep_len)) if ep_len else None,
           "mean_robot_speed_mps": float(np.mean(speeds)), "mean_distance_between_the_two_robots_m": float(np.mean(gaps)),
           "robot0_reward_at_tag_mean": float(np.mean(tag_rew)) if tag_rew else None,
           "distinct_codes_used": int((codes > 0).sum()),
           "config": {"friction_range": [0.4, 1.0], "push": bool(a.push), "control_spd": "engine default", "policy": "mean heading, argmax code, mean action", "policy_on": a.policy}}
    print(json.dumps(rep, indent=1))
    if a.out:
        json.dump(rep, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
