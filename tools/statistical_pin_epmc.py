#!/usr/bin/env python
"""Statistical pin of the terrain physics (SURVEY 8c(3), rows a18-a22): roll the reference's *shipped, Bullet-trained*
environmental-level policies (data/models/environmental_level_{hurdle,hole,cube}.model, host restatement in
lifelike_agility_and_play_b200/policy_epmc.py, argmax code + mean action like test_scripts/environmental_level/
test_environmental_level_env.py:95-100) through this repo's EPMC corridors with that script's environment configuration
(friction 0.4-1.0, target speed 3 m/s, pushes on, auxiliary_radius None) and count how the episodes end: reached the target at the
end of the corridor / fell / ran out of time.  A policy trained in Bullet only clears hurdles, bars and cube steps here if the
contact physics it meets behaves like Bullet's.

    python tools/statistical_pin_epmc.py --stage DIR                      # pack the three weight lists (git-ignored scratch)
    python tools/statistical_pin_epmc.py --staged DIR --engine cuda --element 3 --envs 1024 --steps 1200 --out profiles/...json
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
from lifelike_agility_and_play_b200.policy_epmc import EpmcPolicy  # noqa: E402

NAMES = {1: "hurdle", 2: "hole", 3: "cube"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--engine", default="cuda", choices=["oracle", "cuda"])
    ap.add_argument("--element", type=int, default=3)
    ap.add_argument("--envs", type=int, default=256)
    ap.add_argument("--steps", type=int, default=1200)
    ap.add_argument("--models", default="/root/reference/data/models")
    ap.add_argument("--stage", default="")
    ap.add_argument("--staged", default="")
    ap.add_argument("--sample", type=int, default=0, help="1: sample the code from the logits (the actor's behaviour) instead of argmax")
    ap.add_argument("--push", type=int, default=1)
    ap.add_argument("--aux", type=float, default=0.0, help="auxiliary_radius (the test script passes None, the train script 0.02)")
    ap.add_argument("--cfg", default="{}")
    ap.add_argument("--out", default="")
    ap.add_argument("--policy", default="host", choices=["host", "device"], help="numpy statement or csrc/llq_policy_hier.cu")
    a = ap.parse_args()
    if a.stage:
        from load_reference_model import load
        os.makedirs(a.stage, exist_ok=True)
        for e, nm in NAMES.items():
            w = load(os.path.join(a.models, "environmental_level_%s.model" % nm)).model
            np.savez(os.path.join(a.stage, "epmc_%s.npz" % nm), **{"w%d" % i: np.asarray(x, np.float32) for i, x in enumerate(w)})
        print("staged", a.stage)
        return
    if a.staged:
        wz = np.load(os.path.join(a.staged, "epmc_%s.npz" % NAMES[a.element]))
        weights = [wz["w%d" % i] for i in range(102)]
    else:
        from load_reference_model import load
        weights = load(os.path.join(a.models, "environmental_level_%s.model" % NAMES[a.element])).model
    pol = EpmcPolicy(weights)
    from lifelike_agility_and_play_b200.sim_envs.playground_env import INIT_STATE_RUN_0, epmc_engine_config
    erc = {'element_id': a.element, 'friction_range': [0.4, 1.0], 'cmd_vary_freq_range': [9999, 10000], 'target_spd_range': [3.0, 3.0],
           'hole_config': {'min_gap_height': 0.25, 'max_gap_height': 0.25}, 'auxiliary_radius': a.aux or None,
           'disturb_force_config': {'start_time': 0.5, 'interval_time': 1.0, 'duration_time': 0.2, 'horizontal_force': [0, 50],
                                    'vertical_force': [0, 10]} if a.push else None}
    cfg = epmc_engine_config(50.0, 50.0, 0.5, 16, 1000, erc)
    cfg.update(eval(a.cfg))
    if a.engine == "oracle":
        from oracle import oracle
        lib = oracle.load()
    else:
        lib = capi.load_cuda_library()
    n = a.envs
    eng = capi.VecEngine(lib, n, load_model_blob(), None, seed=2025, auto_reset=0, **cfg)
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
    rng = np.random.default_rng(7) if a.sample else None
    steps_alive, rew_sum = np.zeros(n, int), np.zeros(n)
    start_dist = None
    ep = {"reach": 0, "fall": 0, "timeup": 0, "other": 0}
    ep_len, ep_rew, ep_progress, ep_speed = [], [], [], []
    codes = np.zeros(256, int)
    for t in range(a.steps):
        if dev is not None:
            t_obs = torch.from_numpy(np.ascontiguousarray(obs, np.float32)).cuda(); t_done = torch.from_numpy(mask.astype(np.uint8)).cuda()
            dev.forward(t_obs.data_ptr(), obs.shape[1], n, t_done.data_ptr(), t_state.data_ptr(), t_act.data_ptr(), t_code.data_ptr())
            torch.cuda.synchronize()
            act, code = t_act.cpu().numpy(), t_code.cpu().numpy()
        else:
            act, state, code = pol.act(obs, state, mask, rng=rng, return_code=True)
        codes += np.bincount(code, minlength=256)
        mask[:] = 0
        if start_dist is None:
            aux0, st0 = eng.get(capi.F_AUX), eng.get(capi.F_STATE)
            start_dist = np.hypot(aux0[:, 2] - st0[:, 0], aux0[:, 3] - st0[:, 1])
        obs, r, d = eng.step(act)
        steps_alive += 1; rew_sum += r
        if d.any():
            st, aux = eng.get(capi.F_STATE).astype(np.float64), eng.get(capi.F_AUX)
            for i in np.flatnonzero(d):
                x, y, z, w = st[i, 3:7] / np.linalg.norm(st[i, 3:7])
                r22 = 1 - 2 * (x * x + y * y)
                left_z = 2 * (x * z + y * w) * 2 * (x * y + z * w) - 2 * (y * z - x * w) * (1 - 2 * (y * y + z * z))
                dist = float(np.hypot(aux[i, capi.AUX_TARGET_X] - st[i, 0], aux[i, capi.AUX_TARGET_Y] - st[i, 1]))
                cause = "reach" if dist < 0.5 else ("fall" if (r22 < 0.5 or abs(left_z) > 0.7071) else ("timeup" if aux[i, capi.AUX_COUNTER] >= cfg["max_steps"] else "other"))
                ep[cause] += 1
                ep_len.append(int(steps_alive[i])); ep_rew.append(float(rew_sum[i]))
                ep_progress.append(float(1.0 - dist / max(start_dist[i], 1e-6)))
                ep_speed.append(float((start_dist[i] - dist) / (steps_alive[i] * 0.02)))
            obs_r = eng.reset(d.astype(np.uint8))
            obs = np.where(d[:, None] != 0, obs_r, obs)
            mask = d.astype(np.float32)
            aux0, st0 = eng.get(capi.F_AUX), eng.get(capi.F_STATE)
            nd = np.hypot(aux0[:, 2] - st0[:, 0], aux0[:, 3] - st0[:, 1])
            start_dist = np.where(d != 0, nd, start_dist)
            steps_alive[d != 0] = 0; rew_sum[d != 0] = 0
    tot = max(1, sum(ep.values()))
    rep = {"engine": a.engine, "element": NAMES[a.element], "envs": n, "steps": a.steps, "episodes_finished": int(sum(ep.values())),
           "ended_by": ep, "reach_frac": ep["reach"] / tot, "fall_frac": ep["fall"] / tot,
           "median_episode_steps": float(np.median(ep_len)) if ep_len else None,
           "mean_progress_along_corridor": float(np.mean(ep_progress)) if ep_progress else None,
           "mean_speed_towards_target_mps": float(np.mean(ep_speed)) if ep_speed else None,
           "mean_episode_reward_sum": float(np.mean(ep_rew)) if ep_rew else None,
           "distinct_codes_used": int((codes > 0).sum()), "top_codes": [int(c) for c in np.argsort(-codes)[:8]],
           "config": {"friction_range": [0.4, 1.0], "target_spd": 3.0, "push": bool(a.push), "auxiliary_radius": a.aux or None,
                      "code": "sample" if a.sample else "argmax", "overrides": a.cfg, "policy": a.policy}}
    print(json.dumps(rep, indent=1))
    if a.out:
        json.dump(rep, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
