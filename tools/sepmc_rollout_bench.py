"""Timing of the strategic level's training rollouts on the GPU: the hierarchical policy kernel's deterministic strategic forward
(llq_hier_policy_forward) and strategic training forward (llq_hier_policy_forward_rec_strategic: heading sample, -log p, value tower) at
8192 rows, and the pair-steps/s of `SepmcRolloutWorker` (training forward on seat 0 + the frozen opponent's forward on seat 1 + copies +
fused step + reset per step) at 4096 chase-tag pairs, with random weights of the shipped architecture.  Steady state: one unroll of
pre-roll before any timed window; CUDA events on the stream the work runs on.  The card's name and power limit are read in the same run.
Prints one JSON line.

    python tools/sepmc_rollout_bench.py [--rows 8192] [--pairs 4096] [--unroll 32] [--unrolls 4] [--reps 50]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from hier_rollout_bench import card, timed, worker_rate  # noqa: E402


def sepmc_engine(n_robots):
    from lifelike_agility_and_play_b200 import _capi as capi
    from lifelike_agility_and_play_b200.model.compile_model import load_model_blob
    from lifelike_agility_and_play_b200.sim_envs.playground_env import INIT_STATE_RUN_0
    eng = capi.VecEngine(capi.load_cuda_library(), n_robots, load_model_blob(), None, device=0, seed=1234, auto_reset=1, env_kind=capi.ENV_SEPMC,
                         kp=50.0, kd=0.5, max_tau=16.0, ground_friction=1.0, friction_hi=1.0, max_steps=1000)
    eng.set_init_state(INIT_STATE_RUN_0)
    return eng


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=8192)
    ap.add_argument("--pairs", type=int, default=4096)
    ap.add_argument("--unroll", type=int, default=32)
    ap.add_argument("--unrolls", type=int, default=4)
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("sepmc_rollout_bench.py measures on a CUDA device; none is visible")
    from lifelike_agility_and_play_b200.parallel import SepmcRolloutWorker
    from lifelike_agility_and_play_b200.policy_epmc import DeviceHierPolicy, DeviceSepmcTrainPolicy, random_weights
    det, tr = DeviceHierPolicy(random_weights(True, 1), device=0), DeviceSepmcTrainPolicy(random_weights(True, 1), device=0)
    opp = DeviceHierPolicy(random_weights(True, 2), device=0)
    name, power = card()
    out = {"gpu": name, "power_limit": power, "rows": a.rows, "pairs": a.pairs, "unroll": a.unroll}
    eng = sepmc_engine(2 * a.pairs)
    worker = SepmcRolloutWorker(eng, tr, opp, a.unroll, "cuda:0", seed=3)
    ms, slab = worker_rate(worker, eng.reset(), a.unrolls)
    st = worker.stream
    # the two forwards on rolled-out observations (rows of the last record, repeated up to --rows), on the worker's stream
    n = a.rows
    obs = slab[a.unroll - 1].repeat((n + slab.shape[1] - 1) // slab.shape[1], 1)[:n].contiguous()
    s128, s192 = torch.zeros((n, 128), device="cuda"), torch.zeros((n, 192), device="cuda")
    act, codes = torch.zeros((n, 12), device="cuda"), torch.zeros((n,), dtype=torch.int32, device="cuda")
    hd, val, nlp = (torch.zeros((n,), device="cuda") for _ in range(3))
    with torch.cuda.stream(st):
        t_det = timed(lambda i: det.forward(obs.data_ptr(), obs.shape[1], n, None, s128.data_ptr(), act.data_ptr(), codes.data_ptr(), hd.data_ptr(),
                                            st.cuda_stream), st, a.reps)
        t_tr = timed(lambda i: tr.forward_rec(obs.data_ptr(), obs.shape[1], n, None, s192.data_ptr(), act.data_ptr(), codes.data_ptr(), hd.data_ptr(),
                                              val.data_ptr(), nlp.data_ptr(), 1, 3, 10 ** 6 + i, 0, st.cuda_stream), st, a.reps)
    out.update({"forward_deterministic_ms": round(t_det, 4), "forward_training_ms": round(t_tr, 4),
                "training_over_deterministic": round(t_tr / t_det, 3),
                "worker_pair_steps_per_s": round(a.pairs / (ms / 1e3)), "worker_ms_per_step": round(ms, 4)})
    eng.close(); det.close(); tr.close(); opp.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
