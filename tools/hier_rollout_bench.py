"""Timing of the environmental level's training rollouts on the GPU: the hierarchical policy kernel's deterministic forward
(llq_hier_policy_forward) and training forward (llq_hier_policy_forward_rec: value tower, Gumbel sample, -log p), and the env-steps/s of
`HierRolloutWorker` (training forward + fused step + reset per step), at 8192 EPMC envs on elements 0 and 3 with random weights of the
shipped architecture.  Steady state: one unroll of pre-roll before any timed window (`worker_rate`, which the strategic level's tools
share); CUDA events on the stream the work runs on.  The card's name and power limit are read in the same run.  Prints one JSON line.

    python tools/hier_rollout_bench.py [--envs 8192] [--unroll 32] [--unrolls 4] [--reps 50]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(0), "not read"
    return name, power


def epmc_engine(n, element):
    from lifelike_agility_and_play_b200 import _capi as capi
    from lifelike_agility_and_play_b200.model.compile_model import load_model_blob
    from lifelike_agility_and_play_b200.sim_envs.playground_env import INIT_STATE_RUN_0, epmc_engine_config
    erc = {'element_id': element, 'friction_range': [0.4, 3.0], 'cmd_vary_freq_range': [25, 200], 'target_spd_range': [0.5, 3.0],
           'hole_config': {'min_gap_height': 0.25, 'max_gap_height': 0.25}, 'auxiliary_radius': 0.02,
           'disturb_force_config': {'start_time': 0.5, 'interval_time': 1.0, 'duration_time': 0.2, 'horizontal_force': [0, 50], 'vertical_force': [0, 10]}}
    cfg = epmc_engine_config(50.0, 50.0, 0.5, 16, 1000, erc)       # train_scripts/example_epmc_train.sh:88-117
    eng = capi.VecEngine(capi.load_cuda_library(), n, load_model_blob(), None, device=0, seed=1234, auto_reset=1, **cfg)
    eng.set_init_state(INIT_STATE_RUN_0)
    return eng


def timed(fn, stream, reps):
    import torch
    for i in range(5):
        fn(i)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for i in range(reps):
        fn(i)
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def worker_rate(worker, first_obs, unrolls):
    """Milliseconds per step of a rollout worker: one unroll of pre-roll (module loads, a full unroll of episodes under way), then
    `unrolls` unrolls between CUDA events on the worker's stream.  Returns (ms per step, the pre-roll's slab view, which the timed
    unrolls have refilled since with later records); everything has finished on return."""
    import torch
    worker.start(first_obs)
    for _ in range(worker.T):
        worker.step()
    slab = worker.finish_unroll().slab
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(worker.stream)
    for _ in range(unrolls):
        for _ in range(worker.T):
            worker.step()
        worker.finish_unroll()
    e1.record(worker.stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / (worker.T * unrolls), slab


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=8192)
    ap.add_argument("--unroll", type=int, default=32)
    ap.add_argument("--unrolls", type=int, default=4)
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("hier_rollout_bench.py measures on a CUDA device; none is visible")
    from lifelike_agility_and_play_b200.parallel import HierRolloutWorker
    from lifelike_agility_and_play_b200.policy_epmc import DeviceHierPolicy, random_weights
    n = a.envs
    w = random_weights(False, 1)
    det, tr = DeviceHierPolicy(w, device=0), DeviceHierPolicy(w, device=0, train=True)
    name, power = card()
    out = {"gpu": name, "power_limit": power, "envs": n, "unroll": a.unroll}
    for element in (0, 3):
        eng = epmc_engine(n, element)
        worker = HierRolloutWorker(eng, tr, a.unroll, "cuda:0", seed=3)
        ms, slab = worker_rate(worker, eng.reset(), a.unrolls)
        st = worker.stream
        # the two forwards on rolled-out observations, on the worker's stream
        obs = slab[a.unroll - 1]
        s64, s128 = torch.zeros((n, 64), device="cuda"), torch.zeros((n, 128), device="cuda")
        act, codes = torch.zeros((n, 12), device="cuda"), torch.zeros((n,), dtype=torch.int32, device="cuda")
        val, nlp = torch.zeros((n,), device="cuda"), torch.zeros((n,), device="cuda")
        with torch.cuda.stream(st):
            t_det = timed(lambda i: det.forward(obs.data_ptr(), obs.shape[1], n, None, s64.data_ptr(), act.data_ptr(), codes.data_ptr(), None,
                                                st.cuda_stream), st, a.reps)
            t_tr = timed(lambda i: tr.forward_rec(obs.data_ptr(), obs.shape[1], n, None, s128.data_ptr(), act.data_ptr(), codes.data_ptr(),
                                                  val.data_ptr(), nlp.data_ptr(), 1, 3, 10 ** 6 + i, 0, st.cuda_stream), st, a.reps)
        out["element%d" % element] = {"forward_deterministic_ms": round(t_det, 4), "forward_training_ms": round(t_tr, 4),
                                      "training_over_deterministic": round(t_tr / t_det, 3),
                                      "worker_env_steps_per_s": round(n / (ms / 1e3)), "worker_ms_per_step": round(ms, 4)}
        eng.close()
    det.close(); tr.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
