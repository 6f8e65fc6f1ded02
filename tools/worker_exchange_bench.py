"""Cost of handing the rollout workers' unrolls to the learner rank (parallel/rollout.py `UnrollExchange`), per level: PMC at 4096 envs,
EPMC at 8192 envs (element 0), SEPMC at 4096 chase-tag pairs against one opponent, T = 128, random weights of the shipped architectures.

Per level and rank:
  - the worker's rate (env-steps/s, pair-steps/s at the strategic level) over `--unrolls` unrolls after one of pre-roll, without the
    hand-over and with one `hand_over()` per unroll, alternated twice (without, with, without, with), each run on a fresh worker with the
    same seeds so that both run the same episodes; the window ends after the last transfer;
  - blocking: one hand-over and the wait for it with nothing else running;
  - exposed: (one unroll stepped while the previous one is in flight) - (one unroll alone), minima over `--reps`, as bench.py does for
    its trajectory slab.
On one GPU the exchange runs with `own_copy=True`: the transfer is the learner rank's device copy of its own unroll into the gathered
buffers.  With `--gpus K` (K >= 2) one NCCL rank per GPU steps its own shard (global env offset rank * N), rank 0 is the learner, and the
line holds the maxima over the ranks.  CUDA events on the worker's stream; the card's name and power limit are read in the same run.
Prints one JSON line per level.

    python tools/worker_exchange_bench.py [--gpus 1] [--unrolls 3] [--reps 3] [--levels pmc,epmc,sepmc]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from hier_rollout_bench import card  # noqa: E402
from policy_refresh_bench import pmc_weights  # noqa: E402

UNROLL = 128
ROBOTS = {"pmc": 4096, "epmc": 8192, "sepmc": 8192}


def make_worker(level, rank, device):
    """A worker of `level` on CUDA device `device` for shard `rank`, its first observation and the handles to close."""
    from lifelike_agility_and_play_b200 import _capi as capi
    from lifelike_agility_and_play_b200.model.compile_model import load_model_blob
    from lifelike_agility_and_play_b200.parallel import HierRolloutWorker, RolloutWorker, SepmcRolloutWorker
    from lifelike_agility_and_play_b200.policy_epmc import DeviceHierPolicy, DeviceSepmcTrainPolicy, random_weights
    from lifelike_agility_and_play_b200.sim_envs.playground_env import INIT_STATE_RUN_0, epmc_engine_config
    n, lib, blob, dev = ROBOTS[level], capi.load_cuda_library(), load_model_blob(), "cuda:%d" % device
    if level == "pmc":
        from lifelike_agility_and_play_b200.mocap import synthetic_mocap
        from lifelike_agility_and_play_b200.policy import DevicePolicy
        eng = capi.VecEngine(lib, n, blob, synthetic_mocap(8, seed=2, min_frames=380, max_frames=700), seed=21, device=device, auto_reset=1,
                             global_env_offset=rank * n)
        pol = DevicePolicy(pmc_weights(1), device=device)
        return RolloutWorker(eng, pol, UNROLL, dev, seed=5), eng.reset(), [pol, eng]
    if level == "epmc":
        erc = {'element_id': 0, 'friction_range': [0.4, 3.0], 'cmd_vary_freq_range': [25, 200], 'target_spd_range': [0.5, 3.0],
               'hole_config': {'min_gap_height': 0.25, 'max_gap_height': 0.25}, 'auxiliary_radius': 0.02,
               'disturb_force_config': {'start_time': 0.5, 'interval_time': 1.0, 'duration_time': 0.2, 'horizontal_force': [0, 50],
                                        'vertical_force': [0, 10]}}              # hier_rollout_bench.py (example_epmc_train.sh:88-117)
        eng = capi.VecEngine(lib, n, blob, None, device=device, seed=1234, auto_reset=1, global_env_offset=rank * n,
                             **epmc_engine_config(50.0, 50.0, 0.5, 16, 1000, erc))
        eng.set_init_state(INIT_STATE_RUN_0)
        pol = DeviceHierPolicy(random_weights(False, 1), device=device, train=True)
        return HierRolloutWorker(eng, pol, UNROLL, dev, seed=5), eng.reset(), [pol, eng]
    eng = capi.VecEngine(lib, n, blob, None, device=device, seed=1234, auto_reset=1, env_kind=capi.ENV_SEPMC, kp=50.0, kd=0.5, max_tau=16.0,
                         ground_friction=1.0, friction_hi=1.0, max_steps=1000, global_env_offset=rank * n)     # sepmc_rollout_bench.py
    eng.set_init_state(INIT_STATE_RUN_0)
    pol, opp = DeviceSepmcTrainPolicy(random_weights(True, 1), device=device), DeviceHierPolicy(random_weights(True, 2), device=device)
    return SepmcRolloutWorker(eng, pol, opp, UNROLL, dev, seed=5), eng.reset(), [pol, opp, eng]


def unroll(worker):
    for _ in range(worker.T):
        worker.step()
    return worker.finish_unroll()


def measure(level, rank, device, world, a):
    import torch
    import torch.distributed as dist
    from lifelike_agility_and_play_b200.parallel import UnrollExchange

    def sync():
        torch.cuda.synchronize(device)
        if world > 1:
            dist.barrier()

    def rate(with_exchange):
        worker, o0, handles = make_worker(level, rank, device)
        xch = UnrollExchange(worker, own_copy=True) if with_exchange else None
        worker.start(o0)
        u = unroll(worker)
        b = xch.hand_over(u) if xch else None
        sync()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(worker.stream)
        for _ in range(a.unrolls):
            u = unroll(worker)
            if xch:
                b = xch.hand_over(u)
        if xch:
            xch.core.wait(b, worker.stream)
        e1.record(worker.stream)
        e1.synchronize()
        out = worker.rows * worker.T * a.unrolls / (e0.elapsed_time(e1) / 1e3)
        for h in handles:
            h.close()
        return out, xch.bytes_per_rank if xch else None

    runs = {"without": [], "with": []}
    for mode in ("without", "with", "without", "with"):
        r, nbytes = rate(mode == "with")
        runs[mode].append(r)
        if nbytes:
            bytes_per_rank = nbytes

    worker, o0, handles = make_worker(level, rank, device)
    xch = UnrollExchange(worker, own_copy=True)
    ws = worker.stream
    worker.start(o0)
    u = unroll(worker)

    def timed(fn):
        sync()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(ws)
        fn()
        e1.record(ws)
        e1.synchronize()
        return e0.elapsed_time(e1)

    def alone():
        state["u"] = unroll(worker)

    def overlapped():
        xch.hand_over(state["u"])
        state["u"] = unroll(worker)          # its finish_unroll() waits for the transfer before it writes into that slab

    def blocking():
        xch.core.wait(xch.hand_over(state["u"]), ws)

    state = {"u": u}
    t_alone, t_over, t_block = [], [], []
    for _ in range(a.reps):
        t_alone.append(timed(alone))
        t_over.append(timed(overlapped))
    for _ in range(a.reps):
        state["u"] = unroll(worker)
        t_block.append(timed(blocking))
    for h in handles:
        h.close()
    x = [min(t_alone), min(t_over), max(0.0, min(t_over) - min(t_alone)), sorted(t_block)[len(t_block) // 2]]
    x += runs["without"] + runs["with"]
    if world > 1:
        v = torch.tensor(x, dtype=torch.float64, device="cuda:%d" % device)
        dist.all_reduce(v, op=dist.ReduceOp.MAX)
        x = v.tolist()
    return {"unroll_alone_ms": round(x[0], 3), "unroll_overlapped_ms": round(x[1], 3), "exposed_ms_per_unroll": round(x[2], 3),
            "blocking_ms": round(x[3], 3), "rate_without_handover": [round(r) for r in x[4:6]], "rate_with_handover": [round(r) for r in x[6:8]],
            "bytes_per_rank": bytes_per_rank}


def run(rank, world, a, port):
    import torch
    import torch.distributed as dist
    if world > 1:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    name, power = card()
    for level in a.levels.split(","):
        out = measure(level, rank, rank, world, a)
        if rank == 0:
            unit = "pair-steps/s" if level == "sepmc" else "env-steps/s"
            head = {"level": level, "gpu": name, "power_limit": power, "world": world, "per_rank": ROBOTS[level] // (2 if level == "sepmc" else 1),
                    "unit": unit, "unroll": UNROLL, "unrolls": a.unrolls,
                    "transfer": "learner rank's own device copy" if world == 1 else "NCCL to rank 0 (maxima over ranks)"}
            print(json.dumps({**head, **out}), flush=True)
    if world > 1:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--unrolls", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--levels", default="pmc,epmc,sepmc")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("worker_exchange_bench.py measures on CUDA devices; none is visible")
    if a.gpus > torch.cuda.device_count():
        raise SystemExit("--gpus %d: only %d CUDA devices are visible" % (a.gpus, torch.cuda.device_count()))
    if a.unrolls < 3:
        raise SystemExit("--unrolls must be at least 3")
    if a.gpus == 1:
        run(0, 1, a, None)
    else:
        import torch.multiprocessing as mp
        mp.spawn(run, args=(a.gpus, a, 29700 + os.getpid() % 2000), nprocs=a.gpus)


if __name__ == "__main__":
    main()
