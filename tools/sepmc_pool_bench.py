"""Timing of the strategic level's opponent pool on the GPU: the deterministic strategic forward (llq_hier_policy_forward, one model)
against the pool forward (llq_hier_policy_forward_pool, assign kernel + pool kernel) at 8192 rows for K = 1, 4, 16 and 64 models with
uniform probabilities, the assign kernel alone (the pool call with a row whose model is out of range everywhere: no segment, so the pool
kernel's CTAs return at once), and the pair-steps/s of `SepmcRolloutWorker` at 4096 chase-tag pairs against one opponent and against a
pool of 16, with random weights of the shipped architecture.  Each pool forward sees a quarter of its rows drawing (done set), the rest
keeping a uniformly spread model.  K = 64 models of 1.27 MB each no longer fit in the 50 MB L2; K <= 16 do.  CUDA events on one stream;
the card's name and power limit are read in the same run.  Prints one JSON line.

    python tools/sepmc_pool_bench.py [--rows 8192] [--pairs 4096] [--unroll 32] [--unrolls 4] [--reps 50]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from hier_rollout_bench import card, timed, worker_rate  # noqa: E402
from sepmc_rollout_bench import sepmc_engine  # noqa: E402


def opponent_rate(opponent, pairs, unroll, unrolls):
    """Pair-steps/s of SepmcRolloutWorker against `opponent`, and the [2P, 984] records of one step of the run."""
    from lifelike_agility_and_play_b200.parallel import SepmcRolloutWorker
    from lifelike_agility_and_play_b200.policy_epmc import DeviceSepmcTrainPolicy, random_weights
    tr = DeviceSepmcTrainPolicy(random_weights(True, 1), device=0)
    eng = sepmc_engine(2 * pairs)
    ms, slab = worker_rate(SepmcRolloutWorker(eng, tr, opponent, unroll, "cuda:0", seed=3), eng.reset(), unrolls)
    obs = slab[unroll - 1].clone()
    eng.close(); tr.close()
    return round(pairs / (ms / 1e3)), obs


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
        raise SystemExit("sepmc_pool_bench.py measures on a CUDA device; none is visible")
    from lifelike_agility_and_play_b200.policy_epmc import DeviceHierPolicy, DeviceOpponentPool, random_weights
    name, power = card()
    out = {"gpu": name, "power_limit": power, "rows": a.rows, "pairs": a.pairs, "unroll": a.unroll}
    models = [random_weights(True, 10 + k) for k in range(64)]
    one = DeviceHierPolicy(models[0], device=0)
    rate1, last = opponent_rate(one, a.pairs, a.unroll, a.unrolls)
    pool16 = DeviceOpponentPool(models[:16], device=0, max_rows=a.pairs)
    rate16, _ = opponent_rate(pool16, a.pairs, a.unroll, a.unrolls)
    pool16.close()
    out.update({"worker_pair_steps_per_s_one_opponent": rate1, "worker_pair_steps_per_s_pool16": rate16})
    n = a.rows
    st = torch.cuda.Stream()
    obs = last.repeat((n + last.shape[0] - 1) // last.shape[0], 1)[:n].contiguous()
    state = torch.zeros((n, 128), device="cuda")
    act, codes, hd = torch.zeros((n, 12), device="cuda"), torch.zeros((n,), dtype=torch.int32, device="cuda"), torch.zeros((n,), device="cuda")
    done = (torch.arange(n, device="cuda") % 4 == 0).to(torch.uint8)
    with torch.cuda.stream(st):
        out["forward_deterministic_ms"] = round(timed(lambda i: one.forward(obs.data_ptr(), obs.shape[1], n, done.data_ptr(), state.data_ptr(),
                                                                            act.data_ptr(), codes.data_ptr(), hd.data_ptr(), st.cuda_stream),
                                                      st, a.reps), 4)
        for K in (1, 4, 16, 64):
            pool = DeviceOpponentPool(models[:K], device=0, max_rows=n)
            model = (torch.arange(n, device="cuda", dtype=torch.int32) * K) // n
            out["forward_pool_k%d_ms" % K] = round(timed(lambda i: pool.forward(obs.data_ptr(), obs.shape[1], n, done.data_ptr(), state.data_ptr(),
                                                                                 act.data_ptr(), codes.data_ptr(), hd.data_ptr(), model.data_ptr(),
                                                                                 None, 1, 5, i, 0, st.cuda_stream), st, a.reps), 4)
            if K == 64:
                off = torch.full((n,), -1, dtype=torch.int32, device="cuda")
                out["assign_only_k64_ms"] = round(timed(lambda i: pool.forward(obs.data_ptr(), obs.shape[1], n, None, state.data_ptr(), act.data_ptr(),
                                                                                codes.data_ptr(), hd.data_ptr(), off.data_ptr(), None, 1, 5, i, 0,
                                                                                st.cuda_stream), st, a.reps), 4)
            pool.close()
    one.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
