"""Cost of a model refresh on the GPU: the time of one `set_weights` (host list and device blob) for each handle kind -- the PMC policy
(upload + pack kernel), the environmental- and strategic-level deterministic and training handles and one model of a 16-model opponent
pool (one copy each) -- and the steps/s of the three rollout workers with a refresh every 128 steps (one per 128-step unroll, of the
weights the worker runs, so that the episodes are those of the run without refreshes) against none, at PMC 4096 envs, EPMC 8192 envs and SEPMC 4096 pairs, random weights of the shipped architectures.
Refresh time: CUDA events on the stream the refreshes are queued on, back to back, so the number is the larger of the host's and the
device's cost per refresh.  Worker rates: one unroll of pre-roll, then `--unrolls` timed unrolls between CUDA events on the worker's
stream; the run without refreshes comes first and again last, a bracket on the drift between runs.  The card's name and power limit
are read in the same run.  Prints one JSON line.

    python tools/policy_refresh_bench.py [--unroll 128] [--unrolls 3] [--reps 50]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from hier_rollout_bench import card, epmc_engine, timed  # noqa: E402
from sepmc_rollout_bench import sepmc_engine  # noqa: E402


def pmc_weights(seed):
    import numpy as np
    from lifelike_agility_and_play_b200.policy import PMC_SHAPES
    rng = np.random.default_rng(seed)
    w = [(rng.standard_normal(s) / np.sqrt(s[0] if len(s) == 2 and s[0] > 1 else 1.0)).astype(np.float32) for s in PMC_SHAPES]
    w[1] = np.abs(w[1]) + 0.1; w[3] = np.abs(w[3]) + 0.1
    w[25] *= 0.05; w[27][:] = -2.0
    return w


def refresh_ms(handle, sets, blobs, stream, reps, k=None):
    """ms per refresh from host lists and from device blobs, alternating the two weight sets."""
    head = () if k is None else (k,)
    fn = handle.set_weights if k is None else handle.set_model
    host = timed(lambda i: fn(*head, sets[i % 2], stream=stream.cuda_stream), stream, reps)
    dev = timed(lambda i: fn(*head, blobs[i % 2], stream=stream.cuda_stream), stream, reps)
    return round(host, 4), round(dev, 4)


def worker_rate(worker, first_obs, unrolls, refresh):
    """Steps/s of `worker` over `unrolls` unrolls after one of pre-roll; `refresh(u)` (or None) is called before each timed unroll."""
    import torch
    worker.start(first_obs)
    for _ in range(worker.T):
        worker.step()
    worker.finish_unroll()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(worker.stream)
    for u in range(unrolls):
        if refresh is not None:
            refresh(u)
        for _ in range(worker.T):
            worker.step()
        worker.finish_unroll()
    e1.record(worker.stream)
    e1.synchronize()
    return round(worker.rows * worker.T * unrolls / (e0.elapsed_time(e1) / 1e3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--unroll", type=int, default=128)
    ap.add_argument("--unrolls", type=int, default=3)
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("policy_refresh_bench.py measures on a CUDA device; none is visible")
    from lifelike_agility_and_play_b200 import _capi as capi
    from lifelike_agility_and_play_b200.mocap import synthetic_mocap
    from lifelike_agility_and_play_b200.model.compile_model import load_model_blob
    from lifelike_agility_and_play_b200.parallel import HierRolloutWorker, RolloutWorker, SepmcRolloutWorker
    from lifelike_agility_and_play_b200.policy import DevicePolicy, pack_weights
    from lifelike_agility_and_play_b200.policy_epmc import DeviceHierPolicy, DeviceOpponentPool, DeviceSepmcTrainPolicy, random_weights, weight_blob
    name, power = card()
    out = {"gpu": name, "power_limit": power, "unroll": a.unroll}
    st = torch.cuda.Stream()
    pmc = [pmc_weights(s) for s in (1, 2)]
    epmc, sepmc = [random_weights(False, s) for s in (1, 2)], [random_weights(True, s) for s in (1, 2)]
    pmc_dev = [torch.from_numpy(pack_weights(w)).cuda() for w in pmc]
    epmc_dev = [torch.from_numpy(weight_blob(w)[0]).cuda() for w in epmc]
    sepmc_dev = [torch.from_numpy(weight_blob(w)[0]).cuda() for w in sepmc]
    kinds = (("pmc", lambda: DevicePolicy(pmc[0], device=0), pmc, pmc_dev),
             ("epmc", lambda: DeviceHierPolicy(epmc[0], device=0), epmc, epmc_dev),
             ("epmc_train", lambda: DeviceHierPolicy(epmc[0], device=0, train=True), epmc, epmc_dev),
             ("sepmc", lambda: DeviceHierPolicy(sepmc[0], device=0), sepmc, sepmc_dev),
             ("sepmc_train", lambda: DeviceSepmcTrainPolicy(sepmc[0], device=0), sepmc, sepmc_dev))
    for kind, make, sets, blobs in kinds:
        h = make()
        out["refresh_%s_host_ms" % kind], out["refresh_%s_device_ms" % kind] = refresh_ms(h, sets, blobs, st, a.reps)
        h.close()
    pool = DeviceOpponentPool([random_weights(True, 10 + k) for k in range(16)], device=0, max_rows=4096)
    out["refresh_pool16_model_host_ms"], out["refresh_pool16_model_device_ms"] = refresh_ms(pool, sepmc, sepmc_dev, st, a.reps, k=5)
    pool.close()
    torch.cuda.synchronize()

    mocap = synthetic_mocap(8, seed=2, min_frames=380, max_frames=700)

    def pmc_worker():
        eng = capi.VecEngine(capi.load_cuda_library(), 4096, load_model_blob(), mocap, seed=21, device=0, auto_reset=1)
        return RolloutWorker(eng, DevicePolicy(pmc[0], device=0), a.unroll, "cuda:0", seed=5), eng

    def epmc_worker():
        eng = epmc_engine(8192, 0)
        return HierRolloutWorker(eng, DeviceHierPolicy(epmc[0], device=0, train=True), a.unroll, "cuda:0", seed=5), eng

    def sepmc_worker():
        eng = sepmc_engine(2 * 4096)
        opp = DeviceHierPolicy(sepmc[1], device=0)
        return SepmcRolloutWorker(eng, DeviceSepmcTrainPolicy(sepmc[0], device=0), opp, a.unroll, "cuda:0", seed=5), eng

    for kind, make, sets, blobs in (("pmc_4096", pmc_worker, pmc, pmc_dev), ("epmc_8192", epmc_worker, epmc, epmc_dev),
                                    ("sepmc_4096_pairs", sepmc_worker, sepmc, sepmc_dev)):
        # the refresh re-sends the weights the worker runs: other weights would change the episodes, and with them the engine's cost
        for mode, refresh in (("none", None), ("host", lambda u: w.update_policy(sets[0])), ("device", lambda u: w.update_policy(blobs[0])),
                              ("none_again", None)):
            w, eng = make()
            out["worker_%s_steps_per_s_refresh_%s" % (kind, mode)] = worker_rate(w, eng.reset(), a.unrolls, refresh)
            w.pol.close(); eng.close()
            torch.cuda.synchronize()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
