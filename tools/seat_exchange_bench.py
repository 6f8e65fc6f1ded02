"""The strategic level's learner-seat hand-over (`UnrollExchange(worker, learner_seat_only=True)`) on one GPU, T = 128, P = 4096 chase-tag
pairs, random weights of the shipped architecture, one opponent (as tools/worker_exchange_bench.py).

  - the pack kernel (`pack_learner_seat`, csrc/llq_seat_pack.cu): CUDA events around `--launches` launches after 5 of warm-up, on a
    random `[T, 2P, 984]` slab; bytes moved = read + write of the `[T, P, 984]` seat-0 records (2 x T x P x 984 x 4), over the time,
    against 3.35 TB/s (the H100 SXM data sheet's HBM3 bandwidth);
  - the worker: pair-steps/s over `--unrolls` unrolls after one of pre-roll, with the default exchange (both seats) and the learner-seat
    exchange, alternated twice (default, seat, default, seat), each on a fresh worker with the same seeds; the window ends after the
    last transfer.  On one GPU the transfer is the learner rank's own device copy (`own_copy=True`);
  - per mode: one unroll alone, one unroll with the previous one's hand-over in flight, the exposed difference (minima over `--reps`),
    the blocking hand-over (median), `bytes_per_rank` and the peak of `torch.cuda.max_memory_allocated` over that mode's runs (torch's
    allocations: the slabs, the send and receive buffers; not the engine's and policies' own device memory).
The card's name and power limit are read in the same run.  Prints one JSON line.

    python tools/seat_exchange_bench.py [--unrolls 3] [--reps 3] [--launches 50]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from hier_rollout_bench import card  # noqa: E402
from worker_exchange_bench import UNROLL, make_worker, unroll  # noqa: E402

PAIRS = 4096
HBM_BYTES_PER_S = 3.35e12


def pack_kernel(launches):
    import torch
    from lifelike_agility_and_play_b200.parallel import pack_learner_seat
    from lifelike_agility_and_play_b200.parallel.trajectory import SEPMC_TRAJ_WIDTH as W
    slab = torch.randn((UNROLL, 2 * PAIRS, W), device="cuda")
    out = torch.empty((UNROLL, PAIRS, W), device="cuda")
    for _ in range(5):
        pack_learner_seat(slab, out)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        pack_learner_seat(slab, out)
    e1.record()
    e1.synchronize()
    ms = e0.elapsed_time(e1) / launches
    assert torch.equal(out, slab[:, 0::2])
    nbytes = 2 * out.numel() * 4
    del slab, out
    torch.cuda.empty_cache()
    return {"pack_ms": round(ms, 4), "pack_bytes": nbytes, "pack_bytes_per_s": round(nbytes / (ms / 1e3) / 1e12, 3),
            "pack_share_of_3.35TBps": round(nbytes / (ms / 1e3) / HBM_BYTES_PER_S, 3)}


def exchange(seat_only, worker):
    from lifelike_agility_and_play_b200.parallel import UnrollExchange
    return UnrollExchange(worker, own_copy=True, learner_seat_only=seat_only)


def rate(seat_only, a):
    import torch
    worker, o0, handles = make_worker("sepmc", 0, 0)
    xch = exchange(seat_only, worker)
    worker.start(o0)
    xch.hand_over(unroll(worker))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(worker.stream)
    for _ in range(a.unrolls):
        b = xch.hand_over(unroll(worker))
    xch.core.wait(b, worker.stream)
    e1.record(worker.stream)
    e1.synchronize()
    out = worker.rows * worker.T * a.unrolls / (e0.elapsed_time(e1) / 1e3)
    for h in handles:
        h.close()
    return out, xch.bytes_per_rank


def exposed(seat_only, a):
    import torch
    worker, o0, handles = make_worker("sepmc", 0, 0)
    xch = exchange(seat_only, worker)
    ws = worker.stream
    worker.start(o0)
    state = {"u": unroll(worker)}

    def timed(fn):
        torch.cuda.synchronize()
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
        state["u"] = unroll(worker)

    def blocking():
        xch.core.wait(xch.hand_over(state["u"]), ws)

    t_alone, t_over, t_block = [], [], []
    for _ in range(a.reps):
        t_alone.append(timed(alone))
        t_over.append(timed(overlapped))
    for _ in range(a.reps):
        state["u"] = unroll(worker)
        t_block.append(timed(blocking))
    for h in handles:
        h.close()
    return {"unroll_alone_ms": round(min(t_alone), 3), "unroll_overlapped_ms": round(min(t_over), 3),
            "exposed_ms_per_unroll": round(max(0.0, min(t_over) - min(t_alone)), 3), "blocking_ms": round(sorted(t_block)[len(t_block) // 2], 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--unrolls", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--launches", type=int, default=50)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("seat_exchange_bench.py measures on a CUDA device; none is visible")
    name, power = card()
    out = {"gpu": name, "power_limit": power, "pairs": PAIRS, "unroll": UNROLL, "unrolls": a.unrolls, "unit": "pair-steps/s",
           "transfer": "learner rank's own device copy"}
    out.update(pack_kernel(a.launches))
    modes = {False: "both_seats", True: "learner_seat"}
    peak = {m: 0 for m in modes.values()}
    for seat_only in (False, True, False, True):
        m = modes[seat_only]
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        r, nbytes = rate(seat_only, a)
        peak[m] = max(peak[m], torch.cuda.max_memory_allocated())
        out.setdefault("rate_" + m, []).append(round(r))
        out["bytes_per_rank_" + m] = nbytes
    for seat_only, m in modes.items():
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        for k, v in exposed(seat_only, a).items():
            out[k + "_" + m] = v
        peak[m] = max(peak[m], torch.cuda.max_memory_allocated())
        out["peak_torch_allocated_gb_" + m] = round(peak[m] / 1e9, 2)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
