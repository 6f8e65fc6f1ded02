"""Reset-kernel time per policy step against the size of the prioritized clip table (PMC, 4096 envs).

    python tools/clip_table_bench.py [--envs 4096] [--steps 200] [--rounds 3] [--sizes 66,3902,8192,26814]

Every block of the reset kernel rebuilds the clip table (two sequential fp64 passes over all C clips on one thread) and every
resetting env scans the cdf linearly, after every step.  This script times the reset kernel with the engine's CUDA events
(`set_option("profile", 1)`, `timing()[1]`) over --steps steps per size, the sizes alternating inside each of --rounds rounds, and
prints the card name and power limit of the same run.  Clips are 300..420 synthetic frames; the default configuration steps with
zero actions, so episodes end (and auto-reset) at their natural rate.  Writes nothing."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sizes", default="66,3902,8192,26814")
    a = ap.parse_args()
    from lifelike_agility_and_play_b200 import _capi as capi
    from lifelike_agility_and_play_b200.mocap import synthetic_mocap
    from lifelike_agility_and_play_b200.model.compile_model import load_model_blob
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    lib, blob = capi.load_cuda_library(), load_model_blob()
    sizes = [int(s) for s in a.sizes.split(",")]
    engines = {}
    for C in sizes:
        e = capi.VecEngine(lib, a.envs, blob, synthetic_mocap(C, seed=C, min_frames=300, max_frames=420), seed=1, device=0)
        e.set_option("profile", 1)
        e.reset()
        engines[C] = e
    act = np.zeros((a.envs, 12), np.float32)
    res = {C: [] for C in sizes}
    for r in range(a.rounds):
        for C in sizes:
            e = engines[C]
            for _ in range(a.warmup):
                e.step(act)
            ms = []
            c0 = e.counters()[capi.CNT_EPISODES]
            for _ in range(a.steps):
                e.step(act)
                e.sync()
                ms.append(e.timing()[1])
            resets = int(e.counters()[capi.CNT_EPISODES] - c0)
            res[C].append(dict(reset_ms=float(np.mean(ms)), resets_per_step=resets / a.steps))
            print(json.dumps(dict(round=r, clips=C, reset_ms_mean=round(float(np.mean(ms)), 5), reset_ms_median=round(float(np.median(ms)), 5),
                                  resets_per_step=round(resets / a.steps, 1))), flush=True)
    for e in engines.values():
        e.close()
    print(json.dumps(dict(card=card, envs=a.envs, steps=a.steps, reset_ms={C: [round(x["reset_ms"], 5) for x in res[C]] for C in sizes})))


if __name__ == "__main__":
    main()
