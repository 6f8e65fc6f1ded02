"""Dump every engine field after seeded random stepping, and compare two dumps bit for bit.

    python tools/dump_fields.py --lib lifelike_agility_and_play_b200/csrc/libllq_cuda.so --out head.npz
    python tools/dump_fields.py --compare parent.npz head.npz

Seven configurations (PMC with and without hurdle plates, EPMC elements 0-3 with the edge cylinders on 1-3, SEPMC with pushes) run
300 steps of seeded random actions with auto-reset on N = 4097 robots (SEPMC 4098): partial CTAs and the shadow lanes of the last
env are exercised.  The dump holds each step's reward and done, every field llq_get_field returns at the end, and the counters.
--compare exits non-zero on the first array that is not bit-identical: a refactor that claims bit-identical outputs must pass it.
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lifelike_agility_and_play_b200 import _capi as capi  # noqa: E402

PUSH = {'start_time': 0.5, 'interval_time': 1.0, 'duration_time': 0.2, 'horizontal_force': [0, 50], 'vertical_force': [0, 10]}
CONFIGS = ["pmc", "pmc_hurdles", "epmc0", "epmc1", "epmc2", "epmc3", "sepmc"]
FIELDS = [f for f in capi._FIELDS if f != capi.F_DECISION_MARGIN]     # the margin is an oracle-only field


def make_engine(lib, name, n):
    from lifelike_agility_and_play_b200.model.compile_model import load_model_blob
    from lifelike_agility_and_play_b200.mocap import synthetic_mocap, obstacle_table
    from lifelike_agility_and_play_b200.sim_envs.playground_env import INIT_STATE_RUN_0, epmc_engine_config
    from lifelike_agility_and_play_b200.sim_envs.chase_tag_game_env import sepmc_engine_config
    blob = load_model_blob()
    common = dict(seed=1234, auto_reset=1, device=0)
    if name.startswith("pmc"):
        mc = synthetic_mocap(8, seed=5, min_frames=400, max_frames=600)
        if name == "pmc_hurdles":
            mc.frames[:, 2] += 0.25 * np.exp(-((np.arange(len(mc.frames)) % 400 - 200) / 20.0) ** 2)      # periodic jumps
        eng = capi.VecEngine(lib, n, blob, mc, **common)
        if name == "pmc_hurdles":
            tab, offs = obstacle_table(mc)
            eng.load_obstacles(tab, offs, (0.025, 0.5, 0.2))
        return eng
    if name == "sepmc":
        cfg = sepmc_engine_config(50.0, 50.0, 0.5, 16, 150, {'friction_range': [0.4, 3.0], 'disturb_force_config': PUSH})
    else:
        element = int(name[-1])
        erc = {'element_id': element, 'friction_range': [0.4, 3.0], 'cmd_vary_freq_range': [25, 40], 'target_spd_range': [0.5, 3.0],
               'hole_config': {'min_gap_height': 0.25, 'max_gap_height': 0.25}, 'auxiliary_radius': 0.02 if element else None,
               'disturb_force_config': PUSH}
        cfg = epmc_engine_config(50.0, 50.0, 0.5, 16, 150, erc)
    cfg.update(common)
    eng = capi.VecEngine(lib, n, blob, None, **cfg)
    eng.set_init_state(INIT_STATE_RUN_0)
    return eng


def dump(lib_path, out, steps=300):
    lib = capi.LlqLibrary(lib_path)
    arrays = {}
    for name in CONFIGS:
        n = 4098 if name == "sepmc" else 4097
        eng = make_engine(lib, name, n)
        rng = np.random.default_rng(7)
        arrays[name + "/reset_obs"] = eng.reset()
        rew, done = np.empty((steps, n), np.float32), np.empty((steps, n), np.uint8)
        for t in range(steps):
            obs, rew[t], done[t] = eng.step((0.3 * rng.standard_normal((n, 12))).astype(np.float32))
        arrays.update({name + "/reward": rew, name + "/done": done, name + "/obs": obs, name + "/counters": eng.counters()})
        for f in FIELDS:
            if f in (capi.F_SAMPLE_PROB, capi.F_AVG_REWARD) and eng.n_clips == 0:
                continue
            arrays["%s/field%d" % (name, f)] = eng.get(f)
        print("%-12s episodes finished %d" % (name, int(eng.counters()[capi.CNT_EPISODES])))
        eng.close()
    np.savez_compressed(out, **arrays)


def compare(a, b):
    A, B = np.load(a), np.load(b)
    if sorted(A.files) != sorted(B.files):
        print("different arrays: %s" % sorted(set(A.files) ^ set(B.files)))
        return 1
    for k in A.files:
        a, b = A[k], B[k]
        if a.dtype != b.dtype or a.shape != b.shape or a.tobytes() != b.tobytes():      # bit for bit: NaN rows compare too
            print("DIFFERS: %s (%d of %d entries)" % (k, int(np.sum(a.view(np.uint8) != b.view(np.uint8))), a.size))
            return 1
    print("all %d arrays identical" % len(A.files))
    return 0


if __name__ == "__main__":
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--lib", default=capi.CUDA_LIB_PATH)
    ap.add_argument("--out")
    ap.add_argument("--compare", nargs=2, metavar=("A", "B"))
    a = ap.parse_args()
    if not a.compare and not a.out:
        ap.error("--out is required unless --compare is given")
    sys.exit(compare(*a.compare) if a.compare else dump(a.lib, a.out))
