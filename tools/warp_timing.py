"""Per-warp phase clocks of the step kernel (development aid; needs an H100).  Slots: 0 first CTA barrier, 1 dynamics, 2 collision +
limits, 3 impulse sums + back substitution, 8 row images (incl. pairing), 9 Delassus + warm start, 10 sweep, 11 second CTA barrier
(waiting for the CTA's heaviest warp); "rows+solver" is 3 + 8..11.  Prints the split and writes it as JSON to $OUT (default
warp_timing.json in the current directory).  Needs the -DLLQ16_TIMING build:
nvcc <NVCC_FLAGS of __graft_entry__> -DLLQ16_TIMING -o lifelike_agility_and_play_b200/csrc/variants/libllq_cuda_timing.so llq_cuda.cu"""
import ctypes as C, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from lifelike_agility_and_play_b200 import _capi as capi
from bench import synthetic_inputs, action_pool_np

path = os.path.join(os.path.dirname(capi.CUDA_LIB_PATH), "variants", "libllq_cuda_timing.so")
lib = capi.LlqLibrary(path)
n = int(os.environ.get("ENVS", 4096))
blob, mocap = synthetic_inputs()
dev = torch.device("cuda", 0)
stream = torch.cuda.Stream(device=dev); torch.cuda.set_stream(stream)
eng = capi.VecEngine(lib, n, blob, mocap, seed=1234, auto_reset=1)
eng.reset()
pool = torch.from_numpy(action_pool_np(n, 4, 5678)).to(dev)
obs = torch.empty((n, 207), device=dev); rew = torch.empty((n,), device=dev); done = torch.empty((n,), device=dev, dtype=torch.uint8)
res = {}
for label, warm in (("fresh", 3), ("steady", int(os.environ.get("WARM", 200)))):
    for i in range(warm):
        eng.step_device(pool[i % 4].data_ptr(), obs.data_ptr(), rew.data_ptr(), done.data_ptr(), stream=stream.cuda_stream)
    torch.cuda.synchronize()
    nw = n // 2
    buf = np.zeros((nw, 12), np.uint64)
    assert lib.lib.llq_debug_timing(buf.ctypes.data_as(C.c_void_p), nw) == 0
    t = buf.astype(np.float64)
    sums = t[:, 3].copy()                               # impulse sums + back substitution (the marks inside the solver restart the clock)
    t[:, 3] += t[:, 8] + t[:, 9] + t[:, 10] + t[:, 11]
    names = ["barrier", "dynamics", "collision+limits", "rows+solver", "epilogue(tail,emit)", "integrate", "rows", "total"]
    tot = t[:, 7]
    r = {"warps": nw, "total_mean": tot.mean(), "total_max": tot.max(), "total_p50": np.median(tot), "total_min": tot.min()}
    for j in (0, 1, 2, 3, 4, 5):
        r[names[j]] = {"mean": t[:, j].mean(), "max": t[:, j].max(), "share_of_total": t[:, j].sum() / tot.sum()}
    rows = buf[:, 6]
    two = ((rows >> np.uint64(16)) & np.uint64(0xFF)).astype(np.float64); twop = (rows >> np.uint64(24)).astype(np.float64); cm = ((rows >> np.uint64(8)) & np.uint64(0xFF)).astype(np.float64); lm = (rows & np.uint64(0xFF)).astype(np.float64)
    r["Cmax_sum_per_step"] = {"mean": cm.mean(), "max": cm.max()}; r["Lmax_sum_per_step"] = {"mean": lm.mean(), "max": lm.max()}
    r["substeps_with_an_env_over_16_rows"] = {"mean": two.mean(), "max": two.max(), "warps_with_any": float((two > 0).mean())}
    r["two_pass_substeps"] = {"mean": twop.mean(), "max": twop.max(), "warps_with_any": float((twop > 0).mean())}
    work = t[:, 1] + t[:, 2] + t[:, 3] + t[:, 5]
    r["work_without_barrier"] = {"mean": work.mean(), "max": work.max(), "p99": float(np.percentile(work, 99))}
    r["corr_solver_vs_rows"] = float(np.corrcoef(t[:, 3], cm + lm)[0, 1])
    # solver clocks by row load (Cmax + Lmax summed over the 10 sub-steps)
    load = cm + lm
    bins = [0, 20, 40, 60, 80, 100, 120, 160, 400]
    r["solver_clocks_by_load"] = [{"load": "%d-%d" % (bins[b], bins[b + 1]), "warps": int(((load >= bins[b]) & (load < bins[b + 1])).sum()),
                                   "solver_mean": float(t[(load >= bins[b]) & (load < bins[b + 1]), 3].mean()) if ((load >= bins[b]) & (load < bins[b + 1])).any() else None}
                                  for b in range(len(bins) - 1)]
    for j, nm in ((8, "row_images"), (9, "delassus+warm"), (10, "sweep"), (11, "barrier2")):
        r[nm] = {"mean": t[:, j].mean(), "max": t[:, j].max(), "share_of_total": t[:, j].sum() / tot.sum()}
    r["sums+backsub"] = {"mean": sums.mean(), "max": sums.max(), "share_of_total": sums.sum() / tot.sum()}
    heavy = load >= 100
    r["heavy_warps(load>=100)"] = {"n": int(heavy.sum()), **{nm: float(t[heavy, j].mean()) for j, nm in ((1, "dynamics(+barrier wait)"), (2, "collision"), (3, "solver"), (8, "row_images"), (9, "delassus+warm"), (10, "sweep"), (7, "total"))}} if heavy.any() else None
    r["dynamics_min"] = float(t[:, 1].min())
    cta = tot.reshape(-1, 8).max(1)
    r["cta_total"] = {"mean": cta.mean(), "max": cta.max(), "min": cta.min()}
    res[label] = r
    print(label, json.dumps(r, indent=1, default=float), flush=True)
json.dump(res, open(os.environ.get("OUT", "warp_timing.json"), "w"), indent=1, default=float)
