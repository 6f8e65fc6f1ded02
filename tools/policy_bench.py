"""A/B timing of policy-kernel variants on the GPU: csrc/libllq_policy.so + csrc/variants/libllq_policy_*.so, one subprocess per library
(the path is read at load time)."""
import glob
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def child():
    import numpy as np
    import torch
    from lifelike_agility_and_play_b200.policy import DevicePolicy
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_policy import random_weights
    n = int(os.environ.get("ROWS", 4096))
    pol = DevicePolicy(random_weights(1), device=0)
    obs = torch.randn((n, 207), device="cuda"); act = torch.zeros((n, 12), device="cuda")
    val = torch.zeros((n,), device="cuda"); nlp = torch.zeros((n,), device="cuda")
    st = torch.cuda.Stream(); res = {}
    with torch.cuda.stream(st):
        for name, fn in (("mean", lambda i: pol.forward(obs.data_ptr(), 207, n, act.data_ptr(), None, st.cuda_stream)),
                         ("full", lambda i: pol.forward_ex(obs.data_ptr(), 207, n, act.data_ptr(), None, val.data_ptr(), nlp.data_ptr(), 1, i, st.cuda_stream))):
            for i in range(20):
                fn(i)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            for i in range(200):
                fn(i)
            e1.record(st); st.synchronize()
            res[name] = e0.elapsed_time(e1) / 200
    print(json.dumps(res))


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "child":
        child(); sys.exit(0)
    csrc = os.path.join(ROOT, "lifelike_agility_and_play_b200", "csrc")
    libs = [os.path.join(csrc, "libllq_policy.so")] + sorted(glob.glob(os.path.join(csrc, "variants", "libllq_policy_*.so")))
    for lib in libs:
        e = dict(os.environ, LLQ_POLICY_LIB=lib)
        r = subprocess.run([sys.executable, __file__, "child"], env=e, capture_output=True, text=True)
        print(os.path.basename(lib), r.stdout.strip().splitlines()[-1] if r.stdout.strip() else r.stderr[-500:], flush=True)
