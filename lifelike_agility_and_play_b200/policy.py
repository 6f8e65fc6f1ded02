"""Host-side reference forward of the PMC policy (SURVEY row f2; networks/legged_robot/pmc_net/pmc_net.py:33-58,99-178 with
policy_config of test_scripts/primitive_level/test_primitive_level_env.py:39-57): observation normalisation with the stored
running mean / std clipped to +-5 (layers.py:55, pmc_net.py:130-135), VQ encoder 207 -> 256 -> 256 -> 32 with a 32 x 256
codebook (argmin of the squared distance, pmc_net.py:157-171), low-level controller (prop 135 -> 64) + (z 32 -> 32) -> 256 ->
256 -> 12, ReLU activations; the deterministic action is the mean (agent.step(argmax=True)).

`weights` is the list of 28 arrays of a shipped ``*.model`` file in its stored order:
0-3 prop / future running mean, std | 4-9 value head | 10-15 encoder | 16 codebook | 17-20 bottleneck embeds | 21-26 decoder | 27 logstd
"""
import numpy as np


class PmcPolicy:
    def __init__(self, weights):
        w = [np.asarray(x, dtype=np.float32) for x in weights]
        assert len(w) == 28 and w[10].shape == (207, 256) and w[16].shape == (32, 256) and w[25].shape == (256, 12)
        self.prop_mean, self.prop_std, self.fut_mean, self.fut_std = w[0][0], w[1][0], w[2][0], w[3][0]
        self.enc = [(w[10], w[11]), (w[12], w[13]), (w[14], w[15])]
        self.codebook = w[16]
        self.prop_embed, self.z_embed = (w[17], w[18]), (w[19], w[20])
        self.dec = [(w[21], w[22]), (w[23], w[24]), (w[25], w[26])]
        self.logstd = w[27]
        self.vf = [(w[4], w[5]), (w[6], w[7]), (w[8], w[9])]

    def normalise(self, obs):
        p = np.clip((obs[:, :135] - self.prop_mean) / (self.prop_std + 1e-8), -5.0, 5.0)
        f = np.clip((obs[:, 135:207] - self.fut_mean) / (self.fut_std + 1e-8), -5.0, 5.0)
        return p, f

    def encode(self, p, f):
        x = np.concatenate([p, f], axis=1)
        x = np.maximum(x @ self.enc[0][0] + self.enc[0][1], 0.0)
        x = np.maximum(x @ self.enc[1][0] + self.enc[1][1], 0.0)
        z = x @ self.enc[2][0] + self.enc[2][1]
        d = (z ** 2).sum(1, keepdims=True) - 2.0 * z @ self.codebook + (self.codebook ** 2).sum(0, keepdims=True)
        idx = np.argmax(-d, axis=1)
        return z, idx

    def act(self, obs, return_code=False):
        obs = np.asarray(obs, dtype=np.float32)
        p, f = self.normalise(obs)
        z, idx = self.encode(p, f)
        zq = self.codebook.T[idx]
        pe = np.maximum(p @ self.prop_embed[0] + self.prop_embed[1], 0.0)
        ze = np.maximum(zq @ self.z_embed[0] + self.z_embed[1], 0.0)
        x = np.concatenate([pe, ze], axis=1)
        x = np.maximum(x @ self.dec[0][0] + self.dec[0][1], 0.0)
        x = np.maximum(x @ self.dec[1][0] + self.dec[1][1], 0.0)
        a = x @ self.dec[2][0] + self.dec[2][1]
        return (a, idx) if return_code else a

    def value(self, obs):
        """V(obs): 207 -> 256 -> 256 -> 1 with tanh on the normalised observation (pmc_net.py:139-144)."""
        p, f = self.normalise(np.asarray(obs, dtype=np.float32))
        x = np.concatenate([p, f], axis=1)
        x = np.tanh(x @ self.vf[0][0] + self.vf[0][1])
        x = np.tanh(x @ self.vf[1][0] + self.vf[1][1])
        return (x @ self.vf[2][0] + self.vf[2][1])[:, 0]

    def neglogp(self, action, mean):
        """-log p(action) under the diagonal Gaussian head (mean, exp(logstd)) (pmc_net.py:107-113)."""
        ls = self.logstd.reshape(-1)
        e = (action - mean) / np.exp(ls)
        return 0.5 * (e * e).sum(1) + ls.sum() + 0.5 * e.shape[1] * np.log(2.0 * np.pi)


# ------------------------------------------------------------------------------------------------------------------------
# device side (include/llq_policy.h, csrc/llq_policy.cu)
import ctypes as _C
import os as _os

POLICY_LIB_PATH = _os.path.join(_os.path.dirname(_os.path.abspath(__file__)), "csrc", "libllq_policy.so")
POLICY_EXPORTS = ["llq_policy_create", "llq_policy_destroy", "llq_policy_forward", "llq_policy_forward_ex", "llq_policy_forward_rec",
                  "llq_policy_last_error", "llq_hier_policy_create", "llq_hier_policy_destroy", "llq_hier_policy_forward",
                  "llq_hier_policy_last_error", "llq_hier_policy_create_train", "llq_hier_policy_forward_rec",
                  "llq_hier_policy_create_pool", "llq_hier_policy_set_pool_probs", "llq_hier_policy_forward_pool",
                  "llq_policy_set_weights", "llq_hier_policy_set_weights", "llq_hier_policy_set_pool_model", "llq_seat_pack",
                  "llq_seat_pack_last_error"]
N_WEIGHTS = 358647
# array shapes of a shipped primitive-level *.model file, in their stored order (the 28 arrays of include/llq_policy.h)
PMC_SHAPES = [(1, 135), (1, 135), (1, 72), (1, 72), (207, 256), (256,), (256, 256), (256,), (256, 1), (1,), (207, 256), (256,), (256, 256),
              (256,), (256, 32), (32,), (32, 256), (135, 64), (64,), (32, 32), (32,), (96, 256), (256,), (256, 256), (256,), (256, 12), (12,),
              (1, 12)]


def check_arrays(weights, shapes, what):
    """ValueError unless `weights` is a list of len(shapes) arrays of these shapes (unit axes aside: (1, 135) and (135,) agree)."""
    if isinstance(weights, np.ndarray) or not hasattr(weights, "__len__") or len(weights) != len(shapes):
        raise ValueError("expected the %d arrays of %s, got %s" % (len(shapes), what, len(weights) if hasattr(weights, "__len__") else type(weights)))
    for i, (a, want) in enumerate(zip(weights, shapes)):
        got = np.shape(a)
        if tuple(d for d in got if d != 1) != tuple(d for d in want if d != 1):
            raise ValueError("array %d of %s has shape %s, expected %s" % (i, what, got, tuple(want)))


def check_device_blob(t, n, device):
    """ValueError unless `t` is a contiguous 1-D float32 CUDA tensor of `n` floats on cuda:`device`."""
    import torch
    if not (isinstance(t, torch.Tensor) and t.is_cuda):
        raise ValueError("a device weight blob must be a CUDA tensor")
    if t.dtype != torch.float32 or t.dim() != 1 or not t.is_contiguous() or t.numel() != n:
        raise ValueError("a device weight blob must be a contiguous 1-D float32 tensor of %d floats (got %s %s)" % (n, t.dtype, tuple(t.shape)))
    if t.device.index != device:
        raise ValueError("the weight blob is on %s, the handle on cuda:%d" % (t.device, device))


def is_tensor(x):
    return type(x).__module__.startswith("torch") and hasattr(x, "data_ptr")


def keep_for_stream(t, stream, device):
    """The caching allocator must not hand `t`'s memory out again before the work queued on `stream` (a cudaStream_t, None / 0 = the
    default stream) has read it."""
    import torch
    s = torch.cuda.ExternalStream(stream, device=device) if stream else torch.cuda.default_stream(device)
    t.record_stream(s)


def pack_weights(weights):
    """The blob llq_policy_create() expects: the 28 arrays of a model file in their stored order (include/llq_policy.h)."""
    blob = np.concatenate([np.asarray(w, dtype=np.float32).reshape(-1) for w in weights])
    assert len(weights) == 28 and blob.size == N_WEIGHTS
    return np.ascontiguousarray(blob)


class DevicePolicy:
    """ctypes binding of the CUDA policy forward.  No CPU fallback: construction fails without the library or a GPU."""

    def __init__(self, weights, device=0):
        if not _os.path.exists(POLICY_LIB_PATH):
            raise OSError("%s is missing: run `python __graft_entry__.py` (nvcc) first" % POLICY_LIB_PATH)
        self._lib = _C.CDLL(_os.environ.get("LLQ_POLICY_LIB", POLICY_LIB_PATH))     # the override is for tools/policy_bench.py variants
        L = self._lib
        L.llq_policy_create.argtypes = [_C.c_void_p, _C.c_int64, _C.c_int32, _C.POINTER(_C.c_void_p)]
        L.llq_policy_forward.argtypes = [_C.c_void_p, _C.c_void_p, _C.c_int64, _C.c_int32, _C.c_void_p, _C.c_void_p, _C.c_void_p]
        L.llq_policy_forward_ex.argtypes = [_C.c_void_p, _C.c_void_p, _C.c_int64, _C.c_int32, _C.c_void_p, _C.c_void_p, _C.c_void_p,
                                            _C.c_void_p, _C.c_uint64, _C.c_uint64, _C.c_void_p]
        L.llq_policy_forward_rec.argtypes = [_C.c_void_p, _C.c_void_p, _C.c_int64, _C.c_int32, _C.c_void_p, _C.c_void_p, _C.c_void_p,
                                             _C.c_void_p, _C.c_int64, _C.c_uint64, _C.c_uint64, _C.c_int64, _C.c_void_p]
        L.llq_policy_destroy.argtypes = [_C.c_void_p]
        L.llq_policy_last_error.restype = _C.c_char_p
        blob = pack_weights(weights)
        self.device = int(device)
        self._h = _C.c_void_p()
        rc = L.llq_policy_create(blob.ctypes.data_as(_C.c_void_p), blob.size, device, _C.byref(self._h))
        if rc != 0:
            raise RuntimeError("llq_policy_create failed (%d): %s" % (rc, (L.llq_policy_last_error() or b"").decode()))

    def forward(self, obs_ptr, obs_ld, n, actions_ptr, codes_ptr=None, stream=None):
        """Device pointers (ints); asynchronous on `stream`."""
        rc = self._lib.llq_policy_forward(self._h, obs_ptr, obs_ld, n, actions_ptr, codes_ptr, stream)
        if rc != 0:
            raise RuntimeError("llq_policy_forward failed (%d): %s" % (rc, (self._lib.llq_policy_last_error() or b"").decode()))

    def forward_ex(self, obs_ptr, obs_ld, n, actions_ptr, codes_ptr=None, values_ptr=None, neglogp_ptr=None, seed=0, counter=0,
                   stream=None):
        """Rollout step: optional V(obs) and, when `neglogp_ptr` is given, sampled actions with their -log p."""
        rc = self._lib.llq_policy_forward_ex(self._h, obs_ptr, obs_ld, n, actions_ptr, codes_ptr, values_ptr, neglogp_ptr,
                                             seed, counter, stream)
        if rc != 0:
            raise RuntimeError("llq_policy_forward_ex failed (%d): %s" % (rc, (self._lib.llq_policy_last_error() or b"").decode()))

    def forward_rec(self, obs_ptr, obs_ld, n, actions_ptr, values_ptr, neglogp_ptr, out_ld, seed=0, counter=0, row_gid0=0, stream=None):
        """Rollout step writing V(obs) / -log p with row stride `out_ld` (straight into the columns of a trajectory slab row);
        the sampling noise is keyed by the global row `row_gid0 + i`."""
        rc = self._lib.llq_policy_forward_rec(self._h, obs_ptr, obs_ld, n, actions_ptr, None, values_ptr, neglogp_ptr, out_ld,
                                              seed, counter, row_gid0, stream)
        if rc != 0:
            raise RuntimeError("llq_policy_forward_rec failed (%d): %s" % (rc, (self._lib.llq_policy_last_error() or b"").decode()))

    def set_weights(self, weights, stream=None):
        """The learner's new weights (include/llq_policy.h, llq_policy_set_weights), asynchronous on `stream` (a cudaStream_t, None = the
        default stream): forwards queued there before see the old weights, forwards queued after it the new ones.  `weights`: the 28
        arrays of a model file (the host list may be reused as soon as this returns), or a flat float32 CUDA tensor of N_WEIGHTS floats
        on the handle's device (pack_weights' layout)."""
        if is_tensor(weights):
            check_device_blob(weights, N_WEIGHTS, self.device)
            ptr, on_device = weights.data_ptr(), 1
        else:
            check_arrays(weights, PMC_SHAPES, "a primitive-level model")
            blob = pack_weights(weights)
            ptr, on_device = blob.ctypes.data, 0
        L = self._lib
        L.llq_policy_set_weights.argtypes = [_C.c_void_p, _C.c_void_p, _C.c_int64, _C.c_int32, _C.c_void_p]
        rc = L.llq_policy_set_weights(self._h, ptr, N_WEIGHTS, on_device, stream)
        if rc != 0:
            raise RuntimeError("llq_policy_set_weights failed (%d): %s" % (rc, (L.llq_policy_last_error() or b"").decode()))
        if on_device:
            keep_for_stream(weights, stream, self.device)

    def close(self):
        if getattr(self, "_h", None):
            self._lib.llq_policy_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
