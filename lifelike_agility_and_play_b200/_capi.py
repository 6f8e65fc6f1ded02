"""ctypes binding of the C-ABI declared in ``include/llq.h``.

This module is host plumbing only: it marshals numpy buffers (or raw device
pointers) into the ``llq_*`` entry points.  It never computes anything itself
and has no CPU fallback -- :func:`load_cuda_library` raises if the CUDA engine
has not been built.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

STATE_DIM, ACTION_DIM, PROP_DIM, OBS_DIM, MOCAP_FRAME = 37, 12, 33, 207, 19

LLQ_IO_HOST, LLQ_IO_DEVICE, LLQ_IO_PINNED = 0, 1, 2
(F_STATE, F_CLIP, F_TIME, F_REWARD_SUM, F_EPISODE_STEPS, F_WARMSTART, F_OBS, F_KIN_STATE, F_SAMPLE_PROB,
 F_AVG_REWARD, F_EPISODE_ID, F_FOOT_POS, F_DECISION_MARGIN, F_AUX, F_OB_ID, F_BOXES, F_NBOX) = range(17)
MAX_BOXES = 36
ENV_PMC, ENV_EPMC, ENV_SEPMC, OBS_DIM_EPMC, OBS_DIM_SEPMC, AUX_DIM = 0, 1, 2, 916, 965, 18

# field id -> (dtype, per-env width or None for per-clip tables)
_FIELDS = {
    F_STATE: (np.float32, STATE_DIM), F_CLIP: (np.int32, 1), F_TIME: (np.float64, 1),
    F_REWARD_SUM: (np.float32, 1), F_EPISODE_STEPS: (np.int32, 1), F_WARMSTART: (np.float32, 32),
    F_OBS: (np.float32, OBS_DIM), F_KIN_STATE: (np.float32, STATE_DIM), F_SAMPLE_PROB: (np.float64, None),
    F_AVG_REWARD: (np.float64, None), F_EPISODE_ID: (np.int64, 1), F_FOOT_POS: (np.float32, 12),
    F_DECISION_MARGIN: (np.float32, 1), F_AUX: (np.float64, AUX_DIM), F_OB_ID: (np.int32, 1),
    F_BOXES: (np.float32, 36 * 6), F_NBOX: (np.int32, 1),
}


class LlqConfig(C.Structure):
    """Mirror of ``struct llq_config`` (include/llq.h) -- field order and types must match."""
    _fields_ = [
        ("struct_size", C.c_int32), ("n_envs", C.c_int32), ("device", C.c_int32), ("substeps", C.c_int32),
        ("solver_iters", C.c_int32), ("auto_reset", C.c_int32), ("num_threads", C.c_int32), ("element_id", C.c_int32),
        ("global_env_offset", C.c_int64), ("seed", C.c_uint64),
        ("sim_dt", C.c_double), ("kp", C.c_double), ("kd", C.c_double), ("max_tau", C.c_double),
        ("gravity_z", C.c_double), ("ground_friction", C.c_double), ("foot_friction", C.c_double),
        ("contact_erp", C.c_double), ("joint_erp", C.c_double), ("linear_slop", C.c_double), ("warmstart", C.c_double),
        ("contact_breaking", C.c_double), ("lin_damping", C.c_double), ("ang_damping", C.c_double),
        ("max_coord_vel", C.c_double), ("max_applied_impulse", C.c_double),
        ("w_joint_pos", C.c_double), ("w_joint_vel", C.c_double), ("w_end_effector", C.c_double),
        ("w_root_pose", C.c_double), ("w_root_vel", C.c_double),
        ("prioritized_sample_factor", C.c_double), ("policy_dt", C.c_double),
        ("env_kind", C.c_int32), ("max_steps", C.c_int32), ("cmd_freq_lo", C.c_int32), ("cmd_freq_hi", C.c_int32),
        ("push_start_count", C.c_int32), ("push_interval_steps", C.c_int32), ("push_duration_steps", C.c_int32),
        ("push_enabled", C.c_int32),
        ("friction_lo", C.c_double), ("friction_hi", C.c_double), ("push_h_lo", C.c_double), ("push_h_hi", C.c_double),
        ("push_v_lo", C.c_double), ("push_v_hi", C.c_double), ("target_spd_lo", C.c_double), ("target_spd_hi", C.c_double),
        ("wall_width_lo", C.c_double), ("wall_width_hi", C.c_double), ("wall_gap_lo", C.c_double), ("wall_gap_hi", C.c_double),
        ("hole_gap_lo", C.c_double), ("hole_gap_hi", C.c_double),
        ("knee_contacts", C.c_int32), ("reserved1", C.c_int32), ("link_friction", C.c_double), ("auxiliary_radius", C.c_double),
    ]


class LlqError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("llq error %d: %s" % (code, msg))
        self.code = code


_EXPORTS = ["llq_abi_version", "llq_default_config", "llq_create", "llq_destroy", "llq_load_model", "llq_load_mocap",
            "llq_reset", "llq_reset_to", "llq_step", "llq_step_ex", "llq_get_field", "llq_set_field",
            "llq_get_counters", "llq_set_option", "llq_get_timing", "llq_obs_dim", "llq_set_init_state", "llq_host_alloc", "llq_host_free", "llq_load_obstacles", "llq_sync", "llq_last_error"]


class LlqLibrary:
    """A loaded implementation of include/llq.h (CUDA engine or CPU oracle)."""

    def __init__(self, path):
        if not os.path.exists(path):
            raise FileNotFoundError(path)
        self.path = path
        self.lib = C.CDLL(path, mode=C.RTLD_GLOBAL if False else C.RTLD_LOCAL)
        for name in _EXPORTS:
            if not hasattr(self.lib, name):
                raise AttributeError("%s does not export %s" % (path, name))
        L = self.lib
        vp = C.c_void_p
        L.llq_abi_version.argtypes = [C.POINTER(C.c_int)]
        L.llq_default_config.argtypes = [C.POINTER(LlqConfig)]
        L.llq_create.argtypes = [C.POINTER(LlqConfig), C.POINTER(vp)]
        L.llq_destroy.argtypes = [vp]
        L.llq_load_model.argtypes = [vp, vp, C.c_int64]
        L.llq_load_mocap.argtypes = [vp, vp, vp, C.c_int32, C.c_double]
        L.llq_reset.argtypes = [vp, vp, vp]
        L.llq_reset_to.argtypes = [vp, vp, vp, vp, vp]
        L.llq_step.argtypes = [vp, vp, vp, vp, vp]
        L.llq_step_ex.argtypes = [vp, vp, vp, C.c_int64, vp, vp, C.c_int, vp]
        L.llq_get_field.argtypes = [vp, C.c_int, vp]
        L.llq_set_field.argtypes = [vp, C.c_int, vp]
        L.llq_get_counters.argtypes = [vp, vp, C.c_int32]
        L.llq_sync.argtypes = [vp]
        L.llq_load_obstacles.argtypes = [vp, vp, vp, C.c_int32, C.c_double, C.c_double, C.c_double]
        L.llq_host_alloc.argtypes = [C.POINTER(vp), C.c_int64]
        L.llq_host_free.argtypes = [vp]
        L.llq_obs_dim.argtypes = [vp]
        L.llq_set_init_state.argtypes = [vp, vp]
        L.llq_set_option.argtypes = [vp, C.c_char_p, C.c_double]
        L.llq_get_timing.argtypes = [vp, vp, C.c_int32]
        L.llq_last_error.restype = C.c_char_p
        for name in _EXPORTS[:-1]:
            getattr(L, name).restype = C.c_int
        is_cuda = C.c_int(0)
        self.abi = L.llq_abi_version(C.byref(is_cuda))
        self.is_cuda = bool(is_cuda.value)

    def check(self, rc):
        if rc != 0:
            raise LlqError(rc, (self.lib.llq_last_error() or b"").decode())

    def default_config(self) -> LlqConfig:
        cfg = LlqConfig()
        self.check(self.lib.llq_default_config(C.byref(cfg)))
        return cfg


_HERE = os.path.dirname(os.path.abspath(__file__))
CUDA_LIB_PATH = os.environ.get("LLQ_CUDA_LIB", os.path.join(_HERE, "csrc", "libllq_cuda.so"))   # override: profiling variants only
_cuda_lib = None


def load_cuda_library() -> LlqLibrary:
    """Load the sm_90a engine.  No fallback: a missing build is a hard error."""
    global _cuda_lib
    if _cuda_lib is None:
        if not os.path.exists(CUDA_LIB_PATH):
            raise RuntimeError("CUDA engine %s is not built; run `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(there is no CPU fallback on the product path)" % CUDA_LIB_PATH)
        lib = LlqLibrary(CUDA_LIB_PATH)
        if not lib.is_cuda:
            raise RuntimeError("%s is not the CUDA engine" % CUDA_LIB_PATH)
        _cuda_lib = lib
    return _cuda_lib


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class _PinnedBlock:
    """Page-locked host block (llq_host_alloc).  numpy views made with ``np.asarray(block)`` keep the block alive through
    their ``base``; the memory is returned to the driver only when the last view is gone, not when the engine closes."""

    def __init__(self, lib, shape, dtype):
        self._lib, self.shape, self.dtype = lib, tuple(int(x) for x in shape), np.dtype(dtype)
        self.nbytes = int(np.prod(self.shape)) * self.dtype.itemsize
        p = C.c_void_p()
        lib.check(lib.lib.llq_host_alloc(C.byref(p), self.nbytes))
        self._p = p

    @property
    def __array_interface__(self):
        return {"shape": self.shape, "typestr": self.dtype.str, "data": (self._p.value, False), "version": 3}

    def __del__(self):
        try:
            if self._p:
                self._lib.lib.llq_host_free(self._p)
                self._p = None
        except Exception:
            pass


class VecEngine:
    """N lock-step environments behind one ``llq_handle``.

    Array arguments are numpy (host) arrays; ``step_device`` takes raw device
    pointers (e.g. ``torch.Tensor.data_ptr()``) for the zero-copy path.
    """

    def __init__(self, lib: LlqLibrary, n_envs, model_blob, mocap, **overrides):
        self.lib = lib
        cfg = lib.default_config()
        cfg.n_envs = int(n_envs)
        for k, v in overrides.items():
            if not hasattr(cfg, k):
                raise TypeError("unknown llq_config field %r" % k)
            setattr(cfg, k, v)
        self.cfg = cfg
        self.n = int(n_envs)
        self._h = C.c_void_p()
        lib.check(lib.lib.llq_create(C.byref(cfg), C.byref(self._h)))
        blob = np.ascontiguousarray(model_blob, dtype=np.float64)
        lib.check(lib.lib.llq_load_model(self._h, _ptr(blob), blob.size))
        self.n_clips = 0
        if mocap is not None:
            frames = np.ascontiguousarray(mocap.frames, dtype=np.float64)
            offs = np.ascontiguousarray(mocap.offsets, dtype=np.int32)
            self.n_clips = offs.size - 1
            lib.check(lib.lib.llq_load_mocap(self._h, _ptr(frames), _ptr(offs), self.n_clips, float(mocap.frame_dt)))
        self.obs_dim = int(lib.lib.llq_obs_dim(self._h))
        if self.obs_dim <= 0:
            lib.check(self.obs_dim)

    def load_obstacles(self, table, offsets, half_extents):
        """PMC hurdle plates (mocap.obstacle_table) -- set_obstacle=True of the reference (PLE:173-193)."""
        t = np.ascontiguousarray(table, dtype=np.float64).reshape(-1, 4)
        o = np.ascontiguousarray(offsets, dtype=np.int32)
        hx, hy, hz = [float(v) for v in half_extents]
        self.lib.check(self.lib.lib.llq_load_obstacles(self._h, _ptr(t) if t.size else None, _ptr(o), o.size - 1, hx, hy, hz))

    def set_init_state(self, state37):
        st = np.ascontiguousarray(state37, dtype=np.float64)
        assert st.shape == (STATE_DIM,)
        self.lib.check(self.lib.lib.llq_set_init_state(self._h, _ptr(st)))

    # -- lifecycle
    def close(self):
        if self._h:
            self.lib.lib.llq_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- stepping
    def _mask(self, mask):
        return None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)

    def reset(self, mask=None):
        obs = np.empty((self.n, self.obs_dim), np.float32)
        m = self._mask(mask)
        self.lib.check(self.lib.lib.llq_reset(self._h, _ptr(m), _ptr(obs)))
        return obs

    def reset_to(self, clip, time, mask=None):
        obs = np.empty((self.n, self.obs_dim), np.float32)
        clip = np.ascontiguousarray(np.broadcast_to(clip, (self.n,)), dtype=np.int32)
        time = np.ascontiguousarray(np.broadcast_to(time, (self.n,)), dtype=np.float64)
        m = self._mask(mask)
        self.lib.check(self.lib.lib.llq_reset_to(self._h, _ptr(m), _ptr(clip), _ptr(time), _ptr(obs)))
        return obs

    def step(self, actions, out=None):
        a = np.ascontiguousarray(actions, dtype=np.float32)
        if a.shape != (self.n, ACTION_DIM):
            raise ValueError("actions must have shape (%d, %d)" % (self.n, ACTION_DIM))
        if out is None:
            obs = np.empty((self.n, self.obs_dim), np.float32)
            rew = np.empty((self.n,), np.float32)
            done = np.empty((self.n,), np.uint8)
        else:
            obs, rew, done = out
            for arr, shape, dt in ((obs, (self.n, self.obs_dim), np.float32), (rew, (self.n,), np.float32), (done, (self.n,), np.uint8)):
                if not (isinstance(arr, np.ndarray) and arr.shape == shape and arr.dtype == dt and arr.flags.c_contiguous and arr.flags.writeable):
                    raise ValueError("out arrays must be writeable C-contiguous %s arrays of shape %s" % (np.dtype(dt).name, shape))
        self.lib.check(self.lib.lib.llq_step(self._h, _ptr(a), _ptr(obs), _ptr(rew), _ptr(done)))
        return obs, rew, done

    # -- page-locked I/O (LLQ_IO_PINNED): no staging memcpy on either side
    def pinned_array(self, shape, dtype):
        """numpy array over page-locked host memory; the block is freed when the last view of it is released (it may outlive
        the engine -- TLeague queues observation objects for another thread, distill_actor.py:267-270)."""
        return np.asarray(_PinnedBlock(self.lib, shape, dtype))

    def pinned_io(self):
        """(actions, obs, reward, done) page-locked buffers for step_pinned."""
        return (self.pinned_array((self.n, ACTION_DIM), np.float32), self.pinned_array((self.n, self.obs_dim), np.float32),
                self.pinned_array((self.n,), np.float32), self.pinned_array((self.n,), np.uint8))

    def step_pinned(self, actions, obs, reward, done):
        """Like step(), but the arrays must be page-locked (pinned_io()); results land in obs / reward / done.  obs may be None:
        the observation then stays on the device (llq_get_field / an on-device policy reads it there) and only reward / done
        travel back."""
        self.lib.check(self.lib.lib.llq_step_ex(self._h, _ptr(actions), _ptr(obs), self.obs_dim, _ptr(reward), _ptr(done),
                                                 LLQ_IO_PINNED, None))
        return obs, reward, done

    def step_device(self, actions_ptr, obs_ptr, reward_ptr, done_ptr, obs_ld=None, stream=None):
        obs_ld = self.obs_dim if obs_ld is None else obs_ld
        self.lib.check(self.lib.lib.llq_step_ex(self._h, C.c_void_p(actions_ptr), C.c_void_p(obs_ptr), obs_ld,
                                                 C.c_void_p(reward_ptr), C.c_void_p(done_ptr), LLQ_IO_DEVICE,
                                                 C.c_void_p(stream) if stream else None))

    def sync(self):
        self.lib.check(self.lib.lib.llq_sync(self._h))

    # -- state access
    def get(self, field):
        dt, w = _FIELDS[field]
        if field == F_OBS:
            w = self.obs_dim
        arr = np.empty((self.n_clips,) if w is None else ((self.n,) if w == 1 else (self.n, w)), dt)
        self.lib.check(self.lib.lib.llq_get_field(self._h, field, _ptr(arr)))
        return arr

    def set(self, field, value):
        dt, w = _FIELDS[field]
        if field == F_OBS:
            w = self.obs_dim
        shape = (self.n_clips,) if w is None else ((self.n,) if w == 1 else (self.n, w))
        arr = np.ascontiguousarray(np.broadcast_to(np.asarray(value, dtype=dt), shape), dtype=dt)
        self.lib.check(self.lib.lib.llq_set_field(self._h, field, _ptr(arr)))

    def set_option(self, name, value):
        self.lib.check(self.lib.lib.llq_set_option(self._h, name.encode(), float(value)))

    def timing(self):
        """(step kernel ms, reset kernel ms) of the last step; needs set_option("profile", 1)."""
        out = np.zeros(2, np.float64)
        self.lib.check(self.lib.lib.llq_get_timing(self._h, _ptr(out), 2))
        return float(out[0]), float(out[1])

    def counters(self):
        out = np.zeros(8, np.int64)
        self.lib.check(self.lib.lib.llq_get_counters(self._h, _ptr(out), 8))
        return out
