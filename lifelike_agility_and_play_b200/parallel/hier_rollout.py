"""On-device actor loop of the environmental level (EPMC) producing training unrolls: the recurrent counterpart of `RolloutWorker`.

Per step, the training forward of the hierarchical policy kernel (llq_hier_policy_forward_rec) reads observation row t of the
trajectory slab in place, samples the code, and writes -log p and V into row t; the fused env step (record option 2) writes
a_t | r_t | done_t into row t and observation t+1 into row t+1.  The sampled code goes from the kernel's int32 output into the
code column.  The LSTM states ([N, 128]: code LSTM, then value LSTM) stay on the device, and each forward receives the done flags of
the step before it, so a finished episode's state is wiped exactly where the reference actor's mask is set.  Nothing synchronises with
the host inside an unroll.  Two `[T+1, N, 936]` slabs ping-pong (layout: parallel/trajectory.py, HCOL_*).
"""
from collections import namedtuple

import torch

from .trajectory import ACT_DIM, HCOL_CODE, HCOL_NEGLOGP, HCOL_VALUE, HIER_OBS_DIM, HIER_TRAJ_WIDTH

HierUnroll = namedtuple("HierUnroll", ["slab", "initial_state", "first_mask", "bootstrap_value"])


class HierRolloutWorker:
    def __init__(self, engine, policy, unroll, device, seed=0):
        """`engine`: a `_capi.VecEngine` on the CUDA library for the EPMC env (916-wide observations) with auto_reset=1;
        `policy`: a `policy_epmc.DeviceHierPolicy(..., train=True)` on the same device; `unroll`: T."""
        if engine.obs_dim != HIER_OBS_DIM:
            raise ValueError("HierRolloutWorker drives the EPMC env (916-wide observations)")
        if not getattr(policy, "train", False) or policy.strategic:
            raise ValueError("HierRolloutWorker needs an environmental-level DeviceHierPolicy created with train=True")
        self.eng, self.pol, self.T, self.n = engine, policy, int(unroll), engine.n
        self.dev = torch.device(device)
        z = lambda *shape, dtype=torch.float32: torch.zeros(shape, dtype=dtype, device=self.dev)
        self.bufs = [z(self.T + 1, self.n, HIER_TRAJ_WIDTH) for _ in range(2)]
        self.buf = self.bufs[0]
        self.state = z(self.n, policy.state_dim)
        self.done = z(self.n, dtype=torch.uint8)           # done flags of the last step: the mask of the next forward
        self.act, self.rew = z(self.n, ACT_DIM), z(self.n)
        self.codes = z(self.n, dtype=torch.int32)
        # per slab: the state and mask its first forward started from, V(observation T)
        self.init_states = [z(self.n, policy.state_dim) for _ in range(2)]
        self.first_masks = [z(self.n, dtype=torch.uint8) for _ in range(2)]
        self.boots = [z(self.n) for _ in range(2)]
        self._scratch_state, self._scratch_act = z(self.n, policy.state_dim), z(self.n, ACT_DIM)
        self.seed, self.calls = int(seed), 0
        self.row_gid0 = int(engine.cfg.global_env_offset)       # noise keyed by the global env id: equal seeds on two shards still differ
        engine.set_option("record", 2)
        self.stream = torch.cuda.Stream(self.dev)              # one stream orders the kernels and torch's copies (see RolloutWorker)
        self.stream.wait_stream(torch.cuda.current_stream(self.dev))
        self.t = 0

    def _slab_index(self, buf):
        return 0 if buf is self.bufs[0] else 1

    def start(self, first_obs):
        """`first_obs` [N, 916] (host or device): the observation `engine.reset()` returned.  Every env starts an episode: zero state,
        mask 1."""
        first = torch.as_tensor(first_obs, dtype=torch.float32).to(self.dev)
        self.stream.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(self.stream):
            self.buf[0, :, :HIER_OBS_DIM] = first
            self.state.zero_()
            self.done.fill_(1)
        self.t = 0

    def _forward(self, row, state, act, values_ptr, neglogp_ptr, codes_ptr, out_ld):
        self.pol.forward_rec(row.data_ptr(), HIER_TRAJ_WIDTH, self.n, self.done.data_ptr(), state.data_ptr(), act.data_ptr(), codes_ptr,
                             values_ptr, neglogp_ptr, out_ld, self.seed, self.calls, self.row_gid0, self.stream.cuda_stream)

    def step(self):
        """One training forward + one fused env step; fills record t.  Asynchronous on the worker's stream."""
        assert self.t < self.T, "unroll is full: call finish_unroll()"
        row, nxt = self.buf[self.t], self.buf[self.t + 1]
        fsz = 4
        with torch.cuda.stream(self.stream):
            if self.t == 0:
                i = self._slab_index(self.buf)
                self.init_states[i].copy_(self.state)
                self.first_masks[i].copy_(self.done)
            self._forward(row, self.state, self.act, row.data_ptr() + HCOL_VALUE * fsz, row.data_ptr() + HCOL_NEGLOGP * fsz,
                          self.codes.data_ptr(), HIER_TRAJ_WIDTH)
            row[:, HCOL_CODE].copy_(self.codes)
        self.eng.step_device(self.act.data_ptr(), nxt.data_ptr(), self.rew.data_ptr(), self.done.data_ptr(), obs_ld=HIER_TRAJ_WIDTH,
                             stream=self.stream.cuda_stream)
        self.calls += 1
        self.t += 1

    def finish_unroll(self):
        """`HierUnroll(slab [T, N, 936] view, initial_state [N, 128], first_mask [N] uint8, bootstrap_value [N])`, all valid until the
        end of the NEXT unroll; stepping continues in the other slab, whose row 0 receives observation T.

        bootstrap_value = V(observation T): the training forward on a scratch copy of the state with the current counter, so neither the
        worker's state nor its counter advances and the next unroll's first forward computes the same V bit for bit."""
        assert self.t == self.T
        done_buf = self.buf
        idx = self._slab_index(done_buf)
        self.buf = self.bufs[1 - idx]
        with torch.cuda.stream(self.stream):
            self._scratch_state.copy_(self.state)
            self._forward(done_buf[self.T], self._scratch_state, self._scratch_act, self.boots[idx].data_ptr(), None, None, 1)
            self.buf[0, :, :HIER_OBS_DIM] = done_buf[self.T, :, :HIER_OBS_DIM]
        self.t = 0
        return HierUnroll(done_buf[:self.T], self.init_states[idx], self.first_masks[idx], self.boots[idx])

    def wait(self):
        """Make torch's current stream wait for everything queued so far (call before reading a finished slab there)."""
        torch.cuda.current_stream(self.dev).wait_stream(self.stream)
