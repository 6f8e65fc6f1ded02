"""On-device actor loop of the strategic level (SEPMC, the chase-tag game) producing training unrolls against a frozen opponent.

Robot 2p of each env-pair p is the learning agent (seat 0) and robot 2p+1 its frozen opponent (seat 1), as a TLeague actor plays the
learning model against one from the pool; the game's termination reads robot 0's fall and contacts only.  Per step:
  * the strategic training forward (llq_hier_policy_forward_rec_strategic) on the seat-0 rows of slab row t, read in place with a row
    stride of two records, samples the heading and writes its raw value, -log p and V straight into those records; its noise is keyed by
    the global pair id;
  * the opponent's deterministic forward (llq_hier_policy_forward) on the seat-1 rows; against an opponent pool
    (policy_epmc.DeviceOpponentPool, llq_hier_policy_forward_pool) every pair whose game starts first draws its opponent's model from the
    pool's probabilities, and the model index goes into the opponent column of the pair's seat-0 record;
  * device-side copies interleave both seats' actions into the engine's [2P, 12] action array and put both seats' codes into the code
    column; the fused env step (record option 2) writes a_t | r_t | done_t into row t and observation t+1 into row t+1; the pair's done
    flags (equal on both rows) are copied into each seat's contiguous mask for the next forwards.
The LSTM states ([P, 192] for seat 0: heading, code and value LSTM; [P, 128] for seat 1) and, with a pool, each pair's model index stay on
the device.  Nothing synchronises with
the host inside an unroll.  Two `[T+1, 2P, 984]` slabs ping-pong (layout: parallel/trajectory.py, SCOL_*).
"""
from collections import namedtuple

import torch

from ..policy_epmc import DeviceOpponentPool
from .trajectory import ACT_DIM, SCOL_CODE, SCOL_HEADING, SCOL_NEGLOGP, SCOL_OPPONENT, SCOL_VALUE, SEPMC_OBS_DIM, SEPMC_TRAJ_WIDTH

SepmcUnroll = namedtuple("SepmcUnroll", ["slab", "initial_state", "first_mask", "bootstrap_value"])
_FSZ = 4


class SepmcRolloutWorker:
    def __init__(self, engine, policy, opponent, unroll, device, seed=0):
        """`engine`: a `_capi.VecEngine` on the CUDA library for the SEPMC env (965-wide observations, 2P robots) with auto_reset=1 and an
        even `global_env_offset`; `policy`: a `policy_epmc.DeviceSepmcTrainPolicy` (the learner's weights); `opponent`: a deterministic
        strategic-level `policy_epmc.DeviceHierPolicy` (its own weights), or a `policy_epmc.DeviceOpponentPool` with max_rows >= P (each
        pair draws its opponent's model at every game start; see `set_opponent_probs`), all on the engine's device; `unroll`: T."""
        if engine.obs_dim != SEPMC_OBS_DIM:
            raise ValueError("SepmcRolloutWorker drives the SEPMC env (965-wide observations)")
        if not int(engine.cfg.auto_reset):
            raise ValueError("SepmcRolloutWorker needs an engine with auto_reset=1")
        if int(engine.cfg.global_env_offset) % 2:
            raise ValueError("global_env_offset must be even: robots 2p and 2p+1 form a pair")
        if getattr(policy, "state_dim", None) != 192 or not getattr(policy, "train", False):
            raise ValueError("SepmcRolloutWorker needs a DeviceSepmcTrainPolicy")
        if not getattr(opponent, "strategic", False) or getattr(opponent, "train", True):
            raise ValueError("the opponent must be a deterministic strategic-level DeviceHierPolicy or a DeviceOpponentPool")
        self.pool = isinstance(opponent, DeviceOpponentPool)
        if self.pool and opponent.max_rows < engine.n // 2:
            raise ValueError("the opponent pool's max_rows is below the number of pairs")
        self.eng, self.pol, self.opp, self.T = engine, policy, opponent, int(unroll)
        self.n, self.P = engine.n, engine.n // 2
        self.dev = torch.device(device)
        z = lambda *shape, dtype=torch.float32: torch.zeros(shape, dtype=dtype, device=self.dev)
        P = self.P
        self.bufs = [z(self.T + 1, self.n, SEPMC_TRAJ_WIDTH) for _ in range(2)]
        self.buf = self.bufs[0]
        self.state, self.opp_state = z(P, policy.state_dim), z(P, opponent.state_dim)
        self.done = z(self.n, dtype=torch.uint8)                 # the step's per-robot done flags
        self.masks = z(2, P, dtype=torch.uint8)                  # per seat: the done flags of the last step, the mask of the next forward
        self.act, self.rew = z(self.n, ACT_DIM), z(self.n)
        self.seat_act = z(2, P, ACT_DIM)
        self.codes = z(2, P, dtype=torch.int32)
        self.opp_model = z(P, dtype=torch.int32) if self.pool else None     # each pair's model in the pool, redrawn where masks[1] is set
        # per slab: the state and mask its first forward started from, V(observation T)
        self.init_states = [z(P, policy.state_dim) for _ in range(2)]
        self.first_masks = [z(P, dtype=torch.uint8) for _ in range(2)]
        self.boots = [z(P) for _ in range(2)]
        self._scratch_state, self._scratch_act = z(P, policy.state_dim), z(P, ACT_DIM)
        self.seed, self.calls = int(seed), 0
        self.pair_gid0 = int(engine.cfg.global_env_offset) // 2  # noise keyed by the global pair id: equal seeds on two shards still differ
        engine.set_option("record", 2)
        self.stream = torch.cuda.Stream(self.dev)                # one stream orders the kernels and torch's copies (see RolloutWorker)
        self.stream.wait_stream(torch.cuda.current_stream(self.dev))
        self.t = 0

    def _slab_index(self, buf):
        return 0 if buf is self.bufs[0] else 1

    def start(self, first_obs):
        """`first_obs` [2P, 965] (host or device): the observation `engine.reset()` returned.  Every pair starts an episode: zero
        states, masks 1."""
        first = torch.as_tensor(first_obs, dtype=torch.float32).to(self.dev)
        self.stream.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(self.stream):
            self.buf[0, :, :SEPMC_OBS_DIM] = first
            self.state.zero_()
            self.opp_state.zero_()
            self.masks.fill_(1)
        self.t = 0

    def _forward(self, row, state, act, heading_ptr, values_ptr, neglogp_ptr, codes_ptr, out_ld):
        self.pol.forward_rec(row.data_ptr(), 2 * SEPMC_TRAJ_WIDTH, self.P, self.masks[0].data_ptr(), state.data_ptr(), act.data_ptr(), codes_ptr,
                             heading_ptr, values_ptr, neglogp_ptr, out_ld, self.seed, self.calls, self.pair_gid0, self.stream.cuda_stream)

    def step(self):
        """Two forwards, the copies and one fused env step; fills record t of both seats.  Asynchronous on the worker's stream."""
        assert self.t < self.T, "unroll is full: call finish_unroll()"
        row, nxt = self.buf[self.t], self.buf[self.t + 1]
        p0, p1 = row.data_ptr(), row.data_ptr() + SEPMC_TRAJ_WIDTH * _FSZ    # first seat-0 and seat-1 records of row t
        with torch.cuda.stream(self.stream):
            if self.t == 0:
                i = self._slab_index(self.buf)
                self.init_states[i].copy_(self.state)
                self.first_masks[i].copy_(self.masks[0])
            self._forward(row, self.state, self.seat_act[0], p0 + SCOL_HEADING * _FSZ, p0 + SCOL_VALUE * _FSZ, p0 + SCOL_NEGLOGP * _FSZ,
                          self.codes[0].data_ptr(), 2 * SEPMC_TRAJ_WIDTH)
            if self.pool:
                self.opp.forward(p1, 2 * SEPMC_TRAJ_WIDTH, self.P, self.masks[1].data_ptr(), self.opp_state.data_ptr(), self.seat_act[1].data_ptr(),
                                 self.codes[1].data_ptr(), None, self.opp_model.data_ptr(), p0 + SCOL_OPPONENT * _FSZ, 2 * SEPMC_TRAJ_WIDTH,
                                 self.seed, self.calls, self.pair_gid0, self.stream.cuda_stream)
            else:
                self.opp.forward(p1, 2 * SEPMC_TRAJ_WIDTH, self.P, self.masks[1].data_ptr(), self.opp_state.data_ptr(),
                                 self.seat_act[1].data_ptr(), self.codes[1].data_ptr(), None, self.stream.cuda_stream)
            self.act.view(self.P, 2, ACT_DIM).copy_(self.seat_act.transpose(0, 1))
            row[:, SCOL_CODE].view(self.P, 2).copy_(self.codes.t())
        self.eng.step_device(self.act.data_ptr(), nxt.data_ptr(), self.rew.data_ptr(), self.done.data_ptr(), obs_ld=SEPMC_TRAJ_WIDTH,
                             stream=self.stream.cuda_stream)
        with torch.cuda.stream(self.stream):
            self.masks.copy_(self.done.view(self.P, 2).t())
        self.calls += 1
        self.t += 1

    def finish_unroll(self):
        """`SepmcUnroll(slab [T, 2P, 984] view, initial_state [P, 192], first_mask [P] uint8, bootstrap_value [P])` of seat 0, all valid
        until the end of the NEXT unroll; stepping continues in the other slab, whose row 0 receives observation T.

        bootstrap_value = V(observation T) of seat 0: the training forward on a scratch copy of the state with the current counter, so
        neither the worker's state nor its counter advances and the next unroll's first forward computes the same V bit for bit."""
        assert self.t == self.T
        done_buf = self.buf
        idx = self._slab_index(done_buf)
        self.buf = self.bufs[1 - idx]
        with torch.cuda.stream(self.stream):
            self._scratch_state.copy_(self.state)
            self._forward(done_buf[self.T], self._scratch_state, self._scratch_act, None, self.boots[idx].data_ptr(), None, None, 1)
            self.buf[0, :, :SEPMC_OBS_DIM] = done_buf[self.T, :, :SEPMC_OBS_DIM]
        self.t = 0
        return SepmcUnroll(done_buf[:self.T], self.init_states[idx], self.first_masks[idx], self.boots[idx])

    def set_opponent_probs(self, probs):
        """The opponent pool's draw probabilities (one per model, >= 0, positive sum) for the games that start from the next step on."""
        if not self.pool:
            raise ValueError("the worker plays a single opponent")
        self.opp.set_probs(probs)

    def wait(self):
        """Make torch's current stream wait for everything queued so far (call before reading a finished slab there)."""
        torch.cuda.current_stream(self.dev).wait_stream(self.stream)
