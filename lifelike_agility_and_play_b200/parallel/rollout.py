"""On-device actor loops producing learner-ready unrolls (rows f2 + f3 joined to the hot path), one worker per level.

Replaces, for one GPU's block of environments, the reference actor's per-env loop `obs -> agent.step -> env.step -> queue`
(learning/actors/distill_actor.py:205-270) and its unroll assembly (`:120-167`): the policy kernel (csrc/llq_policy.cu,
csrc/llq_policy_hier.cu) reads observation row t of the trajectory slab in place, the fused env step (llq_step_ex, LLQ_IO_DEVICE,
record option 2) consumes its actions, writes a_t | r_t | done_t into row t and the *next* observation straight into row t+1 of the
slab, so record t = (obs_t, a_t, r_t, done_t) is aligned the way the learner wants it (X = the observation the action was computed
from) without any staging copy.  Nothing synchronises with the host inside an unroll.  Two `[T+1, N, width]` slabs ping-pong:
`finish_unroll()` hands back a view of the finished one (it stays valid for the whole next unroll, so the NCCL gather / unroll
conversion overlaps the stepping) and carries observation T over to row 0 of the other.  Slab layouts: parallel/trajectory.py.

* `RolloutWorker` (primitive level, PMC): the policy kernel writes V and -log p of the sampled action into the record.
* `HierRolloutWorker` (environmental level, EPMC): the training forward (llq_hier_policy_forward_rec) samples the code and writes -log p
  and V into the record; the code goes from the kernel's int32 output into the code column.
* `SepmcRolloutWorker` (strategic level, SEPMC, the chase-tag game): robot 2p of each env-pair p is the learning agent (seat 0) and robot
  2p+1 its frozen opponent (seat 1), as a TLeague actor plays the learning model against one from the pool; the game's termination
  reads robot 0's fall and contacts only.  Per step:
    - the strategic training forward (llq_hier_policy_forward_rec_strategic) on the seat-0 rows of slab row t, read in place with a
      row stride of two records, samples the heading and writes its raw value, -log p and V straight into those records; its noise is
      keyed by the global pair id;
    - the opponent's deterministic forward (llq_hier_policy_forward) on the seat-1 rows; against an opponent pool
      (policy_epmc.DeviceOpponentPool, llq_hier_policy_forward_pool) every pair whose game starts first draws its opponent's model from
      the pool's probabilities, and the model index goes into the opponent column of the pair's seat-0 record;
    - device-side copies interleave both seats' actions into the engine's [2P, 12] action array and put both seats' codes into the code
      column; after the fused step the pair's done flags (equal on both rows) are copied into each seat's contiguous mask for the next
      forwards.
Model refresh: `update_policy(weights)` (every worker) and `SepmcRolloutWorker.update_opponent(weights, k)` queue the new weights on the
worker's stream (set_weights / set_model of the handle: a host list, or a flat CUDA tensor, e.g. the blob the learner rank broadcast);
they take effect from the next `step()`, and the LSTM states, masks, counters and slabs stay as they are: an episode in progress continues
with the new weights.
Several GPUs: `UnrollExchange(worker)` hands each finished unroll to the learner rank in place (the slab and the per-slab state, mask and
bootstrap value go out of the worker's own buffers in one NCCL group); the worker's stream waits on the device for a slab's hand-over
before it writes into that slab again.  At the strategic level `learner_seat_only=True` sends the seat-0 records alone, packed into a
contiguous buffer first (`pack_learner_seat`), half the bytes.
The recurrent levels keep their LSTM states on the device ([N, 128] at the environmental level: code LSTM, then value LSTM; [P, 192]
for seat 0 at the strategic level: heading, code and value LSTM, and [P, 128] for seat 1), and each forward receives the done flags of
the step before it, so a finished episode's state is wiped exactly where the reference actor's mask is set.
"""
import ctypes as C
from collections import namedtuple

import torch

from ..policy_epmc import DeviceHierPolicy, DeviceOpponentPool, DeviceSepmcTrainPolicy, _policy_lib
from .trajectory import (ACT_DIM, COL_NEGLOGP, COL_VALUE, HCOL_CODE, HCOL_NEGLOGP, HCOL_VALUE, HIER_OBS_DIM, HIER_TRAJ_WIDTH, OBS_DIM,
                         SCOL_CODE, SCOL_HEADING, SCOL_NEGLOGP, SCOL_OPPONENT, SCOL_VALUE, SEPMC_OBS_DIM, SEPMC_TRAJ_WIDTH, TRAJ_WIDTH, HandOver)

# what the recurrent workers' finish_unroll() returns: the [T, N, width] slab view, then the learner's state [rows, state_dim] and
# mask [rows] (uint8) its first forward started from, and V(observation T) [rows]; all valid until the end of the NEXT unroll
Unroll = namedtuple("Unroll", ["slab", "initial_state", "first_mask", "bootstrap_value"])
_FSZ = 4                                    # bytes per float: column offsets into a slab row
_seat_lib = None


def pack_learner_seat(slab, out, stream=None):
    """`out` [T, P, 984] = `slab[:, 0::2]` of a strategic-level `[T, 2P, 984]` slab, the learning robots' records, bit for bit, by the
    pack kernel (include/llq_policy.h, llq_seat_pack); both contiguous float32 on one CUDA device.  Asynchronous on `stream` (a
    torch.cuda.Stream; default: the current stream)."""
    global _seat_lib
    W = SEPMC_TRAJ_WIDTH
    if not (isinstance(slab, torch.Tensor) and isinstance(out, torch.Tensor) and slab.dim() == 3 and out.dim() == 3 and out.shape[2] == W
            and tuple(slab.shape) == (out.shape[0], 2 * out.shape[1], W) and slab.dtype == out.dtype == torch.float32
            and slab.is_cuda and slab.device == out.device and slab.is_contiguous() and out.is_contiguous()):
        raise ValueError("pack_learner_seat takes a contiguous float32 [T, 2P, %d] slab and a [T, P, %d] output on one CUDA device, got %s %s"
                         % (W, W, getattr(slab, "shape", slab), getattr(out, "shape", out)))
    T, P = out.shape[:2]
    if _seat_lib is None:
        lib = _policy_lib()
        lib.llq_seat_pack.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]
        lib.llq_seat_pack_last_error.restype = C.c_char_p
        _seat_lib = lib
    s = torch.cuda.current_stream(out.device) if stream is None else stream
    if _seat_lib.llq_seat_pack(slab.data_ptr(), out.data_ptr(), T, P, s.cuda_stream):
        raise RuntimeError("llq_seat_pack: %s" % _seat_lib.llq_seat_pack_last_error().decode())


class _SlabWorker:
    """What the workers of every level share: the two slabs, the side stream, the engine's action / reward / done buffers, the step
    counter and the fused step.  A level sets _OBS_DIM, _WIDTH (the record), _LEVEL, _SEATS (robots per forward row: 1, or 2 for a
    chase-tag pair) and defines `_act(row)` (the forwards and copies of record t, before the env step), `_bootstrap(obs_row, out)`
    (V of observation T into `out`) and `_unroll(slab, i)` (what finish_unroll returns for slab i)."""

    def __init__(self, engine, policy, unroll, device, seed):
        name = type(self).__name__
        if engine.obs_dim != self._OBS_DIM:
            raise ValueError("%s drives the %s env (%d-wide observations)" % (name, self._LEVEL, self._OBS_DIM))
        if not int(engine.cfg.auto_reset):
            raise ValueError("%s needs an engine with auto_reset=1" % name)
        self.eng, self.pol, self.T, self.n = engine, policy, int(unroll), engine.n
        self.rows = self.n // self._SEATS
        self.dev = torch.device(device)
        self.bufs = [self._zeros(self.T + 1, self.n, self._WIDTH) for _ in range(2)]
        self.buf = self.bufs[0]
        self.act, self.rew, self.done = self._zeros(self.n, ACT_DIM), self._zeros(self.n), self._zeros(self.n, dtype=torch.uint8)
        self.boots = [self._zeros(self.rows) for _ in range(2)]     # per slab: V(observation T)
        self.seed, self.calls = int(seed), 0
        self.handed = [None, None]          # per slab: the event that ends its hand-over to the learner rank (UnrollExchange)
        # noise keyed by the global id of the forward's row (env or pair): equal seeds on two shards still differ
        self.gid0 = int(engine.cfg.global_env_offset) // self._SEATS
        engine.set_option("record", 2)      # a_t | r_t | done_t go to the slab row BEFORE the one receiving obs_{t+1}
        # everything the worker launches (kernels through the C-ABI and torch's column copies) is ordered on ONE side stream: a
        # NULL stream would mean "the engine's own non-blocking stream" to llq_step_ex and would not order with torch's work
        self.stream = torch.cuda.Stream(self.dev)
        self.stream.wait_stream(torch.cuda.current_stream(self.dev))
        self.t = 0

    def _zeros(self, *shape, dtype=torch.float32):
        return torch.zeros(shape, dtype=dtype, device=self.dev)

    def _slab_index(self):
        return 0 if self.buf is self.bufs[0] else 1

    def start(self, first_obs):
        """`first_obs` [N, obs] (host or device): the observation `engine.reset()` returned.  Every env starts an episode."""
        first = torch.as_tensor(first_obs, dtype=torch.float32).to(self.dev)
        self.stream.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(self.stream):
            self.buf[0, :, :self._OBS_DIM] = first
            self._start_state()
        self.t = 0

    def _start_state(self):
        pass

    def step(self):
        """The level's forwards + one fused env step; fills record t.  Asynchronous on the worker's stream."""
        assert self.t < self.T, "unroll is full: call finish_unroll()"
        row, nxt = self.buf[self.t], self.buf[self.t + 1]
        self._act(row)
        self.eng.step_device(self.act.data_ptr(), nxt.data_ptr(), self.rew.data_ptr(), self.done.data_ptr(), obs_ld=self._WIDTH,
                             stream=self.stream.cuda_stream)
        self.calls += 1
        self.t += 1

    def finish_unroll(self):
        """Hands back the finished slab (see the worker's class), valid until the end of the NEXT unroll; stepping continues in the
        other slab, whose row 0 receives observation T."""
        assert self.t == self.T
        done_buf, i = self.buf, self._slab_index()
        self.buf = self.bufs[1 - i]
        with torch.cuda.stream(self.stream):
            # V of the observation that follows the last record: the bootstrap of the lambda-return (unroll.py)
            self._bootstrap(done_buf[self.T], self.boots[i])
            self._claim(1 - i)
            self.buf[0, :, :self._OBS_DIM] = done_buf[self.T, :, :self._OBS_DIM]
        self.t = 0
        return self._unroll(done_buf[:self.T], i)

    def _claim(self, i):
        # slab i (and its state, mask and bootstrap value) may still be on its way to the learner rank: the worker's stream waits for the
        # end of that transfer before anything writes into them again (the host does not wait)
        if self.handed[i] is not None:
            self.stream.wait_event(self.handed[i])
            self.handed[i] = None

    def wait(self):
        """Make torch's current stream wait for everything queued so far (call before reading a finished slab there)."""
        torch.cuda.current_stream(self.dev).wait_stream(self.stream)

    def update_policy(self, weights):
        """The learner's new weights for the worker's policy from the next `step()` on: the refresh is queued on the worker's stream
        behind every step queued so far (and behind torch's current stream, where a device blob may just have been broadcast).  `weights`:
        what the policy's `set_weights` takes, the model's arrays or a flat CUDA tensor.  The LSTM states, masks, counters and slabs stay:
        episodes in progress continue with the new weights.  A refresh between `finish_unroll()` and the next `step()` leaves the finished
        unroll's bootstrap V computed with the old weights."""
        self._refresh(self.pol.set_weights, weights)

    def _refresh(self, set_weights, weights, *head):
        self.stream.wait_stream(torch.cuda.current_stream(self.dev))
        set_weights(*head, weights, stream=self.stream.cuda_stream)


class RolloutWorker(_SlabWorker):
    """The primitive level (PMC, 207-wide observations, `[T+1, N, 223]` slabs).  `finish_unroll()` returns the copy-free `[T, N, 223]`
    view of the finished records; `self.bootstrap_value` [N] = V(observation T) of that slab."""
    _OBS_DIM, _WIDTH, _LEVEL, _SEATS = OBS_DIM, TRAJ_WIDTH, "PMC", 1

    def __init__(self, engine, policy, unroll, device, sample=True, seed=0):
        """`engine`: a `_capi.VecEngine` on the CUDA library with auto_reset=1 (PMC, 207-wide observations);
        `policy`: a `policy.DevicePolicy` on the same device; `unroll`: T (128 in example_pmc_train.sh:145);
        `sample`: draw the actions from the Gaussian head and record -log p (training rollouts) instead of the mean (evaluation)."""
        super().__init__(engine, policy, unroll, device, seed)
        self.sample = bool(sample)
        self._scratch_act = self._zeros(self.n, ACT_DIM)
        self.bootstrap_value = self.boots[0]

    def _act(self, row):
        # Every column of record t is written by the two kernels themselves, no copies: the policy kernel reads observation t in
        # place and writes V / -log p into the value / neglogp columns of row t (row stride 223); the fused step writes the rest.
        p = row.data_ptr()
        self.pol.forward_rec(p, TRAJ_WIDTH, self.n, self.act.data_ptr(), p + COL_VALUE * _FSZ, (p + COL_NEGLOGP * _FSZ) if self.sample else None,
                             TRAJ_WIDTH, self.seed, self.calls, self.gid0, self.stream.cuda_stream)

    def _bootstrap(self, obs_row, out):
        self.pol.forward_ex(obs_row.data_ptr(), TRAJ_WIDTH, self.n, self._scratch_act.data_ptr(), None, out.data_ptr(), None, 0, 0,
                            self.stream.cuda_stream)

    def _unroll(self, slab, i):
        self.bootstrap_value = self.boots[i]
        return slab


class _RecurrentWorker(_SlabWorker):
    """The recurrent levels: the learner's LSTM states [rows, state_dim] stay on the device, and each slab keeps the state and mask its
    first forward started from.  A level sets `mask` (the learner's [rows] uint8 mask: the done flags of the last step) and defines
    `_forward(row, state, act, out_ld, values=None, neglogp=None, codes=None, ...)`, the learner's training forward from slab row `row`."""

    def __init__(self, engine, policy, unroll, device, seed):
        super().__init__(engine, policy, unroll, device, seed)
        z, rows, dim = self._zeros, self.rows, policy.state_dim
        self.state = z(rows, dim)
        self.init_states, self.first_masks = [z(rows, dim) for _ in range(2)], [z(rows, dtype=torch.uint8) for _ in range(2)]
        self._scratch_state, self._scratch_act = z(rows, dim), z(rows, ACT_DIM)

    def step(self):
        if self.t == 0:
            i = self._slab_index()
            with torch.cuda.stream(self.stream):
                self.init_states[i].copy_(self.state)
                self.first_masks[i].copy_(self.mask)
        super().step()

    def _bootstrap(self, obs_row, out):
        # the training forward on a scratch copy of the state with the current counter, so neither the worker's state nor its counter
        # advances and the next unroll's first forward computes the same V bit for bit -- unless update_policy() comes between
        # finish_unroll() and that forward: the bootstrap keeps the old weights' V, the next forward has the new weights'
        self._scratch_state.copy_(self.state)
        self._forward(obs_row, self._scratch_state, self._scratch_act, 1, values=out.data_ptr())

    def _unroll(self, slab, i):
        return Unroll(slab, self.init_states[i], self.first_masks[i], self.boots[i])


class HierRolloutWorker(_RecurrentWorker):
    """The environmental level (EPMC, 916-wide observations, `[T+1, N, 936]` slabs).  `finish_unroll()` returns `Unroll(slab [T, N, 936]
    view, initial_state [N, 128], first_mask [N] uint8, bootstrap_value [N])`."""
    _OBS_DIM, _WIDTH, _LEVEL, _SEATS = HIER_OBS_DIM, HIER_TRAJ_WIDTH, "EPMC", 1

    def __init__(self, engine, policy, unroll, device, seed=0):
        """`engine`: a `_capi.VecEngine` on the CUDA library for the EPMC env (916-wide observations) with auto_reset=1;
        `policy`: a `policy_epmc.DeviceHierPolicy(..., train=True)` on the same device; `unroll`: T."""
        if not (isinstance(policy, DeviceHierPolicy) and policy.train and not policy.strategic):
            raise ValueError("HierRolloutWorker needs an environmental-level DeviceHierPolicy created with train=True")
        super().__init__(engine, policy, unroll, device, seed)
        self.mask = self.done
        self.codes = self._zeros(self.n, dtype=torch.int32)

    def _start_state(self):
        self.state.zero_()
        self.done.fill_(1)

    def _forward(self, row, state, act, out_ld, values=None, neglogp=None, codes=None):
        self.pol.forward_rec(row.data_ptr(), HIER_TRAJ_WIDTH, self.n, self.mask.data_ptr(), state.data_ptr(), act.data_ptr(), codes, values, neglogp,
                             out_ld, self.seed, self.calls, self.gid0, self.stream.cuda_stream)

    def _act(self, row):
        p = row.data_ptr()
        with torch.cuda.stream(self.stream):
            self._forward(row, self.state, self.act, HIER_TRAJ_WIDTH, p + HCOL_VALUE * _FSZ, p + HCOL_NEGLOGP * _FSZ, self.codes.data_ptr())
            row[:, HCOL_CODE].copy_(self.codes)


class SepmcRolloutWorker(_RecurrentWorker):
    """The strategic level (SEPMC, 965-wide observations, 2P robots, `[T+1, 2P, 984]` slabs).  `finish_unroll()` returns `Unroll(slab
    [T, 2P, 984] view, initial_state [P, 192], first_mask [P] uint8, bootstrap_value [P])`, the last three of seat 0."""
    _OBS_DIM, _WIDTH, _LEVEL, _SEATS = SEPMC_OBS_DIM, SEPMC_TRAJ_WIDTH, "SEPMC", 2

    def __init__(self, engine, policy, opponent, unroll, device, seed=0):
        """`engine`: a `_capi.VecEngine` on the CUDA library for the SEPMC env (965-wide observations, 2P robots) with auto_reset=1 and an
        even `global_env_offset`; `policy`: a `policy_epmc.DeviceSepmcTrainPolicy` (the learner's weights); `opponent`: a deterministic
        strategic-level `policy_epmc.DeviceHierPolicy` (its own weights), or a `policy_epmc.DeviceOpponentPool` with max_rows >= P (each
        pair draws its opponent's model at every game start; see `set_opponent_probs`), all on the engine's device; `unroll`: T."""
        if int(engine.cfg.global_env_offset) % 2:
            raise ValueError("global_env_offset must be even: robots 2p and 2p+1 form a pair")
        if not isinstance(policy, DeviceSepmcTrainPolicy):
            raise ValueError("SepmcRolloutWorker needs a DeviceSepmcTrainPolicy")
        self.pool = isinstance(opponent, DeviceOpponentPool)
        if not (self.pool or (isinstance(opponent, DeviceHierPolicy) and opponent.strategic and not opponent.train)):
            raise ValueError("the opponent must be a deterministic strategic-level DeviceHierPolicy or a DeviceOpponentPool")
        if self.pool and opponent.max_rows < engine.n // 2:
            raise ValueError("the opponent pool's max_rows is below the number of pairs")
        super().__init__(engine, policy, unroll, device, seed)
        z, P = self._zeros, self.rows
        self.opp, self.opp_state = opponent, z(P, opponent.state_dim)
        self.masks = z(2, P, dtype=torch.uint8)              # per seat: the done flags of the last step, the mask of the next forward
        self.mask = self.masks[0]
        self.seat_act, self.codes = z(2, P, ACT_DIM), z(2, P, dtype=torch.int32)
        self.opp_model = z(P, dtype=torch.int32) if self.pool else None     # each pair's model in the pool, redrawn where masks[1] is set

    def _start_state(self):
        self.state.zero_()
        self.opp_state.zero_()
        self.masks.fill_(1)

    def _forward(self, row, state, act, out_ld, values=None, neglogp=None, codes=None, heading=None):
        self.pol.forward_rec(row.data_ptr(), 2 * SEPMC_TRAJ_WIDTH, self.rows, self.mask.data_ptr(), state.data_ptr(), act.data_ptr(), codes,
                             heading, values, neglogp, out_ld, self.seed, self.calls, self.gid0, self.stream.cuda_stream)

    def _act(self, row):
        P, ld = self.rows, 2 * SEPMC_TRAJ_WIDTH
        p0, p1 = row.data_ptr(), row.data_ptr() + SEPMC_TRAJ_WIDTH * _FSZ    # first seat-0 and seat-1 records of row t
        with torch.cuda.stream(self.stream):
            self._forward(row, self.state, self.seat_act[0], ld, p0 + SCOL_VALUE * _FSZ, p0 + SCOL_NEGLOGP * _FSZ, self.codes[0].data_ptr(),
                          p0 + SCOL_HEADING * _FSZ)
            if self.pool:
                self.opp.forward(p1, ld, P, self.masks[1].data_ptr(), self.opp_state.data_ptr(), self.seat_act[1].data_ptr(),
                                 self.codes[1].data_ptr(), None, self.opp_model.data_ptr(), p0 + SCOL_OPPONENT * _FSZ, ld, self.seed, self.calls,
                                 self.gid0, self.stream.cuda_stream)
            else:
                self.opp.forward(p1, ld, P, self.masks[1].data_ptr(), self.opp_state.data_ptr(), self.seat_act[1].data_ptr(),
                                 self.codes[1].data_ptr(), None, self.stream.cuda_stream)
            self.act.view(P, 2, ACT_DIM).copy_(self.seat_act.transpose(0, 1))
            row[:, SCOL_CODE].view(P, 2).copy_(self.codes.t())

    def step(self):
        """Two forwards, the copies and one fused env step; fills record t of both seats.  Asynchronous on the worker's stream."""
        super().step()
        with torch.cuda.stream(self.stream):
            self.masks.copy_(self.done.view(self.rows, 2).t())

    def update_opponent(self, weights, k=None):
        """New weights for the frozen opponent from the next `step()` on, queued like `update_policy`: the single opponent's (`k` None) or
        model `k` of the opponent pool (`k` required).  `weights`: a strategic-level model (152 arrays) or a flat CUDA tensor in the blob
        layout.  Pairs in a game against the replaced model continue that game with the new weights and the state they carry."""
        if self.pool:
            if k is None:
                raise ValueError("the worker plays an opponent pool: name the model k to replace")
            self._refresh(self.opp.set_model, weights, k)
        else:
            if k is not None:
                raise ValueError("the worker plays a single opponent: k must be None")
            self._refresh(self.opp.set_weights, weights)

    def set_opponent_probs(self, probs):
        """The opponent pool's draw probabilities (one per model, >= 0, positive sum) for the games that start from the next step on."""
        if not self.pool:
            raise ValueError("the worker plays a single opponent")
        self.opp.set_probs(probs)


class UnrollExchange:
    """Hands the finished unrolls of a rollout worker (any level) to the learner rank `dst` of `group`, overlapped with the next unroll.

    `hand_over(u)` takes what `worker.finish_unroll()` returned and posts its transfer (`trajectory.HandOver`) on a side stream behind
    the worker's stream: the `[T, N, W]` slab -- the leading rows of the worker's `[T+1, N, W]` buffer -- and, per slab, the recurrent
    levels' `initial_state` and `first_mask` and every level's `bootstrap_value` (V of observation T) go out in place, in one NCCL group;
    the host does not wait.  The finished slab stays valid during the next unroll and is written again from the end of it
    (`finish_unroll()` puts observation T into row 0 of the other slab): the worker's stream waits there, on the device, for the
    hand-over of that slab.  `gathered(b)` on `dst` returns one `Unroll` per rank, views of the received buffers shaped as the worker
    returns them (the primitive level's with `initial_state` and `first_mask` None), ready for `slab_records` /
    `slab_to_unrolls(u.slab, key, bootstrap_value=u.bootstrap_value)`, `hier_slab_records` or `sepmc_slab_records`; None on the other
    ranks.  A world of 1 returns the worker's own views, with no copy (`own_copy=True` copies them as a learner rank of a larger world
    copies its own unroll).

    The strategic level sends by default the slab as the worker wrote it, both seats: the opponent's model (column 983) travels in the
    seat-0 records, and the seat-1 records, which the learner never reads, double the bytes (4.13 GB per rank and unroll at T = 128,
    P = 4096).  `learner_seat_only=True` (a `SepmcRolloutWorker` only) sends the seat-0 records alone: `hand_over` first packs them into
    one contiguous `[T, P, 984]` send buffer of the exchange (`pack_learner_seat`, on the side stream behind the worker's stream and
    behind the previous transfer out of that buffer), then sends that buffer in the slab's place, with the same state, mask and bootstrap
    value.  The slab's hand-over event is recorded behind the pack and the transfer, so the worker rewrites a slab only after both.
    `gathered(b)` returns `Unroll(slab [T, P, 984], initial_state, first_mask, bootstrap_value)` per rank, for
    `sepmc_slab_records(..., learner_seat_only=True)`; a world of 1 without `own_copy` returns the send buffer itself, which the next
    `hand_over` packs again once the next unroll is complete: valid, like the worker's views, until the end of the next unroll.
    `bytes_per_rank` is 2.07 GB at T = 128, P = 4096, and every rank keeps one send buffer of 2.06 GB.  One buffer is enough: the
    next pack waits for the worker's whole next unroll, which takes far longer than a transfer.

    Memory on the learner rank: `2 x world x bytes_per_rank` bytes of receive buffers, `bytes_per_rank` = T*N*W*4 + state + mask +
    bootstrap, on top of the worker's own two `[T+1, N, W]` slabs.  At T = 128: PMC at N = 4096 sends 0.47 GB per rank (7.5 GB for
    8 ranks); EPMC at N = 8192 3.93 GB (62.9 GB for 8 ranks, plus 7.9 GB of slabs: too much next to an engine on an 80 GB card), at
    N = 4096 1.97 GB (31.4 GB for 8 ranks, plus 4.0 GB of slabs: fits on an 80 GB learner rank); SEPMC at P = 4096 4.13 GB (66.1 GB for
    8 ranks), or with `learner_seat_only` 2.07 GB (33.1 GB for 8 ranks, plus 8.3 GB of slabs and the 2.06 GB send buffer).
    """

    def __init__(self, worker, dst=0, group=None, own_copy=None, learner_seat_only=False):
        if not isinstance(worker, _SlabWorker):
            raise ValueError("UnrollExchange hands over the unrolls of a RolloutWorker, HierRolloutWorker or SepmcRolloutWorker")
        self.learner_seat_only = bool(learner_seat_only)
        if self.learner_seat_only and not isinstance(worker, SepmcRolloutWorker):
            raise ValueError("learner_seat_only is for a SepmcRolloutWorker: the other levels have one seat")
        self.worker = worker
        self.recurrent = isinstance(worker, _RecurrentWorker)
        self.send = worker._zeros(worker.T, worker.rows, SEPMC_TRAJ_WIDTH) if self.learner_seat_only else None
        self.core = HandOver([(x.shape, x.dtype) for x in self._tensors(0)], worker.dev, dst, group, own_copy)
        self.world, self.rank, self.dst, self.bytes_per_rank = self.core.world, self.core.rank, self.core.dst, self.core.bytes_per_rank
        self._last = None                   # the ping-pong index of the last hand-over: its transfer reads the send buffer

    def _tensors(self, i):
        w = self.worker
        slab = self.send if self.learner_seat_only else w.bufs[i][:w.T]
        return (slab, w.init_states[i], w.first_masks[i], w.boots[i]) if self.recurrent else (slab, w.boots[i])

    def hand_over(self, u):
        """`u`: what the worker's `finish_unroll()` just returned (the slab view at the primitive level, an `Unroll` at the other two).
        Starts the transfer of that unroll; returns its slab index (pass it to `gathered` on the learner rank)."""
        w = self.worker
        slab = u.slab if isinstance(u, Unroll) else u
        i = next((k for k in (0, 1) if slab.data_ptr() == w.bufs[k].data_ptr()), None)
        if i is None or i == w._slab_index():
            raise ValueError("hand_over() takes the unroll the worker's finish_unroll() returned last")
        stream = w.stream
        if self.learner_seat_only:
            stream = self.core.side
            stream.wait_stream(w.stream)
            if self._last is not None:
                stream.wait_event(self.core.sent[self._last])      # the previous transfer has left the send buffer
            pack_learner_seat(slab, self.send, stream)
        self.core.post(i, self._tensors(i), stream=stream)
        w.handed[i] = self.core.sent[i]     # recorded behind the pack and the transfer: the worker rewrites slab i after both
        self._last = i
        return i

    def gathered(self, b):
        """Learner rank: one `Unroll` per rank of the unroll handed over as `b`, readable on torch's current stream (the wait is queued
        there); None on the other ranks."""
        g = self.core.gathered(b)
        if g is None:
            return None
        if self.recurrent:
            return [Unroll(*(x[r] for x in g)) for r in range(g[0].shape[0])]
        return [Unroll(g[0][r], None, None, g[1][r]) for r in range(g[0].shape[0])]
