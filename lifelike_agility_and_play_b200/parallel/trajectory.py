"""Multi-GPU plumbing of the rollout: env shards and the trajectory gather to the learner rank.

Environments are independent (SURVEY 8e), so the data path has no collective: rank r owns the contiguous block
[r*N, (r+1)*N) of global env ids (RNG streams are keyed by global id, hence results do not depend on the world size).
The only exchange is the hand-over of a finished unroll -- a [T, N_local, 223] fp32 slab whose record mirrors the
reference's PMCInputs (networks/legged_robot/pmc_net/pmc_net_data.py:7-16; actor->learner push, distill_actor.py:164-167)
-- to the learner rank, one gather per unroll (NCCL over NVLink on GPUs, gloo in the CPU tests).  The fused step kernel
writes the record (observation, and with the "record" option action / reward / done) directly into the slab (llq_step_ex
obs_ld = 223), so there is no staging copy between stepping and the send buffer.  `TrajectoryExchange` is the designed
hand-over (SURVEY 8e): two slabs ping-pong, the finished one travels as grouped point-to-point sends / receives on a side
stream while the next unroll is stepped into the other.  `HandOver` is its transfer, for tensors owned by the caller: the rollout
workers' unrolls (slab, recurrent state, mask, bootstrap value) travel through it in place (parallel/rollout.py, `UnrollExchange`).
"""
import torch
import torch.distributed as dist

OBS_DIM, ACT_DIM = 207, 12
COL_ACTION, COL_REWARD, COL_DONE, COL_NEGLOGP, COL_VALUE = 207, 219, 220, 221, 222
TRAJ_WIDTH = 223
# the environmental level's record (parallel/rollout.py, HierRolloutWorker): obs 916 | action 12 | reward | done (the step kernel, record
# option 2) | -log p | value | sampled code (as a float), padded to a multiple of 4 floats
HIER_OBS_DIM = 916
HCOL_ACTION, HCOL_REWARD, HCOL_DONE, HCOL_NEGLOGP, HCOL_VALUE, HCOL_CODE = 916, 928, 929, 930, 931, 932
HIER_TRAJ_WIDTH = 936
# the strategic level's record, one row per robot (parallel/rollout.py, SepmcRolloutWorker): obs 965 | action 12 | reward | done (the
# step kernel, record option 2) | -log p | value | code (as a float) | raw sampled heading | opponent (as a float), 984 floats, a multiple
# of 4.  The learning robot's rows (seat 0) carry all of them; the frozen opponent's (seat 1) carry the code and leave the rest at 0.
# `opponent` is the index of the model seat 1 plays in an opponent pool (policy_epmc.DeviceOpponentPool), and stays 0 against a single
# opponent.
SEPMC_OBS_DIM = 965
SCOL_ACTION, SCOL_REWARD, SCOL_DONE, SCOL_NEGLOGP, SCOL_VALUE, SCOL_CODE, SCOL_HEADING = 965, 977, 978, 979, 980, 981, 982
SCOL_OPPONENT = 983
SEPMC_TRAJ_WIDTH = 984


def shard_offset(rank, envs_per_rank):
    """Global id of this rank's env 0 (-> llq_config.global_env_offset)."""
    return int(rank) * int(envs_per_rank)


class TrajectorySlab:
    def __init__(self, unroll, n_envs, device):
        self.unroll, self.n = int(unroll), int(n_envs)
        self.buf = torch.zeros((self.unroll, self.n, TRAJ_WIDTH), dtype=torch.float32, device=device)

    def row(self, t):
        return self.buf[t % self.unroll]

    def record(self, t, action, reward, done, obs=None):
        """Fill the non-observation columns of record t (obs is written by the kernel unless given)."""
        r = self.row(t)
        if obs is not None:
            r[:, :OBS_DIM] = obs
        r[:, COL_ACTION:COL_ACTION + ACT_DIM] = action
        r[:, COL_REWARD] = reward
        r[:, COL_DONE] = done

    def gather_to_learner(self, dst=0, recv=None):
        """All ranks call this once per unroll; returns the list of per-rank slabs on `dst`, None elsewhere."""
        if not dist.is_initialized() or dist.get_world_size() == 1:
            return [self.buf]
        if dist.get_rank() == dst:
            if recv is None:
                recv = [torch.empty_like(self.buf) for _ in range(dist.get_world_size())]
            dist.gather(self.buf, recv, dst=dst)
            return recv
        dist.gather(self.buf, None, dst=dst)
        return None


class HandOver:
    """The transfer of one finished unroll per call to the learner rank ``dst``, for tensors the caller owns.

    An unroll is a tuple of tensors (``specs``: one ``(shape, dtype)`` each, dtypes may differ); the caller keeps two of them, ping-pong
    index 0 and 1.  ``post(b, tensors)`` starts the transfer of unroll b on a side stream behind the caller's stream -- one grouped
    ``batch_isend_irecv`` (ncclGroupStart / ncclSend / ncclRecv / ncclGroupEnd underneath) for every tensor of the unroll: every other rank
    sends its tensors in place, no staging copy, and the learner rank posts one receive per sender and tensor into ``[world, *shape]``
    buffers it allocates once per ping-pong index (2 x world x ``bytes_per_rank`` bytes), and copies its own tensors device-to-device.
    ``sent[b]`` (CUDA) completes when the tensors of unroll b may be written again; the caller's stream has to wait for it before it
    overwrites them.  CPU tensors (gloo) take the same path without streams.

    ``own_copy``: whether the learner rank copies its own tensors into the received buffers.  By default only with a world of several
    ranks; a world of 1 then hands back the caller's own tensors, with no copy.  ``own_copy=True`` on one rank runs the learner rank's
    copy of a larger world (how the copy's cost and ordering are measured and tested on one GPU).
    """

    def __init__(self, specs, device, dst=0, group=None, own_copy=None):
        self.specs = [(tuple(int(x) for x in shape), dtype) for shape, dtype in specs]
        self.dst, self.group = int(dst), group
        self.dev = torch.device(device)
        self.cuda = self.dev.type == "cuda"
        if self.cuda and self.dev.index is None:
            self.dev = torch.device("cuda", torch.cuda.current_device())
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        if not 0 <= self.dst < self.world:
            raise ValueError("dst %d is not a rank of a world of %d" % (self.dst, self.world))
        self.own_copy = self.world > 1 if own_copy is None else bool(own_copy)
        if self.world > 1 and not self.own_copy:
            raise ValueError("with several ranks the learner rank's own tensors go into the gathered buffers")
        self.bytes_per_rank = sum(torch.Size(s).numel() * torch.empty((), dtype=d).element_size() for s, d in self.specs)
        self.recv = None
        if self.rank == self.dst and self.own_copy:
            self.recv = [[torch.empty((self.world,) + s, dtype=d, device=self.dev) for s, d in self.specs] for _ in range(2)]
        self.posted = [None, None]                 # per ping-pong index: the tensors of its last transfer
        if self.cuda:
            self.side = torch.cuda.Stream(self.dev)
            self.ready = [torch.cuda.Event() for _ in range(2)]
            self.sent = [torch.cuda.Event() for _ in range(2)]

    def _post(self, b, tensors):
        ops = []
        if self.rank == self.dst:
            if self.recv is None:
                return
            for k, x in enumerate(tensors):
                for r in range(self.world):
                    if r == self.dst:
                        self.recv[b][k][r].copy_(x, non_blocking=True)
                    else:
                        ops.append(dist.P2POp(dist.irecv, self.recv[b][k][r], r, self.group, tag=k))
        else:
            ops = [dist.P2POp(dist.isend, x, self.dst, self.group, tag=k) for k, x in enumerate(tensors)]
        for w in (dist.batch_isend_irecv(ops) if ops else []):
            w.wait()                      # NCCL: orders the side stream behind the transfer (the host does not block); gloo: blocks

    def post(self, b, tensors, stream=None):
        """``tensors`` (one per spec, contiguous) are complete on ``stream`` (default: the current stream): start their transfer as
        unroll ``b`` (0 or 1).  The host does not wait."""
        tensors = tuple(tensors)
        if len(tensors) != len(self.specs) or any(tuple(x.shape) != s or x.dtype != d or x.device != self.dev or not x.is_contiguous()
                                                  for x, (s, d) in zip(tensors, self.specs)):
            raise ValueError("the tensors do not match the exchange's specs (shape, dtype, device, contiguous)")
        if self.cuda:
            self.ready[b].record(torch.cuda.current_stream(self.dev) if stream is None else stream)
            self.side.wait_event(self.ready[b])
            with torch.cuda.stream(self.side):
                self._post(b, tensors)
                self.sent[b].record(self.side)
        else:
            self._post(b, tensors)
        self.posted[b] = tensors

    def wait(self, b, stream=None):
        """Make ``stream`` (default: the current stream) wait for transfer b (CPU: already complete)."""
        if self.cuda and self.posted[b] is not None:
            (torch.cuda.current_stream(self.dev) if stream is None else stream).wait_event(self.sent[b])

    def gathered(self, b):
        """Learner rank: one ``[world, *shape]`` tensor per spec holding unroll b of every rank, readable on the current stream; without
        ``own_copy`` the caller's own tensors, unsqueezed; None on the other ranks."""
        self.wait(b)
        if self.rank != self.dst:
            return None
        if self.recv is None:
            return tuple(x.unsqueeze(0) for x in self.posted[b])
        return tuple(self.recv[b])


class TrajectoryExchange:
    """Double-buffered hand-over of finished unrolls to the learner rank, overlapped with stepping.

    Rank r steps its envs into ``slab()`` (a ``[T, N_local, width]`` device tensor the fused kernel writes in place).  When the
    unroll is complete ``hand_over()`` posts the transfer of that slab (``HandOver``) on a side stream -- every non-learner rank sends
    its slab, the learner posts one receive per sender into ``[world, T, N_local, width]`` and copies its own slab device-to-device
    -- and flips to the other slab, so the 128 steps of unroll k+1 run while unroll k is on the NVLinks.  The stepping stream
    only waits for a transfer when it is about to overwrite that slab again, one whole unroll later.
    CPU tensors (gloo, the world_size-2 tests) take the same path without streams.
    """

    def __init__(self, unroll, n_envs, width, device, dst=0, group=None):
        self.T, self.n, self.width, self.dst, self.group = int(unroll), int(n_envs), int(width), int(dst), group
        self.dev = torch.device(device)
        self.cuda = self.dev.type == "cuda"
        self.slabs = [torch.zeros((self.T, self.n, self.width), dtype=torch.float32, device=self.dev) for _ in range(2)]
        self.core = HandOver([(self.slabs[0].shape, torch.float32)], self.dev, self.dst, group)
        self.world, self.rank, self.bytes_per_rank = self.core.world, self.core.rank, self.core.bytes_per_rank
        self.cur = 0

    def slab(self):
        """The slab the current unroll is written into."""
        return self.slabs[self.cur]

    def hand_over(self):
        """The current slab is complete on the caller's current stream: start its transfer, continue in the other slab.
        Returns the index of the slab now in flight (pass it to ``gathered`` on the learner rank)."""
        b = self.cur
        self.core.post(b, (self.slabs[b],))
        self.cur ^= 1
        self.core.wait(self.cur)          # do not overwrite a slab that is still being sent
        return b

    def wait(self, b):
        """Make the caller's current stream wait for transfer b (CPU: already complete)."""
        self.core.wait(b)

    def gathered(self, b):
        """Learner rank: ``[world, T, N_local, width]`` of unroll b after ``wait(b)``; a single rank gets its own slab; None elsewhere."""
        self.wait(b)
        if self.world == 1:
            return self.slabs[b].unsqueeze(0)
        return self.core.recv[b][0] if self.rank == self.dst else None
