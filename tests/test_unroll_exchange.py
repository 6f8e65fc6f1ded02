"""The hand-over of finished unrolls to the learner rank (parallel/trajectory.py `HandOver`, parallel/rollout.py `UnrollExchange`).

CPU: the tuple core on gloo ranks (worlds of 2 and 3, the learner rank not rank 0, three unrolls so that both ping-pong buffers are
reused, fp32 / uint8 / int32 tensors of different shapes): the learner rank receives what every rank sent, bit for bit.
GPU (-m gpu): the workers of all three levels with the exchange on one rank hand the learner what the bare worker returns, bit for bit,
records included; the worker's stream waits for a slab's transfer before it writes into that slab again (a sleeping side stream); and,
with two or more GPUs, one NCCL rank per GPU: the learner's gathered records equal one process stepping all ranks' envs."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T, N, UNROLLS = 5, 6, 3


def _spec():
    """The tensors of one unroll: (shape, dtype) of each."""
    return [((T, N, 7), torch.float32), ((N,), torch.uint8), ((N, 3), torch.int32), ((N,), torch.float32)]


def _fill(rank, u, b):
    """Unroll u of `rank` in ping-pong buffer b: every element differs between ranks and unrolls, no byte of the mask is 0."""
    base = 1000 * u + 100000 * rank
    return (torch.arange(T * N * 7, dtype=torch.float32).reshape(T, N, 7) + base,
            (torch.arange(N, dtype=torch.int32) * 7 + 3 * u + 50 * rank + 1).remainder(255).add(1).to(torch.uint8),
            torch.arange(N * 3, dtype=torch.int32).reshape(N, 3) * (u + 2) - base,
            torch.full((N,), 0.5, dtype=torch.float32) + base + b)


def _core_worker(rank, world, dst, port, q):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from lifelike_agility_and_play_b200.parallel import HandOver
    x = HandOver(_spec(), "cpu", dst=dst)
    bufs = [[torch.zeros(s, dtype=d) for s, d in _spec()] for _ in range(2)]      # the caller's ping-pong tensors
    got = []
    for u in range(UNROLLS):
        b = u % 2
        for dst_t, src in zip(bufs[b], _fill(rank, u, b)):
            dst_t.copy_(src)
        x.post(b, bufs[b])
        g = x.gathered(b)
        if rank == dst:
            got.append([t.clone().numpy() for t in g])
        else:
            got.append(g)
    if rank == dst:
        q.put(got)
    else:
        assert all(g is None for g in got)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("world,dst", [(2, 1), (3, 2)])
def test_tuple_core_gathers_every_rank_bit_for_bit(built, world, dst):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33500 + 10 * world + (os.getpid() % 2000)
    procs = [ctx.Process(target=_core_worker, args=(r, world, dst, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = q.get(timeout=240)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert len(got) == UNROLLS
    for u in range(UNROLLS):
        for k, (shape, dtype) in enumerate(_spec()):
            assert got[u][k].shape == (world,) + shape and got[u][k].dtype == torch.empty((), dtype=dtype).numpy().dtype
            for r in range(world):
                assert np.array_equal(got[u][k][r], _fill(r, u, u % 2)[k].numpy()), (u, k, r)


def test_one_rank_core_returns_the_callers_tensors(built):
    """A world of 1: the caller's own tensors without a copy, or a copy with own_copy=True; tensors off the specs are refused."""
    from lifelike_agility_and_play_b200.parallel import HandOver
    mine = list(_fill(0, 0, 0))
    x = HandOver(_spec(), "cpu")
    x.post(0, mine)
    g = x.gathered(0)
    assert all(a.shape == (1,) + tuple(b.shape) and a.data_ptr() == b.data_ptr() for a, b in zip(g, mine))
    c = HandOver(_spec(), "cpu", own_copy=True)
    c.post(1, mine)
    g = c.gathered(1)
    assert all(torch.equal(a[0], b) and a.data_ptr() != b.data_ptr() for a, b in zip(g, mine))
    assert c.bytes_per_rank == T * N * 7 * 4 + N + N * 3 * 4 + N * 4
    with pytest.raises(ValueError):
        x.post(0, mine[:3])
    with pytest.raises(ValueError):
        x.post(0, [mine[0], mine[1].to(torch.int32)] + mine[2:])
    with pytest.raises(ValueError):
        x.post(0, [mine[0].transpose(0, 1).contiguous()] + mine[1:])
    with pytest.raises(ValueError):
        HandOver(_spec(), "cpu", dst=1)


# ---------------------------------------------------------------------------------------------------------------------- the workers
SLEEP = int(6e8)          # GPU cycles the exchange's side stream sleeps: two more unrolls are queued and run on the worker's stream meanwhile
LEVELS = ["pmc", "epmc", "sepmc"]


def _level(level, n, device, offset=0, clips=5, pool_rows=None):
    """A worker of `level` over n robots on CUDA device `device` (an int) with global env offset `offset`, its first observation and the
    handles to close.  Equal arguments give equal workers."""
    from lifelike_agility_and_play_b200 import _capi as capi
    from lifelike_agility_and_play_b200.model.compile_model import load_model_blob
    from lifelike_agility_and_play_b200.parallel import HierRolloutWorker, RolloutWorker, SepmcRolloutWorker
    from lifelike_agility_and_play_b200.sim_envs.playground_env import INIT_STATE_RUN_0
    lib, blob, dev = capi.load_cuda_library(), load_model_blob(), "cuda:%d" % device
    if level == "pmc":
        from lifelike_agility_and_play_b200.mocap import synthetic_mocap
        from lifelike_agility_and_play_b200.policy import DevicePolicy
        from test_policy import random_weights
        w = random_weights(9)
        w[25] *= 0.05
        w[27][:] = -2.0
        eng = capi.VecEngine(lib, n, blob, synthetic_mocap(clips, seed=2, min_frames=380, max_frames=420), seed=21, device=device, auto_reset=1,
                             global_env_offset=offset)
        pol = DevicePolicy(w, device=device)
        return RolloutWorker(eng, pol, T, dev, seed=5), eng.reset(), [pol, eng]
    from lifelike_agility_and_play_b200.policy_epmc import DeviceHierPolicy, DeviceOpponentPool, DeviceSepmcTrainPolicy, random_weights
    cfg = dict(kp=50.0, kd=0.5, max_tau=16.0, ground_friction=1.0, max_steps=7, seed=5, friction_hi=1.0, auto_reset=1, global_env_offset=offset)
    if level == "epmc":
        w = random_weights(False, 4)
        w[99] = (0.05 * w[99]).astype(np.float32)
        eng = capi.VecEngine(lib, n, blob, None, device=device, env_kind=capi.ENV_EPMC, element_id=3, cmd_freq_lo=25, cmd_freq_hi=40, **cfg)
        eng.set_init_state(INIT_STATE_RUN_0)
        pol = DeviceHierPolicy(w, device=device, train=True)
        return HierRolloutWorker(eng, pol, T, dev, seed=77), eng.reset(), [pol, eng]
    ws = [random_weights(True, s) for s in (4, 5, 8, 9)]
    for x in ws:
        x[149] = (0.05 * x[149]).astype(np.float32)
    eng = capi.VecEngine(lib, n, blob, None, device=device, env_kind=capi.ENV_SEPMC, **cfg)
    eng.set_init_state(INIT_STATE_RUN_0)
    pol = DeviceSepmcTrainPolicy(ws[0], device=device)
    opp = DeviceOpponentPool(ws[1:], device=device, max_rows=pool_rows or n // 2, probs=[0.25, 0.5, 0.25])
    return SepmcRolloutWorker(eng, pol, opp, T, dev, seed=77), eng.reset(), [pol, opp, eng]


def _clone(u):
    from lifelike_agility_and_play_b200.parallel import Unroll
    return Unroll(*(None if x is None else x.clone() for x in u))


def _run(worker, o0, unrolls, xch=None):
    """`unrolls` unrolls; per unroll, clones of what the learner gets: the bare worker's `Unroll` (the primitive level's with its
    bootstrap value) in a list of one, or the exchange's `gathered` (None off the learner rank)."""
    from lifelike_agility_and_play_b200.parallel import Unroll
    worker.start(o0)
    out = []
    for _ in range(unrolls):
        for _ in range(worker.T):
            worker.step()
        u = worker.finish_unroll()
        if xch is None:
            worker.wait()
            out.append([_clone(u if isinstance(u, Unroll) else Unroll(u, None, None, worker.bootstrap_value))])
        else:
            g = xch.gathered(xch.hand_over(u))
            out.append(None if g is None else [_clone(e) for e in g])
    torch.cuda.synchronize()
    return out


def _bits(x):
    return x.view(torch.int32).cpu().numpy() if x.dtype == torch.float32 else x.cpu().numpy()


def _records(level, u):
    from lifelike_agility_and_play_b200.parallel import hier_slab_records, sepmc_slab_records, slab_records
    if level == "pmc":
        return {"records": slab_records(u.slab, bootstrap_value=u.bootstrap_value)}
    if level == "epmc":
        return hier_slab_records(*u)
    return sepmc_slab_records(*u, with_opponent=True)


def _same(level, got, want, what):
    for name, a, b in zip(("slab", "initial_state", "first_mask", "bootstrap_value"), got, want):
        assert (a is None) == (b is None), (what, name)
        if a is not None:
            assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(_bits(a), _bits(b)), (what, name)
    ra, rb = _records(level, got), _records(level, want)
    for k in rb:
        assert np.array_equal(_bits(ra[k]), _bits(rb[k])), (what, k)


def _close(*handles):
    torch.cuda.synchronize()
    for h in handles:
        h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("own_copy", [False, True])
@pytest.mark.parametrize("level", LEVELS)
def test_one_rank_exchange_hands_over_what_the_worker_returns(built, level, own_copy):
    """Three unrolls through UnrollExchange on one rank (no process group) against a bare worker of the same arguments: slab, initial
    state, first mask, bootstrap value and the records built from them bit for bit (the strategic level's with the opponent column).
    Without own_copy the entries are the worker's own views."""
    from lifelike_agility_and_play_b200.parallel import UnrollExchange
    from lifelike_agility_and_play_b200.parallel.trajectory import SCOL_OPPONENT
    n = 40
    bare, o0, h0 = _level(level, n, 0)
    ref = _run(bare, o0, UNROLLS)
    worker, o1, h1 = _level(level, n, 0)
    assert np.array_equal(o0, o1)
    xch = UnrollExchange(worker, own_copy=own_copy)
    got = _run(worker, o1, UNROLLS, xch)
    for k in range(UNROLLS):
        assert len(got[k]) == 1
        _same(level, got[k][0], ref[k][0], "unroll %d" % k)
    if level == "sepmc":
        assert any(int(r[0].slab[:, 0::2, SCOL_OPPONENT].max()) > 0 for r in ref), "no pair played pool model 1 or 2"
    g = xch.gathered((UNROLLS - 1) % 2)
    assert (g[0].slab.data_ptr() == worker.bufs[(UNROLLS - 1) % 2].data_ptr()) != own_copy
    _close(*(h0 + h1))


@pytest.mark.gpu
@pytest.mark.parametrize("level", LEVELS)
def test_worker_waits_for_a_slab_in_flight(built, level):
    """The exchange's side stream sleeps before it copies unroll 0 (the learner rank's own copy); unrolls 1 and 2 are queued meanwhile,
    and unroll 2 goes into unroll 0's slab.  The received copy of unroll 0 (and of unroll 1, handed over behind it) still equals the bare
    worker's: the worker's stream waited for the transfer before it wrote into the slab again."""
    from lifelike_agility_and_play_b200.parallel import UnrollExchange
    n = 40
    bare, o0, h0 = _level(level, n, 0)
    ref = _run(bare, o0, UNROLLS)
    worker, o1, h1 = _level(level, n, 0)
    xch = UnrollExchange(worker, own_copy=True)
    worker.start(o1)
    handed = []
    for k in range(UNROLLS):
        for _ in range(worker.T):
            worker.step()
        u = worker.finish_unroll()
        if k == 0:
            with torch.cuda.stream(xch.core.side):
                torch.cuda._sleep(SLEEP)
        if k < 2:
            handed.append(xch.hand_over(u))
    assert not xch.core.side.query(), "the side stream woke before the unrolls were queued: the ordering was not exercised"
    got = [_clone(xch.gathered(b)[0]) for b in handed]
    torch.cuda.synchronize()
    assert handed == [0, 1]
    for k, g in enumerate(got):
        _same(level, g, ref[k][0], "unroll %d" % k)
    _close(*(h0 + h1))


# -------------------------------------------------------------------------------------------------------------- one NCCL rank per GPU
N_PER = {"pmc": 64, "epmc": 32, "sepmc": 32}          # robots per rank (16 chase-tag pairs at the strategic level)


def _nccl_rank(rank, world, dst, port, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from lifelike_agility_and_play_b200.parallel import UnrollExchange
    out = {}
    for level in LEVELS:
        n = N_PER[level]
        # one clip: the primitive level's prioritized-sampling table is kept per shard (one per actor process, as in the reference), so
        # with several clips the clip drawn at a reset depends on the shard's own episodes; one clip leaves the draws keyed by global id
        worker, o0, handles = _level(level, n, rank, offset=rank * n, clips=1, pool_rows=world * n // 2)
        got = _run(worker, o0, UNROLLS, UnrollExchange(worker, dst=dst))
        if rank == dst:
            out[level] = [[tuple(None if x is None else x.cpu() for x in e) for e in g] for g in got]
        else:
            assert all(g is None for g in got)
        _close(*handles)
    if rank == dst:
        q.put(out)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_nccl_ranks_gather_what_one_process_steps(built):
    """One NCCL rank per GPU (up to 4), the learner rank the last: each rank steps N envs (N/2 pairs) of every level from global env
    rank*N; the learner's gathered unrolls, concatenated over ranks, equal one process stepping world*N envs with the same seeds, bit
    for bit, records included."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two or more GPUs, one NCCL rank each")
    from lifelike_agility_and_play_b200.parallel import Unroll
    world = min(torch.cuda.device_count(), 4)
    dst = world - 1
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 35500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_nccl_rank, args=(r, world, dst, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = q.get(timeout=800)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for level in LEVELS:
        n = world * N_PER[level]
        worker, o0, handles = _level(level, n, 0, clips=1)
        ref = _run(worker, o0, UNROLLS)
        for k in range(UNROLLS):
            ranks = got[level][k]
            assert len(ranks) == world
            cat = Unroll(*(None if ranks[0][f] is None else torch.cat([e[f] for e in ranks], dim=1 if f == 0 else 0).cuda() for f in range(4)))
            _same(level, cat, ref[k][0], "%s unroll %d" % (level, k))
        _close(*handles)
