"""The strategic level's learner-seat hand-over: `UnrollExchange(worker, learner_seat_only=True)` packs the seat-0 records of a
`[T, 2P, 984]` slab into a `[T, P, 984]` send buffer (csrc/llq_seat_pack.cu, `pack_learner_seat`) and sends that instead of the slab;
`sepmc_slab_records(..., learner_seat_only=True)` reads it.

CPU: the records of a learner-seat slab equal those of the full slab bit for bit, leaf by leaf; slabs on the wrong side of the flag
and the other levels' workers are refused; the C entry refuses null, misaligned, overlapping and out-of-range arguments before it
touches a device; the pack kernel neither spills nor uses local memory.
GPU (-m gpu): the pack kernel against `slab[:, 0::2]` bit for bit with NaNs and sentinels in the seat-1 rows; a worker with the
learner-seat exchange against a twin with the default one over three unrolls (its own slabs, what is gathered, the records); the
worker's stream waits for a slab's pack and transfer before it writes into that slab again; with two or more GPUs, NCCL ranks."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from lifelike_agility_and_play_b200.parallel.trajectory import SCOL_DONE, SCOL_OPPONENT, SCOL_REWARD, SEPMC_TRAJ_WIDTH
from test_unroll_exchange import SLEEP, T, UNROLLS, _bits, _clone, _close, _level, _run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W = SEPMC_TRAJ_WIDTH
LLQ_EINVAL = -1
CANARY = 0x7FBADBAD


@pytest.fixture(scope="module")
def lib(built):
    from lifelike_agility_and_play_b200.policy import POLICY_LIB_PATH
    lib = C.CDLL(POLICY_LIB_PATH)
    lib.llq_seat_pack.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]
    lib.llq_seat_pack_last_error.restype = C.c_char_p
    return lib


# ------------------------------------------------------------------------------------------------------------------------ the records
def _slab(T_, P, seed):
    """A random [T, 2P, 984] slab: done flags equal on both seats and set at t = 0 and t = T-1 for pair 0, integral codes and opponent
    indices, NaNs in the seat-1 columns the learner never reads; with its initial state, first mask and bootstrap value."""
    rng = np.random.default_rng(seed)
    s = rng.standard_normal((T_, 2 * P, W)).astype(np.float32)
    d = (rng.random((T_, P)) < 0.3).astype(np.float32)
    d[0, 0] = d[T_ - 1, 0] = 1.0
    s[:, 0::2, SCOL_DONE] = s[:, 1::2, SCOL_DONE] = d
    s[:, :, SCOL_REWARD] = rng.random((T_, 2 * P)).astype(np.float32)
    s[:, 0::2, SCOL_OPPONENT] = rng.integers(0, 64, (T_, P)).astype(np.float32)
    s[:, 1::2, 979:981] = np.nan
    init = torch.from_numpy(rng.standard_normal((P, 192)).astype(np.float32))
    first = torch.from_numpy((rng.random(P) < 0.5).astype(np.uint8))
    boot = torch.from_numpy(rng.standard_normal(P).astype(np.float32))
    return torch.from_numpy(s), init, first, boot


@pytest.mark.parametrize("T_", [1, 5])
@pytest.mark.parametrize("P", [1, 3, 64])
def test_learner_seat_records_equal_the_full_slab(T_, P):
    from lifelike_agility_and_play_b200.parallel import sepmc_slab_records
    s, init, first, boot = _slab(T_, P, 7 * P + T_)
    want = sepmc_slab_records(s, init, first, boot, with_opponent=True)
    got = sepmc_slab_records(s[:, 0::2].contiguous(), init, first, boot, with_opponent=True, learner_seat_only=True)
    assert list(got) == list(want) and list(want)[-1] == "opponent"
    for k in want:
        assert got[k].dtype == want[k].dtype and got[k].shape == want[k].shape, k
        assert np.array_equal(_bits(got[k]), _bits(want[k])), k
    assert int(want["opponent"].max()) > 0 or P == 1


def test_records_refuse_a_slab_on_the_wrong_side_of_the_flag():
    from lifelike_agility_and_play_b200.parallel import sepmc_slab_records
    s, init, first, boot = _slab(5, 4, 1)
    packed = s[:, 0::2].contiguous()
    for bad in (s, packed[:, :3], packed[:, :, :936], packed[0]):
        with pytest.raises(AssertionError):
            sepmc_slab_records(bad, init, first, boot, learner_seat_only=True)
    for bad in (packed, s[:, :6], s[:, :7]):         # a learner-seat slab (P = 4: an even row count) without the flag
        with pytest.raises(AssertionError):
            sepmc_slab_records(bad, init, first, boot)


def test_learner_seat_only_is_refused_off_the_strategic_level():
    """Device-free: the workers are bare objects; the exchange refuses them before it reads anything from them."""
    from lifelike_agility_and_play_b200.parallel import HierRolloutWorker, RolloutWorker, UnrollExchange
    for cls in (RolloutWorker, HierRolloutWorker):
        with pytest.raises(ValueError, match="learner_seat_only"):
            UnrollExchange(cls.__new__(cls), learner_seat_only=True)
    with pytest.raises(ValueError):
        UnrollExchange(object(), learner_seat_only=True)


# -------------------------------------------------------------------------------------------------------------- the pack entry, no GPU
def test_pack_entry_refuses_bad_arguments_before_the_device(lib):
    """Fake addresses: every refusal below comes before the first CUDA call, so none of them is dereferenced."""
    a, b = 0x10000000, 0x20000000                     # 16-byte aligned, far apart
    cases = [(None, b, 5, 3, b"null"), (a, None, 5, 3, b"null"), (a + 4, b, 5, 3, b"aligned"), (a, b + 8, 5, 3, b"aligned"),
             (a, b, 0, 3, b"positive"), (a, b, 5, 0, b"positive"), (a, b, -1, 3, b"positive"), (a, b, 1 << 40, 1 << 20, b"one launch"),
             (a, a + 16 * 246, 5, 3, b"overlaps"), (a + 16 * 246 * 14, a, 5, 3, b"overlaps")]     # the output: 15 records
    for slab, out, steps, pairs, msg in cases:
        assert lib.llq_seat_pack(slab, out, steps, pairs, None) == LLQ_EINVAL, (slab, out, steps, pairs)
        assert msg in lib.llq_seat_pack_last_error(), (lib.llq_seat_pack_last_error(), msg)


def test_pack_wrapper_refuses_wrong_tensors():
    from lifelike_agility_and_play_b200.parallel import pack_learner_seat
    s = torch.zeros((2, 6, W))
    for slab, out in ((s, torch.zeros((2, 3, W))), (s, torch.zeros((2, 2, W))), (s[:, :, :936], torch.zeros((2, 3, 936))),
                      (s.double(), torch.zeros((2, 3, W), dtype=torch.float64)), (s[:, 0::2], torch.zeros((2, 1, W))), (s.numpy(), None)):
        with pytest.raises(ValueError):
            pack_learner_seat(slab, out)


def test_pack_kernel_has_no_spills_or_local_memory():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "lifelike_agility_and_play_b200", "csrc", "llq_seat_pack.cu")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c", "-o", os.devnull, src],
                         capture_output=True, text=True, check=True).stderr
    blocks = [b for b in out.split("Compiling entry function")[1:] if "seat_pack_kernel" in b.split("\n")[0]]
    assert len(blocks) == 1, out
    assert re.search(r"0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", blocks[0]), blocks[0]
    assert int(re.search(r"Used (\d+) registers", blocks[0]).group(1)) <= 32, blocks[0]


# ------------------------------------------------------------------------------------------------------------------- the pack kernel
@pytest.mark.gpu
@pytest.mark.parametrize("T_", [1, 128])
@pytest.mark.parametrize("P", [1, 3, 4096])
def test_pack_kernel_copies_seat_zero_bit_for_bit(lib, T_, P):
    """Random bit patterns in seat 0 (NaNs and infinities included), quiet and signalling NaNs, -inf and a sentinel in seat 1, a canary
    output with 256 more floats past its end; on a side stream.  Then the refusals of device arguments leave the output untouched."""
    from lifelike_agility_and_play_b200.parallel import pack_learner_seat
    g = torch.Generator(device="cuda").manual_seed(T_ * 10007 + P)
    s = torch.randint(-2 ** 31, 2 ** 31 - 1, (T_, 2 * P, W), dtype=torch.int32, device="cuda", generator=g)
    s1 = s[:, 1::2]
    s1[:, :, 0::4], s1[:, :, 1::4], s1[:, :, 2::4], s1[:, :, 3::4] = 0x7FC00001, CANARY, -8388608, 0x7F800001
    buf = torch.full((T_ * P * W + 256,), CANARY, dtype=torch.int32, device="cuda")
    out = buf[:T_ * P * W].view(T_, P, W)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        pack_learner_seat(s.view(torch.float32), out.view(torch.float32), side)
    torch.cuda.current_stream().wait_stream(side)
    assert torch.equal(out, s[:, 0::2])
    assert bool((buf[T_ * P * W:] == CANARY).all())
    # refused before any launch: the output keeps what it holds
    out.fill_(CANARY)
    host = np.zeros(W, np.float32)                   # refused before anything reads it
    for src, dst in ((s.data_ptr() + 4, out.data_ptr()), (s.data_ptr(), out.data_ptr() + 4), (host.ctypes.data, out.data_ptr()),
                     (s.data_ptr(), s.data_ptr() + 16 * 246)):
        assert lib.llq_seat_pack(src, dst, T_, P, None) == LLQ_EINVAL, lib.llq_seat_pack_last_error()
    torch.cuda.synchronize()
    assert bool((buf == CANARY).all())
    del s, buf, out
    torch.cuda.empty_cache()


# ----------------------------------------------------------------------------------------------------------------- the worker's exchange
def _seat0(u):
    """What the learner-seat exchange must gather from the worker's full `Unroll`: seat 0 of the slab, the rest as it is."""
    from lifelike_agility_and_play_b200.parallel import Unroll
    return Unroll(u.slab[:, 0::2].contiguous(), u.initial_state, u.first_mask, u.bootstrap_value)


def _same_seat(got, full, what):
    """`got` (a learner-seat `Unroll`) against the full-slab `Unroll` `full`: tensors bit for bit, records leaf by leaf."""
    from lifelike_agility_and_play_b200.parallel import sepmc_slab_records
    for name, a, b in zip(("slab", "initial_state", "first_mask", "bootstrap_value"), got, _seat0(full)):
        assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(_bits(a), _bits(b)), (what, name)
    ra = sepmc_slab_records(*got, with_opponent=True, learner_seat_only=True)
    rb = sepmc_slab_records(*full, with_opponent=True)
    assert list(ra) == list(rb)
    for k in rb:
        assert np.array_equal(_bits(ra[k]), _bits(rb[k])), (what, k)


@pytest.mark.gpu
@pytest.mark.parametrize("own_copy", [True, False])
def test_learner_seat_exchange_hands_over_seat_zero(built, own_copy):
    """Three unrolls of a worker with the learner-seat exchange against a twin with the default exchange (own_copy=True): the worker's
    own slabs, both seats, are the twin's bit for bit (the pack adds no hazard to the slab's reuse); what is gathered is seat 0 of the
    twin's unroll with its state, mask and bootstrap value, records included; bytes_per_rank counts the learner seat alone."""
    from lifelike_agility_and_play_b200.parallel import UnrollExchange
    n = 40
    P = n // 2
    twin, o0, h0 = _level("sepmc", n, 0)
    ref = _run(twin, o0, UNROLLS, UnrollExchange(twin, own_copy=True))
    worker, o1, h1 = _level("sepmc", n, 0)
    assert np.array_equal(o0, o1)
    xch = UnrollExchange(worker, own_copy=own_copy, learner_seat_only=True)
    assert xch.bytes_per_rank == T * P * W * 4 + P * 192 * 4 + P + P * 4
    worker.start(o1)
    for k in range(UNROLLS):
        for _ in range(worker.T):
            worker.step()
        u = worker.finish_unroll()
        g = xch.gathered(xch.hand_over(u))
        assert len(g) == 1 and tuple(g[0].slab.shape) == (T, P, W)
        got = _clone(g[0])
        worker.wait()
        mine = _clone(u)
        torch.cuda.synchronize()
        assert np.array_equal(_bits(mine.slab), _bits(ref[k][0].slab)), "unroll %d: the worker's own slab" % k
        _same_seat(got, ref[k][0], "unroll %d" % k)
        assert (g[0].slab.data_ptr() == xch.send.data_ptr()) != own_copy
    assert any(int(r[0].slab[:, 0::2, SCOL_OPPONENT].max()) > 0 for r in ref), "no pair played pool model 1 or 2"
    _close(*(h0 + h1))


@pytest.mark.gpu
def test_worker_waits_for_a_slab_in_flight_learner_seat(built):
    """As test_unroll_exchange.py::test_worker_waits_for_a_slab_in_flight with the learner-seat exchange: the side stream sleeps before
    it packs unroll 0; unrolls 1 and 2 are queued meanwhile, and unroll 2 goes into unroll 0's slab.  The gathered unrolls 0 and 1 still
    equal seat 0 of the bare worker's: the worker's stream waited for the pack and the transfer before it wrote into the slab again, and
    the second pack waited for the first transfer out of the send buffer."""
    from lifelike_agility_and_play_b200.parallel import UnrollExchange
    n = 40
    bare, o0, h0 = _level("sepmc", n, 0)
    ref = _run(bare, o0, UNROLLS)
    worker, o1, h1 = _level("sepmc", n, 0)
    xch = UnrollExchange(worker, own_copy=True, learner_seat_only=True)
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
        _same_seat(g, ref[k][0], "unroll %d" % k)
    _close(*(h0 + h1))


# -------------------------------------------------------------------------------------------------------------- one NCCL rank per GPU
N_PER = 32                  # robots per rank: 16 chase-tag pairs


def _nccl_rank(rank, world, dst, port, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from lifelike_agility_and_play_b200.parallel import UnrollExchange
    worker, o0, handles = _level("sepmc", N_PER, rank, offset=rank * N_PER, clips=1, pool_rows=world * N_PER // 2)
    xch = UnrollExchange(worker, dst=dst, learner_seat_only=True)
    worker.start(o0)
    local, gathered = [], []
    for _ in range(UNROLLS):
        for _ in range(worker.T):
            worker.step()
        u = worker.finish_unroll()
        g = xch.gathered(xch.hand_over(u))
        worker.wait()
        local.append(tuple(x.cpu() for x in _seat0(u)))
        gathered.append(None if g is None else [tuple(x.cpu() for x in e) for e in g])
    q.put((rank, local, gathered))
    _close(*handles)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_nccl_ranks_gather_learner_seats(built):
    """One NCCL rank per GPU (up to 4), the learner rank the last, learner-seat exchange: the learner's gathered unroll of rank r is
    seat 0 of rank r's own finished unroll, with its state, mask and bootstrap value, bit for bit; the other ranks gather None."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two or more GPUs, one NCCL rank each")
    world = min(torch.cuda.device_count(), 4)
    dst = world - 1
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 36500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_nccl_rank, args=(r, world, dst, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = {}
    for _ in range(world):
        rank, local, gathered = q.get(timeout=800)
        res[rank] = (local, gathered)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for r in range(world):
        assert all(g is None for g in res[r][1]) == (r != dst)
    for k in range(UNROLLS):
        ranks = res[dst][1][k]
        assert len(ranks) == world
        for r in range(world):
            for name, a, b in zip(("slab", "initial_state", "first_mask", "bootstrap_value"), ranks[r], res[r][0][k]):
                assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(_bits(a), _bits(b)), (k, r, name)
