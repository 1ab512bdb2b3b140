"""world_size-2 gloo test (CPU) of the multi-GPU host logic (hyperqueue_b200/sharded.py): block ranges,
the all-gather of per-group counts and the derived (counts_all, ranks_before), and that tasks ranked
locally + ranks_before reproduce the single-rank assignment.  The device phases are replaced by a numpy
stand-in that follows the same contract (count per group / emit the tasks whose global rank < k[g])."""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import parity as P


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port, n_total, q, seed, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from hyperqueue_b200.sharded import block_range, shard_exchange
    rng = np.random.default_rng(seed)
    cls = rng.integers(0, q, n_total)
    lvl = rng.integers(0, 4, n_total)
    G = 4 * q
    group = lvl * q + cls
    k = np.minimum(np.bincount(group, minlength=G), rng.integers(0, 40, G))     # "solver": k[g] tasks per group
    lo, hi = block_range(n_total, rank, world)
    local_counts = torch.from_numpy(np.bincount(group[lo:hi], minlength=G).astype(np.int32))
    counts_all, before = shard_exchange(local_counts, rank, world)
    assert np.array_equal(counts_all.numpy(), np.bincount(group, minlength=G))
    assert np.array_equal(before.numpy(), np.bincount(group[:lo], minlength=G))
    # local stable rank inside the group + ranks_before = global rank; emit those below k[g]
    g_loc = group[lo:hi]
    order = np.argsort(g_loc, kind="stable")
    rank_in = np.empty(hi - lo, dtype=np.int64)
    starts = np.searchsorted(g_loc[order], np.arange(G))
    rank_in[order] = np.arange(hi - lo) - starts[g_loc[order]]
    chosen = np.nonzero(rank_in + before.numpy()[g_loc] < k[g_loc])[0] + lo
    ret[rank] = chosen.tolist()
    dist.barrier()
    dist.destroy_process_group()


def test_shard_exchange_reproduces_single_rank_selection():
    n_total, q, seed, world = 5000, 6, 3, 2
    mgr = mp.Manager()
    ret = mgr.dict()
    port = _free_port()
    mp.spawn(_worker, args=(world, port, n_total, q, seed, ret), nprocs=world, join=True)
    got = sorted(ret[0] + ret[1])
    rng = np.random.default_rng(seed)
    cls = rng.integers(0, q, n_total); lvl = rng.integers(0, 4, n_total)
    G = 4 * q
    group = lvl * q + cls
    k = np.minimum(np.bincount(group, minlength=G), rng.integers(0, 40, G))
    exp = []
    seen = np.zeros(G, dtype=np.int64)
    for t in range(n_total):
        if seen[group[t]] < k[group[t]]:
            exp.append(t)
        seen[group[t]] += 1
    assert got == exp


def test_block_ranges_cover_everything_in_order():
    from hyperqueue_b200.sharded import block_range
    for n, w in [(10, 3), (1_000_000, 8), (7, 8), (0, 2)]:
        rs = [block_range(n, r, w) for r in range(w)]
        assert rs[0][0] == 0 and rs[-1][1] == n
        assert all(a[1] == b[0] for a, b in zip(rs, rs[1:]))


class _FakeLib:
    """Stand-in for the three exchange set-up entry points: records what the Python plumbing passes around."""

    def __init__(self, rank):
        self.rank = rank
        self.opened = []
        self.attached = None

    def hqs_shard_xbuf(self, ctx, p_own, handle):
        import ctypes as C
        C.cast(p_own, C.POINTER(C.c_void_p))[0] = 0x1000 + self.rank
        for i in range(64):
            handle[i] = (self.rank * 37 + i) % 256
        return 0

    def hqs_ipc_open(self, ctx, handle, p_out):
        import ctypes as C
        hb = bytes(handle)
        self.opened.append(hb)
        C.cast(p_out, C.POINTER(C.c_void_p))[0] = 0x2000 + hb[0]
        return 0

    def hqs_shard_attach(self, ctx, world, rank, ptrs):
        self.attached = (world, rank, [int(ptrs[r] or 0) for r in range(world)])
        return 0


class _FakeSched:
    def __init__(self, rank):
        self._lib, self._ctx = _FakeLib(rank), None

    def _check(self, rc):
        assert rc == 0


def _attach_worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from hyperqueue_b200.sharded import attach_peers
    s = _FakeSched(rank)
    attach_peers(s, rank, world)
    ret[rank] = (s._lib.opened, s._lib.attached)
    dist.barrier()
    dist.destroy_process_group()


def test_peer_handle_exchange_plumbing():
    """attach_peers: every rank must open exactly the other ranks' 64-byte handles, unmodified, and attach with its own
    buffer at its own index (the device side of the exchange is covered on the GPU)."""
    world = 2
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_attach_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
    for rank in range(world):
        opened, attached = ret[rank]
        other = 1 - rank
        assert opened == [bytes((other * 37 + i) % 256 for i in range(64))]
        assert attached[0] == world and attached[1] == rank
        assert attached[2][rank] == 0x1000 + rank and attached[2][other] == 0x2000 + (other * 37) % 256


class _FakeMirror:
    """The host-side fields of GpuScheduler that ShardedScheduler.tasks_finished touches (no device)."""

    def __init__(self, n_local, W, R):
        self._task_worker = np.full(n_local, -1, dtype=np.int64)
        self._task_class = np.zeros(n_local, dtype=np.uint32)
        self._task_variant = np.zeros(n_local, dtype=np.uint8)
        self._amount_tab = np.zeros((2, 8, R), dtype=np.uint64)
        self._amount_tab[0, 0] = [10000, 0]
        self._amount_tab[1, 0] = [20000, 5000]
        self._all_tab = np.zeros((2, 8, R), dtype=bool)
        self.total = np.full((W, R), 80000, dtype=np.uint64)
        self.free = self.total.copy()


def _finished_worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from hyperqueue_b200.sharded import ShardedScheduler, block_range
    n_total, W, R = 10, 3, 2
    lo, hi = block_range(n_total, rank, world)
    sh = ShardedScheduler.__new__(ShardedScheduler)
    sh.s, sh.rank, sh.world, sh.group, sh.lo, sh.hi, sh.device = _FakeMirror(hi - lo, W, R), rank, world, None, lo, hi, torch.device("cpu")
    # the replicated solve placed global task t of class t % 2 on worker t % 3: every rank saw the same free vectors
    for t in range(n_total):
        amount = sh.s._amount_tab[t % 2, 0]
        sh.s.free[t % 3] -= amount
    a = np.zeros(hi - lo, dtype=[("task", "<u4"), ("worker", "<u2"), ("variant", "u1"), ("kind", "u1")])
    a["task"] = np.arange(hi - lo); a["worker"] = (np.arange(lo, hi) % 3)
    sh.s._task_class[:] = np.arange(lo, hi) % 2
    sh._record(a)
    sh.tasks_finished(np.arange(n_total))          # the same global list on every rank
    ret[rank] = sh.s.free.tobytes()
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_tasks_finished_returns_resources_on_every_rank():
    """Each rank knows where ITS tasks ran; the amounts to give back are summed over the ranks, so the replicated free
    vectors stay identical and return to the totals."""
    world = 2
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_finished_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
    total = np.full((3, 2), 80000, dtype=np.uint64)
    for rank in range(world):
        assert np.array_equal(np.frombuffer(ret[rank], dtype=np.uint64).reshape(3, 2), total)


def _mirror_with_unlimited(n_local, W, R):
    """_FakeMirror with resource 1 of worker 2 unlimited (HQS_AMOUNT_MAX), and the fields the record bookkeeping reads."""
    from hyperqueue_b200 import _lib as L
    s = _FakeMirror(n_local, W, R)
    s.worker_ids = np.arange(W, dtype=np.uint32)
    s._pf_worker = np.full(n_local, -1, dtype=np.int64)
    s.total[2, 1] = L.HQS_AMOUNT_MAX
    s.free = s.total.copy()
    return s


def _finish_on_unlimited(rank, world):
    """Global task t of class t % 2 ran on worker t % 3; task 5 requested resource 1 of worker 2, whose total is
    HQS_AMOUNT_MAX (a tick leaves it unlimited).  All tasks finish; returns the rank's free vectors afterwards."""
    from hyperqueue_b200 import _lib as L
    from hyperqueue_b200.sharded import ShardedScheduler, block_range
    n_total, W, R = 10, 3, 2
    lo, hi = block_range(n_total, rank, world)
    sh = ShardedScheduler.__new__(ShardedScheduler)
    sh.s, sh.rank, sh.world, sh.group, sh.lo, sh.hi, sh.device = (_mirror_with_unlimited(hi - lo, W, R), rank, world, None,
                                                                   lo, hi, torch.device("cpu"))
    for t in range(n_total):
        fr = sh.s.free[t % 3]
        sh.s.free[t % 3] = np.where(fr == np.uint64(L.HQS_AMOUNT_MAX), fr, fr - sh.s._amount_tab[t % 2, 0])
    a = np.zeros(hi - lo, dtype=[("task", "<u4"), ("worker", "<u2"), ("variant", "u1"), ("kind", "u1")])
    a["task"] = np.arange(hi - lo); a["worker"] = (np.arange(lo, hi) % 3)
    sh.s._task_class[:] = np.arange(lo, hi) % 2
    sh._record(a)
    sh.tasks_finished(np.arange(n_total))
    return sh.s.free


def _unlimited_worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ret[rank] = _finish_on_unlimited(rank, world).tobytes()
    dist.barrier()
    dist.destroy_process_group()


def _totals_with_unlimited():
    from hyperqueue_b200 import _lib as L
    total = np.full((3, 2), 80000, dtype=np.uint64)
    total[2, 1] = L.HQS_AMOUNT_MAX
    return total


def test_sharded_tasks_finished_keeps_unlimited_amounts_in_a_world_of_one():
    """A task that requested resource 1 finishes on the worker whose resource 1 is HQS_AMOUNT_MAX: it stays MAX (adding the
    returned amount onto it would wrap to amount - 1)."""
    assert np.array_equal(_finish_on_unlimited(0, 1), _totals_with_unlimited())


def test_sharded_tasks_finished_keeps_unlimited_amounts_on_every_rank():
    """The same over gloo with two ranks: the task on the unlimited worker belongs to rank 1, and both ranks keep MAX."""
    world = 2
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_unlimited_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
    for rank in range(world):
        assert np.array_equal(np.frombuffer(ret[rank], dtype=np.uint64).reshape(3, 2), _totals_with_unlimited())
