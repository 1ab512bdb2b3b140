"""Handle compaction over a sharded task graph (hqs_shard_graph_compact): every rank renumbers the replicated graph alike and
keeps its own tasks.

The harness is the one of tests/test_gpu_sharded_graph.py (a reference context fed the same calls through the single-context
graph API, and 2 or 3 HQS_CREATE_SHARE_DEVICE contexts of one GPU as ranks; fused ticks use 2, as each context's cooperative
tick kernel takes half of the SMs), with ranges that follow the compactions.  Where
the ranks compact, the reference compacts with hqs_handles_compact and the same keep list.  After every compaction every
rank's old_of_new equals the reference's and its new range is [new(lo), new(hi)) (the last rank's ends at n_total); after
every call and every tick each rank's keys equal the reference's over its range, hqs_graph_debug out[0..2] is equal on every
rank and to the reference's, and out[3] sums to the reference's."""
import ctypes as C

import numpy as np
import pytest
import torch

import parity as P
import test_gpu_ready_set as RS
import test_gpu_sharded_graph as SG
from test_gpu_sharded_graph import E_INVALID, E_STATE, VALID, _ptr, csr, prio

pytestmark = pytest.mark.gpu


class Ranks(SG.Ranks):
    """SG.Ranks whose ranges change with the compactions."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.ranges = [(self.cuts[r], self.cuts[r + 1]) for r in range(self.world)]

    def rng_of(self, r):
        return self.ranges[r]

    def compact_call(self, d, keep):
        ptr, k, rng = C.POINTER(C.c_uint32)(), C.c_uint32(0), np.zeros(2, np.uint32)
        rc = d.lib.hqs_shard_graph_compact(d.ctx, keep.size, _ptr(keep), C.byref(ptr), C.byref(k), self.L.ptr(rng))
        old = np.ctypeslib.as_array(ptr, shape=(k.value,)).copy() if k.value else np.zeros(0, np.uint32)
        return rc, old, (int(rng[0]), int(rng[1]))

    def compact(self, keep, label="compact"):
        keep = np.ascontiguousarray(keep, np.uint32)
        ptr, k = C.POINTER(C.c_uint32)(), C.c_uint32(0)
        self.ref.ok(self.ref.lib.hqs_handles_compact(self.ref.ctx, keep.size, _ptr(keep), C.byref(ptr), C.byref(k)))
        want = np.ctypeslib.as_array(ptr, shape=(k.value,)).copy() if k.value else np.zeros(0, np.uint32)

        def new(h):
            return self.n_total if h == self.n_total else int(np.searchsorted(want, h))

        for r, d in enumerate(self.ranks):
            rc, old, rng = self.compact_call(d, keep)
            assert rc == 0, (label, r, d.lib.hqs_last_error(d.ctx))
            assert np.array_equal(old, want), (label, r)
            lo, hi = self.ranges[r]
            assert rng == (new(lo), new(hi)), (label, r, rng)
            self.ranges[r] = rng
        assert self.ranges[0][0] == 0 and self.ranges[-1][1] == self.n_total, label
        assert all(a[1] == b[0] for a, b in zip(self.ranges, self.ranges[1:])), (label, self.ranges)
        kept = want.astype(np.int64)
        for name, fill in (("cls", 0), ("pfw", -1)):
            a = getattr(self, name)
            b = np.full_like(a, fill)
            b[: kept.size] = a[kept]
            setattr(self, name, b)
        self.check(label)
        return want


def make(n_total, world, split, q=2, **kw):
    return Ranks(n_total, SG.splits(n_total, world)[split], q, **kw)


# random sequences --------------------------------------------------------------------------------------------------------
def _random(s, rng, steps, every=4):
    """Pushes (fresh handles from the freed tail after each compaction), cancels across ranks, removes, sharded ticks with
    proactive filling, finishes, and a compaction every `every` steps: the first keeps nothing, the second keeps removed
    handles, the others keep random handles.  Returns how many handles were pushed."""
    q, n_total = s.q, s.n_total
    next_h, free_handles, removed, job, pushed, compactions = 0, [], [], 0, 0, 0
    for step in range(steps):
        live = np.nonzero(s.ref.keys() & VALID)[0]
        k = int(rng.integers(1, 40))
        reuse = [free_handles.pop(int(rng.integers(0, len(free_handles)))) for _ in range(min(len(free_handles), k // 2))]
        fresh = list(range(next_h, min(next_h + k - len(reuse), n_total)))
        next_h += len(fresh)
        hs = reuse + fresh
        if hs:
            if rng.random() < 0.5:
                hs = sorted(hs)
            deps = []
            for i, x in enumerate(hs):
                pool = list(live[-80:]) + hs[:i] + hs[i + 1: i + 3]
                ds = {int(pool[j]) for j in rng.integers(0, len(pool), size=int(rng.integers(0, 4)))} - {x} if pool else set()
                deps.append(sorted(ds))
            s.push(hs, rng.integers(0, q, size=len(hs)), [prio(int(rng.integers(0, 4)), job % 7)] * len(hs), *csr(deps),
                   label=f"push {step}")
            job += 1
            pushed += len(hs)
        live = np.nonzero(s.ref.keys() & VALID)[0]
        if rng.random() < 0.25 and live.size:
            # the lowest and the highest live handles: a closure that crosses the rank boundaries
            gone = s.cancel([int(live[0]), int(live[-1])], f"cancel {step}")
            free_handles += gone
        elif rng.random() < 0.25 and live.size:
            victim = [int(x) for x in rng.choice(live, size=min(4, live.size), replace=False)]
            s.remove(victim, f"remove {step}")
            free_handles += victim
            removed += victim
        exp = s.tick(f"tick {step}")
        done = exp[exp["kind"] != 1]["task"]
        fin = [int(x) for x in done if rng.random() < 0.8]
        if fin:
            s.finished(fin + fin[:1], f"finish {step}")
            free_handles += fin
        if step % every == every - 1 or next_h >= n_total - 40:
            n = s.ref.keys().size
            if compactions == 0:
                keep = []
            elif compactions == 1 and removed:
                keep = [x for x in removed if x < n][:5]
            else:
                keep = [int(x) for x in rng.integers(0, max(n, 1), size=int(rng.integers(0, 6)))] if n else []
            old = s.compact(keep, f"compact {step}")
            if compactions == 1 and keep:
                assert set(keep) <= set(old.tolist())
            compactions += 1
            next_h, free_handles, removed = int(old.size), [], []
    assert compactions >= 2
    return pushed


@pytest.mark.parametrize("world,split,fused,seed", [(2, "even", False, 0), (3, "even", False, 1), (3, "first", False, 2),
                                                    (3, "last", False, 3), (2, "even", True, 4), (2, "last", True, 5)])
def test_random_sequences_with_compactions(world, split, fused, seed):
    n_total = 1500
    s = make(n_total, world, split, q=3, fused=fused, prefill=RS.PREFILL)
    try:
        _random(s, np.random.default_rng(900 + seed), 36)
    finally:
        s.close()


@pytest.mark.parametrize("world,split,fused", [(3, "even", False), (2, "even", True)])
def test_run_past_n_total(world, split, fused):
    n_total = 600
    s = make(n_total, world, split, q=3, fused=fused, prefill=RS.PREFILL)
    try:
        pushed = _random(s, np.random.default_rng(77), 110, every=6)
        assert pushed >= 3 * n_total, pushed
    finally:
        s.close()


# rejections, state rules, cost ---------------------------------------------------------------------------------------------
def _snapshot(s):
    return [(d.keys(), s.debug(d), s.ranges[r]) for r, d in enumerate(s.ranks)]


def _same(a, b):
    return all(np.array_equal(x[0], y[0]) and x[1] == y[1] and x[2] == y[2] for x, y in zip(a, b))


@pytest.mark.parametrize("world,split", [(2, "even"), (3, "last")])
def test_rejections_leave_every_rank_unchanged(world, split):
    s = make(64, world, split, q=2)
    try:
        s.push([0, 1, 2, 40], [0, 1, 0, 1], [prio(1)] * 4, *csr([[], [0], [0, 1], [2]]))
        s.remove([1])
        before = _snapshot(s)
        for r, d in enumerate(s.ranks):
            rc, old, rng = s.compact_call(d, np.array([3, 64], np.uint32))          # a keep entry >= n_total
            assert rc == E_INVALID and old.size == 0 and rng == s.ranges[r]
            ptr, k, out = C.POINTER(C.c_uint32)(), C.c_uint32(0), np.zeros(2, np.uint32)
            assert d.lib.hqs_shard_graph_compact(d.ctx, 2, None, C.byref(ptr), C.byref(k), s.L.ptr(out)) == E_INVALID
        assert _same(before, _snapshot(s))
        # a pending tick: hqs_shard_count, then hqs_shard_solve_emit on every rank, and nothing is fetched yet
        L, W = s.L, s.W
        w = np.zeros(W, dtype=L.worker_dtype)
        w["worker_id"] = np.arange(W)
        w["remaining_time_ms"] = L.HQS_TIME_INF
        free = RS.W_TOTAL.copy()
        ng = C.c_uint32(0)
        for d, cnt in zip(s.ranks, s.counts):
            d.ok(d.lib.hqs_shard_count(d.ctx, W, L.ptr(w), L.ptr(free), L.ptr(RS.W_TOTAL), None, C.c_void_p(cnt.data_ptr()),
                                       cnt.numel(), C.byref(ng)))
        torch.cuda.synchronize()
        allc = torch.stack(s.counts).sum(0, dtype=torch.int32)
        before_r = [torch.stack(s.counts[:r]).sum(0, dtype=torch.int32) if r else torch.zeros_like(allc) for r in range(s.world)]
        torch.cuda.synchronize()
        for d, b in zip(s.ranks, before_r):
            d.ok(d.lib.hqs_shard_solve_emit(d.ctx, C.c_void_p(allc.data_ptr()), C.c_void_p(b.data_ptr()), 64))
        for d in s.ranks:
            assert s.compact_call(d, np.zeros(0, np.uint32))[0] == E_STATE
        for d in s.ranks:
            out = np.zeros(64, dtype=L.assignment_dtype)
            d.ok(d.lib.hqs_tick_fetch(d.ctx, 64, L.ptr(out), C.byref(ng), None))
        s.ref.tick(RS.W_TOTAL.copy(), None, 64)                                     # the reference assigns the same tasks
        assert [x[2] for x in _snapshot(s)] == [x[2] for x in before]
        # hqs_handles_compact is still refused on a sharded graph context
        for d in s.ranks:
            ptr, k = C.POINTER(C.c_uint32)(), C.c_uint32(0)
            assert d.lib.hqs_handles_compact(d.ctx, 0, None, C.byref(ptr), C.byref(k)) == E_STATE
        s.compact([1], "after the rejections")                                      # keeps the removed handle 1
        assert s.ranges[-1][1] == 64
    finally:
        s.close()


def test_state_rules():
    from hyperqueue_b200 import _lib as L
    ptr, k, rng = C.POINTER(C.c_uint32)(), C.c_uint32(0), np.zeros(2, np.uint32)
    plain = RS.Dev(0)
    attached = RS.Dev(L.HQS_CREATE_SHARE_DEVICE)
    try:
        for d in (plain, attached):
            d.classes(1)
        assert plain.lib.hqs_shard_graph_compact(plain.ctx, 0, None, C.byref(ptr), C.byref(k), L.ptr(rng)) == E_STATE
        # a sharded ready set without a graph has no replicated VALID bits
        xb = (C.c_void_p * 1)()
        p = C.c_void_p()
        attached.ok(attached.lib.hqs_shard_xbuf(attached.ctx, C.byref(p), None))
        xb[0] = p
        attached.ok(attached.lib.hqs_shard_attach(attached.ctx, 1, 0, xb))
        assert attached.lib.hqs_shard_graph_compact(attached.ctx, 0, None, C.byref(ptr), C.byref(k), L.ptr(rng)) == E_STATE
    finally:
        plain.close()
        attached.close()


def _compact_cost(n_total):
    s = make(n_total, 2, "even", q=2)
    try:
        h = np.concatenate([np.arange(0, 64), np.arange(n_total - 64, n_total)])
        s.push(h, h % 2, [prio(1)] * h.size, *csr([[]] * 64 + [[int(x)] for x in range(64)]))
        s.finished(h[:8])
        d = s.ranks[1]
        before = d.stats()["kernel_launches"]
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            rc, old, _ = s.compact_call(d, np.zeros(0, np.uint32))
        assert rc == 0 and old.size == 120
        launches = d.stats()["kernel_launches"] - before
        names = [e.name for e in prof.events()]
        syncs = names.count("cudaStreamSynchronize")     # the call's own waits (the profiler adds a device synchronise)
        seen_api = any(x.startswith("cuda") for x in names)
        # the other rank compacts too, so that the ranks stay alike
        assert s.compact_call(s.ranks[0], np.zeros(0, np.uint32))[0] == 0
        return launches, syncs, seen_api
    finally:
        s.close()


def test_cost_does_not_depend_on_n_total():
    small, big = _compact_cost(4096), _compact_cost(1 << 22)
    assert small[0] == big[0] and small[0] <= 9, (small, big)
    for launches, syncs, seen in (small, big):
        if seen:                                    # the profiler saw the CUDA runtime calls of the library
            assert 1 <= syncs <= 2, syncs


# ShardedScheduler.compact_handles end to end -----------------------------------------------------------------------------
@pytest.mark.parametrize("p2p", [False, True])
def test_sharded_scheduler_compact_handles_as_one_rank(p2p):
    from hyperqueue_b200.sharded import ShardedScheduler
    n_total = 1200
    wl = P.make_independent(n_total, 16, 4, seed=5)
    ref = P.gpu_scheduler(wl, add_tasks=False)
    base = P.gpu_scheduler(wl, add_tasks=False)
    sh = ShardedScheduler(base, 0, 1, n_total, torch.device("cuda", 0), p2p=p2p)
    sh.graph_init()
    sh.set_prefill(*RS.PREFILL)
    ref.set_prefill(*RS.PREFILL)
    rng = np.random.default_rng(21)
    cls = np.ascontiguousarray(wl.task_class, np.uint32)
    next_h, pushed, compactions = 0, 0, 0
    try:
        for tick in range(120):
            k = min(int(rng.integers(5, 30)), n_total - next_h)
            if k > 0:
                h = np.arange(next_h, next_h + k)
                keys = _keys(ref)
                live = np.nonzero(keys & VALID)[0]
                deps = [sorted({int(x) for x in rng.choice(live, size=min(live.size, int(rng.integers(0, 3))), replace=False)})
                        if live.size else [] for _ in range(k)]
                off, flat = csr(deps)
                c = cls[h % cls.size]
                p = np.array([prio(int(u), tick % 5) for u in rng.integers(0, 3, k)], np.uint64)
                assert sh.submit_tasks(h, c, p, off, flat) == ref.submit_tasks(h, c, p, off, flat)
                next_h += k
                pushed += k
            got, fa = sh.run_scheduling()
            exp = ref.run_scheduling()
            assert np.array_equal(got, exp.assignments) and np.array_equal(fa, exp.free_after), tick
            pf = exp.assignments[exp.assignments["kind"] == 1]
            if pf.size and tick % 3 == 0:
                t = int(pf["task"][-1])
                sh.on_task_running_prefilled(t, 0)
                ref.on_task_running_prefilled(t, 0)
            done = exp.assignments[exp.assignments["kind"] != 1]["task"]
            fin = done[:-1]
            assert np.array_equal(sh.graph_tasks_finished(fin), ref.graph_tasks_finished(fin))
            victims = done[-1:]
            g1, m1 = sh.graph_cancel_tasks(victims)
            g2, m2 = ref.graph_cancel_tasks(victims)
            assert np.array_equal(g1, g2) and m1 == m2
            assert np.array_equal(base.free, ref.free)
            if tick % 5 == 4 or next_h > n_total - 60:
                o1 = sh.compact_handles()
                o2 = ref.compact_handles()
                assert np.array_equal(o1, o2), tick
                assert (sh.lo, sh.hi) == (0, n_total)
                next_h = int(o1.size)
                compactions += 1
                assert np.array_equal(_keys(base), _keys(ref)), tick
                for a, b in ((base._task_worker, ref._task_worker), (base._pf_worker, ref._pf_worker)):
                    assert np.array_equal(a[: o1.size], b[: o1.size]) and (a[o1.size:] == -1).all(), tick
            assert np.array_equal(base.graph_debug(), ref.graph_debug()), tick
        assert compactions >= 10 and pushed > n_total, (compactions, pushed)
    finally:
        base.close()
        ref.close()


def _keys(s):
    return SG._sched_keys(s)


def _rank_worker(rank, world, port, ret):
    import os
    import torch.distributed as dist
    from hyperqueue_b200.sharded import ShardedScheduler
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    wl = P.make_dag(20_000, 32, 4, seed=1)
    base = P.gpu_scheduler(wl, add_tasks=False, device=rank)
    sh = ShardedScheduler(base, rank, world, wl.n_tasks, torch.device("cuda", rank))
    sh.graph_init()
    from hyperqueue_b200 import priority_from_user
    off, flat = csr(wl.deps)
    sh.submit_tasks(np.arange(wl.n_tasks), wl.task_class, priority_from_user(wl.task_user_priority), off, flat)
    waves, olds = [], []
    while len(waves) < 5000:
        a, _ = sh.run_scheduling()
        t = torch.from_numpy(np.ascontiguousarray(a["task"][a["kind"] != 1]).astype(np.int64))
        sizes = [torch.zeros(1, dtype=torch.int64, device="cuda") for _ in range(world)]
        dist.all_gather(sizes, torch.tensor([t.numel()], device="cuda"))
        parts = [torch.zeros(int(s.item()), dtype=torch.int64, device="cuda") for s in sizes]
        dist.all_gather(parts, t.to("cuda"))
        every = torch.cat(parts).cpu().numpy()
        if every.size == 0:
            break
        sh.graph_tasks_finished(every)
        waves.append(int(every.size))
        if len(waves) % 7 == 0:
            olds.append(int(sh.compact_handles().size))
    ret[rank] = (waves, olds)
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_scheduler_compact_handles_one_process_per_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs: one process per GPU")
    import socket
    import torch.multiprocessing as mp
    sock = socket.socket(); sock.bind(("127.0.0.1", 0)); port = sock.getsockname()[1]; sock.close()
    mgr = mp.Manager(); ret = mgr.dict()
    mp.spawn(_rank_worker, args=(2, port, ret), nprocs=2, join=True)
    wl = P.make_dag(20_000, 32, 4, seed=1)
    ref = P.gpu_scheduler(wl, add_tasks=False)
    from hyperqueue_b200 import priority_from_user
    off, flat = csr(wl.deps)
    ref.submit_tasks(np.arange(wl.n_tasks), wl.task_class, priority_from_user(wl.task_user_priority), off, flat)
    waves = []
    while True:
        t = ref.run_scheduling().assignments["task"]
        if t.size == 0:
            break
        ref.graph_tasks_finished(t)
        waves.append(int(t.size))
    assert ret[0][0] == ret[1][0] == waves
    assert ret[0][1] == ret[1][1] and ret[0][1]
