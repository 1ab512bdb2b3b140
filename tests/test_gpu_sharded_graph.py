"""Task graphs over a sharded ready set (hqs_shard_graph_*): the graph replicated on every rank, each task's key on its owner.

The reference is one context fed the same calls through the single-context graph API with the same declared levels.  The
ranks are 2 or 3 HQS_CREATE_SHARE_DEVICE contexts of one GPU, split evenly, all on the first rank or all on the last rank.
After every call:
  * each rank's output equals the reference's restricted to its range [lo, hi), and the concatenation in rank order equals
    it in full;
  * each rank's keys (hqs_debug_keys) equal the reference keys [lo, hi) bit for bit;
  * hqs_graph_debug's edges, pool capacity and compactions are equal on every rank and to the reference's, and the ranks'
    waiting counts sum to the reference's.
Sharded ticks (unfused: hqs_shard_count + summed counts + hqs_shard_solve_emit; fused: hqs_shard_tick_launch) run between
the calls and must equal the reference tick filtered per rank.  The reference's own graph calls are checked against the
model and the specification in tests/test_gpu_graph.py and tests/test_gpu_graph_cancel.py."""
import ctypes as C

import numpy as np
import pytest
import torch

import parity as P
import test_gpu_ready_set as RS

pytestmark = pytest.mark.gpu
E_INVALID, E_STATE = -1, -6
READY, DONE, VALID = 1 << 31, 1 << 30, 1 << 29


def _ptr(a):
    from hyperqueue_b200 import _lib as L
    return L.ptr(a) if a.size else None


def csr(deps):
    off = np.concatenate([[0], np.cumsum([len(d) for d in deps])]).astype(np.uint32)
    flat = np.array([x for ds in deps for x in ds], dtype=np.uint32)
    return off, flat


def prio(user, job=0):
    return RS.tako_priority(user, job)


def splits(n_total, world):
    """Cut points: even, everything on the first rank, everything on the last rank."""
    even = [n_total * r // world for r in range(world + 1)]
    return {"even": even, "first": [0] + [n_total] * world, "last": [0] * world + [n_total]}


class Ranks:
    """The reference context and one context per rank, driven with the same calls; checks after every call."""

    def __init__(self, n_total, cuts, q, fused=False, prefill=None):
        from hyperqueue_b200 import _lib as L
        self.L = L
        self.n_total, self.cuts, self.fused = n_total, list(cuts), fused
        self.world = len(cuts) - 1
        self.ref = RS.Dev(0)
        self.ranks = [RS.Dev(L.HQS_CREATE_SHARE_DEVICE) for _ in range(self.world)]
        self.q = q
        for d in [self.ref] + self.ranks:
            d.classes(q)
        self.prefill = prefill
        if prefill:
            for d in [self.ref] + self.ranks:
                d.ok(d.lib.hqs_prefill_config(d.ctx, *prefill))
        for r, d in enumerate(self.ranks):
            d.ok(d.lib.hqs_shard_graph_init(d.ctx, n_total, self.cuts[r], self.cuts[r + 1]))
        self.cls = np.zeros(n_total, np.int64)
        self.pfw = np.full(n_total, -1, np.int64)        # worker index each task is prefilled on, -1: none
        self.W = RS.W_TOTAL.shape[0]
        if fused:
            xb = (C.c_void_p * self.world)()
            for r, d in enumerate(self.ranks):
                p = C.c_void_p()
                d.ok(d.lib.hqs_shard_xbuf(d.ctx, C.byref(p), None))
                xb[r] = p
            for r, d in enumerate(self.ranks):
                d.ok(d.lib.hqs_shard_attach(d.ctx, self.world, r, xb))
        self.counts = [torch.zeros(self.L.HQS_MAX_GROUPS, dtype=torch.int32, device="cuda") for _ in range(self.world)]

    def close(self):
        for d in [self.ref] + self.ranks:
            d.close()

    def rng_of(self, r):
        return self.cuts[r], self.cuts[r + 1]

    def debug(self, d):
        out = (C.c_uint64 * 4)()
        d.ok(d.lib.hqs_graph_debug(d.ctx, out))
        return list(out)

    def check(self, label):
        ref = self.ref.keys()
        want = self.debug(self.ref)
        waiting = 0
        for r, d in enumerate(self.ranks):
            lo, hi = self.rng_of(r)
            exp = np.zeros(hi - lo, np.uint32)
            top = max(min(ref.size, hi), lo)
            exp[: top - lo] = ref[lo:top]
            got = np.zeros(hi - lo, np.uint32)
            k = d.keys()
            assert k.size <= hi - lo, (label, r, k.size)
            got[: k.size] = k
            assert np.array_equal(got, exp), (label, r, np.nonzero(got != exp)[0][:8] + lo)
            dbg = self.debug(d)
            assert dbg[:3] == want[:3], (label, r, dbg, want)
            waiting += dbg[3]
        assert waiting == want[3], (label, waiting, want)

    def _split(self, label, got_lists, want):
        for r, got in enumerate(got_lists):
            lo, hi = self.rng_of(r)
            assert got == [x for x in want if lo <= x < hi], (label, r, got[:8])
        assert sum(got_lists, []) == want, label

    def declare(self, p):
        lv = np.ascontiguousarray(np.unique(np.asarray(p, np.uint64)))
        for d in [self.ref] + self.ranks:
            d.ok(d.lib.hqs_levels_add(d.ctx, lv.size, d.L.ptr(lv)))

    # the calls -----------------------------------------------------------------------------------------------------
    def push(self, h, c, p, off, deps, label="push", expect_ok=True):
        h, c, p = np.ascontiguousarray(h, np.uint32), np.ascontiguousarray(c, np.uint32), np.ascontiguousarray(p, np.uint64)
        off, deps = np.ascontiguousarray(off, np.uint32), np.ascontiguousarray(deps, np.uint32)
        self.declare(p)
        n = C.c_uint32(0)
        rc = self.ref.lib.hqs_graph_push(self.ref.ctx, h.size, _ptr(h), _ptr(c), _ptr(p), self.L.ptr(off), _ptr(deps), C.byref(n))
        assert (rc == 0) == expect_ok, (label, rc)
        total = 0
        for r, d in enumerate(self.ranks):
            m = C.c_uint32(0)
            rr = d.lib.hqs_shard_graph_push(d.ctx, h.size, _ptr(h), _ptr(c), _ptr(p), self.L.ptr(off), _ptr(deps), C.byref(m))
            assert rr == rc, (label, r, rr, rc)
            if rc == 0:
                lo, hi = self.rng_of(r)
                keys = self.ref.keys()
                mine = h[(h >= lo) & (h < hi)]
                assert m.value == int(np.count_nonzero(keys[mine] & READY)), (label, r, m.value)
                total += m.value
        if rc == 0:
            assert total == n.value, (label, total, n.value)
            self.cls[h] = c
            self.pfw[h] = -1
        self.check(label)
        return n.value if rc == 0 else None

    def _listing(self, name, ref_name, t, label):
        t = np.ascontiguousarray(t, np.uint32)
        ptr, k = C.POINTER(C.c_uint32)(), C.c_uint32(0)
        self.ref.ok(getattr(self.ref.lib, ref_name)(self.ref.ctx, t.size, _ptr(t), C.byref(ptr), C.byref(k)))
        want = [ptr[i] for i in range(k.value)]
        got = []
        for d in self.ranks:
            ptr, k = C.POINTER(C.c_uint32)(), C.c_uint32(0)
            d.ok(getattr(d.lib, name)(d.ctx, t.size, _ptr(t), C.byref(ptr), C.byref(k)))
            got.append([ptr[i] for i in range(k.value)])
        self._split(label, got, want)
        return want

    def finished(self, t, label="finished"):
        want = self._listing("hqs_shard_graph_finished", "hqs_graph_finished", t, label)
        self.pfw[np.asarray(t, np.int64)] = -1
        self.check(label)
        return want

    def cancel(self, t, label="cancel"):
        launches = [d.stats()["kernel_launches"] for d in self.ranks]
        want = self._listing("hqs_shard_graph_cancel", "hqs_graph_cancel", t, label)
        self.last_cancel_launches = [d.stats()["kernel_launches"] - b for d, b in zip(self.ranks, launches)]
        if want:
            self.pfw[np.asarray(want, np.int64)] = -1
        self.check(label)
        return want

    def remove(self, t, label="remove"):
        t = np.ascontiguousarray(t, np.uint32)
        self.ref.ok(self.ref.lib.hqs_ready_remove(self.ref.ctx, t.size, _ptr(t)))
        for d in self.ranks:
            d.ok(d.lib.hqs_shard_graph_remove(d.ctx, t.size, _ptr(t)))
        self.pfw[t.astype(np.int64)] = -1
        self.check(label)

    def tick(self, label="tick"):
        L = self.L
        W = self.W
        w = np.zeros(W, dtype=L.worker_dtype)
        w["worker_id"] = np.arange(W)
        w["remaining_time_ms"] = L.HQS_TIME_INF
        free = RS.W_TOTAL.copy()
        mask = None
        if self.prefill:
            mask = np.zeros((W, self.q), np.uint8)
            held = np.nonzero(self.pfw >= 0)[0]
            mask[self.pfw[held], self.cls[held]] = 1
        exp, fa = self.ref.tick(free, mask, self.n_total)
        got = []
        for d in self.ranks:
            if mask is not None:
                d.ok(d.lib.hqs_prefill_state(d.ctx, W, L.ptr(mask)))
        if self.fused:
            # contexts of one process wait for each other on the device: nothing may allocate between their launches, and
            # the groups grow with the levels, so every rank reserves before the first launch of each tick
            for d in self.ranks:
                d.ok(d.lib.hqs_tick_reserve(d.ctx, W, self.n_total, 0))
            for d in self.ranks:
                d.ok(d.lib.hqs_shard_tick_launch(d.ctx, W, L.ptr(w), L.ptr(free), L.ptr(RS.W_TOTAL), None, self.n_total))
        else:
            ng = C.c_uint32(0)
            for d, cnt in zip(self.ranks, self.counts):
                d.ok(d.lib.hqs_shard_count(d.ctx, W, L.ptr(w), L.ptr(free), L.ptr(RS.W_TOTAL), None,
                                           C.c_void_p(cnt.data_ptr()), cnt.numel(), C.byref(ng)))
            torch.cuda.synchronize()
            allc = torch.stack(self.counts).sum(0, dtype=torch.int32)
            before = [torch.stack(self.counts[:r]).sum(0, dtype=torch.int32) if r else torch.zeros_like(allc)
                      for r in range(self.world)]
            torch.cuda.synchronize()
            for d, b in zip(self.ranks, before):
                d.ok(d.lib.hqs_shard_solve_emit(d.ctx, C.c_void_p(allc.data_ptr()), C.c_void_p(b.data_ptr()), self.n_total))
        for r, d in enumerate(self.ranks):
            lo, hi = self.rng_of(r)
            out = np.zeros(self.n_total, dtype=L.assignment_dtype)
            n = C.c_uint32(0)
            fr = np.zeros_like(free)
            d.ok(d.lib.hqs_tick_fetch(d.ctx, self.n_total, L.ptr(out), C.byref(n), L.ptr(fr)))
            a = out[: n.value].copy()
            a["task"] += np.uint32(lo)
            want = exp[(exp["task"] >= lo) & (exp["task"] < hi)]
            assert np.array_equal(a, want), (label, r, a[:4], want[:4])
            assert np.array_equal(fr, fa), (label, r)
            got.append(a)
        t = exp["task"].astype(np.int64)
        self.pfw[t[exp["kind"] != 1]] = -1
        self.pfw[t[exp["kind"] == 1]] = exp["worker"][exp["kind"] == 1]
        self.check(label)
        return exp


def make(n_total, world, split, q=2, **kw):
    return Ranks(n_total, splits(n_total, world)[split], q, **kw)


# rejections and state rules --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world,split", [(2, "even"), (3, "even"), (3, "first"), (2, "last")])
def test_rejections_leave_every_rank_unchanged(world, split):
    s = make(64, world, split, q=2)
    try:
        s.push([0, 1, 2, 40], [0, 1, 0, 1], [prio(1)] * 4, *csr([[], [0], [0, 1], [2]]))
        bad = [
            ([3], [2], [prio(1)], [0, 0], []),                       # class id >= n_classes
            ([3, 3], [0, 0], [prio(1)] * 2, [0, 0, 0], []),          # a handle twice
            ([1], [0], [prio(1)], [0, 0], []),                       # a VALID (waiting) handle
            ([40], [0], [prio(1)], [0, 0], []),                      # a VALID handle on the upper rank
            ([3], [0], [prio(1)], [0, 1], [3]),                      # depends on itself
            ([3], [0], [prio(1)], [0, 2], [0, 0]),                   # the same dependency twice
            ([3], [0], [prio(1)], [1, 1], [0]),                      # dep_off[0] != 0
            ([3, 4], [0, 5], [prio(7)] * 2, [0, 0, 1], [3]),         # valid dependencies, a bad class id
        ]
        for args in bad:
            assert s.push(*args, label=f"rejected {args}", expect_ok=False) is None
        # a handle or a dependency >= n_total: only the sharded calls know n_total
        for h, off, deps in (([64], [0, 0], []), ([5], [0, 1], [64])):
            before = [d.keys() for d in s.ranks]
            for d in s.ranks:
                hh, c, p = np.array(h, np.uint32), np.zeros(1, np.uint32), np.array([prio(1)], np.uint64)
                o, dd = np.array(off, np.uint32), np.array(deps, np.uint32)
                assert d.lib.hqs_shard_graph_push(d.ctx, 1, d.L.ptr(hh), d.L.ptr(c), d.L.ptr(p), d.L.ptr(o), _ptr(dd),
                                                  C.byref(C.c_uint32())) == E_INVALID
            assert all(np.array_equal(b, d.keys()) for b, d in zip(before, s.ranks))
        big = np.array([3, 64], np.uint32)
        for d in s.ranks:
            ptr, k = C.POINTER(C.c_uint32)(), C.c_uint32(0)
            assert d.lib.hqs_shard_graph_finished(d.ctx, 2, d.L.ptr(big), C.byref(ptr), C.byref(k)) == E_INVALID
            assert d.lib.hqs_shard_graph_cancel(d.ctx, 2, d.L.ptr(big), C.byref(ptr), C.byref(k)) == E_INVALID
            assert d.lib.hqs_shard_graph_remove(d.ctx, 2, d.L.ptr(big)) == E_INVALID
        # an undeclared priority is refused by the sharded push (the ranks would number the levels differently)
        d = s.ranks[0]
        hh, c, p, o = np.array([7], np.uint32), np.zeros(1, np.uint32), np.array([prio(99)], np.uint64), np.zeros(2, np.uint32)
        assert d.lib.hqs_shard_graph_push(d.ctx, 1, d.L.ptr(hh), d.L.ptr(c), d.L.ptr(p), d.L.ptr(o), None,
                                          C.byref(C.c_uint32())) == E_INVALID
        s.check("after the rejections")
        for d in [s.ref] + s.ranks:
            out = (C.c_uint64 * 4)()
            d.ok(d.lib.hqs_graph_debug(d.ctx, out))
            assert out[2] == 0
    finally:
        s.close()


def test_state_rules():
    from hyperqueue_b200 import _lib as L
    one = np.zeros(1, np.uint32)
    p1 = np.array([prio(0)], np.uint64)
    off = np.zeros(2, np.uint32)
    n, ptr = C.c_uint32(0), C.POINTER(C.c_uint32)()
    d = RS.Dev(L.HQS_CREATE_SHARE_DEVICE)
    try:
        d.classes(1)
        d.ok(d.lib.hqs_levels_add(d.ctx, 1, d.L.ptr(p1)))
        # the sharded calls need hqs_shard_graph_init
        assert d.lib.hqs_shard_graph_push(d.ctx, 1, d.L.ptr(one), d.L.ptr(one), d.L.ptr(p1), d.L.ptr(off), None, C.byref(n)) == E_STATE
        assert d.lib.hqs_shard_graph_finished(d.ctx, 1, d.L.ptr(one), C.byref(ptr), C.byref(n)) == E_STATE
        assert d.lib.hqs_shard_graph_cancel(d.ctx, 1, d.L.ptr(one), C.byref(ptr), C.byref(n)) == E_STATE
        assert d.lib.hqs_shard_graph_remove(d.ctx, 1, d.L.ptr(one)) == E_STATE
        assert d.lib.hqs_shard_graph_init(d.ctx, 10, 6, 5) == E_INVALID
        assert d.lib.hqs_shard_graph_init(d.ctx, 10, 5, 11) == E_INVALID
        # a pending tick refuses it
        w = np.zeros(1, dtype=d.L.worker_dtype)
        w["remaining_time_ms"] = d.L.HQS_TIME_INF
        free = RS.W_TOTAL[:1].copy()
        d.ok(d.lib.hqs_tick_launch(d.ctx, 1, d.L.ptr(w), d.L.ptr(free), d.L.ptr(free), None, 4))
        assert d.lib.hqs_shard_graph_init(d.ctx, 10, 0, 5) == E_STATE
        out = np.zeros(4, dtype=d.L.assignment_dtype)
        d.ok(d.lib.hqs_tick_fetch(d.ctx, 4, d.L.ptr(out), C.byref(n), None))
        d.ok(d.lib.hqs_shard_graph_init(d.ctx, 10, 0, 5))
        assert d.lib.hqs_shard_graph_init(d.ctx, 10, 0, 5) == E_STATE                 # a second time
        # the single-context calls, hqs_ready_push / _range / _remove and hqs_dag_load are refused
        assert d.lib.hqs_graph_push(d.ctx, 1, d.L.ptr(one), d.L.ptr(one), d.L.ptr(p1), d.L.ptr(off), None, C.byref(n)) == E_STATE
        assert d.lib.hqs_graph_finished(d.ctx, 1, d.L.ptr(one), C.byref(ptr), C.byref(n)) == E_STATE
        assert d.lib.hqs_graph_cancel(d.ctx, 1, d.L.ptr(one), C.byref(ptr), C.byref(n)) == E_STATE
        assert d.lib.hqs_ready_push(d.ctx, 1, d.L.ptr(one), d.L.ptr(one), d.L.ptr(p1)) == E_STATE
        assert d.lib.hqs_ready_push_range(d.ctx, 0, 1, d.L.ptr(one), d.L.ptr(p1)) == E_STATE
        assert d.lib.hqs_ready_remove(d.ctx, 1, d.L.ptr(one)) == E_STATE
        assert d.lib.hqs_dag_load(d.ctx, 1, d.L.ptr(one), d.L.ptr(p1), d.L.ptr(one), d.L.ptr(off), None) == E_STATE
        d.ok(d.lib.hqs_shard_graph_push(d.ctx, 1, d.L.ptr(one), d.L.ptr(one), d.L.ptr(p1), d.L.ptr(off), None, C.byref(n)))
        assert n.value == 1
    finally:
        d.close()
    # after a graph push, after hqs_dag_load, on a table with a live key: refused; on an attached context: allowed
    for case in ("graph", "dag", "live", "attached"):
        e = RS.Dev(0)
        try:
            e.classes(1)
            if case == "graph":
                e.ok(e.lib.hqs_graph_push(e.ctx, 1, e.L.ptr(one), e.L.ptr(one), e.L.ptr(p1), e.L.ptr(off), None, C.byref(n)))
            elif case == "dag":
                e.ok(e.lib.hqs_dag_load(e.ctx, 1, e.L.ptr(one), e.L.ptr(p1), e.L.ptr(one), e.L.ptr(off), None))
            elif case == "live":
                e.push([3], [0], [prio(0)], as_range=False)
            else:
                xb = C.c_void_p()
                e.ok(e.lib.hqs_shard_xbuf(e.ctx, C.byref(xb), None))
                e.ok(e.lib.hqs_shard_attach(e.ctx, 1, 0, (C.c_void_p * 1)(xb)))
            rc = e.lib.hqs_shard_graph_init(e.ctx, 8, 0, 8)
            assert rc == (0 if case == "attached" else E_STATE), (case, rc)
        finally:
            e.close()


# cross-rank edges ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world,split", [(2, "even"), (3, "even"), (3, "first"), (3, "last")])
def test_cross_rank_edges(world, split):
    n_total = 90
    s = make(n_total, world, split, q=2)
    try:
        # a chain that alternates ranks: 0 -> 30 -> 1 -> 60 -> 2 -> 89
        chain = [0, 30, 1, 60, 2, 89]
        assert s.push(chain, [0] * 6, [prio(1)] * 6, *csr([[]] + [[chain[i - 1]] for i in range(1, 6)])) == 1
        for i in range(5):
            assert s.finished([chain[i]]) == [chain[i + 1]]
        s.finished([89])
        # a fan-out from rank 0 to every rank, then a diamond across a boundary
        fan = [5] + list(range(10, 90, 7))
        s.push(fan, [1] * len(fan), [prio(2)] * len(fan), *csr([[]] + [[5]] * (len(fan) - 1)))
        assert s.finished([5]) == sorted(fan[1:])
        s.push([44, 46, 29, 32], [0, 1, 0, 1], [prio(3)] * 4, *csr([[], [44], [44], [46, 29]]))
        assert s.finished([44]) == [29, 46]
        assert s.finished([46]) == []
        assert s.finished([29]) == [32]
        # a resubmitted low handle depends on a higher one
        s.push([70], [0], [prio(0)], *csr([[]]))
        assert s.push([0], [1], [prio(0)], *csr([[70]])) == 0
        assert s.finished([70]) == [0]
        s.tick()
        # a cancel whose closure crosses the ranks several times costs the launches of a lone task
        zig = [3, 50, 4, 81, 6, 33, 7, 65]
        s.push(zig, [0] * 8, [prio(4)] * 8, *csr([[]] + [[zig[i - 1]] for i in range(1, 8)]))
        s.push([8], [0], [prio(4)], *csr([[]]))
        assert s.cancel([8]) == [8]
        lone = s.last_cancel_launches
        assert s.cancel([3]) == sorted(zig)
        assert s.last_cancel_launches == lone == [6] * world
    finally:
        s.close()


@pytest.mark.parametrize("world,split", [(2, "even"), (3, "even")])
def test_removed_producer_resubmitted_does_not_release_old_consumers(world, split):
    s = make(60, world, split, q=2)
    try:
        s.push([1, 25, 45], [0, 0, 1], [prio(1)] * 3, *csr([[], [1], [1]]))
        s.remove([1])                                 # the consumers keep waiting, on every rank's replica
        assert s.push([1], [1], [prio(2)], *csr([[]])) == 1
        assert s.finished([1]) == []                  # the new incarnation of 1 has no consumers
        s.cancel([25, 45])
        assert s.debug(s.ref)[3] == 0
    finally:
        s.close()


# random sequences with ticks in between ------------------------------------------------------------------------------------
def _random(s, rng, steps, n_total):
    q = s.q
    next_h, free_handles, job = 0, [], 0
    for step in range(steps):
        keys = s.ref.keys()
        live = np.nonzero(keys & VALID)[0]
        k = int(rng.integers(1, 40))
        reuse = [free_handles.pop(int(rng.integers(0, len(free_handles)))) for _ in range(min(len(free_handles), k // 2))]
        fresh = list(range(next_h, min(next_h + k - len(reuse), n_total)))
        next_h += len(fresh)
        hs = reuse + fresh
        if not hs:
            break
        if rng.random() < 0.5:
            hs = sorted(hs)
        deps = []
        for i, x in enumerate(hs):
            pool = list(live[-80:]) + hs[:i] + hs[i + 1: i + 3]
            ds = {int(pool[j]) for j in rng.integers(0, len(pool), size=int(rng.integers(0, 4)))} - {x} if pool else set()
            deps.append(sorted(ds))
        s.push(hs, rng.integers(0, q, size=len(hs)), [prio(int(rng.integers(0, 4)), job)] * len(hs), *csr(deps), label=f"push {step}")
        job += 1
        live = np.nonzero(s.ref.keys() & VALID)[0]
        if rng.random() < 0.25 and live.size:
            gone = s.cancel([int(x) for x in rng.choice(live, size=min(3, live.size), replace=False)], f"cancel {step}")
            free_handles += gone
        elif rng.random() < 0.2 and live.size:
            victim = [int(x) for x in rng.choice(live, size=min(4, live.size), replace=False)]
            s.remove(victim, f"remove {step}")
            free_handles += victim
        exp = s.tick(f"tick {step}")
        done = exp[exp["kind"] != 1]["task"]
        fin = [int(x) for x in done if rng.random() < 0.8]
        if fin:
            s.finished(fin + fin[:1], f"finish {step}")
            free_handles += fin


@pytest.mark.parametrize("world,split,fused,seed", [(2, "even", False, 0), (3, "even", False, 1), (3, "first", False, 2),
                                                    (3, "last", False, 3), (2, "even", True, 4), (2, "last", True, 5)])
def test_random_sequences_with_sharded_ticks(world, split, fused, seed):
    n_total = 1500
    s = make(n_total, world, split, q=3, fused=fused, prefill=RS.PREFILL)
    try:
        _random(s, np.random.default_rng(700 + seed), 40, n_total)
    finally:
        s.close()


def test_pool_compaction_and_a_rank_past_65536_handles():
    n_total = 140_000                                 # rank 1 holds local handles past 65 536
    s = make(n_total, 2, "even", q=3)
    try:
        prod = np.concatenate([np.arange(50), np.arange(139_900, 139_950)])
        s.push(prod, prod % 3, [prio(2)] * prod.size, *csr([[]] * prod.size))
        keep = np.arange(69_990, 70_040)               # across the boundary
        s.push(keep, keep % 3, [prio(1)] * 50, *csr([[int(prod[i]), int(prod[i + 50])] for i in range(50)]))
        rng = np.random.default_rng(5)
        cons = np.arange(100_000, 101_500)
        for wave in range(6):
            deps = [sorted({int(x) for x in rng.choice(prod, size=2)}) for _ in cons]
            s.push(cons, cons % 3, [prio(0, wave)] * cons.size, *csr(deps), label=f"wave {wave}")
            s.remove(cons)
        assert s.debug(s.ref)[2] >= 2
        assert s.finished(prod) == list(keep)
        s.tick()
    finally:
        s.close()


# the cfg4 DAG over two contexts -------------------------------------------------------------------------------------------
def test_cfg4_drains_like_the_single_context_graph():
    from hyperqueue_b200 import _lib as L, priority_from_user
    wl = P.make_dag(500_000, 256, 16, seed=0)
    n = wl.n_tasks
    ref = P.gpu_scheduler(wl, add_tasks=False)
    cuts = [0, n // 2, n]
    ranks = [P.gpu_scheduler(wl, add_tasks=False, flags=L.HQS_CREATE_SHARE_DEVICE) for _ in range(2)]
    prio_all = priority_from_user(wl.task_user_priority)
    lv = np.ascontiguousarray(np.unique(prio_all))
    for r, s in enumerate(ranks):
        s._sync_classes()
        s._check(s._lib.hqs_levels_add(s._ctx, lv.size, L.ptr(lv)))
        s._check(s._lib.hqs_shard_graph_init(s._ctx, n, cuts[r], cuts[r + 1]))
    ready = 0
    for lo in range(0, n, 10_000):
        hi = min(lo + 10_000, n)
        ds = wl.deps[lo:hi]
        off, flat = csr(ds)
        h = np.arange(lo, hi, dtype=np.uint32)
        c = np.ascontiguousarray(wl.task_class[lo:hi], np.uint32)
        p = np.ascontiguousarray(prio_all[lo:hi])
        ready += ref.submit_tasks(h, c, p, off, flat)
        for s in ranks:
            m = C.c_uint32(0)
            s._check(s._lib.hqs_shard_graph_push(s._ctx, h.size, L.ptr(h), L.ptr(c), L.ptr(p), L.ptr(off), _ptr(flat), C.byref(m)))
    counts = [torch.zeros(L.HQS_MAX_GROUPS, dtype=torch.int32, device="cuda") for _ in ranks]
    outs = [np.zeros(n, dtype=L.assignment_dtype) for _ in ranks]
    waves, left = 0, n
    while left and waves < 5000:
        w = ref._worker_structs(0.0)
        free, total = np.ascontiguousarray(ref.free), np.ascontiguousarray(ref.total)
        ng = C.c_uint32(0)
        for s, cnt in zip(ranks, counts):
            s._check(s._lib.hqs_shard_count(s._ctx, w.shape[0], L.ptr(w), L.ptr(free), L.ptr(total), None,
                                            C.c_void_p(cnt.data_ptr()), cnt.numel(), C.byref(ng)))
        torch.cuda.synchronize()
        allc = counts[0] + counts[1]
        torch.cuda.synchronize()
        got = []
        for r, (s, b) in enumerate(zip(ranks, (torch.zeros_like(allc), counts[0]))):
            s._check(s._lib.hqs_shard_solve_emit(s._ctx, C.c_void_p(allc.data_ptr()), C.c_void_p(b.data_ptr()), n))
            out = outs[r]
            k = C.c_uint32(0)
            s._check(s._lib.hqs_tick_fetch(s._ctx, out.size, L.ptr(out), C.byref(k), None))
            a = out[: k.value].copy()
            a["task"] += np.uint32(cuts[r])
            got.append(a)
        mref = ref.run_scheduling()
        exp = mref.assignments
        for r in range(2):
            assert np.array_equal(got[r], exp[(exp["task"] >= cuts[r]) & (exp["task"] < cuts[r + 1])]), waves
        t = np.ascontiguousarray(exp["task"])
        assert t.size, waves
        made = ref.graph_tasks_finished(t)
        lists = []
        for s in ranks:
            ptr, k = C.POINTER(C.c_uint32)(), C.c_uint32(0)
            s._check(s._lib.hqs_shard_graph_finished(s._ctx, t.size, L.ptr(t), C.byref(ptr), C.byref(k)))
            lists.append([ptr[i] for i in range(k.value)])
        assert lists[0] + lists[1] == made.tolist(), waves
        left -= t.size
        waves += 1
    assert left == 0 and waves == 1234
    for s in ranks:
        dbg = (C.c_uint64 * 4)()
        s._check(s._lib.hqs_graph_debug(s._ctx, dbg))
        assert dbg[0] == 0 and dbg[3] == 0
        s.close()
    ref.close()


# ShardedScheduler ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p2p", [False, True])
def test_sharded_scheduler_as_one_rank(p2p):
    from hyperqueue_b200.sharded import ShardedScheduler
    wl = P.make_independent(2000, 16, 4, seed=3)
    n = 2000
    ref = P.gpu_scheduler(wl, add_tasks=False)
    base = P.gpu_scheduler(wl, add_tasks=False)
    sh = ShardedScheduler(base, 0, 1, n, torch.device("cuda", 0), p2p=p2p)
    sh.graph_init()
    sh.set_prefill(*RS.PREFILL)
    ref.set_prefill(*RS.PREFILL)
    rng = np.random.default_rng(11)
    started = 0
    try:
        cls = np.ascontiguousarray(wl.task_class, np.uint32)
        pr = np.array([prio(int(u), 0) for u in rng.integers(0, 3, n)], np.uint64)
        sh.add_ready_tasks(np.arange(0, 100), cls[:100], pr[:100])          # routed through hqs_shard_graph_push
        ref.submit_tasks(np.arange(0, 100), cls[:100], pr[:100], np.zeros(101, np.uint32), np.zeros(0, np.uint32))
        for lo in range(100, n, 300):
            hi = min(lo + 300, n)
            deps = [sorted({int(x) for x in rng.integers(0, lo, size=int(rng.integers(0, 3)))}) for _ in range(lo, hi)]
            off, flat = csr(deps)
            a = sh.submit_tasks(np.arange(lo, hi), cls[lo:hi], pr[lo:hi], off, flat)
            b = ref.submit_tasks(np.arange(lo, hi), cls[lo:hi], pr[lo:hi], off, flat)
            assert a == b
            got, fa = sh.run_scheduling()
            exp = ref.run_scheduling()
            assert np.array_equal(got, exp.assignments) and np.array_equal(fa, exp.free_after)
            pf = exp.assignments[exp.assignments["kind"] == 1]
            if pf.size:
                # RunningPrefilled: the task leaves the table of every rank, and the worker's resources are taken
                t = int(pf["task"][-1])
                sh.on_task_running_prefilled(t, 0)
                ref.on_task_running_prefilled(t, 0)
                started += 1
                assert np.array_equal(base.free, ref.free)
                assert np.array_equal(_sched_keys(base), _sched_keys(ref))
            done = exp.assignments[exp.assignments["kind"] != 1]["task"]
            fin = done[: done.size // 2]
            assert np.array_equal(sh.graph_tasks_finished(fin), ref.graph_tasks_finished(fin))
            assert np.array_equal(base.free, ref.free)
            victims = done[done.size // 2: done.size // 2 + 2]
            g1, m1 = sh.graph_cancel_tasks(victims)
            g2, m2 = ref.graph_cancel_tasks(victims)
            assert np.array_equal(g1, g2) and m1 == m2
            assert np.array_equal(base.free, ref.free)
            sh.remove_ready_tasks(done[-1:])
            ref.remove_ready_tasks(done[-1:])
            assert np.array_equal(base.graph_debug(), ref.graph_debug())
        assert started > 0
    finally:
        base.close()
        ref.close()


def _sched_keys(s):
    n = C.c_uint32(0)
    s._check(s._lib.hqs_debug_keys(s._ctx, 0, None, C.byref(n)))
    out = np.zeros(n.value, np.uint32)
    s._check(s._lib.hqs_debug_keys(s._ctx, n.value, _ptr(out), C.byref(n)))
    return out


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
    waves = []
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
    ret[rank] = waves
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_scheduler_one_process_per_gpu():
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
    assert ret[0] == ret[1] == waves
    ref.close()
