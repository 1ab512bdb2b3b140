"""Task graphs on the device (hqs_graph_push / hqs_graph_finished) against tests/graph_model.py: after every call the whole
key array (hqs_debug_keys), hqs_graph_debug, every n_ready and every list of newly ready handles must equal the model's, on
two contexts side by side (one per amount width of the solver).  Ticks in between are compared with the sequential
specification (tests/greedy_model.py) and the judge, through tests/test_gpu_ready_set.py's harness.  Then the cfg4 DAG
submitted in batches must drain exactly as hqs_dag_load drains it, and the C++ shim's graph self-test must pass."""
import ctypes as C

import numpy as np
import pytest

import graph_model as GM
import level_model as LM
import parity as P
import test_gpu_ready_set as RS

pytestmark = pytest.mark.gpu
E_INVALID, E_STATE = -1, -6


def _ptr(a):
    from hyperqueue_b200 import _lib as L
    return L.ptr(a) if a.size else None


class Harness(RS.Harness):
    def __init__(self):
        super().__init__()
        self.m = GM.GraphModel()

    def check(self, label):
        super().check(label)
        want = self.m.debug()
        for d in self.devs:
            out = (C.c_uint64 * 4)()
            d.ok(d.lib.hqs_graph_debug(d.ctx, out))
            assert list(out) == want, (label, list(out), want)

    def graph_push(self, h, c, p, off, deps, label="graph_push"):
        h, c, p = np.ascontiguousarray(h, np.uint32), np.ascontiguousarray(c, np.uint32), np.ascontiguousarray(p, np.uint64)
        off, deps = np.ascontiguousarray(off, np.uint32), np.ascontiguousarray(deps, np.uint32)
        if h.size and int(h.max()) < 0xFFFFFFFF:
            hi = h.astype(np.int64)
            if hi.max() >= self.pfw.size:
                self.pfw = np.concatenate([self.pfw, np.full(int(hi.max()) + 1 - self.pfw.size, -1, np.int64)])
        try:
            want = self.m.graph_push(h, c, p, off, deps)
        except LM.Rejected:
            want = None
        for d in self.devs:
            n = C.c_uint32(12345)
            rc = d.lib.hqs_graph_push(d.ctx, h.size, _ptr(h), _ptr(c), _ptr(p), d.L.ptr(off), _ptr(deps), C.byref(n))
            if want is None:
                assert rc == E_INVALID, (label, rc)
            else:
                d.ok(rc)
                assert n.value == want, (label, n.value, want)
        if want is not None:
            self.pfw[h.astype(np.int64)] = -1
        self.check(label)
        return want

    def graph_finished(self, t, label="graph_finished"):
        t = np.ascontiguousarray(t, np.uint32)
        try:
            want = self.m.graph_finished(t)
        except LM.Rejected:
            want = None
        for d in self.devs:
            ptr, k = C.POINTER(C.c_uint32)(), C.c_uint32(0)
            rc = d.lib.hqs_graph_finished(d.ctx, t.size, _ptr(t), C.byref(ptr), C.byref(k))
            if want is None:
                assert rc == E_INVALID, (label, rc)
            else:
                d.ok(rc)
                got = [ptr[i] for i in range(k.value)]
                assert got == want, (label, got[:8], want[:8], len(got), len(want))
        if want is not None:
            ti = t.astype(np.int64)
            self.pfw[ti[ti < self.pfw.size]] = -1
        self.check(label)
        return want


@pytest.fixture
def harness():
    h = Harness()
    yield h
    h.close()


def csr(deps):
    off = np.concatenate([[0], np.cumsum([len(d) for d in deps])]).astype(np.uint32)
    flat = np.array([x for ds in deps for x in ds], dtype=np.uint32)
    return off, flat


def prio(user, job=0):
    return RS.tako_priority(user, job)


# directed cases -------------------------------------------------------------------------------------------------------
def test_every_rejection_leaves_the_context_unchanged(harness):
    h = harness
    h.classes(2)
    assert h.graph_push([0, 1, 2], [0, 1, 0], [prio(1)] * 3, *csr([[], [0], [0, 1]])) == 1
    bad = [
        ([3], [2], [prio(1)], [0, 0], []),                       # class id >= n_classes
        ([3, 3], [0, 0], [prio(1)] * 2, [0, 0, 0], []),          # a handle twice
        ([3, 0xFFFFFFFF], [0, 0], [prio(1)] * 2, [0, 0, 0], []), # the reserved handle
        ([1], [0], [prio(1)], [0, 0], []),                       # a VALID (waiting) handle
        ([0], [0], [prio(1)], [0, 0], []),                       # a VALID (ready) handle
        ([3], [0], [prio(1)], [0, 1], [3]),                      # depends on itself
        ([3], [0], [prio(1)], [0, 2], [0, 0]),                   # the same dependency twice
        ([3], [0], [prio(1)], [0, 1], [40]),                     # neither in the batch nor < n_handles
        ([3], [0], [prio(1)], [1, 1], [0]),                      # dep_off[0] != 0
        ([3, 4], [0, 0], [prio(1)] * 2, [0, 1, 0], [0]),         # dep_off decreases
        ([3, 4], [0, 5], [prio(7)] * 2, [0, 0, 1], [3]),         # valid dependencies, a bad class id: nothing at all
    ]
    for args in bad:
        assert h.graph_push(*args, label=f"rejected {args}") is None
    assert h.graph_finished([0, 3]) is None                    # a handle >= n_handles
    # the pool's first allocation and its compactions happen only for accepted batches
    for d in h.devs:
        out = (C.c_uint64 * 4)()
        d.ok(d.lib.hqs_graph_debug(d.ctx, out))
        assert out[1] == GM.POOL_MIN and out[2] == 0


def test_mode_rules(harness):
    h = harness
    h.classes(1)
    d = h.devs[0]
    n, ptr = C.c_uint32(0), C.POINTER(C.c_uint32)()
    one = np.zeros(1, np.uint32)
    p1 = np.array([prio(0)], np.uint64)
    off = np.zeros(2, np.uint32)
    # a graph context refuses hqs_dag_load
    h.graph_push([0], [0], [prio(0)], *csr([[]]))
    assert d.lib.hqs_dag_load(d.ctx, 1, d.L.ptr(one), d.L.ptr(p1), d.L.ptr(one), d.L.ptr(off), None) == E_STATE
    # a pending tick refuses the graph calls, and they work again after the fetch
    w = np.zeros(1, dtype=d.L.worker_dtype)
    w["remaining_time_ms"] = d.L.HQS_TIME_INF
    free = RS.W_TOTAL[:1].copy()
    d.ok(d.lib.hqs_tick_launch(d.ctx, 1, d.L.ptr(w), d.L.ptr(free), d.L.ptr(free), None, 4))
    two = np.array([1], np.uint32)
    assert d.lib.hqs_graph_push(d.ctx, 1, d.L.ptr(two), d.L.ptr(one), d.L.ptr(p1), d.L.ptr(off), None, C.byref(n)) == E_STATE
    assert d.lib.hqs_graph_finished(d.ctx, 1, d.L.ptr(one), C.byref(ptr), C.byref(n)) == E_STATE
    assert d.lib.hqs_graph_debug(d.ctx, (C.c_uint64 * 4)()) == E_STATE
    out = np.zeros(4, dtype=d.L.assignment_dtype)
    d.ok(d.lib.hqs_tick_fetch(d.ctx, 4, d.L.ptr(out), C.byref(n), None))
    d.ok(d.lib.hqs_graph_debug(d.ctx, (C.c_uint64 * 4)()))
    # a DAG context and an attached context refuse the graph calls
    for attach in (False, True):
        e = RS.Dev(0)
        try:
            e.classes(1)
            if attach:
                xb = C.c_void_p()
                e.ok(e.lib.hqs_shard_xbuf(e.ctx, C.byref(xb), None))
                e.ok(e.lib.hqs_shard_attach(e.ctx, 1, 0, (C.c_void_p * 1)(xb)))
            else:
                e.ok(e.lib.hqs_dag_load(e.ctx, 1, e.L.ptr(one), e.L.ptr(p1), e.L.ptr(one), e.L.ptr(off), None))
            assert e.lib.hqs_graph_push(e.ctx, 1, e.L.ptr(two), e.L.ptr(one), e.L.ptr(p1), e.L.ptr(off), None, C.byref(n)) == E_STATE
            assert e.lib.hqs_graph_finished(e.ctx, 1, e.L.ptr(one), C.byref(ptr), C.byref(n)) == E_STATE
            assert e.lib.hqs_graph_debug(e.ctx, (C.c_uint64 * 4)()) == E_STATE
        finally:
            e.close()


def test_tasks_finished_rejects_handles_outside_the_dag():
    d = RS.Dev(0)
    try:
        d.classes(1)
        c = np.zeros(3, np.uint32)
        p = np.full(3, prio(0), np.uint64)
        nd = np.array([0, 1, 1], np.uint32)
        off = np.array([0, 1, 2, 2], np.uint32)
        cons = np.array([1, 2], np.uint32)
        d.ok(d.lib.hqs_dag_load(d.ctx, 3, d.L.ptr(c), d.L.ptr(p), d.L.ptr(nd), d.L.ptr(off), d.L.ptr(cons)))
        before = d.keys()
        n = C.c_uint32(0)
        t = np.array([0, 3], np.uint32)
        assert d.lib.hqs_tasks_finished(d.ctx, 2, d.L.ptr(t), C.byref(n)) == E_INVALID
        assert np.array_equal(d.keys(), before)
        d.ok(d.lib.hqs_tasks_finished(d.ctx, 1, d.L.ptr(t), C.byref(n)))
        assert n.value == 1
    finally:
        d.close()


def test_cancelled_and_resubmitted_consumer_under_a_live_producer(harness):
    h = harness
    h.classes(2)
    assert h.graph_push([0, 1, 2], [0, 0, 1], [prio(2)] * 3, *csr([[], [0], [0, 1]])) == 1
    h.tick()                                          # producer 0 is assigned (DONE) and stays VALID
    h.remove([1, 2])                                  # the consumers are cancelled; 1's list goes with it
    assert h.graph_push([1, 2], [1, 0], [prio(1)] * 2, *csr([[], [1]])) == 1   # re-submitted: 2 waits on the new 1 only
    assert h.graph_finished([0]) == []               # the old edges 0 -> 1 and 0 -> 2 are stale
    h.tick()
    assert h.graph_finished([1]) == [2]
    h.tick()
    assert h.graph_finished([2]) == []
    assert h.m.debug()[0] == 0 and h.m.debug()[3] == 0


def test_duplicate_and_not_valid_finishes(harness):
    h = harness
    h.classes(1)
    h.graph_push(np.arange(6), np.zeros(6), [prio(0)] * 6, *csr([[], [], [0, 1], [2], [2], [0]]))
    assert h.graph_finished([0, 0, 0]) == [5]        # named thrice, released once
    assert h.graph_finished([0, 1, 1]) == [2]        # 0 already left: ignored
    h.remove([4])
    assert h.graph_finished([4, 2, 2]) == [3]        # 4 was removed: not VALID
    assert h.graph_finished([3, 3]) == []
    assert h.graph_finished([2, 5]) == []            # a ready task that never ran may finish too (it leaves the table)


@pytest.mark.parametrize("q", [2, 4096])
def test_fresh_priorities_carried_only_by_waiting_tasks(harness, q):
    """Exact (2 classes) and coarse (4096 classes: two levels) tables: new priorities arrive only on waiting tasks, the
    older tasks leave, and the levels the waiting tasks pin must survive every pruning."""
    h = harness
    h.classes(q)
    rng = np.random.default_rng(q)
    base = np.arange(200)
    h.graph_push(base, base % q, [prio(0, j) for j in range(200)], *csr([[]] * 200))
    for wave in range(4):
        hs = np.arange(1000 + 100 * wave, 1100 + 100 * wave)
        deps = [[int(x)] for x in rng.choice(base[base % 4 == wave], size=100)]
        h.graph_push(hs, hs % q, [prio(5 + wave, 7 * j) for j in range(100)], *csr(deps))
        h.remove(base[base % 4 == (wave + 1) % 4])   # some producers are cancelled: their consumers keep waiting
        h.push(np.arange(5000 + 300 * wave, 5300 + 300 * wave), np.arange(300) % q, [prio(-1, 50 * wave + j) for j in range(300)],
               as_range=True)
        h.tick()
        h.graph_finished(base[base % 4 == wave])


def test_table_growth_past_65536_handles_with_live_edges(harness):
    h = harness
    h.classes(2)
    h.graph_push(np.arange(64), np.arange(64) % 2, [prio(1)] * 64, *csr([[]] * 64))
    far = np.arange(70000, 70500)
    h.graph_push(far, far % 2, [prio(3)] * 500, *csr([[int(i % 64), int((i * 7 + 1) % 64)] for i in range(500)]))
    h.push(np.arange(200000, 200010), np.zeros(10), [prio(0)] * 10, as_range=True)     # the table grows again
    h.graph_push([131072], [1], [prio(9)], *csr([[70001]]))
    h.graph_finished(np.arange(0, 64, 2))
    h.graph_finished(np.arange(1, 64, 2))
    h.tick()
    h.graph_finished([70001, 70001])


def test_pool_compactions_keep_the_waiting_edges(harness):
    """Consumers that are cancelled while their producers stay live leave stale edges behind; the pool is compacted (at
    least twice) and the edges of the consumers that still wait survive every compaction, across handle re-use."""
    h = harness
    h.classes(3)
    prod = np.arange(100)
    h.graph_push(prod, prod % 3, [prio(2)] * 100, *csr([[]] * 100))
    keep = np.arange(100, 150)
    h.graph_push(keep, keep % 3, [prio(1)] * 50, *csr([[i, i + 50] for i in range(50)]))
    rng = np.random.default_rng(5)
    cons = np.arange(1000, 2500)
    for wave in range(6):
        deps = [sorted({int(x) for x in rng.choice(prod, size=2)}) for _ in cons]
        h.graph_push(cons, cons % 3, [prio(0, wave)] * cons.size, *csr(deps))
        h.remove(cons)                                # the same handles are submitted again in the next wave
    assert h.m.compactions >= 2, h.m.compactions
    assert h.graph_finished(prod) == list(range(100, 150))


# random sequences: graph jobs between ticks, range pushes, cancels, handle re-use, proactive filling -------------------
def _dispose_for(h, released):
    """check_dispose_prefill (taskqueue.rs:146-152): a released task of higher priority than a class's prefilled tasks
    retracts them."""
    m = h.m
    pf = np.nonzero(m.has(LM.KEY_PF))[0]
    for c in sorted({int(m.cls[t]) for t in released}):
        top = max(int(m.prio[t]) for t in released if int(m.cls[t]) == c)
        held = pf[m.cls[pf] == c]
        if held.size and top > int(m.prio[held].min()):
            h.dispose(c)


@pytest.mark.parametrize("seed", range(4))
def test_random_drains_match_the_model_and_the_specification(harness, seed):
    h = harness
    rng = np.random.default_rng(100 + seed)
    q = 3
    h.classes(q)
    if seed % 2:
        h.set_prefill(RS.PREFILL)
    next_h, free_handles, job = 0, [], 0
    for step in range(40):
        m = h.m
        live = np.nonzero(m.has(LM.KEY_VALID))[0]
        # a job with dependencies: new handles and re-used ones of finished / cancelled tasks
        k = int(rng.integers(1, 60))
        reuse = [free_handles.pop(int(rng.integers(0, len(free_handles)))) for _ in range(min(len(free_handles), k // 3))]
        hs = reuse + list(range(next_h, next_h + k - len(reuse)))
        next_h += k - len(reuse)
        if rng.random() < 0.5:
            hs = sorted(hs)
        deps = []
        for i, x in enumerate(hs):
            pool = list(live[-80:]) + hs[:i] + hs[i + 1: i + 3]
            ds = {int(pool[j]) for j in rng.integers(0, len(pool), size=int(rng.integers(0, 4)))} - {x} if pool else set()
            deps.append(sorted(ds))
        h.graph_push(hs, rng.integers(0, q, size=k), [prio(int(rng.integers(0, 4)), job)] * k, *csr(deps))
        job += 1
        if rng.random() < 0.3:                        # a task array without dependencies
            r = list(range(next_h, next_h + 20))
            next_h += 20
            h.push(r, np.arange(20) % q, [prio(int(rng.integers(0, 4)), job)] * 20, as_range=True)
        if rng.random() < 0.3 and live.size:          # a cancel: a task and its waiting consumers leave
            victim = [int(x) for x in rng.choice(live, size=min(3, live.size), replace=False)]
            waiting = [c for v in victim for c, g in h.m.lists.get(v, []) if h.m._edge_waits(c, g)]
            gone = sorted(set(victim + waiting))
            h.remove(gone)
            free_handles += gone
        exp = h.tick(f"tick {step}")
        done = exp[exp["kind"] != 1]["task"] if exp is not None else np.zeros(0, np.uint32)
        fin = [int(x) for x in done if rng.random() < 0.8]
        if fin:
            made = h.graph_finished(fin + fin[:1], f"finish {step}")
            free_handles += fin
            if made and h.prefill is not None:
                _dispose_for(h, made)


# cfg4: the 500 k-node DAG submitted in batches drains exactly as hqs_dag_load drains it -----------------------------------
def test_cfg4_graph_push_drains_like_dag_load():
    wl = P.make_dag(500_000, 256, 16, seed=0)
    a = P.gpu_scheduler(wl)                           # hqs_dag_load
    b = P.gpu_scheduler(wl, add_tasks=False)
    from hyperqueue_b200 import priority_from_user
    prio_all = priority_from_user(wl.task_user_priority)
    n_ready = 0
    for lo in range(0, wl.n_tasks, 10_000):
        hi = min(lo + 10_000, wl.n_tasks)
        ds = wl.deps[lo:hi]
        off = np.concatenate([[0], np.cumsum([len(d) for d in ds])]).astype(np.uint32)
        flat = np.array([x for d in ds for x in d], dtype=np.uint32)
        n_ready += b.submit_tasks(np.arange(lo, hi, dtype=np.uint32), wl.task_class[lo:hi], prio_all[lo:hi], off, flat)
    assert n_ready == sum(1 for d in wl.deps if not d)
    waves, left = 0, wl.n_tasks
    while left and waves < 5000:
        ma, mb = a.run_scheduling(), b.run_scheduling()
        assert np.array_equal(ma.assignments, mb.assignments), waves
        assert np.array_equal(ma.free_after, mb.free_after), waves
        t = ma.assignments["task"]
        assert t.size, waves
        made_a = a.tasks_finished(t, propagate=True)
        made_b = b.graph_tasks_finished(t)
        assert made_b.size == made_a and (np.diff(made_b.astype(np.int64)) > 0).all()
        left -= t.size
        waves += 1
    assert left == 0 and waves == 1234
    assert np.array_equal(a.free, b.free) and np.array_equal(b.free, wl.worker_free)
    dbg = b.graph_debug()
    assert dbg[0] == 0 and dbg[3] == 0
    a.close()
    b.close()


def test_cpp_shim_graph_selftest():
    from hyperqueue_b200 import _lib
    assert _lib.load_shim().hqshim_selftest_graph(0, 1) == 0
