"""hqs_handles_compact / GpuScheduler.compact_handles on the device.  Twin schedulers get the same call sequence: A compacts
its handles now and then, B never does.  A bijection maps each of B's handles to A's; new tasks take the next free handle
on each side (on A sometimes after a gap, whose keys must read 0).  After every call: tick records mapped through the
bijection (order, worker, variant, kind), free vectors, finished / cancel outputs, A's key of each survivor equal bit for bit
to B's key of its handle, the host mirrors, and hqs_graph_debug's waiting tasks (A's linked edges are at most B's: a
compaction drops the stale ones).  A handle of B that A retired
is not VALID on B; a call naming it reaches A without it (it would be ignored or dropped there too).
Then the rejections, a 16 M-slot table with 1 M survivors, the C++ shim's retire self-test, and one compaction script under
compute-sanitizer memcheck."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FR = 10_000
E_INVALID, E_STATE = -1, -6
KEY_VALID = 1 << 29
W_TOTAL = np.array([[12 * FR, 300000], [16 * FR, 400000], [8 * FR, 200000], [20 * FR, 500000]], dtype=np.uint64)
SANITIZER_ERROR = 7


def _sched(flags=0, q=3, prefill=None, workers=W_TOTAL):
    from hyperqueue_b200 import GpuScheduler
    from hyperqueue_b200.scheduler import RequestVariant
    s = GpuScheduler(2, 0, flags)
    for c in range(q):
        s.get_or_create_resource_rq_id([RequestVariant.of({0: (1 + c % 4) * FR, 1: (1 + c // 4) * 100})])
    s.new_workers_bulk(np.arange(10, 10 + workers.shape[0], dtype=np.uint32), workers)
    if prefill:
        s.set_prefill(*prefill)
    return s


def keys(s):
    n = C.c_uint32(0)
    s._check(s._lib.hqs_debug_keys(s._ctx, 0, None, C.byref(n)))
    out = np.zeros(n.value, np.uint32)
    if n.value:
        s._check(s._lib.hqs_debug_keys(s._ctx, n.value, out.ctypes.data_as(C.c_void_p), C.byref(n)))
    return out


class Twin:
    def __init__(self, flags=0, q=3, prefill=None, graph=False, workers=W_TOTAL):
        self.a = _sched(flags, q, prefill, workers)
        self.b = _sched(flags, q, prefill, workers)
        self.graph = graph
        self.b2a = {}
        self.na = self.nb = 0
        self.q = q
        self.compactions = 0

    def close(self):
        self.a.close()
        self.b.close()

    # handles ------------------------------------------------------------------------------------------------------
    def new(self, k, gap=0):
        hb = np.arange(self.nb, self.nb + k, dtype=np.uint32)
        self.na += gap
        ha = np.arange(self.na, self.na + k, dtype=np.uint32)
        self.nb += k
        self.na += k
        self.b2a.update(zip(hb.tolist(), ha.tolist()))
        return hb

    def amap(self, hb):
        """A's handles of B's, in order, without the ones A retired."""
        return np.array([self.b2a[b] for b in np.asarray(hb).tolist() if b in self.b2a], dtype=np.uint32)

    def bmap(self, ha):
        a2b = {v: k for k, v in self.b2a.items()}
        return [a2b[a] for a in np.asarray(ha).tolist()]

    # calls --------------------------------------------------------------------------------------------------------
    def push(self, hb, cls, prio):
        self.b.add_ready_tasks(hb, cls, prio)
        self.a.add_ready_tasks(self.amap(hb), cls, prio)
        self.check()

    def submit(self, hb, cls, prio, deps):
        off = np.cumsum([0] + [len(d) for d in deps]).astype(np.uint32)
        flat = np.array([x for d in deps for x in d], np.uint32)
        ra = self.b.submit_tasks(hb, cls, prio, off, flat)
        da = [self.amap(d) for d in deps]
        offa = np.cumsum([0] + [len(d) for d in da]).astype(np.uint32)
        flata = np.concatenate(da + [np.zeros(0, np.uint32)]).astype(np.uint32)
        assert self.a.submit_tasks(self.amap(hb), cls, prio, offa, flata) == ra
        self.check()

    def finish(self, hb):
        if self.graph:
            rb = self.b.graph_tasks_finished(hb)
            ra = self.a.graph_tasks_finished(self.amap(hb))
            assert self.bmap(ra) == rb.tolist()
        else:                             # a finished task leaves the table (retired with remove_ready_tasks)
            self.b.tasks_finished(hb)
            self.b.remove_ready_tasks(hb)
            self.a.tasks_finished(self.amap(hb))
            self.a.remove_ready_tasks(self.amap(hb))
        self.check()

    def cancel(self, hb):
        gb, mb = self.b.graph_cancel_tasks(hb)
        ga, ma = self.a.graph_cancel_tasks(self.amap(hb))
        assert self.bmap(ga) == gb.tolist()
        assert {w: self.bmap(v) for w, v in ma.items()} == {w: list(v) for w, v in mb.items()}
        self.check()
        return gb

    def remove(self, hb):
        self.b.remove_ready_tasks(hb)
        self.a.remove_ready_tasks(self.amap(hb))
        self.check()

    def tick(self):
        mb = self.b.run_scheduling()
        ma = self.a.run_scheduling()
        xa, xb = ma.assignments, mb.assignments
        assert xa.shape == xb.shape
        assert self.bmap(xa["task"]) == xb["task"].tolist()
        for f in ("worker", "variant", "kind"):
            assert (xa[f] == xb[f]).all(), f
        assert (ma.free_after == mb.free_after).all()
        self.check()
        return xb

    def start_prefilled(self, b, variant=0):
        self.b.on_task_running_prefilled(b, variant)
        self.a.on_task_running_prefilled(self.b2a[b], variant)
        self.check()

    def retract_response(self, wid, hb):
        rb = self.b.on_retract_response(wid, hb)
        ra = self.a.on_retract_response(wid, self.amap(hb))
        assert {w: [(self.bmap([t])[0], v) for t, v in l] for w, l in ra.items()} == rb

    def dispose(self, c):
        rb = self.b.dispose_prefill(c)
        ra = self.a.dispose_prefill(c)
        assert {w: self.bmap(v) for w, v in ra.items()} == rb
        self.check()

    def compact(self, keep_b=()):
        kb = keys(self.b)
        n_b = kb.size
        # B's view of what must survive: VALID keys, what its mirror tracks, and keep
        m = min(n_b, self.b._task_worker.shape[0])
        want_b = set(np.nonzero(kb & KEY_VALID)[0].tolist())
        want_b |= set(np.nonzero((self.b._task_worker[:m] >= 0) | (self.b._pf_worker[:m] >= 0))[0].tolist())
        want_b |= set(self.b.redirects) | set(self.b._retracting_from) | set(int(x) for x in keep_b)
        assert want_b <= set(self.b2a), "a handle B still uses was retired on A"
        before = self.a._lib_stats().kernel_launches
        old = self.a.compact_handles(self.amap(sorted(keep_b)) if len(keep_b) else None)
        launches = self.a._lib_stats().kernel_launches - before
        assert launches <= 8, launches
        assert old.tolist() == sorted(self.b2a[b] for b in want_b)
        new_of_old = {int(o): i for i, o in enumerate(old.tolist())}
        self.b2a = {b: new_of_old[a] for b, a in self.b2a.items() if a in new_of_old}
        self.na = old.size
        assert self.a._lib_stats().n_handles == old.size
        self.compactions += 1
        self.check()
        return old

    # comparison ---------------------------------------------------------------------------------------------------
    def check(self):
        ka, kb = keys(self.a), keys(self.b)
        a_of = np.full(ka.size, -1, np.int64)
        for b, a in self.b2a.items():
            if b < kb.size and a < ka.size:
                assert ka[a] == kb[b], (b, a, hex(ka[a]), hex(kb[b]))
                a_of[a] = b
            elif b < kb.size:
                assert kb[b] & KEY_VALID == 0, b
        assert (ka[a_of < 0] == 0).all(), "a slot A never handed out after a compaction is not zero"
        for b in range(kb.size):
            if b not in self.b2a:
                assert kb[b] & KEY_VALID == 0, b
        # host mirrors of the tracked tasks
        for b, a in self.b2a.items():
            if b < self.b._task_worker.shape[0] and a < self.a._task_worker.shape[0]:
                assert self.a._task_worker[a] == self.b._task_worker[b]
                assert self.a._pf_worker[a] == self.b._pf_worker[b]
                if self.b._task_worker[b] >= 0:
                    assert self.a._task_variant[a] == self.b._task_variant[b]
        assert {self.bmap([t])[0]: v for t, v in self.a.redirects.items()} == self.b.redirects
        assert {self.bmap([t])[0]: v for t, v in self.a._retracting_from.items()} == self.b._retracting_from
        assert (self.a.free == self.b.free).all()
        if self.graph:
            da, db = self.a.graph_debug(), self.b.graph_debug()
            # A's compactions drop the stale edges that B's lists still hold
            assert da[0] <= db[0] and da[3] == db[3], (da, db)


@pytest.fixture
def twins():
    made = []

    def make(**kw):
        t = Twin(**kw)
        made.append(t)
        return t
    yield make
    for t in made:
        t.close()


def prio(user, job=0):
    return (((int(user) & 0xFFFFFFFF) ^ 0x80000000) << 32) | int(job)


def _live(t):
    kb = keys(t.b)
    return np.nonzero(kb & KEY_VALID)[0]


@pytest.mark.parametrize("flags", [0, 2])
@pytest.mark.parametrize("seed", [1, 2])
def test_plain_ready_set_random(twins, flags, seed):
    rng = np.random.default_rng(seed)
    t = twins(flags=flags)
    for step in range(60):
        op = rng.integers(0, 6)
        if op <= 1:
            k = int(rng.integers(1, 300))
            t.push(t.new(k, gap=int(rng.integers(0, 3))), rng.integers(0, 3, k), [prio(int(u)) for u in rng.integers(0, 4, k)])
        elif op == 2:
            x = t.tick()
            done = x["task"][x["kind"] != 1]
            if done.size:
                t.finish(rng.choice(done, size=max(1, done.size // 2), replace=False))
        elif op == 3 and t.nb:
            t.remove(rng.integers(0, t.nb, int(rng.integers(1, 50))))
        elif op == 4:
            t.compact()
        else:
            t.tick()
    assert t.compactions > 0
    t.compact()


def test_proactive_filling_across_compactions(twins):
    rng = np.random.default_rng(7)
    t = twins(prefill=(2, 3))
    kinds = set()
    started = False
    for step in range(60):
        if step % 3 == 0:                 # few new tasks: the prefilled ones are assigned elsewhere (kind 2)
            k = int(rng.integers(5, 40))
            t.push(t.new(k), rng.integers(0, 3, k), [prio(int(u)) for u in rng.integers(0, 2, k)])
        x = t.tick()
        kinds |= set(x["kind"].tolist())
        # a worker starts one of its prefilled tasks: it leaves the table but is still tracked (kept through keep)
        held = [b for b in range(min(t.nb, t.b._pf_worker.shape[0])) if t.b._pf_worker[b] >= 0]
        if held and rng.integers(0, 2):
            b = int(rng.choice(held))
            t.start_prefilled(b)
            started = True
            if rng.integers(0, 2):
                t.compact()
                assert b in t.b2a
        for b, wid in list(t.b._retracting_from.items())[:3]:    # the workers give retracted tasks back
            t.retract_response(wid, [b])
        done = x["task"][x["kind"] == 0]
        if done.size:
            t.finish(done)
        if rng.integers(0, 4) == 0:
            t.dispose(int(rng.integers(0, 3)))
        if rng.integers(0, 3) == 0:
            t.compact()
    assert started and {1, 2} <= kinds, kinds
    t.compact()


@pytest.mark.parametrize("mode", ["declared", "pruned", "coarse"])
def test_levels(twins, mode):
    rng = np.random.default_rng(11)
    t = twins(q=3)
    if mode == "declared":
        for s in (t.a, t.b):
            s._sync_classes()
            p = np.array([prio(u, j) for u in range(3) for j in range(40)], np.uint64)
            s._check(s._lib.hqs_levels_add(s._ctx, p.size, p.ctypes.data_as(C.c_void_p)))
    n_jobs = 3000 if mode == "coarse" else 40
    for step in range(12):
        k = 1500 if mode == "coarse" else 150
        # pruned: new jobs with every push, so the level set keeps doubling and the dead levels are pruned
        jobs = rng.integers(step * 100, step * 100 + 20, k) if mode == "pruned" else rng.integers(0, n_jobs, k)
        t.push(t.new(k), rng.integers(0, 3, k), [prio(int(u), int(j)) for u, j in zip(rng.integers(0, 3, k), jobs)])
        x = t.tick()
        done = x["task"][x["kind"] == 0]
        if done.size:
            t.finish(done)
        if step % 3 == 2:
            t.compact()
    if mode == "coarse":
        assert t.a._lib_stats().coarsened == 1 and t.b._lib_stats().coarsened == 1


@pytest.mark.parametrize("flags", [0, 2])
@pytest.mark.parametrize("seed", [3, 4])
def test_graphs_random(twins, flags, seed):
    rng = np.random.default_rng(seed)
    t = twins(flags=flags, graph=True)
    resubmitted = cancels = 0
    for step in range(80):
        op = rng.integers(0, 8)
        if op <= 2:
            k = int(rng.integers(1, 40))
            hb = t.new(k, gap=int(rng.integers(0, 2)))
            lo = max(0, t.nb - 300)
            deps = [sorted(set(rng.integers(lo, int(hb[i]), int(rng.integers(0, 4))).tolist())) if hb[i] > 0 else []
                    for i in range(k)]
            t.submit(hb, rng.integers(0, 3, k), [prio(int(u)) for u in rng.integers(0, 3, k)], deps)
        elif op == 3:
            x = t.tick()
            done = x["task"][x["kind"] == 0]
            if done.size:
                t.finish(done)
        elif op == 4 and t.nb:
            cancels += len(t.cancel(rng.integers(0, t.nb, int(rng.integers(1, 4)))))
        elif op == 5 and t.nb:
            # a removed handle that B still tracks (named in keep, so A keeps it too) is submitted again
            b = int(rng.integers(max(0, t.nb - 100), t.nb))
            if b in t.b2a and not keys(t.b)[b] & KEY_VALID and t.b._task_worker[b] < 0:
                t.compact(keep_b=[b])
                t.submit(np.array([b], np.uint32), [0], [prio(0)], [sorted(x for x in _live(t)[-3:].tolist() if x < b)])
                resubmitted += 1
            else:
                t.remove([b])
        elif op == 6:
            t.compact()
        else:
            t.tick()
    t.compact()
    assert t.compactions > 3 and cancels > 0


def test_empty_identity_and_keep_nothing(twins):
    t = twins(graph=True)
    old = t.compact()                                       # an empty table
    assert old.size == 0
    hb = t.new(50)
    t.submit(hb, np.zeros(50, np.uint32), [prio(0)] * 50, [[] if i == 0 else [i - 1] for i in range(50)])
    before = keys(t.a)
    old = t.compact()                                       # everything is VALID: the identity
    assert old.tolist() == list(range(50)) and (keys(t.a) == before).all()
    t.cancel([0])                                           # the whole chain leaves
    old = t.compact()
    assert old.size == 0 and keys(t.a).size == 0
    hb = t.new(3)
    assert t.b2a[int(hb[0])] == 0                           # the next push takes handle 0
    t.submit(hb, np.zeros(3, np.uint32), [prio(1)] * 3, [[], [int(hb[0])], []])
    t.tick()


def test_rejections_change_nothing():
    from hyperqueue_b200 import _lib as L
    s = _sched()
    try:
        s.add_ready_tasks(np.arange(100), np.zeros(100, np.uint32), [prio(0)] * 100)
        s.remove_ready_tasks(np.arange(0, 100, 2))
        k0 = keys(s)
        lib, ptr, n = s._lib, C.POINTER(C.c_uint32)(), C.c_uint32(7)
        bad = np.array([3, 100], np.uint32)
        assert lib.hqs_handles_compact(s._ctx, 2, bad.ctypes.data_as(C.c_void_p), C.byref(ptr), C.byref(n)) == E_INVALID
        assert n.value == 0
        assert lib.hqs_handles_compact(s._ctx, 1, None, C.byref(ptr), C.byref(n)) == E_INVALID
        w = s._worker_structs(0.0)
        free = np.ascontiguousarray(s.free)
        s._check(lib.hqs_tick_launch(s._ctx, w.size, L.ptr(w), L.ptr(free), L.ptr(free), None, 200))
        assert lib.hqs_handles_compact(s._ctx, 0, None, C.byref(ptr), C.byref(n)) == E_STATE
        out = np.zeros(200, dtype=L.assignment_dtype)
        s._check(lib.hqs_tick_fetch(s._ctx, 200, L.ptr(out), C.byref(n), None))
        k1 = keys(s)
        assert k1.size == k0.size and ((k1 & KEY_VALID) != 0).sum() == ((k0 & KEY_VALID) != 0).sum()
        # a DAG context, an attached context, a sharded graph context
        for mode in ("dag", "attach", "shard_graph"):
            e = _sched()
            try:
                e._sync_classes()
                one = np.zeros(1, np.uint32)
                if mode == "dag":
                    e._check(lib.hqs_dag_load(e._ctx, 1, L.ptr(one), L.ptr(np.zeros(1, np.uint64)), L.ptr(one),
                                              L.ptr(np.zeros(2, np.uint32)), None))
                elif mode == "attach":
                    xb = C.c_void_p()
                    e._check(lib.hqs_shard_xbuf(e._ctx, C.byref(xb), None))
                    e._check(lib.hqs_shard_attach(e._ctx, 1, 0, (C.c_void_p * 1)(xb)))
                else:
                    e._check(lib.hqs_shard_graph_init(e._ctx, 100, 0, 50))
                assert lib.hqs_handles_compact(e._ctx, 0, None, C.byref(ptr), C.byref(n)) == E_STATE
            finally:
                e.close()
        assert (keys(s) == k1).all()
        s.compact_handles()
        assert keys(s).size == int(((k1 & KEY_VALID) != 0).sum())
    finally:
        s.close()


def test_sixteen_million_slots_with_one_million_survivors(twins):
    n, live = 16 << 20, 1 << 20
    t = twins(workers=np.tile(W_TOTAL, (64, 1)))
    hb = t.new(n)
    cls = (np.arange(n) % 3).astype(np.uint32)
    p = np.full(n, prio(0), np.uint64)
    t.b.add_ready_tasks(hb, cls, p)
    t.a.add_ready_tasks(t.amap(hb), cls, p)
    gone = np.setdiff1d(np.arange(n, dtype=np.uint32), np.linspace(0, n - 1, live).astype(np.uint32))
    t.b.remove_ready_tasks(gone)
    t.a.remove_ready_tasks(t.amap(gone))
    old = t.compact()
    assert old.size == live
    t.tick()
    # a push after a gap: the slots between n_kept and it read 0
    g = t.new(1, gap=1000)
    t.push(g, [0], [prio(1)])
    assert (keys(t.a)[live: live + 1000] == 0).all()
    t.tick()


def test_cpp_shim_retire_selftest():
    from hyperqueue_b200 import _lib as L
    shim = L.load_shim()
    assert shim.hqshim_selftest_retire(0, 1) == 0


# ------------------------------------------------------------------------------------------------------------------------
# one compaction script under compute-sanitizer memcheck (no cooperative launch: no cancel, plain tick kernels)
def exercise() -> None:
    from hyperqueue_b200 import _lib as L
    lib = L.load_library()
    cudart = C.CDLL("libcudart.so.12")
    s = _sched()
    n = 5000
    h = np.arange(n, dtype=np.uint32)
    off = np.concatenate([[0], np.cumsum(np.arange(n) % 3 != 0)]).astype(np.uint32)
    deps = np.array([i - 1 for i in range(n) if i % 3 != 0], np.uint32)
    s.submit_tasks(h, h % 3, np.full(n, prio(0), np.uint64), off, deps)
    s.run_scheduling()
    s.graph_tasks_finished(np.arange(0, n, 3, dtype=np.uint32))
    s.remove_ready_tasks(np.arange(1, n, 7, dtype=np.uint32))
    s.compact_handles()
    s.compact_handles(keep=[0])
    s.run_scheduling()
    s.close()
    assert cudart.cudaDeviceReset() == 0


def test_compaction_under_memcheck():
    tool = shutil.which("compute-sanitizer") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin",
                                                               "compute-sanitizer")
    if not os.path.exists(tool):
        pytest.skip("compute-sanitizer is not installed")
    import __graft_entry__ as ge
    ge.build()
    cmd = [tool, "--tool", "memcheck", "--leak-check", "full", "--error-exitcode", str(SANITIZER_ERROR),
           sys.executable, os.path.abspath(__file__)]
    r = subprocess.run(cmd, env=dict(os.environ, HQS_DEBUG_NO_COOP="1"), cwd=ROOT, capture_output=True, text=True,
                       timeout=900)
    log = r.stdout + r.stderr
    tool_errors = [ln for ln in log.splitlines() if ln.startswith("========= Error: ") and "terminate successfully" not in ln]
    if tool_errors:
        pytest.skip("compute-sanitizer cannot check this process: " + tool_errors[0])
    assert r.returncode == 0 and "ERROR SUMMARY: 0 errors" in log and "Leaked" not in log, log[-4000:]


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    exercise()
