"""hqs_graph_cancel on the device against tests/graph_cancel_model.py: after every call the whole key array, hqs_graph_debug
and every returned list must equal the model's, on two contexts side by side (one per amount width), through
tests/test_gpu_graph.py's harness.  Ticks in between are compared with the sequential specification (tests/greedy_model.py)
and the judge.  Then GpuScheduler.graph_cancel_tasks on the cfg4 DAG against a host closure over its dependencies, and the
C++ shim's cancel self-test."""
import ctypes as C

import numpy as np
import pytest

import graph_cancel_model as CM
import level_model as LM
import parity as P
import test_gpu_graph as TG
import test_gpu_ready_set as RS
from test_gpu_graph import E_INVALID, E_STATE, _ptr, csr, prio

pytestmark = pytest.mark.gpu


class Harness(TG.Harness):
    def __init__(self):
        super().__init__()
        self.m = CM.CancelModel()

    def graph_cancel(self, t, label="graph_cancel"):
        t = np.ascontiguousarray(t, np.uint32)
        try:
            want = self.m.graph_cancel(t)
        except LM.Rejected:
            want = None
        launches = []
        for d in self.devs:
            ptr, k = C.POINTER(C.c_uint32)(), C.c_uint32(12345)
            before = d.stats()["kernel_launches"]
            rc = d.lib.hqs_graph_cancel(d.ctx, t.size, _ptr(t), C.byref(ptr), C.byref(k))
            launches.append(d.stats()["kernel_launches"] - before)
            if want is None:
                assert rc == E_INVALID, (label, rc)
                assert k.value == 0
            else:
                d.ok(rc)
                got = np.ctypeslib.as_array(ptr, shape=(k.value,)).tolist() if k.value else []
                assert got == want, (label, got[:8], want[:8], len(got), len(want))
        if want is not None:
            self.pfw[np.asarray(want, np.int64)] = -1
        self.check(label)
        self.last_launches = launches
        return want


@pytest.fixture
def harness():
    h = Harness()
    yield h
    h.close()


def test_rejections_and_mode_rules(harness):
    h = harness
    h.classes(2)
    h.graph_push([0, 1, 2], [0, 1, 0], [prio(1)] * 3, *csr([[], [0], [1]]))
    assert h.graph_cancel([0, 3]) is None                       # a handle >= n_handles: nothing changes
    assert h.graph_cancel([7]) is None
    assert h.graph_cancel([]) == []
    d = h.devs[0]
    ptr, k = C.POINTER(C.c_uint32)(), C.c_uint32(0)
    assert d.lib.hqs_graph_cancel(d.ctx, 1, None, C.byref(ptr), C.byref(k)) == E_INVALID
    h.check("null task array")
    # a pending tick refuses the call, and it works again after the fetch
    e = RS.Dev(0)
    try:
        e.classes(1)
        one = np.zeros(1, np.uint32)
        e.ok(e.lib.hqs_graph_push(e.ctx, 1, e.L.ptr(one), e.L.ptr(one), e.L.ptr(np.array([prio(0)], np.uint64)),
                                  e.L.ptr(np.zeros(2, np.uint32)), None, C.byref(k)))
        w = np.zeros(1, dtype=e.L.worker_dtype)
        w["remaining_time_ms"] = e.L.HQS_TIME_INF
        free = RS.W_TOTAL[:1].copy()
        e.ok(e.lib.hqs_tick_launch(e.ctx, 1, e.L.ptr(w), e.L.ptr(free), e.L.ptr(free), None, 4))
        assert e.lib.hqs_graph_cancel(e.ctx, 1, e.L.ptr(one), C.byref(ptr), C.byref(k)) == E_STATE
        out = np.zeros(4, dtype=e.L.assignment_dtype)
        e.ok(e.lib.hqs_tick_fetch(e.ctx, 4, e.L.ptr(out), C.byref(k), None))
        assert k.value == 1
        e.ok(e.lib.hqs_graph_cancel(e.ctx, 1, e.L.ptr(one), C.byref(ptr), C.byref(k)))
        assert k.value == 1 and ptr[0] == 0                     # the assigned task leaves
    finally:
        e.close()
    # a DAG context and an attached context refuse it
    p1, off = np.array([prio(0)], np.uint64), np.zeros(2, np.uint32)
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
            assert e.lib.hqs_graph_cancel(e.ctx, 1, e.L.ptr(one), C.byref(ptr), C.byref(k)) == E_STATE
        finally:
            e.close()
    assert h.graph_cancel([1, 1, 2]) == [1, 2]


def test_directed_cases(harness):
    h = harness
    h.classes(1)
    h.graph_push(np.arange(5), np.zeros(5), [prio(0)] * 5, *csr([[], [0], [0], [1, 2], [3]]))
    assert h.graph_cancel([0]) == [0, 1, 2, 3, 4]               # a diamond: 3 is listed once
    h.graph_push(np.arange(10, 14), np.zeros(4), [prio(0)] * 4, *csr([[], [10], [11], []]))
    assert h.graph_cancel([12, 10, 13, 1]) == [10, 11, 12, 13]    # 12 is a consumer of 10; 1 left already
    h.graph_push([20, 21], [0, 0], [prio(0)] * 2, *csr([[], [20]]))
    h.remove([21])
    h.graph_push([21], [0], [prio(0)], *csr([[]]))              # resubmitted without dependencies
    assert h.graph_cancel([20]) == [20]                         # the stale edge 20 -> 21 is not followed
    assert h.graph_cancel([0, 0, 20, 21, 21]) == [21]           # duplicates; 0 and 20 are not VALID


def test_a_chain_leaves_in_as_many_launches_as_a_lone_task(harness):
    h = harness
    h.classes(2)
    n = 20_000
    h.graph_push([n + 5], [0], [prio(0)], *csr([[]]))
    assert h.graph_cancel([n + 5]) == [n + 5]
    lone = h.last_launches
    h.graph_push(np.arange(n), np.arange(n) % 2, [prio(1)] * n, *csr([[]] + [[i] for i in range(n - 1)]))
    assert h.graph_cancel([0]) == list(range(n))
    assert h.last_launches == lone, (h.last_launches, lone)
    assert h.m.debug()[3] == 0


def test_a_fan_out_of_50000(harness):
    h = harness
    h.classes(3)
    n = 50_000
    h.graph_push(np.arange(n + 1), np.arange(n + 1) % 3, [prio(2)] * (n + 1), *csr([[]] + [[0]] * n))
    h.tick()                                                    # the root is assigned (DONE) and still VALID
    assert h.graph_cancel([0]) == list(range(n + 1))
    assert h.tick() is not None and h.m.debug() == [0, h.m.pool_cap, 0, 0]


@pytest.mark.parametrize("seed", range(3))
def test_prefilled_and_assigned_named_tasks(harness, seed):
    """Named tasks that are prefilled (READY | PREFILLED) and assigned (DONE) leave with their waiting consumers; the next
    ticks must equal the specification with the host's prefill mask."""
    h = harness
    rng = np.random.default_rng(seed)
    h.classes(3)
    h.set_prefill(RS.PREFILL)
    k = 400
    deps = [[] if i < 150 else sorted({int(x) for x in rng.integers(0, i, size=2)}) for i in range(k)]
    h.graph_push(np.arange(k), rng.integers(0, 3, size=k), [prio(int(rng.integers(0, 3)), 1) for _ in range(k)], *csr(deps))
    exp = h.tick("tick 0")
    asg = exp[exp["kind"] != 1]["task"].astype(np.int64)
    pf = np.nonzero(h.m.has(LM.KEY_PF))[0]
    assert asg.size and pf.size, (asg.size, pf.size)
    named = list(rng.choice(asg, size=min(5, asg.size), replace=False)) + list(rng.choice(pf, size=min(5, pf.size), replace=False))
    h.graph_cancel(named)
    for i in range(3):
        exp = h.tick(f"tick {i + 1}")
        done = exp[exp["kind"] != 1]["task"] if exp is not None else np.zeros(0, np.uint32)
        if done.size:
            made = h.graph_finished(done)
            if made:
                TG._dispose_for(h, made)


def test_after_a_compaction_and_past_65536_handles(harness):
    h = harness
    h.classes(2)
    prod = np.arange(100)
    h.graph_push(prod, prod % 2, [prio(2)] * 100, *csr([[]] * 100))
    rng = np.random.default_rng(7)
    cons = np.arange(1000, 2500)
    for wave in range(6):
        h.graph_push(cons, cons % 2, [prio(0, wave)] * cons.size, *csr([sorted({int(x) for x in rng.choice(prod, 2)}) for _ in cons]))
        if wave < 5:
            h.remove(cons)
    assert h.m.compactions >= 1
    h.graph_cancel(prod[::3])
    far = np.arange(70000, 70300)
    h.graph_push(far, far % 2, [prio(3)] * far.size, *csr([[int(p)] for p in rng.choice(prod, far.size)]))
    h.push(np.arange(140000, 140010), np.zeros(10), [prio(0)] * 10, as_range=True)
    h.graph_push([140020], [1], [prio(9)], *csr([[70001]]))
    h.graph_cancel(prod[1::3].tolist() + [140005])
    h.tick()
    h.graph_finished(prod[2::3])


@pytest.mark.parametrize("seed", range(4))
def test_random_sequences_match_the_model_and_the_specification(harness, seed):
    h = harness
    rng = np.random.default_rng(200 + seed)
    q = 3
    h.classes(q)
    if seed % 2:
        h.set_prefill(RS.PREFILL)
    next_h, free_handles, job = 0, [], 0
    for step in range(30):
        live = np.nonzero(h.m.has(LM.KEY_VALID))[0]
        k = int(rng.integers(1, 60))
        reuse = [free_handles.pop(int(rng.integers(0, len(free_handles)))) for _ in range(min(len(free_handles), k // 3))]
        hs = reuse + list(range(next_h, next_h + k - len(reuse)))
        next_h += k - len(reuse)
        deps = []
        for i, x in enumerate(hs):
            pool = list(live[-80:]) + hs[:i] * 2
            ds = {int(pool[j]) for j in rng.integers(0, len(pool), size=int(rng.integers(0, 4)))} - {x} if pool else set()
            deps.append(sorted(ds))
        h.graph_push(hs, rng.integers(0, q, size=k), [prio(int(rng.integers(0, 4)), job)] * k, *csr(deps))
        job += 1
        if rng.random() < 0.5 and live.size:
            victim = [int(x) for x in rng.choice(live, size=min(4, live.size), replace=False)]
            if rng.random() < 0.3:
                victim += victim[:1] + [int(rng.integers(0, max(next_h, 1)))]
            free_handles += h.graph_cancel(victim, f"cancel {step}")
        exp = h.tick(f"tick {step}")
        done = exp[exp["kind"] != 1]["task"] if exp is not None else np.zeros(0, np.uint32)
        fin = [int(x) for x in done if rng.random() < 0.8]
        if fin:
            made = h.graph_finished(fin, f"finish {step}")
            free_handles += fin
            if made and h.prefill is not None:
                TG._dispose_for(h, made)


def test_scheduler_messages_for_assigned_and_prefilled_tasks():
    """GpuScheduler.graph_cancel_tasks: CancelTasks lists per worker in the order the tasks were named, resources of the
    assigned tasks back, the prefilled task no longer held."""
    from hyperqueue_b200 import GpuScheduler, RequestVariant
    s = GpuScheduler(1)
    try:
        rid = s.get_or_create_resource_rq_id([RequestVariant.of({0: P.FR})])
        tot = np.array([[2 * P.FR], [2 * P.FR]], np.uint64)
        s.new_workers_bulk(np.array([50, 51], np.uint32), tot, tot.copy())
        s.set_prefill(0, 2)
        cons = {0: [8], 8: [9], 1: [10], 4: [11]}
        s.submit_tasks(np.arange(12), np.full(12, rid), np.full(12, prio(0), np.uint64), *csr([[]] * 8 + [[0], [8], [1], [4]]))
        m = s.run_scheduling()
        run = m.assignments[m.assignments["kind"] != 1]
        asg = run["task"].tolist()
        where = {t: int(s.worker_ids[w]) for t, w in zip(asg, run["worker"].tolist())}
        pf = sorted(s.prefilled_tasks(51).tolist())
        assert len(asg) == 4 and pf and asg[0] != asg[1]
        named = [pf[0], asg[1], 11, asg[1], asg[0]]
        want, stack = set(named), list(named)
        while stack:
            for c in cons.get(stack.pop(), []):
                want.add(c)
                stack.append(c)
        free0 = s.free.copy()
        gone, msgs = s.graph_cancel_tasks(named)
        assert gone.tolist() == sorted(want)
        exp = {}
        for t in (pf[0], asg[1], asg[0]):
            exp.setdefault(51 if t == pf[0] else where[t], []).append(t)
        assert msgs == exp
        assert int((s.free - free0).sum()) == 2 * P.FR
        assert s._pf_worker[pf[0]] == -1 and s._task_worker[asg[0]] == -1
    finally:
        s.close()


def test_cfg4_cancel_of_100_live_tasks_matches_a_host_closure():
    wl = P.make_dag(500_000, 256, 16, seed=0)
    s = P.gpu_scheduler(wl, add_tasks=False)
    from hyperqueue_b200 import priority_from_user
    prio_all = priority_from_user(wl.task_user_priority)
    for lo in range(0, wl.n_tasks, 10_000):
        hi = min(lo + 10_000, wl.n_tasks)
        ds = wl.deps[lo:hi]
        off = np.concatenate([[0], np.cumsum([len(d) for d in ds])]).astype(np.uint32)
        flat = np.array([x for d in ds for x in d], dtype=np.uint32)
        s.submit_tasks(np.arange(lo, hi, dtype=np.uint32), wl.task_class[lo:hi], prio_all[lo:hi], off, flat)
    assigned = np.zeros(wl.n_tasks, np.int64)
    finished = np.zeros(wl.n_tasks, bool)
    for _ in range(5):
        t = s.run_scheduling().assignments["task"]
        assigned[t] += 1
        s.graph_tasks_finished(t)
        finished[t] = True
    cons = [[] for _ in range(wl.n_tasks)]
    for t, ds in enumerate(wl.deps):
        for d in ds:
            cons[d].append(t)
    rng = np.random.default_rng(4)
    live = np.nonzero(~finished)[0]
    named = rng.choice(live, size=100, replace=False)
    want = set(int(x) for x in named)
    stack = list(want)
    while stack:                                                # every consumer of a live task still waits
        for c in cons[stack.pop()]:
            if c not in want:
                want.add(c)
                stack.append(c)
    gone, msgs = s.graph_cancel_tasks(named)
    assert gone.tolist() == sorted(want)
    assert sum(len(v) for v in msgs.values()) == 0              # nothing named was running: everything drains between waves
    cancelled = np.zeros(wl.n_tasks, bool)
    cancelled[gone] = True
    for _ in range(5000):
        t = s.run_scheduling().assignments["task"]
        if not t.size:
            break
        assigned[t] += 1
        s.graph_tasks_finished(t)
    assert (assigned[cancelled] == 0).all()
    assert (assigned[~cancelled] == 1).all()
    dbg = s.graph_debug()
    assert dbg[0] == 0 and dbg[3] == 0
    assert np.array_equal(s.free, wl.worker_free)
    s.close()


def test_cpp_shim_graph_cancel_selftest():
    from hyperqueue_b200 import _lib
    assert _lib.load_shim().hqshim_selftest_graph_cancel(0, 1) == 0
