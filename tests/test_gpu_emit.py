"""The emit step's two finishing passes, record by record: the staged pass (each chunk's assignments written as per-group
runs staged in shared memory, HQS_PATH_EMIT_STAGED) and the per-task pass that HQS_DEBUG_EMIT_PER_TASK forces, both against
the sequential specification.  Cases: the bench shape at reduced size, ragged table tails, more chunks than worker CTAs, a
packed level (the chunk is ranked again after the pack command), out_cap below the assignments, the two-context sharded
tick on one GPU, prefilled tasks in the assigned range (kind 2) and a group count that leaves no room for the staging
buffer.  Every case asserts which pass ran."""
import ctypes as C

import numpy as np
import pytest

import greedy_model as G
import parity as P
import prefill_scenarios as S
from hyperqueue_b200 import _lib as L

pytestmark = pytest.mark.gpu
PER_TASK = "HQS_DEBUG_EMIT_PER_TASK"
STAGED = L.HQS_PATH_EMIT_STAGED


def _set_pass(monkeypatch, per_task):
    if per_task:
        monkeypatch.setenv(PER_TASK, "1")
    else:
        monkeypatch.delenv(PER_TASK, raising=False)


def _both_passes(monkeypatch, wl, staged, flags=0):
    """One tick with each pass: both equal the specification; the staged pass runs iff `staged` (and not forced off)."""
    exp, exp_free = G.model_tick(wl, np.ones(wl.n_tasks, dtype=bool), wl.worker_free.copy(), pack=not (flags & L.HQS_CREATE_NO_PACK))
    for per_task in (False, True):
        _set_pass(monkeypatch, per_task)
        s = P.gpu_scheduler(wl, flags=flags)
        m = s.run_scheduling()
        path = s.stats()["solver_path"]
        s.close()
        assert np.array_equal(m.assignments, exp), (per_task, m.n_assigned(), exp.size)
        assert np.array_equal(m.free_after, exp_free), per_task
        assert bool(path & STAGED) == (staged and not per_task), (per_task, hex(path))
    return exp


CASES = {
    # cfg2-M1 shape (256 workers, Q = 16, 8 levels, every task assignable) at a fifth of the bench's task count
    "bench_shape": (lambda: P.make_independent(200_000, 256, 16, seed=0, free_scale=1024), 0, True),
    # a table that ends inside a row of 32 and inside a chunk; a table shorter than one row
    "ragged_tail": (lambda: P.make_independent(100_003, 64, 12, seed=2, free_scale=1024), 0, True),
    "tiny_table": (lambda: P.make_independent(37, 4, 3, seed=3, free_scale=1024), 0, True),
    # only part of the table is assigned: runs end inside chunks, later chunks have no work
    "partly_assigned": (lambda: P.make_independent(150_001, 64, 16, seed=5, free_scale=1), L.HQS_CREATE_NO_PACK, True),
    # 65 worker CTAs (half of the SMs), 20-row chunks of 10 240 slots: 69 chunks, some CTAs emit two
    "more_chunks_than_ctas": (lambda: P.make_independent(700_001, 64, 8, seed=6, free_scale=1024), L.HQS_CREATE_SHARE_DEVICE, True),
    # a saturated level is packed first: the worker CTAs run a pack command and rank their chunk after it
    "packed_level": (lambda: P.make_independent(80_000, 300, 16, seed=14, free_scale=1), 0, True),
    # 1500 classes x 2 levels = 3000 groups: the run records and the staging buffer do not fit next to the counters
    "many_groups": (lambda: P.Workload(3, [[{"amounts": {c % 3: (c // 3 + 1) * P.FR}}] for c in range(1500)],
                                       np.full((64, 3), 500_000 * P.FR, dtype=np.uint64), np.full((64, 3), 500_000 * P.FR, dtype=np.uint64),
                                       np.random.default_rng(3).integers(0, 1500, 40_000).astype(np.uint32),
                                       np.random.default_rng(4).integers(0, 2, 40_000).astype(np.int32)), 0, False),
}


@pytest.mark.parametrize("name", list(CASES))
def test_staged_and_per_task_pass_equal_the_specification(monkeypatch, name):
    build, flags, staged = CASES[name]
    exp = _both_passes(monkeypatch, build(), staged, flags)
    assert exp.size > 0


@pytest.mark.parametrize("per_task", [False, True], ids=["staged", "per_task"])
def test_out_cap_below_the_assignments(monkeypatch, per_task):
    """The solver sees that out_cap is too small before the emit step: nothing is emitted, the ready set stays intact, and
    the next tick with room emits exactly the specification."""
    _set_pass(monkeypatch, per_task)
    wl = P.make_independent(50_000, 32, 8, seed=7, free_scale=1024)
    exp, exp_free = G.model_tick(wl, np.ones(wl.n_tasks, dtype=bool), wl.worker_free.copy())
    s = P.gpu_scheduler(wl)
    with pytest.raises(Exception):
        s.run_scheduling(out_cap=exp.size - 1)
    assert s.stats()["solver_path"] & STAGED == 0
    s.free = wl.worker_free.copy()
    m = s.run_scheduling()
    assert np.array_equal(m.assignments, exp) and np.array_equal(m.free_after, exp_free)
    assert bool(s.stats()["solver_path"] & STAGED) == (not per_task)
    s.close()


def _shard_workload(wl, lo, hi):
    import copy
    w2 = copy.copy(wl)
    w2.task_class = wl.task_class[lo:hi]
    w2.task_user_priority = wl.task_user_priority[lo:hi]
    return w2


@pytest.mark.parametrize("per_task", [False, True], ids=["staged", "per_task"])
def test_two_context_sharded_tick_on_one_gpu(monkeypatch, per_task):
    """Fused sharded tick, two contexts of one process on half of the SMs each: rank 1 emits its runs behind the counts
    of rank 0 (`before`).  The merged records equal the specification of the whole table."""
    from hyperqueue_b200 import priority_from_user
    from hyperqueue_b200.sharded import block_range
    _set_pass(monkeypatch, per_task)
    n, w = 100_001, 64
    wl = P.make_independent(n, w, 16, seed=4, free_scale=1024)
    exp, exp_free = G.model_tick(wl, np.ones(n, dtype=bool), wl.worker_free.copy())
    parts = []
    xb = (C.c_void_p * 2)()
    lv = np.ascontiguousarray(np.unique(priority_from_user(wl.task_user_priority)))
    for r in range(2):
        lo, hi = block_range(n, r, 2)
        s = P.gpu_scheduler(_shard_workload(wl, lo, hi), add_tasks=False, flags=L.HQS_CREATE_SHARE_DEVICE)
        s._sync_classes()
        s._check(s._lib.hqs_levels_add(s._ctx, lv.size, L.ptr(lv)))
        s.add_ready_tasks(np.arange(hi - lo, dtype=np.uint32), wl.task_class[lo:hi], priority_from_user(wl.task_user_priority[lo:hi]))
        p = C.c_void_p()
        s._check(s._lib.hqs_shard_xbuf(s._ctx, C.byref(p), None))
        xb[r] = p
        parts.append((s, lo, hi))
    for r, (s, lo, hi) in enumerate(parts):
        s._check(s._lib.hqs_shard_attach(s._ctx, 2, r, xb))
        s._check(s._lib.hqs_tick_reserve(s._ctx, w, hi - lo, 0))
    workers = parts[0][0]._worker_structs(0.0)
    free = np.ascontiguousarray(wl.worker_free); total = np.ascontiguousarray(wl.worker_total)
    for s, lo, hi in parts:
        s._check(s._lib.hqs_shard_tick_launch(s._ctx, w, L.ptr(workers), L.ptr(free), L.ptr(total), None, hi - lo))
    merged = []
    for s, lo, hi in parts:
        out = np.zeros(hi - lo, dtype=L.assignment_dtype)
        nn = C.c_uint32(0)
        fa = np.zeros_like(free)
        s._check(s._lib.hqs_tick_fetch(s._ctx, hi - lo, L.ptr(out), C.byref(nn), L.ptr(fa)))
        assert np.array_equal(fa, exp_free)
        assert bool(s.stats()["solver_path"] & STAGED) == (not per_task)
        a = out[: nn.value].copy()
        a["task"] += np.uint32(lo)
        merged.append(a)
    for s, lo, hi in parts:
        s.close()
    got = np.concatenate(merged)
    assert got.size == exp.size > 0
    # each rank emits its own tasks in the specification's order: rank 0's records, then rank 1's, both in order
    for a, (_, lo, hi) in zip(merged, parts):
        sel = (exp["task"] >= lo) & (exp["task"] < hi)
        assert np.array_equal(a, exp[sel])


@pytest.mark.parametrize("per_task", [False, True], ids=["staged", "per_task"])
def test_prefill_scenarios(monkeypatch, per_task):
    """Proactive filling: a tick with a prefill range (kind-1 records behind the assignments) keeps the per-task pass; a
    tick without one emits its retract-and-redirect records (kind 2) through the staged pass."""
    from hyperqueue_b200 import GpuScheduler, RequestVariant, priority_from_user
    _set_pass(monkeypatch, per_task)
    kind2_staged = 0
    for name in sorted(S.SCENARIOS):
        reserve, pmax, cpus, steps = S.SCENARIOS[name]
        _, exp = S.run_spec(name)
        s = GpuScheduler(1)
        c = s.get_or_create_resource_rq_id([RequestVariant.of({0: cpus * S.FR})])
        s.set_prefill(reserve, pmax)
        n_w = n_t = 0
        for tick, (new_w, new_t) in enumerate(steps):
            for cp in new_w:
                s.new_worker(50 + n_w, [cp * S.FR]); n_w += 1
            if new_t:
                h = np.arange(n_t, n_t + new_t, dtype=np.uint32)
                s.add_ready_tasks(h, np.full(new_t, c, dtype=np.uint32), priority_from_user(np.zeros(new_t)))
                n_t += new_t
            m = s.run_scheduling()
            got = m.assignments
            assert np.array_equal(got, exp[tick]), (name, tick)
            path = s.stats()["solver_path"]
            staged = not per_task and not np.any(got["kind"] == 1)
            assert bool(path & STAGED) == staged, (name, tick, hex(path))
            if staged and np.any(got["kind"] == 2):
                kind2_staged += 1
        s.close()
    assert per_task or kind2_staged > 0
