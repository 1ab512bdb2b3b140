"""Edge cases of the CUDA path through the C ABI: maximum sizes (1024 workers, 16 resource kinds, 8 variants),
large class tables (global-memory class path), more (level x class) groups than HQS_MAX_GROUPS, handle re-use,
class-table growth, empty capacity, and the error contract (no partial results, ready set unchanged)."""
import ctypes as C

import numpy as np
import pytest

import greedy_model as G
import parity as P

pytestmark = pytest.mark.gpu
FR = P.FR


def _random_workload(n, w, q, r, vmax, seed, n_prio=5, cap=(8, 64)):
    rng = np.random.default_rng(seed)
    classes = []
    seen = set()
    while len(classes) < q:
        vs = []
        for _ in range(int(rng.integers(1, vmax + 1))):
            k = int(rng.integers(1, min(r, 4) + 1))
            rs = rng.choice(r, size=k, replace=False)
            vs.append({"amounts": {int(x): int(rng.integers(1, 9)) * FR // int(rng.choice([1, 2, 4])) for x in rs}})
        key = repr([sorted(d["amounts"].items()) for d in vs])
        if key not in seen:
            seen.add(key); classes.append(vs)
    total = (rng.integers(cap[0], cap[1], size=(w, r)).astype(np.uint64)) * np.uint64(FR)
    return P.Workload(r, classes, total, total.copy(), rng.integers(0, q, n).astype(np.uint32),
                      rng.integers(0, n_prio, n).astype(np.int32))


def _check_exact(wl, expect_narrow=None, path_bits=0):
    """Both amount widths of the solver (gcd-scaled 32-bit and plain 64-bit) against the sequential spec; path_bits:
    HQS_PATH_* bits both ticks must report."""
    out = None
    for flags in (0, 2):
        s = P.gpu_scheduler(wl, flags=flags)
        fb = s.free.copy()
        m = s.run_scheduling()
        assert P.judge_tick(wl, fb, m.assignments).ok
        exp, exp_free = G.model_tick(wl, np.ones(wl.n_tasks, dtype=bool), fb)
        assert np.array_equal(m.assignments, exp)
        assert np.array_equal(m.free_after, exp_free)
        narrow = s.stats()["narrow_amounts"]
        assert s.stats()["solver_path"] & path_bits == path_bits, (flags, hex(s.stats()["solver_path"]))
        if flags == 2:
            assert narrow == 0
        elif expect_narrow is not None:
            assert narrow == int(expect_narrow)
        s.close()
        out = out or m
    return out


def test_maximum_workers_resources_variants():
    from hyperqueue_b200 import _lib as L
    m = _check_exact(_random_workload(30000, 1024, 12, 16, 8, seed=1), path_bits=L.HQS_PATH_GENERAL)
    assert m.n_assigned() > 1000


def test_eight_resources_path():
    _check_exact(_random_workload(20000, 100, 10, 7, 3, seed=2))


def test_large_class_table_uses_global_class_path():
    # 1500 classes x 648 B > the shared-memory budget of the solver => ClassT read from global memory
    from hyperqueue_b200 import _lib as L
    m = _check_exact(_random_workload(40000, 64, 1500, 4, 1, seed=3, n_prio=2), path_bits=L.HQS_PATH_CLASSES_GLOBAL)
    assert m.n_assigned() > 100


def test_many_live_levels_stay_exact_up_to_the_group_limit():
    """test_many_cuts shape (test_scheduler_sn.rs:1129-1146): 3200 priority levels x 2 classes = 6400 groups fit
    HQS_MAX_GROUPS (8192): no coarsening, the tick equals the specification and strict priority order holds."""
    rng = np.random.default_rng(5)
    n = 6400
    classes = [[{"amounts": {0: 1 * FR}}], [{"amounts": {0: 2 * FR}}]]
    total = np.full((300, 1), 8 * FR, dtype=np.uint64)
    wl = P.Workload(1, classes, total, total.copy(), (np.arange(n) % 2).astype(np.uint32), (np.arange(n) // 2).astype(np.int32))
    s = P.gpu_scheduler(wl)
    fb = s.free.copy()
    m = s.run_scheduling()
    st = s.stats()
    assert st["coarsened"] == 0 and st["n_levels"] == 3200
    exp, exp_free = G.model_tick(wl, np.ones(n, dtype=bool), fb)
    assert np.array_equal(m.assignments, exp) and np.array_equal(m.free_after, exp_free)
    assert (np.diff(wl.task_user_priority[m.assignments["task"]]) <= 0).all()
    cnt = np.bincount(wl.task_class[m.assignments["task"]], minlength=2)
    assert abs(int(cnt[0]) - 800) <= 10 and abs(int(cnt[1]) - 800) <= 10      # the reference pins 800 / 800 +- 10
    s.close()


def test_more_groups_than_the_limit_are_coarsened():
    wl = _random_workload(60000, 128, 300, 4, 2, seed=4, n_prio=40)      # 300 x 40 = 12000 groups > 8192
    s = P.gpu_scheduler(wl)
    fb = s.free.copy()
    m = s.run_scheduling()
    assert s.stats()["coarsened"] == 1 and m.n_assigned() > 100
    assert P.judge_tick(wl, fb, m.assignments).ok
    # coarsening merges adjacent levels but never inverts the order of far-apart priorities:
    pr = wl.task_user_priority[m.assignments["task"]]
    assert pr[: max(1, pr.size // 10)].mean() >= pr[-max(1, pr.size // 10):].mean()
    s.close()


def test_handle_reuse_and_class_table_growth():
    from hyperqueue_b200 import RequestVariant, priority_from_user
    wl = P.make_independent(3000, 8, 4, seed=5)
    s = P.gpu_scheduler(wl)
    first = s.run_scheduling()
    assert first.n_assigned() > 0
    s.tasks_finished(first.assignments["task"])
    # a new class appears after tasks were pushed (ResourceRqMap is append-only) ...
    new_c = s.get_or_create_resource_rq_id([RequestVariant.of({0: 1 * FR})])
    assert new_c == len(wl.classes)
    # ... and the finished handles are re-used for tasks of that class with a higher priority than everything
    h = first.assignments["task"][:50].copy()
    s.add_ready_tasks(h, np.full(h.size, new_c, dtype=np.uint32), priority_from_user(np.full(h.size, 100)))
    second = s.run_scheduling()
    got = set(second.assignments["task"].tolist())
    assert set(h.tolist()) <= got                        # top priority, 1 cpu each: all placed
    assert (second.assignments["task"][: h.size] == np.sort(h)).all()   # and emitted first, in handle order
    s.close()


def test_no_capacity_no_assignment_and_ready_set_kept():
    wl = P.make_independent(2000, 4, 3, seed=6)
    wl.worker_free = np.zeros_like(wl.worker_free)
    s = P.gpu_scheduler(wl)
    assert s.run_scheduling().n_assigned() == 0
    s.free = wl.worker_total.copy()                      # resources come back: the same ready set is still there
    assert s.run_scheduling().n_assigned() > 0
    s.close()


def test_error_contract():
    from hyperqueue_b200 import GpuScheduler, HqsError, RequestVariant, _lib as L, priority_from_user
    with pytest.raises(HqsError):
        GpuScheduler(17)                                  # > HQS_MAX_RESOURCES
    s = GpuScheduler(2)
    with pytest.raises(HqsError):                         # tick before any class exists
        s.new_worker(1, [4 * FR, 0]); s.run_scheduling()
    s.get_or_create_resource_rq_id([RequestVariant.of({0: 1 * FR})])
    with pytest.raises(HqsError):                         # class id out of range
        s.add_ready_tasks(np.arange(3, dtype=np.uint32), np.array([0, 1, 0], dtype=np.uint32), priority_from_user(np.zeros(3)))
    s.add_ready_tasks(np.arange(3, dtype=np.uint32), np.zeros(3, dtype=np.uint32), priority_from_user(np.zeros(3)))
    # unsorted / duplicate worker ids are rejected before anything is launched; the ready set is untouched
    w = s._worker_structs(0.0)
    w2 = np.concatenate([w, w])
    free = np.ascontiguousarray(np.concatenate([s.free, s.free])); tot = np.ascontiguousarray(np.concatenate([s.total, s.total]))
    out = np.zeros(8, dtype=L.assignment_dtype); n = C.c_uint32(0)
    rc = s._lib.hqs_tick(s._ctx, 2, L.ptr(w2), L.ptr(free), L.ptr(tot), None, 8, L.ptr(out), C.byref(n), None)
    assert rc == -1 and n.value == 0
    assert s.run_scheduling().n_assigned() == 3
    # a request that uses a resource the context does not have is refused by hqs_classes_set
    s2 = GpuScheduler(1)
    cls = (L.hqs_class * 1)()
    cls[0].n_variants = 1
    cls[0].variants[0].amount[1] = 1 * FR
    cls[0].variants[0].weight = 10000
    assert s2._lib.hqs_classes_set(s2._ctx, 1, cls) == -1
    assert b"n_resources" in s2._lib.hqs_last_error(s2._ctx)
    s.close(); s2.close()


def test_min_utilization_vectors():
    """test_schedule_min_utilization1/2 (test_scheduler_sn.rs:1391-1445): the rule is enforced inside the tick kernel (a
    violating worker is taken out of the solve, which starts over)."""
    from hyperqueue_b200 import GpuScheduler, RequestVariant, priority_from_user

    def run(n_tasks, w_cpus, mu, running_cpus=0):
        s = GpuScheduler(1)
        c = s.get_or_create_resource_rq_id([RequestVariant.of({0: 3 * FR})])
        s.new_worker(1, [w_cpus * FR], min_utilization=mu, free=[(w_cpus - running_cpus) * FR])
        s.add_ready_tasks(np.arange(n_tasks, dtype=np.uint32), np.full(n_tasks, c, dtype=np.uint32), priority_from_user(np.zeros(n_tasks)))
        m = s.run_scheduling()
        again = s.run_scheduling().n_assigned() if m.n_assigned() == 0 else None
        free = s.free.copy()
        s.close()
        return m.n_assigned(), again, free

    assert run(2, 9, 1.0)[0] == 0
    assert run(3, 9, 1.0)[0] == 3
    assert run(2, 9, 1.0, running_cpus=3)[0] == 2
    for n, mu, exp in [(2, 0.5, 2), (2, 0.51, 0), (3, 0.51, 3), (3, 0.75, 3), (3, 0.76, 0)]:
        got, again, free = run(n, 12, mu)
        assert got == exp, (n, mu, got)
        if exp == 0:
            assert again == 0 and int(free[0, 0]) == 12 * FR      # dropped tasks are ready again; nothing leaked


def test_min_utilization_moves_work_to_other_workers():
    """A worker that cannot reach its minimum utilisation gets nothing — and its tasks go to the workers that can take
    them in the SAME tick (the reference's MILP does this with one boolean per worker, solver.rs:479-518).  Checked
    against the specification bit for bit, on a single-variant and on a three-variant pool."""
    from hyperqueue_b200 import GpuScheduler, RequestVariant, priority_from_user
    # w0 wants to be full (mu = 1.0, 4 cpus), w1 takes anything: one 1-cpu task must land on w1, not starve
    s = GpuScheduler(1)
    c = s.get_or_create_resource_rq_id([RequestVariant.of({0: 1 * FR})])
    s.new_worker(1, [4 * FR], min_utilization=1.0)
    s.new_worker(2, [4 * FR])
    s.add_ready_tasks(np.arange(1, dtype=np.uint32), np.full(1, c, dtype=np.uint32), priority_from_user(np.zeros(1)))
    m = s.run_scheduling()
    assert m.n_assigned() == 1 and m.per_worker() == {2: [(0, 0)]}
    assert int(s.free[0, 0]) == 4 * FR and int(s.free[1, 0]) == 3 * FR
    s.close()
    for seed, v3 in [(31, False), (32, True)]:
        wl = P.make_independent(3000, 12, 6, seed=seed, variants3=v3)
        mu = np.zeros(12, dtype=np.float32)
        mu[[0, 3, 7]] = [1.0, 0.97, 0.9]
        sch = P.gpu_scheduler(wl)
        sch.min_utilization = mu.copy()
        fb = sch.free.copy()
        m = sch.run_scheduling()
        exp, exp_free = G.model_tick(wl, np.ones(wl.n_tasks, dtype=bool), fb, min_utilization=mu)
        assert P.judge_tick(wl, fb, m.assignments).ok
        assert np.array_equal(m.assignments, exp) and np.array_equal(m.free_after, exp_free)
        # the rule itself: every worker with a minimum got either nothing or at least its minimum
        new_cpus = (fb[:, 0].astype(np.float64) - m.free_after[:, 0].astype(np.float64)) / 1e4
        min_cpus = wl.worker_total[:, 0] / 1e4 * (mu.astype(np.float64) - 1.0) + fb[:, 0] / 1e4
        assert ((new_cpus == 0) | (new_cpus >= min_cpus - 1e-9) | (mu <= 0.001)).all()
        sch.close()


def test_too_small_out_cap_fails_before_anything_is_consumed():
    """ABI contract: after a failed hqs_tick the host schedules nothing — so the device must not have consumed anything
    either.  The solver knows the number of assignments before the emit step and skips it."""
    from hyperqueue_b200 import HqsError
    wl = P.make_independent(5000, 8, 4, seed=9, free_scale=64)
    s = P.gpu_scheduler(wl)
    with pytest.raises(HqsError) as ei:
        s.run_scheduling(out_cap=100)
    assert ei.value.code == -5
    m = s.run_scheduling()                                # the whole ready set is still there
    exp, _ = G.model_tick(wl, np.ones(wl.n_tasks, dtype=bool), wl.worker_free)
    assert np.array_equal(m.assignments, exp) and m.n_assigned() > 100
    s.close()


def test_priority_levels_of_departed_tasks_are_pruned():
    """tako priorities carry a per-job component, so a long-running server sees ever new priority values.  Levels that no
    task of the table carries any more are dropped before the level set would have to be coarsened: after 6 waves of
    1500 distinct priorities each (9000 values, far beyond HQS_MAX_GROUPS / 2 classes = 4096 levels) the ticks are still
    exact (priority order is kept), because at most one wave is alive at a time."""
    from hyperqueue_b200 import GpuScheduler, RequestVariant, priority_from_user
    s = GpuScheduler(1)
    c1 = s.get_or_create_resource_rq_id([RequestVariant.of({0: 1 * FR})])
    c2 = s.get_or_create_resource_rq_id([RequestVariant.of({0: 2 * FR})])
    s.new_worker(1, [64 * FR])
    n = 1500
    for wave in range(6):
        h = np.arange(n, dtype=np.uint32)
        up = (wave * n + np.arange(n)).astype(np.int64)                 # 1500 fresh priority values per wave
        cls = np.where(np.arange(n) % 2 == 0, c1, c2).astype(np.uint32)
        s.add_ready_tasks(h, cls, priority_from_user(up))
        st = s.stats()
        assert st["coarsened"] == 0 and st["n_levels"] <= 2 * n + 64, (wave, st)
        m = s.run_scheduling()
        a = m.assignments
        # 64 cpus: the highest priorities first, strictly by priority
        assert a.shape[0] > 0 and (np.diff(up[a["task"]]) < 0).all()
        assert up[a["task"]].min() >= n * wave + n - 64
        s.tasks_finished(a["task"])
        s.remove_ready_tasks(h)                                         # the wave leaves (finished or cancelled)
    s.close()


def test_1024_worker_pool_tick_cfg5_shape():
    """BASELINE configs[4] pool: 1024 workers (32 worker tiles).  Small task count against the specification bit for bit,
    then the per-GPU share of cfg5 (1.25 M tasks, capacity >= demand) through the judge and the exact replay."""
    wl = P.make_independent(30000, 1024, 16, seed=11)
    _check_exact(wl)
    wl = P.make_independent(1_250_000, 1024, 16, seed=12, free_scale=1024)
    s = P.gpu_scheduler(wl)
    fb = s.free.copy()
    m = s.run_scheduling()
    a = m.assignments
    assert a.shape[0] == wl.n_tasks and np.array_equal(np.sort(a["task"]), np.arange(wl.n_tasks, dtype=np.uint32))
    assert P.judge_tick(wl, fb, a).ok
    amounts, allm, _, _ = wl.class_tables()
    from oracle import judge as J
    assert np.array_equal(J.replay_free_after(amounts, allm, fb, wl.worker_total, wl.task_class, a["task"], a["worker"], a["variant"]), m.free_after)
    assert (np.diff(wl.task_user_priority[a["task"]]) <= 0).all()
    s.close()


def test_new_worker_query_is_a_dry_run():
    """Shape of test_query.rs: fake workers, partial descriptors with MAX, nothing consumed."""
    wl = P.make_independent(3000, 4, 4, seed=12)
    s = P.gpu_scheduler(wl)
    fake = np.array([[128 * FR, 8 * FR, 512 * FR, 2048 * FR],            # a full node
                     [1 * FR, 0, 1 * FR, 0],                              # too small for anything
                     [64 * FR, P.J.AMOUNT_MAX, P.J.AMOUNT_MAX, P.J.AMOUNT_MAX]], dtype=np.uint64)   # partial descriptor
    needed, counts, total = s.new_worker_query(fake)
    assert needed.tolist() == [True, False, True] and total == int(counts.sum()) and counts[0] > 0
    again = s.new_worker_query(fake)
    assert np.array_equal(again[1], counts)                              # a query consumes nothing
    real = s.run_scheduling()
    assert real.n_assigned() > 0                                          # and the real tick still sees every task
    s.close()


def test_narrow_amounts_with_remainders_and_all_policy():
    # requests are multiples of 4 units (gcd 4 * FR), worker amounts are not: the scaled solver carries the
    # remainders; an `All` request needs free == total exactly, remainder included
    rng = np.random.default_rng(11)
    classes = [[{"amounts": {0: 4 * FR, 1: 8 * FR}}], [{"amounts": {0: 8 * FR}, "all": (2,)}],
               [{"amounts": {1: 4 * FR, 2: 12 * FR}}], [{"amounts": {0: 12 * FR, 2: 4 * FR}}, {"amounts": {1: 16 * FR}}]]
    w = 48
    total = rng.integers(20, 90, size=(w, 3)).astype(np.uint64) * np.uint64(FR) + rng.integers(0, FR, size=(w, 3)).astype(np.uint64)
    free = total.copy()
    free[::3, 2] -= np.uint64(1)            # a touched resource: `All` on it must not fit there
    free[1::3, 0] -= np.uint64(4 * FR)
    wl = P.Workload(3, classes, total, free, rng.integers(0, 4, 3000).astype(np.uint32), rng.integers(0, 3, 3000).astype(np.int32))
    m = _check_exact(wl, expect_narrow=True)
    assert m.n_assigned() > 50


def test_amounts_beyond_31_bits_use_the_wide_solver():
    # memory in bytes with odd request sizes: gcd 1 and totals ~ 2^50 => not representable in the narrow form
    rng = np.random.default_rng(12)
    gib = 1 << 30
    classes = [[{"amounts": {0: 1 * FR, 1: (3 * gib + 1) * FR}}], [{"amounts": {0: 2 * FR, 1: (5 * gib + 7) * FR}}],
               [{"amounts": {1: 11 * gib * FR}}]]
    w = 20
    total = np.stack([np.full(w, 64 * FR, dtype=np.uint64), rng.integers(200, 900, size=w).astype(np.uint64) * np.uint64(gib * FR)], axis=1)
    wl = P.Workload(2, classes, total, total.copy(), rng.integers(0, 3, 5000).astype(np.uint32), rng.integers(0, 4, 5000).astype(np.int32))
    m = _check_exact(wl, expect_narrow=False)
    assert m.n_assigned() > 100


def test_large_amounts_with_a_common_factor_stay_narrow():
    # the same memory sizes in whole GiB: the per-resource gcd brings them back under 2^31
    rng = np.random.default_rng(13)
    gib = 1 << 30
    classes = [[{"amounts": {0: 1 * FR, 1: 3 * gib * FR}}], [{"amounts": {0: 2 * FR, 1: 5 * gib * FR}}], [{"amounts": {1: 11 * gib * FR}}]]
    w = 20
    total = np.stack([np.full(w, 64 * FR, dtype=np.uint64), rng.integers(200, 900, size=w).astype(np.uint64) * np.uint64(gib * FR) + np.uint64(12345)], axis=1)
    wl = P.Workload(2, classes, total, total.copy(), rng.integers(0, 3, 5000).astype(np.uint32), rng.integers(0, 4, 5000).astype(np.int32))
    m = _check_exact(wl, expect_narrow=True)
    assert m.n_assigned() > 100


def test_cpp_shim_selftest():
    """tako_b200::GpuCore (C++ host side, include/tako_shim.hpp) through scenarios restated from test_scheduler_sn.rs
    and a zero-duration drain with a host replay of every placement."""
    from hyperqueue_b200 import _lib
    assert _lib.load_shim().hqshim_selftest(0, 1) == 0


def _fuzz_workload(seed):
    """Small random tick mixing everything the predicate knows: 1-6 resources, 1-4 variants, `All` entries, blocked
    masks, time limits, partly used workers, amounts with and without a common factor."""
    rng = np.random.default_rng(1000 + seed)
    r = int(rng.integers(1, 7)); w = int(rng.integers(1, 41)); q = int(rng.integers(1, 9)); n = int(rng.integers(1, 1500))
    unit = int(rng.choice([1, 2500, FR, 4 * FR]))                      # request granularity
    classes, seen = [], set()
    while len(classes) < q:
        vs = []
        for _ in range(int(rng.integers(1, 5))):
            k = int(rng.integers(1, min(r, 3) + 1))
            rs = [int(x) for x in rng.choice(r, size=k, replace=False)]
            d = {"amounts": {x: int(rng.integers(1, 12)) * unit for x in rs}}
            if r > 1 and rng.random() < 0.15:
                allr = int(rng.choice([x for x in range(r) if x not in rs] or [rs[0]]))
                if allr not in rs:
                    d["all"] = (allr,)
            if rng.random() < 0.2:
                d["min_time_s"] = float(rng.choice([1.0, 30.0, 120.0]))
            vs.append(d)
        key = repr([(sorted(d["amounts"].items()), d.get("all"), d.get("min_time_s")) for d in vs])
        if key not in seen:
            seen.add(key); classes.append(vs)
    total = rng.integers(4, 64, size=(w, r)).astype(np.uint64) * np.uint64(unit) + (
        rng.integers(0, unit, size=(w, r)).astype(np.uint64) if rng.random() < 0.5 else np.uint64(0))
    free = total.copy()
    used = rng.random((w, r)) < 0.3
    free[used] -= np.minimum(free[used], rng.integers(0, 20, size=int(used.sum())).astype(np.uint64) * np.uint64(unit))
    blocked = None
    if rng.random() < 0.4:
        blocked = np.zeros((w, q, P.MAXV), dtype=bool)
        blocked[:, :, :4] = rng.random((w, q, 4)) < 0.2
    rem = None
    if rng.random() < 0.4:
        rem = np.where(rng.random(w) < 0.5, np.inf, rng.choice([0.5, 10.0, 60.0, 600.0], size=w))
    return P.Workload(r, classes, total, free, rng.integers(0, q, n).astype(np.uint32), rng.integers(0, 5, n).astype(np.int32),
                      blocked=blocked, worker_remaining_s=rem)


@pytest.mark.parametrize("seed", range(40))
def test_random_ticks_match_specification(seed):
    _check_exact(_fuzz_workload(seed))
