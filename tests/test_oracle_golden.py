"""Pins the oracle against the reference's own known-answer vectors (SURVEY.md Appendix B).

Every test below is a transcription of a test in
hyperqueue/crates/tako/src/internal/tests/test_scheduler_sn.rs (line ranges in each docstring),
scheduler/gap.rs:175-246 or scheduler/batches.rs:223-250.  CPU only.
"""
import pytest

from oracle.batches import PriorityCut, create_task_batches, prune_progressive
from oracle.model import priority_from_user
from oracle_env import TaskBuilder as TB, TestCase, TestEnv, WorkerBuilder as WB


# ---------------------------------------------------------------------------------------------
# batching
# ---------------------------------------------------------------------------------------------
def test_prune_progressive():
    """batches.rs:223-250."""
    assert prune_progressive(list(range(40)), 4, 100) == list(range(40))
    assert prune_progressive(list(range(1000)), 4, 32) == [
        0, 1, 2, 3, 4, 5, 9, 16, 26, 38, 53, 71, 91, 115, 140, 169, 201, 235, 272, 311,
        353, 398, 446, 497, 550, 606, 665, 726, 790, 857, 927, 999]
    assert prune_progressive(list(range(40)), 4, 32) == [
        0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22,
        23, 24, 25, 27, 29, 32, 34, 36, 39]


def test_task_grouping_basic():
    """test_scheduler_sn.rs:13-73."""
    rt = TestEnv()
    rt.new_workers_cpus([5, 5, 5])
    assert create_task_batches(rt.core, 0.0) == []
    t1 = rt.new_task(TB().user_priority(123))
    a = create_task_batches(rt.core, 0.0)
    assert len(a) == 1 and a[0].resource_rq_id == rt.task(t1).rq_id
    assert a[0].cuts == [] and a[0].size == 1 and not a[0].limit_reached
    for p in (20, 5, 123, 20):
        rt.new_task(TB().user_priority(p))
    a = create_task_batches(rt.core, 0.0)
    assert len(a) == 1 and a[0].cuts == [] and a[0].size == 5 and not a[0].limit_reached
    t6 = rt.new_task(TB().cpus(2).user_priority(123))
    t7 = rt.new_task(TB().cpus(123).user_priority(123))
    rt.new_task(TB().cpus(2).user_priority(123))
    rt.new_task(TB().cpus(2).user_priority(123))
    a = create_task_batches(rt.core, 0.0)
    assert len(a) == 2
    assert a[0].resource_rq_id == rt.task(t1).rq_id and a[0].size == 5 and not a[0].limit_reached
    assert a[0].cuts == [PriorityCut(2, [(rt.task(t6).rq_id, 3), (rt.task(t7).rq_id, None)])]
    assert a[1].resource_rq_id == rt.task(t6).rq_id and a[1].size == 3 and not a[1].limit_reached
    assert a[1].cuts == []


def test_task_grouping_blocker():
    """test_scheduler_sn.rs:75-87."""
    rt = TestEnv()
    rt.new_workers_cpus([5])
    rt.new_task(TB().user_priority(2))
    rt.new_task(TB().cpus(2).user_priority(1))
    a = create_task_batches(rt.core, 0.0)
    assert len(a) == 2 and a[0].is_blocker and not a[1].is_blocker


def test_task_group_saturation():
    """test_scheduler_sn.rs:89-135."""
    rt = TestEnv()
    rt.new_workers_cpus([5, 5, 5])
    for p in (2, 2, 4, 4, 6, 6):
        rt.new_task(TB().cpus(4).user_priority(p))
    a = create_task_batches(rt.core, 0.0)
    assert len(a) == 1 and a[0].size == 3 and a[0].limit_reached and a[0].cuts == []
    rt.new_task(TB().cpus(1).user_priority(5))
    rt.new_task(TB().cpus(1).user_priority(0))
    a = create_task_batches(rt.core, 0.0)
    assert len(a) == 2
    assert a[0].size == 3 and a[0].limit_reached
    assert a[0].cuts == [PriorityCut(2, [(1, 1)])]
    assert a[1].size == 2 and not a[1].limit_reached
    assert a[1].cuts == [PriorityCut(0, [(0, 2)]), PriorityCut(1, [(0, None)])]


def test_task_batching2():
    """test_scheduler_sn.rs:137-154."""
    rt = TestEnv()
    ws = rt.new_workers_cpus([3, 3, 3])
    rt.new_task_running(TB().cpus(1), ws[0])
    rt.new_task_running(TB().cpus(2), ws[1])
    rt.new_task_running(TB().cpus(3), ws[2])
    rt.new_task(TB().cpus(2)); rt.new_task(TB().cpus(1)); rt.new_task(TB().cpus(3))
    a = create_task_batches(rt.core, 0.0)
    assert len(a) == 3 and all(b.cuts == [] for b in a)


# ---------------------------------------------------------------------------------------------
# gap cache
# ---------------------------------------------------------------------------------------------
def test_compute_gap():
    """gap.rs:175-246 (13 exact values)."""
    rt = TestEnv()
    rt.new_named_resource("foo"); rt.new_named_resource("bar")

    def gap(hi, lo, w):
        core = rt.core
        return core.scheduler_state.gap_cache.get_gap(rt.task(hi).rq_id, rt.task(lo).rq_id,
                                                      core.workers[w].resources, [], core.rq_map)
    w = rt.new_worker(WB(4))
    t1 = rt.new_task_cpus(2); t2 = rt.new_task_cpus(1)
    assert gap(t1, t2, w) == 0
    t1 = rt.new_task_cpus(3)
    assert gap(t1, t2, w) == 1
    t2 = rt.new_task_cpus(2)
    assert gap(t1, t2, w) == 0
    w = rt.new_worker(WB(12).res_sum("foo", 2).res_sum("bar", 1))
    t1 = rt.new_task_cpus(4); t2 = rt.new_task_cpus(2)
    assert gap(t1, t2, w) == 0
    t1 = rt.new_task_cpus(5); t2 = rt.new_task_cpus(1)
    assert gap(t1, t2, w) == 2
    t1 = rt.new_task(TB().cpus(5).add_resource(1, 2))
    assert gap(t1, t2, w) == 7
    t2 = rt.new_task(TB().cpus(1).add_resource(1, 1))
    assert gap(t1, t2, w) == 0
    t1 = rt.new_task(TB().cpus(5).add_resource(1, 2))
    t2 = rt.new_task(TB().cpus(1).add_resource(2, 1))
    assert gap(t1, t2, w) == 1
    t1 = rt.new_task(TB().cpus(8).next_variant().cpus(2).add_resource(1, 2))
    t2 = rt.new_task(TB().cpus(1))
    assert gap(t1, t2, w) == 2
    t1 = rt.new_task(TB().cpus(8).next_variant().cpus(2).add_resource(1, 1))
    assert gap(t1, t2, w) == 0
    t1 = rt.new_task(TB().cpus(8).next_variant().cpus(2).add_resource(1, 2))
    t2 = rt.new_task(TB().cpus(1).add_resource(2, 1))
    assert gap(t1, t2, w) == 1
    w = rt.new_worker(WB(6).res_sum("foo", 2).res_sum("bar", 2))
    t1 = rt.new_task(TB().cpus(2).add_resource(1, 1).next_variant().cpus(2).add_resource(2, 1))
    t2 = rt.new_task_cpus(1)
    assert gap(t1, t2, w) == 0
    w = rt.new_worker(WB(58))
    t1 = rt.new_task(TB().cpus(13).next_variant().cpus(7))
    t2 = rt.new_task_cpus(1)
    assert gap(t1, t2, w) == 2


# ---------------------------------------------------------------------------------------------
# packing without priorities
# ---------------------------------------------------------------------------------------------
def test_schedule_no_priorities():
    """test_scheduler_sn.rs:156-224 (11 cases)."""
    w3, w4 = WB(3), WB(4)
    c = TestCase(); c.w(w4); c.w(w3); c.check()

    c = TestCase(); ts = c.c_tasks([3]); c.w(w3).expect_tasks([ts[0]]); c.check()

    c = TestCase(); ts = c.c_tasks([2]); c.w(w4).expect_tasks([ts[0]]); c.w(w4); c.check()

    c = TestCase(); ts = c.c_tasks([2, 2]); c.w(w4).expect_tasks(ts); c.w(w4); c.check()

    c = TestCase(); ts = c.c_tasks([2, 2, 2])
    c.w(w4).expect_tasks([ts[0], ts[2]]); c.w(w4).expect_tasks([ts[1]]); c.check()

    c = TestCase(); ts = c.c_tasks([2, 2, 2, 2])
    c.w(w4).expect_tasks([ts[0], ts[2]]); c.w(w4).expect_tasks([ts[1], ts[3]]); c.check()

    c = TestCase(); ts = c.c_tasks([2, 2, 2, 2, 2])
    c.w(w4).expect_tasks([ts[0], ts[2]]); c.w(w4).expect_tasks([ts[1], ts[3]]); c.check()

    c = TestCase(); ts = c.c_tasks([2, 3])
    c.w(w4).expect_tasks([ts[1]]); c.w(w4).expect_tasks([ts[0]]); c.check()

    c = TestCase(); ts = c.c_tasks([2, 3])
    c.w(w3).expect_tasks([ts[1]]); c.w(w4).expect_tasks([ts[0]]); c.check()

    c = TestCase(); ts = c.c_tasks([5, 5, 1, 1, 1, 1, 1])
    c.w(w4).expect_tasks([ts[2], ts[4], ts[5], ts[6]]); c.w(w4).expect_tasks([ts[3]]); c.check()

    c = TestCase(); ts = c.c_tasks([3, 4, 2])
    c.w(w4).expect_tasks([ts[1]]); c.w(w4).expect_tasks([ts[0]]); c.check()


# ---------------------------------------------------------------------------------------------
# priorities and cuts
# ---------------------------------------------------------------------------------------------
def test_schedule_priorities():
    """test_scheduler_sn.rs:226-307 (13 cases)."""
    w4, w10 = WB(4), WB(10)
    c = TestCase(); ts = c.pc_tasks([(1, 2), (1, 2)])
    c.w(w4).expect_tasks([ts[0], ts[1]]); c.w(w4); c.check()

    c = TestCase(); ts = c.pc_tasks([(1, 2), (2, 2)])
    c.w(w4).expect_tasks([ts[1], ts[0]]); c.w(w4); c.check()

    c = TestCase(); ts = c.pc_tasks([(0, 4), (0, 4), (1, 2), (2, 3)])
    c.w(w4).expect_tasks([ts[3]]); c.w(w4).expect_tasks([ts[2]]); c.check()

    c = TestCase(); ts = c.pc_tasks([(0, 4), (0, 4), (1, 2), (1, 3)])
    c.w(w4).expect_tasks([ts[3]]); c.w(w4).expect_tasks([ts[2]]); c.check()

    c = TestCase(); ts = c.pc_tasks([(1, 4), (1, 4), (1, 2), (1, 3)])
    c.w(w4).eq_class(0).expect_tasks([ts[0]]); c.w(w4).eq_class(0).expect_tasks([ts[1]]); c.check()

    c = TestCase(); ts = c.pc_tasks([(0, 2), (4, 2), (3, 1), (2, 3)])
    c.w(w4).eq_class(0).expect_tasks([ts[1], ts[0]]); c.w(w4).eq_class(0).expect_tasks([ts[2], ts[3]])
    c.check()

    c = TestCase(); ts = c.pc_tasks([(1, 5), (0, 4)])
    c.w(w4).expect_tasks([ts[1]]); c.w(w4); c.check()

    c = TestCase(); ts = c.pc_tasks([(0, 2), (4, 2), (2, 4)])
    c.w(w4).eq_class(0).expect_tasks([ts[1], ts[0]]); c.w(w4).eq_class(0).expect_tasks([ts[2]]); c.check()

    c = TestCase(); ts = c.pc_tasks([(9, 2), (7, 1), (6, 2)])
    c.w(w4).expect_tasks(ts[:2]); c.check()

    c = TestCase(); ts = c.pc_tasks([(9, 2), (7, 1), (6, 2), (5, 1)])
    c.w(w4).expect_tasks(ts[:2]); c.check()

    c = TestCase()
    ts = c.pc_tasks([(9, 2), (8, 1), (7, 2), (6, 1), (5, 2), (4, 1), (3, 2), (2, 1)])
    c.w(w10).expect_tasks(ts[:6]); c.check()

    c = TestCase(); ts = c.pc_tasks([(1, 3), (1, 3), (1, 3), (0, 1)])
    c.w(w4).expect_tasks([ts[0], ts[3]]); c.check()


def test_schedule_no_irrelevant_blocking():
    """test_scheduler_sn.rs:309-330."""
    w3, w5 = WB(3), WB(5)
    c = TestCase(); ts = c.pc_tasks([(10, 5), (0, 1)]); c.w(w3).expect_tasks([ts[1]]); c.check()
    c = TestCase(); ts = c.pc_tasks([(10, 5), (9, 5), (0, 1)])
    c.w(w3).expect_tasks([ts[2]]); c.w(w5).expect_tasks([ts[0]]); c.check()
    c = TestCase(); ts = c.pc_tasks([(10, 3), (9, 2), (8, 5), (0, 1)])
    c.w(w5).expect_tasks([ts[0], ts[1]]); c.w(w3).expect_tasks([ts[3]]); c.check()


def test_schedule_some_tasks_running():
    """test_scheduler_sn.rs:332-366."""
    w3 = WB(3)
    c = TestCase(); c.pc_tasks([(1, 3)]); c.w(w3).running_c(1).expect_tasks([]); c.check()
    c = TestCase(); ts = c.pc_tasks([(1, 2)]); c.w(w3).running_c(1).expect_tasks([ts[0]]); c.check()
    c = TestCase(); c.pc_tasks([(1, 3), (0, 1)]); c.w(w3).running_c(1).expect_tasks([]); c.check()
    c = TestCase(); ts = c.c_tasks([2, 1, 3])
    c.w(w3).running_c(1).expect_tasks([ts[0]])
    c.w(w3).running_c(2).expect_tasks([ts[1]])
    c.w(w3).running_c(2).running_c(1).expect_tasks([])
    c.check()


@pytest.mark.parametrize("w_cpus,count_a,count_b", [
    (1, 2, 0), (2, 3, 1), (3, 4, 2), (4, 6, 2), (5, 7, 3),
    (6, 8, 4), (7, 10, 4), (8, 12, 4), (9, 12, 5), (10, 12, 5)])
def test_priority_switching(w_cpus, count_a, count_b):
    """test_scheduler_sn.rs:368-405."""
    rt = TestEnv()
    rt.new_named_resource("foo")
    ta, tb = TB().cpus(1), TB().cpus(1).add_resource(1, 1)
    w = WB(w_cpus).res_sum("foo", 10_000)
    rt.new_worker(w); rt.new_worker(w)
    rt.new_tasks(3, ta.user_priority(10)); rt.new_tasks(2, tb.user_priority(9))
    rt.new_tasks(1, ta.user_priority(8)); rt.new_tasks(3, ta.user_priority(7))
    rt.new_tasks(1, tb.user_priority(6)); rt.new_tasks(1, tb.user_priority(5))
    rt.new_tasks(5, ta.user_priority(4)); rt.new_tasks(1, tb.user_priority(3))
    rt.schedule()
    counts = rt.assigned_counts()
    assert (counts[0], counts[1]) == (count_a, count_b)


# ---------------------------------------------------------------------------------------------
# gap filling
# ---------------------------------------------------------------------------------------------
def test_schedule_gap_filling():
    """test_scheduler_sn.rs:410-449."""
    w6, w12, w8 = WB(6), WB(12), WB(8)
    c = TestCase(); ts = c.pc_tasks([(1, 8), (1, 8), (0, 4)])
    c.w(w12).expect_tasks([ts[0], ts[2]]); c.check()
    c = TestCase(); ts = c.pc_tasks([(1, 3), (1, 3), (1, 3), (0, 2)])
    c.w(w6).expect_tasks([ts[0], ts[1]]); c.check()
    c = TestCase(); ts = c.pc_tasks([(1, 3), (1, 3), (1, 3), (0, 1), (0, 1)])
    c.w(w8).expect_tasks([ts[0], ts[1], ts[3], ts[4]]); c.check()
    c = TestCase(); ts = c.pc_tasks([(1, 3), (1, 3), (1, 3), (2, 1), (0, 1)])
    c.w(w8).expect_tasks([ts[3], ts[0], ts[1], ts[4]]); c.check()
    c = TestCase()
    ts = c.pc_tasks([(1, 3), (1, 3), (1, 3), (2, 1), (0, 1), (0, 1), (0, 1), (0, 1)])
    c.w(w8).expect_tasks([ts[3], ts[0], ts[1], ts[4]]); c.check()


@pytest.mark.parametrize("extra", [True, False])
def test_schedule_gap_filling2(extra):
    """test_scheduler_sn.rs:461-494."""
    rt = TestEnv()
    rt.new_named_resource("foo")
    rt.new_worker(WB(8))
    rt.new_workers(3, WB(4).res_sum("foo", 1))
    ta, tb, tc = TB().cpus(1), TB().cpus(3), TB().cpus(4).add_resource(1, 1)
    rt.new_tasks(7, ta.user_priority(1)); rt.new_tasks(3, tb.user_priority(2)); rt.new_tasks(3, tc.user_priority(2))
    if extra:
        rt.new_tasks(2, tb.user_priority(-1)); rt.new_tasks(3, tc.user_priority(-2))
        rt.new_tasks(1, ta.user_priority(-3)); rt.new_tasks(2, tb.user_priority(-4))
        rt.new_tasks(3, tc.user_priority(-5)); rt.new_tasks(1, ta.user_priority(-6))
    rt.schedule()
    assert rt.assigned_counts()[:3] == [2, 2, 3]
    rt.schedule()


def test_schedule_gap_filling3():
    """test_scheduler_sn.rs:496-526."""
    rt = TestEnv()
    rt.new_named_resource("foo")
    ws = rt.new_workers(2, WB(34))
    ta, tb = TB().cpus(3), TB().cpus(9)
    rt.new_tasks(5, ta.user_priority(10))
    ts2 = rt.new_tasks(6, tb.user_priority(10))
    ts3 = rt.new_tasks(5, ta.user_priority(9))
    rt.schedule()
    for w in ws:
        cpus = t3count = 0
        for t in rt.worker(w).assigned_tasks:
            if t in ts2:
                cpus += 9
            else:
                cpus += 3
                t3count += t in ts3
        assert cpus == 33 and t3count <= 2


def test_schedule_gap_filling4():
    """test_scheduler_sn.rs:528-565."""
    rt = TestEnv()
    for n in ("foo", "bar", "goo"):
        rt.new_named_resource(n)
    rt.new_workers(2, WB(3).res_sum("foo", 10).res_sum("goo", 10))
    rt.new_worker(WB(3).res_sum("foo", 10).res_sum("bar", 10))
    rt.new_tasks(5, TB().cpus(2).add_resource(3, 1).user_priority(10))
    rt.new_tasks(2, TB().cpus(1).add_resource(1, 1).user_priority(9))
    rt.new_tasks(10, TB().cpus(3).add_resource(1, 1).add_resource(2, 1).user_priority(8))
    rt.schedule()
    assert rt.assigned_counts() == [2, 2, 1]


# ---------------------------------------------------------------------------------------------
# reservations
# ---------------------------------------------------------------------------------------------
def test_schedule_reservation_simple():
    """test_scheduler_sn.rs:567-580."""
    c = TestCase(); ts = c.pc_tasks([(3, 3), (2, 2)])
    c.w(WB(3)).eq_class(0).running_c(1).expect_tasks([])
    c.w(WB(3)).eq_class(0).running_c(1).expect_tasks([ts[1]])
    c.check()


def test_schedule_reservation2():
    """test_scheduler_sn.rs:582-592."""
    c = TestCase(); ts = c.pc_tasks([(3, 3), (2, 1), (2, 1)])
    c.w(WB(3)).eq_class(0).running_c(1)
    c.w(WB(3)).eq_class(0).running_c(1).expect_tasks([ts[1], ts[2]])
    c.check()


def test_schedule_reservation3():
    """test_scheduler_sn.rs:594-603."""
    c = TestCase(); ts = c.pc_tasks([(3, 3), (2, 1), (2, 1)])
    c.w(WB(3)).running_c(2).expect_tasks([ts[1]])
    c.w(WB(3)).running_c(1)
    c.check()


def test_schedule_reservation4():
    """test_scheduler_sn.rs:605-619."""
    c = TestCase(); ts = c.pc_tasks([(4, 3), (3, 3), (3, 3), (2, 1), (2, 1)])
    c.w(WB(4)).running_c(1).expect_tasks([ts[0]])
    c.w(WB(3)).running_c(2).expect_tasks([ts[3]])
    c.w(WB(3)).running_c(2)
    c.w(WB(3)).running_c(1)
    c.check()


def test_schedule_reservation5():
    """test_scheduler_sn.rs:621-633."""
    c = TestCase(); c.pc_tasks([(4, 3), (3, 3), (3, 3), (2, 1), (2, 1)])
    c.w(WB(3)).running_c(2).expect_request(1, TB())
    c.w(WB(3)).running_c(2)
    c.w(WB(3)).running_c(1)
    c.w(WB(4)).expect_request(1, TB().cpus(3)).expect_request(1, TB())
    c.check()


# ---------------------------------------------------------------------------------------------
# several resources
# ---------------------------------------------------------------------------------------------
def test_schedule_multiple_resources1():
    """test_scheduler_sn.rs:635-686."""
    w4_1, w4_2 = WB(4).res_range("gpus", 1, 1), WB(4).res_range("gpus", 1, 2)
    tb2_1, tb1_2, tb2 = TB().cpus(2).add_resource(1, 1), TB().cpus(1).add_resource(1, 2), TB().cpus(2)
    create = lambda: TestCase().resources(["gpus"])
    c = create(); t1 = c.t(tb2_1); t2 = c.t(tb2_1); c.w(w4_2).expect_tasks([t1, t2]); c.check()
    c = create(); t1 = c.t(tb2_1); c.t(tb2_1); c.w(w4_1).expect_tasks([t1]); c.check()
    c = create(); t1 = c.t(tb2); c.w(w4_2).expect_tasks([t1]); c.check()
    c = create(); t1 = c.t(tb1_2); c.w(w4_2).expect_tasks([t1]); c.check()
    c = create(); c.t(tb1_2); c.w(w4_1).expect_tasks([]); c.check()

    c = TestCase().resources(["gpus", "foo"])
    ta = TB().cpus(2).add_resource(1, 1)
    tb = TB().add_resource(1, 1).add_resource(2, 2)
    tc = TB().cpus(4)
    c.t(ta); c.ts(2, tb); c.ts(2, tc); c.t(tb)
    c.w(WB(6)).expect_request(1, tc)
    c.w(WB(3).res_sum("gpus", 2)).expect_request(1, ta)
    c.w(WB(5).res_sum("gpus", 20).res_sum("foo", 4)).expect_request(2, tb)
    c.check()


def test_schedule_multiple_resources2():
    """test_scheduler_sn.rs:688-721."""
    tb2_1, tb2 = TB().cpus(2).add_resource(1, 1), TB().cpus(2)

    def create():
        c = TestCase().resources(["gpus"]); c.ts(10, tb2); c.ts(10, tb2_1); return c
    c = create(); c.w(WB(6)).expect_request(3, tb2); c.check()
    c = create(); c.w(WB(6).res_sum("gpus", 10)).expect_request(3, tb2_1); c.check()
    c = create(); c.w(WB(6).res_sum("gpus", 2)).expect_request(2, tb2_1).expect_request(1, tb2); c.check()
    c = create()
    c.w(WB(6).res_sum("gpus", 2)).expect_request(2, tb2_1).expect_request(1, tb2)
    c.w(WB(6)).expect_request(3, tb2)
    c.check()


# ---------------------------------------------------------------------------------------------
# variants
# ---------------------------------------------------------------------------------------------
def test_schedule_variants1():
    """test_scheduler_sn.rs:723-754."""
    tb1 = TB().cpus(2).next_variant().cpus(5)
    c = TestCase(); c.ts(2, tb1); c.w(WB(11)).expect_request_v(2, tb1, 1); c.check()
    c = TestCase(); c.ts(3, tb1); c.w(WB(11)).expect_request_v(2, tb1, 1); c.check()
    c = TestCase(); c.ts(3, tb1); c.w(WB(14)).expect_request_v(2, tb1, 1).expect_request_v(1, tb1, 0); c.check()
    c = TestCase(); c.ts(10, tb1); c.w(WB(8)).expect_request_v(4, tb1, 0); c.check()
    c = TestCase(); c.ts(3, tb1); c.w(WB(8)).expect_request_v(1, tb1, 0).expect_request_v(1, tb1, 1); c.check()


def test_schedule_variants2():
    """test_scheduler_sn.rs:756-784."""
    tb1 = TB().cpus(6).next_variant().cpus(2).add_resource(1, 2)
    create = lambda: TestCase().resources(["gpus"])
    c = create(); c.ts(10, tb1); c.w(WB(12)).expect_request_v(2, tb1, 0); c.check()
    c = create(); c.ts(10, tb1)
    c.w(WB(12).res_sum("gpus", 4)).expect_request_v(1, tb1, 0).expect_request_v(2, tb1, 1); c.check()
    c = create(); c.ts(10, tb1); c.w(WB(12).res_sum("gpus", 20)).expect_request_v(6, tb1, 1); c.check()


def test_generic_resource_variants():
    """test_scheduler_sn.rs:1053-1108 (variants1-3)."""
    for (cpus0, w1c, w2c, res, exp1, exp2) in [(2, 4, 4, 2, 2, 2), (8, 4, 4, 2, 0, 2), (3, 2, 5, 1, 0, 2)]:
        rt = TestEnv(); rt.new_generic_resource(1)
        w1 = rt.new_worker(WB(w1c)); w2 = rt.new_worker(WB(w2c).res_range("Res0", 1, res))
        rt.new_tasks(4, TB().cpus(cpus0).next_variant().cpus(1).add_resource(1, 1))
        rt.schedule()
        assert (len(rt.worker_tasks(w1)), len(rt.worker_tasks(w2))) == (exp1, exp2)


def test_schedule_variant_gap1():
    """test_scheduler_sn.rs:1324-1351."""
    for running in (0, 1, 2):
        rt = TestEnv(); rt.new_named_resource("gpus")
        w = rt.new_worker(WB(14).res_sum("gpus", 4))
        for _ in range(running):
            rt.new_task_running(TB(), w)
        rt.new_tasks(10, TB().user_priority(10).cpus(8).next_variant().cpus(4).add_resource(1, 2))
        ts = rt.new_tasks(10, TB())
        rt.schedule()
        assert rt.n_assigned(ts) == 2 - running


# ---------------------------------------------------------------------------------------------
# scattering / compaction / prefill
# ---------------------------------------------------------------------------------------------
def _msg_len(mapping, w):
    up = mapping.workers.get(w)
    return 0 if up is None else len(up.prefills) + len(up.assigned)


def test_no_deps_scattering_1():
    """test_scheduler_sn.rs:793-815."""
    rt = TestEnv(); ws = rt.new_workers_cpus([5, 5, 5])
    rt.new_tasks(4, TB())
    m = rt.schedule()
    assert [_msg_len(m, w) for w in ws] == [4, 0, 0]


def test_no_deps_scattering_2():
    """test_scheduler_sn.rs:817-847."""
    rt = TestEnv(); rt.new_workers_cpus([5, 5, 5])

    def submit_and_check(expected):
        rt.new_task_default(); rt.schedule()
        assert sorted(len(w.assigned_tasks) for w in rt.core.workers.values()) == expected
    for i in range(1, 6):
        submit_and_check([0, 0, i])
    for i in range(1, 6):
        submit_and_check([0, i, 5])
    for i in range(1, 6):
        submit_and_check([i, 5, 5])
    submit_and_check([5, 5, 5]); submit_and_check([5, 5, 5])


def test_no_deps_distribute():
    """test_scheduler_sn.rs:849-871: 150 tasks, 3 x 10 cpus, reserve 10 / max 20 => 30 per message."""
    rt = TestEnv(); rt.set_scheduler_config(10, 20)
    ws = rt.new_workers_cpus([10, 10, 10])
    rt.new_tasks(150, TB())
    m = rt.schedule()
    assert [_msg_len(m, w) for w in ws] == [30, 30, 30]


def test_prefill_basic():
    """test_scheduler_sn.rs:1168-1200."""
    rt = TestEnv(); rt.set_scheduler_config(4, 32)
    ws = rt.new_workers(2, WB(8))
    tasks = rt.new_tasks(300, TB().cpus(4))
    m = rt.schedule()
    for w in ws:
        up = m.workers[w]
        assert len(up.prefills) == 32 and len(up.assigned) == 2       # prefills first in the message
        assert len(rt.worker(w).prefilled_tasks) == 32
    q = rt.core.task_queues.get(rt.task(tasks[0]).rq_id)
    assert list(q.iter_priority_sizes()) == [(priority_from_user(0), 296)]


def test_prefill_choose_waiting():
    """test_scheduler_sn.rs:1202-1223."""
    rt = TestEnv(); rt.set_scheduler_config(3, 6)
    w1 = rt.new_worker(WB(1)); rt.new_tasks(15, TB()); rt.schedule()
    pc = lambda w: len(rt.worker(w).prefilled_tasks)
    assert pc(w1) == 6
    w2 = rt.new_worker(WB(1)); rt.schedule()
    assert (pc(w1), pc(w2)) == (6, 4)
    w3 = rt.new_worker(WB(1)); rt.schedule()
    assert (pc(w1), pc(w2), pc(w3)) == (6, 4, 0)


def test_prefill_steal_first_half():
    """test_scheduler_sn.rs:1225-1270 (up to the retract message; on_retract_response is next-tier)."""
    rt = TestEnv(); rt.set_scheduler_config(3, 6)
    w1 = rt.new_worker(WB(1))
    tasks = rt.new_tasks(9, TB())
    rt.schedule()
    assert len(rt.worker(w1).prefilled_tasks) == 5
    w2 = rt.new_worker(WB(5))
    q = rt.core.task_queues.get(rt.task(tasks[0]).rq_id)
    assert list(q.iter_priority_sizes()) == [(priority_from_user(0), 8)]
    m = rt.core.schedule_mapping(0.0)
    assert len(m.workers[w1].retracts) == 2
    assert len(m.workers[w2].assigned) == 3
    assert sorted(rt.core.scheduler_state.redirects.values()) == [(w2, 0), (w2, 0)]
    assert len(rt.worker(w1).prefilled_tasks) == 3 and len(rt.worker(w2).prefilled_tasks) == 0
    assert len(rt.worker(w1).assigned_tasks) == 1 and len(rt.worker(w2).assigned_tasks) == 5


def test_generic_resource_balancing3():
    """test_scheduler_sn.rs:992-1051."""
    rt = TestEnv(); rt.set_scheduler_config(0, 100); rt.new_generic_resource(1)
    w1 = rt.new_worker(WB(2)); w2 = rt.new_worker(WB(2).res_range("Res0", 1, 1))
    ts1 = rt.new_tasks(80, TB()); ts2 = rt.new_tasks(20, TB().cpus(1).add_resource(1, 1))
    rq1, rq2 = rt.task(ts1[0]).rq_id, rt.task(ts2[0]).rq_id
    rt.schedule()
    a = rt.worker(w1)
    assert len(a.assigned_tasks) == 2 and all(rt.task(t).rq_id == rq1 for t in a.assigned_tasks)
    assert len(a.prefilled_tasks) == 38 and all(rt.task(t).rq_id == rq1 for t in a.prefilled_tasks)
    a = rt.worker(w2)
    assert len(a.assigned_tasks) == 2 and len(a.prefilled_tasks) == 57
    assert sum(rt.task(t).rq_id == rq1 for t in a.prefilled_tasks) == 38
    assert sum(rt.task(t).rq_id == rq2 for t in a.prefilled_tasks) == 19


# ---------------------------------------------------------------------------------------------
# time, generic resources, running tasks
# ---------------------------------------------------------------------------------------------
def test_resource_time_assign():
    """test_scheduler_sn.rs:873-885."""
    rt = TestEnv(); w1 = rt.new_worker(WB(10).time_limit_s(100))
    rt.new_task(TB().time_request(170)); t2 = rt.new_task_default(); t3 = rt.new_task(TB().time_request(99))
    rt.schedule()
    assert rt.worker_tasks(w1) == {t2, t3}


def test_resource_time_balance1():
    """test_scheduler_sn.rs:887-904."""
    rt = TestEnv()
    w1 = rt.new_worker(WB(1).time_limit_s(50)); w2 = rt.new_worker(WB(1).time_limit_s(200))
    w3 = rt.new_worker(WB(1).time_limit_s(100))
    t1 = rt.new_task(TB().time_request(170)); t2 = rt.new_task(TB()); t3 = rt.new_task(TB().time_request(99))
    rt.schedule()
    assert (rt.worker_tasks(w1), rt.worker_tasks(w2), rt.worker_tasks(w3)) == ({t2}, {t1}, {t3})


def _three_generic_workers(rt):
    rt.new_generic_resource(2)
    w1 = rt.new_worker(WB(10).res_range("Res0", 1, 10))
    w2 = rt.new_worker(WB(10))
    w3 = rt.new_worker(WB(10).res_range("Res0", 1, 10).res_sum("Res1", 1_000_000))
    return w1, w2, w3


def test_generic_resource_assign2():
    """test_scheduler_sn.rs:906-936."""
    rt = TestEnv(); w1, w2, w3 = _three_generic_workers(rt)
    ts1 = rt.new_tasks(50, TB().add_resource(1, 1)); rt.new_tasks(50, TB().add_resource(1, 2))
    rt.schedule()
    assert [len(rt.worker_tasks(w)) for w in (w1, w2, w3)] == [10, 0, 10]
    assert all(t in ts1 for t in rt.worker_tasks(w1))


def test_generic_resource_balance1():
    """test_scheduler_sn.rs:938-957."""
    rt = TestEnv(); w1, w2, w3 = _three_generic_workers(rt)
    rt.new_tasks(4, TB().cpus(1).add_resource(1, 5)); rt.schedule()
    assert [len(rt.worker_tasks(w)) for w in (w1, w2, w3)] == [2, 0, 2]


def test_generic_resource_balance2():
    """test_scheduler_sn.rs:959-990."""
    rt = TestEnv(); w1, w2, w3 = _three_generic_workers(rt)
    a, b = TB().cpus(1).add_resource(1, 5), TB().cpus(1).add_resource(1, 5).add_resource(2, 500_000)
    rt.new_task(a); rt.new_task(b); rt.new_task(a); rt.new_task(b)
    rt.schedule()
    assert [len(rt.worker_tasks(w)) for w in (w1, w2, w3)] == [2, 0, 2]


def test_scheduler_two_running_three_waiting():
    """test_scheduler_sn.rs:1110-1127."""
    rt = TestEnv(); rt.new_named_resource("foo")
    w = rt.new_worker(WB(8).res_range("foo", 1, 4))
    ts = rt.new_tasks(4, TB().cpus(1).add_resource(1, 2))
    rt.assign_and_start_task(ts[0], w); rt.assign_and_start_task(ts[1], w)
    t5 = rt.new_task(TB().cpus(2).user_priority(1))
    rt.schedule()
    assert rt.task(t5).is_assigned()
    assert rt.task(ts[0]).state == "running" and rt.task(ts[1]).state == "running"
    assert rt.task(ts[2]).state == "waiting" and rt.task(ts[3]).state == "waiting"


def test_schedule_running():
    """test_scheduler_sn.rs:1308-1322."""
    rt = TestEnv(); w = rt.new_worker(WB(14))
    for _ in range(8):
        rt.new_task_running(TB(), w)
    ts = rt.new_tasks(10, TB()); rt.schedule()
    assert len(rt.worker(w).assigned_tasks) == 14 and rt.n_assigned(ts) == 6


def test_many_cuts():
    """test_scheduler_sn.rs:1129-1146: 300 x 8 cpus, 3200 priority levels x 2 classes => ~800/800."""
    rt = TestEnv(); rt.new_workers(300, WB(8))
    ts1, ts2 = [], []
    for i in range(3200):
        ts1.append(rt.new_task(TB().cpus(1).user_priority(i)))
        ts2.append(rt.new_task(TB().cpus(2).user_priority(i)))
    rt.schedule()
    c1, c2 = rt.n_assigned(ts1), rt.n_assigned(ts2)
    assert abs(c1 - c2) < 10 and abs(c1 - 800) < 10 and abs(c2 - 800) < 10


# ---------------------------------------------------------------------------------------------
# weights, min-utilisation
# ---------------------------------------------------------------------------------------------
def test_schedule_resource_weights1():
    """test_scheduler_sn.rs:1353-1370."""
    rt = TestEnv(); t1 = rt.new_task(TB().cpus(3)); t2 = rt.new_task(TB().cpus(2).weight(1.49))
    rt.new_worker(WB(4)); rt.schedule()
    assert rt.task(t1).is_assigned() and rt.task(t2).state == "waiting"
    rt = TestEnv(); t1 = rt.new_task(TB().cpus(3).weight(1.0)); t2 = rt.new_task(TB().cpus(2).weight(1.51))
    rt.new_worker(WB(4)); rt.schedule()
    assert rt.task(t1).state == "waiting" and rt.task(t2).is_assigned()


def test_schedule_resource_weights2():
    """test_scheduler_sn.rs:1372-1389."""
    rt = TestEnv(); ts = rt.new_tasks(5, TB().cpus(3).weight(1.1)); t1 = rt.new_task(TB().cpus_all())
    rt.new_worker(WB(12)); rt.schedule()
    assert rt.n_assigned(ts) == 4 and rt.task(t1).state == "waiting"
    rt = TestEnv(); ts = rt.new_tasks(5, TB().cpus(3)); t1 = rt.new_task(TB().cpus_all().weight(1.1))
    rt.new_worker(WB(12)); rt.schedule()
    assert rt.n_assigned(ts) == 0 and rt.task(t1).is_assigned()


def test_schedule_min_utilization1():
    """test_scheduler_sn.rs:1391-1412."""
    rt = TestEnv(); ts = rt.new_tasks(2, TB().cpus(3)); rt.new_worker(WB(9).min_utilization(1.0)); rt.schedule()
    assert rt.n_assigned(ts) == 0
    rt = TestEnv(); ts = rt.new_tasks(3, TB().cpus(3)); rt.new_worker(WB(9).min_utilization(1.0)); rt.schedule()
    assert rt.n_assigned(ts) == 3
    rt = TestEnv(); ts = rt.new_tasks(2, TB().cpus(3)); w = rt.new_worker(WB(9).min_utilization(1.0))
    rt.new_task_running(TB().cpus(3), w); rt.schedule()
    assert rt.n_assigned(ts) == 2


def test_schedule_min_utilization2():
    """test_scheduler_sn.rs:1414-1445."""
    for n, mu, exp in [(2, 0.5, 2), (2, 0.51, 0), (3, 0.51, 3), (3, 0.75, 3), (3, 0.76, 0)]:
        rt = TestEnv(); ts = rt.new_tasks(n, TB().cpus(3)); rt.new_worker(WB(12).min_utilization(mu))
        rt.schedule()
        assert rt.n_assigned(ts) == exp, (n, mu)


def test_schedule_min_utilization3():
    """test_scheduler_sn.rs:1447-1463."""
    rt = TestEnv(); ts = rt.new_tasks(3, TB().cpus(3).weight(2.0)); t2 = rt.new_task(TB().cpus_all())
    rt.new_worker(WB(12).min_utilization(1.0)); rt.schedule()
    assert rt.n_assigned(ts) == 0 and rt.task(t2).is_assigned()
    rt = TestEnv(); ts = rt.new_tasks(4, TB().cpus(3).weight(2.0)); t2 = rt.new_task(TB().cpus_all())
    rt.new_worker(WB(12).min_utilization(1.0)); rt.schedule()
    assert rt.n_assigned(ts) == 4 and not rt.task(t2).is_assigned()


def test_schedule_mapping_do_not_change():
    """test_scheduler_mapping.rs:16-44: a second tick emits nothing; a task whose only capable worker is busy stays
    in the queue without disturbing the existing assignment."""
    rt = TestEnv()
    rt.new_named_resource("gpus")
    w1 = rt.new_worker(WB(6).res_sum("gpus", 2))
    rt.new_worker(WB(3))
    t1 = rt.new_task(TB().cpus(5))
    rt.schedule()
    assert rt.task(t1).state == "assigned" and rt.task(t1).worker == w1
    assert t1 in rt.worker(w1).assigned_tasks
    assert not rt.schedule().workers
    rt.new_worker(WB(6))
    rt.new_task(TB().cpus(4).add_resource(1, 2))
    assert not rt.schedule().workers
