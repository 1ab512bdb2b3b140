"""hqs_graph_cancel in the sequential model (tests/graph_cancel_model.py) against the restated server core
(tests/graph_cancel_core.py: on_cancel_tasks, task_failed): random submits with dependencies, assignments, starts,
prefills, retracts, finishes, cancels of tasks in every modelled state (and of finished or unknown ones) and failures of
assigned and running tasks.  After every event the ready set, the prefilled set, the waiting set with its counters, and each
call's list (the tasks that left; for a failure, the consumers) must agree.  Then directed cases."""
import numpy as np
import pytest

import graph_cancel_model as CM
from graph_cancel_core import CancelCore
from level_model import KEY_PF, KEY_READY, Rejected
from oracle.core import Task
from oracle.model import COMPACT, AllocRequest, ResourceRequest, ResourceRequestVariants, Worker, WorkerResources, units

def _oracle():
    core = CancelCore()
    rq = core.get_or_create_resource_rq_id(ResourceRequestVariants((ResourceRequest.new([AllocRequest(0, COMPACT, units(1))]),)))
    core.new_worker(Worker(1, WorkerResources([units(1 << 20)])))
    core.new_worker(Worker(2, WorkerResources([units(1 << 20)])))
    return core, rq


def _records(tasks, worker, kind):
    rec = np.zeros(len(tasks), dtype=[("task", "<u4"), ("worker", "<u2"), ("variant", "u1"), ("kind", "u1")])
    rec["task"], rec["worker"], rec["kind"] = tasks, worker, kind
    return rec


def _compare(m, core, label):
    ready = sorted(int(h) for h in np.nonzero(m.has(KEY_READY))[0])
    assert ready == sorted(t.id for t in core.tasks.values() if t.is_ready() or t.state == "prefilled"), label
    pf = sorted(int(h) for h in np.nonzero(m.has(KEY_PF))[0])
    assert pf == sorted(t.id for t in core.tasks.values() if t.state == "prefilled"), label
    waiting = {t.id: t.unfinished_deps for t in core.tasks.values() if t.state == "waiting" and t.unfinished_deps > 0}
    assert {h: m.gdeps[h] for h in range(m.n_handles) if m.waiting(h)} == waiting, label
    assert m.debug()[3] == len(waiting), label


def _pick(rng, xs, k):
    xs = sorted(xs)
    return [xs[j] for j in sorted(set(rng.integers(0, len(xs), size=min(len(xs), k)).tolist()))] if xs else []


def _prefill(core, t, w):
    """A ready task is prefilled on worker w (mapping.rs:156-230 through TaskQueue::take_tasks_for_prefill)."""
    task = core.tasks[t]
    q = core.task_queues.get(task.rq_id)
    if q.prefill is not None and q.prefill[0] != task.priority:
        return False
    core.remove_from_ready_queue(t)
    q.prefill = (task.priority, (q.prefill[1] if q.prefill else set()) | {t})
    task.state, task.worker = "prefilled", w
    core.workers[w].prefilled_tasks.add(t)
    return True


def _retract(core, t, target):
    """A prefilled task is assigned elsewhere: retracting from its worker, redirected to `target` (mapping.rs:63-101)."""
    task = core.tasks[t]
    core.task_queues.get(task.rq_id).remove_prefilled(t)
    core.workers[task.worker].prefilled_tasks.remove(t)
    core.workers[target].insert_sn_task(t, core.rq_map.get(task.rq_id).variants[0])
    core.scheduler_state.redirects[t] = (target, 0)
    task.state = "retracting"


@pytest.mark.parametrize("seed", range(8))
def test_random_cancels_and_failures_match_the_server_core(seed):
    rng = np.random.default_rng(1000 + seed)
    core, rq = _oracle()
    m = CM.CancelModel()
    m.classes_set(1)
    next_id, gone = 0, []
    seen = dict(cancel_named={}, fail=0, consumers=0)
    for step in range(160):
        ev = int(rng.integers(0, 7)) if next_id else 0
        by = lambda *states: [t.id for t in core.tasks.values() if t.state in states]
        if ev == 0:                                       # a job with dependencies
            k = int(rng.integers(1, 30))
            ids = list(range(next_id, next_id + k))
            next_id += k
            if rng.random() < 0.3:
                rng.shuffle(ids)
            live = list(core.tasks)
            deps = []
            for i, t in enumerate(ids):
                pool = live[-60:] + ids[:i] * 3 + ids[i + 1:] + gone[-20:]
                cand = {int(pool[j]) for j in rng.integers(0, len(pool), size=int(rng.integers(0, 4)))} if pool else set()
                deps.append(sorted(cand - {t}))
            off = np.concatenate([[0], np.cumsum([len(d) for d in deps])]).astype(np.int64)
            m.graph_push(ids, np.zeros(k, np.uint32), np.full(k, 7, np.uint64), off, [d for ds in deps for d in ds])
            core.on_new_tasks([Task(t, rq, 0, deps=tuple(ds)) for t, ds in zip(ids, deps)])
        elif ev == 1:                                     # assignments; some start running
            pick = _pick(rng, [t.id for t in core.tasks.values() if t.is_ready()], 6)
            for t in pick:
                core.assign_task(t, 1)
                if rng.random() < 0.5:
                    core.start_task(t)
            m.apply_tick(_records(pick, 0, 0))
        elif ev == 2:                                     # prefills, and retracts of earlier prefills
            pick = [t for t in _pick(rng, [t.id for t in core.tasks.values() if t.is_ready()], 4) if _prefill(core, t, 1)]
            m.apply_tick(_records(pick, 0, 1))
            red = _pick(rng, [t for t in by("prefilled") if t not in pick], 2)
            for t in red:
                _retract(core, t, 2)
            m.apply_tick(_records(red, 1, 2))
        elif ev == 3:                                     # finishes
            pick = _pick(rng, by("assigned", "running"), 5)
            made = m.graph_finished(pick)
            before = {t.id for t in core.tasks.values() if t.is_ready()}
            for t in pick:
                core.task_finished(core.tasks[t].worker, t)
            gone += pick
            assert made == sorted({t.id for t in core.tasks.values() if t.is_ready()} - before), step
        elif ev in (4, 5):                                # cancels: tasks in any state, finished and unknown ones
            states = ["waiting", "assigned", "running", "prefilled", "retracting"]
            named = []
            for s in rng.permutation(states)[: int(rng.integers(1, 4))]:
                named += _pick(rng, by(str(s)), 2)
            named += _pick(rng, gone, 1)
            if rng.random() < 0.3 and named:
                named = named + named[:1]                 # named twice: counts once
            for t in named:
                st = core.tasks[t].state if t in core.tasks else "gone"
                seen["cancel_named"][st] = seen["cancel_named"].get(st, 0) + 1
            got = m.graph_cancel(named)
            core.on_cancel_tasks(list(dict.fromkeys(named)))   # tako's clients name each task once
            assert got == sorted(core.last_removed), step
            gone += got
        else:                                             # a failure of an assigned or running task
            pick = _pick(rng, by("assigned", "running"), 1)
            if pick:
                t = pick[0]
                got = m.graph_cancel([t])
                cons = core.task_failed(core.tasks[t].worker, t)
                assert [x for x in got if x != t] == cons and t in got, step
                seen["fail"] += 1
                seen["consumers"] += len(cons)
                gone += got
        _compare(m, core, step)
    core.sanity_check()
    assert {"waiting", "assigned", "running", "prefilled", "gone"} <= set(seen["cancel_named"]), seen


def _push(m, deps, first=0):
    ids = list(range(first, first + len(deps)))
    off = np.concatenate([[0], np.cumsum([len(d) for d in deps])]).astype(np.int64)
    return m.graph_push(ids, np.zeros(len(ids), np.uint32), np.full(len(ids), 3, np.uint64), off, [d for ds in deps for d in ds])


def _model():
    m = CM.CancelModel()
    m.classes_set(1)
    return m


def test_a_diamond_lists_the_shared_consumer_once():
    m = _model()
    _push(m, [[], [0], [0], [1, 2], [3]])
    assert m.graph_cancel([0]) == [0, 1, 2, 3, 4]
    assert m.debug()[0] == 0 and m.debug()[3] == 0


def test_a_named_task_that_is_also_a_consumer_of_another_named_task():
    m = _model()
    _push(m, [[], [0], [1], []])
    assert m.graph_cancel([2, 0, 3]) == [0, 1, 2, 3]
    assert m.n_handles == 4 and not m.has(KEY_READY).any()


def test_a_resubmitted_consumer_is_not_cancelled_by_its_old_producer():
    m = _model()
    _push(m, [[], [0]])
    m.remove([1])                                         # the consumer is cancelled alone ...
    _push(m, [[]], first=1)                               # ... and submitted again without dependencies
    assert m.graph_cancel([0]) == [0]                     # the old edge 0 -> 1 is stale
    assert m.has(KEY_READY)[1]
    _push(m, [[], [], [1]], first=2)                      # 4 waits on the new incarnation of 1
    m.graph_cancel([1])
    assert not m.waiting(4) and m.debug()[3] == 0


def test_duplicates_and_not_valid_names():
    m = _model()
    _push(m, [[], [0], [], [2]])
    m.apply_tick(_records([2], 0, 0))
    assert m.graph_finished([2]) == [3]
    keys = m.keys().copy()
    assert m.graph_cancel([2, 2]) == []                   # finished: not VALID, nothing changes
    assert np.array_equal(m.keys(), keys)
    assert m.graph_cancel([0, 0, 1, 0]) == [0, 1]
    assert m.graph_cancel([]) == []
    with pytest.raises(Rejected):
        m.graph_cancel([3, 4])                            # 4 >= n_handles: the whole batch is rejected
    assert m.has(KEY_READY)[3]


def test_a_failed_task_reports_its_waiting_consumers_only():
    core, rq = _oracle()
    core.on_new_tasks([Task(0, rq), Task(1, rq), Task(2, rq, deps=(0,)), Task(3, rq, deps=(2, 1)), Task(4, rq, deps=(1,))])
    core.assign_task(0, 1)
    core.assign_task(1, 2)
    core.start_task(1)
    assert core.task_failed(1, 0) == [2, 3]
    assert sorted(core.tasks) == [1, 4] and core.tasks[4].unfinished_deps == 1
    assert core.workers[1].assigned_tasks == set()
    msgs = core.on_cancel_tasks([1, 9])
    assert msgs == {2: [1]} and core.last_removed == {1, 4} and not core.tasks
