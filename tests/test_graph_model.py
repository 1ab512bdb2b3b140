"""The sequential task-graph model (tests/graph_model.py) against the restated server core (oracle/core.py: on_new_tasks,
assign_task, task_finished): random submits of task batches with dependencies on live, running and finished tasks and on
earlier and later tasks of the same batch (in handle order or shuffled), random assignments and random finishes.  After
every event the ready set, the waiting set with its dependency counters, and each finish's newly ready tasks must agree."""
import numpy as np
import pytest

import graph_model as GM
from level_model import KEY_READY, Rejected
from oracle.core import Core, Task
from oracle.model import (COMPACT, AllocRequest, ResourceRequest, ResourceRequestVariants, Worker, WorkerResources,
                          priority_from_user, units)


def _oracle():
    core = Core()
    rq = core.get_or_create_resource_rq_id(ResourceRequestVariants((ResourceRequest.new([AllocRequest(0, COMPACT, units(1))]),)))
    core.new_worker(Worker(1, WorkerResources([units(1 << 20)])))
    return core, rq


def _compare(m, core, label):
    ready = sorted(int(h) for h in np.nonzero(m.has(KEY_READY))[0])
    assert ready == sorted(t.id for t in core.tasks.values() if t.is_ready()), label
    waiting = {t.id: t.unfinished_deps for t in core.tasks.values() if t.state == "waiting" and t.unfinished_deps > 0}
    assert {h: m.gdeps[h] for h in range(m.n_handles) if m.waiting(h)} == waiting, label
    assert m.debug()[3] == len(waiting), label


@pytest.mark.parametrize("seed", range(6))
def test_random_submits_and_finishes_match_the_server_core(seed):
    rng = np.random.default_rng(seed)
    core, rq = _oracle()
    m = GM.GraphModel()
    m.classes_set(1)
    next_id, finished, running = 0, [], set()
    for step in range(120):
        ev = rng.integers(0, 3)
        if ev == 0 or next_id == 0:
            k = int(rng.integers(1, 40))
            ids = list(range(next_id, next_id + k))
            next_id += k
            if rng.random() < 0.3:
                rng.shuffle(ids)
            live = [t for t in core.tasks]
            deps = []
            for i, t in enumerate(ids):
                pool = live + ids[:i] * 2 + ids[i + 1:] + finished[-50:]
                cand = {int(pool[j]) for j in rng.integers(0, len(pool), size=int(rng.integers(0, 6)))} if pool else set()
                deps.append(sorted(cand - {t}))
            prio = rng.integers(0, 3, size=k)
            off = np.concatenate([[0], np.cumsum([len(d) for d in deps])]).astype(np.int64)
            flat = [d for ds in deps for d in ds]
            before = {t.id for t in core.tasks.values() if t.is_ready()}
            n_ready = m.graph_push(ids, np.zeros(k, np.uint32), priority_from_user_vec(prio), off, flat)
            core.on_new_tasks([Task(t, rq, int(p), deps=tuple(ds)) for t, p, ds in zip(ids, prio.tolist(), deps)])
            after = {t.id for t in core.tasks.values() if t.is_ready()}
            assert n_ready == len(after - before), step
        elif ev == 1:
            ready = sorted(t.id for t in core.tasks.values() if t.is_ready())
            pick = [ready[j] for j in sorted(set(rng.integers(0, len(ready), size=min(len(ready), 8)).tolist()))] if ready else []
            for t in pick:
                core.assign_task(t, 1)
                running.add(t)
            rec = np.zeros(len(pick), dtype=[("task", "<u4"), ("worker", "<u2"), ("variant", "u1"), ("kind", "u1")])
            rec["task"] = pick
            m.apply_tick(rec)
        else:
            run = sorted(running)
            pick = [run[j] for j in sorted(set(rng.integers(0, len(run), size=min(len(run), 6)).tolist()))] if run else []
            if rng.random() < 0.3 and pick:
                pick = pick + pick[:1]                         # a task named twice counts once
            before = {t.id for t in core.tasks.values() if t.is_ready()}
            made = m.graph_finished(pick)
            for t in dict.fromkeys(pick):
                core.task_finished(1, t)
                running.discard(t)
                finished.append(t)
            after = {t.id for t in core.tasks.values() if t.is_ready()}
            assert made == sorted(after - before), step
        _compare(m, core, step)


def priority_from_user_vec(user):
    return np.array([priority_from_user(int(u)) for u in user], dtype=np.uint64)


def test_rejections_leave_the_model_unchanged():
    m = GM.GraphModel()
    m.classes_set(2)
    m.graph_push([0, 1], [0, 1], [5, 5], [0, 0, 1], [0])
    keys, dbg = m.keys().copy(), m.debug()
    bad = [
        ([2], [2], [1], [0, 0], []),                 # class id
        ([2, 2], [0, 0], [1, 1], [0, 0, 0], []),     # a handle twice
        ([0xFFFFFFFF], [0], [1], [0, 0], []),        # the reserved handle
        ([1], [0], [1], [0, 0], []),                 # a live handle
        ([2], [0], [1], [0, 1], [2]),                # depends on itself
        ([2], [0], [1], [0, 2], [0, 0]),             # the same dependency twice
        ([2], [0], [1], [0, 1], [9]),                # neither in the batch nor < n_handles
        ([2], [0], [1], [1, 1], [0]),                # dep_off does not start at 0
        ([2, 3], [0, 0], [1, 1], [0, 1, 0], [0]),    # dep_off decreases
    ]
    for args in bad:
        with pytest.raises(Rejected):
            m.graph_push(*args)
        assert np.array_equal(m.keys(), keys) and m.debug() == dbg, args
    with pytest.raises(Rejected):
        m.graph_finished([0, 5])
    assert np.array_equal(m.keys(), keys) and m.debug() == dbg


def test_a_resubmitted_handle_is_not_released_by_its_old_producers():
    m = GM.GraphModel()
    m.classes_set(1)
    assert m.graph_push([0, 1], [0, 0], [1, 1], [0, 0, 1], [0]) == 1
    m.remove([1])                                    # the consumer is cancelled
    assert m.graph_push([1, 2], [0, 0], [1, 1], [0, 0, 0], []) == 2
    assert m.graph_push([3], [0], [1], [0, 1], [2]) == 0
    m.remove([1])
    assert m.graph_push([1], [0], [1], [0, 1], [2]) == 0   # waits on 2 only
    assert m.graph_finished([0]) == []               # the old edge 0 -> 1 is stale
    assert m.waiting(1)
    assert m.graph_finished([2, 2]) == [1, 3]
    assert m.debug() == [0, GM.POOL_MIN, 0, 0]
