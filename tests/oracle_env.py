"""Test DSL over the oracle, mirroring the reference's own test helpers so that the golden vectors can
be transcribed one to one:
  hyperqueue/crates/tako/src/internal/tests/utils/env.rs        TestEnv (worker ids from 50, task ids from 1)
  .../tests/utils/task.rs        TaskBuilder     .../tests/utils/worker.rs   WorkerBuilder
  .../tests/utils/resources.rs   ResBuilder (adds 1 cpu if no cpu entry: resources.rs:99-109)
  .../tests/utils/scheduler.rs   TestCase (expect_tasks / expect_request_v / eq_class / running_c)
"""
from __future__ import annotations

import copy
from typing import Dict, List, Optional, Sequence, Tuple

from oracle import model as M
from oracle.core import Core, SchedulerConfig, Task
from oracle.mapping import WorkerTaskMapping, WorkerTaskUpdate


class TaskBuilder:
    def __init__(self) -> None:
        self._finished: List[M.ResourceRequest] = []
        self._entries: List[M.AllocRequest] = []
        self._min_time = 0.0
        self._weight = 1.0
        self._user_priority = 0
        self._deps: Tuple = ()

    def _c(self) -> "TaskBuilder":
        return copy.deepcopy(self)

    def user_priority(self, p: int) -> "TaskBuilder":
        b = self._c(); b._user_priority = p; return b

    def task_deps(self, deps: Sequence) -> "TaskBuilder":
        b = self._c(); b._deps = tuple(deps); return b

    def cpus(self, n) -> "TaskBuilder":
        return self.add_resource(0, n)

    def cpus_all(self) -> "TaskBuilder":
        b = self._c(); b._entries.append(M.AllocRequest(0, M.ALL)); return b

    def add_resource(self, rid: int, n) -> "TaskBuilder":
        b = self._c()
        amt = M.units(n) if isinstance(n, int) else M.amount_from_float(n)
        b._entries.append(M.AllocRequest(rid, M.COMPACT, amt))
        return b

    def weight(self, w: float) -> "TaskBuilder":
        b = self._c(); b._weight = w; return b

    def time_request(self, secs: float) -> "TaskBuilder":
        b = self._c(); b._min_time = float(secs); return b

    def _finish_current(self) -> M.ResourceRequest:
        entries = list(self._entries)
        if not any(e.resource_id == 0 for e in entries):
            entries.insert(0, M.AllocRequest(0, M.COMPACT, M.units(1)))
        return M.ResourceRequest.new(entries, 0, self._min_time, self._weight)

    def next_variant(self) -> "TaskBuilder":
        b = self._c()
        b._finished.append(self._finish_current())
        b._entries, b._min_time, b._weight = [], 0.0, 1.0
        return b

    def build_rqv(self) -> M.ResourceRequestVariants:
        rqv = M.ResourceRequestVariants(tuple(self._finished + [self._finish_current()]))
        rqv.validate()
        return rqv


class WorkerBuilder:
    def __init__(self, cpus: Optional[int] = None) -> None:
        self.items: List[Tuple[str, int]] = [] if cpus is None else [("cpus", cpus)]
        self._time_limit: Optional[float] = None
        self._min_utilization = 0.0
        self._group = "default"

    def _c(self) -> "WorkerBuilder":
        return copy.deepcopy(self)

    def res_sum(self, name: str, amount: int) -> "WorkerBuilder":
        b = self._c(); b.items.append((name, amount)); return b

    def res_range(self, name: str, start: int, end: int) -> "WorkerBuilder":
        b = self._c(); b.items.append((name, end - start + 1)); return b

    def time_limit_s(self, secs: float) -> "WorkerBuilder":
        b = self._c(); b._time_limit = float(secs); return b

    def min_utilization(self, v: float) -> "WorkerBuilder":
        b = self._c(); b._min_utilization = v; return b


class TestEnv:
    __test__ = False

    def __init__(self) -> None:
        self.core = Core()
        self.task_id_counter = 1
        self.worker_id_counter = 50
        self.now = 0.0

    def set_scheduler_config(self, reserve: int, maximum: int) -> None:
        self.core.scheduler_state.config = SchedulerConfig(reserve, maximum)

    def new_named_resource(self, name: str) -> int:
        return self.core.get_or_create_resource_id(name)

    def new_generic_resource(self, count: int) -> None:
        for i in range(count):
            self.core.get_or_create_resource_id(f"Res{i}")

    def task(self, task_id) -> Task:
        return self.core.tasks[task_id]

    def new_task(self, builder: TaskBuilder):
        task_id = self.task_id_counter
        self.task_id_counter += 1
        rq_id = self.core.get_or_create_resource_rq_id(builder.build_rqv())
        self.core.on_new_tasks([Task(task_id, rq_id, builder._user_priority, deps=builder._deps)])
        return task_id

    def new_tasks(self, n: int, builder: TaskBuilder) -> list:
        return [self.new_task(builder) for _ in range(n)]

    def new_task_cpus(self, cpus: int):
        return self.new_task(TaskBuilder().cpus(cpus))

    def new_task_default(self):
        return self.new_task(TaskBuilder())

    def new_task_running(self, builder: TaskBuilder, worker_id: int):
        t = self.new_task(builder)
        self.core.assign_task(t, worker_id)
        self.core.start_task(t)
        return t

    def assign_and_start_task(self, task_id, worker_id: int, rv: int = 0) -> None:
        self.core.assign_task(task_id, worker_id, rv)
        self.core.start_task(task_id, rv)

    def new_worker(self, builder: WorkerBuilder) -> int:
        wid = self.worker_id_counter
        self.worker_id_counter += 1
        # WorkerResources::from_description (workerload.rs:48-75): vector as long as the highest
        # resource index present in the descriptor
        ids = [self.core.resource_names.index(n) if n in self.core.resource_names
               else self.core.get_or_create_resource_id(n) for n, _ in builder.items]
        vec = [0] * ((max(ids) + 1) if ids else 0)
        for rid, (_, amount) in zip(ids, builder.items):
            vec[rid] = M.units(amount)
        term = None if builder._time_limit is None else self.now + builder._time_limit
        self.core.new_worker(M.Worker(wid, M.WorkerResources(vec), termination_time=term,
                                      min_utilization=builder._min_utilization, group=builder._group))
        return wid

    def new_workers(self, n: int, builder: WorkerBuilder) -> List[int]:
        return [self.new_worker(builder) for _ in range(n)]

    def new_workers_cpus(self, cpus: Sequence[int]) -> List[int]:
        return [self.new_worker(WorkerBuilder(c)) for c in cpus]

    def worker(self, wid: int) -> M.Worker:
        return self.core.workers[wid]

    def worker_tasks(self, wid: int) -> set:
        return self.core.workers[wid].assigned_tasks

    def schedule(self) -> WorkerTaskMapping:
        mapping = self.core.schedule_mapping(self.now)
        self.core.sanity_check()
        return mapping

    def assigned_counts(self) -> List[int]:
        counts = [0] * len(self.core.rq_map)
        for t in self.core.tasks.values():
            if t.is_assigned():
                counts[t.rq_id] += 1
        return counts

    def n_assigned(self, tasks: Sequence) -> int:
        return sum(1 for t in tasks if self.core.tasks[t].is_assigned())


class _TestWorker:
    def __init__(self, case: "TestCase", worker_id: int) -> None:
        self.case = case
        self.worker_id = worker_id
        self.expect: Optional[object] = None        # None=Empty | list[(task, v)] | dict[(rq, v)] -> n
        self._eq_class: Optional[int] = None

    def eq_class(self, k: int) -> "_TestWorker":
        self._eq_class = k; return self

    def expect_tasks(self, tasks: Sequence) -> "_TestWorker":
        self.expect = [(t, 0) for t in tasks]; return self

    def expect_request(self, count: int, builder: TaskBuilder) -> "_TestWorker":
        return self.expect_request_v(count, builder, 0)

    def expect_request_v(self, count: int, builder: TaskBuilder, variant: int) -> "_TestWorker":
        rq_id = self.case.rt.core.get_or_create_resource_rq_id(builder.build_rqv())
        if not isinstance(self.expect, dict):
            self.expect = {}
        self.expect[(rq_id, variant)] = self.expect.get((rq_id, variant), 0) + count
        return self

    def running(self, builder: TaskBuilder) -> "_TestWorker":
        self.case.rt.new_task_running(builder, self.worker_id); return self

    def running_c(self, cpus: int) -> "_TestWorker":
        return self.running(TaskBuilder().cpus(cpus))


class TestCase:
    __test__ = False

    def __init__(self) -> None:
        self.rt = TestEnv()
        self.workers: List[_TestWorker] = []

    def resources(self, names: Sequence[str]) -> "TestCase":
        for n in names:
            self.rt.new_named_resource(n)
        return self

    def w(self, builder: WorkerBuilder) -> _TestWorker:
        tw = _TestWorker(self, self.rt.new_worker(builder))
        self.workers.append(tw)
        return tw

    def t(self, b: TaskBuilder):
        return self.rt.new_task(b)

    def ts(self, n: int, b: TaskBuilder) -> list:
        return [self.t(b) for _ in range(n)]

    def c_tasks(self, cpus: Sequence[int]) -> list:
        return [self.rt.new_task_cpus(c) for c in cpus]

    def pc_tasks(self, pcs: Sequence[Tuple[int, int]]) -> list:
        return [self.rt.new_task(TaskBuilder().cpus(c).user_priority(p)) for p, c in pcs]

    def mapping_per_worker(self, mapping: WorkerTaskMapping) -> Dict[int, List[Tuple[object, int]]]:
        per = {tw.worker_id: list(mapping.workers.get(tw.worker_id, WorkerTaskUpdate()).assigned)
               for tw in self.workers}
        # normalize_workers (scheduler.rs:97-106): sort the updates of an eq class
        for k in {tw._eq_class for tw in self.workers if tw._eq_class is not None}:
            ids = [tw.worker_id for tw in self.workers if tw._eq_class == k]
            ups = sorted(per[i] for i in ids)
            for i, up in zip(ids, ups):
                per[i] = up
        return per

    def check(self, exact_tasks: bool = True) -> None:
        mapping = self.rt.schedule()
        per = self.mapping_per_worker(mapping)
        for tw in self.workers:
            got = per[tw.worker_id]
            if tw.expect is None:
                assert got == [], (tw.worker_id, got)
            elif isinstance(tw.expect, list):
                if exact_tasks:
                    assert got == tw.expect, (tw.worker_id, got, tw.expect)
                else:
                    assert sorted(got) == sorted(tw.expect), (tw.worker_id, got, tw.expect)
            else:
                cnt: Dict[Tuple[int, int], int] = {}
                for t, v in got:
                    key = (self.rt.task(t).rq_id, v)
                    cnt[key] = cnt.get(key, 0) + 1
                assert cnt == tw.expect, (tw.worker_id, cnt, tw.expect)
