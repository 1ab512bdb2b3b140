"""Autoalloc what-if query, restated (TEST INFRASTRUCTURE — see oracle/__init__.py).

Follows hyperqueue/crates/tako/src/internal/scheduler/query.rs:
  :12-70    fake workers per WorkerTypeQuery (partial descriptors get ResourceAmount::MAX for every resource
            the query does not name)
  :72-95    create_task_batches + run_scheduling_solver over the FAKE workers only; a fake worker is "needed" iff
            it receives at least one task
  :97-131   multi-node allocations — not restated (multi-node requests are outside this path)
Pinned by tests/test_oracle_query.py (transcribed from tests/test_query.rs).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

from .batches import create_task_batches
from .model import AMOUNT_MAX, Worker, WorkerResources, units
from .solver import run_scheduling_solver


@dataclass
class WorkerTypeQuery:
    """control.rs WorkerTypeQuery; `resources` = [(resource name, amount in units)] of the descriptor."""
    resources: Sequence[Tuple[str, int]]
    partial: bool = False
    time_limit: Optional[float] = None          # seconds
    max_sn_workers: int = 1
    max_workers_per_allocation: int = 1
    min_utilization: float = 0.0

    @staticmethod
    def simple_cpus(cpus: int, **kw) -> "WorkerTypeQuery":
        return WorkerTypeQuery([("cpus", cpus)], **kw)


@dataclass
class NewWorkerAllocationResponse:
    single_node_workers_per_query: List[int] = field(default_factory=list)
    multi_node_allocations: list = field(default_factory=list)


def compute_new_worker_query(core, queries: Sequence[WorkerTypeQuery], now: float = 0.0) -> NewWorkerAllocationResponse:
    fake_id = max(core.workers.keys(), default=0) + 1            # query.rs:18-19 (worker_counter + 1)
    for q in queries:                                             # query.rs:21-26
        for name, _ in q.resources:
            core.get_or_create_resource_id(name)
    n_res = core.n_resources()
    fake_workers: List[Worker] = []
    for q in queries:
        for _ in range(q.max_sn_workers):
            ids = [core.resource_names.index(name) for name, _ in q.resources]
            if q.partial:                                         # query.rs:35-46
                vec = [AMOUNT_MAX] * n_res
            else:
                vec = [0] * ((max(ids) + 1) if ids else 0)        # WorkerResources::from_description
            for rid, (_, amount) in zip(ids, q.resources):
                vec[rid] = units(amount)
            term = None if q.time_limit is None else now + q.time_limit
            fake_workers.append(Worker(fake_id, WorkerResources(vec), termination_time=term,
                                       min_utilization=q.min_utilization, group=f"fake-worker-group-{fake_id}"))
            fake_id += 1
    batches = create_task_batches(core, now, fake_workers)
    solution = run_scheduling_solver(core, now, batches, fake_workers)
    loaded = set()
    for counts in solution.sn_counts.values():
        for wid, c in counts.items():
            if c > 0:
                loaded.add(wid)
    out = NewWorkerAllocationResponse()
    i = 0
    for q in queries:
        n = 0
        for _ in range(q.max_sn_workers):
            if fake_workers[i].id in loaded:
                n += 1
            i += 1
        out.single_node_workers_per_query.append(n)
    return out
