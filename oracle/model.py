"""Resource model of the tako scheduler, restated (TEST INFRASTRUCTURE — see oracle/__init__.py).

Follows (paths relative to hyperqueue/crates/tako/src/internal/):
  common/resources/amount.rs:7,26-104      ResourceAmount: u64 fixed point, 10 000 fractions per unit
  common/resources/request.rs:13-83        AllocationRequest (6 policies, `All` has no amount)
  common/resources/request.rs:107-134      ResourceWeight (u32, x10 000)
  common/resources/request.rs:136-227      ResourceRequest (entries sorted by resource id)
  common/resources/request.rs:229-353      ResourceRequestVariants (<= 32 variants)
  common/resources/map.rs:99-109           ResourceRqMap interning -> ResourceRqId
  server/workerload.rs:16-226              WorkerResources
  server/worker.rs:40-84,181-338           Worker predicates
  common/priority.rs:36-48                 Priority from user priority
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, Iterable, List, Optional, Sequence, Set, Tuple

import numpy as np

FRACTIONS_PER_UNIT = 10_000          # amount.rs:7
AMOUNT_MAX = (1 << 64) - 1           # amount.rs:30  ResourceAmount::MAX
MAX_TASK_PER_WORKER = 1024           # workerload.rs:12
CPU_RESOURCE_ID = 0                  # map.rs:7

# AllocationRequest discriminants (request.rs:13-21)
COMPACT, TIGHT, SCATTER, FORCE_COMPACT, FORCE_TIGHT, ALL = range(6)


def units(n: int) -> int:
    """ResourceAmount::new_units (amount.rs:37-39)."""
    return int(n) * FRACTIONS_PER_UNIT


def amount(u: int, fractions: int = 0) -> int:
    """ResourceAmount::new (amount.rs:32-35)."""
    assert 0 <= fractions < FRACTIONS_PER_UNIT
    return int(u) * FRACTIONS_PER_UNIT + int(fractions)


def amount_from_float(value: float) -> int:
    """ResourceAmount::from_float: ceil of an f32 product (amount.rs:41-43)."""
    v = np.float32(value) * np.float32(FRACTIONS_PER_UNIT)
    return int(math.ceil(float(v)))


def as_f64(a: int) -> float:
    """amount.rs:90-92."""
    return float(a) / float(FRACTIONS_PER_UNIT)


def priority_from_user(user_priority: int) -> int:
    """Priority::from_user_priority (priority.rs:43-48): order-preserving i32 -> high 32 bits of a u64."""
    return (((int(user_priority) & 0xFFFFFFFF) ^ 0x8000_0000) << 32) & AMOUNT_MAX


@dataclass(frozen=True)
class AllocRequest:
    """ResourceAllocRequest (request.rs:98-102): one entry of a request."""
    resource_id: int
    policy: int
    amount: int = 0          # ignored for ALL

    def min_amount(self) -> int:
        # request.rs:34-36: amount(ResourceAmount::ONE) -> 1 fraction for All
        return 1 if self.policy == ALL else self.amount

    def amount_or_none_if_all(self) -> Optional[int]:
        return None if self.policy == ALL else self.amount

    def is_all(self) -> bool:
        return self.policy == ALL


@dataclass(frozen=True)
class ResourceRequest:
    """request.rs:136-167.  `entries` is kept sorted by resource id (request.rs:160)."""
    entries: Tuple[AllocRequest, ...]
    n_nodes: int = 0
    min_time: float = 0.0            # seconds
    weight: int = 10_000             # ResourceWeight raw value (request.rs:107-134)

    @staticmethod
    def new(entries: Iterable[AllocRequest], n_nodes: int = 0, min_time: float = 0.0,
            weight: float = 1.0) -> "ResourceRequest":
        es = tuple(sorted(entries, key=lambda e: e.resource_id))
        # ResourceWeight::try_from: (value * 10_000f32).round() as u32 (request.rs:110-118)
        w = int(np.round(np.float32(weight) * np.float32(10_000)))
        assert w > 0
        return ResourceRequest(es, n_nodes, float(min_time), w)

    def is_multi_node(self) -> bool:
        return self.n_nodes > 0

    def weight_f64(self) -> float:
        return self.weight / 10_000.0

    def get_amount(self, r_id: int) -> Optional[int]:
        """request.rs:183-189: Some(amount) / None for All / Some(0) if not requested."""
        for e in self.entries:
            if e.resource_id == r_id:
                return e.amount_or_none_if_all()
        return 0

    def validate(self) -> None:
        # request.rs:191-206 + AllocationRequest::validate (request.rs:24-32)
        if not self.entries and self.n_nodes == 0:
            raise ValueError("Resource request is empty")
        for e in self.entries:
            if e.policy != ALL and e.amount == 0:
                raise ValueError("Zero resources cannot be requested")
        for a, b in zip(self.entries, self.entries[1:]):
            if a.resource_id >= b.resource_id:
                raise ValueError("Request are not sorted or unique")


@dataclass(frozen=True)
class ResourceRequestVariants:
    """request.rs:229-353."""
    variants: Tuple[ResourceRequest, ...]

    def is_multi_node(self) -> bool:
        return self.variants[0].is_multi_node()

    def trivial_request(self) -> Optional[ResourceRequest]:
        return self.variants[0] if len(self.variants) == 1 else None

    def min_time(self) -> float:
        return min((v.min_time for v in self.variants), default=0.0)

    def validate(self) -> None:
        if not self.variants:
            raise ValueError("Resource are empty")
        if len(self.variants) > 32:
            raise ValueError("Too many resource variants")
        mn = self.variants[0].is_multi_node()
        for rq in self.variants:
            rq.validate()
            if rq.is_multi_node() != mn:
                raise ValueError("Resources mixes multi-node and non-multi-node requests")


class ResourceRqMap:
    """Interning of ResourceRequestVariants -> dense ResourceRqId (map.rs:77-109)."""

    def __init__(self) -> None:
        self._ids: Dict[ResourceRequestVariants, int] = {}
        self._rqvs: List[ResourceRequestVariants] = []

    def get_or_create(self, rqv: ResourceRequestVariants) -> Tuple[int, bool]:
        rid = self._ids.get(rqv)
        if rid is not None:
            return rid, False
        rid = len(self._rqvs)
        self._ids[rqv] = rid
        self._rqvs.append(rqv)
        return rid, True

    def get(self, rq_id: int) -> ResourceRequestVariants:
        return self._rqvs[rq_id]

    def __len__(self) -> int:
        return len(self._rqvs)

    def is_empty(self) -> bool:
        return not self._rqvs


class WorkerResources:
    """Per-worker vector of amounts indexed by resource id (workerload.rs:16-226)."""

    __slots__ = ("n",)

    def __init__(self, amounts: Sequence[int]) -> None:
        self.n: List[int] = [int(a) for a in amounts]

    def clone(self) -> "WorkerResources":
        return WorkerResources(self.n)

    def key(self) -> Tuple[int, ...]:
        return tuple(self.n)

    def __eq__(self, other: object) -> bool:
        return isinstance(other, WorkerResources) and self.n == other.n

    def __hash__(self) -> int:
        return hash(tuple(self.n))

    def __repr__(self) -> str:
        return "WR(" + ",".join(str(a / FRACTIONS_PER_UNIT) for a in self.n) + ")"

    def get(self, r_id: int) -> int:
        # workerload.rs:26-31: missing resource => ZERO
        return self.n[r_id] if r_id < len(self.n) else 0

    def _ensure(self, r_id: int) -> None:
        # The reference indexes n_resources[r] directly (would panic when out of range); resource
        # vectors there are always long enough when remove/add is legal.  We grow defensively.
        while len(self.n) <= r_id:
            self.n.append(0)

    def iter_pairs(self) -> Iterable[Tuple[int, int]]:
        # workerload.rs:33-46: only non-zero entries
        return [(i, a) for i, a in enumerate(self.n) if a != 0]

    def is_capable_to_run_request(self, rq: ResourceRequest) -> bool:
        # workerload.rs:77-83
        return all(e.min_amount() <= self.get(e.resource_id) for e in rq.entries)

    def task_max_count_for_request(self, rq: ResourceRequest) -> int:
        # workerload.rs:121-145
        best: Optional[int] = None
        for e in rq.entries:
            a = e.amount_or_none_if_all()
            if a is not None:
                c = min(self.get(e.resource_id) // a, MAX_TASK_PER_WORKER)
            elif self.get(e.resource_id) == 0:
                c = 0
            else:
                c = 1
            best = c if best is None else min(best, c)
        return 0 if best is None else best

    def task_max_count(self, rqv: ResourceRequestVariants) -> int:
        # workerload.rs:147-154: SUM over variants (flagged TODO in the reference)
        return sum(self.task_max_count_for_request(r) for r in rqv.variants)

    def remove(self, rq: ResourceRequest) -> None:
        # workerload.rs:156-165
        self.remove_multiple(rq, 1)

    def remove_multiple(self, rq: ResourceRequest, n: int) -> None:
        # workerload.rs:167-178 (saturating_sub; All => ZERO)
        for e in rq.entries:
            self._ensure(e.resource_id)
            a = e.amount_or_none_if_all()
            if a is not None:
                self.n[e.resource_id] = max(0, self.n[e.resource_id] - a * n)
            else:
                self.n[e.resource_id] = 0

    def add(self, rq: ResourceRequest, total: "WorkerResources") -> None:
        # workerload.rs:194-202
        for e in rq.entries:
            self._ensure(e.resource_id)
            a = e.amount_or_none_if_all()
            if a is not None:
                self.n[e.resource_id] += a
            else:
                self.n[e.resource_id] = total.get(e.resource_id)


@dataclass
class Worker:
    """server/worker.rs:40-84, single-node view only (multi-node assignment: out of first slice)."""
    id: int
    resources: WorkerResources                       # totals
    free: WorkerResources = None                     # sn_assignment().free_resources
    assigned_tasks: Set = field(default_factory=set)
    prefilled_tasks: Set = field(default_factory=set)
    blocked_requests: Set[Tuple[int, int]] = field(default_factory=set)
    termination_time: Optional[float] = None         # absolute seconds; None = no limit
    min_utilization: float = 0.0
    group: str = "default"
    stopping: bool = False
    mn_task: Optional[object] = None                 # WorkerAssignment::Mn marker

    def __post_init__(self) -> None:
        if self.free is None:
            self.free = self.resources.clone()       # WorkerAssignment::empty_sn (worker.rs:53-61)

    def is_sn(self) -> bool:
        return self.mn_task is None

    def is_free(self) -> bool:
        # worker.rs:181-186
        return self.is_sn() and not self.assigned_tasks and not self.stopping

    def has_time_to_run(self, time_request: float, now: float) -> bool:
        # worker.rs:320-326
        return self.termination_time is None or now + time_request <= self.termination_time

    def have_immediate_resources_for_rq(self, rq: ResourceRequest) -> bool:
        # worker.rs:273-278
        return self.is_sn() and self.free.is_capable_to_run_request(rq)

    def is_capable_to_run(self, rq: ResourceRequest, now: float) -> bool:
        # worker.rs:280-289
        if not self.has_time_to_run(rq.min_time, now):
            return False
        return True if rq.is_multi_node() else self.resources.is_capable_to_run_request(rq)

    def is_capable_to_run_rqv(self, rqv: ResourceRequestVariants, now: float) -> bool:
        # worker.rs:291-299
        return any(self.is_capable_to_run(r, now) for r in rqv.variants)

    def is_request_blocked(self, rq_id: int, rv: int) -> bool:
        return (rq_id, rv) in self.blocked_requests

    def insert_sn_task(self, task_id, rq: ResourceRequest) -> None:
        # worker.rs:188-196
        self.free.remove(rq)
        assert task_id not in self.assigned_tasks
        self.assigned_tasks.add(task_id)

    def remove_sn_task(self, task_id, rq: ResourceRequest) -> None:
        # worker.rs:223-234
        self.assigned_tasks.remove(task_id)
        self.free.add(rq, self.resources)
