"""Gap computation ("how many low-priority tasks still fit beside a maximally packed high-priority
class"), restated (TEST INFRASTRUCTURE — see oracle/__init__.py).

Follows hyperqueue/crates/tako/src/internal/scheduler/gap.rs:
  :37-93    GapCache::get_gap
  :96-147   compute_gap_resources (one small LP per non-zero worker resource)
Pinned by the 13 asserts of gap.rs:175-246 (tests/test_oracle_golden.py::test_compute_gap).
"""
from __future__ import annotations

import math
from typing import Dict, Iterable, Tuple

from .lp import MAX, LpSolver
from .model import (ResourceRequestVariants, ResourceRqMap, WorkerResources, amount_from_float, as_f64)


def compute_gap_resources(rqv: ResourceRequestVariants, resources: WorkerResources) -> WorkerResources:
    used_ids = [e.resource_id for rq in rqv.variants for e in rq.entries]
    if not used_ids:
        return WorkerResources([])
    n_resources = max(used_ids) + 1
    gap_res = []
    # NB (reference quirk kept): the result vector is indexed by position in iter_pairs(), i.e. only
    # over the worker's NON-ZERO resources (gap.rs:110-145).
    for r_id, r_amount in resources.iter_pairs():
        lp = LpSolver()
        rows = [[] for _ in range(n_resources)]
        xs = []
        for rq in rqv.variants:
            a = rq.get_amount(r_id)
            if a is None:
                a = resources.get(r_id)
            xs.append(lp.add_nat_variable(as_f64(a)))
        for i, rq in enumerate(rqv.variants):
            for e in rq.entries:
                a = e.amount_or_none_if_all()
                if a is None:
                    a = resources.get(r_id)          # sic: outer r_id (gap.rs:128)
                rows[e.resource_id].append((xs[i], as_f64(a)))
        for idx, terms in enumerate(rows):
            lp.add_constraint(MAX, as_f64(resources.get(idx)), terms)
        sol = lp.solve()
        if sol is None:
            gap_res.append(0)
            continue
        v = sol[1]
        rounded = math.floor(v + 0.5) if v >= 0 else -math.floor(-v + 0.5)
        gap_res.append(r_amount - amount_from_float(float(rounded)))
    return WorkerResources(gap_res)


class GapCache:
    def __init__(self) -> None:
        self._cache: Dict[Tuple[int, Tuple[int, ...]], WorkerResources] = {}
        # memo of the whole (pure) function for workers without assigned tasks: the reference recomputes it
        # per (cut, blocker, worker) in ~a microsecond of Rust; in Python that loop would dominate the tick
        self._memo: Dict[Tuple[int, int, Tuple[int, ...]], int] = {}

    def get_gap(self, high_rq: int, low_rq: int, resources: WorkerResources,
                assigned: Iterable[Tuple[int, int]], rq_map: ResourceRqMap) -> int:
        assigned = list(assigned)
        mkey = None
        if not assigned:
            mkey = (high_rq, low_rq, resources.key())
            hit = self._memo.get(mkey)
            if hit is not None:
                return hit
        out = self._get_gap(high_rq, low_rq, resources, assigned, rq_map)
        if mkey is not None:
            self._memo[mkey] = out
        return out

    def _get_gap(self, high_rq: int, low_rq: int, resources: WorkerResources,
                 assigned: Iterable[Tuple[int, int]], rq_map: ResourceRqMap) -> int:
        h_rqv = rq_map.get(high_rq)
        if h_rqv.is_multi_node():
            return 0
        l_rqv = rq_map.get(low_rq)
        if l_rqv.is_multi_node():
            return 0
        h_rq = h_rqv.trivial_request()
        if h_rq is not None:
            if any(e.is_all() for e in h_rq.entries):
                return 0
            count = resources.task_max_count_for_request(h_rq)
            free = resources.clone()
            free.remove_multiple(h_rq, count)
        else:
            key = (high_rq, resources.key())
            cached = self._cache.get(key)
            if cached is None:
                cached = compute_gap_resources(h_rqv, resources)
                self._cache[key] = cached
            free = cached.clone()
        for rq_id, rv in assigned:
            if rq_id != high_rq:
                free.remove(rq_map.get(rq_id).variants[rv])
        return min((free.task_max_count_for_request(rq) for rq in l_rqv.variants), default=0)
