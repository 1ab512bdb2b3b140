"""Task batches and priority cuts, restated (TEST INFRASTRUCTURE — see oracle/__init__.py).

Follows hyperqueue/crates/tako/src/internal/scheduler/batches.rs:
  :8-9      BATCH_PRUNING_MAX_SIZE = 32, BATCH_PRUNING_FIXED_PREFIX = 4
  :11-40    PriorityCut {size, blockers[(rq, Some(size)|None)]}, TaskBatch {rq, cuts, size, limit,
            limit_reached, is_blocker}
  :42-181   create_task_batches: per-class limit, k-way merge of the per-class priority histograms in
            descending priority, cut emission when classes tie or the leading class changes
  :183-217  prune_progressive (quadratic spacing, first 4 kept)
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

BATCH_PRUNING_MAX_SIZE = 32
BATCH_PRUNING_FIXED_PREFIX = 4


@dataclass
class PriorityCut:
    size: int
    blockers: List[Tuple[int, Optional[int]]]


@dataclass
class TaskBatch:
    resource_rq_id: int
    limit: int
    cuts: List[PriorityCut] = field(default_factory=list)
    size: int = 0
    limit_reached: bool = False
    is_blocker: bool = False


def _round_half_away(x: float) -> int:
    """f64::round for non-negative x."""
    return int(math.floor(x + 0.5))


def prune_progressive(vec: list, prefix_size: int, size_limit: int) -> list:
    """batches.rs:183-217.  Returns the pruned list (the reference prunes in place by swapping)."""
    n = len(vec)
    if n <= size_limit:
        return vec
    remaining = size_limit - prefix_size
    pool = n - prefix_size
    keep = list(range(prefix_size))
    last = prefix_size - 1
    for i in range(remaining):
        t = i / (remaining - 1)
        idx = prefix_size + _round_half_away(t * t * (pool - 1))
        if idx <= last:
            idx = last + 1
        keep.append(idx)
        last = idx
    return [vec[i] for i in keep]


def _batch_limit(core, rqv, now: float, custom_workers) -> int:
    """batches.rs:62-91."""
    if rqv.is_multi_node():
        n_nodes = rqv.variants[0].n_nodes
        n_free = sum(1 for w in core.workers.values() if w.is_free())
        return n_free // n_nodes
    workers = custom_workers if custom_workers is not None else core.workers.values()
    limit = 0
    for w in workers:
        if not w.is_capable_to_run_rqv(rqv, now):
            continue
        runnable = w.free.task_max_count(rqv) if w.is_sn() else 0
        limit += runnable if runnable > 0 else 1       # every capable worker counts at least once
    return limit


def create_task_batches(core, now: float, custom_workers: Optional[Sequence] = None) -> List[TaskBatch]:
    queues = [q for q in core.task_queues if not q.is_empty()]
    if not queues:
        return []
    batches = [TaskBatch(q.resource_rq_id, _batch_limit(core, core.rq_map.get(q.resource_rq_id), now,
                                                         custom_workers)) for q in queues]
    streams = [q.iter_priority_sizes() for q in queues]
    heads: List[Optional[Tuple[int, int]]] = [next(s, None) for s in streams]

    def absorb(i: int) -> None:
        # shared tail of both branches (batches.rs:120-129 / :156-165)
        b = batches[i]
        b.size += heads[i][1]
        if b.size > b.limit:
            b.size = b.limit
            b.limit_reached = True
            heads[i] = None
        else:
            heads[i] = next(streams[i], None)

    leader: Optional[int] = None          # `unique` in the reference
    while True:
        live = [(h[0], i) for i, h in enumerate(heads) if h is not None]
        if not live:
            break
        top = max(p for p, _ in live)
        found = [i for p, i in live if p == top]
        if len(found) == 1 and leader == found[0]:
            absorb(found[0])
            continue
        for i in found:
            size_before = batches[i].size
            blockers = []
            for j, b in enumerate(batches):
                if j != i and (b.size > 0 or b.limit_reached):
                    b.is_blocker = True
                    blockers.append((b.resource_rq_id, None if b.limit_reached else b.size))
            if blockers:
                batches[i].cuts.append(PriorityCut(size_before, blockers))
        for i in found:
            absorb(i)
        leader = found[0] if len(found) == 1 else None

    out = []
    for b in batches:
        b.cuts = prune_progressive(b.cuts, BATCH_PRUNING_FIXED_PREFIX, BATCH_PRUNING_MAX_SIZE)
        if b.size > 0:
            out.append(b)
    return out
