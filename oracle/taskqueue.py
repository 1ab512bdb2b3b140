"""Ready-task queues per request class, restated (TEST INFRASTRUCTURE — see oracle/__init__.py).

Follows hyperqueue/crates/tako/src/internal/scheduler/taskqueue.rs:
  :26-72    TaskQueues (one TaskQueue per ResourceRqId; add_ready_task disposes lower-priority prefills)
  :114-119  TaskQueue {queue: BTreeMap<Reverse<Priority>, OneOrMoreTaskIds>, prefill: Option<(Priority, Set)>}
  :146-152  check_dispose_prefill
  :194-216  remove
  :237-253  top_priority / top_size_no_prefill
  :255-271  remove_prefilled / move_prefilled_task_to_ready
  :273-302  iter_priority_sizes (prefill merged into the histogram)
  :304-318  take_tasks_for_prefill
  :320-355  take_tasks
  :357-420  take_one / drain_prefill / take_from_entry

Order inside one priority level is ascending TaskId (BTreeSet::pop_first).
"""
from __future__ import annotations

from bisect import bisect_left, insort
from typing import Iterator, List, Optional, Tuple

from sortedcontainers import SortedDict


class _Level:
    """OneOrMoreTaskIds: an ordered set of task ids with cheap pop-smallest."""

    __slots__ = ("ids", "head")

    def __init__(self) -> None:
        self.ids: list = []
        self.head = 0

    def __len__(self) -> int:
        return len(self.ids) - self.head

    def add(self, t) -> None:
        if not self.ids or t > self.ids[-1]:
            self.ids.append(t)
        else:
            insort(self.ids, t, lo=self.head)

    def extend_sorted(self, ts: list) -> None:
        if self.head:
            del self.ids[: self.head]
            self.head = 0
        if self.ids and ts and ts[0] < self.ids[-1]:
            self.ids = sorted(self.ids + list(ts))
        else:
            self.ids.extend(ts)

    def remove(self, t) -> bool:
        i = bisect_left(self.ids, t, lo=self.head)
        if i < len(self.ids) and self.ids[i] == t:
            del self.ids[i]
            return True
        return False

    def contains(self, t) -> bool:
        i = bisect_left(self.ids, t, lo=self.head)
        return i < len(self.ids) and self.ids[i] == t

    def pop_first_n(self, n: int) -> list:
        k = min(n, len(self))
        out = self.ids[self.head: self.head + k]
        self.head += k
        return out


class TaskQueue:
    def __init__(self, resource_rq_id: int) -> None:
        self.resource_rq_id = resource_rq_id
        self.queue: SortedDict = SortedDict()          # key = -priority  (Reverse<Priority>)
        self.prefill: Optional[Tuple[int, set]] = None

    # -- maintenance ------------------------------------------------------------------------
    def check_dispose_prefill(self, priority: int, retracted: list) -> None:
        # taskqueue.rs:146-152
        if self.prefill is not None and self.prefill[0] < priority:
            p, ts = self.prefill
            self.prefill = None
            self.add_many(ts, p)
            retracted.extend(ts)

    def add(self, task_id, priority: int) -> None:
        # taskqueue.rs:154-172
        lvl = self.queue.get(-priority)
        if lvl is None:
            lvl = self.queue[-priority] = _Level()
        lvl.add(task_id)

    def add_many(self, task_ids, priority: int) -> None:
        # taskqueue.rs:174-192
        ts = sorted(task_ids)
        if not ts:
            return
        lvl = self.queue.get(-priority)
        if lvl is None:
            lvl = self.queue[-priority] = _Level()
        lvl.extend_sorted(ts)

    def remove(self, task_id, priority: int) -> None:
        # taskqueue.rs:194-216
        if self.prefill is not None and self.prefill[0] == priority and task_id in self.prefill[1]:
            self.prefill[1].remove(task_id)
            return
        lvl = self.queue.get(-priority)
        if lvl is not None:
            lvl.remove(task_id)
            if len(lvl) == 0:
                del self.queue[-priority]

    # -- queries ----------------------------------------------------------------------------
    def size(self) -> int:
        return sum(len(v) for v in self.queue.values())

    def is_empty(self) -> bool:
        return len(self.queue) == 0

    def top_priority(self) -> Optional[int]:
        if not self.queue:
            return None
        return -self.queue.peekitem(0)[0]

    def top_size_no_prefill(self) -> int:
        # taskqueue.rs:237-253
        if not self.queue:
            return 0
        negp, lvl = self.queue.peekitem(0)
        if self.prefill is not None and self.prefill[0] != -negp:
            return 0
        return len(lvl)

    def is_ready(self, task_id, priority: int) -> bool:
        lvl = self.queue.get(-priority)
        return lvl is not None and lvl.contains(task_id)

    def iter_priority_sizes(self) -> Iterator[Tuple[int, int]]:
        # taskqueue.rs:273-302
        items = [(-k, len(v)) for k, v in self.queue.items()]
        if self.prefill is None:
            return iter(items)
        pp, ps = self.prefill
        psize = len(ps)
        if items and items[0][0] == pp:
            return iter([(pp, items[0][1] + psize)] + items[1:])
        return iter([(pp, psize)] + items)

    # -- taking -----------------------------------------------------------------------------
    def _take_from_first_entry(self, count: int, result: list) -> int:
        # take_from_entry (taskqueue.rs:395-420)
        negp, lvl = self.queue.peekitem(0)
        got = lvl.pop_first_n(count)
        result.extend(got)
        if len(lvl) == 0:
            del self.queue[negp]
        return count - len(got)

    def _drain_prefill(self, count: int, result: list) -> int:
        # drain_prefill (taskqueue.rs:377-393).  The reference iterates a hash set (arbitrary
        # order); we take ascending ids, which is one admissible order.
        if self.prefill is None:
            return count
        _, tasks = self.prefill
        while count > 0 and tasks:
            t = min(tasks)
            tasks.remove(t)
            result.append(t)
            count -= 1
        if not tasks:
            self.prefill = None
        return count

    def take_tasks_for_prefill(self, count: int) -> list:
        # taskqueue.rs:304-318
        negp, _ = self.queue.peekitem(0)
        priority = -negp
        result: list = []
        self._take_from_first_entry(count, result)
        if self.prefill is not None:
            assert self.prefill[0] == priority
            self.prefill[1].update(result)
        else:
            self.prefill = (priority, set(result))
        return result

    def take_tasks(self, count: int) -> list:
        # taskqueue.rs:320-355
        result: list = []
        if self.prefill is None:
            while count > 0:
                count = self._take_from_first_entry(count, result)
            return result
        prefill_priority = self.prefill[0]
        if self.top_priority() == prefill_priority:
            if count > 0:
                count = self._take_from_first_entry(count, result)
            count = self._drain_prefill(count, result)
        else:
            count = self._drain_prefill(count, result)
        while count > 0:
            count = self._take_from_first_entry(count, result)
        return result

    def take_one(self):
        # taskqueue.rs:357-375
        if not self.queue:
            return None
        out: list = []
        self._take_from_first_entry(1, out)
        return out[0]

    def remove_prefilled(self, task_id) -> None:
        # taskqueue.rs:255-261
        self.prefill[1].remove(task_id)
        if not self.prefill[1]:
            self.prefill = None

    def move_prefilled_task_to_ready(self, task_id) -> None:
        # taskqueue.rs:263-271
        p = self.prefill[0]
        self.remove_prefilled(task_id)
        self.add(task_id, p)


class TaskQueues:
    def __init__(self) -> None:
        self.queues: List[TaskQueue] = []

    def add_task_queue(self) -> None:
        self.queues.append(TaskQueue(len(self.queues)))

    def add_ready_task(self, task_id, rq_id: int, priority: int, retracted: list) -> None:
        # taskqueue.rs:37-43
        for q in self.queues:
            q.check_dispose_prefill(priority, retracted)
        self.queues[rq_id].add(task_id, priority)

    def add_ready_tasks_bulk(self, task_ids, rq_id: int, priority: int) -> None:
        """Bulk form of add_ready_task for the benchmark harness (no prefills outstanding)."""
        self.queues[rq_id].add_many(task_ids, priority)

    def get(self, rq_id: int) -> TaskQueue:
        return self.queues[rq_id]

    def __iter__(self):
        return iter(self.queues)

    def top_priority(self) -> int:
        # taskqueue.rs:62-68
        tops = [q.top_priority() for q in self.queues]
        tops = [t for t in tops if t is not None]
        return max(tops) if tops else 0
