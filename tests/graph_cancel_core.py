"""Cancelling and failing tasks in the server core, restated (TEST INFRASTRUCTURE, on top of oracle/core.py).

Follows (paths relative to hyperqueue/crates/tako/src/internal/):
  server/reactor.rs:696-770   on_cancel_tasks (per-state host updates, CancelTasks messages, batched removal)
  server/reactor.rs:596-694   task_failed (resources of the failing task, its transitive consumers, removal)
  server/reactor.rs:582-594   try_remove_redirection
  server/task.rs:235-248      Task::collect_recursive_consumers
  server/core.rs:216-243      Core::remove_task / remove_tasks_batched
For the task states oracle/core.py models: waiting, assigned, running, prefilled and retracting.  Multi-node tasks and the
client's answer to on_task_error are out of scope.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Set

from oracle.core import Core


class CancelCore(Core):
    def collect_recursive_consumers(self, task_id, out: Set) -> None:
        # task.rs:235-248
        consumers = self.tasks[task_id].consumers
        out.update(consumers)
        stack = list(consumers)
        while stack:
            for c in self.tasks[stack.pop()].consumers:
                if c not in out:
                    out.add(c)
                    stack.append(c)

    def remove_task(self, task_id) -> str:
        # core.rs:213-233: a waiting task leaves its ready queue and its producers' consumer lists
        task = self.tasks.pop(task_id)
        if task.state == "waiting":
            self.task_queues.get(task.rq_id).remove(task_id, task.priority)
            if task.unfinished_deps > 0:
                for d in task.deps:
                    p = self.tasks.get(d)
                    if p is not None:
                        p.consumers.remove(task_id)
        return task.state

    def _try_remove_redirection(self, task) -> None:
        # reactor.rs:582-594: the redirect target's resources come back
        red = self.scheduler_state.redirects.pop(task.id, None)
        if red is not None:
            w, rv = red
            self.workers[w].remove_sn_task(task.id, self.rq_map.get(task.rq_id).variants[rv])

    def _leave_worker(self, task) -> None:
        """The per-state worker bookkeeping both calls share (reactor.rs:612-659, 720-760)."""
        if task.state in ("assigned", "running"):
            self.workers[task.worker].remove_sn_task(task.id, self.rq_map.get(task.rq_id).variants[task.rv])
        elif task.state == "prefilled":
            self.task_queues.get(task.rq_id).remove_prefilled(task.id)
            self.workers[task.worker].prefilled_tasks.discard(task.id)
        elif task.state == "retracting":
            self._try_remove_redirection(task)

    def on_cancel_tasks(self, task_ids) -> Dict[int, List]:
        """reactor.rs:696-770.  Returns the CancelTasks messages (worker id -> tasks in the order they were named); the
        set of removed tasks is left in self.last_removed."""
        to_unregister: Set = set()
        running_ids: Dict[int, List] = {}
        for t in task_ids:
            task = self.tasks.get(t)
            if task is None:
                continue                                   # "Task is not here"
            to_unregister.add(t)
            self.collect_recursive_consumers(t, to_unregister)
            if task.state != "waiting":
                self._leave_worker(task)
                running_ids.setdefault(task.worker, []).append(t)
        for t in to_unregister:
            self.remove_task(t)
        self.last_removed = to_unregister
        return running_ids

    def task_failed(self, worker_id: Optional[int], task_id) -> Optional[List]:
        """reactor.rs:596-694: returns the failed task's transitive consumers, ascending (the list handed to
        on_task_error), or None for an unknown task."""
        task = self.tasks.get(task_id)
        if task is None:
            return None                                    # "Unknown task failed"
        if worker_id is not None:
            assert task.worker == worker_id
            self._leave_worker(task)
        else:
            assert task.state == "waiting"
        s: Set = set()
        self.collect_recursive_consumers(task_id, s)
        for c in s:
            assert self.remove_task(c) == "waiting"
        self.remove_task(task_id)
        return sorted(s)
