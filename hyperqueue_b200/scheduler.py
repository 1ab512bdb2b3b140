"""Host-side mirror of tako's scheduler seam over the C ABI (include/hqsched.h).

What the Rust shim of INTEGRATION.md does inside `run_scheduling_inner`
(hyperqueue/crates/tako/src/internal/scheduler/main.rs:40-46) is done here in Python so that the
parity tests and the benchmark read like the reference's own tests:

  reference (Rust)                                          here
  --------------------------------------------------------  -----------------------------------------
  get_or_create_resource_rq_id   control.rs:222-227         GpuScheduler.get_or_create_resource_rq_id
  on_new_worker                  reactor.rs:20-32           GpuScheduler.new_worker
  Worker::block_request          worker.rs:336-344          GpuScheduler.block_request / unblock_request
  TaskQueues::add_ready_task     taskqueue.rs:37-43         GpuScheduler.add_ready_tasks
  TaskQueue::remove              taskqueue.rs:194-216       GpuScheduler.remove_ready_tasks
  run_scheduling_inner           main.rs:40-46              GpuScheduler.run_scheduling  -> WorkerTaskMapping
  WorkerTaskMapping::send_messages  mapping.rs:255-288      GpuScheduler.run_scheduling_grouped -> GroupedTaskMapping
  Worker::insert_sn_task         worker.rs:188-196          (free vectors come back from the device)
  task_finished / remove_sn_task reactor.rs:500-580         GpuScheduler.tasks_finished
  on_new_tasks with dependencies reactor.rs:188-220         GpuScheduler.submit_tasks
  task_finished in a task graph  reactor.rs:500-580         GpuScheduler.graph_tasks_finished
  on_cancel_tasks / task_failed  reactor.rs:596-770         GpuScheduler.graph_cancel_tasks

Device memory, streams and the kernels live in libhqsched_b200.so; this module only marshals numpy
arrays.  No CPU fallback exists: without the library or a CUDA device every call raises.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np

from . import _lib as L

FRACTIONS_PER_UNIT = 10_000


def priority_from_user(user_priority) -> np.ndarray:
    """Priority::from_user_priority (common/priority.rs:43-48), vectorised."""
    p = np.asarray(user_priority, dtype=np.int64)
    return ((((p & 0xFFFFFFFF) ^ 0x8000_0000).astype(np.uint64)) << np.uint64(32)).astype(np.uint64)


@dataclass(frozen=True)
class RequestVariant:
    """One ResourceRequest (common/resources/request.rs:136-167) in dense form."""
    amounts: Tuple[Tuple[int, int], ...]          # (resource id, fractions), amount policies
    all_resources: Tuple[int, ...] = ()           # resource ids requested with policy `All`
    weight: float = 1.0
    min_time_s: float = 0.0

    @staticmethod
    def of(amounts: Dict[int, int], all_resources: Iterable[int] = (), weight: float = 1.0,
           min_time_s: float = 0.0) -> "RequestVariant":
        return RequestVariant(tuple(sorted((int(r), int(a)) for r, a in amounts.items())),
                              tuple(sorted(int(r) for r in all_resources)), float(weight), float(min_time_s))


@dataclass
class WorkerTaskMapping:
    """What create_task_mapping returns (mapping.rs:9-21), as arrays."""
    assignments: np.ndarray                       # L.assignment_dtype; `worker` = index into worker_ids
    worker_ids: np.ndarray
    free_after: np.ndarray                        # [W][R] u64

    retract_from: Optional[np.ndarray] = None     # for kind == 2 records: index of the worker the task was prefilled on

    def n_assigned(self) -> int:
        """Assignments of this tick: plain (kind 0) and redirected ones (kind 2); prefill records are not assignments."""
        return int(np.count_nonzero(self.assignments["kind"] != 1))

    def n_prefilled(self) -> int:
        return int(np.count_nonzero(self.assignments["kind"] == 1))

    def messages(self) -> Dict[int, Dict[str, list]]:
        """WorkerTaskMapping::send_messages (mapping.rs:255-288) as data: worker_id -> {"retracts": [task handles] (one
        RetractTasks message, sent first), "compute": [(task handle, variant or None)] (the ComputeTasks list: prefills
        first with variant None, then the assigned tasks in priority-descending order; ComputeTasksBuilder splits it at
        32 MiB of serialised size, server/task.rs:315-414)}.  Redirected tasks (kind 2) are NOT sent to their new worker
        here: that happens when the old worker answers the retract (GpuScheduler.on_retract_response)."""
        out: Dict[int, Dict[str, list]] = {}
        a = self.assignments
        def slot(widx):
            return out.setdefault(int(self.worker_ids[widx]), {"retracts": [], "compute": []})
        pf = a[a["kind"] == 1]
        for t, w in zip(pf["task"].tolist(), pf["worker"].tolist()):
            slot(w)["compute"].append((t, None))
        for t, w, v, k in zip(a["task"].tolist(), a["worker"].tolist(), a["variant"].tolist(), a["kind"].tolist()):
            if k == 0:
                slot(w)["compute"].append((t, v))          # emission order is already priority-descending per worker
        if self.retract_from is not None:
            r2 = a[a["kind"] == 2]
            for t, ow in zip(r2["task"].tolist(), self.retract_from.tolist()):
                slot(ow)["retracts"].append(t)
        return out

    def per_worker(self) -> Dict[int, List[Tuple[int, int]]]:
        """worker_id -> [(task handle, variant)] in emission order (priority descending)."""
        out: Dict[int, List[Tuple[int, int]]] = {}
        a = self.assignments
        for t, w, v, k in zip(a["task"].tolist(), a["worker"].tolist(), a["variant"].tolist(), a["kind"].tolist()):
            if k != 1:
                out.setdefault(int(self.worker_ids[w]), []).append((t, v))
        return out


@dataclass
class GroupedTaskMapping:
    """The same tick result as WorkerTaskMapping with the records grouped by worker on the device (hqs_tick_fetch_grouped):
    with W = len(worker_ids), worker w's prefill records are records[worker_off[2w]:worker_off[2w+1]], its assignments
    records[worker_off[2w+1]:worker_off[2w+2]], both in emission order, and the redirect records (kind 2) are the flat tail
    records[worker_off[2W]:worker_off[2W+1]] in emission order.  The per-worker lists are slices."""
    records: np.ndarray                           # L.assignment_dtype; `worker` = index into worker_ids
    worker_off: np.ndarray                        # [2W + 2] u32
    worker_ids: np.ndarray
    free_after: np.ndarray                        # [W][R] u64
    retract_from: Optional[np.ndarray] = None     # for the tail's records: index of the worker the task was prefilled on

    def redirects(self) -> np.ndarray:
        nw = self.worker_ids.shape[0]
        return self.records[int(self.worker_off[2 * nw]): int(self.worker_off[2 * nw + 1])]

    def n_assigned(self) -> int:
        return int(self.records.shape[0]) - self.n_prefilled()

    def n_prefilled(self) -> int:
        off = self.worker_off.astype(np.int64)
        return int((off[1:-1:2] - off[0:-2:2]).sum())

    def messages(self) -> Dict[int, Dict[str, list]]:
        """What WorkerTaskMapping.messages() returns for the same tick."""
        out: Dict[int, Dict[str, list]] = {}
        off = self.worker_off.tolist()
        task, variant = self.records["task"], self.records["variant"]
        for w, wid in enumerate(self.worker_ids.tolist()):
            p0, a0, a1 = off[2 * w], off[2 * w + 1], off[2 * w + 2]
            if a1 > p0:
                out[wid] = {"retracts": [], "compute": [(t, None) for t in task[p0:a0].tolist()]
                            + list(zip(task[a0:a1].tolist(), variant[a0:a1].tolist()))}
        if self.retract_from is not None:
            for t, ow in zip(self.redirects()["task"].tolist(), self.retract_from.tolist()):
                out.setdefault(int(self.worker_ids[ow]), {"retracts": [], "compute": []})["retracts"].append(t)
        return out

    def per_worker(self) -> Dict[int, List[Tuple[int, int]]]:
        """worker_id -> [(task handle, variant)]: the worker's assignments in emission order, which is what
        WorkerTaskMapping.per_worker() returns for a tick without redirect records.  Tasks redirected to the worker follow
        its assignments here (the grouped layout keeps them in the tail, not at their place in the emission order)."""
        out: Dict[int, List[Tuple[int, int]]] = {}
        off = self.worker_off.tolist()
        task, variant = self.records["task"], self.records["variant"]
        for w, wid in enumerate(self.worker_ids.tolist()):
            a0, a1 = off[2 * w + 1], off[2 * w + 2]
            if a1 > a0:
                out[wid] = list(zip(task[a0:a1].tolist(), variant[a0:a1].tolist()))
        red = self.redirects()
        for t, w, v in zip(red["task"].tolist(), red["worker"].tolist(), red["variant"].tolist()):
            out.setdefault(int(self.worker_ids[w]), []).append((t, v))
        return out


def apply_tick_records(s, a: np.ndarray) -> Optional[np.ndarray]:
    """The host's bookkeeping after a tick, on the scheduler `s` whose task handles the records `a` carry (a GpuScheduler,
    or the per-rank one of a sharded tick): where each assigned task runs, the redirects of kind-2 records and the new
    prefills of kind-1 records.  Returns, for the kind-2 records in order, the index of the worker each was prefilled on
    (None if there are none)."""
    retract_from = None
    if a.size:
        asg = a[a["kind"] != 1]
        s._task_worker[asg["task"]] = asg["worker"]
        s._task_variant[asg["task"]] = asg["variant"]
        red = a[a["kind"] == 2]
        if red.size:
            # a prefilled task was assigned: RetractTasks to the worker that holds it, redirect to the new one; the
            # new worker's resources are already taken (mapping.rs:49-101)
            old = s._pf_worker[red["task"]].copy()
            retract_from = np.searchsorted(s.worker_ids, old)
            for t, ow, nwk, v in zip(red["task"].tolist(), old.tolist(), red["worker"].tolist(), red["variant"].tolist()):
                s.redirects[t] = (int(s.worker_ids[nwk]), int(v))
                s._retracting_from[t] = int(ow)
            s._pf_worker[red["task"]] = -1
        pf = a[a["kind"] == 1]
        if pf.size:
            s._pf_worker[pf["task"]] = s.worker_ids[pf["worker"]]
    return retract_from


def return_resources(s, h: np.ndarray) -> None:
    """The host's bookkeeping of task_finished (Worker::remove_sn_task -> WorkerResources::add, workerload.rs:194-202) on
    the scheduler `s` whose task handles `h` are (a GpuScheduler, or the owner rank's one of a sharded ready set): each
    task's amounts go back to the worker it ran on, an `All` resource gets the worker's total back, and the tasks are no
    longer assigned.  An unlimited amount (HQS_AMOUNT_MAX) is never taken by a tick, so nothing comes back to it."""
    wi = s._task_worker[h]
    cl = s._task_class[h]
    va = s._task_variant[h]
    add = np.zeros_like(s.free)
    np.add.at(add, wi, s._amount_tab[cl, va])                 # [n][R] summed per worker
    s.free = np.where(s.free == L.HQS_AMOUNT_MAX, s.free, s.free + add)
    allm = s._all_tab[cl, va]                                 # [n][R] bool
    if allm.any():
        ws, rs = np.nonzero(allm)
        s.free[wi[ws], rs] = s.total[wi[ws], rs]
    s._task_worker[h] = -1


def cancel_bookkeeping(s, h: np.ndarray, gone: np.ndarray) -> Dict[int, List[int]]:
    """The host's bookkeeping of on_cancel_tasks on the scheduler `s` whose handles `h` (named) and `gone` (what left the
    table) are: a named task that is assigned gives its resources back, a prefilled one is no longer held, a retracting one
    loses its redirect and the resources taken on the redirect target come back.  Returns worker id -> the named tasks to
    cancel there, in the order they were named (the CancelTasks messages)."""
    if h.size:
        s._grow_tasks(int(h.max()) + 1)
    left = set(gone.tolist())
    messages: Dict[int, List[int]] = {}
    assigned = []
    for t in dict.fromkeys(h.tolist()):
        if t not in left:
            continue                                     # "Task is not here"
        if t in s._retracting_from:
            messages.setdefault(s._retracting_from.pop(t), []).append(t)
            s.redirects.pop(t, None)
            assigned.append(t)                           # try_remove_redirection: the target's resources come back
        elif s._task_worker[t] >= 0:
            messages.setdefault(int(s.worker_ids[s._task_worker[t]]), []).append(t)
            assigned.append(t)
        elif s._pf_worker[t] >= 0:
            messages.setdefault(int(s._pf_worker[t]), []).append(t)
            s._pf_worker[t] = -1
    if assigned:
        return_resources(s, np.array(assigned, dtype=np.int64))
    return messages


def tracked_handles(s, n: int) -> np.ndarray:
    """The handles below n that the scheduler `s` still tracks on the host, whether or not their task is in the device table:
    assigned to a worker, prefilled, or with a pending redirect or retract.  A handle compaction must keep them (int64, may
    repeat)."""
    tracked = np.zeros(0, dtype=np.int64)
    if n:
        m = min(n, s._task_worker.shape[0])
        tracked = np.nonzero((s._task_worker[:m] >= 0) | (s._pf_worker[:m] >= 0))[0]
    extra = list(s.redirects.keys()) + list(s._retracting_from.keys())
    return np.concatenate([tracked, np.asarray(extra, dtype=np.int64)])


def renumber_host_mirror(s, kept: np.ndarray) -> None:
    """After a handle compaction: the scheduler `s`'s handle kept[i] (ascending, int64) is now handle i.  The per-handle host
    arrays and the redirect and retract maps follow; the slots past the survivors read as never used.  The arrays must
    already hold every kept handle."""
    def remap(a: np.ndarray, fill) -> np.ndarray:
        out = np.full_like(a, fill)
        out[: kept.size] = a[kept]
        return out

    s._task_class = remap(s._task_class, 0)
    s._task_worker = remap(s._task_worker, -1)
    s._task_variant = remap(s._task_variant, 0)
    s._task_prio = remap(s._task_prio, 0)
    s._pf_worker = remap(s._pf_worker, -1)

    def new_of(t: int) -> int:
        return int(np.searchsorted(kept, t))

    s.redirects = {new_of(t): v for t, v in s.redirects.items()}
    s._retracting_from = {new_of(t): v for t, v in s._retracting_from.items()}


def query_workers(worker_totals: np.ndarray, remaining_s: Optional[np.ndarray] = None,
                  min_utilization: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray]:
    """The fake-worker array of a what-if query (new_worker_query): worker ids 0..n-1, time limits in seconds (inf = none)
    as milliseconds, min_utilization as given.  Returns (workers [L.worker_dtype], totals [W][R] u64); the totals are also
    the free vectors."""
    tot = np.ascontiguousarray(worker_totals, dtype=np.uint64)
    nw = tot.shape[0]
    w = np.zeros(nw, dtype=L.worker_dtype)
    w["worker_id"] = np.arange(nw, dtype=np.uint32)
    rem = np.full(nw, L.HQS_TIME_INF, dtype=np.uint64)
    if remaining_s is not None:
        r = np.asarray(remaining_s, dtype=np.float64)
        finite = ~np.isinf(r)
        rem[finite] = (np.maximum(r[finite], 0.0) * 1000.0).astype(np.uint64)
    w["remaining_time_ms"] = rem
    if min_utilization is not None:
        w["min_utilization"] = np.asarray(min_utilization, dtype=np.float32)
    return w, tot


class GpuScheduler:
    def __init__(self, n_resources: int, device: int = 0, flags: int = 0) -> None:
        self._lib = L.load_library()
        self.R = int(n_resources)
        self._ctx = C.c_void_p()
        rc = self._lib.hqs_create(C.byref(self._ctx), device, self.R, int(flags))
        if rc:
            raise L.HqsError(rc, (self._lib.hqs_last_error(None) or b"").decode())
        self._rq_ids: Dict[Tuple[RequestVariant, ...], int] = {}
        self._classes: List[Tuple[RequestVariant, ...]] = []
        self._classes_dirty = False
        # dense per-class amount table for resource return: [Q][V][R] and an `All` mask [Q][V][R]
        self._amount_tab = np.zeros((0, L.HQS_MAX_VARIANTS, self.R), dtype=np.uint64)
        self._all_tab = np.zeros((0, L.HQS_MAX_VARIANTS, self.R), dtype=bool)
        # workers, kept sorted by id
        self.worker_ids = np.zeros(0, dtype=np.uint32)
        self.total = np.zeros((0, self.R), dtype=np.uint64)
        self.free = np.zeros((0, self.R), dtype=np.uint64)
        self.termination = np.zeros(0, dtype=np.float64)      # absolute seconds, inf = none
        self.min_utilization = np.zeros(0, dtype=np.float32)
        self._blocked: Dict[int, set] = {}
        # per-task host mirror (Task.resource_rq_id / TaskRuntimeState::Assigned{worker_id, rv_id})
        self._task_class = np.zeros(0, dtype=np.uint32)
        self._task_worker = np.zeros(0, dtype=np.int64)
        self._task_variant = np.zeros(0, dtype=np.uint8)
        self._task_prio = np.zeros(0, dtype=np.uint64)
        self._out = np.zeros(1024, dtype=L.assignment_dtype)
        # proactive filling: Worker::prefilled_tasks / SchedulerState::redirects (scheduler/state.rs:23-28), host side
        self._prefill = (0, 0)
        self._pf_worker = np.zeros(0, dtype=np.int64)     # per task: worker ID it is prefilled on, -1 = none
        self.redirects: Dict[int, Tuple[int, int]] = {}   # retracting task -> (target worker id, variant)
        self._retracting_from: Dict[int, int] = {}        # retracting task -> worker id it is being retracted from

    # ------------------------------------------------------------------------------------------
    def close(self) -> None:
        if getattr(self, "_ctx", None) is not None and self._ctx.value:
            self._lib.hqs_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self) -> None:
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int) -> None:
        if rc:
            raise L.HqsError(rc, (self._lib.hqs_last_error(self._ctx) or b"").decode())

    # classes ----------------------------------------------------------------------------------
    def get_or_create_resource_rq_id(self, variants: Sequence[RequestVariant]) -> int:
        key = tuple(variants)
        rid = self._rq_ids.get(key)
        if rid is None:
            if not 1 <= len(key) <= L.HQS_MAX_VARIANTS:
                raise ValueError("1..%d variants per class" % L.HQS_MAX_VARIANTS)
            rid = len(self._classes)
            self._rq_ids[key] = rid
            self._classes.append(key)
            self._classes_dirty = True
        return rid

    @property
    def n_classes(self) -> int:
        return len(self._classes)

    def _sync_classes(self) -> None:
        if not self._classes_dirty:
            return
        q = len(self._classes)
        arr = (L.hqs_class * q)()
        self._amount_tab = np.zeros((q, L.HQS_MAX_VARIANTS, self.R), dtype=np.uint64)
        self._all_tab = np.zeros((q, L.HQS_MAX_VARIANTS, self.R), dtype=bool)
        for c, variants in enumerate(self._classes):
            arr[c].n_variants = len(variants)
            arr[c].n_nodes = 0
            for v, rv in enumerate(variants):
                hv = arr[c].variants[v]
                for r, a in rv.amounts:
                    if a <= 0:
                        raise ValueError("Zero resources cannot be requested")   # request.rs:24-32
                    hv.amount[r] = a
                    self._amount_tab[c, v, r] = a
                mask = 0
                for r in rv.all_resources:
                    mask |= 1 << r
                    self._all_tab[c, v, r] = True
                hv.all_mask = mask
                hv.weight = int(np.round(np.float32(rv.weight) * np.float32(10_000)))
                hv.min_time_ms = int(round(rv.min_time_s * 1000.0))
        self._check(self._lib.hqs_classes_set(self._ctx, q, arr))
        self._classes_dirty = False

    # workers ----------------------------------------------------------------------------------
    def new_worker(self, worker_id: int, resources: Sequence[int], termination_time: Optional[float] = None,
                   min_utilization: float = 0.0, free: Optional[Sequence[int]] = None) -> None:
        if worker_id in self.worker_ids:
            raise ValueError(f"worker {worker_id} exists")
        tot = np.zeros(self.R, dtype=np.uint64)
        tot[: len(resources)] = np.asarray(resources, dtype=np.uint64)
        fr = tot.copy() if free is None else np.asarray(list(free) + [0] * (self.R - len(free)), dtype=np.uint64)
        pos = int(np.searchsorted(self.worker_ids, worker_id))
        self.worker_ids = np.insert(self.worker_ids, pos, worker_id).astype(np.uint32)
        self.total = np.insert(self.total, pos, tot, axis=0)
        self.free = np.insert(self.free, pos, fr, axis=0)
        self.termination = np.insert(self.termination, pos, np.inf if termination_time is None else termination_time)
        self.min_utilization = np.insert(self.min_utilization, pos, min_utilization).astype(np.float32)

    def new_workers_bulk(self, worker_ids: np.ndarray, total: np.ndarray, free: Optional[np.ndarray] = None) -> None:
        order = np.argsort(worker_ids)
        self.worker_ids = np.asarray(worker_ids, dtype=np.uint32)[order]
        self.total = np.ascontiguousarray(np.asarray(total, dtype=np.uint64)[order])
        self.free = self.total.copy() if free is None else np.ascontiguousarray(np.asarray(free, dtype=np.uint64)[order])
        self.termination = np.full(len(order), np.inf)
        self.min_utilization = np.zeros(len(order), dtype=np.float32)

    def block_request(self, worker_id: int, rq_id: int, variant: int) -> None:
        self._blocked.setdefault(worker_id, set()).add((rq_id, variant))

    def unblock_request(self, worker_id: int, rq_id: int, variant: int) -> None:
        self._blocked.get(worker_id, set()).discard((rq_id, variant))

    def set_blocked_mask(self, mask_wcv: Optional[np.ndarray]) -> None:
        """Bulk form: bool [W][Q][HQS_MAX_VARIANTS] over the sorted workers, or None."""
        self._blocked_bulk = None if mask_wcv is None else np.packbits(
            np.asarray(mask_wcv, dtype=bool), axis=2, bitorder="little")[:, :, 0].copy()

    # ready set ----------------------------------------------------------------------------------
    def _grow_tasks(self, n: int) -> None:
        if n > self._task_class.shape[0]:
            m = max(n, 2 * self._task_class.shape[0], 1024)
            self._task_class = np.concatenate([self._task_class, np.zeros(m - self._task_class.shape[0], np.uint32)])
            self._task_worker = np.concatenate([self._task_worker, np.full(m - self._task_worker.shape[0], -1, np.int64)])
            self._task_variant = np.concatenate([self._task_variant, np.zeros(m - self._task_variant.shape[0], np.uint8)])
            self._task_prio = np.concatenate([self._task_prio, np.zeros(m - self._task_prio.shape[0], np.uint64)])
            self._pf_worker = np.concatenate([self._pf_worker, np.full(m - self._pf_worker.shape[0], -1, np.int64)])

    def add_ready_tasks(self, handles, rq_ids, priorities) -> None:
        h = np.ascontiguousarray(handles, dtype=np.uint32)
        c = np.ascontiguousarray(rq_ids, dtype=np.uint32)
        p = np.ascontiguousarray(priorities, dtype=np.uint64)
        if not (h.shape == c.shape == p.shape):
            raise ValueError("shape mismatch")
        if h.size == 0:
            return
        self._sync_classes()
        self._grow_tasks(int(h.max()) + 1)
        self._task_class[h] = c
        self._task_prio[h] = p
        if h.size > 1 and int(h[-1]) - int(h[0]) == h.size - 1 and (np.diff(h.astype(np.int64)) == 1).all():
            # a task array: consecutive handles, no handle array crosses PCIe
            self._check(self._lib.hqs_ready_push_range(self._ctx, int(h[0]), h.size, L.ptr(c), L.ptr(p)))
        else:
            self._check(self._lib.hqs_ready_push(self._ctx, h.size, L.ptr(h), L.ptr(c), L.ptr(p)))

    def remove_ready_tasks(self, handles) -> None:
        h = np.ascontiguousarray(handles, dtype=np.uint32)
        if h.size:
            self._check(self._lib.hqs_ready_remove(self._ctx, h.size, L.ptr(h)))

    def load_dag(self, rq_ids, priorities, n_deps, cons_off, cons) -> None:
        c = np.ascontiguousarray(rq_ids, dtype=np.uint32)
        p = np.ascontiguousarray(priorities, dtype=np.uint64)
        d = np.ascontiguousarray(n_deps, dtype=np.uint32)
        co = np.ascontiguousarray(cons_off, dtype=np.uint32)
        cs = np.ascontiguousarray(cons, dtype=np.uint32)
        self._sync_classes()
        self._grow_tasks(c.size)
        self._task_class[: c.size] = c
        self._task_prio[: c.size] = p
        self._check(self._lib.hqs_dag_load(self._ctx, c.size, L.ptr(c), L.ptr(p), L.ptr(d), L.ptr(co),
                                           L.ptr(cs) if cs.size else None))

    # the tick -----------------------------------------------------------------------------------
    def _worker_structs(self, now: float) -> np.ndarray:
        w = np.zeros(self.worker_ids.shape[0], dtype=L.worker_dtype)
        w["worker_id"] = self.worker_ids
        finite = ~np.isinf(self.termination)
        rem = np.full(self.termination.shape[0], L.HQS_TIME_INF, dtype=np.uint64)
        rem[finite] = (np.maximum(self.termination[finite] - now, 0.0) * 1000.0).astype(np.uint64)
        w["remaining_time_ms"] = rem
        w["min_utilization"] = self.min_utilization
        return w

    def _blocked_bytes(self) -> Optional[np.ndarray]:
        bulk = getattr(self, "_blocked_bulk", None)
        if bulk is not None:
            return np.ascontiguousarray(bulk, dtype=np.uint8)
        if not any(self._blocked.values()):
            return None
        q = len(self._classes)
        b = np.zeros((self.worker_ids.shape[0], q), dtype=np.uint8)
        for wid, pairs in self._blocked.items():
            pos = int(np.searchsorted(self.worker_ids, wid))
            if pos < self.worker_ids.shape[0] and self.worker_ids[pos] == wid:
                for rq, v in pairs:
                    if rq < q:
                        b[pos, rq] |= np.uint8(1 << v)
        return b

    def run_scheduling(self, now: float = 0.0, out_cap: Optional[int] = None) -> WorkerTaskMapping:
        """run_scheduling_inner: one tick over the device-resident ready set.  Assigned tasks leave the
        ready set and the host free vectors are replaced by the post-tick vectors."""
        self._sync_classes()
        w = self._worker_structs(now)
        nw = w.shape[0]
        if out_cap is None:
            out_cap = max(int(self._lib_stats().n_handles), 1)
        if self._out.shape[0] < out_cap:
            self._out = np.zeros(out_cap, dtype=L.assignment_dtype)
        blocked = self._blocked_bytes()
        free = np.ascontiguousarray(self.free)
        total = np.ascontiguousarray(self.total)
        free_after = np.zeros_like(free)
        n = C.c_uint32(0)
        if self._prefill[1] > 0:
            self._check(self._lib.hqs_prefill_state(self._ctx, nw, L.ptr(self.prefill_mask())))
        self._check(self._lib.hqs_tick(self._ctx, nw, L.ptr(w), L.ptr(free), L.ptr(total),
                                       L.ptr(blocked) if blocked is not None else None, out_cap,
                                       L.ptr(self._out), C.byref(n), L.ptr(free_after)))
        a = self._out[: n.value].copy()
        # WorkerConfiguration::min_utilization (solver.rs:154-156, 479-518) is enforced inside the tick kernel: a worker
        # that would receive less than its minimum is taken out of the solve, which then starts over
        self.free = free_after
        retract_from = apply_tick_records(self, a)
        return WorkerTaskMapping(a, self.worker_ids.copy(), free_after, retract_from)

    def run_scheduling_grouped(self, now: float = 0.0, out_cap: Optional[int] = None) -> GroupedTaskMapping:
        """run_scheduling with the records grouped by worker on the device (hqs_tick_grouped): the same tick, the same
        bookkeeping, and per-worker message lists that are slices of one array."""
        self._sync_classes()
        w = self._worker_structs(now)
        nw = w.shape[0]
        if out_cap is None:
            out_cap = max(int(self._lib_stats().n_handles), 1)
        if self._out.shape[0] < out_cap:
            self._out = np.zeros(out_cap, dtype=L.assignment_dtype)
        blocked = self._blocked_bytes()
        free = np.ascontiguousarray(self.free)
        total = np.ascontiguousarray(self.total)
        free_after = np.zeros_like(free)
        off = np.zeros(2 * nw + 2, dtype=np.uint32)
        n = C.c_uint32(0)
        if self._prefill[1] > 0:
            self._check(self._lib.hqs_prefill_state(self._ctx, nw, L.ptr(self.prefill_mask())))
        self._check(self._lib.hqs_tick_grouped(self._ctx, nw, L.ptr(w), L.ptr(free), L.ptr(total),
                                               L.ptr(blocked) if blocked is not None else None, out_cap,
                                               L.ptr(self._out), C.byref(n), off.size, L.ptr(off), L.ptr(free_after)))
        a = self._out[: n.value].copy()
        self.free = free_after
        retract_from = apply_tick_records(self, a)      # kind-2 records keep their relative order in the grouped array
        return GroupedTaskMapping(a, off, self.worker_ids.copy(), free_after, retract_from)

    def prefill_mask(self) -> np.ndarray:
        """"Worker w holds a prefilled task of class c" (Worker::prefilled_tasks) over this scheduler's tasks, the host's
        view at tick start: uint8 [W][Q], the input of hqs_prefill_state."""
        nw = self.worker_ids.shape[0]
        held = np.nonzero(self._pf_worker >= 0)[0]
        pfwc = np.zeros((nw, len(self._classes)), dtype=np.uint8)
        if held.size:
            widx = np.searchsorted(self.worker_ids, self._pf_worker[held])
            ok = (widx < nw) & (self.worker_ids[np.minimum(widx, nw - 1)] == self._pf_worker[held])
            pfwc[widx[ok], self._task_class[held[ok]]] = 1
        return np.ascontiguousarray(pfwc)

    # proactive filling ------------------------------------------------------------------------------
    def set_prefill(self, reserve: int, max_per_worker: int) -> None:
        """SchedulerConfig::proactive_filling_reserve / _max (scheduler/state.rs:14-21; tako's defaults: 16 / 40)."""
        self._prefill = (int(reserve), int(max_per_worker))
        self._check(self._lib.hqs_prefill_config(self._ctx, int(reserve), int(max_per_worker)))

    def prefilled_tasks(self, worker_id: int) -> np.ndarray:
        return np.nonzero(self._pf_worker == worker_id)[0]

    def on_task_running_prefilled(self, handle: int, variant: int) -> None:
        """The worker started one of its prefilled tasks by itself (reactor.rs:263-345, RunningPrefilled): the task leaves
        the ready set and takes the worker's resources."""
        pos = self._start_prefilled(handle, variant)
        self._take_resources(pos, int(self._task_class[handle]), variant)

    def _start_prefilled(self, handle: int, variant: int) -> int:
        """Bookkeeping of on_task_running_prefilled without the free vectors; returns the worker's index."""
        pos = self._prefilled_started(handle, variant)
        self.remove_ready_tasks(np.array([handle], dtype=np.uint32))
        return pos

    def _prefilled_started(self, handle: int, variant: int) -> int:
        """The host half of _start_prefilled: the task now runs on the worker it was prefilled on; returns the worker's
        index.  A sharded graph context takes the task out of its table on every rank instead (hqs_shard_graph_remove)."""
        wid = int(self._pf_worker[handle])
        assert wid >= 0, "task is not prefilled"
        pos = int(np.searchsorted(self.worker_ids, wid))
        self._pf_worker[handle] = -1
        self._task_worker[handle] = pos
        self._task_variant[handle] = variant
        return pos

    def _take_resources(self, pos: int, rq_id: int, variant: int) -> None:
        """A task of class rq_id started on worker index pos with the given variant: it takes the worker's resources.
        An unlimited amount (HQS_AMOUNT_MAX) stays unlimited, as on the device."""
        am = self._amount_tab[rq_id, variant]
        fr = self.free[pos]
        taken = np.where(fr == L.HQS_AMOUNT_MAX, fr, fr - np.minimum(fr, am))
        self.free[pos] = np.where(self._all_tab[rq_id, variant], 0, taken)

    def on_retract_response(self, worker_id: int, handles) -> Dict[int, List[Tuple[int, int]]]:
        """on_retract_response (server/reactor.rs:452-498): the worker gave the listed tasks back.  A task with a redirect
        becomes Assigned on its target (returned as target worker id -> [(task, variant)], one ComputeTasks message each);
        without one it would wait again.  Tasks not being retracted from this worker are ignored."""
        to_workers: Dict[int, List[Tuple[int, int]]] = {}
        for t in np.asarray(handles).tolist():
            if self._retracting_from.get(t) != worker_id:
                continue
            del self._retracting_from[t]
            tgt = self.redirects.pop(t, None)
            if tgt is not None:
                to_workers.setdefault(tgt[0], []).append((t, tgt[1]))
        return to_workers

    def dispose_prefill(self, rq_id: int) -> Dict[int, List[int]]:
        """TaskQueue::check_dispose_prefill (taskqueue.rs:146-152): a task of higher priority became ready, the class's
        prefills are retracted and wait again.  Returns worker id -> [task handles] (RetractTasks messages)."""
        held = np.nonzero((self._pf_worker >= 0) & (self._task_class[: self._pf_worker.shape[0]] == rq_id))[0]
        out: Dict[int, List[int]] = {}
        for t in held.tolist():
            out.setdefault(int(self._pf_worker[t]), []).append(t)
        self._pf_worker[held] = -1
        self._check(self._lib.hqs_prefill_dispose(self._ctx, int(rq_id)))
        return out

    def tasks_finished(self, handles, propagate: bool = False) -> int:
        """task_finished for a batch: returns the resources of each task to its worker
        (Worker::remove_sn_task -> WorkerResources::add, workerload.rs:194-202).  With `propagate`
        (DAG mode) the device also decrements the consumers' dependency counters and marks the
        newly ready ones; returns how many became ready."""
        h = np.ascontiguousarray(handles, dtype=np.uint32)
        if h.size == 0:
            return 0
        return_resources(self, h)
        if propagate:
            n_new = C.c_uint32(0)
            self._check(self._lib.hqs_tasks_finished(self._ctx, h.size, L.ptr(h), C.byref(n_new)))
            return int(n_new.value)
        return 0

    def submit_tasks(self, handles, rq_ids, priorities, dep_off, deps) -> int:
        """on_new_tasks (reactor.rs:188-220) for new tasks with dependencies (hqs_graph_push): the dependencies of
        handles[i] are deps[dep_off[i]:dep_off[i + 1]].  A dependency on a live task or on an earlier task of the batch
        counts; one on a finished, removed or unknown task, or on a later task of the batch, is dropped.  Returns how many of
        the tasks are ready at once; the others wait until graph_tasks_finished releases them."""
        h = np.ascontiguousarray(handles, dtype=np.uint32)
        c = np.ascontiguousarray(rq_ids, dtype=np.uint32)
        p = np.ascontiguousarray(priorities, dtype=np.uint64)
        off = np.ascontiguousarray(dep_off, dtype=np.uint32)
        d = np.ascontiguousarray(deps, dtype=np.uint32)
        if not (h.shape == c.shape == p.shape) or off.shape != (h.size + 1,):
            raise ValueError("shape mismatch")
        if h.size == 0:
            return 0
        self._sync_classes()
        n_ready = C.c_uint32(0)
        self._check(self._lib.hqs_graph_push(self._ctx, h.size, L.ptr(h), L.ptr(c), L.ptr(p), L.ptr(off),
                                             L.ptr(d) if d.size else None, C.byref(n_ready)))
        self._grow_tasks(int(h.max()) + 1)
        self._task_class[h] = c
        self._task_prio[h] = p
        return int(n_ready.value)

    def graph_tasks_finished(self, handles) -> np.ndarray:
        """task_finished for tasks of a task graph (hqs_graph_finished): returns each assigned task's resources to its
        worker, as tasks_finished does, takes the tasks out of the ready set and releases their consumers.  Returns the
        handles that became ready, ascending."""
        h = np.ascontiguousarray(handles, dtype=np.uint32)
        if h.size == 0:
            return np.zeros(0, dtype=np.uint32)
        ptr = C.POINTER(C.c_uint32)()
        k = C.c_uint32(0)
        self._check(self._lib.hqs_graph_finished(self._ctx, h.size, L.ptr(h), C.byref(ptr), C.byref(k)))
        ready = np.ctypeslib.as_array(ptr, shape=(k.value,)).copy() if k.value else np.zeros(0, dtype=np.uint32)
        self._grow_tasks(int(h.max()) + 1)
        assigned = h[self._task_worker[h] >= 0]
        if assigned.size:
            return_resources(self, np.unique(assigned))
        return ready

    def graph_cancel_tasks(self, handles) -> Tuple[np.ndarray, Dict[int, List[int]]]:
        """on_cancel_tasks (reactor.rs:696-770) over a task graph (hqs_graph_cancel): the named tasks that are live and,
        transitively, every consumer still waiting on them leave the ready set.  For a named task that is assigned, its
        resources go back to its worker; prefilled, it is no longer held; retracting, its redirect is dropped and the
        resources taken on the redirect target come back.  Returns (every handle that left, ascending; worker id -> the
        named tasks to cancel there, in the order they were named: the CancelTasks messages).  The consumers are the
        returned handles that were not named; they were waiting, so no worker holds them.  A failed task (task_failed,
        reactor.rs:596-694) is cancelled the same way; its worker gets no message."""
        h = np.ascontiguousarray(handles, dtype=np.uint32)
        if h.size == 0:
            return np.zeros(0, dtype=np.uint32), {}
        ptr = C.POINTER(C.c_uint32)()
        k = C.c_uint32(0)
        self._check(self._lib.hqs_graph_cancel(self._ctx, h.size, L.ptr(h), C.byref(ptr), C.byref(k)))
        gone = np.ctypeslib.as_array(ptr, shape=(k.value,)).copy() if k.value else np.zeros(0, dtype=np.uint32)
        return gone, cancel_bookkeeping(self, h, gone)

    def compact_handles(self, keep=None) -> np.ndarray:
        """Retires the handles of forgotten tasks (hqs_handles_compact): the surviving handles are renumbered 0 ..
        n_kept - 1 in ascending order, so handle order stays TaskId order and a long-running server's tick cost and memory
        follow its live tasks.  A handle survives if its task is in the device table (waiting, ready, prefilled, assigned
        and not finished or removed), if this object still tracks it (assigned to a worker, prefilled, or with a pending
        redirect or retract), or if it is in `keep` (handles the caller tracks).  A finished task stays in the table until
        the caller retires it with remove_ready_tasks (tasks_finished does not take it out).  The host mirror is renumbered
        with the table.  Returns old_of_new: the old handle of each new handle, ascending; the caller renumbers its own
        handles with it (np.searchsorted(old_of_new, old) for a survivor)."""
        n = int(self._lib_stats().n_handles)
        k = np.concatenate([tracked_handles(self, n),
                            np.zeros(0, np.int64) if keep is None else np.asarray(keep, dtype=np.int64).ravel()])
        k = np.ascontiguousarray(np.unique(k), dtype=np.uint32)
        ptr = C.POINTER(C.c_uint32)()
        nk = C.c_uint32(0)
        self._check(self._lib.hqs_handles_compact(self._ctx, k.size, L.ptr(k) if k.size else None, C.byref(ptr),
                                                  C.byref(nk)))
        old_of_new = np.ctypeslib.as_array(ptr, shape=(nk.value,)).copy() if nk.value else np.zeros(0, dtype=np.uint32)
        self._grow_tasks(n)
        renumber_host_mirror(self, old_of_new.astype(np.int64))
        return old_of_new

    def graph_debug(self) -> np.ndarray:
        """hqs_graph_debug: [live edges, edge-pool capacity, pool compactions, waiting tasks]."""
        out = (C.c_uint64 * 4)()
        self._check(self._lib.hqs_graph_debug(self._ctx, out))
        return np.array(list(out), dtype=np.uint64)

    def new_worker_query(self, worker_totals: np.ndarray, now: float = 0.0, remaining_s: Optional[np.ndarray] = None,
                         min_utilization: Optional[np.ndarray] = None):
        """compute_new_worker_query (scheduler/query.rs:12-131): which of these HYPOTHETICAL workers would get
        work from the current ready set?  Nothing is consumed.  Partial descriptors use HQS_AMOUNT_MAX for unknown
        resources (query.rs:35-46); remaining_s = time limits of the allocation (inf = none); min_utilization as in
        WorkerConfiguration.  Returns (needed[bool], counts, total)."""
        self._sync_classes()
        w, tot = query_workers(worker_totals, remaining_s, min_utilization)
        nw = tot.shape[0]
        counts = np.zeros(nw, dtype=np.uint32)
        n = C.c_uint32(0)
        self._check(self._lib.hqs_query(self._ctx, nw, L.ptr(w), L.ptr(tot), L.ptr(tot), None, C.byref(n), L.ptr(counts), None))
        return counts > 0, counts, int(n.value)

    # declared priority levels (sharded ready sets) ------------------------------------------------
    def n_declared_levels(self) -> int:
        n = C.c_uint32(0)
        self._check(self._lib.hqs_levels_live(self._ctx, 0, None, None, C.byref(n)))
        return int(n.value)

    def levels_live(self) -> Tuple[np.ndarray, np.ndarray]:
        """The context's exact level table (u64, descending) and, per level, whether a task of this context carries it
        (uint8 0 / 1)."""
        n = self.n_declared_levels()
        lv = np.zeros(n, dtype=np.uint64)
        live = np.zeros(n, dtype=np.uint8)
        if n:
            got = C.c_uint32(0)
            self._check(self._lib.hqs_levels_live(self._ctx, n, L.ptr(lv), L.ptr(live), C.byref(got)))
        return lv, live

    def levels_retain(self, keep: np.ndarray) -> None:
        """Drops the levels whose entry of `keep` (aligned with levels_live()) is 0; none of them may be carried by a task
        of this context."""
        k = np.ascontiguousarray(keep, dtype=np.uint8)
        self._check(self._lib.hqs_levels_retain(self._ctx, k.size, L.ptr(k)))

    # misc ---------------------------------------------------------------------------------------
    def rearm(self) -> None:
        self._check(self._lib.hqs_ready_rearm(self._ctx))

    def sync(self) -> None:
        self._check(self._lib.hqs_sync(self._ctx))

    def _lib_stats(self) -> L.hqs_stats:
        st = L.hqs_stats()
        self._check(self._lib.hqs_get_stats(self._ctx, C.byref(st)))
        return st

    def stats(self) -> Dict[str, int]:
        st = self._lib_stats()
        return {name: int(getattr(st, name)) for name, _ in L.hqs_stats._fields_}

    @property
    def stream_ptr(self) -> int:
        return int(self._lib.hqs_stream(self._ctx) or 0)
