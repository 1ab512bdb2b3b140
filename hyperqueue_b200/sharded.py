"""Multi-GPU sharding of the ready set (SURVEY.md §8(e)): one process per GPU, the task table is
block-sharded by handle, worker state is replicated.

Per tick:
  1. every rank histograms ITS ready tasks per (priority level, class) group     hqs_shard_count
  2. all-gather of the count vectors (NCCL over NVLink; 4 B x groups per rank — the only data-path
     collective), from which every rank derives   counts_all = sum over ranks
                                                   ranks_before = sum over lower ranks   (shard_exchange)
  3. every rank runs the SAME deterministic solve on counts_all (replicated worker state => identical
     count segments everywhere) and emits only its own tasks: a task's global rank inside its group is
     ranks_before[g] + its local rank                                           hqs_shard_solve_emit
  4. the assignment lists are gathered where they are needed (host, or all-gather of (task, worker) pairs).
No task data moves between GPUs.  The exchange logic is device-agnostic torch code so that it is covered
by world_size-2 gloo tests on CPU (tests/test_sharded_cpu.py).

Fused form (`ShardedScheduler(..., p2p=True)`, the default on GPUs): steps 1-3 are ONE stream of kernels with no
host collective in between — the counting step's vector goes to every peer by NVLink peer stores (CUDA IPC
mapped exchange buffers, hqs_shard_xbuf / hqs_ipc_open / hqs_shard_attach) followed by a release flag, and the
solver kernel acquires all flags and sums the vectors itself (hqs_shard_tick_launch).  torch.distributed is then
used once, at set-up, to pass the 64-byte IPC handles around.

Proactive filling works in both forms.  Each rank keeps the prefill state of its own tasks; before the tick the ranks OR
their "worker holds a prefilled task of the class" masks (reduce_or), so every rank solves with the same global
mask, computes the same prefill ranges and emits the prefill records of its own tasks.

The autoalloc what-if query (ShardedScheduler.new_worker_query) runs the same two forms without the emit step
(hqs_shard_query_launch, or hqs_shard_count + exchange + hqs_shard_query_solve): every rank solves the summed counts and
returns the same answer, the one a single context holding all ranks' tasks gives.

Priority levels are declared on every rank (hqs_levels_add), so that every rank numbers them identically, and are pruned
by all ranks together at the start of a tick or a query (ShardedScheduler.prune_levels): a level is dropped only when no
task of any rank carries it.

Task graphs (ShardedScheduler.graph_init, then submit_tasks / graph_tasks_finished / graph_cancel_tasks): the graph is
replicated on every rank (hqs_shard_graph_init) and every rank makes every graph call with the same GLOBAL arguments, runs
the same propagation, writes the keys it owns and returns the handles it owns.  No graph data moves between ranks; the only
collective is the free-vector all-reduce that finishing and cancelling already need.  ShardedScheduler.compact_handles retires
the handles of forgotten tasks the same way: every rank renumbers the replicated graph alike and keeps its own tasks, and the
ranks' ranges shrink in place.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.distributed as dist

from . import _lib as L
from .scheduler import (WorkerTaskMapping, apply_tick_records, cancel_bookkeeping, query_workers, renumber_host_mirror,
                        return_resources, tracked_handles)


def shard_exchange(counts_local: torch.Tensor, rank: int, world: int,
                   group: Optional[dist.ProcessGroup] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """counts_local: int32 [G] on any device.  Returns (counts_all, ranks_before), int32 [G]."""
    if world == 1:
        return counts_local.clone(), torch.zeros_like(counts_local)
    gathered = torch.empty(world * counts_local.numel(), dtype=counts_local.dtype, device=counts_local.device)
    dist.all_gather_into_tensor(gathered, counts_local.contiguous(), group=group)
    g2 = gathered.view(world, -1).to(torch.int64)
    counts_all = g2.sum(0).to(torch.int32)
    before = g2[:rank].sum(0).to(torch.int32) if rank else torch.zeros_like(counts_local)
    return counts_all, before


def reduce_or(local: np.ndarray, world: int, group: Optional[dist.ProcessGroup] = None,
              device: Optional[torch.device] = None) -> np.ndarray:
    """The element-wise OR of the ranks' uint8 0 / 1 arrays of one shape (one all-reduce, on `device` for NCCL).  Used for
    what must hold over the tasks of ALL ranks while each rank knows only its own: "worker w holds a prefilled task of
    class c" (the [W][Q] mask every rank passes to hqs_prefill_state) and "a task carries priority level i" (the live
    vector every rank passes to hqs_levels_retain)."""
    m = np.ascontiguousarray(local, dtype=np.uint8)
    if world == 1:
        return m
    dev = device if device is not None and dist.get_backend(group) == "nccl" else torch.device("cpu")
    t = torch.from_numpy(m.copy()).to(dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
    return np.ascontiguousarray(t.cpu().numpy())


reduce_prefill_mask = reduce_or          # the name the prefill path has always imported


def levels_need_pruning(n_levels: int, n_classes: int, prefill: bool, pruned_at: int) -> bool:
    """A sharded ready set declares every priority it is given (hqs_levels_add) and never prunes on its own.  The ranks
    prune together when the declared table exceeds what a tick's groups allow (HQS_MAX_GROUPS / Q levels, half of that
    with proactive filling, which doubles the groups) or has more than doubled (+64) since the last pruning.  Declared
    tables are identical on every rank, so every rank decides the same way."""
    budget = L.HQS_MAX_GROUPS // (max(n_classes, 1) * (2 if prefill else 1))
    return n_levels > budget or n_levels > 2 * pruned_at + 64


def gather_peer_handles(sched, rank: int, world: int, group: Optional[dist.ProcessGroup] = None):
    """Collective half of the set-up: allocates this rank's exchange buffer and all-gathers the 64-byte CUDA IPC
    handles (on the host).  Returns (own device pointer, [handle bytes of rank r])."""
    lib = sched._lib
    own = C.c_void_p()
    handle = (C.c_uint8 * L.HQS_IPC_HANDLE_BYTES)()
    sched._check(lib.hqs_shard_xbuf(sched._ctx, C.byref(own), handle))
    if world == 1:
        return own, [bytes(handle)]
    mine = torch.tensor(list(bytes(handle)), dtype=torch.uint8)
    backend = dist.get_backend(group)
    dev = torch.device("cuda", torch.cuda.current_device()) if backend == "nccl" else torch.device("cpu")
    gathered = [torch.zeros(L.HQS_IPC_HANDLE_BYTES, dtype=torch.uint8, device=dev) for _ in range(world)]
    dist.all_gather(gathered, mine.to(dev), group=group)
    return own, [bytes(g.cpu().tolist()) for g in gathered]


def open_and_attach(sched, rank: int, world: int, own, handles) -> None:
    """Local half: maps the other ranks' buffers (cudaIpcOpenMemHandle) and attaches the context."""
    lib = sched._lib
    ptrs = (C.c_void_p * world)()
    for r in range(world):
        if r == rank:
            ptrs[r] = own
            continue
        hb = (C.c_uint8 * L.HQS_IPC_HANDLE_BYTES)(*handles[r])
        p = C.c_void_p()
        sched._check(lib.hqs_ipc_open(sched._ctx, hb, C.byref(p)))
        ptrs[r] = p
    sched._check(lib.hqs_shard_attach(sched._ctx, world, rank, ptrs))


def attach_peers(sched, rank: int, world: int, group: Optional[dist.ProcessGroup] = None) -> None:
    """One-time set-up of the peer-to-peer count exchange: every rank allocates its exchange buffer, the CUDA IPC
    handles are all-gathered (64 bytes per rank, on the host), every rank maps the others' buffers."""
    own, handles = gather_peer_handles(sched, rank, world, group)
    open_and_attach(sched, rank, world, own, handles)


def block_range(n_total: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous handle range [lo, hi) of a rank; ranks are ordered by handle so that lower ranks hold the
    lower (earlier TaskId) handles — the global rank of a task inside its group needs exactly that."""
    per = (n_total + world - 1) // world
    lo = min(rank * per, n_total)
    return lo, min(lo + per, n_total)


class ShardedScheduler:
    """Wraps one GpuScheduler per rank.  Handles given to / returned from this class are GLOBAL."""

    def __init__(self, sched, rank: int, world: int, n_total: int, device: torch.device,
                 group: Optional[dist.ProcessGroup] = None, p2p: bool = False) -> None:
        self.s = sched
        self.rank, self.world, self.group = rank, world, group
        self.n_total = int(n_total)
        self.lo, self.hi = block_range(n_total, rank, world)
        self.graph = False                  # graph_init was called: tasks enter and leave through the graph calls
        self.device = device
        self._counts = torch.zeros(L.HQS_MAX_GROUPS, dtype=torch.int32, device=device)
        self.p2p = bool(p2p)
        self.last_mapping: Optional[WorkerTaskMapping] = None
        self.levels_pruned_at = 0           # declared table size after the last pruning (the same on every rank)
        if self.p2p:
            attach_peers(sched, rank, world, group)

    def add_ready_tasks(self, handles, rq_ids, priorities) -> None:
        if self.graph:                      # the replicated graph must see every live task
            n = np.asarray(handles).size
            self.submit_tasks(handles, rq_ids, priorities, np.zeros(n + 1, dtype=np.uint32), np.zeros(0, dtype=np.uint32))
            return
        h = np.asarray(handles, dtype=np.int64)
        # every rank sees the whole call: number the priority levels identically everywhere
        lv = np.ascontiguousarray(np.unique(np.asarray(priorities, dtype=np.uint64)))
        self.s._sync_classes()
        self.s._check(self.s._lib.hqs_levels_add(self.s._ctx, lv.size, L.ptr(lv)))
        m = (h >= self.lo) & (h < self.hi)
        if m.any():
            self.s.add_ready_tasks((h[m] - self.lo).astype(np.uint32), np.asarray(rq_ids)[m], np.asarray(priorities)[m])

    def remove_ready_tasks(self, handles) -> None:
        """TaskQueue::remove for GLOBAL handles, called with the same list on every rank: the owner of each task takes it
        out of its ready set.  Also the way to retire the handle of a finished task, so that it no longer keeps its
        priority level alive (prune_levels)."""
        if self.graph:                      # every rank's replica forgets the handles too
            h = np.ascontiguousarray(handles, dtype=np.uint32).reshape(-1)
            if h.size:
                self.s._check(self.s._lib.hqs_shard_graph_remove(self.s._ctx, h.size, L.ptr(h)))
            return
        mine = self._mine(handles)
        if mine.size:
            self.s.remove_ready_tasks(mine.astype(np.uint32))

    def prune_levels(self) -> None:
        """Drops the declared priority levels that no task of any rank carries (levels_need_pruning decides when; a
        collective when it does).  Called at the start of run_scheduling and new_worker_query, where no tick is in flight."""
        s = self.s
        n = s.n_declared_levels()
        if not levels_need_pruning(n, s.n_classes, s._prefill[1] > 0, self.levels_pruned_at):
            return
        _, live = s.levels_live()
        keep = reduce_or(live, self.world, self.group, self.device)
        s.levels_retain(keep)
        self.levels_pruned_at = int(np.count_nonzero(keep))

    def run_scheduling(self, now: float = 0.0, out_cap: Optional[int] = None):
        """One sharded tick.  Returns (this rank's records with GLOBAL handles, free vectors after the tick): its assignments
        (kind 0 / 2) in single-context order, then its prefill records (kind 1).  self.last_mapping holds the same records
        as a WorkerTaskMapping (messages(), retracts of kind-2 records)."""
        s = self.s
        s._sync_classes()
        self.prune_levels()
        w = s._worker_structs(now)
        free = np.ascontiguousarray(s.free)
        total = np.ascontiguousarray(s.total)
        blocked = s._blocked_bytes()
        if s._prefill[1] > 0:
            # a host collective at tick start: the previous tick has been fetched, so no collective overlaps a tick in
            # flight (DESIGN.md §6); every rank passes the same global mask
            pfwc = reduce_or(s.prefill_mask(), self.world, self.group, self.device)
            s._check(s._lib.hqs_prefill_state(s._ctx, w.shape[0], L.ptr(pfwc)))
        cap = out_cap or max(self.hi - self.lo, 1)
        if self.p2p:
            s._check(s._lib.hqs_shard_tick_launch(s._ctx, w.shape[0], L.ptr(w), L.ptr(free), L.ptr(total),
                                                  L.ptr(blocked) if blocked is not None else None, cap))
        else:
            ng = C.c_uint32(0)
            s._check(s._lib.hqs_shard_count(s._ctx, w.shape[0], L.ptr(w), L.ptr(free), L.ptr(total),
                                            L.ptr(blocked) if blocked is not None else None,
                                            C.c_void_p(self._counts.data_ptr()), self._counts.numel(), C.byref(ng)))
            counts_all, before = shard_exchange(self._counts, self.rank, self.world, self.group)
            torch.cuda.synchronize(self.device)
            s._check(s._lib.hqs_shard_solve_emit(s._ctx, C.c_void_p(counts_all.data_ptr()), C.c_void_p(before.data_ptr()), cap))
        out = np.zeros(cap, dtype=L.assignment_dtype)
        free_after = np.zeros_like(free)
        n = C.c_uint32(0)
        s._check(s._lib.hqs_tick_fetch(s._ctx, cap, L.ptr(out), C.byref(n), L.ptr(free_after)))
        a = out[: n.value].copy()
        retract_from = self._record(a)
        a["task"] += np.uint32(self.lo)
        s.free = free_after
        self.last_mapping = WorkerTaskMapping(a, s.worker_ids.copy(), free_after, retract_from)
        return a, free_after

    def new_worker_query(self, worker_totals: np.ndarray, now: float = 0.0, remaining_s: Optional[np.ndarray] = None,
                         min_utilization: Optional[np.ndarray] = None):
        """compute_new_worker_query (scheduler/query.rs:12-131) over the ready sets of ALL ranks: GpuScheduler.new_worker_query
        on one context holding every rank's tasks, bit for bit.  Every rank calls it with the same arguments and gets the same
        (needed[bool], counts, total); nothing is consumed.  It is an exchange like a tick: call it when no tick is in flight
        (DESIGN.md §6).  `now` is accepted for symmetry with GpuScheduler: the fake workers' time limits are remaining_s."""
        s = self.s
        s._sync_classes()
        self.prune_levels()
        w, tot = query_workers(worker_totals, remaining_s, min_utilization)
        nw = tot.shape[0]
        if self.p2p:
            # no allocation between the launches of the ranks (contexts of one process wait for each other on the device)
            s._check(s._lib.hqs_tick_reserve(s._ctx, nw, max(self.hi - self.lo, 1), 0))
            s._check(s._lib.hqs_shard_query_launch(s._ctx, nw, L.ptr(w), L.ptr(tot), L.ptr(tot), None))
        else:
            ng = C.c_uint32(0)
            s._check(s._lib.hqs_shard_count(s._ctx, nw, L.ptr(w), L.ptr(tot), L.ptr(tot), None,
                                            C.c_void_p(self._counts.data_ptr()), self._counts.numel(), C.byref(ng)))
            counts_all, _ = shard_exchange(self._counts, self.rank, self.world, self.group)
            torch.cuda.synchronize(self.device)
            s._check(s._lib.hqs_shard_query_solve(s._ctx, C.c_void_p(counts_all.data_ptr())))
        counts = np.zeros(nw, dtype=np.uint32)
        n = C.c_uint32(0)
        s._check(s._lib.hqs_query_fetch(s._ctx, C.byref(n), L.ptr(counts), None))
        return counts > 0, counts, int(n.value)

    def _record(self, a_local):
        """TaskRuntimeState::Assigned{worker_id, rv_id} of this rank's tasks (local handles), as GpuScheduler.run_scheduling
        keeps it (needed to return the resources when the tasks finish), and the rank's redirects and prefills."""
        return apply_tick_records(self.s, a_local)

    def _mine(self, handles) -> np.ndarray:
        """This rank's handles among GLOBAL `handles`, as local handles."""
        h = np.asarray(handles, dtype=np.int64).reshape(-1)
        return h[(h >= self.lo) & (h < self.hi)] - self.lo

    # proactive filling: every rank is called with the same arguments; handles are GLOBAL ---------------------------
    def set_prefill(self, reserve: int, max_per_worker: int) -> None:
        """SchedulerConfig::proactive_filling_reserve / _max; the same on every rank."""
        self.s.set_prefill(reserve, max_per_worker)

    def prefilled_tasks(self, worker_id: int) -> np.ndarray:
        """This rank's tasks prefilled on the worker (global handles)."""
        return self.s.prefilled_tasks(worker_id) + self.lo

    def on_task_running_prefilled(self, handle: int, variant: int) -> None:
        """The worker started one of its prefilled tasks (RunningPrefilled).  Only the owner knows the worker and the class,
        so the owner's (worker index, class) is summed over the ranks (one all-reduce of two integers), and every rank takes
        the same resources from its replicated free vectors.  After graph_init the task leaves the table of every rank
        (remove_ready_tasks: hqs_shard_graph_remove), so that no replica keeps it VALID."""
        s = self.s
        mine = self._mine([handle])
        key = np.zeros(2, dtype=np.int64)
        if mine.size:
            loc = int(mine[0])
            pos = s._prefilled_started(loc, variant) if self.graph else s._start_prefilled(loc, variant)
            key[:] = (pos + 1, int(s._task_class[loc]) + 1)
        if self.world > 1:
            t = torch.from_numpy(key)
            dev = self.device if dist.get_backend(self.group) == "nccl" else torch.device("cpu")
            t = t.to(dev)
            dist.all_reduce(t, group=self.group)
            key = t.cpu().numpy()
        assert key[0] > 0, "task is not prefilled on any rank"
        s._take_resources(int(key[0]) - 1, int(key[1]) - 1, variant)
        if self.graph:
            self.remove_ready_tasks([handle])

    def on_retract_response(self, worker_id: int, handles) -> Dict[int, List[Tuple[int, int]]]:
        """The worker gave the listed tasks back; the owner of a redirected task returns it as target worker id ->
        [(global handle, variant)]."""
        sent = self.s.on_retract_response(worker_id, self._mine(handles))
        return {wid: [(t + self.lo, v) for t, v in lst] for wid, lst in sent.items()}

    def dispose_prefill(self, rq_id: int) -> Dict[int, List[int]]:
        """check_dispose_prefill on every rank: each rank retracts its own prefilled tasks of the class and returns them as
        worker id -> [global handles]."""
        ret = self.s.dispose_prefill(rq_id)
        return {wid: [t + self.lo for t in lst] for wid, lst in ret.items()}

    # task graphs: every rank is called with the same arguments; handles are GLOBAL --------------------------------------
    def graph_init(self) -> None:
        """Replicates the task graph over all n_total handles on this rank (hqs_shard_graph_init); call it on every rank
        before any task is added.  From then on add_ready_tasks and remove_ready_tasks go through the graph calls."""
        self.s._check(self.s._lib.hqs_shard_graph_init(self.s._ctx, self.n_total, self.lo, self.hi))
        self.graph = True

    def submit_tasks(self, handles, rq_ids, priorities, dep_off, deps) -> int:
        """on_new_tasks with dependencies (GpuScheduler.submit_tasks) for GLOBAL handles: the batch's priorities are
        declared first (hqs_levels_add), then every rank links the whole batch and pushes the keys it owns
        (hqs_shard_graph_push).  Returns how many of this rank's tasks are ready at once."""
        s = self.s
        h = np.ascontiguousarray(handles, dtype=np.uint32).reshape(-1)
        c = np.ascontiguousarray(rq_ids, dtype=np.uint32).reshape(-1)
        p = np.ascontiguousarray(priorities, dtype=np.uint64).reshape(-1)
        off = np.ascontiguousarray(dep_off, dtype=np.uint32)
        d = np.ascontiguousarray(deps, dtype=np.uint32)
        if not (h.shape == c.shape == p.shape) or off.shape != (h.size + 1,):
            raise ValueError("shape mismatch")
        if h.size == 0:
            return 0
        s._sync_classes()
        lv = np.ascontiguousarray(np.unique(p))
        s._check(s._lib.hqs_levels_add(s._ctx, lv.size, L.ptr(lv)))
        n_ready = C.c_uint32(0)
        s._check(s._lib.hqs_shard_graph_push(s._ctx, h.size, L.ptr(h), L.ptr(c), L.ptr(p), L.ptr(off),
                                             L.ptr(d) if d.size else None, C.byref(n_ready)))
        m = (h >= self.lo) & (h < self.hi)
        if m.any():
            loc = h[m] - np.uint32(self.lo)
            s._grow_tasks(int(loc.max()) + 1)
            s._task_class[loc] = c[m]
            s._task_prio[loc] = p[m]
        return int(n_ready.value)

    def graph_tasks_finished(self, handles) -> np.ndarray:
        """task_finished in a task graph (GpuScheduler.graph_tasks_finished) for GLOBAL handles: the owners return the
        resources of their assigned tasks and the ranks sum the change of the free vectors, as tasks_finished does; every rank
        releases consumers across the whole graph (hqs_shard_graph_finished).  Returns the newly ready handles this rank owns,
        global and ascending: the ranks' lists in rank order are the single-context list."""
        s = self.s
        h = np.ascontiguousarray(handles, dtype=np.uint32).reshape(-1)
        if h.size == 0:
            return np.zeros(0, dtype=np.uint32)
        ptr = C.POINTER(C.c_uint32)()
        k = C.c_uint32(0)
        s._check(s._lib.hqs_shard_graph_finished(s._ctx, h.size, L.ptr(h), C.byref(ptr), C.byref(k)))
        ready = np.ctypeslib.as_array(ptr, shape=(k.value,)).copy() if k.value else np.zeros(0, dtype=np.uint32)
        mine = self._mine(h)
        before = s.free.copy()
        if mine.size:
            s._grow_tasks(int(mine.max()) + 1)
            assigned = np.unique(mine[s._task_worker[mine] >= 0])
            if assigned.size:
                return_resources(s, assigned)
        self._sum_free_change(before)
        return ready

    def graph_cancel_tasks(self, handles) -> Tuple[np.ndarray, Dict[int, List[int]]]:
        """on_cancel_tasks / task_failed over a task graph (GpuScheduler.graph_cancel_tasks) for GLOBAL handles: every rank
        removes the whole closure from its replica (hqs_shard_graph_cancel) and does the bookkeeping of its own named tasks;
        the ranks then sum the change of the free vectors.  Returns (the part of the closure this rank owns, global and
        ascending; worker id -> this rank's named tasks to cancel there, global handles)."""
        s = self.s
        h = np.ascontiguousarray(handles, dtype=np.uint32).reshape(-1)
        if h.size == 0:
            return np.zeros(0, dtype=np.uint32), {}
        ptr = C.POINTER(C.c_uint32)()
        k = C.c_uint32(0)
        s._check(s._lib.hqs_shard_graph_cancel(s._ctx, h.size, L.ptr(h), C.byref(ptr), C.byref(k)))
        gone = np.ctypeslib.as_array(ptr, shape=(k.value,)).copy() if k.value else np.zeros(0, dtype=np.uint32)
        before = s.free.copy()
        msgs = cancel_bookkeeping(s, self._mine(h), gone.astype(np.int64) - self.lo)
        self._sum_free_change(before)
        return gone, {wid: [t + self.lo for t in lst] for wid, lst in msgs.items()}

    def compact_handles(self, keep=None) -> np.ndarray:
        """Retires the handles of forgotten tasks over the sharded graph (hqs_shard_graph_compact), the counterpart of
        GpuScheduler.compact_handles.  Every rank calls it with the same arguments and gets the same old_of_new: the old
        GLOBAL handle of each new global handle, ascending (np.searchsorted(old_of_new, old) renumbers a survivor).
        A handle survives if its task is in the replicated graph, if any rank still tracks it on the host (assigned to a
        worker, prefilled, with a pending redirect or retract, or a started prefilled task that left the graph), or if it is
        in `keep` (global handles the caller tracks).  What the ranks track is gathered in one variable-length all-gather
        (none with world == 1), so every rank passes the same keep list.  Survivor i becomes global handle i; no key moves
        between ranks: each rank's range [lo, hi) becomes [number of survivors below lo, number below hi), and the last rank
        also takes the freed tail up to n_total.  This rank's host mirror, redirects and retracts are renumbered, and lo / hi
        follow the new range.
        Intake: new tasks carry higher TaskIds than every survivor, so they get the handles of the freed tail and all land on
        the last rank, until the caller compacts again or sets up a new sharded graph.  (Fixed blocks already put a stream of
        TaskId-ordered submits on one rank at a time; ranges are not rebalanced by moving keys.)"""
        s = self.s
        mine = np.unique(tracked_handles(s, s._task_worker.shape[0])) + self.lo
        k = np.concatenate([self._all_gather_handles(mine),
                            np.zeros(0, np.int64) if keep is None else np.asarray(keep, dtype=np.int64).ravel()])
        k = np.ascontiguousarray(np.unique(k), dtype=np.uint32)
        ptr = C.POINTER(C.c_uint32)()
        nk = C.c_uint32(0)
        rng = np.zeros(2, dtype=np.uint32)
        s._check(s._lib.hqs_shard_graph_compact(s._ctx, k.size, L.ptr(k) if k.size else None, C.byref(ptr), C.byref(nk),
                                                L.ptr(rng)))
        old_of_new = np.ctypeslib.as_array(ptr, shape=(nk.value,)).copy() if nk.value else np.zeros(0, dtype=np.uint32)
        a, b = np.searchsorted(old_of_new, [self.lo, self.hi])
        kept = old_of_new[a:b].astype(np.int64) - self.lo          # this rank's survivors, old local handles
        if kept.size:
            s._grow_tasks(int(kept[-1]) + 1)
        renumber_host_mirror(s, kept)
        self.lo, self.hi = int(rng[0]), int(rng[1])
        return old_of_new

    def _all_gather_handles(self, mine: np.ndarray) -> np.ndarray:
        """The concatenation over the ranks of each rank's int64 handle list `mine` (lists of any length)."""
        if self.world == 1:
            return np.asarray(mine, dtype=np.int64)
        dev = self.device if dist.get_backend(self.group) == "nccl" else torch.device("cpu")
        sizes = [torch.zeros(1, dtype=torch.int64, device=dev) for _ in range(self.world)]
        dist.all_gather(sizes, torch.tensor([mine.size], dtype=torch.int64, device=dev), group=self.group)
        sizes = [int(x.item()) for x in sizes]
        buf = torch.zeros(max(max(sizes), 1), dtype=torch.int64)
        buf[: mine.size] = torch.from_numpy(np.asarray(mine, dtype=np.int64))
        parts = [torch.zeros_like(buf, device=dev) for _ in range(self.world)]
        dist.all_gather(parts, buf.to(dev), group=self.group)
        return np.concatenate([p.cpu().numpy()[:n] for p, n in zip(parts, sizes)])

    def _sum_free_change(self, before: np.ndarray) -> None:
        """Returning resources only adds to a free vector: the per-worker change (>= 0, below the worker's total) is summed
        over the ranks (one all-reduce of a [W][R] matrix, or nothing with world == 1)."""
        s = self.s
        if self.world > 1:
            delta = (s.free - before).view(np.int64)
            dev = self.device if dist.get_backend(self.group) == "nccl" else torch.device("cpu")
            t = torch.from_numpy(np.ascontiguousarray(delta)).to(dev)
            dist.all_reduce(t, group=self.group)
            s.free = before + t.cpu().numpy().view(np.uint64)

    def tasks_finished(self, handles) -> None:
        """task_finished for GLOBAL handles, called with the same list on every rank: every rank holds the replicated free
        vectors, but only the owner of a task knows where it ran.  The owner returns the resources as GpuScheduler does
        (scheduler.return_resources: an unlimited amount stays unlimited, `All` gives the total back), and the per-worker change of its
        free vectors is summed over the ranks (one all-reduce of a [W][R] matrix, or nothing with world == 1)."""
        s = self.s
        mine = self._mine(handles)
        before = s.free.copy()
        if mine.size:
            assert (s._task_worker[mine] >= 0).all(), "a finished task of this rank was never assigned"
            return_resources(s, mine)
        self._sum_free_change(before)
