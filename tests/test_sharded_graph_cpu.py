"""Task graphs over a sharded ready set, host side (no GPU).

(1) The sharded design restated per rank (ShardRank) against the single-context model (tests/graph_cancel_model.py): a rank
    keeps the graph replicated over the global handles (a VALID bit, the unfinished-dependency counter, the incarnation and
    the consumer lists), keys only for the handles it owns, and counts a task as waiting while it is VALID with unfinished
    dependencies (the single-context model reads that off the key instead).  For random sequences of pushes, finishes,
    cancels and removes, handle re-use included, and random splits over 1 to 4 ranks: each rank's output is the single
    model's output restricted to its range, the outputs concatenate to the whole, each rank's keys are the model's keys of
    its range, the n_ready counts sum to the model's, and every replica holds the model's edges.
(2) ShardedScheduler's bookkeeping of graph_tasks_finished / graph_cancel_tasks / on_task_running_prefilled over gloo with
    world size 2: the owner of a task returns its resources, clears its prefill and its redirect, the ranks sum the change of
    the free vectors, and a started prefilled task leaves every rank's table.  The library calls are replaced by a stand-in
    that answers what hqs_shard_graph_finished / _cancel answer on each rank and records hqs_shard_graph_remove."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

import graph_cancel_model as CM
import level_model as LM

KEEP = LM.KEY_READY | LM.KEY_VALID | LM.KEY_DONE


class ShardRank:
    """One rank of a sharded graph context, as DESIGN §4 and §6 describe it (batches are validated by the caller)."""

    def __init__(self, lo: int, hi: int) -> None:
        self.lo, self.hi = lo, hi
        self.gvalid = set()
        self.gdeps, self.gen, self.lists = {}, {}, {}
        self.key = {}                                   # owned handle -> READY / VALID bits

    def own(self, h):
        return self.lo <= h < self.hi

    def waits(self, c, g):
        return self.gen.get(c, 0) == g and c in self.gvalid and self.gdeps.get(c, 0) > 0

    def leave(self, h):
        self.gvalid.discard(h)
        self.key.pop(h, None)

    def push(self, hs, off, deps):
        pos = {x: i for i, x in enumerate(hs)}
        for x in hs:
            self.gvalid.add(x)
            if self.own(x):
                self.key[x] = LM.KEY_VALID | LM.KEY_READY
        ready = 0
        for i, x in enumerate(hs):
            g = self.gen.get(x, 0) + 1
            self.gen[x] = g
            cnt = 0
            for y in deps[off[i]: off[i + 1]]:
                if pos.get(y, -1) >= i or y not in self.gvalid:
                    continue                            # a later task of the batch, or not VALID: dropped
                self.lists.setdefault(y, []).append((x, g))
                cnt += 1
            self.gdeps[x] = cnt
            if self.own(x):
                if cnt:
                    self.key[x] &= ~LM.KEY_READY
                else:
                    ready += 1
        return ready

    def finished(self, hs):
        won = [x for x in dict.fromkeys(hs) if x in self.gvalid]
        for x in won:
            self.leave(x)
        made = []
        for x in won:
            for c, g in self.lists.pop(x, []):
                if self.waits(c, g):
                    self.gdeps[c] -= 1
                    if self.gdeps[c] == 0 and self.own(c):
                        self.key[c] |= LM.KEY_READY
                        made.append(c)
        return sorted(made)

    def cancel(self, hs):
        gone = {x for x in hs if x in self.gvalid}
        stack = list(gone)
        while stack:
            for c, g in self.lists.get(stack.pop(), []):
                if c not in gone and self.waits(c, g):
                    gone.add(c)
                    stack.append(c)
        for x in gone:
            self.leave(x)
            self.lists.pop(x, None)
        return sorted(x for x in gone if self.own(x))

    def remove(self, hs):
        for x in hs:
            self.leave(x)
            self.lists.pop(x, None)


def _cuts(rng, n, world):
    return [0] + sorted(int(x) for x in rng.integers(0, n + 1, world - 1)) + [n]


def _csr(deps):
    off = np.concatenate([[0], np.cumsum([len(d) for d in deps])]).astype(np.uint32)
    return off, np.array([x for ds in deps for x in ds], dtype=np.uint32)


@pytest.mark.parametrize("seed", range(8))
def test_rank_model_matches_the_single_context_model(seed):
    rng = np.random.default_rng(seed)
    n_total = 400
    world = 1 + seed % 4
    cuts = _cuts(rng, n_total, world)
    single = CM.CancelModel()
    single.classes_set(3)
    ranks = [ShardRank(cuts[r], cuts[r + 1]) for r in range(world)]

    def live():
        return [h for h in range(single.n_handles) if single.flag(h) & LM.KEY_VALID]

    def check(label, want, got):
        for r, g in enumerate(got):
            assert g == [x for x in want if cuts[r] <= x < cuts[r + 1]], (label, r)
        assert sum(got, []) == want, label
        edges = sorted((p, c, g) for p, lst in single.lists.items() for c, g in lst)
        for r, m in enumerate(ranks):
            assert sorted((p, c, g) for p, lst in m.lists.items() for c, g in lst) == edges, (label, r)
            for h in range(m.lo, m.hi):
                assert m.key.get(h, 0) == single.flag(h) & KEEP, (label, r, h)

    nxt, free = 0, []
    for step in range(60):
        lv = live()
        k = int(rng.integers(1, 12))
        reuse = [free.pop(int(rng.integers(0, len(free)))) for _ in range(min(len(free), k // 2))]
        fresh = list(range(nxt, min(nxt + k - len(reuse), n_total)))
        nxt += len(fresh)
        hs = reuse + fresh
        if hs:
            rng.shuffle(hs)
            deps = []
            for i, x in enumerate(hs):
                pool = lv[-40:] + hs[:i] + hs[i + 1: i + 3]     # live tasks, earlier and later tasks of the batch
                deps.append(sorted({int(pool[j]) for j in rng.integers(0, len(pool), int(rng.integers(0, 4)))} - {x})
                            if pool else [])
            off, flat = _csr(deps)
            want = single.graph_push(np.array(hs), rng.integers(0, 3, len(hs)), np.full(len(hs), 5, np.uint64), off, flat)
            got = [m.push(hs, off.tolist(), flat.tolist()) for m in ranks]
            assert sum(got) == want, step
            check(f"push {step}", [], [[] for _ in ranks])
        lv = live()
        op = rng.random()
        if not lv:
            continue
        pick = [int(x) for x in rng.choice(lv, size=min(len(lv), int(rng.integers(1, 5))), replace=False)]
        if op < 0.55:
            pick += pick[:1]                                    # a handle named twice counts once
            want = single.graph_finished(pick)
            check(f"finish {step}", want, [m.finished(pick) for m in ranks])
            free += sorted(set(pick))
        elif op < 0.8:
            want = single.graph_cancel(pick)
            check(f"cancel {step}", want, [m.cancel(pick) for m in ranks])
            free += want
        else:
            single.remove(pick)
            for m in ranks:
                m.remove(pick)
            check(f"remove {step}", [], [[] for _ in ranks])
            free += pick
    assert nxt > 0


class _Lib:
    """hqs_shard_graph_finished / _cancel on one rank: the answer is fixed by the test."""

    def __init__(self, answer):
        self.answer = np.ascontiguousarray(answer, dtype=np.uint32)

    def _out(self, ptr_ref, k_ref):
        if self.answer.size:
            ptr_ref._obj.contents = C.c_uint32.from_buffer(self.answer)
        k_ref._obj.value = self.answer.size
        return 0

    def hqs_shard_graph_finished(self, ctx, n, task, ptr_ref, k_ref):
        return self._out(ptr_ref, k_ref)

    hqs_shard_graph_cancel = hqs_shard_graph_finished

    def hqs_shard_graph_remove(self, ctx, n, task):
        self.removed = C.cast(task, C.POINTER(C.c_uint32))[:n]
        return 0


class _Sched:
    """The part of GpuScheduler that the sharded graph bookkeeping reads and writes (one resource, two workers)."""

    def __init__(self, lib):
        self._lib, self._ctx = lib, None
        self.worker_ids = np.array([100, 101], np.uint32)
        self.total = np.array([[50], [50]], np.uint64)
        self.free = np.array([[20], [30]], np.uint64)
        self._amount_tab = np.zeros((2, 8, 1), np.uint64)
        self._amount_tab[0, 0, 0], self._amount_tab[1, 0, 0] = 5, 7
        self._all_tab = np.zeros((2, 8, 1), bool)
        self._task_class = np.zeros(0, np.uint32)
        self._task_worker = np.zeros(0, np.int64)
        self._task_variant = np.zeros(0, np.uint8)
        self._pf_worker = np.zeros(0, np.int64)
        self.redirects, self._retracting_from = {}, {}
        self._grow_tasks(10)

    def _grow_tasks(self, n):
        m = n - self._task_class.size
        if m > 0:
            self._task_class = np.concatenate([self._task_class, np.zeros(m, np.uint32)])
            self._task_worker = np.concatenate([self._task_worker, np.full(m, -1, np.int64)])
            self._task_variant = np.concatenate([self._task_variant, np.zeros(m, np.uint8)])
            self._pf_worker = np.concatenate([self._pf_worker, np.full(m, -1, np.int64)])

    def _check(self, rc):
        assert rc == 0

    from hyperqueue_b200.scheduler import GpuScheduler
    _prefilled_started = GpuScheduler._prefilled_started      # the real host bookkeeping
    _take_resources = GpuScheduler._take_resources
    del GpuScheduler


def _worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from hyperqueue_b200.sharded import ShardedScheduler
    # rank 0 owns global handles [0, 10), rank 1 [10, 20)
    s = _Sched(_Lib([3, 5] if rank == 0 else [12, 15, 16]))
    sh = ShardedScheduler(s, rank, world, 20, device=None)
    sh.graph = True
    if rank == 0:
        s._task_worker[3], s._task_class[3] = 0, 0          # task 3 runs on worker 100 (5 units)
    else:
        s._task_worker[2], s._task_class[2] = 1, 1          # task 12 runs on worker 101 (7 units)
        s._pf_worker[5] = 101                                # task 15 is prefilled on worker 101
    gone, msgs = sh.graph_cancel_tasks([3, 12, 15, 18])
    out = {"gone": gone.tolist(), "msgs": msgs, "free": s.free.ravel().tolist(), "pf": s._pf_worker[:10].tolist()}
    # a finish on a fresh assignment: the owner returns the resources, both ranks see them
    s._lib = _Lib([7] if rank == 0 else [])
    if rank == 1:
        s._task_worker[4], s._task_class[4] = 0, 1          # task 14 runs on worker 100 (7 units)
    out["ready"] = sh.graph_tasks_finished([14]).tolist()
    out["free2"] = s.free.ravel().tolist()
    # a worker starts task 17 (rank 1's), prefilled on worker 100: every rank takes its 5 units and removes it from its
    # table (the stand-in has no hqs_ready_remove: an owner-only device remove would fail here)
    s._lib = _Lib([])
    if rank == 1:
        s._pf_worker[7], s._task_class[7] = 100, 0
    sh.on_task_running_prefilled(17, 0)
    out["removed"] = list(s._lib.removed)
    out["free3"] = s.free.ravel().tolist()
    out["run17"] = (int(s._task_worker[7]), int(s._pf_worker[7]))
    ret[rank] = out
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_graph_bookkeeping_over_gloo():
    sock = socket.socket(); sock.bind(("127.0.0.1", 0)); port = sock.getsockname()[1]; sock.close()
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(2, port, ret), nprocs=2, join=True)
    r0, r1 = ret[0], ret[1]
    assert r0["gone"] == [3, 5] and r1["gone"] == [12, 15, 16]
    assert r0["msgs"] == {100: [3]} and r1["msgs"] == {101: [12, 15]}
    assert r1["pf"][5] == -1
    assert r0["free"] == r1["free"] == [25, 37]
    assert r0["ready"] == [7] and r1["ready"] == []
    assert r0["free2"] == r1["free2"] == [32, 37]
    assert r0["removed"] == r1["removed"] == [17]
    assert r0["free3"] == r1["free3"] == [27, 37]
    assert r1["run17"] == (0, -1) and r0["run17"] == (-1, -1)
