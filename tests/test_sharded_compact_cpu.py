"""Handle compaction over a sharded task graph (hqs_shard_graph_compact), host side (no GPU).

(1) One rank of the design (CompactRank: the rank of tests/test_sharded_graph_cpu.py with a compaction of its own) against
    the single-context model with hqs_handles_compact (tests/compact_model.py).  Every rank computes the survivors from its
    replicated VALID bits and the shared keep list, renumbers the replicated graph alike, moves the keys it owns to
    new(h) - new(lo) and takes the range [new(lo), new(hi)), the last rank up to n_total.  For random sequences of pushes
    (the freed tail re-used after every compaction, so new tasks land on the last rank), finishes, cancels, removes and
    compactions over random splits of 1 to 4 ranks, empty ranges included: every rank's old_of_new is the model's, its keys
    are the model's keys over its new range, every replica holds the model's edges, dependency counts and incarnations, and
    the new ranges tile [0, n_total) in rank order.  Mutants that give the tail to the first rank, leave the replicated
    consumers unrenumbered, or let the last rank stop at n_kept each fail.
(2) ShardedScheduler.compact_handles over gloo with world size 2, with a stand-in for the library call: both ranks pass the
    same keep list, the union of what each rank tracks and the caller's list; each rank's host mirror, redirects and retracts
    are renumbered; lo, hi and _mine follow the new ranges."""
import bisect
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

import level_model as LM
import test_sharded_graph_cpu as SG
from compact_model import CompactModel

KEEP = LM.KEY_READY | LM.KEY_VALID | LM.KEY_DONE


class CompactRank(SG.ShardRank):
    """ShardRank with hqs_shard_graph_compact.  `mutant` breaks one rule on purpose: "tail_first" gives the freed tail to the
    first rank (the ranges still tile, shifted), "consumers" leaves the replicated consumers unrenumbered, "no_tail" lets the
    last rank end at n_kept."""

    def __init__(self, lo, hi, n_total, mutant=None):
        super().__init__(lo, hi)
        self.n_total, self.mutant = n_total, mutant

    def compact(self, keep):
        old = sorted(self.gvalid | {int(x) for x in keep})
        new_of = {o: i for i, o in enumerate(old)}
        tail = self.n_total - len(old)

        def new(h):
            if h == self.n_total and self.mutant != "no_tail":
                return self.n_total
            return bisect.bisect_left(old, h)

        lo, hi = new(self.lo), new(self.hi)
        if self.mutant == "tail_first":
            lo, hi = (0 if self.lo == 0 else min(new(self.lo) + tail, self.n_total)), min(new(self.hi) + tail, self.n_total)
        lists = {}
        for p, edges in self.lists.items():
            kept = [(c if self.mutant == "consumers" else new_of[c], g) for c, g in edges if self.waits(c, g)]
            if kept:
                lists[new_of[p]] = kept
        self.lists = lists
        self.key = {new_of[h] - new(self.lo) + lo: v for h, v in self.key.items() if h in new_of}
        self.gvalid = {new_of[h] for h in self.gvalid}
        self.gdeps = {new_of[h]: v for h, v in self.gdeps.items() if h in new_of}
        self.gen = {new_of[h]: v for h, v in self.gen.items() if h in new_of}
        self.lo, self.hi = lo, hi
        return old


def _run(seed, mutant=None):
    """One random sequence; raises AssertionError where a rank departs from the model."""
    rng = np.random.default_rng(seed)
    n_total = 300
    world = 1 + seed % 4
    cuts = SG._cuts(rng, n_total, world)
    if seed % 5 == 1:
        cuts = [0] + [n_total] * world                   # everything on the first rank
    elif seed % 5 == 2:
        cuts = [0] * world + [n_total]                   # everything on the last rank
    single = CompactModel()
    single.classes_set(3)
    ranks = [CompactRank(cuts[r], cuts[r + 1], n_total, mutant) for r in range(world)]

    def live():
        return [h for h in range(single.n_handles) if single.flag(h) & LM.KEY_VALID]

    def check(label):
        assert ranks[0].lo == 0 and ranks[-1].hi == n_total, label
        for a, b in zip(ranks, ranks[1:]):
            assert a.hi == b.lo, (label, a.hi, b.lo)
        edges = sorted((p, c, g) for p, lst in single.lists.items() for c, g in lst)
        valid = set(live())
        for r, m in enumerate(ranks):
            assert sorted((p, c, g) for p, lst in m.lists.items() for c, g in lst) == edges, (label, r)
            assert m.gvalid == valid, (label, r)
            assert {h: m.gdeps.get(h, 0) for h in valid} == {h: single.gdeps.get(h, 0) for h in valid}, (label, r)
            assert {h: g for h, g in m.gen.items() if g} == {h: g for h, g in single.gen.items() if g}, (label, r)
            for h in range(m.lo, m.hi):
                assert m.key.get(h, 0) == single.flag(h) & KEEP, (label, r, h)

    nxt, free, compactions = 0, [], 0
    for step in range(70):
        lv = live()
        k = int(rng.integers(1, 14))
        reuse = [free.pop(int(rng.integers(0, len(free)))) for _ in range(min(len(free), k // 2))]
        fresh = list(range(nxt, min(nxt + k - len(reuse), n_total)))
        nxt += len(fresh)
        hs = reuse + fresh
        if hs:
            rng.shuffle(hs)
            deps = []
            for i, x in enumerate(hs):
                pool = lv[-40:] + hs[:i] + hs[i + 1: i + 3]
                deps.append(sorted({int(pool[j]) for j in rng.integers(0, len(pool), int(rng.integers(0, 4)))} - {x})
                            if pool else [])
            off, flat = SG._csr(deps)
            want = single.graph_push(np.array(hs), rng.integers(0, 3, len(hs)), np.full(len(hs), 5, np.uint64), off, flat)
            assert sum(m.push(hs, off.tolist(), flat.tolist()) for m in ranks) == want, step
            check(f"push {step}")
        lv = live()
        op = rng.random()
        if lv and op < 0.4:
            pick = [int(x) for x in rng.choice(lv, size=min(len(lv), int(rng.integers(1, 5))), replace=False)]
            single.graph_finished(pick)
            for m in ranks:
                m.finished(pick)
            free += sorted(set(pick))
        elif lv and op < 0.55:
            want = single.graph_cancel(lv[:1] + lv[-1:])                    # across rank boundaries
            for m in ranks:
                m.cancel(lv[:1] + lv[-1:])
            free += want
        elif lv and op < 0.65:
            pick = [int(x) for x in rng.choice(lv, size=min(len(lv), 3), replace=False)]
            single.remove(pick)
            for m in ranks:
                m.remove(pick)
            free += pick
        elif op < 0.85 or nxt >= n_total - 10:
            # keep: nothing, or handles in any state (removed and finished ones included), repeated
            n = single.n_handles
            keep = [] if compactions % 3 == 0 or not n else [int(x) for x in rng.integers(0, n, int(rng.integers(1, 8)))]
            want = single.compact(keep)
            for r, m in enumerate(ranks):
                assert m.compact(keep) == want, (step, r)
            compactions += 1
            nxt, free = len(want), []                                       # the freed tail is re-used
        check(f"step {step}")
    assert compactions >= 3
    return compactions


@pytest.mark.parametrize("seed", range(16))
def test_rank_compaction_matches_the_single_context_model(seed):
    _run(seed)


@pytest.mark.parametrize("mutant", ["tail_first", "consumers", "no_tail"])
def test_mutants_are_caught(mutant):
    caught = 0
    for seed in range(16):
        try:
            _run(seed, mutant)
        except AssertionError:
            caught += 1
    assert caught > 0, mutant


# ShardedScheduler.compact_handles over gloo ----------------------------------------------------------------------------
N_TOTAL = 20
VALID = [2, 5, 11, 17]                  # the replicated graph VALID bits, the same on every rank


class _Lib:
    """hqs_shard_graph_compact on one rank, by the rule of the header, over the fixed VALID set; records the keep list."""

    def __init__(self, lo, hi):
        self.lo, self.hi = lo, hi

    def hqs_shard_graph_compact(self, ctx, n, keep, ptr_ref, k_ref, rng):
        self.keep = C.cast(keep, C.POINTER(C.c_uint32))[:n] if n else []
        old = sorted(set(VALID) | set(self.keep))
        self.old = np.array(old, dtype=np.uint32)
        ptr_ref._obj.contents = C.c_uint32.from_buffer(self.old)
        k_ref._obj.value = self.old.size
        new = [N_TOTAL if h == N_TOTAL else bisect.bisect_left(old, h) for h in (self.lo, self.hi)]
        out = C.cast(rng, C.POINTER(C.c_uint32))
        out[0], out[1] = new
        return 0


class _Sched:
    """The part of GpuScheduler that the compaction's host bookkeeping reads and writes."""

    def __init__(self, lib):
        self._lib, self._ctx = lib, None
        self._task_class = np.zeros(0, np.uint32)
        self._task_worker = np.zeros(0, np.int64)
        self._task_variant = np.zeros(0, np.uint8)
        self._task_prio = np.zeros(0, np.uint64)
        self._pf_worker = np.zeros(0, np.int64)
        self.redirects, self._retracting_from = {}, {}
        self._grow_tasks(10)

    def _grow_tasks(self, n):
        m = n - self._task_class.size
        if m > 0:
            self._task_class = np.concatenate([self._task_class, np.zeros(m, np.uint32)])
            self._task_worker = np.concatenate([self._task_worker, np.full(m, -1, np.int64)])
            self._task_variant = np.concatenate([self._task_variant, np.zeros(m, np.uint8)])
            self._task_prio = np.concatenate([self._task_prio, np.zeros(m, np.uint64)])
            self._pf_worker = np.concatenate([self._pf_worker, np.full(m, -1, np.int64)])

    def _check(self, rc):
        assert rc == 0


def _worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from hyperqueue_b200.sharded import ShardedScheduler
    lo, hi = (0, 10) if rank == 0 else (10, 20)
    s = _Sched(_Lib(lo, hi))
    sh = ShardedScheduler(s, rank, world, N_TOTAL, device=None)
    sh.graph = True
    if rank == 0:
        s._task_worker[3], s._task_class[3], s._task_variant[3] = 0, 2, 1     # 3: a started prefilled task, out of the graph
        s._pf_worker[7], s._task_class[7] = 101, 1                            # 7: prefilled on worker 101
        s.redirects[8] = (100, 0)                                             # 8: redirected to worker 100
        s._task_prio[5] = 77
    else:
        s._task_worker[4], s._task_class[4] = 1, 2                            # 14: assigned to worker index 1
        s._retracting_from[6] = 100                                           # 16: being retracted from worker 100
        s._task_prio[7] = 99                                                  # 17
    old = sh.compact_handles(keep=[19, 19])
    ret[rank] = {
        "old": old.tolist(), "keep": list(s._lib.keep), "range": (sh.lo, sh.hi),
        "worker": s._task_worker[:6].tolist(), "pf": s._pf_worker[:6].tolist(), "cls": s._task_class[:6].tolist(),
        "variant": s._task_variant[:6].tolist(), "prio": s._task_prio[:6].tolist(),
        "redirects": dict(s.redirects), "retracting": dict(s._retracting_from),
        "mine": sh._mine([0, 4, 5, 19]).tolist(),
    }
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_compact_handles_over_gloo():
    sock = socket.socket(); sock.bind(("127.0.0.1", 0)); port = sock.getsockname()[1]; sock.close()
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(2, port, ret), nprocs=2, join=True)
    r0, r1 = ret[0], ret[1]
    # what rank 0 tracks (3, 7, 8), what rank 1 tracks (14, 16), the caller's 19: the same list on both ranks
    assert r0["keep"] == r1["keep"] == [3, 7, 8, 14, 16, 19]
    assert r0["old"] == r1["old"] == [2, 3, 5, 7, 8, 11, 14, 16, 17, 19]
    # rank 0 keeps [0, new(10) = 5); rank 1 takes [5, 20), the freed tail [10, 20) included
    assert r0["range"] == (0, 5) and r1["range"] == (5, 20)
    # rank 0: old local 2, 3, 5, 7, 8 are now 0 .. 4
    assert r0["worker"] == [-1, 0, -1, -1, -1, -1] and r0["variant"][1] == 1 and r0["cls"][:4] == [0, 2, 0, 1]
    assert r0["pf"] == [-1, -1, -1, 101, -1, -1] and r0["prio"][2] == 77
    assert r0["redirects"] == {4: (100, 0)} and r0["retracting"] == {}
    # rank 1: old local 1, 4, 6, 7, 9 are now 0 .. 4
    assert r1["worker"] == [-1, 1, -1, -1, -1, -1] and r1["cls"][1] == 2 and r1["prio"][3] == 99
    assert r1["retracting"] == {2: 100} and r1["redirects"] == {}
    assert r0["mine"] == [0, 4] and r1["mine"] == [0, 14]
