"""Proactive filling in sharded ticks, on the CPU.

(1) The per-rank prefill offsets as the tick kernel computes them (numpy stand-in, in the style of test_sharded_cpu.py): the
    specification's single-context records (greedy_model.model_tick with prefill) are split over N ranks by handle blocks;
    each rank places its records with the kernel's formulas and must reproduce the single-context order filtered to its
    handles: assignments (kind 0 / 2) first, then prefill records (kind 1).
      prefill range of the waiting group g:  [k, k + n_el * ps)    (global ranks, the same on every rank)
      this rank's share:                     max(0, min(k + n_el * ps, bef + loc) - max(k, bef))
      offset of g's records:                 running sum of the shares over the ranges in emission order
      output index of global rank r:         n_assigned_local + offset[g] + (r - max(k, bef))
(2) The OR of the ranks' "worker holds a prefilled task of the class" masks over gloo (sharded.reduce_prefill_mask)."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import greedy_model as G
from workloads import FR, Workload


def _workload(rng, n, w, q):
    classes = [[{"amounts": {0: int(c) * FR}}] for c in range(1, q + 1)]
    total = rng.integers(4, 9, size=(w, 1)).astype(np.uint64) * np.uint64(FR)
    cls = rng.integers(0, q, n).astype(np.uint32)
    prio = rng.choice([0, 0, 0, 1, 2], size=n).astype(np.int32)
    return Workload(1, classes, total, total.copy(), cls, prio)


def _spec_ticks(seed, n_ticks=3):
    """Single-context specification ticks with prefill; yields (ready at tick start, pf_worker at tick start, records)."""
    rng = np.random.default_rng(seed)
    wl = _workload(rng, int(rng.integers(150, 400)), int(rng.integers(2, 7)), int(rng.integers(1, 4)))
    ready = np.ones(wl.n_tasks, dtype=bool)
    pf = np.full(wl.n_tasks, -1, dtype=np.int64)
    free = wl.worker_free.copy()
    reserve, pmax = int(rng.integers(0, 6)), int(rng.integers(1, 12))
    for _ in range(n_ticks):
        ready0, pf0 = ready.copy(), pf.copy()
        a, fa = G.model_tick(wl, ready, free, prefill=(reserve, pmax), pf_worker=pf)
        yield wl, ready0, pf0, a
        ready[a["task"][a["kind"] != 1]] = False
        free = wl.worker_free.copy()              # the tasks of the tick finish: every worker is free again


def _groups(wl, ready, pf0):
    """Group id of every task that is ready at tick start: (level, class, prefilled), -1 otherwise."""
    levels = {int(p): i for i, p in enumerate(np.unique(wl.task_user_priority)[::-1].tolist())}
    lv = np.array([levels[int(p)] for p in wl.task_user_priority], dtype=np.int64)
    g = (lv * len(wl.classes) + wl.task_class.astype(np.int64)) * 2 + (pf0 >= 0)
    return np.where(ready, g, -1)


def _per_rank(wl, ready, pf0, a, cuts):
    """Every rank's records placed with the kernel's formulas, from the single-context records."""
    grp = _groups(wl, ready, pf0)
    # prefill ranges in emission order: the kind-1 records of one group are consecutive ranks behind its assigned ones
    pfa = a[a["kind"] == 1]
    ranges = []                                   # (group, k, length)
    rank_of = np.full(wl.n_tasks, -1, dtype=np.int64)
    for gid in np.unique(grp[grp >= 0]).tolist():
        members = np.nonzero(grp == gid)[0]
        rank_of[members] = np.arange(members.size)
    for t in pfa["task"].tolist():
        gid = int(grp[t])
        if not ranges or ranges[-1][0] != gid:
            ranges.append([gid, int(rank_of[t]), 0])
        assert rank_of[t] == ranges[-1][1] + ranges[-1][2], "the prefill range of a group is contiguous"
        ranges[-1][2] += 1
    assert len({r[0] for r in ranges}) == len(ranges)
    n_groups = int(grp.max()) + 1 if (grp >= 0).any() else 0
    out = []
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        bef = np.bincount(grp[:lo][grp[:lo] >= 0], minlength=n_groups)
        loc = np.bincount(grp[lo:hi][grp[lo:hi] >= 0], minlength=n_groups)
        asg = a[(a["kind"] != 1) & (a["task"] >= lo) & (a["task"] < hi)]         # the existing sharded emit: filtered order
        n_loc = asg.size
        offset, share_sum = {}, 0
        for gid, k, m in ranges:
            b, l = int(bef[gid]), int(loc[gid])
            offset[gid] = share_sum
            share_sum += max(0, min(k + m, b + l) - max(k, b))
        rec = np.zeros(n_loc + share_sum, dtype=a.dtype)
        rec[:n_loc] = asg
        filled = np.zeros(rec.size, dtype=bool)
        filled[:n_loc] = True
        for r in pfa:
            t = int(r["task"])
            if not lo <= t < hi:
                continue
            gid = int(grp[t])
            k = next(rg[1] for rg in ranges if rg[0] == gid)
            oi = n_loc + offset[gid] + (int(rank_of[t]) - max(k, int(bef[gid])))
            assert not filled[oi]
            rec[oi] = r
            filled[oi] = True
        assert filled.all()
        out.append((lo, hi, rec, share_sum))
    return out


def _random_cuts(rng, n, world):
    return [0] + sorted(rng.integers(0, n + 1, world - 1).tolist()) + [n]


@pytest.mark.parametrize("seed", range(12))
def test_local_prefill_offsets_reproduce_the_filtered_single_context_order(seed):
    rng = np.random.default_rng(1000 + seed)
    n_prefill_ticks = 0
    for wl, ready, pf0, a in _spec_ticks(seed):
        pfa = a[a["kind"] == 1]
        n_prefill_ticks += pfa.size > 0
        cut_sets = [_random_cuts(rng, wl.n_tasks, world) for world in (1, 2, 3, 4) for _ in range(6)]
        if pfa.size:
            # cut points at the ends of the prefill ranges and inside them, and right after the last assigned task
            t = np.sort(pfa["task"])
            cut_sets += [[0, int(t[0]), wl.n_tasks], [0, int(t[-1]) + 1, wl.n_tasks], [0, int(t[t.size // 2]), wl.n_tasks],
                         [0, int(t[0]), int(t[-1]) + 1, wl.n_tasks]]
        asg = a[a["kind"] != 1]
        if asg.size:
            cut_sets.append([0, int(asg["task"].max()), wl.n_tasks])
        for cuts in cut_sets:
            ranks = _per_rank(wl, ready, pf0, a, cuts)
            assert sum(s for _, _, _, s in ranks) == pfa.size
            for lo, hi, rec, _ in ranks:
                m = (a["task"] >= lo) & (a["task"] < hi)
                want = np.concatenate([a[m & (a["kind"] != 1)], a[m & (a["kind"] == 1)]])
                assert np.array_equal(rec, want), (seed, cuts, lo, hi)
    assert n_prefill_ticks > 0


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _mask_worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from hyperqueue_b200.sharded import reduce_prefill_mask
    rng = np.random.default_rng(50 + rank)
    mask = (rng.random((37, 5)) < 0.1).astype(np.uint8)
    ret[rank] = (mask.tobytes(), reduce_prefill_mask(mask, world).tobytes())
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_prefill_mask_is_the_or_over_the_ranks(world):
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_mask_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
    masks = [np.frombuffer(ret[r][0], dtype=np.uint8).reshape(37, 5) for r in range(world)]
    want = np.bitwise_or.reduce(np.stack(masks), axis=0)
    assert want.any() and not all(np.array_equal(want, m) for m in masks)
    for r in range(world):
        assert np.array_equal(np.frombuffer(ret[r][1], dtype=np.uint8).reshape(37, 5), want)


def test_prefill_mask_world_one_is_the_local_mask():
    from hyperqueue_b200.sharded import reduce_prefill_mask
    m = np.eye(4, 3, dtype=np.uint8)
    assert np.array_equal(reduce_prefill_mask(m, 1), m)


def _live_worker(rank, world, port, ret):
    """Per-rank live vectors of a declared level table: the OR is what every rank passes to hqs_levels_retain."""
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from hyperqueue_b200.sharded import reduce_or
    rng = np.random.default_rng(70 + rank)
    live = (rng.random(300) < 0.05).astype(np.uint8)
    ret[rank] = (live.tobytes(), reduce_or(live, world).tobytes())
    dist.barrier()
    dist.destroy_process_group()


def test_level_live_vectors_are_or_ed_over_the_ranks():
    world = 2
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_live_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
    lives = [np.frombuffer(ret[r][0], dtype=np.uint8) for r in range(world)]
    want = lives[0] | lives[1]
    assert (lives[0] & ~lives[1]).any() and (lives[1] & ~lives[0]).any()        # each rank alone would drop a live level
    for r in range(world):
        assert np.array_equal(np.frombuffer(ret[r][1], dtype=np.uint8), want)


def test_levels_need_pruning_budget_and_doubling():
    from hyperqueue_b200.sharded import levels_need_pruning
    assert not levels_need_pruning(256, 16, True, 200) and levels_need_pruning(257, 16, True, 200)      # 8192 / (2 * 16)
    assert not levels_need_pruning(512, 16, False, 300) and levels_need_pruning(513, 16, False, 300)    # 8192 / 16
    assert not levels_need_pruning(128, 64, False, 32) and levels_need_pruning(129, 64, False, 100)
    assert not levels_need_pruning(84, 2, False, 10) and levels_need_pruning(85, 2, False, 10)          # 2 * 10 + 64
