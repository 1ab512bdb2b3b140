"""What hqs_shard_graph_compact costs, and what it gives back to the fused sharded tick, on the cfg2-M1 shape (1 M ready
tasks, 256 workers, 16 classes, tests/workloads.py::make_independent(seed=0, free_scale=1024)) over 2 and 3
HQS_CREATE_SHARE_DEVICE contexts of one GPU, split evenly.  For D = 4 M and 15 M retired handles the live tasks sit behind D
handles that were pushed through the sharded graph and removed (n_total = D + 1 M), as a long-running server's finished tasks
are.  Sharded tick: fused with 2 ranks (hqs_shard_tick_launch on every rank, then every fetch; each context's cooperative
kernel takes half of the SMs, so 3 fused contexts do not fit on one GPU), unfused with 3 (hqs_shard_count on every rank, the
summed counts, hqs_shard_solve_emit and the fetch); host wall time of the whole tick, median of `reps` ticks after one warm-up, before and after the compaction; every tick must assign the same number of tasks.  Compaction: each
rank's call, its host wall time and the span between two CUDA events on its stream (hqs_set_stream onto a torch stream).
Prints one JSON line with the card's name and power limit, read in the same run.
Usage: python tools/shard_compact_probe.py [reps]"""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def build(wl, dead, world, streams):
    import workloads as W
    from hyperqueue_b200 import _lib as L, priority_from_user
    n_total = dead + wl.n_tasks
    cuts = [n_total * r // world for r in range(world + 1)]
    ranks = [W.gpu_scheduler(wl, add_tasks=False, flags=L.HQS_CREATE_SHARE_DEVICE) for _ in range(world)]
    prio = priority_from_user(wl.task_user_priority)
    lv = np.ascontiguousarray(np.unique(np.concatenate([prio, np.zeros(1, np.uint64)])))
    for r, s in enumerate(ranks):
        s._check(s._lib.hqs_set_stream(s._ctx, C.c_void_p(streams[r].cuda_stream)))
        s._sync_classes()
        s._check(s._lib.hqs_levels_add(s._ctx, lv.size, L.ptr(lv)))
        s._check(s._lib.hqs_shard_graph_init(s._ctx, n_total, cuts[r], cuts[r + 1]))
    n = C.c_uint32(0)

    def push(h, c, p):
        off = np.zeros(h.size + 1, np.uint32)
        for s in ranks:
            s._check(s._lib.hqs_shard_graph_push(s._ctx, h.size, L.ptr(h), L.ptr(c), L.ptr(p), L.ptr(off), None, C.byref(n)))

    step = 1 << 22
    for lo in range(0, dead, step):
        h = np.arange(lo, min(lo + step, dead), dtype=np.uint32)
        push(h, np.zeros(h.size, np.uint32), np.zeros(h.size, np.uint64))
        for s in ranks:
            s._check(s._lib.hqs_shard_graph_remove(s._ctx, h.size, L.ptr(h)))
    push(np.arange(dead, n_total, dtype=np.uint32), np.ascontiguousarray(wl.task_class, np.uint32), np.ascontiguousarray(prio))
    xb = (C.c_void_p * world)()
    for r, s in enumerate(ranks):
        p = C.c_void_p()
        s._check(s._lib.hqs_shard_xbuf(s._ctx, C.byref(p), None))
        xb[r] = p
    if world == 2:
        for r, s in enumerate(ranks):
            s._check(s._lib.hqs_shard_attach(s._ctx, world, r, xb))
    return ranks, n_total


def tick_ms(ranks, wl, n_total, reps):
    import torch
    from hyperqueue_b200 import _lib as L
    ref = ranks[0]
    w = ref._worker_structs(0.0)
    total = np.ascontiguousarray(ref.total)
    out = np.zeros(n_total, dtype=L.assignment_dtype)
    times, assigned = [], set()
    counts = [torch.zeros(L.HQS_MAX_GROUPS, dtype=torch.int32, device="cuda") for _ in ranks]
    for i in range(reps + 1):
        free = np.ascontiguousarray(wl.worker_free)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if len(ranks) == 2:
            for s in ranks:
                s._check(s._lib.hqs_tick_reserve(s._ctx, w.shape[0], n_total, 0))
            for s in ranks:
                s._check(s._lib.hqs_shard_tick_launch(s._ctx, w.shape[0], L.ptr(w), L.ptr(free), L.ptr(total), None, n_total))
        else:
            ng = C.c_uint32(0)
            for s, cnt in zip(ranks, counts):
                s._check(s._lib.hqs_shard_count(s._ctx, w.shape[0], L.ptr(w), L.ptr(free), L.ptr(total), None,
                                                C.c_void_p(cnt.data_ptr()), cnt.numel(), C.byref(ng)))
            allc = torch.stack(counts).sum(0, dtype=torch.int32)
            before = [torch.stack(counts[:r]).sum(0, dtype=torch.int32) if r else torch.zeros_like(allc)
                      for r in range(len(ranks))]
            torch.cuda.synchronize()
            for s, b in zip(ranks, before):
                s._check(s._lib.hqs_shard_solve_emit(s._ctx, C.c_void_p(allc.data_ptr()), C.c_void_p(b.data_ptr()), n_total))
        got = 0
        for s in ranks:
            k = C.c_uint32(0)
            s._check(s._lib.hqs_tick_fetch(s._ctx, n_total, L.ptr(out), C.byref(k), None))
            got += k.value
        if i:
            times.append((time.perf_counter() - t0) * 1e3)
        assigned.add(got)
        for s in ranks:
            s.rearm()
    assert len(assigned) == 1, assigned
    return float(np.median(times)), assigned.pop()


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    import torch
    import workloads as W
    from hyperqueue_b200 import _lib as L
    wl = W.make_independent(1_000_000, 256, 16, seed=0, free_scale=1024)
    torch.cuda.init()
    res = {}
    for world in (2, 3):
        for dead in (4 << 20, 15 << 20):
            streams = [torch.cuda.Stream() for _ in range(world)]
            ranks, n_total = build(wl, dead, world, streams)
            before, n0 = tick_ms(ranks, wl, n_total, reps)
            calls = []
            for s, st in zip(ranks, streams):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record(st)
                t0 = time.perf_counter()
                ptr, k, rng = C.POINTER(C.c_uint32)(), C.c_uint32(0), np.zeros(2, np.uint32)
                s._check(s._lib.hqs_shard_graph_compact(s._ctx, 0, None, C.byref(ptr), C.byref(k), L.ptr(rng)))
                wall = (time.perf_counter() - t0) * 1e3
                e1.record(st)
                torch.cuda.synchronize()
                assert k.value == wl.n_tasks
                calls.append({"wall_ms": wall, "device_ms": e0.elapsed_time(e1), "new_range": rng.tolist()})
            after, n1 = tick_ms(ranks, wl, n_total, reps)
            assert n0 == n1
            res[f"world_{world}_dead_{dead}"] = {"n_total": n_total, "tick_ms_before": before, "tick_ms_after": after,
                                                 "assigned": n0, "compact": calls}
            for s in ranks:
                s.close()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    print(json.dumps({"card": smi[0] if smi else "unknown", "reps": reps, **res}))


if __name__ == "__main__":
    main()
