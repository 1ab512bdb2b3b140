"""Measures the per-worker grouped fetch (hqs_tick_grouped) against the flat one at the benchmark's shapes: cfg2-M1 (1 M tasks,
256 workers) and the per-rank shape of cfg5 (1.25 M tasks, 1024 workers), Q = 16, every task assigned in one tick.
  (a) device time of the three grouping kernels (CUDA events on the context stream, hqs_grouped_kernel_ms) next to the tick
      kernel's (hqs_get_kernel_ms);
  (b) host wall time of the C ABI call alone, flat and grouped, with pinned output buffers;
  (c) host wall time of the call plus the construction of the per-worker lists in C++ (hqshim_time_mapping): hqs_tick + one map
      lookup and push_back per record, against hqs_tick_grouped + one bulk append per worker.
Flat and grouped alternate; each number is the median of --reps ticks after --warmup, with the range.  The card and its power
limit are printed with the numbers.  One JSON line at the end."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import hyperqueue_b200._lib as L
from bench import CFG2, CFG5, make_workload
from group_model import group_model
from workloads import gpu_scheduler


def stat(xs):
    xs = np.asarray(xs, dtype=np.float64)
    return {"median": round(float(np.median(xs)), 4), "min": round(float(xs.min()), 4), "max": round(float(xs.max()), 4)}


def probe(cfg, reps, warmup):
    lib, shim = L.load_library(), L.load_shim()
    wl = make_workload(cfg, seed=0)
    s = gpu_scheduler(wl)
    n, nw = wl.n_tasks, wl.n_workers
    workers = s._worker_structs(0.0)
    free, total = np.ascontiguousarray(wl.worker_free), np.ascontiguousarray(wl.worker_total)
    out = torch.empty(n * 8, dtype=torch.uint8).pin_memory().numpy().view(L.assignment_dtype)
    off = np.zeros(2 * nw + 2, dtype=np.uint32)
    out_n = C.c_uint32(0)
    s._check(lib.hqs_set_profile(s._ctx, 1))

    def tick(grouped):
        s._check(lib.hqs_ready_rearm(s._ctx))
        s._check(lib.hqs_sync(s._ctx))
        t0 = time.perf_counter()
        if grouped:
            rc = lib.hqs_tick_grouped(s._ctx, nw, L.ptr(workers), L.ptr(free), L.ptr(total), None, n, L.ptr(out), C.byref(out_n),
                                      off.size, L.ptr(off), None)
        else:
            rc = lib.hqs_tick(s._ctx, nw, L.ptr(workers), L.ptr(free), L.ptr(total), None, n, L.ptr(out), C.byref(out_n), None)
        ms = (time.perf_counter() - t0) * 1e3
        s._check(rc)
        assert out_n.value == n, (out_n.value, n)
        return ms

    # the two fetches return the same records: checked once at this size before anything is timed
    tick(False)
    flat = out[:n].copy()
    tick(True)
    want, want_off = group_model(flat, nw)
    assert np.array_equal(out[:n], want) and np.array_equal(off, want_off)
    for _ in range(warmup):
        tick(False); tick(True)
    wall = {False: [], True: []}
    dev_tick, dev_group = [], []
    ms4 = (C.c_float * 4)()
    g_ms = C.c_float(0)
    for _ in range(reps):
        for grouped in (False, True):
            wall[grouped].append(tick(grouped))
            s._check(lib.hqs_get_kernel_ms(s._ctx, ms4))
            dev_tick.append(ms4[3])
            if grouped:
                s._check(lib.hqs_grouped_kernel_ms(s._ctx, C.byref(g_ms)))
                dev_group.append(g_ms.value)
    s._check(lib.hqs_set_profile(s._ctx, 0))
    # (c) the call + the per-worker lists in C++
    lists = {}
    digests = []
    for grouped in (0, 1, 0, 1):
        ms = np.zeros(warmup + reps, dtype=np.float64)
        dg = C.c_uint64(0)
        s._check(shim.hqshim_time_mapping(s._ctx, nw, L.ptr(workers), L.ptr(free), L.ptr(total), n, grouped, ms.size, L.ptr(ms),
                                          C.byref(dg)))
        lists.setdefault(grouped, []).extend(ms[warmup:].tolist())
        digests.append(dg.value)
    assert len(set(digests)) == 1, digests
    s.close()
    bytes_moved = 2 * 8 * n + 2 * 4 * (2 * nw + 1) * ((n + 4095) // 4096)      # records in and out, the histogram written and read
    return {"shape": cfg["name"], "tasks": n, "workers": nw, "reps": reps,
            "device_ms_tick_kernel": stat(dev_tick), "device_ms_grouping_kernels": stat(dev_group),
            "grouping_bytes": bytes_moved, "grouping_GBps_achieved": round(bytes_moved / (np.median(dev_group) * 1e-3) / 1e9, 1),
            "wall_ms_hqs_tick": stat(wall[False]), "wall_ms_hqs_tick_grouped": stat(wall[True]),
            "wall_ms_tick_plus_lists_flat": stat(lists[0]), "wall_ms_tick_plus_lists_grouped": stat(lists[1])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("grouped_probe needs a CUDA device: nothing is measured without one")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    res = {"card": card, "shapes": [probe(cfg, args.reps, args.warmup) for cfg in (CFG2, CFG5)]}
    for r in res["shapes"]:
        print(json.dumps(r, indent=1))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
