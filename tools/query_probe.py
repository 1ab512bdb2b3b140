"""Host wall time of the autoalloc what-if query (median of 20 after warm-up), with the card it ran on:
  - hqs_query on one context holding 1 M tasks,
  - the fused sharded query (hqs_shard_query_launch + hqs_query_fetch) on two HQS_CREATE_SHARE_DEVICE contexts of one GPU
    holding 500 k tasks each (one query = both launches and both fetches),
  - ShardedScheduler.new_worker_query, one process per GPU (p2p), when the run has at least 2 GPUs,
each with 64, 512 and 1024 fake workers.  Every sharded answer is checked against hqs_query on the union.
Usage: python tools/query_probe.py [--out FILE]"""
import argparse
import ctypes as C
import json
import os
import socket
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import workloads as WL
from hyperqueue_b200 import _lib as L, priority_from_user
from hyperqueue_b200.scheduler import query_workers

N_TASKS = 1_000_000
POOLS = (64, 512, 1024)
REPS, WARMUP = 20, 3
UNIT = np.array([32, 2, 128, 512], dtype=np.uint64) * np.uint64(WL.FR)


def card():
    """(name, power limit) of GPU 0."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def workload():
    return WL.make_independent(N_TASKS, 16, 16, seed=1)


def pool(nw):
    return query_workers(np.tile(UNIT, (nw, 1)))


def median_ms(fn):
    for _ in range(WARMUP):
        fn()
    ts = []
    for _ in range(REPS):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def single_query(s, w, tot):
    n = C.c_uint32(0)
    counts = np.zeros(w.shape[0], dtype=np.uint32)
    s._check(s._lib.hqs_query(s._ctx, w.shape[0], L.ptr(w), L.ptr(tot), L.ptr(tot), None, C.byref(n), L.ptr(counts), None))
    return int(n.value), counts


def fused_parts(wl):
    prio = priority_from_user(wl.task_user_priority)
    lv = np.ascontiguousarray(np.unique(prio))
    parts, xb = [], (C.c_void_p * 2)()
    for r, (lo, hi) in enumerate([(0, N_TASKS // 2), (N_TASKS // 2, N_TASKS)]):
        s = WL.gpu_scheduler(wl, add_tasks=False, flags=L.HQS_CREATE_SHARE_DEVICE)
        s._sync_classes()
        s._check(s._lib.hqs_levels_add(s._ctx, lv.size, L.ptr(lv)))
        s.add_ready_tasks(np.arange(hi - lo, dtype=np.uint32), wl.task_class[lo:hi], prio[lo:hi])
        p = C.c_void_p()
        s._check(s._lib.hqs_shard_xbuf(s._ctx, C.byref(p), None))
        xb[r] = p
        parts.append(s)
    for r, s in enumerate(parts):
        s._check(s._lib.hqs_shard_attach(s._ctx, 2, r, xb))
        s._check(s._lib.hqs_tick_reserve(s._ctx, max(POOLS), N_TASKS // 2, 0))
    return parts


def fused_query(parts, w, tot):
    for s in parts:
        s._check(s._lib.hqs_shard_query_launch(s._ctx, w.shape[0], L.ptr(w), L.ptr(tot), L.ptr(tot), None))
    res = []
    for s in parts:
        n = C.c_uint32(0)
        counts = np.zeros(w.shape[0], dtype=np.uint32)
        s._check(s._lib.hqs_query_fetch(s._ctx, C.byref(n), L.ptr(counts), None))
        res.append((int(n.value), counts))
    return res


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _rank(rank, world, port, ret):
    import torch.distributed as dist
    from hyperqueue_b200.sharded import ShardedScheduler
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    wl = workload()
    sh = ShardedScheduler(WL.gpu_scheduler(wl, add_tasks=False, device=rank), rank, world, N_TASKS,
                          torch.device("cuda", rank), p2p=True)
    sh.add_ready_tasks(np.arange(N_TASKS), wl.task_class, priority_from_user(wl.task_user_priority))
    out = {}
    for nw in POOLS:
        tot = np.tile(UNIT, (nw, 1))
        out[nw] = (median_ms(lambda: sh.new_worker_query(tot)), int(sh.new_worker_query(tot)[2]))
    ret[rank] = out
    dist.barrier()
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("query_probe: no CUDA device")
    name, power = card()
    wl = workload()
    single = WL.gpu_scheduler(wl)
    parts = fused_parts(wl)
    rows = []
    for nw in POOLS:
        w, tot = pool(nw)
        want = single_query(single, w, tot)
        for n, counts in fused_query(parts, w, tot):
            assert n == want[0] and np.array_equal(counts, want[1]), nw
        rows.append({"workers": nw, "n_would_assign": want[0],
                     "hqs_query_1M_ms": median_ms(lambda: single_query(single, w, tot)),
                     "fused_2x500k_one_gpu_ms": median_ms(lambda: fused_query(parts, w, tot))})
    for s in parts:
        s.close()
    single.close()
    sharded = "not measured (needs at least 2 GPUs)"
    if torch.cuda.device_count() >= 2:
        import torch.multiprocessing as mp
        mgr = mp.Manager(); ret = mgr.dict()
        world = torch.cuda.device_count()
        mp.spawn(_rank, args=(world, _free_port(), ret), nprocs=world, join=True)
        sharded = {f"{nw} workers": {"rank0_ms": ret[0][nw][0], "n_would_assign": ret[0][nw][1]} for nw in POOLS}
        sharded["world"] = world
    report = {"card": name, "power_limit": power, "reps": REPS, "warmup": WARMUP, "rows": rows,
              "sharded_scheduler_one_process_per_gpu": sharded}
    print(f"card: {name}, power limit {power}; host wall time per query, median of {REPS} after {WARMUP} warm-up")
    print(f"{'workers':>8} {'tasks assigned':>15} {'hqs_query 1M (ms)':>18} {'fused 2x500k, one GPU (ms)':>27}")
    for r in rows:
        print(f"{r['workers']:>8} {r['n_would_assign']:>15} {r['hqs_query_1M_ms']:>18.3f} {r['fused_2x500k_one_gpu_ms']:>27.3f}")
    print(f"ShardedScheduler, one process per GPU: {sharded}")
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
