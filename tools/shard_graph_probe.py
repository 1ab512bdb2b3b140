"""Task graphs over a sharded ready set on the cfg4 shape (the 500 k-node DAG of tests/workloads.py::make_dag(500_000, 256,
16, seed=0)): host wall time per hqs_shard_graph_push batch and per hqs_shard_graph_finished wave on each of two
HQS_CREATE_SHARE_DEVICE contexts of one GPU (each owning half of the handles, each holding the whole replicated graph),
against hqs_graph_push / hqs_graph_finished on one reference context.  Each timed call ends in its own synchronise, and the
three calls of a batch or a wave take turns going first.  The waves come from the reference's ticks; each wave's union
over the ranks must equal the reference's list.
Prints one JSON line with the card's name and power limit.
Usage: python tools/shard_graph_probe.py [batch]"""
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


def main():
    batch = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000
    import torch
    import workloads as W
    from hyperqueue_b200 import _lib as L
    from hyperqueue_b200 import priority_from_user
    wl = W.make_dag(500_000, 256, 16, seed=0)
    n = wl.n_tasks
    prio = priority_from_user(wl.task_user_priority)
    ref = W.gpu_scheduler(wl, add_tasks=False)
    cuts = [0, n // 2, n]
    ranks = [W.gpu_scheduler(wl, add_tasks=False, flags=L.HQS_CREATE_SHARE_DEVICE) for _ in range(2)]
    lv = np.ascontiguousarray(np.unique(prio))
    for r, s in enumerate(ranks):
        s._sync_classes()
        s._check(s._lib.hqs_levels_add(s._ctx, lv.size, L.ptr(lv)))
        s._check(s._lib.hqs_shard_graph_init(s._ctx, n, cuts[r], cuts[r + 1]))
    names = ["ref", "rank0", "rank1"]

    def order(i):                                    # call i rotates which context goes first
        return names[i % 3:] + names[:i % 3]

    push = {"ref": [], "rank0": [], "rank1": []}
    for lo in range(0, n, batch):
        hi = min(lo + batch, n)
        ds = wl.deps[lo:hi]
        off = np.concatenate([[0], np.cumsum([len(d) for d in ds])]).astype(np.uint32)
        flat = np.array([x for d in ds for x in d], dtype=np.uint32)
        h = np.arange(lo, hi, dtype=np.uint32)
        c = np.ascontiguousarray(wl.task_class[lo:hi], np.uint32)
        p = np.ascontiguousarray(prio[lo:hi])
        for name in order(lo // batch):
            t0 = time.perf_counter()
            if name == "ref":
                ref.submit_tasks(h, c, p, off, flat)
            else:
                s = ranks[int(name[-1])]
                s._check(s._lib.hqs_shard_graph_push(s._ctx, h.size, L.ptr(h), L.ptr(c), L.ptr(p), L.ptr(off),
                                                     L.ptr(flat) if flat.size else None, C.byref(C.c_uint32(0))))
            push[name].append(time.perf_counter() - t0)
    wave = {"ref": [], "rank0": [], "rank1": []}
    waves, left = 0, n
    while left:
        t = np.ascontiguousarray(ref.run_scheduling().assignments["task"])
        ref.tasks_finished(t)                        # the resources go back on the host (not timed)
        lists = {}
        for name in order(waves):
            s = ref if name == "ref" else ranks[int(name[-1])]
            call = s._lib.hqs_graph_finished if name == "ref" else s._lib.hqs_shard_graph_finished
            ptr, k = C.POINTER(C.c_uint32)(), C.c_uint32(0)
            t0 = time.perf_counter()
            s._check(call(s._ctx, t.size, L.ptr(t), C.byref(ptr), C.byref(k)))
            wave[name].append(time.perf_counter() - t0)
            lists[name] = [ptr[i] for i in range(k.value)]
        assert lists["rank0"] + lists["rank1"] == lists["ref"], waves
        left -= t.size
        waves += 1
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    out = {"card": smi[0] if smi else torch.cuda.get_device_name(0), "waves": waves, "batch": batch}
    for name in push:
        out[f"push_ms_median_{name}"] = float(np.median(push[name]) * 1e3)
        v = np.array(wave[name][5:])                 # the first waves load the kernels
        out[f"wave_us_median_{name}"] = float(np.median(v) * 1e6)
        out[f"wave_us_p90_{name}"] = float(np.percentile(v, 90) * 1e6)
    print(json.dumps(out))
    for s in ranks + [ref]:
        s.close()


if __name__ == "__main__":
    main()
