"""Readiness propagation on the cfg4 shape (the 500 k-node DAG of tests/workloads.py::make_dag(500_000, 256, 16, seed=0)):
device time per completion wave of hqs_graph_finished against hqs_tasks_finished (CUDA events around each call on the
context's stream, from the call's entry to its end: the host's checks, the upload of the finished handles, the kernels
and the copy of the result; the resources go back on the host outside the window), and host wall time of the
hqs_graph_push batches that submit the DAG (tasks and edges per second).  Both contexts drain the same DAG tick by tick.
Prints one JSON line with the card's name and power limit.
Usage: python tools/graph_probe.py [batch]"""
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
    prio = priority_from_user(wl.task_user_priority)
    a = W.gpu_scheduler(wl)
    b = W.gpu_scheduler(wl, add_tasks=False)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for s, st in zip((a, b), streams):
        s._check(s._lib.hqs_set_stream(s._ctx, st.cuda_stream))
    push_s, n_edges = [], 0
    for lo in range(0, wl.n_tasks, batch):
        hi = min(lo + batch, wl.n_tasks)
        ds = wl.deps[lo:hi]
        off = np.concatenate([[0], np.cumsum([len(d) for d in ds])]).astype(np.uint32)
        flat = np.array([x for d in ds for x in d], dtype=np.uint32)
        h = np.arange(lo, hi, dtype=np.uint32)
        b.sync()
        t0 = time.perf_counter()
        b.submit_tasks(h, wl.task_class[lo:hi], prio[lo:hi], off, flat)
        push_s.append(time.perf_counter() - t0)
        n_edges += flat.size
    ms = {"tasks_finished": [], "graph_finished": []}
    waves, left = 0, wl.n_tasks
    while left:
        ma, mb = a.run_scheduling(), b.run_scheduling()
        assert np.array_equal(ma.assignments, mb.assignments), waves
        t = np.ascontiguousarray(ma.assignments["task"])
        n = C.c_uint32(0)
        ptr = C.POINTER(C.c_uint32)()
        calls = (("tasks_finished", a, streams[0], lambda: a._lib.hqs_tasks_finished(a._ctx, t.size, L.ptr(t), C.byref(n))),
                 ("graph_finished", b, streams[1],
                  lambda: b._lib.hqs_graph_finished(b._ctx, t.size, L.ptr(t), C.byref(ptr), C.byref(n))))
        for name, s, st, call in calls:
            s.tasks_finished(t)                      # the resources go back on the host (not timed)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            s._check(call())
            e1.record(st)
            e1.synchronize()
            ms[name].append(e0.elapsed_time(e1))
        left -= t.size
        waves += 1
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    out = {"card": smi[0] if smi else torch.cuda.get_device_name(0), "waves": waves, "batch": batch,
           "push_tasks_per_s": wl.n_tasks / sum(push_s), "push_edges_per_s": n_edges / sum(push_s),
           "push_ms_median": float(np.median(push_s) * 1e3)}
    for name, v in ms.items():
        v = np.array(v[5:])                      # the first waves load the kernels
        out[name + "_us_median"] = float(np.median(v) * 1e3)
        out[name + "_us_mean"] = float(v.mean() * 1e3)
        out[name + "_us_p90"] = float(np.percentile(v, 90) * 1e3)
    print(json.dumps(out))
    a.close()
    b.close()


if __name__ == "__main__":
    main()
