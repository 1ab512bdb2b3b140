"""Host wall time of hqs_graph_cancel (a cancelled task with its transitive consumers leaving the device table) against
hqs_ready_remove of the same handle set, the floor: the same keys cleared without the closure.  Each of the 20 timed calls
of a case runs on a freshly submitted graph (the same handles submitted again: a new incarnation each time), from the
call's entry to its return (the call ends in a stream synchronise).  Cases: one task without consumers; a 100 000-task
chain cancelled at its head; a 1 -> 100 000 fan-out; the 55 954 roots of the cfg4 DAG (tests/workloads.py::make_dag(500_000,
256, 16, seed=0)), on which all 500 000 tasks depend.  Prints one JSON line with the card's name and power limit.
Usage: python tools/graph_cancel_probe.py [reps]"""
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


def csr(deps):
    off = np.concatenate([[0], np.cumsum([len(d) for d in deps])]).astype(np.uint32)
    return off, np.array([x for d in deps for x in d], dtype=np.uint32)


def case(s, batches, named, reps):
    """batches: [(handles, classes, priorities, off, flat)] submitted before every call; named: the handles cancelled."""
    from hyperqueue_b200 import _lib as L
    named = np.ascontiguousarray(named, np.uint32)
    ptr, k = C.POINTER(C.c_uint32)(), C.c_uint32(0)
    t_cancel, t_remove, n_left = [], [], None
    for rep in range(reps + 2):                  # the first two load the kernels and size the pool
        for b in batches:
            s.submit_tasks(*b)
        t0 = time.perf_counter()
        s._check(s._lib.hqs_graph_cancel(s._ctx, named.size, L.ptr(named), C.byref(ptr), C.byref(k)))
        t1 = time.perf_counter()
        left = np.ctypeslib.as_array(ptr, shape=(k.value,)).copy()
        assert n_left is None or left.size == n_left
        n_left = left.size
        for b in batches:
            s.submit_tasks(*b)
        t2 = time.perf_counter()
        s._check(s._lib.hqs_ready_remove(s._ctx, left.size, L.ptr(left)))
        t3 = time.perf_counter()
        if rep >= 2:
            t_cancel.append(t1 - t0)
            t_remove.append(t3 - t2)
    f = lambda v, q: float(np.percentile(np.array(v) * 1e3, q))
    return {"left": int(n_left), "cancel_ms_median": f(t_cancel, 50), "cancel_ms_p90": f(t_cancel, 90),
            "ready_remove_ms_median": f(t_remove, 50), "ready_remove_ms_p90": f(t_remove, 90)}


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    import workloads as W
    from hyperqueue_b200 import GpuScheduler, RequestVariant, priority_from_user
    out = {}

    def plain():
        s = GpuScheduler(1)
        s.get_or_create_resource_rq_id([RequestVariant.of({0: W.FR})])
        s.new_workers_bulk(np.array([0], np.uint32), np.array([[64 * W.FR]], np.uint64))
        return s

    def one(h, deps):
        n = len(deps)
        return (np.asarray(h, np.uint32), np.zeros(n, np.uint32), np.full(n, priority_from_user(0), np.uint64)) + csr(deps)

    n = 100_000
    s = plain()
    out["one_task"] = case(s, [one([n + 1], [[]])], [n + 1], reps)
    out["chain_100k"] = case(s, [one(np.arange(n), [[]] + [[i] for i in range(n - 1)])], [0], reps)
    out["fanout_100k"] = case(s, [one(np.arange(n + 1), [[]] + [[0]] * n)], [0], reps)
    s.close()
    wl = W.make_dag(500_000, 256, 16, seed=0)
    prio = priority_from_user(wl.task_user_priority)
    s = W.gpu_scheduler(wl, add_tasks=False)
    batches = []
    for lo in range(0, wl.n_tasks, 10_000):
        hi = min(lo + 10_000, wl.n_tasks)
        batches.append((np.arange(lo, hi, dtype=np.uint32), wl.task_class[lo:hi], prio[lo:hi]) + csr(wl.deps[lo:hi]))
    roots = np.array([t for t, d in enumerate(wl.deps) if not d], np.uint32)
    out["cfg4_roots"] = dict(case(s, batches, roots, reps), named=int(roots.size))
    s.close()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    print(json.dumps({"card": smi[0] if smi else "unknown", "reps": reps, **out}))


if __name__ == "__main__":
    main()
