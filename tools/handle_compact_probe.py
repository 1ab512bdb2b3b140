"""What dead handles cost the tick, and what hqs_handles_compact costs, on the cfg2-M1 shape (1 M ready tasks, 256 workers,
16 classes, tests/workloads.py::make_independent(seed=0, free_scale=1024)).  For D = 0, 4 M and 15 M retired handles the
live tasks sit behind D handles that were pushed and removed (as a long-running server's finished tasks are), and three
contexts are timed: the table before compaction, the same table after hqs_handles_compact, and a fresh context loaded with
only the live tasks.  Tick time: the tick kernel between two CUDA events (hqs_set_profile, hqs_get_kernel_ms()[3]), median
of `reps` ticks after one warm-up, re-armed in between; every tick must assign the same number of tasks.  Compaction: host
wall time of the call (it ends in a stream synchronise) and its device time between two CUDA events on the context's
stream (hqs_set_stream onto a torch stream), each on its own freshly built table.  Prints one JSON line with the card's
name and power limit, read in the same run.
Usage: python tools/handle_compact_probe.py [reps]"""
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


def build(wl, dead, stream=None):
    import workloads as W
    from hyperqueue_b200 import priority_from_user
    s = W.gpu_scheduler(wl, add_tasks=False)
    if stream is not None:
        s._check(s._lib.hqs_set_stream(s._ctx, C.c_void_p(stream)))
    if dead:
        s.add_ready_tasks(np.arange(dead, dtype=np.uint32), np.zeros(dead, np.uint32), np.zeros(dead, np.uint64))
        s.remove_ready_tasks(np.arange(dead, dtype=np.uint32))
    s.add_ready_tasks(np.arange(dead, dead + wl.n_tasks, dtype=np.uint32), wl.task_class,
                      priority_from_user(wl.task_user_priority))
    return s


def tick_ms(s, wl, reps):
    s._check(s._lib.hqs_set_profile(s._ctx, 1))
    out, assigned = [], set()
    for i in range(reps + 1):
        s.free = wl.worker_free.copy()
        m = s.run_scheduling()
        ms = (C.c_float * 4)()
        s._check(s._lib.hqs_get_kernel_ms(s._ctx, ms))
        if i:
            out.append(float(ms[3]))
        assigned.add(m.n_assigned())
        s.rearm()
    assert len(assigned) == 1, assigned
    return float(np.median(out)), assigned.pop()


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    import torch
    import workloads as W
    wl = W.make_independent(1_000_000, 256, 16, seed=0, free_scale=1024)
    torch.cuda.init()
    res = {}
    fresh = build(wl, 0)
    fresh_ms, fresh_n = tick_ms(fresh, wl, reps)
    fresh.close()
    for dead in (0, 4 << 20, 15 << 20):
        s = build(wl, dead)
        before_ms, n0 = tick_ms(s, wl, reps)
        t0 = time.perf_counter()
        old = s.compact_handles()
        wall = (time.perf_counter() - t0) * 1e3
        assert old.size == wl.n_tasks
        after_ms, n1 = tick_ms(s, wl, reps)
        s.close()
        # the compaction's device time, on a table built anew on a torch stream
        st = torch.cuda.Stream()
        s = build(wl, dead, st.cuda_stream)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(st)
        s.compact_handles()
        e1.record(st)
        torch.cuda.synchronize()
        dev_ms = e0.elapsed_time(e1)
        s.close()
        assert n0 == n1 == fresh_n
        res[f"dead_{dead}"] = {"handles_before": dead + wl.n_tasks, "tick_ms_before": before_ms, "tick_ms_after": after_ms,
                               "tick_ms_fresh": fresh_ms, "assigned": n0, "compact_wall_ms": wall,
                               "compact_device_ms": dev_ms}
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    print(json.dumps({"card": smi[0] if smi else "unknown", "reps": reps, **res}))


if __name__ == "__main__":
    main()
