"""Host wall time of hqs_ready_push on a large table, with exact and with coarse priority levels, for a batch whose
priorities are all registered and for one that brings a single new priority (which registers it: in coarse mode that
prunes over the whole table, rebuilds the level table and re-keys every task).
Usage: python tools/push_probe.py [n_table] [batch] [reps]"""
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    n_table = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
    batch = int(sys.argv[2]) if len(sys.argv) > 2 else 10_000
    reps = int(sys.argv[3]) if len(sys.argv) > 3 else 20
    from hyperqueue_b200 import GpuScheduler, RequestVariant
    for n_prio, mode in ((1000, "exact"), (8000, "coarse")):
        s = GpuScheduler(1)
        for c in range(2):
            s.get_or_create_resource_rq_id([RequestVariant.of({0: (c + 1) * 10_000})])
        rng = np.random.default_rng(0)
        vals = np.arange(1, n_prio + 1, dtype=np.uint64) * np.uint64(1 << 20)
        s.add_ready_tasks(np.arange(n_table, dtype=np.uint32), (np.arange(n_table) % 2).astype(np.uint32),
                          rng.choice(vals, n_table))
        st = s.stats()
        assert st["coarsened"] == (mode == "coarse"), st
        h = np.arange(batch, dtype=np.uint32)            # re-used handles: the table size stays put
        cls = (np.arange(batch) % 2).astype(np.uint32)
        for fresh in (False, True):
            times = []
            for r in range(reps):
                p = rng.choice(vals, batch)
                if fresh:
                    p[0] = np.uint64(r + 1) * np.uint64(1 << 20) + np.uint64(7)   # one priority no task had before
                s.sync()
                t0 = time.perf_counter()
                s.add_ready_tasks(h, cls, p)
                times.append((time.perf_counter() - t0) * 1e3)
            st = s.stats()
            print(f"{mode:6s} table={n_table} batch={batch} new priority={'yes' if fresh else 'no '}: "
                  f"median {np.median(times):.3f} ms, max {np.max(times):.3f} ms (levels {st['n_levels']}, "
                  f"coarsened {st['coarsened']})")
        s.close()


if __name__ == "__main__":
    main()
