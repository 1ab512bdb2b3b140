"""Emit tail of the tick from the measuring build (tools/trace_build.sh, -DHQS_TRACE), in microseconds after the solver
CTA released the emit command: when the last worker CTA saw the command, had staged the group records and the segment
cache, had run the chunk filter, had finished emit_finish and had counted emit_done; when the solver CTA had written the
free vectors and had seen every emit_done.  Plain ticks on pools of up to 512 workers (the wide loop), e.g. the bench shape.
Usage: python tools/trace_emit.py [n_tasks] [n_workers] [n_classes ...]      (HQS_LIB selects another trace build)"""
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from hyperqueue_b200 import _lib as L

L.LIB_PATH = os.path.join(ROOT, "hyperqueue_b200", os.environ.get("HQS_LIB", "libhqsched_b200_trace.so"))
import workloads as WL

WORKER = ["command seen", "staged", "chunk filter", "emit_finish", "emit_done counted"]


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
    w = int(sys.argv[2]) if len(sys.argv) > 2 else 256
    qs = [int(x) for x in sys.argv[3:]] or [16, 1]
    for q in qs:
        wl = WL.make_independent(n, w, q, seed=0, free_scale=1024)
        s = WL.gpu_scheduler(wl)
        for it in range(5):
            s.free = wl.worker_free.copy()
            m = s.run_scheduling()
            d = (C.c_uint64 * 8)()
            s._lib.hqs_debug_read(s._ctx, d)
            f7 = [(d[7] >> (16 * i)) & 0xFFFF for i in range(4)]
            f5 = [(d[5] >> (16 * i)) & 0xFFFF for i in range(4)]
            us = lambda x: f"{x * 16 / 1000:.2f}"
            worker = " | ".join(f"{WORKER[i]} {us(v)}" for i, v in enumerate(f7 + f5[:1]))
            print(f"Q={q} n={n} w={w} path={s.stats()['solver_path']:#x} assigned {m.n_assigned()}: worker CTAs (max, us): {worker} || "
                  f"solver CTA: free vectors {us(f5[1])} | all emit_done seen {us(f5[2])} || CTAs with work {f5[3]}", flush=True)
            s.rearm()
        s.close()


if __name__ == "__main__":
    main()
