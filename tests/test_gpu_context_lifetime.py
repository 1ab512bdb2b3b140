"""Every buffer a context allocates is freed by hqs_destroy, and no call touches memory it does not own.

A short ctypes script (no torch) drives contexts through every call that allocates, then destroys them all: on its own,
and under compute-sanitizer's memcheck with leak checking.  The same script with one allocation of its own that it never
frees is the positive control: the leak it must report shows that the check can fail.  Under the sanitizer, tick kernels
are launched plainly (HQS_DEBUG_NO_COOP=1, as tools/sanitize.sh does); the grid is one CTA per SM, so its CTAs are still
co-resident.
hqs_graph_cancel is left out: it launches cooperatively whatever HQS_DEBUG_NO_COOP says, and the buffers it uses are
allocated by the graph calls the script makes."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FR = 10_000                 # fractions per resource unit
LEAK_BYTES = 4096           # the positive control's allocation
SANITIZER_ERROR = 7         # exit code of a run with a sanitizer finding


def exercise(leak: bool) -> None:
    from hyperqueue_b200 import _lib as L
    lib = L.load_library()
    cudart = C.CDLL("libcudart.so.12")          # the runtime the library is linked against, already loaded
    ctxs = []

    def ok(ctx, rc):
        if rc:
            raise L.HqsError(rc, (lib.hqs_last_error(ctx) or b"").decode())

    def u32(a):
        return np.ascontiguousarray(a, np.uint32)

    def u64(a):
        return np.ascontiguousarray(a, np.uint64)

    def create(q):
        ctx = C.c_void_p()
        ok(None, lib.hqs_create(C.byref(ctx), 0, 2, 0))
        ctxs.append(ctx)
        if q:
            classes(ctx, q)
        return ctx

    def classes(ctx, q):
        arr = (L.hqs_class * q)()
        for c in range(q):
            arr[c].n_variants = 1
            arr[c].variants[0].amount[0] = (1 + c % 4) * FR
            arr[c].variants[0].amount[1] = (1 + c // 4) * 100
            arr[c].variants[0].weight = 10000
        ok(ctx, lib.hqs_classes_set(ctx, q, arr))

    def push(ctx, h, q, prio):
        h = u32(h)
        ok(ctx, lib.hqs_ready_push(ctx, h.size, L.ptr(h), L.ptr(u32(h % q)), L.ptr(u64(prio))))

    def graph_push(ctx, h, deps_of):
        h = u32(h)
        off = u32(np.concatenate([[0], np.cumsum([len(deps_of(int(t))) for t in h])]))
        deps = u32([d for t in h for d in deps_of(int(t))])
        n = C.c_uint32(0)
        ok(ctx, lib.hqs_graph_push(ctx, h.size, L.ptr(h), L.ptr(u32(h % 2)), L.ptr(u64(np.full(h.size, 5))), L.ptr(off),
                                   L.ptr(deps) if deps.size else None, C.byref(n)))

    def graph_finished(ctx, h):
        h = u32(h)
        ready, n = C.POINTER(C.c_uint32)(), C.c_uint32(0)
        ok(ctx, lib.hqs_graph_finished(ctx, h.size, L.ptr(h), C.byref(ready), C.byref(n)))

    # class tables (grown once), the handle table (grown with its contents), ticks with flat and grouped fetch, a query
    W = 4
    tick = create(2)
    classes(tick, 1024)
    classes(tick, 2)
    workers = np.zeros(W, dtype=L.worker_dtype)
    workers["worker_id"] = np.arange(W)
    workers["remaining_time_ms"] = L.HQS_TIME_INF
    free = u64([[8 * FR, 1_000_000]] * W)
    out = np.zeros(1024, dtype=L.assignment_dtype)
    off = np.zeros(2 * W + 2, np.uint32)
    n = C.c_uint32(0)
    ok(tick, lib.hqs_tick_reserve(tick, W, out.size, 1))
    push(tick, np.arange(100), 2, np.arange(100) % 3)
    ok(tick, lib.hqs_tick(tick, W, L.ptr(workers), L.ptr(free), L.ptr(free), None, out.size, L.ptr(out), C.byref(n), None))
    push(tick, np.arange(100, 200), 2, np.zeros(100))
    ok(tick, lib.hqs_tick_grouped(tick, W, L.ptr(workers), L.ptr(free), L.ptr(free), None, out.size, L.ptr(out), C.byref(n),
                                  off.size, L.ptr(off), None))
    push(tick, np.arange(70_000, 70_100), 2, np.ones(100))
    ok(tick, lib.hqs_query(tick, W, L.ptr(workers), L.ptr(free), L.ptr(free), None, C.byref(n), None, None))

    # more priorities than 8192 groups hold for 1024 classes: coarse levels, pruned on the device, then pruned again
    levels = create(1024)
    push(levels, np.arange(40), 1024, np.arange(40))
    h = u32(np.arange(30))
    ok(levels, lib.hqs_ready_remove(levels, h.size, L.ptr(h)))
    push(levels, np.arange(40, 200), 1024, np.arange(40, 200))

    # a fan-out fills a fresh edge pool; once its root is finished a larger one compacts it; then the table grows
    graph = create(2)
    graph_push(graph, np.arange(3000), lambda t: [0] if t else [])
    graph_finished(graph, [0])
    graph_push(graph, np.arange(3000, 6500), lambda t: [3000] if t > 3000 else [])
    graph_finished(graph, [3000])
    graph_push(graph, [70_000], lambda t: [5000])
    stats = (C.c_uint64 * 4)()
    ok(graph, lib.hqs_graph_debug(graph, stats))
    assert stats[2] >= 1, "the edge pool was never compacted"

    # a DAG loaded twice on one context
    dag = create(2)
    for k in (3, 5):
        cons_off = u32([0, k - 1] + [k - 1] * (k - 1))
        ok(dag, lib.hqs_dag_load(dag, k, L.ptr(u32(np.arange(k) % 2)), L.ptr(u64(np.zeros(k))),
                                 L.ptr(u32([0] + [1] * (k - 1))), L.ptr(cons_off), L.ptr(u32(np.arange(1, k)))))

    # the replicated graph of a sharded ready set, and the tick exchange buffers
    shard = create(2)
    ok(shard, lib.hqs_shard_graph_init(shard, 1000, 0, 500))
    xbuf = C.c_void_p()
    ok(shard, lib.hqs_shard_xbuf(shard, C.byref(xbuf), None))

    if leak:
        p = C.c_void_p()
        assert cudart.cudaMalloc(C.byref(p), C.c_size_t(LEAK_BYTES)) == 0
    for ctx in ctxs:
        lib.hqs_destroy(ctx)
    # leaks are reported when the device's context is torn down
    assert cudart.cudaDeviceReset() == 0


def run_script(prefix, leak: bool):
    import __graft_entry__ as ge
    ge.build()
    cmd = prefix + [sys.executable, os.path.abspath(__file__)] + (["--leak"] if leak else [])
    env = dict(os.environ, HQS_DEBUG_NO_COOP="1") if prefix else None
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    return r.returncode, r.stdout + r.stderr


def test_every_allocating_call_then_destroy():
    rc, log = run_script([], leak=False)
    assert rc == 0, log[-4000:]


def test_destroy_frees_every_buffer():
    tool = shutil.which("compute-sanitizer") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin",
                                                               "compute-sanitizer")
    if not os.path.exists(tool):
        pytest.skip("compute-sanitizer is not installed")
    memcheck = [tool, "--tool", "memcheck", "--leak-check", "full", "--error-exitcode", str(SANITIZER_ERROR)]
    rc, log = run_script(memcheck, leak=True)
    # the sanitizer's own errors (an unsupported device, say), not the findings it reports or the script's exit status
    tool_errors = [ln for ln in log.splitlines() if ln.startswith("========= Error: ") and "terminate successfully" not in ln]
    if tool_errors:
        pytest.skip("compute-sanitizer cannot check this process: " + tool_errors[0])
    assert rc == SANITIZER_ERROR and f"Leaked {LEAK_BYTES} bytes" in log, log[-4000:]
    rc, log = run_script(memcheck, leak=False)
    assert rc == 0 and "ERROR SUMMARY: 0 errors" in log and "Leaked" not in log, log[-4000:]


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    exercise(leak="--leak" in sys.argv)
