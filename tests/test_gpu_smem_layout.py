"""The solver CTA's shared-memory layout at the limits the ABI documents (1024 workers, 16 resource slots, 4096 classes, 8192
(level x class) groups), checked against the specification.  Every layout that leaves an array in global memory has a case
that asserts its HQS_PATH_* bit: the group list (HQS_PATH_GROUPS_GLOBAL, ticks whose worker state and group list do not fit
together), the narrow remainders (HQS_PATH_REM_GLOBAL), the blocked mask (HQS_PATH_BLOCKED_GLOBAL) and a sharded tick's
per-group counts (HQS_PATH_COUNTS_GLOBAL).  A judged sweep ticks every (workers, resource slots, amount width, proactive
filling, classes) corner at the largest level count the tick takes, and the bench shapes must keep every array in shared
memory.  The specification of a large corner takes tens of seconds on the host, so each is computed once per workload and
shared by the plain, query, grouped and sharded forms."""
import ctypes as C
import copy

import numpy as np
import pytest

import greedy_model as G
import parity as P
from group_model import group_model
from hyperqueue_b200 import _lib as L
from oracle import judge as J

pytestmark = pytest.mark.gpu
FR = P.FR
WIDE = L.HQS_CREATE_WIDE_AMOUNTS
SPILL = (L.HQS_PATH_GROUPS_GLOBAL | L.HQS_PATH_REM_GLOBAL | L.HQS_PATH_BLOCKED_GLOBAL | L.HQS_PATH_COUNTS_GLOBAL
         | L.HQS_PATH_CLASSES_GLOBAL)
# the solver's shared-memory budget: min(227 KB - the tick kernel's static shared memory, 216 KB); tests/test_abi.py checks
# that the statics leave the 216 KB
BUDGET = 216 * 1024


def mandatory_bytes(W, RT, at, Q, L_, pf, groups=True):
    """Restates the mandatory part of solver_layout (hqsched.cu): 16-byte aligned arrays; `groups`: with the group list."""
    up = lambda n: (n + 15) & ~15
    n_pos = (L_ * Q) << pf
    o = sum(up(b) for b in (W * RT * at, W * 4, W * 8, W, W, W * 2, Q * 2, Q))
    if groups:
        o += up(n_pos * 8) + up(n_pos * 4) + (up(n_pos * 4) if pf else 0)
    return o + (2 * up(Q * 4) if pf else 0)


# -------------------------------------------------------------------------------------------------
# workloads
# -------------------------------------------------------------------------------------------------
def _classes(Q, R):
    """Q distinct one-variant classes over R >= 2 resources: resource 0 is the pool's bottleneck, one other resource varies."""
    return [[{"amounts": {0: (1 + c % 2) * FR, 1 + (c // 2) % (R - 1): (1 + c // (2 * (R - 1))) * 100}}] for c in range(Q)]


def _pool(W, R, rng, lo, hi):
    """Worker w has room for lo..hi units of resource 0 (plus a remainder below the gcd of the requests, so the narrow
    solver carries per-worker remainders); the other resources are ample except the last, which binds now and then."""
    total = np.full((W, R), 1000 * FR + 37, dtype=np.uint64)
    total[:, 0] = rng.integers(lo, hi + 1, W).astype(np.uint64) * np.uint64(FR) + np.uint64(37)
    total[:, R - 1] = rng.integers(30, 200, W).astype(np.uint64) * np.uint64(FR) + np.uint64(11)
    return total


def corner(W, R, Q, L_, per_group, seed, lo=10, hi=22, first=None):
    """per_group tasks in every (level, class) group, handles shuffled over the groups; `first` tasks of class 0 at the top
    level come first (the batch of a warm-up tick)."""
    rng = np.random.default_rng(seed)
    total = _pool(W, R, rng, lo, hi)
    lvl = np.repeat(np.arange(L_), Q * per_group)
    cls = np.tile(np.repeat(np.arange(Q), per_group), L_)
    perm = rng.permutation(lvl.size)
    lvl, cls = lvl[perm], cls[perm]
    if first:
        lvl = np.concatenate([np.full(first, L_ - 1), lvl])
        cls = np.concatenate([np.zeros(first, dtype=cls.dtype), cls])
    return P.Workload(R, _classes(Q, R), total, total.copy(), cls.astype(np.uint32), lvl.astype(np.int32),
                      name=f"corner W={W} R={R} Q={Q} L={L_}")


WORKLOADS = {
    # (a) 1024 workers x 16 resource slots x u64 x 8192 groups (Q = 2, 4096 levels): 245 792 B with the group list
    "a": lambda: corner(1024, 12, 2, 4096, 2, seed=1),
    # (b) the same with 4096 classes and 2 levels: 258 048 B
    "b": lambda: corner(1024, 12, 4096, 2, 2, seed=2),
    # (c) proactive filling, Q = 2, 2048 levels (16 B per list entry): 278 592 B; 600 tasks of class 0 for the warm-up tick
    "c": lambda: corner(1024, 12, 2, 2048, 4, seed=3, first=600),
    # (d) proactive filling, Q = 4096, one level, 512 workers: 249 856 B
    "d": lambda: corner(512, 12, 4096, 1, 4, seed=4, lo=20, hi=44, first=300),
    # 1024 workers x 8 slots x u32 x 8192 groups: everything fits but a sharded tick's counts (2 x 32 KB)
    "counts": lambda: corner(1024, 6, 2, 4096, 2, seed=5),
}
_WL, _SPEC = {}, {}


def workload(name):
    if name not in _WL:
        _WL[name] = WORKLOADS[name]()
    return _WL[name]


def spec(name):
    """(assignments, free_after) of one tick over the whole ready set, computed once per workload."""
    if name not in _SPEC:
        wl = workload(name)
        _SPEC[name] = G.model_tick(wl, np.ones(wl.n_tasks, dtype=bool), wl.worker_free.copy())
    return _SPEC[name]


def blocked_workload():
    """1024 workers x 200 classes (3 variants) over 2 levels: the blocked mask alone is 200 KB."""
    rng = np.random.default_rng(6)
    W, Q, R = 1024, 200, 4
    classes = [[{"amounts": {0: (1 + v) * FR, 1 + v: (1 + c) * 100}} for v in range(3)] for c in range(Q)]
    total = _pool(W, R, rng, 2, 6)
    blocked = np.zeros((W, Q, P.MAXV), dtype=bool)
    blocked[:, :, :3] = rng.random((W, Q, 3)) < 0.05
    n = 6000
    return P.Workload(R, classes, total, total.copy(), rng.integers(0, Q, n).astype(np.uint32),
                      rng.integers(0, 2, n).astype(np.int32), blocked, name="blocked 1024 x 200")


# -------------------------------------------------------------------------------------------------
# drivers
# -------------------------------------------------------------------------------------------------
def _judged(wl, free_before, a, free_after):
    """Feasibility judge and exact replay of the free vectors (prefill records take nothing)."""
    a = a[a["kind"] != 1]
    res = P.judge_tick(wl, free_before, a)
    assert res.ok, res
    amounts, allm, _, _ = wl.class_tables()
    exp = J.replay_free_after(amounts, allm, free_before, wl.worker_total, wl.task_class, a["task"], a["worker"], a["variant"])
    assert np.array_equal(exp, free_after), "free_after differs from the exact replay"


def _tick_exact(s, exp, exp_free, must, grouped=False):
    m = s.run_scheduling_grouped() if grouped else s.run_scheduling()
    path = s.stats()["solver_path"]
    got = m.records if grouped else m.assignments
    want = group_model(exp, s.worker_ids.shape[0])[0] if grouped else exp
    assert got.shape == want.shape and np.array_equal(got, want), (got.size, want.size, hex(path))
    assert np.array_equal(m.free_after, exp_free)
    if grouped:
        assert np.array_equal(m.worker_off, group_model(exp, s.worker_ids.shape[0])[1])
    assert path & must == must, hex(path)
    return m, path


def _shard(wl, lo, hi):
    w2 = copy.copy(wl)
    w2.task_class = wl.task_class[lo:hi]
    w2.task_user_priority = wl.task_user_priority[lo:hi]
    return w2


def sharded_tick(wl, flags):
    """Fused sharded tick over two contexts of one GPU, each on half of the SMs, the table block-split by handle.  A rank
    is launched only after the previous rank's launch returned success, so no rank waits for a peer that never started.
    Returns the merged records (rank order, global handles), every rank's free_after and solver_path."""
    from hyperqueue_b200 import priority_from_user
    from hyperqueue_b200.sharded import block_range
    n, w = wl.n_tasks, wl.n_workers
    parts = []
    try:
        xb = (C.c_void_p * 2)()
        lv = np.ascontiguousarray(np.unique(priority_from_user(wl.task_user_priority)))
        for r in range(2):
            lo, hi = block_range(n, r, 2)
            s = P.gpu_scheduler(_shard(wl, lo, hi), add_tasks=False, flags=flags | L.HQS_CREATE_SHARE_DEVICE)
            parts.append((s, lo, hi))
            s._sync_classes()
            s._check(s._lib.hqs_levels_add(s._ctx, lv.size, L.ptr(lv)))
            s.add_ready_tasks(np.arange(hi - lo, dtype=np.uint32), wl.task_class[lo:hi],
                              priority_from_user(wl.task_user_priority[lo:hi]))
            p = C.c_void_p()
            s._check(s._lib.hqs_shard_xbuf(s._ctx, C.byref(p), None))
            xb[r] = p
        for r, (s, lo, hi) in enumerate(parts):
            s._check(s._lib.hqs_shard_attach(s._ctx, 2, r, xb))
            s._check(s._lib.hqs_tick_reserve(s._ctx, w, hi - lo, 0))
        workers = parts[0][0]._worker_structs(0.0)
        free = np.ascontiguousarray(wl.worker_free)
        total = np.ascontiguousarray(wl.worker_total)
        for s, lo, hi in parts:
            s._check(s._lib.hqs_shard_tick_launch(s._ctx, w, L.ptr(workers), L.ptr(free), L.ptr(total), None, hi - lo))
        merged, frees, paths = [], [], []
        for s, lo, hi in parts:
            out = np.zeros(hi - lo, dtype=L.assignment_dtype)
            nn = C.c_uint32(0)
            fa = np.zeros_like(free)
            s._check(s._lib.hqs_tick_fetch(s._ctx, hi - lo, L.ptr(out), C.byref(nn), L.ptr(fa)))
            a = out[: nn.value].copy()
            a["task"] += np.uint32(lo)
            merged.append(a)
            frees.append(fa)
            paths.append(s.stats()["solver_path"])
        return merged, frees, paths, [(lo, hi) for _, lo, hi in parts]
    finally:
        for s, _, _ in parts:
            s.close()


def _check_sharded(name, flags, must, must_not=0):
    wl = workload(name)
    exp, exp_free = spec(name)
    merged, frees, paths, ranges = sharded_tick(wl, flags)
    for a, fa, path, (lo, hi) in zip(merged, frees, paths, ranges):
        assert path & must == must and path & must_not == 0, hex(path)
        assert np.array_equal(fa, exp_free)
        sel = (exp["task"] >= lo) & (exp["task"] < hi)
        assert np.array_equal(a, exp[sel]), (lo, hi, a.size, int(sel.sum()))
    assert sum(a.size for a in merged) == exp.size


# -------------------------------------------------------------------------------------------------
# the cases: name -> the HQS_PATH_* spill bits the case must reach (tests/test_paths_matrix.py keeps one per bit)
# -------------------------------------------------------------------------------------------------
CASES = {
    "corner_a": L.HQS_PATH_GROUPS_GLOBAL,
    "corner_a_query_grouped": L.HQS_PATH_GROUPS_GLOBAL,
    "corner_b": L.HQS_PATH_GROUPS_GLOBAL,
    "corner_c_prefill": L.HQS_PATH_GROUPS_GLOBAL,
    "corner_d_prefill": L.HQS_PATH_GROUPS_GLOBAL,
    "corner_a_narrow_remainders": L.HQS_PATH_REM_GLOBAL,
    "blocked_mask": L.HQS_PATH_BLOCKED_GLOBAL,
    "sharded_counts": L.HQS_PATH_COUNTS_GLOBAL,
    "sharded_corner_a": L.HQS_PATH_GROUPS_GLOBAL,
}


def _corner_tick(name, flags, must, must_not=0):
    wl = workload(name)
    exp, exp_free = spec(name)
    s = P.gpu_scheduler(wl, flags=flags)
    try:
        _, path = _tick_exact(s, exp, exp_free, must)
        assert path & must_not == 0, hex(path)
        st = s.stats()
        assert st["narrow_amounts"] == (0 if flags & WIDE else 1)
        assert st["n_groups"] == len(np.unique(wl.task_class.astype(np.int64) * 65536 + wl.task_user_priority))
    finally:
        s.close()
    # first-fit walked the whole pool
    assert exp.size > 0 and int(exp["worker"].max()) == wl.n_workers - 1
    assert exp.size < wl.n_tasks


def test_corner_a():
    _corner_tick("a", WIDE, CASES["corner_a"], must_not=L.HQS_PATH_REM_GLOBAL)


def test_corner_a_query_grouped():
    """(a) as hqs_query (per-worker counts of the specification, nothing consumed: a tick afterwards is the specification's)
    and as hqs_tick_grouped."""
    wl = workload("a")
    exp, exp_free = spec("a")
    must = CASES["corner_a_query_grouped"]
    s = P.gpu_scheduler(wl, flags=WIDE)
    try:
        needed, counts, n_total = s.new_worker_query(wl.worker_total)
        assert s.stats()["solver_path"] & must == must
        want = np.bincount(exp["worker"].astype(np.int64), minlength=wl.n_workers)
        assert np.array_equal(counts, want) and n_total == exp.size and np.array_equal(needed, want > 0)
        _tick_exact(s, exp, exp_free, must)
    finally:
        s.close()
    s = P.gpu_scheduler(wl, flags=WIDE)
    try:
        _tick_exact(s, exp, exp_free, must, grouped=True)
    finally:
        s.close()


def test_corner_b():
    _corner_tick("b", WIDE, CASES["corner_b"])


def test_corner_a_narrow_remainders():
    """(a) on 32-bit amounts: the list fits, the remainders (W x 16 x 8 B) do not."""
    _corner_tick("a", 0, CASES["corner_a_narrow_remainders"], must_not=L.HQS_PATH_GROUPS_GLOBAL)


def _prefill_corner(name, first, free_first, prefill=(16, 4)):
    """Tick 1: only the `first` tasks (class 0, top level) on a pool with little room: assignments and prefills.  Tick 2:
    every task, full pool; the prefilled tasks form sub-groups of their own, and the tick redirects some of them (kind 2)
    or prefills again (kind 1).  Both ticks against the specification."""
    from hyperqueue_b200 import priority_from_user
    wl = workload(name)
    n = wl.n_tasks
    prio = priority_from_user(wl.task_user_priority)
    ready = np.zeros(n, dtype=bool)
    ready[:first] = True
    pf = np.full(n, -1, dtype=np.int64)
    exp1, free1 = G.model_tick(wl, ready, free_first.copy(), prefill=prefill, pf_worker=pf)
    assert (exp1["kind"] == 1).sum() > 0 and (pf >= 0).any()
    ready[exp1["task"][exp1["kind"] != 1]] = False
    ready[first:] = True
    exp2, free2 = G.model_tick(wl, ready, wl.worker_free.copy(), prefill=prefill, pf_worker=pf)
    assert (exp2["kind"] != 0).any() and int(exp2["worker"][exp2["kind"] != 1].max()) == wl.n_workers - 1
    s = P.gpu_scheduler(wl, add_tasks=False, flags=WIDE)
    try:
        s.set_prefill(*prefill)
        s.add_ready_tasks(np.arange(first, dtype=np.uint32), wl.task_class[:first], prio[:first])
        s.free = free_first.copy()
        _tick_exact(s, exp1, free1, 0)
        s.add_ready_tasks(np.arange(first, n, dtype=np.uint32), wl.task_class[first:], prio[first:])
        s.free = wl.worker_free.copy()
        _, path = _tick_exact(s, exp2, free2, CASES[f"corner_{name}_prefill"])
        assert s.stats()["narrow_amounts"] == 0
    finally:
        s.close()
    return path


def _little_room(wl, n_room):
    free = wl.worker_free.copy()
    free[:, 0] = np.uint64(37)
    free[:n_room, 0] = np.uint64(2 * FR + 37)
    return free


def test_corner_c_prefill():
    wl = workload("c")
    _prefill_corner("c", 600, _little_room(wl, 128))


def test_corner_d_prefill():
    """(d) reaches the spilled layout in both ticks: Q = 4096 with proactive filling is 8192 groups whatever is ready."""
    wl = workload("d")
    _prefill_corner("d", 300, _little_room(wl, 64), prefill=(0, 4))


def test_blocked_mask():
    wl = blocked_workload()
    exp, exp_free = G.model_tick(wl, np.ones(wl.n_tasks, dtype=bool), wl.worker_free.copy())
    s = P.gpu_scheduler(wl)
    try:
        _, path = _tick_exact(s, exp, exp_free, CASES["blocked_mask"])
        assert path & L.HQS_PATH_GROUPS_GLOBAL == 0 and path & L.HQS_PATH_GENERAL
    finally:
        s.close()
    assert exp.size > 0 and int(exp["worker"].max()) > 900


def test_sharded_counts():
    """1024 workers x 8 slots x u32 x 8192 groups, two ranks: the group list fits, the per-group counts of the ranks do
    not.  The single-context tick at the same shape runs first."""
    _corner_tick("counts", 0, 0, must_not=L.HQS_PATH_GROUPS_GLOBAL | L.HQS_PATH_REM_GLOBAL)
    _check_sharded("counts", 0, CASES["sharded_counts"])


def test_sharded_corner_a():
    """(a) over two ranks: with the group list in global memory, both ranks' counts (2 x 32 KB) fit shared memory."""
    _corner_tick("a", WIDE, L.HQS_PATH_GROUPS_GLOBAL)
    _check_sharded("a", WIDE, CASES["sharded_corner_a"], must_not=L.HQS_PATH_COUNTS_GLOBAL)


# -------------------------------------------------------------------------------------------------
# the judged sweep: every corner at the largest level count the tick takes
# -------------------------------------------------------------------------------------------------
SWEEP = [(W, RT, width, pf, Q) for W in (512, 768, 896, 1024) for RT in (4, 8, 16) for width in ("u32", "u64")
         for pf in (0, 1) for Q in (1, 2, 64, 4096)]


def sweep_workload(W, R, Q, L_, seed):
    """One task per registered level, classes round-robin; every worker has room for 20 or more of them."""
    rng = np.random.default_rng(seed)
    total = _pool(W, R, rng, 40, 48)
    lvl = rng.permutation(L_)
    cls = (np.arange(L_) * 7 + 3) % Q
    return P.Workload(R, _classes(Q, R), total, total.copy(), cls.astype(np.uint32), lvl.astype(np.int32))


@pytest.mark.parametrize("W,RT", sorted({(W, RT) for W, RT, *_ in SWEEP}))
def test_sweep_every_corner_ticks(W, RT):
    for _, _, width, pf, Q in [c for c in SWEEP if c[:2] == (W, RT)]:
        L_ = (L.HQS_MAX_GROUPS >> pf) // Q
        wl = sweep_workload(W, RT, Q, L_, seed=W + RT + Q + pf)
        at = 8 if width == "u64" else 4
        spill = mandatory_bytes(W, RT, at, Q, L_, pf) > BUDGET
        assert mandatory_bytes(W, RT, at, Q, L_, pf, groups=False) <= BUDGET
        s = P.gpu_scheduler(wl, flags=WIDE if width == "u64" else 0)
        tag = (W, RT, width, pf, Q, L_)
        try:
            if pf:
                s.set_prefill(0, 2)
            m = s.run_scheduling()
            st = s.stats()
            assert st["narrow_amounts"] == (width == "u32"), tag
            assert st["n_levels"] == L_ and not st["coarsened"], tag
            assert bool(st["solver_path"] & L.HQS_PATH_GROUPS_GLOBAL) == spill, (tag, hex(st["solver_path"]))
            assert m.n_assigned() == wl.n_tasks, tag            # one task per level: the pool has room for all
            _judged(wl, wl.worker_free, m.assignments, m.free_after)
        finally:
            s.close()


# -------------------------------------------------------------------------------------------------
# the bench shapes keep every array in shared memory
# -------------------------------------------------------------------------------------------------
BENCH_SHAPES = {
    "cfg2": lambda: P.make_independent(20_000, 256, 16, seed=0, free_scale=1024),
    "cfg3": lambda: P.make_independent(20_000, 256, 16, seed=0, free_scale=1, variants3=True, blocked_density=0.05),
    "cfg5_pool": lambda: P.make_independent(20_000, 1024, 16, seed=0, free_scale=4096),
}


@pytest.mark.parametrize("name", list(BENCH_SHAPES))
def test_bench_shapes_keep_the_shared_layout(name):
    wl = BENCH_SHAPES[name]()
    exp, exp_free = G.model_tick(wl, np.ones(wl.n_tasks, dtype=bool), wl.worker_free.copy())
    s = P.gpu_scheduler(wl)
    try:
        _, path = _tick_exact(s, exp, exp_free, 0)
        assert path & SPILL == 0, hex(path)
    finally:
        s.close()
    assert exp.size > 0
