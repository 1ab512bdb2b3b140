"""The autoalloc what-if query over a sharded ready set on the GPU.

Contract: every rank holds the same classes, declared levels, prefill configuration and fake-worker array.  Then every rank
returns the same answer, and it is what hqs_query returns on ONE context holding the union of the ranks' ready sets:
n_would_assign, per-worker counts and free vectors, bit for bit.  Nothing is emitted or consumed on any rank.

The ranks run as contexts of this process: the unfused path (hqs_shard_count, a torch sum of the count vectors,
hqs_shard_query_solve) with 2 and 3 ranks, and the fused path (hqs_shard_query_launch, peer exchange between two
HQS_CREATE_SHARE_DEVICE contexts).  ShardedScheduler.new_worker_query runs as one rank here, and with >= 2 GPUs as one process
per GPU over NCCL and over IPC."""
import ctypes as C
import functools
import os
import socket

import numpy as np
import pytest
import torch

import test_query_spec as T
import workloads as WL
from test_gpu_sharded_prefill import (DRAIN_CLASSES, DRAIN_PREFILL, Ranks, _apply_workers, _crossing_cut, _drain_script,
                                      _drain_setup, _replay, _sched)
from workloads import FR

pytestmark = pytest.mark.gpu

HQS_E_STATE = -6
_gpu_scheduler = WL.gpu_scheduler          # the real one: the spec fixture below replaces the module attribute


def _L():
    from hyperqueue_b200 import _lib as L
    return L


# ---- ranks as contexts of this process -----------------------------------------------------------------------------------
def _make_parts(wl, cuts, flags=0):
    """Rank r owns the tasks [cuts[r], cuts[r + 1]) of `wl` (an empty range is a rank without tasks); every rank has the
    workload's classes and workers and declares every priority level."""
    from hyperqueue_b200 import priority_from_user
    L = _L()
    prio = priority_from_user(wl.task_user_priority)
    lv = np.ascontiguousarray(np.unique(prio))
    parts = []
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        s = _gpu_scheduler(wl, add_tasks=False, flags=flags)
        s._sync_classes()
        s._check(s._lib.hqs_levels_add(s._ctx, lv.size, L.ptr(lv)))
        if hi > lo:
            s.add_ready_tasks(np.arange(hi - lo, dtype=np.uint32), wl.task_class[lo:hi], prio[lo:hi])
        parts.append((s, lo, hi))
    return parts


def _as_ranks(parts, fused):
    """The ranks behind the tick interface of test_gpu_sharded_prefill.Ranks; fused: attached to each other's exchange
    buffers."""
    rk = Ranks.__new__(Ranks)
    rk.L, rk.fused, rk.parts = _L(), fused, parts
    if fused:
        n = len(parts)
        xb = (C.c_void_p * n)()
        for r, (s, _, _) in enumerate(parts):
            p = C.c_void_p()
            s._check(s._lib.hqs_shard_xbuf(s._ctx, C.byref(p), None))
            xb[r] = p
        for r, (s, _, _) in enumerate(parts):
            s._check(s._lib.hqs_shard_attach(s._ctx, n, r, xb))
    return rk


def _launch(rk, w, tot):
    """Launches the sharded query on every rank; returns what must stay alive until the fetch."""
    L = _L()
    nw = w.shape[0]
    if rk.fused:
        # the launches wait for each other on the device: every buffer is allocated before the first one
        for s, lo, hi in rk.parts:
            s._check(s._lib.hqs_tick_reserve(s._ctx, nw, max(hi - lo, 1), 0))
        for s, _, _ in rk.parts:
            s._check(s._lib.hqs_shard_query_launch(s._ctx, nw, L.ptr(w), L.ptr(tot), L.ptr(tot), None))
        return None
    counts = []
    for s, _, _ in rk.parts:
        c = torch.zeros(L.HQS_MAX_GROUPS, dtype=torch.int32, device="cuda")
        ng = C.c_uint32(0)
        s._check(s._lib.hqs_shard_count(s._ctx, nw, L.ptr(w), L.ptr(tot), L.ptr(tot), None,
                                        C.c_void_p(c.data_ptr()), c.numel(), C.byref(ng)))
        counts.append(c)
    all_c = torch.stack(counts).to(torch.int64).sum(0).to(torch.int32)
    torch.cuda.synchronize()
    for s, _, _ in rk.parts:
        s._check(s._lib.hqs_shard_query_solve(s._ctx, C.c_void_p(all_c.data_ptr())))
    return all_c


def _fetch(rk, nw):
    """[(rc, error text, n_would_assign, per-worker counts, free_after)] of every rank."""
    L = _L()
    out = []
    for s, _, _ in rk.parts:
        n = C.c_uint32(0)
        counts = np.zeros(nw, dtype=np.uint32)
        fa = np.zeros((nw, s.R), dtype=np.uint64)
        rc = s._lib.hqs_query_fetch(s._ctx, C.byref(n), L.ptr(counts), L.ptr(fa))
        out.append((rc, (s._lib.hqs_last_error(s._ctx) or b"").decode() if rc else "", int(n.value), counts, fa))
    return out


def _shard_query(rk, w, tot):
    keep = _launch(rk, w, tot)
    res = _fetch(rk, w.shape[0])
    del keep
    return res


def _single_query(s, w, tot):
    """hqs_query on one context: (n_would_assign, per-worker counts, free_after)."""
    L = _L()
    nw = w.shape[0]
    n = C.c_uint32(0)
    counts = np.zeros(nw, dtype=np.uint32)
    fa = np.zeros((nw, s.R), dtype=np.uint64)
    s._check(s._lib.hqs_query(s._ctx, nw, L.ptr(w), L.ptr(tot), L.ptr(tot), None, C.byref(n), L.ptr(counts), L.ptr(fa)))
    return int(n.value), counts, fa


def _assert_same(res, want, tag=""):
    """Every rank succeeded and returned `want` = (n_would_assign, counts, free_after)."""
    n, counts, fa = want
    for r, (rc, text, n_r, c_r, fa_r) in enumerate(res):
        assert rc == 0, (tag, r, text)
        assert n_r == n, (tag, r, n_r, n)
        assert np.array_equal(c_r, counts), (tag, r)
        assert np.array_equal(fa_r, fa), (tag, r)


def _keys(s):
    L = _L()
    n = C.c_uint32(0)
    s._check(s._lib.hqs_debug_keys(s._ctx, 0, None, C.byref(n)))
    k = np.zeros(max(n.value, 1), dtype=np.uint32)
    s._check(s._lib.hqs_debug_keys(s._ctx, k.size, L.ptr(k), None))
    return k[: n.value]


def _pool(nw, unit, seed, extras):
    """A fake pool of nw workers: totals = unit x {1, 2}; with extras, some resources unknown (HQS_AMOUNT_MAX, partial
    descriptors), time limits on some workers and min_utilization on others.  Returns (workers, totals)."""
    from hyperqueue_b200.scheduler import query_workers
    L = _L()
    rng = np.random.default_rng(seed)
    tot = np.tile(np.asarray(unit, dtype=np.uint64), (nw, 1)) * rng.integers(1, 3, size=(nw, 1)).astype(np.uint64)
    rem = mu = None
    if extras:
        tot[rng.random(tot.shape) < 0.15] = L.HQS_AMOUNT_MAX
        rem = np.where(rng.random(nw) < 0.3, rng.uniform(1.0, 500.0, nw), np.inf)
        mu = np.where(rng.random(nw) < 0.2, rng.uniform(0.2, 0.9, nw), 0.0).astype(np.float32)
    return query_workers(tot, rem, mu)


def _cut_points(n, world, cut):
    from hyperqueue_b200.sharded import block_range
    if cut == "even":
        return [block_range(n, r, world)[0] for r in range(world)] + [n]
    if cut == "first":                                     # everything on rank 0, the others hold nothing
        return [0] + [n] * world
    return [0] * world + [n]                               # "last": everything on the last rank


def _split(records):
    return np.concatenate([records[records["kind"] != 1], records[records["kind"] == 1]])


def _check_tick(m, recs, frees, rk, tag):
    """Every rank's records are the single-context tick's records of its handles, order kept; free vectors equal."""
    ra = m.assignments
    for (s, lo, hi), a, fa in zip(rk.parts, recs, frees):
        k = (ra["task"] >= lo) & (ra["task"] < hi)
        assert np.array_equal(a, _split(ra[k])), (tag, lo, hi)
        assert np.array_equal(fa, m.free_after), tag


# ---- 1. every case of tests/test_query_spec.py through the sharded query -------------------------------------------------
class _Tick:
    def __init__(self, n):
        self._n = n

    def n_assigned(self):
        return self._n


class _ShardedStandIn:
    """What test_query_spec.spec_query needs of a GpuScheduler, answered by the ranks: new_worker_query by the sharded query
    (the same answer on every rank), run_scheduling by a sharded tick."""

    def __init__(self, wl, world, fused, cut):
        flags = _L().HQS_CREATE_SHARE_DEVICE if fused else 0
        self.rk = _as_ranks(_make_parts(wl, _cut_points(wl.n_tasks, world, cut), flags), fused)

    @property
    def min_utilization(self):
        return self.rk.parts[0][0].min_utilization

    @min_utilization.setter
    def min_utilization(self, mu):
        for s, _, _ in self.rk.parts:
            s.min_utilization = np.asarray(mu, dtype=np.float32).copy()

    def new_worker_query(self, worker_totals, now=0.0, remaining_s=None, min_utilization=None):
        from hyperqueue_b200.scheduler import query_workers
        w, tot = query_workers(worker_totals, remaining_s, min_utilization)
        res = _shard_query(self.rk, w, tot)
        _, _, n, counts, fa = res[0]
        _assert_same(res, (n, counts, fa))                # every rank gives the same answer
        return counts > 0, counts, n

    def run_scheduling(self):
        recs, _, errs = self.rk.tick()
        assert all(rc == 0 for rc, _ in errs), errs
        return _Tick(sum(int(np.count_nonzero(a["kind"] != 1)) for a in recs))

    def close(self):
        self.rk.close()


_SPEC_MODES = [(world, fused, cut) for world, fused in [(2, False), (3, False), (2, True)] for cut in ("even", "first", "last")]


@pytest.fixture(params=_SPEC_MODES, ids=lambda m: f"w{m[0]}-{'fused' if m[1] else 'unfused'}-{m[2]}")
def sharded_backend(request, monkeypatch):
    world, fused, cut = request.param
    monkeypatch.setattr(T, "_BACKEND", "gpu")
    monkeypatch.setattr(WL, "gpu_scheduler", lambda wl, *a, **kw: _ShardedStandIn(wl, world, fused, cut))
    yield


def _spec_case(fn):
    @functools.wraps(fn)
    def run(*args, **kwargs):
        return fn(*args, **kwargs)
    return pytest.mark.usefixtures("sharded_backend")(run)


for _name in dir(T):
    if _name.startswith("test_"):
        globals()[_name + "_sharded"] = _spec_case(getattr(T, _name))


# ---- 2. larger sets against hqs_query on the union -----------------------------------------------------------------------
_UNIT4 = np.array([128, 8, 512, 2048], dtype=np.uint64) * np.uint64(FR)


@pytest.mark.parametrize("wide", [False, True], ids=["narrow", "wide"])
@pytest.mark.parametrize("world,fused", [(2, False), (3, False), (2, True)])
@pytest.mark.parametrize("n,q,v3,nw,extras", [(200001, 16, False, 1024, False), (200001, 16, True, 512, True),
                                              (100001, 16, False, 512, False), (50000, 8, False, 33, True),
                                              (50000, 8, True, 1, True), (3000, 4, False, 1024, True)])
def test_union_equals_single_context(n, q, v3, nw, extras, world, fused, wide):
    L = _L()
    flags = L.HQS_CREATE_WIDE_AMOUNTS if wide else 0
    wl = WL.make_independent(n, 16, q, seed=13, variants3=v3)
    single = _gpu_scheduler(wl, flags=flags)
    rk = _as_ranks(_make_parts(wl, _cut_points(n, world, "even"), flags | (L.HQS_CREATE_SHARE_DEVICE if fused else 0)), fused)
    try:
        busy = 0
        for seed in range(2):
            w, tot = _pool(nw, _UNIT4 // np.uint64(8), 100 * nw + seed, extras)
            want = _single_query(single, w, tot)
            busy += want[0]
            _assert_same(_shard_query(rk, w, tot), want, (nw, seed))
        assert busy > 0
        # what the query counts is what a real tick over the same workers assigns
        out = np.zeros(n, dtype=L.assignment_dtype)
        n_out = C.c_uint32(0)
        single._check(single._lib.hqs_tick(single._ctx, nw, L.ptr(w), L.ptr(tot), L.ptr(tot), None, n, L.ptr(out),
                                           C.byref(n_out), None))
        assert n_out.value == want[0]
    finally:
        rk.close()
        single.close()


# ---- 3. a dry run: nothing changes on any rank --------------------------------------------------------------------------
@pytest.mark.parametrize("world,fused", [(2, False), (3, False), (2, True)])
def test_query_is_a_dry_run(world, fused):
    L = _L()
    wl = WL.make_independent(30000, 16, 8, seed=4)
    single = _gpu_scheduler(wl)
    rk = _as_ranks(_make_parts(wl, _cut_points(wl.n_tasks, world, "even"), L.HQS_CREATE_SHARE_DEVICE if fused else 0), fused)
    try:
        before = [_keys(s) for s, _, _ in rk.parts]
        w, tot = _pool(64, _UNIT4, 3, True)
        _assert_same(_shard_query(rk, w, tot), _single_query(single, w, tot))
        for (s, _, _), k in zip(rk.parts, before):
            assert np.array_equal(_keys(s), k)
            assert s.stats()["ticks"] == 0                      # a query is not a tick
        m = single.run_scheduling()
        recs, frees, errs = rk.tick()
        assert all(rc == 0 for rc, _ in errs), errs
        assert m.n_assigned() > 0
        _check_tick(m, recs, frees, rk, "tick after the query")
    finally:
        rk.close()
        single.close()


# ---- 4. ticks and queries share the exchange sequence -------------------------------------------------------------------
def test_fused_ticks_and_queries_interleaved():
    L = _L()
    wl = WL.make_independent(60000, 16, 8, seed=9)
    single = _gpu_scheduler(wl)
    rk = _as_ranks(_make_parts(wl, _cut_points(wl.n_tasks, 2, "even"), L.HQS_CREATE_SHARE_DEVICE), True)
    try:
        for step, op in enumerate(["tick", "query", "query", "tick", "query", "tick"]):
            if op == "tick":
                # zero-duration tasks: every worker is free again at each tick, so every tick assigns
                for s in [single] + [p[0] for p in rk.parts]:
                    s.free = wl.worker_free.copy()
                m = single.run_scheduling()
                recs, frees, errs = rk.tick()
                assert all(rc == 0 for rc, _ in errs), (step, errs)
                assert m.n_assigned() > 0
                _check_tick(m, recs, frees, rk, step)
            else:
                w, tot = _pool(48 + step, _UNIT4 // np.uint64(4), step, step == 2)
                _assert_same(_shard_query(rk, w, tot), _single_query(single, w, tot), step)
    finally:
        rk.close()
        single.close()


# ---- 5. proactive filling: a query after every tick of the drain --------------------------------------------------------
class _Both:
    """Replays the drain's host events on the ranks and on a single context at once; returns what the ranks return."""

    def __init__(self, rk, single):
        self.rk, self.single = rk, single

    def on_retract_response(self, w, hs):
        got = self.rk.on_retract_response(w, hs)
        self.single.on_retract_response(w, np.asarray(hs, dtype=np.int64))
        return got

    def tasks_finished(self, h):
        self.rk.tasks_finished(h)
        self.single.tasks_finished(np.asarray(h, dtype=np.uint32))

    def on_task_running_prefilled(self, t, v):
        self.rk.on_task_running_prefilled(t, v)
        self.single.on_task_running_prefilled(t, v)

    def add(self, h, c, p):
        self.rk.add(h, c, p)
        self.single.add_ready_tasks(np.asarray(h, dtype=np.uint32), c, p)

    def dispose_prefill(self, c):
        self.single.dispose_prefill(c)
        return self.rk.dispose_prefill(c)


@pytest.mark.parametrize("world,fused", [(2, False), (3, False), (2, True)])
def test_prefill_drain_with_queries(world, fused):
    script, out, n_all = _drain_script(seed=11)
    _, total, _, _, _, _ = _drain_setup(11)
    cut = _crossing_cut(script, out, n_all)
    cuts = [0, cut, n_all] if world == 2 else [0, cut // 2, cut, n_all]
    rk = Ranks(2, DRAIN_CLASSES, cuts, DRAIN_PREFILL, fused)
    single = _sched(2, DRAIN_CLASSES, 0, DRAIN_PREFILL)
    unit = np.array([8 * FR, 32 * FR], dtype=np.uint64)
    seen = {"busy": 0}
    try:
        _apply_workers(rk, total)
        _apply_workers(single, total)

        def check(tick, m, pfw):
            recs, frees, errs = rk.tick()
            assert all(rc == 0 for rc, _ in errs), errs
            _check_tick(m, recs, frees, rk, tick)
            m1 = single.run_scheduling()
            assert np.array_equal(m1.assignments, m.assignments), tick
            assert np.array_equal(rk.pf_worker(n_all), pfw), tick
            # prefilled tasks count as ready in a query, waiting ones first (both sub-groups of every level)
            w, tot = _pool(40 + tick, unit, tick, tick % 2 == 1)
            want = _single_query(single, w, tot)
            seen["busy"] += int(want[0] > 0)
            _assert_same(_shard_query(rk, w, tot), want, tick)

        _replay(_Both(rk, single), script, out, n_all, check)
    finally:
        rk.close()
        single.close()
    assert seen["busy"] >= 5, seen


# ---- 6. ranks configured differently ------------------------------------------------------------------------------------
def test_fused_query_prefill_mismatch_fails_on_every_rank():
    _, total, cls, prio, n, _ = _drain_setup(5, n=2000, W=32)
    rk = Ranks(2, DRAIN_CLASSES, [0, 1000, n], None, True, prefill_of_rank=[DRAIN_PREFILL, None])
    single = _sched(2, DRAIN_CLASSES, 0, DRAIN_PREFILL)
    unit = np.array([8 * FR, 32 * FR], dtype=np.uint64)
    try:
        for sys_ in (rk, single):
            _apply_workers(sys_, total)
        rk.add(np.arange(n), cls, prio)
        single.add_ready_tasks(np.arange(n, dtype=np.uint32), cls, prio)
        keys = [_keys(s) for s, _, _ in rk.parts]
        w, tot = _pool(24, unit, 1, False)
        res = _shard_query(rk, w, tot)
        for rc, text, n_r, _, _ in res:
            assert rc == HQS_E_STATE and "G=" in text, res
            assert n_r == 0
        for (s, _, _), k in zip(rk.parts, keys):
            assert np.array_equal(_keys(s), k)
        # the same configuration on both ranks: the next query is exact
        rk.parts[1][0].set_prefill(*DRAIN_PREFILL)
        want = _single_query(single, w, tot)
        assert want[0] > 0
        _assert_same(_shard_query(rk, w, tot), want)
    finally:
        rk.close()
        single.close()


# ---- 7. call-sequence errors ---------------------------------------------------------------------------------------------
def _rc_text(s, rc):
    return rc, (s._lib.hqs_last_error(s._ctx) or b"").decode()


def test_call_sequence_errors_single_context():
    L = _L()
    wl = WL.make_independent(20000, 16, 8, seed=2)
    s = _gpu_scheduler(wl)
    ref = _gpu_scheduler(wl)
    try:
        w = s._worker_structs(0.0)
        free, total = np.ascontiguousarray(s.free), np.ascontiguousarray(s.total)
        n = C.c_uint32(0)
        assert s._lib.hqs_query_fetch(s._ctx, C.byref(n), None, None) == HQS_E_STATE          # nothing pending
        # a pending tick: the query calls fail and leave it fetchable
        s._check(s._lib.hqs_tick_launch(s._ctx, w.shape[0], L.ptr(w), L.ptr(free), L.ptr(total), None, wl.n_tasks))
        assert s._lib.hqs_query_fetch(s._ctx, C.byref(n), None, None) == HQS_E_STATE
        rc, text = _rc_text(s, s._lib.hqs_query(s._ctx, w.shape[0], L.ptr(w), L.ptr(free), L.ptr(total), None, C.byref(n),
                                                None, None))
        assert rc == HQS_E_STATE and "has not been fetched" in text
        out = np.zeros(wl.n_tasks, dtype=L.assignment_dtype)
        fa = np.zeros_like(free)
        s._check(s._lib.hqs_tick_fetch(s._ctx, wl.n_tasks, L.ptr(out), C.byref(n), L.ptr(fa)))
        m = ref.run_scheduling()
        assert np.array_equal(out[: n.value], m.assignments) and np.array_equal(fa, m.free_after)
        assert s._lib.hqs_query_fetch(s._ctx, C.byref(n), None, None) == HQS_E_STATE          # fetched: nothing pending
    finally:
        s.close()
        ref.close()


@pytest.mark.parametrize("fused", [False, True])
def test_call_sequence_errors_pending_query(fused):
    L = _L()
    wl = WL.make_independent(20000, 16, 8, seed=2)
    single = _gpu_scheduler(wl)
    rk = _as_ranks(_make_parts(wl, _cut_points(wl.n_tasks, 2, "even"), L.HQS_CREATE_SHARE_DEVICE if fused else 0), fused)
    try:
        s0 = rk.parts[0][0]
        w = s0._worker_structs(0.0)
        free, total = np.ascontiguousarray(s0.free), np.ascontiguousarray(s0.total)
        nw = w.shape[0]
        qw, qtot = _pool(40, _UNIT4, 5, True)
        want = _single_query(single, qw, qtot)
        keep = _launch(rk, qw, qtot)
        n = C.c_uint32(0)
        out = np.zeros(wl.n_tasks, dtype=L.assignment_dtype)
        lib, ctx = s0._lib, s0._ctx
        c = torch.zeros(L.HQS_MAX_GROUPS, dtype=torch.int32, device="cuda")
        ng = C.c_uint32(0)
        # every call that fails while a tick is pending fails the same way while a query is; none launches anything, so
        # no peer waits for it
        calls = {
            "hqs_tick_fetch": lambda: lib.hqs_tick_fetch(ctx, wl.n_tasks, L.ptr(out), C.byref(n), None),
            "hqs_tick_launch": lambda: lib.hqs_tick_launch(ctx, nw, L.ptr(w), L.ptr(free), L.ptr(total), None, wl.n_tasks),
            "hqs_shard_tick_launch": lambda: lib.hqs_shard_tick_launch(ctx, nw, L.ptr(w), L.ptr(free), L.ptr(total), None, 100),
            "hqs_shard_query_launch": lambda: lib.hqs_shard_query_launch(ctx, 40, L.ptr(qw), L.ptr(qtot), L.ptr(qtot), None),
            "hqs_shard_query_solve": lambda: lib.hqs_shard_query_solve(ctx, C.c_void_p(c.data_ptr())),
            "hqs_shard_count": lambda: lib.hqs_shard_count(ctx, nw, L.ptr(w), L.ptr(free), L.ptr(total), None,
                                                           C.c_void_p(c.data_ptr()), c.numel(), C.byref(ng)),
            "hqs_query": lambda: lib.hqs_query(ctx, 40, L.ptr(qw), L.ptr(qtot), L.ptr(qtot), None, C.byref(n), None, None),
            "hqs_debug_keys": lambda: lib.hqs_debug_keys(ctx, 0, None, C.byref(n)),
            "hqs_prefill_config": lambda: lib.hqs_prefill_config(ctx, 0, 0),
        }
        for name, call in calls.items():
            rc, text = _rc_text(s0, call())
            assert rc == HQS_E_STATE, (name, rc, text)
            if name == "hqs_tick_fetch":
                assert "hqs_query_fetch" in text
            elif name.startswith("hqs_shard_") and name.endswith("_launch") and not fused:
                assert "hqs_shard_attach" in text, name          # the unfused ranks are not attached
            else:
                assert "has not been fetched" in text, name
        res = _fetch(rk, 40)
        del keep
        _assert_same(res, want)
        assert all(s.stats()["ticks"] == 0 for s, _, _ in rk.parts)
        assert lib.hqs_query_fetch(ctx, C.byref(n), None, None) == HQS_E_STATE
        # and a tick after all that is exact
        m = single.run_scheduling()
        recs, frees, errs = rk.tick()
        assert all(rc == 0 for rc, _ in errs), errs
        _check_tick(m, recs, frees, rk, "tick after the errors")
    finally:
        rk.close()
        single.close()


# ---- 8. ShardedScheduler.new_worker_query --------------------------------------------------------------------------------
def _sharded_scheduler(wl, rank, world, p2p):
    from hyperqueue_b200 import priority_from_user
    from hyperqueue_b200.sharded import ShardedScheduler
    base = _gpu_scheduler(wl, add_tasks=False, device=rank)
    sh = ShardedScheduler(base, rank, world, wl.n_tasks, torch.device("cuda", rank), p2p=p2p)
    sh.add_ready_tasks(np.arange(wl.n_tasks), wl.task_class, priority_from_user(wl.task_user_priority))
    return sh


def _query_args(seed):
    rng = np.random.default_rng(seed)
    tot = np.tile(_UNIT4 // np.uint64(4), (300, 1))
    tot[rng.random(tot.shape) < 0.1] = _L().HQS_AMOUNT_MAX
    return tot, np.where(rng.random(300) < 0.3, 200.0, np.inf), np.where(rng.random(300) < 0.2, 0.5, 0.0)


@pytest.mark.parametrize("p2p", [False, True])
def test_sharded_scheduler_one_rank(p2p):
    wl = WL.make_independent(40000, 16, 8, seed=6, variants3=True)
    single = _gpu_scheduler(wl)
    sh = _sharded_scheduler(wl, 0, 1, p2p)
    try:
        for seed in range(3):
            tot, rem, mu = _query_args(seed)
            needed, counts, total = sh.new_worker_query(tot, remaining_s=rem, min_utilization=mu)
            n2, c2, t2 = single.new_worker_query(tot, remaining_s=rem, min_utilization=mu)
            assert total == t2 > 0 and np.array_equal(counts, c2) and np.array_equal(needed, n2)
        # and the ready set is untouched: the next sharded tick is the single context's
        a, fa = sh.run_scheduling()
        m = single.run_scheduling()
        assert np.array_equal(a, m.assignments) and np.array_equal(fa, m.free_after)
    finally:
        sh.s.close()
        single.close()


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _query_worker(rank, world, port, p2p, ret):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    wl = WL.make_independent(40000, 16, 8, seed=6, variants3=True)
    sh = _sharded_scheduler(wl, rank, world, p2p)
    got = []
    for seed in range(2):
        tot, rem, mu = _query_args(seed)
        _, counts, total = sh.new_worker_query(tot, remaining_s=rem, min_utilization=mu)
        got.append((counts.tobytes(), total))
    a, _ = sh.run_scheduling()
    ret[rank] = (got, a.tobytes())
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("p2p", [False, True], ids=["nccl", "ipc"])
def test_sharded_scheduler_one_process_per_gpu(p2p):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    L = _L()
    wl = WL.make_independent(40000, 16, 8, seed=6, variants3=True)
    single = _gpu_scheduler(wl)
    try:
        want = []
        for seed in range(2):
            tot, rem, mu = _query_args(seed)
            _, c, t = single.new_worker_query(tot, remaining_s=rem, min_utilization=mu)
            want.append((c.tobytes(), t))
        m = single.run_scheduling()
    finally:
        single.close()
    mgr = mp.Manager(); ret = mgr.dict()
    mp.spawn(_query_worker, args=(2, _free_port(), p2p, ret), nprocs=2, join=True)
    for r in range(2):
        assert ret[r][0] == want, r
    got = np.concatenate([np.frombuffer(ret[r][1], dtype=L.assignment_dtype) for r in range(2)])
    got = got[np.argsort(got["task"], kind="stable")]
    exp = m.assignments[np.argsort(m.assignments["task"], kind="stable")]
    assert np.array_equal(got, exp)
