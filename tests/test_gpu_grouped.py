"""Per-worker grouping of a tick's records on the device (hqs_tick_fetch_grouped / hqs_tick_grouped, hqs_group.cuh).

Every case runs the same tick on two identically loaded contexts, one fetched flat and one fetched grouped, and requires
grouped == group_model(flat) record for record (tests/group_model.py: a stable sort by worker and kind), the same offset
table, equal free vectors and equal device task tables afterwards."""
import ctypes as C

import numpy as np
import pytest

import prefill_scenarios as S
from group_model import group_keys, group_model
from workloads import FR, Workload, gpu_scheduler, make_independent

pytestmark = pytest.mark.gpu


def _inputs(s):
    from hyperqueue_b200 import _lib as L
    s._sync_classes()
    w = s._worker_structs(0.0)
    return L, w, np.ascontiguousarray(s.free), np.ascontiguousarray(s.total)


def tick_flat(s, out_cap=None):
    L, w, free, total = _inputs(s)
    cap = out_cap or max(s.stats()["n_handles"], 1)
    out = np.zeros(cap, dtype=L.assignment_dtype)
    fa = np.zeros_like(free)
    n = C.c_uint32(0)
    s._check(s._lib.hqs_tick(s._ctx, w.shape[0], L.ptr(w), L.ptr(free), L.ptr(total), None, cap, L.ptr(out), C.byref(n), L.ptr(fa)))
    return out[: n.value].copy(), fa


def tick_grouped(s, out_cap=None):
    L, w, free, total = _inputs(s)
    cap = out_cap or max(s.stats()["n_handles"], 1)
    out = np.zeros(cap, dtype=L.assignment_dtype)
    off = np.full(2 * w.shape[0] + 2, 0xDEADBEEF, dtype=np.uint32)
    fa = np.zeros_like(free)
    n = C.c_uint32(0)
    s._check(s._lib.hqs_tick_grouped(s._ctx, w.shape[0], L.ptr(w), L.ptr(free), L.ptr(total), None, cap, L.ptr(out), C.byref(n),
                                     off.size, L.ptr(off), L.ptr(fa)))
    return out[: n.value].copy(), off, fa


def keys(s):
    from hyperqueue_b200 import _lib as L
    n = max(s.stats()["n_handles"], 1)
    k = np.zeros(n, dtype=np.uint32)
    s._check(s._lib.hqs_debug_keys(s._ctx, n, L.ptr(k), None))
    return k


def check_pair(sf, sg, tag, min_records=0):
    """One tick on both schedulers; returns the flat records."""
    nw = sf.worker_ids.shape[0]
    flat, fa_f = tick_flat(sf)
    got, off, fa_g = tick_grouped(sg)
    want, want_off = group_model(flat, nw)
    assert flat.shape[0] >= min_records, (tag, flat.shape[0])
    assert np.array_equal(off, want_off), (tag, off[:8], want_off[:8])
    assert np.array_equal(got, want), (tag, np.nonzero(got != want)[0][:8])
    assert np.array_equal(fa_f, fa_g) and np.array_equal(keys(sf), keys(sg)), tag
    sf.free, sg.free = fa_f, fa_g
    return flat


def pair(wl, flags=0):
    return gpu_scheduler(wl, flags=flags), gpu_scheduler(wl, flags=flags)


@pytest.mark.parametrize("n,w,free_scale,min_records", [
    (200_000, 256, 1024, 200_000),      # the benchmark's shape, every task assigned: 49 tiles, the last one ragged
    (20_000, 1, 4096, 4097),            # one worker: two keys
    (20_000, 33, 64, 4097),
    (30_000, 512, 16, 4097),
    (30_000, 1024, 16, 4097),           # the largest key set: 2049 keys, 72 KB of shared memory in the scatter step
    (1, 5, 1, 1),                       # one task
    (3_000, 1024, 1, 1),                # fewer records than keys, one ragged tile
])
def test_grouped_equals_the_sorted_flat_stream(n, w, free_scale, min_records):
    sf, sg = pair(make_independent(n, w, 16, seed=n + w, free_scale=free_scale))
    check_pair(sf, sg, (n, w), min_records)
    sf.close(); sg.close()


def test_wide_amounts_context():
    from hyperqueue_b200 import _lib as L
    sf, sg = pair(make_independent(12_000, 40, 16, seed=5, free_scale=64), flags=L.HQS_CREATE_WIDE_AMOUNTS)
    check_pair(sf, sg, "wide", 4097)
    assert sg.stats()["narrow_amounts"] == 0
    sf.close(); sg.close()


def test_empty_ready_set_and_partly_assigned_table():
    wl = make_independent(6_000, 12, 16, seed=3)
    sf, sg = pair(wl)
    for s in (sf, sg):
        s.remove_ready_tasks(np.arange(wl.n_tasks, dtype=np.uint32))
    flat = check_pair(sf, sg, "empty")                      # nothing is ready: no records, an all-zero table
    assert flat.size == 0
    sf.close(); sg.close()
    sf, sg = pair(wl)
    total = 0
    for tick in range(3):                                   # later ticks run over a table that is partly DONE
        flat = check_pair(sf, sg, ("drain", tick), 1)
        total += flat.size
        for s in (sf, sg):
            s.free = s.total.copy()                         # everything has finished
    assert total < wl.n_tasks
    sf.close(); sg.close()


def test_one_worker_takes_everything_and_others_get_nothing():
    total = np.tile(np.array([[12_800 * FR]], dtype=np.uint64), (9, 1))
    free = np.zeros_like(total)
    free[4, 0] = total[4, 0]                                # only worker 4 has room
    wl = Workload(1, [[{"amounts": {0: 1 * FR}}]], total, free, np.zeros(10_000, dtype=np.uint32), np.zeros(10_000, dtype=np.int32))
    sf, sg = pair(wl)
    nw = 9
    flat, _ = tick_flat(sf)
    got, off, _ = tick_grouped(sg)
    assert flat.size == 10_000 and (flat["worker"] == 4).all()
    assert np.array_equal(got, flat)                        # one run: the grouped stream is the flat one
    want = np.zeros(2 * nw + 2, dtype=np.uint32)
    want[2 * 4 + 2:] = 10_000                               # empty runs are equal consecutive offsets
    assert np.array_equal(off, want)
    sf.close(); sg.close()


def _scenario_scheduler(name):
    from hyperqueue_b200 import GpuScheduler, RequestVariant
    reserve, pmax, cpus, steps = S.SCENARIOS[name]
    s = GpuScheduler(1)
    c = s.get_or_create_resource_rq_id([RequestVariant.of({0: cpus * FR})])
    s.set_prefill(reserve, pmax)
    return s, c, steps


@pytest.mark.parametrize("name", sorted(S.SCENARIOS))
def test_prefill_scenarios_every_tick(name):
    """Proactive filling through GpuScheduler: kind 1 before kind 0 inside a worker, kind 2 only in the tail, the same
    messages and the same host bookkeeping as the flat path, on every tick (prefill_many_ticks: five ticks)."""
    from hyperqueue_b200 import priority_from_user
    (sf, c, steps), (sg, _, _) = _scenario_scheduler(name), _scenario_scheduler(name)
    _, spec = S.run_spec(name)
    n_w = n_t = 0
    kinds_seen = set()
    for tick, (new_w, new_t) in enumerate(steps):
        for cp in new_w:
            for s in (sf, sg):
                s.new_worker(50 + n_w, [cp * FR])
            n_w += 1
        if new_t:
            h = np.arange(n_t, n_t + new_t, dtype=np.uint32)
            for s in (sf, sg):
                s.add_ready_tasks(h, np.full(new_t, c, dtype=np.uint32), priority_from_user(np.zeros(new_t)))
            n_t += new_t
        m, g = sf.run_scheduling(), sg.run_scheduling_grouped()
        assert np.array_equal(m.assignments, spec[tick])
        want, want_off = group_model(m.assignments, n_w)
        assert np.array_equal(g.records, want) and np.array_equal(g.worker_off, want_off), (name, tick)
        for w in range(n_w):
            p0, a0, a1 = (int(x) for x in g.worker_off[2 * w: 2 * w + 3])
            assert (g.records["kind"][p0:a0] == 1).all() and (g.records["kind"][a0:a1] == 0).all()
            assert (g.records["worker"][p0:a1] == w).all()
        assert (g.redirects()["kind"] == 2).all() and g.redirects().size == int((m.assignments["kind"] == 2).sum())
        assert g.messages() == m.messages(), (name, tick)
        assert g.n_assigned() == m.n_assigned() and g.n_prefilled() == m.n_prefilled()
        if not (m.assignments["kind"] == 2).any():
            assert g.per_worker() == m.per_worker()
        assert np.array_equal(g.free_after, m.free_after) and np.array_equal(keys(sf), keys(sg))
        assert np.array_equal(sf._pf_worker, sg._pf_worker) and sf.redirects == sg.redirects
        kinds_seen |= set(m.assignments["kind"].tolist())
    if name == "prefill_steal":
        assert kinds_seen == {0, 1, 2}
    sf.close(); sg.close()


@pytest.mark.parametrize("fused", [False, True])
def test_sharded_rank_gets_its_own_records_grouped(fused):
    """Two contexts on one GPU as the ranks of a sharded ready set, with proactive filling: each rank's grouped output is the
    single-context grouped output filtered to the rank's handles, order kept.  Two ticks, the second one with redirects."""
    import torch
    from hyperqueue_b200 import priority_from_user
    from hyperqueue_b200.scheduler import apply_tick_records
    from test_gpu_sharded_prefill import Ranks, _sched
    classes, prefill, n_tasks, cuts = [[{0: 1 * FR}], [{0: 2 * FR}]], (3, 6), 60, [0, 23, 60]
    ref = _sched(1, classes, 0, prefill)
    rk = Ranks(1, classes, cuts, prefill, fused)
    L = rk.L
    rng = np.random.default_rng(11)
    cls = rng.integers(0, 2, n_tasks).astype(np.uint32)
    prio = priority_from_user(np.zeros(n_tasks))
    h = np.arange(n_tasks, dtype=np.uint32)
    ref.add_ready_tasks(h, cls, prio)
    rk.add(h, cls, prio)
    n_w = 0
    kinds_seen = set()
    for tick, new_w in enumerate([[4, 4, 8], [80]]):
        for cp in new_w:
            ref.new_worker(50 + n_w, [cp * FR]); rk.new_worker(50 + n_w, [cp * FR]); n_w += 1
        g = ref.run_scheduling_grouped()
        kinds_seen |= set(g.records["kind"].tolist())
        # the ranks' tick, as ShardedScheduler drives it, with the grouped fetch
        s0 = rk.parts[0][0]
        for s, _, _ in rk.parts:
            s._sync_classes()
        w = s0._worker_structs(0.0)
        free, total = np.ascontiguousarray(s0.free), np.ascontiguousarray(s0.total)
        mask = np.ascontiguousarray(np.bitwise_or.reduce(np.stack([s.prefill_mask() for s, _, _ in rk.parts]), axis=0))
        caps = [2 * (hi - lo) for _, lo, hi in rk.parts]
        for (s, _, _), cap in zip(rk.parts, caps):
            s._check(s._lib.hqs_prefill_state(s._ctx, n_w, L.ptr(mask)))
            # contexts that wait for each other on the device allocate and load everything before the first launch
            s._check(s._lib.hqs_tick_reserve(s._ctx, n_w, cap, 0))
            s._check(s._lib.hqs_grouped_reserve(s._ctx, n_w, cap))
        if fused:
            for (s, _, _), cap in zip(rk.parts, caps):
                s._check(s._lib.hqs_shard_tick_launch(s._ctx, n_w, L.ptr(w), L.ptr(free), L.ptr(total), None, cap))
        else:
            counts = []
            for s, _, _ in rk.parts:
                c = torch.zeros(L.HQS_MAX_GROUPS, dtype=torch.int32, device="cuda")
                s._check(s._lib.hqs_shard_count(s._ctx, n_w, L.ptr(w), L.ptr(free), L.ptr(total), None, C.c_void_p(c.data_ptr()),
                                                c.numel(), None))
                counts.append(c)
            st = torch.stack(counts).to(torch.int64)
            all_c = st.sum(0).to(torch.int32)
            befs = [st[:r].sum(0).to(torch.int32) for r in range(len(counts))]
            torch.cuda.synchronize()
        for r, ((s, lo, hi), cap) in enumerate(zip(rk.parts, caps)):
            if not fused:
                s._check(s._lib.hqs_shard_solve_emit(s._ctx, C.c_void_p(all_c.data_ptr()), C.c_void_p(befs[r].data_ptr()), cap))
            out = np.zeros(cap, dtype=L.assignment_dtype)
            off = np.zeros(2 * n_w + 2, dtype=np.uint32)
            fa = np.zeros_like(free)
            n = C.c_uint32(0)
            s._check(s._lib.hqs_tick_fetch_grouped(s._ctx, cap, L.ptr(out), C.byref(n), off.size, L.ptr(off), L.ptr(fa)))
            a = out[: n.value].copy()
            apply_tick_records(s, a)
            s.free = fa
            a["task"] += np.uint32(lo)
            want = g.records[(g.records["task"] >= lo) & (g.records["task"] < hi)]
            assert np.array_equal(a, want), (tick, r)
            want_off = np.zeros(2 * n_w + 2, dtype=np.uint32)
            want_off[1:] = np.cumsum(np.bincount(group_keys(want, n_w), minlength=2 * n_w + 1))
            assert np.array_equal(off, want_off) and np.array_equal(fa, g.free_after), (tick, r)
    assert kinds_seen == {0, 1, 2}
    ref.close(); rk.close()


def test_errors_leave_the_tick_and_the_ready_set_as_hqs_tick_fetch_does():
    from hyperqueue_b200 import _lib as L
    wl = make_independent(5_000, 6, 16, seed=9, free_scale=8)
    sf, sg = pair(wl)
    lib = sg._lib
    _, w, free, total = _inputs(sg)
    nw, cap = w.shape[0], wl.n_tasks
    out = np.zeros(cap, dtype=L.assignment_dtype)
    off = np.zeros(2 * nw + 2, dtype=np.uint32)
    fa = np.zeros_like(free)
    n = C.c_uint32(7)
    # nothing pending
    assert lib.hqs_tick_fetch_grouped(sg._ctx, cap, L.ptr(out), C.byref(n), off.size, L.ptr(off), L.ptr(fa)) == -6
    # out_cap too small: HQS_E_OVERFLOW, nothing emitted, the ready set intact
    before = keys(sg)
    rc = lib.hqs_tick_grouped(sg._ctx, nw, L.ptr(w), L.ptr(free), L.ptr(total), None, 10, L.ptr(out), C.byref(n), off.size, L.ptr(off), L.ptr(fa))
    assert rc == -5 and n.value == 0 and np.array_equal(keys(sg), before)
    # hqs_tick_grouped checks the offset table before it launches anything
    rc = lib.hqs_tick_grouped(sg._ctx, nw, L.ptr(w), L.ptr(free), L.ptr(total), None, cap, L.ptr(out), C.byref(n), 2 * nw + 1, L.ptr(off), L.ptr(fa))
    assert rc == -1 and np.array_equal(keys(sg), before)
    # off_cap too small / null table: HQS_E_INVALID and the tick stays fetchable, by the grouped fetch ...
    flat, fa_f = tick_flat(sf)
    want, want_off = group_model(flat, nw)
    sg._check(lib.hqs_tick_launch(sg._ctx, nw, L.ptr(w), L.ptr(free), L.ptr(total), None, cap))
    assert lib.hqs_tick_fetch_grouped(sg._ctx, cap, L.ptr(out), C.byref(n), 2 * nw + 1, L.ptr(off), L.ptr(fa)) == -1
    assert lib.hqs_tick_fetch_grouped(sg._ctx, cap, L.ptr(out), C.byref(n), off.size, None, L.ptr(fa)) == -1
    sg._check(lib.hqs_tick_fetch_grouped(sg._ctx, cap, L.ptr(out), C.byref(n), off.size, L.ptr(off), L.ptr(fa)))
    assert np.array_equal(out[: n.value], want) and np.array_equal(off, want_off) and np.array_equal(fa, fa_f)
    # ... and by the flat one
    flat2, _ = tick_flat(sf)                                # the same free vectors again: the next tasks
    sg._check(lib.hqs_tick_launch(sg._ctx, nw, L.ptr(w), L.ptr(free), L.ptr(total), None, cap))
    assert lib.hqs_tick_fetch_grouped(sg._ctx, cap, L.ptr(out), C.byref(n), 0, L.ptr(off), L.ptr(fa)) == -1
    sg._check(lib.hqs_tick_fetch(sg._ctx, cap, L.ptr(out), C.byref(n), L.ptr(fa)))
    assert flat2.size > 0 and np.array_equal(out[: n.value], flat2)
    # a pending query is not a tick: HQS_E_STATE, and the query stays fetchable
    xb = (C.c_void_p * 1)()
    p = C.c_void_p()
    sg._check(lib.hqs_shard_xbuf(sg._ctx, C.byref(p), None))
    xb[0] = p
    sg._check(lib.hqs_shard_attach(sg._ctx, 1, 0, xb))
    sg._check(lib.hqs_shard_query_launch(sg._ctx, nw, L.ptr(w), L.ptr(total), L.ptr(total), None))
    assert lib.hqs_tick_fetch_grouped(sg._ctx, cap, L.ptr(out), C.byref(n), off.size, L.ptr(off), L.ptr(fa)) == -6
    assert b"query" in lib.hqs_last_error(sg._ctx)
    would = C.c_uint32(0)
    sg._check(lib.hqs_query_fetch(sg._ctx, C.byref(would), None, None))
    assert would.value > 0
    sf.close(); sg.close()


def test_kernel_launches_flat_unchanged_grouped_plus_three():
    sf, sg = pair(make_independent(9_000, 20, 16, seed=2, free_scale=4))
    deltas = []
    for s, tick in ((sf, tick_flat), (sg, tick_grouped)):
        k0 = s.stats()["kernel_launches"]
        n = tick(s)[0].size
        deltas.append(s.stats()["kernel_launches"] - k0)
        assert n > 0
    assert deltas[0] == 1 and deltas[1] == deltas[0] + 3      # the tick is one kernel; the grouping is three more
    # a tick without records launches nothing beyond the tick kernel
    sg.free = np.zeros_like(sg.free)
    k0 = sg.stats()["kernel_launches"]
    got, off, _ = tick_grouped(sg)
    assert got.size == 0 and not off.any() and sg.stats()["kernel_launches"] - k0 == 1
    sf.close(); sg.close()


def test_cpp_shim_grouped_selftest():
    """tako_b200::GpuCore::run_scheduling_grouped against run_scheduling on two identically loaded cores: equal mappings, list
    order included, on every tick of a drain and through prefill, retract and redirect."""
    from hyperqueue_b200 import _lib as L
    assert L.load_shim().hqshim_selftest_grouped(0, 0) == 0
