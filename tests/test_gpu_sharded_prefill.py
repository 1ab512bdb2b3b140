"""Proactive filling and retract / redirect in sharded ticks on the GPU.

Contract: rank r owns the global handles [lo_r, hi_r); every rank has the same prefill configuration, levels and workers and
is given the same GLOBAL prefill mask.  Then every rank's records equal the single-context tick's records filtered to its
handles with their order kept (assignments, kind 0 / 2, then prefill records, kind 1), every rank's free vectors equal the
single-context ones, and the host bookkeeping (prefilled tasks, redirects) of the ranks together equals the single context's.
The single-context GpuScheduler is the oracle: tests/test_gpu_prefill.py pins it to the specification record by record.

The ranks run as contexts of this process (class Ranks): the unfused path (hqs_shard_count, a torch sum of the count vectors,
hqs_shard_solve_emit) with 2 and 3 ranks, and the fused path (hqs_shard_tick_launch, peer exchange between two
HQS_CREATE_SHARE_DEVICE contexts).  With >= 2 GPUs, ShardedScheduler itself replays the synthetic drain over NCCL."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch

import prefill_scenarios as S
from workloads import FR

pytestmark = pytest.mark.gpu


def _sched(R, classes, flags=0, prefill=None):
    from hyperqueue_b200 import GpuScheduler, RequestVariant
    s = GpuScheduler(R, 0, flags)
    for vs in classes:
        s.get_or_create_resource_rq_id([RequestVariant.of(a) for a in vs])
    s._sync_classes()
    if prefill:
        s.set_prefill(*prefill)
    return s


class Ranks:
    """The ranks of a sharded ready set as contexts of this process; rank r owns the GLOBAL handles [cuts[r], cuts[r + 1])
    (a range may be empty).  The host half follows ShardedScheduler: every rank declares every priority, the prefill mask
    and the live level vectors are OR-ed over the ranks, records are applied to the owner's bookkeeping, host events that
    only the owner can resolve are combined over the ranks, and worker state (free vectors, termination, min-utilisation,
    the blocked mask) is replicated.  Its task calls are GpuScheduler's, with global handles, so that a drain
    (tests/drain_fuzz.py) can drive it like a single context.  `make(flags)`, if given, returns a configured GpuScheduler
    of one rank; otherwise every rank gets the classes and the prefill configuration given here."""

    levels_pruned_at = 0              # declared table size after the last pruning (the same on every rank)

    def __init__(self, R, classes, cuts, prefill, fused, prefill_of_rank=None, make=None, flags=0):
        from hyperqueue_b200 import _lib as L
        self.L, self.fused = L, fused
        flags |= L.HQS_CREATE_SHARE_DEVICE if fused else 0
        self.parts = []
        for r, (lo, hi) in enumerate(zip(cuts[:-1], cuts[1:])):
            pf = prefill if prefill_of_rank is None else prefill_of_rank[r]
            self.parts.append((make(flags) if make else _sched(R, classes, flags, pf), lo, hi))
        if fused:
            n = len(self.parts)
            xb = (C.c_void_p * n)()
            for r, (s, _, _) in enumerate(self.parts):
                p = C.c_void_p()
                s._check(s._lib.hqs_shard_xbuf(s._ctx, C.byref(p), None))
                xb[r] = p
            for r, (s, _, _) in enumerate(self.parts):
                s._check(s._lib.hqs_shard_attach(s._ctx, n, r, xb))

    def close(self):
        for s, _, _ in self.parts:
            s.close()

    def new_worker(self, wid, res):
        for s, _, _ in self.parts:
            s.new_worker(wid, res)

    def add_ready_tasks(self, handles, cls, prio):
        L = self.L
        h = np.asarray(handles, dtype=np.int64)
        lv = np.ascontiguousarray(np.unique(np.asarray(prio, dtype=np.uint64)))
        for s, lo, hi in self.parts:
            s._sync_classes()
            s._check(s._lib.hqs_levels_add(s._ctx, lv.size, L.ptr(lv)))
            m = (h >= lo) & (h < hi)
            if m.any():
                s.add_ready_tasks((h[m] - lo).astype(np.uint32), np.asarray(cls)[m], np.asarray(prio, dtype=np.uint64)[m])

    add = add_ready_tasks             # the name the replays of this module and its importers call

    def remove_ready_tasks(self, handles):
        for s, _, mine in self._mine(handles):
            if mine.size:
                s.remove_ready_tasks(mine.astype(np.uint32))

    def set_blocked_mask(self, mask):
        for s, _, _ in self.parts:
            s.set_blocked_mask(mask)

    def _mine(self, handles):
        h = np.asarray(handles, dtype=np.int64).reshape(-1)
        return [(s, lo, h[(h >= lo) & (h < hi)] - lo) for s, lo, hi in self.parts]

    def tasks_finished(self, handles):
        free0 = self.parts[0][0].free.copy()
        delta = np.zeros_like(free0)
        for s, lo, mine in self._mine(handles):
            if mine.size:
                before = s.free.copy()
                s.tasks_finished(mine)
                delta += s.free - before
        for s, _, _ in self.parts:
            s.free = free0 + delta

    def on_task_running_prefilled(self, t, variant):
        (s, lo, _), = [(s, lo, hi) for s, lo, hi in self.parts if lo <= t < hi]
        pos = s._start_prefilled(int(t) - lo, variant)
        cls = int(s._task_class[int(t) - lo])
        for s2, _, _ in self.parts:
            s2._take_resources(pos, cls, variant)

    def on_retract_response(self, wid, handles):
        out = {}
        for s, lo, mine in self._mine(handles):
            for w, lst in s.on_retract_response(wid, mine).items():
                out.setdefault(w, []).extend((int(t) + lo, int(v)) for t, v in lst)
        return out

    def dispose_prefill(self, c):
        out = {}
        for s, lo, _ in self.parts:
            for w, lst in s.dispose_prefill(c).items():
                out.setdefault(w, []).extend(int(t) + lo for t in lst)
        return {w: sorted(v) for w, v in out.items()}

    def pf_worker(self, n):
        pf = np.full(n, -1, dtype=np.int64)
        for s, lo, hi in self.parts:
            m = max(0, min(hi, n, lo + s._pf_worker.shape[0]) - lo)      # a rank's table grows with its tasks
            pf[lo:lo + m] = s._pf_worker[:m]
        return pf

    def prune_levels(self):
        """ShardedScheduler.prune_levels over the ranks: the same trigger, the OR of the live vectors, the same retain."""
        from hyperqueue_b200.sharded import levels_need_pruning
        s0 = self.parts[0][0]
        if not levels_need_pruning(s0.n_declared_levels(), s0.n_classes, s0._prefill[1] > 0, self.levels_pruned_at):
            return
        tables = [s.levels_live() for s, _, _ in self.parts]
        assert all(np.array_equal(lv, tables[0][0]) for lv, _ in tables)      # declared tables are identical
        lives = [live for _, live in tables]
        keep = np.bitwise_or.reduce(np.stack(lives), axis=0)
        for s, _, _ in self.parts:
            s.levels_retain(keep)
        self.levels_pruned_at = int(np.count_nonzero(keep))

    def tick(self, now=0.0):
        """One sharded tick on every rank at time `now`.  Returns ([records of rank r, global handles], [free after],
        [(rc, text)])."""
        from hyperqueue_b200.scheduler import apply_tick_records
        L = self.L
        s0 = self.parts[0][0]
        for s, _, _ in self.parts:
            s._sync_classes()
            assert np.array_equal(s.free, s0.free)            # the worker state is replicated
        self.prune_levels()
        # every rank passes its own copy of the replicated worker state, as a process of ShardedScheduler does
        ins = []
        for s, _, _ in self.parts:
            blocked = s._blocked_bytes()
            ins.append((s._worker_structs(now), np.ascontiguousarray(s.free), np.ascontiguousarray(s.total), blocked,
                        L.ptr(blocked) if blocked is not None else None))
        nw = ins[0][0].shape[0]
        masks = [s.prefill_mask() for s, _, _ in self.parts if s._prefill[1] > 0]
        if masks:
            mask = np.ascontiguousarray(np.bitwise_or.reduce(np.stack(masks), axis=0))
            for s, _, _ in self.parts:
                if s._prefill[1] > 0:
                    s._check(s._lib.hqs_prefill_state(s._ctx, nw, L.ptr(mask)))
        caps = [max(hi - lo, 1) for _, lo, hi in self.parts]
        if self.fused:
            # the ticks wait for each other on the device: every buffer is allocated before the first launch
            for (s, _, _), cap, (_, _, _, blocked, _) in zip(self.parts, caps, ins):
                s._check(s._lib.hqs_tick_reserve(s._ctx, nw, cap, int(blocked is not None)))
            for (s, _, _), cap, (w, free, total, _, bp) in zip(self.parts, caps, ins):
                s._check(s._lib.hqs_shard_tick_launch(s._ctx, nw, L.ptr(w), L.ptr(free), L.ptr(total), bp, cap))
        else:
            counts = []
            for (s, _, _), (w, free, total, _, bp) in zip(self.parts, ins):
                c = torch.zeros(L.HQS_MAX_GROUPS, dtype=torch.int32, device="cuda")
                ng = C.c_uint32(0)
                s._check(s._lib.hqs_shard_count(s._ctx, nw, L.ptr(w), L.ptr(free), L.ptr(total), bp,
                                                C.c_void_p(c.data_ptr()), c.numel(), C.byref(ng)))
                counts.append(c)
            st = torch.stack(counts).to(torch.int64)
            all_c = st.sum(0).to(torch.int32)
            befs = [st[:r].sum(0).to(torch.int32) for r in range(len(counts))]
            torch.cuda.synchronize()
        recs, frees, errs = [], [], []
        for r, ((s, lo, hi), cap) in enumerate(zip(self.parts, caps)):
            if not self.fused:
                s._check(s._lib.hqs_shard_solve_emit(s._ctx, C.c_void_p(all_c.data_ptr()), C.c_void_p(befs[r].data_ptr()), cap))
            out = np.zeros(cap, dtype=L.assignment_dtype)
            n = C.c_uint32(0)
            fa = np.zeros_like(s.free)
            rc = s._lib.hqs_tick_fetch(s._ctx, cap, L.ptr(out), C.byref(n), L.ptr(fa))
            errs.append((rc, (s._lib.hqs_last_error(s._ctx) or b"").decode() if rc else ""))
            a = out[: n.value].copy()
            if rc == 0:
                apply_tick_records(s, a)
                s.free = fa
            a["task"] += np.uint32(lo)
            recs.append(a)
            frees.append(fa)
        return recs, frees, errs


def _check_tick(ref, m, recs, frees, rk, n_tasks, tag):
    """The per-rank contract of one tick against the single-context tick `m`."""
    ra = m.assignments
    for (s, lo, hi), a, fa in zip(rk.parts, recs, frees):
        k = (ra["task"] >= lo) & (ra["task"] < hi)
        want = np.concatenate([ra[k & (ra["kind"] != 1)], ra[k & (ra["kind"] == 1)]])
        assert np.array_equal(a, want), (tag, lo, hi, a[:6], want[:6])
        assert np.array_equal(fa, m.free_after), tag
    got = np.concatenate(recs)
    W = m.free_after.shape[0]
    assert np.count_nonzero(got["kind"] != 1) == m.n_assigned()
    assert np.array_equal(np.bincount(got["worker"][got["kind"] == 1], minlength=W),
                          np.bincount(ra["worker"][ra["kind"] == 1], minlength=W)), tag
    # the owners' bookkeeping together is the single context's (which tasks are prefilled where)
    assert np.array_equal(rk.pf_worker(n_tasks), ref._pf_worker[:n_tasks]), tag


# ---- (a), (b): the reference's proactive-filling scenarios ---------------------------------------------------------------
def _scenario_cuts(name, world):
    """Cut points: inside the first tick's assigned range, at the ends of and inside its prefill range, right behind the
    assigned tasks (that rank holds no waiting task), and at the first task a later tick redirects."""
    _, recs = S.run_spec(name)
    n = sum(t for _, t in S.SCENARIOS[name][3])
    a0 = recs[0]
    asg, pf = np.sort(a0["task"][a0["kind"] != 1]), np.sort(a0["task"][a0["kind"] == 1])
    pts = set()
    if asg.size:
        pts |= {int(asg[asg.size // 2]), int(asg[-1]) + 1}
    if pf.size:
        pts |= {int(pf[0]), int(pf[pf.size // 2]), int(pf[-1]) + 1}
    for a in recs[1:]:
        k2 = a["task"][a["kind"] == 2]
        if k2.size:
            pts |= {int(k2.min()), int(k2.max()) + 1}
    n0 = S.SCENARIOS[name][3][0][1]                              # every rank holds tasks from the first tick on
    pts = sorted(p for p in pts if 0 < p < n0)
    if world == 2:
        return [[0, p, n] for p in pts]
    return [[0, p, q, n] for p, q in zip(pts, pts[1:])]


def _run_scenario(name, cuts, fused):
    from hyperqueue_b200 import priority_from_user
    reserve, pmax, cpus, steps = S.SCENARIOS[name]
    classes = [[{0: cpus * FR}]]
    ref = _sched(1, classes, 0, (reserve, pmax))
    rk = Ranks(1, classes, cuts, (reserve, pmax), fused)
    n_w = n_t = 0
    kinds = np.zeros(3, dtype=np.int64)
    try:
        for tick, (new_w, new_t) in enumerate(steps):
            for cp in new_w:
                ref.new_worker(50 + n_w, [cp * FR])
                rk.new_worker(50 + n_w, [cp * FR])
                n_w += 1
            if new_t:
                h = np.arange(n_t, n_t + new_t, dtype=np.uint32)
                c = np.zeros(new_t, dtype=np.uint32)
                p = priority_from_user(np.zeros(new_t))
                ref.add_ready_tasks(h, c, p)
                rk.add(h, c, p)
                n_t += new_t
            m = ref.run_scheduling()
            recs, frees, errs = rk.tick()
            assert all(rc == 0 for rc, _ in errs), errs
            _check_tick(ref, m, recs, frees, rk, n_t, (name, cuts, tick))
            kinds += np.bincount(m.assignments["kind"], minlength=3)
    finally:
        rk.close()
        ref.close()
    return kinds


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("name", sorted(S.SCENARIOS))
def test_scenarios_unfused(name, world):
    cut_sets = _scenario_cuts(name, world)
    assert cut_sets
    for cuts in cut_sets:
        kinds = _run_scenario(name, cuts, fused=False)
        assert kinds[1] > 0 or name == "prefill_choose_waiting" and kinds[0] > 0
        if name == "prefill_steal":
            assert kinds[2] == 2                               # the two stolen tasks, on whichever rank owns them


@pytest.mark.parametrize("name", sorted(S.SCENARIOS))
def test_scenarios_fused(name):
    for cuts in _scenario_cuts(name, 2):
        _run_scenario(name, cuts, fused=True)


# ---- (c), (e): a larger synthetic drain with host events between the ticks --------------------------------------------
DRAIN_CLASSES = [[{0: 1 * FR}], [{0: 2 * FR, 1: 4 * FR}], [{0: 1 * FR, 1: 8 * FR}], [{0: 4 * FR}]]
DRAIN_PREFILL = (16, 40)            # tako's defaults (SchedulerConfig::default, scheduler/state.rs:14-21)


def _drain_setup(seed, n=3000, W=48):
    from hyperqueue_b200 import priority_from_user
    rng = np.random.default_rng(seed)
    total = np.tile(np.array([8 * FR, 32 * FR], dtype=np.uint64), (W, 1))
    cls = rng.integers(0, len(DRAIN_CLASSES), n).astype(np.uint32)
    prio = priority_from_user(rng.choice([0, 1, 2], size=n, p=[0.2, 0.3, 0.5]))
    extra = 60                                                  # higher-priority tasks that arrive later (tick 3)
    return rng, total, cls, prio, n, extra


def _apply_workers(sys_, total):
    for i in range(total.shape[0]):
        sys_.new_worker(100 + i, total[i].tolist())


def _drain_script(seed, ticks=7):
    """Runs the drain on a single context and records what happens before every tick (the events are chosen from the
    single context's state) and what every tick returns."""
    from hyperqueue_b200 import priority_from_user
    rng, total, cls, prio, n, extra = _drain_setup(seed)
    ref = _sched(2, DRAIN_CLASSES, 0, DRAIN_PREFILL)
    _apply_workers(ref, total)
    script, out = [], []
    running = []
    try:
        for tick in range(ticks):
            ev = {"add": None, "retract": [], "finish": [], "start": None, "dispose": None}
            res = {}
            if tick == 0:
                ev["add"] = (list(range(n)), cls.tolist(), prio.tolist())
            else:
                for t, ow in sorted(ref._retracting_from.items()):
                    ev["retract"].append((ow, [t]))
                fin = rng.permutation(np.array(running, dtype=np.int64))[: len(running) // 2]
                ev["finish"] = sorted(int(t) for t in fin)
                if tick == 2:
                    wid = next(int(w) for w in ref.worker_ids if ref.prefilled_tasks(int(w)).size)
                    ev["start"] = (int(ref.prefilled_tasks(wid)[0]), 0)
                if tick == 3:
                    h = list(range(n, n + extra))
                    ev["add"] = (h, [0] * extra, priority_from_user(np.full(extra, 5)).tolist())
                    ev["dispose"] = 0                         # check_dispose_prefill: a task of higher priority is ready
            res["retract"] = [ref.on_retract_response(w, hs) for w, hs in ev["retract"]]
            for r in res["retract"]:
                running += [t for lst in r.values() for t, _ in lst]
            ref.tasks_finished(np.array(ev["finish"], dtype=np.uint32))
            done = set(ev["finish"])
            running = [t for t in running if t not in done]
            if ev["start"]:
                ref.on_task_running_prefilled(*ev["start"])
                running.append(ev["start"][0])
            if ev["add"]:
                ref.add_ready_tasks(np.array(ev["add"][0], dtype=np.uint32), np.array(ev["add"][1], dtype=np.uint32),
                                    np.array(ev["add"][2], dtype=np.uint64))
            if ev["dispose"] is not None:
                res["dispose"] = {w: sorted(int(t) for t in v) for w, v in ref.dispose_prefill(ev["dispose"]).items()}
            m = ref.run_scheduling()
            running += m.assignments["task"][m.assignments["kind"] == 0].tolist()
            script.append(ev)
            pfw = np.full(n + extra, -1, dtype=np.int64)
            k = min(n + extra, ref._pf_worker.shape[0])               # the table grows with the tasks
            pfw[:k] = ref._pf_worker[:k]
            out.append((m, res, pfw))
    finally:
        ref.close()
    return script, out, n + extra


def _replay(sys_, script, out, n_all, check):
    """Replays the script on `sys_` (Ranks) and checks every tick against the single context's."""
    for tick, (ev, (m, res, pfw)) in enumerate(zip(script, out)):
        got = [sys_.on_retract_response(w, hs) for w, hs in ev["retract"]]
        assert got == res["retract"], tick
        sys_.tasks_finished(np.array(ev["finish"], dtype=np.int64))
        if ev["start"]:
            sys_.on_task_running_prefilled(*ev["start"])
        if ev["add"]:
            sys_.add(np.array(ev["add"][0], dtype=np.int64), np.array(ev["add"][1], dtype=np.uint32),
                     np.array(ev["add"][2], dtype=np.uint64))
        if ev["dispose"] is not None:
            assert sys_.dispose_prefill(ev["dispose"]) == res["dispose"], tick
        check(tick, m, pfw)


def _task_groups(script, n_all):
    """(priority, class) of every task of the drain, i.e. its (level, class) group."""
    prio = np.zeros(n_all, dtype=np.uint64)
    cls = np.zeros(n_all, dtype=np.int64)
    for ev in script:
        if ev["add"]:
            h = np.array(ev["add"][0], dtype=np.int64)
            cls[h] = ev["add"][1]
            prio[h] = np.array(ev["add"][2], dtype=np.uint64)
    return prio, cls


def _prefill_ranges(a, prio, cls):
    """Tasks of each prefill range of a tick (kind-1 records grouped by their (level, class) group), ascending."""
    pf = a["task"][a["kind"] == 1].astype(np.int64)
    out = {}
    for t in pf.tolist():
        out.setdefault((int(prio[t]), int(cls[t])), []).append(t)
    return [np.sort(np.array(v)) for v in out.values()]


def _crossing_cut(script, out, n_all):
    """A cut inside the first tick's largest prefill range: that range has records on both sides of the rank boundary."""
    prio, cls = _task_groups(script, n_all)
    ranges = _prefill_ranges(out[0][0].assignments, prio, cls)
    assert ranges
    t = max(ranges, key=len)
    assert t.size >= 2
    return int(t[t.size // 2])


@pytest.mark.parametrize("world,fused", [(2, False), (3, False), (2, True)])
def test_synthetic_drain(world, fused):
    script, out, n_all = _drain_script(seed=11)
    _, total, _, _, _, _ = _drain_setup(11)
    cut = _crossing_cut(script, out, n_all)
    prio, cls = _task_groups(script, n_all)
    cuts = [0, cut, n_all] if world == 2 else [0, cut // 2, cut, n_all]
    rk = Ranks(2, DRAIN_CLASSES, cuts, DRAIN_PREFILL, fused)
    _apply_workers(rk, total)
    seen = {"crossed": 0, "k2": 0, "k1": 0}

    def check(tick, m, pfw):
        recs, frees, errs = rk.tick()
        assert all(rc == 0 for rc, _ in errs), errs
        ra = m.assignments
        for (s, lo, hi), a, fa in zip(rk.parts, recs, frees):
            k = (ra["task"] >= lo) & (ra["task"] < hi)
            want = np.concatenate([ra[k & (ra["kind"] != 1)], ra[k & (ra["kind"] == 1)]])
            assert np.array_equal(a, want), (tick, lo, hi)
            assert np.array_equal(fa, m.free_after), tick
        assert np.array_equal(rk.pf_worker(n_all), pfw), tick
        # a prefill range (one group's kind-1 records) with records on both sides of the cut
        if any(t[0] < cut <= t[-1] for t in _prefill_ranges(ra, prio, cls)):
            seen["crossed"] += 1
        seen["k1"] += int(np.count_nonzero(ra["kind"] == 1))
        seen["k2"] += int(np.count_nonzero(ra["kind"] == 2))

    try:
        _replay(rk, script, out, n_all, check)
    finally:
        rk.close()
    assert seen["crossed"] and seen["k1"] and seen["k2"], seen


# ---- (d): ranks configured differently -----------------------------------------------------------------------------------
def test_fused_prefill_mismatch_fails_the_tick_on_every_rank():
    _, total, cls, prio, n, _ = _drain_setup(5, n=2000, W=32)
    cuts = [0, 1000, n]
    rk = Ranks(2, DRAIN_CLASSES, cuts, None, True, prefill_of_rank=[DRAIN_PREFILL, None])
    ref = _sched(2, DRAIN_CLASSES, 0, DRAIN_PREFILL)
    try:
        for sys_ in (rk, ref):
            _apply_workers(sys_, total)
        rk.add(np.arange(n), cls, prio)
        ref.add_ready_tasks(np.arange(n, dtype=np.uint32), cls, prio)
        recs, frees, errs = rk.tick()
        for rc, text in errs:
            assert rc == -6 and "G=" in text, errs                # HQS_E_STATE, naming both group counts
        g = [s.stats() for s, _, _ in rk.parts]
        assert all(x["n_assigned"] == 0 for x in g)
        # the same configuration on both ranks: the ready sets were not touched, the tick equals the single context's
        rk.parts[1][0].set_prefill(*DRAIN_PREFILL)
        m = ref.run_scheduling()
        recs, frees, errs = rk.tick()
        assert all(rc == 0 for rc, _ in errs), errs
        _check_tick(ref, m, recs, frees, rk, n, "after the mismatch")
        assert np.count_nonzero(m.assignments["kind"] == 1)
    finally:
        rk.close()
        ref.close()


# ---- (e): ShardedScheduler over NCCL, one process per GPU -------------------------------------------------------------
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


class _ShardedSys:
    """ShardedScheduler of one rank behind the replay interface; returns what the rank itself returns."""

    def __init__(self, sh):
        self.sh = sh

    def new_worker(self, wid, res):
        self.sh.s.new_worker(wid, res)

    def add(self, h, c, p):
        self.sh.add_ready_tasks(h, c, p)

    def tasks_finished(self, h):
        self.sh.tasks_finished(h)

    def on_task_running_prefilled(self, t, v):
        self.sh.on_task_running_prefilled(t, v)

    def on_retract_response(self, w, hs):
        return self.sh.on_retract_response(w, hs)

    def dispose_prefill(self, c):
        return self.sh.dispose_prefill(c)


def _new_sharded(rank, world, n_all, p2p, total):
    """A ShardedScheduler of the drain (classes, workers, tako's default prefill configuration) on GPU `rank`."""
    from hyperqueue_b200 import GpuScheduler, RequestVariant
    from hyperqueue_b200.sharded import ShardedScheduler
    base = GpuScheduler(2, rank, 0)
    for vs in DRAIN_CLASSES:
        base.get_or_create_resource_rq_id([RequestVariant.of(a) for a in vs])
    sh = ShardedScheduler(base, rank, world, n_all, torch.device("cuda", rank), p2p=p2p)
    sh.set_prefill(*DRAIN_PREFILL)
    sys_ = _ShardedSys(sh)
    _apply_workers(sys_, total)
    return sh, sys_


def _rank_pf_worker(sh, n_all):
    """The rank's prefill bookkeeping over the global handles (-1 elsewhere); the rank's table grows with its tasks."""
    pf = np.full(n_all, -1, dtype=np.int64)
    m = min(sh.hi - sh.lo, sh.s._pf_worker.shape[0])
    pf[sh.lo:sh.lo + m] = sh.s._pf_worker[:m]
    return pf


@pytest.mark.parametrize("p2p", [False, True])
def test_sharded_scheduler_one_rank_drain(p2p):
    """ShardedScheduler itself on one GPU: a world of one rank needs no process group (the exchange, the mask reduction and
    the all-reduces of the host events reduce to the rank's own values), so its prefill surface (set_prefill, the mask
    passed before the tick, on_task_running_prefilled, on_retract_response, dispose_prefill, prefilled_tasks, the records
    applied to the owner's bookkeeping) runs the drain against the single context on both exchange paths."""
    script, out, n_all = _drain_script(seed=11)
    _, total, _, _, _, _ = _drain_setup(11)
    sh, sys_ = _new_sharded(0, 1, n_all, p2p, total)
    seen = {"k1": 0, "k2": 0}

    def check(tick, m, pfw):
        a, fa = sh.run_scheduling()
        ra = m.assignments
        assert np.array_equal(a, np.concatenate([ra[ra["kind"] != 1], ra[ra["kind"] == 1]])), tick
        assert np.array_equal(fa, m.free_after), tick
        assert np.array_equal(_rank_pf_worker(sh, n_all), pfw), tick
        assert sh.last_mapping.messages() == m.messages(), tick        # RetractTasks of kind-2 records included
        for wid in sh.s.worker_ids.tolist():
            assert np.array_equal(np.sort(sh.prefilled_tasks(wid)), np.nonzero(pfw == wid)[0]), (tick, wid)
        seen["k1"] += int(np.count_nonzero(ra["kind"] == 1))
        seen["k2"] += int(np.count_nonzero(ra["kind"] == 2))

    try:
        _replay(sys_, script, out, n_all, check)
    finally:
        sh.s.close()
    assert seen["k1"] and seen["k2"], seen


def _sharded_worker(rank, world, port, p2p, script, n_all, total, ret):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    sh, sys_ = _new_sharded(rank, world, n_all, p2p, total)
    ticks = []
    for ev in script:
        host = {"retract": [sys_.on_retract_response(w, hs) for w, hs in ev["retract"]]}
        sys_.tasks_finished(np.array(ev["finish"], dtype=np.int64))
        if ev["start"]:
            sys_.on_task_running_prefilled(*ev["start"])
        if ev["add"]:
            sys_.add(np.array(ev["add"][0], dtype=np.int64), np.array(ev["add"][1], dtype=np.uint32),
                     np.array(ev["add"][2], dtype=np.uint64))
        if ev["dispose"] is not None:
            host["dispose"] = sys_.dispose_prefill(ev["dispose"])
        a, fa = sh.run_scheduling()
        ticks.append((a.tobytes(), fa.tobytes(), _rank_pf_worker(sh, n_all).tobytes(), host))
    ret[rank] = ticks
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("p2p", [False, True])
def test_sharded_scheduler_drain_over_nccl(p2p):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    from hyperqueue_b200 import _lib as L
    from hyperqueue_b200.sharded import block_range
    script, out, n_all = _drain_script(seed=11)
    _, total, _, _, _, _ = _drain_setup(11)
    mgr = mp.Manager(); ret = mgr.dict()
    mp.spawn(_sharded_worker, args=(2, _free_port(), p2p, script, n_all, total, ret), nprocs=2, join=True)
    for tick, (m, res, pfw) in enumerate(out):
        ra = m.assignments
        pf = np.full(n_all, -1, dtype=np.int64)
        retract = [dict() for _ in res["retract"]]
        dispose = {}
        for r in range(2):
            lo, hi = block_range(n_all, r, 2)
            a_b, fa_b, pf_b, host = ret[r][tick]
            a = np.frombuffer(a_b, dtype=L.assignment_dtype)
            k = (ra["task"] >= lo) & (ra["task"] < hi)
            want = np.concatenate([ra[k & (ra["kind"] != 1)], ra[k & (ra["kind"] == 1)]])
            assert np.array_equal(a, want), (tick, r)
            assert np.array_equal(np.frombuffer(fa_b, dtype=np.uint64).reshape(m.free_after.shape), m.free_after), (tick, r)
            pf[lo:hi] = np.frombuffer(pf_b, dtype=np.int64)[lo:hi]
            for i, d in enumerate(host["retract"]):
                for w, lst in d.items():
                    retract[i].setdefault(w, []).extend(lst)
            for w, lst in host.get("dispose", {}).items():
                dispose.setdefault(w, []).extend(lst)
        assert np.array_equal(pf, pfw), tick
        assert retract == res["retract"], tick
        if "dispose" in res:
            assert {w: sorted(v) for w, v in dispose.items()} == res["dispose"], tick
