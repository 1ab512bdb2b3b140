"""The ready set's key table on the device against tests/level_model.py: after every call the whole key array
(hqs_debug_keys) and the level statistics must equal the model's, and no VALID key may hold a level outside the level
table.  Only then does a tick run, and it must equal the sequential specification (tests/greedy_model.py) on the
level-mapped workload (user priority = -level, so that coarse ticks are compared bit for bit too) and pass the judge.
Every sequence runs on two contexts side by side, one per amount width of the solver."""
import ctypes as C

import numpy as np
import pytest

import greedy_model as G
import level_model as LM
import parity as P

pytestmark = pytest.mark.gpu
FR = P.FR
W_TOTAL = np.array([[12 * FR, 300000], [16 * FR, 400000], [8 * FR, 200000], [20 * FR, 500000]], dtype=np.uint64)
PREFILL = (2, 3)                       # proactive filling reserve / max per worker
E_LIMIT, E_OVERFLOW = -3, -5


def class_def(c):
    """Class c: one variant, distinct for every c < 4096."""
    return [{"amounts": {0: (1 + c % 4) * FR, 1: (1 + c // 4) * 100}}]


def tako_priority(user, job):
    return (((int(user) & 0xFFFFFFFF) ^ 0x80000000) << 32) | int(job)


class Dev:
    """One context driven through the C ABI."""

    def __init__(self, flags):
        from hyperqueue_b200 import _lib as L
        self.L, self.lib = L, L.load_library()
        self.ctx = C.c_void_p()
        rc = self.lib.hqs_create(C.byref(self.ctx), 0, 2, flags)
        if rc:
            raise L.HqsError(rc, (self.lib.hqs_last_error(None) or b"").decode())

    def ok(self, rc):
        if rc:
            raise self.L.HqsError(rc, (self.lib.hqs_last_error(self.ctx) or b"").decode())

    def close(self):
        if self.ctx.value:
            self.lib.hqs_destroy(self.ctx)
            self.ctx = C.c_void_p()

    def classes(self, q):
        arr = (self.L.hqs_class * q)()
        for c in range(q):
            arr[c].n_variants = 1
            for r, a in class_def(c)[0]["amounts"].items():
                arr[c].variants[0].amount[r] = a
            arr[c].variants[0].weight = 10000
        self.ok(self.lib.hqs_classes_set(self.ctx, q, arr))

    def push(self, h, c, p, as_range):
        h, c, p = (np.ascontiguousarray(h, np.uint32), np.ascontiguousarray(c, np.uint32),
                   np.ascontiguousarray(p, np.uint64))
        if as_range:
            assert (np.diff(h.astype(np.int64)) == 1).all()
            self.ok(self.lib.hqs_ready_push_range(self.ctx, int(h[0]), h.size, self.L.ptr(c), self.L.ptr(p)))
        else:
            self.ok(self.lib.hqs_ready_push(self.ctx, h.size, self.L.ptr(h), self.L.ptr(c), self.L.ptr(p)))

    def remove(self, h):
        h = np.ascontiguousarray(h, np.uint32)
        self.ok(self.lib.hqs_ready_remove(self.ctx, h.size, self.L.ptr(h)))

    def keys(self):
        n = C.c_uint32(0)
        self.ok(self.lib.hqs_debug_keys(self.ctx, 0, None, C.byref(n)))
        out = np.zeros(n.value, np.uint32)
        self.ok(self.lib.hqs_debug_keys(self.ctx, n.value, self.L.ptr(out), C.byref(n)))
        assert n.value == out.size
        return out

    def stats(self):
        st = self.L.hqs_stats()
        self.ok(self.lib.hqs_get_stats(self.ctx, C.byref(st)))
        return {name: int(getattr(st, name)) for name, _ in self.L.hqs_stats._fields_}

    def tick(self, free, pf_mask, out_cap):
        W = free.shape[0]
        w = np.zeros(W, dtype=self.L.worker_dtype)
        w["worker_id"] = np.arange(W)
        w["remaining_time_ms"] = self.L.HQS_TIME_INF
        if pf_mask is not None:
            self.ok(self.lib.hqs_prefill_state(self.ctx, W, self.L.ptr(np.ascontiguousarray(pf_mask))))
        out = np.zeros(max(out_cap, 1), dtype=self.L.assignment_dtype)
        n = C.c_uint32(0)
        fa = np.zeros_like(free)
        self.ok(self.lib.hqs_tick(self.ctx, W, self.L.ptr(w), self.L.ptr(free), self.L.ptr(W_TOTAL), None, out_cap,
                                  self.L.ptr(out), C.byref(n), self.L.ptr(fa)))
        return out[: n.value].copy(), fa


class Harness:
    """The same calls on the model and on one context per amount width; checks after every call."""

    def __init__(self, widths=(0, 2)):
        from hyperqueue_b200 import _lib as L
        self.devs = [Dev(f) for f in widths]
        self.m = LM.LevelModel()
        self.pfw = np.zeros(0, np.int64)       # worker index each task is prefilled on, -1: none
        self.prefill = None
        self.L = L
        # what the calls exercised: prefill records, PF bits cleared by a dispose or a remove, coarse -> exact pushes
        self.seen = dict(kind1=0, kind2=0, pf_disposed=0, pf_removed=0, to_exact=0)

    def close(self):
        for d in self.devs:
            d.close()

    def _sync_pf(self):
        if self.pfw.size < self.m.n_handles:
            self.pfw = np.concatenate([self.pfw, np.full(self.m.n_handles - self.pfw.size, -1, np.int64)])

    def check(self, label):
        m = self.m
        exp = m.keys()
        self._sync_pf()
        assert np.array_equal(self.pfw[: m.n_handles] >= 0, m.has(LM.KEY_PF)), label
        for d in self.devs:
            got = d.keys()
            st = d.stats()
            valid = (got & np.uint32(LM.KEY_VALID)) != 0
            lv = (got >> np.uint32(LM.LEVEL_SHIFT)) & np.uint32(LM.LEVEL_MASK)
            bad = valid & (lv >= max(st["n_levels"], 1))
            assert not bad.any(), (f"{label}: {int(bad.sum())} VALID keys hold a level >= max(n_levels, 1) = "
                                   f"{max(st['n_levels'], 1)} (largest {int(lv[bad].max())})")
            assert (st["coarsened"], st["n_levels"]) == (m.coarsened, m.n_levels), (
                f"{label}: device coarsened={st['coarsened']} n_levels={st['n_levels']}, model coarsened={m.coarsened} "
                f"n_levels={m.n_levels}; live priorities {m.live_priorities().size}, budget {LM.max_levels(m.Q)}")
            assert got.size == exp.size, (label, got.size, exp.size)
            diff = np.nonzero(got != exp)[0]
            if diff.size:
                dv = diff[valid[diff]]
                lv_dev = np.unique(lv[dv]).tolist()
                lv_mod = np.unique(m.lvl[dv]).tolist()
                raise AssertionError(
                    f"{label}: {diff.size} keys differ, first handle {int(diff[0])}: device {int(got[diff[0]]):#010x} model "
                    f"{int(exp[diff[0]]):#010x}; {dv.size} of them VALID with {np.unique(m.prio[dv]).size} distinct priorities, "
                    f"device levels {lv_dev[:6]}{'...' if len(lv_dev) > 6 else ''} ({len(lv_dev)} distinct), model levels "
                    f"{lv_mod[:6]}{'...' if len(lv_mod) > 6 else ''} ({len(lv_mod)} distinct)")

    def _both(self, model_call, dev_call, label):
        try:
            model_call()
        except LM.Rejected:
            for d in self.devs:
                with pytest.raises(self.L.HqsError):
                    dev_call(d)
        else:
            for d in self.devs:
                dev_call(d)
        self.check(label)

    # calls ------------------------------------------------------------------------------------------------------------
    def classes(self, q):
        self._both(lambda: self.m.classes_set(q), lambda d: d.classes(q), f"classes_set({q})")

    def set_prefill(self, cfg):
        self.prefill = cfg
        for d in self.devs:
            d.ok(d.lib.hqs_prefill_config(d.ctx, cfg[0], cfg[1]))

    def push(self, h, c, p, as_range=False):
        hi = np.asarray(h, np.int64)
        if hi.size and hi.max() >= self.pfw.size:
            self.pfw = np.concatenate([self.pfw, np.full(int(hi.max()) + 1 - self.pfw.size, -1, np.int64)])
        self.pfw[hi] = -1                                      # a push replaces the whole key
        was_coarse = self.m.coarse
        self._both(lambda: self.m.push(h, c, p), lambda d: d.push(h, c, p, as_range),
                   f"push of {len(h)} tasks ({'range' if as_range else 'handles'})")
        self.seen["to_exact"] += int(was_coarse and not self.m.coarse)

    def remove(self, h):
        h = np.asarray(h, np.uint32)
        hi = h.astype(np.int64)
        hi = hi[hi < self.m.n_handles]
        self.seen["pf_removed"] += int(np.count_nonzero(self.m.has(LM.KEY_PF)[hi]))
        self.pfw[hi] = -1
        self._both(lambda: self.m.remove(h), lambda d: d.remove(h), f"remove of {h.size} handles")

    def rearm(self):
        self._both(self.m.rearm, lambda d: d.ok(d.lib.hqs_ready_rearm(d.ctx)), "rearm")

    def dispose(self, c):
        if c < self.m.Q:
            held = (self.m.cls == c) & self.m.has(LM.KEY_PF)
            self.seen["pf_disposed"] += int(np.count_nonzero(held))
            self.pfw[: self.m.n_handles][held] = -1
        self._both(lambda: self.m.prefill_dispose(c), lambda d: d.ok(d.lib.hqs_prefill_dispose(d.ctx, c)),
                   f"prefill_dispose({c})")

    def levels_add(self, p):
        p = np.ascontiguousarray(p, np.uint64)
        self._both(lambda: self.m.levels_add(p), lambda d: d.ok(d.lib.hqs_levels_add(d.ctx, p.size, d.L.ptr(p))),
                   f"levels_add of {p.size}")

    def levels_retain(self, keep):
        """hqs_levels_live on every context must equal the model's before the retain."""
        want_lv, want_live = self.m.levels_live()
        for d in self.devs:
            n = C.c_uint32(0)
            d.ok(d.lib.hqs_levels_live(d.ctx, 0, None, None, C.byref(n)))
            assert n.value == want_lv.size, ("n_levels", n.value, want_lv.size)
            lv, live = np.zeros(n.value, np.uint64), np.zeros(n.value, np.uint8)
            if n.value:
                d.ok(d.lib.hqs_levels_live(d.ctx, n.value, d.L.ptr(lv), d.L.ptr(live), C.byref(n)))
            assert np.array_equal(lv, want_lv) and np.array_equal(live, want_live), "levels_live"
        keep = np.ascontiguousarray(keep, np.uint8)
        self.seen["retained"] = self.seen.get("retained", 0) + 1
        self._both(lambda: self.m.levels_retain(keep),
                   lambda d: d.ok(d.lib.hqs_levels_retain(d.ctx, keep.size, d.L.ptr(keep))),
                   f"levels_retain of {keep.size} ({int(keep.size - keep.sum())} dropped)")

    def dag_load(self, cls, prio, n_deps, off, cons):
        arrs = [np.ascontiguousarray(cls, np.uint32), np.ascontiguousarray(prio, np.uint64),
                np.ascontiguousarray(n_deps, np.uint32), np.ascontiguousarray(off, np.uint32),
                np.ascontiguousarray(cons, np.uint32)]
        self.pfw = np.full(len(cls), -1, np.int64)
        self._both(lambda: self.m.dag_load(*arrs),
                   lambda d: d.ok(d.lib.hqs_dag_load(d.ctx, arrs[0].size, *[d.L.ptr(a) for a in arrs[:4]],
                                                     d.L.ptr(arrs[4]) if arrs[4].size else None)),
                   f"dag_load of {len(cls)} tasks")

    def finished(self, t):
        t = np.ascontiguousarray(t, np.uint32)
        want = self.m.tasks_finished(t)
        self.pfw[t.astype(np.int64)] = -1
        for d in self.devs:
            n = C.c_uint32(0)
            d.ok(d.lib.hqs_tasks_finished(d.ctx, t.size, d.L.ptr(t), C.byref(n)))
            assert n.value == want, ("n_new_ready", n.value, want)
        self.check(f"tasks_finished of {t.size}")

    def tick(self, label="tick"):
        """One tick on every context, compared with the specification; returns the records (None if the tick has more
        groups than HQS_MAX_GROUPS, which must fail before anything changes)."""
        m = self.m
        self.check(f"before {label}")
        n, Q = m.n_handles, m.Q
        ready = m.ready()
        free = W_TOTAL.copy()
        pf_on = self.prefill is not None and self.prefill[1] > 0
        mask = None
        if pf_on:
            mask = np.zeros((free.shape[0], Q), np.uint8)
            held = np.nonzero(ready & (self.pfw[:n] >= 0))[0]
            mask[self.pfw[held], m.cls[held]] = 1
        # proactive filling doubles the groups (waiting / prefilled) but not the level budget, which is HQS_MAX_GROUPS / Q:
        # a coarse table with proactive filling on always has too many groups, and such a tick must fail untouched
        if max(m.n_levels, 1) * Q * (2 if pf_on else 1) > LM.HQS_MAX_GROUPS:
            for d in self.devs:
                with pytest.raises(self.L.HqsError) as ei:
                    d.tick(free, mask, max(n, 1))
                assert ei.value.code == E_LIMIT
            self.check(f"{label} (too many groups)")
            return None
        wl = P.Workload(2, [class_def(c) for c in range(Q)], W_TOTAL, free, m.cls.copy(),
                        np.where(ready, -m.lvl.astype(np.int64), 0).astype(np.int32))
        pfw = self.pfw[:n].copy() if pf_on else None
        exp, exp_free = G.model_tick(wl, ready, free, prefill=self.prefill if pf_on else None, pf_worker=pfw)
        for d in self.devs:
            got, fa = d.tick(free, mask, max(n, 1))
            assert np.array_equal(got, exp), (label, got.size, exp.size, got[:6], exp[:6])
            assert np.array_equal(fa, exp_free), label
        asg = exp[exp["kind"] != 1]
        self.seen["kind1"] += int(np.count_nonzero(exp["kind"] == 1))
        self.seen["kind2"] += int(np.count_nonzero(exp["kind"] == 2))
        res = P.judge_tick(wl, free, asg, ready)
        assert res.ok, (label, res)
        m.apply_tick(exp)
        self.pfw[asg["task"].astype(np.int64)] = -1
        pf = exp[exp["kind"] == 1]
        self.pfw[pf["task"].astype(np.int64)] = pf["worker"]
        self.check(f"after {label}")
        return exp


@pytest.fixture
def harness():
    h = Harness()
    yield h
    h.close()


# directed sequences -----------------------------------------------------------------------------------------------------
WAVE1 = np.array([tako_priority(0, 1000 + 16 * i) for i in range(5000)], dtype=np.uint64)   # 5000 distinct, ascending


def _classes_of(n):
    return (np.arange(n) % 2).astype(np.uint32)


def _first_wave(h):
    h.classes(2)                                             # budget 8192 / 2 = 4096 levels
    h.push(np.arange(5000), _classes_of(5000), WAVE1, as_range=True)     # > 4096 fresh: the host's distinct pass
    assert h.m.coarsened == 1 and h.m.n_levels == 4096


def test_coarse_table_is_left_when_a_new_wave_fits(harness):
    """All of the first wave leaves; 1500 new priorities above all of it fit the budget exactly again."""
    h = harness
    _first_wave(h)
    h.remove(np.arange(5000))
    up = np.array([tako_priority(5, j) for j in range(1, 1501)], dtype=np.uint64)
    h.push(np.arange(5000, 6500), _classes_of(1500), up)
    assert h.m.coarsened == 0 and h.m.n_levels == 1500
    a = h.tick()
    got = [int(x) for x in up[a["task"].astype(np.int64) - 5000]]
    assert a.size and all(x > y for x, y in zip(got, got[1:]))          # strictly by priority again


def test_lower_wave_keeps_its_order_below_the_kept_tasks_after_a_new_class(harness):
    """100 tasks of the first wave stay; the new wave lies below them; then a class is registered (Q 2 -> 3)."""
    h = harness
    _first_wave(h)
    h.remove(np.arange(4900))                               # the 100 highest priorities stay
    low = np.array([tako_priority(-5, j) for j in range(1, 1501)], dtype=np.uint64)
    h.push(np.arange(5000, 6500), _classes_of(1500), low)
    h.classes(3)
    assert h.m.coarsened == 0 and h.m.n_levels == 1600
    a = h.tick()
    first = a["task"][: min(a.size, 20)].astype(np.int64)
    assert a.size and (first < 5000).all()                  # the 100 kept tasks come first


def test_lower_wave_alone_after_a_new_class(harness):
    """None of the first wave stays; the new wave lies below every priority it had; then Q 2 -> 3."""
    h = harness
    _first_wave(h)
    h.remove(np.arange(5000))
    low = np.array([tako_priority(-5, j) for j in range(1, 1501)], dtype=np.uint64)
    h.push(np.arange(5000, 6500), _classes_of(1500), low)
    h.classes(3)
    assert h.m.coarsened == 0 and h.m.n_levels == 1500
    assert h.tick().size


def test_wave_interleaving_the_old_priorities(harness):
    h = harness
    _first_wave(h)
    h.remove(np.setdiff1d(np.arange(5000), np.arange(0, 5000, 50)))      # 100 spread-out tasks stay
    mid = np.array([tako_priority(0, 1000 + 16 * (3 * i) + 8) for i in range(1500)], dtype=np.uint64)
    h.push(np.arange(5000, 6500), _classes_of(1500), mid)
    assert h.m.coarsened == 0 and h.m.n_levels == 1600
    h.classes(3)
    h.tick()
    # the removed priorities come back on re-used handles, together with the kept ones
    h.push(np.arange(0, 3000, 3), _classes_of(1000), WAVE1[np.arange(0, 3000, 3)])
    h.tick()


def test_overflowing_tick_leaves_the_key_table_unchanged(harness):
    h = harness
    _first_wave(h)                                          # coarse
    for d in h.devs:
        before = d.keys()
        with pytest.raises(h.L.HqsError) as ei:
            d.tick(W_TOTAL.copy(), None, 1)
        assert ei.value.code == E_OVERFLOW
        assert np.array_equal(d.keys(), before)
    h.check("after the failed ticks")
    h.tick()


def test_table_growth_keeps_old_keys_and_zeroes_new_ones(harness):
    h = harness
    h.classes(3)
    h.push(np.arange(1000), np.arange(1000) % 3, np.arange(1000, dtype=np.uint64) * 7, as_range=True)
    h.tick()
    h.push(np.array([70000, 65535, 65536]), np.array([2, 1, 0]), np.array([5, 7, 2 ** 64 - 1], dtype=np.uint64))
    h.push(np.array([140000]), np.array([1]), np.array([0], dtype=np.uint64))           # the second doubling
    h.remove(np.array([200000, 140000, 3]))
    h.rearm()
    h.tick()


# random sequences -------------------------------------------------------------------------------------------------------
def _run_random(h, rng, declared, n_ops, max_q=4096, few_priorities=False):
    used: set = set()
    for _ in range(n_ops):
        op = LM.random_op(rng, h.m, used, declared, max_q=max_q, few_priorities=few_priorities)
        if op[0] == "push":
            h.push(op[1], op[2], op[3], op[4])
        elif op[0] == "remove":
            h.remove(op[1])
        elif op[0] == "tick":
            h.tick()
        elif op[0] == "remove_done":
            h.remove(np.nonzero(h.m.has(LM.KEY_DONE))[0])      # finished tasks leave the table
        elif op[0] == "rearm":
            h.rearm()
        elif op[0] == "dispose":
            h.dispose(op[1])
        elif op[0] == "classes":
            h.classes(op[1])
        elif op[0] == "levels_add":
            h.levels_add(op[1])
        elif op[0] == "levels_retain":
            h.levels_retain(op[1])


@pytest.mark.parametrize("seed", range(30))
def test_random_call_sequences_match_the_model(harness, seed):
    rng = np.random.default_rng(seed)
    if seed % 3 == 0:
        # proactive filling: few classes and few priorities, so that ticks fit the group limit and levels hold more
        # waiting tasks than the reserve
        harness.classes(int(rng.choice([1, 2, 3])))
        harness.set_prefill(PREFILL)
        _run_random(harness, rng, declared=False, n_ops=40, max_q=12, few_priorities=True)
        harness.tick("last tick")
        assert harness.seen["kind1"] > 0, harness.seen
    else:
        harness.classes(int(rng.choice([1, 2, 3, 100, 1000, 2048])))
        _run_random(harness, rng, declared=seed % 5 == 4, n_ops=40)
        harness.tick("last tick")


def test_proactive_filling_sets_and_clears_prefilled_bits(harness):
    """Kind-1 records set PREFILLED, an assigned prefilled task comes out as kind 2, and a dispose and a remove clear the
    bit; the keys equal the model after each call."""
    h = harness
    h.classes(2)
    h.set_prefill(PREFILL)
    top, low = tako_priority(3, 1), tako_priority(1, 1)
    h.push(np.arange(200), np.zeros(200), np.full(200, top, dtype=np.uint64), as_range=True)
    h.push(np.arange(200, 300), np.ones(100), np.full(100, low, dtype=np.uint64), as_range=True)
    a = h.tick("tick 1")
    assert (a["kind"] == 1).any() and h.m.has(LM.KEY_PF).any()
    h.dispose(0)                                            # a task of higher priority arrived
    assert h.seen["pf_disposed"] > 0 and not h.m.has(LM.KEY_PF).any()
    h.tick("tick 2")
    h.remove(np.nonzero(h.m.has(LM.KEY_PF))[0][:2])         # a worker started two of its prefilled tasks
    h.remove(np.nonzero(h.m.has(LM.KEY_DONE))[0])           # and the assigned ones finished
    for k in range(3, 8):
        h.tick(f"tick {k}")
    assert h.seen["kind1"] and h.seen["kind2"] and h.seen["pf_removed"] == 2, h.seen



# DAG mode ---------------------------------------------------------------------------------------------------------------
def _dag(rng, n, n_diamonds):
    deps = []
    for k in range(n_diamonds):                             # a -> b, a -> c, b -> d, c -> d
        a = 4 * k
        deps += [[], [a], [a], [a + 1, a + 2]]
    for t in range(4 * n_diamonds, n):
        k = int(rng.integers(0, 4))
        deps.append(sorted(set(int(x) for x in rng.integers(max(0, t - 500), t, k))) if k else [])
    return deps


def test_dag_mode_keys_follow_the_model(harness):
    h = harness
    rng = np.random.default_rng(7)
    n = 6000
    deps = _dag(rng, n, 100)
    n_deps, off, cons = P.dag_csr(deps)
    # 5500 distinct priorities (more than the 4096 the two classes allow), the diamonds on top
    vals = np.array([tako_priority(9, 10 ** 6 - i) for i in range(5500)], dtype=np.uint64)
    prio = np.concatenate([vals[:400], rng.permutation(np.concatenate([vals[400:], rng.choice(vals[400:], n - 5500)]))])
    h.classes(2)
    h.dag_load(rng.integers(0, 2, n), prio, n_deps, off, cons)
    assert h.m.coarsened == 1
    h.remove(np.array([3, 7]))                               # diamond sinks removed while both producers are unfinished
    for step in range(10):
        a = h.tick(f"tick {step}")
        done = a["task"][a["kind"] != 1].astype(np.int64)
        half = done.size // 2
        h.finished(done[:half])
        h.finished(done[half:])
        waiting = np.nonzero(h.m.has(LM.KEY_VALID) & ~h.m.ready() & (h.m.deps > 0))[0]
        if step % 3 == 1 and waiting.size:
            h.remove(rng.choice(waiting, 3))
        if step == 5:
            h.classes(3)                                     # the budget shrinks: prune and re-level in DAG mode
    assert not (h.m.has(LM.KEY_READY) & np.isin(np.arange(n), [3, 7])).any()
