"""Multi-tick drains on worker pools of 1 to 1024 workers with every tick feature mixed, and the driver that runs them
against the specification (tests/greedy_model.py) and, in lockstep, through the CUDA path.

A scenario is a pure function of its seed (numpy default_rng).  Between ticks the drain does what a server does: assigned
tasks finish after 1 to 3 ticks and their handles are retired (remove_ready_tasks, as the C++ shim does) and later re-used
with another class and priority; new tasks arrive as handle ranges and as scattered handles, some at new priority values
and some above everything in the set; waiting (never prefilled) tasks are cancelled; with proactive filling a worker
starts one of its prefilled tasks, a class's prefills are disposed, and every redirect is answered by the old worker; the
blocked mask changes and `now` advances, so remaining times shrink and some workers run out of time.

Drain(seed).run(check) calls check(tick, inputs, expected) once per tick with the specification's result; the GPU test
passes a check that runs the same tick on the device contexts.  Nothing here is a test by itself."""
from __future__ import annotations

from dataclasses import dataclass, field
from types import SimpleNamespace
from typing import Callable, Dict, List, Optional, Tuple

import numpy as np

import greedy_model as G
from oracle import judge as J
from workloads import FR, MAXV, Workload

AMOUNT_MAX = G.AMOUNT_MAX
POOL_SIZES = (1, 31, 32, 33, 64, 65, 257, 511, 512, 513, 640, 1023, 1024)
SEEDS = tuple(range(26))
TICK_S = 10.0                 # `now` advances by this much per tick; time limits are multiples of it
MAX_GROUPS = 8192             # HQS_MAX_GROUPS: live levels x classes x 2 must stay below it with proactive filling


@dataclass
class Scenario:
    seed: int
    W: int
    R: int
    classes: List[List[dict]]
    total: np.ndarray                              # [W][R] u64
    termination: np.ndarray                        # [W] absolute seconds, inf = none
    min_util: Optional[np.ndarray]                 # [W] f32 or None
    pack: bool
    prefill: Optional[Tuple[int, int]]             # (reserve, max) or None
    n_ticks: int
    plain: bool                                    # one variant per class, nothing else set: the lean / wide loops
    blocked: bool
    n_levels_cap: int
    class_p: np.ndarray = field(default=None)      # class mix of new tasks


def _variant(rng, R: int, units: List[int], big: bool, extras: bool) -> dict:
    """Worker totals are 8 to 63 units of each resource; a big request takes 14 to 40 of them, so it only fits on the
    bigger workers and not on a partly used one: its class is left with tasks and reserves workers."""
    k = int(rng.integers(1, min(R, 4) + 1))
    rs = sorted(int(x) for x in rng.choice(R, size=k, replace=False))
    lo, hi = (14, 40) if big else (1, 12)
    d = {"amounts": {r: int(rng.integers(lo, hi)) * units[r] + (units[r] & 1) for r in rs}}
    if extras:
        if R > 1 and rng.random() < 0.12:
            free_r = [r for r in range(R) if r not in rs]
            if free_r:
                d["all"] = (int(rng.choice(free_r)),)
        if rng.random() < 0.2:
            d["min_time_s"] = float(rng.choice([10.0, 30.0, 60.0, 120.0]))
    w = float(rng.choice([1.0, 1.0, 0.5, 2.0, 3.0]))
    if w != 1.0:
        d["weight"] = w
    return d


def make_scenario(seed: int) -> Scenario:
    rng = np.random.default_rng(7100 + seed)
    W = POOL_SIZES[seed % len(POOL_SIZES)]
    plain = seed % 4 == 1
    big_pool = W > 512
    if seed == 3:
        R = 16
    else:
        R = int(rng.choice([1, 2, 3, 4, 5, 6]) if big_pool else rng.integers(1, 17))
    # amounts: most resources carry a common factor (the 32-bit solve), some seeds have an odd ~2^40 resource (64-bit
    # only), and a resource may be unlimited (AMOUNT_MAX) on a few workers
    units = [int(rng.choice([2500, FR, 4 * FR])) for _ in range(R)]
    wide_r = int(rng.integers(0, R)) if rng.random() < 0.35 else -1
    if wide_r >= 0:
        units[wide_r] = (1 << 40) + 2 * int(rng.integers(0, 1 << 20)) + 1
    total = np.zeros((W, R), dtype=np.uint64)
    for r in range(R):
        t = rng.integers(8, 64, size=W).astype(object) * units[r]
        if units[r] < (1 << 32) and rng.random() < 0.5:
            t = t + rng.integers(0, units[r], size=W).astype(object)          # remainders on the workers
        total[:, r] = np.array([int(x) for x in t], dtype=np.uint64)
    if R > 1 and rng.random() < 0.3:
        r = int(rng.integers(0, R))
        total[rng.choice(W, size=min(W, 3), replace=False), r] = AMOUNT_MAX
    # classes
    if big_pool:
        Q, vmax = int(rng.integers(2, 9)), 3
    elif W > 64:
        Q, vmax = int(rng.integers(2, 13)), 4
    else:
        Q, vmax = int(rng.integers(1, 25)), 8
    classes, seen = [], set()
    while len(classes) < Q:
        nv = 1 if plain else int(rng.integers(1, vmax + 1))
        big = rng.random() < 0.2
        vs = [_variant(rng, R, units, big, not plain) for _ in range(nv)]
        if not plain and rng.random() < 0.2:
            # two variants of equal cost: the lower index must win the tie
            d = dict(vs[0]); d.pop("all", None)
            vs = [dict(d, min_time_s=float(rng.choice([30.0, 60.0]))), dict(d)] + vs[1:]
            if R > 1 and len(d["amounts"]) == 1:
                (r0, a0), = d["amounts"].items()
                vs.append({"amounts": {(r0 + 1) % R: a0}})
            vs = vs[:MAXV]
        key = repr([(sorted(x["amounts"].items()), x.get("all"), x.get("min_time_s"), x.get("weight")) for x in vs])
        if key not in seen:
            seen.add(key)
            classes.append(vs)
    termination = np.full(W, np.inf)
    min_util = None
    blocked = False
    if not plain:
        if rng.random() < 0.6:
            lim = rng.random(W) < 0.4
            termination[lim] = TICK_S * rng.integers(1, 13, size=int(lim.sum()))
        if rng.random() < 0.5 and W > 1:
            min_util = np.zeros(W, dtype=np.float32)
            ws = rng.choice(W, size=max(1, min(W // 8, 24)), replace=False)
            min_util[ws] = rng.choice([0.5, 0.75, 0.9, 0.97, 1.0], size=ws.size)
        blocked = rng.random() < 0.5
    prefill = None
    if (not plain and rng.random() < 0.5) or (plain and seed % 8 == 5):
        prefill = (int(rng.integers(0, 5)), int(rng.integers(1, 7)))
    pack = rng.random() < 0.7
    n_ticks = 4 if W >= 1000 else 5 if W > 256 else int(rng.integers(6, 11))
    # few levels, or many on small pools; live levels x Q x 2 stays under the group limit
    n_levels_cap = int(rng.choice([2, 4, 8])) if W > 65 or rng.random() < 0.5 else int(rng.integers(20, 120))
    if prefill is not None and rng.random() < 0.7:
        n_levels_cap = int(rng.choice([1, 2, 3]))         # a class's top level is often the global one: prefills happen
    n_levels_cap = max(1, min(n_levels_cap, (MAX_GROUPS - 64) // (2 * Q)))
    class_p = 1.0 / np.arange(1, Q + 1) ** 0.8
    return Scenario(seed, W, R, classes, total, termination, min_util, pack, prefill, n_ticks, plain, blocked,
                    n_levels_cap, class_p / class_p.sum())


def remaining_ms(termination: np.ndarray, now: float) -> np.ndarray:
    """GpuScheduler._worker_structs(now)["remaining_time_ms"] of a scheduler with these termination times."""
    from hyperqueue_b200.scheduler import GpuScheduler
    W = termination.shape[0]
    host = SimpleNamespace(worker_ids=np.arange(W, dtype=np.uint32), termination=termination,
                           min_utilization=np.zeros(W, dtype=np.float32))
    return GpuScheduler._worker_structs(host, now)["remaining_time_ms"].copy()


@dataclass
class TickInputs:
    wl: Workload                  # classes, totals, per-handle class and user priority, blocked mask
    ready: np.ndarray
    free: np.ndarray
    levels: np.ndarray
    remaining_ms: np.ndarray
    pf_before: np.ndarray         # per handle: worker index it was prefilled on at tick start, -1 = none
    now: float


class Drain:
    """The host state of one scenario and its events.  Every event is applied to the specification's state and to each
    context in `ctxs` (GpuScheduler objects, attached by the GPU test)."""

    def __init__(self, seed: int, model=None) -> None:
        self.sc = make_scenario(seed)
        self.rng = np.random.default_rng(9100 + seed)
        self.model = model or G.model_tick
        sc = self.sc
        self.ctxs: list = []
        self.H = 0
        self.task_class = np.zeros(0, dtype=np.uint32)
        self.task_prio = np.zeros(0, dtype=np.int32)
        self.ready = np.zeros(0, dtype=bool)
        self.pf = np.zeros(0, dtype=np.int64)
        self.task_worker = np.zeros(0, dtype=np.int64)
        self.task_variant = np.zeros(0, dtype=np.int64)
        self.finish_at: Dict[int, int] = {}       # running handle -> tick before which it finishes
        self.retired: List[int] = []             # handles free for re-use
        self.free = sc.total.copy()
        self.now = 0.0
        self.prio_values = sorted(int(x) for x in self.rng.choice(1000, size=max(1, min(sc.n_levels_cap, 8)), replace=False))
        self.blocked = None
        if sc.blocked:
            self.blocked = np.zeros((sc.W, len(sc.classes), MAXV), dtype=bool)
            self._flip_blocked(0.15)
        self.amounts, self.allm, self.nvar, self.mint = self.workload().class_tables()
        self.capacity = self._capacity()

    def _capacity(self) -> int:
        """Tasks of the class mix (first variants) the empty pool holds, roughly."""
        sc = self.sc
        tot = np.where(sc.total == AMOUNT_MAX, 0, sc.total).astype(np.float64)
        per_worker = 0.0
        for c, p in enumerate(sc.class_p):
            am = self.amounts[c, 0].astype(np.float64)
            used = am > 0
            fit = np.floor(tot[:, used] / am[used]).min(axis=1) if used.any() else np.full(sc.W, 16.0)
            per_worker += p * float(np.mean(np.minimum(fit, 64)))
        return max(4, int(sc.W * per_worker))

    # --- host state ------------------------------------------------------------------------------------------------
    def workload(self) -> Workload:
        sc = self.sc
        return Workload(sc.R, sc.classes, sc.total, self.free.copy(), self.task_class.copy(), self.task_prio.copy(),
                        blocked=None if self.blocked is None else self.blocked.copy())

    def _grow(self, n: int) -> None:
        if n > self.H:
            k = n - self.H
            self.task_class = np.concatenate([self.task_class, np.zeros(k, np.uint32)])
            self.task_prio = np.concatenate([self.task_prio, np.zeros(k, np.int32)])
            self.ready = np.concatenate([self.ready, np.zeros(k, bool)])
            self.pf = np.concatenate([self.pf, np.full(k, -1, np.int64)])
            self.task_worker = np.concatenate([self.task_worker, np.full(k, -1, np.int64)])
            self.task_variant = np.concatenate([self.task_variant, np.zeros(k, np.int64)])
            self.H = n

    def live_levels(self) -> np.ndarray:
        return np.unique(self.task_prio[self.ready].astype(np.int64))[::-1]

    def _new_priorities(self, n: int) -> np.ndarray:
        live = set(self.live_levels().tolist())
        if len(live) < self.sc.n_levels_cap and self.rng.random() < 0.5:
            # a fresh value: inside the range or above everything in the set
            hi = max(live | set(self.prio_values)) if live or self.prio_values else 0
            v = hi + int(self.rng.integers(1, 50)) if self.rng.random() < 0.5 else int(self.rng.integers(0, hi + 2))
            if v not in self.prio_values:
                self.prio_values.append(v)
        # only values that keep the live level count under the cap
        pool = [p for p in self.prio_values if p in live]
        room = self.sc.n_levels_cap - len(live)
        pool += [p for p in self.prio_values if p not in live][:max(room, 0)]
        if not pool:
            pool = [self.prio_values[0]]
        pool = pool[: self.sc.n_levels_cap]
        return np.asarray(self.rng.choice(pool, size=n), dtype=np.int32)

    def push(self, handles: np.ndarray) -> None:
        from hyperqueue_b200 import priority_from_user
        h = np.sort(np.asarray(handles, dtype=np.uint32))
        if h.size == 0:
            return
        self._grow(int(h.max()) + 1)
        cls = self.rng.choice(len(self.sc.classes), size=h.size, p=self.sc.class_p).astype(np.uint32)
        pr = self._new_priorities(h.size)
        self.task_class[h] = cls
        self.task_prio[h] = pr
        self.ready[h] = True
        self.pf[h] = -1
        for s in self.ctxs:
            s.add_ready_tasks(h, cls, priority_from_user(pr))

    def _flip_blocked(self, p: float) -> None:
        sc = self.sc
        nv = np.array([len(vs) for vs in sc.classes])
        flip = self.rng.random(self.blocked.shape) < p
        flip &= np.arange(MAXV)[None, None, :] < nv[None, :, None]
        self.blocked ^= flip
        for s in self.ctxs:
            s.set_blocked_mask(self.blocked)

    def _fits(self, w: int, c: int, v: int) -> bool:
        for r in range(self.sc.R):
            f, t = int(self.free[w, r]), int(self.sc.total[w, r])
            if self.allm[c, v, r]:
                if t == 0 or f != t:
                    return False
            elif self.amounts[c, v, r] and f != AMOUNT_MAX and f < int(self.amounts[c, v, r]):
                return False
        return True

    def _take(self, w: int, c: int, v: int) -> None:
        for r in range(self.sc.R):
            if self.allm[c, v, r]:
                self.free[w, r] = 0
            elif self.amounts[c, v, r] and int(self.free[w, r]) != AMOUNT_MAX:
                self.free[w, r] -= self.amounts[c, v, r]

    def _give(self, w: int, c: int, v: int) -> None:
        for r in range(self.sc.R):
            if self.allm[c, v, r]:
                self.free[w, r] = self.sc.total[w, r]
            elif self.amounts[c, v, r] and int(self.free[w, r]) != AMOUNT_MAX:
                self.free[w, r] += self.amounts[c, v, r]

    # --- events between ticks --------------------------------------------------------------------------------------
    def events(self, tick: int) -> None:
        rng, sc = self.rng, self.sc
        done = sorted(t for t, k in self.finish_at.items() if k <= tick)
        if done:
            h = np.array(done, dtype=np.uint32)
            for t in done:
                del self.finish_at[t]
                self._give(int(self.task_worker[t]), int(self.task_class[t]), int(self.task_variant[t]))
                self.task_worker[t] = -1
            for s in self.ctxs:
                s.tasks_finished(h)
                s.remove_ready_tasks(h)
            self.retired += done
        # cancel a few waiting tasks (never prefilled ones: the host's prefill mirror would keep them)
        waiting = np.nonzero(self.ready & (self.pf < 0))[0]
        if waiting.size and rng.random() < 0.5:
            h = np.sort(rng.choice(waiting, size=max(1, waiting.size // 30), replace=False)).astype(np.uint32)
            self.ready[h] = False
            for s in self.ctxs:
                s.remove_ready_tasks(h)
            self.retired += h.tolist()
        if sc.prefill is not None:
            held = np.nonzero(self.ready & (self.pf >= 0))[0]
            if held.size and rng.random() < 0.6:
                # a worker starts one of its prefilled tasks by itself, with a variant that fits
                for t in rng.permutation(held)[:4].tolist():
                    w, c = int(self.pf[t]), int(self.task_class[t])
                    vs = [v for v in range(int(self.nvar[c])) if self._fits(w, c, v)]
                    if not vs:
                        continue
                    v = int(vs[int(rng.integers(0, len(vs)))])
                    self.ready[t] = False
                    self.pf[t] = -1
                    self.task_worker[t], self.task_variant[t] = w, v
                    self._take(w, c, v)
                    self.finish_at[t] = tick + int(rng.integers(1, 4))
                    for s in self.ctxs:
                        s.on_task_running_prefilled(t, v)
                    break
            held = np.nonzero(self.ready & (self.pf >= 0))[0]
            if held.size and rng.random() < 0.25:
                c = int(self.task_class[int(rng.choice(held))])
                self.pf[(self.pf >= 0) & (self.task_class == c)] = -1
                for s in self.ctxs:
                    s.dispose_prefill(c)
        if self.blocked is not None and rng.random() < 0.5:
            self._flip_blocked(0.05)
        # new tasks: a handle range beyond everything so far, and scattered re-used handles
        # demand: enough to saturate the pool, with the backlog held to a few pool loads
        backlog = int(self.ready.sum())
        # some ticks are lulls: the backlog drains, so prefilled tasks get assigned (kind-2 redirects)
        n_new = int(self.capacity * rng.uniform(1.5, 2.5)) if tick == 0 else int(self.capacity * rng.uniform(0.5, 1.5))
        if tick > 0 and rng.random() < 0.3:
            n_new = int(self.capacity * rng.uniform(0.0, 0.2))
        n_new = max(1, min(n_new, 4 * self.capacity - backlog))
        n_reuse = min(len(self.retired), int(rng.integers(0, n_new // 2 + 1)))
        if n_reuse:
            pick = set(rng.choice(len(self.retired), size=n_reuse, replace=False).tolist())
            h = [x for i, x in enumerate(self.retired) if i in pick]
            self.retired = [x for i, x in enumerate(self.retired) if i not in pick]
            self.push(np.array(h, dtype=np.uint32))
        if n_new - n_reuse > 0:
            self.push(np.arange(self.H, self.H + n_new - n_reuse, dtype=np.uint32))
        self.now = tick * TICK_S

    # --- one tick ------------------------------------------------------------------------------------------------------
    def inputs(self) -> TickInputs:
        return TickInputs(self.workload(), self.ready.copy(), self.free.copy(), self.live_levels(),
                          remaining_ms(self.sc.termination, self.now), self.pf.copy(), self.now)

    def expected(self, inp: TickInputs, trace: Optional[dict] = None):
        sc = self.sc
        pf = inp.pf_before.copy()
        a, fa = self.model(inp.wl, inp.ready, inp.free, inp.levels, remaining_ms=inp.remaining_ms, pack=sc.pack,
                           min_utilization=sc.min_util, prefill=sc.prefill, pf_worker=pf if sc.prefill else None,
                           trace=trace)
        return a, fa, pf

    def apply(self, tick: int, a: np.ndarray, free_after: np.ndarray, pf_after: np.ndarray) -> None:
        asg = a[a["kind"] != 1]
        self.ready[asg["task"]] = False
        self.task_worker[asg["task"]] = asg["worker"]
        self.task_variant[asg["task"]] = asg["variant"]
        for t in asg["task"].tolist():
            self.finish_at[t] = tick + 1 + int(self.rng.integers(0, 3))
        self.free = free_after.copy()
        self.pf = pf_after.copy()

    def run(self, check: Optional[Callable] = None, trace: bool = False):
        """Runs the drain; returns per tick (inputs, records, free_after, trace or None)."""
        out = []
        for tick in range(self.sc.n_ticks):
            self.events(tick)
            inp = self.inputs()
            tr = {} if trace else None
            a, fa, pf = self.expected(inp, tr)
            if check is not None:
                check(tick, inp, a, fa, pf)
            self.apply(tick, a, fa, pf)
            out.append((inp, a, fa, tr))
        return out


def gpu_context(d: Drain, flags: int = 0):
    """A GpuScheduler set up as the scenario's server: classes, workers, termination, min-utilisation, blocked mask,
    proactive filling; `flags` are hqs_create flags (NO_PACK follows the scenario)."""
    from hyperqueue_b200 import GpuScheduler, RequestVariant, _lib as L
    sc = d.sc
    s = GpuScheduler(sc.R, 0, flags | (0 if sc.pack else L.HQS_CREATE_NO_PACK))
    for c, vs in enumerate(sc.classes):
        rid = s.get_or_create_resource_rq_id([RequestVariant.of(v["amounts"], v.get("all", ()), v.get("weight", 1.0),
                                                                v.get("min_time_s", 0.0)) for v in vs])
        assert rid == c
    s.new_workers_bulk(np.arange(sc.W, dtype=np.uint32), sc.total)
    s.termination = sc.termination.copy()
    if sc.min_util is not None:
        s.min_utilization = sc.min_util.copy()
    if d.blocked is not None:
        s.set_blocked_mask(d.blocked)
    if sc.prefill is not None:
        s.set_prefill(*sc.prefill)
    s._sync_classes()
    return s


# --- checks shared by the CPU and GPU tests --------------------------------------------------------------------------
def judge_and_replay(d: Drain, inp: TickInputs, a: np.ndarray, free_after: np.ndarray) -> Optional[str]:
    """The tick's assignments (kind 0 and 2) are feasible, no handle is placed twice, prefill records name ready tasks
    that were not assigned, and free_after is the exact replay.  Returns a message or None."""
    asg = a[a["kind"] != 1]
    res = J.judge_assignments(d.amounts, d.allm, d.nvar, d.mint, inp.free, d.sc.total, inp.remaining_ms, inp.wl.blocked,
                              inp.wl.task_class, asg["task"], asg["worker"], asg["variant"], inp.ready)
    if not res.ok:
        return f"judge: {res.violations}"
    if np.unique(a["task"]).size != a.size:
        return "a handle was placed twice"
    pf = a[a["kind"] == 1]
    if pf.size and not (inp.ready[pf["task"]].all() and (inp.pf_before[pf["task"]] < 0).all()):
        return "a prefill record names a task that was not waiting"
    rep = J.replay_free_after(d.amounts, d.allm, inp.free, d.sc.total, inp.wl.task_class, asg["task"], asg["worker"],
                              asg["variant"])
    if not np.array_equal(rep, free_after):
        return "free_after differs from the exact replay"
    pr = inp.wl.task_user_priority[asg["task"]].astype(np.int64)
    if pr.size and (np.diff(pr) > 0).any():
        return "an assignment is emitted before one of higher priority"
    return None


def first_difference(inp: TickInputs, got: np.ndarray, want: np.ndarray) -> str:
    """The first record where two tick outputs differ, with its task's class, level and variant."""
    n = min(got.size, want.size)
    neq = np.nonzero(got[:n] != want[:n])[0]
    i = int(neq[0]) if neq.size else n
    lvl = {int(p): k for k, p in enumerate(inp.levels.tolist())}

    def rec(a):
        if i >= a.size:
            return "(none)"
        t = int(a[i]["task"])
        return (f"task {t} class {int(inp.wl.task_class[t])} level {lvl.get(int(inp.wl.task_user_priority[t]))} "
                f"-> worker {int(a[i]['worker'])} variant {int(a[i]['variant'])} kind {int(a[i]['kind'])}")
    return f"record {i} of {got.size} / {want.size}: got {rec(got)}, want {rec(want)}"
