"""Sequential CPU specification of the DEVICE algorithm (hyperqueue_b200/csrc/hqsched.cu).

Test infrastructure: it is neither the oracle (which restates the reference's MILP) nor a product
fallback.  It exists so that (a) the design can be compared with the oracle on the CPU-only box and
(b) the CUDA path can be checked for bit-exact equality with a short specification of itself.

The algorithm, per tick:
  levels (distinct priorities, descending) x classes (the tick's class order) = groups; groups are
  processed in that order.  The FIRST level whose demand exceeds the aggregate free capacity is
  "packed": the level's class counts are pre-split over the workers (share proportional to how many
  tasks of the class fit on the worker alone, scaled by phi = the fraction of the level's demand the
  pool can serve, so that every class of the level progresses at the same rate) and every worker then
  fills ITSELF, independently: per class it considers the variant that costs the smallest share of what
  the worker has left (min over variants of max_r amount_r / free_r), and takes from the class whose such
  variant is best aligned with its remaining capacity (normalised dot product, the vector-bin-packing
  heuristic) — this is what makes one tick use cpus, gpus and memory together the way the reference's
  MILP objective (sum of normalised utilisations, solver.rs:520-549) does.  Everything else — levels
  before and after, and whatever the packed level could not place — is priority-ordered first-fit over
  workers in ascending id (compaction, solver.rs (n - w_idx)/n); a worker tries the variants of a class in
  ascending order of the same "share of what I have left" cost, re-evaluated after each variant.
Mirrors tick_orders() (hqsched.cu), solver_cta() / emit_chunk() (hqs_tick.cuh) and pack_body() (hqs_solver.cuh).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import numpy as np

from workloads import FR, MAXV, Workload

AMOUNT_MAX = (1 << 64) - 1
TIME_INF = (1 << 64) - 1
U64 = (1 << 64) - 1
PACK_MAX_CAND = 64        # candidates (class, variant) of the packed level; more => plain first-fit
PACK_MAX_ITER = 64        # fill iterations per worker
PACK_CHUNK_DIV = 8        # a pick takes at most max(1, quota / 8) tasks

assignment_dtype = np.dtype([("task", "<u4"), ("worker", "<u2"), ("variant", "u1"), ("kind", "u1")])


def class_order(wl: Workload, free: np.ndarray, total: np.ndarray) -> List[int]:
    W, R = free.shape
    S = [0.0] * R
    T = [0.0] * R
    for w in range(W):
        for r in range(R):
            f = int(free[w, r]); t = int(total[w, r])
            S[r] += 1.0 if f == AMOUNT_MAX else f / 10000.0
            T[r] += 1.0 if t == AMOUNT_MAX else t / 10000.0
    scores = []
    for c, vs in enumerate(wl.classes):
        best = 0.0
        for d in vs:
            s = 0.0
            for r in range(R):
                if S[r] < 1e-6:
                    continue
                if r in d.get("all", ()):
                    s += (T[r] / max(W, 1)) / S[r]
                else:
                    s += (int(d["amounts"].get(r, 0)) / 10000.0) / S[r]
            s *= int(np.round(np.float32(d.get("weight", 1.0)) * np.float32(10000))) / 10000.0
            best = max(best, s)
        scores.append((best, c))
    return [c for _, c in sorted(scores, key=lambda sc: -sc[0])]      # stable


def variant_order(wl: Workload, free: np.ndarray) -> List[List[int]]:
    """Per class: variants by ascending dominant share max_r amount_r / S_r (S_r = total free of r at tick
    start): the variant that costs least of the scarcest thing it touches is tried first."""
    W, R = free.shape
    S = [0.0] * R
    for w in range(W):
        for r in range(R):
            f = int(free[w, r])
            S[r] += 1.0 if f == AMOUNT_MAX else f / 10000.0
    out = []
    for vs in wl.classes:
        doms = []
        for v, d in enumerate(vs):
            dom = 0.0
            for r in range(R):
                a = int(d["amounts"].get(r, 0))
                if a:
                    x = float("inf") if S[r] < 1e-6 else (a / 10000.0) / S[r]
                    dom = x if x > dom else dom
            if d.get("all", ()):
                dom = float("inf")
            doms.append((dom, v))
        out.append([v for _, v in sorted(doms, key=lambda dv: dv[0])])      # stable
    return out


def _sat_add(a: int, b: int) -> int:
    return min(a + b, U64)


def _sat_mul(a: int, b: int) -> int:
    return min(a * b, U64)


class _Tick:
    def __init__(self, wl: Workload, free: np.ndarray, remaining_ms: np.ndarray) -> None:
        self.wl = wl
        self.W, self.R = free.shape
        self.fr = [[int(x) for x in free[w]] for w in range(self.W)]
        self.fr0 = [list(x) for x in self.fr]
        self.tot = [[int(x) for x in wl.worker_total[w]] for w in range(self.W)]
        self.rem_ms = [int(x) for x in remaining_ms]
        self.am = [[{r: int(a) for r, a in d["amounts"].items()} for d in vs] for vs in wl.classes]
        self.alls = [[tuple(d.get("all", ())) for d in vs] for vs in wl.classes]
        self.min_ms = [[int(round(d.get("min_time_s", 0.0) * 1000)) for d in vs] for vs in wl.classes]
        self.excluded = None
        self.trace = None                        # model_tick's `trace` dict, or None
        self.pass_no = 0
        self.touched = [False] * self.W          # the worker received something in this tick
        self.noresv = set()                      # classes for which no worker can be reserved any more

    def capable(self, w: int, c: int) -> bool:
        """Worker::is_capable_to_run_rqv (worker.rs:280-299): some variant fits the TOTALS and the remaining time."""
        tot, rt = self.tot[w], self.rem_ms[w]
        for v in range(len(self.am[c])):
            if rt != TIME_INF and self.min_ms[c][v] > rt:
                continue
            if all(a <= tot[r] for r, a in self.am[c][v].items()) and all(tot[r] != 0 for r in self.alls[c][v]):
                return True
        return False

    def reserve(self, c: int, n_all: int, remaining: int) -> None:
        """Reservations (solver.rs:133-151): a class that is left with unplaced tasks may claim workers that are big
        enough for it (by their totals) but cannot take a single task of it right now — such a worker receives nothing
        in this tick, so that running tasks drain and the waiting class gets in instead of being starved by lower
        priorities.  As in the reference: only workers without a placement variable for the class (nothing of it fits at
        tick start) and without any assignment in this tick, at most one per unplaced task, only while the class's count
        does not exceed the batch limit (batches.rs:80-91: every capable worker counts at least once), and the MILP's
        preference for HIGH worker indices (coefficient w_idx / (100 n)) is kept."""
        if c in self.noresv:
            return
        cap = [w for w in range(self.W) if self.capable(w, c)]
        limit = 0
        for w in cap:
            limit += max(1, sum(min(self.fit_start(w, c, v), 1024) for v in range(len(self.am[c]))))
        got = 0
        if n_all <= limit:
            for w in reversed(cap):
                if got >= remaining:
                    break
                if (self.excluded is not None and self.excluded[w]) or self.touched[w]:
                    continue
                if any(self.fit_start(w, c, v) > 0 for v in range(len(self.am[c]))):
                    continue
                self.excluded[w] = True
                got += 1
                if self.trace is not None:
                    self.trace["reserved"].append((self.pass_no, w, c))
        if got < remaining:
            self.noresv.add(c)            # eligibility only shrinks during a tick

    def fit_start(self, w: int, c: int, v: int) -> int:
        """task_max_count of variant v against the free vector at tick start, blocked requests ignored (workerload.rs:121-145)."""
        fr, tot = self.fr0[w], self.tot[w]
        cnt = U64
        for r in range(self.R):
            if r in self.alls[c][v]:
                cnt = min(cnt, 1 if fr[r] != 0 else 0)
            elif r in self.am[c][v] and fr[r] != AMOUNT_MAX:
                cnt = min(cnt, fr[r] // self.am[c][v][r])
        return cnt

    def admissible(self, w: int, c: int, v: int) -> bool:
        if self.excluded is not None and self.excluded[w]:
            return False
        if self.wl.blocked is not None and self.wl.blocked[w, c, v]:
            return False
        rt = self.rem_ms[w]
        return rt == TIME_INF or self.min_ms[c][v] <= rt

    def fit(self, w: int, c: int, v: int, cap: int) -> int:
        """How many tasks of (c, v) fit on worker w now, at most `cap`."""
        if not self.admissible(w, c, v):
            if self.trace is not None and not (self.excluded is not None and self.excluded[w]):
                self._trace_rejection(w, c, v)
            return 0
        cnt = cap
        fr, tot = self.fr[w], self.tot[w]
        for r in range(self.R):
            if r in self.alls[c][v]:
                cnt = min(cnt, 1 if (tot[r] != 0 and fr[r] == tot[r]) else 0)
            elif r in self.am[c][v] and fr[r] != AMOUNT_MAX:
                cnt = min(cnt, fr[r] // self.am[c][v][r])
        return cnt

    def _trace_rejection(self, w: int, c: int, v: int) -> None:
        """Records a blocked or time-limited (worker, class, variant) cell whose resources would take a task now."""
        fr, tot = self.fr[w], self.tot[w]
        for r in range(self.R):
            if r in self.alls[c][v]:
                if not (tot[r] != 0 and fr[r] == tot[r]):
                    return
            elif r in self.am[c][v] and fr[r] != AMOUNT_MAX and fr[r] < self.am[c][v][r]:
                return
        why = "blocked" if self.wl.blocked is not None and self.wl.blocked[w, c, v] else "time"
        self.trace["rejected"].append((why, w, c, v))

    def next_variant(self, w: int, c: int, tried: int) -> int:
        """The untried variant of class c that costs the smallest share of what worker w has left:
        min over variants of max_r f32(amount_r) * (1 / f32(free_r)) in IEEE single (u64 -> double -> single,
        both round-to-nearest); a variant with an `All` entry costs +inf; ties: lower variant index."""
        nv = len(self.am[c])
        if nv == 1:
            return 0
        fr = self.fr[w]
        best, best_d = -1, np.float32(0)
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            inv = [np.float32(1.0) / np.float32(float(fr[r])) for r in range(self.R)]
            for v in range(nv):
                if (tried >> v) & 1:
                    continue
                dom = np.float32(0)
                if self.alls[c][v]:
                    dom = np.float32(np.inf)
                else:
                    for r in range(self.R):
                        a = self.am[c][v].get(r)
                        if a is None or fr[r] == AMOUNT_MAX:
                            continue
                        x = np.float32(float(a)) * inv[r]
                        dom = x if x > dom else dom
                if best < 0 or dom < best_d:
                    best, best_d = v, dom
        return best

    def take(self, w: int, c: int, v: int, k: int) -> None:
        fr = self.fr[w]
        if k:
            self.touched[w] = True
        for r in range(self.R):
            if r in self.alls[c][v]:
                fr[r] = 0
            elif r in self.am[c][v] and fr[r] != AMOUNT_MAX:
                fr[r] -= k * self.am[c][v][r]

    def give_back(self, w: int, c: int, v: int, k: int) -> None:
        fr = self.fr[w]
        for r, a in self.am[c][v].items():
            if fr[r] != AMOUNT_MAX:
                fr[r] += k * a


def _level_is_saturated(t: _Tick, groups: List[Tuple[int, int]], vorder: List[List[int]]) -> Tuple[bool, float]:
    """Demand of the level (each class with its first variant of the tick's variant order) against the
    aggregate free capacity, exact saturating u64 arithmetic.  Returns (saturated, phi) with
    phi = min(1, min_r capacity_r / demand_r) in IEEE double (u64 -> double round-to-nearest) when at
    least two resources are over-subscribed, else 1."""
    R, W = t.R, t.W
    C = [0] * R
    for r in range(R):
        s = 0
        for w in range(W):
            if t.excluded is not None and t.excluded[w]:
                continue
            s = U64 if t.fr[w][r] == AMOUNT_MAX else _sat_add(s, t.fr[w][r])
            if s == U64:
                break
        C[r] = s
    tot_max = [max(t.tot[w][r] for w in range(W)) for r in range(R)]
    D = [0] * R
    for c, n in groups:
        am = t.am[c][vorder[c][0]]
        if any(a > tot_max[r] for r, a in am.items()):
            continue            # no worker is big enough for it: it is not demand that capacity could serve
        for r, a in am.items():
            D[r] = _sat_add(D[r], _sat_mul(n, a))
    n_sat = sum(1 for r in range(R) if C[r] != U64 and D[r] > C[r])
    phi = 1.0
    if n_sat >= 2:
        # two or more scarce resources: classes complement each other, so each gets the same fraction of its
        # demand this tick.  With a single scarce resource every split drains at the same rate and the
        # alignment order alone (the reference objective's preference) decides.
        for r in range(R):
            if C[r] != U64 and D[r] > 0:
                x = float(C[r]) / float(D[r])
                phi = x if x < phi else phi
    return n_sat > 0, phi


def _pack_quota(n: int, cn: int, T: int, phi: float) -> int:
    """A worker's share of a packed class: ceil(n * cn / T), scaled by phi and rounded up again."""
    return int(math.ceil(float(-(-n * cn // T)) * phi))


def _pack_level(t: _Tick, groups: List[Tuple[int, int]], phi: float) -> Dict[Tuple[int, int], List[int]]:
    """Every worker fills itself (its free vector is consumed).  Returns taken[(group index, variant)][w]."""
    W, R = t.W, t.R
    cands = [(gi, c, v) for gi, (c, n) in enumerate(groups) for v in range(len(t.am[c]))]
    # a. per-worker quotas
    quota = [[0] * len(groups) for _ in range(W)]
    for gi, (c, n) in enumerate(groups):
        cn = [max(t.fit(w, c, v, n) for v in range(len(t.am[c]))) for w in range(W)]
        T = sum(cn)
        if T:
            for w in range(W):
                quota[w][gi] = _pack_quota(n, cn[w], T, phi)
    # b. every worker fills itself
    taken: Dict[Tuple[int, int], int] = {}       # (w, candidate index) -> count
    for w in range(W):
        tot = t.tot[w]
        # reciprocals once per worker / candidate: the per-iteration score is multiply-add only
        inv_tot = [(1.0 / float(tot[r])) if (tot[r] != 0 and tot[r] != AMOUNT_MAX) else 0.0 for r in range(R)]
        dvec, inv_norm = [], []
        for (gi, c, v) in cands:
            d = [0.0] * R
            for r, a in t.am[c][v].items():
                d[r] = float(a) * inv_tot[r]
            s2 = 0.0
            for r in range(R):
                s2 = s2 + d[r] * d[r]
            nrm = math.sqrt(s2)
            dvec.append(d)
            inv_norm.append((1.0 / nrm) if nrm > 0.0 else 0.0)
        for _ in range(PACK_MAX_ITER):
            fr = t.fr[w]
            u = [float(fr[r]) * inv_tot[r] for r in range(R)]
            inv_u = [(1.0 / u[r]) if u[r] != 0.0 else float("inf") for r in range(R)]
            # per group: the feasible variant with the smallest dominant share (ties: lower candidate index)
            pick: Dict[int, Tuple[float, int]] = {}
            for ci, (gi, c, v) in enumerate(cands):
                if quota[w][gi] <= 0 or not t.admissible(w, c, v):
                    continue
                if any(fr[r] != AMOUNT_MAX and a > fr[r] for r, a in t.am[c][v].items()):
                    continue
                # dominant share of what the worker has left: max_r (amount_r / total_r) * (1 / (free_r / total_r))
                dom = 0.0
                for r in range(R):
                    if dvec[ci][r] > 0.0:
                        x = dvec[ci][r] * inv_u[r]
                        dom = x if x > dom else dom
                if gi not in pick or dom < pick[gi][0]:
                    pick[gi] = (dom, ci)
            best, best_s = -1, 0.0
            for ci, (gi, c, v) in enumerate(cands):
                if gi not in pick or pick[gi][1] != ci:
                    continue
                dot = 0.0
                for r in range(R):
                    dot = dot + dvec[ci][r] * u[r]
                s = dot * inv_norm[ci]
                if best < 0 or s > best_s:
                    best, best_s = ci, s
            if best < 0:
                break
            gi, c, v = cands[best]
            q = quota[w][gi]
            k = min(t.fit(w, c, v, q), max(1, q // PACK_CHUNK_DIV))
            t.take(w, c, v, k)
            quota[w][gi] -= k
            taken[(w, best)] = taken.get((w, best), 0) + k
    res: Dict[Tuple[int, int], List[int]] = {}
    for ci, (gi, c, v) in enumerate(cands):
        res[(gi, v)] = [taken.get((w, ci), 0) for w in range(W)]
    return res


def model_tick(wl: Workload, ready: np.ndarray, free: np.ndarray, levels: Optional[np.ndarray] = None,
               remaining_ms: Optional[np.ndarray] = None, pack: bool = True,
               min_utilization: Optional[np.ndarray] = None, prefill: Optional[Tuple[int, int]] = None,
               pf_worker: Optional[np.ndarray] = None, trace: Optional[dict] = None) -> Tuple[np.ndarray, np.ndarray]:
    """Returns (assignments in device emission order, free_after).

    trace: an optional dict that collects the tick's decisions (it does not change them): "reserved" [(pass, worker,
    class)], "mu_excluded" [[workers newly excluded by pass p] ...] (one list per restart), "give_back" [(worker, class,
    variant, count)] of pack, "variant_takes" [(worker, class, variant, try)] of first-fit takes that were not the worker's
    first variant choice (try > 0), "rejected" [("blocked" | "time", worker, class, variant)] of cells whose resources
    would have taken a task.

    min_utilization (solver.rs:154-156, 479-518): a worker either receives at least
    min_cpus = total * (mu - 1) + free cpus of new work in this tick, or nothing.  A violating worker is taken out of
    the tick and the solve starts over (at most MU_MAX_PASSES - 1 times), so its tasks go to the other workers."""
    W = free.shape[0]
    excluded = np.zeros(W, dtype=bool)
    if trace is not None:
        for k in ("reserved", "mu_excluded", "give_back", "variant_takes", "rejected"):
            trace.setdefault(k, [])
    for p in range(MU_MAX_PASSES):
        a, fa = _solve_pass(wl, ready, free, levels, remaining_ms, pack, excluded, pf_worker, trace, p)
        if min_utilization is None or p + 1 >= MU_MAX_PASSES:
            return _with_prefill(wl, ready, a, levels, prefill, pf_worker), fa
        viol = False
        newly = []
        for w in range(W):
            mu = float(np.float32(min_utilization[w]))
            t0, f0 = int(wl.worker_total[w, 0]), int(free[w, 0])
            if excluded[w] or not (np.float32(min_utilization[w]) > np.float32(0.001)) or t0 == AMOUNT_MAX or f0 == AMOUNT_MAX:
                continue
            min_cpus = (float(t0) / 10000.0) * (mu - 1.0) + float(f0) / 10000.0
            new_cpus = float(f0 - int(fa[w, 0])) / 10000.0
            if min_cpus >= 0.0001 and new_cpus > 0.0 and new_cpus < min_cpus - 1e-9:
                excluded[w] = True
                viol = True
                newly.append(w)
        if trace is not None and newly:
            trace["mu_excluded"].append(newly)
        if not viol:
            return _with_prefill(wl, ready, a, levels, prefill, pf_worker), fa
    raise AssertionError("unreachable")


def _with_prefill(wl: Workload, ready: np.ndarray, a: np.ndarray, levels, prefill, pf_worker) -> np.ndarray:
    """Proactive filling (mapping.rs:156-230) and the retract / redirect marking (mapping.rs:63-101) on top of a tick's
    assignments.  pf_worker[t] = worker a ready task is prefilled on (-1: none) is updated in place:
      * an assigned task that was prefilled comes out with kind = 2 (RetractTasks to its old worker + redirect to the
        new one, even if they are the same worker, as in the reference) and is no longer prefilled,
      * then, for every class whose best waiting (not prefilled) priority level is the best one over all classes:
        size = waiting tasks of that level - reserve (0 if the class still has prefilled tasks at another level,
        taskqueue.rs:237-253); eligible workers = those that received an ASSIGNMENT (kind 0) of the class in this tick and
        held no prefilled task of it at tick start (the host's mirror; the reference looks after this tick's retracts);
        each gets min(size // eligible, max) of the level's next waiting tasks in handle
        order: records with kind = 1 after all assignments, classes ascending, workers ascending.  The tasks stay ready."""
    if prefill is None or prefill[1] <= 0:
        return a
    reserve, pmax = prefill
    if pf_worker is None:
        raise ValueError("prefill needs the pf_worker state array")
    W = wl.n_workers
    out = a.copy()
    pf_start = pf_worker.copy()          # "holds a prefilled task of the class" is the host's view at tick start
    was_pf = pf_worker[out["task"]] >= 0
    out["kind"][was_pf] = 2
    pf_worker[out["task"][was_pf]] = -1
    prio = wl.task_user_priority.astype(np.int64)
    if levels is None:
        levels = np.unique(prio)[::-1]
    still = ready.copy()
    still[out["task"]] = False
    waiting = np.nonzero(still & (pf_worker < 0))[0]
    if waiting.size == 0:
        return out
    lvl_of = {int(p): i for i, p in enumerate(np.asarray(levels).tolist())}
    lv = np.array([lvl_of[int(p)] for p in prio[waiting]])
    cls = wl.task_class[waiting]
    top_c = {}
    for c in np.unique(cls).tolist():
        top_c[int(c)] = int(lv[cls == c].min())
    g_top = min(top_c.values())
    extra = []
    for c in sorted(top_c):
        if top_c[c] != g_top:
            continue
        pf_here = np.nonzero(ready & (pf_worker >= 0) & (wl.task_class == c))[0]
        if pf_here.size and any(lvl_of[int(p)] != g_top for p in prio[pf_here]):
            continue
        cand = waiting[(cls == c) & (lv == g_top)]                    # ascending handle
        size = cand.size - reserve
        if size <= 0:
            continue
        got = np.unique(out["worker"][(out["kind"] == 0) & (wl.task_class[out["task"]] == c)])
        elig = [int(w) for w in got.tolist() if not _holds_prefill(pf_start, ready, wl.task_class, w, c)]
        if not elig:
            continue
        ps = min(size // len(elig), pmax)
        if ps == 0:
            continue
        pos = 0
        for w in elig:
            for t in cand[pos: pos + ps].tolist():
                extra.append((t, w, 255, 1))          # variant = None
                pf_worker[t] = w
            pos += ps
    if extra:
        out = np.concatenate([out, np.array(extra, dtype=assignment_dtype)])
    return out


def _holds_prefill(pf_start: np.ndarray, ready: np.ndarray, task_class: np.ndarray, w: int, c: int) -> bool:
    """Worker w held a prefilled task of class c at tick start (Worker::prefilled_tasks, the host's mirror)."""
    return bool(np.any((pf_start == w) & ready & (task_class == c)))


MU_MAX_PASSES = 8


def _solve_pass(wl: Workload, ready: np.ndarray, free: np.ndarray, levels, remaining_ms, pack: bool,
                excluded: np.ndarray, pf_worker: Optional[np.ndarray] = None, trace: Optional[dict] = None,
                pass_no: int = 0) -> Tuple[np.ndarray, np.ndarray]:
    W, R = free.shape
    prio = wl.task_user_priority.astype(np.int64)
    if levels is None:
        levels = np.unique(prio)[::-1]
    if remaining_ms is None:
        remaining_ms = wl.remaining_ms()
    t = _Tick(wl, free, remaining_ms)
    t.excluded = [bool(x) for x in excluded]
    t.trace, t.pass_no = trace, pass_no
    # reservations can only exist when some worker is partly occupied at tick start (free != total)
    t.any_partial = any(t.fr0[w][r] != t.tot[w][r] for w in range(W) for r in range(R))
    order = class_order(wl, free, wl.worker_total)
    vorder = variant_order(wl, free)
    out: List[Tuple[int, int, int, int]] = []
    ready_idx = np.nonzero(ready)[0]
    key_p = prio[ready_idx]
    packed = not pack
    for lvl in levels.tolist():
        in_lvl = ready_idx[key_p == lvl]
        if in_lvl.size == 0:
            continue
        cls_lvl = wl.task_class[in_lvl]
        if pf_worker is None:
            tasks_of = {c: in_lvl[cls_lvl == c] for c in order}
            groups = [(c, int(tasks_of[c].size)) for c in order if tasks_of[c].size]
            gkeys = [c for c, _ in groups]
        else:
            # prefilled tasks of a (level, class) come after its waiting ones (take_tasks, taskqueue.rs:320-355): two groups
            pf_lvl = pf_worker[in_lvl] >= 0
            tasks_of, groups, gkeys = {}, [], []
            for c in order:
                for pfb in (False, True):
                    sel = in_lvl[(cls_lvl == c) & (pf_lvl == pfb)]
                    if sel.size:
                        tasks_of[(c, pfb)] = sel
                        groups.append((c, int(sel.size)))
                        gkeys.append((c, pfb))
        taken: Dict[Tuple[int, int], List[int]] = {}
        if not packed:
            n_cand = sum(len(t.am[c]) for c, _ in groups)
            has_all = any(t.alls[c][v] for c, _ in groups for v in range(len(t.am[c])))
            if n_cand <= PACK_MAX_CAND and len(groups) <= PACK_MAX_CAND and not has_all:
                saturated, phi = _level_is_saturated(t, groups, vorder)
                if saturated:
                    before = list(t.touched)
                    taken = _pack_level(t, groups, phi)
                    packed = True
                    # a worker whose pack takes are all handed back below received no assignment: it can still be
                    # reserved.  The capping of every group is known now, so `touched` is what the workers keep.
                    t.touched = before
                    for gi, (c, n) in enumerate(groups):
                        pos = 0
                        for v in range(len(t.am[c])):
                            for w, k in enumerate(taken[(gi, v)]):
                                use = min(k, n - pos)
                                if use > 0:
                                    t.touched[w] = True
                                    pos += use
        for gi, (c, n) in enumerate(groups):
            tasks = tasks_of[gkeys[gi]]
            pos = 0
            # cap what the workers took for this class at its count, (variant, worker) order; hand the
            # excess back
            for v in range(len(t.am[c])):
                tk = taken.get((gi, v))
                if tk is None:
                    continue
                for w in range(W):
                    k = tk[w]
                    if not k:
                        continue
                    use = min(k, n - pos)
                    if use < k:
                        t.give_back(w, c, v, k - use)
                        if trace is not None:
                            trace["give_back"].append((w, c, v, k - use))
                    for tt in tasks[pos: pos + use].tolist():
                        out.append((tt, w, v, 0))
                    pos += use
            remaining = n - pos
            nv = len(t.am[c])
            tried = [0] * W
            for vi in range(nv):
                if remaining == 0:
                    break
                for w in range(W):
                    if remaining == 0:
                        break
                    v = t.next_variant(w, c, tried[w])
                    tried[w] |= 1 << v
                    cnt = t.fit(w, c, v, remaining)
                    if cnt <= 0:
                        continue
                    t.take(w, c, v, cnt)
                    if trace is not None and vi:
                        trace["variant_takes"].append((w, c, v, vi))
                    for tt in tasks[pos: pos + cnt].tolist():
                        out.append((tt, w, v, 0))
                    pos += cnt
                    remaining -= cnt
            if remaining and t.any_partial:
                t.reserve(c, n, remaining)
    a = np.array(out, dtype=assignment_dtype) if out else np.zeros(0, dtype=assignment_dtype)
    return a, np.array(t.fr, dtype=np.uint64)


def model_drain(wl: Workload, max_ticks: int = 100000, pack: bool = True):
    """Zero-duration drain with the model (independent tasks or DAG)."""
    n = wl.n_tasks
    if wl.deps is None:
        ready = np.ones(n, dtype=bool)
        unfinished = None
    else:
        unfinished = np.array([len(d) for d in wl.deps], dtype=np.int64)
        ready = unfinished == 0
        consumers = [[] for _ in range(n)]
        for t, ds in enumerate(wl.deps):
            for d in ds:
                consumers[d].append(t)
    levels = np.unique(wl.task_user_priority.astype(np.int64))[::-1]
    remaining = n
    per_tick = []
    while remaining > 0 and len(per_tick) < max_ticks:
        a, _ = model_tick(wl, ready, wl.worker_free, levels, pack=pack)
        if a.size == 0:
            raise RuntimeError("model drain stalled")
        ready[a["task"]] = False
        if unfinished is not None:
            for t in a["task"].tolist():
                for c in consumers[t]:
                    unfinished[c] -= 1
                    if unfinished[c] == 0:
                        ready[c] = True
        remaining -= a.size
        per_tick.append(int(a.size))
    return len(per_tick), per_tick
