"""The specification (tests/greedy_model.py) alone over the multi-tick drains of tests/drain_fuzz.py: every tick is feasible
and exactly replayable, and the seed set reaches the states where the solve loops' tile bookkeeping matters (reservations
and pack hand-backs beyond the first tile, minimum-utilisation restarts, prefills and redirects on workers >= 32, blocked
and time-limited cells that turn a fitting task away).  Mutants of the specification, each a small plausible slip of the
device, must change some tick of the seed set: the GPU comparison (tests/test_gpu_drain_fuzz.py) sees those decisions."""
import dataclasses
import math

import numpy as np
import pytest

import drain_fuzz as D
import greedy_model as G
from workloads import FR, Workload

RESULTS: dict = {}           # seed -> [(inputs, records, free_after, trace)] per tick
MUTANT_SEEDS = tuple(s for s in D.SEEDS if D.POOL_SIZES[s % len(D.POOL_SIZES)] <= 256)


def _drain(seed):
    if seed not in RESULTS:
        RESULTS[seed] = D.Drain(seed).run(trace=True)
    return RESULTS[seed]


@pytest.mark.parametrize("seed", D.SEEDS)
def test_specification_drain_is_feasible(seed):
    d = D.Drain(seed)

    def check(tick, inp, a, fa, pf):
        msg = D.judge_and_replay(d, inp, a, fa)
        assert msg is None, f"seed {seed} tick {tick}: {msg}"
        # the drain's prefill state is the specification's: every ready task prefilled at most once, on a real worker
        assert ((pf >= -1) & (pf < d.sc.W)).all() and (pf[~inp.ready] < 0).all()
    RESULTS[seed] = d.run(check, trace=True)


def test_seed_set_reaches_the_tile_states():
    stats = {"resv32": 0, "resv512": 0, "mu32": 0, "gb_tile1": 0, "k1_32": 0, "k2_32": 0, "blocked": 0, "time": 0,
             "other_variant": 0, "ticks": 0, "left": 0, "empty": 0}
    for seed in D.SEEDS:
        for inp, a, fa, tr in _drain(seed):
            res = [w for _, w, _ in tr["reserved"]]
            stats["resv32"] += sum(w >= 32 for w in res)
            stats["resv512"] += sum(w >= 512 for w in res)
            stats["mu32"] += sum(w >= 32 for ws in tr["mu_excluded"] for w in ws)      # each list is followed by a restart
            stats["gb_tile1"] += sum(w >= 32 for w, *_ in tr["give_back"])
            stats["k1_32"] += int(np.count_nonzero((a["kind"] == 1) & (a["worker"] >= 32)))
            stats["k2_32"] += int(np.count_nonzero((a["kind"] == 2) & (a["worker"] >= 32)))
            stats["blocked"] += sum(r[0] == "blocked" for r in tr["rejected"])
            stats["time"] += sum(r[0] == "time" for r in tr["rejected"])
            stats["other_variant"] += sum(v != 0 for _, _, v, _ in tr["variant_takes"])
            n_asg = int(np.count_nonzero(a["kind"] != 1))
            stats["ticks"] += 1
            stats["left"] += int(inp.ready.sum()) > n_asg
            stats["empty"] += n_asg == 0
    for k in ("resv32", "resv512", "mu32", "gb_tile1", "k1_32", "k2_32", "blocked", "time", "other_variant"):
        assert stats[k] > 0, (k, stats)
    assert 2 * stats["left"] >= stats["ticks"] and 10 * stats["empty"] <= stats["ticks"], stats


# --- mutants of the specification -------------------------------------------------------------------------------------
def _reserve_ascending(self, c, n_all, remaining):
    """_Tick.reserve with the workers walked from the LOWEST index up."""
    if c in self.noresv:
        return
    cap = [w for w in range(self.W) if self.capable(w, c)]
    limit = sum(max(1, sum(min(self.fit_start(w, c, v), 1024) for v in range(len(self.am[c])))) for w in cap)
    got = 0
    if n_all <= limit:
        for w in cap:
            if got >= remaining:
                break
            if self.excluded[w] or self.touched[w] or any(self.fit_start(w, c, v) > 0 for v in range(len(self.am[c]))):
                continue
            self.excluded[w] = True
            got += 1
    if got < remaining:
        self.noresv.add(c)


def _variant_cost(t, w, c, v):
    fr = t.fr[w]
    if t.alls[c][v]:
        return np.float32(np.inf)
    dom = np.float32(0)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for r, a in t.am[c][v].items():
            if fr[r] != G.AMOUNT_MAX:
                x = np.float32(float(a)) * (np.float32(1.0) / np.float32(float(fr[r])))
                dom = x if x > dom else dom
    return dom


def _mutate(mp, name):
    T = G._Tick
    if name == "reservations ascending":
        mp.setattr(T, "reserve", _reserve_ascending)
    elif name == "reservations off":
        mp.setattr(T, "reserve", lambda self, c, n_all, remaining: None)
    elif name == "min-utilisation checked once":
        mp.setattr(G, "MU_MAX_PASSES", 2)
    elif name == "variant ties to the higher index":
        orig = T.next_variant

        def next_variant(self, w, c, tried):
            v = orig(self, w, c, tried)
            cost = _variant_cost(self, w, c, v)
            ties = [u for u in range(len(self.am[c])) if not (tried >> u) & 1 and _variant_cost(self, w, c, u) == cost]
            return max(ties) if ties else v
        mp.setattr(T, "next_variant", next_variant)
    elif name == "variant cost from the tick-start free vector":
        orig = T.next_variant

        def next_variant(self, w, c, tried):
            now, self.fr[w] = self.fr[w], self.fr0[w]
            try:
                return orig(self, w, c, tried)
            finally:
                self.fr[w] = now
        mp.setattr(T, "next_variant", next_variant)
    elif name == "stale frontier after a hand-back":
        orig_pack, orig_fit = G._pack_level, T.fit

        def pack(t, groups, phi):
            taken = orig_pack(t, groups, phi)
            t.stale = {(w, c) for c in range(len(t.am)) for w in range(t.W)
                       if all(orig_fit(t, w, c, v, 1) == 0 for v in range(len(t.am[c])))}
            return taken

        def fit(self, w, c, v, cap):
            return 0 if (w, c) in getattr(self, "stale", ()) else orig_fit(self, w, c, v, cap)
        mp.setattr(G, "_pack_level", pack)
        mp.setattr(T, "fit", fit)
    elif name == "pack quota rounded down":
        mp.setattr(G, "_pack_quota", lambda n, cn, T_, phi: int(math.floor(float(n * cn // T_) * phi)))
    elif name == "class weights ignored":
        orig = G.class_order

        def class_order(wl, free, total):
            plain = [[{k: x for k, x in d.items() if k != "weight"} for d in vs] for vs in wl.classes]
            return orig(dataclasses.replace(wl, classes=plain), free, total)
        mp.setattr(G, "class_order", class_order)
    elif name in ("time limit compared with <", "blocked mask on variant 0 only"):
        strict = name.startswith("time")

        def admissible(self, w, c, v):
            if self.excluded is not None and self.excluded[w]:
                return False
            if self.wl.blocked is not None and self.wl.blocked[w, c, v] and (strict or v == 0):
                return False
            rt = self.rem_ms[w]
            return rt == G.TIME_INF or (self.min_ms[c][v] < rt if strict else self.min_ms[c][v] <= rt)
        mp.setattr(T, "admissible", admissible)
    elif name == "prefill ignores a held prefill of the class":
        mp.setattr(G, "_holds_prefill", lambda *args: False)
    elif name == "redirects emitted as kind 0":
        orig = G._with_prefill

        def with_prefill(*args):
            out = orig(*args)
            out["kind"][out["kind"] == 2] = 0
            return out
        mp.setattr(G, "_with_prefill", with_prefill)
    else:
        raise KeyError(name)


MUTANTS = ("reservations ascending", "reservations off", "min-utilisation checked once", "variant ties to the higher index",
           "variant cost from the tick-start free vector", "stale frontier after a hand-back", "pack quota rounded down",
           "class weights ignored", "time limit compared with <", "blocked mask on variant 0 only",
           "prefill ignores a held prefill of the class", "redirects emitted as kind 0")


class _Caught(Exception):
    pass


@pytest.mark.parametrize("name", MUTANTS)
def test_mutant_changes_some_tick(name, monkeypatch):
    """The first (seed, tick) of the seed set (pools of at most 256 workers) whose records or free vectors the mutant
    changes; the drain stops there, because the events that follow depend on the records."""
    base = {seed: _drain(seed) for seed in MUTANT_SEEDS}
    _mutate(monkeypatch, name)
    for seed in MUTANT_SEEDS:
        want = base[seed]

        def check(tick, inp, a, fa, pf):
            _, a0, fa0, _ = want[tick]
            if not (np.array_equal(a, a0) and np.array_equal(fa, fa0)):
                raise _Caught(f"seed {seed} tick {tick}")
        try:
            D.Drain(seed).run(check)
        except _Caught as e:
            print(f"mutant '{name}' caught at {e}")
            return
    pytest.fail(f"mutant '{name}' changes no tick of seeds {MUTANT_SEEDS}")


# --- directed cases of what the drains found ------------------------------------------------------------------------
def handed_back_worker_case() -> Workload:
    """Worker 1 is partly used (4 of 10 cpus free).  Level 1 holds one 1-cpu task (class 0) and two 8-cpu tasks
    (class 1): 17 cpus of demand on 14, so the level is packed.  Both workers take the 1-cpu task in the pack; worker 0
    keeps it and worker 1 hands it back, so worker 1 receives no assignment.  Class 1 is left with a task it cannot place:
    it reserves worker 1 (big enough by its totals, nothing of the class fits now), and the 1-cpu tasks of level 0 must not
    go there."""
    classes = [[{"amounts": {0: 1 * FR}}], [{"amounts": {0: 8 * FR}}]]
    total = np.array([[10 * FR], [10 * FR]], dtype=np.uint64)
    free = np.array([[10 * FR], [4 * FR]], dtype=np.uint64)
    return Workload(1, classes, total, free, np.array([0, 1, 1, 0, 0, 0], dtype=np.uint32),
                    np.array([1, 1, 1, 0, 0, 0], dtype=np.int32))


def test_pack_take_handed_back_in_full_leaves_the_worker_reservable():
    wl = handed_back_worker_case()
    tr = {}
    a, fa = G.model_tick(wl, np.ones(wl.n_tasks, dtype=bool), wl.worker_free, trace=tr)
    assert tr["give_back"] == [(1, 0, 0, 1)] and tr["reserved"] == [(0, 1, 1)]
    assert a.tolist() == [(1, 0, 0, 0), (0, 0, 0, 0), (3, 0, 0, 0)]
    assert fa[:, 0].tolist() == [0, 4 * FR]


def test_host_keeps_unlimited_amounts_unlimited():
    """A worker with an unlimited resource (HQS_AMOUNT_MAX, which a tick never takes from) keeps it unlimited when its
    tasks finish or a prefilled task starts; a limited resource of the same worker is returned and taken as usual."""
    from hyperqueue_b200 import GpuScheduler
    s = object.__new__(GpuScheduler)
    s.free = np.array([[G.AMOUNT_MAX, 2 * FR]], dtype=np.uint64)
    s.total = s.free.copy()
    s._amount_tab = np.zeros((1, 8, 2), dtype=np.uint64)
    s._amount_tab[0, 0] = [5 * FR, 1 * FR]
    s._all_tab = np.zeros((1, 8, 2), dtype=bool)
    s._task_worker = np.array([0, -1], dtype=np.int64)
    s._task_class = np.zeros(2, dtype=np.uint32)
    s._task_variant = np.zeros(2, dtype=np.uint8)
    s.free[0, 1] = 1 * FR                                 # task 0 runs: 1 of 2 limited units used
    s.tasks_finished(np.array([0], dtype=np.uint32))
    assert s.free.tolist() == [[G.AMOUNT_MAX, 2 * FR]]
    s._take_resources(0, 0, 0)
    assert s.free.tolist() == [[G.AMOUNT_MAX, 1 * FR]]
