"""hqs_handles_compact in the sequential model (tests/compact_model.py): over seeded random sequences of pushes, graph
submits, finishes, removes, cancels and compactions, a model that compacts must equal a model that never does, through the
bijection of their handles, after every step: every key bit for bit (the retired handles are not VALID on the reference),
the priorities, the consumer lists' waiting edges, the dependency counts of the waiting tasks, every returned list, and the
level table.  New tasks take the next free handle on each side.  Then the mutants the comparison must catch, the
rejections and directed cases."""
import numpy as np
import pytest

from compact_model import CompactModel
from level_model import KEY_VALID, Rejected


def _prio(user, job=0):
    return (((int(user) & 0xFFFFFFFF) ^ 0x80000000) << 32) | int(job)


class Pair:
    """c compacts, r never does; r2c maps r's handles to c's."""

    def __init__(self, mutant=None, q=3):
        self.c, self.r = CompactModel(mutant), CompactModel()
        for m in (self.c, self.r):
            m.classes_set(q)
        self.r2c = {}
        self.nc = self.nr = 0

    def new(self, k):
        hr = list(range(self.nr, self.nr + k))
        self.r2c.update(zip(hr, range(self.nc, self.nc + k)))
        self.nr += k
        self.nc += k
        return hr

    def cmap(self, hr):
        return [self.r2c[h] for h in hr if h in self.r2c]

    def rmap(self, hc):
        c2r = {v: k for k, v in self.r2c.items()}
        return [c2r[h] for h in hc]

    def waiting_edges(self, m, to_r):
        out = set()
        for prod, edges in m.lists.items():
            for cn, g in edges:
                if m._edge_waits(cn, g):
                    out.add((to_r(prod), to_r(cn), g))
        return out

    def check(self):
        c, r = self.c, self.r
        kc, kr = c.keys(), r.keys()
        c2r = {v: k for k, v in self.r2c.items()}
        for hr in range(r.n_handles):
            hc = self.r2c.get(hr)
            if hc is None or hc >= c.n_handles:
                assert not kr[hr] & KEY_VALID, hr
                continue
            assert kc[hc] == kr[hr], (hr, hc, hex(kc[hc]), hex(kr[hr]))
            assert c.prio[hc] == r.prio[hr]
            if r.waiting(hr):
                assert c.gdeps[hc] == r.gdeps[hr] and c.gen.get(hc, 0) == r.gen.get(hr, 0)
        assert all(h in c2r for h in range(c.n_handles) if kc[h])
        to_r = lambda h: c2r.get(h, -1)
        assert self.waiting_edges(c, to_r) == self.waiting_edges(r, lambda h: h)
        assert c.levels == r.levels and c.table == r.table and c.coarse == r.coarse
        assert c.debug()[0] >= len(self.waiting_edges(c, to_r)) and c.debug()[3] == r.debug()[3]

    # the calls, on both models ---------------------------------------------------------------------------------------
    def push(self, hr, cls, prio):
        self.r.push(hr, cls, prio)
        self.c.push(self.cmap(hr), cls, prio)

    def graph_push(self, hr, cls, prio, deps):
        off = np.cumsum([0] + [len(d) for d in deps])
        dc = [self.cmap(d) for d in deps]
        offc = np.cumsum([0] + [len(d) for d in dc])
        a = self.r.graph_push(hr, cls, prio, off, [x for d in deps for x in d])
        assert self.c.graph_push(self.cmap(hr), cls, prio, offc, [x for d in dc for x in d]) == a

    def finished(self, hr):
        assert self.rmap(self.c.graph_finished(self.cmap(hr))) == self.r.graph_finished(hr)

    def cancel(self, hr):
        assert self.rmap(self.c.graph_cancel(self.cmap(hr))) == self.r.graph_cancel(hr)

    def remove(self, hr):
        self.r.remove(hr)
        self.c.remove(self.cmap(hr))

    def compact(self, keep_r=()):
        kr = self.r.keys()
        want = sorted(self.r2c[h] for h in set(np.nonzero(kr & KEY_VALID)[0].tolist()) | set(keep_r))
        old = self.c.compact(self.cmap(sorted(keep_r)))
        assert old == want
        new_of = {o: i for i, o in enumerate(old)}
        self.r2c = {h: new_of[c] for h, c in self.r2c.items() if c in new_of}
        self.nc = len(old)


def _run(seed, mutant=None, steps=150):
    rng = np.random.default_rng(seed)
    p = Pair(mutant)
    kept = set()                                        # handles the "host" still tracks: named in every keep
    for step in range(steps):
        op = int(rng.integers(0, 9))
        if op <= 2:
            k = int(rng.integers(1, 12))
            hr = p.new(k)
            deps = [sorted(set(rng.integers(max(0, h - 40), h, int(rng.integers(0, 4))).tolist())) if h else [] for h in hr]
            p.graph_push(hr, rng.integers(0, 3, k), [_prio(u, j) for u, j in zip(rng.integers(0, 3, k), rng.integers(0, 20, k))],
                         deps)
        elif op == 3:
            k = int(rng.integers(1, 8))
            p.push(p.new(k), rng.integers(0, 3, k), [_prio(u, 0) for u in rng.integers(0, 3, k)])
        elif op == 4 and p.nr:
            p.finished(rng.integers(0, p.nr, int(rng.integers(1, 6))).tolist())
        elif op == 5 and p.nr:
            p.cancel(rng.integers(0, p.nr, int(rng.integers(1, 3))).tolist())
        elif op == 6 and p.nr:
            h = int(rng.integers(0, p.nr))
            p.remove([h])
            if rng.integers(0, 2) and h in p.r2c:
                kept.add(h)                             # e.g. a prefilled task a worker started
        elif op == 7 and kept and rng.integers(0, 2):
            h = sorted(kept)[int(rng.integers(0, len(kept)))]
            if not p.r.flag(h) & KEY_VALID:            # a tracked handle is submitted again: a new incarnation
                kept.discard(h)
                live = [x for x in range(max(0, h - 30), h) if p.r.flag(x) & KEY_VALID and x in p.r2c]
                p.graph_push([h], [0], [_prio(1)], [live[-2:]])
        else:
            kept = {h for h in kept if h in p.r2c}
            p.compact(sorted(kept))
        p.check()
    return p


@pytest.mark.parametrize("seed", range(12))
def test_compacting_model_equals_the_model_that_never_compacts(seed):
    _run(seed)


@pytest.mark.parametrize("mutant", ["edge_remap", "incarnation"])
def test_the_comparison_catches_a_broken_compaction(mutant):
    caught = 0
    for seed in range(12):
        try:
            _run(seed, mutant)
        except (AssertionError, KeyError, IndexError):
            caught += 1
    assert caught > 0


def test_rejections_and_directed_cases():
    m = CompactModel()
    m.classes_set(1)
    m.graph_push([0, 1, 2], [0, 0, 0], [_prio(0)] * 3, [0, 0, 1, 2], [0, 1])
    m.remove([0])                                       # 1 keeps waiting on 0's edge: the list went with 0
    before = m.keys().copy()
    with pytest.raises(Rejected):
        m.compact([3])
    assert (m.keys() == before).all()
    assert m.compact([]) == [1, 2]                      # 0 is gone; 1 and 2 become 0 and 1
    assert m.debug()[0] == 1 and m.lists == {0: [(1, 1)]}
    assert m.graph_finished([0]) == [1]                 # the renumbered edge releases the renumbered consumer
    assert m.compact([]) == [1] and m.n_handles == 1
    m.graph_finished([0])
    assert m.compact([]) == [] and m.n_handles == 0
    assert m.graph_push([0], [0], [_prio(0)], [0, 0], []) == 1    # the next push takes handle 0
