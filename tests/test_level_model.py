"""CPU checks of tests/level_model.py, the model of the ready set's key table and priority-level policy that
tests/test_gpu_ready_set.py compares the device with: the bucket formula at its edges, the lookup against a scalar
restatement, and the policy's invariants over random call sequences."""
import numpy as np
import pytest

import level_model as LM

U64_MAX = (1 << 64) - 1


def _scalar_find(table, p, coarse):
    """find_level of hqs_ready_set.cuh, one value at a time."""
    lo, hi = 0, len(table)
    while lo < hi:
        mid = (lo + hi) // 2
        if table[mid] <= p:
            hi = mid
        else:
            lo = mid + 1
    if coarse:
        return min(lo, len(table) - 1)
    return lo if lo < len(table) and table[lo] == p else -1


@pytest.mark.parametrize("m", [1, 2, 3, 8, 81, 4096])
def test_bucket_bounds_at_one_and_two_levels_per_bucket(m):
    # L = M + 1: the first M - 1 levels keep a bucket each, the last bucket takes the two lowest
    levels = [U64_MAX] + list(range(10 * m, 9 * m + 1, -1))[: m - 1] + [0]
    assert len(levels) == m + 1 and levels == sorted(levels, reverse=True)
    b = LM.bucket_bounds(levels, m)
    assert len(b) == m and b[-1] == 0 and b[:-1] == levels[: m - 1]
    lv = LM.find_levels(np.array(b, dtype=np.uint64), np.array(levels, dtype=np.uint64), True)
    assert lv.tolist() == list(range(m - 1)) + [m - 1, m - 1]
    # L = 2M: bucket b holds levels 2b and 2b + 1, its bound is the lower one
    levels = [U64_MAX] + [U64_MAX - 1 - 3 * i for i in range(2 * m - 2)] + [0]
    b = LM.bucket_bounds(levels, m)
    assert b[:-1] == levels[1:-1:2][: m - 1] and b[-1] == 0
    lv = LM.find_levels(np.array(b, dtype=np.uint64), np.array(levels, dtype=np.uint64), True)
    assert lv.tolist() == [i // 2 for i in range(2 * m)]
    # the extremes: 2^64 - 1 is in the first bucket, 0 in the last, priorities between the registered ones go to the
    # bucket whose bound is the first one at or below them
    probe = np.array([U64_MAX, 0, U64_MAX - 2], dtype=np.uint64)
    got = LM.find_levels(np.array(b, dtype=np.uint64), probe, True).tolist()
    assert got == [_scalar_find(b, int(p), True) for p in probe.tolist()]
    assert got[0] == 0 and got[1] == m - 1


def test_find_levels_equals_the_scalar_search():
    rng = np.random.default_rng(0)
    for n in (1, 2, 7, 64, 1000):
        table = sorted(set(int(x) * 2 for x in rng.integers(0, 1 << 63, n, dtype=np.int64)), reverse=True)
        probe = [int(x) for x in rng.choice(np.array(table, dtype=np.uint64), 50)] + \
                [int(x) * 2 + 1 for x in rng.integers(0, 1 << 62, 50)] + [0, U64_MAX]
        for coarse in (False, True):
            got = LM.find_levels(np.array(table, dtype=np.uint64), np.array(probe, dtype=np.uint64), coarse).tolist()
            assert got == [_scalar_find(table, p, coarse) for p in probe], (n, coarse)


def _check_invariants(m: LM.LevelModel, pushed_fresh: bool):
    valid = m.has(LM.KEY_VALID)
    lvl, prio = m.lvl[valid].astype(np.int64), m.prio[valid]
    assert (lvl < max(m.n_levels, 1)).all()
    if not m.coarse:
        rank = {p: i for i, p in enumerate(m.levels)}
        assert all(int(p) in rank for p in prio.tolist()), "an exact table misses a live priority"
        assert lvl.tolist() == [rank[int(p)] for p in prio.tolist()]
    # the level never increases as the priority increases
    order = np.argsort(prio, kind="stable")
    assert (np.diff(lvl[order]) <= 0).all()
    if pushed_fresh and not m.declared:
        assert m.coarse == (m.live_priorities().size > LM.max_levels(m.Q)), (m.live_priorities().size, m.Q)


def _fake_tick(rng, m: LM.LevelModel):
    """Records of some tick: a few ready tasks are assigned (kind 0, or 2 if prefilled), a few others prefilled."""
    ready = np.nonzero(m.ready())[0]
    if ready.size == 0:
        return
    pick = rng.choice(ready, min(ready.size, int(rng.integers(1, 64))), replace=False)
    rec = np.zeros(pick.size, dtype=[("task", "<u4"), ("worker", "<u2"), ("variant", "u1"), ("kind", "u1")])
    rec["task"] = pick
    pf = m.has(LM.KEY_PF)[pick]
    rec["kind"] = np.where(pf, 2, np.where(rng.random(pick.size) < 0.3, 1, 0))
    m.apply_tick(rec)


def _run(seed, declared, check=True):
    """A random sequence on the model; returns how many calls took a coarse table back to exact levels."""
    rng = np.random.default_rng(seed)
    m = LM.LevelModel()
    m.classes_set(int(rng.choice([1, 2, 3, 100, 1000, 2048])))
    used: set = set()
    to_exact = 0
    for _ in range(40):
        op = LM.random_op(rng, m, used, declared)
        fresh = False
        if op[0] == "push":
            fresh = not set(int(p) for p in op[3].tolist()) <= set(m.levels)
            was = m.coarse
            m.push(op[1], op[2], op[3])
            to_exact += int(was and not m.coarse)
        elif op[0] == "remove":
            m.remove(op[1])
        elif op[0] == "tick":
            _fake_tick(rng, m)
        elif op[0] == "remove_done":
            m.remove(np.nonzero(m.has(LM.KEY_DONE))[0])
        elif op[0] == "rearm":
            m.rearm()
        elif op[0] == "dispose":
            m.prefill_dispose(op[1])
        elif op[0] == "classes":
            was = m.coarse
            m.classes_set(op[1])
            to_exact += int(was and not m.coarse)
        elif op[0] == "levels_add":
            m.levels_add(op[1])
        if check:
            _check_invariants(m, fresh)
    return to_exact


@pytest.mark.parametrize("seed", range(12))
def test_random_sequences_keep_the_invariants(seed):
    _run(1000 + seed, declared=seed % 4 == 3)


def test_random_sequences_alternate_between_exact_and_coarse():
    """The sequences must not only go coarse and stay there: pushes and class changes bring coarse tables back to exact
    levels."""
    assert sum(_run(seed, declared=False, check=False) for seed in range(20)) >= 20


def test_coarse_pushes_register_their_priorities():
    """The sequences of the ready-set tests: a coarse table is left as soon as the live priorities fit again."""
    m = LM.LevelModel()
    m.classes_set(2)
    m.push(np.arange(5000), np.zeros(5000), np.arange(5000, dtype=np.uint64) * 8 + 1000)
    assert m.coarsened == 1 and m.n_levels == 4096
    m.remove(np.arange(5000))
    top = np.arange(1500, dtype=np.uint64) + 10 ** 6
    m.push(np.arange(5000, 6500), np.ones(1500), top)
    assert m.coarsened == 0 and m.n_levels == 1500
    assert m.lvl[5000:].tolist() == list(range(1499, -1, -1))
    # a new class shrinks the budget; what is registered still fits
    m.classes_set(3)
    assert m.coarsened == 0 and m.n_levels == 1500
    _check_invariants(m, False)


def test_levels_live_and_retain():
    """Declared levels: live flags follow the VALID keys; a retain that drops a carried level or has another length is
    rejected with nothing changed; a valid one drops the dead levels, leaves coarse mode when the rest fits, re-levels."""
    m = LM.LevelModel()
    m.classes_set(4096)                                   # budget 2 levels
    m.levels_add([50, 40, 30, 20])
    assert m.coarsened == 1
    m.push([0, 1, 2], [0, 1, 2], [40, 20, 40])
    lv, live = m.levels_live()
    assert lv.tolist() == [50, 40, 30, 20] and live.tolist() == [0, 1, 0, 1]
    keys = m.keys().copy()
    for bad in ([1, 0, 1, 1], [0, 1, 0, 1, 1], [0, 1, 0]):
        with pytest.raises(LM.Rejected):
            m.levels_retain(bad)
        assert np.array_equal(m.keys(), keys) and m.levels == [50, 40, 30, 20]
    m.levels_retain([1, 1, 0, 1])                          # another rank still holds 50
    assert m.levels == [50, 40, 20] and m.coarsened == 1 and m.pruned_at == 3
    m.remove([0, 2])
    m.levels_retain(m.levels_live()[1])
    assert m.levels == [20] and m.coarsened == 0 and m.pruned_at == 1
    assert int(m.lvl[1]) == 0 and not m.need_pruning()    # declared: never prunes on its own


def test_random_declared_sequences_retain_levels():
    rng = np.random.default_rng(3)
    m = LM.LevelModel()
    m.classes_set(2)
    used: set = set()
    kinds = {}
    for _ in range(400):
        op = LM.random_op(rng, m, used, declared=True)
        kinds[op[0]] = kinds.get(op[0], 0) + 1
        try:
            if op[0] == "push":
                m.push(op[1], op[2], op[3])
            elif op[0] == "remove":
                m.remove(op[1])
            elif op[0] == "levels_add":
                m.levels_add(op[1])
            elif op[0] == "levels_retain":
                m.levels_retain(op[1])
            elif op[0] == "classes":
                m.classes_set(op[1])
        except LM.Rejected:
            continue
        # every carried priority stays registered
        assert set(int(p) for p in m.live_priorities().tolist()) <= set(m.levels)
    assert kinds.get("levels_retain", 0) > 5, kinds
