"""Parity tests proper: the CUDA path, called through the C ABI, against
  (1) the feasibility judge — every emitted assignment must pass the reference's own admission predicate
      and capacity rows, bit-exact (oracle/judge.py),
  (2) an exact replay of the free vectors (Worker::sanity_check),
  (3) the sequential specification of the device algorithm (tests/greedy_model.py) — bit-exact,
  (4) the oracle (restated reference tick): per-tick fill and drain makespan,
and, at BASELINE.json's full size (1M tasks x 256 workers x 4 resource kinds), size-independent
properties: every task assigned exactly once, output sorted by priority, idempotence of a second tick.
"""
import ctypes as C
import json
import os

import numpy as np
import pytest

import greedy_model as G
import parity as P
from oracle import judge as J

pytestmark = pytest.mark.gpu
FR = P.FR
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "oracle_drains.json")


def _tick_vs_model(wl, levels=None, stats=None):
    s = P.gpu_scheduler(wl)
    free_before = s.free.copy()
    m = s.run_scheduling()
    if stats is not None:
        stats.update(s.stats())
    ready = np.ones(wl.n_tasks, dtype=bool)
    exp, exp_free = G.model_tick(wl, ready, free_before, levels)
    res = P.judge_tick(wl, free_before, m.assignments, ready)
    assert res.ok, res
    assert np.array_equal(m.assignments, exp), (m.assignments[:10], exp[:10])
    assert np.array_equal(m.free_after, exp_free)
    s.close()
    return m


# ---------------------------------------------------------------------------------------------------
# single tick, bit-exact against the specification + judge
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,w,q,seed", [(1, 1, 1, 0), (37, 3, 2, 1), (1000, 8, 6, 2), (4097, 16, 12, 3),
                                        (50000, 64, 16, 4), (200001, 256, 16, 5)])
def test_tick_matches_specification(n, w, q, seed):
    _tick_vs_model(P.make_independent(n, w, q, seed))


@pytest.mark.parametrize("n,w,q,seed,scale", [(30000, 33, 8, 11, 1024), (120000, 300, 16, 12, 1024), (150000, 512, 16, 13, 1024),
                                              (80000, 300, 16, 14, 1), (90000, 512, 12, 15, 1), (40000, 513, 8, 16, 1024)])
def test_wide_first_fit_pool_shapes(n, w, q, seed, scale):
    """Plain ticks on pools of up to 512 workers run the wide first-fit (every worker a lane, one warp per 32 workers): ragged
    last warp (33, 300), all 16 warps (512), every task assignable (scale 1024) and saturated pools (scale 1: pack first, then
    dead classes are skipped); 513 workers fall back to the one-warp loop.  Bit-exact against the specification."""
    from hyperqueue_b200 import _lib as L
    st = {}
    _tick_vs_model(P.make_independent(n, w, q, seed, free_scale=scale), stats=st)
    path = st["solver_path"]
    if w <= 512:
        assert path & L.HQS_PATH_WIDE and not path & (L.HQS_PATH_LEAN | L.HQS_PATH_LEAN_EXTRAS), hex(path)
    else:
        assert path & L.HQS_PATH_LEAN and not path & L.HQS_PATH_WIDE, hex(path)
    if scale == 1:
        assert path & L.HQS_PATH_PACKED, hex(path)


def test_tick_variants_and_blocked():
    _tick_vs_model(P.make_independent(20000, 32, 12, seed=7, variants3=True, blocked_density=0.05))


def test_tick_capacity_exceeds_demand_m1():
    m = _tick_vs_model(P.make_independent(60000, 32, 16, seed=8, free_scale=1024))
    assert m.n_assigned() == 60000


def test_tick_time_limits_all_policy_and_max_sentinel():
    classes = [[{"amounts": {0: 2 * FR}, "min_time_s": 100.0}],        # needs 100 s
               [{"amounts": {1: 5000}, "all": (0,)}],                  # all cpus + 0.5 gpu
               [{"amounts": {0: 1 * FR, 2: 3 * FR}}],
               [{"amounts": {0: 3 * FR}}, {"amounts": {0: 1 * FR, 1: 1 * FR}}]]
    total = np.array([[8 * FR, 2 * FR, 10 * FR], [8 * FR, 0, P.J.AMOUNT_MAX], [4 * FR, 1 * FR, 6 * FR],
                      [16 * FR, 4 * FR, 0]], dtype=np.uint64)
    free = total.copy()
    free[2, 0] = 3 * FR                                              # a running task holds one cpu
    rng = np.random.default_rng(5)
    wl = P.Workload(3, classes, total, free, rng.integers(0, 4, 300).astype(np.uint32),
                    rng.integers(-3, 3, 300).astype(np.int32),
                    worker_remaining_s=np.array([np.inf, 50.0, 200.0, np.inf]))
    m = _tick_vs_model(wl)
    cls = wl.task_class[m.assignments["task"]]
    # class 0 (100 s) never lands on worker 1 (50 s left); `All` never on the partially used worker 2
    assert not ((cls == 0) & (m.assignments["worker"] == 1)).any()
    assert not ((cls == 1) & (m.assignments["worker"] == 2)).any()


def test_tick_empty_and_idempotent():
    wl = P.make_independent(5000, 8, 4, seed=9)
    s = P.gpu_scheduler(wl, add_tasks=False)
    assert s.run_scheduling().n_assigned() == 0                      # nothing ever pushed
    from hyperqueue_b200 import priority_from_user
    s.add_ready_tasks(np.arange(wl.n_tasks, dtype=np.uint32), wl.task_class, priority_from_user(wl.task_user_priority))
    first = s.run_scheduling()
    assert first.n_assigned() > 0
    # a second tick with no change emits nothing (test_scheduler_mapping.rs:38-44)
    assert s.run_scheduling().n_assigned() == 0
    # removing every remaining ready task empties the tick even after resources return
    s.tasks_finished(first.assignments["task"])
    left = np.setdiff1d(np.arange(wl.n_tasks, dtype=np.uint32), first.assignments["task"])
    s.remove_ready_tasks(left)
    assert s.run_scheduling().n_assigned() == 0
    s.close()


def test_tick_out_cap_overflow_is_an_error_without_partial_results():
    from hyperqueue_b200 import HqsError
    wl = P.make_independent(3000, 8, 4, seed=10)
    s = P.gpu_scheduler(wl)
    with pytest.raises(HqsError) as e:
        s.run_scheduling(out_cap=5)
    assert e.value.code == -5
    s.close()


def test_many_priority_levels_are_exact_up_to_the_group_limit():
    """Shape of test_many_cuts (test_scheduler_sn.rs:1129-1146): 300 x 8 cpus, 3200 levels x 2 classes = 6400 groups, inside
    HQS_MAX_GROUPS (8192): no coarsening (round 1 merged levels at 4096 groups)."""
    classes = [[{"amounts": {0: 1 * FR}}], [{"amounts": {0: 2 * FR}}]]
    total = np.full((300, 1), 8 * FR, dtype=np.uint64)
    cls = np.tile(np.array([0, 1], dtype=np.uint32), 3200)
    up = np.repeat(np.arange(3200, dtype=np.int32), 2)
    wl = P.Workload(1, classes, total, total.copy(), cls, up)
    s = P.gpu_scheduler(wl)
    m = s.run_scheduling()
    assert P.judge_tick(wl, wl.worker_free, m.assignments).ok
    c = np.bincount(wl.task_class[m.assignments["task"]], minlength=2)
    assert abs(int(c[0]) - int(c[1])) < 10 and abs(int(c[0]) - 800) < 10, c
    assert s.stats()["coarsened"] == 0
    exp, _ = G.model_tick(wl, np.ones(wl.n_tasks, dtype=bool), wl.worker_free)
    assert np.array_equal(m.assignments, exp)
    s.close()


# ---------------------------------------------------------------------------------------------------
# drain (mode M2): feasibility every tick, resources conserved, makespan
# ---------------------------------------------------------------------------------------------------
ALL_DRAINS = sorted(k for k in json.load(open(GOLDEN)).keys() if not k.startswith("big_") or os.environ.get("HQS_BIG_DRAINS"))


@pytest.mark.parametrize("key", ALL_DRAINS)
def test_drain_makespan_vs_oracle(key):
    """north_star: the zero-duration drain takes at most 2 % more ticks than the reference scheduler (finishing
    earlier is fine).  Six cases were used while designing the packing rules, eight (see make_oracle_drains.py)
    were generated afterwards as held-out checks."""
    golden = json.load(open(GOLDEN))[key]
    wl = (P.make_dag if "dag" in key.split("_")[:2] else P.make_independent)(*golden["args"], **golden.get("kwargs", {}))
    ticks, per_tick = P.gpu_drain(wl)
    assert sum(per_tick) == wl.n_tasks
    if key.startswith("w256_"):
        assert ticks == golden["max_ticks"]            # = the specification's makespan, recorded by the generator (minutes in Python)
    else:
        assert ticks == G.model_drain(wl)[0]
    assert ticks <= golden["max_ticks"], (ticks, golden)                       # the pinned value can only shrink
    assert ticks - golden["oracle_ticks"] <= 0.02 * golden["oracle_ticks"], (ticks, golden)


def test_drain_with_running_tasks_matches_specification():
    """Tasks run for 1-3 ticks, so workers are partly occupied (free != total) at every tick start — the situation in which
    reservations (solver.rs:133-151) exist.  Every tick of the CUDA path must equal the specification's tick on the same
    ready set and free vectors, and the makespan must be the recorded one (tests/golden/duration_drains.json)."""
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    import make_duration_drains as D
    g = json.load(open(os.path.join(os.path.dirname(GOLDEN), "duration_drains.json")))["dur_indep3_3000_8_6_53"]
    wl = P.make_independent(*g["args"], **g["kwargs"])
    dur = D.durations(wl.n_tasks, g["args"][-1])
    s = P.gpu_scheduler(wl)
    amounts, _, _, _ = wl.class_tables()
    ready = np.ones(wl.n_tasks, dtype=bool)
    levels = np.unique(wl.task_user_priority.astype(np.int64))[::-1]
    remaining, tick, finish_at = wl.n_tasks, 0, {}
    while remaining > 0 and tick < 10000:
        for (t, w, v) in finish_at.pop(tick, []):
            s.free[w] += amounts[wl.task_class[t], v]
        fb = s.free.copy()
        m = s.run_scheduling()
        a = m.assignments
        exp, exp_free = G.model_tick(wl, ready, fb, levels)
        assert np.array_equal(a, exp) and np.array_equal(m.free_after, exp_free), tick
        assert P.judge_tick(wl, fb, a, ready).ok
        ready[a["task"]] = False
        for t, w, v in zip(a["task"].tolist(), a["worker"].tolist(), a["variant"].tolist()):
            finish_at.setdefault(tick + int(dur[t]), []).append((t, w, v))
        remaining -= a.size
        tick += 1
    s.close()
    assert tick + max((k - tick for k in finish_at), default=0) == g["model_ticks"]


def test_dag_drain_readiness_propagation():
    wl = P.make_dag(20000, 16, 8, seed=6, window=512)
    ticks, per_tick = P.gpu_drain(wl)          # checks n_new_ready against a host replay every wave
    assert sum(per_tick) == wl.n_tasks and ticks > 10


# ---------------------------------------------------------------------------------------------------
# full size (BASELINE.json configs[1]): size-independent properties
# ---------------------------------------------------------------------------------------------------
def test_full_size_single_tick_properties():
    wl = P.make_independent(1_000_000, 256, 16, seed=0, free_scale=1024)
    s = P.gpu_scheduler(wl)
    free_before = s.free.copy()
    m = s.run_scheduling()
    a = m.assignments
    assert a.shape[0] == wl.n_tasks
    assert np.array_equal(np.sort(a["task"]), np.arange(wl.n_tasks, dtype=np.uint32))      # a permutation
    res = P.judge_tick(wl, free_before, a)
    assert res.ok, res
    amounts, allm, _, _ = wl.class_tables()
    exp = J.replay_free_after(amounts, allm, free_before, wl.worker_total, wl.task_class, a["task"], a["worker"], a["variant"])
    assert np.array_equal(exp, m.free_after)
    # emission order: priority descending, then ascending handle inside one (priority, class) group
    pr = wl.task_user_priority[a["task"]]
    assert (np.diff(pr) <= 0).all()
    same = (np.diff(pr) == 0) & (np.diff(wl.task_class[a["task"]].astype(np.int64)) == 0)
    assert (np.diff(a["task"].astype(np.int64))[same] > 0).all()
    assert s.run_scheduling().n_assigned() == 0
    s.close()


def test_full_size_drain_first_ticks_feasible():
    wl = P.make_independent(1_000_000, 256, 16, seed=1)
    s = P.gpu_scheduler(wl)
    assigned = 0
    for _ in range(5):
        free_before = s.free.copy()
        m = s.run_scheduling()
        assert m.n_assigned() > 1000
        assert P.judge_tick(wl, free_before, m.assignments).ok
        assert (wl.task_user_priority[m.assignments["task"]] >= 6).all() or m.n_assigned() > 0
        assigned += m.n_assigned()
        s.tasks_finished(m.assignments["task"])
        assert np.array_equal(s.free, wl.worker_free)
    s.close()
