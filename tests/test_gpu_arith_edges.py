"""Ticks at the edges of the solver's fit-count arithmetic, through the C ABI, on both amount widths (gcd-scaled 32-bit
and plain 64-bit): free amounts at the top of the u64 range, binding quotients above 2^20 (the u64 path's exact-division
fallback), the narrow/wide boundary of the gcd scaling, and HQS_AMOUNT_MAX in a tick.  Every tick is compared bit for
bit with the sequential specification (assignments and free vectors) and goes through the feasibility judge."""
import numpy as np
import pytest

import greedy_model as G
import parity as P
from hyperqueue_b200 import _lib as L

pytestmark = pytest.mark.gpu
FR = P.FR
MAX = (1 << 64) - 1
LOOPS = L.HQS_PATH_WIDE | L.HQS_PATH_LEAN | L.HQS_PATH_LEAN_EXTRAS | L.HQS_PATH_GENERAL


def _tick_both_widths(wl, narrow=None, loop=None):
    """flags 0 (narrow when the tick allows it) and flags 2 (HQS_CREATE_WIDE_AMOUNTS) against the specification.
    narrow: expected hqs_stats.narrow_amounts of the flags-0 tick; loop: the expected first-fit loop bits."""
    ready = np.ones(wl.n_tasks, dtype=bool)
    exp, exp_free = G.model_tick(wl, ready, wl.worker_free)
    out = {}
    for flags in (0, L.HQS_CREATE_WIDE_AMOUNTS):
        s = P.gpu_scheduler(wl, flags=flags)
        fb = s.free.copy()
        m = s.run_scheduling()
        st = s.stats()
        s.close()
        assert np.array_equal(m.assignments, exp), (flags, m.n_assigned(), exp.shape[0])
        assert np.array_equal(m.free_after, exp_free), flags
        res = P.judge_tick(wl, fb, m.assignments, ready)
        assert res.ok, res
        assert st["narrow_amounts"] == (0 if flags else (st["narrow_amounts"] if narrow is None else int(narrow)))
        if loop is not None:
            assert st["solver_path"] & LOOPS == loop, (flags, hex(st["solver_path"]))
        out[flags] = (m, st)
    return out


@pytest.mark.parametrize("R", [2, 6])
def test_free_amounts_at_the_top_of_the_u64_range(R):
    """Workers whose free amount of a resource lies within d of 2^64 (free + d > 2^64) for requests of d >= 2^45: the fp32
    quotient estimate is 2^64 / d there.  free = 2^64 - 2 and d = 2^45 fit 524287 tasks, not 524290."""
    big = R - 1
    classes = [[{"amounts": {0: 1 * FR, big: 1 << 45}}],
               [{"amounts": {0: 1 * FR, big: 3 << 45}}],
               [{"amounts": {0: 1 * FR}}],
               [{"amounts": {big: (1 << 45) + 1}}]]
    W = 4
    total = np.full((W, R), 4_000_000 * FR, dtype=np.uint64)
    total[:, big] = [MAX - 1, (1 << 64) - (1 << 45) + 5, (1 << 64) - (3 << 45) + 1, 1 << 50]
    n = [700_000, 300_000, 5_000, 2_000]
    task_class = np.repeat(np.arange(4, dtype=np.uint32), n)
    prio = np.repeat(np.array([3, 2, 1, 0], dtype=np.int32), n)
    wl = P.Workload(R, classes, total, total.copy(), task_class, prio)
    out = _tick_both_widths(wl, narrow=False, loop=L.HQS_PATH_WIDE)
    m = out[0][0]
    a = m.assignments
    first = a[(wl.task_class[a["task"]] == 0) & (a["worker"] == 0)]
    assert first.shape[0] == ((1 << 64) - 2) // (1 << 45) == 524287


def _big_quotient_workload(shape, W):
    """1.5 M tasks of one class at one level; three workers that fit about 1.2 M, 0.2 M and 0.5 M of them (shape 1: one
    resource; shape 2: two resources that both bind above 2^20, at different values), and W - 3 workers with half a cpu."""
    if shape == 1:
        R, classes = 1, [[{"amounts": {0: 1 * FR}}]]
        head = np.array([[1_200_000 * FR + 3], [200_000 * FR + 7], [500_000 * FR + 1]], dtype=np.uint64)
    else:
        R, classes = 2, [[{"amounts": {0: 1 * FR, 1: 2 * FR}}]]
        head = np.array([[1_300_000 * FR + 11, 2 * 1_250_000 * FR + 5],
                         [300_000 * FR, 2 * 200_000 * FR + 3],
                         [500_000 * FR + 9, 2 * 2_000_000 * FR]], dtype=np.uint64)
    tail = np.full((W - 3, R), FR // 2, dtype=np.uint64)
    total = np.concatenate([head, tail])
    n = 1_500_000
    return P.Workload(R, classes, total, total.copy(), np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.int32))


@pytest.mark.parametrize("shape", [1, 2])
@pytest.mark.parametrize("W,loop", [(3, L.HQS_PATH_WIDE), (600, L.HQS_PATH_LEAN)], ids=["wide-loop", "one-warp-loop"])
def test_binding_quotients_above_2_20(shape, W, loop):
    """A worker takes over 2^20 tasks of one group: the u64 fit count leaves its fp32 estimate for an exact division."""
    wl = _big_quotient_workload(shape, W)
    out = _tick_both_widths(wl, narrow=True, loop=loop)
    a = out[0][0].assignments
    per_worker = np.bincount(a["worker"], minlength=W)
    assert per_worker[0] > (1 << 20) and a.shape[0] == wl.n_tasks


def _boundary_workload(extra):
    rng = np.random.default_rng(21)
    classes = [[{"amounts": {0: 1 * FR, 1: 4 * FR}}], [{"amounts": {0: 2 * FR}}], [{"amounts": {1: 8 * FR}}]]
    W = 24
    total = np.stack([rng.integers(4, 64, W).astype(np.uint64) * np.uint64(FR) + rng.integers(1, FR, W).astype(np.uint64),
                      rng.integers(4, 200, W).astype(np.uint64) * np.uint64(4 * FR) + rng.integers(1, 4 * FR, W).astype(np.uint64)],
                     axis=1)
    total[0, 1] = 4 * FR * ((1 << 31) - 1) + extra           # the gcd of resource 1 is 4 FR: its narrow limit
    n = 20_000
    return P.Workload(2, classes, total, total.copy(), rng.integers(0, 3, n).astype(np.uint32), rng.integers(0, 3, n).astype(np.int32))


def test_narrow_wide_boundary_of_the_gcd_scaling():
    """A free amount of exactly gscale * (2^31 - 1) is still solved narrow; one fraction more is solved on 64-bit amounts.
    The two ticks place the same tasks the same way (the extra fraction is a remainder nobody can use)."""
    at = _tick_both_widths(_boundary_workload(0), narrow=True)
    over = _tick_both_widths(_boundary_workload(1), narrow=False)
    m0, m1 = at[0][0], over[0][0]
    assert m0.n_assigned() > 1000
    assert np.array_equal(m0.assignments, m1.assignments)
    diff = m1.free_after.astype(object) - m0.free_after.astype(object)
    assert diff[0, 1] == 1 and np.count_nonzero(diff) == 1


def test_amount_max_in_a_tick():
    """HQS_AMOUNT_MAX (unknown / unbounded) free amounts on some resources of some workers, in a real tick: never the
    binding resource, never consumed."""
    rng = np.random.default_rng(22)
    classes = [[{"amounts": {0: 1 * FR, 1: 3 * FR}}], [{"amounts": {1: 2 * FR, 2: 5 * FR}}], [{"amounts": {0: 2 * FR, 2: 1 * FR}}],
               [{"amounts": {2: 7 * FR}}]]
    W = 16
    total = rng.integers(8, 64, size=(W, 3)).astype(np.uint64) * np.uint64(FR)
    total[::3, 1] = MAX
    total[1::4, 2] = MAX
    total[5, :] = MAX                                          # unbounded everywhere
    n = 20_000
    wl = P.Workload(3, classes, total, total.copy(), rng.integers(0, 4, n).astype(np.uint32), rng.integers(0, 3, n).astype(np.int32))
    out = _tick_both_widths(wl, narrow=True)
    m = out[0][0]
    assert m.n_assigned() > 1000
    assert (m.free_after[total == MAX] == MAX).all()
