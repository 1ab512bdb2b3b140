"""Which solve loop a tick runs, asserted through hqs_stats.solver_path, with one constructed workload per reachable
cell of {first-fit loop} x {RT 4, 8, 16 resource slots} x {u32, u64 amounts}, plus the class table in global memory,
packing on and off and the minimum-utilisation restart.  Every case is also compared bit for bit with the sequential
specification and goes through the feasibility judge, so a change in dispatch cannot move a case off its loop unnoticed.

Loops (hqs_tick.cuh): the wide loop (plain tick, every worker of a pool of <= 512 a lane, free vectors of at most 16
32-bit words: not RT 16 on u64), the one-warp lean loop (plain tick on a larger pool), the lean loop with reservation
bookkeeping (plain tick with a partly occupied worker) and the general loop (several variants, `All`, blocked masks,
time limits, minimum utilisation, packed levels)."""
import numpy as np
import pytest

import greedy_model as G
import parity as P
from hyperqueue_b200 import _lib as L

pytestmark = pytest.mark.gpu
FR = P.FR
LOOPS = {"wide": L.HQS_PATH_WIDE, "lean": L.HQS_PATH_LEAN, "lean_extras": L.HQS_PATH_LEAN_EXTRAS, "general": L.HQS_PATH_GENERAL}
LOOP_MASK = L.HQS_PATH_WIDE | L.HQS_PATH_LEAN | L.HQS_PATH_LEAN_EXTRAS | L.HQS_PATH_GENERAL
R_OF_RT = {4: 3, 8: 6, 16: 12}
WIDE_POOL, LEAN_POOL = 64, 600           # <= 512 workers: the wide loop can run; more: one warp walks the worker tiles


def _workload(R, W, variants=1, partial=False, n=20_000, q=6, seed=0):
    """q distinct classes over R resources, whole-unit amounts (narrow-capable), capacity well above demand."""
    rng = np.random.default_rng(seed)
    classes = []
    for c in range(q):
        vs = []
        for v in range(variants):
            a = {(c + v) % R: (c + 1) * FR}
            a[(c + 2 * v + 1) % R] = a.get((c + 2 * v + 1) % R, 0) + (v + 1) * FR
            vs.append({"amounts": a})
        classes.append(vs)
    total = np.full((W, R), 2_000 * FR, dtype=np.uint64)
    free = total.copy()
    if partial:
        free[::5, 0] -= np.uint64(3 * FR)                 # partly occupied workers: reservations are possible
    return P.Workload(R, classes, total, free, rng.integers(0, q, n).astype(np.uint32), rng.integers(0, 4, n).astype(np.int32))


def _loop_case(loop, rt):
    R = R_OF_RT[rt]
    if loop == "wide":
        return _workload(R, WIDE_POOL)
    if loop == "lean":
        return _workload(R, LEAN_POOL)
    if loop == "lean_extras":
        return _workload(R, WIDE_POOL, partial=True)
    return _workload(R, WIDE_POOL, variants=2)


def reachable_cells():
    """(loop, RT, width) cells the dispatch can reach.  The wide loop keeps a free vector in registers: at most 16 words."""
    cells = []
    for loop in LOOPS:
        for rt in (4, 8, 16):
            for width in ("u32", "u64"):
                words = rt * (1 if width == "u32" else 2)
                if loop == "wide" and words > 16:
                    continue
                cells.append((loop, rt, width))
    return cells


EXTRA_CELLS = ("classes_global", "pack_on", "pack_off", "mu_restart")

# every reachable cell has a case: (workload builder, flags, min_utilization or None, bits that must be set,
# bits that must be clear, the exact loop bits)
CASES = {}
for _loop, _rt, _width in reachable_cells():
    CASES[(_loop, _rt, _width)] = (lambda lp=_loop, rt=_rt: _loop_case(lp, rt),
                                   L.HQS_CREATE_WIDE_AMOUNTS if _width == "u64" else 0, None, 0, L.HQS_PATH_PACKED,
                                   LOOPS[_loop])


def _mu_workload():
    return _workload(3, 12, n=400, q=3, seed=5)


_MU = np.zeros(12, dtype=np.float32)
_MU[[0, 3]] = [1.0, 0.97]
CASES["classes_global"] = (lambda: P.Workload(3, [[{"amounts": {c % 3: (c // 3 + 1) * FR}}] for c in range(1500)],
                                              np.full((64, 3), 500_000 * FR, dtype=np.uint64), np.full((64, 3), 500_000 * FR, dtype=np.uint64),
                                              np.random.default_rng(3).integers(0, 1500, 40_000).astype(np.uint32),
                                              np.random.default_rng(4).integers(0, 2, 40_000).astype(np.int32)),
                           0, None, L.HQS_PATH_CLASSES_GLOBAL, 0, L.HQS_PATH_LEAN)
CASES["pack_on"] = (lambda: P.make_independent(80_000, 300, 16, seed=14, free_scale=1), 0, None,
                    L.HQS_PATH_PACKED | L.HQS_PATH_GENERAL, L.HQS_PATH_CLASSES_GLOBAL, None)
CASES["pack_off"] = (lambda: P.make_independent(80_000, 300, 16, seed=14, free_scale=1), L.HQS_CREATE_NO_PACK, None,
                     0, L.HQS_PATH_PACKED, L.HQS_PATH_WIDE)
CASES["mu_restart"] = (_mu_workload, 0, _MU, L.HQS_PATH_MU_RESTART, 0, L.HQS_PATH_GENERAL)


def _ids():
    return ["-".join(str(x) for x in k) if isinstance(k, tuple) else k for k in CASES]


@pytest.mark.parametrize("key", list(CASES), ids=_ids())
def test_solver_path_cell(key):
    build, flags, mu, must, must_not, loops = CASES[key]
    wl = build()
    s = P.gpu_scheduler(wl, flags=flags)
    if mu is not None:
        s.min_utilization = mu.copy()
    fb = s.free.copy()
    m = s.run_scheduling()
    st = s.stats()
    s.close()
    path = st["solver_path"]
    print(f"{key}: solver_path {path:#04x} narrow {st['narrow_amounts']} assigned {m.n_assigned()}")
    exp, exp_free = G.model_tick(wl, np.ones(wl.n_tasks, dtype=bool), fb, pack=not (flags & L.HQS_CREATE_NO_PACK),
                                 min_utilization=mu)
    assert np.array_equal(m.assignments, exp) and np.array_equal(m.free_after, exp_free)
    assert P.judge_tick(wl, fb, m.assignments).ok
    assert m.n_assigned() > 0
    if isinstance(key, tuple):
        assert st["narrow_amounts"] == (1 if key[2] == "u32" else 0)
    assert path & must == must, hex(path)
    assert path & must_not == 0, hex(path)
    if loops is not None:
        assert path & LOOP_MASK == loops, hex(path)
