"""The per-worker grouped layout on the CPU: the numpy model (tests/group_model.py, what tests/test_gpu_grouped.py holds the
device to) against a naive per-worker bucket loop, and GroupedTaskMapping's sliced message lists against the ones
WorkerTaskMapping builds record by record from the same flat stream."""
import numpy as np
import pytest

from group_model import group_model
from hyperqueue_b200 import GroupedTaskMapping, WorkerTaskMapping
from hyperqueue_b200._lib import assignment_dtype


def random_stream(rng, n, n_workers, kinds=(0, 1, 2)):
    """A flat stream in the tick's shape: assignments and redirects (kind 0 / 2) first, prefill records (kind 1) behind them."""
    a = np.zeros(n, dtype=assignment_dtype)
    a["task"] = rng.permutation(n).astype(np.uint32)
    a["worker"] = rng.integers(0, n_workers, n)
    a["variant"] = rng.integers(0, 8, n)
    kind = rng.choice(np.array(kinds), n)
    a["kind"] = np.concatenate([kind[kind != 1], kind[kind == 1]])
    return a


def naive(flat, n_workers):
    pre = [[] for _ in range(n_workers)]
    asg = [[] for _ in range(n_workers)]
    tail = []
    for i, (w, k) in enumerate(zip(flat["worker"].tolist(), flat["kind"].tolist())):
        (tail if k == 2 else pre[w] if k == 1 else asg[w]).append(i)
    order, off = [], [0]
    for w in range(n_workers):
        order += pre[w]; off.append(len(order))
        order += asg[w]; off.append(len(order))
    order += tail; off.append(len(order))
    return flat[np.array(order, dtype=np.int64)], np.array(off, dtype=np.uint32)


@pytest.mark.parametrize("n,n_workers,kinds", [(0, 5, (0, 1, 2)), (1, 1, (0,)), (5000, 1, (0, 1, 2)), (3000, 7, (2,)),
                                               (20000, 1024, (0, 1, 2)), (4097, 33, (0, 1)), (600, 512, (0,))])
def test_model_equals_a_bucket_loop(n, n_workers, kinds):
    rng = np.random.default_rng(n + n_workers)
    flat = random_stream(rng, n, n_workers, kinds)
    got, off = group_model(flat, n_workers)
    want, want_off = naive(flat, n_workers)
    assert np.array_equal(got, want) and np.array_equal(off, want_off)
    assert off.shape == (2 * n_workers + 2,) and off[0] == 0 and off[-1] == n and (np.diff(off.astype(np.int64)) >= 0).all()
    assert (got["kind"][off[-2]:] == 2).all() and (got["kind"][:off[-2]] != 2).all()


@pytest.mark.parametrize("seed,n,n_workers", [(0, 0, 3), (1, 400, 6), (2, 3000, 40), (3, 50, 1)])
def test_grouped_mapping_builds_the_same_messages(seed, n, n_workers):
    rng = np.random.default_rng(seed)
    flat = random_stream(rng, n, n_workers)
    ids = np.sort(rng.choice(10 * n_workers, n_workers, replace=False)).astype(np.uint32) + 50
    n_red = int((flat["kind"] == 2).sum())
    retract_from = rng.integers(0, n_workers, n_red) if n_red else None
    free_after = np.zeros((n_workers, 1), dtype=np.uint64)
    grouped, off = group_model(flat, n_workers)
    m = WorkerTaskMapping(flat, ids, free_after, retract_from)
    g = GroupedTaskMapping(grouped, off, ids, free_after, retract_from)
    assert g.messages() == m.messages()
    assert g.n_assigned() == m.n_assigned() and g.n_prefilled() == m.n_prefilled()
    # per_worker: the same lists once the redirected tasks (kind 2) are set aside; equal outright without them
    plain = WorkerTaskMapping(flat[flat["kind"] != 2], ids, free_after)
    gp, off_p = group_model(flat[flat["kind"] != 2], n_workers)
    assert GroupedTaskMapping(gp, off_p, ids, free_after).per_worker() == plain.per_worker()
    assert {w: sorted(v) for w, v in g.per_worker().items()} == {w: sorted(v) for w, v in m.per_worker().items()}


def test_cpp_shim_exports_the_grouped_tick():
    import subprocess
    import __graft_entry__ as ge
    ge.build()
    from hyperqueue_b200 import _lib
    shim = _lib.load_shim()
    assert hasattr(shim, "hqshim_selftest_grouped") and hasattr(shim, "hqshim_time_mapping")
    syms = subprocess.run(["nm", "-DC", _lib.SHIM_PATH], capture_output=True, text=True).stdout
    assert "tako_b200::GpuCore::run_scheduling_grouped" in syms
