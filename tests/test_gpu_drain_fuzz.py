"""Multi-tick drains (tests/drain_fuzz.py) on pools of 1 to 1024 workers with every tick feature mixed, run on two device
contexts in lockstep (32-bit gcd-scaled amounts where they fit, and always 64-bit) and compared bit for bit with the
specification every tick: the records with their kinds and order, free_after, the host's prefill and redirect
bookkeeping, and on odd ticks the worker-grouped fetch of the 64-bit context against tests/group_model.py."""
import numpy as np
import pytest

import drain_fuzz as D
import group_model as GM

pytestmark = pytest.mark.gpu

SEEN: dict = {}          # seed -> per-seed summary (loop bits per context, record kinds, ...)


def _contexts(d: D.Drain):
    from hyperqueue_b200 import _lib as L
    return [D.gpu_context(d, wide) for wide in (0, L.HQS_CREATE_WIDE_AMOUNTS)]


def run_seed(seed: int) -> dict:
    from hyperqueue_b200 import _lib as L
    d = D.Drain(seed)
    ctxs = _contexts(d)
    d.ctxs = ctxs
    sc = d.sc
    summary = {"W": sc.W, "R": sc.R, "Q": len(sc.classes), "ticks": sc.n_ticks, "paths": [0, 0], "narrow": set(),
               "kinds": [0, 0, 0], "per_task_emit": 0}

    def check(tick, inp, a, fa, pf):
        msg = D.judge_and_replay(d, inp, a, fa)
        assert msg is None, f"seed {seed} tick {tick}: the specification itself: {msg}"
        for i, s in enumerate(ctxs):
            where = f"seed {seed} tick {tick} context {'u64' if i else 'default'}"
            assert np.array_equal(s.free, inp.free), f"{where}: host free vectors differ from the drain's"
            assert np.array_equal(s._worker_structs(inp.now)["remaining_time_ms"], inp.remaining_ms), where
            grouped = i == 1 and tick % 2 == 1
            m = s.run_scheduling_grouped(inp.now) if grouped else s.run_scheduling(inp.now)
            st = s.stats()
            where += f" solver_path {st['solver_path']:#x} narrow_amounts {st['narrow_amounts']}"
            assert st["coarsened"] == 0, where
            if grouped:
                want, off = GM.group_model(a, sc.W)
                got = m.records
                assert np.array_equal(m.worker_off, off), f"{where}: worker offsets differ"
            else:
                got, want = m.assignments, a
            assert np.array_equal(got, want), f"{where}: {D.first_difference(inp, got, want)}"
            assert np.array_equal(m.free_after, fa), f"{where}: free_after differs"
            # host bookkeeping: prefills as the specification holds them; every redirect answered by the old worker
            n_pf = s._pf_worker.shape[0]
            assert np.array_equal(s._pf_worker[: d.H], pf) and (s._pf_worker[d.H:] < 0).all(), f"{where}: prefills"
            for w in np.unique(pf[pf >= 0]).tolist()[:8]:
                assert np.array_equal(s.prefilled_tasks(w), np.nonzero(pf == w)[0]), where
            red = a[a["kind"] == 2]
            for ow in np.unique(inp.pf_before[red["task"]]).tolist():
                mine = red[inp.pf_before[red["task"]] == ow]
                sent = s.on_retract_response(int(ow), mine["task"])
                exp = {}
                for t, w, v in zip(mine["task"].tolist(), mine["worker"].tolist(), mine["variant"].tolist()):
                    exp.setdefault(w, []).append((t, v))
                assert sent == exp, f"{where}: redirects of worker {ow}"
            assert s.redirects == {}, where
            assert n_pf >= d.H
            summary["paths"][i] |= st["solver_path"]
            if i == 0:
                summary["narrow"].add(st["narrow_amounts"])
            if a.size and not st["solver_path"] & L.HQS_PATH_EMIT_STAGED:
                summary["per_task_emit"] += 1
        for k in range(3):
            summary["kinds"][k] += int(np.count_nonzero(a["kind"] == k))

    try:
        out = d.run(check, trace=True)
    finally:
        for s in ctxs:
            s.close()
    tr = [t for *_, t in out]
    summary["reserved"] = sum(len(t["reserved"]) for t in tr)
    summary["restarts"] = sum(len(t["mu_excluded"]) for t in tr)
    summary["give_back"] = sum(len(t["give_back"]) for t in tr)
    print(f"seed {seed}: {summary}")
    return summary


@pytest.mark.parametrize("seed", D.SEEDS)
def test_drain_matches_specification(seed):
    SEEN[seed] = run_seed(seed)


def test_seed_set_reaches_every_solve_loop():
    """Over the whole seed set (seeds not run in this session are run here): every first-fit loop, the packed level,
    the minimum-utilisation restart and both emit passes ran, and the default context solved in both amount widths."""
    from hyperqueue_b200 import _lib as L
    for seed in D.SEEDS:
        if seed not in SEEN:
            SEEN[seed] = run_seed(seed)
    paths = 0
    narrow = set()
    per_task = 0
    for sm in SEEN.values():
        paths |= sm["paths"][0] | sm["paths"][1]
        narrow |= sm["narrow"]
        per_task += sm["per_task_emit"]
    want = (L.HQS_PATH_WIDE | L.HQS_PATH_LEAN | L.HQS_PATH_LEAN_EXTRAS | L.HQS_PATH_GENERAL | L.HQS_PATH_PACKED
            | L.HQS_PATH_MU_RESTART | L.HQS_PATH_EMIT_STAGED)
    assert paths & want == want, hex(paths)
    assert per_task > 0
    assert narrow == {0, 1}


def test_handed_back_pack_take_leaves_the_worker_reservable():
    """tests/test_drain_fuzz_spec.py::handed_back_worker_case on both amount widths: the worker whose pack take was handed
    back in full is reserved, and the lower level's tasks do not go there."""
    import greedy_model as G
    import parity as P
    from test_drain_fuzz_spec import handed_back_worker_case
    wl = handed_back_worker_case()
    exp, exp_free = G.model_tick(wl, np.ones(wl.n_tasks, dtype=bool), wl.worker_free)
    for flags in (0, 2):
        s = P.gpu_scheduler(wl, flags=flags)
        m = s.run_scheduling()
        assert np.array_equal(m.assignments, exp) and np.array_equal(m.free_after, exp_free), (flags, m.assignments)
        s.close()
