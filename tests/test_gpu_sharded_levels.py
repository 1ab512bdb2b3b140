"""Pruning the declared priority levels of a sharded ready set across its ranks.

Every rank declares every priority it is given (hqs_levels_add), so that all ranks number the levels alike, and no
declared context prunes on its own.  Without pruning the table grows with every distinct priority ever submitted: past
HQS_MAX_GROUPS / Q levels the table is coarsened for good (tasks of merged levels are no longer ordered by priority), and
with proactive filling every tick fails past HQS_MAX_GROUPS / (2 Q) levels.  The ranks prune together at tick start:
each reports which levels its tasks carry, the vectors are OR-ed, and every rank keeps the same levels.

Waves of tasks at about 30 never-used priorities each run through 2 ranks (unfused and fused) and through
ShardedScheduler as a world of one rank; the assigned tasks finish and their handles are retired between ticks.  One old
level is held only by tasks of rank 1 whose class is blocked on every worker: it must survive every pruning on rank 0
too, and once unblocked its tasks come out where a single context puts them.  Every tick of every rank equals a single
GpuScheduler holding all the tasks (which prunes on its own), reports coarsened == 0 and keeps its levels within the
budget."""
import numpy as np
import pytest
import torch

from test_gpu_sharded_prefill import Ranks, _sched
from workloads import FR, MAXV

pytestmark = pytest.mark.gpu

W, H, N_WAVES, PER_WAVE, TASKS_PER_PRIO = 10, 1200, 10, 30, 2
N_HELD = 6                                    # the blocked tasks of the old level: the top handles, owned by rank 1
OLD_USER_PRIORITY = 61                        # odd: the waves use even user priorities
BUDGETS = {"prefill_q16": (16, (0, 2)), "plain_q64": (64, None)}


class _OneRank:
    """ShardedScheduler as a world of one rank, behind the tick interface of Ranks."""

    def __init__(self, classes, prefill):
        from hyperqueue_b200.sharded import ShardedScheduler
        self.sh = ShardedScheduler(_sched(1, classes, 0, prefill), 0, 1, H, torch.device("cuda", 0))
        self.parts = [(self.sh.s, 0, H)]

    def __getattr__(self, name):               # the task calls, with global handles
        return getattr(self.sh, name)

    def new_worker(self, wid, res):
        self.sh.s.new_worker(wid, res)

    def set_blocked_mask(self, m):
        self.sh.s.set_blocked_mask(m)

    def tick(self):
        a, fa = self.sh.run_scheduling()
        return [a], [fa], [(0, "")]

    def close(self):
        self.sh.s.close()


@pytest.mark.parametrize("mode", ["unfused", "fused", "sharded"])
@pytest.mark.parametrize("budget", sorted(BUDGETS))
def test_declared_levels_are_pruned_across_ranks(budget, mode):
    from hyperqueue_b200 import _lib as L, priority_from_user
    Q, prefill = BUDGETS[budget]
    classes = [[{0: FR + c}] for c in range(Q)]             # distinct classes; 7 tasks fill a worker
    held_class = Q - 1
    max_levels = L.HQS_MAX_GROUPS // (Q * (2 if prefill else 1))
    rng = np.random.default_rng(Q)
    ref = _sched(1, classes, 0, prefill)
    sys_ = _OneRank(classes, prefill) if mode == "sharded" else Ranks(1, classes, [0, H // 2, H], prefill, mode == "fused")
    blocked = np.zeros((W, Q, MAXV), dtype=bool)
    blocked[:, held_class, :] = True
    pushed = set()
    try:
        for x in (ref, sys_):
            for i in range(W):
                x.new_worker(i, [8 * FR])
            x.set_blocked_mask(blocked)
        held = np.arange(H - N_HELD, H)
        p_old = priority_from_user(np.full(N_HELD, OLD_USER_PRIORITY))
        ref.add_ready_tasks(held.astype(np.uint32), np.full(N_HELD, held_class, np.uint32), p_old)
        sys_.add_ready_tasks(held, np.full(N_HELD, held_class, np.uint32), p_old)
        pushed.add(OLD_USER_PRIORITY)
        free_handles = set(range(H - N_HELD))

        def tick(label):
            m = ref.run_scheduling()
            recs, frees, errs = sys_.tick()
            assert all(rc == 0 for rc, _ in errs), (label, errs)
            ra = m.assignments
            for r, ((s, lo, hi), a, fa) in enumerate(zip(sys_.parts, recs, frees)):
                st = s.stats()
                assert st["coarsened"] == 0 and st["n_levels"] <= max_levels, (label, r, st)
                k = (ra["task"] >= lo) & (ra["task"] < hi)
                want = np.concatenate([ra[k & (ra["kind"] != 1)], ra[k & (ra["kind"] == 1)]])
                assert np.array_equal(a, want), (label, r, a[:6], want[:6])
                assert np.array_equal(fa, m.free_after), (label, r)
            assert ref.stats()["coarsened"] == 0, label
            return ra

        for wave in range(N_WAVES):
            users = 2 * (PER_WAVE * wave + np.arange(PER_WAVE))
            pushed |= set(users.tolist())
            h = np.sort(rng.choice(sorted(free_handles), PER_WAVE * TASKS_PER_PRIO, replace=False))
            free_handles -= set(h.tolist())
            c = rng.integers(0, held_class, h.size).astype(np.uint32)
            p = priority_from_user(rng.permutation(np.repeat(users, TASKS_PER_PRIO)))
            ref.add_ready_tasks(h.astype(np.uint32), c, p)
            sys_.add_ready_tasks(h, c, p)
            ra = tick(f"wave {wave}")
            done = np.sort(ra["task"][ra["kind"] != 1]).astype(np.int64)
            assert not np.isin(done, held).any()
            # the assigned tasks finish and their handles are retired (they no longer keep their levels alive)
            ref.tasks_finished(done.astype(np.uint32))
            ref.remove_ready_tasks(done.astype(np.uint32))
            sys_.tasks_finished(done)
            sys_.remove_ready_tasks(done)
            free_handles |= set(done.tolist())
        assert len(pushed) > max_levels, (len(pushed), max_levels)
        # the old level is live only on the rank that owns the held tasks, and every rank still has it
        for s, lo, hi in sys_.parts:
            lv, live = s.levels_live()
            k = np.nonzero(lv == p_old[0])[0]
            assert k.size == 1, (lo, hi)
            assert bool(live[k[0]]) == (lo < H <= hi)
        assert len(sys_.parts[0][0].levels_live()[0]) < len(pushed)          # the ranks did prune
        for x in (ref, sys_):
            x.set_blocked_mask(None)
        ra = tick("unblocked")
        assert np.isin(held, ra["task"][ra["kind"] != 1]).all()
    finally:
        sys_.close()
        ref.close()
