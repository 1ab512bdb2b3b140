"""The multi-tick drains of tests/drain_fuzz.py (pools of 1 to 1024 workers, every tick feature mixed) on sharded ready
sets, compared with the specification every tick.

For every seed the drain first runs on the specification alone, which gives its final handle count H and the records of
every tick (the drain is deterministic).  Then it runs once more with these systems attached in lockstep:
  * 2 ranks, unfused (hqs_shard_count + hqs_shard_solve_emit), cut at block_range(H): the upper rank starts empty;
  * 3 ranks, unfused, 64-bit amounts: one rank owns no handle at all, one cut lies inside some tick's assigned range of a
    (level, class) group;
  * 2 ranks, fused (hqs_shard_tick_launch, two HQS_CREATE_SHARE_DEVICE contexts), cut inside the first tick's largest
    prefill range (or assigned range when it has none);
  * ShardedScheduler itself as a world of one rank, with the unfused and with the peer-to-peer exchange.
Every tick, every rank must return the specification's records of its handles in order (kind 0 / 2, then kind 1) and its
free_after; the host free vectors before the tick are the drain's; the ranks' prefill bookkeeping together is the
specification's; every redirect is answered by its owner; no rank is coarsened, and the ranks report the same solver
path apart from the emit pass (HQS_PATH_EMIT_STAGED is decided per rank)."""
import numpy as np
import pytest
import torch

import drain_fuzz as D
from test_gpu_sharded_prefill import Ranks

pytestmark = pytest.mark.gpu

SEEN: dict = {}          # seed -> coverage summary


def _group_ranges(inp, a, kind1):
    """The tasks of each (level, class) group among the records of one kind class (assigned: kind 0 / 2; prefill: kind 1),
    ascending."""
    sel = a[(a["kind"] == 1) == kind1]["task"].astype(np.int64)
    out = {}
    for t in sel.tolist():
        out.setdefault((int(inp.wl.task_user_priority[t]), int(inp.wl.task_class[t])), []).append(t)
    return [np.sort(np.array(v)) for v in out.values()]


def _cut_inside(ranges):
    r = [t for t in ranges if t.size >= 2]
    if not r:
        return None
    t = max(r, key=len)
    return int(t[t.size // 2])


def plan(seed):
    """The specification's run: (H, cuts of the three rank configurations)."""
    from hyperqueue_b200.sharded import block_range
    d = D.Drain(seed)
    out = d.run()
    H = d.H
    half = block_range(H, 0, 2)[1]
    inp0, a0 = out[0][0], out[0][1]
    c3 = _cut_inside(_group_ranges(inp0, a0, True)) or _cut_inside(_group_ranges(inp0, a0, False)) or half
    c2 = None
    for inp, a, *_ in reversed(out):                       # a later tick than the fused cut's, where there is one
        c2 = _cut_inside(_group_ranges(inp, a, False))
        if c2 is not None:
            break
    c2 = c2 or half
    three = ([0, 0, c2, H], [0, c2, c2, H], [0, c2, H, H])[seed % 3]
    return H, [0, half, H], three, [0, c3, H]


class OneRank:
    """ShardedScheduler as a world of one rank behind the drain's GpuScheduler-shaped calls; the replicated worker state
    is set on its GpuScheduler.  Counts finished tasks that requested a resource whose total on their worker is MAX."""

    def __init__(self, d, H, p2p):
        from hyperqueue_b200.sharded import ShardedScheduler
        self.sh = ShardedScheduler(D.gpu_context(d, 0), 0, 1, H, torch.device("cuda", 0), p2p=p2p)
        self.max_finished = 0

    def close(self):
        self.sh.s.close()

    def add_ready_tasks(self, h, c, p):
        self.sh.add_ready_tasks(h, c, p)

    def remove_ready_tasks(self, h):
        self.sh.remove_ready_tasks(h)

    def set_blocked_mask(self, m):
        self.sh.s.set_blocked_mask(m)

    def tasks_finished(self, h):
        from hyperqueue_b200 import _lib as L
        s = self.sh.s
        t = np.asarray(h, dtype=np.int64)
        wi = s._task_worker[t]
        asked = s._amount_tab[s._task_class[t], s._task_variant[t]] > 0
        self.max_finished += int((asked & (s.total[wi] == np.uint64(L.HQS_AMOUNT_MAX))).any(axis=1).sum())
        self.sh.tasks_finished(h)

    def on_task_running_prefilled(self, t, v):
        self.sh.on_task_running_prefilled(int(t), v)

    def dispose_prefill(self, c):
        return self.sh.dispose_prefill(c)

    def on_retract_response(self, w, hs):
        return self.sh.on_retract_response(w, hs)

    # the tick interface of Ranks ------------------------------------------------------------------------------------
    @property
    def parts(self):
        return [(self.sh.s, self.sh.lo, self.sh.hi)]

    def tick(self, now):
        a, fa = self.sh.run_scheduling(now)
        return [a], [fa], [(0, "")]

    def pf_worker(self, n):
        pf = np.full(n, -1, dtype=np.int64)
        m = min(n, self.sh.s._pf_worker.shape[0])
        pf[:m] = self.sh.s._pf_worker[:m]
        return pf


def run_seed(seed):
    from hyperqueue_b200 import _lib as L
    H, two, three, fused = plan(seed)
    d = D.Drain(seed)
    mk = lambda flags: D.gpu_context(d, flags)                       # noqa: E731
    systems = []
    try:
        systems = [("2 ranks", Ranks(None, None, two, None, False, make=mk)),
                   ("3 ranks u64", Ranks(None, None, three, None, False, make=mk, flags=L.HQS_CREATE_WIDE_AMOUNTS)),
                   ("2 ranks fused", Ranks(None, None, fused, None, True, make=mk)),
                   ("sharded", OneRank(d, H, False)), ("sharded p2p", OneRank(d, H, True))]
        d.ctxs = [x for _, x in systems]
        sm = {"paths": 0, "narrow": set(), "per_task_emit": 0, "k1_upper": 0, "k2_upper": 0, "asg_cross": 0,
              "pf_cross": 0, "idle_rank": 0, "max_finished": 0}

        def check(tick, inp, a, fa, pf):
            msg = D.judge_and_replay(d, inp, a, fa)
            assert msg is None, f"seed {seed} tick {tick}: the specification itself: {msg}"
            red = a[a["kind"] == 2]
            for name, sys_ in systems:
                where = f"seed {seed} tick {tick} {name}"
                for s, _, _ in sys_.parts:
                    assert np.array_equal(s.free, inp.free), f"{where}: host free vectors differ from the drain's"
                recs, frees, errs = sys_.tick(inp.now)
                assert all(rc == 0 for rc, _ in errs), f"{where}: {errs}"
                paths = set()
                for r, ((s, lo, hi), got, fa_r) in enumerate(zip(sys_.parts, recs, frees)):
                    k = (a["task"] >= lo) & (a["task"] < hi)
                    want = np.concatenate([a[k & (a["kind"] != 1)], a[k & (a["kind"] == 1)]])
                    st = s.stats()
                    w = f"{where} rank {r} [{lo}, {hi}) solver_path {st['solver_path']:#x}"
                    assert np.array_equal(got, want), f"{w}: {D.first_difference(inp, got, want)}"
                    assert np.array_equal(fa_r, fa), f"{w}: free_after differs"
                    assert st["coarsened"] == 0, w
                    paths.add(st["solver_path"] & ~L.HQS_PATH_EMIT_STAGED)
                    sm["paths"] |= st["solver_path"]
                    sm["narrow"].add(st["narrow_amounts"])
                    if got.size and not st["solver_path"] & L.HQS_PATH_EMIT_STAGED:
                        sm["per_task_emit"] += 1
                    if r > 0:
                        sm["k1_upper"] += int(np.count_nonzero(got["kind"] == 1))
                        sm["k2_upper"] += int(np.count_nonzero(got["kind"] == 2))
                    if not inp.ready[lo:hi].any():
                        sm["idle_rank"] += 1
                assert len(paths) == 1, f"{where}: solver paths differ across ranks: {[hex(p) for p in paths]}"
                assert np.array_equal(sys_.pf_worker(d.H), pf), f"{where}: prefills"
                for ow in np.unique(inp.pf_before[red["task"]]).tolist():
                    mine = red[inp.pf_before[red["task"]] == ow]
                    sent = sys_.on_retract_response(int(ow), mine["task"])
                    exp = {}
                    for t, w_, v in zip(mine["task"].tolist(), mine["worker"].tolist(), mine["variant"].tolist()):
                        exp.setdefault(w_, []).append((t, v))
                    assert {w_: sorted(x) for w_, x in sent.items()} == {w_: sorted(x) for w_, x in exp.items()}, \
                        f"{where}: redirects of worker {ow}"
                for s, _, _ in sys_.parts:
                    assert s.redirects == {}, where
                if isinstance(sys_, Ranks):
                    inner = [lo for _, lo, _ in sys_.parts[1:] if 0 < lo < d.H]
                    for kind1, key in ((False, "asg_cross"), (True, "pf_cross")):
                        for t in _group_ranges(inp, a, kind1):
                            sm[key] += int(any(t[0] < c <= t[-1] for c in inner))

        d.run(check)
        sm["max_finished"] = sum(x.max_finished for _, x in systems if isinstance(x, OneRank))
    finally:
        for _, x in systems:
            x.close()
    print(f"seed {seed}: W {d.sc.W} R {d.sc.R} Q {len(d.sc.classes)} H {H} {sm}")
    return sm


@pytest.mark.parametrize("seed", D.SEEDS)
def test_sharded_drain_matches_specification(seed):
    SEEN[seed] = run_seed(seed)


def test_seed_set_reaches_every_sharded_case():
    """Over the whole seed set (seeds not run in this session are run here): every first-fit loop, the packed level, the
    minimum-utilisation restart and both emit passes ran on sharded ranks in both amount widths; a rank above rank 0
    emitted prefill (kind 1) and redirect (kind 2) records; an assigned range and a prefill range crossed a cut; some
    rank ticked with no task of its own; and a task that requested a resource finished on a worker whose total of it is
    HQS_AMOUNT_MAX."""
    from hyperqueue_b200 import _lib as L
    for seed in D.SEEDS:
        if seed not in SEEN:
            SEEN[seed] = run_seed(seed)
    tot = {k: 0 for k in ("per_task_emit", "k1_upper", "k2_upper", "asg_cross", "pf_cross", "idle_rank", "max_finished")}
    paths, narrow = 0, set()
    for sm in SEEN.values():
        paths |= sm["paths"]
        narrow |= sm["narrow"]
        for k in tot:
            tot[k] += sm[k]
    want = (L.HQS_PATH_WIDE | L.HQS_PATH_LEAN | L.HQS_PATH_LEAN_EXTRAS | L.HQS_PATH_GENERAL | L.HQS_PATH_PACKED
            | L.HQS_PATH_MU_RESTART | L.HQS_PATH_EMIT_STAGED)
    assert paths & want == want, hex(paths)
    assert narrow == {0, 1}, narrow
    assert all(v > 0 for v in tot.values()), tot
