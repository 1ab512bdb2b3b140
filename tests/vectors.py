"""Known-answer vectors of the reference's scheduler tests in a neutral form, for running the SAME cases
through the sequential specification (CPU) and the CUDA path (GPU).

Each case: workers (cpus[, extra resources]), tasks (priority, request variants), expected per-worker result as
a multiset of (class key, variant) counts — or None where only a predicate is pinned.  Source lines refer to
hyperqueue/crates/tako/src/internal/tests/test_scheduler_sn.rs.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import numpy as np

from workloads import FR, Workload


def case(workers, tasks, expect, name, running=None, resources=1, eq=None, worker_time=None, check=None):
    """workers: per worker (cpus[, extra resource units]); tasks: (priority, class key); running: worker -> cpus in use;
    eq: groups of interchangeable workers (the reference's eq_class); worker_time: worker -> remaining seconds;
    check: extra predicate over (per-worker class-key lists) for cases that pin a property instead of a placement."""
    return {"workers": workers, "tasks": tasks, "expect": expect, "name": name, "running": running or {}, "R": resources,
            "eq": eq or [], "worker_time": worker_time or {}, "check": check}


def c(cpus, **extra):          # single-variant request: cpus + {rid: units}
    d = {0: cpus}
    d.update({int(k[1:]): v for k, v in extra.items()})
    return (tuple(sorted(d.items())),)


def cv(*variants):             # variants: dicts rid -> units
    return tuple(tuple(sorted(v.items())) for v in variants)


def cw(cpus, weight=1.0, time=0.0, all_cpus=False):     # single variant with weight / min_time / cpus = All
    d = {} if all_cpus else {0: cpus}
    return (tuple(sorted(d.items())) + (("w", weight), ("t", time)) + ((("all", 0),) if all_cpus else ()),)


def _gap3(per):
    """test_schedule_gap_filling3 :496-526: both 34-cpu workers are filled to 33 cpus and at most two of the lower-priority
    3-cpu tasks land on each."""
    for lst in per:
        cpus = sum(dict(k[0])[0] for k, _p in lst)
        low = sum(1 for k, p in lst if p == 9)
        if cpus != 33 or low > 2:
            return f"worker holds {cpus} cpus, {low} low-priority tasks"
    return None


CASES = [
    # test_schedule_no_priorities :156-224  (expected: per worker list of cpu sizes)
    case([(3,)], [(0, c(3))], [[c(3)]], "nop-1"),
    case([(4,), (4,)], [(0, c(2))], [[c(2)], []], "nop-2"),
    case([(4,), (4,)], [(0, c(2))] * 2, [[c(2)] * 2, []], "nop-3"),
    case([(4,), (4,)], [(0, c(2))] * 3, [[c(2)] * 2, [c(2)]], "nop-4"),
    case([(4,), (4,)], [(0, c(2))] * 4, [[c(2)] * 2, [c(2)] * 2], "nop-5"),
    case([(4,), (4,)], [(0, c(2))] * 5, [[c(2)] * 2, [c(2)] * 2], "nop-6"),
    case([(4,), (4,)], [(0, c(2)), (0, c(3))], [[c(3)], [c(2)]], "nop-7"),
    case([(3,), (4,)], [(0, c(2)), (0, c(3))], [[c(3)], [c(2)]], "nop-8"),
    case([(4,), (4,)], [(0, c(5))] * 2 + [(0, c(1))] * 5, [[c(1)] * 4, [c(1)]], "nop-9"),
    case([(4,), (4,)], [(0, c(3)), (0, c(4)), (0, c(2))], [[c(4)], [c(3)]], "nop-10"),
    # test_schedule_priorities :226-307
    case([(4,), (4,)], [(1, c(2)), (1, c(2))], [[c(2)] * 2, []], "prio-1"),
    case([(4,), (4,)], [(1, c(2)), (2, c(2))], [[c(2)] * 2, []], "prio-2"),
    case([(4,), (4,)], [(0, c(4)), (0, c(4)), (1, c(2)), (2, c(3))], [[c(3)], [c(2)]], "prio-3"),
    case([(4,), (4,)], [(0, c(4)), (0, c(4)), (1, c(2)), (1, c(3))], [[c(3)], [c(2)]], "prio-4"),
    case([(4,), (4,)], [(1, c(4)), (1, c(4)), (1, c(2)), (1, c(3))], [[c(4)], [c(4)]], "prio-5"),
    case([(4,), (4,)], [(0, c(2)), (4, c(2)), (3, c(1)), (2, c(3))], "set:" , "prio-6-all-four"),     # MILP places all 4
    case([(4,), (4,)], [(1, c(5)), (0, c(4))], [[c(4)], []], "prio-7"),
    case([(4,)], [(9, c(2)), (7, c(1)), (6, c(2))], [[c(2), c(1)]], "prio-9"),
    case([(4,)], [(9, c(2)), (7, c(1)), (6, c(2)), (5, c(1))], [[c(2), c(1)]], "prio-10"),
    case([(10,)], [(9, c(2)), (8, c(1)), (7, c(2)), (6, c(1)), (5, c(2)), (4, c(1)), (3, c(2)), (2, c(1))],
         [[c(2), c(1), c(2), c(1), c(2), c(1)]], "prio-11"),
    case([(4,)], [(1, c(3))] * 3 + [(0, c(1))], [[c(3), c(1)]], "prio-12"),
    # test_schedule_no_irrelevant_blocking :309-330
    case([(3,)], [(10, c(5)), (0, c(1))], [[c(1)]], "noblock-1"),
    case([(3,), (5,)], [(10, c(5)), (9, c(5)), (0, c(1))], [[c(1)], [c(5)]], "noblock-2"),
    case([(5,), (3,)], [(10, c(3)), (9, c(2)), (8, c(5)), (0, c(1))], [[c(3), c(2)], [c(1)]], "noblock-3"),
    # test_schedule_gap_filling :410-449
    case([(12,)], [(1, c(8)), (1, c(8)), (0, c(4))], [[c(8), c(4)]], "gap-1"),
    case([(6,)], [(1, c(3))] * 3 + [(0, c(2))], [[c(3), c(3)]], "gap-2"),
    case([(8,)], [(1, c(3))] * 3 + [(0, c(1))] * 2, [[c(3), c(3), c(1), c(1)]], "gap-3"),
    case([(8,)], [(1, c(3))] * 3 + [(2, c(1)), (0, c(1))], [[c(1), c(3), c(3), c(1)]], "gap-4"),
    # test_schedule_multiple_resources1/2 :635-721 (gpus = resource 1)
    case([(4, 2)], [(0, c(2, r1=1))] * 2, [[c(2, r1=1)] * 2], "mres-1", resources=2),
    case([(4, 1)], [(0, c(2, r1=1))] * 2, [[c(2, r1=1)]], "mres-2", resources=2),
    case([(4, 1)], [(0, c(1, r1=2))], [[]], "mres-5", resources=2),
    case([(6, 0)], [(0, c(2))] * 10 + [(0, c(2, r1=1))] * 10, [[c(2)] * 3], "mres2-1", resources=2),
    case([(6, 10)], [(0, c(2))] * 10 + [(0, c(2, r1=1))] * 10, [[c(2, r1=1)] * 3], "mres2-2", resources=2),
    case([(6, 2)], [(0, c(2))] * 10 + [(0, c(2, r1=1))] * 10, [[c(2, r1=1)] * 2 + [c(2)]], "mres2-3", resources=2),
    case([(6, 2), (6, 0)], [(0, c(2))] * 10 + [(0, c(2, r1=1))] * 10, [[c(2, r1=1)] * 2 + [c(2)], [c(2)] * 3], "mres2-4", resources=2),
    # test_schedule_variants1 :723-754   (variant 0 = 2 cpus, variant 1 = 5 cpus)
    case([(11,)], [(0, cv({0: 2}, {0: 5}))] * 2, "count:2", "var1-1"),
    case([(8,)], [(0, cv({0: 2}, {0: 5}))] * 10, "count:4", "var1-4"),
    # test_generic_resource_variants1-3 :1053-1108
    case([(4, 0), (4, 2)], [(0, cv({0: 2}, {0: 1, 1: 1}))] * 4, "perworker:2,2", "gvar-1", resources=2),
    case([(4, 0), (4, 2)], [(0, cv({0: 8}, {0: 1, 1: 1}))] * 4, "perworker:0,2", "gvar-2", resources=2),
    case([(2, 0), (5, 1)], [(0, cv({0: 3}, {0: 1, 1: 1}))] * 4, "perworker:0,2", "gvar-3", resources=2),
    # test_no_deps_scattering_1 :793-815 (compaction)
    case([(5,), (5,), (5,)], [(0, c(1))] * 4, "perworker:4,0,0", "scatter-1"),
    # test_schedule_running :1308-1322
    case([(14,)], [(0, c(1))] * 10, "count:6", "running-1", running={0: 8}),
    # test_schedule_some_tasks_running :332-366
    case([(3,)], [(1, c(3))], "count:0", "somerun-1", running={0: 1}),
    case([(3,)], [(1, c(2))], "count:1", "somerun-2", running={0: 1}),
    case([(3,)], [(1, c(3)), (0, c(1))], "count:0", "somerun-3", running={0: 1}),
    case([(3,)], [(0, c(2)), (0, c(1)), (0, c(3))], [[c(2)]], "somerun-4a", running={0: 1}),
    case([(3,)], [(0, c(2)), (0, c(1)), (0, c(3))], [[c(1)]], "somerun-4b", running={0: 2}),
    case([(3,)], [(0, c(2)), (0, c(1)), (0, c(3))], [[]], "somerun-4c", running={0: 3}),
    # test_priority_switching :368-405: two workers x (w cpus, 10000 foo); a = 1 cpu, b = 1 cpu + 1 foo
] + [
    case([(w, 10000), (w, 10000)],
         [(10, c(1))] * 3 + [(9, c(1, r1=1))] * 2 + [(8, c(1))] + [(7, c(1))] * 3 + [(6, c(1, r1=1))] + [(5, c(1, r1=1))] +
         [(4, c(1))] * 5 + [(3, c(1, r1=1))], f"classcounts:{a},{b}", f"switch-{w}", resources=2)
    for w, a, b in [(1, 2, 0), (2, 3, 1), (3, 4, 2), (4, 6, 2), (5, 7, 3), (6, 8, 4), (7, 10, 4), (8, 12, 4), (9, 12, 5), (10, 12, 5)]
] + [
    # test_schedule_gap_filling :410-449, last case
    case([(8,)], [(1, c(3))] * 3 + [(2, c(1))] + [(0, c(1))] * 4, [[c(1), c(3), c(3), c(1)]], "gap-5"),
    # test_schedule_gap_filling2 :461-494 (foo = resource 1): a = 1 cpu, b = 3 cpus, c = 4 cpus + 1 foo
    case([(8, 0), (4, 1), (4, 1), (4, 1)], [(1, c(1))] * 7 + [(2, c(3))] * 3 + [(2, c(4, r1=1))] * 3, "classcounts:2,2,3", "gap2-plain", resources=2),
    case([(8, 0), (4, 1), (4, 1), (4, 1)], [(1, c(1))] * 7 + [(2, c(3))] * 3 + [(2, c(4, r1=1))] * 3 + [(-1, c(3))] * 2 +
         [(-2, c(4, r1=1))] * 3 + [(-3, c(1))] + [(-4, c(3))] * 2 + [(-5, c(4, r1=1))] * 3 + [(-6, c(1))], "classcounts:2,2,3", "gap2-extra", resources=2),
    # test_schedule_gap_filling3 :496-526
    case([(34,), (34,)], [(10, c(3))] * 5 + [(10, c(9))] * 6 + [(9, c(3))] * 5, "pred", "gap3", check=_gap3),
    # test_schedule_gap_filling4 :528-565 (foo = 1, bar = 2, goo = 3)
    case([(3, 10, 0, 10), (3, 10, 0, 10), (3, 10, 10, 0)], [(10, c(2, r3=1))] * 5 + [(9, c(1, r1=1))] * 2 + [(8, c(3, r1=1, r2=1))] * 10,
         "classcounts:2,2,1", "gap4", resources=4),
    # test_schedule_reservation_simple..5 :567-633
    case([(3,), (3,)], [(3, c(3)), (2, c(2))], [[], [c(2)]], "resv-1", running={0: 1, 1: 1}, eq=[[0, 1]]),
    case([(3,), (3,)], [(3, c(3)), (2, c(1)), (2, c(1))], [[], [c(1), c(1)]], "resv-2", running={0: 1, 1: 1}, eq=[[0, 1]]),
    case([(3,), (3,)], [(3, c(3)), (2, c(1)), (2, c(1))], [[c(1)], []], "resv-3", running={0: 2, 1: 1}),
    case([(4,), (3,), (3,), (3,)], [(4, c(3)), (3, c(3)), (3, c(3)), (2, c(1)), (2, c(1))], [[c(3)], [c(1)], [], []], "resv-4",
         running={0: 1, 1: 2, 2: 2, 3: 1}),
    case([(3,), (3,), (3,), (4,)], [(4, c(3)), (3, c(3)), (3, c(3)), (2, c(1)), (2, c(1))], [[c(1)], [], [], [c(3), c(1)]], "resv-5",
         running={0: 2, 1: 2, 2: 1}),
    # test_resource_time_assign / _balance1 :873-904 (worker time limits, task time requests)
    case([(10,)], [(0, cw(1, time=170.0)), (0, cw(1)), (0, cw(1, time=99.0))], [[cw(1), cw(1, time=99.0)]], "time-assign", worker_time={0: 100.0}),
    case([(1,), (1,), (1,)], [(0, cw(1, time=170.0)), (0, cw(1)), (0, cw(1, time=99.0))], [[cw(1)], [cw(1, time=170.0)], [cw(1, time=99.0)]],
         "time-balance1", worker_time={0: 50.0, 1: 200.0, 2: 100.0}),
    # test_schedule_variant_gap1 :1324-1351: 8 cpus OR 4 cpus + 2 gpus at priority 10, then 1-cpu tasks
] + [
    case([(14, 4)], [(10, cv({0: 8}, {0: 4, 1: 2}))] * 10 + [(0, c(1))] * 10, f"classcounts:*,{2 - r}", f"vargap-{r}", running={0: r}, resources=2)
    for r in (0, 1, 2)
] + [
    # test_schedule_resource_weights1/2 :1353-1389
    case([(4,)], [(0, cw(3)), (0, cw(2, weight=1.49))], [[cw(3)]], "weight1-a"),
    case([(4,)], [(0, cw(3, weight=1.0)), (0, cw(2, weight=1.51))], [[cw(2, weight=1.51)]], "weight1-b"),
    case([(12,)], [(0, cw(3, weight=1.1))] * 5 + [(0, cw(0, all_cpus=True))], [[cw(3, weight=1.1)] * 4], "weight2-a"),
    case([(12,)], [(0, cw(3))] * 5 + [(0, cw(0, weight=1.1, all_cpus=True))], [[cw(0, weight=1.1, all_cpus=True)]], "weight2-b"),
    # test_schedule_min_utilization3 :1447-1463 is in tests/test_gpu_edges.py (needs worker options)
    # test_schedule_variants2 :757-784: 10 tasks of {6 cpus} | {2 cpus + 2 gpus} on 12 cpus with 0 / 4 / 20 gpus
    case([(12, 0)], [(0, cv({0: 6}, {0: 2, 1: 2}))] * 10, "varcounts:2,0", "var2-nogpu", resources=2),
    case([(12, 4)], [(0, cv({0: 6}, {0: 2, 1: 2}))] * 10, "varcounts:1,2", "var2-4gpus", resources=2),
    case([(12, 20)], [(0, cv({0: 6}, {0: 2, 1: 2}))] * 10, "varcounts:0,6", "var2-20gpus", resources=2),
    # test_no_deps_scattering_2 :816-847: one new 1-cpu task per tick on 3 x 5 cpus; the running tasks of the earlier ticks
    # keep their cpus (the reference compares sorted counts; first-fit fills the lowest worker id)
    case([(5,), (5,), (5,)], [(0, c(1))], "perworker:1,0,0", "scatter2-a", running={0: 3}),
    case([(5,), (5,), (5,)], [(0, c(1))], "perworker:0,1,0", "scatter2-b", running={0: 5, 1: 2}),
    case([(5,), (5,), (5,)], [(0, c(1))], "perworker:0,0,1", "scatter2-c", running={0: 5, 1: 5, 2: 4}),
    case([(5,), (5,), (5,)], [(0, c(1))], "perworker:0,0,0", "scatter2-d", running={0: 5, 1: 5, 2: 5}),
    # test_generic_resource_assign2 :906-937: w1 (10 cpus, 10 Res0), w2 (10 cpus), w3 (10 cpus, 10 Res0, 1e6 Res1);
    # 50 x {1 cpu, 1 Res0} + 50 x {1 cpu, 2 Res0}: 10 tasks of the first kind on w1 and on w3, nothing on w2
    case([(10, 10, 0), (10, 0, 0), (10, 10, 1000000)], [(0, c(1, r1=1))] * 50 + [(0, c(1, r1=2))] * 50,
         [[c(1, r1=1)] * 10, [], [c(1, r1=1)] * 10], "gres-assign2", resources=3),
    # test_generic_resource_balance1/2 :939-990
    case([(10, 10, 0), (10, 0, 0), (10, 10, 1000000)], [(0, c(1, r1=5))] * 4, "perworker:2,0,2", "gres-balance1", resources=3),
    case([(10, 10, 0), (10, 0, 0), (10, 10, 1000000)],
         [(0, c(1, r1=5)), (0, c(1, r1=5, r2=500000)), (0, c(1, r1=5)), (0, c(1, r1=5, r2=500000))],
         [[c(1, r1=5)] * 2, [], [c(1, r1=5, r2=500000)] * 2], "gres-balance2", resources=3),
    # test_scheduler_two_running_three_waiting :1110-1127: 8 cpus + 4 foo, two running {1 cpu, 2 foo} tasks hold all foo;
    # the 2-cpu task at priority 1 is assigned, the two waiting {1 cpu, 2 foo} tasks stay
    case([(8, 4)], [(1, c(2)), (0, c(1, r1=2)), (0, c(1, r1=2))], [[c(2)]], "two-running-three-waiting", running={0: (2, 4)}, resources=2),
]


def to_workload(cs) -> Tuple[Workload, List[Tuple]]:
    R = cs["R"]
    classes: List = []
    keys: List[Tuple] = []
    cls_of = []
    for prio, key in cs["tasks"]:
        if key not in keys:
            keys.append(key)
            vs = []
            for var in key:
                d = {"amounts": {r: int(u * FR) for r, u in var if isinstance(r, int)}}
                opts = {r: u for r, u in var if not isinstance(r, int)}
                if "w" in opts:
                    d["weight"] = opts["w"]
                if opts.get("t"):
                    d["min_time_s"] = opts["t"]
                if "all" in opts:
                    d["all"] = (opts["all"],)
                vs.append(d)
            classes.append(vs)
        cls_of.append(keys.index(key))
    W = len(cs["workers"])
    total = np.zeros((W, R), dtype=np.uint64)
    for w, res in enumerate(cs["workers"]):
        for r, u in enumerate(res):
            total[w, r] = u * FR
    free = total.copy()
    for w, used in cs["running"].items():          # cpus in use, or units in use per resource
        for r, u in enumerate(used if isinstance(used, tuple) else (used,)):
            free[w, r] -= np.uint64(u * FR)
    rem = None
    if cs.get("worker_time"):
        rem = np.full(W, np.inf)
        for w, t in cs["worker_time"].items():
            rem[w] = t
    wl = Workload(R, classes, total, free, np.array(cls_of, dtype=np.uint32),
                  np.array([p for p, _ in cs["tasks"]], dtype=np.int32), worker_remaining_s=rem, name=cs["name"])
    return wl, keys


def check(cs, wl, keys, a) -> Optional[str]:
    """a: assignment array (task, worker, variant).  Returns None if the expectation holds, else a message."""
    W = wl.n_workers
    exp = cs["expect"]
    per = [[] for _ in range(W)]
    for t, w, v in zip(a["task"].tolist(), a["worker"].tolist(), a["variant"].tolist()):
        per[w].append(keys[wl.task_class[t]])
    if isinstance(exp, str):
        kind, _, arg = exp.partition(":")
        if kind == "classcounts":      # assigned tasks per class, classes in order of first appearance ("*" = any)
            got = np.bincount(wl.task_class[a["task"]], minlength=len(keys)).tolist()
            want = arg.split(",")
            ok = all(x == "*" or int(x) == g for x, g in zip(want, got))
            return None if ok else f"class counts {got} != {want}"
        if kind == "pred":
            prio = wl.task_user_priority
            perp = [[] for _ in range(W)]
            for t, w in zip(a["task"].tolist(), a["worker"].tolist()):
                perp[w].append((keys[wl.task_class[t]], int(prio[t])))
            return cs["check"](perp)
        if kind == "count":
            return None if a.shape[0] == int(arg) else f"assigned {a.shape[0]} != {arg}"
        if kind == "varcounts":        # assigned tasks per variant id
            got = np.bincount(a["variant"], minlength=8).tolist()
            want = [int(x) for x in arg.split(",")]
            return None if got[:len(want)] == want and sum(got[len(want):]) == 0 else f"variant counts {got} != {want}"
        if kind == "perworker":
            want = [int(x) for x in arg.split(",")]
            got = [len(p) for p in per]
            return None if got == want else f"per-worker {got} != {want}"
        if kind == "set":
            return None if a.shape[0] == len(cs["tasks"]) else f"assigned {a.shape[0]} of {len(cs['tasks'])}"
        raise ValueError(exp)
    got = [sorted(map(repr, p)) for p in per]
    want = [sorted(map(repr, e)) for e in exp]
    for grp in cs.get("eq", []):       # interchangeable workers: compare as multisets
        g_got = sorted(got[w] for w in grp)
        g_want = sorted(want[w] for w in grp)
        for w, x in zip(grp, g_got):
            got[w] = x
        for w, x in zip(grp, g_want):
            want[w] = x
    return None if got == want else f"{got} != {want}"
