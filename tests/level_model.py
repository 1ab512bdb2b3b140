"""Sequential model of the device task table's keys and of the priority-level policy (include/hqsched.h, DESIGN.md §4).

Test infrastructure: tests/test_gpu_ready_set.py runs the same call sequence on a context and on this model and compares
the whole key array (hqs_debug_keys) after every call.  The model keeps, per handle, the key's READY / DONE / VALID /
PREFILLED bits, its level field, its class and its u64 priority; per context, the registered priorities (descending),
the table the device searches (the same list, or coarse bucket bounds), the size of the set after its last pruning and
whether the levels were declared (hqs_levels_add).

The policy:
  * max_levels = max(1, HQS_MAX_GROUPS // Q).
  * A push registers every priority of the batch that is not registered yet, in exact and in coarse mode alike.  When
    something was registered, the levels are pruned if there are more than max_levels of them or more than
    2 * (size after the last pruning) + 64 (pruning keeps the priorities that a VALID key carries), then the device table
    is rebuilt and every VALID key is re-levelled.
  * The device table is the registered list when it has at most max_levels entries (exact: a key's level is the rank of
    its priority).  Otherwise it has M = max_levels buckets, entry b = levels[(b + 1) * L // M - 1] (the lowest priority
    of the bucket) and the last entry 0 (coarse: a key's level is the first bucket whose bound is <= its priority).
  * hqs_classes_set with another Q prunes (same triggers), rebuilds and re-levels; hqs_levels_add registers without ever
    pruning; hqs_dag_load replaces the table and registers exactly the DAG's priorities.
  * hqs_levels_live returns the registered list and, per entry, whether a VALID key carries it; hqs_levels_retain(keep)
    (the caller's pruning of declared levels, over all ranks) rejects a keep vector of another length or one that drops
    a carried level; otherwise it drops the unflagged levels, sets the size after the last pruning, and when something
    was dropped rebuilds the device table and re-levels every VALID key.
Levels are only ever written into VALID keys; a key that leaves the table keeps its level and class bits.
"""
from __future__ import annotations

from typing import List, Sequence

import numpy as np

HQS_MAX_GROUPS = 8192
KEY_READY, KEY_DONE, KEY_VALID, KEY_PF = 1 << 31, 1 << 30, 1 << 29, 1 << 28
LEVEL_SHIFT, LEVEL_MASK, CLASS_MASK = 14, 0x3FFF, 0x3FFF
NO_HANDLE = 0xFFFFFFFF


class Rejected(Exception):
    """The library rejects the call and leaves the context as it was."""


def max_levels(q: int) -> int:
    return max(1, HQS_MAX_GROUPS // max(q, 1))


def bucket_bounds(levels: Sequence[int], m: int) -> List[int]:
    """Device table of L > m registered priorities (descending): m buckets of adjacent levels, entry b = the lowest
    priority of bucket b, the last bucket takes everything below (bound 0)."""
    n = len(levels)
    out = [int(levels[(b + 1) * n // m - 1]) for b in range(m)]
    out[-1] = 0
    return out


def find_levels(table: np.ndarray, prio: np.ndarray, coarse: bool) -> np.ndarray:
    """Level of each priority: index of the first entry of the descending table that is <= p; coarse: clamped to the
    last bucket; exact: -1 unless that entry equals p."""
    table = np.asarray(table, dtype=np.uint64)
    prio = np.asarray(prio, dtype=np.uint64)
    n = table.size
    lo = n - np.searchsorted(table[::-1], prio, side="right")         # entries > p
    if coarse:
        return np.minimum(lo, n - 1).astype(np.int64)
    hit = lo < n
    hit[hit] = table[lo[hit]] == prio[hit]
    return np.where(hit, lo, -1).astype(np.int64)


class LevelModel:
    def __init__(self) -> None:
        self.Q = 0
        self.levels: List[int] = []          # registered priorities, descending
        self.table: List[int] = []           # what the device searches
        self.coarse = False
        self.declared = False
        self.pruned_at = 0
        self.dag = False
        self.n_handles = 0
        self.flags = np.zeros(0, dtype=np.uint32)
        self.lvl = np.zeros(0, dtype=np.uint32)
        self.cls = np.zeros(0, dtype=np.uint32)
        self.prio = np.zeros(0, dtype=np.uint64)
        self.deps = self.cons_off = self.cons = None

    # outputs --------------------------------------------------------------------------------------
    def keys(self) -> np.ndarray:
        return (self.flags | (self.lvl << np.uint32(LEVEL_SHIFT)) | (self.cls & np.uint32(CLASS_MASK))).astype(np.uint32)

    @property
    def n_levels(self) -> int:
        return len(self.table)

    @property
    def coarsened(self) -> int:
        return int(self.coarse)

    def has(self, bit: int) -> np.ndarray:
        return (self.flags & np.uint32(bit)) != 0

    def ready(self) -> np.ndarray:
        return self.has(KEY_READY)

    def live_priorities(self) -> np.ndarray:
        return np.unique(self.prio[self.has(KEY_VALID)])

    # policy ---------------------------------------------------------------------------------------
    def _grow(self, n: int) -> None:
        if n > self.n_handles:
            extra = n - self.n_handles
            self.flags = np.concatenate([self.flags, np.zeros(extra, np.uint32)])
            self.lvl = np.concatenate([self.lvl, np.zeros(extra, np.uint32)])
            self.cls = np.concatenate([self.cls, np.zeros(extra, np.uint32)])
            self.prio = np.concatenate([self.prio, np.zeros(extra, np.uint64)])
            self.n_handles = n

    def _merge(self, prios) -> bool:
        fresh = set(int(p) for p in np.unique(np.asarray(prios, dtype=np.uint64)).tolist()) - set(self.levels)
        if not fresh:
            return False
        self.levels = sorted(set(self.levels) | fresh, reverse=True)
        return True

    def need_pruning(self) -> bool:
        n = len(self.levels)
        return not self.declared and (n > max_levels(self.Q) or n > 2 * self.pruned_at + 64)

    def _prune(self) -> bool:
        if self.declared or not self.levels or self.n_handles == 0:
            return False
        live = set(int(p) for p in self.live_priorities().tolist())
        kept = [p for p in self.levels if p in live]
        dropped = len(kept) != len(self.levels)
        self.levels = kept
        self.pruned_at = len(kept)
        return dropped

    def _upload(self) -> None:
        m = max_levels(self.Q)
        if len(self.levels) <= m:
            self.table, self.coarse = list(self.levels), False
        else:
            self.table, self.coarse = bucket_bounds(self.levels, m), True

    def _find(self, prio: np.ndarray) -> np.ndarray:
        lv = find_levels(np.array(self.table, dtype=np.uint64), prio, self.coarse)
        return np.where(lv < 0, 0, lv).astype(np.uint32)            # not registered: provisionally level 0

    def _relevel(self) -> None:
        v = np.nonzero(self.has(KEY_VALID))[0]
        if v.size:
            self.lvl[v] = self._find(self.prio[v])

    def _register(self, prios) -> None:
        if self._merge(prios):
            if self.need_pruning():
                self._prune()
            self._upload()
            self._relevel()

    # operations -----------------------------------------------------------------------------------
    def push(self, handles, cls, prio) -> None:
        h = np.asarray(handles, dtype=np.int64)
        c = np.asarray(cls, dtype=np.uint32)
        p = np.asarray(prio, dtype=np.uint64)
        if h.size == 0:
            return
        assert np.unique(h).size == h.size, "a batch names each handle once"
        if self.Q == 0 or self.dag or int(h.max()) >= NO_HANDLE or int(c.max()) >= self.Q:
            raise Rejected()
        self._grow(int(h.max()) + 1)
        self.flags[h] = KEY_READY | KEY_VALID
        self.lvl[h] = self._find(p)
        self.cls[h] = c
        self.prio[h] = p
        self._register(p)

    def remove(self, handles) -> None:
        h = np.asarray(handles, dtype=np.int64)
        h = h[h < self.n_handles]
        self.flags[h] &= np.uint32(~(KEY_READY | KEY_VALID | KEY_DONE | KEY_PF) & 0xFFFFFFFF)

    def rearm(self) -> None:
        d = self.has(KEY_DONE)
        self.flags[d] = (self.flags[d] & np.uint32(~KEY_DONE & 0xFFFFFFFF)) | np.uint32(KEY_READY)

    def prefill_dispose(self, c: int) -> None:
        if c >= self.Q:
            raise Rejected()
        sel = self.has(KEY_PF) & ((self.cls & np.uint32(CLASS_MASK)) == c)
        self.flags[sel] &= np.uint32(~KEY_PF & 0xFFFFFFFF)

    def classes_set(self, q: int) -> None:
        changed = q != self.Q
        self.Q = q
        if changed and self.levels:
            was_coarse, old_n = self.coarse, len(self.table)
            dropped = self._prune() if self.need_pruning() else False
            self._upload()
            if dropped or was_coarse or self.coarse or old_n != len(self.table):
                self._relevel()

    def levels_add(self, prios) -> None:
        if len(prios) == 0:
            return
        self.declared = True
        if self._merge(prios):
            self._upload()
            self._relevel()

    def levels_live(self):
        """(registered priorities, descending; uint8 flag per entry: a VALID key carries it)."""
        live = set(int(p) for p in self.live_priorities().tolist()) if self.n_handles else set()
        return (np.array(self.levels, dtype=np.uint64),
                np.array([1 if p in live else 0 for p in self.levels], dtype=np.uint8))

    def levels_retain(self, keep) -> None:
        k = np.asarray(keep, dtype=np.uint8)
        _, live = self.levels_live()
        if k.size != len(self.levels) or (live.astype(bool) & (k == 0)).any():
            raise Rejected()
        kept = [p for p, f in zip(self.levels, k.tolist()) if f]
        self.pruned_at = len(kept)
        if len(kept) != len(self.levels):
            self.levels = kept
            self._upload()
            self._relevel()

    def dag_load(self, cls, prio, n_deps, cons_off, cons) -> None:
        c = np.asarray(cls, dtype=np.uint32)
        if self.Q == 0 or int(c.max()) >= self.Q:
            raise Rejected()
        n = c.size
        self.n_handles = n                                  # the new table replaces the old one, every key starts at 0
        self.flags = np.zeros(n, np.uint32)
        self.lvl = np.zeros(n, np.uint32)
        self.cls = np.zeros(n, np.uint32)
        self.prio = np.zeros(n, np.uint64)
        self.levels = []
        self._merge(prio)
        self._upload()
        self.deps = np.asarray(n_deps, dtype=np.int64).copy()
        self.cons_off = np.asarray(cons_off, dtype=np.int64)
        self.cons = np.asarray(cons, dtype=np.int64)
        self.cls[:] = c
        self.prio[:] = np.asarray(prio, dtype=np.uint64)
        self.lvl[:] = self._find(self.prio)
        self.flags[:] = np.where(self.deps == 0, KEY_VALID | KEY_READY, KEY_VALID).astype(np.uint32)
        self.dag = True

    def tasks_finished(self, tasks) -> int:
        """DAG mode: the tasks' consumers lose a dependency; a VALID consumer reaching zero becomes ready.  Returns how
        many did (n_new_ready).  A batch must not name a task twice or a task together with one of its producers."""
        if not self.dag:
            raise Rejected()
        t = np.asarray(tasks, dtype=np.int64)
        assert np.unique(t).size == t.size
        made = 0
        for x in t.tolist():
            for cn in self.cons[self.cons_off[x]: self.cons_off[x + 1]].tolist():
                self.deps[cn] -= 1
                if self.deps[cn] == 0 and self.flags[cn] & KEY_VALID:
                    self.flags[cn] |= np.uint32(KEY_READY)
                    made += 1
        self.flags[t] &= np.uint32(~(KEY_VALID | KEY_DONE | KEY_READY | KEY_PF) & 0xFFFFFFFF)
        return made

    def apply_tick(self, records: np.ndarray) -> None:
        """A tick's records: assigned tasks (kind 0 / 2) leave the ready set (DONE), prefilled ones (kind 1) stay ready."""
        asg = records["task"][records["kind"] != 1].astype(np.int64)
        self.flags[asg] = (self.flags[asg] & np.uint32(~(KEY_READY | KEY_PF) & 0xFFFFFFFF)) | np.uint32(KEY_DONE)
        pf = records["task"][records["kind"] == 1].astype(np.int64)
        self.flags[pf] |= np.uint32(KEY_PF)


# random call sequences ----------------------------------------------------------------------------
U64_MAX = (1 << 64) - 1
BATCH_SIZES = (1, 2, 31, 32, 33, 63, 255, 256, 257, 1000, 1023, 4097, 5000, 20000)


def _fresh_priorities(rng, k: int, used: set) -> List[int]:
    """k new priority values: tako priorities (user part in the high word, a nonzero job part in the low word), raw u64
    values, and the extremes 0 and 2^64 - 1."""
    out: List[int] = []
    while len(out) < k:
        kind = rng.integers(0, 10)
        if kind == 0:
            p = U64_MAX if rng.random() < 0.5 else 0
        elif kind < 6:
            user = int(rng.integers(-50, 50))
            p = (((user & 0xFFFFFFFF) ^ 0x80000000) << 32) | int(rng.integers(1, 1 << 32))
        else:
            p = int(rng.integers(0, 1 << 63)) * 2 + int(rng.integers(0, 2))
        if p not in used:
            used.add(p)
            out.append(p)
    return out


def _pool(used: set) -> np.ndarray:
    return np.array(sorted(used), dtype=np.uint64)


def random_op(rng, m: LevelModel, used: set, declared: bool, max_q: int = 4096, few_priorities: bool = False):
    """One call for a non-DAG context in state m: ("push", handles, classes, priorities, as_range), ("remove", handles),
    ("tick",), ("remove_done",), ("rearm",), ("dispose", class), ("classes", Q), ("levels_add", priorities) or, once
    levels were declared, ("levels_retain", keep) with keep = the live flags of levels_live() OR some dead levels another
    rank would still hold, and now and then a keep vector that drops a live level or has the wrong length (rejected).  `used`
    collects every priority handed out so far.  few_priorities: a batch brings at most one new priority, so that levels
    hold many tasks (proactive filling needs more waiting tasks in a level than its reserve)."""
    r = rng.random()
    if r < 0.40 or m.n_handles == 0:
        n = int(rng.choice(BATCH_SIZES)) if rng.random() < 0.6 else int(np.exp(rng.uniform(0, np.log(20000))))
        if few_priorities:
            n_fresh = min(n, 3) if len(used) < 3 else int(rng.random() < 0.3)
            prios = _fresh_priorities(rng, n_fresh, used)
            if len(prios) < n:
                prios += [int(x) for x in rng.choice(_pool(used), n - len(prios))]
        elif rng.random() < 0.08:
            n = 5000                                            # more fresh priorities than the device reports back
            prios = _fresh_priorities(rng, 4200, used) + [int(x) for x in rng.choice(_pool(used), 800)]
        else:
            n_fresh = min(n, int(rng.choice([0, 1, 3, 40, 300, n]))) if used else n
            prios = _fresh_priorities(rng, n_fresh, used)
            if len(prios) < n:
                # the rest mostly re-uses live priorities (a job's later tasks), sometimes any earlier one
                live = m.live_priorities()
                pool = live if live.size and rng.random() < 0.7 else _pool(used)
                prios += [int(x) for x in rng.choice(pool, n - len(prios))]
        prios = np.array(prios, dtype=np.uint64)
        rng.shuffle(prios)
        as_range = rng.random() < 0.5
        if as_range:
            first = int(rng.integers(0, m.n_handles + 1))
            handles = np.arange(first, first + n, dtype=np.int64)
        else:
            hi = max(m.n_handles + n // 4, n)
            handles = np.sort(rng.choice(hi, n, replace=False)).astype(np.int64)
            rng.shuffle(handles)
        cls = rng.integers(0, m.Q, n).astype(np.uint32)
        return ("push", handles.astype(np.uint32), cls, prios, as_range)
    if r < 0.50:
        # most tasks leave: only those of a few live priorities stay, fewer than the budget, so that the next push with a
        # new priority brings a coarse table back to exact levels
        live = m.live_priorities()
        valid = np.nonzero(m.has(KEY_VALID))[0]
        keep = rng.choice(live, min(live.size, max(1, max_levels(m.Q) // 2)), replace=False) if live.size else live
        return ("remove", valid[~np.isin(m.prio[valid], keep)].astype(np.uint32))
    if r < 0.57:
        k = int(rng.integers(1, m.n_handles + 1))
        h = rng.choice(m.n_handles, k, replace=False).astype(np.int64)
        beyond = rng.integers(m.n_handles, NO_HANDLE, int(rng.integers(0, 4)))   # past the table: ignored
        return ("remove", np.concatenate([h, beyond]).astype(np.uint32))
    if r < 0.71:
        return ("tick",)
    if r < 0.77:
        return ("remove_done",)
    if r < 0.82:
        return ("rearm",)
    if r < 0.87:
        return ("dispose", int(rng.integers(0, m.Q)))
    if r < 0.91 or not declared:
        q = min(max_q, m.Q + int(rng.choice([1, 1, 3, 7])))
        return ("classes", q)
    if r < 0.95 and m.declared:
        _, live = m.levels_live()
        keep = live | (rng.random(live.size) < rng.choice([0.0, 0.1, 0.5])).astype(np.uint8)
        u = rng.random()
        if u < 0.08 and live.any():
            keep[int(rng.choice(np.nonzero(live)[0]))] = 0          # drops a level a task carries
        elif u < 0.12:
            keep = np.concatenate([keep, [1]]).astype(np.uint8)   # not the table's length
        return ("levels_retain", keep)
    k = int(rng.choice([1, 10, 500]))
    return ("levels_add", np.array(_fresh_priorities(rng, k, used) + [int(x) for x in rng.choice(_pool(used), k)],
                                   dtype=np.uint64))
