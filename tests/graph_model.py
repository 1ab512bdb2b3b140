"""Sequential model of task graphs on the device (hqs_graph_push / hqs_graph_finished / hqs_graph_debug, include/hqsched.h).

Test infrastructure.  GraphModel extends tests/level_model.py's key table by what the graph calls keep per handle (the
unfinished-dependency counter, the incarnation and the consumer list) and by the edge pool's bookkeeping:

  * hqs_graph_push(handles, classes, priorities, dep_off, deps): validated as a whole first (Rejected, nothing changed).
    A dependency counts if its handle is VALID or is an earlier task of the batch; a later task of the batch or a handle
    that is not VALID is dropped.  Every pushed handle starts a new incarnation; each counted dependency becomes an edge
    (consumer, incarnation) in its producer's list.  The keys are written as hqs_ready_push writes them (the same level
    policy), and a task with a counted dependency is VALID without READY.  The pool: the first push allocates
    max(2 * E, 4096) slots, E = the batch's dependencies that are not on later tasks of the batch; a push that finds
    used + E > capacity first compacts (keeps the edges whose consumer still waits on their incarnation; used = their
    number L; capacity = max(capacity, 2 * L + E); one more compaction); then used += E.
  * hqs_graph_finished(handles): every VALID handle leaves the table (a second mention or a handle that is not VALID does
    nothing), then each of them walks its list: a consumer that is waiting (VALID, not READY, not DONE) on the edge's
    incarnation loses a dependency and becomes READY at zero.  The lists of the finished handles are emptied.  Returns
    the newly READY handles, ascending.
  * hqs_ready_remove also empties the removed handles' lists (their consumers keep waiting).
  * hqs_graph_debug: [edges in all lists, pool capacity, compactions, waiting tasks].
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import numpy as np

import level_model as LM
from level_model import KEY_DONE, KEY_READY, KEY_VALID, NO_HANDLE, Rejected

POOL_MIN = 4096
WAIT_MASK = KEY_VALID | KEY_READY | KEY_DONE


class GraphModel(LM.LevelModel):
    def __init__(self) -> None:
        super().__init__()
        self.gdeps: Dict[int, int] = {}
        self.gen: Dict[int, int] = {}
        self.lists: Dict[int, List[Tuple[int, int]]] = {}     # producer -> [(consumer, incarnation)]
        self.pool_cap = 0
        self.pool_used = 0
        self.compactions = 0
        self.graph = False
        self.sharded = False

    # helpers --------------------------------------------------------------------------------------
    def flag(self, h: int) -> int:
        return int(self.flags[h]) if h < self.n_handles else 0

    def waiting(self, h: int) -> bool:
        return self.flag(h) & WAIT_MASK == KEY_VALID

    def _edge_waits(self, cons: int, g: int) -> bool:
        return self.gen.get(cons, 0) == g and self.waiting(cons)

    def _mode_check(self) -> None:
        if self.dag or self.sharded:
            raise Rejected()

    # calls ----------------------------------------------------------------------------------------
    def graph_push(self, handles, cls, prio, dep_off, deps) -> int:
        self._mode_check()
        h = [int(x) for x in np.asarray(handles, dtype=np.int64).tolist()]
        c = np.asarray(cls, dtype=np.uint32)
        p = np.asarray(prio, dtype=np.uint64)
        off = [int(x) for x in np.asarray(dep_off, dtype=np.int64).tolist()]
        d = [int(x) for x in np.asarray(deps, dtype=np.int64).tolist()]
        n = len(h)
        if n == 0:
            return 0
        if self.Q == 0:
            raise Rejected()
        if off[0] != 0 or any(off[i + 1] < off[i] for i in range(n)) or off[n] > len(d):
            raise Rejected()
        pos = {x: i for i, x in enumerate(h)}
        if len(pos) != n or NO_HANDLE in pos or int(c.max()) >= self.Q:
            raise Rejected()
        if any(self.flag(x) & KEY_VALID for x in h):
            raise Rejected()
        kept: List[List[int]] = []
        for i, x in enumerate(h):
            ds = d[off[i]: off[i + 1]]
            if len(set(ds)) != len(ds) or x in ds:
                raise Rejected()
            k = []
            for y in ds:
                j = pos.get(y)
                if j is None:
                    if y >= self.n_handles:
                        raise Rejected()
                    k.append(y)
                elif j < i:
                    k.append(y)
            kept.append(k)
        e = sum(len(k) for k in kept)
        # the pool, before anything is written
        if self.pool_cap == 0:
            self.pool_cap = max(2 * e, POOL_MIN)
        elif self.pool_used + e > self.pool_cap:
            self._compact(e)
        self.pool_used += e
        # the keys as hqs_ready_push writes them, then the dependencies (VALID at link time: the batch is VALID by now)
        valid_before = {y: bool(self.flag(y) & KEY_VALID) for k in kept for y in k if y not in pos}
        self.push(h, c, p)
        n_ready = 0
        for i, x in enumerate(h):
            g = self.gen.get(x, 0) + 1
            self.gen[x] = g
            cnt = 0
            for y in kept[i]:
                if y in pos or valid_before[y]:
                    self.lists.setdefault(y, []).append((x, g))
                    cnt += 1
            self.gdeps[x] = cnt
            if cnt:
                self.flags[x] &= np.uint32(~KEY_READY & 0xFFFFFFFF)
            else:
                n_ready += 1
        self.graph = True
        return n_ready

    def _compact(self, e: int) -> None:
        live = 0
        for prod in list(self.lists):
            kept = [(cn, g) for cn, g in self.lists[prod] if self._edge_waits(cn, g)]
            if kept:
                self.lists[prod] = kept
            else:
                del self.lists[prod]
            live += len(kept)
        self.pool_cap = max(self.pool_cap, 2 * live + e)
        self.pool_used = live
        self.compactions += 1

    def graph_finished(self, handles) -> List[int]:
        self._mode_check()
        h = [int(x) for x in np.asarray(handles, dtype=np.int64).tolist()]
        if any(x >= self.n_handles for x in h):
            raise Rejected()
        won = []
        for x in h:
            if self.flag(x) & KEY_VALID:
                self.flags[x] &= np.uint32(~(KEY_READY | KEY_VALID | KEY_DONE | LM.KEY_PF) & 0xFFFFFFFF)
                won.append(x)
        made = []
        for x in won:
            for cn, g in self.lists.pop(x, []):
                if self._edge_waits(cn, g):
                    self.gdeps[cn] -= 1
                    if self.gdeps[cn] == 0:
                        self.flags[cn] |= np.uint32(KEY_READY)
                        made.append(cn)
        return sorted(made)

    def remove(self, handles) -> None:
        super().remove(handles)
        for x in np.asarray(handles, dtype=np.int64).tolist():
            if x < self.n_handles:
                self.lists.pop(int(x), None)

    def dag_load(self, *a, **k) -> None:
        if self.graph:
            raise Rejected()
        super().dag_load(*a, **k)

    def debug(self) -> List[int]:
        edges = sum(len(v) for v in self.lists.values())
        waiting = int(np.count_nonzero((self.flags & np.uint32(WAIT_MASK)) == KEY_VALID)) if self.n_handles else 0
        return [edges, self.pool_cap, self.compactions, waiting]
