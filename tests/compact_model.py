"""hqs_handles_compact (include/hqsched.h) added to the sequential task-graph model (tests/graph_cancel_model.py).

Test infrastructure.  CompactModel.compact(keep): a keep entry >= n_handles rejects the call (Rejected, nothing changed), and
so does a DAG or sharded context.  The survivors are the VALID handles and the handles in keep; survivor i, in ascending old
handle, becomes handle i with its key, priority, dependency count and incarnation; each survivor's consumer list keeps, in
order, the edges whose consumer still waits on the edge's incarnation, with the consumers renumbered.  n_handles becomes the
number of survivors; the level table is unchanged.  Returns old_of_new.

`mutant` breaks one rule on purpose, so that the tests can show they would catch it: "edge_remap" leaves the consumers of
the edges unrenumbered, "incarnation" does not carry the incarnation (it restarts at 0).
"""
from __future__ import annotations

from typing import Iterable, List, Optional

import numpy as np

from graph_cancel_model import CancelModel
from level_model import KEY_VALID, Rejected


class CompactModel(CancelModel):
    def __init__(self, mutant: Optional[str] = None) -> None:
        super().__init__()
        self.mutant = mutant

    def compact(self, keep: Iterable[int] = ()) -> List[int]:
        self._mode_check()
        k = [int(x) for x in np.asarray(list(keep), dtype=np.int64).tolist()]
        if any(x >= self.n_handles for x in k):
            raise Rejected()
        valid = np.nonzero(self.flags[: self.n_handles] & np.uint32(KEY_VALID))[0].tolist() if self.n_handles else []
        old = sorted(set(valid) | set(k))
        new_of = {o: i for i, o in enumerate(old)}
        lists = {}                          # against the old table: an edge's consumer waits, so it is VALID and survives
        for prod, edges in self.lists.items():
            kept = [(cn if self.mutant == "edge_remap" else new_of[cn], g) for cn, g in edges if self._edge_waits(cn, g)]
            if kept:
                lists[new_of[prod]] = kept
        idx = np.asarray(old, dtype=np.int64)
        self.flags, self.lvl, self.cls, self.prio = (a[idx].copy() for a in (self.flags, self.lvl, self.cls, self.prio))
        self.n_handles = len(old)
        self.gdeps = {new_of[h]: v for h, v in self.gdeps.items() if h in new_of}
        self.gen = {} if self.mutant == "incarnation" else {new_of[h]: v for h, v in self.gen.items() if h in new_of}
        self.lists = lists
        self.pool_used = sum(len(v) for v in lists.values())
        return old
