"""hqs_graph_cancel (include/hqsched.h) added to the sequential task-graph model (tests/graph_model.py).

Test infrastructure.  CancelModel.graph_cancel(handles): a handle >= n_handles rejects the batch (Rejected, nothing
changed).  Every named handle that is VALID leaves the table, and so does, transitively, every consumer that still waits on
the incarnation its edge was made for (the same test hqs_graph_finished applies before it releases a consumer).  All of
them leave as hqs_ready_remove makes a handle leave (key bits cleared, consumer list emptied).  Returns them, ascending.
"""
from __future__ import annotations

from typing import List

import numpy as np

from graph_model import GraphModel
from level_model import KEY_VALID, Rejected


class CancelModel(GraphModel):
    def graph_cancel(self, handles) -> List[int]:
        self._mode_check()
        h = [int(x) for x in np.asarray(handles, dtype=np.int64).tolist()]
        if any(x >= self.n_handles for x in h):
            raise Rejected()
        gone = {x for x in h if self.flag(x) & KEY_VALID}
        stack = list(gone)
        while stack:
            for cn, g in self.lists.get(stack.pop(), []):
                if cn not in gone and self._edge_waits(cn, g):
                    gone.add(cn)
                    stack.append(cn)
        out = sorted(gone)
        self.remove(out)
        return out
