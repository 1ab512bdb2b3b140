"""LP/MIP facade over HiGHS, restated (TEST INFRASTRUCTURE — see oracle/__init__.py).

Follows hyperqueue/crates/tako/src/internal/solver/mod.rs:27-41 (LpInnerSolver trait) and
solver/highs.rs:4-63 (HiGHS backend: integer columns 0..=1 / 0.., rows `..=v`, `v..`, `v..=v`,
`optimise(Sense::Maximise).solve()`, result only when HighsModelStatus::Optimal).

The reference links HiGHS through crate `highs 1.12.0` / `highs-sys 1.12.1` (Cargo.lock:1106-1123,
source not in the reference repository).  Here the same HiGHS release (1.12.0, bundled in scipy 1.18) is
driven through scipy.optimize.milp.  Among tied optima the two drivers may differ (option defaults
of the `highs` crate are not verifiable here); the reference's own tests tolerate that (eq_class).
"""
from __future__ import annotations

from typing import Iterable, List, Optional, Tuple

import numpy as np
import scipy.sparse as sp
from scipy.optimize import Bounds, LinearConstraint, milp

MAX, MIN, EQ = "max", "min", "eq"      # ConstraintType (solver/mod.rs:20-25)


class LpSolver:
    def __init__(self) -> None:
        self.obj: List[float] = []
        self.lb: List[float] = []
        self.ub: List[float] = []
        self.integrality: List[int] = []
        self.rows: List[int] = []
        self.cols: List[int] = []
        self.vals: List[float] = []
        self.row_lo: List[float] = []
        self.row_hi: List[float] = []

    # variables ----------------------------------------------------------------------------
    def _add(self, weight: float, lo: float, hi: float, integer: int) -> int:
        self.obj.append(float(weight))
        self.lb.append(lo)
        self.ub.append(hi)
        self.integrality.append(integer)
        return len(self.obj) - 1

    def add_variable(self, weight: float, lo: float, hi: float) -> int:
        return self._add(weight, lo, hi, 0)

    def add_bool_variable(self, weight: float) -> int:
        return self._add(weight, 0.0, 1.0, 1)          # highs.rs:22-24

    def add_nat_variable(self, weight: float) -> int:
        return self._add(weight, 0.0, np.inf, 1)       # highs.rs:27-29

    # constraints --------------------------------------------------------------------------
    def add_constraint(self, ctype: str, value: float, terms: Iterable[Tuple[int, float]]) -> None:
        r = len(self.row_lo)
        # HiGHS' RowProblem sums duplicate (row, col) entries; scipy's COO->CSR does the same.
        n = 0
        for v, c in terms:
            self.rows.append(r)
            self.cols.append(v)
            self.vals.append(float(c))
            n += 1
        if ctype == MAX:
            lo, hi = -np.inf, float(value)
        elif ctype == MIN:
            lo, hi = float(value), np.inf
        else:
            lo = hi = float(value)
        self.row_lo.append(lo)
        self.row_hi.append(hi)

    # solve --------------------------------------------------------------------------------
    def solve(self, time_limit: Optional[float] = None, mip_rel_gap: Optional[float] = None,
              accept_incumbent: bool = False) -> Optional[Tuple[np.ndarray, float]]:
        """Maximise.  Returns (values, objective) or None unless the status is Optimal.

        Defaults reproduce the reference (HiGHS defaults, Optimal only).  The two relaxations exist
        because the reference's MILP is a multi-dimensional knapsack that HiGHS cannot close to its
        default 0.01 % gap in bounded time on many-class inputs (seconds to minutes for ~130 variables,
        see DESIGN.md "oracle practicality"): `mip_rel_gap` loosens the optimality tolerance and
        `accept_incumbent` returns the best feasible point when `time_limit` strikes (where the
        reference would return None and schedule nothing, solver.rs:412-415)."""
        n = len(self.obj)
        if n == 0:
            return np.zeros(0), 0.0
        c = -np.asarray(self.obj, dtype=np.float64)
        constraints = []
        if self.row_lo:
            a = sp.csr_matrix((self.vals, (self.rows, self.cols)), shape=(len(self.row_lo), n))
            constraints.append(LinearConstraint(a, np.asarray(self.row_lo), np.asarray(self.row_hi)))
        options = {"disp": False}
        if time_limit is not None:
            options["time_limit"] = time_limit
        if mip_rel_gap is not None:
            options["mip_rel_gap"] = mip_rel_gap
        res = milp(c, constraints=constraints, integrality=np.asarray(self.integrality),
                   bounds=Bounds(np.asarray(self.lb), np.asarray(self.ub)), options=options)
        self.last_status = res.status
        if res.x is None:
            return None
        if res.status != 0 and not (accept_incumbent and res.status == 1):   # 0 = Optimal, 1 = limit reached
            return None
        return res.x, -float(res.fun)
