"""CPU oracle: a restatement of HyperQueue's tako scheduler tick (v0.26.0, commit d3575d0).

TEST INFRASTRUCTURE ONLY.  Nothing under ``hyperqueue_b200/`` may import this package; only
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline / ``--impl reference``
legs use it, and there only as the checker (or as the timed CPU baseline), never as the product.

The reference is Rust + HiGHS (crate ``highs 1.12.0`` / ``highs-sys 1.12.1``, not vendored in the
reference repository) and is not built here (it needs cargo/rustc).  This package restates the
algorithm in Python/numpy, solving the MIP with the same HiGHS version (1.12.0) bundled in scipy
(``scipy.optimize.milp``).  Parity is PINNED: ``tests/test_oracle_golden.py`` replays the
known-answer vectors of the reference's own tests
(crates/tako/src/internal/tests/test_scheduler_sn.rs, scheduler/gap.rs:175-246,
scheduler/batches.rs:223-250) against this restatement.

Module map (reference file each one follows, paths relative to crates/tako/src/internal/):
  model.py      common/resources/{amount,request,map}.rs, server/{workerload,worker}.rs, common/priority.rs
  taskqueue.py  scheduler/taskqueue.rs
  batches.py    scheduler/batches.rs
  lp.py         solver/{mod,highs}.rs
  gap.py        scheduler/gap.rs
  solver.py     scheduler/solver.rs
  mapping.py    scheduler/mapping.rs
  core.py       server/{core,reactor,task}.rs (only the parts that feed the tick), scheduler/{main,state}.rs
  judge.py      the stand-alone feasibility judge (server/worker.rs:236-271 sanity_check replay)
"""
