"""tests/test_gpu_paths.py must keep one case per reachable (solve loop, RT, amount width) cell and per extra path
(class table in global memory, packing on and off, minimum-utilisation restart).  Runs without a GPU."""
import test_gpu_paths as T


def test_every_reachable_solver_path_cell_has_a_case():
    cells = T.reachable_cells()
    assert len(cells) == 4 * 3 * 2 - 1                       # the wide loop cannot hold RT 16 on u64 amounts
    assert ("wide", 16, "u64") not in cells
    missing = [c for c in list(cells) + list(T.EXTRA_CELLS) if c not in T.CASES]
    assert not missing, missing


def test_path_cases_name_their_loop():
    for key, (_, flags, _, must, must_not, loops) in T.CASES.items():
        if isinstance(key, tuple):
            assert loops == T.LOOPS[key[0]], key
            assert bool(flags & T.L.HQS_CREATE_WIDE_AMOUNTS) == (key[2] == "u64"), key
        assert must & must_not == 0, key
