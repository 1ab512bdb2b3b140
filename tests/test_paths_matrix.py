"""tests/test_gpu_paths.py must keep one case per reachable (solve loop, RT, amount width) cell and per extra path
(class table in global memory, packing on and off, minimum-utilisation restart); tests/test_gpu_smem_layout.py one case per
array the solver layout can leave in global memory.  Runs without a GPU."""
import test_gpu_paths as T


def test_every_reachable_solver_path_cell_has_a_case():
    cells = T.reachable_cells()
    assert len(cells) == 4 * 3 * 2 - 1                       # the wide loop cannot hold RT 16 on u64 amounts
    assert ("wide", 16, "u64") not in cells
    missing = [c for c in list(cells) + list(T.EXTRA_CELLS) if c not in T.CASES]
    assert not missing, missing


def test_every_spill_bit_has_a_layout_case():
    """tests/test_gpu_smem_layout.py keeps a case for every array the solver layout can leave in global memory."""
    import test_gpu_smem_layout as S
    spill = (T.L.HQS_PATH_GROUPS_GLOBAL, T.L.HQS_PATH_REM_GLOBAL, T.L.HQS_PATH_BLOCKED_GLOBAL, T.L.HQS_PATH_COUNTS_GLOBAL)
    for bit in spill:
        assert any(must & bit for must in S.CASES.values()), hex(bit)
    assert all(hasattr(S, "test_" + name) for name in S.CASES), sorted(S.CASES)
    # the worst corner with the group list in global memory fits the budget; the refused corners need the fallback
    assert S.mandatory_bytes(1024, 16, 8, 4096, 1, 1, groups=False) == 192_512 <= S.BUDGET
    for W, RT, Q, L_, pf, need in [(1024, 16, 2, 4096, 0, 245_792), (1024, 16, 4096, 2, 0, 258_048),
                                   (1024, 16, 2, 2048, 1, 278_592), (512, 16, 4096, 1, 1, 249_856)]:
        assert S.mandatory_bytes(W, RT, 8, Q, L_, pf) == need > S.BUDGET


def test_path_cases_name_their_loop():
    for key, (_, flags, _, must, must_not, loops) in T.CASES.items():
        if isinstance(key, tuple):
            assert loops == T.LOOPS[key[0]], key
            assert bool(flags & T.L.HQS_CREATE_WIDE_AMOUNTS) == (key[2] == "u64"), key
        assert must & must_not == 0, key
