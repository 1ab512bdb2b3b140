"""CPU-only checks of the drop-in boundary: the C-ABI library loads, exports every symbol that
include/hqsched.h declares, struct layouts match the header, and — with no CUDA device — fails loudly
instead of falling back to a CPU path."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    from hyperqueue_b200 import _lib
    return _lib.load_library()


def test_header_symbols_exported(lib):
    hdr = open(os.path.join(ROOT, "include", "hqsched.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(hqs_[a-z_]+)\s*\(", hdr))
    assert len(declared) >= 18
    from hyperqueue_b200 import _lib
    assert declared == set(_lib.ABI_SYMBOLS)
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.hqs_abi_version() == 1


def test_struct_layouts():
    from hyperqueue_b200 import _lib
    assert C.sizeof(_lib.hqs_variant) == 16 * 8 + 16
    assert C.sizeof(_lib.hqs_class) == 8 + 8 * C.sizeof(_lib.hqs_variant)
    assert C.sizeof(_lib.hqs_worker) == 24 == _lib.worker_dtype.itemsize
    assert _lib.assignment_dtype.itemsize == 8
    assert _lib.assignment_dtype.fields["worker"][1] == 4 and _lib.assignment_dtype.fields["variant"][1] == 6


def test_no_cpu_fallback(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    ctx = C.c_void_p()
    rc = lib.hqs_create(C.byref(ctx), 0, 4, 0)
    assert rc == -2 and not ctx.value                       # HQS_E_CUDA
    assert b"no CPU fallback" in lib.hqs_last_error(None)
    from hyperqueue_b200 import GpuScheduler, HqsError
    with pytest.raises(HqsError):
        GpuScheduler(4)


def test_product_does_not_import_oracle():
    """The product path may not import, link or execute anything under oracle/ (or the test-only model)."""
    pkg = os.path.join(ROOT, "hyperqueue_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            src = open(os.path.join(dirpath, f), errors="ignore").read() if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp", ".hpp")) else ""
            if f.endswith(".py"):
                assert not re.search(r"^\s*(import|from)\s+(oracle|greedy_model|parity)\b", src, flags=re.M), f
            if f.endswith((".cu", ".cuh", ".h", ".cpp", ".hpp")):
                assert not re.search(r"#include\s+[\"<][^\">]*oracle", src), f
    so = os.path.join(pkg, "libhqsched_b200.so")
    out = __import__("subprocess").run(["ldd", so], capture_output=True, text=True).stdout
    assert "hqjudge" not in out and "oracle" not in out


def test_priority_mapping_matches_oracle():
    from hyperqueue_b200 import priority_from_user
    from oracle.model import priority_from_user as ref
    ups = np.array([-2**31, -5, -1, 0, 1, 7, 123, 2**31 - 1])
    got = priority_from_user(ups)
    assert [int(x) for x in got] == [ref(int(u)) for u in ups]
    assert (np.diff(got.astype(np.float64)) > 0).all()


def test_cpp_shim_builds_and_exports_the_reference_interface(lib):
    """The host side above the C ABI is C++ (the reference's is Rust): libhqtako_shim.so links against the C-ABI
    library only and exports tako_b200::GpuCore with the reference's operation names."""
    import subprocess
    from hyperqueue_b200 import _lib
    shim = _lib.load_shim()
    assert hasattr(shim, "hqshim_selftest")
    syms = subprocess.run(["nm", "-DC", _lib.SHIM_PATH], capture_output=True, text=True).stdout
    for name in ("tako_b200::GpuCore::get_or_create_resource_rq_id", "tako_b200::GpuCore::on_new_worker",
                 "tako_b200::GpuCore::add_ready_task", "tako_b200::GpuCore::remove_ready_task",
                 "tako_b200::GpuCore::run_scheduling", "tako_b200::GpuCore::on_task_finished",
                 "tako_b200::GpuCore::block_request"):
        assert name in syms, name
    ldd = subprocess.run(["ldd", _lib.SHIM_PATH], capture_output=True, text=True).stdout
    assert "libhqsched_b200.so" in ldd and "hqjudge" not in ldd
    import torch
    if not torch.cuda.is_available():
        # no device: the shim fails loudly (exception caught by the self-test => one failed check), no CPU path
        assert shim.hqshim_selftest(0, 0) >= 1


def test_solver_shared_memory_budget(lib):
    """The solver CTA's dynamic shared memory may be min(227 KB - the kernel's static shared memory, 216 KB) (hqs_create).
    Its mandatory arrays without the group list, which moves to global memory when it does not fit next to them, must fit
    that budget at every corner of the documented limits (HQS_MAX_WORKERS, 16 resource slots, u32 / u64 amounts, proactive
    filling on / off, HQS_MAX_CLASSES, HQS_MAX_GROUPS), or a tick there fails with HQS_E_LIMIT on every call."""
    import subprocess
    from hyperqueue_b200 import _lib
    out = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True).stdout
    statics = [int(m) for blk in re.findall(r"Function [^\n]*tick_k[^\n]*\n[^\n]*", out) for m in re.findall(r"SHARED:(\d+)", blk)]
    assert len(statics) == 6
    budget = min(227 * 1024 - max(statics), 216 * 1024)
    assert budget == 216 * 1024                      # tests/test_gpu_smem_layout.py predicts the layout with this budget
    up = lambda n: (n + 15) & ~15                    # solver_layout aligns every array to 16 bytes
    for W in (1, 1024):
        for RT in (4, 8, 16):
            for at in (4, 8):
                for pf in (0, 1):
                    for Q in (1, _lib.HQS_MAX_CLASSES):
                        # free amounts [W][RT]; unt, remtime, excl, touch, td per worker; frontier, noresv per class;
                        # with proactive filling top and pflvl per class
                        need = sum(up(b) for b in (W * RT * at, W * 4, W * 8, W, W, W * 2, Q * 2, Q))
                        need += 2 * up(Q * 4) if pf else 0
                        assert need <= budget, (W, RT, at, pf, Q, need, budget)
    # worst corner: 1024 workers x 16 slots x u64, proactive filling, 4096 classes
    assert need == 192_512
    # the emit step of the worker CTAs: <= 128 KB of counters (+ the group records when they fit) + the segment cache
    assert 128 * 1024 + 8 * 1024 <= budget
