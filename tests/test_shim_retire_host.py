"""Host logic of the C++ shim's handle retirement (tako_b200::GpuCore::retire_handles) without a GPU: the shim's sources,
tako_shim_retire.cpp included, are compiled against the test double of the C ABI with its compaction call
(tests/mock/fake_hqsched_retire.cpp, on top of fake_hqsched_graph_cancel.cpp) and driven through
tests/mock/shim_retire_host_test.cpp.  The real library is exercised by the same shim on the GPU
(tests/test_gpu_handle_compact.py::test_cpp_shim_retire_selftest)."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_shim_retire_against_the_abi_double(tmp_path):
    exe = str(tmp_path / "shim_retire_host_test")
    srcs = [os.path.join(ROOT, "tests", "mock", "shim_retire_host_test.cpp"),
            os.path.join(ROOT, "hyperqueue_b200", "csrc", "tako_shim.cpp"),
            os.path.join(ROOT, "hyperqueue_b200", "csrc", "tako_shim_graph.cpp"),
            os.path.join(ROOT, "hyperqueue_b200", "csrc", "tako_shim_graph_cancel.cpp"),
            os.path.join(ROOT, "hyperqueue_b200", "csrc", "tako_shim_retire.cpp"),
            os.path.join(ROOT, "tests", "mock", "fake_hqsched_retire.cpp")]
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-o", exe] + srcs, check=True, cwd=ROOT)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
