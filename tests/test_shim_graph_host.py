"""Host logic of the C++ shim's task graphs (tako_b200::GpuCore::on_new_tasks with dependencies) without a GPU: tako_shim.cpp
and tako_shim_graph.cpp are compiled against the test double of the C ABI with its graph calls
(tests/mock/fake_hqsched_graph.cpp, which builds on tests/mock/fake_hqsched.cpp) and driven through dependency resolution,
the batched graph push, releases through hqs_graph_finished and cancellation (tests/mock/shim_graph_host_test.cpp).  The
real library is exercised by the same shim on the GPU (tests/test_gpu_graph.py::test_cpp_shim_graph_selftest)."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_shim_graph_bookkeeping_against_the_abi_double(tmp_path):
    exe = str(tmp_path / "shim_graph_host_test")
    srcs = [os.path.join(ROOT, "tests", "mock", "shim_graph_host_test.cpp"),
            os.path.join(ROOT, "hyperqueue_b200", "csrc", "tako_shim.cpp"),
            os.path.join(ROOT, "hyperqueue_b200", "csrc", "tako_shim_graph.cpp"),
            os.path.join(ROOT, "tests", "mock", "fake_hqsched_graph.cpp")]
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-o", exe] + srcs, check=True, cwd=ROOT)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
