"""The narrow solver divides by an invariant amount with a magic number that hqs_classes_set derives on the host
(pack_var32 in hyperqueue_b200/csrc/hqs_solver.cuh).  This compiles tests/cuda/div_magic_check.cpp against the
library's own packing code and replays the device arithmetic on the CPU: every d < 2^20, every 2^l + delta
(|delta| <= 3) and 10^7 random d < 2^31, each at the numerators where a wrong magic or shift shows first."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_pack_var32_magic_divides_exactly(tmp_path):
    exe = str(tmp_path / "div_magic_check")
    subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-o", exe, os.path.join(ROOT, "tests", "cuda", "div_magic_check.cpp")],
                   check=True)
    res = subprocess.run([exe, "10000000"], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    checks = int(res.stdout.split()[-3])
    assert checks >= 6 * (10_000_000 + (1 << 20) - 1), res.stdout
