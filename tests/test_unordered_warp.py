"""CPU: the warp-parallel write-out order of the `top1` container (kb::unorderedSetOrderWarp in kiwi_b200/csrc/unordered_emu.h, called
by the Viterbi kernels' reorderTop1) against libstdc++'s std::unordered_set and the sequential restatement kb::unorderedSetOrder.
tests/native/emu_warp_check.cpp runs it on the 32-lane host simulation of a warp (tests/hostsim/shim32), compiled here with g++."""
import os, subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_warp_unordered_set_order_matches_libstdcxx(tmp_path):
    exe = str(tmp_path / "kb_emu_warp_check")
    subprocess.run(["g++", "-O2", "-std=c++17", "-DKB_HOSTSIM=32", "-I", os.path.join(ROOT, "tests", "hostsim", "shim32"), "-o", exe,
                    os.path.join(ROOT, "tests", "native", "emu_warp_check.cpp"), "-ldl"], check=True)
    out = subprocess.run([exe, "5"], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "mismatching 0" in out.stdout, out.stdout
