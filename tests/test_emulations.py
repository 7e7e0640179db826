"""CPU: the two libstdc++ behaviours that are part of the reference's RESULT and that the kernels therefore restate on the device:
  * std::sort is not stable: which of several equal-score end-node candidates comes first (PathEvaluator.hpp:1359-1368) decides the
    emitted morpheme id -> kiwi_b200/csrc/std_sort_emu.h;
  * the `top1` container (> 512 incoming paths) is an std::unordered_set that is written out in iteration order
    (BestPathContainer.hpp:229-276) -> kiwi_b200/csrc/unordered_emu.h.
tests/native/emu_check.cpp compares both restatements with the real library on random inputs (many ties / collisions, re-used sets,
median-of-3 killer sequences); it is compiled here with g++ (libstdc++ is the library the reference is built against)."""
import os, subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_std_sort_and_unordered_set_restatements_match_libstdcxx(tmp_path):
    exe = str(tmp_path / "kb_emu_check")
    subprocess.run(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "native", "emu_check.cpp")], check=True)
    out = subprocess.run([exe, "1"], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "mismatching 0" in out.stdout, out.stdout


def test_skipbigram_float_restatement_matches_the_c_library(tmp_path):
    """kiwi_b200/csrc/sbg_math.h (the SkipBigram logSumExp as the device computes it): its logf against glibc's for every float in
    [1, 16], its logSumExp16 against the reference's operation order with the library logf on 2 M random score arrays - bit for bit."""
    exe = str(tmp_path / "kb_sbg_math_check")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-o", exe, os.path.join(ROOT, "tests", "native", "sbg_math_check.cpp")], check=True)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "mismatches 0" in out.stdout, out.stdout
