"""CPU: the model loader resolves the suffix walk after every leaf edge of the Knlm and CoNg tries once, and stores the resulting state in
the edge's table entry (kiwi_b200/csrc/lm_tables.h), so the Viterbi kernels never walk suffixes.  tests/native/lm_leaf_check.cpp builds
those tables from the fabricated model images and checks every entry against the LM step of the oracle restatement, which walks the
suffix chain as the reference does: the state after each leaf edge, and the child's ll / context id on each inner edge."""
import os, subprocess
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODELS = os.path.join(ROOT, "oracle", "_ref", "models")


def test_stored_leaf_states_match_the_suffix_walk(tmp_path):
    knlm_img = os.path.join(MODELS, "knlm_small.img"); cong_img = os.path.join(MODELS, "cong_small.img")
    if not (os.path.exists(knlm_img) and os.path.exists(cong_img)):
        pytest.skip("model images missing: run __graft_entry__.build()")
    exe = str(tmp_path / "kb_lm_leaf_check")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    subprocess.run(["g++", "-O2", "-std=c++17", "-I" + os.path.join(cuda, "include"), "-o", exe,
                    os.path.join(ROOT, "tests", "native", "lm_leaf_check.cpp")], check=True)
    out = subprocess.run([exe, knlm_img, cong_img], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "knlm:" in out.stdout and "cong:" in out.stdout and out.stdout.count(" 0 mismatches") == 2, out.stdout
