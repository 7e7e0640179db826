"""CPU: native readers of the reference's language-model files (kiwi_b200/csrc/native_lm.cpp, exported as kiwi_b200_native_knlm /
kiwi_b200_native_sbg / kiwi_b200_native_cong; SURVEY 8f-2, first pieces of a loader that does not link the reference).  tests/native/native_lm_check.cpp
compares their output with the Knlm / SkipBigram / CoNg sections of the model images that flatten_model dumped from the reference's own
in-memory models: every section byte for byte, and the scalars the reference computes at load time (suffix links, BOS state, unk_ll)."""
import os, subprocess
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODELS = os.path.join(ROOT, "oracle", "_ref", "models")


def test_native_knlm_and_sbg_sections_equal_the_flattened_image(tmp_path):
    lib = os.path.join(ROOT, "kiwi_b200", "libkiwi_b200.so")
    knlm_img = os.path.join(MODELS, "knlm_small.img"); knlm_file = os.path.join(MODELS, "knlm_small", "sj.knlm")
    if not (os.path.exists(lib) and os.path.exists(knlm_img) and os.path.exists(knlm_file)):
        pytest.skip("library, model image or the reference-format model directory missing: run __graft_entry__.build()")
    exe = str(tmp_path / "kb_native_lm_check")
    subprocess.run(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "native", "native_lm_check.cpp"), "-ldl"], check=True)
    args = [exe, lib, knlm_img, knlm_file]
    sbg_img = os.path.join(MODELS, "sbg_small.img"); sbg_file = os.path.join(MODELS, "sbg_small", "skipbigram.mdl")
    args += [sbg_img, sbg_file] if os.path.exists(sbg_img) and os.path.exists(sbg_file) else ["-", "-"]
    cong_img = os.path.join(MODELS, "cong_small.img"); cong_file = os.path.join(MODELS, "cong_small", "cong.mdl")
    args += [cong_img, cong_file] if os.path.exists(cong_img) and os.path.exists(cong_file) else ["-", "-"]
    out = subprocess.run(args, capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "mismatching sections 0" in out.stdout, out.stdout + out.stderr
    assert "KN_NODES" in out.stdout and "knlm scalars identical" in out.stdout
    if os.path.exists(cong_file): assert "CG_OUT_EMB" in out.stdout and "cong scalars identical" in out.stdout


def test_native_reader_rejects_damaged_files(tmp_path):
    import ctypes as C
    lib = os.path.join(ROOT, "kiwi_b200", "libkiwi_b200.so")
    knlm_file = os.path.join(MODELS, "knlm_small", "sj.knlm")
    if not (os.path.exists(lib) and os.path.exists(knlm_file)):
        pytest.skip("library or model file missing")
    L = C.CDLL(lib)
    L.kiwi_b200_native_knlm.argtypes = [C.c_char_p, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
    L.kiwi_b200_native_error.restype = C.c_char_p
    data = open(knlm_file, "rb").read()
    for name, blob in [("truncated", data[:len(data) // 2]), ("tiny", data[:40]), ("offsets", data[:8] + b"\xff" * 8 + data[16:])]:
        p = tmp_path / (name + ".knlm"); p.write_bytes(blob)
        out = C.c_void_p(); size = C.c_uint64()
        assert L.kiwi_b200_native_knlm(os.fsencode(str(p)), C.byref(out), C.byref(size)) == -1, name
        assert L.kiwi_b200_native_error()
    out = C.c_void_p(); size = C.c_uint64()
    assert L.kiwi_b200_native_knlm(b"/nonexistent/sj.knlm", C.byref(out), C.byref(size)) == -1
