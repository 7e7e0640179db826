"""CPU: the sentence splitter (Kiwi::splitIntoSents, src/Kiwi.cpp:417-450) without a GPU, against the unmodified reference's vectors
over the documents of tests/golden/docs_sents.jsonl (Knlm and CoNg models):
  1. the shared rule core (kiwi_b200/csrc/sentences.h) on the reference's own tokenizedResultOut tokens gives the reference's ranges;
  2. sents.cu - the device source - on a simulated 32-lane warp gives them from the reference's token rows, and a sample of short
     documents goes through the whole simulated pipeline (lattice -> Viterbi -> emit -> sents);
  3. the C ABI exports the new symbols and keeps the reference's handle / index error convention."""
import ctypes as C, os, subprocess
import numpy as np
import pytest
from tests.orc import IMAGE, CONG_IMAGE
from tests.sentsio import read_docs, read_sents_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HS = os.path.join(ROOT, "tests", "hostsim")
OBJS = ["lattice.o", "viterbi.o", "viterbi_cong.o", "viterbi_sbg.o", "emit.o", "model.o"]
MATCH_ALL_WITH_NORMALIZING = (1 << 0) | (1 << 1) | (1 << 2) | (1 << 3) | (1 << 4) | (1 << 5) | (1 << 23) | (1 << 16)
OWN_TAGS = set(range(21, 39)) | {0}      # sf..w_emoji and unknown: tokens that carry their own surface form


def u16(text):
    return np.ascontiguousarray(np.frombuffer(text.encode("utf-16-le", "surrogatepass"), dtype="<u2"))


@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    """tests/hostsim/sents_sim32.cpp + pipeline_sim32.cpp + sents.cu (as C++) over the simulator objects the build leaves in tests/hostsim/obj32"""
    objs = [os.path.join(HS, "obj32", o) for o in OBJS]
    if not all(os.path.exists(o) for o in objs):
        pytest.skip("tests/hostsim/obj32 missing: run __graft_entry__.build()")
    lib = str(tmp_path_factory.mktemp("sents_sim") / "libsents_sim32.so")
    cmd = [os.environ.get("CXX", "g++"), "-std=c++20", "-O1", "-ffp-contract=off", "-fPIC", "-DKB_HOSTSIM=32", "-I" + os.path.join(HS, "shim32"),
           "-I" + os.path.join(ROOT, "include"), "-shared", "-o", lib, os.path.join(HS, "sents_sim32.cpp"), os.path.join(HS, "pipeline_sim32.cpp"),
           "-x", "c++", os.path.join(ROOT, "kiwi_b200", "csrc", "sents.cu"), "-x", "none"] + objs + ["-lpthread"]
    subprocess.run(cmd, check=True)
    L = C.CDLL(lib)
    L.ss_core_ranges.argtypes = [C.c_int] + [C.c_void_p] * 7 + [C.c_uint32, C.c_void_p]
    L.ss32_open.restype = C.c_void_p; L.ss32_open.argtypes = [C.c_char_p]
    L.ss32_close.argtypes = [C.c_void_p]
    L.ss32_rows.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_int] + [C.c_void_p] * 6
    L.hs32_open.restype = C.c_void_p; L.hs32_open.argtypes = [C.c_char_p]
    L.hs32_close.argtypes = [C.c_void_p]
    L.hs32_analyze.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_uint32] + [C.c_void_p] * 5 + [C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_int), C.c_void_p]
    return L


def core_ranges(L, text, gold):
    toks, forms = gold["tokens"], gold["forms"]
    n = len(toks)
    units = u16(text)
    pos = np.array([t[2] for t in toks], np.uint32); ln = np.array([t[3] for t in toks], np.uint32); tag = np.array([t[1] for t in toks], np.uint8)
    fu = [u16(f[1]) for f in forms]
    off = np.zeros(n + 1, np.uint32); off[1:] = np.cumsum([len(x) for x in fu])
    blob = np.ascontiguousarray(np.concatenate(fu + [np.zeros(1, "<u2")]))
    is_yo = np.array([1 if f[1] == "요" else 0 for f in forms] + [0], np.uint8)
    out = np.zeros(2 * n + 2, np.uint32)
    k = L.ss_core_ranges(n, pos.ctypes.data, ln.ctypes.data, tag.ctypes.data, blob.ctypes.data, off.ctypes.data, is_yo.ctypes.data,
                         units.ctypes.data if len(units) else None, len(units), out.ctypes.data)
    return [(int(out[2 * i]), int(out[2 * i + 1])) for i in range(k)]


def sim_ranges(L, h, text, morph, tag, pos, ln, flags):
    units = u16(text)
    n = len(morph)
    out = np.zeros(2 * n + 2, np.uint32)
    arrs = [np.ascontiguousarray(a) for a in (morph, tag, pos, ln, flags)]
    k = L.ss32_rows(h, units.ctypes.data if len(units) else None, len(units), n, *[a.ctypes.data for a in arrs], out.ctypes.data)
    assert k >= 0, text
    return [(int(out[2 * i]), int(out[2 * i + 1])) for i in range(k)]


def rows_of(gold):
    """the reference's tokens as emit_kernel rows: own-substring flag on the symbol / foreign / unknown tags (their form is the text)"""
    toks = gold["tokens"]
    morph = np.array([t[0] if t[0] != 0xFFFFFFFF else 0 for t in toks], np.uint32)
    tag = np.array([t[1] for t in toks], np.uint8); pos = np.array([t[2] for t in toks], np.uint32); ln = np.array([t[3] for t in toks], np.uint16)
    flags = np.array([1 if ((t[1] & 0x7F) in OWN_TAGS or t[0] == 0xFFFFFFFF) else 0 for t in toks], np.uint8)
    return morph, tag, pos, ln, flags


def test_fixture_covers_the_document_shapes():
    docs = read_docs()
    assert len(docs) >= 400
    for needle in ["\r\n", "\n\n", "\v", "\f", " ", '"', "(", "①", "(가)", "요", "ㅋ", "2024.01.02.", "https://", "@", "😀", "𠀀"]:
        assert any(needle in d for d in docs), needle
    assert "" in docs and any(d and not d.strip() for d in docs)
    assert sum(len(d.encode("utf-16-le")) // 2 >= 2000 for d in docs) >= 3


def test_vectors_belong_to_the_committed_images():
    """docs_sents.MANIFEST.json (tests/golden/make_docs.py --golden): the vector files are the ones it names, made with the model images
    of tests/golden/MANIFEST.json"""
    import gzip, hashlib, json
    golden = os.path.join(ROOT, "tests", "golden")
    m = json.load(open(os.path.join(golden, "docs_sents.MANIFEST.json")))
    images = json.load(open(os.path.join(golden, "MANIFEST.json")))
    for prefix in ("", "cong_"):
        assert m[prefix + "image_md5"] == images[prefix + "image_md5"], prefix
        data = gzip.open(os.path.join(golden, prefix + "docs_sents.golden.txt.gz"), "rb").read()
        assert hashlib.md5(data).hexdigest() == m["files"][prefix + "docs_sents"]["md5"], prefix


@pytest.mark.parametrize("prefix", ["", "cong_"])
def test_core_reproduces_reference_ranges(sim, prefix):
    docs, gold = read_docs(), read_sents_golden(prefix)
    assert len(gold) == len(docs)
    for i, (d, g) in enumerate(zip(docs, gold)):
        assert core_ranges(sim, d, g) == g["ranges"], (prefix, i, d[:80])


@pytest.mark.parametrize("prefix,image", [("", IMAGE), ("cong_", CONG_IMAGE)])
def test_simulated_kernel_reproduces_reference_ranges(sim, prefix, image):
    if not os.path.exists(image):
        pytest.skip("model image missing: run __graft_entry__.build()")
    h = sim.ss32_open(os.fsencode(image))
    assert h
    try:
        docs, gold = read_docs(), read_sents_golden(prefix)
        for i, (d, g) in enumerate(zip(docs, gold)):
            assert sim_ranges(sim, h, d, *rows_of(g)) == g["ranges"], (prefix, i, d[:80])
    finally:
        sim.ss32_close(h)


def test_simulated_pipeline_splits_like_reference(sim):
    """short documents through lattice -> Viterbi -> emit -> sents, all simulated: tokens and ranges of the reference"""
    docs, gold = read_docs(), read_sents_golden("")
    sample = [i for i, d in enumerate(docs) if 0 < len(d) <= 48][:24]
    assert len(sample) >= 12
    hs = sim.hs32_open(os.fsencode(IMAGE)); ss = sim.ss32_open(os.fsencode(IMAGE))
    assert hs and ss
    cap = 4096
    morph = np.zeros(cap, np.uint32); tag = np.zeros(cap, np.uint8); pos = np.zeros(cap, np.uint32); ln = np.zeros(cap, np.uint16)
    sc = np.zeros(cap, np.float32); fl = np.zeros(cap, np.uint8)
    try:
        for i in sample:
            units = u16(docs[i])
            s = C.c_float(0); nn = C.c_int(0)
            n = sim.hs32_analyze(hs, units.ctypes.data, len(units), MATCH_ALL_WITH_NORMALIZING, morph.ctypes.data, tag.ctypes.data, pos.ctypes.data,
                                 ln.ctypes.data, sc.ctypes.data, cap, C.byref(s), C.byref(nn), fl.ctypes.data)
            assert n >= 0, (i, docs[i])
            assert [(int(morph[k]), int(tag[k]), int(pos[k]), int(ln[k])) for k in range(n)] == [t[:4] for t in gold[i]["tokens"]], (i, docs[i])
            assert sim_ranges(sim, ss, docs[i], morph[:n], tag[:n], pos[:n], ln[:n], fl[:n]) == gold[i]["ranges"], (i, docs[i])
    finally:
        sim.hs32_close(hs); sim.ss32_close(ss)


def test_split_symbols_and_error_convention():
    import kiwi_b200
    lib = kiwi_b200.load_library()
    for n in ["kiwi_split_into_sents_w", "kiwi_split_into_sents", "kiwi_ss_size", "kiwi_ss_begin_position", "kiwi_ss_end_position",
              "kiwi_ss_close", "kiwi_b200_split_batch", "kiwi_b200_sents_free"]:
        assert hasattr(lib, n), n
    text = u16("문장이다.\0")
    assert not lib.kiwi_split_into_sents_w(None, text.ctypes.data, MATCH_ALL_WITH_NORMALIZING, None)
    assert not lib.kiwi_split_into_sents(None, "문장이다.".encode(), MATCH_ALL_WITH_NORMALIZING, None)
    assert lib.kiwi_ss_size(None) == -2 and lib.kiwi_ss_begin_position(None, 0) == -2 and lib.kiwi_ss_end_position(None, 0) == -2
    assert lib.kiwi_ss_close(None) == -2
    lib.kiwi_clear_error()
    off = np.array([0, len(text) - 1], np.uint32)
    assert not lib.kiwi_b200_split_batch(None, text.ctypes.data, off.ctypes.data, 1, MATCH_ALL_WITH_NORMALIZING)
    assert lib.kiwi_error() == b"invalid handle"
    lib.kiwi_b200_sents_free(None)
