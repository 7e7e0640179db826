"""CPU: the token-joining match options (joinAffixTokens, src/Kiwi.cpp:495-588; KIWI_MATCH_JOIN_*, MERGE_SAISIOT, JOIN_PARTICLE_YO and
COMPATIBLE_JAMO) without a GPU, against the unmodified reference's join vectors (tests/golden/make_join.py, sets in tests/joinio.py):
every sentence goes through the simulated lattice -> Viterbi -> emit_join_kernel (the device sources on 32-lane warps) and the product's
host assembly, and must give the reference's morpheme ids (-1 for a joined token), tags, positions, lengths, forms, sentence fields and
scores exactly."""
import ctypes as C, gzip, hashlib, json, os, subprocess
import numpy as np
import pytest
from tests.goldenio import read_golden, read_inputs
from tests.joinio import SETS, RULES, read_manifest, rule_counts
from tests.orc import IMAGE, CONG_IMAGE, TYPO_IMAGES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HS = os.path.join(ROOT, "tests", "hostsim")
OBJS = ["lattice.o", "viterbi.o", "viterbi_cong.o", "viterbi_sbg.o", "emit.o", "model.o"]
GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    """tests/hostsim/join_sim32.cpp over the simulator objects the build leaves in tests/hostsim/obj32"""
    objs = [os.path.join(HS, "obj32", o) for o in OBJS]
    if not all(os.path.exists(o) for o in objs):
        pytest.skip("tests/hostsim/obj32 missing: run __graft_entry__.build()")
    lib = str(tmp_path_factory.mktemp("join_sim") / "libjoin_sim32.so")
    cmd = [os.environ.get("CXX", "g++"), "-std=c++20", "-O1", "-ffp-contract=off", "-fPIC", "-DKB_HOSTSIM=32", "-I" + os.path.join(HS, "shim32"),
           "-I" + os.path.join(ROOT, "include"), "-shared", "-o", lib, os.path.join(HS, "join_sim32.cpp")] + objs + ["-lpthread"]
    subprocess.run(cmd, check=True)
    L = C.CDLL(lib)
    L.hj32_open.restype = C.c_void_p; L.hj32_open.argtypes = [C.c_char_p, C.c_char_p]
    L.hj32_close.argtypes = [C.c_void_p]
    L.hj32_analyze.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_uint32, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_float)]
    return L


def test_join_vectors_belong_to_the_committed_images():
    m = read_manifest()
    images = json.load(open(os.path.join(GOLDEN, "MANIFEST.json")))
    for key in ("image_md5", "cong_image_md5", "typo_basic_image_md5"):
        assert m[key] == images[key], key
    assert set(m["files"]) == set(SETS)
    for name, (opts, *_rest) in SETS.items():
        data = gzip.open(os.path.join(GOLDEN, name + ".golden.txt.gz"), "rb").read()
        assert hashlib.md5(data).hexdigest() == m["files"][name]["md5"], name
        assert m["files"][name]["match"] == opts, name


def test_every_rule_fires_in_the_vectors():
    """the per-rule counts of the manifest are those of the committed vectors, and every rule fired at least once"""
    m = read_manifest()["rule_counts"]
    total = dict.fromkeys(RULES, 0)
    for name in SETS:
        c = rule_counts(name)
        assert c == m[name], name
        for r in RULES: total[r] += c[r]
    assert total == m["total"]
    assert all(total[r] > 0 for r in RULES), total


def _u16(text):
    return np.ascontiguousarray(np.frombuffer(text.encode("utf-16-le", "surrogatepass"), dtype="<u2"))


@pytest.mark.parametrize("name", sorted(SETS))
def test_simulated_join_matches_reference(sim, name):
    opts, mtype, typo, inputs, _ = SETS[name]
    image = CONG_IMAGE if mtype == "cong" else IMAGE
    typo_path = TYPO_IMAGES[typo] if typo else None
    if not os.path.exists(image) or (typo_path and not os.path.exists(typo_path)):
        pytest.skip("model image missing: run __graft_entry__.build()")
    h = sim.hj32_open(os.fsencode(image), os.fsencode(typo_path) if typo_path else None)
    assert h
    cap = 8192
    rows = np.zeros(10 * cap, np.uint32); blob = np.zeros(4 * cap, np.uint16); off = np.zeros(cap + 1, np.uint32)
    try:
        texts, gold = read_inputs(inputs), read_golden(name)
        assert len(gold) == len(texts) and gold
        for i, (t, g) in enumerate(zip(texts, gold)):
            u = _u16(t)
            s = C.c_float(0)
            n = sim.hj32_analyze(h, u.ctypes.data if len(u) else None, len(u), opts, rows.ctypes.data, cap, blob.ctypes.data, off.ctypes.data, len(blob), C.byref(s))
            assert n >= 0, (name, i, n, t)
            r = rows[:10 * n].reshape(n, 10).astype(np.int64)
            got = [(int(x[0]) & 0xFFFFFFFF, int(x[1]), int(x[2]), int(x[3])) for x in r]
            assert got == [x[:4] for x in g["tokens"]], (name, i, t)
            assert [np.float32(v) for v in r[:, 4].astype(np.uint32).view(np.float32)] == [np.float32(x[4]) for x in g["tokens"]], (name, i, t)
            fields = [(int(x[5]), int(x[6]), int(x[7]), int(x[8]), int(np.int32(np.uint32(x[9])))) for x in r]
            assert fields == [f[0] for f in g.get("forms", [])], (name, i, t)
            forms = [blob[off[k]:off[k + 1]].tobytes().decode("utf-16-le", "replace") for k in range(n)]
            assert forms == [f[1] for f in g.get("forms", [])], (name, i, t)
            assert np.float32(s.value) == np.float32(g["score"]), (name, i, t)
    finally:
        sim.hj32_close(h)
