"""GPU: the token-joining match options through the C ABI (kiwi_b200_analyze_batch, kiwi_analyze_w) against the unmodified reference's join
vectors (tests/golden/make_join.py; sets in tests/joinio.py), through the retry arena, several passes and a two-engine handle, and without
join options on the same handle before and after (rows unchanged, no form array)."""
import ctypes as C
import os
import subprocess
import sys
import numpy as np
import pytest
import kiwi_b200
from tests.goldenio import read_golden, read_inputs
from tests.joinio import SETS, J1, J2
from tests.orc import IMAGE, CONG_IMAGE, TYPO_IMAGES

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M = kiwi_b200.MATCH_ALL_WITH_NORMALIZING
HEAVY = ". ".join(["다" * 100] * 30) + "."      # (its paths overflow the first arena: retried)


class TokenInfo(C.Structure):      # kiwi_token_info_t
    _fields_ = [("chr_position", C.c_uint32), ("word_position", C.c_uint32), ("sent_position", C.c_uint32), ("line_number", C.c_uint32),
                ("length", C.c_uint16), ("tag", C.c_uint8), ("sense_id", C.c_uint8), ("score", C.c_float), ("typo_cost", C.c_float),
                ("typo_form_id", C.c_uint32), ("paired_token", C.c_uint32), ("sub_sent_position", C.c_uint32), ("dialect", C.c_uint16)]


def _close(a, b):
    return abs(a - b) <= 1e-4 * max(1.0, abs(b))


@pytest.fixture(scope="module")
def typo():
    if not os.path.exists(TYPO_IMAGES["basic"]):
        pytest.skip("typo image missing")
    t = kiwi_b200.PreparedTypo(path=TYPO_IMAGES["basic"])
    yield t
    t.close()


def rows_of(r, i):
    """sentence i of a BatchResult as (morph id or -1, tag, position, length, score, form of a joined token or None)"""
    out = []
    for k, t in enumerate(r.sentence(i)):
        j = r.joined_form(i, k)
        out.append((-1 if j else int(t["morph_id"]), int(t["tag"]), int(t["position"]), int(t["length"]), float(t["score"]), j[0] if j else None))
    return out


def check_rows(got, g, where):
    want = [(x[0] if x[0] != 0xFFFFFFFF else -1, x[1], x[2], x[3]) for x in g["tokens"]]
    assert [x[:4] for x in got] == want, where
    assert all(_close(a[4], b[4]) for a, b in zip(got, g["tokens"])), where
    forms = [f[1] for f in g.get("forms", [])]
    assert [x[5] for x in got if x[0] == -1] == [f for f, x in zip(forms, want) if x[0] == -1], where


@pytest.mark.parametrize("name", sorted(SETS))
def test_batch_matches_join_vectors(kiwi, kiwi_cong, typo, name):
    opts, mtype, tset, inputs, _ = SETS[name]
    kw = kiwi_cong if mtype == "cong" else kiwi
    texts, gold = read_inputs(inputs), read_golden(name)
    r = kw.analyze_batch(texts, kiwi_b200.default_option(opts, typo=typo if tset else None))
    assert (r.status == 0).all()
    for i, g in enumerate(gold):
        check_rows(rows_of(r, i), g, (name, i, texts[i]))
        assert _close(float(r.scores[i]), g["score"]), (name, i)


@pytest.mark.parametrize("name", ["join1_inputs_web", "join1_inputs_ref_tests", "join2_inputs_saisiot", "join2_inputs_ref_tests"])
def test_analyze_w_matches_join_vectors(kiwi, name):
    """kiwi_analyze_w: forms (kiwi_res_form_w), morpheme ids (-1 for a joined token) and every kiwi_token_info_t field the vectors hold"""
    opts, _, _, inputs, _ = SETS[name]
    lib = kiwi._lib
    lib.kiwi_res_token_info.restype = C.POINTER(TokenInfo); lib.kiwi_res_token_info.argtypes = [C.c_void_p, C.c_int, C.c_int]
    lib.kiwi_res_form_w.restype = C.c_void_p; lib.kiwi_res_form_w.argtypes = [C.c_void_p, C.c_int, C.c_int]
    lib.kiwi_res_morpheme_id.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    texts, gold = read_inputs(inputs), read_golden(name)
    for i, (t, g) in enumerate(zip(texts, gold)):
        buf = np.ascontiguousarray(np.frombuffer((t + "\0").encode("utf-16-le", "surrogatepass"), dtype="<u2"))
        res = lib.kiwi_analyze_w(kiwi._h, buf.ctypes.data, 1, kiwi_b200.default_option(opts), None)
        assert res, kiwi_b200._last_error(lib)
        try:
            n = lib.kiwi_res_word_num(res, 0)
            assert n == len(g["tokens"]), (name, i, t)
            for k in range(n):
                info = lib.kiwi_res_token_info(res, 0, k).contents
                morph, tag, pos, ln, score = g["tokens"][k]
                assert (lib.kiwi_res_morpheme_id(res, 0, k, None), info.tag, info.chr_position, info.length) == (morph if morph != 0xFFFFFFFF else -1, tag, pos, ln), (name, i, k)
                assert _close(info.score, score), (name, i, k)
                fields = (info.word_position, info.sent_position, info.line_number, info.sub_sent_position,
                          -1 if info.paired_token == 0xFFFFFFFF else info.paired_token)
                assert fields == g["forms"][k][0], (name, i, k)
                p = lib.kiwi_res_form_w(res, 0, k)
                form = _u16_at(p)
                assert form == g["forms"][k][1], (name, i, k, form)
        finally:
            lib.kiwi_res_close(res)


def _u16_at(p):
    out = []
    a = C.cast(p, C.POINTER(C.c_uint16))
    while a[len(out)]:
        out.append(a[len(out)])
    return np.array(out, np.uint16).tobytes().decode("utf-16-le", "replace")      # (the vectors hold U+FFFD for an unpaired surrogate)


def _sample():
    """J1 / Knlm sentences of all four files with the retry-bound sentence at index len(texts) // 2, and their vectors"""
    texts, gold = [], []
    for name in ["join1_inputs_web", "join1_inputs_written", "join1_inputs_ref_tests", "join1_inputs_dialect_typos"]:
        texts += read_inputs(SETS[name][3]); gold += read_golden(name)
    mid = (len(texts) + 1) // 2
    return texts[:mid] + [HEAVY] + texts[mid:], gold[:mid] + [None] + gold[mid:]


def test_retry_arena_and_two_engines_give_the_same_rows(kiwi):
    texts, gold = _sample()
    r = kiwi.analyze_batch(texts, kiwi_b200.default_option(J1))
    assert kiwi.last_stats().retried >= 1
    single = kiwi.analyze_batch([HEAVY], kiwi_b200.default_option(J1))
    ref = [rows_of(r, i) for i in range(len(texts))]
    assert ref[len(texts) // 2] == rows_of(single, 0)
    for i, g in enumerate(gold):
        if g is not None:
            check_rows(ref[i], g, i)
    with open(IMAGE, "rb") as f:
        img = f.read()
    two = kiwi_b200.Kiwi(image_bytes=img, devices=[0, 0])
    try:
        r2 = two.analyze_batch(texts, kiwi_b200.default_option(J1))
        assert [rows_of(r2, i) for i in range(len(texts))] == ref
    finally:
        two.close()


def test_many_passes_give_the_same_rows(kiwi, tmp_path):
    """KIWI_B200_PASS_SENT=16 cuts the batch into many passes (a later pass's joined rows point behind the forms of the earlier ones)"""
    texts, _ = _sample()
    ref = kiwi.analyze_batch(texts, kiwi_b200.default_option(J1))
    path = str(tmp_path / "join.npy")
    code = ("import sys, numpy as np; sys.path.insert(0, %r); import kiwi_b200; from tests.test_gpu_join import _sample, rows_of\n"
            "from tests.orc import IMAGE\n"
            "texts, _ = _sample(); kw = kiwi_b200.Kiwi(IMAGE); r = kw.analyze_batch(texts, kiwi_b200.default_option(%d))\n"
            "np.save(%r, np.array([repr(rows_of(r, i)) for i in range(len(texts))], dtype=object), allow_pickle=True)\n") % (ROOT, J1, path)
    subprocess.run([sys.executable, "-c", code], check=True, env=dict(os.environ, KIWI_B200_PASS_SENT="16"), timeout=900)
    got = np.load(path, allow_pickle=True).tolist()
    assert got == [repr(rows_of(ref, i)) for i in range(len(texts))]


def test_calls_without_join_options_are_unchanged(kiwi):
    lib = kiwi._lib
    texts = read_inputs("inputs_web") + read_inputs("inputs_written")
    blob, off = kiwi_b200.encode_batch(texts)

    def plain():
        p = lib.kiwi_b200_analyze_batch(kiwi._h, blob.ctypes.data, off.ctypes.data, len(texts), kiwi_b200.default_option(M))
        assert p
        try:
            b = p.contents
            assert not b.forms and b.forms_size == 0
            n = b.token_offsets[len(texts)]
            return C.string_at(b.tokens, n * kiwi_b200.TOKEN_DTYPE.itemsize)
        finally:
            lib.kiwi_b200_batch_free(p)

    before = plain()
    kiwi.analyze_batch(texts, kiwi_b200.default_option(J1)); kiwi.analyze_batch(texts, kiwi_b200.default_option(J2))
    assert plain() == before
    for name in ["inputs_web", "inputs_written"]:
        gold = read_golden(name)
        r = kiwi.analyze_batch(read_inputs(name))
        for i, g in enumerate(gold):
            assert [tuple(int(v) for v in (t["morph_id"], t["tag"], t["position"], t["length"])) for t in r.sentence(i)] == [x[:4] for x in g["tokens"]]


def test_refusals_still_hold(kiwi):
    lib = kiwi._lib
    text = np.ascontiguousarray(np.frombuffer("문장이다.\0".encode("utf-16-le"), dtype="<u2"))
    for bit in (1 << 8, 1 << 9, 1 << 30):
        assert not lib.kiwi_analyze_w(kiwi._h, text.ctypes.data, 1, kiwi_b200.default_option(M | bit), None)
        assert b"outside the kiwi_b200 hot path" in lib.kiwi_error()
        lib.kiwi_clear_error()
    for bit in (1 << 17, 1 << 24, 1 << 26, 1 << 27):
        assert not lib.kiwi_split_into_sents_w(kiwi._h, text.ctypes.data, M | bit, None)
        lib.kiwi_clear_error()
        with pytest.raises(kiwi_b200.KiwiError):
            kiwi.split_batch(["문장."], match_options=M | bit)
        with pytest.raises(kiwi_b200.KiwiError):
            kiwi.analyze_device(0, 0, 1, 1, kiwi_b200.default_option(M | bit))
    assert kiwi.analyze("나뭇잎이 바람에 흔들린다.", option=kiwi_b200.default_option(J2))[0][1] != 0
