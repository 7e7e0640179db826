"""GPU (-m gpu): the CUDA hot path, called through the C ABI, against (a) the golden vectors of the unmodified
reference and (b) the oracle restatement.  Integer / index fields must be bit-exact; the float path score and
word scores must agree within 1e-4 relative (BASELINE.json) — the tests also report how many are bit-exact."""
import numpy as np
import pytest
import kiwi_b200
from tests.goldenio import read_golden, read_inputs

pytestmark = pytest.mark.gpu
RTOL = 1e-4


def _tok4(arr):
    return [(int(k["morph_id"]), int(k["tag"]), int(k["position"]), int(k["length"])) for k in arr]


def _close(a, b):
    return abs(a - b) <= RTOL * max(1.0, abs(b))


@pytest.mark.parametrize("name", ["inputs_ref_tests", "inputs_web", "inputs_written", "inputs_dialect_typos"])
def test_tokens_and_scores_match_reference_golden(kiwi, name):
    texts = read_inputs(name); gold = read_golden(name)
    res = kiwi.analyze_batch(texts)
    exact = 0
    for i, (t, g) in enumerate(zip(texts, gold)):
        got = res.sentence(i)
        assert _tok4(got) == [x[:4] for x in g["tokens"]], (i, t)
        assert _close(float(res.scores[i]), g["score"]), (i, t, float(res.scores[i]), g["score"])
        for k, x in zip(got, g["tokens"]):
            assert _close(float(k["score"]), x[4]), (i, t)
        exact += int(np.float32(res.scores[i]) == np.float32(g["score"]))
    print("%s: %d/%d sentence scores bit-exact" % (name, exact, len(texts)))
    assert exact >= 0.99 * len(texts)


@pytest.mark.parametrize("name", ["inputs_ref_tests", "inputs_web"])
def test_lattice_matches_reference_golden(kiwi, name):
    texts = read_inputs(name); gold = read_golden(name)
    for t, g in list(zip(texts, gold))[::2]:
        assert kiwi.debug_lattice(t).tolist() == g["lattice"], t


def test_batch_8192_properties_and_sampled_oracle(kiwi, oracle):
    """Full benchmark size: size-independent properties + a sampled comparison with the oracle."""
    from kiwi_b200.synth import synth_batch, u16len
    texts = synth_batch(8192)
    r1 = kiwi.analyze_batch(texts)
    r2 = kiwi.analyze_batch(texts)
    # determinism / idempotence of the whole batch
    assert (r1.token_offsets == r2.token_offsets).all() and r1.tokens.tobytes() == r2.tokens.tobytes() and (r1.scores == r2.scores).all()
    # batch-composition invariance: a sentence's result does not depend on its neighbours
    perm = np.random.RandomState(7).permutation(len(texts))[:512]
    r3 = kiwi.analyze_batch([texts[i] for i in perm])
    for k, i in enumerate(perm):
        assert r3.sentence(k).tobytes() == r1.sentence(int(i)).tobytes() and r3.scores[k] == r1.scores[i]
    # coverage property of the reference's EmptyResult test: tokens are in order and end at the end of the text
    for i, t in enumerate(texts):
        s = r1.sentence(i)
        assert len(s) > 0
        pos = s["position"].astype(np.int64); end = pos + s["length"]
        assert (np.diff(pos) >= 0).all()
        assert int(end.max()) == u16len(t.rstrip(" "))
    # sampled oracle parity
    for i in range(0, len(texts), 32):
        otoks, oscore = oracle.analyze(texts[i])
        assert _tok4(r1.sentence(i)) == [x[:4] for x in otoks], texts[i]
        assert _close(float(r1.scores[i]), oscore)


def test_capacity_retry_path(kiwi, oracle):
    """A pathological sentence overflows the first-pass scratch and must come back through the larger second pass."""
    texts = ["가" * 50, "안녕하세요", "가나다라마바사아자차카타파하" * 20]
    res = kiwi.analyze_batch(texts)
    for i, t in enumerate(texts):
        otoks, oscore = oracle.analyze(t)
        assert _tok4(res.sentence(i)) == [x[:4] for x in otoks]
        assert _close(float(res.scores[i]), oscore)


def test_reference_c_api_single_and_multi(kiwi, oracle):
    """kiwi_analyze_w / kiwi_res_* and kiwi_analyze_mw (reader / receiver, results in input order)."""
    import ctypes as C
    lib = kiwi_b200.load_library()
    opt = kiwi_b200.default_option()
    text = "안녕하세요. 반갑습니다!"
    buf = (C.c_uint16 * (len(text) + 1))(*[ord(c) for c in text], 0)
    r = lib.kiwi_analyze_w(kiwi._h, buf, 1, opt, None)
    assert r
    otoks, oscore = oracle.analyze(text)
    n = lib.kiwi_res_word_num(r, 0)
    got = [(lib.kiwi_res_morpheme_id(r, 0, i, kiwi._h), lib.kiwi_res_position(r, 0, i), lib.kiwi_res_length(r, 0, i)) for i in range(n)]
    assert got == [(x[0], x[2], x[3]) for x in otoks]
    assert [lib.kiwi_res_tag(r, 0, i).decode() for i in range(n)] == [kiwi_b200.tag_to_string(x[1]) for x in otoks]
    assert _close(lib.kiwi_res_prob(r, 0), oscore)
    assert lib.kiwi_res_close(r) == 0
    # unsupported option -> NULL + error message, never a silent fallback
    bad = kiwi_b200.default_option(); bad.match_options |= (1 << 8)
    assert not lib.kiwi_analyze_w(kiwi._h, buf, 1, bad, None)
    assert b"outside the kiwi_b200 hot path" in lib.kiwi_error()
    lib.kiwi_clear_error()

    texts = read_inputs("inputs_web")[:40]
    READER = C.CFUNCTYPE(C.c_int, C.c_int, C.POINTER(C.c_uint16), C.c_void_p)
    RECEIVER = C.CFUNCTYPE(C.c_int, C.c_int, C.c_void_p, C.c_void_p)
    order = []; counts = []

    def reader(idx, out, ud):
        if idx >= len(texts): return 0
        enc = np.frombuffer(texts[idx].encode("utf-16-le"), dtype="<u2")
        if out:
            for k, v in enumerate(enc): out[k] = int(v)
        return len(enc)

    def receiver(idx, res, ud):
        order.append(idx); counts.append(lib.kiwi_res_word_num(res, 0)); lib.kiwi_res_close(res); return 0

    lib.kiwi_analyze_mw.argtypes = [C.c_void_p, READER, RECEIVER, C.c_void_p, C.c_int, kiwi_b200.AnalyzeOption]
    n = lib.kiwi_analyze_mw(kiwi._h, READER(reader), RECEIVER(receiver), None, 1, opt)
    assert n == len(texts) and order == list(range(len(texts)))
    assert counts == [len(oracle.analyze(t)[0]) for t in texts]


def test_large_batch_is_split_into_passes(kiwi):
    """40 000 sentences exceed one device pass (16 384 sentences / 1.5 Mi units): the engine cuts the batch and
    the concatenated result must equal the per-pass results (batch-composition invariance at scale)."""
    from kiwi_b200.synth import synth_batch
    base = synth_batch(2000, 12345)
    texts = (base * 20)[:40000]
    r = kiwi.analyze_batch(texts)
    assert len(r.token_offsets) == len(texts) + 1
    ref = kiwi.analyze_batch(base)
    for i in range(0, len(texts), 997):
        j = i % len(base)
        assert r.sentence(i).tobytes() == ref.sentence(j).tobytes() and r.scores[i] == ref.scores[j]


class _TokenInfo(__import__("ctypes").Structure):      # kiwi_token_info_t, include/kiwi_b200.h (capi.h:43-61)
    import ctypes as _C
    _fields_ = [("chr_position", _C.c_uint32), ("word_position", _C.c_uint32), ("sent_position", _C.c_uint32), ("line_number", _C.c_uint32),
                ("length", _C.c_uint16), ("tag", _C.c_uint8), ("sense_id", _C.c_uint8), ("score", _C.c_float), ("typo_cost", _C.c_float),
                ("typo_form_id", _C.c_uint32), ("paired_token", _C.c_uint32), ("sub_sent_position", _C.c_uint32), ("dialect", _C.c_uint16)]


@pytest.mark.parametrize("name", ["inputs_web", "inputs_written"])
def test_result_assembly_forms_and_word_positions(kiwi, name):
    """SURVEY 8f-1 (result assembly): kiwi_res_form and the kiwi_token_info_t fields word / sentence / line / sub-sentence
    position and paired token of every token, through kiwi_analyze_mw, against TokenInfo of the unmodified reference
    (insertPathIntoResults src/Kiwi.cpp:696-756, fillPairedTokenInfo 98-143, fillSentLineInfo 322-415)."""
    import ctypes as C
    lib = kiwi_b200.load_library()
    texts = read_inputs(name); gold = read_golden(name)
    READER = C.CFUNCTYPE(C.c_int, C.c_int, C.POINTER(C.c_uint16), C.c_void_p)
    RECEIVER = C.CFUNCTYPE(C.c_int, C.c_int, C.c_void_p, C.c_void_p)
    lib.kiwi_res_token_info.restype = C.POINTER(_TokenInfo)
    lib.kiwi_res_token_info.argtypes = [C.c_void_p, C.c_int, C.c_int]
    lib.kiwi_res_form.restype = C.c_char_p
    got = {}

    def reader(idx, out, ud):
        if idx >= len(texts): return 0
        enc = np.frombuffer(texts[idx].encode("utf-16-le"), dtype="<u2")
        if out:
            for k, v in enumerate(enc): out[k] = int(v)
        return len(enc)

    def receiver(idx, res, ud):
        n = lib.kiwi_res_word_num(res, 0)
        got[idx] = []
        for i in range(n):
            ti = lib.kiwi_res_token_info(res, 0, i).contents
            paired = int(ti.paired_token); paired = -1 if paired == 0xFFFFFFFF else paired
            got[idx].append(((int(ti.word_position), int(ti.sent_position), int(ti.line_number), int(ti.sub_sent_position), paired), lib.kiwi_res_form(res, 0, i).decode("utf-8")))
        lib.kiwi_res_close(res); return 0

    lib.kiwi_analyze_mw.argtypes = [C.c_void_p, READER, RECEIVER, C.c_void_p, C.c_int, kiwi_b200.AnalyzeOption]
    assert lib.kiwi_analyze_mw(kiwi._h, READER(reader), RECEIVER(receiver), None, 1, kiwi_b200.default_option()) == len(texts)
    for i, g in enumerate(gold):
        assert got[i] == g["forms"], (i, texts[i], got[i], g["forms"])


def test_global_config_round_trip(kiwi, oracle):
    """kiwi_get_global_config returns the KiwiConfig of the image (reference defaults, include/kiwi/Kiwi.h:150-167);
    setting the same values back refreshes the constant-memory model view and must leave results untouched; a larger
    cut-off threshold keeps more paths alive but cannot change the top-1 result of this sentence."""
    c = kiwi.get_global_config()
    assert (c.integrate_allomorph, c.cut_off_threshold, c.oov_rule_scale, c.oov_rule_bias, c.space_penalty, c.typo_cost_weight) == (1, 8.0, 4.0, 4.0, 7.0, 6.0)
    assert (c.max_unk_form_size, c.max_unk_form_size_followed_by_j_class, c.space_tolerance) == (6, 0xFFFFFFFF, 0)
    assert (c.oov_chr_bias, c.oov_global_weight, c.oov_local_weight, c.oov_global_min_freq) == (0.0, 35.0, 3.0, 4.0)
    t = "설정 값을 다시 써도 분석 결과는 그대로여야 합니다."
    before = kiwi.analyze_batch([t])
    kiwi.set_global_config(c)
    after = kiwi.analyze_batch([t])
    assert before.sentence(0).tobytes() == after.sentence(0).tobytes() and before.scores[0] == after.scores[0]
    otoks, oscore = oracle.analyze(t)
    assert _tok4(after.sentence(0)) == [x[:4] for x in otoks] and _close(float(after.scores[0]), oscore)
    c2 = kiwi.get_global_config()
    assert c2.cut_off_threshold == 8.0 and c2.space_tolerance == 0
