"""GPU (-m gpu): sentence splitting on the device (kiwi_split_into_sents[_w], kiwi_ss_*, kiwi_b200_split_batch) against the unmodified
reference's Kiwi::splitIntoSents over every document of tests/golden/docs_sents.jsonl, Knlm and CoNg: ranges in UTF-16 units and in
UTF-8 bytes, the tokenized result, the batched call through several passes and the retry arena, a multi-device handle, the error
convention, and no state left behind in the handle."""
import ctypes as C
import os
import subprocess
import sys
import numpy as np
import pytest
import kiwi_b200
from tests.orc import IMAGE, CONG_IMAGE
from tests.sentsio import read_docs, read_sents_golden

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M = kiwi_b200.MATCH_ALL_WITH_NORMALIZING


class TokenInfo(C.Structure):      # kiwi_token_info_t
    _fields_ = [("chr_position", C.c_uint32), ("word_position", C.c_uint32), ("sent_position", C.c_uint32), ("line_number", C.c_uint32),
                ("length", C.c_uint16), ("tag", C.c_uint8), ("sense_id", C.c_uint8), ("score", C.c_float), ("typo_cost", C.c_float),
                ("typo_form_id", C.c_uint32), ("paired_token", C.c_uint32), ("sub_sent_position", C.c_uint32), ("dialect", C.c_uint16)]


def _u16z(text):
    return np.ascontiguousarray(np.frombuffer((text + "\0").encode("utf-16-le", "surrogatepass"), dtype="<u2"))


def _ss_ranges(lib, ss):
    return [(lib.kiwi_ss_begin_position(ss, i), lib.kiwi_ss_end_position(ss, i)) for i in range(lib.kiwi_ss_size(ss))]


@pytest.mark.parametrize("which", ["knlm", "cong"])
def test_split_w_matches_reference(which, kiwi, kiwi_cong):
    kw, prefix = (kiwi, "") if which == "knlm" else (kiwi_cong, "cong_")
    docs, gold = read_docs(), read_sents_golden(prefix)
    bad = [i for i, (d, g) in enumerate(zip(docs, gold)) if kw.split_into_sents(d) != g["ranges"]]
    assert not bad, (which, len(bad), bad[:10], [docs[i][:60] for i in bad[:3]])


def test_split_utf8_returns_reference_byte_offsets(kiwi):
    lib = kiwi._lib
    docs, gold = read_docs(), read_sents_golden("")
    for i, (d, g) in enumerate(zip(docs, gold)):
        ss = lib.kiwi_split_into_sents(kiwi._h, d.encode("utf-8"), M, None)
        assert ss, kiwi_b200._last_error(lib)
        try:
            assert _ss_ranges(lib, ss) == g["byte_ranges"], (i, d[:60])
        finally:
            lib.kiwi_ss_close(ss)


def test_tokenized_res_matches_reference(kiwi):
    lib = kiwi._lib
    lib.kiwi_res_token_info.restype = C.POINTER(TokenInfo)
    lib.kiwi_res_token_info.argtypes = [C.c_void_p, C.c_int, C.c_int]
    docs, gold = read_docs(), read_sents_golden("")
    for i, (d, g) in enumerate(zip(docs, gold)):
        res = C.c_void_p(None)
        u = _u16z(d)      # (kept alive for the call)
        ss = lib.kiwi_split_into_sents_w(kiwi._h, u.ctypes.data, M, C.byref(res))
        assert ss and res.value, kiwi_b200._last_error(lib)
        try:
            ranges = _ss_ranges(lib, ss)
            n = lib.kiwi_res_word_num(res.value, 0)
            assert n == len(g["tokens"]), (i, d[:60])
            derived, last = [], None
            for k in range(n):
                info = lib.kiwi_res_token_info(res.value, 0, k).contents
                morph, tag, pos, ln, score = g["tokens"][k]
                assert (lib.kiwi_res_morpheme_id(res.value, 0, k, None), info.tag, info.chr_position, info.length) == (morph, tag, pos, ln), (i, k)
                assert abs(info.score - score) <= 1e-4 * max(1.0, abs(score)), (i, k, info.score, score)
                fields = (info.word_position, info.sent_position, info.line_number, info.sub_sent_position,
                          -1 if info.paired_token == 0xFFFFFFFF else info.paired_token)
                assert fields == g["forms"][k][0], (i, k, fields, g["forms"][k][0])
                if info.sent_position != last:
                    derived.append([pos, pos + ln]); last = info.sent_position
                else:
                    derived[-1][1] = pos + ln
            assert ranges == [tuple(r) for r in derived] == g["ranges"], (i, d[:60])
        finally:
            lib.kiwi_ss_close(ss)
            lib.kiwi_res_close(res.value)


def test_split_batch_equals_per_document_calls_and_reference(kiwi):
    docs, gold = read_docs(), read_sents_golden("")
    r = kiwi.split_batch(docs)
    assert (r.status == 0).all()
    for i, (d, g) in enumerate(zip(docs, gold)):
        got = [tuple(int(v) for v in x) for x in r.ranges(i)]
        assert got == g["ranges"], (i, d[:60])
    assert r.timings_ms["sents"] > 0 and r.timings_ms["total"] >= r.timings_ms["sents"]


def test_split_batch_over_many_passes_and_the_retry_arena(tmp_path):
    """KIWI_B200_PASS_SENT=16 cuts the documents into 26 passes; the repeated-syllable document overflows its first arena and is split
    from the retry arena's rows.  Ranges equal the reference's, and the retry arena was used."""
    path = str(tmp_path / "split.npz")
    code = ("import sys, numpy as np; sys.path.insert(0, %r); import kiwi_b200; from tests.sentsio import read_docs\n"
            "kw = kiwi_b200.Kiwi(%r); r = kw.split_batch(read_docs())\n"
            "np.savez(sys.argv[1], off=r.sent_offsets, b=r.begin, e=r.end, st=r.status, retried=kw.last_stats().retried)") % (ROOT, IMAGE)
    subprocess.run([sys.executable, "-c", code, path], check=True, env=dict(os.environ, KIWI_B200_PASS_SENT="16"), timeout=600)
    z = dict(np.load(path))
    assert int(z["retried"]) > 0 and (z["st"] == 0).all()
    for i, g in enumerate(read_sents_golden("")):
        a, b = int(z["off"][i]), int(z["off"][i + 1])
        assert list(zip(z["b"][a:b].tolist(), z["e"][a:b].tolist())) == g["ranges"], i


def test_split_batch_on_several_devices_keeps_input_order():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one device visible")
    docs, gold = read_docs(), read_sents_golden("")
    kw = kiwi_b200.Kiwi(IMAGE, devices=list(range(torch.cuda.device_count())))
    try:
        r = kw.split_batch(docs)
        for i, g in enumerate(gold):
            assert [tuple(int(v) for v in x) for x in r.ranges(i)] == g["ranges"], i
    finally:
        kw.close()


def test_split_error_paths(kiwi):
    lib = kiwi._lib
    short = _u16z("문장.")
    assert not lib.kiwi_split_into_sents_w(None, short.ctypes.data, M, None)
    assert lib.kiwi_ss_size(None) == -2 and lib.kiwi_ss_close(None) == -2
    docs, gold = read_docs(), read_sents_golden("")
    i = next(i for i, g in enumerate(gold) if len(g["ranges"]) >= 2)
    u = _u16z(docs[i])
    ss = lib.kiwi_split_into_sents_w(kiwi._h, u.ctypes.data, M, None)
    assert ss
    try:
        n = lib.kiwi_ss_size(ss)
        assert n == len(gold[i]["ranges"])
        for idx in (-1, n, n + 5):
            assert lib.kiwi_ss_begin_position(ss, idx) == -3 and lib.kiwi_ss_end_position(ss, idx) == -3
    finally:
        assert lib.kiwi_ss_close(ss) == 0
    lib.kiwi_clear_error()
    assert not lib.kiwi_split_into_sents_w(kiwi._h, short.ctypes.data, M | (1 << 17), None)      # a join* flag: outside the path
    assert b"outside the kiwi_b200 hot path" in lib.kiwi_error()
    lib.kiwi_clear_error()
    with pytest.raises(kiwi_b200.KiwiError):
        kiwi.split_batch(["문장."], match_options=M | (1 << 17))
    empty = kiwi.split_batch([])
    assert len(empty.sent_offsets) == 1 and len(empty.status) == 0


def test_split_leaves_no_state_behind(kiwi):
    from kiwi_b200.synth import synth_batch
    texts = synth_batch(3000, 7)
    a = kiwi.analyze_batch(texts)
    a = (a.token_offsets.copy(), a.tokens.copy(), a.scores.copy(), a.status.copy())
    kiwi.split_batch(read_docs())
    kiwi.split_into_sents("그는 \"밥 먹었어?\"라고 물었다.", return_tokens=True)
    b = kiwi.analyze_batch(texts)
    assert (a[0] == b.token_offsets).all() and a[1].tobytes() == b.tokens.tobytes() and (a[2] == b.scores).all() and (a[3] == b.status).all()


def test_split_into_sents_returns_tokens_like_analyze(kiwi):
    text = "첫 문장이다. 둘째 문장이에요?\n셋째."
    ranges, toks = kiwi.split_into_sents(text, return_tokens=True)
    assert ranges == kiwi.split_into_sents(text)
    ref = kiwi.analyze(text)
    assert [t[:4] for t in toks[0][0]] == [t[:4] for t in ref[0][0]] and abs(toks[0][1] - ref[0][1]) <= 1e-4 * max(1.0, abs(ref[0][1]))
