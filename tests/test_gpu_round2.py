"""GPU (-m gpu), round 2: parity of the BENCH batches themselves against the UNMODIFIED reference (tokens that oracle/_ref/ref_bench
dumped for the whole batch, stored for a fixed sample of sentences in tests/golden/refbench_*.npz by tests/golden/make_refbench.py),
the engine-ownership / multi-device / pass-pipelining paths, and the remaining reference C-ABI entry points (kiwi_analyze,
kiwi_analyze_m, kiwi_res_word_position / kiwi_res_sent_position)."""
import ctypes as C
import os
import subprocess
import tempfile
import numpy as np
import pytest
import kiwi_b200
from tests.goldenio import read_golden, read_inputs
from tests.orc import IMAGE, CONG_IMAGE, TYPO_IMAGES

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
RTOL = 1e-4


def _reference_golden(name):
    """(sentence indices, token counts, sentence scores, token rows) of the unmodified reference for one stored batch"""
    z = np.load(os.path.join(GOLDEN, "refbench_%s.npz" % name))
    counts = z["counts"].astype(np.int64)
    off = np.concatenate([[0], np.cumsum(counts)])
    toks = np.frombuffer(z["tokens"].tobytes(), dtype=kiwi_b200.TOKEN_DTYPE)
    return z["index"].astype(np.int64), counts, z["scores"], [toks[off[i]:off[i + 1]] for i in range(len(counts))]


def _compare_with_reference(res, idx, counts, scores, rows, texts, what):
    got_counts = np.diff(res.token_offsets.astype(np.int64))[idx]
    bad = np.nonzero(got_counts != counts)[0]
    assert len(bad) == 0, (what, "token counts differ", int(idx[bad[0]]), texts[int(idx[bad[0]])])
    ref = np.concatenate(rows) if rows else np.zeros(0, kiwi_b200.TOKEN_DTYPE)
    got = np.concatenate([res.sentence(int(i)) for i in idx]) if len(idx) else np.zeros(0, kiwi_b200.TOKEN_DTYPE)
    off = np.concatenate([[0], np.cumsum(counts)])
    for f in ("morph_id", "position", "length", "tag"):
        d = np.nonzero(got[f] != ref[f])[0]
        if len(d):
            s = int(idx[np.searchsorted(off, d[0], side="right") - 1])
            raise AssertionError((what, f, "differs in sentence", s, texts[s]))
    tol = RTOL * np.maximum(1.0, np.abs(ref["score"]))
    assert (np.abs(got["score"] - ref["score"]) <= tol).all(), what
    got_scores = res.scores[idx]
    assert (np.abs(got_scores - scores) <= RTOL * np.maximum(1.0, np.abs(scores))).all(), what
    exact = float((got_scores == scores).mean())
    print("%s: %d sampled sentences, %d tokens identical to the unmodified reference; %.2f %% of the sentence scores bit-exact" % (what, len(idx), len(ref), 100 * exact))
    assert exact >= 0.99


def test_bench_batch_config2_all_sentences_match_reference(kiwi):
    """the config-2 bench batch (8192, Knlm) against the reference's own tokens (stored sample)"""
    import bench
    from kiwi_b200.synth import SEED
    texts = bench.gen_sentences(bench.CONFIGS[2], 0, 8192, SEED)
    res = kiwi.analyze_batch(texts)
    _compare_with_reference(res, *_reference_golden("cfg2"), texts, "config 2")


def test_bench_batch_config3_cong_65536_matches_reference(kiwi_cong):
    """config 3 at its stated size: 65536 sentences, CoNg model, against the reference (stored sample; multi-pass engine path)"""
    import bench
    from kiwi_b200.synth import SEED
    texts = bench.gen_sentences(bench.CONFIGS[3], 0, 65536, SEED)
    res = kiwi_cong.analyze_batch(texts)
    _compare_with_reference(res, *_reference_golden("cfg3"), texts, "config 3")


def test_bench_batch_config4_typo_65536_matches_reference(kiwi):
    """config 4 at its stated size: 65536 sentences (30 % typo eojeols), Knlm + basic typo lattice, against the reference with
    option.typoTransformer = basicTypoSet.prepare(true)"""
    import bench
    from kiwi_b200.synth import SEED
    cfg = bench.CONFIGS[4]
    texts = bench.gen_sentences(cfg, 0, 65536, SEED)
    typo = kiwi_b200.PreparedTypo(path=TYPO_IMAGES["basic"])
    res = kiwi.analyze_batch(texts, kiwi_b200.default_option(typo=typo))
    _compare_with_reference(res, *_reference_golden("cfg4"), texts, "config 4")
    plain = kiwi.analyze_batch(texts[:4096])
    changed = sum(1 for i in range(4096) if plain.sentence(i).tobytes() != res.sentence(i).tobytes())
    print("config 4: the typo lattice changes %d of the first 4096 analyses" % changed)
    assert changed > 0
    typo.close()


def test_constant_view_ownership_use_a_create_b_use_a():
    """ADVICE r1 (high): handle A analyses, handle B (another model) is created and analyses, A analyses again - A must run with
    its own model view, not B's (the constant-memory view is re-uploaded when its owner changed)."""
    texts = read_inputs("inputs_web")[:64]
    gk = read_golden("inputs_web"); gc = read_golden("cong_inputs_web")
    a = kiwi_b200.Kiwi(IMAGE)
    ra1 = a.analyze_batch(texts)
    b = kiwi_b200.Kiwi(CONG_IMAGE)            # created AFTER a was used
    ra2 = a.analyze_batch(texts)              # a again, before b ever ran
    rb = b.analyze_batch(texts)
    ra3 = a.analyze_batch(texts)
    for r in (ra1, ra2, ra3):
        for i in range(len(texts)):
            assert [(int(k["morph_id"]), int(k["tag"]), int(k["position"]), int(k["length"])) for k in r.sentence(i)] == [x[:4] for x in gk[i]["tokens"]], i
    for i in range(len(texts)):
        assert [(int(k["morph_id"]), int(k["tag"]), int(k["position"]), int(k["length"])) for k in rb.sentence(i)] == [x[:4] for x in gc[i]["tokens"]], i
    b.close()
    ra4 = a.analyze_batch(texts)              # b's engine is gone: the owner pointer must not dangle
    assert ra4.tokens.tobytes() == ra1.tokens.tobytes()
    a.close()


def test_two_handles_from_two_threads():
    """ADVICE r1 (medium): two threads analysing on two handles of one device take turns on the device lock"""
    import threading
    texts = read_inputs("inputs_web")
    gk = read_golden("inputs_web"); gc = read_golden("cong_inputs_web")
    a = kiwi_b200.Kiwi(IMAGE); b = kiwi_b200.Kiwi(CONG_IMAGE)
    errs = []

    def run(kw, gold):
        try:
            for _ in range(6):
                r = kw.analyze_batch(texts)
                for i in range(len(texts)):
                    if [int(k["morph_id"]) for k in r.sentence(i)] != [x[0] for x in gold[i]["tokens"]]: errs.append(i)
        except Exception as e:
            errs.append(repr(e))

    ts = [threading.Thread(target=run, args=(a, gk)), threading.Thread(target=run, args=(b, gc))]
    for t in ts: t.start()
    for t in ts: t.join()
    assert not errs, errs[:5]
    a.close(); b.close()


def test_multi_device_handle_round_robin_ordered_merge(kiwi):
    """kiwi_b200_init_multi: ONE handle, several engines, sentence i -> engine i mod N, one host thread per engine, results in input
    order.  With a single GPU in the box the two engines share device 0 (the fan-out / merge logic is the same)."""
    import torch
    from kiwi_b200.synth import synth_batch
    ndev = torch.cuda.device_count()
    devices = [0, 1] if ndev >= 2 else [0, 0]
    multi = kiwi_b200.Kiwi(IMAGE, devices=devices + ([2] if ndev >= 3 else []))
    texts = synth_batch(3001, 4242)
    rm = multi.analyze_batch(texts)
    rs = kiwi.analyze_batch(texts)
    assert (rm.token_offsets == rs.token_offsets).all() and rm.tokens.tobytes() == rs.tokens.tobytes() and (rm.scores == rs.scores).all()
    multi.close()


def test_small_passes_overlap_and_keep_order():
    """KIWI_B200_PASS_SENT forces many small passes through the two-slot pipeline: the result must equal the single-pass result"""
    from kiwi_b200.synth import synth_batch
    texts = synth_batch(5000, 99)
    code = ("import os, sys, numpy as np; sys.path.insert(0, %r); import kiwi_b200; from kiwi_b200.synth import synth_batch; "
            "kw = kiwi_b200.Kiwi(%r); r = kw.analyze_batch(synth_batch(5000, 99)); "
            "np.savez(sys.argv[1], off=r.token_offsets, tok=r.tokens, sc=r.scores)") % (ROOT, IMAGE)
    outs = []
    for ps in ("16384", "700"):
        path = tempfile.mktemp(suffix=".npz")
        subprocess.run([os.sys.executable, "-c", code, path], check=True, env=dict(os.environ, KIWI_B200_PASS_SENT=ps), timeout=600)
        outs.append(np.load(path)); os.unlink(path)
    assert (outs[0]["off"] == outs[1]["off"]).all() and outs[0]["tok"].tobytes() == outs[1]["tok"].tobytes() and (outs[0]["sc"] == outs[1]["sc"]).all()


def test_utf8_entry_points_and_position_accessors(kiwi, oracle):
    """kiwi_analyze (UTF-8), kiwi_analyze_m (UTF-8 reader) and kiwi_res_word_position / kiwi_res_sent_position (capi.h:698, 724, 897, 907)"""
    lib = kiwi_b200.load_library()
    opt = kiwi_b200.default_option()
    lib.kiwi_analyze.restype = C.c_void_p
    lib.kiwi_analyze.argtypes = [C.c_void_p, C.c_char_p, C.c_int, kiwi_b200.AnalyzeOption, C.c_void_p]
    for fn in ("kiwi_res_word_position", "kiwi_res_sent_position"): getattr(lib, fn).argtypes = [C.c_void_p, C.c_int, C.c_int]
    texts = read_inputs("inputs_web")[:30]; gold = read_golden("inputs_web")
    for t, g in zip(texts, gold):
        r = lib.kiwi_analyze(kiwi._h, t.encode("utf-8"), 1, opt, None)
        assert r, lib.kiwi_error()
        n = lib.kiwi_res_word_num(r, 0)
        got = [(lib.kiwi_res_morpheme_id(r, 0, i, kiwi._h), lib.kiwi_res_position(r, 0, i), lib.kiwi_res_length(r, 0, i)) for i in range(n)]
        assert got == [(x[0], x[2], x[3]) for x in g["tokens"]], t
        assert [(lib.kiwi_res_word_position(r, 0, i), lib.kiwi_res_sent_position(r, 0, i)) for i in range(n)] == [f[0][:2] for f in g["forms"]], t
        assert lib.kiwi_res_word_position(r, 0, n) < 0 and lib.kiwi_res_sent_position(r, 0, -1) < 0
        lib.kiwi_res_close(r)
    READER = C.CFUNCTYPE(C.c_int, C.c_int, C.POINTER(C.c_char), C.c_void_p)
    RECEIVER = C.CFUNCTYPE(C.c_int, C.c_int, C.c_void_p, C.c_void_p)
    order = []; toks = []

    def reader(idx, out, ud):
        if idx >= len(texts): return 0
        enc = texts[idx].encode("utf-8")
        if out: C.memmove(out, enc, len(enc))
        return len(enc)

    def receiver(idx, res, ud):
        n = lib.kiwi_res_word_num(res, 0)
        order.append(idx); toks.append([lib.kiwi_res_morpheme_id(res, 0, i, kiwi._h) for i in range(n)]); lib.kiwi_res_close(res); return 0

    lib.kiwi_analyze_m.argtypes = [C.c_void_p, READER, RECEIVER, C.c_void_p, C.c_int, kiwi_b200.AnalyzeOption]
    assert lib.kiwi_analyze_m(kiwi._h, READER(reader), RECEIVER(receiver), None, 1, opt) == len(texts)
    assert order == list(range(len(texts)))
    assert toks == [[x[0] for x in g["tokens"]] for g in gold[:len(texts)]]


def test_top1_container_and_full_bucket_cases_match_reference(kiwi, oracle):
    """DESIGN.md's documented deviation, probed on purpose: nodes with more than 512 incoming paths use the reference's `top1`
    container (an unordered_set whose iteration order the kernels replace by insertion order), and 128-slot buckets that fill up
    drop insertions.  The oracle's counters pick the bench sentences that really exercise these rules; the expected values are the
    UNMODIFIED reference's tokens for exactly those sentences."""
    import bench
    from kiwi_b200.synth import SEED
    texts = bench.gen_sentences(bench.CONFIGS[2], 0, 2048, SEED)
    hard = []; prev = oracle.counters2()
    for i, t in enumerate(texts):
        oracle.analyze(t); c = oracle.counters2()
        if c["top1Mode"] > prev["top1Mode"] or c["bucketFull"] > prev["bucketFull"]: hard.append(i)
        prev = c
    print("%d of %d bench sentences use the top1 container or hit a full bucket" % (len(hard), len(texts)))
    assert len(hard) >= 8
    idx, counts, scores, rows = _reference_golden("top1")
    assert hard == idx.tolist()
    sub = [texts[i] for i in hard]
    res = kiwi.analyze_batch(sub)
    _compare_with_reference(res, np.arange(len(sub)), counts, scores, rows, sub, "top1 / full-bucket sentences")


def test_input_text_never_fails_the_batch(kiwi, oracle):
    """ADVICE r1 (medium / low): a sentence whose lattice does not fit the device structures (here: one chunk with more than 65535
    nodes - 'a b a b ...' never meets the chunk-break condition) comes back with a non-zero status and no tokens; its neighbours in
    the batch are analysed normally and nothing throws."""
    texts = ["안녕하세요. 반갑습니다!", "a b " * 40000, "형태소 분석기입니다."]
    res = kiwi.analyze_batch(texts)
    assert int(res.status[0]) == 0 and int(res.status[2]) == 0
    assert int(res.status[1]) != 0 and len(res.sentence(1)) == 0
    for i in (0, 2):
        otoks, oscore = oracle.analyze(texts[i])
        assert [(int(k["morph_id"]), int(k["tag"]), int(k["position"]), int(k["length"])) for k in res.sentence(i)] == [x[:4] for x in otoks]
