"""GPU (-m gpu): the SkipBigram path (SURVEY 8a row a13: Knlm + SkipBigramModel::evaluate + logSumExp over the 8-token history state),
called through the C ABI, against the golden vectors of the unmodified reference (ModelType::sbg, tests/golden/sbg_*: one fresh
thread per sentence, see tests/golden/make_golden.py) and the oracle restatement.  Bit-exact: morpheme ids, tags, positions, lengths
and every float score - the device restates the AVX2 exp polynomial, glibc's logf and the reference's path containers as they behave
(kiwi_b200/csrc/sbg_math.h, viterbi.cu exactInsertRound)."""
import numpy as np
import pytest
from tests.goldenio import read_golden, read_inputs

pytestmark = pytest.mark.gpu


def _tok4(arr):
    return [(int(k["morph_id"]), int(k["tag"]), int(k["position"]), int(k["length"])) for k in arr]


@pytest.fixture(scope="module")
def kiwi_sbg():
    import kiwi_b200
    from tests.orc import SBG_IMAGE
    kw = kiwi_b200.Kiwi(SBG_IMAGE)      # raises when the CUDA extension or the GPU is missing: no fallback
    yield kw
    kw.close()


# The SkipBigram kernel inserts paths one at a time and is slow on inputs whose path sets explode (the reference itself needs minutes
# and tens of GB on the later sentences of inputs_ref_tests), so the suite keeps to the two corpus files, and this file sorts last among
# the GPU tests.
@pytest.mark.timeout(1200)
@pytest.mark.parametrize("name,limit", [("inputs_written", None), ("inputs_web", 80)])
def test_sbg_tokens_and_scores_match_reference_golden(kiwi_sbg, name, limit):
    assert kiwi_sbg.model_type() == 3
    gold = read_golden("sbg_" + name)
    n = min(len(gold), limit or len(gold))
    texts = read_inputs(name)[:n]; gold = gold[:n]
    res = kiwi_sbg.analyze_batch(texts)
    assert not res.status.any(), np.nonzero(res.status)[0][:10]
    for i, (t, g) in enumerate(zip(texts, gold)):
        got = res.sentence(i)
        assert _tok4(got) == [x[:4] for x in g["tokens"]], (i, t)
        assert np.float32(res.scores[i]) == np.float32(g["score"]), (i, t, float(res.scores[i]), g["score"])
        assert [np.float32(k["score"]) for k in got] == [np.float32(x[4]) for x in g["tokens"]], (i, t)


@pytest.mark.timeout(600)
def test_three_model_types_coexist(kiwi, kiwi_sbg, oracle, oracle_sbg):
    """Knlm and SkipBigram handles in one process: each launch uploads its own model view"""
    t = "키위는 형태소 분석기입니다. 두 모델을 번갈아 씁니다."
    for _ in range(2):
        for kw, orc in ((kiwi, oracle), (kiwi_sbg, oracle_sbg)):
            r = kw.analyze_batch([t])
            otoks, oscore = orc.analyze(t)
            assert _tok4(r.sentence(0)) == [x[:4] for x in otoks]
            assert np.float32(r.scores[0]) == np.float32(oscore)
