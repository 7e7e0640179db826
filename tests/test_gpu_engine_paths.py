"""GPU (-m gpu): the engine's pass and retry paths with retried sentences in more than one pass - analyze_device cut into several
passes (on-device offset rebase), and host passes much smaller than the batch.  Both entry points must retry the same sentences
and return what one pass over the batch returns."""
import os
import subprocess
import sys
import numpy as np
import pytest
import kiwi_b200
from tests.orc import IMAGE

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# sentences whose paths overflow a main arena and fit the retry arena's first round (host simulation of the kernels at both sizes)
RETRY = ["다" * 100, "가나" * 50, "이가" * 60, "가" * 200]
TOO_LONG = "a b " * 40000     # one chunk beyond the 16-bit node index: ST_TOO_LONG in every arena, never retried
ST_TOO_LONG = 5


def test_device_multi_pass_retries_like_host_path():
    """70 000 sentences exceed one analyze_device pass (65 536 sentences / 6 Mi units): it cuts the batch and rebases the offsets
    on the device.  Sentences that need the retry arena sit in the first and the last pass.  analyze_device must count the tokens
    analyze_batch returns, and both must retry the same sentences."""
    import torch
    from kiwi_b200.synth import synth_batch
    # (the first 16 characters of each sentence: the first pass's arena takes ~17 GB instead of the 46 GB of a 6 Mi-unit pass)
    texts = [t[:16] for t in synth_batch(70000, 2024)]
    plants = dict(zip((10, 20000, 50000, 69990), RETRY))
    for i, t in plants.items():
        texts[i] = t
    texts[35000] = TOO_LONG
    blob, off = kiwi_b200.encode_batch(texts)
    kw = kiwi_b200.Kiwi(IMAGE)      # (its own handle: close() gives the device pass's arena back)
    try:
        res = kw.analyze_batch(texts)
        host = kw.last_stats()
        d_blob = torch.from_numpy(blob.view(np.int16)).cuda()
        d_off = torch.from_numpy(off.view(np.int32)).cuda()
        torch.cuda.synchronize()
        _, n_tokens, launches = kw.analyze_device(d_blob.data_ptr(), d_off.data_ptr(), len(texts), int(blob.size))
        dev = kw.last_stats()
    finally:
        kw.close()
    assert int(res.status[35000]) == ST_TOO_LONG and len(res.sentence(35000)) == 0
    for i in plants:
        assert int(res.status[i]) == 0 and len(res.sentence(i)) > 0, i
    assert host.retried >= len(plants)
    assert launches >= 3 * 6, "two device passes and a retry launch"
    assert n_tokens == int(res.token_offsets[-1]) == dev.tokens
    assert dev.retried == host.retried


def test_retries_in_several_small_passes_match_one_pass(kiwi, tmp_path):
    """KIWI_B200_PASS_SENT=700 cuts 5 000 sentences into eight host passes, with sentences that need the retry arena in several of
    them: offsets, tokens, scores and statuses must equal those of one pass, and each retried sentence its result alone."""
    plants = dict(zip((3, 1500, 2900, 4999), RETRY))
    code = ("import sys, numpy as np; sys.path.insert(0, %r); import kiwi_b200; from kiwi_b200.synth import synth_batch\n"
            "texts = synth_batch(5000, 99)\n"
            "for i, t in %r.items(): texts[i] = t\n"
            "kw = kiwi_b200.Kiwi(%r); r = kw.analyze_batch(texts)\n"
            "np.savez(sys.argv[1], off=r.token_offsets, tok=r.tokens, sc=r.scores, st=r.status, retried=kw.last_stats().retried)") % (ROOT, plants, IMAGE)
    outs = []
    for ps in ("16384", "700"):
        path = str(tmp_path / ("pass_sent_%s.npz" % ps))
        subprocess.run([sys.executable, "-c", code, path], check=True, env=dict(os.environ, KIWI_B200_PASS_SENT=ps), timeout=600)
        outs.append(dict(np.load(path)))
    one, small = outs
    assert int(one["retried"]) >= len(plants) and int(small["retried"]) == int(one["retried"])
    assert (one["off"] == small["off"]).all() and one["tok"].tobytes() == small["tok"].tobytes()
    assert (one["sc"] == small["sc"]).all() and (one["st"] == small["st"]).all()
    for i, t in plants.items():
        alone = kiwi.analyze_batch([t])
        got = small["tok"][small["off"][i]:small["off"][i + 1]]
        assert got.tobytes() == alone.sentence(0).tobytes() and small["sc"][i] == alone.scores[0] and small["st"][i] == alone.status[0], i
