#!/usr/bin/env python3
"""Builds tests/golden/docs_sents.jsonl: seeded multi-sentence DOCUMENTS for the sentence splitter (Kiwi::splitIntoSents), one JSON
string per line (documents hold newlines).  They are made from the committed input lines (inputs_written / inputs_web) and cover:
sentences joined by spaces, LF, CR LF, blank lines, VT / FF / U+2028; quoted and bracketed sub-sentences, nested and unbalanced;
bullets; "...요" endings, z_coda endings, final punctuation followed by numbers; URLs, e-mails, emoji; non-BMP characters; empty and
whitespace-only documents; long documents of several thousand UTF-16 units, one of them made of repeated syllables whose paths
overflow the engine's first arena (so it goes through the retry arena).
`python make_docs.py` writes the documents; `python make_docs.py --golden` then runs the unmodified reference on them (needs
oracle/_ref) and writes docs_sents.golden.txt.gz / cong_docs_sents.golden.txt.gz and docs_sents.MANIFEST.json (the md5 of each
vector file and of the model images they were made with)."""
import gzip, hashlib, json, os, random, struct, subprocess, sys
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "docs_sents.jsonl")
SEED = 20261018


def _lines(name):
    with open(os.path.join(HERE, name), encoding="utf-8") as f:
        return [l.rstrip("\n").split("\t")[0] for l in f if l.strip()]


def make_docs():
    rng = random.Random(SEED)
    sents = [s for s in _lines("inputs_written.txt") + _lines("inputs_web.txt") if 4 <= len(s) <= 160]
    pick = lambda: rng.choice(sents)
    seps = [" ", "\n", "\r\n", "\n\n", "\r\n\r\n", "\v", "\f", "\u2028", "  ", " \n "]
    docs = []
    # plain sentences with every kind of separator
    for _ in range(220):
        k = rng.randint(2, 6)
        parts = [pick() for _ in range(k)]
        doc = parts[0]
        for p in parts[1:]:
            doc += rng.choice(seps) + p
        docs.append(doc)
    # quoted / bracketed sub-sentences, nested and unbalanced
    quoted = ['그는 "밥 먹었어?"라고 물었다.', '그녀는 "좋아요. 내일 봐요."라고 말했다. 그리고 떠났다.', "'정말요?' 그가 되물었다.",
              '그는 "나는 \'괜찮다\'고 했어. 정말이야."라고 전했다.', '(이 문장은 괄호 안에 있다. 두 문장이다.) 밖의 문장이다.',
              '「낫표 안의 문장이다.」 다음 문장이다.', '《책 이름》을 읽었다. 재미있었다.', '"열린 따옴표만 있다. 닫히지 않는다.',
              '닫는 괄호만 있다) 그리고 끝난다.', '[대괄호 안. 두 번째.] 뒤.', '{"key": "값"} 이런 것도 있다.', '그가 "왜?"하고 물었다.']
    for _ in range(70):
        q = rng.choice(quoted)
        templates = ["{q}", "{s} {q}", "{q} {s}", "{s}\n{q}\n{s}", '그는 "{s}"라고 말했다. {q}', "({s}) {q}", '"{s} "{q}"', "{s} ({q}"]
        docs.append(rng.choice(templates).format(q=q, s=pick()))
    # bullets
    bullets = [["1.", "2.", "3."], ["(가)", "(나)", "(다)"], ["①", "②", "③"], ["가.", "나.", "다."], ["1)", "2)", "3)"], ["ㄱ.", "ㄴ.", "ㄷ."], ["Ⅰ.", "Ⅱ.", "Ⅲ."]]
    for _ in range(40):
        b = rng.choice(bullets)
        sep = rng.choice([" ", "\n", "\r\n"])
        docs.append(sep.join("%s %s" % (x, pick()) for x in b[:rng.randint(2, 3)]))
    # endings: ...요, z_coda, final punctuation followed by numbers
    endings = ["좋아요 정말요 그래서요.", "그래요? 맞아요! 네요", "먹었엌ㅋㅋ 그래섴ㅋ 알았어욬ㅋㅋ", "했닼ㅋㅋ 그랬짘ㅋ", "2024.01.02. 회의가 있다. 3.14는 원주율이다.",
               "가격은 1,000원. 2,000원도 있다.", "버전 1.2.3. 다음 버전은 2.0이다.", "U.S.A. 에서 왔다. Mr. Kim 이 말했다.", "끝났다... 정말 끝?!", "왜요?? 몰라요!!"]
    for _ in range(40):
        docs.append(rng.choice(["{e}", "{s} {e}", "{e}\n{s}", "{s}\n\n{e} {s}"]).format(e=rng.choice(endings), s=pick()))
    # URLs, e-mails, emoji, non-BMP characters
    specials = ["https://github.com/bab2min/Kiwi 에서 받으세요. 좋아요.", "메일은 mail@example.com 으로 보내주세요. 감사합니다.", "😀 웃었다. 😀😀 또 웃었다.",
                "👨‍👩‍👧‍👦 가족이다. 👍🏽 좋아요.", "𠀀𠀁 한자를 씁니다. 𠀂은 드문 글자다.", "🇰🇷 대한민국이다. 만세!", "#해시태그 입니다. @kiwi_bot 안녕.", "漢字 かな カナ. 섞였다."]
    for _ in range(30):
        docs.append(rng.choice(["{x}", "{s} {x}", "{x}\n{s}", "{s} {x}"]).format(x=rng.choice(specials), s=pick()))
    # empty and whitespace-only
    docs += ["", " ", "\n", "\r\n\r\n", " \t ", "　", "\v\f", "\u2028"]
    # long documents (several thousand units)
    for _ in range(5):
        parts = []
        while sum(len(p) + 1 for p in parts) < rng.randint(2000, 6000):
            parts.append(pick())
        doc = parts[0]
        for p in parts[1:]:
            doc += rng.choice(seps) + p
        docs.append(doc)
    docs.append(". ".join(["다" * 100] * 30) + ".")      # (paths overflow the first arena: retried)
    return docs


def write_docs():
    docs = make_docs()
    with open(OUT, "w", encoding="utf-8", newline="\n") as f:
        for d in docs:
            f.write(json.dumps(d, ensure_ascii=False) + "\n")
    return docs


def read_docs():
    with open(OUT, encoding="utf-8", newline="\n") as f:
        return [json.loads(l) for l in f if l.strip()]


def make_sents_golden():
    """oracle/_ref/split_sents (oracle/ref_build/tools/split_sents.cpp) over every document, Knlm and CoNg: docs_sents / cong_docs_sents"""
    refdir = os.path.join(ROOT, "oracle", "_ref")
    manifest = {"files": {}}
    subprocess.run(["make", "-C", os.path.join(ROOT, "oracle", "ref_build"), "../_ref/split_sents"], check=True)
    docs = read_docs()
    u16 = [d.encode("utf-16-le", "surrogatepass") for d in docs]
    off = [0]
    for u in u16: off.append(off[-1] + len(u) // 2)
    blob = "/tmp/docs_sents.u16"
    with open(blob, "wb") as f:
        f.write(struct.pack("<I", len(docs)) + struct.pack("<%dI" % len(off), *off) + b"".join(u16))
    for model, mtype, prefix in [("knlm_small", "knlm", ""), ("cong_small", "cong", "cong_")]:
        tmp = os.path.join("/tmp", prefix + "docs_sents.golden.txt")
        env = dict(os.environ, KIWI_ARCH_TYPE="avx2", KB_MODEL_TYPE=mtype)
        subprocess.run([os.path.join(refdir, "split_sents"), os.path.join(refdir, "models", model), blob, tmp], check=True, env=env, timeout=1200)
        data = open(tmp, "rb").read()
        with gzip.GzipFile(os.path.join(HERE, prefix + "docs_sents.golden.txt.gz"), "wb", mtime=0) as f:
            f.write(data)
        manifest["files"][prefix + "docs_sents"] = {"lines": data.count(b"\nS ") + (1 if data.startswith(b"S ") else 0), "md5": hashlib.md5(data).hexdigest()}
        manifest[prefix + "image_md5"] = hashlib.md5(open(os.path.join(refdir, "models", model + ".img"), "rb").read()).hexdigest()
    with open(os.path.join(HERE, "docs_sents.MANIFEST.json"), "w") as f:
        json.dump(manifest, f, indent=1)


if __name__ == "__main__":
    if "--golden" in sys.argv:
        make_sents_golden()
    else:
        print(len(write_docs()), "documents")
