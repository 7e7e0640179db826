#!/usr/bin/env python3
"""Vectors of the token-joining match options from the UNMODIFIED reference (needs oracle/_ref): the golden-vector dumper with the
match options of each set (tests/golden/dump_join.cpp, built here against oracle/_ref/libkiwi_ref.so):
  J1 = MATCH_ALL_WITH_NORMALIZING | joinAffix | joinParticleYo   Knlm over the four inputs_*.txt files, CoNg over inputs_written /
                                                                  inputs_web, the basic typo set over inputs_dialect_typos
  J2 = MATCH_ALL_WITH_NORMALIZING | mergeSaisiot | compatibleJamo  Knlm over the same four files and inputs_saisiot.txt (사이시옷
                                                                  compounds: the fabricated model joins few of them elsewhere)
The set names and options are tests/joinio.py SETS.  join.MANIFEST.json records the md5 of every vector file, the model images they
belong to and the rows where each join rule fired (tests/joinio.py rule_counts).  MANIFEST.json and the other vectors are not touched."""
import gzip, hashlib, json, os, subprocess, sys
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from tests.joinio import SETS, RULES, rule_counts      # noqa: E402

REFDIR = os.path.join(ROOT, "oracle", "_ref")
REF = os.environ.get("REF", "/root/reference")
# the reference tools' flags (oracle/ref_build/Makefile TOOLFLAGS)
TOOLFLAGS = ["-std=c++17", "-O2", "-pthread", "-fno-access-control", "-DKIWI_ARCH_X86_64=1", "-DKIWI_AVX_VNNI_SUPPORTED=1",
             "-I" + os.path.join(REF, "include"), "-I" + os.path.join(REF, "src"), "-I" + os.path.join(ROOT, "oracle", "ref_build", "shim"), "-w"]


def build_dumper():
    out = os.path.join(REFDIR, "dump_join")
    subprocess.run([os.environ.get("CXX", "g++")] + TOOLFLAGS + [os.path.join(HERE, "dump_join.cpp"), "-o", out, "-L" + REFDIR, "-lkiwi_ref",
                    "-Wl,-rpath," + REFDIR], check=True)
    return out


def main():
    dumper = build_dumper()
    manifest = {"files": {}, "rule_counts": {}}
    for name, (opts, mtype, typo, inputs, _) in SETS.items():
        tmp = os.path.join("/tmp", name + ".golden.txt")
        env = dict(os.environ, KIWI_ARCH_TYPE="avx2", KB_MODEL_TYPE=mtype, KB_MATCH=str(opts))
        if typo: env["KB_TYPO"] = typo
        model = "cong_small" if mtype == "cong" else "knlm_small"
        subprocess.run([dumper, os.path.join(REFDIR, "models", model), os.path.join(HERE, inputs + ".txt"), tmp],
                       check=True, env=env, timeout=1200)
        data = open(tmp, "rb").read()
        with gzip.GzipFile(os.path.join(HERE, name + ".golden.txt.gz"), "wb", mtime=0) as f:
            f.write(data)
        manifest["files"][name] = {"match": opts, "lines": data.count(b"\nS ") + (1 if data.startswith(b"S ") else 0), "md5": hashlib.md5(data).hexdigest()}
    for key, img in [("image_md5", "knlm_small.img"), ("cong_image_md5", "cong_small.img"), ("typo_basic_image_md5", "typo_basic.img")]:
        manifest[key] = hashlib.md5(open(os.path.join(REFDIR, "models", img), "rb").read()).hexdigest()
    total = dict.fromkeys(RULES, 0)
    for name in SETS:
        c = rule_counts(name)
        manifest["rule_counts"][name] = c
        for r in RULES: total[r] += c[r]
    manifest["rule_counts"]["total"] = total
    with open(os.path.join(HERE, "join.MANIFEST.json"), "w") as f:
        json.dump(manifest, f, indent=1)
    print(json.dumps(total))


if __name__ == "__main__":
    main()
