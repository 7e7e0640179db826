"""The token-joining vector sets (tests/golden/make_join.py) and the per-rule count of the joins in them (test infrastructure)."""
import json, os
from tests.goldenio import read_golden

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MATCH_ALL_WITH_NORMALIZING = (1 << 0) | (1 << 1) | (1 << 2) | (1 << 3) | (1 << 4) | (1 << 5) | (1 << 23) | (1 << 16)
JOIN_AFFIX = 0x1F << 17
JOIN_PARTICLE_YO, MERGE_SAISIOT, COMPATIBLE_JAMO = 1 << 27, 1 << 26, 1 << 24
J1 = MATCH_ALL_WITH_NORMALIZING | JOIN_AFFIX | JOIN_PARTICLE_YO
J2 = MATCH_ALL_WITH_NORMALIZING | MERGE_SAISIOT | COMPATIBLE_JAMO
INPUTS = ["inputs_ref_tests", "inputs_web", "inputs_written", "inputs_dialect_typos"]
# vector name -> (match options, model ("knlm" / "cong"), typo set or None, input file, vectors of the same model without join options)
SETS = {}
for _n in INPUTS:
    SETS["join1_" + _n] = (J1, "knlm", None, _n, _n)
    SETS["join2_" + _n] = (J2, "knlm", None, _n, None)
for _n in ["inputs_written", "inputs_web"]:
    SETS["cong_join1_" + _n] = (J1, "cong", None, _n, "cong_" + _n)
SETS["typo6_join1_inputs_dialect_typos"] = (J1, "knlm", "basic", "inputs_dialect_typos", "typo6_inputs_dialect_typos")
SETS["join2_inputs_saisiot"] = (J2, "knlm", None, "inputs_saisiot", None)
RULES = ["noun_prefix", "noun_suffix", "verb_suffix", "adj_suffix", "adv_suffix", "saisiot", "particle_yo"]
JOINED = 0xFFFFFFFF      # (the reference's morphToId(nullptr), as goldenio reads it)
T_NNG, T_VV, T_VA, T_MAG, T_XPN, T_XSN, T_XSV, T_XSA, T_XSM, T_JX, T_EF, T_EC = 1, 4, 5, 6, 13, 14, 15, 16, 17, 46, 49, 50


def read_manifest():
    with open(os.path.join(HERE, "join.MANIFEST.json")) as f:
        return json.load(f)


def rule_counts(name):
    """rows of the vectors `name` where each rule fired.  J2 joins only NN + Z_SIOT + NN (an NNG row); a J1 row is told apart by the tags
    of the tokens it covers in the same model's vectors without join options (the affix / particle rules do not change the best path)"""
    opts, _, _, _, plain_name = SETS[name]
    counts = dict.fromkeys(RULES, 0)
    gold = read_golden(name)
    plain = read_golden(plain_name) if plain_name else None
    for i, g in enumerate(gold):
        for t in g["tokens"]:
            if t[0] != JOINED:
                continue
            if opts & MERGE_SAISIOT:
                counts["saisiot"] += 1
                continue
            parts = [p for p in plain[i]["tokens"] if t[2] <= p[2] < t[2] + t[3]]
            tags = [p[1] & 0x7F for p in parts]
            if tags and tags[0] == T_XPN: counts["noun_prefix"] += 1
            for tag in tags[1:]:
                key = {T_XSN: "noun_suffix", T_XSV: "verb_suffix", T_XSA: "adj_suffix", T_XSM: "adv_suffix", T_JX: "particle_yo"}.get(tag)
                if key: counts[key] += 1
    return counts
