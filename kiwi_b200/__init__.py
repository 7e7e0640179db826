"""kiwi_b200 — Python host-side mirror of the reference's analysis interface, over the C ABI of
libkiwi_b200.so (include/kiwi_b200.h).  The compute path is the CUDA library only: there is no CPU
fallback, and importing/using this module on a box without the built extension or without a GPU fails loudly.

Mirrors (reference file:line under /root/reference/):
  Kiwi.analyze(text, top_n=1)            include/kiwi/Kiwi.h:333-400, src/Kiwi.cpp:1014-1158
  Kiwi.analyze(iterable) -> ordered list include/kiwi/Kiwi.h:402-454 (reader/receiver batch mode)
  Kiwi.split_into_sents(text)            src/Kiwi.cpp:417-450 (Kiwi::splitIntoSents)
  Token fields                           include/kiwi/Types.h:344-391 (TokenInfo)
"""
from __future__ import annotations
import ctypes as C
import os
from dataclasses import dataclass
from typing import Iterable, List, Sequence, Tuple
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("KIWI_B200_LIB", os.path.join(_HERE, "libkiwi_b200.so"))   # env override: kernel-variant experiments only

MATCH_ALL = 1 | 2 | 4 | 8 | 16 | 32 | (1 << 23)
MATCH_ALL_WITH_NORMALIZING = MATCH_ALL | (1 << 16)
# token-joining options (include/kiwi_b200.h KIWI_MATCH_*): joined tokens have morph_id JOINED_TOKEN | k, their form is BatchResult.joined_form
MATCH_JOIN_NOUN_PREFIX = 1 << 17
MATCH_JOIN_NOUN_SUFFIX = 1 << 18
MATCH_JOIN_VERB_SUFFIX = 1 << 19
MATCH_JOIN_ADJ_SUFFIX = 1 << 20
MATCH_JOIN_ADV_SUFFIX = 1 << 21
MATCH_JOIN_AFFIX = MATCH_JOIN_NOUN_PREFIX | MATCH_JOIN_NOUN_SUFFIX | MATCH_JOIN_VERB_SUFFIX | MATCH_JOIN_ADJ_SUFFIX | MATCH_JOIN_ADV_SUFFIX
MATCH_COMPATIBLE_JAMO = 1 << 24
MATCH_SPLIT_SAISIOT = 1 << 25
MATCH_MERGE_SAISIOT = 1 << 26
MATCH_JOIN_PARTICLE_YO = 1 << 27
JOINED_TOKEN = 0x80000000

TAG_NAMES = ["UN", "NNG", "NNP", "NNB", "VV", "VA", "MAG", "NR", "NP", "VX", "MM", "MAJ", "IC", "XPN", "XSN", "XSV", "XSA", "XSM", "XR",
             "VCP", "VCN", "SF", "SP", "SS", "SSO", "SSC", "SE", "SO", "SW", "SB", "SL", "SH", "SN", "W_URL", "W_EMAIL", "W_MENTION",
             "W_HASHTAG", "W_SERIAL", "W_EMOJI", "JKS", "JKC", "JKG", "JKO", "JKB", "JKV", "JKQ", "JX", "JC", "EP", "EF", "EC", "ETN", "ETM",
             "Z_CODA", "Z_SIOT", "USER0", "USER1", "USER2", "USER3", "USER4", "P", "@"]


def tag_to_string(tag: int) -> str:
    if tag & 0x80:
        return {4: "VV-I", 5: "VA-I", 9: "VX-I", 16: "XSA-I"}.get(tag & 0x7F, "@")
    return TAG_NAMES[tag] if tag < len(TAG_NAMES) else "@"


class AnalyzeOption(C.Structure):
    """kiwi_analyze_option_t, passed by value (capi.h:662-670)."""
    _fields_ = [("match_options", C.c_int), ("blocklist", C.c_void_p), ("open_ending", C.c_int), ("allowed_dialects", C.c_int),
                ("dialect_cost", C.c_float), ("typo_transformer", C.c_void_p), ("typo_threshold", C.c_float)]


def default_option(match_options: int = MATCH_ALL_WITH_NORMALIZING, typo: "PreparedTypo" = None, typo_threshold: float = 2.5, open_ending: bool = False,
                   blocklist: "MorphSet" = None) -> AnalyzeOption:
    """AnalyzeOption{match} / .withTypoTransformer(typo, typo_threshold) / .openEnding / .blocklist (include/kiwi/Kiwi.h:69-133); keep `typo` and
    `blocklist` alive while the option is used"""
    return AnalyzeOption(match_options, blocklist.handle if blocklist is not None else None, 1 if open_ending else 0, 0, 3.0,
                         typo.handle if typo is not None else None, typo_threshold)


class MorphSet:
    """kiwi_morphset_h (capi.h:36, 660, 1243-1263): a set of morphemes for AnalyzeOption::blocklist.  `add(form, tag)` resolves like
    Kiwi::findMorphemes and returns how many morphemes it added (tag None = any tag)."""

    def __init__(self, kiwi: "Kiwi"):
        self._lib = load_library()
        self.handle = self._lib.kiwi_new_morphset(kiwi._h)
        if not self.handle:
            raise KiwiError(_last_error(self._lib))

    def add(self, form: str, tag: str = None) -> int:
        n = self._lib.kiwi_morphset_add(self.handle, form.encode("utf-8"), tag.encode("ascii") if tag else None)
        if n < 0:
            raise KiwiError(_last_error(self._lib))
        return n

    def close(self):
        if getattr(self, "handle", None):
            self._lib.kiwi_morphset_close(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


TYPO_WITHOUT, TYPO_BASIC, TYPO_CONTINUAL, TYPO_BASIC_WITH_CONTINUAL, TYPO_LENGTHENING, TYPO_BASIC_WITH_CONTINUAL_AND_LENGTHENING, TYPO_DIALECT = range(7)   # capi.h:484-492


class PreparedTypo:
    """kiwi_prepared_typo_h: a prepared typo transformer resident on the device.  `PreparedTypo(path=...)` loads a flat typo image
    (include/kiwi_b200_typo.h); `PreparedTypo(default_set=TYPO_BASIC)` is kiwi_typo_prepare(kiwi_typo_get_default(set))."""

    def __init__(self, path: str = None, default_set: int = None, image_bytes: bytes = None):
        self._lib = load_library()
        if image_bytes is not None:
            buf = (C.c_char * len(image_bytes)).from_buffer_copy(image_bytes)
            self.handle = self._lib.kiwi_b200_typo_from_image(buf, len(image_bytes))
        elif path is not None:
            self.handle = self._lib.kiwi_b200_typo_load(os.fsencode(path))
        else:
            t = self._lib.kiwi_typo_get_default(TYPO_BASIC if default_set is None else default_set)
            self.handle = self._lib.kiwi_typo_prepare(t) if t else None
        if not self.handle:
            raise KiwiError(_last_error(self._lib))

    def close(self):
        if getattr(self, "handle", None):
            self._lib.kiwi_prepared_typo_close(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


TOKEN_DTYPE = np.dtype([("morph_id", "<u4"), ("position", "<u4"), ("score", "<f4"), ("length", "<u2"), ("tag", "u1"), ("flags", "u1")])


class Config(C.Structure):
    """kiwi_config_t (capi.h:72-86), passed and returned by value"""
    _fields_ = [("integrate_allomorph", C.c_uint8), ("cut_off_threshold", C.c_float), ("oov_rule_scale", C.c_float), ("oov_rule_bias", C.c_float),
                ("oov_chr_bias", C.c_float), ("oov_global_weight", C.c_float), ("oov_local_weight", C.c_float), ("oov_global_min_freq", C.c_float),
                ("space_penalty", C.c_float), ("typo_cost_weight", C.c_float), ("max_unk_form_size", C.c_uint32),
                ("max_unk_form_size_followed_by_j_class", C.c_uint32), ("space_tolerance", C.c_uint32)]


class _Batch(C.Structure):
    _fields_ = [("n_sentences", C.c_int), ("token_offsets", C.POINTER(C.c_uint32)), ("tokens", C.c_void_p), ("scores", C.POINTER(C.c_float)),
                ("status", C.POINTER(C.c_uint32)), ("ms_h2d", C.c_float), ("ms_lattice", C.c_float), ("ms_viterbi", C.c_float),
                ("ms_pack", C.c_float), ("ms_d2h", C.c_float), ("ms_total", C.c_float), ("forms", C.POINTER(C.c_uint16)), ("forms_size", C.c_uint32)]


class _Sents(C.Structure):
    _fields_ = [("n_docs", C.c_int), ("sent_offsets", C.POINTER(C.c_uint32)), ("begin", C.POINTER(C.c_uint32)), ("end", C.POINTER(C.c_uint32)),
                ("status", C.POINTER(C.c_uint32)), ("ms_h2d", C.c_float), ("ms_lattice", C.c_float), ("ms_viterbi", C.c_float),
                ("ms_sents", C.c_float), ("ms_d2h", C.c_float), ("ms_total", C.c_float)]


class Stats(C.Structure):
    _fields_ = [("n_sentences", C.c_uint64), ("raw_units", C.c_uint64), ("norm_units", C.c_uint64), ("lattice_nodes", C.c_uint64),
                ("tokens", C.c_uint64), ("paths", C.c_uint64), ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64), ("kernel_launches", C.c_uint64), ("retried", C.c_uint64),
                ("ms_lattice", C.c_float), ("ms_viterbi", C.c_float), ("ms_pack", C.c_float)]


_lib = None


def load_library() -> C.CDLL:
    """Loads libkiwi_b200.so; raises (never falls back) when the CUDA extension has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    path = os.environ.get("KIWI_B200_LIB", LIB_PATH)      # kernel experiments: another build of the same library
    if not os.path.exists(path):
        raise ImportError(f"{path} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(kiwi_b200 has no CPU fallback)")
    lib = C.CDLL(path)
    lib.kiwi_version.restype = C.c_char_p
    lib.kiwi_error.restype = C.c_char_p
    lib.kiwi_init.restype = C.c_void_p
    lib.kiwi_init.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int]
    lib.kiwi_close.argtypes = [C.c_void_p]
    lib.kiwi_b200_init_from_image.restype = C.c_void_p
    lib.kiwi_b200_init_from_image.argtypes = [C.c_void_p, C.c_uint64]
    lib.kiwi_b200_init_multi.restype = C.c_void_p
    lib.kiwi_b200_init_multi.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_int), C.c_int]
    lib.kiwi_b200_num_devices.argtypes = [C.c_void_p]
    lib.kiwi_b200_analyze_batch.restype = C.POINTER(_Batch)
    lib.kiwi_b200_analyze_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, AnalyzeOption]
    lib.kiwi_b200_batch_free.argtypes = [C.POINTER(_Batch)]
    lib.kiwi_b200_analyze_device.restype = C.c_float
    lib.kiwi_b200_analyze_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_uint64, AnalyzeOption, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    lib.kiwi_b200_last_stats.argtypes = [C.c_void_p, C.POINTER(Stats)]
    lib.kiwi_b200_debug_lattice.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, AnalyzeOption]
    lib.kiwi_b200_debug_cong.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 8
    lib.kiwi_b200_model_type.argtypes = [C.c_void_p]
    lib.kiwi_new_morphset.restype = C.c_void_p
    lib.kiwi_new_morphset.argtypes = [C.c_void_p]
    lib.kiwi_morphset_add.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
    lib.kiwi_morphset_close.argtypes = [C.c_void_p]
    lib.kiwi_get_global_config.argtypes = [C.c_void_p]
    lib.kiwi_get_global_config.restype = Config
    lib.kiwi_set_global_config.argtypes = [C.c_void_p, Config]
    lib.kiwi_set_global_config.restype = None
    lib.kiwi_b200_debug_timing.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    lib.kiwi_b200_set_device.argtypes = [C.c_int]
    lib.kiwi_b200_read_image.argtypes = [C.c_char_p, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
    lib.kiwi_b200_free.argtypes = [C.c_void_p]
    for fn in ("kiwi_typo_get_default", "kiwi_typo_get_basic", "kiwi_typo_prepare", "kiwi_b200_typo_load", "kiwi_b200_typo_from_image"):
        getattr(lib, fn).restype = C.c_void_p
    lib.kiwi_typo_get_default.argtypes = [C.c_int]
    lib.kiwi_typo_prepare.argtypes = [C.c_void_p]
    lib.kiwi_typo_close.argtypes = [C.c_void_p]
    lib.kiwi_b200_typo_load.argtypes = [C.c_char_p]
    lib.kiwi_b200_typo_from_image.argtypes = [C.c_void_p, C.c_uint64]
    lib.kiwi_prepared_typo_close.argtypes = [C.c_void_p]
    lib.kiwi_analyze_w.restype = C.c_void_p
    lib.kiwi_analyze_w.argtypes = [C.c_void_p, C.c_void_p, C.c_int, AnalyzeOption, C.c_void_p]
    lib.kiwi_res_close.argtypes = [C.c_void_p]
    lib.kiwi_res_word_num.argtypes = [C.c_void_p, C.c_int]
    lib.kiwi_res_prob.restype = C.c_float
    lib.kiwi_res_prob.argtypes = [C.c_void_p, C.c_int]
    for fn in ("kiwi_res_position", "kiwi_res_length"):
        getattr(lib, fn).argtypes = [C.c_void_p, C.c_int, C.c_int]
    lib.kiwi_res_morpheme_id.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    lib.kiwi_res_score.restype = C.c_float
    lib.kiwi_res_score.argtypes = [C.c_void_p, C.c_int, C.c_int]
    lib.kiwi_res_tag.restype = C.c_char_p
    lib.kiwi_res_tag.argtypes = [C.c_void_p, C.c_int, C.c_int]
    lib.kiwi_res_form.restype = C.c_char_p
    lib.kiwi_res_form.argtypes = [C.c_void_p, C.c_int, C.c_int]
    for fn, text_t in (("kiwi_split_into_sents_w", C.c_void_p), ("kiwi_split_into_sents", C.c_char_p)):
        getattr(lib, fn).restype = C.c_void_p
        getattr(lib, fn).argtypes = [C.c_void_p, text_t, C.c_int, C.POINTER(C.c_void_p)]
    for fn in ("kiwi_ss_size", "kiwi_ss_close"):
        getattr(lib, fn).argtypes = [C.c_void_p]
    for fn in ("kiwi_ss_begin_position", "kiwi_ss_end_position"):
        getattr(lib, fn).argtypes = [C.c_void_p, C.c_int]
    lib.kiwi_b200_split_batch.restype = C.POINTER(_Sents)
    lib.kiwi_b200_split_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    lib.kiwi_b200_sents_free.argtypes = [C.POINTER(_Sents)]
    _lib = lib
    return lib


class KiwiError(RuntimeError):
    pass


def _last_error(lib) -> str:
    e = lib.kiwi_error()
    return e.decode("utf-8", "replace") if e else "unknown error"


def encode_batch(texts: Sequence[str]) -> Tuple[np.ndarray, np.ndarray]:
    """UTF-16 blob + offsets[n+1] (the marshalling format of kiwi_b200_analyze_batch)."""
    chunks = [np.frombuffer(t.encode("utf-16-le", "surrogatepass"), dtype="<u2") for t in texts]
    offsets = np.zeros(len(texts) + 1, dtype=np.uint32)
    if chunks:
        offsets[1:] = np.cumsum([len(c) for c in chunks], dtype=np.uint64).astype(np.uint32)
    blob = np.concatenate(chunks) if chunks else np.zeros(0, dtype="<u2")
    return np.ascontiguousarray(blob), offsets


class _BatchOwner:
    """keeps the C-side batch (kiwi_b200_batch_t / kiwi_b200_sents_t) alive while numpy views of its arrays are in use"""
    def __init__(self, lib, p, free="kiwi_b200_batch_free"):
        self.lib, self.p, self.free = lib, p, free

    def __del__(self):
        try:
            if self.p:
                getattr(self.lib, self.free)(self.p); self.p = None
        except Exception:
            pass


@dataclass
class BatchResult:
    token_offsets: np.ndarray      # uint32 [n + 1]
    tokens: np.ndarray             # TOKEN_DTYPE
    scores: np.ndarray             # float32 [n]
    timings_ms: dict
    status: np.ndarray = None      # uint32 [n]: 0 = analysed; non-zero = the sentence exceeded even the escalated device capacity (no tokens)
    _owner: object = None          # the arrays above are views into the library's result buffers (no copy)
    forms: np.ndarray = None       # uint16: the joined tokens' entries (token-joining options; empty otherwise)

    def sentence(self, i: int) -> np.ndarray:
        return self.tokens[self.token_offsets[i]:self.token_offsets[i + 1]]

    def joined_form(self, i: int, k: int):
        """token k of sentence i made by a token-joining option: (form, morpheme id of its first component); None for any other token"""
        m = int(self.sentence(i)[k]["morph_id"])
        if not m & JOINED_TOKEN:
            return None
        e = m & ~JOINED_TOKEN
        end = e + 2
        while self.forms[end]:
            end += 1
        return self.forms[e + 2:end].tobytes().decode("utf-16-le", "surrogatepass"), int(self.forms[e]) | (int(self.forms[e + 1]) << 16)


@dataclass
class SentsResult:
    """kiwi_b200_split_batch: the sentence ranges of every document, [begin, end) in UTF-16 units relative to the document"""
    sent_offsets: np.ndarray       # uint32 [n + 1] into begin / end
    begin: np.ndarray              # uint32
    end: np.ndarray                # uint32
    status: np.ndarray             # uint32 [n]: 0 = analysed; non-zero = the document exceeded even the escalated device capacity (no ranges)
    timings_ms: dict
    _owner: object = None          # the arrays above are views into the library's result buffers (no copy)

    def ranges(self, i: int) -> np.ndarray:
        """(k, 2) array of document i's sentence ranges"""
        a, b = int(self.sent_offsets[i]), int(self.sent_offsets[i + 1])
        return np.stack([self.begin[a:b], self.end[a:b]], axis=1)


class Kiwi:
    """Analysis handle.  `model_path` is a kiwi_b200 model image (or a directory containing kiwi_b200.img)."""

    def __init__(self, model_path: str = None, num_threads: int = 0, device: int = None, image_bytes: bytes = None, devices: Sequence[int] = None):
        """`devices=[0, 1, ...]`: ONE handle over several GPUs of the box (kiwi_b200_init_multi): batches are sharded round-robin,
        one host thread per device, results in input order."""
        self._lib = load_library()
        if device is not None:
            self._lib.kiwi_b200_set_device(int(device))
        if devices is not None:
            if image_bytes is None:
                with open(model_path if not os.path.isdir(model_path) else os.path.join(model_path, "kiwi_b200.img"), "rb") as f:
                    image_bytes = f.read()
            buf = (C.c_char * len(image_bytes)).from_buffer_copy(image_bytes)
            arr = (C.c_int * len(devices))(*[int(d) for d in devices])
            self._h = self._lib.kiwi_b200_init_multi(C.cast(buf, C.c_void_p), len(image_bytes), arr, len(devices))
        elif image_bytes is not None:
            buf = (C.c_char * len(image_bytes)).from_buffer_copy(image_bytes)
            self._h = self._lib.kiwi_b200_init_from_image(C.cast(buf, C.c_void_p), len(image_bytes))
        else:
            self._h = self._lib.kiwi_init(os.fsencode(model_path), int(num_threads), 0, 0)
        if not self._h:
            raise KiwiError(_last_error(self._lib))

    def close(self):
        if getattr(self, "_h", None):
            self._lib.kiwi_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def analyze_batch_arrays(self, blob: np.ndarray, offsets: np.ndarray, option: AnalyzeOption = None) -> BatchResult:
        option = option or default_option()
        blob = np.ascontiguousarray(blob, dtype="<u2"); offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
        n = len(offsets) - 1
        p = self._lib.kiwi_b200_analyze_batch(self._h, blob.ctypes.data, offsets.ctypes.data, n, option)
        if not p:
            raise KiwiError(_last_error(self._lib))
        owner = _BatchOwner(self._lib, p)
        b = p.contents
        tok_off = np.ctypeslib.as_array(b.token_offsets, shape=(n + 1,))
        total = int(tok_off[n])
        if total:
            raw = (C.c_char * (total * TOKEN_DTYPE.itemsize)).from_address(b.tokens)
            tokens = np.frombuffer(raw, dtype=TOKEN_DTYPE)
        else:
            tokens = np.zeros(0, dtype=TOKEN_DTYPE)
        scores = np.ctypeslib.as_array(b.scores, shape=(n,)) if n else np.zeros(0, np.float32)
        status = np.ctypeslib.as_array(b.status, shape=(n,)) if n else np.zeros(0, np.uint32)
        tm = dict(h2d=b.ms_h2d, lattice=b.ms_lattice, viterbi=b.ms_viterbi, pack=b.ms_pack, d2h=b.ms_d2h, total=b.ms_total)
        forms = np.ctypeslib.as_array(b.forms, shape=(b.forms_size,)) if b.forms else np.zeros(0, np.uint16)
        return BatchResult(tok_off, tokens, scores, tm, status, owner, forms)

    def analyze_batch(self, texts: Sequence[str], option: AnalyzeOption = None) -> BatchResult:
        blob, offsets = encode_batch(texts)
        return self.analyze_batch_arrays(blob, offsets, option)

    def analyze(self, text, top_n: int = 1, option: AnalyzeOption = None):
        """str -> [(tokens, score)] like the reference's Kiwi::analyze; iterable of str -> list of those, in order."""
        if top_n != 1:
            raise KiwiError("kiwi_b200 implements the top_n == 1 path only")
        single = isinstance(text, str)
        texts = [text] if single else list(text)
        r = self.analyze_batch(texts, option)
        out = []
        for i, t in enumerate(texts):
            # (a token made by a token-joining option has no morpheme: -1, as the reference's morphToId(nullptr))
            toks = [(-1 if int(k["morph_id"]) & JOINED_TOKEN else int(k["morph_id"]), tag_to_string(int(k["tag"])), int(k["position"]), int(k["length"]),
                     float(k["score"])) for k in r.sentence(i)]
            out.append([(toks, float(r.scores[i]))])
        return out[0] if single else out

    def split_into_sents(self, text: str, match_options: int = MATCH_ALL_WITH_NORMALIZING, return_tokens: bool = False):
        """Kiwi::splitIntoSents: [(begin, end), ...] in UTF-16 units of `text`; with return_tokens, (ranges, tokens) where tokens is what
        analyze(text) returns for the same call (the analysis the ranges come from)."""
        u = np.ascontiguousarray(np.frombuffer((text + "\0").encode("utf-16-le", "surrogatepass"), dtype="<u2"))
        res = C.c_void_p(None)
        ss = self._lib.kiwi_split_into_sents_w(self._h, u.ctypes.data, int(match_options), C.byref(res) if return_tokens else None)
        if not ss:
            raise KiwiError(_last_error(self._lib))
        try:
            ranges = [(self._lib.kiwi_ss_begin_position(ss, i), self._lib.kiwi_ss_end_position(ss, i)) for i in range(self._lib.kiwi_ss_size(ss))]
        finally:
            self._lib.kiwi_ss_close(ss)
        if not return_tokens:
            return ranges
        try:
            lib, r = self._lib, res.value
            toks = [(lib.kiwi_res_morpheme_id(r, 0, k, None), lib.kiwi_res_tag(r, 0, k).decode("ascii"), lib.kiwi_res_position(r, 0, k),
                     lib.kiwi_res_length(r, 0, k), float(lib.kiwi_res_score(r, 0, k))) for k in range(lib.kiwi_res_word_num(r, 0))]
            return ranges, [(toks, float(lib.kiwi_res_prob(r, 0)))]
        finally:
            self._lib.kiwi_res_close(res.value)

    def split_batch(self, texts, match_options: int = MATCH_ALL_WITH_NORMALIZING) -> SentsResult:
        """kiwi_b200_split_batch over a list of documents or a (UTF-16 blob, offsets[n + 1]) pair"""
        if isinstance(texts, tuple):
            blob, offsets = texts
        else:
            blob, offsets = encode_batch(texts)
        blob = np.ascontiguousarray(blob, dtype="<u2"); offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
        n = len(offsets) - 1
        p = self._lib.kiwi_b200_split_batch(self._h, blob.ctypes.data, offsets.ctypes.data, n, int(match_options))
        if not p:
            raise KiwiError(_last_error(self._lib))
        owner = _BatchOwner(self._lib, p, "kiwi_b200_sents_free")
        b = p.contents
        off = np.ctypeslib.as_array(b.sent_offsets, shape=(n + 1,))
        total = int(off[n])
        begin = np.ctypeslib.as_array(b.begin, shape=(total,)) if total else np.zeros(0, np.uint32)
        end = np.ctypeslib.as_array(b.end, shape=(total,)) if total else np.zeros(0, np.uint32)
        status = np.ctypeslib.as_array(b.status, shape=(n,)) if n else np.zeros(0, np.uint32)
        tm = dict(h2d=b.ms_h2d, lattice=b.ms_lattice, viterbi=b.ms_viterbi, sents=b.ms_sents, d2h=b.ms_d2h, total=b.ms_total)
        return SentsResult(off, begin, end, status, tm, owner)

    def analyze_device(self, d_text_ptr: int, d_offsets_ptr: int, n: int, total_units: int, option: AnalyzeOption = None):
        """Inputs already resident in device memory (raw pointers); returns (elapsed_ms, n_tokens, launches)."""
        option = option or default_option()
        nt = C.c_uint64(0); nl = C.c_uint64(0)
        ms = self._lib.kiwi_b200_analyze_device(self._h, C.c_void_p(d_text_ptr), C.c_void_p(d_offsets_ptr), n, total_units, option, C.byref(nt), C.byref(nl))
        if ms < 0:
            raise KiwiError(_last_error(self._lib))
        return ms, nt.value, nl.value

    def last_stats(self) -> Stats:
        s = Stats()
        self._lib.kiwi_b200_last_stats(self._h, C.byref(s))
        return s

    def debug_lattice(self, text: str, option: AnalyzeOption = None, max_rows: int = 65536) -> np.ndarray:
        option = option or default_option()
        blob = np.frombuffer(text.encode("utf-16-le", "surrogatepass"), dtype="<u2")
        blob = np.ascontiguousarray(blob)
        rows = np.zeros((max_rows, 9), dtype=np.int32)
        n = self._lib.kiwi_b200_debug_lattice(self._h, blob.ctypes.data, len(blob), rows.ctypes.data, max_rows, option)
        if n < 0:
            raise KiwiError(_last_error(self._lib))
        return rows[:n].copy()

    def model_type(self) -> int:
        """(int)ModelType of the loaded image: 2 knlm, 4 cong"""
        return int(self._lib.kiwi_b200_model_type(self._h))

    def debug_cong(self, ctx, wid, node):
        """CoNg scorer self-test on the device (kiwi_b200_debug_cong): arrays of context ids, output ids and trie nodes ->
        dict(dot=int32[n], eps=float32[n,3] (scalar / small / gemv epilogue), node=int32[n], ctx=uint32[n] after one
        context-trie step, tile=int32[min(n,64), min(n,32)] from the tensor-core tile)."""
        ctx = np.ascontiguousarray(ctx, np.uint32); wid = np.ascontiguousarray(wid, np.uint32); node = np.ascontiguousarray(node, np.int32)
        n = len(ctx)
        assert len(wid) == n and len(node) == n
        dot = np.zeros(n, np.int32); eps = np.zeros((n, 3), np.float32); onode = np.zeros(n, np.int32); octx = np.zeros(n, np.uint32)
        tile = np.zeros((min(n, 64), min(n, 32)), np.int32)
        rc = self._lib.kiwi_b200_debug_cong(self._h, n, ctx.ctypes.data, wid.ctypes.data, node.ctypes.data,
                                            dot.ctypes.data, eps.ctypes.data, onode.ctypes.data, octx.ctypes.data, tile.ctypes.data)
        if rc != 0:
            raise KiwiError(_last_error(self._lib))
        return dict(dot=dot, eps=eps, node=onode, ctx=octx, tile=tile)

    def debug_timing(self, n: int) -> np.ndarray:
        """{start, end} ns (%globaltimer) of every sentence's Viterbi in the last batch launch -> uint64[n, 2]"""
        out = np.zeros((n, 2), np.uint64)
        if self._lib.kiwi_b200_debug_timing(self._h, n, out.ctypes.data) != 0:
            raise KiwiError(_last_error(self._lib))
        return out

    def get_global_config(self) -> Config:
        return self._lib.kiwi_get_global_config(self._h)

    def set_global_config(self, config: Config):
        self._lib.kiwi_set_global_config(self._h, config)
