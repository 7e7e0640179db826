/* kiwi_b200 — C ABI of the GPU-native (sm_90a) replacement for Kiwi's lattice-analysis hot path.
 *
 * The entry points below are exactly the ones the reference's FFI for this path binds
 * (/root/reference/include/kiwi/capi.h, implementation src/capi/kiwi_c.cpp); each declaration cites the
 * reference declaration it replaces.  Types are plain C: pointers, sizes, opaque handles; no torch or CUDA
 * types cross the boundary.  `kiwi_b200_*` functions are additive (batched flat-array interface, model
 * image handling, device control); everything else keeps the reference's name, argument meaning and
 * error convention (never throws across the ABI; NULL / KIWIERR_* + kiwi_error() per calling thread).
 *
 * Out of scope (SURVEY.md section 8b): builder, user-defined typo rule sets, pretokenized spans, joiner,
 * sub-word tokenizer — passing a non-NULL handle for one of those is an error.  The sentence splitter
 * (kiwi_split_into_sents[_w], kiwi_ss_*) runs its rules on the device, after the analysis.
 */
#ifndef KIWI_B200_H
#define KIWI_B200_H
#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KIWIERR_FAIL -1             /* capi.h:17 */
#define KIWIERR_INVALID_HANDLE -2   /* capi.h:18 */
#define KIWIERR_INVALID_INDEX -3    /* capi.h:19 */

#define KIWI_MATCH_URL 1
#define KIWI_MATCH_EMAIL 2
#define KIWI_MATCH_HASHTAG 4
#define KIWI_MATCH_MENTION 8
#define KIWI_MATCH_SERIAL 16
#define KIWI_MATCH_EMOJI 32
#define KIWI_MATCH_NORMALIZE_CODA (1 << 16)
#define KIWI_MATCH_JOIN_NOUN_PREFIX (1 << 17)
#define KIWI_MATCH_JOIN_NOUN_SUFFIX (1 << 18)
#define KIWI_MATCH_JOIN_VERB_SUFFIX (1 << 19)
#define KIWI_MATCH_JOIN_ADJ_SUFFIX (1 << 20)
#define KIWI_MATCH_JOIN_ADV_SUFFIX (1 << 21)
#define KIWI_MATCH_SPLIT_COMPLEX (1 << 22)
#define KIWI_MATCH_Z_CODA (1 << 23)
#define KIWI_MATCH_COMPATIBLE_JAMO (1 << 24)
#define KIWI_MATCH_SPLIT_SAISIOT (1 << 25)
#define KIWI_MATCH_MERGE_SAISIOT (1 << 26)
#define KIWI_MATCH_JOIN_PARTICLE_YO (1 << 27)
#define KIWI_MATCH_JOIN_AFFIX (KIWI_MATCH_JOIN_NOUN_PREFIX | KIWI_MATCH_JOIN_NOUN_SUFFIX | KIWI_MATCH_JOIN_VERB_SUFFIX | KIWI_MATCH_JOIN_ADJ_SUFFIX | KIWI_MATCH_JOIN_ADV_SUFFIX)
#define KIWI_MATCH_ALL (KIWI_MATCH_URL | KIWI_MATCH_EMAIL | KIWI_MATCH_HASHTAG | KIWI_MATCH_MENTION | KIWI_MATCH_SERIAL | KIWI_MATCH_EMOJI | KIWI_MATCH_Z_CODA)
#define KIWI_MATCH_ALL_WITH_NORMALIZING (KIWI_MATCH_ALL | KIWI_MATCH_NORMALIZE_CODA)

typedef struct kiwi_s* kiwi_h;                        /* capi.h:29 */
typedef struct kiwi_res* kiwi_res_h;                  /* capi.h:31 */
typedef struct kiwi_morphset* kiwi_morphset_h;        /* capi.h:36 */
typedef struct kiwi_pretokenized* kiwi_pretokenized_h;/* capi.h:37 */
typedef struct kiwi_prepared_typo* kiwi_prepared_typo_h; /* capi.h:38 */
typedef struct kiwi_typo* kiwi_typo_h;                   /* capi.h:35 */
typedef struct kiwi_ss* kiwi_ss_h;                       /* capi.h:33 */
typedef unsigned short kchar16_t;                     /* capi.h:39 */

typedef struct {                                      /* capi.h:43-61 */
	uint32_t chr_position;
	uint32_t word_position;
	uint32_t sent_position;
	uint32_t line_number;
	uint16_t length;
	uint8_t tag;
	union { uint8_t sense_id; uint8_t script; };
	float score;
	float typo_cost;
	uint32_t typo_form_id;
	uint32_t paired_token;
	uint32_t sub_sent_position;
	uint16_t dialect;
} kiwi_token_info_t;

typedef struct {                                      /* capi.h:72-86 (KiwiConfig, include/kiwi/Kiwi.h:150-167) */
	uint8_t integrate_allomorph;
	float cut_off_threshold;
	float oov_rule_scale;
	float oov_rule_bias;
	float oov_chr_bias;
	float oov_global_weight;
	float oov_local_weight;
	float oov_global_min_freq;
	float space_penalty;
	float typo_cost_weight;
	uint32_t max_unk_form_size;
	uint32_t max_unk_form_size_followed_by_j_class;
	uint32_t space_tolerance;
} kiwi_config_t;

typedef struct {                                      /* capi.h:662-670, passed BY VALUE */
	int match_options;
	kiwi_morphset_h blocklist;
	int open_ending;
	int allowed_dialects;
	float dialect_cost;
	kiwi_prepared_typo_h typo_transformer;
	float typo_threshold;
} kiwi_analyze_option_t;

typedef int (*kiwi_reader_t)(int, char*, void*);         /* capi.h:104 */
typedef int (*kiwi_reader_w_t)(int, kchar16_t*, void*);  /* capi.h:105 */
typedef int (*kiwi_receiver_t)(int, kiwi_res_h, void*);  /* capi.h:144 */

const char* kiwi_version(void);                          /* capi.h:238 */
const char* kiwi_error(void);                            /* capi.h:245 */
void kiwi_clear_error(void);                             /* capi.h:252 */

/* capi.h:599.  model_path: a directory holding `kiwi_b200.img` or the path of an image file.  num_threads sizes
 * only the host-side marshalling pool; options / enabled_dialects are recorded in the image at flatten time. */
kiwi_h kiwi_init(const char* model_path, int num_threads, int options, int enabled_dialects);
int kiwi_close(kiwi_h handle);                           /* capi.h:771 */
/* capi.h:607-615 (src/capi/kiwi_c.cpp:738-795).  The fields the hot path reads (cut-off threshold, oov rule scale / bias, space
 * penalty, typo cost weight, unknown-form size limits, space tolerance) take effect at the next launch; the chr-model oov
 * weights are stored and returned only (their match options are outside the path). */
void kiwi_set_global_config(kiwi_h handle, kiwi_config_t config);
kiwi_config_t kiwi_get_global_config(kiwi_h handle);

/* Typo-tolerant analysis (BASELINE.json config 4): kiwi_analyze_option_t::typo_transformer / typo_threshold.
 * kiwi_typo_get_default (capi.h:501; sets capi.h:484-492), kiwi_typo_get_basic (capi.h:480), kiwi_typo_prepare (capi.h:580),
 * kiwi_prepared_typo_close (capi.h:588), kiwi_typo_close (capi.h:570).  A default set is prepared by loading the flat image
 * typo_<set>.img (include/kiwi_b200_typo.h; <set> = basic, continual, ...; written by oracle/ref_build/tools/typo_tool.cpp
 * from the reference's own prepared transformer) from the directory of the model opened last, or from $KIWI_B200_TYPO_DIR;
 * kiwi_typo_init/add/copy/update/scale_cost (user-defined rule sets) are not provided.  Lengthening typo sets are refused. */
kiwi_typo_h kiwi_typo_get_default(int kiwi_typo_set);
kiwi_typo_h kiwi_typo_get_basic(void);
int kiwi_typo_close(kiwi_typo_h handle);
kiwi_prepared_typo_h kiwi_typo_prepare(kiwi_typo_h handle);
int kiwi_prepared_typo_close(kiwi_prepared_typo_h handle);

/* ---- morpheme sets: kiwi_analyze_option_t::blocklist (capi.h:660, 1243-1263; src/capi/kiwi_c.cpp:851-864, 1780-1825) --------------
 * kiwi_morphset_add[_w] resolves (form, tag) like Kiwi::findMorphemes (src/Kiwi.cpp:1281-1297; tag NULL = any tag) and returns the number
 * of morphemes added; the analysis skips every candidate for which Morpheme::hasMorpheme(blocklist) holds (src/PathEvaluator.hpp:385). */
kiwi_morphset_h kiwi_new_morphset(kiwi_h handle);
int kiwi_morphset_add(kiwi_morphset_h handle, const char* form, const char* tag);
int kiwi_morphset_add_w(kiwi_morphset_h handle, const kchar16_t* form, const char* tag);
int kiwi_morphset_close(kiwi_morphset_h handle);
/* additive: a prepared transformer straight from a flat typo image (file / memory) */
kiwi_prepared_typo_h kiwi_b200_typo_load(const char* typo_image_path);
kiwi_prepared_typo_h kiwi_b200_typo_from_image(const void* bytes, size_t size);

kiwi_res_h kiwi_analyze_w(kiwi_h handle, const kchar16_t* text, int top_n, kiwi_analyze_option_t option, kiwi_pretokenized_h pretokenized);  /* capi.h:684 */
kiwi_res_h kiwi_analyze(kiwi_h handle, const char* text, int top_n, kiwi_analyze_option_t option, kiwi_pretokenized_h pretokenized);        /* capi.h:698 */
int kiwi_analyze_mw(kiwi_h handle, kiwi_reader_w_t reader, kiwi_receiver_t receiver, void* user_data, int top_n, kiwi_analyze_option_t option); /* capi.h:711 */
int kiwi_analyze_m(kiwi_h handle, kiwi_reader_t reader, kiwi_receiver_t receiver, void* user_data, int top_n, kiwi_analyze_option_t option);   /* capi.h:724 */

int kiwi_res_size(kiwi_res_h result);                                        /* capi.h:788 */
float kiwi_res_prob(kiwi_res_h result, int index);                           /* capi.h:797 */
int kiwi_res_word_num(kiwi_res_h result, int index);                         /* capi.h:806 */
const kiwi_token_info_t* kiwi_res_token_info(kiwi_res_h result, int index, int num); /* capi.h:816 */
int kiwi_res_morpheme_id(kiwi_res_h result, int index, int num, kiwi_h kiwi_handle); /* capi.h:827 */
const kchar16_t* kiwi_res_form_w(kiwi_res_h result, int index, int num);     /* capi.h:837 */
const kchar16_t* kiwi_res_tag_w(kiwi_res_h result, int index, int num);      /* capi.h:847 */
const char* kiwi_res_form(kiwi_res_h result, int index, int num);            /* capi.h:857 */
const char* kiwi_res_tag(kiwi_res_h result, int index, int num);             /* capi.h:867 */
int kiwi_res_position(kiwi_res_h result, int index, int num);                /* capi.h:877 */
int kiwi_res_length(kiwi_res_h result, int index, int num);                  /* capi.h:887 */
int kiwi_res_word_position(kiwi_res_h result, int index, int num);          /* capi.h:897 */
int kiwi_res_sent_position(kiwi_res_h result, int index, int num);          /* capi.h:907 */
float kiwi_res_score(kiwi_res_h result, int index, int num);                 /* capi.h:917 */
float kiwi_res_typo_cost(kiwi_res_h result, int index, int num);             /* capi.h:927 */
int kiwi_res_close(kiwi_res_h result);                                       /* capi.h:937 */

/* ---- sentence splitting: Kiwi::splitIntoSents (src/Kiwi.cpp:417-450, src/capi/kiwi_c.cpp:973-1009, 1660-1720) ------------------
 * The text is analysed top-1 with match_options (checked like kiwi_analyze_option_t::match_options) and its sentences are found on the
 * device from the token rows (sentence rules: fillSentLineInfo, src/Kiwi.cpp:322-415).  Ranges are [begin, end) in UTF-16 units of the
 * text (kiwi_split_into_sents_w) or in bytes of the UTF-8 text (kiwi_split_into_sents).  tokenized_res (may be NULL) receives the
 * analysis the ranges come from, equal to what kiwi_analyze_w(text, 1, {match_options}) returns.  NULL handle: NULL; otherwise
 * NULL + kiwi_error() on failure.  A text that overflows even the retry capacity has no tokens and no sentence. */
kiwi_ss_h kiwi_split_into_sents_w(kiwi_h handle, const kchar16_t* text, int match_options, kiwi_res_h* tokenized_res);   /* capi.h:738 */
kiwi_ss_h kiwi_split_into_sents(kiwi_h handle, const char* text, int match_options, kiwi_res_h* tokenized_res);          /* capi.h:752 */
int kiwi_ss_size(kiwi_ss_h result);                                          /* capi.h:1166; KIWIERR_INVALID_HANDLE on NULL */
int kiwi_ss_begin_position(kiwi_ss_h result, int index);                     /* capi.h:1175; KIWIERR_INVALID_INDEX out of range */
int kiwi_ss_end_position(kiwi_ss_h result, int index);                       /* capi.h:1184 */
int kiwi_ss_close(kiwi_ss_h result);                                         /* capi.h:1194 */

/* ---- additive batched interface (flat arrays; what kiwi_analyze_mw drains into) -------------------- */
/* A token the token-joining options (KIWI_MATCH_JOIN_*, KIWI_MATCH_MERGE_SAISIOT, KIWI_MATCH_JOIN_PARTICLE_YO; joinAffixTokens,
 * src/Kiwi.cpp:495-588) made of several has no morpheme: its morph_id is KIWI_B200_JOINED_TOKEN | k, where k indexes the batch's
 * `forms` array (morpheme ids stay far below 2^31).  The entry at forms[k] is
 *   forms[k], forms[k + 1]   the morpheme id of the token's FIRST component, low 16 bits then high 16 bits (its sense_id and dialect)
 *   forms[k + 2] ...         the joined form (TokenInfo::str: joinHangul per component, compatibility jamo with KIWI_MATCH_COMPATIBLE_JAMO,
 *                            coda ㅅ for a merged 사이시옷), terminated by 0.
 * The row keeps its first component's position, score and flags; its length reaches to the end of its last component. */
#define KIWI_B200_JOINED_TOKEN 0x80000000u
typedef struct {
	uint32_t morph_id;      /* morphToId(PathNode.morph) after unifyMorpheme (PathEvaluator.hpp:1054-1058), or KIWI_B200_JOINED_TOKEN | k */
	uint32_t position;      /* original UTF-16 units (Kiwi.cpp:734-737) */
	float score;            /* PathNode.wordScore */
	uint16_t length;
	uint8_t tag;            /* POSTag incl. the irregular bit, after script re-tagging (Kiwi.cpp:590-605) */
	uint8_t flags;          /* bit0: the token carries its own surface form (OOV / special run / pattern);
	                         * bits 1-3: typo cost of the token's lattice node in units of 0.5, bits 4-7: tokens of that node - 1;
	                         * TokenInfo::typoCost = cost / tokens (0 without a typo transformer) */
} kiwi_b200_token_t;

typedef struct {
	int n_sentences;
	const uint32_t* token_offsets;      /* [n_sentences + 1] into tokens */
	const kiwi_b200_token_t* tokens;
	const float* scores;                /* top-1 path score per sentence (sum over chunks, Kiwi.cpp:759) */
	const uint32_t* status;             /* 0 = ok */
	/* device timing of the last call, milliseconds (CUDA events on the engine's stream) */
	float ms_h2d, ms_lattice, ms_viterbi, ms_pack, ms_d2h, ms_total;
	/* the joined tokens' entries (see KIWI_B200_JOINED_TOKEN), forms_size UTF-16 units; NULL when the call had no token-joining option
	 * (or nothing joined).  KIWI_MATCH_COMPATIBLE_JAMO applies to these forms; forms a caller builds itself from the text or the
	 * morphemes are the caller's to convert. */
	const kchar16_t* forms;
	uint32_t forms_size;
} kiwi_b200_batch_t;

/* Analyze n sentences given as one UTF-16 blob + offsets[n+1].  Returns NULL and sets kiwi_error() on failure
 * (including any sentence that overflowed even the retry capacity).  Free with kiwi_b200_batch_free. */
const kiwi_b200_batch_t* kiwi_b200_analyze_batch(kiwi_h handle, const kchar16_t* text, const uint32_t* offsets, int n, kiwi_analyze_option_t option);
void kiwi_b200_batch_free(const kiwi_b200_batch_t* batch);

/* Additive: the sentence ranges of n documents (one UTF-16 blob + offsets[n+1], as kiwi_b200_analyze_batch takes them).  Only the
 * ranges come back from the device, not the token rows.  Document i's ranges are [sent_offsets[i], sent_offsets[i+1]) of begin / end,
 * UTF-16 units relative to the document; a document with a non-zero status has none.  ms_sents: the sentence kernels.  NULL +
 * kiwi_error() on failure.  Free with kiwi_b200_sents_free. */
typedef struct {
	int n_docs;
	const uint32_t* sent_offsets;       /* [n_docs + 1] into begin / end */
	const uint32_t* begin;              /* UTF-16 units, relative to the document */
	const uint32_t* end;
	const uint32_t* status;             /* 0 = ok */
	float ms_h2d, ms_lattice, ms_viterbi, ms_sents, ms_d2h, ms_total;
} kiwi_b200_sents_t;
const kiwi_b200_sents_t* kiwi_b200_split_batch(kiwi_h handle, const kchar16_t* text, const uint32_t* offsets, int n, int match_options);
void kiwi_b200_sents_free(const kiwi_b200_sents_t* sents);

/* Same work with inputs already resident in device memory (used by bench.py's device-resident leg). The
 * text / offsets pointers are DEVICE pointers; results stay on the device; returns elapsed device ms or < 0. */
float kiwi_b200_analyze_device(kiwi_h handle, const void* d_text, const void* d_offsets, int n, uint64_t total_units, kiwi_analyze_option_t option, uint64_t* out_tokens, uint64_t* out_launches);

/* Counters of the last batch (for the roofline arithmetic): kernel times, launches, bytes moved. */
typedef struct {
	uint64_t n_sentences, raw_units, norm_units, lattice_nodes, tokens, paths;
	uint64_t h2d_bytes, d2h_bytes, kernel_launches;
	uint64_t retried;          /* sentences that overflowed the first-pass scratch and went through the larger arena */
	float ms_lattice, ms_viterbi, ms_pack;
} kiwi_b200_stats_t;
int kiwi_b200_last_stats(kiwi_h handle, kiwi_b200_stats_t* out);

/* Lattice of one sentence (stage-level parity tests): nodes as 9 x int32 rows
 * {form, uform_off|-1, uform_len, prev, sibling, start, end, space_errors, chunk}.  Returns node count or < 0. */
int kiwi_b200_debug_lattice(kiwi_h handle, const kchar16_t* text, int len, int32_t* out_rows, int max_rows, kiwi_analyze_option_t option);

/* CoNg scorer self-test on the device (stage-level parity tests of the int8 scorer, SURVEY.md 8a rows a14/a15): for n
 * (context id, output id, trie node) triples returns the integer dot product minus hsum (dp4a path), the three float
 * epilogues (scalar / small / gemv association, src/qgemm.hpp:68-80, src/archImpl/avx2_qgemm.hpp:124,435), the context
 * trie transition (src/CoNgramModel.hpp:271-385) and, in out_tile[min(n,64) x min(n,32)], the same integers computed by
 * the tensor-core tile (mma.sync m16n8k32 u8 x s8) over the first contexts x first output ids. */
int kiwi_b200_debug_cong(kiwi_h handle, int n, const uint32_t* ctx, const uint32_t* wid, const int32_t* node,
	int32_t* out_dot, float* out_eps, int32_t* out_node, uint32_t* out_ctx, int32_t* out_tile);
int kiwi_b200_model_type(kiwi_h handle);
/* Diagnostics: {start, end} of every sentence's Viterbi in the last batch launch, %globaltimer ns, out[2 * n]. */
int kiwi_b200_debug_timing(kiwi_h handle, int n, uint64_t* out_start_end_ns);         /* (int)ModelType of the loaded image: 2 knlm, 4 cong */

int kiwi_b200_device_count(void);
int kiwi_b200_set_device(int device);            /* call before kiwi_init; default: current device */
/* raw model image access so a launcher can broadcast it (NCCL) and hand it to every rank */
int kiwi_b200_read_image(const char* model_path, void** out_bytes, uint64_t* out_size);   /* malloc'ed */
kiwi_h kiwi_b200_init_from_image(const void* bytes, uint64_t size);
/* One handle over several GPUs of one box: the read-only model is made resident on every listed device; kiwi_analyze_m[w] and
 * kiwi_b200_analyze_batch shard each batch round-robin (sentence i -> devices[i mod n]), one host thread per device, and deliver
 * results in input order (the reference's ordered pool, include/kiwi/Kiwi.h:402-454).  No collective in steady state. */
kiwi_h kiwi_b200_init_multi(const void* bytes, uint64_t size, const int* devices, int n_devices);
int kiwi_b200_num_devices(kiwi_h handle);
void kiwi_b200_free(void* p);

/* ---- native model loading, first pieces (SURVEY 8f-2) -------------------------------------------------------------------------
 * Read the reference's language-model FILES without the reference library and return the corresponding sections of the model image
 * (kiwi_b200_image.h) - byte for byte what oracle/ref_build/tools/flatten_model.cpp dumps from the reference's in-memory model:
 *   sj.knlm         KnLangModel constructor, /root/reference/src/Knlm.hpp:1003-1167 (header include/kiwi/Knlm.h:10-16)
 *   skipbigram.mdl  SkipBigramModel constructor, src/SkipBigramModel.hpp:40-105 (header include/kiwi/SkipBigramModel.h:9-13)
 * out: a malloc'ed blob that starts with the struct below; offsets are from the blob's start; release with kiwi_b200_free.
 * Returns 0, or -1 with a message in kiwi_b200_native_error().  Host code only (no GPU needed). */
typedef struct kiwi_b200_native_knlm_t {
	uint32_t num_nodes, num_edges, htx_vocab, has_htx, order, vocab_size;   /* = kb2_header kn_* / lang_vocab_size */
	int32_t  bos_node; float unk_ll;
	uint64_t nodes_off, nodes_bytes;     /* KB2_SEC_KN_NODES  kb2_kn_node[num_nodes] */
	uint64_t keys_off, keys_bytes;       /* KB2_SEC_KN_KEYS   uint32_t[num_edges]    */
	uint64_t values_off, values_bytes;   /* KB2_SEC_KN_VALUES int32_t[num_edges]     */
	uint64_t root_off, root_bytes;       /* KB2_SEC_KN_ROOT   int32_t[htx_vocab]     */
	uint64_t htx_off, htx_bytes;         /* KB2_SEC_KN_HTX    uint32_t[vocab_size] or empty */
} kiwi_b200_native_knlm_t;
typedef struct kiwi_b200_native_sbg_t {
	uint32_t vocab_size, window_size, num_pairs, pad;                       /* = kb2_header sb_* */
	uint64_t ptrs_off, ptrs_bytes;       /* KB2_SEC_SB_PTRS    uint32_t[vocab_size + 1] */
	uint64_t keys_off, keys_bytes;       /* KB2_SEC_SB_KEYS    uint32_t[num_pairs]      */
	uint64_t comps_off, comps_bytes;     /* KB2_SEC_SB_COMPS   float[num_pairs]         */
	uint64_t discnts_off, discnts_bytes; /* KB2_SEC_SB_DISCNTS float[vocab_size]        */
	uint64_t valid_off, valid_bytes;     /* KB2_SEC_SB_VALID   uint8_t[vocab_size]      */
} kiwi_b200_native_sbg_t;
typedef struct kiwi_b200_native_cong_t {
	uint32_t num_nodes, num_edges, root_size, dim, context_size, key_size, flags, vocab_size;   /* = kb2_header cg_* / lang_vocab_size */
	uint64_t nodes_off, nodes_bytes;         /* KB2_SEC_CG_NODES     kb2_cg_node[num_nodes] */
	uint64_t keys_off, keys_bytes;           /* KB2_SEC_CG_KEYS      uint32_t[num_edges]    */
	uint64_t values_off, values_bytes;       /* KB2_SEC_CG_VALUES    int32_t[num_edges]     */
	uint64_t root_off, root_bytes;           /* KB2_SEC_CG_ROOT      int32_t[root_size]     */
	uint64_t ctx_emb_off, ctx_emb_bytes;     /* KB2_SEC_CG_CTX_EMB   */
	uint64_t out_emb_off, out_emb_bytes;     /* KB2_SEC_CG_OUT_EMB   */
	uint64_t inv_vocab_off, inv_vocab_bytes; /* KB2_SEC_CG_INV_VOCAB (may be empty) */
	uint64_t out_bias_off, out_bias_bytes;   /* KB2_SEC_CG_OUT_BIAS  (may be empty) */
} kiwi_b200_native_cong_t;
int kiwi_b200_native_knlm(const char* sj_knlm_path, void** out_bytes, uint64_t* out_size);
/*   cong.mdl        CoNgramModel<..., windowSize 0, quantized> constructor, src/CoNgramModel.cpp:425-790 (8-bit embedding rows) */
int kiwi_b200_native_cong(const char* cong_mdl_path, void** out_bytes, uint64_t* out_size);
int kiwi_b200_native_sbg(const char* skipbigram_mdl_path, void** out_bytes, uint64_t* out_size);
/* host-only helper behind kiwi_morphset_add (no GPU needed): the morpheme ids (form, tag) resolves to in a model image; returns the count
 * (at most `cap` ids are written), -1 on error */
int kiwi_b200_image_find_morphemes(const void* image_bytes, uint64_t size, const kchar16_t* form, const char* tag, uint32_t* out_ids, int cap);
const char* kiwi_b200_native_error(void);

#ifdef __cplusplus
}
#endif
#endif
