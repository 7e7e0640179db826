// kiwi_b200: device-resident model view and the derived per-morpheme / per-form feature words.
//
// The read-only model lives in HBM as one contiguous copy of the image file (include/kiwi_b200_image.h)
// followed by tables derived once on the host at load time (model.cpp).  The derived tables turn the
// string-chasing predicates of the reference's rule scorer into single 4..16-byte loads:
//   RuleBasedScorer ctor / operator()   /root/reference/src/PathEvaluator.hpp:88-184
//   FormEvaluator                       /root/reference/src/PathEvaluator.hpp:253-311
//   FeatureTestor::isMatched            /root/reference/src/FeatureTestor.cpp:6-80
#pragma once
#include <stdint.h>
#include "../../include/kiwi_b200_image.h"
#include "kb_batch.h"

#if defined(__CUDACC__)
#define KB_HD __host__ __device__ __forceinline__
#else
#define KB_HD inline
#endif

namespace kb
{
	// POSTag values of the reference (include/kiwi/Types.h:195-227)
	enum Tag : uint8_t
	{
		T_unknown = 0, T_nng, T_nnp, T_nnb, T_vv, T_va, T_mag, T_nr, T_np, T_vx, T_mm, T_maj, T_ic,
		T_xpn, T_xsn, T_xsv, T_xsa, T_xsm, T_xr, T_vcp, T_vcn,
		T_sf, T_sp, T_ss, T_sso, T_ssc, T_se, T_so, T_sw, T_sb, T_sl, T_sh, T_sn,
		T_w_url, T_w_email, T_w_mention, T_w_hashtag, T_w_serial, T_w_emoji,
		T_jks, T_jkc, T_jkg, T_jko, T_jkb, T_jkv, T_jkq, T_jx, T_jc,
		T_ep, T_ef, T_ec, T_etn, T_etm, T_z_coda, T_z_siot,
		T_user0, T_user1, T_user2, T_user3, T_user4, T_p, T_max,
	};
	enum { CV_none = 0, CV_any, CV_vowel, CV_vocalic, CV_vocalic_h, CV_non_vowel, CV_non_vocalic, CV_non_vocalic_h, CV_applosive };
	enum { CP_none = 0, CP_positive, CP_negative, CP_non_adj };

	KB_HD uint8_t clearIrregular(uint8_t t) { return t & 0x7F; }
	KB_HD bool isIrregular(uint8_t t) { return (t & 0x80) != 0; }
	KB_HD bool isEClass(uint8_t t) { return T_ep <= t && t <= T_etm; }
	KB_HD bool isJClass(uint8_t t) { return T_jks <= t && t <= T_jc; }
	KB_HD bool isNNClass(uint8_t t) { return T_nng <= t && t <= T_nnb; }
	KB_HD bool isVerbClass(uint8_t t)
	{
		t = clearIrregular(t);
		return t == T_vv || t == T_va || t == T_vx || t == T_xsv || t == T_xsa || t == T_vcp || t == T_vcn;
	}
	KB_HD bool isHangulSyllable(uint32_t c) { return 0xAC00 <= c && c < 0xD7A4; }
	KB_HD bool isHangulCoda(uint32_t c) { return 0x11A8 <= c && c < 0x11A8 + 27; }
	KB_HD bool isHighSurrogate(uint32_t c) { return (c & 0xFC00) == 0xD800; }
	// Match::compatibleJamo: a conjoining consonant becomes its Hangul Compatibility Jamo (U+3131-314E, the 30 consonants ㄱ..ㅎ in
	// Unicode order).  The 19 choseong U+1100-1112 are the compatibility consonants without the 11 clusters ㄳ ㄵ ㄶ ㄺ-ㅀ ㅄ; the 27
	// jongseong U+11A8-11C2 are the compatibility consonants without the 3 that never close a syllable, ㄸ ㅃ ㅉ.  Others: unchanged.
	KB_HD uint32_t nthSetBit(uint32_t mask, uint32_t n)
	{
		uint32_t j = 0;
		for (;; ++j) if ((mask >> j) & 1) { if (!n) break; --n; }
		return j;
	}
	KB_HD uint16_t toCompatibleJamo(uint16_t c)
	{
		constexpr uint32_t all = (1u << 30) - 1;
		constexpr uint32_t onsets = all & ~((1u << 2) | (1u << 4) | (1u << 5) | (0x7Fu << 9) | (1u << 19));
		constexpr uint32_t codas = all & ~((1u << 7) | (1u << 18) | (1u << 24));
		if (0x1100 <= c && c < 0x1113) return (uint16_t)(0x3131 + nthSetBit(onsets, c - 0x1100u));
		if (0x11A8 <= c && c < 0x11C3) return (uint16_t)(0x3131 + nthSetBit(codas, c - 0x11A8u));
		return c;
	}
	KB_HD uint32_t mergeSurrogate(uint32_t h, uint32_t l) { return (((h & 0x3FF) << 10) | (l & 0x3FF)) + 0x10000; }

	// ---- morpheme feature word (DMorph::feat)
	enum : uint32_t
	{
		MF_TAG_MASK = 0xFFu,
		MF_VERB = 1u << 8,            // isVerbClass(tag)
		MF_INFL_NP = 1u << 9,         // isInflectendaNP          PathEvaluator.hpp:46-50
		MF_VERB_L = 1u << 10,         // isVerbL                  :58-61
		MF_POS_VERB = 1u << 11,       // isPositiveVerb           :69-72
		MF_VERB_VOWEL = 1u << 12,     // isVerbVowel              :79-82
		MF_SPECIAL_SHIFT = 13,        // 3 bits: Kiwi::SpecialMorph 0..5, 7 = none
		MF_SBTYPE_SHIFT = 16,         // 5 bits: getSBType() for SB morphemes
		MF_VOWEL_E = 1u << 21,
		MF_INF_J = 1u << 22,
		MF_BADPAIR_L = 1u << 23,
		MF_CONTRACT_E = 1u << 24,
		MF_SINGLE = 1u << 25,         // Morpheme::isSingle       Form.h:174
		MF_POLAR_SHIFT = 26,          // 2 bits CondPolarity
		MF_VOWEL_SHIFT = 28,          // 4 bits CondVowel
	};

	enum : uint32_t { MM_COMPLEX = 1u, MM_SAISIOT = 2u, MM_KFORM_YO = 4u };      // MM_KFORM_YO: kform is "요" (the sentence splitter's jx-요 rule)
	struct alignas(16) DMorph             // 32 B, one vector load
	{
		uint32_t feat;
		uint32_t lm_id;       // lmMorphemeId
		int32_t combined;     // relative index of the combined morpheme
		uint32_t chunk_off;
		float user_score;
		int32_t form_idx;     // kform
		uint8_t chunk_cnt, combine_socket, sense_id, nonstd_dialect;
		uint32_t misc;        // MM_* bits
	};

	// static per-candidate data of evalSingleMorpheme (PathEvaluator.hpp:531-556) and of the path it creates
	enum : uint8_t { MX_FIRST_IS_P = 1, MX_CHUNK_HAS_P = 2 };
	struct alignas(16) DMorphX            // 16 B
	{
		uint32_t first_wid;       // isSingle ? lmMorphemeId : chunks[0]->lmMorphemeId
		uint32_t last_seq_id;     // `lastSeqId` = wid of the created path
		uint32_t last_seq_feat;   // DMorph::feat of morphemes[last_seq_id]
		uint32_t fw_x;            // bits 0-23: filter word (kb_batch.h FW_*) of the created path when it has no own form, without FW_COMMON_ROOT; bits 24-31: MX_*
	};

	// Static record of ONE candidate entry of a form (parallel to form_cands[], + 2 trailing records for the default unknown
	// morphemes NNG / NNP): everything PathEvaluator::operator() and evalSingleMorpheme derive from the candidate morpheme alone
	// (PathEvaluator.hpp:382-448, 531-560, RuleBasedScorer ctor 88-113), resolved at model load.  The candidates of a form are
	// contiguous, so a lattice node's candidate block is ONE bulk copy (cp.async.bulk) into shared memory.
	enum : uint8_t
	{
		DK_DIALECT = 1,           // non-standard dialect morpheme: never a candidate
		DK_COMPLEX = 2,           // hasComplex(): dropped when Match::splitComplex
		DK_SHORTCUT_CODA = 4, DK_SHORTCUT_SIOT = 8,
		DK_HA = 16,               // contracted 하+다/게/지: dropped after a space (PathEvaluator.hpp:435-448)
		DK_FIRST_IS_P = 32, DK_CHUNK_HAS_P = 64,
		DK_IS_SN = 128,           // tag SN: snEndswithPoint is decided per node
	};
	enum : uint8_t { CS_POSITIVE_E = 1, CS_SN_POINT = 2, CS_SINGLE = 4, CS_NO_LM = 8, CS_FORK = 16, CS_SOCKET_CHUNK = 32 };
	struct alignas(16) DCand              // 48 B
	{
		int32_t cur_id; uint32_t first_wid; uint32_t last_seq_id; uint32_t last_seq_feat;
		uint32_t feat; float user_score; uint32_t chunk_off;
		uint32_t fw_new;          // filter word of the created path (no own form, FW_COMMON_ROOT clear)
		uint8_t chunk_cnt;
		uint8_t flags;            // CS_* known statically (CS_POSITIVE_E uses the form's first character)
		uint8_t path_socket;      // combineSocket of the created path (single morphemes only)
		uint8_t sense_id;
		uint8_t cur_socket;       // the morpheme's own combine socket
		uint8_t kind;             // DK_*
		uint8_t tag_clean;        // clearIrregular(tag): index into tag_left_boundary
		uint8_t pad0;
		uint32_t pad1[2];
	};
	static_assert(sizeof(DCand) == 48, "DCand rows are bulk-copied: a multiple of 16 bytes");

	// ---- form feature record
	enum : uint8_t
	{
		FF_ZCODA = 1, FF_ZSIOT = 2, FF_HASFULL = 8,
		FF_HAS_SPECIAL = 4,       // a candidate is a z_coda / z_siot shortcut or a forking (quote / bullet) morpheme: the node takes the general evaluation path
		FF_HASJ_OR_STAG = 16,     // form.hasJClass || (len == 1 && sf <= cls(form[0]) <= sw)     KTrie.cpp:970-972
		FF_FIRST_IS_CODA = 32,    // isHangulCoda(form[0])                                       KTrie.cpp:968
		FF_ALL_PARTIAL = 64,      // every candidate is combineSocket or chunked non-single      PathEvaluator.hpp:1277-1280
		FF_FIRST_IS_A = 128,      // form[0] == '아' (positiveE)                                 PathEvaluator.hpp:104
	};
	enum : uint8_t
	{
		FP_POLAR_POS = 1,         // FeatureTestor::isMatched(form, CondPolarity::positive)
		FP_POLAR_NEG = 2,         // FeatureTestor::isMatched(form, CondPolarity::negative)
		FP_LAST_SSC = 4,          // identifySpecialChr(form.back()) == ssc
	};
	struct alignas(16) DForm              // 16 B
	{
		uint32_t cand_off;
		uint16_t cand_cnt;
		uint16_t str_len;
		uint16_t size_no_space;   // sizeWithoutSpace()
		uint16_t last_chr;        // 0 when empty
		uint16_t num_spaces;
		uint8_t flags;            // FF_*
		uint8_t pol;              // FP_*
	};

	struct DevModel           // passed to kernels by value
	{
		// raw image sections (device pointers)
		const kb2_trie_node* trie_nodes;
		const uint16_t* trie_keys;
		const int32_t* trie_diffs;
		const kb2_form* forms_raw;
		const uint16_t* form_chars;
		const uint32_t* form_cands;
		const kb2_chunk* chunks;
		const kb2_kn_node* kn_nodes;
		const uint32_t* kn_keys;
		const int32_t* kn_values;
		const int32_t* kn_root;
		const uint32_t* kn_htx;        // nullptr when absent
		const kb2_chr_run* chr_runs;
		// derived
		const DMorph* morphs;
		const DMorphX* morphx;
		const DCand* cands;            // [n_form_cands + 2]: static candidate records parallel to form_cands, then the unknown NNG / NNP records
		uint32_t cand_unk;             // index of the NNG record (NNP follows)
		const uint32_t* chunk_lm;      // lmMorphemeId of every chunk entry (parallel to `chunks`)
		const DForm* forms;
		const uint32_t* chr_bmp;       // [65536] cls | script << 8 | flags << 16
		const int32_t* trie_root_next; // [65536] child node index of the root, -1 = none
		// Knlm re-laid out for one-probe child lookup (model.cu): open-addressing table over all non-root edges,
		// entry = {node, token, value, ll of the child node}; per-node backoff pair; root children via direct tables
		const uint4* kn_hash; uint32_t kn_hash_mask;
		const float2* kn_backoff;      // [node] {lower as int bits, gamma}
		const float* kn_root_ll;       // [htx_vocab] ll of the root's child for token t (valid when kn_root[t] > 0)
		// CoNg (model_type cong; all null / 0 for Knlm images).  Context trie re-laid out like the Knlm one: one
		// open-addressing table over all non-root edges, entry = {node, key, value, contextIdx of the child node};
		// per-node {lower, value}; root children via the direct table.  Embedding rows stay in the image layout
		// (src/CoNgramModel.hpp:89-105): context row = u8[dim] (s8 + 128), float scale, float bias;
		// output row = s8[dim], float scale, int32 hsum.
		const uint4* cg_hash; uint32_t cg_hash_mask;
		const int2* cg_nodes;          // [node] {lower, value (= contextIdx)}
		const int32_t* cg_root;        // [cg_root_size]
		const uint8_t* cg_ctx_emb;
		const uint8_t* cg_out_emb;
		const uint32_t* cg_inv_vocab;  // nullptr when absent
		const float* cg_out_bias;      // nullptr when absent
		uint32_t cg_dim, cg_stride, cg_key_size, cg_root_size, cg_context_size;
		// SkipBigram (model_type sbg; null / 0 otherwise): the image sections as they are (src/SkipBigramModel.hpp:24-32) - per target token a
		// sorted list of history tokens with their compensations, per token a discount and the validity flag
		const uint32_t* sb_ptrs; const uint32_t* sb_keys; const float* sb_comps; const float* sb_discnts; const uint8_t* sb_valid;
		uint32_t sb_vocab_size; float sb_log_window;
		uint32_t model_type;           // (int)ModelType: 2 knlm, 3 sbg, 4 cong
		// scalars
		uint32_t n_chr_runs, n_morphs, n_forms, n_trie_nodes;
		uint32_t default_tag_size, lang_vocab_size;
		uint32_t script_latin, script_variation_selectors;
		uint32_t kn_root_num_nexts;
		uint32_t kn_htx_vocab;
		uint32_t* debug;               // [64] anomaly record (diagnostics)
		int32_t kn_bos_node;
		float kn_unk_ll;
		uint32_t special_morph_ids[6];
		kb2_config cfg;
		float tag_left_boundary[2][KB2_POSTAG_MAX];
	};

	// code-point attributes: cls = identifySpecialChr, script = chr2ScriptType, flags = KB2_CHR_*
	KB_HD uint32_t chrAttr(const DevModel& m, uint32_t c)
	{
		if (c < 0x10000) return m.chr_bmp[c];
		uint32_t lo = 0, hi = m.n_chr_runs;
		while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (m.chr_runs[mid].start <= c) lo = mid; else hi = mid; }
		const kb2_chr_run r = m.chr_runs[lo];
		return (uint32_t)r.cls | ((uint32_t)r.script << 8) | ((uint32_t)r.flags << 16);
	}
	KB_HD uint8_t attrCls(uint32_t a) { return a & 0xFF; }
	KB_HD uint8_t attrScript(uint32_t a) { return (a >> 8) & 0xFF; }
	KB_HD bool attrSpace(uint32_t a) { return (a >> 16) & KB2_CHR_SPACE; }
	KB_HD bool isSpaceChr(const DevModel& m, uint16_t c) { return attrSpace(m.chr_bmp[c]); }
	KB_HD int isEmoji(const DevModel& m, uint32_t c0, uint32_t c1)
	{
		const uint32_t f = chrAttr(m, c0 <= 0x10FFFF ? c0 : 0) >> 16;
		if (f & KB2_CHR_EMOJI1) return 1;
		if (!(c1 == 0xfe0f || (0x1f3fb <= c1 && c1 <= 0x1f3ff))) return 0;
		return (f & KB2_CHR_EMOJI2) ? 2 : 0;
	}

	// FeatureTestor::isMatched(begin, end, CondVowel) reduced to (empty?, last char)   FeatureTestor.cpp:6-60
	KB_HD bool ftVowel(bool empty, uint16_t c, uint8_t vowel)
	{
		if (vowel == CV_none) return true;
		if (empty) return false;
		if (vowel == CV_any) return true;
		if (vowel == CV_applosive)
		{
			switch (c) { case 0x11A8: case 0x11A9: case 0x11AA: case 0x11AE: case 0x11B8: case 0x11B9: case 0x11BA: case 0x11BB: case 0x11BD: case 0x11BE: case 0x11BF: case 0x11C0: case 0x11C1: return true; }
			return false;
		}
		if (!(0xAC00 <= c && c <= 0xD7A4) && !(0x11A8 <= c && c <= 0x11C2)) return true;
		switch (vowel)
		{
		case CV_vocalic_h: if (c == 0x11C2) return true;
		case CV_vocalic: if (c == 0x11AF) return true;
		case CV_vowel: if (0x11A8 <= c && c <= 0x11C2) return false; return true;
		case CV_non_vocalic_h: if (c == 0x11C2) return false;
		case CV_non_vocalic: if (c == 0x11AF) return false;
		case CV_non_vowel: if (0xAC00 <= c && c <= 0xD7A4) return false; return true;
		default: return false;
		}
	}
	// FeatureTestor::isMatched(begin, end, CondPolarity)   FeatureTestor.cpp:62-80
	template<class Ptr>
	KB_HD bool ftPolar(Ptr b, uint32_t len, uint8_t polar)
	{
		if (polar == CP_none || polar == CP_non_adj) return true;
		if (len == 0) return true;
		for (int32_t i = (int32_t)len - 1; i >= 0; --i)
		{
			const uint16_t c = b[i];
			if (0x11A8 <= c && c <= 0x11C2) continue;
			if (c == 0x1161 || c == 0x1163 || c == 0x1169 || c == 0x116D || c == 0x119E) return polar == CP_positive;
			if (!(0xAC00 <= c && c <= 0xD7A4)) break;
			const int v = ((c - 0xAC00) / 28) % 21;
			if (v == 0 || v == 2 || v == 8 || v == 12) return polar == CP_positive;
			if (v == 18 && i == (int32_t)len - 1) continue;
			return polar == CP_negative;
		}
		return polar == CP_negative;
	}
	// FeatureTestor::isMatched(CondVowel) only distinguishes these classes of the last code unit (FeatureTestor.cpp:6-60)
	KB_HD uint32_t lastClass(uint32_t c)
	{
		if (0xAC00 <= c && c <= 0xD7A4) return LC_SYLLABLE;
		if (!(0x11A8 <= c && c <= 0x11C2)) return LC_OTHER;
		if (c == 0x11AF) return LC_CODA_L;
		if (c == 0x11C2) return LC_CODA_H;
		switch (c) { case 0x11A8: case 0x11A9: case 0x11AA: case 0x11AE: case 0x11B8: case 0x11B9: case 0x11BA: case 0x11BB: case 0x11BD: case 0x11BE: case 0x11BF: case 0x11C0: case 0x11C1: return LC_CODA_APPLOSIVE; }
		return LC_CODA_OTHER;
	}
	// left-form part of a path's filter word from (last code unit, LP_* bits)
	KB_HD uint32_t fwOfLeft(uint16_t last, uint8_t lp)
	{
		uint32_t w = lastClass(last);
		if (lp & LP_EMPTY) w |= FW_EMPTY;
		if (lp & LP_POLAR_POS) w |= FW_POLAR_POS;
		if (lp & LP_POLAR_NEG) w |= FW_POLAR_NEG;
		if (lp & LP_LAST_SSC) w |= FW_NOCOND;
		if (lp & LP_MORPH_SOCKET) w |= FW_MORPH_SOCKET;
		return w;
	}
	// tag / socket part: SSC tag switches the conditions off, Z_SIOT is filtered by its successors, the path's combine socket
	KB_HD uint32_t fwOfTag(uint8_t morphTag, uint8_t pathSocket)
	{
		uint32_t w = (uint32_t)pathSocket << FW_SOCKET_SHIFT;
		if (morphTag == T_ssc) w |= FW_NOCOND;
		if (morphTag == T_z_siot) w |= FW_ZSIOT;
		return w;
	}
	// float epilogues of the CoNg int8 scorer (see oracle/restate/cong.hpp for the reference kernels each one restates)
	enum : uint32_t { CG_E_SCALAR = 0, CG_E_SMALL = 1, CG_E_GEMV = 2 };
	KB_HD uint32_t cgEpilogueOf(uint32_t m, uint32_t n)      // m, n = unique contexts / outputs, saturated at 4 (qgemm.hpp:157-201)
	{
		if (m <= 3 && n <= 3) return CG_E_SMALL;
		if (n == 1) return CG_E_GEMV;
		if (m >= 4 && n == 2) return CG_E_GEMV;
		return CG_E_SMALL;
	}
	KB_HD uint32_t knHashFn(uint32_t node, uint32_t token) { uint32_t x = node * 0x9E3779B1u ^ token * 0x85EBCA6Bu; x ^= x >> 15; x *= 0x2C1B3C6Du; x ^= x >> 13; return x; }
	KB_HD uint8_t hashSbTypeOrder(uint8_t type, uint8_t order) { return ((type << 1) ^ (type >> 7) ^ order) % 63 + 1; }   // PathEvaluator.hpp:83-86
}
