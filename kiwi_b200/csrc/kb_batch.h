// kiwi_b200: device batch layout.  One batch = B sentences (raw UTF-16, concatenated) + per-sentence scratch.
// All per-sentence regions are addressed arithmetically from the raw-text offsets, so no offset tables other
// than `text_off` travel to the device:
//   n_s   = text_off[s+1] - text_off[s]             raw length
//   W_s   = 2 * n_s + 4                              capacity in normalized code units (every syllable may split)
//   wbase = 2 * text_off[s] + 4 * s                  start of the W-sized regions of sentence s
//   NC_s  = nodes_per_unit * W_s                     lattice-node capacity; nbase = nodes_per_unit * wbase
#pragma once
#include <stdint.h>
#include "../../include/kiwi_b200_typo.h"

namespace kb
{
	constexpr uint32_t KB_DEFAULT_NODES_PER_UNIT = 12;
	constexpr uint32_t KB_MAX_CHUNKS_SHIFT = 2;      // chunk capacity = W_s >> 2 (a chunk has >= 4 units) + 2

	struct alignas(16) DNode          // 32 B lattice node (KGraphNode, /root/reference/src/KTrie.h:57-77, index based)
	{
		int32_t form;            // form index, -1 = none
		uint32_t uform_off;      // offset into the sentence's normalized text (valid when uform_len > 0)
		uint32_t uform_len;
		uint32_t start_pos, end_pos;   // non-space coordinates while building, normalized-text offsets in the final lattice
		uint16_t prev, sibling;  // relative offsets exactly as the reference: prev = back-offset to the first predecessor
		uint16_t space_errors;
		uint16_t reserved;
		float typo_cost;
	};

	struct alignas(16) DChunk { uint32_t start, end, node_off, n_nodes; };   // normalized offsets [start,end), nodes in the final lattice region

	struct DPattern { uint32_t end, len, tag; };

	// filter word of a path: everything the per-(candidate, path) filter of evalSingleMorpheme (PathEvaluator.hpp:566-594) and the
	// pruning rule need to know about the path's left context, computed ONCE when the path is created
	enum : uint32_t
	{
		FW_CLS_MASK = 7,            // class of the last code unit of the left form (LC_*): all FeatureTestor::isMatched(CondVowel) distinguishes
		FW_EMPTY = 8, FW_POLAR_POS = 16, FW_POLAR_NEG = 32,
		FW_NOCOND = 64,             // FormEvaluator skips the conditions: the left form ends in a closing bracket, or the morpheme's tag is SSC
		FW_ZSIOT = 128,             // morpheme tag is Z_SIOT
		FW_COMMON_ROOT = 256,       // rootId == commonRootId
		FW_MORPH_SOCKET = 512,      // the path's morpheme has a combine socket (excluded from the pruning maximum, PathEvaluator.hpp:480)
		FW_SOCKET_SHIFT = 16,       // 8 bits: WordLL::combineSocket
		FW_PATH_MASK = 0x00FFFFFFu,
	};
	enum : uint32_t { LC_OTHER = 0, LC_SYLLABLE = 1, LC_CODA_L = 2, LC_CODA_H = 3, LC_CODA_APPLOSIVE = 4, LC_CODA_OTHER = 5 };

	struct alignas(16) DPath          // 48 B search path (WordLL, /root/reference/src/BestPathContainer.hpp:21-67), index based
	{
		// segment 0: what a successor's LM step and score need (one 16-byte load)
		int32_t lm_state; float acc_score; float acc_typo_cost;
		uint32_t wid_feat;       // Knlm build: DMorph::feat of morphemes[wid]; CoNg build: CoNgramState::contextIdx
		// segment 1
		uint8_t sp_state;        // SpecialState
		uint8_t root_id, prev_root_id, morph_tag;
		uint32_t fw;             // FW_* filter word (combine socket in bits 16-23)
		float first_chunk_score; uint32_t wid;
		// segment 2: what the back-trace (emit_kernel) needs
		int32_t morpheme; uint32_t parent; uint32_t own_off;
		uint16_t own_len;        // own form (ownFormId != 0): own_off >= 0 -> normalized text offset, own_off has bit 31 -> ~form index
		uint16_t node;           // lattice node (chunk relative) this path ends at
	};
	static_assert(sizeof(DPath) == 48, "DPath is three 16-byte segments");
	enum : uint8_t { LP_POLAR_POS = 1, LP_POLAR_NEG = 2, LP_LAST_SSC = 4, LP_EMPTY = 8, LP_MORPH_SOCKET = 128 };   // leftFeat()'s intermediate form

	struct alignas(16) DToken { uint32_t morph; uint32_t position; float score; uint16_t length; uint8_t tag; uint8_t flags; };

	struct alignas(16) DRec { int32_t parent_rec; uint32_t end_parent; uint32_t chunk; float score; };

	struct VitView
	{
		uint32_t paths_per_unit, paths_const;   // path capacity of sentence s = paths_per_unit * W_s + paths_const
		uint32_t path_stride;        // bytes per path record: sizeof(DPath), or 96 for SkipBigram images (DPath + the 8-token history, viterbi.cu PathS)
		uint32_t n_team;             // the first n_team sentences of the launch order are analysed by a team of warps each (viterbi.cu, team mode)
		uint32_t solo_blocks, solo_warps;   // work-queue build: the first solo_blocks blocks keep only solo_warps warps, which start with the heaviest sentences
		uint32_t* work_counter;      // work-queue build: next position of the launch order to hand out (zeroed before every launch)
		DPath* paths;                // pool, index pbase = paths_per_unit * wbase + paths_const * s
		uint32_t* node_path_off;     // per lattice node (nbase + chunk.node_off + i)
		uint32_t* node_path_cnt;
		uint2* node_cand;            // per lattice node: {first row of the node's candidate block in DevModel::cands, row count | DForm::flags << 16}
		uint8_t* reachable;          // per lattice node
		DRec* recs;                  // 2 per chunk slot: 2 * ((wbase >> 2) + 2 * s)
		DToken* tokens;              // output, W_s per sentence at wbase
		uint32_t* n_tokens;          // [n_sent]
		int32_t* best_rec;           // [n_sent] record of the best stitched result, -1 = none
		float* score;                // [n_sent]
		unsigned long long* timing;  // [2 * n_sent] %globaltimer at the start / end of every sentence's Viterbi (diagnostics: the kernel time is its slowest sentence)
		// token-joining options only (emit_join_kernel): the joined forms of sentence s, forms_per_unit * W_s units at forms_per_unit * wbase
		// (entry layout: JOINED_TOKEN below); n_forms[s] = units used.  nullptr without a join option.
		uint16_t* forms;
		uint32_t* n_forms;           // [n_sent + 1]
		uint32_t forms_per_unit;
	};

	// Match bits of the token-joining fold (joinAffixTokens, /root/reference/src/Kiwi.cpp:495-588) and of the form conversion
	enum : uint32_t
	{
		MO_JOIN_NOUN_PREFIX = 1u << 17, MO_JOIN_NOUN_SUFFIX = 1u << 18, MO_JOIN_VERB_SUFFIX = 1u << 19, MO_JOIN_ADJ_SUFFIX = 1u << 20,
		MO_JOIN_ADV_SUFFIX = 1u << 21, MO_COMPATIBLE_JAMO = 1u << 24, MO_MERGE_SAISIOT = 1u << 26, MO_JOIN_PARTICLE_YO = 1u << 27,
		MO_JOIN_ANY = MO_JOIN_NOUN_PREFIX | MO_JOIN_NOUN_SUFFIX | MO_JOIN_VERB_SUFFIX | MO_JOIN_ADJ_SUFFIX | MO_JOIN_ADV_SUFFIX | MO_MERGE_SAISIOT | MO_JOIN_PARTICLE_YO,
	};
	// DToken::morph of a joined token: JOINED_TOKEN | k, k = offset of its entry in the forms array.  An entry is the first component's
	// morpheme id (low 16 bits, high 16 bits) followed by the joined form and a terminating 0 (include/kiwi_b200.h KIWI_B200_JOINED_TOKEN).
	constexpr uint32_t JOINED_TOKEN = 0x80000000u;

	enum : uint32_t { ST_OK = 0, ST_NODE_OVERFLOW = 1, ST_CHUNK_OVERFLOW = 2, ST_PATH_OVERFLOW = 3, ST_TOKEN_OVERFLOW = 4, ST_TOO_LONG = 5, ST_INTERNAL = 6, ST_TYPO_OVERFLOW = 7 };

	// ---- typo lattice (AnalyzeOption::typoTransformer, BASELINE.json config 4) -------------------------------
	struct alignas(8) DTypoNode       // 24 B typo-graph node (TypoGraphNode, /root/reference/include/kiwi/TypoTransformer.h:130-156)
	{
		uint32_t end_pos; float typo_cost;
		uint32_t prev, sibling;       // relative offsets in the final graph (absolute ids while it is being built)
		uint32_t off; uint16_t len;   // form: chunk[off, off+len) or pool[off, off+len)
		uint8_t from_pool, continual_idx;
	};
	struct alignas(16) DTypoState     // 32 B search state (Splitter::SearchState, /root/reference/src/KTrie.cpp:672-707)
	{
		int32_t node; float acc_cost; uint32_t min_form_len; int32_t start_pos_offset;
		uint32_t special_start, unk_form_start, last_space_boundary, last_chr;
	};
	struct DTypoMatch { uint32_t end_pos, repl_off, size, pat_len; };

	struct TypoView
	{
		// prepared typo transformer, device resident (include/kiwi_b200_typo.h); nodes == nullptr: no typo lattice
		const kb2_typo_node* nodes; const uint16_t* keys; const int32_t* diffs; const kb2_typo_pat* pats; const kb2_typo_repl* repls; const uint16_t* pool;
		float threshold;              // AnalyzeOption::typoThreshold
		float continual_threshold;    // PreparedTypoTransformer::continualTypoThreshold, INFINITY = off
		// per-sentence scratch: graph-node regions at graph_per_unit * wbase (capacity graph_per_unit * W_s), states at states_per_unit * wbase
		uint32_t graph_per_unit, states_per_unit;
		DTypoNode* tmp; DTypoNode* graph; uint32_t* remap;      // insertion-ordered nodes, final graph, old -> new index
		uint2* state_range;           // per final graph node: [first, last) in `states`
		DTypoState* states;
		DTypoMatch* matches;          // graph_per_unit * W_s as well
	};

	struct BatchView
	{
		uint32_t n_sent;
		const uint16_t* text;        // raw UTF-16
		const uint32_t* text_off;    // [n_sent + 1]
		uint32_t match_options;      // kiwi::Match bits (include/kiwi/PatternMatcher.h:10-45)
		uint32_t nodes_per_unit;
		const uint32_t* order;       // [n_sent] launch order: longest sentence first (LPT), so that no long sentence starts in the last wave
		// W-sized scratch (index wbase + i)
		uint16_t* norm;              // normalized text
		uint32_t* norm_len;          // [n_sent]
		uint32_t* pos_table;         // raw index -> normalized index, n_s + 1 entries at text_off[s] + s
		uint32_t* ns_to_pos;
		uint32_t* pos_to_ns;
		uint2* end_pos_map;
		uint32_t* ctr;               // counting-sort scratch
		DPattern* patterns;
		// node regions (index nbase + i)
		DNode* build_nodes;          // insertion-ordered nodes of the chunk being built
		DNode* nodes;                // final lattices of all chunks of the sentence, concatenated
		uint32_t* new_index;         // build index -> final index
		// chunk table: (wbase >> 2) + 2 * s
		DChunk* chunks;
		uint32_t* n_chunks;          // [n_sent]
		uint32_t* status;            // [n_sent]
		uint32_t* debug;             // [64] anomaly record of the first internal-consistency failure (diagnostics)
		TypoView typo;
	};
}
