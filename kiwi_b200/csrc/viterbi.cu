// kiwi_b200 kernel B: pruned Viterbi over the morpheme lattice with Knlm scoring, one warp per sentence.
//
// Replaces (reference file:line under /root/reference/):
//   BestPathFinder<KnLangModel>::findBestPath (topN == 1)   src/PathEvaluator.hpp:1178-1419
//   PathEvaluator::operator() / evalSingleMorpheme           src/PathEvaluator.hpp:347-634
//   RuleBasedScorer, insertToPathContainer, FormEvaluator    src/PathEvaluator.hpp:88-311
//   BucketedHashContainer (top1Small / top1Medium)           src/BestPathContainer.hpp:291-483
//   KnLangModel::progress                                    src/Knlm.cpp:44-130
//   UnkFormScorer::ruleBasedScore                            src/UnkFormScorer.cpp:28-51
//   generateTokenList, isDisconnected                        src/PathEvaluator.hpp:1038-1176
//   chunk loop + insertPathIntoResults (selection part)      src/Kiwi.cpp:1095-1141, 615-783
//
// Parallel mapping.  Lattice nodes are visited in index (= end position) order.  Because kernel A emits the
// nodes that end at one position contiguously and every node appends its surviving paths to one pool, the
// incoming paths of a node are ONE contiguous pool range.  For each candidate morpheme the lanes take the
// incoming paths 32 at a time ("pairs"): filters, Knlm progress (a per-lane pointer chase with binary
// searches), rule scores.  The reference's per-(node, candidate) de-duplication container is reproduced with
// warp primitives: __match_any groups equal (lmState, prevRootId, spState) keys inside a round, a redux picks
// the best score (earliest pair wins ties, like the reference's strict '>'), a shared-memory open-addressing
// table finds keys inserted by earlier rounds, and new keys are appended in pair order so that the output
// order - which fixes all later tie-breaks - is the reference's insertion order (bucket-major in the
// 4 x 128 "medium" mode).  Pruning is a warp max-reduction followed by a ballot compaction.
// Compile with -fmad=false: the reference's float sums are not contracted (x86-64 baseline, no FMA).
#include <cstdlib>
#ifdef KB_HOSTSIM
#include <array>
#include <cstdio>
#include <unordered_map>
#include <unordered_set>
#endif
#include <cuda_runtime.h>
#include <math_constants.h>
#include "kb_model.h"
#include "sbg_math.h"
#include "kb_batch.h"
#include "std_sort_emu.h"
#include "unordered_emu.h"

// This file is compiled twice (csrc/Makefile): KB_CONG=0 -> viterbi_kernel for Knlm images (the code described above),
// KB_CONG=1 -> viterbi_cong_kernel for quantized CoNg images.  The CoNg build replaces, behind `#if KB_CONG`:
//   * the LM step: int8 dot product of a context row and an output row with the reference's float epilogues +
//     one context-trie transition (src/CoNgramModel.cpp:869-903, src/CoNgramModel.hpp:271-385);
//   * the per-node evaluation order of the "transposed" evaluator (PathEvaluator.hpp:860-1035,
//     MorphemeEvaluator<CoNgramState>::eval src/CoNgramModel.cpp:17-317): shortcuts first, then regular, left-half and
//     right-half candidates, every candidate through the per-candidate path `evalCand`;
//   * progressMatrix (src/CoNgramModel.cpp:1494-1611): the (unique context x candidate) int8 products of a node are
//     computed as warp-level tensor-core tiles (mma.sync m16n8k32 u8 x s8 -> s32) into shared memory, `congGroupDots`.
// A CoNg path keeps CoNgramState::contextIdx in the DPath::wid_feat slot (the feature word is re-read from morphs[wid]).
// KB_SBG=1 -> viterbi_sbg_kernel for SkipBigram images (Knlm + an 8-token history per path, src/SkipBigramModel.hpp:113-185).  Its states
// rarely merge, which puts the path containers of the reference into the regime where BucketedHashContainer::insertOptimized behaves
// unlike its comments (see exactInsertRound); that is restated exactly, item by item, so the build takes the per-candidate path
// `evalCand` for every candidate and leaves the item pipeline to the other two builds.
#ifndef KB_CONG
#define KB_CONG 0
#endif
#ifndef KB_SBG
#define KB_SBG 0
#endif
#if KB_SBG
#define KB_VIT_NS vit_sbg
#define KB_VIT_KERNEL viterbi_sbg_kernel
#define P_WID_FEAT(p) ((p).wid_feat)
#define KB_NO_TMA 1
#ifndef KB_TEAM
#define KB_TEAM 1      // (team mode moves 48-byte records)
#endif
#elif KB_CONG
#define KB_VIT_NS vit_cong
#define KB_VIT_KERNEL viterbi_cong_kernel
#define P_WID_FEAT(p) (c_m.morphs[(p).wid].feat)
#define P_CTX(p) ((p).wid_feat)
#else
#define KB_VIT_NS vit_knlm
#define KB_VIT_KERNEL viterbi_kernel
#define P_WID_FEAT(p) ((p).wid_feat)
#endif

namespace kb
{
namespace KB_VIT_NS
{
	// the model view lives in constant memory: every `c_m.field` is an immediate-offset constant-bank load
	__constant__ DevModel c_m;

#if KB_PHASE_CLOCKS
	// Diagnostic build only (`make variant VFLAGS="... -DKB_PHASE_CLOCKS"`, scripts/phase_clocks.py): clock64 cycles of the phases of
	// each sentence's Viterbi, summed over the sentence, lane 0 of its warp, and what its `top1` containers held (count, entries, bucket
	// count after each, rehashes); sentences with index >= KB_PHASE_SENT are not counted.  Inside `evaluate`: path staging, candidate
	// classification, the candidate walk (enumeration and everything it calls), the per-candidate path `evalGeneralCand` on `top1` nodes
	// of more than HT_MAX_ENTRIES incoming paths ("big") and on all others, the exact group redo, and how many big nodes / candidates
	enum { PH_TOP1_ORDER, PH_TOP1_REORDER, PH_FLUSH, PH_EVALUATE, PH_PRUNE, PH_NODE_LOOP, PH_FIND_BEST_PATH,
	       PH_N_TOP1, PH_SUM_E, PH_SUM_B, PH_REHASHES,
	       PH_STAGE, PH_CLASSIFY, PH_WALK, PH_GEN_SMALL, PH_GEN_BIG, PH_REDO, PH_N_BIG_NODES, PH_N_BIG_CANDS, PH_COUNT };
	constexpr uint32_t KB_PHASE_SENT = 8192;
	__device__ unsigned long long phaseClocks[KB_PHASE_SENT * PH_COUNT];
#define KB_PH_START(t) const long long t = clock64()
#define KB_PH_ADD(ph, t, sent) do { if (lane == 0 && (sent) < KB_PHASE_SENT) phaseClocks[(sent) * PH_COUNT + (ph)] += (unsigned long long)(clock64() - (t)); } while (0)
#define KB_PH_COUNT(ph, v, sent) do { if (lane == 0 && (sent) < KB_PHASE_SENT) phaseClocks[(sent) * PH_COUNT + (ph)] += (v); } while (0)
#else
#define KB_PH_COUNT(ph, v, sent) do { } while (0)
#define KB_PH_START(t) do { } while (0)
#define KB_PH_ADD(ph, t, sent) do { } while (0)
#endif

	// a path record: DPath (kb_batch.h); the SkipBigram build appends the rest of the LM state - the ring of the last 8 valid tokens
	// and its position - and the container hash the entry was appended with (VitView::path_stride tells emit.cu the record size)
#if KB_SBG
	struct alignas(16) PathS : DPath { uint32_t hist[8]; uint32_t hpos; uint32_t hpad; unsigned long long hcode; };
	static_assert(sizeof(PathS) == 96, "SkipBigram path record");
	using PathT = PathS;
#else
	using PathT = DPath;
#endif

	static constexpr unsigned FULL = 0xFFFFFFFFu;
	static constexpr uint32_t NPOS = 0xFFFFFFFFu;
	static constexpr uint8_t COMMON_ROOT = 0xFF;
	// Staging capacity of the item pipeline.  Containers of <= 512 incoming paths are the reference's top1Small / top1Medium
	// modes; with KB_STAGE_CAP > 512 the unbounded `top1` mode (> 512 incoming paths, insertion order, no bucket capacity)
	// also goes through the pipeline up to that many incoming paths - these nodes dominate the heaviest sentences of a
	// batch, and the kernel time is the time of its heaviest sentence.
	// A larger capacity costs shared memory (one byte per path and warp), and the L1 cache shrinks with every step of the shared-memory
	// carveout: the Knlm build (one block of 12 warps per SM) stages 1024 paths (csrc/Makefile), the other builds 512.  The mode-2
	// pipeline is kept for a staging area outside shared memory.
#ifndef KB_CG_UCAP
#define KB_CG_UCAP 32
#endif
#ifndef KB_CG_CANDS
#define KB_CG_CANDS 128
#endif
#ifndef KB_STAGE_CAP
#define KB_STAGE_CAP 512
#endif
#ifndef KB_HT_SIZE
#define KB_HT_SIZE 1024
#endif
	static constexpr uint32_t HT_SIZE = KB_HT_SIZE, HT_MAX_ENTRIES = KB_HT_SIZE * 3 / 4;
#ifndef KB_ITEM_CAP
#define KB_ITEM_CAP 512
#endif
	static constexpr uint32_t STAGE_CAP = KB_STAGE_CAP, ITEM_CAP = KB_ITEM_CAP, GROUP = 32;
	static constexpr uint32_t TILE_W = ITEM_CAP / 32 < 16 ? ITEM_CAP / 32 : 16;      // bitmap words (of 32 paths) enumerated per pass: one item buffer
	static_assert(ITEM_CAP % 32 == 0 && ITEM_CAP >= 256, "item buffer");
	static_assert(STAGE_CAP % 512 == 0 && STAGE_CAP <= HT_MAX_ENTRIES * 2 && (HT_SIZE & (HT_SIZE - 1)) == 0, "staging / index capacities");

	// per-node data of one candidate of the current group of 32 (the static part is the DCand row next to it in shared memory)
	struct alignas(8) CandDyn { float additionalScore; uint8_t flags, cls, pad0, pad1; };
	enum : uint8_t { CLS_SKIP = 0, CLS_ITEM = 1, CLS_GENERAL = 2, CLS_SHORTCUT = 3 };
	static constexpr uint32_t FWTAB_CAP = 64;

	struct CandMask { uint32_t valid, condFail, sets; };

	struct WarpSmem
	{
		alignas(16) DCand dcandBuf[2][GROUP];   // static candidate rows of the current group, double buffered: the NEXT node's block arrives by one
		                                        // bulk copy (cp.async.bulk -> mbarrier) while the current node is evaluated; other groups by lane stores
		alignas(8) unsigned long long mbar[2];  // one transaction barrier per buffer
		alignas(16) DCand dcandGen[GROUP];      // rows stored from registers (groups that were not bulk-staged): the bulk buffers are only ever
		                                        // written by the copy engine, so no generic-to-async proxy fence is needed before a copy
		CandDyn cdyn[GROUP];
		uint8_t pcls[STAGE_CAP];                // class index of every incoming path (classes = distinct filter words)
		uint32_t fclass[32];                    // the distinct filter words: FW_* bits | combine_socket << 16
		uint16_t ht[HT_SIZE];
		uint32_t item[ITEM_CAP];                // slot << 27 | fwIdx << 20 | q << 3 | spacePen << 2 | r << 1 | condFail
		CandMask cmask[GROUP];                  // per candidate: which path classes survive the filter / fail the soft condition / override firstWid
		uint32_t candNew[GROUP];                // entries created per candidate of the current group
		uint32_t fwTab[FWTAB_CAP];              // first-wid overrides of socket chunks (PathEvaluator.hpp:590), index 0 unused
		uint32_t exactInsert;                   // != 0: evalCand inserts item by item (exactInsertRound) - set while a group is re-run (redoGroupExact)
#if KB_CONG
		int32_t dots[KB_CG_UCAP][33];           // (unique context, candidate of the group) -> sum u8*s8 - hsum, from the tensor-core tiles
		uint32_t uctx[KB_CG_UCAP];              // the node's unique context ids (regular incoming paths)
		uint8_t pslot[STAGE_CAP];               // incoming path -> index into uctx, 0xFF = none (socket path / more than 64 contexts)
		uint32_t colWid[GROUP];                 // first wid of every candidate of the group
		uint32_t candOrder[KB_CG_CANDS];        // the node's candidates in the transposed evaluator's order (indices into the node's candidate block)
#endif
	};
#ifndef KB_VIT_WARPS
#define KB_VIT_WARPS 4
#endif
	static constexpr uint32_t WARPS_PER_BLOCK = KB_VIT_WARPS;
#ifndef KB_EXACT_FROM
#define KB_EXACT_FROM 64u      // states per bucket from which a group is re-run item by item (tests lower it to drive that path through every sentence)
#endif
	static constexpr uint32_t MAX_RESULTS = 16;

	__device__ __forceinline__ float asFloat(int32_t v) { return __int_as_float(v); }

	__device__ __forceinline__ bool ftVowelCls(bool empty, uint32_t cls, uint32_t vowel)
	{
		if (vowel == CV_none) return true;
		if (empty) return false;
		if (vowel == CV_any) return true;
		if (vowel == CV_applosive) return cls == LC_CODA_APPLOSIVE;
		if (cls == LC_OTHER) return true;
		const bool coda = cls >= LC_CODA_L;
		switch (vowel)
		{
		case CV_vocalic_h: if (cls == LC_CODA_H) return true;
		case CV_vocalic: if (cls == LC_CODA_L) return true;
		case CV_vowel: return !coda;
		case CV_non_vocalic_h: if (cls == LC_CODA_H) return false;
		case CV_non_vocalic: if (cls == LC_CODA_L) return false;
		case CV_non_vowel: return cls != LC_SYLLABLE;
		default: return false;
		}
	}

	// ---- KnLangModel::progress, src/Knlm.cpp:44-130 (one lane) -------------------------------------
	// Same arithmetic (float adds in the reference's order), different table layout: the per-node sorted key
	// arrays + binary search of the reference become ONE probe into an open-addressing table over all edges whose
	// entry also carries a second word, and the root uses direct tables (lm_tables.h, built by model.cu at load).
	// That word is returned as raw bits: the child's ll for an inner edge (v > 0), the state after the edge for a leaf (v <= 0).
	__device__ __forceinline__ bool knLookup(uint32_t node, uint32_t key, int32_t& v, uint32_t& w)
	{
		uint32_t h = knHashFn(node, key) & c_m.kn_hash_mask;
		while (true)
		{
			const uint4 e = c_m.kn_hash[h];
			if (e.x == node && e.y == key) { v = (int32_t)e.z; w = e.w; return true; }
			if (e.x == 0xFFFFFFFFu) return false;
			h = (h + 1) & c_m.kn_hash_mask;
		}
	}
	// (state in, {log-probability, state} out - both in registers: a reference parameter would pin the caller's state to local memory)
	struct KnRes { float ll; int32_t node; };
	__device__ __forceinline__ KnRes knProgressI(int32_t nodeIdx, uint32_t next)
	{
		float acc = 0;
		while (true)
		{
			if (nodeIdx == 0)
			{
				const int32_t v = c_m.kn_root[next];
				if (v > 0) return KnRes{ acc + c_m.kn_root_ll[next], v };
				// unknown token (v == 0) or a leaf of the root (v < 0, whose ll it holds): the root has no suffix to fall back to
				const int32_t st = c_m.kn_htx ? c_m.kn_root[c_m.kn_htx[next]] : 0;
				return KnRes{ acc + (v == 0 ? c_m.kn_unk_ll : asFloat(v)), st };
			}
			const float2 bo = c_m.kn_backoff[nodeIdx];            // issued together with the probe
			int32_t v; uint32_t w;
			if (!knLookup((uint32_t)nodeIdx, next, v, w))
			{
				acc += bo.y;
				nodeIdx += __float_as_int(bo.x);
				continue;
			}
			if (v > 0) return KnRes{ acc + __uint_as_float(w), nodeIdx + v };
			return KnRes{ acc + asFloat(v), (int32_t)w };         // leaf: v holds its ll, w the next state
		}
	}
	__device__ __noinline__ KnRes knProgressV(int32_t nodeIdx, uint32_t next) { return knProgressI(nodeIdx, next); }
#if defined(KB_HOSTSIM) && !KB_SBG
	// tests/hostsim (scripts/lm_chain.py): the serial dependent loads of every LM step, i.e. the probe slots of its chain (root table
	// reads included; CoNg also reads a node's suffix link only after the probe missed) and its backoff levels, and the loads the
	// kernels spent after a leaf before lm_tables.h stored the leaf's next state.  Those come in two kinds, counted apart: the suffix
	// walk after a leaf edge of a non-root node (re-done here and checked against the stored state), and the single read of the root's
	// empty suffix link after a leaf of the root.  Per flushItems round, the largest sum over the round's active lanes is kept three
	// ways: with both (the kernels before), with neither (now), and with the non-root walk only.  A round lasts as long as its slowest lane.
	struct HsChain { uint64_t steps, probes, backoffs, leafSteps, walkLevels, walkLoads, rootLeafSteps, rounds, roundMax[3]; };
	static HsChain g_chain;
	static uint32_t g_chainLane[512][3];           // per thread: loads of its LM steps since its round began {before, now, non-root walk only}
	static uint32_t g_chainFlush[512];             // per thread: flushItems calls
	static std::unordered_map<uint64_t, std::array<uint32_t, 3>> g_chainRounds;      // (warp, call, round) -> maxima over its lanes
	static bool hsProbe(const uint4* tab, uint32_t mask, uint32_t node, uint32_t key, int32_t& v, uint32_t& w, uint32_t& loads)
	{
		for (uint32_t h = knHashFn(node, key) & mask;; h = (h + 1) & mask)
		{
			++loads;
			const uint4 e = tab[h];
			if (e.x == node && e.y == key) { v = (int32_t)e.z; w = e.w; return true; }
			if (e.x == 0xFFFFFFFFu) return false;
		}
	}
	// after: the step's loads now; walk: the non-root leaf walk's loads; rootLeaf: 1 when the step ended on a leaf of the root
	static void hsChainAdd(uint32_t after, uint32_t walk, uint32_t rootLeaf)
	{
		++g_chain.steps; g_chain.probes += after; g_chain.walkLoads += walk; g_chain.rootLeafSteps += rootLeaf;
		uint32_t* l = g_chainLane[threadIdx.x];
		l[0] += after + walk + rootLeaf; l[1] += after; l[2] += after + walk;
	}
	static void hsChainMismatch(int32_t node, uint32_t next, uint32_t stored, int32_t walked)
	{
		std::fprintf(stderr, "[hs32] leaf edge (%d, %u): stored state %u, suffix walk %d\n", node, next, stored, walked);
		std::abort();
	}
#if !KB_CONG
	static void hsChainStep(int32_t node, uint32_t next)
	{
		uint32_t after = 0, walk = 0, rootLeaf = 0;
		while (true)
		{
			if (node == 0)
			{
				const int32_t v = c_m.kn_root[next]; ++after;
				if (v <= 0 && c_m.kn_htx) after += 2;                    // kn_htx[next], then its root entry
				rootLeaf = v < 0;                                          // the kernels read the root's (empty) suffix link first
				break;
			}
			int32_t v; uint32_t w;
			if (!hsProbe(c_m.kn_hash, c_m.kn_hash_mask, (uint32_t)node, next, v, w, after))
			{
				++g_chain.backoffs; node += __float_as_int(c_m.kn_backoff[node].x); continue;      // link read with the probe
			}
			if (v > 0) break;
			++g_chain.leafSteps;
			int32_t cur = node, st = -1;
			while (true)
			{
				++walk;                                                    // kn_backoff[cur]
				const int32_t lower = __float_as_int(c_m.kn_backoff[cur].x);
				if (!lower) break;
				cur += lower; ++g_chain.walkLevels;
				int32_t lv = 0; uint32_t lw; bool f;
				if (cur == 0) { ++walk; f = (lv = c_m.kn_root[next]) != 0; }
				else f = hsProbe(c_m.kn_hash, c_m.kn_hash_mask, (uint32_t)cur, next, lv, lw, walk);
				if (f && lv > 0) { st = cur + lv; break; }
			}
			if (st < 0) { if (c_m.kn_htx) walk += 2; st = c_m.kn_htx ? c_m.kn_root[c_m.kn_htx[next]] : 0; }
			if ((uint32_t)st != w) hsChainMismatch(node, next, w, st);
			break;
		}
		hsChainAdd(after, walk, rootLeaf);
	}
	extern "C" void hs32_lm_chain_stats(uint64_t* out)
#else
	static void hsChainStep(int32_t node, uint32_t next)
	{
		uint32_t after = 0, walk = 0, rootLeaf = 0;
		while (true)
		{
			if (node == 0)
			{
				const int32_t v = next < c_m.cg_root_size ? c_m.cg_root[next] : 0; ++after;
				if (v > 0) ++after;                                        // cg_nodes[v].y
				rootLeaf = v < 0;                                          // the kernels read the root's (empty) suffix link first
				break;
			}
			int32_t v; uint32_t w;
			if (!hsProbe(c_m.cg_hash, c_m.cg_hash_mask, (uint32_t)node, next, v, w, after))
			{
				++after; ++g_chain.backoffs;                               // cg_nodes[node].x, read after the miss
				const int32_t lower = c_m.cg_nodes[node].x;
				if (!lower) break;
				node += lower; continue;
			}
			if (v > 0) break;
			++g_chain.leafSteps;
			int32_t cur = node, st = 0;
			while (true)
			{
				++walk;                                                    // cg_nodes[cur].x
				const int32_t lower = c_m.cg_nodes[cur].x;
				if (!lower) break;
				cur += lower; ++g_chain.walkLevels;
				int32_t lv = 0; uint32_t lw; bool f;
				if (cur == 0) { ++walk; lv = next < c_m.cg_root_size ? c_m.cg_root[next] : 0; f = lv != 0; }
				else f = hsProbe(c_m.cg_hash, c_m.cg_hash_mask, (uint32_t)cur, next, lv, lw, walk);
				if (f && lv > 0) { st = cur + lv; break; }
			}
			if ((uint32_t)st != w) hsChainMismatch(node, next, w, st);
			break;
		}
		hsChainAdd(after, walk, rootLeaf);
	}
	extern "C" void hs32_cg_chain_stats(uint64_t* out)
#endif
	{
		// {steps, chain loads, backoff levels, non-root leaf steps, their walk levels, their walk loads, root-leaf steps, flushItems rounds,
		//  sums of the round maxima: before, now, non-root walk only}
		for (const auto& r : g_chainRounds) { ++g_chain.rounds; for (int k = 0; k < 3; ++k) g_chain.roundMax[k] += r.second[k]; }
		const uint64_t v[11] = { g_chain.steps, g_chain.probes, g_chain.backoffs, g_chain.leafSteps, g_chain.walkLevels, g_chain.walkLoads,
		                         g_chain.rootLeafSteps, g_chain.rounds, g_chain.roundMax[0], g_chain.roundMax[1], g_chain.roundMax[2] };
		for (int i = 0; i < 11; ++i) out[i] = v[i];
		g_chain = HsChain{}; g_chainRounds.clear();
	}
	static void hsChainRound(uint32_t ib)
	{
		const uint32_t t = threadIdx.x;
		auto& m = g_chainRounds[(uint64_t)(t >> 5) << 56 | (uint64_t)g_chainFlush[t] << 24 | ib];
		for (int k = 0; k < 3; ++k) m[k] = std::max(m[k], g_chainLane[t][k]);
	}
#define KB_HS_CHAIN_STEP(node, next) hsChainStep((node), (next))
#define KB_HS_CHAIN_FLUSH() (++g_chainFlush[threadIdx.x])
#define KB_HS_CHAIN_ROUND_BEGIN() (g_chainLane[threadIdx.x][0] = g_chainLane[threadIdx.x][1] = g_chainLane[threadIdx.x][2] = 0)
#define KB_HS_CHAIN_ROUND_END(ib) hsChainRound(ib)
#else
#define KB_HS_CHAIN_STEP(node, next) ((void)0)
#define KB_HS_CHAIN_FLUSH() ((void)0)
#define KB_HS_CHAIN_ROUND_BEGIN() ((void)0)
#define KB_HS_CHAIN_ROUND_END(ib) ((void)0)
#endif
#if defined(KB_HOSTSIM) && !KB_CONG && !KB_SBG
	// tests/hostsim: LM steps and distinct (state, wid) pairs of one sentence (scripts/lm_repeat.py reads and resets them per sentence)
	static uint64_t g_lmSteps, g_lmDistinct;
	static std::unordered_set<uint64_t> g_lmPairs;
	extern "C" void hs32_lm_repeat_stats(uint64_t* out)
	{
		out[0] = g_lmSteps; out[1] = g_lmDistinct;
		g_lmSteps = g_lmDistinct = 0; g_lmPairs.clear();
	}
	// ... and where they were taken (scripts/lm_sites.py): flushItems, evalCand on a node of at most / more than HT_MAX_ENTRIES
	// incoming paths (g_lmBigNode, set by evalCand), anywhere else
	static uint64_t g_lmSite[4];
	static bool g_lmBigNode;
	extern "C" void hs32_lm_site_stats(uint64_t* out)
	{
		for (int i = 0; i < 4; ++i) { out[i] = g_lmSite[i]; g_lmSite[i] = 0; }
	}
#endif
	__device__ __forceinline__ float knProgress(int32_t& nodeIdx, uint32_t next, uint32_t site = 0)
	{
#if defined(KB_HOSTSIM) && !KB_CONG && !KB_SBG
		++g_lmSteps; g_lmDistinct += g_lmPairs.insert((uint64_t)(uint32_t)nodeIdx << 32 | next).second;
		++g_lmSite[site == 1 || site == 2 ? 0 : site == 3 || site == 4 ? (g_lmBigNode ? 2 : 1) : 3];
		KB_HS_CHAIN_STEP(nodeIdx, next);
#else
		(void)site;
#endif
		const KnRes r = knProgressV(nodeIdx, next);
		nodeIdx = r.node;
		return r.ll;
	}


#if KB_CONG
	// ---- CoNg language model ----------------------------------------------------------------------------
	static constexpr uint32_t CG_UCAP = KB_CG_UCAP;  // unique contexts of a node held in the tensor-core tile (else per-pair dp4a); 32 keeps 4 blocks per SM
	static constexpr uint32_t CG_CANDS = KB_CG_CANDS; // candidates of one lattice node (the largest candidate list of the test models has 90 entries)

	// as knLookup: the fourth word is the child's context id for an inner edge, the node after the edge for a leaf (lm_tables.h)
	__device__ __forceinline__ bool cgLookup(uint32_t node, uint32_t key, int32_t& v, uint32_t& w)
	{
		uint32_t h = knHashFn(node, key) & c_m.cg_hash_mask;
		while (true)
		{
			const uint4 e = c_m.cg_hash[h];
			if (e.x == node && e.y == key) { v = (int32_t)e.z; w = e.w; return true; }
			if (e.x == 0xFFFFFFFFu) return false;
			h = (h + 1) & c_m.cg_hash_mask;
		}
	}
	// progressContextNodeVl, src/CoNgramModel.hpp:314-385 (one lane)
	__device__ __noinline__ uint32_t cgStepVl(int32_t& nodeIdx, uint32_t next)
	{
		if ((uint32_t)nodeIdx >= 0x10000000u)
		{
			if (atomicCAS(&c_m.debug[0], 0u, 1u) == 0u) { c_m.debug[1] = 77; c_m.debug[2] = next; c_m.debug[3] = (uint32_t)nodeIdx; c_m.debug[4] = blockIdx.x; c_m.debug[5] = threadIdx.x; }
			nodeIdx = 0; return 0;
		}
		KB_HS_CHAIN_STEP(nodeIdx, next);
		while (true)
		{
			if (nodeIdx == 0)
			{
				const int32_t v = next < c_m.cg_root_size ? c_m.cg_root[next] : 0;
				if (v == 0) return 0;
				if (v > 0) { nodeIdx = v; return (uint32_t)c_m.cg_nodes[v].y; }
				return (uint32_t)-v;                               // a leaf of the root: the root has no suffix, the state stays 0
			}
			int32_t v; uint32_t w;
			if (!cgLookup((uint32_t)nodeIdx, next, v, w))
			{
				const int32_t lower = c_m.cg_nodes[nodeIdx].x;
				if (!lower) return 0;
				nodeIdx += lower;
				continue;
			}
			if (v > 0) { nodeIdx += v; return w; }
			nodeIdx = (int32_t)w;                                 // leaf: -v is its context id, w the next node
			return (uint32_t)-v;
		}
	}
	// progressContextNode, src/CoNgramModel.hpp:271-297
	__device__ __forceinline__ uint32_t cgStep(int32_t& nodeIdx, uint32_t next)
	{
		if (c_m.cg_inv_vocab) next = c_m.cg_inv_vocab[next];
		if (c_m.cg_key_size != 3) return cgStepVl(nodeIdx, next);
		const uint32_t tMax = (1u << 16) - (1u << 10) * 2;
		if (next < tMax) return cgStepVl(nodeIdx, next);
		next -= tMax;
		cgStepVl(nodeIdx, tMax + (next >> 10));
		return cgStepVl(nodeIdx, tMax + (1u << 10) + (next & 0x3FF));
	}
	// sum_k ctx_u8[k] * out_s8[k] - hsum  ==  sum_k (ctx_u8[k] - 128) * out_s8[k]   (hsum = 128 * sum out, CoNgramModel.cpp:672)
	__device__ __noinline__ int32_t cgDot(uint32_t ctx, uint32_t wid)
	{
		const uint4* a = reinterpret_cast<const uint4*>(c_m.cg_ctx_emb + (size_t)ctx * c_m.cg_stride);
		const uint4* b = reinterpret_cast<const uint4*>(c_m.cg_out_emb + (size_t)wid * c_m.cg_stride);
		// rows are 8-byte aligned (stride = dim + 8): read 8 bytes at a time
		const uint2* a2 = reinterpret_cast<const uint2*>(a); const uint2* b2 = reinterpret_cast<const uint2*>(b);
		int32_t acc = 0;
		const uint32_t n8 = c_m.cg_dim >> 3;
		#pragma unroll 4
		for (uint32_t k = 0; k < n8; ++k)
		{
			const uint2 x = a2[k], y = b2[k];
			acc = __dp4a((int)(x.x ^ 0x80808080u), (int)y.x, acc);
			acc = __dp4a((int)(x.y ^ 0x80808080u), (int)y.y, acc);
		}
		return acc;
	}
	// the three float epilogues of the reference's kernels (kb_model.h CG_E_*, oracle/restate/cong.hpp)
	__device__ __forceinline__ float cgFinish(int32_t x, uint32_t ctx, uint32_t wid, uint32_t ep)
	{
		const float2 cs = *reinterpret_cast<const float2*>(c_m.cg_ctx_emb + (size_t)ctx * c_m.cg_stride + c_m.cg_dim);   // {scale, bias}
		const float os = *reinterpret_cast<const float*>(c_m.cg_out_emb + (size_t)wid * c_m.cg_stride + c_m.cg_dim);
		const float xf = __int2float_rn(x);
		if (ep == CG_E_SCALAR)
		{
			float ll = __fadd_rn(__fmul_rn(__fmul_rn(xf, cs.x), os), cs.y);
			if (c_m.cg_out_bias) ll = __fadd_rn(ll, c_m.cg_out_bias[wid]);
			return ll;
		}
		if (ep == CG_E_SMALL) return __fmaf_rn(__fmul_rn(xf, cs.x), os, cs.y);
		return __fmaf_rn(__fmul_rn(xf, os), cs.x, cs.y);
	}
	// CoNgramState::next (scalar path)
	__device__ __forceinline__ float cgNext(int32_t& node, uint32_t& ctx, uint32_t wid)
	{
		const float ll = cgFinish(cgDot(ctx, wid), ctx, wid, CG_E_SCALAR);
		ctx = cgStep(node, wid);
		return ll;
	}

	// progressMatrix's gather GEMM for one group of <= 32 candidates (src/CoNgramModel.cpp:1575-1579, qgemm.hpp:36-87):
	// dots[u][c] = sum_k ctx_u8[uctx[u]][k] * out_s8[colWid[c]][k] - hsum[colWid[c]] as warp-level tensor-core tiles,
	// mma.sync.m16n8k32 (u8 x s8 -> s32); rows are gathered straight from the resident embedding tables (L2).
	// Fragment layout (g = lane / 4, t = lane % 4): A row-major 16x32: a0 (row g, k 4t..4t+3), a1 (row g+8, same k), a2 (row g, k 16+4t..),
	// a3 (row g+8, k 16+4t..); B col-major 32x8: b0 (k 4t..4t+3, col g), b1 (k 16+4t.., col g); C: c0 (g, 2t), c1 (g, 2t+1), c2 (g+8, 2t), c3 (g+8, 2t+1).
	__device__ __noinline__ void cgTileDots(const uint32_t* uctx, const uint32_t* colWid, int32_t (*dots)[33], uint32_t nU, uint32_t colMask, uint32_t lane)
	{
		const uint32_t g = lane >> 2, t = lane & 3;
		const uint32_t mTiles = (nU + 15) >> 4, kSteps = c_m.cg_dim >> 5, stride = c_m.cg_stride;
		#pragma unroll 1
		for (uint32_t nt = 0; nt < 4; ++nt)
		{
			if (!((colMask >> (nt * 8)) & 0xFFu)) continue;
			const uint32_t col = nt * 8 + g;
			const uint32_t wid = ((colMask >> col) & 1u) ? colWid[col] : 0u;
			const uint8_t* pb = c_m.cg_out_emb + (size_t)wid * stride;
			// hsum of the two columns this lane's accumulators belong to (2t, 2t + 1)
			const uint32_t c0col = nt * 8 + t * 2, c1col = c0col + 1;
			const uint32_t w0 = ((colMask >> c0col) & 1u) ? colWid[c0col] : 0u, w1 = ((colMask >> c1col) & 1u) ? colWid[c1col] : 0u;
			const int32_t h0 = *reinterpret_cast<const int32_t*>(c_m.cg_out_emb + (size_t)w0 * stride + c_m.cg_dim + 4);
			const int32_t h1 = *reinterpret_cast<const int32_t*>(c_m.cg_out_emb + (size_t)w1 * stride + c_m.cg_dim + 4);
			#pragma unroll 1
			for (uint32_t mt = 0; mt < mTiles; ++mt)
			{
				const uint32_t r0 = mt * 16 + g, r1 = r0 + 8;
				const uint8_t* pa0 = c_m.cg_ctx_emb + (size_t)uctx[r0 < nU ? r0 : 0] * stride;
				const uint8_t* pa1 = c_m.cg_ctx_emb + (size_t)uctx[r1 < nU ? r1 : 0] * stride;
				int32_t c0 = 0, c1 = 0, c2 = 0, c3 = 0;
				#pragma unroll 2
				for (uint32_t kk = 0; kk < kSteps; ++kk)
				{
					const uint32_t ko = kk * 32 + t * 4;
					const uint32_t a0 = *reinterpret_cast<const uint32_t*>(pa0 + ko), a1 = *reinterpret_cast<const uint32_t*>(pa1 + ko);
					const uint32_t a2 = *reinterpret_cast<const uint32_t*>(pa0 + ko + 16), a3 = *reinterpret_cast<const uint32_t*>(pa1 + ko + 16);
					const uint32_t b0 = *reinterpret_cast<const uint32_t*>(pb + ko), b1 = *reinterpret_cast<const uint32_t*>(pb + ko + 16);
#ifdef KB_HOSTSIM
					simt::mma_m16n8k32_u8s8(c0, c1, c2, c3, a0, a1, a2, a3, b0, b1);      // tests/hostsim: the fragment semantics in C++
#else
					asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
						: "+r"(c0), "+r"(c1), "+r"(c2), "+r"(c3) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
#endif
				}
				if (r0 < nU) { dots[r0][c0col] = c0 - h0; dots[r0][c1col] = c1 - h1; }
				if (r1 < nU) { dots[r1][c0col] = c2 - h0; dots[r1][c1col] = c3 - h1; }
			}
		}
		__syncwarp();
	}
#endif

	// ------------------------------------------------------------------------------------------------
	struct PathRes { float score; uint32_t endParent; uint8_t prevState, curState; };

	// ---- team mode ------------------------------------------------------------------------------------------------------
	// A batch's kernel time is the time of its heaviest sentence (10 x the mean work in the bench batch).  The first
	// VitView::n_team sentences of the launch order are therefore analysed by TEAMS of KB_TEAM warps: all warps of a team walk the
	// lattice together; the candidates of a node are dealt round-robin to the warps, each warp evaluates its candidates
	// (classification, enumeration, LM chase, de-duplication: all per-candidate state) into a private staging region of the
	// sentence's path pool, and after a team barrier the per-candidate segments are copied to their final places in candidate
	// order - the pool ends up byte-identical to the single-warp result.  Order-dependent steps (shortcut / general candidates,
	// pruning, reachability, the end node, stitching) stay on the team's first warp and their results are broadcast.
#ifndef KB_TEAM
#define KB_TEAM 4
#endif
#ifndef KB_QUEUE
#define KB_QUEUE 0      // 1: persistent warps draw sentences from a work queue (needs KB_TEAM=1)
#endif
	static constexpr uint32_t TEAM = KB_TEAM, TEAMS_PER_BLOCK = KB_VIT_WARPS / KB_TEAM > 0 ? KB_VIT_WARPS / KB_TEAM : 1;
	static_assert(KB_VIT_WARPS % KB_TEAM == 0 || KB_VIT_WARPS < KB_TEAM, "teams tile the block");
	struct TeamSmem
	{
		uint32_t cnt[GROUP];         // entries per candidate of the current group (written by the owning warp)
		uint32_t val[2][4];          // broadcast slots (alternating, see Vit::teamBroadcast)
		uint32_t err;
	};

	// functions with ONE call site: inlined with -DKB_INLINE_MORE (kernel experiments), out of line otherwise
#ifdef KB_INLINE_MORE
#define KB_INL1 __forceinline__
#else
#define KB_INL1 __noinline__
#endif
#ifdef KB_INLINE_EVAL
#define KB_INL_EVAL __forceinline__
#else
#define KB_INL_EVAL __noinline__
#endif
	// Vit lives in local memory (its address is `this` of the out-of-line members), and every member a loop reads through `this` is
	// re-read from there after each store the compiler cannot tell apart from it.  The hot loops (flushItems, evaluate) therefore work
	// on register copies of the members they read.  The kernel parameters are not referenced from here: a reference would give them
	// a local copy too.
	struct Vit
	{
		const uint32_t lane;
		uint32_t err = 0;
		// sentence
		const uint16_t* norm;
		PathT* pool; uint32_t poolCap, top;
		// chunk
		const DNode* nodes; uint32_t N;
		uint32_t* npOff; uint32_t* npCnt; uint8_t* reach;
		uint8_t uniq[2]; uint32_t nUniq;
		uint16_t* ht; uint32_t htUsed;
		uint32_t top1Buckets = 1;           // bucket count of the reference's `top1` unordered_set, per sentence (unordered_emu.h)
#if KB_PHASE_CLOCKS
		uint32_t phSent = 0;                // the sentence's index (phaseClocks)
#endif
#if KB_SBG
		uint32_t sbIdxCap = 0;              // slots of the current candidate's `top1` index at the end of the sentence's pool region (0 = none yet)
#endif
		DCand* dcur = nullptr; uint32_t curBuf = 0, pfPhase = 0; const DCand* pfBase[2] = { nullptr, nullptr };      // candidate-row staging (see prefetchCands)
		uint2* nodeCand = nullptr;
		WarpSmem* sm; uint32_t stagedNode = 0xFFFFFFFFu; uint32_t htBase = 0, htCount = 0;
		uint32_t nClasses = 0, classCommon = 0; bool classOverflow = false;
		// team mode (the heaviest sentences): KB_TEAM warps share one sentence, see TeamSmem
#if KB_TEAM > 1
		uint32_t teamRank = 0, teamSize = 1, teamBar = 0, teamSeq = 0; struct TeamSmem* tm = nullptr;
#else
		static constexpr uint32_t teamRank = 0, teamSize = 1, teamBar = 0; uint32_t teamSeq = 0; struct TeamSmem* tm = nullptr;      // KB_TEAM=1: every team branch folds away
#endif
		bool splitComplex, splitSaisiot, mergeSaisiot;

		__device__ explicit Vit(uint32_t _lane) : lane{ _lane } {}

		// ---- team primitives (no-ops for a single warp)
		__device__ __forceinline__ bool leader() const { return teamRank == 0; }
		__device__ __forceinline__ void teamSync()
		{
			if (teamSize == 1) return;
			__syncwarp();
#ifdef KB_HOSTSIM
			simt::bar_sync(teamBar, teamSize * 32);
#else
			asm volatile("bar.sync %0, %1;" :: "r"(teamBar), "r"(teamSize * 32) : "memory");
#endif
		}
		// the first warp's (a, b, c) and the team's error state become everybody's: one barrier; the two slots alternate so that a
		// slot is rewritten only after every reader has passed one more barrier
		__device__ __forceinline__ void teamBroadcast(uint32_t& a, uint32_t& b, uint32_t& c)
		{
			if (teamSize == 1) return;
			uint32_t* slot = tm->val[teamSeq & 1]; ++teamSeq;
			if (leader() && lane == 0) { slot[0] = a; slot[1] = b; slot[2] = c; }
			if (err && lane == 0) atomicMax(&tm->err, err);
			teamSync();
			a = slot[0]; b = slot[1]; c = slot[2];
			err = tm->err;
		}
		__device__ __forceinline__ void teamBroadcast(uint32_t& a) { uint32_t b = 0, c = 0; teamBroadcast(a, b, c); }

		// ---- left-form features of a path (what FormEvaluator will see), uniform per candidate ------
		__device__ __noinline__ void leftFeat(uint32_t ownOff, uint32_t ownLen, uint32_t wid, int32_t morpheme, uint16_t& last, uint8_t& pol) const
		{
			pol = 0; last = 0;
			if (ownLen)
			{
				if (ownOff & 0x80000000u)
				{
					const DForm f = c_m.forms[~ownOff];
					last = f.last_chr;
					pol = (f.pol & (FP_POLAR_POS | FP_POLAR_NEG | FP_LAST_SSC));
				}
				else
				{
					const uint16_t* p = norm + ownOff;
					last = p[ownLen - 1];
					if (ftPolar(p, ownLen, CP_positive)) pol |= LP_POLAR_POS;
					if (ftPolar(p, ownLen, CP_negative)) pol |= LP_POLAR_NEG;
					if (attrCls(c_m.chr_bmp[last]) == T_ssc) pol |= LP_LAST_SSC;
				}
				return;
			}
			int32_t fi = c_m.morphs[wid].form_idx;
			if (!(fi >= 0 && c_m.forms[fi].str_len)) fi = c_m.morphs[morpheme].form_idx;
			if (fi < 0 || c_m.forms[fi].str_len == 0) { pol = LP_EMPTY | LP_POLAR_POS | LP_POLAR_NEG; return; }
			const DForm f = c_m.forms[fi];
			last = f.last_chr;
			pol = (f.pol & (FP_POLAR_POS | FP_POLAR_NEG | FP_LAST_SSC));
		}

		// ---- UnkFormScorer::ruleBasedScore, src/UnkFormScorer.cpp:28-51 ------------------------------
		template<class Ptr>
		__device__ float unkFormScore(Ptr form, uint32_t len) const
		{
			float penalty = 0;
			if (len > 0)
			{
				uint32_t chrs[2] = { 0, 0 };
				for (uint32_t i = 0, j = 0; i < len && j < 2; ++j)
				{
					if (isHighSurrogate(form[i])) { chrs[j] = mergeSurrogate(form[i], i + 1 < len ? form[i + 1] : 0); i += 2; }
					else { chrs[j] = form[i]; ++i; }
				}
				if (isEmoji(c_m, chrs[0], chrs[1])) penalty = -10.f;
			}
			return penalty - ((float)len * c_m.cfg.oov_rule_scale + c_m.cfg.oov_rule_bias);
		}

		// PathEvaluator.hpp:22-44
		__device__ bool hasLeftBoundary(uint32_t i) const
		{
			const DNode nd = nodes[i];
			const DNode pv = nodes[i - nd.prev];
			if (pv.end_pos == 0) return true;
			if (pv.end_pos < nd.start_pos) return true;
			if (pv.uform_len)
			{
				const uint32_t c = norm[pv.uform_off + pv.uform_len - 1];
				const uint32_t tag = attrCls(c_m.chr_bmp[c]);
				if (tag == T_ssc || c == '"' || c == '\'') return false;
				if (T_sf <= tag && tag <= T_sb) return true;
			}
			return false;
		}

		__device__ void htClear()
		{
			if (!htUsed) return;
			for (uint32_t i = lane; i < HT_SIZE / 8; i += 32) reinterpret_cast<uint4*>(ht)[i] = make_uint4(0, 0, 0, 0);
			htUsed = 0;
			__syncwarp();
		}
		static __device__ __forceinline__ uint32_t htHash(int32_t lm, uint32_t prevRoot, uint32_t sp)
		{
			uint32_t h = (uint32_t)lm * 0x9E3779B1u ^ (prevRoot * 0x85EBCA6Bu) ^ (sp * 0xC2B2AE35u);
			h ^= h >> 15;
			return h & (HT_SIZE - 1);
		}

#if KB_SBG
		// ---- SkipBigram LM step: SbgState::nextImpl + SkipBigramModel::evaluate (src/SkipBigramModel.hpp:113-142, 169-182) ------------
		__device__ __noinline__ float sbgEvaluate(const uint32_t* hist, uint32_t next, float base)
		{
			float arr[16];
			#pragma unroll
			for (int i = 0; i < 8; ++i) { arr[i] = base; arr[8 + i] = -CUDART_INF_F; }
			const uint32_t b = c_m.sb_ptrs[next], e = c_m.sb_ptrs[next + 1];
			#pragma unroll 1
			for (int i = 0; i < 8; ++i)
			{
				const uint32_t hv = hist[i];
				arr[i] = c_m.sb_discnts[hv] + base;
				// nst::search over the target's key list = exact lookup; the image keeps the keys ascending
				uint32_t lo = b, hi = e;
				while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (c_m.sb_keys[mid] < hv) lo = mid + 1; else hi = mid; }
				if (lo < e && c_m.sb_keys[lo] == hv) arr[8 + i] = c_m.sb_comps[lo];
			}
			return sbgLogSumExp16(arr) - c_m.sb_log_window;
		}
		__device__ __forceinline__ float sbgNext(int32_t& node, uint32_t* hist, uint32_t& hpos, uint32_t wid)
		{
			float ll = knProgress(node, wid, 6);
			if (wid < c_m.sb_vocab_size && c_m.sb_valid[wid])
			{
#ifdef KB_HOSTSIM
				const float ll0 = ll;
#endif
				if (ll > -13.f) ll = sbgEvaluate(hist, wid, ll);
#ifdef KB_HOSTSIM
				if (std::getenv("HS32_TRACE_SBG")) std::fprintf(stderr, "[hs32] sbg wid %u base %a -> %a hist %u %u %u %u %u %u %u %u pos %u\n", wid, ll0, ll, hist[0], hist[1], hist[2], hist[3], hist[4], hist[5], hist[6], hist[7], hpos);
#endif
				#pragma unroll
				for (int i = 0; i < 8; ++i) if ((uint32_t)i == hpos) hist[i] = wid;      // (no dynamic register indexing)
				hpos = (hpos + 1) & 7;
			}
			return ll;
		}

#endif

		// ---- the path container of one candidate, item by item (BestPathContainer.hpp) -------------------------------------------------
		// The reference inserts a candidate's paths one after the other, and once a bucket holds 64 states the outcome depends on that order
		// in ways the parallel insert cannot model.  The SkipBigram build (states rarely merge) inserts every candidate this way; the Knlm /
		// CoNg builds re-run a group of candidates this way when one of their buckets has reached 64 states (evaluate: `exactInsert`):
		//  modes 0 / 1 (BucketedHashContainer::insertOptimized<avx2>, 316-383, with nst::findAll<avx2>, search.cpp:948-968), as the code
		//  BEHAVES on x86-64:
		//   - a bucket with fewer than 64 entries is searched properly (hash byte, then equalTo);
		//   - from 64 entries on, the candidate mask of the first 64 is ANDed with ((size_t)1 << 64) - 1, which the hardware evaluates as 0:
		//     none of them is ever found again;
		//   - the candidates among entries 64.. are tested with value[i] where value[64 + i] is meant: when entry i IS the new state,
		//     entry 64 + i (some other state with the same hash byte, or an earlier duplicate) is compared by score and overwritten;
		//   - 32 < size < 64: a match at byte 31 sign-extends the low mask, every position 32 .. size-1 becomes a candidate;
		//   - nothing found: the state is appended (again) while the bucket has room (128), else dropped.
		//  mode 2 (`top1`, an unordered_set, 229-276): plain set semantics, the better score replaces the entry.
		// Shared memory (the hash index `ht` of the other builds, unused here): modes 0 / 1 keep per bucket the entry index of every position
		// (bIdx) and the hash byte it was appended with (hb); mode 2 keeps an open-addressing index over all entries in global memory.
		__device__ __noinline__ void exactInsertRound(unsigned vmask, const PathT& np, uint32_t candBeg, uint32_t& E, uint32_t* bucketCnt, uint32_t mode)
		{
			uint16_t* bIdx = sm->ht;                                             // [4][128]
			uint8_t* hb = reinterpret_cast<uint8_t*>(sm->ht + 512);              // [4][128]
			static_assert(HT_SIZE >= 768, "bucket index fits the hash-index array");
			htUsed = 1;      // (the next htClear must really clear: the array holds bucket positions or index slots from here on)
			#pragma unroll 1
			while (vmask)
			{
				const int L = __ffs(vmask) - 1; vmask &= vmask - 1;
				const int32_t lm = __shfl_sync(FULL, np.lm_state, L);
				const float sc = __shfl_sync(FULL, np.acc_score, L);
#if KB_SBG
				const uint32_t idw = __shfl_sync(FULL, (uint32_t)np.prev_root_id | ((uint32_t)np.sp_state << 8) | (np.hpos << 16), L);
				uint32_t hh[8];
				#pragma unroll
				for (int i = 0; i < 8; ++i) hh[i] = __shfl_sync(FULL, np.hist[i], L);
				const unsigned long long h = __shfl_sync(FULL, np.hcode, L);
				auto eq = [&](const PathT* t)
				{
					if (t->lm_state != lm || ((uint32_t)t->prev_root_id | ((uint32_t)t->sp_state << 8) | (t->hpos << 16)) != idw) return false;
					bool same = true;
					#pragma unroll
					for (int i = 0; i < 8; ++i) same = same && t->hist[i] == hh[i];
					return same;
				};
#else
				// WordLL::equalTo: prevRootId, spState, LM state (the Knlm node; CoNg: the context-trie node only, CoNgramModel.hpp:491-494)
				const uint32_t idw = __shfl_sync(FULL, (uint32_t)np.prev_root_id | ((uint32_t)np.sp_state << 8), L);
				unsigned long long h;
				{
					// Hash<WordLL> (BestPathContainer.hpp:79-84) over Hash<LmState>: std::hash<int32_t> (Knlm.hpp:1170-1178) / Hash<uint32_t>(node) (CoNg)
#if KB_CONG
					const unsigned long long v = (uint32_t)lm;
					const unsigned long long h0 = (v * 2305843009213693951ull) ^ ((v << 33) | (v >> 31));
#else
					const unsigned long long h0 = (unsigned long long)(long long)lm;
#endif
					h = (unsigned long long)idw ^ ((h0 << 3) | (h0 >> 61));
				}
				auto eq = [&](const PathT* t) { return t->lm_state == lm && ((uint32_t)t->prev_root_id | ((uint32_t)t->sp_state << 8)) == idw; };
#endif
				uint32_t target = NPOS; bool append = false;
				uint32_t b = 0, n = 0;
#if KB_SBG
				if (mode == 2)
				{
					// open-addressing index over ALL entries of the candidate (slot = entry + 1), kept at the far end of the sentence's pool
					// region and doubled (rebuilt by lane 0) when half full: a candidate with tens of thousands of distinct states stays linear
					uint32_t* gi = reinterpret_cast<uint32_t*>(pool + poolCap) - sbIdxCap;
					if (2 * (E + 1) > sbIdxCap)
					{
						uint32_t cap = sbIdxCap ? sbIdxCap * 2 : 2048u;
						while (2 * (E + 1) > cap) cap *= 2;
						uint32_t* ng = reinterpret_cast<uint32_t*>(pool + poolCap) - cap;
						if (reinterpret_cast<const char*>(ng) < reinterpret_cast<const char*>(pool + candBeg + E + 2)) { err = ST_PATH_OVERFLOW; return; }
						#pragma unroll 1
						for (uint32_t i = lane; i < cap; i += 32) ng[i] = 0;
						__syncwarp();
						if (lane == 0)
						{
							#pragma unroll 1
							for (uint32_t e = 0; e < E; ++e)
							{
								const unsigned long long hc = pool[candBeg + e].hcode;
								uint32_t sl = ((uint32_t)(hc ^ (hc >> 29)) * 0x9E3779B1u) >> 7 & (cap - 1);
								while (ng[sl]) sl = (sl + 1) & (cap - 1);
								ng[sl] = e + 1;
							}
						}
						__syncwarp();
						sbIdxCap = cap; gi = ng;
					}
					else if (reinterpret_cast<const char*>(gi) < reinterpret_cast<const char*>(pool + candBeg + E + 2)) { err = ST_PATH_OVERFLOW; return; }
					const uint32_t imask = sbIdxCap - 1;
					uint32_t slot = ((uint32_t)(h ^ (h >> 29)) * 0x9E3779B1u) >> 7 & imask;
					#pragma unroll 1
					while (true)
					{
						const uint32_t e = gi[slot];
						if (!e) break;
						const PathT* t = pool + candBeg + (e - 1);
						if (t->hcode == h && eq(t)) { target = e - 1; break; }
						slot = (slot + 1) & imask;
					}
					append = target == NPOS;
					if (append && lane == 0) gi[slot] = E + 1;      // (the probe stopped at the first empty slot of this key's sequence)
				}
				else
#endif
				{
					b = mode == 1 ? ((uint32_t)(h >> 8) & 3u) : 0u; n = bucketCnt[b];
					const uint8_t hbNew = (uint8_t)h;
					const uint16_t* bi = bIdx + b * 128; const uint8_t* hv = hb + b * 128;
					uint32_t pos = NPOS;
					if (n < 64)
					{
						bool c0 = false;
						if (lane < n && hv[lane] == hbNew) c0 = eq(pool + candBeg + bi[lane]);
						const unsigned m0 = __ballot_sync(FULL, c0);
						if (m0) pos = __ffs(m0) - 1;
						else if (n > 32)
						{
							const uint32_t i = 32 + lane;
							bool c1 = false;
							if (i < n && (hv[i] == hbNew || hv[31] == hbNew)) c1 = eq(pool + candBeg + bi[i]);
							const unsigned m1 = __ballot_sync(FULL, c1);
							if (m1) pos = 32 + __ffs(m1) - 1;
						}
					}
					else
					{
						const uint32_t m = n - 64;
						if (m > 0 && m < 64)
						{
							bool c0 = false;
							if (lane < m && hv[64 + lane] == hbNew) c0 = eq(pool + candBeg + bi[lane]);      // value[i], as the reference reads it
							const unsigned m0 = __ballot_sync(FULL, c0);
							if (m0) pos = 64 + __ffs(m0) - 1;
							else if (m > 32)
							{
								const uint32_t i = 32 + lane;
								bool c1 = false;
								if (i < m && (hv[64 + i] == hbNew || hv[64 + 31] == hbNew)) c1 = eq(pool + candBeg + bi[i]);
								const unsigned m1 = __ballot_sync(FULL, c1);
								if (m1) pos = 64 + 32 + __ffs(m1) - 1;
							}
						}
					}
					if (pos != NPOS) target = bi[pos];
					append = target == NPOS && n < 128;
				}
				if (target != NPOS)
				{
					const PathT* t = pool + candBeg + target;
					if (sc > t->acc_score && lane == (uint32_t)L)
					{
						PathT w = np;
#if KB_SBG
						if (mode != 2) { w.prev_root_id = t->prev_root_id; w.hcode = t->hcode; }      // neither prevRootId nor the stored hash byte is refreshed (370-381)
#else
						w.prev_root_id = t->prev_root_id;
#endif
						pool[candBeg + target] = w;
					}
				}
				else if (append)
				{
					if (candBeg + E + 1 > poolCap) { err = ST_PATH_OVERFLOW; return; }
					if (E >= 0xFFFEu && mode != 2) { err = ST_PATH_OVERFLOW; return; }
					if (lane == (uint32_t)L) pool[candBeg + E] = np;
					if (mode != 2)
					{
						if (lane == 0) { bIdx[b * 128 + n] = (uint16_t)E; hb[b * 128 + n] = (uint8_t)h; }
						bucketCnt[b] = n + 1;
					}
					++E;
				}
				__syncwarp();
			}
		}

		// ---- evalSingleMorpheme, PathEvaluator.hpp:514-634 -------------------------------------------
		struct CandCtx
		{
			int32_t curId; DMorph cur; bool single;
			uint32_t firstWid0, lastSeqId;
			float additionalScore, ignoreCondScore;
			uint32_t specialType, sbType, sbOrder; bool positiveE, snEndswithPoint, fork;
			uint32_t ownOff, ownLen;
			uint32_t fwNew; uint8_t morphTag; uint32_t widFeat;      // fwNew: filter word of the created path (own form resolved, FW_COMMON_ROOT clear)
			bool spaceBefore;
#if KB_CONG
			uint32_t epFirst;        // epilogue of the first-wid score of a regular candidate (shape of the node's gather GEMM), CG_E_*
			int32_t dotCol;          // column of this candidate in sm->dots, -1 = not computed
#endif
		};

		// writeTo of the `top1` container (BestPathContainer.hpp:229-276): the candidate's E entries [candBeg, candBeg + E) are in
		// first-insertion order; the reference emits them in its unordered_set's iteration order (unordered_emu.h)
		// `bucketsBefore`: the set's bucket count before this container's first insertion; returns the count after it.  `scratch`: first
		// free pool slot (the segment may be followed by other candidates' entries)
		__device__ __noinline__ uint32_t reorderTop1(uint32_t candBeg, uint32_t E, uint32_t bucketsBefore, uint32_t scratch)
		{
			KB_PH_START(tReorder);
			if (E == 0) return bucketsBefore;
			const uint32_t Bafter = unorderedBucketsAfter(bucketsBefore, E);
			if (!Bafter) { err = ST_INTERNAL; return bucketsBefore; }
			if (E == 1) return Bafter;
			// (the reservation is 16 bytes per entry, of which the order takes 12; the containers that overflow the pool are the same as
			// when the order kept 64-bit hash codes in the scratch)
			const size_t need = (size_t)E * sizeof(PathT) + (size_t)E * 16 + (size_t)Bafter * 4;
			if ((size_t)scratch * sizeof(PathT) + need > (size_t)poolCap * sizeof(PathT)) { err = ST_PATH_OVERFLOW; return bucketsBefore; }
			PathT* tmp = pool + scratch;
			int32_t* first = reinterpret_cast<int32_t*>(pool + scratch + (size_t)E); int32_t* runs = first + E; int32_t* order = runs + E; int32_t* buckets = order + E;
			#pragma unroll 1
			for (uint32_t e = lane; e < E; e += 32) tmp[e] = pool[candBeg + e];
			__syncwarp();
			// Hash<WordLL> (BestPathContainer.hpp:79-84) over Hash<LmState>: std::hash<int32_t> for Knlm (Knlm.hpp:1170-1178), Hash<uint32_t>(node) for CoNg
			const auto codeOf = [tmp](int32_t i) -> unsigned long long
			{
				const PathT& p = tmp[i];
#if KB_SBG
				return p.hcode;
#else
#if KB_CONG
				const unsigned long long v = (uint32_t)p.lm_state;
				unsigned long long h = (v * 2305843009213693951ull) ^ ((v << 33) | (v >> 31));
#else
				unsigned long long h = (unsigned long long)(long long)p.lm_state;
#endif
				return (unsigned long long)((uint32_t)p.prev_root_id | ((uint32_t)p.sp_state << 8)) ^ ((h << 3) | (h >> 61));
#endif
			};
			uint32_t B = bucketsBefore;
			KB_PH_START(tOrder);
			if (!unorderedSetOrderWarp(codeOf, (int32_t)E, B, first, runs, buckets, order, lane)) { err = ST_INTERNAL; return bucketsBefore; }
			KB_PH_ADD(PH_TOP1_ORDER, tOrder, phSent);
			KB_PH_COUNT(PH_N_TOP1, 1, phSent); KB_PH_COUNT(PH_SUM_E, E, phSent); KB_PH_COUNT(PH_SUM_B, Bafter, phSent);
#if KB_PHASE_CLOCKS
			for (uint32_t b = bucketsBefore == 1 ? 13u : bucketsBefore; b != Bafter; b = unorderedNextBuckets(b)) KB_PH_COUNT(PH_REHASHES, 1, phSent);
#endif
			#pragma unroll 1
			for (uint32_t j = lane; j < E; j += 32) pool[candBeg + j] = tmp[order[j]];
			__syncwarp();
			KB_PH_ADD(PH_TOP1_REORDER, tReorder, phSent);
			return Bafter;
		}

		__device__ __noinline__ void evalCand(uint32_t nodeIdx, const DNode& node, const CandCtx& cc, uint32_t inBeg, uint32_t inEnd, uint32_t mode)
		{
			const uint32_t P = inEnd - inBeg;
			const uint32_t nRoot = cc.fork ? nUniq : 1;
			const uint32_t pairsPerRound = 32 / nRoot;
			const uint32_t candBeg = top;
			uint32_t E = 0;                           // entries of this candidate (all buckets)
			uint32_t bucketCnt[4] = { 0, 0, 0, 0 };
			uint32_t fwCarry = cc.firstWid0;
			htClear();
#if KB_SBG
			sbIdxCap = 0;      // (the `top1` index of the previous candidate is dead)
#endif
#if defined(KB_HOSTSIM) && !KB_CONG && !KB_SBG
			g_lmBigNode = P > HT_MAX_ENTRIES;
#endif
			const bool allowedSpaceBetweenChunk = c_m.cfg.space_tolerance > 0;

			for (uint32_t qb = 0; qb < P; qb += pairsPerRound)
			{
				const uint32_t pr = lane / nRoot, rr = lane % nRoot;
				const uint32_t q = qb + pr;
				bool valid = pr < pairsPerRound && q < P;
				PathT pp;
				if (valid) pp = pool[inBeg + q];
				float candScore = 0, firstChunkScore = 0;
				bool setsFW = false; uint32_t fwVal = 0;
				if (valid)
				{
#if KB_CONG
					// only the regular-candidate loop of the transposed evaluator has the z_siot test (CoNgramModel.cpp:184-189 vs 208-246)
					if (cc.cur.combine_socket == 0)
#endif
					if (pp.morph_tag == T_z_siot && (!isNNClass(cc.cur.feat & MF_TAG_MASK) || cc.spaceBefore)) valid = false;
				}
				if (valid)
				{
					candScore = pp.acc_score + cc.additionalScore;
					firstChunkScore = cc.additionalScore;
					if (pp.fw >> FW_SOCKET_SHIFT)
					{
						if ((pp.fw >> FW_SOCKET_SHIFT) != cc.cur.combine_socket || cc.single) valid = false;
						else if (cc.spaceBefore)
						{
							if (allowedSpaceBetweenChunk) candScore -= c_m.cfg.space_penalty;
							else valid = false;
						}
						if (valid)
						{
							setsFW = true;
							const DMorph pw = c_m.morphs[pp.wid];
							fwVal = c_m.morphs[(int32_t)pp.wid + pw.combined].lm_id;
						}
					}
				}
#if KB_CONG
				// right halves only see combining paths, and their first wid is local to the pair (CoNgramModel.cpp:248-286)
				if (valid && cc.cur.combine_socket && !cc.single && !(pp.fw >> FW_SOCKET_SHIFT)) valid = false;
				const uint32_t firstWid = setsFW ? fwVal : cc.firstWid0;
				(void)fwCarry;
				const bool regular = cc.cur.combine_socket == 0;
				float ignAdd = 0.f; bool ignLate = false;
#else
				// the reference mutates `firstWid` in place (PathEvaluator.hpp:590): later pairs inherit it
				uint32_t firstWid;
				{
					const unsigned smask = __ballot_sync(FULL, setsFW);
					const unsigned le = smask & (lane == 31 ? FULL : ((2u << lane) - 1));
					const int src = le ? 31 - __clz(le) : 0;
					const uint32_t got = __shfl_sync(FULL, fwVal, src);
					firstWid = le ? got : fwCarry;
					if (smask) fwCarry = __shfl_sync(FULL, fwVal, 31 - __clz(smask));
				}
#endif
				if (valid)
				{
					// FormEvaluator, PathEvaluator.hpp:253-311
					const bool empty = (pp.fw & FW_EMPTY) != 0;
					if (pp.fw & FW_NOCOND) {}      // SSC tag or a left form ending in a closing bracket
					else
					{
						const uint32_t cv = (cc.cur.feat >> MF_VOWEL_SHIFT) & 15, cp = (cc.cur.feat >> MF_POLAR_SHIFT) & 3;
						bool ok = ftVowelCls(empty, pp.fw & FW_CLS_MASK, cv);
						if (ok && (cp == CP_positive || cp == CP_negative))
						{
							ok = empty ? true : ((pp.fw & (cp == CP_positive ? FW_POLAR_POS : FW_POLAR_NEG)) != 0);
						}
#if KB_CONG
						// regular candidates: `score = acc + morphScore + lm` comes first, FormEvaluator adds afterwards (CoNgramModel.cpp:175-179)
						if (cc.ignoreCondScore != 0.f) { if (regular) { ignAdd = ok ? 0.f : cc.ignoreCondScore; ignLate = true; } else candScore += ok ? 0.f : cc.ignoreCondScore; }
						else if (!ok) valid = false;
#else
						if (cc.ignoreCondScore != 0.f) candScore += ok ? 0.f : cc.ignoreCondScore;
						else if (!ok) valid = false;
#endif
					}
				}
				int32_t lmState = 0;
#if KB_CONG
				uint32_t ctxIdx = 0;
				if (valid)
				{
					lmState = pp.lm_state; ctxIdx = P_CTX(pp);
					if (cc.cur.combine_socket && cc.single) {}
					else
					{
						if ((c_m.morphs[firstWid].feat & MF_TAG_MASK) == T_p) valid = false;
						else
						{
							float ll;
							if (regular)
							{
								// progressMatrix entry: tensor-core tile when this path's context is in the node's tile, else a dp4a dot
								const uint32_t ps = q < STAGE_CAP ? sm->pslot[q] : 0xFFu;
								const int32_t x = (cc.dotCol >= 0 && ps != 0xFFu) ? sm->dots[ps][cc.dotCol] : cgDot(ctxIdx, firstWid);
								ll = cgFinish(x, ctxIdx, firstWid, cc.epFirst);
								ctxIdx = cgStep(lmState, firstWid);
							}
							else ll = cgNext(lmState, ctxIdx, firstWid);
							candScore += ll;
							firstChunkScore += ll;
							if (ignLate) candScore += ignAdd;
							if (!cc.single)
							{
								for (uint32_t i = 1; i < cc.cur.chunk_cnt; ++i)
								{
									const uint32_t wid = c_m.morphs[c_m.chunks[cc.cur.chunk_off + i].morph].lm_id;
									if ((c_m.morphs[wid].feat & MF_TAG_MASK) == T_p) { valid = false; break; }
									ll = cgNext(lmState, ctxIdx, wid);
									candScore += ll;
								}
							}
						}
					}
				}
#else
#if KB_SBG
				uint32_t hist[8] = { 0, 0, 0, 0, 0, 0, 0, 0 }, hpos = 0;
				if (valid) { for (int i = 0; i < 8; ++i) hist[i] = pp.hist[i]; hpos = pp.hpos; }
#define KB_LM_STEP(w, site) sbgNext(lmState, hist, hpos, (w))
#else
#define KB_LM_STEP(w, site) knProgress(lmState, (w), (site))
#endif
				if (valid)
				{
					lmState = pp.lm_state;
					if (cc.cur.combine_socket && cc.single) {}
					else
					{
						if ((c_m.morphs[firstWid].feat & MF_TAG_MASK) == T_p) valid = false;
						else
						{
							float ll = KB_LM_STEP(firstWid, 3);
							candScore += ll;
							firstChunkScore += ll;
							if (!cc.single)
							{
								for (uint32_t i = 1; i < cc.cur.chunk_cnt; ++i)
								{
									const uint32_t wid = c_m.morphs[c_m.chunks[cc.cur.chunk_off + i].morph].lm_id;
									if ((c_m.morphs[wid].feat & MF_TAG_MASK) == T_p) { valid = false; break; }
									ll = KB_LM_STEP(wid, 4);
									candScore += ll;
								}
							}
						}
					}
				}
#endif
				// insertToPathContainer, PathEvaluator.hpp:193-251
				uint8_t spState = 0, rootId = COMMON_ROOT;
				float accScore = 0, fcs = 0;
				if (valid)
				{
					const bool doFork = cc.fork && pp.root_id == COMMON_ROOT;
					if (!doFork && rr != 0) valid = false;
					else
					{
						rootId = doFork ? (uint8_t)rr : COMMON_ROOT;
						spState = doFork ? uniq[rr] : pp.sp_state;
						// RuleBasedScorer::operator(), PathEvaluator.hpp:115-183
						const uint32_t pf = P_WID_FEAT(pp);
						const uint32_t ptag = pf & MF_TAG_MASK;
						float rs = 0;
						if ((cc.cur.feat & MF_VOWEL_E) && isIrregular((uint8_t)ptag)) rs -= 10;
						if ((cc.cur.feat & MF_INF_J) && (pf & MF_INFL_NP)) rs -= 5;
						if ((cc.cur.feat & MF_BADPAIR_L) && (pf & MF_VERB_L)) rs -= 7;
						if (cc.positiveE && !(pf & MF_POS_VERB)) rs -= 100;
						if ((cc.cur.feat & MF_CONTRACT_E) && (pf & MF_VERB_VOWEL)) rs -= 3;
						if (((cc.cur.feat >> MF_POLAR_SHIFT) & 3) == CP_non_adj && (ptag == T_va || ptag == T_xsa)) rs -= 10;
						const uint32_t sq = spState & 1, dq = (spState >> 1) & 1, bh = spState >> 2;
						if (cc.specialType <= 2) { if (cc.specialType != sq) rs -= 2; }
						else if (cc.specialType <= 5) { if (cc.specialType - 3 != dq) rs -= 2; }
						if (cc.sbType == 5) rs -= 5;
						if (cc.sbType && isEClass((uint8_t)ptag) && ptag != T_ef) rs -= 10;
						if (cc.sbType && bh == hashSbTypeOrder((uint8_t)cc.sbType, (uint8_t)cc.sbOrder)) rs += 3;
						if (cc.snEndswithPoint && (ptag == T_unknown || ptag == T_ef || ptag == T_sf)) rs -= 5;
						accScore = candScore + rs;
						fcs = firstChunkScore + rs;
						if (cc.specialType == 0) spState |= 1;
						else if (cc.specialType == 1) spState &= ~1;
						else if (cc.specialType == 3) spState |= 2;
						else if (cc.specialType == 4) spState &= ~2;
						if (cc.sbType) spState = (spState & 3) | (uint8_t)(hashSbTypeOrder((uint8_t)cc.sbType, (uint8_t)(cc.sbOrder + 1)) << 2);
						accScore = accScore - 0.f;      // curDialectCost (standard dialect only)
						fcs = fcs - 0.f;
					}
				}

				// ---- warp-cooperative BucketedHashContainer::insert for the (<= 32) items of this round
				const uint32_t prevRoot = pp.root_id;
				const unsigned vmask = __ballot_sync(FULL, valid);
				if (!vmask) continue;
				if (KB_SBG || (mode != 2 && sm->exactInsert))
				{
					// every valid lane prepares its path record; the container takes them one at a time, in pair order (exactInsertRound)
					PathT np;
					if (valid)
					{
						np.lm_state = lmState; np.acc_score = accScore; np.first_chunk_score = fcs; np.wid = cc.lastSeqId;
						np.morpheme = cc.curId; np.parent = inBeg + q; np.own_off = cc.single ? cc.ownOff : 0; np.acc_typo_cost = pp.acc_typo_cost + node.typo_cost;
						np.own_len = cc.single ? (uint16_t)cc.ownLen : 0; np.node = (uint16_t)nodeIdx;
						np.sp_state = spState;
						np.root_id = rootId != COMMON_ROOT ? rootId : pp.root_id;
						np.fw = cc.fwNew | (np.root_id == COMMON_ROOT ? (uint32_t)FW_COMMON_ROOT : 0u);
						np.prev_root_id = (uint8_t)prevRoot; np.morph_tag = cc.morphTag;
#if KB_CONG
						P_CTX(np) = ctxIdx;
#else
						np.wid_feat = cc.widFeat;
#endif
#if KB_SBG
						for (int i = 0; i < 8; ++i) np.hist[i] = hist[i];
						np.hpos = hpos; np.hpad = 0;
						// Hash<WordLL<SbgState>>: Knlm node, the 8 ring slots, then prevRootId | spState << 8 (SkipBigramModel.hpp:188-203, BestPathContainer.hpp:79-84)
						unsigned long long h = (unsigned long long)(long long)lmState;
						for (int i = 0; i < 8; ++i) h = (unsigned long long)hist[i] ^ ((h << 3) | (h >> 61));
						np.hcode = (unsigned long long)((prevRoot & 0xFFu) | ((uint32_t)spState << 8)) ^ ((h << 3) | (h >> 61));
#endif
					}
					exactInsertRound(vmask, np, candBeg, E, bucketCnt, mode);
					if (err) return;
					continue;
				}
				const unsigned long long key = valid
					? ((unsigned long long)(uint32_t)lmState | ((unsigned long long)prevRoot << 32) | ((unsigned long long)spState << 40))
					: (0xFFFF000000000000ull | lane);
				const unsigned grp = __match_any_sync(FULL, key);
				// best of the group: max score, earliest lane on ties
				uint32_t ord = __float_as_uint(accScore);
				ord = (ord & 0x80000000u) ? ~ord : (ord | 0x80000000u);
				const uint32_t gmax = __reduce_max_sync(grp, ord);
				const unsigned bestMask = __ballot_sync(FULL, valid && ord == gmax) & grp;
				const uint32_t bestLane = __ffs(bestMask) - 1;
				const uint32_t leader = __ffs(grp) - 1;
				const bool isLeader = valid && lane == leader;
				// lookup among the entries of earlier rounds
				uint32_t found = NPOS;
#if KB_CONG
				// Hash<CoNgramState> = Hash<uint32_t>(node) = node * (2^61 - 1) ^ rol(node, 33): its bits 5-6 are those of -node (CoNgramModel.hpp:505-541)
				const uint32_t bucket = mode == 1 ? ((spState ^ ((0u - (uint32_t)lmState) >> 5)) & 3) : 0;
#else
				const uint32_t bucket = mode == 1 ? ((spState ^ ((uint32_t)lmState >> 5)) & 3) : 0;
#endif
				if (isLeader && E)
				{
					uint32_t slot = htHash(lmState, prevRoot, spState);
					while (true)
					{
						const uint32_t e = ht[slot];
						if (!e) break;
						const PathT* t = pool + candBeg + (e - 1);
						if (t->lm_state == lmState && t->prev_root_id == prevRoot && t->sp_state == spState) { found = e - 1; break; }
						slot = (slot + 1) & (HT_SIZE - 1);
					}
				}
				// new keys are appended in lane (= pair) order; a full 128-slot bucket drops the key (BestPathContainer.hpp:363-367)
				const bool isNew = isLeader && found == NPOS;
				uint32_t newIdx = NPOS;
				{
					const unsigned nmask = __ballot_sync(FULL, isNew);
					if (mode == 2)
					{
						if (isNew) newIdx = E + __popc(nmask & ((1u << lane) - 1));
					}
					else
					{
						// capacity per bucket; rank inside the bucket in lane order
						uint32_t accepted = 0;
#pragma unroll
						for (uint32_t b = 0; b < 4; ++b)
						{
							const unsigned bm = __ballot_sync(FULL, isNew && bucket == b);
							if (isNew && bucket == b)
							{
								const uint32_t r = __popc(bm & ((1u << lane) - 1));
								if (bucketCnt[b] + r < 128) accepted = 1;
							}
							const uint32_t add = min((uint32_t)__popc(bm), 128u - bucketCnt[b]);
							bucketCnt[b] += add;
						}
						const unsigned amask = __ballot_sync(FULL, accepted != 0);
						if (accepted) newIdx = E + __popc(amask & ((1u << lane) - 1));
						if (isNew && !accepted) newIdx = NPOS;
						// total new entries this round
						const uint32_t totalNew = __popc(amask);
						if (candBeg + E + totalNew > poolCap) { err = ST_PATH_OVERFLOW; return; }
						if (E + totalNew > HT_MAX_ENTRIES) { err = ST_PATH_OVERFLOW; return; }
						// insert into the hash index
						if (accepted)
						{
							uint32_t slot = htHash(lmState, prevRoot, spState);
							while (atomicCAS_u16(ht, slot, newIdx + 1)) slot = (slot + 1) & (HT_SIZE - 1);
						}
						E += totalNew;
						htUsed = 1;
						goto inserted;
					}
					{
						const uint32_t totalNew = __popc(nmask);
						if (candBeg + E + totalNew > poolCap) { err = ST_PATH_OVERFLOW; return; }
						if (E + totalNew > HT_MAX_ENTRIES) { err = ST_PATH_OVERFLOW; return; }
						if (isNew)
						{
							uint32_t slot = htHash(lmState, prevRoot, spState);
							while (atomicCAS_u16(ht, slot, newIdx + 1)) slot = (slot + 1) & (HT_SIZE - 1);
						}
						E += totalNew;
						htUsed = 1;
					}
				}
			inserted:
				__syncwarp();
				// the group's best lane writes the entry: new key -> create, existing key -> strict '>' update
				{
					const uint32_t tgtNew = __shfl_sync(FULL, newIdx, leader);
					const uint32_t tgtOld = __shfl_sync(FULL, found, leader);
					if (valid && lane == bestLane)
					{
						uint32_t tgt = tgtOld != NPOS ? tgtOld : tgtNew;
						bool write = tgt != NPOS;
						if (write && tgtOld != NPOS) write = accScore > pool[candBeg + tgt].acc_score;
						if (write)
						{
							PathT np;
							np.lm_state = lmState; np.acc_score = accScore; np.first_chunk_score = fcs; np.wid = cc.lastSeqId;
							np.morpheme = cc.curId; np.parent = inBeg + q; np.own_off = cc.single ? cc.ownOff : 0; np.acc_typo_cost = pp.acc_typo_cost + node.typo_cost;
							np.own_len = cc.single ? (uint16_t)cc.ownLen : 0; np.node = (uint16_t)nodeIdx;
							np.sp_state = spState;
							np.root_id = rootId != COMMON_ROOT ? rootId : pp.root_id;
							np.fw = cc.fwNew | (np.root_id == COMMON_ROOT ? (uint32_t)FW_COMMON_ROOT : 0u);
							np.prev_root_id = (uint8_t)prevRoot; np.morph_tag = cc.morphTag;
#if KB_CONG
							P_CTX(np) = ctxIdx;
#else
							np.wid_feat = cc.widFeat;
#endif
							pool[candBeg + tgt] = np;
						}
					}
				}
				__syncwarp();
			}
			// writeTo (BestPathContainer.hpp:451-469): bucket-major order in medium mode
			if (mode == 1 && E > 1 && (bucketCnt[0] != E))
			{
				if (candBeg + 2 * E > poolCap) { err = ST_PATH_OVERFLOW; return; }
				uint32_t base[4]; base[0] = 0; base[1] = bucketCnt[0]; base[2] = base[1] + bucketCnt[1]; base[3] = base[2] + bucketCnt[2];
				uint32_t fill[4] = { 0, 0, 0, 0 };
				for (uint32_t eb = 0; eb < E; eb += 32)
				{
					const uint32_t e = eb + lane;
					PathT p; uint32_t b = 0xFF;
#if KB_SBG
					if (e < E) { p = pool[candBeg + e]; b = (uint32_t)(p.hcode >> 8) & 3; }
#elif KB_CONG
					if (e < E) { p = pool[candBeg + e]; b = (p.sp_state ^ ((0u - (uint32_t)p.lm_state) >> 5)) & 3; }
#else
					if (e < E) { p = pool[candBeg + e]; b = (p.sp_state ^ ((uint32_t)p.lm_state >> 5)) & 3; }
#endif
#pragma unroll
					for (uint32_t k = 0; k < 4; ++k)
					{
						const unsigned bm = __ballot_sync(FULL, b == k);
						if (b == k) pool[candBeg + E + base[k] + fill[k] + __popc(bm & ((1u << lane) - 1))] = p;
						fill[k] += __popc(bm);
					}
				}
				__syncwarp();
				for (uint32_t e = lane; e < E; e += 32) pool[candBeg + e] = pool[candBeg + E + e];
				__syncwarp();
			}
#ifdef KB_HOSTSIM
			if (lane == 0 && std::getenv("HS32_TRACE_CAND")) std::fprintf(stderr, "[cand] node %u cand %d mode %u E %u buckets %u %u %u %u\n", nodeIdx, cc.curId, mode, E, bucketCnt[0], bucketCnt[1], bucketCnt[2], bucketCnt[3]);
#endif
			top = candBeg + E;      // (mode 2: the container's write-out order is applied per candidate segment by fixupGroup)
		}

		static __device__ __forceinline__ bool atomicCAS_u16(uint16_t* ht, uint32_t slot, uint32_t val)
		{
			// returns true when the slot was occupied (caller probes on).  16-bit CAS on a 32-bit word.
			uint32_t* w = reinterpret_cast<uint32_t*>(ht) + (slot >> 1);
			const uint32_t shift = (slot & 1) * 16;
			while (true)
			{
				const uint32_t old = *reinterpret_cast<volatile uint32_t*>(w);
				if ((old >> shift) & 0xFFFF) return true;
				if (atomicCAS(w, old, old | (val << shift)) == old) return false;
			}
		}


		// ---- candidate rows: TMA-style bulk staging --------------------------------------------------------------------
		// The candidate rows of a lattice node are one contiguous block of DevModel::cands, known before the node is evaluated
		// (node_cand, filled per chunk by lane-parallel loads).  While node i is evaluated, lane 0 issues ONE bulk copy
		// (cp.async.bulk.shared.global with an mbarrier transaction count) of node i+1's first 32 rows into the other buffer; node
		// i+1 then only waits on the barrier's phase.  Groups beyond the first 32 candidates, the unknown-form re-evaluations and the
		// CoNg build (reordered candidates) store their rows from registers instead.
#if !KB_CONG && !defined(KB_HOSTSIM) && !defined(KB_NO_TMA)
#define KB_TMA_ROWS 1
		static __device__ __forceinline__ uint32_t smemAddr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
		__device__ void pfInit()
		{
			if (lane == 0)
			{
				asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smemAddr(&sm->mbar[0])) : "memory");
				asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smemAddr(&sm->mbar[1])) : "memory");
				asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
			}
			__syncwarp();
		}
		// issue the copy of `cnt` rows (1..32) into buffer `buf`; every issue is matched by exactly one pfWait on that buffer
		__device__ __forceinline__ void pfIssue(const DCand* base, uint32_t cnt, uint32_t buf)
		{
			__syncwarp();      // all lanes are done reading the buffer's previous contents
			if (lane == 0)
			{
				const uint32_t bytes = cnt * (uint32_t)sizeof(DCand), bar = smemAddr(&sm->mbar[buf]);
				asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory");
				asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
					:: "r"(smemAddr(&sm->dcandBuf[buf][0])), "l"(base), "r"(bytes), "r"(bar) : "memory");
			}
			pfBase[buf] = base;
		}
		__device__ __forceinline__ void pfWait(uint32_t buf)
		{
			const uint32_t bar = smemAddr(&sm->mbar[buf]), parity = (pfPhase >> buf) & 1u;
			asm volatile("{\n.reg .pred P1;\nLAB_WAIT:\nmbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n@P1 bra DONE;\nbra LAB_WAIT;\nDONE:\n}" :: "r"(bar), "r"(parity) : "memory");
			pfPhase ^= 1u << buf;
			pfBase[buf] = nullptr;
		}
		// a sentence that stopped on an error may leave a copy in flight: wait for it before the buffers serve the next sentence
		__device__ void pfDrain() { if (pfBase[0] != nullptr) pfWait(0); if (pfBase[1] != nullptr) pfWait(1); }
#else
#define KB_TMA_ROWS 0
#endif

		// ---- the item pipeline (containers of <= 512 incoming paths: the reference's top1Small / top1Medium) --------
		// Every path carries its filter word (DPath::fw, computed when the path was created); the distinct words of a node's
		// incoming paths become "path classes" (a handful per node).  Candidates are classified 32 at a time, one lane per
		// candidate, from their static DCand rows; each lane decides per path class whether a pair survives the reference's
		// filter (z_siot / combine socket / FormEvaluator conditions), so the per-pair filter is a bit test.  For every
		// candidate, in order, the survivors are compacted by ballot into an item list that is drained 32 items at a time
		// ACROSS candidate boundaries, so the Knlm pointer chase runs with full lanes.
		// Items are in (candidate, path, root) order and new container entries are appended in item order, hence the
		// pool receives them candidate-major in first-insertion order = the write-out order of the reference's
		// per-candidate containers.  Keys are independent of each other, so the 128-slot capacity of a container
		// bucket ("skip insertion if container is full", BestPathContainer.hpp:363-367) and the bucket-major order of
		// the 4 x 128 medium container are applied afterwards per candidate segment (fixupGroup).
		__device__ KB_INL1 void stagePaths(uint32_t nodeIdx, uint32_t inBeg, uint32_t P)
		{
			if (stagedNode == nodeIdx) return;
			nClasses = 0; classCommon = 0; classOverflow = false;
			uint32_t myTab = 0;      // lane z keeps class z's filter word
			#pragma unroll 1
			for (uint32_t qb = 0; qb < P; qb += 32)
			{
				const uint32_t q = qb + lane;
				const uint32_t w = q < P ? pool[inBeg + q].fw : 0xFFFFFFFFu;
				unsigned rem = __ballot_sync(FULL, q < P);
				uint32_t myIdx = 0;
				while (rem)
				{
					const int src = __ffs(rem) - 1;
					const uint32_t v = __shfl_sync(FULL, w, src);
					const unsigned hit = __ballot_sync(FULL, lane < nClasses && myTab == v);
					uint32_t idx;
					if (hit) idx = __ffs(hit) - 1;
					else if (nClasses >= 32) { classOverflow = true; idx = 0; }
					else
					{
						idx = nClasses++;
						if (lane == idx) myTab = v;
						if (v & FW_COMMON_ROOT) classCommon |= 1u << idx;
					}
					const unsigned same = __ballot_sync(FULL, w == v);
					if (w == v) myIdx = idx;
					rem &= ~same;
				}
				if (q < P) sm->pcls[q] = (uint8_t)myIdx;
			}
			if (lane < nClasses) sm->fclass[lane] = myTab;
			stagedNode = nodeIdx;
			__syncwarp();
		}

		struct FlushCtx
		{
			uint32_t nodeIdx; uint32_t inBeg; float ignoreCondScore; float nodeTypoCost; uint32_t ownOff, ownLen;
			uint32_t ownFw;      // left-form part of the filter word of a path that keeps the node's own form
			uint32_t inEnd, mode, spaceBefore;      // (for the cold group redo: kept here, not in registers)
#if KB_CONG
			uint32_t epFirst, dotMask;      // epilogue of the node's gather GEMM; candidates of the current group that have a column in sm->dots
#endif
		};

		// the `nItems` items in sm->item; false when the pool overflowed (err is set).  Out of line: it has several call sites, and
		// instruction-cache misses are the kernel's other large stall.  The members it reads are copied to registers (see Vit), and
		// htCount / htUsed / top are written back once.
		__device__ __noinline__ bool flushItems(const FlushCtx& fcIn, uint32_t nItems)
		{
			if (!nItems) return true;
			const FlushCtx fc = fcIn;
			PathT* const pool = this->pool; WarpSmem* const sm = this->sm; uint16_t* const ht = this->ht; const DCand* const dcur = this->dcur;
			const uint32_t lane = this->lane, poolCap = this->poolCap, htBase = this->htBase;
			const uint8_t uniq0 = uniq[0], uniq1 = uniq[1];
			uint32_t htCount = this->htCount, htUsed = this->htUsed;
			KB_HS_CHAIN_FLUSH();
			__syncwarp();
			#pragma unroll 1
			for (uint32_t ib = 0; ib < nItems; ib += 32)
			{
				const uint32_t i = ib + lane;
				KB_HS_CHAIN_ROUND_BEGIN();
				const bool valid = i < nItems;
				uint32_t slot = 0, q = 0, r = 0, fwIdx = 0; bool condFail = false, spacePen = false;
				if (valid) { const uint32_t it = sm->item[i]; slot = it >> 27; fwIdx = (it >> 20) & 63; q = (it >> 3) & 0x1FFFF; spacePen = (it >> 2) & 1; r = (it >> 1) & 1; condFail = it & 1; }
				const DCand* cs = &dcur[slot];
				const CandDyn cd = sm->cdyn[slot];
				const uint32_t csFeat = cs->feat;
				const int32_t csCurId = cs->cur_id;
				int32_t lmState = 0; float accScore = 0, fcs = 0, typoAcc = 0; uint32_t prevRoot = 0; uint8_t spState = 0, rootId = COMMON_ROOT;
#if KB_CONG
				uint32_t ctxIdx = 0;
#endif
				if (valid)
				{
					const PathT* pp = pool + fc.inBeg + q;
					const uint4 s0 = *reinterpret_cast<const uint4*>(&pp->lm_state);      // lm_state, acc_score, acc_typo_cost, wid_feat
					const uint32_t meta = *reinterpret_cast<const uint32_t*>(&pp->sp_state);   // sp_state | root_id << 8 | prev_root_id << 16 | morph_tag << 24
					prevRoot = (meta >> 8) & 0xFF;
					const bool doFork = (cd.flags & CS_FORK) && prevRoot == COMMON_ROOT;
					spState = doFork ? (r ? uniq1 : uniq0) : (uint8_t)(meta & 0xFF);
					rootId = doFork ? (uint8_t)r : COMMON_ROOT;
					typoAcc = __uint_as_float(s0.z);
					float candScore = __uint_as_float(s0.y) + cd.additionalScore;
					float firstChunkScore = cd.additionalScore;
					if (spacePen) candScore -= c_m.cfg.space_penalty;
#if KB_CONG
					// regular candidates: FormEvaluator's soft penalty comes after `acc + morphScore + lm` (CoNgramModel.cpp:175-179)
					const bool cgRegular = !(cd.flags & (CS_NO_LM | CS_SOCKET_CHUNK));
					if (condFail && !cgRegular) candScore += fc.ignoreCondScore;
					ctxIdx = s0.w;
					const uint32_t pf = c_m.morphs[pp->wid].feat;
#else
					if (condFail) candScore += fc.ignoreCondScore;
					const uint32_t pf = s0.w;
#endif
					lmState = (int32_t)s0.x;
					const uint32_t firstWid = fwIdx ? sm->fwTab[fwIdx] : cs->first_wid;
#if KB_CONG
					if (!(cd.flags & CS_NO_LM))
					{
						float ll;
						if (cgRegular)
						{
							const uint32_t ps = q < STAGE_CAP ? sm->pslot[q] : 0xFFu;
							const int32_t x = (((fc.dotMask >> slot) & 1u) && ps != 0xFFu) ? sm->dots[ps][slot] : cgDot(ctxIdx, firstWid);
							ll = cgFinish(x, ctxIdx, firstWid, fc.epFirst);
							ctxIdx = cgStep(lmState, firstWid);
						}
						else ll = cgNext(lmState, ctxIdx, firstWid);
						candScore += ll; firstChunkScore += ll;
						if (condFail && cgRegular) candScore += fc.ignoreCondScore;
						if (!(cd.flags & CS_SINGLE))
						{
							const uint32_t co = cs->chunk_off, cc = cs->chunk_cnt;
							#pragma unroll 1
							for (uint32_t c = 1; c < cc; ++c) { ll = cgNext(lmState, ctxIdx, c_m.chunk_lm[co + c]); candScore += ll; }
						}
					}
#else
					if (!(cd.flags & CS_NO_LM))
					{
#ifdef KB_INLINE_KN
						const KnRes kr0 = knProgressI(lmState, firstWid); lmState = kr0.node;
						float ll = kr0.ll;
#else
						float ll = knProgress(lmState, firstWid, 1);
#endif
						candScore += ll; firstChunkScore += ll;
						if (!(cd.flags & CS_SINGLE))
						{
							const uint32_t co = cs->chunk_off, cc = cs->chunk_cnt;
							#pragma unroll 1
							for (uint32_t c = 1; c < cc; ++c) { ll = knProgress(lmState, c_m.chunk_lm[co + c], 2); candScore += ll; }
						}
					}
#endif
					KB_HS_CHAIN_ROUND_END(ib);
					// RuleBasedScorer::operator() + special-state update (PathEvaluator.hpp:115-183, 208-230)
					const uint32_t ptag = pf & MF_TAG_MASK;
					const uint32_t specialType = (csFeat >> MF_SPECIAL_SHIFT) & 7, sbType = (csFeat >> MF_SBTYPE_SHIFT) & 31;
					float rs = 0;
					if ((csFeat & MF_VOWEL_E) && isIrregular((uint8_t)ptag)) rs -= 10;
					if ((csFeat & MF_INF_J) && (pf & MF_INFL_NP)) rs -= 5;
					if ((csFeat & MF_BADPAIR_L) && (pf & MF_VERB_L)) rs -= 7;
					if ((cd.flags & CS_POSITIVE_E) && !(pf & MF_POS_VERB)) rs -= 100;
					if ((csFeat & MF_CONTRACT_E) && (pf & MF_VERB_VOWEL)) rs -= 3;
					if (((csFeat >> MF_POLAR_SHIFT) & 3) == CP_non_adj && (ptag == T_va || ptag == T_xsa)) rs -= 10;
					const uint32_t sq = spState & 1, dq = (spState >> 1) & 1;
					if (specialType <= 2) { if (specialType != sq) rs -= 2; }
					else if (specialType <= 5) { if (specialType - 3 != dq) rs -= 2; }
					if (sbType)
					{
						const uint32_t sbOrder = cs->sense_id, bh = spState >> 2;
						if (sbType == 5) rs -= 5;
						if (isEClass((uint8_t)ptag) && ptag != T_ef) rs -= 10;
						if (bh == hashSbTypeOrder((uint8_t)sbType, (uint8_t)sbOrder)) rs += 3;
					}
					if ((cd.flags & CS_SN_POINT) && (ptag == T_unknown || ptag == T_ef || ptag == T_sf)) rs -= 5;
					accScore = candScore + rs;
					fcs = firstChunkScore + rs;
					if (specialType == 0) spState |= 1;
					else if (specialType == 1) spState &= ~1;
					else if (specialType == 3) spState |= 2;
					else if (specialType == 4) spState &= ~2;
					if (sbType) spState = (spState & 3) | (uint8_t)(hashSbTypeOrder((uint8_t)sbType, (uint8_t)(cs->sense_id + 1)) << 2);
					accScore = accScore - 0.f; fcs = fcs - 0.f;        // curDialectCost (standard dialect only)
				}
				// de-duplication by (candidate, lmState, prevRootId, spState): best score, earliest item on ties
				const unsigned long long key = valid
					? ((unsigned long long)(uint32_t)lmState | ((unsigned long long)prevRoot << 32) | ((unsigned long long)spState << 40) | ((unsigned long long)slot << 48))
					: (0xFFFF000000000000ull | lane);
				const unsigned grp = __match_any_sync(FULL, key);
				uint32_t ord = __float_as_uint(accScore);
				ord = (ord & 0x80000000u) ? ~ord : (ord | 0x80000000u);
				uint32_t gmax = ord;
				if (grp != (1u << lane)) gmax = __reduce_max_sync(grp, ord);          // most keys are unique inside a round
				const unsigned bestMask = __ballot_sync(FULL, valid && ord == gmax) & grp;
				const uint32_t bestLane = __ffs(bestMask) - 1;
				const uint32_t leader = __ffs(grp) - 1;
				const bool isLeader = valid && lane == leader;
				uint32_t found = NPOS;
				const uint32_t h0 = htHash(lmState, prevRoot | (slot << 8), spState);
				if (isLeader && htCount)
				{
					uint32_t hs = h0;
					while (true)
					{
						const uint32_t e = ht[hs];
						if (!e) break;
						const PathT* tp = pool + htBase + (e - 1);
						if (tp->lm_state == lmState && tp->morpheme == csCurId && tp->prev_root_id == prevRoot && tp->sp_state == spState) { found = e - 1; break; }
						hs = (hs + 1) & (HT_SIZE - 1);
					}
				}
				const bool isNew = isLeader && found == NPOS;
				const unsigned nmask = __ballot_sync(FULL, isNew);
				const uint32_t totalNew = __popc(nmask);
				uint32_t newIdx = NPOS;
				if (isNew) newIdx = htCount + __popc(nmask & ((1u << lane) - 1));
				if (htBase + htCount + totalNew > poolCap || htCount + totalNew > HT_MAX_ENTRIES)
				{
					err = ST_PATH_OVERFLOW; this->htCount = htCount; this->htUsed = htUsed;
					return false;
				}
				if (isNew)
				{
					uint32_t hs = h0;
					while (atomicCAS_u16(ht, hs, newIdx + 1)) hs = (hs + 1) & (HT_SIZE - 1);
					atomicAdd(&sm->candNew[slot], 1u);
				}
				if (totalNew) htUsed = 1;
				htCount += totalNew;
				__syncwarp();
				const uint32_t tgtNew = __shfl_sync(FULL, newIdx, leader);
				const uint32_t tgtOld = __shfl_sync(FULL, found, leader);
				if (valid && lane == bestLane)
				{
					const uint32_t tgt = tgtOld != NPOS ? tgtOld : tgtNew;
					bool write = true;
					if (tgtOld != NPOS) write = accScore > pool[htBase + tgt].acc_score;
					if (write)
					{
						const bool own = (cd.flags & CS_SINGLE) && fc.ownLen;
						const uint8_t tag = (uint8_t)(csFeat & MF_TAG_MASK);
						PathT np;
						np.lm_state = lmState; np.acc_score = accScore; np.acc_typo_cost = typoAcc + fc.nodeTypoCost;
#if KB_CONG
						P_CTX(np) = ctxIdx;
#else
						np.wid_feat = cs->last_seq_feat;
#endif
						np.sp_state = spState; np.root_id = rootId != COMMON_ROOT ? rootId : (uint8_t)prevRoot; np.prev_root_id = (uint8_t)prevRoot; np.morph_tag = tag;
						const uint32_t fwNew = cs->fw_new;
						np.fw = (own ? (fc.ownFw | (fwNew & FW_MORPH_SOCKET) | fwOfTag(tag, cs->path_socket)) : fwNew) | (np.root_id == COMMON_ROOT ? (uint32_t)FW_COMMON_ROOT : 0u);
						np.first_chunk_score = fcs; np.wid = cs->last_seq_id;
						np.morpheme = csCurId; np.parent = fc.inBeg + q; np.own_off = own ? fc.ownOff : 0;
						np.own_len = own ? (uint16_t)fc.ownLen : 0; np.node = (uint16_t)fc.nodeIdx;
						pool[htBase + tgt] = np;
					}
				}
				__syncwarp();
			}
			this->htCount = htCount; this->htUsed = htUsed;
			top = htBase + htCount;
			return true;
		}

		__device__ void resetIndex()
		{
			htClear();
			htBase = top; htCount = 0;
		}

		// the group's candidates whose container has a bucket of 64 (distinct) states or more (bit k: candidate k).  Segments: candidate k's
		// entries follow candidate k - 1's, sm->candNew[k] of them, in first-insertion order
		__device__ __noinline__ uint32_t groupExactMask(uint32_t groupBase, uint32_t gcount, uint32_t mode)
		{
			const uint32_t cn = lane < gcount ? sm->candNew[lane] : 0;
			const uint8_t cl = lane < gcount ? sm->cdyn[lane].cls : CLS_SKIP;
			const unsigned big = __ballot_sync(FULL, cn >= KB_EXACT_FROM && (cl == CLS_ITEM || cl == CLS_GENERAL));
			if (!big || mode == 0) return big;
			// medium mode: 4 buckets, count the largest one of every big candidate
			uint32_t r = groupBase;
			uint32_t need = 0;
			#pragma unroll 1
			for (uint32_t k = 0; k < gcount; ++k)
			{
				const uint32_t cnt = sm->candNew[k];
				if ((big >> k) & 1u)
				{
					uint32_t c0 = 0, c1 = 0, c2 = 0, c3 = 0;
					#pragma unroll 1
					for (uint32_t e = 0; e < cnt; e += 32)
					{
						uint32_t b = 0xFF;
						if (e + lane < cnt)
						{
							const PathT* p = pool + r + e + lane;
#if KB_CONG
							b = (p->sp_state ^ ((0u - (uint32_t)p->lm_state) >> 5)) & 3;
#else
							b = (p->sp_state ^ ((uint32_t)p->lm_state >> 5)) & 3;
#endif
						}
						c0 += __popc(__ballot_sync(FULL, b == 0)); c1 += __popc(__ballot_sync(FULL, b == 1));
						c2 += __popc(__ballot_sync(FULL, b == 2)); c3 += __popc(__ballot_sync(FULL, b == 3));
					}
					if (max(max(c0, c1), max(c2, c3)) >= KB_EXACT_FROM) need |= 1u << k;
				}
				r += cnt;
			}
			return need;
		}

		// capacity + write-out order per candidate segment (see the comment above stagePaths)
		__device__ KB_INL1 void fixupGroup(uint32_t groupBase, uint32_t gcount, uint32_t mode, bool deferTop1)
		{
			if (mode == 2)
			{
				// `top1` container: no buckets, no capacity, but the write-out order of an unordered_set - per candidate segment, in candidate
				// order (the set's bucket count carries over from one candidate to the next).  Team mode defers this until every warp's
				// entry counts are known (evaluate).
				if (deferTop1) return;
				uint32_t r = groupBase;
				#pragma unroll 1
				for (uint32_t k = 0; k < gcount; ++k)
				{
					const uint32_t cnt = sm->candNew[k];
					if (!cnt) continue;
					if (sm->cdyn[k].cls != CLS_SHORTCUT) { top1Buckets = reorderTop1(r, cnt, top1Buckets, top); if (err) return; }
					r += cnt;
				}
				return;
			}
			// is any fix-up needed at all?
			bool need = false;
			{
				const uint32_t cnt = lane < gcount ? sm->candNew[lane] : 0;
				const uint8_t cls = lane < gcount ? sm->cdyn[lane].cls : CLS_SKIP;
				need = mode != 2 && cls == CLS_ITEM && ((mode == 1 && cnt > 1) || cnt > 128);     // the top1 container has neither buckets nor a capacity
			}
			if (!__any_sync(FULL, need)) return;
			uint32_t w = groupBase, r = groupBase;
			const uint32_t tmp = top;
			#pragma unroll 1
			for (uint32_t k = 0; k < gcount; ++k)
			{
				const uint32_t cnt = sm->candNew[k];
				if (!cnt) continue;
				const bool fix = mode != 2 && sm->cdyn[k].cls == CLS_ITEM && ((mode == 1 && cnt > 1) || cnt > 128);
				if (!fix)
				{
					if (w != r)
					{
						#pragma unroll 1
						for (uint32_t e = 0; e < cnt; e += 32)
						{
							PathT p; const bool ok = e + lane < cnt;
							if (ok) p = pool[r + e + lane];
							__syncwarp();
							if (ok) pool[w + e + lane] = p;
							__syncwarp();
						}
					}
					w += cnt; r += cnt;
					continue;
				}
				if (tmp + cnt > poolCap) { err = ST_PATH_OVERFLOW; return; }
				#pragma unroll 1
				for (uint32_t e = lane; e < cnt; e += 32) pool[tmp + e] = pool[r + e];
				__syncwarp();
				const uint32_t nb = mode == 1 ? 4 : 1;
				uint32_t kept = 0;
				#pragma unroll 1
				for (uint32_t b = 0; b < nb; ++b)
				{
					uint32_t inBucket = 0;
					#pragma unroll 1
					for (uint32_t e = 0; e < cnt; e += 32)
					{
						PathT p; bool ok = e + lane < cnt;
#if KB_CONG
						if (ok) { p = pool[tmp + e + lane]; if (mode == 1) ok = ((p.sp_state ^ ((0u - (uint32_t)p.lm_state) >> 5)) & 3) == b; }
#else
						if (ok) { p = pool[tmp + e + lane]; if (mode == 1) ok = ((p.sp_state ^ ((uint32_t)p.lm_state >> 5)) & 3) == b; }
#endif
						const unsigned bm = __ballot_sync(FULL, ok);
						const uint32_t pos = inBucket + __popc(bm & ((1u << lane) - 1));
						if (ok && pos < 128) pool[w + kept + pos] = p;
						inBucket += __popc(bm);
					}
					kept += min(inBucket, 128u);
				}
				__syncwarp();
				if (lane == 0) sm->candNew[k] = kept;      // (team mode publishes the final per-candidate counts)
				w += kept; r += cnt;
			}
			// every lane has read sm->cdyn / sm->candNew of this group: the caller overwrites them for the next group
			// (found by the 32-lane host simulation, tests/hostsim: a lane that leaves this loop early must not race ahead)
			__syncwarp();
			top = w;
		}


#if KB_CONG
		// ---- transposed evaluator, node-level preparation ------------------------------------------------------
		struct CongNode { uint32_t nOrdered, epFirst, nU; };

		// (a) the node's unique context ids among the regular (non-socket) incoming paths -> sm->uctx / sm->pslot, and
		//     (b) the candidates in evaluation order -> sm->candOrder (indices into the node's candidate block): z_coda shortcut,
		//     z_siot shortcut, regular, left halves, right halves (PathEvaluator.hpp:883-963, CoNgramModel.cpp:76-121); dropped
		//     candidates are left out.
		//     The shape (unique contexts m, unique first wids n) of the node's gather GEMM selects the float epilogue.
		__device__ __noinline__ CongNode congPrepare(const DNode& node, bool spaceBefore, const DCand* candBase, uint32_t nCandsIn, uint32_t inBeg, uint32_t P)
		{
			CongNode cn; cn.nOrdered = 0; cn.epFirst = CG_E_SMALL; cn.nU = 0;
			// ---- (a)
			uint32_t nU = 0, nUtrue = 0, Preg = 0;
			#pragma unroll 1
			for (uint32_t qb = 0; qb < P; qb += 32)
			{
				const uint32_t q = qb + lane;
				bool reg = false; uint32_t ctx = 0;
				if (q < P) { const PathT* pth = pool + inBeg + q; reg = (pth->fw >> FW_SOCKET_SHIFT) == 0; ctx = P_CTX(*pth); }
				unsigned rem = __ballot_sync(FULL, reg);
				Preg += __popc(rem);
				uint32_t mySlot = 0xFFu;
				while (rem)
				{
					const int src = __ffs(rem) - 1;
					const uint32_t v = __shfl_sync(FULL, ctx, src);
					uint32_t slot = 0xFFu;
					for (uint32_t base = 0; base < nU; base += 32)
					{
						const unsigned hit = __ballot_sync(FULL, base + lane < nU && sm->uctx[base + lane] == v);
						if (hit) { slot = base + __ffs(hit) - 1; break; }
					}
					if (slot == 0xFFu)
					{
						// not in the tile list: either new, or (list full) an overflow context that is scored per pair
						if (nU < CG_UCAP) { slot = nU; if (lane == 0) sm->uctx[nU] = v; ++nU; ++nUtrue; __syncwarp(); }
						else ++nUtrue;      // nUtrue only needs to be exact up to 4
					}
					const unsigned same = __ballot_sync(FULL, reg && ctx == v);
					if (reg && ctx == v) mySlot = slot;
					rem &= ~same;
				}
				if (q < P && q < STAGE_CAP) sm->pslot[q] = (uint8_t)mySlot;
			}
			cn.nU = nU;
			// ---- (b)
			if (nCandsIn > CG_CANDS) { err = ST_INTERNAL; return cn; }
			uint32_t W = 0, nDistinct = 0, known[4] = { 0, 0, 0, 0 };
			int32_t lastCoda = -1, lastSiot = -1;
			#pragma unroll 1
			for (uint32_t cb = 0; cb < nCandsIn; cb += 32)
			{
				const uint32_t ci = cb + lane;
				uint32_t key = 7, fw = 0;
				if (ci < nCandsIn)
				{
					const DCand* dc = candBase + ci;
					const uint32_t kind = dc->kind;
					bool drop = (kind & DK_DIALECT) || (splitComplex && (kind & DK_COMPLEX));
					if (drop) key = 7;
					else if (kind & DK_SHORTCUT_CODA) key = 0;
					else if (kind & DK_SHORTCUT_SIOT) key = 1;
					else
					{
						if ((kind & DK_HA) && node.prev && spaceBefore) drop = true;
						if (drop) key = 7;
						else if (dc->cur_socket) key = (dc->flags & CS_SINGLE) ? 3 : 4;
						else if (kind & DK_FIRST_IS_P) key = 7;
						else { key = 2; fw = dc->first_wid; }
					}
				}
				sm->item[ci < ITEM_CAP ? ci : 0] = ci < nCandsIn ? key : 7u;      // nCandsIn <= CG_CANDS <= ITEM_CAP
				const unsigned codaM = __ballot_sync(FULL, key == 0), siotM = __ballot_sync(FULL, key == 1);
				if (codaM) lastCoda = (int32_t)(cb + 31 - __clz(codaM));
				if (siotM) lastSiot = (int32_t)(cb + 31 - __clz(siotM));
				unsigned rem = __ballot_sync(FULL, key == 2);
				W += __popc(rem);
				while (rem && nDistinct < 4)
				{
					const int src = __ffs(rem) - 1;
					const uint32_t v = __shfl_sync(FULL, fw, src);
					bool seen = false;
					for (uint32_t z = 0; z < nDistinct; ++z) if (known[z] == v) seen = true;
					if (!seen) known[nDistinct++] = v;
					rem &= ~__ballot_sync(FULL, key == 2 && fw == v);
				}
			}
			__syncwarp();
			uint32_t nOut = 0;
			#pragma unroll 1
			for (uint32_t k = 0; k <= 4; ++k)
			{
				#pragma unroll 1
				for (uint32_t cb = 0; cb < nCandsIn; cb += 32)
				{
					const uint32_t ci = cb + lane;
					bool take = ci < nCandsIn && sm->item[ci] == k;
					if (k == 0 && take && (int32_t)ci != lastCoda) take = false;       // `zCodaMorph = curMorph`: the last one wins
					if (k == 1 && take && (int32_t)ci != lastSiot) take = false;
					const unsigned tm = __ballot_sync(FULL, take);
					if (take) sm->candOrder[nOut + __popc(tm & ((1u << lane) - 1))] = ci;
					nOut += __popc(tm);
				}
			}
			__syncwarp();
			cn.nOrdered = nOut;
			const uint32_t m4 = min(nUtrue, 4u), n4 = min(nDistinct, 4u);
			cn.epFirst = (Preg == 1 && W == 1) ? (uint32_t)CG_E_SCALAR : cgEpilogueOf(m4, n4);
			return cn;
		}

		__device__ __forceinline__ void congGroupDots(uint32_t nU, uint32_t colMask) { cgTileDots(sm->uctx, sm->colWid, sm->dots, nU, colMask, lane); }
#endif

		// ---- candidates that do not go through the item pipeline: the z_coda / z_siot shortcuts (PathEvaluator.hpp:389-432) and
		// the per-candidate path evalCand (> 512 incoming paths, medium-mode forks, class-table overflow).  Cold: kept out of line.
		struct GenCtx
		{
			uint32_t nodeIdx, inBeg, inEnd, mode, ownOff, ownLen, ownFw; float ignoreCondScore; bool spaceBefore;
#if KB_CONG
			uint32_t epFirst; int32_t dotCol;
#endif
		};
		__device__ __noinline__ void evalGeneralCand(uint32_t k, const DNode& node, const GenCtx& g)
		{
			const uint32_t P = g.inEnd - g.inBeg, inBeg = g.inBeg;
			const DCand dk = dcur[k];
			const CandDyn cd = sm->cdyn[k];
			const int32_t curId = dk.cur_id;
			const DMorph cur = c_m.morphs[curId];
			const uint32_t tag = cur.feat & MF_TAG_MASK;
			if (cd.cls == CLS_SHORTCUT)
			{
				// shortcut (PathEvaluator.hpp:389-432): copy qualifying incoming paths, no LM step
				const float add = cur.user_score * c_m.cfg.typo_cost_weight;
				const DMorph lmM = c_m.morphs[cur.lm_id];
				#pragma unroll 1
				for (uint32_t qb = 0; qb < P; qb += 32)
				{
					const uint32_t q = qb + lane;
					PathT p; bool ok = false;
					if (q < P)
					{
						p = pool[inBeg + q];
						const uint32_t lastTag = P_WID_FEAT(p) & MF_TAG_MASK;
						ok = tag == T_z_coda ? (isJClass((uint8_t)lastTag) || isEClass((uint8_t)lastTag)) : isNNClass((uint8_t)lastTag);
					}
					const unsigned om = __ballot_sync(FULL, ok);
					if (top + __popc(om) > poolCap) { err = ST_PATH_OVERFLOW; return; }
					if (ok)
					{
						PathT np = p;
						np.acc_score += add;
						np.acc_typo_cost -= cur.user_score;
						np.parent = inBeg + q;
						np.morpheme = (int32_t)cur.lm_id;
						np.wid = cur.lm_id;
						np.node = (uint16_t)g.nodeIdx;
						np.morph_tag = (uint8_t)(lmM.feat & MF_TAG_MASK);
#if !KB_CONG
						np.wid_feat = lmM.feat;
#endif
						uint16_t ll; uint8_t lp;
						leftFeat(np.own_len ? np.own_off : 0, np.own_len, np.wid, np.morpheme, ll, lp);
						if (lmM.combine_socket) lp |= LP_MORPH_SOCKET;
						np.fw = fwOfLeft(ll, lp) | fwOfTag(np.morph_tag, (uint8_t)(p.fw >> FW_SOCKET_SHIFT)) | (p.fw & FW_COMMON_ROOT);
						pool[top + __popc(om & ((1u << lane) - 1))] = np;
					}
					top += __popc(om);
				}
				__syncwarp();
				return;
			}
			const bool single = (cur.feat & MF_SINGLE) != 0;
			CandCtx cc;
			cc.curId = curId; cc.cur = cur; cc.single = single;
			cc.firstWid0 = dk.first_wid; cc.lastSeqId = dk.last_seq_id;
			cc.additionalScore = cd.additionalScore;
			cc.ignoreCondScore = g.ignoreCondScore;
			cc.specialType = (cur.feat >> MF_SPECIAL_SHIFT) & 7;
			cc.sbType = (cur.feat >> MF_SBTYPE_SHIFT) & 31;
			cc.sbOrder = cc.sbType ? cur.sense_id : 0;
			cc.positiveE = (cd.flags & CS_POSITIVE_E) != 0;
			cc.snEndswithPoint = (cd.flags & CS_SN_POINT) != 0;
			cc.fork = (cd.flags & CS_FORK) != 0;
			cc.ownOff = g.ownOff; cc.ownLen = g.ownLen;
			cc.spaceBefore = g.spaceBefore;
			cc.morphTag = (uint8_t)tag;
			cc.widFeat = dk.last_seq_feat;
			const bool own = single && g.ownLen;
			cc.fwNew = own ? (g.ownFw | (dk.fw_new & FW_MORPH_SOCKET) | fwOfTag((uint8_t)tag, dk.path_socket)) : dk.fw_new;
#if KB_CONG
			cc.epFirst = g.epFirst; cc.dotCol = g.dotCol;
#endif
			evalCand(g.nodeIdx, node, cc, g.inBeg, g.inEnd, g.mode);
		}

#if !KB_SBG
		// (cold) the group's candidates once more, one after the other, with the item-by-item container (see evaluate)
		__device__ __noinline__ void redoGroupExact(const DNode& node, const FlushCtx& fc, uint32_t groupBase, uint32_t gcount)
		{
			const uint32_t inEnd = fc.inEnd, mode = fc.mode; const bool spaceBefore = fc.spaceBefore != 0;
#ifdef KB_HOSTSIM
			if (lane == 0 && std::getenv("HS32_TRACE_REDO")) std::fprintf(stderr, "[redo] node %u mode %u group of %u\n", fc.nodeIdx, mode, gcount);
#endif
			top = groupBase;
			resetIndex();
			if (lane == 0) sm->exactInsert = 1;
			__syncwarp();
			#pragma unroll 1
			for (uint32_t k = 0; k < gcount; ++k)
			{
				const uint8_t cls = sm->cdyn[k].cls;
				const uint32_t before = top;
				if (cls != CLS_SKIP)
				{
					GenCtx g;
					g.nodeIdx = fc.nodeIdx; g.inBeg = fc.inBeg; g.inEnd = inEnd; g.mode = mode; g.ownOff = fc.ownOff; g.ownLen = fc.ownLen; g.ownFw = fc.ownFw;
					g.ignoreCondScore = fc.ignoreCondScore; g.spaceBefore = spaceBefore;
#if KB_CONG
					g.epFirst = fc.epFirst; g.dotCol = ((fc.dotMask >> k) & 1u) ? (int32_t)k : -1;
#endif
					evalGeneralCand(k, node, g);
					if (err) { __syncwarp(); if (lane == 0) sm->exactInsert = 0; __syncwarp(); return; }
				}
				__syncwarp();
				if (lane == 0) { sm->candNew[k] = top - before; if (cls == CLS_ITEM) sm->cdyn[k].cls = CLS_GENERAL; }      // capacity and order are final
				__syncwarp();
				resetIndex();
			}
			if (lane == 0) sm->exactInsert = 0;
			__syncwarp();
		}

		// (cold) only the candidates in `need` once more, item by item; the other candidates' containers never reached 64 states in a bucket,
		// where the parallel insert is the reference's container, and keep their entries.  The re-runs append behind the group, then every
		// segment is gathered in candidate order behind them and moved back to groupBase.  Returns false when that scratch does not fit the
		// pool (err is clear then, nothing of the group has moved: the caller re-runs the whole group in place)
		__device__ __noinline__ bool redoCandsExact(const DNode& node, const FlushCtx& fc, uint32_t groupBase, uint32_t gcount, uint32_t need)
		{
			const uint32_t cn = lane < gcount ? sm->candNew[lane] : 0;
			uint32_t incl = cn;
			for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(FULL, incl, d); if (lane >= (uint32_t)d) incl += t; }
			uint32_t mySrc = groupBase + incl - cn, myCnt = cn;      // lane k: where candidate k's final entries are
			const uint32_t groupEnd = groupBase + __shfl_sync(FULL, incl, 31);
			top = groupEnd;
			if (lane == 0) sm->exactInsert = 1;
			__syncwarp();
			#pragma unroll 1
			for (uint32_t rem = need; rem; rem &= rem - 1)
			{
				const uint32_t k = __ffs(rem) - 1;
				resetIndex();
				const uint32_t before = top;
				GenCtx g;
				g.nodeIdx = fc.nodeIdx; g.inBeg = fc.inBeg; g.inEnd = fc.inEnd; g.mode = fc.mode; g.ownOff = fc.ownOff; g.ownLen = fc.ownLen; g.ownFw = fc.ownFw;
				g.ignoreCondScore = fc.ignoreCondScore; g.spaceBefore = fc.spaceBefore != 0;
#if KB_CONG
				g.epFirst = fc.epFirst; g.dotCol = ((fc.dotMask >> k) & 1u) ? (int32_t)k : -1;
#endif
				evalGeneralCand(k, node, g);
				if (err) break;
				if (lane == k) { mySrc = before; myCnt = top - before; }
			}
			__syncwarp();
			if (lane == 0) sm->exactInsert = 0;
			__syncwarp();
			uint32_t total = myCnt;
			for (int d = 16; d > 0; d >>= 1) total += __shfl_xor_sync(FULL, total, d);
			const uint32_t gather = top;
			if (err == ST_PATH_OVERFLOW || gather + total > poolCap) { err = 0; top = groupEnd; resetIndex(); return false; }
			if (err) return true;
			// gather in candidate order, then back to groupBase (48-byte records as 3 x 16 bytes)
			uint32_t dst = gather;
			#pragma unroll 1
			for (uint32_t k = 0; k < gcount; ++k)
			{
				const uint32_t src = __shfl_sync(FULL, mySrc, k), c = __shfl_sync(FULL, myCnt, k);
				#pragma unroll 1
				for (uint32_t e = lane; e < c; e += 32) pool[dst + e] = pool[src + e];
				dst += c;
			}
			__syncwarp();
			#pragma unroll 1
			for (uint32_t e = lane; e < total; e += 32) pool[groupBase + e] = pool[gather + e];
			__syncwarp();
			if (lane < gcount)
			{
				sm->candNew[lane] = myCnt;
				if (((need >> lane) & 1u) && sm->cdyn[lane].cls == CLS_ITEM) sm->cdyn[lane].cls = CLS_GENERAL;      // capacity and order are final
			}
			top = groupBase + total;
			__syncwarp();
			resetIndex();
			return true;
		}
#endif

		// ---- PathEvaluator::operator(), PathEvaluator.hpp:347-512 ------------------------------------
		// candBase: the node's static candidate rows (a form's block of c_m.cands, or the unknown NNG / NNP rows)
		__device__ KB_INL_EVAL void evaluate(uint32_t nodeIdx, uint32_t nodeBeg, const DCand* candBase, uint32_t nCandsIn,
			float unkFormDiscount, uint32_t ownOff, uint32_t ownLen, uint32_t inBeg, uint32_t inEnd, bool first)
		{
			// register copies (see Vit)
			WarpSmem* const sm = this->sm; PathT* const pool = this->pool; const uint32_t lane = this->lane, nUniq = this->nUniq;
			// `first`: the node's first evaluation - its candidate block may be waiting in the other staging buffer
			bool rowsStaged = false;
#if KB_TMA_ROWS
			if (first)
			{
				curBuf ^= 1u;
				if (pfBase[curBuf] != nullptr) { const bool hit = pfBase[curBuf] == candBase; pfWait(curBuf); rowsStaged = hit; }
			}
#else
			(void)first;
#endif
			const DNode node = nodes[nodeIdx];
			float whitespaceDiscount = 0;
			if (node.uform_len == 0 && node.form >= 0 && c_m.forms[node.form].str_len && node.space_errors)
				whitespaceDiscount = -c_m.cfg.space_penalty * (float)node.space_errors;
			const float typoDiscount = -node.typo_cost * c_m.cfg.typo_cost_weight;
			const float nodeLevelDiscount = whitespaceDiscount + typoDiscount + unkFormDiscount;
			const uint32_t P = inEnd - inBeg;
			const uint32_t mode = P <= 128 ? 0 : (P <= 512 ? 1 : 2);
			const bool spaceBefore = nodes[nodeIdx - node.prev].end_pos < node.start_pos;
			const bool hasLB = hasLeftBoundary(nodeIdx);
#if KB_CONG
#ifndef KB_CONG_PIPELINE
#define KB_CONG_PIPELINE 1
#endif
			const bool itemOK = KB_CONG_PIPELINE && P <= STAGE_CAP;      // else every candidate goes through evalCand; always in the transposed evaluator's order
			const CongNode cgn = congPrepare(node, spaceBefore, candBase, nCandsIn, inBeg, P);
			if (err) return;
			const uint32_t nCands = cgn.nOrdered;
#else
			const bool itemOK = !KB_SBG && P <= STAGE_CAP;          // modes 0 / 1 always; mode 2 (`top1`, an unordered_set in the reference) up to the staging capacity
			const uint32_t nCands = nCandsIn;
#endif
			FlushCtx fc;
			fc.nodeIdx = nodeIdx; fc.inBeg = inBeg; fc.nodeTypoCost = node.typo_cost; fc.ownOff = ownOff; fc.ownLen = ownLen; fc.ownFw = 0;
			fc.inEnd = inEnd; fc.mode = mode; fc.spaceBefore = spaceBefore ? 1u : 0u;
			if (mode == 2 && P > HT_MAX_ENTRIES) { KB_PH_COUNT(PH_N_BIG_NODES, 1, phSent); KB_PH_COUNT(PH_N_BIG_CANDS, nCands, phSent); }
			KB_PH_START(tStage);
			if (itemOK) stagePaths(nodeIdx, inBeg, P);
			KB_PH_ADD(PH_STAGE, tStage, phSent);
			const bool itemOK2 = itemOK && !classOverflow;
			const uint32_t nClasses = this->nClasses, classCommon = this->classCommon;
			if (ownLen) { uint16_t ol; uint8_t op; leftFeat(ownOff, ownLen, 0, 0, ol, op); fc.ownFw = fwOfLeft(ol, op); }
			uint32_t nItems = 0;      // items waiting in sm->item
			uint32_t nFw = 1;         // entries of sm->fwTab (index 0 unused)
			auto flush = [&]() { KB_PH_START(tFlush); const bool ok = flushItems(fc, nItems); KB_PH_ADD(PH_FLUSH, tFlush, phSent); nItems = 0; return ok; };
			const bool snPoint = node.uform_len && norm[node.uform_off + node.uform_len - 1] == '.';
			const uint32_t nWords = (P + 31) >> 5;
			// class of lane's path in each of the first 6 words of 32 incoming paths, 5 bits each (+ which words have a path for this lane): the
			// enumeration below tests (candidate's valid-class mask >> class) per word without touching shared memory
			uint32_t clsPack = 0, clsHave = 0;
			if (itemOK)
			{
				#pragma unroll
				for (uint32_t w = 0; w < 6; ++w)
				{
					const uint32_t q = (w << 5) | lane;
					if (q < P) { clsPack |= (uint32_t)sm->pcls[q] << (5 * w); clsHave |= 1u << w; }
				}
			}

			#pragma unroll 1
			for (int ignoreCond = 0; ignoreCond < 2; ++ignoreCond)
			{
				fc.ignoreCondScore = ignoreCond ? -10.f : 0.f;
				#pragma unroll 1
				for (uint32_t gb = 0; gb < nCands; gb += GROUP)
				{
					const uint32_t gcount = min(GROUP, nCands - gb);
#if KB_TMA_ROWS
					dcur = (rowsStaged && gb == 0) ? sm->dcandBuf[curBuf] : sm->dcandGen;
#endif
					// ---- classification, one lane per candidate (PathEvaluator.hpp:382-448 + evalSingleMorpheme head 531-560), from the static rows
					KB_PH_START(tClassify);
					uint32_t myPack = CLS_SKIP, myValid = 0, myCondFail = 0, mySets = 0;
					{
						uint8_t cls = CLS_SKIP, flags = 0;
						float additionalScore = 0;
						uint32_t feat = 0, kind = 0, curSocket = 0;
						if (lane < gcount)
						{
#if KB_CONG
							const DCand* src = candBase + sm->candOrder[gb + lane];
#else
							const DCand* src = candBase + gb + lane;
#endif
							uint4 r0, r1, r2;
							uint4* dst = reinterpret_cast<uint4*>(&dcur[lane]);
							if (rowsStaged && gb == 0) { r1 = dst[1]; r2 = dst[2]; }      // the block is already in shared memory (bulk copy)
							else
							{
								r0 = reinterpret_cast<const uint4*>(src)[0]; r1 = reinterpret_cast<const uint4*>(src)[1]; r2 = reinterpret_cast<const uint4*>(src)[2];
								dst[0] = r0; dst[1] = r1; dst[2] = r2;
							}
							feat = r1.x;
							flags = (uint8_t)(r2.x >> 8); curSocket = r2.y & 0xFF; kind = (r2.y >> 8) & 0xFF;
							const uint32_t tagClean = (r2.y >> 16) & 0xFF;
							bool skip = (kind & DK_DIALECT) || (splitComplex && (kind & DK_COMPLEX));
							if (!skip && (kind & (DK_SHORTCUT_CODA | DK_SHORTCUT_SIOT)))
							{
								if ((kind & DK_SHORTCUT_SIOT) && !(splitSaisiot || mergeSaisiot)) skip = true;
								else cls = CLS_SHORTCUT;
							}
							else if (!skip)
							{
								// contracted '하다/하게/하지' after a space is not a candidate (PathEvaluator.hpp:435-448)
								if ((kind & DK_HA) && node.prev && spaceBefore) skip = true;
								if (!skip)
								{
									const bool fork = (flags & CS_FORK) != 0, socketChunk = (flags & CS_SOCKET_CHUNK) != 0, noLm = (flags & CS_NO_LM) != 0;
									// a forking candidate creates up to 2 entries per path; medium-mode forks keep the bucket-aware general path
									if (!itemOK2 || (mode == 1 && fork) || (mode == 2 && (fork ? 2 * P : P) > HT_MAX_ENTRIES)) cls = CLS_GENERAL;
									else if (!noLm && !socketChunk && (kind & (DK_FIRST_IS_P | DK_CHUNK_HAS_P))) cls = CLS_SKIP;     // every pair hits `goto continueFor`
									else if (socketChunk && (kind & DK_CHUNK_HAS_P)) cls = CLS_SKIP;
									else cls = CLS_ITEM;
									if ((kind & DK_IS_SN) && snPoint) flags |= CS_SN_POINT;
								}
							}
							additionalScore = __uint_as_float(r1.y) + nodeLevelDiscount + c_m.tag_left_boundary[hasLB ? 1 : 0][tagClean];
						}
						CandDyn cd; cd.additionalScore = additionalScore; cd.flags = flags; cd.cls = cls; cd.pad0 = 0; cd.pad1 = 0;
						sm->cdyn[lane] = cd;
						sm->candNew[lane] = 0;
						// which path classes pass this candidate's filter (PathEvaluator.hpp:566-594), decided once per class
						CandMask cm; cm.valid = 0; cm.condFail = 0; cm.sets = 0;
						if (cls == CLS_ITEM)
						{
							const uint32_t curTag = feat & MF_TAG_MASK;
							const uint32_t cv = (feat >> MF_VOWEL_SHIFT) & 15, cp = (feat >> MF_POLAR_SHIFT) & 3;
							const bool curNN = isNNClass((uint8_t)curTag);
							const bool socketChunk = (flags & CS_SOCKET_CHUNK) != 0;
							for (uint32_t c = 0; c < nClasses; ++c)
							{
								const uint32_t f = sm->fclass[c];
								const uint32_t socket = f >> FW_SOCKET_SHIFT;
								bool valid = true;
#if KB_CONG
								// the z_siot test exists only in the regular-candidate loop, and right halves only see combining paths
								// (CoNgramModel.cpp:184-189, 208-246, 248-286)
								if ((f & FW_ZSIOT) && curSocket == 0 && (!curNN || spaceBefore)) valid = false;
								else if (socketChunk && !socket) valid = false;
#else
								if ((f & FW_ZSIOT) && (!curNN || spaceBefore)) valid = false;
#endif
								else if (socket)
								{
									// merge <v> <chunk> with only the same socket (PathEvaluator.hpp:578-591)
									if (!socketChunk || socket != curSocket) valid = false;
									else if (spaceBefore && !(c_m.cfg.space_tolerance > 0)) valid = false;
									if (valid) cm.sets |= 1u << c;
								}
								if (valid && !(f & FW_NOCOND))
								{
									const bool empty = (f & FW_EMPTY) != 0;
									bool ok = ftVowelCls(empty, f & FW_CLS_MASK, cv);
									if (ok && (cp == CP_positive || cp == CP_negative)) ok = empty ? true : ((f & (cp == CP_positive ? FW_POLAR_POS : FW_POLAR_NEG)) != 0);
									if (ignoreCond) { if (!ok) cm.condFail |= 1u << c; }
									else if (!ok) valid = false;
								}
								if (valid) cm.valid |= 1u << c;
							}
							// prohibit <v> without <chunk> (PathEvaluator.hpp:603-607): a socket chunk whose first wid is the tag-P
							// placeholder only survives behind a path that overrides firstWid; without such a path nothing survives
							if (socketChunk && !cm.sets && (kind & DK_FIRST_IS_P)) cm.valid = 0;
						}
						sm->cmask[lane] = cm;
						myPack = cls | ((uint32_t)flags << 8); myValid = cm.valid; myCondFail = cm.condFail; mySets = cm.sets;
					}
					__syncwarp();
					KB_PH_ADD(PH_CLASSIFY, tClassify, phSent);
#if KB_CONG
					// tensor-core tile for the regular candidates of this group
					uint32_t dotMask = 0;
					{
						const CandDyn cdl = sm->cdyn[lane];
						const bool regular = lane < gcount && (cdl.cls == CLS_GENERAL || cdl.cls == CLS_ITEM) && dcur[lane].cur_socket == 0 && !(dcur[lane].kind & DK_FIRST_IS_P);
						sm->colWid[lane] = lane < gcount ? dcur[lane].first_wid : 0u;
						dotMask = __ballot_sync(FULL, regular);
						__syncwarp();
						if (dotMask && cgn.nU && cgn.epFirst != CG_E_SCALAR) congGroupDots(cgn.nU, dotMask);
						else dotMask = 0;
						fc.epFirst = cgn.epFirst; fc.dotMask = dotMask;
					}
#endif
					// team mode: a group whose candidates all take the item pipeline is dealt to the warps of the team (candidate k -> warp k mod
					// team size), every warp writing into its own staging region of the pool; any other group is the first warp's alone
					const bool teamGroup = teamSize > 1 && !__any_sync(FULL, (myPack & 0xFF) >= CLS_GENERAL);
					const uint32_t groupBase = top, poolCap0 = poolCap;
					uint32_t half = 0, myBase = top;
					if (teamGroup)
					{
						half = (poolCap0 - top) / 2;
						const uint32_t regionSize = half / teamSize;
						myBase = top + half + teamRank * regionSize;
						poolCap = myBase + regionSize; top = myBase;
					}
					auto walk = [&]()
					{
					resetIndex();
					nFw = 1;

					// ---- ordered walk over the candidates of the group
					#pragma unroll 1
					for (uint32_t k = 0; k < gcount; ++k)
					{
						const uint32_t packK = __shfl_sync(FULL, myPack, k);
						const uint32_t cls = packK & 0xFF, kfl = packK >> 8;
						if (cls == CLS_SKIP) continue;
						if (teamGroup && (k % teamSize) != teamRank) continue;
						if (cls == CLS_ITEM)
						{
							const uint32_t vmK = __shfl_sync(FULL, myValid, k), setsK = __shfl_sync(FULL, mySets, k);
							if (!(vmK | setsK)) continue;
							const uint32_t cfK = __shfl_sync(FULL, myCondFail, k);
							// the entry index is shared by consecutive candidates while it is small; a top1-mode candidate (up to P entries) starts with an empty one
							if (mode == 2 ? (htCount | nItems) != 0 : htCount + nItems > 256) { if (!flush()) return; resetIndex(); }
							if (!(kfl & CS_FORK) && !setsK)
							{
								// common case: the survivors of every 32 incoming paths are compacted by one ballot, in path order
								#pragma unroll 1
								for (uint32_t w = 0; w < nWords; ++w)
								{
									const uint32_t q = (w << 5) | lane;
									uint32_t c; bool on;
									if (w < 6) { c = (clsPack >> (5 * w)) & 31u; on = ((clsHave >> w) & (vmK >> c) & 1u) != 0; }
									else { c = q < P ? sm->pcls[q] : 31u; on = q < P && ((vmK >> c) & 1u); }
									const unsigned m = __ballot_sync(FULL, on);
									if (!m) continue;
									const uint32_t cnt = __popc(m);
									if (nItems + cnt > ITEM_CAP) { if (!flush()) return; }
									if (on) sm->item[nItems + __popc(m & ((1u << lane) - 1))] = (k << 27) | (q << 3) | ((cfK >> c) & 1u);
									nItems += cnt;
								}
								continue;
							}
							// filter pass (PathEvaluator.hpp:566-594): lanes = (path, root) pairs in order; the per-pair work is a
							// table lookup because the decision only depends on (candidate, path class)
							const bool fork = (kfl & CS_FORK) != 0, socketChunk = (kfl & CS_SOCKET_CHUNK) != 0;
							const uint32_t rshift = (fork && nUniq == 2) ? 1 : 0;
							const uint32_t perRound = 32u >> rshift;
							const bool spacePen = socketChunk && spaceBefore;          // only socket matches survive `spaceBefore` (with tolerance) and they pay the penalty
							uint32_t fwCarry = 0;                     // index into fwTab of the inherited first-wid override, 0 = none
							const bool firstIsP = socketChunk && (dcur[k].kind & DK_FIRST_IS_P) != 0;
							#pragma unroll 1
							for (uint32_t qb = 0; qb < P; qb += perRound)
							{
								if (nItems + 32 > ITEM_CAP) { if (!flush()) return; }
								const uint32_t pr = lane >> rshift, rr = lane & ((1u << rshift) - 1);
								const uint32_t q = qb + pr;
								bool valid = false, condFail = false, setsFW = false, isSock = false;
								if (q < P)
								{
									const uint32_t c = sm->pcls[q];
									valid = (vmK >> c) & 1;
									condFail = (cfK >> c) & 1;
									setsFW = (setsK >> c) & 1;
									isSock = setsFW;
									if (rr != 0 && !((classCommon >> c) & 1)) valid = false;      // only common-root paths fork over the root states
								}
								uint32_t fwIdx = 0;
								if (setsK)
								{
									// the reference overwrites `firstWid` in place: every later pair inherits the latest override
									const unsigned smask = __ballot_sync(FULL, setsFW);
									uint32_t myIdx = 0;
									if (smask)
									{
										uint32_t fwVal = 0;
										if (setsFW) { const uint32_t pw = pool[inBeg + q].wid; fwVal = c_m.morphs[(int32_t)pw + c_m.morphs[pw].combined].lm_id; }
										unsigned rem = smask;
										while (rem)
										{
											const int src = __ffs(rem) - 1;
											const uint32_t v = __shfl_sync(FULL, fwVal, src);
											uint32_t idx = 0;
											for (uint32_t z = 1; z < nFw; ++z) if (sm->fwTab[z] == v) { idx = z; break; }
											if (!idx)
											{
												if (nFw >= FWTAB_CAP) { err = ST_INTERNAL; return; }
												idx = nFw++;
												if (lane == 0) sm->fwTab[idx] = v;
												__syncwarp();
											}
											if ((int)lane == src) myIdx = idx;
											rem &= rem - 1;
										}
									}
									const unsigned le = smask & (lane == 31 ? FULL : ((2u << lane) - 1));
									const int src = le ? 31 - __clz(le) : 0;
									const uint32_t got = __shfl_sync(FULL, myIdx, src);
									fwIdx = le ? got : fwCarry;
									if (smask) fwCarry = __shfl_sync(FULL, myIdx, 31 - __clz(smask));
								}
								// prohibit <v> without <chunk>: tag P first wid (PathEvaluator.hpp:603-607)
								if (valid && socketChunk && (fwIdx ? ((c_m.morphs[sm->fwTab[fwIdx]].feat & MF_TAG_MASK) == T_p) : firstIsP)) valid = false;
								const unsigned vm = __ballot_sync(FULL, valid);
								if (valid) sm->item[nItems + __popc(vm & ((1u << lane) - 1))] = (k << 27) | (fwIdx << 20) | (q << 3) | ((spacePen && isSock) ? 4u : 0u) | (rr << 1) | (condFail ? 1u : 0u);
								nItems += __popc(vm);
								__syncwarp();
							}
							continue;
						}
						// general path and shortcuts: drain the pipeline first so that entries stay candidate-major
						if (!flush()) return;
						const uint32_t before = top;
						GenCtx g;
						g.nodeIdx = nodeIdx; g.inBeg = inBeg; g.inEnd = inEnd; g.mode = mode; g.ownOff = ownOff; g.ownLen = ownLen; g.ownFw = fc.ownFw;
						g.ignoreCondScore = fc.ignoreCondScore; g.spaceBefore = spaceBefore;
#if KB_CONG
						g.epFirst = cgn.epFirst; g.dotCol = ((dotMask >> k) & 1u) ? (int32_t)k : -1;
#endif
						KB_PH_START(tGen);
						evalGeneralCand(k, node, g);
						if (mode == 2 && P > HT_MAX_ENTRIES) KB_PH_ADD(PH_GEN_BIG, tGen, phSent); else KB_PH_ADD(PH_GEN_SMALL, tGen, phSent);
						if (err) return;
						if (lane == 0) sm->candNew[k] = top - before;
						__syncwarp();
						resetIndex();
					}
					if (!flush()) return;
#if !KB_SBG && !defined(KB_NO_EXACT_REDO)
					// The parallel insert above is the reference's container as long as no bucket reaches 64 states (0.02 % of the containers
					// of the bench batches do).  Beyond that the reference's insertOptimized behaves differently (exactInsertRound): the
					// candidates whose container got there are evaluated again, one after the other, item by item.
					if (mode != 2 && teamSize == 1 && __any_sync(FULL, lane < gcount && sm->candNew[lane] >= KB_EXACT_FROM))
					{
						const uint32_t need = groupExactMask(myBase, gcount, mode);
						if (need)
						{
							KB_PH_START(tRedo);
							if (!redoCandsExact(node, fc, myBase, gcount, need)) redoGroupExact(node, fc, myBase, gcount);
							KB_PH_ADD(PH_REDO, tRedo, phSent);
							if (err) return;
						}
					}
#endif
					if (itemOK || mode == 2) { fixupGroup(myBase, gcount, mode, teamGroup); if (err) return; }
					};
					KB_PH_START(tWalk);
					if (teamSize == 1 || teamGroup || leader()) walk();      // (one call site: the walk is the bulk of this function's code)
					KB_PH_ADD(PH_WALK, tWalk, phSent);
					if (teamSize == 1) { if (err) return; }
					else if (teamGroup)
					{
						// publish the per-candidate entry counts of my candidates, then place every segment in candidate order
						if (lane < gcount && (lane % teamSize) == teamRank) tm->cnt[lane] = sm->candNew[lane];
						if (err && lane == 0) atomicMax(&tm->err, err);
						teamSync();
						err = tm->err;
						if (err) { poolCap = poolCap0; return; }
						const uint32_t cnt = lane < gcount ? tm->cnt[lane] : 0;
						if (mode == 2)
						{
							// write-out order of the `top1` container for my candidates: candidate k starts with the bucket count the set has after
							// the candidates before it (of any warp) - it only grows, so that is a function of their largest entry count
							uint32_t pmax = cnt;
							for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(FULL, pmax, d); if (lane >= (uint32_t)d) pmax = max(pmax, t); }
							const uint32_t before = __shfl_up_sync(FULL, pmax, 1);      // max entry count of the candidates before lane's
							uint32_t seg = myBase;
							#pragma unroll 1
							for (uint32_t k = teamRank; k < gcount; k += teamSize)
							{
								const uint32_t c = __shfl_sync(FULL, cnt, k), mb = k ? __shfl_sync(FULL, before, k) : 0u;
								if (c) { reorderTop1(seg, c, unorderedBucketsAfter(top1Buckets, mb), top); seg += c; }
							}
							top1Buckets = unorderedBucketsAfter(top1Buckets, __shfl_sync(FULL, pmax, 31));
							if (err && lane == 0) atomicMax(&tm->err, err);
							teamSync();
							err = tm->err;
							if (err) { poolCap = poolCap0; return; }
						}
						poolCap = poolCap0;
						uint32_t incl = cnt;
						for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(FULL, incl, d); if (lane >= (uint32_t)d) incl += t; }
						const uint32_t total = __shfl_sync(FULL, incl, 31), excl = incl - cnt;
						if (total > half) { err = ST_PATH_OVERFLOW; return; }
						uint32_t src = myBase;
						#pragma unroll 1
						for (uint32_t k = teamRank; k < gcount; k += teamSize)
						{
							const uint32_t c = __shfl_sync(FULL, cnt, k), dst = groupBase + __shfl_sync(FULL, excl, k);
							#pragma unroll 1
							for (uint32_t e = lane; e < c; e += 32)
							{
								const uint4* sp = reinterpret_cast<const uint4*>(pool + src + e); uint4* dp = reinterpret_cast<uint4*>(pool + dst + e);
								const uint4 a = sp[0], b = sp[1], cc = sp[2];
								dp[0] = a; dp[1] = b; dp[2] = cc;
								static_assert(!KB_SBG || TEAM == 1, "team mode moves 48-byte records");
							}
							src += c;
						}
						teamSync();
						top = groupBase + total;
					}
					else
					{
						uint32_t t = top; teamBroadcast(t); top = t;
						if (err) return;
					}
				}
				if (top > nodeBeg) break;
			}

			// prune (PathEvaluator.hpp:475-511): per root slot the best score of the paths whose morpheme has no combine socket;
			// scores are compared as order-preserving unsigned keys, the threshold test itself stays a float comparison
			KB_PH_START(tPrune);
			if (leader())
			{
			const uint32_t cntAll = top - nodeBeg;
			const uint32_t NEG_INF_ORD = 0x007FFFFFu;      // key of -inf
			uint32_t mxo0 = NEG_INF_ORD, mxo1 = NEG_INF_ORD, mxo2 = NEG_INF_ORD;
			#pragma unroll 1
			for (uint32_t eb = 0; eb < cntAll; eb += 32)
			{
				const uint32_t e = eb + lane;
				uint32_t o = 0, slot = 3;
				if (e < cntAll)
				{
					const PathT* p = pool + nodeBeg + e;
					const uint32_t meta = *reinterpret_cast<const uint32_t*>(&p->sp_state);
					const uint32_t root = (meta >> 8) & 0xFF;
					slot = root == COMMON_ROOT ? 0 : root + 1;
					o = NEG_INF_ORD;
					if (!(p->fw & FW_MORPH_SOCKET)) { const uint32_t u = __float_as_uint(p->acc_score); o = (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
				}
				mxo0 = max(mxo0, __reduce_max_sync(FULL, slot == 0 ? o : 0u));
				if (nUniq > 0) mxo1 = max(mxo1, __reduce_max_sync(FULL, slot == 1 ? o : 0u));
				if (nUniq > 1) mxo2 = max(mxo2, __reduce_max_sync(FULL, slot == 2 ? o : 0u));
			}
			const float mx0 = __uint_as_float((mxo0 & 0x80000000u) ? (mxo0 ^ 0x80000000u) : ~mxo0);
			const float mx1 = __uint_as_float((mxo1 & 0x80000000u) ? (mxo1 ^ 0x80000000u) : ~mxo1);
			const float mx2 = __uint_as_float((mxo2 & 0x80000000u) ? (mxo2 ^ 0x80000000u) : ~mxo2);
			uint32_t valid = 0;
			#pragma unroll 1
			for (uint32_t eb = 0; eb < cntAll; eb += 32)
			{
				const uint32_t e = eb + lane;
				bool keep = false;
				if (e < cntAll)
				{
					const PathT* p = pool + nodeBeg + e;
					const uint32_t root = p->root_id;
					const float mxs = root == COMMON_ROOT ? mx0 : (root == 0 ? mx1 : mx2);
					keep = !(p->acc_score + c_m.cfg.cut_off_threshold < mxs);
				}
				const unsigned km = __ballot_sync(FULL, keep);
				const uint32_t dst = valid + __popc(km & ((1u << lane) - 1));
				const uint32_t remE = cntAll - eb;
				if (valid != eb || km != (remE >= 32 ? FULL : ((1u << remE) - 1)))
				{
					// something was dropped at or before this round: move the survivors down (read all, then write)
					constexpr uint32_t SEGS = sizeof(PathT) / 16;      // 3 (DPath), 6 with the SkipBigram history
					uint4 seg[SEGS];
					if (keep) { const uint4* sp = reinterpret_cast<const uint4*>(pool + nodeBeg + e); for (uint32_t z = 0; z < SEGS; ++z) seg[z] = sp[z]; }
					__syncwarp();
					if (keep && dst != e) { uint4* dp = reinterpret_cast<uint4*>(pool + nodeBeg + dst); for (uint32_t z = 0; z < SEGS; ++z) dp[z] = seg[z]; }
					__syncwarp();
				}
				valid += __popc(km);
			}
			top = nodeBeg + valid;
			}
			KB_PH_ADD(PH_PRUNE, tPrune, phSent);
			if (teamSize > 1) { uint32_t t = top; teamBroadcast(t); top = t; }
		}

		// PathEvaluator.hpp:1159-1176; predecessors of a node are the contiguous group [k - prev, ...] linked by sibling == 1
		__device__ __noinline__ bool isDisconnected(uint32_t scanStart)
		{
			if (reach[scanStart - 1]) return false;
			__syncwarp();
			for (uint32_t k = scanStart; k < N; ++k)
			{
				const DNode nd = nodes[k];
				uint32_t r = 0;
				uint32_t q = k - nd.prev;
				if (nd.prev)
				{
					while (true)
					{
						if (reach[q]) { r = 1; break; }
						if (!nodes[q].sibling) break;
						q += nodes[q].sibling;
					}
				}
				if (lane == 0) reach[k] = (uint8_t)r;
				__syncwarp();
			}
			return reach[N - 1] == 0;
		}

		__device__ bool anyNonSocket(uint32_t beg, uint32_t end) const
		{
			bool any = false;
			for (uint32_t eb = beg; eb < end; eb += 32)
			{
				const uint32_t e = eb + lane;
				const bool ok = e < end && (pool[e].fw >> FW_SOCKET_SHIFT) == 0;
				if (__any_sync(FULL, ok)) { any = true; break; }
			}
			return any;
		}

		// incoming pool range of node i
		__device__ void incoming(uint32_t i, uint32_t& inBeg, uint32_t& inEnd) const
		{
			const DNode nd = nodes[i];
			uint32_t q = i - nd.prev;
			inBeg = npOff[q];
			while (nodes[q].sibling) q += nodes[q].sibling;
			inEnd = npOff[q] + npCnt[q];
		}

		// ---- one chunk: findBestPath, returns the selected results in res[] ----------------------------
		__device__ __noinline__ uint32_t findBestPath(const DChunk& ch, PathRes* res, bool openEnding)
		{
			const uint32_t chunkBase = top;
			stagedNode = NPOS;
			// BOS path (PathEvaluator.hpp:1224-1226)
			if (top + 1 > poolCap) { err = ST_PATH_OVERFLOW; return 0; }
			if (lane == 0 && leader())
			{
				PathT b;
#if KB_CONG
				b.lm_state = 0;            // CoNgramState(const ILangModel*): node 0, contextIdx 0 (CoNgramModel.hpp:479-485)
#else
				b.lm_state = c_m.kn_bos_node;
#if KB_SBG
				for (int i = 0; i < 8; ++i) b.hist[i] = 0;      // SbgState(const ILangModel*): empty ring (SkipBigramModel.hpp:144-154)
				b.hpos = 0; b.hpad = 0; b.hcode = 0;
#endif
#endif
				b.acc_score = 0; b.first_chunk_score = 0; b.wid = 0; b.morpheme = 0; b.parent = NPOS; b.own_off = 0; b.acc_typo_cost = 0;
				b.own_len = 0; b.node = 0; b.sp_state = 0; b.root_id = COMMON_ROOT; b.prev_root_id = 0;
				const DMorph m0 = c_m.morphs[0];
				b.morph_tag = (uint8_t)(m0.feat & MF_TAG_MASK);
#if KB_CONG
				P_CTX(b) = 0;
#else
				b.wid_feat = m0.feat;
#endif
				uint16_t ll; uint8_t lp;
				leftFeat(0, 0, 0, 0, ll, lp);
				b.fw = fwOfLeft(ll, lp) | fwOfTag(b.morph_tag, 0) | FW_COMMON_ROOT;
				pool[top] = b;
				npOff[0] = top; npCnt[0] = 1; reach[0] = 1;
			}
			if (leader()) for (uint32_t i = lane + 1; i < N; i += 32) reach[i] = 0;
			top += 1;
			__syncwarp();

			// per node: where its candidate rows are (a form's block of the static table, or the unknown NNG / NNP rows) - lane-parallel
			if (leader()) for (uint32_t j = 1 + lane; j + 1 < N; j += 32)
			{
				const int32_t fm = nodes[j].form;
				uint2 ci;
				if (fm >= 0) { const DForm f = c_m.forms[fm]; ci.x = f.cand_off; ci.y = (uint32_t)f.cand_cnt | ((uint32_t)f.flags << 16); }
				else { ci.x = c_m.cand_unk; ci.y = 2u; }
				nodeCand[j] = ci;
			}
			__syncwarp();
			teamSync();
#if KB_TMA_ROWS
			if (N > 2) { const uint2 c1 = nodeCand[1]; pfIssue(c_m.cands + c1.x, min(c1.y & 0xFFFFu, GROUP), curBuf ^ 1u); }
#endif

			KB_PH_START(tNodes);
			for (uint32_t i = 1; i + 1 < N; ++i)
			{
				const DNode node = nodes[i];
				const uint2 ci = nodeCand[i];
				uint32_t inBeg, inEnd;
				incoming(i, inBeg, inEnd);
				const uint32_t nodeBeg = top;
#if KB_TMA_ROWS
				// node i's rows sit in buffer curBuf ^ 1 (issued one node ago); node i + 1's go to curBuf, whose last reader was node i - 1
				if (i + 2 < N) { const uint2 cn = nodeCand[i + 1]; pfIssue(c_m.cands + cn.x, min(cn.y & 0xFFFFu, GROUP), curBuf); }
#endif
				// up to three evaluations of the node (PathEvaluator.hpp:1255-1306), ONE call site: (0) the form's candidates, or NNG + NNP for an
				// unknown span; (1) a form whose candidates are all partial: additionally as an unknown NNP; (2) a form node after which the
				// rest of the lattice is unreachable: the raw substring as unknown NNG + NNP
				const uint32_t fflags = ci.y >> 16;
				#pragma unroll 1
				for (uint32_t pass = 0; pass < 3; ++pass)
				{
					const DCand* cb; uint32_t cn, oo, ol; float disc;
					if (pass == 0)
					{
						if (node.form >= 0) { cb = c_m.cands + ci.x; cn = ci.y & 0xFFFFu; disc = 0.f; }
						else { cb = c_m.cands + c_m.cand_unk; cn = 2; disc = unkFormScore(norm + node.uform_off, node.uform_len); }
						oo = node.uform_off; ol = node.uform_len;
					}
					else if (pass == 1)
					{
						if (node.form < 0) break;
						if (!(node.typo_cost == 0.f && (fflags & FF_ALL_PARTIAL))) continue;
						const DForm f = c_m.forms[node.form];
						cb = c_m.cands + c_m.cand_unk + 1; cn = 1; disc = unkFormScore(c_m.form_chars + c_m.forms_raw[node.form].str_off, f.str_len);
						oo = ~(uint32_t)node.form; ol = f.str_len;
					}
					else
					{
						uint32_t dc = 0;
						if (leader())
						{
							const bool r = anyNonSocket(nodeBeg, top);
							if (lane == 0) reach[i] = r ? 1 : 0;
							__syncwarp();
							dc = isDisconnected(i + 1) ? 1u : 0u;
						}
						teamBroadcast(dc);
						if (err) return 0;
						if (!dc) break;
						ol = node.end_pos - node.start_pos; oo = node.start_pos;
						cb = c_m.cands + c_m.cand_unk; cn = 2; disc = unkFormScore(norm + node.start_pos, ol);
					}
					KB_PH_START(tEval);
					evaluate(i, nodeBeg, cb, cn, disc, oo, ol, inBeg, inEnd, pass == 0);
					KB_PH_ADD(PH_EVALUATE, tEval, phSent);
					if (err) return 0;
				}
				if (lane == 0 && leader()) { npOff[i] = nodeBeg; npCnt[i] = top - nodeBeg; }
				__syncwarp();
				teamSync();
			}
			KB_PH_ADD(PH_NODE_LOOP, tNodes, phSent);
			if (!leader()) return 0;      // the end node and the stitching are the first warp's; the others wait for its broadcast

			// ---- end node (PathEvaluator.hpp:1320-1357): candidates go to the pool tail as temporary records
			uint32_t inBeg, inEnd;
			incoming(N - 1, inBeg, inEnd);
			const uint32_t P = inEnd - inBeg;
			const uint32_t candBeg = top;
			uint32_t nCand = 0;
			const uint32_t perPath = nUniq;
			if (top + P * perPath > poolCap) { err = ST_PATH_OVERFLOW; return 0; }
			for (uint32_t qb = 0; qb < P; qb += 32)
			{
				const uint32_t q = qb + lane;
				PathT p; bool ok = false; float c = 0;
				if (q < P)
				{
					p = pool[inBeg + q];
					ok = (p.fw >> FW_SOCKET_SHIFT) == 0;
					if (ok)
					{
						const DMorph pm = c_m.morphs[p.morpheme];
						const bool single = (pm.feat & MF_SINGLE) != 0;
						if (!single && pm.chunk_cnt <= (pm.combine_socket ? 2u : 1u) && ((pm.feat >> MF_VOWEL_SHIFT) & 15) != CV_none) ok = false;
						if (p.morph_tag == T_z_siot) ok = false;
					}
					if (ok)
					{
						c = p.acc_score;
						if (!openEnding)
						{
							int32_t st = p.lm_state;
#if KB_CONG
							uint32_t sctx = P_CTX(p);
							c += cgNext(st, sctx, 1);
#elif KB_SBG
							uint32_t eh[8]; for (int i = 0; i < 8; ++i) eh[i] = p.hist[i];
							uint32_t ep = p.hpos;
							c += sbgNext(st, eh, ep, 1);
#else
							c += knProgress(st, 1, 5);
#endif
							if (p.sp_state & 1) c -= 2;
							if (p.sp_state & 2) c -= 2;
						}
					}
				}
				const unsigned om = __ballot_sync(FULL, ok);
				const uint32_t before = __popc(om & ((1u << lane) - 1));
				if (ok)
				{
					// cand record reuses PathT: acc_score = c, parent, root_id, sp_state
					if (p.root_id == COMMON_ROOT)
					{
						for (uint32_t r = 0; r < nUniq; ++r)
						{
							PathT cnd = p; cnd.acc_score = c; cnd.parent = inBeg + q; cnd.root_id = (uint8_t)r; cnd.sp_state = uniq[r]; cnd.wid = 1;
							pool[candBeg + (nCand + before) * perPath + r] = cnd;
						}
					}
					else
					{
						PathT cnd = p; cnd.acc_score = c; cnd.parent = inBeg + q; cnd.wid = 1;
						pool[candBeg + (nCand + before) * perPath] = cnd;
						for (uint32_t r = 1; r < nUniq; ++r) { PathT z = cnd; z.wid = 0; pool[candBeg + (nCand + before) * perPath + r] = z; }
					}
				}
				nCand += __popc(om);
			}
			__syncwarp();
			const uint32_t nRec = nCand * perPath;      // records with wid == 1 are real candidates, in the reference's emplace order
			// sort(cand) by (rootId, spState, score desc) EXACTLY as libstdc++'s std::sort does (std_sort_emu.h): equal-score candidates
			// - two morphemes with the same LM id - tie regularly, and which one comes first decides the emitted morpheme id
			SortRec* sr = reinterpret_cast<SortRec*>(pool + candBeg + nRec);
			uint32_t nReal = 0;
			for (uint32_t eb = 0; eb < nRec; eb += 32)
			{
				const uint32_t e = eb + lane;
				bool real = false; unsigned long long key = 0;
				if (e < nRec)
				{
					const PathT* r = pool + candBeg + e;
					real = r->wid != 0;
					uint32_t o = __float_as_uint(r->acc_score);
					o = (o & 0x80000000u) ? ~o : (o | 0x80000000u);
					key = ((unsigned long long)r->root_id << 40) | ((unsigned long long)r->sp_state << 32) | (unsigned long long)(~o);
				}
				const unsigned rm = __ballot_sync(FULL, real);
				const uint32_t k = nReal + __popc(rm & ((1u << lane) - 1));
				if ((size_t)(candBeg + nRec) * sizeof(PathT) + (size_t)(nReal + __popc(rm)) * sizeof(SortRec) > (size_t)poolCap * sizeof(PathT)) { err = ST_PATH_OVERFLOW; return 0; }
				if (real) { SortRec x; x.key = key; x.idx = e; x.pad = 0; sr[k] = x; }
				nReal += __popc(rm);
			}
			if (nReal == 0) return 0;
			__syncwarp();
#ifdef KB_HOSTSIM
			if (lane == 0 && std::getenv("HS32_TRACE_END")) { std::fprintf(stderr, "[hs32] end cands %u:", nReal); for (uint32_t z = 0; z < nReal; ++z) { const PathT* r = pool + candBeg + sr[z].idx; std::fprintf(stderr, " (%d,%d,%a,n%d,p%u)", r->root_id, r->sp_state, r->acc_score, pool[r->parent].node, r->parent); } std::fprintf(stderr, "\n"); }
#endif
			if (lane == 0) stdSortEmu(sr, (long)nReal);
			__syncwarp();
			// groups = runs of equal (rootId, spState) in the sorted order; keep the first ceil(2 / #groups) of every group
			uint32_t nGroups = 0;
			for (uint32_t eb = 0; eb < nReal; eb += 32)
			{
				const uint32_t e = eb + lane;
				const bool start = e < nReal && (e == 0 || (sr[e].key >> 32) != (sr[e - 1].key >> 32));
				nGroups += __popc(__ballot_sync(FULL, start));
			}
			const uint32_t perGroup = (2 + nGroups - 1) / nGroups;        // ceil(topN * 2 / numUniq), topN == 1
			uint32_t nRes = 0;
			for (uint32_t eb = 0; eb < nReal; eb += 32)
			{
				const uint32_t e = eb + lane;
				bool take = false;
				if (e < nReal)
				{
					const unsigned long long g = sr[e].key >> 32;
					take = e == 0 || (sr[e - 1].key >> 32) != g;                                    // first of its group
					if (!take && perGroup == 2) take = e == 1 || (sr[e - 2].key >> 32) != g;       // second of its group (single-group case only)
				}
				unsigned tm = __ballot_sync(FULL, take);
				while (tm)
				{
					const uint32_t src = __ffs(tm) - 1; tm &= tm - 1;
					if (nRes >= MAX_RESULTS) { err = ST_INTERNAL; return 0; }
					const PathT* r = pool + candBeg + sr[eb + src].idx;
					res[nRes].score = r->acc_score; res[nRes].endParent = r->parent;
					res[nRes].prevState = uniq[r->root_id]; res[nRes].curState = r->sp_state;
					++nRes;
				}
			}
			// sort(ret) by score desc (<= 16 elements: libstdc++ std::sort is an insertion sort -> stable)
			for (uint32_t a = 1; a < nRes; ++a)
			{
				const PathRes k = res[a]; uint32_t b = a;
				while (b && res[b - 1].score < k.score) { res[b] = res[b - 1]; --b; }
				res[b] = k;
			}
			(void)chunkBase;
			return nRes;
		}
	};

	// registers: 4 resident blocks for the Knlm kernel (128 registers); the CoNg kernel's larger per-warp state spills less at 3 blocks.
	// The Makefile overrides both per build.
	#ifndef KB_VIT_MIN_BLOCKS
#define KB_VIT_MIN_BLOCKS (KB_CONG ? 3 : 4)
#endif
	__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32, KB_VIT_MIN_BLOCKS) KB_VIT_KERNEL(const BatchView bv, const VitView vv)
	{
#ifdef KB_HOSTSIM
		alignas(16) static unsigned char smRaw[sizeof(WarpSmem) * WARPS_PER_BLOCK + sizeof(TeamSmem) * TEAMS_PER_BLOCK];      // tests/hostsim: one static arena
#else
		extern __shared__ __align__(16) unsigned char smRaw[];
#endif
		WarpSmem* smAll = reinterpret_cast<WarpSmem*>(smRaw);
		TeamSmem* teamSm = reinterpret_cast<TeamSmem*>(smRaw + sizeof(WarpSmem) * WARPS_PER_BLOCK);
		const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
		// The first n_team sentences of the launch order (the heaviest) get a TEAM of warps each: the blocks [0, nTeamBlocks) hold
		// TEAMS_PER_BLOCK teams; every other sentence gets one warp.
		const uint32_t nTeam = TEAM > 1 ? min(vv.n_team, bv.n_sent) : 0u;
		const uint32_t nTeamBlocks = (nTeam + TEAMS_PER_BLOCK - 1) / TEAMS_PER_BLOCK;
		if (threadIdx.x < TEAMS_PER_BLOCK) teamSm[threadIdx.x].err = 0;
		__syncthreads();
		uint32_t slot, teamRank = 0, teamSize = 1, teamIdx = 0;
#if KB_QUEUE
		// Work queue: the grid is one wave of resident blocks; every warp analyses one sentence after the other, taking the next position
		// of the launch order (heaviest predicted sentence first) from a global counter - a warp that drew a light sentence is back for
		// more at once, so the launch ends when its heaviest sentence does, not when the last statically assigned block has been scheduled.
		// The first solo_blocks blocks keep only solo_warps warps, which start with the very heaviest sentences (positions
		// 0 .. solo_blocks * solo_warps - 1) and so run them with little competition for their SM's issue slots and instruction cache.
		static_assert(TEAM == 1, "the work queue hands sentences to single warps");
		const uint32_t nSolo = min(vv.solo_blocks * vv.solo_warps, bv.n_sent);
		const bool soloBlock = blockIdx.x < vv.solo_blocks;
		if (soloBlock && wib >= vv.solo_warps) return;
		bool firstDraw = true;
		uint32_t pfPhaseKeep = 0, curBufKeep = 0;
#if KB_TMA_ROWS
		{ Vit v0{ lane }; v0.sm = &smAll[wib]; v0.pfInit(); }
#endif
		for (;;)
		{
		if (soloBlock && firstDraw && blockIdx.x * vv.solo_warps + wib < nSolo) slot = blockIdx.x * vv.solo_warps + wib;
		else
		{
			uint32_t d = 0;
			if (lane == 0) d = atomicAdd(vv.work_counter, 1u);
			slot = nSolo + __shfl_sync(0xFFFFFFFFu, d, 0);
		}
		firstDraw = false;
		if (slot >= bv.n_sent) return;
		const uint32_t s = bv.order[slot];
		if (bv.status[s]) { if (lane == 0) { vv.best_rec[s] = -1; vv.score[s] = 0; } continue; }
#else
		if (TEAM > 1 && blockIdx.x < nTeamBlocks)
		{
			teamIdx = wib / TEAM; teamRank = wib % TEAM; teamSize = TEAM;
			slot = blockIdx.x * TEAMS_PER_BLOCK + teamIdx;
			if (slot >= nTeam || wib >= TEAMS_PER_BLOCK * TEAM) return;      // (whole teams leave together)
		}
		else slot = nTeam + (blockIdx.x - nTeamBlocks) * WARPS_PER_BLOCK + wib;
		if (slot >= bv.n_sent) return;
		const uint32_t s = bv.order[slot];
		if (bv.status[s]) { if (lane == 0 && teamRank == 0) { vv.best_rec[s] = -1; vv.score[s] = 0; } return; }
#endif

#ifndef KB_HOSTSIM
		if (lane == 0 && teamRank == 0) { unsigned long long tns; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(tns)); vv.timing[2 * s] = tns; }
#endif
		const uint32_t t0 = bv.text_off[s], t1 = bv.text_off[s + 1];
		const uint32_t n = t1 - t0;
		const uint32_t W = 2 * n + 4;
		const size_t wbase = 2 * (size_t)t0 + 4 * (size_t)s;
		const size_t nbase = (size_t)bv.nodes_per_unit * wbase;
		const size_t pbase = (size_t)vv.paths_per_unit * wbase + (size_t)vv.paths_const * s;

		Vit v{ lane };
		v.norm = bv.norm + wbase;
		v.pool = reinterpret_cast<PathT*>(vv.paths) + pbase;      // (records of VitView::path_stride bytes)
		v.poolCap = vv.paths_per_unit * W + vv.paths_const;
		v.top = 0;
		v.sm = &smAll[wib]; v.ht = smAll[wib].ht; v.htUsed = 1;
		v.dcur = smAll[wib].dcandGen;
#if KB_TEAM > 1
		v.teamRank = teamRank; v.teamSize = teamSize; v.teamBar = 1 + teamIdx; v.tm = &teamSm[teamIdx];
#endif
#if KB_PHASE_CLOCKS
		v.phSent = s;
#endif
		v.splitComplex = (bv.match_options >> 22) & 1; v.splitSaisiot = (bv.match_options >> 25) & 1; v.mergeSaisiot = (bv.match_options >> 26) & 1;
		v.htClear();
		if (lane == 0) smAll[wib].exactInsert = 0;
		__syncwarp();
#if KB_TMA_ROWS
#if KB_QUEUE
		v.pfPhase = pfPhaseKeep; v.curBuf = curBufKeep;      // the warp's transaction barriers live across its sentences
#else
		v.pfInit();
#endif
#endif

		const DChunk* chunks = bv.chunks + (wbase >> 2) + 2 * (size_t)s;
		const uint32_t nChunks = bv.n_chunks[s];
		DRec* recs = vv.recs + 2 * ((wbase >> 2) + 2 * (size_t)s);
		const uint32_t normLen = bv.norm_len[s];

		// running results of insertPathIntoResults (<= 2 survive each chunk)
		uint32_t retN = 0; float retScore[2] = { 0, 0 }; uint8_t retSp[2] = { 0, 0 }; int32_t retRec[2] = { -1, -1 };
		uint32_t nRecs = 0;

		for (uint32_t c = 0; c < nChunks && !v.err; ++c)
		{
			const DChunk ch = chunks[c];
			v.nodes = bv.nodes + nbase + ch.node_off; v.N = ch.n_nodes;
			v.npOff = vv.node_path_off + nbase + ch.node_off; v.npCnt = vv.node_path_cnt + nbase + ch.node_off;
			v.reach = vv.reachable + nbase + ch.node_off;
			v.nodeCand = vv.node_cand + nbase + ch.node_off;
			// uniqStates = sorted unique of spStatesByRet, or {0} (PathEvaluator.hpp:1212-1218)
			if (retN == 0) { v.uniq[0] = 0; v.nUniq = 1; }
			else if (retN == 1 || retSp[0] == retSp[1]) { v.uniq[0] = retSp[0]; v.nUniq = 1; }
			else { v.uniq[0] = min(retSp[0], retSp[1]); v.uniq[1] = max(retSp[0], retSp[1]); v.nUniq = 2; }

			PathRes res[MAX_RESULTS];
			// AnalyzeOption::openEnding (bit 31 of the option word, capi.cu): no end-of-sentence step on the chunk that ends the text (src/Kiwi.cpp:1122-1131)
			KB_PH_START(tFind);
			const uint32_t K = v.findBestPath(ch, res, (bv.match_options >> 31) != 0 && ch.end == normLen);
			KB_PH_ADD(PH_FIND_BEST_PATH, tFind, s);

			// ---- insertPathIntoResults, topN == 1 (src/Kiwi.cpp:629-782), all lanes redundantly (team mode: the first warp's lanes)
			auto stitch = [&]()
			{
			struct Ret { float score; uint8_t sp; int32_t rec; uint32_t parent; };
			Ret ret[2 + MAX_RESULTS]; uint32_t nRet = 0;
			if (retN == 0)      // `ret.empty()` in the reference: also true again after a chunk that kept nothing
			{
				const uint32_t nn = min(K, 2u);
				for (uint32_t i = 0; i < nn; ++i) ret[nRet++] = Ret{ 0.f, 0, -1, i };
			}
			else
			{
				uint8_t ppKey[4]; uint32_t ppVal[4]; uint32_t nPP = 0;      // prevParents map
				bool selected[MAX_RESULTS];
				for (uint32_t i = 0; i < K; ++i) selected[i] = false;
				for (uint32_t i = 0; i < retN; ++i)
				{
					const uint8_t st = retSp[i];
					uint32_t from = 0; int32_t ppi = -1;
					for (uint32_t k = 0; k < nPP; ++k) if (ppKey[k] == st) { from = ppVal[k]; ppi = (int32_t)k; }
					uint32_t parent = from;
					for (; parent < K; ++parent) if (res[parent].prevState == st) break;
					if (parent >= K && from) { for (parent = 0; parent < K; ++parent) if (res[parent].prevState == st) break; }
					ret[nRet++] = Ret{ retScore[i], st, retRec[i], parent };
					if (ppi < 0) { ppi = (int32_t)nPP; ppKey[nPP] = st; ppVal[nPP] = 0; ++nPP; }   // operator[] default-inserts 0
					if (parent < K) { selected[parent] = true; ppVal[ppi] = parent + 1; }
				}
				for (uint32_t i = 0; i < K; ++i)
				{
					if (selected[i]) continue;
					uint32_t parent = 0;
					for (; parent < nRet; ++parent) if (ret[parent].sp == res[i].prevState) break;
					// NB: the reference searches spStatesByRet, which grows together with ret
					if (parent < nRet) { Ret r = ret[parent]; r.parent = i; ret[nRet++] = r; }
					else { v.err = ST_INTERNAL; break; }
				}
			}
			if (v.err) return;
			// keep the first path per curState, accumulate, then sort by score and keep 2
			Ret kept[2 + MAX_RESULTS]; uint32_t nKept = 0;
			uint8_t seenSt[2 + MAX_RESULTS]; uint32_t nSeen = 0;
			for (uint32_t i = 0; i < nRet; ++i)
			{
				if (!(ret[i].parent < K)) continue;
				const PathRes& r = res[ret[i].parent];
				bool dup = false;
				for (uint32_t k = 0; k < nSeen; ++k) if (seenSt[k] == r.curState) dup = true;
				if (dup) continue;
				seenSt[nSeen++] = r.curState;
				Ret o; o.score = ret[i].score + r.score; o.sp = r.curState; o.rec = ret[i].rec; o.parent = ret[i].parent;
				kept[nKept++] = o;
			}
			for (uint32_t a = 1; a < nKept; ++a)
			{
				const Ret k = kept[a]; uint32_t b = a;
				while (b && kept[b - 1].score < k.score) { kept[b] = kept[b - 1]; --b; }
				kept[b] = k;
			}
			retN = min(nKept, 2u);
			for (uint32_t i = 0; i < retN; ++i)
			{
				retScore[i] = kept[i].score; retSp[i] = kept[i].sp;
				if (lane == 0) recs[nRecs] = DRec{ kept[i].rec, res[kept[i].parent].endParent, c, kept[i].score };
				retRec[i] = (int32_t)nRecs;
				++nRecs;
			}
			__syncwarp();
			};
			if (v.leader() && !v.err) stitch();
			if (v.teamSize > 1)
			{
				// what the other warps of the team need for the next chunk: how many results survive and their special states, the pool top
				uint32_t a = retN | ((uint32_t)retSp[0] << 8) | ((uint32_t)retSp[1] << 16), b = v.top, cc = 0;
				v.teamBroadcast(a, b, cc);
				retN = a & 0xFF; retSp[0] = (uint8_t)(a >> 8); retSp[1] = (uint8_t)(a >> 16); v.top = b;
			}
			if (v.err) break;
		}

		// the best stitched result (ret[0]); tokens are materialised by emit_kernel
		(void)normLen;
#ifndef KB_HOSTSIM
		if (lane == 0 && teamRank == 0) { unsigned long long tns; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(tns)); vv.timing[2 * s + 1] = tns; }
#endif
		if (lane == 0 && teamRank == 0)
		{
			vv.best_rec[s] = (!v.err && retN) ? retRec[0] : -1;
			vv.score[s] = (!v.err && retN) ? retScore[0] : 0.f;
			if (v.err) bv.status[s] = v.err;
		}
#if KB_QUEUE
#if KB_TMA_ROWS
		v.pfDrain(); pfPhaseKeep = v.pfPhase; curBufKeep = v.curBuf;
#endif
		__syncwarp();
		}      // next sentence of the queue
#endif
	}

#if KB_CONG
	// ---- device self-test of the CoNg scorer pieces (kiwi_b200_debug_cong): one thread per (context, wid, node) triple for the
	// dp4a dot, the three epilogues and one context-trie transition; warp 0 of block 0 additionally runs the tensor-core tile over
	// the first min(n, 64) contexts x first min(n, 32) wids.
	__global__ void cong_debug_kernel(uint32_t n, const uint32_t* ctx, const uint32_t* wid, const int32_t* node,
		int32_t* outDot, float* outEps, int32_t* outNode, uint32_t* outCtx, int32_t* outTile)
	{
		__shared__ uint32_t sU[64]; __shared__ uint32_t sW[32]; __shared__ int32_t sD[64][33];
		const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
		if (i < n)
		{
			const int32_t x = cgDot(ctx[i], wid[i]);
			outDot[i] = x;
			outEps[3 * i + 0] = cgFinish(x, ctx[i], wid[i], CG_E_SCALAR);
			outEps[3 * i + 1] = cgFinish(x, ctx[i], wid[i], CG_E_SMALL);
			outEps[3 * i + 2] = cgFinish(x, ctx[i], wid[i], CG_E_GEMV);
			int32_t nd = node[i];
			outCtx[i] = cgStep(nd, wid[i]);
			outNode[i] = nd;
		}
		if (blockIdx.x == 0 && threadIdx.x < 32)
		{
			const uint32_t lane = threadIdx.x, nU = min(n, 64u), nW = min(n, 32u);
			for (uint32_t k = lane; k < nU; k += 32) sU[k] = ctx[k];
			if (lane < nW) sW[lane] = wid[lane];
			__syncwarp();
			cgTileDots(sU, sW, sD, nU, nW == 32 ? 0xFFFFFFFFu : ((1u << nW) - 1), lane);
			for (uint32_t k = lane; k < nU * nW; k += 32) outTile[k] = sD[k / nW][k % nW];
		}
	}
#endif
}   // namespace KB_VIT_NS
	using namespace KB_VIT_NS;

#if KB_CONG && !defined(KB_HOSTSIM)
	cudaError_t launch_cong_debug(uint32_t n, const uint32_t* ctx, const uint32_t* wid, const int32_t* node,
		int32_t* outDot, float* outEps, int32_t* outNode, uint32_t* outCtx, int32_t* outTile, cudaStream_t stream)
	{
		cong_debug_kernel<<<(n + 127) / 128, 128, 0, stream>>>(n, ctx, wid, node, outDot, outEps, outNode, outCtx, outTile);
		return cudaGetLastError();
	}
#endif

#if KB_SBG
#define KB_SET_MODEL set_model_viterbi_sbg
#define KB_LAUNCH launch_viterbi_sbg
#elif KB_CONG
#define KB_SET_MODEL set_model_viterbi_cong
#define KB_LAUNCH launch_viterbi_cong
#else
#define KB_SET_MODEL set_model_viterbi
#define KB_LAUNCH launch_viterbi
#endif
	cudaError_t KB_SET_MODEL(const DevModel& m) { return cudaMemcpyToSymbol(c_m, &m, sizeof(DevModel)); }

	cudaError_t KB_LAUNCH(const DevModel&, const BatchView& bv, const VitView& vv, cudaStream_t stream)
	{
		if (bv.n_sent == 0) return cudaSuccess;
		if (vv.path_stride != sizeof(PathT)) return (cudaError_t)1;      // the arena was sized for another record type
		const uint32_t nTeam = TEAM > 1 ? (vv.n_team < bv.n_sent ? vv.n_team : bv.n_sent) : 0u;
		const uint32_t blocks = (nTeam + TEAMS_PER_BLOCK - 1) / TEAMS_PER_BLOCK + (bv.n_sent - nTeam + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK;
		static bool attrSetOn[64] = {};      // function attributes are per device (the caller holds that device's lock)
		int devId = 0;
#ifndef KB_HOSTSIM
		cudaGetDevice(&devId);
#endif
		bool& attrSet = attrSetOn[devId & 63];
		const size_t smemBytes = sizeof(WarpSmem) * WARPS_PER_BLOCK + sizeof(TeamSmem) * TEAMS_PER_BLOCK;
		if (!attrSet)
		{
			cudaFuncSetAttribute(KB_VIT_KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smemBytes);
			// kernel experiments: KIWI_B200_CARVEOUT=<percent> overrides the shared-memory / L1 split the driver picks
			if (const char* co = getenv("KIWI_B200_CARVEOUT")) cudaFuncSetAttribute(KB_VIT_KERNEL, cudaFuncAttributePreferredSharedMemoryCarveout, atoi(co));
			attrSet = true;
		}
#if KB_QUEUE
		// work queue: one wave of resident blocks (SM count x blocks per SM at this register / shared-memory footprint)
		VitView vq = vv;
		if (!vq.work_counter) return (cudaError_t)1;      // cudaErrorInvalidValue
		uint32_t grid = blocks;
#ifndef KB_HOSTSIM
		static int residentOn[64] = {};
		int& resident = residentOn[devId & 63];
		if (!resident)
		{
			int perSm = 0, sms = 0;
			cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, KB_VIT_KERNEL, WARPS_PER_BLOCK * 32, smemBytes);
			cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, devId);
			resident = perSm > 0 && sms > 0 ? perSm * sms : 132;
		}
		if (vq.solo_warps == 0 || vq.solo_warps > WARPS_PER_BLOCK) vq.solo_blocks = 0;
		// the solo blocks' missing warps are made up for by as many extra blocks only if they would still be resident: they are not, so the
		// wave stays at `resident` blocks and the solo blocks trade (WARPS_PER_BLOCK - solo_warps) warp slots each for an undisturbed SM
		grid = blocks + vq.solo_blocks < (uint32_t)resident ? blocks + vq.solo_blocks : (uint32_t)resident;
		if (vq.solo_blocks > grid / 2) vq.solo_blocks = grid / 2;
		if (cudaError_t e = cudaMemsetAsync(vq.work_counter, 0, sizeof(uint32_t), stream)) return e;
#else
		vq.solo_blocks = 0; *vq.work_counter = 0;
#endif
#define KB_VV vq
#define KB_GRID grid
#else
#define KB_VV vv
#define KB_GRID blocks
#endif
#ifdef KB_HOSTSIM
		// tests/hostsim: one sentence, one block of WARPS_PER_BLOCK warps (one warp works, or - n_team == 1 - one team)
		if (bv.n_sent != 1) return 1;
		(void)stream; (void)smemBytes;
		simt::launch(KB_GRID, WARPS_PER_BLOCK * 32, [&] { KB_VIT_KERNEL(bv, KB_VV); });
		return cudaSuccess;
#else
		KB_VIT_KERNEL<<<KB_GRID, WARPS_PER_BLOCK * 32, smemBytes, stream>>>(bv, KB_VV);
		return cudaGetLastError();
#endif
	}
}

#if KB_PHASE_CLOCKS && !KB_CONG && !KB_SBG && !defined(KB_HOSTSIM)
// diagnostic build only: copies phaseClocks ([KB_PHASE_SENT][PH_COUNT] cycles) to `out` and zeroes them
extern "C" __attribute__((visibility("default"))) int kiwi_b200_debug_phase_clocks(unsigned long long* out)
{
	using namespace kb::vit_knlm;
	static unsigned long long zero[KB_PHASE_SENT * PH_COUNT];
	if (cudaDeviceSynchronize() || cudaMemcpyFromSymbol(out, phaseClocks, sizeof(zero)) || cudaMemcpyToSymbol(phaseClocks, zero, sizeof(zero))) return -1;
	return PH_COUNT;
}
#endif
