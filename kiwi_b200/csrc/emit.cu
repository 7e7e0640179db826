// kiwi_b200 kernel C: token emission, one thread per sentence.
//
// Replaces generateTokenList (/root/reference/src/PathEvaluator.hpp:1038-1157) and the token part of
// insertPathIntoResults (src/Kiwi.cpp:696-751: space pseudo-tokens dropped, position/length mapped back to the
// original string through the position table, script re-tagging of sl/sh/sw/w_emoji tokens).  The Viterbi
// kernel leaves, per sentence, the record chain of the best stitched result; this kernel walks the parent
// links of each chunk's best path (a short, inherently serial pointer walk) and writes the token rows.
#include <cuda_runtime.h>
#include "kb_model.h"
#include "kb_batch.h"

namespace kb
{
	__constant__ DevModel c_m;
	static constexpr uint32_t NPOS = 0xFFFFFFFFu;

	__device__ __forceinline__ uint32_t upperBound(const uint32_t* t, uint32_t n, uint32_t v)
	{
		uint32_t lo = 0, hi = n;
		while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (t[mid] <= v) lo = mid + 1; else hi = mid; }
		return lo;
	}
	__device__ __forceinline__ uint32_t lowerBound(const uint32_t* t, uint32_t n, uint32_t v)
	{
		uint32_t lo = 0, hi = n;
		while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (t[mid] < v) lo = mid + 1; else hi = mid; }
		return lo;
	}

	// JOIN: the token-joining fold runs over every chunk's rows (emit_join_kernel), which needs each row's own surface form: src[i] = the
	// {own_off, own_len} its pushTok had
	template<bool JOIN> struct Emitter
	{
		const uint16_t* norm; const uint32_t* posTable; uint32_t n, W;
		DToken* out; uint32_t nTok = 0; uint32_t err = 0;
		DToken backTok; uint32_t backBegin = 0, backEnd = 0; bool backValid = false, backSkip = false;
		uint2* src; uint32_t backOwnOff = 0, backOwnLen = 0;

		__device__ Emitter() {}

		__device__ void flushBack()
		{
			if (!backValid) return;
			if (!backSkip)
			{
				if (nTok >= W) { err = ST_TOKEN_OVERFLOW; return; }
				DToken t = backTok;
				const uint32_t beginPos = upperBound(posTable, n + 1, backBegin) - 1;
				const uint32_t endPos = lowerBound(posTable, n + 1, backEnd);
				t.position = beginPos; t.length = (uint16_t)(endPos - beginPos);
				if constexpr (JOIN) src[nTok] = make_uint2(backOwnOff, backOwnLen);
				out[nTok++] = t;
			}
			backValid = false;
		}
		__device__ uint16_t ownChar(uint32_t ownOff, uint32_t k) const
		{
			return (ownOff & 0x80000000u) ? c_m.form_chars[c_m.forms_raw[~ownOff].str_off + k] : norm[ownOff + k];
		}
		// PathNode::typoCost = the node's typo cost / the number of tokens the node yields (PathEvaluator.hpp:1066-1074) travels in
		// DToken::flags: bits 1-3 the node's cost in units of 0.5 (the default typo sets use 1, 1.5 and 2; saturates at 3.5),
		// bits 4-7 the token count - 1; the host divides as the reference does
		uint8_t typoBits = 0;
		__device__ void setTypoCost(float typoCostDiff, uint32_t numNewTokens)
		{
			const float q = typoCostDiff * 2.f + 0.5f;
			const uint32_t v = q <= 0.f ? 0u : (q >= 7.f ? 7u : (uint32_t)q);
			const uint32_t n1 = (numNewTokens > 16 ? 16u : numNewTokens) - 1;
			typoBits = v ? (uint8_t)((v << 1) | (n1 << 4)) : 0;
		}
		__device__ void pushTok(uint32_t morph, uint32_t begin, uint32_t end, float score, uint32_t ownOff, uint32_t ownLen)
		{
			flushBack();
			const DMorph mm = c_m.morphs[morph];
			backTok.morph = morph; backTok.tag = (uint8_t)(mm.feat & MF_TAG_MASK); backTok.score = score; backTok.flags = (uint8_t)((ownLen ? 1 : 0) | typoBits);
			backTok.position = 0; backTok.length = 0;
			backBegin = begin; backEnd = end; backValid = true; backSkip = false;
			if constexpr (JOIN) { backOwnOff = ownOff; backOwnLen = ownLen; }
			if (ownLen)
			{
				const uint32_t c0 = ownChar(ownOff, 0);
				if (c0 == ' ') backSkip = true;
				// updateTokenInfoScript (src/Kiwi.cpp:590-605)
				const uint32_t tg = backTok.tag;
				if ((tg == T_sl || tg == T_sh || tg == T_sw || tg == T_w_emoji) && !(mm.form_idx >= 0 && c_m.forms[mm.form_idx].str_len))
				{
					uint32_t cc = c0;
					if (isHighSurrogate(cc)) cc = mergeSurrogate(cc, ownLen > 1 ? ownChar(ownOff, 1) : 0);
					if (attrScript(chrAttr(c_m, cc)) == c_m.script_latin) backTok.tag = T_sl;
				}
			}
		}
		__device__ uint32_t unify(uint32_t morph) const      // PathEvaluator.hpp:1054-1058
		{
			if (!(morph < c_m.lang_vocab_size) || c_m.morphs[morph].combined) return morph;
			return c_m.morphs[morph].lm_id;
		}
	};

	// ---- token joining (Match::join*, mergeSaisiot, joinParticleYo): joinAffixTokens, /root/reference/src/Kiwi.cpp:495-588 ----------
	// A joined row keeps its first token's position, score and flags (concatTokens, Kiwi.cpp:487-493), spans to the end of its last one
	// and carries JOINED_TOKEN | k: its form is not a substring of the text, so it is written to the sentence's form pool at k.
	struct JoinPool { uint16_t* p = nullptr; uint32_t len = 0, cap = 0; };

	__device__ __forceinline__ bool kformIsYo(uint32_t morph)
	{
		const int32_t fi = c_m.morphs[morph].form_idx;
		return fi >= 0 && c_m.forms_raw[fi].str_len == 1 && c_m.form_chars[c_m.forms_raw[fi].str_off] == 0xC694;
	}

	// appends one component's TokenInfo::str (Kiwi.cpp:723-729): joinHangul over its own form (OOV / pattern tokens) or its morpheme's
	// kform, then, with Match::compatibleJamo, the compatibility jamo.  false: the pool is full.
	__device__ bool appendForm(JoinPool& jp, const uint16_t* norm, uint32_t morph, uint2 own, bool compat)
	{
		const uint16_t* srcChars; uint32_t srcLen;
		if (own.y) srcChars = (own.x & 0x80000000u) ? c_m.form_chars + c_m.forms_raw[~own.x].str_off : norm + own.x, srcLen = own.y;
		else
		{
			const int32_t fi = c_m.morphs[morph].form_idx;
			srcChars = fi >= 0 ? c_m.form_chars + c_m.forms_raw[fi].str_off : nullptr; srcLen = fi >= 0 ? c_m.forms_raw[fi].str_len : 0;
		}
		const uint32_t start = jp.len;
		for (uint32_t k = 0; k < srcLen; ++k)
		{
			if (jp.len + 4 > jp.cap) return false;      // (3 units at most, and the entry's terminating 0)
			const uint32_t c = srcChars[k];
			uint16_t* back = jp.p + jp.len - 1;
			// joinHangul, include/kiwi/Utils.h:167-205
			if (jp.len > start && isHangulSyllable(*back) && (*back - 0xAC00u) % 28 == 0)
			{
				if (isHangulCoda(c)) { *back = (uint16_t)(*back + (c - 0x11A7)); continue; }
				if ((0x11A8 <= c && c < 0x1200) || (0xD7CB <= c && c < 0xD800))
				{
					const uint32_t onset = (*back - 0xAC00u) / 28 / 21, vowel = (*back - 0xAC00u) / 28 % 21;
					*back = (uint16_t)(0x1100 + onset);
					jp.p[jp.len++] = (uint16_t)(0x1161 + vowel);
				}
			}
			jp.p[jp.len++] = (uint16_t)c;
		}
		if (compat) for (uint32_t i = start; i < jp.len; ++i) jp.p[i] = toCompatibleJamo(jp.p[i]);
		return true;
	}

	// the fold over the rows [c0, nTok), in place and in the reference's rule order.  The reference folds the whole token list again after
	// each chunk (insertPathIntoResults, Kiwi.cpp:756), which leaves the earlier chunks' rows as they were except the last two: the last row
	// may join the new chunk's first, and a trailing Z_SIOT may merge into the new chunk's first noun.  So c0 is the start of the chunk's
	// rows minus two, and a joined row there gets its entry (the pool's last) reopened.
	__device__ void joinChunk(DToken* out, uint2* src, uint32_t c0, uint32_t& nTok, uint32_t opt, const uint16_t* norm, JoinPool& jp, uint32_t& err)
	{
		const uint32_t c1 = nTok;
		if (c1 < c0 + 2) return;
		const bool compat = (opt & MO_COMPATIBLE_JAMO) != 0;
		uint32_t f = c0;
		DToken cur = out[f];
		bool joined = false; uint32_t entry = 0;
		for (uint32_t nx = c0 + 1; nx < c1;)
		{
			const DToken nt = out[nx];
			const uint8_t ct = cur.tag, ntg = nt.tag;
			const bool curNN = isNNClass(ct), curStem = curNN || ct == T_xr;
			uint32_t last = nx; uint8_t tag; bool saisiot = false;
			if ((opt & MO_JOIN_NOUN_PREFIX) && ct == T_xpn && (isNNClass(ntg) || ntg == T_sn)) tag = ntg;
			else if ((opt & MO_JOIN_NOUN_SUFFIX) && ntg == T_xsn && (curNN || ct == T_sn)) tag = ct;
			else if ((opt & MO_JOIN_VERB_SUFFIX) && clearIrregular(ntg) == T_xsv && curStem) tag = (uint8_t)(T_vv | (ntg & 0x80));
			else if ((opt & MO_JOIN_ADJ_SUFFIX) && clearIrregular(ntg) == T_xsa && curStem) tag = (uint8_t)(T_va | (ntg & 0x80));
			else if ((opt & MO_JOIN_ADV_SUFFIX) && ntg == T_xsm && curStem) tag = T_mag;
			else if ((opt & MO_MERGE_SAISIOT) && ntg == T_z_siot && curNN && nx + 1 < c1 && isNNClass(out[nx + 1].tag)) { tag = T_nng; last = nx + 1; saisiot = true; }
			else if ((opt & MO_JOIN_PARTICLE_YO) && ntg == T_jx && kformIsYo(nt.morph) && (ct == T_ec || ct == T_ef)) tag = ct;
			else
			{
				if (joined) jp.p[jp.len++] = 0;
				out[f++] = cur;
				cur = nt; src[f] = src[nx];
				joined = false;
				++nx;
				continue;
			}
			if (!joined && (cur.morph & JOINED_TOKEN))
			{
				// a row an earlier chunk's fold joined: its entry is the last in the pool; drop its terminating 0 and go on appending
				entry = cur.morph & ~JOINED_TOKEN;
				if (!jp.len || jp.p[jp.len - 1] != 0) { err = ST_INTERNAL; return; }
				--jp.len;
				joined = true;
			}
			if (!joined)
			{
				// a new entry: the first component's morpheme id, then its form
				if (jp.len + 3 > jp.cap) { err = ST_TOKEN_OVERFLOW; return; }
				entry = jp.len;
				jp.p[jp.len++] = (uint16_t)(cur.morph & 0xFFFF); jp.p[jp.len++] = (uint16_t)(cur.morph >> 16);
				if (!appendForm(jp, norm, cur.morph, src[f], compat)) { err = ST_TOKEN_OVERFLOW; return; }
				cur.morph = JOINED_TOKEN | entry;
				joined = true;
			}
			if (saisiot && jp.len > entry + 2) jp.p[jp.len - 1] = (uint16_t)(jp.p[jp.len - 1] + (0x11BA - 0x11A7));      // coda ㅅ on the left form's last unit
			if (!appendForm(jp, norm, out[last].morph, src[last], compat)) { err = ST_TOKEN_OVERFLOW; return; }
			cur.tag = tag;
			cur.length = (uint16_t)(out[last].position + out[last].length - cur.position);
			nx = last + 1;
		}
		if (joined) jp.p[jp.len++] = 0;
		out[f] = cur;
		nTok = f + 1;
	}

	template<bool JOIN> __device__ __forceinline__ void emitSentence(const BatchView& bv, const VitView& vv, uint32_t s)
	{
		const int32_t best = vv.best_rec[s];
		if (best < 0 || bv.status[s]) { vv.n_tokens[s] = 0; if constexpr (JOIN) vv.n_forms[s] = 0; return; }
		const uint32_t t0 = bv.text_off[s], t1 = bv.text_off[s + 1];
		const uint32_t n = t1 - t0;
		const uint32_t W = 2 * n + 4;
		const size_t wbase = 2 * (size_t)t0 + 4 * (size_t)s;
		const size_t nbase = (size_t)bv.nodes_per_unit * wbase;
		const size_t pbase = (size_t)vv.paths_per_unit * wbase + (size_t)vv.paths_const * s;
		// (records of vv.path_stride bytes: the SkipBigram build appends its history to DPath)
		const char* poolBytes = reinterpret_cast<const char*>(vv.paths) + pbase * (size_t)vv.path_stride;
		const uint32_t stride = vv.path_stride;
		auto P = [&](uint32_t i) -> const DPath& { return *reinterpret_cast<const DPath*>(poolBytes + (size_t)i * stride); };
		const DChunk* chunks = bv.chunks + (wbase >> 2) + 2 * (size_t)s;
		const DRec* recs = vv.recs + 2 * ((wbase >> 2) + 2 * (size_t)s);
		const bool splitSaisiot = (bv.match_options >> 25) & 1;

		Emitter<JOIN> e;
		e.norm = bv.norm + wbase; e.posTable = bv.pos_table + t0 + s; e.n = n; e.W = W; e.out = vv.tokens + wbase;
		JoinPool jp{};
		if constexpr (JOIN)
		{
			e.src = bv.end_pos_map + wbase;      // (the lattice's end-position map is free once the lattice is built; a join call runs no sentence kernel)
			jp.p = vv.forms + (size_t)vv.forms_per_unit * wbase; jp.cap = vv.forms_per_unit * W;
		}

		// record chain, last chunk first
		uint32_t* chain = bv.ctr + wbase;                // W entries, free after kernel A
		uint32_t L = 0;
		for (int32_t r = best; r >= 0; r = recs[r].parent_rec) chain[L++] = (uint32_t)r;
		uint32_t* steps = bv.ns_to_pos + wbase;          // backtrack scratch (W entries)
		for (int32_t ci = (int32_t)L - 1; ci >= 0 && !e.err; --ci)
		{
			const uint32_t chunkTok0 = e.nTok;
			const DRec rec = recs[chain[ci]];
			const DChunk ch = chunks[rec.chunk];
			const DNode* gnodes = bv.nodes + nbase + ch.node_off;
			uint32_t nSteps = 0;
			for (uint32_t p = rec.end_parent; P(p).parent != NPOS; p = P(p).parent)
			{
				if (nSteps >= W) { e.err = ST_TOKEN_OVERFLOW; break; }
				steps[nSteps++] = p;
			}
			if (e.err || !nSteps) break;
			uint32_t prevIdx = P(steps[nSteps - 1]).parent;
			for (int32_t si = (int32_t)nSteps - 1; si >= 0 && !e.err; --si)
			{
				const DPath cur = P(steps[si]);
				const float prevAcc = P(prevIdx).acc_score, prevTypo = P(prevIdx).acc_typo_cost;
				const float scoreDiff = cur.acc_score - prevAcc;
				const float typoCostDiff = cur.acc_typo_cost - prevTypo;
				const DMorph mm = c_m.morphs[cur.morpheme];
				const bool single = (mm.feat & MF_SINGLE) != 0;
				const bool saisiot = (mm.misc & MM_SAISIOT) != 0;
				const uint32_t numNewTokens = ((splitSaisiot && saisiot) || !single) ? mm.chunk_cnt : 1;
				const DNode g = gnodes[cur.node];
				const float firstScore = cur.first_chunk_score + typoCostDiff * c_m.cfg.typo_cost_weight;
				const float restScores = numNewTokens > 1 ? (scoreDiff - cur.first_chunk_score) / (float)(numNewTokens - 1) : 0.f;
				e.setTypoCost(typoCostDiff, numNewTokens);
				if (splitSaisiot && saisiot)
				{
					for (uint32_t chn = 0; chn < numNewTokens; ++chn)
					{
						const kb2_chunk ck = c_m.chunks[mm.chunk_off + chn];
						e.pushTok(e.unify(ck.morph), g.start_pos + ck.begin, g.start_pos + ck.end, chn == 0 ? firstScore : restScores, 0, 0);
					}
					e.backEnd = g.end_pos;
				}
				else if (single)
				{
					e.pushTok(e.unify((uint32_t)cur.morpheme), g.start_pos, g.end_pos, firstScore, cur.own_off, cur.own_len);
				}
				else if (mm.combine_socket)
				{
					// ret.back() is merged with the left half (PathEvaluator.hpp:1111-1134)
					e.backTok.morph = e.backTok.morph + c_m.morphs[e.backTok.morph].combined;
					e.backTok.tag = (uint8_t)(c_m.morphs[e.backTok.morph].feat & MF_TAG_MASK);
					e.backEnd = g.start_pos + c_m.chunks[mm.chunk_off].end;
					e.backTok.score = firstScore;
					e.backTok.flags = (uint8_t)((e.backTok.flags & 1) | e.typoBits);
					for (uint32_t chn = 1; chn < numNewTokens; ++chn)
					{
						const kb2_chunk ck = c_m.chunks[mm.chunk_off + chn];
						e.pushTok(e.unify(ck.morph), g.start_pos + ck.begin, g.start_pos + ck.end, restScores, 0, 0);
					}
					e.backEnd = g.end_pos;
				}
				else
				{
					for (uint32_t chn = 0; chn < numNewTokens; ++chn)
					{
						const kb2_chunk ck = c_m.chunks[mm.chunk_off + chn];
						e.pushTok(e.unify(ck.morph), g.start_pos + ck.begin, g.start_pos + ck.end, chn == 0 ? firstScore : restScores, 0, 0);
					}
					e.backEnd = g.end_pos;
				}
				prevIdx = steps[si];
			}
			e.flushBack();
			if constexpr (JOIN) if (!e.err) joinChunk(e.out, e.src, chunkTok0 > 2 ? chunkTok0 - 2 : 0, e.nTok, bv.match_options, e.norm, jp, e.err);
		}
		if (e.err) { bv.status[s] = e.err; vv.n_tokens[s] = 0; vv.score[s] = 0.f; }
		else vv.n_tokens[s] = e.nTok;
		if constexpr (JOIN) vv.n_forms[s] = e.err ? 0 : jp.len;
	}

	__global__ void __launch_bounds__(128) emit_kernel(const BatchView bv, const VitView vv)
	{
		const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
		if (s >= bv.n_sent) return;
		emitSentence<false>(bv, vv, s);
	}

	// launched instead of emit_kernel when a token-joining match option is set: the same emission, then the fold over every chunk
	__global__ void __launch_bounds__(128) emit_join_kernel(const BatchView bv, const VitView vv)
	{
		const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
		if (s >= bv.n_sent) return;
		emitSentence<true>(bv, vv, s);
	}

	cudaError_t set_model_emit(const DevModel& m) { return cudaMemcpyToSymbol(c_m, &m, sizeof(DevModel)); }

	cudaError_t launch_emit(const DevModel&, const BatchView& bv, const VitView& vv, cudaStream_t stream)
	{
		if (bv.n_sent == 0) return cudaSuccess;
#ifdef KB_HOSTSIM
		(void)stream;
		if (bv.n_sent != 1) return 1;
		if (bv.match_options & MO_JOIN_ANY) simt::launch(1, 1, [&] { emit_join_kernel(bv, vv); });      // thread-per-sentence kernel: one lane
		else simt::launch(1, 1, [&] { emit_kernel(bv, vv); });
		return cudaSuccess;
#else
		if (bv.match_options & MO_JOIN_ANY) emit_join_kernel<<<(bv.n_sent + 127) / 128, 128, 0, stream>>>(bv, vv);
		else emit_kernel<<<(bv.n_sent + 127) / 128, 128, 0, stream>>>(bv, vv);
		return cudaGetLastError();
#endif
	}
}
