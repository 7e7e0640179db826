// kiwi_b200 kernel D: sentence ranges of every document of a pass (Kiwi::splitIntoSents, src/Kiwi.cpp:417-436), one warp per
// document, launched after emit_kernel only when a split was asked for.
//
// The lanes build the per-token inputs of the sentence rules (sentences.h) from the unpacked token rows and the raw text: the
// newline count before every position, and each token's bracket / bullet family, "하" and "요" bits.  Lane 0 then runs the
// pairing, the sentence fold and the range derivation, which are serial by nature and cost a few operations per token.
// Scratch is the document's own W-sized regions that the lattice kernel used and nothing reads after it: the newline counts in
// bv.ctr, the tokens and the two pairing stacks in bv.build_nodes (48 of its >= 384 bytes per unit), the ranges in bv.end_pos_map.
#include <cuda_runtime.h>
#include "kb_model.h"
#include "kb_batch.h"
#include "sentences.h"

namespace kb
{
	__constant__ DevModel c_ms;

	__device__ __forceinline__ void sents_document(const BatchView& bv, const VitView& vv, uint32_t s, uint32_t lane, uint32_t* nSents)
	{
		const uint32_t t0 = bv.text_off[s], n = bv.text_off[s + 1] - t0;
		const size_t wbase = 2 * (size_t)t0 + 4 * (size_t)s;
		const uint32_t cnt = bv.status[s] ? 0u : vv.n_tokens[s];
		if (cnt == 0) { if (lane == 0) nSents[s] = 0; return; }
		const uint16_t* text = bv.text + t0;
		const DToken* rows = vv.tokens + wbase;
		uint32_t* nlBefore = bv.ctr + wbase;                       // [n + 1] newlines before each position
		SentTok* toks = reinterpret_cast<SentTok*>(bv.build_nodes + (size_t)bv.nodes_per_unit * wbase);
		uint2* stacks = reinterpret_cast<uint2*>(toks + cnt);     // 2 x cnt pairing stack entries
		uint2* ranges = bv.end_pos_map + wbase;

		uint32_t carry = 0;
		for (uint32_t base = 0; base <= n; base += 32)
		{
			const uint32_t i = base + lane;
			const unsigned nl = __ballot_sync(0xFFFFFFFFu, i < n && isNewlineAt(text, i));
			if (i <= n) nlBefore[i] = carry + __popc(nl & ((1u << lane) - 1u));
			carry += __popc(nl);
		}
		__syncwarp();
		for (uint32_t i = lane; i < cnt; i += 32)
		{
			const DToken d = rows[i];
			const DMorph mm = c_ms.morphs[d.morph];
			SentTok t{};
			t.position = d.position; t.length = d.length; t.tag = d.tag; t.pairedToken = NO_PAIR;
			t.flags = (mm.misc & MM_KFORM_YO) ? SF_YO : 0;
			t.lineNumber = nlBefore[d.position < n ? d.position : n];
			// the token's form as makeRes takes it: its own substring of the text, else the morpheme's form
			if (d.flags & 1) setSentForm(t, text + d.position, d.length);
			else if (mm.form_idx >= 0) setSentForm(t, c_ms.form_chars + c_ms.forms_raw[mm.form_idx].str_off, c_ms.forms[mm.form_idx].str_len);
			toks[i] = t;
		}
		__syncwarp();
		if (lane == 0)
		{
			pairTokens(toks, cnt, stacks, stacks + cnt);
			foldSentLine(toks, cnt);
			nSents[s] = sentRanges(toks, cnt, ranges);
		}
	}

	cudaError_t set_model_sents(const DevModel& m) { return cudaMemcpyToSymbol(c_ms, &m, sizeof(DevModel)); }

#ifndef KB_HOSTSIM
	__global__ void __launch_bounds__(128) sents_kernel(const BatchView bv, const VitView vv, uint32_t* __restrict__ nSents)
	{
		const uint32_t s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
		if (s >= bv.n_sent) return;
		sents_document(bv, vv, s, threadIdx.x & 31, nSents);
	}

	// the documents' ranges, contiguous: begin / end of document s at sentOff[s]
	__global__ void sents_pack_kernel(const BatchView bv, const uint32_t* __restrict__ nSents, const uint32_t* __restrict__ sentOff,
		uint32_t* __restrict__ begin, uint32_t* __restrict__ end)
	{
		const uint32_t lane = threadIdx.x & 31;
		const uint32_t s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
		if (s >= bv.n_sent) return;
		const size_t wbase = 2 * (size_t)bv.text_off[s] + 4 * (size_t)s;
		const uint32_t k = nSents[s], o = sentOff[s];
		for (uint32_t i = lane; i < k; i += 32) { const uint2 r = bv.end_pos_map[wbase + i]; begin[o + i] = r.x; end[o + i] = r.y; }
	}

	// nSents[s] and the document-relative ranges in bv.end_pos_map + wbase of every document of the launch
	cudaError_t launch_sents(const BatchView& bv, const VitView& vv, uint32_t* nSents, cudaStream_t stream)
	{
		if (bv.n_sent == 0) return cudaSuccess;
		const uint32_t threads = 128, blocks = (bv.n_sent * 32 + threads - 1) / threads;
		sents_kernel<<<blocks, threads, 0, stream>>>(bv, vv, nSents);
		return cudaGetLastError();
	}

	cudaError_t launch_sents_pack(const BatchView& bv, const uint32_t* nSents, const uint32_t* sentOff, uint32_t* begin, uint32_t* end, cudaStream_t stream)
	{
		if (bv.n_sent == 0) return cudaSuccess;
		const uint32_t threads = 256, blocks = (bv.n_sent * 32 + threads - 1) / threads;
		sents_pack_kernel<<<blocks, threads, 0, stream>>>(bv, nSents, sentOff, begin, end);
		return cudaGetLastError();
	}
#else
	// host simulation (tests/hostsim): one 32-lane warp per document, ranges left unpacked
	cudaError_t launch_sents(const BatchView& bv, const VitView& vv, uint32_t* nSents, cudaStream_t)
	{
		for (uint32_t s = 0; s < bv.n_sent; ++s) simt::launch(1, 32, [&] { sents_document(bv, vv, s, simt::lane, nSents); });
		return cudaSuccess;
	}
#endif
}
