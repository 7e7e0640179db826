// TEST INFRASTRUCTURE: the sentence splitter without a GPU, behind a small C API for tests/test_sents.py.
//  * ss_core_ranges: the shared rule core (kiwi_b200/csrc/sentences.h) on host tokens given with their surface forms;
//  * ss32_rows: kiwi_b200/csrc/sents.cu - the device source - compiled as C++ and run on a simulated 32-lane warp
//    (tests/hostsim/shim32) over one document's token rows;
//  * hs32_* (pipeline_sim32.cpp, linked in): the simulated lattice -> Viterbi -> emit pipeline, whose rows ss32_rows then takes.
// tests/test_sents.py compiles this file, pipeline_sim32.cpp and sents.cu with the objects the build leaves in tests/hostsim/obj32.
#include <cuda_runtime.h>
#include <algorithm>
#include <mutex>
#include <vector>
#include "../../kiwi_b200/csrc/engine.h"
#include "../../kiwi_b200/csrc/sentences.h"

namespace kb
{
	cudaError_t launch_sents(const BatchView& bv, const VitView& vv, uint32_t* nSents, cudaStream_t stream);
	cudaError_t set_model_sents(const DevModel& m);
}

namespace { std::mutex g_ssMtx; }

extern "C" {

// tokens (position, length, tag, surface form, kform-is-요) of one text -> ranges[2 * k]; returns k
int ss_core_ranges(int n, const uint32_t* pos, const uint32_t* len, const uint8_t* tag, const uint16_t* formBlob, const uint32_t* formOff,
	const uint8_t* isYo, const uint16_t* text, uint32_t textLen, uint32_t* out)
{
	using namespace kb;
	std::vector<uint32_t> nlBefore(textLen + 1, 0);
	for (uint32_t i = 0; i < textLen; ++i) nlBefore[i + 1] = nlBefore[i] + (isNewlineAt(text, i) ? 1 : 0);
	std::vector<SentTok> t((size_t)n);
	for (int i = 0; i < n; ++i)
	{
		t[i] = SentTok{};
		t[i].position = pos[i]; t[i].length = len[i]; t[i].tag = tag[i]; t[i].flags = isYo[i] ? SF_YO : 0; t[i].pairedToken = NO_PAIR;
		t[i].lineNumber = nlBefore[std::min(pos[i], textLen)];
		setSentForm(t[i], formBlob + formOff[i], formOff[i + 1] - formOff[i]);
	}
	std::vector<uint2> stacks(2 * (size_t)n + 2), ranges((size_t)n + 1);
	pairTokens(t.data(), (uint32_t)n, stacks.data(), stacks.data() + n + 1);
	foldSentLine(t.data(), (uint32_t)n);
	const uint32_t k = sentRanges(t.data(), (uint32_t)n, ranges.data());
	for (uint32_t i = 0; i < k; ++i) { out[2 * i] = ranges[i].x; out[2 * i + 1] = ranges[i].y; }
	return (int)k;
}

void* ss32_open(const char* imagePath)
{
	try
	{
		auto blob = kb::readImageFile(imagePath);
		auto* m = new kb::Model;
		m->load(blob.data(), blob.size());
		return m;
	}
	catch (...) { return nullptr; }
}
void ss32_close(void* p) { delete reinterpret_cast<kb::Model*>(p); }

// one document's token rows (as emit_kernel writes them) -> ranges[2 * k] from sents.cu on a simulated warp; returns k
int ss32_rows(void* p, const uint16_t* text, uint32_t textLen, int n, const uint32_t* morph, const uint8_t* tag, const uint32_t* pos, const uint16_t* len,
	const uint8_t* flags, uint32_t* out)
{
	using namespace kb;
	std::lock_guard<std::mutex> lk(g_ssMtx);
	const Model& m = *reinterpret_cast<const Model*>(p);
	set_model_sents(m.dev);
	const size_t W = 2 * (size_t)textLen + 4, npu = KB_DEFAULT_NODES_PER_UNIT;
	if ((size_t)n > W) return -1;
	const uint32_t off[2] = { 0, textLen };
	std::vector<DToken> rows(W);
	for (int i = 0; i < n; ++i) rows[i] = DToken{ morph[i], pos[i], 0.f, len[i], tag[i], flags[i] };
	std::vector<uint32_t> ctr(W), nTok(1, (uint32_t)n), status(1, 0), nSents(1, 0);
	std::vector<DNode> nodes(W * npu);
	std::vector<uint2> ranges(W);
	BatchView bv{}; VitView vv{};
	bv.n_sent = 1; bv.text = text; bv.text_off = off; bv.nodes_per_unit = (uint32_t)npu; bv.ctr = ctr.data(); bv.build_nodes = nodes.data();
	bv.end_pos_map = ranges.data(); bv.status = status.data();
	vv.tokens = rows.data(); vv.n_tokens = nTok.data();
	if (launch_sents(bv, vv, nSents.data(), nullptr)) return -1;
	for (uint32_t i = 0; i < nSents[0]; ++i) { out[2 * i] = ranges[i].x; out[2 * i + 1] = ranges[i].y; }
	return (int)nSents[0];
}

}
