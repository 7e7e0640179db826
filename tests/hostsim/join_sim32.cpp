// TEST INFRASTRUCTURE: the token-joining fold without a GPU, behind a small C API for tests/test_join.py.  One sentence through the simulated
// lattice -> Viterbi -> emit_join_kernel (lattice.cu, viterbi.cu, emit.cu compiled as C++ on 32-lane warps, tests/hostsim/shim32), with the
// match options of the call; the rows then go through the product's host assembly (kiwi_b200/csrc/assemble.h assembleRows, what
// kiwi_analyze_w reports): morpheme id (-1 for a joined token), forms and the sentence fields.
// tests/test_join.py compiles this file with the objects the build leaves in tests/hostsim/obj32.
#include <cuda_runtime.h>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <vector>
#include "../../kiwi_b200/csrc/engine.h"
#include "../../kiwi_b200/csrc/assemble.h"

namespace kb
{
	cudaError_t launch_lattice(const DevModel& m, const BatchView& bv, cudaStream_t stream);
	cudaError_t launch_viterbi(const DevModel& m, const BatchView& bv, const VitView& vv, cudaStream_t stream);
	cudaError_t launch_viterbi_cong(const DevModel& m, const BatchView& bv, const VitView& vv, cudaStream_t stream);
	cudaError_t launch_emit(const DevModel& m, const BatchView& bv, const VitView& vv, cudaStream_t stream);
	cudaError_t set_model_lattice(const DevModel& m);
	cudaError_t set_model_viterbi(const DevModel& m);
	cudaError_t set_model_viterbi_cong(const DevModel& m);
	cudaError_t set_model_emit(const DevModel& m);
}

namespace
{
	struct Sim { kb::Model model; std::vector<char> typo; };
	std::mutex g_mtx;
}

extern "C" {

void* hj32_open(const char* imagePath, const char* typoPath)
{
	try
	{
		auto blob = kb::readImageFile(imagePath);
		auto* s = new Sim;
		s->model.load(blob.data(), blob.size());
		if (typoPath)
		{
			FILE* f = std::fopen(typoPath, "rb");
			if (!f) { delete s; return nullptr; }
			std::fseek(f, 0, SEEK_END); const long n = std::ftell(f); std::fseek(f, 0, SEEK_SET);
			s->typo.resize((size_t)n);
			const bool ok = std::fread(s->typo.data(), 1, (size_t)n, f) == (size_t)n;
			std::fclose(f);
			if (!ok) { delete s; return nullptr; }
		}
		return s;
	}
	catch (...) { return nullptr; }
}
void hj32_close(void* p) { delete reinterpret_cast<Sim*>(p); }

// rows[10 * i] = {morph id or -1, tag, position, length, score bits, wordPosition, sentPosition, lineNumber, subSentPosition, pairedToken};
// token i's form is formBlob[formOff[i], formOff[i + 1]) (formCap units in all).  Returns the token count, -status on a kernel status,
// -100 on an error.
int hj32_analyze(void* p, const uint16_t* text, int len, uint32_t matchOptions, uint32_t* rows, int maxTokens, uint16_t* formBlob, uint32_t* formOff,
	int formCap, float* sentScore)
{
	try
	{
		std::lock_guard<std::mutex> lk(g_mtx);
		Sim& s = *reinterpret_cast<Sim*>(p);
		using namespace kb;
		const uint32_t off[2] = { 0, (uint32_t)len }, order[1] = { 0 };
		const size_t U = 2 * (size_t)len + 4, npu = KB_DEFAULT_NODES_PER_UNIT, ppu = 128, pc = 8192, fpu = 4;
		auto norm = std::vector<uint16_t>(U + 32); std::vector<uint32_t> normLen(1), posTable(len + 2), nsToPos(U), posToNs(U), ctr(U);
		std::vector<uint2> endPosMap(U); std::vector<DPattern> pats(U); std::vector<DNode> build(U * npu), nodes(U * npu); std::vector<uint32_t> newIndex(U * npu);
		const size_t chunkSlots = U / 4 + 10;
		std::vector<DChunk> chunks(chunkSlots); std::vector<uint32_t> nChunks(1), status(1), debug(64);
		std::vector<DPath> paths(ppu * U + pc); std::vector<uint32_t> npOff(U * npu), npCnt(U * npu); std::vector<uint2> nodeCand(U * npu); std::vector<uint8_t> reach(U * npu);
		std::vector<DRec> recs(2 * chunkSlots); std::vector<DToken> toks(U); std::vector<uint32_t> nTok(2), nF(2); std::vector<int32_t> bestRec(1); std::vector<float> sc(1);
		std::vector<unsigned long long> timing(2); std::vector<uint32_t> workCounter(4); std::vector<uint16_t> pool(U * fpu);
		BatchView bv{}; VitView vv{};
		bv.n_sent = 1; bv.text = text; bv.text_off = off; bv.match_options = matchOptions; bv.nodes_per_unit = (uint32_t)npu; bv.order = order;
		bv.norm = norm.data(); bv.norm_len = normLen.data(); bv.pos_table = posTable.data(); bv.ns_to_pos = nsToPos.data(); bv.pos_to_ns = posToNs.data();
		bv.end_pos_map = endPosMap.data(); bv.ctr = ctr.data(); bv.patterns = pats.data(); bv.build_nodes = build.data(); bv.nodes = nodes.data();
		bv.new_index = newIndex.data(); bv.chunks = chunks.data(); bv.n_chunks = nChunks.data(); bv.status = status.data(); bv.debug = debug.data();
		vv.work_counter = workCounter.data(); vv.solo_blocks = 0; vv.solo_warps = 1;
		vv.paths_per_unit = (uint32_t)ppu; vv.paths_const = (uint32_t)pc; vv.path_stride = sizeof(DPath); vv.paths = paths.data(); vv.node_path_off = npOff.data();
		vv.node_path_cnt = npCnt.data(); vv.node_cand = nodeCand.data(); vv.reachable = reach.data(); vv.recs = recs.data(); vv.tokens = toks.data();
		vv.n_tokens = nTok.data(); vv.best_rec = bestRec.data(); vv.score = sc.data(); vv.timing = timing.data();
		vv.forms = pool.data(); vv.n_forms = nF.data(); vv.forms_per_unit = (uint32_t)fpu;
		std::vector<DTypoNode> tgTmp, tg; std::vector<uint32_t> tgRemap; std::vector<uint2> tgRange; std::vector<DTypoState> tgStates; std::vector<DTypoMatch> tgMatches;
		if (!s.typo.empty())
		{
			const auto* th = reinterpret_cast<const kb2_typo_header*>(s.typo.data());
			size_t o = sizeof(kb2_typo_header);
			auto take = [&](size_t bytes) { o = (o + 15) / 16 * 16; const char* q = s.typo.data() + o; o += bytes; return q; };
			TypoView& tv = bv.typo;
			tv.nodes = reinterpret_cast<const kb2_typo_node*>(take(sizeof(kb2_typo_node) * th->n_nodes));
			tv.keys = reinterpret_cast<const uint16_t*>(take(2 * (size_t)th->n_edges));
			tv.diffs = reinterpret_cast<const int32_t*>(take(4 * (size_t)th->n_edges));
			tv.pats = reinterpret_cast<const kb2_typo_pat*>(take(sizeof(kb2_typo_pat) * th->n_pats));
			tv.repls = reinterpret_cast<const kb2_typo_repl*>(take(sizeof(kb2_typo_repl) * th->n_repls));
			tv.pool = reinterpret_cast<const uint16_t*>(take(2 * (size_t)th->n_pool));
			tv.threshold = 2.5f; tv.continual_threshold = th->continual_typo_threshold;
			tv.graph_per_unit = 6; tv.states_per_unit = 6;
			tgTmp.resize(U * 6); tg.resize(U * 6); tgRemap.resize(U * 6); tgRange.resize(U * 6); tgMatches.resize(U * 6); tgStates.resize(U * 6);
			tv.tmp = tgTmp.data(); tv.graph = tg.data(); tv.remap = tgRemap.data(); tv.state_range = tgRange.data(); tv.matches = tgMatches.data(); tv.states = tgStates.data();
		}
		const bool cong = s.model.dev.model_type == 4;
		set_model_lattice(s.model.dev); set_model_emit(s.model.dev);
		if (cong) set_model_viterbi_cong(s.model.dev); else set_model_viterbi(s.model.dev);
		if (launch_lattice(s.model.dev, bv, nullptr)) return -100;
		if (status[0]) return -(int)status[0];
		if (cong ? launch_viterbi_cong(s.model.dev, bv, vv, nullptr) : launch_viterbi(s.model.dev, bv, vv, nullptr)) return -100;
		if (status[0]) return -(int)status[0];
		if (s.model.dev.debug[0] || debug[0]) return -101;
		if (launch_emit(s.model.dev, bv, vv, nullptr)) return -100;
		if (status[0]) return -(int)status[0];
		const int n = (int)nTok[0];
		if (n > maxTokens) return -100;
		const Model& m = s.model;
		const std::vector<ResTok> rt = assembleRows(m.hMorphs, m.hForms, m.hFormChars, m.hChrBmp.data(), text, (uint32_t)len, toks.data(), (uint32_t)n,
			pool.data(), (matchOptions & MO_JOIN_ANY) ? nF[0] : 0, matchOptions);
		formOff[0] = 0;
		for (int i = 0; i < n; ++i)
		{
			uint32_t bits; std::memcpy(&bits, &toks[i].score, 4);
			const AsmTok& a = rt[i].a;
			const uint32_t r[10] = { rt[i].morphId, toks[i].tag, toks[i].position, toks[i].length, bits, a.wordPosition, a.sentPosition, a.lineNumber, a.subSentPosition, a.pairedToken };
			std::memcpy(rows + 10 * i, r, sizeof(r));
			if (formOff[i] + a.form.size() > (size_t)formCap) return -100;
			std::memcpy(formBlob + formOff[i], a.form.data(), a.form.size() * 2);
			formOff[i + 1] = formOff[i] + (uint32_t)a.form.size();
		}
		*sentScore = sc[0];
		return n;
	}
	catch (...) { return -100; }
}

}
