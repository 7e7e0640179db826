// kiwi_b200: host engine.  Owns the device-resident model, the per-batch scratch arena and the stream; turns
// one batch of raw UTF-16 sentences into flat token arrays with exactly four compute launches
// (lattice_kernel, viterbi_kernel, emit_kernel, pack_kernel) plus one cub scan.
//
// Host role (the reference does all of this per sentence on CPU threads, src/Kiwi.cpp:1014-1158 and
// include/kiwi/Kiwi.h:402-454): here the host only copies the text blob + offsets in and the packed
// tokens out; normalisation, chunking, lattice, Viterbi, stitching and position mapping run on the GPU.
// Sentences whose scratch demand exceeds the arithmetic capacity (rare, e.g. 50 x the same syllable) are
// re-run in a larger-capacity retry arena (two escalation rounds); a sentence that still does not fit keeps its
// status and comes back without tokens - the batch itself never fails on input text.
// Batches larger than one pass alternate between two arenas on two streams (H2D / kernels / D2H of neighbouring
// passes overlap); one lock per CUDA device serialises engines that share the device's constant-memory model view.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <stdexcept>
#include <string>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_radix_sort.cuh>
#include "engine.h"

namespace kb
{
	cudaError_t launch_lattice(const DevModel& m, const BatchView& bv, cudaStream_t stream);
	cudaError_t launch_viterbi(const DevModel& m, const BatchView& bv, const VitView& vv, cudaStream_t stream);
	cudaError_t launch_emit(const DevModel& m, const BatchView& bv, const VitView& vv, cudaStream_t stream);
	cudaError_t set_model_lattice(const DevModel& m);
	cudaError_t set_model_viterbi(const DevModel& m);
	cudaError_t launch_viterbi_cong(const DevModel& m, const BatchView& bv, const VitView& vv, cudaStream_t stream);
	cudaError_t set_model_viterbi_cong(const DevModel& m);
	cudaError_t launch_viterbi_sbg(const DevModel& m, const BatchView& bv, const VitView& vv, cudaStream_t stream);
	cudaError_t set_model_viterbi_sbg(const DevModel& m);
	cudaError_t launch_cong_debug(uint32_t n, const uint32_t* ctx, const uint32_t* wid, const int32_t* node,
		int32_t* outDot, float* outEps, int32_t* outNode, uint32_t* outCtx, int32_t* outTile, cudaStream_t stream);
	cudaError_t set_model_emit(const DevModel& m);
	cudaError_t launch_sents(const BatchView& bv, const VitView& vv, uint32_t* nSents, cudaStream_t stream);
	cudaError_t launch_sents_pack(const BatchView& bv, const uint32_t* nSents, const uint32_t* sentOff, uint32_t* begin, uint32_t* end, cudaStream_t stream);
	cudaError_t set_model_sents(const DevModel& m);

	static void ck(cudaError_t e, const char* what)
	{
		if (e != cudaSuccess) throw std::runtime_error(std::string("CUDA error in ") + what + ": " + cudaGetErrorString(e));
	}

	static constexpr uint32_t DEFAULT_PATHS_PER_UNIT = 128, DEFAULT_PATHS_CONST = 8192;
#ifndef KB_DEFAULT_SOLO_BLOCKS
#define KB_DEFAULT_SOLO_BLOCKS 0
#define KB_DEFAULT_SOLO_WARPS 1
#endif
#ifndef KB_DEFAULT_TEAM_PERMILLE
#define KB_DEFAULT_TEAM_PERMILLE 0
#endif
	static uint32_t teamPermille();
	static std::pair<uint32_t, uint32_t> soloConfig();
	// typo graph nodes / search states per normalised-unit slot (W_s = 2 n + 4 slots per sentence): the basic typo set needs < 4
	// on the reference's evaluation texts (tests/test_hostsim_lattice.py); overflow -> ST_TYPO_OVERFLOW -> retry arena
	static constexpr uint32_t DEFAULT_TYPO_GRAPH_PER_UNIT = 6, DEFAULT_TYPO_STATES_PER_UNIT = 6;

	__global__ void length_kernel(uint32_t nSent, const uint32_t* __restrict__ textOff, uint32_t* __restrict__ keys, uint32_t* __restrict__ idx)
	{
		const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
		if (s >= nSent) return;
		keys[s] = textOff[s + 1] - textOff[s];
		idx[s] = s;
	}

	// predicted Viterbi cost of a sentence = sum over its lattice nodes of (candidate count)^2: the launch order of the Viterbi kernel
	// (heaviest first) and the choice of the sentences that get a team of warps.  Measured on the bench batch against the oracle's work
	// counters: correlation 0.92 with the LM-step count (sentence length: 0.87); the top 20 % by this key hold 91 % of the heaviest 5 %.
	__global__ void cost_kernel(BatchView bv, const DForm* __restrict__ forms, uint32_t* __restrict__ keys, uint32_t* __restrict__ idx)
	{
		const uint32_t lane = threadIdx.x & 31;
		const uint32_t s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
		if (s >= bv.n_sent) return;
		unsigned long long cost = 0;
		if (!bv.status[s])
		{
			const size_t wbase = 2 * (size_t)bv.text_off[s] + 4 * (size_t)s;
			const size_t nbase = (size_t)bv.nodes_per_unit * wbase;
			const DChunk* chunks = bv.chunks + (wbase >> 2) + 2 * (size_t)s;
			const uint32_t nChunks = bv.n_chunks[s];
			for (uint32_t c = 0; c < nChunks; ++c)
			{
				const DChunk ch = chunks[c];
				const DNode* nodes = bv.nodes + nbase + ch.node_off;
				for (uint32_t j = 1 + lane; j + 1 < ch.n_nodes; j += 32)
				{
					const int32_t fm = nodes[j].form;
					const unsigned long long k = fm >= 0 ? forms[fm].cand_cnt : 2u;
					cost += k * k;
				}
			}
		}
		for (int d = 16; d; d >>= 1) cost += __shfl_xor_sync(0xFFFFFFFFu, cost, d);
		if (lane == 0) { keys[s] = cost > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)cost; idx[s] = s; }
	}

	__global__ void pack_kernel(uint32_t nSent, const uint32_t* __restrict__ textOff, const uint32_t* __restrict__ nTokens,
		const uint32_t* __restrict__ tokOff, const DToken* __restrict__ tokens, DToken* __restrict__ packed)
	{
		const uint32_t lane = threadIdx.x & 31;
		const uint32_t s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
		if (s >= nSent) return;
		const size_t wbase = 2 * (size_t)textOff[s] + 4 * (size_t)s;
		const uint32_t n = nTokens[s], o = tokOff[s];
		for (uint32_t i = lane; i < n; i += 32) packed[o + i] = tokens[wbase + i];
	}

	// token-joining options: the joined forms of every sentence to their place in the packed form array, and the flagged rows' entry offsets
	// from sentence-relative to array-relative
	__global__ void join_pack_kernel(uint32_t nSent, const uint32_t* __restrict__ textOff, uint32_t formsPerUnit, const uint16_t* __restrict__ pools,
		const uint32_t* __restrict__ nForms, const uint32_t* __restrict__ formOff, const uint32_t* __restrict__ nTokens, const uint32_t* __restrict__ tokOff,
		DToken* __restrict__ packed, uint16_t* __restrict__ packedForms)
	{
		const uint32_t lane = threadIdx.x & 31;
		const uint32_t s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
		if (s >= nSent) return;
		const size_t fbase = (size_t)formsPerUnit * (2 * (size_t)textOff[s] + 4 * (size_t)s);
		const uint32_t nf = nForms[s], fo = formOff[s];
		for (uint32_t i = lane; i < nf; i += 32) packedForms[fo + i] = pools[fbase + i];
		if (!fo) return;
		const uint32_t nt = nTokens[s], to = tokOff[s];
		for (uint32_t i = lane; i < nt; i += 32) if (packed[to + i].morph & JOINED_TOKEN) packed[to + i].morph += fo;
	}

	// adds `base` to the entry offset of every joined row (the forms of a later pass are appended behind the earlier passes' forms)
	__global__ void rebase_joined_kernel(uint32_t n, uint32_t base, DToken* __restrict__ rows)
	{
		const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
		if (i < n && (rows[i].morph & JOINED_TOKEN)) rows[i].morph += base;
	}

	// ---- per-device state: one lock and one owner of the kernels' __constant__ model view per CUDA device --------------
	namespace
	{
		// (sentsOwner: the model view of the sentence kernel, uploaded by the first split only)
		struct DevState { std::recursive_mutex mtx; const Model* owner = nullptr; const Model* sentsOwner = nullptr; };
		DevState g_devState[64];
	}
	DeviceGuard::DeviceGuard(int device) : dev{ device < 0 || device >= 64 ? 0 : device }
	{
		g_devState[dev].mtx.lock();
		if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
		if (prev != dev) cudaSetDevice(dev);
	}
	DeviceGuard::~DeviceGuard()
	{
		if (prev >= 0 && prev != dev) cudaSetDevice(prev);
		g_devState[dev].mtx.unlock();
	}

	Engine::Engine(const void* imageBytes, size_t size)
	{
		ck(cudaGetDevice(&device), "cudaGetDevice");
		DeviceGuard g{ device };
		model.load(imageBytes, size);
		// (the constant-memory model view is uploaded by the first launch: uploading here would overwrite the view of another
		// engine on this device without it noticing)
		for (auto& sl : slot_)
		{
			ck(cudaStreamCreateWithFlags(&sl.stream, cudaStreamNonBlocking), "cudaStreamCreate");
			for (auto& e : sl.ev) ck(cudaEventCreate(&e), "cudaEventCreate");
			for (auto& e : sl.evSents) ck(cudaEventCreate(&e), "cudaEventCreate");
		}
		stream = slot_[0].stream;
	}

	Engine::~Engine()
	{
		DeviceGuard g{ device };
		if (g_devState[g.dev].owner == &model) g_devState[g.dev].owner = nullptr;
		if (g_devState[g.dev].sentsOwner == &model) g_devState[g.dev].sentsOwner = nullptr;
		for (auto& sl : slot_)
		{
			freeScratch(sl.sc);
			if (sl.hPinText) cudaFreeHost(sl.hPinText);
			if (sl.hPinOff) cudaFreeHost(sl.hPinOff);
			if (sl.hPinOut) cudaFreeHost(sl.hPinOut);
			for (auto& e : sl.ev) if (e) cudaEventDestroy(e);
			for (auto& e : sl.evSents) if (e) cudaEventDestroy(e);
			if (sl.stream) cudaStreamDestroy(sl.stream);
		}
		freeScratch(retry_);
	}

	void Engine::freeScratch(Scratch& sc)
	{
		for (void* p : sc.bufs) cudaFree(p);
		for (void* p : sc.typoBufs) cudaFree(p);
		for (void* p : sc.sentBufs) cudaFree(p);
		for (void* p : sc.joinBufs) cudaFree(p);
		sc = Scratch{};
	}

	// ---- typo lattice: the device-resident transformer and the per-sentence graph / state scratch ----------------
	void TypoDev::load(const void* bytes, size_t size)
	{
		if (size < sizeof(kb2_typo_header)) throw std::runtime_error("typo image: too small");
		blob.assign(reinterpret_cast<const char*>(bytes), reinterpret_cast<const char*>(bytes) + size);
		const auto* h = reinterpret_cast<const kb2_typo_header*>(blob.data());
		if (h->magic != KB2_TYPO_MAGIC) throw std::runtime_error("typo image: bad magic");
		size_t o = sizeof(kb2_typo_header);
		auto take = [&](size_t bytesOf) { o = (o + 15) / 16 * 16; const size_t at = o; o += bytesOf; return at; };
		const size_t oNodes = take(sizeof(kb2_typo_node) * h->n_nodes), oKeys = take(2 * (size_t)h->n_edges), oDiffs = take(4 * (size_t)h->n_edges);
		const size_t oPats = take(sizeof(kb2_typo_pat) * h->n_pats), oRepls = take(sizeof(kb2_typo_repl) * h->n_repls), oPool = take(2 * (size_t)h->n_pool);
		if (o > size) throw std::runtime_error("typo image: truncated");
		if (std::isfinite(h->lengthening_typo_threshold)) throw std::runtime_error("typo image: lengthening typo sets are outside the kiwi_b200 hot path");
		ck(cudaMalloc(&dBlob, size), "cudaMalloc(typo image)");
		ck(cudaMemcpy(dBlob, blob.data(), size, cudaMemcpyHostToDevice), "cudaMemcpy(typo image)");
		const char* d = reinterpret_cast<const char*>(dBlob);
		view = TypoView{};
		view.nodes = reinterpret_cast<const kb2_typo_node*>(d + oNodes); view.keys = reinterpret_cast<const uint16_t*>(d + oKeys);
		view.diffs = reinterpret_cast<const int32_t*>(d + oDiffs); view.pats = reinterpret_cast<const kb2_typo_pat*>(d + oPats);
		view.repls = reinterpret_cast<const kb2_typo_repl*>(d + oRepls); view.pool = reinterpret_cast<const uint16_t*>(d + oPool);
		view.continual_threshold = h->continual_typo_threshold;
	}

	TypoDev::~TypoDev() { if (dBlob) cudaFree(dBlob); }

	void Engine::ensureTypoScratch(Scratch& sc, uint32_t gpu0, uint32_t spu0, uint32_t mul)
	{
		const uint32_t gpu = gpu0 * mul, spu = spu0 * mul;
		if (sc.typoCapUnits >= sc.capUnits && sc.typoGraphPerUnit == gpu && sc.typoStatesPerUnit == spu) return;
		for (void* p : sc.typoBufs) cudaFree(p);
		sc.typoBufs.clear();
		auto alloc = [&](size_t bytes) { void* p = nullptr; ck(cudaMalloc(&p, std::max<size_t>(bytes, 256)), "cudaMalloc(typo scratch)"); sc.typoBufs.push_back(p); return p; };
		const size_t G = sc.capUnits * gpu, S = sc.capUnits * spu;
		TypoView& t = sc.typoScratch;
		t = TypoView{};
		t.graph_per_unit = gpu; t.states_per_unit = spu;
		t.tmp = (DTypoNode*)alloc(G * sizeof(DTypoNode)); t.graph = (DTypoNode*)alloc(G * sizeof(DTypoNode));
		t.remap = (uint32_t*)alloc(G * 4); t.state_range = (uint2*)alloc(G * 8); t.matches = (DTypoMatch*)alloc(G * sizeof(DTypoMatch));
		t.states = (DTypoState*)alloc(S * sizeof(DTypoState));
		sc.typoCapUnits = sc.capUnits; sc.typoGraphPerUnit = gpu; sc.typoStatesPerUnit = spu;
	}

	void Engine::ensureScratch(Scratch& sc, cudaStream_t st, size_t U, size_t B, uint32_t ppu, uint32_t pc, uint32_t npu)
	{
		const size_t T = (U - 4 * B) / 2 + 1;
		if (U <= sc.capUnits && B <= sc.capSent && ppu == sc.pathsPerUnit && pc == sc.pathsConst && npu == sc.nodesPerUnit && T <= sc.capText) return;
		const size_t capU = std::max(U, sc.capUnits), capB = std::max(B, sc.capSent), capT = std::max(T, sc.capText);
		freeScratch(sc);
		auto alloc = [&](size_t bytes) { void* p = nullptr; ck(cudaMalloc(&p, std::max<size_t>(bytes, 256)), "cudaMalloc(scratch)"); sc.bufs.push_back(p); return p; };
		BatchView& bv = sc.bv; VitView& vv = sc.vv;
		bv.nodes_per_unit = npu;
		bv.norm = (uint16_t*)alloc(capU * 2 + 64);
		bv.norm_len = (uint32_t*)alloc(capB * 4);
		bv.pos_table = (uint32_t*)alloc((capT + capB + 1) * 4);
		bv.ns_to_pos = (uint32_t*)alloc(capU * 4);
		bv.pos_to_ns = (uint32_t*)alloc(capU * 4);
		bv.end_pos_map = (uint2*)alloc(capU * 8);
		bv.ctr = (uint32_t*)alloc(capU * 4);
		bv.patterns = (DPattern*)alloc(capU * sizeof(DPattern));
		bv.build_nodes = (DNode*)alloc(capU * npu * sizeof(DNode));
		bv.nodes = (DNode*)alloc(capU * npu * sizeof(DNode));
		bv.new_index = (uint32_t*)alloc(capU * npu * 4);
		const size_t chunkSlots = capU / 4 + 2 * capB + 8;
		bv.chunks = (DChunk*)alloc(chunkSlots * sizeof(DChunk));
		bv.n_chunks = (uint32_t*)alloc(capB * 4);
		bv.status = (uint32_t*)alloc(capB * 4);
		bv.debug = (uint32_t*)alloc(64 * 4);
		ck(cudaMemset(bv.debug, 0, 64 * 4), "memset");
		vv.paths_per_unit = ppu; vv.paths_const = pc;
		vv.path_stride = pathStride();
		vv.paths = (DPath*)alloc(((size_t)ppu * capU + (size_t)pc * capB) * vv.path_stride);
		vv.node_path_off = (uint32_t*)alloc(capU * npu * 4);
		vv.node_path_cnt = (uint32_t*)alloc(capU * npu * 4);
		vv.node_cand = (uint2*)alloc(capU * npu * 8);
		vv.reachable = (uint8_t*)alloc(capU * npu);
		vv.recs = (DRec*)alloc(2 * chunkSlots * sizeof(DRec));
		vv.tokens = (DToken*)alloc(capU * sizeof(DToken));
		vv.n_tokens = (uint32_t*)alloc((capB + 1) * 4);
		vv.best_rec = (int32_t*)alloc(capB * 4);
		vv.score = (float*)alloc(capB * 4);
		vv.timing = (unsigned long long*)alloc(capB * 16);
		vv.work_counter = (uint32_t*)alloc(16);
		sc.tokOff = (uint32_t*)alloc((capB + 1) * 4);
		sc.packed = (DToken*)alloc(capU * sizeof(DToken));
		sc.dText = (uint16_t*)alloc(capT * 2 + 64);
		sc.dOff = (uint32_t*)alloc((capB + 1) * 4);
		size_t tb = 0;
		cub::DeviceScan::ExclusiveSum(nullptr, tb, vv.n_tokens, sc.tokOff, (int)(capB + 1), st);
		sc.cubTempBytes = tb; sc.cubTemp = alloc(tb);
		sc.lenKeys = (uint32_t*)alloc(capB * 4); sc.lenKeysOut = (uint32_t*)alloc(capB * 4); sc.idxIn = (uint32_t*)alloc(capB * 4); sc.order = (uint32_t*)alloc(capB * 4); sc.orderVit = (uint32_t*)alloc(capB * 4);
		size_t sb = 0;
		cub::DeviceRadixSort::SortPairsDescending(nullptr, sb, sc.lenKeys, sc.lenKeysOut, sc.idxIn, sc.order, (int)capB, 0, 32, st);
		sc.sortTempBytes = sb; sc.sortTemp = alloc(sb);
		sc.capUnits = capU; sc.capSent = capB; sc.capText = capT; sc.pathsPerUnit = ppu; sc.pathsConst = pc; sc.nodesPerUnit = npu;
	}

	// form pool units per normalised-unit slot: a joined form is at most 3 units per unit of its components' sources plus a 3-unit entry frame;
	// overflow -> ST_TOKEN_OVERFLOW -> retry arena, which carries capMul x the pool like its node capacity
	static constexpr uint32_t DEFAULT_FORMS_PER_UNIT = 4;

	void Engine::ensureJoinScratch(Scratch& sc, uint32_t perUnit)
	{
		if (sc.joinCapUnits < sc.capUnits || sc.joinCapSent < sc.capSent || sc.joinPerUnit != perUnit)
		{
			for (void* p : sc.joinBufs) cudaFree(p);
			sc.joinBufs.clear();
			auto alloc = [&](size_t bytes) { void* p = nullptr; ck(cudaMalloc(&p, std::max<size_t>(bytes, 256)), "cudaMalloc(join scratch)"); sc.joinBufs.push_back(p); return p; };
			const size_t units = sc.capUnits * perUnit;
			sc.vv.forms = (uint16_t*)alloc(units * 2); sc.vv.n_forms = (uint32_t*)alloc((sc.capSent + 1) * 4);
			sc.formOff = (uint32_t*)alloc((sc.capSent + 1) * 4); sc.packedForms = (uint16_t*)alloc(units * 2);
			sc.joinCapUnits = sc.capUnits; sc.joinCapSent = sc.capSent; sc.joinPerUnit = perUnit;
		}
		sc.vv.forms = (uint16_t*)sc.joinBufs[0]; sc.vv.n_forms = (uint32_t*)sc.joinBufs[1]; sc.vv.forms_per_unit = perUnit;
	}

	void Engine::bind(Scratch& sc, const uint16_t* dText, const uint32_t* dOffsets, uint32_t n, uint32_t matchOptions, uint32_t capMul)
	{
		sc.bv.n_sent = n; sc.bv.text = dText; sc.bv.text_off = dOffsets; sc.bv.match_options = matchOptions;
		if (matchOptions & MO_JOIN_ANY) ensureJoinScratch(sc, DEFAULT_FORMS_PER_UNIT * capMul);
		else { sc.vv.forms = nullptr; sc.vv.n_forms = nullptr; sc.vv.forms_per_unit = 0; }
		sc.bv.typo = TypoView{};
		if (typo_)
		{
			// a retry arena carries capMul x the graph / state capacity, like its node capacity
			ensureTypoScratch(sc, DEFAULT_TYPO_GRAPH_PER_UNIT, DEFAULT_TYPO_STATES_PER_UNIT, capMul);
			TypoView v = sc.typoScratch;
			v.nodes = typo_->view.nodes; v.keys = typo_->view.keys; v.diffs = typo_->view.diffs; v.pats = typo_->view.pats; v.repls = typo_->view.repls; v.pool = typo_->view.pool;
			v.continual_threshold = typo_->view.continual_threshold; v.threshold = typoThreshold_;
			sc.bv.typo = v;
		}
	}

	// caller holds the device lock and no kernel of another engine is in flight on this device (every public entry point
	// synchronises its streams before it releases the lock)
	void Engine::uploadConstants()
	{
		DevState& ds = g_devState[device < 0 || device >= 64 ? 0 : device];
		if (ds.owner == &model) return;
		DevModel vm = model.dev;
		if (candsOverride_) vm.cands = candsOverride_;      // (AnalyzeOption::blocklist: only the Viterbi kernels read the candidate table)
		ck(set_model_lattice(model.dev), "constant upload"); ck(model.dev.model_type == 4 ? set_model_viterbi_cong(vm) : model.dev.model_type == 3 ? set_model_viterbi_sbg(vm) : set_model_viterbi(vm), "constant upload"); ck(set_model_emit(model.dev), "constant upload");
		ds.owner = &model;
	}

	void Engine::setCandsOverride(const DCand* deviceTable)
	{
		if (deviceTable == candsOverride_) return;
		DeviceGuard g{ device };
		for (auto& sl : slot_) if (sl.stream) cudaStreamSynchronize(sl.stream);      // (no kernel of this engine may still read the old table)
		candsOverride_ = deviceTable;
		g_devState[device < 0 || device >= 64 ? 0 : device].owner = nullptr;      // the next launch uploads the model view again
	}

	void Engine::launchAll(Scratch& sc, cudaStream_t st, cudaEvent_t* ev, uint32_t n)
	{
		uploadConstants();
		ck(cudaEventRecord(ev[1], st), "event");
		// longest-processing-time-first launch order (sentence cost grows with its length)
		length_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, sc.bv.text_off, sc.lenKeys, sc.idxIn);
		ck(cudaGetLastError(), "length_kernel launch");
		size_t sb = sc.sortTempBytes;
		ck(cub::DeviceRadixSort::SortPairsDescending(sc.sortTemp, sb, sc.lenKeys, sc.lenKeysOut, sc.idxIn, sc.order, (int)n, 0, 32, st), "cub sort");
		sc.bv.order = sc.order;
		ck(launch_lattice(model.dev, sc.bv, st), "lattice_kernel launch");
		// Viterbi launch order: heaviest predicted sentence first; the first n_team of them get a team of warps each
		{
			const uint32_t threads = 256, blocks = (n * 32 + threads - 1) / threads;
			cost_kernel<<<blocks, threads, 0, st>>>(sc.bv, model.dev.forms, sc.lenKeys, sc.idxIn);
			ck(cudaGetLastError(), "cost_kernel launch");
			size_t sb2 = sc.sortTempBytes;
			ck(cub::DeviceRadixSort::SortPairsDescending(sc.sortTemp, sb2, sc.lenKeys, sc.lenKeysOut, sc.idxIn, sc.orderVit, (int)n, 0, 32, st), "cub sort");
			static const bool byLength = [] { const char* e = std::getenv("KIWI_B200_LPT"); return e && std::string(e) == "len"; }();      // experiments: keep the length order
			if (!byLength) sc.bv.order = sc.orderVit;
			sc.vv.n_team = (uint32_t)((unsigned long long)n * teamPermille() / 1000);
			sc.vv.solo_blocks = soloConfig().first; sc.vv.solo_warps = soloConfig().second;
		}
		ck(cudaEventRecord(ev[2], st), "event");
		ck(model.dev.model_type == 4 ? launch_viterbi_cong(model.dev, sc.bv, sc.vv, st) : model.dev.model_type == 3 ? launch_viterbi_sbg(model.dev, sc.bv, sc.vv, st) : launch_viterbi(model.dev, sc.bv, sc.vv, st), "viterbi_kernel launch");
		ck(cudaEventRecord(ev[3], st), "event");
		ck(launch_emit(model.dev, sc.bv, sc.vv, st), "emit_kernel launch");
		ck(cudaMemsetAsync(sc.vv.n_tokens + n, 0, 4, st), "memset");
		size_t tb = sc.cubTempBytes;
		ck(cub::DeviceScan::ExclusiveSum(sc.cubTemp, tb, sc.vv.n_tokens, sc.tokOff, (int)(n + 1), st), "cub scan");
		const uint32_t threads = 256, blocks = (n * 32 + threads - 1) / threads;
		pack_kernel<<<blocks, threads, 0, st>>>(n, sc.bv.text_off, sc.vv.n_tokens, sc.tokOff, sc.vv.tokens, sc.packed);
		ck(cudaGetLastError(), "pack_kernel launch");
		if (sc.bv.match_options & MO_JOIN_ANY)
		{
			ck(cudaMemsetAsync(sc.vv.n_forms + n, 0, 4, st), "memset");
			size_t tb2 = sc.cubTempBytes;
			ck(cub::DeviceScan::ExclusiveSum(sc.cubTemp, tb2, sc.vv.n_forms, sc.formOff, (int)(n + 1), st), "cub scan");
			join_pack_kernel<<<blocks, threads, 0, st>>>(n, sc.bv.text_off, sc.vv.forms_per_unit, sc.vv.forms, sc.vv.n_forms, sc.formOff, sc.vv.n_tokens, sc.tokOff, sc.packed, sc.packedForms);
			ck(cudaGetLastError(), "join_pack_kernel launch");
			last.kernelLaunches += 2;
		}
		ck(cudaEventRecord(ev[4], st), "event");
		last.kernelLaunches += 6;
	}

	// CUDA-event times of the launch whose events launchAll recorded into ev[1..4]
	struct KernelMs { float lattice = 0, viterbi = 0, pack = 0, total = 0; };
	static KernelMs kernelMs(const cudaEvent_t* ev)
	{
		KernelMs t;
		cudaEventElapsedTime(&t.lattice, ev[1], ev[2]);
		cudaEventElapsedTime(&t.viterbi, ev[2], ev[3]);
		cudaEventElapsedTime(&t.pack, ev[3], ev[4]);
		cudaEventElapsedTime(&t.total, ev[1], ev[4]);
		return t;
	}

	// ---- sentence ranges (Kiwi::splitIntoSents): sents_kernel over the unpacked token rows, then a scan and a pack like the tokens' ----
	void Engine::ensureSentScratch(Scratch& sc)
	{
		if (sc.sentCapUnits >= sc.capUnits && sc.sentCapSent >= sc.capSent) return;
		for (void* p : sc.sentBufs) cudaFree(p);
		sc.sentBufs.clear();
		auto alloc = [&](size_t bytes) { void* p = nullptr; ck(cudaMalloc(&p, std::max<size_t>(bytes, 256)), "cudaMalloc(sentence scratch)"); sc.sentBufs.push_back(p); return (uint32_t*)p; };
		// (a document has at most as many sentences as tokens, and at most W_s tokens: the packed ranges fit capUnits)
		sc.nSents = alloc((sc.capSent + 1) * 4); sc.sentOff = alloc((sc.capSent + 1) * 4);
		sc.sentBegin = alloc(sc.capUnits * 4); sc.sentEnd = alloc(sc.capUnits * 4);
		sc.sentCapUnits = sc.capUnits; sc.sentCapSent = sc.capSent;
	}

	// after launchAll on the same stream (ensureSentScratch first)
	void Engine::launchSents(Scratch& sc, cudaStream_t st, cudaEvent_t* evSents, uint32_t n)
	{
		DevState& ds = g_devState[device < 0 || device >= 64 ? 0 : device];
		if (ds.sentsOwner != &model) { ck(set_model_sents(model.dev), "constant upload"); ds.sentsOwner = &model; }
		ck(cudaEventRecord(evSents[0], st), "event");
		ck(launch_sents(sc.bv, sc.vv, sc.nSents, st), "sents_kernel launch");
		ck(cudaMemsetAsync(sc.nSents + n, 0, 4, st), "memset");
		size_t tb = sc.cubTempBytes;
		ck(cub::DeviceScan::ExclusiveSum(sc.cubTemp, tb, sc.nSents, sc.sentOff, (int)(n + 1), st), "cub scan");
		ck(launch_sents_pack(sc.bv, sc.nSents, sc.sentOff, sc.sentBegin, sc.sentEnd, st), "sents_pack_kernel launch");
		ck(cudaEventRecord(evSents[1], st), "event");
		last.kernelLaunches += 3;
	}

	// appends the ranges of the n sentences of a finished launch (hSentOff: its sentOff scan, on the host) to `out`; its kernel time counts
	// as msSents, the copy as D2H
	void Engine::copySents(Scratch& sc, cudaStream_t st, cudaEvent_t* evSents, uint32_t n, const uint32_t* hSentOff, BatchOutput& out)
	{
		const size_t base = out.sentBegin.size(), total = hSentOff[n];
		out.sentBegin.resize(base + total); out.sentEnd.resize(base + total);
		ck(cudaEventRecord(evSents[2], st), "event");
		if (total)
		{
			ck(cudaMemcpyAsync(out.sentBegin.data() + base, sc.sentBegin, total * 4, cudaMemcpyDeviceToHost, st), "D2H sentence ranges");
			ck(cudaMemcpyAsync(out.sentEnd.data() + base, sc.sentEnd, total * 4, cudaMemcpyDeviceToHost, st), "D2H sentence ranges");
		}
		ck(cudaEventRecord(evSents[3], st), "event");
		ck(cudaEventSynchronize(evSents[3]), "sync (sentence ranges)");
		for (uint32_t k = 1; k <= n; ++k) out.sentOff.push_back((uint32_t)(base + hSentOff[k]));
		float ms = 0;
		cudaEventElapsedTime(&ms, evSents[0], evSents[1]); out.msSents += ms;
		cudaEventElapsedTime(&ms, evSents[2], evSents[3]); out.msD2H += ms; out.msTotal += ms;
		last.d2hBytes += total * 8;
	}

	// appends the packed forms of a finished launch of n sentences (nForms units, the total of its formOff scan) to `out.forms`, and moves the
	// entry offsets of its joined rows, out.tokens[tokBegin, end), behind the forms already there
	void Engine::copyForms(Scratch& sc, uint32_t nForms, size_t tokBegin, BatchOutput& out)
	{
		const size_t base = out.forms.size();
		out.forms.resize(base + nForms);
		if (nForms) ck(cudaMemcpy(out.forms.data() + base, sc.packedForms, (size_t)nForms * 2, cudaMemcpyDeviceToHost), "D2H joined forms");
		if (base) for (size_t t = tokBegin; t < out.tokens.size(); ++t) if (out.tokens[t].morph & JOINED_TOKEN) out.tokens[t].morph += (uint32_t)base;
		last.d2hBytes += (size_t)nForms * 2;
	}

	// KIWI_B200_SOLO=<blocks>,<warps> (work-queue kernel build): the first <blocks> blocks of the Viterbi wave keep only <warps> warps,
	// which start with the heaviest sentences of the launch order
	static std::pair<uint32_t, uint32_t> soloConfig()
	{
		static const std::pair<uint32_t, uint32_t> v = []
		{
			unsigned b = KB_DEFAULT_SOLO_BLOCKS, w = KB_DEFAULT_SOLO_WARPS;
			if (const char* e = std::getenv("KIWI_B200_SOLO")) { if (std::sscanf(e, "%u,%u", &b, &w) != 2) { b = KB_DEFAULT_SOLO_BLOCKS; w = KB_DEFAULT_SOLO_WARPS; } }
			return std::make_pair((uint32_t)std::min(b, 64u), (uint32_t)std::min(w, 32u));
		}();
		return v;
	}

	// KIWI_B200_TEAM_PERMILLE: share (in 1/1000) of a pass's sentences, heaviest first, that are analysed by a team of warps
	static uint32_t teamPermille()
	{
		static const uint32_t v = [] { const char* e = std::getenv("KIWI_B200_TEAM_PERMILLE"); const long x = e ? std::atol(e) : KB_DEFAULT_TEAM_PERMILLE; return (uint32_t)std::min<long>(std::max<long>(x, 0), 1000); }();
		return v;
	}

	static void growPinned(void** p, size_t* cap, size_t bytes)
	{
		if (bytes <= *cap) return;
		if (*p) cudaFreeHost(*p);
		const size_t nb = std::max(bytes, *cap * 2);
		ck(cudaMallocHost(p, nb), "cudaMallocHost");
		*cap = nb;
	}

	void Engine::checkDebug(Scratch& sc)
	{
		uint32_t dbg[16];
		ck(cudaMemcpy(dbg, sc.bv.debug, sizeof(dbg), cudaMemcpyDeviceToHost), "D2H debug");
		if (!dbg[0]) ck(cudaMemcpy(dbg, model.dev.debug, sizeof(dbg), cudaMemcpyDeviceToHost), "D2H debug");
		if (dbg[0])
		{
			std::string msg = "internal consistency failure in viterbi_kernel:";
			for (int i = 1; i < 16; ++i) msg += " " + std::to_string(dbg[i]);
			throw std::runtime_error(msg);
		}
	}

	// Layout of a slot's pinned head buffer: [tokOff n+1][scores n][status n][debug flag 2 words], + [sentOff n+1] with OUT_SENTS.  The packed tokens go straight into
	// the caller's (page-locked) result array:
	//  - the FIRST pass of a call knows where its tokens start (offset 0), so an ESTIMATE of them (5/8 token per raw UTF-16 unit + 8 per
	//    sentence; web text needs ~0.55) is enqueued behind the kernels together with the head - a single-pass call needs one stream
	//    synchronisation and no host copy; finishPass fetches the rest when the estimate was too small;
	//  - a later pass starts where its predecessor ends, which is known only when that one has finished: finishPass enqueues its token
	//    copy then and does not wait for it (drainTokenCopies at the end of the call, or before the array has to grow).
	static size_t tokenEstimate(size_t rawUnits, uint32_t n) { return rawUnits * 5 / 8 + 8 * (size_t)n + 64; }

	// End of the pass that starts at sentence i0 of the batch offsets[0..n]: sentences (W_s = 2 n_s + 4 units each) are added while
	// fits(units, sentences) holds for the pass with them; the first one is always taken.
	template<class Fits> static uint32_t passEnd(const uint32_t* offsets, uint32_t i0, uint32_t n, Fits fits)
	{
		uint32_t i1 = i0;
		for (size_t units = 0; i1 < n; ++i1)
		{
			const size_t u = 2 * (size_t)(offsets[i1 + 1] - offsets[i1]) + 4;
			if (i1 > i0 && !fits(units + u, (size_t)(i1 - i0) + 1)) break;
			units += u;
		}
		return i1;
	}

	// a sentence that overflowed an arena may fit a larger one; a chunk beyond the 16-bit node index (ST_TOO_LONG) fits none
	static bool retryable(uint32_t status) { return status && status != ST_TOO_LONG; }

	void Engine::submitPass(Slot& s, const uint16_t* text, const uint32_t* off, uint32_t i0, uint32_t pn, uint32_t matchOptions, DToken* directDst, uint32_t outputs)
	{
		const size_t t0 = off[i0], pT = off[i0 + pn] - t0;
		const size_t U = 2 * pT + 4 * (size_t)pn;
		ensureScratch(s.sc, s.stream, U, pn, DEFAULT_PATHS_PER_UNIT * pathScale(), DEFAULT_PATHS_CONST * pathScale(), KB_DEFAULT_NODES_PER_UNIT);
		growPinned((void**)&s.hPinText, &s.pinTextCap, pT * 2 + 64);
		growPinned((void**)&s.hPinOff, &s.pinOffCap, ((size_t)pn + 1) * 4);
		std::memcpy(s.hPinText, text + t0, pT * 2);
		for (uint32_t k = 0; k <= pn; ++k) s.hPinOff[k] = off[i0 + k] - (uint32_t)t0;
		ck(cudaEventRecord(s.ev[0], s.stream), "event");
		ck(cudaMemcpyAsync(s.sc.dText, s.hPinText, pT * 2, cudaMemcpyHostToDevice, s.stream), "H2D text");
		ck(cudaMemcpyAsync(s.sc.dOff, s.hPinOff, ((size_t)pn + 1) * 4, cudaMemcpyHostToDevice, s.stream), "H2D offsets");
		bind(s.sc, s.sc.dText, s.sc.dOff, pn, matchOptions, 1);
		const bool sents = (outputs & OUT_SENTS) != 0;
		if (sents) ensureSentScratch(s.sc);
		launchAll(s.sc, s.stream, s.ev, pn);
		if (sents) launchSents(s.sc, s.stream, s.evSents, pn);
		const bool join = (matchOptions & MO_JOIN_ANY) != 0;
		const size_t headWords = ((size_t)pn + 1) + 2 * (size_t)pn + 2 + (sents ? (size_t)pn + 1 : 0) + (join ? 1 : 0);
		const size_t est = directDst ? std::min(tokenEstimate(pT, pn), (size_t)U) : 0;
		growPinned(&s.hPinOut, &s.pinOutCap, headWords * 4 + 16);
		uint32_t* hTokOff = (uint32_t*)s.hPinOut; float* hScore = (float*)(hTokOff + pn + 1); uint32_t* hStatus = (uint32_t*)(hScore + pn); uint32_t* hDbg = hStatus + pn;
		ck(cudaMemcpyAsync(hTokOff, s.sc.tokOff, ((size_t)pn + 1) * 4, cudaMemcpyDeviceToHost, s.stream), "D2H offsets");
		ck(cudaMemcpyAsync(hScore, s.sc.vv.score, (size_t)pn * 4, cudaMemcpyDeviceToHost, s.stream), "D2H scores");
		ck(cudaMemcpyAsync(hStatus, s.sc.bv.status, (size_t)pn * 4, cudaMemcpyDeviceToHost, s.stream), "D2H status");
		ck(cudaMemcpyAsync(hDbg, s.sc.bv.debug, 4, cudaMemcpyDeviceToHost, s.stream), "D2H debug");
		ck(cudaMemcpyAsync(hDbg + 1, model.dev.debug, 4, cudaMemcpyDeviceToHost, s.stream), "D2H debug");
		if (sents) ck(cudaMemcpyAsync(hDbg + 2, s.sc.sentOff, ((size_t)pn + 1) * 4, cudaMemcpyDeviceToHost, s.stream), "D2H sentence offsets");
		if (join) ck(cudaMemcpyAsync(hDbg + 2 + (sents ? pn + 1 : 0), s.sc.formOff + pn, 4, cudaMemcpyDeviceToHost, s.stream), "D2H form total");
		if (est) ck(cudaMemcpyAsync(directDst, s.sc.packed, est * sizeof(DToken), cudaMemcpyDeviceToHost, s.stream), "D2H tokens");
		ck(cudaEventRecord(s.ev[5], s.stream), "event");
		s.busy = true; s.n = pn; s.tokCopied = est;
		last.h2dBytes += pT * 2 + ((size_t)pn + 1) * 4;
	}

	// waits for the token copies still in flight into `out.tokens` (their time counts as D2H)
	void Engine::drainTokenCopies(BatchOutput& out)
	{
		for (auto& s : slot_)
		{
			if (!s.tokPending) continue;
			ck(cudaEventSynchronize(s.ev[7]), "sync (token copy)");
			s.tokPending = false;
			float ms = 0;
			cudaEventElapsedTime(&ms, s.ev[6], s.ev[7]); out.msD2H += ms; out.msTotal += ms;
		}
	}

	// waits for the slot's pass, appends its sentences (they are the next ones in input order) to `out`
	void Engine::finishPass(Slot& s, BatchOutput& out, uint32_t outputs)
	{
		if (!s.busy) return;
		ck(cudaStreamSynchronize(s.stream), "sync (a kernel fault surfaces here)");
		s.busy = false;
		if (s.tokPending)      // (the stream is idle: the slot's previous token copy is done as well)
		{
			s.tokPending = false;
			float ms = 0;
			cudaEventElapsedTime(&ms, s.ev[6], s.ev[7]); out.msD2H += ms; out.msTotal += ms;
		}
		const uint32_t pn = s.n;
		const bool tokens = (outputs & OUT_TOKENS) != 0, sents = (outputs & OUT_SENTS) != 0, join = (s.sc.bv.match_options & MO_JOIN_ANY) != 0;
		const size_t headWords = ((size_t)pn + 1) + 2 * (size_t)pn + 2 + (sents ? (size_t)pn + 1 : 0) + (join ? 1 : 0);
		const uint32_t* hTokOff = (const uint32_t*)s.hPinOut; const float* hScore = (const float*)(hTokOff + pn + 1); const uint32_t* hStatus = (const uint32_t*)(hScore + pn); const uint32_t* hDbg = hStatus + pn;
		if (hDbg[0] || hDbg[1]) checkDebug(s.sc);
		const uint32_t total = tokens ? hTokOff[pn] : 0;
		const size_t base = out.tokens.size();
		// what the first pass copied on its own is in place already (base == 0 there); make it part of the array before anything can move it
		const size_t first = std::min<size_t>(total, s.tokCopied);
		if (first) out.tokens.resize(base + first);
		const size_t formBase = out.forms.size();
		if (join && tokens)
		{
			// (the rows still to be copied get their entry offsets moved on the device; a pass with a base has no early copy: only the first does)
			const uint32_t nForms = hDbg[2 + (sents ? pn + 1 : 0)];
			out.forms.resize(formBase + nForms);
			if (nForms) ck(cudaMemcpy(out.forms.data() + formBase, s.sc.packedForms, (size_t)nForms * 2, cudaMemcpyDeviceToHost), "D2H joined forms");
			if (formBase && total)
			{
				if (first) throw std::runtime_error("joined forms: a later pass has an early token copy");
				rebase_joined_kernel<<<(total + 255) / 256, 256, 0, s.stream>>>(total, (uint32_t)formBase, s.sc.packed);
				ck(cudaGetLastError(), "rebase_joined_kernel launch");
			}
			last.d2hBytes += (size_t)nForms * 2;
		}
		if (total > first)
		{
			if (base + total > out.tokens.capacity()) drainTokenCopies(out);      // the array is about to move
			out.tokens.resize(base + total);
			ck(cudaEventRecord(s.ev[6], s.stream), "event");
			ck(cudaMemcpyAsync(out.tokens.data() + base + first, s.sc.packed + first, (size_t)(total - first) * sizeof(DToken), cudaMemcpyDeviceToHost, s.stream), "D2H tokens");
			ck(cudaEventRecord(s.ev[7], s.stream), "event");
			s.tokPending = true;
		}
		for (uint32_t k = 0; k < pn; ++k)
		{
			out.tokOff.push_back((uint32_t)(base + (tokens ? hTokOff[k + 1] : 0)));
			out.scores.push_back(hScore[k]); out.status.push_back(hStatus[k]);
		}
		const KernelMs t = kernelMs(s.ev);
		out.msLattice += t.lattice; out.msViterbi += t.viterbi; out.msPack += t.pack;
		float ms;
		cudaEventElapsedTime(&ms, s.ev[0], s.ev[1]); out.msH2D += ms;
		cudaEventElapsedTime(&ms, s.ev[4], s.ev[5]); out.msD2H += ms;
		cudaEventElapsedTime(&ms, s.ev[0], s.ev[5]); out.msTotal += ms;
		last.d2hBytes += headWords * 4 + (size_t)std::max<size_t>(total, s.tokCopied) * sizeof(DToken);
		if (sents) copySents(s.sc, s.stream, s.evSents, pn, hDbg + 2, out);
	}

	// Sentences that overflowed the arithmetic capacity of a main arena are re-run in the retry arena with 8 x the path and 4 x the
	// node capacity (round 0), then, what still fails, with 64 x / 16 x (round 1); a round is cut into sub-passes that fit a memory
	// budget.  runRetry runs round `round` and the rounds after it over the n sentences of the contiguous sub-batch text / offsets:
	// `out.status` holds on entry the status each of them failed with, and `out` receives their results.  A sentence that fails even
	// then keeps its status and has no tokens: the caller reports it per sentence instead of failing the whole batch.
	void Engine::runRetry(const uint16_t* text, const uint32_t* offsets, uint32_t n, uint32_t matchOptions, int round, BatchOutput& out, uint32_t outputs)
	{
		const bool tokens = (outputs & OUT_TOKENS) != 0, sents = (outputs & OUT_SENTS) != 0;
		static const uint32_t pathMul[2] = { 8, 64 }, nodeMul[2] = { 4, 16 };
		const size_t budget = (size_t)4 << 30;       // bytes of path pool per sub-pass (the retry arena stays allocated with its handle)
		const uint32_t ppu = DEFAULT_PATHS_PER_UNIT * pathScale() * pathMul[round], pc = DEFAULT_PATHS_CONST * pathScale() * pathMul[round], npu = KB_DEFAULT_NODES_PER_UNIT * nodeMul[round];
		const auto fits = [&](size_t units, size_t count) { return (units * ppu + count * pc) * pathStride() <= budget; };
		Slot& s = slot_[0];
		out.tokOff.assign(1, 0); out.tokens.clear(); out.forms.clear(); out.scores.assign(n, 0.f);
		if (sents) { out.sentOff.assign(1, 0); out.sentBegin.clear(); out.sentEnd.clear(); }
		std::vector<uint32_t> subOff, tokOff, sentOff;
		for (uint32_t i0 = 0, i1; i0 < n; i0 = i1)
		{
			i1 = passEnd(offsets, i0, n, fits);
			const uint32_t pn = i1 - i0;
			const size_t t0 = offsets[i0], pT = offsets[i1] - t0, U = 2 * pT + 4 * (size_t)pn;
			try { ensureScratch(retry_, s.stream, U, pn, ppu, pc, npu); if (sents) ensureSentScratch(retry_); }
			catch (const std::exception&)
			{
				// the escalated arena does not fit the device: these sentences keep their overflow status (no tokens), the batch goes on
				cudaGetLastError();
				freeScratch(retry_);
				out.tokOff.resize(out.tokOff.size() + pn, (uint32_t)out.tokens.size());
				if (sents) out.sentOff.resize(out.sentOff.size() + pn, (uint32_t)out.sentBegin.size());
				continue;
			}
			subOff.resize((size_t)pn + 1);
			for (uint32_t k = 0; k <= pn; ++k) subOff[k] = offsets[i0 + k] - (uint32_t)t0;
			ck(cudaMemcpyAsync(retry_.dText, text + t0, pT * 2, cudaMemcpyHostToDevice, s.stream), "H2D text");
			ck(cudaMemcpyAsync(retry_.dOff, subOff.data(), ((size_t)pn + 1) * 4, cudaMemcpyHostToDevice, s.stream), "H2D offsets");
			bind(retry_, retry_.dText, retry_.dOff, pn, matchOptions, nodeMul[round]);
			launchAll(retry_, s.stream, s.ev, pn);
			if (sents) launchSents(retry_, s.stream, s.evSents, pn);
			tokOff.resize((size_t)pn + 1);
			ck(cudaMemcpyAsync(tokOff.data(), retry_.tokOff, ((size_t)pn + 1) * 4, cudaMemcpyDeviceToHost, s.stream), "D2H offsets");
			ck(cudaMemcpyAsync(out.scores.data() + i0, retry_.vv.score, (size_t)pn * 4, cudaMemcpyDeviceToHost, s.stream), "D2H scores");
			ck(cudaMemcpyAsync(out.status.data() + i0, retry_.bv.status, (size_t)pn * 4, cudaMemcpyDeviceToHost, s.stream), "D2H status");
			if (sents) { sentOff.resize((size_t)pn + 1); ck(cudaMemcpyAsync(sentOff.data(), retry_.sentOff, ((size_t)pn + 1) * 4, cudaMemcpyDeviceToHost, s.stream), "D2H sentence offsets"); }
			ck(cudaStreamSynchronize(s.stream), "sync (retry pass)");
			checkDebug(retry_);
			if (!tokens) std::fill(tokOff.begin(), tokOff.end(), 0u);
			const size_t base = out.tokens.size(), nTok = tokOff[pn];
			out.tokens.resize(base + nTok);
			if (nTok) ck(cudaMemcpy(out.tokens.data() + base, retry_.packed, nTok * sizeof(DToken), cudaMemcpyDeviceToHost), "D2H tokens");
			if (tokens && (matchOptions & MO_JOIN_ANY))
			{
				uint32_t nForms = 0;
				ck(cudaMemcpy(&nForms, retry_.formOff + pn, 4, cudaMemcpyDeviceToHost), "D2H form total");
				copyForms(retry_, nForms, base, out);
			}
			for (uint32_t k = 1; k <= pn; ++k) out.tokOff.push_back((uint32_t)(base + tokOff[k]));
			out.msTotal += kernelMs(s.ev).total;
			last.h2dBytes += pT * 2 + ((size_t)pn + 1) * 4; last.d2hBytes += ((size_t)pn * 3 + 1) * 4 + nTok * sizeof(DToken);
			if (sents)
			{
				const float msSents0 = out.msSents;
				copySents(retry_, s.stream, s.evSents, pn, sentOff.data(), out);
				out.msTotal += out.msSents - msSents0;
				last.d2hBytes += ((size_t)pn + 1) * 4;
			}
		}
		if (round + 1 < 2) retryFailed(text, offsets, matchOptions, round + 1, out, outputs);
	}

	// Gathers the retryable sentences of `out` (the results of the batch text / offsets), in input order, into one contiguous
	// sub-batch, runs it through retry round `round` and the rounds after it, and puts the results in their places.  Returns how many
	// sentences it re-ran.
	size_t Engine::retryFailed(const uint16_t* text, const uint32_t* offsets, uint32_t matchOptions, int round, BatchOutput& out, uint32_t outputs)
	{
		std::vector<uint32_t> ids;
		for (uint32_t i = 0; i < (uint32_t)out.status.size(); ++i) if (retryable(out.status[i])) ids.push_back(i);
		if (ids.empty()) return 0;
		std::vector<uint16_t> subText; std::vector<uint32_t> subOff{ 0 };
		BatchOutput sub;
		for (uint32_t id : ids)
		{
			subText.insert(subText.end(), text + offsets[id], text + offsets[id + 1]);
			subOff.push_back((uint32_t)subText.size());
			sub.status.push_back(out.status[id]);
		}
		runRetry(subText.data(), subOff.data(), (uint32_t)ids.size(), matchOptions, round, sub, outputs);
		// splice the retried sentences into the token stream and the sentence ranges (rare path: rebuild)
		const bool sents = (outputs & OUT_SENTS) != 0;
		TokenVec toks; std::vector<uint32_t> tokOff(1, 0), sentOff(1, 0), sentBegin, sentEnd;
		// (the retried sentences' forms go behind the batch's: a sentence that failed has none in `out`)
		const uint32_t subFormBase = (uint32_t)out.forms.size();
		out.forms.insert(out.forms.end(), sub.forms.begin(), sub.forms.end());
		toks.reserve(out.tokens.size() + sub.tokens.size());
		for (uint32_t i = 0, k = 0; i < (uint32_t)out.status.size(); ++i)
		{
			const bool retried = k < ids.size() && ids[k] == i;
			const BatchOutput& src = retried ? sub : out;
			const uint32_t j = retried ? k++ : i;
			const size_t at = toks.size();
			toks.insert(toks.end(), src.tokens.begin() + src.tokOff[j], src.tokens.begin() + src.tokOff[j + 1]);
			if (retried && subFormBase) for (size_t t = at; t < toks.size(); ++t) if (toks[t].morph & JOINED_TOKEN) toks[t].morph += subFormBase;
			out.scores[i] = src.scores[j]; out.status[i] = src.status[j];
			tokOff.push_back((uint32_t)toks.size());
			if (sents)
			{
				sentBegin.insert(sentBegin.end(), src.sentBegin.begin() + src.sentOff[j], src.sentBegin.begin() + src.sentOff[j + 1]);
				sentEnd.insert(sentEnd.end(), src.sentEnd.begin() + src.sentOff[j], src.sentEnd.begin() + src.sentOff[j + 1]);
				sentOff.push_back((uint32_t)sentBegin.size());
			}
		}
		out.tokens.swap(toks); out.tokOff.swap(tokOff);
		if (sents) { out.sentOff.swap(sentOff); out.sentBegin.swap(sentBegin); out.sentEnd.swap(sentEnd); out.msSents += sub.msSents; }
		out.msTotal += sub.msTotal;
		return ids.size();
	}

	// Public entry: batches of any size.  The scratch arenas are sized per pass, so a large batch (65536 / 1 M sentences)
	// is cut into passes of at most MAX_UNITS_PER_PASS normalised units / MAX_SENT_PER_PASS sentences.  A slot's arena costs about
	// 7.3 KB per unit (128 48-byte paths, 12 nodes), so 1.5 Mi units are ~11 GB per slot: an 8192-sentence batch of web-shaped text
	// (~1.3 M units) stays one pass, and two handles with both slots grown, their retry arenas and the device path of one of them fit
	// the 80 GB of an H100.
	static constexpr size_t MAX_UNITS_PER_PASS = 3u << 19, MAX_SENT_PER_PASS = 16384;
	static size_t passSentLimit()
	{
		// KIWI_B200_PASS_SENT: sentences per pass (experiments with the overlap of small passes); default 16384
		static const size_t v = [] { const char* e = std::getenv("KIWI_B200_PASS_SENT"); const long x = e ? std::atol(e) : 0; return x > 0 ? std::min<size_t>((size_t)x, MAX_SENT_PER_PASS) : MAX_SENT_PER_PASS; }();
		return v;
	}

	void Engine::analyze(const uint16_t* text, const uint32_t* offsets, uint32_t n, uint32_t matchOptions, BatchOutput& out, uint32_t outputs)
	{
		DeviceGuard g{ device };
		last = Stats{};
		const bool tokens = (outputs & OUT_TOKENS) != 0;
		// (the caller may hand in a recycled BatchOutput: keep the vectors' capacity)
		out.tokOff.assign(1, 0); out.tokens.clear(); out.forms.clear(); out.scores.clear(); out.status.clear();
		out.sentOff.clear(); out.sentBegin.clear(); out.sentEnd.clear();
		if (outputs & OUT_SENTS) out.sentOff.push_back(0);
		out.msH2D = out.msLattice = out.msViterbi = out.msPack = out.msSents = out.msD2H = out.msTotal = 0;
		if (n == 0) return;
		if (offsets[0] != 0) throw std::runtime_error("offsets[0] must be 0");
		for (uint32_t i = 0; i < n; ++i) if (offsets[i + 1] < offsets[i]) throw std::runtime_error("offsets must be non-decreasing");
		out.tokOff.reserve((size_t)n + 1); out.scores.reserve(n); out.status.reserve(n);
		if (tokens) out.tokens.reserve(tokenEstimate(offsets[n], n));
		const size_t sentLimit = std::max<size_t>(passSentLimit() / passDivisor(), 1), unitLimit = MAX_UNITS_PER_PASS / passDivisor();
		const auto fits = [&](size_t units, size_t count) { return units <= unitLimit && count <= sentLimit; };
		uint32_t i0 = 0, k = 0;
		try
		{
			while (i0 < n)
			{
				const uint32_t i1 = passEnd(offsets, i0, n, fits);
				Slot& s = slot_[k & 1];
				// results are appended in input order: the slot's previous pass (k - 2) is older than the other slot's (k - 1)
				finishPass(s, out, outputs);
				submitPass(s, text, offsets, i0, i1 - i0, matchOptions, k == 0 && tokens ? out.tokens.data() : nullptr, outputs);      // (capacity reserved above)
				i0 = i1; ++k;
			}
			finishPass(slot_[k & 1], out, outputs);
			finishPass(slot_[(k + 1) & 1], out, outputs);
			drainTokenCopies(out);
		}
		catch (...)
		{
			for (auto& sl : slot_) { if (sl.busy || sl.tokPending) { cudaStreamSynchronize(sl.stream); sl.busy = false; sl.tokPending = false; } }
			throw;
		}
		last.retried = retryFailed(text, offsets, matchOptions, 0, out, outputs);
		last.nSentences = n; last.rawUnits = offsets[n]; last.tokens = out.tokens.size();
		last.msLattice = out.msLattice; last.msViterbi = out.msViterbi; last.msPack = out.msPack;
	}

	__global__ void rebase_kernel(uint32_t n, const uint32_t* __restrict__ off, uint32_t i0, uint32_t* __restrict__ out)
	{
		const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
		if (k <= n) out[k] = off[i0 + k] - off[i0];
	}

	// Device-resident inputs (bench.py's `value`): passes run back to back on ONE stream so that every kernel's CUDA-event time is
	// its own; sentences that overflow the arena are re-run through the host retry path (their text comes back from the device).
	float Engine::analyzeDevice(const uint16_t* dText, const uint32_t* dOffsets, uint32_t n, uint64_t totalUnits, uint32_t matchOptions, uint64_t* nTokens)
	{
		DeviceGuard g{ device };
		last = Stats{};
		if (nTokens) *nTokens = 0;
		if (n == 0) return 0.f;
		Slot& s = slot_[0];
		std::vector<uint32_t> off;
		const size_t Uall = 2 * (size_t)totalUnits + 4 * (size_t)n;
		const size_t devUnits = 4 * MAX_UNITS_PER_PASS / passDivisor(), devSent = 4 * MAX_SENT_PER_PASS / passDivisor();
		const bool single = Uall <= devUnits && n <= devSent;      // (one launch set keeps the longest-first order over the whole batch)
		const auto fits = [&](size_t units, size_t count) { return units <= devUnits && count <= devSent; };
		if (!single)
		{
			off.resize((size_t)n + 1);
			ck(cudaMemcpy(off.data(), dOffsets, ((size_t)n + 1) * 4, cudaMemcpyDeviceToHost), "D2H offsets");
		}
		float msTotal = 0; uint64_t total = 0;
		std::vector<uint32_t> failed;
		BatchOutput retry;      // (retry.status: the status each failed sentence came back with)
		for (uint32_t i0 = 0, i1; i0 < n; i0 = i1)
		{
			i1 = single ? n : passEnd(off.data(), i0, n, fits);
			const uint32_t pn = i1 - i0;
			const size_t pT = single ? totalUnits : off[i1] - off[i0], U = 2 * pT + 4 * (size_t)pn;
			ensureScratch(s.sc, s.stream, U, pn, DEFAULT_PATHS_PER_UNIT * pathScale(), DEFAULT_PATHS_CONST * pathScale(), KB_DEFAULT_NODES_PER_UNIT);
			const uint16_t* pText = dText; const uint32_t* pOff = dOffsets;
			if (!single)
			{
				rebase_kernel<<<(pn + 256) / 256, 256, 0, s.stream>>>(pn, dOffsets, i0, s.sc.dOff);
				ck(cudaGetLastError(), "rebase_kernel launch");
				pText = dText + off[i0]; pOff = s.sc.dOff;
			}
			bind(s.sc, pText, pOff, pn, matchOptions, 1);
			launchAll(s.sc, s.stream, s.ev, pn);
			growPinned(&s.hPinOut, &s.pinOutCap, (size_t)pn * 4 + 64);
			uint32_t* hStatus = (uint32_t*)s.hPinOut; uint32_t* hTotal = hStatus + pn;
			ck(cudaMemcpyAsync(hTotal, s.sc.tokOff + pn, 4, cudaMemcpyDeviceToHost, s.stream), "D2H total");
			ck(cudaMemcpyAsync(hStatus, s.sc.bv.status, (size_t)pn * 4, cudaMemcpyDeviceToHost, s.stream), "D2H status");
			ck(cudaStreamSynchronize(s.stream), "sync (a kernel fault surfaces here)");
			const KernelMs t = kernelMs(s.ev);
			msTotal += t.total; last.msLattice += t.lattice; last.msViterbi += t.viterbi; last.msPack += t.pack;
			total += *hTotal;
			last.d2hBytes += 4 + (size_t)pn * 4;
			for (uint32_t k = 0; k < pn; ++k) if (retryable(hStatus[k])) { failed.push_back(i0 + k); retry.status.push_back(hStatus[k]); }
		}
		last.nSentences = n; last.rawUnits = totalUnits; last.retried = failed.size();
		if (!failed.empty())
		{
			// overflowed sentences (rare) go through the escalating retry arena; their text comes back from the device
			if (off.empty()) { off.resize((size_t)n + 1); ck(cudaMemcpy(off.data(), dOffsets, ((size_t)n + 1) * 4, cudaMemcpyDeviceToHost), "D2H offsets"); }
			std::vector<uint16_t> subText; std::vector<uint32_t> subOff{ 0 };
			for (uint32_t id : failed)
			{
				const size_t len = off[id + 1] - off[id], at = subText.size();
				subText.resize(at + len);
				if (len) ck(cudaMemcpy(subText.data() + at, dText + off[id], len * 2, cudaMemcpyDeviceToHost), "D2H text");
				subOff.push_back((uint32_t)subText.size());
			}
			runRetry(subText.data(), subOff.data(), (uint32_t)failed.size(), matchOptions, 0, retry);
			msTotal += retry.msTotal;
			total += retry.tokens.size();
		}
		last.tokens = total;
		if (nTokens) *nTokens = total;
		return msTotal;
	}

	void Engine::debugCong(uint32_t n, const uint32_t* ctx, const uint32_t* wid, const int32_t* node,
		int32_t* outDot, float* outEps, int32_t* outNode, uint32_t* outCtx, int32_t* outTile)
	{
		if (model.dev.model_type != 4) throw std::runtime_error("debugCong needs a CoNg model image");
		if (n == 0) return;
		for (uint32_t i = 0; i < n; ++i)
		{
			if (ctx[i] >= model.dev.cg_context_size || wid[i] >= model.dev.lang_vocab_size || node[i] < 0 || (uint32_t)node[i] >= model.header.cg_num_nodes)
				throw std::runtime_error("debugCong: index out of range");
		}
		DeviceGuard g{ device };
		uploadConstants();
		const uint32_t nU = std::min(n, 64u), nW = std::min(n, 32u);
		uint32_t* d = nullptr;
		const size_t words = (size_t)n * 9 + (size_t)nU * nW;
		ck(cudaMalloc(&d, words * 4), "cudaMalloc(debugCong)");
		uint32_t* dCtx = d; uint32_t* dWid = d + n; int32_t* dNode = reinterpret_cast<int32_t*>(d + 2 * n);
		int32_t* dDot = reinterpret_cast<int32_t*>(d + 3 * n); float* dEps = reinterpret_cast<float*>(d + 4 * n);
		int32_t* dNodeOut = reinterpret_cast<int32_t*>(d + 7 * n); uint32_t* dCtxOut = d + 8 * n; int32_t* dTile = reinterpret_cast<int32_t*>(d + 9 * n);
		cudaError_t e = cudaMemcpyAsync(dCtx, ctx, n * 4, cudaMemcpyHostToDevice, stream);
		if (e == cudaSuccess) e = cudaMemcpyAsync(dWid, wid, n * 4, cudaMemcpyHostToDevice, stream);
		if (e == cudaSuccess) e = cudaMemcpyAsync(dNode, node, n * 4, cudaMemcpyHostToDevice, stream);
		if (e == cudaSuccess) e = launch_cong_debug(n, dCtx, dWid, dNode, dDot, dEps, dNodeOut, dCtxOut, dTile, stream);
		if (e == cudaSuccess) e = cudaMemcpyAsync(outDot, dDot, n * 4, cudaMemcpyDeviceToHost, stream);
		if (e == cudaSuccess) e = cudaMemcpyAsync(outEps, dEps, n * 12, cudaMemcpyDeviceToHost, stream);
		if (e == cudaSuccess) e = cudaMemcpyAsync(outNode, dNodeOut, n * 4, cudaMemcpyDeviceToHost, stream);
		if (e == cudaSuccess) e = cudaMemcpyAsync(outCtx, dCtxOut, n * 4, cudaMemcpyDeviceToHost, stream);
		if (e == cudaSuccess) e = cudaMemcpyAsync(outTile, dTile, (size_t)nU * nW * 4, cudaMemcpyDeviceToHost, stream);
		if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
		cudaFree(d);
		ck(e, "debugCong");
	}

	void Engine::setConfig(const kb2_config& cfg)
	{
		DeviceGuard g{ device };
		model.dev.cfg = cfg;
		model.header.config = cfg;
		if (g_devState[g.dev].owner == &model) g_devState[g.dev].owner = nullptr;
	}

	void Engine::debugTiming(uint32_t n, unsigned long long* out)
	{
		DeviceGuard g{ device };
		const Scratch& sc = slot_[0].sc;
		if (!sc.vv.timing || n > sc.capSent) throw std::runtime_error("debugTiming: no launch of that size yet");
		ck(cudaMemcpy(out, sc.vv.timing, (size_t)n * 16, cudaMemcpyDeviceToHost), "debugTiming");
	}

	int Engine::debugLattice(const uint16_t* text, uint32_t len, uint32_t matchOptions, std::vector<int32_t>& rows)
	{
		const uint32_t off[2] = { 0, len };
		const size_t U = 2 * (size_t)len + 4;
		DeviceGuard g{ device };
		Scratch& sc = slot_[0].sc;
		ensureScratch(sc, stream, U, 1, DEFAULT_PATHS_PER_UNIT * pathScale(), DEFAULT_PATHS_CONST * pathScale(), KB_DEFAULT_NODES_PER_UNIT);
		ck(cudaMemcpyAsync(sc.dText, text, (size_t)len * 2, cudaMemcpyHostToDevice, stream), "H2D");
		ck(cudaMemcpyAsync(sc.dOff, off, 8, cudaMemcpyHostToDevice, stream), "H2D");
		bind(sc, sc.dText, sc.dOff, 1, matchOptions, 1);
		ck(cudaMemsetAsync(sc.order, 0, 4, stream), "memset");
		sc.bv.order = sc.order;
		uploadConstants();
		ck(launch_lattice(model.dev, sc.bv, stream), "lattice launch");
		uint32_t nChunks = 0, status = 0;
		ck(cudaMemcpyAsync(&nChunks, sc.bv.n_chunks, 4, cudaMemcpyDeviceToHost, stream), "D2H");
		ck(cudaMemcpyAsync(&status, sc.bv.status, 4, cudaMemcpyDeviceToHost, stream), "D2H");
		ck(cudaStreamSynchronize(stream), "sync");
		if (status) return -(int)status;
		std::vector<DChunk> chunks(nChunks);
		if (nChunks) ck(cudaMemcpy(chunks.data(), sc.bv.chunks, nChunks * sizeof(DChunk), cudaMemcpyDeviceToHost), "D2H chunks");
		rows.clear();
		int total = 0;
		for (uint32_t c = 0; c < nChunks; ++c)
		{
			std::vector<DNode> nodes(chunks[c].n_nodes);
			ck(cudaMemcpy(nodes.data(), sc.bv.nodes + chunks[c].node_off, nodes.size() * sizeof(DNode), cudaMemcpyDeviceToHost), "D2H nodes");
			for (auto& nd : nodes)
			{
				const int32_t r[9] = { nd.form, nd.uform_len ? (int32_t)nd.uform_off : -1, (int32_t)nd.uform_len, nd.prev, nd.sibling,
					(int32_t)nd.start_pos, (int32_t)nd.end_pos, nd.space_errors, (int32_t)c };
				rows.insert(rows.end(), r, r + 9);
				++total;
			}
		}
		return total;
	}
}
