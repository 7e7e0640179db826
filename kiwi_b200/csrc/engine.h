// kiwi_b200: host engine (model residency, batch marshalling, kernel launches, result packing).
#pragma once
#include <cstdint>
#include <memory>
#include <string>
#include <utility>
#include <vector>
#include <unordered_map>
#include <string>
#include <cuda_runtime.h>
#include "kb_model.h"
#include "kb_batch.h"

namespace kb
{
	std::vector<char> readImageFile(const std::string& modelPath);

	struct Model
	{
		std::vector<char> blob;
		kb2_header header;
		DevModel dev;
		std::vector<void*> owned;
		size_t deviceBytes = 0;
		const kb2_form* hForms = nullptr; const uint16_t* hFormChars = nullptr; const kb2_morph* hMorphs = nullptr;
		std::vector<uint32_t> hChrBmp;      // host copy of chr_bmp (cls | script << 8 | flags << 16) for result assembly
		std::vector<DCand> hCands;          // host copy of the static candidate table (AnalyzeOption::blocklist patches a copy of it)
		// AnalyzeOption::blocklist: the candidate table with every candidate that Morpheme::hasMorpheme(blocklist) would reject marked like a
		// non-standard dialect candidate (DK_DIALECT: the kernels skip it at the very place the reference tests the blocklist, PathEvaluator.hpp:384-386)
		std::vector<DCand> blockedCands(const std::vector<uint32_t>& sortedMorphemeIds) const;
		// Kiwi::findMorphemes (src/Kiwi.cpp:1281-1297): the morphemes of the form spelled `form` (any code units; codas are normalised here) with tag
		// `tag` (0 = any; the irregular bit is ignored), combining-socket candidates left out
		std::vector<uint32_t> findMorphemes(const uint16_t* form, size_t len, uint8_t tag) const;
		mutable std::unordered_map<std::u16string, uint32_t> formIndex_;      // form string -> first form of that spelling (built on first use)
		uint32_t hostChrAttr(uint16_t c) const { return hChrBmp[c]; }
		void load(const void* bytes, size_t size);
		~Model();
	};

	// a prepared typo transformer resident on the device (flat typo image, include/kiwi_b200_typo.h); an analysis option
	// (kiwi_analyze_option_t::typo_transformer), shared read-only by any number of engines
	struct TypoDev
	{
		std::vector<char> blob;
		void* dBlob = nullptr;
		TypoView view{};             // device pointers of the image sections + continual threshold; no scratch
		void load(const void* bytes, size_t size);
		~TypoDev();
	};

	// Allocator of the result token arrays: page-locked host memory (any device of the process can copy into it), and resize() leaves
	// the trivially-constructible rows uninitialised - the device-to-host copies of a pass land in the caller's result array itself,
	// there is no staging copy on the host.  Result holders are recycled (capi.cu), so the page-locking cost is paid once per holder.
	template<class T> struct PinnedNoInitAlloc
	{
		using value_type = T;
		PinnedNoInitAlloc() = default;
		template<class U> PinnedNoInitAlloc(const PinnedNoInitAlloc<U>&) {}
		T* allocate(size_t n)
		{
			void* p = nullptr;
			if (cudaHostAlloc(&p, n * sizeof(T), cudaHostAllocPortable) != cudaSuccess) { cudaGetLastError(); throw std::bad_alloc(); }
			return static_cast<T*>(p);
		}
		void deallocate(T* p, size_t) { cudaFreeHost(p); }
		template<class U, class... A> void construct(U* p, A&&... a)
		{
			if constexpr (sizeof...(A) == 0) ::new ((void*)p) U; else ::new ((void*)p) U(std::forward<A>(a)...);
		}
		template<class U> bool operator==(const PinnedNoInitAlloc<U>&) const { return true; }
		template<class U> bool operator!=(const PinnedNoInitAlloc<U>&) const { return false; }
	};
	using TokenVec = std::vector<DToken, PinnedNoInitAlloc<DToken>>;

	// what Engine::analyze brings back besides scores and statuses: the token rows, the sentence ranges (Kiwi::splitIntoSents), or both
	enum : uint32_t { OUT_TOKENS = 1, OUT_SENTS = 2 };

	struct BatchOutput
	{
		std::vector<uint32_t> tokOff;      // [n + 1]; all 0 without OUT_TOKENS
		TokenVec tokens;
		std::vector<float> scores;
		std::vector<uint32_t> status;
		// OUT_SENTS: the ranges of sentence s are [sentOff[s], sentOff[s + 1]) of sentBegin / sentEnd, UTF-16 units relative to the sentence's text
		std::vector<uint32_t> sentOff, sentBegin, sentEnd;
		// token-joining options: the joined forms the flagged rows (DToken::morph = JOINED_TOKEN | k) point into; empty otherwise
		std::vector<uint16_t> forms;
		float msH2D = 0, msLattice = 0, msViterbi = 0, msPack = 0, msSents = 0, msD2H = 0, msTotal = 0;
	};

	struct Stats
	{
		uint64_t nSentences = 0, rawUnits = 0, normUnits = 0, latticeNodes = 0, tokens = 0, paths = 0;
		uint64_t h2dBytes = 0, d2hBytes = 0, kernelLaunches = 0, retried = 0;
		float msLattice = 0, msViterbi = 0, msPack = 0;
	};

	class Engine
	{
	public:
		Model model;
		cudaStream_t stream = nullptr;      // stream of pass slot 0 (single-pass calls, debug entry points)
		Stats last;
		int device = 0;                     // CUDA device the model and the scratch arenas live on

		explicit Engine(const void* imageBytes, size_t size);
		~Engine();

		// host buffers in, host buffers out (H2D / D2H inside).  Batches larger than one pass are cut into passes that alternate
		// between two scratch arenas on two streams: pass k+1's H2D and kernels overlap pass k's tail and D2H.
		// A sentence that overflows even the escalated retry capacity keeps a non-zero status and an empty token list (no throw).
		// `outputs` (OUT_*): OUT_SENTS adds the sentence kernel (sents.cu) after the token emission; without OUT_TOKENS no token row is copied back.
		void analyze(const uint16_t* text, const uint32_t* offsets, uint32_t n, uint32_t matchOptions, BatchOutput& out, uint32_t outputs = OUT_TOKENS);
		// AnalyzeOption::blocklist: a patched copy of the candidate table (device memory of this engine's device, Model::blockedCands) replaces
		// the model's for the calls that follow; nullptr = the model's own table
		void setCandsOverride(const DCand* deviceTable);
		// device-resident inputs; results stay on the device.  returns elapsed ms (CUDA events on the engine stream)
		float analyzeDevice(const uint16_t* dText, const uint32_t* dOffsets, uint32_t n, uint64_t totalUnits, uint32_t matchOptions, uint64_t* nTokens);
		// lattice of one sentence for stage-level parity tests
		int debugLattice(const uint16_t* text, uint32_t len, uint32_t matchOptions, std::vector<int32_t>& rows);
		// per-sentence {start, end} ns of the last Viterbi launch of the main scratch (diagnostics)
		void debugTiming(uint32_t n, unsigned long long* out);
		// KiwiConfig fields read by the kernels; the constant-memory model view is refreshed at the next launch
		void setConfig(const kb2_config& cfg);
		// AnalyzeOption::typoTransformer / typoThreshold for the following analyze* calls (nullptr: plain lattice)
		void setTypo(const TypoDev* typo, float threshold) { typo_ = typo; typoThreshold_ = threshold; }
		// CoNg scorer self-test on the device (see cong_debug_kernel): n triples in, per-triple results + the tensor-core tile out
		void debugCong(uint32_t n, const uint32_t* ctx, const uint32_t* wid, const int32_t* node,
			int32_t* outDot, float* outEps, int32_t* outNode, uint32_t* outCtx, int32_t* outTile);

	private:
		struct Scratch
		{
			size_t capUnits = 0, capSent = 0, capText = 0;
			uint32_t pathsPerUnit = 0, pathsConst = 0, nodesPerUnit = 0;
			std::vector<void*> bufs;
			std::vector<void*> typoBufs; size_t typoCapUnits = 0; uint32_t typoGraphPerUnit = 0, typoStatesPerUnit = 0;
			TypoView typoScratch{};
			BatchView bv{};
			VitView vv{};
			uint32_t* tokOff = nullptr;      // [capSent + 1]
			DToken* packed = nullptr;        // [capUnits]
			void* cubTemp = nullptr; size_t cubTempBytes = 0;
			uint16_t* dText = nullptr; uint32_t* dOff = nullptr;
			uint32_t* lenKeys = nullptr; uint32_t* lenKeysOut = nullptr; uint32_t* idxIn = nullptr; uint32_t* order = nullptr; uint32_t* orderVit = nullptr; void* sortTemp = nullptr; size_t sortTempBytes = 0;
			// sentence ranges (allocated by the first split): per-sentence counts and their scan [capSent + 1], the packed ranges [capUnits]
			std::vector<void*> sentBufs; size_t sentCapUnits = 0, sentCapSent = 0;
			uint32_t* nSents = nullptr; uint32_t* sentOff = nullptr; uint32_t* sentBegin = nullptr; uint32_t* sentEnd = nullptr;
			// joined forms (allocated by the first call with a token-joining option): the per-sentence pools live in vv.forms; their scan [capSent + 1]
			// and the packed forms [joinCapUnits]
			std::vector<void*> joinBufs; size_t joinCapUnits = 0, joinCapSent = 0; uint32_t joinPerUnit = 0;
			uint32_t* formOff = nullptr; uint16_t* packedForms = nullptr;
		};
		// one in-flight pass: its own scratch arena, stream, events and pinned staging
		struct Slot
		{
			Scratch sc;
			cudaStream_t stream = nullptr;
			cudaEvent_t ev[8] = { nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr };      // [6], [7]: around the deferred token copy
			cudaEvent_t evSents[4] = { nullptr, nullptr, nullptr, nullptr };      // [0], [1]: around the sentence kernels; [2], [3]: around the copy of the ranges
			uint16_t* hPinText = nullptr; uint32_t* hPinOff = nullptr; size_t pinTextCap = 0, pinOffCap = 0;
			void* hPinOut = nullptr; size_t pinOutCap = 0;
			// the pass in flight
			bool busy = false; uint32_t n = 0; size_t tokCopied = 0;
			bool tokPending = false;      // a token copy into the caller's result array is still in flight on `stream`
		};
		const TypoDev* typo_ = nullptr; float typoThreshold_ = 2.5f;
		const DCand* candsOverride_ = nullptr;
		void ensureTypoScratch(Scratch& sc, uint32_t graphPerUnit, uint32_t statesPerUnit, uint32_t mul);
		Slot slot_[2];
		Scratch retry_;                  // larger per-sentence capacity, only for sentences that overflowed a main arena

		void ensureScratch(Scratch& sc, cudaStream_t st, size_t totalUnits, size_t nSent, uint32_t pathsPerUnit, uint32_t pathsConst, uint32_t nodesPerUnit);
		void freeScratch(Scratch& sc);
		void bind(Scratch& sc, const uint16_t* dText, const uint32_t* dOffsets, uint32_t n, uint32_t matchOptions, uint32_t capMul);
		void uploadConstants();
		void launchAll(Scratch& sc, cudaStream_t st, cudaEvent_t* ev, uint32_t n);
		void ensureSentScratch(Scratch& sc);
		void ensureJoinScratch(Scratch& sc, uint32_t perUnit);
		void copyForms(Scratch& sc, uint32_t nForms, size_t tokBegin, BatchOutput& out);
		void launchSents(Scratch& sc, cudaStream_t st, cudaEvent_t* evSents, uint32_t n);
		void copySents(Scratch& sc, cudaStream_t st, cudaEvent_t* evSents, uint32_t n, const uint32_t* sentOff, BatchOutput& out);
		void submitPass(Slot& s, const uint16_t* text, const uint32_t* off, uint32_t i0, uint32_t n, uint32_t matchOptions, DToken* directDst, uint32_t outputs);
		void drainTokenCopies(BatchOutput& out);
		// SkipBigram states (Knlm node + 8-token history) rarely merge: 8 x the paths per sentence from the start (the first retry round of the
		// other models), passes 16 x smaller so that the arena stays the same size
		uint32_t pathScale() const { return model.dev.model_type == 3 ? 8u : 1u; }
		size_t passDivisor() const { return model.dev.model_type == 3 ? 16 : 1; }
		size_t pathStride() const { return model.dev.model_type == 3 ? 96 : sizeof(DPath); }      // SkipBigram paths carry their 8-token history (viterbi.cu PathS)
		void finishPass(Slot& s, BatchOutput& out, uint32_t outputs);
		void runRetry(const uint16_t* text, const uint32_t* offsets, uint32_t n, uint32_t matchOptions, int round, BatchOutput& out, uint32_t outputs = OUT_TOKENS);
		size_t retryFailed(const uint16_t* text, const uint32_t* offsets, uint32_t matchOptions, int round, BatchOutput& out, uint32_t outputs);
		void checkDebug(Scratch& sc);
	};

	// one lock per CUDA device: the kernels' model view lives in __constant__ memory (one copy per device and module), so
	// engines that share a device take turns; engines on different devices run concurrently
	struct DeviceGuard
	{
		int dev; int prev = -1;
		explicit DeviceGuard(int device);
		~DeviceGuard();
	};
}
