// kiwi_b200: extern "C" boundary (include/kiwi_b200.h).  Mirrors the error convention of the reference's
// C API (/root/reference/src/capi/kiwi_c.cpp:84-113): nothing is thrown across the ABI, failures return
// NULL / KIWIERR_* and leave a message for the calling thread in kiwi_error().
#include <cstring>
#include <algorithm>
#include <cctype>
#include <map>
#include <memory>
#include <mutex>
#include <chrono>
#include <thread>
#include <stdexcept>
#include <string>
#include <vector>
#include "../../include/kiwi_b200.h"
#include "engine.h"
#include "assemble.h"

using namespace kb;

struct kiwi_s
{
	std::unique_ptr<Engine> engine;                      // primary engine (device of kiwi_init / first device of kiwi_b200_init_multi)
	std::vector<std::unique_ptr<Engine>> extra;          // kiwi_b200_init_multi: one more engine per further device; batches are sharded round-robin
	std::mutex mtx;           // scratch arenas and streams belong to the handle: calls on one handle are serialised
	// result scratch that lives with the handle (used under mtx): the token arrays are page-locked, so they are made once and reused
	std::vector<BatchOutput> shardOut;                   // per device of a sharded batch
	BatchOutput callOut;                                 // single-sentence calls and the reader-driven batches
	int numThreads = 0;
	float oovChrBias = 0, oovGlobalWeight = 35, oovLocalWeight = 3, oovGlobalMinFreq = 4;      // KiwiConfig defaults of the chr-model oov scorers (stored only)
};

// typo handles (capi.h:35-38).  A kiwi_typo names one of the reference's default typo sets; preparing it loads the flat image
// of that set as the reference prepared it (oracle/ref_build/tools/typo_tool.cpp writes typo_<set>.img): building a
// PreparedTypoTransformer from rules natively is a host-side "next" row (DESIGN.md).
struct kiwi_typo { int set; };
struct kiwi_prepared_typo
{
	std::vector<char> blob;
	std::mutex m;
	std::map<int, std::unique_ptr<kb::TypoDev>> perDevice;      // the flat typo image resident on every device that used it
	const kb::TypoDev* forDevice(int device)
	{
		std::lock_guard<std::mutex> lk(m);
		auto& p = perDevice[device];
		if (!p)
		{
			kb::DeviceGuard g{ device };
			p.reset(new kb::TypoDev);
			p->load(blob.data(), blob.size());
		}
		return p.get();
	}
};
static kiwi_typo g_defaultTypos[7] = { {0}, {1}, {2}, {3}, {4}, {5}, {6} };
static std::string g_typoDir;      // directory of the last model image opened by kiwi_init

struct TypoScope      // AnalyzeOption::typoTransformer for the calls made while the handle's mutex is held
{
	Engine* e;
	TypoScope(Engine* _e, const kiwi_analyze_option_t& o) : e{ _e } { e->setTypo(o.typo_transformer ? o.typo_transformer->forDevice(e->device) : nullptr, o.typo_threshold); }
	~TypoScope() { e->setTypo(nullptr, 2.5f); }
};

// kiwi_morphset (capi.h:36): morpheme ids + one patched candidate table per engine that has used the set (device memory of that engine's device)
struct kiwi_morphset
{
	kiwi_s* inst;
	std::vector<uint32_t> ids;      // sorted, unique
	uint64_t version = 0;
	std::mutex m;
	struct Table { void* dev = nullptr; uint64_t version = ~0ull; int device = 0; };
	std::map<Engine*, Table> tables;
	const DCand* forEngine(Engine* e)
	{
		std::lock_guard<std::mutex> lk(m);
		Table& t = tables[e];
		if (t.version != version)
		{
			const std::vector<DCand> rows = e->model.blockedCands(ids);
			DeviceGuard g{ e->device };
			if (!t.dev && cudaMalloc(&t.dev, rows.size() * sizeof(DCand)) != cudaSuccess) { cudaGetLastError(); throw std::runtime_error("cudaMalloc(blocklist candidate table) failed"); }
			e->setCandsOverride(nullptr);      // (nothing reads the table while it is rewritten)
			if (cudaMemcpy(t.dev, rows.data(), rows.size() * sizeof(DCand), cudaMemcpyHostToDevice) != cudaSuccess) { cudaGetLastError(); throw std::runtime_error("upload of the blocklist candidate table failed"); }
			t.version = version; t.device = e->device;
		}
		return static_cast<const DCand*>(t.dev);
	}
	~kiwi_morphset() { for (auto& kv : tables) if (kv.second.dev) { DeviceGuard g{ kv.second.device }; cudaFree(kv.second.dev); } }
};
struct BlockScope      // AnalyzeOption::blocklist for the calls made while the handle's mutex is held
{
	Engine* e;
	BlockScope(Engine* _e, const kiwi_analyze_option_t& o) : e{ _e } { e->setCandsOverride(o.blocklist && !o.blocklist->ids.empty() ? o.blocklist->forEngine(e) : nullptr); }
	~BlockScope() { e->setCandsOverride(nullptr); }
};

struct kiwi_ss { std::vector<std::pair<uint32_t, uint32_t>> ranges; };      // capi/kiwi_c.cpp: kiwi_ss = vector<pair<size_t, size_t>>

struct kiwi_res
{
	struct Tok { kiwi_token_info_t info; uint32_t morphId; std::u16string form; std::string form8; };
	std::vector<Tok> toks;
	float score = 0;
	bool empty = false;
};

static thread_local std::string g_error;
static thread_local bool g_hasError = false;
static int g_device = -1;

static void setError(const std::exception& e) { g_error = e.what(); g_hasError = true; }
static void setError(const char* s) { g_error = s; g_hasError = true; }

static const char* tagName(uint8_t t)
{
	static const char* tags[] = { "UN", "NNG", "NNP", "NNB", "VV", "VA", "MAG", "NR", "NP", "VX", "MM", "MAJ", "IC", "XPN", "XSN", "XSV", "XSA", "XSM", "XR",
		"VCP", "VCN", "SF", "SP", "SS", "SSO", "SSC", "SE", "SO", "SW", "SB", "SL", "SH", "SN", "W_URL", "W_EMAIL", "W_MENTION", "W_HASHTAG", "W_SERIAL", "W_EMOJI",
		"JKS", "JKC", "JKG", "JKO", "JKB", "JKV", "JKQ", "JX", "JC", "EP", "EF", "EC", "ETN", "ETM", "Z_CODA", "Z_SIOT", "USER0", "USER1", "USER2", "USER3", "USER4", "P", "@" };
	if (t & 0x80)
	{
		switch (t & 0x7F) { case T_vv: return "VV-I"; case T_va: return "VA-I"; case T_vx: return "VX-I"; case T_xsa: return "XSA-I"; default: return "@"; }
	}
	return t <= T_max ? tags[t] : "@";
}
static const char16_t* tagNameW(uint8_t t)
{
	static thread_local std::u16string buf[4]; static thread_local int rot = 0;
	const char* s = tagName(t);
	auto& b = buf[rot++ & 3];
	b.assign(s, s + std::strlen(s));
	return b.c_str();
}

// bytePositions (optional): the byte offset of the character every UTF-16 unit belongs to, + the length (utf8To16, src/StrUtils.h:236-300)
static std::u16string utf8To16(const char* s, std::vector<uint32_t>* bytePositions = nullptr)
{
	std::u16string out;
	const size_t n = std::strlen(s);
	for (size_t i = 0; i < n;)
	{
		uint32_t c = (uint8_t)s[i]; size_t k = 1;
		if (c >= 0xF0) { c &= 7; k = 4; } else if (c >= 0xE0) { c &= 15; k = 3; } else if (c >= 0xC0) { c &= 31; k = 2; }
		for (size_t j = 1; j < k && i + j < n; ++j) c = (c << 6) | ((uint8_t)s[i + j] & 63);
		if (bytePositions) bytePositions->insert(bytePositions->end(), c >= 0x10000 ? 2 : 1, (uint32_t)i);
		i += k;
		if (c >= 0x10000) { c -= 0x10000; out.push_back((char16_t)(0xD800 | (c >> 10))); out.push_back((char16_t)(0xDC00 | (c & 0x3FF))); }
		else out.push_back((char16_t)c);
	}
	if (bytePositions) bytePositions->push_back((uint32_t)n);
	return out;
}
static std::string utf16To8(const std::u16string& s)
{
	std::string out;
	for (size_t i = 0; i < s.size(); ++i)
	{
		uint32_t c = s[i];
		if ((c & 0xFC00) == 0xD800 && i + 1 < s.size()) { c = (((c & 0x3FF) << 10) | (s[i + 1] & 0x3FF)) + 0x10000; ++i; }
		if (c < 0x80) out.push_back((char)c);
		else if (c < 0x800) { out.push_back((char)(0xC0 | (c >> 6))); out.push_back((char)(0x80 | (c & 63))); }
		else if (c < 0x10000) { out.push_back((char)(0xE0 | (c >> 12))); out.push_back((char)(0x80 | ((c >> 6) & 63))); out.push_back((char)(0x80 | (c & 63))); }
		else { out.push_back((char)(0xF0 | (c >> 18))); out.push_back((char)(0x80 | ((c >> 12) & 63))); out.push_back((char)(0x80 | ((c >> 6) & 63))); out.push_back((char)(0x80 | (c & 63))); }
	}
	return out;
}
// the kernels' option word: the reference's Match bits (include/kiwi/Types.h) + bit 31 = AnalyzeOption::openEnding (no Match flag lives there)
static uint32_t optionWord(const kiwi_analyze_option_t& o) { return ((uint32_t)o.match_options & 0x7FFFFFFFu) | (o.open_ending ? 0x80000000u : 0u); }

// joins: the call honours the token-joining options (join*, mergeSaisiot, joinParticleYo) and compatibleJamo - the analysis calls do; the
// sentence splitter and the device-resident call refuse them
static void checkOption(const kiwi_analyze_option_t& o, int topN, kiwi_pretokenized_h pt, bool joins = false)
{
	if (topN != 1) throw std::invalid_argument("kiwi_b200 implements the top_n == 1 path only");
	if (o.allowed_dialects) throw std::invalid_argument("dialects other than standard are outside the kiwi_b200 hot path");
	if (pt) throw std::invalid_argument("pretokenized spans are outside the kiwi_b200 hot path");
	const uint32_t joinBits = MO_JOIN_ANY | MO_COMPATIBLE_JAMO;
	const uint32_t unsupported = (3u << 8) | (1u << 30) | (joins ? 0u : joinBits);
	if ((uint32_t)o.match_options & unsupported)
		throw std::invalid_argument(joins ? "match_options contain a flag outside the kiwi_b200 hot path (oov models, useOldSplitter)"
			: "match_options contain a flag outside the kiwi_b200 hot path (oov models, join*, compatibleJamo, mergeSaisiot, useOldSplitter)");
}

static kiwi_res* makeRes(kiwi_s* h, const uint16_t* text, uint32_t rawLen, const BatchOutput& bo, uint32_t idx, uint32_t matchOptions)
{
	auto* r = new kiwi_res;
	r->score = bo.scores[idx];
	const Model& m = h->engine->model;
	const uint32_t t0 = bo.tokOff[idx], n = bo.tokOff[idx + 1] - t0;
	std::vector<ResTok> rt = assembleRows(m.hMorphs, m.hForms, m.hFormChars, m.hChrBmp.data(), text, rawLen, bo.tokens.data() + t0, n, bo.forms.data(), bo.forms.size(), matchOptions);
	r->toks.resize(n);
	for (uint32_t t = 0; t < n; ++t)
	{
		const DToken& d = bo.tokens[t0 + t];
		const AsmTok& a = rt[t].a;
		kiwi_res::Tok& k = r->toks[t];
		std::memset(&k.info, 0, sizeof(k.info));
		k.info.chr_position = d.position; k.info.length = d.length; k.info.tag = d.tag; k.info.score = d.score;
		// TokenInfo::typoCost (src/Kiwi.cpp:739) = node cost / tokens of the node (PathEvaluator.hpp:1074), both in the device row's flags
		k.info.typo_cost = ((d.flags >> 1) & 7) ? (float)((d.flags >> 1) & 7) * 0.5f / (float)((d.flags >> 4) + 1) : 0.f;
		k.info.sense_id = rt[t].senseId; k.info.dialect = rt[t].dialect;
		k.info.word_position = a.wordPosition; k.info.sent_position = a.sentPosition; k.info.line_number = a.lineNumber;
		k.info.sub_sent_position = a.subSentPosition; k.info.paired_token = a.pairedToken;
		k.morphId = rt[t].morphId;
		k.form = a.form;
		k.form8 = utf16To8(k.form);
	}
	return r;
}

// One batch through the handle's engine(s).  With several devices (kiwi_b200_init_multi) sentence i goes to device i mod N
// (BASELINE.json config 5); one host thread per device gathers its shard, runs it, and scatters its rows back into the batch's
// output arrays in input order - the reference's ordered delivery (include/kiwi/Kiwi.h:402-454) without a collective.
// `outputs` (OUT_*): the token rows and / or the sentence ranges (kiwi_split_into_sents, kiwi_b200_split_batch), merged alike.
static void analyzeSharded(kiwi_s* h, const uint16_t* text, const uint32_t* offsets, uint32_t n, const kiwi_analyze_option_t& option, BatchOutput& out,
	uint32_t outputs = OUT_TOKENS)
{
	const uint32_t N = 1 + (uint32_t)h->extra.size();
	if (N == 1 || n < 2 * N)
	{
		TypoScope ts{ h->engine.get(), option };
		BlockScope bs{ h->engine.get(), option };
		h->engine->analyze(text, offsets, n, optionWord(option), out, outputs);
		return;
	}
	if (h->shardOut.size() != N) h->shardOut.resize(N);
	std::vector<BatchOutput>& part = h->shardOut;
	std::vector<std::string> errors(N);
	static const bool trace = std::getenv("KIWI_B200_TRACE") != nullptr;      // stderr: where the host time of a sharded batch goes
	using Clock = std::chrono::steady_clock;
	const auto tStart = Clock::now();
	std::vector<double> msGather(N, 0.0), msEngine(N, 0.0);
	std::vector<Stats> stats(N);
	auto work = [&](uint32_t r)
	{
		try
		{
			Engine* e = r == 0 ? h->engine.get() : h->extra[r - 1].get();
			const auto t0 = Clock::now();
			std::vector<uint16_t> sub; std::vector<uint32_t> off{ 0 };
			size_t units = 0;
			for (uint32_t i = r; i < n; i += N) units += offsets[i + 1] - offsets[i];
			sub.reserve(units); off.reserve(n / N + 2);
			for (uint32_t i = r; i < n; i += N) { sub.insert(sub.end(), text + offsets[i], text + offsets[i + 1]); off.push_back((uint32_t)sub.size()); }
			const auto t1 = Clock::now();
			TypoScope ts{ e, option };
			BlockScope bs{ e, option };
			e->analyze(sub.data(), off.data(), (uint32_t)off.size() - 1, optionWord(option), part[r], outputs);
			stats[r] = e->last;
			msGather[r] = std::chrono::duration<double, std::milli>(t1 - t0).count();
			msEngine[r] = std::chrono::duration<double, std::milli>(Clock::now() - t1).count();
		}
		catch (const std::exception& ex) { errors[r] = ex.what(); if (errors[r].empty()) errors[r] = "error"; }
	};
	std::vector<std::thread> th;
	for (uint32_t r = 1; r < N; ++r) th.emplace_back(work, r);
	work(0);
	for (auto& t : th) t.join();
	for (auto& e : errors) if (!e.empty()) throw std::runtime_error(e);
	// ordered merge: token offsets by prefix sum over the round-robin order, then every shard scatters its rows
	// (`out` may be a recycled holder: its arrays keep their capacity)
	const auto tMerge = Clock::now();
	out.msH2D = out.msLattice = out.msViterbi = out.msPack = out.msSents = out.msD2H = out.msTotal = 0;
	out.tokens.clear();
	out.tokOff.assign((size_t)n + 1, 0); out.scores.resize(n); out.status.resize(n);
	// joined forms: the shards' arrays one after the other; a shard's joined rows move by the forms in front of its own
	std::vector<uint32_t> formBase(N, 0);
	out.forms.clear();
	for (uint32_t r = 0; r < N; ++r) { formBase[r] = (uint32_t)out.forms.size(); out.forms.insert(out.forms.end(), part[r].forms.begin(), part[r].forms.end()); }
	const bool sents = (outputs & OUT_SENTS) != 0;
	out.sentOff.assign(sents ? (size_t)n + 1 : 0, 0);
	for (uint32_t i = 0; i < n; ++i)
	{
		const BatchOutput& p = part[i % N]; const uint32_t k = i / N;
		out.tokOff[i + 1] = out.tokOff[i] + (p.tokOff[k + 1] - p.tokOff[k]);
		out.scores[i] = p.scores[k]; out.status[i] = p.status[k];
		if (sents) out.sentOff[i + 1] = out.sentOff[i] + (p.sentOff[k + 1] - p.sentOff[k]);
	}
	out.tokens.resize(out.tokOff[n]);
	out.sentBegin.resize(sents ? out.sentOff[n] : 0); out.sentEnd.resize(sents ? out.sentOff[n] : 0);
	auto scatter = [&](uint32_t r)
	{
		const BatchOutput& p = part[r];
		for (uint32_t i = r, k = 0; i < n; i += N, ++k)
		{
			const uint32_t cnt = p.tokOff[k + 1] - p.tokOff[k];
			if (cnt) std::memcpy(out.tokens.data() + out.tokOff[i], p.tokens.data() + p.tokOff[k], (size_t)cnt * sizeof(DToken));
			if (formBase[r]) for (uint32_t t = out.tokOff[i]; t < out.tokOff[i] + cnt; ++t) if (out.tokens[t].morph & JOINED_TOKEN) out.tokens[t].morph += formBase[r];
			if (!sents) continue;
			const uint32_t ns = p.sentOff[k + 1] - p.sentOff[k];
			std::copy_n(p.sentBegin.data() + p.sentOff[k], ns, out.sentBegin.data() + out.sentOff[i]);
			std::copy_n(p.sentEnd.data() + p.sentOff[k], ns, out.sentEnd.data() + out.sentOff[i]);
		}
	};
	th.clear();
	for (uint32_t r = 1; r < N; ++r) th.emplace_back(scatter, r);
	scatter(0);
	for (auto& t : th) t.join();
	Stats agg{};
	for (uint32_t r = 0; r < N; ++r)
	{
		const BatchOutput& p = part[r];
		out.msH2D = std::max(out.msH2D, p.msH2D); out.msLattice = std::max(out.msLattice, p.msLattice); out.msViterbi = std::max(out.msViterbi, p.msViterbi);
		out.msPack = std::max(out.msPack, p.msPack); out.msSents = std::max(out.msSents, p.msSents); out.msD2H = std::max(out.msD2H, p.msD2H); out.msTotal = std::max(out.msTotal, p.msTotal);
		agg.h2dBytes += stats[r].h2dBytes; agg.d2hBytes += stats[r].d2hBytes; agg.kernelLaunches += stats[r].kernelLaunches; agg.retried += stats[r].retried;
		agg.rawUnits += stats[r].rawUnits;
	}
	agg.nSentences = n; agg.tokens = out.tokens.size(); agg.msLattice = out.msLattice; agg.msViterbi = out.msViterbi; agg.msPack = out.msPack;
	h->engine->last = agg;
	if (trace)
	{
		const double msAll = std::chrono::duration<double, std::milli>(Clock::now() - tStart).count(), msM = std::chrono::duration<double, std::milli>(Clock::now() - tMerge).count();
		std::fprintf(stderr, "[kiwi_b200] sharded batch n=%u devices=%u: total %.1f ms, merge %.1f ms, per device gather/engine/device-busy ms:", n, N, msAll, msM);
		for (uint32_t r = 0; r < N; ++r) std::fprintf(stderr, " %.1f/%.1f/%.1f", msGather[r], msEngine[r], part[r].msTotal);
		std::fprintf(stderr, "\n");
	}
}

// Drains the reader into batches (the reference primes pool->size()*2 futures, include/kiwi/Kiwi.h:402-454);
// results are delivered to the receiver in input order, which owns and closes them (kiwi_c.cpp:932-936).
template<class ReadFn>
static int analyzeMulti(kiwi_h handle, ReadFn&& readOne, kiwi_receiver_t receiver, void* user_data, int top_n, kiwi_analyze_option_t option)
{
	if (!handle) return KIWIERR_INVALID_HANDLE;
	try
	{
		checkOption(option, top_n, nullptr, true);
		const size_t maxBatch = 65536, maxUnits = 16u << 20;
		int idx = 0, delivered = 0;
		bool done = false;
		BatchOutput bo;      // (page-locked token array: one per call, reused by every batch of it)
		while (!done)
		{
			std::vector<uint16_t> text; std::vector<uint32_t> off{ 0 };
			while (off.size() - 1 < maxBatch && text.size() < maxUnits)
			{
				std::u16string s;
				if (!readOne(idx, s)) { done = true; break; }
				++idx;
				text.insert(text.end(), s.begin(), s.end());
				off.push_back((uint32_t)text.size());
			}
			const uint32_t n = (uint32_t)off.size() - 1;
			if (!n) break;
			{
				std::lock_guard<std::mutex> lk(handle->mtx);
				analyzeSharded(handle, text.data(), off.data(), n, option, bo);
			}
			for (uint32_t i = 0; i < n; ++i)
			{
				kiwi_res* r = makeRes(handle, text.data() + off[i], off[i + 1] - off[i], bo, i, (uint32_t)option.match_options);
				// positions are relative to the sentence already (each sentence has its own position table)
				(*receiver)(delivered++, r, user_data);
			}
		}
		return delivered;
	}
	catch (const std::exception& e) { setError(e); return KIWIERR_FAIL; }
}


// result buffers of kiwi_b200_analyze_batch are recycled (a 5 MB allocation + first-touch page faults per 8192-sentence call otherwise);
// the pool outlives the handle for batches the caller frees late
struct BatchHolder;
struct BatchPool
{
	std::mutex m; std::vector<BatchHolder*> free; bool closed = false;
	~BatchPool();
};
struct BatchHolder { kiwi_b200_batch_t pub; BatchOutput bo; std::shared_ptr<BatchPool> pool; };
BatchPool::~BatchPool() { for (auto* h : free) delete h; }
static std::mutex g_poolMapMtx;
static std::map<kiwi_s*, std::shared_ptr<BatchPool>> g_pools;
static std::shared_ptr<BatchPool> poolOf(kiwi_s* h)
{
	std::lock_guard<std::mutex> lk(g_poolMapMtx);
	auto& p = g_pools[h];
	if (!p) p = std::make_shared<BatchPool>();
	return p;
}


extern "C" {
#pragma GCC visibility push(default)

const char* kiwi_version(void) { return "0.23.1-b200.1"; }
const char* kiwi_error(void) { return g_hasError ? g_error.c_str() : nullptr; }
void kiwi_clear_error(void) { g_hasError = false; g_error.clear(); }

int kiwi_b200_device_count(void) { int n = 0; if (cudaGetDeviceCount(&n) != cudaSuccess) return 0; return n; }
int kiwi_b200_set_device(int device) { g_device = device; return 0; }

int kiwi_b200_read_image(const char* model_path, void** out_bytes, uint64_t* out_size)
{
	try
	{
		auto blob = readImageFile(model_path);
		void* p = std::malloc(blob.size());
		if (!p) throw std::bad_alloc();
		std::memcpy(p, blob.data(), blob.size());
		*out_bytes = p; *out_size = blob.size();
		return 0;
	}
	catch (const std::exception& e) { setError(e); return KIWIERR_FAIL; }
}
void kiwi_b200_free(void* p) { std::free(p); }

kiwi_h kiwi_b200_init_from_image(const void* bytes, uint64_t size)
{
	try
	{
		int n = 0;
		if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) throw std::runtime_error("kiwi_b200 needs a CUDA device (sm_90a); there is no CPU fallback");
		if (g_device >= 0 && cudaSetDevice(g_device) != cudaSuccess) throw std::runtime_error("cudaSetDevice failed");
		auto* h = new kiwi_s;
		h->engine.reset(new Engine(bytes, size));
		return h;
	}
	catch (const std::exception& e) { setError(e); return nullptr; }
}

kiwi_h kiwi_b200_init_multi(const void* bytes, uint64_t size, const int* devices, int n_devices)
{
	try
	{
		int n = 0;
		if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) throw std::runtime_error("kiwi_b200 needs a CUDA device (sm_90a); there is no CPU fallback");
		if (n_devices < 1) throw std::invalid_argument("kiwi_b200_init_multi: n_devices < 1");
		for (int i = 0; i < n_devices; ++i) if (devices[i] < 0 || devices[i] >= n) throw std::invalid_argument("kiwi_b200_init_multi: no such device");
		auto h = std::unique_ptr<kiwi_s>(new kiwi_s);
		int prev = 0; cudaGetDevice(&prev);
		// one resident copy of the read-only model per device; the copies are made concurrently (one host thread per device)
		std::vector<std::unique_ptr<Engine>> eng((size_t)n_devices);
		std::vector<std::string> errors((size_t)n_devices);
		std::vector<std::thread> th;
		for (int i = 0; i < n_devices; ++i) th.emplace_back([&, i]
		{
			try { if (cudaSetDevice(devices[i]) != cudaSuccess) throw std::runtime_error("cudaSetDevice failed"); eng[i].reset(new Engine(bytes, size)); }
			catch (const std::exception& e) { errors[i] = e.what(); }
		});
		for (auto& t : th) t.join();
		cudaSetDevice(prev);
		for (auto& e : errors) if (!e.empty()) throw std::runtime_error(e);
		h->engine = std::move(eng[0]);
		for (int i = 1; i < n_devices; ++i) h->extra.push_back(std::move(eng[i]));
		return h.release();
	}
	catch (const std::exception& e) { setError(e); return nullptr; }
}

int kiwi_b200_num_devices(kiwi_h handle) { return handle ? 1 + (int)handle->extra.size() : KIWIERR_INVALID_HANDLE; }

kiwi_h kiwi_init(const char* model_path, int num_threads, int options, int enabled_dialects)
{
	(void)options; (void)enabled_dialects;
	try
	{
		auto blob = readImageFile(model_path);
		kiwi_h h = kiwi_b200_init_from_image(blob.data(), blob.size());
		if (h) h->numThreads = num_threads;
		if (h)
		{
			// typo_<set>.img files are looked up next to the model image (or inside the model directory)
			std::string p = model_path;
			FILE* probe = std::fopen((p + "/kiwi_b200.img").c_str(), "rb");
			if (probe) std::fclose(probe);
			else { const size_t sl = p.find_last_of('/'); p = sl == std::string::npos ? "." : p.substr(0, sl); }
			g_typoDir = p;
		}
		return h;
	}
	catch (const std::exception& e) { setError(e); return nullptr; }
}

// ---- typo transformers (capi.h:469-588, the subset the analysis option needs) -------------------------------------
kiwi_typo_h kiwi_typo_get_default(int kiwi_typo_set)
{
	if (kiwi_typo_set < 0 || kiwi_typo_set > 6) { setError("kiwi_typo_get_default: unknown typo set"); return nullptr; }
	return &g_defaultTypos[kiwi_typo_set];
}

kiwi_typo_h kiwi_typo_get_basic() { return &g_defaultTypos[1]; }

int kiwi_typo_close(kiwi_typo_h handle)
{
	if (!handle) return KIWIERR_INVALID_HANDLE;
	if (handle >= g_defaultTypos && handle < g_defaultTypos + 7) { setError("default typo sets must not be closed"); return KIWIERR_FAIL; }
	return KIWIERR_INVALID_HANDLE;      // no other kiwi_typo is ever created by this build
}

kiwi_prepared_typo_h kiwi_b200_typo_from_image(const void* bytes, size_t size)
{
	try
	{
		auto* t = new kiwi_prepared_typo;
		try
		{
			t->blob.assign(reinterpret_cast<const char*>(bytes), reinterpret_cast<const char*>(bytes) + size);
			int dev = 0;
			if (g_device >= 0) dev = g_device; else cudaGetDevice(&dev);
			t->forDevice(dev);      // validates the image and makes it resident on the current device
		}
		catch (...) { delete t; throw; }
		return t;
	}
	catch (const std::exception& e) { setError(e); return nullptr; }
}

kiwi_prepared_typo_h kiwi_b200_typo_load(const char* path)
{
	try
	{
		FILE* f = std::fopen(path, "rb");
		if (!f) throw std::runtime_error(std::string("cannot open typo image '") + path + "'");
		std::fseek(f, 0, SEEK_END); const long n = std::ftell(f); std::fseek(f, 0, SEEK_SET);
		std::vector<char> blob((size_t)std::max(n, 0l));
		const bool ok = std::fread(blob.data(), 1, blob.size(), f) == blob.size();
		std::fclose(f);
		if (!ok) throw std::runtime_error(std::string("short read on ") + path);
		return kiwi_b200_typo_from_image(blob.data(), blob.size());
	}
	catch (const std::exception& e) { setError(e); return nullptr; }
}

kiwi_prepared_typo_h kiwi_typo_prepare(kiwi_typo_h handle)
{
	if (!handle) { setError("invalid handle"); return nullptr; }
	static const char* names[7] = { "none", "basic", "continual", "basic_continual", "lengthening", "basic_continual_lengthening", "dialect" };
	const char* env = std::getenv("KIWI_B200_TYPO_DIR");
	const std::string dir = env ? env : g_typoDir;
	if (dir.empty()) { setError("kiwi_typo_prepare: open a model with kiwi_init first or set KIWI_B200_TYPO_DIR (typo_<set>.img is looked up there)"); return nullptr; }
	return kiwi_b200_typo_load((dir + "/typo_" + names[handle->set] + ".img").c_str());
}

int kiwi_prepared_typo_close(kiwi_prepared_typo_h handle)
{
	if (!handle) return KIWIERR_INVALID_HANDLE;
	delete handle;
	return 0;
}

// POSTag names (include/kiwi/Types.h:39-93, toPOSTag in src/TagUtils.cpp): the index is the enum value; "-I" marks the irregular variants
static uint8_t parseTag(const char* tag)
{
	static const char* names[] = { "UN", "NNG", "NNP", "NNB", "VV", "VA", "MAG", "NR", "NP", "VX", "MM", "MAJ", "IC", "XPN", "XSN", "XSV", "XSA", "XSM", "XR",
		"VCP", "VCN", "SF", "SP", "SS", "SSO", "SSC", "SE", "SO", "SW", "SB", "SL", "SH", "SN", "W_URL", "W_EMAIL", "W_MENTION", "W_HASHTAG", "W_SERIAL", "W_EMOJI",
		"JKS", "JKC", "JKG", "JKO", "JKB", "JKV", "JKQ", "JX", "JC", "EP", "EF", "EC", "ETN", "ETM", "Z_CODA", "Z_SIOT", "USER0", "USER1", "USER2", "USER3", "USER4", "P" };
	if (!tag) return 0;
	std::string t{ tag };
	for (auto& c : t) c = (char)std::toupper((unsigned char)c);
	bool irregular = false;
	if (t.size() > 2 && t.compare(t.size() - 2, 2, "-I") == 0) { irregular = true; t.resize(t.size() - 2); }
	for (size_t i = 0; i < sizeof(names) / sizeof(names[0]); ++i) if (t == names[i]) return (uint8_t)(i | (irregular ? 0x80 : 0));
	throw std::invalid_argument(std::string{ "Unknown POSTag : " } + tag);
}

kiwi_morphset_h kiwi_new_morphset(kiwi_h handle)
{
	if (!handle) return nullptr;
	try { auto* s = new kiwi_morphset; s->inst = handle; return s; }
	catch (const std::exception& e) { setError(e); return nullptr; }
}

int kiwi_morphset_add_w(kiwi_morphset_h handle, const kchar16_t* form, const char* tag)
{
	if (!handle) return KIWIERR_INVALID_HANDLE;
	try
	{
		size_t len = 0; while (form[len]) ++len;
		const std::vector<uint32_t> found = handle->inst->engine->model.findMorphemes(reinterpret_cast<const uint16_t*>(form), len, parseTag(tag));
		std::lock_guard<std::mutex> lk(handle->m);
		handle->ids.insert(handle->ids.end(), found.begin(), found.end());
		std::sort(handle->ids.begin(), handle->ids.end());
		handle->ids.erase(std::unique(handle->ids.begin(), handle->ids.end()), handle->ids.end());
		++handle->version;
		return (int)found.size();
	}
	catch (const std::exception& e) { setError(e); return KIWIERR_FAIL; }
}

int kiwi_morphset_add(kiwi_morphset_h handle, const char* form, const char* tag)
{
	if (!handle) return KIWIERR_INVALID_HANDLE;
	try
	{
		const std::u16string w = utf8To16(form);
		return kiwi_morphset_add_w(handle, reinterpret_cast<const kchar16_t*>(w.c_str()), tag);
	}
	catch (const std::exception& e) { setError(e); return KIWIERR_FAIL; }
}

int kiwi_morphset_close(kiwi_morphset_h handle)
{
	if (!handle) return KIWIERR_INVALID_HANDLE;
	delete handle;
	return 0;
}

int kiwi_b200_image_find_morphemes(const void* image_bytes, uint64_t size, const kchar16_t* form, const char* tag, uint32_t* out_ids, int cap)
{
	try
	{
		// host-side view of the image only: the sections findMorphemes reads (no device, no derived tables)
		if (size < sizeof(kb2_header)) throw std::runtime_error("model image too small");
		Model m;
		m.blob.assign(static_cast<const char*>(image_bytes), static_cast<const char*>(image_bytes) + size);
		std::memcpy(&m.header, m.blob.data(), sizeof(kb2_header));
		if (m.header.magic != KB2_IMAGE_MAGIC || m.header.total_bytes != size) throw std::runtime_error("not a kiwi_b200 model image");
		m.hForms = reinterpret_cast<const kb2_form*>(m.blob.data() + m.header.sec[KB2_SEC_FORMS].offset);
		m.hFormChars = reinterpret_cast<const uint16_t*>(m.blob.data() + m.header.sec[KB2_SEC_FORM_CHARS].offset);
		m.hMorphs = reinterpret_cast<const kb2_morph*>(m.blob.data() + m.header.sec[KB2_SEC_MORPHS].offset);
		size_t len = 0; while (form[len]) ++len;
		const std::vector<uint32_t> found = m.findMorphemes(reinterpret_cast<const uint16_t*>(form), len, parseTag(tag));
		for (size_t i = 0; i < found.size() && (int)i < cap; ++i) out_ids[i] = found[i];
		return (int)found.size();
	}
	catch (const std::exception& e) { setError(e); return -1; }
}

int kiwi_close(kiwi_h handle)
{
	if (!handle) return KIWIERR_INVALID_HANDLE;
	{
		std::shared_ptr<BatchPool> pool;
		{ std::lock_guard<std::mutex> lk(g_poolMapMtx); auto it = g_pools.find(handle); if (it != g_pools.end()) { pool = it->second; g_pools.erase(it); } }
		if (pool) { std::lock_guard<std::mutex> lk(pool->m); pool->closed = true; for (auto* h : pool->free) delete h; pool->free.clear(); }
	}
	try { delete handle; return 0; }
	catch (const std::exception& e) { setError(e); return KIWIERR_FAIL; }
}

kiwi_res_h kiwi_analyze_w(kiwi_h handle, const kchar16_t* text, int top_n, kiwi_analyze_option_t option, kiwi_pretokenized_h pretokenized)
{
	if (!handle) return nullptr;
	try
	{
		checkOption(option, top_n, pretokenized, true);
		uint32_t len = 0;
		while (text[len]) ++len;
		const uint32_t off[2] = { 0, len };
		std::lock_guard<std::mutex> lk(handle->mtx);
		BatchOutput& bo = handle->callOut;
		TypoScope ts{ handle->engine.get(), option };
		BlockScope bs{ handle->engine.get(), option };
		handle->engine->analyze(text, off, 1, optionWord(option), bo);
		return makeRes(handle, text, len, bo, 0, (uint32_t)option.match_options);
	}
	catch (const std::exception& e) { setError(e); return nullptr; }
}

kiwi_res_h kiwi_analyze(kiwi_h handle, const char* text, int top_n, kiwi_analyze_option_t option, kiwi_pretokenized_h pretokenized)
{
	if (!handle) return nullptr;
	try
	{
		const std::u16string w = utf8To16(text);
		// NB: positions are reported in UTF-16 units of the converted text, as the reference does for its internal string
		return kiwi_analyze_w(handle, reinterpret_cast<const kchar16_t*>(w.c_str()), top_n, option, pretokenized);
	}
	catch (const std::exception& e) { setError(e); return nullptr; }
}

int kiwi_analyze_mw(kiwi_h handle, kiwi_reader_w_t reader, kiwi_receiver_t receiver, void* user_data, int top_n, kiwi_analyze_option_t option)
{
	return analyzeMulti(handle, [&](int idx, std::u16string& s)
	{
		const int len = (*reader)(idx, nullptr, user_data);        // kiwi_c.cpp:924-931
		if (len <= 0) return false;
		s.resize((size_t)len);
		(*reader)(idx, reinterpret_cast<kchar16_t*>(&s[0]), user_data);
		return true;
	}, receiver, user_data, top_n, option);
}

int kiwi_analyze_m(kiwi_h handle, kiwi_reader_t reader, kiwi_receiver_t receiver, void* user_data, int top_n, kiwi_analyze_option_t option)
{
	return analyzeMulti(handle, [&](int idx, std::u16string& s)
	{
		const int len = (*reader)(idx, nullptr, user_data);
		if (len <= 0) return false;
		std::string buf((size_t)len, '\0');
		(*reader)(idx, &buf[0], user_data);
		s = utf8To16(buf.c_str());
		return true;
	}, receiver, user_data, top_n, option);
}

int kiwi_res_size(kiwi_res_h result) { if (!result) return KIWIERR_INVALID_HANDLE; return 1; }
float kiwi_res_prob(kiwi_res_h result, int index) { if (!result || index != 0) return 0; return result->score; }
int kiwi_res_word_num(kiwi_res_h result, int index) { if (!result) return KIWIERR_INVALID_HANDLE; if (index != 0) return KIWIERR_INVALID_INDEX; return (int)result->toks.size(); }
#define KB_TOK_OR(ret) if (!result) return ret; if (index != 0 || num < 0 || num >= (int)result->toks.size()) return ret;
const kiwi_token_info_t* kiwi_res_token_info(kiwi_res_h result, int index, int num) { KB_TOK_OR(nullptr) return &result->toks[num].info; }
int kiwi_res_morpheme_id(kiwi_res_h result, int index, int num, kiwi_h kiwi_handle) { (void)kiwi_handle; KB_TOK_OR(KIWIERR_INVALID_INDEX) return (int)result->toks[num].morphId; }
const kchar16_t* kiwi_res_form_w(kiwi_res_h result, int index, int num) { KB_TOK_OR(nullptr) return reinterpret_cast<const kchar16_t*>(result->toks[num].form.c_str()); }
const kchar16_t* kiwi_res_tag_w(kiwi_res_h result, int index, int num) { KB_TOK_OR(nullptr) return reinterpret_cast<const kchar16_t*>(tagNameW(result->toks[num].info.tag)); }
const char* kiwi_res_form(kiwi_res_h result, int index, int num) { KB_TOK_OR(nullptr) return result->toks[num].form8.c_str(); }
const char* kiwi_res_tag(kiwi_res_h result, int index, int num) { KB_TOK_OR(nullptr) return tagName(result->toks[num].info.tag); }
int kiwi_res_position(kiwi_res_h result, int index, int num) { KB_TOK_OR(KIWIERR_INVALID_INDEX) return (int)result->toks[num].info.chr_position; }
int kiwi_res_length(kiwi_res_h result, int index, int num) { KB_TOK_OR(KIWIERR_INVALID_INDEX) return (int)result->toks[num].info.length; }
int kiwi_res_word_position(kiwi_res_h result, int index, int num) { KB_TOK_OR(KIWIERR_INVALID_INDEX) return (int)result->toks[num].info.word_position; }
int kiwi_res_sent_position(kiwi_res_h result, int index, int num) { KB_TOK_OR(KIWIERR_INVALID_INDEX) return (int)result->toks[num].info.sent_position; }
float kiwi_res_score(kiwi_res_h result, int index, int num) { KB_TOK_OR(0.f) return result->toks[num].info.score; }
float kiwi_res_typo_cost(kiwi_res_h result, int index, int num) { KB_TOK_OR(0.f) return result->toks[num].info.typo_cost; }
int kiwi_res_close(kiwi_res_h result) { if (!result) return KIWIERR_INVALID_HANDLE; delete result; return 0; }

// ---- sentence splitting (Kiwi::splitIntoSents): one engine call brings the ranges and, for tokenized_res, the token rows ----
kiwi_ss_h kiwi_split_into_sents_w(kiwi_h handle, const kchar16_t* text, int match_options, kiwi_res_h* tokenized_res)
{
	if (!handle) return nullptr;
	try
	{
		kiwi_analyze_option_t option{};
		option.match_options = match_options;
		checkOption(option, 1, nullptr);
		uint32_t len = 0;
		while (text[len]) ++len;
		const uint32_t off[2] = { 0, len };
		std::lock_guard<std::mutex> lk(handle->mtx);
		BatchOutput& bo = handle->callOut;
		analyzeSharded(handle, text, off, 1, option, bo, OUT_SENTS | (tokenized_res ? OUT_TOKENS : 0));
		auto ss = std::make_unique<kiwi_ss>();
		for (uint32_t k = bo.sentOff[0]; k < bo.sentOff[1]; ++k) ss->ranges.emplace_back(bo.sentBegin[k], bo.sentEnd[k]);
		if (tokenized_res) *tokenized_res = makeRes(handle, text, len, bo, 0, (uint32_t)match_options);
		return ss.release();
	}
	catch (const std::exception& e) { setError(e); return nullptr; }
}

kiwi_ss_h kiwi_split_into_sents(kiwi_h handle, const char* text, int match_options, kiwi_res_h* tokenized_res)
{
	if (!handle) return nullptr;
	try
	{
		std::vector<uint32_t> bytePositions;
		const std::u16string w = utf8To16(text, &bytePositions);
		kiwi_ss_h ss = kiwi_split_into_sents_w(handle, reinterpret_cast<const kchar16_t*>(w.c_str()), match_options, tokenized_res);
		if (ss) for (auto& r : ss->ranges) { r.first = bytePositions[r.first]; r.second = bytePositions[r.second]; }      // (Kiwi.cpp:438-450)
		return ss;
	}
	catch (const std::exception& e) { setError(e); return nullptr; }
}

int kiwi_ss_size(kiwi_ss_h result) { if (!result) return KIWIERR_INVALID_HANDLE; return (int)result->ranges.size(); }
int kiwi_ss_begin_position(kiwi_ss_h result, int index)
{
	if (!result) return KIWIERR_INVALID_HANDLE;
	if (index < 0 || index >= (int)result->ranges.size()) return KIWIERR_INVALID_INDEX;
	return (int)result->ranges[index].first;
}
int kiwi_ss_end_position(kiwi_ss_h result, int index)
{
	if (!result) return KIWIERR_INVALID_HANDLE;
	if (index < 0 || index >= (int)result->ranges.size()) return KIWIERR_INVALID_INDEX;
	return (int)result->ranges[index].second;
}
int kiwi_ss_close(kiwi_ss_h result) { if (!result) return KIWIERR_INVALID_HANDLE; delete result; return 0; }

const kiwi_b200_batch_t* kiwi_b200_analyze_batch(kiwi_h handle, const kchar16_t* text, const uint32_t* offsets, int n, kiwi_analyze_option_t option)
{
	if (!handle) { setError("invalid handle"); return nullptr; }
	try
	{
		checkOption(option, 1, nullptr, true);
		if (n < 0) throw std::invalid_argument("n < 0");
		auto pool = poolOf(handle);
		BatchHolder* h = nullptr;
		{
			std::lock_guard<std::mutex> lk(pool->m);
			if (!pool->free.empty()) { h = pool->free.back(); pool->free.pop_back(); }
		}
		if (!h) h = new BatchHolder;
		h->pool = pool;
		try
		{
			std::lock_guard<std::mutex> lk(handle->mtx);
			analyzeSharded(handle, text, offsets, (uint32_t)n, option, h->bo);
		}
		catch (...) { delete h; throw; }
		static_assert(sizeof(kiwi_b200_token_t) == sizeof(DToken), "token layout");
		h->pub.n_sentences = n;
		h->pub.token_offsets = h->bo.tokOff.data();
		h->pub.tokens = reinterpret_cast<const kiwi_b200_token_t*>(h->bo.tokens.data());
		h->pub.scores = h->bo.scores.data();
		h->pub.status = h->bo.status.data();
		h->pub.ms_h2d = h->bo.msH2D; h->pub.ms_lattice = h->bo.msLattice; h->pub.ms_viterbi = h->bo.msViterbi; h->pub.ms_pack = h->bo.msPack;
		h->pub.ms_d2h = h->bo.msD2H; h->pub.ms_total = h->bo.msTotal;
		h->pub.forms = (option.match_options & MO_JOIN_ANY) && !h->bo.forms.empty() ? reinterpret_cast<const kchar16_t*>(h->bo.forms.data()) : nullptr;
		h->pub.forms_size = (uint32_t)h->bo.forms.size();
		return &h->pub;
	}
	catch (const std::exception& e) { setError(e); return nullptr; }
}

struct SentsHolder { kiwi_b200_sents_t pub; BatchOutput bo; };

const kiwi_b200_sents_t* kiwi_b200_split_batch(kiwi_h handle, const kchar16_t* text, const uint32_t* offsets, int n, int match_options)
{
	if (!handle) { setError("invalid handle"); return nullptr; }
	try
	{
		kiwi_analyze_option_t option{};
		option.match_options = match_options;
		checkOption(option, 1, nullptr);
		if (n < 0) throw std::invalid_argument("n < 0");
		auto h = std::make_unique<SentsHolder>();
		{
			std::lock_guard<std::mutex> lk(handle->mtx);
			analyzeSharded(handle, text, offsets, (uint32_t)n, option, h->bo, OUT_SENTS);
		}
		h->pub.n_docs = n;
		h->pub.sent_offsets = h->bo.sentOff.data(); h->pub.begin = h->bo.sentBegin.data(); h->pub.end = h->bo.sentEnd.data(); h->pub.status = h->bo.status.data();
		h->pub.ms_h2d = h->bo.msH2D; h->pub.ms_lattice = h->bo.msLattice; h->pub.ms_viterbi = h->bo.msViterbi; h->pub.ms_sents = h->bo.msSents;
		h->pub.ms_d2h = h->bo.msD2H; h->pub.ms_total = h->bo.msTotal;
		return &h.release()->pub;
	}
	catch (const std::exception& e) { setError(e); return nullptr; }
}

void kiwi_b200_sents_free(const kiwi_b200_sents_t* sents)
{
	delete reinterpret_cast<SentsHolder*>(const_cast<kiwi_b200_sents_t*>(sents));
}

void kiwi_b200_batch_free(const kiwi_b200_batch_t* batch)
{
	if (!batch) return;
	auto* h = reinterpret_cast<BatchHolder*>(const_cast<kiwi_b200_batch_t*>(batch));
	std::shared_ptr<BatchPool> pool = std::move(h->pool);
	if (pool)
	{
		std::lock_guard<std::mutex> lk(pool->m);
		// (large holders - hundreds of MB of page-locked memory each - are kept more sparingly)
		const size_t keep = h->bo.tokens.capacity() * sizeof(DToken) > ((size_t)256 << 20) ? 2 : 4;
		if (!pool->closed && pool->free.size() < keep) { pool->free.push_back(h); return; }
	}
	delete h;
}

float kiwi_b200_analyze_device(kiwi_h handle, const void* d_text, const void* d_offsets, int n, uint64_t total_units, kiwi_analyze_option_t option, uint64_t* out_tokens, uint64_t* out_launches)
{
	if (!handle) { setError("invalid handle"); return -1.f; }
	try
	{
		checkOption(option, 1, nullptr);
		std::lock_guard<std::mutex> lk(handle->mtx);
		TypoScope ts{ handle->engine.get(), option };
		BlockScope bs{ handle->engine.get(), option };
		const float ms = handle->engine->analyzeDevice(reinterpret_cast<const uint16_t*>(d_text), reinterpret_cast<const uint32_t*>(d_offsets), (uint32_t)n, total_units, optionWord(option), out_tokens);
		if (out_launches) *out_launches = handle->engine->last.kernelLaunches;
		return ms;
	}
	catch (const std::exception& e) { setError(e); return -1.f; }
}

int kiwi_b200_last_stats(kiwi_h handle, kiwi_b200_stats_t* out)
{
	if (!handle || !out) return KIWIERR_INVALID_HANDLE;
	const Stats& s = handle->engine->last;
	out->n_sentences = s.nSentences; out->raw_units = s.rawUnits; out->norm_units = s.normUnits; out->lattice_nodes = s.latticeNodes; out->tokens = s.tokens; out->paths = s.paths;
	out->h2d_bytes = s.h2dBytes; out->d2h_bytes = s.d2hBytes; out->kernel_launches = s.kernelLaunches; out->retried = s.retried;
	out->ms_lattice = s.msLattice; out->ms_viterbi = s.msViterbi; out->ms_pack = s.msPack;
	return 0;
}

int kiwi_b200_debug_lattice(kiwi_h handle, const kchar16_t* text, int len, int32_t* out_rows, int max_rows, kiwi_analyze_option_t option)
{
	if (!handle) return KIWIERR_INVALID_HANDLE;
	try
	{
		std::lock_guard<std::mutex> lk(handle->mtx);
		std::vector<int32_t> rows;
		TypoScope ts{ handle->engine.get(), option };
		const int n = handle->engine->debugLattice(text, (uint32_t)len, (uint32_t)option.match_options, rows);
		if (n < 0) throw std::runtime_error("lattice build failed with status " + std::to_string(-n));
		if (n > max_rows) throw std::runtime_error("lattice has more rows than the caller's buffer");
		std::memcpy(out_rows, rows.data(), rows.size() * 4);
		return n;
	}
	catch (const std::exception& e) { setError(e); return KIWIERR_FAIL; }
}

int kiwi_b200_debug_cong(kiwi_h handle, int n, const uint32_t* ctx, const uint32_t* wid, const int32_t* node,
	int32_t* out_dot, float* out_eps, int32_t* out_node, uint32_t* out_ctx, int32_t* out_tile)
{
	if (!handle) return KIWIERR_INVALID_HANDLE;
	try
	{
		std::lock_guard<std::mutex> lk(handle->mtx);
		handle->engine->debugCong((uint32_t)n, ctx, wid, node, out_dot, out_eps, out_node, out_ctx, out_tile);
		return 0;
	}
	catch (const std::exception& e) { setError(e); return KIWIERR_FAIL; }
}

int kiwi_b200_debug_timing(kiwi_h handle, int n, uint64_t* out_start_end_ns)
{
	if (!handle) return KIWIERR_INVALID_HANDLE;
	try
	{
		std::lock_guard<std::mutex> lk(handle->mtx);
		handle->engine->debugTiming((uint32_t)n, reinterpret_cast<unsigned long long*>(out_start_end_ns));
		return 0;
	}
	catch (const std::exception& e) { setError(e); return KIWIERR_FAIL; }
}

void kiwi_set_global_config(kiwi_h handle, kiwi_config_t config)
{
	if (!handle) return;
	try
	{
		std::lock_guard<std::mutex> lk(handle->mtx);
		kb2_config c = handle->engine->model.header.config;
		c.integrate_allomorph = config.integrate_allomorph ? 1u : 0u;
		c.cut_off_threshold = config.cut_off_threshold; c.oov_rule_scale = config.oov_rule_scale; c.oov_rule_bias = config.oov_rule_bias;
		c.space_penalty = config.space_penalty; c.typo_cost_weight = config.typo_cost_weight;
		c.max_unk_form_size = config.max_unk_form_size; c.max_unk_form_size_followed_by_jclass = config.max_unk_form_size_followed_by_j_class;
		c.space_tolerance = config.space_tolerance;
		handle->engine->setConfig(c);
		for (auto& e : handle->extra) e->setConfig(c);
		handle->oovChrBias = config.oov_chr_bias; handle->oovGlobalWeight = config.oov_global_weight;
		handle->oovLocalWeight = config.oov_local_weight; handle->oovGlobalMinFreq = config.oov_global_min_freq;
	}
	catch (const std::exception& e) { setError(e); }
}

kiwi_config_t kiwi_get_global_config(kiwi_h handle)
{
	kiwi_config_t config{};
	if (!handle) return config;
	const kb2_config& c = handle->engine->model.header.config;
	config.integrate_allomorph = c.integrate_allomorph ? 1 : 0;
	config.cut_off_threshold = c.cut_off_threshold; config.oov_rule_scale = c.oov_rule_scale; config.oov_rule_bias = c.oov_rule_bias;
	config.oov_chr_bias = handle->oovChrBias; config.oov_global_weight = handle->oovGlobalWeight;
	config.oov_local_weight = handle->oovLocalWeight; config.oov_global_min_freq = handle->oovGlobalMinFreq;
	config.space_penalty = c.space_penalty; config.typo_cost_weight = c.typo_cost_weight;
	config.max_unk_form_size = c.max_unk_form_size; config.max_unk_form_size_followed_by_j_class = c.max_unk_form_size_followed_by_jclass;
	config.space_tolerance = c.space_tolerance;
	return config;
}

int kiwi_b200_model_type(kiwi_h handle)
{
	if (!handle) return KIWIERR_INVALID_HANDLE;
	return (int)handle->engine->model.header.model_type;
}

#pragma GCC visibility pop
}
