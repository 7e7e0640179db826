// CPU check (tests/test_unordered_warp.py): kb::unorderedSetOrderWarp (kiwi_b200/csrc/unordered_emu.h), the warp-parallel iteration
// order of std::unordered_set that the Viterbi kernels use, run by the 32-lane host simulation of a warp (tests/hostsim/shim32) and
// compared with the real libstdc++ container and with the sequential restatement kb::unorderedSetOrder.  Cases: sets re-used by a
// "sentence" (cleared, never shrunk), every step of the prime chain from 1 (the first insertion of a fresh set has 1 bucket), 1 to
// 6000 keys, heavy bucket collisions, and the hash codes of the Knlm, CoNg and SkipBigram builds.
#include <cuda_runtime.h>
#include "../../kiwi_b200/csrc/unordered_emu.h"
#include <random>
#include <unordered_set>

struct Key { unsigned long long code; int id; bool operator==(const Key& o) const { return id == o.id; } };
struct H { size_t operator()(const Key& k) const { return (size_t)k.code; } };

static long bad = 0, sets = 0;

// one container: `codes` in first-insertion order, the set's bucket count before it in `B` (updated)
static void check(std::unordered_set<Key, H>& s, const std::vector<unsigned long long>& codes, uint32_t& B)
{
	const int n = (int)codes.size();
	s.clear();
	for (int i = 0; i < n; ++i) s.insert(Key{ codes[i], i });
	const uint32_t after = kb::unorderedBucketsAfter(B, n);
	std::vector<int32_t> next(n + 1), seqOrder(n + 1), seqBuckets(after ? after : 1);
	uint32_t seqB = B;
	const bool seqOk = kb::unorderedSetOrder(codes.data(), n, seqB, next.data(), seqBuckets.data(), seqOrder.data());
	// the warp's scratch is poisoned: nothing may depend on what it held before
	std::vector<int32_t> first(n + 1, 0x5A5A5A5A), runs(n + 1, 0x5A5A5A5A), buckets(after ? after : 1, 0x5A5A5A5A), order(n + 1, -7);
	uint32_t warpB = 0; bool warpOk = false;
	simt::launch(1, 32, [&]
	{
		uint32_t b = B;
		const bool ok = kb::unorderedSetOrderWarp([&](int32_t i) { return codes[i]; }, n, b, first.data(), runs.data(), buckets.data(), order.data(), simt::lane);
		if (simt::lane == 0) { warpB = b; warpOk = ok; }
	});
	++sets;
	bool diff = !seqOk || !warpOk || warpB != s.bucket_count() || seqB != warpB || warpB != after;
	int j = 0;
	for (auto& k : s) { if (j >= n || order[j] != k.id || seqOrder[j] != k.id) diff = true; ++j; }
	if (j != n) diff = true;
	if (diff && bad < 10) std::printf("mismatch: n %d, buckets before %u, after %u / %u / %zu\n", n, B, warpB, seqB, s.bucket_count());
	bad += diff;
	B = warpB;
}

int main(int argc, char** argv)
{
	const int scale = argc > 1 ? std::atoi(argv[1]) : 1;
	std::mt19937_64 rng(11);
	// hash codes as the three Viterbi builds form them from (lmState, prevRootId, spState) - or, SkipBigram, from the history ring too
	auto knlm = [&](int32_t lm, uint32_t prevRoot, uint32_t sp) { unsigned long long h = (unsigned long long)(long long)lm; return (unsigned long long)(prevRoot | (sp << 8)) ^ ((h << 3) | (h >> 61)); };
	auto cong = [&](uint32_t node, uint32_t prevRoot, uint32_t sp) { const unsigned long long v = node; unsigned long long h = (v * 2305843009213693951ull) ^ ((v << 33) | (v >> 31)); return (unsigned long long)(prevRoot | (sp << 8)) ^ ((h << 3) | (h >> 61)); };
	auto sbg = [&](int32_t lm, const uint32_t* hist, uint32_t prevRoot, uint32_t sp) { unsigned long long h = (unsigned long long)(long long)lm; for (int i = 0; i < 8; ++i) h = (unsigned long long)hist[i] ^ ((h << 3) | (h >> 61)); return (unsigned long long)(prevRoot | (sp << 8)) ^ ((h << 3) | (h >> 61)); };
	auto makeCodes = [&](int n, int kind, uint32_t B)
	{
		std::vector<unsigned long long> c(n);
		const uint32_t states = 1 + rng() % 4000;
		for (int i = 0; i < n; ++i)
		{
			const uint32_t prevRoot = rng() % 4 == 0 ? rng() % 256 : 0, sp = rng() % 3;
			switch (kind)
			{
			case 0: c[i] = knlm((int32_t)(rng() % states), prevRoot, sp); break;
			case 1: c[i] = cong((uint32_t)(rng() % states), prevRoot, sp); break;
			case 2: { uint32_t hist[8]; for (auto& x : hist) x = rng() % 50; c[i] = sbg((int32_t)(rng() % states), hist, prevRoot, sp); break; }
			case 3: c[i] = (rng() % 64) * 8 + rng() % 3; break;                                  // few distinct buckets
			case 4: c[i] = (unsigned long long)(rng() % 5) * B + (rng() % 3) * 2357; break;     // whole runs in a handful of buckets
			default: c[i] = rng(); break;
			}
		}
		return c;
	};
	const uint32_t chain[] = { 1u, 13u, 29u, 59u, 127u, 257u, 541u, 1109u, 2357u, 5087u };
	// every step of the prime chain: a fresh set grown to it, then containers just below, at and just above its bucket count
	for (uint32_t b : chain)
		for (int dn : { -1, 0, 1, 2 })
			for (int kind = 0; kind < 6; ++kind)
			{
				std::unordered_set<Key, H> fresh; uint32_t B = 1;
				if (b > 1) { check(fresh, makeCodes((int)b, kind, b), B); }
				const int n = (int)b + dn;
				if (n >= 0) check(fresh, makeCodes(n, kind, B), B);
			}
	// re-used sets: a "sentence" of containers of 1 to 6000 keys
	for (int trial = 0; trial < 60 * scale; ++trial)
	{
		std::unordered_set<Key, H> sent; uint32_t B = 1;
		const int rounds = 1 + rng() % 8;
		for (int r = 0; r < rounds; ++r)
		{
			const int n = rng() % 4 == 0 ? 1 + rng() % 6000 : 1 + rng() % 800;
			check(sent, makeCodes(n, (int)(rng() % 6), B), B);
		}
	}
	std::printf("sets %ld mismatching %ld\n", sets, bad);
	return bad != 0;
}
