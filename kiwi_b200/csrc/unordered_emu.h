// kiwi_b200: the iteration order of libstdc++'s std::unordered_set, restated (bits/hashtable.h: _M_insert_unique_node /
// _M_insert_bucket_begin, _M_rehash_aux(unique keys), _Prime_rehash_policy with max_load_factor 1 and growth factor 2).
//
// Why: with more than 512 incoming paths the reference collects a candidate's paths in BestPathConatiner<top1> - an
// std::unordered_set - and writes them out in the set's ITERATION order (/root/reference/src/BestPathContainer.hpp:229-276).  That
// order fixes the order of the node's paths and through it every later tie-break (first-inserted wins in the containers, std::sort of
// equal end-node scores), so it is part of the result.  The order is a function of (a) the bucket count the set has grown to - the
// set is cleared, never shrunk, between uses - and (b) the hash codes of the distinct keys in first-insertion order; the kernels know
// both: keys are appended in first-insertion order, and the bucket count is a per-sentence state that starts at 1 like the oracle's
// (the reference's thread_local set additionally remembers earlier sentences of its thread: not reproducible by definition).
// unorderedSetOrder is the sequential statement; the kernels run unorderedSetOrderWarp, the same order computed by a whole warp.
// n = distinct keys of one candidate's container (hundreds).
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define KB_UO_HD __host__ __device__ inline
#else
#define KB_UO_HD inline
#endif

namespace kb
{
	// bucket counts libstdc++ walks through from a default-constructed set: 1 -> 13 on the first insertion, then the smallest prime of its
	// __prime_list that is >= twice the current count, whenever an insertion would push the size above the bucket count
	KB_UO_HD uint32_t unorderedNextBuckets(uint32_t b)
	{
		const uint32_t chain[] = { 1u, 13u, 29u, 59u, 127u, 257u, 541u, 1109u, 2357u, 5087u, 10273u, 20753u, 42043u, 85229u, 172933u, 351061u, 712697u, 1447153u, 2938679u };
		for (unsigned i = 0; i + 1 < sizeof(chain) / sizeof(chain[0]); ++i) if (chain[i] == b) return chain[i + 1];
		return 0;      // not on the chain: the caller treats it as an internal error
	}
	// the bucket count after a container that held `n` distinct keys, starting from `b`
	KB_UO_HD uint32_t unorderedBucketsAfter(uint32_t b, uint32_t n)
	{
		while (n > (b == 1 ? 0u : b)) { b = unorderedNextBuckets(b); if (!b) return 0; }
		return b;
	}

	// codes[i]: hash code of the i-th distinct key in first-insertion order.  bucketCount: in = the set's bucket count before the first
	// insertion, out = after the last.  next[n], buckets[bucketCount after]: scratch.  order[j] = insertion index of the j-th element in
	// iteration order.  Returns false when the bucket chain is exhausted.
	KB_UO_HD bool unorderedSetOrder(const unsigned long long* codes, int32_t n, uint32_t& bucketCount, int32_t* next, int32_t* buckets, int32_t* order)
	{
		const int32_t EMPTY = -2, BEFORE_BEGIN = -1;
		uint32_t B = bucketCount;
		int32_t beginNext = -1;      // _M_before_begin._M_nxt
		for (uint32_t b = 0; b < B; ++b) buckets[b] = EMPTY;
		for (int32_t i = 0; i < n; ++i)
		{
			if ((uint32_t)i + 1 > (B == 1 ? 0u : B))
			{
				// _M_rehash_aux(n, unique keys): relink every node into the new bucket array, walking the old list from its head
				const uint32_t nb = unorderedNextBuckets(B);
				if (!nb) return false;
				B = nb;
				for (uint32_t b = 0; b < B; ++b) buckets[b] = EMPTY;
				int32_t p = beginNext; beginNext = -1;
				uint32_t bbeginBkt = 0;
				while (p >= 0)
				{
					const int32_t nx = next[p];
					const uint32_t bkt = (uint32_t)(codes[p] % B);
					if (buckets[bkt] == EMPTY)
					{
						next[p] = beginNext; beginNext = p;
						buckets[bkt] = BEFORE_BEGIN;
						if (next[p] >= 0) buckets[bbeginBkt] = p;
						bbeginBkt = bkt;
					}
					else
					{
						const int32_t before = buckets[bkt];
						if (before == BEFORE_BEGIN) { next[p] = beginNext; beginNext = p; }
						else { next[p] = next[before]; next[before] = p; }
					}
					p = nx;
				}
			}
			// _M_insert_bucket_begin
			const uint32_t bkt = (uint32_t)(codes[i] % B);
			if (buckets[bkt] != EMPTY)
			{
				const int32_t before = buckets[bkt];
				if (before == BEFORE_BEGIN) { next[i] = beginNext; beginNext = i; }
				else { next[i] = next[before]; next[before] = i; }
			}
			else
			{
				next[i] = beginNext; beginNext = i;
				if (next[i] >= 0) buckets[(uint32_t)(codes[next[i]] % B)] = i;
				buckets[bkt] = BEFORE_BEGIN;
			}
		}
		int32_t j = 0;
		for (int32_t p = beginNext; p >= 0; p = next[p]) order[j++] = p;
		bucketCount = B;
		return j == n;
	}

#if defined(__CUDACC__) || defined(KB_HOSTSIM)
	// The same order computed by a whole warp; unorderedSetOrder above is its specification.  Every lane calls it with the same arguments.
	//
	// _M_insert_bucket_begin and the relink loop of _M_rehash_aux apply one rule: a node whose bucket already holds nodes goes to the
	// front of that bucket's run, any other node to the head of the list.  So within an epoch (a stretch with one bucket count B), whose
	// ARRIVALS are the list left by the rehash followed by the epoch's insertions, the list is: buckets by descending arrival of their
	// first node, and within a bucket, nodes by descending arrival.  Per epoch: (1) bucket and first arrival of every node, 32 arrivals
	// a round, node count per bucket kept at the bucket's first arrival; (2) suffix sum of those counts over the arrivals = where each
	// bucket's run starts; (3) scatter, arrivals in descending order, each bucket's run filled from its start.
	//
	// codeOf(i): hash code of the i-th distinct key in first-insertion order.  bucketCount: in = the set's bucket count before the first
	// insertion, out = after the last.  first[n], runs[n], buckets[bucketCount after]: scratch.  order[n] as in unorderedSetOrder.
	// Returns false when the bucket chain is exhausted.
	template<class CodeOf>
	__device__ inline bool unorderedSetOrderWarp(CodeOf codeOf, int32_t n, uint32_t& bucketCount, int32_t* first, int32_t* runs, int32_t* buckets, int32_t* order, uint32_t lane)
	{
		const unsigned FULL = 0xFFFFFFFFu;
		uint32_t B = bucketCount;
		int32_t m = 0;      // nodes in the list; order[0, m) is the list
		while (m < n)
		{
			if ((uint32_t)m + 1 > (B == 1 ? 0u : B)) { B = unorderedNextBuckets(B); if (!B) return false; }
			const int32_t m1 = (int32_t)B < n ? (int32_t)B : n;      // insertions m .. m1 - 1 keep this bucket count
			for (uint32_t b = lane; b < B; b += 32) buckets[b] = -1;
			for (int32_t t = (int32_t)lane; t < m1; t += 32) runs[t] = 0;
			__syncwarp();
			// (1) arrival t is node order[t] (t < m: the relinked list) or node t (this epoch's insertions)
			for (int32_t base = 0; base < m1; base += 32)
			{
				const int32_t t = base + (int32_t)lane;
				const bool valid = t < m1;
				const uint32_t bkt = valid ? (uint32_t)(codeOf(t < m ? order[t] : t) % B) : 0xFFFFFFFFu;
				const unsigned grp = __match_any_sync(FULL, bkt);
				const int32_t leader = __ffs(grp) - 1;
				int32_t f = 0;
				if (valid && (int32_t)lane == leader)
				{
					f = buckets[bkt];
					if (f < 0) { f = t; buckets[bkt] = t; }
					runs[f] += __popc(grp);
				}
				f = __shfl_sync(FULL, f, leader);
				if (valid) first[t] = f;
				__syncwarp();
			}
			// (2) runs[t] = nodes of the buckets whose first arrival is after t = start of the run of the bucket first reached at t
			int32_t carry = 0;
			for (int32_t base = (m1 - 1) & ~31; base >= 0; base -= 32)
			{
				const int32_t t = base + (int32_t)lane;
				const int32_t c = t < m1 ? runs[t] : 0;
				int32_t incl = c;      // inclusive suffix sum inside the round
				for (int d = 1; d < 32; d <<= 1) { const int32_t o = __shfl_down_sync(FULL, incl, d); if (lane + d < 32) incl += o; }
				if (t < m1) runs[t] = carry + incl - c;
				carry += __shfl_sync(FULL, incl, 0);
			}
			__syncwarp();
			// (3) the bucket array is dead: it receives the new list.  Later arrivals of a bucket come first.
			for (int32_t base = (m1 - 1) & ~31; base >= 0; base -= 32)
			{
				const int32_t t = base + (int32_t)lane;
				const bool valid = t < m1;
				const int32_t f = valid ? first[t] : -1;
				const unsigned grp = __match_any_sync(FULL, f);
				const int32_t leader = __ffs(grp) - 1;
				int32_t at = 0;
				if (valid && (int32_t)lane == leader) { at = runs[f]; runs[f] = at + __popc(grp); }
				at = __shfl_sync(FULL, at, leader);
				if (valid) buckets[at + __popc(grp & ~((2u << lane) - 1u))] = t < m ? order[t] : t;
				__syncwarp();
			}
			for (int32_t t = (int32_t)lane; t < m1; t += 32) order[t] = buckets[t];
			__syncwarp();
			m = m1;
		}
		bucketCount = B;
		return true;
	}
#endif
}
