// kiwi_b200: the one-probe edge tables of the Knlm and CoNg tries, built once on the host when a model is loaded (model.cu) and
// probed by the Viterbi kernels (viterbi.cu knLookup / cgLookup).  Host code only.
//
// Every edge (node, key) of a non-root trie node becomes one 16-byte entry {node, key, v, w} of an open-addressing table on
// knHashFn; v is the image's value (> 0: relative index of the child node, <= 0: a leaf).  The fourth word has two meanings:
//   inner edge (v > 0)  what the step needs from the child: its ll (Knlm, float bits) or its context id (CoNg);
//   leaf edge (v <= 0)  the state that follows the edge.  The reference finds it by walking the suffix chain of `node` for the
//                       deepest suffix with a non-leaf child `key` (KnLangModel::progress, src/Knlm.cpp:44-130;
//                       progressContextNodeVl, src/CoNgramModel.hpp:314-385).  That walk depends on the edge alone, so it is done
//                       here, once per leaf edge, and a leaf step on the device costs the one probe an inner step costs.
#pragma once
#include <algorithm>
#include <cstring>
#include <vector>
#include <cuda_runtime.h>
#include "kb_model.h"

namespace kb
{
	// child value of `key` below a node whose keys are sorted ascending (the image's layout); false when absent
	inline bool lmSortedFind(const uint32_t* keys, const int32_t* values, uint32_t off, uint32_t n, uint32_t key, int32_t& v)
	{
		const uint32_t* it = std::lower_bound(keys + off, keys + off + n, key);
		if (it == keys + off + n || *it != key) return false;
		v = values[it - keys];
		return true;
	}

	struct KnTables
	{
		std::vector<uint4> hash;       // {node, key, v, w}; empty slots have node 0xFFFFFFFF
		std::vector<float2> backoff;   // [node] {lower as int bits, gamma}
		std::vector<float> rootLl;     // [token] ll of the root's child
	};

	// Knlm: the state after the leaf edge (node, next): the deepest proper suffix of `node` with a non-leaf child `next`, else the
	// root's child of the history token of `next` (kn_htx), else the root
	inline int32_t knLeafState(const kb2_header* h, const kb2_kn_node* nodes, const uint32_t* keys, const int32_t* values,
	                           const int32_t* root, const uint32_t* htx, int32_t node, uint32_t next)
	{
		for (int32_t cur = node; nodes[cur].lower; )
		{
			cur += nodes[cur].lower;
			int32_t lv = 0;
			const bool found = cur == 0 ? (next < h->kn_htx_vocab && (lv = root[next]) != 0)
			                            : lmSortedFind(keys, values, nodes[cur].next_offset, nodes[cur].num_nexts, next, lv);
			if (found && lv > 0) return cur + lv;
		}
		return htx ? root[htx[next]] : 0;
	}

	inline KnTables buildKnTables(const kb2_header* h, const kb2_kn_node* nodes, const uint32_t* keys, const int32_t* values,
	                              const int32_t* root, const uint32_t* htx)
	{
		KnTables t;
		uint32_t hashSize = 1024;
		while (hashSize < 2 * (size_t)h->kn_num_edges + 16) hashSize <<= 1;
		t.hash.assign(hashSize, make_uint4(0xFFFFFFFFu, 0, 0, 0));
		t.backoff.resize(h->kn_num_nodes);
		for (uint32_t i = 0; i < h->kn_num_nodes; ++i)
		{
			const kb2_kn_node& nd = nodes[i];
			float2 b; std::memcpy(&b.x, &nd.lower, 4); b.y = nd.gamma;
			t.backoff[i] = b;
			if (i == 0) continue;
			for (uint32_t j = 0; j < nd.num_nexts; ++j)
			{
				const uint32_t key = keys[nd.next_offset + j];
				const int32_t v = values[nd.next_offset + j];
				uint32_t w;
				if (v > 0) std::memcpy(&w, &nodes[i + v].ll, 4);                                         // inner edge: the child's ll
				else w = (uint32_t)knLeafState(h, nodes, keys, values, root, htx, (int32_t)i, key);      // leaf edge: the next state
				uint32_t hh = knHashFn(i, key) & (hashSize - 1);
				while (t.hash[hh].x != 0xFFFFFFFFu) hh = (hh + 1) & (hashSize - 1);
				t.hash[hh] = make_uint4(i, key, (uint32_t)v, w);
			}
		}
		t.rootLl.assign(h->kn_htx_vocab, 0.f);
		for (uint32_t tkn = 0; tkn < h->kn_htx_vocab; ++tkn) if (root[tkn] > 0 && (uint32_t)root[tkn] < h->kn_num_nodes) t.rootLl[tkn] = nodes[root[tkn]].ll;
		return t;
	}

	struct CgTables
	{
		std::vector<uint4> hash;       // {node, key, v, w}; empty slots have node 0xFFFFFFFF
		std::vector<int2> nodes;       // [node] {lower, context id}
	};

	// CoNg: the node after the leaf edge (node, next): the deepest proper suffix of `node` with a non-leaf child `next`, else the root
	inline int32_t cgLeafState(const kb2_header* h, const kb2_cg_node* nodes, const uint32_t* keys, const int32_t* values,
	                           const int32_t* root, int32_t node, uint32_t next)
	{
		for (int32_t cur = node; nodes[cur].lower; )
		{
			cur += nodes[cur].lower;
			int32_t lv = 0;
			const bool found = cur == 0 ? (next < h->cg_root_size && (lv = root[next]) != 0)
			                            : lmSortedFind(keys, values, nodes[cur].next_offset, nodes[cur].num_nexts, next, lv);
			if (found && lv > 0) return cur + lv;
		}
		return 0;
	}

	inline CgTables buildCgTables(const kb2_header* h, const kb2_cg_node* nodes, const uint32_t* keys, const int32_t* values, const int32_t* root)
	{
		CgTables t;
		uint32_t hashSize = 1024;
		while (hashSize < 2 * (size_t)h->cg_num_edges + 16) hashSize <<= 1;
		t.hash.assign(hashSize, make_uint4(0xFFFFFFFFu, 0, 0, 0));
		t.nodes.resize(h->cg_num_nodes);
		for (uint32_t i = 0; i < h->cg_num_nodes; ++i)
		{
			t.nodes[i] = make_int2(nodes[i].lower, (int32_t)nodes[i].value);
			if (i == 0) continue;
			for (uint32_t j = 0; j < nodes[i].num_nexts; ++j)
			{
				const uint32_t key = keys[nodes[i].next_offset + j];
				const int32_t v = values[nodes[i].next_offset + j];
				const uint32_t w = v > 0 ? nodes[i + v].value                                             // inner edge: the child's context id
				                         : (uint32_t)cgLeafState(h, nodes, keys, values, root, (int32_t)i, key);   // leaf edge: the next node
				uint32_t hh = knHashFn(i, key) & (hashSize - 1);
				while (t.hash[hh].x != 0xFFFFFFFFu) hh = (hh + 1) & (hashSize - 1);
				t.hash[hh] = make_uint4(i, key, (uint32_t)v, w);
			}
		}
		return t;
	}
}
