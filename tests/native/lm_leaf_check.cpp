// CPU check of the leaf states the model loader stores in the Knlm and CoNg edge tables (kiwi_b200/csrc/lm_tables.h): for every
// leaf edge (node, key) of the table, the stored state must be the state the oracle restatement's LM step reaches from `node` with
// `key` (oracle/restate/knlm.hpp Knlm::progress, cong.hpp Cong::stepVl, which walk the suffix chain), and every inner edge must carry
// the child's ll / context id.
//   lm_leaf_check <knlm image> [<cong image> | -]
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include "../../oracle/restate/knlm.hpp"
#include "../../oracle/restate/cong.hpp"
#include "../../kiwi_b200/csrc/lm_tables.h"

static int checkKnlm(const char* path)
{
	orc::Image im; im.load(path);
	orc::Knlm kn(im);
	const kb::KnTables t = kb::buildKnTables(im.h, im.knNodes, im.knKeys, im.knValues, im.knRoot, im.knHtx);
	uint64_t leaves = 0, inner = 0, bad = 0;
	for (const uint4& e : t.hash)
	{
		if (e.x == 0xFFFFFFFFu) continue;
		int32_t node = (int32_t)e.x;
		const float ll = kn.progress(node, e.y);
		float ell; std::memcpy(&ell, &e.w, 4);
		const int32_t v = (int32_t)e.z;
		bool ok;
		if (v > 0) { ++inner; ok = node == (int32_t)e.x + v && std::memcmp(&ll, &ell, 4) == 0; }
		else { ++leaves; ok = (uint32_t)node == e.w && std::memcmp(&ll, &v, 4) == 0; }
		if (!ok && bad++ < 10) std::printf("knlm edge (%u, %u) v %d: stored %u, oracle state %d\n", e.x, e.y, v, e.w, node);
	}
	std::printf("knlm: %llu leaf edges, %llu inner edges, %llu mismatches\n", (unsigned long long)leaves, (unsigned long long)inner, (unsigned long long)bad);
	return leaves && !bad ? 0 : 1;
}

static int checkCong(const char* path)
{
	orc::Image im; im.load(path);
	orc::Cong cg(im);
	const kb2_header* h = im.h;
	const kb::CgTables t = kb::buildCgTables(h, cg.nodes, cg.keys, cg.values, cg.root);
	uint64_t leaves = 0, inner = 0, bad = 0;
	for (const uint4& e : t.hash)
	{
		if (e.x == 0xFFFFFFFFu) continue;
		int32_t node = (int32_t)e.x;
		const uint32_t ctx = cg.stepVl(node, e.y);
		const int32_t v = (int32_t)e.z;
		bool ok;
		if (v > 0) { ++inner; ok = node == (int32_t)e.x + v && ctx == e.w; }
		else { ++leaves; ok = (uint32_t)node == e.w && ctx == (uint32_t)-v; }
		if (!ok && bad++ < 10) std::printf("cong edge (%u, %u) v %d: stored %u, oracle state %d\n", e.x, e.y, v, e.w, node);
	}
	std::printf("cong: %llu leaf edges, %llu inner edges, %llu mismatches\n", (unsigned long long)leaves, (unsigned long long)inner, (unsigned long long)bad);
	return leaves && !bad ? 0 : 1;
}

int main(int argc, char** argv)
{
	if (argc < 2) { std::fprintf(stderr, "usage: %s <knlm image> [<cong image> | -]\n", argv[0]); return 2; }
	try
	{
		int rc = checkKnlm(argv[1]);
		if (argc > 2 && std::strcmp(argv[2], "-") != 0) rc |= checkCong(argv[2]);
		return rc;
	}
	catch (const std::exception& e) { std::fprintf(stderr, "%s\n", e.what()); return 2; }
}
