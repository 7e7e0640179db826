// Sentence-splitting vectors: runs the UNMODIFIED reference's Kiwi::splitIntoSents (src/Kiwi.cpp:417-450), both the UTF-16 and
// the UTF-8 overload, with Match::allWithNormalizing, on every document of a binary document file, and writes per document
//   S <idx> <nTokens> <score> 0 0
//   T ... x nTokens          the tokenizedResultOut tokens, in dump_golden's T line format
//   R <nRanges> <begin>,<end> ...   ranges in UTF-16 units (UTF-16 overload)
//   B <nRanges> <begin>,<end> ...   ranges in bytes of the UTF-8 text (UTF-8 overload)
// Input: uint32 n, uint32 offsets[n + 1], UTF-16 text (tests/golden/make_docs.py writes it from docs_sents.jsonl).  The model type
// follows KB_MODEL_TYPE (knlm, default, or cong).  TEST INFRASTRUCTURE.
// usage: split_sents <model_dir> <docs.u16> <out.txt>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iostream>
#include <string>
#include <vector>
#include <kiwi/Kiwi.h>
#include "StrUtils.h"

using namespace kiwi;

static std::string toUtf8Lenient(const std::u16string& s)
{
	std::string out;
	for (size_t i = 0; i < s.size(); ++i)
	{
		uint32_t c = s[i];
		if (0xD800 <= c && c < 0xDC00 && i + 1 < s.size() && 0xDC00 <= s[i + 1] && s[i + 1] < 0xE000) { c = 0x10000 + ((c - 0xD800) << 10) + (s[i + 1] - 0xDC00); ++i; }
		else if (0xD800 <= c && c < 0xE000) c = 0xFFFD;
		if (c < 0x80) out.push_back((char)c);
		else if (c < 0x800) { out.push_back((char)(0xC0 | (c >> 6))); out.push_back((char)(0x80 | (c & 63))); }
		else if (c < 0x10000) { out.push_back((char)(0xE0 | (c >> 12))); out.push_back((char)(0x80 | ((c >> 6) & 63))); out.push_back((char)(0x80 | (c & 63))); }
		else { out.push_back((char)(0xF0 | (c >> 18))); out.push_back((char)(0x80 | ((c >> 12) & 63))); out.push_back((char)(0x80 | ((c >> 6) & 63))); out.push_back((char)(0x80 | (c & 63))); }
	}
	return out;
}

static void writeRanges(FILE* fo, char key, const std::vector<std::pair<size_t, size_t>>& r)
{
	std::fprintf(fo, "%c %zu", key, r.size());
	for (auto& p : r) std::fprintf(fo, " %zu,%zu", p.first, p.second);
	std::fprintf(fo, "\n");
}

int main(int argc, char** argv)
{
	if (argc < 4) { std::cerr << "usage: split_sents <model_dir> <docs.u16> <out.txt>\n"; return 2; }
	if (!getenv("KIWI_ARCH_TYPE")) setenv("KIWI_ARCH_TYPE", "avx2", 1);
	try
	{
		std::ifstream ifs{ argv[2], std::ios::binary };
		uint32_t n = 0;
		ifs.read(reinterpret_cast<char*>(&n), 4);
		std::vector<uint32_t> off(n + 1);
		ifs.read(reinterpret_cast<char*>(off.data()), (std::streamsize)(4 * (n + 1)));
		std::u16string all(off[n], u'\0');
		ifs.read(reinterpret_cast<char*>(&all[0]), (std::streamsize)(2 * off[n]));
		if (!ifs) throw std::runtime_error("short read on the document file");
		const char* mt = getenv("KB_MODEL_TYPE");
		KiwiBuilder kb{ argv[1], 1, BuildOption::default_, (mt && std::string{ mt } == "cong") ? ModelType::cong : ModelType::knlm };
		Kiwi kw = kb.build();
		FILE* fo = std::fopen(argv[3], "w");
		for (uint32_t idx = 0; idx < n; ++idx)
		{
			const std::u16string doc = all.substr(off[idx], off[idx + 1] - off[idx]);
			TokenResult res;
			const auto r16 = kw.splitIntoSents(doc, Match::allWithNormalizing, &res);
			const auto r8 = kw.splitIntoSents(toUtf8Lenient(doc), Match::allWithNormalizing);
			std::fprintf(fo, "S %u %zu %a 0 0\n", idx, res.first.size(), res.second);
			for (auto& t : res.first)
			{
				std::fprintf(fo, "T %zu %u %u %u %a %u,%u,%u,%u,%d %s\n", t.morph ? kw.morphToId(t.morph) : (size_t)-1, (unsigned)t.tag, t.position, (unsigned)t.length, t.score,
					(unsigned)t.wordPosition, (unsigned)t.sentPosition, (unsigned)t.lineNumber, (unsigned)t.subSentPosition, (int)t.pairedToken, toUtf8Lenient(t.str).c_str());
			}
			writeRanges(fo, 'R', r16);
			writeRanges(fo, 'B', r8);
		}
		std::fclose(fo);
		std::cerr << "split " << n << " documents\n";
	}
	catch (const std::exception& e)
	{
		std::cerr << "split_sents failed: " << e.what() << std::endl;
		return 1;
	}
	return 0;
}
