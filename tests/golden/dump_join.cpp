// Dumper of the token-joining vectors (tests/golden/make_join.py): the golden-vector dumper oracle/ref_build/tools/dump_golden.cpp,
// compiled unchanged, with AnalyzeOption::match taken from the environment variable KB_MATCH (an integer; unset: the default
// MATCH_ALL_WITH_NORMALIZING).  The dumper's headers are included first, so that the macro below renames only the option object the
// dumper declares (`AnalyzeOption option;`): it becomes the subclass here, whose constructor reads KB_MATCH.  Output format, model
// selection (KB_MODEL_TYPE) and the typo set (KB_TYPO) are the dumper's.  make_join.py builds it against oracle/_ref/libkiwi_ref.so
// with the reference tools' flags (oracle/ref_build/Makefile TOOLFLAGS).
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iostream>
#include <string>
#include <thread>
#include <unordered_set>
#include <algorithm>
#include <kiwi/Kiwi.h>
#include <kiwi/TypoTransformer.h>
#include "StrUtils.h"
#include "KTrie.h"
#include "PathEvaluator.h"

struct KbJoinOption : kiwi::AnalyzeOption
{
	KbJoinOption()
	{
		if (const char* mo = std::getenv("KB_MATCH")) match = (kiwi::Match)std::stoul(mo, nullptr, 0);
	}
};

#define AnalyzeOption KbJoinOption
#include "../../oracle/ref_build/tools/dump_golden.cpp"
