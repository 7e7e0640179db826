// kiwi_b200: host-side result assembly — the token-list post-processing the reference runs after the hot path
// (SURVEY.md 8f-1).  Pure functions over the finished token list; nothing here touches the device.
//   fillPairedTokenInfo   /root/reference/src/Kiwi.cpp:98-143
//   fillSentLineInfo      src/Kiwi.cpp:322-415
//   allNewLinePositions   src/Kiwi.cpp:69-96
// The sentence rules themselves live in sentences.h, which the device sentence kernel (sents.cu) shares; the functions here
// convert the host's token records to its POD tokens and back.
#pragma once
#include <algorithm>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>
#include "kb_model.h"
#include "sentences.h"

namespace kb
{
	struct AsmTok
	{
		// in
		uint32_t position = 0, length = 0;
		uint8_t tag = 0;
		std::u16string form;          // TokenInfo::str
		bool kformIsYo = false;       // *morph->kform == u"요"
		uint32_t wordPosition = 0;    // in: word index in the whole text (getWordPositions); out: word index inside its sentence
		// out
		uint32_t sentPosition = 0, lineNumber = 0, subSentPosition = 0, pairedToken = 0xFFFFFFFFu;
		uint32_t endPos() const { return position + length; }
	};

	// ---- surface form of a token that keeps its own substring (TokenInfo::str = joinHangul(PathNode::str), src/Kiwi.cpp:721):
	// the substring is taken from the NORMALISED text (normalizeHangulWithPosition src/StrUtils.h:493-520, then normalizeCoda
	// 636-710 when Match::normalizeCoda is set), whose codas are separate units; a token may begin at the coda of a raw
	// character or end before it.  The device reports raw positions only, but tokens tile the text, so such a split shows
	// as two tokens sharing one raw character.
	struct NormText { std::u16string norm; std::vector<uint32_t> pos; };      // pos[i] = first normalised unit of raw unit i, pos[n] = size

	inline NormText normalizeWithPosition(const uint16_t* text, size_t n, bool normalizeCodaOpt)
	{
		NormText nt;
		nt.pos.reserve(n + 1); nt.norm.reserve(n * 2);
		for (size_t i = 0; i < n; ++i)
		{
			uint32_t c = text[i];
			nt.pos.push_back((uint32_t)nt.norm.size());
			if (c == 0xB42C) c = 0xB410;
			if (0xAC00 <= c && c < 0xD7A4)
			{
				const uint32_t coda = (c - 0xAC00) % 28;
				nt.norm.push_back((char16_t)(c - coda));
				if (coda) nt.norm.push_back((char16_t)(coda + 0x11A7));
			}
			else nt.norm.push_back((char16_t)c);
		}
		nt.pos.push_back((uint32_t)nt.norm.size());
		if (normalizeCodaOpt)
		{
			// a coda followed by the compatibility jamo of the same consonant ("몈ㅋㅋ") becomes that jamo, or the first half of a double coda
			static const char16_t toOnset[27] = { 0x3131, 0x3131, 0x3145, 0x3134, 0x3148, 0x314E, 0x3137, 0x3139, 0x3131, 0x3141, 0x3142, 0x3145, 0x314C, 0x314D,
				0x314E, 0x3141, 0x3142, 0x3145, 0x3145, 0x3145, 0x3147, 0x3148, 0x314A, 0x314B, 0x314C, 0x314D, 0x314E };
			static const char16_t reduced[27] = { 0, 0x11A8, 0x11A8, 0, 0x11AB, 0x11AB, 0, 0, 0x11AF, 0x11AF, 0x11AF, 0x11AF, 0x11AF, 0x11AF, 0x11AF, 0, 0, 0x11B8, 0, 0x11BA,
				0, 0, 0, 0, 0, 0, 0 };
			char16_t before = 0;
			for (size_t i = 0; i < nt.norm.size(); ++i)
			{
				const char16_t cur = nt.norm[i];
				if (0x11A8 <= before && before <= 0x11C2 && cur == toOnset[before - 0x11A8])
				{
					const char16_t r = reduced[before - 0x11A8];
					nt.norm[i - 1] = r ? r : cur;
				}
				before = cur;
			}
		}
		return nt;
	}

	// joinHangul, include/kiwi/Utils.h:167-205
	inline std::u16string joinHangulUnits(const char16_t* p, size_t n)
	{
		std::u16string ret;
		ret.reserve(n);
		for (size_t i = 0; i < n; ++i)
		{
			const char16_t c = p[i];
			if (!ret.empty() && 0xAC00 <= ret.back() && ret.back() < 0xD7A4 && (ret.back() - 0xAC00) % 28 == 0)
			{
				if (0x11A8 <= c && c < 0x11A8 + 27) ret.back() = (char16_t)(ret.back() + (c - 0x11A7));
				else if ((0x11A8 <= c && c < 0x1200) || (0xD7CB <= c && c < 0xD800))
				{
					const uint32_t onset = (ret.back() - 0xAC00) / 28 / 21, vowel = (ret.back() - 0xAC00) / 28 % 21;
					ret.back() = (char16_t)(0x1100 + onset);
					ret.push_back((char16_t)(0x1161 + vowel));
					ret.push_back(c);
				}
				else ret.push_back(c);
			}
			else ret.push_back(c);
		}
		return ret;
	}

	inline std::u16string ownSubstringForm(const NormText& nt, uint32_t position, uint32_t length, bool beginsAtCoda, bool endsBeforeCoda)
	{
		if ((size_t)position + length >= nt.pos.size()) return {};
		uint32_t b = nt.pos[position] + (beginsAtCoda ? 1u : 0u), e = nt.pos[position + length] - (endsBeforeCoda ? 1u : 0u);
		if (e < b) e = b;
		return joinHangulUnits(nt.norm.data() + b, e - b);
	}

	inline std::vector<size_t> newlinePositions(const uint16_t* text, size_t n)
	{
		std::vector<size_t> ret;
		for (size_t i = 0; i < n; ++i) if (isNewlineAt(text, (uint32_t)i)) ret.push_back(i);
		return ret;
	}

	inline std::vector<SentTok> toSentToks(const std::vector<AsmTok>& toks)
	{
		std::vector<SentTok> st(toks.size());
		for (size_t i = 0; i < toks.size(); ++i)
		{
			const AsmTok& t = toks[i];
			SentTok& o = st[i];
			o = SentTok{};
			o.position = t.position; o.length = t.length; o.tag = t.tag; o.flags = t.kformIsYo ? SF_YO : 0;
			o.wordPosition = t.wordPosition; o.pairedToken = t.pairedToken;
			setSentForm(o, reinterpret_cast<const uint16_t*>(t.form.data()), (uint32_t)t.form.size());
		}
		return st;
	}

	inline void fillPaired(std::vector<AsmTok>& toks)
	{
		std::vector<SentTok> st = toSentToks(toks);
		std::vector<uint2> stacks(2 * st.size() + 2);
		pairTokens(st.data(), (uint32_t)st.size(), stacks.data(), stacks.data() + st.size() + 1);
		for (size_t i = 0; i < toks.size(); ++i) toks[i].pairedToken = st[i].pairedToken;
	}

	// (pairedToken filled by fillPaired)
	inline void fillSentLine(std::vector<AsmTok>& toks, const std::vector<size_t>& newlines)
	{
		std::vector<SentTok> st = toSentToks(toks);
		for (auto& t : st) t.lineNumber = (uint32_t)(std::lower_bound(newlines.begin(), newlines.end(), (size_t)t.position) - newlines.begin());
		foldSentLine(st.data(), (uint32_t)st.size());
		for (size_t i = 0; i < toks.size(); ++i)
		{
			AsmTok& t = toks[i];
			t.wordPosition = st[i].wordPosition; t.sentPosition = st[i].sentPosition; t.lineNumber = st[i].lineNumber; t.subSentPosition = st[i].subSentPosition;
		}
	}

	// ---- one sentence's device rows -> the reference's TokenInfo list (insertPathIntoResults src/Kiwi.cpp:714-751, then fillPairedTokenInfo /
	// fillSentLineInfo, Kiwi.cpp:1149-1154).  The model's host view: morphemes, forms, form characters, character attributes (chr_bmp).
	struct ResTok { AsmTok a; uint32_t morphId; uint8_t senseId; uint16_t dialect; };
	inline std::vector<ResTok> assembleRows(const kb2_morph* morphs, const kb2_form* forms, const uint16_t* formChars, const uint32_t* chrBmp,
		const uint16_t* text, uint32_t rawLen, const DToken* rows, uint32_t n, const uint16_t* joined, size_t joinedSize, uint32_t matchOptions)
	{
		// word index of every raw position: getWordPositions, src/Kiwi.cpp:464-485 (a run of spaces ends one word)
		std::vector<uint16_t> wordPos(rawLen + 1, 0);
		{
			uint32_t position = 0; bool continuousSpace = false;
			for (uint32_t i = 0; i <= rawLen; ++i)
			{
				wordPos[i] = (uint16_t)position;
				if (i < rawLen && attrSpace(chrBmp[text[i]])) { if (!continuousSpace) ++position; continuousSpace = true; }
				else continuousSpace = false;
			}
		}
		const NormText nt = normalizeWithPosition(text, rawLen, (matchOptions & (1u << 16)) != 0);
		std::vector<ResTok> out(n);
		std::vector<AsmTok> at(n);
		for (uint32_t t = 0; t < n; ++t)
		{
			const DToken& d = rows[t];
			ResTok& r = out[t];
			AsmTok& a = at[t];
			a.position = d.position; a.length = d.length; a.tag = d.tag; a.wordPosition = wordPos[d.position];
			// a joined row (token-joining options) has no morpheme (morphToId(nullptr) = -1); its entry in `joined` holds the first
			// component's morpheme id (sense id, dialect) and the form the device built (kb_batch.h JOINED_TOKEN)
			const bool isJoined = (d.morph & JOINED_TOKEN) != 0;
			const uint32_t entry = d.morph & ~JOINED_TOKEN;
			if (isJoined && (size_t)entry + 2 >= joinedSize) throw std::runtime_error("joined token without its form");
			const uint32_t first = isJoined ? (uint32_t)joined[entry] | ((uint32_t)joined[entry + 1] << 16) : d.morph;
			const kb2_morph& mm = morphs[first];
			r.morphId = isJoined ? 0xFFFFFFFFu : d.morph;
			r.senseId = mm.sense_id; r.dialect = mm.dialect;
			// an OOV noun (own surface form) has no sense (Kiwi.cpp:738-741)
			if ((d.flags & 1) && ((mm.tag & 0x7F) == T_nng || (mm.tag & 0x7F) == T_nnp)) r.senseId = 0xFF;
			if (isJoined)
			{
				const uint16_t* f = joined + entry + 2;
				a.form.assign(reinterpret_cast<const char16_t*>(f), std::find(f, joined + joinedSize, (uint16_t)0) - f);
				continue;      // (never the jx "요" of the sentence rules: Kiwi.cpp:211 tests t.morph)
			}
			if (d.flags & 1)
			{
				// own substring: two tokens sharing a raw character = that character's syllable body / coda split
				const bool beginsAtCoda = t > 0 && rows[t - 1].position + rows[t - 1].length > d.position;
				const bool endsBeforeCoda = t + 1 < n && rows[t + 1].position < d.position + d.length;
				a.form = ownSubstringForm(nt, d.position, d.length, beginsAtCoda, endsBeforeCoda);
			}
			else if (mm.form_idx >= 0) a.form = joinHangulUnits(reinterpret_cast<const char16_t*>(formChars + forms[mm.form_idx].str_off), forms[mm.form_idx].str_len);
			// Match::compatibleJamo converts every token's form (Kiwi.cpp:726-729); the device converted the joined ones already
			if (matchOptions & MO_COMPATIBLE_JAMO) for (auto& c : a.form) c = (char16_t)toCompatibleJamo((uint16_t)c);
			a.kformIsYo = mm.form_idx >= 0 && forms[mm.form_idx].str_len == 1 && formChars[forms[mm.form_idx].str_off] == 0xC694;
		}
		fillPaired(at);
		fillSentLine(at, newlinePositions(text, rawLen));
		for (uint32_t t = 0; t < n; ++t) out[t].a = std::move(at[t]);
		return out;
	}
}
