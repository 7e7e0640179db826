// kiwi_b200: sentence boundaries over a finished token list - the one restatement of the reference's rules, compiled for the host
// (assemble.h: per-token fields of kiwi_res) and for the device (sents.cu: kiwi_split_into_sents*, kiwi_b200_split_batch).
//   bracket / bullet pairing   fillPairedTokenInfo, src/Kiwi.cpp:98-143   (getSSType src/Utils.cpp:184-261, getSBType 263-298)
//   SentenceSplitter           SentenceParser, src/Kiwi.cpp:145-290
//   foldSentLine               fillSentLineInfo, src/Kiwi.cpp:322-415   (hasSentences / isNestedLeft / isNestedRight 292-313)
//   sentRanges                 Kiwi::splitIntoSents, src/Kiwi.cpp:417-436
// Works on POD tokens and caller-provided scratch (no allocation), so that one warp lane can run it on the device.
#pragma once
#include <stdint.h>
#include "kb_model.h"

namespace kb
{
	enum : uint8_t { SF_YO = 1, SF_HA = 2 };      // SentTok::flags: the morpheme's kform is "요"; the token's form is "하"
	static constexpr uint32_t NO_PAIR = 0xFFFFFFFFu;

	struct SentTok
	{
		// in
		uint32_t position, length;
		uint8_t tag;                  // with the irregular bit, as TokenInfo::tag
		uint8_t ssType;               // ssTypeOf(form[0]) of an SSO / SSC token, else 0
		uint8_t sbType;               // sbTypeOf(form) of an SB token, else 0
		uint8_t flags;                // SF_*
		uint32_t wordPosition;        // in: word index in the whole text; out: word index inside its sentence
		uint32_t lineNumber;          // in: newlines before `position`; out: TokenInfo::lineNumber
		// out
		uint32_t sentPosition, subSentPosition, pairedToken;
		KB_HD uint32_t endPos() const { return position + length; }
	};

	// bracket / quote family of an opening or closing character, 0 = none
	KB_HD uint32_t ssTypeOf(uint32_t c)
	{
		switch (c)
		{
		case u'\'': return 1; case u'"': return 2; case u'(': case u')': return 3; case u'<': case u'>': return 4; case u'[': case u']': return 5;
		case u'{': case u'}': return 6; case 0x2018: case 0x2019: return 7; case 0x201c: case 0x201d: return 8; case 0x226a: case 0x226b: return 9;
		case 0x3008: case 0x3009: return 10; case 0x300a: case 0x300b: return 11; case 0x300c: case 0x300d: return 12; case 0x300e: case 0x300f: return 13;
		case 0x3010: case 0x3011: return 14; case 0x3014: case 0x3015: return 15; case 0x3016: case 0x3017: return 16; case 0x3018: case 0x3019: return 17;
		case 0x301a: case 0x301b: return 18; case 0xff08: case 0xff09: return 19; case 0xff1c: case 0xff1e: return 20; case 0xff3b: case 0xff3d: return 21;
		case 0xff5b: case 0xff5d: return 22; case 0xff5f: case 0xff60: return 23; case 0xff62: case 0xff63: return 24;
		}
		return 0;
	}

	// bullet family of an SB token's surface form
	KB_HD uint32_t sbTypeOf(const uint16_t* form, uint32_t len)
	{
		if (!len) return 0;
		uint32_t format = 0, group = 0;
		uint32_t chr = form[0];
		if (form[len - 1] == u'.') format = 1;
		else if (form[len - 1] == u')')
		{
			if (form[0] == u'(') { chr = len > 1 ? form[1] : 0; format = 2; }
			else format = 3;
		}
		if (0xAC00 <= chr && chr <= 0xD7A3) group = 1;
		else if (0x3131 <= chr && chr <= 0x314E) group = 2;
		else if (u'0' <= chr && chr <= u'9') group = 3;
		else if (0x2160 <= chr && chr <= 0x216B) group = 4;
		else if (0x2170 <= chr && chr <= 0x217B) group = 5;
		else if (0x2460 <= chr && chr <= 0x2473) return 24;
		else if (0x2780 <= chr && chr <= 0x2789) return 24;
		else if (0x2776 <= chr && chr <= 0x277F) return 25;
		else if (0x278A <= chr && chr <= 0x2793) return 25;
		else if (0x2474 <= chr && chr <= 0x2487) return 26;
		else if (0x2488 <= chr && chr <= 0x249B) return 27;
		return format | (group << 2);
	}

	// the per-token inputs that depend on the token's surface form
	KB_HD void setSentForm(SentTok& t, const uint16_t* form, uint32_t len)
	{
		const uint8_t tag = t.tag;
		t.ssType = (tag == T_sso || tag == T_ssc) && len ? (uint8_t)ssTypeOf(form[0]) : 0;
		t.sbType = tag == T_sb ? (uint8_t)sbTypeOf(form, len) : 0;
		if (len == 1 && form[0] == 0xD558) t.flags |= SF_HA;
	}

	// pairs opening with closing brackets and bullets with the next bullet of their family; qStack / bStack hold up to n entries each
	KB_HD void pairTokens(SentTok* toks, uint32_t n, uint2* qStack, uint2* bStack)
	{
		uint32_t nq = 0, nb = 0;      // stack entries: (token index, family)
		for (uint32_t i = 0; i < n; ++i)
		{
			SentTok& t = toks[i];
			if (t.tag == T_sso)
			{
				if (t.ssType) qStack[nq++] = uint2{ i, t.ssType };
			}
			else if (t.tag == T_ssc)
			{
				if (!t.ssType) continue;
				for (uint32_t j = nq; j-- > 0;)
				{
					if (qStack[j].y != t.ssType) continue;
					t.pairedToken = qStack[j].x;
					toks[qStack[j].x].pairedToken = i;
					nq = j;
					break;
				}
			}
			else if (t.tag == T_sb)
			{
				if (!t.sbType) continue;
				for (uint32_t j = nb; j-- > 0;)
				{
					if (bStack[j].y != t.sbType) continue;
					toks[bStack[j].x].pairedToken = i;
					nb = j;
					break;
				}
				bStack[nb++] = uint2{ i, t.sbType };
			}
		}
	}

	// sentence boundary automaton: a sentence ends after a final ending (+ optional "요", z_coda) or final punctuation,
	// followed by any run of closing symbols; see the rule comment at src/Kiwi.cpp:145-150
	class SentenceSplitter
	{
		enum { S_none, S_ef, S_efjx, S_zcoda, S_sf } state = S_none;
		uint32_t lastPosition = 0, lastLineNumber = 0;
		KB_HD static bool trailingSymbol(uint8_t tag) { return tag == T_so || tag == T_sw || tag == T_sh || tag == T_sp || tag == T_se || tag == T_ssc; }
	public:
		KB_HD bool next(uint8_t tag, bool isYo, uint32_t position, uint32_t length, uint32_t lineNumber, bool forceNewSent = false)
		{
			bool ret = false;
			if (forceNewSent)
			{
				state = S_none;
				lastPosition = position + length;
				return true;
			}
			if (state == S_none)
			{
				if (tag == T_ef) state = S_ef;
				else if (tag == T_sf) state = S_sf;
			}
			else if (state == S_ef || state == S_efjx)
			{
				if (state == S_ef && tag == T_vx) state = S_none;
				else if (tag == T_z_coda) state = S_zcoda;
				else if (isJClass(tag) || tag == T_vcp || tag == T_etm || tag == T_ec)
				{
					if (tag == T_jx && isYo)
					{
						if (state == S_ef) state = S_efjx;
						else { ret = true; state = S_none; }
					}
					else state = S_none;
				}
				else if (trailingSymbol(tag)) {}
				else if (tag == T_sf) state = S_sf;
				else if (tag == T_sso && lineNumber == lastLineNumber) {}
				else { ret = true; state = S_none; }
			}
			else if (state == S_zcoda)
			{
				if (trailingSymbol(tag) || tag == T_sf) {}
				else if (tag == T_sso && lineNumber == lastLineNumber) {}
				else { ret = true; state = S_none; }
			}
			else      // S_sf
			{
				if (trailingSymbol(tag)) {}
				else if (tag == T_sso)
				{
					if (lineNumber != lastLineNumber) { ret = true; state = S_none; }
				}
				else if ((tag == T_sl || tag == T_sn) && lastPosition == position) state = S_none;
				else { ret = true; state = S_none; }
			}
			lastPosition = position + length;
			lastLineNumber = lineNumber;
			return ret;
		}
		KB_HD bool next(const SentTok& t, uint32_t lineNumber, bool forceNewSent = false)
		{
			return next(t.tag, (t.flags & SF_YO) != 0, t.position, t.length, lineNumber, forceNewSent);
		}
	};

	KB_HD bool hasSentences(const SentTok* first, const SentTok* last)
	{
		SentenceSplitter sp;
		for (; first != last; ++first) if (sp.next(*first, 0)) return true;
		return sp.next(0, false, 0, 0, 0);      // (a default TokenInfo)
	}
	KB_HD bool isNestedLeft(const SentTok& t) { return isJClass(t.tag) || (isEClass(t.tag) && t.tag != T_ef) || t.tag == T_sp; }
	KB_HD bool isNestedRight(const SentTok& t) { return isJClass(t.tag) || isEClass(t.tag) || (isVerbClass(t.tag) && (t.flags & SF_HA)) || t.tag == T_vcp || t.tag == T_sp; }

	// sentence / line / sub-sentence numbers and the sentence-relative word index of every token (pairedToken filled by pairTokens)
	KB_HD void foldSentLine(SentTok* toks, uint32_t n)
	{
		SentenceSplitter sp;
		uint32_t sentPos = 0, lastSentPos = 0, subSentPos = 0, accumSubSent = 1, accumWordPos = 0, lastWordPos = 0;
		uint32_t nlPos = 0, lastNlPos = 0, nestedSentEnd = 0, nestedEnd = 0;
		for (uint32_t i = 0; i < n; ++i)
		{
			SentTok& t = toks[i];
			if (i >= nestedEnd && sp.next(t, nlPos, nestedSentEnd && i == nestedSentEnd))
			{
				// (rewrites token i - 1, whose sentPosition is already final otherwise: ranges are derived after the whole fold)
				const bool includePrevToken = i > 1
					&& (toks[i - 1].tag == T_so || toks[i - 1].tag == T_sw || toks[i - 1].tag == T_sp || toks[i - 1].tag == T_se || toks[i - 1].tag == T_sso)
					&& toks[i - 1].endPos() == toks[i].position
					&& toks[i - 1].position > toks[i - 2].endPos();
				if (nestedSentEnd)
				{
					subSentPos++;
					accumSubSent++;
					if (includePrevToken) toks[i - 1].subSentPosition = subSentPos;
				}
				else
				{
					sentPos++;
					accumSubSent = 1;
					if (includePrevToken)
					{
						toks[i - 1].sentPosition = sentPos;
						toks[i - 1].wordPosition = 0;
						accumWordPos = 0;
					}
				}
			}

			if (!nestedSentEnd && !nestedEnd && t.tag == T_sso && t.pairedToken != NO_PAIR)
			{
				if (!hasSentences(&toks[i], &toks[t.pairedToken]))
				{
					nestedEnd = t.pairedToken;
					subSentPos = 0;
				}
				else if ((t.pairedToken + 1 < n && isNestedRight(toks[t.pairedToken + 1])) || (i > 0 && isNestedLeft(toks[i - 1])))
				{
					nestedSentEnd = t.pairedToken;
					subSentPos = accumSubSent;
				}
			}
			else if (nestedSentEnd && i > nestedSentEnd) { nestedSentEnd = 0; subSentPos = 0; }
			else if (nestedEnd && i >= nestedEnd) { nestedEnd = 0; subSentPos = 0; }

			// (the reference advances one cursor over the newline list: the count so far never decreases)
			if (t.lineNumber > nlPos) nlPos = t.lineNumber;
			t.lineNumber = nlPos;
			if (nlPos > lastNlPos + 1 && sentPos == lastSentPos && !nestedSentEnd) sentPos++;
			t.sentPosition = sentPos;
			t.subSentPosition = (i == nestedSentEnd || i == toks[nestedSentEnd].pairedToken) ? 0 : subSentPos;

			if (sentPos != lastSentPos) { accumWordPos = 0; accumSubSent = 1; }
			else if (t.wordPosition != lastWordPos) accumWordPos++;
			lastWordPos = t.wordPosition;
			t.wordPosition = accumWordPos;

			lastSentPos = sentPos;
			lastNlPos = nlPos;
		}
	}

	// {begin, end} of every sentence from the final sentPosition of the folded tokens; returns the count (<= n)
	KB_HD uint32_t sentRanges(const SentTok* toks, uint32_t n, uint2* out)
	{
		uint32_t k = 0;
		for (uint32_t i = 0; i < n; ++i)
		{
			if (i == 0 || toks[i].sentPosition != toks[i - 1].sentPosition) out[k++] = uint2{ toks[i].position, toks[i].endPos() };
			else out[k - 1].y = toks[i].endPos();
		}
		return k;
	}

	// newline test of allNewLinePositions (src/Kiwi.cpp:69-96) at unit i: CR, LF not after a CR, VT, FF, NEL, LS, PS
	KB_HD bool isNewlineAt(const uint16_t* text, uint32_t i)
	{
		const uint16_t c = text[i];
		if (c == 0x0A) return !(i > 0 && text[i - 1] == 0x0D);
		return c == 0x0D || c == 0x0B || c == 0x0C || c == 0x85 || c == 0x2028 || c == 0x2029;
	}
}
