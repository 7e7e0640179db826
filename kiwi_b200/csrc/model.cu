// kiwi_b200: host-side model loading.  Reads a model image (include/kiwi_b200_image.h), derives the feature
// tables described in kb_model.h and uploads everything to the current device.
#include <cstdio>
#include <cstring>
#include <algorithm>
#include <cmath>
#include <stdexcept>
#include <string>
#include <vector>
#include <cuda_runtime.h>
#include "kb_model.h"
#include "engine.h"
#include "lm_tables.h"

namespace kb
{
	static void cudaCheck(cudaError_t e, const char* what)
	{
		if (e != cudaSuccess) throw std::runtime_error(std::string("CUDA error in ") + what + ": " + cudaGetErrorString(e));
	}

	std::vector<char> readImageFile(const std::string& modelPath)
	{
		std::string path = modelPath;
		FILE* f = std::fopen(path.c_str(), "rb");
		bool isDir = false;
		if (f)
		{
			// fopen succeeds on directories on Linux; detect by a failing read
			char probe;
			if (std::fread(&probe, 1, 1, f) != 1) { std::fclose(f); f = nullptr; isDir = true; }
			else std::fseek(f, 0, SEEK_SET);
		}
		if (!f)
		{
			path = modelPath + "/kiwi_b200.img";
			f = std::fopen(path.c_str(), "rb");
		}
		(void)isDir;
		if (!f) throw std::runtime_error("cannot open model image '" + modelPath + "' (expected an image file or a directory containing kiwi_b200.img)");
		std::fseek(f, 0, SEEK_END);
		const long n = std::ftell(f);
		std::fseek(f, 0, SEEK_SET);
		std::vector<char> blob((size_t)n);
		if (std::fread(blob.data(), 1, (size_t)n, f) != (size_t)n) { std::fclose(f); throw std::runtime_error("short read on " + path); }
		std::fclose(f);
		return blob;
	}

	// src/Utils.cpp:264-298 evaluated on the un-joined kform (joining codas cannot change the tested classes)
	static uint32_t getSBType(const uint16_t* form, uint32_t len)
	{
		if (!len) return 0;
		uint32_t format = 0, group = 0;
		uint32_t chr = form[0];
		if (form[len - 1] == '.') format = 1;
		else if (form[len - 1] == ')')
		{
			if (form[0] == '(') { chr = len > 1 ? form[1] : 0; format = 2; }
			else format = 3;
		}
		if (0xAC00 <= chr && chr <= 0xD7A3) group = 1;
		else if (0x3131 <= chr && chr <= 0x314E) group = 2;
		else if ('0' <= chr && chr <= '9') group = 3;
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

	template<class T> static T* upload(const std::vector<T>& v, std::vector<void*>& owned)
	{
		void* d = nullptr;
		const size_t bytes = std::max<size_t>(v.size() * sizeof(T), 16);
		cudaCheck(cudaMalloc(&d, bytes), "cudaMalloc(model)");
		if (!v.empty()) cudaCheck(cudaMemcpy(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice), "cudaMemcpy(model)");
		owned.push_back(d);
		return reinterpret_cast<T*>(d);
	}

	void Model::load(const void* bytes, size_t size)
	{
		blob.assign(reinterpret_cast<const char*>(bytes), reinterpret_cast<const char*>(bytes) + size);
		if (size < sizeof(kb2_header)) throw std::runtime_error("model image too small");
		const kb2_header* h = reinterpret_cast<const kb2_header*>(blob.data());
		if (h->magic != KB2_IMAGE_MAGIC) throw std::runtime_error("not a kiwi_b200 model image (bad magic)");
		if (h->version != KB2_IMAGE_VERSION) throw std::runtime_error("model image version mismatch: rebuild the image with this build's flatten tool");
		if (h->total_bytes != size) throw std::runtime_error("model image is truncated");
		if (h->model_type != 2 && h->model_type != 3 && h->model_type != 4) throw std::runtime_error("only Knlm, SkipBigram and CoNg (quantized, no window) images are supported by this build");
		if (h->model_type == 3 && (h->sb_window_size != 8 || h->sb_vocab_size == 0)) throw std::runtime_error("SkipBigram image: window size must be 8");
		const bool cong = h->model_type == 4;
		if (cong && (h->cg_dim == 0 || h->cg_dim % 32 != 0 || h->cg_dim > 1024)) throw std::runtime_error("CoNg image: dim must be a multiple of 32 (tensor-core tile depth)");
		header = *h;
		auto sec = [&](int id) { return blob.data() + h->sec[id].offset; };
		const kb2_trie_node* trieNodes = reinterpret_cast<const kb2_trie_node*>(sec(KB2_SEC_TRIE_NODES));
		const uint16_t* trieKeys = reinterpret_cast<const uint16_t*>(sec(KB2_SEC_TRIE_KEYS));
		const int32_t* trieDiffs = reinterpret_cast<const int32_t*>(sec(KB2_SEC_TRIE_DIFFS));
		const kb2_form* forms = reinterpret_cast<const kb2_form*>(sec(KB2_SEC_FORMS));
		const uint16_t* formChars = reinterpret_cast<const uint16_t*>(sec(KB2_SEC_FORM_CHARS));
		const uint32_t* formCands = reinterpret_cast<const uint32_t*>(sec(KB2_SEC_FORM_CANDS));
		const kb2_morph* morphs = reinterpret_cast<const kb2_morph*>(sec(KB2_SEC_MORPHS));
		const kb2_chr_run* runs = reinterpret_cast<const kb2_chr_run*>(sec(KB2_SEC_CHR_RUNS));
		hForms = forms; hFormChars = formChars; hMorphs = morphs;

		// ---- code point table
		std::vector<uint32_t> bmp(0x10000, 0);
		for (uint32_t i = 0; i < h->n_chr_runs; ++i)
		{
			const uint32_t s = runs[i].start, e = i + 1 < h->n_chr_runs ? runs[i + 1].start : 0x110000u;
			for (uint32_t c = s; c < e && c < 0x10000; ++c) bmp[c] = (uint32_t)runs[i].cls | ((uint32_t)runs[i].script << 8) | ((uint32_t)runs[i].flags << 16);
		}
		hChrBmp = bmp;
		// ---- root direct table
		std::vector<int32_t> rootNext(0x10000, -1);
		for (uint32_t i = 0; i < trieNodes[0].num_nexts; ++i) rootNext[trieKeys[trieNodes[0].next_offset + i]] = trieDiffs[trieNodes[0].next_offset + i];

		// ---- form features
		std::vector<DForm> dforms(h->n_forms);
		for (uint32_t i = 0; i < h->n_forms; ++i)
		{
			const kb2_form& f = forms[i];
			const uint16_t* s = formChars + f.str_off;
			DForm d;
			d.cand_off = f.cand_off; d.cand_cnt = f.cand_cnt; d.str_len = f.str_len;
			d.size_no_space = (uint16_t)(f.str_len - f.num_spaces);
			d.last_chr = f.str_len ? s[f.str_len - 1] : 0;
			d.num_spaces = f.num_spaces;
			uint8_t fl = f.flags & (FF_ZCODA | FF_ZSIOT | FF_HASFULL);
			const uint16_t c0 = f.str_len ? s[0] : 0;
			const uint8_t cls0 = attrCls(bmp[c0]);
			const bool isSTag = f.str_len == 1 && cls0 >= T_sf && cls0 <= T_sw;
			if ((f.flags & KB2_FORM_HASJ) || isSTag) fl |= FF_HASJ_OR_STAG;
			if (isHangulCoda(c0)) fl |= FF_FIRST_IS_CODA;
			bool allPartial = true;
			for (uint32_t c = 0; c < f.cand_cnt; ++c)
			{
				const kb2_morph& m = morphs[formCands[f.cand_off + c]];
				const bool single = m.chunk_cnt == 0 || (m.flags & (KB2_MORPH_COMPLEX | KB2_MORPH_SAISIOT));
				if (!(m.combine_socket || !single)) { allPartial = false; break; }
			}
			if (allPartial) fl |= FF_ALL_PARTIAL;
			if (c0 == 0xC544) fl |= FF_FIRST_IS_A;
			d.flags = fl;
			uint8_t pol = 0;
			if (ftPolar(s, f.str_len, CP_positive)) pol |= FP_POLAR_POS;
			if (ftPolar(s, f.str_len, CP_negative)) pol |= FP_POLAR_NEG;
			if (f.str_len && attrCls(bmp[d.last_chr]) == T_ssc) pol |= FP_LAST_SSC;
			d.pol = pol;
			dforms[i] = d;
		}
		// ---- morpheme features
		std::vector<DMorph> dmorphs(h->n_morphs);
		for (uint32_t i = 0; i < h->n_morphs; ++i)
		{
			const kb2_morph& m = morphs[i];
			const uint16_t* kf = m.form_idx >= 0 ? formChars + forms[m.form_idx].str_off : nullptr;
			const uint32_t kl = m.form_idx >= 0 ? forms[m.form_idx].str_len : 0;
			const uint16_t k0 = kl ? kf[0] : 0, kb = kl ? kf[kl - 1] : 0;
			uint32_t feat = m.tag;
			const bool verb = isVerbClass(m.tag);
			if (verb) feat |= MF_VERB;
			if (m.tag == T_np && kl == 1 && (k0 == 0xB098 || k0 == 0xB108 || k0 == 0xC800)) feat |= MF_INFL_NP;
			if (verb && kf && kl && kb == 0x11AF) feat |= MF_VERB_L;
			if (verb && ftPolar(kf, kl, CP_positive)) feat |= MF_POS_VERB;          // null kform -> begin == end -> matched
			if (verb && kf && kl && !isHangulCoda(kb)) feat |= MF_VERB_VOWEL;
			uint32_t special = 7;
			for (uint32_t k = 0; k < 6; ++k) if (h->special_morph_ids[k] == i) { special = k; break; }
			feat |= special << MF_SPECIAL_SHIFT;
			const uint32_t sb = m.tag == T_sb ? getSBType(kf, kl) : 0;
			feat |= (sb & 31) << MF_SBTYPE_SHIFT;
			if (isEClass(m.tag) && kf && (0xC544 <= k0 && k0 <= 0xC774)) feat |= MF_VOWEL_E;
			if ((m.tag == T_jks || m.tag == T_jkc) && kl == 1 && k0 == 0xAC00) feat |= MF_INF_J;
			if (k0 == 0xC73C || k0 == 0xB290 || (0xC0AC <= k0 && k0 <= 0xC2DC)) feat |= MF_BADPAIR_L;
			if (isEClass(m.tag) && kf && kl && k0 == 0xC5B4) feat |= MF_CONTRACT_E;
			const bool single = m.chunk_cnt == 0 || (m.flags & (KB2_MORPH_COMPLEX | KB2_MORPH_SAISIOT));
			if (single) feat |= MF_SINGLE;
			feat |= ((uint32_t)m.polar & 3) << MF_POLAR_SHIFT;
			feat |= ((uint32_t)m.vowel & 15) << MF_VOWEL_SHIFT;
			DMorph d;
			d.feat = feat; d.lm_id = m.lm_morpheme_id; d.combined = m.combined; d.chunk_off = m.chunk_off; d.user_score = m.user_score;
			d.form_idx = m.form_idx; d.chunk_cnt = m.chunk_cnt; d.combine_socket = m.combine_socket; d.sense_id = m.sense_id;
			d.nonstd_dialect = m.dialect != 0;
			d.misc = ((m.flags & KB2_MORPH_COMPLEX) ? MM_COMPLEX : 0) | ((m.flags & KB2_MORPH_SAISIOT) ? MM_SAISIOT : 0) | (kl == 1 && k0 == 0xC694 ? MM_KFORM_YO : 0);
			dmorphs[i] = d;
		}

		// ---- static candidate data
		const kb2_chunk* chunksH = reinterpret_cast<const kb2_chunk*>(sec(KB2_SEC_MORPH_CHUNKS));
		std::vector<uint32_t> chunkLm(h->n_chunks);
		for (uint32_t i = 0; i < h->n_chunks; ++i) chunkLm[i] = morphs[chunksH[i].morph].lm_morpheme_id;
		std::vector<DMorphX> dmx(h->n_morphs);
		for (uint32_t i = 0; i < h->n_morphs; ++i)
		{
			const kb2_morph& m = morphs[i];
			const bool single = (dmorphs[i].feat & MF_SINGLE) != 0;
			DMorphX x;
			int64_t lastMorph;
			if (single) { lastMorph = m.combined ? (int64_t)i + m.combined : (int64_t)i; x.first_wid = m.lm_morpheme_id; }
			else { lastMorph = chunksH[m.chunk_off + m.chunk_cnt - 1].morph; x.first_wid = chunkLm[m.chunk_off]; }
			if (lastMorph < 0 || lastMorph >= (int64_t)h->n_morphs) lastMorph = i;
			if ((uint64_t)lastMorph >= h->lang_vocab_size) x.last_seq_id = (uint32_t)lastMorph;
			else x.last_seq_id = morphs[lastMorph].lm_morpheme_id;
			if (x.last_seq_id >= h->n_morphs) x.last_seq_id = 0;
			if (x.first_wid >= h->n_morphs) x.first_wid = 0;
			x.last_seq_feat = dmorphs[x.last_seq_id].feat;
			// left form seen by FormEvaluator when the path has no own form: kform of morphemes[wid], else of the morpheme
			int32_t fi = morphs[x.last_seq_id].form_idx;
			if (!(fi >= 0 && forms[fi].str_len)) fi = m.form_idx;
			uint16_t leftLast; uint8_t leftPol;
			if (fi < 0 || forms[fi].str_len == 0) { leftLast = 0; leftPol = LP_EMPTY | LP_POLAR_POS | LP_POLAR_NEG; }
			else { leftLast = dforms[fi].last_chr; leftPol = dforms[fi].pol & (FP_POLAR_POS | FP_POLAR_NEG | FP_LAST_SSC); }
			if (m.combine_socket) leftPol |= LP_MORPH_SOCKET;
			uint8_t xf = 0;
			if ((dmorphs[x.first_wid].feat & MF_TAG_MASK) == T_p) xf |= MX_FIRST_IS_P;
			if (!single) for (uint32_t c = 1; c < m.chunk_cnt; ++c) if ((dmorphs[chunkLm[m.chunk_off + c]].feat & MF_TAG_MASK) == T_p) xf |= MX_CHUNK_HAS_P;
			// the created path: morph_tag = the candidate's tag, combineSocket only for single morphemes (BestPathContainer.hpp:451-469)
			x.fw_x = fwOfLeft(leftLast, leftPol) | fwOfTag(m.tag, single ? m.combine_socket : 0) | ((uint32_t)xf << 24);
			dmx[i] = x;
		}

		// ---- static candidate records, parallel to form_cands (+ the unknown NNG / NNP records): kb_model.h DCand
		const uint32_t nFormCands = (uint32_t)(h->sec[KB2_SEC_FORM_CANDS].nbytes / 4);
		std::vector<DCand> dcands(nFormCands + 2);
		auto makeCand = [&](uint32_t curId, bool formStartsWithA)
		{
			DCand c; std::memset(&c, 0, sizeof(c));
			const kb2_morph& m = morphs[curId];
			const DMorph& dm = dmorphs[curId];
			const DMorphX& mx = dmx[curId];
			const bool single = (dm.feat & MF_SINGLE) != 0;
			const uint32_t tag = dm.feat & MF_TAG_MASK;
			c.cur_id = (int32_t)curId; c.first_wid = mx.first_wid; c.last_seq_id = mx.last_seq_id; c.last_seq_feat = mx.last_seq_feat;
			c.feat = dm.feat; c.user_score = m.user_score; c.chunk_off = m.chunk_off; c.fw_new = mx.fw_x & FW_PATH_MASK;
			c.chunk_cnt = m.chunk_cnt; c.sense_id = m.sense_id; c.cur_socket = m.combine_socket; c.path_socket = single ? m.combine_socket : 0;
			c.tag_clean = clearIrregular((uint8_t)tag);
			uint8_t kind = 0;
			if (m.dialect != 0) kind |= DK_DIALECT;
			{
				bool cx = (dmorphs[(int64_t)curId + m.combined].misc & MM_COMPLEX) != 0;
				for (uint32_t k = 0; k < m.chunk_cnt && !cx; ++k) if (dmorphs[chunksH[m.chunk_off + k].morph].misc & MM_COMPLEX) cx = true;
				if (cx) kind |= DK_COMPLEX;
			}
			if (tag == T_z_coda) kind |= DK_SHORTCUT_CODA;
			if (tag == T_z_siot) kind |= DK_SHORTCUT_SIOT;
			if (!single && m.form_idx >= 0 && forms[m.form_idx].str_len == 1)
			{
				const uint16_t k0 = formChars[forms[m.form_idx].str_off];
				if (k0 == 0xB2E4 || k0 == 0xAC8C || k0 == 0xC9C0)
				{
					const kb2_morph& c0 = morphs[chunksH[m.chunk_off].morph];
					if (c0.form_idx >= 0 && forms[c0.form_idx].str_len == 1 && formChars[forms[c0.form_idx].str_off] == 0xD558) kind |= DK_HA;
				}
			}
			const uint8_t xf = (uint8_t)(mx.fw_x >> 24);
			if (xf & MX_FIRST_IS_P) kind |= DK_FIRST_IS_P;
			if (xf & MX_CHUNK_HAS_P) kind |= DK_CHUNK_HAS_P;
			if (tag == T_sn) kind |= DK_IS_SN;
			c.kind = kind;
			const uint32_t specialType = (dm.feat >> MF_SPECIAL_SHIFT) & 7, sbType = (dm.feat >> MF_SBTYPE_SHIFT) & 31;
			const bool fork = sbType != 0 || specialType == 0 || specialType == 1 || specialType == 3 || specialType == 4;
			uint8_t fl = 0;
			if (isEClass((uint8_t)tag) && formStartsWithA) fl |= CS_POSITIVE_E;
			if (single) fl |= CS_SINGLE;
			if (m.combine_socket && single) fl |= CS_NO_LM;
			if (fork) fl |= CS_FORK;
			if (m.combine_socket && !single) fl |= CS_SOCKET_CHUNK;
			c.flags = fl;
			return c;
		};
		for (uint32_t i = 0; i < h->n_forms; ++i)
		{
			const kb2_form& f = forms[i];
			const bool startsA = f.str_len && formChars[f.str_off] == 0xC544;
			bool special = false;
			for (uint32_t c = 0; c < f.cand_cnt; ++c)
			{
				const DCand dc = makeCand(formCands[f.cand_off + c], startsA);
				dcands[f.cand_off + c] = dc;
				if ((dc.kind & (DK_SHORTCUT_CODA | DK_SHORTCUT_SIOT)) || (dc.flags & CS_FORK)) special = true;
			}
			if (special) dforms[i].flags |= FF_HAS_SPECIAL;
		}
		dcands[nFormCands] = makeCand(T_nng + 1u, false);          // getDefaultMorphemeId, Kiwi.h:64-67
		dcands[nFormCands + 1] = makeCand(T_nnp + 1u, false);

		// ---- Knlm and CoNg one-probe layouts (lm_tables.h): the fourth word of an entry is the child's ll / context id for an inner
		// edge and the state after the edge for a leaf, so no LM step walks a suffix chain on the device
		const kb2_kn_node* knNodes = reinterpret_cast<const kb2_kn_node*>(sec(KB2_SEC_KN_NODES));
		KnTables kn = buildKnTables(h, knNodes, reinterpret_cast<const uint32_t*>(sec(KB2_SEC_KN_KEYS)), reinterpret_cast<const int32_t*>(sec(KB2_SEC_KN_VALUES)),
		                            reinterpret_cast<const int32_t*>(sec(KB2_SEC_KN_ROOT)), h->kn_has_htx ? reinterpret_cast<const uint32_t*>(sec(KB2_SEC_KN_HTX)) : nullptr);
		CgTables cg;
		if (cong)
			cg = buildCgTables(h, reinterpret_cast<const kb2_cg_node*>(sec(KB2_SEC_CG_NODES)), reinterpret_cast<const uint32_t*>(sec(KB2_SEC_CG_KEYS)),
			                   reinterpret_cast<const int32_t*>(sec(KB2_SEC_CG_VALUES)), reinterpret_cast<const int32_t*>(sec(KB2_SEC_CG_ROOT)));

		// ---- upload
		void* dBlob = nullptr;
		cudaCheck(cudaMalloc(&dBlob, size), "cudaMalloc(image)");
		owned.push_back(dBlob);
		cudaCheck(cudaMemcpy(dBlob, blob.data(), size, cudaMemcpyHostToDevice), "cudaMemcpy(image)");
		auto dsec = [&](int id) { return reinterpret_cast<const char*>(dBlob) + h->sec[id].offset; };
		DevModel& d = dev;
		std::memset(&d, 0, sizeof(d));
		d.trie_nodes = reinterpret_cast<const kb2_trie_node*>(dsec(KB2_SEC_TRIE_NODES));
		d.trie_keys = reinterpret_cast<const uint16_t*>(dsec(KB2_SEC_TRIE_KEYS));
		d.trie_diffs = reinterpret_cast<const int32_t*>(dsec(KB2_SEC_TRIE_DIFFS));
		d.forms_raw = reinterpret_cast<const kb2_form*>(dsec(KB2_SEC_FORMS));
		d.form_chars = reinterpret_cast<const uint16_t*>(dsec(KB2_SEC_FORM_CHARS));
		d.form_cands = reinterpret_cast<const uint32_t*>(dsec(KB2_SEC_FORM_CANDS));
		d.chunks = reinterpret_cast<const kb2_chunk*>(dsec(KB2_SEC_MORPH_CHUNKS));
		d.kn_nodes = reinterpret_cast<const kb2_kn_node*>(dsec(KB2_SEC_KN_NODES));
		d.kn_keys = reinterpret_cast<const uint32_t*>(dsec(KB2_SEC_KN_KEYS));
		d.kn_values = reinterpret_cast<const int32_t*>(dsec(KB2_SEC_KN_VALUES));
		d.kn_root = reinterpret_cast<const int32_t*>(dsec(KB2_SEC_KN_ROOT));
		d.kn_htx = h->kn_has_htx ? reinterpret_cast<const uint32_t*>(dsec(KB2_SEC_KN_HTX)) : nullptr;
		d.chr_runs = reinterpret_cast<const kb2_chr_run*>(dsec(KB2_SEC_CHR_RUNS));
		d.morphs = upload(dmorphs, owned);
		d.morphx = upload(dmx, owned);
		d.cands = upload(dcands, owned); d.cand_unk = nFormCands;
		hCands = dcands;
		d.chunk_lm = upload(chunkLm, owned);
		d.kn_hash = upload(kn.hash, owned); d.kn_hash_mask = (uint32_t)kn.hash.size() - 1;
		d.kn_backoff = upload(kn.backoff, owned);
		d.kn_root_ll = upload(kn.rootLl, owned);
		d.forms = upload(dforms, owned);
		d.chr_bmp = upload(bmp, owned);
		d.trie_root_next = upload(rootNext, owned);
		d.model_type = h->model_type;
		if (cong)
		{
			d.cg_hash = upload(cg.hash, owned); d.cg_hash_mask = (uint32_t)cg.hash.size() - 1;
			d.cg_nodes = upload(cg.nodes, owned);
			d.cg_root = reinterpret_cast<const int32_t*>(dsec(KB2_SEC_CG_ROOT));
			d.cg_ctx_emb = reinterpret_cast<const uint8_t*>(dsec(KB2_SEC_CG_CTX_EMB));
			d.cg_out_emb = reinterpret_cast<const uint8_t*>(dsec(KB2_SEC_CG_OUT_EMB));
			d.cg_inv_vocab = h->sec[KB2_SEC_CG_INV_VOCAB].nbytes ? reinterpret_cast<const uint32_t*>(dsec(KB2_SEC_CG_INV_VOCAB)) : nullptr;
			d.cg_out_bias = h->sec[KB2_SEC_CG_OUT_BIAS].nbytes ? reinterpret_cast<const float*>(dsec(KB2_SEC_CG_OUT_BIAS)) : nullptr;
			d.cg_dim = h->cg_dim; d.cg_stride = h->cg_dim + 8; d.cg_key_size = h->cg_key_size; d.cg_root_size = h->cg_root_size; d.cg_context_size = h->cg_context_size;
		}
		if (h->model_type == 3)
		{
			d.sb_ptrs = reinterpret_cast<const uint32_t*>(dsec(KB2_SEC_SB_PTRS)); d.sb_keys = reinterpret_cast<const uint32_t*>(dsec(KB2_SEC_SB_KEYS));
			d.sb_comps = reinterpret_cast<const float*>(dsec(KB2_SEC_SB_COMPS)); d.sb_discnts = reinterpret_cast<const float*>(dsec(KB2_SEC_SB_DISCNTS));
			d.sb_valid = reinterpret_cast<const uint8_t*>(dsec(KB2_SEC_SB_VALID));
			d.sb_vocab_size = h->sb_vocab_size; d.sb_log_window = std::log((float)h->sb_window_size);      // (SkipBigramModel.hpp:104)
		}
		d.n_chr_runs = h->n_chr_runs; d.n_morphs = h->n_morphs; d.n_forms = h->n_forms; d.n_trie_nodes = h->n_trie_nodes;
		d.default_tag_size = h->default_tag_size; d.lang_vocab_size = h->lang_vocab_size;
		d.script_latin = h->script_latin; d.script_variation_selectors = h->script_variation_selectors;
		d.kn_bos_node = h->kn_bos_node; d.kn_unk_ll = h->kn_unk_ll; d.kn_htx_vocab = h->kn_htx_vocab;
		{ std::vector<uint32_t> z(64, 0); d.debug = upload(z, owned); }
		for (int i = 0; i < 6; ++i) d.special_morph_ids[i] = h->special_morph_ids[i];
		d.cfg = h->config;
		std::memcpy(d.tag_left_boundary, h->tag_left_boundary, sizeof(d.tag_left_boundary));
		deviceBytes = size + dmorphs.size() * sizeof(DMorph) + dforms.size() * sizeof(DForm) + bmp.size() * 4 + rootNext.size() * 4;
	}

	std::vector<DCand> Model::blockedCands(const std::vector<uint32_t>& ids) const
	{
		std::vector<DCand> out = hCands;
		if (ids.empty()) return out;
		const kb2_chunk* chunksH = reinterpret_cast<const kb2_chunk*>(blob.data() + header.sec[KB2_SEC_MORPH_CHUNKS].offset);
		auto listed = [&](uint32_t m) { return std::binary_search(ids.begin(), ids.end(), m); };
		for (DCand& c : out)
		{
			const kb2_morph& m = hMorphs[c.cur_id];
			bool hit = listed((uint32_t)(c.cur_id + m.combined));      // Morpheme::hasMorpheme (include/kiwi/Form.h:187-196): getCombined() or a chunk
			for (uint32_t k = 0; k < m.chunk_cnt && !hit; ++k) hit = listed(chunksH[m.chunk_off + k].morph);
			if (hit) c.kind |= DK_DIALECT;
		}
		return out;
	}

	std::vector<uint32_t> Model::findMorphemes(const uint16_t* form, size_t len, uint8_t tag) const
	{
		// normalizeHangul (src/StrUtils.h:493-520): a syllable with a coda becomes the open syllable + the coda jamo
		std::u16string key;
		for (size_t i = 0; i < len; ++i)
		{
			const uint16_t c = form[i];
			if (c >= 0xAC00 && c <= 0xD7A3 && (c - 0xAC00) % 28) { const uint16_t t = (uint16_t)((c - 0xAC00) % 28); key.push_back((char16_t)(c - t)); key.push_back((char16_t)(0x11A7 + t)); }
			else key.push_back((char16_t)c);
		}
		if (formIndex_.empty())
		{
			formIndex_.reserve(header.n_forms * 2);
			for (uint32_t i = 0; i < header.n_forms; ++i)
			{
				const kb2_form& f = hForms[i];
				formIndex_.emplace(std::u16string(reinterpret_cast<const char16_t*>(hFormChars + f.str_off), f.str_len), i);      // (the trie keeps the first form of a spelling)
			}
		}
		std::vector<uint32_t> out;
		const auto it = formIndex_.find(key);
		if (it == formIndex_.end()) return out;
		const uint32_t* formCands = reinterpret_cast<const uint32_t*>(blob.data() + header.sec[KB2_SEC_FORM_CANDS].offset);
		const kb2_form& f = hForms[it->second];
		tag &= 0x7F;
		for (uint32_t c = 0; c < f.cand_cnt; ++c)
		{
			const uint32_t id = formCands[f.cand_off + c];
			const kb2_morph& m = hMorphs[id];
			if (m.combine_socket || (tag != 0 && (m.tag & 0x7F) != tag)) continue;
			out.push_back(id);
		}
		return out;
	}

	Model::~Model()
	{
		for (void* p : owned) cudaFree(p);
	}
}
