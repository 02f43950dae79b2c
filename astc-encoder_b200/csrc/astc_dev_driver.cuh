// CUDA-native ASTC block compressor: trial functions and the compress_block search driver
// (astcenc_compress_symbolic.cpp:353-1455). Control flow is uniform across the warp.
#pragma once

ASTC_FN float min_ep_cutoff(float e0, float e1, float cur) {
	float ep = (1.0f - e0) / (e1 - e0);
	bool use = (ep > 0.5f) && (ep < cur);
	return use ? ep : cur;
}

// Quantise the decimated ideal weights of one winning block mode straight into the work candidate
// (the reference keeps every mode's quantised set in dec_weights_uquant; we recompute the winners).
// (dst: 64 bytes, plane 2 at +32; no barrier inside - the caller synchronises once after its last call)
ASTC_FN void quantize_candidate_weights_to(const WCtx& w, SPtr<uint8_t> dst, int decimation_mode, int quant_mode, int nplanes, float cutoff1, float cutoff2) {
	DecView di = dec_view((unsigned int)decimation_mode);
	int W = di.W;
	SPtr<float> dwi = dwi_of(w) + di.dwi_offset;
	ASTC_NOUNROLL
	for (int id = w.lane; id < W * nplanes; id += ASTC_WARP) {
		int pl = id >= W ? 1 : 0;
		int k = id - pl * W;
		float low, high;
		mode_low_high(w, decimation_mode, quant_mode, pl, pl ? cutoff2 : cutoff1, low, high);
		WeightQuantizer z = make_weight_quantizer(low, high, quant_mode);
		dst[pl * 32 + k] = (uint8_t)quantize_weight(z, dwi[id]);
	}
}
ASTC_FN void quantize_candidate_weights_t(const WCtx& w, int decimation_mode, int quant_mode, int nplanes, float cutoff1, float cutoff2) {
	quantize_candidate_weights_to(w, work_weights_of(w), decimation_mode, quant_mode, nplanes, cutoff1, cutoff2);
	wsync();
}
ASTC_COOP void quantize_candidate_weights(WCtx w, int decimation_mode, int quant_mode, int nplanes, float cutoff1, float cutoff2) {
	quantize_candidate_weights_t(w, decimation_mode, quant_mode, nplanes, cutoff1, cutoff2);
}

ASTC_FN void copy_work_to_best_t(const WCtx& w) {
	// best_weights[64] best_colors[32] | work_weights[64] work_colors[32]: one word per lane
	SPtr<uint32_t> dst = sptr<uint32_t>(w.base + A_SCB);
	SPtr<uint32_t> src = sptr<uint32_t>(w.base + A_SCB + 96);
	ASTC_NOUNROLL
	for (int i = w.lane; i < 24; i += ASTC_WARP) {
		dst[i] = src[i];
	}
	wsync();
}
ASTC_COOP void copy_work_to_best(WCtx w) {
	copy_work_to_best_t(w);
}

// Pack the endpoints of partitions 0..pc-1 of the work candidate at quant_level into colors (work_colors or
// mod_colors). LDR formats: lanes over partitions; HDR formats: one partition after the other, the warp running the
// format's sub-mode ladder lane-parallel. The resulting formats come back packed 8 bits each (exchanged via tmpf).
// L1: one partition and LDR formats are compile-time facts; the RGB / RGBA contest is inlined, the HDR packers are left out.
template <bool L1> ASTC_FN uint32_t pack_work_endpoints_t(const WCtx& w, unsigned int pc_in, uint32_t formats_in, int quant_level, uint32_t colors_off) {
	const unsigned int pc = L1 ? 1u : pc_in;
	SPtr<f4> ep = ep_of(w);
	SPtr<uint8_t> colors = sptr<uint8_t>(colors_off);
	SPtr<uint32_t> colors32 = sptr<uint32_t>(colors_off);
	SPtr<uint32_t> xch = sptr<uint32_t>(w.base + A_TMPF);
	ASTC_NOUNROLL
	for (int k = w.lane; k < 2 * (int)pc; k += ASTC_WARP) {
		colors32[k] = 0;
	}
	wsync();
	// one partition, RGB / RGBA (nearly every LDR candidate): the four encodings of the pair run on four lanes
	const int fmt0 = (int)(formats_in & 0xFF);
#if defined(ASTC_PACK_ONE_LANE)
	const bool rgb_coop = false;
#else
	const bool rgb_coop = pc == 1 && (fmt0 == FMT_RGB || fmt0 == FMT_RGBA);
#endif
	if (rgb_coop) {
		uint8_t fmt = L1 ? pack_rgb_endpoints_coop_t<true>(w.lane, ep[EP_WORK_0], ep[EP_WORK_1], fmt0, &colors[0], quant_level)
		                 : pack_rgb_endpoints_coop(w.lane, ep[EP_WORK_0], ep[EP_WORK_1], fmt0, &colors[0], quant_level);
		if (w.lane == 0) {
			xch[0] = fmt;
		}
	}
	ASTC_NOUNROLL
	for (unsigned int j = (unsigned int)w.lane; j < pc && !rgb_coop; j += ASTC_WARP) {
		int fmt_in = (int)((formats_in >> (8 * j)) & 0xFF);
		if (L1 || !is_hdr_format(fmt_in)) {
			// (packed straight into the shared arena: a local byte array behind a pointer would live in local memory)
			xch[(int)j] = pack_color_endpoints(ep[EP_WORK_0 + (int)j], ep[EP_WORK_1 + (int)j], ep[EP_RGBS + (int)j], ep[EP_RGBO + (int)j], fmt_in, &colors[(int)j * 8], quant_level);
		}
	}
	ASTC_NOUNROLL
	for (unsigned int j = 0; j < pc; j++) {
		int fmt_in = (int)((formats_in >> (8 * j)) & 0xFF);
		if (!L1 && is_hdr_format(fmt_in)) {
			uint8_t fmt = pack_hdr_endpoints(w.lane, ep[EP_WORK_0 + (int)j], ep[EP_WORK_1 + (int)j], ep[EP_RGBO + (int)j], fmt_in, &colors[(int)j * 8], quant_level);
			if (w.lane == 0) {
				xch[(int)j] = fmt;
			}
		}
	}
	wsync();
	uint32_t r = 0;
	for (unsigned int j = 0; j < 4; j++) {
		if (j < pc) {
			r |= (xch[(int)j] & 0xFF) << (8 * j);
		}
	}
	wsync();
	return r;
}
ASTC_COOP uint32_t pack_work_endpoints(WCtx w, unsigned int pc, uint32_t formats_in, int quant_level, uint32_t colors_off) {
	return pack_work_endpoints_t<false>(w, pc, formats_in, quant_level, colors_off);
}

ASTC_FN void set_formats(ScbHdr& h, uint32_t f) {
	h.color_formats[0] = (uint8_t)f;
	h.color_formats[1] = (uint8_t)(f >> 8);
	h.color_formats[2] = (uint8_t)(f >> 16);
	h.color_formats[3] = (uint8_t)(f >> 24);
}

// The candidate refinement loop shared by both trial kinds (:504-699 and :886-1044).
// base endpoints are in slots EP_BASE_*; returns best_errorval_in_mode.
ASTC_COOP float refine_candidates(WCtx w, unsigned int pc, unsigned int packed, bool dual, unsigned int partition_index,
                                  int plane2_component, unsigned int candidate_count, float cutoff1, float cutoff2,
                                  float tune_errorval_threshold, ScbHdr& scb) {
	PartView pi = part_view_packed(pc, packed);
	unsigned int partition_count = pc;
	unsigned int refinement_limit = CFG.tune_refinement_limit;
	float best_errorval_in_mode = ERROR_CALC_DEFAULT;
	float best_errorval_in_scb = scb.errorval;
	SPtr<Candidate> cands = cand_of(w);
	SPtr<f4> ep = ep_of(w);
	ASTC_NOUNROLL
	for (unsigned int i = 0; i < candidate_count; i++) {
		Candidate cd = cands[(int)i];
		const DevBlockMode* qw_bm = BSD.block_modes + cd.block_mode;
		int dmode = ASTC_LDG(&qw_bm->decimation_mode);
		int qmode = ASTC_LDG(&qw_bm->quant_mode);
		uint16_t mode_index = ASTC_LDG(&qw_bm->mode_index);
		uint32_t cd_formats = (uint32_t)cd.formats[0] | ((uint32_t)cd.formats[1] << 8) | ((uint32_t)cd.formats[2] << 16) | ((uint32_t)cd.formats[3] << 24);
		quantize_candidate_weights(w, dmode, qmode, dual ? 2 : 1, cutoff1, cutoff2);
		ASTC_NOUNROLL
		for (int k = w.lane; k < 4; k += ASTC_WARP) {
			ep[EP_WORK_0 + k] = ep[EP_BASE_0 + k];
			ep[EP_WORK_1 + k] = ep[EP_BASE_1 + k];
			ep[EP_RGBS + k] = splat4(0.0f);
			ep[EP_RGBO + k] = splat4(0.0f);
		}
		{
			SPtr<uint32_t> wc32 = sptr<uint32_t>(work_colors_of(w).off);
			ASTC_NOUNROLL
			for (int k = w.lane; k < 8; k += ASTC_WARP) {
				wc32[k] = 0;
			}
		}
		wsync();
		ScbHdr work;
		work.errorval = 0.0f;
		work.color_formats[0] = work.color_formats[1] = work.color_formats[2] = work.color_formats[3] = 0;
		work.constant_color[0] = work.constant_color[1] = work.constant_color[2] = work.constant_color[3] = 0;
		ASTC_NOUNROLL
		for (unsigned int l = 0; l < refinement_limit; l++) {
			uint32_t formats;
			if (dual) {
				recompute_ideal_colors_2planes(w, (unsigned int)dmode, plane2_component);
				formats = pack_work_endpoints(w, 1, cd_formats, cd.quant_level, work_colors_of(w).off);
				set_formats(work, formats & 0xFF);
				work.partition_count = 1;
				work.partition_index = 0;
				work.quant_mode = cd.quant_level;
				work.color_formats_matched = 0;
				work.block_mode = mode_index;
				work.plane2_component = static_cast<int8_t>(plane2_component);
				work.block_type = SYM_BTYPE_NONCONST;
			} else {
				recompute_ideal_colors_1plane(w, pi, (unsigned int)dmode);
				formats = pack_work_endpoints(w, partition_count, cd_formats, cd.quant_level, work_colors_of(w).off);
				bool all_same = cd.quant_level != cd.quant_level_mod;
				for (unsigned int j = 1; j < 4; j++) {
					if (j < partition_count) {
						all_same = all_same && ((formats >> (8 * j)) & 0xFF) == (formats & 0xFF);
					}
				}
				work.color_formats_matched = 0;
				if (partition_count >= 2 && all_same) {
					{
						SPtr<uint32_t> mc32 = sptr<uint32_t>(mod_colors_of(w).off);
						ASTC_NOUNROLL
						for (int k = w.lane; k < 8; k += ASTC_WARP) {
							mc32[k] = 0;
						}
					}
					wsync();
					// (the reference stops packing at the first format mismatch; the later partitions' values are then unused)
					uint32_t formats_mod = pack_work_endpoints(w, partition_count, cd_formats, cd.quant_level_mod, mod_colors_of(w).off);
					bool all_same_mod = true;
					uint32_t kept = formats_mod & 0xFF;
					for (unsigned int j = 1; j < 4; j++) {
						if (j < partition_count && all_same_mod) {
							uint32_t fj = (formats_mod >> (8 * j)) & 0xFF;
							if (fj != (formats_mod & 0xFF)) {
								all_same_mod = false;
							} else {
								kept |= fj << (8 * j);
							}
						}
					}
					if (all_same_mod) {
						work.color_formats_matched = 1;
						SPtr<uint32_t> wc32 = sptr<uint32_t>(work_colors_of(w).off);
						SPtr<uint32_t> mc32 = sptr<uint32_t>(mod_colors_of(w).off);
						ASTC_NOUNROLL
						for (int k = w.lane; k < 8; k += ASTC_WARP) {
							wc32[k] = mc32[k];
						}
						formats = kept;
						wsync();
					}
				}
				set_formats(work, formats);
				work.partition_count = static_cast<uint8_t>(partition_count);
				work.partition_index = static_cast<uint16_t>(partition_index);
				work.plane2_component = -1;
				work.quant_mode = work.color_formats_matched ? cd.quant_level_mod : cd.quant_level;
				work.block_mode = mode_index;
				work.block_type = SYM_BTYPE_NONCONST;
			}

			unpack_work_endpoints(w, partition_count, formats, ends_off_of(w));
			bool stop_all = false;
			if (l == 0) {
				float errorval = compute_symbolic_block_difference(w, partition_count, formats, plane2_component, pi, (unsigned int)dmode, dual);
				TRACE_F("err_pre", errorval);
				if (errorval == -ERROR_CALC_DEFAULT) {
					errorval = -errorval;
					work.block_type = SYM_BTYPE_ERROR;
				}
				best_errorval_in_mode = minf(errorval, best_errorval_in_mode);
				unsigned int iters_remaining = refinement_limit - l;
				float threshold = (0.045f * static_cast<float>(iters_remaining)) + 1.08f;
				if (errorval > (threshold * best_errorval_in_scb)) {
					break;
				}
				if (errorval < best_errorval_in_scb) {
					best_errorval_in_scb = errorval;
					work.errorval = errorval;
					scb = work;
					copy_work_to_best(w);
					if (errorval < tune_errorval_threshold) {
						stop_all = true;
					}
				}
			}
			if (stop_all) {
				i = candidate_count;
				break;
			}
			bool adjustments = realign_weights(w, partition_count, formats, plane2_component, pi, qmode, dual, (unsigned int)dmode);
			float errorval = ERROR_CALC_DEFAULT;
			if (work.block_type != SYM_BTYPE_ERROR) {
				errorval = compute_symbolic_block_difference(w, partition_count, formats, plane2_component, pi, (unsigned int)dmode, dual);
			}
			TRACE_F("err_post", errorval);
			if (errorval == -ERROR_CALC_DEFAULT) {
				errorval = -errorval;
				work.block_type = SYM_BTYPE_ERROR;
			}
			best_errorval_in_mode = minf(errorval, best_errorval_in_mode);
			unsigned int iters_remaining = refinement_limit - 1 - l;
			float threshold = (0.045f * static_cast<float>(iters_remaining)) + 1.0f;
			if (errorval > (threshold * best_errorval_in_scb)) {
				break;
			}
			if (errorval < best_errorval_in_scb) {
				best_errorval_in_scb = errorval;
				work.errorval = errorval;
				scb = work;
				copy_work_to_best(w);
				if (errorval < tune_errorval_threshold) {
					i = candidate_count;
					break;
				}
			}
			if (!adjustments) {
				break;
			}
		}
	}
	return best_errorval_in_mode;
}

// compress_symbolic_block_for_partition_1plane :353-712
ASTC_COOP float compress_symbolic_block_for_partition_1plane(WCtx w, bool only_always, float tune_errorval_threshold, unsigned int partition_count,
                                                             unsigned int partition_index, ScbHdr& scb, int quant_limit) {
	int max_weight_quant = mini((int)QUANT_32, quant_limit);
	unsigned int packed = part_packed_index(partition_count, partition_index);
	PartView pi = part_view_packed(partition_count, packed);
	compute_ideal_colors_and_weights_1plane(w, pi);

	unsigned int max_decimation_modes = only_always ? BSD.decimation_mode_count_always : BSD.decimation_mode_count_selected;
	uint16_t refmask = (uint16_t)((1u << (max_weight_quant + 1)) - 1);
	ASTC_NOUNROLL
	for (unsigned int i = 0; i < max_decimation_modes; i++) {
		if ((ASTC_LDG(&BSD.dec_modes[i].refprec_1plane) & refmask) == 0) {
			continue;
		}
		compute_ideal_weights_for_decimation(w, i, 1);
	}
	SPtr<f4> ep = ep_of(w);
	f4 min_ep = splat4(10.0f);
	ASTC_NOUNROLL
	for (unsigned int i = 0; i < partition_count; i++) {
		f4 e0 = ep[EP_EI1_0 + (int)i];
		f4 e1 = ep[EP_EI1_1 + (int)i];
		min_ep.x = min_ep_cutoff(e0.x, e1.x, min_ep.x);
		min_ep.y = min_ep_cutoff(e0.y, e1.y, min_ep.y);
		min_ep.z = min_ep_cutoff(e0.z, e1.z, min_ep.z);
		min_ep.w = min_ep_cutoff(e0.w, e1.w, min_ep.w);
	}
	float min_wt_cutoff = hmin_s(min_ep);
	TRACE("trial1p pc=%u pidx=%u only_always=%d maxq=%d\n", partition_count, partition_index, (int)only_always, max_weight_quant);
	TRACE_F("min_wt_cutoff", min_wt_cutoff);

	compute_angular_endpoints(w, only_always, 1, (unsigned int)max_weight_quant);

	unsigned int max_block_modes = only_always ? BSD.block_mode_count_1plane_always : BSD.block_mode_count_1plane_selected;
	quantize_and_score_modes(w, 0, max_block_modes, 1, partition_count, max_weight_quant, min_wt_cutoff, min_wt_cutoff);

	unsigned int candidate_count = compute_ideal_endpoint_formats(w, pi, EP_EI1_0, EP_EI1_1, 1, 0, max_block_modes);
	ASTC_NOUNROLL
	for (int k = w.lane; k < 4; k += ASTC_WARP) {
		ep[EP_BASE_0 + k] = ep[EP_EI1_0 + k];
		ep[EP_BASE_1 + k] = ep[EP_EI1_1 + k];
	}
	wsync();
	return refine_candidates(w, partition_count, packed, false, partition_index, -1, candidate_count, min_wt_cutoff, min_wt_cutoff, tune_errorval_threshold, scb);
}

// compress_symbolic_block_for_partition_2planes :715-1044
ASTC_COOP float compress_symbolic_block_for_partition_2planes(WCtx w, float tune_errorval_threshold, unsigned int plane2_component, ScbHdr& scb, int quant_limit) {
	int max_weight_quant = mini((int)QUANT_32, quant_limit);
	compute_ideal_colors_and_weights_2planes(w, plane2_component);
	uint16_t refmask = (uint16_t)((1u << (max_weight_quant + 1)) - 1);
	unsigned int ndm = BSD.decimation_mode_count_selected;
	ASTC_NOUNROLL
	for (unsigned int i = 0; i < ndm; i++) {
		if ((ASTC_LDG(&BSD.dec_modes[i].refprec_2planes) & refmask) == 0) {
			continue;
		}
		compute_ideal_weights_for_decimation(w, i, 2);
	}
	SPtr<f4> ep = ep_of(w);
	f4 a0 = ep[EP_EI1_0], a1 = ep[EP_EI1_1], b0 = ep[EP_EI2_0], b1 = ep[EP_EI2_1];
	f4 min_ep1 = mk4(min_ep_cutoff(a0.x, a1.x, 10.0f), min_ep_cutoff(a0.y, a1.y, 10.0f), min_ep_cutoff(a0.z, a1.z, 10.0f), min_ep_cutoff(a0.w, a1.w, 10.0f));
	f4 min_ep2 = mk4(min_ep_cutoff(b0.x, b1.x, 10.0f), min_ep_cutoff(b0.y, b1.y, 10.0f), min_ep_cutoff(b0.z, b1.z, 10.0f), min_ep_cutoff(b0.w, b1.w, 10.0f));
	f4 m1 = min_ep1;
	set_lane(m1, (int)plane2_component, ERROR_CALC_DEFAULT);
	float min_wt_cutoff1 = hmin_s(m1);
	f4 m2 = splat4(ERROR_CALC_DEFAULT);
	set_lane(m2, (int)plane2_component, lane(min_ep2, (int)plane2_component));
	float min_wt_cutoff2 = hmin_s(m2);

	compute_angular_endpoints(w, false, 2, (unsigned int)max_weight_quant);

	unsigned int start_2plane = BSD.block_mode_count_1plane_selected;
	unsigned int end_2plane = BSD.block_mode_count_1plane_2plane_selected;
	quantize_and_score_modes(w, start_2plane, end_2plane, 2, 1, max_weight_quant, min_wt_cutoff1, min_wt_cutoff2);

	// merge_endpoints :37-66
	f4 epm0 = a0, epm1 = a1;
	set_lane(epm0, (int)plane2_component, lane(b0, (int)plane2_component));
	set_lane(epm1, (int)plane2_component, lane(b1, (int)plane2_component));
	if (w.lane == 0) {
		ep[EP_BASE_0] = epm0;
		ep[EP_BASE_1] = epm1;
	}
	wsync();
	PartView pi = part_view_packed(1, 0);
	unsigned int candidate_count = compute_ideal_endpoint_formats(w, pi, EP_BASE_0, EP_BASE_1, 2, start_2plane, end_2plane);
	return refine_candidates(w, 1, 0, true, 0, (int)plane2_component, candidate_count, min_wt_cutoff1, min_wt_cutoff2, tune_errorval_threshold, scb);
}

// prepare_block_statistics :1047-1159 - 15 ordered chains over the texels:
//   0 rs, 1 gs, 2 bs, 3 as, 4 rr, 5 gg, 6 bb, 7 aa, 8 rg, 9 rb, 10 ra, 11 gb, 12 ga, 13 ba, 14 weight_sum
ASTC_COOP float prepare_block_statistics(WCtx w) {
	int T = w.T;
	float weight = hadd_s(bi_of(w).channel_weight) / 4.0f;
	SPtr<float> tmpf = tmpf_of(w);
	SPtr<float> b0 = blk_of(w, 0);
	uint32_t cs = tp4(w);
	ASTC_NOUNROLL
	for (int id = w.lane; id < 15; id += ASTC_WARP) {
		tmpf[id] = 0.0f;
	}
	wsync();
	chain_sums<15>(w, T, su_of(w), tmpf, 15,
		[&](int i, float* term) {
			SPtr<float> tx = b0 + i;
			float r = tx[0], g = sptr<float>(tx.off + cs)[0], b = sptr<float>(tx.off + 2 * cs)[0], a = sptr<float>(tx.off + 3 * cs)[0];
			float rw = r * weight, gw = g * weight, bw = b * weight, aw = a * weight;
			term[0] = rw;
			term[1] = gw;
			term[2] = bw;
			term[3] = aw;
			term[4] = r * rw;
			term[5] = g * gw;
			term[6] = b * bw;
			term[7] = a * aw;
			term[8] = g * rw;
			term[9] = b * rw;
			term[10] = a * rw;
			term[11] = b * gw;
			term[12] = a * gw;
			term[13] = a * bw;
			term[14] = weight;
		},
		[&](int id, int& k, int& lo, int& hi, int& step) {
			k = id;
			lo = 0;
			hi = T;
			step = 1;
		});
	SPtr<float> t = tmpf;
	float rs = t[0], gs = t[1], bs = t[2], as = t[3];
	float rr_var = t[4], gg_var = t[5], bb_var = t[6], aa_var = t[7];
	float rg_cov = t[8], rb_cov = t[9], ra_cov = t[10], gb_cov = t[11], ga_cov = t[12], ba_cov = t[13];
	float weight_sum = t[14];
	wsync();
	float rpt = 1.0f / maxf(weight_sum, 1e-7f);
	rr_var -= rs * (rs * rpt);
	rg_cov -= gs * (rs * rpt);
	rb_cov -= bs * (rs * rpt);
	ra_cov -= as * (rs * rpt);
	gg_var -= gs * (gs * rpt);
	gb_cov -= bs * (gs * rpt);
	ga_cov -= as * (gs * rpt);
	bb_var -= bs * (bs * rpt);
	ba_cov -= as * (bs * rpt);
	aa_var -= as * (as * rpt);
	rg_cov *= 1.0f / sqrtf(rr_var * gg_var);
	rb_cov *= 1.0f / sqrtf(rr_var * bb_var);
	ra_cov *= 1.0f / sqrtf(rr_var * aa_var);
	gb_cov *= 1.0f / sqrtf(gg_var * bb_var);
	ga_cov *= 1.0f / sqrtf(gg_var * aa_var);
	ba_cov *= 1.0f / sqrtf(bb_var * aa_var);
	if (rg_cov != rg_cov) rg_cov = 1.0f;
	if (rb_cov != rb_cov) rb_cov = 1.0f;
	if (ra_cov != ra_cov) ra_cov = 1.0f;
	if (gb_cov != gb_cov) gb_cov = 1.0f;
	if (ga_cov != ga_cov) ga_cov = 1.0f;
	if (ba_cov != ba_cov) ba_cov = 1.0f;
	float lowest_correlation = minf(fabsf(rg_cov), fabsf(rb_cov));
	lowest_correlation = minf(lowest_correlation, fabsf(ra_cov));
	lowest_correlation = minf(lowest_correlation, fabsf(gb_cov));
	lowest_correlation = minf(lowest_correlation, fabsf(ga_cov));
	lowest_correlation = minf(lowest_correlation, fabsf(ba_cov));
	return lowest_correlation;
}

ASTC_FN void constant_color_u16(const WCtx& w, ScbHdr& scb) {
	scb.block_type = SYM_BTYPE_CONST_U16;
	f4 c = vclamp4(0.0f, 1.0f, bi_of(w).origin_texel) * 65535.0f;
	scb.constant_color[0] = f2i_rtn(c.x);
	scb.constant_color[1] = f2i_rtn(c.y);
	scb.constant_color[2] = f2i_rtn(c.z);
	scb.constant_color[3] = f2i_rtn(c.w);
}

// compress_block :1162-1455. The block is already loaded (arena block texels + BlkInfo). Writes 16 bytes to out.
ASTC_COOP void compress_block(WCtx w, uint8_t* out) {
	int decode_mode = CFG.profile;
	ScbHdr scb;
	scb.block_type = SYM_BTYPE_ERROR;
	scb.partition_count = 0;
	scb.color_formats_matched = 0;
	scb.plane2_component = -1;
	scb.block_mode = 0;
	scb.partition_index = 0;
	scb.color_formats[0] = scb.color_formats[1] = scb.color_formats[2] = scb.color_formats[3] = 0;
	scb.quant_mode = 0;
	scb.errorval = 0.0f;
	scb.constant_color[0] = scb.constant_color[1] = scb.constant_color[2] = scb.constant_color[3] = 0;

	const BlkInfo& bi = bi_of(w);
	f4 dmn = bi.data_min, dmx = bi.data_max;
	if (dmn.x == dmx.x && dmn.y == dmx.y && dmn.z == dmx.z && dmn.w == dmx.w) {
		scb.partition_count = 0;
		if (decode_mode == PRF_HDR || decode_mode == PRF_HDR_RGB_LDR_A) {
			f4 ot = bi.origin_texel;
			scb.block_type = SYM_BTYPE_CONST_F16;
			scb.constant_color[0] = float_to_sf16(ot.x);
			scb.constant_color[1] = float_to_sf16(ot.y);
			scb.constant_color[2] = float_to_sf16(ot.z);
			scb.constant_color[3] = float_to_sf16(ot.w);
		} else {
			constant_color_u16(w, scb);
		}
		if (w.lane == 0) {
			symbolic_to_physical(w, scb, out);
		}
		wsync();
		return;
	}

	bool block_is_l = is_luminance(w);
	float block_is_l_scale = block_is_l ? 1.0f / 1.5f : 1.0f;
	bool block_is_la = is_luminancealpha(w);
	float block_is_la_scale = block_is_la ? 1.0f / 1.05f : 1.0f;
	int max_partitions = (int)CFG.tune_partition_count_limit;
	bool grayscale = bi.grayscale != 0;

	float error_weight_sum = hadd_s(bi.channel_weight) * BSD.texel_count;
	float error_threshold = CFG.tune_db_limit * error_weight_sum * block_is_l_scale * block_is_la_scale;
	TRACE_F("error_threshold", error_threshold);

	scb.errorval = ERROR_CALC_DEFAULT;
	scb.block_type = SYM_BTYPE_ERROR;
	float best_pc1 = ERROR_CALC_DEFAULT;     // best_errorvals_for_pcount[0]
	const float errorval_overshoot = 1.0f / CFG.tune_mse_overshoot;
	int start_trial = 1;
	if (CFG.tune_search_mode0_enable >= 0.85f && BSD.dim_z == 1) {
		start_trial = 0;
	}
	int quant_limit = QUANT_32;
	bool done = false;
	ASTC_NOUNROLL
	for (int i = start_trial; i < 2 && !done; i++) {
		float mult = i == 0 ? 1.0f / CFG.tune_mse_overshoot : 1.0f;       // errorval_mult[i]
		float errorval = compress_symbolic_block_for_partition_1plane(w, i == 0, error_threshold * mult * errorval_overshoot, 1, 0, scb, QUANT_32);
		if (scb.block_type != SYM_BTYPE_ERROR) {
			quant_limit = ASTC_LDG(&BSD.block_modes[ASTC_LDG(&BSD.block_mode_packed_index[scb.block_mode])].quant_mode);
		}
		best_pc1 = minf(best_pc1, errorval);
		if (errorval < (error_threshold * mult)) {
			done = true;
		}
	}
	if (!done) {
		float lowest_correl = prepare_block_statistics(w);
		bool block_skip_two_plane = lowest_correl > CFG.tune_2plane_early_out_limit_correlation;
		ASTC_NOUNROLL
		for (int i = 3; i >= 0 && !done; i--) {
			if (block_skip_two_plane) {
				continue;
			}
			if (grayscale && i != 3) {
				continue;
			}
			if (is_constant_channel(w, i)) {
				continue;
			}
			float errorval = compress_symbolic_block_for_partition_2planes(w, error_threshold * errorval_overshoot, (unsigned int)i, scb, quant_limit);
			if (errorval > (best_pc1 * 1.85f)) {
				break;
			}
			if (errorval < error_threshold) {
				done = true;
			}
		}
	}
	float best_error_in_prev = best_pc1;
	ASTC_NOUNROLL
	for (int partition_count = 2; partition_count <= max_partitions && !done; partition_count++) {
		unsigned int partition_indices[8];
		unsigned int requested_indices = CFG.tune_partition_index_limit[partition_count - 2];
		unsigned int requested_trials = CFG.tune_partitioning_candidate_limit[partition_count - 2];
		requested_trials = requested_trials < requested_indices ? requested_trials : requested_indices;
		unsigned int actual_trials = find_best_partition_candidates(w, (unsigned int)partition_count, requested_indices, partition_indices, requested_trials);
		// exit_thresholds_for_pcount = {0, 2partition factor, 3partition factor, 0}
		float exit_threshold = partition_count == 2 ? CFG.tune_2partition_early_out_limit_factor : partition_count == 3 ? CFG.tune_3partition_early_out_limit_factor : 0.0f;
		float best_error = ERROR_CALC_DEFAULT;          // best_errorvals_for_pcount[partition_count - 1]
		ASTC_NOUNROLL
		for (unsigned int i = 0; i < actual_trials && !done; i++) {
			float errorval = compress_symbolic_block_for_partition_1plane(w, false, error_threshold * errorval_overshoot, (unsigned int)partition_count,
			                                                              partition_indices[i], scb, quant_limit);
			best_error = minf(best_error, errorval);
			float best_error_scale = exit_threshold * 1.85f;
			if (best_error > (best_error_in_prev * best_error_scale)) {
				done = true;
				break;
			}
			if (errorval < error_threshold) {
				done = true;
				break;
			}
		}
		if (done) {
			break;
		}
		if (best_error > (best_error_in_prev * exit_threshold)) {
			done = true;
		}
		best_error_in_prev = best_error;
	}
	if (scb.block_type == SYM_BTYPE_ERROR) {
		constant_color_u16(w, scb);
	}
	if (w.lane == 0) {
		symbolic_to_physical(w, scb, out);
	}
	wsync();
}
