// CUDA-native ASTC block compressor: warp-cooperative device code, part 2
// (per-mode weight quantisation + error, endpoint format choice, candidate refinement, error scoring,
//  weight realignment, partition search, physical packing, the compress_block driver).
#pragma once
#include "astc_dev_core.cuh"

// su (union scratch) sub-layouts. Each phase owns the whole union while it runs.
//   decimation          : infilled[2][T]
//   angular search      : table rows, pair ranges, step records         (see compute_angular_endpoints)
//   quantise+error pass : per-lane quantised weight rows                 UQ_ROW_STRIDE * 32
//   endpoint formats    : best_error/format tables, combined tables     (EfTables)
//   refinement          : undecimated weights, int weights, chain staging tile (RefineScratch)
//   partition search    : mismatch counts, ordering, histogram, k-means state, candidate errors
#define UQ_ROW_STRIDE 68    /* 17 words: conflict-free lane-private rows */

// =============================================================================================
// Per block mode: quantise the decimated ideal weights and measure the weight-set error
// (astcenc_compress_symbolic.cpp:434-485 / :803-868 + ideal_endpoints.cpp:688-842, :974-1080).
// Lanes over block modes; the texel error sum keeps the reference's 4-lane accumulator order per mode.
// =============================================================================================
// S1: one plane and one partition are compile-time facts (the wave-0 set-up of an LDR profile inlines that instantiation)
template <bool S1> ASTC_FN void quantize_and_score_modes_t(const WCtx& w, unsigned int start_mode, unsigned int end_mode, int nplanes_in,
                                                          unsigned int partition_count_in, int max_weight_quant, float min_wt_cutoff1, float min_wt_cutoff2) {
	const int nplanes = S1 ? 1 : nplanes_in;
	const unsigned int partition_count = S1 ? 1u : partition_count_in;
	int free_bits = partition_count == 1 ? 115 - 4 : partition_count == 2 ? 111 - 4 - 10 : partition_count == 3 ? 108 - 4 - 10 : 105 - 4 - 10;
	SPtr<uint8_t> uqrow = sptr<uint8_t>(su_of(w) + (uint32_t)w.lane * UQ_ROW_STRIDE);
	SPtr<float> mode_err = mode_err_of(w);
	SPtr<float> dwi = dwi_of(w);
	SPtr<float> eiw1 = eiw_of(w, 0), eis1 = eis_of(w, 0), eiw2 = eiw_of(w, 1), eis2 = eis_of(w, 1);
	int T = w.T;
	ASTC_NOUNROLL
	for (unsigned int i = start_mode + (unsigned int)w.lane; i < end_mode; i += ASTC_WARP) {
		const DevBlockMode* bmp = BSD.block_modes + i;
		int quant_mode = ASTC_LDG(&bmp->quant_mode);
		int dmode = ASTC_LDG(&bmp->decimation_mode);
		if (quant_mode > max_weight_quant) {
			mode_err[(int)i] = 1e38f;
			continue;
		}
		if (nplanes == 1) {
			int bitcount = free_bits - (int)ASTC_LDG(&bmp->weight_bits);
			if (bitcount <= 0) {
				mode_err[(int)i] = 1e38f;
				continue;
			}
		}
		DecView di = dec_view((unsigned int)dmode);
		int W = di.W;
		float low1, high1, low2 = 0.0f, high2 = 1.0f;
		mode_low_high(w, dmode, quant_mode, 0, min_wt_cutoff1, low1, high1);
		WeightQuantizer z1 = make_weight_quantizer(low1, high1, quant_mode);
		float rscale2 = z1.rscale, lowb2 = z1.low_bound;
		SPtr<float> ideal1 = dwi + di.dwi_offset;
		ASTC_UNROLL_S2
		for (int k = 0; k < W; k++) {
			uqrow[k] = (uint8_t)quantize_weight(z1, ideal1[k]);
		}
		if (nplanes == 2) {
			mode_low_high(w, dmode, quant_mode, 1, min_wt_cutoff2, low2, high2);
			WeightQuantizer z2 = make_weight_quantizer(low2, high2, quant_mode);
			rscale2 = z2.rscale;
			lowb2 = z2.low_bound;
			SPtr<float> ideal2 = ideal1 + W;
			ASTC_UNROLL_X2
			for (int k = 0; k < W; k++) {
				uqrow[32 + k] = (uint8_t)quantize_weight(z2, ideal2[k]);
			}
		}
		// compute_error_of_weight_set_1plane / _2planes: texel t feeds accumulator lane t & 3 - four texels per trip, one per
		// accumulator (no selection chain), the odd texels of footprints that are not a multiple of four afterwards
		float acc0 = 0.0f, acc1 = 0.0f, acc2 = 0.0f, acc3 = 0.0f;
		float rscale1 = z1.rscale, lowb1 = z1.low_bound;
		auto texel_error = [&](int t) -> float {
			uint32_t ix = ASTC_LDD(&di.twi[t]);
			f4 cf = dec_contribs(di, t);
			int i0 = (int)(ix & 0xFF), i1 = (int)((ix >> 8) & 0xFF), i2 = (int)((ix >> 16) & 0xFF), i3 = (int)(ix >> 24);
			float c0 = cf.x, c1 = cf.y, c2 = cf.z, c3 = cf.w;
			float cur1 = ((static_cast<float>(uqrow[i0]) * rscale1 + lowb1) * c0 + (static_cast<float>(uqrow[i1]) * rscale1 + lowb1) * c1) +
			             ((static_cast<float>(uqrow[i2]) * rscale1 + lowb1) * c2 + (static_cast<float>(uqrow[i3]) * rscale1 + lowb1) * c3);
			float diff = cur1 - eiw1[t];
			float error = diff * diff * eis1[t];
			if (nplanes == 2) {
				float cur2 = ((static_cast<float>(uqrow[32 + i0]) * rscale2 + lowb2) * c0 + (static_cast<float>(uqrow[32 + i1]) * rscale2 + lowb2) * c1) +
				             ((static_cast<float>(uqrow[32 + i2]) * rscale2 + lowb2) * c2 + (static_cast<float>(uqrow[32 + i3]) * rscale2 + lowb2) * c3);
				float diff2 = cur2 - eiw2[t];
				float error2 = diff2 * diff2 * eis2[t];
				error = error + error2;
			}
			return error;
		};
		int t = 0;
		ASTC_NOUNROLL
		for (; t + 4 <= T; t += 4) {
			acc0 = acc0 + texel_error(t);
			acc1 = acc1 + texel_error(t + 1);
			acc2 = acc2 + texel_error(t + 2);
			acc3 = acc3 + texel_error(t + 3);
		}
		ASTC_NOUNROLL
		for (; t < T; t++) {
			float error = texel_error(t);
			int a = t & 3;
			if (a == 0) acc0 = acc0 + error;
			else if (a == 1) acc1 = acc1 + error;
			else acc2 = acc2 + error;
		}
		mode_err[(int)i] = (acc0 + acc2) + (acc1 + acc3);
	}
	wsync();
}
ASTC_COOP void quantize_and_score_modes(WCtx w, unsigned int start_mode, unsigned int end_mode, int nplanes, unsigned int partition_count,
                                        int max_weight_quant, float min_wt_cutoff1, float min_wt_cutoff2) {
	quantize_and_score_modes_t<false>(w, start_mode, end_mode, nplanes, partition_count, max_weight_quant, min_wt_cutoff1, min_wt_cutoff2);
}

// =============================================================================================
// Endpoint format choice (astcenc_pick_best_endpoint_format.cpp)
// =============================================================================================
struct EncodingChoiceErrors {
	float rgb_scale_error, rgb_luma_error, luminance_error, alpha_drop_error;
	bool can_offset_encode, can_blue_contract;
};

ASTC_FN f4 dot3_splat(f4 a, f4 b) {
	float d = dot3_s(a, b);
	return mk4(d, d, d, 0.0f);
}

// layout of su during endpoint format selection
struct EfTables {
	float best_error[4][21][4];
	float combined_error[21][13];
	uint8_t format_of_choice[4][21][4];
	uint8_t combined_format[21][13][4];
};
#define EF_OF(w) (*reinterpret_cast<EfTables*>(astc_smem + su_of(w)))
// (the chain staging tile of compute_encoding_choice_errors uses the same bytes first: its sums are done
//  before the tables are written)

// compute_encoding_choice_errors :222-312 with compute_error_squared_rgb_single_partition :72-219.
// Terms per texel: 0 alpha drop, 1 uncorrelated line, 2 same-chroma line, 3 rgb-luma line, 4 luminance line;
// one chain per (partition, term, texel index mod 4).
// (S1 here and below: one partition, one plane, LDR endpoint formats - see quantize_and_score_modes_t)
template <bool S1> ASTC_FN void compute_encoding_choice_errors_t(const WCtx& w, const PartView& pi, int ep0slot, int ep1slot, EncodingChoiceErrors eci[4]) {
	const int pc = S1 ? 1 : (int)pi.partition_count;
	PartitionMetrics pms[4];
	if (S1) {
		compute_avgs_and_dirs_3_comp_rgb_t<true>(w, pi, pms);
	} else {
		compute_avgs_and_dirs_3_comp_rgb(w, pi, pms);
	}
	SPtr<float> tmpf = tmpf_of(w);
	SPtr<float> lines = tmpf + 80;          // per partition: uncor.amod[3] uncor.bs[3] samec.bs[3] rgbl.amod[3]
	if (w.lane == 0) {
		for (int i = 0; i < pc; i++) {
			f4 uncor_a = pms[i].avg;
			f4 uncor_b = normalize_safe4(pms[i].dir, unit3());
			f4 samec_b = normalize_safe4(pms[i].avg, unit3());
			f4 luma_a = pms[i].avg;
			f4 luma_b = unit3();
			f4 uncor_amod = uncor_a - uncor_b * dot3_splat(uncor_a, uncor_b);
			f4 rgbl_amod = luma_a - luma_b * dot3_splat(luma_a, luma_b);
			SPtr<float> l = lines + i * 12;
			l[0] = uncor_amod.x; l[1] = uncor_amod.y; l[2] = uncor_amod.z;
			l[3] = uncor_b.x; l[4] = uncor_b.y; l[5] = uncor_b.z;
			l[6] = samec_b.x; l[7] = samec_b.y; l[8] = samec_b.z;
			l[9] = rgbl_amod.x; l[10] = rgbl_amod.y; l[11] = rgbl_amod.z;
		}
	}
	int nchains = pc * 20;
	ASTC_NOUNROLL
	for (int id = w.lane; id < nchains; id += ASTC_WARP) {
		tmpf[id] = 0.0f;
	}
	wsync();
	f4 ews = bi_of(w).channel_weight;
	float default_a = default_alpha(w);
	SPtr<float> br = blk_of(w, 0), bg = blk_of(w, 1), bb = blk_of(w, 2), ba = blk_of(w, 3);
	const float u3 = 0.577350258827209473f;
	chain_sums<5>(w, w.T, su_of(w), tmpf, nchains,
		[&](int pos, float* term) {
			int t = S1 ? pos : pv_texel(pi, pos);
			int p = pc > 1 ? (int)ASTC_LDG(&pi.partition_of_texel[t]) : 0;
			SPtr<float> l = lines + p * 12;
			float dr = br[t], dg = bg[t], db = bb[t];
			float alpha_diff = ba[t] - default_a;
			term[0] = alpha_diff * alpha_diff;
			{
				float bx = l[3], by = l[4], bz = l[5];
				float param = dr * bx + dg * by + db * bz;
				float dist0 = (l[0] + param * bx) - dr;
				float dist1 = (l[1] + param * by) - dg;
				float dist2 = (l[2] + param * bz) - db;
				term[1] = dist0 * dist0 * ews.x + dist1 * dist1 * ews.y + dist2 * dist2 * ews.z;
			}
			{
				float bx = l[6], by = l[7], bz = l[8];
				float param = dr * bx + dg * by + db * bz;
				float dist0 = (param * bx) - dr;
				float dist1 = (param * by) - dg;
				float dist2 = (param * bz) - db;
				term[2] = dist0 * dist0 * ews.x + dist1 * dist1 * ews.y + dist2 * dist2 * ews.z;
			}
			{
				float param = dr * u3 + dg * u3 + db * u3;
				float dist0 = (l[9] + param * u3) - dr;
				float dist1 = (l[10] + param * u3) - dg;
				float dist2 = (l[11] + param * u3) - db;
				term[3] = dist0 * dist0 * ews.x + dist1 * dist1 * ews.y + dist2 * dist2 * ews.z;
				float e0 = (param * u3) - dr;
				float e1 = (param * u3) - dg;
				float e2 = (param * u3) - db;
				term[4] = e0 * e0 * ews.x + e1 * e1 * ews.y + e2 * e2 * ews.z;
			}
		},
		[&](int id, int& k, int& lo, int& hi, int& step) {
			int p = id / 20;
			int r = id - p * 20;
			k = r >> 2;
			lo = pv_start(pi, (unsigned int)p) + (r & 3);
			hi = pv_start(pi, (unsigned int)p) + pv_count(pi, (unsigned int)p);
			step = 4;
		});
	SPtr<f4> ep = ep_of(w);
	bool blue_contract = !is_luminance(w);
	for (int i = 0; i < pc; i++) {
		SPtr<float> a = tmpf + i * 20;
		float alpha_drop_error = ((a[0] + a[2]) + (a[1] + a[3])) * ews.w;
		float uncorr_rgb_error = (a[4] + a[6]) + (a[5] + a[7]);
		float samechroma_rgb_error = (a[8] + a[10]) + (a[9] + a[11]);
		float rgb_luma_error = (a[12] + a[14]) + (a[13] + a[15]);
		float luminance_rgb_error = (a[16] + a[18]) + (a[17] + a[19]);
		f4 d = ep[ep1slot + i] - ep[ep0slot + i];
		const float lim = 0.12f * 65535.0f;
		eci[i].can_offset_encode = (absf(d.x) < lim) && (absf(d.y) < lim) && (absf(d.z) < lim);
		eci[i].rgb_scale_error = (samechroma_rgb_error - uncorr_rgb_error) * 0.7f;
		eci[i].rgb_luma_error = (rgb_luma_error - uncorr_rgb_error) * 1.5f;
		eci[i].luminance_error = (luminance_rgb_error - uncorr_rgb_error) * 3.0f;
		eci[i].alpha_drop_error = alpha_drop_error * 3.0f;
		eci[i].can_blue_contract = blue_contract;
	}
	wsync();
}
ASTC_COOP void compute_encoding_choice_errors(WCtx w, const PartView& pi, int ep0slot, int ep1slot, EncodingChoiceErrors eci[4]) {
	compute_encoding_choice_errors_t<false>(w, pi, ep0slot, ep1slot, eci);
}

// 5^2 7^2 9^2 11^2 15^2 19^2 23^2 31^2 39^2 47^2 63^2 79^2 95^2 127^2 159^2 191^2 255^2: (levels - 1)^2 from QUANT_6 up
ASTC_FN float quant_den(int q) {
	float m = static_cast<float>(quant_level_count(q) - 1u);
	return m * m;
}

// compute_color_error_for_every_integer_count_and_quant_level :315-675. Lanes over quant levels.
// (the one-partition, one-plane set-up calls this out-of-line function too: as an inlined template instantiation the general
// function compiled to different code)
ASTC_COOP void compute_color_error_tables(WCtx w, int partition_size, int partition_index, const EncodingChoiceErrors& eci, int ep0slot, int ep1slot) {
	const BlkInfo& bi = bi_of(w);
	EfTables& ef = EF_OF(w);
	bool encode_hdr_rgb = bi.rgb_lns0 != 0;
	bool encode_hdr_alpha = bi.alpha_lns0 != 0;
	f4 error_weight = bi.channel_weight;
	SPtr<f4> ep = ep_of(w);
	f4 ep0 = ep[ep0slot + partition_index];
	f4 ep1 = ep[ep1slot + partition_index];
	float ep1_min = hmin_s(mk4(ep1.x, ep1.y, ep1.z, ep1.x));
	ep1_min = maxf(ep1_min, 0.0f);
	float error_weight_rgbsum = hadd_rgb_s(error_weight);
	float range_upper_limit_rgb = encode_hdr_rgb ? 61440.0f : 65535.0f;
	float range_upper_limit_alpha = encode_hdr_alpha ? 61440.0f : 65535.0f;
	f4 offset = mk4(range_upper_limit_rgb, range_upper_limit_rgb, range_upper_limit_rgb, range_upper_limit_alpha);
	f4 zero = splat4(0.0f);
	f4 ep0_high = max4(ep0 - offset, zero);
	f4 ep1_high = max4(ep1 - offset, zero);
	f4 ep0_low = min4(ep0, zero);
	f4 ep1_low = min4(ep1, zero);
	f4 sum_range_error = (ep0_low * ep0_low) + (ep1_low * ep1_low) + (ep0_high * ep0_high) + (ep1_high * ep1_high);
	float rgb_range_error = dot3_s(sum_range_error, error_weight) * 0.5f * static_cast<float>(partition_size);
	float alpha_range_error = sum_range_error.w * error_weight.w * 0.5f * static_cast<float>(partition_size);
	float (*best_error)[4] = ef.best_error[partition_index];
	uint8_t (*format_of_choice)[4] = ef.format_of_choice[partition_index];

	if (encode_hdr_rgb) {
		float af, cf;
		if (ep1.x > ep1.y && ep1.x > ep1.z) {
			af = ep1.x;
			cf = ep1.x - ep0.x;
		} else if (ep1.y > ep1.z) {
			af = ep1.y;
			cf = ep1.y - ep0.y;
		} else {
			af = ep1.z;
			cf = ep1.z - ep0.z;
		}
		float bf = af - ep1_min;
		f4 prd = mk4(ep1.x - cf, ep1.y - cf, ep1.z - cf, 0.0f);
		f4 pdif = prd - mk4(ep0.x, ep0.y, ep0.z, 0.0f);
		float df = hmax_s(mk4(absf(pdif.x), absf(pdif.y), absf(pdif.z), absf(pdif.w)));
		int b = static_cast<int>(clampf(bf, 0.0f, 65536.0f));
		int c = static_cast<int>(clampf(cf, 0.0f, 65536.0f));
		int d = static_cast<int>(clampf(df, 0.0f, 65536.0f));
		int rgbo_mode = 5;
		if (b < 32768 && c < 16384) rgbo_mode = 4;
		if (b < 8192 && c < 16384) rgbo_mode = 3;
		if (b < 2048 && c < 16384) rgbo_mode = 2;
		if (b < 2048 && c < 1024) rgbo_mode = 1;
		if (b < 1024 && c < 4096) rgbo_mode = 0;
		int rgb_mode = 8;
		if (b < 16384 && c < 8192 && d < 8192) rgb_mode = 0;
		if (b < 32768 && c < 8192 && d < 4096) rgb_mode = 1;
		if (b < 4096 && c < 8192 && d < 4096) rgb_mode = 2;
		if (b < 8192 && c < 8192 && d < 2048) rgb_mode = 3;
		if (b < 8192 && c < 2048 && d < 512) rgb_mode = 4;
		if (b < 2048 && c < 8192 && d < 1024) rgb_mode = 5;
		if (b < 2048 && c < 2048 && d < 256) rgb_mode = 6;
		if (b < 1024 && c < 2048 && d < 512) rgb_mode = 7;
		const float rgbo_error_scales[6] = {4.0f, 4.0f, 16.0f, 64.0f, 256.0f, 1024.0f};
		const float rgb_error_scales[9] = {64.0f, 64.0f, 16.0f, 16.0f, 4.0f, 4.0f, 1.0f, 1.0f, 384.0f};
		float mode7mult = rgbo_error_scales[rgbo_mode] * 0.0015f;
		float mode11mult = rgb_error_scales[rgb_mode] * 0.010f;
		float lum_high = hadd_rgb_s(ep1) * (1.0f / 3.0f);
		float lum_low = hadd_rgb_s(ep0) * (1.0f / 3.0f);
		float lumdif = lum_high - lum_low;
		float mode23mult = lumdif < 960 ? 4.0f : lumdif < 3968 ? 16.0f : 128.0f;
		mode23mult *= 0.0005f;
		ASTC_NOUNROLL
		for (int i = w.lane; i <= QUANT_256; i += ASTC_WARP) {
			format_of_choice[i][3] = static_cast<uint8_t>(encode_hdr_alpha ? FMT_HDR_RGBA : FMT_HDR_RGB_LDR_ALPHA);
			format_of_choice[i][2] = FMT_HDR_RGB;
			format_of_choice[i][1] = FMT_HDR_RGB_SCALE;
			format_of_choice[i][0] = FMT_HDR_LUMINANCE_LARGE_RANGE;
			if (i < QUANT_16) {
				best_error[i][3] = ERROR_CALC_DEFAULT;
				best_error[i][2] = ERROR_CALC_DEFAULT;
				best_error[i][1] = ERROR_CALC_DEFAULT;
				best_error[i][0] = ERROR_CALC_DEFAULT;
				continue;
			}
			float base_quant_error = ((65536.0f * 65536.0f / 18.0f) / quant_den(i)) * static_cast<float>(partition_size);
			float rgb_quantization_error = error_weight_rgbsum * base_quant_error * 2.0f;
			float alpha_quantization_error = error_weight.w * base_quant_error * 2.0f;
			float rgba_quantization_error = rgb_quantization_error + alpha_quantization_error;
			best_error[i][3] = rgba_quantization_error + rgb_range_error + alpha_range_error;
			best_error[i][2] = (rgb_quantization_error * mode11mult) + rgb_range_error + eci.alpha_drop_error;
			best_error[i][1] = (rgb_quantization_error * mode7mult) + rgb_range_error + eci.alpha_drop_error + eci.rgb_luma_error;
			best_error[i][0] = (rgb_quantization_error * mode23mult) + rgb_range_error + eci.alpha_drop_error + eci.luminance_error;
		}
	} else {
		float base_quant_error_rgb = error_weight_rgbsum * static_cast<float>(partition_size);
		float base_quant_error_a = error_weight.w * static_cast<float>(partition_size);
		float base_quant_error_rgba = base_quant_error_rgb + base_quant_error_a;
		float error_scale_bc_rgba = eci.can_blue_contract ? 0.625f : 1.0f;
		float error_scale_bc_rgb = eci.can_blue_contract ? 0.5f : 1.0f;
		ASTC_NOUNROLL
		for (int i = w.lane; i <= QUANT_256; i += ASTC_WARP) {
			if (i < QUANT_6) {
				best_error[i][3] = ERROR_CALC_DEFAULT;
				best_error[i][2] = ERROR_CALC_DEFAULT;
				best_error[i][1] = ERROR_CALC_DEFAULT;
				best_error[i][0] = ERROR_CALC_DEFAULT;
				format_of_choice[i][3] = FMT_RGBA;
				format_of_choice[i][2] = FMT_RGB;
				format_of_choice[i][1] = FMT_RGB_SCALE;
				format_of_choice[i][0] = FMT_LUMINANCE;
				continue;
			}
			float error_scale_oe_rgba = eci.can_offset_encode ? 0.5f : 1.0f;
			float error_scale_oe_rgb = eci.can_offset_encode ? 0.25f : 1.0f;
			if (i >= QUANT_192) {
				error_scale_oe_rgba = 1.0f;
				error_scale_oe_rgb = 1.0f;
			}
			float base_quant_error = (65536.0f * 65536.0f / 18.0f) / quant_den(i);
			float quant_error_rgb = base_quant_error_rgb * base_quant_error;
			float quant_error_rgba = base_quant_error_rgba * base_quant_error;
			best_error[i][3] = quant_error_rgba * error_scale_bc_rgba * error_scale_oe_rgba + rgb_range_error + alpha_range_error;
			format_of_choice[i][3] = FMT_RGBA;
			float full_ldr_rgb_error = quant_error_rgb * error_scale_bc_rgb * error_scale_oe_rgb + rgb_range_error + eci.alpha_drop_error;
			float rgbs_alpha_error = quant_error_rgba + eci.rgb_scale_error + rgb_range_error + alpha_range_error;
			if (rgbs_alpha_error < full_ldr_rgb_error) {
				best_error[i][2] = rgbs_alpha_error;
				format_of_choice[i][2] = FMT_RGB_SCALE_ALPHA;
			} else {
				best_error[i][2] = full_ldr_rgb_error;
				format_of_choice[i][2] = FMT_RGB;
			}
			float ldr_rgbs_error = quant_error_rgb + rgb_range_error + eci.alpha_drop_error + eci.rgb_scale_error;
			float lum_alpha_error = quant_error_rgba + rgb_range_error + alpha_range_error + eci.luminance_error;
			if (ldr_rgbs_error < lum_alpha_error) {
				best_error[i][1] = ldr_rgbs_error;
				format_of_choice[i][1] = FMT_RGB_SCALE;
			} else {
				best_error[i][1] = lum_alpha_error;
				format_of_choice[i][1] = FMT_LUMINANCE_ALPHA;
			}
			best_error[i][0] = quant_error_rgb + rgb_range_error + eci.alpha_drop_error + eci.luminance_error;
			format_of_choice[i][0] = FMT_LUMINANCE;
		}
	}
	wsync();
}

// N-partition combination tables (:728-1093): lanes over quant levels, the combination scan inside a
// level is sequential (the reference's "<=" update order matters). The reference walks nested loops over the
// per-partition integer counts and prunes every prefix whose counts differ by more than one; the tuples that
// survive are listed here in the same (lexicographic) order, 2 bits per partition, first partition on top.
#if defined(ASTC_HOSTSIM)
	#define ASTC_DEV_TABLE static const
#else
	#define ASTC_DEV_TABLE __constant__ const
#endif
ASTC_DEV_TABLE uint8_t g_combo_tuples[10 + 22 + 46] = {
	0, 1, 4, 5, 6, 9, 10, 11, 14, 15,
	0, 1, 4, 5, 16, 17, 20, 21, 22, 25, 26, 37, 38, 41, 42, 43, 46, 47, 58, 59, 62, 63,
	0, 1, 4, 5, 16, 17, 20, 21, 64, 65, 68, 69, 80, 81, 84, 85, 86, 89, 90, 101, 102, 105, 106, 149, 150, 153, 154, 165, 166, 169, 170,
	171, 174, 175, 186, 187, 190, 191, 234, 235, 238, 239, 250, 251, 254, 255};

ASTC_COOP void multi_partition_find_best_combination(WCtx w, int pc) {
	EfTables& ef = EF_OF(w);
	int width = pc == 2 ? 7 : pc == 3 ? 10 : 13;
	int combos = pc == 2 ? 10 : pc == 3 ? 22 : 46;
	const uint8_t* tuples = g_combo_tuples + (pc == 2 ? 0 : pc == 3 ? 10 : 32);
	ASTC_NOUNROLL
	for (int quant = w.lane; quant <= QUANT_256; quant += ASTC_WARP) {
		ASTC_NOUNROLL
		for (int j = 0; j < width; j++) {
			ef.combined_error[quant][j] = ERROR_CALC_DEFAULT;
		}
		if (quant < QUANT_6) {
			continue;
		}
		ASTC_NOUNROLL
		for (int n = 0; n < combos; n++) {
			unsigned int tup = tuples[n];
			int sh = 2 * (pc - 1);
			int dg = (int)(tup >> sh) & 3;
			float errorterm = ef.best_error[0][quant][dg];
			int intcnt = dg;
			ASTC_NOUNROLL
			for (int k = 1; k < pc; k++) {
				sh -= 2;
				dg = (int)(tup >> sh) & 3;
				errorterm = errorterm + ef.best_error[k][quant][dg];
				intcnt += dg;
			}
			errorterm = minf(errorterm, 1e10f);
			if (errorterm <= ef.combined_error[quant][intcnt]) {
				ef.combined_error[quant][intcnt] = errorterm;
				sh = 2 * pc;
				ASTC_NOUNROLL
				for (int k = 0; k < pc; k++) {
					sh -= 2;
					ef.combined_format[quant][intcnt][k] = ef.format_of_choice[k][quant][(tup >> sh) & 3];
				}
			}
		}
	}
	wsync();
}

// one_partition_/N-partition _find_best_combination_for_bitcount (:678-725, :768-1093)
template <bool S1> ASTC_FN float find_best_combination_for_bitcount_t(int pc, uint32_t ef_off, int bits_available, uint8_t& best_quant_level, uint8_t& best_quant_level_mod,
                                                                 uint8_t* best_formats) {
	const DevConstTables* ct = ASTC_CT;
	const EfTables& ef = *reinterpret_cast<const EfTables*>(astc_smem + ef_off);
	if (S1 || pc == 1) {
		int best_integer_count = 0;
		float best_integer_count_error = ERROR_CALC_DEFAULT;
		ASTC_NOUNROLL
		for (int integer_count = 1; integer_count <= 4; integer_count++) {
			int quant_level = ASTC_LDG(&ct->quant_mode_table[integer_count][bits_available]);
			if (quant_level < QUANT_6) {
				continue;
			}
			float integer_count_error = ef.best_error[0][quant_level][integer_count - 1];
			if (integer_count_error < best_integer_count_error) {
				best_integer_count_error = integer_count_error;
				best_integer_count = integer_count - 1;
			}
		}
		int ql = ASTC_LDG(&ct->quant_mode_table[best_integer_count + 1][bits_available]);
		best_quant_level = static_cast<uint8_t>(ql);
		best_quant_level_mod = best_quant_level;
		best_formats[0] = FMT_LUMINANCE;
		if (ql >= QUANT_6) {
			best_formats[0] = ef.format_of_choice[0][ql][best_integer_count];
		}
		return best_integer_count_error;
	}
	int best_integer_count = 0;
	float best_integer_count_error = ERROR_CALC_DEFAULT;
	int first = pc;
	int last = pc == 2 ? 8 : 9;
	int mod_bits = pc == 2 ? 2 : pc == 3 ? 5 : 8;
	ASTC_NOUNROLL
	for (int integer_count = first; integer_count <= last; integer_count++) {
		int quant_level = ASTC_LDG(&ct->quant_mode_table[integer_count][bits_available]);
		if (quant_level < QUANT_6) {
			break;
		}
		float integer_count_error = ef.combined_error[quant_level][integer_count - first];
		if (integer_count_error < best_integer_count_error) {
			best_integer_count_error = integer_count_error;
			best_integer_count = integer_count;
		}
	}
	int ql = ASTC_LDG(&ct->quant_mode_table[best_integer_count][bits_available]);
	int ql_mod = ASTC_LDG(&ct->quant_mode_table[best_integer_count][bits_available + mod_bits]);
	best_quant_level = static_cast<uint8_t>(ql);
	best_quant_level_mod = static_cast<uint8_t>(ql_mod);
	if (ql >= QUANT_6) {
		for (int i = 0; i < pc; i++) {
			best_formats[i] = ef.combined_format[ql][best_integer_count - first][i];
		}
	} else {
		for (int i = 0; i < pc; i++) {
			best_formats[i] = FMT_LUMINANCE;
		}
	}
	return best_integer_count_error;
}
ASTC_NOINLINE float find_best_combination_for_bitcount(int pc, uint32_t ef_off, int bits_available, uint8_t& best_quant_level, uint8_t& best_quant_level_mod, uint8_t* best_formats) {
	return find_best_combination_for_bitcount_t<false>(pc, ef_off, bits_available, best_quant_level, best_quant_level_mod, best_formats);
}

// candidate record kept in the arena (8 bytes each)
struct Candidate {
	uint16_t block_mode;       // packed index
	uint8_t quant_level, quant_level_mod;
	uint8_t formats[4];
};
ASTC_FN SPtr<Candidate> cand_of(const WCtx& w) { return sptr<Candidate>(w.base + A_CAND); }

ASTC_FN int mode_bitcount(int weight_bits, int nplanes, int pc) {
	int free_bits = pc == 1 ? 115 - 4 : pc == 2 ? 111 - 4 - 10 : pc == 3 ? 108 - 4 - 10 : 105 - 4 - 10;
	return nplanes == 2 ? 109 - weight_bits : free_bits - weight_bits;
}

// compute_ideal_endpoint_formats :1096-1357, in two parts.
// Part 1: error tables + the total error of every block mode in [start, end) (overwrites the weight error in place).
template <bool S1> ASTC_FN void endpoint_formats_prepare_t(const WCtx& w, const PartView& pi, int ep0slot, int ep1slot, int nplanes_in,
                                                          unsigned int start_block_mode, unsigned int end_block_mode) {
	const int pc = S1 ? 1 : (int)pi.partition_count;
	const int nplanes = S1 ? 1 : nplanes_in;
	EncodingChoiceErrors eci[4];
	if (S1) {
		compute_encoding_choice_errors_t<true>(w, pi, ep0slot, ep1slot, eci);
		compute_color_error_tables(w, pv_count(pi, 0), 0, eci[0], ep0slot, ep1slot);
	} else {
		compute_encoding_choice_errors(w, pi, ep0slot, ep1slot, eci);
		for (int i = 0; i < pc; i++) {
			compute_color_error_tables(w, pv_count(pi, (unsigned int)i), i, eci[i], ep0slot, ep1slot);
		}
	}
	if (pc >= 2) {
		multi_partition_find_best_combination(w, pc);
	}
	uint32_t ef_off = su_of(w);
	SPtr<float> mode_err = mode_err_of(w);
	ASTC_NOUNROLL
	for (unsigned int i = start_block_mode + (unsigned int)w.lane; i < end_block_mode; i += ASTC_WARP) {
		float qwt = mode_err[(int)i];
		if (qwt >= ERROR_CALC_DEFAULT) {
			mode_err[(int)i] = ERROR_CALC_DEFAULT;
			continue;
		}
		uint8_t ql, qlm, fmts[4];
		int bits = mode_bitcount(ASTC_LDG(&BSD.block_modes[i].weight_bits), nplanes, pc);
		float error_of_best = S1 ? find_best_combination_for_bitcount_t<true>(1, ef_off, bits, ql, qlm, fmts)
		                         : find_best_combination_for_bitcount(pc, ef_off, bits, ql, qlm, fmts);
		mode_err[(int)i] = error_of_best + qwt;
	}
	wsync();
}
ASTC_COOP void endpoint_formats_prepare(WCtx w, const PartView& pi, int ep0slot, int ep1slot, int nplanes,
                                        unsigned int start_block_mode, unsigned int end_block_mode) {
	endpoint_formats_prepare_t<false>(w, pi, ep0slot, ep1slot, nplanes, start_block_mode, end_block_mode);
}

// Part 2: the tune_candidate_limit lowest totals of [start, end), lowest index first among equals (:1286-1333), written
// to the Candidate array at cand_off. With keep_errors the totals survive (a second selection over another range follows).
template <bool S1> ASTC_FN unsigned int endpoint_formats_select_t(const WCtx& w, int pc_in, int nplanes_in, unsigned int start_block_mode, unsigned int end_block_mode,
                                                                 uint32_t cand_off, bool keep_errors) {
	const int pc = S1 ? 1 : pc_in;
	const int nplanes = S1 ? 1 : nplanes_in;
	uint32_t ef_off = su_of(w);
	SPtr<float> mode_err = mode_err_of(w);
	unsigned int limit = CFG.tune_candidate_limit;
	unsigned int count = 0;
	SPtr<Candidate> cands = sptr<Candidate>(cand_off);
	SPtr<float> taken = tmpf_of(w);             // [8] x (index, value) of the entries knocked out
	ASTC_NOUNROLL
	for (unsigned int k = 0; k < limit; k++) {
		float best = ERROR_CALC_DEFAULT;
		int best_idx = 0x7FFFFFFF;
		ASTC_NOUNROLL
		for (unsigned int i = start_block_mode + (unsigned int)w.lane; i < end_block_mode; i += ASTC_WARP) {
			float e = mode_err[(int)i];
			if (e < best) {
				best = e;
				best_idx = (int)i;
			}
		}
		wargmin(best, best_idx);
		if (!(best < ERROR_CALC_DEFAULT)) {
			break;
		}
		if (w.lane == 0) {
			taken[2 * (int)k] = ASTC_U2F((uint32_t)best_idx);
			taken[2 * (int)k + 1] = best;
			mode_err[best_idx] = ERROR_CALC_DEFAULT;
		}
		count++;
		wsync();
	}
	// the winners' quant levels and formats: one lane per candidate (the look-up chain is long and serial)
	ASTC_NOUNROLL
	for (unsigned int k = (unsigned int)w.lane; k < count; k += ASTC_WARP) {
		int best_idx = (int)ASTC_F2U(taken[2 * (int)k]);
		Candidate c;
		c.block_mode = (uint16_t)best_idx;
		c.formats[0] = c.formats[1] = c.formats[2] = c.formats[3] = 0;
		int bits = mode_bitcount(ASTC_LDG(&BSD.block_modes[best_idx].weight_bits), nplanes, pc);
		if (S1) {
			find_best_combination_for_bitcount_t<true>(1, ef_off, bits, c.quant_level, c.quant_level_mod, c.formats);
		} else {
			find_best_combination_for_bitcount(pc, ef_off, bits, c.quant_level, c.quant_level_mod, c.formats);
		}
		cands[(int)k] = c;
	}
	wsync();
	if (keep_errors && w.lane == 0) {
		for (unsigned int k = 0; k < count; k++) {
			mode_err[(int)ASTC_F2U(taken[2 * (int)k])] = taken[2 * (int)k + 1];
		}
	}
	wsync();
	return count;
}
ASTC_COOP unsigned int endpoint_formats_select(WCtx w, int pc, int nplanes, unsigned int start_block_mode, unsigned int end_block_mode,
                                               uint32_t cand_off, bool keep_errors) {
	return endpoint_formats_select_t<false>(w, pc, nplanes, start_block_mode, end_block_mode, cand_off, keep_errors);
}

ASTC_COOP unsigned int compute_ideal_endpoint_formats(WCtx w, const PartView& pi, int ep0slot, int ep1slot, int nplanes,
                                                      unsigned int start_block_mode, unsigned int end_block_mode) {
	endpoint_formats_prepare(w, pi, ep0slot, ep1slot, nplanes, start_block_mode, end_block_mode);
	return endpoint_formats_select(w, (int)pi.partition_count, nplanes, start_block_mode, end_block_mode, w.base + A_CAND, false);
}

// =============================================================================================
// Least-squares endpoint refit (astcenc_ideal_endpoints_and_weights.cpp:1099-1650)
// =============================================================================================
ASTC_NOINLINE f4 compute_rgbo_vector(f4 rgba_weight_sum, f4 weight_weight_sum, f4 rgbq_sum, float psum) {
	float X = rgba_weight_sum.x, Y = rgba_weight_sum.y, Z = rgba_weight_sum.z;
	float P = weight_weight_sum.x, Q = weight_weight_sum.y, R = weight_weight_sum.z;
	float S = psum;
	float PP = P * P, QQ = Q * Q, RR = R * R;
	float SZmRR = S * Z - RR;
	float DT = SZmRR * Y - Z * QQ;
	float YP = Y * P, QX = Q * X, YX = Y * X;
	float mZYP = -Z * YP, mZQX = -Z * QX, mRYX = -R * YX;
	float ZQP = Z * Q * P, RYP = R * YP, RQX = R * QX;
	float rdet = 1.0f / (DT * X + mZYP * P);
	f4 mat0 = mk4(DT, ZQP, RYP, mZYP);
	f4 mat1 = mk4(ZQP, SZmRR * X - Z * PP, RQX, mZQX);
	f4 mat2 = mk4(RYP, RQX, (S * Y - QQ) * X - Y * PP, mRYX);
	f4 mat3 = mk4(mZYP, mZQX, mRYX, Z * YX);
	f4 vect = rgbq_sum * rdet;
	return mk4(dot_s(mat0, vect), dot_s(mat1, vect), dot_s(mat2, vect), dot_s(mat3, vect));
}

ASTC_FN f4 sel4(f4 a, f4 b, bool m0, bool m1, bool m2, bool m3) {
	return mk4(m0 ? b.x : a.x, m1 ? b.y : a.y, m2 ? b.z : a.z, m3 ? b.w : a.w);
}

ASTC_FN void rgbo_fallback(f4& rgbo, const f4& v0, const f4& v1) {
	float dd = dot_s(rgbo, rgbo);
	if (dd != dd) {
		float avgdif = hadd_rgb_s(v1 - v0) * (1.0f / 3.0f);
		avgdif = maxf(avgdif, 0.0f);
		f4 avg = (v0 + v1) * 0.5f;
		f4 ep0 = avg - splat4(avgdif) * 0.5f;
		rgbo = mk4(ep0.x, ep0.y, ep0.z, avgdif);
	}
}

// refinement scratch inside su (byte offsets in the shared window), laid out from the block size
struct RefineScratch {
	uint32_t undec[2];    // float[T] undecimated float weights per plane
	uint32_t texel_err;   // float[T] per-texel error terms for the ordered sums
	uint32_t uqf;         // float[64] realign: float copy of the quantised weights
	uint32_t iw[2];       // u8[T] integer undecimated weights (0..64) per plane
	uint32_t tile;        // chain staging tile: 20 x CHAIN_STRIDE floats
};
#define REFINE_TILE_BYTES (20 * CHAIN_STRIDE * 4)
// realign_weights: the wavefront replay is taken when pending weights * DEN > fronts * NUM (see there)
#if defined(ASTC_HOSTSIM)
static unsigned int g_hostsim_wavefront_replays;
#endif
#ifndef ASTC_REALIGN_WAVE_NUM
	#define ASTC_REALIGN_WAVE_NUM 1
	#define ASTC_REALIGN_WAVE_DEN 1
#endif

ASTC_FN RefineScratch make_refine_scratch(const WCtx& w) {
	RefineScratch r;
	uint32_t t4 = tp4(w);
	uint32_t f = su_of(w);
	r.undec[0] = f;
	r.undec[1] = f + t4;
	r.texel_err = f + 2 * t4;
	r.uqf = f + 3 * t4;
	r.tile = f + 3 * t4 + 256;
	r.iw[0] = r.tile + REFINE_TILE_BYTES;
	r.iw[1] = r.iw[0] + (t4 >> 2);
	return r;
}

// undecimate the quantised weights of `planes` planes: lanes over texels
ASTC_FN void undecimate_weights_t(const WCtx& w, unsigned int d, int planes) {
	RefineScratch rs = make_refine_scratch(w);
	DecView di = dec_view(d);
	int T = w.T;
	SPtr<uint8_t> uquant = work_weights_of(w);
	ASTC_NOUNROLL
	for (int id = w.lane; id < T * planes; id += ASTC_WARP) {
		int pl = id >= T ? 1 : 0;
		int t = id - pl * T;
		SPtr<uint8_t> uq = uquant + pl * 32;
		float v;
		if (di.max_twc == 1) {
			v = static_cast<float>(uq[t]) * (1.0f / 64.0f);
		} else {
			uint32_t ix = ASTC_LDD(&di.twi[t]);
			f4 c = dec_contribs(di, t);
			v = ((static_cast<float>(uq[(int)(ix & 0xFF)]) * (1.0f / 64.0f)) * c.x + (static_cast<float>(uq[(int)((ix >> 8) & 0xFF)]) * (1.0f / 64.0f)) * c.y) +
			    ((static_cast<float>(uq[(int)((ix >> 16) & 0xFF)]) * (1.0f / 64.0f)) * c.z + (static_cast<float>(uq[(int)(ix >> 24)]) * (1.0f / 64.0f)) * c.w);
		}
		sptr<float>(rs.undec[pl])[t] = v;
	}
	wsync();
}
ASTC_COOP void undecimate_weights(WCtx w, unsigned int d, int planes) {
	undecimate_weights_t(w, d, planes);
}

// recompute_ideal_colors_1plane :1146-1366. Per-texel terms (in partition-texel order):
//   0 left, 1 middle, 2 right, 3 weight_weight, 4-7 color_vec_x, 8-11 color_vec_y, 12-13 scale_vec;
// one chain per (partition, term).
// L1: one partition and LDR endpoints are compile-time facts (the refinement step of the one-partition, one-plane LDR trial inlines
// this instantiation; the out-of-line function is the general one).
template <bool L1> ASTC_FN void recompute_ideal_colors_1plane_t(const WCtx& w, const PartView& pi, unsigned int d) {
	RefineScratch rs = make_refine_scratch(w);
	const unsigned int pc = L1 ? 1u : pi.partition_count;
	if (L1) {
		undecimate_weights_t(w, d, 1);
	} else {
		undecimate_weights(w, d, 1);
	}
	SPtr<float> undec = sptr<float>(rs.undec[0]);
	SPtr<float> tmpf = tmpf_of(w);
	SPtr<float> sdv = tmpf + 64;            // scale_dir per partition, 4 floats each
	const BlkInfo& bi = bi_of(w);
	f4 color_weight = bi.channel_weight;
	float ls_weight = hadd_rgb_s(color_weight);
	SPtr<float> b0 = blk_of(w, 0);
	uint32_t cs = tp4(w);
	// phase A: per-partition colour sums (needed for scale_dir)
	if (pc > 1) {
		ASTC_NOUNROLL
		for (int id = w.lane; id < (int)pc * 4; id += ASTC_WARP) {
			unsigned int p = (unsigned int)id >> 2;
			int c = id & 3;
			const uint8_t* tix = pi.texels + pv_start(pi, p);
			int n = pv_count(pi, p);
			SPtr<float> dch = sptr<float>(b0.off + (uint32_t)c * cs);
			float s = 0.0f;
			ASTC_UNROLL_R4
			for (int j = 0; j < n; j++) {
				s = s + dch[ASTC_LDG(&tix[j])];
			}
			tmpf[96 + id] = s;
		}
		wsync();
	}
	// scale_dir per partition -> sdv (shared), read back by the term and solve phases
	if (w.lane == 0) {
		ASTC_NOUNROLL
		for (unsigned int p = 0; p < pc; p++) {
			f4 rgba_sum = pc > 1 ? mk4(tmpf[96 + (int)p * 4], tmpf[96 + (int)p * 4 + 1], tmpf[96 + (int)p * 4 + 2], tmpf[96 + (int)p * 4 + 3])
			                     : bi.data_mean * static_cast<float>(w.T);
			rgba_sum = rgba_sum * color_weight;
			f4 rws = max4(color_weight * static_cast<float>(pv_count(pi, p)), splat4(1e-17f));
			f4 q = rgba_sum / rws;
			f4 sd = normalize4(mk4(q.x, q.y, q.z, 0.0f));
			sdv[(int)p * 4] = sd.x;
			sdv[(int)p * 4 + 1] = sd.y;
			sdv[(int)p * 4 + 2] = sd.z;
			sdv[(int)p * 4 + 3] = sd.w;
		}
	}
	int nchains = (int)pc * 14;
	ASTC_NOUNROLL
	for (int id = w.lane; id < nchains; id += ASTC_WARP) {
		tmpf[id] = (id % 14) == 3 ? 1e-17f : 0.0f;
	}
	wsync();
	// phase B: the weighted sums
	chain_sums<14>(w, w.T, rs.tile, tmpf, nchains,
		[&](int pos, float* term) {
			int t = pv_texel(pi, pos);
			int p = pc > 1 ? (int)ASTC_LDG(&pi.partition_of_texel[t]) : 0;
			float idx0 = undec[t];
			float om_idx0 = 1.0f - idx0;
			SPtr<float> tx = b0 + t;
			float r = tx[0], g = sptr<float>(tx.off + cs)[0], b = sptr<float>(tx.off + 2 * cs)[0], a = sptr<float>(tx.off + 3 * cs)[0];
			term[0] = om_idx0 * om_idx0;
			term[1] = om_idx0 * idx0;
			term[2] = idx0 * idx0;
			term[3] = idx0;
			float ri = r * idx0, gi = g * idx0, bi2 = b * idx0, ai = a * idx0;
			term[4] = r - ri;
			term[5] = g - gi;
			term[6] = b - bi2;
			term[7] = a - ai;
			term[8] = ri;
			term[9] = gi;
			term[10] = bi2;
			term[11] = ai;
			SPtr<float> sd = sdv + p * 4;
			float scale = (sd[0] * r + sd[1] * g) + sd[2] * b;
			term[12] = om_idx0 * (scale * ls_weight);
			term[13] = idx0 * (scale * ls_weight);
		},
		[&](int id, int& k, int& lo, int& hi, int& step) {
			int p = id / 14;
			k = id - p * 14;
			lo = pv_start(pi, (unsigned int)p);
			hi = lo + pv_count(pi, (unsigned int)p);
			step = 1;
		});
	SPtr<float> mm = tmpf + 112;            // per partition: weight min, weight max, scale min, scale max
	ASTC_NOUNROLL
	for (unsigned int p = 0; p < pc; p++) {
		const uint8_t* tix = pi.texels + pv_start(pi, p);
		int n = pv_count(pi, p);
		SPtr<float> sdp = sdv + (int)p * 4;
		f4 sd = mk4(sdp[0], sdp[1], sdp[2], sdp[3]);
		float a = 1.0f, b = 0.0f, c = 1e10f, dd = 0.0f;
		ASTC_NOUNROLL
		for (int j = w.lane; j < n; j += ASTC_WARP) {
			int t = pc > 1 ? (int)ASTC_LDG(&tix[j]) : j;
			float idx0 = undec[t];
			a = minf(idx0, a);
			b = maxf(idx0, b);
			float scale = dot3_s(sd, texel4(w, t));
			c = minf(scale, c);
			dd = maxf(scale, dd);
		}
		a = wmin_f(a);
		b = wmax_f(b);
		c = wmin_f(c);
		dd = wmax_f(dd);
		if (w.lane == 0) {
			mm[(int)p * 4] = a;
			mm[(int)p * 4 + 1] = b;
			mm[(int)p * 4 + 2] = c;
			mm[(int)p * 4 + 3] = dd;
		}
	}
	wsync();
	// phase C: the solves, one lane per (partition, channel): every channel of the reference's vfloat4 algebra is
	// independent, the per-partition scalars are recomputed by the four lanes of a partition
	SPtr<float> epf = sptr<float>(ep_of(w).off);          // endpoint slots as floats: slot * 4 + channel
	ASTC_NOUNROLL
	for (unsigned int k = (unsigned int)w.lane; k < pc * 4; k += ASTC_WARP) {
		unsigned int i = k >> 2;
		int c = (int)(k & 3);
		SPtr<float> a = tmpf + (int)i * 14;
		float left_sum_s = a[0], middle_sum_s = a[1], right_sum_s = a[2];
		float cw_c = lane(color_weight, c);
		float color_vec_x = a[4 + c] * cw_c;
		float color_vec_y = a[8 + c] * cw_c;
		float scale_vec_x = a[12], scale_vec_y = a[13];
		float sdir_c = sdv[(int)i * 4 + c];
		float rws_c = maxf(cw_c * static_cast<float>(pv_count(pi, i)), 1e-17f);
		float wmn = mm[(int)i * 4], wmx = mm[(int)i * 4 + 1], smn = mm[(int)i * 4 + 2], smx = mm[(int)i * 4 + 3];
		float left_sum = left_sum_s * cw_c;
		float middle_sum = middle_sum_s * cw_c;
		float right_sum = right_sum_s * cw_c;
		float lmrs_x = left_sum_s * ls_weight, lmrs_y = middle_sum_s * ls_weight, lmrs_z = right_sum_s * ls_weight;
		float scalediv = smn / maxf(smx, 1e-10f);
		scalediv = clamp1f(scalediv);
		float rgbs_c = c < 3 ? sdir_c * smx : scalediv;
		float e0 = epf[(EP_WORK_0 + (int)i) * 4 + c], e1 = epf[(EP_WORK_1 + (int)i) * 4 + c];
		if (wmn >= wmx * 0.999f) {
			float avg = (color_vec_x + color_vec_y) / rws_c;
			if (avg == avg) {
				e0 = avg;
				e1 = avg;
			}
			if (c == 3) {
				rgbs_c = 1.0f;
			}
		} else {
			float color_det1 = (left_sum * right_sum) - (middle_sum * middle_sum);
			float color_rdet1 = 1.0f / color_det1;
			float ls_det1 = (lmrs_x * lmrs_z) - (lmrs_y * lmrs_y);
			float ls_rdet1 = 1.0f / ls_det1;
			float color_mss1 = (left_sum * left_sum) + (2.0f * middle_sum * middle_sum) + (right_sum * right_sum);
			float ls_mss1 = (lmrs_x * lmrs_x) + (2.0f * lmrs_y * lmrs_y) + (lmrs_z * lmrs_z);
			float ep0 = (right_sum * color_vec_x - middle_sum * color_vec_y) * color_rdet1;
			float ep1 = (left_sum * color_vec_y - middle_sum * color_vec_x) * color_rdet1;
			float thr = color_mss1 * 1e-4f;
			if (absf(color_det1) > thr && ep0 == ep0 && ep1 == ep1) {
				e0 = ep0;
				e1 = ep1;
			}
			float scale_ep0 = (lmrs_z * scale_vec_x - lmrs_y * scale_vec_y) * ls_rdet1;
			float scale_ep1 = (lmrs_x * scale_vec_y - lmrs_y * scale_vec_x) * ls_rdet1;
			if (fabsf(ls_det1) > (ls_mss1 * 1e-4f) && scale_ep0 == scale_ep0 && scale_ep1 == scale_ep1 && scale_ep0 < scale_ep1) {
				rgbs_c = c < 3 ? sdir_c * scale_ep1 : scale_ep0 / scale_ep1;
			}
		}
		epf[(EP_WORK_0 + (int)i) * 4 + c] = e0;
		epf[(EP_WORK_1 + (int)i) * 4 + c] = e1;
		epf[(EP_RGBS + (int)i) * 4 + c] = rgbs_c;
	}
	wsync();
	if (!L1 && (bi.rgb_lns0 || bi.alpha_lns0)) {
		// HDR: the RGBO fit mixes the channels - one lane per partition
		SPtr<f4> ep = ep_of(w);
		ASTC_NOUNROLL
		for (unsigned int i = (unsigned int)w.lane; i < pc; i += ASTC_WARP) {
			SPtr<float> a = tmpf + (int)i * 14;
			float right_sum_s = a[2], weight_weight_sum_s = a[3];
			f4 color_vec_x = mk4(a[4], a[5], a[6], a[7]) * color_weight;
			f4 color_vec_y = mk4(a[8], a[9], a[10], a[11]) * color_weight;
			f4 rws = max4(color_weight * static_cast<float>(pv_count(pi, i)), splat4(1e-17f));
			f4 weight_weight_sum = splat4(weight_weight_sum_s) * color_weight;
			float psum = right_sum_s * hadd_rgb_s(color_weight);
			f4 rgbq_sum = color_vec_x + color_vec_y;
			rgbq_sum.w = hadd_rgb_s(color_vec_y);
			f4 rgbovec = compute_rgbo_vector(rws, weight_weight_sum, rgbq_sum, psum);
			rgbo_fallback(rgbovec, ep[EP_WORK_0 + (int)i], ep[EP_WORK_1 + (int)i]);
			ep[EP_RGBO + (int)i] = rgbovec;
		}
		wsync();
	}
}
ASTC_COOP void recompute_ideal_colors_1plane(WCtx w, const PartView& pi, unsigned int d) {
	recompute_ideal_colors_1plane_t<false>(w, pi, d);
}

// recompute_ideal_colors_2planes :1369-1650. Per-texel terms (texel order):
//   0-2 left/middle/right plane 1, 3-5 plane 2, 6-9 color_vec_x, 10-13 color_vec_y, 14-15 scale_vec, 16-19 weight_weight_sum
ASTC_COOP void recompute_ideal_colors_2planes(WCtx w, unsigned int d, int plane2_component) {
	RefineScratch rs = make_refine_scratch(w);
	int T = w.T;
	undecimate_weights(w, d, 2);
	SPtr<float> undec1 = sptr<float>(rs.undec[0]);
	SPtr<float> undec2 = sptr<float>(rs.undec[1]);
	SPtr<float> tmpf = tmpf_of(w);
	const BlkInfo& bi = bi_of(w);
	f4 color_weight = bi.channel_weight;
	float ls_weight = hadd_rgb_s(color_weight);
	f4 rgba_weight_sum = max4(color_weight * static_cast<float>(T), splat4(1e-17f));
	f4 dmean = bi.data_mean;
	f4 scale_dir = normalize4(mk4(dmean.x, dmean.y, dmean.z, 0.0f));
	SPtr<float> b0 = blk_of(w, 0);
	uint32_t cs = tp4(w);
	ASTC_NOUNROLL
	for (int id = w.lane; id < 20; id += ASTC_WARP) {
		tmpf[id] = id >= 16 ? 1e-17f : 0.0f;
	}
	wsync();
	chain_sums<20>(w, T, rs.tile, tmpf, 20,
		[&](int j, float* term) {
			float idx0 = undec1[j];
			float om_idx0 = 1.0f - idx0;
			float idx1 = undec2[j];
			float om_idx1 = 1.0f - idx1;
			SPtr<float> tx = b0 + j;
			float r = tx[0], g = sptr<float>(tx.off + cs)[0], b = sptr<float>(tx.off + 2 * cs)[0], a = sptr<float>(tx.off + 3 * cs)[0];
			term[0] = om_idx0 * om_idx0;
			term[1] = om_idx0 * idx0;
			term[2] = idx0 * idx0;
			term[3] = om_idx1 * om_idx1;
			term[4] = om_idx1 * idx1;
			term[5] = idx1 * idx1;
			float i_r = plane2_component == 0 ? idx1 : idx0;
			float i_g = plane2_component == 1 ? idx1 : idx0;
			float i_b = plane2_component == 2 ? idx1 : idx0;
			float i_a = plane2_component == 3 ? idx1 : idx0;
			float ri = r * i_r, gi = g * i_g, bi2 = b * i_b, ai = a * i_a;
			term[6] = r - ri;
			term[7] = g - gi;
			term[8] = b - bi2;
			term[9] = a - ai;
			term[10] = ri;
			term[11] = gi;
			term[12] = bi2;
			term[13] = ai;
			float scale = (scale_dir.x * r + scale_dir.y * g) + scale_dir.z * b;
			term[14] = om_idx0 * (ls_weight * scale);
			term[15] = idx0 * (ls_weight * scale);
			term[16] = i_r;
			term[17] = i_g;
			term[18] = i_b;
			term[19] = i_a;
		},
		[&](int id, int& k, int& lo, int& hi, int& step) {
			k = id;
			lo = 0;
			hi = T;
			step = 1;
		});
	float a = 1.0f, b = 0.0f, a2 = 1.0f, b2 = 0.0f, c = 1e10f, dd = 0.0f;
	ASTC_NOUNROLL
	for (int j = w.lane; j < T; j += ASTC_WARP) {
		float idx0 = undec1[j];
		float idx1 = undec2[j];
		a = minf(idx0, a);
		b = maxf(idx0, b);
		a2 = minf(idx1, a2);
		b2 = maxf(idx1, b2);
		float scale = dot3_s(scale_dir, texel4(w, j));
		c = minf(scale, c);
		dd = maxf(scale, dd);
	}
	float wmin1 = wmin_f(a), wmax1 = wmax_f(b), wmin2 = wmin_f(a2), wmax2 = wmax_f(b2);
	float scale_min = wmin_f(c), scale_max = wmax_f(dd);
	wsync();
	// the solves: one lane per channel (the plane-2 component uses the plane-2 sums, the others the plane-1 sums)
	{
		SPtr<float> t = tmpf;
		SPtr<float> epf = sptr<float>(ep_of(w).off);
		ASTC_NOUNROLL
		for (int c = w.lane; c < 4; c += ASTC_WARP) {
			bool p2 = c == plane2_component;
			float cw_c = lane(color_weight, c);
			float color_vec_x = t[6 + c] * cw_c;
			float color_vec_y = t[10 + c] * cw_c;
			float rws_c = lane(rgba_weight_sum, c);
			float left_s = p2 ? t[3] : t[0], middle_s = p2 ? t[4] : t[1], right_s = p2 ? t[5] : t[2];
			float wmn = p2 ? wmin2 : wmin1, wmx = p2 ? wmax2 : wmax1;
			float left_sum = left_s * cw_c, middle_sum = middle_s * cw_c, right_sum = right_s * cw_c;
			float e0 = epf[EP_WORK_0 * 4 + c], e1 = epf[EP_WORK_1 * 4 + c];
			if (wmn >= wmx * 0.999f) {
				float avg = (color_vec_x + color_vec_y) / rws_c;
				if (avg == avg) {
					e0 = avg;
					e1 = avg;
				}
			} else {
				float color_det = (left_sum * right_sum) - (middle_sum * middle_sum);
				float color_rdet = 1.0f / color_det;
				float color_mss = (left_sum * left_sum) + (2.0f * middle_sum * middle_sum) + (right_sum * right_sum);
				float ep0 = (right_sum * color_vec_x - middle_sum * color_vec_y) * color_rdet;
				float ep1 = (left_sum * color_vec_y - middle_sum * color_vec_x) * color_rdet;
				if (absf(color_det) > color_mss * 1e-4f && ep0 == ep0 && ep1 == ep1) {
					e0 = ep0;
					e1 = ep1;
				}
			}
			// the RGBS vector always comes from plane 1
			float lmrs_x = t[0] * ls_weight, lmrs_y = t[1] * ls_weight, lmrs_z = t[2] * ls_weight;
			float scalediv = scale_min / maxf(scale_max, 1e-10f);
			scalediv = clamp1f(scalediv);
			float sdir_c = lane(scale_dir, c);
			float rgbs_c = c < 3 ? sdir_c * scale_max : scalediv;
			if (wmin1 >= wmax1 * 0.999f) {
				if (c == 3) {
					rgbs_c = 1.0f;
				}
			} else {
				float ls_det1 = (lmrs_x * lmrs_z) - (lmrs_y * lmrs_y);
				float ls_rdet1 = 1.0f / ls_det1;
				float ls_mss1 = (lmrs_x * lmrs_x) + (2.0f * lmrs_y * lmrs_y) + (lmrs_z * lmrs_z);
				float scale_ep0 = (lmrs_z * t[14] - lmrs_y * t[15]) * ls_rdet1;
				float scale_ep1 = (lmrs_x * t[15] - lmrs_y * t[14]) * ls_rdet1;
				if (fabsf(ls_det1) > (ls_mss1 * 1e-4f) && scale_ep0 == scale_ep0 && scale_ep1 == scale_ep1 && scale_ep0 < scale_ep1) {
					rgbs_c = c < 3 ? sdir_c * scale_ep1 : scale_ep0 / scale_ep1;
				}
			}
			epf[EP_WORK_0 * 4 + c] = e0;
			epf[EP_WORK_1 * 4 + c] = e1;
			epf[EP_RGBS * 4 + c] = rgbs_c;
		}
	}
	wsync();
	if ((bi.rgb_lns0 || bi.alpha_lns0) && w.lane == 0) {
		// HDR: the RGBO fit mixes the channels
		SPtr<float> t = tmpf;
		SPtr<f4> ep = ep_of(w);
		bool p20 = plane2_component == 0, p21 = plane2_component == 1, p22 = plane2_component == 2, p23 = plane2_component == 3;
		f4 color_vec_x = mk4(t[6], t[7], t[8], t[9]) * color_weight;
		f4 color_vec_y = mk4(t[10], t[11], t[12], t[13]) * color_weight;
		f4 weight_weight_sum = mk4(t[16], t[17], t[18], t[19]) * color_weight;
		f4 right1_sum = splat4(t[2]) * color_weight;
		f4 right2_sum = splat4(t[5]) * color_weight;
		f4 rsel = mk4(p20 ? right2_sum.x : right1_sum.x, p21 ? right2_sum.y : right1_sum.y, p22 ? right2_sum.z : right1_sum.z,
		              p23 ? right2_sum.w : right1_sum.w);
		float psum = dot3_s(rsel, color_weight);
		f4 rgbq_sum = color_vec_x + color_vec_y;
		rgbq_sum.w = hadd_rgb_s(color_vec_y);
		f4 rgbo_vector = compute_rgbo_vector(rgba_weight_sum, weight_weight_sum, rgbq_sum, psum);
		rgbo_fallback(rgbo_vector, ep[EP_WORK_0], ep[EP_WORK_1]);
		ep[EP_RGBO] = rgbo_vector;
	}
	wsync();
}

// =============================================================================================
// Decompress-and-diff scoring (astcenc_decompress_symbolic.cpp:89-618)
// =============================================================================================
ASTC_FN bool u8_mask(const WCtx& w) { return bi_of(w).decode_unorm8 || CFG.profile == PRF_LDR_SRGB; }

ASTC_FN int lerp1(bool u8, int c0, int c1, int w1) {   // lerp_color_int :37-61
	int w0 = 64 - w1;
	int color = (c0 * w0) + (c1 * w1) + 32;
	color = color >> 6;
	if (u8) {
		color = (color >> 8) * 257;
	}
	return color;
}

// Unpack the integer endpoints of the work candidate into the arena: ends[p * 8 + 0..3] = endpoint 0 (rgba), + 4..7 = endpoint 1.
template <bool L1> ASTC_FN void unpack_work_endpoints_t(const WCtx& w, unsigned int pc_in, uint32_t formats, uint32_t ends_off) {
	const unsigned int pc = L1 ? 1u : pc_in;
	SPtr<int> ends = sptr<int>(ends_off);
	SPtr<uint8_t> wc = work_colors_of(w);
	ASTC_NOUNROLL
	for (unsigned int p = (unsigned int)w.lane; p < pc; p += ASTC_WARP) {
		const uint8_t* in = &wc[(int)p * 8];      // (straight from the shared arena: no local copy)
		bool rgb_lns, a_lns;
		i4 e0, e1;
		unpack_color_endpoints_inl<L1>(CFG.profile, (int)((formats >> (8 * p)) & 0xFF), in, rgb_lns, a_lns, e0, e1);
		SPtr<int> o = ends + (int)p * 8;
		o[0] = e0.x; o[1] = e0.y; o[2] = e0.z; o[3] = e0.w;
		o[4] = e1.x; o[5] = e1.y; o[6] = e1.z; o[7] = e1.w;
	}
	wsync();
}
ASTC_COOP void unpack_work_endpoints(WCtx w, unsigned int pc, uint32_t formats, uint32_t ends_off) {
	unpack_work_endpoints_t<false>(w, pc, formats, ends_off);
}
ASTC_FN uint32_t pack_formats(const ScbHdr& h) {
	return (uint32_t)h.color_formats[0] | ((uint32_t)h.color_formats[1] << 8) | ((uint32_t)h.color_formats[2] << 16) | ((uint32_t)h.color_formats[3] << 24);
}
// the unpacked endpoints live in tmpf[96..128) (32 ints) from the end of the packing stage of a refinement step until its
// last score: packing is the only thing that changes them, scoring and realignment only read them
ASTC_FN uint32_t ends_off_of(const WCtx& w) { return w.base + A_TMPF + 96 * 4; }

// compute_symbolic_block_difference_{2plane,1plane,1plane_1partition} (:313-618) on the work candidate.
// Per-texel terms by lanes over texels (integer infill :89-167 inlined), then the reference's summation order:
// 4-lane accumulator (1 partition, 1 plane, no RGBM) or one scalar chain.
template <bool L1> ASTC_FN float compute_symbolic_block_difference_t(const WCtx& w, unsigned int pc_in, uint32_t formats, int plane2_in, const PartView& pi, unsigned int d, bool dual_in) {
	const unsigned int pc = L1 ? 1u : pc_in;
	const int plane2_component = L1 ? -1 : plane2_in;
	const bool dual = L1 ? false : dual_in;
	RefineScratch rs = make_refine_scratch(w);
	DecView di = dec_view(d);
	int T = w.T;
	bool rgbm = (CFG.flags & FLG_MAP_RGBM) != 0;
	float rgbm_scale = CFG.rgbm_m_scale;
	bool fast = !dual && pc == 1 && !rgbm;
	bool u8 = u8_mask(w);
	(void)formats;      // the caller unpacked the work candidate's endpoints (unpack_work_endpoints) after packing them
	SPtr<int> ends = sptr<int>(ends_off_of(w));
	SPtr<uint8_t> uq = work_weights_of(w);
	SPtr<float> texel_err = sptr<float>(rs.texel_err);
	SPtr<float> tmpf = tmpf_of(w);
	f4 cw = bi_of(w).channel_weight;
	SPtr<float> b0 = blk_of(w, 0);
	uint32_t cs = tp4(w);
	bool reject = false;
	ASTC_NOUNROLL
	for (int t = w.lane; t < T; t += ASTC_WARP) {
		uint32_t ix = ASTC_LDD(&di.twi[t]);
		uint32_t cx = ASTC_LDD(&di.tci[t]);
		int i0 = (int)(ix & 0xFF), i1 = (int)((ix >> 8) & 0xFF), i2 = (int)((ix >> 16) & 0xFF), i3 = (int)(ix >> 24);
		int c0 = (int)(cx & 0xFF), c1 = (int)((cx >> 8) & 0xFF), c2 = (int)((cx >> 16) & 0xFF), c3 = (int)(cx >> 24);
		int w1 = (8 + uq[i0] * c0 + uq[i1] * c1 + uq[i2] * c2 + uq[i3] * c3) >> 4;
		int w2 = w1;
		if (dual) {
			w2 = (8 + uq[32 + i0] * c0 + uq[32 + i1] * c1 + uq[32 + i2] * c2 + uq[32 + i3] * c3) >> 4;
		}
		int p = pc > 1 ? (int)ASTC_LDG(&pi.partition_of_texel[t]) : 0;
		SPtr<int> e = ends + p * 8;
		float cr = (float)lerp1(u8, e[0], e[4], plane2_component == 0 ? w2 : w1);
		float cg = (float)lerp1(u8, e[1], e[5], plane2_component == 1 ? w2 : w1);
		float cb = (float)lerp1(u8, e[2], e[6], plane2_component == 2 ? w2 : w1);
		float ca = (float)lerp1(u8, e[3], e[7], plane2_component == 3 ? w2 : w1);
		SPtr<float> tx = b0 + t;
		float orr = tx[0], og = sptr<float>(tx.off + cs)[0], ob = sptr<float>(tx.off + 2 * cs)[0], oa = sptr<float>(tx.off + 3 * cs)[0];
		float metric;
		if (fast) {
			float er = minf(absf(orr - cr), 1e15f);
			float eg = minf(absf(og - cg), 1e15f);
			float eb = minf(absf(ob - cb), 1e15f);
			float ea = minf(absf(oa - ca), 1e15f);
			er = er * er;
			eg = eg * eg;
			eb = eb * eb;
			ea = ea * ea;
			metric = er * cw.x + eg * cw.y + eb * cw.z + ea * cw.w;
		} else {
			f4 color = mk4(cr, cg, cb, ca);
			f4 old = mk4(orr, og, ob, oa);
			if (rgbm) {
				if (color.w == 0.0f) {
					reject = true;
				}
				color = mk4(color.x * color.w * rgbm_scale, color.y * color.w * rgbm_scale, color.z * color.w * rgbm_scale, 1.0f);
				old = mk4(old.x * old.w * rgbm_scale, old.y * old.w * rgbm_scale, old.z * old.w * rgbm_scale, 1.0f);
			}
			f4 error = old - color;
			error = min4(mk4(absf(error.x), absf(error.y), absf(error.z), absf(error.w)), splat4(1e15f));
			error = error * error;
			metric = minf(dot_s(error, cw), ERROR_CALC_DEFAULT);
		}
		texel_err[t] = metric;
	}
	// The reference returns -1e30 at the first texel (in its iteration order) whose decoded alpha is 0; any
	// such texel makes the result -1e30, so the order does not matter for the rejection itself.
	reject = wany(reject);
	wsync();
	if (reject) {
		return -ERROR_CALC_DEFAULT;
	}
	if (fast) {
		ASTC_NOUNROLL
		for (int l = w.lane; l < 4; l += ASTC_WARP) {
			float s = 0.0f;
			ASTC_UNROLL_R4
			for (int t = l; t < T; t += 4) {
				s = s + texel_err[t];
			}
			tmpf[l] = s;
		}
		wsync();
		float r = (tmpf[0] + tmpf[2]) + (tmpf[1] + tmpf[3]);
		wsync();
		return r;
	}
	if (w.lane == 0) {
		float summa = 0.0f;
		if (dual || pc == 1) {
			ASTC_NOUNROLL
			for (int t = 0; t < T; t++) {
				summa += texel_err[t];
			}
		} else {
			ASTC_NOUNROLL
			for (int t = 0; t < T; t++) {
				summa += texel_err[ASTC_LDG(&pi.texels[t])];
			}
		}
		tmpf[0] = summa;
	}
	wsync();
	float r = tmpf[0];
	wsync();
	return r;
}
ASTC_COOP float compute_symbolic_block_difference(WCtx w, unsigned int pc, uint32_t formats, int plane2_component, const PartView& pi, unsigned int d, bool dual) {
	return compute_symbolic_block_difference_t<false>(w, pc, formats, plane2_component, pi, d, dual);
}

// =============================================================================================
// Weight realignment (astcenc_compress_symbolic.cpp:69-350)
// =============================================================================================
// Decimated grids (:188-350): weights are visited in order and a changed weight feeds the following ones, so
// the outer loop is sequential. Per weight, lane = (texel slot 0..7, channel 0..3): eight of the weight's texels
// at a time compute their squared channel differences for the current / previous / next quantised value into a
// [12][8] tile; twelve chain lanes (3 candidates x 4 channels) then add them in texel order, and a few shuffles fold
// the channel sums the way the reference's dot product does. The bilinear infill of every texel (wb) is kept
// current instead of being rebuilt for every weight: it only changes for the texels of a weight that moved.
template <bool L1> ASTC_FN bool realign_weights_t(const WCtx& w, unsigned int pc_in, uint32_t formats, int plane2_in, const PartView& pi, int quant_mode, bool dual_in, unsigned int d) {
	const unsigned int pc = L1 ? 1u : pc_in;
	const int plane2_component = L1 ? -1 : plane2_in;
	const bool is_dual = L1 ? false : dual_in;
	const DevConstTables* ct = ASTC_CT;
	RefineScratch rs = make_refine_scratch(w);
	DecView di = dec_view(d);
	const uint16_t* prev_next = ct->wq_prev_next[quant_mode];
	int weight_count = di.W;
	int T = w.T;
	bool decimated = weight_count != T;
	unsigned int max_plane = is_dual ? 1u : 0u;
	(void)formats;      // endpoints already unpacked by the caller (once per refinement step)
	SPtr<int> ends = sptr<int>(ends_off_of(w));
	f4 ew = bi_of(w).channel_weight;
	SPtr<float> uqf = sptr<float>(rs.uqf);
	SPtr<float> wb = sptr<float>(rs.undec[0]);        // per-texel infill of uqf (free here: recompute rebuilds its own)
	SPtr<float> tmpf = tmpf_of(w);
	SPtr<float> eb = tmpf + 32;                       // endpoint 0 as float, [partition][channel]
	SPtr<float> eo = tmpf + 48;                       // (endpoint 1 - endpoint 0) / 64, plane-masked
	SPtr<float> b0 = blk_of(w, 0);
	uint32_t cs = tp4(w);
	bool adjustments = false;
	ASTC_NOUNROLL
	for (unsigned int pl = 0; pl <= max_plane; pl++) {
		SPtr<uint8_t> dec_weights_uquant = work_weights_of(w) + (int)pl * 32;
		// plane_mask: for plane 1 the plane-2 component is zeroed, for plane 2 all others
		ASTC_NOUNROLL
		for (int k = w.lane; k < (int)pc * 4; k += ASTC_WARP) {
			int p = k >> 2, c = k & 3;
			int e0 = ends[p * 8 + c], e1 = ends[p * 8 + 4 + c];
			bool masked = (plane2_component == c) != (pl == 1);
			eb[k] = static_cast<float>(e0);
			eo[k] = static_cast<float>(masked ? 0 : e1 - e0) * (1.0f / 64.0f);
		}
		wsync();
		if (!decimated) {
			// realign_weights_undecimated :69-185 - texels are independent
			ASTC_NOUNROLL
			for (int texel = w.lane; texel < T; texel += ASTC_WARP) {
				int uqw = dec_weights_uquant[texel];
				uint32_t pn = ASTC_LDG(&prev_next[uqw]);
				int uqw_down = pn & 0xFF;
				int uqw_up = (pn >> 8) & 0xFF;
				float weight_base = static_cast<float>(uqw);
				float weight_down = static_cast<float>(uqw_down - uqw);
				float weight_up = static_cast<float>(uqw_up - uqw);
				int partition = pc > 1 ? (int)ASTC_LDG(&pi.partition_of_texel[texel]) : 0;
				float t0[4], t1[4], t2[4];
				for (int c = 0; c < 4; c++) {
					float color_offset = eo[partition * 4 + c];
					float color = eb[partition * 4 + c] + color_offset * weight_base;
					float orig = sptr<float>(b0.off + (uint32_t)c * cs)[texel];
					float color_diff = color - orig;
					float color_diff_down = color_diff + color_offset * weight_down;
					float color_diff_up = color_diff + color_offset * weight_up;
					float ewc = lane(ew, c);
					t0[c] = color_diff * color_diff * ewc;
					t1[c] = color_diff_down * color_diff_down * ewc;
					t2[c] = color_diff_up * color_diff_up * ewc;
				}
				float ebs = (t0[0] + t0[2]) + (t0[1] + t0[3]);      // dot_s: (x + z) + (y + w)
				float ed = (t1[0] + t1[2]) + (t1[1] + t1[3]);
				float eu = (t2[0] + t2[2]) + (t2[1] + t2[3]);
				if ((eu < ebs) && (eu < ed) && (uqw < 64)) {
					dec_weights_uquant[texel] = static_cast<uint8_t>(uqw_up);
					adjustments = true;
				} else if ((ed < ebs) && (uqw > 0)) {
					dec_weights_uquant[texel] = static_cast<uint8_t>(uqw_down);
					adjustments = true;
				}
			}
			wsync();
			continue;
		}
		// Stage everything the sequential weight loop reads in shared memory (the staging tile is free here), so an
		// iteration never waits for global memory: per weight its previous/next quantised value and list range,
		// the list entries, the partition of every texel.
		SPtr<uint16_t> s_pn = sptr<uint16_t>(rs.tile);                       // [64]
		SPtr<uint16_t> s_wto = sptr<uint16_t>(rs.tile + 128);                // [65]
		const uint32_t tp = (uint32_t)((T + 3) & ~3);                        // (T <= 216: 264 + 216 + 1728 + 64 <= REFINE_TILE_BYTES)
		SPtr<uint8_t> s_pot = sptr<uint8_t>(rs.tile + 128 + 136);           // [T]
		SPtr<uint16_t> s_wtc = sptr<uint16_t>(rs.tile + 128 + 136 + tp);     // [E] (<= 4 T)
		ASTC_NOUNROLL
		for (int we = w.lane; we <= weight_count; we += ASTC_WARP) {
			s_wto[we] = ASTC_LDD(&di.wto[we]);
			if (we < weight_count) {
				int uq = dec_weights_uquant[we];
				uqf[we] = static_cast<float>(uq);
				s_pn[we] = ASTC_LDG(&prev_next[uq]);
			}
		}
		ASTC_NOUNROLL
		for (int t = w.lane; t < T; t += ASTC_WARP) {
			s_pot[t] = pc > 1 ? ASTC_LDG(&pi.partition_of_texel[t]) : (uint8_t)0;
		}
		wsync();
		int E = s_wto[weight_count];
		ASTC_NOUNROLL
		for (int e = w.lane; e < E; e += ASTC_WARP) {
			s_wtc[e] = ASTC_LDD(&di.wtc[e]);
		}
		ASTC_NOUNROLL
		for (int t = w.lane; t < T; t += ASTC_WARP) {
			wb[t] = bilinear_infill(di, uqf, t);
		}
		wsync();
#if ASTC_WARP == 1
		// serial form (one simulated lane / the single-lane debug build): the reference's loop as it stands
		ASTC_NOUNROLL
		for (int we = 0; we < weight_count; we++) {
			uint32_t pn = s_pn[we];
			float uqw_base = uqf[we];
			int uqw = (int)uqw_base;
			float uqw_down = static_cast<float>(pn & 0xFF);
			float uqw_up = static_cast<float>((pn >> 8) & 0xFF);
			float uqw_diff_down = uqw_down - uqw_base;
			float uqw_diff_up = uqw_up - uqw_base;
			int off = s_wto[we];
			int cnt = s_wto[we + 1] - off;
			// 12 ordered channel sums, then the weighted (x + z) + (y + w) fold
			float acc[12];
			for (int k = 0; k < 12; k++) acc[k] = 0.0f;
			for (int te = 0; te < cnt; te++) {
				uint32_t e = s_wtc[off + te];
				int texel = (int)(e & 0xFF);
				float tw_base = static_cast<float>(e >> 8) * (1.0f / 16.0f);
				float weight_base = wb[texel];
				float weight_down = weight_base + uqw_diff_down * tw_base - weight_base;
				float weight_up = weight_base + uqw_diff_up * tw_base - weight_base;
				int partition = s_pot[texel];
				for (int c = 0; c < 4; c++) {
					float color_offset = eo[partition * 4 + c];
					float color = eb[partition * 4 + c] + color_offset * weight_base;
					float orig = sptr<float>(b0.off + (uint32_t)c * cs)[texel];
					float color_diff = color - orig;
					float color_down_diff = color_diff + color_offset * weight_down;
					float color_up_diff = color_diff + color_offset * weight_up;
					acc[c] = acc[c] + color_diff * color_diff;
					acc[4 + c] = acc[4 + c] + color_down_diff * color_down_diff;
					acc[8 + c] = acc[8 + c] + color_up_diff * color_up_diff;
				}
			}
			for (int k = 0; k < 12; k++) acc[k] = acc[k] * lane(ew, k & 3);
			float error_base = (acc[0] + acc[2]) + (acc[1] + acc[3]);
			float error_down = (acc[4] + acc[6]) + (acc[5] + acc[7]);
			float error_up = (acc[8] + acc[10]) + (acc[9] + acc[11]);
			float new_uqw = -1.0f;
			if ((error_up < error_base) && (error_up < error_down) && (uqw < 64)) {
				new_uqw = uqw_up;
			} else if ((error_down < error_base) && (uqw > 0)) {
				new_uqw = uqw_down;
			}
			if (new_uqw >= 0.0f) {
				uqf[we] = new_uqw;
				dec_weights_uquant[we] = static_cast<uint8_t>(new_uqw);
				adjustments = true;
				for (int te = 0; te < cnt; te++) {
					int texel = (int)(s_wtc[off + te] & 0xFF);
					wb[texel] = bilinear_infill(di, uqf, texel);
				}
			}
		}
#else
		// The reference visits the weights in index order and a weight that moves changes the infill its grid neighbours see,
		// so the loop is sequential - but only about 1 weight in 7 moves at 6x6 -medium. So: evaluate EVERY
		// weight against the current state at once (group of four lanes = one weight, one lane per channel, each lane walking its
		// weight's texels in order - eight weights per pass), then replay the reference's order over the outcomes: the first
		// weight that wants to move moves; the only outcomes this can invalidate are those of its LATER grid neighbours
		// (x+1, y), (x-1, y+1), (x, y+1), (x+1, y+1) - weights further away share no texel with it - so exactly those are
		// evaluated again (four groups at once) before the scan goes on. Every weight is therefore decided on the state the
		// sequential loop would show it: same decisions, a handful of sequential steps instead of weight_count.
		// (3D block sizes: seven later neighbours, see below.)
		const DevDecMode* dmp = BSD.dec_modes + d;
		const int gw = ASTC_LDG(&dmp->weight_x);
		const bool volume = BSD.dim_z > 1;
		const int grp = w.lane >> 2;
		const int lc = w.lane & 3;
		const float ew_c = lane(ew, lc);
		SPtr<uint8_t> s_new = sptr<uint8_t>(rs.tile + 128 + 136 + tp + 8 * tp);   // [64] the value a weight wants to move to
		// decision of weight `we` on the current state; all 32 lanes call it (shuffles inside), act = group has a weight
		auto evaluate = [&](int we, bool act) -> int {
			int off = 0, cnt = 0, uqw = 0;
			float uqw_down = 0.0f, uqw_up = 0.0f, uqw_diff_down = 0.0f, uqw_diff_up = 0.0f;
			if (act) {
				uint32_t pn = s_pn[we];
				float uqw_base = uqf[we];
				uqw = (int)uqw_base;
				uqw_down = static_cast<float>(pn & 0xFF);
				uqw_up = static_cast<float>((pn >> 8) & 0xFF);
				uqw_diff_down = uqw_down - uqw_base;
				uqw_diff_up = uqw_up - uqw_base;
				off = s_wto[we];
				cnt = s_wto[we + 1] - off;
			}
			float sb = 0.0f, sd = 0.0f, su = 0.0f;
			ASTC_UNROLL_R2
			for (int te = 0; te < cnt; te++) {
				uint32_t e = s_wtc[off + te];
				int texel = (int)(e & 0xFF);
				float tw_base = static_cast<float>(e >> 8) * (1.0f / 16.0f);
				float weight_base = wb[texel];
				float weight_down = weight_base + uqw_diff_down * tw_base - weight_base;
				float weight_up = weight_base + uqw_diff_up * tw_base - weight_base;
				int pidx = s_pot[texel] * 4 + lc;
				float color_offset = eo[pidx];
				float color = eb[pidx] + color_offset * weight_base;
				float orig = sptr<float>(b0.off + (uint32_t)lc * cs)[texel];
				float color_diff = color - orig;
				float color_down_diff = color_diff + color_offset * weight_down;
				float color_up_diff = color_diff + color_offset * weight_up;
				sb = sb + color_diff * color_diff;
				sd = sd + color_down_diff * color_down_diff;
				su = su + color_up_diff * color_up_diff;
			}
			// dot with the channel weights: (x + z) + (y + w); fp addition commutes, so the four lanes get the same bits
			float vb = sb * ew_c, vd = sd * ew_c, vu = su * ew_c;
			vb = vb + __shfl_xor_sync(0xffffffffu, vb, 2);
			vd = vd + __shfl_xor_sync(0xffffffffu, vd, 2);
			vu = vu + __shfl_xor_sync(0xffffffffu, vu, 2);
			float error_base = vb + __shfl_xor_sync(0xffffffffu, vb, 1);
			float error_down = vd + __shfl_xor_sync(0xffffffffu, vd, 1);
			float error_up = vu + __shfl_xor_sync(0xffffffffu, vu, 1);
			int nv = -1;
			if (act) {
				if ((error_up < error_base) && (error_up < error_down) && (uqw < 64)) {
					nv = (int)uqw_up;
				} else if ((error_down < error_base) && (uqw > 0)) {
					nv = (int)uqw_down;
				}
			}
			return nv;
		};
		// pass 1: everybody against the state at entry; pending = the weights that want to move (bit we of a 64-bit set)
		uint32_t pend_lo = 0, pend_hi = 0;
		ASTC_NOUNROLL
		for (int we0 = 0; we0 < weight_count; we0 += 8) {
			int we = we0 + grp;
			bool act = we < weight_count;
			int nv = evaluate(we, act);
			if (act && lc == 0 && nv >= 0) {
				s_new[we] = (uint8_t)nv;
			}
			uint32_t m = __ballot_sync(0xffffffffu, act && lc == 0 && nv >= 0);
			// lane 4 g -> bit we0 + g
			uint32_t bits = (m & 1u) | ((m >> 3) & 2u) | ((m >> 6) & 4u) | ((m >> 9) & 8u) | ((m >> 12) & 16u) | ((m >> 15) & 32u) | ((m >> 18) & 64u) | ((m >> 21) & 128u);
			if (we0 < 32) pend_lo |= bits << we0;
			else pend_hi |= bits << (we0 - 32);
		}
		wsync();
		// pass 2: the reference's order over the outcomes.
		// Two ways to replay it. (a) Speculative: take the pending weights in index order; a move invalidates the outcomes of the
		// weight's later grid neighbours only, which are evaluated again. One sequential step per MOVE: cheap for the typical step
		// (~1 weight in 7 moves) but the tail is long - a noisy block moves most of its weights, and with one CTA-wide vote per
		// refinement round the slowest warp of 24 sets the pace.
		// (b) Wavefront: in a bilinear grid the earlier neighbours of (x, y) are (x-1, y), (x+1, y-1), (x, y-1), (x-1, y-1); with
		// k = x + 2 y they sit on fronts k-1, k-1, k-2, k-3, so the weights of one front are independent and all their earlier
		// neighbours are final: gw + 2 (gh - 1) sequential steps whatever the content (16 for a 6x6 grid), up to ceil(gw / 2) <= 8
		// weights per step, one group of four lanes each. Used when the pending set of pass 1 says (a) would take longer:
		// pending > fronts: 71.2 ms per pass against 74.4 ms with the wavefront never used (H100 80GB HBM3 at 400 W, 4K 6x6 -medium). (Computing the twelve
		// squared differences of a front's (weight, texel) pairs by one lane per pair into a tile and letting four lanes per weight
		// add the columns in order - less latency per front on paper - measured slower: more instructions, more barriers; removed.)
		const int npend = __popc(pend_lo) + __popc(pend_hi);
		const int gh = ASTC_LDG(&dmp->weight_y);
		const int nfronts = gw + 2 * (gh - 1);
		if (!volume && npend * ASTC_REALIGN_WAVE_DEN > nfronts * ASTC_REALIGN_WAVE_NUM) {
#if defined(ASTC_HOSTSIM)
			if (w.lane == 0) {
				g_hostsim_wavefront_replays++;      // (tests assert that their inputs reach this branch)
			}
#endif
			ASTC_NOUNROLL
			for (int k = 0; k < nfronts; k++) {
				int ylo = k - (gw - 1);
				ylo = ylo > 0 ? (ylo + 1) >> 1 : 0;
				int yhi = k >> 1;
				yhi = yhi < gh - 1 ? yhi : gh - 1;
				int y = ylo + grp;
				bool act = y <= yhi;
				int j = act ? y * gw + (k - 2 * y) : 0;
				int nv = evaluate(j, act);
				bool mv = act && nv >= 0;
				if (!wany(mv)) {
					continue;
				}
				adjustments = true;
				wsync();                   // (every group has read the state it decides on)
				int off = 0, cnt = 0;
				if (mv) {
					off = s_wto[j];
					cnt = s_wto[j + 1] - off;
					if (lc == 0) {
						uqf[j] = static_cast<float>(nv);
						dec_weights_uquant[j] = (uint8_t)nv;
					}
				}
				wsync();
				// the infill changes for the texels of the moved weights only (weights of one front share no texel)
				ASTC_NOUNROLL
				for (int te = lc; te < cnt; te += 4) {
					int texel = (int)(s_wtc[off + te] & 0xFF);
					wb[texel] = bilinear_infill(di, uqf, texel);
				}
				wsync();
			}
			continue;
		}
		ASTC_NOUNROLL
		while ((pend_lo | pend_hi) != 0) {
			int f = pend_lo != 0 ? __ffs((int)pend_lo) - 1 : 32 + __ffs((int)pend_hi) - 1;
			if (f < 32) pend_lo &= ~(1u << f);
			else pend_hi &= ~(1u << (f - 32));
			adjustments = true;
			int off = s_wto[f];
			int cnt = s_wto[f + 1] - off;
			float nvf = static_cast<float>(s_new[f]);
			wsync();                       // (everybody has read s_new[f] / the old state before lane 0 overwrites it)
			if (w.lane == 0) {
				uqf[f] = nvf;
				dec_weights_uquant[f] = (uint8_t)s_new[f];
			}
			wsync();
			// the infill changed for this weight's texels only
			ASTC_NOUNROLL
			for (int te = w.lane; te < cnt; te += ASTC_WARP) {
				int texel = (int)(s_wtc[off + te] & 0xFF);
				wb[texel] = bilinear_infill(di, uqf, texel);
			}
			wsync();
			// later grid neighbours of f: the weights of higher index that share a texel with it, one per group of four lanes.
			// 2D (bilinear cells): (fx+1, fy), (fx-1, fy+1), (fx, fy+1), (fx+1, fy+1). 3D (simplex cells: the corners of a texel's
			// simplex differ by vectors of {0,1}^3): the seven (fx+a, fy+b, fz+c), (a, b, c) != 0 - groups 0..6.
			int j;
			bool act;
			if (!volume) {
				int fy = f / gw;
				int fx = f - fy * gw;
				int dx = grp == 1 ? -1 : (grp == 2 ? 0 : 1);
				int dy = grp == 0 ? 0 : 1;
				int nx = fx + dx;
				j = f + dy * gw + dx;
				act = grp < 4 && nx >= 0 && nx < gw && j < weight_count;
			} else {
				const int gd = ASTC_LDG(&dmp->weight_z);
				const int gwh = gw * gh;
				int fz = f / gwh;
				int fr = f - fz * gwh;
				int fy = fr / gw;
				int fx = fr - fy * gw;
				int v = grp + 1;      // 1..7: bits = (dx, dy, dz)
				int dx = v & 1, dy = (v >> 1) & 1, dz = (v >> 2) & 1;
				j = f + dz * gwh + dy * gw + dx;
				act = grp < 7 && fx + dx < gw && fy + dy < gh && fz + dz < gd;
			}
			int nv = evaluate(j, act);
			if (act && lc == 0 && nv >= 0) {
				s_new[j] = (uint8_t)nv;
			}
			uint32_t redo = __ballot_sync(0xffffffffu, act && lc == 0);
			uint32_t want = __ballot_sync(0xffffffffu, act && lc == 0 && nv >= 0);
			// every lane folds the outcomes into its copy of the pending set (lane 4 g <-> neighbour g)
			if (!volume) {
				ASTC_NOUNROLL
				for (int g = 0; g < 4; g++) {
					if ((redo >> (4 * g)) & 1u) {
						int gdx = g == 1 ? -1 : (g == 2 ? 0 : 1);
						int jj = f + (g == 0 ? 0 : gw) + gdx;
						uint32_t on = (want >> (4 * g)) & 1u;
						if (jj < 32) pend_lo = (pend_lo & ~(1u << jj)) | (on << jj);
						else pend_hi = (pend_hi & ~(1u << (jj - 32))) | (on << (jj - 32));
					}
				}
			} else {
				ASTC_NOUNROLL
				while (redo != 0) {
					int l0 = __ffs((int)redo) - 1;
					redo &= redo - 1;
					int jj = __shfl_sync(0xffffffffu, j, l0);
					uint32_t on = (want >> l0) & 1u;
					if (jj < 32) pend_lo = (pend_lo & ~(1u << jj)) | (on << jj);
					else pend_hi = (pend_hi & ~(1u << (jj - 32))) | (on << (jj - 32));
				}
			}
			wsync();
		}
#endif
	}
	return wany(adjustments);
}
ASTC_COOP bool realign_weights(WCtx w, unsigned int pc, uint32_t formats, int plane2_component, const PartView& pi, int quant_mode, bool is_dual, unsigned int d) {
	return realign_weights_t<false>(w, pc, formats, plane2_component, pi, quant_mode, is_dual, d);
}

// =============================================================================================
// Physical block packing (astcenc_symbolic_physical.cpp:102-286, astcenc_integer_sequence.cpp:493-648).
// Pure bit twiddling on ~100 values: executed by lane 0.
// =============================================================================================
// The 128-bit block is assembled in two 64-bit registers; fields never overlap, so OR-ing a field in is
// equivalent to the reference's masked byte writes (symbolic_physical.cpp:63-85).
struct Bits128 {
	uint64_t lo, hi;
};

ASTC_FN void put_bits(Bits128& b, unsigned int value, unsigned int bitcount, unsigned int bitoffset) {
	uint64_t v = (uint64_t)(value & ((1u << bitcount) - 1u));
	if (bitoffset < 64) {
		b.lo |= v << bitoffset;
		if (bitoffset + bitcount > 64) {
			b.hi |= v >> (64 - bitoffset);
		}
	} else if (bitoffset < 128) {
		b.hi |= v << (bitoffset - 64);
	}
}

ASTC_FN uint64_t brev64(uint64_t v) {
#if defined(ASTC_HOSTSIM)
	v = ((v >> 1) & 0x5555555555555555ULL) | ((v & 0x5555555555555555ULL) << 1);
	v = ((v >> 2) & 0x3333333333333333ULL) | ((v & 0x3333333333333333ULL) << 2);
	v = ((v >> 4) & 0x0F0F0F0F0F0F0F0FULL) | ((v & 0x0F0F0F0F0F0F0F0FULL) << 4);
	v = ((v >> 8) & 0x00FF00FF00FF00FFULL) | ((v & 0x00FF00FF00FF00FFULL) << 8);
	v = ((v >> 16) & 0x0000FFFF0000FFFFULL) | ((v & 0x0000FFFF0000FFFFULL) << 16);
	return (v >> 32) | (v << 32);
#else
	return __brevll(v);
#endif
}

// Source of the values of one integer sequence: the block's weights (scrambled quantised values, planes
// interleaved for dual-plane modes :127-150) or its colour values (partition after partition :268-285).
struct IseSource {
	uint32_t arr;                    // shared offset of best_weights / best_colors
	const uint8_t* table;            // scramble map / uquant -> scrambled pquant
	float weight_quant_levels_m1;    // weights only
	int is_dual_plane;               // weights only
	int is_color;
	uint32_t n0, n1, n2;             // colours only: values in partitions 0, 1, 2
};

ASTC_NOINLINE unsigned int ise_value(const IseSource& s, unsigned int i, unsigned int count) {
	if (i >= count) {
		return 0u;
	}
	SPtr<uint8_t> a = sptr<uint8_t>(s.arr);
	if (!s.is_color) {
		unsigned int src = s.is_dual_plane ? ((i >> 1) + ((i & 1) ? 32u : 0u)) : i;
		float uqw = static_cast<float>(a[(int)src]);
		float qw = (uqw / 64.0f) * s.weight_quant_levels_m1;
		int qwi = static_cast<int>(qw + 0.5f);
		return ASTC_LDG(&s.table[qwi]);
	}
	unsigned int p = 0;
	if (i >= s.n0) { i -= s.n0; p = 1; if (i >= s.n1) { i -= s.n1; p = 2; if (i >= s.n2) { i -= s.n2; p = 3; } } }
	return ASTC_LDG(&s.table[a[(int)(p * 8 + i)]]);
}

// encode_ise (astcenc_integer_sequence.cpp:493-648)
ASTC_NOINLINE void encode_ise(int quant_level, unsigned int character_count, const IseSource& src, Bits128& out, unsigned int bit_offset) {
	const DevConstTables* ct = ASTC_CT;
	unsigned int bits, trits, quints;
	ise_btq(quant_level, bits, trits, quints);
	unsigned int mask = (1u << bits) - 1;
	if (trits) {
		// five values share one packed trit byte T; element j carries T bits [sh, sh + n): 2 2 1 2 1
		ASTC_NOUNROLL
		for (unsigned int i = 0; i < character_count; i += 5) {
			unsigned int v[5];
			unsigned int tr = 0;
			for (int j = 4; j >= 0; j--) {
				v[j] = ise_value(src, i + (unsigned int)j, character_count);
				tr = tr * 3 + (v[j] >> bits);
			}
			unsigned int T = ASTC_LDG(&ct->integer_of_trits[tr]);
			unsigned int sh = 0;
			for (int j = 0; j < 5; j++) {
				if (i + (unsigned int)j >= character_count) break;
				unsigned int n = (j == 2 || j == 4) ? 1u : 2u;
				put_bits(out, (v[j] & mask) | (((T >> sh) & ((1u << n) - 1)) << bits), bits + n, bit_offset);
				bit_offset += bits + n;
				sh += n;
			}
		}
	} else if (quints) {
		// three values share one packed quint byte Q; element j carries Q bits: 3 2 2
		ASTC_NOUNROLL
		for (unsigned int i = 0; i < character_count; i += 3) {
			unsigned int v[3];
			unsigned int qv = 0;
			for (int j = 2; j >= 0; j--) {
				v[j] = ise_value(src, i + (unsigned int)j, character_count);
				qv = qv * 5 + (v[j] >> bits);
			}
			unsigned int Q = ASTC_LDG(&ct->integer_of_quints[qv]);
			unsigned int sh = 0;
			for (int j = 0; j < 3; j++) {
				if (i + (unsigned int)j >= character_count) break;
				unsigned int n = j == 0 ? 3u : 2u;
				put_bits(out, (v[j] & mask) | (((Q >> sh) & ((1u << n) - 1)) << bits), bits + n, bit_offset);
				bit_offset += bits + n;
				sh += n;
			}
		}
	} else {
		ASTC_NOUNROLL
		for (unsigned int i = 0; i < character_count; i++) {
			put_bits(out, ise_value(src, i, character_count), bits, bit_offset);
			bit_offset += bits;
		}
	}
}

// Writes the 16 physical bytes of the best block (header scb, arrays in the arena's best_* slots) to out. Lane 0 only.
ASTC_NOINLINE void symbolic_to_physical(WCtx w, const ScbHdr& scb, uint8_t* out) {
	Bits128 pcb;
	pcb.lo = 0;
	pcb.hi = 0;
	if (scb.block_type == SYM_BTYPE_CONST_U16 || scb.block_type == SYM_BTYPE_CONST_F16) {
		// FC FD FF .. FF (UNORM16) or FC FF FF .. FF (FP16), then the four 16-bit components
		pcb.lo = scb.block_type == SYM_BTYPE_CONST_U16 ? 0xFFFFFFFFFFFFFDFCULL : 0xFFFFFFFFFFFFFFFCULL;
		pcb.hi = ((uint64_t)(scb.constant_color[0] & 0xFFFF)) | ((uint64_t)(scb.constant_color[1] & 0xFFFF) << 16) |
		         ((uint64_t)(scb.constant_color[2] & 0xFFFF) << 32) | ((uint64_t)(scb.constant_color[3] & 0xFFFF) << 48);
	} else {
		const DevConstTables* ct = ASTC_CT;
		unsigned int partition_count = scb.partition_count;
		const DevBlockMode* bm = BSD.block_modes + ASTC_LDG(&BSD.block_mode_packed_index[scb.block_mode]);
		int weight_count = ASTC_LDG(&BSD.dec_modes[ASTC_LDG(&bm->decimation_mode)].weight_count);
		int weight_quant_method = ASTC_LDG(&bm->quant_mode);
		int is_dual_plane = ASTC_LDG(&bm->is_dual_plane);
		int real_weight_count = is_dual_plane ? 2 * weight_count : weight_count;
		int bits_for_weights = (int)ise_sequence_bitcount((unsigned int)real_weight_count, weight_quant_method);
		IseSource ws;
		ws.arr = best_weights_of(w).off;
		ws.table = ct->wq_scramble_map[weight_quant_method];
		ws.weight_quant_levels_m1 = static_cast<float>(quant_level_count(weight_quant_method)) - 1.0f;
		ws.is_dual_plane = is_dual_plane;
		ws.is_color = 0;
		ws.n0 = ws.n1 = ws.n2 = 0;
		Bits128 wb;
		wb.lo = 0;
		wb.hi = 0;
		encode_ise(weight_quant_method, (unsigned int)real_weight_count, ws, wb, 0);
		// the weight stream is stored bit-reversed from the top of the block (:153-156)
		pcb.lo = brev64(wb.hi);
		pcb.hi = brev64(wb.lo);
		put_bits(pcb, scb.block_mode, 11, 0);
		put_bits(pcb, partition_count - 1, 2, 11);
		int below_weights_pos = 128 - bits_for_weights;
		if (partition_count > 1) {
			put_bits(pcb, scb.partition_index, 6, 13);
			put_bits(pcb, scb.partition_index >> 6, 10 - 6, 19);
			if (scb.color_formats_matched) {
				put_bits(pcb, (unsigned int)scb.color_formats[0] << 2, 6, 13 + 10);
			} else {
				int low_class = 4;
				for (unsigned int i = 0; i < partition_count; i++) {
					int class_of_format = scb.color_formats[i] >> 2;
					low_class = mini(class_of_format, low_class);
				}
				if (low_class == 3) {
					low_class = 2;
				}
				int encoded_type = low_class + 1;
				int bitpos = 2;
				for (unsigned int i = 0; i < partition_count; i++) {
					int classbit_of_format = (scb.color_formats[i] >> 2) - low_class;
					encoded_type |= classbit_of_format << bitpos;
					bitpos++;
				}
				for (unsigned int i = 0; i < partition_count; i++) {
					int lowbits_of_format = scb.color_formats[i] & 3;
					encoded_type |= lowbits_of_format << bitpos;
					bitpos += 2;
				}
				int encoded_type_lowpart = encoded_type & 0x3F;
				int encoded_type_highpart = encoded_type >> 6;
				int encoded_type_highpart_size = (3 * (int)partition_count) - 4;
				int encoded_type_highpart_pos = 128 - bits_for_weights - encoded_type_highpart_size;
				put_bits(pcb, (unsigned int)encoded_type_lowpart, 6, 13 + 10);
				put_bits(pcb, (unsigned int)encoded_type_highpart, (unsigned int)encoded_type_highpart_size, (unsigned int)encoded_type_highpart_pos);
				below_weights_pos -= encoded_type_highpart_size;
			}
		} else {
			put_bits(pcb, scb.color_formats[0], 4, 13);
		}
		if (is_dual_plane) {
			put_bits(pcb, (unsigned int)scb.plane2_component, 2, (unsigned int)(below_weights_pos - 2));
		}
		// colour values: partition after partition, 2 * (class + 1) values each (:268-285)
		IseSource cs;
		cs.arr = best_colors_of(w).off;
		cs.table = ct->color_uquant_to_scrambled_pquant[scb.quant_mode - QUANT_6];
		cs.weight_quant_levels_m1 = 0.0f;
		cs.is_dual_plane = 0;
		cs.is_color = 1;
		cs.n0 = 2u * (scb.color_formats[0] >> 2) + 2u;
		cs.n1 = partition_count > 1 ? 2u * (scb.color_formats[1] >> 2) + 2u : 0u;
		cs.n2 = partition_count > 2 ? 2u * (scb.color_formats[2] >> 2) + 2u : 0u;
		unsigned int n3 = partition_count > 3 ? 2u * (scb.color_formats[3] >> 2) + 2u : 0u;
		encode_ise(scb.quant_mode, cs.n0 + cs.n1 + cs.n2 + n3, cs, pcb, scb.partition_count == 1 ? 17 : 19 + 10);
	}
	uint32_t* o32 = reinterpret_cast<uint32_t*>(out);
	o32[0] = (uint32_t)pcb.lo;
	o32[1] = (uint32_t)(pcb.lo >> 32);
	o32[2] = (uint32_t)pcb.hi;
	o32[3] = (uint32_t)(pcb.hi >> 32);
}

#include "astc_dev_partition.cuh"
#include "astc_dev_driver.cuh"
#include "astc_dev_lockstep.cuh"
#include "astc_dev_alpha.cuh"
#include "astc_dev_wave.cuh"
#include "astc_dev_decode.cuh"
