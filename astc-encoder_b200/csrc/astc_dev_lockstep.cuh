// CUDA-native ASTC block compressor: the phase-aligned ("lockstep") CTA driver.
//
// Why: the block search is ~150 KB of hot, branchy code that every block walks once per trial. With each warp
// of an SM at a different point of it, nearly every instruction line is fetched from L2 again (the SM instruction cache
// misses, the instruction path to L2 saturates and the issue slots idle).
// When all warps of a CTA run the SAME stage at the same time - each on its own block - one fetch feeds all of
// them.
//
// How: every trial of astcenc_compress_symbolic.cpp has the same shape - ideal endpoints/weights, decimated weights,
// angular ranges, per-mode quantisation error, endpoint formats, then refinement steps (refit colours, pack,
// score, realign, score). The CTA walks that stage list round after round with a barrier in front of every stage;
// in each round every warp runs the next trial of ITS OWN block (1 plane / 2 planes / n partitions), and fetches
// a new block whenever its search has finished. The per-block decision tree (compress_block :1162-1455) is a
// small state machine advanced between rounds. Results are bit-identical to the per-warp driver.
#pragma once

ASTC_FN bool block_has_alpha(const WCtx& w, const float* averages, float threshold, unsigned int pos_x, unsigned int pos_y);

#if defined(ASTC_ONE_LANE)
ASTC_FN void cta_sync() {}
ASTC_FN bool cta_any(bool p) { return p; }
#else
ASTC_FN void cta_sync() { __syncthreads(); }
ASTC_FN bool cta_any(bool p) { return __syncthreads_or(p ? 1 : 0) != 0; }
#endif

// Progress and cancellation of an astcenc_compress_image pass: two device words per context, null when the pass has none.
// The cancel flag is written by a DMA from the host while the kernels run; one lane reads it (from L2) wherever a warp takes
// new work, and a raised flag looks exactly like an empty queue / exhausted ticket feed, so the warps leave through their usual
// exits. The done counter gets one add per block whose search has ended (its result is final).
#if defined(ASTC_HOSTSIM)
// (a harness may watch every look at the flag: tests/hostsim/hostsim_progress.cpp raises it after a number of pops)
static void (*g_hostsim_cancel_look)() = nullptr;
ASTC_FN bool pass_cancelled(const uint32_t* flag) {
	if (flag == nullptr) {
		return false;
	}
	if (g_hostsim_cancel_look != nullptr) {
		g_hostsim_cancel_look();
	}
	return *flag != 0;
}
ASTC_FN void pass_done_add(uint32_t* done) { if (done != nullptr) *done += 1u; }
#else
ASTC_FN bool pass_cancelled(const uint32_t* flag) { return flag != nullptr && __ldcg(flag) != 0u; }
ASTC_FN void pass_done_add(uint32_t* done) { if (done != nullptr) atomicAdd(done, 1u); }
#endif
// a block's search has ended (called by the whole warp)
ASTC_FN void pass_block_done(const WCtx& w, uint32_t* done) {
	if (w.lane == 0) {
		pass_done_add(done);
	}
}

// where the next block index comes from (device: a global ticket counter; host simulation: a plain counter)
struct BlockFeed {
	unsigned int* ticket;
	unsigned int total;
	unsigned int blocks_x;
	const uint32_t* cancel = ASTC_PASS_CANCEL_DEFAULT;      // raised: the feed is exhausted (may be null)
};

ASTC_FN bool feed_next(const WCtx& w, const BlockFeed& f, unsigned int& b) {
#if defined(ASTC_HOSTSIM) && defined(ASTC_ONE_LANE)
	b = pass_cancelled(f.cancel) ? 0xFFFFFFFFu : (*f.ticket)++;
#elif defined(ASTC_DEBUG_SINGLE_LANE)
	b = pass_cancelled(f.cancel) ? 0xFFFFFFFFu : atomicAdd(f.ticket, 1u);
#else
	unsigned int v = 0xFFFFFFFFu;
	if (w.lane == 0 && !pass_cancelled(f.cancel)) {
		v = atomicAdd(f.ticket, 1u);
	}
	b = __shfl_sync(0xffffffffu, v, 0);
#endif
	return b < f.total;
}

// Search state of the block a warp currently owns (compress_block's locals).
struct BlockSearch {
	ScbHdr scb;
	float error_threshold, errorval_overshoot;
	float best_pc1;                 // best_errorvals_for_pcount[0]
	float best_error_in_prev;       // best error of the previous partition count
	float best_error_cur;           // best error of the current partition count
	int quant_limit;
	int phase;                      // 0: 1 partition 1 plane, 1: 2 planes, 2: 2..4 partitions, 3: finished
	int idx;                        // trial index inside the phase
	int pc;                         // partition count (phase 2)
	unsigned int actual_trials;     // phase 2
	bool phase_entered;
	bool skip_two_plane;
	unsigned int out_index;
};

// The trial a warp runs in the current round.
struct Trial {
	int dual;                       // 0: 1 plane, 1: 2 planes
	int only_always;
	unsigned int partition_count, partition_index, packed;
	int plane2_component;
	float tune_errorval_threshold;
	float done_threshold;           // errorval below this finishes the block
	int max_weight_quant;
	float cutoff1, cutoff2;
	unsigned int start_mode, end_mode;
	unsigned int candidate_count;
	unsigned int candidate_count_next;   // wave pipeline: candidates already selected for the following trial (A_CAND2), 0 = none
};

ASTC_FN SPtr<uint16_t> partition_list_of(const WCtx& w) { return sptr<uint16_t>(w.base + A_STATE + (uint32_t)offsetof(BlkInfo, partition_list)); }

// THE SEARCH STATE (BlockSearch, Trial, Refine) EXISTS ONCE PER WARP, IN SHARED MEMORY (as per-lane automatic variables the
// three structs were 32 copies per warp in local memory). The discipline that makes this independent of how the lanes of a
// warp are scheduled: lanes READ the state into registers; a __syncwarp() separates the last read from the next write;
// LANE 0 ALONE WRITES; a __syncwarp() publishes the write before anybody reads again. Scalar bookkeeping that only the
// state itself needs (the decision tree) runs on lane 0 in place and its verdict is broadcast with a shuffle.
#define ST_WRITE_BEGIN(w) wsync(); if ((w).lane == 0) {
#define ST_WRITE_END(w) } wsync();

ASTC_FN void block_search_begin(const WCtx& w, BlockSearch& s, unsigned int out_index) {
	ST_WRITE_BEGIN(w)
		const BlkInfo& bi = bi_of(w);
		s.scb.block_type = SYM_BTYPE_ERROR;
		s.scb.partition_count = 0;
		s.scb.color_formats_matched = 0;
		s.scb.plane2_component = -1;
		s.scb.block_mode = 0;
		s.scb.partition_index = 0;
		s.scb.color_formats[0] = s.scb.color_formats[1] = s.scb.color_formats[2] = s.scb.color_formats[3] = 0;
		s.scb.quant_mode = 0;
		s.scb.errorval = ERROR_CALC_DEFAULT;
		s.scb.constant_color[0] = s.scb.constant_color[1] = s.scb.constant_color[2] = s.scb.constant_color[3] = 0;
		bool block_is_l = is_luminance(w);
		float block_is_l_scale = block_is_l ? 1.0f / 1.5f : 1.0f;
		bool block_is_la = is_luminancealpha(w);
		float block_is_la_scale = block_is_la ? 1.0f / 1.05f : 1.0f;
		float error_weight_sum = hadd_s(bi.channel_weight) * BSD.texel_count;
		s.error_threshold = CFG.tune_db_limit * error_weight_sum * block_is_l_scale * block_is_la_scale;
		s.errorval_overshoot = 1.0f / CFG.tune_mse_overshoot;
		s.best_pc1 = ERROR_CALC_DEFAULT;
		s.best_error_in_prev = ERROR_CALC_DEFAULT;
		s.best_error_cur = ERROR_CALC_DEFAULT;
		s.quant_limit = QUANT_32;
		s.phase = 0;
		s.idx = (CFG.tune_search_mode0_enable >= 0.85f && BSD.dim_z == 1) ? 0 : 1;      // (compress_symbolic.cpp:1287: no mode-0 trial for 3D block sizes)
		s.pc = 2;
		s.actual_trials = 0;
		s.phase_entered = false;
		s.skip_two_plane = false;
		s.out_index = out_index;
	ST_WRITE_END(w)
}

// Pick the next trial of the block (compress_block :1236-1443 unrolled into a state machine).
//   NEXT_TRIAL    : t describes the trial to run
//   NEXT_PREPARE  : the phase just entered needs the block statistics (2 planes) or the partition search first
//   NEXT_FINISHED : the search is over
enum { NEXT_TRIAL = 0, NEXT_PREPARE = 1, NEXT_FINISHED = 2 };

ASTC_FN int block_search_advance_on(const WCtx& w, BlockSearch& s, Trial& t) {
	const BlkInfo& bi = bi_of(w);
	while (true) {
		if (s.phase == 0) {
			if (s.idx < 2) {
				float mult = s.idx == 0 ? 1.0f / CFG.tune_mse_overshoot : 1.0f;       // errorval_mult[i]
				t.dual = 0;
				t.only_always = s.idx == 0;
				t.partition_count = 1;
				t.partition_index = 0;
				t.packed = 0;
				t.plane2_component = -1;
				t.tune_errorval_threshold = s.error_threshold * mult * s.errorval_overshoot;
				t.done_threshold = s.error_threshold * mult;
				t.max_weight_quant = (int)QUANT_32;
				return NEXT_TRIAL;
			}
			s.phase = 1;
			s.idx = 3;
			s.phase_entered = false;
			continue;
		}
		if (s.phase == 1) {
			if (!s.phase_entered) {
				return NEXT_PREPARE;
			}
			bool found = false;
			while (s.idx >= 0) {
				int i = s.idx;
				if (s.skip_two_plane || (bi.grayscale && i != 3) || is_constant_channel(w, i)) {
					s.idx--;
					continue;
				}
				found = true;
				break;
			}
			if (found) {
				t.dual = 1;
				t.only_always = 0;
				t.partition_count = 1;
				t.partition_index = 0;
				t.packed = 0;
				t.plane2_component = s.idx;
				t.tune_errorval_threshold = s.error_threshold * s.errorval_overshoot;
				t.done_threshold = s.error_threshold;
				t.max_weight_quant = mini((int)QUANT_32, s.quant_limit);
				return NEXT_TRIAL;
			}
			s.phase = 2;
			s.pc = 2;
			s.phase_entered = false;
			s.best_error_in_prev = s.best_pc1;
			continue;
		}
		if (s.phase == 2) {
			if (s.pc > (int)CFG.tune_partition_count_limit) {
				s.phase = 3;
				continue;
			}
			if (!s.phase_entered) {
				return NEXT_PREPARE;
			}
			if ((unsigned int)s.idx < s.actual_trials) {
				t.dual = 0;
				t.only_always = 0;
				t.partition_count = (unsigned int)s.pc;
				t.partition_index = partition_list_of(w)[s.idx];
				t.packed = part_packed_index(t.partition_count, t.partition_index);
				t.plane2_component = -1;
				t.tune_errorval_threshold = s.error_threshold * s.errorval_overshoot;
				t.done_threshold = s.error_threshold;
				t.max_weight_quant = mini((int)QUANT_32, s.quant_limit);
				return NEXT_TRIAL;
			}
			// all trials of this partition count done (:1434-1441)
			float exit_threshold = s.pc == 2 ? CFG.tune_2partition_early_out_limit_factor : s.pc == 3 ? CFG.tune_3partition_early_out_limit_factor : 0.0f;
			if (s.best_error_cur > (s.best_error_in_prev * exit_threshold)) {
				s.phase = 3;
				continue;
			}
			s.best_error_in_prev = s.best_error_cur;
			s.pc++;
			s.phase_entered = false;
			continue;
		}
		return NEXT_FINISHED;
	}
}

// The decision tree runs on lane 0, in place on the shared state; every lane gets the verdict.
ASTC_FN int block_search_advance(const WCtx& w, BlockSearch& s, Trial& t) {
	int next = 0;
	wsync();
	if (w.lane == 0) {
		next = block_search_advance_on(w, s, t);
	}
	next = (int)wbroadcast0(w, (uint32_t)next);
	wsync();
	return next;
}

// The work a phase needs before its first trial: block statistics (2 planes, :1283-1289) or the partition search
// of the current partition count (:1341-1360).
ASTC_COOP void block_search_prepare(WCtx w, BlockSearch& s) {
	int phase = s.phase;
	int pc = s.pc;
	if (phase == 1) {
		float lowest_correl = prepare_block_statistics(w);
		ST_WRITE_BEGIN(w)
			s.skip_two_plane = lowest_correl > CFG.tune_2plane_early_out_limit_correlation;
			s.phase_entered = true;
		ST_WRITE_END(w)
		return;
	}
	unsigned int partition_indices[8];
	unsigned int requested_indices = CFG.tune_partition_index_limit[pc - 2];
	unsigned int requested_trials = CFG.tune_partitioning_candidate_limit[pc - 2];
	requested_trials = requested_trials < requested_indices ? requested_trials : requested_indices;
	unsigned int actual_trials = find_best_partition_candidates(w, (unsigned int)pc, requested_indices, partition_indices, requested_trials);
	SPtr<uint16_t> pl = partition_list_of(w);
	ST_WRITE_BEGIN(w)
		for (unsigned int k = 0; k < 8; k++) {
			if (k < actual_trials) {
				pl[(int)k] = (uint16_t)partition_indices[k];
			}
		}
		s.actual_trials = actual_trials;
		s.best_error_cur = ERROR_CALC_DEFAULT;
		s.idx = 0;
		s.phase_entered = true;
	ST_WRITE_END(w)
}

ASTC_COOP bool block_search_next(WCtx w, BlockSearch& s, Trial& t) {
	while (true) {
		int k = block_search_advance(w, s, t);
		if (k == NEXT_PREPARE) {
			block_search_prepare(w, s);
			continue;
		}
		return k == NEXT_TRIAL;
	}
}

// Book-keeping after a trial returned errorval (= best_errorval_in_mode of the trial).
ASTC_FN void block_search_after_trial_on(const WCtx& w, BlockSearch& s, const Trial& t, float errorval) {
	if (s.phase == 0) {
		if (s.scb.block_type != SYM_BTYPE_ERROR) {
			s.quant_limit = ASTC_LDG(&BSD.block_modes[ASTC_LDG(&BSD.block_mode_packed_index[s.scb.block_mode])].quant_mode);
		}
		s.best_pc1 = minf(s.best_pc1, errorval);
		if (errorval < t.done_threshold) {
			s.phase = 3;
		}
		s.idx++;
	} else if (s.phase == 1) {
		if (errorval > (s.best_pc1 * 1.85f)) {
			s.phase = 2;                 // break out of the 2-plane loop
			s.pc = 2;
			s.phase_entered = false;
			s.best_error_in_prev = s.best_pc1;
		} else if (errorval < t.done_threshold) {
			s.phase = 3;
		} else {
			s.idx--;
		}
	} else {
		s.best_error_cur = minf(s.best_error_cur, errorval);
		float exit_threshold = s.pc == 2 ? CFG.tune_2partition_early_out_limit_factor : s.pc == 3 ? CFG.tune_3partition_early_out_limit_factor : 0.0f;
		float best_error_scale = exit_threshold * 1.85f;
		if (s.best_error_cur > (s.best_error_in_prev * best_error_scale)) {
			s.phase = 3;
		} else if (errorval < t.done_threshold) {
			s.phase = 3;
		} else {
			s.idx++;
		}
	}
}
ASTC_FN void block_search_after_trial(const WCtx& w, BlockSearch& s, const Trial& t, float errorval) {
	ST_WRITE_BEGIN(w)
		block_search_after_trial_on(w, s, t, errorval);
	ST_WRITE_END(w)
}

ASTC_FN void emit_block(const WCtx& w, BlockSearch& s) {
	ST_WRITE_BEGIN(w)
		if (s.scb.block_type == SYM_BTYPE_ERROR) {
			constant_color_u16(w, s.scb);
		}
		symbolic_to_physical(w, s.scb, IMG.out + (size_t)s.out_index * 16);
	ST_WRITE_END(w)
}

// Constant-colour blocks never enter the search (compress_block :1176-1222). Returns true when the block was emitted.
ASTC_FN bool emit_if_constant(const WCtx& w, unsigned int out_index) {
	const BlkInfo& bi = bi_of(w);
	f4 dmn = bi.data_min, dmx = bi.data_max;
	if (!(dmn.x == dmx.x && dmn.y == dmx.y && dmn.z == dmx.z && dmn.w == dmx.w)) {
		return false;
	}
	ScbHdr scb;
	scb.partition_count = 0;
	scb.color_formats_matched = 0;
	scb.plane2_component = -1;
	scb.block_mode = 0;
	scb.partition_index = 0;
	scb.color_formats[0] = scb.color_formats[1] = scb.color_formats[2] = scb.color_formats[3] = 0;
	scb.quant_mode = 0;
	scb.errorval = 0.0f;
	int decode_mode = CFG.profile;
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
		symbolic_to_physical(w, scb, IMG.out + (size_t)out_index * 16);
	}
	wsync();
	return true;
}

// ---- trial stages (compress_symbolic_block_for_partition_1plane :353-712 / _2planes :715-1044) ----
// Each stage exists in two instantiations of the same source. S1 = false: the general stage, an out-of-line function that reads
// the trial's shape (partitions, planes, HDR endpoints) at run time. S1 = true: the trial has one partition and one plane in an
// LDR profile - compile-time facts; the wave-0 set-up inlines this instantiation with the two-plane, n-partition and HDR
// branches folded away.
template <bool S1> ASTC_FN void stage_ideal_t(const WCtx& w, const Trial& t) {
	if (S1) {
		compute_ideal_colors_and_weights_1plane_t<true>(w, part_view_packed(1, 0));
	} else if (t.dual) {
		compute_ideal_colors_and_weights_2planes(w, (unsigned int)t.plane2_component);
	} else {
		PartView pi = part_view_packed(t.partition_count, t.packed);
		compute_ideal_colors_and_weights_1plane(w, pi);
	}
}
ASTC_COOP void stage_ideal(WCtx w, const Trial& t) {
	stage_ideal_t<false>(w, t);
}

template <bool S1> ASTC_FN void stage_decimate_t(const WCtx& w, const Trial& t) {
	unsigned int ndm = ((S1 || !t.dual) && t.only_always) ? BSD.decimation_mode_count_always : BSD.decimation_mode_count_selected;
	uint16_t refmask = (uint16_t)((1u << (t.max_weight_quant + 1)) - 1);
	// (one grid after the other: a single pass over the weights of all grids through a slot map was measured slower - the
	//  per-slot table look-ups cost more than the fuller warps gain)
	ASTC_NOUNROLL
	for (unsigned int i = 0; i < ndm; i++) {
		uint16_t ref = (!S1 && t.dual) ? ASTC_LDG(&BSD.dec_modes[i].refprec_2planes) : ASTC_LDG(&BSD.dec_modes[i].refprec_1plane);
		if ((ref & refmask) == 0) {
			continue;
		}
		if (S1) {
			compute_ideal_weights_for_decimation_t<true>(w, i, 1);
		} else {
			compute_ideal_weights_for_decimation(w, i, t.dual ? 2 : 1);
		}
	}
}
ASTC_COOP void stage_decimate(WCtx w, const Trial& t) {
	stage_decimate_t<false>(w, t);
}

// weight cut-offs (:430-432 / :791-798) and the block-mode range of the trial
ASTC_FN void trial_cutoffs(const WCtx& w, Trial& t) {
	SPtr<f4> ep = ep_of(w);
	int dual = t.dual, only_always = t.only_always, plane2_component = t.plane2_component;
	unsigned int partition_count = t.partition_count;
	float cutoff1, cutoff2;
	unsigned int start_mode, end_mode;
	if (!dual) {
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
		cutoff1 = hmin_s(min_ep);
		cutoff2 = cutoff1;
		start_mode = 0;
		end_mode = only_always ? BSD.block_mode_count_1plane_always : BSD.block_mode_count_1plane_selected;
	} else {
		f4 a0 = ep[EP_EI1_0], a1 = ep[EP_EI1_1], b0 = ep[EP_EI2_0], b1 = ep[EP_EI2_1];
		f4 min_ep1 = mk4(min_ep_cutoff(a0.x, a1.x, 10.0f), min_ep_cutoff(a0.y, a1.y, 10.0f), min_ep_cutoff(a0.z, a1.z, 10.0f), min_ep_cutoff(a0.w, a1.w, 10.0f));
		f4 min_ep2 = mk4(min_ep_cutoff(b0.x, b1.x, 10.0f), min_ep_cutoff(b0.y, b1.y, 10.0f), min_ep_cutoff(b0.z, b1.z, 10.0f), min_ep_cutoff(b0.w, b1.w, 10.0f));
		f4 m1 = min_ep1;
		set_lane(m1, plane2_component, ERROR_CALC_DEFAULT);
		cutoff1 = hmin_s(m1);
		f4 m2 = splat4(ERROR_CALC_DEFAULT);
		set_lane(m2, plane2_component, lane(min_ep2, plane2_component));
		cutoff2 = hmin_s(m2);
		start_mode = BSD.block_mode_count_1plane_selected;
		end_mode = BSD.block_mode_count_1plane_2plane_selected;
	}
	ST_WRITE_BEGIN(w)
		t.cutoff1 = cutoff1;
		t.cutoff2 = cutoff2;
		t.start_mode = start_mode;
		t.end_mode = end_mode;
	ST_WRITE_END(w)
}

template <bool S1> ASTC_FN void stage_formats_t(const WCtx& w, Trial& t) {
	SPtr<f4> ep = ep_of(w);
	unsigned int count;
	if (S1) {
		PartView pi = part_view_packed(1, 0);
		endpoint_formats_prepare_t<true>(w, pi, EP_EI1_0, EP_EI1_1, 1, t.start_mode, t.end_mode);
		count = endpoint_formats_select_t<true>(w, 1, 1, t.start_mode, t.end_mode, w.base + A_CAND, false);
		ASTC_NOUNROLL
		for (int k = w.lane; k < 4; k += ASTC_WARP) {
			ep[EP_BASE_0 + k] = ep[EP_EI1_0 + k];
			ep[EP_BASE_1 + k] = ep[EP_EI1_1 + k];
		}
	} else if (!t.dual) {
		PartView pi = part_view_packed(t.partition_count, t.packed);
		count = compute_ideal_endpoint_formats(w, pi, EP_EI1_0, EP_EI1_1, 1, t.start_mode, t.end_mode);
		ASTC_NOUNROLL
		for (int k = w.lane; k < 4; k += ASTC_WARP) {
			ep[EP_BASE_0 + k] = ep[EP_EI1_0 + k];
			ep[EP_BASE_1 + k] = ep[EP_EI1_1 + k];
		}
	} else {
		// merge_endpoints :37-66
		int plane2_component = t.plane2_component;
		f4 a0 = ep[EP_EI1_0], a1 = ep[EP_EI1_1], b0 = ep[EP_EI2_0], b1 = ep[EP_EI2_1];
		f4 epm0 = a0, epm1 = a1;
		set_lane(epm0, plane2_component, lane(b0, plane2_component));
		set_lane(epm1, plane2_component, lane(b1, plane2_component));
		wsync();
		if (w.lane == 0) {
			ep[EP_BASE_0] = epm0;
			ep[EP_BASE_1] = epm1;
		}
		wsync();
		PartView pi = part_view_packed(1, 0);
		count = compute_ideal_endpoint_formats(w, pi, EP_BASE_0, EP_BASE_1, 2, t.start_mode, t.end_mode);
	}
	ST_WRITE_BEGIN(w)
		t.candidate_count = count;
	ST_WRITE_END(w)
}
ASTC_COOP void stage_formats(WCtx w, Trial& t) {
	stage_formats_t<false>(w, t);
}

// Refinement state of the candidate a warp is working on (the loop nest of :504-699 / :886-1044 flattened into steps).
struct Refine {
	unsigned int i, l;              // candidate, refinement iteration
	bool running;                   // more steps to do in this trial
	bool in_step;                   // still inside the current step (no early break yet)
	float best_errorval_in_mode, best_errorval_in_scb;
	ScbHdr work;
	uint32_t formats, cd_formats;
	int dmode, qmode, quant_level, quant_level_mod;
	uint16_t mode_index;
	bool adjustments;
	bool from_candw;                // candidate weights were quantised by the setup kernel (A_CANDW) instead of being derived here
};

// a trial begins: no candidate refined yet
ASTC_FN void refine_begin_trial(const WCtx& w, const Trial& t, Refine& r, const BlockSearch& s, bool from_candw) {
	unsigned int candidate_count = t.candidate_count;
	float scb_errorval = s.scb.errorval;
	ST_WRITE_BEGIN(w)
		r.i = 0;
		r.l = 0;
		r.running = candidate_count > 0;
		r.in_step = false;
		r.best_errorval_in_mode = ERROR_CALC_DEFAULT;
		r.best_errorval_in_scb = scb_errorval;
		r.adjustments = false;
		r.from_candw = from_candw;
	ST_WRITE_END(w)
}

// The refinement step exists in two instantiations of the same source. L1 = false: the general step, every part an
// out-of-line function that reads the trial's shape (partitions, planes, HDR formats) at run time. L1 = true: the trial has
// one partition, one plane and an LDR profile (so LDR endpoint formats) - compile-time facts, and every part of the step is
// inlined into its caller with the two-plane, n-partition and HDR branches folded away.

// start candidate r.i (quantise its weights, reset the work endpoints): the part of the candidate loop before `for l`
template <bool L1> ASTC_FN void refine_begin_candidate_t(const WCtx& w, const Trial& t, Refine& r) {
	unsigned int ci = r.i;
	bool from_candw = r.from_candw;
	Candidate cd = cand_of(w)[(int)ci];
	const DevBlockMode* qw_bm = BSD.block_modes + cd.block_mode;
	int dmode = ASTC_LDG(&qw_bm->decimation_mode);
	int qmode = ASTC_LDG(&qw_bm->quant_mode);
	uint16_t mode_index = ASTC_LDG(&qw_bm->mode_index);
	if (from_candw) {
		SPtr<uint32_t> ww = sptr<uint32_t>(work_weights_of(w).off);
		SPtr<uint32_t> cw = sptr<uint32_t>(w.base + A_CANDW + ci * 64u);
		ASTC_NOUNROLL
		for (int k = w.lane; k < 16; k += ASTC_WARP) {
			ww[k] = cw[k];
		}
	} else if (L1) {
		quantize_candidate_weights_t(w, dmode, qmode, 1, t.cutoff1, t.cutoff2);
	} else {
		quantize_candidate_weights(w, dmode, qmode, t.dual ? 2 : 1, t.cutoff1, t.cutoff2);
	}
	SPtr<f4> ep = ep_of(w);
	ASTC_NOUNROLL
	for (int k = w.lane; k < 4; k += ASTC_WARP) {
		ep[EP_WORK_0 + k] = ep[EP_BASE_0 + k];
		ep[EP_WORK_1 + k] = ep[EP_BASE_1 + k];
		ep[EP_RGBS + k] = splat4(0.0f);
		ep[EP_RGBO + k] = splat4(0.0f);
	}
	SPtr<uint32_t> wc32 = sptr<uint32_t>(work_colors_of(w).off);
	ASTC_NOUNROLL
	for (int k = w.lane; k < 8; k += ASTC_WARP) {
		wc32[k] = 0;
	}
	ST_WRITE_BEGIN(w)
		r.dmode = dmode;
		r.qmode = qmode;
		r.mode_index = mode_index;
		r.quant_level = cd.quant_level;
		r.quant_level_mod = cd.quant_level_mod;
		r.cd_formats = (uint32_t)cd.formats[0] | ((uint32_t)cd.formats[1] << 8) | ((uint32_t)cd.formats[2] << 16) | ((uint32_t)cd.formats[3] << 24);
		r.work.errorval = 0.0f;
		r.work.color_formats[0] = r.work.color_formats[1] = r.work.color_formats[2] = r.work.color_formats[3] = 0;
		r.work.constant_color[0] = r.work.constant_color[1] = r.work.constant_color[2] = r.work.constant_color[3] = 0;
	ST_WRITE_END(w)
}
ASTC_COOP void refine_begin_candidate(WCtx w, const Trial& t, Refine& r) {
	refine_begin_candidate_t<false>(w, t, r);
}

// the trial's partitioning (L1: the single partition)
template <bool L1> ASTC_FN PartView refine_part_view(const Trial& t) {
	return L1 ? part_view_packed(1, 0) : part_view_packed(t.partition_count, t.packed);
}

// step part 1: refit the endpoint colours
template <bool L1> ASTC_FN void refine_recompute_t(const WCtx& w, const Trial& t, Refine& r) {
	bool first = r.l == 0;
	ST_WRITE_BEGIN(w)
		r.in_step = true;
	ST_WRITE_END(w)
	if (first) {
		if (L1) {
			refine_begin_candidate_t<true>(w, t, r);
		} else {
			refine_begin_candidate(w, t, r);
		}
	}
	if (!L1 && t.dual) {
		recompute_ideal_colors_2planes(w, (unsigned int)r.dmode, t.plane2_component);
	} else if (L1) {
		recompute_ideal_colors_1plane_t<true>(w, refine_part_view<true>(t), (unsigned int)r.dmode);
	} else {
		PartView pi = part_view_packed(t.partition_count, t.packed);
		recompute_ideal_colors_1plane(w, pi, (unsigned int)r.dmode);
	}
}
ASTC_COOP void refine_recompute(WCtx w, const Trial& t, Refine& r) {
	refine_recompute_t<false>(w, t, r);
}

// step part 2: quantise the endpoints (with the matched-format retry of :560-601)
template <bool L1> ASTC_FN void refine_pack_t(const WCtx& w, const Trial& t, Refine& r) {
	uint32_t cd_formats = r.cd_formats;
	int quant_level = r.quant_level, quant_level_mod = r.quant_level_mod;
	uint16_t mode_index = r.mode_index;
	int dual = L1 ? 0 : t.dual;
	unsigned int partition_count = L1 ? 1u : (dual ? 1u : t.partition_count);
	unsigned int partition_index = L1 ? 0u : (dual ? 0u : t.partition_index);
	int plane2_component = dual ? t.plane2_component : -1;      // (L1: folds to -1)
	uint32_t formats;
	int matched = 0;
	if (dual) {
		formats = pack_work_endpoints(w, 1, cd_formats, quant_level, work_colors_of(w).off);
		formats &= 0xFF;
	} else {
		formats = L1 ? pack_work_endpoints_t<true>(w, 1, cd_formats, quant_level, work_colors_of(w).off)
		             : pack_work_endpoints(w, partition_count, cd_formats, quant_level, work_colors_of(w).off);
		bool all_same = quant_level != quant_level_mod;
		for (unsigned int j = 1; j < 4; j++) {
			if (j < partition_count) {
				all_same = all_same && ((formats >> (8 * j)) & 0xFF) == (formats & 0xFF);
			}
		}
		if (partition_count >= 2 && all_same) {
			SPtr<uint32_t> wc32 = sptr<uint32_t>(work_colors_of(w).off);
			SPtr<uint32_t> mc32 = sptr<uint32_t>(mod_colors_of(w).off);
			ASTC_NOUNROLL
			for (int k = w.lane; k < 8; k += ASTC_WARP) {
				mc32[k] = 0;
			}
			wsync();
			// (the reference stops packing at the first format mismatch; the later partitions' values are then unused)
			uint32_t formats_mod = pack_work_endpoints(w, partition_count, cd_formats, quant_level_mod, mod_colors_of(w).off);
			bool all_same_mod = true;
			for (unsigned int j = 1; j < 4; j++) {
				if (j < partition_count) {
					all_same_mod = all_same_mod && ((formats_mod >> (8 * j)) & 0xFF) == (formats_mod & 0xFF);
				}
			}
			if (all_same_mod) {
				matched = 1;
				ASTC_NOUNROLL
				for (int k = w.lane; k < 8; k += ASTC_WARP) {
					wc32[k] = mc32[k];
				}
				formats = formats_mod;
				wsync();
			}
		}
	}
	ST_WRITE_BEGIN(w)
		ScbHdr& work = r.work;
		work.partition_count = static_cast<uint8_t>(partition_count);
		work.partition_index = static_cast<uint16_t>(partition_index);
		work.plane2_component = static_cast<int8_t>(plane2_component);
		work.color_formats_matched = static_cast<uint8_t>(matched);
		work.quant_mode = (uint8_t)(matched ? quant_level_mod : quant_level);
		set_formats(work, formats);
		work.block_mode = mode_index;
		work.block_type = SYM_BTYPE_NONCONST;
		r.formats = formats;
	ST_WRITE_END(w)
	// integer endpoints of the packed candidate, once per step: both scores and the realignment read them
	if (L1) {
		unpack_work_endpoints_t<true>(w, 1, formats, ends_off_of(w));
	} else {
		unpack_work_endpoints(w, partition_count, formats, ends_off_of(w));
	}
}
ASTC_COOP void refine_pack(WCtx w, const Trial& t, Refine& r) {
	refine_pack_t<false>(w, t, r);
}

template <bool L1> ASTC_FN float refine_score(const WCtx& w, const Trial& t, const Refine& r) {
	PartView pi = refine_part_view<L1>(t);
	if (L1) {
		return compute_symbolic_block_difference_t<true>(w, 1, r.formats, -1, pi, (unsigned int)r.dmode, false);
	}
	return compute_symbolic_block_difference(w, t.partition_count, r.formats, t.plane2_component, pi, (unsigned int)r.dmode, t.dual != 0);
}

// What a score does to the candidate loop. The flags are computed by every lane from registers; the state changes
// they imply are written by lane 0 in one go (refine_apply).
enum { RF_KEEP = 0, RF_NEXT_CANDIDATE = 1, RF_STOP_ALL = 2, RF_NEXT_ITERATION = 3 };

// advance to the next candidate / the next refinement iteration / finish the trial
template <bool L1> ASTC_FN void refine_apply(const WCtx& w, const Trial& t, Refine& r, BlockSearch& s, int action, bool error_block, float best_in_mode, bool new_best, float errorval) {
	unsigned int i = r.i, l = r.l;
	unsigned int candidate_count = t.candidate_count;
	ST_WRITE_BEGIN(w)
		if (error_block) {
			r.work.block_type = SYM_BTYPE_ERROR;
		}
		r.best_errorval_in_mode = best_in_mode;
		if (new_best) {
			r.best_errorval_in_scb = errorval;
			r.work.errorval = errorval;
			s.scb = r.work;
		}
		if (action == RF_NEXT_CANDIDATE || action == RF_STOP_ALL) {
			i = action == RF_STOP_ALL ? candidate_count : i + 1;
			r.in_step = false;
			r.l = 0;
			r.i = i;
			if (i >= candidate_count) {
				r.running = false;
			}
		} else if (action == RF_NEXT_ITERATION) {
			r.l = l + 1;
			r.in_step = false;
		}
	ST_WRITE_END(w)
	if (new_best) {
		if (L1) {
			copy_work_to_best_t(w);
		} else {
			copy_work_to_best(w);
		}
	}
}

// step part 3 (first iteration of a candidate only): score before realignment (:606-640)
template <bool L1> ASTC_FN void refine_first_score_t(const WCtx& w, const Trial& t, Refine& r, BlockSearch& s) {
	float errorval = refine_score<L1>(w, t, r);
	float best_in_mode = r.best_errorval_in_mode, best_in_scb = r.best_errorval_in_scb;
	unsigned int l = r.l;
	bool error_block = false;
	if (errorval == -ERROR_CALC_DEFAULT) {
		errorval = -errorval;
		error_block = true;
	}
	best_in_mode = minf(errorval, best_in_mode);
	unsigned int iters_remaining = CFG.tune_refinement_limit - l;
	float threshold = (0.045f * static_cast<float>(iters_remaining)) + 1.08f;
	int action = RF_KEEP;
	bool new_best = false;
	if (errorval > (threshold * best_in_scb)) {
		action = RF_NEXT_CANDIDATE;
	} else if (errorval < best_in_scb) {
		new_best = true;
		if (errorval < t.tune_errorval_threshold) {
			action = RF_STOP_ALL;
		}
	}
	refine_apply<L1>(w, t, r, s, action, error_block, best_in_mode, new_best, errorval);
}
ASTC_FN void refine_first_score(const WCtx& w, const Trial& t, Refine& r, BlockSearch& s) {
	refine_first_score_t<false>(w, t, r, s);
}

// step part 5: score after realignment and decide how to go on (:642-698)
template <bool L1> ASTC_FN void refine_second_score_t(const WCtx& w, const Trial& t, Refine& r, BlockSearch& s) {
	float errorval = ERROR_CALC_DEFAULT;
	if (r.work.block_type != SYM_BTYPE_ERROR) {
		errorval = refine_score<L1>(w, t, r);
	}
	float best_in_mode = r.best_errorval_in_mode, best_in_scb = r.best_errorval_in_scb;
	unsigned int l = r.l;
	bool adjustments = r.adjustments;
	bool error_block = false;
	if (errorval == -ERROR_CALC_DEFAULT) {
		errorval = -errorval;
		error_block = true;
	}
	best_in_mode = minf(errorval, best_in_mode);
	unsigned int refinement_limit = CFG.tune_refinement_limit;
	unsigned int iters_remaining = refinement_limit - 1 - l;
	float threshold = (0.045f * static_cast<float>(iters_remaining)) + 1.0f;
	int action;
	bool new_best = false;
	if (errorval > (threshold * best_in_scb)) {
		action = RF_NEXT_CANDIDATE;
	} else {
		new_best = errorval < best_in_scb;
		if (new_best && errorval < t.tune_errorval_threshold) {
			action = RF_STOP_ALL;
		} else if (!adjustments || l + 1 >= refinement_limit) {
			action = RF_NEXT_CANDIDATE;
		} else {
			action = RF_NEXT_ITERATION;
		}
	}
	refine_apply<L1>(w, t, r, s, action, error_block, best_in_mode, new_best, errorval);
}
ASTC_FN void refine_second_score(const WCtx& w, const Trial& t, Refine& r, BlockSearch& s) {
	refine_second_score_t<false>(w, t, r, s);
}

// step part 4: realign the weights of the work candidate
template <bool L1> ASTC_FN void refine_realign_t(const WCtx& w, const Trial& t, Refine& r) {
	PartView pi = refine_part_view<L1>(t);
	bool adjustments = L1 ? realign_weights_t<true>(w, 1, r.formats, -1, pi, r.qmode, false, (unsigned int)r.dmode)
	                      : realign_weights(w, t.partition_count, r.formats, t.plane2_component, pi, r.qmode, t.dual != 0, (unsigned int)r.dmode);
	ST_WRITE_BEGIN(w)
		r.adjustments = adjustments;
	ST_WRITE_END(w)
}
ASTC_FN void refine_realign(const WCtx& w, const Trial& t, Refine& r) {
	refine_realign_t<false>(w, t, r);
}

#if defined(ASTC_HOSTSIM) && defined(ASTC_TRIAL_STATS)
#include <stdio.h>
static unsigned int g_trial_steps;
#endif

// The CTA main loop. Every warp of the CTA must call this (barriers inside). The search state lives in the warp's arena
// slots (BlockSearch, Trial) and in the Refine slot the caller provides (shared memory, ASTC_REFINE_STATE_BYTES).
ASTC_COOP void compress_blocks_lockstep(WCtx w, BlockFeed feed, uint32_t refine_state_off) {
	BlockSearch& s = *reinterpret_cast<BlockSearch*>(astc_smem + w.base + A_SEARCH);
	Trial& t = *reinterpret_cast<Trial*>(astc_smem + w.base + A_TRIAL);
	Refine& r = *reinterpret_cast<Refine*>(astc_smem + refine_state_off);
	bool has_block = false;
	bool exhausted = false;
	ST_WRITE_BEGIN(w)
		s.phase = 3;
		t.candidate_count = 0;
		t.dual = 0;
		t.partition_count = 1;
		t.packed = 0;
		r.running = false;
	ST_WRITE_END(w)
	while (true) {
		// ---- between rounds: finish / fetch blocks until this warp has a trial to run
		bool active = false;
		while (!exhausted) {
			if (!has_block) {
				unsigned int b;
				if (!feed_next(w, feed, b)) {
					exhausted = true;
					break;
				}
				unsigned int by = b / feed.blocks_x;
				unsigned int bx = b - by * feed.blocks_x;
				if (IMG.alpha_avg != nullptr && !block_has_alpha(w, IMG.alpha_avg, IMG.alpha_threshold, bx * BSD.dim_x, (by + IMG.block_row0) * BSD.dim_y)) {
					wsync();
					if (w.lane == 0) {
						BlkInfo& bi = bi_of(w);
						bi.origin_texel = bi.data_min = bi.data_mean = bi.data_max = splat4(0.0f);
						bi.grayscale = 1;
					}
					wsync();
					emit_if_constant(w, b);
					pass_block_done(w, IMG.done);
					continue;
				}
				load_block(w, bx, by + IMG.block_row0);
				if (emit_if_constant(w, b)) {
					pass_block_done(w, IMG.done);
					continue;
				}
				block_search_begin(w, s, b);
				has_block = true;
			}
			if (block_search_next(w, s, t)) {
				active = true;
				break;
			}
			emit_block(w, s);
			pass_block_done(w, IMG.done);
			has_block = false;
		}
		if (!cta_any(active)) {
			break;
		}
		// ---- the trial, stage by stage
		if (active) stage_ideal(w, t);
		cta_sync();
		if (active) stage_decimate(w, t);
		cta_sync();
		if (active) {
			trial_cutoffs(w, t);
			compute_angular_endpoints(w, t.only_always != 0, t.dual ? 2 : 1, (unsigned int)t.max_weight_quant);
		}
		cta_sync();
		if (active) quantize_and_score_modes(w, t.start_mode, t.end_mode, t.dual ? 2 : 1, t.partition_count, t.max_weight_quant, t.cutoff1, t.cutoff2);
		cta_sync();
		if (active) stage_formats(w, t);
		// ---- refinement steps
		if (active) {
			refine_begin_trial(w, t, r, s, false);
		}
		bool running = active && r.running;
#if defined(ASTC_HOSTSIM) && defined(ASTC_TRIAL_STATS)
		g_trial_steps = 0;
#endif
		while (cta_any(running)) {
			if (running) {
#if defined(ASTC_HOSTSIM) && defined(ASTC_TRIAL_STATS)
				g_trial_steps++;
#endif
				refine_recompute(w, t, r);
			}
			cta_sync();
			if (running) refine_pack(w, t, r);
			cta_sync();
			if (running && r.l == 0) refine_first_score(w, t, r, s);
			cta_sync();
			if (running && r.running && r.in_step) refine_realign(w, t, r);
			cta_sync();
			if (running && r.running && r.in_step) refine_second_score(w, t, r, s);
			running = running && r.running;
		}
#if defined(ASTC_HOSTSIM) && defined(ASTC_TRIAL_STATS)
		if (active) {
			fprintf(stderr, "TRIAL blk=%u dual=%d pc=%u cands=%u steps=%u\n", s.out_index, t.dual, t.partition_count, t.candidate_count, g_trial_steps);
		}
#endif
		if (active) {
			block_search_after_trial(w, s, t, r.best_errorval_in_mode);
		}
	}
}
