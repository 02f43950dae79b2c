// CUDA-native ASTC block compressor: the stage-kernel ("wave") pipeline.
//
// The per-block search is a chain of trials; every trial is [setup: ideal endpoints/weights, decimated weights,
// angular ranges, per-mode errors, endpoint formats] followed by [refinement steps]. Running the whole chain in one
// kernel leaves the SMs starved for instructions (each warp is somewhere else in ~150 KB of code); aligning the
// warps of a CTA on a common stage list fixes the fetch problem but makes them wait for each other, because blocks
// need different numbers of refinement steps. So the chain is cut into four kernels that exchange small per-block
// records through HBM, and every kernel only ever runs ONE kind of work:
//
//   setup    (S) : one trial setup per popped item, warps of a CTA phase-aligned stage by stage
//   refine   (R) : refinement steps; a warp pops the next item as soon as its trial ends - every step is the same
//                  code, so warps never wait for a slower block's extra steps; then the block's decision tree
//                  (compress_block) picks what comes next and routes the block to the matching queue
//   prepare  (P) : block statistics / partition search for blocks entering the 2-plane / n-partition phases
//   emit     (E) : symbolic -> physical packing, one block per LANE
//
// One "wave" = S, R, P over the blocks still searching; the host enqueues as many waves as a block can have trials
// (kernels whose queue is empty return at once) and one E at the end. A block's record is the persistent head of
// its arena plus its texels (DevBsd::record_bytes, 2.4 KB at 6x6): 466 k blocks x ~7 KB moved per trial is
// noise next to 6.5 TB/s of HBM. Results are bit-identical to the single-kernel drivers.
#pragma once

#define ASTC_MAX_WAVES 64
// Set-up and refinement items are queued by the kind of trial they belong to (class 0: one partition, one or two
// planes; class p-1: p partitions): a late wave holds a mix of 2-plane and n-partition trials whose steps differ ~2x in
// length, and warps of a CTA wait for each other every round. Each warp drains class 0, then 1, ... so that the warps
// voting together are (almost always) doing the same kind of step.
#define ASTC_Q_CLASSES 4
// Refinement items have one class more: the one-partition trials are split by planes (class 0: one partition, one plane - the
// mode-0 trial and the full one-plane trial of every block, most of the refinement work; class 1: two planes; class p: p
// partitions). Class 0 of an LDR profile runs the specialised refinement step (astc_dev_lockstep.cuh, L1).
#define ASTC_Q_RCLASSES (ASTC_Q_CLASSES + 1)
// Set-up items are queued by the trial's weight quantisation limit as well (Trial::max_weight_quant, 12 values): a later trial of
// a block searches only the modes up to the limit its best result so far allows, and the cost of a set-up follows it (a
// two-plane set-up at QUANT_32 costs several times one at QUANT_2). Mixed in one queue, every round of a CTA lasts as long as
// its most expensive item.
// A class is drained from the expensive end, so the warps that vote together hold items of the same cost and the cheap ones fill
// the tail of the launch.
#define ASTC_Q_SUB 12
// Preparation items by what they prepare: 0 block statistics (two-plane phase), 1..3 the partition search for 2..4 partitions
// (the search costs several times the statistics; the kernel votes once per item).
#define ASTC_Q_PREP 4
// Refinement items may be sub-queued too (experiment builds, ASTC_RSORT: 1 by the number of candidates, 2 by the kind of weight grid
// of the first candidate, 3 by the trial's weight quantisation limit); the shipped build has one queue per class (ASTC_Q_RSUB 1).
#ifndef ASTC_RSORT
	#define ASTC_RSORT 0
#endif
#if ASTC_RSORT == 0
	#define ASTC_Q_RSUB 1
#else
	#define ASTC_Q_RSUB 4
#endif
enum { Q_SETUP = 0, Q_REFINE = ASTC_Q_CLASSES * ASTC_Q_SUB, Q_PREPARE = Q_REFINE + ASTC_Q_RCLASSES * ASTC_Q_RSUB, Q_EMIT = Q_PREPARE + ASTC_Q_PREP, ASTC_Q_KINDS = Q_EMIT + 1 };

struct WaveArgs {
	uint8_t* records;            // [blocks] x record_bytes
	uint32_t* queues;            // item lists (block indices): list k at queues + k * queue_stride, capacity = blocks each
	size_t queue_stride;
	uint32_t* count;             // [ASTC_Q_KINDS][ASTC_MAX_WAVES] items pushed (Q_EMIT uses wave slot 0)
	uint32_t* head;              // [ASTC_Q_KINDS][ASTC_MAX_WAVES] items popped
	unsigned int total;          // blocks of the slab (capacity of every queue)
	unsigned int blocks_x;
	// wave 0 reads the image; the host may cut it into bands of block rows (upload of band k+1 under the set-up of band k):
	// a wave-0 launch takes blocks [first_block, first_block + band_blocks) from its own ticket counter
	uint32_t* ticket;
	unsigned int first_block, band_blocks;
	// set-up launches of waves >= 1 may be split by class of trial: [cls_lo, cls_hi) of the ASTC_Q_CLASSES queues (the one-plane
	// classes run on the compact arena plan)
	int cls_lo, cls_hi;
	int wave;
	unsigned int sync_mask;      // tuning: which stage barriers are active (bit i = i-th barrier of the kernel loop)
	uint32_t stage_bytes_setup;  // set-up kernel: the same (decimation tables only)
	uint32_t refine_state_off;   // refine kernel: offset of the per-warp Refine slots (ASTC_REFINE_STATE_BYTES each) in the shared window
	uint32_t stage_bytes;        // refine kernel: bytes of tables staged between the header and the arenas (0 = none)
	// (the progress and cancellation words of the pass are in the launch constants, IMG.cancel / IMG.done: kept out of this
	// struct, which the item loops take by value)
};

#if defined(ASTC_HOSTSIM)
ASTC_FN uint32_t q_atomic_add(uint32_t* p, uint32_t v) { uint32_t o = *p; *p = o + v; return o; }
ASTC_FN uint32_t q_load(const uint32_t* p) { return *p; }
#else
ASTC_FN uint32_t q_atomic_add(uint32_t* p, uint32_t v) { return atomicAdd(p, v); }
ASTC_FN uint32_t q_load(const uint32_t* p) { return __ldcg(p); }
#endif

// q_pop without the look at the cancel flag: the refinement kernel looks once per item in its drain loop instead (wave_refine).
// (The look inside each pop of q_pop_classes costs the refinement kernels more spill code, -Xptxas -v.)
ASTC_FN bool q_pop_plain(const WCtx& w, const WaveArgs& a, int kind, int wave, unsigned int& b) {
	uint32_t i = 0;
	if (w.lane == 0) {
		i = q_atomic_add(a.head + kind * ASTC_MAX_WAVES + wave, 1u);
	}
	i = wbroadcast0(w, i);
	if (i >= q_load(a.count + kind * ASTC_MAX_WAVES + wave)) {
		return false;
	}
	b = q_load(a.queues + (size_t)kind * a.queue_stride + i);
	return true;
}
// one item of a queue; false once the queue is empty or the pass is cancelled (the flag is looked at before the item is taken)
ASTC_FN bool q_pop(const WCtx& w, const WaveArgs& a, int kind, int wave, unsigned int& b) {
	uint32_t i = 0xFFFFFFFFu;      // (past the end of every queue: what a warp sees once the pass is cancelled)
	if (w.lane == 0 && !pass_cancelled(IMG.cancel)) {
		i = q_atomic_add(a.head + kind * ASTC_MAX_WAVES + wave, 1u);
	}
	i = wbroadcast0(w, i);
	if (i >= q_load(a.count + kind * ASTC_MAX_WAVES + wave)) {
		return false;
	}
	b = q_load(a.queues + (size_t)kind * a.queue_stride + i);
	return true;
}

// pop from the classes of a kind in order; cls is the warp's cursor (the caller looks at the cancel flag)
ASTC_FN bool q_pop_classes(const WCtx& w, const WaveArgs& a, int kind, int wave, int& cls, unsigned int& b, int cls_end = ASTC_Q_CLASSES) {
	while (cls < cls_end) {
		if (q_pop_plain(w, a, kind + cls, wave, b)) {
			return true;
		}
		cls++;
	}
	return false;
}

// set-up items: the classes' sub-queues in order, each class from the expensive end; cls is the warp's cursor over
// [cls_lo * ASTC_Q_SUB, cls_end * ASTC_Q_SUB). Empty sub-queues are skipped 32 at a time with plain loads (a look that can be
// stale only in the harmless direction: the atomic pop decides), so a drained launch costs a warp one round trip, not one per queue.
ASTC_FN int sorted_kind_of_cursor(int base_kind, int nsub, int cls) {
	int klass = cls / nsub;
	return base_kind + klass * nsub + (nsub - 1 - (cls - klass * nsub));
}
// queues base_kind + klass * nsub + sub; cls = cursor over [.., cls_end * nsub)
ASTC_FN bool q_pop_sorted(const WCtx& w, const WaveArgs& a, int base_kind, int nsub, int wave, int& cls, unsigned int& b, int cls_end) {
	const int end = cls_end * nsub;
	bool look = (cls % nsub) == 0;      // entering a class: find its first queue with items; otherwise pop where the last item came from
	while (cls < end) {
#if !defined(ASTC_ONE_LANE)
		if (look) {
			int k = cls + w.lane;
			bool has = false;
			if (k < end) {
				int kind = sorted_kind_of_cursor(base_kind, nsub, k);
				has = q_load(a.count + kind * ASTC_MAX_WAVES + wave) > q_load(a.head + kind * ASTC_MAX_WAVES + wave);
			}
			uint32_t m = __ballot_sync(0xffffffffu, has);
			if (m == 0) {
				cls += ASTC_WARP;
				continue;
			}
			cls += __ffs((int)m) - 1;
		}
#endif
		if (q_pop(w, a, sorted_kind_of_cursor(base_kind, nsub, cls), wave, b)) {
			return true;
		}
		cls++;
		look = true;
	}
	return false;
}
ASTC_FN bool q_pop_setup(const WCtx& w, const WaveArgs& a, int wave, int& cls, unsigned int& b, int cls_end) {
	return q_pop_sorted(w, a, Q_SETUP, ASTC_Q_SUB, wave, cls, b, cls_end);
}
ASTC_FN int setup_queue_of(const Trial& t, int klass) {
	int q = t.max_weight_quant;
	q = q < 0 ? 0 : (q >= ASTC_Q_SUB ? ASTC_Q_SUB - 1 : q);
	return Q_SETUP + klass * ASTC_Q_SUB + q;
}

ASTC_FN int refine_queue_of(const WCtx& w, const Trial& t, int klass) {
#if ASTC_RSORT == 1
	int k = (int)t.candidate_count - 1;
#elif ASTC_RSORT == 2
	// 0: the first candidate's grid is the full grid (no realignment replay to speak of), 1: up to 16 weights, 2: up to 32, 3: more
	Candidate c0 = sptr<Candidate>(w.base + A_CAND)[0];
	const DevDecMode* dm = BSD.dec_modes + ASTC_LDG(&BSD.block_modes[c0.block_mode].decimation_mode);
	int W = ASTC_LDG(&dm->weight_count);
	int k = W == w.T ? 0 : (W <= 16 ? 1 : (W <= 32 ? 2 : 3));
#elif ASTC_RSORT == 3
	int k = t.max_weight_quant / 3;
#else
	int k = 0;
	(void)w; (void)t;
#endif
	k = k < 0 ? 0 : (k >= ASTC_Q_RSUB ? ASTC_Q_RSUB - 1 : k);
	return Q_REFINE + klass * ASTC_Q_RSUB + k;
}

ASTC_FN void q_push(const WCtx& w, const WaveArgs& a, int kind, int wave, unsigned int b) {
	if (w.lane == 0) {
		uint32_t i = q_atomic_add(a.count + kind * ASTC_MAX_WAVES + wave, 1u);
		a.queues[(size_t)kind * a.queue_stride + i] = b;
	}
}

// record <-> arena: the persistent head [0, A_PERSIST) and the block texels.
// On the device both directions are BULK ASYNCHRONOUS COPIES (the 1-D form of TMA, cp.async.bulk): one lane hands the two
// ranges to the copy engine of the SM - global -> shared completes on the warp's mbarrier (A_MBAR), shared -> global as a
// bulk group - instead of 32 lanes moving 16 bytes per trip through registers. Addresses and sizes are multiples of 16
// bytes by construction (arena bases, A_BLK, record_bytes). The host simulation copies word by word.
// (the texels never change after the first save: later saves write the head only)
struct alignas(16) U128 {
	uint32_t x, y, z, w;
};
#if defined(ASTC_HOSTSIM)
ASTC_FN void record_mbar_init(const WCtx& w) { (void)w; }
ASTC_FN void record_copy(const WCtx& w, const WaveArgs& a, unsigned int b, bool save, bool with_texels, uint32_t& phase) {
	(void)phase;
	U128* g = reinterpret_cast<U128*>(a.records + (size_t)b * BSD.record_bytes);
	const int n1 = A_PERSIST / 16;
	int n2 = with_texels ? ((w.T + 3) & ~3) : 0;      // 4 channels x Tp floats = Tp x 16 bytes
	SPtr<U128> h = sptr<U128>(w.base);
	SPtr<U128> t = sptr<U128>(w.base + A_BLK);
	ASTC_NOUNROLL
	for (int i = w.lane; i < n1 + n2; i += ASTC_WARP) {
		if (save) {
			g[i] = i < n1 ? h[i] : t[i - n1];
		} else {
			U128 v = g[i];
			if (i < n1) h[i] = v;
			else t[i - n1] = v;
		}
	}
	wsync();
}
#else
ASTC_FN uint32_t smem_addr(uint32_t off) { return (uint32_t)__cvta_generic_to_shared(astc_smem + off); }
// once per warp, before its first restore: one pending arrival per phase (the lane that issues the copies)
ASTC_FN void record_mbar_init(const WCtx& w) {
	if (w.lane == 0) {
		asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_addr(w.base + A_MBAR)));
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	__syncwarp();
}
ASTC_FN void record_copy(const WCtx& w, const WaveArgs& a, unsigned int b, bool save, bool with_texels, uint32_t& phase) {
	const uint8_t* g = a.records + (size_t)b * BSD.record_bytes;
	const uint32_t n1 = A_PERSIST;
	const uint32_t n2 = with_texels ? (uint32_t)((w.T + 3) & ~3) * 16u : 0u;
	const uint32_t s_head = smem_addr(w.base), s_tex = smem_addr(w.base + A_BLK), bar = smem_addr(w.base + A_MBAR);
	__syncwarp();      // every lane is done with the arena contents that are about to be replaced / has written what is saved
	if (save) {
		if (w.lane == 0) {
			// the lanes' (generic proxy) stores to shared memory must be visible to the copy engine (async proxy)
			asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
			asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(g), "r"(s_head), "r"(n1) : "memory");
			if (n2) {
				asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(g + n1), "r"(s_tex), "r"(n2) : "memory");
			}
			asm volatile("cp.async.bulk.commit_group;" ::: "memory");
			// the arena may be overwritten as soon as the engine has READ it (the stores to HBM complete behind our back;
			// the consumer is a later kernel launch)
			asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
		}
		__syncwarp();
		return;
	}
	if (w.lane == 0) {
		asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
		asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(n1 + n2) : "memory");
		asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(s_head), "l"(g), "r"(n1), "r"(bar) : "memory");
		if (n2) {
			asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(s_tex), "l"(g + n1), "r"(n2), "r"(bar) : "memory");
		}
	}
	// every lane waits for the phase to complete: the bytes are then visible to it
	uint32_t done = 0;
	unsigned int spins = 0;
	while (!done) {
		asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(bar), "r"(phase) : "memory");
		if (!done && ++spins > (1u << 26)) {
			__trap();      // (a copy that never completes would otherwise hang the GPU: fail loudly instead)
		}
	}
	phase ^= 1u;
	__syncwarp();
}
#endif

ASTC_FN BlockSearch& search_of(const WCtx& w) { return *reinterpret_cast<BlockSearch*>(astc_smem + w.base + A_SEARCH); }
ASTC_FN Trial& trial_of(const WCtx& w) { return *reinterpret_cast<Trial*>(astc_smem + w.base + A_TRIAL); }
static_assert(sizeof(BlockSearch) <= 128 && sizeof(Trial) <= 64, "search state must fit its arena slots");

// the search state already lives in its arena slots: saving / restoring a record moves it with the rest of the head
ASTC_FN void record_save(const WCtx& w, const WaveArgs& a, unsigned int b, bool with_texels = false) {
	uint32_t unused = 0;
	wsync();
	record_copy(w, a, b, true, with_texels, unused);
}
// phase: the parity of the warp's mbarrier, kept by the caller's item loop (flips with every restore)
ASTC_FN void record_restore(const WCtx& w, const WaveArgs& a, unsigned int b, uint32_t& phase) {
	record_copy(w, a, b, false, true, phase);
}

ASTC_FN int trial_class(const Trial& t) {
	int c = t.dual ? 0 : (int)t.partition_count - 1;
	return c < 0 ? 0 : (c >= ASTC_Q_CLASSES ? ASTC_Q_CLASSES - 1 : c);
}
// the class of a trial's refinement queue (ASTC_Q_RCLASSES)
ASTC_FN int refine_class(const Trial& t) {
	return (!t.dual && t.partition_count == 1) ? 0 : trial_class(t) + 1;
}

#if defined(ASTC_STEP_STATS)
// dev instrumentation (make -C astc-encoder_b200 variant NAME=stats DEFS=-DASTC_STEP_STATS=1): cycles per part, printed by the emit kernel.
// refinement: [class][part]; class = realign path (0 undecimated, 1 dense, 2 sparse) + 3 for the first step of a candidate;
//             parts: recompute, pack, score1, realign, score2, block change, wait at the vote, number of steps
// set-up:     [kind][part]; kind 0 shared 1-plane set-up (wave 0), 1 two planes, 2 n partitions;
//             parts: ideal, decimate, angular, quantise+score, formats + candidate weights, record save, wait, items
__device__ unsigned long long g_step_stats[6][8];
__device__ unsigned long long g_setup_stats[3][8];
__device__ unsigned long long g_setup_bar[3];
__device__ unsigned long long g_setup_q[3][12][3];      // by max_weight_quant: items, cycles before / after the stage barrier
__device__ unsigned int g_setup_hist[3][2][32];
// tails: histograms (4096-cycle buckets) of a step's parts over all kinds of step: 0 recompute, 1 pack, 2 score1, 3 realign, 4 score2,
// 5 the whole step's work, 6 block change (only the warps that changed block), 7 wait at the vote
__device__ unsigned int g_step_hist[8][32];
__device__ __forceinline__ void stat_hist(int part, long long cycles) {
	int b = (int)(cycles >> 12);
	atomicAdd(&g_step_hist[part][b < 0 ? 0 : (b > 31 ? 31 : b)], 1u);
}
#define STAT_T(v) long long v = clock64()
#else
#define STAT_T(v)
#endif

// ---------------------------------------------------------------------------------------------
// S: trial setup. Wave 0 reads the image (load_block, constant-colour blocks are emitted on the spot).
// S1 = true: the wave-0 launches of an LDR profile. The first trial of every block has one partition and one plane, so its
// stages run the S1 instantiation (astc_dev_lockstep.cuh, "trial stages"), inlined here; a trial of another shape would take
// the general stages.
// ---------------------------------------------------------------------------------------------
template <bool S1>
ASTC_COOP void wave_setup_t(WCtx w, WaveArgs a) {
	// one copy of the search state per warp, in the arena slots the record keeps it in (discipline: astc_dev_lockstep.cuh,
	// "THE SEARCH STATE ..."); the widened copy of the trial used by the shared set-up sits in the work / mod colour slots,
	// which only refinement uses
	BlockSearch& s = search_of(w);
	Trial& t = trial_of(w);
	Trial& tf = *reinterpret_cast<Trial*>(astc_smem + w.base + A_SCB + 160);
	BlockFeed feed;
	feed.ticket = a.ticket;      // wave 0 has no queue: a ticket counter hands out the band's blocks
	feed.total = a.band_blocks;
	feed.blocks_x = a.blocks_x;
	feed.cancel = IMG.cancel;
	int cls = a.cls_lo * ASTC_Q_SUB;
	uint32_t rec_phase = 0;
	record_mbar_init(w);
	while (true) {
		bool active = false;
		unsigned int b = 0;
		if (a.wave == 0) {
			while (feed_next(w, feed, b)) {
				b += a.first_block;
				unsigned int by = b / a.blocks_x;
				unsigned int bx = b - by * a.blocks_x;
				if (IMG.alpha_avg != nullptr && !block_has_alpha(w, IMG.alpha_avg, IMG.alpha_threshold, bx * BSD.dim_x, (by + IMG.block_row0) * BSD.dim_y)) {
					// alpha-scale RDO (astcenc_entry.cpp:1021-1030): the block is treated as all-zero
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
				block_search_advance(w, s, t);       // phase 0 always yields a trial
				active = true;
				break;
			}
		} else if (q_pop_setup(w, a, a.wave, cls, b, a.cls_hi)) {
			record_restore(w, a, b, rec_phase);
			active = true;
		}
		// one CTA-wide vote per round: it doubles as the barrier that keeps the warps loosely phase-aligned
		// (without it the pass is much slower)
		STAT_T(sv);
		if (!cta_any(active)) {
			break;
		}
		STAT_T(s0);
		// The mode-0 trial (only the "always" modes) and the full 1-plane trial that follows it differ in nothing but
		// the range of grids / block modes they look at: ideal weights, decimated weights, angular ranges and per-mode
		// errors of the shared modes are identical (compress_symbolic.cpp:1243-1270 runs the same code twice).
		// One set-up over the full range therefore serves both; the second candidate list waits in A_CAND2.
		bool shared = active && !t.dual && t.only_always && t.partition_count == 1;
		// (the restored trial's own shape is checked too: only a one-partition, one-plane trial may run the folded stages)
		const bool s1 = S1 && active && !t.dual && t.partition_count == 1;
		if (active) {
			ST_WRITE_BEGIN(w)
				tf = t;
				if (shared) {
					tf.only_always = 0;
				}
			ST_WRITE_END(w)
		}
		if (active) {
			if (s1) stage_ideal_t<true>(w, tf);
			else stage_ideal(w, tf);
		}
		STAT_T(st1);
		if (a.sync_mask & 1) cta_sync();
		if (active) {
			if (s1) stage_decimate_t<true>(w, tf);
			else stage_decimate(w, tf);
		}
		STAT_T(s2);
		if (a.sync_mask & 2) cta_sync();
		if (active) {
			trial_cutoffs(w, tf);
			if (s1) compute_angular_endpoints_t<true>(w, tf.only_always != 0, 1, (unsigned int)tf.max_weight_quant);
			else compute_angular_endpoints(w, tf.only_always != 0, tf.dual ? 2 : 1, (unsigned int)tf.max_weight_quant);
		}
		STAT_T(s3);
		if (a.sync_mask & 4) cta_sync();
		if (active) {
			if (s1) quantize_and_score_modes_t<true>(w, tf.start_mode, tf.end_mode, 1, 1, tf.max_weight_quant, tf.cutoff1, tf.cutoff2);
			else quantize_and_score_modes(w, tf.start_mode, tf.end_mode, tf.dual ? 2 : 1, tf.partition_count, tf.max_weight_quant, tf.cutoff1, tf.cutoff2);
		}
		STAT_T(s4);
		if (a.sync_mask & 8) cta_sync();
		STAT_T(s4b);
		if (active) {
			unsigned int count = 0, count_next = 0;
			if (shared) {
				PartView pi = part_view_packed(1, 0);
				SPtr<f4> ep = ep_of(w);
				unsigned int end_full = tf.end_mode;
				if (s1) {
					endpoint_formats_prepare_t<true>(w, pi, EP_EI1_0, EP_EI1_1, 1, 0, end_full);
					count = endpoint_formats_select_t<true>(w, 1, 1, 0, BSD.block_mode_count_1plane_always, w.base + A_CAND, true);
					count_next = endpoint_formats_select_t<true>(w, 1, 1, 0, end_full, w.base + A_CAND2, false);
				} else {
					endpoint_formats_prepare(w, pi, EP_EI1_0, EP_EI1_1, 1, 0, end_full);
					count = endpoint_formats_select(w, 1, 1, 0, BSD.block_mode_count_1plane_always, w.base + A_CAND, true);
					count_next = endpoint_formats_select(w, 1, 1, 0, end_full, w.base + A_CAND2, false);
				}
				ASTC_NOUNROLL
				for (int k = w.lane; k < 4; k += ASTC_WARP) {
					ep[EP_BASE_0 + k] = ep[EP_EI1_0 + k];
					ep[EP_BASE_1 + k] = ep[EP_EI1_1 + k];
				}
			}
			ST_WRITE_BEGIN(w)
				t.cutoff1 = tf.cutoff1;
				t.cutoff2 = tf.cutoff2;
				t.start_mode = tf.start_mode;
				t.end_mode = shared ? BSD.block_mode_count_1plane_always : tf.end_mode;
				t.candidate_count_next = count_next;
				if (shared) {
					t.candidate_count = count;
				}
			ST_WRITE_END(w)
			if (!shared) {
				if (s1) stage_formats_t<true>(w, t);
				else stage_formats(w, t);
			}
			// the refinement kernel has no decimated ideal weights: quantise every candidate's weights now, straight into the
			// candidates' slots (unused bytes of a slot are never read), one barrier at the end
			int nplanes = s1 ? 1 : (t.dual ? 2 : 1);
			float cutoff1 = t.cutoff1, cutoff2 = t.cutoff2;
			ASTC_NOUNROLL
			for (int list = 0; list < 2; list++) {
				unsigned int n = list == 0 ? t.candidate_count : t.candidate_count_next;
				SPtr<Candidate> cl = sptr<Candidate>(w.base + (list == 0 ? A_CAND : A_CAND2));
				SPtr<uint8_t> cw = sptr<uint8_t>(w.base + (list == 0 ? A_CANDW : A_CANDW2));
				ASTC_NOUNROLL
				for (unsigned int i = 0; i < n; i++) {
					Candidate cd = cl[(int)i];
					const DevBlockMode* bm = BSD.block_modes + cd.block_mode;
					quantize_candidate_weights_to(w, cw + (int)i * 64, ASTC_LDG(&bm->decimation_mode), ASTC_LDG(&bm->quant_mode), nplanes, cutoff1, cutoff2);
				}
			}
			wsync();
			STAT_T(s5);
			record_save(w, a, b, a.wave == 0);
			q_push(w, a, refine_queue_of(w, t, refine_class(t)), a.wave, b);
#if defined(ASTC_STEP_STATS)
			if (w.lane == 0) {
				long long s6 = clock64();
				int kind = t.dual ? 1 : (t.partition_count > 1 ? 2 : 0);
				atomicAdd(&g_setup_stats[kind][0], (unsigned long long)(st1 - s0));
				atomicAdd(&g_setup_stats[kind][1], (unsigned long long)(s2 - st1));
				atomicAdd(&g_setup_stats[kind][2], (unsigned long long)(s3 - s2));
				atomicAdd(&g_setup_stats[kind][3], (unsigned long long)(s4 - s3));
				atomicAdd(&g_setup_stats[kind][4], (unsigned long long)(s5 - s4b));
				atomicAdd(&g_setup_bar[kind], (unsigned long long)(s4b - s4));
				{
					int q = t.max_weight_quant < 0 ? 0 : (t.max_weight_quant > 11 ? 11 : t.max_weight_quant);
					atomicAdd(&g_setup_q[kind][q][0], 1ull);
					atomicAdd(&g_setup_q[kind][q][1], (unsigned long long)(s4 - s0));
					atomicAdd(&g_setup_q[kind][q][2], (unsigned long long)(s5 - s4b));
				}
				{
					// tails: item work up to the stage barrier / after it, 8192-cycle buckets
					int b1 = (int)((s4 - s0) >> 13), b2 = (int)((s5 - s4b) >> 13);
					atomicAdd(&g_setup_hist[kind][0][b1 > 31 ? 31 : b1], 1u);
					atomicAdd(&g_setup_hist[kind][1][b2 > 31 ? 31 : b2], 1u);
				}
				atomicAdd(&g_setup_stats[kind][5], (unsigned long long)(s6 - s5));
				atomicAdd(&g_setup_stats[kind][6], (unsigned long long)(s0 - sv));
				atomicAdd(&g_setup_stats[kind][7], 1ull);
			}
#endif
		}
	}
}

// which instantiation a set-up launch of wave a.wave runs: S1 for wave 0 of an LDR or sRGB profile, the general one otherwise
// (the rule the host code applies when it picks the set-up kernel, astcenc_b200.cu setup_kernel; the host simulation calls this)
ASTC_COOP void wave_setup(WCtx w, WaveArgs a) {
	if (a.wave == 0 && (CFG.profile == PRF_LDR || CFG.profile == PRF_LDR_SRGB)) {
		wave_setup_t<true>(w, a);
	} else {
		wave_setup_t<false>(w, a);
	}
}

// ---------------------------------------------------------------------------------------------
// R: refinement steps + the decision what the block does next.
// ---------------------------------------------------------------------------------------------
ASTC_COOP void wave_finish_trial(WCtx w, const WaveArgs& a, unsigned int b, BlockSearch& s, Trial& t, float errorval) {
	unsigned int ready = t.candidate_count_next;
	block_search_after_trial(w, s, t, errorval);
	int next = block_search_advance(w, s, t);
	bool straight = ready != 0 && next == NEXT_TRIAL && s.phase == 0;
	ST_WRITE_BEGIN(w)
		t.candidate_count_next = 0;
		if (straight) {
			t.candidate_count = ready;
		}
	ST_WRITE_END(w)
	if (straight) {
		// the set-up of the trial just finished already selected this trial's candidates: go straight to refinement
		SPtr<uint32_t> dst = sptr<uint32_t>(w.base + A_CAND);
		SPtr<uint32_t> src = sptr<uint32_t>(w.base + A_CAND2);
		ASTC_NOUNROLL
		for (int k = w.lane; k < (64 + 512) / 4; k += ASTC_WARP) {
			dst[k] = src[k];
		}
		record_save(w, a, b);
		q_push(w, a, refine_queue_of(w, t, refine_class(t)), a.wave + 1, b);
		return;
	}
	record_save(w, a, b);
	if (next == NEXT_TRIAL) {
		q_push(w, a, setup_queue_of(t, trial_class(t)), a.wave + 1, b);
	} else if (next == NEXT_PREPARE) {
		int pk = s.phase == 1 ? 0 : (s.pc < 2 ? 1 : (s.pc > ASTC_Q_PREP ? ASTC_Q_PREP - 1 : s.pc - 1));
		q_push(w, a, Q_PREPARE + pk, a.wave, b);
	} else {
		q_push(w, a, Q_EMIT, 0, b);
		pass_block_done(w, IMG.done);
	}
}

// The refine kernel works on ONE copy of the search state per warp in shared memory: BlockSearch and Trial in their arena
// slots (where the record keeps them anyway), Refine in a slot behind the arenas (as per-lane automatic variables the three
// structs were ~10 KB of local memory per warp: ncu showed an L1 hit rate of 39 % and long-scoreboard stalls on local loads).
// Reads and writes follow the lane-0-publishes discipline of astc_dev_lockstep.cuh, so the result does not depend on how
// the lanes of a warp are scheduled (the thread-per-lane host simulation runs this very code).
#define ASTC_REFINE_STATE_BYTES 128
static_assert(sizeof(Refine) <= ASTC_REFINE_STATE_BYTES, "Refine must fit its shared-memory slot");

// L1_STEP = false compiles the specialised step out (the kernel of the HDR profiles, which never take it)
template <bool L1_STEP = true>
ASTC_COOP void wave_refine(WCtx w, WaveArgs a, uint32_t warp_index) {
	BlockSearch& s = search_of(w);
	Trial& t = trial_of(w);
	Refine& r = *reinterpret_cast<Refine*>(astc_smem + a.refine_state_off + warp_index * ASTC_REFINE_STATE_BYTES);
	bool has_item = false;
	bool drained = false;
	unsigned int b = 0;
	unsigned int round = 0;
	int cls = 0;
	uint32_t rec_phase = 0;
	record_mbar_init(w);
	const unsigned int vote_mask = (1u << ((a.sync_mask >> 8) & 7)) - 1u;
	// class 0 of an LDR profile: the step with every part inlined (one partition, one plane, LDR endpoint formats). The warp's
	// queue cursor says which class the item came from; the classes are drained in order, so the specialised items come first.
	const bool ldr = L1_STEP && (CFG.profile == PRF_LDR || CFG.profile == PRF_LDR_SRGB);
	bool l1 = false;
#if defined(ASTC_STEP_STATS)
	int st_prev_class = -1;
	long long st_prev_end = 0;
#endif
	while (true) {
		while (!has_item && !drained) {
#if ASTC_Q_RSUB == 1
			// (a raised cancel flag drains the queues; a pass without one skips the look)
			bool stop = false;
			if (IMG.cancel != nullptr) {
				uint32_t c = 0;
				if (w.lane == 0) c = pass_cancelled(IMG.cancel) ? 1u : 0u;
				stop = wbroadcast0(w, c) != 0u;
			}
			if (stop || !q_pop_classes(w, a, Q_REFINE, a.wave, cls, b, ASTC_Q_RCLASSES)) {
#else
			if (!q_pop_sorted(w, a, Q_REFINE, ASTC_Q_RSUB, a.wave, cls, b, ASTC_Q_RCLASSES)) {
#endif
				drained = true;
				break;
			}
			record_restore(w, a, b, rec_phase);
			// (the restored trial's own shape is checked too: only a one-partition, one-plane trial may run the folded step)
			l1 = ldr && cls < ASTC_Q_RSUB && !t.dual && t.partition_count == 1;
			refine_begin_trial(w, t, r, s, true);
			if (!r.running) {
				wave_finish_trial(w, a, b, s, t, r.best_errorval_in_mode);
				continue;
			}
			has_item = true;
		}
		STAT_T(tv);
		// (vote_period: tuning knob - vote only every 2^n-th round)
		if ((round++ & vote_mask) == 0) {
			if (!cta_any(has_item)) {
				break;
			}
		}
		STAT_T(t0);
#if defined(ASTC_STEP_STATS)
		bool st_on = has_item;
		int st_first = has_item && r.l == 0 ? 3 : 0;
		if (st_on && w.lane == 0 && st_prev_class >= 0) {
			atomicAdd(&g_step_stats[st_prev_class][5], (unsigned long long)(tv - st_prev_end));
			atomicAdd(&g_step_stats[st_prev_class][6], (unsigned long long)(t0 - tv));
			if (tv - st_prev_end > 512) stat_hist(6, tv - st_prev_end);
			stat_hist(7, t0 - tv);
		}
#endif
		if (has_item) {
			if (l1) refine_recompute_t<true>(w, t, r);
			else refine_recompute(w, t, r);
		}
		STAT_T(t1);
		if (a.sync_mask & 16) cta_sync();
		if (has_item) {
			if (l1) refine_pack_t<true>(w, t, r);
			else refine_pack(w, t, r);
		}
		STAT_T(t2);
		if (a.sync_mask & 32) cta_sync();
		if (has_item && r.l == 0) {
			if (l1) refine_first_score_t<true>(w, t, r, s);
			else refine_first_score(w, t, r, s);
		}
		STAT_T(t3);
		if (a.sync_mask & 64) cta_sync();
		if (has_item && r.running && r.in_step) {
			if (l1) refine_realign_t<true>(w, t, r);
			else refine_realign(w, t, r);
		}
		STAT_T(t4);
		if (a.sync_mask & 128) cta_sync();
		if (has_item && r.running && r.in_step) {
			if (l1) refine_second_score_t<true>(w, t, r, s);
			else refine_second_score(w, t, r, s);
		}
		STAT_T(t5);
#if defined(ASTC_STEP_STATS)
		if (st_on) {
			const DevDecMode* dmp = BSD.dec_modes + r.dmode;
			int cls = (dec_view((unsigned int)r.dmode).W == w.T ? 0 : (ASTC_LDG(&dmp->max_weight_texels) <= 6 ? 1 : 2)) + st_first;
			if (w.lane == 0) {
				atomicAdd(&g_step_stats[cls][0], (unsigned long long)(t1 - t0));
				atomicAdd(&g_step_stats[cls][1], (unsigned long long)(t2 - t1));
				atomicAdd(&g_step_stats[cls][2], (unsigned long long)(t3 - t2));
				atomicAdd(&g_step_stats[cls][3], (unsigned long long)(t4 - t3));
				atomicAdd(&g_step_stats[cls][4], (unsigned long long)(t5 - t4));
				atomicAdd(&g_step_stats[cls][7], 1ull);
				stat_hist(0, t1 - t0);
				stat_hist(1, t2 - t1);
				stat_hist(2, t3 - t2);
				stat_hist(3, t4 - t3);
				stat_hist(4, t5 - t4);
				stat_hist(5, t5 - t0);
			}
			st_prev_class = cls;
			st_prev_end = t5;
		}
#endif
		if (has_item && !r.running) {
			wave_finish_trial(w, a, b, s, t, r.best_errorval_in_mode);
			has_item = false;
		}
	}
}

// ---------------------------------------------------------------------------------------------
// P: block statistics / partition search.
// ---------------------------------------------------------------------------------------------
ASTC_COOP void wave_prepare(WCtx w, WaveArgs a) {
	BlockSearch& s = search_of(w);
	Trial& t = trial_of(w);
	uint32_t rec_phase = 0;
	int pcls = 0;
	record_mbar_init(w);
	while (true) {
		unsigned int b = 0;
		// (the expensive kinds first)
		bool active = q_pop_sorted(w, a, Q_PREPARE, ASTC_Q_PREP, a.wave, pcls, b, 1);
		if (!cta_any(active)) {
			break;
		}
		if (active) {
			record_restore(w, a, b, rec_phase);
			int next;
			do {
				block_search_prepare(w, s);
				next = block_search_advance(w, s, t);
			} while (next == NEXT_PREPARE);
			int klass = trial_class(t);
			record_save(w, a, b);
			if (next == NEXT_TRIAL) {
				q_push(w, a, setup_queue_of(t, klass), a.wave + 1, b);
			} else {
				q_push(w, a, Q_EMIT, 0, b);
				pass_block_done(w, IMG.done);
			}
		}
	}
}

// ---------------------------------------------------------------------------------------------
// E: symbolic -> physical, one block per lane. Each lane gets a private 96-byte slice holding its block's
// best_weights / best_colors, addressed through a lane-private context so symbolic_to_physical() runs unchanged.
// ---------------------------------------------------------------------------------------------
#define EMIT_SLICE 96
ASTC_COOP void wave_emit(int lane, uint32_t slices_base, WaveArgs a) {
#if defined(ASTC_STEP_STATS)
	if (blockIdx.x == 0 && threadIdx.x == 0) {
		for (int c = 0; c < 3; c++) {
			unsigned long long n = g_setup_stats[c][7];
			printf("setup kind %d n %llu: ideal %llu decimate %llu angular %llu quantscore %llu formats %llu save %llu wait %llu (cycles per item)\n", c, n,
			       g_setup_stats[c][0] / (n ? n : 1), g_setup_stats[c][1] / (n ? n : 1), g_setup_stats[c][2] / (n ? n : 1), g_setup_stats[c][3] / (n ? n : 1),
			       g_setup_stats[c][4] / (n ? n : 1), g_setup_stats[c][5] / (n ? n : 1), g_setup_stats[c][6] / (n ? n : 1));
			printf("setup kind %d: wait at the stage barrier %llu\n", c, g_setup_bar[c] / (n ? n : 1));
			g_setup_bar[c] = 0;
			printf("setup kind %d by max_weight_quant (items : cycles before / after the barrier):", c);
			for (int q = 0; q < 12; q++) {
				unsigned long long m = g_setup_q[c][q][0];
				printf(" q%d %llu : %llu / %llu,", q, m, g_setup_q[c][q][1] / (m ? m : 1), g_setup_q[c][q][2] / (m ? m : 1));
				g_setup_q[c][q][0] = g_setup_q[c][q][1] = g_setup_q[c][q][2] = 0;
			}
			printf("\n");
			for (int h = 0; h < 2; h++) {
				printf("hist setup kind %d %s (8192-cycle buckets):", c, h == 0 ? "before the barrier" : "after the barrier ");
				for (int b = 0; b < 32; b++) {
					printf(" %u", g_setup_hist[c][h][b]);
					g_setup_hist[c][h][b] = 0;
				}
				printf("\n");
			}
			for (int k = 0; k < 8; k++) g_setup_stats[c][k] = 0;
		}
		for (int c = 0; c < 6; c++) {
			unsigned long long n = g_step_stats[c][7];
			printf("steps class %d n %llu: recompute %llu pack %llu score1 %llu realign %llu score2 %llu change %llu wait %llu (cycles per step)\n", c, n,
			       g_step_stats[c][0] / (n ? n : 1), g_step_stats[c][1] / (n ? n : 1), g_step_stats[c][2] / (n ? n : 1), g_step_stats[c][3] / (n ? n : 1),
			       g_step_stats[c][4] / (n ? n : 1), g_step_stats[c][5] / (n ? n : 1), g_step_stats[c][6] / (n ? n : 1));
			for (int k = 0; k < 8; k++) g_step_stats[c][k] = 0;
		}
		const char* names[8] = {"recompute", "pack", "score1", "realign", "score2", "step work", "block change", "wait"};
		for (int p = 0; p < 8; p++) {
			printf("hist %-12s (4096-cycle buckets):", names[p]);
			for (int b = 0; b < 32; b++) {
				printf(" %u", g_step_hist[p][b]);
				g_step_hist[p][b] = 0;
			}
			printf("\n");
		}
	}
#endif
	uint32_t n = q_load(a.count + Q_EMIT * ASTC_MAX_WAVES);
	while (true) {
		uint32_t i0 = 0;
		if (lane == 0) {
			i0 = q_atomic_add(a.head + Q_EMIT * ASTC_MAX_WAVES, (uint32_t)ASTC_WARP);
		}
		WCtx wl;
		wl.lane = lane;
		wl.T = BSD.texel_count;
		i0 = wbroadcast0(wl, i0);
		if (i0 >= n) {
			break;
		}
		uint32_t i = i0 + (uint32_t)lane;
		if (i < n) {
			unsigned int b = q_load(a.queues + (size_t)Q_EMIT * a.queue_stride + i);
			const uint8_t* rec = a.records + (size_t)b * BSD.record_bytes;
			uint32_t slice = slices_base + (uint32_t)lane * EMIT_SLICE;
			const uint32_t* src = reinterpret_cast<const uint32_t*>(rec + A_SCB);
			SPtr<uint32_t> dst = sptr<uint32_t>(slice);
			ASTC_NOUNROLL
			for (int k = 0; k < EMIT_SLICE / 4; k++) {
				dst[k] = src[k];
			}
			ScbHdr scb = reinterpret_cast<const BlockSearch*>(rec + A_SEARCH)->scb;
			if (scb.block_type == SYM_BTYPE_ERROR) {
				f4 ot = reinterpret_cast<const BlkInfo*>(rec + A_STATE)->origin_texel;
				scb.block_type = SYM_BTYPE_CONST_U16;
				f4 c = vclamp4(0.0f, 1.0f, ot) * 65535.0f;
				scb.constant_color[0] = f2i_rtn(c.x);
				scb.constant_color[1] = f2i_rtn(c.y);
				scb.constant_color[2] = f2i_rtn(c.z);
				scb.constant_color[3] = f2i_rtn(c.w);
			}
			wl.base = slice - A_SCB;
			symbolic_to_physical(wl, scb, IMG.out + (size_t)b * 16);
		}
	}
}
