// libastcenc_b200: the tuning knobs of a context and the launch plan of its kernels, free of CUDA runtime calls so that the
// host tests run the same code. Included after astc_dev_search.cuh (shared-window layout, ASTC_MAX_WAVES).
#pragma once
#include <cstdlib>
#include <cstring>

#define ASTC_CTA_THREADS_MAX 512        /* single-kernel drivers: at most 16 warps */
#define ASTC_SETUP_THREADS_MAX 640      /* 20 warps x <= 102 registers (registers are granted per 4 warps: 21 warps would be charged as 24 and cap the kernel at 80) */
#ifndef ASTC_REFINE_THREADS_MAX
#define ASTC_REFINE_THREADS_MAX 768      /* 24 warps x 80 registers; 28 warps x 72 registers: 71.6 vs 71.1 ms per pass (H100 80GB HBM3 at 400 W, 4K 6x6 -medium) */
#endif
#define ASTC_CQ_BYTES (17 * 512)        /* colour quantisation tables the refine kernel can stage */
#define ASTC_MAX_PIPES 8
#define ASTC_MAX_BANDS 8

// Tuning / experiment knobs, read ONCE when the context is created (INTEGRATION.md lists them). None changes the output.
struct Knobs {
	size_t batch_blocks = (size_t)1 << 20;   // ASTCENC_B200_BATCH_BLOCKS: blocks per batch of a slab (records are reused batch after batch)
	// stage barriers of the wave kernels (bit i = i-th barrier of the kernel loop): the one in front of the endpoint-format stage
	// of the set-up kernel (bit 3) is on. With the queues sorted by cost the mask hardly matters: no barrier at all measures
	// 71.35 against 71.57 ms per pass (H100 80GB HBM3 at 400 W, 4K 6x6 -medium), inside the run-to-run spread of 71.1-71.7 ms
	unsigned int sync_mask = 8;              // ASTCENC_B200_SYNC_MASK
	unsigned int sync_mask_tail = 8;         // ASTCENC_B200_SYNC_MASK_TAIL: the waves after the first (default: the same mask)
	int coherence_probe = 0;                 // ASTCENC_B200_COHERENCE_PROBE (single-kernel driver experiment)
	int stage_print = 0;                     // ASTCENC_B200_STAGE_PRINT
	int upload_bands = 4;                    // ASTCENC_B200_UPLOAD_BANDS: bands the host-pointer path cuts an image into (1 = one copy)
	// ASTCENC_B200_PIPES: independent sub-slab pipelines of one pass (1 = the plain wave loop). 1 / 2 / 4 pipelines = 71.6 / 71.9 /
	// 73.7 ms per pass (H100 80GB HBM3 at 400 W, 4K 6x6 -medium): the idle warps are inside the CTAs, not between kernels
	int pipes = 1;
	int ctas_per_sm = 1;                     // ASTCENC_B200_CTAS_PER_SM (1 .. 8): CTAs per SM of the set-up kernels and the single-kernel driver
	int refine_ctas = 1;                     // ASTCENC_B200_REFINE_CTAS (1 .. 4): CTAs per SM of the refine kernel
	int driver = 0;                          // ASTCENC_B200_DRIVER=lockstep|warp: single kernel (1) instead of the wave pipeline (0)
	int lockstep = 1;                        //   with a phase-aligned CTA (1) or independent warps (0)
	int stage_refine = 0;                    // ASTCENC_B200_STAGE_REFINE (set): stage the tables in the refine kernel when that costs no warp
	int stage_setup = -1;                    // ASTCENC_B200_STAGE_SETUP: -1 unset (stage when it costs at most one warp), 0 never, 1 whenever it fits
	// warps per CTA as given; the plan takes them only inside its own bounds. -1 = unset (every negative value acts as unset)
	int warps = -1;                          // ASTCENC_B200_WARPS: single-kernel driver
	int warps_setup = -1;                    // ASTCENC_B200_WARPS_SETUP
	int warps_refine = -1;                   // ASTCENC_B200_WARPS_REFINE
	int warps_setup_1p = -1;                 // ASTCENC_B200_WARPS_SETUP_1P (0 = no compact plan)
};

static inline Knobs read_knobs() {
	Knobs k;
	if (const char* e = getenv("ASTCENC_B200_BATCH_BLOCKS")) {
		long v = atol(e);
		if (v > 0) k.batch_blocks = (size_t)v;
	}
	if (const char* e = getenv("ASTCENC_B200_SYNC_MASK")) {
		k.sync_mask = (unsigned int)strtoul(e, nullptr, 0);
	}
	k.sync_mask_tail = k.sync_mask;
	if (const char* e = getenv("ASTCENC_B200_SYNC_MASK_TAIL")) {
		k.sync_mask_tail = (unsigned int)strtoul(e, nullptr, 0);
	}
	k.coherence_probe = getenv("ASTCENC_B200_COHERENCE_PROBE") ? 1 : 0;
	k.stage_print = getenv("ASTCENC_B200_STAGE_PRINT") ? 1 : 0;
	// knobs with a fixed range: a value outside it keeps the default
	auto in_range = [](const char* name, int lo, int hi, int& knob) {
		if (const char* e = getenv(name)) {
			int v = atoi(e);
			if (v >= lo && v <= hi) knob = v;
		}
	};
	in_range("ASTCENC_B200_PIPES", 1, ASTC_MAX_PIPES, k.pipes);
	in_range("ASTCENC_B200_UPLOAD_BANDS", 1, ASTC_MAX_BANDS, k.upload_bands);
	in_range("ASTCENC_B200_CTAS_PER_SM", 1, 8, k.ctas_per_sm);
	in_range("ASTCENC_B200_REFINE_CTAS", 1, 4, k.refine_ctas);
	if (const char* e = getenv("ASTCENC_B200_DRIVER")) {
		if (!strcmp(e, "lockstep")) { k.driver = 1; k.lockstep = 1; }
		else if (!strcmp(e, "warp")) { k.driver = 1; k.lockstep = 0; }
	}
	k.stage_refine = getenv("ASTCENC_B200_STAGE_REFINE") ? 1 : 0;
	if (const char* e = getenv("ASTCENC_B200_STAGE_SETUP")) {
		k.stage_setup = atoi(e) != 0 ? 1 : 0;
	}
	// knobs whose bound depends on the plan: kept as given
	auto raw = [](const char* name, int& knob) {
		if (const char* e = getenv(name)) knob = atoi(e);
	};
	raw("ASTCENC_B200_WARPS", k.warps);
	raw("ASTCENC_B200_WARPS_SETUP", k.warps_setup);
	raw("ASTCENC_B200_WARPS_REFINE", k.warps_refine);
	raw("ASTCENC_B200_WARPS_SETUP_1P", k.warps_setup_1p);
	return k;
}

// Launch geometry of a compressing context's kernels.
struct KernelPlan {
	int warps_per_cta = 0;          // single-kernel driver: warps per CTA
	int grid = 0;                   // CTAs of one launch of the set-up kernels and of the single-kernel driver
	size_t smem_bytes = 0;          // single-kernel driver: shared window
	int lockstep = 1;               // single-kernel drivers: phase-aligned CTA (1) or independent warps (0)
	int driver = 0;                 // 0 = wave pipeline (default), 1 = single kernel
	int warps_setup = 0;            // warps per CTA of the set-up kernel on the general plan
	int warps_setup_1p = 0;         // set-up kernel on the compact one-plane plan (0 = plan not used)
	int warps_small = 0;            // warps per CTA of the refine kernel (the prepare kernel takes half of them)
	int refine_ctas = 1;            // CTAs per SM of the refine kernel
	size_t smem_setup = 0, smem_setup_1p = 0, smem_refine = 0;
	uint32_t setup_stage_bytes = 0;  // decimation tables staged behind the sin/cos tables of the set-up kernel's window (0 = none)
	uint32_t refine_stage_bytes = 0; // tables staged behind the header of the refine kernel's shared window (0 = none)
	int max_waves = 0;              // waves of the pipeline: a block runs at most this many trials
};

// The plan of a compressing context whose tables are `bsd` (and `bsd_1p`, the compact one-plane plan), on an SM of smem_limit bytes
// of opt-in shared memory. ASTCENC_ERR_NOT_IMPLEMENTED: the block size / preset's working set exceeds one SM's shared memory.
static inline astcenc_error plan_kernels(const DevBsd& bsd, const DevBsd& bsd_1p, const astcenc_config& cfg, size_t smem_limit, int sm_count, const Knobs& knobs,
                                         KernelPlan& p) {
	// The per-warp arena lives in shared memory only: one CTA per SM with as many warps as fit (at most 16).
	size_t arena = bsd.arena_bytes;
	int warps = (int)((smem_limit - ASTC_SMEM_HDR - ASTC_SMEM_SINCOS_BYTES) / (arena + ASTC_REFINE_STATE_BYTES));
	if (warps > ASTC_CTA_THREADS_MAX / 32) warps = ASTC_CTA_THREADS_MAX / 32;
	if (warps < 1) {
		return ASTCENC_ERR_NOT_IMPLEMENTED;
	}
	p.warps_per_cta = knobs.warps >= 1 && knobs.warps <= warps ? knobs.warps : warps;
	p.grid = sm_count * knobs.ctas_per_sm;
	p.lockstep = knobs.lockstep;
	p.driver = knobs.driver;
	p.smem_bytes = ASTC_SMEM_HDR + ASTC_SMEM_SINCOS_BYTES + (arena + ASTC_REFINE_STATE_BYTES) * p.warps_per_cta;
	// wave pipeline: the setup kernel needs the full arena, refinement / preparation only up to the union scratch
	size_t arena_small = bsd.arena_bytes_small;
	int ws = (int)((smem_limit - ASTC_SMEM_HDR - ASTC_SMEM_SINCOS_BYTES) / arena);
	if (ws > ASTC_SETUP_THREADS_MAX / 32) ws = ASTC_SETUP_THREADS_MAX / 32;
	p.refine_ctas = knobs.refine_ctas;
	// (per CTA: 1 KB of shared memory is reserved by the system)
	int wr = (int)((smem_limit / p.refine_ctas - (p.refine_ctas > 1 ? 1024 : 0) - ASTC_SMEM_HDR) / (arena_small + ASTC_REFINE_STATE_BYTES));
	if (wr > ASTC_REFINE_THREADS_MAX / 32) wr = ASTC_REFINE_THREADS_MAX / 32;
	// Staging the decimation (+ colour quantisation) tables in the refine kernel's spare shared memory is possible
	// without losing a warp at 6x6, but gains nothing (71.63 vs 71.57 ms per pass, H100 80GB HBM3 at 400 W, 4K 6x6 -medium: L1 already serves these loads): opt-in.
	size_t stage = (((size_t)bsd.dec_stage_bytes + 15) & ~(size_t)15) + ASTC_CQ_BYTES;
	p.refine_stage_bytes = 0;
	if (knobs.stage_refine && smem_limit > ASTC_SMEM_HDR + stage && (int)((smem_limit - ASTC_SMEM_HDR - stage) / (arena_small + ASTC_REFINE_STATE_BYTES)) >= wr) {
		p.refine_stage_bytes = (uint32_t)stage;
	}
	if (knobs.warps_setup >= 1 && knobs.warps_setup <= ws) ws = knobs.warps_setup;
	if (knobs.warps_refine >= 1 && knobs.warps_refine <= wr) wr = knobs.warps_refine;
	p.warps_setup = ws;
	p.warps_small = wr;
	// The set-up kernel walks the decimation tables of every grid for every block (decimated ideal weights, per-mode
	// scoring): with them in shared memory it is faster even with one warp less (6x6 medium: 21 KB of tables, 15
	// instead of 16 warps; 71.6 against 73.3 ms per pass unstaged, H100 80GB HBM3 at 400 W, 4K 6x6 -medium). Done when it costs at most one warp (ASTCENC_B200_STAGE_SETUP=0/1 forces).
	p.setup_stage_bytes = 0;
	{
		size_t st = ((size_t)bsd.dec_stage_bytes + 15) & ~(size_t)15;
		int ws2 = smem_limit > ASTC_SMEM_HDR + ASTC_SMEM_SINCOS_BYTES + st ? (int)((smem_limit - ASTC_SMEM_HDR - ASTC_SMEM_SINCOS_BYTES - st) / arena) : 0;
		bool want = ws2 >= 1 && ws2 >= ws - 1;
		if (knobs.stage_setup >= 0) {
			want = knobs.stage_setup != 0 && ws2 >= 1;
		}
		if (want) {
			if (ws2 < ws) ws = ws2;
			p.warps_setup = ws;
			p.setup_stage_bytes = (uint32_t)st;
		}
	}
	p.smem_setup = ASTC_SMEM_HDR + ASTC_SMEM_SINCOS_BYTES + p.setup_stage_bytes + arena * ws;
	// wave 0 (every block's first trial has one weight plane) runs on the compact plan: more arenas per SM
	{
		size_t arena1 = bsd_1p.arena_bytes;
		int w1 = (int)((smem_limit - ASTC_SMEM_HDR - ASTC_SMEM_SINCOS_BYTES - p.setup_stage_bytes) / arena1);
		if (w1 > ASTC_SETUP_THREADS_MAX / 32) w1 = ASTC_SETUP_THREADS_MAX / 32;
		if (knobs.warps_setup_1p >= 0 && knobs.warps_setup_1p < w1) w1 = knobs.warps_setup_1p;
		p.warps_setup_1p = w1 > ws ? w1 : 0;      // only when it buys warps
		p.smem_setup_1p = ASTC_SMEM_HDR + ASTC_SMEM_SINCOS_BYTES + p.setup_stage_bytes + arena1 * (size_t)w1;
	}
	p.smem_refine = ASTC_SMEM_HDR + p.refine_stage_bytes + arena_small * wr + (size_t)ASTC_REFINE_STATE_BYTES * wr;
	// a block runs at most this many trials (compress_block: mode-0 + full 1-plane, 4 two-plane, then the partition candidates)
	int waves = 2 + 4;
	const unsigned int cl[3] = {cfg.tune_2partitioning_candidate_limit, cfg.tune_3partitioning_candidate_limit, cfg.tune_4partitioning_candidate_limit};
	for (unsigned int pc = 2; pc <= cfg.tune_partition_count_limit && pc <= 4; pc++) {
		waves += (int)cl[pc - 2];
	}
	if (waves > ASTC_MAX_WAVES - 1) waves = ASTC_MAX_WAVES - 1;
	p.max_waves = waves;
	return ASTCENC_SUCCESS;
}
