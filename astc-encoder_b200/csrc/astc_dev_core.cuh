// CUDA-native ASTC block compressor: warp-cooperative device code, part 1
// (platform layer, block load, ideal endpoints/weights, decimated weights, angular search, weight quantisation).
//
// Execution model: ONE WARP OWNS ONE IMAGE BLOCK for its whole search. All lanes follow the same
// control flow (the decision tree only depends on the block); lanes are spread over independent
// work items (texels, grid weights, decimation grids, block modes, accumulation chains, candidate
// partitionings). Every fp32 sum whose order is fixed by the reference is computed as a *chain*: one
// lane adds the terms in the reference's order; chains run side by side in different lanes.
//
// Memory model: the whole per-warp working set is an arena in SHARED memory, addressed through 32-bit
// byte offsets (SPtr<T>) from the CTA's shared window, so every access is an LDS/STS with an immediate
// or register offset. The first ASTC_SMEM_HDR bytes of the window hold the launch constants (block-size
// descriptor + search configuration), copied there once per CTA.
// The kernel image is deliberately compact (no unrolling, few inlined copies): the search is
// instruction-fetch bound, not ALU bound, when its hot loops do not fit the SM instruction caches.
//
// The same source compiles for the host with ASTC_HOSTSIM (1 "lane", used by tests/hostsim to check
// lane-independent logic against the oracle without a GPU). It is not a product path.
#pragma once

#include <stdint.h>
#include <math.h>
#include <string.h>
#include <stddef.h>
#include "astc_dev_tables.h"

#if defined(ASTC_HOSTSIM)
	#define ASTC_FN static inline
	#define ASTC_MFN inline
	#define ASTC_NOINLINE static
	#define ASTC_COOP static
	#if defined(ASTC_HOSTSIM_LANES32)
		#define ASTC_WARP 32      /* tests/hostsim/simt_emul.h: 32 host threads stand in for the lanes */
	#else
		#define ASTC_WARP 1
		#define ASTC_ONE_LANE 1
	#endif
	#define ASTC_NOUNROLL
	#define ASTC_UNROLL_S2
	#define ASTC_UNROLL_S4
	#define ASTC_UNROLL_R2
	#define ASTC_UNROLL_R4
	#define ASTC_UNROLL_C4
	#define ASTC_UNROLL_X2
	#define ASTC_UNROLL_X4
	#define ASTC_RINT(a) nearbyintf(a)
	static inline uint32_t astc_f2u(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
	static inline float astc_u2f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
	#define ASTC_F2U(f) astc_f2u(f)
	#define ASTC_U2F(u) astc_u2f(u)
	#define ASTC_CLZ(v) __builtin_clz(v)
	#define ASTC_POPCLL(v) __builtin_popcountll(v)
	#if !defined(ASTC_LDG)      /* (a host simulation may define its own: tests/hostsim/hostsim_pack_lists.cpp checks every read) */
		#define ASTC_LDG(p) (*(p))
	#endif
	static const DevConstTables* g_astc_ct;
	#define ASTC_CT g_astc_ct
	static uint8_t* astc_smem;           // stands in for the CTA's shared window
#else
	#define ASTC_FN static __device__ __forceinline__
	#define ASTC_MFN __device__ __forceinline__
	#define ASTC_NOINLINE static __device__ __noinline__
	#define ASTC_COOP static __device__ __noinline__
	#if defined(ASTC_DEBUG_SINGLE_LANE)
		#define ASTC_WARP 1       /* debug build: lane 0 of each warp does all the work serially */
		#define ASTC_ONE_LANE 1
	#else
		#define ASTC_WARP 32
	#endif
	#if defined(ASTC_UNROLL_DEFAULT)
		#define ASTC_NOUNROLL                     /* experiment: leave loop unrolling to the compiler */
	#else
		#define ASTC_NOUNROLL _Pragma("unroll 1")
	#endif
	// The warps are latency bound (one warp issues ~1 instruction in 20 cycles): the few short loops that sit on every
	// item's critical path - an LDS feeding an ordered add, a chain of dependent table look-ups per texel - are unrolled a
	// little so that the loads of the next trips are in flight while the current one computes. Everything else stays
	// rolled: the kernels are instruction-cache sensitive (unrolling everything is much slower). Groups (ASTC_UNROLL_GROUPS): 1 set-up kernel loops, 2 refinement loops (realign / score), 4 the ordered-sum chains,
	// 8 further set-up loops.
	#ifndef ASTC_UNROLL_GROUPS
		#define ASTC_UNROLL_GROUPS 5      /* groups 1+4: 71.1 ms per pass, group 1 alone: 71.4 ms (H100 80GB HBM3 at 400 W, 4K 6x6 -medium) */
	#endif
	#define ASTC_PRAGMA_(x) _Pragma(#x)
	#define ASTC_PRAGMA(x) ASTC_PRAGMA_(x)
	#if (ASTC_UNROLL_GROUPS & 1)
		#define ASTC_UNROLL_S2 ASTC_PRAGMA(unroll 2)
		#define ASTC_UNROLL_S4 ASTC_PRAGMA(unroll 4)
	#else
		#define ASTC_UNROLL_S2 ASTC_PRAGMA(unroll 1)
		#define ASTC_UNROLL_S4 ASTC_PRAGMA(unroll 1)
	#endif
	#if (ASTC_UNROLL_GROUPS & 2)
		#define ASTC_UNROLL_R2 ASTC_PRAGMA(unroll 2)
		#define ASTC_UNROLL_R4 ASTC_PRAGMA(unroll 4)
	#else
		#define ASTC_UNROLL_R2 ASTC_PRAGMA(unroll 1)
		#define ASTC_UNROLL_R4 ASTC_PRAGMA(unroll 1)
	#endif
	#if (ASTC_UNROLL_GROUPS & 4)
		#define ASTC_UNROLL_C4 ASTC_PRAGMA(unroll 4)
	#else
		#define ASTC_UNROLL_C4 ASTC_PRAGMA(unroll 1)
	#endif
	#if (ASTC_UNROLL_GROUPS & 8)
		#define ASTC_UNROLL_X2 ASTC_PRAGMA(unroll 2)
		#define ASTC_UNROLL_X4 ASTC_PRAGMA(unroll 4)
	#else
		#define ASTC_UNROLL_X2 ASTC_PRAGMA(unroll 1)
		#define ASTC_UNROLL_X4 ASTC_PRAGMA(unroll 1)
	#endif
	#define ASTC_RINT(a) rintf(a)
	#define ASTC_F2U(f) __float_as_uint(f)
	#define ASTC_U2F(u) __uint_as_float(u)
	#define ASTC_CLZ(v) __clz((int)(v))
	#define ASTC_POPCLL(v) __popcll(v)
	#define ASTC_LDG(p) __ldg(p)
	__constant__ const DevConstTables* g_astc_ct;
	#define ASTC_CT g_astc_ct
	extern __shared__ __align__(16) uint8_t astc_smem[];
#endif

#include "astc_dev_math.cuh"

// Optional tracing of intermediate values (debug builds only: -DASTC_TRACE), printed by lane 0.
#if defined(ASTC_TRACE)
	#include <stdio.h>
	#define TRACE(...) do { if (w.lane == 0) printf(__VA_ARGS__); } while (0)
	#define TRACE_F(name, v) TRACE("%s %08x\n", name, ASTC_F2U(v))
#else
	#define TRACE(...) do { } while (0)
	#define TRACE_F(name, v) do { } while (0)
#endif

static const float ERROR_CALC_DEFAULT = 1e30f;
#define TUNE_MAX_ANGULAR_QUANT 7
#define TUNE_MAX_TRIAL_CANDIDATES 8

enum { FLG_MAP_NORMAL = 1, FLG_USE_DECODE_UNORM8 = 2, FLG_USE_ALPHA_WEIGHT = 4, FLG_USE_PERCEPTUAL = 8,
       FLG_DECOMPRESS_ONLY = 16, FLG_SELF_DECOMPRESS_ONLY = 32, FLG_MAP_RGBM = 64 };
enum { SYM_BTYPE_ERROR = 0, SYM_BTYPE_CONST_F16 = 1, SYM_BTYPE_CONST_U16 = 2, SYM_BTYPE_NONCONST = 3 };

// ---------------------------------------------------------------------------------------------
// Shared-memory pointers
// ---------------------------------------------------------------------------------------------
template <typename T> struct SPtr {
	uint32_t off;
	ASTC_MFN T& operator[](int i) const { return *reinterpret_cast<T*>(astc_smem + off + (uint32_t)i * (uint32_t)sizeof(T)); }
	ASTC_MFN SPtr<T> operator+(int n) const { SPtr<T> r; r.off = off + (uint32_t)n * (uint32_t)sizeof(T); return r; }
};
template <typename T> ASTC_FN SPtr<T> sptr(uint32_t off) { SPtr<T> r; r.off = off; return r; }

// launch constants at the start of the shared window
struct SmemHdr {
	DevBsd bsd;
	DevConfig cfg;
	DevImage img;
	// tables a kernel staged behind the header (offsets into the shared window, 0 = read them from global memory):
	// the packed decimation tables [0, bsd.dec_stage_bytes) and color_unquant_to_uquant
	uint32_t dec_smem_off;
	uint32_t cq_smem_off;
};
#define ASTC_SMEM_HDR 512
static_assert(sizeof(SmemHdr) <= ASTC_SMEM_HDR, "launch constants must fit the shared header");
// kernels that run the angular search also stage its sin/cos tables behind the header (6 KB, shared by the CTA)
#define ASTC_SMEM_SINCOS_BYTES (2 * 64 * ASTC_ANGULAR_STEPS * 4)
#define BSD (reinterpret_cast<const SmemHdr*>(astc_smem)->bsd)
#define CFG (reinterpret_cast<const SmemHdr*>(astc_smem)->cfg)
#define IMG (reinterpret_cast<const SmemHdr*>(astc_smem)->img)
#define STAGED (*reinterpret_cast<const SmemHdr*>(astc_smem))
// loads of decimation-table entries: generic, the tables may live in shared memory (staged) or in global memory
#define ASTC_LDD(p) (*(p))

#include "astc_dev_color.cuh"

// ---------------------------------------------------------------------------------------------
// Warp primitives
// ---------------------------------------------------------------------------------------------
#if defined(ASTC_ONE_LANE)
ASTC_FN void wsync() {}
ASTC_FN float wmin_f(float v) { return v; }
ASTC_FN float wmax_f(float v) { return v; }
ASTC_FN bool wall(bool p) { return p; }
ASTC_FN bool wany(bool p) { return p; }
ASTC_FN void wargmin(float& err, int& idx) {}
ASTC_FN int wsame_key_rank(int key, int lane) { (void)key; (void)lane; return 0; }
ASTC_FN int wsame_key_count(int key) { (void)key; return 1; }
ASTC_FN int wscan_incl(int v, int lane) { (void)lane; return v; }
ASTC_FN int wcount(bool p) { return p ? 1 : 0; }
#else
ASTC_FN void wsync() { __syncwarp(); }
ASTC_FN float wmin_f(float v) {
	ASTC_NOUNROLL
	for (int o = 16; o > 0; o >>= 1) {
		float t = __shfl_xor_sync(0xffffffffu, v, o);
		v = t < v ? t : v;
	}
	return v;
}
ASTC_FN float wmax_f(float v) {
	ASTC_NOUNROLL
	for (int o = 16; o > 0; o >>= 1) {
		float t = __shfl_xor_sync(0xffffffffu, v, o);
		v = t > v ? t : v;
	}
	return v;
}
ASTC_FN bool wall(bool p) { return __all_sync(0xffffffffu, p) != 0; }
ASTC_FN bool wany(bool p) { return __any_sync(0xffffffffu, p) != 0; }
// lowest error, lowest index among equal errors; every lane receives the winner
ASTC_FN void wargmin(float& err, int& idx) {
	ASTC_NOUNROLL
	for (int o = 16; o > 0; o >>= 1) {
		float e2 = __shfl_xor_sync(0xffffffffu, err, o);
		int i2 = __shfl_xor_sync(0xffffffffu, idx, o);
		bool take = (e2 < err) || (e2 == err && (unsigned int)i2 < (unsigned int)idx);
		err = take ? e2 : err;
		idx = take ? i2 : idx;
	}
}
ASTC_FN int wsame_key_rank(int key, int lane) {
	unsigned int m = __match_any_sync(0xffffffffu, key);
	return __popc(m & ((1u << lane) - 1));
}
ASTC_FN int wsame_key_count(int key) {
	return __popc(__match_any_sync(0xffffffffu, key));
}
ASTC_FN int wscan_incl(int v, int lane) {
	ASTC_NOUNROLL
	for (int o = 1; o < 32; o <<= 1) {
		int t = __shfl_up_sync(0xffffffffu, v, o);
		if (lane >= o) v += t;
	}
	return v;
}
ASTC_FN int wcount(bool p) { return __popc(__ballot_sync(0xffffffffu, p)); }
#endif

// ---------------------------------------------------------------------------------------------
// Per-warp context and arena
// ---------------------------------------------------------------------------------------------
struct WCtx;
ASTC_FN uint32_t wbroadcast0(const WCtx& w, uint32_t v) {     // lane 0's value for everybody
	(void)w;
#if defined(ASTC_ONE_LANE)
	return v;
#else
	return __shfl_sync(0xffffffffu, v, 0);
#endif
}

struct BlkInfo {
	f4 origin_texel, data_min, data_mean, data_max, channel_weight;
	uint8_t grayscale, decode_unorm8, rgb_lns0, alpha_lns0;
	uint8_t ei_const_wes[2];
	uint8_t pad[10];
	uint16_t partition_list[8];   // partition candidates of the current partition count (lockstep driver)
};

struct ScbHdr {            // scalar part of symbolic_compressed_block (arrays live in the arena)
	uint8_t block_type, partition_count, color_formats_matched;
	int8_t plane2_component;
	uint16_t block_mode, partition_index;
	uint8_t color_formats[4];
	uint8_t quant_mode;
	float errorval;
	int constant_color[4];
};

// The context is three registers and is passed by value.
struct WCtx {
	int lane;
	uint32_t base;         // byte offset of this warp's arena in the shared window
	int T;                 // texels per block
};

// Head of the arena (byte offsets from base). [0, A_PERSIST) plus the block texels at A_BLK are a block's record:
// what has to survive from one stage kernel to the next. The block-size dependent tail follows at A_BLK
// (layout planned by the host: astc_host_pack.h, offsets in DevBsd): block texels, union scratch, and - for the
// trial-setup kernel only - ideal weights, decimated weights, angular ranges, per-mode errors.
enum {
	A_STATE = 0,           // BlkInfo (112)
	A_SEARCH = 112,        // BlockSearch (128): where the block's decision tree stands
	A_TRIAL = 240,         // Trial (64): the trial in flight
	A_SCB = 304,           // best_weights[64] best_colors[32] work_weights[64] work_colors[32] mod_colors[32] (224)
	A_CAND = 528,          // Candidate[8]
	A_CANDW = 592,         // quantised weights of the candidates, 8 x 64
	A_CAND2 = 1104,        // candidates + weights of the FOLLOWING trial when one set-up serves two trials
	A_CANDW2 = 1168,       //   (the mode-0 trial and the full 1-plane trial share everything but the mode range)
	A_EP = 1680,           // f4[EP_COUNT] endpoint slots (640), the trial's base endpoints first
	A_PERSIST = ASTC_ARENA_PERSIST_HEAD,   // = A_EP + 128
	A_TMPF = 2320,         // float[128] chain results / partial sums
	A_MBAR = 2832,         // the warp's mbarrier for bulk (TMA) copies of its record (8 bytes used)
	A_BLK = ASTC_ARENA_FIXED   // float[4][Tp] block texels
};
static_assert(sizeof(BlkInfo) == 112, "BlkInfo layout");
static_assert(A_TMPF + 512 == A_MBAR && A_MBAR + 16 == A_BLK && A_EP + 128 == A_PERSIST && A_EP + 640 == A_TMPF, "arena head layout");

// endpoint slots (f4 units)
enum { EP_BASE_0 = 0, EP_BASE_1 = 4, EP_EI1_0 = 8, EP_EI1_1 = 12, EP_EI2_0 = 16, EP_EI2_1 = 20, EP_WORK_0 = 24, EP_WORK_1 = 28, EP_RGBS = 32, EP_RGBO = 36, EP_COUNT = 40 };

ASTC_FN uint32_t tp4(const WCtx& w) { return (uint32_t)((w.T + 3) & ~3) * 4u; }
ASTC_FN BlkInfo& bi_of(const WCtx& w) { return *reinterpret_cast<BlkInfo*>(astc_smem + w.base + A_STATE); }
ASTC_FN SPtr<f4> ep_of(const WCtx& w) { return sptr<f4>(w.base + A_EP); }
ASTC_FN SPtr<uint8_t> best_weights_of(const WCtx& w) { return sptr<uint8_t>(w.base + A_SCB); }
ASTC_FN SPtr<uint8_t> best_colors_of(const WCtx& w) { return sptr<uint8_t>(w.base + A_SCB + 64); }
ASTC_FN SPtr<uint8_t> work_weights_of(const WCtx& w) { return sptr<uint8_t>(w.base + A_SCB + 96); }
ASTC_FN SPtr<uint8_t> work_colors_of(const WCtx& w) { return sptr<uint8_t>(w.base + A_SCB + 160); }
ASTC_FN SPtr<uint8_t> mod_colors_of(const WCtx& w) { return sptr<uint8_t>(w.base + A_SCB + 192); }
ASTC_FN SPtr<float> tmpf_of(const WCtx& w) { return sptr<float>(w.base + A_TMPF); }
ASTC_FN SPtr<float> blk_of(const WCtx& w, int c) { return sptr<float>(w.base + A_BLK + (uint32_t)c * tp4(w)); }
ASTC_FN SPtr<float> eiw_of(const WCtx& w, int pl) { return sptr<float>(w.base + BSD.off_ei + (uint32_t)(2 * pl) * tp4(w)); }
ASTC_FN SPtr<float> eis_of(const WCtx& w, int pl) { return sptr<float>(w.base + BSD.off_ei + (uint32_t)(2 * pl + 1) * tp4(w)); }
ASTC_FN SPtr<float> dwi_of(const WCtx& w) { return sptr<float>(w.base + BSD.off_dwi); }
ASTC_FN SPtr<float> lowhigh_of(const WCtx& w) { return sptr<float>(w.base + BSD.off_lowhigh); }
ASTC_FN SPtr<float> mode_err_of(const WCtx& w) { return sptr<float>(w.base + BSD.off_mode_err); }
ASTC_FN uint32_t su_of(const WCtx& w) { return w.base + BSD.off_scratch; }

ASTC_FN float cw_lane(const WCtx& w, int c) { return reinterpret_cast<const float*>(&bi_of(w).channel_weight)[c]; }
ASTC_FN f4 texel4(const WCtx& w, int i) {
	uint32_t s = tp4(w);
	SPtr<float> b = blk_of(w, 0) + i;
	return mk4(b[0], sptr<float>(b.off + s)[0], sptr<float>(b.off + 2 * s)[0], sptr<float>(b.off + 3 * s)[0]);
}
ASTC_FN float default_alpha(const WCtx& w) { return bi_of(w).alpha_lns0 ? static_cast<float>(0x7800) : static_cast<float>(0xFFFF); }
ASTC_FN bool is_constant_channel(const WCtx& w, int ch) {
	const BlkInfo& bi = bi_of(w);
	return reinterpret_cast<const float*>(&bi.data_min)[ch] == reinterpret_cast<const float*>(&bi.data_max)[ch];
}
ASTC_FN bool is_luminance(const WCtx& w) {
	const BlkInfo& bi = bi_of(w);
	float da = default_alpha(w);
	bool alpha1 = (bi.data_min.w == da) && (bi.data_max.w == da);
	return bi.grayscale && alpha1;
}
ASTC_FN bool is_luminancealpha(const WCtx& w) {
	const BlkInfo& bi = bi_of(w);
	float da = default_alpha(w);
	bool alpha1 = (bi.data_min.w == da) && (bi.data_max.w == da);
	return bi.grayscale && !alpha1;
}

// ---------------------------------------------------------------------------------------------
// Table accessors (global memory, read-only)
// ---------------------------------------------------------------------------------------------
struct DecView {
	const float* tcf;         // [T][4] contributions as floats
	const uint32_t* twi;      // [T] 4 x u8 grid weight indices
	const uint32_t* tci;      // [T] 4 x u8 contributions in 1/16ths
	const uint16_t* wto;      // [W + 1]
	const uint16_t* wtc;      // [E] texel | contribution << 8
	int T, W, max_twc, dwi_offset;
};

ASTC_FN DecView dec_view(unsigned int d) {
	DecView v;
	const DevDecMode* dm = BSD.dec_modes + d;
	const uint8_t* blob = (STAGED.dec_smem_off != 0 ? astc_smem + STAGED.dec_smem_off : BSD.dec_blob) + ASTC_LDG(&dm->blob_offset);
	v.T = BSD.texel_count;
	v.W = ASTC_LDG(&dm->weight_count);
	v.max_twc = ASTC_LDG(&dm->max_texel_weight_count);
	v.dwi_offset = BSD.layout_planes == 1 ? ASTC_LDG(&dm->dwi_offset_1p) : ASTC_LDG(&dm->dwi_offset);
	v.tcf = reinterpret_cast<const float*>(blob);
	v.twi = reinterpret_cast<const uint32_t*>(blob + 16 * v.T);
	v.tci = reinterpret_cast<const uint32_t*>(blob + 20 * v.T);
	v.wto = reinterpret_cast<const uint16_t*>(blob + 24 * v.T);
	v.wtc = reinterpret_cast<const uint16_t*>(blob + ASTC_LDG(&dm->wtc_offset));
	return v;
}

// the four float contributions of texel t
ASTC_FN f4 dec_contribs(const DecView& di, int t) {
#if defined(ASTC_HOSTSIM)
	const float* p = di.tcf + 4 * t;
	return mk4(p[0], p[1], p[2], p[3]);
#else
	float4 v = *(reinterpret_cast<const float4*>(di.tcf) + t);
	return mk4(v.x, v.y, v.z, v.w);
#endif
}

struct PartView {
	const uint8_t* partition_of_texel;
	const uint8_t* texels;    // concatenated texels_of_partition
	unsigned int partition_count;
	unsigned int partition_index;
	uint32_t counts;          // 4 x u8 texel counts
	uint32_t starts;          // 4 x u8 first position of each partition in texels[]
};
ASTC_FN int pv_count(const PartView& v, unsigned int p) { return (int)((v.counts >> (8 * p)) & 0xFF); }
ASTC_FN int pv_start(const PartView& v, unsigned int p) { return (int)((v.starts >> (8 * p)) & 0xFF); }
// texel at position pos of the concatenated texels_of_partition lists. With one partition the list is the identity
// (partition_tables.cpp: texels_of_partition[0][i] = i), so the look-up - a dependent load in front of every per-texel
// computation of the latency-bound loops - is skipped.
ASTC_FN int pv_texel(const PartView& v, int pos) { return v.partition_count > 1 ? (int)ASTC_LDG(&v.texels[pos]) : pos; }

ASTC_FN PartView part_view_packed(unsigned int pc, unsigned int packed) {
	PartView v;
	const uint8_t* e = BSD.partitions[pc] + (size_t)packed * BSD.part_stride;
	v.partition_count = pc;
	uint32_t h0 = ASTC_LDG(reinterpret_cast<const uint32_t*>(e));
	uint32_t h1 = ASTC_LDG(reinterpret_cast<const uint32_t*>(e + 4));
	v.partition_index = h0 & 0xFFFF;
	uint32_t c0 = (h0 >> 16) & 0xFF, c1 = h0 >> 24, c2 = h1 & 0xFF, c3 = (h1 >> 8) & 0xFF;
	v.counts = c0 | (c1 << 8) | (c2 << 16) | (c3 << 24);
	v.starts = (c0 << 8) | ((c0 + c1) << 16) | ((c0 + c1 + c2) << 24);
	v.partition_of_texel = e + ASTC_PART_HDR;
	v.texels = e + ASTC_PART_HDR + BSD.texel_count;
	return v;
}

ASTC_FN unsigned int part_packed_index(unsigned int pc, unsigned int partition_index) {
	return pc >= 2 ? ASTC_LDG(&BSD.partitioning_packed_index[pc - 2][partition_index]) : 0u;
}

ASTC_FN unsigned int quant_level_count(int q) {
	// 2 3 4 5 6 8 10 12 16 20 24 32 40 48 64 80 96 128 160 192 256: (2, 3 or 5) << shift, period 3 from QUANT_4
	if (q < 4) {
		return (unsigned int)(q + 2);
	}
	unsigned int r = (unsigned int)(q - 4) % 3u, s = (unsigned int)(q - 4) / 3u;
	unsigned int b = r == 0 ? 6u : r == 1 ? 8u : 10u;
	return b << s;
}

// bits / trits / quints of a BISE level (astcenc_integer_sequence.cpp:301-327)
//   level  0 1 2 3 4 5 6 7 8 9 10 11 ...  = 2 3 4 5 6 8 10 12 16 20 24 32 ... values
//   trits at levels 1, 4, 7, ...; quints at 3, 6, 9, ...; the rest is plain bits
ASTC_FN void ise_btq(int q, unsigned int& bits, unsigned int& trits, unsigned int& quints) {
	trits = (q % 3 == 1) ? 1u : 0u;
	quints = (q >= 3 && q % 3 == 0) ? 1u : 0u;
	if (q < 4) {
		bits = q == 0 ? 1u : q == 2 ? 2u : 0u;
	} else {
		unsigned int r = (unsigned int)(q - 4) % 3u, sh = (unsigned int)(q - 4) / 3u;
		bits = (r == 1 ? 3u : 1u) + sh;   // 6,10 << sh: 1 + sh bits next to the trit / quint; 8 << sh: 3 + sh bits
	}
}

ASTC_FN unsigned int ise_sequence_bitcount(unsigned int count, int q) {   // :419-435
	unsigned int bits, trits, quints;
	ise_btq(q, bits, trits, quints);
	if (trits) return ((8 + 5 * bits) * count + 4) / 5;
	if (quints) return ((7 + 3 * bits) * count + 2) / 3;
	return bits * count;
}

// ---------------------------------------------------------------------------------------------
// Ordered sums ("chains") over a list of positions, without per-lane switches.
//   term phase : lane l of each 32-position chunk computes the K terms of position base + l and parks
//                them in a staging tile st[k * 33 + l]
//   chain phase: chain id (k, lo, hi, step) adds st[k][p] for p = lo, lo + step, ... < hi, in order.
// The running sums live in acc[id] (shared) so that more than 32 chains and the 1-lane debug build work.
// TermFn(pos, float t[K]); ChainFn(id, k, lo, hi, step).
// ---------------------------------------------------------------------------------------------
#define CHAIN_STRIDE 33
template <int K, typename TermFn, typename ChainFn>
ASTC_FN void chain_sums(const WCtx& w, int n, uint32_t tile, SPtr<float> acc, int nchains, TermFn termfn, ChainFn chainfn) {
	SPtr<float> st = sptr<float>(tile);
	ASTC_NOUNROLL
	for (int base = 0; base < n; base += 32) {
		ASTC_NOUNROLL
		for (int l = w.lane; l < 32; l += ASTC_WARP) {
			if (base + l < n) {
				float t[K];
				termfn(base + l, t);
				for (int k = 0; k < K; k++) {
					st[k * CHAIN_STRIDE + l] = t[k];
				}
			}
		}
		wsync();
		int top = n - base < 32 ? n : base + 32;
		ASTC_NOUNROLL
		for (int id = w.lane; id < nchains; id += ASTC_WARP) {
			int k, lo, hi, step;
			chainfn(id, k, lo, hi, step);
			if (hi > top) hi = top;
			// first position of this chain inside the chunk
			int p = lo;
			if (p < base) {
				p = lo + ((base - lo + step - 1) / step) * step;
			}
			float s = acc[id];
			SPtr<float> row = st + (k * CHAIN_STRIDE - base);
			ASTC_UNROLL_C4
			for (; p < hi; p += step) {
				s = s + row[p];
			}
			acc[id] = s;
		}
		wsync();
	}
}

// =============================================================================================
// Block load (astcenc_image.cpp:162-342). Lanes over texels; the per-channel mean is a chain.
// =============================================================================================
// (block_x, block_row): block coordinates; for 3D block sizes block_row counts layer * IMG.blocks_y + row and the texels of a
// block run x fastest, then y, then z (:221-270)
ASTC_COOP void load_block(WCtx w, unsigned int block_x, unsigned int block_row) {
	const DevImage& img = IMG;
	int profile = CFG.profile;
	bool needs_swz = img.swz[0] != 0 || img.swz[1] != 1 || img.swz[2] != 2 || img.swz[3] != 3;
	bool needs_hdr = profile == PRF_HDR || profile == PRF_HDR_RGB_LDR_A;
	const bool volume = BSD.dim_z > 1;
	bool fast = !needs_swz && !needs_hdr && img.data_type == 0 && !volume;      // (astcenc_entry.cpp:946-947)
	unsigned int pos_x = block_x * BSD.dim_x, pos_y = block_row * BSD.dim_y, pos_z = 0;
	if (volume) {
		unsigned int layer = block_row / img.blocks_y;
		pos_y = (block_row - layer * img.blocks_y) * BSD.dim_y;
		pos_z = layer * BSD.dim_z;
	}
	uint8_t rgb_lns = needs_hdr ? 1 : 0;
	uint8_t a_lns = profile == PRF_HDR ? 1 : 0;
	int T = w.T;
	unsigned int bx = BSD.dim_x;
	uint32_t cs = tp4(w);
	SPtr<float> b0 = blk_of(w, 0);
	SPtr<float> tmpf = tmpf_of(w);

	f4 dmin = splat4(1e38f), dmax = splat4(-1e38f);
	bool gray = true;
	ASTC_NOUNROLL
	for (int t = w.lane; t < T; t += ASTC_WARP) {
		unsigned int x = pos_x + (unsigned int)t % bx;
		unsigned int ty = (unsigned int)t / bx;
		size_t off = 0;
		if (volume) {
			unsigned int tz = ty / BSD.dim_y;
			ty -= tz * BSD.dim_y;
			unsigned int z = pos_z + tz;
			unsigned int zi = z < img.dim_z - 1 ? z : img.dim_z - 1;
			off = 4 * (size_t)img.dim_x * img.dim_y * zi;
		}
		unsigned int y = pos_y + ty;
		unsigned int xi = x < img.dim_x - 1 ? x : img.dim_x - 1;
		unsigned int yi = y < img.dim_y - 1 ? y : img.dim_y - 1;
		off += (4 * (size_t)img.dim_x * yi) + (4 * xi);
		f4 v;
		if (fast) {
			uint32_t px = ASTC_LDG(reinterpret_cast<const uint32_t*>(static_cast<const uint8_t*>(img.data) + off));
			v = mk4(static_cast<float>(px & 0xFF), static_cast<float>((px >> 8) & 0xFF), static_cast<float>((px >> 16) & 0xFF),
			        static_cast<float>(px >> 24)) * (65535.0f / 255.0f);
		} else {
			if (img.data_type == 0) {
				uint32_t px = ASTC_LDG(reinterpret_cast<const uint32_t*>(static_cast<const uint8_t*>(img.data) + off));
				v = mk4(static_cast<float>(px & 0xFF), static_cast<float>((px >> 8) & 0xFF), static_cast<float>((px >> 16) & 0xFF),
				        static_cast<float>(px >> 24)) / 255.0f;
			} else if (img.data_type == 1) {
				const uint16_t* p = static_cast<const uint16_t*>(img.data) + off;
				v = mk4(sf16_to_float(p[0]), sf16_to_float(p[1]), sf16_to_float(p[2]), sf16_to_float(p[3]));
			} else {
				const float* p = static_cast<const float*>(img.data) + off;
				v = mk4(p[0], p[1], p[2], p[3]);
			}
			if (needs_swz) {
				float s0 = img.swz[0] < 4 ? lane(v, img.swz[0]) : (img.swz[0] == 4 ? 0.0f : 1.0f);
				float s1 = img.swz[1] < 4 ? lane(v, img.swz[1]) : (img.swz[1] == 4 ? 0.0f : 1.0f);
				float s2 = img.swz[2] < 4 ? lane(v, img.swz[2]) : (img.swz[2] == 4 ? 0.0f : 1.0f);
				float s3 = img.swz[3] < 4 ? lane(v, img.swz[3]) : (img.swz[3] == 4 ? 0.0f : 1.0f);
				v = mk4(s0, s1, s2, s3);
			}
			f4 un = vclamp4(0.0f, 65535.0f, v * 65535.0f);
			if (rgb_lns || a_lns) {
				f4 l = mk4(float_to_lns(v.x), float_to_lns(v.y), float_to_lns(v.z), float_to_lns(v.w));
				v = mk4(rgb_lns ? l.x : un.x, rgb_lns ? l.y : un.y, rgb_lns ? l.z : un.z, a_lns ? l.w : un.w);
			} else {
				v = un;
			}
		}
		dmin = min4(dmin, v);
		dmax = max4(dmax, v);
		gray = gray && (v.x == v.y) && (v.x == v.z);
		SPtr<float> d = b0 + t;
		d[0] = v.x;
		sptr<float>(d.off + cs)[0] = v.y;
		sptr<float>(d.off + 2 * cs)[0] = v.z;
		sptr<float>(d.off + 3 * cs)[0] = v.w;
	}
	// block data never holds NaN (the clamps and float_to_lns flush it), so min/max are order independent
	dmin = mk4(wmin_f(dmin.x), wmin_f(dmin.y), wmin_f(dmin.z), wmin_f(dmin.w));
	dmax = mk4(wmax_f(dmax.x), wmax_f(dmax.y), wmax_f(dmax.z), wmax_f(dmax.w));
	gray = wall(gray);
	wsync();
	// per-channel mean: chain in texel order
	float mean_scale = 1.0f / static_cast<float>(T);
	ASTC_NOUNROLL
	for (int c = w.lane; c < 4; c += ASTC_WARP) {
		float s = 0.0f;
		SPtr<float> d = blk_of(w, c);
		if (fast) {
			ASTC_NOUNROLL
			for (int t = 0; t < T; t++) s = s + d[t];
			s = s / static_cast<float>(T);
		} else {
			ASTC_NOUNROLL
			for (int t = 0; t < T; t++) s = s + d[t] * mean_scale;
		}
		tmpf[c] = s;
	}
	wsync();
	if (w.lane == 0) {
		BlkInfo& bi = bi_of(w);
		bi.data_mean = mk4(tmpf[0], tmpf[1], tmpf[2], tmpf[3]);
		bi.data_min = dmin;
		bi.data_max = dmax;
		bi.grayscale = gray ? 1 : 0;
		bi.decode_unorm8 = (CFG.flags & FLG_USE_DECODE_UNORM8) != 0 ? 1 : 0;
		f4 cwt = mk4(CFG.cw[0], CFG.cw[1], CFG.cw[2], CFG.cw[3]);
		f4 enc = texel4(w, 0);
		if (fast) {
			bi.origin_texel = enc / 65535.0f;
			bi.rgb_lns0 = 0;
			bi.alpha_lns0 = 0;
		} else {
			f4 enc_unorm = enc / 65535.0f;
			f4 enc_lns = splat4(0.0f);
			if (rgb_lns || a_lns) {
				enc_lns = mk4(sf16_to_float((uint16_t)lns_to_sf16(f2i(enc.x))), sf16_to_float((uint16_t)lns_to_sf16(f2i(enc.y))),
				              sf16_to_float((uint16_t)lns_to_sf16(f2i(enc.z))), sf16_to_float((uint16_t)lns_to_sf16(f2i(enc.w))));
			}
			bi.origin_texel = mk4(rgb_lns ? enc_lns.x : enc_unorm.x, rgb_lns ? enc_lns.y : enc_unorm.y,
			                      rgb_lns ? enc_lns.z : enc_unorm.z, a_lns ? enc_lns.w : enc_unorm.w);
			bi.rgb_lns0 = rgb_lns;
			bi.alpha_lns0 = a_lns;
		}
		if (CFG.flags & FLG_USE_ALPHA_WEIGHT) {   // astcenc_entry.cpp:1017-1024
			float alpha_scale = dmax.w * (1.0f / 65535.0f);
			cwt = mk4(cwt.x * alpha_scale, cwt.y * alpha_scale, cwt.z * alpha_scale, cwt.w);
		}
		bi.channel_weight = cwt;
		bi.ei_const_wes[0] = bi.ei_const_wes[1] = 0;
	}
	wsync();
}

// =============================================================================================
// Averages and directions (astcenc_averages_and_directions.cpp:47-720)
// =============================================================================================
struct PartitionMetrics {
	f4 avg;
	f4 dir;
};

// Partition means. For >= 2 partitions the reference accumulates with masked haccumulate: texel i adds
// to lane (i mod 4) of its partition's accumulator -> one chain per (partition, channel, i mod 4).
// ncomp = 4 (rgba) or 3 (rgb, lane 3 zero).
// (S1 in this section and the next: the trial has one partition and one plane, a compile-time fact - the wave-0 set-up of an
// LDR profile inlines that instantiation, astc_dev_wave.cuh; the out-of-line function is the general one)
template <bool S1> ASTC_FN void compute_partition_averages_t(const WCtx& w, const PartView& pi, int ncomp, f4 averages[4]) {
	const unsigned int pc = S1 ? 1u : pi.partition_count;
	f4 dm = bi_of(w).data_mean;
	f4 mean = ncomp == 4 ? dm : mk4(dm.x, dm.y, dm.z, 0.0f);
	if (pc == 1) {
		averages[0] = mean;
		return;
	}
	int T = w.T;
	SPtr<float> tmpf = tmpf_of(w);
	int nchains = (int)(pc - 1) * ncomp * 4;
	ASTC_NOUNROLL
	for (int id = w.lane; id < nchains; id += ASTC_WARP) {
		int l = id & 3;
		int c = (id >> 2) % ncomp;
		unsigned int p = (unsigned int)((id >> 2) / ncomp);
		SPtr<float> d = blk_of(w, c);
		float s = 0.0f;
		ASTC_NOUNROLL
		for (int i = l; i < T; i += 4) {
			if (ASTC_LDG(&pi.partition_of_texel[i]) == p) {
				s = s + d[i];
			}
		}
		tmpf[id] = s;
	}
	wsync();
	f4 block_total = mean * static_cast<float>(T);
	f4 rest = block_total;
	for (unsigned int p = 0; p < pc - 1; p++) {
		f4 total = splat4(0.0f);
		for (int c = 0; c < ncomp; c++) {
			SPtr<float> a = tmpf + ((int)p * ncomp + c) * 4;
			set_lane(total, c, (a[0] + a[2]) + (a[1] + a[3]));
		}
		rest = rest - total;
		averages[p] = total / static_cast<float>(pv_count(pi, p));
	}
	averages[pc - 1] = rest / static_cast<float>(pv_count(pi, pc - 1));
	wsync();
}
ASTC_COOP void compute_partition_averages(WCtx w, const PartView& pi, int ncomp, f4 averages[4]) {
	compute_partition_averages_t<false>(w, pi, ncomp, averages);
}

// Sign-split direction sums: one chain per (partition, split axis K, component c), in partition-texel order.
// chan = the ncomp block channels taking part, 4 bits each (channel c of the fit is block channel (chan >> 4c) & 15).
template <bool S1> ASTC_FN void compute_dirs_t(const WCtx& w, const PartView& pi, uint32_t chan, int ncomp, const f4 averages[4], PartitionMetrics pm[4]) {
	const unsigned int pc = S1 ? 1u : pi.partition_count;
	SPtr<float> tmpf = tmpf_of(w);
	int per_part = ncomp * ncomp;
	int nchains = (int)pc * per_part;
	ASTC_NOUNROLL
	for (int id = w.lane; id < nchains; id += ASTC_WARP) {
		int p = id / per_part;
		int r = id - p * per_part;
		int K = r / ncomp;
		int c = r - K * ncomp;
		f4 av = averages[0];
		if (p == 1) av = averages[1];
		else if (p == 2) av = averages[2];
		else if (p == 3) av = averages[3];
		float avgK = lane(av, K);
		float avgc = lane(av, c);
		SPtr<float> dK = blk_of(w, (int)((chan >> (4 * K)) & 15));
		SPtr<float> dc = blk_of(w, (int)((chan >> (4 * c)) & 15));
		const uint8_t* tix = pi.texels + pv_start(pi, (unsigned int)p);
		int n = pv_count(pi, (unsigned int)p);
		float s = 0.0f;
		ASTC_UNROLL_S4
		for (int i = 0; i < n; i++) {
			int t = pc > 1 ? (int)ASTC_LDG(&tix[i]) : i;
			float vK = dK[t] - avgK;
			float vc = dc[t] - avgc;
			s = s + (vK > 0.0f ? vc : 0.0f);
		}
		tmpf[id] = s;
	}
	wsync();
	for (unsigned int p = 0; p < pc; p++) {
		SPtr<float> a = tmpf + (int)p * per_part;
		f4 best_vector = splat4(0.0f);
		float best_sum = 0.0f;
		ASTC_NOUNROLL
		for (int K = 0; K < ncomp; K++) {
			f4 sum = splat4(0.0f);
			sum.x = a[K * ncomp];
			sum.y = a[K * ncomp + 1];
			if (ncomp > 2) sum.z = a[K * ncomp + 2];
			if (ncomp > 3) sum.w = a[K * ncomp + 3];
			float prod = dot_s(sum, sum);
			if (K == 0 || prod > best_sum) {
				best_vector = sum;
				best_sum = prod;
			}
		}
		pm[p].avg = averages[p];
		pm[p].dir = best_vector;
	}
	wsync();
}
ASTC_COOP void compute_dirs(WCtx w, const PartView& pi, uint32_t chan, int ncomp, const f4 averages[4], PartitionMetrics pm[4]) {
	compute_dirs_t<false>(w, pi, chan, ncomp, averages, pm);
}

ASTC_FN uint32_t chan_list(int a, int b, int c, int d) { return (uint32_t)a | ((uint32_t)b << 4) | ((uint32_t)c << 8) | ((uint32_t)d << 12); }

template <bool S1> ASTC_FN void compute_avgs_and_dirs_4_comp_t(const WCtx& w, const PartView& pi, PartitionMetrics pm[4]) {
	f4 averages[4];
	if (S1) {
		compute_partition_averages_t<true>(w, pi, 4, averages);
		compute_dirs_t<true>(w, pi, chan_list(0, 1, 2, 3), 4, averages, pm);
	} else {
		compute_partition_averages(w, pi, 4, averages);
		compute_dirs(w, pi, chan_list(0, 1, 2, 3), 4, averages, pm);
	}
}
ASTC_COOP void compute_avgs_and_dirs_4_comp(WCtx w, const PartView& pi, PartitionMetrics pm[4]) {
	compute_avgs_and_dirs_4_comp_t<false>(w, pi, pm);
}

ASTC_COOP void compute_avgs_and_dirs_3_comp(WCtx w, const PartView& pi, unsigned int omitted, PartitionMetrics pm[4]) {
	f4 averages[4] = {splat4(0.0f), splat4(0.0f), splat4(0.0f), splat4(0.0f)};
	compute_partition_averages(w, pi, 4, averages);
	for (int i = 0; i < 4; i++) {
		f4 a = averages[i];
		if (omitted == 0) averages[i] = mk4(a.y, a.z, a.w, 0.0f);
		else if (omitted == 1) averages[i] = mk4(a.x, a.z, a.w, 0.0f);
		else if (omitted == 2) averages[i] = mk4(a.x, a.y, a.w, 0.0f);
		else averages[i] = mk4(a.x, a.y, a.z, 0.0f);
	}
	uint32_t chan = omitted == 0 ? chan_list(1, 2, 3, 3) : omitted == 1 ? chan_list(0, 2, 3, 3) : omitted == 2 ? chan_list(0, 1, 3, 3) : chan_list(0, 1, 2, 2);
	compute_dirs(w, pi, chan, 3, averages, pm);
}

template <bool S1> ASTC_FN void compute_avgs_and_dirs_3_comp_rgb_t(const WCtx& w, const PartView& pi, PartitionMetrics pm[4]) {
	f4 averages[4];
	if (S1) {
		compute_partition_averages_t<true>(w, pi, 3, averages);
		compute_dirs_t<true>(w, pi, chan_list(0, 1, 2, 2), 3, averages, pm);
	} else {
		compute_partition_averages(w, pi, 3, averages);
		compute_dirs(w, pi, chan_list(0, 1, 2, 2), 3, averages, pm);
	}
}
ASTC_COOP void compute_avgs_and_dirs_3_comp_rgb(WCtx w, const PartView& pi, PartitionMetrics pm[4]) {
	compute_avgs_and_dirs_3_comp_rgb_t<false>(w, pi, pm);
}

ASTC_COOP void compute_avgs_and_dirs_2_comp(WCtx w, const PartView& pt, unsigned int comp1, unsigned int comp2, PartitionMetrics pm[4]) {
	SPtr<float> vr = blk_of(w, (int)comp1);
	SPtr<float> vg = blk_of(w, (int)comp2);
	f4 averages[4];
	unsigned int pc = pt.partition_count;
	f4 dmean = bi_of(w).data_mean;
	// only ever called with the single-partition table (2-plane trials), keep the general form anyway
	for (unsigned int p = 0; p < pc; p++) {
		f4 average = mk4(lane(dmean, (int)comp1), lane(dmean, (int)comp2), 0.0f, 0.0f);
		if (pc > 1) {
			average = splat4(0.0f);
			unsigned int n = (unsigned int)pv_count(pt, p);
			for (unsigned int i = 0; i < n; i++) {
				unsigned int iwt = pt.texels[pv_start(pt, p) + (int)i];
				average = average + mk4(vr[(int)iwt], vg[(int)iwt], 0.0f, 0.0f);
			}
			average = average / static_cast<float>(n);
		}
		averages[p] = average;
	}
	compute_dirs(w, pt, chan_list((int)comp1, (int)comp2, (int)comp2, (int)comp2), 2, averages, pm);
}

// =============================================================================================
// Ideal endpoints and weights (astcenc_ideal_endpoints_and_weights.cpp:107-683)
// =============================================================================================
// One-component fit (:107-206). which = 0/1 selects the ei slot, epslot the endpoint slot pair.
ASTC_COOP void compute_ideal_colors_and_weights_1_comp(WCtx w, const PartView& pi, int which, int ep0slot, int ep1slot, unsigned int component) {
	unsigned int pc = pi.partition_count;
	SPtr<float> data_vr = blk_of(w, (int)component);
	float error_weight = cw_lane(w, (int)component);
	SPtr<float> weights = eiw_of(w, which);
	SPtr<float> wes = eis_of(w, which);
	SPtr<f4> ep = ep_of(w);
	bool is_constant_wes = true;
	float partition0_len_sq = 0.0f;
	ASTC_NOUNROLL
	for (unsigned int i = 0; i < pc; i++) {
		const uint8_t* tix = pi.texels + pv_start(pi, i);
		int n = pv_count(pi, i);
		float lowvalue = 1e10f, highvalue = -1e10f;
		ASTC_NOUNROLL
		for (int j = w.lane; j < n; j += ASTC_WARP) {
			float value = data_vr[pc > 1 ? (int)ASTC_LDG(&tix[j]) : j];
			lowvalue = minf(value, lowvalue);
			highvalue = maxf(value, highvalue);
		}
		lowvalue = wmin_f(lowvalue);
		highvalue = wmax_f(highvalue);
		if (highvalue <= lowvalue) {
			lowvalue = 0.0f;
			highvalue = 1e-7f;
		}
		float length = highvalue - lowvalue;
		float length_squared = length * length;
		float scale = 1.0f / length;
		if (i == 0) {
			partition0_len_sq = length_squared;
		} else {
			is_constant_wes = is_constant_wes && length_squared == partition0_len_sq;
		}
		ASTC_NOUNROLL
		for (int j = w.lane; j < n; j += ASTC_WARP) {
			int t = pc > 1 ? (int)ASTC_LDG(&tix[j]) : j;
			float value = (data_vr[t] - lowvalue) * scale;
			value = clamp1f(value);
			weights[t] = value;
			wes[t] = length_squared * error_weight;
		}
		if (w.lane == 0) {
			f4 e0 = bi_of(w).data_min, e1 = bi_of(w).data_max;
			set_lane(e0, (int)component, lowvalue);
			set_lane(e1, (int)component, highvalue);
			ep[ep0slot + (int)i] = e0;
			ep[ep1slot + (int)i] = e1;
		}
	}
	if (w.lane == 0) {
		bi_of(w).ei_const_wes[which] = is_constant_wes ? 1 : 0;
	}
	wsync();
}

// Projection on the partition lines (shared tail of the 2/3/4 component fits).
template <bool S1> ASTC_FN void ideal_project_t(const WCtx& w, const PartView& pi, int which, const PartitionMetrics pms[4], int ncomp, uint32_t chan,
                                               float error_weight, f4 lowv[4], f4 highv[4]) {
	const unsigned int pc = S1 ? 1u : pi.partition_count;
	SPtr<float> weights = eiw_of(w, which);
	SPtr<float> wes = eis_of(w, which);
	SPtr<float> c0 = blk_of(w, (int)(chan & 15)), c1 = blk_of(w, (int)((chan >> 4) & 15)), c2 = blk_of(w, (int)((chan >> 8) & 15)),
	            c3 = blk_of(w, (int)((chan >> 12) & 15));
	bool is_constant_wes = true;
	float partition0_len_sq = 0.0f;
	ASTC_NOUNROLL
	for (unsigned int i = 0; i < pc; i++) {
		f4 dir = pms[i].dir;
		float dsum = ncomp == 2 ? hadd_s(dir) : hadd_rgb_s(dir);
		if (dsum < 0.0f) {
			dir = splat4(0.0f) - dir;
		}
		f4 la = pms[i].avg;
		f4 lb = normalize_safe4(dir, ncomp == 2 ? unit2() : ncomp == 3 ? unit3() : unit4());
		const uint8_t* tix = pi.texels + pv_start(pi, i);
		int n = pv_count(pi, i);
		float lowparam = 1e10f, highparam = -1e10f;
		ASTC_NOUNROLL
		for (int j = w.lane; j < n; j += ASTC_WARP) {
			int t = pc > 1 ? (int)ASTC_LDG(&tix[j]) : j;
			f4 point = mk4(c0[t], c1[t], ncomp > 2 ? c2[t] : 0.0f, ncomp > 3 ? c3[t] : 0.0f);
			float param = ncomp == 3 ? dot3_s(point - la, lb) : dot_s(point - la, lb);
			weights[t] = param;
			lowparam = minf(param, lowparam);
			highparam = maxf(param, highparam);
		}
		// params may be NaN only if the block data is, which load_block excludes -> order independent
		lowparam = wmin_f(lowparam);
		highparam = wmax_f(highparam);
		if (highparam <= lowparam) {
			lowparam = 0.0f;
			highparam = 1e-7f;
		}
		float length = highparam - lowparam;
		float length_squared = length * length;
		float scale = 1.0f / length;
		if (i == 0) {
			partition0_len_sq = length_squared;
		} else {
			is_constant_wes = is_constant_wes && length_squared == partition0_len_sq;
		}
		wsync();
		ASTC_NOUNROLL
		for (int j = w.lane; j < n; j += ASTC_WARP) {
			int t = pc > 1 ? (int)ASTC_LDG(&tix[j]) : j;
			float idx = (weights[t] - lowparam) * scale;
			idx = clamp1f(idx);
			weights[t] = idx;
			wes[t] = length_squared * error_weight;
		}
		lowv[i] = la + lb * lowparam;
		highv[i] = la + lb * highparam;
	}
	if (w.lane == 0) {
		bi_of(w).ei_const_wes[which] = is_constant_wes ? 1 : 0;
	}
	wsync();
}
ASTC_COOP void ideal_project(WCtx w, const PartView& pi, int which, const PartitionMetrics pms[4], int ncomp, uint32_t chan, float error_weight,
                             f4 lowv[4], f4 highv[4]) {
	ideal_project_t<false>(w, pi, which, pms, ncomp, chan, error_weight, lowv, highv);
}

ASTC_COOP void compute_ideal_colors_and_weights_2_comp(WCtx w, const PartView& pi, int which, int ep0slot, int ep1slot, int comp1, int comp2) {   // :217-351
	f4 cw = bi_of(w).channel_weight;
	float error_weight = ((lane(cw, comp1) + 0.0f) + (lane(cw, comp2) + 0.0f)) / 2.0f;
	PartitionMetrics pms[4];
	compute_avgs_and_dirs_2_comp(w, pi, (unsigned int)comp1, (unsigned int)comp2, pms);
	f4 lowv[4], highv[4];
	ideal_project(w, pi, which, pms, 2, chan_list(comp1, comp2, comp2, comp2), error_weight, lowv, highv);
	SPtr<f4> ep = ep_of(w);
	for (unsigned int i = 0; i < pi.partition_count; i++) {
		f4 e0 = bi_of(w).data_min, e1 = bi_of(w).data_max;
		set_lane(e0, comp1, lowv[i].x);
		set_lane(e1, comp1, highv[i].x);
		set_lane(e0, comp2, lowv[i].y);
		set_lane(e1, comp2, highv[i].y);
		if (w.lane == 0) {
			ep[ep0slot + (int)i] = e0;
			ep[ep1slot + (int)i] = e1;
		}
	}
	wsync();
}

// (S1: only the one-plane fit without alpha, omitted = 3, reaches this instantiation)
template <bool S1> ASTC_FN void compute_ideal_colors_and_weights_3_comp_t(const WCtx& w, const PartView& pi, int which, int ep0slot, int ep1slot, unsigned int omitted_in) {
	const unsigned int omitted = S1 ? 3u : omitted_in;
	f4 cw = bi_of(w).channel_weight;
	uint32_t chan;
	float error_weight;
	if (omitted == 0) {
		error_weight = (cw.x + cw.z) + (cw.y + 0.0f);
		chan = chan_list(1, 2, 3, 3);
	} else if (omitted == 1) {
		error_weight = (cw.x + cw.w) + (cw.z + 0.0f);
		chan = chan_list(0, 2, 3, 3);
	} else if (omitted == 2) {
		error_weight = (cw.x + cw.w) + (cw.y + 0.0f);
		chan = chan_list(0, 1, 3, 3);
	} else {
		error_weight = (cw.x + cw.z) + (cw.y + 0.0f);
		chan = chan_list(0, 1, 2, 2);
	}
	error_weight = error_weight * (1.0f / 3.0f);
	PartitionMetrics pms[4];
	if (S1) {
		compute_avgs_and_dirs_3_comp_rgb_t<true>(w, pi, pms);
	} else if (omitted == 3) {
		compute_avgs_and_dirs_3_comp_rgb(w, pi, pms);
	} else {
		compute_avgs_and_dirs_3_comp(w, pi, omitted, pms);
	}
	f4 lowv[4], highv[4];
	if (S1) {
		ideal_project_t<true>(w, pi, which, pms, 3, chan, error_weight, lowv, highv);
	} else {
		ideal_project(w, pi, which, pms, 3, chan, error_weight, lowv, highv);
	}
	SPtr<f4> ep = ep_of(w);
	f4 bmin = bi_of(w).data_min, bmax = bi_of(w).data_max;
	for (unsigned int i = 0; i < (S1 ? 1u : pi.partition_count); i++) {
		f4 e0 = lowv[i], e1 = highv[i];
		f4 r0, r1;
		switch (omitted) {
		case 0: r0 = mk4(bmin.x, e0.x, e0.y, e0.z); r1 = mk4(bmax.x, e1.x, e1.y, e1.z); break;
		case 1: r0 = mk4(e0.x, bmin.y, e0.y, e0.z); r1 = mk4(e1.x, bmax.y, e1.y, e1.z); break;
		case 2: r0 = mk4(e0.x, e0.y, bmin.z, e0.z); r1 = mk4(e1.x, e1.y, bmax.z, e1.z); break;
		default: r0 = mk4(e0.x, e0.y, e0.z, bmin.w); r1 = mk4(e1.x, e1.y, e1.z, bmax.w); break;
		}
		if (w.lane == 0) {
			ep[ep0slot + (int)i] = r0;
			ep[ep1slot + (int)i] = r1;
		}
	}
	wsync();
}
ASTC_COOP void compute_ideal_colors_and_weights_3_comp(WCtx w, const PartView& pi, int which, int ep0slot, int ep1slot, unsigned int omitted) {   // :354-517
	compute_ideal_colors_and_weights_3_comp_t<false>(w, pi, which, ep0slot, ep1slot, omitted);
}

template <bool S1> ASTC_FN void compute_ideal_colors_and_weights_4_comp_t(const WCtx& w, const PartView& pi, int which, int ep0slot, int ep1slot) {
	float error_weight = hadd_s(bi_of(w).channel_weight) / 4.0f;
	PartitionMetrics pms[4];
	f4 lowv[4], highv[4];
	if (S1) {
		compute_avgs_and_dirs_4_comp_t<true>(w, pi, pms);
		ideal_project_t<true>(w, pi, which, pms, 4, chan_list(0, 1, 2, 3), error_weight, lowv, highv);
	} else {
		compute_avgs_and_dirs_4_comp(w, pi, pms);
		ideal_project(w, pi, which, pms, 4, chan_list(0, 1, 2, 3), error_weight, lowv, highv);
	}
	SPtr<f4> ep = ep_of(w);
	for (unsigned int i = 0; i < (S1 ? 1u : pi.partition_count); i++) {
		if (w.lane == 0) {
			ep[ep0slot + (int)i] = lowv[i];
			ep[ep1slot + (int)i] = highv[i];
		}
	}
	wsync();
}
ASTC_COOP void compute_ideal_colors_and_weights_4_comp(WCtx w, const PartView& pi, int which, int ep0slot, int ep1slot) {   // :520-609
	compute_ideal_colors_and_weights_4_comp_t<false>(w, pi, which, ep0slot, ep1slot);
}

// S1: pi is the one-partition view
template <bool S1> ASTC_FN void compute_ideal_colors_and_weights_1plane_t(const WCtx& w, const PartView& pi) {   // :612-627
	bool uses_alpha = !is_constant_channel(w, 3);
	if (S1) {
		if (uses_alpha) {
			compute_ideal_colors_and_weights_4_comp_t<true>(w, pi, 0, EP_EI1_0, EP_EI1_1);
		} else {
			compute_ideal_colors_and_weights_3_comp_t<true>(w, pi, 0, EP_EI1_0, EP_EI1_1, 3);
		}
	} else if (uses_alpha) {
		compute_ideal_colors_and_weights_4_comp(w, pi, 0, EP_EI1_0, EP_EI1_1);
	} else {
		compute_ideal_colors_and_weights_3_comp(w, pi, 0, EP_EI1_0, EP_EI1_1, 3);
	}
}
ASTC_COOP void compute_ideal_colors_and_weights_1plane(WCtx w, const PartView& pi) {
	compute_ideal_colors_and_weights_1plane_t<false>(w, pi);
}

ASTC_COOP void compute_ideal_colors_and_weights_2planes(WCtx w, unsigned int plane2_component) {   // :630-683
	PartView pi = part_view_packed(1, 0);
	bool uses_alpha = !is_constant_channel(w, 3);
	if (plane2_component == 3 || uses_alpha) {
		compute_ideal_colors_and_weights_3_comp(w, pi, 0, EP_EI1_0, EP_EI1_1, plane2_component);
	} else {
		int c1 = plane2_component == 0 ? 1 : 0;
		int c2 = plane2_component == 2 ? 1 : 2;
		compute_ideal_colors_and_weights_2_comp(w, pi, 0, EP_EI1_0, EP_EI1_1, c1, c2);
	}
	compute_ideal_colors_and_weights_1_comp(w, pi, 1, EP_EI2_0, EP_EI2_1, plane2_component);
}

// bilinear infill (:38-104): (w0*c0 + w1*c1) + (w2*c2 + w3*c3); contributions are exact multiples of 1/16.
// Grids whose texels touch at most two weights skip the second pair in the reference; adding its (+0.0 + +0.0)
// here leaves the non-negative sum unchanged bit for bit, so one form serves every grid.
ASTC_FN float bilinear_infill(const DecView& di, SPtr<float> weights, int t) {
	uint32_t ix = ASTC_LDD(&di.twi[t]);
	f4 c = dec_contribs(di, t);
	return (weights[(int)(ix & 0xFF)] * c.x + weights[(int)((ix >> 8) & 0xFF)] * c.y) +
	       (weights[(int)((ix >> 16) & 0xFF)] * c.z + weights[(int)(ix >> 24)] * c.w);
}

// compute_ideal_weights_for_decimation (:845-971) for one grid; nplanes = 1 or 2 (second plane: ei slot 1,
// output W floats further on). Lanes over grid weights / texels; the per-weight sums are chains.
template <bool S1> ASTC_FN void compute_ideal_weights_for_decimation_t(const WCtx& w, unsigned int d, int nplanes_in) {
	const int nplanes = S1 ? 1 : nplanes_in;
	DecView di = dec_view(d);
	int T = di.T;
	int W = di.W;
	SPtr<float> out = dwi_of(w) + di.dwi_offset;
	SPtr<float> eiw0 = eiw_of(w, 0);
	uint32_t plane_stride = 2 * tp4(w);           // eiw[1] - eiw[0] == eis[1] - eis[0] in bytes
	uint32_t wes_off = tp4(w);                    // eis[pl] - eiw[pl]
	if (T == W) {
		ASTC_NOUNROLL
		for (int i = w.lane; i < T * nplanes; i += ASTC_WARP) {
			int pl = i >= T ? 1 : 0;
			int t = i - pl * T;
			out[pl * W + t] = sptr<float>(eiw0.off + (uint32_t)pl * plane_stride)[t];
		}
		wsync();
		return;
	}
	SPtr<float> infilled = sptr<float>(su_of(w));   // [nplanes][T]
	const BlkInfo& bi = bi_of(w);
	ASTC_NOUNROLL
	for (int id = w.lane; id < W * nplanes; id += ASTC_WARP) {
		int pl = id >= W ? 1 : 0;
		int i = id - pl * W;
		SPtr<float> eiw = sptr<float>(eiw0.off + (uint32_t)pl * plane_stride);
		SPtr<float> eis = sptr<float>(eiw.off + wes_off);
		bool constant_wes = bi.ei_const_wes[pl] != 0;
		float wes0 = eis[0];
		float weight_weight = 1e-10f;
		float initial_weight = 0.0f;
		int off = ASTC_LDD(&di.wto[i]);
		int end = ASTC_LDD(&di.wto[i + 1]);
		ASTC_UNROLL_S4
		for (int j = off; j < end; j++) {
			uint32_t e = ASTC_LDD(&di.wtc[j]);
			int texel = (int)(e & 0xFF);
			float weight = static_cast<float>(e >> 8);
			float wes = constant_wes ? wes0 : eis[texel];
			float contrib_weight = weight * wes;
			weight_weight += contrib_weight;
			initial_weight += eiw[texel] * contrib_weight;
		}
		out[id] = initial_weight / weight_weight;
	}
	wsync();
	ASTC_NOUNROLL
	for (int id = w.lane; id < T * nplanes; id += ASTC_WARP) {
		int pl = id >= T ? 1 : 0;
		int t = id - pl * T;
		infilled[id] = bilinear_infill(di, out + pl * W, t);
	}
	wsync();
	const float stepsize = 0.25f;
	const float chd_scale = -16.0f;
	ASTC_NOUNROLL
	for (int id = w.lane; id < W * nplanes; id += ASTC_WARP) {
		int pl = id >= W ? 1 : 0;
		int i = id - pl * W;
		SPtr<float> eiw = sptr<float>(eiw0.off + (uint32_t)pl * plane_stride);
		SPtr<float> eis = sptr<float>(eiw.off + wes_off);
		SPtr<float> inf = infilled + pl * T;
		bool constant_wes = bi.ei_const_wes[pl] != 0;
		float wes0 = eis[0];
		float weight_val = out[id];
		float error_change0 = 1e-10f;
		float error_change1 = 0.0f;
		int off = ASTC_LDD(&di.wto[i]);
		int end = ASTC_LDD(&di.wto[i + 1]);
		ASTC_UNROLL_S4
		for (int j = off; j < end; j++) {
			uint32_t e = ASTC_LDD(&di.wtc[j]);
			int texel = (int)(e & 0xFF);
			float contrib_weight = static_cast<float>(e >> 8);
			float wes = constant_wes ? wes0 : eis[texel];
			float scale = wes * contrib_weight;
			float old_weight = inf[texel];
			float ideal_weight = eiw[texel];
			error_change0 += contrib_weight * scale;
			error_change1 += (old_weight - ideal_weight) * scale;
		}
		float step = (error_change1 * chd_scale) / error_change0;
		step = vclampf(-stepsize, stepsize, step);
		out[id] = weight_val + step;
	}
	wsync();
}
ASTC_COOP void compute_ideal_weights_for_decimation(WCtx w, unsigned int d, int nplanes) {
	compute_ideal_weights_for_decimation_t<false>(w, d, nplanes);
}

// =============================================================================================
// Angular weight-range search (astcenc_weight_align.cpp:94-355).
// Work items are (grid, plane, angular step) triples, compacted so that every lane has one:
//   setup  : lanes over (grid, plane) pairs: step count, weight min/max, prefix sum -> item ranges
//   phase 1: lanes over items: walk the grid's weights twice (offset sums, then error / cut sums - all
//            chains in weight order) and park six results per step in scratch
//   phase 2: lanes over pairs replay the reference's sequential best-of scan over the pair's steps.
// Pairs are taken in rounds of up to 32 whose items fit the scratch.
// =============================================================================================
struct alignas(8) AngStep {
	float offset, minidx, error, cut_low_err, cut_high_err;
	int span;
};

ASTC_FN int steps_for_quant_level(unsigned int q) {     // 2 3 4 5 6 8 10 12 16 20 24 32
	return (int)quant_level_count((int)q);
}

// decimation mode d: is it searched in this trial, and with how many angular steps?
ASTC_FN int angular_steps_of(unsigned int d, int nplanes, uint16_t mask, unsigned int max_weight_quant, unsigned int& max_precision_out) {
	const DevDecMode* dm = BSD.dec_modes + d;
	uint16_t ref = nplanes == 1 ? ASTC_LDG(&dm->refprec_1plane) : ASTC_LDG(&dm->refprec_2planes);
	max_precision_out = 0;
	if ((ref & mask) == 0) {
		return 0;
	}
	unsigned int max_precision = (unsigned int)(nplanes == 1 ? ASTC_LDG(&dm->maxprec_1plane) : ASTC_LDG(&dm->maxprec_2planes));
	if (max_precision > TUNE_MAX_ANGULAR_QUANT) max_precision = TUNE_MAX_ANGULAR_QUANT;
	if (max_precision > max_weight_quant) max_precision = max_weight_quant;
	max_precision_out = max_precision;
	return steps_for_quant_level(max_precision);
}

// compute_angular_endpoints_1plane / _2planes (:358-500)
template <bool S1> ASTC_FN void compute_angular_endpoints_t(const WCtx& w, bool only_always, int nplanes_in, unsigned int max_weight_quant) {
	const int nplanes = S1 ? 1 : nplanes_in;
	unsigned int max_dm = (nplanes == 1 && only_always) ? BSD.decimation_mode_count_always : BSD.decimation_mode_count_selected;
	uint16_t mask = (uint16_t)((1u << (max_weight_quant + 1)) - 1);
	int pairs = (int)max_dm * nplanes;
	SPtr<float> dwi = dwi_of(w);
	SPtr<float> lowhigh = lowhigh_of(w);
	const float mult = 1.0f / (2.0f * 3.14159265358979323846f);

	// scratch: isamp u8[dwi floats] | pmin[32] pmax[32] | pfirst u8[32] | map u8[cap] | rec AngStep[cap]
	int ndwi = (int)((BSD.off_lowhigh - BSD.off_dwi) >> 2);
	uint32_t so = su_of(w);
	SPtr<uint8_t> isamp = sptr<uint8_t>(so);
	so += (uint32_t)((ndwi + 15) & ~15);
	SPtr<float> pmin = sptr<float>(so);
	SPtr<float> pmax = sptr<float>(so + 128);
	SPtr<uint8_t> pfirst = sptr<uint8_t>(so + 256);
	so += 288;
	int cap = (int)((su_of(w) + BSD.scratch_bytes - so) / 25u) & ~7;
	if (cap > 240) cap = 240;
	SPtr<uint8_t> map = sptr<uint8_t>(so);
	SPtr<AngStep> rec = sptr<AngStep>(so + (uint32_t)cap);

	// the table row of every decimated ideal weight (stale slots of unsearched grids convert harmlessly)
	ASTC_NOUNROLL
	for (int i = w.lane; i < ndwi; i += ASTC_WARP) {
		float sample = clampzo(dwi[i]) * (64 - 1.0f);
		isamp[i] = (uint8_t)(f2i_rtn(sample) & 63);
	}
	wsync();

	int pair0 = 0;
	ASTC_NOUNROLL
	while (pair0 < pairs) {
		// setup: one lane per pair of this round
		int id = pair0 + (ASTC_WARP == 1 ? 0 : w.lane);
		int steps = 0, d = 0, pl = 0, W = 0, doff = 0;
		unsigned int max_precision = 0;
		if (id < pairs) {
			d = id / nplanes;
			pl = id - d * nplanes;
			steps = angular_steps_of((unsigned int)d, nplanes, mask, max_weight_quant, max_precision);
			const DevDecMode* dm = BSD.dec_modes + d;
			W = ASTC_LDG(&dm->weight_count);
			doff = (int)(BSD.layout_planes == 1 ? ASTC_LDG(&dm->dwi_offset_1p) : ASTC_LDG(&dm->dwi_offset)) + pl * W;
		}
		int incl = wscan_incl(steps, w.lane);
		bool in_round = id < pairs && incl <= cap;
		int npair = wcount(id < pairs && incl <= cap);      // a prefix of the lanes (incl is monotone)
		int nitems = 0;
#if defined(ASTC_ONE_LANE)
		nitems = incl;
#else
		nitems = __shfl_sync(0xffffffffu, incl, npair - 1);
#endif
		int first = incl - steps;
		if (in_round) {
			float mn = 3.402823466e+38f, mx = -3.402823466e+38f;
			if (steps != 0) {
				SPtr<float> v = dwi + doff;
				ASTC_UNROLL_X4
				for (int i = 0; i < W; i++) {
					float x = v[i];
					mn = minf(x, mn);
					mx = maxf(x, mx);
				}
			}
			int L = ASTC_WARP == 1 ? 0 : w.lane;
			pmin[L] = mn;
			pmax[L] = mx;
			pfirst[L] = (uint8_t)first;
			ASTC_NOUNROLL
			for (int s = 0; s < steps; s++) {
				map[first + s] = (uint8_t)L;
			}
		}
		wsync();
		// phase 1
		ASTC_NOUNROLL
		for (int it = w.lane; it < nitems; it += ASTC_WARP) {
			int pr = map[it];
			int sp = it - pfirst[pr];
			int pid = pair0 + pr;
			int pd = pid / nplanes;
			int ppl = pid - pd * nplanes;
			const DevDecMode* dm = BSD.dec_modes + pd;
			int pW = ASTC_LDG(&dm->weight_count);
			int pdoff = (int)(BSD.layout_planes == 1 ? ASTC_LDG(&dm->dwi_offset_1p) : ASTC_LDG(&dm->dwi_offset)) + ppl * pW;
			unsigned int mp;
			int psteps = angular_steps_of((unsigned int)pd, nplanes, mask, max_weight_quant, mp);
			SPtr<float> v = dwi + pdoff;
			SPtr<uint8_t> is = isamp + pdoff;
			// compute_angular_offsets :94-157
			float anglesum_x = 0.0f, anglesum_y = 0.0f;
			SPtr<float> cosp = sptr<float>(ASTC_SMEM_HDR) + sp;
			SPtr<float> sinp = cosp + 64 * ASTC_ANGULAR_STEPS;
			ASTC_UNROLL_S4
			for (int j = 0; j < pW; j++) {
				int row = is[j] * ASTC_ANGULAR_STEPS;
				anglesum_x += cosp[row];
				anglesum_y += sinp[row];
			}
			float angle = approx_atan2(anglesum_y, anglesum_x);
			angle = (angle == angle) ? angle : 0.0f;
			float offset = angle * mult;
			// compute_lowest_and_highest_weight :160-253
			float rcp_stepsize = static_cast<float>(sp) + 1.0f;
			float minidx = ASTC_RINT(pmin[pr] * rcp_stepsize - offset);
			float maxidx = ASTC_RINT(pmax[pr] * rcp_stepsize - offset);
			float errval = 0.0f, cut_low = 0.0f, cut_high = 0.0f;
			ASTC_UNROLL_S4
			for (int j = 0; j < pW; j++) {
				float sval = v[j] * rcp_stepsize - offset;
				float svalrte = ASTC_RINT(sval);
				float diff = sval - svalrte;
				errval += diff * diff;
				if (svalrte == minidx) {
					cut_low = cut_low + 1.0f - 2.0f * diff;
				}
				if (svalrte == maxidx) {
					cut_high = cut_high + 1.0f + 2.0f * diff;
				}
			}
			int span = f2i(maxidx - minidx + 1.0f);
			span = mini(span, psteps + 3);
			span = maxi(span, 2);
			float ssize = 1.0f / rcp_stepsize;
			float errscale = ssize * ssize;
			AngStep r;
			r.offset = offset;
			r.minidx = minidx;
			r.error = errval * errscale;
			r.cut_low_err = cut_low * errscale;
			r.cut_high_err = cut_high * errscale;
			r.span = span;
			rec[it] = r;
		}
		wsync();
		// phase 2 (:298-355): the reference walks a pair's steps once and keeps, per span bucket, the best
		// (error, step, cut) in three arrays; only the buckets of the quant levels 0..max_precision are ever read. Here one
		// lane owns one (pair, quant level): it scans the pair's step records for ITS bucket in the same order with the
		// same strict comparisons, so it ends with exactly the entry the arrays would hold - in registers, all lanes busy.
		{
			int nitems2 = npair * 8;
			ASTC_NOUNROLL
			for (int it0 = 0; it0 < nitems2; it0 += ASTC_WARP) {
#if defined(ASTC_ONE_LANE)
				ASTC_NOUNROLL
				for (int it = it0; it < nitems2; it++) {
				int qi = it & 7;
				int p_steps = steps, p_first = first, p_d = d, p_pl = pl;
				unsigned int p_mp = max_precision;
				bool act = true;
#else
				{
				int it = it0 + w.lane;
				int qi = it & 7;
				bool act = it < nitems2;
				int src = act ? (it >> 3) : 0;
				int p_steps = __shfl_sync(0xffffffffu, steps, src);
				int p_first = __shfl_sync(0xffffffffu, first, src);
				int p_d = __shfl_sync(0xffffffffu, d, src);
				int p_pl = __shfl_sync(0xffffffffu, pl, src);
				unsigned int p_mp = __shfl_sync(0xffffffffu, max_precision, src);
#endif
				if (act && p_steps != 0 && (unsigned int)qi <= p_mp) {
					int q = steps_for_quant_level((unsigned int)qi);
					float best = ERROR_CALC_DEFAULT;
					int bidx = -1;
					float bcut = 0.0f;
					SPtr<AngStep> rp = rec + p_first;
					ASTC_UNROLL_X2
					for (int sp = 0; sp < p_steps; sp++) {
						AngStep r = rp[sp];
						int span = r.span;
						float error = r.error;
						if (span == q) {
							if (best > error) {
								best = error;
								bidx = sp;
								bcut = 0.0f;
							}
						} else if (span - 1 == q) {
							float error_cut_low = error + r.cut_low_err;
							float error_cut_high = error + r.cut_high_err;
							if (best > error_cut_low) {
								best = error_cut_low;
								bidx = sp;
								bcut = 1.0f;
							}
							if (best > error_cut_high) {
								best = error_cut_high;
								bidx = sp;
								bcut = 0.0f;
							}
						} else if (span - 2 == q) {
							float error_cut_low_high = error + r.cut_low_err + r.cut_high_err;
							if (best > error_cut_low_high) {
								best = error_cut_low_high;
								bidx = sp;
								bcut = 1.0f;
							}
						}
					}
					int bsi = maxi(0, bidx);
					AngStep r = rp[bsi];
					float lwi = r.minidx + bcut;
					float hwi = lwi + static_cast<float>(q) - 1.0f;
					float stepsize = 1.0f / (1.0f + static_cast<float>(bsi));
					SPtr<float> lh = lowhigh + (p_d * (int)BSD.layout_planes + p_pl) * 16;
					lh[2 * qi] = (r.offset + lwi) * stepsize;
					lh[2 * qi + 1] = (r.offset + hwi) * stepsize;
				}
				}
			}
		}
		wsync();
		pair0 += npair;
	}
}
ASTC_COOP void compute_angular_endpoints(WCtx w, bool only_always, int nplanes, unsigned int max_weight_quant) {
	compute_angular_endpoints_t<false>(w, only_always, nplanes, max_weight_quant);
}

// The (low, high) weight range of a packed block mode, including the "snap high to 1.0" rule of
// astcenc_compress_symbolic.cpp:459 / :819-827.
ASTC_FN void mode_low_high(const WCtx& w, int decimation_mode, int quant_mode, int plane, float min_wt_cutoff, float& low, float& high) {
	if (quant_mode <= TUNE_MAX_ANGULAR_QUANT) {
		SPtr<float> lh = lowhigh_of(w) + ((decimation_mode * (int)BSD.layout_planes + plane) * 16 + quant_mode * 2);
		low = lh[0];
		high = lh[1];
	} else {
		low = 0.0f;
		high = 1.0f;
	}
	if (high > 1.02f * min_wt_cutoff) {
		high = 1.0f;
	}
}

// compute_quantized_weights_for_decimation (:974-1080), one weight
struct WeightQuantizer {
	float scale, scaled_low_bound, quant_level_m1, rscale, low_bound;
	int steps_m1;
	const uint8_t* q2u;
};

ASTC_FN WeightQuantizer make_weight_quantizer(float low_bound, float high_bound, int quant_level) {
	WeightQuantizer z;
	z.steps_m1 = (int)quant_level_count(quant_level) - 1;
	z.quant_level_m1 = static_cast<float>(z.steps_m1);
	if (high_bound <= low_bound) {
		low_bound = 0.0f;
		high_bound = 1.0f;
	}
	float rscale = high_bound - low_bound;
	z.scale = 1.0f / rscale;
	z.scaled_low_bound = low_bound * z.scale;
	z.rscale = rscale * (1.0f / 64.0f);
	z.low_bound = low_bound;
	z.q2u = ASTC_CT->wq_quant_to_unquant[quant_level];
	return z;
}

ASTC_FN int quantize_weight(const WeightQuantizer& z, float ideal) {
	float ix = ideal * z.scale - z.scaled_low_bound;
	ix = clampzo(ix);
	float ix1 = ix * z.quant_level_m1;
	int weightl = f2i(ix1);
	int weighth = mini(weightl + 1, z.steps_m1);
	int ixli = ASTC_LDG(&z.q2u[weightl]);
	int ixhi = ASTC_LDG(&z.q2u[weighth]);
	float ixl = static_cast<float>(ixli);
	float ixh = static_cast<float>(ixhi);
	bool mask = (ixl + ixh) < (128.0f * ix);
	return mask ? ixhi : ixli;
}
ASTC_FN float quantized_weight_value(const WeightQuantizer& z, int uq) {
	return static_cast<float>(uq) * z.rscale + z.low_bound;
}
