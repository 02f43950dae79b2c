// libastcenc_b200: the astcenc.h C ABI on top of hand-written sm_90a (H100) kernels.
//
// Host side of the drop-in boundary. Behavioural spec: /root/reference/Source/astcenc_entry.cpp
//   astcenc_context_alloc :726-860, astcenc_compress_image :1113-1228 (check order :1134-1182),
//   astcenc_compress_reset :1231, astcenc_compress_cancel :1251, astcenc_context_free :862,
//   ParallelManager protocol astcenc_internal_entry.h:97-324 (N callers, first arrival initialises,
//   everyone returns when the image is done).
// There is deliberately no CPU compression path in this library: without a usable CUDA device
// astcenc_context_alloc() fails (ASTCENC_ERR_BAD_CONTEXT) instead of falling back.
#include <cuda_runtime.h>
#include <mutex>
#include <condition_variable>
#include <atomic>
#include <vector>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cstddef>
#include <new>
#include <thread>
#include <chrono>

#include "astc_dev_search.cuh"
#include "astc_dev_metrics.cuh"
#include "astc_dev_gather.cuh"
#include "astc_host_pack.h"
#include "astc_host_config.h"

// ---------------------------------------------------------------------------------------------
// The kernel: persistent warps, one block per warp at a time, dynamic ticket scheduling (the GPU analogue
// of the reference's ParallelManager::get_task_assignment ticket counter).
// ---------------------------------------------------------------------------------------------
#define ASTC_CTA_THREADS_MAX 512

// Shared window: [0, ASTC_SMEM_HDR) launch constants, then one arena per warp.
static __device__ __forceinline__ void stage_launch_constants(const DevBsd& bsd, const DevConfig& cfg, const DevImage& img) {
	// all threads help copy the launch constants from the parameter bank
	uint32_t* dst = reinterpret_cast<uint32_t*>(astc_smem);
	const uint32_t* s0 = reinterpret_cast<const uint32_t*>(&bsd);
	const uint32_t* s1 = reinterpret_cast<const uint32_t*>(&cfg);
	const uint32_t* s2 = reinterpret_cast<const uint32_t*>(&img);
	for (unsigned int i = threadIdx.x; i < sizeof(DevBsd) / 4; i += blockDim.x) {
		dst[offsetof(SmemHdr, bsd) / 4 + i] = s0[i];
	}
	for (unsigned int i = threadIdx.x; i < sizeof(DevConfig) / 4; i += blockDim.x) {
		dst[offsetof(SmemHdr, cfg) / 4 + i] = s1[i];
	}
	for (unsigned int i = threadIdx.x; i < sizeof(DevImage) / 4; i += blockDim.x) {
		dst[offsetof(SmemHdr, img) / 4 + i] = s2[i];
	}
	if (threadIdx.x == 0) {
		dst[offsetof(SmemHdr, dec_smem_off) / 4] = 0;
		dst[offsetof(SmemHdr, cq_smem_off) / 4] = 0;
	}
	__syncthreads();
}

// Refinement reads the packed decimation tables (infill in every score / refit / realignment) and, from single lanes in
// long dependent chains, the colour quantisation tables; its arenas leave ~50 KB of the shared window free at 6x6, so
// both are copied behind the header once per CTA and read from there (when they fit without costing a warp).
#define ASTC_CQ_BYTES (17 * 512)
static __device__ __forceinline__ void stage_tables(uint32_t stage_bytes, uint32_t at, bool with_colour) {
	if (stage_bytes == 0) {
		return;
	}
	const DevBsd& bsd = BSD;
	uint32_t dec_bytes = (bsd.dec_stage_bytes + 15u) & ~15u;
	uint4* dst = reinterpret_cast<uint4*>(astc_smem + at);
	const uint4* src = reinterpret_cast<const uint4*>(bsd.dec_blob);
	for (unsigned int i = threadIdx.x; i < dec_bytes / 16; i += blockDim.x) {
		dst[i] = __ldg(src + i);
	}
	if (with_colour) {
		uint4* dst2 = reinterpret_cast<uint4*>(astc_smem + at + dec_bytes);
		const uint4* src2 = reinterpret_cast<const uint4*>(&ASTC_CT->color_unquant_to_uquant[0][0]);
		for (unsigned int i = threadIdx.x; i < ASTC_CQ_BYTES / 16; i += blockDim.x) {
			dst2[i] = __ldg(src2 + i);
		}
	}
	if (threadIdx.x == 0) {
		uint32_t* hdr = reinterpret_cast<uint32_t*>(astc_smem);
		hdr[offsetof(SmemHdr, dec_smem_off) / 4] = at;
		if (with_colour) {
			hdr[offsetof(SmemHdr, cq_smem_off) / 4] = at + dec_bytes;
		}
	}
	__syncthreads();
}

// cos_table then sin_table, [64][ASTC_ANGULAR_STEPS] each, right behind the header (kernels that run the angular search)
static __device__ __forceinline__ void stage_sincos_tables() {
	float* dst = reinterpret_cast<float*>(astc_smem + ASTC_SMEM_HDR);
	const DevConstTables* ct = ASTC_CT;
	const float* c = &ct->cos_table[0][0];
	const float* sn = &ct->sin_table[0][0];
	for (unsigned int i = threadIdx.x; i < 64 * ASTC_ANGULAR_STEPS; i += blockDim.x) {
		dst[i] = __ldg(c + i);
		dst[64 * ASTC_ANGULAR_STEPS + i] = __ldg(sn + i);
	}
	__syncthreads();
}

// ---- the stage kernels of the wave pipeline (astc_dev_wave.cuh) ----
// nothing queued in any class of this kind for the launch's wave?
static __device__ __forceinline__ bool wave_queue_empty(const WaveArgs& a, int kind, int c0 = 0, int c1 = ASTC_Q_CLASSES) {
	uint32_t n = 0;
	for (int c = c0; c < c1; c++) {
		n += __ldcg(a.count + (kind + c) * ASTC_MAX_WAVES + a.wave);
	}
	return n == 0;
}
// (the set-up classes have ASTC_Q_SUB sub-queues each; a thread per sub-queue looks, the CTA votes)
static __device__ __forceinline__ bool wave_setup_queues_empty(const WaveArgs& a) {
	bool any = false;
	for (int k = a.cls_lo * ASTC_Q_SUB + (int)threadIdx.x; k < a.cls_hi * ASTC_Q_SUB; k += (int)blockDim.x) {
		any = any || __ldcg(a.count + (Q_SETUP + k) * ASTC_MAX_WAVES + a.wave) != 0;
	}
	return __syncthreads_or(any ? 1 : 0) == 0;
}

#define ASTC_SETUP_THREADS_MAX 640      /* 20 warps x <= 102 registers (registers are granted per 4 warps: 21 warps would be charged as 24 and cap the kernel at 80) */
#ifndef ASTC_REFINE_THREADS_MAX
#define ASTC_REFINE_THREADS_MAX 768      /* 24 warps x 80 registers; 28 warps x 72 registers: 71.6 vs 71.1 ms per pass (H100 80GB HBM3 at 400 W, 4K 6x6 -medium) */
#endif
#define ASTC_EMIT_THREADS 256

// Two instantiations: S1 = true for the wave-0 launches of the LDR profiles (the first trial of every block, one partition and
// one plane, runs the specialised set-up stages inlined beside the general ones), false for every later wave and for the HDR
// profiles - their kernel carries the general stages alone, laid out as it was before the specialised stages existed.
template <bool S1>
__global__ void __launch_bounds__(ASTC_SETUP_THREADS_MAX, 1)
astc_wave_setup_kernel(const __grid_constant__ DevBsd bsd, const __grid_constant__ DevConfig cfg, const __grid_constant__ DevImage img, const __grid_constant__ WaveArgs a) {
	if (a.wave != 0 && wave_setup_queues_empty(a)) {
		return;
	}
	stage_launch_constants(bsd, cfg, img);
	stage_sincos_tables();
	stage_tables(a.stage_bytes_setup, ASTC_SMEM_HDR + ASTC_SMEM_SINCOS_BYTES, false);
	WCtx w;
	w.lane = threadIdx.x & 31;
	w.base = ASTC_SMEM_HDR + ASTC_SMEM_SINCOS_BYTES + a.stage_bytes_setup + (uint32_t)(threadIdx.x >> 5) * bsd.arena_bytes;
	w.T = bsd.texel_count;
	wave_setup_t<S1>(w, a);
}

#ifndef ASTC_REFINE_MIN_CTAS
#define ASTC_REFINE_MIN_CTAS 1
#endif
// Two instantiations: L1_STEP = true for the LDR profiles (the specialised one-partition, one-plane step inlined beside the
// general one), false for the HDR profiles, which never take it - their kernel carries the general step alone, laid out as
// it was before the specialised step existed.
template <bool L1_STEP>
__global__ void __launch_bounds__(ASTC_REFINE_THREADS_MAX, ASTC_REFINE_MIN_CTAS)
astc_wave_refine_kernel(const __grid_constant__ DevBsd bsd, const __grid_constant__ DevConfig cfg, const __grid_constant__ DevImage img, const __grid_constant__ WaveArgs a) {
	if (wave_queue_empty(a, Q_REFINE, 0, ASTC_Q_RCLASSES * ASTC_Q_RSUB)) {
		return;
	}
	stage_launch_constants(bsd, cfg, img);
	stage_tables(a.stage_bytes, ASTC_SMEM_HDR, true);
	WCtx w;
	w.lane = threadIdx.x & 31;
	w.base = ASTC_SMEM_HDR + a.stage_bytes + (uint32_t)(threadIdx.x >> 5) * bsd.arena_bytes_small;
	w.T = bsd.texel_count;
	wave_refine<L1_STEP>(w, a, threadIdx.x >> 5);
}

// which refinement kernel a context launches
static inline bool refine_l1_step(const DevConfig& cfg) { return cfg.profile == PRF_LDR || cfg.profile == PRF_LDR_SRGB; }
// which set-up kernel a launch of wave `wave` takes (the same profiles as the refinement kernel, wave 0 only)
typedef void (*SetupKernel)(const DevBsd, const DevConfig, const DevImage, const WaveArgs);
static inline SetupKernel setup_kernel(const DevConfig& cfg, int wave) {
	return (wave == 0 && refine_l1_step(cfg)) ? astc_wave_setup_kernel<true> : astc_wave_setup_kernel<false>;
}

__global__ void __launch_bounds__(ASTC_REFINE_THREADS_MAX, 1)
astc_wave_prepare_kernel(const __grid_constant__ DevBsd bsd, const __grid_constant__ DevConfig cfg, const __grid_constant__ DevImage img, const __grid_constant__ WaveArgs a) {
	if (wave_queue_empty(a, Q_PREPARE, 0, ASTC_Q_PREP)) {
		return;
	}
	stage_launch_constants(bsd, cfg, img);
	WCtx w;
	w.lane = threadIdx.x & 31;
	w.base = ASTC_SMEM_HDR + (uint32_t)(threadIdx.x >> 5) * bsd.arena_bytes_small;
	w.T = bsd.texel_count;
	wave_prepare(w, a);
}

__global__ void __launch_bounds__(ASTC_EMIT_THREADS, 1)
astc_wave_emit_kernel(const __grid_constant__ DevBsd bsd, const __grid_constant__ DevConfig cfg, const __grid_constant__ DevImage img, const __grid_constant__ WaveArgs a) {
	// a cancelled pass packs nothing (one look per CTA, so that the whole CTA leaves together; no barrier when the pass has no flag)
	if (img.cancel != nullptr && __syncthreads_or(threadIdx.x == 0 && pass_cancelled(img.cancel) ? 1 : 0)) {
		return;
	}
	stage_launch_constants(bsd, cfg, img);
	wave_emit(threadIdx.x & 31, ASTC_SMEM_HDR + (uint32_t)(threadIdx.x >> 5) * (32 * EMIT_SLICE), a);
}

// ---- alpha-scale pre-pass (SURVEY.md section 8f): one CTA per 32 x 32 tile ----
// The grid covers tile rows [tile_row0, tile_row0 + gridDim.x / tiles_x): the window of one slab (alpha_window).
#define ASTC_ALPHA_THREADS 128
__global__ void __launch_bounds__(ASTC_ALPHA_THREADS, 1)
astc_alpha_average_kernel(const __grid_constant__ DevImage img, unsigned int radius, unsigned int tiles_x, unsigned int tile_row0, float* __restrict__ averages) {
	// (a cancelled pass reads no averages: wave 0 finds the same raised flag)
	if (img.cancel != nullptr && __syncthreads_or(threadIdx.x == 0 && pass_cancelled(img.cancel) ? 1 : 0)) {
		return;
	}
	unsigned int ty = blockIdx.x / tiles_x;
	unsigned int tx = blockIdx.x - ty * tiles_x;
	ty += tile_row0;
	alpha_average_tile(img, radius, tx * ALPHA_TILE, ty * ALPHA_TILE, 0, averages, (int)threadIdx.x, (int)blockDim.x);
}

// ---- block lists (astc_dev_gather.cuh): one warp per listed block, grid-stride ----
#define ASTC_GATHER_THREADS 256
__global__ void __launch_bounds__(ASTC_GATHER_THREADS)
astc_gather_blocks_kernel(const __grid_constant__ GatherArgs g) {
	const unsigned int warps = blockDim.x >> 5;
	for (unsigned int i = blockIdx.x * warps + (threadIdx.x >> 5); i < g.n; i += gridDim.x * warps) {
		gather_block(g, i, (int)(threadIdx.x & 31), 32);
	}
}

// staging block i -> payload block indices[i] (duplicates write the same bytes); one thread per block
__global__ void __launch_bounds__(ASTC_GATHER_THREADS)
astc_scatter_blocks_kernel(const uint8_t* __restrict__ staged, const uint32_t* __restrict__ indices, unsigned int n, uint8_t* payload, int aligned16) {
	unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) {
		return;
	}
	uint8_t* dst = payload + (size_t)__ldg(indices + i) * 16;
	uint4 v = __ldg(reinterpret_cast<const uint4*>(staged) + i);
	if (aligned16) {
		*reinterpret_cast<uint4*>(dst) = v;
	} else {
		const uint8_t* b = reinterpret_cast<const uint8_t*>(&v);
		for (int k = 0; k < 16; k++) {
			dst[k] = b[k];
		}
	}
}

// ---- decompression (SURVEY.md section 8f): one warp per block, grid-stride ----
#define ASTC_DECODE_THREADS 256
__global__ void __launch_bounds__(ASTC_DECODE_THREADS, 2)
astc_decompress_kernel(const __grid_constant__ DevBsd bsd, const __grid_constant__ DevConfig cfg, const __grid_constant__ DevImage img,
                       const uint8_t* __restrict__ blocks, unsigned int block_count) {
	stage_launch_constants(bsd, cfg, img);
	const int lane = threadIdx.x & 31;
	const unsigned int warps_per_cta = blockDim.x >> 5;
	const uint32_t slice = ASTC_SMEM_HDR + (threadIdx.x >> 5) * D_SLICE;
	for (unsigned int b = blockIdx.x * warps_per_cta + (threadIdx.x >> 5); b < block_count; b += gridDim.x * warps_per_cta) {
		unsigned int by = b / img.blocks_x;
		unsigned int bx = b - by * img.blocks_x;
		decompress_block(lane, slice, blocks + (size_t)b * 16, bx, by);
	}
}

__global__ void __launch_bounds__(32, 1)
astc_block_info_kernel(const __grid_constant__ DevBsd bsd, const __grid_constant__ DevConfig cfg, const __grid_constant__ DevImage img,
                       unsigned long long lo, unsigned long long hi, DevBlockInfo* out) {
	stage_launch_constants(bsd, cfg, img);
	block_info(threadIdx.x & 31, ASTC_SMEM_HDR, lo, hi, out);
}

// ---- the single-kernel drivers (kept for A/B measurements: ASTCENC_B200_DRIVER=lockstep|warp) ----
__global__ void __launch_bounds__(ASTC_CTA_THREADS_MAX, 1)
astc_compress_kernel(const __grid_constant__ DevBsd bsd, const __grid_constant__ DevConfig cfg, const __grid_constant__ DevImage img,
                     unsigned int* __restrict__ ticket, int coherence_probe, int lockstep) {
	const int lane = threadIdx.x & 31;
	const int warp = threadIdx.x >> 5;
	stage_launch_constants(bsd, cfg, img);
	stage_sincos_tables();
	WCtx w;
	w.lane = lane;
	w.base = ASTC_SMEM_HDR + ASTC_SMEM_SINCOS_BYTES + (uint32_t)warp * bsd.arena_bytes;
	w.T = bsd.texel_count;
	const unsigned int total = img.blocks_x * img.block_rows;
	const unsigned int blocks_x = img.blocks_x;
#if defined(ASTC_DEBUG_SINGLE_LANE)
	if (lane != 0) {
		return;
	}
#endif
	if (lockstep) {
		BlockFeed feed;
		feed.ticket = ticket;
		feed.total = total;
		feed.blocks_x = blocks_x;
		feed.cancel = img.cancel;
		// (the Refine slots sit behind the arenas: the host sizes the window for them)
		compress_blocks_lockstep(w, feed, ASTC_SMEM_HDR + ASTC_SMEM_SINCOS_BYTES + (uint32_t)(blockDim.x >> 5) * bsd.arena_bytes + (uint32_t)warp * ASTC_REFINE_STATE_BYTES);
		return;
	}
	while (true) {
		unsigned int b = 0;
#if !defined(ASTC_DEBUG_SINGLE_LANE)
		if (coherence_probe) {
			// experiment only: every warp of the CTA compresses the SAME block (measures what instruction-cache
			// sharing between phase-aligned warps is worth); results are identical, so the duplicate stores are benign
			unsigned int* cta_ticket = reinterpret_cast<unsigned int*>(astc_smem + ASTC_SMEM_HDR - 4);
			__syncthreads();
			if (threadIdx.x == 0) {
				*cta_ticket = pass_cancelled(img.cancel) ? 0xFFFFFFFFu : atomicAdd(ticket, 1u);
			}
			__syncthreads();
			b = *cta_ticket;
		} else
#endif
		{
			if (lane == 0) {
				b = pass_cancelled(img.cancel) ? 0xFFFFFFFFu : atomicAdd(ticket, 1u);
			}
#if !defined(ASTC_DEBUG_SINGLE_LANE)
			b = __shfl_sync(0xffffffffu, b, 0);
#endif
		}
		if (b >= total) {
			break;
		}
		unsigned int by = b / blocks_x;
		unsigned int bx = b - by * blocks_x;
		load_block(w, bx, by + IMG.block_row0);
		compress_block(w, IMG.out + (size_t)b * 16);
		pass_block_done(w, img.done);
	}
}

// ---------------------------------------------------------------------------------------------
// Context
// ---------------------------------------------------------------------------------------------
static const bool g_debug_cuda = getenv("ASTCENC_B200_DEBUG") != nullptr;
#define CUDA_TRY(expr, onfail) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) { \
	if (g_debug_cuda) fprintf(stderr, "astcenc_b200: %s failed: %s\n", #expr, cudaGetErrorString(e_)); onfail; } } while (0)

// Every entry point runs on the context's device and leaves the caller's current device as it found it
// (single-process multi-GPU callers such as PyTorch keep their own notion of the current device).
struct DeviceGuard {
	int prev, target;
	bool ok;
	explicit DeviceGuard(int device) : prev(device), target(device), ok(true) {
		ok = cudaGetDevice(&prev) == cudaSuccess;
		if (ok && prev != target) {
			ok = cudaSetDevice(target) == cudaSuccess;
		}
	}
	~DeviceGuard() {
		if (ok && prev != target) {
			cudaSetDevice(prev);
		}
	}
};

// Tuning / experiment knobs, read ONCE when the context is created (INTEGRATION.md lists them).
struct Knobs {
	size_t batch_blocks;         // ASTCENC_B200_BATCH_BLOCKS: blocks per batch of a slab (records are reused batch after batch)
	unsigned int sync_mask;      // ASTCENC_B200_SYNC_MASK: stage barriers of the wave kernels
	unsigned int sync_mask_tail; // ASTCENC_B200_SYNC_MASK_TAIL: the same for the waves after the first (default: the same mask)
	int coherence_probe;         // ASTCENC_B200_COHERENCE_PROBE (single-kernel driver experiment)
	int upload_bands;            // ASTCENC_B200_UPLOAD_BANDS: bands the host-pointer path cuts an image into (1 = one copy)
	int stage_print;             // ASTCENC_B200_STAGE_PRINT
	int pipes;                   // ASTCENC_B200_PIPES: independent sub-slab pipelines of one pass (1 = the plain wave loop)
};
#define ASTC_MAX_PIPES 8
#define ASTC_MAX_BANDS 8
#define ASTC_COUNTER_WORDS (2 * ASTC_Q_KINDS * ASTC_MAX_WAVES + ASTC_MAX_BANDS)

struct DeviceTables {            // shared between a parent context and its children
	std::atomic<int> refcount;
	uint8_t* d_blob;
	DevBsd bsd;                  // device pointers
	DevBsd bsd_1p;               // the same tables, compact one-plane arena plan (wave 0 of the pipeline)
	astc_host::BlockSizeTables* host_tables;
};

struct astcenc_context {
	astcenc_config config;
	unsigned int thread_count;
	int device;
	DeviceTables* tables;
	DevConfig dcfg;
	cudaStream_t stream;
	cudaEvent_t ev0, ev1;
	unsigned int* d_ticket;
	int warps_per_cta;
	int grid;
	size_t smem_bytes;
	int lockstep;                // single-kernel drivers: phase-aligned CTA (1) or independent warps (0)
	int driver;                  // 0 = wave pipeline (default), 1 = single kernel
	int warps_setup, warps_small;   // warps per CTA of the setup / refine+prepare kernels
	int refine_ctas;                // CTAs per SM of the refine kernel (experiment: ASTCENC_B200_REFINE_CTAS)
	int warps_setup_1p;             // set-up kernel on the compact one-plane plan (0 = plan not used)
	size_t smem_setup, smem_setup_1p, smem_small, smem_refine;
	uint32_t setup_stage_bytes;
	uint32_t refine_stage_bytes;   // tables staged behind the header of the refine kernel's shared window (0 = none)
	int max_waves;
	unsigned int volume_dim_z;      // slices of the volume the current pass reads (3D block sizes; 1 otherwise), set under launch_mtx
	uint32_t* pass_cancel;          // the progress words the current pass's kernels see (null for the device-resident paths), set under launch_mtx
	uint32_t* pass_done;
	bool pass_alpha_staged;         // the pass reads averages gathered into d_alpha beforehand and runs no pre-pass (block lists), set under launch_mtx
	// wave pipeline buffers, grown on demand
	uint8_t* d_records;
	size_t d_records_bytes;
	uint32_t* d_queues;          // ASTC_Q_KINDS x capacity
	size_t queue_capacity;
	uint32_t* d_counters;        // count[ASTC_Q_KINDS][MAX_WAVES] head[ASTC_Q_KINDS][MAX_WAVES]
	float* d_alpha;              // alpha-scale pre-pass: one average per texel
	size_t d_alpha_bytes;
	float alpha_threshold;
	// optional per-stage timing (astcenc_b200_stage_timing): an event after every launch of the next call
	int stage_timing;
	std::vector<cudaEvent_t> stage_events;
	std::vector<int> stage_kinds;
	// staging buffers for the host-pointer API, grown on demand
	uint8_t* d_image;
	size_t d_image_bytes;
	uint8_t* d_out;
	size_t d_out_bytes;
	// block lists (astcenc_b200_compress_device_blocks), grown on demand: the list, the staging image and payload of one chunk,
	// the pre-pass averages of the source image
	uint8_t* d_list;
	size_t d_list_bytes;
	uint8_t* d_list_image;
	size_t d_list_image_bytes;
	uint8_t* d_list_out;
	size_t d_list_out_bytes;
	uint8_t* d_list_alpha;
	size_t d_list_alpha_bytes;
	Knobs knobs;
	// The per-context scratch (records, queues, counters, alpha averages) serves ONE pipeline pass at a time: launch_mtx
	// serialises the host side, scratch_done orders a pass on one stream behind the previous pass on another.
	std::mutex launch_mtx;
	cudaEvent_t scratch_done;
	bool scratch_used;
	// host-pointer path: uploads run on copy_stream, band by band, under the set-up of the previous band
	cudaStream_t copy_stream;
	cudaEvent_t band_ready[ASTC_MAX_BANDS];
	cudaEvent_t out_ready;
	// sub-slab pipelines of one pass (launch_pipes): one stream each, joined to the caller's stream by events
	cudaStream_t pipe_stream[ASTC_MAX_PIPES];
	cudaEvent_t pipe_done[ASTC_MAX_PIPES];
	cudaEvent_t pipe_start;
	uint8_t* d_image2;           // second image buffer of the batch API (double-buffered uploads)
	size_t d_image2_bytes;
	// multi-GPU (astc_host_multi.inl): one process per GPU, NCCL for the payload gather
	void* nccl_comm;
	int rank, world;
	cudaEvent_t ev_g0, ev_g1;
	float last_gather_ms, last_compress_ms;
	// caller protocol
	std::mutex mtx;
	std::condition_variable cv;
	int state;                   // 0 idle, 1 running, 2 done
	astcenc_error result;
	int dstate;                  // the same for decompression
	astcenc_error dresult;
	std::atomic<bool> cancel;
	// Progress and cancellation of astcenc_compress_image (astc_dev_lockstep.cuh, pass_cancelled): d_words = {cancel flag, done
	// counter}; h_words (pinned) = {0, 1, counter read-back}: the flag is written by 4-byte DMAs from h_words[0] / [1] and the
	// counter read by one into h_words[2], all on ctl_stream, which never waits for the pass. flag_mtx makes "set ctx->cancel,
	// enqueue the matching flag write" one step, so that the device flag always ends on the value ctx->cancel holds.
	uint32_t* d_words;
	uint32_t* h_words;
	cudaStream_t ctl_stream;
	cudaEvent_t ctl_ready;          // after the last flag clear: a pass starts behind it
	std::mutex flag_mtx;
	bool flag_raised;               // a raise was enqueued since the last clear (under flag_mtx)
	// stats
	unsigned long long launches;
	float last_kernel_ms;
	size_t last_h2d, last_d2h;
};

static std::mutex g_const_mtx;
static DevConstTables* g_d_consts[64];

static astcenc_error ensure_const_tables(int device) {
	std::lock_guard<std::mutex> lk(g_const_mtx);
	if (device < 0 || device >= 64) {
		return ASTCENC_ERR_BAD_CONTEXT;
	}
	if (g_d_consts[device]) {
		return ASTCENC_SUCCESS;
	}
	DevConstTables* h = new DevConstTables;
	astc_host::fill_dev_const_tables(*h);
	DevConstTables* d = nullptr;
	CUDA_TRY(cudaMalloc(&d, sizeof(DevConstTables)), { delete h; return ASTCENC_ERR_OUT_OF_MEM; });
	CUDA_TRY(cudaMemcpy(d, h, sizeof(DevConstTables), cudaMemcpyHostToDevice), { delete h; return ASTCENC_ERR_BAD_CONTEXT; });
	const DevConstTables* dc = d;
	CUDA_TRY(cudaMemcpyToSymbol(g_astc_ct, &dc, sizeof(dc)), { delete h; return ASTCENC_ERR_BAD_CONTEXT; });
	delete h;
	g_d_consts[device] = d;
	return ASTCENC_SUCCESS;
}

static void release_tables(DeviceTables* t) {
	if (t && t->refcount.fetch_sub(1) == 1) {
		cudaFree(t->d_blob);
		astc_host::free_block_size_tables(t->host_tables);
		delete t;
	}
}

extern "C" {

astcenc_error astcenc_config_init(astcenc_profile profile, unsigned int block_x, unsigned int block_y, unsigned int block_z, float quality,
                                  unsigned int flags, astcenc_config* config) {
	return astc_host::config_init(profile, block_x, block_y, block_z, quality, flags, config);
}

void astcenc_context_free(astcenc_context* ctx);

astcenc_error astcenc_context_alloc(const astcenc_config* configp, unsigned int thread_count, astcenc_context** context, const astcenc_context* parent) {
	astcenc_error status = astc_host::validate_cpu_float();
	if (status != ASTCENC_SUCCESS) {
		return status;
	}
	if (thread_count == 0) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	bool has_config = configp != nullptr;
	bool has_parent = parent != nullptr;
	if (!(has_config ^ has_parent)) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	if (has_parent) {
		configp = &parent->config;
	}
	astcenc_context* ctx = new (std::nothrow) astcenc_context;
	if (!ctx) {
		return ASTCENC_ERR_OUT_OF_MEM;
	}
	// every resource starts out null, so that astcenc_context_free() can release a partially built context
	ctx->config = *configp;
	ctx->thread_count = thread_count;
	ctx->device = -1;
	ctx->tables = nullptr;
	ctx->stream = nullptr;
	ctx->copy_stream = nullptr;
	ctx->ev0 = ctx->ev1 = nullptr;
	ctx->scratch_done = nullptr;
	ctx->scratch_used = false;
	ctx->out_ready = nullptr;
	for (int i = 0; i < ASTC_MAX_BANDS; i++) {
		ctx->band_ready[i] = nullptr;
	}
	for (int i = 0; i < ASTC_MAX_PIPES; i++) {
		ctx->pipe_stream[i] = nullptr;
		ctx->pipe_done[i] = nullptr;
	}
	ctx->pipe_start = nullptr;
	ctx->d_ticket = nullptr;
	ctx->d_records = nullptr;
	ctx->d_records_bytes = 0;
	ctx->d_queues = nullptr;
	ctx->queue_capacity = 0;
	ctx->d_counters = nullptr;
	ctx->d_alpha = nullptr;
	ctx->d_alpha_bytes = 0;
	ctx->alpha_threshold = 0.0f;
	ctx->stage_timing = 0;
	ctx->d_image = nullptr;
	ctx->d_image2 = nullptr;
	ctx->d_out = nullptr;
	ctx->d_image_bytes = ctx->d_image2_bytes = ctx->d_out_bytes = 0;
	ctx->d_list = ctx->d_list_image = ctx->d_list_out = ctx->d_list_alpha = nullptr;
	ctx->d_list_bytes = ctx->d_list_image_bytes = ctx->d_list_out_bytes = ctx->d_list_alpha_bytes = 0;
	ctx->nccl_comm = nullptr;
	ctx->rank = 0;
	ctx->world = 1;
	ctx->ev_g0 = ctx->ev_g1 = nullptr;
	ctx->last_gather_ms = ctx->last_compress_ms = 0.0f;
	ctx->state = 0;
	ctx->result = ASTCENC_SUCCESS;
	ctx->dstate = 0;
	ctx->dresult = ASTCENC_SUCCESS;
	ctx->cancel = false;
	ctx->d_words = nullptr;
	ctx->h_words = nullptr;
	ctx->ctl_stream = nullptr;
	ctx->ctl_ready = nullptr;
	ctx->flag_raised = false;
	ctx->pass_cancel = ctx->pass_done = nullptr;
	ctx->pass_alpha_staged = false;
	ctx->launches = 0;
	ctx->last_kernel_ms = 0.0f;
	ctx->last_h2d = ctx->last_d2h = 0;
	ctx->warps_per_cta = ctx->grid = 0;
	ctx->warps_setup_1p = 0;
	ctx->max_waves = 0;
	ctx->volume_dim_z = 1;
	// environment knobs: read here, once
	ctx->knobs.batch_blocks = (size_t)1 << 20;
	if (const char* e = getenv("ASTCENC_B200_BATCH_BLOCKS")) {
		long v = atol(e);
		if (v > 0) ctx->knobs.batch_blocks = (size_t)v;
	}
	// stage barriers of the wave kernels (bit i = i-th barrier of the kernel loop): the one in front of the endpoint-format stage
	// of the set-up kernel (bit 3) is on. With the queues sorted by cost the mask hardly matters: no barrier at all measures
	// 71.35 against 71.57 ms per pass (H100 80GB HBM3 at 400 W, 4K 6x6 -medium), inside the run-to-run spread of 71.1-71.7 ms
	ctx->knobs.sync_mask = 8;
	if (const char* e = getenv("ASTCENC_B200_SYNC_MASK")) {
		ctx->knobs.sync_mask = (unsigned int)strtoul(e, nullptr, 0);
	}
	ctx->knobs.sync_mask_tail = ctx->knobs.sync_mask;
	if (const char* e = getenv("ASTCENC_B200_SYNC_MASK_TAIL")) {
		ctx->knobs.sync_mask_tail = (unsigned int)strtoul(e, nullptr, 0);
	}
	ctx->knobs.coherence_probe = getenv("ASTCENC_B200_COHERENCE_PROBE") ? 1 : 0;
	ctx->knobs.stage_print = getenv("ASTCENC_B200_STAGE_PRINT") ? 1 : 0;
	ctx->knobs.pipes = 1;      // 1 / 2 / 4 pipelines = 71.6 / 71.9 / 73.7 ms per pass (H100 80GB HBM3 at 400 W, 4K 6x6 -medium): the idle warps are inside the CTAs, not between kernels
	if (const char* e = getenv("ASTCENC_B200_PIPES")) {
		int v = atoi(e);
		if (v >= 1 && v <= ASTC_MAX_PIPES) ctx->knobs.pipes = v;
	}
	ctx->knobs.upload_bands = 4;
	if (const char* e = getenv("ASTCENC_B200_UPLOAD_BANDS")) {
		int v = atoi(e);
		if (v >= 1 && v <= ASTC_MAX_BANDS) ctx->knobs.upload_bands = v;
	}
	// one exit for every failure: whatever was built so far is released by astcenc_context_free()
	#define ALLOC_FAIL(code) do { astcenc_context_free(ctx); return (code); } while (0)
	status = astc_host::validate_config(ctx->config);
	if (status != ASTCENC_SUCCESS) {
		ALLOC_FAIL(status);
	}
	// The GPU is mandatory: no device, no context.
	int device = 0;
	CUDA_TRY(cudaGetDevice(&device), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
	ctx->device = device;
	status = ensure_const_tables(device);
	if (status != ASTCENC_SUCCESS) {
		ALLOC_FAIL(status);
	}
	const astcenc_config& cfg = ctx->config;
	if (has_parent) {
		ctx->tables = parent->tables;
		ctx->tables->refcount.fetch_add(1);
	} else {
		DeviceTables* t = new DeviceTables;
		t->refcount = 1;
		t->d_blob = nullptr;
		t->host_tables = nullptr;
		ctx->tables = t;
		astc_host::PackedTables pk;
		t->host_tables = astc_host::build_packed_tables(cfg, pk);
		CUDA_TRY(cudaMalloc(&t->d_blob, pk.blob.size()), ALLOC_FAIL(ASTCENC_ERR_OUT_OF_MEM));
		CUDA_TRY(cudaMemcpy(t->d_blob, pk.blob.data(), pk.blob.size(), cudaMemcpyHostToDevice), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
		astc_host::relocate_tables(pk, t->d_blob);
		t->bsd = pk.bsd;
		t->bsd_1p = pk.bsd_1p;
	}
	astc_host::make_device_config(cfg, ctx->dcfg);

	if (!(cfg.flags & ASTCENC_FLG_DECOMPRESS_ONLY)) {
		cudaDeviceProp prop;
		CUDA_TRY(cudaGetDeviceProperties(&prop, device), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
		// The per-warp arena lives in shared memory only: one CTA per SM with as many warps as fit (at most 16).
		size_t smem_limit = prop.sharedMemPerBlockOptin;
		size_t arena = ctx->tables->bsd.arena_bytes;
		int warps = (int)((smem_limit - ASTC_SMEM_HDR - ASTC_SMEM_SINCOS_BYTES) / (arena + ASTC_REFINE_STATE_BYTES));
		if (warps > ASTC_CTA_THREADS_MAX / 32) warps = ASTC_CTA_THREADS_MAX / 32;
		if (warps < 1) {
			// block sizes / presets whose working set exceeds one SM's shared memory are not supported by this build
			ALLOC_FAIL(ASTCENC_ERR_NOT_IMPLEMENTED);
		}
		ctx->warps_per_cta = warps;
		ctx->grid = prop.multiProcessorCount;
		// tuning overrides (experiments): warps per CTA and CTAs per SM
		if (const char* e = getenv("ASTCENC_B200_WARPS")) {
			int v = atoi(e);
			if (v >= 1 && v <= warps) ctx->warps_per_cta = v;
		}
		if (const char* e = getenv("ASTCENC_B200_CTAS_PER_SM")) {
			int v = atoi(e);
			if (v >= 1 && v <= 8) ctx->grid = prop.multiProcessorCount * v;
		}
		ctx->lockstep = 1;
		ctx->driver = 0;
		if (const char* e = getenv("ASTCENC_B200_DRIVER")) {
			if (!strcmp(e, "lockstep")) { ctx->driver = 1; ctx->lockstep = 1; }
			else if (!strcmp(e, "warp")) { ctx->driver = 1; ctx->lockstep = 0; }
		}
		ctx->smem_bytes = ASTC_SMEM_HDR + ASTC_SMEM_SINCOS_BYTES + (arena + ASTC_REFINE_STATE_BYTES) * ctx->warps_per_cta;
		CUDA_TRY(cudaFuncSetAttribute(astc_compress_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_limit), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
		// wave pipeline: the setup kernel needs the full arena, refinement / preparation only up to the union scratch
		{
			size_t arena_small = ctx->tables->bsd.arena_bytes_small;
			int ws = (int)((smem_limit - ASTC_SMEM_HDR - ASTC_SMEM_SINCOS_BYTES) / arena);
			if (ws > ASTC_SETUP_THREADS_MAX / 32) ws = ASTC_SETUP_THREADS_MAX / 32;
			ctx->refine_ctas = 1;
			if (const char* e = getenv("ASTCENC_B200_REFINE_CTAS")) {
				int v = atoi(e);
				if (v >= 1 && v <= 4) ctx->refine_ctas = v;
			}
			// (per CTA: 1 KB of shared memory is reserved by the system)
			int wr = (int)((smem_limit / ctx->refine_ctas - (ctx->refine_ctas > 1 ? 1024 : 0) - ASTC_SMEM_HDR) / (arena_small + ASTC_REFINE_STATE_BYTES));
			if (wr > ASTC_REFINE_THREADS_MAX / 32) wr = ASTC_REFINE_THREADS_MAX / 32;
			// Staging the decimation (+ colour quantisation) tables in the refine kernel's spare shared memory is possible
			// without losing a warp at 6x6, but gains nothing (71.63 vs 71.57 ms per pass, H100 80GB HBM3 at 400 W, 4K 6x6 -medium: L1 already serves these loads): opt-in.
			size_t stage = (((size_t)ctx->tables->bsd.dec_stage_bytes + 15) & ~(size_t)15) + ASTC_CQ_BYTES;
			ctx->refine_stage_bytes = 0;
			if (getenv("ASTCENC_B200_STAGE_REFINE") && smem_limit > ASTC_SMEM_HDR + stage && (int)((smem_limit - ASTC_SMEM_HDR - stage) / (arena_small + ASTC_REFINE_STATE_BYTES)) >= wr) {
				ctx->refine_stage_bytes = (uint32_t)stage;
			}
			if (const char* e = getenv("ASTCENC_B200_WARPS_SETUP")) {
				int v = atoi(e);
				if (v >= 1 && v <= ws) ws = v;
			}
			if (const char* e = getenv("ASTCENC_B200_WARPS_REFINE")) {
				int v = atoi(e);
				if (v >= 1 && v <= wr) wr = v;
			}
			ctx->warps_setup = ws;
			ctx->warps_small = wr;
			// The set-up kernel walks the decimation tables of every grid for every block (decimated ideal weights, per-mode
			// scoring): with them in shared memory it is faster even with one warp less (6x6 medium: 21 KB of tables, 15
			// instead of 16 warps; 71.6 against 73.3 ms per pass unstaged, H100 80GB HBM3 at 400 W, 4K 6x6 -medium). Done when it costs at most one warp (ASTCENC_B200_STAGE_SETUP=0/1 forces).
			ctx->setup_stage_bytes = 0;
			{
				size_t st = ((size_t)ctx->tables->bsd.dec_stage_bytes + 15) & ~(size_t)15;
				int ws2 = smem_limit > ASTC_SMEM_HDR + ASTC_SMEM_SINCOS_BYTES + st ? (int)((smem_limit - ASTC_SMEM_HDR - ASTC_SMEM_SINCOS_BYTES - st) / arena) : 0;
				bool want = ws2 >= 1 && ws2 >= ws - 1;
				if (const char* e = getenv("ASTCENC_B200_STAGE_SETUP")) {
					want = atoi(e) != 0 && ws2 >= 1;
				}
				if (want) {
					if (ws2 < ws) ws = ws2;
					ctx->warps_setup = ws;
					ctx->setup_stage_bytes = (uint32_t)st;
				}
			}
			ctx->smem_setup = ASTC_SMEM_HDR + ASTC_SMEM_SINCOS_BYTES + ctx->setup_stage_bytes + arena * ws;
			// wave 0 (every block's first trial has one weight plane) runs on the compact plan: more arenas per SM
			{
				size_t arena1 = ctx->tables->bsd_1p.arena_bytes;
				int w1 = (int)((smem_limit - ASTC_SMEM_HDR - ASTC_SMEM_SINCOS_BYTES - ctx->setup_stage_bytes) / arena1);
				if (w1 > ASTC_SETUP_THREADS_MAX / 32) w1 = ASTC_SETUP_THREADS_MAX / 32;
				if (const char* e = getenv("ASTCENC_B200_WARPS_SETUP_1P")) {
					int v = atoi(e);
					if (v >= 0 && v < w1) w1 = v;
				}
				ctx->warps_setup_1p = w1 > ws ? w1 : 0;      // only when it buys warps
				ctx->smem_setup_1p = ASTC_SMEM_HDR + ASTC_SMEM_SINCOS_BYTES + ctx->setup_stage_bytes + arena1 * (size_t)w1;
			}
			ctx->smem_small = ASTC_SMEM_HDR + arena_small * wr;
			ctx->smem_refine = ASTC_SMEM_HDR + ctx->refine_stage_bytes + arena_small * wr + (size_t)ASTC_REFINE_STATE_BYTES * wr;
			CUDA_TRY(cudaFuncSetAttribute(astc_wave_setup_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_limit), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
			CUDA_TRY(cudaFuncSetAttribute(astc_wave_setup_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_limit), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
			CUDA_TRY(cudaFuncSetAttribute(astc_wave_refine_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_limit), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
			CUDA_TRY(cudaFuncSetAttribute(astc_wave_refine_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_limit), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
			CUDA_TRY(cudaFuncSetAttribute(astc_wave_prepare_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_limit), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
			// a block runs at most this many trials (compress_block: mode-0 + full 1-plane, 4 two-plane, then the partition candidates)
			int waves = 2 + 4;
			const unsigned int cl[3] = {cfg.tune_2partitioning_candidate_limit, cfg.tune_3partitioning_candidate_limit, cfg.tune_4partitioning_candidate_limit};
			for (unsigned int pc = 2; pc <= cfg.tune_partition_count_limit && pc <= 4; pc++) {
				waves += (int)cl[pc - 2];
			}
			if (waves > ASTC_MAX_WAVES - 1) waves = ASTC_MAX_WAVES - 1;
			ctx->max_waves = waves;
			// count[kinds][waves], head[kinds][waves], then one image ticket per upload band
			CUDA_TRY(cudaMalloc(&ctx->d_counters, sizeof(uint32_t) * ASTC_COUNTER_WORDS * ASTC_MAX_PIPES), ALLOC_FAIL(ASTCENC_ERR_OUT_OF_MEM));
		}
		CUDA_TRY(cudaMalloc(&ctx->d_ticket, sizeof(unsigned int)), ALLOC_FAIL(ASTCENC_ERR_OUT_OF_MEM));
		// progress and cancellation: the device words start cleared
		CUDA_TRY(cudaMalloc(&ctx->d_words, 2 * sizeof(uint32_t)), ALLOC_FAIL(ASTCENC_ERR_OUT_OF_MEM));
		CUDA_TRY(cudaMemset(ctx->d_words, 0, 2 * sizeof(uint32_t)), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
		CUDA_TRY(cudaHostAlloc(&ctx->h_words, 3 * sizeof(uint32_t), cudaHostAllocDefault), ALLOC_FAIL(ASTCENC_ERR_OUT_OF_MEM));
		ctx->h_words[0] = 0;
		ctx->h_words[1] = 1;
		ctx->h_words[2] = 0;
		CUDA_TRY(cudaStreamCreateWithFlags(&ctx->ctl_stream, cudaStreamNonBlocking), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
		CUDA_TRY(cudaEventCreateWithFlags(&ctx->ctl_ready, cudaEventDisableTiming), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
	}
	CUDA_TRY(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
	CUDA_TRY(cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
	CUDA_TRY(cudaEventCreate(&ctx->ev0), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
	CUDA_TRY(cudaEventCreate(&ctx->ev1), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
	CUDA_TRY(cudaEventCreate(&ctx->ev_g0), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
	CUDA_TRY(cudaEventCreate(&ctx->ev_g1), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
	CUDA_TRY(cudaEventCreateWithFlags(&ctx->scratch_done, cudaEventDisableTiming), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
	CUDA_TRY(cudaEventCreateWithFlags(&ctx->out_ready, cudaEventDisableTiming), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
	for (int i = 0; i < ASTC_MAX_BANDS; i++) {
		CUDA_TRY(cudaEventCreateWithFlags(&ctx->band_ready[i], cudaEventDisableTiming), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
	}
	for (int i = 0; i < ASTC_MAX_PIPES; i++) {
		CUDA_TRY(cudaStreamCreateWithFlags(&ctx->pipe_stream[i], cudaStreamNonBlocking), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
		CUDA_TRY(cudaEventCreateWithFlags(&ctx->pipe_done[i], cudaEventDisableTiming), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
	}
	CUDA_TRY(cudaEventCreateWithFlags(&ctx->pipe_start, cudaEventDisableTiming), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
	#undef ALLOC_FAIL
	*context = ctx;
	return ASTCENC_SUCCESS;
}

static void comm_destroy(astcenc_context* ctx);

void astcenc_context_free(astcenc_context* ctx) {
	if (!ctx) {
		return;
	}
	if (ctx->device < 0) {
		// nothing on the device yet (astcenc_context_alloc failed before it picked one)
		delete ctx;
		return;
	}
	DeviceGuard guard(ctx->device);
	if (ctx->stream) cudaStreamSynchronize(ctx->stream);
	if (ctx->copy_stream) cudaStreamSynchronize(ctx->copy_stream);
	comm_destroy(ctx);
	cudaFree(ctx->d_ticket);
	cudaFree(ctx->d_records);
	cudaFree(ctx->d_queues);
	cudaFree(ctx->d_counters);
	cudaFree(ctx->d_alpha);
	for (cudaEvent_t e : ctx->stage_events) {
		cudaEventDestroy(e);
	}
	cudaFree(ctx->d_image);
	cudaFree(ctx->d_image2);
	cudaFree(ctx->d_out);
	cudaFree(ctx->d_list);
	cudaFree(ctx->d_list_image);
	cudaFree(ctx->d_list_out);
	cudaFree(ctx->d_list_alpha);
	if (ctx->ev0) cudaEventDestroy(ctx->ev0);
	if (ctx->ev1) cudaEventDestroy(ctx->ev1);
	if (ctx->ev_g0) cudaEventDestroy(ctx->ev_g0);
	if (ctx->ev_g1) cudaEventDestroy(ctx->ev_g1);
	if (ctx->scratch_done) cudaEventDestroy(ctx->scratch_done);
	if (ctx->out_ready) cudaEventDestroy(ctx->out_ready);
	for (int i = 0; i < ASTC_MAX_BANDS; i++) {
		if (ctx->band_ready[i]) cudaEventDestroy(ctx->band_ready[i]);
	}
	for (int i = 0; i < ASTC_MAX_PIPES; i++) {
		if (ctx->pipe_stream[i]) {
			cudaStreamSynchronize(ctx->pipe_stream[i]);
			cudaStreamDestroy(ctx->pipe_stream[i]);
		}
		if (ctx->pipe_done[i]) cudaEventDestroy(ctx->pipe_done[i]);
	}
	if (ctx->pipe_start) cudaEventDestroy(ctx->pipe_start);
	if (ctx->ctl_stream) {
		cudaStreamSynchronize(ctx->ctl_stream);
		cudaStreamDestroy(ctx->ctl_stream);
	}
	if (ctx->ctl_ready) cudaEventDestroy(ctx->ctl_ready);
	cudaFree(ctx->d_words);
	if (ctx->h_words) cudaFreeHost(ctx->h_words);
	if (ctx->stream) cudaStreamDestroy(ctx->stream);
	if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
	release_tables(ctx->tables);
	delete ctx;
}

static astcenc_error validate_compression_swizzle(const astcenc_swizzle& s) {
	const int v[4] = {(int)s.r, (int)s.g, (int)s.b, (int)s.a};
	for (int i = 0; i < 4; i++) {
		if (v[i] < ASTCENC_SWZ_R || v[i] > ASTCENC_SWZ_1) {
			return ASTCENC_ERR_BAD_SWIZZLE;
		}
	}
	return ASTCENC_SUCCESS;
}

static size_t mul_safe(size_t a, size_t b, bool& overflow) {
	size_t r = a * b;
	overflow = overflow || ((b != 0) && ((r / b) != a));
	return r;
}

static size_t block_count_axis(size_t dim, size_t blk) {
	size_t n = dim / blk;
	if (dim != blk * n) {
		n++;
	}
	return n;
}

// Upload plan of the host-pointer path: the image (one 2D slice) is copied to the device in bands of block rows on the
// context's copy stream; wave 0 of the pipeline - the only reader of the image - is launched band by band, each launch
// waiting for its band only, so the copy of band k+1 runs under the set-up of band k.
struct UploadPlan {
	const uint8_t* host;         // first byte of the slice in host memory (pageable or pinned)
	uint8_t* device;             // where the slice goes
	size_t row_bytes;            // bytes per image row
	int bands;                   // 1 .. ASTC_MAX_BANDS
};

static astcenc_error launch_batch(astcenc_context* ctx, const void* d_pixels, int data_type, unsigned int dim_x, unsigned int dim_y, const int swz[4],
                                  unsigned int block_row0, unsigned int block_rows, uint8_t* d_out, cudaStream_t stream, const UploadPlan* up);

// A slab of block rows is processed in batches of at most ~1 M blocks: the per-block search records (a few KB each)
// are the only buffer that grows with the image, and the batches reuse them in stream order.
// The context's scratch buffers serve one pass at a time. Calls may come from several host threads and on different
// streams: launch_mtx serialises the enqueueing, and every pass starts by making its stream wait for the event that
// closes the previous pass (a no-op when both ran on the same stream).
static astcenc_error launch_slab_locked(astcenc_context* ctx, const void* d_pixels, int data_type, unsigned int dim_x, unsigned int dim_y, const int swz[4],
                                        unsigned int block_row0, unsigned int block_rows, uint8_t* d_out, cudaStream_t stream, const UploadPlan* up);

// d_cancel / d_done: the progress words of an astcenc_compress_image pass (null: no progress, no cancellation).
static astcenc_error launch_slab(astcenc_context* ctx, const void* d_pixels, int data_type, unsigned int dim_x, unsigned int dim_y, const int swz[4],
                                 unsigned int block_row0, unsigned int block_rows, uint8_t* d_out, cudaStream_t stream, const UploadPlan* up = nullptr,
                                 unsigned int volume_dim_z = 1, uint32_t* d_cancel = nullptr, uint32_t* d_done = nullptr) {
	std::lock_guard<std::mutex> lk(ctx->launch_mtx);
	ctx->volume_dim_z = volume_dim_z;
	ctx->pass_cancel = d_cancel;
	ctx->pass_done = d_done;
	if (ctx->scratch_used) {
		CUDA_TRY(cudaStreamWaitEvent(stream, ctx->scratch_done, 0), return ASTCENC_ERR_BAD_CONTEXT);
	}
	astcenc_error st = launch_slab_locked(ctx, d_pixels, data_type, dim_x, dim_y, swz, block_row0, block_rows, d_out, stream, up);
	CUDA_TRY(cudaEventRecord(ctx->scratch_done, stream), return ASTCENC_ERR_BAD_CONTEXT);
	ctx->scratch_used = true;
	return st;
}

// Image rows [y0, y1) that a pass over block rows [block_row0, block_row0 + block_rows) of a 2D image reads: the slab's own
// rows, or with alpha-scale the rows its pre-pass window reads (a superset of them).
static void slab_image_rows(const astcenc_context* ctx, unsigned int dim_y, unsigned int block_row0, unsigned int block_rows, size_t& y0, size_t& y1) {
	const unsigned int by = ctx->tables->bsd.dim_y;
	y0 = (size_t)block_row0 * by;
	y1 = (size_t)(block_row0 + block_rows) * by;
	if (y1 > dim_y) y1 = dim_y;
	const unsigned int radius = ctx->tables->bsd.dim_z > 1 ? 0 : ctx->config.a_scale_radius;
	if (radius != 0 && y1 > y0) {
		AlphaWindow w = alpha_window(dim_y, radius, (unsigned int)y0, (unsigned int)y1);
		y0 = w.read_row0;
		y1 = w.read_row1;
	}
}

static astcenc_error upload_rows(astcenc_context* ctx, const UploadPlan& up, size_t y0, size_t y1, cudaStream_t stream) {
	CUDA_TRY(cudaMemcpyAsync(up.device + y0 * up.row_bytes, up.host + y0 * up.row_bytes, up.row_bytes * (y1 - y0), cudaMemcpyHostToDevice, ctx->copy_stream),
	         return ASTCENC_ERR_BAD_CONTEXT);
	CUDA_TRY(cudaEventRecord(ctx->band_ready[0], ctx->copy_stream), return ASTCENC_ERR_BAD_CONTEXT);
	CUDA_TRY(cudaStreamWaitEvent(stream, ctx->band_ready[0], 0), return ASTCENC_ERR_BAD_CONTEXT);
	return ASTCENC_SUCCESS;
}

// One pass as P independent sub-slab pipelines. The search is a chain of waves (set-up -> refine -> prepare, ~10 times) and
// every kernel of the chain ends with a drain: the last blocks of a wave keep a few SMs busy while the others idle, and the
// late waves never fill the GPU's SMs at all. Blocks are independent, so the slab is cut into P ranges of block rows, each with
// its own records / queues / counters, and the P chains are enqueued breadth-first on P streams: while the kernel of one
// chain drains, the CTAs of the next chain's kernel take over the SMs that became free (every kernel is one CTA per SM,
// so the hardware block scheduler does the interleaving). Same kernels, same results; wave 0 of chain p waits only for the
// upload of its own rows (the band scheme of the host-pointer path with bands = pipelines).
static astcenc_error launch_pipes(astcenc_context* ctx, int pipes, const void* d_pixels, int data_type, unsigned int dim_x, unsigned int dim_y, const int swz[4],
                                  unsigned int block_row0, unsigned int block_rows, uint8_t* d_out, cudaStream_t stream, const UploadPlan* up) {
	const DevBsd& bsd = ctx->tables->bsd;
	unsigned int blocks_x = (dim_x + bsd.dim_x - 1) / bsd.dim_x;
	size_t total = (size_t)blocks_x * block_rows;
	if (total > ctx->queue_capacity) {
		cudaFree(ctx->d_queues);
		ctx->d_queues = nullptr;
		ctx->queue_capacity = 0;
		CUDA_TRY(cudaMalloc(&ctx->d_queues, sizeof(uint32_t) * ASTC_Q_KINDS * total), return ASTCENC_ERR_OUT_OF_MEM);
		ctx->queue_capacity = total;
	}
	size_t rec_bytes = total * (size_t)bsd.record_bytes;
	if (rec_bytes > ctx->d_records_bytes) {
		cudaFree(ctx->d_records);
		ctx->d_records = nullptr;
		ctx->d_records_bytes = 0;
		CUDA_TRY(cudaMalloc(&ctx->d_records, rec_bytes), return ASTCENC_ERR_OUT_OF_MEM);
		ctx->d_records_bytes = rec_bytes;
	}
	DevImage img[ASTC_MAX_PIPES];
	WaveArgs a[ASTC_MAX_PIPES];
	if (up != nullptr && ctx->scratch_used) {
		CUDA_TRY(cudaStreamWaitEvent(ctx->copy_stream, ctx->scratch_done, 0), return ASTCENC_ERR_BAD_CONTEXT);
	}
	CUDA_TRY(cudaEventRecord(ctx->pipe_start, stream), return ASTCENC_ERR_BAD_CONTEXT);
	for (int p = 0; p < pipes; p++) {
		unsigned int r0 = (unsigned int)((size_t)block_rows * p / pipes), r1 = (unsigned int)((size_t)block_rows * (p + 1) / pipes);
		size_t first = (size_t)r0 * blocks_x;
		cudaStream_t ps = ctx->pipe_stream[p];
		CUDA_TRY(cudaStreamWaitEvent(ps, ctx->pipe_start, 0), return ASTCENC_ERR_BAD_CONTEXT);
		DevImage& im = img[p];
		im.data = d_pixels;
		im.data_type = data_type;
		im.dim_x = dim_x;
		im.dim_y = dim_y;
		im.dim_z = ctx->volume_dim_z;
		im.blocks_x = blocks_x;
		im.blocks_y = (dim_y + bsd.dim_y - 1) / bsd.dim_y;
		im.block_row0 = block_row0 + r0;
		im.block_rows = r1 - r0;
		for (int i = 0; i < 4; i++) {
			im.swz[i] = swz[i];
		}
		im.out = d_out + first * 16;
		im.alpha_avg = ctx->config.a_scale_radius != 0 && bsd.dim_z == 1 ? ctx->d_alpha : nullptr;
		im.alpha_threshold = ctx->alpha_threshold;
		im.cancel = ctx->pass_cancel;
		im.done = ctx->pass_done;
		uint32_t* counters = ctx->d_counters + (size_t)p * ASTC_COUNTER_WORDS;
		CUDA_TRY(cudaMemsetAsync(counters, 0, sizeof(uint32_t) * ASTC_COUNTER_WORDS, ps), return ASTCENC_ERR_BAD_CONTEXT);
		WaveArgs& w = a[p];
		w.records = ctx->d_records + first * (size_t)bsd.record_bytes;
		w.queues = ctx->d_queues + first;
		w.queue_stride = ctx->queue_capacity;
		w.count = counters;
		w.head = counters + ASTC_Q_KINDS * ASTC_MAX_WAVES;
		w.total = (r1 - r0) * blocks_x;
		w.blocks_x = blocks_x;
		w.ticket = counters + 2 * ASTC_Q_KINDS * ASTC_MAX_WAVES;
		w.first_block = 0;
		w.band_blocks = w.total;
		w.cls_lo = 0;
		w.cls_hi = ASTC_Q_CLASSES;
		w.stage_bytes = ctx->refine_stage_bytes;
		w.refine_state_off = (uint32_t)(ASTC_SMEM_HDR + ctx->refine_stage_bytes + (size_t)bsd.arena_bytes_small * ctx->warps_small);
		w.stage_bytes_setup = ctx->setup_stage_bytes;
		w.sync_mask = ctx->knobs.sync_mask;
		if (up != nullptr) {
			// this pipeline's rows go up on the copy stream; only its wave 0 waits for them
			size_t y0 = (size_t)(block_row0 + r0) * bsd.dim_y, y1 = (size_t)(block_row0 + r1) * bsd.dim_y;
			if (y1 > dim_y) y1 = dim_y;
			if (y1 > y0) {
				CUDA_TRY(cudaMemcpyAsync(up->device + y0 * up->row_bytes, up->host + y0 * up->row_bytes, (y1 - y0) * up->row_bytes, cudaMemcpyHostToDevice, ctx->copy_stream),
				         return ASTCENC_ERR_BAD_CONTEXT);
			}
			CUDA_TRY(cudaEventRecord(ctx->band_ready[p], ctx->copy_stream), return ASTCENC_ERR_BAD_CONTEXT);
			CUDA_TRY(cudaStreamWaitEvent(ps, ctx->band_ready[p], 0), return ASTCENC_ERR_BAD_CONTEXT);
		}
	}
	int grid = ctx->grid;
	int wp = ctx->warps_small >= 2 ? ctx->warps_small / 2 : 1;
	for (int wave = 0; wave < ctx->max_waves; wave++) {
		for (int p = 0; p < pipes; p++) {
			if (a[p].total == 0) {
				continue;
			}
			a[p].wave = wave;
			a[p].sync_mask = wave == 0 ? ctx->knobs.sync_mask : ctx->knobs.sync_mask_tail;
			cudaStream_t ps = ctx->pipe_stream[p];
			if (ctx->warps_setup_1p) {
				if (wave != 0) {
					a[p].cls_lo = 0;
					a[p].cls_hi = 1;
					astc_wave_setup_kernel<false><<<grid, ctx->warps_setup * 32, ctx->smem_setup, ps>>>(bsd, ctx->dcfg, img[p], a[p]);
					ctx->launches++;
					a[p].cls_lo = 1;
					a[p].cls_hi = ASTC_Q_CLASSES;
				}
				setup_kernel(ctx->dcfg, wave)<<<grid, ctx->warps_setup_1p * 32, ctx->smem_setup_1p, ps>>>(ctx->tables->bsd_1p, ctx->dcfg, img[p], a[p]);
				a[p].cls_lo = 0;
				a[p].cls_hi = ASTC_Q_CLASSES;
			} else {
				setup_kernel(ctx->dcfg, wave)<<<grid, ctx->warps_setup * 32, ctx->smem_setup, ps>>>(bsd, ctx->dcfg, img[p], a[p]);
			}
			if (refine_l1_step(ctx->dcfg)) {
				astc_wave_refine_kernel<true><<<grid * ctx->refine_ctas, ctx->warps_small * 32, ctx->smem_refine, ps>>>(bsd, ctx->dcfg, img[p], a[p]);
			} else {
				astc_wave_refine_kernel<false><<<grid * ctx->refine_ctas, ctx->warps_small * 32, ctx->smem_refine, ps>>>(bsd, ctx->dcfg, img[p], a[p]);
			}
			astc_wave_prepare_kernel<<<grid * 2, wp * 32, ASTC_SMEM_HDR + (size_t)bsd.arena_bytes_small * wp, ps>>>(bsd, ctx->dcfg, img[p], a[p]);
			ctx->launches += 3;
		}
	}
	for (int p = 0; p < pipes; p++) {
		cudaStream_t ps = ctx->pipe_stream[p];
		if (a[p].total != 0) {
			a[p].wave = 0;
			astc_wave_emit_kernel<<<grid * 4, ASTC_EMIT_THREADS, ASTC_SMEM_HDR + (ASTC_EMIT_THREADS / 32) * 32 * EMIT_SLICE, ps>>>(bsd, ctx->dcfg, img[p], a[p]);
			ctx->launches++;
		}
		CUDA_TRY(cudaEventRecord(ctx->pipe_done[p], ps), return ASTCENC_ERR_BAD_CONTEXT);
		CUDA_TRY(cudaStreamWaitEvent(stream, ctx->pipe_done[p], 0), return ASTCENC_ERR_BAD_CONTEXT);
	}
	CUDA_TRY(cudaGetLastError(), return ASTCENC_ERR_BAD_CONTEXT);
	return ASTCENC_SUCCESS;
}

// The alpha-scale pre-pass over image rows [y0, y1) of a 2D image (alpha_window: the 32 x 32 tiles that cover them, reading up to
// a_scale_radius rows beyond); the averages land at their image positions in `averages` (dim_x * dim_y floats). Sets the
// threshold the set-up stage compares them with.
static astcenc_error alpha_prepass(astcenc_context* ctx, const void* d_pixels, int data_type, unsigned int dim_x, unsigned int dim_y, const int swz[4],
                                   unsigned int y0, unsigned int y1, float* averages, cudaStream_t stream) {
	const DevBsd& bsd = ctx->tables->bsd;
	const unsigned int radius = ctx->config.a_scale_radius;
	size_t pad = (size_t)ALPHA_TILE + 2 * (size_t)radius + 1;
	size_t smem = pad * pad * sizeof(float);
	if (smem > 200 * 1024) {
		return ASTCENC_ERR_NOT_IMPLEMENTED;      // radius > ~94: the padded tile no longer fits shared memory
	}
	if (smem > 48 * 1024) {
		CUDA_TRY(cudaFuncSetAttribute(astc_alpha_average_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), return ASTCENC_ERR_BAD_CONTEXT);
	}
	DevImage aimg{};
	aimg.data = d_pixels;
	aimg.data_type = data_type;
	aimg.dim_x = dim_x;
	aimg.dim_y = dim_y;
	for (int i = 0; i < 4; i++) {
		aimg.swz[i] = swz[i];
	}
	aimg.cancel = ctx->pass_cancel;
	unsigned int tiles_x = (dim_x + ALPHA_TILE - 1) / ALPHA_TILE;
	AlphaWindow win = alpha_window(dim_y, radius, y0, y1);
	astc_alpha_average_kernel<<<tiles_x * win.tile_rows, ASTC_ALPHA_THREADS, smem, stream>>>(aimg, radius, tiles_x, win.tile_row0, averages);
	CUDA_TRY(cudaGetLastError(), return ASTCENC_ERR_BAD_CONTEXT);
	ctx->launches++;
	// astcenc_entry.cpp:983-988
	size_t x_footprint = bsd.dim_x + 2 * ((size_t)radius - 1);
	size_t y_footprint = bsd.dim_y + 2 * ((size_t)radius - 1);
	float footprint = static_cast<float>(x_footprint * y_footprint);
	ctx->alpha_threshold = 0.9f / (255.0f * footprint);
	return ASTCENC_SUCCESS;
}

static astcenc_error launch_slab_locked(astcenc_context* ctx, const void* d_pixels, int data_type, unsigned int dim_x, unsigned int dim_y, const int swz[4],
                                        unsigned int block_row0, unsigned int block_rows, uint8_t* d_out, cudaStream_t stream, const UploadPlan* up) {
	const DevBsd& bsd = ctx->tables->bsd;
	size_t blocks_x = (dim_x + bsd.dim_x - 1) / bsd.dim_x;
	size_t rows_per_batch = ctx->knobs.batch_blocks / (blocks_x ? blocks_x : 1);
	if (rows_per_batch < 1) rows_per_batch = 1;
	const unsigned int radius = bsd.dim_z > 1 ? 0 : ctx->config.a_scale_radius;      // (the averages only steer 2D block sizes, astcenc_entry.cpp:975)
	// big single-batch slabs run as independent sub-slab pipelines (launch_pipes); per-launch timing wants one stream
	bool single_batch = (size_t)block_rows <= rows_per_batch;
	int pipes = ctx->knobs.pipes;
	bool use_pipes = pipes > 1 && ctx->driver == 0 && !ctx->stage_timing && single_batch && block_rows >= (unsigned int)pipes * 4 &&
	                 blocks_x * block_rows >= (size_t)pipes * 8192;
	// banded uploads need the whole slab in one batch on the wave pipeline, and no pre-pass that reads the window first
	bool banded = up != nullptr && radius == 0 && ctx->driver == 0 && single_batch && (use_pipes || (up->bands > 1 && block_rows >= (unsigned int)up->bands * 4));
	if (up != nullptr && !banded) {
		// the upload streams on the copy stream; it must not overtake a pass that still reads the image buffer
		if (ctx->scratch_used) {
			CUDA_TRY(cudaStreamWaitEvent(ctx->copy_stream, ctx->scratch_done, 0), return ASTCENC_ERR_BAD_CONTEXT);
		}
		size_t y0, y1;
		slab_image_rows(ctx, dim_y, block_row0, block_rows, y0, y1);
		astcenc_error st = upload_rows(ctx, *up, y0, y1, stream);
		if (st != ASTCENC_SUCCESS) {
			return st;
		}
		up = nullptr;
	}
	if (radius != 0 && !ctx->pass_alpha_staged) {
		// alpha-scale pre-pass over the tiles that cover the slab's rows: the box filter reaches across slab borders, so
		// the window reads up to `radius` rows beyond the tiles (alpha_window); the averages stay at their image positions
		size_t need = (size_t)dim_x * dim_y * sizeof(float);
		if (need > ctx->d_alpha_bytes) {
			cudaFree(ctx->d_alpha);
			ctx->d_alpha = nullptr;
			ctx->d_alpha_bytes = 0;
			CUDA_TRY(cudaMalloc(&ctx->d_alpha, need), return ASTCENC_ERR_OUT_OF_MEM);
			ctx->d_alpha_bytes = need;
		}
		size_t y1 = (size_t)(block_row0 + block_rows) * bsd.dim_y;
		astcenc_error st = alpha_prepass(ctx, d_pixels, data_type, dim_x, dim_y, swz, block_row0 * bsd.dim_y, y1 < dim_y ? (unsigned int)y1 : dim_y, ctx->d_alpha, stream);
		if (st != ASTCENC_SUCCESS) {
			return st;
		}
	}
	if (use_pipes) {
		return launch_pipes(ctx, pipes, d_pixels, data_type, dim_x, dim_y, swz, block_row0, block_rows, d_out, stream, banded ? up : nullptr);
	}
	unsigned int done = 0;
	while (done < block_rows) {
		unsigned int rows = block_rows - done;
		if ((size_t)rows > rows_per_batch) rows = (unsigned int)rows_per_batch;
		astcenc_error st = launch_batch(ctx, d_pixels, data_type, dim_x, dim_y, swz, block_row0 + done, rows, d_out + (size_t)done * blocks_x * 16, stream, banded ? up : nullptr);
		if (st != ASTCENC_SUCCESS) {
			return st;
		}
		done += rows;
	}
	return ASTCENC_SUCCESS;
}

static astcenc_error launch_batch(astcenc_context* ctx, const void* d_pixels, int data_type, unsigned int dim_x, unsigned int dim_y, const int swz[4],
                                  unsigned int block_row0, unsigned int block_rows, uint8_t* d_out, cudaStream_t stream, const UploadPlan* up) {
	const DevBsd& bsd = ctx->tables->bsd;
	DevImage img;
	img.data = d_pixels;
	img.data_type = data_type;
	img.dim_x = dim_x;
	img.dim_y = dim_y;
	img.dim_z = ctx->volume_dim_z;
	img.blocks_x = (dim_x + bsd.dim_x - 1) / bsd.dim_x;
	img.blocks_y = (dim_y + bsd.dim_y - 1) / bsd.dim_y;
	img.block_row0 = block_row0;
	img.block_rows = block_rows;
	for (int i = 0; i < 4; i++) {
		img.swz[i] = swz[i];
	}
	img.out = d_out;
	img.alpha_avg = ctx->config.a_scale_radius != 0 && bsd.dim_z == 1 ? ctx->d_alpha : nullptr;
	img.alpha_threshold = ctx->alpha_threshold;
	img.cancel = ctx->pass_cancel;
	img.done = ctx->pass_done;
	size_t total = (size_t)img.blocks_x * block_rows;
	if (ctx->driver == 0) {
		// ---- wave pipeline ----
		if (total > ctx->queue_capacity) {
			cudaFree(ctx->d_queues);
			ctx->d_queues = nullptr;
			ctx->queue_capacity = 0;
			CUDA_TRY(cudaMalloc(&ctx->d_queues, sizeof(uint32_t) * ASTC_Q_KINDS * total), return ASTCENC_ERR_OUT_OF_MEM);
			ctx->queue_capacity = total;
		}
		size_t rec_bytes = total * (size_t)bsd.record_bytes;
		if (rec_bytes > ctx->d_records_bytes) {
			cudaFree(ctx->d_records);
			ctx->d_records = nullptr;
			ctx->d_records_bytes = 0;
			CUDA_TRY(cudaMalloc(&ctx->d_records, rec_bytes), return ASTCENC_ERR_OUT_OF_MEM);
			ctx->d_records_bytes = rec_bytes;
		}
		CUDA_TRY(cudaMemsetAsync(ctx->d_counters, 0, sizeof(uint32_t) * ASTC_COUNTER_WORDS, stream), return ASTCENC_ERR_BAD_CONTEXT);
		WaveArgs a;
		a.records = ctx->d_records;
		a.queues = ctx->d_queues;
		a.queue_stride = ctx->queue_capacity;
		a.count = ctx->d_counters;
		a.head = ctx->d_counters + ASTC_Q_KINDS * ASTC_MAX_WAVES;
		a.total = (unsigned int)total;
		a.blocks_x = img.blocks_x;
		a.ticket = ctx->d_counters + 2 * ASTC_Q_KINDS * ASTC_MAX_WAVES;
		a.first_block = 0;
		a.band_blocks = (unsigned int)total;
		a.cls_lo = 0;
		a.cls_hi = ASTC_Q_CLASSES;
		a.stage_bytes = ctx->refine_stage_bytes;
		a.refine_state_off = (uint32_t)(ASTC_SMEM_HDR + ctx->refine_stage_bytes + (size_t)bsd.arena_bytes_small * ctx->warps_small);
		a.stage_bytes_setup = ctx->setup_stage_bytes;
		a.sync_mask = ctx->knobs.sync_mask;
		int grid = ctx->grid;
		size_t ev_used = 0;
		auto mark = [&](int kind) {
			if (!ctx->stage_timing) {
				return;
			}
			if (ev_used == ctx->stage_events.size()) {
				cudaEvent_t e;
				if (cudaEventCreate(&e) != cudaSuccess) {
					return;
				}
				ctx->stage_events.push_back(e);
				ctx->stage_kinds.push_back(kind);
			}
			ctx->stage_kinds[ev_used] = kind;
			cudaEventRecord(ctx->stage_events[ev_used++], stream);
		};
		if (ctx->stage_timing) {
			ctx->stage_kinds.clear();
			ctx->stage_kinds.resize(ctx->stage_events.size(), -1);
		}
		mark(-1);
		for (int wave = 0; wave < ctx->max_waves; wave++) {
			a.wave = wave;
			a.sync_mask = wave == 0 ? ctx->knobs.sync_mask : ctx->knobs.sync_mask_tail;
			if (wave == 0 && up != nullptr) {
				// bands of block rows, growing (1 : 3 : 4 : 8 ...) so that the first copy - the only one nothing hides - is short
				static const unsigned int shares[ASTC_MAX_BANDS] = {1, 3, 4, 8, 8, 8, 8, 8};
				unsigned int sum = 0;
				for (int k = 0; k < up->bands; k++) sum += shares[k];
				if (ctx->scratch_used) {
					CUDA_TRY(cudaStreamWaitEvent(ctx->copy_stream, ctx->scratch_done, 0), return ASTCENC_ERR_BAD_CONTEXT);
				}
				unsigned int row = 0, acc = 0;
				for (int k = 0; k < up->bands; k++) {
					acc += shares[k];
					unsigned int row_end = k == up->bands - 1 ? block_rows : (unsigned int)((size_t)block_rows * acc / sum);
					if (row_end <= row) {
						continue;
					}
					// image rows of block rows [row, row_end) of this slab
					size_t y0 = (size_t)(block_row0 + row) * bsd.dim_y;
					size_t y1 = (size_t)(block_row0 + row_end) * bsd.dim_y;
					if (y1 > dim_y) y1 = dim_y;
					if (y1 > y0) {
						CUDA_TRY(cudaMemcpyAsync(up->device + y0 * up->row_bytes, up->host + y0 * up->row_bytes, (y1 - y0) * up->row_bytes, cudaMemcpyHostToDevice, ctx->copy_stream),
						         return ASTCENC_ERR_BAD_CONTEXT);
					}
					CUDA_TRY(cudaEventRecord(ctx->band_ready[k], ctx->copy_stream), return ASTCENC_ERR_BAD_CONTEXT);
					CUDA_TRY(cudaStreamWaitEvent(stream, ctx->band_ready[k], 0), return ASTCENC_ERR_BAD_CONTEXT);
					a.ticket = ctx->d_counters + 2 * ASTC_Q_KINDS * ASTC_MAX_WAVES + k;
					a.first_block = row * img.blocks_x;
					a.band_blocks = (row_end - row) * img.blocks_x;
					if (ctx->warps_setup_1p) {
						setup_kernel(ctx->dcfg, 0)<<<grid, ctx->warps_setup_1p * 32, ctx->smem_setup_1p, stream>>>(ctx->tables->bsd_1p, ctx->dcfg, img, a);
					} else {
						setup_kernel(ctx->dcfg, 0)<<<grid, ctx->warps_setup * 32, ctx->smem_setup, stream>>>(bsd, ctx->dcfg, img, a);
					}
					ctx->launches++;
					row = row_end;
				}
				mark(0);
				ctx->launches--;      // (the loop below counts one set-up launch per wave)
			} else if (ctx->warps_setup_1p) {
				// class 0 of the later waves holds the two-plane trials (general plan); wave 0 and the n-partition classes have
				// one weight plane and run on the compact plan with more warps per SM
				if (wave != 0) {
					a.cls_lo = 0;
					a.cls_hi = 1;
					astc_wave_setup_kernel<false><<<grid, ctx->warps_setup * 32, ctx->smem_setup, stream>>>(bsd, ctx->dcfg, img, a);
					ctx->launches++;
					a.cls_lo = 1;
					a.cls_hi = ASTC_Q_CLASSES;
				}
				setup_kernel(ctx->dcfg, wave)<<<grid, ctx->warps_setup_1p * 32, ctx->smem_setup_1p, stream>>>(ctx->tables->bsd_1p, ctx->dcfg, img, a);
				a.cls_lo = 0;
				a.cls_hi = ASTC_Q_CLASSES;
				mark(0);
			} else {
				setup_kernel(ctx->dcfg, wave)<<<grid, ctx->warps_setup * 32, ctx->smem_setup, stream>>>(bsd, ctx->dcfg, img, a);
				mark(0);
			}
			if (refine_l1_step(ctx->dcfg)) {
				astc_wave_refine_kernel<true><<<grid * ctx->refine_ctas, ctx->warps_small * 32, ctx->smem_refine, stream>>>(bsd, ctx->dcfg, img, a);
			} else {
				astc_wave_refine_kernel<false><<<grid * ctx->refine_ctas, ctx->warps_small * 32, ctx->smem_refine, stream>>>(bsd, ctx->dcfg, img, a);
			}
			mark(1);
			// (statistics / partition search gain nothing from phase alignment: two half-size CTAs per SM wait less)
			int wp = ctx->warps_small >= 2 ? ctx->warps_small / 2 : 1;
			astc_wave_prepare_kernel<<<grid * 2, wp * 32, ASTC_SMEM_HDR + (size_t)bsd.arena_bytes_small * wp, stream>>>(bsd, ctx->dcfg, img, a);
			mark(2);
			ctx->launches += 3;
		}
		a.wave = 0;
		astc_wave_emit_kernel<<<grid * 4, ASTC_EMIT_THREADS, ASTC_SMEM_HDR + (ASTC_EMIT_THREADS / 32) * 32 * EMIT_SLICE, stream>>>(bsd, ctx->dcfg, img, a);
		mark(3);
		if (ctx->stage_timing) {
			ctx->stage_kinds.resize(ev_used);
		}
		ctx->launches++;
		CUDA_TRY(cudaGetLastError(), return ASTCENC_ERR_BAD_CONTEXT);
		return ASTCENC_SUCCESS;
	}
	CUDA_TRY(cudaMemsetAsync(ctx->d_ticket, 0, sizeof(unsigned int), stream), return ASTCENC_ERR_BAD_CONTEXT);
	int grid = ctx->grid;
	size_t needed = (total + ctx->warps_per_cta - 1) / ctx->warps_per_cta;
	if ((size_t)grid > needed) {
		grid = (int)(needed ? needed : 1);
	}
	astc_compress_kernel<<<grid, ctx->warps_per_cta * 32, ctx->smem_bytes, stream>>>(bsd, ctx->dcfg, img, ctx->d_ticket, ctx->knobs.coherence_probe, ctx->lockstep);
	CUDA_TRY(cudaGetLastError(), return ASTCENC_ERR_BAD_CONTEXT);
	ctx->launches++;
	return ASTCENC_SUCCESS;
}

static astcenc_error ensure_buffer(uint8_t*& buf, size_t& have, size_t need) {
	if (have < need) {
		cudaFree(buf);
		buf = nullptr;
		have = 0;
		CUDA_TRY(cudaMalloc(&buf, need), return ASTCENC_ERR_OUT_OF_MEM);
		have = need;
	}
	return ASTCENC_SUCCESS;
}

// Progress of one astcenc_compress_image call, reported like the reference's task pool (astcenc_internal_entry.h:199-295):
// value = done / total * 100 over the blocks of the whole image, a call whenever it has moved by more than
// max(1 %, 4096 blocks) since the last call, and exactly one call with 100 once the payload is in the caller's buffer.
// The counter is read every ASTC_POLL_US: 1 ms is a tenth of the 1 % step of a 100 ms pass (a pass that short needs no
// finer bar), a read costs the host thread one 4-byte copy (~10 us), and a finished or cancelled pass is noticed within 1 ms.
#define ASTC_POLL_US 1000
struct PassProgress {
	astcenc_progress_callback callback;     // null: no polling, the pass is waited for with a plain synchronise
	float total;                            // blocks of the whole image
	float min_diff;
	float last;
};

// Waits until `end` (recorded on the pass stream after the pass's kernels) has completed; with a callback, polls the done
// counter meanwhile and reports progress. The callback may call astcenc_compress_cancel.
static astcenc_error wait_pass(astcenc_context* ctx, cudaEvent_t end, PassProgress& pp) {
	if (!pp.callback) {
		CUDA_TRY(cudaEventSynchronize(end), return ASTCENC_ERR_BAD_CONTEXT);
		return ASTCENC_SUCCESS;
	}
	while (true) {
		cudaError_t q = cudaEventQuery(end);
		if (q == cudaSuccess) {
			return ASTCENC_SUCCESS;
		}
		if (q != cudaErrorNotReady) {
			CUDA_TRY(q, return ASTCENC_ERR_BAD_CONTEXT);
		}
		std::this_thread::sleep_for(std::chrono::microseconds(ASTC_POLL_US));
		CUDA_TRY(cudaMemcpyAsync(ctx->h_words + 2, ctx->d_words + 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->ctl_stream), return ASTCENC_ERR_BAD_CONTEXT);
		CUDA_TRY(cudaStreamSynchronize(ctx->ctl_stream), return ASTCENC_ERR_BAD_CONTEXT);
		float value = (static_cast<float>(ctx->h_words[2]) / pp.total) * 100.0f;
		// (100 is reported once, after the payload copy; nothing is reported once the pass is cancelled)
		if (value < 100.0f && value - pp.last > pp.min_diff && !ctx->cancel.load()) {
			pp.callback(value);
			pp.last = value;
		}
	}
}

// The host-pointer path (what the reference's callers use: astcenccli_toplevel.cpp:2195-2215 passes plain heap memory).
// The image goes up in bands on the copy stream while wave 0 already works on the bands that arrived; the payload comes
// back with one copy when the emit kernel is done. Works with pageable and with pinned host memory alike (with pageable
// memory the driver stages each band through its own pinned buffers and the call blocks for the band's duration -
// the kernels of the earlier bands are running meanwhile).
// A cancelled call (astcenc_compress_cancel) skips the remaining slices and copies no payload back: the caller's buffer keeps
// its bytes, and the call still returns ASTCENC_SUCCESS (astcenc.h: the data is then undefined).
static astcenc_error compress_image_gpu(astcenc_context* ctx, const astcenc_image& image, const astcenc_swizzle& swizzle, uint8_t* data_out) {
	const DevBsd& bsd = ctx->tables->bsd;
	DeviceGuard guard(ctx->device);
	if (!guard.ok) {
		return ASTCENC_ERR_BAD_CONTEXT;
	}
	size_t bpt = image.data_type == ASTCENC_TYPE_U8 ? 4 : image.data_type == ASTCENC_TYPE_F16 ? 8 : 16;
	size_t slice_bytes = (size_t)image.dim_x * image.dim_y * bpt;
	size_t blocks_x = block_count_axis(image.dim_x, bsd.dim_x);
	size_t blocks_y = block_count_axis(image.dim_y, bsd.dim_y);
	size_t out_bytes = blocks_x * blocks_y * 16;
	astcenc_error st = ensure_buffer(ctx->d_image, ctx->d_image_bytes, slice_bytes);
	if (st == ASTCENC_SUCCESS) {
		st = ensure_buffer(ctx->d_out, ctx->d_out_bytes, out_bytes);
	}
	if (st != ASTCENC_SUCCESS) {
		return st;
	}
	int swz[4] = {(int)swizzle.r, (int)swizzle.g, (int)swizzle.b, (int)swizzle.a};
	ctx->last_h2d = ctx->last_d2h = 0;
	ctx->last_kernel_ms = 0.0f;
	float total_ms = 0.0f;
	// the pass starts behind the last flag clear (astcenc_compress_reset), with its done counter at zero
	uint32_t* d_cancel = ctx->d_words;
	uint32_t* d_done = ctx->d_words + 1;
	CUDA_TRY(cudaStreamWaitEvent(ctx->stream, ctx->ctl_ready, 0), return ASTCENC_ERR_BAD_CONTEXT);
	CUDA_TRY(cudaMemsetAsync(d_done, 0, sizeof(uint32_t), ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
	PassProgress pp;
	pp.callback = ctx->config.progress_callback;
	pp.total = static_cast<float>(blocks_x * blocks_y * (bsd.dim_z > 1 ? block_count_axis(image.dim_z, bsd.dim_z) : (size_t)image.dim_z));
	pp.min_diff = (4096.0f / pp.total) * 100.0f;
	pp.min_diff = pp.min_diff > 1.0f ? pp.min_diff : 1.0f;
	pp.last = 0.0f;
	if (bsd.dim_z > 1) {
		// 3D block sizes (astcenc_entry.cpp:906-1043): the slices go up into one contiguous volume, the blocks come out in (z, y, x)
		// order; "block rows" of the pass count layer * blocks_y + row
		size_t blocks_z = block_count_axis(image.dim_z, bsd.dim_z);
		size_t vol_out = out_bytes * blocks_z;
		st = ensure_buffer(ctx->d_image, ctx->d_image_bytes, slice_bytes * image.dim_z);
		if (st == ASTCENC_SUCCESS) {
			st = ensure_buffer(ctx->d_out, ctx->d_out_bytes, vol_out);
		}
		if (st != ASTCENC_SUCCESS) {
			return st;
		}
		if (ctx->cancel.load()) {
			return ASTCENC_SUCCESS;
		}
		for (unsigned int z = 0; z < image.dim_z; z++) {
			CUDA_TRY(cudaMemcpyAsync(ctx->d_image + (size_t)z * slice_bytes, image.data[z], slice_bytes, cudaMemcpyHostToDevice, ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
		}
		CUDA_TRY(cudaEventRecord(ctx->ev0, ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
		st = launch_slab(ctx, ctx->d_image, (int)image.data_type, image.dim_x, image.dim_y, swz, 0, (unsigned int)(blocks_y * blocks_z), ctx->d_out, ctx->stream, nullptr, image.dim_z,
		                 d_cancel, d_done);
		if (st != ASTCENC_SUCCESS) {
			return st;
		}
		CUDA_TRY(cudaEventRecord(ctx->ev1, ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
		st = wait_pass(ctx, ctx->ev1, pp);
		if (st != ASTCENC_SUCCESS) {
			return st;
		}
		if (ctx->cancel.load()) {
			return ASTCENC_SUCCESS;
		}
		CUDA_TRY(cudaMemcpyAsync(data_out, ctx->d_out, vol_out, cudaMemcpyDeviceToHost, ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
		CUDA_TRY(cudaStreamSynchronize(ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
		cudaEventElapsedTime(&total_ms, ctx->ev0, ctx->ev1);
		ctx->last_kernel_ms = total_ms;
		ctx->last_h2d = slice_bytes * image.dim_z;
		ctx->last_d2h = vol_out;
		if (pp.callback) {
			pp.callback(100.0f);
		}
		return ASTCENC_SUCCESS;
	}
	// 3D images with 2D blocks are an array of independent 2D slices (astcenc.h:94-100); progress runs over all of them
	for (unsigned int z = 0; z < image.dim_z; z++) {
		if (ctx->cancel.load()) {
			return ASTCENC_SUCCESS;
		}
		UploadPlan up;
		up.host = static_cast<const uint8_t*>(image.data[z]);
		up.device = ctx->d_image;
		up.row_bytes = (size_t)image.dim_x * bpt;
		up.bands = ctx->knobs.upload_bands;
		CUDA_TRY(cudaEventRecord(ctx->ev0, ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
		st = launch_slab(ctx, ctx->d_image, (int)image.data_type, image.dim_x, image.dim_y, swz, 0, (unsigned int)blocks_y, ctx->d_out, ctx->stream, &up, 1, d_cancel, d_done);
		if (st != ASTCENC_SUCCESS) {
			return st;
		}
		CUDA_TRY(cudaEventRecord(ctx->ev1, ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
		st = wait_pass(ctx, ctx->ev1, pp);
		if (st != ASTCENC_SUCCESS) {
			return st;
		}
		if (ctx->cancel.load()) {
			return ASTCENC_SUCCESS;
		}
		CUDA_TRY(cudaMemcpyAsync(data_out + (size_t)z * out_bytes, ctx->d_out, out_bytes, cudaMemcpyDeviceToHost, ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
		CUDA_TRY(cudaStreamSynchronize(ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
		float ms = 0.0f;
		cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1);
		total_ms += ms;
		ctx->last_h2d += slice_bytes;
		ctx->last_d2h += out_bytes;
	}
	ctx->last_kernel_ms = total_ms;
	if (pp.callback) {
		pp.callback(100.0f);
	}
	return ASTCENC_SUCCESS;
}

astcenc_error astcenc_compress_reset(astcenc_context* ctx);

astcenc_error astcenc_compress_image(astcenc_context* ctx, astcenc_image* imagep, const astcenc_swizzle* swizzle, uint8_t* data_out, size_t data_len,
                                     unsigned int thread_index) {
	if (ctx->config.flags & ASTCENC_FLG_DECOMPRESS_ONLY) {
		return ASTCENC_ERR_BAD_CONTEXT;
	}
	astcenc_error status = validate_compression_swizzle(*swizzle);
	if (status != ASTCENC_SUCCESS) {
		return status;
	}
	if (thread_index >= ctx->thread_count) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	const astcenc_image& image = *imagep;
	bool overflow = false;
	size_t texel_count = mul_safe(mul_safe(image.dim_x, image.dim_y, overflow), image.dim_z, overflow);
	if (overflow || texel_count == 0) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	size_t blocks_x = block_count_axis(image.dim_x, ctx->config.block_x);
	size_t blocks_y = block_count_axis(image.dim_y, ctx->config.block_y);
	size_t blocks_z = block_count_axis(image.dim_z, ctx->config.block_z);
	overflow = false;
	size_t block_count = mul_safe(mul_safe(blocks_x, blocks_y, overflow), blocks_z, overflow);
	mul_safe(block_count, 16, overflow);
	if (overflow || block_count == 0) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	if (data_len < block_count * 16) {
		return ASTCENC_ERR_OUT_OF_MEM;
	}
	if (ctx->config.a_scale_radius != 0 && image.dim_z != 1 && ctx->config.block_z <= 1) {
		// the alpha-scale pre-pass is built for 2D images; volumes would average across slices (compute_variance.cpp have_z)
		return ASTCENC_ERR_NOT_IMPLEMENTED;
	}
	if (ctx->thread_count == 1) {
		astcenc_compress_reset(ctx);
	}
	std::unique_lock<std::mutex> lk(ctx->mtx);
	if (ctx->state == 0) {
		ctx->state = 1;
		lk.unlock();
		astcenc_error r = compress_image_gpu(ctx, image, *swizzle, data_out);
		lk.lock();
		ctx->result = r;
		ctx->state = 2;
		ctx->cv.notify_all();
		return r;
	}
	ctx->cv.wait(lk, [ctx] { return ctx->state == 2; });
	return ctx->result;
}

astcenc_error astcenc_compress_reset(astcenc_context* ctx) {
	if (ctx->config.flags & ASTCENC_FLG_DECOMPRESS_ONLY) {
		return ASTCENC_ERR_BAD_CONTEXT;
	}
	std::lock_guard<std::mutex> lk(ctx->mtx);
	if (ctx->state != 1) {
		ctx->state = 0;
	}
	std::lock_guard<std::mutex> fl(ctx->flag_mtx);
	ctx->cancel = false;
	if (ctx->flag_raised) {
		// clear the device flag on the control stream (behind any raise enqueued before) and start the next pass behind it
		DeviceGuard guard(ctx->device);
		CUDA_TRY(cudaMemcpyAsync(ctx->d_words, ctx->h_words, sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->ctl_stream), return ASTCENC_ERR_BAD_CONTEXT);
		CUDA_TRY(cudaEventRecord(ctx->ctl_ready, ctx->ctl_stream), return ASTCENC_ERR_BAD_CONTEXT);
		ctx->flag_raised = false;
	}
	return ASTCENC_SUCCESS;
}

// Takes neither ctx->mtx nor launch_mtx: it is called from other threads while a pass runs, and from inside the progress
// callback on the thread that runs the pass.
astcenc_error astcenc_compress_cancel(astcenc_context* ctx) {
	if (ctx->config.flags & ASTCENC_FLG_DECOMPRESS_ONLY) {
		return ASTCENC_ERR_BAD_CONTEXT;
	}
	std::lock_guard<std::mutex> fl(ctx->flag_mtx);
	ctx->cancel = true;
	// a 4-byte DMA from pinned memory on the control stream: it lands while the pass's kernels run, and their next look at the
	// flag finds every queue empty
	DeviceGuard guard(ctx->device);
	CUDA_TRY(cudaMemcpyAsync(ctx->d_words, ctx->h_words + 1, sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->ctl_stream), return ASTCENC_ERR_BAD_CONTEXT);
	ctx->flag_raised = true;
	return ASTCENC_SUCCESS;
}

static astcenc_error validate_decompression_swizzle(const astcenc_swizzle& s) {   // astcenc_entry.cpp:279-300: r,g,b,a,0,1 and Z
	const int v[4] = {(int)s.r, (int)s.g, (int)s.b, (int)s.a};
	for (int i = 0; i < 4; i++) {
		if (v[i] < ASTCENC_SWZ_R || v[i] > ASTCENC_SWZ_Z) {
			return ASTCENC_ERR_BAD_SWIZZLE;
		}
	}
	return ASTCENC_SUCCESS;
}

static astcenc_error decompress_image_gpu(astcenc_context* ctx, const uint8_t* data, astcenc_image& image, const astcenc_swizzle& swizzle) {
	const DevBsd& bsd = ctx->tables->bsd;
	DeviceGuard guard(ctx->device);
	if (!guard.ok) {
		return ASTCENC_ERR_BAD_CONTEXT;
	}
	std::lock_guard<std::mutex> launch_lock(ctx->launch_mtx);      // (shares d_image / d_out with the compression path)
	if (ctx->scratch_used) {
		CUDA_TRY(cudaStreamWaitEvent(ctx->stream, ctx->scratch_done, 0), return ASTCENC_ERR_BAD_CONTEXT);
	}
	size_t bpt = image.data_type == ASTCENC_TYPE_U8 ? 4 : image.data_type == ASTCENC_TYPE_F16 ? 8 : 16;
	size_t slice_bytes = (size_t)image.dim_x * image.dim_y * bpt;
	size_t blocks_x = block_count_axis(image.dim_x, bsd.dim_x);
	size_t blocks_y = block_count_axis(image.dim_y, bsd.dim_y);
	// 3D block sizes decode the volume in one pass (blocks in z, y, x order); 2D block sizes take it slice by slice
	const bool volume = bsd.dim_z > 1;
	size_t blocks_z = volume ? block_count_axis(image.dim_z, bsd.dim_z) : 1;
	size_t in_bytes = blocks_x * blocks_y * blocks_z * 16;
	size_t image_bytes = volume ? slice_bytes * image.dim_z : slice_bytes;
	if (ctx->d_image_bytes < image_bytes) {
		cudaFree(ctx->d_image);
		ctx->d_image = nullptr;
		ctx->d_image_bytes = 0;
		CUDA_TRY(cudaMalloc(&ctx->d_image, image_bytes), return ASTCENC_ERR_OUT_OF_MEM);
		ctx->d_image_bytes = image_bytes;
	}
	if (ctx->d_out_bytes < in_bytes) {
		cudaFree(ctx->d_out);
		ctx->d_out = nullptr;
		ctx->d_out_bytes = 0;
		CUDA_TRY(cudaMalloc(&ctx->d_out, in_bytes), return ASTCENC_ERR_OUT_OF_MEM);
		ctx->d_out_bytes = in_bytes;
	}
	DevImage img;
	img.data = ctx->d_image;
	img.data_type = (int)image.data_type;
	img.dim_x = image.dim_x;
	img.dim_y = image.dim_y;
	img.dim_z = volume ? image.dim_z : 1;
	img.blocks_x = (unsigned int)blocks_x;
	img.blocks_y = (unsigned int)blocks_y;
	img.block_row0 = 0;
	img.block_rows = (unsigned int)(blocks_y * blocks_z);
	img.swz[0] = (int)swizzle.r;
	img.swz[1] = (int)swizzle.g;
	img.swz[2] = (int)swizzle.b;
	img.swz[3] = (int)swizzle.a;
	img.out = nullptr;
	img.alpha_avg = nullptr;
	img.alpha_threshold = 0.0f;
	img.cancel = nullptr;
	img.done = nullptr;
	cudaDeviceProp prop;
	CUDA_TRY(cudaGetDeviceProperties(&prop, ctx->device), return ASTCENC_ERR_BAD_CONTEXT);
	unsigned int nblocks = (unsigned int)(blocks_x * blocks_y * blocks_z);
	int warps = ASTC_DECODE_THREADS / 32;
	int grid = (int)((nblocks + warps - 1) / warps);
	if (grid > prop.multiProcessorCount * 8) {
		grid = prop.multiProcessorCount * 8;
	}
	if (volume) {
		CUDA_TRY(cudaMemcpyAsync(ctx->d_out, data, in_bytes, cudaMemcpyHostToDevice, ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
		astc_decompress_kernel<<<grid, ASTC_DECODE_THREADS, ASTC_SMEM_HDR + warps * D_SLICE, ctx->stream>>>(bsd, ctx->dcfg, img, ctx->d_out, nblocks);
		CUDA_TRY(cudaGetLastError(), return ASTCENC_ERR_BAD_CONTEXT);
		ctx->launches++;
		for (unsigned int z = 0; z < image.dim_z; z++) {
			CUDA_TRY(cudaMemcpyAsync(image.data[z], ctx->d_image + (size_t)z * slice_bytes, slice_bytes, cudaMemcpyDeviceToHost, ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
		}
		CUDA_TRY(cudaStreamSynchronize(ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
		return ASTCENC_SUCCESS;
	}
	// 3D images with 2D blocks are an array of independent 2D slices; blocks of slice z follow those of slice z - 1
	for (unsigned int z = 0; z < image.dim_z; z++) {
		CUDA_TRY(cudaMemcpyAsync(ctx->d_out, data + (size_t)z * in_bytes, in_bytes, cudaMemcpyHostToDevice, ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
		astc_decompress_kernel<<<grid, ASTC_DECODE_THREADS, ASTC_SMEM_HDR + warps * D_SLICE, ctx->stream>>>(bsd, ctx->dcfg, img, ctx->d_out, nblocks);
		CUDA_TRY(cudaGetLastError(), return ASTCENC_ERR_BAD_CONTEXT);
		ctx->launches++;
		CUDA_TRY(cudaMemcpyAsync(image.data[z], ctx->d_image, slice_bytes, cudaMemcpyDeviceToHost, ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
		CUDA_TRY(cudaStreamSynchronize(ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
	}
	return ASTCENC_SUCCESS;
}

// astcenc_decompress_image (astcenc_entry.cpp:1274-1385): same check order; the decode mode follows the output type
astcenc_error astcenc_decompress_image(astcenc_context* ctx, const uint8_t* data, size_t data_len, astcenc_image* image_outp, const astcenc_swizzle* swizzle,
                                       unsigned int thread_index) {
	if (thread_index >= ctx->thread_count) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	astcenc_error status = validate_decompression_swizzle(*swizzle);
	if (status != ASTCENC_SUCCESS) {
		return status;
	}
	astcenc_image& image = *image_outp;
	bool overflow = false;
	size_t texel_count = mul_safe(mul_safe(image.dim_x, image.dim_y, overflow), image.dim_z, overflow);
	if (overflow || texel_count == 0) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	size_t blocks_x = block_count_axis(image.dim_x, ctx->config.block_x);
	size_t blocks_y = block_count_axis(image.dim_y, ctx->config.block_y);
	size_t blocks_z = block_count_axis(image.dim_z, ctx->config.block_z);
	overflow = false;
	size_t block_count = mul_safe(mul_safe(blocks_x, blocks_y, overflow), blocks_z, overflow);
	mul_safe(block_count, 16, overflow);
	if (overflow || block_count == 0) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	if (data_len < block_count * 16) {
		return ASTCENC_ERR_OUT_OF_MEM;
	}
	// any subset of the thread_count callers may call; the image is decoded once, everybody returns when it is done
	if (ctx->thread_count == 1) {
		astcenc_decompress_reset(ctx);
	}
	std::unique_lock<std::mutex> lk(ctx->mtx);
	if (ctx->dstate == 0) {
		ctx->dstate = 1;
		lk.unlock();
		astcenc_error r = decompress_image_gpu(ctx, data, image, *swizzle);
		lk.lock();
		ctx->dresult = r;
		ctx->dstate = 2;
		ctx->cv.notify_all();
		return r;
	}
	ctx->cv.wait(lk, [ctx] { return ctx->dstate == 2; });
	return ctx->dresult;
}

astcenc_error astcenc_decompress_reset(astcenc_context* ctx) {
	std::lock_guard<std::mutex> lk(ctx->mtx);
	if (ctx->dstate != 1) {
		ctx->dstate = 0;
	}
	return ASTCENC_SUCCESS;
}

// astcenc_get_block_info (astcenc_entry.cpp:1401-1517). A query for tools: one 32-thread launch per call.
astcenc_error astcenc_get_block_info(astcenc_context* ctx, const uint8_t data[16], astcenc_block_info* info) {
	memset(info, 0, sizeof(*info));
	info->profile = ctx->config.profile;
	info->block_x = ctx->config.block_x;
	info->block_y = ctx->config.block_y;
	info->block_z = ctx->config.block_z;
	info->texel_count = ctx->tables->bsd.texel_count;
	DeviceGuard guard(ctx->device);
	if (!guard.ok) {
		return ASTCENC_ERR_BAD_CONTEXT;
	}
	DevBlockInfo* d_info = nullptr;
	CUDA_TRY(cudaMalloc(&d_info, sizeof(DevBlockInfo)), return ASTCENC_ERR_OUT_OF_MEM);
	cudaMemsetAsync(d_info, 0, sizeof(DevBlockInfo), ctx->stream);
	unsigned long long lo, hi;
	memcpy(&lo, data, 8);
	memcpy(&hi, data + 8, 8);
	DevImage img{};
	astc_block_info_kernel<<<1, 32, ASTC_SMEM_HDR + D_SLICE, ctx->stream>>>(ctx->tables->bsd, ctx->dcfg, img, lo, hi, d_info);
	ctx->launches++;
	DevBlockInfo h;
	cudaError_t e = cudaMemcpyAsync(&h, d_info, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream);
	if (e == cudaSuccess) {
		e = cudaStreamSynchronize(ctx->stream);
	}
	cudaFree(d_info);
	if (e != cudaSuccess) {
		return ASTCENC_ERR_BAD_CONTEXT;
	}
	info->is_error_block = h.is_error_block != 0;
	if (info->is_error_block) {
		return ASTCENC_SUCCESS;
	}
	info->is_constant_block = h.is_constant_block != 0;
	if (info->is_constant_block) {
		return ASTCENC_SUCCESS;
	}
	info->is_hdr_block = h.is_hdr_block != 0;
	info->is_dual_plane_block = h.is_dual_plane_block != 0;
	info->partition_count = h.partition_count;
	info->partition_index = h.partition_index;
	info->dual_plane_component = h.dual_plane_component;
	info->color_level_count = h.color_level_count;
	info->weight_level_count = h.weight_level_count;
	info->weight_x = h.weight_x;
	info->weight_y = h.weight_y;
	info->weight_z = h.weight_z;
	for (unsigned int p = 0; p < h.partition_count && p < 4; p++) {
		info->color_endpoint_modes[p] = h.color_endpoint_modes[p];
		memcpy(info->color_endpoints[p], h.color_endpoints[p], sizeof(h.color_endpoints[p]));
	}
	for (unsigned int i = 0; i < info->texel_count; i++) {
		info->weight_values_plane1[i] = h.weight_values_plane1[i];
		if (info->is_dual_plane_block) {
			info->weight_values_plane2[i] = h.weight_values_plane2[i];
		}
		info->partition_assignment[i] = h.partition_assignment[i];
	}
	return ASTCENC_SUCCESS;
}

// astcenc_b200_compute_error_metrics: the CLI's compute_error_metrics (astcenccli_error_metrics.cpp:109-413) with the
// per-texel work and the reductions on the device; the final dB figures are computed here exactly as the CLI prints them.
astcenc_error astcenc_b200_compute_error_metrics(astcenc_context* ctx, int compute_hdr_metrics, int compute_normal_metrics, int input_components,
                                                 const astcenc_image* img1, const astcenc_image* img2, int fstop_lo, int fstop_hi,
                                                 astcenc_b200_error_metrics* out) {
	if (!ctx || !img1 || !img2 || !out || input_components < 1 || input_components > 4 || !img1->data || !img2->data) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	if (fstop_lo < -125 || fstop_hi > 125) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	if ((int)img1->data_type < 0 || (int)img1->data_type > 2 || (int)img2->data_type < 0 || (int)img2->data_type > 2) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	memset(out, 0, sizeof(*out));
	unsigned int dim_x = img1->dim_x < img2->dim_x ? img1->dim_x : img2->dim_x;
	unsigned int dim_y = img1->dim_y < img2->dim_y ? img1->dim_y : img2->dim_y;
	unsigned int dim_z = img1->dim_z < img2->dim_z ? img1->dim_z : img2->dim_z;
	if (dim_x == 0 || dim_y == 0 || dim_z == 0) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	DeviceGuard guard(ctx->device);
	if (!guard.ok) {
		return ASTCENC_ERR_BAD_CONTEXT;
	}
	static const size_t comp_bytes[3] = {1, 2, 4};
	size_t slice1 = (size_t)img1->dim_x * img1->dim_y * 4 * comp_bytes[img1->data_type];
	size_t slice2 = (size_t)img2->dim_x * img2->dim_y * 4 * comp_bytes[img2->data_type];
	// a fixed partition of the sums (not one derived from the SM count), so the figures are the same on every GPU
	int ctas = 592;
	size_t texels = (size_t)dim_x * dim_y;
	if ((size_t)ctas * 256 > texels) {
		ctas = (int)((texels + 255) / 256);
	}
	uint8_t* d1 = nullptr;
	uint8_t* d2 = nullptr;
	double* d_part = nullptr;
	astcenc_error status = ASTCENC_SUCCESS;
	double sums[ASTC_METRIC_SUMS];
	do {
		if (cudaMalloc(&d1, slice1) != cudaSuccess || cudaMalloc(&d2, slice2) != cudaSuccess ||
		    cudaMalloc(&d_part, ((size_t)ctas * dim_z + 1) * ASTC_METRIC_SUMS * sizeof(double)) != cudaSuccess) {
			status = ASTCENC_ERR_OUT_OF_MEM;
			break;
		}
		MetricArgs a;
		a.img1.type = (int)img1->data_type;
		a.img1.dim_x = img1->dim_x;
		a.img2.type = (int)img2->data_type;
		a.img2.dim_x = img2->dim_x;
		a.dim_x = dim_x;
		a.dim_y = dim_y;
		a.hdr = compute_hdr_metrics != 0;
		a.normal = compute_normal_metrics != 0;
		a.fstop_lo = fstop_lo;
		a.fstop_hi = fstop_hi;
		a.inv_pixels = 1.0 / (double)(dim_x * dim_y * dim_z);      // (unsigned product, like the reference's :281)
		cudaError_t e = cudaSuccess;
		for (unsigned int z = 0; z < dim_z && e == cudaSuccess; z++) {
			// (stream-ordered: the next slice's copy waits for this slice's kernel)
			e = cudaMemcpyAsync(d1, img1->data[z], slice1, cudaMemcpyHostToDevice, ctx->stream);
			if (e == cudaSuccess) e = cudaMemcpyAsync(d2, img2->data[z], slice2, cudaMemcpyHostToDevice, ctx->stream);
			a.img1.data = d1;
			a.img2.data = d2;
			a.partials = d_part + (size_t)z * ctas * ASTC_METRIC_SUMS;
			astc_error_metrics_kernel<<<ctas, 256, 0, ctx->stream>>>(a);
			ctx->launches++;
		}
		double* d_out = d_part + (size_t)ctas * dim_z * ASTC_METRIC_SUMS;
		astc_error_metrics_finish_kernel<<<1, 32, 0, ctx->stream>>>(d_part, ctas * (int)dim_z, d_out);
		ctx->launches++;
		if (e == cudaSuccess) e = cudaMemcpyAsync(sums, d_out, sizeof(sums), cudaMemcpyDeviceToHost, ctx->stream);
		if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
		if (e == cudaSuccess) e = cudaGetLastError();
		if (e != cudaSuccess) {
			status = ASTCENC_ERR_BAD_CONTEXT;
		}
	} while (false);
	cudaFree(d1);
	cudaFree(d2);
	cudaFree(d_part);
	if (status != ASTCENC_SUCCESS) {
		return status;
	}
	// the closing arithmetic of compute_error_metrics (:285-411)
	static const int componentmasks[5] = {0x00, 0x07, 0x0C, 0x07, 0x0F};
	int mask = componentmasks[input_components];
	double pixels = (double)(dim_x * dim_y * dim_z);
	double samples = 0.0, num = 0.0, alpha_num = 0.0, log_num = 0.0, mpsnr_num = 0.0;
	for (int c = 0; c < 4; c++) {
		if (mask & (1 << c)) {
			num += sums[MS_ERR + c];
			alpha_num += sums[MS_AERR + c];
			if (c < 3) {
				log_num += sums[MS_LOG + c];
				mpsnr_num += sums[MS_MPSNR + c];
			}
			samples += pixels;
		}
	}
	double stopcount = (double)(fstop_hi - fstop_lo + 1);
	double mpsnr_denom = pixels * 3.0 * stopcount * 255.0 * 255.0;
	double psnr = num == 0.0 ? 999.0 : 10.0 * log10(samples / num);
	double rgb_psnr = psnr;
	out->psnr = psnr;
	out->alpha_psnr = psnr;
	if (mask & 8) {
		out->alpha_psnr = alpha_num == 0.0 ? 999.0 : 10.0 * log10(samples / alpha_num);
		double rgb_num = sums[MS_ERR + 0] + sums[MS_ERR + 1] + sums[MS_ERR + 2];
		rgb_psnr = rgb_num == 0.0 ? 999.0 : 10.0 * log10(pixels * 3.0 / rgb_num);
	}
	out->rgb_psnr = rgb_psnr;
	out->rgb_peak = sums[MS_PEAK];
	if (compute_hdr_metrics) {
		out->peak_psnr = rgb_psnr + 20.0 * log10(sums[MS_PEAK]);
		out->mpsnr = mpsnr_num == 0.0 ? 999.0 : 10.0 * log10(mpsnr_denom / mpsnr_num);
		out->log_rmse = sqrt(log_num / pixels);
	}
	if (compute_normal_metrics) {
		out->mean_angular_error = sums[MS_ANG_MEAN];
		out->worst_angular_error = sums[MS_ANG_WORST];
	}
	for (int c = 0; c < 4; c++) {
		out->sum_squared_error[c] = sums[MS_ERR + c];
	}
	return ASTCENC_SUCCESS;
}

const char* astcenc_get_error_string(astcenc_error status) {
	switch (static_cast<int>(status)) {
	case ASTCENC_SUCCESS: return "ASTCENC_SUCCESS";
	case ASTCENC_ERR_OUT_OF_MEM: return "ASTCENC_ERR_OUT_OF_MEM";
	case ASTCENC_ERR_BAD_CPU_FLOAT: return "ASTCENC_ERR_BAD_CPU_FLOAT";
	case ASTCENC_ERR_BAD_PARAM: return "ASTCENC_ERR_BAD_PARAM";
	case ASTCENC_ERR_BAD_BLOCK_SIZE: return "ASTCENC_ERR_BAD_BLOCK_SIZE";
	case ASTCENC_ERR_BAD_PROFILE: return "ASTCENC_ERR_BAD_PROFILE";
	case ASTCENC_ERR_BAD_QUALITY: return "ASTCENC_ERR_BAD_QUALITY";
	case ASTCENC_ERR_BAD_FLAGS: return "ASTCENC_ERR_BAD_FLAGS";
	case ASTCENC_ERR_BAD_SWIZZLE: return "ASTCENC_ERR_BAD_SWIZZLE";
	case ASTCENC_ERR_BAD_CONTEXT: return "ASTCENC_ERR_BAD_CONTEXT";
	case ASTCENC_ERR_NOT_IMPLEMENTED: return "ASTCENC_ERR_NOT_IMPLEMENTED";
	case ASTCENC_ERR_BAD_DECODE_MODE: return "ASTCENC_ERR_BAD_DECODE_MODE";
	default: return nullptr;
	}
}

// ---- extensions ----
astcenc_error astcenc_b200_compress_device(astcenc_context* ctx, const void* d_pixels, astcenc_type data_type, unsigned int dim_x, unsigned int dim_y,
                                           const astcenc_swizzle* swizzle, unsigned int block_row0, unsigned int block_rows, uint8_t* d_out, void* cuda_stream) {
	if (ctx->config.flags & ASTCENC_FLG_DECOMPRESS_ONLY) {
		return ASTCENC_ERR_BAD_CONTEXT;
	}
	astcenc_error status = validate_compression_swizzle(*swizzle);
	if (status != ASTCENC_SUCCESS) {
		return status;
	}
	if (dim_x == 0 || dim_y == 0 || !d_pixels || !d_out) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	if (ctx->config.block_z > 1) {
		return ASTCENC_ERR_NOT_IMPLEMENTED;      // the device-resident entry takes one 2D image; volumes go through astcenc_compress_image
	}
	size_t blocks_y = block_count_axis(dim_y, ctx->config.block_y);
	if ((size_t)block_row0 + block_rows > blocks_y) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	if (block_rows == 0) {
		return ASTCENC_SUCCESS;
	}
	DeviceGuard guard(ctx->device);
	if (!guard.ok) {
		return ASTCENC_ERR_BAD_CONTEXT;
	}
	int swz[4] = {(int)swizzle->r, (int)swizzle->g, (int)swizzle->b, (int)swizzle->a};
	cudaStream_t s = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : ctx->stream;
	return launch_slab(ctx, d_pixels, (int)data_type, dim_x, dim_y, swz, block_row0, block_rows, d_out, s);
}

// Block lists (astc_dev_gather.cuh): gather -> one ordinary pass over the staging row -> scatter, chunk by chunk (a staging row is
// one block row, which the batching of launch_slab_locked cannot split: a chunk holds at most knobs.batch_blocks blocks). The
// whole call is one turn of the context's scratch (launch_mtx, scratch_done), like a launch_slab.
static astcenc_error launch_blocks(astcenc_context* ctx, const void* d_pixels, int data_type, unsigned int dim_x, unsigned int dim_y, unsigned int dim_z,
                                   const int swz[4], const std::vector<uint32_t>& list, unsigned int row_lo, unsigned int row_hi, uint8_t* d_payload, cudaStream_t stream) {
	const DevBsd& bsd = ctx->tables->bsd;
	const bool volume = bsd.dim_z > 1;
	const unsigned int radius = volume ? 0 : ctx->config.a_scale_radius;
	const size_t n = list.size();
	const size_t chunk = n < ctx->knobs.batch_blocks ? n : ctx->knobs.batch_blocks;
	const unsigned int words = data_type == ASTCENC_TYPE_U8 ? 1 : data_type == ASTCENC_TYPE_F16 ? 2 : 4;
	std::lock_guard<std::mutex> lk(ctx->launch_mtx);
	ctx->volume_dim_z = volume ? bsd.dim_z : 1;      // (the staging volume is one layer deep)
	ctx->pass_cancel = ctx->pass_done = nullptr;
	if (ctx->scratch_used) {
		CUDA_TRY(cudaStreamWaitEvent(stream, ctx->scratch_done, 0), return ASTCENC_ERR_BAD_CONTEXT);
	}
	astcenc_error st = ensure_buffer(ctx->d_list, ctx->d_list_bytes, n * sizeof(uint32_t));
	if (st == ASTCENC_SUCCESS) st = ensure_buffer(ctx->d_list_image, ctx->d_list_image_bytes, chunk * bsd.texel_count * words * 4);
	if (st == ASTCENC_SUCCESS) st = ensure_buffer(ctx->d_list_out, ctx->d_list_out_bytes, chunk * 16);
	if (st == ASTCENC_SUCCESS && radius != 0) {
		st = ensure_buffer(ctx->d_list_alpha, ctx->d_list_alpha_bytes, (size_t)dim_x * dim_y * sizeof(float));
		if (st == ASTCENC_SUCCESS && chunk * bsd.texel_count * sizeof(float) > ctx->d_alpha_bytes) {
			cudaFree(ctx->d_alpha);
			ctx->d_alpha = nullptr;
			ctx->d_alpha_bytes = 0;
			CUDA_TRY(cudaMalloc(&ctx->d_alpha, chunk * bsd.texel_count * sizeof(float)), st = ASTCENC_ERR_OUT_OF_MEM);
			if (st == ASTCENC_SUCCESS) ctx->d_alpha_bytes = chunk * bsd.texel_count * sizeof(float);
		}
	}
	if (st == ASTCENC_SUCCESS) {
		// (from pageable memory: staged by the driver before the call returns, so `list` may go when this function does)
		CUDA_TRY(cudaMemcpyAsync(ctx->d_list, list.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice, stream), st = ASTCENC_ERR_BAD_CONTEXT);
	}
	if (st == ASTCENC_SUCCESS && radius != 0) {
		// the averages of the listed blocks' rows, at their image positions; the staging pass must not filter its own image,
		// whose box filter would reach across the seams between unrelated blocks
		unsigned int y1 = (row_hi + 1) * bsd.dim_y;
		st = alpha_prepass(ctx, d_pixels, data_type, dim_x, dim_y, swz, row_lo * bsd.dim_y, y1 < dim_y ? y1 : dim_y,
		                   reinterpret_cast<float*>(ctx->d_list_alpha), stream);
	}
	GatherArgs g;
	g.src = d_pixels;
	g.dst = ctx->d_list_image;
	g.avg_src = radius != 0 ? reinterpret_cast<const float*>(ctx->d_list_alpha) : nullptr;
	g.avg_dst = radius != 0 ? ctx->d_alpha : nullptr;
	g.words = words;
	g.dim_x = dim_x;
	g.dim_y = dim_y;
	g.dim_z = dim_z;
	g.blocks_x = (unsigned int)block_count_axis(dim_x, bsd.dim_x);
	g.blocks_y = (unsigned int)block_count_axis(dim_y, bsd.dim_y);
	g.bx = bsd.dim_x;
	g.by = bsd.dim_y;
	g.bz = bsd.dim_z;
	const int aligned16 = (reinterpret_cast<uintptr_t>(d_payload) & 15) == 0;
	for (size_t first = 0; first < n && st == ASTCENC_SUCCESS; first += chunk) {
		const unsigned int m = (unsigned int)(n - first < chunk ? n - first : chunk);
		const uint32_t* d_idx = reinterpret_cast<const uint32_t*>(ctx->d_list) + first;
		g.indices = d_idx;
		g.n = m;
		const unsigned int warps = ASTC_GATHER_THREADS / 32;
		astc_gather_blocks_kernel<<<(m + warps - 1) / warps < (unsigned int)ctx->grid * 16 ? (m + warps - 1) / warps : (unsigned int)ctx->grid * 16, ASTC_GATHER_THREADS, 0, stream>>>(g);
		ctx->launches++;
		ctx->pass_alpha_staged = radius != 0;
		st = launch_slab_locked(ctx, ctx->d_list_image, data_type, m * bsd.dim_x, bsd.dim_y, swz, 0, 1, ctx->d_list_out, stream, nullptr);
		ctx->pass_alpha_staged = false;
		if (st == ASTCENC_SUCCESS) {
			astc_scatter_blocks_kernel<<<(m + ASTC_GATHER_THREADS - 1) / ASTC_GATHER_THREADS, ASTC_GATHER_THREADS, 0, stream>>>(ctx->d_list_out, d_idx, m, d_payload, aligned16);
			ctx->launches++;
			CUDA_TRY(cudaGetLastError(), st = ASTCENC_ERR_BAD_CONTEXT);
		}
	}
	CUDA_TRY(cudaEventRecord(ctx->scratch_done, stream), return ASTCENC_ERR_BAD_CONTEXT);
	ctx->scratch_used = true;
	return st;
}

astcenc_error astcenc_b200_compress_device_blocks(astcenc_context* ctx, const void* d_pixels, astcenc_type data_type, unsigned int dim_x, unsigned int dim_y,
                                                  unsigned int dim_z, const astcenc_swizzle* swizzle, const uint32_t* block_indices, unsigned int block_count,
                                                  uint8_t* d_payload, void* cuda_stream) {
	if (ctx->config.flags & ASTCENC_FLG_DECOMPRESS_ONLY) {
		return ASTCENC_ERR_BAD_CONTEXT;
	}
	if (!swizzle) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	astcenc_error status = validate_compression_swizzle(*swizzle);
	if (status != ASTCENC_SUCCESS) {
		return status;
	}
	if (dim_x == 0 || dim_y == 0 || dim_z == 0 || !d_pixels || !d_payload || (block_count != 0 && !block_indices)) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	if ((int)data_type < 0 || (int)data_type > 2) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	if (ctx->config.a_scale_radius != 0 && dim_z != 1 && ctx->config.block_z <= 1) {
		return ASTCENC_ERR_NOT_IMPLEMENTED;      // as astcenc_compress_image: the pre-pass is built for 2D images
	}
	size_t blocks_x = block_count_axis(dim_x, ctx->config.block_x);
	size_t blocks_y = block_count_axis(dim_y, ctx->config.block_y);
	size_t blocks_z = block_count_axis(dim_z, ctx->config.block_z);
	bool overflow = false;
	size_t total = mul_safe(mul_safe(blocks_x, blocks_y, overflow), blocks_z, overflow);
	if (overflow) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	// the list is checked whole before anything is enqueued, and copied: the caller may free it when the call returns
	std::vector<uint32_t> list(block_indices, block_indices + block_count);
	unsigned int row_lo = 0xFFFFFFFFu, row_hi = 0;
	for (uint32_t b : list) {
		if (b >= total) {
			return ASTCENC_ERR_BAD_PARAM;
		}
		unsigned int row = (unsigned int)(b / blocks_x);      // (2D images: the block row, for the alpha-scale pre-pass window)
		row_lo = row < row_lo ? row : row_lo;
		row_hi = row > row_hi ? row : row_hi;
	}
	if (block_count == 0) {
		return ASTCENC_SUCCESS;
	}
	DeviceGuard guard(ctx->device);
	if (!guard.ok) {
		return ASTCENC_ERR_BAD_CONTEXT;
	}
	int swz[4] = {(int)swizzle->r, (int)swizzle->g, (int)swizzle->b, (int)swizzle->a};
	cudaStream_t s = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : ctx->stream;
	return launch_blocks(ctx, d_pixels, (int)data_type, dim_x, dim_y, dim_z, swz, list, row_lo, row_hi, d_payload, s);
}

astcenc_error astcenc_b200_stage_timing(astcenc_context* ctx, int enable, float stage_ms[4], unsigned int stage_launches[4]) {
	if (!ctx) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	DeviceGuard guard(ctx->device);
	std::lock_guard<std::mutex> launch_lock(ctx->launch_mtx);
	if (stage_ms && stage_launches && ctx->stage_timing && ctx->stage_kinds.size() > 1) {
		// durations of the launches of the last astcenc_b200_compress_device() call, summed per kernel
		cudaEventSynchronize(ctx->stage_events[ctx->stage_kinds.size() - 1]);
		for (int k = 0; k < 4; k++) {
			stage_ms[k] = 0.0f;
			stage_launches[k] = 0;
		}
		for (size_t i = 1; i < ctx->stage_kinds.size(); i++) {
			float ms = 0.0f;
			cudaEventElapsedTime(&ms, ctx->stage_events[i - 1], ctx->stage_events[i]);
			int k = ctx->stage_kinds[i];
			if (ctx->knobs.stage_print) {
				fprintf(stderr, "launch %zu kind %d %.3f ms\n", i - 1, k, ms);
			}
			if (k >= 0 && k < 4) {
				stage_ms[k] += ms;
				stage_launches[k]++;
			}
		}
	}
	ctx->stage_timing = enable ? 1 : 0;
	return ASTCENC_SUCCESS;
}

}  // extern "C"

#include "astc_host_multi.inl"

extern "C" {

// dev aid (tools/diag_*.py): the per-block search records of the last pass, for post-mortem comparison of two passes
__attribute__((visibility("default"))) astcenc_error astcenc_b200_debug_records(astcenc_context* ctx, void** records, size_t* record_bytes, size_t* capacity_bytes) {
	if (!ctx || !records || !record_bytes || !capacity_bytes) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	*records = ctx->d_records;
	*record_bytes = ctx->tables->bsd.record_bytes;
	*capacity_bytes = ctx->d_records_bytes;
	return ASTCENC_SUCCESS;
}

unsigned long long astcenc_b200_launch_count(astcenc_context* ctx) {
	return ctx->launches;
}

astcenc_error astcenc_b200_last_timing(astcenc_context* ctx, float* kernel_ms, size_t* h2d_bytes, size_t* d2h_bytes) {
	if (kernel_ms) *kernel_ms = ctx->last_kernel_ms;
	if (h2d_bytes) *h2d_bytes = ctx->last_h2d;
	if (d2h_bytes) *d2h_bytes = ctx->last_d2h;
	return ASTCENC_SUCCESS;
}

}  // extern "C"
