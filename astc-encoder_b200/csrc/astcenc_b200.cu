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
#include "astc_dev_gather.cuh"
#include "astc_dev_metrics.cuh"
#include "astc_dev_select.cuh"
#include "astc_host_pack.h"
#include "astc_host_config.h"
#include "astc_host_slab.h"
#include "astc_host_launch.h"

// ---------------------------------------------------------------------------------------------
// The kernel: persistent warps, one block per warp at a time, dynamic ticket scheduling (the GPU analogue
// of the reference's ParallelManager::get_task_assignment ticket counter).
// ---------------------------------------------------------------------------------------------

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

// ---- block lists and image tables (astc_dev_gather.cuh): one warp per staging block, grid-stride ----
#define ASTC_GATHER_THREADS 256
__global__ void __launch_bounds__(ASTC_GATHER_THREADS)
astc_gather_blocks_kernel(const __grid_constant__ GatherArgs g) {
	const unsigned int warps = blockDim.x >> 5;
	for (unsigned int i = blockIdx.x * warps + (threadIdx.x >> 5); i < g.n; i += gridDim.x * warps) {
		gather_block(g, i, (int)(threadIdx.x & 31), 32);
	}
}

// staging block i -> its payload position (duplicate list entries write the same bytes); one thread per block
__global__ void __launch_bounds__(ASTC_GATHER_THREADS)
astc_scatter_blocks_kernel(const uint8_t* __restrict__ staged, const __grid_constant__ GatherArgs g) {
	unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= g.n) {
		return;
	}
	const uint4 v = __ldg(reinterpret_cast<const uint4*>(staged) + i);      // (read while the target is looked up)
	uint8_t* dst = scatter_target(g, i);
	if (dst == nullptr) {
		return;      // (an invalid list slot)
	}
	if ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
		*reinterpret_cast<uint4*>(dst) = v;
	} else {
		const uint8_t* b = reinterpret_cast<const uint8_t*>(&v);
		for (int k = 0; k < 16; k++) {
			dst[k] = b[k];
		}
	}
}

// ---- decompression (SURVEY.md section 8f) over image tables (astcenc_decompress_image, astcenc_b200_decompress_device_images):
// one warp per block, each CTA over a contiguous share of the call's blocks; img carries the call's data type and swizzle ----
#define ASTC_DECODE_THREADS 256
__global__ void __launch_bounds__(ASTC_DECODE_THREADS, 2)
astc_decompress_images_kernel(const __grid_constant__ DevBsd bsd, const __grid_constant__ DevConfig cfg, const __grid_constant__ DevImage img,
                              const GatherImage* __restrict__ images, unsigned int image_count, size_t total) {
	stage_launch_constants(bsd, cfg, img);
	const size_t per = (total + gridDim.x - 1) / gridDim.x;
	const size_t c0 = blockIdx.x * per;
	const size_t c1 = c0 + per < total ? c0 + per : total;
	decode_table_blocks(images, image_count, c0, c1, (int)(threadIdx.x >> 5), (int)(blockDim.x >> 5), (int)(threadIdx.x & 31),
	                    ASTC_SMEM_HDR + (threadIdx.x >> 5) * D_SLICE);
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

#define ASTC_COUNTER_WORDS (2 * ASTC_Q_KINDS * ASTC_MAX_WAVES + ASTC_MAX_BANDS)

struct DeviceTables {            // shared between a parent context and its children
	std::atomic<int> refcount{1};
	uint8_t* d_blob = nullptr;
	DevBsd bsd;                  // device pointers
	DevBsd bsd_1p;               // the same tables, compact one-plane arena plan (wave 0 of the pipeline)
	astc_host::BlockSizeTables* host_tables = nullptr;
};

// A device buffer grown on demand (never shrunk): `bytes` bytes at `ptr`.
struct DevBuffer {
	uint8_t* ptr = nullptr;
	size_t bytes = 0;
	template <typename T> T* as() const { return reinterpret_cast<T*>(ptr); }
};

static astcenc_error ensure_buffer(DevBuffer& b, size_t need) {
	if (b.bytes < need) {
		cudaFree(b.ptr);
		b.ptr = nullptr;
		b.bytes = 0;
		CUDA_TRY(cudaMalloc(&b.ptr, need), return ASTCENC_ERR_OUT_OF_MEM);
		b.bytes = need;
	}
	return ASTCENC_SUCCESS;
}

// "The first caller does the work, the others wait for its result" (the reference's ParallelManager): one per kind of call.
struct CallerGate {
	int state = 0;               // 0 idle, 1 running, 2 done
	astcenc_error result = ASTCENC_SUCCESS;
	void reset() {               // (under astcenc_context::mtx) ready for the next image, unless a call is running
		if (state != 1) {
			state = 0;
		}
	}
};

// Every member starts out null / idle, so that astcenc_context_free() can release a partially built context.
struct astcenc_context {
	astcenc_config config;
	unsigned int thread_count = 0;
	int device = -1;
	DeviceTables* tables = nullptr;
	DevConfig dcfg;
	cudaStream_t stream = nullptr;
	cudaEvent_t ev0 = nullptr, ev1 = nullptr;
	unsigned int* d_ticket = nullptr;
	Knobs knobs;
	KernelPlan plan;
	// wave pipeline buffers, grown on demand
	DevBuffer records;
	DevBuffer queues;            // ASTC_Q_KINDS lists of one entry per block (uint32_t)
	uint32_t* d_counters = nullptr;   // count[ASTC_Q_KINDS][MAX_WAVES] head[ASTC_Q_KINDS][MAX_WAVES]
	DevBuffer alpha;             // alpha-scale pre-pass: one average per texel (float)
	// optional per-stage timing (astcenc_b200_stage_timing): an event after every launch of the next call
	int stage_timing = 0;
	std::vector<cudaEvent_t> stage_events;
	std::vector<int> stage_kinds;
	// staging buffers for the host-pointer API, grown on demand; image2 is the second image buffer of the batch API
	// (double-buffered uploads)
	DevBuffer image, image2, out;
	// staging calls (astc_dev_gather.cuh), grown on demand: the table with its lists, the staging image and payload of one chunk,
	// the pre-pass averages of the source images
	DevBuffer list, list_image, list_out, list_alpha;
	// metrics calls: the partial sums of every virtual CTA and the sums of every pair, grown on demand
	DevBuffer metric_partials;
	// selection calls: the entries, their histograms and the tile counts
	DevBuffer select;
	// The per-context scratch (records, queues, counters, alpha averages, table and staging buffers) serves ONE pass at a time
	// (scratch_turn): launch_mtx serialises the host side, scratch_done orders a pass on one stream behind the previous pass on
	// another.
	std::mutex launch_mtx;
	cudaEvent_t scratch_done = nullptr;
	bool scratch_used = false;
	int sm_count = 0;            // the device's SMs (grids of the decode and pipeline launches)
	// host-pointer path: uploads run on copy_stream, band by band, under the set-up of the previous band
	cudaStream_t copy_stream = nullptr;
	cudaEvent_t band_ready[ASTC_MAX_BANDS] = {};
	// sub-slab pipelines of one pass (launch_pipes): one stream each, joined to the caller's stream by events
	cudaStream_t pipe_stream[ASTC_MAX_PIPES] = {};
	cudaEvent_t pipe_done[ASTC_MAX_PIPES] = {};
	cudaEvent_t pipe_start = nullptr;
	// multi-GPU (astc_host_multi.inl): one process per GPU, NCCL for the payload gather
	void* nccl_comm = nullptr;
	int rank = 0, world = 1;
	cudaEvent_t ev_g0 = nullptr, ev_g1 = nullptr;
	float last_gather_ms = 0.0f, last_compress_ms = 0.0f;
	// caller protocol
	std::mutex mtx;
	std::condition_variable cv;
	CallerGate compress_gate, decompress_gate;
	std::atomic<bool> cancel{false};
	// Progress and cancellation of astcenc_compress_image (astc_dev_lockstep.cuh, pass_cancelled): d_words = {cancel flag, done
	// counter}; h_words (pinned) = {0, 1, counter read-back}: the flag is written by 4-byte DMAs from h_words[0] / [1] and the
	// counter read by one into h_words[2], all on ctl_stream, which never waits for the pass. flag_mtx makes "set ctx->cancel,
	// enqueue the matching flag write" one step, so that the device flag always ends on the value ctx->cancel holds.
	uint32_t* d_words = nullptr;
	uint32_t* h_words = nullptr;
	cudaStream_t ctl_stream = nullptr;
	cudaEvent_t ctl_ready = nullptr;          // after the last flag clear: a pass starts behind it
	std::mutex flag_mtx;
	bool flag_raised = false;                 // a raise was enqueued since the last clear (under flag_mtx)
	// stats
	unsigned long long launches = 0;
	float last_kernel_ms = 0.0f;
	size_t last_h2d = 0, last_d2h = 0;
};

// Runs `work` for the first caller through `gate`; every other caller waits for that call and returns its result.
template <typename F>
static astcenc_error run_once(astcenc_context* ctx, CallerGate& gate, F work) {
	std::unique_lock<std::mutex> lk(ctx->mtx);
	if (gate.state == 0) {
		gate.state = 1;
		lk.unlock();
		astcenc_error r = work();
		lk.lock();
		gate.result = r;
		gate.state = 2;
		ctx->cv.notify_all();
		return r;
	}
	ctx->cv.wait(lk, [&gate] { return gate.state == 2; });
	return gate.result;
}

// Orders `stream` behind the last turn of the scratch (a no-op when that ran on the same stream). Under launch_mtx.
static astcenc_error wait_for_scratch(astcenc_context* ctx, cudaStream_t stream) {
	if (ctx->scratch_used) {
		CUDA_TRY(cudaStreamWaitEvent(stream, ctx->scratch_done, 0), return ASTCENC_ERR_BAD_CONTEXT);
	}
	return ASTCENC_SUCCESS;
}

// One turn of the context's scratch: `work` enqueues a pass on `stream`. Calls may come from several host threads and on
// different streams: launch_mtx serialises the enqueueing, the pass starts behind the event that closed the previous turn, and
// every exit records that event behind this one. Returns the first error.
template <typename F>
static astcenc_error scratch_turn(astcenc_context* ctx, cudaStream_t stream, F work) {
	std::lock_guard<std::mutex> lk(ctx->launch_mtx);
	astcenc_error st = wait_for_scratch(ctx, stream);
	if (st == ASTCENC_SUCCESS) {
		st = work();
	}
	CUDA_TRY(cudaEventRecord(ctx->scratch_done, stream), return st != ASTCENC_SUCCESS ? st : ASTCENC_ERR_BAD_CONTEXT);
	ctx->scratch_used = true;
	return st;
}

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
	ctx->config = *configp;
	ctx->thread_count = thread_count;
	ctx->knobs = read_knobs();      // environment knobs: read here, once
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
	CUDA_TRY(cudaDeviceGetAttribute(&ctx->sm_count, cudaDevAttrMultiProcessorCount, device), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));

	if (!(cfg.flags & ASTCENC_FLG_DECOMPRESS_ONLY)) {
		cudaDeviceProp prop;
		CUDA_TRY(cudaGetDeviceProperties(&prop, device), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
		status = plan_kernels(ctx->tables->bsd, ctx->tables->bsd_1p, cfg, prop.sharedMemPerBlockOptin, ctx->sm_count, ctx->knobs, ctx->plan);
		if (status != ASTCENC_SUCCESS) {
			ALLOC_FAIL(status);
		}
		const int smem_limit = (int)prop.sharedMemPerBlockOptin;
		CUDA_TRY(cudaFuncSetAttribute(astc_compress_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_limit), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
		CUDA_TRY(cudaFuncSetAttribute(astc_wave_setup_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_limit), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
		CUDA_TRY(cudaFuncSetAttribute(astc_wave_setup_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_limit), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
		CUDA_TRY(cudaFuncSetAttribute(astc_wave_refine_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_limit), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
		CUDA_TRY(cudaFuncSetAttribute(astc_wave_refine_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_limit), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
		CUDA_TRY(cudaFuncSetAttribute(astc_wave_prepare_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_limit), ALLOC_FAIL(ASTCENC_ERR_BAD_CONTEXT));
		// count[kinds][waves], head[kinds][waves], then one image ticket per upload band
		CUDA_TRY(cudaMalloc(&ctx->d_counters, sizeof(uint32_t) * ASTC_COUNTER_WORDS * ASTC_MAX_PIPES), ALLOC_FAIL(ASTCENC_ERR_OUT_OF_MEM));
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
	cudaFree(ctx->d_counters);
	for (DevBuffer* b : {&ctx->records, &ctx->queues, &ctx->alpha, &ctx->image, &ctx->image2, &ctx->out, &ctx->list, &ctx->list_image, &ctx->list_out,
	                     &ctx->list_alpha, &ctx->metric_partials, &ctx->select}) {
		cudaFree(b->ptr);
	}
	for (cudaEvent_t e : ctx->stage_events) {
		cudaEventDestroy(e);
	}
	if (ctx->ev0) cudaEventDestroy(ctx->ev0);
	if (ctx->ev1) cudaEventDestroy(ctx->ev1);
	if (ctx->ev_g0) cudaEventDestroy(ctx->ev_g0);
	if (ctx->ev_g1) cudaEventDestroy(ctx->ev_g1);
	if (ctx->scratch_done) cudaEventDestroy(ctx->scratch_done);
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

// Every component a selector from ASTCENC_SWZ_R to `highest`: ASTCENC_SWZ_1 for compression, ASTCENC_SWZ_Z for decompression
// (astcenc_entry.cpp:279-300).
static astcenc_error check_swizzle(const astcenc_swizzle& s, astcenc_swz highest) {
	const int v[4] = {(int)s.r, (int)s.g, (int)s.b, (int)s.a};
	for (int i = 0; i < 4; i++) {
		if (v[i] < ASTCENC_SWZ_R || v[i] > (int)highest) {
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

static size_t texel_bytes(int data_type) {
	return data_type == ASTCENC_TYPE_U8 ? 4 : data_type == ASTCENC_TYPE_F16 ? 8 : 16;
}

static size_t block_count_axis(size_t dim, size_t blk) {
	size_t n = dim / blk;
	if (dim != blk * n) {
		n++;
	}
	return n;
}

// Geometry of one image in combined block rows (astc_host_slab.h): `layers` layers (3D block sizes) or slices of blocks_y rows.
// A 3D block size takes the volume in one pass; a 2D one takes an array one slice per pass.
struct SlabGeometry {
	size_t blocks_x, blocks_y, layers;
	size_t blocks;               // blocks_x * blocks_y * layers
	bool overflow;               // the block count does not fit a size_t
	size_t texel_bytes;          // bytes per texel of the image's data type
	size_t slice_bytes;          // bytes of one image slice
	size_t row_out;              // payload bytes of one combined row
	unsigned int dim_z;
	bool volume;
	unsigned int rows() const { return (unsigned int)(blocks_y * layers); }
	size_t out_bytes() const { return row_out * blocks_y * layers; }
	unsigned int passes() const { return volume ? 1 : dim_z; }
	unsigned int pass_slices() const { return volume ? dim_z : 1; }      // image slices one pass reads
	unsigned int pass_rows() const { return volume ? rows() : (unsigned int)blocks_y; }
	size_t pass_out_bytes() const { return row_out * pass_rows(); }
	bool payload_overflow() const { return overflow || blocks > SIZE_MAX / 16; }      // block count or payload bytes
};

static SlabGeometry slab_geometry(const astcenc_context* ctx, unsigned int dim_x, unsigned int dim_y, unsigned int dim_z, int data_type) {
	const DevBsd& bsd = ctx->tables->bsd;
	SlabGeometry g;
	g.volume = bsd.dim_z > 1;
	g.dim_z = dim_z;
	g.blocks_x = block_count_axis(dim_x, bsd.dim_x);
	g.blocks_y = block_count_axis(dim_y, bsd.dim_y);
	g.layers = g.volume ? block_count_axis(dim_z, bsd.dim_z) : dim_z;
	g.overflow = false;
	g.blocks = mul_safe(mul_safe(g.blocks_x, g.blocks_y, g.overflow), g.layers, g.overflow);
	g.row_out = g.blocks_x * 16;
	g.texel_bytes = texel_bytes(data_type);
	g.slice_bytes = (size_t)dim_x * dim_y * g.texel_bytes;
	return g;
}

// ---- argument checks: every entry point calls the ones it makes, in its own order (astcenc_compress_image in the reference's) ----
static astcenc_error check_compress_context(const astcenc_context* ctx) {
	return (ctx->config.flags & ASTCENC_FLG_DECOMPRESS_ONLY) ? ASTCENC_ERR_BAD_CONTEXT : ASTCENC_SUCCESS;
}

// texel count non-zero and free of overflow
static astcenc_error check_texel_count(unsigned int dim_x, unsigned int dim_y, unsigned int dim_z) {
	bool overflow = false;
	size_t texels = mul_safe(mul_safe(dim_x, dim_y, overflow), dim_z, overflow);
	return overflow || texels == 0 ? ASTCENC_ERR_BAD_PARAM : ASTCENC_SUCCESS;
}

static astcenc_error check_data_type(astcenc_type data_type) {
	return (int)data_type < 0 || (int)data_type > 2 ? ASTCENC_ERR_BAD_PARAM : ASTCENC_SUCCESS;
}

// the alpha-scale pre-pass is built for 2D images; arrays would average across slices (compute_variance.cpp have_z)
static astcenc_error check_alpha_scale(const astcenc_context* ctx, unsigned int dim_z) {
	return ctx->config.a_scale_radius != 0 && dim_z != 1 && ctx->config.block_z <= 1 ? ASTCENC_ERR_NOT_IMPLEMENTED : ASTCENC_SUCCESS;
}

// The scratch of a pass, grown on demand: records and queues for `blocks` blocks of the wave pipeline, `alpha` averages of the
// alpha-scale pre-pass.
static astcenc_error ensure_scratch(astcenc_context* ctx, size_t blocks, size_t alpha) {
	astcenc_error st = ensure_buffer(ctx->queues, sizeof(uint32_t) * ASTC_Q_KINDS * blocks);
	if (st == ASTCENC_SUCCESS) st = ensure_buffer(ctx->records, blocks * (size_t)ctx->tables->bsd.record_bytes);
	if (st == ASTCENC_SUCCESS) st = ensure_buffer(ctx->alpha, alpha * sizeof(float));
	return st;
}

// The image a pass reads: dim_x x dim_y texels at `pixels`, `dim_z` slices of them for a volume pass (3D block sizes; 1
// otherwise), no alpha averages and no progress words. The pass fills in the block rows it covers and where their payload goes.
static DevImage pass_image(const astcenc_context* ctx, const void* pixels, int data_type, unsigned int dim_x, unsigned int dim_y, unsigned int dim_z,
                           const astcenc_swizzle& swizzle) {
	const DevBsd& bsd = ctx->tables->bsd;
	DevImage img{};
	img.data = pixels;
	img.data_type = data_type;
	img.dim_x = dim_x;
	img.dim_y = dim_y;
	img.dim_z = dim_z;
	img.blocks_x = (dim_x + bsd.dim_x - 1) / bsd.dim_x;
	img.blocks_y = (dim_y + bsd.dim_y - 1) / bsd.dim_y;
	img.swz[0] = (int)swizzle.r;
	img.swz[1] = (int)swizzle.g;
	img.swz[2] = (int)swizzle.b;
	img.swz[3] = (int)swizzle.a;
	img.cancel = nullptr;
	img.done = nullptr;
	return img;
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

// Image rows [y0, y1) go up on the copy stream; band event k marks their arrival, and `stream` waits for it.
static astcenc_error upload_rows(astcenc_context* ctx, const UploadPlan& up, size_t y0, size_t y1, int k, cudaStream_t stream) {
	if (y1 > y0) {
		CUDA_TRY(cudaMemcpyAsync(up.device + y0 * up.row_bytes, up.host + y0 * up.row_bytes, (y1 - y0) * up.row_bytes, cudaMemcpyHostToDevice, ctx->copy_stream),
		         return ASTCENC_ERR_BAD_CONTEXT);
	}
	CUDA_TRY(cudaEventRecord(ctx->band_ready[k], ctx->copy_stream), return ASTCENC_ERR_BAD_CONTEXT);
	CUDA_TRY(cudaStreamWaitEvent(stream, ctx->band_ready[k], 0), return ASTCENC_ERR_BAD_CONTEXT);
	return ASTCENC_SUCCESS;
}

// Slices [z0, z1) of a host image to their places in a device buffer of slice_bytes per slice, one copy each on `stream`.
static astcenc_error upload_slices(uint8_t* device, void* const* slices, unsigned int z0, unsigned int z1, size_t slice_bytes, cudaStream_t stream) {
	for (unsigned int z = z0; z < z1; z++) {
		CUDA_TRY(cudaMemcpyAsync(device + (size_t)z * slice_bytes, slices[z], slice_bytes, cudaMemcpyHostToDevice, stream), return ASTCENC_ERR_BAD_CONTEXT);
	}
	return ASTCENC_SUCCESS;
}

// Image rows [y0, y1) that a pass over block rows [block_row0, block_row0 + block_rows) of a 2D image reads: the slab's own
// rows, or with alpha-scale the rows its pre-pass window reads (a superset of them).
static void slab_image_rows(const astcenc_context* ctx, unsigned int dim_y, unsigned int block_row0, unsigned int block_rows, size_t& y0, size_t& y1) {
	image_rows(block_row0, block_row0 + block_rows, ctx->tables->bsd.dim_y, dim_y, y0, y1);
	const unsigned int radius = ctx->tables->bsd.dim_z > 1 ? 0 : ctx->config.a_scale_radius;
	if (radius != 0 && y1 > y0) {
		AlphaWindow w = alpha_window(dim_y, radius, (unsigned int)y0, (unsigned int)y1);
		y0 = w.read_row0;
		y1 = w.read_row1;
	}
}

// Per-stage timing (astcenc_b200_stage_timing): an event on `stream` behind the launches of one stage of a batch (kind 0 set-up,
// 1 refine, 2 prepare, 3 emit; -1 opens the batch).
static void stage_mark(astcenc_context* ctx, int kind, cudaStream_t stream) {
	if (!ctx->stage_timing) {
		return;
	}
	const size_t i = ctx->stage_kinds.size();
	if (i == ctx->stage_events.size()) {
		cudaEvent_t e;
		if (cudaEventCreate(&e) != cudaSuccess) {
			return;
		}
		ctx->stage_events.push_back(e);
	}
	ctx->stage_kinds.push_back(kind);
	cudaEventRecord(ctx->stage_events[i], stream);
}

// The WaveArgs of one pipeline over `blocks` blocks (blocks_x per row): its counter block, and its first block `first` in the
// context's records and queues.
static WaveArgs wave_args(const astcenc_context* ctx, uint32_t* counters, size_t first, unsigned int blocks, unsigned int blocks_x) {
	const DevBsd& bsd = ctx->tables->bsd;
	WaveArgs a;
	a.records = ctx->records.ptr + first * (size_t)bsd.record_bytes;
	a.queues = ctx->queues.as<uint32_t>() + first;
	a.queue_stride = ctx->queues.bytes / (sizeof(uint32_t) * ASTC_Q_KINDS);
	a.count = counters;
	a.head = counters + ASTC_Q_KINDS * ASTC_MAX_WAVES;
	a.total = blocks;
	a.blocks_x = blocks_x;
	a.ticket = counters + 2 * ASTC_Q_KINDS * ASTC_MAX_WAVES;
	a.first_block = 0;
	a.band_blocks = blocks;
	a.cls_lo = 0;
	a.cls_hi = ASTC_Q_CLASSES;
	a.wave = 0;
	a.sync_mask = ctx->knobs.sync_mask;
	a.stage_bytes_setup = ctx->plan.setup_stage_bytes;
	a.refine_state_off = (uint32_t)(ASTC_SMEM_HDR + ctx->plan.refine_stage_bytes + (size_t)bsd.arena_bytes_small * ctx->plan.warps_small);
	a.stage_bytes = ctx->plan.refine_stage_bytes;
	return a;
}

// The set-up launch(es) of wave a.wave of one pipeline. Wave 0 of a banded upload (`up`) runs one launch per band, each behind
// the copy of its band's rows and taking the band's blocks from its own ticket. On the compact one-plane plan, class 0 of the
// later waves (the two-plane trials) runs on the general plan; wave 0 and the n-partition classes have one weight plane and run
// on the compact plan with more warps per SM.
static astcenc_error enqueue_setup(astcenc_context* ctx, const DevImage& img, WaveArgs a, cudaStream_t stream, const UploadPlan* up) {
	const SetupKernel kernel = setup_kernel(ctx->dcfg, a.wave);
	const KernelPlan& p = ctx->plan;
	const bool compact = p.warps_setup_1p != 0;
	auto launch = [&](bool on_compact) {
		if (on_compact) {
			kernel<<<p.grid, p.warps_setup_1p * 32, p.smem_setup_1p, stream>>>(ctx->tables->bsd_1p, ctx->dcfg, img, a);
		} else {
			kernel<<<p.grid, p.warps_setup * 32, p.smem_setup, stream>>>(ctx->tables->bsd, ctx->dcfg, img, a);
		}
		ctx->launches++;
	};
	if (a.wave == 0 && up != nullptr) {
		uint32_t* const ticket = a.ticket;
		for (int k = 0; k < up->bands; k++) {
			unsigned int r0, r1;
			if (!band_of(img.block_rows, up->bands, k, r0, r1)) {
				continue;
			}
			size_t y0, y1;
			image_rows(img.block_row0 + r0, img.block_row0 + r1, ctx->tables->bsd.dim_y, img.dim_y, y0, y1);
			astcenc_error st = upload_rows(ctx, *up, y0, y1, k, stream);
			if (st != ASTCENC_SUCCESS) {
				return st;
			}
			a.ticket = ticket + k;
			a.first_block = r0 * img.blocks_x;
			a.band_blocks = (r1 - r0) * img.blocks_x;
			launch(compact);
		}
	} else {
		if (compact && a.wave != 0) {
			a.cls_lo = 0;
			a.cls_hi = 1;
			launch(false);
			a.cls_lo = 1;
			a.cls_hi = ASTC_Q_CLASSES;
		}
		launch(compact);
	}
	stage_mark(ctx, 0, stream);
	return ASTCENC_SUCCESS;
}

// Refinement and preparation of wave a.wave of one pipeline.
static void enqueue_refine_prepare(astcenc_context* ctx, const DevImage& img, const WaveArgs& a, cudaStream_t stream) {
	const DevBsd& bsd = ctx->tables->bsd;
	const KernelPlan& p = ctx->plan;
	if (refine_l1_step(ctx->dcfg)) {
		astc_wave_refine_kernel<true><<<p.grid * p.refine_ctas, p.warps_small * 32, p.smem_refine, stream>>>(bsd, ctx->dcfg, img, a);
	} else {
		astc_wave_refine_kernel<false><<<p.grid * p.refine_ctas, p.warps_small * 32, p.smem_refine, stream>>>(bsd, ctx->dcfg, img, a);
	}
	ctx->launches++;
	stage_mark(ctx, 1, stream);
	// (statistics / partition search gain nothing from phase alignment: two half-size CTAs per SM wait less)
	const int wp = p.warps_small >= 2 ? p.warps_small / 2 : 1;
	astc_wave_prepare_kernel<<<p.grid * 2, wp * 32, ASTC_SMEM_HDR + (size_t)bsd.arena_bytes_small * wp, stream>>>(bsd, ctx->dcfg, img, a);
	ctx->launches++;
	stage_mark(ctx, 2, stream);
}

// The emit launch of one pipeline: the chosen encoding of every block into the payload.
static void enqueue_emit(astcenc_context* ctx, const DevImage& img, WaveArgs a, cudaStream_t stream) {
	a.wave = 0;
	astc_wave_emit_kernel<<<ctx->plan.grid * 4, ASTC_EMIT_THREADS, ASTC_SMEM_HDR + (ASTC_EMIT_THREADS / 32) * 32 * EMIT_SLICE, stream>>>(ctx->tables->bsd, ctx->dcfg, img, a);
	ctx->launches++;
	stage_mark(ctx, 3, stream);
}

// One batch of a slab on the wave pipeline: the waves of the search, then emit, on `stream`.
static astcenc_error launch_batch(astcenc_context* ctx, const DevImage& img, cudaStream_t stream, const UploadPlan* up) {
	CUDA_TRY(cudaMemsetAsync(ctx->d_counters, 0, sizeof(uint32_t) * ASTC_COUNTER_WORDS, stream), return ASTCENC_ERR_BAD_CONTEXT);
	WaveArgs a = wave_args(ctx, ctx->d_counters, 0, img.blocks_x * img.block_rows, img.blocks_x);
	if (ctx->stage_timing) {
		ctx->stage_kinds.clear();
	}
	stage_mark(ctx, -1, stream);
	for (int wave = 0; wave < ctx->plan.max_waves; wave++) {
		a.wave = wave;
		a.sync_mask = wave == 0 ? ctx->knobs.sync_mask : ctx->knobs.sync_mask_tail;
		astcenc_error st = enqueue_setup(ctx, img, a, stream, up);
		if (st != ASTCENC_SUCCESS) {
			return st;
		}
		enqueue_refine_prepare(ctx, img, a, stream);
	}
	enqueue_emit(ctx, img, a, stream);
	CUDA_TRY(cudaGetLastError(), return ASTCENC_ERR_BAD_CONTEXT);
	return ASTCENC_SUCCESS;
}

// One pass as P independent sub-slab pipelines. The search is a chain of waves (set-up -> refine -> prepare, ~10 times) and
// every kernel of the chain ends with a drain: the last blocks of a wave keep a few SMs busy while the others idle, and the
// late waves never fill the GPU's SMs at all. Blocks are independent, so the slab is cut into P ranges of block rows, each with
// its own records / queues / counters, and the P chains are enqueued breadth-first on P streams: while the kernel of one
// chain drains, the CTAs of the next chain's kernel take over the SMs that became free (every kernel is one CTA per SM,
// so the hardware block scheduler does the interleaving). Same kernels, same results; wave 0 of chain p waits only for the
// upload of its own rows (the band scheme of the host-pointer path with bands = pipelines).
static astcenc_error launch_pipes(astcenc_context* ctx, int pipes, const DevImage& slab, cudaStream_t stream, const UploadPlan* up) {
	DevImage img[ASTC_MAX_PIPES];
	WaveArgs a[ASTC_MAX_PIPES];
	CUDA_TRY(cudaEventRecord(ctx->pipe_start, stream), return ASTCENC_ERR_BAD_CONTEXT);
	for (int p = 0; p < pipes; p++) {
		unsigned int r0, r1;
		slab_of(slab.block_rows, pipes, p, r0, r1);
		cudaStream_t ps = ctx->pipe_stream[p];
		CUDA_TRY(cudaStreamWaitEvent(ps, ctx->pipe_start, 0), return ASTCENC_ERR_BAD_CONTEXT);
		img[p] = slab;
		img[p].block_row0 = slab.block_row0 + r0;
		img[p].block_rows = r1 - r0;
		img[p].out = slab.out + (size_t)r0 * slab.blocks_x * 16;
		uint32_t* counters = ctx->d_counters + (size_t)p * ASTC_COUNTER_WORDS;
		CUDA_TRY(cudaMemsetAsync(counters, 0, sizeof(uint32_t) * ASTC_COUNTER_WORDS, ps), return ASTCENC_ERR_BAD_CONTEXT);
		a[p] = wave_args(ctx, counters, (size_t)r0 * slab.blocks_x, (r1 - r0) * slab.blocks_x, slab.blocks_x);
		if (up != nullptr) {
			// this pipeline's rows go up on the copy stream; only its wave 0 waits for them
			size_t y0, y1;
			image_rows(slab.block_row0 + r0, slab.block_row0 + r1, ctx->tables->bsd.dim_y, slab.dim_y, y0, y1);
			astcenc_error st = upload_rows(ctx, *up, y0, y1, p, ps);
			if (st != ASTCENC_SUCCESS) {
				return st;
			}
		}
	}
	for (int wave = 0; wave < ctx->plan.max_waves; wave++) {
		for (int p = 0; p < pipes; p++) {
			if (a[p].total == 0) {
				continue;
			}
			a[p].wave = wave;
			a[p].sync_mask = wave == 0 ? ctx->knobs.sync_mask : ctx->knobs.sync_mask_tail;
			astcenc_error st = enqueue_setup(ctx, img[p], a[p], ctx->pipe_stream[p], nullptr);
			if (st != ASTCENC_SUCCESS) {
				return st;
			}
			enqueue_refine_prepare(ctx, img[p], a[p], ctx->pipe_stream[p]);
		}
	}
	for (int p = 0; p < pipes; p++) {
		cudaStream_t ps = ctx->pipe_stream[p];
		if (a[p].total != 0) {
			enqueue_emit(ctx, img[p], a[p], ps);
		}
		CUDA_TRY(cudaEventRecord(ctx->pipe_done[p], ps), return ASTCENC_ERR_BAD_CONTEXT);
		CUDA_TRY(cudaStreamWaitEvent(stream, ctx->pipe_done[p], 0), return ASTCENC_ERR_BAD_CONTEXT);
	}
	CUDA_TRY(cudaGetLastError(), return ASTCENC_ERR_BAD_CONTEXT);
	return ASTCENC_SUCCESS;
}

// One batch of a slab on a single-kernel driver (ASTCENC_B200_DRIVER=lockstep|warp).
static astcenc_error launch_driver(astcenc_context* ctx, const DevImage& img, cudaStream_t stream) {
	CUDA_TRY(cudaMemsetAsync(ctx->d_ticket, 0, sizeof(unsigned int), stream), return ASTCENC_ERR_BAD_CONTEXT);
	const KernelPlan& p = ctx->plan;
	int grid = p.grid;
	size_t total = (size_t)img.blocks_x * img.block_rows;
	size_t needed = (total + p.warps_per_cta - 1) / p.warps_per_cta;
	if ((size_t)grid > needed) {
		grid = (int)(needed ? needed : 1);
	}
	astc_compress_kernel<<<grid, p.warps_per_cta * 32, p.smem_bytes, stream>>>(ctx->tables->bsd, ctx->dcfg, img, ctx->d_ticket, ctx->knobs.coherence_probe, p.lockstep);
	CUDA_TRY(cudaGetLastError(), return ASTCENC_ERR_BAD_CONTEXT);
	ctx->launches++;
	return ASTCENC_SUCCESS;
}

// The alpha-scale pre-pass over the image rows of block rows [r0, r1) of a 2D image (alpha_window: the 32 x 32 tiles that cover
// them, reading up to a_scale_radius rows beyond); the averages land at their image positions in `averages` (dim_x * dim_y
// floats), and `threshold` receives the value the set-up stage compares them with.
static astcenc_error alpha_prepass(astcenc_context* ctx, const DevImage& src, unsigned int r0, unsigned int r1, float* averages, cudaStream_t stream,
                                   float& threshold) {
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
	size_t y0, y1;
	image_rows(r0, r1, bsd.dim_y, src.dim_y, y0, y1);
	unsigned int tiles_x = (src.dim_x + ALPHA_TILE - 1) / ALPHA_TILE;
	AlphaWindow win = alpha_window(src.dim_y, radius, (unsigned int)y0, (unsigned int)y1);
	astc_alpha_average_kernel<<<tiles_x * win.tile_rows, ASTC_ALPHA_THREADS, smem, stream>>>(src, radius, tiles_x, win.tile_row0, averages);
	CUDA_TRY(cudaGetLastError(), return ASTCENC_ERR_BAD_CONTEXT);
	ctx->launches++;
	// astcenc_entry.cpp:983-988
	size_t x_footprint = bsd.dim_x + 2 * ((size_t)radius - 1);
	size_t y_footprint = bsd.dim_y + 2 * ((size_t)radius - 1);
	float footprint = static_cast<float>(x_footprint * y_footprint);
	threshold = 0.9f / (255.0f * footprint);
	return ASTCENC_SUCCESS;
}

// A slab of block rows is processed in batches of at most ~1 M blocks: the per-block search records (a few KB each)
// are the only buffer that grows with the image, and the batches reuse them in stream order. A 2D pass given no alpha
// averages with a_scale_radius set runs its own pre-pass over the slab's window first.
static astcenc_error launch_slab_locked(astcenc_context* ctx, const DevImage& src, unsigned int block_row0, unsigned int block_rows, uint8_t* d_out,
                                        cudaStream_t stream, const UploadPlan* up) {
	const DevBsd& bsd = ctx->tables->bsd;
	DevImage img = src;
	img.block_row0 = block_row0;
	img.block_rows = block_rows;
	img.out = d_out;
	const size_t blocks_x = img.blocks_x;
	size_t rows_per_batch = ctx->knobs.batch_blocks / (blocks_x ? blocks_x : 1);
	if (rows_per_batch < 1) rows_per_batch = 1;
	const unsigned int radius = bsd.dim_z > 1 ? 0 : ctx->config.a_scale_radius;      // (the averages only steer 2D block sizes, astcenc_entry.cpp:975)
	// big single-batch slabs run as independent sub-slab pipelines (launch_pipes); per-launch timing wants one stream
	bool single_batch = (size_t)block_rows <= rows_per_batch;
	int pipes = ctx->knobs.pipes;
	bool use_pipes = pipes > 1 && ctx->plan.driver == 0 && !ctx->stage_timing && single_batch && block_rows >= (unsigned int)pipes * 4 &&
	                 blocks_x * block_rows >= (size_t)pipes * 8192;
	// banded uploads need the whole slab in one batch on the wave pipeline, and no pre-pass that reads the window first
	bool banded = up != nullptr && radius == 0 && ctx->plan.driver == 0 && single_batch && (use_pipes || (up->bands > 1 && block_rows >= (unsigned int)up->bands * 4));
	if (up != nullptr) {
		// the upload streams on the copy stream; it must not overtake a pass that still reads the image buffer
		astcenc_error st = wait_for_scratch(ctx, ctx->copy_stream);
		if (st != ASTCENC_SUCCESS) {
			return st;
		}
	}
	if (up != nullptr && !banded) {
		size_t y0, y1;
		slab_image_rows(ctx, img.dim_y, block_row0, block_rows, y0, y1);
		astcenc_error st = upload_rows(ctx, *up, y0, y1, 0, stream);
		if (st != ASTCENC_SUCCESS) {
			return st;
		}
		up = nullptr;
	}
	if (radius != 0 && img.alpha_avg == nullptr) {
		// the box filter reaches across slab borders: the window reads up to `radius` rows beyond the tiles that cover the
		// slab's rows (alpha_window); the averages stay at their image positions
		astcenc_error st = ensure_scratch(ctx, 0, (size_t)img.dim_x * img.dim_y);
		if (st == ASTCENC_SUCCESS) {
			st = alpha_prepass(ctx, img, block_row0, block_row0 + block_rows, ctx->alpha.as<float>(), stream, img.alpha_threshold);
		}
		if (st != ASTCENC_SUCCESS) {
			return st;
		}
		img.alpha_avg = ctx->alpha.as<float>();
	}
	if (ctx->plan.driver == 0) {
		astcenc_error st = ensure_scratch(ctx, blocks_x * (single_batch ? block_rows : rows_per_batch), 0);
		if (st != ASTCENC_SUCCESS) {
			return st;
		}
	}
	if (use_pipes) {
		return launch_pipes(ctx, pipes, img, stream, up);
	}
	for (unsigned int done = 0; done < block_rows;) {
		DevImage batch = img;
		batch.block_row0 = block_row0 + done;
		batch.block_rows = block_rows - done < rows_per_batch ? block_rows - done : (unsigned int)rows_per_batch;
		batch.out = d_out + (size_t)done * blocks_x * 16;
		astcenc_error st = ctx->plan.driver == 0 ? launch_batch(ctx, batch, stream, up) : launch_driver(ctx, batch, stream);
		if (st != ASTCENC_SUCCESS) {
			return st;
		}
		done += batch.block_rows;
	}
	return ASTCENC_SUCCESS;
}

static astcenc_error launch_slab(astcenc_context* ctx, const DevImage& src, unsigned int block_row0, unsigned int block_rows, uint8_t* d_out, cudaStream_t stream,
                                 const UploadPlan* up = nullptr) {
	return scratch_turn(ctx, stream, [&] { return launch_slab_locked(ctx, src, block_row0, block_rows, d_out, stream, up); });
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
static astcenc_error compress_image_gpu(astcenc_context* ctx, const astcenc_image& image, const SlabGeometry& geo, const astcenc_swizzle& swizzle,
                                        uint8_t* data_out) {
	DeviceGuard guard(ctx->device);
	if (!guard.ok) {
		return ASTCENC_ERR_BAD_CONTEXT;
	}
	// 3D block sizes (astcenc_entry.cpp:906-1043): one pass over the volume, whose slices go up into one contiguous buffer before
	// it; its blocks come out in (z, y, x) order and its "block rows" count layer * blocks_y + row. 3D images with 2D blocks are
	// an array of independent 2D slices (astcenc.h:94-100): one banded pass per slice. Progress runs over all passes.
	const size_t slice_bytes = geo.slice_bytes;
	const size_t out_bytes = geo.pass_out_bytes();
	astcenc_error st = ensure_buffer(ctx->image, slice_bytes * geo.pass_slices());
	if (st == ASTCENC_SUCCESS) {
		st = ensure_buffer(ctx->out, out_bytes);
	}
	if (st != ASTCENC_SUCCESS) {
		return st;
	}
	ctx->last_h2d = ctx->last_d2h = 0;
	ctx->last_kernel_ms = 0.0f;
	float total_ms = 0.0f;
	// the pass starts behind the last flag clear (astcenc_compress_reset), with its done counter at zero
	DevImage src = pass_image(ctx, ctx->image.ptr, (int)image.data_type, image.dim_x, image.dim_y, geo.pass_slices(), swizzle);
	src.cancel = ctx->d_words;
	src.done = ctx->d_words + 1;
	CUDA_TRY(cudaStreamWaitEvent(ctx->stream, ctx->ctl_ready, 0), return ASTCENC_ERR_BAD_CONTEXT);
	CUDA_TRY(cudaMemsetAsync(src.done, 0, sizeof(uint32_t), ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
	PassProgress pp;
	pp.callback = ctx->config.progress_callback;
	pp.total = static_cast<float>(geo.blocks);
	pp.min_diff = (4096.0f / pp.total) * 100.0f;
	pp.min_diff = pp.min_diff > 1.0f ? pp.min_diff : 1.0f;
	pp.last = 0.0f;
	for (unsigned int z = 0; z < geo.passes(); z++) {
		if (ctx->cancel.load()) {
			return ASTCENC_SUCCESS;
		}
		UploadPlan up = {static_cast<const uint8_t*>(image.data[z]), ctx->image.ptr, (size_t)image.dim_x * geo.texel_bytes, ctx->knobs.upload_bands};
		if (geo.volume) {
			st = upload_slices(ctx->image.ptr, image.data, 0, image.dim_z, slice_bytes, ctx->stream);
			if (st != ASTCENC_SUCCESS) {
				return st;
			}
		}
		CUDA_TRY(cudaEventRecord(ctx->ev0, ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
		st = launch_slab(ctx, src, 0, geo.pass_rows(), ctx->out.ptr, ctx->stream, geo.volume ? nullptr : &up);
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
		CUDA_TRY(cudaMemcpyAsync(data_out + (size_t)z * out_bytes, ctx->out.ptr, out_bytes, cudaMemcpyDeviceToHost, ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
		CUDA_TRY(cudaStreamSynchronize(ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
		float ms = 0.0f;
		cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1);
		total_ms += ms;
		ctx->last_h2d += slice_bytes * geo.pass_slices();
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
	astcenc_error status = check_compress_context(ctx);
	if (status == ASTCENC_SUCCESS) status = check_swizzle(*swizzle, ASTCENC_SWZ_1);
	if (status == ASTCENC_SUCCESS && thread_index >= ctx->thread_count) status = ASTCENC_ERR_BAD_PARAM;
	if (status != ASTCENC_SUCCESS) {
		return status;
	}
	const astcenc_image& image = *imagep;
	const SlabGeometry geo = slab_geometry(ctx, image.dim_x, image.dim_y, image.dim_z, (int)image.data_type);
	status = check_texel_count(image.dim_x, image.dim_y, image.dim_z);
	if (status == ASTCENC_SUCCESS && geo.payload_overflow()) status = ASTCENC_ERR_BAD_PARAM;
	if (status == ASTCENC_SUCCESS && data_len < geo.out_bytes()) status = ASTCENC_ERR_OUT_OF_MEM;
	if (status == ASTCENC_SUCCESS) status = check_alpha_scale(ctx, image.dim_z);
	if (status != ASTCENC_SUCCESS) {
		return status;
	}
	if (ctx->thread_count == 1) {
		astcenc_compress_reset(ctx);
	}
	return run_once(ctx, ctx->compress_gate, [&] { return compress_image_gpu(ctx, image, geo, *swizzle, data_out); });
}

astcenc_error astcenc_compress_reset(astcenc_context* ctx) {
	if (ctx->config.flags & ASTCENC_FLG_DECOMPRESS_ONLY) {
		return ASTCENC_ERR_BAD_CONTEXT;
	}
	std::lock_guard<std::mutex> lk(ctx->mtx);
	ctx->compress_gate.reset();
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

// Entry e of an image table: dim_z slices of dim_x * dim_y texels of `data_type` at `data`, its payload at `payload`, call blocks
// [first, first + its blocks). Advances `first`. ASTCENC_ERR_BAD_PARAM when the image's payload does not fit a size_t, the image
// has 2^32 blocks or more (the table walks index an image's blocks with 32 bits, as block lists do) or the call's total does
// not fit a size_t.
static astcenc_error table_entry(const astcenc_context* ctx, int data_type, unsigned int dim_x, unsigned int dim_y, unsigned int dim_z, const void* data,
                                 uint8_t* payload, size_t& first, GatherImage& e) {
	const SlabGeometry geo = slab_geometry(ctx, dim_x, dim_y, dim_z, data_type);
	if (geo.payload_overflow() || geo.blocks > 0xFFFFFFFFu || geo.blocks > SIZE_MAX - first) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	e.data = data;
	e.payload = payload;
	e.first = first;
	e.avg_offset = 0;
	e.dim_x = dim_x;
	e.dim_y = dim_y;
	e.dim_z = dim_z;
	e.blocks_x = (unsigned int)geo.blocks_x;
	e.blocks_y = (unsigned int)geo.blocks_y;
	first += geo.blocks;
	return ASTCENC_SUCCESS;
}

// One launch decodes the `blocks` call blocks of an image table on `stream` (inside a scratch turn: the table goes up into the
// context's table buffer, ctx->list).
static astcenc_error launch_decode(astcenc_context* ctx, const GatherImage* table, unsigned int image_count, size_t blocks, int data_type,
                                   const astcenc_swizzle& swizzle, cudaStream_t stream) {
	astcenc_error st = ensure_buffer(ctx->list, image_count * sizeof(GatherImage));
	if (st != ASTCENC_SUCCESS) {
		return st;
	}
	// (from pageable memory: staged by the driver before the call returns)
	CUDA_TRY(cudaMemcpyAsync(ctx->list.ptr, table, image_count * sizeof(GatherImage), cudaMemcpyHostToDevice, stream), return ASTCENC_ERR_BAD_CONTEXT);
	const unsigned int warps = ASTC_DECODE_THREADS / 32;
	const size_t ctas = (blocks + warps - 1) / warps;
	const unsigned int grid = ctas < (size_t)ctx->sm_count * 8 ? (unsigned int)ctas : (unsigned int)ctx->sm_count * 8;
	astc_decompress_images_kernel<<<grid, ASTC_DECODE_THREADS, ASTC_SMEM_HDR + warps * D_SLICE, stream>>>(
	    ctx->tables->bsd, ctx->dcfg, pass_image(ctx, nullptr, data_type, 0, 0, 0, swizzle), ctx->list.as<const GatherImage>(), image_count, blocks);
	ctx->launches++;
	CUDA_TRY(cudaGetLastError(), return ASTCENC_ERR_BAD_CONTEXT);
	return ASTCENC_SUCCESS;
}

// The host-pointer twin of astcenc_b200_decompress_device_images: the whole payload goes up into ctx->out, a one-entry table
// points it at ctx->image (the image's dim_z slices: an array, or the volume of a 3D block size), one launch decodes it and each
// slice comes back into image.data[z]. The buffers are shared with the compression path: everything up to the copies back is
// one scratch turn, and the call waits for them outside it.
static astcenc_error decompress_image_gpu(astcenc_context* ctx, const uint8_t* data, astcenc_image& image, const SlabGeometry& geo, const astcenc_swizzle& swizzle) {
	DeviceGuard guard(ctx->device);
	if (!guard.ok) {
		return ASTCENC_ERR_BAD_CONTEXT;
	}
	astcenc_error st = scratch_turn(ctx, ctx->stream, [&]() -> astcenc_error {
		const size_t slice_bytes = geo.slice_bytes;
		astcenc_error r = ensure_buffer(ctx->image, slice_bytes * image.dim_z);
		if (r == ASTCENC_SUCCESS) r = ensure_buffer(ctx->out, geo.out_bytes());
		GatherImage e;
		size_t blocks = 0;
		if (r == ASTCENC_SUCCESS) r = table_entry(ctx, (int)image.data_type, image.dim_x, image.dim_y, image.dim_z, ctx->image.ptr, ctx->out.ptr, blocks, e);
		if (r != ASTCENC_SUCCESS) {
			return r;
		}
		CUDA_TRY(cudaMemcpyAsync(ctx->out.ptr, data, geo.out_bytes(), cudaMemcpyHostToDevice, ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
		r = launch_decode(ctx, &e, 1, blocks, (int)image.data_type, swizzle, ctx->stream);
		for (unsigned int z = 0; z < image.dim_z && r == ASTCENC_SUCCESS; z++) {
			CUDA_TRY(cudaMemcpyAsync(image.data[z], ctx->image.ptr + (size_t)z * slice_bytes, slice_bytes, cudaMemcpyDeviceToHost, ctx->stream),
			         return ASTCENC_ERR_BAD_CONTEXT);
		}
		return r;
	});
	if (st != ASTCENC_SUCCESS) {
		return st;
	}
	CUDA_TRY(cudaStreamSynchronize(ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
	return ASTCENC_SUCCESS;
}

// astcenc_decompress_image (astcenc_entry.cpp:1274-1385): same check order; the decode mode follows the output type
astcenc_error astcenc_decompress_image(astcenc_context* ctx, const uint8_t* data, size_t data_len, astcenc_image* image_outp, const astcenc_swizzle* swizzle,
                                       unsigned int thread_index) {
	if (thread_index >= ctx->thread_count) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	astcenc_error status = check_swizzle(*swizzle, ASTCENC_SWZ_Z);
	if (status != ASTCENC_SUCCESS) {
		return status;
	}
	astcenc_image& image = *image_outp;
	const SlabGeometry geo = slab_geometry(ctx, image.dim_x, image.dim_y, image.dim_z, (int)image.data_type);
	status = check_texel_count(image.dim_x, image.dim_y, image.dim_z);
	if (status == ASTCENC_SUCCESS && geo.payload_overflow()) status = ASTCENC_ERR_BAD_PARAM;
	if (status == ASTCENC_SUCCESS && data_len < geo.out_bytes()) status = ASTCENC_ERR_OUT_OF_MEM;
	if (status != ASTCENC_SUCCESS) {
		return status;
	}
	// any subset of the thread_count callers may call; the image is decoded once, everybody returns when it is done
	if (ctx->thread_count == 1) {
		astcenc_decompress_reset(ctx);
	}
	return run_once(ctx, ctx->decompress_gate, [&] { return decompress_image_gpu(ctx, data, image, geo, *swizzle); });
}

astcenc_error astcenc_decompress_reset(astcenc_context* ctx) {
	std::lock_guard<std::mutex> lk(ctx->mtx);
	ctx->decompress_gate.reset();
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

// One metrics call of a planned table (plan_metrics) on `stream`, inside a scratch turn: the table and the map list go up into
// the context's table buffer (ctx->list) in one copy, the metrics kernel and the finish kernel run, then the map kernel when
// an entry asks for a map. The sums of entry j are left at ctx->metric_partials + (plan.ctas + j) * ASTC_METRIC_SUMS doubles.
static astcenc_error launch_metrics(astcenc_context* ctx, const std::vector<MetricEntry>& table, const MetricPlan& plan, int hdr, int normal,
                                    int input_components, int fstop_lo, int fstop_hi, cudaStream_t stream) {
	const size_t table_bytes = table.size() * sizeof(MetricEntry);
	const size_t map_bytes = plan.maps.size() * sizeof(MetricMap);
	std::vector<uint8_t> up(table_bytes + map_bytes);
	memcpy(up.data(), table.data(), table_bytes);
	if (map_bytes != 0) {
		memcpy(up.data() + table_bytes, plan.maps.data(), map_bytes);
	}
	astcenc_error st = ensure_buffer(ctx->list, up.size());
	if (st == ASTCENC_SUCCESS) st = ensure_buffer(ctx->metric_partials, plan.partial_doubles * sizeof(double));
	if (st != ASTCENC_SUCCESS) {
		return st;
	}
	// (from pageable memory: staged by the driver before the call returns)
	CUDA_TRY(cudaMemcpyAsync(ctx->list.ptr, up.data(), up.size(), cudaMemcpyHostToDevice, stream), return ASTCENC_ERR_BAD_CONTEXT);
	MetricArgs a;
	a.entries = ctx->list.as<const MetricEntry>();
	a.count = (unsigned int)table.size();
	a.maps = reinterpret_cast<const MetricMap*>(ctx->list.ptr + table_bytes);
	a.map_count = (unsigned int)plan.maps.size();
	a.map_blocks = plan.map_blocks;
	a.bx = ctx->config.block_x;
	a.by = ctx->config.block_y;
	a.bz = ctx->config.block_z > 1 ? ctx->config.block_z : 1;
	a.hdr = hdr != 0;
	a.normal = normal != 0;
	a.components = input_components;
	a.fstop_lo = fstop_lo;
	a.fstop_hi = fstop_hi;
	a.ctas = plan.ctas;
	a.partials = ctx->metric_partials.as<double>();
	astc_error_metrics_kernel<<<(unsigned int)plan.ctas, ASTC_METRIC_THREADS, 0, stream>>>(a);
	ctx->launches++;
	astc_error_metrics_finish_kernel<<<plan.finish_grid, ASTC_METRIC_FINISH_GROUPS * ASTC_METRIC_SUMS, 0, stream>>>(a);
	ctx->launches++;
	if (plan.map_grid != 0) {
		astc_block_error_kernel<<<plan.map_grid, ASTC_METRIC_MAP_WARPS * 32, 0, stream>>>(a);
		ctx->launches++;
	}
	CUDA_TRY(cudaGetLastError(), return ASTCENC_ERR_BAD_CONTEXT);
	return ASTCENC_SUCCESS;
}

// astcenc_b200_compute_error_metrics: the CLI's compute_error_metrics (astcenccli_error_metrics.cpp:109-413) with the
// per-texel work and the reductions on the device; the final dB figures are computed here exactly as the CLI prints them.
// A one-entry metrics call: both images' slices go up into ctx->image and ctx->image2, the table compares their intersection,
// and the 17 sums come back.
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
	std::vector<MetricEntry> table(1);
	MetricEntry& e = table[0];
	e.type1 = (int)img1->data_type;
	e.type2 = (int)img2->data_type;
	e.pitch1 = img1->dim_x;
	e.pitch2 = img2->dim_x;
	e.stride1 = (size_t)img1->dim_x * img1->dim_y;
	e.stride2 = (size_t)img2->dim_x * img2->dim_y;
	e.dim_x = dim_x;
	e.dim_y = dim_y;
	e.dim_z = dim_z;
	e.metrics = nullptr;
	e.block_error = nullptr;
	MetricPlan plan;
	if (!plan_metrics(table, ctx->config.block_x, ctx->config.block_y, ctx->config.block_z > 1 ? ctx->config.block_z : 1, plan)) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	const size_t slice1 = e.stride1 * texel_bytes(e.type1);
	const size_t slice2 = e.stride2 * texel_bytes(e.type2);
	double sums[ASTC_METRIC_SUMS];
	astcenc_error st = scratch_turn(ctx, ctx->stream, [&]() -> astcenc_error {
		astcenc_error r = ensure_buffer(ctx->image, slice1 * dim_z);
		if (r == ASTCENC_SUCCESS) r = ensure_buffer(ctx->image2, slice2 * dim_z);
		if (r == ASTCENC_SUCCESS) r = upload_slices(ctx->image.ptr, img1->data, 0, dim_z, slice1, ctx->stream);
		if (r == ASTCENC_SUCCESS) r = upload_slices(ctx->image2.ptr, img2->data, 0, dim_z, slice2, ctx->stream);
		if (r != ASTCENC_SUCCESS) {
			return r;
		}
		e.img1 = ctx->image.ptr;
		e.img2 = ctx->image2.ptr;
		r = launch_metrics(ctx, table, plan, compute_hdr_metrics, compute_normal_metrics, input_components, fstop_lo, fstop_hi, ctx->stream);
		if (r == ASTCENC_SUCCESS) {
			CUDA_TRY(cudaMemcpyAsync(sums, ctx->metric_partials.as<double>() + plan.ctas * ASTC_METRIC_SUMS, sizeof(sums), cudaMemcpyDeviceToHost, ctx->stream),
			         return ASTCENC_ERR_BAD_CONTEXT);
		}
		return r;
	});
	if (st != ASTCENC_SUCCESS) {
		return st;
	}
	CUDA_TRY(cudaStreamSynchronize(ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
	metric_close(sums, compute_hdr_metrics, compute_normal_metrics, input_components, fstop_lo, fstop_hi, (double)(dim_x * dim_y * dim_z), out);
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
	astcenc_error status = check_compress_context(ctx);
	if (status == ASTCENC_SUCCESS) status = check_swizzle(*swizzle, ASTCENC_SWZ_1);
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
	cudaStream_t s = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : ctx->stream;
	return launch_slab(ctx, pass_image(ctx, d_pixels, (int)data_type, dim_x, dim_y, 1, *swizzle), block_row0, block_rows, d_out, s);
}

// One entry of a staging call: an image and its payload (plan_blocks sets `first` and `avg_offset`), its list (null: every
// block), the staging blocks it owns (the image's blocks, or the list's capacity) and the block rows [row0, row1) of its
// alpha-scale pre-pass, clamped to the image: the rows a host list touches, else the whole image.
struct BlockEntry {
	GatherImage image{};
	const GatherList* list = nullptr;
	size_t blocks = 0;
	unsigned int row0 = 0, row1 = 0xFFFFFFFFu;
};

// What launch_blocks compresses: a block-list table (astc_dev_gather.cuh). Entry j is table[j], lists[j] (no lists: every block
// of each image) and the block rows of its alpha-scale pre-pass (rows[j]). `words` go up behind the lists: a host list's count
// word and indices, at which its GatherList (count and indices null here) is pointed.
struct BlockCall {
	std::vector<GatherImage> table;
	std::vector<GatherList> lists;
	std::vector<std::pair<unsigned int, unsigned int>> rows;
	std::vector<uint32_t> words;
	size_t blocks = 0;                 // staging blocks of the whole call
	int data_type = 0;
};

// The staging call of checked `entries`: each owns the staging blocks and averages that follow those of the entries before it;
// entries of no staging blocks (lists of capacity 0) are left out. ASTCENC_ERR_BAD_PARAM when the total does not fit a size_t.
static astcenc_error plan_blocks(const std::vector<BlockEntry>& entries, astcenc_type data_type, BlockCall& call) {
	call.data_type = (int)data_type;
	size_t avg_offset = 0;
	for (const BlockEntry& en : entries) {
		if (en.blocks == 0) {
			continue;
		}
		if (en.blocks > SIZE_MAX - call.blocks) {
			return ASTCENC_ERR_BAD_PARAM;
		}
		GatherImage e = en.image;
		e.first = call.blocks;
		e.avg_offset = avg_offset;
		call.table.push_back(e);
		if (en.list != nullptr) {
			call.lists.push_back(*en.list);
		}
		call.rows.push_back({en.row0, en.row1 < e.blocks_y ? en.row1 : e.blocks_y});
		call.blocks += en.blocks;
		avg_offset += (size_t)e.dim_x * e.dim_y;
	}
	return ASTCENC_SUCCESS;
}

// Staging calls (astc_dev_gather.cuh): gather -> one ordinary pass over the staging row -> scatter, chunk by chunk (a staging
// row is one block row, which the batching of launch_slab_locked cannot split: a chunk holds at most knobs.batch_blocks
// blocks). A chunk may span several entries. The whole call is one scratch turn (launch_blocks), like a launch_slab.
static astcenc_error launch_blocks_locked(astcenc_context* ctx, const BlockCall& call, const astcenc_swizzle& swizzle, cudaStream_t stream) {
	const DevBsd& bsd = ctx->tables->bsd;
	const bool volume = bsd.dim_z > 1;
	const unsigned int radius = volume ? 0 : ctx->config.a_scale_radius;
	const size_t n = call.blocks;
	const size_t chunk = n < ctx->knobs.batch_blocks ? n : ctx->knobs.batch_blocks;
	const size_t avg_floats = call.table.back().avg_offset + (size_t)call.table.back().dim_x * call.table.back().dim_y;
	const size_t table_bytes = call.table.size() * sizeof(GatherImage);
	const size_t lists_bytes = call.lists.size() * sizeof(GatherList);
	const size_t list_bytes = table_bytes + lists_bytes + call.words.size() * sizeof(uint32_t);
	astcenc_error st = ensure_buffer(ctx->list, list_bytes);
	if (st == ASTCENC_SUCCESS) st = ensure_buffer(ctx->list_image, chunk * bsd.texel_count * texel_bytes(call.data_type));
	if (st == ASTCENC_SUCCESS) st = ensure_buffer(ctx->list_out, chunk * 16);
	if (st == ASTCENC_SUCCESS && radius != 0) {
		st = ensure_buffer(ctx->list_alpha, avg_floats * sizeof(float));
		if (st == ASTCENC_SUCCESS) st = ensure_scratch(ctx, 0, chunk * bsd.texel_count);
	}
	if (st == ASTCENC_SUCCESS) {
		// the table, its lists and the words in one copy, from pageable memory: staged by the driver before the call returns, so
		// a host list may go when this function does
		std::vector<GatherList> lists = call.lists;
		for (GatherList& l : lists) {
			if (l.count == nullptr) {
				l.count = reinterpret_cast<const uint32_t*>(ctx->list.ptr + table_bytes + lists_bytes);
				l.indices = l.count + 1;
			}
		}
		std::vector<uint8_t> up(reinterpret_cast<const uint8_t*>(call.table.data()), reinterpret_cast<const uint8_t*>(call.table.data()) + table_bytes);
		up.insert(up.end(), reinterpret_cast<const uint8_t*>(lists.data()), reinterpret_cast<const uint8_t*>(lists.data()) + lists_bytes);
		up.insert(up.end(), reinterpret_cast<const uint8_t*>(call.words.data()), reinterpret_cast<const uint8_t*>(call.words.data()) + call.words.size() * sizeof(uint32_t));
		CUDA_TRY(cudaMemcpyAsync(ctx->list.ptr, up.data(), list_bytes, cudaMemcpyHostToDevice, stream), st = ASTCENC_ERR_BAD_CONTEXT);
	}
	// The staging pass reads averages gathered from the sources', so it runs no pre-pass of its own: its box filter would reach
	// across the seams between unrelated blocks. A source's averages cover its window's rows, at their image positions, in the
	// source's region of list_alpha. The threshold depends on the footprint and the radius alone: one value serves every source.
	float threshold = 0.0f;
	for (size_t k = 0; k < call.table.size() && st == ASTCENC_SUCCESS && radius != 0; k++) {
		const GatherImage& e = call.table[k];
		const DevImage src = pass_image(ctx, e.data, call.data_type, e.dim_x, e.dim_y, e.dim_z, swizzle);
		st = alpha_prepass(ctx, src, call.rows[k].first, call.rows[k].second, ctx->list_alpha.as<float>() + e.avg_offset, stream, threshold);
	}
	GatherArgs g;
	g.dst = ctx->list_image.ptr;
	g.avg_src = radius != 0 ? ctx->list_alpha.as<const float>() : nullptr;
	g.avg_dst = radius != 0 ? ctx->alpha.as<float>() : nullptr;
	g.words = (unsigned int)(texel_bytes(call.data_type) / 4);
	g.bx = bsd.dim_x;
	g.by = bsd.dim_y;
	g.bz = bsd.dim_z;
	g.images = ctx->list.as<const GatherImage>();
	g.image_count = (unsigned int)call.table.size();
	g.lists = call.lists.empty() ? nullptr : reinterpret_cast<const GatherList*>(ctx->list.ptr + table_bytes);
	for (size_t first = 0; first < n && st == ASTCENC_SUCCESS; first += chunk) {
		const unsigned int m = (unsigned int)(n - first < chunk ? n - first : chunk);
		g.base = first;
		g.n = m;
		const unsigned int warps = ASTC_GATHER_THREADS / 32;
		astc_gather_blocks_kernel<<<(m + warps - 1) / warps < (unsigned int)ctx->plan.grid * 16 ? (m + warps - 1) / warps : (unsigned int)ctx->plan.grid * 16, ASTC_GATHER_THREADS, 0, stream>>>(g);
		ctx->launches++;
		// (the staging volume is one layer deep)
		DevImage staged = pass_image(ctx, ctx->list_image.ptr, call.data_type, m * bsd.dim_x, bsd.dim_y, volume ? bsd.dim_z : 1, swizzle);
		staged.alpha_avg = radius != 0 ? ctx->alpha.as<float>() : nullptr;
		staged.alpha_threshold = threshold;
		st = launch_slab_locked(ctx, staged, 0, 1, ctx->list_out.ptr, stream, nullptr);
		if (st == ASTCENC_SUCCESS) {
			astc_scatter_blocks_kernel<<<(m + ASTC_GATHER_THREADS - 1) / ASTC_GATHER_THREADS, ASTC_GATHER_THREADS, 0, stream>>>(ctx->list_out.ptr, g);
			ctx->launches++;
			CUDA_TRY(cudaGetLastError(), st = ASTCENC_ERR_BAD_CONTEXT);
		}
	}
	return st;
}

// A staging call on `cuda_stream` (null: the context's stream); a call of no staging blocks launches nothing.
static astcenc_error launch_blocks(astcenc_context* ctx, const BlockCall& call, const astcenc_swizzle& swizzle, void* cuda_stream) {
	if (call.blocks == 0) {
		return ASTCENC_SUCCESS;
	}
	DeviceGuard guard(ctx->device);
	if (!guard.ok) {
		return ASTCENC_ERR_BAD_CONTEXT;
	}
	cudaStream_t stream = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : ctx->stream;
	return scratch_turn(ctx, stream, [&] { return launch_blocks_locked(ctx, call, swizzle, stream); });
}

// A host list is a one-entry block-list table: its count word and indices go up with the table (BlockCall::words).
astcenc_error astcenc_b200_compress_device_blocks(astcenc_context* ctx, const void* d_pixels, astcenc_type data_type, unsigned int dim_x, unsigned int dim_y,
                                                  unsigned int dim_z, const astcenc_swizzle* swizzle, const uint32_t* block_indices, unsigned int block_count,
                                                  uint8_t* d_payload, void* cuda_stream) {
	astcenc_error status = check_compress_context(ctx);
	if (status == ASTCENC_SUCCESS && !swizzle) status = ASTCENC_ERR_BAD_PARAM;
	if (status == ASTCENC_SUCCESS) status = check_swizzle(*swizzle, ASTCENC_SWZ_1);
	if (status == ASTCENC_SUCCESS && (dim_x == 0 || dim_y == 0 || dim_z == 0 || !d_pixels || !d_payload || (block_count != 0 && !block_indices))) {
		status = ASTCENC_ERR_BAD_PARAM;
	}
	if (status == ASTCENC_SUCCESS) status = check_data_type(data_type);
	if (status == ASTCENC_SUCCESS) status = check_alpha_scale(ctx, dim_z);
	const SlabGeometry geo = slab_geometry(ctx, dim_x, dim_y, dim_z, (int)data_type);
	if (status == ASTCENC_SUCCESS && geo.overflow) status = ASTCENC_ERR_BAD_PARAM;
	if (status != ASTCENC_SUCCESS) {
		return status;
	}
	// Every index is checked below, so the list's bound is the block count clamped to 32 bits; the one index that skips,
	// 0xFFFFFFFF in an image of more than 2^32 blocks, lies in an image of at least 256 GiB.
	const GatherList list{nullptr, nullptr, block_count, geo.blocks < 0xFFFFFFFFu ? (unsigned int)geo.blocks : 0xFFFFFFFFu};
	BlockEntry e{{d_pixels, d_payload, 0, 0, dim_x, dim_y, dim_z, (unsigned int)geo.blocks_x, (unsigned int)geo.blocks_y}, &list, block_count, 0xFFFFFFFFu, 0};
	// the list is checked whole before anything is enqueued; the pre-pass window is the block rows it touches (2D images)
	for (unsigned int i = 0; i < block_count; i++) {
		if (block_indices[i] >= geo.blocks) {
			return ASTCENC_ERR_BAD_PARAM;
		}
		const unsigned int row = (unsigned int)(block_indices[i] / geo.blocks_x);
		e.row0 = row < e.row0 ? row : e.row0;
		e.row1 = row + 1 > e.row1 ? row + 1 : e.row1;
	}
	BlockCall call;
	plan_blocks({e}, data_type, call);      // (one entry of fewer than 2^32 blocks: nothing to refuse)
	call.words.push_back(block_count);
	call.words.insert(call.words.end(), block_indices, block_indices + block_count);
	return launch_blocks(ctx, call, *swizzle, cuda_stream);
}

// The image table of a multi-image call, checked whole before anything is enqueued (the caller has checked the context, the
// swizzle and the pointers): zero dimensions and the data type (ASTCENC_ERR_BAD_PARAM), a_scale_radius on a texture array
// (ASTCENC_ERR_NOT_IMPLEMENTED), then the block counts (table_entry). Fills one entry per image, of all its blocks.
static astcenc_error check_image_table(const astcenc_context* ctx, const astcenc_b200_device_image* images, unsigned int image_count, astcenc_type data_type,
                                       std::vector<BlockEntry>& entries) {
	astcenc_error status = ASTCENC_SUCCESS;
	for (unsigned int i = 0; i < image_count && status == ASTCENC_SUCCESS; i++) {
		status = check_texel_count(images[i].dim_x, images[i].dim_y, images[i].dim_z);
	}
	if (status == ASTCENC_SUCCESS) status = check_data_type(data_type);
	for (unsigned int i = 0; i < image_count && status == ASTCENC_SUCCESS; i++) {
		status = check_alpha_scale(ctx, images[i].dim_z);
	}
	entries.resize(image_count);
	size_t first = 0;
	for (unsigned int i = 0; i < image_count && status == ASTCENC_SUCCESS; i++) {
		const astcenc_b200_device_image& im = images[i];
		status = table_entry(ctx, (int)data_type, im.dim_x, im.dim_y, im.dim_z, im.data, im.payload, first, entries[i].image);
		entries[i].blocks = first - entries[i].image.first;
	}
	return status;
}

astcenc_error astcenc_b200_compress_device_images(astcenc_context* ctx, const astcenc_b200_device_image* images, unsigned int image_count, astcenc_type data_type,
                                                  const astcenc_swizzle* swizzle, void* cuda_stream) {
	astcenc_error status = check_compress_context(ctx);
	if (status == ASTCENC_SUCCESS && !swizzle) status = ASTCENC_ERR_BAD_PARAM;
	if (status == ASTCENC_SUCCESS) status = check_swizzle(*swizzle, ASTCENC_SWZ_1);
	if (status == ASTCENC_SUCCESS && image_count != 0 && !images) status = ASTCENC_ERR_BAD_PARAM;
	for (unsigned int i = 0; i < image_count && status == ASTCENC_SUCCESS; i++) {
		if (!images[i].data || !images[i].payload) {
			status = ASTCENC_ERR_BAD_PARAM;
		}
	}
	std::vector<BlockEntry> entries;
	if (status == ASTCENC_SUCCESS) status = check_image_table(ctx, images, image_count, data_type, entries);
	BlockCall call;
	if (status == ASTCENC_SUCCESS) status = plan_blocks(entries, data_type, call);
	return status == ASTCENC_SUCCESS ? launch_blocks(ctx, call, *swizzle, cuda_stream) : status;
}

// The host-pointer twin: every image goes up into one device buffer (ctx->image), the table is pointed at it and at one payload
// buffer (ctx->out), one device-image call runs on the context's stream, and each payload comes back into data_out[i].
astcenc_error astcenc_b200_compress_images(astcenc_context* ctx, astcenc_image* const* images, unsigned int image_count, const astcenc_swizzle* swizzle,
                                           uint8_t* const* data_out, const size_t* data_len) {
	astcenc_error status = check_compress_context(ctx);
	if (status == ASTCENC_SUCCESS && !swizzle) status = ASTCENC_ERR_BAD_PARAM;
	if (status == ASTCENC_SUCCESS) status = check_swizzle(*swizzle, ASTCENC_SWZ_1);
	if (status == ASTCENC_SUCCESS && image_count != 0 && (!images || !data_out || !data_len)) status = ASTCENC_ERR_BAD_PARAM;
	std::vector<astcenc_b200_device_image> descs;
	for (unsigned int i = 0; i < image_count && status == ASTCENC_SUCCESS; i++) {
		const astcenc_image* im = images[i];
		if (!im || !im->data || !data_out[i] || im->data_type != images[0]->data_type) {
			status = ASTCENC_ERR_BAD_PARAM;
		} else {
			// (planned with the host pointers; pointed at the device copies below)
			descs.push_back({im->data, im->dim_x, im->dim_y, im->dim_z, data_out[i]});
		}
	}
	std::vector<BlockEntry> entries;
	BlockCall call;
	if (status == ASTCENC_SUCCESS && image_count != 0) {
		status = check_image_table(ctx, descs.data(), image_count, images[0]->data_type, entries);
		if (status == ASTCENC_SUCCESS) status = plan_blocks(entries, images[0]->data_type, call);
	}
	for (unsigned int i = 0; i < image_count && status == ASTCENC_SUCCESS; i++) {
		if (data_len[i] < entries[i].blocks * 16) {
			status = ASTCENC_ERR_OUT_OF_MEM;
		}
	}
	if (status != ASTCENC_SUCCESS || image_count == 0) {
		return status;
	}
	DeviceGuard guard(ctx->device);
	if (!guard.ok) {
		return ASTCENC_ERR_BAD_CONTEXT;
	}
	// each image starts 256-byte aligned in the upload buffer
	std::vector<size_t> in_offset(image_count);
	size_t in_bytes = 0;
	for (unsigned int i = 0; i < image_count; i++) {
		in_offset[i] = in_bytes;
		in_bytes += ((size_t)images[i]->dim_x * images[i]->dim_y * images[i]->dim_z * texel_bytes(call.data_type) + 255) & ~(size_t)255;
	}
	astcenc_error st = ensure_buffer(ctx->image, in_bytes);
	if (st == ASTCENC_SUCCESS) st = ensure_buffer(ctx->out, call.blocks * 16);
	if (st != ASTCENC_SUCCESS) {
		return st;
	}
	ctx->last_h2d = ctx->last_d2h = 0;
	ctx->last_kernel_ms = 0.0f;
	for (unsigned int i = 0; i < image_count; i++) {
		const astcenc_image& im = *images[i];
		uint8_t* d_data = ctx->image.ptr + in_offset[i];
		const size_t slice_bytes = (size_t)im.dim_x * im.dim_y * texel_bytes(call.data_type);
		st = upload_slices(d_data, im.data, 0, im.dim_z, slice_bytes, ctx->stream);
		if (st != ASTCENC_SUCCESS) {
			return st;
		}
		ctx->last_h2d += slice_bytes * im.dim_z;
		call.table[i].data = d_data;
		call.table[i].payload = ctx->out.ptr + call.table[i].first * 16;
	}
	CUDA_TRY(cudaEventRecord(ctx->ev0, ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
	st = launch_blocks(ctx, call, *swizzle, ctx->stream);
	if (st != ASTCENC_SUCCESS) {
		return st;
	}
	CUDA_TRY(cudaEventRecord(ctx->ev1, ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
	for (unsigned int i = 0; i < image_count; i++) {
		const size_t bytes = entries[i].blocks * 16;
		CUDA_TRY(cudaMemcpyAsync(data_out[i], call.table[i].payload, bytes, cudaMemcpyDeviceToHost, ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
		ctx->last_d2h += bytes;
	}
	CUDA_TRY(cudaStreamSynchronize(ctx->stream), return ASTCENC_ERR_BAD_CONTEXT);
	cudaEventElapsedTime(&ctx->last_kernel_ms, ctx->ev0, ctx->ev1);
	return ASTCENC_SUCCESS;
}

// Decode calls: every image is checked before anything is enqueued; the table goes up in one copy and one launch decodes every
// block of the call, in one scratch turn (the launch takes the context's table buffer, ctx->list).
astcenc_error astcenc_b200_decompress_device_images(astcenc_context* ctx, const astcenc_b200_device_decode_image* images, unsigned int image_count,
                                                    astcenc_type data_type, const astcenc_swizzle* swizzle, void* cuda_stream) {
	astcenc_error status = swizzle ? check_swizzle(*swizzle, ASTCENC_SWZ_Z) : ASTCENC_ERR_BAD_PARAM;
	if (status == ASTCENC_SUCCESS && image_count != 0 && !images) status = ASTCENC_ERR_BAD_PARAM;
	for (unsigned int i = 0; i < image_count && status == ASTCENC_SUCCESS; i++) {
		if (!images[i].payload || !images[i].data) {
			status = ASTCENC_ERR_BAD_PARAM;
		} else {
			status = check_texel_count(images[i].dim_x, images[i].dim_y, images[i].dim_z);
		}
	}
	if (status == ASTCENC_SUCCESS) status = check_data_type(data_type);
	std::vector<GatherImage> table(image_count);
	size_t blocks = 0;
	for (unsigned int i = 0; i < image_count && status == ASTCENC_SUCCESS; i++) {
		const astcenc_b200_device_decode_image& im = images[i];
		// (the payload is read, never written)
		status = table_entry(ctx, (int)data_type, im.dim_x, im.dim_y, im.dim_z, im.data, const_cast<uint8_t*>(im.payload), blocks, table[i]);
	}
	if (status != ASTCENC_SUCCESS || image_count == 0) {
		return status;
	}
	DeviceGuard guard(ctx->device);
	if (!guard.ok) {
		return ASTCENC_ERR_BAD_CONTEXT;
	}
	cudaStream_t s = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : ctx->stream;
	return scratch_turn(ctx, s, [&] { return launch_decode(ctx, table.data(), image_count, blocks, (int)data_type, *swizzle, s); });
}

// Metrics calls: every pair is checked before anything is enqueued; the table goes up in one copy and the call is two
// launches, three with a map, in one scratch turn.
astcenc_error astcenc_b200_compute_error_metrics_device_images(astcenc_context* ctx, int compute_hdr_metrics, int compute_normal_metrics,
                                                               int input_components, const astcenc_b200_device_metrics_image* images,
                                                               unsigned int image_count, int fstop_lo, int fstop_hi, void* cuda_stream) {
	if (!ctx || input_components < 1 || input_components > 4) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	if (fstop_lo < -125 || fstop_hi > 125) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	if (image_count != 0 && !images) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	auto aligned = [](const void* p, size_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; };
	std::vector<MetricEntry> table(image_count);
	for (unsigned int i = 0; i < image_count; i++) {
		const astcenc_b200_device_metrics_image& im = images[i];
		if (!im.original || !im.decoded || !im.metrics || check_texel_count(im.dim_x, im.dim_y, im.dim_z) != ASTCENC_SUCCESS ||
		    check_data_type(im.original_type) != ASTCENC_SUCCESS || check_data_type(im.decoded_type) != ASTCENC_SUCCESS ||
		    !aligned(im.original, texel_bytes(im.original_type)) || !aligned(im.decoded, texel_bytes(im.decoded_type)) || !aligned(im.metrics, 8) ||
		    !aligned(im.block_error, 4)) {
			return ASTCENC_ERR_BAD_PARAM;
		}
		MetricEntry& e = table[i];
		e.img1 = im.original;
		e.img2 = im.decoded;
		e.type1 = (int)im.original_type;
		e.type2 = (int)im.decoded_type;
		e.pitch1 = e.pitch2 = im.dim_x;
		e.stride1 = e.stride2 = (size_t)im.dim_x * im.dim_y;
		e.dim_x = im.dim_x;
		e.dim_y = im.dim_y;
		e.dim_z = im.dim_z;
		e.metrics = im.metrics;
		e.block_error = im.block_error;
	}
	MetricPlan plan;
	if (!plan_metrics(table, ctx->config.block_x, ctx->config.block_y, ctx->config.block_z > 1 ? ctx->config.block_z : 1, plan)) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	if (image_count == 0) {
		return ASTCENC_SUCCESS;
	}
	DeviceGuard guard(ctx->device);
	if (!guard.ok) {
		return ASTCENC_ERR_BAD_CONTEXT;
	}
	cudaStream_t s = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : ctx->stream;
	return scratch_turn(ctx, s, [&] {
		return launch_metrics(ctx, table, plan, compute_hdr_metrics, compute_normal_metrics, input_components, fstop_lo, fstop_hi, s);
	});
}

// Device block lists: an image table whose entry j owns capacity[j] staging blocks, the slots of its device list (GatherList).
// Checked whole before anything is enqueued, in the image-table order of astcenc_b200_compress_device_images; entries with a
// capacity of 0 are checked and then left out of the call.
astcenc_error astcenc_b200_compress_device_block_lists(astcenc_context* ctx, const astcenc_b200_device_block_list* lists, unsigned int list_count,
                                                       astcenc_type data_type, const astcenc_swizzle* swizzle, void* cuda_stream) {
	astcenc_error status = check_compress_context(ctx);
	if (status == ASTCENC_SUCCESS && !swizzle) status = ASTCENC_ERR_BAD_PARAM;
	if (status == ASTCENC_SUCCESS) status = check_swizzle(*swizzle, ASTCENC_SWZ_1);
	if (status == ASTCENC_SUCCESS && list_count != 0 && !lists) status = ASTCENC_ERR_BAD_PARAM;
	auto aligned4 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3) == 0; };
	std::vector<astcenc_b200_device_image> descs;
	for (unsigned int i = 0; i < list_count && status == ASTCENC_SUCCESS; i++) {
		const astcenc_b200_device_block_list& l = lists[i];
		if (!l.data || !l.payload || (l.capacity != 0 && (!l.indices || !l.count)) || !aligned4(l.indices) || !aligned4(l.count)) {
			status = ASTCENC_ERR_BAD_PARAM;
		}
		descs.push_back({l.data, l.dim_x, l.dim_y, l.dim_z, l.payload});
	}
	std::vector<BlockEntry> entries;
	if (status == ASTCENC_SUCCESS) status = check_image_table(ctx, descs.data(), list_count, data_type, entries);
	std::vector<GatherList> gather_lists(list_count);
	for (unsigned int i = 0; i < list_count && status == ASTCENC_SUCCESS; i++) {
		gather_lists[i] = {lists[i].indices, lists[i].count, lists[i].capacity, (unsigned int)entries[i].blocks};
		entries[i].list = &gather_lists[i];
		entries[i].blocks = lists[i].capacity;
	}
	BlockCall call;
	if (status == ASTCENC_SUCCESS) status = plan_blocks(entries, data_type, call);
	return status == ASTCENC_SUCCESS ? launch_blocks(ctx, call, *swizzle, cuda_stream) : status;
}

// Selection calls (astc_dev_select.cuh): every entry is checked before anything is enqueued; in one scratch turn the table goes
// up, the histograms are cleared and SELECT_KERNELS kernels run, whatever the number of entries.
astcenc_error astcenc_b200_select_blocks(astcenc_context* ctx, const astcenc_b200_block_selection* entries, unsigned int entry_count, void* cuda_stream) {
	if (!ctx || (entry_count != 0 && !entries)) {
		return ASTCENC_ERR_BAD_PARAM;
	}
	auto aligned4 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3) == 0; };
	std::vector<SelectEntry> table(entry_count);
	for (unsigned int i = 0; i < entry_count; i++) {
		const astcenc_b200_block_selection& x = entries[i];
		if (!x.count || (x.block_count != 0 && !x.map) || (x.capacity != 0 && !x.indices) || !aligned4(x.map) || !aligned4(x.indices) ||
		    !aligned4(x.count) || x.threshold != x.threshold) {
			return ASTCENC_ERR_BAD_PARAM;
		}
		SelectEntry& e = table[i];
		e.map = x.map;
		e.indices = x.indices;
		e.count = x.count;
		e.threshold = x.threshold;
		e.capacity = x.capacity;
		e.block_count = x.block_count;
	}
	if (entry_count == 0) {
		return ASTCENC_SUCCESS;
	}
	const size_t tiles = plan_select(table);
	DeviceGuard guard(ctx->device);
	if (!guard.ok) {
		return ASTCENC_ERR_BAD_CONTEXT;
	}
	cudaStream_t s = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : ctx->stream;
	return scratch_turn(ctx, s, [&]() -> astcenc_error {
		const size_t table_bytes = table.size() * sizeof(SelectEntry);
		const size_t hist_bytes = table.size() * 1024 * sizeof(uint32_t);
		astcenc_error r = ensure_buffer(ctx->select, table_bytes + hist_bytes + tiles * 2 * sizeof(uint32_t));
		if (r != ASTCENC_SUCCESS) {
			return r;
		}
		// (from pageable memory: staged by the driver before the call returns)
		CUDA_TRY(cudaMemcpyAsync(ctx->select.ptr, table.data(), table_bytes, cudaMemcpyHostToDevice, s), return ASTCENC_ERR_BAD_CONTEXT);
		CUDA_TRY(cudaMemsetAsync(ctx->select.ptr + table_bytes, 0, hist_bytes, s), return ASTCENC_ERR_BAD_CONTEXT);
		SelectArgs a;
		a.entries = ctx->select.as<const SelectEntry>();
		a.count = entry_count;
		a.tiles = tiles;
		a.hist = reinterpret_cast<uint32_t*>(ctx->select.ptr + table_bytes);
		a.tile_counts = reinterpret_cast<uint32_t*>(ctx->select.ptr + table_bytes + hist_bytes);
		// grid-stride launches of SELECT_WARPS warps per CTA, at least one CTA, so that every call makes the same launches
		const size_t cap = (size_t)ctx->sm_count * 16;
		auto grid = [cap](size_t warps) {
			const size_t g = (warps + SELECT_WARPS - 1) / SELECT_WARPS;
			return (unsigned int)(g == 0 ? 1 : g < cap ? g : cap);
		};
		for (int digit = 0; digit < 4; digit++) {
			astc_select_hist_kernel<<<grid(tiles), SELECT_WARPS * 32, 0, s>>>(a, digit);
		}
		astc_select_count_kernel<<<grid(tiles), SELECT_WARPS * 32, 0, s>>>(a);
		astc_select_scan_kernel<<<grid(entry_count), SELECT_WARPS * 32, 0, s>>>(a);
		astc_select_write_kernel<<<grid(tiles), SELECT_WARPS * 32, 0, s>>>(a);
		ctx->launches += SELECT_KERNELS;
		CUDA_TRY(cudaGetLastError(), return ASTCENC_ERR_BAD_CONTEXT);
		return ASTCENC_SUCCESS;
	});
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
	*records = ctx->records.ptr;
	*record_bytes = ctx->tables->bsd.record_bytes;
	*capacity_bytes = ctx->records.bytes;
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
