// TEST TOOL (not a product path): the device source's endpoint packers on the GPU, one call over an array of vectors
// (astc-encoder_b200/Makefile target `devunit`, built with the product's NVFLAGS into libastc_devunit.so).
//   PACK_SERIAL    pack_color_endpoints: 32 different vectors per warp, one per lane, as the multi-partition path runs it
//   PACK_COOP      pack_rgb_endpoints_coop: one vector per warp, all lanes converged, as pack_work_endpoints_t runs it
//   PACK_COOP_INL  pack_rgb_endpoints_coop_t<true>: the same, inlined
//   PACK_HDR       pack_hdr_endpoints: one vector per warp, all lanes converged
// The shared window holds the SmemHdr, then (staged) the 17 x 512-byte color_unquant_to_uquant at cq_smem_off, then one
// 32 x 8-byte output slot per warp. The packers write into shared memory like the product; the slots start as the
// caller's bytes (a sentinel) and go back as they end, so a byte a format does not define must come back unchanged.
// A returned format that differs between the lanes of the warp comes back as 0xFF.
#include "../../astc-encoder_b200/csrc/astc_dev_core.cuh"
#include "../../astc-encoder_b200/csrc/astc_host_pack.h"
#include "pack_endpoints_args.h"
#include <cuda_runtime.h>
#include <cstdio>

#define CQ_BYTES ((int)sizeof(((DevConstTables*)0)->color_unquant_to_uquant))
#define WARPS_PER_CTA 4
#define SLOT_BASE (ASTC_SMEM_HDR + CQ_BYTES)

__global__ void __launch_bounds__(32 * WARPS_PER_CTA) pack_endpoints_kernel(int variant, int staged, unsigned int n, const float* __restrict__ colors,
                                                                           const int* __restrict__ fmt_quant, uint8_t* out, uint8_t* out_format) {
	const int lane = (int)(threadIdx.x & 31u);
	const int warp = (int)(threadIdx.x >> 5);
	SmemHdr* hdr = reinterpret_cast<SmemHdr*>(astc_smem);
	if (threadIdx.x == 0) {
		hdr->dec_smem_off = 0;
		hdr->cq_smem_off = staged ? ASTC_SMEM_HDR : 0;
	}
	if (staged) {
		const uint8_t* src = &g_astc_ct->color_unquant_to_uquant[0][0];
		for (int i = (int)threadIdx.x; i < CQ_BYTES; i += (int)blockDim.x) {
			astc_smem[ASTC_SMEM_HDR + i] = src[i];
		}
	}
	__syncthreads();
	uint8_t* slots = astc_smem + SLOT_BASE + warp * 32 * 8;
	const unsigned int gwarp = blockIdx.x * WARPS_PER_CTA + (unsigned int)warp;
	const unsigned int nwarps = gridDim.x * WARPS_PER_CTA;
	if (variant == PACK_SERIAL) {
		for (unsigned int base = gwarp * 32u; base < n; base += nwarps * 32u) {
			const unsigned int i = base + (unsigned int)lane;
			uint8_t* o = slots + lane * 8;
			if (i < n) {
				for (int b = 0; b < 8; b++) {
					o[b] = out[8 * (size_t)i + b];
				}
				const float* c = colors + 16 * (size_t)i;
				f4 c0 = mk4(c[0], c[1], c[2], c[3]), c1 = mk4(c[4], c[5], c[6], c[7]);
				f4 rgbs = mk4(c[8], c[9], c[10], c[11]), rgbo = mk4(c[12], c[13], c[14], c[15]);
				out_format[i] = pack_color_endpoints(c0, c1, rgbs, rgbo, fmt_quant[2 * i], o, fmt_quant[2 * i + 1]);
				for (int b = 0; b < 8; b++) {
					out[8 * (size_t)i + b] = o[b];
				}
			}
			__syncwarp();
		}
		return;
	}
	for (unsigned int i = gwarp; i < n; i += nwarps) {
		if (lane < 8) {
			slots[lane] = out[8 * (size_t)i + lane];
		}
		__syncwarp();
		const float* c = colors + 16 * (size_t)i;
		f4 c0 = mk4(c[0], c[1], c[2], c[3]), c1 = mk4(c[4], c[5], c[6], c[7]), rgbo = mk4(c[12], c[13], c[14], c[15]);
		const int format = fmt_quant[2 * i], q = fmt_quant[2 * i + 1];
		uint8_t f;
		if (variant == PACK_COOP) {
			f = pack_rgb_endpoints_coop(lane, c0, c1, format, slots, q);
		} else if (variant == PACK_COOP_INL) {
			f = pack_rgb_endpoints_coop_t<true>(lane, c0, c1, format, slots, q);
		} else {
			f = pack_hdr_endpoints(lane, c0, c1, rgbo, format, slots, q);
		}
		const bool uniform = __all_sync(0xffffffffu, __shfl_sync(0xffffffffu, (int)f, 0) == (int)f);
		__syncwarp();
		if (lane < 8) {
			out[8 * (size_t)i + lane] = slots[lane];
		}
		if (lane == 0) {
			out_format[i] = uniform ? f : (uint8_t)0xFF;
		}
		__syncwarp();
	}
}

// 0 = done, 1 = refused inputs (nothing ran), 2 = a CUDA call failed (its error string in devunit_last_error())
static char g_last_error[256];
#define DU_EXPORT extern "C" __attribute__((visibility("default")))
DU_EXPORT const char* devunit_last_error() { return g_last_error; }

#define DU_CHECK(call)                                                                                 \
	do {                                                                                               \
		cudaError_t e_ = (call);                                                                       \
		if (e_ != cudaSuccess) {                                                                       \
			snprintf(g_last_error, sizeof(g_last_error), "%s: %s", #call, cudaGetErrorString(e_));     \
			rc = 2;                                                                                    \
			goto done;                                                                                 \
		}                                                                                              \
	} while (0)

DU_EXPORT int devunit_pack_endpoints(int variant, int staged, unsigned int n, const float* colors, const int* fmt_quant, uint8_t* out, uint8_t* out_format) {
	g_last_error[0] = 0;
	if (pack_args_check(variant, n, colors, fmt_quant) != 0 || (n != 0 && (out == nullptr || out_format == nullptr))) {
		return 1;
	}
	if (n == 0) {
		return 0;
	}
	int rc = 0;
	DevConstTables* h_ct = new DevConstTables;
	DevConstTables* d_ct = nullptr;
	float* d_colors = nullptr;
	int* d_fq = nullptr;
	uint8_t* d_out = nullptr;
	uint8_t* d_fmt = nullptr;
	const unsigned int warps = variant == PACK_SERIAL ? (n + 31u) / 32u : n;
	const unsigned int ctas = (warps + WARPS_PER_CTA - 1) / WARPS_PER_CTA < 4096u ? (warps + WARPS_PER_CTA - 1) / WARPS_PER_CTA : 4096u;
	const size_t smem = SLOT_BASE + WARPS_PER_CTA * 32 * 8;
	astc_host::fill_dev_const_tables(*h_ct);
	DU_CHECK(cudaMalloc(&d_ct, sizeof(DevConstTables)));
	DU_CHECK(cudaMemcpy(d_ct, h_ct, sizeof(DevConstTables), cudaMemcpyHostToDevice));
	DU_CHECK(cudaMemcpyToSymbol(g_astc_ct, &d_ct, sizeof(d_ct)));
	DU_CHECK(cudaMalloc(&d_colors, 16 * sizeof(float) * (size_t)n));
	DU_CHECK(cudaMalloc(&d_fq, 2 * sizeof(int) * (size_t)n));
	DU_CHECK(cudaMalloc(&d_out, 8 * (size_t)n));
	DU_CHECK(cudaMalloc(&d_fmt, (size_t)n));
	DU_CHECK(cudaMemcpy(d_colors, colors, 16 * sizeof(float) * (size_t)n, cudaMemcpyHostToDevice));
	DU_CHECK(cudaMemcpy(d_fq, fmt_quant, 2 * sizeof(int) * (size_t)n, cudaMemcpyHostToDevice));
	DU_CHECK(cudaMemcpy(d_out, out, 8 * (size_t)n, cudaMemcpyHostToDevice));
	DU_CHECK(cudaMemset(d_fmt, 0xFE, (size_t)n));
	pack_endpoints_kernel<<<ctas, 32 * WARPS_PER_CTA, smem>>>(variant, staged, n, d_colors, d_fq, d_out, d_fmt);
	DU_CHECK(cudaGetLastError());
	DU_CHECK(cudaDeviceSynchronize());
	DU_CHECK(cudaMemcpy(out, d_out, 8 * (size_t)n, cudaMemcpyDeviceToHost));
	DU_CHECK(cudaMemcpy(out_format, d_fmt, (size_t)n, cudaMemcpyDeviceToHost));
done:
	cudaFree(d_fmt);
	cudaFree(d_out);
	cudaFree(d_fq);
	cudaFree(d_colors);
	cudaFree(d_ct);
	delete h_ct;
	return rc;
}
