// CUDA-native ASTC codec: image error metrics on the device (SURVEY.md §8f rank 3).
//
// What the reference's CLI computes on the host after a -t* round trip (astcenccli_error_metrics.cpp:109-413,
// compute_error_metrics): per-channel sums of squared differences, the same with RGB scaled by the original alpha,
// and for HDR images log2 / multi-exposure (mPSNR) differences, for normal maps the angular error. Per-texel values
// use the reference's float arithmetic (its polynomial log2, astcenc_vecmathlib.h:416-441; DPPS-ordered dot products);
// the sums are double accumulators there (:31-58) - here the image is reduced in parallel (thread -> warp -> CTA ->
// a second pass in fixed order), so results are deterministic but differ from the reference's raster-order
// double sums in the last bits (tests/test_metrics.py states the tolerance).
//
// A call measures a table of image pairs (MetricEntry). Each slice of an entry owns a fixed number of virtual CTAs
// (metric_ctas: a function of the slice's texel count only, never of the GPU), so an entry's sums do not depend on the
// device, on the other entries of the call or on their order. A CTA of the launch finds its entry by binary search over
// the prefix of the entries' virtual-CTA counts (find_image) and runs the grid-stride loop over its slice as virtual CTA
// v of `ctas`. Partials go out [slice][virtual CTA] per entry, and the finish kernel walks them in that order.
//
// The per-block error map (block_error_sum) is one warp per block of the context's footprint, in astcenc_compress_image's
// block order; it compiles for the host simulation too (tests/hostsim/hostsim_metrics.cpp). A list refresh
// (astcenc_b200_compute_block_errors_device_block_lists) runs the same function at the slots of device block lists, one warp per
// slot (tests/hostsim/hostsim_map_lists.cpp). A map measures one enum astcenc_b200_block_metric (metric_block_terms): the
// squared error on astc_block_error_kernel / astc_block_error_lists_kernel, the alpha-weighted, log2 and angular errors on
// astc_block_metric_kernel<M> / astc_block_metric_lists_kernel<M>, all through block_error_sum<M>.
#pragma once
#include <vector>
#include "../../include/astcenc.h"

#define ASTC_METRIC_SUMS 17
// [0..3] squared error r,g,b,a; [4..7] alpha-scaled; [8..10] log2 error r,g,b; [11..13] mPSNR error r,g,b;
// [14] sum of angular error / pixel count; [15] worst angular error (max); [16] rgb peak of image 1 (max)
enum { MS_ERR = 0, MS_AERR = 4, MS_LOG = 8, MS_MPSNR = 11, MS_ANG_MEAN = 14, MS_ANG_WORST = 15, MS_PEAK = 16 };

#define ASTC_METRIC_THREADS 256
#define ASTC_METRIC_MAX_CTAS 592            // virtual CTAs per slice at most
#define ASTC_METRIC_FINISH_GROUPS 8         // finish kernel: entries per CTA, ASTC_METRIC_SUMS threads each
#define ASTC_METRIC_MAP_WARPS 8             // map kernel: blocks per CTA, one warp each

#if defined(ASTC_HOSTSIM)
	#define ASTC_HD static inline
#else
	#define ASTC_HD static __host__ __device__ inline
#endif

// One image pair of a metrics call: the dim_x x dim_y x dim_z intersection of two images, each with its own row pitch and slice
// stride (in texels), so that a one-entry table compares two images of different sizes as the host entry does.
struct MetricEntry {
	const void* img1;                 // the original: slices of texels of type1 (ASTCENC_TYPE_*)
	const void* img2;                 // the decoded image
	int type1, type2;
	unsigned int pitch1, pitch2;
	size_t stride1, stride2;
	unsigned int dim_x, dim_y, dim_z;
	// filled in by plan_metrics
	unsigned int ctas;                // virtual CTAs per slice
	size_t first;                     // the entry's first virtual CTA in the call; its partials start there too
	double inv_pixels;                // 1 / (dim_x * dim_y * dim_z), the product in unsigned arithmetic like the reference's :281
	unsigned int blocks_x, blocks_y;  // block grid of the map footprint
	astcenc_b200_error_metrics* metrics;   // receives the figures (device), or null: the sums are read back instead
	float* block_error;               // the per-block map (device), or null
};

// A mapped entry of a call: map warps [first, first + its block count) belong to table entry `entry`.
struct MetricMap {
	size_t first;
	unsigned int entry;
};

struct MetricArgs {
	const MetricEntry* entries;
	unsigned int count;
	const MetricMap* maps;
	unsigned int map_count;
	size_t map_blocks;                // blocks of every mapped entry
	unsigned int bx, by, bz;          // the map footprint
	int hdr, normal, components;
	int fstop_lo, fstop_hi;
	size_t ctas;                      // virtual CTAs of the call
	double* partials;                 // [virtual CTA][ASTC_METRIC_SUMS], then the sums [entry][ASTC_METRIC_SUMS]
};

// ---- host planning (no CUDA calls: the host tests run it) ----

// Virtual CTAs of one slice of texels texels: the partition the sums are defined by.
static inline unsigned int metric_ctas(size_t texels) {
	size_t ctas = (texels + ASTC_METRIC_THREADS - 1) / ASTC_METRIC_THREADS;
	return (unsigned int)(ctas < ASTC_METRIC_MAX_CTAS ? ctas : ASTC_METRIC_MAX_CTAS);
}

struct MetricPlan {
	std::vector<MetricMap> maps;
	size_t ctas = 0;                  // grid of the metrics kernel
	size_t map_blocks = 0;            // warps of the map kernel
	size_t partial_doubles = 0;       // the partials and the per-entry sums
	unsigned int finish_grid = 0;     // CTAs of the finish kernel
	unsigned int map_grid = 0;        // CTAs of the map kernel (0: no map asked for)
};

// Fills in the planned fields of `table` (its images, types, pitches, strides, dims and outputs set) for the footprint
// bx x by x bz. false: the call does not fit a launch (an entry with a map has 2^32 blocks or more, or a grid exceeds 2^31 - 1).
static inline bool plan_metrics(std::vector<MetricEntry>& table, unsigned int bx, unsigned int by, unsigned int bz, MetricPlan& p) {
	const size_t grid_max = 0x7FFFFFFF;
	p = MetricPlan();
	for (size_t i = 0; i < table.size(); i++) {
		MetricEntry& e = table[i];
		e.ctas = metric_ctas((size_t)e.dim_x * e.dim_y);
		e.first = p.ctas;
		e.inv_pixels = 1.0 / (double)(e.dim_x * e.dim_y * e.dim_z);
		e.blocks_x = (e.dim_x + bx - 1) / bx;
		e.blocks_y = (e.dim_y + by - 1) / by;
		p.ctas += (size_t)e.ctas * e.dim_z;
		if (p.ctas > grid_max) {
			return false;
		}
		if (e.block_error != nullptr) {
			const size_t blocks = (size_t)e.blocks_x * e.blocks_y * ((e.dim_z + bz - 1) / bz);
			if (blocks > 0xFFFFFFFFu) {
				return false;
			}
			p.maps.push_back({p.map_blocks, (unsigned int)i});
			p.map_blocks += blocks;
		}
	}
	const size_t map_grid = (p.map_blocks + ASTC_METRIC_MAP_WARPS - 1) / ASTC_METRIC_MAP_WARPS;
	if (map_grid > grid_max) {
		return false;
	}
	p.map_grid = (unsigned int)map_grid;
	p.finish_grid = (unsigned int)((table.size() + ASTC_METRIC_FINISH_GROUPS - 1) / ASTC_METRIC_FINISH_GROUPS);
	p.partial_doubles = (p.ctas + table.size()) * ASTC_METRIC_SUMS;
	return true;
}

// ---- map refreshes over block lists (astcenc_b200_compute_block_errors_device_block_lists) ----
// Entry j of the call owns the slots [maps[j].first, maps[j].first + lists[j].capacity): slot s of the entry refreshes map value
// indices[s] of its pair when list_slot finds it valid, and does nothing otherwise. maps[j].entry is j.
struct MetricListArgs {
	const MetricEntry* entries;
	const MetricMap* maps;            // one per entry: its first slot
	const GatherList* lists;          // one per entry
	unsigned int count;
	size_t slots;                     // the sum of the capacities: warps of the launch
	unsigned int bx, by, bz;          // the map footprint
	int components;
};

struct MetricListPlan {
	std::vector<MetricMap> maps;
	size_t slots = 0;
	unsigned int grid = 0;            // CTAs of ASTC_METRIC_MAP_WARPS warps
};

// Fills in the planned fields of `table` (images, types, pitches, strides, dims and block_error set; every entry has a map) and the
// slots of its lists, whose capacities are capacities[j], for the footprint bx x by x bz. The map values depend on the same fields
// plan_metrics fills, so a list refresh and a whole map agree bit for bit. false: the call does not fit a launch (an entry has
// 2^32 blocks or more, the sum of the capacities overflows, or the grid exceeds 2^31 - 1).
static inline bool plan_block_error_lists(std::vector<MetricEntry>& table, const unsigned int* capacities, unsigned int bx, unsigned int by, unsigned int bz,
                                          MetricListPlan& p) {
	const size_t grid_max = 0x7FFFFFFF;
	p = MetricListPlan();
	for (size_t i = 0; i < table.size(); i++) {
		MetricEntry& e = table[i];
		e.ctas = 0;
		e.first = 0;
		e.inv_pixels = 0.0;
		e.blocks_x = (e.dim_x + bx - 1) / bx;
		e.blocks_y = (e.dim_y + by - 1) / by;
		const size_t blocks = (size_t)e.blocks_x * e.blocks_y * ((e.dim_z + bz - 1) / bz);
		if (blocks > 0xFFFFFFFFu || capacities[i] > SIZE_MAX - p.slots) {
			return false;
		}
		p.maps.push_back({p.slots, (unsigned int)i});
		p.slots += capacities[i];
	}
	const size_t grid = (p.slots + ASTC_METRIC_MAP_WARPS - 1) / ASTC_METRIC_MAP_WARPS;
	if (grid > grid_max) {
		return false;
	}
	p.grid = (unsigned int)grid;
	return true;
}

// ---- per-texel values ----

// Texel t (index in texels) of an image of `type`: U8 scaled to 0..1, F16 / F32 clamped to [0, 65504] (:187, :200). One vector
// load per texel: the data is aligned to its texel (4, 8 or 16 bytes).
ASTC_FN f4 metric_texel(const void* data, int type, size_t t) {
	f4 c;
	if (type == 0) {
		const uint32_t v = ASTC_LDG(static_cast<const uint32_t*>(data) + t);
		c = mk4((float)(v & 0xFF) / 255.0f, (float)((v >> 8) & 0xFF) / 255.0f, (float)((v >> 16) & 0xFF) / 255.0f, (float)(v >> 24) / 255.0f);
	} else if (type == 1) {
		const unsigned long long v = ASTC_LDG(static_cast<const unsigned long long*>(data) + t);
		c = mk4(sf16_to_float((uint16_t)v), sf16_to_float((uint16_t)(v >> 16)), sf16_to_float((uint16_t)(v >> 32)), sf16_to_float((uint16_t)(v >> 48)));
	} else {
#if defined(ASTC_HOSTSIM)
		const float* p = static_cast<const float*>(data) + 4 * t;
		c = mk4(p[0], p[1], p[2], p[3]);
#else
		const float4 v = __ldg(static_cast<const float4*>(data) + t);
		c = mk4(v.x, v.y, v.z, v.w);
#endif
	}
	if (type != 0) {
		c.x = fminf(fmaxf(c.x, 0.0f), 65504.0f);
		c.y = fminf(fmaxf(c.y, 0.0f), 65504.0f);
		c.z = fminf(fmaxf(c.z, 0.0f), 65504.0f);
		c.w = fminf(fmaxf(c.w, 0.0f), 65504.0f);
	}
	return c;
}

// The channels input_components counts (compute_error_metrics :283-284): 1 RGB, 2 BA, 3 RGB, 4 RGBA.
ASTC_HD int metric_component_mask(int input_components) {
	return input_components == 2 ? 0x0C : input_components == 4 ? 0x0F : 0x07;
}

// the reference's approximate log2 (astcenc_vecmathlib.h:416-441), unfused
ASTC_FN float metric_log2(float x) {
	int i = (int)ASTC_F2U(x);
	float e = (float)(((i & 0x7F800000) >> 23) - 127);
	float m = ASTC_U2F((uint32_t)((i & 0x007FFFFF) | 0x3F800000));
	float p = 0.0596515482674574969533f;
	p = p * m + -0.465725644288844778798f;
	p = p * m + 1.48116647521213171641f;
	p = p * m + -2.52074962577807006663f;
	p = p * m + 2.8882704548164776201f;
	p = p * (m - 1.0f);
	return p + e;
}

// (c - 0.5) * 2, normalize_safe(xyz, unit3) (:269-275; astcenc_vecmathlib.h:362-371), dot in DPPS order; w is 0
ASTC_FN f4 metric_normal(f4 c) {
	float x = (c.x - 0.5f) * 2.0f, y = (c.y - 0.5f) * 2.0f, z = (c.z - 0.5f) * 2.0f;
	float len = (x * x + y * y) + (z * z + 0.0f);
	if (len != 0.0f) {
		float s = sqrtf(len);
		return mk4(x / s, y / s, z / s, 0.0f);
	}
	float u = 0.57735026918962576451f;      // unit3()
	return mk4(u, u, u, 0.0f);
}

// The angle in degrees between the normals of the RGB of c1 and c2 (:276-281): the float dot product in DPPS order clamped to
// [-1, 1] (a NaN dot gives -1: 180 degrees), acos in double. The per-texel term of mean_angular_error and worst_angular_error.
ASTC_FN double metric_angle(f4 c1, f4 c2) {
	f4 n1 = metric_normal(c1);
	f4 n2 = metric_normal(c2);
	float d = (n1.x * n2.x + n1.y * n2.y) + (n1.z * n2.z + 0.0f);
	d = fminf(fmaxf(d, -1.0f), 1.0f);
	float rad_to_degrees = 180.0f / 3.14159265358979323846f;
	return acos((double)d) * (double)rad_to_degrees;
}

// ---- the per-block error map ----

// How a map of metric M combines its terms, within a lane and across lanes: the largest for WORST_ANGULAR_ERROR (fmax does not
// depend on the order), the double sum for every other metric.
template <int M>
ASTC_FN double metric_combine(double acc, double term) {
	return M == ASTCENC_B200_BLOCK_WORST_ANGULAR_ERROR ? fmax(acc, term) : acc + term;
}

// The terms of one texel of a map of metric M (enum astcenc_b200_block_metric) over the channels in `mask`, c1 the original and
// c2 the decoded texel, combined into acc (metric_combine) in channel order. Each term but the angle is a float square of float
// values, combined in double:
//   SQUARED_ERROR         (c1 - c2)^2 per channel, the MS_ERR terms of the sums
//   ALPHA_WEIGHTED_ERROR  ((c1 - c2) * c1.w)^2 per RGB channel and (c1.w - c2.w)^2 for alpha, the MS_AERR terms
//   LOG2_ERROR            (log2(c1) - log2(c2))^2 per RGB channel, the MS_LOG terms
//   ANGULAR_ERROR and WORST_ANGULAR_ERROR  metric_angle of the RGB whatever the mask, the MS_ANG_MEAN / MS_ANG_WORST term
template <int M>
ASTC_FN void metric_block_terms(const f4& c1, const f4& c2, int mask, double& acc) {
	if (M == ASTCENC_B200_BLOCK_ANGULAR_ERROR || M == ASTCENC_B200_BLOCK_WORST_ANGULAR_ERROR) {
		acc = metric_combine<M>(acc, metric_angle(c1, c2));
		return;
	}
	if (M == ASTCENC_B200_BLOCK_LOG2_ERROR) {
		const float o[3] = {c1.x, c1.y, c1.z}, q[3] = {c2.x, c2.y, c2.z};
		for (int k = 0; k < 3; k++) {
			if (mask & (1 << k)) {
				const float l = metric_log2(o[k]) - metric_log2(q[k]);
				acc = metric_combine<M>(acc, (double)(l * l));
			}
		}
		return;
	}
	const float d[4] = {c1.x - c2.x, c1.y - c2.y, c1.z - c2.z, c1.w - c2.w};
	for (int k = 0; k < 4; k++) {
		if (mask & (1 << k)) {
			const float v = M == ASTCENC_B200_BLOCK_ALPHA_WEIGHTED_ERROR && k < 3 ? d[k] * c1.w : d[k];
			acc = metric_combine<M>(acc, (double)(v * v));
		}
	}
}

// Map block `index` of entry e (astcenc_compress_image's block order for the footprint bx x by x bz; a 2D footprint's index
// counts the slices of a texture array), by `lanes` lanes of one warp, against the decoded texels `decoded` gives: the terms of
// metric M (metric_block_terms) of the channels in `mask` over the block's texels inside the image, combined in double
// (metric_combine: a sum, or the largest for WORST_ANGULAR_ERROR). decoded(t, x, y, z) is the decoded texel of footprint texel t
// at image position (x, y, z). Lane l takes texels l, l + lanes, ... in footprint order, then the lanes are combined in a fixed
// xor-shuffle order. Every lane returns the value. So a value depends on where the decoded texels live only through what
// `decoded` returns.
template <int M, typename Decoded>
ASTC_FN double block_error_sum_of(const MetricEntry& e, unsigned int bx, unsigned int by, unsigned int bz, uint32_t index, int mask, int lane, int lanes,
                                  const Decoded& decoded) {
	double acc = 0.0;
	for (unsigned int t = (unsigned int)lane; t < bx * by * bz; t += (unsigned int)lanes) {
		unsigned int tx, ty, tz, x, y, z;
		footprint_texel(e.blocks_x, e.blocks_y, bx, by, bz, index, t, tx, ty, tz, x, y, z);
		if (x >= e.dim_x || y >= e.dim_y || z >= e.dim_z) {
			continue;
		}
		const f4 c1 = metric_texel(e.img1, e.type1, z * e.stride1 + (size_t)e.pitch1 * y + x);
		const f4 c2 = decoded(t, x, y, z);
		metric_block_terms<M>(c1, c2, mask, acc);
	}
#if !defined(ASTC_ONE_LANE)
	for (int o = lanes / 2; o > 0; o >>= 1) {
		acc = metric_combine<M>(acc, __shfl_xor_sync(0xffffffffu, acc, o));
	}
#endif
	return acc;
}

// block_error_sum_of against the pair's decoded image (img2).
template <int M = ASTCENC_B200_BLOCK_SQUARED_ERROR>
ASTC_FN double block_error_sum(const MetricEntry& e, unsigned int bx, unsigned int by, unsigned int bz, uint32_t index, int mask, int lane, int lanes) {
	return block_error_sum_of<M>(e, bx, by, bz, index, mask, lane, lanes, [&](unsigned int, unsigned int x, unsigned int y, unsigned int z) {
		return metric_texel(e.img2, e.type2, z * e.stride2 + (size_t)e.pitch2 * y + x);
	});
}

// Slot w < a.slots of a list refresh, by `lanes` lanes of one warp: block_error_sum<M> of the listed block into its map value. An
// entry with capacity 0 owns no slot, and a slot past the count or out of range writes nothing.
template <int M = ASTCENC_B200_BLOCK_SQUARED_ERROR>
ASTC_FN void block_error_list_slot(const MetricListArgs& a, size_t w, int lane, int lanes) {
	const MetricMap& m = a.maps[find_image(a.maps, a.count, w)];
	const uint32_t index = list_slot(a.lists[m.entry], w - m.first);
	if (index == GATHER_INVALID) {
		return;      // (the whole warp)
	}
	const MetricEntry& e = a.entries[m.entry];
	const double s = block_error_sum<M>(e, a.bx, a.by, a.bz, index, metric_component_mask(a.components), lane, lanes);
	if (lane == 0) {
		e.block_error[index] = (float)s;
	}
}

// ---- the closing arithmetic of compute_error_metrics (:285-411) ----

// The figures of one entry from its 17 sums; `pixels` = (double)(dim_x * dim_y * dim_z), the product in unsigned arithmetic.
// Runs on the device (the finish kernel) and on the host (astcenc_b200_compute_error_metrics).
ASTC_HD void metric_close(const double* sums, int hdr, int normal, int input_components, int fstop_lo, int fstop_hi, double pixels,
                          astcenc_b200_error_metrics* out) {
	const int mask = metric_component_mask(input_components);
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
	memset(out, 0, sizeof(*out));
	out->psnr = psnr;
	out->alpha_psnr = psnr;
	if (mask & 8) {
		out->alpha_psnr = alpha_num == 0.0 ? 999.0 : 10.0 * log10(samples / alpha_num);
		double rgb_num = sums[MS_ERR + 0] + sums[MS_ERR + 1] + sums[MS_ERR + 2];
		rgb_psnr = rgb_num == 0.0 ? 999.0 : 10.0 * log10(pixels * 3.0 / rgb_num);
	}
	out->rgb_psnr = rgb_psnr;
	out->rgb_peak = sums[MS_PEAK];
	if (hdr) {
		out->peak_psnr = rgb_psnr + 20.0 * log10(sums[MS_PEAK]);
		out->mpsnr = mpsnr_num == 0.0 ? 999.0 : 10.0 * log10(mpsnr_denom / mpsnr_num);
		out->log_rmse = sqrt(log_num / pixels);
	}
	if (normal) {
		out->mean_angular_error = sums[MS_ANG_MEAN];
		out->worst_angular_error = sums[MS_ANG_WORST];
	}
	for (int c = 0; c < 4; c++) {
		out->sum_squared_error[c] = sums[MS_ERR + c];
	}
}

#if !defined(ASTC_HOSTSIM)
// mpsnr_operator / mpsnr_sumdiff (astcenccli_error_metrics.cpp:69-107)
static __device__ __forceinline__ float metric_mpsnr_operator(float val, int fstop) {
	float scale = __uint_as_float(0x3f800000u + ((unsigned int)fstop << 23));
	val = powf(val * scale, 1.0f / 2.2f);
	return fminf(fmaxf(val * 255.0f, 0.0f), 255.0f);
}
static __device__ __forceinline__ float metric_mpsnr_sumdiff(float v1, float v2, int lo, int hi) {
	float summa = 0.0f;
	for (int i = lo; i <= hi; i++) {
		float d = metric_mpsnr_operator(v1, i) - metric_mpsnr_operator(v2, i);
		summa += d * d;
	}
	return summa;
}

// CTA b of the launch is virtual CTA b - first of its entry: slice z, CTA v of that slice's `ctas`.
__global__ void __launch_bounds__(ASTC_METRIC_THREADS)
astc_error_metrics_kernel(const __grid_constant__ MetricArgs a) {
	const MetricEntry& e = a.entries[find_image(a.entries, a.count, blockIdx.x)];
	const unsigned int ctas = e.ctas;
	const unsigned int vz = (unsigned int)(blockIdx.x - e.first);
	const unsigned int z = vz / ctas, v = vz - z * ctas;
	const unsigned int dim_x = e.dim_x, pitch1 = e.pitch1, pitch2 = e.pitch2;
	const int type1 = e.type1, type2 = e.type2;
	// the slice: 4 << type bytes per texel
	const void* img1 = static_cast<const uint8_t*>(e.img1) + ((z * e.stride1) << (2 + type1));
	const void* img2 = static_cast<const uint8_t*>(e.img2) + ((z * e.stride2) << (2 + type2));
	const double inv_pixels = e.inv_pixels;
	double acc[ASTC_METRIC_SUMS];
	for (int k = 0; k < ASTC_METRIC_SUMS; k++) {
		acc[k] = 0.0;
	}
	size_t n = (size_t)dim_x * e.dim_y;
	for (size_t p = (size_t)v * blockDim.x + threadIdx.x; p < n; p += (size_t)ctas * blockDim.x) {
		unsigned int y = (unsigned int)(p / dim_x);
		unsigned int x = (unsigned int)(p - (size_t)y * dim_x);
		f4 c1 = metric_texel(img1, type1, (size_t)pitch1 * y + x);
		f4 c2 = metric_texel(img2, type2, (size_t)pitch2 * y + x);
		acc[MS_PEAK] = fmax(fmax(fmax((double)c1.x, (double)c1.y), (double)c1.z), acc[MS_PEAK]);
		float dx = c1.x - c2.x, dy = c1.y - c2.y, dz = c1.z - c2.z, dw = c1.w - c2.w;
		acc[MS_ERR + 0] += (double)(dx * dx);
		acc[MS_ERR + 1] += (double)(dy * dy);
		acc[MS_ERR + 2] += (double)(dz * dz);
		acc[MS_ERR + 3] += (double)(dw * dw);
		float ax = dx * c1.w, ay = dy * c1.w, az = dz * c1.w;
		acc[MS_AERR + 0] += (double)(ax * ax);
		acc[MS_AERR + 1] += (double)(ay * ay);
		acc[MS_AERR + 2] += (double)(az * az);
		acc[MS_AERR + 3] += (double)(dw * dw);
		if (a.hdr) {
			float lx = metric_log2(c1.x) - metric_log2(c2.x);
			float ly = metric_log2(c1.y) - metric_log2(c2.y);
			float lz = metric_log2(c1.z) - metric_log2(c2.z);
			acc[MS_LOG + 0] += (double)(lx * lx);
			acc[MS_LOG + 1] += (double)(ly * ly);
			acc[MS_LOG + 2] += (double)(lz * lz);
			acc[MS_MPSNR + 0] += (double)metric_mpsnr_sumdiff(c1.x, c2.x, a.fstop_lo, a.fstop_hi);
			acc[MS_MPSNR + 1] += (double)metric_mpsnr_sumdiff(c1.y, c2.y, a.fstop_lo, a.fstop_hi);
			acc[MS_MPSNR + 2] += (double)metric_mpsnr_sumdiff(c1.z, c2.z, a.fstop_lo, a.fstop_hi);
		}
		if (a.normal) {
			double deg = metric_angle(c1, c2);
			acc[MS_ANG_MEAN] += deg * inv_pixels;
			acc[MS_ANG_WORST] = fmax(acc[MS_ANG_WORST], deg);
		}
	}
	// thread -> warp -> CTA, fixed order
	__shared__ double red[ASTC_METRIC_THREADS / 32][ASTC_METRIC_SUMS];
	for (int k = 0; k < ASTC_METRIC_SUMS; k++) {
		double v = acc[k];
		bool is_max = k >= MS_ANG_WORST;
		for (int o = 16; o > 0; o >>= 1) {
			double t = __shfl_xor_sync(0xffffffffu, v, o);
			v = is_max ? fmax(v, t) : v + t;
		}
		if ((threadIdx.x & 31) == 0) {
			red[threadIdx.x >> 5][k] = v;
		}
	}
	__syncthreads();
	if (threadIdx.x < ASTC_METRIC_SUMS) {
		int k = threadIdx.x;
		bool is_max = k >= MS_ANG_WORST;
		double v = red[0][k];
		for (unsigned int wi = 1; wi < blockDim.x / 32; wi++) {
			v = is_max ? fmax(v, red[wi][k]) : v + red[wi][k];
		}
		a.partials[(size_t)blockIdx.x * ASTC_METRIC_SUMS + k] = v;
	}
}

// Second pass: one group of ASTC_METRIC_SUMS threads per entry; thread k walks the entry's partials of sum k in order
// ([slice][virtual CTA]) into the entry's sums, and the group's first thread closes them into the entry's figures.
__global__ void __launch_bounds__(ASTC_METRIC_FINISH_GROUPS * ASTC_METRIC_SUMS)
astc_error_metrics_finish_kernel(const __grid_constant__ MetricArgs a) {
	__shared__ double sums[ASTC_METRIC_FINISH_GROUPS][ASTC_METRIC_SUMS];
	const unsigned int g = threadIdx.x / ASTC_METRIC_SUMS, k = threadIdx.x - g * ASTC_METRIC_SUMS;
	const unsigned int j = blockIdx.x * ASTC_METRIC_FINISH_GROUPS + g;
	if (j < a.count) {
		const MetricEntry& e = a.entries[j];
		const size_t n = (size_t)e.ctas * e.dim_z;
		const double* p = a.partials + e.first * ASTC_METRIC_SUMS + k;
		bool is_max = k >= MS_ANG_WORST;
		double v = p[0];
		for (size_t c = 1; c < n; c++) {
			double t = p[c * ASTC_METRIC_SUMS];
			v = is_max ? fmax(v, t) : v + t;
		}
		sums[g][k] = v;
		a.partials[(a.ctas + j) * ASTC_METRIC_SUMS + k] = v;
	}
	__syncthreads();
	if (j < a.count && k == 0 && a.entries[j].metrics != nullptr) {
		const MetricEntry& e = a.entries[j];
		astcenc_b200_error_metrics m;
		metric_close(sums[g], a.hdr, a.normal, a.components, a.fstop_lo, a.fstop_hi, (double)(e.dim_x * e.dim_y * e.dim_z), &m);
		*e.metrics = m;
	}
}

// The map of metric M: warp w of the launch is block w - first of its mapped entry.
template <int M>
static __device__ __forceinline__ void block_map_warp(const MetricArgs& a) {
	const size_t w = (size_t)blockIdx.x * ASTC_METRIC_MAP_WARPS + (threadIdx.x >> 5);
	if (w >= a.map_blocks) {
		return;      // (the whole warp)
	}
	const MetricMap& m = a.maps[find_image(a.maps, a.map_count, w)];
	const MetricEntry& e = a.entries[m.entry];
	const uint32_t index = (uint32_t)(w - m.first);      // (a mapped entry has fewer than 2^32 blocks)
	const double s = block_error_sum<M>(e, a.bx, a.by, a.bz, index, metric_component_mask(a.components), threadIdx.x & 31, ASTC_WARP);
	if ((threadIdx.x & 31) == 0) {
		e.block_error[index] = (float)s;
	}
}

// The squared-error map (ASTCENC_B200_BLOCK_SQUARED_ERROR).
__global__ void __launch_bounds__(ASTC_METRIC_MAP_WARPS * 32)
astc_block_error_kernel(const __grid_constant__ MetricArgs a) {
	block_map_warp<ASTCENC_B200_BLOCK_SQUARED_ERROR>(a);
}

// The maps of the other metrics: one instantiation each (ALPHA_WEIGHTED_ERROR, LOG2_ERROR, ANGULAR_ERROR, WORST_ANGULAR_ERROR).
template <int M>
__global__ void __launch_bounds__(ASTC_METRIC_MAP_WARPS * 32)
astc_block_metric_kernel(const __grid_constant__ MetricArgs a) {
	block_map_warp<M>(a);
}

// A list refresh of squared-error maps: warp w of the launch is slot w of the call.
__global__ void __launch_bounds__(ASTC_METRIC_MAP_WARPS * 32)
astc_block_error_lists_kernel(const __grid_constant__ MetricListArgs a) {
	const size_t w = (size_t)blockIdx.x * ASTC_METRIC_MAP_WARPS + (threadIdx.x >> 5);
	if (w < a.slots) {
		block_error_list_slot(a, w, threadIdx.x & 31, ASTC_WARP);
	}
}

// A list refresh of maps of metric M (every metric but SQUARED_ERROR).
template <int M>
__global__ void __launch_bounds__(ASTC_METRIC_MAP_WARPS * 32)
astc_block_metric_lists_kernel(const __grid_constant__ MetricListArgs a) {
	const size_t w = (size_t)blockIdx.x * ASTC_METRIC_MAP_WARPS + (threadIdx.x >> 5);
	if (w < a.slots) {
		block_error_list_slot<M>(a, w, threadIdx.x & 31, ASTC_WARP);
	}
}
#endif
