// CUDA-native ASTC: totals of per-block error maps, and the selection weights they gate (astcenc_b200_total_block_maps).
//
// An entry's total is a double sum in an order fixed by its block_count alone, the metrics call's scheme: the entry owns
// ctas = metric_ctas(block_count) virtual CTAs, and virtual CTA v takes the runs of ASTC_METRIC_THREADS values
// v, v + ctas, v + 2 * ctas, ... Each virtual CTA is one warp of TOTAL_SLOTS slots; slot s adds, from 0.0 and in index order,
// its CTA's values i with i % TOTAL_SLOTS == s (so the lanes of a warp read consecutive values). The CTA's partial is
//   ((0.0 + slot 0) + slot 1) + ... + slot 31,
// written at the entry's first virtual CTA + v, and the finish walks the entry's partials in order from 0.0. A slot's sum and
// the walk over the slots do not depend on how many lanes share the work (lane l of `lanes` takes slots l, l + lanes, ...;
// each round's slot sums are added in slot order through shuffles), so one simulated lane, 32 and the device give the same bits.
// The entry's total never depends on the GPU, on the other entries of the call or on their order; an entry with no blocks owns
// no virtual CTA and totals 0.
//
// The finish (one thread per entry) writes the total and the weight: 0 unless total > limit and total > 0 (a NaN total gives 0),
// otherwise 1 (ASTCENC_B200_WEIGHT_ONE) or (float)(1.0 / total) (ASTCENC_B200_WEIGHT_INVERSE_TOTAL).
//
// Launches, whatever the number of entries: the partial kernel (one warp per virtual CTA of the call, find_image over the
// entries' first virtual CTAs) and the finish kernel. Both bodies take (lane, lanes) or none and compile for the host
// simulation (tests/hostsim/hostsim_map_totals.cpp).
#pragma once
#include <vector>

#define TOTAL_SLOTS 32                // slots of a virtual CTA (one warp)
#define TOTAL_WARPS 8                 // partial kernel: virtual CTAs per CTA
#define TOTAL_FINISH_THREADS 256      // finish kernel: entries per CTA
#define TOTAL_KERNELS 2               // kernel launches per call

// One entry of a totals call, as the device reads it.
struct TotalEntry {
	const float* map;
	double* total;                    // or null
	float* weight;                    // or null
	double limit;
	unsigned int block_count;
	unsigned int ctas;                // metric_ctas(block_count)
	size_t first;                     // the entry's first virtual CTA in the call; its partials start there too
};

struct TotalArgs {
	const TotalEntry* entries;
	unsigned int count;
	int rule;                         // enum astcenc_b200_weight_rule
	size_t ctas;                      // virtual CTAs of the call
	double* partials;                 // [virtual CTA]
};

// ---- host planning (no CUDA calls) ----
// Fills in the virtual CTAs and first virtual CTA of every entry and the call's virtual CTAs. false: the call does not fit a
// launch (more than 2^31 - 1 virtual CTAs, the metrics call's limit).
static inline bool plan_map_totals(std::vector<TotalEntry>& table, size_t& ctas) {
	ctas = 0;
	for (TotalEntry& e : table) {
		e.ctas = metric_ctas(e.block_count);
		e.first = ctas;
		ctas += e.ctas;
		if (ctas > 0x7FFFFFFF) {
			return false;
		}
	}
	return true;
}

// Lane l's value, for every lane.
#if defined(ASTC_ONE_LANE)
ASTC_FN double total_lane_value(double v, int l) { (void)l; return v; }
#else
ASTC_FN double total_lane_value(double v, int l) { return __shfl_sync(0xffffffffu, v, l); }
#endif

// ---- per virtual CTA / per entry ----
// The partial of virtual CTA v of entry e, by `lanes` lanes of one warp (a divisor of TOTAL_SLOTS); every lane returns it.
ASTC_FN double map_total_partial(const TotalEntry& e, unsigned int v, int lane, int lanes) {
	const size_t n = e.block_count, step = (size_t)e.ctas * ASTC_METRIC_THREADS;
	double acc = 0.0;
	for (int s0 = 0; s0 < TOTAL_SLOTS; s0 += lanes) {
		const size_t s = (size_t)(s0 + lane);
		double slot = 0.0;
		for (size_t c = (size_t)v * ASTC_METRIC_THREADS; c < n; c += step) {
			for (size_t i = c + s; i < c + ASTC_METRIC_THREADS && i < n; i += TOTAL_SLOTS) {
				slot += (double)ASTC_LDG(e.map + i);
			}
		}
		for (int l = 0; l < lanes; l++) {
			acc += total_lane_value(slot, l);
		}
	}
	return acc;
}

// Entry e's total from its partials (partials: the call's), and its weight under `rule`, into the outputs it has.
ASTC_FN void map_total_finish(const TotalEntry& e, const double* partials, int rule) {
	double t = 0.0;
	for (unsigned int v = 0; v < e.ctas; v++) {
		t += partials[e.first + v];
	}
	if (e.total != nullptr) {
		*e.total = t;
	}
	if (e.weight != nullptr) {
		*e.weight = t > e.limit && t > 0.0 ? (rule == ASTCENC_B200_WEIGHT_INVERSE_TOTAL ? (float)(1.0 / t) : 1.0f) : 0.0f;
	}
}

#if !defined(ASTC_HOSTSIM)
// Warp w of the launch is virtual CTA w of the call. (Entries with no blocks share their first virtual CTA with the next entry;
// find_image returns the last entry whose first is at or before w, the one that owns it.)
__global__ void __launch_bounds__(TOTAL_WARPS * 32)
astc_map_total_partial_kernel(const __grid_constant__ TotalArgs a) {
	const size_t w = (size_t)blockIdx.x * TOTAL_WARPS + (threadIdx.x >> 5);
	if (w >= a.ctas) {
		return;      // (the whole warp)
	}
	const int lane = threadIdx.x & 31;
	const TotalEntry& e = a.entries[find_image(a.entries, a.count, w)];
	const double s = map_total_partial(e, (unsigned int)(w - e.first), lane, 32);
	if (lane == 0) {
		a.partials[w] = s;
	}
}

// Thread j of the launch finishes entry j.
__global__ void __launch_bounds__(TOTAL_FINISH_THREADS)
astc_map_total_finish_kernel(const __grid_constant__ TotalArgs a) {
	const size_t j = (size_t)blockIdx.x * TOTAL_FINISH_THREADS + threadIdx.x;
	if (j < a.count) {
		map_total_finish(a.entries[j], a.partials, a.rule);
	}
}
#endif
