// CUDA-native ASTC: packing of block-list tables (astcenc_b200_compress_device_block_lists_packed,
// astcenc_b200_refine_device_block_lists_packed).
//
// The host plans a packed call as an unpacked one (every entry of capacity > 0 in the table, in call order) and sizes its staging
// row from min(budget, sum of capacities). Once the table is on the device, one launch of pack_lists gives entry j the packed
// position of its first listed slot, first[j] = v_0 + ... + v_(j-1) with v_i = min(*count_i, capacity_i), and writes the packed
// total T = min(sum of v, budget) into the sentinel after the table (images[count].first) and the excess of the sum over the
// budget, saturated to 32 bits, into *overflow. Only the count words are read, never the indices.
//
// The walk takes tiles of lanes * PACK_PER_LANE entries: lane l sums the v of its PACK_PER_LANE consecutive entries, a shuffle
// scan over the lanes gives each lane the sum before its own, and a 64-bit running sum carries from tile to tile. Every sum is
// an integer sum, so one simulated lane, 32 and the device write the same values.
#pragma once

#define PACK_PER_LANE 8               // entries per lane of a tile

// The inclusive sum of v over lanes 0..lane, and lane l's value, for every lane.
#if defined(ASTC_ONE_LANE)
ASTC_FN unsigned long long pack_inclusive_sum(unsigned long long v, int lane, int lanes) { (void)lane; (void)lanes; return v; }
ASTC_FN unsigned long long pack_lane_value(unsigned long long v, int l) { (void)l; return v; }
#else
ASTC_FN unsigned long long pack_inclusive_sum(unsigned long long v, int lane, int lanes) {
	for (int d = 1; d < lanes; d *= 2) {
		const unsigned long long u = __shfl_up_sync(0xffffffffu, v, d);
		if (lane >= d) {
			v += u;
		}
	}
	return v;
}
ASTC_FN unsigned long long pack_lane_value(unsigned long long v, int l) { return __shfl_sync(0xffffffffu, v, l); }
#endif

// The packed firsts of the count entries of images / lists (a staging table whose entries all have capacity > 0), the sentinel
// images[count].first = T and *overflow (when not null), by `lanes` lanes of one warp (1, or 32 with the warp's shuffles).
ASTC_FN void pack_lists(GatherImage* images, const GatherList* lists, unsigned int count, uint32_t budget, uint32_t* overflow, int lane, int lanes) {
	unsigned long long before = 0;      // sum of v over the tiles already walked
	const unsigned int tile = (unsigned int)lanes * PACK_PER_LANE;
	for (unsigned int t0 = 0; t0 < count; t0 += tile) {
		const unsigned int j0 = t0 + (unsigned int)lane * PACK_PER_LANE;
		uint32_t v[PACK_PER_LANE];
		unsigned long long sum = 0;
		for (int k = 0; k < PACK_PER_LANE; k++) {
			v[k] = 0;
			if (j0 + k < count) {
				const GatherList& l = lists[j0 + k];
				const uint32_t c = ASTC_LDG(l.count);
				v[k] = c < l.capacity ? c : l.capacity;
			}
			sum += v[k];
		}
		const unsigned long long inclusive = pack_inclusive_sum(sum, lane, lanes);
		unsigned long long p = before + inclusive - sum;
		for (int k = 0; k < PACK_PER_LANE; k++) {
			if (j0 + k < count) {
				images[j0 + k].first = (size_t)p;
			}
			p += v[k];
		}
		before += pack_lane_value(inclusive, lanes - 1);
	}
	if (lane == 0) {
		images[count].first = (size_t)(before < budget ? before : budget);
		if (overflow != nullptr) {
			const unsigned long long excess = before > budget ? before - budget : 0;
			*overflow = excess < 0xFFFFFFFFull ? (uint32_t)excess : 0xFFFFFFFFu;
		}
	}
}

#if !defined(ASTC_HOSTSIM)
// One CTA of one warp packs the whole table.
__global__ void __launch_bounds__(32, 1)
astc_pack_lists_kernel(GatherImage* __restrict__ images, const GatherList* __restrict__ lists, unsigned int count, uint32_t budget, uint32_t* overflow) {
	pack_lists(images, lists, count, budget, overflow, (int)threadIdx.x, 32);
}
#endif
