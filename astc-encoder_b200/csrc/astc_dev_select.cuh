// CUDA-native ASTC: block selection from error maps (astcenc_b200_select_blocks, astcenc_b200_select_blocks_pooled).
//
// A call's entries are split into pools, consecutive runs of entries. Block b of entry j has the product p = map[b] * weight_j
// (weight 1 when the entry has none: the product is then the map value, bit for bit); it is a candidate when p is greater than
// its pool's threshold (NaN never is; -0.0 counts as 0.0). Of a pool's c candidates the k = min(capacity, c) largest products are
// kept, ties to the lower entry position in the pool, then to the lower block index, and each entry's kept indices are written
// in ascending order. astcenc_b200_select_blocks is the call with one pool per entry and no weights.
//
// A radix select over order-preserving 32-bit keys (select_key), one 8-bit digit per pass from the top, with one histogram of
// 256 counts per pool and digit. k, the k-th largest key K and the number of keys equal to K that are kept (krem) are a pure
// function of the pool's histograms (select_state), so every warp that needs them derives them again and no launch has to
// publish them. Then an ordered compaction: each tile counts its candidates above K and equal to K; one warp per pool walks its
// entries in order and turns the counts into exclusive prefixes, the above-K counts within each entry and the equal-to-K counts
// across the whole pool, and writes each entry's count:
//   (the entry's candidates above K) + min(eq_end, krem) - min(eq_start, krem),
// eq_start and eq_end being the pool's equal-to-K prefixes at the entry's first tile and just past its last. Each tile then
// writes a kept block of entry j at
//   (candidates above K before it in j) + min(q, krem) - min(eq_start, krem),
// q being the candidates equal to K before it in the pool. In a one-entry pool eq_start is 0 and both reduce to the per-entry
// compaction: (above K before it) + min(q, krem), count k. Each entry carries its pool's threshold and capacity, so the per-tile
// functions need nothing but the entry; the per-entry scan (select_scan_entry) is the scan of a one-entry pool.
//
// A tile is SELECT_TILE consecutive values of one map and is one warp's work; the tiles of a call are numbered across its
// entries (SelectEntry::first, find_image). Launches, whatever the number of pools and entries: a memset of the histograms, then
// seven kernels - four histogram passes, the tile counts, the per-pool scan, the write. The histograms are integer counts, whose
// atomic sums do not depend on the order they arrive in, so a pool's output depends only on the pool. Every per-tile and
// per-pool function takes (lane, lanes) and compiles for the host simulation (tests/hostsim/hostsim_select.cpp).
#pragma once
#include <vector>

#define SELECT_TILE 1024              // map values per tile (one warp)
#define SELECT_WARPS 8                // tiles (or pools) per CTA
#define SELECT_KERNELS 7              // kernel launches per call (and one memset)

// One pool of a selection call: entries [first, first + entries) of the table, which share one histogram set.
struct SelectPool {
	unsigned int first;
	unsigned int entries;
};

// One entry of a selection call, as the device reads it.
struct SelectEntry {
	const float* map;
	uint32_t* indices;
	uint32_t* count;
	float threshold;                  // the pool's
	unsigned int capacity;            // the pool's
	unsigned int block_count;
	unsigned int tiles;               // ceil(block_count / SELECT_TILE)
	size_t first;                     // the entry's first tile in the call
	const float* weight;              // one float, or NULL: weight 1
	unsigned int pool;                // the entry's pool
};

struct SelectArgs {
	const SelectEntry* entries;
	const SelectPool* pools;
	unsigned int count;               // entries
	unsigned int pool_count;
	size_t tiles;                     // tiles of the call
	uint32_t* hist;                   // [pool][digit][256]
	uint32_t* tile_counts;            // [tile][2]: candidates above K, equal to K; the scan makes them exclusive prefixes (see above)
};

// ---- host planning (no CUDA calls) ----
// Fills in the first entry of every pool (pools[i].entries set, summing to table.size()) and the tiles, first tile and pool of
// every entry; returns the call's tiles. The entries' thresholds and capacities are their pools'.
static inline size_t plan_select(std::vector<SelectEntry>& table, std::vector<SelectPool>& pools) {
	size_t tiles = 0;
	unsigned int j = 0;
	for (unsigned int p = 0; p < (unsigned int)pools.size(); p++) {
		pools[p].first = j;
		for (unsigned int n = 0; n < pools[p].entries; n++, j++) {
			SelectEntry& e = table[j];
			e.tiles = (unsigned int)(((size_t)e.block_count + SELECT_TILE - 1) / SELECT_TILE);
			e.first = tiles;
			e.pool = p;
			tiles += e.tiles;
		}
	}
	return tiles;
}

// The pools of one pool per entry (astcenc_b200_select_blocks), and the plan of a table of such pools.
static inline std::vector<SelectPool> select_pools_one_each(size_t entries) {
	std::vector<SelectPool> pools(entries);
	for (SelectPool& p : pools) {
		p.entries = 1;
	}
	return pools;
}
static inline size_t plan_select(std::vector<SelectEntry>& table) {
	std::vector<SelectPool> pools = select_pools_one_each(table.size());
	return plan_select(table, pools);
}

// ---- keys ----
// Unsigned order of the keys = float order of the values; -0.0 maps to the key of 0.0. (NaN gets a key too, but never is a
// candidate.)
ASTC_FN uint32_t select_key(float v) {
	uint32_t b = ASTC_F2U(v);
	b = b == 0x80000000u ? 0u : b;
	return (b & 0x80000000u) ? ~b : b | 0x80000000u;
}

// The entry's weight, read once per tile: 1 without one (x * 1 is x for every value but NaN, which is never a candidate).
ASTC_FN float select_weight(const SelectEntry& e) {
	return e.weight ? ASTC_LDG(e.weight) : 1.0f;
}

// ---- warp helpers over unsigned counts ----
#if defined(ASTC_ONE_LANE)
ASTC_FN uint32_t select_scan(uint32_t v, int lane) { (void)lane; return v; }
ASTC_FN uint32_t select_max(uint32_t v) { return v; }
#else
ASTC_FN uint32_t select_scan(uint32_t v, int lane) {      // inclusive prefix sum over the lanes
	for (int o = 1; o < 32; o <<= 1) {
		uint32_t t = __shfl_up_sync(0xffffffffu, v, o);
		if (lane >= o) v += t;
	}
	return v;
}
ASTC_FN uint32_t select_max(uint32_t v) {
	for (int o = 16; o > 0; o >>= 1) {
		uint32_t t = __shfl_xor_sync(0xffffffffu, v, o);
		v = t > v ? t : v;
	}
	return v;
}
#endif
// the sum over the lanes, for every lane (the inclusive prefix never decreases: its maximum is the last lane's)
ASTC_FN uint32_t select_sum(uint32_t v, int lane) { return select_max(select_scan(v, lane)); }

// ---- the state a histogram pass leaves ----
struct SelectState {
	uint32_t k;                       // blocks kept: min(capacity, candidates)
	uint32_t key;                     // the digits of K found so far (all four: K); 0xFFFFFFFF when k == 0, which no candidate matches
	uint32_t krem;                    // of the candidates that match `key` in those digits, how many are kept
};

// Candidates counted in one 256-bin histogram. The lanes hold the bins from the top down: lane l the 256 / lanes bins below
// 256 - l * (256 / lanes).
ASTC_FN uint32_t select_total(const uint32_t* h, int lane, int lanes) {
	const int per = 256 / lanes;
	uint32_t sum = 0;
	for (int p = lane * per; p < (lane + 1) * per; p++) {
		sum += ASTC_LDG(h + 255 - p);
	}
	return select_sum(sum, lane);
}

// The bin that holds the krem-th largest key of histogram h (1 <= krem <= its total), and how many keys lie in higher bins.
ASTC_FN void select_pick(const uint32_t* h, uint32_t krem, int lane, int lanes, uint32_t& bin, uint32_t& above) {
	const int per = 256 / lanes;
	uint32_t sum = 0;
	for (int p = lane * per; p < (lane + 1) * per; p++) {
		sum += ASTC_LDG(h + 255 - p);
	}
	const uint32_t incl = select_scan(sum, lane);
	uint32_t acc = incl - sum, b = 0, ab = 0;
	if (acc < krem && krem <= incl) {      // (exactly one lane)
		for (int p = lane * per; p < (lane + 1) * per; p++) {
			const uint32_t c = ASTC_LDG(h + 255 - p);
			if (acc + c >= krem) {
				b = 255u - (uint32_t)p;
				ab = acc;
				break;
			}
			acc += c;
		}
	}
	bin = select_max(b);
	above = select_max(ab);
}

// The state after `digits` (1-4) complete histograms of the pool (hist: its 4 x 256 counts).
ASTC_FN SelectState select_state(const uint32_t* hist, unsigned int capacity, int digits, int lane, int lanes) {
	SelectState s;
	const uint32_t c = select_total(hist, lane, lanes);
	s.k = capacity < c ? capacity : c;
	s.key = s.k == 0 ? 0xFFFFFFFFu : 0u;
	s.krem = s.k;
	for (int d = 0; d < digits && s.k != 0; d++) {
		uint32_t bin, above;
		select_pick(hist + d * 256, s.krem, lane, lanes, bin, above);
		s.key |= bin << (24 - 8 * d);
		s.krem -= above;
	}
	return s;
}

// ---- per tile / per pool ----
// Tile `tile` of entry e into the histogram of digit `digit` (hist: the pool's 4 x 256 counts): the candidates whose higher
// digits are those of `key`. One atomic per distinct bin and round of the warp.
ASTC_FN void select_hist_tile(const SelectEntry& e, unsigned int tile, int digit, uint32_t key, uint32_t* hist, int lane, int lanes) {
	const float w = select_weight(e);
	const int shift = 24 - 8 * digit;
	const uint32_t hi = digit == 0 ? 0u : 0xFFFFFFFFu << (shift + 8);
	const size_t i0 = (size_t)tile * SELECT_TILE;
	const size_t end = i0 + SELECT_TILE < e.block_count ? i0 + SELECT_TILE : e.block_count;
	for (size_t r = i0; r < end; r += (size_t)lanes) {
		const size_t i = r + (size_t)lane;
		int bin = -1;
		if (i < end) {
			const float v = ASTC_LDG(e.map + i) * w;
			const uint32_t k = select_key(v);
			if (v > e.threshold && (k & hi) == (key & hi)) {
				bin = (int)((k >> shift) & 255u);
			}
		}
		const int rank = wsame_key_rank(bin, lane);
		const int n = wsame_key_count(bin);
		if (bin >= 0 && rank == 0) {
			atomicAdd(hist + digit * 256 + bin, (unsigned int)n);
		}
	}
}

// Candidates of tile `tile` above s.key and equal to it, into counts[0] and counts[1].
ASTC_FN void select_count_tile(const SelectEntry& e, unsigned int tile, const SelectState& s, uint32_t* counts, int lane, int lanes) {
	const float w = select_weight(e);
	const size_t i0 = (size_t)tile * SELECT_TILE;
	const size_t end = i0 + SELECT_TILE < e.block_count ? i0 + SELECT_TILE : e.block_count;
	uint32_t gt = 0, eq = 0;
	for (size_t i = i0 + (size_t)lane; i < end; i += (size_t)lanes) {
		const float v = ASTC_LDG(e.map + i) * w;
		const uint32_t k = select_key(v);
		if (v > e.threshold) {
			gt += k > s.key ? 1u : 0u;
			eq += k == s.key ? 1u : 0u;
		}
	}
	gt = select_sum(gt, lane);
	eq = select_sum(eq, lane);
	if (lane == 0) {
		counts[0] = gt;
		counts[1] = eq;
	}
}

// Pool p's tile counts into exclusive prefixes, in place: above K within each entry, equal to K across the pool (entries: the
// call's table, tile_counts: the call's pairs, hist: the pool's 4 x 256 counts); each entry's *count as in the file comment.
ASTC_FN void select_scan_pool(const SelectPool& p, const SelectEntry* entries, const uint32_t* hist, uint32_t* tile_counts, int lane, int lanes) {
	if (p.entries == 0) {
		return;
	}
	const SelectState s = select_state(hist, entries[p.first].capacity, 4, lane, lanes);
	uint32_t eq_carry = 0;
	for (unsigned int j = p.first; j < p.first + p.entries; j++) {
		const SelectEntry& e = entries[j];
		uint32_t* counts = tile_counts + 2 * e.first;
		const uint32_t eq_start = eq_carry;
		uint32_t gt_carry = 0;
		for (unsigned int r = 0; r < e.tiles; r += (unsigned int)lanes) {
			const unsigned int t = r + (unsigned int)lane;
			const uint32_t g = t < e.tiles ? counts[2 * (size_t)t] : 0u;
			const uint32_t q = t < e.tiles ? counts[2 * (size_t)t + 1] : 0u;
			const uint32_t gi = select_scan(g, lane), qi = select_scan(q, lane);
			if (t < e.tiles) {
				counts[2 * (size_t)t] = gt_carry + gi - g;
				counts[2 * (size_t)t + 1] = eq_carry + qi - q;
			}
			gt_carry += select_max(gi);
			eq_carry += select_max(qi);
		}
		if (lane == 0) {
			*e.count = gt_carry + (eq_carry < s.krem ? eq_carry : s.krem) - (eq_start < s.krem ? eq_start : s.krem);
		}
	}
}

// Entry e's tile counts (counts: its tiles' pairs) as the scan of a pool of e alone: exclusive prefixes over its tiles, and
// *e.count = k.
ASTC_FN void select_scan_entry(const SelectEntry& e, const uint32_t* hist, uint32_t* counts, int lane, int lanes) {
	SelectPool p;
	p.first = 0;
	p.entries = 1;
	select_scan_pool(p, &e, hist, counts - 2 * e.first, lane, lanes);
}

// The kept blocks of tile `tile`, in index order, at their places in e.indices (before: the tile's two exclusive prefixes after
// the scan, within the run of the entry's pairs, whose first pair holds eq_start).
ASTC_FN void select_write_tile(const SelectEntry& e, unsigned int tile, const SelectState& s, const uint32_t* before, int lane, int lanes) {
	const float w = select_weight(e);
	const uint32_t eq_start = (before - 2 * (size_t)tile)[1];
	const size_t i0 = (size_t)tile * SELECT_TILE;
	const size_t end = i0 + SELECT_TILE < e.block_count ? i0 + SELECT_TILE : e.block_count;
	const uint32_t skip = eq_start < s.krem ? eq_start : s.krem;
	uint32_t gt_before = before[0], eq_before = before[1];
	for (size_t r = i0; r < end; r += (size_t)lanes) {
		const size_t i = r + (size_t)lane;
		uint32_t gt = 0, eq = 0;
		if (i < end) {
			const float v = ASTC_LDG(e.map + i) * w;
			const uint32_t k = select_key(v);
			if (v > e.threshold) {
				gt = k > s.key ? 1u : 0u;
				eq = k == s.key ? 1u : 0u;
			}
		}
		const uint32_t gi = select_scan(gt, lane), qi = select_scan(eq, lane);
		const uint32_t g = gt_before + gi - gt, q = eq_before + qi - eq;
		if (gt != 0 || (eq != 0 && q < s.krem)) {
			e.indices[g + (q < s.krem ? q : s.krem) - skip] = (uint32_t)i;
		}
		gt_before += select_max(gi);
		eq_before += select_max(qi);
	}
}

#if !defined(ASTC_HOSTSIM)
// ---- kernels: warp w of the launch (grid-stride) is tile w of the call, or pool w for the scan ----
// The tile's entry and its index among the entry's tiles.
static __device__ __forceinline__ const SelectEntry& select_tile_entry(const SelectArgs& a, size_t w, unsigned int& tile) {
	const SelectEntry& e = a.entries[find_image(a.entries, a.count, w)];
	tile = (unsigned int)(w - e.first);
	return e;
}

__global__ void __launch_bounds__(SELECT_WARPS * 32)
astc_select_hist_kernel(const __grid_constant__ SelectArgs a, int digit) {
	const int lane = threadIdx.x & 31;
	for (size_t w = (size_t)blockIdx.x * SELECT_WARPS + (threadIdx.x >> 5); w < a.tiles; w += (size_t)gridDim.x * SELECT_WARPS) {
		unsigned int tile;
		const SelectEntry& e = select_tile_entry(a, w, tile);
		uint32_t* hist = a.hist + (size_t)e.pool * 1024;
		uint32_t key = 0;
		if (digit > 0) {
			const SelectState s = select_state(hist, e.capacity, digit, lane, 32);
			if (s.k == 0) {
				continue;      // (the whole warp)
			}
			key = s.key;
		}
		select_hist_tile(e, tile, digit, key, hist, lane, 32);
	}
}

__global__ void __launch_bounds__(SELECT_WARPS * 32)
astc_select_count_kernel(const __grid_constant__ SelectArgs a) {
	const int lane = threadIdx.x & 31;
	for (size_t w = (size_t)blockIdx.x * SELECT_WARPS + (threadIdx.x >> 5); w < a.tiles; w += (size_t)gridDim.x * SELECT_WARPS) {
		unsigned int tile;
		const SelectEntry& e = select_tile_entry(a, w, tile);
		const SelectState s = select_state(a.hist + (size_t)e.pool * 1024, e.capacity, 4, lane, 32);
		select_count_tile(e, tile, s, a.tile_counts + 2 * w, lane, 32);
	}
}

__global__ void __launch_bounds__(SELECT_WARPS * 32)
astc_select_scan_kernel(const __grid_constant__ SelectArgs a) {
	const int lane = threadIdx.x & 31;
	for (size_t j = (size_t)blockIdx.x * SELECT_WARPS + (threadIdx.x >> 5); j < a.pool_count; j += (size_t)gridDim.x * SELECT_WARPS) {
		select_scan_pool(a.pools[j], a.entries, a.hist + j * 1024, a.tile_counts, lane, 32);
	}
}

__global__ void __launch_bounds__(SELECT_WARPS * 32)
astc_select_write_kernel(const __grid_constant__ SelectArgs a) {
	const int lane = threadIdx.x & 31;
	for (size_t w = (size_t)blockIdx.x * SELECT_WARPS + (threadIdx.x >> 5); w < a.tiles; w += (size_t)gridDim.x * SELECT_WARPS) {
		unsigned int tile;
		const SelectEntry& e = select_tile_entry(a, w, tile);
		const SelectState s = select_state(a.hist + (size_t)e.pool * 1024, e.capacity, 4, lane, 32);
		if (s.k != 0) {
			select_write_tile(e, tile, s, a.tile_counts + 2 * w, lane, 32);
		}
	}
}
#endif
