// TEST TOOL (not a product path): pooled block selection (astc_dev_select.cuh) on the host simulation. Everything of
// hostsim_select.cpp, plus:
//   hostsim_select_pooled  one selection call over pools of entries with weights, as astcenc_b200_select_blocks_pooled plans
//                          it: the launches in order (four histogram passes, the tile counts, the per-pool scan, the write),
//                          each tile and each pool run by one simulated warp (one lane or 32)
#include "hostsim_select.cpp"

// Pool p: the next pool_entries[p] entries, pool_thresholds[p], pool_capacities[p]. Entry j: maps[j] (block_counts[j] floats),
// weights[j] (one float, or NULL); its kept indices go to indices[j], its count to counts[j].
extern "C" void hostsim_select_pooled(const unsigned int* pool_entries, const float* pool_thresholds, const unsigned int* pool_capacities,
                                      unsigned int pool_count, const float* const* maps, const unsigned int* block_counts,
                                      const float* const* weights, uint32_t* const* indices, uint32_t* counts, unsigned int entry_count) {
	std::vector<SelectEntry> table(entry_count);
	std::vector<SelectPool> pools(pool_count);
	for (unsigned int p = 0, j = 0; p < pool_count; p++) {
		pools[p].entries = pool_entries[p];
		for (unsigned int n = 0; n < pool_entries[p]; n++, j++) {
			SelectEntry& e = table[j];
			e.map = maps[j];
			e.weight = weights[j];
			e.indices = indices[j];
			e.count = counts + j;
			e.threshold = pool_thresholds[p];
			e.capacity = pool_capacities[p];
			e.block_count = block_counts[j];
		}
	}
	const size_t tiles = plan_select(table, pools);
	std::vector<uint32_t> hist(pools.size() * 1024, 0u), tile_counts(2 * tiles, 0u);
	auto each_tile = [&](auto fn) {
		for (const SelectEntry& e : table) {
			for (unsigned int t = 0; t < e.tiles; t++) {
				run_lanes([&](int lane) { fn(e, hist.data() + (size_t)e.pool * 1024, t, e.first + t, lane); });
			}
		}
	};
	for (int digit = 0; digit < 4; digit++) {
		each_tile([&](const SelectEntry& e, uint32_t* h, unsigned int t, size_t, int lane) {
			uint32_t key = 0;
			if (digit > 0) {
				const SelectState s = select_state(h, e.capacity, digit, lane, ASTC_WARP);
				if (s.k == 0) {
					return;
				}
				key = s.key;
			}
			select_hist_tile(e, t, digit, key, h, lane, ASTC_WARP);
		});
	}
	each_tile([&](const SelectEntry& e, uint32_t* h, unsigned int t, size_t w, int lane) {
		const SelectState s = select_state(h, e.capacity, 4, lane, ASTC_WARP);
		select_count_tile(e, t, s, tile_counts.data() + 2 * w, lane, ASTC_WARP);
	});
	for (size_t p = 0; p < pools.size(); p++) {
		run_lanes([&](int lane) { select_scan_pool(pools[p], table.data(), hist.data() + p * 1024, tile_counts.data(), lane, ASTC_WARP); });
	}
	each_tile([&](const SelectEntry& e, uint32_t* h, unsigned int t, size_t w, int lane) {
		const SelectState s = select_state(h, e.capacity, 4, lane, ASTC_WARP);
		if (s.k != 0) {
			select_write_tile(e, t, s, tile_counts.data() + 2 * w, lane, ASTC_WARP);
		}
	});
}
