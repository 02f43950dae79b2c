// TEST TOOL (not a product path): block selection (astc_dev_select.cuh) on the host simulation of hostsim.cpp. Everything of
// hostsim.cpp, plus:
//   hostsim_select_key     select_key over an array of floats
//   hostsim_select_blocks  one selection call over a table of entries, the launches of astcenc_b200_select_blocks in order
//                          (four histogram passes, the tile counts, the per-entry scan, the write), each tile and each entry
//                          run by one simulated warp (one lane or 32)
#include "hostsim.cpp"
#if !defined(ASTC_HOSTSIM_LANES32)
static inline unsigned int atomicAdd(unsigned int* p, unsigned int v) { unsigned int o = *p; *p = o + v; return o; }
#endif
#include "../../astc-encoder_b200/csrc/astc_dev_select.cuh"

extern "C" void hostsim_select_key(const float* v, size_t n, uint32_t* out) {
	for (size_t i = 0; i < n; i++) {
		out[i] = select_key(v[i]);
	}
}

// Entry j: maps[j] (block_counts[j] floats), thresholds[j], capacities[j]; its kept indices go to indices[j], its count to
// counts[j].
extern "C" void hostsim_select_blocks(const float* const* maps, const unsigned int* block_counts, const float* thresholds, const unsigned int* capacities,
                                      uint32_t* const* indices, uint32_t* counts, unsigned int entry_count) {
	std::vector<SelectEntry> table(entry_count);
	for (unsigned int j = 0; j < entry_count; j++) {
		SelectEntry& e = table[j];
		e.map = maps[j];
		e.indices = indices[j];
		e.count = counts + j;
		e.threshold = thresholds[j];
		e.capacity = capacities[j];
		e.block_count = block_counts[j];
	}
	const size_t tiles = plan_select(table);
	std::vector<uint32_t> hist((size_t)entry_count * 1024, 0u), tile_counts(2 * tiles, 0u);
	auto each_tile = [&](auto fn) {
		for (unsigned int j = 0; j < entry_count; j++) {
			for (unsigned int t = 0; t < table[j].tiles; t++) {
				run_lanes([&](int lane) { fn(table[j], hist.data() + (size_t)j * 1024, t, table[j].first + t, lane); });
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
	for (unsigned int j = 0; j < entry_count; j++) {
		run_lanes([&](int lane) { select_scan_entry(table[j], hist.data() + (size_t)j * 1024, tile_counts.data() + 2 * table[j].first, lane, ASTC_WARP); });
	}
	each_tile([&](const SelectEntry& e, uint32_t* h, unsigned int t, size_t w, int lane) {
		const SelectState s = select_state(h, e.capacity, 4, lane, ASTC_WARP);
		if (s.k != 0) {
			select_write_tile(e, t, s, tile_counts.data() + 2 * w, lane, ASTC_WARP);
		}
	});
}
