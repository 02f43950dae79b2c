// TEST TOOL (not a product path): map totals and gated weights (astc_dev_totals.cuh) on the host simulation of hostsim.cpp.
// Everything of hostsim.cpp, plus:
//   hostsim_map_totals  one totals call over a table of maps, as astcenc_b200_total_block_maps plans it: the partial of every
//                       virtual CTA (one simulated warp each; one lane or 32), then the finish of every entry
#include "hostsim.cpp"
#include "../../astc-encoder_b200/csrc/astc_dev_metrics.cuh"
#include "../../astc-encoder_b200/csrc/astc_dev_totals.cuh"

// Entry j: maps[j] (block_counts[j] floats), limits[j]; its total goes to *totals[j] and its weight to *weights[j] (either may be
// NULL). Returns 0, or 1 when the call does not fit a launch.
extern "C" int hostsim_map_totals(const float* const* maps, const unsigned int* block_counts, const double* limits, double* const* totals,
                                  float* const* weights, unsigned int entry_count, int rule) {
	std::vector<TotalEntry> table(entry_count);
	for (unsigned int j = 0; j < entry_count; j++) {
		table[j] = {maps[j], totals[j], weights[j], limits[j], block_counts[j], 0, 0};
	}
	size_t ctas = 0;
	if (!plan_map_totals(table, ctas)) {
		return 1;
	}
	std::vector<double> partials(ctas);
	for (const TotalEntry& e : table) {
		for (unsigned int v = 0; v < e.ctas; v++) {
			run_lanes([&](int lane) {
				const double s = map_total_partial(e, v, lane, ASTC_WARP);
				if (lane == 0) {
					partials[e.first + v] = s;
				}
			});
		}
	}
	for (const TotalEntry& e : table) {
		map_total_finish(e, partials.data(), rule);
	}
	return 0;
}
