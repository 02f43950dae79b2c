// TEST TOOL (not a product path): metrics calls (astc_dev_metrics.cuh) on the host simulation of hostsim.cpp. Everything of
// hostsim.cpp, plus:
//   hostsim_plan_metrics   plan_metrics over a table of pairs, as both metrics entry points plan their calls
//   hostsim_block_error    block_error_sum over every block of one pair, as astc_block_error_kernel runs it (one simulated warp
//                          per block; one lane or 32)
#include "hostsim.cpp"
#include "../../astc-encoder_b200/csrc/astc_dev_metrics.cuh"

// dims: dim_x, dim_y, dim_z per pair; mapped[i] != 0: pair i asks for a map. Out: per pair its virtual CTAs per slice, first
// virtual CTA and map blocks x / y; maps: (first map block, pair) per mapped pair; totals: virtual CTAs, map blocks, partial
// doubles, finish grid, map grid. Returns 0, or 1 when the call does not fit a launch.
extern "C" int hostsim_plan_metrics(const unsigned int* dims, const int* mapped, unsigned int count, unsigned int bx, unsigned int by, unsigned int bz,
                                    unsigned int* ctas, size_t* first, unsigned int* blocks_xy, size_t* maps, size_t* totals) {
	static float dummy;
	std::vector<MetricEntry> table(count);
	for (unsigned int i = 0; i < count; i++) {
		MetricEntry& e = table[i];
		memset(&e, 0, sizeof(e));
		e.dim_x = dims[3 * i];
		e.dim_y = dims[3 * i + 1];
		e.dim_z = dims[3 * i + 2];
		e.block_error = mapped[i] ? &dummy : nullptr;
	}
	MetricPlan p;
	if (!plan_metrics(table, bx, by, bz, p)) {
		return 1;
	}
	for (unsigned int i = 0; i < count; i++) {
		ctas[i] = table[i].ctas;
		first[i] = table[i].first;
		blocks_xy[2 * i] = table[i].blocks_x;
		blocks_xy[2 * i + 1] = table[i].blocks_y;
	}
	for (size_t m = 0; m < p.maps.size(); m++) {
		maps[2 * m] = p.maps[m].first;
		maps[2 * m + 1] = p.maps[m].entry;
	}
	totals[0] = p.ctas;
	totals[1] = p.map_blocks;
	totals[2] = p.partial_doubles;
	totals[3] = p.finish_grid;
	totals[4] = p.map_grid;
	return 0;
}

// The map of one pair of dim_z slices of dim_x * dim_y texels each into `out` (one float per block of bx x by x bz).
extern "C" void hostsim_block_error(const void* original, int original_type, const void* decoded, int decoded_type, unsigned int dim_x, unsigned int dim_y,
                                    unsigned int dim_z, unsigned int bx, unsigned int by, unsigned int bz, int input_components, float* out) {
	std::vector<MetricEntry> table(1);
	MetricEntry& e = table[0];
	memset(&e, 0, sizeof(e));
	e.img1 = original;
	e.img2 = decoded;
	e.type1 = original_type;
	e.type2 = decoded_type;
	e.pitch1 = e.pitch2 = dim_x;
	e.stride1 = e.stride2 = (size_t)dim_x * dim_y;
	e.dim_x = dim_x;
	e.dim_y = dim_y;
	e.dim_z = dim_z;
	e.block_error = out;
	MetricPlan p;
	plan_metrics(table, bx, by, bz, p);
	const int mask = metric_component_mask(input_components);
	run_lanes([&](int lane) {
		for (size_t b = 0; b < p.map_blocks; b++) {
			const double s = block_error_sum(e, bx, by, bz, (uint32_t)b, mask, lane, ASTC_WARP);
			if (lane == 0) {
				out[b] = (float)s;
			}
		}
	});
}
