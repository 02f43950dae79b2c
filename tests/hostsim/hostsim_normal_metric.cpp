// TEST TOOL (not a product path): per-block maps, list refreshes and refine decisions of every enum astcenc_b200_block_metric,
// the normal-map metrics (ANGULAR_ERROR, WORST_ANGULAR_ERROR) included, on the host simulation. Everything of hostsim_refine.cpp
// (and so of hostsim_block_metric.cpp), plus the same three walks over any metric:
//   hostsim_any_metric               block_error_sum<M> over every block of one pair, as astc_block_metric_kernel<M> runs it
//   hostsim_any_metric_lists         block_error_list_slot<M> over every slot of a list refresh, as astc_block_metric_lists_kernel<M>
//   hostsim_any_metric_refine_decide refine_decide_block<M> over staging blocks [base, base + n), as astc_refine_decide_kernel<M>
// (one simulated warp per block or slot; one lane or 32). The arguments are those of hostsim_block_metric,
// hostsim_block_metric_lists and hostsim_refine_decide.
#include "hostsim_refine.cpp"

// Runs f(std::integral_constant<int, M>) for the metric `block_metric` (0-2, 4, 5; anything else runs the squared error).
template <class F>
static void with_any_metric(int block_metric, F f) {
	switch (block_metric) {
	case ASTCENC_B200_BLOCK_ANGULAR_ERROR: f(std::integral_constant<int, ASTCENC_B200_BLOCK_ANGULAR_ERROR>()); break;
	case ASTCENC_B200_BLOCK_WORST_ANGULAR_ERROR: f(std::integral_constant<int, ASTCENC_B200_BLOCK_WORST_ANGULAR_ERROR>()); break;
	default: with_metric(block_metric, f); break;
	}
}

extern "C" void hostsim_any_metric(const void* original, int original_type, const void* decoded, int decoded_type, unsigned int dim_x, unsigned int dim_y,
                                   unsigned int dim_z, unsigned int bx, unsigned int by, unsigned int bz, int input_components, int block_metric, float* out) {
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
	with_any_metric(block_metric, [&](auto m) {
		run_lanes([&](int lane) {
			for (size_t b = 0; b < p.map_blocks; b++) {
				const double s = block_error_sum<decltype(m)::value>(e, bx, by, bz, (uint32_t)b, mask, lane, ASTC_WARP);
				if (lane == 0) {
					out[b] = (float)s;
				}
			}
		});
	});
}

// Returns 0, or 1 when the call does not fit a launch.
extern "C" int hostsim_any_metric_lists(const void* const* originals, const int* original_types, const void* const* decodeds, const int* decoded_types,
                                        const unsigned int* dims, unsigned int count, unsigned int bx, unsigned int by, unsigned int bz, int input_components,
                                        int block_metric, float* const* maps, const uint32_t* const* indices, const uint32_t* counts,
                                        const unsigned int* capacities) {
	std::vector<MetricEntry> table(count);
	for (unsigned int i = 0; i < count; i++) {
		MetricEntry& e = table[i];
		memset(&e, 0, sizeof(e));
		e.img1 = originals[i];
		e.img2 = decodeds[i];
		e.type1 = original_types[i];
		e.type2 = decoded_types[i];
		e.dim_x = dims[3 * i];
		e.dim_y = dims[3 * i + 1];
		e.dim_z = dims[3 * i + 2];
		e.pitch1 = e.pitch2 = e.dim_x;
		e.stride1 = e.stride2 = (size_t)e.dim_x * e.dim_y;
		e.block_error = maps[i];
	}
	MetricListPlan p;
	if (!plan_block_error_lists(table, capacities, bx, by, bz, p)) {
		return 1;
	}
	std::vector<GatherList> lists(count);
	for (unsigned int i = 0; i < count; i++) {
		lists[i] = {indices[i], counts + i, capacities[i], table[i].blocks_x * table[i].blocks_y * ((table[i].dim_z + bz - 1) / bz)};
	}
	MetricListArgs a;
	a.entries = table.data();
	a.maps = p.maps.data();
	a.lists = lists.data();
	a.count = count;
	a.slots = p.slots;
	a.bx = bx;
	a.by = by;
	a.bz = bz;
	a.components = input_components;
	with_any_metric(block_metric, [&](auto m) {
		run_lanes([&](int lane) {
			for (size_t w = 0; w < p.slots; w++) {
				block_error_list_slot<decltype(m)::value>(a, w, lane, ASTC_WARP);
			}
		});
	});
	return 0;
}

extern "C" void hostsim_any_metric_refine_decide(SIM_REFINE_PARAMS, int block_metric) {
	SimRefine c(SIM_REFINE_ARGS);
	with_any_metric(block_metric, [&](auto m) {
		run_lanes([&](int lane) {
			for (unsigned int i = 0; i < n; i++) {
				refine_decide_block<decltype(m)::value>(c.g, c.r, i, lane, ASTC_WARP);
			}
		});
	});
}
