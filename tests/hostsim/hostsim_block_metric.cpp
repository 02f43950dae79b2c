// TEST TOOL (not a product path): per-block maps of any enum astcenc_b200_block_metric (astc_dev_metrics.cuh) on the host
// simulation. Everything of hostsim_map_lists.cpp (and so of hostsim_metrics.cpp), plus:
//   hostsim_block_metric        block_error_sum<M> over every block of one pair, as astc_block_error_kernel (SQUARED_ERROR) and
//                               astc_block_metric_kernel<M> run it (one simulated warp per block; one lane or 32)
//   hostsim_block_metric_lists  block_error_list_slot<M> over every slot of a list refresh, as astc_block_error_lists_kernel and
//                               astc_block_metric_lists_kernel<M> run it (one simulated warp per slot; one lane or 32)
#include <type_traits>
#include "hostsim_map_lists.cpp"

// Runs f(std::integral_constant<int, M>) for the metric `block_metric` (0-2; anything else runs the squared error).
template <class F>
static void with_metric(int block_metric, F f) {
	switch (block_metric) {
	case ASTCENC_B200_BLOCK_ALPHA_WEIGHTED_ERROR: f(std::integral_constant<int, ASTCENC_B200_BLOCK_ALPHA_WEIGHTED_ERROR>()); break;
	case ASTCENC_B200_BLOCK_LOG2_ERROR: f(std::integral_constant<int, ASTCENC_B200_BLOCK_LOG2_ERROR>()); break;
	default: f(std::integral_constant<int, ASTCENC_B200_BLOCK_SQUARED_ERROR>()); break;
	}
}

// The map of metric `block_metric` of one pair of dim_z slices of dim_x * dim_y texels each into `out` (one float per block of
// bx x by x bz).
extern "C" void hostsim_block_metric(const void* original, int original_type, const void* decoded, int decoded_type, unsigned int dim_x, unsigned int dim_y,
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
	with_metric(block_metric, [&](auto m) {
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

// A refresh of metric `block_metric` of `count` pairs (dims: dim_x, dim_y, dim_z per pair; originals / decodeds of the given types,
// dim_z slices of dim_x * dim_y texels each) into maps[i] at the blocks of list i: indices[i], the count word counts[i] and
// capacities[i]. Returns 0, or 1 when the call does not fit a launch.
extern "C" int hostsim_block_metric_lists(const void* const* originals, const int* original_types, const void* const* decodeds, const int* decoded_types,
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
	with_metric(block_metric, [&](auto m) {
		run_lanes([&](int lane) {
			for (size_t w = 0; w < p.slots; w++) {
				block_error_list_slot<decltype(m)::value>(a, w, lane, ASTC_WARP);
			}
		});
	});
	return 0;
}
