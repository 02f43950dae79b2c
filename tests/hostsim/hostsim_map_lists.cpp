// TEST TOOL (not a product path): map refreshes over device block lists (astc_dev_metrics.cuh) on the host simulation.
// Everything of hostsim_metrics.cpp, plus:
//   hostsim_plan_block_error_lists  plan_block_error_lists over a table of pairs, as astcenc_b200_compute_block_errors_device_block_lists
//                                   plans its call
//   hostsim_block_error_lists       block_error_list_slot over every slot of such a call, as astc_block_error_lists_kernel runs it
//                                   (one simulated warp per slot; one lane or 32)
#include "hostsim_metrics.cpp"

// dims: dim_x, dim_y, dim_z per pair; capacities: per pair. Out: per pair its first slot and map blocks x / y; totals: slots,
// grid. Returns 0, or 1 when the call does not fit a launch.
extern "C" int hostsim_plan_block_error_lists(const unsigned int* dims, const unsigned int* capacities, unsigned int count, unsigned int bx, unsigned int by,
                                              unsigned int bz, size_t* first, unsigned int* blocks_xy, size_t* totals) {
	static float dummy;
	std::vector<MetricEntry> table(count);
	for (unsigned int i = 0; i < count; i++) {
		MetricEntry& e = table[i];
		memset(&e, 0, sizeof(e));
		e.dim_x = dims[3 * i];
		e.dim_y = dims[3 * i + 1];
		e.dim_z = dims[3 * i + 2];
		e.block_error = &dummy;
	}
	MetricListPlan p;
	if (!plan_block_error_lists(table, capacities, bx, by, bz, p)) {
		return 1;
	}
	for (unsigned int i = 0; i < count; i++) {
		first[i] = p.maps[i].first;
		blocks_xy[2 * i] = table[i].blocks_x;
		blocks_xy[2 * i + 1] = table[i].blocks_y;
	}
	totals[0] = p.slots;
	totals[1] = p.grid;
	return 0;
}

// A refresh of `count` pairs (dims as above; originals / decodeds of the given types, dim_z slices of dim_x * dim_y texels each)
// into maps[i] at the blocks of list i: indices[i], the count word counts[i] and capacities[i]. Returns as the planner does.
extern "C" int hostsim_block_error_lists(const void* const* originals, const int* original_types, const void* const* decodeds, const int* decoded_types,
                                         const unsigned int* dims, unsigned int count, unsigned int bx, unsigned int by, unsigned int bz, int input_components,
                                         float* const* maps, const uint32_t* const* indices, const uint32_t* counts, const unsigned int* capacities) {
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
	run_lanes([&](int lane) {
		for (size_t w = 0; w < p.slots; w++) {
			block_error_list_slot(a, w, lane, ASTC_WARP);
		}
	});
	return 0;
}
