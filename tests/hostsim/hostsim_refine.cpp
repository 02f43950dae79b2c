// TEST TOOL (not a product path): the decisions and commits of refine calls (astc_dev_refine.cuh) on the host simulation.
// Everything of hostsim_block_metric.cpp, plus:
//   hostsim_refine_decide  refine_decide_block<M> over staging blocks [base, base + n) of a refine call, as
//                          astc_refine_decide_kernel<M> runs it on one chunk (one simulated warp per staging block; one lane or 32)
//   hostsim_refine_commit  refine_commit_block over the same staging blocks, as astc_refine_commit_kernel runs it
// The table is built as astcenc_b200_refine_device_block_lists builds it (plan_blocks): entries of capacity 0 are left out, and
// entry j owns the capacities[j] staging blocks that follow those of the entries before it. The chunk's staged candidates and
// their decode row are the caller's: one row of n blocks in the staging layout, texels of decoded_type.
#include "hostsim_block_metric.cpp"
#include "../../astc-encoder_b200/csrc/astc_dev_refine.cuh"

// A refine call's chunk: entry j has data[j] (data_type), dims[3j..3j+2], payloads[j], decodeds[j] (decoded_type, or null),
// maps[j] and the list indices[j] / counts[j] / capacities[j].
struct SimRefine {
	std::vector<GatherImage> table;
	std::vector<GatherList> lists;
	std::vector<MetricEntry> pairs;
	GatherArgs g{};
	RefineArgs r{};
	SimRefine(const void* const* data, const unsigned int* dims, unsigned int count, int data_type, int decoded_type, unsigned int bx, unsigned int by,
	          unsigned int bz, uint8_t* const* payloads, void* const* decodeds, float* const* maps, const uint32_t* const* indices, const uint32_t* counts,
	          const unsigned int* capacities, int components, size_t base, unsigned int n, const void* row, float* values, uint8_t* keep) {
		size_t first = 0;
		for (unsigned int j = 0; j < count; j++) {
			if (capacities[j] == 0) {
				continue;
			}
			GatherImage e{};
			e.data = data[j];
			e.payload = payloads[j];
			e.first = first;
			e.dim_x = dims[3 * j];
			e.dim_y = dims[3 * j + 1];
			e.dim_z = dims[3 * j + 2];
			e.blocks_x = (e.dim_x + bx - 1) / bx;
			e.blocks_y = (e.dim_y + by - 1) / by;
			table.push_back(e);
			lists.push_back({indices[j], counts + j, capacities[j], e.blocks_x * e.blocks_y * ((e.dim_z + bz - 1) / bz)});
			MetricEntry p;
			memset(&p, 0, sizeof(p));
			p.img1 = data[j];
			p.img2 = decodeds[j];
			p.type1 = data_type;
			p.type2 = decoded_type;
			p.pitch1 = p.pitch2 = e.dim_x;
			p.stride1 = p.stride2 = (size_t)e.dim_x * e.dim_y;
			p.dim_x = e.dim_x;
			p.dim_y = e.dim_y;
			p.dim_z = e.dim_z;
			p.blocks_x = e.blocks_x;
			p.blocks_y = e.blocks_y;
			p.block_error = maps[j];
			pairs.push_back(p);
			first += capacities[j];
		}
		g.n = n;
		g.words = data_type == 0 ? 1 : data_type == 1 ? 2 : 4;
		g.bx = bx;
		g.by = by;
		g.bz = bz;
		g.images = table.data();
		g.image_count = (unsigned int)table.size();
		g.base = base;
		g.lists = lists.data();
		r.pairs = pairs.data();
		r.row = row;
		r.values = values;
		r.keep = keep;
		r.components = components;
	}
};

// The arguments of both walks: the table as SimRefine takes it, the chunk (staging blocks [base, base + n)), its decode row and
// its values and decisions.
#define SIM_REFINE_PARAMS                                                                                                              \
	const void* const* data, const unsigned int* dims, unsigned int count, int data_type, int decoded_type, unsigned int bx,         \
	unsigned int by, unsigned int bz, uint8_t* const* payloads, void* const* decodeds, float* const* maps,                          \
	const uint32_t* const* indices, const uint32_t* counts, const unsigned int* capacities, int components, size_t base, unsigned int n, \
	const void* row, float* values, uint8_t* keep
#define SIM_REFINE_ARGS data, dims, count, data_type, decoded_type, bx, by, bz, payloads, decodeds, maps, indices, counts, capacities, components, base, n, row, values, keep

// The decisions of staging blocks [base, base + n) for maps of `block_metric`: values[i] and keep[i] of staging block base + i.
extern "C" void hostsim_refine_decide(SIM_REFINE_PARAMS, int block_metric) {
	SimRefine c(SIM_REFINE_ARGS);
	with_metric(block_metric, [&](auto m) {
		run_lanes([&](int lane) {
			for (unsigned int i = 0; i < n; i++) {
				refine_decide_block<decltype(m)::value>(c.g, c.r, i, lane, ASTC_WARP);
			}
		});
	});
}

// The commits of the same staging blocks; staged: their candidates, 16 bytes each.
extern "C" void hostsim_refine_commit(SIM_REFINE_PARAMS, const uint8_t* staged) {
	SimRefine c(SIM_REFINE_ARGS);
	run_lanes([&](int lane) {
		for (unsigned int i = 0; i < n; i++) {
			refine_commit_block(c.g, c.r, staged, i, lane, ASTC_WARP);
		}
	});
}
