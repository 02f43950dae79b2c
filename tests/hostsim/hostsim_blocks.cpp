// TEST TOOL (not a product path): staging calls (astc_dev_gather.cuh) on the host simulation of hostsim.cpp.
//   hostsim_gather_table      gather_block over staging blocks [base, base + n) of a block-list table, as
//                             astc_gather_blocks_kernel runs it: every block of each image, or the slots of each entry's list
//   hostsim_scatter_table     scatter_target for the same staging blocks: each staged block to its image's payload, nothing for an
//                             invalid list slot
//   hostsim_alpha_averages_2d the alpha-scale pre-pass over a whole 2D image (the source averages the gather copies)
//   hostsim_compress_staged   hostsim_compress_volume on a staging image, with the gathered averages in place of its own
//                             pre-pass: the staging pass of the library filters nothing, it reads what the gather wrote
// The table is built as plan_blocks builds it (image_table). A host list of n blocks is a one-entry table whose list has
// capacity n and count n. Built like hostsim.cpp, with one simulated lane or with -DASTC_HOSTSIM_LANES32=1; the gather and the
// scatter run on the simulated lanes.
#define ASTC_HOSTSIM 1
#if defined(ASTC_HOSTSIM_LANES32)
#include "simt_emul.h"
#endif
#include "../../astc-encoder_b200/csrc/astc_dev_search.cuh"
#include "../../astc-encoder_b200/csrc/astc_dev_gather.cuh"

static const float* g_staged_averages = nullptr;

// hostsim_compress_volume's pre-pass calls this for every 32 x 32 tile: with staged averages it copies the tile's part of them
static inline void staged_alpha_tile(const DevImage& img, unsigned int radius, unsigned int ox, unsigned int oy, uint32_t buf_off, float* averages,
                                     int tid, int nthreads) {
	if (g_staged_averages == nullptr) {
		alpha_average_tile(img, radius, ox, oy, buf_off, averages, tid, nthreads);
		return;
	}
	unsigned int size_x = img.dim_x - ox < ALPHA_TILE ? img.dim_x - ox : ALPHA_TILE;
	unsigned int size_y = img.dim_y - oy < ALPHA_TILE ? img.dim_y - oy : ALPHA_TILE;
	for (unsigned int i = (unsigned int)tid; i < size_x * size_y; i += (unsigned int)nthreads) {
		size_t o = (size_t)(oy + i / size_x) * img.dim_x + ox + i % size_x;
		averages[o] = g_staged_averages[o];
	}
	cta_sync();
}
#define alpha_average_tile staged_alpha_tile
#include "hostsim.cpp"
#undef alpha_average_tile

// The table of a staging call over image_count images (dims: dim_x, dim_y, dim_z of each): entry j owns the staging blocks that
// follow those of the entries before it - its image's blocks, or capacities[j] when the call has lists - and its averages
// follow theirs (dim_x * dim_y floats each). data or payloads may be null where the caller reads neither.
static std::vector<GatherImage> image_table(const void* const* data, const unsigned int* dims, unsigned int image_count, unsigned int bx, unsigned int by,
                                            unsigned int bz, uint8_t* const* payloads, const unsigned int* capacities = nullptr) {
	std::vector<GatherImage> table(image_count);
	size_t first = 0, avg_offset = 0;
	for (unsigned int j = 0; j < image_count; j++) {
		GatherImage& e = table[j];
		e.data = data != nullptr ? data[j] : nullptr;
		e.payload = payloads != nullptr ? payloads[j] : nullptr;
		e.dim_x = dims[3 * j];
		e.dim_y = dims[3 * j + 1];
		e.dim_z = dims[3 * j + 2];
		e.blocks_x = (e.dim_x + bx - 1) / bx;
		e.blocks_y = (e.dim_y + by - 1) / by;
		e.first = first;
		e.avg_offset = avg_offset;
		first += capacities != nullptr ? capacities[j] : (size_t)e.blocks_x * e.blocks_y * ((e.dim_z + bz - 1) / bz);
		avg_offset += (size_t)e.dim_x * e.dim_y;
	}
	return table;
}

// A staging call: its table, its lists (indices null: none; else indices[j], the count word counts[j] and capacities[j] of
// entry j) and the gather arguments of staging blocks [base, base + n).
struct SimCall {
	std::vector<GatherImage> table;
	std::vector<GatherList> lists;
	GatherArgs g{};
	SimCall(const void* const* data, const unsigned int* dims, unsigned int image_count, int data_type, unsigned int bx, unsigned int by, unsigned int bz,
	        uint8_t* const* payloads, const uint32_t* const* indices, const uint32_t* counts, const unsigned int* capacities, size_t base, unsigned int n)
	    : table(image_table(data, dims, image_count, bx, by, bz, payloads, indices != nullptr ? capacities : nullptr)) {
		for (unsigned int j = 0; j < image_count && indices != nullptr; j++) {
			const GatherImage& e = table[j];
			lists.push_back({indices[j], counts + j, capacities[j], e.blocks_x * e.blocks_y * ((e.dim_z + bz - 1) / bz)});
		}
		g.n = n;
		g.words = data_type == 0 ? 1 : data_type == 1 ? 2 : 4;
		g.bx = bx;
		g.by = by;
		g.bz = bz;
		g.images = table.data();
		g.image_count = image_count;
		g.base = base;
		g.lists = indices != nullptr ? lists.data() : nullptr;
	}
};

extern "C" void hostsim_gather_table(const void* const* data, const unsigned int* dims, unsigned int image_count, int data_type, unsigned int bx,
                                     unsigned int by, unsigned int bz, const uint32_t* const* indices, const uint32_t* counts, const unsigned int* capacities,
                                     size_t base, unsigned int n, const float* avg_src, void* dst, float* avg_dst) {
	SimCall c(data, dims, image_count, data_type, bx, by, bz, nullptr, indices, counts, capacities, base, n);
	c.g.dst = dst;
	c.g.avg_src = avg_src;
	c.g.avg_dst = avg_dst;
	run_lanes([&](int lane) {
		for (unsigned int i = 0; i < n; i++) {
			gather_block(c.g, i, lane, ASTC_WARP);
		}
	});
}

extern "C" void hostsim_scatter_table(const unsigned int* dims, unsigned int image_count, unsigned int bx, unsigned int by, unsigned int bz,
                                      const uint32_t* const* indices, const uint32_t* counts, const unsigned int* capacities, size_t base, unsigned int n,
                                      const uint8_t* staged, uint8_t* const* payloads) {
	SimCall c(nullptr, dims, image_count, 0, bx, by, bz, payloads, indices, counts, capacities, base, n);
	run_lanes([&](int lane) {
		for (unsigned int i = (unsigned int)lane; i < n; i += ASTC_WARP) {
			uint8_t* dst = scatter_target(c.g, i);
			if (dst != nullptr) {
				memcpy(dst, staged + (size_t)i * 16, 16);
			}
		}
	});
}

extern "C" void hostsim_alpha_averages_2d(const void* data, int data_type, unsigned int dim_x, unsigned int dim_y, const int* swz, unsigned int radius, float* averages) {
	DevImage img{};
	img.data = data;
	img.data_type = data_type;
	img.dim_x = dim_x;
	img.dim_y = dim_y;
	img.dim_z = 1;
	for (int i = 0; i < 4; i++) img.swz[i] = swz ? swz[i] : i;
	size_t pad = ALPHA_TILE + 2 * (size_t)radius + 1;
	std::vector<uint8_t> tile_mem(pad * pad * 4 + 64);
	uint8_t* saved = astc_smem;
	astc_smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(tile_mem.data()) + 15) & ~(uintptr_t)15);
	run_lanes([&](int lane) {
		for (unsigned int oy = 0; oy < dim_y; oy += ALPHA_TILE) {
			for (unsigned int ox = 0; ox < dim_x; ox += ALPHA_TILE) {
				alpha_average_tile(img, radius, ox, oy, 0, averages, lane, ASTC_WARP);
				cta_sync();
			}
		}
	});
	astc_smem = saved;
}

extern "C" int hostsim_compress_staged(int profile, unsigned int bx, unsigned int by, unsigned int bz, float quality, unsigned int flags, unsigned int radius,
                                       const void* data, int data_type, unsigned int dim_x, unsigned int dim_y, unsigned int dim_z, const float* averages, uint8_t* out) {
	g_hostsim_a_scale_radius = radius;
	g_staged_averages = averages;
	int rc = hostsim_compress_volume(profile, bx, by, bz, quality, flags, data, data_type, dim_x, dim_y, dim_z, nullptr, out);
	g_staged_averages = nullptr;
	g_hostsim_a_scale_radius = 0;
	return rc;
}
