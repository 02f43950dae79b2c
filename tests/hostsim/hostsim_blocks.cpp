// TEST TOOL (not a product path): block lists (astc_dev_gather.cuh) on the host simulation of hostsim.cpp.
//   hostsim_gather            gather_block over a list, exactly as astc_gather_blocks_kernel runs it (one simulated lane)
//   hostsim_alpha_averages_2d the alpha-scale pre-pass over a whole 2D image (the source averages the gather copies)
//   hostsim_compress_staged   hostsim_compress_volume on a staging image, with the gathered averages in place of its own
//                             pre-pass: the staging pass of the library filters nothing, it reads what the gather wrote
// Built like hostsim.cpp, with one simulated lane or with -DASTC_HOSTSIM_LANES32=1.
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

extern "C" void hostsim_gather(const void* src, int data_type, unsigned int dim_x, unsigned int dim_y, unsigned int dim_z, unsigned int bx, unsigned int by,
                               unsigned int bz, const uint32_t* indices, unsigned int n, const float* avg_src, void* dst, float* avg_dst) {
	GatherArgs g;
	g.src = src;
	g.dst = dst;
	g.avg_src = avg_src;
	g.avg_dst = avg_dst;
	g.indices = indices;
	g.n = n;
	g.words = data_type == 0 ? 1 : data_type == 1 ? 2 : 4;
	g.dim_x = dim_x;
	g.dim_y = dim_y;
	g.dim_z = dim_z;
	g.blocks_x = (dim_x + bx - 1) / bx;
	g.blocks_y = (dim_y + by - 1) / by;
	g.bx = bx;
	g.by = by;
	g.bz = bz;
	for (unsigned int i = 0; i < n; i++) {
		gather_block(g, i, 0, 1);
	}
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
