// TEST TOOL (not a product path): the slab arithmetic of the multi-GPU entry points and the alpha-scale pre-pass over one
// slab's window, compiled for the host from the library's own sources:
//   astc_host_slab.h   slab_of / slab_slices / slab_part (combined block rows of volumes and texture arrays)
//   astc_dev_alpha.cuh alpha_window (the tile rows and image rows of a slab's pre-pass) and alpha_average_tile
// hostsim_alpha_averages runs alpha_average_tile over tile rows [tile_row0, tile_row0 + tile_rows) of the 32 x 32 grid, all
// tiles of each row, as astc_alpha_average_kernel does (one simulated lane stands in for the CTA's threads).
#define ASTC_HOSTSIM 1
#include "../../astc-encoder_b200/csrc/astc_dev_search.cuh"
#include "../../astc-encoder_b200/csrc/astc_host_slab.h"
#include <vector>

extern "C" void hostsim_alpha_window(unsigned int dim_y, unsigned int radius, unsigned int y0, unsigned int y1, unsigned int* out) {
	AlphaWindow w = alpha_window(dim_y, radius, y0, y1);
	out[0] = w.tile_row0;
	out[1] = w.tile_rows;
	out[2] = w.read_row0;
	out[3] = w.read_row1;
}

extern "C" void hostsim_alpha_averages(const void* data, int data_type, unsigned int dim_x, unsigned int dim_y, const int* swz, unsigned int radius,
                                       unsigned int tile_row0, unsigned int tile_rows, float* averages) {
	DevImage img{};
	img.data = data;
	img.data_type = data_type;
	img.dim_x = dim_x;
	img.dim_y = dim_y;
	img.dim_z = 1;
	for (int i = 0; i < 4; i++) img.swz[i] = swz ? swz[i] : i;
	size_t pad = ALPHA_TILE + 2 * (size_t)radius + 1;
	std::vector<uint8_t> tile_mem(pad * pad * 4 + 64);
	astc_smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(tile_mem.data()) + 15) & ~(uintptr_t)15);
	unsigned int tiles_x = (dim_x + ALPHA_TILE - 1) / ALPHA_TILE;
	for (unsigned int ty = tile_row0; ty < tile_row0 + tile_rows; ty++) {
		for (unsigned int tx = 0; tx < tiles_x; tx++) {
			alpha_average_tile(img, radius, tx * ALPHA_TILE, ty * ALPHA_TILE, 0, averages, 0, 1);
		}
	}
	astc_smem = nullptr;
}

extern "C" void hostsim_slab_of(unsigned int rows, int world, int g, unsigned int* out) { slab_of(rows, world, g, out[0], out[1]); }

extern "C" void hostsim_slab_slices(unsigned int r0, unsigned int r1, unsigned int blocks_y, unsigned int block_z, unsigned int dim_z, unsigned int* out) {
	slab_slices(r0, r1, blocks_y, block_z, dim_z, out[0], out[1]);
}

extern "C" void hostsim_slab_part(unsigned int r0, unsigned int r1, unsigned int blocks_y, unsigned int s, unsigned int* out) {
	slab_part(r0, r1, blocks_y, s, out[0], out[1]);
}
