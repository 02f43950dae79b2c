// libastcenc_b200: the slab arithmetic of the multi-GPU entry points (astc_host_multi.inl), free of CUDA and NCCL so that the
// host tests run the same code.
//
// A slab is a range of COMBINED block rows: row r of a volume (3D block sizes) or of a texture array (2D block size, dim_z > 1)
// is layer_or_slice * blocks_y + row, the order in which astcenc_compress_image lays out the payload (row r at r * blocks_x * 16,
// astcenc_entry.cpp:1036). A 2D image is the case of one slice.
#pragma once

// combined block rows [first, last) of rank g when `rows` of them are cut into `world` slabs (the same rule on every rank)
static inline void slab_of(unsigned int rows, int world, int g, unsigned int& first, unsigned int& last) {
	first = (unsigned int)((size_t)rows * (size_t)g / (size_t)world);
	last = (unsigned int)((size_t)rows * (size_t)(g + 1) / (size_t)world);
}

// The image slices [z0, z1) that combined rows [r0, r1) (r0 < r1) read: the slices of the layers they touch, block_z of them per
// layer and clipped to dim_z (texture arrays: block_z = 1, one slice per layer).
static inline void slab_slices(unsigned int r0, unsigned int r1, unsigned int blocks_y, unsigned int block_z, unsigned int dim_z, unsigned int& z0,
                               unsigned int& z1) {
	unsigned int layer0 = r0 / blocks_y, layer1 = (r1 + blocks_y - 1) / blocks_y;
	size_t a = (size_t)layer0 * block_z, b = (size_t)layer1 * block_z;
	z0 = (unsigned int)(a < dim_z ? a : dim_z);
	z1 = (unsigned int)(b < dim_z ? b : dim_z);
}

// The part of combined rows [r0, r1) that lies in layer (or slice) s: block rows [first, last) of that layer, empty if first == last.
static inline void slab_part(unsigned int r0, unsigned int r1, unsigned int blocks_y, unsigned int s, unsigned int& first, unsigned int& last) {
	size_t lo = (size_t)s * blocks_y, hi = lo + blocks_y;
	size_t a = r0 > lo ? r0 : lo, b = r1 < hi ? r1 : hi;
	first = (unsigned int)(a - lo);
	last = (unsigned int)(b > a ? b - lo : a - lo);
}
