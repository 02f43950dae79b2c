// CUDA-native ASTC: keep-the-better re-encodes of device block lists (astcenc_b200_refine_device_block_lists).
//
// The call is a staging call (astc_dev_gather.cuh): each chunk's listed blocks are gathered into a staging row and one pass of
// the wave pipeline compresses it into the chunk's staged candidates. Where compress_device_block_lists scatters them, a refine
// call instead
//   1. decodes the staged candidates into a staging decode row of the same layout (astc_decompress_images_kernel over a one-entry
//      table: the row is an image of m x 1 blocks), with the context that encoded them;
//   2. decides (refine_decide_block, one warp per staging block): the candidate value v' is block_error_sum_of<M> of the block's
//      original texels against the decoded candidate in the row, the same terms in the same lane and shuffle order as the whole
//      map, so v' is bit for bit the map value of that block under the candidate; the block is kept iff v' < block_error[index];
//   3. commits (refine_commit_block, one warp per staging block): a kept block's 16 bytes go to the payload, its footprint's
//      texels inside the image from the row to the caller's decode (when there is one), and v' to the map.
// Deciding and committing are separate launches, so every decision of a chunk reads the map as it stood before the chunk: two
// slots of one block in a chunk decide alike and commit the same bytes, and a copy in a later chunk meets a map value equal to
// its own v' and keeps nothing. Ties and NaN on either side keep the old block.
#pragma once

// The pairs of a refine call, one per entry of its staging table (GatherArgs::images): entry j's original (img1, type1, pitch1,
// stride1: the image the gather reads), its decode (img2, the caller's decoded image or null; type2, the decoded type), its map
// (block_error), dims and footprint block counts. row: the chunk's decoded candidates in the staging layout, texels of type2;
// values / keep: one candidate value and one decision per staging block of the chunk.
struct RefineArgs {
	const MetricEntry* pairs;
	const void* row;
	float* values;
	uint8_t* keep;
	int components;
};

// Staging block i of the chunk, by `lanes` lanes of one warp: its candidate value and decision (0 for an invalid list slot).
// PACKED: a packed table (astc_dev_gather.cuh).
template <int M, bool PACKED = false>
ASTC_FN void refine_decide_block(const GatherArgs& g, const RefineArgs& r, unsigned int i, int lane, int lanes) {
	unsigned int j;
	const uint32_t index = staged_block<PACKED>(g, i, j);
	if (index == GATHER_INVALID) {
		if (lane == 0) {
			r.keep[i] = 0;
		}
		return;      // (the whole warp)
	}
	const MetricEntry& e = r.pairs[j];
	const GatherImage& im = g.images[j];
	const double s = block_error_sum_of<M>(e, g.bx, g.by, g.bz, index, metric_component_mask(r.components), lane, lanes,
	                                       [&](unsigned int t, unsigned int, unsigned int, unsigned int) {
		                                       return metric_texel(r.row, e.type2, gather_texel(g, im, i, index, t).dst);
	                                       });
	if (lane == 0) {
		const float v = (float)s;
		r.values[i] = v;
		r.keep[i] = v < ASTC_LDG(e.block_error + index) ? 1 : 0;
	}
}

// Staging block i of the chunk, by `lanes` lanes of one warp, when it was kept: its staged bytes (staged + 16 i) into the payload,
// the texels of its footprint inside the image from the row into the decode (when the pair has one) and its value into the map.
template <bool PACKED = false>
ASTC_FN void refine_commit_block(const GatherArgs& g, const RefineArgs& r, const uint8_t* staged, unsigned int i, int lane, int lanes) {
	if (ASTC_LDG(r.keep + i) == 0) {
		return;      // (the whole warp)
	}
	unsigned int j;
	const uint32_t index = staged_block<PACKED>(g, i, j);      // (a kept block is a valid slot)
	const MetricEntry& e = r.pairs[j];
	const GatherImage& im = g.images[j];
	if (lane == 0) {
#if defined(ASTC_HOSTSIM)
		memcpy(im.payload + (size_t)index * 16, staged + (size_t)i * 16, 16);
#else
		store_block(im.payload + (size_t)index * 16, __ldg(reinterpret_cast<const uint4*>(staged) + i));
#endif
		e.block_error[index] = ASTC_LDG(r.values + i);
	}
	if (e.img2 == nullptr) {
		return;
	}
	const unsigned int words = e.type2 == 0 ? 1 : e.type2 == 1 ? 2 : 4;
	const uint32_t* src = static_cast<const uint32_t*>(r.row);
	uint32_t* dst = static_cast<uint32_t*>(const_cast<void*>(e.img2));
	for (unsigned int w = (unsigned int)lane; w < g.bx * g.by * g.bz * words; w += (unsigned int)lanes) {
		const unsigned int t = w / words, k = w - t * words;
		unsigned int tx, ty, tz, x, y, z;
		footprint_texel(im.blocks_x, im.blocks_y, g.bx, g.by, g.bz, index, t, tx, ty, tz, x, y, z);
		if (x < im.dim_x && y < im.dim_y && z < im.dim_z) {
			const GatherTexel p = gather_texel(g, im, i, index, t);      // (inside the image: p.src is the texel's own position)
			dst[p.src * words + k] = ASTC_LDG(src + p.dst * words + k);
		}
	}
}

#if !defined(ASTC_HOSTSIM)
#define ASTC_REFINE_LIST_WARPS 8            // decide and commit kernels: staging blocks per CTA, one warp each

// The decisions of a chunk for maps of metric M: warp i of the launch is staging block i.
template <int M>
__global__ void __launch_bounds__(ASTC_REFINE_LIST_WARPS * 32)
astc_refine_decide_kernel(const __grid_constant__ GatherArgs g, const __grid_constant__ RefineArgs r) {
	const unsigned int i = blockIdx.x * ASTC_REFINE_LIST_WARPS + (threadIdx.x >> 5);
	if (i < g.n) {
		refine_decide_block<M>(g, r, i, threadIdx.x & 31, ASTC_WARP);
	}
}

// The commits of a chunk: warp i of the launch is staging block i.
__global__ void __launch_bounds__(ASTC_REFINE_LIST_WARPS * 32)
astc_refine_commit_kernel(const uint8_t* __restrict__ staged, const __grid_constant__ GatherArgs g, const __grid_constant__ RefineArgs r) {
	const unsigned int i = blockIdx.x * ASTC_REFINE_LIST_WARPS + (threadIdx.x >> 5);
	if (i < g.n) {
		refine_commit_block(g, r, staged, i, threadIdx.x & 31, ASTC_WARP);
	}
}

// The same two kernels over a packed table (astc_dev_gather.cuh).
template <int M>
__global__ void __launch_bounds__(ASTC_REFINE_LIST_WARPS * 32)
astc_refine_decide_packed_kernel(const __grid_constant__ GatherArgs g, const __grid_constant__ RefineArgs r) {
	const unsigned int i = blockIdx.x * ASTC_REFINE_LIST_WARPS + (threadIdx.x >> 5);
	if (i < g.n) {
		refine_decide_block<M, true>(g, r, i, threadIdx.x & 31, ASTC_WARP);
	}
}

__global__ void __launch_bounds__(ASTC_REFINE_LIST_WARPS * 32)
astc_refine_commit_packed_kernel(const uint8_t* __restrict__ staged, const __grid_constant__ GatherArgs g, const __grid_constant__ RefineArgs r) {
	const unsigned int i = blockIdx.x * ASTC_REFINE_LIST_WARPS + (threadIdx.x >> 5);
	if (i < g.n) {
		refine_commit_block<true>(g, r, staged, i, threadIdx.x & 31, ASTC_WARP);
	}
}
#endif
