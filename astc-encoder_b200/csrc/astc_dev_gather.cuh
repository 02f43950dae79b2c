// CUDA-native ASTC: staging calls over block-list tables (astcenc_b200_compress_device_images, astcenc_b200_compress_images,
// astcenc_b200_compress_device_block_lists, astcenc_b200_compress_device_blocks). A block's 16 bytes depend on its texels after
// clamp-to-edge, the alpha-scale test over its footprint and the context - not on where it sits (void extents carry no
// coordinates, partition tables are indexed by seed). So the call's blocks are copied, footprint by footprint, into a staging
// image that is ONE ROW of blocks, an ordinary pass of the wave pipeline compresses that row, and a scatter puts each staging
// block at its payload position. The stage kernels never see the table.
//
// Staging layout of n blocks of a bx x by (x bz) footprint: (n * bx) x by texels (x bz slices for 3D block sizes), block i at
// x = i * bx. Every staged texel lies inside the staging image, so load_block reads it without clamping; the gather has done the
// clamping against the source image, exactly as load_block clamps in place (astcenc_image.cpp:162-342).
//
// Entry j of the table owns the call's staging blocks [first[j], first[j + 1]): every block of image j in payload order, or,
// when the call has lists, the capacity[j] slots of list j. Staging block c is then slot s = c - first[j] of list j: block
// indices[s] of image j while s < min(*count, capacity) and that index lies inside the image. Any other slot is invalid: the
// gather stages all-zero texels and zero alpha averages for it, which the pipeline emits as a constant block in wave 0, and the
// scatter writes nothing for it. The gather and the scatter find j by binary search over first[]. A chunk of the call
// (GatherArgs::base) may span several entries, and an entry several chunks. A host list of n blocks of one image is a one-entry
// table whose list has capacity n and *count n.
//
// A decode call (astcenc_b200_decompress_device_images) walks the same kind of table without lists: each entry's payload is
// read and its data written.
#pragma once

// One image of an image table.
struct GatherImage {
	const void* data;           // dim_z slices of dim_x * dim_y texels, contiguous
	uint8_t* payload;           // the image's whole payload
	size_t first;               // call block of the entry's first staging block (decode: of the image's block 0)
	size_t avg_offset;          // where the image's alpha-scale averages start in GatherArgs::avg_src
	unsigned int dim_x, dim_y, dim_z;
	unsigned int blocks_x, blocks_y;
};

// The list of one entry of a block-list table (beside its GatherImage).
struct GatherList {
	const uint32_t* indices;    // device: block positions in the image's payload order
	const uint32_t* count;      // device: how many of them are listed (at most `capacity` are read)
	unsigned int capacity;
	unsigned int blocks;        // the image's block count: indices at or beyond it are skipped
};

struct GatherArgs {
	void* dst;                  // the staging image
	const float* avg_src;       // alpha-scale averages of every entry's slice 0 at image positions (dim_x * dim_y each), or null
	float* avg_dst;             // the averages in the staging layout ((n * bx) x by), or null
	unsigned int n;             // staging blocks of this gather
	unsigned int words;         // 32-bit words per texel: 1 (U8), 2 (F16), 4 (F32)
	unsigned int bx, by, bz;    // footprint; bz = 1 for 2D block sizes, whose block index then counts slice z of a texture array
	// staging block i is call block base + i of the table
	const GatherImage* images;
	unsigned int image_count;
	size_t base;
	const GatherList* lists;    // one per entry, or null: every block of each image
};

#define GATHER_INVALID 0xFFFFFFFFu

// The block of slot s < capacity of list l, or GATHER_INVALID for a slot past min(*count, capacity) or an index beyond the image.
// (The slot is read together with the count: it lies inside the list's capacity either way.)
ASTC_FN uint32_t list_slot(const GatherList& l, size_t s) {
	const uint32_t count = ASTC_LDG(l.count);
	const uint32_t index = ASTC_LDG(l.indices + s);
	return s < (count < l.capacity ? count : l.capacity) && index < l.blocks ? index : GATHER_INVALID;
}

// Texel t (x fastest, then y, then z) of a staged block: where it comes from in the source image (a texel index, clamped to the
// image's edges) and where it goes in the staging image. inside: the unclamped texel lies in the image (block_has_alpha counts
// only those).
struct GatherTexel {
	size_t src, dst;
	bool inside;
};

// Texel t (x fastest, then y, then z) of the footprint of block `index` of an image of blocks_x x blocks_y blocks per layer:
// its place (tx, ty, tz) in the footprint and its image coordinates (x, y, z), unclamped: they may lie beyond the image's edges.
ASTC_FN void footprint_texel(unsigned int blocks_x, unsigned int blocks_y, unsigned int bx, unsigned int by, unsigned int bz, uint32_t index,
                             unsigned int t, unsigned int& tx, unsigned int& ty, unsigned int& tz, unsigned int& x, unsigned int& y, unsigned int& z) {
	unsigned int col = index % blocks_x;
	unsigned int rest = index / blocks_x;
	unsigned int row = rest % blocks_y;
	unsigned int layer = rest / blocks_y;
	tx = t % bx;
	ty = (t / bx) % by;
	tz = t / (bx * by);
	x = col * bx + tx, y = row * by + ty, z = layer * bz + tz;
}

// Texel t of block `index` of image im, staged as staging block i.
ASTC_FN GatherTexel gather_texel(const GatherArgs& g, const GatherImage& im, unsigned int i, uint32_t index, unsigned int t) {
	unsigned int tx, ty, tz, x, y, z;
	footprint_texel(im.blocks_x, im.blocks_y, g.bx, g.by, g.bz, index, t, tx, ty, tz, x, y, z);
	unsigned int xi = x < im.dim_x - 1 ? x : im.dim_x - 1;
	unsigned int yi = y < im.dim_y - 1 ? y : im.dim_y - 1;
	unsigned int zi = z < im.dim_z - 1 ? z : im.dim_z - 1;
	GatherTexel r;
	r.src = ((size_t)zi * im.dim_y + yi) * im.dim_x + xi;
	r.dst = ((size_t)tz * g.by + ty) * ((size_t)g.n * g.bx) + (size_t)i * g.bx + tx;
	r.inside = x < im.dim_x && y < im.dim_y;
	return r;
}

// The table entry that holds item c of a call: the last entry whose first item is at or before c (every entry has at least one
// item, so there is exactly one). The entries are images of an image table (items: call blocks), pairs of a metrics call
// (virtual CTAs) or the mapped pairs of one (map blocks).
template <typename E>
ASTC_FN unsigned int find_image(const E* images, unsigned int image_count, size_t c) {
	unsigned int lo = 0, hi = image_count - 1;
	while (lo < hi) {
		unsigned int mid = (lo + hi + 1) / 2;
		if (images[mid].first <= c) {
			lo = mid;
		} else {
			hi = mid - 1;
		}
	}
	return lo;
}

// Staging block i: the entry that holds it (j) and its block in the entry's image, or GATHER_INVALID for an invalid list slot.
ASTC_FN uint32_t staged_block(const GatherArgs& g, unsigned int i, unsigned int& j) {
	j = find_image(g.images, g.image_count, g.base + i);
	const size_t s = g.base + i - g.images[j].first;
	return g.lists != nullptr ? list_slot(g.lists[j], s) : (uint32_t)s;      // (an image has fewer than 2^32 blocks)
}

// Staging block i, by the lanes of one warp (lane / lanes): the texels word by word, so that consecutive lanes read consecutive
// words of a footprint row; then the alpha averages (0 for texels outside the image). An invalid slot stages zeros: a constant
// block, emitted in wave 0 and never scattered. The host simulation calls it with 0 / 1 or on its 32 simulated lanes.
ASTC_FN void gather_block(const GatherArgs& g, unsigned int i, int lane, int lanes) {
	unsigned int j;
	const uint32_t index = staged_block(g, i, j);
	const bool valid = index != GATHER_INVALID;
	const GatherImage im = g.images[j];      // (a copy: the stores below cannot alias it, so its fields stay in registers)
	const unsigned int T = g.bx * g.by * g.bz;
	const uint32_t* src = static_cast<const uint32_t*>(im.data);
	uint32_t* dst = static_cast<uint32_t*>(g.dst);
	for (unsigned int w = (unsigned int)lane; w < T * g.words; w += (unsigned int)lanes) {
		unsigned int t = w / g.words, k = w - t * g.words;
		GatherTexel p = gather_texel(g, im, i, valid ? index : 0, t);
		dst[p.dst * g.words + k] = valid ? ASTC_LDG(src + p.src * g.words + k) : 0u;
	}
	if (g.avg_dst != nullptr) {
		const float* avg = g.avg_src + im.avg_offset;
		for (unsigned int t = (unsigned int)lane; t < T; t += (unsigned int)lanes) {
			GatherTexel p = gather_texel(g, im, i, valid ? index : 0, t);
			g.avg_dst[p.dst] = valid && p.inside ? ASTC_LDG(avg + p.src) : 0.0f;
		}
	}
}

// Where staging block i goes in its image's payload; null for an invalid list slot.
ASTC_FN uint8_t* scatter_target(const GatherArgs& g, unsigned int i) {
	unsigned int j;
	const uint32_t index = staged_block(g, i, j);
	return index == GATHER_INVALID ? nullptr : g.images[j].payload + (size_t)index * 16;
}

// ---- image tables of a decode call (astc_decompress_images_kernel) ----
// Call block c is block c - first[j] of image j, found by find_image. decompress_block reads its image from the CTA's launch
// constants (IMG), so a CTA decodes its blocks one plane at a time and restages IMG between planes behind a barrier. A plane is
// an image of a 3D block size (its blocks count layer * blocks_y + row) or one slice of an image of a 2D block size (a texture
// array's combined row slice * blocks_y + row, with IMG.data at the slice).
//
// Call blocks [c0, c1) by the `warps` warps of one CTA; this is warp `warp` (the host simulation runs warp 0 of 1). On entry IMG
// holds the call's data type and swizzle; its pointer and dimensions are restaged here.
ASTC_FN void decode_table_blocks(const GatherImage* images, unsigned int image_count, size_t c0, size_t c1, int warp, int warps, int lane,
                                 uint32_t slice) {
	DevImage& img = reinterpret_cast<SmemHdr*>(astc_smem)->img;
	const unsigned int bz = BSD.dim_z;
	const size_t texel_bytes = img.data_type == 0 ? 4 : img.data_type == 1 ? 8 : 16;
	for (size_t c = c0; c < c1;) {
		const GatherImage& im = images[find_image(images, image_count, c)];
		const size_t plane_blocks = (size_t)im.blocks_x * im.blocks_y * (bz > 1 ? (im.dim_z + bz - 1) / bz : 1);
		const size_t plane = (c - im.first) / plane_blocks;
		const size_t p0 = im.first + plane * plane_blocks;
		const size_t end = p0 + plane_blocks < c1 ? p0 + plane_blocks : c1;
		cta_sync();      // every warp is done with the previous plane
		if (warp == 0 && lane == 0) {
			img.data = static_cast<const uint8_t*>(im.data) + plane * (size_t)im.dim_x * im.dim_y * texel_bytes;
			img.dim_x = im.dim_x;
			img.dim_y = im.dim_y;
			img.dim_z = bz > 1 ? im.dim_z : 1;
			img.blocks_x = im.blocks_x;
			img.blocks_y = im.blocks_y;
		}
		cta_sync();
		for (size_t b = c + (size_t)warp; b < end; b += (size_t)warps) {
			const unsigned int k = (unsigned int)(b - p0);      // (a plane has fewer than 2^32 blocks)
			const unsigned int by = k / im.blocks_x;
			decompress_block(lane, slice, im.payload + (b - im.first) * 16, k - by * im.blocks_x, by);
		}
		c = end;
	}
}
