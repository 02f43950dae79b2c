// CUDA-native ASTC: the alpha-scale pre-pass (SURVEY.md section 8f, second "next" row; `-a <radius>`).
//   compute_averages                 astcenc_entry.cpp:1056-1108   (32 x 32 tiles)
//   compute_pixel_region_variance    astcenc_compute_variance.cpp:103-500 (alpha lane of the 2D path)
//   brent_kung_prefix_sum            astcenc_compute_variance.cpp:52-100
// One CTA per tile: the padded tile of alpha values sits in shared memory, one thread per row (then per column) runs
// the reference's Brent-Kung prefix sum in its exact association order, then every texel reads its box sum from the
// summed-area table. Output: one float per texel; the set-up kernel turns it into "does this block have any alpha".
#pragma once

ASTC_FN void brent_kung_prefix_sum(SPtr<float> d, int items, int stride) {
	if (items < 2) {
		return;
	}
	int lc_stride = 2;
	int log2_stride = 1;
	do {
		int step = lc_stride >> 1;
		int start = lc_stride - 1;
		int iters = items >> log2_stride;
		int pos = start * stride;
		int ofs = step * stride;
		int ofs_stride = stride << log2_stride;
		ASTC_NOUNROLL
		while (iters) {
			d[pos] = d[pos] + d[pos - ofs];
			pos += ofs_stride;
			iters--;
		}
		log2_stride += 1;
		lc_stride <<= 1;
	} while (lc_stride <= items);
	do {
		log2_stride -= 1;
		lc_stride >>= 1;
		int step = lc_stride >> 1;
		int start = step + lc_stride - 1;
		int iters = (items - step) >> log2_stride;
		int pos = start * stride;
		int ofs = step * stride;
		int ofs_stride = stride << log2_stride;
		ASTC_NOUNROLL
		while (iters) {
			d[pos] = d[pos] + d[pos - ofs];
			pos += ofs_stride;
			iters--;
		}
	} while (lc_stride > 2);
}

// the alpha channel of the swizzled input texel as the averaging pass sees it (compute_variance.cpp:158-360)
ASTC_FN float alpha_for_average(const DevImage& img, unsigned int x, unsigned int y) {
	size_t o = (4 * (size_t)img.dim_x * y) + 4 * (size_t)x;
	int sa = img.swz[3];
	if (img.data_type == 0) {
		const uint8_t* p = static_cast<const uint8_t*>(img.data) + o;
		int v = sa < 4 ? (int)ASTC_LDG(&p[sa]) : (sa == 4 ? 0 : 255);
		return static_cast<float>(v) * (1.0f / 255.0f);
	}
	if (img.data_type == 1) {
		const uint16_t* p = static_cast<const uint16_t*>(img.data) + o;
		int v = sa < 4 ? (int)ASTC_LDG(&p[sa]) : (sa == 4 ? 0 : 0x3C00);
		// the reference's F16C builds saturate the packed half (astcenc_vecmathlib_sse_4.h:1001)
		return sf16_to_float((uint16_t)(v > 0x7FFF ? 0x7FFF : v));
	}
	const float* p = static_cast<const float*>(img.data) + o;
	return sa < 4 ? ASTC_LDG(&p[sa]) : (sa == 4 ? 0.0f : 1.0f);
}

#define ALPHA_TILE 32

// One tile at (ox, oy). buf = shared offset of (ALPHA_TILE + 2 r + 1)^2 floats. tid / nthreads: the calling thread's
// share of the loops (the host simulation calls it with 0 / 1).
ASTC_FN void alpha_average_tile(const DevImage& img, unsigned int radius, unsigned int ox, unsigned int oy, uint32_t buf_off, float* averages,
                                int tid, int nthreads) {
	SPtr<float> buf = sptr<float>(buf_off);
	int dim_x = (int)img.dim_x, dim_y = (int)img.dim_y;
	int r = (int)radius;
	int kerneldim = 2 * r + 1;
	int size_x = dim_x - (int)ox < ALPHA_TILE ? dim_x - (int)ox : ALPHA_TILE;
	int size_y = dim_y - (int)oy < ALPHA_TILE ? dim_y - (int)oy : ALPHA_TILE;
	int padsize_x = size_x + kerneldim, padsize_y = size_y + kerneldim;
	int yst = padsize_x;
	ASTC_NOUNROLL
	for (int i = tid; i < padsize_x * padsize_y; i += nthreads) {
		int y = i / padsize_x, x = i - y * padsize_x;
		float v = 0.0f;               // row 0 and column 0 are the zero edge of the table
		if (x != 0 && y != 0) {
			int y_src = (y - 1) + (int)oy;
			y_src = y_src <= r ? 0 : y_src - r;
			y_src = y_src < dim_y - 1 ? y_src : dim_y - 1;
			int x_src = (x - 1) + (int)ox;
			x_src = x_src <= r ? 0 : x_src - r;
			x_src = x_src < dim_x - 1 ? x_src : dim_x - 1;
			v = alpha_for_average(img, (unsigned int)x_src, (unsigned int)y_src);
		}
		buf[i] = v;
	}
	cta_sync();
	ASTC_NOUNROLL
	for (int y = 1 + tid; y < padsize_y; y += nthreads) {
		brent_kung_prefix_sum(buf + (y * yst + 1), padsize_x - 1, 1);
	}
	cta_sync();
	ASTC_NOUNROLL
	for (int x = 1 + tid; x < padsize_x; x += nthreads) {
		brent_kung_prefix_sum(buf + (yst + x), padsize_y - 1, yst);
	}
	cta_sync();
	float alpha_kdim = static_cast<float>(2 * radius + 1);
	float alpha_rsamples = 1.0f / (alpha_kdim * alpha_kdim);
	ASTC_NOUNROLL
	for (int i = tid; i < size_x * size_y; i += nthreads) {
		int y = i / size_x, x = i - y * size_x;
		int y_low = y, y_high = y + 2 * r + 1;        // (y + r) -/+ r (+ 1)
		int x_low = x, x_high = x + 2 * r + 1;
		float vasum = buf[y_low * yst + x_low] - buf[y_low * yst + x_high] - buf[y_high * yst + x_low] + buf[y_high * yst + x_high];
		averages[(size_t)(y + (int)oy) * img.dim_x + (size_t)(x + (int)ox)] = vasum * alpha_rsamples;
	}
	cta_sync();
}

// The pre-pass window of image rows [y0, y1) (a slab's rows, y0 < y1 <= dim_y): tile rows [tile_row0, tile_row0 + tile_rows) of
// the 32 x 32 grid cover them, and those tiles read image rows [read_row0, read_row1). The grid stays anchored at (0, 0) for
// every slab: a texel's average depends on its whole padded tile (the prefix sums' association order follows padsize), so a
// shifted grid would change the bytes. A pass over the slab needs the averages of its own texels only, which the window's
// tiles write; outside the read rows the image may hold anything.
struct AlphaWindow {
	unsigned int tile_row0, tile_rows;
	unsigned int read_row0, read_row1;
};

static inline AlphaWindow alpha_window(unsigned int dim_y, unsigned int radius, unsigned int y0, unsigned int y1) {
	AlphaWindow w;
	unsigned int t1 = (y1 + ALPHA_TILE - 1) / ALPHA_TILE;
	w.tile_row0 = y0 / ALPHA_TILE;
	w.tile_rows = t1 - w.tile_row0;
	// alpha_average_tile clamps its source rows to [0, dim_y - 1]: the first tile reads from oy - r, the last up to oy + size_y + r - 1
	size_t lo = (size_t)w.tile_row0 * ALPHA_TILE, hi = (size_t)t1 * ALPHA_TILE + radius;
	w.read_row0 = lo > radius ? (unsigned int)(lo - radius) : 0u;
	w.read_row1 = hi < dim_y ? (unsigned int)hi : dim_y;
	return w;
}

// Alpha-scale RDO test of one block (astcenc_entry.cpp:973-1003): false = no texel of the block has an alpha average above
// the threshold, the block is emitted as constant zero without looking at it.
ASTC_FN bool block_has_alpha(const WCtx& w, const float* averages, float threshold, unsigned int pos_x, unsigned int pos_y) {
	const DevImage& img = IMG;
	unsigned int bx = BSD.dim_x;
	bool any = false;
	ASTC_NOUNROLL
	for (int t = w.lane; t < w.T; t += ASTC_WARP) {
		unsigned int x = pos_x + (unsigned int)t % bx, y = pos_y + (unsigned int)t / bx;
		if (x < img.dim_x && y < img.dim_y) {
			any = any || ASTC_LDG(&averages[(size_t)y * img.dim_x + x]) > threshold;
		}
	}
	return wany(any);
}
