// ORACLE (test infrastructure): flat C entry points for ctypes-based tests and bench.py's cpu_baseline leg.
#include "astc_codec.h"
#include <cstring>

using namespace ao;

extern "C" {

// Returns an opaque context or nullptr. `tune_overrides` may be null; otherwise 3 entries:
// {tune_partition_count_limit (0 = keep), tune_2plane_early_out_limit_correlation (<0 = keep), a_scale_radius (0 = off)}.
void* oracle_context_create(int profile, unsigned int block_x, unsigned int block_y, float quality, unsigned int flags, const float* tune_overrides) {
	Config cfg;
	if (config_init(profile, block_x, block_y, quality, flags, cfg) != 0) {
		return nullptr;
	}
	if (tune_overrides) {
		if (tune_overrides[0] > 0.0f) cfg.tune_partition_count_limit = (unsigned int)tune_overrides[0];
		if (tune_overrides[1] >= 0.0f) cfg.tune_2plane_early_out_limit_correlation = tune_overrides[1];
		if (tune_overrides[2] > 0.0f) cfg.a_scale_radius = (unsigned int)tune_overrides[2];
	}
	if (config_finalize(cfg) != 0) {
		return nullptr;
	}
	return context_create(cfg);
}

// The same for any block size: block_z > 1 selects one of the ten 3D footprints.
void* oracle_context_create_3d(int profile, unsigned int block_x, unsigned int block_y, unsigned int block_z, float quality, unsigned int flags) {
	Config cfg;
	if (config_init(profile, block_x, block_y, quality, flags, cfg, block_z) != 0) {
		return nullptr;
	}
	if (config_finalize(cfg) != 0) {
		return nullptr;
	}
	return context_create(cfg);
}

void oracle_context_destroy(void* ctx) {
	context_destroy(static_cast<Context*>(ctx));
}

// data_type: 0 = U8, 1 = F16, 2 = F32; swz = 4 ints (0..5) or null for identity. out = blocks * 16 bytes.
int oracle_compress_image(void* ctx, const void* data, int data_type, unsigned int dim_x, unsigned int dim_y, const int* swz, uint8_t* out) {
	static const int ident[4] = {0, 1, 2, 3};
	compress_image(*static_cast<Context*>(ctx), data, data_type, dim_x, dim_y, swz ? swz : ident, out);
	return 0;
}

// blocks -> image. out has dim_x * dim_y * 4 components of data_type (0 = U8, 1 = F16, 2 = F32)
int oracle_decompress_image(void* ctx, const uint8_t* data, void* out, int data_type, unsigned int dim_x, unsigned int dim_y, const int* swz) {
	static const int ident[4] = {0, 1, 2, 3};
	decompress_image(*static_cast<Context*>(ctx), data, out, data_type, dim_x, dim_y, swz ? swz : ident);
	return 0;
}

// Volumes: data / out hold dim_z slices of dim_x * dim_y texels, contiguous; blocks come out in (z, y, x) order.
int oracle_compress_volume(void* ctx, const void* data, int data_type, unsigned int dim_x, unsigned int dim_y, unsigned int dim_z, const int* swz, uint8_t* out) {
	static const int ident[4] = {0, 1, 2, 3};
	compress_image(*static_cast<Context*>(ctx), data, data_type, dim_x, dim_y, swz ? swz : ident, out, dim_z);
	return 0;
}

int oracle_decompress_volume(void* ctx, const uint8_t* data, void* out, int data_type, unsigned int dim_x, unsigned int dim_y, unsigned int dim_z, const int* swz) {
	static const int ident[4] = {0, 1, 2, 3};
	decompress_image(*static_cast<Context*>(ctx), data, out, data_type, dim_x, dim_y, swz ? swz : ident, dim_z);
	return 0;
}

// Copy the finalized config (as floats/uints in declaration order) for host-logic tests.
void oracle_get_config(void* ctx, Config* out) {
	*out = static_cast<Context*>(ctx)->config;
}

// pack_color_endpoints on n vectors. colors: 16 floats per vector (color0, color1, rgbs_color, rgbo_color);
// fmt_quant: (format, quant_level) per vector; out: 8 bytes per vector, bytes the format does not define are left as
// they are; out_format: the format used. The caller checks the inputs (finite values, quant level 4..20, a known format).
void oracle_pack_color_endpoints(unsigned int n, const float* colors, const int* fmt_quant, uint8_t* out, uint8_t* out_format) {
	for (unsigned int i = 0; i < n; i++) {
		const float* c = colors + 16 * (size_t)i;
		out_format[i] = pack_color_endpoints(mk4(c[0], c[1], c[2], c[3]), mk4(c[4], c[5], c[6], c[7]), mk4(c[8], c[9], c[10], c[11]),
		                                     mk4(c[12], c[13], c[14], c[15]), fmt_quant[2 * i], out + 8 * (size_t)i, fmt_quant[2 * i + 1]);
	}
}

}

#include "astc_error_metrics.inl"
