// TEST TOOL: the argument check shared by the two harnesses that run the device source's endpoint packers on arrays of
// vectors (tests/hostsim/hostsim_endpoints.cpp on the host, tests/devunit/pack_endpoints.cu on the GPU).
//
// Vector i: colors[16 i .. 16 i + 15] = color0, color1, rgbs_color, rgbo_color; fmt_quant[2 i], [2 i + 1] = format, quant level.
// A non-finite input makes f2i_rtn return INT_MIN and the table look-ups index outside color_unquant_to_uquant, so such inputs,
// quant levels outside QUANT_6..QUANT_256 and formats the variant does not pack are refused before anything runs.
#pragma once
#include <cmath>
#include <cstdint>

enum PackVariant {
	PACK_SERIAL = 0,      // pack_color_endpoints: one vector per lane, the LDR formats of multi-partition candidates
	PACK_COOP = 1,        // pack_rgb_endpoints_coop (pack_rgb_endpoints_coop_t<false>): RGB / RGBA, one vector per warp
	PACK_COOP_INL = 2,    // pack_rgb_endpoints_coop_t<true>: the same, inlined (one-partition LDR paths)
	PACK_HDR = 3,         // pack_hdr_endpoints: the HDR formats, one vector per warp
	PACK_VARIANTS = 4
};

static inline bool pack_format_allowed(int variant, int format) {
	switch (variant) {
	case PACK_SERIAL:
		return format == 0 || format == 4 || format == 6 || format == 8 || format == 10 || format == 12;
	case PACK_COOP:
	case PACK_COOP_INL:
		return format == 8 || format == 12;
	case PACK_HDR:
		return format == 2 || format == 3 || format == 7 || format == 11 || format == 14 || format == 15;
	default:
		return false;
	}
}

// 0 when every vector can be packed by `variant`, else 1
static inline int pack_args_check(int variant, unsigned int n, const float* colors, const int* fmt_quant) {
	if (variant < 0 || variant >= PACK_VARIANTS || (n != 0 && (colors == nullptr || fmt_quant == nullptr))) {
		return 1;
	}
	for (unsigned int i = 0; i < n; i++) {
		for (int j = 0; j < 16; j++) {
			if (!std::isfinite(colors[16 * (size_t)i + j])) {
				return 1;
			}
		}
		int q = fmt_quant[2 * (size_t)i + 1];
		if (q < 4 || q > 20 || !pack_format_allowed(variant, fmt_quant[2 * (size_t)i])) {
			return 1;
		}
	}
	return 0;
}
