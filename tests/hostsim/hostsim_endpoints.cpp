// TEST TOOL (not a product path): the device source's endpoint packers (astc_dev_color.cuh, astc_dev_color_hdr_pack.cuh) on
// the host, one call over an array of vectors. Built like hostsim.cpp, with one simulated lane or with -DASTC_HOSTSIM_LANES32=1.
//   PACK_SERIAL    pack_color_endpoints, each lane its own vector (32 vectors at a time in the 32-lane build)
//   PACK_COOP      pack_rgb_endpoints_coop, every lane on the same vector
//   PACK_COOP_INL  pack_rgb_endpoints_coop_t<true>, every lane on the same vector
//   PACK_HDR       pack_hdr_endpoints, every lane on the same vector
// staged != 0 reads color_unquant_to_uquant from a copy behind the shared header (SmemHdr::cq_smem_off), else from the
// constant tables. The packers write straight into `out`, which the caller fills with a sentinel: bytes a format does not
// define must come back as they were. A result that is not the same on every lane comes back as format 0xFF.
#define ASTC_HOSTSIM 1
#if defined(ASTC_HOSTSIM_LANES32)
#include "simt_emul.h"
#endif
#include "../../astc-encoder_b200/csrc/astc_dev_core.cuh"
#include "../../astc-encoder_b200/csrc/astc_host_pack.h"
#include "../devunit/pack_endpoints_args.h"
#include <vector>

template <typename F> static void run_lanes(F fn) {
#if defined(ASTC_HOSTSIM_LANES32)
	simt::run_warp(fn);
#else
	fn(0);
#endif
}
extern "C" int hostsim_lanes() { return ASTC_WARP; }

static inline f4 vec_at(const float* c) { return mk4(c[0], c[1], c[2], c[3]); }

extern "C" int hostsim_pack_endpoints(int variant, int staged, unsigned int n, const float* colors, const int* fmt_quant, uint8_t* out, uint8_t* out_format) {
	if (pack_args_check(variant, n, colors, fmt_quant) != 0 || (n != 0 && (out == nullptr || out_format == nullptr))) {
		return 1;
	}
	DevConstTables* ct = new DevConstTables;
	astc_host::fill_dev_const_tables(*ct);
	g_astc_ct = ct;
	std::vector<uint8_t> window(ASTC_SMEM_HDR + sizeof(ct->color_unquant_to_uquant) + 16, 0xCD);
	astc_smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(window.data()) + 15) & ~(uintptr_t)15);
	SmemHdr* hdr = reinterpret_cast<SmemHdr*>(astc_smem);
	memset(hdr, 0, sizeof(SmemHdr));
	if (staged) {
		hdr->cq_smem_off = ASTC_SMEM_HDR;
		memcpy(astc_smem + ASTC_SMEM_HDR, ct->color_unquant_to_uquant, sizeof(ct->color_unquant_to_uquant));
	}
	// every lane's returned format, to check that the warp agrees
	std::vector<uint8_t> lane_fmt((size_t)ASTC_WARP * n, 0);
	run_lanes([&](int lane) {
		if (variant == PACK_SERIAL) {
			for (unsigned int i = (unsigned int)lane; i < n; i += ASTC_WARP) {
				const float* c = colors + 16 * (size_t)i;
				out_format[i] = pack_color_endpoints(vec_at(c), vec_at(c + 4), vec_at(c + 8), vec_at(c + 12), fmt_quant[2 * i], out + 8 * (size_t)i, fmt_quant[2 * i + 1]);
			}
			return;
		}
		for (unsigned int i = 0; i < n; i++) {
			const float* c = colors + 16 * (size_t)i;
			int format = fmt_quant[2 * i], q = fmt_quant[2 * i + 1];
			uint8_t* o = out + 8 * (size_t)i;
			uint8_t f;
			if (variant == PACK_COOP) {
				f = pack_rgb_endpoints_coop(lane, vec_at(c), vec_at(c + 4), format, o, q);
			} else if (variant == PACK_COOP_INL) {
				f = pack_rgb_endpoints_coop_t<true>(lane, vec_at(c), vec_at(c + 4), format, o, q);
			} else {
				f = pack_hdr_endpoints(lane, vec_at(c), vec_at(c + 4), vec_at(c + 12), format, o, q);
			}
			lane_fmt[(size_t)lane * n + i] = f;
		}
	});
	if (variant != PACK_SERIAL) {
		for (unsigned int i = 0; i < n; i++) {
			out_format[i] = lane_fmt[i];
			for (int l = 1; l < ASTC_WARP; l++) {
				if (lane_fmt[(size_t)l * n + i] != lane_fmt[i]) {
					out_format[i] = 0xFF;
				}
			}
		}
	}
	g_astc_ct = nullptr;
	astc_smem = nullptr;
	delete ct;
	return 0;
}
