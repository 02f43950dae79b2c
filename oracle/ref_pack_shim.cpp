// Reference-side shim (checker only): exposes the reference's pack_color_endpoints() - an internal function of the
// UNMODIFIED astcenc_color_quantize.cpp (declared in astcenc_internal.h) - as a C symbol over arrays of inputs. oracle/Makefile
// links it against the reference's own objects into oracle/_ref/libastcenc_ref_pack.so.
#include "astcenc_internal.h"

// colors: 16 floats per vector (color0, color1, rgbs_color, rgbo_color); fmt_quant: (format, quant_level) per vector;
// out: 8 bytes per vector (bytes the format does not define are left as they are); out_format: the format used.
extern "C" __attribute__((visibility("default")))
void ref_pack_color_endpoints(unsigned int n, const float* colors, const int* fmt_quant, uint8_t* out, uint8_t* out_format) {
	for (unsigned int i = 0; i < n; i++) {
		const float* c = colors + 16 * (size_t)i;
		out_format[i] = pack_color_endpoints(vfloat4(c[0], c[1], c[2], c[3]), vfloat4(c[4], c[5], c[6], c[7]), vfloat4(c[8], c[9], c[10], c[11]),
		                                     vfloat4(c[12], c[13], c[14], c[15]), fmt_quant[2 * i], out + 8 * (size_t)i,
		                                     static_cast<quant_method>(fmt_quant[2 * i + 1]));
	}
}
