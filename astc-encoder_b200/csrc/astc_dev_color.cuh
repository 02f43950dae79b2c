// Device-side colour endpoint quantisation / unquantisation (one lane per partition).
//   pack side   : astcenc_color_quantize.cpp:72-1909 (LDR formats here; HDR formats in astc_dev_color_hdr_pack.cuh)
//   unpack side : astcenc_color_unquantize.cpp:61-1022
#pragma once

enum {
	FMT_LUMINANCE = 0, FMT_LUMINANCE_DELTA = 1, FMT_HDR_LUMINANCE_LARGE_RANGE = 2, FMT_HDR_LUMINANCE_SMALL_RANGE = 3,
	FMT_LUMINANCE_ALPHA = 4, FMT_LUMINANCE_ALPHA_DELTA = 5, FMT_RGB_SCALE = 6, FMT_HDR_RGB_SCALE = 7,
	FMT_RGB = 8, FMT_RGB_DELTA = 9, FMT_RGB_SCALE_ALPHA = 10, FMT_HDR_RGB = 11,
	FMT_RGBA = 12, FMT_RGBA_DELTA = 13, FMT_HDR_RGB_LDR_ALPHA = 14, FMT_HDR_RGBA = 15
};

enum { PRF_LDR_SRGB = 0, PRF_LDR = 1, PRF_HDR_RGB_LDR_A = 2, PRF_HDR = 3 };

// ---------------------------------------------------------------------------------------------
// Unpack (astcenc_color_unquantize.cpp)
// ---------------------------------------------------------------------------------------------
ASTC_FN i4 uncontract_color(i4 in) {          // :33-40 lanes r,g <- (c + b) >> 1
	return mki4((in.x + in.z) >> 1, (in.y + in.z) >> 1, in.z, in.w);
}

ASTC_FN void bit_transfer_signed1(int& in0, int& in1) {   // astcenc_vecmathlib_common_4.h:367-380
	in1 = (int)((unsigned int)in1 >> 1) | (in0 & 0x80);
	in0 = (int)((unsigned int)in0 >> 1) & 0x3F;
	if (in0 & 0x20) {
		in0 = in0 - 0x40;
	}
}

ASTC_FN void bit_transfer_signed4(i4& a, i4& b) {
	bit_transfer_signed1(a.x, b.x);
	bit_transfer_signed1(a.y, b.y);
	bit_transfer_signed1(a.z, b.z);
	bit_transfer_signed1(a.w, b.w);
}

ASTC_FN void rgba_delta_unpack(i4 in0, i4 in1, i4& out0, i4& out1) {   // :61-102
	bit_transfer_signed4(in1, in0);
	int rgb_sum = in1.x + in1.y + in1.z;
	in1 = mki4(in1.x + in0.x, in1.y + in0.y, in1.z + in0.z, in1.w + in0.w);
	if (rgb_sum < 0) {
		in0 = uncontract_color(in0);
		in1 = uncontract_color(in1);
		i4 t = in0; in0 = in1; in1 = t;
	}
	out0 = mki4(clampi(in0.x, 0, 255), clampi(in0.y, 0, 255), clampi(in0.z, 0, 255), clampi(in0.w, 0, 255));
	out1 = mki4(clampi(in1.x, 0, 255), clampi(in1.y, 0, 255), clampi(in1.z, 0, 255), clampi(in1.w, 0, 255));
}

ASTC_FN void rgba_unpack(i4 in0, i4 in1, i4& out0, i4& out1) {   // :105-135
	if ((in0.x + in0.y + in0.z) > (in1.x + in1.y + in1.z)) {
		in0 = uncontract_color(in0);
		in1 = uncontract_color(in1);
		i4 t = in0; in0 = in1; in1 = t;
	}
	out0 = in0;
	out1 = in1;
}

#include "astc_dev_color_hdr_unpack.cuh"

// unpack_color_endpoints (astcenc_color_unquantize.cpp:844-1022)
// (the _inl form lets a caller keep the results in registers: reference parameters of an out-of-line function force the
// caller's variables into local memory)
// LDR_ONLY: the caller decodes in an LDR profile, so the HDR unpackers are left out. An HDR format still ends as the error
// colour below, exactly as in the general form (an LDR decode replaces any HDR endpoint pair by it).
template <bool LDR_ONLY = false>
ASTC_FN void unpack_color_endpoints_inl(int decode_mode, int format, const uint8_t* in, bool& rgb_hdr, bool& alpha_hdr, i4& o0, i4& o1) {
	rgb_hdr = false;
	alpha_hdr = false;
	bool alpha_hdr_default = false;
	switch (format) {
	case FMT_LUMINANCE:
		o0 = mki4(in[0], in[0], in[0], 255);
		o1 = mki4(in[1], in[1], in[1], 255);
		break;
	case FMT_LUMINANCE_DELTA: {
		int v0 = in[0], v1 = in[1];
		int l0 = (v0 >> 2) | (v1 & 0xC0);
		int l1 = l0 + (v1 & 0x3F);
		l1 = mini(l1, 255);
		o0 = mki4(l0, l0, l0, 255);
		o1 = mki4(l1, l1, l1, 255);
		break;
	}
	case FMT_HDR_LUMINANCE_SMALL_RANGE:
		if (LDR_ONLY) { rgb_hdr = true; o0 = o1 = mki4(0, 0, 0, 0); break; }
		rgb_hdr = true;
		alpha_hdr_default = true;
		hdr_luminance_small_range_unpack(in, o0, o1);
		break;
	case FMT_HDR_LUMINANCE_LARGE_RANGE:
		if (LDR_ONLY) { rgb_hdr = true; o0 = o1 = mki4(0, 0, 0, 0); break; }
		rgb_hdr = true;
		alpha_hdr_default = true;
		hdr_luminance_large_range_unpack(in, o0, o1);
		break;
	case FMT_LUMINANCE_ALPHA:
		o0 = mki4(in[0], in[0], in[0], in[2]);
		o1 = mki4(in[1], in[1], in[1], in[3]);
		break;
	case FMT_LUMINANCE_ALPHA_DELTA: {
		int lum0 = in[0], lum1 = in[1], alpha0 = in[2], alpha1 = in[3];
		lum0 |= (lum1 & 0x80) << 1;
		alpha0 |= (alpha1 & 0x80) << 1;
		lum1 &= 0x7F;
		alpha1 &= 0x7F;
		if (lum1 & 0x40) lum1 -= 0x80;
		if (alpha1 & 0x40) alpha1 -= 0x80;
		lum0 >>= 1;
		lum1 >>= 1;
		alpha0 >>= 1;
		alpha1 >>= 1;
		lum1 += lum0;
		alpha1 += alpha0;
		lum1 = clampi(lum1, 0, 255);
		alpha1 = clampi(alpha1, 0, 255);
		o0 = mki4(lum0, lum0, lum0, alpha0);
		o1 = mki4(lum1, lum1, lum1, alpha1);
		break;
	}
	case FMT_RGB_SCALE: {
		int scale = in[3];
		o1 = mki4(in[0], in[1], in[2], 255);
		o0 = mki4((in[0] * scale) >> 8, (in[1] * scale) >> 8, (in[2] * scale) >> 8, 255);
		break;
	}
	case FMT_RGB_SCALE_ALPHA: {
		int scale = in[3];
		o1 = mki4(in[0], in[1], in[2], in[5]);
		o0 = mki4((in[0] * scale) >> 8, (in[1] * scale) >> 8, (in[2] * scale) >> 8, in[4]);
		break;
	}
	case FMT_HDR_RGB_SCALE:
		if (LDR_ONLY) { rgb_hdr = true; o0 = o1 = mki4(0, 0, 0, 0); break; }
		rgb_hdr = true;
		alpha_hdr_default = true;
		hdr_rgbo_unpack(in, o0, o1);
		break;
	case FMT_RGB:
		rgba_unpack(mki4(in[0], in[2], in[4], 0), mki4(in[1], in[3], in[5], 0), o0, o1);
		o0.w = 255;
		o1.w = 255;
		break;
	case FMT_RGB_DELTA:
		rgba_delta_unpack(mki4(in[0], in[2], in[4], 0), mki4(in[1], in[3], in[5], 0), o0, o1);
		o0.w = 255;
		o1.w = 255;
		break;
	case FMT_HDR_RGB:
		if (LDR_ONLY) { rgb_hdr = true; o0 = o1 = mki4(0, 0, 0, 0); break; }
		rgb_hdr = true;
		alpha_hdr_default = true;
		hdr_rgb_unpack(in, o0, o1);
		break;
	case FMT_RGBA:
		rgba_unpack(mki4(in[0], in[2], in[4], in[6]), mki4(in[1], in[3], in[5], in[7]), o0, o1);
		break;
	case FMT_RGBA_DELTA:
		rgba_delta_unpack(mki4(in[0], in[2], in[4], in[6]), mki4(in[1], in[3], in[5], in[7]), o0, o1);
		break;
	case FMT_HDR_RGB_LDR_ALPHA:
		if (LDR_ONLY) { rgb_hdr = true; o0 = o1 = mki4(0, 0, 0, 0); break; }
		rgb_hdr = true;
		hdr_rgb_unpack(in, o0, o1);
		o0.w = in[6];
		o1.w = in[7];
		break;
	case FMT_HDR_RGBA: {
		if (LDR_ONLY) { rgb_hdr = true; o0 = o1 = mki4(0, 0, 0, 0); break; }
		rgb_hdr = true;
		alpha_hdr = true;
		hdr_rgb_unpack(in, o0, o1);
		int a0, a1;
		hdr_alpha_unpack(in + 6, a0, a1);
		o0.w = a0;
		o1.w = a1;
		break;
	}
	}
	if (alpha_hdr_default) {
		if (decode_mode == PRF_HDR) {
			o0.w = 0x7800;
			o1.w = 0x7800;
			alpha_hdr = true;
		} else {
			o0.w = 0x00FF;
			o1.w = 0x00FF;
			alpha_hdr = false;
		}
	}
	if (decode_mode == PRF_LDR) {
		if (rgb_hdr || alpha_hdr) {
			o0 = mki4(0xFF, 0x00, 0xFF, 0xFF);
			o1 = mki4(0xFF, 0x00, 0xFF, 0xFF);
			rgb_hdr = false;
			alpha_hdr = false;
		}
		o0 = mki4(o0.x * 257, o0.y * 257, o0.z * 257, o0.w * 257);
		o1 = mki4(o1.x * 257, o1.y * 257, o1.z * 257, o1.w * 257);
	} else if (decode_mode == PRF_LDR_SRGB) {
		if (rgb_hdr || alpha_hdr) {
			o0 = mki4(0xFF, 0x00, 0xFF, 0xFF);
			o1 = mki4(0xFF, 0x00, 0xFF, 0xFF);
			rgb_hdr = false;
			alpha_hdr = false;
		}
		o0 = mki4((o0.x << 8) | 0x80, (o0.y << 8) | 0x80, (o0.z << 8) | 0x80, (o0.w << 8) | 0x80);
		o1 = mki4((o1.x << 8) | 0x80, (o1.y << 8) | 0x80, (o1.z << 8) | 0x80, (o1.w << 8) | 0x80);
	} else {
		int sr = rgb_hdr ? 1 : 257;
		int sa = alpha_hdr ? 1 : 257;
		o0 = mki4(o0.x * sr, o0.y * sr, o0.z * sr, o0.w * sa);
		o1 = mki4(o1.x * sr, o1.y * sr, o1.z * sr, o1.w * sa);
	}
}

ASTC_NOINLINE void unpack_color_endpoints(int decode_mode, int format, const uint8_t* in, bool& rgb_hdr, bool& alpha_hdr, i4& o0, i4& o1) {
	unpack_color_endpoints_inl(decode_mode, format, in, rgb_hdr, alpha_hdr, o0, o1);
}

// ---------------------------------------------------------------------------------------------
// Pack (astcenc_color_quantize.cpp)
// ---------------------------------------------------------------------------------------------
struct QuantCtx {
	const uint8_t* tab;   // color_unquant_to_uquant[quant_level - QUANT_6]
	int quant_level;
};

ASTC_FN int quant_color(QuantCtx q, int value) {   // :72-79 (round to nearest, ties up)
	return q.tab[value * 2 + 1];
}
ASTC_FN int quant_color_f(QuantCtx q, int value, float valuef) {   // :109-126
	int index = value * 2;
	float residual = valuef - static_cast<float>(value);
	if (residual >= -0.1f) {
		index++;
	}
	return q.tab[index];
}
ASTC_FN i4 quant_color3(QuantCtx q, i4 v) {
	return mki4(quant_color(q, v.x), quant_color(q, v.y), quant_color(q, v.z), 0);
}
ASTC_FN i4 quant_color3_f(QuantCtx q, i4 v, f4 vf) {
	return mki4(quant_color_f(q, v.x, vf.x), quant_color_f(q, v.y, vf.y), quant_color_f(q, v.z, vf.z), 0);
}
ASTC_FN i4 f4_to_i4_rtn(f4 a) { return mki4(f2i_rtn(a.x), f2i_rtn(a.y), f2i_rtn(a.z), f2i_rtn(a.w)); }

ASTC_FN float get_rgba_encoding_error(f4 uq0, f4 uq1, i4 q0, i4 q1) {   // :50-60
	f4 e0 = uq0 - mk4((float)q0.x, (float)q0.y, (float)q0.z, (float)q0.w);
	f4 e1 = uq1 - mk4((float)q1.x, (float)q1.y, (float)q1.z, (float)q1.w);
	return hadd_s(e0 * e0 + e1 * e1);
}

// Results of the out-of-line quantisers come back BY VALUE (registers); the inline wrappers below keep the reference
// style of the reference code without forcing the caller's endpoints into local memory.
struct QEnds {
	i4 a, b;
	bool ok;
};

// (each out-of-line quantiser below is also instantiated inline, _inl, by the one-partition LDR refinement step)
ASTC_FN QEnds quantize_rgb_inl(f4 c0, f4 c1, QuantCtx q) {   // :169-193
	i4 c0i, c1i;
	do {
		i4 a = f4_to_i4_rtn(c0);
		i4 c0q = mki4(maxi(a.x, 0), maxi(a.y, 0), maxi(a.z, 0), maxi(a.w, 0));
		c0i = quant_color3_f(q, c0q, c0);
		c0 = c0 - splat4(0.2f);
		i4 b = f4_to_i4_rtn(c1);
		i4 c1q = mki4(mini(b.x, 255), mini(b.y, 255), mini(b.z, 255), mini(b.w, 255));
		c1i = quant_color3_f(q, c1q, c1);
		c1 = c1 + splat4(0.2f);
	} while ((c0i.x + c0i.y + c0i.z) > (c1i.x + c1i.y + c1i.z));
	QEnds r;
	r.a = c0i;
	r.b = c1i;
	r.ok = true;
	return r;
}
ASTC_NOINLINE QEnds quantize_rgb_v(f4 c0, f4 c1, QuantCtx q) { return quantize_rgb_inl(c0, c1, q); }
ASTC_FN void quantize_rgb(f4 c0, f4 c1, i4& o0, i4& o1, QuantCtx q) {
	QEnds r = quantize_rgb_v(c0, c1, q);
	o0 = r.a;
	o1 = r.b;
}

ASTC_FN void quantize_rgba(f4 c0, f4 c1, i4& o0, i4& o1, QuantCtx q) {   // :207-220
	quantize_rgb(c0, c1, o0, o1, q);
	o0.w = quant_color_f(q, f2i_rtn(c0.w), c0.w);
	o1.w = quant_color_f(q, f2i_rtn(c1.w), c1.w);
}

ASTC_FN bool in_0_255(f4 c) {
	// any((c < 0) | (c > 255)) over all four lanes
	return !((c.x < 0.0f) || (c.x > 255.0f) || (c.y < 0.0f) || (c.y > 255.0f) ||
	         (c.z < 0.0f) || (c.z > 255.0f) || (c.w < 0.0f) || (c.w > 255.0f));
}

ASTC_FN f4 blue_contract_fwd(f4 c) {   // c += c - c.bbba
	return mk4(c.x + (c.x - c.z), c.y + (c.y - c.z), c.z + (c.z - c.z), c.w + (c.w - c.w));
}

ASTC_FN QEnds try_quantize_rgb_blue_contract_inl(f4 c0, f4 c1, QuantCtx q) {   // :237-267
	QEnds r;
	r.a = r.b = mki4(0, 0, 0, 0);
	r.ok = false;
	c0 = blue_contract_fwd(c0);
	c1 = blue_contract_fwd(c1);
	if (!in_0_255(c0) || !in_0_255(c1)) {
		return r;
	}
	i4 c0i = quant_color3_f(q, f4_to_i4_rtn(c0), c0);
	i4 c1i = quant_color3_f(q, f4_to_i4_rtn(c1), c1);
	if ((c1i.x + c1i.y + c1i.z) <= (c0i.x + c0i.y + c0i.z)) {
		return r;
	}
	r.a = c1i;
	r.b = c0i;
	r.ok = true;
	return r;
}
ASTC_NOINLINE QEnds try_quantize_rgb_blue_contract_v(f4 c0, f4 c1, QuantCtx q) { return try_quantize_rgb_blue_contract_inl(c0, c1, q); }
// (a failed attempt leaves o0 / o1 untouched, like the reference)
ASTC_FN bool try_quantize_rgb_blue_contract(f4 c0, f4 c1, i4& o0, i4& o1, QuantCtx q) {
	QEnds r = try_quantize_rgb_blue_contract_v(c0, c1, q);
	if (r.ok) {
		o0 = r.a;
		o1 = r.b;
	}
	return r.ok;
}

ASTC_FN bool try_quantize_rgba_blue_contract(f4 c0, f4 c1, i4& o0, i4& o1, QuantCtx q) {   // :283-303
	if (try_quantize_rgb_blue_contract(c0, c1, o0, o1, q)) {
		o0.w = quant_color_f(q, f2i_rtn(c1.w), c1.w);
		o1.w = quant_color_f(q, f2i_rtn(c0.w), c0.w);
		return true;
	}
	return false;
}

// common body of try_quantize_rgb_delta (:321-400) and ..._delta_blue_contract (:403-488)
ASTC_FN QEnds rgb_delta_core_inl(f4 c0, f4 c1, QuantCtx q, bool want_negative_sum) {
	QEnds res;
	res.a = res.b = mki4(0, 0, 0, 0);
	res.ok = false;
	i4 c0a = f4_to_i4_rtn(c0);
	c0a = mki4(c0a.x << 1, c0a.y << 1, c0a.z << 1, c0a.w << 1);
	i4 c0b = mki4(c0a.x & 0xFF, c0a.y & 0xFF, c0a.z & 0xFF, c0a.w & 0xFF);
	i4 c0be = quant_color3(q, c0b);
	c0b = mki4(c0be.x | (c0a.x & 0x100), c0be.y | (c0a.y & 0x100), c0be.z | (c0a.z & 0x100), c0be.w | (c0a.w & 0x100));
	i4 c1d = f4_to_i4_rtn(c1);
	c1d = mki4((c1d.x << 1) - c0b.x, (c1d.y << 1) - c0b.y, (c1d.z << 1) - c0b.z, 0);
	if (c1d.x > 63 || c1d.x < -64 || c1d.y > 63 || c1d.y < -64 || c1d.z > 63 || c1d.z < -64) {
		return res;
	}
	c1d = mki4((c1d.x & 0x7F) | ((c0b.x & 0x100) >> 1), (c1d.y & 0x7F) | ((c0b.y & 0x100) >> 1),
	           (c1d.z & 0x7F) | ((c0b.z & 0x100) >> 1), (c1d.w & 0x7F) | ((c0b.w & 0x100) >> 1));
	i4 c1de = quant_color3(q, c1d);
	if ((((c1d.x ^ c1de.x) | (c1d.y ^ c1de.y) | (c1d.z ^ c1de.z)) & 0xC0) != 0) {
		return res;
	}
	i4 ep0 = c0be;
	i4 ep1 = c1de;
	bit_transfer_signed4(ep1, ep0);
	int sum = ep1.x + ep1.y + ep1.z;
	if (want_negative_sum ? (sum >= 0) : (sum < 0)) {
		return res;
	}
	ep0 = mki4(ep0.x + ep1.x, ep0.y + ep1.y, ep0.z + ep1.z, ep0.w + ep1.w);
	if (ep0.x < 0 || ep0.x > 0xFF || ep0.y < 0 || ep0.y > 0xFF || ep0.z < 0 || ep0.z > 0xFF || ep0.w < 0 || ep0.w > 0xFF) {
		return res;
	}
	res.a = c0be;
	res.b = c1de;
	res.ok = true;
	return res;
}
ASTC_NOINLINE QEnds rgb_delta_core_v(f4 c0, f4 c1, QuantCtx q, bool want_negative_sum) { return rgb_delta_core_inl(c0, c1, q, want_negative_sum); }
ASTC_FN bool rgb_delta_core(f4 c0, f4 c1, i4& o0, i4& o1, QuantCtx q, bool want_negative_sum) {
	QEnds r = rgb_delta_core_v(c0, c1, q, want_negative_sum);
	if (r.ok) {
		o0 = r.a;
		o1 = r.b;
	}
	return r.ok;
}

ASTC_FN bool try_quantize_rgb_delta(f4 c0, f4 c1, i4& o0, i4& o1, QuantCtx q) {
	return rgb_delta_core(c0, c1, o0, o1, q, false);
}

ASTC_FN bool try_quantize_rgb_delta_blue_contract(f4 c0, f4 c1, i4& o0, i4& o1, QuantCtx q) {
	f4 t = c0; c0 = c1; c1 = t;
	c0 = blue_contract_fwd(c0);
	c1 = blue_contract_fwd(c1);
	if (!in_0_255(c0) || !in_0_255(c1)) {
		return false;
	}
	return rgb_delta_core(c0, c1, o0, o1, q, true);
}

struct QAlpha {
	int a0, a1;
	bool ok;
};
ASTC_FN QAlpha try_quantize_alpha_delta_inl(f4 c0, f4 c1, QuantCtx q) {   // :504-570
	QAlpha res;
	res.a0 = res.a1 = 0;
	res.ok = false;
	float a0 = c0.w, a1 = c1.w;
	int a0a = f2i_rtn(a0);
	a0a <<= 1;
	int a0b = a0a & 0xFF;
	int a0be = quant_color(q, a0b);
	a0b = a0be;
	a0b |= a0a & 0x100;
	int a1d = f2i_rtn(a1);
	a1d <<= 1;
	a1d -= a0b;
	if (a1d > 63 || a1d < -64) {
		return res;
	}
	a1d &= 0x7F;
	a1d |= (a0b & 0x100) >> 1;
	int a1de = quant_color(q, a1d);
	int a1du = a1de;
	if ((a1d ^ a1du) & 0xC0) {
		return res;
	}
	a1du &= 0x7F;
	if (a1du & 0x40) {
		a1du -= 0x80;
	}
	a1du += a0b;
	if (a1du < 0 || a1du > 0x1FF) {
		return res;
	}
	res.a0 = a0be;
	res.a1 = a1de;
	res.ok = true;
	return res;
}
ASTC_NOINLINE QAlpha try_quantize_alpha_delta_v(f4 c0, f4 c1, QuantCtx q) { return try_quantize_alpha_delta_inl(c0, c1, q); }
ASTC_FN bool try_quantize_alpha_delta(f4 c0, f4 c1, i4& o0, i4& o1, QuantCtx q) {
	QAlpha r = try_quantize_alpha_delta_v(c0, c1, q);
	if (r.ok) {
		o0.w = r.a0;
		o1.w = r.a1;
	}
	return r.ok;
}

ASTC_NOINLINE bool try_quantize_luminance_alpha_delta(f4 c0, f4 c1, uint8_t out[4], QuantCtx q) {   // :573-694
	float l0 = hadd_rgb_s(c0) * (1.0f / 3.0f);
	float l1 = hadd_rgb_s(c1) * (1.0f / 3.0f);
	float a0 = c0.w, a1 = c1.w;
	int l0a = f2i_rtn(l0), a0a = f2i_rtn(a0);
	l0a <<= 1;
	a0a <<= 1;
	int l0b = l0a & 0xFF, a0b = a0a & 0xFF;
	int l0be = quant_color(q, l0b), a0be = quant_color(q, a0b);
	l0b = l0be;
	a0b = a0be;
	l0b |= l0a & 0x100;
	a0b |= a0a & 0x100;
	int l1d = f2i_rtn(l1), a1d = f2i_rtn(a1);
	l1d <<= 1;
	a1d <<= 1;
	l1d -= l0b;
	a1d -= a0b;
	if (l1d > 63 || l1d < -64) return false;
	if (a1d > 63 || a1d < -64) return false;
	l1d &= 0x7F;
	a1d &= 0x7F;
	l1d |= (l0b & 0x100) >> 1;
	a1d |= (a0b & 0x100) >> 1;
	int l1de = quant_color(q, l1d), a1de = quant_color(q, a1d);
	int l1du = l1de, a1du = a1de;
	if ((l1d ^ l1du) & 0xC0) return false;
	if ((a1d ^ a1du) & 0xC0) return false;
	l1du &= 0x7F;
	a1du &= 0x7F;
	if (l1du & 0x40) l1du -= 0x80;
	if (a1du & 0x40) a1du -= 0x80;
	l1du += l0b;
	a1du += a0b;
	if (l1du < 0 || l1du > 0x1FF) return false;
	if (a1du < 0 || a1du > 0x1FF) return false;
	out[0] = (uint8_t)l0be;
	out[1] = (uint8_t)l1de;
	out[2] = (uint8_t)a0be;
	out[3] = (uint8_t)a1de;
	return true;
}

ASTC_NOINLINE void quantize_rgbs(f4 color, uint8_t out[4], QuantCtx q) {   // :734-763
	float scale = 1.0f / 257.0f;
	float r = clampf(color.x * scale, 0.0f, 255.0f);
	float g = clampf(color.y * scale, 0.0f, 255.0f);
	float b = clampf(color.z * scale, 0.0f, 255.0f);
	int ri = quant_color_f(q, f2i_rtn(r), r);
	int gi = quant_color_f(q, f2i_rtn(g), g);
	int bi = quant_color_f(q, f2i_rtn(b), b);
	float oldcolorsum = hadd_rgb_s(color) * scale;
	float newcolorsum = static_cast<float>(ri + gi + bi);
	float scalea = clamp1f(color.w * (oldcolorsum + 1e-10f) / (newcolorsum + 1e-10f));
	int scale_idx = f2i_rtn(scalea * 256.0f);
	scale_idx = clampi(scale_idx, 0, 255);
	out[0] = (uint8_t)ri;
	out[1] = (uint8_t)gi;
	out[2] = (uint8_t)bi;
	out[3] = (uint8_t)quant_color(q, scale_idx);
}

ASTC_FN void quantize_luminance(f4 c0, f4 c1, uint8_t out[2], QuantCtx q) {   // :795-815
	float lum0 = hadd_rgb_s(c0) * (1.0f / 3.0f);
	float lum1 = hadd_rgb_s(c1) * (1.0f / 3.0f);
	if (lum0 > lum1) {
		float avg = (lum0 + lum1) * 0.5f;
		lum0 = avg;
		lum1 = avg;
	}
	out[0] = (uint8_t)quant_color_f(q, f2i_rtn(lum0), lum0);
	out[1] = (uint8_t)quant_color_f(q, f2i_rtn(lum1), lum1);
}

ASTC_FN void quantize_luminance_alpha(f4 c0, f4 c1, uint8_t out[4], QuantCtx q) {   // :828-846
	float lum0 = hadd_rgb_s(c0) * (1.0f / 3.0f);
	float lum1 = hadd_rgb_s(c1) * (1.0f / 3.0f);
	out[0] = (uint8_t)quant_color_f(q, f2i_rtn(lum0), lum0);
	out[1] = (uint8_t)quant_color_f(q, f2i_rtn(lum1), lum1);
	out[2] = (uint8_t)quant_color_f(q, f2i_rtn(c0.w), c0.w);
	out[3] = (uint8_t)quant_color_f(q, f2i_rtn(c1.w), c1.w);
}

#include "astc_dev_color_hdr_pack.cuh"

// pack_color_endpoints (astcenc_color_quantize.cpp:1909-2147)
ASTC_NOINLINE uint8_t pack_color_endpoints(f4 color0, f4 color1, f4 rgbs_color, f4 rgbo_color, int format, uint8_t* output, int quant_level) {
	QuantCtx q;
	q.tab = STAGED.cq_smem_off != 0 ? astc_smem + STAGED.cq_smem_off + 512 * (quant_level - QUANT_6)
	                                : ASTC_CT->color_unquant_to_uquant[quant_level - QUANT_6];
	q.quant_level = quant_level;

	color0 = vclamp4(0.0f, 65535.0f, color0);
	color1 = vclamp4(0.0f, 65535.0f, color1);
	f4 c0l = color0 * (1.0f / 257.0f);
	f4 c1l = color1 * (1.0f / 257.0f);

	uint8_t retval = 0;
	float best_error = 1e30f;
	i4 o0 = mki4(0, 0, 0, 0), o1 = mki4(0, 0, 0, 0), p0 = o0, p1 = o1, u0, u1;

	switch (format) {
	case FMT_RGB:
	case FMT_RGBA: {
		bool has_a = format == FMT_RGBA;
		if (quant_level <= QUANT_160) {
			bool ok = has_a ? (try_quantize_rgb_delta_blue_contract(c0l, c1l, o0, o1, q) && try_quantize_alpha_delta(c1l, c0l, o0, o1, q))
			                : try_quantize_rgb_delta_blue_contract(c0l, c1l, o0, o1, q);
			if (ok) {
				rgba_delta_unpack(o0, o1, u0, u1);
				retval = has_a ? FMT_RGBA_DELTA : FMT_RGB_DELTA;
				best_error = get_rgba_encoding_error(c0l, c1l, u0, u1);
			}
			ok = has_a ? (try_quantize_rgb_delta(c0l, c1l, p0, p1, q) && try_quantize_alpha_delta(c0l, c1l, p0, p1, q))
			           : try_quantize_rgb_delta(c0l, c1l, p0, p1, q);
			if (ok) {
				rgba_delta_unpack(p0, p1, u0, u1);
				float error = get_rgba_encoding_error(c0l, c1l, u0, u1);
				if (error < best_error) {
					retval = has_a ? FMT_RGBA_DELTA : FMT_RGB_DELTA;
					best_error = error;
					o0 = p0;
					o1 = p1;
				}
			}
		}
		if (quant_level < QUANT_256) {
			bool ok = has_a ? try_quantize_rgba_blue_contract(c0l, c1l, p0, p1, q) : try_quantize_rgb_blue_contract(c0l, c1l, p0, p1, q);
			if (ok) {
				rgba_unpack(p0, p1, u0, u1);
				float error = get_rgba_encoding_error(c0l, c1l, u0, u1);
				if (error < best_error) {
					retval = has_a ? FMT_RGBA : FMT_RGB;
					best_error = error;
					o0 = p0;
					o1 = p1;
				}
			}
		}
		{
			if (has_a) {
				quantize_rgba(c0l, c1l, p0, p1, q);
			} else {
				quantize_rgb(c0l, c1l, p0, p1, q);
			}
			rgba_unpack(p0, p1, u0, u1);
			float error = get_rgba_encoding_error(c0l, c1l, u0, u1);
			if (error < best_error) {
				retval = has_a ? FMT_RGBA : FMT_RGB;
				o0 = p0;
				o1 = p1;
			}
		}
		output[0] = (uint8_t)o0.x;
		output[1] = (uint8_t)o1.x;
		output[2] = (uint8_t)o0.y;
		output[3] = (uint8_t)o1.y;
		output[4] = (uint8_t)o0.z;
		output[5] = (uint8_t)o1.z;
		if (has_a) {
			output[6] = (uint8_t)o0.w;
			output[7] = (uint8_t)o1.w;
		}
		break;
	}
	case FMT_RGB_SCALE:
		quantize_rgbs(rgbs_color, output, q);
		retval = FMT_RGB_SCALE;
		break;
	case FMT_RGB_SCALE_ALPHA:
		output[4] = (uint8_t)quant_color_f(q, f2i_rtn(c0l.w), c0l.w);
		output[5] = (uint8_t)quant_color_f(q, f2i_rtn(c1l.w), c1l.w);
		quantize_rgbs(rgbs_color, output, q);
		retval = FMT_RGB_SCALE_ALPHA;
		break;
	case FMT_LUMINANCE:
		quantize_luminance(c0l, c1l, output, q);
		retval = FMT_LUMINANCE;
		break;
	case FMT_LUMINANCE_ALPHA:
		if (quant_level <= 18) {
			if (try_quantize_luminance_alpha_delta(c0l, c1l, output, q)) {
				retval = FMT_LUMINANCE_ALPHA_DELTA;
				break;
			}
		}
		quantize_luminance_alpha(c0l, c1l, output, q);
		retval = FMT_LUMINANCE_ALPHA;
		break;
	}
	return retval;
}

// The HDR formats (2, 3, 7, 11, 14, 15) are packed by the whole warp: their sub-mode ladders run lane-parallel
// (astc_dev_color_hdr_pack.cuh). Every lane passes the same arguments; `output` is shared memory (the winning lane of each
// ladder stores the bytes, the caller synchronises); returns the format used.
ASTC_FN bool is_hdr_format(int format) { return ((0xC88Cu >> format) & 1u) != 0; }

ASTC_NOINLINE uint8_t pack_hdr_endpoints(int lane, f4 color0, f4 color1, f4 rgbo_color, int format, uint8_t* output, int quant_level) {
	QuantCtx q;
	q.tab = STAGED.cq_smem_off != 0 ? astc_smem + STAGED.cq_smem_off + 512 * (quant_level - QUANT_6)
	                                : ASTC_CT->color_unquant_to_uquant[quant_level - QUANT_6];
	q.quant_level = quant_level;
	color0 = vclamp4(0.0f, 65535.0f, color0);
	color1 = vclamp4(0.0f, 65535.0f, color1);
	switch (format) {
	case FMT_HDR_RGB_SCALE:
		quantize_hdr_rgbo(lane, rgbo_color, output, q);
		return FMT_HDR_RGB_SCALE;
	case FMT_HDR_RGB:
		quantize_hdr_rgb(lane, color0, color1, output, q);
		return FMT_HDR_RGB;
	case FMT_HDR_RGB_LDR_ALPHA:
		if (lane == 0) {      // (:1791-1817: LDR alpha beside the HDR colour)
			float a0 = clampf(color0.w * (1.0f / 257.0f), 0.0f, 255.0f);
			float a1 = clampf(color1.w * (1.0f / 257.0f), 0.0f, 255.0f);
			output[6] = (uint8_t)quant_color_f(q, f2i_rtn(a0), a0);
			output[7] = (uint8_t)quant_color_f(q, f2i_rtn(a1), a1);
		}
		quantize_hdr_rgb(lane, color0, color1, output, q);
		return FMT_HDR_RGB_LDR_ALPHA;
	case FMT_HDR_RGBA:
		quantize_hdr_rgb(lane, color0, color1, output, q);
		quantize_hdr_alpha(lane, color0.w, color1.w, output + 6, q);
		return FMT_HDR_RGBA;
	default:      // FMT_HDR_LUMINANCE_SMALL_RANGE / _LARGE_RANGE: the small range form when it fits
		return (uint8_t)quantize_hdr_luminance(lane, color0, color1, output, q);
	}
}

// FMT_RGB / FMT_RGBA, the formats of nearly every candidate of an LDR image, are a contest of four encodings of the same
// endpoint pair (:1953-2050): base + offset with blue contraction, base + offset, blue contraction, plain - the one with the
// smallest round-trip error wins, the earlier one on a tie. For a single-partition candidate the four run on four lanes
// (the two offset forms share their instruction stream, as do the four round-trip error evaluations); the winner stores
// the bytes. `output` is shared memory, every lane passes the same arguments, the caller synchronises.
// INL: the quantisers are inlined (the one-partition LDR refinement step) instead of called
template <bool INL> ASTC_FN uint8_t pack_rgb_endpoints_coop_t(int lane, f4 color0, f4 color1, int format, uint8_t* output, int quant_level) {
	QuantCtx q;
	q.tab = STAGED.cq_smem_off != 0 ? astc_smem + STAGED.cq_smem_off + 512 * (quant_level - QUANT_6)
	                                : ASTC_CT->color_unquant_to_uquant[quant_level - QUANT_6];
	q.quant_level = quant_level;
	color0 = vclamp4(0.0f, 65535.0f, color0);
	color1 = vclamp4(0.0f, 65535.0f, color1);
	const f4 c0l = color0 * (1.0f / 257.0f);
	const f4 c1l = color1 * (1.0f / 257.0f);
	const bool has_a = format == FMT_RGBA;
	float best = 3.0e38f;
	int best_k = 0x7FFFFFFF;
	i4 b0 = mki4(0, 0, 0, 0), b1 = b0;
	ASTC_NOUNROLL
	for (int k = lane; k < 4; k += ASTC_WARP) {
		// which encodings the quant level admits (:1957, :1999)
		if ((k < 2 && quant_level > QUANT_160) || (k == 2 && quant_level >= QUANT_256)) {
			continue;
		}
		i4 o0 = mki4(0, 0, 0, 0), o1 = o0;
		bool ok;
		if (k < 2) {
			// base + offset; the blue-contracted form starts from the swapped, contracted pair and wants a negative offset sum
			const bool bc = k == 0;
			f4 a = bc ? c1l : c0l, b = bc ? c0l : c1l;
			ok = true;
			if (bc) {
				a = blue_contract_fwd(a);
				b = blue_contract_fwd(b);
				ok = in_0_255(a) && in_0_255(b);
			}
			if (ok) {
				QEnds r = INL ? rgb_delta_core_inl(a, b, q, bc) : rgb_delta_core_v(a, b, q, bc);
				ok = r.ok;
				o0 = r.a;
				o1 = r.b;
			}
			if (ok && has_a) {
				QAlpha ra = INL ? try_quantize_alpha_delta_inl(bc ? c1l : c0l, bc ? c0l : c1l, q) : try_quantize_alpha_delta_v(bc ? c1l : c0l, bc ? c0l : c1l, q);
				ok = ra.ok;
				o0.w = ra.a0;
				o1.w = ra.a1;
			}
		} else if (k == 2) {
			QEnds r = INL ? try_quantize_rgb_blue_contract_inl(c0l, c1l, q) : try_quantize_rgb_blue_contract_v(c0l, c1l, q);
			ok = r.ok;
			o0 = r.a;
			o1 = r.b;
			if (ok && has_a) {
				o0.w = quant_color_f(q, f2i_rtn(c1l.w), c1l.w);
				o1.w = quant_color_f(q, f2i_rtn(c0l.w), c0l.w);
			}
		} else {
			QEnds r = INL ? quantize_rgb_inl(c0l, c1l, q) : quantize_rgb_v(c0l, c1l, q);
			ok = true;
			o0 = r.a;
			o1 = r.b;
			if (has_a) {
				o0.w = quant_color_f(q, f2i_rtn(c0l.w), c0l.w);
				o1.w = quant_color_f(q, f2i_rtn(c1l.w), c1l.w);
			}
		}
		if (ok) {
			i4 u0, u1;
			if (k < 2) {
				rgba_delta_unpack(o0, o1, u0, u1);
			} else {
				rgba_unpack(o0, o1, u0, u1);
			}
			float error = get_rgba_encoding_error(c0l, c1l, u0, u1);
			if (error < best) {
				best = error;
				best_k = k;
				b0 = o0;
				b1 = o1;
			}
		}
	}
#if !defined(ASTC_ONE_LANE)
	// smallest error, the earlier encoding on a tie; every lane learns the winner
	{
		float e = best;
		int ik = best_k;
		ASTC_NOUNROLL
		for (int o = 16; o > 0; o >>= 1) {
			float e2 = __shfl_xor_sync(0xffffffffu, e, o);
			int i2 = __shfl_xor_sync(0xffffffffu, ik, o);
			bool take = (e2 < e) || (e2 == e && i2 < ik);
			e = take ? e2 : e;
			ik = take ? i2 : ik;
		}
		if (ik != best_k) {
			best_k = ik;
			best = -1.0f;      // not this lane's
		}
	}
#endif
	if (best >= 0.0f) {
		output[0] = (uint8_t)b0.x;
		output[1] = (uint8_t)b1.x;
		output[2] = (uint8_t)b0.y;
		output[3] = (uint8_t)b1.y;
		output[4] = (uint8_t)b0.z;
		output[5] = (uint8_t)b1.z;
		if (has_a) {
			output[6] = (uint8_t)b0.w;
			output[7] = (uint8_t)b1.w;
		}
	}
	return (uint8_t)(best_k < 2 ? (has_a ? FMT_RGBA_DELTA : FMT_RGB_DELTA) : (has_a ? FMT_RGBA : FMT_RGB));
}
ASTC_NOINLINE uint8_t pack_rgb_endpoints_coop(int lane, f4 color0, f4 color1, int format, uint8_t* output, int quant_level) {
	return pack_rgb_endpoints_coop_t<false>(lane, color0, color1, format, output, quant_level);
}
