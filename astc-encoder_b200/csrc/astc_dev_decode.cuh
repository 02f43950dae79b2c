// CUDA-native ASTC: block DECOMPRESSION (SURVEY.md section 8f, first "next" row).
//   physical_to_symbolic        astcenc_symbolic_physical.cpp:291-556   (lane 0: ~100 sequential bit-field reads)
//   decode_ise                  astcenc_integer_sequence.cpp:651-760
//   decompress_symbolic_block   astcenc_decompress_symbolic.cpp:170-306 (lanes over texels)
//   store_image_block           astcenc_image.cpp:345-563               (lanes over texels, straight to the image)
// One warp per block. The warp's slice of shared memory holds the symbolic block: weights[64], colour values
// [4][8], the unpacked endpoints and a few scalars.
#pragma once
#include "../../include/astcenc.h"

// decode slice layout (bytes from the slice base)
enum { D_WEIGHTS = 0, D_COLORS = 64, D_ENDS = 96 /* int[4][8] + lns flags */, D_HDR = 96 + 128 + 16, D_SLICE = 304 };

struct DecodeHdr {
	int block_type, partition_count, partition_index, block_mode_packed, plane2_component, quant_mode;
	int color_formats[4];
	int constant_color[4];
};
static_assert(D_HDR + sizeof(DecodeHdr) <= D_SLICE, "decode slice");

// read up to 16 bits at a bit offset of the 128-bit block held in two registers (read_bits :52-63; bits past 127 read 0)
ASTC_FN unsigned int rd_bits(uint64_t lo, uint64_t hi, unsigned int bitcount, unsigned int bitoffset) {
	uint64_t v;
	if (bitoffset >= 128) {
		v = 0;
	} else if (bitoffset >= 64) {
		v = hi >> (bitoffset - 64);
	} else {
		v = lo >> bitoffset;
		if (bitoffset != 0) {
			v |= hi << (64 - bitoffset);
		}
	}
	return (unsigned int)v & ((1u << bitcount) - 1u);
}

// decode_ise: the values go to out[0..count) in shared memory, mapped through `table` (unscramble / unquantise)
ASTC_NOINLINE void decode_ise_mapped(int quant_level, unsigned int count, uint64_t lo, uint64_t hi, unsigned int bit_offset, const uint8_t* table,
                                     uint32_t out_off, int dual_interleave) {
	const DevConstTables* ct = ASTC_CT;
	SPtr<uint8_t> out = sptr<uint8_t>(out_off);
	unsigned int bits, trits, quints;
	ise_btq(quant_level, bits, trits, quints);
	unsigned int group = trits ? 5u : quints ? 3u : 1u;
	ASTC_NOUNROLL
	for (unsigned int i = 0; i < count; i += group) {
		unsigned int m[5] = {0, 0, 0, 0, 0};
		unsigned int tq = 0;
		for (unsigned int j = 0; j < 5; j++) {
			if (j < group && i + j < count) {
				m[j] = rd_bits(lo, hi, bits, bit_offset);
				bit_offset += bits;
				if (trits) {
					unsigned int n = (j == 2 || j == 4) ? 1u : 2u;
					unsigned int sh = j == 0 ? 0u : j == 1 ? 2u : j == 2 ? 4u : j == 3 ? 5u : 7u;
					tq |= rd_bits(lo, hi, n, bit_offset) << sh;
					bit_offset += n;
				} else if (quints) {
					unsigned int n = j == 0 ? 3u : 2u;
					unsigned int sh = j == 0 ? 0u : j == 1 ? 3u : 5u;
					tq |= rd_bits(lo, hi, n, bit_offset) << sh;
					bit_offset += n;
				}
			}
		}
		for (unsigned int j = 0; j < 5; j++) {
			if (j < group && i + j < count) {
				unsigned int v = m[j];
				if (trits) {
					v |= (unsigned int)ASTC_LDG(&ct->trits_of_integer[tq & 0xFF][j]) << bits;
				} else if (quints) {
					v |= (unsigned int)ASTC_LDG(&ct->quints_of_integer[tq & 0x7F][j < 3 ? j : 0]) << bits;
				}
				unsigned int k = i + j;
				// dual-plane weights arrive interleaved: even -> plane 1, odd -> plane 2 (+32)
				unsigned int dst = dual_interleave ? ((k >> 1) + ((k & 1) ? 32u : 0u)) : k;
				out[(int)dst] = ASTC_LDG(&table[v & 0xFF]);
			}
		}
	}
}

// The header stage of physical_to_symbolic (astcenc_symbolic_physical.cpp:291-556 without the two ISE decodes and the constant
// colour), in registers: the block-type verdict (void extents 2D and 3D, reserved bits, the block-mode table, dual plane with
// four partitions, partition-table validity, more than 18 colour integers, colour quant below QUANT_6) and the header fields.
// An error block keeps the fields read before the rule it breaks; nothing reads them.
struct BlockHeader {
	int block_type, partition_count, partition_index, block_mode_packed, plane2_component, quant_mode;
	int color_formats[4];
	int weight_count;              // the weights of both planes
	int weight_quant;
	int color_integer_count;       // the colour values of all partitions
	bool dual;
};

ASTC_FN BlockHeader block_header(uint64_t lo, uint64_t hi) {
	const DevConstTables* ct = ASTC_CT;
	BlockHeader h;
	h.block_type = SYM_BTYPE_NONCONST;
	h.partition_count = 0;
	h.partition_index = 0;
	h.block_mode_packed = 0;
	h.plane2_component = -1;
	h.quant_mode = 0;
	for (int i = 0; i < 4; i++) {
		h.color_formats[i] = 0;
	}
	h.weight_count = 0;
	h.weight_quant = 0;
	h.color_integer_count = 0;
	h.dual = false;
	int block_mode = (int)rd_bits(lo, hi, 11, 0);
	if ((block_mode & 0x1FF) == 0x1FC) {
		h.block_type = (block_mode & 0x200) ? SYM_BTYPE_CONST_F16 : SYM_BTYPE_CONST_U16;
		if (BSD.dim_z > 1) {
			// 3D void extent (astcenc_symbolic_physical.cpp:348-366): six 9-bit coordinates, no reserved bits
			int v[6];
			bool ones = true;
			for (int k = 0; k < 6; k++) {
				v[k] = (int)rd_bits(lo, hi, 9, 10 + 9 * (unsigned int)k);
				ones = ones && v[k] == 0x1FF;
			}
			if ((v[0] >= v[1] || v[2] >= v[3] || v[4] >= v[5]) && !ones) {
				h.block_type = SYM_BTYPE_ERROR;
			}
			return h;
		}
		int rsvbits = (int)rd_bits(lo, hi, 2, 10);
		if (rsvbits != 3) {
			h.block_type = SYM_BTYPE_ERROR;
			return h;
		}
		int vx_low_s = (int)rd_bits(lo, hi, 13, 12);
		int vx_high_s = (int)rd_bits(lo, hi, 13, 25);
		int vx_low_t = (int)rd_bits(lo, hi, 13, 38);
		int vx_high_t = (int)rd_bits(lo, hi, 13, 51);
		bool all_ones = vx_low_s == 0x1FFF && vx_high_s == 0x1FFF && vx_low_t == 0x1FFF && vx_high_t == 0x1FFF;
		if ((vx_low_s >= vx_high_s || vx_low_t >= vx_high_t) && !all_ones) {
			h.block_type = SYM_BTYPE_ERROR;
		}
		return h;
	}
	unsigned int packed_index = ASTC_LDG(&BSD.block_mode_packed_index[block_mode]);
	if (packed_index == 0xFFFF) {
		h.block_type = SYM_BTYPE_ERROR;
		return h;
	}
	const DevBlockMode* bm = BSD.block_modes + packed_index;
	int weight_count = ASTC_LDG(&BSD.dec_modes[ASTC_LDG(&bm->decimation_mode)].weight_count);
	h.weight_quant = ASTC_LDG(&bm->quant_mode);
	h.dual = ASTC_LDG(&bm->is_dual_plane) != 0;
	h.weight_count = h.dual ? 2 * weight_count : weight_count;
	int partition_count = (int)rd_bits(lo, hi, 2, 11) + 1;
	h.block_mode_packed = (int)packed_index;
	h.partition_count = partition_count;
	int bits_for_weights = (int)ise_sequence_bitcount((unsigned int)h.weight_count, h.weight_quant);
	int below_weights_pos = 128 - bits_for_weights;
	if (h.dual && partition_count == 4) {
		h.block_type = SYM_BTYPE_ERROR;
		return h;
	}
	int encoded_type_highpart_size = 0;
	if (partition_count == 1) {
		h.color_formats[0] = (int)rd_bits(lo, hi, 4, 13);
	} else {
		encoded_type_highpart_size = (3 * partition_count) - 4;
		below_weights_pos -= encoded_type_highpart_size;
		int encoded_type = (int)rd_bits(lo, hi, 6, 13 + 10) | ((int)rd_bits(lo, hi, (unsigned int)encoded_type_highpart_size, (unsigned int)below_weights_pos) << 6);
		int baseclass = encoded_type & 0x3;
		if (baseclass == 0) {
			for (int i = 0; i < 4; i++) {
				if (i < partition_count) h.color_formats[i] = (encoded_type >> 2) & 0xF;
			}
			below_weights_pos += encoded_type_highpart_size;
			encoded_type_highpart_size = 0;
		} else {
			int bitpos = 2;
			baseclass--;
			for (int i = 0; i < 4; i++) {
				if (i < partition_count) {
					h.color_formats[i] = (((encoded_type >> bitpos) & 1) + baseclass) << 2;
					bitpos++;
				}
			}
			for (int i = 0; i < 4; i++) {
				if (i < partition_count) {
					h.color_formats[i] |= (encoded_type >> bitpos) & 3;
					bitpos += 2;
				}
			}
		}
		h.partition_index = (int)rd_bits(lo, hi, 10, 13);
		if (ASTC_LDG(&BSD.partitioning_packed_index[partition_count - 2][h.partition_index]) == 0xFFFF) {
			h.block_type = SYM_BTYPE_ERROR;
			return h;
		}
	}
	int color_integer_count = 0;
	for (int i = 0; i < 4; i++) {
		if (i < partition_count) {
			color_integer_count += ((h.color_formats[i] >> 2) + 1) * 2;
		}
	}
	h.color_integer_count = color_integer_count;
	if (color_integer_count > 18) {
		h.block_type = SYM_BTYPE_ERROR;
		return h;
	}
	int color_bits = (partition_count == 1 ? 115 - 4 : 113 - 4 - 10) - bits_for_weights - encoded_type_highpart_size;
	if (h.dual) {
		color_bits -= 2;
	}
	if (color_bits < 0) {
		color_bits = 0;
	}
	int color_quant_level = ASTC_LDG(&ct->quant_mode_table[color_integer_count >> 1][color_bits]);
	if (color_quant_level < QUANT_6) {
		h.block_type = SYM_BTYPE_ERROR;
		return h;
	}
	h.quant_mode = color_quant_level;
	if (h.dual) {
		h.plane2_component = (int)rd_bits(lo, hi, 2, (unsigned int)(below_weights_pos - 2));
	}
	return h;
}

// physical_to_symbolic: the header stage, then the weight and colour ISE decodes and the constant colour. Executed by lane 0;
// the result lands in the slice.
ASTC_NOINLINE void physical_to_symbolic(uint32_t slice, uint64_t lo, uint64_t hi) {
	const DevConstTables* ct = ASTC_CT;
	DecodeHdr& h = *reinterpret_cast<DecodeHdr*>(astc_smem + slice + D_HDR);
	const BlockHeader b = block_header(lo, hi);
	h.block_type = b.block_type;
	h.partition_count = b.partition_count;
	h.partition_index = b.partition_index;
	h.block_mode_packed = b.block_mode_packed;
	h.plane2_component = b.plane2_component;
	h.quant_mode = b.quant_mode;
	for (int i = 0; i < 4; i++) {
		h.color_formats[i] = b.color_formats[i];
	}
	if (b.block_type == SYM_BTYPE_CONST_F16 || b.block_type == SYM_BTYPE_CONST_U16) {
		for (int i = 0; i < 4; i++) {
			h.constant_color[i] = (int)rd_bits(hi, 0, 16, 16 * (unsigned int)i);
		}
		return;
	}
	if (b.block_type != SYM_BTYPE_NONCONST) {
		return;
	}
	// the weight stream is read from the top of the block, bit-reversed (:404-407)
	decode_ise_mapped(b.weight_quant, (unsigned int)b.weight_count, brev64(hi), brev64(lo), 0, ct->wq_unscramble_and_unquant[b.weight_quant],
	                  slice + D_WEIGHTS, b.dual ? 1 : 0);
	// the colour values of all partitions are one sequence; partition p's values start at 8 * p in the slice
	SPtr<uint8_t> colors = sptr<uint8_t>(slice + D_COLORS);
	SPtr<uint8_t> tmp = sptr<uint8_t>(slice + D_ENDS);      // staging (the endpoints are unpacked afterwards)
	decode_ise_mapped(b.quant_mode, (unsigned int)b.color_integer_count, lo, hi, b.partition_count == 1 ? 17u : 19u + 10u,
	                  ct->color_scrambled_pquant_to_uquant[b.quant_mode - QUANT_6], slice + D_ENDS, 0);
	int k = 0;
	for (int i = 0; i < 4; i++) {
		if (i < b.partition_count) {
			int vals = 2 * (b.color_formats[i] >> 2) + 2;
			for (int j = 0; j < 8; j++) {
				if (j < vals) {
					colors[i * 8 + j] = tmp[k + j];
				}
			}
			k += vals;
		}
	}
}

ASTC_FN float error_color_nan() { return ASTC_U2F(0xFFFFE000u); }

ASTC_FN float decode_component(int v, bool lns) {   // decode_texel :66-87
	int sf = lns ? lns_to_sf16(v) : unorm16_to_sf16(v);
	return sf16_to_float((uint16_t)sf);
}

// n bytes from src to dst, one at a time (an output that starts at any byte)
ASTC_FN void store_bytes(uint8_t* dst, const uint8_t* src, int n) {
	for (int k = 0; k < n; k++) {
		dst[k] = src[k];
	}
}

// store one texel (store_image_block); swz uses astcenc_swz numbering (4 = 0, 5 = 1, 6 = Z). img.data may start at any byte
// (decode calls over image tables), and a texel that is not aligned to its components is stored byte by byte.
ASTC_FN void store_texel(const DevImage& img, unsigned int x, unsigned int y, unsigned int z, f4 d) {
	bool needs_swz = img.swz[0] != 0 || img.swz[1] != 1 || img.swz[2] != 2 || img.swz[3] != 3;
	bool needs_z = img.swz[0] == 6 || img.swz[1] == 6 || img.swz[2] == 6 || img.swz[3] == 6;
	size_t o = (4 * (size_t)img.dim_x * img.dim_y * z) + (4 * (size_t)img.dim_x * y) + 4 * (size_t)x;
	void* base = const_cast<void*>(img.data);
	if (img.data_type == 0) {
		int vr = f2i_rtn(clampzo(d.x) * 255.0f), vg = f2i_rtn(clampzo(d.y) * 255.0f), vb = f2i_rtn(clampzo(d.z) * 255.0f), va = f2i_rtn(clampzo(d.w) * 255.0f);
		int o0 = vr, o1 = vg, o2 = vb, o3 = va;
		if (needs_swz) {
			int vz = 0;
			if (needs_z) {
				float data_x = (d.x * 2.0f) - 1.0f;
				float data_y = (d.w * 2.0f) - 1.0f;
				float data_z = 1.0f - (data_x * data_x) - (data_y * data_y);
				data_z = maxf(data_z, 0.0f);
				data_z = (sqrtf(data_z) * 0.5f) + 0.5f;
				vz = f2i_rtn(minf(data_z, 1.0f) * 255.0f);
			}
			int sel[4];
			for (int k = 0; k < 4; k++) {
				int s = img.swz[k];
				sel[k] = s == 0 ? vr : s == 1 ? vg : s == 2 ? vb : s == 3 ? va : s == 4 ? 0 : s == 5 ? 255 : vz;
			}
			o0 = sel[0]; o1 = sel[1]; o2 = sel[2]; o3 = sel[3];
		}
		if (d.x != d.x) {      // errors are NaN encoded -> magenta
			o0 = 0xFF; o1 = 0x00; o2 = 0xFF; o3 = 0xFF;
		}
		uint32_t px = (uint32_t)(o0 & 0xFF) | ((uint32_t)(o1 & 0xFF) << 8) | ((uint32_t)(o2 & 0xFF) << 16) | ((uint32_t)(o3 & 0xFF) << 24);
		uint8_t* dst = static_cast<uint8_t*>(base) + o;
		if ((reinterpret_cast<uintptr_t>(dst) & 3) != 0) {
			store_bytes(dst, reinterpret_cast<const uint8_t*>(&px), 4);
		} else {
			*reinterpret_cast<uint32_t*>(dst) = px;
		}
		return;
	}
	f4 ov = d;
	if (needs_swz) {
		float vz = 0.0f;
		if (needs_z) {
			float xN = (d.x * 2.0f) - 1.0f;
			float yN = (d.w * 2.0f) - 1.0f;
			float zN = 1.0f - xN * xN - yN * yN;
			if (zN < 0.0f) {
				zN = 0.0f;
			}
			vz = (sqrtf(zN) * 0.5f) + 0.5f;
			// A NaN input gives a NaN Z. The reference's x86 arithmetic passes on the first NaN operand's payload (quieted),
			// which through 1 - xN * xN - yN * yN is R's, else A's; the GPU's arithmetic would give its canonical NaN instead.
			if (d.x != d.x || d.w != d.w) {
				vz = ASTC_U2F(ASTC_F2U(d.x != d.x ? d.x : d.w) | 0x00400000u);
			}
		}
		float sel[4];
		for (int k = 0; k < 4; k++) {
			int s = img.swz[k];
			sel[k] = s == 0 ? d.x : s == 1 ? d.y : s == 2 ? d.z : s == 3 ? d.w : s == 4 ? 0.0f : s == 5 ? 1.0f : vz;
		}
		ov = mk4(sel[0], sel[1], sel[2], sel[3]);
	}
	if (img.data_type == 1) {
		uint16_t* p = static_cast<uint16_t*>(base) + o;
		if ((reinterpret_cast<uintptr_t>(p) & 1) != 0) {
			const uint16_t h[4] = {float_to_sf16(ov.x), float_to_sf16(ov.y), float_to_sf16(ov.z), float_to_sf16(ov.w)};
			store_bytes(reinterpret_cast<uint8_t*>(p), reinterpret_cast<const uint8_t*>(h), 8);
			return;
		}
		p[0] = float_to_sf16(ov.x);
		p[1] = float_to_sf16(ov.y);
		p[2] = float_to_sf16(ov.z);
		p[3] = float_to_sf16(ov.w);
	} else {
		float* p = static_cast<float*>(base) + o;
		if ((reinterpret_cast<uintptr_t>(p) & 3) != 0) {
			const float f[4] = {ov.x, ov.y, ov.z, ov.w};
			store_bytes(reinterpret_cast<uint8_t*>(p), reinterpret_cast<const uint8_t*>(f), 16);
			return;
		}
		p[0] = ov.x;
		p[1] = ov.y;
		p[2] = ov.z;
		p[3] = ov.w;
	}
}

// Decompress block (bx_i, by_i) of the image described by IMG (IMG.data = output image, IMG.out unused).
ASTC_COOP void decompress_block(int lane, uint32_t slice, const uint8_t* pcb, unsigned int bx_i, unsigned int by_i) {
	const DevImage& img = IMG;
	int T = BSD.texel_count;
	unsigned int bdx = BSD.dim_x;
	DecodeHdr& h = *reinterpret_cast<DecodeHdr*>(astc_smem + slice + D_HDR);
	if (lane == 0) {
		const uint32_t* p32 = reinterpret_cast<const uint32_t*>(pcb);
		uint64_t lo = (uint64_t)ASTC_LDG(p32) | ((uint64_t)ASTC_LDG(p32 + 1) << 32);
		uint64_t hi = (uint64_t)ASTC_LDG(p32 + 2) | ((uint64_t)ASTC_LDG(p32 + 3) << 32);
		physical_to_symbolic(slice, lo, hi);
	}
	wsync();
	int decode_mode = CFG.profile;
	int block_type = h.block_type;
	bool u8 = img.data_type == 0 || decode_mode == PRF_LDR_SRGB;
	// 3D block sizes: by_i counts layer * IMG.blocks_y + row; texels run x fastest, then y, then z (store_image_block, astcenc_image.cpp:366-420)
	const bool volume = BSD.dim_z > 1;
	unsigned int pos_x = bx_i * bdx, pos_y = by_i * BSD.dim_y, pos_z = 0;
	unsigned int lim_z = 1;
	if (volume) {
		unsigned int layer = by_i / img.blocks_y;
		pos_y = (by_i - layer * img.blocks_y) * BSD.dim_y;
		pos_z = layer * BSD.dim_z;
		lim_z = img.dim_z;
	}
	if (block_type != SYM_BTYPE_NONCONST) {
		f4 c = splat4(error_color_nan());
		if (block_type == SYM_BTYPE_CONST_U16) {
			int v[4];
			for (int k = 0; k < 4; k++) {
				int ci = h.constant_color[k];
				if (u8) {
					ci = (ci >> 8) * 257;
				}
				v[k] = unorm16_to_sf16(ci);
			}
			c = mk4(sf16_to_float((uint16_t)v[0]), sf16_to_float((uint16_t)v[1]), sf16_to_float((uint16_t)v[2]), sf16_to_float((uint16_t)v[3]));
		} else if (block_type == SYM_BTYPE_CONST_F16 && (decode_mode == PRF_HDR || decode_mode == PRF_HDR_RGB_LDR_A)) {
			// the reference's F16C builds saturate the packed half-floats (astcenc_vecmathlib_sse_4.h:1001): sign bit set -> 0x7FFF
			int v[4];
			for (int k = 0; k < 4; k++) {
				v[k] = h.constant_color[k] > 0x7FFF ? 0x7FFF : h.constant_color[k];
			}
			c = mk4(sf16_to_float((uint16_t)v[0]), sf16_to_float((uint16_t)v[1]), sf16_to_float((uint16_t)v[2]), sf16_to_float((uint16_t)v[3]));
		}
		ASTC_NOUNROLL
		for (int t = lane; t < T; t += ASTC_WARP) {
			unsigned int tyz = (unsigned int)t / bdx, tz = volume ? tyz / BSD.dim_y : 0u;
			unsigned int x = pos_x + (unsigned int)t % bdx, y = pos_y + tyz - tz * BSD.dim_y, z = pos_z + tz;
			if (x < img.dim_x && y < img.dim_y && z < lim_z) {
				store_texel(img, x, y, z, c);
			}
		}
		wsync();
		return;
	}
	int pc = h.partition_count;
	// endpoints: lanes over partitions -> ends[p][0..3] = endpoint 0, [4..7] = endpoint 1, flags behind
	SPtr<int> ends = sptr<int>(slice + D_ENDS);
	SPtr<uint8_t> lnsf = sptr<uint8_t>(slice + D_ENDS + 128);
	SPtr<uint8_t> colors = sptr<uint8_t>(slice + D_COLORS);
	wsync();
	ASTC_NOUNROLL
	for (int p = lane; p < pc; p += ASTC_WARP) {
		uint8_t in[8];
		for (int k = 0; k < 8; k++) {
			in[k] = colors[p * 8 + k];
		}
		bool rgb_lns, a_lns;
		i4 e0, e1;
		unpack_color_endpoints(decode_mode, h.color_formats[p], in, rgb_lns, a_lns, e0, e1);
		SPtr<int> o = ends + p * 8;
		o[0] = e0.x; o[1] = e0.y; o[2] = e0.z; o[3] = e0.w;
		o[4] = e1.x; o[5] = e1.y; o[6] = e1.z; o[7] = e1.w;
		lnsf[p * 2] = rgb_lns ? 1 : 0;
		lnsf[p * 2 + 1] = a_lns ? 1 : 0;
	}
	wsync();
	const DevBlockMode* bm = BSD.block_modes + h.block_mode_packed;
	DecView di = dec_view(ASTC_LDG(&bm->decimation_mode));
	bool dual = ASTC_LDG(&bm->is_dual_plane) != 0;
	int plane2_component = h.plane2_component;
	PartView pi = part_view_packed((unsigned int)pc, part_packed_index((unsigned int)pc, (unsigned int)h.partition_index));
	SPtr<uint8_t> uq = sptr<uint8_t>(slice + D_WEIGHTS);
	ASTC_NOUNROLL
	for (int t = lane; t < T; t += ASTC_WARP) {
		uint32_t ix = ASTC_LDD(&di.twi[t]);
		uint32_t cx = ASTC_LDD(&di.tci[t]);
		int i0 = (int)(ix & 0xFF), i1 = (int)((ix >> 8) & 0xFF), i2 = (int)((ix >> 16) & 0xFF), i3 = (int)(ix >> 24);
		int c0 = (int)(cx & 0xFF), c1 = (int)((cx >> 8) & 0xFF), c2 = (int)((cx >> 16) & 0xFF), c3 = (int)(cx >> 24);
		int w1 = (8 + uq[i0] * c0 + uq[i1] * c1 + uq[i2] * c2 + uq[i3] * c3) >> 4;
		int w2 = w1;
		if (dual) {
			w2 = (8 + uq[32 + i0] * c0 + uq[32 + i1] * c1 + uq[32 + i2] * c2 + uq[32 + i3] * c3) >> 4;
		}
		int p = pc > 1 ? (int)ASTC_LDG(&pi.partition_of_texel[t]) : 0;
		SPtr<int> e = ends + p * 8;
		bool rgb_lns = lnsf[p * 2] != 0, a_lns = lnsf[p * 2 + 1] != 0;
		f4 d = mk4(decode_component(lerp1(u8, e[0], e[4], plane2_component == 0 ? w2 : w1), rgb_lns),
		           decode_component(lerp1(u8, e[1], e[5], plane2_component == 1 ? w2 : w1), rgb_lns),
		           decode_component(lerp1(u8, e[2], e[6], plane2_component == 2 ? w2 : w1), rgb_lns),
		           decode_component(lerp1(u8, e[3], e[7], plane2_component == 3 ? w2 : w1), a_lns));
		unsigned int tyz = (unsigned int)t / bdx, tz = volume ? tyz / BSD.dim_y : 0u;
		unsigned int x = pos_x + (unsigned int)t % bdx, y = pos_y + tyz - tz * BSD.dim_y, z = pos_z + tz;
		if (x < img.dim_x && y < img.dim_y && z < lim_z) {
			store_texel(img, x, y, z, d);
		}
	}
	wsync();
}

// ---------------------------------------------------------------------------------------------
// astcenc_get_block_info (astcenc_entry.cpp:1401-1517): the decoded view of one block, written straight into the public
// astcenc_block_info layout by one warp (astcenc_get_block_info, astcenc_b200_get_block_info_device_block_lists).
// ---------------------------------------------------------------------------------------------
// The fields astcenc_get_block_info takes from the context rather than from the block.
struct BlockInfoHead {
	int profile;
	unsigned int block_x, block_y, block_z, texel_count;
};

// Every byte of *out (4-byte aligned): zeros where the reference leaves its memset's zeros. The lanes zero the struct word by
// word; the barrier after the parse orders those stores before the fields'.
ASTC_COOP void block_info(int lane, uint32_t slice, uint64_t lo, uint64_t hi, const BlockInfoHead& head, astcenc_block_info* out) {
	int T = BSD.texel_count;
	DecodeHdr& h = *reinterpret_cast<DecodeHdr*>(astc_smem + slice + D_HDR);
	uint32_t* words = reinterpret_cast<uint32_t*>(out);
	for (int k = lane; k < (int)(sizeof(astcenc_block_info) / 4); k += ASTC_WARP) {
		words[k] = 0;
	}
	if (lane == 0) {
		physical_to_symbolic(slice, lo, hi);
	}
	wsync();
	int block_type = h.block_type;
	if (lane == 0) {
		out->profile = (astcenc_profile)head.profile;
		out->block_x = head.block_x;
		out->block_y = head.block_y;
		out->block_z = head.block_z;
		out->texel_count = head.texel_count;
		out->is_error_block = block_type == SYM_BTYPE_ERROR;
		out->is_constant_block = block_type == SYM_BTYPE_CONST_F16 || block_type == SYM_BTYPE_CONST_U16;
	}
	if (block_type != SYM_BTYPE_NONCONST) {
		return;
	}
	int pc = h.partition_count;
	int decode_mode = CFG.profile;
	const DevBlockMode* bm = BSD.block_modes + h.block_mode_packed;
	unsigned int d = ASTC_LDG(&bm->decimation_mode);
	bool dual = ASTC_LDG(&bm->is_dual_plane) != 0;
	SPtr<uint8_t> colors = sptr<uint8_t>(slice + D_COLORS);
	if (lane == 0) {
		out->weight_x = ASTC_LDG(&BSD.dec_modes[d].weight_x);
		out->weight_y = ASTC_LDG(&BSD.dec_modes[d].weight_y);
		out->weight_z = ASTC_LDG(&BSD.dec_modes[d].weight_z);
		out->is_dual_plane_block = dual;
		out->partition_count = (unsigned int)pc;
		out->partition_index = (unsigned int)h.partition_index;
		out->dual_plane_component = (unsigned int)h.plane2_component;
		out->color_level_count = quant_level_count(h.quant_mode);
		out->weight_level_count = quant_level_count(ASTC_LDG(&bm->quant_mode));
		bool is_hdr = false;
		for (int p = 0; p < 4; p++) {
			if (p >= pc) {
				break;
			}
			uint8_t in[8];
			for (int k = 0; k < 8; k++) {
				in[k] = colors[p * 8 + k];
			}
			bool rgb_hdr, a_hdr;
			i4 e[2];
			unpack_color_endpoints(decode_mode, h.color_formats[p], in, rgb_hdr, a_hdr, e[0], e[1]);
			out->color_endpoint_modes[p] = (unsigned int)h.color_formats[p];
			is_hdr = is_hdr || rgb_hdr || a_hdr;
			for (int j = 0; j < 2; j++) {
				out->color_endpoints[p][j][0] = decode_component(e[j].x, rgb_hdr);
				out->color_endpoints[p][j][1] = decode_component(e[j].y, rgb_hdr);
				out->color_endpoints[p][j][2] = decode_component(e[j].z, rgb_hdr);
				out->color_endpoints[p][j][3] = decode_component(e[j].w, a_hdr);
			}
		}
		out->is_hdr_block = is_hdr;
	}
	DecView di = dec_view(d);
	PartView pi = part_view_packed((unsigned int)pc, part_packed_index((unsigned int)pc, (unsigned int)h.partition_index));
	SPtr<uint8_t> uq = sptr<uint8_t>(slice + D_WEIGHTS);
	ASTC_NOUNROLL
	for (int t = lane; t < T; t += ASTC_WARP) {
		uint32_t ix = ASTC_LDD(&di.twi[t]);
		uint32_t cx = ASTC_LDD(&di.tci[t]);
		int i0 = (int)(ix & 0xFF), i1 = (int)((ix >> 8) & 0xFF), i2 = (int)((ix >> 16) & 0xFF), i3 = (int)(ix >> 24);
		int c0 = (int)(cx & 0xFF), c1 = (int)((cx >> 8) & 0xFF), c2 = (int)((cx >> 16) & 0xFF), c3 = (int)(cx >> 24);
		int w1 = (8 + uq[i0] * c0 + uq[i1] * c1 + uq[i2] * c2 + uq[i3] * c3) >> 4;
		out->weight_values_plane1[t] = static_cast<float>(w1) * (1.0f / 16.0f);
		if (dual) {
			int w2 = (8 + uq[32 + i0] * c0 + uq[32 + i1] * c1 + uq[32 + i2] * c2 + uq[32 + i3] * c3) >> 4;
			out->weight_values_plane2[t] = static_cast<float>(w2) * (1.0f / 16.0f);
		}
		out->partition_assignment[t] = ASTC_LDG(&pi.partition_of_texel[t]);
	}
}

// ---------------------------------------------------------------------------------------------
// astcenc_b200_get_block_summaries_device_images: the 16-byte summary of one block (struct astcenc_b200_block_summary) from the
// header stage alone, by one lane. Each field is the same-named field block_info writes, narrowed; error and constant blocks
// get their flag and zeros, as block_info returns early for them.
// ---------------------------------------------------------------------------------------------
// The 16 bytes of a block as two little-endian halves. A 16-byte aligned block is one vector load on the device.
ASTC_FN void load_block_bits(const uint8_t* pcb, uint64_t& lo, uint64_t& hi) {
#if !defined(ASTC_HOSTSIM)
	if ((reinterpret_cast<uintptr_t>(pcb) & 15) == 0) {
		const uint4 v = __ldg(reinterpret_cast<const uint4*>(pcb));
		lo = (uint64_t)v.x | ((uint64_t)v.y << 32);
		hi = (uint64_t)v.z | ((uint64_t)v.w << 32);
		return;
	}
#endif
	const uint32_t* p32 = reinterpret_cast<const uint32_t*>(pcb);
	lo = (uint64_t)ASTC_LDG(p32) | ((uint64_t)ASTC_LDG(p32 + 1) << 32);
	hi = (uint64_t)ASTC_LDG(p32 + 2) | ((uint64_t)ASTC_LDG(p32 + 3) << 32);
}

// *out (16-byte aligned) from four little-endian words in the struct's byte order: one vector store on the device.
ASTC_FN void store_summary(astcenc_b200_block_summary* out, uint32_t x, uint32_t y, uint32_t z, uint32_t w) {
#if defined(ASTC_HOSTSIM)
	uint32_t* p = reinterpret_cast<uint32_t*>(out);
	p[0] = x;
	p[1] = y;
	p[2] = z;
	p[3] = w;
#else
	*reinterpret_cast<uint4*>(out) = make_uint4(x, y, z, w);
#endif
}

ASTC_FN void block_summary(uint64_t lo, uint64_t hi, astcenc_b200_block_summary* out) {
	const BlockHeader h = block_header(lo, hi);
	if (h.block_type == SYM_BTYPE_ERROR) {
		store_summary(out, ASTCENC_B200_BLOCK_IS_ERROR, 0u, 0u, 0u);
		return;
	}
	if (h.block_type != SYM_BTYPE_NONCONST) {
		store_summary(out, ASTCENC_B200_BLOCK_IS_CONSTANT, 0u, 0u, 0u);
		return;
	}
	const DevBlockMode* bm = BSD.block_modes + h.block_mode_packed;
	const unsigned int d = ASTC_LDG(&bm->decimation_mode);
	// is_hdr_block is rgb_hdr || alpha_hdr of unpack_color_endpoints under the context's profile. The flags depend on the
	// endpoint mode and the profile alone, never on the colour values, so the modes are unpacked from zeros and the values are
	// not decoded. The LDR_ONLY form leaves out the HDR unpackers (and their local arrays); it sets rgb_hdr for every HDR mode,
	// as the general form does, so the disjunction is the same under every profile.
	bool is_hdr = false;
	unsigned int modes = 0;
	for (int p = 0; p < 4; p++) {
		if (p < h.partition_count) {
			const uint8_t zeros[8] = {0, 0, 0, 0, 0, 0, 0, 0};
			bool rgb_hdr, a_hdr;
			i4 e0, e1;
			unpack_color_endpoints_inl<true>(CFG.profile, h.color_formats[p], zeros, rgb_hdr, a_hdr, e0, e1);
			is_hdr = is_hdr || rgb_hdr || a_hdr;
			modes |= (unsigned int)h.color_formats[p] << (8 * p);
		}
	}
	const unsigned int flags = (is_hdr ? ASTCENC_B200_BLOCK_IS_HDR : 0u) | (h.dual ? ASTCENC_B200_BLOCK_IS_DUAL_PLANE : 0u);
	store_summary(out, flags | ((unsigned int)h.partition_count << 8) | ((unsigned int)h.partition_index << 16),
	              ((unsigned int)h.plane2_component & 0xFFu) | ((unsigned int)ASTC_LDG(&BSD.dec_modes[d].weight_x) << 8) |
	                  ((unsigned int)ASTC_LDG(&BSD.dec_modes[d].weight_y) << 16) | ((unsigned int)ASTC_LDG(&BSD.dec_modes[d].weight_z) << 24),
	              modes, quant_level_count(h.quant_mode) | (quant_level_count(h.weight_quant) << 16));
}
