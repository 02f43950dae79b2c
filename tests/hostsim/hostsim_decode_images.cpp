// TEST TOOL (not a product path): decode calls over image tables (decode_table_blocks, astc_dev_gather.cuh) on the host
// simulation of hostsim.cpp. Everything of hostsim_blocks.cpp, plus:
//   hostsim_decompress_images  decode_table_blocks over every block of a decode call, in shares of `share` call blocks, as the
//                              CTAs of astc_decompress_images_kernel take them (one simulated warp per CTA; one lane or 32)
// The table is built as astcenc_b200_decompress_device_images builds it (image_table: first[] is the exclusive prefix sum of
// the images' block counts); each entry's payload is read and its data written.
#include "hostsim_blocks.cpp"

// payloads[j] -> outs[j] (dim_z slices of dim_x * dim_y texels of data_type); swz uses astcenc_swz numbering.
extern "C" int hostsim_decompress_images(int profile, unsigned int bx, unsigned int by, unsigned int bz, unsigned int flags, const uint8_t* const* payloads,
                                         void* const* outs, const unsigned int* dims, unsigned int image_count, int data_type, const int* swz, size_t share) {
	astcenc_config cfg;
	if (astc_host::config_init((astcenc_profile)profile, bx, by, bz, 60.0f, flags, &cfg) != ASTCENC_SUCCESS) return 1;
	if (astc_host::validate_config(cfg) != ASTCENC_SUCCESS) return 2;
	if (image_count == 0 || share == 0) return 3;
	astc_host::PackedTables pk;
	astc_host::BlockSizeTables* t = astc_host::build_packed_tables(cfg, pk);
	astc_host::relocate_tables(pk, pk.blob.data());
	astc_host::fill_dev_const_tables(pk.consts);
	g_astc_ct = &pk.consts;
	DevConfig dcfg;
	astc_host::make_device_config(cfg, dcfg);
	std::vector<uint8_t> window(ASTC_SMEM_HDR + D_SLICE + 64, 0xCD);
	astc_smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(window.data()) + 15) & ~(uintptr_t)15);
	std::vector<GatherImage> table = image_table(const_cast<const void* const*>(outs), dims, image_count, bx, by, bz, const_cast<uint8_t* const*>(payloads));
	const GatherImage& last = table.back();
	const size_t total = last.first + (size_t)last.blocks_x * last.blocks_y * ((last.dim_z + bz - 1) / bz);
	// the launch's DevImage: the call's data type and swizzle, nothing else
	DevImage img{};
	img.data_type = data_type;
	for (int i = 0; i < 4; i++) img.swz[i] = swz ? swz[i] : i;
	SmemHdr* hdr = reinterpret_cast<SmemHdr*>(astc_smem);
	hdr->bsd = pk.bsd;
	hdr->cfg = dcfg;
	hdr->img = img;
	hdr->dec_smem_off = 0;
	hdr->cq_smem_off = 0;
	run_lanes([&](int lane) {
		for (size_t c0 = 0; c0 < total; c0 += share) {
			decode_table_blocks(table.data(), image_count, c0, c0 + share < total ? c0 + share : total, 0, 1, lane, ASTC_SMEM_HDR);
		}
	});
	astc_host::free_block_size_tables(t);
	return 0;
}
