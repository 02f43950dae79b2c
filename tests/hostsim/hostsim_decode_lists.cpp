// TEST TOOL (not a product path): decode calls over device block lists (decode_list_blocks, astc_dev_gather.cuh) on the host
// simulation of hostsim.cpp. Everything of hostsim_blocks.cpp, plus:
//   hostsim_decompress_block_lists  decode_list_blocks over every slot of a list decode call, in shares of `share` slots, as the
//                                   one-warp CTAs of astc_decompress_block_lists_kernel take them (one lane or 32)
// The table is built as astcenc_b200_decompress_device_block_lists builds it: entries of capacity 0 are left out, and first[] is the
// exclusive prefix sum of the other entries' capacities.
#include "hostsim_blocks.cpp"

// payloads[j] -> outs[j] (dim_z slices of dim_x * dim_y texels of data_type) at the blocks of list j: indices[j], the count word
// counts[j] and capacities[j]. swz uses astcenc_swz numbering. Returns 0, or non-zero for a configuration that is refused.
extern "C" int hostsim_decompress_block_lists(int profile, unsigned int bx, unsigned int by, unsigned int bz, unsigned int flags, const uint8_t* const* payloads,
                                              void* const* outs, const unsigned int* dims, unsigned int image_count, int data_type, const int* swz,
                                              const uint32_t* const* indices, const uint32_t* counts, const unsigned int* capacities, size_t share) {
	astcenc_config cfg;
	if (astc_host::config_init((astcenc_profile)profile, bx, by, bz, 60.0f, flags, &cfg) != ASTCENC_SUCCESS) return 1;
	if (astc_host::validate_config(cfg) != ASTCENC_SUCCESS) return 2;
	if (share == 0) return 3;
	std::vector<GatherImage> table;
	std::vector<GatherList> lists;
	size_t total = 0;
	for (unsigned int j = 0; j < image_count; j++) {
		if (capacities[j] == 0) {
			continue;
		}
		GatherImage e = image_table(const_cast<const void* const*>(outs) + j, dims + 3 * j, 1, bx, by, bz, const_cast<uint8_t* const*>(payloads) + j)[0];
		e.first = total;
		table.push_back(e);
		lists.push_back({indices[j], counts + j, capacities[j], e.blocks_x * e.blocks_y * ((e.dim_z + bz - 1) / bz)});
		total += capacities[j];
	}
	if (total == 0) {
		return 0;      // (the library launches nothing)
	}
	astc_host::PackedTables pk;
	astc_host::BlockSizeTables* t = astc_host::build_packed_tables(cfg, pk);
	astc_host::relocate_tables(pk, pk.blob.data());
	astc_host::fill_dev_const_tables(pk.consts);
	g_astc_ct = &pk.consts;
	DevConfig dcfg;
	astc_host::make_device_config(cfg, dcfg);
	std::vector<uint8_t> window(ASTC_SMEM_HDR + D_SLICE + 64, 0xCD);
	astc_smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(window.data()) + 15) & ~(uintptr_t)15);
	// the launch's DevImage: the call's data type and swizzle, nothing else
	DevImage img{};
	img.data_type = data_type;
	for (int i = 0; i < 4; i++) img.swz[i] = swz ? swz[i] : i;
	SmemHdr* hdr = reinterpret_cast<SmemHdr*>(astc_smem);
	hdr->bsd = pk.bsd;
	hdr->cfg = dcfg;
	hdr->dec_smem_off = 0;
	hdr->cq_smem_off = 0;
	run_lanes([&](int lane) {
		for (size_t c0 = 0; c0 < total; c0 += share) {
			// every CTA starts from the launch constants: nothing staged
			cta_sync();
			if (lane == 0) {
				hdr->img = img;
			}
			cta_sync();
			decode_list_blocks(table.data(), lists.data(), (unsigned int)table.size(), c0, c0 + share < total ? c0 + share : total, lane, ASTC_SMEM_HDR);
		}
	});
	astc_host::free_block_size_tables(t);
	return 0;
}
