// TEST TOOL (not a product path): block info of device payloads (astc_dev_gather.cuh, astc_dev_decode.cuh) on the host
// simulation of hostsim.cpp. Everything of hostsim_blocks.cpp, plus:
//   hostsim_block_summaries   summarize_table_blocks over every block of a summary call, lane-strided over the simulated lanes
//                             (one lane or 32), as the threads of astc_block_summaries_kernel take them grid-stride
//   hostsim_block_info_lists  info_list_slot over every slot of a list call, each slot by the whole simulated warp, as the warps
//                             of astc_block_info_lists_kernel take them
// The tables are built as the library builds them: a summary call's entry j owns its image's blocks; a list call leaves out the
// entries of capacity 0, and first[] is the exclusive prefix sum of the other entries' capacities.
#include "hostsim_blocks.cpp"

namespace {
// The context's tables and launch constants in the simulated shared window (one decode slice behind the header).
struct InfoSim {
	astcenc_config cfg;
	astc_host::PackedTables pk;
	astc_host::BlockSizeTables* t = nullptr;
	std::vector<uint8_t> window;
	BlockInfoHead head;
	int init(int profile, unsigned int bx, unsigned int by, unsigned int bz, unsigned int flags) {
		if (astc_host::config_init((astcenc_profile)profile, bx, by, bz, 60.0f, flags, &cfg) != ASTCENC_SUCCESS) return 1;
		if (astc_host::validate_config(cfg) != ASTCENC_SUCCESS) return 2;
		t = astc_host::build_packed_tables(cfg, pk);
		astc_host::relocate_tables(pk, pk.blob.data());
		astc_host::fill_dev_const_tables(pk.consts);
		g_astc_ct = &pk.consts;
		DevConfig dcfg;
		astc_host::make_device_config(cfg, dcfg);
		window.assign(ASTC_SMEM_HDR + D_SLICE + 64, 0xCD);
		astc_smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(window.data()) + 15) & ~(uintptr_t)15);
		SmemHdr* hdr = reinterpret_cast<SmemHdr*>(astc_smem);
		hdr->bsd = pk.bsd;
		hdr->cfg = dcfg;
		hdr->img = DevImage{};
		hdr->dec_smem_off = 0;
		hdr->cq_smem_off = 0;
		head = {(int)cfg.profile, cfg.block_x, cfg.block_y, cfg.block_z, pk.bsd.texel_count};
		return 0;
	}
	~InfoSim() {
		if (t) astc_host::free_block_size_tables(t);
	}
};
}

// payloads[j] -> summaries[j] (one 16-byte summary per block). dims: dim_x, dim_y, dim_z of each image.
extern "C" int hostsim_block_summaries(int profile, unsigned int bx, unsigned int by, unsigned int bz, unsigned int flags, const uint8_t* const* payloads,
                                       void* const* summaries, const unsigned int* dims, unsigned int image_count) {
	InfoSim sim;
	int rc = sim.init(profile, bx, by, bz, flags);
	if (rc != 0) return rc;
	if (image_count == 0) return 0;      // (the library launches nothing)
	std::vector<GatherImage> table = image_table(const_cast<const void* const*>(summaries), dims, image_count, bx, by, bz, const_cast<uint8_t* const*>(payloads));
	const size_t total = table.back().first + (size_t)table.back().blocks_x * table.back().blocks_y * ((table.back().dim_z + bz - 1) / bz);
	run_lanes([&](int lane) { summarize_table_blocks(table.data(), image_count, (size_t)lane, total, ASTC_WARP); });
	return 0;
}

// payloads[j] at the slots of list j (indices[j], the count word counts[j], capacities[j]) -> infos[j] (capacities[j] structs).
extern "C" int hostsim_block_info_lists(int profile, unsigned int bx, unsigned int by, unsigned int bz, unsigned int flags, const uint8_t* const* payloads,
                                        void* const* infos, const unsigned int* dims, unsigned int image_count, const uint32_t* const* indices,
                                        const uint32_t* counts, const unsigned int* capacities) {
	InfoSim sim;
	int rc = sim.init(profile, bx, by, bz, flags);
	if (rc != 0) return rc;
	std::vector<GatherImage> table;
	std::vector<GatherList> lists;
	size_t total = 0;
	for (unsigned int j = 0; j < image_count; j++) {
		if (capacities[j] == 0) {
			continue;
		}
		GatherImage e = image_table(const_cast<const void* const*>(infos) + j, dims + 3 * j, 1, bx, by, bz, const_cast<uint8_t* const*>(payloads) + j)[0];
		e.first = total;
		table.push_back(e);
		lists.push_back({indices[j], counts + j, capacities[j], e.blocks_x * e.blocks_y * ((e.dim_z + bz - 1) / bz)});
		total += capacities[j];
	}
	run_lanes([&](int lane) {
		for (size_t c = 0; c < total; c++) {
			info_list_slot(table.data(), lists.data(), (unsigned int)table.size(), c, lane, ASTC_SMEM_HDR, sim.head);
		}
	});
	return 0;
}
