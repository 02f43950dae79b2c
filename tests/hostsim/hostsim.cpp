// TEST TOOL (not a product path): compiles the warp-cooperative device source for the host (ASTC_HOSTSIM), so the
// kernels' logic can be checked against the oracle / reference without a GPU. Two builds:
//   default               one simulated lane: state machines, arithmetic order, table layouts (fast)
//   -DASTC_HOSTSIM_LANES32 32 host threads emulate the lanes of one warp, the CUDA warp primitives are collectives over
//                         them (simt_emul.h): shuffle partners, ordered sums across lanes, results that must be uniform
//                         across the warp, missing __syncwarp between producer and consumer lanes (slow: small images)
// The product library never links this.
#define ASTC_HOSTSIM 1
#if defined(ASTC_HOSTSIM_LANES32)
#include "simt_emul.h"
#endif
#include "../../astc-encoder_b200/csrc/astc_dev_search.cuh"
#include "../../astc-encoder_b200/csrc/astc_dev_gather.cuh"
#include "../../astc-encoder_b200/csrc/astc_host_pack.h"
#include "../../astc-encoder_b200/csrc/astc_host_config.h"
#include "../../astc-encoder_b200/csrc/astc_host_launch.h"
#include <vector>
#include <cstdio>
#include <cstring>
#include <cstdlib>

// run fn(lane) for every simulated lane
template <typename F> static void run_lanes(F fn) {
#if defined(ASTC_HOSTSIM_LANES32)
	simt::run_warp(fn);
#else
	fn(0);
#endif
}
extern "C" int hostsim_lanes() { return ASTC_WARP; }
// realign_weights calls that took the wavefront replay since the last call (32-lane build; the one-lane build runs the serial form)
extern "C" unsigned int hostsim_wavefront_replays() { unsigned int n = g_hostsim_wavefront_replays; g_hostsim_wavefront_replays = 0; return n; }

static unsigned int g_hostsim_a_scale_radius = 0;
extern "C" void hostsim_set_a_scale_radius(unsigned int r) { g_hostsim_a_scale_radius = r; }

// Volumes / 3D block sizes: data holds dim_z slices of dim_x * dim_y texels, contiguous; bz > 1 selects a 3D footprint and the
// blocks come out in (z, y, x) order. (2D block sizes: dim_z must be 1 here.)
extern "C" int hostsim_compress_volume(int profile, unsigned int bx, unsigned int by, unsigned int bz, float quality, unsigned int flags,
                                       const void* data, int data_type, unsigned int dim_x, unsigned int dim_y, unsigned int dim_z, const int* swz, uint8_t* out) {
	astcenc_config cfg;
	if (astc_host::config_init((astcenc_profile)profile, bx, by, bz, quality, flags, &cfg) != ASTCENC_SUCCESS) return 1;
	cfg.a_scale_radius = bz > 1 ? 0 : g_hostsim_a_scale_radius;
	if (astc_host::validate_config(cfg) != ASTCENC_SUCCESS) return 2;
	if (bz <= 1 && dim_z != 1) return 3;
	astc_host::PackedTables pk;
	astc_host::BlockSizeTables* t = astc_host::build_packed_tables(cfg, pk);
	astc_host::relocate_tables(pk, pk.blob.data());
	const DevBsd bsd_1p = pk.bsd_1p;
	astc_host::fill_dev_const_tables(pk.consts);
	g_astc_ct = &pk.consts;
	DevConfig dcfg;
	astc_host::make_device_config(cfg, dcfg);
	// the simulated shared window: launch constants, then one arena (16-byte aligned like the device's)
	std::vector<uint8_t> window(ASTC_SMEM_HDR + ASTC_SMEM_SINCOS_BYTES + pk.bsd.arena_bytes + 64 + 32 * EMIT_SLICE + ASTC_REFINE_STATE_BYTES, 0xCD);
	astc_smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(window.data()) + 15) & ~(uintptr_t)15);
	DevImage img;
	img.data = data;
	img.data_type = data_type;
	img.dim_x = dim_x;
	img.dim_y = dim_y;
	img.dim_z = dim_z;
	img.blocks_x = (dim_x + bx - 1) / bx;
	img.blocks_y = (dim_y + by - 1) / by;
	img.block_row0 = 0;
	img.block_rows = img.blocks_y * (bz > 1 ? (dim_z + bz - 1) / bz : 1);
	for (int i = 0; i < 4; i++) img.swz[i] = swz ? swz[i] : i;
	img.out = out;
	img.alpha_avg = nullptr;
	img.alpha_threshold = 0.0f;
	std::vector<float> alpha_avg;
	if (cfg.a_scale_radius != 0) {
		// the pre-pass, tile by tile, through the device source (the simulated lanes stand in for the CTA's threads)
		unsigned int r = cfg.a_scale_radius;
		alpha_avg.resize((size_t)dim_x * dim_y);
		size_t pad = ALPHA_TILE + 2 * (size_t)r + 1;
		std::vector<uint8_t> tile_mem(pad * pad * 4 + 64);
		uint8_t* saved = astc_smem;
		astc_smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(tile_mem.data()) + 15) & ~(uintptr_t)15);
		run_lanes([&](int lane) {
			for (unsigned int oy = 0; oy < dim_y; oy += ALPHA_TILE) {
				for (unsigned int ox = 0; ox < dim_x; ox += ALPHA_TILE) {
					alpha_average_tile(img, r, ox, oy, 0, alpha_avg.data(), lane, ASTC_WARP);
					cta_sync();      // (on the device every tile is its own CTA; here the same lanes reuse the tile buffer)
				}
			}
		});
		astc_smem = saved;
		img.alpha_avg = alpha_avg.data();
		size_t x_footprint = bx + 2 * ((size_t)r - 1), y_footprint = by + 2 * ((size_t)r - 1);
		img.alpha_threshold = 0.9f / (255.0f * static_cast<float>(x_footprint * y_footprint));
	}
	SmemHdr* hdr = reinterpret_cast<SmemHdr*>(astc_smem);
	hdr->bsd = pk.bsd;
	hdr->cfg = dcfg;
	hdr->img = img;
	hdr->dec_smem_off = 0;
	hdr->cq_smem_off = 0;
	const uint32_t arena_base = ASTC_SMEM_HDR + ASTC_SMEM_SINCOS_BYTES;
	{
		float* sc = reinterpret_cast<float*>(astc_smem + ASTC_SMEM_HDR);
		for (int j = 0; j < 64; j++) {
			for (int i = 0; i < ASTC_ANGULAR_STEPS; i++) {
				sc[j * ASTC_ANGULAR_STEPS + i] = pk.consts.cos_table[j][i];
				sc[64 * ASTC_ANGULAR_STEPS + j * ASTC_ANGULAR_STEPS + i] = pk.consts.sin_table[j][i];
			}
		}
	}
	const char* driver = getenv("HOSTSIM_DRIVER");
	unsigned int counter = 0;
	unsigned int total = img.blocks_x * img.block_rows;
	std::vector<uint8_t> records((size_t)total * pk.bsd.record_bytes + 16);
	std::vector<uint32_t> queues((size_t)ASTC_Q_KINDS * total);
	std::vector<uint32_t> counters(2 * ASTC_Q_KINDS * ASTC_MAX_WAVES, 0);
	run_lanes([&](int lane) {
		WCtx w;
		w.lane = lane;
		w.base = arena_base;
		w.T = pk.bsd.texel_count;
		if (driver && !strcmp(driver, "warp")) {
			for (unsigned int y = 0; y < img.block_rows; y++) {
				for (unsigned int x = 0; x < img.blocks_x; x++) {
					load_block(w, x, y);
					compress_block(w, out + ((size_t)y * img.blocks_x + x) * 16);
				}
			}
		} else if (driver && !strcmp(driver, "lockstep")) {
			BlockFeed feed;
			feed.ticket = &counter;
			feed.total = img.blocks_x * img.block_rows;
			feed.blocks_x = img.blocks_x;
			compress_blocks_lockstep(w, feed, ASTC_SMEM_HDR + ASTC_SMEM_SINCOS_BYTES + pk.bsd.arena_bytes + 32 * EMIT_SLICE + 16);
		} else {
			// the wave pipeline, driven like the CUDA host code does (one simulated warp per "kernel")
			WaveArgs a;
			a.records = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(records.data()) + 15) & ~(uintptr_t)15);
			a.queues = queues.data();
			a.queue_stride = total;
			a.count = counters.data();
			a.head = counters.data() + ASTC_Q_KINDS * ASTC_MAX_WAVES;
			a.total = total;
			a.blocks_x = img.blocks_x;
			a.ticket = &counter;
			a.first_block = 0;
			a.band_blocks = total;
			a.cls_lo = 0;
			a.cls_hi = ASTC_Q_CLASSES;
			a.sync_mask = 0xFF;
			a.stage_bytes = 0;
			a.refine_state_off = ASTC_SMEM_HDR + ASTC_SMEM_SINCOS_BYTES + pk.bsd.arena_bytes + 32 * EMIT_SLICE + 16;
			a.stage_bytes_setup = 0;
			for (int wave = 0; wave < ASTC_MAX_WAVES - 1; wave++) {
				a.wave = wave;
				// (like the CUDA host code: trials with one weight plane - wave 0, the n-partition classes - run on the compact plan)
				const bool compact = !getenv("HOSTSIM_NO_1P");
				if (wave != 0 && compact) {
					cta_sync();
					if (lane == 0) {
						hdr->bsd = pk.bsd;
					}
					cta_sync();
					a.cls_lo = 0;
					a.cls_hi = 1;
					wave_setup(w, a);
					a.cls_lo = 1;
					a.cls_hi = ASTC_Q_CLASSES;
				}
				cta_sync();
				if (lane == 0) {
					hdr->bsd = compact ? bsd_1p : pk.bsd;
				}
				cta_sync();
				wave_setup(w, a);
				a.cls_lo = 0;
				a.cls_hi = ASTC_Q_CLASSES;
				cta_sync();
				if (lane == 0) {
					hdr->bsd = pk.bsd;
				}
				cta_sync();
				wave_refine(w, a, 0);
				wave_prepare(w, a);
			}
			a.wave = 0;
			wave_emit(lane, ASTC_SMEM_HDR + ASTC_SMEM_SINCOS_BYTES + pk.bsd.arena_bytes, a);
		}
	});
	astc_host::free_block_size_tables(t);
	return 0;
}

extern "C" int hostsim_compress_image(int profile, unsigned int bx, unsigned int by, float quality, unsigned int flags,
                                      const void* data, int data_type, unsigned int dim_x, unsigned int dim_y, const int* swz, uint8_t* out) {
	return hostsim_compress_volume(profile, bx, by, 1, quality, flags, data, data_type, dim_x, dim_y, 1, swz, out);
}

// decompression through the device source (one simulated lane): the table walk of astc_decompress_images_kernel over a one-entry
// table, as astcenc_decompress_image builds it. swz uses astcenc_swz numbering.
extern "C" int hostsim_decompress_volume(int profile, unsigned int bx, unsigned int by, unsigned int bz, unsigned int flags, const uint8_t* blocks, void* out, int data_type,
                                         unsigned int dim_x, unsigned int dim_y, unsigned int dim_z, const int* swz) {
	astcenc_config cfg;
	if (astc_host::config_init((astcenc_profile)profile, bx, by, bz, 60.0f, flags, &cfg) != ASTCENC_SUCCESS) return 1;
	if (astc_host::validate_config(cfg) != ASTCENC_SUCCESS) return 2;
	if (bz <= 1 && dim_z != 1) return 3;
	astc_host::PackedTables pk;
	astc_host::BlockSizeTables* t = astc_host::build_packed_tables(cfg, pk);
	astc_host::relocate_tables(pk, pk.blob.data());
	astc_host::fill_dev_const_tables(pk.consts);
	g_astc_ct = &pk.consts;
	DevConfig dcfg;
	astc_host::make_device_config(cfg, dcfg);
	std::vector<uint8_t> window(ASTC_SMEM_HDR + D_SLICE + 64, 0xCD);
	astc_smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(window.data()) + 15) & ~(uintptr_t)15);
	GatherImage e;
	e.data = out;
	e.payload = const_cast<uint8_t*>(blocks);
	e.first = 0;
	e.avg_offset = 0;
	e.dim_x = dim_x;
	e.dim_y = dim_y;
	e.dim_z = dim_z;
	e.blocks_x = (dim_x + bx - 1) / bx;
	e.blocks_y = (dim_y + by - 1) / by;
	const size_t total = (size_t)e.blocks_x * e.blocks_y * (bz > 1 ? (dim_z + bz - 1) / bz : 1);
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
		decode_table_blocks(&e, 1, 0, total, 0, 1, lane, ASTC_SMEM_HDR);
	});
	astc_host::free_block_size_tables(t);
	return 0;
}

extern "C" int hostsim_decompress_image(int profile, unsigned int bx, unsigned int by, unsigned int flags, const uint8_t* blocks, void* out, int data_type,
                                        unsigned int dim_x, unsigned int dim_y, const int* swz) {
	return hostsim_decompress_volume(profile, bx, by, 1, flags, blocks, out, data_type, dim_x, dim_y, 1, swz);
}

extern "C" unsigned int hostsim_arena_bytes_3d(int profile, unsigned int bx, unsigned int by, unsigned int bz, float quality, unsigned int flags) {
	astcenc_config cfg;
	if (astc_host::config_init((astcenc_profile)profile, bx, by, bz, quality, flags, &cfg) != ASTCENC_SUCCESS) return 0;
	astc_host::validate_config(cfg);
	astc_host::PackedTables pk;
	astc_host::free_block_size_tables(astc_host::build_packed_tables(cfg, pk));
	fprintf(stderr, "%ux%ux%u arena %u (1-plane plan %u) small %u | scratch@%u (%u B) ei@%u dwi@%u lowhigh@%u mode_err@%u record %u | dec modes %u block modes %u | dec tables %u B\n",
	        bx, by, bz, pk.bsd.arena_bytes, pk.bsd_1p.arena_bytes, pk.bsd.arena_bytes_small, pk.bsd.off_scratch, pk.bsd.scratch_bytes, pk.bsd.off_ei, pk.bsd.off_dwi,
	        pk.bsd.off_lowhigh, pk.bsd.off_mode_err, pk.bsd.record_bytes, pk.bsd.decimation_mode_count_selected, pk.bsd.block_mode_count_1plane_2plane_selected, pk.bsd.dec_stage_bytes);
	return pk.bsd.arena_bytes;
}

extern "C" unsigned int hostsim_arena_bytes(int profile, unsigned int bx, unsigned int by, float quality, unsigned int flags) {
	astcenc_config cfg;
	if (astc_host::config_init((astcenc_profile)profile, bx, by, 1, quality, flags, &cfg) != ASTCENC_SUCCESS) return 0;
	astc_host::validate_config(cfg);
	astc_host::PackedTables pk;
	astc_host::free_block_size_tables(astc_host::build_packed_tables(cfg, pk));
	if (getenv("HOSTSIM_ARENA_PRINT")) {
		fprintf(stderr, "arena %u small %u | fixed %u scratch@%u (%u B) ei@%u dwi@%u lowhigh@%u mode_err@%u record %u | dec modes %u block modes %u | dec tables %u B\n",
		        pk.bsd.arena_bytes, pk.bsd.arena_bytes_small, (unsigned)ASTC_ARENA_FIXED, pk.bsd.off_scratch, pk.bsd.scratch_bytes, pk.bsd.off_ei, pk.bsd.off_dwi,
		        pk.bsd.off_lowhigh, pk.bsd.off_mode_err, pk.bsd.record_bytes, pk.bsd.decimation_mode_count_selected, pk.bsd.block_mode_count_1plane_2plane_selected, pk.bsd.dec_stage_bytes);
	}
	return pk.bsd.arena_bytes;
}

// The launch plan (astc_host_launch.h) of a compressing context with these knobs on an SM of smem_limit bytes of opt-in shared memory.
// Returns the astcenc_error of plan_kernels, or -1 when the configuration itself is refused.
extern "C" int hostsim_kernel_plan(int profile, unsigned int bx, unsigned int by, unsigned int bz, float quality, unsigned int flags, size_t smem_limit,
                                   int sm_count, const Knobs* knobs, KernelPlan* out) {
	astcenc_config cfg;
	if (astc_host::config_init((astcenc_profile)profile, bx, by, bz, quality, flags, &cfg) != ASTCENC_SUCCESS) return -1;
	if (astc_host::validate_config(cfg) != ASTCENC_SUCCESS) return -1;
	astc_host::PackedTables pk;
	astc_host::BlockSizeTables* t = astc_host::build_packed_tables(cfg, pk);
	int status = (int)plan_kernels(pk.bsd, pk.bsd_1p, cfg, smem_limit, sm_count, *knobs, *out);
	astc_host::free_block_size_tables(t);
	return status;
}
