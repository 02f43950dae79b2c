// Table layouts shared by the host packer (astc_host_tables.cpp) and the sm_90a kernels.
// Everything is plain-old-data addressed through raw pointers so one struct can be copied to the GPU.
//
// What each table restates (reference file:line, relative to /root/reference/Source):
//   block_mode / decimation_mode        astcenc_internal.h:418-512
//   decimation_info (bilinear tables)   astcenc_internal.h:347-413   -> compact blob per grid (see DecBlob)
//   partition_info                      astcenc_internal.h:313-334   -> compact entry per partitioning
//   quant_and_xfer_tables, colour quant astcenc_weight_quant_xfer_tables.cpp:26, astcenc_quantization.cpp:27
#pragma once
#include <stdint.h>

#define ASTC_MAX_TEXELS 216     /* 6x6x6; the largest 2D block (12x12) has 144 */
#define ASTC_MAX_WEIGHTS 64
#define ASTC_MAX_PARTITIONINGS 1024
#define ASTC_MAX_BLOCK_MODES 2048
#define ASTC_MAX_DECIMATION_MODES 87
#define ASTC_MAX_KMEANS_TEXELS 64
/* Per-warp arena head (astc_dev_core.cuh A_*): bytes before the block texels, and the part of it that, together with the
   block texels, forms a block's persistent record between stage kernels */
#define ASTC_ARENA_FIXED 2848      /* head 2320 + chain results 512 + 16 for the warp's bulk-copy mbarrier */
#define ASTC_ARENA_PERSIST_HEAD 1808
#define ASTC_ANGULAR_STEPS 12     /* TUNE_MAX_ANGULAR_QUANT = 7 -> at most 12 steps are ever evaluated */

enum { QUANT_2 = 0, QUANT_3, QUANT_4, QUANT_5, QUANT_6, QUANT_8, QUANT_10, QUANT_12, QUANT_16, QUANT_20, QUANT_24,
       QUANT_32, QUANT_40, QUANT_48, QUANT_64, QUANT_80, QUANT_96, QUANT_128, QUANT_160, QUANT_192, QUANT_256 };

struct DevConstTables {
	uint8_t integer_of_trits[243];          // [((t4*3+t3)*3+t2)*3+t1)*3+t0]
	uint8_t integer_of_quints[125];         // [(q2*5+q1)*5+q0]
	uint8_t color_unquant_to_uquant[17][512];
	uint8_t color_uquant_to_scrambled_pquant[17][256];
	int8_t quant_mode_table[10][128];
	uint8_t wq_quant_to_unquant[12][32];
	uint8_t wq_scramble_map[12][32];
	uint16_t wq_prev_next[12][65];
	// decompression only
	uint8_t trits_of_integer[256][5];
	uint8_t quints_of_integer[128][3];
	uint8_t wq_unscramble_and_unquant[12][32];
	uint8_t color_scrambled_pquant_to_uquant[17][256];
	float sin_table[64][ASTC_ANGULAR_STEPS];
	float cos_table[64][ASTC_ANGULAR_STEPS];
};

struct DevBlockMode {
	uint16_t mode_index;
	uint8_t decimation_mode;
	uint8_t quant_mode;
	uint8_t weight_bits;
	uint8_t is_dual_plane;
};

// Per weight grid. The bilinear tables live in a blob (16-byte aligned), packed so that one texel / one list
// entry is one load:
//   tcf[T] float4    the (up to) 4 contributions of a texel as floats, c / 16 (0 = unused)   (texel_weight_contribs_float_tr)
//   twi[T] u32       the 4 grid weights a texel reads, one byte each                          (texel_weights_tr)
//   tci[T] u32       the 4 contributions in 1/16ths, one byte each                            (texel_weight_contribs_int_tr)
//   wto[W+1] u16     CSR offsets of the weight -> texel lists
//   wtc[E] u16       list entries: texel | contribution-in-1/16ths << 8    (weight_texels_tr, weights_texel_contribs_tr)
// Float contributions are c * (1/16) resp. float(c): both are exact, so the values equal the reference's
// stored floats bit for bit.
struct DevDecMode {
	int8_t maxprec_1plane;
	int8_t maxprec_2planes;
	uint16_t refprec_1plane;
	uint16_t refprec_2planes;
	uint8_t weight_count;
	uint8_t weight_x;
	uint8_t weight_y;
	uint8_t max_texel_weight_count;
	uint16_t dwi_offset;      // float offset of this grid's ideal weights in the per-warp arena
	uint16_t wto_offset;      // byte offset of wto inside the blob (= 24 * T)
	uint16_t wtc_offset;      // byte offset of wtc
	uint16_t max_weight_texels;   // longest weight -> texel list of this grid
	uint16_t dwi_offset_1p;   // the same in the compact one-plane arena layout (DevBsd::layout_planes == 1)
	uint8_t weight_z;         // 1 for the grids of 2D block sizes
	uint8_t pad_[1];
	uint32_t blob_offset;     // byte offset of the blob in dec_blob
};

// Partition entry, stride part_stride bytes:
//   u16 partition_index (the 10-bit seed); u8 count[4]; u8 pad[2];
//   u8 partition_of_texel[T]; u8 texels[T]  (texels_of_partition concatenated in partition order)
#define ASTC_PART_HDR 8

struct DevBsd {
	uint8_t dim_x, dim_y, texel_count, max_weight_texel_count;
	uint8_t dim_z, pad_[3];      // dim_z > 1: one of the ten 3D footprints (astcenc_block_sizes.cpp:1025)
	uint32_t decimation_mode_count_always, decimation_mode_count_selected, decimation_mode_count_all;
	uint32_t block_mode_count_1plane_always, block_mode_count_1plane_selected, block_mode_count_1plane_2plane_selected, block_mode_count_all;
	uint32_t partitioning_count_selected[4];
	uint32_t part_stride;
	const DevBlockMode* block_modes;
	const uint16_t* block_mode_packed_index;    // [2048]
	const DevDecMode* dec_modes;
	const uint8_t* dec_blob;
	uint32_t dec_stage_bytes;                   // prefix of dec_blob that holds every grid the search can select
	const uint8_t* partitions[5];               // [1]: single entry, [2..4]: packed partitionings
	const uint16_t* partitioning_packed_index[3];
	const uint64_t* coverage_bitmaps[5];        // [pc][packed * pc + p]
	uint8_t kmeans_texels[ASTC_MAX_KMEANS_TEXELS];
	// per-warp arena layout (byte offsets from the arena base, 16-byte aligned) and size. The fixed part
	// (state, endpoint slots, symbolic block arrays, chain results, candidates, block texels, ideal weights) is
	// laid out by astc_dev_core.cuh (A_* constants); the block-size dependent tail is planned by the host.
	uint32_t arena_bytes;        // everything (the trial-setup kernel)
	uint32_t arena_bytes_small;  // up to the end of the union scratch (refinement / partition-search kernels)
	uint32_t off_scratch, off_ei, off_dwi, off_lowhigh, off_mode_err;
	uint32_t scratch_bytes;      // size of the union scratch at off_scratch
	uint32_t record_bytes;       // ASTC_ARENA_PERSIST_HEAD + 16 * Tp, rounded to 16
	// Two plans of the set-up tail exist: the general one (ideal weights, decimated weights and angular ranges for TWO weight
	// planes) and a compact one for trials with ONE plane (wave 0 - every block's first trial - never has two): fewer bytes
	// per block, more blocks in flight per SM. The kernel is told which plan its launch uses.
	uint32_t layout_planes;      // 2 (general) or 1 (compact)
};

// The search configuration consumed on the device (subset of astcenc_config, astcenc.h:427-605).
struct DevConfig {
	int profile;
	unsigned int flags;
	float cw[4];
	float rgbm_m_scale;
	unsigned int tune_partition_count_limit;
	unsigned int tune_partition_index_limit[3];
	unsigned int tune_refinement_limit;
	unsigned int tune_candidate_limit;
	unsigned int tune_partitioning_candidate_limit[3];
	float tune_db_limit;
	float tune_mse_overshoot;
	float tune_2partition_early_out_limit_factor;
	float tune_3partition_early_out_limit_factor;
	float tune_2plane_early_out_limit_correlation;
	float tune_search_mode0_enable;
};

// Where a DevImage's progress words point unless they are set: nowhere (progress and cancellation off). A host-simulation
// harness may define these to its own words before it includes the device source (tests/hostsim/hostsim_progress.cpp).
#ifndef ASTC_PASS_CANCEL_DEFAULT
#define ASTC_PASS_CANCEL_DEFAULT nullptr
#endif
#ifndef ASTC_PASS_DONE_DEFAULT
#define ASTC_PASS_DONE_DEFAULT nullptr
#endif

// One image (or slab) to compress.
struct DevImage {
	const void* data;          // RGBA texels, row-major, tightly packed
	int data_type;             // 0 = U8, 1 = F16, 2 = F32
	unsigned int dim_x, dim_y; // full image size (for clamp-to-edge)
	unsigned int dim_z;        // slices of a volume (3D block sizes only; 2D block sizes see one slice per pass), contiguous in data
	unsigned int blocks_x;
	unsigned int blocks_y;     // 3D block sizes: block rows per layer of blocks; a "block row" index then counts layer * blocks_y + row
	unsigned int block_row0;   // first block row of this launch (slab sharding)
	unsigned int block_rows;   // number of block rows in this launch
	int swz[4];
	uint8_t* out;              // 16 bytes per block, slab-relative
	const float* alpha_avg;    // per-texel alpha averages of the alpha-scale pre-pass, or NULL
	float alpha_threshold;     // blocks with no average above this are emitted as constant zero
	// progress and cancellation (astc_dev_lockstep.cuh, pass_cancelled) for the kernels that take no WaveArgs: the alpha-scale
	// pre-pass and the single-kernel drivers; null = off
	const uint32_t* cancel = ASTC_PASS_CANCEL_DEFAULT;
	uint32_t* done = ASTC_PASS_DONE_DEFAULT;
};
