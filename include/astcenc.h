/*
 * astcenc.h - C ABI of the CUDA-native ASTC block compressor for the NVIDIA H100 (libastcenc_b200.so).
 *
 * This is the drop-in boundary: the library exports exactly the entry points that the reference
 * codec's public header declares, with identical names, argument meaning, struct layouts and error
 * behaviour, so the reference command line tool, its unit tests and any application written against
 * the reference API can be relinked against this library unchanged.
 *
 * Reference interface replaced by each declaration (file:line in /root/reference/Source):
 *   astcenc_error / profile / swz / type enums ....... astcenc.h:207-236, 241-256, 284-313, 318-329
 *   astcenc_config ................................... astcenc.h:427-605
 *   astcenc_image .................................... astcenc.h:613-629
 *   astcenc_block_info ............................... astcenc.h:637-717
 *   astcenc_config_init .............................. astcenc.h:725-749  (impl astcenc_entry.cpp:504)
 *   astcenc_context_alloc ............................ astcenc.h:751-772  (impl astcenc_entry.cpp:726)
 *   astcenc_compress_image ........................... astcenc.h:774-799  (impl astcenc_entry.cpp:1113)
 *   astcenc_compress_reset / _cancel ................. astcenc.h:801-823  (impl astcenc_entry.cpp:1231, :1251)
 *   astcenc_decompress_image / _reset ................ astcenc.h:825-861  (impl astcenc_entry.cpp:1274, :1389)
 *   astcenc_context_free ............................. astcenc.h:863-868  (impl astcenc_entry.cpp:862)
 *   astcenc_get_block_info ........................... astcenc.h:870-884  (impl astcenc_entry.cpp:1401)
 *   astcenc_get_error_string ......................... astcenc.h:886-894  (impl astcenc_entry.cpp:1520)
 *
 * Threading contract (same as the reference): a context compresses one image at a time; up to
 * `thread_count` callers may enter astcenc_compress_image() with distinct thread_index values, any
 * subset may actually call, and all of them return once the image is complete. Here the first
 * arrival drives the GPU (upload, kernel, download) and the others simply wait.
 *
 * Extensions (prefix astcenc_b200_) expose device-resident buffers and slab sharding for multi-GPU use.
 */
#ifndef ASTCENC_B200_PUBLIC_H
#define ASTCENC_B200_PUBLIC_H

#include <stddef.h>
#include <stdint.h>

#if defined(__cplusplus)
	#define ASTCENC_B200_EXTERN extern "C"
#else
	#include <stdbool.h>
	#define ASTCENC_B200_EXTERN
#endif
#define ASTCENC_PUBLIC ASTCENC_B200_EXTERN __attribute__((visibility("default")))

struct astcenc_context;

enum astcenc_error {
	ASTCENC_SUCCESS = 0,
	ASTCENC_ERR_OUT_OF_MEM,
	ASTCENC_ERR_BAD_CPU_FLOAT,
	ASTCENC_ERR_BAD_PARAM,
	ASTCENC_ERR_BAD_BLOCK_SIZE,
	ASTCENC_ERR_BAD_PROFILE,
	ASTCENC_ERR_BAD_QUALITY,
	ASTCENC_ERR_BAD_SWIZZLE,
	ASTCENC_ERR_BAD_FLAGS,
	ASTCENC_ERR_BAD_CONTEXT,
	ASTCENC_ERR_NOT_IMPLEMENTED,
	ASTCENC_ERR_BAD_DECODE_MODE
};

enum astcenc_profile { ASTCENC_PRF_LDR_SRGB = 0, ASTCENC_PRF_LDR, ASTCENC_PRF_HDR_RGB_LDR_A, ASTCENC_PRF_HDR };

/* search quality presets (any value in [0, 100] is accepted and interpolated) */
static const float ASTCENC_PRE_FASTEST = 0.0f;
static const float ASTCENC_PRE_FAST = 10.0f;
static const float ASTCENC_PRE_MEDIUM = 60.0f;
static const float ASTCENC_PRE_THOROUGH = 98.0f;
static const float ASTCENC_PRE_VERYTHOROUGH = 99.0f;
static const float ASTCENC_PRE_EXHAUSTIVE = 100.0f;

enum astcenc_swz { ASTCENC_SWZ_R = 0, ASTCENC_SWZ_G = 1, ASTCENC_SWZ_B = 2, ASTCENC_SWZ_A = 3, ASTCENC_SWZ_0 = 4, ASTCENC_SWZ_1 = 5, ASTCENC_SWZ_Z = 6 };

struct astcenc_swizzle {
	enum astcenc_swz r;
	enum astcenc_swz g;
	enum astcenc_swz b;
	enum astcenc_swz a;
};

enum astcenc_type { ASTCENC_TYPE_U8 = 0, ASTCENC_TYPE_F16 = 1, ASTCENC_TYPE_F32 = 2 };

ASTCENC_B200_EXTERN typedef void (*astcenc_progress_callback)(float);

static const unsigned int ASTCENC_FLG_MAP_NORMAL = 1 << 0;
static const unsigned int ASTCENC_FLG_USE_DECODE_UNORM8 = 1 << 1;
static const unsigned int ASTCENC_FLG_USE_ALPHA_WEIGHT = 1 << 2;
static const unsigned int ASTCENC_FLG_USE_PERCEPTUAL = 1 << 3;
static const unsigned int ASTCENC_FLG_DECOMPRESS_ONLY = 1 << 4;
static const unsigned int ASTCENC_FLG_SELF_DECOMPRESS_ONLY = 1 << 5;
static const unsigned int ASTCENC_FLG_MAP_RGBM = 1 << 6;
static const unsigned int ASTCENC_ALL_FLAGS = (1 << 0) | (1 << 1) | (1 << 2) | (1 << 3) | (1 << 4) | (1 << 5) | (1 << 6);

struct astcenc_config {
	enum astcenc_profile profile;
	unsigned int flags;
	unsigned int block_x;
	unsigned int block_y;
	unsigned int block_z;
	float cw_r_weight;
	float cw_g_weight;
	float cw_b_weight;
	float cw_a_weight;
	unsigned int a_scale_radius;
	float rgbm_m_scale;
	unsigned int tune_partition_count_limit;
	unsigned int tune_2partition_index_limit;
	unsigned int tune_3partition_index_limit;
	unsigned int tune_4partition_index_limit;
	unsigned int tune_block_mode_limit;
	unsigned int tune_refinement_limit;
	unsigned int tune_candidate_limit;
	unsigned int tune_2partitioning_candidate_limit;
	unsigned int tune_3partitioning_candidate_limit;
	unsigned int tune_4partitioning_candidate_limit;
	float tune_db_limit;
	float tune_mse_overshoot;
	float tune_2partition_early_out_limit_factor;
	float tune_3partition_early_out_limit_factor;
	float tune_2plane_early_out_limit_correlation;
	float tune_search_mode0_enable;
	astcenc_progress_callback progress_callback;
};

/* data[z] points at slice z: dim_x * dim_y RGBA texels of data_type, row-major, tightly packed */
struct astcenc_image {
	unsigned int dim_x;
	unsigned int dim_y;
	unsigned int dim_z;
	enum astcenc_type data_type;
	void** data;
};

struct astcenc_block_info {
	enum astcenc_profile profile;
	unsigned int block_x;
	unsigned int block_y;
	unsigned int block_z;
	unsigned int texel_count;
	bool is_error_block;
	bool is_constant_block;
	bool is_hdr_block;
	bool is_dual_plane_block;
	unsigned int partition_count;
	unsigned int partition_index;
	unsigned int dual_plane_component;
	unsigned int color_endpoint_modes[4];
	unsigned int color_level_count;
	unsigned int weight_level_count;
	unsigned int weight_x;
	unsigned int weight_y;
	unsigned int weight_z;
	float color_endpoints[4][2][4];
	float weight_values_plane1[216];
	float weight_values_plane2[216];
	uint8_t partition_assignment[216];
};

ASTCENC_PUBLIC enum astcenc_error astcenc_config_init(enum astcenc_profile profile, unsigned int block_x, unsigned int block_y, unsigned int block_z,
                                                      float quality, unsigned int flags, struct astcenc_config* config);

ASTCENC_PUBLIC enum astcenc_error astcenc_context_alloc(const struct astcenc_config* config, unsigned int thread_count,
                                                        struct astcenc_context** context, const struct astcenc_context* parent_context);

ASTCENC_PUBLIC enum astcenc_error astcenc_compress_image(struct astcenc_context* context, struct astcenc_image* image, const struct astcenc_swizzle* swizzle,
                                                         uint8_t* data_out, size_t data_len, unsigned int thread_index);

ASTCENC_PUBLIC enum astcenc_error astcenc_compress_reset(struct astcenc_context* context);

ASTCENC_PUBLIC enum astcenc_error astcenc_compress_cancel(struct astcenc_context* context);

ASTCENC_PUBLIC enum astcenc_error astcenc_decompress_image(struct astcenc_context* context, const uint8_t* data, size_t data_len,
                                                           struct astcenc_image* image_out, const struct astcenc_swizzle* swizzle, unsigned int thread_index);

ASTCENC_PUBLIC enum astcenc_error astcenc_decompress_reset(struct astcenc_context* context);

ASTCENC_PUBLIC void astcenc_context_free(struct astcenc_context* context);

ASTCENC_PUBLIC enum astcenc_error astcenc_get_block_info(struct astcenc_context* context, const uint8_t data[16], struct astcenc_block_info* info);

ASTCENC_PUBLIC const char* astcenc_get_error_string(enum astcenc_error status);

/* ---- astcenc_b200_* extensions --------------------------------------------------------------------- */

/* Behaviour notes for the ten reference entry points above, where the GPU implementation differs in timing (never in
 * results) from the reference's thread pool:
 *  - progress_callback is called as blocks complete, like the reference's task pool (astcenc_internal_entry.h:199-295): with
 *    done / total * 100 over the blocks of the whole image (all slices of a volume), whenever the value has moved by more
 *    than max(1 %, 4096 blocks) since the last call, and exactly once with 100 after the payload is in data_out. Only the
 *    calling thread that runs the pass calls it; the library polls a device counter about every millisecond.
 *  - astcenc_compress_cancel() stops a running pass at once: the kernels stop taking blocks (the flag is written into device
 *    memory while they run), remaining slices are skipped, and the call returns ASTCENC_SUCCESS without writing data_out and
 *    without the 100 % call. It takes no lock a pass holds, so it may be called from the progress callback. The
 *    astcenc_b200_* device-resident and multi-GPU entry points have neither progress nor cancellation.
 *  - Every entry point runs on the CUDA device that was current in astcenc_context_alloc() and restores the caller's
 *    current device before it returns.
 *  - Block sizes: the fourteen 2D and the ten 3D footprints (block_z > 1: 3x3x3 .. 6x6x6, astcenc_block_sizes.cpp:1025). With a
 *    3D block size the slices of astcenc_image::data are uploaded into one volume and compressed in one pass, blocks in
 *    (z, y, x) order like the reference's (astcenc_entry.cpp:1036); a_scale_radius is ignored like the reference does
 *    (astcenc_entry.cpp:975). The multi-GPU entry points (slab and batch mode) take the same images: 2D, texture arrays and
 *    volumes. The device-resident entry astcenc_b200_compress_device and astcenc_b200_slab_rows stay 2D (3D block sizes:
 *    ASTCENC_ERR_NOT_IMPLEMENTED); the device-resident block-list entry astcenc_b200_compress_device_blocks takes volumes.
 *  - a_scale_radius with a 2D block size and dim_z > 1 gives ASTCENC_ERR_NOT_IMPLEMENTED from every compressing entry point.
 *    The alpha-scale pre-pass of a pass over some block rows filters only the 32 x 32 tiles that cover those rows, and reads
 *    the image rows of those tiles plus a_scale_radius rows on either side; nothing else of the image is read.
 *  - A context owns ONE set of search scratch buffers: passes of the same context are serialised - on the host by a mutex,
 *    on the device by an event chain - whatever streams they are enqueued on. Use one context per concurrent stream.
 */

/* Compress block rows [block_row0, block_row0 + block_rows) of an image that is ALREADY RESIDENT in device
 * memory (d_pixels: the whole dim_x * dim_y image), writing block_rows * blocks_x * 16 bytes to the device
 * buffer d_out. Enqueued on `cuda_stream` (a cudaStream_t passed as void*, 0 = the context's own stream);
 * returns without synchronising. Used for slab sharding across GPUs and by bench.py's device-resident timing.
 * Calls on different streams of the same context are ordered one after the other (see above). */
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_compress_device(struct astcenc_context* context, const void* d_pixels, enum astcenc_type data_type,
                                                               unsigned int dim_x, unsigned int dim_y, const struct astcenc_swizzle* swizzle,
                                                               unsigned int block_row0, unsigned int block_rows, uint8_t* d_out, void* cuda_stream);

/* Recompress a list of blocks of an image that is ALREADY RESIDENT in device memory, in place in its device-resident payload:
 * for a texture whose source changes a few tiles at a time (painting tools, procedural or virtual-texture pages, atlases).
 *  - d_pixels: the whole image, dim_z slices of dim_x * dim_y texels, contiguous. Image shapes are those astcenc_compress_image
 *    takes: 2D images, texture arrays (2D block size, dim_z > 1) and volumes of 3D block sizes.
 *  - d_payload: the whole image's payload in astcenc_compress_image's order (blocks in z, y, x order; for 2D block sizes z
 *    counts slices). block_indices (a HOST array, which the caller may free as soon as the call returns) are positions in that
 *    order. Exactly the 16 bytes of each listed block are written - the bytes astcenc_compress_image produces for that block -
 *    and every other byte of d_payload is left untouched. Duplicate indices write the same bytes; block_count == 0 does nothing.
 *  - Errors, in this order: ASTCENC_ERR_BAD_CONTEXT for a decompress-only context, ASTCENC_ERR_BAD_SWIZZLE, ASTCENC_ERR_BAD_PARAM
 *    for NULL or zero-sized arguments, ASTCENC_ERR_NOT_IMPLEMENTED for a_scale_radius on a texture array (with a 3D block size
 *    the radius is ignored), ASTCENC_ERR_BAD_PARAM for an index at or beyond the image's block count. On error nothing is
 *    launched and nothing is written.
 *  - Enqueued on `cuda_stream` (0 = the context's own stream), without synchronising, in order with every other pass of the
 *    context (see above). No progress callback, no cancellation.
 * The listed blocks are gathered into a staging row of blocks, compressed by one ordinary pass of the wave pipeline (one per
 * ASTCENC_B200_BATCH_BLOCKS blocks of a longer list) and scattered to their positions; the block count of the list, not the
 * image's, sets the cost. */
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_compress_device_blocks(struct astcenc_context* context, const void* d_pixels, enum astcenc_type data_type,
                                                                      unsigned int dim_x, unsigned int dim_y, unsigned int dim_z, const struct astcenc_swizzle* swizzle,
                                                                      const uint32_t* block_indices, unsigned int block_count, uint8_t* d_payload, void* cuda_stream);

/* Compress many images - the levels of a mip chain, a set of small textures - in shared pipeline passes: for callers whose
 * images are small, each of which would otherwise pay the fixed cost of a pass of its own (a few milliseconds, whatever the
 * image's size).
 *  - astcenc_b200_compress_device_images: images[i] describes an image ALREADY RESIDENT in device memory (data: dim_z slices
 *    of dim_x * dim_y texels, contiguous) and its device payload. Every block of every image is written to that image's
 *    payload, in astcenc_compress_image's order, and the bytes are those astcenc_compress_image writes for the image alone.
 *    Images may differ in size and take the shapes astcenc_compress_image takes: 2D images, texture arrays (2D block size,
 *    dim_z > 1) and volumes of 3D block sizes. All share data_type and swizzle. Payloads must not overlap (not checked). The
 *    descriptor array is copied: the caller may free it when the call returns. Enqueued on `cuda_stream` (0 = the context's
 *    own stream), without synchronising, in order with every other pass of the context (see above). No progress callback, no
 *    cancellation.
 *  - astcenc_b200_compress_images: the host-pointer twin. Every image goes up into one device buffer, the device path runs on
 *    the context's stream, payload i is copied into data_out[i] (data_len[i] bytes, which must hold it), and the call returns
 *    when that is done. All images must have the same data_type. astcenc_b200_last_timing() reports its device time and its
 *    H2D / D2H bytes. It uses the context's host-path buffers: one host-pointer call at a time per context.
 *  - Errors, in this order; on error nothing is launched and nothing is written: ASTCENC_ERR_BAD_CONTEXT for a decompress-only
 *    context; ASTCENC_ERR_BAD_PARAM for a NULL swizzle, then ASTCENC_ERR_BAD_SWIZZLE; ASTCENC_ERR_BAD_PARAM for images == NULL
 *    with a non-zero count, a NULL data, payload or output pointer, a zero dimension, a bad data type or (host entry) mixed
 *    data types; ASTCENC_ERR_NOT_IMPLEMENTED for a_scale_radius on a texture array; ASTCENC_ERR_BAD_PARAM when the block count
 *    of an image (2^32 blocks or more) or of the whole call overflows; (host entry) ASTCENC_ERR_OUT_OF_MEM when a data_len[i]
 *    is too short. All images are checked before anything is enqueued. image_count == 0 does nothing.
 * The images' blocks are gathered, in call order, into staging rows of at most ASTCENC_B200_BATCH_BLOCKS blocks, as block lists
 * are: one ordinary pass per staging row, which may span several images, then a scatter to each image's payload. With
 * a_scale_radius (2D block sizes) each image gets its own alpha-scale pre-pass over the whole image: one extra launch per image. */
struct astcenc_b200_device_image {
	const void* data;              /* device: dim_z slices of dim_x * dim_y texels, contiguous */
	unsigned int dim_x, dim_y, dim_z;
	uint8_t* payload;              /* device: the image's whole payload, astcenc_compress_image's block order */
};
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_compress_device_images(struct astcenc_context* context, const struct astcenc_b200_device_image* images,
                                                                      unsigned int image_count, enum astcenc_type data_type, const struct astcenc_swizzle* swizzle,
                                                                      void* cuda_stream);
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_compress_images(struct astcenc_context* context, struct astcenc_image* const* images, unsigned int image_count,
                                                               const struct astcenc_swizzle* swizzle, uint8_t* const* data_out, const size_t* data_len);

/**
 * Device-resident decompression of many images in one launch, such as the levels of a mip chain or a set of textures.
 * images[i] describes a payload ALREADY RESIDENT in device memory (astcenc_compress_image's block order, 16 bytes per block) and
 * the device image it decodes into (dim_z slices of dim_x * dim_y texels of data_type, contiguous). Image i's data receives
 * exactly the texels astcenc_decompress_image writes for payload i alone, with the same data_type and swizzle: Z
 * reconstruction, the error colour of illegal blocks and the F16 void-extent behaviour included. Images may differ in size and
 * take the shapes astcenc_decompress_image takes: 2D images, texture arrays (2D block size, dim_z > 1) and volumes of 3D block
 * sizes. Outputs must not overlap each other or any payload (not checked); they need no alignment. The descriptor array is
 * copied: the caller may free it when the call returns. Enqueued on `cuda_stream` (0 = the context's own stream), without
 * synchronising, in order with every other pass of the context. Works on decompress-only contexts. No progress callback, no
 * cancellation. A single image is a call with image_count == 1.
 * Errors, in this order; on error nothing is launched and nothing is written: ASTCENC_ERR_BAD_PARAM for a NULL swizzle, then
 * ASTCENC_ERR_BAD_SWIZZLE (r, g, b, a, 0, 1 and Z are allowed); ASTCENC_ERR_BAD_PARAM for images == NULL with a non-zero count, a
 * NULL payload or data pointer, a zero dimension or a bad data type; ASTCENC_ERR_BAD_PARAM when the block count of an image
 * (2^32 blocks or more) or of the whole call overflows. All images are checked before anything is enqueued. image_count == 0
 * does nothing. The call's table goes up in one small copy and every block of the call is decoded by one kernel launch.
 */
struct astcenc_b200_device_decode_image {
	const uint8_t* payload;        /* device: the image's whole payload, astcenc_compress_image's block order */
	void* data;                    /* device: dim_z slices of dim_x * dim_y texels of data_type, contiguous */
	unsigned int dim_x, dim_y, dim_z;
};
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_decompress_device_images(struct astcenc_context* context, const struct astcenc_b200_device_decode_image* images,
                                                                        unsigned int image_count, enum astcenc_type data_type,
                                                                        const struct astcenc_swizzle* swizzle, void* cuda_stream);

/**
 * Multi-GPU sharding: one process per GPU, each with its own context; the only exchange is the gather of the compressed
 * payload over NCCL (loaded at run time: "libnccl.so.2"; ASTCENC_ERR_NOT_IMPLEMENTED when it cannot be loaded).
 * The reference has no counterpart - its unit of distribution is the block ticket of one process
 * (astcenc_internal_entry.h:97-324); the payload layout the ranks agree on is astcenc_entry.cpp:1036.
 *
 * astcenc_b200_comm_unique_id   rank 0 makes the 128-byte rendezvous id; the caller ships it to the other ranks
 * astcenc_b200_comm_init        collective: joins `world` ranks (world == 1: no communicator, the calls below run locally)
 * astcenc_b200_slab_rows        the block rows [first, first + rows) rank `rank` of `world` owns for a 2D image of height dim_y
 * astcenc_b200_compress_image_sharded
 *     collective, SLAB MODE: every rank passes the same image (host pointers) and compresses its slab of the COMBINED block
 *     rows: layer * blocks_y + row for 3D block sizes, slice * blocks_y + row for a texture array (2D block size, dim_z > 1),
 *     the rows of a 2D image. A rank reads and uploads only what its slab needs: the image rows of its block rows (with
 *     a_scale_radius, the pre-pass window around them), or the slices of its layers. The slabs are gathered into the root's
 *     device buffer (grouped ncclSend/ncclRecv) and copied to data_out on the root (data_out is ignored elsewhere); bytes are
 *     identical to astcenc_compress_image(). astcenc_b200_last_timing() reports the bytes this rank uploaded.
 * astcenc_b200_compress_batch
 *     collective, BATCH MODE: image i of `images` belongs to rank i % world (other entries are not touched on this rank and
 *     may be NULL); all images share dim_x, dim_y, dim_z and type (ASTCENC_ERR_BAD_PARAM otherwise) and data_len_each must
 *     hold one image's payload. Each rank searches its images one after the other with the upload of the next image
 *     overlapped (two device image buffers), a volume in one pass, a texture array slice by slice; payload i arrives in
 *     data_out[i] on the root.
 * astcenc_b200_comm_last_timing device milliseconds of the last sharded call on this rank: search, and the gather alone
 */
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_comm_unique_id(void* id_out, size_t id_bytes);
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_comm_init(struct astcenc_context* context, int rank, int world, const void* id, size_t id_bytes);
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_comm_free(struct astcenc_context* context);
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_slab_rows(struct astcenc_context* context, unsigned int dim_y, int rank, int world,
                                                         unsigned int* first_block_row, unsigned int* block_rows);
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_compress_image_sharded(struct astcenc_context* context, struct astcenc_image* image,
                                                                      const struct astcenc_swizzle* swizzle, uint8_t* data_out, size_t data_len, int root);
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_compress_batch(struct astcenc_context* context, struct astcenc_image* const* images, unsigned int image_count,
                                                              const struct astcenc_swizzle* swizzle, uint8_t* const* data_out, size_t data_len_each, int root);
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_comm_last_timing(struct astcenc_context* context, float* compress_ms, float* gather_ms);

/* Number of kernel launches issued by this context so far (bench.py reports it as gpu_launches). */
ASTCENC_PUBLIC unsigned long long astcenc_b200_launch_count(struct astcenc_context* context);

/**
 * Per-stage timing of the wave pipeline (measurement aid). enable != 0 makes the following
 * astcenc_b200_compress_device() calls record a CUDA event after every kernel launch; a later call with non-NULL
 * arrays returns, for the last such call, the summed launch durations and launch counts per kernel
 * (0 setup, 1 refine, 2 prepare, 3 emit). Leave it off for production use.
 */
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_stage_timing(struct astcenc_context* context, int enable, float stage_ms[4], unsigned int stage_launches[4]);

/* Milliseconds of device time (CUDA events on the launching stream) spent in the compress kernel by the most
 * recent astcenc_compress_image() or astcenc_b200_compress_images() call on this context, and its H2D / D2H byte counts. */
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_last_timing(struct astcenc_context* context, float* kernel_ms, size_t* h2d_bytes, size_t* d2h_bytes);

/**
 * Image error metrics on the device: what the reference's command line tool computes on the host after a -t* round trip
 * (Source/astcenccli_error_metrics.cpp:109-413, compute_error_metrics(); it prints, this returns). img1 is the
 * original, img2 the decoded image (host pointers, any mix of U8 / F16 / F32; only the intersection is compared).
 * input_components (1-4) selects the channels that count, as in the reference (1: RGB, 2: BA, 3: RGB, 4: RGBA).
 * Fields not requested (HDR / normal-map metrics) are zero. PSNR values are 999.0 for identical images.
 */
struct astcenc_b200_error_metrics {
	double psnr;                  /* "PSNR (LDR-RGBA)" when alpha counts, else "PSNR (LDR-RGB)" */
	double alpha_psnr;            /* "Alpha-weighted PSNR" (= psnr when alpha does not count) */
	double rgb_psnr;              /* "PSNR (LDR-RGB)" */
	double rgb_peak;              /* largest R/G/B value of img1 */
	double peak_psnr;             /* HDR: "PSNR (RGB norm to peak)" */
	double mpsnr;                 /* HDR: "mPSNR (RGB)" over fstop_lo..fstop_hi */
	double log_rmse;              /* HDR: "LogRMSE (RGB)" */
	double mean_angular_error;    /* normal maps: degrees */
	double worst_angular_error;   /* normal maps: degrees */
	double sum_squared_error[4];  /* per channel, values scaled to 0..1 (LDR) */
};
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_compute_error_metrics(struct astcenc_context* context, int compute_hdr_metrics, int compute_normal_metrics,
                                                                     int input_components, const struct astcenc_image* img1, const struct astcenc_image* img2,
                                                                     int fstop_lo, int fstop_hi, struct astcenc_b200_error_metrics* metrics);

/**
 * Error metrics of many device-resident image pairs in one call, such as the levels of a mip chain or a texture set against
 * their decodes (astcenc_b200_decompress_device_images), with an optional per-block error map.
 * What each entry gets: *metrics receives the figures astcenc_b200_compute_error_metrics returns for that pair alone, on host
 * copies of the same images. sum_squared_error, rgb_peak, mean_angular_error, worst_angular_error and log_rmse are bit for bit
 * the same. The dB figures (psnr, alpha_psnr, rgb_psnr, peak_psnr, mpsnr) are computed on the device, whose log10 may differ
 * from the host's in the last bits: they agree within 1e-12 dB. Fields not requested are zero.
 * The per-block error map: block_error, when not NULL, receives one float per block of the context's footprint
 * (block_x / block_y / block_z) in astcenc_compress_image's block order, the index astcenc_b200_compress_device_blocks takes (a 2D
 * footprint's z counts the slices of a texture array). Each value is the sum, over the block's texels inside the image, of the
 * squared differences of the channels input_components selects, in the units of sum_squared_error (U8 scaled to 0..1, F16 / F32
 * clamped to [0, 65504]); it is accumulated in double in a fixed order and rounded to float once, and depends only on that
 * block's texels.
 * The figures are deterministic and do not depend on which other entries share the call or on their order. The call is
 * enqueued on `cuda_stream` (0 = the context's own stream) without synchronising, in order with every other pass of the
 * context. Works on decompress-only contexts. No progress callback, no cancellation. image_count == 0 does nothing. The
 * descriptor array is copied: the caller may free it when the call returns. Outputs must not overlap any input (not checked).
 * Errors, in this order; on error nothing is launched and nothing is written: ASTCENC_ERR_BAD_PARAM for a NULL context or
 * input_components outside 1-4, then for fstop_lo < -125 or fstop_hi > 125, then for images == NULL with a non-zero count, then
 * for an entry with a NULL original, decoded or metrics, a zero or overflowing dimension, a bad data type, or a pointer not
 * aligned to its element (4 / 8 / 16 bytes for a U8 / F16 / F32 texel, 8 for metrics, 4 for block_error; decode outputs of
 * one type packed tightly into a cudaMalloc buffer always are), then when the call does not fit a launch (an image with 2^32
 * blocks or more that asks for a map, or a grid beyond 2^31 - 1 CTAs). All entries are checked before anything is enqueued.
 * The table goes up in one small copy; the call is two kernel launches, three when any entry asks for a map.
 */
struct astcenc_b200_device_metrics_image {
	const void* original;                         /* device: dim_z slices of dim_x * dim_y texels of original_type, contiguous */
	const void* decoded;                          /* device: the same shape, texels of decoded_type */
	enum astcenc_type original_type, decoded_type;
	unsigned int dim_x, dim_y, dim_z;
	struct astcenc_b200_error_metrics* metrics;   /* device: receives this image's figures */
	float* block_error;                           /* device, or NULL: one float per block of the context's footprint */
};
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_compute_error_metrics_device_images(struct astcenc_context* context, int compute_hdr_metrics,
                                                                                  int compute_normal_metrics, int input_components,
                                                                                  const struct astcenc_b200_device_metrics_image* images,
                                                                                  unsigned int image_count, int fstop_lo, int fstop_hi, void* cuda_stream);

/**
 * What a per-block error map measures (astcenc_b200_compute_block_metric_device_images and
 * astcenc_b200_compute_block_metric_device_block_lists). Every map value is a sum over the block's texels inside the image, with
 * o the original texel and d the decoded one in the units of sum_squared_error (U8 scaled to 0..1, F16 / F32 clamped to
 * [0, 65504]) and m the channels input_components selects. Each term is computed in float, added in double in a fixed order, and
 * the block's sum is rounded to float once; a value depends only on that block's texels.
 * ASTCENC_B200_BLOCK_SQUARED_ERROR: (o_c - d_c)^2 for c in m; the map of astcenc_b200_compute_error_metrics_device_images. Summed
 *   over the image, the masked sum of sum_squared_error.
 * ASTCENC_B200_BLOCK_ALPHA_WEIGHTED_ERROR: ((o_c - d_c) * o_A)^2 for c in m among R, G, B, plus (o_A - d_A)^2 when A is in m. The
 *   block's share of the error sum behind alpha_psnr: RGB error under transparent texels does not count. Summed over the image
 *   with input_components == 4, samples / 10^(alpha_psnr / 10).
 * ASTCENC_B200_BLOCK_LOG2_ERROR: (L(o_c) - L(d_c))^2 for c in m among R, G, B, L the polynomial log2 the HDR figures use. The
 *   block's share of the error sum behind log_rmse, measured whether or not HDR figures are asked for: errors in dark and mid
 *   tones weigh as much as errors in the brightest blocks. Summed over the image and divided by the pixel count, log_rmse^2.
 * The image sums agree with the figures up to the per-block float rounding.
 * The normal-map metrics measure the angle theta(o, d) in degrees of each texel, the per-texel term of mean_angular_error and
 * worst_angular_error: each texel's RGB becomes a normal (c - 0.5) * 2, normalised (a zero-length vector becomes the unit
 * vector (1, 1, 1) / sqrt(3)); the dot product of the two normals is taken in float in DPPS order ((x1 x2 + y1 y2) + (z1 z2 + 0))
 * and clamped to [-1, 1] with fminf(fmaxf(dot, -1), 1), so a NaN dot gives -1, 180 degrees; theta is acos of it in double
 * times (double)(180.0f / pi). Both read R, G and B whatever input_components selects (input_components is still checked to be
 * 1-4), and neither depends on compute_normal_metrics or compute_hdr_metrics.
 * ASTCENC_B200_BLOCK_ANGULAR_ERROR: the sum of theta over the block's texels inside the image, added in double and rounded to
 *   float once. Summed over the image and divided by the pixel count, mean_angular_error.
 * ASTCENC_B200_BLOCK_WORST_ANGULAR_ERROR: the largest theta over the same texels, combined with fmax in double (the order does
 *   not matter) and rounded to float once. The largest value of the map is exactly (float)worst_angular_error, as rounding to
 *   float is monotone. Its total over the image is a sum of maxima, not a figure.
 * Valid values are 0, 1, 2, 4 and 5. Any other value, 3 included, is ASTCENC_ERR_BAD_PARAM wherever a call takes a block_metric.
 */
enum astcenc_b200_block_metric {
	ASTCENC_B200_BLOCK_SQUARED_ERROR = 0,
	ASTCENC_B200_BLOCK_ALPHA_WEIGHTED_ERROR = 1,
	ASTCENC_B200_BLOCK_LOG2_ERROR = 2,
	/* 3 is not assigned */
	ASTCENC_B200_BLOCK_ANGULAR_ERROR = 4,        /* sum over the block's texels of the angle, in degrees */
	ASTCENC_B200_BLOCK_WORST_ANGULAR_ERROR = 5   /* the largest angle over the block's texels, in degrees */
};

/**
 * astcenc_b200_compute_error_metrics_device_images with a chosen per-block error map: every block_error map receives
 * block_metric (enum astcenc_b200_block_metric) instead of the squared error. Everything else is that call's: the figures (bit for
 * bit the same), the stream, the descriptor table, decompress-only contexts, the launch count (two kernel launches, three when any
 * entry asks for a map) and the error order, into which one check is inserted: ASTCENC_ERR_BAD_PARAM for block_metric not one of 0, 1, 2, 4, 5
 * comes right after the check of input_components. With ASTCENC_B200_BLOCK_SQUARED_ERROR the call is
 * astcenc_b200_compute_error_metrics_device_images.
 */
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_compute_block_metric_device_images(struct astcenc_context* context, int compute_hdr_metrics,
                                                                                 int compute_normal_metrics, int input_components,
                                                                                 enum astcenc_b200_block_metric block_metric,
                                                                                 const struct astcenc_b200_device_metrics_image* images,
                                                                                 unsigned int image_count, int fstop_lo, int fstop_hi, void* cuda_stream);

/**
 * Block selection on the device: turn per-block error maps (astcenc_b200_compute_error_metrics_device_images) into device block
 * lists (astcenc_b200_compress_device_block_lists) without a trip through host memory.
 * One rule per entry: a block is a candidate when map[b] > threshold (NaN never is; -0.0 counts as 0.0). Of c candidates the
 * k = min(capacity, c) largest values are kept, ties going to the lower block index; their indices are written to indices[0, k)
 * in ascending order, *count receives k, and indices past k are left untouched. A threshold of -INFINITY with capacity k gives
 * the k worst blocks; a finite threshold with a large capacity gives every block worse than the threshold. In numpy terms, with
 * m[~(m > threshold)] = -inf: np.sort(np.argsort(-m, kind="stable")[:k]).
 * Each entry's output depends only on that entry, never on the other entries of the call or on the GPU. The call is a radix
 * select over the values' 32-bit keys and an ordered compaction: one memset and 7 kernel launches, whatever the number of
 * entries, reading each map six times. It uses the context's scratch and works on any context, decompress-only ones included.
 * Enqueued on `cuda_stream` (0 = the context's own stream) without synchronising, in order with every other pass of the
 * context. The descriptor array is copied: the caller may free it when the call returns. Outputs must not overlap any map or
 * each other (not checked). entry_count == 0 does nothing.
 * Errors, in this order; on error nothing is launched and nothing is written: ASTCENC_ERR_BAD_PARAM for a NULL context or
 * entries == NULL with a non-zero count, then for an entry with a NULL count, a NULL map with block_count > 0, NULL indices
 * with capacity > 0, a pointer not aligned to 4 bytes or a NaN threshold. All entries are checked before anything is enqueued.
 */
struct astcenc_b200_block_selection {
	const float* map;              /* device: block_count values, e.g. a per-block error map */
	unsigned int block_count;
	float threshold;               /* candidates are the values above it; -INFINITY: every value but NaN and -INFINITY */
	unsigned int capacity;         /* at most this many blocks are kept */
	uint32_t* indices;             /* device: receives the kept block indices, ascending (room for capacity) */
	uint32_t* count;               /* device: receives how many were kept */
};
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_select_blocks(struct astcenc_context* context, const struct astcenc_b200_block_selection* entries,
                                                             unsigned int entry_count, void* cuda_stream);

/**
 * Block selection over a set of maps under one shared budget, such as the worst blocks of a texture set or of a mip chain:
 * "the K worst blocks of the whole set", in a unit chosen per image by a device-resident weight.
 * The pools split the entry array into consecutive runs, in order: pools[0] owns the first pools[0].entry_count entries, and so
 * on. The rule for each pool:
 * - Product. Block b of entry j has the product p = map[b] * *weight, one float multiply. Without a weight, p = map[b].
 * - Candidates. A block is a candidate when p > threshold. NaN is never a candidate, and -0.0 counts as 0.0, as in
 *   astcenc_b200_select_blocks.
 * - Which blocks are kept. Of the pool's c candidates, the k = min(capacity, c) largest products are kept. Ties go to the lower
 *   entry position in the pool, then to the lower block index.
 * - Output. Each entry gets its own kept indices in ascending order and its own *count, which is 0 when none of its blocks are
 *   kept. Indices past the count are left untouched.
 * - In numpy terms: concatenate the entries' products in order, set non-candidates to -inf, run
 *   np.argsort(-pp, kind="stable")[:k], split the result by entry, and sort each part.
 * - Independence. A pool's outputs depend only on that pool, never on the other pools in the call, their order, or the GPU.
 * astcenc_b200_select_blocks is this call with one pool per entry and no weights, and writes the same bytes.
 * The weight is read on the device when the call runs, so a weight derived from device figures (for example
 * 1 / sum_squared_error from an astcenc_b200_error_metrics record) needs no host round trip. As first-order statements, not
 * promises, with each map an image's per-block error (astcenc_b200_compute_block_metric_device_images) and a -INFINITY
 * threshold, a block ranks by its share of:
 * - NULL weights: the pool's total map sum;
 * - 1 / texels_j (texels of image j): the mean over the images of the per-texel error;
 * - 1 / E_j, E_j being image j's map total: the mean PSNR over the images (a block of error e holds image j's PSNR down by
 *   about (10 / ln 10) * e / E_j dB).
 * Stream, scratch and tables are those of astcenc_b200_select_blocks: enqueued on `cuda_stream` (0 = the context's own stream)
 * without synchronising, on any context, decompress-only ones included. The descriptor arrays are copied. The call costs one
 * memset and 7 kernel launches, whatever the number of pools and entries, reading each map six times; entry_count == 0 launches
 * nothing. Outputs must not overlap any map, weight or each other (not checked).
 * Errors, in this order; on error nothing is launched and nothing is written:
 *   1. ASTCENC_ERR_BAD_PARAM for a NULL context, pools == NULL with pool_count > 0, or entries == NULL with entry_count > 0;
 *   2. ASTCENC_ERR_BAD_PARAM for a pool with a NaN threshold, or when the pools' entry_counts, summed without overflow, differ
 *      from entry_count;
 *   3. ASTCENC_ERR_BAD_PARAM for an entry with a NULL count, a NULL map with block_count > 0, NULL indices when its pool's
 *      capacity is > 0, or a map, weight, indices or count not aligned to 4 bytes.
 * All entries are checked before anything is enqueued.
 */
struct astcenc_b200_block_pool {
	unsigned int entry_count;      /* the next entry_count entries of the call share this pool */
	float threshold;               /* candidates are the products above it */
	unsigned int capacity;         /* at most this many blocks are kept, over all the pool's entries */
};
struct astcenc_b200_pooled_selection {
	const float* map;              /* device: block_count values, e.g. a per-block error map */
	unsigned int block_count;
	const float* weight;           /* device: one float, read when the call runs; NULL = no weight */
	uint32_t* indices;             /* device: room for min(pool capacity, block_count) indices */
	uint32_t* count;               /* device: receives how many of this entry's blocks were kept */
};
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_select_blocks_pooled(struct astcenc_context* context, const struct astcenc_b200_block_pool* pools,
                                                                    unsigned int pool_count, const struct astcenc_b200_pooled_selection* entries,
                                                                    unsigned int entry_count, void* cuda_stream);

/**
 * Recompress block lists that live in device memory, such as the output of astcenc_b200_select_blocks or a GPU tool's list of
 * dirty tiles, for many device-resident images in shared pipeline passes.
 * lists[i] describes an image ALREADY RESIDENT in device memory (data: dim_z slices of dim_x * dim_y texels, contiguous; the
 * shapes astcenc_compress_image takes), its device payload, a device index list and a device count. The call reads the first
 * min(*count, capacity) indices; an index at or beyond the image's block count is skipped. Each listed block's 16 bytes are
 * written, the bytes astcenc_compress_image writes for that block; every other byte of the payload is left untouched, and
 * duplicate indices write the same bytes. A one-entry call is the single-image case. All entries share data_type and swizzle;
 * payloads must not overlap (not checked). The descriptor array is copied. Enqueued on `cuda_stream` (0 = the context's own
 * stream), without synchronising, in order with every other pass of the context: *count and the indices are read on the device
 * when the call runs. No progress callback, no cancellation.
 * Cost: the host does not know the counts, so a call costs what astcenc_b200_compress_device_images costs over the sum of
 * the capacities, not over the counts: each entry owns `capacity` staging blocks, and a slot past the count (or with an index
 * out of range) is staged as an all-zero block, which the pipeline finishes as a constant block in its first wave and which is
 * never written back. With a_scale_radius (2D block sizes) each entry gets an alpha-scale pre-pass over its whole image, one
 * extra launch per entry. Entries with capacity == 0 do nothing; a call whose capacities are all zero launches nothing.
 * Errors, in this order; on error nothing is launched and nothing is written: ASTCENC_ERR_BAD_CONTEXT for a decompress-only
 * context; ASTCENC_ERR_BAD_PARAM for a NULL swizzle, then ASTCENC_ERR_BAD_SWIZZLE; ASTCENC_ERR_BAD_PARAM for lists == NULL with
 * a non-zero count, or an entry with a NULL data or payload, a NULL indices or count with capacity > 0, indices or count not
 * aligned to 4 bytes, a zero dimension, or a bad data type; ASTCENC_ERR_NOT_IMPLEMENTED for a_scale_radius on a texture array;
 * ASTCENC_ERR_BAD_PARAM for an image of 2^32 blocks or more, or when the sum of the capacities overflows. All entries are checked
 * before anything is enqueued.
 */
struct astcenc_b200_device_block_list {
	const void* data;              /* device: dim_z slices of dim_x * dim_y texels, contiguous */
	unsigned int dim_x, dim_y, dim_z;
	uint8_t* payload;              /* device: the image's whole payload, astcenc_compress_image's block order */
	const uint32_t* indices;       /* device: block positions in that order */
	const uint32_t* count;         /* device: how many of the indices are listed */
	unsigned int capacity;         /* at most this many indices are read; the call's cost */
};
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_compress_device_block_lists(struct astcenc_context* context, const struct astcenc_b200_device_block_list* lists,
                                                                          unsigned int list_count, enum astcenc_type data_type,
                                                                          const struct astcenc_swizzle* swizzle, void* cuda_stream);

/**
 * Decode block lists that live in device memory into device images: bring a decoded copy up to date after
 * astcenc_b200_compress_device_block_lists (or compress_device_blocks) has re-encoded some of its blocks, without decoding the
 * whole payload again.
 * lists[i] describes a payload ALREADY RESIDENT in device memory (astcenc_compress_image's block order), the device image it
 * decodes into (dim_z slices of dim_x * dim_y texels of data_type, contiguous, starting at any byte), a device index list and a
 * device count. The list rule is that of astcenc_b200_compress_device_block_lists: the call reads the first min(*count, capacity)
 * indices, and an index at or beyond the image's block count is skipped. For each listed block, the texels of its footprint that
 * lie inside the image receive exactly the bytes astcenc_b200_decompress_device_images writes there for the whole payload (the
 * swizzle, Z reconstruction, the error colour and the F16 void-extent behaviour included); every other byte of data is left
 * untouched, and duplicate indices write the same texels. Takes 2D images, texture arrays (2D block sizes; z counts the slices)
 * and volumes of 3D block sizes; works on decompress-only contexts. Outputs must not overlap each other or any payload (not
 * checked). The descriptor array is copied. Enqueued on `cuda_stream` (0 = the context's own stream) without synchronising, in
 * order with every other pass of the context: *count and the indices are read on the device when the call runs.
 * Cost: the host does not know the counts, so the call is one table copy and one kernel launch over the sum of the capacities;
 * a slot past the count does no work. Entries with capacity == 0 do nothing; a call whose capacities are all zero launches nothing.
 * Errors, in this order; on error nothing is launched and nothing is written: ASTCENC_ERR_BAD_PARAM for a NULL swizzle, then
 * ASTCENC_ERR_BAD_SWIZZLE; ASTCENC_ERR_BAD_PARAM for lists == NULL with a non-zero count, an entry with a NULL payload or data, a
 * NULL indices or count with capacity > 0, indices or count not aligned to 4 bytes, or a zero or overflowing dimension, then for a
 * bad data type, then for an image of 2^32 blocks or more, or when the sum of the capacities overflows. All entries are checked
 * before anything is enqueued.
 */
struct astcenc_b200_device_decode_block_list {
	const uint8_t* payload;        /* device: the image's whole payload, astcenc_compress_image's block order */
	void* data;                    /* device: dim_z slices of dim_x * dim_y texels of data_type, contiguous */
	unsigned int dim_x, dim_y, dim_z;
	const uint32_t* indices;       /* device: block positions in that order */
	const uint32_t* count;         /* device: how many of the indices are listed */
	unsigned int capacity;         /* at most this many indices are read; the call's cost */
};
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_decompress_device_block_lists(struct astcenc_context* context,
                                                                            const struct astcenc_b200_device_decode_block_list* lists,
                                                                            unsigned int list_count, enum astcenc_type data_type,
                                                                            const struct astcenc_swizzle* swizzle, void* cuda_stream);

/**
 * Refresh per-block error maps at the blocks of device block lists: after listed blocks have been re-encoded and re-decoded
 * (astcenc_b200_decompress_device_block_lists), bring the map of astcenc_b200_compute_error_metrics_device_images up to date
 * without measuring the whole image pair again.
 * lists[i] describes an image pair ALREADY RESIDENT in device memory (as astcenc_b200_device_metrics_image does), its whole map
 * (one float per block of the context's footprint, in astcenc_compress_image's block order), a device index list and a device
 * count, read by the list rule of astcenc_b200_decompress_device_block_lists. For each listed block, block_error[index] receives
 * bit for bit the value astcenc_b200_compute_error_metrics_device_images writes for that block of the same pair with the same
 * input_components; every other map value is left untouched. No PSNR figures are produced. Works on decompress-only contexts.
 * The descriptor array is copied. Enqueued on `cuda_stream` (0 = the context's own stream) without synchronising, in order with
 * every other pass of the context. Cost: one table copy and one kernel launch, one warp per slot over the sum of the capacities.
 * Entries with capacity == 0 do nothing; a call whose capacities are all zero launches nothing.
 * Errors, in this order; on error nothing is launched and nothing is written: ASTCENC_ERR_BAD_PARAM for a NULL context or
 * input_components outside 1-4, then for lists == NULL with a non-zero count, then for an entry with a NULL original or decoded, a
 * NULL block_error, indices or count with capacity > 0, a zero or overflowing dimension, a bad data type, or a pointer not aligned
 * to its element (4 / 8 / 16 bytes for a U8 / F16 / F32 texel, 4 for block_error, indices and count), then when the call does not
 * fit a launch (an image of 2^32 blocks or more, or a grid beyond 2^31 - 1 CTAs). All entries are checked before anything is
 * enqueued.
 */
struct astcenc_b200_device_block_error_list {
	const void* original;          /* device: dim_z slices of dim_x * dim_y texels of original_type, contiguous */
	const void* decoded;           /* device: the same shape, texels of decoded_type */
	enum astcenc_type original_type, decoded_type;
	unsigned int dim_x, dim_y, dim_z;
	float* block_error;            /* device: the image's whole map, one float per block of the context's footprint */
	const uint32_t* indices;       /* device: block positions in astcenc_compress_image's order */
	const uint32_t* count;         /* device: how many of the indices are listed */
	unsigned int capacity;         /* at most this many indices are read; the call's cost */
};
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_compute_block_errors_device_block_lists(struct astcenc_context* context, int input_components,
                                                                                      const struct astcenc_b200_device_block_error_list* lists,
                                                                                      unsigned int list_count, void* cuda_stream);

/**
 * astcenc_b200_compute_block_errors_device_block_lists for a map of block_metric (enum astcenc_b200_block_metric): each listed
 * value receives bit for bit what astcenc_b200_compute_block_metric_device_images writes for that block with the same
 * input_components and block_metric, and every other value is left untouched. Everything else is that call's: the list rule, the
 * stream, decompress-only contexts, one kernel launch (none when the capacities are all zero) and the error order, into which one
 * check is inserted: ASTCENC_ERR_BAD_PARAM for block_metric not one of 0, 1, 2, 4, 5 comes right after the check of input_components. With
 * ASTCENC_B200_BLOCK_SQUARED_ERROR the call is astcenc_b200_compute_block_errors_device_block_lists.
 */
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_compute_block_metric_device_block_lists(struct astcenc_context* context, int input_components,
                                                                                      enum astcenc_b200_block_metric block_metric,
                                                                                      const struct astcenc_b200_device_block_error_list* lists,
                                                                                      unsigned int list_count, void* cuda_stream);

/**
 * Re-encode device block lists and keep each new block only where it lowers the block's error: one round of a device refinement
 * loop (compress, decode, map, astcenc_b200_select_blocks, then this call, repeated) that never makes a block worse under the
 * caller's own metric. It replaces astcenc_b200_compress_device_block_lists followed by the list decode and the list map, and
 * needs no decode context of its own: each candidate is decoded by the context that encoded it.
 * lists[i] describes an image ALREADY RESIDENT in device memory (data: dim_z slices of dim_x * dim_y texels of data_type,
 * contiguous), its payload (astcenc_compress_image's block order), its decode (the same shape, texels of decoded_type) or NULL,
 * its per-block map of block_metric (one float per block of the context's footprint) and a device index list with a device count.
 * - List rule: that of astcenc_b200_compress_device_block_lists. The call reads the first min(*count, capacity) indices; an index
 *   at or beyond the image's block count is skipped.
 * - Candidate: for each listed block, the 16 bytes astcenc_b200_compress_device_block_lists would write with this context,
 *   data_type and swizzle.
 * - Candidate value v': bit for bit what astcenc_b200_compute_block_metric_device_images writes for that block with
 *   input_components and block_metric when it compares data against this context's decode of the candidate, the decode
 *   astcenc_b200_decompress_device_images on this context writes with decoded_type and decode_swizzle.
 * - Commit rule: the block is committed iff v' < block_error[index] as a float comparison, with the map as it stood before the
 *   call: ties keep the old block, and a NaN on either side never commits. A committed block gets its 16 payload bytes replaced,
 *   the texels of its footprint inside the image replaced in decoded (when decoded is not NULL), and block_error[index] = v'.
 *   Nothing else is written: payload bytes and texels of blocks that are not committed, invalid slots and unlisted blocks keep
 *   their values. A block listed more than once ends as if listed once (its candidates are the same bytes with the same value).
 * - Consistency: if payload, decoded and block_error agree on entry (decoded is what this context decodes from payload, and
 *   block_error is the whole map of data against decoded), they agree after the call. The call does not check that they agree.
 *   So the decode and map the caller passes in should come from a context with the same profile and the same
 *   ASTCENC_FLG_USE_DECODE_UNORM8 flag as this one, and the same decoded_type, decode_swizzle, input_components and block_metric.
 * All entries share data_type, swizzle, decoded_type and decode_swizzle; payloads, decodes and maps must not overlap each other
 * (not checked). The descriptor array is copied. Enqueued on `cuda_stream` (0 = the context's own stream) without
 * synchronising, in order with every other pass of the context: *count, the indices and the map are read on the device when the
 * call runs. No progress callback, no cancellation.
 * Cost: that of astcenc_b200_compress_device_block_lists over the sum of the capacities, with each chunk's scatter replaced by
 * three launches (a decode of the chunk's candidates, the decisions, the commits). With a_scale_radius (2D block sizes) each
 * entry gets an alpha-scale pre-pass over its whole image. Entries with capacity == 0 do nothing; a call whose capacities are all
 * zero launches nothing.
 * Errors, in this order; on error nothing is launched and nothing is written:
 *   1. ASTCENC_ERR_BAD_CONTEXT for a decompress-only context;
 *   2. ASTCENC_ERR_BAD_PARAM for a NULL swizzle, then ASTCENC_ERR_BAD_SWIZZLE for a swizzle with a selector beyond
 *      ASTCENC_SWZ_1; then the same two for decode_swizzle, whose selectors may go up to ASTCENC_SWZ_Z;
 *   3. ASTCENC_ERR_BAD_PARAM for input_components outside 1-4;
 *   4. ASTCENC_ERR_BAD_PARAM for block_metric not one of 0, 1, 2, 4, 5;
 *   5. ASTCENC_ERR_BAD_PARAM for lists == NULL with a non-zero count, then for a bad data_type, then for a bad decoded_type,
 *      then for an entry with a NULL data or payload, a NULL indices, count or block_error with capacity > 0, indices, count or
 *      block_error not aligned to 4 bytes, or data or decoded not aligned to its texel (4 / 8 / 16 bytes for U8 / F16 / F32:
 *      the call reads the original one texel per vector load), then for a zero or overflowing dimension;
 *   6. ASTCENC_ERR_NOT_IMPLEMENTED for a_scale_radius on a texture array;
 *   7. ASTCENC_ERR_BAD_PARAM for an image of 2^32 blocks or more, or when the sum of the capacities overflows.
 * All entries are checked before anything is enqueued.
 */
struct astcenc_b200_device_refine_list {
	const void* data;              /* device: the original, dim_z slices of dim_x * dim_y texels of data_type, contiguous */
	unsigned int dim_x, dim_y, dim_z;
	uint8_t* payload;              /* device: the image's whole payload (astcenc_compress_image's block order) */
	void* decoded;                 /* device: its decode, texels of decoded_type, or NULL */
	float* block_error;            /* device: its per-block map of block_metric, one float per block */
	const uint32_t* indices;       /* device: block positions */
	const uint32_t* count;         /* device: how many are listed */
	unsigned int capacity;         /* at most this many are read; the call's cost */
};
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_refine_device_block_lists(struct astcenc_context* context, const struct astcenc_b200_device_refine_list* lists,
                                                                        unsigned int list_count, enum astcenc_type data_type,
                                                                        const struct astcenc_swizzle* swizzle, enum astcenc_type decoded_type,
                                                                        const struct astcenc_swizzle* decode_swizzle, int input_components,
                                                                        enum astcenc_b200_block_metric block_metric, void* cuda_stream);

/**
 * Packed block lists: astcenc_b200_compress_device_block_lists and astcenc_b200_refine_device_block_lists at a cost set by a
 * budget the caller states rather than by the sum of the capacities. After astcenc_b200_select_blocks_pooled keeps the K worst
 * blocks of a texture set, each image's list needs capacity min(K, n_j), because the split of K between the images is known
 * only on the device; the unpacked calls stage every one of those slots, the packed calls stage at most `budget` of them.
 * The descriptors are those of the unpacked calls, and so are the arguments after `overflow`.
 * - Listed slots. Entry j lists v_j = min(*count_j, capacity_j) slots; the count is read on the device when the call runs. An
 *   entry of capacity 0 lists none, and its count is not read.
 * - Packing. Slot s < v_j of entry j gets the packed position P_j + s, P_j being the sum of v_i over the entries i < j in call
 *   order (summed in 64 bits, without overflow). Packing reads only the count words, never the indices: a slot whose index is
 *   out of range still takes a position, and the list rule then skips it.
 * - Budget. A slot at a packed position below `budget` is processed exactly as the unpacked call processes it: the list rule,
 *   skipped indices and duplicates, and for refine calls the candidate, its value v', the commit rule and the consistency of
 *   payload, decode and map. A slot at or beyond `budget` is not processed, and its block keeps every byte. Truncation
 *   therefore drops the trailing slots in entry order, deterministically.
 * - Equivalence. When the sum of v_j is at most `budget`, the packed call writes the same payload bytes as the unpacked call
 *   with the same table, byte for byte, and a refine call the same decoded texels and map values, bit for bit. With the lists
 *   of astcenc_b200_select_blocks_pooled and `budget` the sum of the capacities of the pools that cover the entries, this
 *   always holds.
 * - overflow. A device word, or NULL, aligned to 4 bytes. It receives the sum of v_j minus `budget` when that is positive and 0
 *   otherwise, saturated at 0xFFFFFFFF. Every successful call in which some entry has capacity > 0 writes it, budget == 0
 *   included.
 * Cost: the staging row has min(budget, sum of capacity_j) slots (the host knows both), so a packed call never stages more
 * than the unpacked one. The call makes the unpacked call's launches over that many slots plus one, the packing kernel,
 * launched after the table copy and before the first gather. A call whose capacities are all 0 launches nothing and writes
 * nothing; a call with budget == 0 and some capacity is the packing launch alone. With a_scale_radius (2D block sizes) each
 * entry gets its whole-image alpha-scale pre-pass, as in the unpacked call.
 * Errors: those of the unpacked call, in its order; after them ASTCENC_ERR_BAD_PARAM for an overflow pointer not aligned to 4
 * bytes. On error nothing is launched and nothing is written. Any budget is accepted.
 */
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_compress_device_block_lists_packed(
    struct astcenc_context* context, const struct astcenc_b200_device_block_list* lists, unsigned int list_count,
    unsigned int budget, uint32_t* overflow, enum astcenc_type data_type, const struct astcenc_swizzle* swizzle, void* cuda_stream);

ASTCENC_PUBLIC enum astcenc_error astcenc_b200_refine_device_block_lists_packed(
    struct astcenc_context* context, const struct astcenc_b200_device_refine_list* lists, unsigned int list_count,
    unsigned int budget, uint32_t* overflow, enum astcenc_type data_type, const struct astcenc_swizzle* swizzle,
    enum astcenc_type decoded_type, const struct astcenc_swizzle* decode_swizzle, int input_components,
    enum astcenc_b200_block_metric block_metric, void* cuda_stream);

/**
 * Totals of device-resident per-block maps, and from each total a selection weight that is zero once the image meets a target:
 * the device side of a per-image quality target ("every texture at 40 dB or better") in the refinement loop.
 * - Total. The sum of the entry's block_count map values, accumulated in double in a fixed order that depends only on
 *   block_count: never on the GPU, on the other entries of the call or on their order. NaN values propagate into the total;
 *   block_count == 0 gives 0.
 * - Weight. 0 unless total > limit and total > 0 (so a NaN total gives 0); otherwise 1.0f under ASTCENC_B200_WEIGHT_ONE and
 *   (float)(1.0 / total) under ASTCENC_B200_WEIGHT_INVERSE_TOTAL (0 for an infinite total). A weight of 0 in
 *   astcenc_b200_select_blocks_pooled with a pool threshold of 0 makes none of the image's blocks a candidate (the product is 0,
 *   or NaN where the map holds inf): that is how an image that meets its target leaves the pool.
 * - Targets. With each map a whole per-block map of astcenc_b200_compute_block_metric_device_images (and the identities stated
 *   above enum astcenc_b200_block_metric), the image meets a target when total <= limit with:
 *     SQUARED_ERROR, PSNR of at least P dB:               limit = samples * 10^(-P / 10);
 *     ALPHA_WEIGHTED_ERROR, alpha_psnr of at least P dB:  limit = samples * 10^(-P / 10), input_components == 4;
 *     LOG2_ERROR, log_rmse of at most R:                  limit = R^2 * pixels;
 *     ANGULAR_ERROR, mean_angular_error of at most D deg: limit = D * pixels;
 *   samples being pixels times the number of channels input_components selects. A total agrees with the figure's error sum up
 *   to the per-block float rounding of the map, so a target met within that rounding may be judged either way. limit
 *   = -INFINITY never meets the target. The total of a WORST_ANGULAR_ERROR map is a sum of maxima and is not a target. For "no
 *   texel worse than T degrees", call astcenc_b200_select_blocks (or astcenc_b200_select_blocks_pooled with no weight) on that
 *   map with threshold T and a capacity, then refine with the same metric: the candidates are exactly the blocks that still
 *   have a texel beyond T, so a round in which none is left lists nothing.
 * - The closed loop. Compress, decode and map the set once; then enqueue every round up front, each one this call (then the
 *   weights are current), astcenc_b200_select_blocks_pooled with these weights, a threshold of 0 and the round's budget K, and
 *   astcenc_b200_refine_device_block_lists_packed with budget K, which keeps the maps current and stages K slots rather than
 *   the sum of the capacities min(K, n_j). Images that reach their target get no blocks in later rounds and the budget goes
 *   to those that still miss theirs, with no host synchronisation between rounds.
 *   ASTCENC_B200_WEIGHT_INVERSE_TOTAL gives the weights 1 / E_j (rule (d) of the pooled selection: a block ranks by its share
 *   of its image's error) with the same gate.
 * Enqueued on `cuda_stream` (0 = the context's own stream) without synchronising, in order with every other pass of the
 * context; works on any context, decompress-only ones included. The descriptor array is copied. The call is one table copy and
 * two kernel launches, whatever the number of entries; entry_count == 0 launches nothing. Outputs must not overlap any map or
 * each other (not checked).
 * Errors, in this order; on error nothing is launched and nothing is written:
 *   1. ASTCENC_ERR_BAD_PARAM for a NULL context or entries == NULL with entry_count > 0;
 *   2. ASTCENC_ERR_BAD_PARAM for a rule outside 0-1;
 *   3. ASTCENC_ERR_BAD_PARAM for an entry with a NULL map and block_count > 0, a NaN limit, a map or weight not aligned to 4
 *      bytes, or a total not aligned to 8;
 *   4. ASTCENC_ERR_BAD_PARAM when the call does not fit a launch (more than 2^31 - 1 virtual CTAs: a few million entries of
 *      large maps).
 * All entries are checked before anything is enqueued.
 */
enum astcenc_b200_weight_rule {
	ASTCENC_B200_WEIGHT_ONE = 0,            /* weight 1 while the image misses its target */
	ASTCENC_B200_WEIGHT_INVERSE_TOTAL = 1   /* weight 1 / total while the image misses its target (rule (d)) */
};
struct astcenc_b200_block_map_total {
	const float* map;              /* device: block_count values, e.g. a map of astcenc_b200_compute_block_metric_device_images */
	unsigned int block_count;
	double limit;                  /* the image meets its target when total <= limit; -INFINITY: never */
	double* total;                 /* device, or NULL: receives the map's total */
	float* weight;                 /* device, or NULL: receives the selection weight */
};
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_total_block_maps(struct astcenc_context* context, const struct astcenc_b200_block_map_total* entries,
                                                                unsigned int entry_count, enum astcenc_b200_weight_rule rule, void* cuda_stream);

/**
 * Block info of device-resident payloads on the device: what astcenc_get_block_info reports, for whole payloads or for the
 * blocks of device lists, without copying a block to the host. For callers who want to see what a refinement round did to an
 * encoding (which blocks now use two partitions or dual planes, which are constant, which weight grids a mip chain's small
 * levels use), or whether a payload loaded from a file holds error blocks, and where, before it is decoded or shipped.
 *
 * astcenc_b200_get_block_summaries_device_images: a 16-byte summary of every block of whole payloads.
 * images[i] describes a payload ALREADY RESIDENT in device memory (astcenc_compress_image's block order, 16 bytes per block, of
 * an image of dim_x * dim_y * dim_z texels in the context's footprint) and a device array of one summary per block, in the
 * same order. Every field of summaries[b] equals the same-named field astcenc_get_block_info on this context writes for block
 * b's 16 bytes, narrowed to the field's width (every value fits): flags holds its four is_* fields as the bits below, and
 * dual_plane_component is 0xFF where astcenc_get_block_info reports 0xFFFFFFFF (a block with one plane). An error or constant
 * block therefore gets its flag and zeros, as astcenc_get_block_info returns early for them. reserved is written as 0.
 *
 * astcenc_b200_get_block_info_device_block_lists: the full astcenc_block_info of the blocks of device lists, for drilling into
 * the blocks a selection picked. lists[i] describes a payload ALREADY RESIDENT in device memory, a device index list with a
 * device count, and a device array of capacity structs. The list rule is that of astcenc_b200_decompress_device_block_lists:
 * the call reads the first min(*count, capacity) slots, and a slot whose index is at or beyond the image's block count is
 * skipped. The output is indexed by slot, not by block: each read slot s receives in infos[s], byte for byte, the whole struct
 * astcenc_get_block_info on this context writes for block indices[s], its zeros included. Skipped slots and slots past the
 * count are left untouched; duplicate indices write the same bytes.
 *
 * Both calls:
 * - Take 2D images, texture arrays (2D block sizes; z counts the slices) and volumes of 3D block sizes, and work on
 *   decompress-only contexts. Outputs must not overlap each other or any payload (not checked).
 * - Are enqueued on `cuda_stream` (0 = the context's own stream) without synchronising, in order with every other pass of the
 *   context: the counts and the indices are read on the device when the call runs. The descriptor array is copied.
 * - Cost one table copy and one kernel launch (one lane per block for summaries, one warp per slot for lists, over the sum of
 *   the capacities). A call with nothing to do (no images, or capacities all zero) launches nothing.
 * - Errors, in this order; on error nothing is launched and nothing is written:
 *     1. ASTCENC_ERR_BAD_PARAM for a NULL context;
 *     2. ASTCENC_ERR_BAD_PARAM for a NULL table with a non-zero count;
 *     3. ASTCENC_ERR_BAD_PARAM for an entry with a NULL payload or output (summaries; for lists, infos, indices or count with
 *        capacity > 0), or an output not aligned: summaries to 16 bytes, indices, count and infos to 4;
 *     4. ASTCENC_ERR_BAD_PARAM for a zero or overflowing dimension;
 *     5. ASTCENC_ERR_BAD_PARAM for an image of 2^32 blocks or more, or a call whose block or slot total overflows.
 *   Every entry is checked before anything is enqueued.
 */
static const unsigned int ASTCENC_B200_BLOCK_IS_ERROR = 1, ASTCENC_B200_BLOCK_IS_CONSTANT = 2, ASTCENC_B200_BLOCK_IS_HDR = 4,
                          ASTCENC_B200_BLOCK_IS_DUAL_PLANE = 8;
struct astcenc_b200_block_summary {    /* 16 bytes */
	uint8_t flags;                     /* ASTCENC_B200_BLOCK_IS_* */
	uint8_t partition_count;
	uint16_t partition_index;
	uint8_t dual_plane_component;      /* 0xFF for a block with one plane */
	uint8_t weight_x, weight_y, weight_z;
	uint8_t color_endpoint_modes[4];
	uint16_t color_level_count;
	uint8_t weight_level_count;
	uint8_t reserved;                  /* written as 0 */
};
struct astcenc_b200_device_block_summary_image {
	const uint8_t* payload;            /* device: the whole payload, astcenc_compress_image's block order */
	unsigned int dim_x, dim_y, dim_z;
	struct astcenc_b200_block_summary* summaries;   /* device: one per block, same order; 16-byte aligned */
};
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_get_block_summaries_device_images(struct astcenc_context* context,
                                                                                 const struct astcenc_b200_device_block_summary_image* images,
                                                                                 unsigned int image_count, void* cuda_stream);

struct astcenc_b200_device_block_info_list {
	const uint8_t* payload;            /* device: the whole payload, astcenc_compress_image's block order */
	unsigned int dim_x, dim_y, dim_z;
	const uint32_t* indices;           /* device: block positions in that order */
	const uint32_t* count;             /* device: how many are listed */
	unsigned int capacity;             /* at most this many are read; the call's cost */
	struct astcenc_block_info* infos;  /* device: capacity structs; slot s describes block indices[s] */
};
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_get_block_info_device_block_lists(struct astcenc_context* context,
                                                                                 const struct astcenc_b200_device_block_info_list* lists,
                                                                                 unsigned int list_count, void* cuda_stream);

/**
 * The .astc container (Docs/FileFormat.md; Source/astcenccli_image_load_store.cpp:2573-2760, load_cimage / store_cimage):
 * a 16-byte header - magic 13 AB A1 5C, block dimensions (one byte each), image dimensions (24 bits each, little endian)
 * - followed by the blocks as astcenc_compress_image() wrote them.
 * store: data_len must be the size of the block grid the header describes.
 * load: call with data == NULL to get the header and the payload size in *data_len, then again with a buffer;
 * corrupt files (bad magic, zero dimensions, size overflow, fewer payload bytes than the header promises) give
 * ASTCENC_ERR_BAD_PARAM, a buffer smaller than the payload ASTCENC_ERR_OUT_OF_MEM.
 */
struct astcenc_b200_cimage_header {
	unsigned int block_x, block_y, block_z;
	unsigned int dim_x, dim_y, dim_z;
};
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_store_cimage(const char* filename, const struct astcenc_b200_cimage_header* header,
                                                            const uint8_t* data, size_t data_len);
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_load_cimage(const char* filename, struct astcenc_b200_cimage_header* header,
                                                           uint8_t* data, size_t data_capacity, size_t* data_len);

/**
 * The same payload in a KTX 1 container (Source/astcenccli_image_load_store.cpp:870-905 header, :1294-1440
 * load_ktx_compressed_image / store_ktx_compressed_image): 64-byte header with glInternalFormat =
 * GL_COMPRESSED_RGBA_ASTC_<footprint> (or the SRGB8_ALPHA8 variant when is_srgb), one mip level, no key/value data, then
 * the 32-bit payload size and the blocks. load accepts files of either byte order, skips key/value data and reads the first
 * mip level; the two-call protocol (data == NULL first) and the error codes are those of astcenc_b200_load_cimage, a footprint
 * without a GL enum gives ASTCENC_ERR_BAD_BLOCK_SIZE on store.
 */
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_store_ktx_cimage(const char* filename, const struct astcenc_b200_cimage_header* header, int is_srgb,
                                                                const uint8_t* data, size_t data_len);
ASTCENC_PUBLIC enum astcenc_error astcenc_b200_load_ktx_cimage(const char* filename, struct astcenc_b200_cimage_header* header, int* is_srgb,
                                                               uint8_t* data, size_t data_capacity, size_t* data_len);

#endif
