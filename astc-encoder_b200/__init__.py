"""astc-encoder_b200: CUDA-native ASTC block compressor (NVIDIA H100, sm_90a) behind the astcenc.h C ABI.

This module is the thin Python mirror of the C interface (same names and argument meaning as
astcenc.h: config_init -> context_alloc -> compress_image); all compression happens in
libastcenc_b200.so (hand-written sm_90a kernels). There is no CPU fallback: importing works
anywhere, but creating a context without a CUDA device raises.

PyTorch is used only as plumbing (device buffers, streams, torch.distributed); see
compress_device() for the device-resident entry point used by bench.py and the multi-GPU path.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("ASTCENC_B200_LIB") or os.path.join(_HERE, "libastcenc_b200.so")      # (the override is for A/B builds in tools/)

PRF_LDR_SRGB, PRF_LDR, PRF_HDR_RGB_LDR_A, PRF_HDR = 0, 1, 2, 3
PRE_FASTEST, PRE_FAST, PRE_MEDIUM, PRE_THOROUGH, PRE_VERYTHOROUGH, PRE_EXHAUSTIVE = 0.0, 10.0, 60.0, 98.0, 99.0, 100.0
FLG_MAP_NORMAL, FLG_USE_DECODE_UNORM8, FLG_USE_ALPHA_WEIGHT, FLG_USE_PERCEPTUAL = 1, 2, 4, 8
FLG_DECOMPRESS_ONLY, FLG_SELF_DECOMPRESS_ONLY, FLG_MAP_RGBM = 16, 32, 64
TYPE_U8, TYPE_F16, TYPE_F32 = 0, 1, 2
ERROR_NAMES = ["ASTCENC_SUCCESS", "ASTCENC_ERR_OUT_OF_MEM", "ASTCENC_ERR_BAD_CPU_FLOAT", "ASTCENC_ERR_BAD_PARAM", "ASTCENC_ERR_BAD_BLOCK_SIZE",
               "ASTCENC_ERR_BAD_PROFILE", "ASTCENC_ERR_BAD_QUALITY", "ASTCENC_ERR_BAD_SWIZZLE", "ASTCENC_ERR_BAD_FLAGS", "ASTCENC_ERR_BAD_CONTEXT",
               "ASTCENC_ERR_NOT_IMPLEMENTED", "ASTCENC_ERR_BAD_DECODE_MODE"]


ERR_OUT_OF_MEM, ERR_BAD_PARAM, ERR_BAD_BLOCK_SIZE, ERR_BAD_SWIZZLE, ERR_BAD_CONTEXT, ERR_NOT_IMPLEMENTED = 1, 3, 4, 7, 9, 10
# enum astcenc_b200_block_metric: what a per-block error map measures
BLOCK_SQUARED_ERROR, BLOCK_ALPHA_WEIGHTED_ERROR, BLOCK_LOG2_ERROR = 0, 1, 2
# normal maps: the sum of each texel's angle in degrees, and the largest one (3 is not assigned)
BLOCK_ANGULAR_ERROR, BLOCK_WORST_ANGULAR_ERROR = 4, 5
# enum astcenc_b200_weight_rule: the selection weight of an image that misses its target
WEIGHT_ONE, WEIGHT_INVERSE_TOTAL = 0, 1
# the flags of struct astcenc_b200_block_summary
BLOCK_IS_ERROR, BLOCK_IS_CONSTANT, BLOCK_IS_HDR, BLOCK_IS_DUAL_PLANE = 1, 2, 4, 8
# sizeof(struct astcenc_block_info): the slot size of get_block_info_device_block_lists outputs
BLOCK_INFO_BYTES = 2144


class AstcencError(RuntimeError):
    def __init__(self, code, what):
        self.code = code
        RuntimeError.__init__(self, "%s: %s" % (what, ERROR_NAMES[code] if 0 <= code < len(ERROR_NAMES) else code))


class Config(C.Structure):
    """astcenc_config (astcenc.h:427-605)."""
    _fields_ = [
        ("profile", C.c_int), ("flags", C.c_uint), ("block_x", C.c_uint), ("block_y", C.c_uint), ("block_z", C.c_uint),
        ("cw_r_weight", C.c_float), ("cw_g_weight", C.c_float), ("cw_b_weight", C.c_float), ("cw_a_weight", C.c_float),
        ("a_scale_radius", C.c_uint), ("rgbm_m_scale", C.c_float),
        ("tune_partition_count_limit", C.c_uint), ("tune_2partition_index_limit", C.c_uint),
        ("tune_3partition_index_limit", C.c_uint), ("tune_4partition_index_limit", C.c_uint),
        ("tune_block_mode_limit", C.c_uint), ("tune_refinement_limit", C.c_uint), ("tune_candidate_limit", C.c_uint),
        ("tune_2partitioning_candidate_limit", C.c_uint), ("tune_3partitioning_candidate_limit", C.c_uint),
        ("tune_4partitioning_candidate_limit", C.c_uint),
        ("tune_db_limit", C.c_float), ("tune_mse_overshoot", C.c_float),
        ("tune_2partition_early_out_limit_factor", C.c_float), ("tune_3partition_early_out_limit_factor", C.c_float),
        ("tune_2plane_early_out_limit_correlation", C.c_float), ("tune_search_mode0_enable", C.c_float),
        ("progress_callback", C.c_void_p),
    ]


class Image(C.Structure):
    _fields_ = [("dim_x", C.c_uint), ("dim_y", C.c_uint), ("dim_z", C.c_uint), ("data_type", C.c_int), ("data", C.POINTER(C.c_void_p))]


class Swizzle(C.Structure):
    _fields_ = [("r", C.c_int), ("g", C.c_int), ("b", C.c_int), ("a", C.c_int)]


class DeviceImage(C.Structure):
    """struct astcenc_b200_device_image (include/astcenc.h)."""
    _fields_ = [("data", C.c_void_p), ("dim_x", C.c_uint), ("dim_y", C.c_uint), ("dim_z", C.c_uint), ("payload", C.c_void_p)]


class DeviceDecodeImage(C.Structure):
    """struct astcenc_b200_device_decode_image (include/astcenc.h)."""
    _fields_ = [("payload", C.c_void_p), ("data", C.c_void_p), ("dim_x", C.c_uint), ("dim_y", C.c_uint), ("dim_z", C.c_uint)]


class DeviceMetricsImage(C.Structure):
    """struct astcenc_b200_device_metrics_image (include/astcenc.h)."""
    _fields_ = [("original", C.c_void_p), ("decoded", C.c_void_p), ("original_type", C.c_int), ("decoded_type", C.c_int), ("dim_x", C.c_uint),
                ("dim_y", C.c_uint), ("dim_z", C.c_uint), ("metrics", C.c_void_p), ("block_error", C.c_void_p)]


class BlockSelection(C.Structure):
    """struct astcenc_b200_block_selection (include/astcenc.h)."""
    _fields_ = [("map", C.c_void_p), ("block_count", C.c_uint), ("threshold", C.c_float), ("capacity", C.c_uint), ("indices", C.c_void_p),
                ("count", C.c_void_p)]


class BlockPool(C.Structure):
    """struct astcenc_b200_block_pool (include/astcenc.h)."""
    _fields_ = [("entry_count", C.c_uint), ("threshold", C.c_float), ("capacity", C.c_uint)]


class PooledSelection(C.Structure):
    """struct astcenc_b200_pooled_selection (include/astcenc.h)."""
    _fields_ = [("map", C.c_void_p), ("block_count", C.c_uint), ("weight", C.c_void_p), ("indices", C.c_void_p), ("count", C.c_void_p)]


class BlockMapTotal(C.Structure):
    """struct astcenc_b200_block_map_total (include/astcenc.h)."""
    _fields_ = [("map", C.c_void_p), ("block_count", C.c_uint), ("limit", C.c_double), ("total", C.c_void_p), ("weight", C.c_void_p)]


class DeviceBlockList(C.Structure):
    """struct astcenc_b200_device_block_list (include/astcenc.h)."""
    _fields_ = [("data", C.c_void_p), ("dim_x", C.c_uint), ("dim_y", C.c_uint), ("dim_z", C.c_uint), ("payload", C.c_void_p), ("indices", C.c_void_p),
                ("count", C.c_void_p), ("capacity", C.c_uint)]


class DeviceDecodeBlockList(C.Structure):
    """struct astcenc_b200_device_decode_block_list (include/astcenc.h)."""
    _fields_ = [("payload", C.c_void_p), ("data", C.c_void_p), ("dim_x", C.c_uint), ("dim_y", C.c_uint), ("dim_z", C.c_uint), ("indices", C.c_void_p),
                ("count", C.c_void_p), ("capacity", C.c_uint)]


class DeviceBlockErrorList(C.Structure):
    """struct astcenc_b200_device_block_error_list (include/astcenc.h)."""
    _fields_ = [("original", C.c_void_p), ("decoded", C.c_void_p), ("original_type", C.c_int), ("decoded_type", C.c_int), ("dim_x", C.c_uint),
                ("dim_y", C.c_uint), ("dim_z", C.c_uint), ("block_error", C.c_void_p), ("indices", C.c_void_p), ("count", C.c_void_p),
                ("capacity", C.c_uint)]


class DeviceRefineList(C.Structure):
    """struct astcenc_b200_device_refine_list (include/astcenc.h)."""
    _fields_ = [("data", C.c_void_p), ("dim_x", C.c_uint), ("dim_y", C.c_uint), ("dim_z", C.c_uint), ("payload", C.c_void_p), ("decoded", C.c_void_p),
                ("block_error", C.c_void_p), ("indices", C.c_void_p), ("count", C.c_void_p), ("capacity", C.c_uint)]


class BlockSummary(C.Structure):
    """struct astcenc_b200_block_summary (include/astcenc.h): 16 bytes per block."""
    _fields_ = [("flags", C.c_uint8), ("partition_count", C.c_uint8), ("partition_index", C.c_uint16), ("dual_plane_component", C.c_uint8),
                ("weight_x", C.c_uint8), ("weight_y", C.c_uint8), ("weight_z", C.c_uint8), ("color_endpoint_modes", C.c_uint8 * 4),
                ("color_level_count", C.c_uint16), ("weight_level_count", C.c_uint8), ("reserved", C.c_uint8)]


# The same layout as a numpy structured dtype: a torch uint8 buffer of summaries, copied to the host as numpy, is read field by
# field with buf.view(BLOCK_SUMMARY_DTYPE)["partition_count"].
BLOCK_SUMMARY_DTYPE = np.dtype([("flags", np.uint8), ("partition_count", np.uint8), ("partition_index", "<u2"), ("dual_plane_component", np.uint8),
                                ("weight_x", np.uint8), ("weight_y", np.uint8), ("weight_z", np.uint8), ("color_endpoint_modes", np.uint8, (4,)),
                                ("color_level_count", "<u2"), ("weight_level_count", np.uint8), ("reserved", np.uint8)])
assert BLOCK_SUMMARY_DTYPE.itemsize == C.sizeof(BlockSummary) == 16


class DeviceBlockSummaryImage(C.Structure):
    """struct astcenc_b200_device_block_summary_image (include/astcenc.h)."""
    _fields_ = [("payload", C.c_void_p), ("dim_x", C.c_uint), ("dim_y", C.c_uint), ("dim_z", C.c_uint), ("summaries", C.c_void_p)]


class DeviceBlockInfoList(C.Structure):
    """struct astcenc_b200_device_block_info_list (include/astcenc.h)."""
    _fields_ = [("payload", C.c_void_p), ("dim_x", C.c_uint), ("dim_y", C.c_uint), ("dim_z", C.c_uint), ("indices", C.c_void_p), ("count", C.c_void_p),
                ("capacity", C.c_uint), ("infos", C.c_void_p)]


class ErrorMetrics(C.Structure):
    """struct astcenc_b200_error_metrics (include/astcenc.h)."""
    _fields_ = [(n, C.c_double) for n in ("psnr", "alpha_psnr", "rgb_psnr", "rgb_peak", "peak_psnr", "mpsnr", "log_rmse",
                                          "mean_angular_error", "worst_angular_error")] + [("sum_squared_error", C.c_double * 4)]


class CImageHeader(C.Structure):
    """struct astcenc_b200_cimage_header (include/astcenc.h): the fields of the 16-byte .astc header."""
    _fields_ = [(n, C.c_uint) for n in ("block_x", "block_y", "block_z", "dim_x", "dim_y", "dim_z")]


def build(verbose=False):
    """Compile libastcenc_b200.so for sm_90a in-tree (nvcc cross-compiles without a GPU)."""
    r = subprocess.run(["make", "-C", _HERE], capture_output=True, text=True)
    if verbose or r.returncode != 0:
        print(r.stdout[-4000:], r.stderr[-4000:])
    if r.returncode != 0:
        raise RuntimeError("building libastcenc_b200.so failed")
    return LIB_PATH


_lib = None


def lib():
    """The loaded C library. Fails loudly if it was not built - there is no Python/CPU fallback."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("libastcenc_b200.so is missing: run `make -C %s` (or __graft_entry__.build())" % _HERE)
        l = C.CDLL(LIB_PATH, mode=os.RTLD_LOCAL)
        l.astcenc_config_init.argtypes = [C.c_int, C.c_uint, C.c_uint, C.c_uint, C.c_float, C.c_uint, C.POINTER(Config)]
        l.astcenc_config_init.restype = C.c_int
        l.astcenc_context_alloc.argtypes = [C.POINTER(Config), C.c_uint, C.POINTER(C.c_void_p), C.c_void_p]
        l.astcenc_context_alloc.restype = C.c_int
        l.astcenc_compress_image.argtypes = [C.c_void_p, C.POINTER(Image), C.POINTER(Swizzle), C.c_void_p, C.c_size_t, C.c_uint]
        l.astcenc_compress_image.restype = C.c_int
        l.astcenc_compress_reset.argtypes = [C.c_void_p]
        l.astcenc_compress_reset.restype = C.c_int
        l.astcenc_decompress_image.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(Image), C.POINTER(Swizzle), C.c_uint]
        l.astcenc_decompress_image.restype = C.c_int
        l.astcenc_compress_cancel.argtypes = [C.c_void_p]
        l.astcenc_compress_cancel.restype = C.c_int
        l.astcenc_context_free.argtypes = [C.c_void_p]
        l.astcenc_context_free.restype = None
        l.astcenc_get_error_string.argtypes = [C.c_int]
        l.astcenc_get_error_string.restype = C.c_char_p
        l.astcenc_b200_compress_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_uint, C.c_uint, C.POINTER(Swizzle), C.c_uint, C.c_uint, C.c_void_p, C.c_void_p]
        l.astcenc_b200_compress_device.restype = C.c_int
        l.astcenc_b200_compress_device_blocks.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_uint, C.c_uint, C.c_uint, C.POINTER(Swizzle), C.c_void_p,
                                                          C.c_uint, C.c_void_p, C.c_void_p]
        l.astcenc_b200_compress_device_blocks.restype = C.c_int
        l.astcenc_b200_compress_device_images.argtypes = [C.c_void_p, C.POINTER(DeviceImage), C.c_uint, C.c_int, C.POINTER(Swizzle), C.c_void_p]
        l.astcenc_b200_compress_device_images.restype = C.c_int
        l.astcenc_b200_compress_images.argtypes = [C.c_void_p, C.POINTER(C.POINTER(Image)), C.c_uint, C.POINTER(Swizzle), C.POINTER(C.c_void_p),
                                                   C.POINTER(C.c_size_t)]
        l.astcenc_b200_compress_images.restype = C.c_int
        l.astcenc_b200_decompress_device_images.argtypes = [C.c_void_p, C.POINTER(DeviceDecodeImage), C.c_uint, C.c_int, C.POINTER(Swizzle), C.c_void_p]
        l.astcenc_b200_decompress_device_images.restype = C.c_int
        l.astcenc_b200_launch_count.argtypes = [C.c_void_p]
        l.astcenc_b200_launch_count.restype = C.c_ulonglong
        l.astcenc_b200_last_timing.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
        l.astcenc_b200_last_timing.restype = C.c_int
        l.astcenc_b200_stage_timing.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_uint)]
        l.astcenc_b200_stage_timing.restype = C.c_int
        l.astcenc_b200_compute_error_metrics.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(Image), C.POINTER(Image), C.c_int, C.c_int,
                                                         C.POINTER(ErrorMetrics)]
        l.astcenc_b200_compute_error_metrics.restype = C.c_int
        l.astcenc_b200_compute_error_metrics_device_images.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(DeviceMetricsImage), C.c_uint,
                                                                       C.c_int, C.c_int, C.c_void_p]
        l.astcenc_b200_compute_error_metrics_device_images.restype = C.c_int
        l.astcenc_b200_compute_block_metric_device_images.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(DeviceMetricsImage), C.c_uint,
                                                                      C.c_int, C.c_int, C.c_void_p]
        l.astcenc_b200_compute_block_metric_device_images.restype = C.c_int
        l.astcenc_b200_select_blocks.argtypes = [C.c_void_p, C.POINTER(BlockSelection), C.c_uint, C.c_void_p]
        l.astcenc_b200_select_blocks.restype = C.c_int
        l.astcenc_b200_select_blocks_pooled.argtypes = [C.c_void_p, C.POINTER(BlockPool), C.c_uint, C.POINTER(PooledSelection), C.c_uint, C.c_void_p]
        l.astcenc_b200_select_blocks_pooled.restype = C.c_int
        l.astcenc_b200_total_block_maps.argtypes = [C.c_void_p, C.POINTER(BlockMapTotal), C.c_uint, C.c_int, C.c_void_p]
        l.astcenc_b200_total_block_maps.restype = C.c_int
        l.astcenc_b200_compress_device_block_lists.argtypes = [C.c_void_p, C.POINTER(DeviceBlockList), C.c_uint, C.c_int, C.POINTER(Swizzle), C.c_void_p]
        l.astcenc_b200_compress_device_block_lists.restype = C.c_int
        l.astcenc_b200_decompress_device_block_lists.argtypes = [C.c_void_p, C.POINTER(DeviceDecodeBlockList), C.c_uint, C.c_int, C.POINTER(Swizzle),
                                                                 C.c_void_p]
        l.astcenc_b200_decompress_device_block_lists.restype = C.c_int
        l.astcenc_b200_compute_block_errors_device_block_lists.argtypes = [C.c_void_p, C.c_int, C.POINTER(DeviceBlockErrorList), C.c_uint, C.c_void_p]
        l.astcenc_b200_compute_block_errors_device_block_lists.restype = C.c_int
        l.astcenc_b200_compute_block_metric_device_block_lists.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(DeviceBlockErrorList), C.c_uint,
                                                                           C.c_void_p]
        l.astcenc_b200_compute_block_metric_device_block_lists.restype = C.c_int
        l.astcenc_b200_refine_device_block_lists.argtypes = [C.c_void_p, C.POINTER(DeviceRefineList), C.c_uint, C.c_int, C.POINTER(Swizzle), C.c_int,
                                                             C.POINTER(Swizzle), C.c_int, C.c_int, C.c_void_p]
        l.astcenc_b200_refine_device_block_lists.restype = C.c_int
        l.astcenc_b200_compress_device_block_lists_packed.argtypes = [C.c_void_p, C.POINTER(DeviceBlockList), C.c_uint, C.c_uint, C.c_void_p, C.c_int,
                                                                      C.POINTER(Swizzle), C.c_void_p]
        l.astcenc_b200_compress_device_block_lists_packed.restype = C.c_int
        l.astcenc_b200_refine_device_block_lists_packed.argtypes = [C.c_void_p, C.POINTER(DeviceRefineList), C.c_uint, C.c_uint, C.c_void_p, C.c_int,
                                                                    C.POINTER(Swizzle), C.c_int, C.POINTER(Swizzle), C.c_int, C.c_int, C.c_void_p]
        l.astcenc_b200_refine_device_block_lists_packed.restype = C.c_int
        l.astcenc_b200_get_block_summaries_device_images.argtypes = [C.c_void_p, C.POINTER(DeviceBlockSummaryImage), C.c_uint, C.c_void_p]
        l.astcenc_b200_get_block_summaries_device_images.restype = C.c_int
        l.astcenc_b200_get_block_info_device_block_lists.argtypes = [C.c_void_p, C.POINTER(DeviceBlockInfoList), C.c_uint, C.c_void_p]
        l.astcenc_b200_get_block_info_device_block_lists.restype = C.c_int
        l.astcenc_b200_store_cimage.argtypes = [C.c_char_p, C.POINTER(CImageHeader), C.c_void_p, C.c_size_t]
        l.astcenc_b200_store_cimage.restype = C.c_int
        l.astcenc_b200_load_cimage.argtypes = [C.c_char_p, C.POINTER(CImageHeader), C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        l.astcenc_b200_load_cimage.restype = C.c_int
        l.astcenc_b200_store_ktx_cimage.argtypes = [C.c_char_p, C.POINTER(CImageHeader), C.c_int, C.c_void_p, C.c_size_t]
        l.astcenc_b200_store_ktx_cimage.restype = C.c_int
        l.astcenc_b200_load_ktx_cimage.argtypes = [C.c_char_p, C.POINTER(CImageHeader), C.POINTER(C.c_int), C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        l.astcenc_b200_load_ktx_cimage.restype = C.c_int
        l.astcenc_b200_comm_unique_id.argtypes = [C.c_void_p, C.c_size_t]
        l.astcenc_b200_comm_unique_id.restype = C.c_int
        l.astcenc_b200_comm_init.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_size_t]
        l.astcenc_b200_comm_init.restype = C.c_int
        l.astcenc_b200_comm_free.argtypes = [C.c_void_p]
        l.astcenc_b200_comm_free.restype = C.c_int
        l.astcenc_b200_slab_rows.argtypes = [C.c_void_p, C.c_uint, C.c_int, C.c_int, C.POINTER(C.c_uint), C.POINTER(C.c_uint)]
        l.astcenc_b200_slab_rows.restype = C.c_int
        l.astcenc_b200_compress_image_sharded.argtypes = [C.c_void_p, C.POINTER(Image), C.POINTER(Swizzle), C.c_void_p, C.c_size_t, C.c_int]
        l.astcenc_b200_compress_image_sharded.restype = C.c_int
        l.astcenc_b200_compress_batch.argtypes = [C.c_void_p, C.POINTER(C.POINTER(Image)), C.c_uint, C.POINTER(Swizzle), C.POINTER(C.c_void_p), C.c_size_t, C.c_int]
        l.astcenc_b200_compress_batch.restype = C.c_int
        l.astcenc_b200_comm_last_timing.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float)]
        l.astcenc_b200_comm_last_timing.restype = C.c_int
        _lib = l
    return _lib


COMM_ID_BYTES = 128


def comm_unique_id():
    """astcenc_b200_comm_unique_id: the 128-byte NCCL rendezvous id (made on one rank, shipped to the others by the caller)."""
    buf = (C.c_uint8 * COMM_ID_BYTES)()
    err = lib().astcenc_b200_comm_unique_id(buf, COMM_ID_BYTES)
    if err:
        raise AstcencError(err, "astcenc_b200_comm_unique_id")
    return bytes(buf)


def config_init(profile, block_x, block_y, quality, flags=0, block_z=1, **overrides):
    """astcenc_config_init (astcenc.h:725-749); keyword overrides edit tune_* fields like the CLI's power-user switches."""
    cfg = Config()
    err = lib().astcenc_config_init(profile, block_x, block_y, block_z, quality, flags, C.byref(cfg))
    if err:
        raise AstcencError(err, "astcenc_config_init")
    for k, v in overrides.items():
        setattr(cfg, k, v)
    return cfg


_DTYPES = {np.dtype(np.uint8): TYPE_U8, np.dtype(np.float16): TYPE_F16, np.dtype(np.float32): TYPE_F32}

PROGRESS_CALLBACK = C.CFUNCTYPE(None, C.c_float)      # astcenc_progress_callback


class Context:
    """astcenc_context (astcenc_context_alloc / astcenc_compress_image / astcenc_context_free).

    progress: optional callable(float), the config's progress_callback. compress_image calls it from the thread that runs
    the pass while blocks complete, and exactly once with 100.0 when the payload is in place (not after cancel()); it may
    call cancel(). parent: another Context whose tables this one shares (astcenc_context_alloc's parent argument); the
    config then comes from the parent."""

    def __init__(self, config=None, thread_count=1, progress=None, parent=None):
        self.handle = None
        self._progress = None
        if parent is not None:
            config = parent.config
        cfg = Config.from_buffer_copy(config)
        if progress is not None:
            # the trampoline must outlive every call that can reach it: it is kept with the context
            self._progress = PROGRESS_CALLBACK(lambda value: progress(float(value)))
            cfg.progress_callback = C.cast(self._progress, C.c_void_p)
        self.config = cfg
        self.thread_count = thread_count
        handle = C.c_void_p()
        if parent is not None:
            err = lib().astcenc_context_alloc(None, thread_count, C.byref(handle), parent.handle)
        else:
            err = lib().astcenc_context_alloc(C.byref(cfg), thread_count, C.byref(handle), None)
        if err:
            raise AstcencError(err, "astcenc_context_alloc")
        self.handle = handle

    def cancel(self):
        """astcenc_compress_cancel: a running compress_image stops handing out blocks and returns without writing its output;
        safe from any thread and from inside the progress callback."""
        err = lib().astcenc_compress_cancel(self.handle)
        if err:
            raise AstcencError(err, "astcenc_compress_cancel")

    def reset(self):
        """astcenc_compress_reset: ready for the next image (clears a cancel)."""
        err = lib().astcenc_compress_reset(self.handle)
        if err:
            raise AstcencError(err, "astcenc_compress_reset")

    def close(self):
        if self.handle:
            lib().astcenc_context_free(self.handle)
            self.handle = None

    __del__ = close

    def blocks(self, dim_x, dim_y):
        bx, by = self.config.block_x, self.config.block_y
        return (dim_x + bx - 1) // bx, (dim_y + by - 1) // by

    def compress_image(self, img, swizzle=(0, 1, 2, 3), out=None, thread_index=0):
        """Host-pointer path: img is a (H, W, 4) or (D, H, W, 4) numpy array of uint8 / float16 / float32."""
        img, slices, image, nbytes = self._image(img)
        sw = Swizzle(*swizzle)
        if out is None:
            out = np.empty(nbytes, dtype=np.uint8)
        err = lib().astcenc_compress_image(self.handle, C.byref(image), C.byref(sw), out.ctypes.data, out.nbytes, thread_index)
        if err:
            raise AstcencError(err, "astcenc_compress_image")
        return out

    def decompress_image(self, blocks, dim_x, dim_y, dtype=np.uint8, swizzle=(0, 1, 2, 3), dim_z=1, thread_index=0):
        """astcenc_decompress_image: 16-byte blocks -> (H, W, 4) (or (D, H, W, 4)) array of uint8 / float16 / float32."""
        blocks = np.ascontiguousarray(blocks, dtype=np.uint8)
        out = np.zeros((dim_z, dim_y, dim_x, 4), dtype=dtype)
        slices = (C.c_void_p * dim_z)(*[out[z].ctypes.data for z in range(dim_z)])
        image = Image(dim_x, dim_y, dim_z, _DTYPES[np.dtype(dtype)], slices)
        sw = Swizzle(*swizzle)
        err = lib().astcenc_decompress_image(self.handle, blocks.ctypes.data, blocks.nbytes, C.byref(image), C.byref(sw), thread_index)
        if err:
            raise AstcencError(err, "astcenc_decompress_image")
        return out[0] if dim_z == 1 else out

    def compress_device(self, d_pixels_ptr, data_type, dim_x, dim_y, d_out_ptr, block_row0=0, block_rows=None, swizzle=(0, 1, 2, 3), stream=0):
        """Device-resident path (astcenc_b200_compress_device): raw device pointers, enqueued on `stream`, no sync."""
        nbx, nby = self.blocks(dim_x, dim_y)
        if block_rows is None:
            block_rows = nby - block_row0
        sw = Swizzle(*swizzle)
        err = lib().astcenc_b200_compress_device(self.handle, C.c_void_p(d_pixels_ptr), data_type, dim_x, dim_y, C.byref(sw), block_row0, block_rows,
                                                 C.c_void_p(d_out_ptr), C.c_void_p(stream))
        if err:
            raise AstcencError(err, "astcenc_b200_compress_device")

    def compress_device_blocks(self, d_pixels_ptr, data_type, dim_x, dim_y, dim_z, indices, d_payload_ptr, swizzle=(0, 1, 2, 3), stream=0):
        """Block-list path (astcenc_b200_compress_device_blocks): recompress the listed blocks of a device-resident image into its
        device-resident payload, in place. indices: any integer array-like of block positions in payload order (z, y, x);
        enqueued on `stream`, no sync."""
        idx = np.asarray(indices).reshape(-1)
        if idx.size and (idx.min() < 0 or idx.max() > 0xFFFFFFFF):
            raise AstcencError(ERR_BAD_PARAM, "astcenc_b200_compress_device_blocks")      # (no position the C interface could take)
        idx = np.ascontiguousarray(idx, dtype=np.uint32)
        sw = Swizzle(*swizzle)
        err = lib().astcenc_b200_compress_device_blocks(self.handle, C.c_void_p(d_pixels_ptr), data_type, dim_x, dim_y, dim_z, C.byref(sw),
                                                        idx.ctypes.data if idx.size else None, idx.size, C.c_void_p(d_payload_ptr), C.c_void_p(stream))
        if err:
            raise AstcencError(err, "astcenc_b200_compress_device_blocks")

    def compress_device_images(self, images, data_type, swizzle=(0, 1, 2, 3), stream=0):
        """Many device-resident images in shared passes (astcenc_b200_compress_device_images). images: a sequence of
        (d_pixels_ptr, dim_x, dim_y, dim_z, d_payload_ptr); every payload receives its image's whole payload, the bytes
        compress_image gives for that image. Enqueued on `stream`, no sync."""
        n = len(images)
        table = (DeviceImage * n)(*[DeviceImage(C.c_void_p(p), x, y, z, C.c_void_p(q)) for p, x, y, z, q in images])
        sw = Swizzle(*swizzle)
        err = lib().astcenc_b200_compress_device_images(self.handle, table if n else None, n, data_type, C.byref(sw), C.c_void_p(stream))
        if err:
            raise AstcencError(err, "astcenc_b200_compress_device_images")

    def compress_images(self, arrays, swizzle=(0, 1, 2, 3)):
        """Host-pointer twin (astcenc_b200_compress_images): (H, W, 4) / (D, H, W, 4) numpy arrays of one dtype -> their payloads
        (uint8 arrays), compressed in shared passes."""
        n = len(arrays)
        prepared = [self._image(a) for a in arrays]
        ptrs = (C.POINTER(Image) * n)(*[C.pointer(p[2]) for p in prepared])
        outs = [np.empty(p[3], dtype=np.uint8) for p in prepared]
        optr = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
        lens = (C.c_size_t * n)(*[o.nbytes for o in outs])
        sw = Swizzle(*swizzle)
        err = lib().astcenc_b200_compress_images(self.handle, ptrs, n, C.byref(sw), optr, lens)
        if err:
            raise AstcencError(err, "astcenc_b200_compress_images")
        return outs

    def decompress_device_images(self, images, data_type, swizzle=(0, 1, 2, 3), stream=0):
        """Many device-resident payloads into device images in one launch (astcenc_b200_decompress_device_images). images: a
        sequence of (d_payload_ptr, d_image_ptr, dim_x, dim_y, dim_z); every image receives the texels decompress_image gives
        for its payload alone. Enqueued on `stream`, no sync; works on decompress-only contexts."""
        n = len(images)
        table = (DeviceDecodeImage * n)(*[DeviceDecodeImage(C.c_void_p(p), C.c_void_p(d), x, y, z) for p, d, x, y, z in images])
        sw = Swizzle(*swizzle) if swizzle is not None else None
        err = lib().astcenc_b200_decompress_device_images(self.handle, table if n else None, n, data_type, C.byref(sw) if sw is not None else None,
                                                          C.c_void_p(stream))
        if err:
            raise AstcencError(err, "astcenc_b200_decompress_device_images")

    def launch_count(self):
        return int(lib().astcenc_b200_launch_count(self.handle))

    # ---- multi-GPU (one process per GPU; include/astcenc.h "Multi-GPU sharding") ----
    def comm_init(self, rank, world, unique_id=None):
        self.rank, self.world = rank, world
        buf = (C.c_uint8 * COMM_ID_BYTES).from_buffer_copy(unique_id) if unique_id is not None else None
        err = lib().astcenc_b200_comm_init(self.handle, rank, world, buf, COMM_ID_BYTES if buf is not None else 0)
        if err:
            raise AstcencError(err, "astcenc_b200_comm_init")

    def comm_free(self):
        if self.handle:
            lib().astcenc_b200_comm_free(self.handle)

    def slab_rows(self, dim_y, rank, world):
        a = C.c_uint(); n = C.c_uint()
        err = lib().astcenc_b200_slab_rows(self.handle, dim_y, rank, world, C.byref(a), C.byref(n))
        if err:
            raise AstcencError(err, "astcenc_b200_slab_rows")
        return a.value, n.value

    def _image(self, img):
        """(H, W, 4) or (D, H, W, 4) numpy array -> (contiguous array, slice pointers, Image, payload bytes)."""
        img = np.ascontiguousarray(img)
        if img.ndim == 3:
            img = img[None]
        d, h, w = img.shape[:3]
        slices = (C.c_void_p * d)(*[img[z].ctypes.data for z in range(d)])
        nbx, nby = self.blocks(w, h)
        bz = max(1, self.config.block_z)      # 3D block sizes: blocks come out in (z, y, x) order
        return img, slices, Image(w, h, d, _DTYPES[img.dtype], slices), nbx * nby * ((d + bz - 1) // bz) * 16

    def compress_image_sharded(self, img, out=None, root=0, swizzle=(0, 1, 2, 3)):
        """Slab mode (collective): every rank passes the same (H, W, 4) image or (D, H, W, 4) volume / texture array; the root
        gets the whole payload in `out`."""
        img, slices, image, nbytes = self._image(img)
        sw = Swizzle(*swizzle)
        is_root = getattr(self, "rank", 0) == root
        if out is None and is_root:
            out = np.empty(nbytes, dtype=np.uint8)
        err = lib().astcenc_b200_compress_image_sharded(self.handle, C.byref(image), C.byref(sw), out.ctypes.data if out is not None else None,
                                                        out.nbytes if out is not None else 0, root)
        if err:
            raise AstcencError(err, "astcenc_b200_compress_image_sharded")
        return out

    def compress_batch(self, images, outs=None, root=0, swizzle=(0, 1, 2, 3)):
        """Batch mode (collective): images[i] ((H, W, 4) or (D, H, W, 4); None for images of other ranks) -> outs[i] on the root."""
        n = len(images)
        keep = []
        ptrs = (C.POINTER(Image) * n)()
        for i, im in enumerate(images):
            if im is None:
                continue
            im, slices, st, _ = self._image(im)
            keep.append((im, slices, st))
            ptrs[i] = C.pointer(st)
        sw = Swizzle(*swizzle)
        optr = None
        each = 0
        if outs is not None:
            optr = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
            each = outs[0].nbytes
        err = lib().astcenc_b200_compress_batch(self.handle, ptrs, n, C.byref(sw), optr, each, root)
        if err:
            raise AstcencError(err, "astcenc_b200_compress_batch")
        return outs

    def comm_last_timing(self):
        a = C.c_float(); b = C.c_float()
        lib().astcenc_b200_comm_last_timing(self.handle, C.byref(a), C.byref(b))
        return a.value, b.value

    def stage_timing(self, enable, fetch=False):
        """Enable / disable per-launch events; with fetch=True also return ({kernel: ms}, {kernel: launches}) of the last call."""
        names = ("setup", "refine", "prepare", "emit")
        if fetch:
            ms = (C.c_float * 4)(); n = (C.c_uint * 4)()
            lib().astcenc_b200_stage_timing(self.handle, 1 if enable else 0, ms, n)
            return {k: float(ms[i]) for i, k in enumerate(names)}, {k: int(n[i]) for i, k in enumerate(names)}
        lib().astcenc_b200_stage_timing(self.handle, 1 if enable else 0, None, None)
        return None

    def compute_error_metrics(self, img1, img2, hdr=False, normal=False, input_components=4, fstop_lo=-10, fstop_hi=10):
        """astcenc_b200_compute_error_metrics: the CLI's compute_error_metrics (astcenccli_error_metrics.cpp:109-413) on the
        device. img1 = original, img2 = decoded, numpy (H, W, 4) uint8 / float16 / float32. Returns a dict."""
        imgs = []
        for im in (img1, img2):
            im = np.ascontiguousarray(im)
            slices = (C.c_void_p * 1)(im.ctypes.data)
            imgs.append((im, slices, Image(im.shape[1], im.shape[0], 1, _DTYPES[im.dtype], slices)))
        out = ErrorMetrics()
        err = lib().astcenc_b200_compute_error_metrics(self.handle, int(hdr), int(normal), input_components, C.byref(imgs[0][2]), C.byref(imgs[1][2]),
                                                       fstop_lo, fstop_hi, C.byref(out))
        if err:
            raise AstcencError(err, "astcenc_b200_compute_error_metrics")
        d = {n: getattr(out, n) for n, _ in ErrorMetrics._fields_[:9]}
        d["sum_squared_error"] = list(out.sum_squared_error)
        return d

    def compute_error_metrics_device_images(self, images, hdr=False, normal=False, input_components=4, fstop_lo=-10, fstop_hi=10, stream=0):
        """Error metrics of many device-resident image pairs in one call (astcenc_b200_compute_error_metrics_device_images).
        images: a sequence of (d_original_ptr, d_decoded_ptr, original_type, decoded_type, dim_x, dim_y, dim_z, d_metrics_ptr,
        d_block_error_ptr or 0); every metrics pointer receives an ErrorMetrics, the figures compute_error_metrics gives for that
        pair alone, and every block_error pointer one float per block of the context's footprint. Enqueued on `stream`, no sync;
        works on decompress-only contexts. ErrorMetrics.from_buffer_copy reads a struct back."""
        n = len(images)
        table = _metrics_table(images)
        err = lib().astcenc_b200_compute_error_metrics_device_images(self.handle, int(hdr), int(normal), input_components, table if n else None, n,
                                                                     fstop_lo, fstop_hi, C.c_void_p(stream))
        if err:
            raise AstcencError(err, "astcenc_b200_compute_error_metrics_device_images")

    def compute_block_metric_device_images(self, images, block_metric, hdr=False, normal=False, input_components=4, fstop_lo=-10, fstop_hi=10,
                                           stream=0):
        """compute_error_metrics_device_images with maps of `block_metric` (astcenc_b200_compute_block_metric_device_images):
        BLOCK_SQUARED_ERROR, BLOCK_ALPHA_WEIGHTED_ERROR (each block's share of alpha_psnr's error sum), BLOCK_LOG2_ERROR (each
        block's share of log_rmse's), BLOCK_ANGULAR_ERROR (the sum of its texels' normal angles in degrees: the block's share of
        mean_angular_error times the pixel count) or BLOCK_WORST_ANGULAR_ERROR (its largest texel angle: the map's maximum is
        worst_angular_error). The angular maps read RGB whatever input_components is and need no `normal`. Same tuples, same
        figures; enqueued on `stream`, no sync."""
        n = len(images)
        table = _metrics_table(images)
        err = lib().astcenc_b200_compute_block_metric_device_images(self.handle, int(hdr), int(normal), input_components, block_metric, table if n else None,
                                                                    n, fstop_lo, fstop_hi, C.c_void_p(stream))
        if err:
            raise AstcencError(err, "astcenc_b200_compute_block_metric_device_images")

    def select_blocks(self, entries, stream=0):
        """Block selection from device maps (astcenc_b200_select_blocks). entries: a sequence of (d_map_ptr, block_count,
        threshold, capacity, d_indices_ptr, d_count_ptr); each keeps the min(capacity, candidates) largest values above its
        threshold, ties to the lower index, and writes their indices ascending and their number. Enqueued on `stream`, no sync;
        works on any context."""
        n = len(entries)
        table = (BlockSelection * n)(*[BlockSelection(C.c_void_p(m or None), b, t, c, C.c_void_p(i or None), C.c_void_p(k or None))
                                       for m, b, t, c, i, k in entries])
        err = lib().astcenc_b200_select_blocks(self.handle, table if n else None, n, C.c_void_p(stream))
        if err:
            raise AstcencError(err, "astcenc_b200_select_blocks")

    def select_blocks_pooled(self, pools, entries, stream=0):
        """Block selection under shared budgets (astcenc_b200_select_blocks_pooled). pools: a sequence of (entry_count,
        threshold, capacity), splitting `entries` into consecutive runs; entries: a sequence of (d_map_ptr, block_count,
        d_weight_ptr or 0, d_indices_ptr, d_count_ptr). Each pool keeps its min(capacity, candidates) largest products
        map[b] * *weight above its threshold, ties to the earlier entry, then the lower index; each entry receives its kept
        indices ascending and their number. Enqueued on `stream`, no sync; works on any context."""
        np_, n = len(pools), len(entries)
        ptab = (BlockPool * np_)(*[BlockPool(e, t, c) for e, t, c in pools])
        etab = (PooledSelection * n)(*[PooledSelection(C.c_void_p(m or None), b, C.c_void_p(w or None), C.c_void_p(i or None), C.c_void_p(k or None))
                                       for m, b, w, i, k in entries])
        err = lib().astcenc_b200_select_blocks_pooled(self.handle, ptab if np_ else None, np_, etab if n else None, n, C.c_void_p(stream))
        if err:
            raise AstcencError(err, "astcenc_b200_select_blocks_pooled")

    def total_block_maps(self, entries, rule, stream=0):
        """Map totals and gated selection weights (astcenc_b200_total_block_maps). entries: a sequence of (d_map_ptr, block_count,
        limit, d_total_ptr or 0, d_weight_ptr or 0); each total pointer receives the map's double total, in a fixed order set by
        block_count alone, and each weight pointer 0 unless total > limit and total > 0, else 1 (WEIGHT_ONE) or 1 / total
        (WEIGHT_INVERSE_TOTAL) as a float. Enqueued on `stream`, no sync; works on any context."""
        n = len(entries)
        table = (BlockMapTotal * n)(*[BlockMapTotal(C.c_void_p(m or None), b, lim, C.c_void_p(t or None), C.c_void_p(w or None))
                                      for m, b, lim, t, w in entries])
        err = lib().astcenc_b200_total_block_maps(self.handle, table if n else None, n, rule, C.c_void_p(stream))
        if err:
            raise AstcencError(err, "astcenc_b200_total_block_maps")

    def compress_device_block_lists(self, lists, data_type, swizzle=(0, 1, 2, 3), stream=0):
        """Recompress device-resident block lists (astcenc_b200_compress_device_block_lists). lists: a sequence of
        (d_pixels_ptr, dim_x, dim_y, dim_z, d_payload_ptr, d_indices_ptr, d_count_ptr, capacity); the first min(*count, capacity)
        indices in range are recompressed into the payload, in place. Enqueued on `stream`, no sync."""
        n = len(lists)
        table = (DeviceBlockList * n)(*[DeviceBlockList(C.c_void_p(p), x, y, z, C.c_void_p(q), C.c_void_p(i or None), C.c_void_p(k or None), c)
                                        for p, x, y, z, q, i, k, c in lists])
        sw = Swizzle(*swizzle)
        err = lib().astcenc_b200_compress_device_block_lists(self.handle, table if n else None, n, data_type, C.byref(sw), C.c_void_p(stream))
        if err:
            raise AstcencError(err, "astcenc_b200_compress_device_block_lists")

    def compress_device_block_lists_packed(self, lists, budget, data_type, swizzle=(0, 1, 2, 3), overflow=0, stream=0):
        """compress_device_block_lists at a cost set by `budget` (astcenc_b200_compress_device_block_lists_packed): the listed
        slots v_j = min(*count_j, capacity_j) of the same tuples take consecutive packed positions in entry order, and only those
        below `budget` are processed; `overflow` (a device uint32 pointer, or 0) receives max(sum of v_j - budget, 0). Stages
        min(budget, sum of capacities) slots. Enqueued on `stream`, no sync."""
        n = len(lists)
        table = (DeviceBlockList * n)(*[DeviceBlockList(C.c_void_p(p), x, y, z, C.c_void_p(q), C.c_void_p(i or None), C.c_void_p(k or None), c)
                                        for p, x, y, z, q, i, k, c in lists])
        sw = Swizzle(*swizzle)
        err = lib().astcenc_b200_compress_device_block_lists_packed(self.handle, table if n else None, n, budget, C.c_void_p(overflow or None), data_type,
                                                                    C.byref(sw), C.c_void_p(stream))
        if err:
            raise AstcencError(err, "astcenc_b200_compress_device_block_lists_packed")

    def decompress_device_block_lists(self, lists, data_type, swizzle=(0, 1, 2, 3), stream=0):
        """Decode device-resident block lists into device images (astcenc_b200_decompress_device_block_lists). lists: a sequence of
        (d_payload_ptr, d_image_ptr, dim_x, dim_y, dim_z, d_indices_ptr, d_count_ptr, capacity); for the first min(*count, capacity)
        indices in range, the block's texels receive what decompress_device_images writes there for the whole payload, and no other
        byte changes. Enqueued on `stream`, no sync; works on decompress-only contexts."""
        n = len(lists)
        table = (DeviceDecodeBlockList * n)(*[DeviceDecodeBlockList(C.c_void_p(p), C.c_void_p(d), x, y, z, C.c_void_p(i or None), C.c_void_p(k or None), c)
                                              for p, d, x, y, z, i, k, c in lists])
        sw = Swizzle(*swizzle) if swizzle is not None else None
        err = lib().astcenc_b200_decompress_device_block_lists(self.handle, table if n else None, n, data_type, C.byref(sw) if sw is not None else None,
                                                               C.c_void_p(stream))
        if err:
            raise AstcencError(err, "astcenc_b200_decompress_device_block_lists")

    def get_block_summaries_device_images(self, images, stream=0):
        """Summaries of every block of device-resident payloads (astcenc_b200_get_block_summaries_device_images). images: a
        sequence of (d_payload_ptr, dim_x, dim_y, dim_z, d_summaries_ptr); summaries[b] (16 bytes, BLOCK_SUMMARY_DTYPE) holds the
        fields get_block_info reports for block b, narrowed. Enqueued on `stream`, no sync; works on decompress-only contexts."""
        n = len(images)
        table = (DeviceBlockSummaryImage * n)(*[DeviceBlockSummaryImage(C.c_void_p(p), x, y, z, C.c_void_p(q)) for p, x, y, z, q in images])
        err = lib().astcenc_b200_get_block_summaries_device_images(self.handle, table if n else None, n, C.c_void_p(stream))
        if err:
            raise AstcencError(err, "astcenc_b200_get_block_summaries_device_images")

    def get_block_info_device_block_lists(self, lists, stream=0):
        """The full astcenc_block_info of the blocks of device lists (astcenc_b200_get_block_info_device_block_lists). lists: a
        sequence of (d_payload_ptr, dim_x, dim_y, dim_z, d_indices_ptr, d_count_ptr, capacity, d_infos_ptr); for each of the first
        min(*count, capacity) slots whose index is in range, infos[s] (BLOCK_INFO_BYTES bytes) receives what get_block_info writes
        for block indices[s]; other slots are left untouched. Enqueued on `stream`, no sync; works on decompress-only contexts."""
        n = len(lists)
        table = (DeviceBlockInfoList * n)(*[DeviceBlockInfoList(C.c_void_p(p), x, y, z, C.c_void_p(i or None), C.c_void_p(k or None), c, C.c_void_p(o or None))
                                            for p, x, y, z, i, k, c, o in lists])
        err = lib().astcenc_b200_get_block_info_device_block_lists(self.handle, table if n else None, n, C.c_void_p(stream))
        if err:
            raise AstcencError(err, "astcenc_b200_get_block_info_device_block_lists")

    def compute_block_errors_device_block_lists(self, lists, input_components=4, stream=0):
        """Refresh per-block error maps at device-resident block lists (astcenc_b200_compute_block_errors_device_block_lists).
        lists: a sequence of (d_original_ptr, d_decoded_ptr, original_type, decoded_type, dim_x, dim_y, dim_z, d_block_error_ptr,
        d_indices_ptr, d_count_ptr, capacity); each listed map value receives what compute_error_metrics_device_images writes for
        that block, and no other value changes. Enqueued on `stream`, no sync; works on decompress-only contexts."""
        n = len(lists)
        table = _block_error_list_table(lists)
        err = lib().astcenc_b200_compute_block_errors_device_block_lists(self.handle, input_components, table if n else None, n, C.c_void_p(stream))
        if err:
            raise AstcencError(err, "astcenc_b200_compute_block_errors_device_block_lists")

    def compute_block_metric_device_block_lists(self, lists, block_metric, input_components=4, stream=0):
        """compute_block_errors_device_block_lists for maps of `block_metric` (astcenc_b200_compute_block_metric_device_block_lists):
        each listed map value receives what compute_block_metric_device_images writes for that block with the same metric, and no
        other value changes; any metric compute_block_metric_device_images takes. Same tuples; enqueued on `stream`, no sync."""
        n = len(lists)
        table = _block_error_list_table(lists)
        err = lib().astcenc_b200_compute_block_metric_device_block_lists(self.handle, input_components, block_metric, table if n else None, n,
                                                                         C.c_void_p(stream))
        if err:
            raise AstcencError(err, "astcenc_b200_compute_block_metric_device_block_lists")

    def refine_device_block_lists(self, lists, data_type, decoded_type, block_metric, swizzle=(0, 1, 2, 3), decode_swizzle=(0, 1, 2, 3),
                                  input_components=4, stream=0):
        """Re-encode device-resident block lists and keep each new block only where it lowers the block's value in its map
        (astcenc_b200_refine_device_block_lists). lists: a sequence of (d_pixels_ptr, dim_x, dim_y, dim_z, d_payload_ptr,
        d_decoded_ptr or 0, d_block_error_ptr, d_indices_ptr, d_count_ptr, capacity). For the first min(*count, capacity) indices
        in range, the candidate (what compress_device_block_lists would write) is decoded by this context to decoded_type with
        decode_swizzle and measured in block_metric over input_components; where that value is below the map's, the payload
        bytes, the decoded texels and the map value are replaced. block_metric is any metric of compute_block_metric_device_images;
        for a normal map encoded with the rrrg swizzle, decode with decode_swizzle (0, 3, 6, 5), (R, A, Z, 1), and measure in
        BLOCK_ANGULAR_ERROR or BLOCK_WORST_ANGULAR_ERROR. Enqueued on `stream`, no sync."""
        n = len(lists)
        table = (DeviceRefineList * n)(*[DeviceRefineList(C.c_void_p(p), x, y, z, C.c_void_p(q), C.c_void_p(d or None), C.c_void_p(b or None),
                                                          C.c_void_p(i or None), C.c_void_p(k or None), c)
                                         for p, x, y, z, q, d, b, i, k, c in lists])
        sw = Swizzle(*swizzle)
        dsw = Swizzle(*decode_swizzle)
        err = lib().astcenc_b200_refine_device_block_lists(self.handle, table if n else None, n, data_type, C.byref(sw), decoded_type, C.byref(dsw),
                                                           input_components, block_metric, C.c_void_p(stream))
        if err:
            raise AstcencError(err, "astcenc_b200_refine_device_block_lists")

    def refine_device_block_lists_packed(self, lists, budget, data_type, decoded_type, block_metric, swizzle=(0, 1, 2, 3), decode_swizzle=(0, 1, 2, 3),
                                         input_components=4, overflow=0, stream=0):
        """refine_device_block_lists at a cost set by `budget` (astcenc_b200_refine_device_block_lists_packed): the same tuples,
        packed and truncated as in compress_device_block_lists_packed; `overflow` (a device uint32 pointer, or 0) receives
        max(sum of v_j - budget, 0). Enqueued on `stream`, no sync."""
        n = len(lists)
        table = (DeviceRefineList * n)(*[DeviceRefineList(C.c_void_p(p), x, y, z, C.c_void_p(q), C.c_void_p(d or None), C.c_void_p(b or None),
                                                          C.c_void_p(i or None), C.c_void_p(k or None), c)
                                         for p, x, y, z, q, d, b, i, k, c in lists])
        sw = Swizzle(*swizzle)
        dsw = Swizzle(*decode_swizzle)
        err = lib().astcenc_b200_refine_device_block_lists_packed(self.handle, table if n else None, n, budget, C.c_void_p(overflow or None), data_type,
                                                                  C.byref(sw), decoded_type, C.byref(dsw), input_components, block_metric, C.c_void_p(stream))
        if err:
            raise AstcencError(err, "astcenc_b200_refine_device_block_lists_packed")

    def last_timing(self):
        ms = C.c_float(); a = C.c_size_t(); b = C.c_size_t()
        lib().astcenc_b200_last_timing(self.handle, C.byref(ms), C.byref(a), C.byref(b))
        return ms.value, a.value, b.value


def _metrics_table(images):
    """The astcenc_b200_device_metrics_image array of (d_original_ptr, d_decoded_ptr, original_type, decoded_type, dim_x, dim_y,
    dim_z, d_metrics_ptr, d_block_error_ptr or 0) tuples."""
    return (DeviceMetricsImage * len(images))(*[DeviceMetricsImage(C.c_void_p(o), C.c_void_p(d), ot, dt, x, y, z, C.c_void_p(m), C.c_void_p(b or None))
                                                for o, d, ot, dt, x, y, z, m, b in images])


def _block_error_list_table(lists):
    """The astcenc_b200_device_block_error_list array of (d_original_ptr, d_decoded_ptr, original_type, decoded_type, dim_x, dim_y,
    dim_z, d_block_error_ptr, d_indices_ptr, d_count_ptr, capacity) tuples."""
    return (DeviceBlockErrorList * len(lists))(*[DeviceBlockErrorList(C.c_void_p(o), C.c_void_p(d), ot, dt, x, y, z, C.c_void_p(b or None),
                                                                      C.c_void_p(i or None), C.c_void_p(k or None), c)
                                                 for o, d, ot, dt, x, y, z, b, i, k, c in lists])


def store_cimage(filename, blocks, dim_x, dim_y, block_x, block_y, dim_z=1, block_z=1):
    """Write a .astc file (store_cimage, astcenccli_image_load_store.cpp:2691-2730): 16-byte header + the blocks."""
    data = np.ascontiguousarray(np.frombuffer(bytes(blocks), dtype=np.uint8) if not isinstance(blocks, np.ndarray) else blocks.view(np.uint8).reshape(-1))
    hdr = CImageHeader(block_x, block_y, block_z, dim_x, dim_y, dim_z)
    err = lib().astcenc_b200_store_cimage(os.fsencode(filename), C.byref(hdr), data.ctypes.data, data.nbytes)
    if err:
        raise AstcencError(err, "astcenc_b200_store_cimage")


def load_cimage(filename):
    """Read a .astc file (load_cimage, astcenccli_image_load_store.cpp:2599-2688). Returns (blocks uint8 array, header dict);
    corrupt files raise AstcencError like the reference tool refuses them."""
    hdr = CImageHeader()
    n = C.c_size_t()
    err = lib().astcenc_b200_load_cimage(os.fsencode(filename), C.byref(hdr), None, 0, C.byref(n))
    if err:
        raise AstcencError(err, "astcenc_b200_load_cimage")
    data = np.empty(n.value, dtype=np.uint8)
    err = lib().astcenc_b200_load_cimage(os.fsencode(filename), C.byref(hdr), data.ctypes.data, data.nbytes, C.byref(n))
    if err:
        raise AstcencError(err, "astcenc_b200_load_cimage")
    return data, {k: getattr(hdr, k) for k, _ in CImageHeader._fields_}


def store_ktx_cimage(filename, blocks, dim_x, dim_y, block_x, block_y, is_srgb=False, dim_z=1, block_z=1):
    """Write the blocks as a KTX 1 file (store_ktx_compressed_image, astcenccli_image_load_store.cpp:1396-1440)."""
    data = np.ascontiguousarray(np.frombuffer(bytes(blocks), dtype=np.uint8) if not isinstance(blocks, np.ndarray) else blocks.view(np.uint8).reshape(-1))
    hdr = CImageHeader(block_x, block_y, block_z, dim_x, dim_y, dim_z)
    err = lib().astcenc_b200_store_ktx_cimage(os.fsencode(filename), C.byref(hdr), int(is_srgb), data.ctypes.data, data.nbytes)
    if err:
        raise AstcencError(err, "astcenc_b200_store_ktx_cimage")


def load_ktx_cimage(filename):
    """Read an ASTC payload from a KTX 1 file (load_ktx_compressed_image, :1294-1385). Returns (blocks, header dict, is_srgb)."""
    hdr = CImageHeader()
    n = C.c_size_t()
    srgb = C.c_int()
    err = lib().astcenc_b200_load_ktx_cimage(os.fsencode(filename), C.byref(hdr), C.byref(srgb), None, 0, C.byref(n))
    if err:
        raise AstcencError(err, "astcenc_b200_load_ktx_cimage")
    data = np.empty(n.value, dtype=np.uint8)
    err = lib().astcenc_b200_load_ktx_cimage(os.fsencode(filename), C.byref(hdr), C.byref(srgb), data.ctypes.data, data.nbytes, C.byref(n))
    if err:
        raise AstcencError(err, "astcenc_b200_load_ktx_cimage")
    return data, {k: getattr(hdr, k) for k, _ in CImageHeader._fields_}, bool(srgb.value)


def slab_rows(blocks_y, rank, world):
    """Block-row slab [r0, r1) of `rank` among `world` ranks (SURVEY.md section 8e)."""
    r0 = (blocks_y * rank) // world
    r1 = (blocks_y * (rank + 1)) // world
    return r0, r1
