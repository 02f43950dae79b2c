"""CPU: the launch plan of a compressing context (astc-encoder_b200/csrc/astc_host_launch.h, plan_kernels), pinned.

astcenc_context_alloc takes every kernel's warps per CTA, grid and dynamic shared memory from plan_kernels, with the H100's
opt-in shared memory per block (232448 bytes) and SM count (132). The literals below were computed by the launch arithmetic as it
stood inside astcenc_context_alloc before it moved to plan_kernels; any change to them changes what the library launches.
DESIGN.md's 6x6 -medium plan is the second BASELINE row: set-up 15 warps (480 threads) on the general plan and 19 (608) on the
compact one-plane plan, refine 24 warps (768), prepare 2 x 12 warps per SM, 21456 bytes of decimation tables staged."""
import ctypes as C

import pytest

from astc_ref import *  # noqa: F401,F403

S = FLG_SELF_DECOMPRESS_ONLY
H100_SMEM, H100_SMS = 232448, 132
NOT_IMPLEMENTED = 10

FIELDS = ["status", "warps_per_cta", "grid", "smem_bytes", "lockstep", "driver", "warps_setup", "warps_setup_1p", "warps_small", "refine_ctas",
          "smem_setup", "smem_setup_1p", "smem_refine", "setup_stage_bytes", "refine_stage_bytes", "max_waves"]


class Knobs(C.Structure):
    """struct Knobs (astc_host_launch.h), field for field."""
    _fields_ = [("batch_blocks", C.c_size_t), ("sync_mask", C.c_uint), ("sync_mask_tail", C.c_uint), ("coherence_probe", C.c_int),
                ("stage_print", C.c_int), ("upload_bands", C.c_int), ("pipes", C.c_int), ("ctas_per_sm", C.c_int), ("refine_ctas", C.c_int),
                ("driver", C.c_int), ("lockstep", C.c_int), ("stage_refine", C.c_int), ("stage_setup", C.c_int), ("warps", C.c_int),
                ("warps_setup", C.c_int), ("warps_refine", C.c_int), ("warps_setup_1p", C.c_int)]


DEFAULT_KNOBS = dict(batch_blocks=1 << 20, sync_mask=8, sync_mask_tail=8, coherence_probe=0, stage_print=0, upload_bands=4, pipes=1, ctas_per_sm=1,
                     refine_ctas=1, driver=0, lockstep=1, stage_refine=0, stage_setup=-1, warps=-1, warps_setup=-1, warps_refine=-1, warps_setup_1p=-1)


class KernelPlan(C.Structure):
    """struct KernelPlan (astc_host_launch.h), field for field."""
    _fields_ = [("warps_per_cta", C.c_int), ("grid", C.c_int), ("smem_bytes", C.c_size_t), ("lockstep", C.c_int), ("driver", C.c_int),
                ("warps_setup", C.c_int), ("warps_setup_1p", C.c_int), ("warps_small", C.c_int), ("refine_ctas", C.c_int),
                ("smem_setup", C.c_size_t), ("smem_setup_1p", C.c_size_t), ("smem_refine", C.c_size_t), ("setup_stage_bytes", C.c_uint32),
                ("refine_stage_bytes", C.c_uint32), ("max_waves", C.c_int)]


def plan(hostsim, profile, bx, by, bz, quality, flags=S, smem=H100_SMEM, sms=H100_SMS, **knobs):
    hostsim.hostsim_kernel_plan.argtypes = [C.c_int, C.c_uint, C.c_uint, C.c_uint, C.c_float, C.c_uint, C.c_size_t, C.c_int, C.POINTER(Knobs),
                                            C.POINTER(KernelPlan)]
    hostsim.hostsim_kernel_plan.restype = C.c_int
    k = Knobs(**dict(DEFAULT_KNOBS, **knobs))
    p = KernelPlan()
    status = hostsim.hostsim_kernel_plan(profile, bx, by, bz, quality, flags, smem, sms, C.byref(k), C.byref(p))
    if status != 0:
        return (status,)
    return (status,) + tuple(getattr(p, f) for f in FIELDS[1:])


# (profile, block, quality, knobs, smem_limit) -> the plan, as FIELDS
CASES = [
    # BASELINE.json configs 0-3
    ((PRF_LDR, (4, 4, 1), PRE_FAST, {}, H100_SMEM), (0, 16, 132, 129280, 1, 0, 20, 0, 24, 1, 157840, 152720, 171008, 464, 0, 10)),
    ((PRF_LDR, (6, 6, 1), PRE_MEDIUM, {}, H100_SMEM), (0, 16, 132, 226048, 1, 0, 15, 19, 24, 1, 231872, 229968, 178688, 21456, 0, 10)),
    ((PRF_LDR, (8, 8, 1), PRE_THOROUGH, {}, H100_SMEM), (0, 9, 132, 224240, 1, 0, 9, 12, 24, 1, 223088, 220352, 205952, 0, 0, 13)),
    ((PRF_HDR, (6, 6, 1), PRE_MEDIUM, {}, H100_SMEM), (0, 16, 132, 226048, 1, 0, 15, 19, 24, 1, 231872, 229968, 178688, 21456, 0, 10)),
    # every other 2D block size at -fast and -thorough
    ((PRF_LDR, (5, 4, 1), PRE_FAST, {}, H100_SMEM), (0, 16, 132, 139776, 1, 0, 20, 0, 24, 1, 172272, 161072, 172544, 1776, 0, 10)),
    ((PRF_LDR, (5, 5, 1), PRE_FAST, {}, H100_SMEM), (0, 16, 132, 154112, 1, 0, 20, 0, 24, 1, 192112, 173552, 175616, 3696, 0, 10)),
    ((PRF_LDR, (6, 5, 1), PRE_FAST, {}, H100_SMEM), (0, 16, 132, 170752, 1, 0, 20, 0, 24, 1, 216320, 188480, 177152, 7104, 0, 10)),
    ((PRF_LDR, (6, 6, 1), PRE_FAST, {}, H100_SMEM), (0, 16, 132, 192256, 1, 0, 18, 20, 24, 1, 226128, 210032, 178688, 12976, 0, 10)),
    ((PRF_LDR, (8, 5, 1), PRE_FAST, {}, H100_SMEM), (0, 16, 132, 210432, 1, 0, 16, 20, 24, 1, 226224, 228976, 180224, 17840, 0, 10)),
    ((PRF_LDR, (8, 6, 1), PRE_FAST, {}, H100_SMEM), (0, 15, 132, 230336, 1, 0, 15, 19, 24, 1, 228416, 228272, 183296, 0, 0, 10)),
    ((PRF_LDR, (8, 8, 1), PRE_FAST, {}, H100_SMEM), (0, 11, 132, 216800, 1, 0, 11, 15, 24, 1, 215392, 228656, 195584, 0, 0, 8)),
    ((PRF_LDR, (10, 5, 1), PRE_FAST, {}, H100_SMEM), (0, 14, 132, 227520, 1, 0, 14, 18, 24, 1, 225728, 226688, 184832, 0, 0, 10)),
    ((PRF_LDR, (10, 6, 1), PRE_FAST, {}, H100_SMEM), (0, 12, 132, 230144, 1, 0, 12, 15, 24, 1, 228608, 221216, 192128, 0, 0, 10)),
    ((PRF_LDR, (10, 8, 1), PRE_FAST, {}, H100_SMEM), (0, 9, 132, 210128, 1, 0, 10, 12, 24, 1, 231456, 217856, 210944, 0, 0, 8)),
    ((PRF_LDR, (10, 10, 1), PRE_FAST, {}, H100_SMEM), (0, 8, 132, 225536, 1, 0, 8, 10, 24, 1, 224512, 218016, 231296, 0, 0, 8)),
    ((PRF_LDR, (12, 10, 1), PRE_FAST, {}, H100_SMEM), (0, 7, 132, 210160, 1, 0, 7, 9, 23, 1, 209264, 210992, 232352, 0, 0, 8)),
    ((PRF_LDR, (12, 12, 1), PRE_FAST, {}, H100_SMEM), (0, 6, 132, 200480, 1, 0, 7, 8, 21, 1, 231888, 208512, 226640, 0, 0, 8)),
    ((PRF_LDR, (4, 4, 1), PRE_THOROUGH, {}, H100_SMEM), (0, 16, 132, 148992, 1, 0, 20, 0, 24, 1, 184816, 167536, 171008, 2800, 0, 13)),
    ((PRF_LDR, (5, 4, 1), PRE_THOROUGH, {}, H100_SMEM), (0, 16, 132, 164864, 1, 0, 20, 0, 24, 1, 207136, 180576, 172544, 5280, 0, 13)),
    ((PRF_LDR, (5, 5, 1), PRE_THOROUGH, {}, H100_SMEM), (0, 16, 132, 188672, 1, 0, 19, 20, 24, 1, 229856, 202064, 175616, 9488, 0, 13)),
    ((PRF_LDR, (6, 5, 1), PRE_THOROUGH, {}, H100_SMEM), (0, 16, 132, 211456, 1, 0, 16, 20, 24, 1, 224464, 223632, 177152, 15056, 0, 13)),
    ((PRF_LDR, (6, 6, 1), PRE_THOROUGH, {}, H100_SMEM), (0, 15, 132, 227216, 1, 0, 15, 20, 24, 1, 225296, 230656, 178688, 0, 0, 13)),
    ((PRF_LDR, (8, 5, 1), PRE_THOROUGH, {}, H100_SMEM), (0, 14, 132, 228640, 1, 0, 14, 18, 24, 1, 226848, 220928, 180224, 0, 0, 13)),
    ((PRF_LDR, (8, 6, 1), PRE_THOROUGH, {}, H100_SMEM), (0, 12, 132, 227072, 1, 0, 12, 16, 24, 1, 225536, 223488, 183680, 0, 0, 13)),
    ((PRF_LDR, (10, 5, 1), PRE_THOROUGH, {}, H100_SMEM), (0, 11, 132, 215568, 1, 0, 11, 16, 24, 1, 214160, 231424, 186752, 0, 0, 13)),
    ((PRF_LDR, (10, 6, 1), PRE_THOROUGH, {}, H100_SMEM), (0, 9, 132, 210272, 1, 0, 10, 13, 24, 1, 231616, 223600, 199808, 0, 0, 13)),
    ((PRF_LDR, (10, 8, 1), PRE_THOROUGH, {}, H100_SMEM), (0, 7, 132, 209040, 1, 0, 7, 10, 24, 1, 208144, 220096, 225152, 0, 0, 13)),
    ((PRF_LDR, (10, 10, 1), PRE_THOROUGH, {}, H100_SMEM), (0, 6, 132, 208352, 1, 0, 6, 9, 22, 1, 207584, 230576, 225088, 0, 0, 13)),
    ((PRF_LDR, (12, 10, 1), PRE_THOROUGH, {}, H100_SMEM), (0, 6, 132, 230048, 1, 0, 6, 8, 21, 1, 229280, 227712, 229664, 0, 0, 13)),
    ((PRF_LDR, (12, 12, 1), PRE_THOROUGH, {}, H100_SMEM), (0, 5, 132, 211376, 1, 0, 5, 7, 19, 1, 210736, 219904, 222128, 0, 0, 13)),
    # 3D block sizes
    ((PRF_LDR, (3, 3, 3), PRE_MEDIUM, {}, H100_SMEM), (0, 16, 132, 171520, 1, 0, 20, 0, 24, 1, 216320, 187840, 175616, 6144, 0, 10)),
    ((PRF_LDR, (4, 4, 4), PRE_MEDIUM, {}, H100_SMEM), (0, 12, 132, 224384, 1, 0, 12, 16, 24, 1, 222848, 226816, 189440, 0, 0, 10)),
    ((PRF_LDR, (6, 6, 6), PRE_MEDIUM, {}, H100_SMEM), (0, 5, 132, 223296, 1, 0, 5, 6, 18, 1, 222656, 205472, 231488, 0, 0, 10)),
    # a smaller shared window: 12x12 -thorough fits one warp at 47600 bytes and nothing at 47599; 4x4 -fast at 48 KB
    ((PRF_LDR, (12, 12, 1), PRE_THOROUGH, {}, 47600), (0, 1, 132, 47600, 1, 0, 1, 0, 4, 1, 47472, 37120, 47168, 0, 0, 13)),
    ((PRF_LDR, (12, 12, 1), PRE_THOROUGH, {}, 47599), (NOT_IMPLEMENTED,)),
    ((PRF_LDR, (4, 4, 1), PRE_FAST, {}, 49152), (0, 5, 132, 44976, 1, 0, 5, 0, 6, 1, 44800, 43520, 43136, 464, 0, 10)),
    # the knob overrides the GPU tests use
    ((PRF_LDR, (6, 6, 1), PRE_MEDIUM, dict(stage_setup=0), H100_SMEM), (0, 16, 132, 226048, 1, 0, 16, 20, 24, 1, 224000, 219136, 178688, 0, 0, 10)),
    ((PRF_LDR, (6, 6, 1), PRE_MEDIUM, dict(stage_setup=1), H100_SMEM), (0, 16, 132, 226048, 1, 0, 15, 19, 24, 1, 231872, 229968, 178688, 21456, 0, 10)),
    ((PRF_LDR, (6, 6, 1), PRE_MEDIUM, dict(stage_refine=1), H100_SMEM), (0, 16, 132, 226048, 1, 0, 15, 19, 24, 1, 231872, 229968, 208848, 21456, 30160, 10)),
    ((PRF_LDR, (6, 6, 1), PRE_MEDIUM, dict(warps_setup_1p=0), H100_SMEM), (0, 16, 132, 226048, 1, 0, 15, 0, 24, 1, 231872, 28112, 178688, 21456, 0, 10)),
    ((PRF_LDR, (6, 6, 1), PRE_MEDIUM, dict(refine_ctas=2), H100_SMEM), (0, 16, 132, 226048, 1, 0, 15, 19, 15, 2, 231872, 229968, 111872, 21456, 0, 10)),
]


def _id(case):
    (prof, fp, q, knobs, smem), _ = case
    return "p%d-%s-q%g-%s-%d" % (prof, "x".join(map(str, fp)), q, "-".join("%s=%d" % kv for kv in sorted(knobs.items())) or "default", smem)


@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
def test_kernel_plan_is_pinned(hostsim, case):
    (prof, (bx, by, bz), q, knobs, smem), want = case
    assert plan(hostsim, prof, bx, by, bz, q, smem=smem, **knobs) == want
