"""GPU: the error code every entry point returns for each class of bad argument, and for pairs of bad arguments, which pin the
order of its checks. A refused call enqueues nothing: astcenc_b200_launch_count does not move.

Each entry point has its own order and its own codes (astcenc_compress_image and astcenc_decompress_image follow the
reference's); this file records them as they are."""
import ctypes as C

import numpy as np
import pytest

from astc_ref import *  # noqa: F401,F403

pytestmark = pytest.mark.gpu
S = FLG_SELF_DECOMPRESS_ONLY
OK, OOM, PARAM, SWZ, CTX, NI = 0, 1, 3, 7, 9, 10
HUGE = 0xFFFFFFFF
W, H = 8, 8                      # 2 x 2 blocks of 6x6: 64 payload bytes per slice


@pytest.fixture(scope="module")
def env(pkg):
    import torch
    assert torch.cuda.is_available(), "these tests need a CUDA device"
    ctxs = {
        "plain": pkg.Context(pkg.config_init(PRF_LDR, 6, 6, PRE_FAST, S)),
        "radius": pkg.Context(pkg.config_init(PRF_LDR, 6, 6, PRE_FAST, S, a_scale_radius=2)),
        "dec_only": pkg.Context(pkg.config_init(PRF_LDR, 6, 6, PRE_FAST, pkg.FLG_DECOMPRESS_ONLY)),
    }
    host = np.zeros((2, H, W, 4), np.uint8)
    dev = torch.zeros(2 * H * W * 4, dtype=torch.uint8, device="cuda")
    dev_out = torch.zeros(2 * 4 * 16, dtype=torch.uint8, device="cuda")
    yield pkg, ctxs, host, dev, dev_out
    for c in ctxs.values():
        c.close()


def _image(pkg, host, dim_x=W, dim_y=H, dim_z=1, data_type=TYPE_U8, data=True):
    slices = (C.c_void_p * 2)(host[0].ctypes.data, host[1].ctypes.data)
    image = pkg.Image(dim_x, dim_y, dim_z, data_type, slices if data else None)
    return image, slices


def compress_image(env, ctx="plain", swizzle=(0, 1, 2, 3), out_len=64, thread_index=0, **img):
    pkg, ctxs, host, _, _ = env
    image, keep = _image(pkg, host, **img)
    out = np.zeros(256, np.uint8)
    return pkg.lib().astcenc_compress_image(ctxs[ctx].handle, C.byref(image), C.byref(pkg.Swizzle(*swizzle)), out.ctypes.data, out_len, thread_index)


def decompress_image(env, ctx="plain", swizzle=(0, 1, 2, 3), data_len=64, thread_index=0, **img):
    pkg, ctxs, host, _, _ = env
    image, keep = _image(pkg, host, **img)
    data = np.zeros(256, np.uint8)
    return pkg.lib().astcenc_decompress_image(ctxs[ctx].handle, data.ctypes.data, data_len, C.byref(image), C.byref(pkg.Swizzle(*swizzle)), thread_index)


def compress_device(env, ctx="plain", swizzle=(0, 1, 2, 3), pixels=True, out=True, dim_x=W, dim_y=H, data_type=TYPE_U8, row0=0, rows=2):
    pkg, ctxs, _, dev, dev_out = env
    return pkg.lib().astcenc_b200_compress_device(ctxs[ctx].handle, C.c_void_p(dev.data_ptr() if pixels else 0), data_type, dim_x, dim_y,
                                                  C.byref(pkg.Swizzle(*swizzle)), row0, rows, C.c_void_p(dev_out.data_ptr() if out else 0), None)


def compress_device_blocks(env, ctx="plain", swizzle=(0, 1, 2, 3), pixels=True, payload=True, dim_x=W, dim_y=H, dim_z=1, data_type=TYPE_U8,
                           indices=(0, 3), null_indices=False):
    pkg, ctxs, _, dev, dev_out = env
    idx = np.asarray(indices, np.uint32)
    sw = None if swizzle is None else C.byref(pkg.Swizzle(*swizzle))
    return pkg.lib().astcenc_b200_compress_device_blocks(ctxs[ctx].handle, C.c_void_p(dev.data_ptr() if pixels else 0), data_type, dim_x, dim_y, dim_z, sw,
                                                         None if null_indices else idx.ctypes.data, len(idx),
                                                         C.c_void_p(dev_out.data_ptr() if payload else 0), None)


def compress_sharded(env, ctx="plain", swizzle=(0, 1, 2, 3), out_len=64, null_out=False, null_image=False, root=0, **img):
    pkg, ctxs, host, _, _ = env
    image, keep = _image(pkg, host, **img)
    out = np.zeros(256, np.uint8)
    sw = None if swizzle is None else C.byref(pkg.Swizzle(*swizzle))
    return pkg.lib().astcenc_b200_compress_image_sharded(ctxs[ctx].handle, None if null_image else C.byref(image), sw, None if null_out else out.ctypes.data,
                                                         out_len, root)


def compress_batch(env, ctx="plain", swizzle=(0, 1, 2, 3), out_len=64, count=2, null_out=False, null_images=False, root=0, second=None, **img):
    pkg, ctxs, host, _, _ = env
    image, keep = _image(pkg, host, **img)
    other, keep2 = _image(pkg, host, **(second if second is not None else img))
    ptrs = (C.POINTER(pkg.Image) * 2)(C.pointer(image), C.pointer(other))
    outs = [np.zeros(256, np.uint8) for _ in range(2)]
    optr = (C.c_void_p * 2)(*[o.ctypes.data for o in outs])
    sw = None if swizzle is None else C.byref(pkg.Swizzle(*swizzle))
    return pkg.lib().astcenc_b200_compress_batch(ctxs[ctx].handle, None if null_images else ptrs, count, sw, None if null_out else optr, out_len, root)


CASES = [
    # astcenc_compress_image: context, swizzle, thread_index, dimensions, block count, output length, alpha-scale on an array
    (compress_image, {}, OK),
    (compress_image, dict(ctx="dec_only"), CTX),
    (compress_image, dict(swizzle=(0, 1, 2, 6)), SWZ),
    (compress_image, dict(thread_index=1), PARAM),
    (compress_image, dict(dim_x=0), PARAM),
    (compress_image, dict(dim_z=0), PARAM),
    (compress_image, dict(dim_x=HUGE, dim_y=HUGE, dim_z=HUGE), PARAM),
    (compress_image, dict(out_len=63), OOM),
    (compress_image, dict(ctx="radius", dim_z=2, out_len=128), NI),
    (compress_image, dict(ctx="dec_only", swizzle=(0, 1, 2, 6)), CTX),
    (compress_image, dict(swizzle=(0, 1, 2, 6), thread_index=1), SWZ),
    (compress_image, dict(swizzle=(0, 1, 2, 6), dim_x=0), SWZ),
    (compress_image, dict(dim_x=HUGE, dim_y=HUGE, dim_z=HUGE, out_len=0), PARAM),
    (compress_image, dict(ctx="radius", dim_z=2, out_len=64), OOM),
    (compress_image, dict(ctx="radius", dim_z=2, out_len=128, swizzle=(9, 1, 2, 3)), SWZ),
    # astcenc_decompress_image: thread_index, swizzle (Z allowed), dimensions, input length; any context decodes
    (decompress_image, {}, OK),
    (decompress_image, dict(ctx="dec_only"), OK),
    (decompress_image, dict(swizzle=(0, 1, 2, 6)), OK),
    (decompress_image, dict(thread_index=1), PARAM),
    (decompress_image, dict(swizzle=(0, 1, 2, 7)), SWZ),
    (decompress_image, dict(dim_y=0), PARAM),
    (decompress_image, dict(dim_x=HUGE, dim_y=HUGE, dim_z=HUGE), PARAM),
    (decompress_image, dict(data_len=63), OOM),
    (decompress_image, dict(thread_index=1, swizzle=(0, 1, 2, 7)), PARAM),
    (decompress_image, dict(swizzle=(0, 1, 2, 7), dim_y=0), SWZ),
    (decompress_image, dict(dim_y=0, data_len=0), PARAM),
    # astcenc_b200_compress_device: context, swizzle, dimensions and pointers, block-row range
    (compress_device, {}, OK),
    (compress_device, dict(rows=0), OK),
    (compress_device, dict(ctx="dec_only"), CTX),
    (compress_device, dict(swizzle=(0, 1, 2, 6)), SWZ),
    (compress_device, dict(pixels=False), PARAM),
    (compress_device, dict(out=False), PARAM),
    (compress_device, dict(dim_x=0), PARAM),
    (compress_device, dict(row0=1, rows=2), PARAM),
    (compress_device, dict(dim_x=HUGE, dim_y=HUGE, row0=HUGE, rows=HUGE), PARAM),
    (compress_device, dict(ctx="dec_only", swizzle=(0, 1, 2, 6)), CTX),
    (compress_device, dict(swizzle=(0, 1, 2, 6), pixels=False), SWZ),
    (compress_device, dict(dim_y=0, rows=0), PARAM),
    # astcenc_b200_compress_device_blocks: context, swizzle pointer, swizzle, dimensions and pointers, data type, alpha-scale on an
    # array, block count, the list
    (compress_device_blocks, {}, OK),
    (compress_device_blocks, dict(indices=()), OK),
    (compress_device_blocks, dict(indices=(), null_indices=True), OK),
    (compress_device_blocks, dict(ctx="dec_only"), CTX),
    (compress_device_blocks, dict(swizzle=None), PARAM),
    (compress_device_blocks, dict(swizzle=(0, 1, 2, 6)), SWZ),
    (compress_device_blocks, dict(pixels=False), PARAM),
    (compress_device_blocks, dict(payload=False), PARAM),
    (compress_device_blocks, dict(null_indices=True), PARAM),
    (compress_device_blocks, dict(dim_z=0), PARAM),
    (compress_device_blocks, dict(data_type=3), PARAM),
    (compress_device_blocks, dict(ctx="radius", dim_z=2), NI),
    (compress_device_blocks, dict(dim_x=HUGE, dim_y=HUGE, dim_z=HUGE), PARAM),
    (compress_device_blocks, dict(indices=(0, 4)), PARAM),
    (compress_device_blocks, dict(ctx="dec_only", swizzle=None), CTX),
    (compress_device_blocks, dict(swizzle=None, pixels=False), PARAM),
    (compress_device_blocks, dict(swizzle=(0, 1, 2, 6), pixels=False), SWZ),
    (compress_device_blocks, dict(swizzle=(0, 1, 2, 6), data_type=3), SWZ),
    (compress_device_blocks, dict(ctx="radius", dim_z=2, data_type=3), PARAM),
    (compress_device_blocks, dict(ctx="radius", dim_x=HUGE, dim_y=HUGE, dim_z=HUGE), NI),
    (compress_device_blocks, dict(ctx="radius", dim_z=2, indices=(10 ** 6,)), NI),
    # astcenc_b200_compress_image_sharded (world 1): pointers, context, swizzle, dimensions, data type, alpha-scale on an array,
    # root, output
    (compress_sharded, {}, OK),
    (compress_sharded, dict(null_image=True), PARAM),
    (compress_sharded, dict(swizzle=None), PARAM),
    (compress_sharded, dict(data=False), PARAM),
    (compress_sharded, dict(ctx="dec_only"), CTX),
    (compress_sharded, dict(swizzle=(0, 1, 2, 6)), SWZ),
    (compress_sharded, dict(dim_x=0), PARAM),
    (compress_sharded, dict(dim_x=HUGE, dim_y=HUGE, dim_z=HUGE), PARAM),
    (compress_sharded, dict(data_type=3), PARAM),
    (compress_sharded, dict(ctx="radius", dim_z=2, out_len=128), NI),
    (compress_sharded, dict(root=1), PARAM),
    (compress_sharded, dict(out_len=63), OOM),
    (compress_sharded, dict(null_out=True), PARAM),
    (compress_sharded, dict(ctx="dec_only", swizzle=None), PARAM),
    (compress_sharded, dict(ctx="dec_only", swizzle=(0, 1, 2, 6)), CTX),
    (compress_sharded, dict(swizzle=(0, 1, 2, 6), dim_x=0), SWZ),
    (compress_sharded, dict(dim_x=0, data_type=3), PARAM),
    (compress_sharded, dict(ctx="radius", dim_z=2, data_type=3), PARAM),
    (compress_sharded, dict(ctx="radius", dim_z=2, out_len=0), NI),
    (compress_sharded, dict(root=1, out_len=0), PARAM),
    # astcenc_b200_compress_batch (world 1): pointers and count, root, every image's checks, matching geometry, outputs
    (compress_batch, {}, OK),
    (compress_batch, dict(null_images=True), PARAM),
    (compress_batch, dict(count=0), PARAM),
    (compress_batch, dict(swizzle=None), PARAM),
    (compress_batch, dict(root=1), PARAM),
    (compress_batch, dict(ctx="dec_only"), CTX),
    (compress_batch, dict(swizzle=(0, 1, 2, 6)), SWZ),
    (compress_batch, dict(dim_y=0), PARAM),
    (compress_batch, dict(data_type=3), PARAM),
    (compress_batch, dict(ctx="radius", dim_z=2, out_len=128), NI),
    (compress_batch, dict(second=dict(dim_x=W - 1)), PARAM),
    (compress_batch, dict(second=dict(data_type=3)), PARAM),
    (compress_batch, dict(out_len=63), OOM),
    (compress_batch, dict(null_out=True), PARAM),
    (compress_batch, dict(ctx="dec_only", root=1), PARAM),
    (compress_batch, dict(ctx="dec_only", swizzle=(0, 1, 2, 6)), CTX),
    (compress_batch, dict(swizzle=(0, 1, 2, 6), out_len=0), SWZ),
    (compress_batch, dict(second=dict(dim_x=W - 1), out_len=0), PARAM),
    (compress_batch, dict(ctx="radius", dim_z=2, out_len=0), NI),
    (compress_batch, dict(second=dict(dim_y=0), out_len=0), PARAM),
]


def _id(case):
    fn, kw, code = case
    return "%s-%s-%d" % (fn.__name__, "-".join("%s=%s" % (k, v) for k, v in sorted(kw.items())) or "ok", code)


@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
def test_entry_point_error_codes(env, case):
    import torch
    fn, kw, want = case
    pkg, ctxs = env[0], env[1]
    ctx = ctxs[kw.get("ctx", "plain")]
    before = ctx.launch_count()
    assert fn(env, **kw) == want
    torch.cuda.synchronize()
    if want != OK:
        assert ctx.launch_count() == before
