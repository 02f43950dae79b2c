"""Decode calls over image tables: astcenc_b200_decompress_device_images decodes many device-resident payloads into device
images in one launch (astc_decompress_images_kernel; the table walk is decode_table_blocks in astc_dev_gather.cuh).

CPU: the table walk compiled for the host (tests/hostsim/hostsim_decode_images.cpp, one lane and 32 lanes) over calls that mix image
sizes, a 1 x 1 image, a texture array and volumes, in CTA shares that split and span images, against the oracle's decode of
each image alone.
GPU: every output against Context.decompress_image of the same payload, with sentinel bytes around every output."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import astc_blockgen as G
from astc_ref import *  # noqa: F401,F403
from hostsim_build import host_sim

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
from make_golden_decode import DCASES, make_blocks  # noqa: E402
from test_multi_image import mip_chain  # noqa: E402

import astc_images as I  # noqa: E402

NP = {TYPE_U8: np.uint8, TYPE_F16: np.float16, TYPE_F32: np.float32}
PROFILES = (PRF_LDR_SRGB, PRF_LDR, PRF_HDR_RGB_LDR_A, PRF_HDR)
GAP = 37
SENTINEL = 0xA5


_SIMS = {}


def decode_sim(lanes32=False):
    """tests/hostsim/hostsim_decode_images.cpp compiled for the host (one simulated lane, or 32 lanes on 32 threads)."""
    if lanes32 in _SIMS:
        return _SIMS[lanes32]
    lib = host_sim("hostsim_decode_images", lanes32)
    lib.hostsim_decompress_images.argtypes = [C.c_int, C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_int,
                                              C.POINTER(C.c_int), C.c_size_t]
    _SIMS[lanes32] = lib
    return lib


def block_pool(fp, golden, seed):
    """Blocks of the footprint: its astc_blockgen set (every legal mode, partitioning and endpoint mode, void extents, illegal
    encodings), real encodings of the golden decode cases of that footprint, and random bytes."""
    parts = [G.mosaic(fp).blocks.reshape(-1, 16)]
    for i, c in enumerate(DCASES):
        if fp[2] == 1 and (c[4], c[5]) == fp[:2]:
            parts.append(make_blocks(c[1], c[2], c[4], c[5], golden, 100 + i).reshape(-1, 16))
    parts.append(np.random.default_rng(seed).integers(0, 256, size=(64, 16), dtype=np.uint8))
    return np.ascontiguousarray(np.concatenate(parts))


def nblocks(shape, fp):
    d, h, w = shape
    return -(-w // fp[0]) * -(-h // fp[1]) * (-(-d // fp[2]) if fp[2] > 1 else d)


def payloads_for(shapes, fp, pool, start=0):
    """One payload per (D, H, W) shape, consecutive blocks of the pool (wrapping), so the call covers the whole pool."""
    out, k = [], start
    for s in shapes:
        n = nblocks(s, fp)
        idx = (k + np.arange(n)) % len(pool)
        out.append(np.ascontiguousarray(pool[idx].reshape(-1)))
        k += n
    return out


def oracle_decode(oracle, payload, shape, fp, profile, out_type, swz, flags=0):
    """The oracle's decode of one image alone: (D, H, W, 4); a texture array slice by slice."""
    d, h, w = shape
    if fp[2] > 1:
        return oracle.decompress_volume(payload, w, h, d, profile, fp[0], fp[1], fp[2], out_type=out_type, flags=flags, swz=list(swz))
    per = nblocks((1, h, w), fp) * 16
    return np.stack([oracle.decompress(payload[z * per:(z + 1) * per], w, h, profile, fp[0], fp[1], out_type, flags, list(swz)) for z in range(d)])


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
SHAPES_6X6 = [(1, 37, 29), (1, 1, 1), (3, 13, 17), (1, 6, 6), (1, 5, 61), (2, 7, 1)]      # (D, H, W); (3, 13, 17) is a texture array
SHAPES_4X4X4 = [(5, 7, 9), (1, 1, 1), (4, 4, 4), (9, 3, 13)]
# (name, footprint, shapes, profile, output type, swizzle)
SIM_CASES = [
    ("6x6_ldr_u8", (6, 6, 1), SHAPES_6X6, PRF_LDR, TYPE_U8, (0, 1, 2, 3)),
    ("6x6_hdr_f16_z", (6, 6, 1), SHAPES_6X6, PRF_HDR, TYPE_F16, (0, 3, 6, 5)),
    ("6x6_srgb_f32_bgr0", (6, 6, 1), SHAPES_6X6[::-1], PRF_LDR_SRGB, TYPE_F32, (2, 1, 0, 4)),
    ("4x4x4_ldr_u8", (4, 4, 4), SHAPES_4X4X4, PRF_LDR, TYPE_U8, (0, 1, 2, 3)),
    ("4x4x4_hdr_ldra_f32_z", (4, 4, 4), SHAPES_4X4X4[::-1], PRF_HDR_RGB_LDR_A, TYPE_F32, (3, 6, 1, 0)),
]


def sim_decode(lib, payloads, shapes, fp, profile, out_type, swz, share):
    outs = [np.zeros(s + (4,), NP[out_type]) for s in shapes]
    pays = (C.c_void_p * len(payloads))(*[p.ctypes.data for p in payloads])
    optr = (C.c_void_p * len(outs))(*[o.ctypes.data for o in outs])
    dims = np.array([[s[2], s[1], s[0]] for s in shapes], np.uint32).reshape(-1)
    sw = (C.c_int * 4)(*swz)
    assert lib.hostsim_decompress_images(profile, fp[0], fp[1], fp[2], 0, pays, optr, dims.ctypes.data, len(shapes), out_type, sw, share) == 0
    return outs


@pytest.mark.parametrize("lanes32", [False, True], ids=["lanes1", "lanes32"])
@pytest.mark.parametrize("case", SIM_CASES, ids=[c[0] for c in SIM_CASES])
def test_hostsim_table_walk_equals_oracle_per_image(case, lanes32, oracle, golden):
    """Every image of one decode call equals the oracle's decode of that image alone, byte for byte, whether one CTA takes the
    whole call or the CTA shares split images and slices (7 blocks) or hold one block each."""
    _, fp, shapes, profile, out_type, swz = case
    lib = decode_sim(lanes32)
    pool = block_pool(fp, golden, 3)
    if lanes32:
        pool = pool[::7]      # (the 32-lane simulation is slow: a sample of the set)
    # one more image, with ragged edges, is large enough to take in the rest of the pool
    cols = 48
    rows = -(-len(pool) // (cols * (2 if fp[2] > 1 else 1)))
    shapes = shapes[:2] + [((2 * fp[2] if fp[2] > 1 else 1), rows * fp[1] - 1, cols * fp[0] - 1)] + shapes[2:]
    payloads = payloads_for(shapes, fp, pool)
    want = [oracle_decode(oracle, p, s, fp, profile, out_type, swz) for p, s in zip(payloads, shapes)]
    total = sum(nblocks(s, fp) for s in shapes)
    for share in (total, 7, 1):
        got = sim_decode(lib, payloads, shapes, fp, profile, out_type, swz, share)
        for k, (g, w) in enumerate(zip(got, want)):
            assert np.array_equal(g.view(np.uint8), w.view(np.uint8)), "image %d %s, share %d" % (k, shapes[k], share)


# ---------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu(pkg):
    import torch
    assert torch.cuda.is_available(), "the GPU tests need a CUDA device"
    torch.cuda.set_device(0)
    return pkg


def out_bytes(shape, out_type):
    return int(np.prod(shape)) * 4 * np.dtype(NP[out_type]).itemsize


def out_layout(shapes, out_type, odd=False):
    """Output offsets in one allocation, GAP sentinel bytes before and after every image; aligned to the texel's components
    unless `odd` (then every output starts at an odd byte)."""
    align = 1 if odd else np.dtype(NP[out_type]).itemsize
    offs, pos = [], GAP
    for s in shapes:
        pos = -(-pos // align) * align
        if odd and pos % 2 == 0:
            pos += 1
        offs.append(pos)
        pos += out_bytes(s, out_type) + GAP
    return offs, pos


def decode_device(ctx, payloads, shapes, out_type, swizzle=(0, 1, 2, 3), odd=False, per_image=False, stream=None):
    """The outputs of decompress_device_images over the payloads (one call, or one call per image), decoded into one
    sentinel-filled allocation; checks that no byte outside the outputs changed and that each call is one launch."""
    import torch
    dev = torch.device("cuda", 0)
    d_pays = [torch.from_numpy(p).to(dev) for p in payloads]
    offs, total = out_layout(shapes, out_type, odd)
    d_out = torch.full((total,), SENTINEL, dtype=torch.uint8, device=dev)
    base = d_out.data_ptr()
    table = [(d.data_ptr(), base + o, s[2], s[1], s[0]) for d, o, s in zip(d_pays, offs, shapes)]
    st = stream or torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    calls = [[e] for e in table] if per_image else [table]
    for c in calls:
        n0 = ctx.launch_count()
        ctx.decompress_device_images(c, out_type, swizzle=swizzle, stream=st.cuda_stream)
        assert ctx.launch_count() == n0 + 1
    torch.cuda.synchronize()
    got = d_out.cpu().numpy()
    outs, mask = [], np.ones(total, bool)
    for s, o in zip(shapes, offs):
        n = out_bytes(s, out_type)
        outs.append(got[o:o + n].copy().view(NP[out_type]).reshape(s + (4,)))
        mask[o:o + n] = False
    assert np.all(got[mask] == SENTINEL), "a byte outside the outputs changed"
    return outs


def check_against_decompress_image(ctx, payloads, shapes, out_type, swizzle=(0, 1, 2, 3), **kw):
    got = decode_device(ctx, payloads, shapes, out_type, swizzle, **kw)
    for k, (p, s, g) in enumerate(zip(payloads, shapes, got)):
        want = ctx.decompress_image(p, s[2], s[1], dtype=NP[out_type], swizzle=swizzle, dim_z=s[0])
        want = want.reshape(s + (4,))
        assert np.array_equal(g.view(np.uint8), want.view(np.uint8)), "image %d %s type %d swizzle %s" % (k, s, out_type, swizzle)


@pytest.mark.gpu
@pytest.mark.parametrize("profile", PROFILES)
def test_golden_cases_in_one_call_and_one_call_each(profile, gpu, golden):
    """The golden decode cases' payloads of each block size, under every output type and swizzles with Z, 0 and 1, in one call
    and as one call per image."""
    by_fp = {}
    for i, c in enumerate(DCASES):
        by_fp.setdefault((c[4], c[5]), []).append((make_blocks(c[1], c[2], c[4], c[5], golden, 100 + i), (1,) + tuple(c[2])))
    for (bx, by), cases in sorted(by_fp.items()):
        ctx = gpu.Context(gpu.config_init(profile, bx, by, PRE_MEDIUM, 0))
        try:
            payloads = [np.ascontiguousarray(b) for b, _ in cases]
            shapes = [s for _, s in cases]
            for t in (TYPE_U8, TYPE_F16, TYPE_F32):
                for swz in ((0, 1, 2, 3), (0, 3, 6, 5), (2, 1, 0, 4)):
                    check_against_decompress_image(ctx, payloads, shapes, t, swz)
            check_against_decompress_image(ctx, payloads, shapes, TYPE_F16, (0, 3, 6, 5), per_image=True)
        finally:
            ctx.close()


BLOCKGEN_FPS = [(4, 4, 1), (6, 6, 1), (8, 5, 1), (12, 12, 1), (5, 5, 4)]


@pytest.mark.gpu
@pytest.mark.parametrize("fp", BLOCKGEN_FPS, ids=["%dx%dx%d" % f for f in BLOCKGEN_FPS])
def test_blockgen_sets(fp, gpu, golden):
    """Every legal block mode, partitioning and endpoint mode, void extents and illegal encodings (astc_blockgen), laid out as
    the footprint's mosaic and as a call of mixed shapes (arrays for 2D footprints, ragged volumes for 3D ones)."""
    mo = G.mosaic(fp)
    w, h, d = mo.dims
    shapes = [(d, h, w)] + ([(3, 13, 17), (1, 1, 1), (2, 29, 31)] if fp[2] == 1 else [(7, 9, 11), (1, 1, 1), (fp[2], fp[1], fp[0])])
    pool = block_pool(fp, golden, 5)
    payloads = [np.ascontiguousarray(mo.blocks)] + payloads_for(shapes[1:], fp, pool, 11)
    for profile in PROFILES:
        ctx = gpu.Context(gpu.config_init(profile, fp[0], fp[1], PRE_MEDIUM, 0, block_z=fp[2]))
        try:
            for t in (TYPE_U8, TYPE_F16, TYPE_F32):
                check_against_decompress_image(ctx, payloads, shapes, t, (0, 1, 2, 3) if t != TYPE_F16 else (0, 3, 6, 5))
        finally:
            ctx.close()


@pytest.mark.gpu
def test_round_trip_of_compress_device_images(gpu):
    """compress_device_images of a 300 x 257 mip chain and of 64 textures of 128 x 128, then decompress_device_images on the
    same device payloads: each output equals decompress_image of the payload."""
    import torch
    dev = torch.device("cuda", 0)
    chain = mip_chain(I.photo_like(257, 300, seed=8))
    assert chain[-1].shape[:2] == (1, 1)
    textures = [I.photo_like(128, 128, seed=100 + k) for k in range(64)]
    for imgs, (bx, by) in ((chain, (6, 6)), (textures, (4, 4))):
        ctx = gpu.Context(gpu.config_init(PRF_LDR, bx, by, PRE_FAST, 0))
        try:
            d_imgs = [torch.from_numpy(np.ascontiguousarray(im)).to(dev) for im in imgs]
            sizes = [nblocks((1,) + im.shape[:2], (bx, by, 1)) * 16 for im in imgs]
            d_pays = [torch.zeros(n, dtype=torch.uint8, device=dev) for n in sizes]
            d_outs = [torch.zeros(im.size, dtype=torch.uint8, device=dev) for im in imgs]
            st = torch.cuda.Stream(device=dev)
            torch.cuda.synchronize()
            ctx.compress_device_images([(d.data_ptr(), im.shape[1], im.shape[0], 1, p.data_ptr()) for d, im, p in zip(d_imgs, imgs, d_pays)], TYPE_U8,
                                       stream=st.cuda_stream)
            ctx.decompress_device_images([(p.data_ptr(), o.data_ptr(), im.shape[1], im.shape[0], 1) for p, o, im in zip(d_pays, d_outs, imgs)], TYPE_U8,
                                         stream=st.cuda_stream)
            torch.cuda.synchronize()
            for k, (p, o, im) in enumerate(zip(d_pays, d_outs, imgs)):
                want = ctx.decompress_image(p.cpu().numpy(), im.shape[1], im.shape[0])
                assert np.array_equal(o.cpu().numpy().reshape(im.shape), want), "image %d %s" % (k, im.shape)
        finally:
            ctx.close()


@pytest.mark.gpu
def test_outputs_at_odd_byte_offsets(gpu, golden):
    """Outputs may start at any byte: U8 (and F16 / F32) images at odd offsets, with sentinels around each."""
    fp = (6, 6, 1)
    shapes = [(1, 37, 29), (1, 1, 1), (3, 13, 17), (1, 64, 64)]
    payloads = payloads_for(shapes, fp, block_pool(fp, golden, 9))
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_MEDIUM, 0))
    try:
        for t in (TYPE_U8, TYPE_F16, TYPE_F32):
            check_against_decompress_image(ctx, payloads, shapes, t, (0, 3, 6, 5), odd=True)
    finally:
        ctx.close()


@pytest.mark.gpu
def test_decompress_only_context(gpu, golden):
    fp = (8, 8, 1)
    shapes = [(1, 64, 64), (2, 9, 70), (1, 1, 1)]
    payloads = payloads_for(shapes, fp, block_pool(fp, golden, 4))
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 8, 8, PRE_MEDIUM, gpu.FLG_DECOMPRESS_ONLY))
    try:
        check_against_decompress_image(ctx, payloads, shapes, TYPE_U8)
        check_against_decompress_image(ctx, payloads, shapes, TYPE_F16, (0, 3, 6, 5))
    finally:
        ctx.close()


@pytest.mark.gpu
def test_compress_and_decode_passes_on_two_streams_are_ordered(gpu):
    """A compress_device_images pass and a decompress_device_images pass of ONE context on two streams share its table
    buffer: the library orders them, so each decode sees its own table."""
    import torch
    dev = torch.device("cuda", 0)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_MEDIUM, 0))
    try:
        imgs = mip_chain(I.photo_like(300, 310, seed=1))
        pays = [ctx.compress_image(im).copy() for im in imgs]
        want = [ctx.decompress_image(p, im.shape[1], im.shape[0]) for p, im in zip(pays, imgs)]
        other = [I.photo_like(96, 80, seed=k) for k in range(6)]
        want_other = [ctx.compress_image(im).copy() for im in other]
        d_imgs = [torch.from_numpy(im).to(dev) for im in other]
        d_cpay = [torch.zeros(p.size, dtype=torch.uint8, device=dev) for p in want_other]
        d_pays = [torch.from_numpy(p).to(dev) for p in pays]
        d_outs = [torch.zeros(im.size, dtype=torch.uint8, device=dev) for im in imgs]
        streams = [torch.cuda.Stream(device=dev) for _ in range(2)]
        torch.cuda.synchronize()
        for rep in range(3):
            ctx.compress_device_images([(d.data_ptr(), 80, 96, 1, p.data_ptr()) for d, p in zip(d_imgs, d_cpay)], TYPE_U8, stream=streams[0].cuda_stream)
            ctx.decompress_device_images([(p.data_ptr(), o.data_ptr(), im.shape[1], im.shape[0], 1) for p, o, im in zip(d_pays, d_outs, imgs)], TYPE_U8,
                                         stream=streams[1].cuda_stream)
        torch.cuda.synchronize()
        for k, (o, w) in enumerate(zip(d_outs, want)):
            assert np.array_equal(o.cpu().numpy().reshape(w.shape), w), "level %d" % k
        for k, (p, w) in enumerate(zip(d_cpay, want_other)):
            assert np.array_equal(p.cpu().numpy(), w), "texture %d" % k
    finally:
        ctx.close()


@pytest.mark.gpu
def test_error_order_launches_nothing_and_writes_nothing(gpu):
    import torch
    dev = torch.device("cuda", 0)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, 0))
    d_pay = torch.zeros(4096, dtype=torch.uint8, device=dev)
    nbytes = 65536
    d_out = torch.full((nbytes,), SENTINEL, dtype=torch.uint8, device=dev)
    big = 0xFFFFFFFF
    l = gpu.lib()
    sw = gpu.Swizzle(0, 1, 2, 3)

    def table(**edit):
        t = [[d_pay.data_ptr(), d_out.data_ptr(), 44, 40, 1], [d_pay.data_ptr() + 2048, d_out.data_ptr() + 32768, 13, 12, 2]]
        for k, (i, f, v) in edit.items():
            t[i][f] = v
        return [tuple(e) for e in t]

    def _raise(err):
        if err:
            raise gpu.AstcencError(err, "call")

    def expect(code, images=None, data_type=TYPE_U8, swizzle=(0, 1, 2, 3), raw=None):
        n0 = ctx.launch_count()
        call = raw or (lambda: ctx.decompress_device_images(table() if images is None else images, data_type, swizzle=swizzle))
        if code == 0:
            call()
        else:
            with pytest.raises(gpu.AstcencError) as e:
                call()
            assert e.value.code == code
        torch.cuda.synchronize()
        assert ctx.launch_count() == n0
        assert np.all(d_out.cpu().numpy() == SENTINEL)

    try:
        expect(gpu.ERR_BAD_PARAM, swizzle=None)
        expect(gpu.ERR_BAD_PARAM, swizzle=None, images=table(a=(0, 0, 0)))          # (a NULL swizzle comes first)
        expect(gpu.ERR_BAD_SWIZZLE, swizzle=(0, 1, 2, 7))
        expect(gpu.ERR_BAD_SWIZZLE, swizzle=(0, 1, 2, 7), images=table(a=(1, 2, 0)))  # (the swizzle comes before the images)
        expect(gpu.ERR_BAD_PARAM, raw=lambda: _raise(l.astcenc_b200_decompress_device_images(ctx.handle, None, 2, TYPE_U8, C.byref(sw), None)))
        expect(gpu.ERR_BAD_PARAM, images=table(a=(1, 0, 0)))
        expect(gpu.ERR_BAD_PARAM, images=table(a=(0, 1, 0)))
        expect(gpu.ERR_BAD_PARAM, images=table(a=(1, 3, 0)))
        expect(gpu.ERR_BAD_PARAM, images=table(a=(0, 4, 0)))
        expect(gpu.ERR_BAD_PARAM, data_type=3)
        expect(gpu.ERR_BAD_PARAM, images=table(a=(0, 2, big), b=(0, 3, big), c=(0, 4, big)))      # (texel count overflow)
        expect(gpu.ERR_BAD_PARAM, images=table(a=(0, 2, 6 * 65536), b=(0, 3, 6 * 65536)))         # (2^32 blocks: one image too many)
        expect(0, images=[])
        expect(0, raw=lambda: _raise(l.astcenc_b200_decompress_device_images(ctx.handle, None, 0, TYPE_U8, C.byref(sw), None)))
    finally:
        ctx.close()
