"""Image tables: astcenc_b200_compress_device_images / astcenc_b200_compress_images compress every block of many images - mip
chains, texture sets - in shared pipeline passes (gather into staging rows, one ordinary pass per row, scatter to each image's
payload; astc_dev_gather.cuh).

CPU: the image-table gather and scatter (tests/hostsim/hostsim_blocks.cpp compiles astc_dev_gather.cuh for the host) against a
numpy restatement of load_block's clamp-to-edge and of the alpha averages, and the device source's pass over a multi-image
staging row (one lane and 32 lanes) against the oracle's blocks of each image.
GPU: every payload against Context.compress_image of that image alone, with sentinel gaps between the payloads."""
import ctypes as C
import os

import numpy as np
import pytest

import astc_images as I
from astc_ref import *  # noqa: F401,F403
from test_block_list import blocks_sim

S = FLG_SELF_DECOMPRESS_ONLY
_DT = {np.dtype(np.uint8): TYPE_U8, np.dtype(np.float16): TYPE_F16, np.dtype(np.float32): TYPE_F32}


def grid(shape, fp):
    """(blocks_x, blocks_y, layers) of a (D, H, W, 4) image: layers = slices for 2D footprints, layers of blocks for 3D ones."""
    d, h, w = shape[:3]
    return -(-w // fp[0]), -(-h // fp[1]), -(-d // fp[2])


def nblocks(shape, fp):
    return int(np.prod(grid(shape, fp)))


def staged_reference(vol, fp):
    """Every block of one image, staged as load_block reads it (clamped to the image's edges), block i at x = i * bx:
    (bz, by, blocks * bx, 4)."""
    d, h, w = vol.shape[:3]
    bx, by, bz = fp
    nbx, nby, nl = grid(vol.shape, fp)
    out = np.zeros((bz, by, nbx * nby * nl * bx, 4), vol.dtype)
    for b in range(nbx * nby * nl):
        col, rest = b % nbx, b // nbx
        row, layer = rest % nby, rest // nby
        xs = np.minimum(col * bx + np.arange(bx), w - 1)
        ys = np.minimum(row * by + np.arange(by), h - 1)
        zs = np.minimum(layer * bz + np.arange(bz), d - 1)
        out[:, :, b * bx:(b + 1) * bx] = vol[zs][:, ys][:, :, xs]
    return out


def averages_reference(h, w, avg, fp):
    """The staged averages of every block of one 2D image: its averages, 0 outside the image. (by, blocks * bx)."""
    bx, by, _ = fp
    nbx, nby, _ = grid((1, h, w), fp)
    padded = np.zeros((nby * by, nbx * bx), np.float32)
    padded[:h, :w] = avg
    return np.concatenate([padded[r * by:(r + 1) * by, c * bx:(c + 1) * bx] for r in range(nby) for c in range(nbx)], axis=1)


def sim_gather(lib, vols, fp, base, n, avgs=None):
    """Staging blocks [base, base + n) of the call over `vols`, gathered by the host-compiled gather."""
    vols = [np.ascontiguousarray(v) for v in vols]
    ptrs = (C.c_void_p * len(vols))(*[v.ctypes.data for v in vols])
    dims = np.array([[v.shape[2], v.shape[1], v.shape[0]] for v in vols], np.uint32).reshape(-1)
    staged = np.zeros((fp[2], fp[1], n * fp[0], 4), vols[0].dtype)
    avg = savg = None
    if avgs is not None:
        avg = np.ascontiguousarray(np.concatenate([a.reshape(-1) for a in avgs]).astype(np.float32))
        savg = np.full((fp[1], n * fp[0]), -1.0, np.float32)
    lib.hostsim_gather_table(ptrs, dims.ctypes.data, len(vols), _DT[vols[0].dtype], fp[0], fp[1], fp[2], None, None, None, base, n,
                             avg.ctypes.data if avg is not None else None, staged.ctypes.data, savg.ctypes.data if savg is not None else None)
    return staged, savg


def sim_scatter(lib, shapes, fp, base, staged_blocks, payloads):
    dims = np.array([[s[2], s[1], s[0]] for s in shapes], np.uint32).reshape(-1)
    ptrs = (C.c_void_p * len(payloads))(*[p.ctypes.data for p in payloads])
    lib.hostsim_scatter_table(dims.ctypes.data, len(shapes), fp[0], fp[1], fp[2], None, None, None, base, len(staged_blocks),
                              np.ascontiguousarray(staged_blocks).ctypes.data, ptrs)


def random_image(rng, dtype, shape):
    if dtype == np.uint8:
        return rng.integers(0, 256, size=shape + (4,), dtype=np.uint8)
    return rng.standard_normal(shape + (4,)).astype(dtype)


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
SIZES_2D = [(1, 1, 1), (1, 3, 5), (1, 19, 37), (1, 64, 64)]      # (D, H, W)
GATHER = [
    ("u8_2d_4x4", np.uint8, SIZES_2D, (4, 4, 1)),
    ("f16_2d_6x6", np.float16, SIZES_2D, (6, 6, 1)),
    ("f32_2d_12x12", np.float32, SIZES_2D, (12, 12, 1)),
    ("u8_2d_5x4", np.uint8, SIZES_2D[::-1], (5, 4, 1)),
    ("f16_array_and_2d_8x8", np.float16, [(3, 19, 21), (1, 5, 3), (2, 1, 1)], (8, 8, 1)),
    ("u8_volumes_4x4x4", np.uint8, [(1, 1, 1), (7, 9, 11), (4, 4, 4), (5, 3, 2)], (4, 4, 4)),
    ("f32_volumes_3x3x3", np.float32, [(5, 8, 7), (1, 1, 1), (2, 3, 5)], (3, 3, 3)),
    ("f16_volumes_6x5x5", np.float16, [(6, 11, 13), (1, 5, 3)], (6, 5, 5)),
]


@pytest.mark.parametrize("case", GATHER, ids=[c[0] for c in GATHER])
def test_gather_and_scatter_follow_the_image_table(case):
    """Every block of every image lands in call order in the staging row, as load_block reads it, whatever the chunking; the
    scatter puts each staged block at its image's payload position."""
    _, dtype, shapes, fp = case
    lib = blocks_sim()
    rng = np.random.default_rng(17)
    vols = [random_image(rng, dtype, s) for s in shapes]
    flat = all(s[0] == 1 for s in shapes) and fp[2] == 1
    avgs = [rng.random(s[1:3], dtype=np.float32) for s in shapes] if flat else None
    want = np.concatenate([staged_reference(v, fp) for v in vols], axis=2)
    want_avg = np.concatenate([averages_reference(s[1], s[2], a, fp) for s, a in zip(shapes, avgs)], axis=1) if flat else None
    counts = [nblocks(s, fp) for s in shapes]
    total = sum(counts)
    # one chunk; chunks of 7 (which split images and span several); chunks of one block
    for chunk in (total, 7, 1):
        payloads = [np.zeros(c * 16, np.uint8) for c in counts]
        for base in range(0, total, chunk):
            n = min(chunk, total - base)
            staged, savg = sim_gather(lib, vols, fp, base, n, avgs)
            cols = slice(base * fp[0], (base + n) * fp[0])
            assert np.array_equal(staged.view(np.uint8), want[:, :, cols].view(np.uint8)), "chunk at %d" % base
            if flat:
                assert np.array_equal(savg, want_avg[:, cols]), "averages of the chunk at %d" % base
            # (staged block c carries its call position)
            marks = np.zeros((n, 16), np.uint8)
            marks[:, :8] = np.arange(base, base + n, dtype=np.uint64)[:, None].view(np.uint8)
            sim_scatter(lib, shapes, fp, base, marks, payloads)
        got = np.concatenate([p.reshape(-1, 16)[:, :8].copy().view(np.uint64).reshape(-1) for p in payloads])
        assert np.array_equal(got, np.arange(total, dtype=np.uint64))


def transparent_image(h, w, seed, rect):
    """LDR RGBA8 with alpha noise and a fully transparent rectangle rect = (y0, y1, x0, x1), whose inner blocks the
    alpha-scale test turns into constant zero."""
    img = I.photo_like(h, w, seed=seed).copy()
    img[..., 3] = np.random.default_rng(seed).integers(0, 256, size=(h, w), dtype=np.uint8)
    y0, y1, x0, x1 = rect
    img[y0:y1, x0:x1, 3] = 0
    return np.ascontiguousarray(img)


def ldr_image(h, w, d, seed, dtype=np.uint8):
    img = np.ascontiguousarray(I.photo_like(h * d, w, seed=seed).reshape(d, h, w, 4))
    if dtype == np.uint8:
        return img
    return np.ascontiguousarray((img.astype(np.float32) / 255.0).astype(dtype))


def hdr_image(h, w, d, seed, dtype):
    return np.ascontiguousarray(I.hdr_noise(h * d, w, seed=seed, dtype=dtype).reshape(d, h, w, 4))


PASS_SHAPES_2D = [(1, 1, 1), (1, 3, 5), (1, 13, 17), (1, 9, 14)]
# (name, profile, dtype, footprint, quality, a_scale_radius, lanes32)
PARITY = [
    ("ldr_u8_4x4_fast", PRF_LDR, np.uint8, (4, 4, 1), PRE_FAST, 0, False),
    ("ldr_u8_4x4_fast_32lanes", PRF_LDR, np.uint8, (4, 4, 1), PRE_FAST, 0, True),
    ("srgb_u8_6x6_medium", PRF_LDR_SRGB, np.uint8, (6, 6, 1), PRE_MEDIUM, 0, False),
    ("ldr_f32_12x12_fast", PRF_LDR, np.float32, (12, 12, 1), PRE_FAST, 0, False),
    ("srgb_f16_5x4_medium_32lanes", PRF_LDR_SRGB, np.float16, (5, 4, 1), PRE_MEDIUM, 0, True),
    ("hdr_f16_6x6_fast", PRF_HDR, np.float16, (6, 6, 1), PRE_FAST, 0, False),
    ("hdr_rgb_ldr_a_f32_4x4_fast_32lanes", PRF_HDR_RGB_LDR_A, np.float32, (4, 4, 1), PRE_FAST, 0, True),
    ("ldr_u8_4x4_fast_radius3", PRF_LDR, np.uint8, (4, 4, 1), PRE_FAST, 3, False),
    ("ldr_u8_6x6_medium_radius3_32lanes", PRF_LDR, np.uint8, (6, 6, 1), PRE_MEDIUM, 3, True),
    ("ldr_u8_volumes_4x4x4_fast", PRF_LDR, np.uint8, (4, 4, 4), PRE_FAST, 0, False),
    ("hdr_f16_volumes_3x3x3_fast_32lanes", PRF_HDR, np.float16, (3, 3, 3), PRE_FAST, 0, True),
]


@pytest.mark.parametrize("case", PARITY, ids=[c[0] for c in PARITY])
def test_pass_over_multi_image_row_equals_each_image(case, oracle):
    """The device source's pass over one staging row of several images, scattered, gives the oracle's payload of each image."""
    _, prof, dtype, fp, q, radius, lanes32 = case
    lib = blocks_sim(lanes32)
    hdr = prof in (PRF_HDR, PRF_HDR_RGB_LDR_A)
    if radius:
        vols = [transparent_image(1, 1, 2, (0, 1, 0, 1))[None], transparent_image(7, 5, 3, (0, 0, 0, 0))[None],
                transparent_image(36, 40, 4, (6, 30, 8, 34))[None]]
    elif fp[2] > 1:
        shapes = [(1, 1, 1), (5, 6, 7), (3, 2, 9)]
        vols = [hdr_image(s[1], s[2], s[0], 5 + k, dtype) if hdr else ldr_image(s[1], s[2], s[0], 5 + k, dtype) for k, s in enumerate(shapes)]
    else:
        vols = [hdr_image(s[1], s[2], 1, 5 + k, dtype) if hdr else ldr_image(s[1], s[2], 1, 5 + k, dtype) for k, s in enumerate(PASS_SHAPES_2D)]
    shapes = [v.shape[:3] for v in vols]
    if fp[2] > 1:
        want = [oracle.compress_volume(v, prof, fp[0], fp[1], fp[2], q, S) for v in vols]
    else:
        want = [oracle.compress(v[0], prof, fp[0], fp[1], q, S, a_scale_radius=radius) for v in vols]
    avgs = None
    if radius:
        avgs = []
        for v in vols:
            a = np.zeros(v.shape[1:3], np.float32)
            lib.hostsim_alpha_averages_2d(np.ascontiguousarray(v[0]).ctypes.data, TYPE_U8, v.shape[2], v.shape[1], None, radius, a.ctypes.data)
            avgs.append(a)
    total = sum(nblocks(s, fp) for s in shapes)
    staged, savg = sim_gather(lib, vols, fp, 0, total, avgs)
    out = np.zeros(total * 16, np.uint8)
    rc = lib.hostsim_compress_staged(prof, fp[0], fp[1], fp[2], q, S, radius, staged.ctypes.data, _DT[staged.dtype], total * fp[0], fp[1], fp[2],
                                     savg.ctypes.data if savg is not None else None, out.ctypes.data)
    assert rc == 0
    payloads = [np.zeros(nblocks(s, fp) * 16, np.uint8) for s in shapes]
    sim_scatter(lib, shapes, fp, 0, out.reshape(-1, 16), payloads)
    for k, (got, w) in enumerate(zip(payloads, want)):
        bad = block_diff(got, w)
        assert len(bad) == 0, "image %d: blocks %s differ" % (k, list(bad)[:8])
    if radius:
        assert np.any(np.all(want[2].reshape(-1, 16)[:, 8:] == 0, axis=1)), "the call should hold constant-zero blocks"


# ---------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu(pkg):
    import torch
    assert torch.cuda.is_available(), "these tests need a CUDA device"
    return pkg


GAP = 48      # sentinel bytes before, between and after the payloads


def sentinel(nbytes):
    return (np.arange(nbytes, dtype=np.uint32) * 131 + 7).astype(np.uint8)


def payload_bytes(ctx, vol):
    fp = (ctx.config.block_x, ctx.config.block_y, max(1, ctx.config.block_z))
    return nblocks(vol.shape, fp) * 16


def layout(ctx, vols):
    """Payload offsets in one allocation with GAP sentinel bytes around every payload (odd gaps misalign some payloads)."""
    offs, pos = [], GAP
    for k, v in enumerate(vols):
        offs.append(pos)
        pos += payload_bytes(ctx, v) + GAP + (k % 3)
    return offs, pos


def as_volume(v):
    v = np.ascontiguousarray(v)
    return v[None] if v.ndim == 3 else v


def run_images(ctx, vols, swizzle=(0, 1, 2, 3), stream=None):
    """The payloads of one compress_device_images call over `vols`, in one sentinel-filled allocation; checks that no sentinel
    byte changed."""
    import torch
    dev = torch.device("cuda", 0)
    vols = [as_volume(v) for v in vols]
    d_imgs = [torch.from_numpy(v.view(np.uint8).reshape(-1)).to(dev) for v in vols]
    offs, total = layout(ctx, vols)
    d_pay = torch.from_numpy(sentinel(total)).to(dev)
    base = d_pay.data_ptr()
    table = [(d.data_ptr(), v.shape[2], v.shape[1], v.shape[0], base + o) for d, v, o in zip(d_imgs, vols, offs)]
    st = stream or torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    ctx.compress_device_images(table, _DT[vols[0].dtype], swizzle=swizzle, stream=st.cuda_stream)
    torch.cuda.synchronize()
    got = d_pay.cpu().numpy()
    outs, mask = [], np.ones(total, bool)
    for v, o in zip(vols, offs):
        n = payload_bytes(ctx, v)
        outs.append(got[o:o + n].copy())
        mask[o:o + n] = False
    assert np.array_equal(got[mask], sentinel(total)[mask]), "a byte outside the payloads changed"
    return outs


def check_images(ctx, vols, swizzle=(0, 1, 2, 3)):
    got = run_images(ctx, vols, swizzle)
    for k, (v, g) in enumerate(zip(vols, got)):
        want = ctx.compress_image(v, swizzle=swizzle)
        bad = block_diff(g, want)
        assert len(bad) == 0, "image %d (%s): %d blocks differ" % (k, v.shape, len(bad))
    return got


def mip_chain(img):
    """img and its levels down to 1 x 1 (2 x 2 box filter, odd edges dropped), in img's dtype."""
    levels = [np.ascontiguousarray(img)]
    while levels[-1].shape[0] > 1 or levels[-1].shape[1] > 1:
        a = levels[-1].astype(np.float32)
        h, w = a.shape[:2]
        h2, w2 = max(1, h // 2), max(1, w // 2)
        a = a[:h2 * 2 if h > 1 else 1, :w2 * 2 if w > 1 else 1]
        a = a.reshape(h2, a.shape[0] // h2, w2, a.shape[1] // w2, 4).mean(axis=(1, 3))
        if img.dtype == np.uint8:
            a = np.round(a)
        levels.append(np.ascontiguousarray(a.astype(img.dtype)))
    return levels


_QN = {PRE_FAST: "fast", PRE_MEDIUM: "medium", PRE_THOROUGH: "thorough"}
CHAINS = [((4, 4), PRE_FAST), ((6, 6), PRE_MEDIUM), ((8, 8), PRE_THOROUGH), ((12, 12), PRE_MEDIUM)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CHAINS, ids=["%dx%d_%s" % (c[0][0], c[0][1], _QN[c[1]]) for c in CHAINS])
def test_mip_chain_equals_compress_image(case, gpu):
    (bx, by), q = case
    levels = mip_chain(I.photo_like(600, 1000, seed=31))
    assert levels[-1].shape[:2] == (1, 1)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, bx, by, q, S))
    try:
        check_images(ctx, levels)
    finally:
        ctx.close()


@pytest.mark.gpu
def test_hdr_srgb_and_swizzled_chains_equal_compress_image(gpu):
    hdr = mip_chain(I.hdr_noise(300, 500, seed=4, dtype=np.float16))
    ctx = gpu.Context(gpu.config_init(PRF_HDR, 6, 6, PRE_MEDIUM, S))
    try:
        check_images(ctx, hdr)
    finally:
        ctx.close()
    ldr = mip_chain(I.photo_like(300, 500, seed=5))
    ctx = gpu.Context(gpu.config_init(PRF_LDR_SRGB, 6, 6, PRE_MEDIUM, S))
    try:
        check_images(ctx, ldr)
    finally:
        ctx.close()
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 5, 4, PRE_FAST, S))
    try:
        check_images(ctx, ldr, swizzle=(2, 0, 1, 5))
        check_images(ctx, ldr, swizzle=(3, 3, 3, 4))
    finally:
        ctx.close()


def texture_set(count, seed, max_dim=150):
    rng = np.random.default_rng(seed)
    return [I.photo_like(int(rng.integers(1, max_dim)), int(rng.integers(1, max_dim)), seed=seed * 1000 + k) for k in range(count)]


@pytest.mark.gpu
def test_texture_set_of_random_sizes_equals_compress_image(gpu):
    textures = texture_set(200, 7)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_MEDIUM, S))
    try:
        check_images(ctx, textures)
    finally:
        ctx.close()


@pytest.mark.gpu
def test_texture_arrays_with_2d_images_equal_compress_image(gpu):
    vols = [ldr_image(41, 53, 3, 9), ldr_image(1, 1, 1, 2), ldr_image(17, 6, 5, 3), ldr_image(64, 64, 1, 4), ldr_image(7, 9, 2, 5)]
    for prof, dtype, fp, q in ((PRF_LDR, np.uint8, (6, 6), PRE_MEDIUM), (PRF_LDR, np.float32, (4, 4), PRE_FAST)):
        ctx = gpu.Context(gpu.config_init(prof, fp[0], fp[1], q, S))
        try:
            check_images(ctx, [v if dtype == np.uint8 else (v.astype(np.float32) / 255.0) for v in vols])
        finally:
            ctx.close()


FOOTPRINTS_3D = [(3, 3, 3), (4, 3, 3), (4, 4, 3), (4, 4, 4), (5, 4, 4), (5, 5, 4), (5, 5, 5), (6, 5, 5), (6, 6, 5), (6, 6, 6)]


@pytest.mark.gpu
def test_ragged_volumes_at_every_3d_footprint_equal_compress_image(gpu):
    shapes = [(11, 17, 19), (1, 1, 1), (3, 5, 7), (7, 2, 13), (6, 6, 6)]
    for fp in FOOTPRINTS_3D:
        vols = [ldr_image(s[1], s[2], s[0], fp[0] * 10 + fp[2] + k) for k, s in enumerate(shapes)]
        ctx = gpu.Context(gpu.config_init(PRF_LDR, fp[0], fp[1], PRE_FAST, S, block_z=fp[2]))
        try:
            check_images(ctx, vols)
        finally:
            ctx.close()
    ctx = gpu.Context(gpu.config_init(PRF_HDR, 4, 4, PRE_FAST, S, block_z=4))
    try:
        check_images(ctx, [hdr_image(s[1], s[2], s[0], k, np.float16) for k, s in enumerate(shapes)])
    finally:
        ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("radius", [1, 5, 17])
def test_alpha_scale_images_equal_compress_image(radius, gpu):
    imgs = [transparent_image(300, 259, radius, (75, 123, 51, 115)), transparent_image(1, 1, 2, (0, 1, 0, 1)),
            transparent_image(70, 90, 3, (10, 60, 10, 80)), transparent_image(13, 29, 4, (0, 13, 0, 29)), I.photo_like(45, 33, seed=radius)]
    for bx, by in ((6, 6), (4, 4)):
        cfg = gpu.config_init(PRF_LDR, bx, by, PRE_MEDIUM, S | FLG_USE_ALPHA_WEIGHT)
        cfg.a_scale_radius = radius
        ctx = gpu.Context(cfg)
        try:
            got = check_images(ctx, imgs)
            zero = [np.all(g.reshape(-1, 16)[:, 8:] == 0, axis=1) & (g.reshape(-1, 16)[:, 0] == 0xFC) for g in got]
            assert np.any(zero[0]), "the call should hold blocks the alpha-scale test zeroes"
        finally:
            ctx.close()


@pytest.mark.gpu
def test_chunks_that_split_and_span_images(gpu):
    """ASTCENC_B200_BATCH_BLOCKS (read when the context is made) = 37: staging rows of 37 blocks split the larger images and
    span several small ones; same bytes."""
    old = os.environ.get("ASTCENC_B200_BATCH_BLOCKS")
    os.environ["ASTCENC_B200_BATCH_BLOCKS"] = "37"
    try:
        ctx = gpu.Context(gpu.config_init(PRF_LDR, 5, 4, PRE_MEDIUM, S))
        cfg = gpu.config_init(PRF_LDR, 6, 6, PRE_MEDIUM, S)
        cfg.a_scale_radius = 2
        ctx_r = gpu.Context(cfg)
    finally:
        if old is None:
            del os.environ["ASTCENC_B200_BATCH_BLOCKS"]
        else:
            os.environ["ASTCENC_B200_BATCH_BLOCKS"] = old
    try:
        imgs = [I.photo_like(90, 130, seed=8)] + texture_set(30, 9, max_dim=25) + mip_chain(I.photo_like(70, 100, seed=10))
        check_images(ctx, imgs)
        check_images(ctx, [ldr_image(21, 23, 3, 11), ldr_image(5, 5, 1, 12), ldr_image(40, 9, 2, 13)])
        check_images(ctx_r, [transparent_image(80, 70, 5, (10, 60, 10, 60))] + texture_set(12, 14, max_dim=30))
    finally:
        ctx.close()
        ctx_r.close()


@pytest.mark.gpu
def test_host_entry_equals_device_entry_and_compress_image(gpu):
    imgs = mip_chain(I.photo_like(200, 300, seed=15)) + texture_set(20, 16, max_dim=60)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_MEDIUM, S))
    try:
        dev = run_images(ctx, imgs)
        host = ctx.compress_images(imgs)
        assert len(host) == len(imgs)
        for k, (h, d, im) in enumerate(zip(host, dev, imgs)):
            assert np.array_equal(h, d), "image %d: host and device entries differ" % k
            assert np.array_equal(h, ctx.compress_image(im)), "image %d differs from compress_image" % k
        host = ctx.compress_images(imgs)
        _, h2d, d2h = ctx.last_timing()
        assert h2d == sum(im.nbytes for im in imgs)
        assert d2h == sum(len(h) for h in host)
        vols = [ldr_image(9, 11, 3, 17, np.float16), ldr_image(30, 20, 1, 18, np.float16)]
        for h, v in zip(ctx.compress_images(vols), vols):
            assert np.array_equal(h, ctx.compress_image(v))
    finally:
        ctx.close()


@pytest.mark.gpu
def test_full_size_mip_chain_equals_per_level_compress_device(gpu):
    """The mip chain of the full-size config 1 image (4096^2 LDR 6x6 -medium) against a compress_device call per level."""
    import torch
    dev = torch.device("cuda", 0)
    levels = mip_chain(I.photo_like(4096, 4096, seed=2024))
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_MEDIUM, S))
    try:
        st = torch.cuda.Stream(device=dev)
        want = []
        for lv in levels:
            h, w = lv.shape[:2]
            nbx, nby = ctx.blocks(w, h)
            d_img = torch.from_numpy(lv).to(dev)
            d_out = torch.zeros(nbx * nby * 16, dtype=torch.uint8, device=dev)
            ctx.compress_device(d_img.data_ptr(), TYPE_U8, w, h, d_out.data_ptr(), stream=st.cuda_stream)
            torch.cuda.synchronize()
            want.append(d_out.cpu().numpy())
        got = run_images(ctx, levels)
        for k, (g, w) in enumerate(zip(got, want)):
            assert len(block_diff(g, w)) == 0, "level %d differs" % k
    finally:
        ctx.close()


@pytest.mark.gpu
def test_errors_launch_nothing_and_write_nothing(gpu):
    import torch
    dev = torch.device("cuda", 0)
    vols = [ldr_image(40, 44, 1, 1), ldr_image(12, 13, 2, 2)]
    d_imgs = [torch.from_numpy(v.reshape(-1)).to(dev) for v in vols]
    nbytes = 4096
    d_pay = torch.from_numpy(sentinel(nbytes)).to(dev)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, S))
    cfg_r = gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, S)
    cfg_r.a_scale_radius = 2
    ctx_r = gpu.Context(cfg_r)
    ctx_d = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, gpu.FLG_DECOMPRESS_ONLY))
    big = 0xFFFFFFFF
    l = gpu.lib()

    def table(**edit):
        t = [[d_imgs[0].data_ptr(), 44, 40, 1, d_pay.data_ptr()], [d_imgs[1].data_ptr(), 13, 12, 2, d_pay.data_ptr() + 2048]]
        for k, (i, f, v) in edit.items():
            t[i][f] = v
        return [tuple(e) for e in t]

    def expect(c, code, images=None, data_type=TYPE_U8, swizzle=(0, 1, 2, 3), raw=None):
        n0 = c.launch_count()
        call = raw or (lambda: c.compress_device_images(table() if images is None else images, data_type, swizzle=swizzle))
        if code == 0:
            call()
        else:
            with pytest.raises(gpu.AstcencError) as e:
                call()
            assert e.value.code == code
        torch.cuda.synchronize()
        assert c.launch_count() == n0
        assert np.array_equal(d_pay.cpu().numpy(), sentinel(nbytes))

    def _raise(err):
        if err:
            raise gpu.AstcencError(err, "call")

    sw = gpu.Swizzle(0, 1, 2, 3)
    try:
        expect(ctx_d, gpu.ERR_BAD_CONTEXT)
        expect(ctx_d, gpu.ERR_BAD_CONTEXT, swizzle=(0, 1, 2, 9))
        expect(ctx, gpu.ERR_BAD_SWIZZLE, swizzle=(0, 1, 2, 9))
        expect(ctx, gpu.ERR_BAD_SWIZZLE, swizzle=(0, 1, 2, 9), images=table(a=(1, 1, 0)))
        expect(ctx, gpu.ERR_BAD_PARAM, raw=lambda: _raise(l.astcenc_b200_compress_device_images(ctx.handle, None, 2, TYPE_U8, C.byref(sw), None)))
        expect(ctx, gpu.ERR_BAD_PARAM, raw=lambda: _raise(l.astcenc_b200_compress_device_images(ctx.handle, None, 1, TYPE_U8, None, None)))
        expect(ctx, gpu.ERR_BAD_PARAM, images=table(a=(1, 0, 0)))
        expect(ctx, gpu.ERR_BAD_PARAM, images=table(a=(0, 4, 0)))
        expect(ctx, gpu.ERR_BAD_PARAM, images=table(a=(1, 3, 0)))
        expect(ctx, gpu.ERR_BAD_PARAM, images=table(a=(0, 2, 0)))
        expect(ctx, gpu.ERR_BAD_PARAM, data_type=3)
        expect(ctx_r, gpu.ERR_BAD_PARAM, images=table(a=(0, 1, 0)))       # (a zero dimension comes before the radius check)
        expect(ctx_r, gpu.ERR_NOT_IMPLEMENTED)
        expect(ctx_r, gpu.ERR_NOT_IMPLEMENTED, images=table(a=(0, 1, big), b=(0, 2, big)))      # (the radius comes before overflow)
        expect(ctx, gpu.ERR_BAD_PARAM, images=table(a=(0, 1, big), b=(0, 2, big), c=(0, 3, big)))
        expect(ctx, gpu.ERR_BAD_PARAM, images=table(a=(0, 1, 6 * 65536), b=(0, 2, 6 * 65536)))      # (2^32 blocks: one image too many)
        expect(ctx, 0, images=[])

        # the host entry
        imgs = [gpu.Context._image(ctx, v) for v in vols]
        outs = [np.full(payload_bytes(ctx, v), 7, np.uint8) for v in vols]

        def host(c, imgs=imgs, lens=None, ptrs=None):
            n = len(imgs)
            arr = (C.POINTER(gpu.Image) * n)(*[C.pointer(p[2]) if p is not None else None for p in imgs])
            optr = (C.c_void_p * n)(*[o.ctypes.data for o in outs]) if ptrs is None else ptrs
            ln = (C.c_size_t * n)(*([o.nbytes for o in outs] if lens is None else lens))
            return lambda: _raise(l.astcenc_b200_compress_images(c.handle, arr, n, C.byref(sw), optr, ln))

        expect(ctx_d, gpu.ERR_BAD_CONTEXT, raw=host(ctx_d))
        expect(ctx, gpu.ERR_BAD_PARAM, raw=lambda: _raise(l.astcenc_b200_compress_images(ctx.handle, None, 1, C.byref(sw), None, None)))
        expect(ctx, gpu.ERR_BAD_PARAM, raw=host(ctx, imgs=[imgs[0], None]))
        expect(ctx, gpu.ERR_BAD_PARAM, raw=host(ctx, ptrs=(C.c_void_p * 2)(outs[0].ctypes.data, None)))
        mixed = gpu.Context._image(ctx, vols[1].astype(np.float16))
        expect(ctx, gpu.ERR_BAD_PARAM, raw=host(ctx, imgs=[imgs[0], mixed]))
        expect(ctx, gpu.ERR_BAD_PARAM, raw=host(ctx, imgs=[imgs[0], mixed], lens=[0, 0]))      # (mixed types come before length)
        expect(ctx_r, gpu.ERR_NOT_IMPLEMENTED, raw=host(ctx_r, lens=[0, 0]))
        expect(ctx, gpu.ERR_OUT_OF_MEM, raw=host(ctx, lens=[outs[0].nbytes, outs[1].nbytes - 1]))
        expect(ctx, 0, raw=lambda: _raise(l.astcenc_b200_compress_images(ctx.handle, None, 0, C.byref(sw), None, None)))
        assert all(np.all(o == 7) for o in outs)
    finally:
        ctx.close()
        ctx_r.close()
        ctx_d.close()


@pytest.mark.gpu
def test_multi_image_and_whole_image_passes_on_two_streams_are_ordered(gpu):
    """compress_device_images and compress_device calls of ONE context on two streams share its scratch: the library orders
    them."""
    import torch
    dev = torch.device("cuda", 0)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_MEDIUM, S))
    try:
        imgs = mip_chain(I.photo_like(300, 310, seed=1))
        whole = I.photo_like(300, 310, seed=2)
        want = [ctx.compress_image(im).copy() for im in imgs]
        want_whole = ctx.compress_image(whole).copy()
        d_imgs = [torch.from_numpy(im).to(dev) for im in imgs]
        d_whole_img = torch.from_numpy(whole).to(dev)
        sizes = [payload_bytes(ctx, im[None]) for im in imgs]
        d_pays = [torch.zeros(n, dtype=torch.uint8, device=dev) for n in sizes]
        nbx, nby = ctx.blocks(310, 300)
        d_whole = torch.zeros(nbx * nby * 16, dtype=torch.uint8, device=dev)
        table = [(d.data_ptr(), im.shape[1], im.shape[0], 1, p.data_ptr()) for d, im, p in zip(d_imgs, imgs, d_pays)]
        streams = [torch.cuda.Stream(device=dev) for _ in range(2)]
        torch.cuda.synchronize()
        for rep in range(3):
            ctx.compress_device_images(table, TYPE_U8, stream=streams[0].cuda_stream)
            ctx.compress_device(d_whole_img.data_ptr(), TYPE_U8, 310, 300, d_whole.data_ptr(), stream=streams[1].cuda_stream)
        torch.cuda.synchronize()
        for k, (p, w) in enumerate(zip(d_pays, want)):
            assert np.array_equal(p.cpu().numpy(), w), "image %d" % k
        assert np.array_equal(d_whole.cpu().numpy(), want_whole)
    finally:
        ctx.close()
