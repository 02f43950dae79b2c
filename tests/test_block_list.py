"""Block lists: astcenc_b200_compress_device_blocks recompresses the listed blocks of a device-resident image in place in its
device-resident payload (gather into a staging row of blocks, one ordinary pass, scatter; astc_dev_gather.cuh).

CPU: the gather's addressing (tests/hostsim/hostsim_blocks.cpp compiles astc_dev_gather.cuh for the host) against a numpy
restatement of load_block's clamp-to-edge, and the device source's pass over the staging image (one lane and 32 lanes) against
the oracle's whole-image blocks at the listed positions.
GPU: the C ABI against astcenc_compress_image / compress_device / the reference build on the same images: listed blocks equal,
every other payload byte untouched."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import astc_images as I
from astc_ref import *  # noqa: F401,F403

S = FLG_SELF_DECOMPRESS_ONLY
HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "astc-encoder_b200", "csrc")
_DT = {np.dtype(np.uint8): TYPE_U8, np.dtype(np.float16): TYPE_F16, np.dtype(np.float32): TYPE_F32}
_SIMS = {}


def blocks_sim(lanes32=False):
    """tests/hostsim/hostsim_blocks.cpp compiled for the host (one simulated lane, or 32 lanes on 32 threads)."""
    if lanes32 in _SIMS:
        return _SIMS[lanes32]
    so = os.path.join(HERE, "_build", "libhostsim_blocks%s.so" % ("32" if lanes32 else ""))
    hs = os.path.join(HERE, "hostsim")
    newest = max([os.path.getmtime(os.path.join(CSRC, f)) for f in os.listdir(CSRC)] + [os.path.getmtime(os.path.join(hs, f)) for f in os.listdir(hs)])
    if not os.path.exists(so) or os.path.getmtime(so) < newest:
        os.makedirs(os.path.dirname(so), exist_ok=True)
        cmd = ["g++", "-std=c++14", "-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-shared"] + \
              (["-pthread", "-DASTC_HOSTSIM_LANES32=1"] if lanes32 else []) + \
              ["-x", "c++", os.path.join(hs, "hostsim_blocks.cpp"), os.path.join(CSRC, "astc_host_tables.cpp"), os.path.join(CSRC, "astc_host_config.cpp"), "-o", so]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(so)
    lib.hostsim_gather.argtypes = [C.c_void_p, C.c_int, C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.c_void_p, C.c_uint, C.c_void_p,
                                   C.c_void_p, C.c_void_p]
    lib.hostsim_alpha_averages_2d.argtypes = [C.c_void_p, C.c_int, C.c_uint, C.c_uint, C.c_void_p, C.c_uint, C.c_void_p]
    lib.hostsim_compress_staged.argtypes = [C.c_int, C.c_uint, C.c_uint, C.c_uint, C.c_float, C.c_uint, C.c_uint, C.c_void_p, C.c_int, C.c_uint, C.c_uint,
                                            C.c_uint, C.c_void_p, C.c_void_p]
    assert lib.hostsim_lanes() == (32 if lanes32 else 1)
    _SIMS[lanes32] = lib
    return lib


def grid(shape, fp):
    """(blocks_x, blocks_y, layers) of a (D, H, W, 4) image: layers = slices for 2D footprints, layers of blocks for 3D ones."""
    d, h, w = shape[:3]
    return -(-w // fp[0]), -(-h // fp[1]), -(-d // fp[2])


def edge_blocks(shape, fp):
    nbx, nby, nl = grid(shape, fp)
    b = np.arange(nbx * nby * nl)
    col, row = b % nbx, (b // nbx) % nby
    return b[(col == nbx - 1) | (row == nby - 1)]


def random_list(rng, total, k, dups=0):
    idx = rng.choice(total, size=min(k, total), replace=False)
    if dups:
        idx = np.concatenate([idx, rng.choice(idx, size=dups)])
        rng.shuffle(idx)
    return idx.astype(np.uint32)


def staged_reference(vol, fp, idx):
    """The staging image a list gathers, restated with numpy: footprint texels of every listed block, clamped to the image's
    edges as load_block clamps them, block i at x = i * bx. (bz, by, n * bx, 4)."""
    d, h, w = vol.shape[:3]
    bx, by, bz = fp
    nbx, nby, _ = grid(vol.shape, fp)
    out = np.zeros((bz, by, len(idx) * bx, 4), vol.dtype)
    for i, b in enumerate(idx.tolist()):
        col, rest = b % nbx, b // nbx
        row, layer = rest % nby, rest // nby
        xs = np.minimum(col * bx + np.arange(bx), w - 1)
        ys = np.minimum(row * by + np.arange(by), h - 1)
        zs = np.minimum(layer * bz + np.arange(bz), d - 1)
        out[:, :, i * bx:(i + 1) * bx] = vol[zs][:, ys][:, :, xs]
    return out


def sim_gather(lib, vol, fp, idx, avg=None):
    vol = np.ascontiguousarray(vol)
    d, h, w = vol.shape[:3]
    staged = np.zeros((fp[2], fp[1], len(idx) * fp[0], 4), vol.dtype)
    savg = np.full((fp[1], len(idx) * fp[0]), -1.0, np.float32) if avg is not None else None
    lib.hostsim_gather(vol.ctypes.data, _DT[vol.dtype], w, h, d, fp[0], fp[1], fp[2], idx.ctypes.data, len(idx),
                       avg.ctypes.data if avg is not None else None, staged.ctypes.data, savg.ctypes.data if savg is not None else None)
    return staged, savg


def ldr_image(h, w, d, seed):
    return np.ascontiguousarray(I.photo_like(h * d, w, seed=seed).reshape(d, h, w, 4))


def image_of(dtype, h, w, d, seed, hdr=False):
    if hdr:
        return np.ascontiguousarray(I.hdr_noise(h * d, w, seed=seed, dtype=dtype).reshape(d, h, w, 4))
    img = ldr_image(h, w, d, seed)
    if dtype == np.uint8:
        return img
    return np.ascontiguousarray((img.astype(np.float32) / 255.0).astype(dtype))


def transparent_image(h, w, seed):
    """LDR RGBA8 with a fully transparent rectangle (blocks inside it are turned into constant zero by the alpha-scale test)
    and alpha noise elsewhere."""
    img = I.photo_like(h, w, seed=seed).copy()
    img[..., 3] = np.random.default_rng(seed).integers(0, 256, size=(h, w), dtype=np.uint8)
    img[h // 4:h // 4 + 48, w // 5:w // 5 + 64, 3] = 0
    return np.ascontiguousarray(img)


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
GATHER = [
    ("u8_2d_6x6_ragged", np.uint8, (1, 23, 37), (6, 6, 1)),
    ("f16_2d_5x4_ragged", np.float16, (1, 31, 29), (5, 4, 1)),
    ("f32_2d_12x12_ragged", np.float32, (1, 17, 13), (12, 12, 1)),
    ("u8_array3_8x8", np.uint8, (3, 19, 21), (8, 8, 1)),
    ("f16_volume_4x4x4", np.float16, (7, 9, 11), (4, 4, 4)),
    ("f32_volume_3x3x3", np.float32, (5, 8, 7), (3, 3, 3)),
    ("u8_volume_6x5x5", np.uint8, (6, 11, 13), (6, 5, 5)),
]


@pytest.mark.parametrize("case", GATHER, ids=[c[0] for c in GATHER])
def test_gather_copies_what_load_block_reads(case):
    _, dtype, shape, fp = case
    lib = blocks_sim()
    rng = np.random.default_rng(7)
    d, h, w = shape
    if dtype == np.uint8:
        vol = rng.integers(0, 256, size=(d, h, w, 4), dtype=np.uint8)
    else:
        vol = rng.standard_normal((d, h, w, 4)).astype(dtype)
    total = int(np.prod(grid(shape, fp)))
    for idx in (random_list(rng, total, total // 2 + 1, dups=3), edge_blocks(shape, fp).astype(np.uint32), np.array([total - 1], np.uint32)):
        avg = rng.random((h, w), dtype=np.float32) if d == 1 else None
        staged, savg = sim_gather(lib, vol, fp, idx, avg)
        assert np.array_equal(staged.view(np.uint8), staged_reference(vol, fp, idx).view(np.uint8))
        if avg is not None:
            # averages of texels outside the image are 0: block_has_alpha skips those texels, it does not clamp them
            padded = np.zeros((h + fp[1], w + fp[0]), np.float32)
            padded[:h, :w] = avg
            nbx = grid(shape, fp)[0]
            for i, b in enumerate(idx.tolist()):
                y0, x0 = (b // nbx) * fp[1], (b % nbx) * fp[0]
                assert np.array_equal(savg[:, i * fp[0]:(i + 1) * fp[0]], padded[y0:y0 + fp[1], x0:x0 + fp[0]])


# (name, profile, dtype, footprint, quality, a_scale_radius, lanes32)
PARITY = [
    ("ldr_u8_4x4_fast", PRF_LDR, np.uint8, (4, 4, 1), PRE_FAST, 0, False),
    ("ldr_u8_4x4_fast_32lanes", PRF_LDR, np.uint8, (4, 4, 1), PRE_FAST, 0, True),
    ("srgb_u8_6x6_medium", PRF_LDR_SRGB, np.uint8, (6, 6, 1), PRE_MEDIUM, 0, False),
    ("ldr_u8_8x8_fast", PRF_LDR, np.uint8, (8, 8, 1), PRE_FAST, 0, False),
    ("ldr_f32_12x12_fast", PRF_LDR, np.float32, (12, 12, 1), PRE_FAST, 0, False),
    ("srgb_f16_5x4_medium", PRF_LDR_SRGB, np.float16, (5, 4, 1), PRE_MEDIUM, 0, False),
    ("hdr_f16_6x6_fast", PRF_HDR, np.float16, (6, 6, 1), PRE_FAST, 0, False),
    ("hdr_rgb_ldr_a_f32_6x6_fast_32lanes", PRF_HDR_RGB_LDR_A, np.float32, (6, 6, 1), PRE_FAST, 0, True),
    ("ldr_u8_6x6_medium_radius2", PRF_LDR, np.uint8, (6, 6, 1), PRE_MEDIUM, 2, False),
    ("ldr_u8_4x4_fast_radius5_32lanes", PRF_LDR, np.uint8, (4, 4, 1), PRE_FAST, 5, True),
    ("ldr_u8_volume_4x4x4_fast", PRF_LDR, np.uint8, (4, 4, 4), PRE_FAST, 0, False),
    ("hdr_f16_volume_3x3x3_fast_32lanes", PRF_HDR, np.float16, (3, 3, 3), PRE_FAST, 0, True),
]


@pytest.mark.parametrize("case", PARITY, ids=[c[0] for c in PARITY])
def test_pass_over_staging_row_equals_whole_image(case, oracle):
    """The device source's pass over the gathered staging row gives the oracle's whole-image blocks at the listed positions."""
    _, prof, dtype, fp, q, radius, lanes32 = case
    lib = blocks_sim(lanes32)
    rng = np.random.default_rng(11)
    volume = fp[2] > 1
    if radius:
        vol = transparent_image(96, 101, 3)[None]
    else:
        shape = (9, 10, 11) if volume else (1, 29, 41)
        vol = image_of(dtype, shape[1], shape[2], shape[0], 5, hdr=prof in (PRF_HDR, PRF_HDR_RGB_LDR_A))
    d, h, w = vol.shape[:3]
    if volume:
        want = oracle.compress_volume(vol, prof, fp[0], fp[1], fp[2], q, S)
    else:
        want = oracle.compress(vol[0], prof, fp[0], fp[1], q, S, a_scale_radius=radius)
    total = len(want) // 16
    idx = random_list(rng, total, 4 if lanes32 else 10, dups=1)
    idx = np.concatenate([idx, edge_blocks(vol.shape, fp)[-1:].astype(np.uint32)])
    avg = None
    if radius:
        # blocks of the transparent rectangle, which the alpha-scale test turns into constant zero
        nbx = grid(vol.shape, fp)[0]
        inner = ((h // 4 + 16) // fp[1]) * nbx + (w // 5 + 16) // fp[0]
        idx = np.concatenate([idx, np.array([inner, inner + 1], np.uint32)])
        avg = np.zeros((h, w), np.float32)
        lib.hostsim_alpha_averages_2d(vol[0].ctypes.data, TYPE_U8, w, h, None, radius, avg.ctypes.data)
    staged, savg = sim_gather(lib, vol, fp, idx, avg)
    out = np.zeros(len(idx) * 16, np.uint8)
    rc = lib.hostsim_compress_staged(prof, fp[0], fp[1], fp[2], q, S, radius, staged.ctypes.data, _DT[staged.dtype], len(idx) * fp[0], fp[1], fp[2],
                                     savg.ctypes.data if savg is not None else None, out.ctypes.data)
    assert rc == 0
    want_blocks = want.reshape(-1, 16)[idx.astype(np.int64)]
    bad = np.nonzero(np.any(out.reshape(-1, 16) != want_blocks, axis=1))[0]
    assert len(bad) == 0, "listed blocks %s differ" % idx[bad][:8]
    if radius:
        assert np.all(want_blocks[-2:, 8:] == 0), "the list should hold constant-zero blocks"


# ---------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu(pkg):
    import torch
    assert torch.cuda.is_available(), "these tests need a CUDA device"
    return pkg


def sentinel(nbytes):
    return (np.arange(nbytes, dtype=np.uint32) * 131 + 7).astype(np.uint8)


def run_blocks(pkg, ctx, vol, idx, stream=None):
    """The payload after one block-list call on a sentinel-filled device payload."""
    import torch
    dev = torch.device("cuda", 0)
    vol = np.ascontiguousarray(vol)
    d, h, w = vol.shape[:3]
    d_img = torch.from_numpy(vol.view(np.uint8).reshape(-1)).to(dev)
    fp = (ctx.config.block_x, ctx.config.block_y, max(1, ctx.config.block_z))
    nbytes = int(np.prod(grid(vol.shape, fp))) * 16
    d_pay = torch.from_numpy(sentinel(nbytes)).to(dev)
    st = stream or torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    ctx.compress_device_blocks(d_img.data_ptr(), _DT[vol.dtype], w, h, d, idx, d_pay.data_ptr(), stream=st.cuda_stream)
    torch.cuda.synchronize()
    return d_pay.cpu().numpy()


def check(got, want, idx):
    listed = np.zeros(len(want) // 16, bool)
    listed[np.asarray(idx, np.int64)] = True
    g, w, s = got.reshape(-1, 16), want.reshape(-1, 16), sentinel(len(want)).reshape(-1, 16)
    bad = np.nonzero(np.any(g[listed] != w[listed], axis=1))[0]
    assert len(bad) == 0, "%d listed blocks differ" % len(bad)
    assert np.array_equal(g[~listed], s[~listed]), "a byte outside the listed blocks changed"


# (profile, dtype, footprint, quality)
GPU_CASES = [
    (PRF_LDR, np.uint8, (4, 4), PRE_FAST),
    (PRF_LDR, np.uint8, (6, 6), PRE_MEDIUM),
    (PRF_LDR_SRGB, np.uint8, (8, 8), PRE_THOROUGH),
    (PRF_LDR, np.float16, (12, 12), PRE_MEDIUM),
    (PRF_LDR, np.float32, (5, 4), PRE_FAST),
    (PRF_LDR_SRGB, np.uint8, (5, 4), PRE_MEDIUM),
    (PRF_HDR, np.float16, (6, 6), PRE_MEDIUM),
    (PRF_HDR, np.float32, (8, 8), PRE_FAST),
    (PRF_HDR_RGB_LDR_A, np.float32, (4, 4), PRE_THOROUGH),
    (PRF_HDR_RGB_LDR_A, np.float16, (12, 12), PRE_FAST),
]
_PN = {PRF_LDR: "ldr", PRF_LDR_SRGB: "srgb", PRF_HDR: "hdr", PRF_HDR_RGB_LDR_A: "hdr_rgb_ldr_a"}
_QN = {PRE_FAST: "fast", PRE_MEDIUM: "medium", PRE_THOROUGH: "thorough"}


@pytest.mark.gpu
@pytest.mark.parametrize("case", GPU_CASES, ids=["%s_%s_%dx%d_%s" % (_PN[c[0]], np.dtype(c[1]).name, c[2][0], c[2][1], _QN[c[3]]) for c in GPU_CASES])
def test_listed_blocks_equal_whole_image(case, gpu):
    prof, dtype, (bx, by), q = case
    vol = image_of(dtype, 150, 203, 1, 21, hdr=prof in (PRF_HDR, PRF_HDR_RGB_LDR_A))
    ctx = gpu.Context(gpu.config_init(prof, bx, by, q, S))
    try:
        want = ctx.compress_image(vol[0]).copy()
        total = len(want) // 16
        rng = np.random.default_rng(bx * 100 + by)
        lists = [rng.integers(0, total, size=1), random_list(rng, total, max(1, total // 100)), rng.permutation(total),
                 random_list(rng, total, 40, dups=25), edge_blocks(vol.shape, (bx, by, 1))]
        for idx in lists:
            check(run_blocks(gpu, ctx, vol, idx), want, idx)
    finally:
        ctx.close()


FULL = [("config1_4096_6x6_medium", "photo_like", 4096, PRF_LDR, np.uint8), ("config3_2048_hdr_6x6_medium", "hdr_noise", 2048, PRF_HDR, np.float16)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", FULL, ids=[c[0] for c in FULL])
def test_full_size_list_equals_reference_build(case, gpu, reference):
    """A seeded 1 % list of the full-size workload image gives the reference build's blocks at those positions (the stored
    answer is the whole image's digest: the whole device-resident pass is checked against it, the list against that pass)."""
    import torch
    name, gen, dim, prof, dtype = case
    img = getattr(I, gen)(dim, dim, seed=2024)
    ctx = gpu.Context(gpu.config_init(prof, 6, 6, PRE_MEDIUM, S))
    try:
        dev = torch.device("cuda", 0)
        d_img = torch.from_numpy(np.ascontiguousarray(img).view(np.uint8).reshape(-1)).to(dev)
        nbx, nby = ctx.blocks(dim, dim)
        d_whole = torch.zeros(nbx * nby * 16, dtype=torch.uint8, device=dev)
        st = torch.cuda.Stream(device=dev)
        ctx.compress_device(d_img.data_ptr(), _DT[img.dtype], dim, dim, d_whole.data_ptr(), stream=st.cuda_stream)
        torch.cuda.synchronize()
        whole = d_whole.cpu().numpy()
        assert len(block_diff(whole, reference.compress(img, prof, 6, 6, PRE_MEDIUM, S))) == 0
        idx = random_list(np.random.default_rng(2024), nbx * nby, nbx * nby // 100)
        check(run_blocks(gpu, ctx, img[None], idx), whole, idx)
    finally:
        ctx.close()


FOOTPRINTS_3D = [(3, 3, 3), (4, 3, 3), (4, 4, 3), (4, 4, 4), (5, 4, 4), (5, 5, 4), (5, 5, 5), (6, 5, 5), (6, 6, 5), (6, 6, 6)]


@pytest.mark.gpu
def test_texture_arrays_and_volumes_equal_compress_image(gpu):
    rng = np.random.default_rng(3)
    arr = ldr_image(41, 53, 3, 9)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_MEDIUM, S))
    try:
        want = ctx.compress_image(arr).copy()
        total = len(want) // 16
        for idx in (random_list(rng, total, total // 3, dups=4), edge_blocks(arr.shape, (6, 6, 1)), rng.permutation(total)):
            check(run_blocks(gpu, ctx, arr, idx), want, idx)
    finally:
        ctx.close()
    for fp in FOOTPRINTS_3D:
        vol = ldr_image(17, 19, 11, fp[0] * 10 + fp[2])
        for prof, v in ((PRF_LDR, vol), (PRF_HDR, image_of(np.float16, 17, 19, 11, 4, hdr=True))):
            ctx = gpu.Context(gpu.config_init(prof, fp[0], fp[1], PRE_FAST, S, block_z=fp[2]))
            try:
                want = ctx.compress_image(v).copy()
                total = len(want) // 16
                for idx in (random_list(rng, total, total // 4 + 1, dups=2), edge_blocks(v.shape, fp), rng.permutation(total)):
                    check(run_blocks(gpu, ctx, v, idx), want, idx)
            finally:
                ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("radius", [1, 5, 17])
def test_alpha_scale_lists_equal_compress_image(radius, gpu):
    img = transparent_image(300, 259, radius)
    rng = np.random.default_rng(radius)
    for bx, by in ((6, 6), (4, 4)):
        cfg = gpu.config_init(PRF_LDR, bx, by, PRE_MEDIUM, S | FLG_USE_ALPHA_WEIGHT)
        cfg.a_scale_radius = radius
        ctx = gpu.Context(cfg)
        try:
            want = ctx.compress_image(img).copy()
            wb = want.reshape(-1, 16)
            zero = np.nonzero(np.all(wb[:, 8:] == 0, axis=1) & (wb[:, 0] == 0xFC))[0]
            assert len(zero) > 0
            total = len(wb)
            for idx in (np.concatenate([random_list(rng, total, total // 20), zero[::3].astype(np.uint32)]), edge_blocks(img[None].shape, (bx, by, 1)),
                        rng.permutation(total)):
                check(run_blocks(gpu, ctx, img[None], idx), want, idx)
        finally:
            ctx.close()


@pytest.mark.gpu
def test_lists_longer_than_one_batch(gpu):
    """A list longer than ASTCENC_B200_BATCH_BLOCKS (read when the context is made) runs as several staging rows: same bytes."""
    img = image_of(np.uint8, 90, 130, 1, 8)
    rng = np.random.default_rng(5)
    old = os.environ.get("ASTCENC_B200_BATCH_BLOCKS")
    os.environ["ASTCENC_B200_BATCH_BLOCKS"] = "37"
    try:
        ctx = gpu.Context(gpu.config_init(PRF_LDR, 5, 4, PRE_MEDIUM, S))
    finally:
        if old is None:
            del os.environ["ASTCENC_B200_BATCH_BLOCKS"]
        else:
            os.environ["ASTCENC_B200_BATCH_BLOCKS"] = old
    try:
        want = ctx.compress_image(img[0]).copy()
        total = len(want) // 16
        for idx in (random_list(rng, total, 200, dups=10), rng.permutation(total)):
            check(run_blocks(gpu, ctx, img, idx), want, idx)
    finally:
        ctx.close()


@pytest.mark.gpu
def test_errors_launch_nothing_and_write_nothing(gpu):
    import torch
    dev = torch.device("cuda", 0)
    img = image_of(np.uint8, 40, 44, 2, 1)
    d_img = torch.from_numpy(img.reshape(-1)).to(dev)
    nbytes = 8 * 7 * 2 * 16
    d_pay = torch.from_numpy(sentinel(nbytes)).to(dev)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, S))
    cfg_r = gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, S)
    cfg_r.a_scale_radius = 2
    ctx_r = gpu.Context(cfg_r)
    ctx_d = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, gpu.FLG_DECOMPRESS_ONLY))

    def expect(c, code, **kw):
        a = dict(d_pixels_ptr=d_img.data_ptr(), data_type=TYPE_U8, dim_x=44, dim_y=40, dim_z=2, indices=[0, 5], d_payload_ptr=d_pay.data_ptr())
        a.update(kw)
        n0 = c.launch_count()
        if code == 0:
            c.compress_device_blocks(**a)
        else:
            with pytest.raises(gpu.AstcencError) as e:
                c.compress_device_blocks(**a)
            assert e.value.code == code
        torch.cuda.synchronize()
        assert c.launch_count() == n0
        assert np.array_equal(d_pay.cpu().numpy(), sentinel(nbytes))

    try:
        expect(ctx, gpu.ERR_BAD_PARAM, indices=[3, nbytes // 16])
        expect(ctx, gpu.ERR_BAD_PARAM, indices=[-1])
        expect(ctx, gpu.ERR_BAD_PARAM, d_pixels_ptr=0)
        expect(ctx, gpu.ERR_BAD_PARAM, d_payload_ptr=0)
        expect(ctx, gpu.ERR_BAD_PARAM, dim_z=0)
        expect(ctx, gpu.ERR_BAD_SWIZZLE, swizzle=(0, 1, 2, 9))
        expect(ctx_d, gpu.ERR_BAD_CONTEXT)
        expect(ctx_r, gpu.ERR_NOT_IMPLEMENTED)
        expect(ctx_r, gpu.ERR_NOT_IMPLEMENTED, indices=[10 ** 6])      # (the radius check comes before the list's)
        expect(ctx, 0, indices=[])
    finally:
        ctx.close()
        ctx_r.close()
        ctx_d.close()


@pytest.mark.gpu
def test_list_and_whole_image_passes_on_two_streams_are_ordered(gpu):
    """Block-list calls and compress_device calls of ONE context on two streams share its scratch: the library orders them."""
    import torch
    dev = torch.device("cuda", 0)
    cfg = gpu.config_init(PRF_LDR, 6, 6, PRE_MEDIUM, S)
    ctx = gpu.Context(cfg)
    try:
        imgs = [I.photo_like(300, 310, seed=s) for s in (1, 2)]
        want = [ctx.compress_image(im).copy() for im in imgs]
        d_imgs = [torch.from_numpy(im).to(dev) for im in imgs]
        nbx, nby = ctx.blocks(310, 300)
        total = nbx * nby
        d_list = torch.from_numpy(sentinel(total * 16)).to(dev)
        d_whole = torch.zeros(total * 16, dtype=torch.uint8, device=dev)
        streams = [torch.cuda.Stream(device=dev) for _ in range(2)]
        idx = np.random.default_rng(1).permutation(total)[:total // 2]
        torch.cuda.synchronize()
        for rep in range(3):
            ctx.compress_device_blocks(d_imgs[0].data_ptr(), TYPE_U8, 310, 300, 1, idx, d_list.data_ptr(), stream=streams[0].cuda_stream)
            ctx.compress_device(d_imgs[1].data_ptr(), TYPE_U8, 310, 300, d_whole.data_ptr(), stream=streams[1].cuda_stream)
        torch.cuda.synchronize()
        check(d_list.cpu().numpy(), want[0], idx)
        assert np.array_equal(d_whole.cpu().numpy(), want[1])
    finally:
        ctx.close()
