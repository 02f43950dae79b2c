"""Volumes, texture arrays and the alpha-scale pre-pass through the multi-GPU entry points (astcenc_b200_compress_image_sharded,
astcenc_b200_compress_batch).

CPU: the library's slab arithmetic (astc_host_slab.h) and the pre-pass over one slab's window (alpha_window,
alpha_average_tile), compiled for the host by tests/hostsim/hostsim_slab.cpp. The window's averages must equal a whole-image run
bit for bit while every row outside the window holds poison.
GPU: every case gives the bytes of astcenc_compress_image on the same context; with two or more GPUs,
tests/sharded_volumes_worker.py runs the same over NCCL."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import astc_images as I
from astc_ref import *  # noqa: F401,F403

S = FLG_SELF_DECOMPRESS_ONLY
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "astc-encoder_b200", "csrc")
_DT = {np.dtype(np.uint8): TYPE_U8, np.dtype(np.float16): TYPE_F16, np.dtype(np.float32): TYPE_F32}
TILE = 32


def alpha_window_rows(dim_y, radius, y0, y1):
    """Image rows [read0, read1) that the pre-pass over the 32-row tiles covering rows [y0, y1) reads (alpha_window)."""
    t0, t1 = y0 // TILE, (y1 + TILE - 1) // TILE
    return max(0, t0 * TILE - radius), min(dim_y, t1 * TILE + radius)


def slab_rows(rows, world, g):
    return rows * g // world, rows * (g + 1) // world


_SIM = []


def slab_sim():
    """tests/hostsim/hostsim_slab.cpp compiled for the host."""
    if _SIM:
        return _SIM[0]
    so = os.path.join(HERE, "_build", "libhostsim_slab.so")
    src = os.path.join(HERE, "hostsim", "hostsim_slab.cpp")
    newest = max([os.path.getmtime(os.path.join(CSRC, f)) for f in os.listdir(CSRC)] + [os.path.getmtime(src)])
    if not os.path.exists(so) or os.path.getmtime(so) < newest:
        os.makedirs(os.path.dirname(so), exist_ok=True)
        r = subprocess.run(["g++", "-std=c++14", "-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-shared", "-x", "c++", src, "-o", so],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(so)
    u4 = C.POINTER(C.c_uint)
    lib.hostsim_alpha_window.argtypes = [C.c_uint, C.c_uint, C.c_uint, C.c_uint, u4]
    lib.hostsim_alpha_averages.argtypes = [C.c_void_p, C.c_int, C.c_uint, C.c_uint, C.POINTER(C.c_int), C.c_uint, C.c_uint, C.c_uint, C.c_void_p]
    lib.hostsim_slab_of.argtypes = [C.c_uint, C.c_int, C.c_int, u4]
    lib.hostsim_slab_slices.argtypes = [C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.c_uint, u4]
    lib.hostsim_slab_part.argtypes = [C.c_uint, C.c_uint, C.c_uint, C.c_uint, u4]
    lib.hostsim_image_rows.argtypes = [C.c_uint, C.c_uint, C.c_uint, C.c_uint, u4]
    lib.hostsim_band_of.argtypes = [C.c_uint, C.c_int, C.c_int, u4]
    _SIM.append(lib)
    return lib


def _call(fn, *args, n=2):
    out = (C.c_uint * n)()
    fn(*args, out)
    return tuple(out)


def sim_averages(lib, img, radius, tile_row0, tile_rows):
    """Averages of tile rows [tile_row0, tile_row0 + tile_rows); every other texel stays NaN."""
    img = np.ascontiguousarray(img)
    h, w = img.shape[:2]
    out = np.full((h, w), np.nan, np.float32)
    lib.hostsim_alpha_averages(img.ctypes.data, _DT[img.dtype], w, h, None, radius, tile_row0, tile_rows, out.ctypes.data)
    return out


def _alpha_image(h, w, dtype, seed):
    """Alpha everywhere below opaque (the poison), varied down to single texels."""
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (h, w, 4)).astype(np.uint8)
    img[..., 3] = (I.alpha_mask(h, w, seed)[..., 3] // 2) ^ rng.integers(0, 64, (h, w)).astype(np.uint8)
    return img if dtype == np.uint8 else (img.astype(np.float32) / 255.0).astype(dtype)


def _opaque(dtype):
    return 255 if dtype == np.uint8 else 1.0


# (dim_x, dim_y, block_y, world): slab borders off the 32-row grid, one-tile windows, images smaller than one tile
WINDOW_CASES = [
    (70, 200, 6, 3),        # borders at block rows 11 and 22: image rows 66 and 132
    (45, 161, 5, 4),        # ragged last tile (161 = 5 * 32 + 1)
    (64, 128, 4, 16),       # slabs of two block rows: one-tile windows
    (20, 13, 5, 2),         # smaller than one tile
    (33, 40, 12, 6),        # more ranks than block rows: empty slabs
]


@pytest.mark.parametrize("dtype", [np.uint8, np.float32], ids=["u8", "f32"])
@pytest.mark.parametrize("radius", [1, 5, 17])
@pytest.mark.parametrize("case", WINDOW_CASES, ids=["%dx%d_b%d_w%d" % c for c in WINDOW_CASES])
def test_windowed_pre_pass_equals_whole_image_run(case, radius, dtype):
    lib = slab_sim()
    w, h, by, world = case
    img = _alpha_image(h, w, dtype, seed=w * 7 + h + radius)
    tiles_y = (h + TILE - 1) // TILE
    whole = sim_averages(lib, img, radius, 0, tiles_y)
    assert not np.isnan(whole).any()
    blocks_y = (h + by - 1) // by
    covered = 0
    for g in range(world):
        r0, r1 = slab_rows(blocks_y, world, g)
        if r1 == r0:
            continue
        y0, y1 = r0 * by, min(r1 * by, h)
        t0, nt, read0, read1 = _call(lib.hostsim_alpha_window, h, radius, y0, y1, n=4)
        assert (t0, t0 + nt) == (y0 // TILE, (y1 + TILE - 1) // TILE)
        assert (read0, read1) == alpha_window_rows(h, radius, y0, y1)
        poisoned = img.copy()
        poisoned[:read0] = _opaque(dtype)
        poisoned[read1:] = _opaque(dtype)
        got = sim_averages(lib, poisoned, radius, t0, nt)
        # the slab's texels, bit for bit; nothing written outside the window's tiles
        assert np.array_equal(got[y0:y1].view(np.uint32), whole[y0:y1].view(np.uint32)), (g, y0, y1)
        assert np.isnan(got[:t0 * TILE]).all() and np.isnan(got[(t0 + nt) * TILE:]).all()
        covered += y1 - y0
        # the window is tight: its first and last rows are read
        for row in {read0, read1 - 1}:
            edge = poisoned.copy()
            edge[row] = _opaque(dtype)
            assert not np.array_equal(sim_averages(lib, edge, radius, t0, nt)[t0 * TILE:(t0 + nt) * TILE],
                                      got[t0 * TILE:(t0 + nt) * TILE], equal_nan=True), (g, row)
    assert covered == h


# (dim_z, blocks_y, block_z): volumes (block_z > 1) and texture arrays (block_z = 1)
SPLIT_CASES = [(7, 5, 3), (10, 3, 4), (6, 6, 6), (4, 1, 4), (3, 4, 1), (5, 1, 1), (1, 9, 1)]


@pytest.mark.parametrize("case", SPLIT_CASES, ids=["z%d_by%d_bz%d" % c for c in SPLIT_CASES])
def test_combined_rows_split_into_slices_and_rows(case):
    lib = slab_sim()
    dim_z, blocks_y, bz = case
    layers = (dim_z + bz - 1) // bz
    rows = layers * blocks_y
    for world in (1, 2, 3, 5, rows + 3):
        seen = []
        for g in range(world):
            r0, r1 = _call(lib.hostsim_slab_of, rows, world, g)
            assert (r0, r1) == slab_rows(rows, world, g)
            if r1 == r0:
                continue
            z0, z1 = _call(lib.hostsim_slab_slices, r0, r1, blocks_y, bz, dim_z)
            need = sorted({z for r in range(r0, r1) for z in range((r // blocks_y) * bz, min((r // blocks_y + 1) * bz, dim_z))})
            assert list(range(z0, z1)) == need, (world, g)
            # per layer (or slice) s: its part of the slab, in order, without gaps
            parts = []
            for s in range(r0 // blocks_y, (r1 + blocks_y - 1) // blocks_y):
                a, b = _call(lib.hostsim_slab_part, r0, r1, blocks_y, s)
                assert 0 <= a < b <= blocks_y
                parts += [s * blocks_y + k for k in range(a, b)]
            assert parts == list(range(r0, r1))
            seen += parts
        assert seen == list(range(rows))


# ---- GPU: one H100, world of one ----

@pytest.fixture(scope="module")
def gpu(pkg):
    import torch
    assert torch.cuda.is_available(), "these tests need a CUDA device"
    return pkg


FOOTPRINTS_3D = [(3, 3, 3), (4, 3, 3), (4, 4, 3), (4, 4, 4), (5, 4, 4), (5, 5, 4), (5, 5, 5), (6, 5, 5), (6, 6, 5), (6, 6, 6)]


def _volume(d, h, w, seed, hdr=False):
    if hdr:
        return np.stack([I.hdr_noise(h, w, seed=seed + z) for z in range(d)])
    return np.stack([I.photo_like(h, w, seed=seed + z) for z in range(d)])


def _check_world_of_one(gpu, cfg, imgs):
    """Slab mode on every image and batch mode over all of them equal astcenc_compress_image on the same context."""
    ctx = gpu.Context(cfg)
    try:
        ctx.comm_init(0, 1)
        want = [ctx.compress_image(im).copy() for im in imgs]
        for im, w in zip(imgs, want):
            assert np.array_equal(ctx.compress_image_sharded(im), w)
            assert ctx.last_timing()[1] == im.nbytes
        outs = [np.full_like(w, 0xA5) for w in want]
        ctx.compress_batch(imgs, outs)
        for o, w in zip(outs, want):
            assert np.array_equal(o, w)
        assert ctx.last_timing()[1] == sum(im.nbytes for im in imgs)
    finally:
        ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fp", FOOTPRINTS_3D, ids=["%dx%dx%d" % f for f in FOOTPRINTS_3D])
def test_3d_footprints_fastest_world_of_one(gpu, fp):
    cfg = gpu.config_init(PRF_LDR, fp[0], fp[1], PRE_FASTEST, S, block_z=fp[2])
    # 23 x 17 x 7: ragged in x, y and z for every footprint
    _check_world_of_one(gpu, cfg, [_volume(7, 17, 23, seed=10 * k + fp[0]) for k in range(3)])


@pytest.mark.gpu
@pytest.mark.parametrize("prof", [PRF_LDR, PRF_HDR], ids=["ldr", "hdr"])
@pytest.mark.parametrize("b", [4, 6])
def test_3d_footprints_medium_world_of_one(gpu, prof, b):
    cfg = gpu.config_init(prof, b, b, PRE_MEDIUM, S, block_z=b)
    _check_world_of_one(gpu, cfg, [_volume(9, 30, 41, seed=7 * k + b, hdr=prof == PRF_HDR) for k in range(2)])


@pytest.mark.gpu
def test_texture_array_world_of_one(gpu):
    cfg = gpu.config_init(PRF_LDR, 6, 6, PRE_MEDIUM, S)
    _check_world_of_one(gpu, cfg, [_volume(3, 50, 61, seed=30 + 5 * k) for k in range(3)])


@pytest.mark.gpu
@pytest.mark.parametrize("radius", [1, 4, 8])
def test_alpha_scale_2d_world_of_one(gpu, radius):
    cfg = gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, S | FLG_USE_ALPHA_WEIGHT, a_scale_radius=radius)
    _check_world_of_one(gpu, cfg, [I.alpha_mask(150, 131, seed=radius + k) for k in range(3)])


@pytest.mark.gpu
def test_device_slabs_read_only_their_alpha_window(gpu):
    """astcenc_b200_compress_device slab by slab with radius 8: each slab's pass filters only its window, so an image that
    holds poison outside the window gives the slab's bytes of the whole-image pass."""
    import torch
    radius, h, w = 8, 250, 300
    cfg = gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, S | FLG_USE_ALPHA_WEIGHT, a_scale_radius=radius)
    ctx = gpu.Context(cfg)
    try:
        img = I.alpha_mask(h, w, seed=5)
        want = ctx.compress_image(img).copy()
        nbx, nby = ctx.blocks(w, h)
        # the radius matters on this image: without it the payload differs
        plain = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, S | FLG_USE_ALPHA_WEIGHT))
        assert not np.array_equal(plain.compress_image(img), want)
        plain.close()
        for r0, r1 in ((0, 7), (7, 19), (19, 30), (30, nby), (12, 13)):
            y0, y1 = r0 * 6, min(r1 * 6, h)
            read0, read1 = alpha_window_rows(h, radius, y0, y1)
            poisoned = img.copy()
            poisoned[:read0] = 255
            poisoned[read1:] = 255
            d_img = torch.from_numpy(poisoned).cuda()
            d_out = torch.zeros((r1 - r0) * nbx * 16, dtype=torch.uint8, device="cuda")
            ctx.compress_device(d_img.data_ptr(), gpu.TYPE_U8, w, h, d_out.data_ptr(), block_row0=r0, block_rows=r1 - r0)
            torch.cuda.synchronize()
            assert np.array_equal(d_out.cpu().numpy(), want[r0 * nbx * 16:r1 * nbx * 16]), (r0, r1)
    finally:
        ctx.close()


@pytest.mark.gpu
def test_error_codes(gpu):
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FASTEST, S))
    try:
        ctx.comm_init(0, 1)
        arr = _volume(3, 20, 20, seed=1)
        with pytest.raises(gpu.AstcencError) as e:
            ctx.compress_batch([arr, arr[:2]], [np.zeros(4 * 4 * 3 * 16, np.uint8)] * 2)
        assert e.value.code == gpu.ERR_BAD_PARAM
        with pytest.raises(gpu.AstcencError) as e:
            ctx.compress_image_sharded(arr, out=np.zeros(4 * 4 * 2 * 16, np.uint8))
        assert e.value.code == gpu.ERR_OUT_OF_MEM
        with pytest.raises(gpu.AstcencError) as e:
            ctx.compress_batch([arr], [np.zeros(4 * 4 * 2 * 16, np.uint8)])
        assert e.value.code == gpu.ERR_OUT_OF_MEM
    finally:
        ctx.close()
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FASTEST, S, a_scale_radius=2))
    try:
        ctx.comm_init(0, 1)
        with pytest.raises(gpu.AstcencError) as e:
            ctx.compress_image_sharded(arr)
        assert e.value.code == gpu.ERR_NOT_IMPLEMENTED
        with pytest.raises(gpu.AstcencError) as e:
            ctx.compress_batch([arr], [np.zeros(4 * 4 * 3 * 16, np.uint8)])
        assert e.value.code == gpu.ERR_NOT_IMPLEMENTED
    finally:
        ctx.close()


# ---- GPU: two or more H100s ----

@pytest.mark.gpu
def test_ranks_nccl_volumes_arrays_and_alpha_windows(gpu, tmp_path):
    """Every GPU of the box (skipped with fewer than two): slab borders inside a layer and inside a slice, more ranks than
    combined rows, radius 8 with borders off the tile grid, batches of volumes with a ragged last round, and every rank's
    uploaded bytes; the root's payloads equal one GPU's."""
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs two GPUs")
    script = os.path.join(HERE, "sharded_volumes_worker.py")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=%d" % min(n, 4), "--master-addr", "127.0.0.1",
                        "--master-port", "29617", script, str(tmp_path)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert os.path.exists(os.path.join(str(tmp_path), "ok"))
