"""The launch plan of a compression pass: how a pass is cut into upload bands and sub-slab pipelines, and what it enqueues.

CPU: the band, pipe and image-row arithmetic of the host pass code (astc_host_slab.h), compiled for the host by
tests/hostsim/hostsim_slab.cpp.
GPU: per entry point and knob setting, the kernel launches a pass makes (astcenc_b200_launch_count), the launches per kernel
kind of its stage timing (astcenc_b200_stage_timing) and the bytes it moves (astcenc_b200_last_timing). The expected values
are literals: a change to the host pass code that adds, drops or reorders work shows up here before it shows up as a timing
or parity difference."""

import numpy as np
import pytest

import astc_images as I
from astc_ref import *  # noqa: F401,F403
from test_sharded_volumes import _call, slab_sim

S = FLG_SELF_DECOMPRESS_ONLY
SHARES = [1, 3, 4, 8, 8, 8, 8, 8]      # the first band is short: its copy is the only one nothing hides


def _bands(lib, rows, bands):
    """[(first, last)] of the bands that are launched, and the boundaries of all of them."""
    launched, ends = [], []
    for k in range(bands):
        a, b, on = _call(lib.hostsim_band_of, rows, bands, k, n=3)
        assert on == (b > a), (rows, bands, k)
        ends.append(b)
        if on:
            launched.append((a, b))
    return launched, ends


def test_bands_tile_the_slab_in_share_order():
    lib = slab_sim()
    for bands in range(1, 9):
        total = sum(SHARES[:bands])
        for rows in range(1, 3001):
            launched, ends = _bands(lib, rows, bands)
            # in order, without gaps or overlaps, no launched band empty
            assert launched[0][0] == 0 and launched[-1][1] == rows, (rows, bands)
            assert all(b0[1] == b1[0] for b0, b1 in zip(launched, launched[1:])), (rows, bands)
            assert all(a < b for a, b in launched)
            # the boundaries follow the shares; the last band takes the rest
            acc = np.cumsum(SHARES[:bands])
            assert ends == [rows * int(c) // total for c in acc[:-1]] + [rows], (rows, bands)


def test_pipes_tile_the_slab():
    lib = slab_sim()
    for pipes in range(1, 9):
        for rows in range(1, 3001):
            parts = [_call(lib.hostsim_slab_of, rows, pipes, p) for p in range(pipes)]
            assert parts[0][0] == 0 and parts[-1][1] == rows
            assert all(p0[1] == p1[0] and p0[0] <= p0[1] for p0, p1 in zip(parts, parts[1:]))
            assert all(a == rows * p // pipes for p, (a, _) in enumerate(parts))


def test_image_rows_of_block_rows():
    lib = slab_sim()
    for by in (4, 5, 6, 8, 12):
        for dim_y in list(range(1, 40)) + [1000, 1001, 2999, 3000]:
            blocks_y = -(-dim_y // by)
            for r0 in range(0, blocks_y, max(1, blocks_y // 7)):
                for r1 in range(r0 + 1, blocks_y + 1, max(1, blocks_y // 5)):
                    assert _call(lib.hostsim_image_rows, r0, r1, by, dim_y) == (r0 * by, min(r1 * by, dim_y)), (by, dim_y, r0, r1)


# ---- GPU: the launch plan of each entry point, pinned ----

@pytest.fixture(scope="module")
def gpu(pkg):
    import torch
    assert torch.cuda.is_available(), "these tests need a CUDA device"
    return pkg


def _context(gpu, monkeypatch, env, prof, bx, by, q, bz=1, radius=0):
    for k, v in env.items():
        monkeypatch.setenv("ASTCENC_B200_" + k, v)      # (the knobs are read when the context is made)
    cfg = gpu.config_init(prof, bx, by, q, S | (FLG_USE_ALPHA_WEIGHT if radius else 0), block_z=bz, a_scale_radius=radius)
    ctx = gpu.Context(cfg)
    for k in env:
        monkeypatch.delenv("ASTCENC_B200_" + k)
    return ctx


def _device(gpu, ctx, img, r0=0, rows=None):
    import torch
    h, w = img.shape[:2]
    nbx, nby = ctx.blocks(w, h)
    rows = nby - r0 if rows is None else rows
    d_img = torch.from_numpy(np.ascontiguousarray(img)).cuda()
    d_out = torch.zeros(rows * nbx * 16, dtype=torch.uint8, device="cuda")
    dt = {np.dtype(np.uint8): TYPE_U8, np.dtype(np.float16): TYPE_F16, np.dtype(np.float32): TYPE_F32}[img.dtype]
    ctx.compress_device(d_img.data_ptr(), dt, w, h, d_out.data_ptr(), block_row0=r0, block_rows=rows)
    torch.cuda.synchronize()


def _blocks(gpu, ctx, img, idx):
    import torch
    img = np.ascontiguousarray(img if img.ndim == 4 else img[None])
    d, h, w = img.shape[:3]
    nbx, nby = ctx.blocks(w, h)
    d_img = torch.from_numpy(img.reshape(-1)).cuda()
    d_pay = torch.zeros(nbx * nby * d * 16, dtype=torch.uint8, device="cuda")
    ctx.compress_device_blocks(d_img.data_ptr(), TYPE_U8, w, h, d, idx, d_pay.data_ptr())
    torch.cuda.synchronize()


def _world_of_one(ctx, what, img):
    ctx.comm_init(0, 1)
    if what == "sharded":
        ctx.compress_image_sharded(img)
    else:
        ctx.compress_batch([img, img], [np.empty(ctx._image(img)[3], np.uint8) for _ in range(2)])


_RNG_LIST = np.random.default_rng(5).permutation(26 * 23)[:200]

# name -> (context: env, profile, block x / y, quality, block z, radius; call)
CASES = {
    "device_6x6_medium": (({}, PRF_LDR, 6, 6, PRE_MEDIUM), lambda g, c: _device(g, c, I.photo_like(96, 96, seed=3))),
    "device_4x4_fast": (({}, PRF_LDR, 4, 4, PRE_FAST), lambda g, c: _device(g, c, I.photo_like(64, 80, seed=4))),
    "device_hdr_6x6_medium": (({}, PRF_HDR, 6, 6, PRE_MEDIUM), lambda g, c: _device(g, c, I.hdr_noise(60, 70, seed=5))),
    "image_bands1_ragged": (({"UPLOAD_BANDS": "1"}, PRF_LDR, 6, 6, PRE_FAST), lambda g, c: c.compress_image(I.photo_like(1001, 333, seed=6))),
    "image_bands4_ragged": (({"UPLOAD_BANDS": "4"}, PRF_LDR, 6, 6, PRE_FAST), lambda g, c: c.compress_image(I.photo_like(1001, 333, seed=6))),
    "image_bands8_ragged": (({"UPLOAD_BANDS": "8"}, PRF_LDR, 6, 6, PRE_FAST), lambda g, c: c.compress_image(I.photo_like(1001, 333, seed=6))),
    "image_bands8_too_small": (({"UPLOAD_BANDS": "8"}, PRF_LDR, 6, 6, PRE_FAST), lambda g, c: c.compress_image(I.photo_like(40, 64, seed=7))),
    "device_pipes2": (({"PIPES": "2"}, PRF_LDR, 5, 5, PRE_FAST), lambda g, c: _device(g, c, I.photo_like(700, 1210, seed=8))),
    "image_pipes4": (({"PIPES": "4"}, PRF_LDR, 5, 5, PRE_FAST), lambda g, c: c.compress_image(I.photo_like(1500, 1210, seed=8))),
    "device_three_batches": (({"BATCH_BLOCKS": "112"}, PRF_LDR, 6, 6, PRE_MEDIUM), lambda g, c: _device(g, c, I.photo_like(120, 96, seed=9))),
    "image_three_batches": (({"BATCH_BLOCKS": "112"}, PRF_LDR, 6, 6, PRE_MEDIUM), lambda g, c: c.compress_image(I.photo_like(120, 96, seed=9))),
    "image_radius5": (({}, PRF_LDR, 6, 6, PRE_FAST, 1, 5), lambda g, c: c.compress_image(I.alpha_mask(150, 131, seed=10))),
    "device_slab_radius5": (({}, PRF_LDR, 6, 6, PRE_FAST, 1, 5), lambda g, c: _device(g, c, I.alpha_mask(150, 131, seed=10), r0=7, rows=12)),
    "image_volume_4x4x4": (({}, PRF_LDR, 4, 4, PRE_FAST, 4), lambda g, c: c.compress_image(_volume(9, 30, 41))),
    "sharded_volume_4x4x4": (({}, PRF_LDR, 4, 4, PRE_FAST, 4), lambda g, c: _world_of_one(c, "sharded", _volume(9, 30, 41))),
    "batch_volume_4x4x4": (({}, PRF_LDR, 4, 4, PRE_FAST, 4), lambda g, c: _world_of_one(c, "batch", _volume(9, 30, 41))),
    "image_array_6x6": (({}, PRF_LDR, 6, 6, PRE_FAST), lambda g, c: c.compress_image(_volume(3, 50, 61))),
    "sharded_array_6x6": (({}, PRF_LDR, 6, 6, PRE_FAST), lambda g, c: _world_of_one(c, "sharded", _volume(3, 50, 61))),
    "batch_array_6x6": (({}, PRF_LDR, 6, 6, PRE_FAST), lambda g, c: _world_of_one(c, "batch", _volume(3, 50, 61))),
    "batch_image_6x6": (({}, PRF_LDR, 6, 6, PRE_FAST), lambda g, c: _world_of_one(c, "batch", I.photo_like(100, 90, seed=11))),
    "blocks_long_list": (({"BATCH_BLOCKS": "37"}, PRF_LDR, 5, 4, PRE_MEDIUM), lambda g, c: _blocks(g, c, I.photo_like(90, 130, seed=12), _RNG_LIST)),
    "blocks_long_list_radius3": (({"BATCH_BLOCKS": "37"}, PRF_LDR, 5, 4, PRE_MEDIUM, 1, 3),
                                 lambda g, c: _blocks(g, c, I.alpha_mask(90, 130, seed=12), _RNG_LIST)),
    "image_lockstep": (({"DRIVER": "lockstep"}, PRF_LDR, 6, 6, PRE_MEDIUM), lambda g, c: c.compress_image(I.photo_like(96, 96, seed=3))),
    "device_lockstep": (({"DRIVER": "lockstep"}, PRF_LDR, 6, 6, PRE_MEDIUM), lambda g, c: _device(g, c, I.photo_like(96, 96, seed=3))),
}


def _volume(d, h, w):
    return np.stack([I.photo_like(h, w, seed=20 + z) for z in range(d)])


def observe(gpu, monkeypatch, name):
    """(launches, per-kind stage-timing launches {setup, refine, prepare, emit}, h2d bytes, d2h bytes) of one call."""
    (env, prof, bx, by, q, *rest), call = CASES[name]
    ctx = _context(gpu, monkeypatch, env, prof, bx, by, q, *rest)
    try:
        n0 = ctx.launch_count()
        call(gpu, ctx)
        launches = ctx.launch_count() - n0
        _, h2d, d2h = ctx.last_timing()
        # the same call again with per-launch events (which keep a pass to the plain wave loop on one stream)
        ctx.stage_timing(True)
        call(gpu, ctx)
        kinds = ctx.stage_timing(False, fetch=True)[1]
    finally:
        ctx.close()
    return launches, [kinds[k] for k in ("setup", "refine", "prepare", "emit")], h2d, d2h


# The values every case gives; DESIGN.md "Launches per pass" explains the first two.
PLAN = {
    "batch_array_6x6": (240, [10, 10, 10, 1], 73200, 9504),
    "batch_image_6x6": (83, [10, 10, 10, 1], 72000, 8160),
    "batch_volume_4x4x4": (64, [8, 8, 8, 1], 88560, 8448),
    "blocks_long_list": (234, [12, 12, 12, 1], 0, 0),
    "blocks_long_list_radius3": (235, [12, 12, 12, 1], 0, 0),
    "device_4x4_fast": (31, [10, 10, 10, 1], 0, 0),
    "device_6x6_medium": (40, [10, 10, 10, 1], 0, 0),
    "device_hdr_6x6_medium": (40, [10, 10, 10, 1], 0, 0),
    "device_lockstep": (1, [0, 0, 0, 0], 0, 0),
    "device_pipes2": (62, [10, 10, 10, 1], 0, 0),
    "device_slab_radius5": (41, [10, 10, 10, 1], 0, 0),
    "device_three_batches": (120, [10, 10, 10, 1], 0, 0),
    "image_array_6x6": (120, [10, 10, 10, 1], 36600, 4752),
    "image_bands1_ragged": (40, [10, 10, 10, 1], 1333332, 149632),
    "image_bands4_ragged": (43, [10, 10, 10, 1], 1333332, 149632),
    "image_bands8_ragged": (47, [10, 10, 10, 1], 1333332, 149632),
    "image_bands8_too_small": (40, [10, 10, 10, 1], 10240, 1232),
    "image_lockstep": (1, [0, 0, 0, 0], 36864, 4096),
    "image_pipes4": (124, [10, 10, 10, 1], 7260000, 1161600),
    "image_radius5": (41, [10, 10, 10, 1], 78600, 8800),
    "image_three_batches": (120, [10, 10, 10, 1], 46080, 5120),
    "image_volume_4x4x4": (32, [8, 8, 8, 1], 44280, 4224),
    "sharded_array_6x6": (120, [10, 10, 10, 1], 36600, 4752),
    "sharded_volume_4x4x4": (32, [8, 8, 8, 1], 44280, 4224),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_launch_plan(gpu, monkeypatch, name):
    assert observe(gpu, monkeypatch, name) == PLAN[name]
