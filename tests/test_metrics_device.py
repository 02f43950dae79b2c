"""Metrics calls over image tables: astcenc_b200_compute_error_metrics_device_images measures many device-resident image pairs in
one call, with an optional per-block error map (astc_dev_metrics.cuh).

CPU: the call planner (plan_metrics: virtual CTAs per slice, their prefix, the partial offsets, the map list and the refusals) and
the per-block error function compiled for the host simulation (tests/hostsim/hostsim_metrics.cpp, one lane and 32 lanes)
against numpy.
GPU: every entry's figures against astcenc_b200_compute_error_metrics on host copies of the same pair, alone and inside a
shuffled 40-entry table; the maps against numpy, with guard bytes around every output; the locality of the map under
compress_device_blocks; the error order and the launch count."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from astc_ref import *  # noqa: F401,F403
import astc_images as I

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "astc-encoder_b200", "csrc")
GOLD = os.path.join(HERE, "golden", "golden_metrics.npz")
NP = {TYPE_U8: np.uint8, TYPE_F16: np.float16, TYPE_F32: np.float32}
DT = {np.dtype(np.uint8): TYPE_U8, np.dtype(np.float16): TYPE_F16, np.dtype(np.float32): TYPE_F32}
MASKS = {1: (0, 1, 2), 2: (2, 3), 3: (0, 1, 2), 4: (0, 1, 2, 3)}
GRID_MAX = 2 ** 31 - 1

# Figures that are sums (or come from them by IEEE double arithmetic only) are bit for bit those of the host entry; the dB
# figures go through the device's double log10 (include/astcenc.h states the tolerance).
EXACT = ("rgb_peak", "log_rmse", "mean_angular_error", "worst_angular_error")
DB = ("psnr", "alpha_psnr", "rgb_psnr", "peak_psnr", "mpsnr")
DB_ATOL = 1e-12

_SIMS = {}


def metrics_sim(lanes32=False):
    """tests/hostsim/hostsim_metrics.cpp compiled for the host (one simulated lane, or 32 lanes on 32 threads)."""
    if lanes32 in _SIMS:
        return _SIMS[lanes32]
    so = os.path.join(HERE, "_build", "libhostsim_metrics%s.so" % ("32" if lanes32 else ""))
    hs = os.path.join(HERE, "hostsim")
    newest = max([os.path.getmtime(os.path.join(CSRC, f)) for f in os.listdir(CSRC)] + [os.path.getmtime(os.path.join(hs, f)) for f in os.listdir(hs)])
    if not os.path.exists(so) or os.path.getmtime(so) < newest:
        os.makedirs(os.path.dirname(so), exist_ok=True)
        cmd = ["g++", "-std=c++14", "-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-shared"] + \
              (["-pthread", "-DASTC_HOSTSIM_LANES32=1"] if lanes32 else []) + \
              ["-x", "c++", os.path.join(hs, "hostsim_metrics.cpp"), os.path.join(CSRC, "astc_host_tables.cpp"), os.path.join(CSRC, "astc_host_config.cpp"),
               "-o", so]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(so)
    lib.hostsim_plan_metrics.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p]
    lib.hostsim_block_error.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.c_int,
                                        C.c_void_p]
    assert lib.hostsim_lanes() == (32 if lanes32 else 1)
    _SIMS[lanes32] = lib
    return lib


def plan(shapes, fp, mapped=None):
    """plan_metrics over pairs of (D, H, W) shapes: None when refused, else a dict of the planned fields."""
    lib = metrics_sim()
    n = len(shapes)
    mapped = np.asarray(mapped if mapped is not None else [0] * n, np.int32)
    dims = np.array([[s[2], s[1], s[0]] for s in shapes], np.uint32).reshape(-1)
    ctas = np.zeros(n, np.uint32)
    first = np.zeros(n, np.uint64)
    bxy = np.zeros(2 * n, np.uint32)
    maps = np.zeros(2 * n, np.uint64)
    totals = np.zeros(5, np.uint64)
    if lib.hostsim_plan_metrics(dims.ctypes.data, mapped.ctypes.data, n, fp[0], fp[1], fp[2], ctas.ctypes.data, first.ctypes.data, bxy.ctypes.data,
                                maps.ctypes.data, totals.ctypes.data):
        return None
    k = int(mapped.astype(bool).sum())
    return dict(ctas=ctas.tolist(), first=first.tolist(), blocks=bxy.reshape(-1, 2).tolist(), maps=maps.reshape(-1, 2)[:k].tolist(),
                total_ctas=int(totals[0]), map_blocks=int(totals[1]), partial_doubles=int(totals[2]), finish_grid=int(totals[3]), map_grid=int(totals[4]))


def nblocks(shape, fp):
    d, h, w = shape
    return -(-w // fp[0]) * -(-h // fp[1]) * (-(-d // fp[2]) if fp[2] > 1 else d)


# ---------------------------------------------------------------------------------------------------------------------------
# CPU: the planner
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hw,ctas", [((1, 1), 1), ((16, 16), 1), ((1, 257), 2), ((37, 29), 5), ((151, 151), 90), ((101, 1500), 592),
                                     ((101, 1501), 592), ((4096, 4096), 592)])
def test_virtual_ctas_per_slice(hw, ctas):
    """min(592, ceil(texels / 256)) per slice: the partition the host entry has always used for one slice."""
    p = plan([(3, hw[0], hw[1])], (6, 6, 1))
    assert p["ctas"] == [ctas]
    assert p["total_ctas"] == 3 * ctas


def test_prefix_and_partial_offsets_of_a_mixed_table():
    """2D images, a texture array and a volume: each entry's first virtual CTA is the prefix of dim_z * ctas, its partials start
    there, the sums follow all partials, and only mapped entries take map blocks, in call order."""
    shapes = [(1, 45, 67), (4, 13, 17), (1, 1, 1), (9, 21, 19), (1, 4096, 4096)]
    for fp in ((6, 6, 1), (4, 4, 4)):
        mapped = [1, 1, 0, 1, 0]
        p = plan(shapes, fp, mapped)
        ctas = [min(592, -(-h * w // 256)) for _, h, w in shapes]
        first = list(np.cumsum([0] + [c * s[0] for c, s in zip(ctas, shapes)])[:-1])
        assert p["ctas"] == ctas and p["first"] == first
        assert p["total_ctas"] == sum(c * s[0] for c, s in zip(ctas, shapes))
        assert p["partial_doubles"] == (p["total_ctas"] + len(shapes)) * 17
        assert p["finish_grid"] == 1
        assert p["blocks"] == [[-(-w // fp[0]), -(-h // fp[1])] for _, h, w in shapes]
        want_maps, at = [], 0
        for j, (s, m) in enumerate(zip(shapes, mapped)):
            if m:
                want_maps.append([at, j])
                at += nblocks(s, fp)
        assert p["maps"] == want_maps and p["map_blocks"] == at and p["map_grid"] == -(-at // 8)
    assert plan([(1, 8, 8)] * 9, (4, 4, 1))["finish_grid"] == 2
    assert plan([(1, 8, 8)], (4, 4, 1))["map_grid"] == 0


def test_calls_that_do_not_fit_a_launch_are_refused():
    big = (1, 2 ** 18, 2 ** 18)      # 2^32 blocks of 4x4
    assert plan([big], (4, 4, 1)) is not None
    assert plan([big], (4, 4, 1), [1]) is None
    assert plan([(1, 6 * 2 ** 16, 6 * 2 ** 16)], (6, 6, 1), [1]) is None
    assert plan([(1, 6 * 2 ** 16, 6 * 2 ** 16 - 6)], (6, 6, 1), [1]) is not None
    under = (1, 2 ** 18, 2 ** 18 - 4)      # 2^32 - 2^16 blocks each: five of them need more than 2^31 - 1 map CTAs
    assert plan([under] * 4, (4, 4, 1), [1] * 4) is not None
    assert plan([under] * 5, (4, 4, 1), [1] * 5) is None
    assert plan([(GRID_MAX, 16, 16)], (4, 4, 1)) is not None
    assert plan([(GRID_MAX, 16, 16), (1, 1, 1)], (4, 4, 1)) is None


# ---------------------------------------------------------------------------------------------------------------------------
# CPU: the per-block error function
# ---------------------------------------------------------------------------------------------------------------------------
def texel_values(img):
    """metric_load's per-texel values: U8 / 255 in float, F16 / F32 clamped to [0, 65504]."""
    if img.dtype == np.uint8:
        return img.astype(np.float32) / np.float32(255.0)
    return np.fmin(np.fmax(img.astype(np.float32), np.float32(0.0)), np.float32(65504.0))


def numpy_map(a, b, fp, components):
    """One float per block: the float64 sum of the block's float squared differences over its texels inside the image and the
    selected channels, rounded to float32 once."""
    d = texel_values(a) - texel_values(b)
    sq = (d * d).astype(np.float64)[..., list(MASKS[components])]
    D, H, W = a.shape[:3]
    bx, by, bz = fp
    gz = -(-D // bz) * bz if bz > 1 else D
    pad = np.zeros((gz, -(-H // by) * by, -(-W // bx) * bx, sq.shape[-1]), np.float64)
    pad[:D, :H, :W] = sq
    lz = gz // bz
    blocks = pad.reshape(lz, bz, pad.shape[1] // by, by, pad.shape[2] // bx, bx, sq.shape[-1]).sum(axis=(1, 3, 5, 6))
    return blocks.reshape(-1).astype(np.float32)


def random_pair(rng, shape, t1, t2):
    def one(t, base=None):
        if t == TYPE_U8:
            v = rng.integers(0, 256, shape + (4,)).astype(np.uint8)
            if base is not None:
                v = np.clip(base.astype(np.int32) + rng.integers(-9, 10, v.shape), 0, 255).astype(np.uint8)
            return v
        v = rng.uniform(-0.5, 4.0, shape + (4,)).astype(NP[t])
        v.reshape(-1)[rng.integers(0, v.size, 3)] = np.array([np.inf, 65504.0 if t == TYPE_F16 else 70000.0, np.nan], NP[t])
        return v
    a = one(t1)
    b = one(t2, a if t1 == t2 == TYPE_U8 else None)
    return a, b


def sim_map(lib, a, b, fp, components):
    D, H, W = a.shape[:3]
    out = np.full(nblocks((D, H, W), fp), np.nan, np.float32)
    lib.hostsim_block_error(a.ctypes.data, DT[a.dtype], b.ctypes.data, DT[b.dtype], W, H, D, fp[0], fp[1], fp[2], components, out.ctypes.data)
    return out


# (footprint, (D, H, W)): ragged on every axis; a 2D footprint over a texture array; whole blocks
MAP_SHAPES = [((6, 6, 1), (1, 37, 29)), ((6, 6, 1), (3, 13, 17)), ((6, 6, 1), (1, 12, 18)), ((6, 6, 1), (2, 1, 1)),
              ((4, 4, 4), (5, 7, 9)), ((4, 4, 4), (8, 8, 4)), ((4, 4, 4), (1, 1, 1)), ((4, 4, 4), (9, 3, 13))]
TYPE_PAIRS = [(TYPE_U8, TYPE_U8), (TYPE_F16, TYPE_F16), (TYPE_F32, TYPE_F32), (TYPE_U8, TYPE_F32), (TYPE_F16, TYPE_U8), (TYPE_F32, TYPE_F16)]


@pytest.mark.parametrize("lanes32", [False, True], ids=["lanes1", "lanes32"])
def test_hostsim_block_error_equals_numpy(lanes32):
    lib = metrics_sim(lanes32)
    rng = np.random.default_rng(11)
    n = 0
    for fp, shape in MAP_SHAPES:
        for t1, t2 in TYPE_PAIRS:
            a, b = random_pair(rng, shape, t1, t2)
            for components in (1, 2, 3, 4):
                if lanes32 and components != (n % 4) + 1:
                    continue      # (the 32-lane simulation is slow: one component count per pair)
                got = sim_map(lib, a, b, fp, components)
                want = numpy_map(a, b, fp, components)
                assert np.array_equal(got, want), (fp, shape, t1, t2, components)
            n += 1


def test_hostsim_block_error_depends_only_on_the_block():
    """Changing the texels of one block, or any texel outside the image's selected channels, moves no other block's value."""
    lib = metrics_sim()
    rng = np.random.default_rng(5)
    fp, shape = (6, 6, 1), (2, 20, 25)
    a, b = random_pair(rng, shape, TYPE_U8, TYPE_U8)
    before = sim_map(lib, a, b, fp, 3)
    b2 = b.copy()
    b2[1, 6:12, 12:18] ^= 0x55      # block (slice 1, row 1, col 2)
    b2[..., 3] ^= 0x0F              # alpha does not count for 3 components
    after = sim_map(lib, a, b2, fp, 3)
    k = (1 * 4 + 1) * 5 + 2
    changed = np.nonzero(before != after)[0].tolist()
    assert changed == [k]


# ---------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------
GUARD = 64
GUARD_BYTE = 0x5A
METRICS_BYTES = C.sizeof(ErrorMetrics)


@pytest.fixture(scope="module")
def gpu(pkg):
    import torch
    assert torch.cuda.is_available(), "the GPU tests need a CUDA device"
    torch.cuda.set_device(0)
    return pkg


def golden_pairs():
    g = np.load(GOLD)
    for name in g["names"]:
        name = str(name)
        hdr, normal, comps, lo, hi = [int(v) for v in g[name + "/args"]]
        yield name, g[name + "/img1"], g[name + "/img2"], dict(hdr=bool(hdr), normal=bool(normal), input_components=comps, fstop_lo=lo, fstop_hi=hi)


def host_metrics(pkg, ctx, a, b, hdr=False, normal=False, input_components=4, fstop_lo=-10, fstop_hi=10):
    """astcenc_b200_compute_error_metrics on host arrays ((H, W, 4) or (D, H, W, 4)) -> ErrorMetrics."""
    keep, imgs = [], []
    for im in (a, b):
        im = np.ascontiguousarray(im)
        im = im[None] if im.ndim == 3 else im
        slices = (C.c_void_p * im.shape[0])(*[im[z].ctypes.data for z in range(im.shape[0])])
        keep.append((im, slices))
        imgs.append(pkg.Image(im.shape[2], im.shape[1], im.shape[0], DT[im.dtype], slices))
    out = pkg.ErrorMetrics()
    err = pkg.lib().astcenc_b200_compute_error_metrics(ctx.handle, int(hdr), int(normal), input_components, C.byref(imgs[0]), C.byref(imgs[1]),
                                                       fstop_lo, fstop_hi, C.byref(out))
    assert err == 0, err
    return out


class Pair:
    """One entry of a device call: its two images, its arguments and whether it asks for a map."""

    def __init__(self, name, a, b, kw, fp, want_map=True):
        self.name = name
        self.a = np.ascontiguousarray(a if a.ndim == 4 else a[None])
        self.b = np.ascontiguousarray(b if b.ndim == 4 else b[None])
        assert self.a.shape == self.b.shape
        self.kw = kw
        self.blocks = nblocks(self.a.shape[:3], fp) if want_map else 0


def device_call(ctx, pairs, kw, order=None, stream=None):
    """One compute_error_metrics_device_images call over `pairs` (in `order`), every output inside guard bytes in one allocation.
    Returns ([ErrorMetrics], [map or None]) in the pairs' order; checks the guard bytes and the launch count."""
    import torch
    dev = torch.device("cuda", 0)
    order = list(range(len(pairs))) if order is None else order
    ins = [(torch.from_numpy(p.a.view(np.uint8).reshape(-1)).to(dev), torch.from_numpy(p.b.view(np.uint8).reshape(-1)).to(dev)) for p in pairs]
    offs, pos = [], GUARD
    for p in pairs:
        m = pos
        pos += METRICS_BYTES + GUARD
        e = pos
        pos += 4 * p.blocks + GUARD
        offs.append((m, e))
        pos = -(-pos // 8) * 8
    out = torch.full((pos,), GUARD_BYTE, dtype=torch.uint8, device=dev)
    base = out.data_ptr()
    table = []
    for j in order:
        p, (i1, i2), (m, e) = pairs[j], ins[j], offs[j]
        D, H, W = p.a.shape[:3]
        table.append((i1.data_ptr(), i2.data_ptr(), DT[p.a.dtype], DT[p.b.dtype], W, H, D, base + m, base + e if p.blocks else 0))
    st = stream or torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    n0 = ctx.launch_count()
    ctx.compute_error_metrics_device_images(table, stream=st.cuda_stream, **kw)
    assert ctx.launch_count() == n0 + (3 if any(p.blocks for p in pairs) else 2)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    mask = np.ones(pos, bool)
    mets, maps = [], []
    for p, (m, e) in zip(pairs, offs):
        mets.append(ErrorMetrics.from_buffer_copy(got[m:m + METRICS_BYTES].tobytes()))
        mask[m:m + METRICS_BYTES] = False
        if p.blocks:
            maps.append(got[e:e + 4 * p.blocks].copy().view(np.float32))
            mask[e:e + 4 * p.blocks] = False
        else:
            maps.append(None)
    assert np.all(got[mask] == GUARD_BYTE), "a guard byte changed"
    return mets, maps


def raw(m):
    return bytes(m)


def check_like_host(got, want, name):
    for c in range(4):
        assert got.sum_squared_error[c] == want.sum_squared_error[c], (name, c)
    for k in EXACT:
        assert getattr(got, k) == getattr(want, k), (name, k)
    for k in DB:
        assert abs(getattr(got, k) - getattr(want, k)) <= DB_ATOL, (name, k, getattr(got, k), getattr(want, k))


def golden_entries(fp):
    out = []
    for name, a, b, kw in golden_pairs():
        h, w = min(a.shape[0], b.shape[0]), min(a.shape[1], b.shape[1])
        out.append((name, a, b, kw, Pair(name, a[:h, :w], b[:h, :w], kw, fp)))
    return out


@pytest.mark.gpu
def test_golden_pairs_alone_equal_the_host_entry(gpu):
    """Each golden pair alone: sums bit for bit those of the host entry (which compares the intersection of a cropped pair),
    dB figures within DB_ATOL; the map against numpy and its masked sum against sum_squared_error."""
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, gpu.FLG_DECOMPRESS_ONLY))
    try:
        for name, a, b, kw, p in golden_entries((6, 6, 1)):
            want = host_metrics(gpu, ctx, a, b, **kw)
            (got,), (mp,) = device_call(ctx, [p], kw)
            check_like_host(got, want, name)
            assert np.array_equal(mp, numpy_map(p.a, p.b, (6, 6, 1), kw["input_components"])), name
            sse = sum(want.sum_squared_error[c] for c in MASKS[kw["input_components"]])
            assert float(mp.astype(np.float64).sum()) == pytest.approx(sse, rel=1e-6, abs=1e-30), name
    finally:
        ctx.close()


def round_trip_entries(gpu):
    """A seeded 1024^2 round trip (6x6 -fast, decoded to U8 and to F16), a texture array and its decode, and a volume of a 3D
    footprint is measured on its own context."""
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, gpu.FLG_SELF_DECOMPRESS_ONLY))
    try:
        img = I.photo_like(1024, 1024, seed=9)
        blocks = ctx.compress_image(img)
        dec8 = ctx.decompress_image(blocks, 1024, 1024)
        dec16 = ctx.decompress_image(blocks, 1024, 1024, dtype=np.float16)
        arr = np.stack([I.photo_like(67, 93, seed=40 + z) for z in range(4)])
        arr_dec = ctx.decompress_image(ctx.compress_image(arr), 93, 67, dim_z=4)
    finally:
        ctx.close()
    kw4 = dict(input_components=4)
    return [("rt_u8", img, dec8, dict(normal=True, input_components=3)), ("rt_f16", img, dec16, kw4), ("array", arr, arr_dec, kw4)]


@pytest.mark.gpu
def test_round_trip_and_array_equal_the_host_entry(gpu):
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, gpu.FLG_DECOMPRESS_ONLY))
    try:
        for name, a, b, kw in round_trip_entries(gpu):
            want = host_metrics(gpu, ctx, a, b, **kw)
            p = Pair(name, a, b, kw, (6, 6, 1))
            (got,), (mp,) = device_call(ctx, [p], kw)
            check_like_host(got, want, name)
            assert 20.0 < got.psnr < 80.0
            assert np.array_equal(mp, numpy_map(p.a, p.b, (6, 6, 1), kw["input_components"])), name
            sse = sum(want.sum_squared_error[c] for c in MASKS[kw["input_components"]])
            assert float(mp.astype(np.float64).sum()) == pytest.approx(sse, rel=1e-6), name
    finally:
        ctx.close()


@pytest.mark.gpu
def test_volume_at_a_3d_footprint_equals_the_host_entry(gpu):
    ctx = gpu.Context(gpu.config_init(PRF_HDR, 4, 4, PRE_FAST, gpu.FLG_SELF_DECOMPRESS_ONLY, block_z=4))
    try:
        vol = I.hdr_noise(21, 19, seed=3, dtype=np.float16)
        vol = np.stack([vol * np.float16(1 + z / 8) for z in range(9)])
        dec = ctx.decompress_image(ctx.compress_image(vol), 19, 21, dtype=np.float16, dim_z=9)
        for kw in (dict(hdr=True, input_components=4, fstop_lo=-4, fstop_hi=6), dict(input_components=2)):
            want = host_metrics(gpu, ctx, vol, dec, **kw)
            p = Pair("volume", vol, dec, kw, (4, 4, 4))
            (got,), (mp,) = device_call(ctx, [p], kw)
            check_like_host(got, want, "volume")
            assert np.array_equal(mp, numpy_map(p.a, p.b, (4, 4, 4), kw["input_components"]))
    finally:
        ctx.close()


@pytest.mark.gpu
def test_entries_inside_a_shuffled_40_entry_table_equal_the_entry_alone(gpu):
    """Every entry's figures and map are bitwise those of the entry alone, whatever shares the call and in whatever order,
    and two runs of the call are bitwise equal."""
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, gpu.FLG_DECOMPRESS_ONLY))
    try:
        kw = dict(input_components=4, normal=True)
        pairs = [p for _, _, _, _, p in golden_entries((6, 6, 1)) if p.a.dtype == np.uint8 and p.b.dtype == np.uint8]
        pairs += [Pair(n, a, b, kw, (6, 6, 1)) for n, a, b, _ in round_trip_entries(gpu)]
        rng = np.random.default_rng(40)
        types = [TYPE_U8, TYPE_F16, TYPE_F32]
        while len(pairs) < 40:
            k = len(pairs)
            shape = (int(rng.integers(1, 4)), int(rng.integers(1, 90)), int(rng.integers(1, 90)))
            a, b = random_pair(rng, shape, types[k % 3], types[(k // 3) % 3])
            pairs.append(Pair("rand%d" % k, a, b, kw, (6, 6, 1), want_map=k % 4 != 0))
        alone = [device_call(ctx, [p], kw) for p in pairs]
        order = rng.permutation(len(pairs)).tolist()
        mets, maps = device_call(ctx, pairs, kw, order=order)
        again = device_call(ctx, pairs, kw, order=order)
        for j, p in enumerate(pairs):
            assert raw(mets[j]) == raw(alone[j][0][0]) == raw(again[0][j]), p.name
            if p.blocks:
                assert maps[j].tobytes() == alone[j][1][0].tobytes() == again[1][j].tobytes(), p.name
    finally:
        ctx.close()


@pytest.mark.gpu
def test_re_encoding_the_worst_blocks_moves_only_their_map_values(gpu):
    """Compress a texture set at -fast and measure it; re-encode the 1 % worst blocks of each texture at -thorough through
    compress_device_blocks, decode and measure again: every block that was not listed keeps its map value bit for bit."""
    import torch
    dev = torch.device("cuda", 0)
    fast = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, gpu.FLG_SELF_DECOMPRESS_ONLY))
    thorough = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_THOROUGH, gpu.FLG_SELF_DECOMPRESS_ONLY))
    try:
        imgs = [I.photo_like(h, w, seed=70 + k) for k, (h, w) in enumerate([(256, 256), (200, 311), (128, 96), (97, 143)])]
        d_img = [torch.from_numpy(im.reshape(-1)).to(dev) for im in imgs]
        d_pay = [torch.zeros(nblocks((1,) + im.shape[:2], (6, 6, 1)) * 16, dtype=torch.uint8, device=dev) for im in imgs]
        d_dec = [torch.zeros(im.size, dtype=torch.uint8, device=dev) for im in imgs]
        d_met = torch.zeros(len(imgs) * METRICS_BYTES, dtype=torch.uint8, device=dev)
        d_map = [torch.zeros(nblocks((1,) + im.shape[:2], (6, 6, 1)), dtype=torch.float32, device=dev) for im in imgs]
        dims = [(im.shape[1], im.shape[0]) for im in imgs]
        fast.compress_device_images([(d.data_ptr(), w, h, 1, p.data_ptr()) for d, (w, h), p in zip(d_img, dims, d_pay)], TYPE_U8)

        def measure():
            fast.decompress_device_images([(p.data_ptr(), o.data_ptr(), w, h, 1) for p, o, (w, h) in zip(d_pay, d_dec, dims)], TYPE_U8)
            fast.compute_error_metrics_device_images([(d.data_ptr(), o.data_ptr(), TYPE_U8, TYPE_U8, w, h, 1, d_met.data_ptr() + k * METRICS_BYTES, m.data_ptr())
                                                      for k, (d, o, (w, h), m) in enumerate(zip(d_img, d_dec, dims, d_map))], input_components=4)
            torch.cuda.synchronize()
            return [m.cpu().numpy() for m in d_map], [ErrorMetrics.from_buffer_copy(d_met.cpu().numpy()[k * METRICS_BYTES:(k + 1) * METRICS_BYTES].tobytes())
                                                     for k in range(len(imgs))]

        before, _ = measure()
        lists = []
        for k, (d, (w, h), p) in enumerate(zip(d_img, dims, d_pay)):
            worst = np.argsort(-before[k], kind="stable")[:max(1, len(before[k]) // 100)].astype(np.uint32)
            lists.append(worst)
            thorough.compress_device_blocks(d.data_ptr(), TYPE_U8, w, h, 1, worst, p.data_ptr())
        torch.cuda.synchronize()
        after, _ = measure()
        for k in range(len(imgs)):
            keep = np.ones(len(before[k]), bool)
            keep[lists[k]] = False
            assert np.array_equal(before[k][keep].view(np.uint32), after[k][keep].view(np.uint32)), k
            assert not np.array_equal(before[k][lists[k]], after[k][lists[k]]), k      # (the listed blocks were re-encoded)
    finally:
        fast.close()
        thorough.close()


# ---- errors ----
OK, PARAM = 0, 3


@pytest.mark.gpu
def test_errors_follow_the_documented_order_and_launch_nothing(gpu):
    import torch
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, gpu.FLG_DECOMPRESS_ONLY))
    dev = torch.device("cuda", 0)
    buf = torch.zeros(4096, dtype=torch.uint8, device=dev)
    base = buf.data_ptr()
    met = base + 2048
    mp = base + 3072

    def call(components=4, lo=-10, hi=10, images=True, count=None, **e):
        d = dict(original=base, decoded=base + 1024, original_type=TYPE_U8, decoded_type=TYPE_U8, dim_x=8, dim_y=8, dim_z=1, metrics=met,
                 block_error=mp)
        d.update(e)
        t = (gpu.DeviceMetricsImage * 2)(*[gpu.DeviceMetricsImage(C.c_void_p(d["original"]), C.c_void_p(d["decoded"]), d["original_type"],
                                                                  d["decoded_type"], d["dim_x"], d["dim_y"], d["dim_z"], C.c_void_p(d["metrics"]),
                                                                  C.c_void_p(d["block_error"] or None))] * 2)
        n0 = ctx.launch_count()
        r = gpu.lib().astcenc_b200_compute_error_metrics_device_images(ctx.handle, 0, 0, components, t if images else None, 2 if count is None else count,
                                                                       lo, hi, None)
        torch.cuda.synchronize()
        launched = ctx.launch_count() - n0
        assert launched == (0 if r != OK else (0 if count == 0 else 3 if d["block_error"] else 2)), (r, launched)
        return r

    try:
        assert call() == OK
        assert call(block_error=0) == OK
        assert call(count=0) == OK
        assert call(images=False, count=0) == OK
        singles = [dict(components=0), dict(components=5), dict(lo=-126), dict(hi=126), dict(images=False), dict(original=0), dict(decoded=0),
                   dict(metrics=0), dict(dim_x=0), dict(dim_y=0), dict(dim_z=0), dict(dim_x=0xFFFFFFFF, dim_y=0xFFFFFFFF, dim_z=2),
                   dict(original_type=3), dict(decoded_type=-1), dict(original=base + 2), dict(decoded_type=TYPE_F16, decoded=base + 1028),
                   dict(original_type=TYPE_F32, original=base + 8), dict(metrics=met + 4), dict(block_error=mp + 2),
                   dict(dim_x=6 * 2 ** 16, dim_y=6 * 2 ** 16)]      # (2^32 blocks of 6x6 with a map)
        for s in singles:
            assert call(**s) == PARAM, s
        # pairs of classes on different arguments: the earlier class decides (every code is ASTCENC_ERR_BAD_PARAM, and nothing runs)
        for s1 in singles:
            for s2 in singles[::3]:
                if not set(s1) & set(s2):
                    assert call(**{**s1, **s2}) == PARAM, (s1, s2)
        assert gpu.lib().astcenc_b200_compute_error_metrics_device_images(None, 0, 0, 4, None, 0, -10, 10, None) == PARAM
    finally:
        ctx.close()
