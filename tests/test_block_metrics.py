"""Per-block error maps of a chosen metric: astcenc_b200_compute_block_metric_device_images and
astcenc_b200_compute_block_metric_device_block_lists (metric_block_terms / block_error_sum<M> in astc_dev_metrics.cuh;
astc_block_metric_kernel<M> and astc_block_metric_lists_kernel<M>).

CPU: the whole maps and list refreshes of the host simulation (tests/hostsim/hostsim_block_metric.cpp, one lane and 32 lanes)
against a numpy restatement and against each other; the per-block values against the oracle's alpha_psnr and log_rmse of each
block's crop; the locality of a value.
GPU: whole maps against the 32-lane simulation, alone and inside a shuffled 40-entry table, with the figures of
compute_error_metrics_device_images and guard bytes around every output; ASTCENC_B200_BLOCK_SQUARED_ERROR against the existing
calls; list refreshes after a re-encode and a list decode; the HDR refine loop on one stream against the host round trip; the
error order and the launch counts."""
import ctypes as C

import numpy as np
import pytest

from astc_ref import *  # noqa: F401,F403
from hostsim_build import host_sim
from test_block_list_decode import KINDS, MAP_CASES, MAP_POISON, make_list
from test_metrics_device import (DT, GUARD, GUARD_BYTE, MAP_SHAPES, MASKS, METRICS_BYTES, TYPE_PAIRS, Pair, golden_entries, nblocks, random_pair,
                                 round_trip_entries, texel_values)
import astc_images as I

SQUARED, ALPHA, LOG2 = 0, 1, 2      # enum astcenc_b200_block_metric
NEW_METRICS = (ALPHA, LOG2)
METRIC_IDS = {SQUARED: "squared", ALPHA: "alpha", LOG2: "log2"}
S = FLG_SELF_DECOMPRESS_ONLY


_SIMS = {}


def sim(lanes32=False):
    """tests/hostsim/hostsim_block_metric.cpp compiled for the host (one simulated lane, or 32 lanes on 32 threads)."""
    if lanes32 in _SIMS:
        return _SIMS[lanes32]
    lib = host_sim("hostsim_block_metric", lanes32)
    lib.hostsim_block_metric.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.c_int,
                                         C.c_int, C.c_void_p]
    lib.hostsim_block_metric_lists.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_uint, C.c_uint,
                                               C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    _SIMS[lanes32] = lib
    return lib


def sim_metric_map(lib, a, b, fp, components, metric):
    """The host simulation's map of (D, H, W, 4) arrays a (original) and b (decoded)."""
    a = np.ascontiguousarray(a if a.ndim == 4 else a[None])
    b = np.ascontiguousarray(b if b.ndim == 4 else b[None])
    D, H, W = a.shape[:3]
    out = np.full(nblocks((D, H, W), fp), np.nan, np.float32)
    lib.hostsim_block_metric(a.ctypes.data, DT[a.dtype], b.ctypes.data, DT[b.dtype], W, H, D, fp[0], fp[1], fp[2], components, metric, out.ctypes.data)
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# The numpy restatement
# ---------------------------------------------------------------------------------------------------------------------------
LOG2_POLY = [np.float32(v) for v in (0.0596515482674574969533, -0.465725644288844778798, 1.48116647521213171641, -2.52074962577807006663,
                                     2.8882704548164776201)]


def np_log2(x):
    """metric_log2 in float32: the exponent plus a polynomial of the mantissa in [1, 2), unfused."""
    i = np.ascontiguousarray(x, np.float32).view(np.int32)
    e = (((i & 0x7F800000) >> 23) - 127).astype(np.float32)
    m = ((i & 0x007FFFFF) | 0x3F800000).astype(np.int32).view(np.float32)
    p = LOG2_POLY[0]
    for c in LOG2_POLY[1:]:
        p = p * m + c
    p = p * (m - np.float32(1.0))
    return p + e


def texel_terms(a, b, components, metric):
    """(..., terms) float32: each texel's terms in channel order (metric_block_terms)."""
    o, d = texel_values(a), texel_values(b)
    mask = MASKS[components]
    if metric == LOG2:
        v = [np_log2(o[..., c]) - np_log2(d[..., c]) for c in mask if c < 3]
    elif metric == ALPHA:
        v = [(o[..., c] - d[..., c]) * o[..., 3] if c < 3 else o[..., 3] - d[..., 3] for c in mask]
    else:
        v = [o[..., c] - d[..., c] for c in mask]
    v = np.stack(v, axis=-1)
    return v * v


def numpy_metric_map(a, b, fp, components, metric):
    """One float per block: the float64 sum of the block's float32 terms over its texels inside the image, rounded once."""
    a = a if a.ndim == 4 else a[None]
    b = b if b.ndim == 4 else b[None]
    sq = texel_terms(a, b, components, metric).astype(np.float64)
    D, H, W = a.shape[:3]
    bx, by, bz = fp
    gz = -(-D // bz) * bz if bz > 1 else D
    pad = np.zeros((gz, -(-H // by) * by, -(-W // bx) * bx, sq.shape[-1]), np.float64)
    pad[:D, :H, :W] = sq
    blocks = pad.reshape(gz // bz, bz, pad.shape[1] // by, by, pad.shape[2] // bx, bx, sq.shape[-1]).sum(axis=(1, 3, 5, 6))
    return blocks.reshape(-1).astype(np.float32)


def soft_alpha(h, w, seed):
    """photo_like with a soft alpha mask: a ramp of its green channel, zero on its darkest 20 % of texels."""
    img = I.photo_like(h, w, seed=seed)
    g = img[..., 1].astype(np.float32)
    lo = np.percentile(g, 20)
    img[..., 3] = np.clip((g - lo) * 3.0, 0, 255).astype(np.uint8)
    return img


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", NEW_METRICS, ids=lambda m: METRIC_IDS[m])
@pytest.mark.parametrize("lanes32", [False, True], ids=["lanes1", "lanes32"])
def test_hostsim_block_metric_equals_numpy(lanes32, metric):
    """Ragged footprints, texture arrays and 3D footprints; every type pair, with inf, NaN and out-of-range texels; input_components
    1-4: the simulation's map equals the numpy restatement bit for bit."""
    lib = sim(lanes32)
    rng = np.random.default_rng(11 + metric)
    n = 0
    for fp, shape in MAP_SHAPES:
        for t1, t2 in TYPE_PAIRS:
            a, b = random_pair(rng, shape, t1, t2)
            for components in (1, 2, 3, 4):
                if lanes32 and components != (n % 4) + 1:
                    continue      # (the 32-lane simulation is slow: one component count per pair)
                got = sim_metric_map(lib, a, b, fp, components, metric)
                want = numpy_metric_map(a, b, fp, components, metric)
                assert np.array_equal(got, want), (fp, shape, t1, t2, components)
            n += 1


def sim_metric_lists(lib, pairs, fp, components, metric, lists, maps):
    """The host simulation's list refresh of `metric` into `maps` at the blocks of `lists` (one per pair)."""
    n = len(pairs)
    o = (C.c_void_p * n)(*[a.ctypes.data for a, _ in pairs])
    d = (C.c_void_p * n)(*[b.ctypes.data for _, b in pairs])
    ot = np.array([DT[a.dtype] for a, _ in pairs], np.int32)
    dt = np.array([DT[b.dtype] for _, b in pairs], np.int32)
    dims = np.array([[a.shape[2], a.shape[1], a.shape[0]] for a, _ in pairs], np.uint32).reshape(-1)
    mp = (C.c_void_p * n)(*[m.ctypes.data for m in maps])
    padded = [l.padded() for l in lists]
    ip = (C.c_void_p * n)(*[p.ctypes.data for p in padded])
    counts = np.array([l.count for l in lists], np.uint32)
    caps = np.array([l.capacity for l in lists], np.uint32)
    assert lib.hostsim_block_metric_lists(o, ot.ctypes.data, d, dt.ctypes.data, dims.ctypes.data, n, fp[0], fp[1], fp[2], components, metric, mp, ip,
                                          counts.ctypes.data, caps.ctypes.data) == 0


@pytest.mark.parametrize("metric", (SQUARED,) + NEW_METRICS, ids=lambda m: METRIC_IDS[m])
@pytest.mark.parametrize("lanes32", [False, True], ids=["lanes1", "lanes32"])
@pytest.mark.parametrize("fp,shapes", MAP_CASES, ids=["6x6", "4x4x4"])
def test_hostsim_list_refresh_equals_the_whole_map_at_listed_blocks(fp, shapes, lanes32, metric):
    """Mixed types, every list kind (garbage past the count, duplicates, count > capacity, count 0, capacity 0, indices out of
    range), one table: listed values equal the simulation's whole map of the same metric bit for bit, every other value keeps its
    poison."""
    lib = sim(lanes32)
    rng = np.random.default_rng(23 + metric)
    types = [(TYPE_U8, TYPE_U8), (TYPE_F16, TYPE_F16), (TYPE_F32, TYPE_U8), (TYPE_U8, TYPE_F16), (TYPE_F16, TYPE_F32)]
    pairs = [random_pair(rng, s, *types[k % len(types)]) for k, s in enumerate(shapes)]
    kinds = [KINDS[k % len(KINDS)] for k in range(len(shapes))]
    lists = [make_list(rng, nblocks(s, fp), k) for s, k in zip(shapes, kinds)]
    for components in ((1, 2, 3, 4) if not lanes32 else (4,)):
        maps = [np.full(nblocks(s, fp), MAP_POISON, np.uint32).view(np.float32) for s in shapes]
        sim_metric_lists(lib, pairs, fp, components, metric, lists, maps)
        for k, ((a, b), s, l, m) in enumerate(zip(pairs, shapes, lists, maps)):
            want = np.full(nblocks(s, fp), MAP_POISON, np.uint32)
            listed = l.listed(len(want))
            want[listed] = sim_metric_map(lib, a, b, fp, components, metric).view(np.uint32)[listed]
            assert np.array_equal(m.view(np.uint32), want), "pair %d %s (%s list), components %d" % (k, s, kinds[k], components)


def test_numpy_log2_is_the_reference_polynomial():
    """Spot values of the restated log2: exact at powers of two, -127 at 0, close to log2 elsewhere."""
    x = np.array([1.0, 2.0, 0.5, 1024.0, 65504.0, 0.0, 3.0, 1.0 / 255.0], np.float32)
    got = np_log2(x)
    assert np.array_equal(got[:4], [0.0, 1.0, -1.0, 10.0]) and got[5] == -127.0
    assert np.allclose(got[[4, 6, 7]], np.log2(x[[4, 6, 7]]), atol=1e-4)


def oracle_pairs(oracle):
    """The 2D golden pairs (cropped to their intersection) and -fast round trips through the oracle: hdr_noise in F16 with the
    HDR profile, and photo_like with a soft alpha mask in U8. (name, original, decoded, input_components)."""
    out = []
    for name, a, b, kw, p in golden_entries((6, 6, 1)):
        out.append((name, p.a[0], p.b[0], kw["input_components"]))
    hdr = I.hdr_noise(42, 47, seed=21, dtype=np.float16)
    dec = oracle.decompress(oracle.compress(hdr, PRF_HDR, 6, 6, PRE_FAST), 47, 42, PRF_HDR, 6, 6, out_type=TYPE_F16)
    out.append(("hdr_noise", hdr, dec, 4))
    out.append(("hdr_noise_rgb", hdr, dec, 3))
    ldr = soft_alpha(40, 53, seed=5)
    dec = oracle.decompress(oracle.compress(ldr, PRF_LDR, 6, 6, PRE_FAST), 53, 40, PRF_LDR, 6, 6, out_type=TYPE_U8)
    out.append(("alpha_photo", ldr, dec, 4))
    return out


def test_block_values_equal_the_oracle_figures_of_each_block(oracle):
    """Each block's texels cropped and measured by the oracle: log_rmse^2 * texels is the LOG2 value and, with 4 components,
    4 * texels / 10^(alpha_psnr / 10) the ALPHA value (999 dB: 0), within 1e-6."""
    lib = sim()
    checked = 0
    for name, a, b, comps in oracle_pairs(oracle):
        h, w = a.shape[:2]
        maps = {m: sim_metric_map(lib, a, b, (6, 6, 1), comps, m) for m in NEW_METRICS}
        bxs = -(-w // 6)
        for k in range(len(maps[LOG2])):
            y0, x0 = (k // bxs) * 6, (k % bxs) * 6
            ca, cb = a[y0:y0 + 6, x0:x0 + 6], b[y0:y0 + 6, x0:x0 + 6]
            texels = ca.shape[0] * ca.shape[1]
            fig = oracle.error_metrics(ca, cb, hdr=True, components=comps)
            assert float(maps[LOG2][k]) == pytest.approx(fig["log_rmse"] ** 2 * texels, rel=1e-6, abs=1e-30), (name, k)
            if comps == 4:
                want = 0.0 if fig["alpha_psnr"] == 999.0 else 4 * texels / 10.0 ** (fig["alpha_psnr"] / 10.0)
                assert float(maps[ALPHA][k]) == pytest.approx(want, rel=1e-6, abs=1e-30), (name, k)
            checked += 1
    assert checked > 500


@pytest.mark.parametrize("metric", (SQUARED,) + NEW_METRICS, ids=lambda m: METRIC_IDS[m])
def test_block_metric_depends_only_on_the_block(metric):
    """Changing the texels of one block, original alpha included, moves that block's value and no other."""
    lib = sim()
    rng = np.random.default_rng(5)
    fp, shape = (6, 6, 1), (2, 20, 25)
    a, b = random_pair(rng, shape, TYPE_U8, TYPE_U8)
    before = sim_metric_map(lib, a, b, fp, 4, metric)
    a2, b2 = a.copy(), b.copy()
    b2[1, 6:12, 12:18, :3] ^= 0x55      # block (slice 1, row 1, col 2)
    a2[1, 6:12, 12:18, 3] ^= 0x3C
    after = sim_metric_map(lib, a2, b2, fp, 4, metric)
    assert np.nonzero(before != after)[0].tolist() == [(1 * 4 + 1) * 5 + 2]


# ---------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu(pkg):
    import torch
    assert torch.cuda.is_available(), "the GPU tests need a CUDA device"
    torch.cuda.set_device(0)
    return pkg


def device_call(ctx, pairs, kw, metric=None, order=None):
    """One call over `pairs` (in `order`): compute_block_metric_device_images with `metric`, or compute_error_metrics_device_images
    when metric is None. Every output sits inside guard bytes in one allocation. Returns (the allocation's bytes, [raw figures],
    [map or None]) in the pairs' order; checks the guard bytes and the launch count."""
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
    st = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    n0 = ctx.launch_count()
    if metric is None:
        ctx.compute_error_metrics_device_images(table, stream=st.cuda_stream, **kw)
    else:
        ctx.compute_block_metric_device_images(table, metric, stream=st.cuda_stream, **kw)
    assert ctx.launch_count() == n0 + (3 if any(p.blocks for p in pairs) else 2)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    mask = np.ones(pos, bool)
    mets, maps = [], []
    for p, (m, e) in zip(pairs, offs):
        mets.append(got[m:m + METRICS_BYTES].tobytes())
        mask[m:m + METRICS_BYTES] = False
        if p.blocks:
            maps.append(got[e:e + 4 * p.blocks].copy().view(np.float32))
            mask[e:e + 4 * p.blocks] = False
        else:
            maps.append(None)
    assert np.all(got[mask] == GUARD_BYTE), "a guard byte changed"
    return got, mets, maps


def hdr_round_trip(gpu):
    """hdr_noise through a -fast HDR context, decoded to F16."""
    ctx = gpu.Context(gpu.config_init(PRF_HDR, 6, 6, PRE_FAST, S))
    try:
        img = I.hdr_noise(181, 203, seed=21, dtype=np.float16)
        return img, ctx.decompress_image(ctx.compress_image(img), 203, 181, dtype=np.float16)
    finally:
        ctx.close()


def all_2d_entries(gpu):
    """(name, Pair, kw) at 6x6: the golden pairs, the LDR round trips and texture array, the HDR round trip and a soft-alpha one."""
    fp = (6, 6, 1)
    out = [(name, p, kw) for name, _, _, kw, p in golden_entries(fp)]
    out += [(name, Pair(name, a, b, kw, fp), kw) for name, a, b, kw in round_trip_entries(gpu)]
    hdr, hdr_dec = hdr_round_trip(gpu)
    kw = dict(hdr=True, input_components=4, fstop_lo=-6, fstop_hi=6)
    out.append(("hdr_rt", Pair("hdr_rt", hdr, hdr_dec, kw, fp), kw))
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, S))
    try:
        img = soft_alpha(157, 211, seed=5)
        dec = ctx.decompress_image(ctx.compress_image(img), 211, 157)
    finally:
        ctx.close()
    kw = dict(input_components=4)
    out.append(("alpha_rt", Pair("alpha_rt", img, dec, kw, fp), kw))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("metric", NEW_METRICS, ids=lambda m: METRIC_IDS[m])
def test_whole_maps_equal_the_32_lane_simulation(metric, gpu):
    """Golden pairs, U8 / F16 / HDR / soft-alpha round trips, a texture array and a volume at a 3D footprint, each alone: the map
    is bit for bit the 32-lane simulation's, the figures bit for bit those of compute_error_metrics_device_images."""
    lib = sim(True)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, FLG_DECOMPRESS_ONLY))
    try:
        for name, p, kw in all_2d_entries(gpu):
            _, (mets,), (mp,) = device_call(ctx, [p], kw, metric)
            _, (want_mets,), _ = device_call(ctx, [p], kw)
            assert mets == want_mets, name
            assert np.array_equal(mp.view(np.uint32), sim_metric_map(lib, p.a, p.b, (6, 6, 1), kw["input_components"], metric).view(np.uint32)), name
    finally:
        ctx.close()
    ctx = gpu.Context(gpu.config_init(PRF_HDR, 4, 4, PRE_FAST, S, block_z=4))
    try:
        vol = I.hdr_noise(21, 19, seed=3, dtype=np.float16)
        vol = np.stack([vol * np.float16(1 + z / 8) for z in range(9)])
        dec = ctx.decompress_image(ctx.compress_image(vol), 19, 21, dtype=np.float16, dim_z=9)
        for kw in (dict(hdr=True, input_components=4, fstop_lo=-4, fstop_hi=6), dict(input_components=2)):
            p = Pair("volume", vol, dec, kw, (4, 4, 4))
            _, (mets,), (mp,) = device_call(ctx, [p], kw, metric)
            _, (want_mets,), _ = device_call(ctx, [p], kw)
            assert mets == want_mets
            assert np.array_equal(mp.view(np.uint32), sim_metric_map(lib, vol, dec, (4, 4, 4), kw["input_components"], metric).view(np.uint32))
    finally:
        ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("metric", NEW_METRICS, ids=lambda m: METRIC_IDS[m])
def test_maps_inside_a_shuffled_40_entry_table_equal_the_entry_alone(metric, gpu):
    """Every entry's map is bitwise the entry's map alone, whatever shares the call and in whatever order; the figures of the
    table are bitwise those of compute_error_metrics_device_images on the same table."""
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, FLG_DECOMPRESS_ONLY))
    try:
        kw = dict(input_components=4, hdr=True)
        pairs = [p for _, p, _ in all_2d_entries(gpu)]
        rng = np.random.default_rng(40)
        types = [TYPE_U8, TYPE_F16, TYPE_F32]
        while len(pairs) < 40:
            k = len(pairs)
            shape = (int(rng.integers(1, 4)), int(rng.integers(1, 90)), int(rng.integers(1, 90)))
            a, b = random_pair(rng, shape, types[k % 3], types[(k // 3) % 3])
            pairs.append(Pair("rand%d" % k, a, b, kw, (6, 6, 1), want_map=k % 4 != 0))
        alone = [device_call(ctx, [p], kw, metric)[2][0] for p in pairs]
        order = rng.permutation(len(pairs)).tolist()
        _, mets, maps = device_call(ctx, pairs, kw, metric, order=order)
        _, want_mets, _ = device_call(ctx, pairs, kw, order=order)
        assert mets == want_mets
        for j, p in enumerate(pairs):
            if p.blocks:
                assert maps[j].tobytes() == alone[j].tobytes(), p.name
            else:
                assert maps[j] is None
    finally:
        ctx.close()


@pytest.mark.gpu
def test_squared_error_calls_write_what_the_existing_calls_write(gpu):
    """With ASTCENC_B200_BLOCK_SQUARED_ERROR, the whole call writes the bytes of compute_error_metrics_device_images (figures, maps
    and guards) and the list call those of compute_block_errors_device_block_lists."""
    import torch
    dev = torch.device("cuda", 0)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, FLG_DECOMPRESS_ONLY))
    try:
        entries = all_2d_entries(gpu)
        pairs = [p for _, p, _ in entries]
        for kw in (dict(input_components=4, hdr=True, normal=True), dict(input_components=2)):
            got, _, _ = device_call(ctx, pairs, kw, SQUARED)
            want, _, _ = device_call(ctx, pairs, kw)
            assert np.array_equal(got, want)
        rng = np.random.default_rng(8)
        lists = [make_list(rng, p.blocks, KINDS[k % len(KINDS)]) for k, p in enumerate(pairs)]
        d_a = [torch.from_numpy(p.a.reshape(-1).view(np.uint8)).to(dev) for p in pairs]
        d_b = [torch.from_numpy(p.b.reshape(-1).view(np.uint8)).to(dev) for p in pairs]
        d_idx = [torch.from_numpy(l.padded().view(np.int32)).to(dev) for l in lists]
        d_cnt = torch.from_numpy(np.array([l.count for l in lists] + [0], np.uint32).view(np.int32)).to(dev)
        outs = []
        for metric in (SQUARED, None):
            maps = [torch.from_numpy(np.full(p.blocks, MAP_POISON, np.uint32).view(np.int32)).to(dev) for p in pairs]
            table = [(a.data_ptr(), b.data_ptr(), DT[p.a.dtype], DT[p.b.dtype], p.a.shape[2], p.a.shape[1], p.a.shape[0], m.data_ptr(), ix.data_ptr(),
                      d_cnt.data_ptr() + 4 * k, l.capacity) for k, (a, b, p, m, ix, l) in enumerate(zip(d_a, d_b, pairs, maps, d_idx, lists))]
            torch.cuda.synchronize()
            n0 = ctx.launch_count()
            if metric is None:
                ctx.compute_block_errors_device_block_lists(table, input_components=3)
            else:
                ctx.compute_block_metric_device_block_lists(table, metric, input_components=3)
            assert ctx.launch_count() == n0 + 1
            torch.cuda.synchronize()
            outs.append([m.cpu().numpy() for m in maps])
        for k, (x, y) in enumerate(zip(*outs)):
            assert np.array_equal(x, y), pairs[k].name
        assert any(not np.all(x.view(np.uint32) == MAP_POISON) for x in outs[0])
    finally:
        ctx.close()


def refresh_group(gpu, profile, imgs, out_type, metric, kw, rng):
    """Compress `imgs` at -fast, decode, re-encode lists of every kind at -thorough and list-decode them; then a list refresh of
    `metric` into poisoned maps against the whole map of the re-decoded images."""
    import torch
    dev = torch.device("cuda", 0)
    fp = (6, 6, 1)
    fast = gpu.Context(gpu.config_init(profile, 6, 6, PRE_FAST, S))
    thorough = gpu.Context(gpu.config_init(profile, 6, 6, PRE_THOROUGH, S))
    meas = gpu.Context(gpu.config_init(profile, 6, 6, PRE_FAST, FLG_DECOMPRESS_ONLY))      # (decodes the -thorough blocks too)
    try:
        in_type = DT[imgs[0].dtype]
        dims = [(im.shape[1], im.shape[0]) for im in imgs]
        nb = [nblocks((1,) + im.shape[:2], fp) for im in imgs]
        d_img = [torch.from_numpy(im.reshape(-1).view(np.uint8)).to(dev) for im in imgs]
        d_pay = [torch.zeros(n * 16, dtype=torch.uint8, device=dev) for n in nb]
        d_dec = [torch.zeros(im.shape[0] * im.shape[1] * 4 * (2 if out_type == TYPE_F16 else 1), dtype=torch.uint8, device=dev) for im in imgs]
        lists = [make_list(rng, n, KINDS[k % len(KINDS)]) for k, n in enumerate(nb)]
        d_idx = [torch.from_numpy(l.padded().view(np.int32)).to(dev) for l in lists]
        d_cnt = torch.from_numpy(np.array([l.count for l in lists] + [0], np.uint32).view(np.int32)).to(dev)
        fast.compress_device_images([(d.data_ptr(), w, h, 1, p.data_ptr()) for d, (w, h), p in zip(d_img, dims, d_pay)], in_type)
        meas.decompress_device_images([(p.data_ptr(), o.data_ptr(), w, h, 1) for p, o, (w, h) in zip(d_pay, d_dec, dims)], out_type)
        thorough.compress_device_block_lists([(d.data_ptr(), w, h, 1, p.data_ptr(), ix.data_ptr(), d_cnt.data_ptr() + 4 * k, l.capacity)
                                              for k, (d, (w, h), p, ix, l) in enumerate(zip(d_img, dims, d_pay, d_idx, lists))], in_type)
        meas.decompress_device_block_lists([(p.data_ptr(), o.data_ptr(), w, h, 1, ix.data_ptr(), d_cnt.data_ptr() + 4 * k, l.capacity)
                                            for k, (p, o, (w, h), ix, l) in enumerate(zip(d_pay, d_dec, dims, d_idx, lists))], out_type)
        whole = [torch.zeros(n, dtype=torch.float32, device=dev) for n in nb]
        d_met = torch.zeros(len(imgs) * METRICS_BYTES, dtype=torch.uint8, device=dev)
        meas.compute_block_metric_device_images([(d.data_ptr(), o.data_ptr(), in_type, out_type, w, h, 1, d_met.data_ptr() + k * METRICS_BYTES, m.data_ptr())
                                                 for k, (d, o, (w, h), m) in enumerate(zip(d_img, d_dec, dims, whole))], metric, **kw)
        maps = [torch.from_numpy(np.full(n, MAP_POISON, np.uint32).view(np.int32)).to(dev) for n in nb]
        torch.cuda.synchronize()
        n0 = meas.launch_count()
        meas.compute_block_metric_device_block_lists([(d.data_ptr(), o.data_ptr(), in_type, out_type, w, h, 1, m.data_ptr(), ix.data_ptr(),
                                                       d_cnt.data_ptr() + 4 * k, l.capacity)
                                                      for k, (d, o, (w, h), m, ix, l) in enumerate(zip(d_img, d_dec, dims, maps, d_idx, lists))],
                                                     metric, input_components=kw["input_components"])
        assert meas.launch_count() == n0 + 1
        torch.cuda.synchronize()
        for k, (m, wm, l, n) in enumerate(zip(maps, whole, lists, nb)):
            want = np.full(n, MAP_POISON, np.uint32)
            listed = l.listed(n)
            want[listed] = wm.cpu().numpy().view(np.uint32)[listed]
            assert np.array_equal(m.cpu().numpy().view(np.uint32), want), (k, KINDS[k % len(KINDS)])
        # the re-encode changed listed blocks: the refresh measured new decodes
        assert any(len(l.listed(n)) for l, n in zip(lists, nb))
    finally:
        fast.close()
        thorough.close()
        meas.close()


@pytest.mark.gpu
@pytest.mark.parametrize("metric", (SQUARED,) + NEW_METRICS, ids=lambda m: METRIC_IDS[m])
def test_list_refresh_after_a_re_encode_equals_the_whole_map(metric, gpu):
    """Soft-alpha U8 textures and HDR F16 images: after a -thorough list re-encode and a list decode, every listed value is bit for
    bit the whole map's, every other value keeps its poison; garbage past the count, duplicates, count > capacity, count 0,
    capacity 0 and indices out of range."""
    rng = np.random.default_rng(60 + metric)
    ldr = [soft_alpha(h, w, seed=80 + k) for k, (h, w) in enumerate([(96, 131), (64, 64), (37, 29), (120, 77), (13, 50)])]
    refresh_group(gpu, PRF_LDR, ldr, TYPE_U8, metric, dict(input_components=4), rng)
    hdr = [I.hdr_noise(h, w, seed=90 + k, dtype=np.float16) for k, (h, w) in enumerate([(90, 101), (48, 48), (31, 43), (72, 60), (12, 19)])]
    refresh_group(gpu, PRF_HDR, hdr, TYPE_F16, metric, dict(input_components=3, hdr=True), rng)


@pytest.mark.gpu
def test_hdr_log2_loop_on_one_stream_equals_the_host_round_trip(gpu):
    """256^2 hdr_noise in F16, HDR profile: -fast, decode, LOG2 map, select the worst 5 %, -thorough list re-encode, list decode,
    LOG2 list refresh, all on one stream with no host copy. The payload equals the host round trip's (argsort of the downloaded
    map, compress_device_blocks); the map equals a whole LOG2 map of the final decode."""
    import torch
    dev = torch.device("cuda", 0)
    fast = gpu.Context(gpu.config_init(PRF_HDR, 6, 6, PRE_FAST, S))
    thorough = gpu.Context(gpu.config_init(PRF_HDR, 6, 6, PRE_THOROUGH, S))
    meas = gpu.Context(gpu.config_init(PRF_HDR, 6, 6, PRE_FAST, FLG_DECOMPRESS_ONLY))      # (decodes the -thorough blocks too)
    try:
        img = I.hdr_noise(256, 256, seed=33, dtype=np.float16)
        W = H = 256
        n = nblocks((1, H, W), (6, 6, 1))
        cap = n // 20
        d_img = torch.from_numpy(img.reshape(-1).view(np.uint8)).to(dev)
        d_pay = torch.zeros(n * 16, dtype=torch.uint8, device=dev)
        d_dec = torch.zeros(img.nbytes, dtype=torch.uint8, device=dev)
        d_met = torch.zeros(METRICS_BYTES, dtype=torch.uint8, device=dev)
        d_map = torch.zeros(n, dtype=torch.float32, device=dev)
        d_idx = torch.zeros(cap, dtype=torch.int32, device=dev)
        d_cnt = torch.zeros(1, dtype=torch.int32, device=dev)
        h_pay, h_dec, h_map = torch.zeros_like(d_pay), torch.zeros_like(d_dec), torch.zeros_like(d_map)      # the host round trip's
        f_dec, f_map = torch.zeros_like(d_dec), torch.zeros_like(d_map)                                        # the final whole calls'
        st = torch.cuda.Stream(device=dev)
        torch.cuda.synchronize()      # (the buffers are zeroed on the current stream; every call below runs on st)
        s = st.cuda_stream
        kw = dict(hdr=True, input_components=3, stream=s)
        whole = lambda dec, mp: meas.compute_block_metric_device_images([(d_img.data_ptr(), dec.data_ptr(), TYPE_F16, TYPE_F16, W, H, 1, d_met.data_ptr(),
                                                                          mp.data_ptr())], LOG2, **kw)
        fast.compress_device_images([(d_img.data_ptr(), W, H, 1, d_pay.data_ptr())], TYPE_F16, stream=s)
        meas.decompress_device_images([(d_pay.data_ptr(), d_dec.data_ptr(), W, H, 1)], TYPE_F16, stream=s)
        whole(d_dec, d_map)
        meas.select_blocks([(d_map.data_ptr(), n, -np.inf, cap, d_idx.data_ptr(), d_cnt.data_ptr())], stream=s)
        thorough.compress_device_block_lists([(d_img.data_ptr(), W, H, 1, d_pay.data_ptr(), d_idx.data_ptr(), d_cnt.data_ptr(), cap)], TYPE_F16, stream=s)
        meas.decompress_device_block_lists([(d_pay.data_ptr(), d_dec.data_ptr(), W, H, 1, d_idx.data_ptr(), d_cnt.data_ptr(), cap)], TYPE_F16, stream=s)
        meas.compute_block_metric_device_block_lists([(d_img.data_ptr(), d_dec.data_ptr(), TYPE_F16, TYPE_F16, W, H, 1, d_map.data_ptr(), d_idx.data_ptr(),
                                                       d_cnt.data_ptr(), cap)], LOG2, input_components=3, stream=s)
        st.synchronize()
        assert int(d_cnt.cpu()[0]) == cap
        # the host round trip
        fast.compress_device_images([(d_img.data_ptr(), W, H, 1, h_pay.data_ptr())], TYPE_F16, stream=s)
        meas.decompress_device_images([(h_pay.data_ptr(), h_dec.data_ptr(), W, H, 1)], TYPE_F16, stream=s)
        whole(h_dec, h_map)
        st.synchronize()
        fast_pay = h_pay.cpu().numpy()
        m = h_map.cpu().numpy()
        worst = np.sort(np.argsort(-m, kind="stable")[:cap]).astype(np.uint32)
        thorough.compress_device_blocks(d_img.data_ptr(), TYPE_F16, W, H, 1, worst, h_pay.data_ptr(), stream=s)
        st.synchronize()
        assert np.array_equal(np.sort(d_idx.cpu().numpy().astype(np.uint32)), worst), "the device selection differs from argsort"
        assert np.array_equal(d_pay.cpu().numpy(), h_pay.cpu().numpy()), "the payload differs from the host round trip's"
        assert not np.array_equal(d_pay.cpu().numpy(), fast_pay), "the loop left the -fast payload unchanged"
        # the refreshed map is a whole map of the final decode
        meas.decompress_device_images([(d_pay.data_ptr(), f_dec.data_ptr(), W, H, 1)], TYPE_F16, stream=s)
        whole(f_dec, f_map)
        st.synchronize()
        assert np.array_equal(d_dec.cpu().numpy(), f_dec.cpu().numpy()), "the list decode differs from a whole decode"
        assert np.array_equal(d_map.cpu().numpy().view(np.uint32), f_map.cpu().numpy().view(np.uint32)), "the refreshed map differs from a whole map"
        assert float(f_map.sum()) < float(h_map.sum()), "the -thorough re-encode did not lower the summed log2 error"
    finally:
        fast.close()
        thorough.close()
        meas.close()


@pytest.mark.gpu
def test_errors_and_launch_counts(gpu):
    """A block_metric outside 0-2 is ASTCENC_ERR_BAD_PARAM right after input_components: before the fstop, table and entry checks,
    and even for a call that would do nothing. Nothing launches and nothing is written. Otherwise a whole call with a map is three
    launches (two without), a refresh one (none when every capacity is 0)."""
    import torch
    dev = torch.device("cuda", 0)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, FLG_DECOMPRESS_ONLY))
    buf = torch.zeros(65536, dtype=torch.uint8, device=dev)
    base = buf.data_ptr()
    met, mp, idx, cnt = base + 32768, base + 33792, base + 40960, base + 49152
    buf[40960:].zero_()
    poison = torch.from_numpy(np.full(256, MAP_POISON, np.uint32).view(np.uint8)).to(dev)
    l = gpu.lib()
    P = gpu.ERR_BAD_PARAM

    def whole(metric=LOG2, components=4, lo=-10, hi=10, count=2, images=True, **e):
        d = dict(original=base, decoded=base + 16384, original_type=TYPE_U8, decoded_type=TYPE_U8, dim_x=40, dim_y=40, dim_z=1, metrics=met,
                 block_error=mp)
        d.update(e)
        t = (gpu.DeviceMetricsImage * 2)(*[gpu.DeviceMetricsImage(C.c_void_p(d["original"]), C.c_void_p(d["decoded"]), d["original_type"],
                                                                  d["decoded_type"], d["dim_x"], d["dim_y"], d["dim_z"], C.c_void_p(d["metrics"]),
                                                                  C.c_void_p(d["block_error"] or None))] * 2)
        buf[33792:33792 + 1024].copy_(poison)
        torch.cuda.synchronize()
        n0 = ctx.launch_count()
        r = l.astcenc_b200_compute_block_metric_device_images(ctx.handle, 0, 0, components, metric, t if images else None, count, lo, hi, None)
        torch.cuda.synchronize()
        launched = ctx.launch_count() - n0
        if r != 0:
            assert launched == 0 and torch.equal(buf[33792:33792 + 1024], poison)
        return r, launched

    def lists(metric=LOG2, components=4, n=1, capacity=4, **e):
        d = dict(original=base, decoded=base + 16384, original_type=TYPE_U8, decoded_type=TYPE_U8, dim_x=40, dim_y=40, dim_z=1, block_error=mp,
                 indices=idx, count=cnt)
        d.update(e)
        t = (gpu.DeviceBlockErrorList * 1)(gpu.DeviceBlockErrorList(C.c_void_p(d["original"]), C.c_void_p(d["decoded"]), d["original_type"],
                                                                    d["decoded_type"], d["dim_x"], d["dim_y"], d["dim_z"], C.c_void_p(d["block_error"] or None),
                                                                    C.c_void_p(d["indices"] or None), C.c_void_p(d["count"] or None), capacity))
        buf[33792:33792 + 1024].copy_(poison)
        buf[49152:49156].copy_(torch.tensor([3], dtype=torch.int32, device=dev).view(torch.uint8))
        torch.cuda.synchronize()
        n0 = ctx.launch_count()
        r = l.astcenc_b200_compute_block_metric_device_block_lists(ctx.handle, components, metric, t if n else None, n, None)
        torch.cuda.synchronize()
        launched = ctx.launch_count() - n0
        if r != 0:
            assert launched == 0 and torch.equal(buf[33792:33792 + 1024], poison)
        return r, launched

    try:
        for m in (SQUARED, ALPHA, LOG2):
            assert whole(m) == (0, 3)
            assert whole(m, block_error=0) == (0, 2)
            assert whole(m, count=0, images=False) == (0, 0)
            assert lists(m) == (0, 1)
            assert lists(m, capacity=0, block_error=0, indices=0, count=0) == (0, 0)
            assert lists(m, n=0) == (0, 0)
        later = [dict(lo=-126), dict(hi=126), dict(images=False), dict(original=0), dict(metrics=0), dict(dim_x=0), dict(original_type=3),
                 dict(block_error=mp + 2), dict(dim_x=6 * 2 ** 16, dim_y=6 * 2 ** 16)]
        later_lists = [dict(original=0), dict(block_error=0), dict(indices=0), dict(dim_x=0), dict(decoded_type=-1), dict(count=cnt + 1),
                       dict(dim_x=6 * 2 ** 16, dim_y=6 * 2 ** 16)]
        for bad in (3, -1, 0x7FFFFFFF):
            assert whole(bad) == (P, 0)
            assert whole(bad, block_error=0) == (P, 0)
            assert whole(bad, count=0, images=False) == (P, 0)      # (a call that would do nothing)
            assert lists(bad) == (P, 0)
            assert lists(bad, n=0) == (P, 0)
            assert lists(bad, capacity=0, block_error=0, indices=0, count=0) == (P, 0)
            for e in later:
                assert whole(bad, **e) == (P, 0), e
            for e in later_lists:
                assert lists(bad, **e) == (P, 0), e
            for c in (0, 5):
                assert whole(bad, components=c) == (P, 0)
                assert lists(bad, components=c) == (P, 0)
        for e in later:
            assert whole(LOG2, **e) == (P, 0), e
        for e in later_lists:
            assert lists(ALPHA, **e) == (P, 0), e
        assert l.astcenc_b200_compute_block_metric_device_images(None, 0, 0, 4, LOG2, None, 0, -10, 10, None) == P
        assert l.astcenc_b200_compute_block_metric_device_block_lists(None, 4, LOG2, None, 0, None) == P
        with pytest.raises(gpu.AstcencError) as e:
            ctx.compute_block_metric_device_images([], 7)
        assert e.value.code == P
    finally:
        ctx.close()
