"""Normal-map block metrics: ASTCENC_B200_BLOCK_ANGULAR_ERROR and ASTCENC_B200_BLOCK_WORST_ANGULAR_ERROR (metric_angle,
metric_combine and block_error_sum_of<M> in astc_dev_metrics.cuh; astc_block_metric_kernel<4, 5>, astc_block_metric_lists_kernel<4,
5> and the refine decisions of astc_dev_refine.cuh).

CPU: the host simulation's maps (tests/hostsim/hostsim_normal_metric.cpp, one lane and 32 lanes) against a numpy restatement of
the definition in include/astcenc.h, within one float ulp (numpy's and the C library's double acos may differ in the last bit);
list refreshes against the whole maps under every list rule; refine decisions and commits against the keep-the-better rule;
each block's value against the oracle's angular figures of that block's crop; the locality of a value.
GPU: whole maps against the 32-lane simulation, the figures against compute_error_metrics_device_images, list refreshes, keep-
the-better refine calls (unpacked and packed), the worst-angle loop on one stream, the error order and the launch counts."""
import ctypes as C
import os

import numpy as np
import pytest

from astc_ref import *  # noqa: F401,F403
from test_block_list_decode import KINDS, MAP_CASES, MAP_POISON, BlockList, make_list
from hostsim_build import host_sim
from test_block_list_decode import block_texels
from test_block_metrics import LOG2, device_call, sim_metric_lists, sim_metric_map
from test_metrics_device import DT, MAP_SHAPES, METRICS_BYTES, TYPE_PAIRS, Pair, nblocks, random_pair, texel_values
from test_refine_lists import GUARD, POISON, Guarded, State, candidates, old_map, sim_refine, slots
import astc_images as I

ANGULAR, WORST = 4, 5      # enum astcenc_b200_block_metric
ANGLE_METRICS = (ANGULAR, WORST)
METRIC_IDS = {ANGULAR: "angular", WORST: "worst"}
BAD_METRICS = (3, 6, 7, -1, 0x7FFFFFFF)
RRRG = (0, 0, 0, 1)        # the CLI's normal-map encode swizzle
RAZ1 = (0, 3, 6, 5)        # its decode: X from R, Y from A, Z rebuilt, 1
GOLDEN_XY = ("px_ldr-xy-00", "px_ldr-xy-02")
S = FLG_SELF_DECOMPRESS_ONLY


class _AnyMetricSim:
    """tests/hostsim/hostsim_normal_metric.cpp under the names the map, list and refine helpers of test_block_metrics and
    test_refine_lists call: its walks take every metric, the normal-map ones included."""

    def __init__(self, lib):
        self.hostsim_block_metric = lib.hostsim_any_metric
        self.hostsim_block_metric_lists = lib.hostsim_any_metric_lists
        self.hostsim_refine_decide = lib.hostsim_any_metric_refine_decide
        self.hostsim_refine_commit = lib.hostsim_refine_commit


_SIMS = {}


def sim(lanes32=False):
    """The simulation with one simulated lane, or 32 lanes on 32 threads."""
    if lanes32 not in _SIMS:
        lib = host_sim("hostsim_normal_metric", lanes32)
        lib.hostsim_any_metric.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.c_int,
                                           C.c_int, C.c_void_p]
        lib.hostsim_any_metric_lists.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_uint, C.c_uint,
                                                 C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        common = [C.c_void_p, C.c_void_p, C.c_uint, C.c_int, C.c_int, C.c_uint, C.c_uint, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                  C.c_void_p, C.c_void_p, C.c_int, C.c_size_t, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.hostsim_any_metric_refine_decide.argtypes = common + [C.c_int]
        lib.hostsim_refine_commit.argtypes = common + [C.c_void_p]
        _SIMS[lanes32] = _AnyMetricSim(lib)
    return _SIMS[lanes32]


# ---------------------------------------------------------------------------------------------------------------------------
# The numpy restatement
# ---------------------------------------------------------------------------------------------------------------------------
def np_normal(c):
    """metric_normal: (c - 0.5) * 2 of the RGB, normalised in float32; a zero-length vector becomes unit3()."""
    f = np.float32
    x, y, z = [(c[..., k] - f(0.5)) * f(2.0) for k in range(3)]
    ln = (x * x + y * y) + (z * z + f(0.0))
    with np.errstate(invalid="ignore", divide="ignore"):
        s = np.sqrt(ln)
        n = np.stack([x / s, y / s, z / s], axis=-1)
    n[ln == 0] = f(0.57735026918962576451)
    return n


def np_angles(a, b):
    """theta(o, d) of every texel, in float64 degrees."""
    f = np.float32
    n1, n2 = np_normal(texel_values(a)), np_normal(texel_values(b))
    with np.errstate(invalid="ignore"):
        d = (n1[..., 0] * n2[..., 0] + n1[..., 1] * n2[..., 1]) + (n1[..., 2] * n2[..., 2] + f(0.0))
    d = np.fmin(np.fmax(d, f(-1.0)), f(1.0))
    return np.arccos(d.astype(np.float64)) * np.float64(f(180.0) / f(np.pi))


def numpy_angle_map(a, b, fp, metric):
    """One float per block: the sum (ANGULAR) or the largest (WORST) of the angles of the block's texels inside the image."""
    a = a if a.ndim == 4 else a[None]
    b = b if b.ndim == 4 else b[None]
    t = np_angles(a, b)
    D, H, W = a.shape[:3]
    bx, by, bz = fp
    gz = -(-D // bz) * bz if bz > 1 else D
    pad = np.zeros((gz, -(-H // by) * by, -(-W // bx) * bx), np.float64)      # (outside texels: 0, neutral to both)
    pad[:D, :H, :W] = t
    blocks = pad.reshape(gz // bz, bz, pad.shape[1] // by, by, pad.shape[2] // bx, bx)
    v = blocks.sum(axis=(1, 3, 5)) if metric == ANGULAR else blocks.max(axis=(1, 3, 5))
    return v.reshape(-1).astype(np.float32)


def assert_within_ulp(got, want, what):
    """Bit patterns of non-negative floats differ by at most one."""
    assert got.shape == want.shape, what
    assert np.all(got >= 0) and np.all(want >= 0), what
    d = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
    assert d.max(initial=0) <= 1, (what, int(np.argmax(d)), got[np.argmax(d)], want[np.argmax(d)])


def special_pair(dtype):
    """Zero-length normals (texels of 0.5), NaN, inf, negative and out-of-range texels, against decodes of the same kinds."""
    vals = np.array([0.5, 0.5, 0.5, 1.0, np.nan, 0.0, 1.0, 2.0, -1.0, 70000.0 if dtype == np.float32 else 65504.0, np.inf, 0.25], np.float64)
    rng = np.random.default_rng(3)
    a = rng.choice(vals, (2, 11, 13, 4)).astype(dtype)
    b = rng.choice(vals, (2, 11, 13, 4)).astype(dtype)
    a[0, :3, :3, :3] = 0.5      # a whole zero-length region, against itself and against the decode
    b[0, :2, :2, :3] = 0.5
    return a, b


def normal_map(h, w, seed):
    """A U8 normal map: central differences of a smooth height field, normalised and packed as (n + 1) / 2; alpha 255."""
    rng = np.random.default_rng(seed)
    g = rng.standard_normal((h // 8 + 3, w // 8 + 3))
    yy, xx = np.linspace(0, g.shape[0] - 2.01, h), np.linspace(0, g.shape[1] - 2.01, w)
    y0, x0 = yy.astype(int), xx.astype(int)
    fy, fx = (yy - y0)[:, None], (xx - x0)[None, :]
    ht = (g[y0][:, x0] * (1 - fy) * (1 - fx) + g[y0 + 1][:, x0] * fy * (1 - fx) + g[y0][:, x0 + 1] * (1 - fy) * fx + g[y0 + 1][:, x0 + 1] * fy * fx) * 6
    dx = np.gradient(ht, axis=1)
    dy = np.gradient(ht, axis=0)
    n = np.stack([-dx, -dy, np.ones_like(ht)], axis=-1)
    n /= np.linalg.norm(n, axis=-1, keepdims=True)
    out = np.full((h, w, 4), 255, np.uint8)
    out[..., :3] = np.clip(np.rint((n + 1) * 0.5 * 255), 0, 255).astype(np.uint8)
    return out


def golden_xy():
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_images.npz"))
    return [(name, np.ascontiguousarray(g[name])) for name in GOLDEN_XY]


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ANGLE_METRICS, ids=lambda m: METRIC_IDS[m])
@pytest.mark.parametrize("lanes32", [False, True], ids=["lanes1", "lanes32"])
def test_hostsim_angle_maps_equal_numpy(lanes32, metric):
    """The map shapes and type pairs of the other metrics (inf, NaN, out-of-range texels), zero-length normals, a texture array
    and 4x4x4 footprints: within one float ulp of numpy, and the same bits for input_components 1-4."""
    lib = sim(lanes32)
    rng = np.random.default_rng(31 + metric)
    cases = [(fp, random_pair(rng, shape, t1, t2)) for fp, shape in MAP_SHAPES for t1, t2 in TYPE_PAIRS]
    cases += [(fp, special_pair(dt)) for fp in ((6, 6, 1), (4, 4, 4)) for dt in (np.float16, np.float32)]
    for k, (fp, (a, b)) in enumerate(cases):
        want = numpy_angle_map(a, b, fp, metric)
        maps = [sim_metric_map(lib, a, b, fp, c, metric) for c in ((1, 2, 3, 4) if not lanes32 or k % 4 == 0 else (k % 4 + 1,))]
        assert_within_ulp(maps[0], want, (k, fp, a.shape, a.dtype, b.dtype))
        for m in maps[1:]:
            assert np.array_equal(m.view(np.uint32), maps[0].view(np.uint32)), (k, "input_components changed the map")


def test_numpy_angle_special_values():
    """Identical normals give 0, opposite ones 180, a NaN texel reads as 0 (metric_texel's clamp) and zero-length normals both
    become unit3()."""
    f = np.float32
    a = np.array([[0.9, 0.2, 0.7, 1], [1.0, 0.5, 0.5, 1], [np.nan, 0.5, 0.5, 1], [0.5, 0.5, 0.5, 1]], f)
    b = np.array([[0.9, 0.2, 0.7, 1], [0.0, 0.5, 0.5, 1], [0.0, 0.5, 0.5, 1], [0.5, 0.5, 0.5, 1]], f)
    t = np_angles(a, b)
    assert t[0] < 0.03 and t[1] == pytest.approx(180.0, abs=1e-4) and t[2] < 0.03 and t[3] < 0.03


@pytest.mark.parametrize("metric", ANGLE_METRICS, ids=lambda m: METRIC_IDS[m])
@pytest.mark.parametrize("lanes32", [False, True], ids=["lanes1", "lanes32"])
@pytest.mark.parametrize("fp,shapes", MAP_CASES, ids=["6x6", "4x4x4"])
def test_hostsim_list_refresh_equals_the_whole_map_at_listed_blocks(fp, shapes, lanes32, metric):
    """Mixed types and every list kind (count above capacity, out-of-range indices, duplicates, count 0, capacity 0): listed values
    equal the simulation's whole map bit for bit, every other value keeps its poison."""
    lib = sim(lanes32)
    rng = np.random.default_rng(43 + metric)
    types = [(TYPE_U8, TYPE_U8), (TYPE_F16, TYPE_F16), (TYPE_F32, TYPE_U8), (TYPE_U8, TYPE_F16), (TYPE_F16, TYPE_F32)]
    pairs = [random_pair(rng, s, *types[k % len(types)]) for k, s in enumerate(shapes)]
    kinds = [KINDS[k % len(KINDS)] for k in range(len(shapes))]
    lists = [make_list(rng, nblocks(s, fp), k) for s, k in zip(shapes, kinds)]
    maps = [np.full(nblocks(s, fp), MAP_POISON, np.uint32).view(np.float32) for s in shapes]
    sim_metric_lists(lib, pairs, fp, 3, metric, lists, maps)
    for k, ((a, b), s, l, m) in enumerate(zip(pairs, shapes, lists, maps)):
        want = np.full(nblocks(s, fp), MAP_POISON, np.uint32)
        listed = l.listed(len(want))
        want[listed] = sim_metric_map(lib, a, b, fp, 3, metric).view(np.uint32)[listed]
        assert np.array_equal(m.view(np.uint32), want), "pair %d %s (%s list)" % (k, s, kinds[k])


@pytest.mark.parametrize("metric", ANGLE_METRICS, ids=lambda m: METRIC_IDS[m])
@pytest.mark.parametrize("lanes32", [False, True], ids=["lanes1", "lanes32"])
def test_hostsim_refine_keeps_the_better_block(oracle, lanes32, metric):
    """Oracle -medium candidates of U8 normal maps (ragged, a texture array) decoded to U8, lists of several kinds, and old maps
    below, equal to, above, NaN, inf and 0 against the candidate values, in one chunk: each valid slot's value is bit for bit the
    whole-map simulation's on the candidate's decode, and exactly the blocks whose value is below the old one get the candidate's
    bytes, texels and value; every other byte keeps its poison or its old value."""
    lib = sim(lanes32)
    rng = np.random.default_rng(17 + metric)
    fp = (6, 6, 1)
    imgs = [normal_map(37, 29, seed=1)[None], np.stack([normal_map(13, 17, seed=2 + z) for z in range(3)]), normal_map(25, 31, seed=6)[None]]
    shapes = [a.shape[:3] for a in imgs]
    pays, decs = zip(*[candidates(oracle, a, fp, PRF_LDR, PRE_MEDIUM, TYPE_U8) for a in imgs])
    lists = [make_list(rng, nblocks(s, fp), kind) for s, kind in zip(shapes, ("mixed", "sorted", "past"))]
    want = [sim_metric_map(lib, a, d, fp, 3, metric) for a, d in zip(imgs, decs)]
    maps = [old_map(rng, w) for w in want]
    call = slots(lists, shapes, fp)
    out_pay, out_dec, out_map, values = sim_refine(lib, imgs, pays, decs, fp, 3, metric, lists, maps, len(call), True, rng)
    for s, (j, b) in enumerate(call):
        if b is not None:
            assert values[s].view(np.uint32) == want[j][b].view(np.uint32), (s, j, b)
    committed = 0
    for j, (s, l) in enumerate(zip(shapes, lists)):
        listed = np.unique(l.listed(nblocks(s, fp)))
        keep = listed[want[j][listed] < maps[j][listed]]
        exp_map = maps[j].copy()
        exp_map[keep] = want[j][keep]
        assert np.array_equal(out_map[j].view(np.uint32), exp_map.view(np.uint32)), j
        exp_pay = np.full(len(out_pay[j]), POISON, np.uint8)
        for k in keep:
            exp_pay[16 * k:16 * k + 16] = pays[j][k]
        assert np.array_equal(out_pay[j], exp_pay), j
        exp_dec = np.full(decs[j].shape, POISON, np.uint8)
        mask = block_texels(s, fp, keep)
        exp_dec[mask] = decs[j][mask]
        assert np.array_equal(out_dec[j], exp_dec), j
        committed += len(keep)
    assert committed > 0


def oracle_round_trips(oracle):
    """The golden LDR-XY images through the oracle at 6x6 -fast, MAP_NORMAL with the rrrg swizzle, decoded to (R, A, Z, 1)."""
    out = []
    for name, img in golden_xy():
        h, w = img.shape[:2]
        pay = oracle.compress(img, PRF_LDR, 6, 6, PRE_FAST, FLG_MAP_NORMAL, swz=RRRG)
        dec = oracle.decompress(pay, w, h, PRF_LDR, 6, 6, out_type=TYPE_U8, flags=FLG_MAP_NORMAL, swz=RAZ1)
        out.append((name, img, dec))
    return out


def test_block_values_equal_the_oracle_figures_of_each_block(oracle):
    """Each 6x6 block cropped and measured by the oracle as its own image: mean_angular_error * texels is the ANGULAR value within
    1e-6 relative, worst_angular_error the WORST value within one float ulp."""
    lib = sim()
    checked = 0
    for name, a, b in oracle_round_trips(oracle):
        h, w = a.shape[:2]
        maps = {m: sim_metric_map(lib, a, b, (6, 6, 1), 3, m) for m in ANGLE_METRICS}
        bxs = -(-w // 6)
        for k in range(len(maps[ANGULAR])):
            y0, x0 = (k // bxs) * 6, (k % bxs) * 6
            ca, cb = a[y0:y0 + 6, x0:x0 + 6], b[y0:y0 + 6, x0:x0 + 6]
            fig = oracle.error_metrics(ca, cb, normal=True, components=3)
            texels = ca.shape[0] * ca.shape[1]
            assert float(maps[ANGULAR][k]) == pytest.approx(fig["mean_angular_error"] * texels, rel=1e-6, abs=1e-30), (name, k)
            assert_within_ulp(maps[WORST][k:k + 1], np.array([fig["worst_angular_error"]], np.float32), (name, k))
            checked += 1
        assert np.max(maps[WORST]) > 1.0, name      # (the round trip is lossy)
    assert checked == 2 * 43 * 43


@pytest.mark.parametrize("metric", ANGLE_METRICS, ids=lambda m: METRIC_IDS[m])
def test_angle_metric_depends_only_on_the_block(metric):
    """Changing the texels of one block moves that block's value and no other."""
    lib = sim()
    img = normal_map(20, 25, seed=4)
    a, b = np.stack([img, img[::-1]]), np.stack([img[:, ::-1], img]).copy()
    before = sim_metric_map(lib, a, b, (6, 6, 1), 4, metric)
    b2 = b.copy()
    b2[1, 6:12, 12:18, :3] ^= 0x35      # block (slice 1, row 1, col 2)
    after = sim_metric_map(lib, a, b2, (6, 6, 1), 4, metric)
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


def gpu_round_trips(gpu):
    """(name, Pair, kw): the golden LDR-XY images at 6x6 -fast with MAP_NORMAL and rrrg, decoded with (R, A, Z, 1) into U8 and
    F16; a texture array of generated normal maps; their input_components vary."""
    fp = (6, 6, 1)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, FLG_MAP_NORMAL | S))
    out = []
    try:
        for k, (name, img) in enumerate(golden_xy()):
            h, w = img.shape[:2]
            pay = ctx.compress_image(img, swizzle=RRRG)
            for dt in (np.uint8, np.float16):
                kw = dict(normal=True, input_components=(3, 4)[k])
                out.append(("%s_%s" % (name, np.dtype(dt).name), Pair(name, img, ctx.decompress_image(pay, w, h, dtype=dt, swizzle=RAZ1), kw, fp), kw))
        arr = np.stack([normal_map(67, 93, seed=50 + z) for z in range(3)])
        dec = ctx.decompress_image(ctx.compress_image(arr, swizzle=RRRG), 93, 67, swizzle=RAZ1, dim_z=3)
        kw = dict(normal=True, input_components=2)
        out.append(("array", Pair("array", arr, dec, kw, fp), kw))
    finally:
        ctx.close()
    return out


def figures_and_map_agree(mets, mp, metric, pixels, what):
    got = ErrorMetrics.from_buffer_copy(mets)
    if metric == WORST:
        assert np.max(mp) == np.float32(got.worst_angular_error), what
    else:
        assert float(mp.astype(np.float64).sum()) / pixels == pytest.approx(got.mean_angular_error, rel=1e-6), what


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ANGLE_METRICS, ids=lambda m: METRIC_IDS[m])
def test_whole_maps_equal_the_32_lane_simulation(metric, gpu):
    """Each pair alone: the map within one float ulp of the 32-lane simulation, the figures bit for bit those of
    compute_error_metrics_device_images, max(WORST) == (float)worst_angular_error and sum(ANGULAR) / pixels == mean_angular_error
    within 1e-6; then a 4x4x4 volume, and a shuffled 40-entry table whose maps are bit for bit those of each entry alone."""
    lib = sim(True)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, FLG_DECOMPRESS_ONLY))
    try:
        entries = gpu_round_trips(gpu)
        for name, p, kw in entries:
            _, (mets,), (mp,) = device_call(ctx, [p], kw, metric)
            _, (want_mets,), _ = device_call(ctx, [p], kw)
            assert mets == want_mets, name
            assert_within_ulp(mp, sim_metric_map(lib, p.a, p.b, (6, 6, 1), kw["input_components"], metric), name)
            figures_and_map_agree(mets, mp, metric, p.a.shape[0] * p.a.shape[1] * p.a.shape[2], name)
        pairs = [p for _, p, _ in entries]
        rng = np.random.default_rng(40)
        types = [TYPE_U8, TYPE_F16, TYPE_F32]
        while len(pairs) < 40:
            k = len(pairs)
            shape = (int(rng.integers(1, 4)), int(rng.integers(1, 90)), int(rng.integers(1, 90)))
            a, b = random_pair(rng, shape, types[k % 3], types[(k // 3) % 3])
            pairs.append(Pair("rand%d" % k, a, b, {}, (6, 6, 1), want_map=k % 4 != 0))
        kw = dict(normal=True, input_components=4)
        alone = [device_call(ctx, [p], kw, metric)[2][0] for p in pairs]
        order = rng.permutation(len(pairs)).tolist()
        _, mets, maps = device_call(ctx, pairs, kw, metric, order=order)
        _, want_mets, _ = device_call(ctx, pairs, kw, order=order)
        assert mets == want_mets
        for j, p in enumerate(pairs):
            assert (maps[j] is None) == (p.blocks == 0)
            if p.blocks:
                assert maps[j].tobytes() == alone[j].tobytes(), p.name
    finally:
        ctx.close()
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 4, 4, PRE_FAST, FLG_MAP_NORMAL | S, block_z=4))
    try:
        v = np.stack([normal_map(21, 19, seed=60 + z) for z in range(9)])
        dec = ctx.decompress_image(ctx.compress_image(v, swizzle=RRRG), 19, 21, swizzle=RAZ1, dim_z=9)
        kw = dict(normal=True, input_components=3)
        p = Pair("volume", v, dec, kw, (4, 4, 4))
        _, (mets,), (mp,) = device_call(ctx, [p], kw, metric)
        _, (want_mets,), _ = device_call(ctx, [p], kw)
        assert mets == want_mets
        assert_within_ulp(mp, sim_metric_map(lib, v, dec, (4, 4, 4), 3, metric), "volume")
        figures_and_map_agree(mets, mp, metric, v.shape[0] * v.shape[1] * v.shape[2], "volume")
    finally:
        ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ANGLE_METRICS, ids=lambda m: METRIC_IDS[m])
def test_list_refresh_equals_the_whole_map(metric, gpu):
    """After a -thorough list re-encode and a list decode, a refresh into poisoned maps inside guard bytes: every listed value is
    bit for bit the whole map's, every other value keeps its poison, under every list kind."""
    import torch
    rng = np.random.default_rng(70 + metric)
    fp = (6, 6, 1)
    imgs = [normal_map(h, w, seed=80 + k) for k, (h, w) in enumerate([(96, 131), (64, 64), (37, 29), (120, 77), (13, 50)])]
    fast = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, FLG_MAP_NORMAL))      # (it decodes the -thorough blocks too)
    thorough = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_THOROUGH, FLG_MAP_NORMAL | S))
    try:
        states = [State(im, make_list(rng, nblocks((1,) + im.shape[:2], fp), KINDS[k % len(KINDS)]), fp, TYPE_U8) for k, im in enumerate(imgs)]
        fast.compress_device_images([(s.d_img.data_ptr(), *s.dims(), s.pay.ptr) for s in states], TYPE_U8, swizzle=RRRG)
        fast.decompress_device_images([(s.pay.ptr, s.dec.ptr, *s.dims()) for s in states], TYPE_U8, swizzle=RAZ1)
        thorough.compress_device_block_lists([(s.d_img.data_ptr(), *s.dims(), s.pay.ptr, s.d_idx.data_ptr(), s.d_cnt.data_ptr(), s.lst.capacity)
                                              for s in states], TYPE_U8, swizzle=RRRG)
        fast.decompress_device_block_lists([(s.pay.ptr, s.dec.ptr, *s.dims(), s.d_idx.data_ptr(), s.d_cnt.data_ptr(), s.lst.capacity) for s in states],
                                           TYPE_U8, swizzle=RAZ1)
        met = torch.zeros(len(states) * METRICS_BYTES, dtype=torch.uint8, device="cuda")
        fast.compute_block_metric_device_images([(s.d_img.data_ptr(), s.dec.ptr, TYPE_U8, TYPE_U8, *s.dims(), met.data_ptr() + k * METRICS_BYTES, s.map.ptr)
                                                 for k, s in enumerate(states)], metric, input_components=3)
        refreshed = [Guarded(s.map.n, np.full(s.blocks, MAP_POISON, np.uint32)) for s in states]
        torch.cuda.synchronize()
        n0 = fast.launch_count()
        fast.compute_block_metric_device_block_lists([(s.d_img.data_ptr(), s.dec.ptr, TYPE_U8, TYPE_U8, *s.dims(), r.ptr, s.d_idx.data_ptr(),
                                                       s.d_cnt.data_ptr(), s.lst.capacity) for s, r in zip(states, refreshed)], metric, input_components=3)
        assert fast.launch_count() == n0 + 1
        torch.cuda.synchronize()
        for k, (s, r) in enumerate(zip(states, refreshed)):
            want = np.full(s.blocks, MAP_POISON, np.uint32)
            listed = s.lst.listed(s.blocks)
            want[listed] = s.map.get().view(np.uint32)[listed]
            assert np.array_equal(r.get().view(np.uint32), want), (k, KINDS[k % len(KINDS)])
        assert any(len(s.lst.listed(s.blocks)) for s in states)
    finally:
        fast.close()
        thorough.close()


def refine_states(gpu, fast, imgs, lists, fp, metric, out_type, stream=0):
    """States with a -fast payload (rrrg), its (R, A, Z, 1) decode and the whole map of `metric`."""
    import torch
    states = [State(a, l, fp, out_type) for a, l in zip(imgs, lists)]
    fast.compress_device_images([(s.d_img.data_ptr(), *s.dims(), s.pay.ptr) for s in states], TYPE_U8, swizzle=RRRG, stream=stream)
    fast.decompress_device_images([(s.pay.ptr, s.dec.ptr, *s.dims()) for s in states], out_type, swizzle=RAZ1, stream=stream)
    met = torch.zeros(len(states) * 128, dtype=torch.uint8, device="cuda")
    fast.compute_block_metric_device_images([(s.d_img.data_ptr(), s.dec.ptr, TYPE_U8, out_type, *s.dims(), met.data_ptr() + 128 * k, s.map.ptr)
                                             for k, s in enumerate(states)], metric, input_components=3, stream=stream)
    torch.cuda.synchronize()      # (met is freed on return, and the calls run on the context's stream, not torch's)
    return states


def refine_tuples(states):
    return [(s.d_img.data_ptr(), *s.dims(), s.pay.ptr, s.dec.ptr, s.map.ptr, s.d_idx.data_ptr(), s.d_cnt.data_ptr(), s.lst.capacity) for s in states]


def whole_again(ctx, s, metric, out_type):
    """A whole decode of the state's payload and a whole map of that decode."""
    import torch
    dec, mp = Guarded(s.dec.n), Guarded(s.map.n)
    met = torch.zeros(128, dtype=torch.uint8, device="cuda")
    ctx.decompress_device_images([(s.pay.ptr, dec.ptr, *s.dims())], out_type, swizzle=RAZ1)
    ctx.compute_block_metric_device_images([(s.d_img.data_ptr(), dec.ptr, TYPE_U8, out_type, *s.dims(), met.data_ptr(), mp.ptr)], metric, input_components=3)
    torch.cuda.synchronize()
    return dec.get(), mp.get().view(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ANGLE_METRICS, ids=lambda m: METRIC_IDS[m])
def test_refine_keeps_the_better_block(metric, gpu):
    """A -thorough refine round (unpacked, and packed with a budget at least the listed total) over every list kind, decoded to U8
    and to F16: afterwards the map is bit for bit a whole map of a whole decode of the payload, the decode is that decode, no
    value rose, some blocks were committed, and packed equals unpacked byte for byte."""
    import torch
    rng = np.random.default_rng(90 + metric)
    fp = (6, 6, 1)
    imgs = [normal_map(h, w, seed=100 + k) for k, (h, w) in enumerate([(97, 131), (64, 64), (37, 29), (120, 77), (13, 50)])]
    imgs[0] = golden_xy()[0][1]
    fast = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, FLG_MAP_NORMAL))      # (it decodes the -thorough blocks too)
    thorough = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_THOROUGH, FLG_MAP_NORMAL | S))
    try:
        for out_type in (TYPE_U8, TYPE_F16):
            lists = [make_list(rng, nblocks((1,) + a.shape[:2], fp), KINDS[k % len(KINDS)]) for k, a in enumerate(imgs)]
            lists[0] = BlockList(np.argsort(rng.random(nblocks((1, 256, 256), fp)))[:300].astype(np.uint32), 300, 300)
            unpacked = refine_states(gpu, fast, imgs, lists, fp, metric, out_type)
            packed = refine_states(gpu, fast, imgs, lists, fp, metric, out_type)
            torch.cuda.synchronize()
            before = [s.map.get().view(np.float32) for s in unpacked]
            thorough.refine_device_block_lists(refine_tuples(unpacked), TYPE_U8, out_type, metric, swizzle=RRRG, decode_swizzle=RAZ1, input_components=3)
            total = sum(min(l.count, l.capacity) for l in lists)      # (every listed slot, in range or not)
            thorough.refine_device_block_lists_packed(refine_tuples(packed), total, TYPE_U8, out_type, metric, swizzle=RRRG, decode_swizzle=RAZ1,
                                                      input_components=3)
            torch.cuda.synchronize()
            committed = 0
            for k, (u, p, b) in enumerate(zip(unpacked, packed, before)):
                pay, dec, mp = u.host()
                assert np.all(mp <= b), (k, "a map value rose")
                committed += int(np.sum(mp < b))
                wdec, wmap = whole_again(fast, u, metric, out_type)
                assert np.array_equal(wdec, dec), (k, "the decode differs from a whole decode of the payload")
                assert np.array_equal(wmap.view(np.uint32), mp.view(np.uint32)), (k, "the map differs from a whole map of the decode")
                ppay, pdec, pmp = p.host()
                assert np.array_equal(pay, ppay) and np.array_equal(dec, pdec) and np.array_equal(mp.view(np.uint32), pmp.view(np.uint32)), (k, "packed")
            assert committed > 0
    finally:
        fast.close()
        thorough.close()


@pytest.mark.gpu
def test_worst_angle_loop_on_one_stream(gpu):
    """No texel worse than T degrees: a WORST map of a -fast normal map, then three rounds enqueued up front on one stream, each
    select_blocks with threshold T and a capacity, then a -thorough refine with WORST. Snapshots taken on the stream show the
    number of blocks above T never rising, each round listing exactly the blocks above T (up to the capacity), and every block
    that changed lowering its value."""
    import torch
    fp = (6, 6, 1)
    img = normal_map(256, 256, seed=7)
    n = nblocks((1, 256, 256), fp)
    fast = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, FLG_MAP_NORMAL))      # (it decodes the -thorough blocks too)
    thorough = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_THOROUGH, FLG_MAP_NORMAL | S))
    try:
        cap = n // 10
        st = State(img, BlockList(np.zeros(cap, np.uint32), 0, cap), fp, TYPE_U8)
        stream = torch.cuda.Stream()
        s = stream.cuda_stream
        torch.cuda.synchronize()
        fast.compress_device_images([(st.d_img.data_ptr(), 256, 256, 1, st.pay.ptr)], TYPE_U8, swizzle=RRRG, stream=s)
        fast.decompress_device_images([(st.pay.ptr, st.dec.ptr, 256, 256, 1)], TYPE_U8, swizzle=RAZ1, stream=s)
        met = torch.zeros(128, dtype=torch.uint8, device="cuda")
        fast.compute_block_metric_device_images([(st.d_img.data_ptr(), st.dec.ptr, TYPE_U8, TYPE_U8, 256, 256, 1, met.data_ptr(), st.map.ptr)], WORST,
                                                input_components=3, stream=s)
        stream.synchronize()
        first = st.map.get().view(np.float32)
        T = float(np.percentile(first, 80))
        snaps, idx_snaps, cnt_snaps = [], [], []
        m_view = st.map.buf[GUARD:GUARD + 4 * n]
        with torch.cuda.stream(stream):
            snaps.append(m_view.clone())
            for r in range(3):
                thorough.select_blocks([(st.map.ptr, n, T, cap, st.d_idx.data_ptr(), st.d_cnt.data_ptr())], stream=s)
                cnt_snaps.append(st.d_cnt.clone())
                idx_snaps.append(st.d_idx.clone())
                thorough.refine_device_block_lists([(st.d_img.data_ptr(), 256, 256, 1, st.pay.ptr, st.dec.ptr, st.map.ptr, st.d_idx.data_ptr(),
                                                     st.d_cnt.data_ptr(), cap)], TYPE_U8, TYPE_U8, WORST, swizzle=RRRG, decode_swizzle=RAZ1,
                                                   input_components=3, stream=s)
                snaps.append(m_view.clone())
        stream.synchronize()
        maps = [x.cpu().numpy().view(np.float32) for x in snaps]
        above = [int(np.sum(m > T)) for m in maps]
        assert above[0] > 0
        for r in range(3):
            prev, cur = maps[r], maps[r + 1]
            assert above[r + 1] <= above[r], above
            changed = cur.view(np.uint32) != prev.view(np.uint32)
            assert np.all(cur[changed] < prev[changed]), r
            k = int(cnt_snaps[r].cpu()[0])
            listed = np.sort(idx_snaps[r].cpu().numpy().view(np.uint32)[:min(k, cap)])
            cand = np.nonzero(prev > T)[0]
            assert k == min(len(cand), cap) and np.all(np.isin(listed, cand)), r
            assert not np.any(changed & ~np.isin(np.arange(n), listed)), r
        assert above[-1] < above[0], above
    finally:
        fast.close()
        thorough.close()


@pytest.mark.gpu
def test_errors_launch_counts_and_the_mean_angle_gate(gpu):
    """Metrics 3, 6, 7, -1 and 0x7FFFFFFF are ASTCENC_ERR_BAD_PARAM on every entry point that takes a metric, right after
    input_components (before the later checks, even for a call that would do nothing), with nothing launched and nothing written.
    4 and 5 launch what LOG2_ERROR launches. A total_block_maps gate with limit = D * pixels on an ANGULAR map zeroes the
    weight exactly when the total is at most the limit."""
    import torch
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, FLG_MAP_NORMAL))
    dec_only = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, FLG_DECOMPRESS_ONLY))
    buf = torch.full((1 << 17,), 0x33, dtype=torch.uint8, device="cuda")
    base = buf.data_ptr()
    data, dec, pay, met, mp, idx, cnt, ovf = base, base + 8192, base + 16384, base + 32768, base + 33792, base + 40960, base + 49152, base + 49664
    buf[cnt - base:cnt - base + 4].copy_(torch.tensor([3], dtype=torch.int32, device="cuda").view(torch.uint8))
    buf[idx - base:idx - base + 16].copy_(torch.tensor([0, 1, 2, 3], dtype=torch.int32, device="cuda").view(torch.uint8))
    l = gpu.lib()
    P = gpu.ERR_BAD_PARAM
    swz = gpu.Swizzle(0, 1, 2, 3)

    def run(c, f):
        before = buf.cpu()
        torch.cuda.synchronize()
        n0 = c.launch_count()
        r = f()
        torch.cuda.synchronize()
        launched = c.launch_count() - n0
        if r != 0:
            assert launched == 0 and torch.equal(buf.cpu(), before), "an error launched or wrote something"
        return r, launched

    def whole(metric, comps=4, count=1, lo=-10, **e):
        d = dict(original=data, decoded=dec, dim_x=40)
        d.update(e)
        t = (gpu.DeviceMetricsImage * 1)(gpu.DeviceMetricsImage(C.c_void_p(d["original"] or None), C.c_void_p(d["decoded"]), TYPE_U8, TYPE_U8, d["dim_x"],
                                                                40, 1, C.c_void_p(met), C.c_void_p(mp)))
        return run(dec_only, lambda: l.astcenc_b200_compute_block_metric_device_images(dec_only.handle, 0, 1, comps, metric, t if count else None, count,
                                                                                       lo, 10, None))

    def lists(metric, comps=4, count=1, **e):
        d = dict(original=data, dim_x=40)
        d.update(e)
        t = (gpu.DeviceBlockErrorList * 1)(gpu.DeviceBlockErrorList(C.c_void_p(d["original"] or None), C.c_void_p(dec), TYPE_U8, TYPE_U8, d["dim_x"], 40, 1,
                                                                    C.c_void_p(mp), C.c_void_p(idx), C.c_void_p(cnt), 4))
        return run(dec_only, lambda: l.astcenc_b200_compute_block_metric_device_block_lists(dec_only.handle, comps, metric, t if count else None, count, None))

    def refine(metric, packed=False, comps=4, count=1, **e):
        d = dict(data=data, dim_x=40)
        d.update(e)
        t = (gpu.DeviceRefineList * 1)(gpu.DeviceRefineList(C.c_void_p(d["data"] or None), d["dim_x"], 40, 1, C.c_void_p(pay), C.c_void_p(dec), C.c_void_p(mp),
                                                            C.c_void_p(idx), C.c_void_p(cnt), 4))
        tt = t if count else None
        if packed:
            return run(ctx, lambda: l.astcenc_b200_refine_device_block_lists_packed(ctx.handle, tt, count, 8, C.c_void_p(ovf), TYPE_U8, C.byref(swz), TYPE_U8,
                                                                                   C.byref(swz), comps, metric, None))
        return run(ctx, lambda: l.astcenc_b200_refine_device_block_lists(ctx.handle, tt, count, TYPE_U8, C.byref(swz), TYPE_U8, C.byref(swz), comps, metric,
                                                                        None))

    try:
        for m in ANGLE_METRICS:
            assert whole(m) == whole(LOG2) == (0, 3)
            assert whole(m, count=0) == (0, 0)
            assert lists(m) == lists(LOG2) == (0, 1)
            assert refine(m) == refine(LOG2)
            assert refine(m)[0] == 0 and refine(m)[1] > 0
            assert refine(m, packed=True) == refine(LOG2, packed=True)
            assert refine(m, packed=True)[0] == 0
        for bad in BAD_METRICS:
            for later in (dict(), dict(count=0), dict(lo=-126), dict(original=0), dict(dim_x=0)):
                assert whole(bad, **later) == (P, 0), (bad, later)
            for later in (dict(), dict(count=0), dict(original=0), dict(dim_x=0)):
                assert lists(bad, **later) == (P, 0), (bad, later)
            for packed in (False, True):
                for later in (dict(), dict(count=0), dict(data=0), dict(dim_x=0)):
                    assert refine(bad, packed, **later) == (P, 0), (bad, packed, later)
            for c in (0, 5):      # (input_components is checked first: the same error)
                assert whole(bad, comps=c) == (P, 0) and lists(bad, comps=c) == (P, 0) and refine(bad, comps=c) == (P, 0)
        with pytest.raises(gpu.AstcencError) as e:
            ctx.compute_block_metric_device_images([], 3)
        assert e.value.code == P
        # the mean-angle gate
        img = golden_xy()[0][1]
        h, w = img.shape[:2]
        blocks = nblocks((1, h, w), (6, 6, 1))
        st, = refine_states(gpu, ctx, [img], [BlockList(np.zeros(1, np.uint32), 0, 1)], (6, 6, 1), ANGULAR, TYPE_U8)
        figs = torch.zeros(128, dtype=torch.uint8, device="cuda")
        ctx.compute_error_metrics_device_images([(st.d_img.data_ptr(), st.dec.ptr, TYPE_U8, TYPE_U8, w, h, 1, figs.data_ptr(), 0)], normal=True,
                                                input_components=3)
        torch.cuda.synchronize()
        mean = ErrorMetrics.from_buffer_copy(figs.cpu().numpy()[:METRICS_BYTES].tobytes()).mean_angular_error
        assert mean > 0
        out = torch.zeros(64, dtype=torch.float64, device="cuda")
        ws = torch.zeros(64, dtype=torch.float32, device="cuda")
        total_ptr, w_ptr = out.data_ptr(), ws.data_ptr()
        limits = [D * h * w for D in (0.0, mean * 0.99, mean * 1.01, 2 * mean)]
        ctx.total_block_maps([(st.map.ptr, blocks, lim, total_ptr + 8 * k, w_ptr + 4 * k) for k, lim in enumerate(limits)], gpu.WEIGHT_ONE)
        torch.cuda.synchronize()
        totals, weights = out.cpu().numpy()[:len(limits)], ws.cpu().numpy()[:len(limits)]
        assert totals[0] == pytest.approx(mean * h * w, rel=1e-6)
        for t, wt, lim in zip(totals, weights, limits):
            assert (wt == 0) == (t <= lim), (t, lim, wt)
        assert weights.tolist() == [1.0, 1.0, 0.0, 0.0]
    finally:
        ctx.close()
        dec_only.close()
