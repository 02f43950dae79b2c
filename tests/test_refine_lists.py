"""Keep-the-better re-encodes of device block lists: astcenc_b200_refine_device_block_lists (astc_dev_refine.cuh:
refine_decide_block / refine_commit_block; astc_refine_decide_kernel<M> and astc_refine_commit_kernel).

CPU: the decisions and commits of the host simulation (tests/hostsim/hostsim_refine.cpp, one lane and 32 lanes) against a numpy
statement of the rule, with candidates from oracle encodes and decodes, chunk by chunk; every byte the rule does not write keeps
its poison. Candidate values are bit for bit the whole-map simulation's on an image that holds the candidate's decode.
GPU: the call against the three-call round (compress_device_block_lists, list decode, list map) on a copy; guard bytes; the
invariants of a -fast -> -medium -> -thorough ladder; the launch counts and the error order."""
import ctypes as C

import numpy as np
import pytest

from astc_ref import *  # noqa: F401,F403
from hostsim_build import host_sim
from test_block_list_decode import KINDS, BlockList, block_texels, make_list
from test_block_metrics import ALPHA, LOG2, METRIC_IDS, SQUARED, numpy_metric_map, sim_metric_map, soft_alpha
from test_block_metrics import sim as metric_sim
from test_metrics_device import DT, nblocks
import astc_images as I

METRICS = (SQUARED, ALPHA, LOG2)
S = FLG_SELF_DECOMPRESS_ONLY
POISON = 0xA5

_SIMS = {}


def sim(lanes32=False):
    """tests/hostsim/hostsim_refine.cpp compiled for the host (one simulated lane, or 32 lanes on 32 threads)."""
    if lanes32 in _SIMS:
        return _SIMS[lanes32]
    lib = host_sim("hostsim_refine", lanes32)
    common = [C.c_void_p, C.c_void_p, C.c_uint, C.c_int, C.c_int, C.c_uint, C.c_uint, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
              C.c_void_p, C.c_void_p, C.c_int, C.c_size_t, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.hostsim_refine_decide.argtypes = common + [C.c_int]
    lib.hostsim_refine_commit.argtypes = common + [C.c_void_p]
    _SIMS[lanes32] = lib
    return lib


def vol(a):
    return a if a.ndim == 4 else a[None]


def candidates(oracle, img, fp, profile, preset, out_type):
    """An oracle encode of (D, H, W, 4) `img` at `preset` and its oracle decode to out_type: ((blocks, 16) uint8, (D, H, W, 4)).
    A 2D footprint takes the slices one by one (a texture array's block order); a 3D one the volume."""
    D, H, W = img.shape[:3]
    if fp[2] > 1:
        pay = oracle.compress_volume(img, profile, fp[0], fp[1], fp[2], preset)
        dec = oracle.decompress_volume(pay, W, H, D, profile, fp[0], fp[1], fp[2], out_type=out_type)
    else:
        pays = [oracle.compress(img[z], profile, fp[0], fp[1], preset) for z in range(D)]
        pay = np.concatenate(pays)
        dec = np.stack([oracle.decompress(p, W, H, profile, fp[0], fp[1], out_type=out_type) for p in pays])
    return pay.reshape(-1, 16), dec


def footprint(shape, fp, b):
    """Image positions (z, y, x) and footprint positions (tz, ty, tx) of block b's texels that lie inside the image."""
    D, H, W = shape
    bx_n, by_n = -(-W // fp[0]), -(-H // fp[1])
    col, row, layer = b % bx_n, (b // bx_n) % by_n, b // (bx_n * by_n)
    out = []
    for tz in range(fp[2]):
        for ty in range(fp[1]):
            for tx in range(fp[0]):
                z, y, x = layer * fp[2] + tz, row * fp[1] + ty, col * fp[0] + tx
                if z < D and y < H and x < W:
                    out.append(((z, y, x), (tz, ty, tx)))
    return out


def slots(lists, shapes, fp):
    """The call's staging blocks in order: (entry, block or None) per slot; entries of capacity 0 own none."""
    out = []
    for j, (l, s) in enumerate(zip(lists, shapes)):
        for k in range(l.capacity):
            b = int(l.idx[k])
            out.append((j, b if k < min(l.count, l.capacity) and b < nblocks(s, fp) else None))
    return out


def old_map(rng, want):
    """A map around the candidate values `want`: below (no commit), equal (a tie: no commit), above (commit), NaN, +inf, 0."""
    m = want.copy()
    kind = rng.integers(0, 6, len(want))
    m[kind == 0] = want[kind == 0] * np.float32(0.5)
    m[kind == 2] = want[kind == 2] * np.float32(2.0) + np.float32(1e-3)
    m[kind == 3] = np.nan
    m[kind == 4] = np.inf
    m[kind == 5] = 0.0
    return m


def sim_refine(lib, imgs, pays, decs, fp, components, metric, lists, maps, chunk, with_decoded, rng):
    """The simulated call, chunk by chunk: the candidates and their decode row staged as the pipeline stages them (texels of the
    footprint outside the image and whole invalid slots hold garbage), then the decisions and the commits. Returns the payloads,
    decodes (None without) and maps it leaves, and each slot's candidate value (NaN where the slot is invalid)."""
    n = len(imgs)
    shapes = [vol(a).shape[:3] for a in imgs]
    dims = np.array([[s[2], s[1], s[0]] for s in shapes], np.uint32).reshape(-1)
    out_pay = [np.full(nblocks(s, fp) * 16, POISON, np.uint8) for s in shapes]
    out_dec = [np.full(d.nbytes, POISON, np.uint8).view(d.dtype).reshape(d.shape) if with_decoded else None for d in decs]
    out_map = [m.copy() for m in maps]
    data = (C.c_void_p * n)(*[vol(a).ctypes.data for a in imgs])
    pp = (C.c_void_p * n)(*[p.ctypes.data for p in out_pay])
    dp = (C.c_void_p * n)(*[d.ctypes.data if d is not None else None for d in out_dec])
    mp = (C.c_void_p * n)(*[m.ctypes.data for m in out_map])
    padded = [l.padded() for l in lists]
    ip = (C.c_void_p * n)(*[p.ctypes.data for p in padded])
    counts = np.array([l.count for l in lists], np.uint32)
    caps = np.array([l.capacity for l in lists], np.uint32)
    dt = DT[vol(imgs[0]).dtype]
    ot = DT[decs[0].dtype]
    call = slots(lists, shapes, fp)
    values = np.full(len(call), np.nan, np.float32)
    for base in range(0, len(call), chunk):
        m = min(chunk, len(call) - base)
        row = rng.integers(0, 256, (fp[2], fp[1], m * fp[0], 4 * decs[0].itemsize), dtype=np.uint8).view(decs[0].dtype)
        staged = rng.integers(0, 256, (m, 16), dtype=np.uint8)
        for i in range(m):
            j, b = call[base + i]
            if b is None:
                continue
            staged[i] = pays[j][b]
            for (z, y, x), (tz, ty, tx) in footprint(shapes[j], fp, b):
                row[tz, ty, i * fp[0] + tx] = decs[j][z, y, x]
        v = np.full(m, np.nan, np.float32)
        keep = np.full(m, 0xEE, np.uint8)
        args = (data, dims.ctypes.data, n, dt, ot, fp[0], fp[1], fp[2], pp, dp, mp, ip, counts.ctypes.data, caps.ctypes.data, components, base, m,
                row.ctypes.data, v.ctypes.data, keep.ctypes.data)
        lib.hostsim_refine_decide(*args, metric)
        assert set(keep.tolist()) <= {0, 1}
        lib.hostsim_refine_commit(*args, staged.ctypes.data)
        values[base:base + m] = np.where([call[base + i][1] is not None for i in range(m)], v, np.nan)
    return out_pay, out_dec, out_map, values


def numpy_refine(imgs, pays, decs, fp, components, metric, lists, maps, chunk, with_decoded):
    """The rule: per chunk, a valid slot's block is committed iff its candidate value is below the map as it stood before the
    chunk; a committed block gets the candidate's bytes, its decode's texels inside the image and the value. Nothing else
    changes. Returns what the call leaves, as sim_refine does, and the candidate value of each block."""
    shapes = [vol(a).shape[:3] for a in imgs]
    want = [numpy_metric_map(vol(a), d, fp, components, metric) for a, d in zip(imgs, decs)]
    out_pay = [np.full(nblocks(s, fp) * 16, POISON, np.uint8) for s in shapes]
    out_dec = [np.full(d.nbytes, POISON, np.uint8).view(d.dtype).reshape(d.shape) if with_decoded else None for d in decs]
    out_map = [m.copy() for m in maps]
    call = slots(lists, shapes, fp)
    for base in range(0, len(call), chunk):
        before = [m.copy() for m in out_map]
        for j, b in call[base:base + chunk]:
            if b is None or not want[j][b] < before[j][b]:
                continue
            out_pay[j][16 * b:16 * b + 16] = pays[j][b]
            out_map[j][b] = want[j][b]
            if with_decoded:
                mask = block_texels(shapes[j], fp, np.array([b]))
                out_dec[j][mask] = decs[j][mask]
    return out_pay, out_dec, out_map, want


def check_case(lanes32, imgs, pays, decs, fp, components, metric, lists, chunk, rng, with_decoded=True):
    lib = sim(lanes32)
    shapes = [vol(a).shape[:3] for a in imgs]
    want_values = [numpy_metric_map(vol(a), d, fp, components, metric) for a, d in zip(imgs, decs)]
    maps = [old_map(rng, w) for w in want_values]
    got = sim_refine(lib, imgs, pays, decs, fp, components, metric, lists, maps, chunk, with_decoded, rng)
    want = numpy_refine(imgs, pays, decs, fp, components, metric, lists, maps, chunk, with_decoded)
    for j in range(len(imgs)):
        assert np.array_equal(got[0][j], want[0][j]), "payload of entry %d" % j
        if with_decoded:
            assert got[1][j].tobytes() == want[1][j].tobytes(), "decode of entry %d" % j
        assert got[2][j].view(np.uint32).tolist() == want[2][j].view(np.uint32).tolist(), "map of entry %d" % j
    # every valid slot's value is bit for bit the whole-map simulation's on the candidate's decode
    call = slots(lists, shapes, fp)
    for s, (j, b) in enumerate(call):
        if b is not None:
            assert got[3][s].view(np.uint32) == want_values[j][b].view(np.uint32), (s, j, b)
    committed = sum(int(np.sum(g.view(np.uint32) != m.view(np.uint32))) for g, m in zip(got[2], maps))
    return committed, sum(b is not None for _, b in call)


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
def ldr_set(rng):
    """Ragged 2D images, a texture array and soft alpha, in U8."""
    shapes = [(1, 37, 29), (3, 13, 17), (1, 1, 1), (1, 25, 31), (2, 8, 14)]
    imgs = []
    for k, (d, h, w) in enumerate(shapes):
        imgs.append(np.stack([soft_alpha(h, w, seed=10 * k + z) if k % 2 else I.photo_like(h, w, seed=10 * k + z) for z in range(d)]))
    return imgs


@pytest.mark.parametrize("metric", METRICS, ids=lambda m: METRIC_IDS[m])
@pytest.mark.parametrize("lanes32", [False, True], ids=["lanes1", "lanes32"])
def test_hostsim_refine_ldr_equals_the_rule(oracle, lanes32, metric):
    """U8 images at 6x6 (ragged edges, a texture array, soft alpha), -medium candidates decoded to U8, F16 and F32; every list kind
    (invalid slots, count > capacity, duplicates in a chunk, count 0, capacity 0); chunks of 7 slots and of the whole call."""
    rng = np.random.default_rng(100 + metric)
    fp = (6, 6, 1)
    imgs = ldr_set(rng)
    lists = [make_list(rng, nblocks(vol(a).shape[:3], fp), KINDS[k % len(KINDS)]) for k, a in enumerate(imgs)]
    total = 0
    for out_type, chunk in ((TYPE_U8, 7), (TYPE_F16, 1000), (TYPE_F32, 7)):
        if lanes32 and out_type != TYPE_U8:
            continue      # (the 32-lane simulation is slow: one decoded type)
        cands = [candidates(oracle, a, fp, PRF_LDR, PRE_MEDIUM, out_type) for a in imgs]
        committed, valid = check_case(lanes32, imgs, [c[0] for c in cands], [c[1] for c in cands], fp, 4, metric, lists, chunk, rng)
        total += committed
        assert valid > 10
    assert total > 0


@pytest.mark.parametrize("metric", METRICS, ids=lambda m: METRIC_IDS[m])
@pytest.mark.parametrize("lanes32", [False, True], ids=["lanes1", "lanes32"])
def test_hostsim_refine_hdr_equals_the_rule(oracle, lanes32, metric):
    """F16 HDR images at 6x6 (ragged, an array) with -fast HDR candidates decoded to F16; input_components 3; with and without a
    decode."""
    rng = np.random.default_rng(200 + metric)
    fp = (6, 6, 1)
    imgs = [np.stack([I.hdr_noise(h, w, seed=7 * k + z, dtype=np.float16) for z in range(d)]) for k, (d, h, w) in enumerate([(1, 31, 23), (2, 12, 19)])]
    lists = [make_list(rng, nblocks(vol(a).shape[:3], fp), kind) for a, kind in zip(imgs, ("mixed", "sorted"))]
    cands = [candidates(oracle, a, fp, PRF_HDR, PRE_FAST, TYPE_F16) for a in imgs]
    for with_decoded in (True, False):
        check_case(lanes32, imgs, [c[0] for c in cands], [c[1] for c in cands], fp, 3, metric, lists, 5, rng, with_decoded)


@pytest.mark.parametrize("metric", METRICS, ids=lambda m: METRIC_IDS[m])
def test_hostsim_refine_volume_equals_the_rule(oracle, metric):
    """A 4x4x4 footprint on ragged volumes in U8 (one lane and 32)."""
    rng = np.random.default_rng(300 + metric)
    fp = (4, 4, 4)
    imgs = [np.stack([I.photo_like(h, w, seed=5 * k + z) for z in range(d)]) for k, (d, h, w) in enumerate([(5, 7, 9), (8, 8, 4), (1, 1, 1)])]
    lists = [make_list(rng, nblocks(a.shape[:3], fp), kind) for a, kind in zip(imgs, ("mixed", "past", "sorted"))]
    cands = [candidates(oracle, a, fp, PRF_LDR, PRE_MEDIUM, TYPE_U8) for a in imgs]
    for lanes32 in (False, True):
        check_case(lanes32, imgs, [c[0] for c in cands], [c[1] for c in cands], fp, 4, metric, lists, 4, rng)


@pytest.mark.parametrize("lanes32", [False, True], ids=["lanes1", "lanes32"])
def test_hostsim_refine_nan_and_inf_texels(lanes32):
    """F32 originals and candidate decodes full of NaN, inf and out-of-range texels: the texels are clamped as the whole map clamps
    them, so the candidate value is the map's value (never NaN) and the rule holds; NaN map values never commit."""
    from test_metrics_device import random_pair
    rng = np.random.default_rng(17)
    fp = (6, 6, 1)
    shapes = [(1, 20, 27), (2, 9, 13)]
    imgs, decs, pays = [], [], []
    for s in shapes:
        a, b = random_pair(rng, s, TYPE_F32, TYPE_F32)
        imgs.append(a)
        decs.append(b)
        pays.append(rng.integers(0, 256, (nblocks(s, fp), 16), dtype=np.uint8))
    lists = [make_list(rng, nblocks(s, fp), "mixed") for s in shapes]
    for metric in METRICS:
        for d in decs:
            assert not np.all(np.isfinite(d))
        check_case(lanes32, imgs, pays, decs, fp, 4, metric, lists, 6, rng)
        assert not np.any(np.isnan(np.concatenate([numpy_metric_map(a, d, fp, 4, metric) for a, d in zip(imgs, decs)])))


def test_hostsim_candidate_values_equal_the_whole_map_simulation(oracle):
    """The 32-lane decide's values against hostsim_block_metric (the whole map of the simulation) on the candidates' decodes,
    every metric, U8 and F16 decodes."""
    rng = np.random.default_rng(400)
    fp = (6, 6, 1)
    img = soft_alpha(29, 41, seed=3)[None]
    lists = [BlockList(np.arange(nblocks(img.shape[:3], fp)), 1 << 20, nblocks(img.shape[:3], fp))]
    lib = sim(True)
    for out_type in (TYPE_U8, TYPE_F16):
        pay, dec = candidates(oracle, img, fp, PRF_LDR, PRE_THOROUGH, out_type)
        for metric in METRICS:
            maps = [np.full(len(pay), np.inf, np.float32)]
            _, _, got, values = sim_refine(lib, [img], [pay], [dec], fp, 4, metric, lists, maps, 1000, True, rng)
            want = sim_metric_map(metric_sim(True), img, dec, fp, 4, metric)
            assert values.view(np.uint32).tolist() == want.view(np.uint32).tolist()
            assert got[0].view(np.uint32).tolist() == want.view(np.uint32).tolist()      # (every value is below +inf)


# ---------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------
GUARD = 256
GUARD_BYTE = 0x5A


@pytest.fixture(scope="module")
def gpu(pkg):
    import torch
    assert torch.cuda.is_available(), "the GPU tests need a CUDA device"
    torch.cuda.set_device(0)
    return pkg


class Guarded:
    """`nbytes` device bytes inside GUARD guard bytes on each side."""

    def __init__(self, nbytes, fill=None):
        import torch
        self.n = nbytes
        self.buf = torch.full((nbytes + 2 * GUARD,), GUARD_BYTE, dtype=torch.uint8, device="cuda")
        if fill is not None:
            self.buf[GUARD:GUARD + nbytes].copy_(torch.from_numpy(np.ascontiguousarray(fill).reshape(-1).view(np.uint8)).cuda())
        self.ptr = self.buf.data_ptr() + GUARD

    def get(self):
        b = self.buf.cpu().numpy()
        assert np.all(b[:GUARD] == GUARD_BYTE) and np.all(b[GUARD + self.n:] == GUARD_BYTE), "a guard byte changed"
        return b[GUARD:GUARD + self.n].copy()


class State:
    """One entry of a refine test on the device: the image, its payload, decode and map (each inside guard bytes), its list."""

    def __init__(self, img, lst, fp, out_type):
        import torch
        self.img = vol(img)
        self.shape = self.img.shape[:3]
        self.blocks = nblocks(self.shape, fp)
        self.lst = lst
        self.out_type = out_type
        self.d_img = torch.from_numpy(self.img.reshape(-1).view(np.uint8)).cuda()
        self.pay = Guarded(self.blocks * 16)
        self.dec = Guarded(int(np.prod(self.shape)) * 4 * {TYPE_U8: 1, TYPE_F16: 2, TYPE_F32: 4}[out_type])
        self.map = Guarded(self.blocks * 4)
        self.d_idx = torch.from_numpy(lst.padded().view(np.int32)).cuda()
        self.d_cnt = torch.from_numpy(np.array([lst.count], np.uint32).view(np.int32)).cuda()

    def dims(self):
        return self.shape[2], self.shape[1], self.shape[0]

    def copy(self):
        import copy
        c = copy.copy(self)
        c.pay, c.dec, c.map = Guarded(self.pay.n, self.pay.get()), Guarded(self.dec.n, self.dec.get()), Guarded(self.map.n, self.map.get())
        return c

    def host(self):
        return self.pay.get(), self.dec.get(), self.map.get().view(np.float32)


def start(ctx, fast, states, data_type, out_type, metric, components, stream=0):
    """Every entry's -fast payload, this context's decode of it and the whole map of `metric`."""
    import torch
    fast.compress_device_images([(s.d_img.data_ptr(), *s.dims(), s.pay.ptr) for s in states], data_type, stream=stream)
    ctx.decompress_device_images([(s.pay.ptr, s.dec.ptr, *s.dims()) for s in states], out_type, stream=stream)
    met = torch.zeros(len(states) * 128, dtype=torch.uint8, device="cuda")
    ctx.compute_block_metric_device_images([(s.d_img.data_ptr(), s.dec.ptr, data_type, out_type, *s.dims(), met.data_ptr() + 128 * k, s.map.ptr)
                                            for k, s in enumerate(states)], metric, input_components=components, stream=stream)


def refine_table(states, with_decoded=True):
    return [(s.d_img.data_ptr(), *s.dims(), s.pay.ptr, s.dec.ptr if with_decoded else 0, s.map.ptr, s.d_idx.data_ptr(), s.d_cnt.data_ptr(), s.lst.capacity)
            for s in states]


def three_call_round(ctx, states, data_type, out_type, metric, components, stream=0):
    ctx.compress_device_block_lists([(s.d_img.data_ptr(), *s.dims(), s.pay.ptr, s.d_idx.data_ptr(), s.d_cnt.data_ptr(), s.lst.capacity) for s in states],
                                    data_type, stream=stream)
    ctx.decompress_device_block_lists([(s.pay.ptr, s.dec.ptr, *s.dims(), s.d_idx.data_ptr(), s.d_cnt.data_ptr(), s.lst.capacity) for s in states],
                                      out_type, stream=stream)
    ctx.compute_block_metric_device_block_lists([(s.d_img.data_ptr(), s.dec.ptr, data_type, out_type, *s.dims(), s.map.ptr, s.d_idx.data_ptr(),
                                                  s.d_cnt.data_ptr(), s.lst.capacity) for s in states], metric, input_components=components, stream=stream)


def equivalence(gpu, ctx, fast, imgs, lists, fp, data_type, out_type, metric, components, order=None, with_decoded=True, poke=True, chunks=1):
    """The call (A) against the three-call round on a copy (B): every listed block of A holds B's bytes, texels and value where
    B's value is below the old one, and the old ones otherwise; nothing else changes, guard bytes included. Returns how many
    listed blocks committed and how many were listed."""
    import torch
    states = [State(a, l, fp, out_type) for a, l in zip(imgs, lists)]
    start(ctx, fast, states, data_type, out_type, metric, components)
    torch.cuda.synchronize()
    rng = np.random.default_rng(5)
    for s in states:
        if poke and s.blocks > 3:
            m = s.map.get().view(np.float32)
            k = rng.choice(s.blocks, 3, replace=False)
            m[k] = [0.0, np.nan, np.inf]      # (never, never and always below)
            s.map = Guarded(s.map.n, m)
    old = [s.host() for s in states]
    b_states = [s.copy() for s in states]
    torch.cuda.synchronize()
    n0 = ctx.launch_count()
    three_call_round(ctx, b_states, data_type, out_type, metric, components)
    n1 = ctx.launch_count()
    order = list(range(len(states))) if order is None else order
    ctx.refine_device_block_lists(refine_table([states[j] for j in order], with_decoded), data_type, out_type, metric, input_components=components)
    n2 = ctx.launch_count()
    torch.cuda.synchronize()
    # the same launches as compress_device_block_lists, with one scatter replaced by three launches per chunk
    assert n2 - n1 == (n1 - n0 - 2) + 2 * chunks
    committed = listed_total = 0
    for s, b, (opay, odec, omap) in zip(states, b_states, old):
        pay, dec, mp = s.host()
        bpay, bdec, bmap = b.host()
        want_pay, want_dec, want_map = opay.copy(), odec.copy(), omap.copy()
        listed = np.unique(s.lst.listed(s.blocks))
        keep = listed[bmap[listed] < omap[listed]]
        for k in keep:
            want_pay[16 * k:16 * k + 16] = bpay[16 * k:16 * k + 16]
        want_map[keep] = bmap[keep]
        if with_decoded:
            mask = block_texels(s.shape, fp, keep).reshape(-1)
            tb = len(want_dec) // mask.size
            m8 = np.repeat(mask, tb)
            want_dec[m8] = bdec[m8]
        assert np.array_equal(pay, want_pay), "payload"
        assert np.array_equal(dec, want_dec), "decode"
        assert np.array_equal(mp.view(np.uint32), want_map.view(np.uint32)), "map"
        committed += len(keep)
        listed_total += len(listed)
    return committed, listed_total


def contexts(gpu, profile, preset, fp=(6, 6, 1), flags=0, **kw):
    return (gpu.Context(gpu.config_init(profile, fp[0], fp[1], preset, flags, block_z=fp[2], **kw)),
            gpu.Context(gpu.config_init(profile, fp[0], fp[1], PRE_FAST, flags, block_z=fp[2], **kw)))


@pytest.mark.gpu
@pytest.mark.parametrize("metric", METRICS, ids=lambda m: METRIC_IDS[m])
def test_equals_the_three_call_round(metric, gpu):
    """LDR U8 (ragged, every list kind), a texture array, soft alpha with 4 components, a decode to F16, a decode left NULL and an
    HDR F16 image on a SELF_DECOMPRESS_ONLY -thorough context: the call keeps exactly the three-call round's blocks whose value
    dropped below the old one."""
    rng = np.random.default_rng(10 + metric)
    fp = (6, 6, 1)
    ctx, fast = contexts(gpu, PRF_LDR, PRE_THOROUGH)
    try:
        imgs = [I.photo_like(97, 131, seed=1), soft_alpha(64, 64, seed=2), np.stack([I.photo_like(37, 29, seed=3 + z) for z in range(3)]),
                I.photo_like(120, 77, seed=4), soft_alpha(13, 50, seed=5)]
        lists = [make_list(rng, nblocks(vol(a).shape[:3], fp), KINDS[k % len(KINDS)]) for k, a in enumerate(imgs)]
        c, n = equivalence(gpu, ctx, fast, imgs, lists, fp, TYPE_U8, TYPE_U8, metric, 4)
        assert 0 < c <= n
        equivalence(gpu, ctx, fast, imgs[:2], lists[:2], fp, TYPE_U8, TYPE_F16, metric, 3)
        equivalence(gpu, ctx, fast, imgs, lists, fp, TYPE_U8, TYPE_U8, metric, 4, with_decoded=False)
    finally:
        ctx.close()
        fast.close()
    ctx, fast = contexts(gpu, PRF_HDR, PRE_THOROUGH, flags=S)
    try:
        imgs = [I.hdr_noise(90, 101, seed=6, dtype=np.float16), I.hdr_noise(31, 43, seed=7, dtype=np.float16)]
        lists = [make_list(rng, nblocks(vol(a).shape[:3], fp), kind) for a, kind in zip(imgs, ("sorted", "mixed"))]
        c, n = equivalence(gpu, ctx, fast, imgs, lists, fp, TYPE_F16, TYPE_F16, metric, 3)
        assert 0 < c <= n
    finally:
        ctx.close()
        fast.close()


@pytest.mark.gpu
def test_volume_shuffled_table_alpha_scale_and_chunks(gpu, monkeypatch):
    """A 4x4x4 volume; a shuffled 40-entry table; entries with a_scale_radius; staging rows of 37 blocks with duplicates that land
    in different chunks: each equals the three-call round."""
    rng = np.random.default_rng(77)
    ctx, fast = contexts(gpu, PRF_LDR, PRE_MEDIUM, fp=(4, 4, 4))
    try:
        v = [np.stack([I.photo_like(21, 19, seed=z) for z in range(9)]), np.stack([I.photo_like(8, 8, seed=20 + z) for z in range(4)])]
        lists = [make_list(rng, nblocks(a.shape[:3], (4, 4, 4)), kind) for a, kind in zip(v, ("mixed", "sorted"))]
        for metric in METRICS:
            equivalence(gpu, ctx, fast, v, lists, (4, 4, 4), TYPE_U8, TYPE_U8, metric, 4)
    finally:
        ctx.close()
        fast.close()
    fp = (6, 6, 1)
    ctx, fast = contexts(gpu, PRF_LDR, PRE_MEDIUM)
    try:
        imgs, lists = [], []
        for k in range(40):
            h, w = int(rng.integers(1, 70)), int(rng.integers(1, 70))
            imgs.append(soft_alpha(h, w, seed=100 + k) if k % 3 else I.photo_like(h, w, seed=100 + k))
            lists.append(make_list(rng, nblocks((1, h, w), fp), KINDS[k % len(KINDS)]))
        equivalence(gpu, ctx, fast, imgs, lists, fp, TYPE_U8, TYPE_U8, ALPHA, 4, order=rng.permutation(40).tolist())
    finally:
        ctx.close()
        fast.close()
    ctx, fast = contexts(gpu, PRF_LDR, PRE_MEDIUM, a_scale_radius=2)
    try:
        imgs = [soft_alpha(70, 90, seed=9), soft_alpha(33, 20, seed=10)]
        lists = [make_list(rng, nblocks((1,) + a.shape[:2], fp), kind) for a, kind in zip(imgs, ("sorted", "mixed"))]
        equivalence(gpu, ctx, fast, imgs, lists, fp, TYPE_U8, TYPE_U8, SQUARED, 4)
    finally:
        ctx.close()
        fast.close()
    monkeypatch.setenv("ASTCENC_B200_BATCH_BLOCKS", "37")
    ctx, fast = contexts(gpu, PRF_LDR, PRE_THOROUGH)
    monkeypatch.delenv("ASTCENC_B200_BATCH_BLOCKS")
    try:
        img = I.photo_like(120, 150, seed=11)
        n = nblocks((1, 120, 150), fp)
        idx = rng.integers(0, n, 100).astype(np.uint32)
        idx[60:100] = idx[0:40]      # (each repeat lies in a later chunk of 37)
        idx[5] = idx[4]              # (and one in the same chunk)
        lst = BlockList(idx, 100, 100)
        for metric in METRICS:
            c, _ = equivalence(gpu, ctx, fast, [img], [lst], fp, TYPE_U8, TYPE_U8, metric, 4, chunks=3)
            assert c > 0
    finally:
        ctx.close()
        fast.close()


@pytest.mark.gpu
@pytest.mark.parametrize("profile,metric", [(PRF_LDR, SQUARED), (PRF_LDR, ALPHA), (PRF_HDR, LOG2)], ids=["ldr-squared", "ldr-alpha", "hdr-log2"])
def test_ladder_invariants(profile, metric, gpu):
    """-fast, then -medium on the worst 10 % and -thorough on the worst 5 % with the new call, all on one stream: after every
    round the map never increased, equals a whole map of the decode, and the decode equals a whole decode of the payload."""
    import torch
    fp = (6, 6, 1)
    hdr = profile == PRF_HDR
    img = I.hdr_noise(150, 170, seed=8, dtype=np.float16) if hdr else soft_alpha(150, 170, seed=8)
    dt = DT[img.dtype]
    ot = TYPE_F16 if hdr else TYPE_U8
    comps = 3 if hdr else 4
    ctxs = [gpu.Context(gpu.config_init(profile, 6, 6, p)) for p in (PRE_FAST, PRE_MEDIUM, PRE_THOROUGH)]
    try:
        n = nblocks((1, 150, 170), fp)
        st = State(img, BlockList(np.zeros(n), 0, n), fp, ot)
        stream = torch.cuda.Stream()
        s = stream.cuda_stream
        torch.cuda.synchronize()
        start(ctxs[0], ctxs[0], [st], dt, ot, metric, comps, stream=s)
        stream.synchronize()
        prev = st.map.get().view(np.float32)
        kept = []
        for ctx, share in zip(ctxs[1:], (0.10, 0.05)):
            cap = int(n * share)
            ctx.select_blocks([(st.map.ptr, n, -np.inf, cap, st.d_idx.data_ptr(), st.d_cnt.data_ptr())], stream=s)
            ctx.refine_device_block_lists([(st.d_img.data_ptr(), 170, 150, 1, st.pay.ptr, st.dec.ptr, st.map.ptr, st.d_idx.data_ptr(), st.d_cnt.data_ptr(),
                                            cap)], dt, ot, metric, input_components=comps, stream=s)
            stream.synchronize()
            pay, dec, mp = st.host()
            assert np.all(mp <= prev), "a map value increased"
            kept.append(int(np.sum(mp < prev)))
            # whole decode of the payload and whole map of the decode
            whole_dec = Guarded(st.dec.n)
            whole_map = Guarded(st.map.n)
            met = torch.zeros(128, dtype=torch.uint8, device="cuda")
            ctx.decompress_device_images([(st.pay.ptr, whole_dec.ptr, 170, 150, 1)], ot, stream=s)
            ctx.compute_block_metric_device_images([(st.d_img.data_ptr(), st.dec.ptr, dt, ot, 170, 150, 1, met.data_ptr(), whole_map.ptr)], metric,
                                                   input_components=comps, stream=s)
            stream.synchronize()
            assert np.array_equal(whole_dec.get(), dec), "the decode differs from a whole decode of the payload"
            assert np.array_equal(whole_map.get(), mp.view(np.uint8)), "the map differs from a whole map of the decode"
            prev = mp
        assert kept[0] > 0
    finally:
        for c in ctxs:
            c.close()


@pytest.mark.gpu
def test_errors_and_launch_counts(gpu):
    """Every documented error in the documented order, with nothing launched and nothing written; an all-zero-capacity call
    launches nothing."""
    import torch
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, 0))
    dec_only = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, FLG_DECOMPRESS_ONLY))
    radius = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, 0, a_scale_radius=2))
    buf = torch.full((1 << 17,), 0x33, dtype=torch.uint8, device="cuda")
    base = buf.data_ptr()
    data, pay, dec, mp, idx, cnt = base, base + 32768, base + 40960, base + 81920, base + 90112, base + 98304
    buf[cnt - base:cnt - base + 4].copy_(torch.tensor([3], dtype=torch.int32, device="cuda").view(torch.uint8))
    buf[idx - base:idx - base + 16].copy_(torch.tensor([0, 1, 2, 3], dtype=torch.int32, device="cuda").view(torch.uint8))
    l = gpu.lib()
    P, SW = gpu.ERR_BAD_PARAM, gpu.ERR_BAD_SWIZZLE
    ok_swz = gpu.Swizzle(0, 1, 2, 3)

    def call(c=ctx, n=1, lists=True, swz=ok_swz, dswz=ok_swz, comps=4, metric=LOG2, data_type=TYPE_U8, decoded_type=TYPE_U8, **e):
        d = dict(data=data, dim_x=40, dim_y=40, dim_z=1, payload=pay, decoded=dec, block_error=mp, indices=idx, count=cnt, capacity=4)
        d.update(e)
        t = (gpu.DeviceRefineList * max(n, 1))(*[gpu.DeviceRefineList(*[C.c_void_p(d[k] or None) if k not in ("dim_x", "dim_y", "dim_z", "capacity")
                                                                         else d[k] for k, _ in gpu.DeviceRefineList._fields_])] * max(n, 1))
        before = buf.cpu()
        torch.cuda.synchronize()
        n0 = c.launch_count()
        r = l.astcenc_b200_refine_device_block_lists(c.handle, t if lists else None, n, data_type, C.byref(swz) if swz is not None else None, decoded_type,
                                                     C.byref(dswz) if dswz is not None else None, comps, metric, None)
        torch.cuda.synchronize()
        launched = c.launch_count() - n0
        if r != 0:
            assert launched == 0 and torch.equal(buf.cpu(), before), "an error launched or wrote something"
        return r, launched

    def compress_launches(c):
        t = (gpu.DeviceBlockList * 1)(gpu.DeviceBlockList(C.c_void_p(data), 40, 40, 1, C.c_void_p(pay), C.c_void_p(idx), C.c_void_p(cnt), 4))
        torch.cuda.synchronize()
        n0 = c.launch_count()
        assert l.astcenc_b200_compress_device_block_lists(c.handle, t, 1, TYPE_U8, C.byref(ok_swz), None) == 0
        torch.cuda.synchronize()
        return c.launch_count() - n0

    try:
        # the launches of compress_device_block_lists with the chunk's scatter replaced by a decode, the decisions and the commits
        launched = compress_launches(ctx) + 2
        assert call() == (0, launched)
        assert call(capacity=0, indices=0, count=0, block_error=0) == (0, 0)
        assert call(n=0, lists=False) == (0, 0)
        assert call(decoded=0) == (0, launched)
        assert call(c=radius) == (0, compress_launches(radius) + 2)      # (with the alpha-scale pre-pass)
        # each check, with every later one failing too
        bad_swz, bad_dswz = gpu.Swizzle(0, 1, 2, 7), gpu.Swizzle(0, 1, 2, 7)
        later = dict(comps=0, metric=3, lists=False, decoded_type=5, data=0, dim_x=0, data_type=9)
        assert call(c=dec_only, swz=None, **later) == (gpu.ERR_BAD_CONTEXT, 0)
        assert call(swz=None, dswz=None, **later) == (P, 0)
        assert call(swz=bad_swz, dswz=None, **later) == (SW, 0)
        assert call(dswz=None, **later) == (P, 0)
        assert call(dswz=bad_dswz, **later) == (SW, 0)
        assert call(dswz=gpu.Swizzle(0, 1, 2, 6)) == (0, launched)      # (Z is a decode selector)
        assert call(swz=gpu.Swizzle(0, 1, 2, 6)) == (SW, 0)
        for c in (0, 5):
            assert call(comps=c, metric=3, lists=False) == (P, 0)
        for m in (3, -1):
            assert call(metric=m, lists=False) == (P, 0)
        assert call(lists=False, decoded_type=5) == (P, 0)
        entry = [dict(data=0), dict(payload=0), dict(indices=0), dict(count=0), dict(block_error=0), dict(indices=idx + 2), dict(count=cnt + 1),
                 dict(block_error=mp + 2), dict(decoded=dec + 2), dict(decoded=dec + 4, decoded_type=TYPE_F16), dict(dim_x=0), dict(data_type=3),
                 dict(data=data + 4, data_type=TYPE_F16), dict(data=data + 4, data_type=TYPE_F32), dict(data=data + 8, data_type=TYPE_F32),
                 dict(data=data + 2)]
        for e in entry:
            assert call(**e) == (P, 0), e
        assert call(decoded=dec + 4) == (0, launched)      # (a U8 decode is aligned to 4 bytes)
        assert call(data=data + 4) == (0, launched)         # (and so is U8 data)
        # a bad data_type comes before the entries' checks, the alignment of data among them
        assert call(data_type=3, data=0) == (P, 0)
        assert call(data=data + 4, data_type=TYPE_F32, dim_x=0) == (P, 0)
        assert call(c=radius, dim_z=2, dim_x=0) == (P, 0)
        assert call(c=radius, dim_z=2) == (gpu.ERR_NOT_IMPLEMENTED, 0)
        assert call(c=radius, dim_z=2, dim_x=6 * 2 ** 16, dim_y=6 * 2 ** 16) == (gpu.ERR_NOT_IMPLEMENTED, 0)
        assert call(dim_x=6 * 2 ** 16, dim_y=6 * 2 ** 16) == (P, 0)
        with pytest.raises(gpu.AstcencError) as e:
            ctx.refine_device_block_lists([], TYPE_U8, TYPE_U8, 7)
        assert e.value.code == P
    finally:
        ctx.close()
        dec_only.close()
        radius.close()
