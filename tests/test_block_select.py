"""Block selection on the device (astcenc_b200_select_blocks, astc_dev_select.cuh) and block lists that live in device memory
(astcenc_b200_compress_device_block_lists, astc_dev_gather.cuh).

CPU: the selection compiled for the host (tests/hostsim/hostsim_select.cpp, one lane and 32 lanes) against the numpy rule of
the header, and the key order; the count-limited gather (tests/hostsim/hostsim_blocks.cpp) against the staging image of the
valid slots, with zeros for the invalid ones.
GPU: selection against numpy, alone and inside a shuffled table, twice, inside guard bytes, in a fixed number of launches;
device block lists against compress_device_blocks with the host list they stand for; the closed loop compress -> decode ->
measure -> select -> re-encode on one stream; launch counts; the error order of both entries."""
import ctypes as C

import numpy as np
import pytest

import astc_images as I
from astc_ref import *  # noqa: F401,F403
from hostsim_build import host_sim
from test_block_list import blocks_sim, sim_gather, sim_gather_list, staged_reference

S = FLG_SELF_DECOMPRESS_ONLY
_DT = {np.dtype(np.uint8): TYPE_U8, np.dtype(np.float16): TYPE_F16, np.dtype(np.float32): TYPE_F32}
SELECT_LAUNCHES = 7
_SIMS = {}


def select_sim(lanes32=False):
    """tests/hostsim/hostsim_select.cpp: the selection's launches in order."""
    if lanes32 in _SIMS:
        return _SIMS[lanes32]
    lib = host_sim("hostsim_select", lanes32)
    lib.hostsim_select_key.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
    lib.hostsim_select_blocks.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint]
    _SIMS[lanes32] = lib
    return lib


def numpy_select(m, t, capacity):
    """The header's rule: np.sort(np.argsort(-m, kind="stable")[:min(capacity, c)]) with m[~(m > t)] = -inf."""
    m = np.asarray(m, np.float32)
    cand = m > np.float32(t)
    mm = np.where(cand, m, np.float32(-np.inf))
    k = min(int(capacity), int(cand.sum()))
    return np.sort(np.argsort(-mm, kind="stable")[:k]).astype(np.uint32)


def sim_select(lib, cases):
    """One simulated call over cases [(map, threshold, capacity)] -> [(indices written, count)]; index slots past the count
    keep their poison."""
    maps = [np.ascontiguousarray(m, np.float32) for m, _, _ in cases]
    outs = [np.full(max(1, c), 0xA5A5A5A5, np.uint32) for _, _, c in cases]
    n = len(cases)
    mp = (C.c_void_p * n)(*[m.ctypes.data for m in maps])
    bc = np.array([len(m) for m in maps], np.uint32)
    th = np.array([t for _, t, _ in cases], np.float32)
    cap = np.array([c for _, _, c in cases], np.uint32)
    op = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
    counts = np.full(n, 0xFFFFFFFF, np.uint32)
    lib.hostsim_select_blocks(mp, bc.ctypes.data, th.ctypes.data, cap.ctypes.data, op, counts.ctypes.data, n)
    res = []
    for o, k, (_, _, c) in zip(outs, counts.tolist(), cases):
        assert np.all(o[k:] == 0xA5A5A5A5), "an index past the count was written"
        res.append((o[:k].copy(), k))
    return res


def select_maps(rng):
    """Maps with many ties (quantised), NaN, +-inf, negatives and -0.0; all-equal maps; sizes 0, 1 and sizes that are not
    multiples of a tile (1024 values) or of a warp."""
    out = []
    for n in (0, 1, 2, 31, 33, 1023, 1024, 1025, 2500):
        q = np.round(rng.normal(size=n) * 3).astype(np.float32) / 4      # (many ties, negatives and zeros)
        sp = rng.random(n)
        q[sp < 0.03] = np.nan
        q[(sp >= 0.03) & (sp < 0.05)] = np.inf
        q[(sp >= 0.05) & (sp < 0.07)] = -np.inf
        q[(sp >= 0.07) & (sp < 0.12)] = -0.0
        out.append(q)
        out.append(rng.random(n).astype(np.float32) * 1e-3)            # (distinct values, error-map-like)
    out.append(np.full(1500, 0.25, np.float32))
    out.append(np.full(77, -0.0, np.float32))
    out.append(np.zeros(40, np.float32))
    out.append(np.full(65, np.nan, np.float32))
    return out


def select_cases(rng):
    cases = []
    for m in select_maps(rng):
        finite = m[np.isfinite(m)]
        ts = [-np.inf, 0.0, np.inf]                                      # (all but NaN and -inf; the positives; none)
        if finite.size:
            ts.append(float(np.quantile(finite, 0.6)))                   # (some)
            ts.append(float(finite.min()) - 1.0)                         # (every finite value)
        for t in ts:
            c = int(np.sum(m > np.float32(t)))
            for cap in sorted({0, 1, max(1, c // 3), c, c + 5, 4096}):
                cases.append((m, t, cap))
    return cases


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
def test_select_key_is_order_preserving():
    lib = select_sim()
    rng = np.random.default_rng(1)
    v = np.concatenate([rng.normal(size=20000).astype(np.float32) * np.float32(10) ** rng.integers(-40, 38, 20000).astype(np.float32),
                        np.array([0.0, -0.0, np.inf, -np.inf, 1e-45, -1e-45, 3.4e38, -3.4e38], np.float32)]).astype(np.float32)
    v = v[~np.isnan(v)]
    keys = np.empty(len(v), np.uint32)
    lib.hostsim_select_key(v.ctypes.data, len(v), keys.ctypes.data)
    order = np.argsort(v, kind="stable")
    assert np.all(np.diff(keys[order].astype(np.int64)) >= 0)
    z = np.array([0.0, -0.0], np.float32)
    kz = np.empty(2, np.uint32)
    lib.hostsim_select_key(z.ctypes.data, 2, kz.ctypes.data)
    assert kz[0] == kz[1]      # (-0.0 counts as 0.0)
    # strictly increasing on distinct values
    u = np.unique(v)
    ku = np.empty(len(u), np.uint32)
    lib.hostsim_select_key(u.ctypes.data, len(u), ku.ctypes.data)
    assert np.all(np.diff(ku.astype(np.int64)) > 0)


@pytest.mark.parametrize("lanes32", [False, True], ids=["1lane", "32lanes"])
def test_hostsim_selection_equals_numpy(lanes32):
    rng = np.random.default_rng(2)
    cases = select_cases(rng)
    if lanes32:
        cases = [c for c in cases if len(c[0]) <= 1100][::3]      # (32 threads per simulated warp: a subset)
    lib = select_sim(lanes32)
    for (m, t, cap), (got, k) in zip(cases, sim_select(lib, cases)):
        want = numpy_select(m, t, cap)
        assert k == len(want), (len(m), t, cap)
        assert np.array_equal(got, want), (len(m), t, cap)


GATHER_LISTS = [
    ("u8_2d_6x6", np.uint8, (1, 23, 37), (6, 6, 1), False),
    ("f16_array_5x4", np.float16, (3, 31, 29), (5, 4, 1), False),
    ("u8_2d_6x6_avg", np.uint8, (1, 40, 50), (6, 6, 1), True),
    ("f32_volume_4x4x4", np.float32, (7, 9, 11), (4, 4, 4), False),
]


@pytest.mark.parametrize("lanes32", [False, True], ids=["1lane", "32lanes"])
@pytest.mark.parametrize("case", GATHER_LISTS, ids=[c[0] for c in GATHER_LISTS])
def test_count_limited_gather_stages_valid_slots_and_zeros(case, lanes32):
    """The first min(count, capacity) slots with an index inside the image stage what staged_reference gives; every other
    slot (past the count, whatever its poison, or out of range) stages zero texels and zero averages."""
    _, dtype, shape, fp, with_avg = case
    lib = blocks_sim(lanes32)
    rng = np.random.default_rng(3)
    vol = np.ascontiguousarray(rng.integers(1, 255, size=shape + (4,)).astype(dtype) if dtype == np.uint8 else
                               (rng.random(shape + (4,)) + 0.5).astype(dtype))
    nbx, nby, nl = -(-shape[2] // fp[0]), -(-shape[1] // fp[1]), -(-shape[0] // fp[2])
    total = nbx * nby * nl
    avg = (rng.random((shape[1], shape[2])).astype(np.float32) + 0.5) if with_avg else None
    for count, capacity in ((5, 12), (12, 12), (20, 12), (0, 6)):
        idx = rng.integers(0, total, size=capacity).astype(np.uint32)
        if capacity > 3:
            idx[1] = total + 7                      # (out of range: skipped)
            idx[2] = idx[0]                         # (a duplicate)
        idx[min(count, capacity):] = rng.integers(0, 2 ** 32, size=capacity - min(count, capacity), dtype=np.uint64).astype(np.uint32)
        valid = np.array([s < min(count, capacity) and idx[s] < total for s in range(capacity)], bool)
        staged, savg = sim_gather_list(lib, vol, fp, idx, count, avg, fill=77)
        ref_idx = np.where(valid, idx, 0).astype(np.uint32)
        want = staged_reference(vol, fp, ref_idx)
        want_avg = sim_gather(lib, vol, fp, ref_idx, avg)[1] if with_avg else None
        for s in range(capacity):
            sl = slice(s * fp[0], (s + 1) * fp[0])
            if valid[s]:
                assert np.array_equal(staged[:, :, sl], want[:, :, sl]), (count, capacity, s)
                if with_avg:
                    assert np.array_equal(savg[:, sl], want_avg[:, sl]), (count, capacity, s)
            else:
                assert np.all(staged[:, :, sl] == 0), (count, capacity, s)
                if with_avg:
                    assert np.all(savg[:, sl] == 0.0), (count, capacity, s)


# ---------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------
GUARD = 64
POISON = 0xA5


@pytest.fixture(scope="module")
def gpu(pkg):
    import torch
    assert torch.cuda.is_available(), "these tests need a CUDA device"
    torch.cuda.set_device(0)
    return pkg


def device_select(ctx, cases, order=None, stream=None):
    """One select_blocks call over cases [(map, threshold, capacity)] in `order`, every output inside guard bytes of one buffer.
    Returns [(indices, count)] in the cases' order; checks the guards, the poison past each count and the launch count."""
    import torch
    dev = torch.device("cuda", 0)
    order = list(range(len(cases))) if order is None else order
    maps = [torch.from_numpy(np.ascontiguousarray(m, np.float32)).to(dev) if len(m) else None for m, _, _ in cases]
    offs, pos = [], GUARD
    for _, _, cap in cases:
        i = pos
        pos += 4 * cap + GUARD
        k = pos
        pos += 4 + GUARD
        offs.append((i, k))
    out = torch.full((pos,), POISON, dtype=torch.uint8, device=dev)
    base = out.data_ptr()
    entries = [(maps[j].data_ptr() if maps[j] is not None else 0, len(cases[j][0]), cases[j][1], cases[j][2], base + offs[j][0], base + offs[j][1])
               for j in order]
    st = stream or torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    n0 = ctx.launch_count()
    ctx.select_blocks(entries, stream=st.cuda_stream)
    assert ctx.launch_count() == n0 + (SELECT_LAUNCHES if cases else 0)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    mask = np.ones(pos, bool)
    res = []
    for (i, k), (_, _, cap) in zip(offs, cases):
        cnt = int(got[k:k + 4].view(np.uint32)[0])
        assert cnt <= cap
        res.append((got[i:i + 4 * cnt].view(np.uint32).copy(), cnt))
        mask[i:i + 4 * cnt] = False
        mask[k:k + 4] = False
    assert np.all(got[mask] == POISON), "a guard byte or an index past a count changed"
    return res


@pytest.mark.gpu
def test_select_blocks_equals_numpy(gpu):
    rng = np.random.default_rng(4)
    cases = select_cases(rng)
    big = rng.random(466489).astype(np.float32)
    big[rng.random(466489) < 0.01] = 0.5                # (ties)
    cases += [(big, -np.inf, 4664), (big, 0.999, 10 ** 6), (big, 0.5, 100), (big, -np.inf, 466489)]
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, gpu.FLG_DECOMPRESS_ONLY))
    try:
        for (m, t, cap), (got, k) in zip(cases, device_select(ctx, cases)):
            want = numpy_select(m, t, cap)
            assert k == len(want) and np.array_equal(got, want), (len(m), t, cap)
    finally:
        ctx.close()


@pytest.mark.gpu
def test_entries_alone_equal_the_same_entries_in_a_shuffled_40_entry_table(gpu):
    rng = np.random.default_rng(5)
    cases = select_cases(rng)
    pick = rng.choice(len(cases), size=38, replace=False).tolist()
    cases = [cases[p] for p in pick] + [(rng.random(70000).astype(np.float32), -np.inf, 700), (np.zeros(0, np.float32), -np.inf, 3)]
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 4, 4, PRE_FAST, S))
    try:
        alone = [device_select(ctx, [c])[0] for c in cases]
        order = rng.permutation(len(cases)).tolist()
        table = device_select(ctx, cases, order=order)
        again = device_select(ctx, cases, order=order)
        for j, c in enumerate(cases):
            assert alone[j][1] == table[j][1] == again[j][1]
            assert alone[j][0].tobytes() == table[j][0].tobytes() == again[j][0].tobytes(), j
            assert np.array_equal(table[j][0], numpy_select(*c)), j
    finally:
        ctx.close()


# ---- device block lists ----
def nblocks(shape, fp):
    d, h, w = shape[:3]
    return -(-w // fp[0]) * -(-h // fp[1]) * -(-d // fp[2])


class ListEntry:
    """One entry of a block-list call: an image ((D, H, W, 4)), the device list's contents (indices, garbage past the count
    included), its count and capacity."""

    def __init__(self, vol, fp, idx, count, capacity):
        self.vol = np.ascontiguousarray(vol if vol.ndim == 4 else vol[None])
        self.blocks = nblocks(self.vol.shape, fp)
        self.idx = np.asarray(idx, np.uint32)
        self.count = count
        self.capacity = capacity

    def host_list(self):
        """The host list the device list stands for."""
        s = self.idx[:min(self.count, self.capacity)]
        return s[s < self.blocks]


def sentinel(n, seed):
    return np.random.default_rng(seed).integers(0, 256, size=n, dtype=np.uint8)


def run_lists(ctx, entries, stream=None, swizzle=(0, 1, 2, 3)):
    """compress_device_block_lists over `entries` against compress_device_blocks with each entry's host list, both on
    sentinel payloads; returns the launches of the list call."""
    import torch
    dev = torch.device("cuda", 0)
    d_img = [torch.from_numpy(e.vol.reshape(-1)).to(dev) for e in entries]
    pays = [sentinel(e.blocks * 16, 100 + k) for k, e in enumerate(entries)]
    d_pay = [torch.from_numpy(p.copy()).to(dev) for p in pays]
    d_want = [torch.from_numpy(p.copy()).to(dev) for p in pays]
    d_idx = [torch.from_numpy(np.concatenate([e.idx, np.array([0], np.uint32)]).view(np.int32)).to(dev) for e in entries]
    d_cnt = torch.from_numpy(np.array([e.count for e in entries] + [0], np.uint32).view(np.int32)).to(dev)
    dt = _DT[entries[0].vol.dtype]
    st = stream or torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    n0 = ctx.launch_count()
    ctx.compress_device_block_lists([(im.data_ptr(), e.vol.shape[2], e.vol.shape[1], e.vol.shape[0], p.data_ptr(), ix.data_ptr(), d_cnt.data_ptr() + 4 * k,
                                      e.capacity) for k, (e, im, p, ix) in enumerate(zip(entries, d_img, d_pay, d_idx))], dt, swizzle=swizzle,
                                    stream=st.cuda_stream)
    launches = ctx.launch_count() - n0
    torch.cuda.synchronize()
    for e, im, w in zip(entries, d_img, d_want):
        ctx.compress_device_blocks(im.data_ptr(), dt, e.vol.shape[2], e.vol.shape[1], e.vol.shape[0], e.host_list(), w.data_ptr(), swizzle=swizzle)
    torch.cuda.synchronize()
    for k, (e, p, w, s) in enumerate(zip(entries, d_pay, d_want, pays)):
        got, want = p.cpu().numpy(), w.cpu().numpy()
        assert np.array_equal(got, want), "entry %d differs from compress_device_blocks" % k
        keep = np.ones(e.blocks, bool)
        keep[e.host_list()] = False
        assert np.array_equal(got.reshape(-1, 16)[keep], s.reshape(-1, 16)[keep]), "entry %d: an unlisted block changed" % k
    return launches


def garbage_list(rng, total, capacity, count, dups=0):
    idx = rng.integers(0, total, size=capacity).astype(np.uint32)
    if dups and capacity > dups:
        idx[1:1 + dups] = idx[0]
    c = min(count, capacity)
    idx[c:] = rng.integers(0, 2 ** 32, size=capacity - c, dtype=np.uint64).astype(np.uint32)      # (garbage past the count)
    return idx


def vol_of(h, w, d, seed, dtype=np.uint8):
    img = np.ascontiguousarray(I.photo_like(h * d, w, seed=seed).reshape(d, h, w, 4))
    return img if dtype == np.uint8 else np.ascontiguousarray((img.astype(np.float32) / 255.0).astype(dtype))


@pytest.mark.gpu
def test_device_lists_equal_host_lists_on_a_mixed_table(gpu):
    """2D images and a texture array in one call: garbage past the count, duplicates, count > capacity, count 0, capacity 0,
    an index out of range."""
    rng = np.random.default_rng(6)
    fp = (6, 6, 1)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_MEDIUM, S))
    try:
        vols = [vol_of(90, 130, 1, 1), vol_of(37, 41, 1, 2), vol_of(25, 31, 3, 3), vol_of(64, 64, 1, 4), vol_of(13, 7, 1, 5), vol_of(50, 50, 1, 6)]
        tot = [nblocks(v.shape, fp) for v in vols]
        entries = [ListEntry(vols[0], fp, garbage_list(rng, tot[0], 40, 25, dups=3), 25, 40),
                   ListEntry(vols[1], fp, garbage_list(rng, tot[1], 10, 99), 99, 10),          # (count > capacity)
                   ListEntry(vols[2], fp, garbage_list(rng, tot[2], 30, 30), 30, 30),
                   ListEntry(vols[3], fp, garbage_list(rng, tot[3], 16, 0), 0, 16),            # (count 0)
                   ListEntry(vols[4], fp, garbage_list(rng, tot[4], 0, 0), 5, 0),              # (capacity 0)
                   ListEntry(vols[5], fp, np.array([3, tot[5], tot[5] + 100, 7, 3], np.uint32), 5, 5)]      # (out of range)
        run_lists(ctx, entries)
        run_lists(ctx, entries[:1])                                                              # (a one-entry call)
        f16 = [ListEntry(vol_of(40, 33, 1, 7, np.float16), fp, garbage_list(rng, 42, 20, 12), 12, 20),
               ListEntry(vol_of(20, 20, 2, 8, np.float16), fp, garbage_list(rng, 32, 8, 8), 8, 8)]
        run_lists(ctx, f16, swizzle=(2, 1, 0, 3))
    finally:
        ctx.close()


@pytest.mark.gpu
def test_device_lists_on_a_volume_of_a_3d_footprint(gpu):
    rng = np.random.default_rng(7)
    fp = (4, 4, 4)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 4, 4, PRE_FAST, S, block_z=4))
    try:
        vols = [vol_of(19, 21, 9, 11), vol_of(8, 8, 4, 12)]
        entries = [ListEntry(vols[0], fp, garbage_list(rng, nblocks(vols[0].shape, fp), 30, 20, dups=2), 20, 30),
                   ListEntry(vols[1], fp, garbage_list(rng, nblocks(vols[1].shape, fp), 4, 9), 9, 4)]
        run_lists(ctx, entries)
    finally:
        ctx.close()


@pytest.mark.gpu
def test_device_lists_with_alpha_scale_and_small_chunks(gpu, monkeypatch):
    """a_scale_radius (a whole-image pre-pass per entry) and staging rows of 37 blocks (ASTCENC_B200_BATCH_BLOCKS, read when
    the context is made) that split entries and span several; the launches are those of compress_device_images over the same
    number of staging blocks: a gather, a pass and a scatter per chunk, and a pre-pass per 2D entry with a radius."""
    rng = np.random.default_rng(8)
    fp = (5, 4, 1)
    monkeypatch.setenv("ASTCENC_B200_BATCH_BLOCKS", "37")
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 5, 4, PRE_MEDIUM, S))
    ctx_r = gpu.Context(gpu.config_init(PRF_LDR, 5, 4, PRE_MEDIUM, S | FLG_USE_ALPHA_WEIGHT, a_scale_radius=3))
    monkeypatch.delenv("ASTCENC_B200_BATCH_BLOCKS")
    try:
        vols = [I.alpha_mask(90, 130, seed=12), I.alpha_mask(33, 47, seed=13), I.photo_like(20, 25, seed=14)]
        tot = [nblocks((1,) + v.shape[:2], fp) for v in vols]
        entries = [ListEntry(vols[0], fp, garbage_list(rng, tot[0], 120, 100, dups=4), 100, 120),      # 200 staging blocks in all
                   ListEntry(vols[1], fp, garbage_list(rng, tot[1], 50, 60), 60, 50),
                   ListEntry(vols[2], fp, garbage_list(rng, tot[2], 30, 3), 3, 30)]
        # 200 staging blocks in chunks of 37: 6 x (gather + a 37-launch pass of 5x4 -medium + scatter), as blocks_long_list
        assert run_lists(ctx, entries) == 234
        assert run_lists(ctx_r, entries) == 234 + 3
    finally:
        ctx.close()
        ctx_r.close()


@pytest.mark.gpu
def test_closed_loop_on_one_stream(gpu):
    """compress_device_images (-fast) -> decode -> maps -> select_blocks (the 1 % worst) -> compress_device_block_lists
    (-thorough), enqueued on one non-default stream with no synchronise until the end: each payload is the -fast payload with
    the selected blocks replaced by the -thorough compress_image bytes, and the lists are the host argsort lists, sorted."""
    import torch
    dev = torch.device("cuda", 0)
    fp = (6, 6, 1)
    fast = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, S))
    thorough = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_THOROUGH, S))
    try:
        imgs = [I.photo_like(h, w, seed=70 + k) for k, (h, w) in enumerate([(256, 256), (200, 311), (128, 96), (97, 143)])]
        nb = [nblocks((1,) + im.shape[:2], fp) for im in imgs]
        caps = [max(1, n // 100) for n in nb]
        dims = [(im.shape[1], im.shape[0]) for im in imgs]
        d_img = [torch.from_numpy(im.reshape(-1)).to(dev) for im in imgs]
        d_pay = [torch.zeros(n * 16, dtype=torch.uint8, device=dev) for n in nb]
        d_dec = [torch.zeros(im.size, dtype=torch.uint8, device=dev) for im in imgs]
        d_met = torch.zeros(len(imgs) * C.sizeof(gpu.ErrorMetrics), dtype=torch.uint8, device=dev)
        d_map = [torch.zeros(n, dtype=torch.float32, device=dev) for n in nb]
        d_idx = [torch.zeros(c, dtype=torch.int32, device=dev) for c in caps]
        d_cnt = torch.zeros(len(imgs), dtype=torch.int32, device=dev)
        st = torch.cuda.Stream(device=dev)
        torch.cuda.synchronize()
        s = st.cuda_stream
        fast.compress_device_images([(d.data_ptr(), w, h, 1, p.data_ptr()) for d, (w, h), p in zip(d_img, dims, d_pay)], TYPE_U8, stream=s)
        with torch.cuda.stream(st):
            d_fast = [p.clone() for p in d_pay]
        fast.decompress_device_images([(p.data_ptr(), o.data_ptr(), w, h, 1) for p, o, (w, h) in zip(d_pay, d_dec, dims)], TYPE_U8, stream=s)
        mb = C.sizeof(gpu.ErrorMetrics)
        fast.compute_error_metrics_device_images([(d.data_ptr(), o.data_ptr(), TYPE_U8, TYPE_U8, w, h, 1, d_met.data_ptr() + k * mb, m.data_ptr())
                                                  for k, (d, o, (w, h), m) in enumerate(zip(d_img, d_dec, dims, d_map))], input_components=4, stream=s)
        fast.select_blocks([(m.data_ptr(), n, -np.inf, c, ix.data_ptr(), d_cnt.data_ptr() + 4 * k)
                            for k, (m, n, c, ix) in enumerate(zip(d_map, nb, caps, d_idx))], stream=s)
        thorough.compress_device_block_lists([(d.data_ptr(), w, h, 1, p.data_ptr(), ix.data_ptr(), d_cnt.data_ptr() + 4 * k, c)
                                              for k, (d, (w, h), p, ix, c) in enumerate(zip(d_img, dims, d_pay, d_idx, caps))], TYPE_U8, stream=s)
        st.synchronize()
        counts = d_cnt.cpu().numpy()
        for k, im in enumerate(imgs):
            m = d_map[k].cpu().numpy()
            want_list = np.sort(np.argsort(-m, kind="stable")[:caps[k]]).astype(np.uint32)
            assert counts[k] == caps[k]
            got_list = d_idx[k].cpu().numpy().view(np.uint32)
            assert np.array_equal(got_list, want_list), k
            want = d_fast[k].cpu().numpy().reshape(-1, 16).copy()
            want[want_list] = thorough.compress_image(im).reshape(-1, 16)[want_list]
            assert np.array_equal(d_pay[k].cpu().numpy().reshape(-1, 16), want), k
    finally:
        fast.close()
        thorough.close()


# ---- errors ----
@pytest.mark.gpu
def test_select_errors_follow_the_documented_order_and_launch_nothing(gpu):
    import torch
    dev = torch.device("cuda", 0)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, gpu.FLG_DECOMPRESS_ONLY))
    buf = torch.full((4096,), POISON, dtype=torch.uint8, device=dev)
    base = buf.data_ptr()
    l = gpu.lib()

    def call(entries=True, count=None, **e):
        d = dict(map=base, block_count=64, threshold=-np.inf, capacity=8, indices=base + 1024, count=base + 2048)
        d.update(e)
        t = (gpu.BlockSelection * 2)(*[gpu.BlockSelection(C.c_void_p(d["map"] or None), d["block_count"], d["threshold"], d["capacity"],
                                                          C.c_void_p(d["indices"] or None), C.c_void_p(d["count"] or None))] * 2)
        torch.cuda.synchronize()
        before = buf.cpu().numpy()
        n0 = ctx.launch_count()
        r = l.astcenc_b200_select_blocks(ctx.handle, t if entries else None, 2 if count is None else count, None)
        torch.cuda.synchronize()
        if r != 0 or count == 0:
            assert ctx.launch_count() == n0
            assert np.array_equal(buf.cpu().numpy(), before)
        else:
            assert ctx.launch_count() == n0 + SELECT_LAUNCHES
        return r

    try:
        assert call() == 0
        assert call(count=0) == 0
        assert call(entries=False, count=0) == 0
        assert call(map=0, block_count=0) == 0
        assert call(indices=0, capacity=0) == 0
        singles = [dict(entries=False), dict(map=0), dict(indices=0), dict(map=base + 2), dict(indices=base + 1026), dict(threshold=float("nan"))]
        for s in singles:
            assert call(**s) == gpu.ERR_BAD_PARAM, s
        t = (gpu.BlockSelection * 1)(gpu.BlockSelection(C.c_void_p(base), 64, 0.0, 8, C.c_void_p(base + 1024), None))
        assert l.astcenc_b200_select_blocks(ctx.handle, t, 1, None) == gpu.ERR_BAD_PARAM       # (a NULL count)
        t = (gpu.BlockSelection * 1)(gpu.BlockSelection(C.c_void_p(base), 64, 0.0, 8, C.c_void_p(base + 1024), C.c_void_p(base + 2049)))
        assert l.astcenc_b200_select_blocks(ctx.handle, t, 1, None) == gpu.ERR_BAD_PARAM       # (a misaligned count)
        assert l.astcenc_b200_select_blocks(None, None, 0, None) == gpu.ERR_BAD_PARAM
        torch.cuda.synchronize()
    finally:
        ctx.close()


@pytest.mark.gpu
def test_block_list_errors_follow_the_documented_order_and_launch_nothing(gpu):
    import torch
    dev = torch.device("cuda", 0)
    vol = vol_of(40, 44, 1, 1)
    d_img = torch.from_numpy(vol.reshape(-1)).to(dev)
    d_arr = torch.from_numpy(vol_of(12, 13, 2, 2).reshape(-1)).to(dev)
    nbytes = 4096
    d_pay = torch.from_numpy(sentinel(nbytes, 1)).to(dev)
    d_idx = torch.zeros(64, dtype=torch.int32, device=dev)
    d_cnt = torch.full((4,), 3, dtype=torch.int32, device=dev)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, S))
    cfg_r = gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, S)
    cfg_r.a_scale_radius = 2
    ctx_r = gpu.Context(cfg_r)
    ctx_d = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, gpu.FLG_DECOMPRESS_ONLY))
    l = gpu.lib()
    E = dict(data=d_img.data_ptr(), dim_x=44, dim_y=40, dim_z=1, payload=d_pay.data_ptr(), indices=d_idx.data_ptr(), count=d_cnt.data_ptr(), capacity=8)

    def table(**edit):
        d = dict(E)
        d.update(edit)
        e2 = dict(E, data=d_arr.data_ptr(), dim_x=13, dim_y=12, dim_z=2, payload=d_pay.data_ptr() + 2048)
        return [(d["data"], d["dim_x"], d["dim_y"], d["dim_z"], d["payload"], d["indices"], d["count"], d["capacity"]),
                (e2["data"], e2["dim_x"], e2["dim_y"], e2["dim_z"], e2["payload"], e2["indices"], e2["count"], e2["capacity"])]

    def expect(c, code, lists=None, data_type=TYPE_U8, swizzle=(0, 1, 2, 3), raw=None):
        torch.cuda.synchronize()
        n0 = c.launch_count()
        call = raw or (lambda: c.compress_device_block_lists(table() if lists is None else lists, data_type, swizzle=swizzle))
        if code == 0:
            call()
        else:
            with pytest.raises(gpu.AstcencError) as e:
                call()
            assert e.value.code == code, (e.value.code, code)
        torch.cuda.synchronize()
        assert c.launch_count() == n0
        assert np.array_equal(d_pay.cpu().numpy(), sentinel(nbytes, 1))

    def _raise(err):
        if err:
            raise gpu.AstcencError(err, "call")

    sw = gpu.Swizzle(0, 1, 2, 3)
    P = gpu.ERR_BAD_PARAM
    try:
        expect(ctx_d, gpu.ERR_BAD_CONTEXT)
        expect(ctx_d, gpu.ERR_BAD_CONTEXT, swizzle=(0, 1, 2, 9))
        expect(ctx, P, raw=lambda: _raise(l.astcenc_b200_compress_device_block_lists(ctx.handle, None, 0, TYPE_U8, None, None)))
        expect(ctx, gpu.ERR_BAD_SWIZZLE, swizzle=(0, 1, 2, 9))
        expect(ctx, gpu.ERR_BAD_SWIZZLE, lists=table(data=0), swizzle=(0, 1, 2, 9))
        expect(ctx, P, raw=lambda: _raise(l.astcenc_b200_compress_device_block_lists(ctx.handle, None, 2, TYPE_U8, C.byref(sw), None)))
        for edit in (dict(data=0), dict(payload=0), dict(indices=0), dict(count=0), dict(indices=d_idx.data_ptr() + 2), dict(count=d_cnt.data_ptr() + 1),
                     dict(dim_x=0), dict(dim_y=0), dict(dim_z=0)):
            expect(ctx, P, lists=table(**edit))
            expect(ctx_r, P, lists=table(**{"dim_z": 2, **edit}))      # (before NOT_IMPLEMENTED)
        expect(ctx, P, data_type=3)
        expect(ctx_r, P, lists=table(dim_z=2), data_type=3)
        expect(ctx_r, gpu.ERR_NOT_IMPLEMENTED, lists=table(dim_z=2))
        expect(ctx_r, gpu.ERR_NOT_IMPLEMENTED, lists=table(dim_x=6 * 2 ** 16, dim_y=6 * 2 ** 16, dim_z=2))      # (before the block count)
        expect(ctx, P, lists=table(dim_x=6 * 2 ** 16, dim_y=6 * 2 ** 16))      # (2^32 blocks)
        # capacity 0: NULL lists are allowed, and nothing runs
        expect(ctx, 0, lists=[t[:5] + (0, 0, 0) for t in table()])
        expect(ctx, 0, lists=[])
        expect(ctx, 0, raw=lambda: _raise(l.astcenc_b200_compress_device_block_lists(ctx.handle, None, 0, TYPE_U8, C.byref(sw), None)))
    finally:
        ctx.close()
        ctx_r.close()
        ctx_d.close()
