"""Map totals and gated selection weights (astcenc_b200_total_block_maps, astc_dev_totals.cuh).

CPU: the totals call compiled for the host (tests/hostsim/hostsim_map_totals.cpp, one lane and 32 lanes) against a numpy
restatement of the fixed order, bit for bit, over sizes from 0 to several rounds of virtual CTAs, NaN, inf, -0.0 and denormal
values, both rules and every kind of limit; an entry's outputs alone and in other tables; the totals against np.sum.
GPU: the call against the 32-lane simulation inside guard bytes, twice and in a shuffled table of real -fast maps of a texture
set and a mip chain; NULL outputs; a decompress-only context; launch counts and the error order; weights read by
select_blocks_pooled on the same stream; the gated closed loop (total -> pooled select -> refine, three rounds enqueued up
front) on the mixed 64-texture set with PSNR targets, and on an F16 HDR set with log_rmse targets."""
import ctypes as C

import numpy as np
import pytest

import astc_images as I
from astc_ref import *  # noqa: F401,F403
from hostsim_build import host_sim
from test_select_pooled import numpy_pooled

ONE, INVERSE = 0, 1                   # enum astcenc_b200_weight_rule
RULES = (ONE, INVERSE)
TOTAL_LAUNCHES = 2
METRIC_THREADS, METRIC_MAX_CTAS, SLOTS = 256, 592, 32      # metric_ctas and TOTAL_SLOTS
S = FLG_SELF_DECOMPRESS_ONLY
POISON_F64 = np.array([0x5A5A5A5A5A5A5A5A], np.uint64).view(np.float64)[0]
POISON_F32 = np.array([0x5A5A5A5A], np.uint32).view(np.float32)[0]
_SIMS = {}


def sim(lanes32=False):
    """tests/hostsim/hostsim_map_totals.cpp compiled for the host (one simulated lane, or 32 lanes on 32 threads)."""
    if lanes32 in _SIMS:
        return _SIMS[lanes32]
    lib = host_sim("hostsim_map_totals", lanes32)
    lib.hostsim_map_totals.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_int]
    _SIMS[lanes32] = lib
    return lib


# ---------------------------------------------------------------------------------------------------------------------------
# The numpy restatement
# ---------------------------------------------------------------------------------------------------------------------------
def serial(a, axis=-1):
    """Left-to-right double sums from 0.0 along `axis` (np.cumsum adds in order)."""
    a = np.moveaxis(np.asarray(a, np.float64), axis, -1)
    z = np.zeros(a.shape[:-1] + (1,))
    return np.cumsum(np.concatenate([z, a], axis=-1), axis=-1)[..., -1]


def numpy_total(m):
    """The fixed order: ctas = min(ceil(n / 256), 592) virtual CTAs; CTA v takes the runs of 256 values v, v + ctas, ...; its
    slot s adds the values i % 32 == s of its runs in index order; the CTA adds its 32 slots in order, the total its CTAs."""
    m = np.asarray(m, np.float32)
    n = len(m)
    if n == 0:
        return 0.0
    with np.errstate(invalid="ignore"):
        return _numpy_total(m, n)


def _numpy_total(m, n):
    ctas = min(-(-n // METRIC_THREADS), METRIC_MAX_CTAS)
    rounds = -(-n // (METRIC_THREADS * ctas))
    pad = np.zeros(rounds * ctas * METRIC_THREADS, np.float64)      # (adding 0.0 to a sum that started at 0.0 changes no bit)
    pad[:n] = m
    x = pad.reshape(rounds, ctas, METRIC_THREADS // SLOTS, SLOTS)      # [round, v, q, s]: value (round * ctas + v) * 256 + 32 q + s
    slots = serial(x.transpose(1, 3, 0, 2).reshape(ctas, SLOTS, -1))
    return float(serial(serial(slots)))


def numpy_weight(total, limit, rule):
    if not (total > limit and total > 0):
        return np.float32(0.0)
    with np.errstate(over="ignore"):
        return np.float32(1.0) if rule == ONE else np.float32(1.0 / total)


def same(a, b):
    """Equal bits, any NaN equal to any NaN."""
    a, b = np.asarray(a), np.asarray(b)
    if np.isnan(a) or np.isnan(b):
        return bool(np.isnan(a) and np.isnan(b))
    return a.tobytes() == b.tobytes()


def sim_totals(lib, entries, rule):
    """One simulated call. entries: [(map, limit, has_total, has_weight)]. Returns [(total or None, weight or None)]."""
    n = len(entries)
    maps = [np.ascontiguousarray(m, np.float32) for m, _, _, _ in entries]
    tots = [np.full(1, POISON_F64) for _ in entries]
    wts = [np.full(1, POISON_F32) for _ in entries]
    mp = (C.c_void_p * max(1, n))(*[m.ctypes.data for m in maps])
    bc = np.array([len(m) for m in maps] or [0], np.uint32)
    lim = np.array([l for _, l, _, _ in entries] or [0.0], np.float64)
    tp = (C.c_void_p * max(1, n))(*[t.ctypes.data if e[2] else None for t, e in zip(tots, entries)])
    wp = (C.c_void_p * max(1, n))(*[w.ctypes.data if e[3] else None for w, e in zip(wts, entries)])
    assert lib.hostsim_map_totals(mp, bc.ctypes.data, lim.ctypes.data, tp, wp, n, rule) == 0
    res = []
    for t, w, e in zip(tots, wts, entries):
        assert e[2] or t.tobytes() == np.full(1, POISON_F64).tobytes()
        assert e[3] or w.tobytes() == np.full(1, POISON_F32).tobytes()
        res.append((float(t[0]) if e[2] else None, np.float32(w[0]) if e[3] else None))
    return res


def same_out(a, b):
    """Two (total or None, weight or None) pairs with the same bits."""
    return all((x is None and y is None) or (x is not None and y is not None and same(x, y)) for x, y in zip(a, b))


def check_entries(res, entries, rule, what):
    for j, ((t, w), (m, limit, ht, hw)) in enumerate(zip(res, entries)):
        want = numpy_total(m)
        if ht:
            assert same(t, want), (what, j, len(m), t, want)
        if hw:
            assert same(w, numpy_weight(want, limit, rule)), (what, j, len(m), limit, w, want)


def special_map(rng, n, kind):
    """A map of n values: non-negative floats at several scales, with NaN, +inf, -0.0, denormals or negatives mixed in."""
    m = (rng.random(n) * 10.0 ** rng.integers(-6, 4, size=n)).astype(np.float32)
    if n == 0 or kind == "plain":
        return m
    k = rng.integers(0, n, size=max(1, n // 50))
    if kind == "nan":
        m[k[:1]] = np.nan
    elif kind == "inf":
        m[k[:1]] = np.inf
    elif kind == "negzero":
        m[:] = -0.0
    elif kind == "denormal":
        m[k] = np.float32(1e-42) * rng.integers(1, 100, size=len(k)).astype(np.float32)
    elif kind == "tiny":
        m[:] = np.float32(1e-44)
    elif kind == "mixed_sign":
        m[k] = -m[k]
    return m


SIZES = [0, 1, 31, 32, 33, 255, 256, 257, 1000, 256 * 3 + 5, 256 * 592 - 1, 256 * 592, 256 * 592 + 1, 256 * 592 * 3 + 777]
KINDS = ("plain", "nan", "inf", "negzero", "denormal", "tiny", "mixed_sign")


def table_cases(rng, small=False):
    """[(map, limit, has_total, has_weight)]: every size with plain values (small: up to 40 virtual CTAs, for the slow 32-lane
    simulation), small sizes with every kind, and for each map the limits -inf, +inf, 0, the exact total (weight 0) and the next
    double below it."""
    maps = [special_map(rng, n, "plain") for n in SIZES if not small or n <= 256 * 40]
    maps += [special_map(rng, n, k) for n in (1, 33, 1000, 256 * 9 + 3) for k in KINDS[1:]]
    maps += [np.array([np.inf, 1.0, np.inf], np.float32), np.array([np.inf, -np.inf], np.float32), np.zeros(40, np.float32)]
    entries = []
    for i, m in enumerate(maps):
        t = numpy_total(m)
        lims = [-np.inf, np.inf, 0.0, t, np.nextafter(t, -np.inf)] if np.isfinite(t) else [-np.inf, np.inf, 0.0]
        for k, lim in enumerate(lims):
            entries.append((m, lim, (i + k) % 5 != 3, (i + k) % 7 != 5))
    return entries


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
def test_numpy_restatement_small_cases():
    """The restatement by hand: 40 values are one CTA whose slots 0-7 hold two values each."""
    m = np.arange(40, dtype=np.float32)
    slots = [float(m[s]) + (float(m[s + 32]) if s + 32 < 40 else 0.0) for s in range(32)]
    want = 0.0
    for v in slots:
        want += v
    assert numpy_total(m) == want
    assert numpy_total(np.zeros(0, np.float32)) == 0.0
    assert same(numpy_total(np.full(5, -0.0, np.float32)), 0.0)


@pytest.mark.parametrize("rule", RULES, ids=["one", "inverse"])
@pytest.mark.parametrize("lanes32", [False, True], ids=["1lane", "32lanes"])
def test_hostsim_totals_equal_numpy(lanes32, rule):
    rng = np.random.default_rng(40 + rule)
    entries = table_cases(rng, small=lanes32)
    check_entries(sim_totals(sim(lanes32), entries, rule), entries, rule, "table")


def test_hostsim_one_lane_equals_32_lanes():
    rng = np.random.default_rng(41)
    entries = table_cases(rng, small=True)
    for rule in RULES:
        a = sim_totals(sim(False), entries, rule)
        b = sim_totals(sim(True), entries, rule)
        for j, (x, y) in enumerate(zip(a, b)):
            assert same_out(x, y), j


def test_hostsim_weights_of_special_totals():
    """A total equal to the limit gives 0; limits of +-inf; a total of 0, a negative total, NaN and inf totals."""
    lib = sim()
    cases = [(np.array([2.0, 2.0], np.float32), 4.0, 0.0, 0.0), (np.array([2.0, 2.0], np.float32), 3.999, 1.0, 0.25),
             (np.array([2.0], np.float32), -np.inf, 1.0, 0.5), (np.array([2.0], np.float32), np.inf, 0.0, 0.0),
             (np.zeros(7, np.float32), -np.inf, 0.0, 0.0), (np.zeros(0, np.float32), -np.inf, 0.0, 0.0),
             (np.array([-1.0], np.float32), -np.inf, 0.0, 0.0), (np.array([np.nan], np.float32), -np.inf, 0.0, 0.0),
             (np.array([np.inf], np.float32), -np.inf, 1.0, 0.0), (np.array([np.inf], np.float32), np.inf, 0.0, 0.0),
             (np.array([3.0], np.float32), -np.inf, 1.0, np.float32(1.0 / 3.0))]
    for rule, col in ((ONE, 2), (INVERSE, 3)):
        res = sim_totals(lib, [(m, lim, True, True) for m, lim, _, _ in cases], rule)
        for (t, w), c in zip(res, cases):
            assert same(w, np.float32(c[col])), (c, rule, w)


def test_hostsim_entries_do_not_depend_on_the_table():
    """An entry's outputs alone equal its outputs in tables with other entries added, removed and reordered."""
    lib = sim()
    rng = np.random.default_rng(42)
    entries = table_cases(rng)
    for rule in RULES:
        base = sim_totals(lib, entries, rule)
        for trial in range(3):
            keep = np.sort(rng.choice(len(entries), size=len(entries) // 2, replace=False))
            extra = [(special_map(rng, int(rng.integers(0, 5000)), "plain"), -np.inf, True, True) for _ in range(5)]
            order = rng.permutation(len(keep) + len(extra)).tolist()
            table = [entries[keep[i]] if i < len(keep) else extra[i - len(keep)] for i in order]
            got = sim_totals(lib, table, rule)
            for pos, i in enumerate(order):
                if i < len(keep):
                    assert same_out(got[pos], base[keep[i]]), (trial, i)
        for j in range(0, len(entries), 17):
            alone = sim_totals(lib, [entries[j]], rule)[0]
            assert same_out(alone, base[j]), j


def test_totals_agree_with_np_sum():
    """Non-negative maps: |total - np.sum(map, float64)| <= n * 2^-52 * total (two double sums of n terms each)."""
    lib = sim()
    rng = np.random.default_rng(43)
    maps = [special_map(rng, n, "plain") for n in SIZES[1:]] + [rng.random(2_000_000).astype(np.float32)]
    res = sim_totals(lib, [(m, -np.inf, True, False) for m in maps], ONE)
    for m, (t, _) in zip(maps, res):
        ref = float(np.sum(m, dtype=np.float64))
        assert abs(t - ref) <= len(m) * 2.0 ** -52 * ref, (len(m), t, ref)


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


def device_totals(ctx, entries, rule, order=None, maps=None, stream=None):
    """One total_block_maps call over `entries` ([(map, limit, has_total, has_weight)]) in table order `order`, every total and
    weight inside guard bytes of one buffer. maps: device tensors of the maps (uploaded when None). Returns
    [(total or None, weight or None)] in the entries' order; checks the guards and the launch count."""
    import torch
    dev = torch.device("cuda", 0)
    order = list(range(len(entries))) if order is None else order
    if maps is None:
        maps = [torch.from_numpy(np.ascontiguousarray(m, np.float32)).to(dev) if len(m) else None for m, _, _, _ in entries]
    offs, pos = [], GUARD
    for _ in entries:
        offs.append((pos, pos + 8 + GUARD))
        pos += 8 + GUARD + 8 + GUARD
    host = np.full(pos, POISON, np.uint8)
    out = torch.from_numpy(host.copy()).to(dev)
    base = out.data_ptr()
    table = []
    for j in order:
        m, lim, ht, hw = entries[j]
        table.append((maps[j].data_ptr() if maps[j] is not None else 0, len(m), lim, base + offs[j][0] if ht else 0, base + offs[j][1] if hw else 0))
    st = stream or torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    n0 = ctx.launch_count()
    ctx.total_block_maps(table, rule, stream=st.cuda_stream)
    assert ctx.launch_count() == n0 + (TOTAL_LAUNCHES if entries else 0)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    mask = np.ones(pos, bool)
    res = []
    for (to, wo), (_, _, ht, hw) in zip(offs, entries):
        t = float(got[to:to + 8].view(np.float64)[0]) if ht else None
        w = got[wo:wo + 4].view(np.float32)[0] if hw else None
        if ht:
            mask[to:to + 8] = False
        if hw:
            mask[wo:wo + 4] = False
        res.append((t, w))
    assert np.array_equal(got[mask], host[mask]), "a guard byte or an output left NULL changed"
    return res


def check_against_sim(res, entries, rule, what):
    want = sim_totals(sim(True), entries, rule)
    for j, (x, y) in enumerate(zip(res, want)):
        assert same_out(x, y), (what, j, x, y)


@pytest.mark.gpu
def test_totals_equal_the_simulation_twice(gpu):
    """Synthetic maps (every size up to one full round of virtual CTAs and the special values) on a decompress-only context,
    both rules, NULL totals and weights mixed in; twice each."""
    rng = np.random.default_rng(44)
    entries = table_cases(rng, small=True)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, gpu.FLG_DECOMPRESS_ONLY))
    try:
        for rule in RULES:
            a = device_totals(ctx, entries, rule)
            b = device_totals(ctx, entries, rule)
            check_against_sim(a, entries, rule, "first")
            check_against_sim(b, entries, rule, "second")
            check_entries(a, entries, rule, "numpy")
    finally:
        ctx.close()


def fast_maps(gpu, imgs, fp=(6, 6)):
    """-fast encode, decode and SQUARED_ERROR maps of U8 images (one stream), downloaded."""
    import torch
    dev = torch.device("cuda", 0)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, fp[0], fp[1], PRE_FAST, S))
    try:
        dims = [(im.shape[1], im.shape[0]) for im in imgs]
        nb = [-(-w // fp[0]) * -(-h // fp[1]) for w, h in dims]
        d_img = [torch.from_numpy(im.reshape(-1)).to(dev) for im in imgs]
        pay = [torch.zeros(n * 16, dtype=torch.uint8, device=dev) for n in nb]
        dec = [torch.zeros(im.size, dtype=torch.uint8, device=dev) for im in imgs]
        mp = [torch.zeros(n, dtype=torch.float32, device=dev) for n in nb]
        met = torch.zeros(len(imgs) * 128, dtype=torch.uint8, device=dev)
        torch.cuda.synchronize()
        ctx.compress_device_images([(d.data_ptr(), w, h, 1, p.data_ptr()) for d, (w, h), p in zip(d_img, dims, pay)], TYPE_U8)
        ctx.decompress_device_images([(p.data_ptr(), o.data_ptr(), w, h, 1) for p, o, (w, h) in zip(pay, dec, dims)], TYPE_U8)
        ctx.compute_block_metric_device_images([(d.data_ptr(), o.data_ptr(), TYPE_U8, TYPE_U8, w, h, 1, met.data_ptr() + 128 * k, m.data_ptr())
                                                for k, (d, o, (w, h), m) in enumerate(zip(d_img, dec, dims, mp))], gpu.BLOCK_SQUARED_ERROR)
        torch.cuda.synchronize()
        return [m.cpu().numpy() for m in mp]
    finally:
        ctx.close()


def mip_chain(img):
    levels = [np.ascontiguousarray(img)]
    while levels[-1].shape[0] > 1 or levels[-1].shape[1] > 1:
        a = levels[-1].astype(np.float32)
        h, w = a.shape[:2]
        h2, w2 = max(1, h // 2), max(1, w // 2)
        a = a[:h2 * 2 if h > 1 else 1, :w2 * 2 if w > 1 else 1]
        a = a.reshape(h2, a.shape[0] // h2, w2, a.shape[1] // w2, 4).mean(axis=(1, 3))
        levels.append(np.ascontiguousarray(np.round(a).astype(np.uint8)))
    return levels


@pytest.mark.gpu
def test_real_maps_in_a_shuffled_table(gpu):
    """The -fast maps of 36 textures and of a 600x400 mip chain (its smallest levels 1 block each), with NULL outputs and
    limits around each total, in one shuffled table of more than 40 entries: each entry equals itself alone and the 32-lane
    simulation, under both rules, on a decompress-only context."""
    rng = np.random.default_rng(45)
    kinds = (I.photo_like, I.uniform_noise, I.smooth_gradient, I.voronoi_flat, I.alpha_mask)
    imgs = [np.ascontiguousarray(kinds[k % 5](int(rng.choice((16, 48, 128, 200))), int(rng.choice((16, 64, 150))), seed=900 + k)) for k in range(36)]
    chain = mip_chain(I.photo_like(400, 600, seed=46))
    maps = fast_maps(gpu, imgs + chain)
    assert sum(1 for m in maps if len(m) == 1) >= 3
    entries = []
    for j, m in enumerate(maps):
        t = numpy_total(m)
        lim = [-np.inf, t, t * 0.5, t * 2.0, np.nextafter(t, -np.inf)][j % 5]
        entries.append((m, lim, j % 6 != 4, j % 4 != 2))
    assert len(entries) > 40
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, gpu.FLG_DECOMPRESS_ONLY))
    try:
        for rule in RULES:
            order = rng.permutation(len(entries)).tolist()
            table = device_totals(ctx, entries, rule, order=order)
            check_against_sim(table, entries, rule, "table")
            check_entries(table, entries, rule, "numpy")
            for j in range(0, len(entries), 5):
                alone = device_totals(ctx, [entries[j]], rule)[0]
                assert same_out(alone, table[j]), j
    finally:
        ctx.close()


@pytest.mark.gpu
def test_launch_counts(gpu):
    """Two launches whatever the number of entries; none for an empty call."""
    import torch
    rng = np.random.default_rng(47)
    m = rng.random(5000).astype(np.float32)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, gpu.FLG_DECOMPRESS_ONLY))
    try:
        device_totals(ctx, [(m, -np.inf, True, True)], ONE)
        device_totals(ctx, [(m, 1.0, True, False)] * 600, INVERSE)
        device_totals(ctx, [(np.zeros(0, np.float32), 0.0, True, True)] * 3, ONE)      # (no virtual CTA at all: still two launches)
        n0 = ctx.launch_count()
        ctx.total_block_maps([], ONE)
        ctx.total_block_maps([], INVERSE)
        torch.cuda.synchronize()
        assert ctx.launch_count() == n0
    finally:
        ctx.close()


@pytest.mark.gpu
def test_errors_follow_the_documented_order_and_launch_nothing(gpu):
    import torch
    dev = torch.device("cuda", 0)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, gpu.FLG_DECOMPRESS_ONLY))
    buf = torch.full((4096,), POISON, dtype=torch.uint8, device=dev)
    base = buf.data_ptr()
    l = gpu.lib()
    P = gpu.ERR_BAD_PARAM

    def call(entries=True, entry_count=None, rule=ONE, table=None, **e):
        d = dict(map=base, block_count=64, limit=0.0, total=base + 1024, weight=base + 2048)
        d.update(e)
        et = table if table is not None else (gpu.BlockMapTotal * 2)(
            gpu.BlockMapTotal(C.c_void_p(d["map"] or None), d["block_count"], d["limit"], C.c_void_p(d["total"] or None), C.c_void_p(d["weight"] or None)),
            gpu.BlockMapTotal(C.c_void_p(base + 512), 8, 0.0, C.c_void_p(base + 1536), C.c_void_p(base + 2560)))
        torch.cuda.synchronize()
        before = buf.cpu().numpy()
        n0 = ctx.launch_count()
        ec = 2 if entry_count is None else entry_count
        r = l.astcenc_b200_total_block_maps(ctx.handle, et if entries else None, ec, rule, None)
        torch.cuda.synchronize()
        if r != 0 or ec == 0:
            assert ctx.launch_count() == n0
            assert np.array_equal(buf.cpu().numpy(), before)
        else:
            assert ctx.launch_count() == n0 + TOTAL_LAUNCHES
        return r

    try:
        assert call() == 0
        assert call(rule=INVERSE) == 0
        assert call(total=0, weight=0) == 0
        assert call(map=0, block_count=0) == 0
        assert call(limit=-np.inf) == 0 and call(limit=np.inf) == 0
        assert call(entry_count=0) == 0
        assert call(entries=False, entry_count=0) == 0
        nan = float("nan")
        bad_later = dict(rule=7, map=0, limit=nan, total=base + 4)
        # step 1, with every later check failing too
        assert l.astcenc_b200_total_block_maps(None, None, 0, ONE, None) == P
        assert l.astcenc_b200_total_block_maps(None, None, 0, 7, None) == P
        assert call(entries=False, **bad_later) == P
        # step 2
        for r in (2, -1, 7):
            assert call(rule=r, map=0, limit=nan) == P
        # step 3
        for s in (dict(map=0), dict(limit=nan), dict(map=base + 2), dict(weight=base + 2049), dict(total=base + 1028), dict(total=base + 1025)):
            assert call(**s) == P, s
        # step 4: more than 2^31 - 1 virtual CTAs (entries of 592 each; nothing is read)
        n = (0x7FFFFFFF // 592) + 1
        tab = np.zeros(n, dtype=np.dtype([("map", np.uint64), ("block_count", np.uint32), ("limit", np.float64), ("total", np.uint64),
                                          ("weight", np.uint64)], align=True))
        assert tab.dtype.itemsize == C.sizeof(gpu.BlockMapTotal)
        tab["map"] = base
        tab["block_count"] = 0xFFFFFFFF
        big = C.cast(tab.ctypes.data, C.POINTER(gpu.BlockMapTotal))
        assert call(table=big, entry_count=n) == P
    finally:
        ctx.close()


@pytest.mark.gpu
def test_weights_feed_select_blocks_pooled_on_the_stream(gpu):
    """total_block_maps writes the weights and select_blocks_pooled (one pool, threshold 0) reads them on the same stream with no
    host sync; the selection equals the numpy pooled rule run with the weights read back, under both rules."""
    import torch
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(48)
    maps = [(rng.random(int(n)) * s).astype(np.float32) for n, s in zip(rng.integers(1, 3000, size=12), (0.1, 1, 10, 100) * 3)]
    maps[3][5] = np.inf
    totals = [numpy_total(m) for m in maps]
    limits = [-np.inf, np.inf, totals[2], totals[3], totals[4] * 2, totals[5] * 0.5, 0.0, -np.inf, totals[8] * 1.01, totals[9] * 0.99, -np.inf, 1.0]
    d_maps = [torch.from_numpy(m).to(dev) for m in maps]
    K = 700
    d_w = torch.full((len(maps),), 7.0, dtype=torch.float32, device=dev)
    d_t = torch.zeros(len(maps), dtype=torch.float64, device=dev)
    d_idx = [torch.full((min(K, len(m)),), -1, dtype=torch.int32, device=dev) for m in maps]
    d_cnt = torch.zeros(len(maps), dtype=torch.int32, device=dev)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, gpu.FLG_DECOMPRESS_ONLY))
    st = torch.cuda.Stream(device=dev)
    try:
        for rule in RULES:
            torch.cuda.synchronize()
            ctx.total_block_maps([(d.data_ptr(), len(m), lim, d_t.data_ptr() + 8 * k, d_w.data_ptr() + 4 * k)
                                  for k, (d, m, lim) in enumerate(zip(d_maps, maps, limits))], rule, stream=st.cuda_stream)
            ctx.select_blocks_pooled([(len(maps), 0.0, K)], [(d.data_ptr(), len(m), d_w.data_ptr() + 4 * k, ix.data_ptr(), d_cnt.data_ptr() + 4 * k)
                                                            for k, (d, m, ix) in enumerate(zip(d_maps, maps, d_idx))], stream=st.cuda_stream)
            st.synchronize()
            w = d_w.cpu().numpy()
            for k in range(len(maps)):
                assert same(w[k], numpy_weight(totals[k], limits[k], rule)), (rule, k)
                assert same(float(d_t[k].item()), totals[k]), (rule, k)
            assert np.sum(w == 0) >= 4 and np.sum(w > 0) >= 4
            want = numpy_pooled([(len(maps), 0.0, K)], [(m, float(x)) for m, x in zip(maps, w)])
            cnt = d_cnt.cpu().numpy()
            for k in range(len(maps)):
                assert cnt[k] == len(want[k]), (rule, k)
                assert np.array_equal(d_idx[k].cpu().numpy()[:cnt[k]].view(np.uint32), want[k]), (rule, k)
                if w[k] == 0:
                    assert cnt[k] == 0, (rule, k)
    finally:
        ctx.close()


# ---- the gated closed loop ----
def mixed_set():
    """The 64-texture mixed set of tools/pooled_select_probe.py: sizes 32-512, five kinds of content."""
    kinds = (I.photo_like, I.uniform_noise, I.smooth_gradient, I.voronoi_flat, I.alpha_mask)
    sizes = (32, 64, 128, 256, 512)
    rng = np.random.default_rng(7)
    out = []
    for k in range(64):
        h, w = int(rng.choice(sizes)), int(rng.choice(sizes))
        out.append(np.ascontiguousarray(kinds[k % len(kinds)](h, w, seed=500 + k)))
    return out


class Ladder:
    """A set of images resident on the device with a payload, a decode and a map of `metric` each, for the contexts of `profile`
    at 6x6 (-fast to start, -thorough to refine)."""

    def __init__(self, gpu, imgs, profile, metric, comps):
        import torch
        self.gpu, self.imgs, self.metric, self.comps = gpu, imgs, metric, comps
        self.dev = torch.device("cuda", 0)
        self.hdr = profile == PRF_HDR
        self.dt = TYPE_F16 if self.hdr else TYPE_U8
        self.dims = [(im.shape[1], im.shape[0]) for im in imgs]
        self.nb = [-(-w // 6) * -(-h // 6) for w, h in self.dims]
        self.fast = gpu.Context(gpu.config_init(profile, 6, 6, PRE_FAST, S))
        self.thorough = gpu.Context(gpu.config_init(profile, 6, 6, PRE_THOROUGH, S))
        self.d_img = [torch.from_numpy(im.reshape(-1).view(np.uint8)).to(self.dev) for im in imgs]
        self.pay = [torch.zeros(n * 16, dtype=torch.uint8, device=self.dev) for n in self.nb]
        self.dec = [torch.zeros(im.nbytes, dtype=torch.uint8, device=self.dev) for im in imgs]
        self.map = [torch.zeros(n, dtype=torch.float32, device=self.dev) for n in self.nb]
        self.met = torch.zeros(len(imgs) * 128, dtype=torch.uint8, device=self.dev)

    def close(self):
        self.fast.close()
        self.thorough.close()

    def measure(self, ctx, maps, s):
        ctx.compute_block_metric_device_images([(d.data_ptr(), o.data_ptr(), self.dt, self.dt, w, h, 1, self.met.data_ptr() + 128 * k, m.data_ptr())
                                                for k, (d, o, (w, h), m) in enumerate(zip(self.d_img, self.dec, self.dims, maps))], self.metric,
                                               hdr=self.hdr, input_components=self.comps, stream=s)

    def start(self, s):
        self.fast.compress_device_images([(d.data_ptr(), w, h, 1, p.data_ptr()) for d, (w, h), p in zip(self.d_img, self.dims, self.pay)], self.dt, stream=s)
        self.fast.decompress_device_images([(p.data_ptr(), o.data_ptr(), w, h, 1) for p, o, (w, h) in zip(self.pay, self.dec, self.dims)], self.dt, stream=s)
        self.measure(self.fast, self.map, s)

    def totals(self, limits, d_t, d_w, s):
        self.fast.total_block_maps([(m.data_ptr(), n, lim, d_t.data_ptr() + 8 * k, d_w.data_ptr() + 4 * k)
                                    for k, (m, n, lim) in enumerate(zip(self.map, self.nb, limits))], self.gpu.WEIGHT_ONE, stream=s)

    def round(self, K, d_w, d_idx, d_cnt, s):
        self.fast.select_blocks_pooled([(len(self.imgs), 0.0, K)], [(m.data_ptr(), n, d_w.data_ptr() + 4 * k, ix.data_ptr(), d_cnt.data_ptr() + 4 * k)
                                                                  for k, (m, n, ix) in enumerate(zip(self.map, self.nb, d_idx))], stream=s)
        self.thorough.refine_device_block_lists([(d.data_ptr(), w, h, 1, p.data_ptr(), o.data_ptr(), m.data_ptr(), ix.data_ptr(), d_cnt.data_ptr() + 4 * k,
                                                  ix.numel()) for k, (d, (w, h), p, o, m, ix) in
                                                 enumerate(zip(self.d_img, self.dims, self.pay, self.dec, self.map, d_idx))],
                                                self.dt, self.dt, self.metric, input_components=self.comps, stream=s)


def gated_ladder(gpu, imgs, profile, metric, comps, limits_from_totals, frac, rounds=3):
    """-fast, decode, map, then `rounds` rounds of total_block_maps(ONE) -> select_blocks_pooled (one pool, threshold 0, K = frac
    of the set's blocks) -> refine_device_block_lists at -thorough, and a last total, all enqueued on one stream before any host
    read. The limits come from a -fast pass run before (limits_from_totals of its totals). Checks the gate, the maps, the final
    totals against numpy and a whole re-measure of the final decodes; returns (totals per round, counts per round, limits)."""
    import torch
    lad = Ladder(gpu, imgs, profile, metric, comps)
    try:
        st = torch.cuda.Stream(device=lad.dev)
        s = st.cuda_stream
        N = len(imgs)
        K = max(1, int(sum(lad.nb) * frac))
        torch.cuda.synchronize()
        lad.start(s)
        st.synchronize()
        limits = limits_from_totals(np.array([numpy_total(m.cpu().numpy()) for m in lad.map]), lad)
        # the ladder, from scratch, with no host read until the end
        d_t = torch.zeros((rounds + 1, N), dtype=torch.float64, device=lad.dev)
        d_w = torch.zeros((rounds + 1, N), dtype=torch.float32, device=lad.dev)
        d_cnt = torch.zeros((rounds, N), dtype=torch.int32, device=lad.dev)
        d_idx = [[torch.zeros(min(K, n), dtype=torch.int32, device=lad.dev) for n in lad.nb] for _ in range(rounds)]
        torch.cuda.synchronize()
        lad.start(s)
        snaps = []
        for r in range(rounds):
            with torch.cuda.stream(st):
                snaps.append([m.clone() for m in lad.map])
            lad.totals(limits, d_t[r], d_w[r], s)
            lad.round(K, d_w[r], d_idx[r], d_cnt[r], s)
        with torch.cuda.stream(st):
            snaps.append([m.clone() for m in lad.map])
        lad.totals(limits, d_t[rounds], d_w[rounds], s)
        st.synchronize()
        tot, cnt = d_t.cpu().numpy(), d_cnt.cpu().numpy()
        snaps = [[m.cpu().numpy() for m in sn] for sn in snaps]
        for r in range(rounds):
            for j in range(N):
                if tot[r, j] <= limits[j]:
                    assert cnt[r, j] == 0, ("an image at its target got blocks", r, j)
                assert np.all(snaps[r + 1][j] <= snaps[r][j]), ("a map value rose", r, j)
        assert np.sum(cnt) > 0
        final = snaps[rounds]
        for j in range(N):
            assert same(tot[rounds, j], numpy_total(final[j])), j
        # a whole re-measure of the final decodes: the same maps, and figures that agree with the totals up to the map's rounding
        re = [torch.zeros_like(m) for m in lad.map]
        lad.measure(lad.fast, re, s)
        st.synchronize()
        figs = [gpu.ErrorMetrics.from_buffer_copy(lad.met.cpu().numpy()[128 * k:128 * k + C.sizeof(gpu.ErrorMetrics)].tobytes()) for k in range(N)]
        for j, ((w, h), f) in enumerate(zip(lad.dims, figs)):
            assert np.array_equal(re[j].cpu().numpy().view(np.uint32), final[j].view(np.uint32)), j
            err = f.log_rmse ** 2 * w * h if metric == gpu.BLOCK_LOG2_ERROR else sum(f.sum_squared_error[c] for c in range(4 if comps == 4 else 3))
            assert abs(err - tot[rounds, j]) <= 2.0 ** -22 * tot[rounds, j] + 1e-300, (j, err, tot[rounds, j])
        return tot, cnt, limits
    finally:
        lad.close()


@pytest.mark.gpu
def test_gated_ladder_on_the_mixed_set(gpu):
    """PSNR targets around each texture's -fast PSNR (some already met, some just above, some far above), turned into SQUARED_ERROR
    limits samples * 10^(-P / 10); 2 % of the set's blocks per round."""
    deltas = (-0.5, 0.02, 0.1, 0.5, 3.0)

    def limits(t0, lad):
        out = []
        for j, ((w, h), t) in enumerate(zip(lad.dims, t0)):
            samples = 4.0 * w * h
            psnr = 10 * np.log10(samples / t) if t > 0 else 999.0
            out.append(samples * 10 ** (-(psnr + deltas[j % len(deltas)]) / 10))
        return out

    tot, cnt, lim = gated_ladder(gpu, mixed_set(), PRF_LDR, gpu.BLOCK_SQUARED_ERROR, 4, limits, 0.02)
    met0 = tot[0] <= lim
    assert np.any(met0) and not np.all(met0)
    assert np.all(cnt[:, met0] == 0)


@pytest.mark.gpu
def test_gated_ladder_on_an_hdr_set(gpu):
    """F16 HDR textures, LOG2_ERROR maps over RGB, log_rmse targets R around each texture's -fast figure turned into limits
    R^2 * pixels; 5 % of the set's blocks per round."""
    imgs = [np.ascontiguousarray(I.hdr_noise(h, w, seed=60 + k, dtype=np.float16)) for k, (h, w) in
            enumerate([(64, 64), (96, 40), (128, 128), (30, 50), (72, 90), (6, 6), (200, 120), (48, 48)])]
    factors = (1.2, 0.999, 0.98, 0.9, 0.5)

    def limits(t0, lad):
        return [(np.sqrt(t / (w * h)) * factors[j % len(factors)]) ** 2 * (w * h) for j, ((w, h), t) in enumerate(zip(lad.dims, t0))]

    tot, cnt, lim = gated_ladder(gpu, imgs, PRF_HDR, gpu.BLOCK_LOG2_ERROR, 3, limits, 0.05)
    met0 = tot[0] <= lim
    assert np.any(met0) and not np.all(met0)
