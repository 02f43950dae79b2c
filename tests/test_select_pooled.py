"""Block selection under shared budgets (astcenc_b200_select_blocks_pooled, astc_dev_select.cuh).

CPU: the selection compiled for the host (tests/hostsim/hostsim_select_pooled.cpp, one lane and 32 lanes) against the numpy
rule of the header, over the select_maps shapes, pools of 1, 2 and 300 entries, empty entries and empty pools, ties across entries, every
kind of capacity and weight; one-entry pools without weights against hostsim_select_blocks; weight 1.0 against NULL; a pool's
output against the same pool in a shuffled table.
GPU: the call against numpy inside guard bytes, twice and in a shuffled table of 40+ pools; launch counts; one-entry pools
against select_blocks; weights written on the stream just before the call; the error order; the closed loop -fast -> decode ->
map -> pooled select -> refine_device_block_lists on one stream against the host round trip, on a texture set and a mip chain."""
import ctypes as C

import numpy as np
import pytest

import astc_images as I
from astc_ref import *  # noqa: F401,F403
from hostsim_build import host_sim
from test_block_select import numpy_select, select_maps, sim_select

S = FLG_SELF_DECOMPRESS_ONLY
SELECT_LAUNCHES = 7
POISON32 = 0xA5A5A5A5
# NULL, one, powers of two, scales float32 cannot hold exactly, zero, negatives, NaN, and one whose products overflow to inf
WEIGHTS = [None, 1.0, 2.0, 0.25, 2.0 ** -20, 0.1, 1.0 / 484, 0.0, -1.0, -0.5, float("nan"), 1e38]
_SIMS = {}


def pooled_sim(lanes32=False):
    """tests/hostsim/hostsim_select_pooled.cpp: hostsim_select.cpp with hostsim_select_pooled."""
    if lanes32 in _SIMS:
        return _SIMS[lanes32]
    lib = host_sim("hostsim_select_pooled", lanes32)
    lib.hostsim_select_blocks.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint]
    lib.hostsim_select_pooled.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_uint]
    _SIMS[lanes32] = lib
    return lib


def products(entries):
    """Each entry's products: map * float32(weight), or the map without a weight."""
    with np.errstate(invalid="ignore", over="ignore"):
        return [np.asarray(m, np.float32) if w is None else np.asarray(m, np.float32) * np.float32(w) for m, w in entries]


def numpy_pooled(pools, entries):
    """The header's numpy statement. pools: [(entry_count, threshold, capacity)]; entries: [(map, weight or None)]. Returns
    each entry's kept indices, ascending."""
    out, j = [], 0
    for n, t, cap in pools:
        prods = products(entries[j:j + n])
        pp = np.concatenate(prods) if prods else np.zeros(0, np.float32)
        cand = pp > np.float32(t)
        pp = np.where(cand, pp, np.float32(-np.inf))
        k = min(int(cap), int(cand.sum()))
        kept = np.argsort(-pp, kind="stable")[:k]
        o = 0
        for p in prods:
            part = kept[(kept >= o) & (kept < o + len(p))] - o
            out.append(np.sort(part).astype(np.uint32))
            o += len(p)
        j += n
    return out


def candidates(entries, t):
    return int(sum(np.sum(p > np.float32(t)) for p in products(entries)))


def sim_pooled(lib, pools, entries):
    """One simulated call -> [(indices written, count)] per entry; index slots past each count keep their poison."""
    maps = [np.ascontiguousarray(m, np.float32) for m, _ in entries]
    weights = [None if w is None else np.array([w], np.float32) for _, w in entries]
    caps = [cap for n, _, cap in pools for _ in range(n)]
    outs = [np.full(max(1, min(c, len(m))), POISON32, np.uint32) for c, m in zip(caps, maps)]
    n = len(entries)
    pe = np.array([p[0] for p in pools], np.uint32)
    pt = np.array([p[1] for p in pools], np.float32)
    pc = np.array([p[2] for p in pools], np.uint32)
    mp = (C.c_void_p * max(1, n))(*[m.ctypes.data for m in maps])
    bc = np.array([len(m) for m in maps] or [0], np.uint32)
    wp = (C.c_void_p * max(1, n))(*[None if w is None else w.ctypes.data for w in weights])
    op = (C.c_void_p * max(1, n))(*[o.ctypes.data for o in outs])
    counts = np.full(max(1, n), 0xFFFFFFFF, np.uint32)
    lib.hostsim_select_pooled(pe.ctypes.data, pt.ctypes.data, pc.ctypes.data, len(pools), mp, bc.ctypes.data, wp, op, counts.ctypes.data, n)
    res = []
    for o, k in zip(outs, counts[:n].tolist()):
        assert k <= len(o) or k == 0, "a count beyond the entry's room"
        assert np.all(o[k:] == POISON32), "an index past the count was written"
        res.append((o[:k].copy(), k))
    return res


def check(res, want, what):
    assert len(res) == len(want)
    for j, ((got, k), w) in enumerate(zip(res, want)):
        assert k == len(w), (what, j, k, len(w))
        assert np.array_equal(got, w), (what, j)


def caps_for(c, total):
    return sorted({0, 1, max(1, c // 3), c, c + 5, total + 7})


def pool_cases(rng, small=False):
    """[(pools, entries)] calls: one-entry and two-entry pools over the select_maps shapes with every weight and threshold kind,
    a 300-entry pool with ties across entries, empty entries and pools with no entries."""
    maps = select_maps(rng)
    if small:
        maps = [m for m in maps if len(m) <= 1100]
    calls = []
    # one-entry pools: every map, a weight each, the usual thresholds and capacities
    for i, m in enumerate(maps):
        w = WEIGHTS[i % len(WEIGHTS)]
        pools, entries = [], []
        for t in (-np.inf, 0.0, 0.5):
            c = candidates([(m, w)], t)
            for cap in caps_for(c, len(m)):
                pools.append((1, t, cap))
                entries.append((m, w))
        calls.append((pools, entries))
    # two-entry pools: neighbouring maps, mixed weights, and an empty pool between them
    pools, entries = [], []
    for i in range(0, len(maps) - 1, 2 if not small else 3):
        pair = [(maps[i], WEIGHTS[(i + 3) % len(WEIGHTS)]), (maps[i + 1], WEIGHTS[(i + 7) % len(WEIGHTS)])]
        t = -np.inf if i % 4 == 0 else 0.0
        c = candidates(pair, t)
        for cap in caps_for(c, len(pair[0][0]) + len(pair[1][0]))[1:4]:
            pools.append((2, t, cap))
            entries += pair
        pools.append((0, 0.0, 5))
    calls.append((pools, entries))
    # a 300-entry pool: small quantised maps (ties inside and across entries), 0-block entries, weights that keep ties
    big = []
    for j in range(300):
        n = 0 if j % 37 == 0 else int(rng.integers(1, 12 if small else 40))
        q = (np.round(rng.normal(size=n) * 2).astype(np.float32) / 4)
        big.append((q, [None, 1.0, 2.0, 0.5][j % 4]))
    c = candidates(big, 0.0)
    total = sum(len(m) for m, _ in big)
    pools = [(0, -np.inf, 3)] + [(300, 0.0, cap) for cap in (0, 1, c // 2, c, c + 5, total + 1)] + [(0, 1.0, 0)]
    calls.append((pools, big * 6))
    return calls


def ties_across_entries():
    """Entries of one constant: every product ties, and the capacity cuts inside an entry, at an entry's end and inside the
    next; a -0.0 entry ties with 0.0."""
    e = [(np.full(5, 0.5, np.float32), None), (np.full(3, 0.25, np.float32), 2.0), (np.zeros(0, np.float32), None), (np.full(4, 0.5, np.float32), None)]
    z = [(np.full(3, -0.0, np.float32), None), (np.zeros(4, np.float32), None)]
    pools = [(4, -np.inf, cap) for cap in (0, 3, 5, 8, 9, 12, 13)] + [(2, -1.0, cap) for cap in (2, 3, 5)]
    return pools, e * 7 + z * 3


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lanes32", [False, True], ids=["1lane", "32lanes"])
def test_hostsim_pooled_equals_numpy(lanes32):
    lib = pooled_sim(lanes32)
    rng = np.random.default_rng(20)
    for k, (pools, entries) in enumerate(pool_cases(rng, small=lanes32) + [ties_across_entries()]):
        check(sim_pooled(lib, pools, entries), numpy_pooled(pools, entries), k)


def test_hostsim_pooled_no_entries():
    lib = pooled_sim()
    assert sim_pooled(lib, [], []) == []
    assert sim_pooled(lib, [(0, 0.0, 4), (0, -np.inf, 0)], []) == []


def test_hostsim_one_entry_pools_equal_select_blocks():
    """Every index, count and untouched poison word of hostsim_select_blocks."""
    lib = pooled_sim()
    rng = np.random.default_rng(21)
    cases = []
    for m in select_maps(rng):
        for t in (-np.inf, 0.0, np.inf):
            c = int(np.sum(m > np.float32(t)))
            cases += [(m, t, cap) for cap in caps_for(c, len(m))]
    # hostsim_select_blocks over index buffers of max(1, capacity) words; the same buffers here
    maps = [np.ascontiguousarray(m, np.float32) for m, _, _ in cases]
    outs = [np.full(max(1, c), POISON32, np.uint32) for _, _, c in cases]
    n = len(cases)
    pe = np.ones(n, np.uint32)
    pt = np.array([t for _, t, _ in cases], np.float32)
    pc = np.array([c for _, _, c in cases], np.uint32)
    mp = (C.c_void_p * n)(*[m.ctypes.data for m in maps])
    bc = np.array([len(m) for m in maps], np.uint32)
    wp = (C.c_void_p * n)(*([None] * n))
    op = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
    counts = np.full(n, 0xFFFFFFFF, np.uint32)
    lib.hostsim_select_pooled(pe.ctypes.data, pt.ctypes.data, pc.ctypes.data, n, mp, bc.ctypes.data, wp, op, counts.ctypes.data, n)
    want = sim_select(lib, cases)
    for j, ((w, wk), o) in enumerate(zip(want, outs)):
        assert counts[j] == wk, j
        assert np.array_equal(o[:wk], w), j
        assert np.all(o[wk:] == POISON32), j
        assert np.array_equal(w, numpy_select(*cases[j])), j


def test_hostsim_weight_one_equals_no_weight():
    lib = pooled_sim()
    rng = np.random.default_rng(22)
    for pools, entries in pool_cases(rng, small=True):
        plain = [(m, None) for m, _ in entries]
        ones = [(m, 1.0) for m, _ in entries]
        assert [(g.tobytes(), k) for g, k in sim_pooled(lib, pools, plain)] == [(g.tobytes(), k) for g, k in sim_pooled(lib, pools, ones)]


def test_hostsim_shuffled_pools_keep_their_outputs():
    lib = pooled_sim()
    rng = np.random.default_rng(23)
    for pools, entries in pool_cases(rng, small=True)[-2:] + [ties_across_entries()]:
        runs, j = [], 0
        for p in pools:
            runs.append((p, entries[j:j + p[0]]))
            j += p[0]
        base = sim_pooled(lib, pools, entries)
        order = rng.permutation(len(runs)).tolist()
        sp = [runs[i][0] for i in order]
        se = [e for i in order for e in runs[i][1]]
        shuffled = sim_pooled(lib, sp, se)
        starts = np.cumsum([0] + [p[0] for p in pools])
        sstarts = np.cumsum([0] + [p[0] for p in sp])
        for pos, i in enumerate(order):
            a = base[starts[i]:starts[i + 1]]
            b = shuffled[sstarts[pos]:sstarts[pos + 1]]
            assert [(g.tobytes(), k) for g, k in a] == [(g.tobytes(), k) for g, k in b], i


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


def device_pooled(ctx, pools, entries, order=None, stream=None):
    """One select_blocks_pooled call over `pools` (their runs of `entries`) in pool order `order`, every index list, count and
    weight inside guard bytes of one buffer. Returns [(indices, count)] in the entries' order; checks the guards, the poison past
    each count, the weights and the launch count."""
    import torch
    dev = torch.device("cuda", 0)
    starts = np.cumsum([0] + [p[0] for p in pools]).tolist()
    order = list(range(len(pools))) if order is None else order
    caps = [cap for n, _, cap in pools for _ in range(n)]
    maps = [torch.from_numpy(np.ascontiguousarray(m, np.float32)).to(dev) if len(m) else None for m, _ in entries]
    offs, pos = [], GUARD
    for (m, w), cap in zip(entries, caps):
        i = pos
        pos += 4 * min(cap, len(m)) + GUARD
        k = pos
        pos += 4 + GUARD
        wo = pos
        pos += 4 + GUARD
        offs.append((i, k, wo))
    host = np.full(pos, POISON, np.uint8)
    for (_, w), (_, _, wo) in zip(entries, offs):
        if w is not None:
            host[wo:wo + 4] = np.array([w], np.float32).view(np.uint8)
    out = torch.from_numpy(host.copy()).to(dev)
    base = out.data_ptr()
    table_pools, table_entries = [], []
    for p in order:
        table_pools.append(pools[p])
        for j in range(starts[p], starts[p + 1]):
            m, w = entries[j]
            table_entries.append((maps[j].data_ptr() if maps[j] is not None else 0, len(m), base + offs[j][2] if w is not None else 0,
                                  base + offs[j][0], base + offs[j][1]))
    st = stream or torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    n0 = ctx.launch_count()
    ctx.select_blocks_pooled(table_pools, table_entries, stream=st.cuda_stream)
    assert ctx.launch_count() == n0 + (SELECT_LAUNCHES if entries else 0)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    mask = np.ones(pos, bool)
    res = []
    for (i, k, wo), cap in zip(offs, caps):
        cnt = int(got[k:k + 4].view(np.uint32)[0])
        assert cnt <= cap
        res.append((got[i:i + 4 * cnt].view(np.uint32).copy(), cnt))
        mask[i:i + 4 * cnt] = False
        mask[k:k + 4] = False
    assert np.array_equal(got[mask], host[mask]), "a guard byte, a weight or an index past a count changed"
    return res


def gpu_cases(rng):
    calls = pool_cases(rng)
    big = rng.random(300000).astype(np.float32)
    big[rng.random(300000) < 0.01] = 0.5
    other = rng.random(70000).astype(np.float32) * 2
    entries = [(big, None), (other, 0.25), (big, 1.0 / 484), (np.zeros(0, np.float32), 2.0), (other, 1e38)]
    c = candidates(entries, -np.inf)
    calls.append(([(5, -np.inf, cap) for cap in (4664, 100000, c, c + 5)], entries * 4))
    return calls


@pytest.mark.gpu
def test_pooled_equals_numpy_twice(gpu):
    rng = np.random.default_rng(24)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, gpu.FLG_DECOMPRESS_ONLY))
    try:
        for k, (pools, entries) in enumerate(gpu_cases(rng) + [ties_across_entries()]):
            want = numpy_pooled(pools, entries)
            a = device_pooled(ctx, pools, entries)
            b = device_pooled(ctx, pools, entries)
            check(a, want, k)
            check(b, want, k)
    finally:
        ctx.close()


@pytest.mark.gpu
def test_pools_alone_equal_the_same_pools_in_a_shuffled_table(gpu):
    """At least 40 pools in one call, in shuffled order: each pool's outputs equal the pool alone and the numpy rule."""
    rng = np.random.default_rng(25)
    pools, entries = [], []
    for p_, e_ in pool_cases(rng)[:-1] + [ties_across_entries()]:
        pools += p_
        entries += e_
    runs, j = [], 0
    for p in pools:
        runs.append((p, entries[j:j + p[0]]))
        j += p[0]
    pick = rng.choice(len(runs), size=min(len(runs), 60), replace=False).tolist()
    runs = [runs[i] for i in pick]
    assert len(runs) >= 40
    pools = [r[0] for r in runs]
    entries = [e for r in runs for e in r[1]]
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 4, 4, PRE_FAST, S))
    try:
        order = rng.permutation(len(pools)).tolist()
        table = device_pooled(ctx, pools, entries, order=order)
        want = numpy_pooled(pools, entries)
        check(table, want, "table")
        j = 0
        for p, e in runs:
            alone = device_pooled(ctx, [p], e)
            assert [(g.tobytes(), k) for g, k in alone] == [(g.tobytes(), k) for g, k in table[j:j + p[0]]]
            j += p[0]
    finally:
        ctx.close()


@pytest.mark.gpu
def test_launch_counts(gpu):
    """One memset and 7 launches whatever the number of pools and entries; none without entries."""
    import torch
    rng = np.random.default_rng(26)
    m = rng.random(5000).astype(np.float32)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, gpu.FLG_DECOMPRESS_ONLY))
    try:
        device_pooled(ctx, [(1, -np.inf, 10)], [(m, None)])
        device_pooled(ctx, [(3, 0.5, 100)] * 200, [(m, 2.0)] * 600)
        device_pooled(ctx, [(0, 0.0, 5)] * 4, [])
        n0 = ctx.launch_count()
        ctx.select_blocks_pooled([], [])
        ctx.select_blocks_pooled([(0, 1.0, 3)] * 7, [])
        torch.cuda.synchronize()
        assert ctx.launch_count() == n0
    finally:
        ctx.close()


@pytest.mark.gpu
def test_one_entry_pools_equal_select_blocks(gpu):
    from test_block_select import device_select, select_cases
    rng = np.random.default_rng(27)
    cases = select_cases(rng)[::2]
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, gpu.FLG_DECOMPRESS_ONLY))
    try:
        a = device_select(ctx, cases)
        b = device_pooled(ctx, [(1, t, cap) for _, t, cap in cases], [(m, None) for m, _, _ in cases])
        for j, ((ga, ka), (gb, kb)) in enumerate(zip(a, b)):
            assert ka == kb and ga.tobytes() == gb.tobytes(), j
    finally:
        ctx.close()


@pytest.mark.gpu
def test_weights_written_on_the_stream_just_before_the_call_are_used(gpu):
    """The weights are read when the call runs: a kernel on the same stream rewrites them right before it."""
    import torch
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(28)
    maps = [rng.random(3000).astype(np.float32) for _ in range(3)]
    d_maps = [torch.from_numpy(m).to(dev) for m in maps]
    d_w = torch.ones(3, dtype=torch.float32, device=dev)
    d_idx = torch.full((3, 500), -1, dtype=torch.int32, device=dev)
    d_cnt = torch.zeros(3, dtype=torch.int32, device=dev)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, gpu.FLG_DECOMPRESS_ONLY))
    st = torch.cuda.Stream(device=dev)
    try:
        new_w = np.array([0.01, 3.0, 0.5], np.float32)
        torch.cuda.synchronize()
        with torch.cuda.stream(st):
            d_w.copy_(torch.from_numpy(new_w).to(dev, non_blocking=False) * 1.0)      # (a kernel on st)
            ctx.select_blocks_pooled([(3, -np.inf, 500)], [(d.data_ptr(), 3000, d_w.data_ptr() + 4 * k, d_idx[k].data_ptr(), d_cnt.data_ptr() + 4 * k)
                                                           for k, d in enumerate(d_maps)], stream=st.cuda_stream)
        st.synchronize()
        want = numpy_pooled([(3, -np.inf, 500)], [(m, float(w)) for m, w in zip(maps, new_w)])
        stale = numpy_pooled([(3, -np.inf, 500)], [(m, 1.0) for m in maps])
        assert [len(w) for w in want] != [len(w) for w in stale]
        cnt = d_cnt.cpu().numpy()
        idx = d_idx.cpu().numpy().view(np.uint32)
        for k in range(3):
            assert cnt[k] == len(want[k]) and np.array_equal(idx[k, :cnt[k]], want[k]), k
    finally:
        ctx.close()


@pytest.mark.gpu
def test_pooled_errors_follow_the_documented_order_and_launch_nothing(gpu):
    import torch
    dev = torch.device("cuda", 0)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, gpu.FLG_DECOMPRESS_ONLY))
    buf = torch.full((4096,), POISON, dtype=torch.uint8, device=dev)
    base = buf.data_ptr()
    l = gpu.lib()
    P = gpu.ERR_BAD_PARAM

    def call(pools=True, entries=True, pool_count=None, entry_count=None, pool=None, pool2=None, **e):
        p = dict(entry_count=1, threshold=-np.inf, capacity=8)
        p.update(pool or {})
        p2 = dict(entry_count=1, threshold=0.0, capacity=8)
        p2.update(pool2 or {})
        d = dict(map=base, block_count=64, weight=base + 3072, indices=base + 1024, count=base + 2048)
        d.update(e)
        pt = (gpu.BlockPool * 2)(gpu.BlockPool(p["entry_count"], p["threshold"], p["capacity"]),
                                 gpu.BlockPool(p2["entry_count"], p2["threshold"], p2["capacity"]))
        et = (gpu.PooledSelection * 2)(*[gpu.PooledSelection(C.c_void_p(d["map"] or None), d["block_count"], C.c_void_p(d["weight"] or None),
                                                              C.c_void_p(d["indices"] or None), C.c_void_p(d["count"] or None))] * 2)
        torch.cuda.synchronize()
        before = buf.cpu().numpy()
        n0 = ctx.launch_count()
        ec = 2 if entry_count is None else entry_count
        r = l.astcenc_b200_select_blocks_pooled(ctx.handle, pt if pools else None, 2 if pool_count is None else pool_count, et if entries else None, ec,
                                                None)
        torch.cuda.synchronize()
        if r != 0 or ec == 0:
            assert ctx.launch_count() == n0
            assert np.array_equal(buf.cpu().numpy(), before)
        else:
            assert ctx.launch_count() == n0 + SELECT_LAUNCHES
        return r

    try:
        assert call() == 0
        assert call(weight=0) == 0
        assert call(map=0, block_count=0) == 0
        assert call(indices=0, pool=dict(capacity=0), pool2=dict(capacity=0)) == 0
        assert call(pool=dict(entry_count=0), pool2=dict(entry_count=0), entry_count=0) == 0
        assert call(pools=False, pool_count=0, entries=False, entry_count=0) == 0
        assert call(pools=False, pool_count=0, entry_count=0) == 0
        # step 1, with every later check failing too
        nan = float("nan")
        bad_later = dict(pool=dict(threshold=nan, entry_count=5), map=0, indices=base + 2, count=0)
        assert l.astcenc_b200_select_blocks_pooled(None, None, 0, None, 0, None) == P
        assert call(pools=False, **bad_later) == P
        assert call(entries=False, **bad_later) == P
        assert call(pools=False, pool_count=2, entries=False, entry_count=0) == P
        # step 2
        for s in (dict(pool=dict(threshold=nan)), dict(pool2=dict(threshold=nan)), dict(pool=dict(entry_count=2)), dict(entry_count=1),
                  dict(pool=dict(entry_count=0xFFFFFFFF), pool2=dict(entry_count=3)),      # (the sum wraps to 2 in 32 bits)
                  dict(pool=dict(threshold=nan), map=0, count=0)):
            assert call(**s) == P, s
        # step 3
        for s in (dict(count=0), dict(map=0), dict(indices=0), dict(map=base + 2), dict(weight=base + 3073), dict(indices=base + 1026),
                  dict(count=base + 2049), dict(indices=0, pool=dict(capacity=0))):
            assert call(**s) == P, s
        torch.cuda.synchronize()
    finally:
        ctx.close()


# ---- the closed loop ----
def nblocks(h, w, fp):
    return -(-w // fp[0]) * -(-h // fp[1])


def block_mask(h, w, fp, blocks):
    """Texels of the listed blocks of an (h, w) image."""
    bx = -(-w // fp[0])
    m = np.zeros((h, w), bool)
    for b in blocks:
        y, x = divmod(int(b), bx)
        m[y * fp[1]:(y + 1) * fp[1], x * fp[0]:(x + 1) * fp[0]] = True
    return m


def closed_loop(gpu, imgs, fp, frac):
    """-fast compress, decode and squared-error maps of every image, a pooled select of K = frac of the set's blocks with no
    weight, then refine_device_block_lists (-thorough) with capacity min(K, n_j) per entry, all on one stream; against the host
    round trip: the maps downloaded, the numpy rule, compress_device_blocks per image on a copy, its whole decode and map as
    the candidates, and the keep rule (a candidate replaces its block where its value is below the old one)."""
    import torch
    dev = torch.device("cuda", 0)
    fast = gpu.Context(gpu.config_init(PRF_LDR, fp[0], fp[1], PRE_FAST, S))
    thorough = gpu.Context(gpu.config_init(PRF_LDR, fp[0], fp[1], PRE_THOROUGH, S))
    try:
        dims = [(im.shape[1], im.shape[0]) for im in imgs]
        nb = [nblocks(h, w, fp) for w, h in dims]
        K = max(1, int(sum(nb) * frac))
        caps = [min(K, n) for n in nb]
        d_img = [torch.from_numpy(im.reshape(-1)).to(dev) for im in imgs]
        d_pay = [torch.zeros(n * 16, dtype=torch.uint8, device=dev) for n in nb]
        d_dec = [torch.zeros(im.size, dtype=torch.uint8, device=dev) for im in imgs]
        d_met = torch.zeros(len(imgs) * 128, dtype=torch.uint8, device=dev)
        d_map = [torch.zeros(n, dtype=torch.float32, device=dev) for n in nb]
        d_idx = [torch.zeros(c, dtype=torch.int32, device=dev) for c in caps]
        d_cnt = torch.zeros(len(imgs), dtype=torch.int32, device=dev)
        st = torch.cuda.Stream(device=dev)
        torch.cuda.synchronize()
        s = st.cuda_stream
        fast.compress_device_images([(d.data_ptr(), w, h, 1, p.data_ptr()) for d, (w, h), p in zip(d_img, dims, d_pay)], TYPE_U8, stream=s)
        fast.decompress_device_images([(p.data_ptr(), o.data_ptr(), w, h, 1) for p, o, (w, h) in zip(d_pay, d_dec, dims)], TYPE_U8, stream=s)
        fast.compute_block_metric_device_images([(d.data_ptr(), o.data_ptr(), TYPE_U8, TYPE_U8, w, h, 1, d_met.data_ptr() + 128 * k, m.data_ptr())
                                                 for k, (d, o, (w, h), m) in enumerate(zip(d_img, d_dec, dims, d_map))], gpu.BLOCK_SQUARED_ERROR, stream=s)
        with torch.cuda.stream(st):
            old = [(p.clone(), o.clone(), m.clone()) for p, o, m in zip(d_pay, d_dec, d_map)]
        fast.select_blocks_pooled([(len(imgs), -np.inf, K)], [(m.data_ptr(), n, 0, ix.data_ptr(), d_cnt.data_ptr() + 4 * k)
                                                               for k, (m, n, ix) in enumerate(zip(d_map, nb, d_idx))], stream=s)
        thorough.refine_device_block_lists([(d.data_ptr(), w, h, 1, p.data_ptr(), o.data_ptr(), m.data_ptr(), ix.data_ptr(), d_cnt.data_ptr() + 4 * k, c)
                                            for k, (d, (w, h), p, o, m, ix, c) in enumerate(zip(d_img, dims, d_pay, d_dec, d_map, d_idx, caps))],
                                           TYPE_U8, TYPE_U8, gpu.BLOCK_SQUARED_ERROR, stream=s)
        st.synchronize()
        # the host round trip
        old_h = [(p.cpu().numpy(), o.cpu().numpy(), m.cpu().numpy()) for p, o, m in old]
        lists = numpy_pooled([(len(imgs), -np.inf, K)], [(m, None) for _, _, m in old_h])
        assert sum(len(x) for x in lists) == K
        counts = d_cnt.cpu().numpy()
        cand_pay = [p.clone() for p, _, _ in old]
        for k, (d, (w, h)) in enumerate(zip(d_img, dims)):
            assert counts[k] == len(lists[k]), k
            assert np.array_equal(d_idx[k].cpu().numpy().view(np.uint32)[:counts[k]], lists[k]), k
            thorough.compress_device_blocks(d.data_ptr(), TYPE_U8, w, h, 1, lists[k], cand_pay[k].data_ptr())
        cand_dec = [torch.zeros_like(o) for _, o, _ in old]
        cand_map = [torch.zeros_like(m) for _, _, m in old]
        thorough.decompress_device_images([(p.data_ptr(), o.data_ptr(), w, h, 1) for p, o, (w, h) in zip(cand_pay, cand_dec, dims)], TYPE_U8)
        thorough.compute_block_metric_device_images([(d.data_ptr(), o.data_ptr(), TYPE_U8, TYPE_U8, w, h, 1, d_met.data_ptr() + 128 * k, m.data_ptr())
                                                     for k, (d, o, (w, h), m) in enumerate(zip(d_img, cand_dec, dims, cand_map))], gpu.BLOCK_SQUARED_ERROR)
        torch.cuda.synchronize()
        committed = 0
        for k, (w, h) in enumerate(dims):
            opay, odec, omap = old_h[k]
            cpay, cdec, cmap = cand_pay[k].cpu().numpy(), cand_dec[k].cpu().numpy(), cand_map[k].cpu().numpy()
            keep = lists[k][cmap[lists[k]] < omap[lists[k]]]
            committed += len(keep)
            want_pay, want_dec, want_map = opay.reshape(-1, 16).copy(), odec.reshape(h, w, 4).copy(), omap.copy()
            want_pay[keep] = cpay.reshape(-1, 16)[keep]
            tm = block_mask(h, w, fp, keep)
            want_dec[tm] = cdec.reshape(h, w, 4)[tm]
            want_map[keep] = cmap[keep]
            assert np.array_equal(d_pay[k].cpu().numpy().reshape(-1, 16), want_pay), ("payload", k)
            assert np.array_equal(d_dec[k].cpu().numpy().reshape(h, w, 4), want_dec), ("decode", k)
            assert np.array_equal(d_map[k].cpu().numpy().view(np.uint32), want_map.view(np.uint32)), ("map", k)
        assert committed > 0
        return lists
    finally:
        fast.close()
        thorough.close()


@pytest.mark.gpu
def test_closed_loop_on_a_texture_set(gpu):
    """256 textures of 128² at 6x6, K = 1 % of the set's blocks."""
    imgs = [I.photo_like(128, 128, seed=1000 + k) for k in range(256)]
    closed_loop(gpu, imgs, (6, 6, 1), 0.01)


@pytest.mark.gpu
def test_closed_loop_on_a_mip_chain(gpu):
    """The chain of a 300x200 image down to 1x1 at 6x6: its smallest levels have 1 block each."""
    levels = [np.ascontiguousarray(I.photo_like(200, 300, seed=31))]
    while levels[-1].shape[0] > 1 or levels[-1].shape[1] > 1:
        a = levels[-1].astype(np.float32)
        h, w = a.shape[:2]
        h2, w2 = max(1, h // 2), max(1, w // 2)
        a = a[:h2 * 2 if h > 1 else 1, :w2 * 2 if w > 1 else 1]
        a = a.reshape(h2, a.shape[0] // h2, w2, a.shape[1] // w2, 4).mean(axis=(1, 3))
        levels.append(np.ascontiguousarray(np.round(a).astype(np.uint8)))
    assert sum(1 for l in levels if nblocks(l.shape[0], l.shape[1], (6, 6)) == 1) >= 3
    closed_loop(gpu, levels, (6, 6, 1), 0.1)
