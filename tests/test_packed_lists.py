"""Packed block lists: astcenc_b200_compress_device_block_lists_packed and astcenc_b200_refine_device_block_lists_packed
(astc_dev_pack.cuh: pack_lists, astc_pack_lists_kernel; the PACKED staged_block of astc_dev_gather.cuh and its users).

CPU: the packing body of the host simulation (tests/hostsim/hostsim_pack_lists.cpp, one lane and 32 lanes) against numpy
(np.minimum, np.cumsum); the packed resolution of every staging slot against numpy, with every read of list memory checked
(no index at or beyond min(*count, capacity) of any list, no count of a list of capacity 0); the packed refine decisions and
commits against the unpacked ones.
GPU: each packed call against its unpacked call on the same lists, inside guard bytes; truncation against the unpacked call on
lists truncated by the numpy rule; the overflow word; counts written by select_blocks_pooled on the stream; launch counts and
the error order; the gated three-round loop with packed refine against the same loop unpacked."""
import ctypes as C

import numpy as np
import pytest

from astc_ref import *  # noqa: F401,F403
from hostsim_build import host_sim
from test_block_list_decode import KINDS, BlockList, make_list
from test_block_metrics import ALPHA, LOG2, METRIC_IDS, SQUARED, numpy_metric_map, soft_alpha
from test_metrics_device import DT, nblocks
from test_refine_lists import (GUARD, Guarded, State, candidates, contexts, footprint, ldr_set, numpy_refine, old_map, refine_table, sim_refine,
                               start, vol)
import astc_images as I

METRICS = (SQUARED, ALPHA, LOG2)
U32 = 0xFFFFFFFF
PACK_GUARD_WORDS = 64      # (hostsim_pack_lists.cpp: list words past the capacity that are checked too)
_SIMS = {}


def sim(lanes32=False):
    """tests/hostsim/hostsim_pack_lists.cpp compiled for the host (one simulated lane, or 32 lanes on 32 threads)."""
    if lanes32 in _SIMS:
        return _SIMS[lanes32]
    lib = host_sim("hostsim_pack_lists", lanes32)
    lib.hostsim_pack_lists.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.hostsim_pack_lists.restype = C.c_uint
    lib.hostsim_pack_slots.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_size_t, C.c_uint, C.c_void_p, C.c_void_p]
    lib.hostsim_pack_slots.restype = C.c_uint
    lib.hostsim_unpacked_slots.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_size_t, C.c_uint, C.c_void_p, C.c_void_p]
    lib.hostsim_unpacked_slots.restype = C.c_uint
    common = [C.c_void_p, C.c_void_p, C.c_uint, C.c_int, C.c_int, C.c_uint, C.c_uint, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
              C.c_void_p, C.c_void_p, C.c_int, C.c_size_t, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.hostsim_refine_decide.argtypes = common + [C.c_int]
    lib.hostsim_refine_commit.argtypes = common + [C.c_void_p]
    lib.hostsim_refine_decide_packed.argtypes = common + [C.c_int, C.c_uint]
    lib.hostsim_refine_decide_packed.restype = C.c_uint
    lib.hostsim_refine_commit_packed.argtypes = common + [C.c_void_p, C.c_uint]
    lib.hostsim_refine_commit_packed.restype = C.c_uint
    _SIMS[lanes32] = lib
    return lib


# ---- the numpy rule ----
def numpy_pack(counts, caps, budget):
    """(firsts (uint64; all ones for an entry of capacity 0), total T, overflow) of a packed call's table."""
    counts, caps = np.asarray(counts, np.uint64), np.asarray(caps, np.uint64)
    v = np.minimum(counts, caps)
    firsts = np.cumsum(v) - v
    firsts[caps == 0] = np.uint64(2 ** 64 - 1)
    s = int(np.sum(v, dtype=object)) if len(v) else 0
    return firsts, min(s, budget), min(max(s - budget, 0), U32)


def numpy_slots(lists, blocks, budget):
    """The packed call's staging slots, min(budget, sum of capacities) of them: (entry, block) per slot, or None for an invalid
    one (past the packed total, or an index out of range)."""
    out = []
    for j, (l, n) in enumerate(zip(lists, blocks)):
        for s in range(min(l.count, l.capacity)):
            b = int(l.idx[s])
            out.append((j, b) if b < n else None)
    n = min(budget, sum(l.capacity for l in lists))
    out = out[:min(len(out), budget)]
    return out + [None] * (n - len(out))


def truncated(lists, budget):
    """The lists the packed call processes under `budget`: entry j keeps its first clip(budget - P_j, 0, v_j) listed slots."""
    out, p = [], 0
    for l in lists:
        v = min(l.count, l.capacity)
        k = int(np.clip(budget - p, 0, v))
        out.append(BlockList(l.idx, k, l.capacity))
        p += v
    return out


def test_numpy_rule_small_cases():
    f, t, o = numpy_pack([3, 9, 0, 2, 7], [5, 4, 0, 2, 3], 6)
    assert f.tolist() == [0, 3, 2 ** 64 - 1, 7, 9] and t == 6 and o == 6
    assert numpy_pack([U32] * 3, [U32] * 3, 5)[1:] == (5, U32)
    ls = [BlockList([4, 1, 9], 2, 3), BlockList([0, 0], 5, 2), BlockList([], 1, 0)]
    assert numpy_slots(ls, [5, 5, 5], 3) == [(0, 4), (0, 1), (1, 0)]
    assert numpy_slots(ls, [5, 5, 5], 100) == [(0, 4), (0, 1), (1, 0), (1, 0), None]
    assert [l.count for l in truncated(ls, 3)] == [2, 1, 0]


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
def pack_tables(rng):
    """(counts, capacities) tables: counts of 0, below, at and above the capacity and 0xFFFFFFFF; capacity-0 entries; 1 entry to
    several thousand (several tiles of 256); sums beyond 2^32."""
    out = []
    for n in (1, 2, 7, 8, 9, 255, 256, 257, 600, 3001):
        caps = rng.integers(0, 40, n).astype(np.uint32)
        caps[rng.random(n) < 0.2] = 0
        kind = rng.integers(0, 5, n)
        counts = np.where(kind == 0, 0, np.where(kind == 1, caps // 2, np.where(kind == 2, caps, np.where(kind == 3, caps + 3, U32)))).astype(np.uint32)
        out.append((counts, caps))
    big = np.array([U32, U32, 7, U32, 0x80000000], np.uint32)
    out.append((big, np.array([U32, U32 - 1, 3, 0, U32], np.uint32)))
    out.append((np.zeros(3, np.uint32), np.zeros(3, np.uint32)))
    return out


def budgets(s):
    return sorted({b for b in (0, 1, s - 1, s, s + 1, U32) if 0 <= b <= U32})


@pytest.mark.parametrize("lanes32", [False, True], ids=["lanes1", "lanes32"])
def test_hostsim_packing_equals_numpy(lanes32):
    lib = sim(lanes32)
    rng = np.random.default_rng(1)
    for counts, caps in pack_tables(rng):
        n = len(counts)
        s = int(np.sum(np.minimum(counts, caps).astype(np.uint64), dtype=object))
        for budget in budgets(s):
            firsts = np.zeros(n, np.uint64)
            total = np.zeros(1, np.uint64)
            ovf = np.full(1, 0xA5A5A5A5, np.uint32)
            stray = lib.hostsim_pack_lists(counts.ctypes.data, caps.ctypes.data, n, budget, firsts.ctypes.data, total.ctypes.data, ovf.ctypes.data)
            f, t, o = numpy_pack(counts, caps, budget)
            assert stray == 0, "a count of a capacity-0 entry was read"
            assert firsts.tolist() == f.tolist(), (n, budget)
            assert int(total[0]) == t and int(ovf[0]) == o, (n, budget, int(total[0]), t, int(ovf[0]), o)
    # a null overflow pointer is not written
    counts, caps = pack_tables(rng)[3]
    firsts, total = np.zeros(len(counts), np.uint64), np.zeros(1, np.uint64)
    assert lib.hostsim_pack_lists(counts.ctypes.data, caps.ctypes.data, len(counts), 5, firsts.ctypes.data, total.ctypes.data, None) == 0
    assert firsts.tolist() == numpy_pack(counts, caps, 5)[0].tolist()


def slot_lists(rng, n_lists, blocks):
    """Lists of every kind over images of `blocks` blocks, each padded by PACK_GUARD_WORDS checked words."""
    return [make_list(rng, b, KINDS[k % len(KINDS)]) for k, b in zip(range(n_lists), blocks)]


def run_slots(lib, lists, blocks, budget, base, n, packed=True):
    padded = [np.concatenate([l.idx, np.full(PACK_GUARD_WORDS + 1, 7, np.uint32)]) for l in lists]
    ip = (C.c_void_p * len(lists))(*[p.ctypes.data for p in padded])
    counts = np.array([min(l.count, U32) for l in lists], np.uint32)
    caps = np.array([l.capacity for l in lists], np.uint32)
    nb = np.array(blocks, np.uint32)
    ent, blk = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
    if packed:
        stray = lib.hostsim_pack_slots(ip, counts.ctypes.data, caps.ctypes.data, nb.ctypes.data, len(lists), budget, base, n, ent.ctypes.data, blk.ctypes.data)
    else:
        stray = lib.hostsim_unpacked_slots(ip, counts.ctypes.data, caps.ctypes.data, nb.ctypes.data, len(lists), base, n, ent.ctypes.data, blk.ctypes.data)
    return [None if e == U32 else (int(e), int(b)) for e, b in zip(ent, blk)], stray


@pytest.mark.parametrize("lanes32", [False, True], ids=["lanes1", "lanes32"])
def test_hostsim_packed_slots_equal_numpy_and_read_no_unlisted_word(lanes32):
    """Every staging slot of packed calls over lists of every kind (invalid indices, count > capacity, slots past the count,
    count 0, capacity 0) at budgets 0, 1, sum - 1, sum, sum + 1 and 0xFFFFFFFF, whole and from chunk bases: the (entry, block)
    of numpy, with no read of an index at or beyond min(*count, capacity) nor of a capacity-0 count."""
    lib = sim(lanes32)
    rng = np.random.default_rng(2)
    for n_lists in (1, 5, 23, 300 if not lanes32 else 40):
        blocks = rng.integers(1, 60, n_lists).tolist()
        lists = slot_lists(rng, n_lists, blocks)
        s = sum(min(l.count, l.capacity) for l in lists)
        for budget in budgets(s):
            want = numpy_slots(lists, blocks, budget)
            got, stray = run_slots(lib, lists, blocks, budget, 0, len(want))
            assert stray == 0 and got == want, (n_lists, budget)
            for base in (1, 3, len(want) // 2):
                if base < len(want):
                    got, stray = run_slots(lib, lists, blocks, budget, base, len(want) - base)
                    assert stray == 0 and got == want[base:], (n_lists, budget, base)
    # the check sees a stray read: the unpacked resolution reads the index of a slot past the count
    lists = [BlockList([1, 2, 3, 4], 2, 4)]
    got, stray = run_slots(lib, lists, [10], 0, 0, 4, packed=False)
    assert got == [(0, 1), (0, 2), None, None] and stray > 0


def sim_refine_packed(lib, imgs, pays, decs, fp, components, metric, lists, maps, chunk, with_decoded, rng, budget):
    """sim_refine (test_refine_lists.py) for the packed call: the candidates staged at their packed positions, chunk by chunk
    over min(budget, sum of capacities) staging blocks; returns the payloads, decodes and maps it leaves."""
    n = len(imgs)
    shapes = [vol(a).shape[:3] for a in imgs]
    dims = np.array([[s[2], s[1], s[0]] for s in shapes], np.uint32).reshape(-1)
    out_pay = [np.full(nblocks(s, fp) * 16, 0xA5, np.uint8) for s in shapes]
    out_dec = [np.full(d.nbytes, 0xA5, np.uint8).view(d.dtype).reshape(d.shape) if with_decoded else None for d in decs]
    out_map = [m.copy() for m in maps]
    data = (C.c_void_p * n)(*[vol(a).ctypes.data for a in imgs])
    pp = (C.c_void_p * n)(*[p.ctypes.data for p in out_pay])
    dp = (C.c_void_p * n)(*[d.ctypes.data if d is not None else None for d in out_dec])
    mp = (C.c_void_p * n)(*[m.ctypes.data for m in out_map])
    padded = [np.concatenate([l.idx, np.zeros(PACK_GUARD_WORDS + 1, np.uint32)]) for l in lists]      # (the checked words are ours)
    ip = (C.c_void_p * n)(*[p.ctypes.data for p in padded])
    counts = np.array([l.count for l in lists], np.uint32)
    caps = np.array([l.capacity for l in lists], np.uint32)
    call = numpy_slots(lists, [nblocks(s, fp) for s in shapes], budget)
    for base in range(0, len(call), chunk):
        m = min(chunk, len(call) - base)
        row = rng.integers(0, 256, (fp[2], fp[1], m * fp[0], 4 * decs[0].itemsize), dtype=np.uint8).view(decs[0].dtype)
        staged = rng.integers(0, 256, (m, 16), dtype=np.uint8)
        for i in range(m):
            if call[base + i] is None:
                continue
            j, b = call[base + i]
            staged[i] = pays[j][b]
            for (z, y, x), (tz, ty, tx) in footprint(shapes[j], fp, b):
                row[tz, ty, i * fp[0] + tx] = decs[j][z, y, x]
        v = np.full(m, np.nan, np.float32)
        keep = np.full(m, 0xEE, np.uint8)
        args = (data, dims.ctypes.data, n, DT[vol(imgs[0]).dtype], DT[decs[0].dtype], fp[0], fp[1], fp[2], pp, dp, mp, ip, counts.ctypes.data,
                caps.ctypes.data, components, base, m, row.ctypes.data, v.ctypes.data, keep.ctypes.data)
        assert lib.hostsim_refine_decide_packed(*args, metric, budget) == 0, "the decisions read an unlisted word"
        assert set(keep.tolist()) <= {0, 1}
        assert lib.hostsim_refine_commit_packed(*args, staged.ctypes.data, budget) == 0, "the commits read an unlisted word"
    return out_pay, out_dec, out_map


def check_packed_refine(lib, imgs, cands, fp, components, metric, lists, rng, with_decoded=True):
    """The packed simulation at budgets sum(v), sum(capacities) and 0xFFFFFFFF equals the unpacked simulation (and the numpy
    rule) with chunks of 7; below sum(v) it equals the unpacked simulation on the truncated lists."""
    pays, decs = [c[0] for c in cands], [c[1] for c in cands]
    want_values = [numpy_metric_map(vol(a), d, fp, components, metric) for a, d in zip(imgs, decs)]
    maps = [old_map(rng, w) for w in want_values]
    s = sum(min(l.count, l.capacity) for l in lists)
    for budget in (s, sum(l.capacity for l in lists), U32, s - 1, s // 2, 1):
        eff = lists if budget >= s else truncated(lists, budget)
        want = sim_refine(lib, imgs, pays, decs, fp, components, metric, eff, maps, 7, with_decoded, rng)
        rule = numpy_refine(imgs, pays, decs, fp, components, metric, eff, maps, 7, with_decoded)
        got = sim_refine_packed(lib, imgs, pays, decs, fp, components, metric, lists, maps, 7, with_decoded, rng, budget)
        for j in range(len(imgs)):
            assert np.array_equal(got[0][j], want[0][j]) and np.array_equal(got[0][j], rule[0][j]), ("payload", budget, j)
            if with_decoded:
                assert got[1][j].tobytes() == want[1][j].tobytes() == rule[1][j].tobytes(), ("decode", budget, j)
            assert got[2][j].view(np.uint32).tolist() == want[2][j].view(np.uint32).tolist() == rule[2][j].view(np.uint32).tolist(), ("map", budget, j)


@pytest.mark.parametrize("metric", METRICS, ids=lambda m: METRIC_IDS[m])
@pytest.mark.parametrize("lanes32", [False, True], ids=["lanes1", "lanes32"])
def test_hostsim_packed_refine_equals_unpacked(oracle, lanes32, metric):
    """U8 images at 6x6 (ragged, a texture array, soft alpha) with every list kind, -medium candidates decoded to U8; with and
    without a decode."""
    rng = np.random.default_rng(300 + metric)
    fp = (6, 6, 1)
    imgs = ldr_set(rng)
    lists = [make_list(rng, nblocks(vol(a).shape[:3], fp), KINDS[k % len(KINDS)]) for k, a in enumerate(imgs)]
    cands = [candidates(oracle, a, fp, PRF_LDR, PRE_MEDIUM, TYPE_U8) for a in imgs]
    for with_decoded in ((True, False) if not lanes32 else (True,)):
        check_packed_refine(sim(lanes32), imgs, cands, fp, 4, metric, lists, rng, with_decoded)


def test_hostsim_packed_refine_volume(oracle):
    """A 4x4x4 footprint on ragged volumes in U8."""
    rng = np.random.default_rng(9)
    fp = (4, 4, 4)
    imgs = [np.stack([I.photo_like(h, w, seed=5 * k + z) for z in range(d)]) for k, (d, h, w) in enumerate([(5, 7, 9), (8, 8, 4), (1, 1, 1)])]
    lists = [make_list(rng, nblocks(a.shape[:3], fp), kind) for a, kind in zip(imgs, ("mixed", "past", "sorted"))]
    cands = [candidates(oracle, a, fp, PRF_LDR, PRE_MEDIUM, TYPE_U8) for a in imgs]
    check_packed_refine(sim(False), imgs, cands, fp, 4, SQUARED, lists, rng)


# ---------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu(pkg):
    import torch
    assert torch.cuda.is_available(), "the GPU tests need a CUDA device"
    torch.cuda.set_device(0)
    return pkg


def dev_u32(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a, np.uint32)).view(np.int32)).cuda()


class Entry:
    """One image of a compress test on the device: its texels and a list (indices and count on the device)."""

    def __init__(self, img, lst):
        import torch
        self.img = vol(img)
        self.shape = self.img.shape[:3]
        self.lst = lst
        self.d_img = torch.from_numpy(self.img.reshape(-1).view(np.uint8)).cuda()
        self.d_idx = dev_u32(lst.padded())
        self.d_cnt = dev_u32([min(lst.count, U32)])

    def dims(self):
        return self.shape[2], self.shape[1], self.shape[0]


def compress_both(ctx, entries, fp, data_type, budget, start_bytes, counts=None, order=None):
    """The packed call (budget) on payload copies A and the unpacked call on copies B, from the same bytes, each inside guard
    bytes. counts: device count words for the unpacked call (default: the lists' own). Returns (A, B, overflow word)."""
    import torch
    a = [Guarded(len(p), p) for p in start_bytes]
    b = [Guarded(len(p), p) for p in start_bytes]
    ovf = Guarded(4, np.full(4, 0xA5, np.uint8))
    order = list(range(len(entries))) if order is None else order
    cnt = [e.d_cnt.data_ptr() for e in entries] if counts is None else counts
    ctx.compress_device_block_lists_packed([(entries[j].d_img.data_ptr(), *entries[j].dims(), a[j].ptr, entries[j].d_idx.data_ptr(),
                                             entries[j].d_cnt.data_ptr(), entries[j].lst.capacity) for j in order], budget, data_type, overflow=ovf.ptr)
    ctx.compress_device_block_lists([(entries[j].d_img.data_ptr(), *entries[j].dims(), b[j].ptr, entries[j].d_idx.data_ptr(), cnt[j], entries[j].lst.capacity)
                                     for j in order], data_type)
    torch.cuda.synchronize()
    return [g.get() for g in a], [g.get() for g in b], int(ovf.get().view(np.uint32)[0])


def check_compress(ctx, imgs, lists, fp, data_type, budgets_of=None, order=None):
    """For each budget (default: sum v - 1, sum v, sum v + 1, sum of capacities, 0, 0xFFFFFFFF): the packed call equals the
    unpacked call on the lists truncated by the numpy rule, and the overflow word holds the excess."""
    import torch
    entries = [Entry(a, l) for a, l in zip(imgs, lists)]
    rng = np.random.default_rng(3)
    start_bytes = [rng.integers(0, 256, nblocks(e.shape, fp) * 16, dtype=np.uint8) for e in entries]
    s = sum(min(l.count, l.capacity) for l in lists)
    caps = sum(l.capacity for l in lists)
    changed = 0
    order = list(range(len(lists))) if order is None else order
    for budget in (budgets_of(s, caps) if budgets_of else sorted({max(s - 1, 0), s, s + 1, caps, 0, U32})):
        tr = [None] * len(lists)      # (truncation follows the call's order)
        for j, t in zip(order, truncated([lists[j] for j in order], budget)):
            tr[j] = t
        cnt = [dev_u32([l.count]) for l in tr]
        got, want, ovf = compress_both(ctx, entries, fp, data_type, budget, start_bytes, [c.data_ptr() for c in cnt], order)
        torch.cuda.synchronize()
        for j, (g, w) in enumerate(zip(got, want)):
            assert np.array_equal(g, w), ("payload", budget, j)
            changed += int(np.sum(g != start_bytes[j]))
        assert ovf == (min(max(s - budget, 0), U32) if caps else 0xA5A5A5A5), (budget, ovf, s)
    return changed


def pooled_lists(gpu, ctx, maps, K, stream=0):
    """select_blocks_pooled over device maps (one pool, capacity K): each entry's device indices (capacity min(K, n)) and count."""
    import torch
    idx = [torch.zeros(max(min(K, m.numel()), 1), dtype=torch.int32, device="cuda") for m in maps]
    cnt = torch.zeros(len(maps), dtype=torch.int32, device="cuda")
    ctx.select_blocks_pooled([(len(maps), -np.inf, K)], [(m.data_ptr(), m.numel(), 0, i.data_ptr(), cnt.data_ptr() + 4 * k) for k, (m, i) in
                                                          enumerate(zip(maps, idx))], stream=stream)
    return idx, cnt


@pytest.mark.gpu
def test_compress_packed_equals_unpacked_256_textures_with_pooled_selections(gpu):
    """256 textures of 40x40 at 6x6 with lists from select_blocks_pooled (capacities min(K, n_j), counts written on the stream by
    the selection just before each packed call): the packed call with budget K writes the unpacked call's bytes."""
    import torch
    rng = np.random.default_rng(4)
    fp = (6, 6, 1)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, 0))
    try:
        imgs = [I.photo_like(40, 40, seed=k) for k in range(256)]
        nb = nblocks((1, 40, 40), fp)
        d_img = [torch.from_numpy(a.reshape(-1).view(np.uint8)).cuda() for a in imgs]
        maps = [torch.from_numpy(rng.random(nb).astype(np.float32)).cuda() for _ in imgs]
        start_bytes = rng.integers(0, 256, nb * 16, dtype=np.uint8)
        for K in (1, 256, int(0.05 * nb * 256), nb * 256 + 3):
            stream = torch.cuda.Stream()
            s = stream.cuda_stream
            a = [Guarded(nb * 16, start_bytes) for _ in imgs]
            b = [Guarded(nb * 16, start_bytes) for _ in imgs]
            ovf = Guarded(4, np.full(4, 0xA5, np.uint8))
            torch.cuda.synchronize()
            # the counts go through a poisoned state: each call reads them as the selection on its stream leaves them
            idx, cnt = pooled_lists(gpu, ctx, maps, K, stream=s)
            table = lambda g: [(d.data_ptr(), 40, 40, 1, g[k].ptr, idx[k].data_ptr(), cnt.data_ptr() + 4 * k, min(K, nb)) for k, d in enumerate(d_img)]
            ctx.compress_device_block_lists_packed(table(a), K, TYPE_U8, overflow=ovf.ptr, stream=s)
            ctx.compress_device_block_lists(table(b), TYPE_U8, stream=s)
            stream.synchronize()
            assert int(cnt.sum().item()) == min(K, nb * 256)
            for k in range(len(imgs)):
                assert np.array_equal(a[k].get(), b[k].get()), (K, k)
            assert int(ovf.get().view(np.uint32)[0]) == 0
            assert any(not np.array_equal(a[k].get(), start_bytes) for k in range(len(imgs)))
    finally:
        ctx.close()


def mip_chain(img):
    out = [img]
    while out[-1].shape[0] > 1 or out[-1].shape[1] > 1:
        p = out[-1]
        h, w = max(1, p.shape[0] // 2), max(1, p.shape[1] // 2)
        out.append(np.ascontiguousarray(p[:2 * h:2, :2 * w:2][:h, :w]))
    return out


@pytest.mark.gpu
def test_compress_packed_mips_arrays_volumes_alpha_scale_and_types(gpu):
    """A mip chain down to 1-block levels, a texture array, a 4x4x4 volume, a context with a_scale_radius, and U8, F16 and F32
    data, each over lists of every kind at budgets around the listed total and the capacities; a shuffled table order."""
    rng = np.random.default_rng(5)
    fp = (6, 6, 1)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, 0))
    try:
        chain = mip_chain(I.photo_like(150, 200, seed=1))
        lists = [make_list(rng, nblocks((1,) + a.shape[:2], fp), KINDS[k % len(KINDS)]) for k, a in enumerate(chain)]
        assert check_compress(ctx, chain, lists, fp, TYPE_U8) > 0
        assert check_compress(ctx, chain, lists, fp, TYPE_U8, order=rng.permutation(len(chain)).tolist()) > 0
        arr = [np.stack([I.photo_like(37, 29, seed=3 + z) for z in range(3)]), I.photo_like(20, 20, seed=9)]
        lists = [make_list(rng, nblocks(vol(a).shape[:3], fp), kind) for a, kind in zip(arr, ("mixed", "sorted"))]
        assert check_compress(ctx, arr, lists, fp, TYPE_U8) > 0
        f32 = [I.photo_like(30, 41, seed=4).astype(np.float32) / 255, I.photo_like(13, 7, seed=5).astype(np.float32) / 255]
        lists = [make_list(rng, nblocks((1,) + a.shape[:2], fp), kind) for a, kind in zip(f32, ("mixed", "past"))]
        assert check_compress(ctx, f32, lists, fp, TYPE_F32) > 0
    finally:
        ctx.close()
    ctx = gpu.Context(gpu.config_init(PRF_HDR, 6, 6, PRE_FAST, 0))
    try:
        hdr = [I.hdr_noise(50, 33, seed=6, dtype=np.float16), I.hdr_noise(6, 6, seed=7, dtype=np.float16)]
        lists = [make_list(rng, nblocks((1,) + a.shape[:2], fp), kind) for a, kind in zip(hdr, ("sorted", "mixed"))]
        assert check_compress(ctx, hdr, lists, fp, TYPE_F16) > 0
    finally:
        ctx.close()
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 4, 4, PRE_FAST, 0, block_z=4))
    try:
        v = [np.stack([I.photo_like(21, 19, seed=z) for z in range(9)]), np.stack([I.photo_like(8, 8, seed=20 + z) for z in range(4)])]
        lists = [make_list(rng, nblocks(a.shape[:3], (4, 4, 4)), kind) for a, kind in zip(v, ("mixed", "sorted"))]
        assert check_compress(ctx, v, lists, (4, 4, 4), TYPE_U8) > 0
    finally:
        ctx.close()
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, 0, a_scale_radius=2))
    try:
        imgs = [soft_alpha(70, 90, seed=9), soft_alpha(33, 20, seed=10)]
        lists = [make_list(rng, nblocks((1,) + a.shape[:2], fp), kind) for a, kind in zip(imgs, ("sorted", "mixed"))]
        assert check_compress(ctx, imgs, lists, fp, TYPE_U8) > 0
    finally:
        ctx.close()


@pytest.mark.gpu
def test_compress_packed_across_chunk_edges(gpu, monkeypatch):
    """Staging rows of 37 blocks: budgets and packed totals inside and across chunk edges, and whole chunks past the total."""
    rng = np.random.default_rng(6)
    fp = (6, 6, 1)
    monkeypatch.setenv("ASTCENC_B200_BATCH_BLOCKS", "37")
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, 0))
    monkeypatch.delenv("ASTCENC_B200_BATCH_BLOCKS")
    try:
        imgs = [I.photo_like(120, 150, seed=11), I.photo_like(60, 40, seed=12), I.photo_like(90, 90, seed=13)]
        lists = []
        for a, count in zip(imgs, (30, 50, 5)):
            n = nblocks((1,) + a.shape[:2], fp)
            lists.append(BlockList(rng.integers(0, n, 200), count, 200))      # (capacities 600: whole chunks lie past the packed total)
        s = 85
        check_compress(ctx, imgs, lists, fp, TYPE_U8, budgets_of=lambda s_, c: [36, 37, 38, 74, 75, s - 1, s, s + 1, 111, 600, U32])
    finally:
        ctx.close()


def refine_both(ctx, fast, imgs, lists, fp, data_type, out_type, metric, components, budget, with_decoded=True):
    """The packed refine call (A) and the unpacked one on the lists truncated by the numpy rule (B), from the same -fast state;
    returns the host copies of both and the overflow word."""
    import torch
    states = [State(a, l, fp, out_type) for a, l in zip(imgs, lists)]
    start(ctx, fast, states, data_type, out_type, metric, components)
    torch.cuda.synchronize()
    b_states = [s.copy() for s in states]
    for s, t in zip(b_states, truncated(lists, budget)):
        s.d_cnt = dev_u32([t.count])
    ovf = Guarded(4, np.full(4, 0xA5, np.uint8))
    ctx.refine_device_block_lists_packed(refine_table(states, with_decoded), budget, data_type, out_type, metric, input_components=components, overflow=ovf.ptr)
    ctx.refine_device_block_lists(refine_table(b_states, with_decoded), data_type, out_type, metric, input_components=components)
    torch.cuda.synchronize()
    return [s.host() for s in states], [s.host() for s in b_states], int(ovf.get().view(np.uint32)[0])


@pytest.mark.gpu
@pytest.mark.parametrize("metric", METRICS, ids=lambda m: METRIC_IDS[m])
def test_refine_packed_equals_unpacked(metric, gpu):
    """LDR U8 (ragged, an array, soft alpha, every list kind) and HDR F16: payload, decode and map of the packed refine equal the
    unpacked call's, with a decode and with none, at budgets at and above the listed total; below it they equal the unpacked call
    on the truncated lists and the overflow word holds the excess."""
    rng = np.random.default_rng(20 + metric)
    fp = (6, 6, 1)
    ctx, fast = contexts(gpu, PRF_LDR, PRE_THOROUGH)
    try:
        imgs = [I.photo_like(97, 131, seed=1), soft_alpha(64, 64, seed=2), np.stack([I.photo_like(37, 29, seed=3 + z) for z in range(3)]),
                I.photo_like(120, 77, seed=4), soft_alpha(13, 50, seed=5)]
        lists = [make_list(rng, nblocks(vol(a).shape[:3], fp), KINDS[k % len(KINDS)]) for k, a in enumerate(imgs)]
        s = sum(min(l.count, l.capacity) for l in lists)
        for budget, with_decoded in ((s, True), (s, False), (U32, True), (s // 2, True), (s - 1, False), (0, True)):
            got, want, ovf = refine_both(ctx, fast, imgs, lists, fp, TYPE_U8, TYPE_U8, metric, 4, budget, with_decoded)
            for g, w in zip(got, want):
                for x, y in zip(g, w):
                    assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8)), (budget, with_decoded)
            assert ovf == max(s - budget, 0)
    finally:
        ctx.close()
        fast.close()
    ctx, fast = contexts(gpu, PRF_HDR, PRE_THOROUGH, flags=FLG_SELF_DECOMPRESS_ONLY)
    try:
        imgs = [I.hdr_noise(90, 101, seed=6, dtype=np.float16), I.hdr_noise(31, 43, seed=7, dtype=np.float16)]
        lists = [make_list(rng, nblocks(vol(a).shape[:3], fp), kind) for a, kind in zip(imgs, ("sorted", "mixed"))]
        s = sum(min(l.count, l.capacity) for l in lists)
        for budget in (s, s // 3):
            got, want, ovf = refine_both(ctx, fast, imgs, lists, fp, TYPE_F16, TYPE_F16, metric, 3, budget)
            for g, w in zip(got, want):
                for x, y in zip(g, w):
                    assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8)), budget
            assert ovf == max(s - budget, 0)
    finally:
        ctx.close()
        fast.close()


@pytest.mark.gpu
def test_launch_counts_errors_and_null_overflow(gpu):
    """Launches: the unpacked call's over min(budget, sum of capacities) slots plus the packing; none when every capacity is 0;
    the packing alone at budget 0. Errors: the unpacked call's, in its order, then a misaligned overflow; nothing launched or
    written on error. A NULL overflow works."""
    import torch
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, 0))
    dec_only = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, FLG_DECOMPRESS_ONLY))
    radius = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, 0, a_scale_radius=2))
    buf = torch.full((1 << 17,), 0x33, dtype=torch.uint8, device="cuda")
    base = buf.data_ptr()
    data, pay, dec, mp, idx, cnt, ovf = base, base + 32768, base + 40960, base + 81920, base + 90112, base + 98304, base + 98312
    buf[cnt - base:cnt - base + 4].copy_(torch.tensor([3], dtype=torch.int32, device="cuda").view(torch.uint8))
    buf[idx - base:idx - base + 16].copy_(torch.tensor([0, 1, 2, 3], dtype=torch.int32, device="cuda").view(torch.uint8))
    l = gpu.lib()
    P, SW = gpu.ERR_BAD_PARAM, gpu.ERR_BAD_SWIZZLE
    ok = gpu.Swizzle(0, 1, 2, 3)

    def measure(c, fn):
        before = buf.cpu()
        torch.cuda.synchronize()
        n0 = c.launch_count()
        r = fn()
        torch.cuda.synchronize()
        launched = c.launch_count() - n0
        if r != 0:
            assert launched == 0 and torch.equal(buf.cpu(), before), "an error launched or wrote something"
        return r, launched

    def compress(c=ctx, n=1, lists=True, swz=ok, packed=True, budget=4, overflow=ovf, data_type=TYPE_U8, **e):
        d = dict(data=data, dim_x=40, dim_y=40, dim_z=1, payload=pay, indices=idx, count=cnt, capacity=4)
        d.update(e)
        t = (gpu.DeviceBlockList * max(n, 1))(*[gpu.DeviceBlockList(*[C.c_void_p(d[k] or None) if k not in ("dim_x", "dim_y", "dim_z", "capacity")
                                                                      else d[k] for k, _ in gpu.DeviceBlockList._fields_])] * max(n, 1))
        sw = C.byref(swz) if swz is not None else None
        if packed:
            return measure(c, lambda: l.astcenc_b200_compress_device_block_lists_packed(c.handle, t if lists else None, n, budget, C.c_void_p(overflow or None),
                                                                                         data_type, sw, None))
        return measure(c, lambda: l.astcenc_b200_compress_device_block_lists(c.handle, t if lists else None, n, data_type, sw, None))

    def refine(c=ctx, n=1, lists=True, swz=ok, dswz=ok, comps=4, metric=LOG2, data_type=TYPE_U8, decoded_type=TYPE_U8, packed=True, budget=4,
               overflow=ovf, **e):
        d = dict(data=data, dim_x=40, dim_y=40, dim_z=1, payload=pay, decoded=dec, block_error=mp, indices=idx, count=cnt, capacity=4)
        d.update(e)
        t = (gpu.DeviceRefineList * max(n, 1))(*[gpu.DeviceRefineList(*[C.c_void_p(d[k] or None) if k not in ("dim_x", "dim_y", "dim_z", "capacity")
                                                                        else d[k] for k, _ in gpu.DeviceRefineList._fields_])] * max(n, 1))
        sw, dsw = (C.byref(swz) if swz is not None else None), (C.byref(dswz) if dswz is not None else None)
        if packed:
            return measure(c, lambda: l.astcenc_b200_refine_device_block_lists_packed(c.handle, t if lists else None, n, budget, C.c_void_p(overflow or None),
                                                                                       data_type, sw, decoded_type, dsw, comps, metric, None))
        return measure(c, lambda: l.astcenc_b200_refine_device_block_lists(c.handle, t if lists else None, n, data_type, sw, decoded_type, dsw, comps, metric,
                                                                            None))

    try:
        for call in (compress, refine):
            for c in (ctx, radius):
                # the unpacked call over min(budget, sum of capacities) slots, plus the packing launch
                assert call(c=c) == (0, call(c=c, packed=False)[1] + 1)
                # (three entries: a pre-pass each with a_scale_radius)
                assert call(c=c, n=3, budget=5) == (0, call(c=c, n=1, capacity=5, packed=False)[1] + 1 + (2 if c is radius else 0))
                assert call(c=c, budget=2, overflow=0) == (0, call(c=c, capacity=2, packed=False)[1] + 1)
                assert call(c=c, budget=0) == (0, 1)
                assert call(c=c, capacity=0, indices=0, count=0) == (0, 0)
                assert call(c=c, n=0, lists=False) == (0, 0)
            assert int(buf[ovf - base:ovf - base + 4].view(torch.int32).item()) == 3      # (budget 0: all 3 listed slots over it)
            buf[ovf - base:ovf - base + 4] = 0x77
            assert call(capacity=0, indices=0, count=0) == (0, 0)
            assert int(buf[ovf - base:ovf - base + 4].view(torch.int32).item()) == 0x77777777      # (nothing written)
            assert call(budget=3)[0] == 0 and int(buf[ovf - base:ovf - base + 4].view(torch.int32).item()) == 0
            for misaligned in (ovf + 1, ovf + 2, ovf + 3):
                assert call(overflow=misaligned) == (P, 0)
                assert call(overflow=misaligned, budget=0) == (P, 0)
                assert call(overflow=misaligned, capacity=0, indices=0, count=0) == (P, 0)
            # every error of the unpacked call comes first
            assert call(c=dec_only, swz=None, overflow=ovf + 1) == (gpu.ERR_BAD_CONTEXT, 0)
            assert call(swz=None, overflow=ovf + 1) == (P, 0)
            assert call(swz=gpu.Swizzle(0, 1, 2, 7), overflow=ovf + 1) == (SW, 0)
            assert call(lists=False, overflow=ovf + 1) == (P, 0)
            for e in (dict(data=0), dict(payload=0), dict(indices=0), dict(count=0), dict(indices=idx + 2), dict(count=cnt + 1), dict(dim_x=0),
                      dict(data_type=3)):
                assert call(overflow=ovf + 1, **e) == (P, 0), e
            assert call(c=radius, dim_z=2, overflow=ovf + 1) == (gpu.ERR_NOT_IMPLEMENTED, 0)
            assert call(dim_x=6 * 2 ** 16, dim_y=6 * 2 ** 16, overflow=ovf + 1) == (P, 0)
        assert refine(dswz=None, overflow=ovf + 1) == (P, 0)
        assert refine(dswz=gpu.Swizzle(0, 1, 2, 7), overflow=ovf + 1) == (SW, 0)
        assert refine(comps=0, overflow=ovf + 1) == (P, 0)
        assert refine(metric=3, overflow=ovf + 1) == (P, 0)
        assert refine(decoded_type=5, overflow=ovf + 1) == (P, 0)
        assert refine(block_error=0, overflow=ovf + 1) == (P, 0)
        assert refine(decoded=dec + 2, overflow=ovf + 1) == (P, 0)
        with pytest.raises(gpu.AstcencError) as e:
            ctx.refine_device_block_lists_packed([], 4, TYPE_U8, TYPE_U8, 7)
        assert e.value.code == P
    finally:
        ctx.close()
        dec_only.close()
        radius.close()


@pytest.mark.gpu
def test_gated_loop_with_packed_refine_equals_unpacked(gpu):
    """The mixed 64-texture set: three rounds of total_block_maps -> select_blocks_pooled (threshold 0, K = 2 % of the set's
    blocks) -> refine, all enqueued on one stream up front, with refine_device_block_lists_packed (budget K) and with the unpacked
    call: the same payloads, decodes and maps after every round; the packed rounds' overflow is 0."""
    import torch
    from test_map_totals import Ladder, mixed_set
    imgs = mixed_set()
    rounds = 3
    ladders = [Ladder(gpu, imgs, PRF_LDR, gpu.BLOCK_SQUARED_ERROR, 4) for _ in range(2)]
    try:
        st = torch.cuda.Stream()
        s = st.cuda_stream
        N = len(imgs)
        nb = ladders[0].nb
        K = max(1, int(sum(nb) * 0.02))
        for lad in ladders:
            lad.start(s)
        st.synchronize()
        t0 = np.array([float(m.double().sum().item()) for m in ladders[0].map])
        limits = [t * f for t, f in zip(t0, np.resize([1.01, 0.999, 0.99, 0.9, 0.5], N))]      # (some met, some just missed, some far)
        ovf = torch.full((rounds,), -1, dtype=torch.int32, device="cuda")
        outs = []
        for packed, lad in zip((False, True), ladders):
            d_t = torch.zeros((rounds, N), dtype=torch.float64, device="cuda")
            d_w = torch.zeros((rounds, N), dtype=torch.float32, device="cuda")
            d_cnt = torch.zeros((rounds, N), dtype=torch.int32, device="cuda")
            d_idx = [[torch.zeros(min(K, n), dtype=torch.int32, device="cuda") for n in nb] for _ in range(rounds)]
            snaps = []
            for r in range(rounds):
                lad.totals(limits, d_t[r], d_w[r], s)
                lad.fast.select_blocks_pooled([(N, 0.0, K)], [(m.data_ptr(), n, d_w[r].data_ptr() + 4 * k, ix.data_ptr(), d_cnt[r].data_ptr() + 4 * k)
                                                              for k, (m, n, ix) in enumerate(zip(lad.map, nb, d_idx[r]))], stream=s)
                table = [(d.data_ptr(), w, h, 1, p.data_ptr(), o.data_ptr(), m.data_ptr(), ix.data_ptr(), d_cnt[r].data_ptr() + 4 * k, ix.numel())
                         for k, (d, (w, h), p, o, m, ix) in enumerate(zip(lad.d_img, lad.dims, lad.pay, lad.dec, lad.map, d_idx[r]))]
                if packed:
                    lad.thorough.refine_device_block_lists_packed(table, K, lad.dt, lad.dt, lad.metric, input_components=4, overflow=ovf.data_ptr() + 4 * r,
                                                                  stream=s)
                else:
                    lad.thorough.refine_device_block_lists(table, lad.dt, lad.dt, lad.metric, input_components=4, stream=s)
                with torch.cuda.stream(st):
                    snaps.append([torch.cat([p, o, m.view(torch.uint8)]) for p, o, m in zip(lad.pay, lad.dec, lad.map)])
            outs.append((snaps, d_cnt))
        st.synchronize()
        for r in range(rounds):
            for j in range(N):
                assert torch.equal(outs[0][0][r][j], outs[1][0][r][j]), (r, j)
        assert torch.equal(outs[0][1], outs[1][1])
        cnt = outs[0][1].cpu().numpy()
        assert np.sum(cnt) > 0 and np.any(cnt[0] == 0)
        assert ovf.cpu().tolist() == [0] * rounds
    finally:
        for lad in ladders:
            lad.close()
