"""List refreshes: astcenc_b200_decompress_device_block_lists decodes the listed blocks of device payloads into device images
(astc_decompress_block_lists_kernel; the walk is decode_list_blocks in astc_dev_gather.cuh), and
astcenc_b200_compute_block_errors_device_block_lists refreshes per-block error maps at the listed blocks
(astc_block_error_lists_kernel; block_error_list_slot and plan_block_error_lists in astc_dev_metrics.cuh).

CPU: both walks compiled for the host (tests/hostsim/hostsim_decode_lists.cpp and hostsim_map_lists.cpp, one lane and 32 lanes)
over whole tables: the listed blocks against the oracle's decode of the whole image and against hostsim_block_error's whole map,
poison everywhere else; and the planner's slots and refusals.
GPU: list decodes against decompress_device_images of the whole payload, guard bytes everywhere else; list maps against whole
maps; an iterated select / re-encode / re-decode / re-measure loop on one stream; launch counts and both error orders."""
import ctypes as C

import numpy as np
import pytest

from astc_ref import *  # noqa: F401,F403
from hostsim_build import host_sim
from test_decode_device import NP, SIM_CASES, block_pool, nblocks, oracle_decode, payloads_for
from test_metrics_device import DT, metrics_sim, random_pair, sim_map
import astc_images as I

POISON = 0xA5
MAP_POISON = np.uint32(0x7FA5A5A5)      # (a NaN no map value is: compared bit for bit)
S = FLG_SELF_DECOMPRESS_ONLY

_SIMS = {}


def lists_sim(name, lanes32=False):
    """tests/hostsim/<name>.cpp compiled for the host (one simulated lane, or 32 lanes on 32 threads)."""
    key = (name, lanes32)
    if key in _SIMS:
        return _SIMS[key]
    lib = host_sim(name, lanes32)
    if name == "hostsim_decode_lists":
        lib.hostsim_decompress_block_lists.argtypes = [C.c_int, C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_int,
                                                       C.POINTER(C.c_int), C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
    else:
        lib.hostsim_plan_block_error_lists.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.hostsim_block_error_lists.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_uint, C.c_uint,
                                                  C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    _SIMS[key] = lib
    return lib


class BlockList:
    """A device list's contents: indices (garbage past the count included), its count and capacity."""

    def __init__(self, idx, count, capacity):
        self.idx = np.ascontiguousarray(np.asarray(idx, np.uint32).reshape(-1)[:capacity])
        self.count = count
        self.capacity = capacity

    def listed(self, blocks):
        """The blocks the list stands for: its first min(count, capacity) indices that lie in the image."""
        s = self.idx[:min(self.count, self.capacity)]
        return s[s < blocks]

    def padded(self):
        """The indices with one spare word, so that a list of capacity 0 still has an address."""
        return np.concatenate([self.idx, np.zeros(1, np.uint32)])


def make_list(rng, n, kind):
    """A list over an image of n blocks. kind: "mixed" (unsorted, duplicates, indices out of range, count > capacity), "past"
    (valid blocks past the count: garbage that must not be read), "sorted" (what select_blocks writes), "empty" (count 0),
    "none" (capacity 0)."""
    if kind == "mixed":
        cap = max(4, n // 2)
        idx = rng.integers(0, n, cap).astype(np.uint32)
        idx[1] = idx[0]
        idx[2] = n
        idx[3] = 0xFFFFFFFF
        return BlockList(idx, cap + 5, cap)
    if kind == "past":
        cap = min(n, 6) + 2
        return BlockList(rng.integers(0, n, cap), 2, cap)
    if kind == "sorted":
        idx = np.sort(rng.choice(n, max(1, n // 3), replace=False))
        return BlockList(idx, len(idx), len(idx))
    if kind == "empty":
        return BlockList(rng.integers(0, n, 4), 0, 4)
    return BlockList(np.zeros(0), 3, 0)


KINDS = ("mixed", "past", "sorted", "empty", "none")


def block_texels(shape, fp, blocks):
    """(D, H, W) mask of the texels of the listed blocks' footprints that lie inside the image."""
    d, h, w = shape
    bxs, bys = -(-w // fp[0]), -(-h // fp[1])
    m = np.zeros(shape, bool)
    for b in np.unique(blocks):
        b = int(b)
        col, rest = b % bxs, b // bxs
        row, layer = rest % bys, rest // bys
        z0 = layer * fp[2]
        m[z0:z0 + fp[2], row * fp[1]:(row + 1) * fp[1], col * fp[0]:(col + 1) * fp[0]] = True
    return m


def expected_decode(full, shape, fp, lst, poison_bytes):
    """The list decode of an image whose whole decode is `full`: its texels at the listed blocks, `poison_bytes` elsewhere."""
    m = block_texels(shape, fp, lst.listed(nblocks(shape, fp)))
    out = poison_bytes.copy().reshape(shape + (-1,))
    out[m] = full.view(np.uint8).reshape(shape + (-1,))[m]
    return out.reshape(-1)


# ---------------------------------------------------------------------------------------------------------------------------
# CPU: the decode walk
# ---------------------------------------------------------------------------------------------------------------------------
def sim_decode_lists(lib, payloads, shapes, lists, fp, profile, out_type, swz, share):
    outs = [np.full(int(np.prod(s)) * 4 * np.dtype(NP[out_type]).itemsize, POISON, np.uint8) for s in shapes]
    pays = (C.c_void_p * len(payloads))(*[p.ctypes.data for p in payloads])
    optr = (C.c_void_p * len(outs))(*[o.ctypes.data for o in outs])
    dims = np.array([[s[2], s[1], s[0]] for s in shapes], np.uint32).reshape(-1)
    padded = [l.padded() for l in lists]
    iptr = (C.c_void_p * len(lists))(*[p.ctypes.data for p in padded])
    counts = np.array([l.count for l in lists], np.uint32)
    caps = np.array([l.capacity for l in lists], np.uint32)
    assert lib.hostsim_decompress_block_lists(profile, fp[0], fp[1], fp[2], 0, pays, optr, dims.ctypes.data, len(shapes), out_type, (C.c_int * 4)(*swz),
                                              iptr, counts.ctypes.data, caps.ctypes.data, share) == 0
    return outs


@pytest.mark.parametrize("lanes32", [False, True], ids=["lanes1", "lanes32"])
@pytest.mark.parametrize("case", SIM_CASES, ids=[c[0] for c in SIM_CASES])
def test_hostsim_list_walk_decodes_listed_blocks_only(case, lanes32, oracle, golden):
    """Every listed block of every entry equals the oracle's decode of the whole image at its texels, every other byte keeps its
    poison: garbage past the count, count > capacity, count 0, capacity 0, indices out of range, duplicates, unsorted and sorted
    lists, edge blocks, a texture array, volumes and a 1 x 1 image; one CTA over the whole call, and shares of 7 slots and of 1
    that split entries and planes."""
    _, fp, shapes, profile, out_type, swz = case
    lib = lists_sim("hostsim_decode_lists", lanes32)
    pool = block_pool(fp, golden, 3)
    if lanes32:
        pool = pool[::7]      # (the 32-lane simulation is slow: a sample of the set)
    cols = 48
    rows = -(-len(pool) // (cols * (2 if fp[2] > 1 else 1)))
    shapes = shapes[:2] + [((2 * fp[2] if fp[2] > 1 else 1), rows * fp[1] - 1, cols * fp[0] - 1)] + shapes[2:]
    payloads = payloads_for(shapes, fp, pool)
    full = [oracle_decode(oracle, p, s, fp, profile, out_type, swz) for p, s in zip(payloads, shapes)]
    rng = np.random.default_rng(17)
    kinds = ["mixed", "past", "sorted"] + [KINDS[k % len(KINDS)] for k in range(len(shapes) - 3)]
    lists = [make_list(rng, nblocks(s, fp), k) for s, k in zip(shapes, kinds)]
    total = sum(l.capacity for l in lists)
    for share in (total, 7, 1):
        got = sim_decode_lists(lib, payloads, shapes, lists, fp, profile, out_type, swz, share)
        for k, (g, f, s, l) in enumerate(zip(got, full, shapes, lists)):
            want = expected_decode(f, s, fp, l, np.full(g.size, POISON, np.uint8))
            assert np.array_equal(g, want), "image %d %s (%s list), share %d" % (k, s, kinds[k], share)


# ---------------------------------------------------------------------------------------------------------------------------
# CPU: the map walk and its planner
# ---------------------------------------------------------------------------------------------------------------------------
def list_plan(shapes, caps, fp):
    lib = lists_sim("hostsim_map_lists")
    n = len(shapes)
    dims = np.array([[s[2], s[1], s[0]] for s in shapes], np.uint32).reshape(-1)
    caps = np.asarray(caps, np.uint32)
    first = np.zeros(n, np.uint64)
    bxy = np.zeros(2 * n, np.uint32)
    totals = np.zeros(2, np.uint64)
    if lib.hostsim_plan_block_error_lists(dims.ctypes.data, caps.ctypes.data, n, fp[0], fp[1], fp[2], first.ctypes.data, bxy.ctypes.data, totals.ctypes.data):
        return None
    return dict(first=first.tolist(), blocks=bxy.reshape(-1, 2).tolist(), slots=int(totals[0]), grid=int(totals[1]))


def test_list_planner_slots_and_refusals():
    """Entry j's slots start at the prefix of the capacities (capacity 0 included), the grid is one CTA per 8 slots, and a call
    is refused for an image of 2^32 blocks or more (whatever its capacity) or a grid beyond 2^31 - 1 CTAs."""
    shapes = [(1, 45, 67), (4, 13, 17), (1, 1, 1), (9, 21, 19)]
    caps = [5, 0, 300, 17]
    for fp in ((6, 6, 1), (4, 4, 4)):
        p = list_plan(shapes, caps, fp)
        assert p["first"] == [0, 5, 5, 305] and p["slots"] == 322 and p["grid"] == 41
        assert p["blocks"] == [[-(-w // fp[0]), -(-h // fp[1])] for _, h, w in shapes]
    assert list_plan([], [], (4, 4, 1)) == dict(first=[], blocks=[], slots=0, grid=0)
    assert list_plan([(1, 2 ** 18, 2 ** 18)], [0], (4, 4, 1)) is None      # (2^32 blocks)
    assert list_plan([(1, 2 ** 18, 2 ** 18 - 4)], [0], (4, 4, 1)) is not None
    big = 2 ** 32 - 1
    assert list_plan([(1, 1, 1)] * 3, [big] * 3, (4, 4, 1)) is not None     # (3 * (2^32 - 1) slots: 1.6e9 CTAs)
    assert list_plan([(1, 1, 1)] * 5, [big] * 5, (4, 4, 1)) is None         # (2.7e9 CTAs)


def sim_map_lists(lib, pairs, fp, components, lists, maps):
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
    assert lib.hostsim_block_error_lists(o, ot.ctypes.data, d, dt.ctypes.data, dims.ctypes.data, n, fp[0], fp[1], fp[2], components, mp, ip,
                                         counts.ctypes.data, caps.ctypes.data) == 0


MAP_CASES = [((6, 6, 1), [(1, 37, 29), (3, 13, 17), (1, 1, 1), (1, 12, 18), (2, 1, 1)]), ((4, 4, 4), [(5, 7, 9), (1, 1, 1), (8, 8, 4), (9, 3, 13)])]


@pytest.mark.parametrize("lanes32", [False, True], ids=["lanes1", "lanes32"])
@pytest.mark.parametrize("fp,shapes", MAP_CASES, ids=["6x6", "4x4x4"])
def test_hostsim_list_maps_equal_whole_maps_at_listed_blocks(fp, shapes, lanes32):
    """Listed values equal hostsim_block_error's whole map bit for bit; every other value keeps its poison. Mixed types, every
    list kind, one table."""
    lib = lists_sim("hostsim_map_lists", lanes32)
    whole_lib = metrics_sim()
    rng = np.random.default_rng(23)
    types = [(TYPE_U8, TYPE_U8), (TYPE_F16, TYPE_F16), (TYPE_F32, TYPE_U8), (TYPE_U8, TYPE_F16), (TYPE_F16, TYPE_F32)]
    pairs = [random_pair(rng, s, *types[k % len(types)]) for k, s in enumerate(shapes)]
    kinds = [KINDS[k % len(KINDS)] for k in range(len(shapes))]
    lists = [make_list(rng, nblocks(s, fp), k) for s, k in zip(shapes, kinds)]
    for components in ((1, 2, 3, 4) if not lanes32 else (4,)):
        maps = [np.full(nblocks(s, fp), MAP_POISON, np.uint32).view(np.float32) for s in shapes]
        sim_map_lists(lib, pairs, fp, components, lists, maps)
        for k, ((a, b), s, l, m) in enumerate(zip(pairs, shapes, lists, maps)):
            want = np.full(nblocks(s, fp), MAP_POISON, np.uint32)
            listed = l.listed(len(want))
            want[listed] = sim_map(whole_lib, a, b, fp, components).view(np.uint32)[listed]
            assert np.array_equal(m.view(np.uint32), want), "pair %d %s (%s list), components %d" % (k, s, kinds[k], components)


# ---------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------
GAP = 37


@pytest.fixture(scope="module")
def gpu(pkg):
    import torch
    assert torch.cuda.is_available(), "the GPU tests need a CUDA device"
    torch.cuda.set_device(0)
    return pkg


def out_bytes(shape, out_type):
    return int(np.prod(shape)) * 4 * np.dtype(NP[out_type]).itemsize


def layout(shapes, out_type, odd):
    align = 1 if odd else np.dtype(NP[out_type]).itemsize
    offs, pos = [], GAP
    for s in shapes:
        pos = -(-pos // align) * align
        if odd and pos % 2 == 0:
            pos += 1
        offs.append(pos)
        pos += out_bytes(s, out_type) + GAP
    return offs, pos


class DecodeCall:
    """Payloads, shapes and lists on the device: the whole decodes (decompress_device_images, one call) and list decodes into
    one guard-filled allocation."""

    def __init__(self, payloads, shapes, lists, out_type, odd=False):
        import torch
        self.dev = torch.device("cuda", 0)
        self.shapes, self.lists, self.out_type = shapes, lists, out_type
        self.d_pay = [torch.from_numpy(p).to(self.dev) for p in payloads]
        self.d_idx = [torch.from_numpy(l.padded().view(np.int32)).to(self.dev) for l in lists]
        self.d_cnt = torch.from_numpy(np.array([l.count for l in lists] + [0], np.uint32).view(np.int32)).to(self.dev)
        self.offs, self.total = layout(shapes, out_type, odd)
        self.guard = np.random.default_rng(len(shapes)).integers(0, 256, self.total, dtype=np.uint8)

    def whole(self, ctx, swizzle):
        import torch
        d_full = [torch.zeros(out_bytes(s, self.out_type), dtype=torch.uint8, device=self.dev) for s in self.shapes]
        ctx.decompress_device_images([(p.data_ptr(), f.data_ptr(), s[2], s[1], s[0]) for p, f, s in zip(self.d_pay, d_full, self.shapes)], self.out_type,
                                     swizzle=swizzle)
        torch.cuda.synchronize()
        return [f.cpu().numpy() for f in d_full]

    def entry(self, k, base):
        s = self.shapes[k]
        return (self.d_pay[k].data_ptr(), base + self.offs[k], s[2], s[1], s[0], self.d_idx[k].data_ptr(), self.d_cnt.data_ptr() + 4 * k,
                self.lists[k].capacity)

    def lists_decode(self, ctx, swizzle, order=None, one_call=True, stream=None):
        """The list decode (one call in `order`, or one call per entry) into the guard-filled allocation; each call is one launch,
        none when its capacities are all zero. Returns the allocation's bytes."""
        import torch
        d_out = torch.from_numpy(self.guard.copy()).to(self.dev)
        base = d_out.data_ptr()
        order = list(range(len(self.shapes))) if order is None else order
        calls = [order] if one_call else [[k] for k in order]
        st = stream or torch.cuda.Stream(device=self.dev)
        torch.cuda.synchronize()
        for c in calls:
            n0 = ctx.launch_count()
            ctx.decompress_device_block_lists([self.entry(k, base) for k in c], self.out_type, swizzle=swizzle, stream=st.cuda_stream)
            assert ctx.launch_count() == n0 + (1 if any(self.lists[k].capacity for k in c) else 0)
        torch.cuda.synchronize()
        return d_out.cpu().numpy()

    def expected(self, full, fp):
        want = self.guard.copy()
        for s, o, f, l in zip(self.shapes, self.offs, full, self.lists):
            n = out_bytes(s, self.out_type)
            want[o:o + n] = expected_decode(f, s, fp, l, self.guard[o:o + n])
        return want


def check_decode(ctx, fp, payloads, shapes, lists, out_type, swizzle, odd=False, shuffled=False):
    call = DecodeCall(payloads, shapes, lists, out_type, odd)
    want = call.expected(call.whole(ctx, swizzle), fp)
    assert np.array_equal(call.lists_decode(ctx, swizzle), want)
    assert np.array_equal(call.lists_decode(ctx, swizzle, one_call=False), want)
    if shuffled:
        order = [int(k) for k in np.random.default_rng(3).permutation(len(shapes))]
        assert np.array_equal(call.lists_decode(ctx, swizzle, order=order), want)


SHAPES_2D = [(1, 37, 29), (1, 1, 1), (3, 13, 17), (1, 64, 64), (1, 5, 61), (2, 7, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("profile", (PRF_LDR, PRF_HDR))
def test_list_decode_equals_whole_decode_at_listed_blocks(profile, gpu, golden):
    """Alone (one call per entry), in one call and inside a shuffled 40-entry table: every listed block's texels equal
    decompress_device_images of the whole payload, every other byte keeps its guard; U8, F16 and F32 with a Z swizzle."""
    fp = (6, 6, 1)
    rng = np.random.default_rng(5)
    shapes = [SHAPES_2D[k % len(SHAPES_2D)] for k in range(40)]
    payloads = payloads_for(shapes, fp, block_pool(fp, golden, 7))
    lists = [make_list(rng, nblocks(s, fp), KINDS[k % len(KINDS)]) for k, s in enumerate(shapes)]
    ctx = gpu.Context(gpu.config_init(profile, 6, 6, PRE_MEDIUM, 0))
    try:
        for t in (TYPE_U8, TYPE_F16, TYPE_F32):
            check_decode(ctx, fp, payloads, shapes, lists, t, (0, 3, 6, 5), shuffled=True)
    finally:
        ctx.close()


@pytest.mark.gpu
def test_list_decode_at_odd_offsets_on_volumes_and_decompress_only_contexts(gpu, golden):
    """Outputs at odd byte offsets; volumes of a 3D footprint; a decompress-only context."""
    rng = np.random.default_rng(9)
    fp = (6, 6, 1)
    payloads = payloads_for(SHAPES_2D, fp, block_pool(fp, golden, 9))
    lists = [make_list(rng, nblocks(s, fp), KINDS[k % len(KINDS)]) for k, s in enumerate(SHAPES_2D)]
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_MEDIUM, 0))
    try:
        for t in (TYPE_U8, TYPE_F16, TYPE_F32):
            check_decode(ctx, fp, payloads, SHAPES_2D, lists, t, (0, 3, 6, 5), odd=True)
    finally:
        ctx.close()
    fp3 = (4, 4, 4)
    shapes3 = [(5, 7, 9), (1, 1, 1), (4, 4, 4), (9, 3, 13), (12, 20, 24)]
    payloads3 = payloads_for(shapes3, fp3, block_pool(fp3, golden, 4))
    lists3 = [make_list(rng, nblocks(s, fp3), k) for s, k in zip(shapes3, ("past", "mixed", "none", "empty", "sorted"))]
    for flags in (0, FLG_DECOMPRESS_ONLY):
        ctx = gpu.Context(gpu.config_init(PRF_HDR_RGB_LDR_A, 4, 4, PRE_MEDIUM, flags, block_z=4))
        try:
            check_decode(ctx, fp3, payloads3, shapes3, lists3, TYPE_F32, (3, 6, 1, 0))
            check_decode(ctx, fp3, payloads3, shapes3, lists3, TYPE_U8, (0, 1, 2, 3))
        finally:
            ctx.close()
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_MEDIUM, FLG_DECOMPRESS_ONLY))
    try:
        check_decode(ctx, fp, payloads, SHAPES_2D, lists, TYPE_F16, (0, 3, 6, 5))
    finally:
        ctx.close()


@pytest.mark.gpu
def test_list_maps_equal_whole_maps_at_listed_blocks(gpu):
    """Mixed types, a texture array, a volume of a 3D footprint, every list kind, alone and in one call: listed values equal the
    whole map of compute_error_metrics_device_images bit for bit, every other value keeps its poison; a decompress-only context."""
    import torch
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(31)
    types = [(TYPE_U8, TYPE_U8), (TYPE_F16, TYPE_F16), (TYPE_F32, TYPE_U8), (TYPE_U8, TYPE_F16), (TYPE_F16, TYPE_F32)]
    mb = C.sizeof(gpu.ErrorMetrics)
    for fp, shapes in MAP_CASES + [((6, 6, 1), [(1, 300, 257), (2, 64, 64)] * 4)]:
        ctx = gpu.Context(gpu.config_init(PRF_LDR, fp[0], fp[1], PRE_FAST, FLG_DECOMPRESS_ONLY, block_z=fp[2]))
        try:
            pairs = [random_pair(rng, s, *types[k % len(types)]) for k, s in enumerate(shapes)]
            lists = [make_list(rng, nblocks(s, fp), KINDS[k % len(KINDS)]) for k, s in enumerate(shapes)]
            d_a = [torch.from_numpy(a.reshape(-1).view(np.uint8)).to(dev) for a, _ in pairs]
            d_b = [torch.from_numpy(b.reshape(-1).view(np.uint8)).to(dev) for _, b in pairs]
            d_idx = [torch.from_numpy(l.padded().view(np.int32)).to(dev) for l in lists]
            d_cnt = torch.from_numpy(np.array([l.count for l in lists] + [0], np.uint32).view(np.int32)).to(dev)
            d_met = torch.zeros(len(shapes) * mb, dtype=torch.uint8, device=dev)
            for components in (1, 2, 4):
                whole = [torch.zeros(nblocks(s, fp), dtype=torch.float32, device=dev) for s in shapes]
                ctx.compute_error_metrics_device_images([(a.data_ptr(), b.data_ptr(), DT[p[0].dtype], DT[p[1].dtype], s[2], s[1], s[0], d_met.data_ptr() + k * mb,
                                                          w.data_ptr()) for k, (a, b, p, s, w) in enumerate(zip(d_a, d_b, pairs, shapes, whole))],
                                                        input_components=components)
                torch.cuda.synchronize()
                want = []
                for w, s, l in zip(whole, shapes, lists):
                    v = np.full(nblocks(s, fp), MAP_POISON, np.uint32)
                    listed = l.listed(len(v))
                    v[listed] = w.cpu().numpy().view(np.uint32)[listed]
                    want.append(v)
                entries = lambda maps, ks: [(d_a[k].data_ptr(), d_b[k].data_ptr(), DT[pairs[k][0].dtype], DT[pairs[k][1].dtype], shapes[k][2], shapes[k][1],
                                             shapes[k][0], maps[k].data_ptr(), d_idx[k].data_ptr(), d_cnt.data_ptr() + 4 * k, lists[k].capacity) for k in ks]
                for one_call in (True, False):
                    maps = [torch.from_numpy(np.full(nblocks(s, fp), MAP_POISON, np.uint32).view(np.int32)).to(dev) for s in shapes]
                    torch.cuda.synchronize()
                    calls = [[int(k) for k in rng.permutation(len(shapes))]] if one_call else [[k] for k in range(len(shapes))]
                    for c in calls:
                        n0 = ctx.launch_count()
                        ctx.compute_block_errors_device_block_lists(entries(maps, c), input_components=components)
                        assert ctx.launch_count() == n0 + (1 if any(lists[k].capacity for k in c) else 0)
                    torch.cuda.synchronize()
                    for k, (m, v) in enumerate(zip(maps, want)):
                        assert np.array_equal(m.cpu().numpy().view(np.uint32), v), (fp, k, shapes[k], components, one_call)
        finally:
            ctx.close()


@pytest.mark.gpu
def test_iterated_refine_loop_on_one_stream(gpu):
    """-fast, then two rounds of select -> compress_device_block_lists -> list decode -> list map (-medium on the worst 10 %, then
    -thorough on the worst 1 %), enqueued on one stream with one synchronise at the end. The decoded images equal
    decompress_device_images of the final payloads, and the maps equal whole maps of those pairs, bit for bit."""
    import torch
    dev = torch.device("cuda", 0)
    fp = (6, 6, 1)
    ctxs = {q: gpu.Context(gpu.config_init(PRF_LDR, 6, 6, q, S)) for q in (PRE_FAST, PRE_MEDIUM, PRE_THOROUGH)}
    fast = ctxs[PRE_FAST]
    try:
        imgs = [I.photo_like(h, w, seed=90 + k) for k, (h, w) in enumerate([(256, 256), (200, 311), (128, 96), (97, 143)])]
        nb = [nblocks((1,) + im.shape[:2], fp) for im in imgs]
        dims = [(im.shape[1], im.shape[0]) for im in imgs]
        d_img = [torch.from_numpy(im.reshape(-1)).to(dev) for im in imgs]
        d_pay = [torch.zeros(n * 16, dtype=torch.uint8, device=dev) for n in nb]
        d_dec = [torch.zeros(im.size, dtype=torch.uint8, device=dev) for im in imgs]
        mb = C.sizeof(gpu.ErrorMetrics)
        d_met = torch.zeros(len(imgs) * mb, dtype=torch.uint8, device=dev)
        d_map = [torch.zeros(n, dtype=torch.float32, device=dev) for n in nb]
        d_idx = [torch.zeros(n, dtype=torch.int32, device=dev) for n in nb]
        d_cnt = torch.zeros(len(imgs), dtype=torch.int32, device=dev)
        st = torch.cuda.Stream(device=dev)
        torch.cuda.synchronize()
        s = st.cuda_stream
        fast.compress_device_images([(d.data_ptr(), w, h, 1, p.data_ptr()) for d, (w, h), p in zip(d_img, dims, d_pay)], TYPE_U8, stream=s)
        fast.decompress_device_images([(p.data_ptr(), o.data_ptr(), w, h, 1) for p, o, (w, h) in zip(d_pay, d_dec, dims)], TYPE_U8, stream=s)
        fast.compute_error_metrics_device_images([(d.data_ptr(), o.data_ptr(), TYPE_U8, TYPE_U8, w, h, 1, d_met.data_ptr() + k * mb, m.data_ptr())
                                                  for k, (d, o, (w, h), m) in enumerate(zip(d_img, d_dec, dims, d_map))], input_components=4, stream=s)
        for q, share in ((PRE_MEDIUM, 10), (PRE_THOROUGH, 100)):
            caps = [max(1, n // share) for n in nb]
            fast.select_blocks([(m.data_ptr(), n, -np.inf, c, ix.data_ptr(), d_cnt.data_ptr() + 4 * k)
                                for k, (m, n, c, ix) in enumerate(zip(d_map, nb, caps, d_idx))], stream=s)
            ctxs[q].compress_device_block_lists([(d.data_ptr(), w, h, 1, p.data_ptr(), ix.data_ptr(), d_cnt.data_ptr() + 4 * k, c)
                                                 for k, (d, (w, h), p, ix, c) in enumerate(zip(d_img, dims, d_pay, d_idx, caps))], TYPE_U8, stream=s)
            fast.decompress_device_block_lists([(p.data_ptr(), o.data_ptr(), w, h, 1, ix.data_ptr(), d_cnt.data_ptr() + 4 * k, c)
                                                for k, (p, o, (w, h), ix, c) in enumerate(zip(d_pay, d_dec, dims, d_idx, caps))], TYPE_U8, stream=s)
            fast.compute_block_errors_device_block_lists([(d.data_ptr(), o.data_ptr(), TYPE_U8, TYPE_U8, w, h, 1, m.data_ptr(), ix.data_ptr(),
                                                           d_cnt.data_ptr() + 4 * k, c)
                                                          for k, (d, o, (w, h), m, ix, c) in enumerate(zip(d_img, d_dec, dims, d_map, d_idx, caps))],
                                                         input_components=4, stream=s)
        st.synchronize()
        assert np.array_equal(d_cnt.cpu().numpy(), [max(1, n // 100) for n in nb])
        want_dec = [torch.zeros_like(o) for o in d_dec]
        want_map = [torch.zeros_like(m) for m in d_map]
        fast.decompress_device_images([(p.data_ptr(), o.data_ptr(), w, h, 1) for p, o, (w, h) in zip(d_pay, want_dec, dims)], TYPE_U8)
        fast.compute_error_metrics_device_images([(d.data_ptr(), o.data_ptr(), TYPE_U8, TYPE_U8, w, h, 1, d_met.data_ptr() + k * mb, m.data_ptr())
                                                  for k, (d, o, (w, h), m) in enumerate(zip(d_img, want_dec, dims, want_map))], input_components=4)
        torch.cuda.synchronize()
        for k in range(len(imgs)):
            assert np.array_equal(d_dec[k].cpu().numpy(), want_dec[k].cpu().numpy()), k
            assert np.array_equal(d_map[k].cpu().numpy().view(np.uint32), want_map[k].cpu().numpy().view(np.uint32)), k
        # the rounds changed blocks: the loop did not refresh a payload that stayed the -fast one
        fast_pay = fast.compress_image(imgs[0])
        assert not np.array_equal(d_pay[0].cpu().numpy(), fast_pay)
    finally:
        for c in ctxs.values():
            c.close()


@pytest.mark.gpu
def test_list_decode_errors_follow_the_documented_order(gpu):
    import torch
    dev = torch.device("cuda", 0)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, FLG_DECOMPRESS_ONLY))
    d_pay = torch.zeros(4096, dtype=torch.uint8, device=dev)
    d_idx = torch.zeros(64, dtype=torch.int32, device=dev)
    d_cnt = torch.full((4,), 3, dtype=torch.int32, device=dev)
    nbytes = 65536
    d_out = torch.full((nbytes,), POISON, dtype=torch.uint8, device=dev)
    l = gpu.lib()
    sw = gpu.Swizzle(0, 1, 2, 3)
    E = dict(payload=d_pay.data_ptr(), data=d_out.data_ptr(), dim_x=44, dim_y=40, dim_z=1, indices=d_idx.data_ptr(), count=d_cnt.data_ptr(), capacity=8)
    F = ("payload", "data", "dim_x", "dim_y", "dim_z", "indices", "count", "capacity")

    def table(**edit):
        d = dict(E, **edit)
        e2 = dict(E, payload=d_pay.data_ptr() + 2048, data=d_out.data_ptr() + 32768, dim_x=13, dim_y=12, dim_z=2, count=d_cnt.data_ptr() + 4)
        return [tuple(d[f] for f in F), tuple(e2[f] for f in F)]

    def _raise(err):
        if err:
            raise gpu.AstcencError(err, "call")

    def expect(code, lists=None, data_type=TYPE_U8, swizzle=(0, 1, 2, 3), raw=None, launches=0):
        torch.cuda.synchronize()
        n0 = ctx.launch_count()
        call = raw or (lambda: ctx.decompress_device_block_lists(table() if lists is None else lists, data_type, swizzle=swizzle))
        if code == 0:
            call()
        else:
            with pytest.raises(gpu.AstcencError) as e:
                call()
            assert e.value.code == code, (e.value.code, code)
        torch.cuda.synchronize()
        assert ctx.launch_count() == n0 + launches
        if launches == 0:
            assert np.all(d_out.cpu().numpy() == POISON)

    P = gpu.ERR_BAD_PARAM
    try:
        expect(P, swizzle=None)
        expect(P, swizzle=None, lists=table(data=0))                          # (a NULL swizzle comes first)
        expect(gpu.ERR_BAD_SWIZZLE, swizzle=(0, 1, 2, 7))
        expect(gpu.ERR_BAD_SWIZZLE, swizzle=(0, 1, 2, 7), lists=table(payload=0))
        expect(P, raw=lambda: _raise(l.astcenc_b200_decompress_device_block_lists(ctx.handle, None, 2, TYPE_U8, C.byref(sw), None)))
        for edit in (dict(payload=0), dict(data=0), dict(indices=0), dict(count=0), dict(indices=d_idx.data_ptr() + 2), dict(count=d_cnt.data_ptr() + 1),
                     dict(dim_x=0), dict(dim_y=0), dict(dim_z=0), dict(dim_x=2 ** 32 - 1, dim_y=2 ** 32 - 1, dim_z=2 ** 32 - 1)):
            expect(P, lists=table(**edit))
            expect(P, lists=table(**edit), data_type=3)
        expect(P, data_type=3)
        expect(P, data_type=3, lists=table(dim_x=6 * 2 ** 16, dim_y=6 * 2 ** 16))      # (the data type before the block count)
        expect(P, lists=table(dim_x=6 * 2 ** 16, dim_y=6 * 2 ** 16))                   # (2^32 blocks)
        expect(P, lists=table(dim_x=6 * 2 ** 16, dim_y=6 * 2 ** 16, capacity=0, indices=0, count=0))
        # capacity 0: NULL lists are allowed, and nothing runs
        expect(0, lists=[t[:5] + (0, 0, 0) for t in table()])
        expect(0, lists=[])
        expect(0, raw=lambda: _raise(l.astcenc_b200_decompress_device_block_lists(ctx.handle, None, 0, TYPE_U8, C.byref(sw), None)))
        expect(0, lists=[table()[0][:5] + (0, 0, 0), table()[1]], launches=1)
    finally:
        ctx.close()


@pytest.mark.gpu
def test_list_map_errors_follow_the_documented_order(gpu):
    import torch
    dev = torch.device("cuda", 0)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, FLG_DECOMPRESS_ONLY))
    d_img = torch.zeros(65536, dtype=torch.uint8, device=dev)
    d_idx = torch.zeros(64, dtype=torch.int32, device=dev)
    d_cnt = torch.full((4,), 3, dtype=torch.int32, device=dev)
    d_map = torch.from_numpy(np.full(4096, MAP_POISON, np.uint32).view(np.int32)).to(dev)
    l = gpu.lib()
    F = ("original", "decoded", "original_type", "decoded_type", "dim_x", "dim_y", "dim_z", "block_error", "indices", "count", "capacity")
    E = dict(original=d_img.data_ptr(), decoded=d_img.data_ptr() + 32768, original_type=TYPE_U8, decoded_type=TYPE_F16, dim_x=44, dim_y=40, dim_z=1,
             block_error=d_map.data_ptr(), indices=d_idx.data_ptr(), count=d_cnt.data_ptr(), capacity=8)

    def table(**edit):
        d = dict(E, **edit)
        e2 = dict(E, dim_x=13, dim_y=12, dim_z=2, block_error=d_map.data_ptr() + 8192, count=d_cnt.data_ptr() + 4)
        return [tuple(d[f] for f in F), tuple(e2[f] for f in F)]

    def _raise(err):
        if err:
            raise gpu.AstcencError(err, "call")

    def expect(code, lists=None, components=4, raw=None, launches=0):
        torch.cuda.synchronize()
        n0 = ctx.launch_count()
        call = raw or (lambda: ctx.compute_block_errors_device_block_lists(table() if lists is None else lists, input_components=components))
        if code == 0:
            call()
        else:
            with pytest.raises(gpu.AstcencError) as e:
                call()
            assert e.value.code == code, (e.value.code, code)
        torch.cuda.synchronize()
        assert ctx.launch_count() == n0 + launches
        if launches == 0:
            assert np.all(d_map.cpu().numpy().view(np.uint32) == MAP_POISON)

    P = gpu.ERR_BAD_PARAM
    try:
        assert l.astcenc_b200_compute_block_errors_device_block_lists(None, 4, None, 0, None) == P
        for c in (0, 5):
            expect(P, components=c)
            expect(P, components=c, raw=lambda: _raise(l.astcenc_b200_compute_block_errors_device_block_lists(ctx.handle, c, None, 2, None)))
        expect(P, raw=lambda: _raise(l.astcenc_b200_compute_block_errors_device_block_lists(ctx.handle, 4, None, 2, None)))
        for edit in (dict(original=0), dict(decoded=0), dict(block_error=0), dict(indices=0), dict(count=0), dict(dim_x=0), dict(dim_z=0),
                     dict(dim_x=2 ** 32 - 1, dim_y=2 ** 32 - 1, dim_z=2 ** 32 - 1), dict(original_type=3), dict(decoded_type=-1),
                     dict(original=d_img.data_ptr() + 2), dict(decoded=d_img.data_ptr() + 32772), dict(block_error=d_map.data_ptr() + 2),
                     dict(indices=d_idx.data_ptr() + 2), dict(count=d_cnt.data_ptr() + 1), dict(dim_x=6 * 2 ** 16, dim_y=6 * 2 ** 16),
                     dict(dim_x=6 * 2 ** 16, dim_y=6 * 2 ** 16, capacity=0)):
            expect(P, lists=table(**edit))
        # capacity 0: NULL maps and lists are allowed, and nothing runs
        expect(0, lists=[t[:7] + (0, 0, 0, 0) for t in table()])
        expect(0, lists=[])
        expect(0, raw=lambda: _raise(l.astcenc_b200_compute_block_errors_device_block_lists(ctx.handle, 4, None, 0, None)))
        expect(0, lists=[table()[0][:7] + (0, 0, 0, 0), table()[1]], launches=1)
    finally:
        ctx.close()
