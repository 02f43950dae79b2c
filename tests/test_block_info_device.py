"""Block info of device-resident payloads: astcenc_b200_get_block_summaries_device_images writes a 16-byte summary of every
block of whole payloads (astc_block_summaries_kernel; summarize_table_blocks and block_summary, which runs the parser's header
stage block_header alone), and astcenc_b200_get_block_info_device_block_lists writes the full astcenc_block_info of the blocks
of device lists (astc_block_info_lists_kernel; info_list_slot and block_info, the body astcenc_get_block_info runs too).

CPU: both walks compiled for the host (tests/hostsim/hostsim_block_info.cpp, one lane and 32 lanes). On every footprint's
astc_blockgen set the summaries equal the parser's header fields (test_decode_modes.expected_info_fields), narrowed, and the
narrowed fields and HDR flag of the list structs; the list structs of the whole set equal the reference build's structs byte
for byte (stored answers) under the LDR and HDR profiles. Shuffled lists with duplicates, out-of-range indices, counts above
the capacity and zero counts leave their other slots' poison untouched. Ragged tables of images, arrays and volumes: an
entry's output does not depend on the rest of its table.
GPU: the library against the simulation and against astcenc_get_block_info per block under all four profiles, inside guard
bytes; a shuffled table of real payloads (-fast and -thorough LDR, F16 HDR, a mip chain down to 1-block levels, a texture
array, a 4x4x4 volume); the list call with counts from astcenc_b200_select_blocks on the same stream; launch counts,
decompress-only contexts and the error order."""
import ctypes as C
import os

import numpy as np
import pytest

import astc_blockgen as G
import astc_images as I
from astc_ref import *  # noqa: F401,F403
from hostsim_build import host_sim
from test_decode_device import block_pool, nblocks, payloads_for
from test_decode_modes import IDS, expected_info_fields

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROFILES = (PRF_LDR_SRGB, PRF_LDR, PRF_HDR_RGB_LDR_A, PRF_HDR)
INFO_PROFILES = (PRF_LDR, PRF_HDR)      # the profiles whose reference structs are stored
INFO_BYTES = 2144                       # sizeof(astcenc_block_info)
POISON = 0xA5

# struct astcenc_block_info (include/astcenc.h), the fields a summary narrows
INFO_DTYPE = np.dtype({"names": ["is_error", "is_constant", "is_hdr", "is_dual", "partition_count", "partition_index", "dual_plane_component",
                                 "color_endpoint_modes", "color_level_count", "weight_level_count", "weight_x", "weight_y", "weight_z"],
                       "formats": ["u1", "u1", "u1", "u1", "<u4", "<u4", "<u4", ("<u4", (4,)), "<u4", "<u4", "<u4", "<u4", "<u4"],
                       "offsets": [20, 21, 22, 23, 24, 28, 32, 36, 52, 56, 60, 64, 68], "itemsize": INFO_BYTES})
SUMMARY_DTYPE = np.dtype([("flags", np.uint8), ("partition_count", np.uint8), ("partition_index", "<u2"), ("dual_plane_component", np.uint8),
                          ("weight_x", np.uint8), ("weight_y", np.uint8), ("weight_z", np.uint8), ("color_endpoint_modes", np.uint8, (4,)),
                          ("color_level_count", "<u2"), ("weight_level_count", np.uint8), ("reserved", np.uint8)])

_SIMS = {}


def info_sim(lanes32=False):
    if lanes32 in _SIMS:
        return _SIMS[lanes32]
    lib = host_sim("hostsim_block_info", lanes32)
    lib.hostsim_block_summaries.argtypes = [C.c_int, C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint]
    lib.hostsim_block_info_lists.argtypes = [C.c_int, C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_void_p,
                                             C.c_void_p, C.c_void_p]
    _SIMS[lanes32] = lib
    return lib


def _ptrs(arrays):
    return (C.c_void_p * max(1, len(arrays)))(*[a.ctypes.data for a in arrays])


def _dims(shapes):
    return np.array([[s[2], s[1], s[0]] for s in shapes], np.uint32).reshape(-1)


def sim_summaries(lib, payloads, shapes, fp, profile, flags=0):
    """One summary call over (D, H, W) images: their summaries as uint8 (n, 16) arrays."""
    outs = [np.full((nblocks(s, fp), 16), POISON, np.uint8) for s in shapes]
    dims = _dims(shapes)
    assert lib.hostsim_block_summaries(profile, fp[0], fp[1], fp[2], flags, _ptrs(payloads), _ptrs(outs), dims.ctypes.data, len(shapes)) == 0
    return outs


def sim_info_lists(lib, payloads, shapes, fp, profile, lists):
    """One list call: lists[j] = (indices, count, capacity); returns each entry's capacity structs (uint8 (cap, 2144)),
    poison where nothing was written."""
    outs = [np.full((max(1, c), INFO_BYTES), POISON, np.uint8) for _, _, c in lists]
    idx = [np.concatenate([np.asarray(i, np.uint32).reshape(-1), np.zeros(1, np.uint32)]) for i, _, _ in lists]
    counts = np.array([k for _, k, _ in lists], np.uint32)
    caps = np.array([c for _, _, c in lists], np.uint32)
    dims = _dims(shapes)
    assert lib.hostsim_block_info_lists(profile, fp[0], fp[1], fp[2], 0, _ptrs(payloads), _ptrs(outs), dims.ctypes.data, len(shapes), _ptrs(idx),
                                        counts.ctypes.data, caps.ctypes.data) == 0
    return [o[:c] for o, (_, _, c) in zip(outs, lists)]


def narrow(structs):
    """astcenc_block_info structs (uint8 (n, 2144), or a list of raw bytes) -> the summaries the rule asks for (uint8 (n, 16))."""
    raw = np.frombuffer(b"".join(structs), np.uint8) if isinstance(structs, list) else np.ascontiguousarray(structs).reshape(-1)
    f = raw.view(INFO_DTYPE)
    s = np.zeros(len(f), SUMMARY_DTYPE)
    s["flags"] = f["is_error"] | (f["is_constant"] << 1) | (f["is_hdr"] << 2) | (f["is_dual"] << 3)
    dpc = f["dual_plane_component"]
    assert np.all((dpc < 4) | (dpc == 0xFFFFFFFF))
    s["dual_plane_component"] = np.where(dpc == 0xFFFFFFFF, 0xFF, dpc)
    for name, bits in (("partition_count", 8), ("partition_index", 16), ("weight_x", 8), ("weight_y", 8), ("weight_z", 8),
                       ("color_endpoint_modes", 8), ("color_level_count", 16), ("weight_level_count", 8)):
        assert np.all(f[name] < (1 << bits)), name      # every value fits its narrowed field
        s[name] = f[name]
    return s.view(np.uint8).reshape(-1, 16)


def narrow_fields(rows):
    """test_decode_modes.expected_info_fields rows (no HDR flag) -> summaries without the HDR bit."""
    r = np.asarray(rows, np.uint64)
    s = np.zeros(len(r), SUMMARY_DTYPE)
    s["flags"] = r[:, 0] | (r[:, 1] << 1) | (r[:, 2] << 3)
    s["partition_count"], s["partition_index"] = r[:, 3], r[:, 4]
    s["dual_plane_component"] = np.where(r[:, 5] == 0xFFFFFFFF, 0xFF, r[:, 5])
    s["color_endpoint_modes"] = r[:, 6:10]
    s["color_level_count"], s["weight_level_count"] = r[:, 10], r[:, 11]
    s["weight_x"], s["weight_y"], s["weight_z"] = r[:, 12], r[:, 13], r[:, 14]
    return s.view(np.uint8).reshape(-1, 16)


def first_row(a, b):
    rows = np.nonzero((np.asarray(a) != np.asarray(b)).reshape(len(a), -1).any(axis=1))[0]
    return None if len(rows) == 0 else int(rows[0])


def set_image(fp):
    """A footprint's blockgen set as one payload of one image (block k = set block k), and that image's (D, H, W) shape."""
    flat = np.ascontiguousarray(np.concatenate(G.mosaic(fp).set_blocks))
    n = len(flat) // 16
    return flat, (fp[2], fp[1], n * fp[0])


_HEADERS = {}


def headers(fp):
    if fp not in _HEADERS:
        _HEADERS[fp] = [G.parse(b, fp) for b in G.mosaic(fp).set_blocks]
    return _HEADERS[fp]


# ------------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lanes32", [False, True], ids=["lanes1", "lanes32"])
@pytest.mark.parametrize("fp", G.FOOTPRINTS, ids=IDS)
def test_hostsim_summaries_match_parser_and_reference_structs(fp, lanes32, reference):
    """On the footprint's set, under all four profiles: the summaries equal the parser's header fields, narrowed (the HDR bit
    aside), and the narrowed list structs of the whole set, HDR bit included; under LDR and HDR those structs equal the
    reference build's, byte for byte. So the HDR flag is pinned on every endpoint mode under every profile."""
    lib = info_sim(lanes32)
    flat, shape = set_image(fp)
    n = len(flat) // 16
    want_fields = narrow_fields([expected_info_fields(h) for h in headers(fp)])
    hdr_bit = np.zeros(16, np.uint8)
    hdr_bit[0] = 4
    hdr_seen = set()
    for p in PROFILES:
        got = sim_summaries(lib, [flat], [shape], fp, p)[0]
        k = first_row(got & ~hdr_bit, want_fields)
        assert k is None, "%s profile=%d: set block %d: summary %s, parser %s (%s)" % (IDS[G.FOOTPRINTS.index(fp)], p, k, got[k].tobytes().hex(),
                                                                                       want_fields[k].tobytes().hex(), headers(fp)[k].describe())
        structs = sim_info_lists(lib, [flat], [shape], fp, p, [(np.arange(n), n, n)])[0]
        if p in INFO_PROFILES:
            assert same([bytes(r) for r in structs], reference.block_infos(flat, p, fp[0], fp[1], bz=fp[2])), \
                "%s profile=%d: the simulated list structs differ from the reference build's" % (IDS[G.FOOTPRINTS.index(fp)], p)
        want = narrow(structs)
        k = first_row(got, want)
        assert k is None, "%s profile=%d: set block %d: summary %s, narrowed struct %s" % (IDS[G.FOOTPRINTS.index(fp)], p, k, got[k].tobytes().hex(),
                                                                                           want[k].tobytes().hex())
        hdr_seen.add((p, bool((got[:, 0] & 4).any())))
    # an LDR decode never reports HDR; the HDR profiles report it for the HDR endpoint modes the set holds
    assert hdr_seen == {(PRF_LDR_SRGB, False), (PRF_LDR, False), (PRF_HDR_RGB_LDR_A, True), (PRF_HDR, True)}


def _shuffled_lists(rng, n):
    """(indices, count, capacity) of lists over an image of n blocks: shuffled with duplicates and out-of-range indices; count
    above the capacity; count 0; capacity 0; a sorted tail past the count."""
    a = rng.permutation(max(n, 8))[: max(8, n // 3)].astype(np.uint32)      # (indices >= n of a small image: skipped)
    a[1] = a[0]
    a[2] = n
    a[3] = 0xFFFFFFFF
    a[5] = a[4]
    b = rng.integers(0, n, 40).astype(np.uint32)
    return [(a, len(a) + 7, len(a)), (b, 25, 40), (rng.integers(0, n, 6), 0, 6), (np.zeros(0), 3, 0), (np.arange(n), n, n)]


@pytest.mark.parametrize("lanes32", [False, True], ids=["lanes1", "lanes32"])
@pytest.mark.parametrize("fp", [(6, 6, 1), (12, 12, 1), (4, 4, 4), (6, 6, 6)], ids=["6x6", "12x12", "4x4x4", "6x6x6"])
def test_hostsim_lists_write_read_slots_only(fp, lanes32, reference):
    """Shuffled lists over the set (the last one lists every block in order, checked against the reference build's structs):
    slot s of a read slot holds the struct of block indices[s], byte for byte; skipped slots and slots past the count keep
    their poison."""
    lib = info_sim(lanes32)
    flat, shape = set_image(fp)
    n = len(flat) // 16
    rng = np.random.default_rng(sum(fp))
    for p in INFO_PROFILES:
        lists = _shuffled_lists(rng, n)
        outs = sim_info_lists(lib, [flat] * len(lists), [shape] * len(lists), fp, p, lists)
        ref = outs[-1]
        assert same([bytes(r) for r in ref], reference.block_infos(flat, p, fp[0], fp[1], bz=fp[2]))
        for j, ((idx, count, cap), out) in enumerate(zip(lists, outs)):
            idx = np.asarray(idx, np.uint32)
            for s in range(cap):
                if s < min(count, cap) and idx[s] < n:
                    assert np.array_equal(out[s], ref[idx[s]]), (p, j, s)
                else:
                    assert np.all(out[s] == POISON), (p, j, s)


TABLE_CASES = [((6, 6, 1), [(1, 37, 29), (1, 1, 1), (3, 13, 17), (1, 6, 6), (1, 5, 61), (2, 7, 1), (1, 200, 3), (4, 1, 90)]),
               ((4, 4, 4), [(5, 7, 9), (1, 1, 1), (4, 4, 4), (9, 3, 13), (13, 21, 2)])]


@pytest.mark.parametrize("lanes32", [False, True], ids=["lanes1", "lanes32"])
@pytest.mark.parametrize("fp,shapes", TABLE_CASES, ids=["6x6", "4x4x4"])
def test_hostsim_table_walks_do_not_depend_on_the_rest_of_the_table(fp, shapes, lanes32, golden):
    """Many ragged entries (2D images, texture arrays, volumes), repeated and shuffled: each entry's summaries equal a call of
    that entry alone, and those equal the summaries of the same blocks as one flat image; the list call over the same table
    writes what the list call of each entry alone writes."""
    lib = info_sim(lanes32)
    pool = block_pool(fp, golden, 7)
    rng = np.random.default_rng(11)
    shapes = [shapes[k] for k in rng.permutation(len(shapes))] * 3
    pays = payloads_for(shapes, fp, pool)
    flat = np.concatenate(pays)
    nflat = len(flat) // 16
    whole = sim_summaries(lib, [flat], [(1, 1, nflat * fp[0])] if fp[2] == 1 else [(fp[2], fp[1], nflat * fp[0])], fp, PRF_HDR)[0]
    got = sim_summaries(lib, pays, shapes, fp, PRF_HDR)
    assert np.array_equal(np.concatenate(got), whole)
    for j in rng.choice(len(shapes), 4, replace=False):
        assert np.array_equal(sim_summaries(lib, [pays[j]], [shapes[j]], fp, PRF_HDR)[0], got[j]), j
    lists = [_shuffled_lists(rng, nblocks(s, fp))[k % 4] for k, s in enumerate(shapes)]
    table = sim_info_lists(lib, pays, shapes, fp, PRF_LDR, lists)
    for j in rng.choice(len(shapes), 5, replace=False):
        alone = sim_info_lists(lib, [pays[j]], [shapes[j]], fp, PRF_LDR, [lists[j]])[0]
        assert np.array_equal(alone, table[j]), j


# ------------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu(pkg):
    import torch
    assert torch.cuda.is_available(), "the GPU tests need a CUDA device"
    torch.cuda.set_device(0)
    return pkg


GUARD = 256


class Guarded:
    """Device outputs of the given byte sizes inside one guard-filled allocation (each output 16-byte aligned, GUARD random
    bytes before, between and after)."""

    def __init__(self, sizes, seed=0):
        import torch
        self.offsets, o = [], GUARD
        for n in sizes:
            self.offsets.append(o)
            o += (n + 15) // 16 * 16 + GUARD
        self.guard = np.random.default_rng(seed).integers(0, 256, o, dtype=np.uint8)
        self.sizes = sizes
        self.buf = torch.from_numpy(self.guard.copy()).cuda()

    def ptr(self, j):
        return self.buf.data_ptr() + self.offsets[j]

    def read(self):
        """The outputs, after checking that every guard byte is intact."""
        host = self.buf.cpu().numpy()
        mask = np.ones(len(host), bool)
        for o, n in zip(self.offsets, self.sizes):
            mask[o:o + n] = False
        assert np.array_equal(host[mask], self.guard[mask]), "a guard byte changed"
        return [host[o:o + n] for o, n in zip(self.offsets, self.sizes)]


def device_summaries(ctx, payloads, shapes, fp, stream=0, order=None):
    """One summary call (entries in `order`) into guarded outputs: the summaries as uint8 (n, 16) arrays in input order."""
    import torch
    d_pay = [torch.from_numpy(p).cuda() for p in payloads]
    out = Guarded([nblocks(s, fp) * 16 for s in shapes], seed=len(shapes))
    order = range(len(shapes)) if order is None else order
    ctx.get_block_summaries_device_images([(d_pay[j].data_ptr(), shapes[j][2], shapes[j][1], shapes[j][0], out.ptr(j)) for j in order], stream=stream)
    torch.cuda.synchronize()
    return [o.reshape(-1, 16) for o in out.read()]


@pytest.mark.gpu
@pytest.mark.parametrize("fp", G.FOOTPRINTS, ids=IDS)
def test_summaries_match_simulation_and_get_block_info(fp, gpu):
    """On the footprint's set, under all four profiles: the summaries equal the simulation's and the narrowed
    astcenc_get_block_info of every block, inside guard bytes, one launch per call."""
    lib = info_sim()
    flat, shape = set_image(fp)
    prod = AstcencLib(os.path.join(ROOT, "astc-encoder_b200", "libastcenc_b200.so"))
    for p in PROFILES:
        ctx = gpu.Context(gpu.config_init(p, fp[0], fp[1], PRE_MEDIUM, FLG_DECOMPRESS_ONLY, block_z=fp[2]))
        try:
            n0 = ctx.launch_count()
            got = device_summaries(ctx, [flat], [shape], fp)[0]
            assert ctx.launch_count() == n0 + 1
        finally:
            ctx.close()
        assert np.array_equal(got, sim_summaries(lib, [flat], [shape], fp, p)[0]), p
        want = narrow(prod.block_infos(flat, p, fp[0], fp[1], bz=fp[2]))
        k = first_row(got, want)
        assert k is None, "profile=%d: set block %d: summary %s, get_block_info %s" % (p, k, got[k].tobytes().hex(), want[k].tobytes().hex())


def _real_payloads(gpu):
    """Real 6x6 payloads of many shapes: -fast and -thorough LDR, F16 HDR, a mip chain down to 1-block levels and a texture
    array; and 4x4x4 volumes. Returns {footprint: [(payload, (D, H, W))]}."""
    out = {(6, 6, 1): [], (4, 4, 4): []}
    for q in (PRE_FAST, PRE_THOROUGH):
        ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, q, FLG_SELF_DECOMPRESS_ONLY))
        for k, (h, w) in enumerate([(128, 128), (61, 97), (200, 33), (6, 6), (13, 250)]):
            im = I.photo_like(h, w, seed=40 + k) if k % 2 == 0 else I.voronoi_flat(h, w, seed=40 + k)
            out[(6, 6, 1)].append((ctx.compress_image(im), (1, h, w)))
        s = 256
        while True:
            out[(6, 6, 1)].append((ctx.compress_image(I.photo_like(s, s, seed=s)), (1, s, s)))
            if s == 1:
                break
            s //= 2
        arr = np.stack([I.alpha_mask(40, 50, seed=z) for z in range(3)])
        out[(6, 6, 1)].append((ctx.compress_image(arr), (3, 40, 50)))
        ctx.close()
    ctx = gpu.Context(gpu.config_init(PRF_HDR, 6, 6, PRE_FAST, FLG_SELF_DECOMPRESS_ONLY))
    for k, (h, w) in enumerate([(64, 64), (37, 90)]):
        out[(6, 6, 1)].append((ctx.compress_image(I.hdr_noise(h, w, seed=k)), (1, h, w)))
    ctx.close()
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 4, 4, PRE_FAST, FLG_SELF_DECOMPRESS_ONLY, block_z=4))
    for k, (d, h, w) in enumerate([(8, 16, 16), (5, 7, 9), (1, 1, 1)]):
        vol = np.stack([I.photo_like(h, w, seed=60 + k + z) for z in range(d)])
        out[(4, 4, 4)].append((ctx.compress_image(vol), (d, h, w)))
    ctx.close()
    return out


@pytest.mark.gpu
def test_shuffled_table_of_real_payloads(gpu):
    """More than 40 real payloads in one shuffled call per footprint, under an LDR and an HDR context: every entry's summaries
    equal the simulation of that payload alone, inside guard bytes."""
    lib = info_sim()
    real = _real_payloads(gpu)
    rng = np.random.default_rng(5)
    for fp, items in real.items():
        items = items * 2 if fp == (6, 6, 1) else items * 4
        assert fp != (6, 6, 1) or len(items) > 40
        pays, shapes = [p for p, _ in items], [s for _, s in items]
        for prof in (PRF_LDR, PRF_HDR):
            ctx = gpu.Context(gpu.config_init(prof, fp[0], fp[1], PRE_FAST, FLG_DECOMPRESS_ONLY, block_z=fp[2]))
            try:
                got = device_summaries(ctx, pays, shapes, fp, order=list(rng.permutation(len(items))))
            finally:
                ctx.close()
            for j in range(len(items)):
                assert np.array_equal(got[j], sim_summaries(lib, [pays[j]], [shapes[j]], fp, prof)[0]), (fp, prof, j, shapes[j])
    # the -thorough payload of a photo uses more than one partition somewhere (the table above was not all one kind of block)
    s = sim_summaries(lib, [real[(6, 6, 1)][15][0]], [real[(6, 6, 1)][15][1]], (6, 6, 1), PRF_LDR)[0].reshape(-1).view(SUMMARY_DTYPE)
    assert (s["partition_count"] > 1).any()


@pytest.mark.gpu
def test_list_call_with_selected_counts_matches_get_block_info(gpu):
    """-fast payloads, decoded, mapped and the worst blocks selected on one stream; the list call on the same stream reads the
    counts select_blocks wrote. Every read slot equals astcenc_get_block_info of its block byte for byte, every other byte of
    the guarded outputs keeps its guard; the shuffled set lists of 4x4x4 too."""
    import torch
    dev = torch.device("cuda", 0)
    prod = AstcencLib(os.path.join(ROOT, "astc-encoder_b200", "libastcenc_b200.so"))
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, FLG_SELF_DECOMPRESS_ONLY))
    try:
        imgs = [I.photo_like(h, w, seed=70 + k) for k, (h, w) in enumerate([(120, 96), (61, 200), (6, 6)])]
        nb = [nblocks((1,) + im.shape[:2], (6, 6, 1)) for im in imgs]
        dims = [(im.shape[1], im.shape[0]) for im in imgs]
        caps = [max(1, n // 5) + 3 for n in nb]
        d_img = [torch.from_numpy(im.reshape(-1)).to(dev) for im in imgs]
        d_pay = [torch.zeros(n * 16, dtype=torch.uint8, device=dev) for n in nb]
        d_dec = [torch.zeros(im.size, dtype=torch.uint8, device=dev) for im in imgs]
        mb = C.sizeof(gpu.ErrorMetrics)
        d_met = torch.zeros(len(imgs) * mb, dtype=torch.uint8, device=dev)
        d_map = [torch.zeros(n, dtype=torch.float32, device=dev) for n in nb]
        d_idx = [torch.zeros(c, dtype=torch.int32, device=dev) for c in caps]
        d_cnt = torch.zeros(len(imgs), dtype=torch.int32, device=dev)
        out = Guarded([c * INFO_BYTES for c in caps], seed=3)
        st = torch.cuda.Stream(device=dev)
        torch.cuda.synchronize()
        s = st.cuda_stream
        ctx.compress_device_images([(d.data_ptr(), w, h, 1, p.data_ptr()) for d, (w, h), p in zip(d_img, dims, d_pay)], TYPE_U8, stream=s)
        ctx.decompress_device_images([(p.data_ptr(), o.data_ptr(), w, h, 1) for p, o, (w, h) in zip(d_pay, d_dec, dims)], TYPE_U8, stream=s)
        ctx.compute_error_metrics_device_images([(d.data_ptr(), o.data_ptr(), TYPE_U8, TYPE_U8, w, h, 1, d_met.data_ptr() + k * mb, m.data_ptr())
                                                 for k, (d, o, (w, h), m) in enumerate(zip(d_img, d_dec, dims, d_map))], input_components=4, stream=s)
        # capacity - 3 of them: the last three slots of each list lie past the count
        ctx.select_blocks([(m.data_ptr(), n, -np.inf, c - 3, ix.data_ptr(), d_cnt.data_ptr() + 4 * k)
                           for k, (m, n, c, ix) in enumerate(zip(d_map, nb, caps, d_idx))], stream=s)
        n0 = ctx.launch_count()
        ctx.get_block_info_device_block_lists([(p.data_ptr(), w, h, 1, ix.data_ptr(), d_cnt.data_ptr() + 4 * k, c, out.ptr(k))
                                               for k, (p, (w, h), ix, c) in enumerate(zip(d_pay, dims, d_idx, caps))], stream=s)
        assert ctx.launch_count() == n0 + 1
        st.synchronize()
        got = out.read()
        cnt = d_cnt.cpu().numpy()
        for k in range(len(imgs)):
            pay = d_pay[k].cpu().numpy().reshape(-1, 16)
            idx = d_idx[k].cpu().numpy().view(np.uint32)
            assert cnt[k] == caps[k] - 3
            slots = got[k].reshape(caps[k], INFO_BYTES)
            want = prod.block_infos(pay[idx[:cnt[k]]].reshape(-1), PRF_LDR, 6, 6)
            for s_ in range(caps[k]):
                if s_ < cnt[k]:
                    assert slots[s_].tobytes() == want[s_], (k, s_)
                else:
                    assert np.array_equal(slots[s_], out.guard[out.offsets[k] + s_ * INFO_BYTES:out.offsets[k] + (s_ + 1) * INFO_BYTES]), (k, s_)
    finally:
        ctx.close()
    # the 4x4x4 set, shuffled lists with duplicates and out-of-range indices, against the simulation
    fp = (4, 4, 4)
    flat, shape = set_image(fp)
    n = len(flat) // 16
    lists = _shuffled_lists(np.random.default_rng(9), n)
    ctx = gpu.Context(gpu.config_init(PRF_HDR, 4, 4, PRE_FAST, FLG_DECOMPRESS_ONLY, block_z=4))
    try:
        d_flat = torch.from_numpy(flat).cuda()
        d_idx = [torch.from_numpy(np.concatenate([np.asarray(i, np.uint32), np.zeros(1, np.uint32)]).view(np.int32)).cuda() for i, _, _ in lists]
        d_cnt = torch.from_numpy(np.array([k for _, k, _ in lists], np.uint32).view(np.int32)).cuda()
        out = Guarded([max(1, c) * INFO_BYTES for _, _, c in lists], seed=4)
        ctx.get_block_info_device_block_lists([(d_flat.data_ptr(), shape[2], shape[1], shape[0], ix.data_ptr(), d_cnt.data_ptr() + 4 * j, c, out.ptr(j))
                                               for j, (ix, (_, _, c)) in enumerate(zip(d_idx, lists))])
        torch.cuda.synchronize()
        got = out.read()
    finally:
        ctx.close()
    want = sim_info_lists(info_sim(), [flat] * len(lists), [shape] * len(lists), fp, PRF_HDR, lists)
    for j, (_, _, c) in enumerate(lists):
        g = got[j][:c * INFO_BYTES].reshape(c, INFO_BYTES)
        # (the simulation's poison stands for the untouched slots; the device keeps its guard bytes there)
        written = ~np.all(want[j] == POISON, axis=1)
        assert np.array_equal(g[written], want[j][written]), j
        gb = out.guard[out.offsets[j]:out.offsets[j] + c * INFO_BYTES].reshape(c, INFO_BYTES)
        assert np.array_equal(g[~written], gb[~written]), j


@pytest.mark.gpu
@pytest.mark.parametrize("call", ["summaries", "lists"])
def test_errors_follow_the_documented_order(call, gpu):
    """The error order of include/astcenc.h, with nothing launched and nothing written; empty calls launch nothing; both
    calls run on decompress-only contexts, one launch each."""
    import torch
    dev = torch.device("cuda", 0)
    ctx = gpu.Context(gpu.config_init(PRF_LDR, 6, 6, PRE_FAST, FLG_DECOMPRESS_ONLY))
    d_pay = torch.zeros(4096, dtype=torch.uint8, device=dev)
    d_idx = torch.zeros(64, dtype=torch.int32, device=dev)
    d_cnt = torch.full((4,), 3, dtype=torch.int32, device=dev)
    d_out = torch.full((65536,), POISON, dtype=torch.uint8, device=dev)
    l = gpu.lib()
    if call == "summaries":
        F = ("payload", "dim_x", "dim_y", "dim_z", "summaries")
        E = dict(payload=d_pay.data_ptr(), dim_x=44, dim_y=40, dim_z=1, summaries=d_out.data_ptr())
        E2 = dict(E, payload=d_pay.data_ptr() + 2048, dim_x=13, dim_y=12, dim_z=2, summaries=d_out.data_ptr() + 32768)
        method, fn, S = ctx.get_block_summaries_device_images, l.astcenc_b200_get_block_summaries_device_images, gpu.DeviceBlockSummaryImage
        bad = [dict(payload=0), dict(summaries=0), dict(summaries=d_out.data_ptr() + 4), dict(summaries=d_out.data_ptr() + 8)]
    else:
        F = ("payload", "dim_x", "dim_y", "dim_z", "indices", "count", "capacity", "infos")
        E = dict(payload=d_pay.data_ptr(), dim_x=44, dim_y=40, dim_z=1, indices=d_idx.data_ptr(), count=d_cnt.data_ptr(), capacity=8, infos=d_out.data_ptr())
        E2 = dict(E, payload=d_pay.data_ptr() + 2048, dim_x=13, dim_y=12, dim_z=2, count=d_cnt.data_ptr() + 4, infos=d_out.data_ptr() + 32768)
        method, fn, S = ctx.get_block_info_device_block_lists, l.astcenc_b200_get_block_info_device_block_lists, gpu.DeviceBlockInfoList
        bad = [dict(payload=0), dict(infos=0), dict(indices=0), dict(count=0), dict(indices=d_idx.data_ptr() + 2), dict(count=d_cnt.data_ptr() + 1),
               dict(infos=d_out.data_ptr() + 2)]

    def table(**edit):
        d = dict(E, **edit)
        return [tuple(d[f] for f in F), tuple(E2[f] for f in F)]

    def _raise(err):
        if err:
            raise gpu.AstcencError(err, "call")

    def expect(code, entries=None, raw=None, launches=0):
        torch.cuda.synchronize()
        n0 = ctx.launch_count()
        run = raw or (lambda: method(table() if entries is None else entries))
        if code == 0:
            run()
        else:
            with pytest.raises(gpu.AstcencError) as e:
                run()
            assert e.value.code == code, (e.value.code, code)
        torch.cuda.synchronize()
        assert ctx.launch_count() == n0 + launches
        if launches == 0:
            assert np.all(d_out.cpu().numpy() == POISON)

    P = gpu.ERR_BAD_PARAM
    try:
        one = (S * 1)(S(*[C.c_void_p(v) if isinstance(v, int) and f in ("payload", "summaries", "indices", "count", "infos") else v
                           for f, v in zip(F, table()[0])]))
        expect(P, raw=lambda: _raise(fn(None, one, 1, None)))                  # 1. a NULL context
        expect(P, raw=lambda: _raise(fn(None, None, 2, None)))
        expect(P, raw=lambda: _raise(fn(ctx.handle, None, 2, None)))           # 2. a NULL table with a non-zero count
        for edit in bad + [dict(dim_x=0), dict(dim_y=0), dict(dim_z=0), dict(dim_x=2 ** 32 - 1, dim_y=2 ** 32 - 1, dim_z=2 ** 32 - 1),
                           dict(dim_x=6 * 2 ** 16, dim_y=6 * 2 ** 16)]:       # 3. pointers, 4. dimensions, 5. 2^32 blocks
            expect(P, entries=table(**edit))
            expect(P, entries=table(**edit)[::-1])
        expect(0, entries=[])
        expect(0, raw=lambda: _raise(fn(ctx.handle, None, 0, None)))
        if call == "lists":
            # capacity 0: NULL lists and outputs are allowed, and nothing runs
            expect(0, entries=[t[:4] + (0, 0, 0, 0) for t in table()])
            expect(P, entries=[t[:4] + (0, 0, 0, 0) for t in table(dim_x=6 * 2 ** 16, dim_y=6 * 2 ** 16)])
            expect(0, entries=[table()[0][:4] + (0, 0, 0, 0), table()[1]], launches=1)
        else:
            expect(0, launches=1)
    finally:
        ctx.close()
