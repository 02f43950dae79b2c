"""Decoding every legal block mode, partitioning and endpoint mode of every block size.

astcenc_decompress_image and astcenc_get_block_info must handle any legal block, not only the blocks this encoder writes.
Real encodings reach only the block modes and partitionings that the presets select, and random bytes are mostly illegal
blocks. So each footprint gets a set built from the header fields up (tests/astc_blockgen.py, written from the ASTC
specification): every legal block mode, every partition index of 2, 3 and 4 partitions, every endpoint mode, the class
form of the endpoint-mode field, the sub-modes of the HDR endpoint modes, each dual-plane component, all-zero and all-one
payloads, void extents and one or more illegal blocks per illegal-encoding rule. The block modes the compressor never
searches and the partitionings it drops have table entries that only decoding reads.

CPU (-m "not gpu"): the sets' coverage, the parser's legal/illegal verdict against the oracle's decode, the oracle and the
one-lane host simulation of the device source against the reference build's decode, the parser against the reference
build's block info. GPU: the CUDA library through the C ABI against the reference build, byte for byte.

The reference build's answers are stored in tests/golden/golden_reference.npz; reference_answers() makes every call both
the CPU and the GPU tests compare against, so recording the CPU tests (ASTCENC_RECORD_REFERENCE, tests/conftest.py) records
the GPU tests' answers as well."""
import ctypes as C
import os

import numpy as np
import pytest

import astc_blockgen as G
from astc_ref import *  # noqa: F401,F403

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROFILES = (PRF_LDR_SRGB, PRF_LDR, PRF_HDR_RGB_LDR_A, PRF_HDR)
OUT_TYPES = (TYPE_U8, TYPE_F16, TYPE_F32)
NP = {TYPE_U8: np.uint8, TYPE_F16: np.float16, TYPE_F32: np.float32}
IDENTITY = (0, 1, 2, 3)
SWIZZLE = (0, 3, 6, 5)            # r from R, g from A, b the Z of a normal map reconstructed from R and A, a = 1
INFO_PROFILES = (PRF_LDR, PRF_HDR)
IDS = ["%dx%d" % fp[:2] if fp[2] == 1 else "%dx%dx%d" % fp for fp in G.FOOTPRINTS]


def decode_calls():
    """(profile, output type, swizzle) of every decode compared: all profiles and output types, unswizzled and swizzled."""
    return [(p, t, s) for s in (IDENTITY, SWIZZLE) for p in PROFILES for t in OUT_TYPES]


_ANSWERS = {}


def reference_answers(reference, fp):
    """The reference build's decode of the footprint's mosaic for every decode_calls() entry, and its block info (raw structs
    and header fields) of every set block under INFO_PROFILES."""
    key = (id(reference), fp)
    if key not in _ANSWERS:
        mo = G.mosaic(fp)
        flat = np.concatenate(mo.set_blocks)
        (w, h, d), (bx, by, bz) = mo.dims, fp
        dec = {c: reference.decompress_volume(mo.blocks, w, h, d, c[0], bx, by, bz, out_type=c[1], swz=c[2]) for c in decode_calls()}
        infos = {p: reference.block_infos(flat, p, bx, by, bz=bz) for p in INFO_PROFILES}
        fields = {p: reference.block_info_fields(flat, p, bx, by, bz=bz) for p in INFO_PROFILES}
        _ANSWERS[key] = dec, infos, fields
    return _ANSWERS[key]


@pytest.fixture(scope="module")
def headers():
    return {fp: [G.parse(b, fp) for b in G.mosaic(fp).set_blocks] for fp in G.FOOTPRINTS}


def _image_blocks(img, fp):
    """(d, h, w, 4) image -> list of per-block texel arrays in block order (ragged edge blocks are cut)."""
    bx, by, bz = fp
    d, h, w = img.shape[:3]
    return [img[z:z + bz, y:y + by, x:x + bx] for z in range(0, d, bz) for y in range(0, h, by) for x in range(0, w, bx)]


def _texel(t):
    """A texel's values and bit patterns (NaNs that differ only in their bits print alike)."""
    return "%s (%s)" % (t, " ".join("%x" % u for u in t.view({1: np.uint8, 2: np.uint16, 4: np.uint32}[t.dtype.itemsize])))


def explain(fp, got, want, call, headers):
    """A message naming the first block where two decodes of the mosaic differ (`want` from another implementation when the
    reference's answer is a digest), with its parsed header."""
    mo = G.mosaic(fp)
    for k, (a, b) in enumerate(zip(_image_blocks(got, fp), _image_blocks(want, fp))):
        if a.tobytes() != b.tobytes():
            j = int(mo.index[k])
            texel = int(np.argmax((a.view(np.uint8) != b.view(np.uint8)).reshape(a.shape[0] * a.shape[1] * a.shape[2], -1).any(axis=1)))
            return ("%s profile=%d type=%d swizzle=%s: image block %d (set block %d, %s, %s) first differs at texel %d: got %s, want %s; header: %s"
                    % (IDS[G.FOOTPRINTS.index(fp)], call[0], call[1], call[2], k, j, mo.kinds[j], mo.set_blocks[j].tobytes().hex(), texel,
                       _texel(a.reshape(-1, 4)[texel]), _texel(b.reshape(-1, 4)[texel]), headers[fp][j].describe()))
    return "%s profile=%d type=%d swizzle=%s: no block differs from the other implementation's decode, which the reference's answer does not match" % (
        IDS[G.FOOTPRINTS.index(fp)], call[0], call[1], call[2])


def _oracle_decode(oracle, fp, call):
    mo = G.mosaic(fp)
    return oracle.decompress_volume(mo.blocks, *mo.dims, call[0], fp[0], fp[1], fp[2], out_type=call[1], swz=list(call[2]))


def _bits(block, pos, n):
    return (int.from_bytes(block.tobytes(), "little") >> pos) & ((1 << n) - 1)


def _fill(block, lo, hi):
    """0 or 1 when bits lo..hi-1 of the block are all that bit, else None."""
    if hi <= lo:
        return None
    v = _bits(block, lo, hi - lo)
    return 0 if v == 0 else 1 if v == (1 << (hi - lo)) - 1 else None


def expected_info_fields(h):
    """The header fields astcenc_get_block_info reports for a block with parsed header h (astc_ref.BLOCK_INFO_FIELDS)."""
    row = [0] * 15
    if not h.legal:
        row[0] = 1
    elif h.void:
        row[1] = 1
    else:
        row[2], row[3], row[4] = int(h.dual), h.partitions, h.partition_index
        row[5] = h.ccs if h.dual else 0xFFFFFFFF
        row[6:6 + h.partitions] = h.cems
        row[10], row[11] = G.RANGES[h.colour_quant], G.WEIGHT_RANGES[h.weight_quant]
        row[12:15] = h.grid
    return row


# ------------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fp", G.FOOTPRINTS, ids=IDS)
def test_set_coverage(fp, headers):
    """The set reaches everything it is meant to; a generator edit that drops a block mode, index or rule fails here."""
    name = IDS[G.FOOTPRINTS.index(fp)]
    kinds, set_blocks = G.mosaic(fp).kinds, G.mosaic(fp).set_blocks
    hs = headers[fp]
    legal = [h for h in hs if h.legal and not h.void]
    missing = []

    seen = {(h.mode, h.partitions) for h in legal}
    for m in G.legal_block_modes(fp):
        if (m, 1) not in seen:
            missing.append("block mode %d with 1 partition" % m)
        p = G.max_partitions(m, fp)
        if p > 1 and (m, p) not in seen:
            missing.append("block mode %d with %d partitions" % (m, p))

    for p in (2, 3, 4):
        got = {h.partition_index for h in legal if h.partitions == p}
        missing += ["partition index %d of %d partitions" % (i, p) for i in range(1024) if i not in got]

    firsts = {(h.cems[0], h.partitions) for h in legal}
    for cem in range(16):
        c = cem >> 2
        for p in (1, 2, 3, 4):
            # the fewest colour values with this first mode: the others one class lower (class 0 stays 0)
            if 2 * (c + 1) + (p - 1) * 2 * max(c, 1) <= 18 and (cem, p) not in firsts:
                missing.append("endpoint mode %d first of %d partitions" % (cem, p))

    offsets = {(h.partitions, h.cem_selector, i, o) for h in legal if h.cem_selector for i, o in enumerate(h.cem_offsets)}
    for p in (2, 3, 4):
        for sel in (1, 2, 3):
            for i in range(p):
                for o in (0, 1):
                    if 2 * sel * (p - 1) + 2 * (sel + o) <= 18 and (p, sel, i, o) not in offsets:
                        missing.append("class form: %d partitions, class base %d, partition %d class offset %d" % (p, sel - 1, i, o))

    for cem in G.HDR_MODES:
        got = {G.hdr_submode(cem, h.endpoint_values) for h in legal if h.cems == [cem] and h.endpoint_values}
        missing += ["HDR endpoint mode %d sub-mode %s" % (cem, s) for s in G.hdr_submodes(cem) if s not in got]

    ccs = {(h.ccs, h.partitions) for h in legal if h.dual}
    missing += ["dual-plane component %d with %d partitions" % (c, p) for c in range(4) for p in (1, 2, 3) if (c, p) not in ccs]

    fills = set()
    for h, b in zip(hs, set_blocks):
        if h.legal and not h.void:
            fills.add(("colour", _fill(b, h.colour_start, h.colour_end)))
            fills.add(("weight", _fill(b, 128 - h.weight_bits, 128)))
    missing += ["%s payload all %d" % (a, f) for a in ("colour", "weight") for f in (0, 1) if (a, f) not in fills]

    ones = 0x1FFF if fp[2] == 1 else 0x1FF
    voids = {(h.void_hdr, h.legal, all(x == ones for x in h.extent)) for h in hs if h.void}
    for hdr in (False, True):
        for want, what in (((hdr, True, False), "valid extent"), ((hdr, True, True), "all-ones extent"), ((hdr, False, False), "invalid extent")):
            if want not in voids:
                missing.append("%s void extent with %s" % ("HDR" if hdr else "LDR", what))
    if fp[2] > 1 and any(len(h.extent) != 6 for h in hs if h.void):
        missing.append("3D void extents only")

    alone = {h.rules[0] for h in hs if len(h.rules) == 1}
    broken = {r for h in hs for r in h.rules}
    for rule in G.RULES:
        if rule == "void_extent_reserved_bits" and fp[2] > 1:
            continue            # 3D void extents have no reserved bits
        # a block-mode rule some block mode of this footprint breaks (alone); 12x12 and 6x6x6 hold every weight grid
        mode_rules = [G.block_mode_rules(m, fp) for m in range(2048) if m & 0x1FF != 0x1FC] if rule in G.BLOCK_MODE_RULES else [[rule]]
        isolable = [rule] in mode_rules
        if rule not in broken and any(rule in r for r in mode_rules):
            missing.append("an illegal block breaking %s" % rule)
        elif isolable and rule not in alone:
            missing.append("an illegal block breaking only %s" % rule)
    assert not missing, "%s: the set lacks %d items, first: %s" % (name, len(missing), missing[:10])
    assert kinds.count("partitioning") == 3 * 1024


@pytest.mark.parametrize("fp", G.FOOTPRINTS, ids=IDS)
def test_validity_agrees_with_oracle(fp, oracle, headers):
    """Under the HDR profile an illegal block decodes to the error colour (float NaN 0xFFFFE000) on every texel; a legal one does not."""
    img = _oracle_decode(oracle, fp, (PRF_HDR, TYPE_F32, IDENTITY))
    mo = G.mosaic(fp)
    bad = []
    for k, tex in enumerate(_image_blocks(img, fp)):
        s = int(mo.index[k])
        error = bool((tex.view(np.uint32) == 0xFFFFE000).all())
        if mo.whole[k] and error == headers[fp][s].legal:
            bad.append("set block %d (%s, %s): decoded %s, header %s" % (s, mo.kinds[s], mo.set_blocks[s].tobytes().hex(),
                                                                         "as error" if error else "as legal", headers[fp][s].describe()))
    assert not bad, "%s: %d blocks, first: %s" % (IDS[G.FOOTPRINTS.index(fp)], len(bad), bad[:3])


@pytest.mark.parametrize("fp", G.FOOTPRINTS, ids=IDS)
def test_oracle_matches_reference(fp, oracle, hostsim, reference, headers):
    """The oracle's decode of the set equals the reference build's: 4 profiles x 3 output types, unswizzled and swizzled.
    (A stored answer is a digest; on a mismatch the device source's decode, an independent implementation, names the block.)"""
    dec, _, _ = reference_answers(reference, fp)
    for call in decode_calls():
        got = _oracle_decode(oracle, fp, call)
        if not same(got, dec[call]):
            other = dec[call] if isinstance(dec[call], np.ndarray) else _hostsim_decode(hostsim, fp, call)
            pytest.fail(explain(fp, got, other, call, headers))


def _hostsim_decode(hostsim, fp, call):
    mo = G.mosaic(fp)
    blocks, (w, h, d) = mo.blocks, mo.dims
    out = np.zeros((d, h, w, 4), dtype=NP[call[1]])
    hostsim.hostsim_decompress_volume.argtypes = [C.c_int, C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.c_void_p, C.c_void_p, C.c_int,
                                                  C.c_uint, C.c_uint, C.c_uint, C.POINTER(C.c_int)]
    rc = hostsim.hostsim_decompress_volume(call[0], fp[0], fp[1], fp[2], 0, blocks.ctypes.data, out.ctypes.data, call[1], w, h, d,
                                           (C.c_int * 4)(*call[2]))
    assert rc == 0
    return out


@pytest.mark.parametrize("fp", G.FOOTPRINTS, ids=IDS)
def test_host_simulation_matches_reference(fp, hostsim, oracle, reference, headers):
    """The device decode source (one simulated lane, the shipped block-mode and partition tables) equals the reference build."""
    dec, _, _ = reference_answers(reference, fp)
    for call in decode_calls():
        got = _hostsim_decode(hostsim, fp, call)
        assert same(got, dec[call]), explain(fp, got, _oracle_decode(oracle, fp, call), call, headers)


@pytest.mark.parametrize("fp", G.FOOTPRINTS, ids=IDS)
def test_parser_matches_reference_block_info(fp, reference, headers):
    """The parser reads every header field as the reference build's astcenc_get_block_info does."""
    _, _, fields = reference_answers(reference, fp)
    want = np.array([expected_info_fields(h) for h in headers[fp]], dtype=np.uint32)
    for p in INFO_PROFILES:
        ref = fields[p]
        if isinstance(ref, np.ndarray):
            rows = np.nonzero((ref != want).any(axis=1))[0]
            assert len(rows) == 0, "%s profile=%d: %d blocks, first set block %d: reference %s, parser %s (%s)" % (
                IDS[G.FOOTPRINTS.index(fp)], p, len(rows), rows[0], list(ref[rows[0]]), list(want[rows[0]]), headers[fp][rows[0]].describe())
        else:
            assert same(want, ref), "%s profile=%d: the parser's fields differ from the reference's (stored as a digest: record live to see which)" % (
                IDS[G.FOOTPRINTS.index(fp)], p)


# ------------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------------
def _gpu_decode(ctx, fp, call):
    mo = G.mosaic(fp)
    (w, h, d) = mo.dims
    img = ctx.decompress_image(mo.blocks, w, h, dtype=NP[call[1]], swizzle=call[2], dim_z=d)
    return img.reshape(d, h, w, 4)


def _gpu_check(pkg, oracle, reference, headers, fp, calls, quality=PRE_MEDIUM, flags=0):
    dec, _, _ = reference_answers(reference, fp)
    for prof in sorted({c[0] for c in calls}):
        ctx = pkg.Context(pkg.config_init(prof, fp[0], fp[1], quality, flags, block_z=fp[2]))
        try:
            for call in [c for c in calls if c[0] == prof]:
                got = _gpu_decode(ctx, fp, call)
                assert same(got, dec[call]), "quality=%s flags=%d: %s" % (quality, flags, explain(fp, got, _oracle_decode(oracle, fp, call), call, headers))
        finally:
            ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fp", G.FOOTPRINTS, ids=IDS)
def test_cuda_decode_matches_reference(fp, pkg, oracle, reference, headers):
    """astcenc_decompress_image on the set equals the reference build byte for byte: every profile and output type."""
    _gpu_check(pkg, oracle, reference, headers, fp, [c for c in decode_calls() if c[2] == IDENTITY])


@pytest.mark.gpu
@pytest.mark.parametrize("fp", G.FOOTPRINTS, ids=IDS)
def test_cuda_decode_swizzle(fp, pkg, oracle, reference, headers):
    """A swizzle with Z reconstruction, every profile and output type. The error blocks' NaN texels reach the Z arithmetic,
    whose NaN result must keep the input's NaN bits as the reference's does."""
    _gpu_check(pkg, oracle, reference, headers, fp, [c for c in decode_calls() if c[2] == SWIZZLE])


@pytest.mark.gpu
@pytest.mark.parametrize("fp", G.FOOTPRINTS, ids=IDS)
def test_cuda_decode_independent_of_preset(fp, pkg, oracle, reference, headers):
    """The block modes and partitionings a preset does not search are decoded the same: contexts made at -fastest and
    -exhaustive, and decompression-only contexts, give the reference's bytes too."""
    calls = [(PRF_LDR, TYPE_U8, IDENTITY), (PRF_HDR, TYPE_F32, IDENTITY)]
    for quality, flags in ((PRE_FASTEST, 0), (PRE_EXHAUSTIVE, 0), (PRE_FASTEST, FLG_DECOMPRESS_ONLY), (PRE_MEDIUM, FLG_DECOMPRESS_ONLY)):
        _gpu_check(pkg, oracle, reference, headers, fp, calls, quality, flags)


@pytest.mark.gpu
@pytest.mark.parametrize("fp", G.FOOTPRINTS, ids=IDS)
def test_cuda_block_info(fp, pkg, reference, headers):
    """astcenc_get_block_info on every set block equals the reference build's struct, and its header fields equal the parser's."""
    _, infos, _ = reference_answers(reference, fp)
    prod = AstcencLib(os.path.join(ROOT, "astc-encoder_b200", "libastcenc_b200.so"))
    flat = np.concatenate(G.mosaic(fp).set_blocks)
    want = np.array([expected_info_fields(h) for h in headers[fp]], dtype=np.uint32)
    for p in INFO_PROFILES:
        got = prod.block_infos(flat, p, fp[0], fp[1], bz=fp[2])
        fields = block_info_fields(got)
        rows = np.nonzero((fields != want).any(axis=1))[0]
        assert len(rows) == 0, "%s profile=%d: %d blocks, first set block %d: library %s, parser %s (%s)" % (
            IDS[G.FOOTPRINTS.index(fp)], p, len(rows), rows[0], list(fields[rows[0]]), list(want[rows[0]]), headers[fp][rows[0]].describe())
        assert same(got, infos[p]), "%s profile=%d: block info structs differ from the reference's (header fields agree)" % (IDS[G.FOOTPRINTS.index(fp)], p)
