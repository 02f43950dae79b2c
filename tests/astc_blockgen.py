"""ASTC block headers, read and written from the Khronos ASTC specification (Khronos Data Format Specification, chapter
"ASTC Compressed Texture Image Formats": block mode layouts, partition and endpoint-mode fields, void-extent blocks,
integer sequence encoding sizes and the illegal-encoding rules).

parse() reads the header of one 16-byte block; write_block() puts chosen header fields into a seeded random block and
leaves the endpoint and weight payloads random. Every bit pattern is a decodable integer-sequence payload, so a block
with a legal header is a valid block. block_set() builds, per footprint, the decode test set of tests/test_decode_modes.py.

Bits are numbered as in the specification: bit k of a block is bit k % 8 of byte k // 8.
"""
import collections
import functools

import numpy as np

FOOTPRINTS_2D = ((4, 4, 1), (5, 4, 1), (5, 5, 1), (6, 5, 1), (6, 6, 1), (8, 5, 1), (8, 6, 1), (8, 8, 1),
                 (10, 5, 1), (10, 6, 1), (10, 8, 1), (10, 10, 1), (12, 10, 1), (12, 12, 1))
FOOTPRINTS_3D = ((3, 3, 3), (4, 3, 3), (4, 4, 3), (4, 4, 4), (5, 4, 4), (5, 5, 4), (5, 5, 5), (6, 5, 5), (6, 6, 5), (6, 6, 6))
FOOTPRINTS = FOOTPRINTS_2D + FOOTPRINTS_3D

# the 21 ranges of the integer sequence encoding; a quant level is an index into this table
RANGES = (2, 3, 4, 5, 6, 8, 10, 12, 16, 20, 24, 32, 40, 48, 64, 80, 96, 128, 160, 192, 256)
QUANT_6, QUANT_256 = 4, 20
# weight quant levels are the first twelve ranges: 2 .. 32
WEIGHT_RANGES = RANGES[:12]

HDR_MODES = (2, 3, 7, 11, 14, 15)

# the rules that make a block illegal, in the order parse() reports them
RULES = (
    "reserved_block_mode",          # a block-mode encoding the specification reserves
    "too_many_weights",             # more than 64 weights (both planes counted)
    "weight_bits_out_of_range",     # the weights take fewer than 24 or more than 96 bits
    "grid_exceeds_block",           # a weight grid dimension larger than the block's
    "dual_plane_4_partitions",      # dual plane with four partitions
    "too_many_colour_values",       # the endpoint modes need more than 18 colour values
    "colour_bits_insufficient",     # the colour values do not fit the remaining bits even at range 6
    "void_extent_reserved_bits",    # 2D void extent whose bits 10..11 are not both one
    "void_extent_bad_extent",       # void extent with a low coordinate not below its high one (and not all ones)
)
BLOCK_MODE_RULES = RULES[:4]


def _range_shape(r):
    """(bits, trits, quints) of one value of range r: r = 2^bits, 3 * 2^bits or 5 * 2^bits."""
    for t, m in ((0, 1), (1, 3), (2, 5)):
        if r % m == 0 and (r // m) & (r // m - 1) == 0:
            bits = (r // m).bit_length() - 1
            return bits, t == 1, t == 2
    raise ValueError(r)


def ise_bits(count, quant):
    """Bits of an integer sequence of `count` values of range RANGES[quant]: trits pack five values in 8 bits, quints three in 7."""
    bits, trits, quints = _range_shape(RANGES[quant])
    extra = (8 * count + 4) // 5 if trits else (7 * count + 2) // 3 if quints else 0
    return count * bits + extra


def _block_mode_2d(m):
    """The 2D block-mode layout: ((wx, wy, 1), weight quant level, dual plane), or None for a reserved encoding."""
    h, d = (m >> 9) & 1, (m >> 10) & 1
    a = (m >> 5) & 3
    if m & 3:
        r = ((m & 3) << 1) | ((m >> 4) & 1)
        b = (m >> 7) & 3
        sel = (m >> 2) & 3
        if sel == 0:
            grid = (b + 4, a + 2)
        elif sel == 1:
            grid = (b + 8, a + 2)
        elif sel == 2:
            grid = (a + 2, b + 8)
        elif (m >> 8) & 1:
            grid = ((b & 1) + 2, a + 2)
        else:
            grid = (a + 2, (b & 1) + 6)
    else:
        r = (((m >> 2) & 3) << 1) | ((m >> 4) & 1)
        if (m >> 2) & 3 == 0:
            return None
        sel = (m >> 7) & 3
        if sel == 0:
            grid = (12, a + 2)
        elif sel == 1:
            grid = (a + 2, 12)
        elif sel == 2:
            grid = (a + 6, ((m >> 9) & 3) + 6)
            h = d = 0
        elif a == 0:
            grid = (6, 10)
        elif a == 1:
            grid = (10, 6)
        else:
            return None
    return (grid[0], grid[1], 1), (r - 2) + 6 * h, bool(d)


def _block_mode_3d(m):
    """The 3D block-mode layout: ((wx, wy, wz), weight quant level, dual plane), or None for a reserved encoding."""
    h, d = (m >> 9) & 1, (m >> 10) & 1
    a = (m >> 5) & 3
    if m & 3:
        r = ((m & 3) << 1) | ((m >> 4) & 1)
        grid = (a + 2, ((m >> 7) & 3) + 2, ((m >> 2) & 3) + 2)
    else:
        r = (((m >> 2) & 3) << 1) | ((m >> 4) & 1)
        if (m >> 2) & 3 == 0:
            return None
        b = (m >> 9) & 3
        sel = (m >> 7) & 3
        if sel == 0:
            grid = (6, b + 2, a + 2)
        elif sel == 1:
            grid = (a + 2, 6, b + 2)
        elif sel == 2:
            grid = (a + 2, b + 2, 6)
        elif a == 3:
            return None
        else:
            grid = ((6, 2, 2), (2, 6, 2), (2, 2, 6))[a]
        if sel != 3:
            h = d = 0
    return grid, (r - 2) + 6 * h, bool(d)


@functools.lru_cache(maxsize=None)
def block_mode(m, is_3d):
    """Header facts of block mode m (0..2047) that do not depend on the footprint. None for reserved and void-extent encodings."""
    if m & 0x1FF == 0x1FC:
        return None
    dm = _block_mode_3d(m) if is_3d else _block_mode_2d(m)
    if dm is None:
        return None
    grid, wq, dual = dm
    count = grid[0] * grid[1] * grid[2] * (2 if dual else 1)
    return grid, wq, dual, count, ise_bits(count, wq)


def block_mode_rules(m, fp):
    """The block-mode rules mode m breaks in footprint fp (empty: a legal block mode there)."""
    bm = block_mode(m, fp[2] > 1)
    if bm is None:
        return ["reserved_block_mode"]
    grid, wq, dual, count, wbits = bm
    rules = []
    if count > 64:
        rules.append("too_many_weights")
    if not 24 <= wbits <= 96:
        rules.append("weight_bits_out_of_range")
    if any(g > b for g, b in zip(grid, fp)):
        rules.append("grid_exceeds_block")
    return rules


@functools.lru_cache(maxsize=None)
def legal_block_modes(fp):
    """Every block mode that is legal in footprint fp, in index order."""
    return tuple(m for m in range(2048) if m & 0x1FF != 0x1FC and not block_mode_rules(m, fp))


def _bits(v, pos, n):
    return (v >> pos) & ((1 << n) - 1)


def colour_quant(values, budget):
    """The colour quant level of `values` endpoint values in `budget` bits: the largest range whose sequence fits; None if none fits."""
    fit = [q for q in range(len(RANGES)) if ise_bits(values, q) <= budget]
    return fit[-1] if fit else None


class Header:
    """The parsed header of one block. Fields that a block does not have are None."""
    void = void_hdr = extent = None
    mode = grid = weight_quant = dual = weight_count = weight_bits = None
    partitions = partition_index = cems = cem_selector = cem_offsets = cem_low = None
    ccs = colour_values = colour_bits = colour_quant = colour_start = colour_end = None
    endpoint_values = None

    def __init__(self):
        self.rules = []

    @property
    def legal(self):
        return not self.rules

    def describe(self):
        if self.void:
            return "void extent %s extent=%s rules=%s" % ("HDR" if self.void_hdr else "LDR", self.extent, self.rules)
        return ("mode=%d grid=%s wq=%s dual=%s wbits=%s parts=%s index=%s cems=%s selector=%s ccs=%s colour_bits=%s cq=%s rules=%s"
                % (self.mode, self.grid, self.weight_quant, self.dual, self.weight_bits, self.partitions, self.partition_index, self.cems,
                   self.cem_selector, self.ccs, self.colour_bits, self.colour_quant, self.rules))


def parse(block, fp):
    """Parse the header of one 16-byte block (bytes or uint8 array) of footprint fp = (x, y, z)."""
    v = int.from_bytes(bytes(block), "little")
    h = Header()
    h.mode = m = _bits(v, 0, 11)
    if m & 0x1FF == 0x1FC:
        h.void, h.void_hdr = True, bool(m & 0x200)
        if fp[2] == 1:
            if _bits(v, 10, 2) != 3:
                h.rules.append("void_extent_reserved_bits")
            h.extent = tuple(_bits(v, 12 + 13 * i, 13) for i in range(4))
            ones = 0x1FFF
        else:
            h.extent = tuple(_bits(v, 10 + 9 * i, 9) for i in range(6))
            ones = 0x1FF
        e = h.extent
        if any(e[i] >= e[i + 1] for i in range(0, len(e), 2)) and any(x != ones for x in e):
            h.rules.append("void_extent_bad_extent")
        return h
    h.void = False
    h.rules = block_mode_rules(m, fp)
    if h.rules:
        return h
    h.grid, h.weight_quant, h.dual, h.weight_count, h.weight_bits = block_mode(m, fp[2] > 1)
    h.partitions = p = _bits(v, 11, 2) + 1
    below = 128 - h.weight_bits           # the weights fill the block from bit 127 down
    if p == 1:
        h.partition_index = 0
        h.cems = [_bits(v, 13, 4)]
        h.cem_selector = 0
        h.colour_start = 17
    else:
        h.partition_index = _bits(v, 13, 10)
        h.cem_low = _bits(v, 23, 6)
        h.cem_selector = sel = h.cem_low & 3
        if sel == 0:
            h.cems = [h.cem_low >> 2] * p
        else:
            extra = 3 * p - 4         # the rest of the endpoint-mode field sits just below the weights
            below -= extra
            field = h.cem_low | (_bits(v, below, extra) << 6)
            h.cem_offsets = [(field >> (2 + i)) & 1 for i in range(p)]
            h.cems = [((sel - 1 + h.cem_offsets[i]) << 2) | ((field >> (2 + p + 2 * i)) & 3) for i in range(p)]
        h.colour_start = 29
    if h.dual:
        below -= 2                    # the dual-plane component selector sits below that
        h.ccs = _bits(v, below, 2)
    h.colour_end = below
    if h.dual and p == 4:
        h.rules.append("dual_plane_4_partitions")
    h.colour_values = sum(2 * ((c >> 2) + 1) for c in h.cems)
    h.colour_bits = max(0, below - h.colour_start)
    if h.colour_values > 18:
        h.rules.append("too_many_colour_values")
    else:
        q = colour_quant(h.colour_values, h.colour_bits)
        if q is None or q < QUANT_6:
            h.rules.append("colour_bits_insufficient")
        else:
            h.colour_quant = q
            if q == QUANT_256 and p == 1:      # range 256 stores each value as its own 8 bits, unchanged by unquantisation
                h.endpoint_values = [_bits(v, 17 + 8 * i, 8) for i in range(h.colour_values)]
    return h


def hdr_submode(cem, ev):
    """The specification's sub-mode selection of the HDR endpoint modes, from the endpoint values ev (a label)."""
    def rgb(v):
        majcomp = (v[4] >> 7) | ((v[5] >> 7) << 1)
        if majcomp == 3:
            return "direct"
        return "major%d.mode%d" % (majcomp, (v[1] >> 7) | ((v[2] >> 7) << 1) | ((v[3] >> 7) << 2))
    if cem == 2:
        return "swapped" if ev[1] < ev[0] else "ordered"
    if cem == 3:
        return "mode%d" % (ev[0] >> 7)
    if cem == 7:
        return "modeval%d" % ((ev[0] >> 6) | ((ev[1] >> 7) << 2) | ((ev[2] >> 7) << 3))
    if cem in (11, 14):
        return rgb(ev)
    if cem == 15:
        return rgb(ev) + ".alpha%d" % ((ev[6] >> 7) | ((ev[7] >> 7) << 1))
    return None


def hdr_submodes(cem):
    """Every label hdr_submode() can give for one HDR endpoint mode."""
    rgb = ["major%d.mode%d" % (j, k) for j in range(3) for k in range(8)] + ["direct"]
    return {2: ["ordered", "swapped"], 3: ["mode0", "mode1"], 7: ["modeval%d" % i for i in range(16)],
            11: rgb, 14: rgb, 15: ["%s.alpha%d" % (r, a) for r in rgb for a in range(4)]}[cem]


def _set_bits(v, pos, n, x):
    mask = ((1 << n) - 1) << pos
    return (v & ~mask) | ((x << pos) & mask)


def write_block(rng, fp, mode, partitions=1, partition_index=0, cems=(0,), ccs=0, shared=None, offsets=None,
                colour_fill=None, weight_fill=None, endpoint_values=None):
    """A random 16-byte block with the given header fields (a uint8 array).

    cems: one endpoint mode per partition (one value is repeated). shared: write them in the one-mode form (default: when all
    are equal); otherwise in the class form, whose class base is the smallest class unless `offsets` gives each partition's
    class offset. colour_fill / weight_fill: 0 or 1 fills the colour or weight area with that bit. endpoint_values: the
    endpoint values of a one-partition block whose colour quant level is range 256."""
    v = int.from_bytes(rng.integers(0, 256, 16, dtype=np.uint8).tobytes(), "little")
    v = _set_bits(v, 0, 11, mode)
    v = _set_bits(v, 11, 2, partitions - 1)
    bm = block_mode(mode, fp[2] > 1)
    wbits = bm[4] if bm and bm[4] <= 96 else 0     # an illegal block mode: the fields below the weights stay random
    below = 128 - wbits
    cems = list(cems) * partitions if len(cems) == 1 else list(cems)
    if partitions == 1:
        v = _set_bits(v, 13, 4, cems[0])
        start = 17
    else:
        v = _set_bits(v, 13, 10, partition_index)
        if shared is None:
            shared = len(set(cems)) == 1
        if shared:
            v = _set_bits(v, 23, 6, cems[0] << 2)
        else:
            if offsets is None:
                base = min(2, min(c >> 2 for c in cems))
                offsets = [(c >> 2) - base for c in cems]
            else:
                base = (cems[0] >> 2) - offsets[0]
            assert all((c >> 2) - base == o for c, o in zip(cems, offsets)) and all(o in (0, 1) for o in offsets) and base <= 2, (cems, offsets)
            field = base + 1
            for i in range(partitions):
                field |= offsets[i] << (2 + i)
                field |= (cems[i] & 3) << (2 + partitions + 2 * i)
            extra = 3 * partitions - 4
            below -= extra
            v = _set_bits(v, 23, 6, field)
            v = _set_bits(v, below, extra, field >> 6)
        start = 29
    if wbits and bm[2]:
        below -= 2
        v = _set_bits(v, below, 2, ccs)
    if colour_fill is not None and below > start:
        v = _set_bits(v, start, below - start, -colour_fill)
    if weight_fill is not None and wbits:
        v = _set_bits(v, 128 - wbits, wbits, -weight_fill)
    if endpoint_values is not None:
        for i, x in enumerate(endpoint_values):
            v = _set_bits(v, 17 + 8 * i, 8, x)
    return np.frombuffer(v.to_bytes(16, "little"), np.uint8).copy()


def write_void_extent(rng, fp, hdr, extent, colour=None, reserved=3):
    """A void-extent block: extent = 4 (2D) or 6 (3D) coordinates (13 or 9 bits each), colour = four 16-bit values."""
    v = 0x1FC | (int(hdr) << 9)
    if fp[2] == 1:
        v |= (reserved & 3) << 10
        for i, x in enumerate(extent):
            v = _set_bits(v, 12 + 13 * i, 13, x)
    else:
        for i, x in enumerate(extent):
            v = _set_bits(v, 10 + 9 * i, 9, x)
    if colour is None:
        colour = [int(c) for c in rng.integers(0, 1 << 16, 4)]
    for i, c in enumerate(colour):
        v = _set_bits(v, 64 + 16 * i, 16, c)
    return np.frombuffer(v.to_bytes(16, "little"), np.uint8).copy()


def _random_f16(rng):
    """A random finite, non-negative half float (the bit pattern)."""
    return int(rng.integers(0, 0x7C00))


def _legal(block, fp):
    return parse(block, fp).legal


def _first(blocks_fn, fp, tries=64):
    """The first block blocks_fn(attempt) makes whose header is legal; None if none is."""
    for t in range(tries):
        b = blocks_fn(t)
        if b is not None and _legal(b, fp):
            return b
    return None


def random_cems(rng, p, first=None):
    """Endpoint modes of p partitions: `first` (default random) for the first, then either that mode in every partition or
    random modes of its class and an adjacent one (the class form)."""
    c0 = int(rng.integers(0, 16)) if first is None else first
    if p == 1 or rng.integers(0, 2) == 0:
        return [c0] * p
    base = min(2, max(0, (c0 >> 2) - int(rng.integers(0, 2))))
    return [c0] + [((base + int(rng.integers(0, 2))) << 2) | int(rng.integers(0, 4)) for _ in range(p - 1)]


def max_partitions(mode, fp):
    """The most partitions a block of this block mode can have: with endpoint mode 0 in every partition, the cheapest form."""
    rng = np.random.default_rng(0)
    for p in (4, 3, 2):
        if _legal(write_block(rng, fp, mode, partitions=p, cems=(0,)), fp):
            return p
    return 1


def block_set(fp, seed=1):
    """The deterministic decode test set of footprint fp: a list of (kind, block) pairs. Kinds name the section each block is for."""
    rng = np.random.default_rng(seed + 1000 * fp[0] + 100 * fp[1] + 10 * fp[2])
    out = []

    def add(kind, b):
        if b is not None:
            out.append((kind, b))

    modes = legal_block_modes(fp)
    one_plane = [m for m in modes if not block_mode(m, fp[2] > 1)[2]]
    dual_modes = [m for m in modes if block_mode(m, fp[2] > 1)[2]]
    by_wbits = sorted(one_plane, key=lambda m: (block_mode(m, fp[2] > 1)[4], m))
    cheap = by_wbits[0]                 # the most colour bits
    costly = by_wbits[-1]               # the fewest colour bits

    # every legal block mode: one partition with a random endpoint mode, and the most partitions the bits allow
    # (after eight tries with random endpoint modes, endpoint mode 0 everywhere: the fewest colour values)
    for m in modes:
        add("block_mode", _first(lambda t: write_block(rng, fp, m, cems=random_cems(rng, 1, None if t < 8 else 0),
                                                       ccs=int(rng.integers(0, 4))), fp))
        p = max_partitions(m, fp)
        if p > 1:
            add("block_mode", _first(lambda t: write_block(rng, fp, m, partitions=p, partition_index=int(rng.integers(0, 1024)),
                                                           cems=random_cems(rng, p, None if t < 8 else 0), ccs=int(rng.integers(0, 4))), fp))

    # every partition index of 2, 3 and 4 partitions, on block modes that allow that many
    for p in (2, 3, 4):
        fit = [m for m in one_plane if max_partitions(m, fp) >= p]
        for i in range(1024):
            m = fit[(i * 7) % len(fit)]
            add("partitioning", _first(lambda t: write_block(rng, fp, m, partitions=p, partition_index=i,
                                                             cems=random_cems(rng, p, None if t < 8 else 0)), fp))

    # every endpoint mode as the first partition's, with one to four partitions (after eight tries with random modes in the
    # other partitions, the cheapest: the class below, or class 0)
    for cem in range(16):
        for p in (1, 2, 3, 4):
            cheapest = [cem] + [max(0, (cem >> 2) - 1) << 2] * (p - 1)
            add("endpoint_mode", _first(lambda t: write_block(rng, fp, by_wbits[int(rng.integers(0, max(1, len(by_wbits) // 4)))], partitions=p,
                                                              partition_index=int(rng.integers(0, 1024)),
                                                              cems=random_cems(rng, p, cem) if t < 8 else cheapest), fp))
    # the class form: each class base, each partition's class offset
    for p in (2, 3, 4):
        for base in range(3):
            for pattern in range(1 << p):
                offsets = [(pattern >> i) & 1 for i in range(p)]
                cems = [((base + o) << 2) | int(rng.integers(0, 4)) for o in offsets]
                add("class_form", write_block(rng, fp, cheap, partitions=p, partition_index=int(rng.integers(0, 1024)), cems=cems,
                                              shared=False, offsets=offsets))
    # the HDR endpoint modes' sub-modes, on one-partition blocks whose endpoint values are stored as plain bytes (range 256)
    for cem in HDR_MODES:
        for label in hdr_submodes(cem):
            ev = _force_submode(cem, label, [int(x) for x in rng.integers(0, 256, 2 * ((cem >> 2) + 1))])
            assert hdr_submode(cem, ev) == label
            add("hdr_submode", write_block(rng, fp, cheap, cems=(cem,), endpoint_values=ev))

    # dual plane: each component selector, with one to three partitions
    for ccs in range(4):
        for p in (1, 2, 3):
            add("dual_plane", _first(lambda t: write_block(rng, fp, dual_modes[int(rng.integers(0, len(dual_modes)))], partitions=p,
                                                           partition_index=int(rng.integers(0, 1024)),
                                                           cems=random_cems(rng, p, None if t < 8 else 0), ccs=ccs), fp))

    # extreme payloads: all-zero and all-one colour and weight areas
    for m in (cheap, costly, dual_modes[0], dual_modes[-1]):
        for cf in (None, 0, 1):
            for wf in (None, 0, 1):
                if cf is None and wf is None:
                    continue
                add("extreme", _first(lambda t: write_block(rng, fp, m, cems=random_cems(rng, 1, None if t < 8 else 0),
                                                            ccs=int(rng.integers(0, 4)), colour_fill=cf, weight_fill=wf), fp))

    # void extents: LDR and HDR; valid, all-ones and invalid extents
    dims = 2 if fp[2] == 1 else 3
    top = 0x1FFF if dims == 2 else 0x1FF
    for hdr in (False, True):
        colour = (lambda: [_random_f16(rng) for _ in range(4)]) if hdr else (lambda: [int(x) for x in rng.integers(0, 1 << 16, 4)])
        for _ in range(3):
            ext = []
            for _ in range(dims):
                lo = int(rng.integers(0, top))
                ext += [lo, int(rng.integers(lo + 1, top + 1))]
            add("void_extent", write_void_extent(rng, fp, hdr, ext, colour()))
        add("void_extent", write_void_extent(rng, fp, hdr, [top] * (2 * dims), colour()))
        add("void_extent", write_void_extent(rng, fp, hdr, [top] * (2 * dims), [0xFFFF, 0, 0x8000, 0xFFFF] if not hdr else [0x3C00, 0, 0x7BFF, 0x3800]))
        if hdr:     # negative and NaN half floats: -NaN, -0, NaN, -65504
            add("void_extent", write_void_extent(rng, fp, hdr, [top] * (2 * dims), [0xFC01, 0x8000, 0x7E00, 0xFBFF]))
        for axis in range(dims):
            for equal in (True, False):
                ext = [0, top] * dims
                lo = int(rng.integers(1, top))
                ext[2 * axis], ext[2 * axis + 1] = (lo, lo) if equal else (lo, lo - 1)
                add("illegal", write_void_extent(rng, fp, hdr, ext, colour()))
        if dims == 2:
            for rsv in (0, 1, 2):
                add("illegal", write_void_extent(rng, fp, hdr, [0, top, 0, top], colour(), reserved=rsv))

    # illegal blocks: each rule, alone where the footprint allows
    for rule in BLOCK_MODE_RULES:
        alone = [m for m in range(2048) if m & 0x1FF != 0x1FC and block_mode_rules(m, fp) == [rule]]
        some = alone or [m for m in range(2048) if m & 0x1FF != 0x1FC and rule in block_mode_rules(m, fp)]
        for m in [some[int(k)] for k in rng.choice(len(some), min(4, len(some)), replace=False)] if some else []:
            add("illegal", write_block(rng, fp, m, partitions=int(rng.integers(1, 4)), partition_index=int(rng.integers(0, 1024)),
                                       cems=(int(rng.integers(0, 4)),)))
    for m in dual_modes[:2] + dual_modes[-2:]:
        add("illegal", write_block(rng, fp, m, partitions=4, partition_index=int(rng.integers(0, 1024)), cems=(0,)))
    for cems in ((15, 15, 15), (12, 13, 8), (8, 8, 8, 8), (11, 11, 7, 7), (15, 11, 11, 11)):
        add("illegal", write_block(rng, fp, cheap, partitions=len(cems), partition_index=int(rng.integers(0, 1024)), cems=cems))
    for cem in (15, 12, 8, 4):
        for m in by_wbits[-8:]:
            b = write_block(rng, fp, m, cems=(cem,))
            if parse(b, fp).rules == ["colour_bits_insufficient"]:
                add("illegal", b)
                break
        for m in by_wbits[-8:]:
            b = write_block(rng, fp, m, partitions=2, partition_index=int(rng.integers(0, 1024)), cems=(cem, cem))
            if parse(b, fp).rules == ["colour_bits_insufficient"]:
                add("illegal", b)
                break
    return out


def _force_submode(cem, label, ev):
    """Set the sub-mode bits of endpoint values ev to those of `label` (the inverse of hdr_submode)."""
    ev = list(ev)

    def bit7(i, b):
        ev[i] = (ev[i] & 0x7F) | (b << 7)
    if cem == 2:
        lo, hi = sorted(ev[:2])
        if lo == hi:
            lo, hi = (lo - 1, lo) if lo else (0, 1)
        ev[:2] = [lo, hi] if label == "ordered" else [hi, lo]
    elif cem == 3:
        bit7(0, int(label[-1]))
    elif cem == 7:
        mv = int(label[len("modeval"):])
        ev[0] = (ev[0] & 0x3F) | ((mv & 3) << 6)
        bit7(1, (mv >> 2) & 1)
        bit7(2, (mv >> 3) & 1)
    elif cem in (11, 14, 15):
        rgb = label.split(".alpha")[0]
        if rgb == "direct":
            bit7(4, 1)
            bit7(5, 1)
        else:
            major, mode = int(rgb[5]), int(rgb.split("mode")[1])
            bit7(4, major & 1)
            bit7(5, major >> 1)
            for k in range(3):
                bit7(1 + k, (mode >> k) & 1)
        if cem == 15:
            a = int(label.split(".alpha")[1])
            bit7(6, a & 1)
            bit7(7, a >> 1)
    return ev


Mosaic = collections.namedtuple("Mosaic", "blocks dims index whole kinds set_blocks")


@functools.lru_cache(maxsize=None)
def mosaic(fp):
    """The footprint's set laid out as an image. Mosaic fields: blocks (the image's blocks, a flat uint8 array), dims (w, h, d),
    index (the set block each image block is), whole (the image block lies inside the image), kinds and set_blocks (the set).

    The set fills all but the last block column and row (and, in 3D, layer); those are ragged, partly outside the image,
    and repeat blocks of the set, so every set block is decoded whole and the edge handling is exercised too."""
    entries = block_set(fp)
    n = len(entries)
    bx, by, bz = fp
    layers = 3 if bz > 1 else 1
    cols = int(np.ceil(np.sqrt(n / layers * by / bx)))
    rows = -(-n // (cols * layers))
    nbx, nby, nbz = cols + 1, rows + 1, (layers + 1 if bz > 1 else 1)
    w, h = cols * bx + (bx + 1) // 2, rows * by + (by + 1) // 2
    d = layers * bz + (bz + 1) // 2 if bz > 1 else 1
    grid = np.zeros((nbz, nby, nbx, 16), np.uint8)
    index = np.zeros((nbz, nby, nbx), np.int64)
    whole = np.zeros((nbz, nby, nbx), bool)
    k = 0
    for z in range(nbz):
        for y in range(nby):
            for x in range(nbx):
                whole[z, y, x] = x < cols and y < rows and (z < layers or bz == 1)
                if whole[z, y, x] and k < n:
                    index[z, y, x] = k
                    k += 1
                else:
                    index[z, y, x] = (x * 31 + y * 17 + z * 7) % n
                grid[z, y, x] = entries[index[z, y, x]][1]
    assert k == n
    return Mosaic(grid.reshape(-1), (w, h, d), index.reshape(-1), whole.reshape(-1), [e[0] for e in entries], [e[1] for e in entries])
