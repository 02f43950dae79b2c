"""Generates tests/golden/golden_endpoints.npz from the UNMODIFIED reference build (oracle/_ref): endpoint packing fixtures.

sweep() is the input set, a seeded, deterministic function of this file that tests/test_endpoint_pack.py imports: for every
input format the search hands pack_color_endpoints (LDR 0, 4, 6, 8, 10, 12; HDR 2, 3, 7, 11, 14, 15) and every colour quant
level QUANT_6 .. QUANT_256, boundary vectors (the edges of each encoding's value ranges, rounding ties, tied components,
out-of-range finite values) and random vectors drawn inside each HDR sub-mode's ranges. No NaN or infinity: the packers'
behaviour on those is undefined (f2i_rtn gives INT_MIN and the table look-ups leave the table).

Stored per vector: the format the reference returned and the 8 output bytes (the buffer starts as SENTINEL, so bytes the
format does not define stay SENTINEL); plus the SHA-256 of the generated inputs, so that a change of the generator shows as
"inputs changed" rather than as a packer mismatch. Run it with the reference build in place (oracle/Makefile `ref`)."""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from astc_ref import ref_pack_color_endpoints  # noqa: E402

OUT = os.path.join(HERE, "golden_endpoints.npz")

LDR_FORMATS = (0, 4, 6, 8, 10, 12)
HDR_FORMATS = (2, 3, 7, 11, 14, 15)
FORMATS = LDR_FORMATS + HDR_FORMATS
QUANT_6, QUANT_160, QUANT_256 = 4, 18, 20
QUANT_LEVELS = tuple(range(QUANT_6, QUANT_256 + 1))
SENTINEL = 0xA5
N_RANDOM = 96           # random vectors per (format, quant level)

# HDR RGB + offset (format 7), sub-modes 0..4: scale shift, width of the difference / offset fields, log2 of the value
# ranges of the differences and of the offset (the format's definition of each sub-mode)
RGBO_MODES = [(5, 5, 7, 10, 12), (5, 6, 5, 11, 10), (6, 5, 8, 11, 14), (7, 6, 7, 13, 14), (8, 7, 6, 15, 14)]
# HDR RGB (formats 11, 14, 15), sub-modes 0..7: scale shift, widths of the b / c / d fields, log2 of the ranges of b, c, d
RGB_MODES = [(7, 7, 6, 7, 14, 13, 13), (7, 8, 6, 6, 15, 13, 12), (6, 6, 7, 7, 12, 13, 12), (6, 7, 7, 6, 13, 13, 11),
             (5, 8, 6, 5, 13, 11, 9), (5, 6, 8, 6, 11, 13, 10), (4, 7, 7, 5, 11, 11, 8), (4, 6, 7, 6, 10, 11, 9)]


def _perm(v, major):
    """(major, other1, other2) -> (r, g, b) with the major value in component `major`."""
    m, o1, o2 = v
    return [(m, o1, o2), (o1, m, o2), (o2, o1, m)][major]


class _Set:
    def __init__(self):
        self.rows, self.boundary = [], []

    def add(self, c0, c1, rgbs=(0, 0, 0, 0), rgbo=(0, 0, 0, 0), boundary=True):
        self.rows.append(list(c0) + list(c1) + list(rgbs) + list(rgbo))
        self.boundary.append(boundary)


def _ldr_boundary(s):
    k = np.arange(0, 256, 17)
    # endpoints at 0 / 65535, 257 k +- eps, the .5 ties of the /257 scaling and the -0.1 residual edge of quant_color_f
    for e in (0.0, 0.5, -0.5, 1.0, -1.0, 128.5, -25.7, -26.0, 1e-3):
        for kk in k:
            v = 257.0 * kk + e
            s.add((v, v, v, v), (65535 - v, v + 257, 65535 - v, 65535 - v), (v, v, v, kk / 255.0), (v, v, v, v))
    s.add((0, 0, 0, 0), (65535, 65535, 65535, 65535), (0, 0, 0, 0), (0, 0, 0, 0))
    s.add((65535, 65535, 65535, 65535), (0, 0, 0, 0), (65535, 65535, 65535, 1), (0, 0, 0, 0))
    # out-of-range finite values
    for a, b in ((-1.0, 70000.0), (-1e6, 1e6), (65536.0, -0.5), (1e6, 1e6), (-3.0, -7.0)):
        s.add((a, b, a, b), (b, a, b, a), (a, b, a, 1.5), (a, b, a, b))
    # luminance / alpha deltas of +-63 / -64 after the x2 to unorm9 (deltas of +-31.5 .. 32.5 in unorm8)
    for base in (10.0, 100.0, 127.5, 200.0, 230.0):
        for d in (-32.5, -32.0, -31.75, -31.5, -31.0, 31.0, 31.5, 31.75, 32.0, 32.5):
            b0, b1 = base * 257.0, (base + d) * 257.0
            s.add((b0, b0, b0, b0), (b1, b1, b1, b1))
            s.add((b0, b0, b0, b1), (b1, b1, b1, b0))
            s.add((b0, b1, b0, b0), (b1, b0, b1, b1))
    # blue contraction: c + (c - b) at 0 and at 255 (unorm8), one step inside and outside
    for b in (0.0, 30.0, 100.0, 254.0, 255.0):
        for edge in (b / 2.0, (b + 255.0) / 2.0):
            for e in (-0.5, -0.25, 0.0, 0.25, 0.5):
                r = (edge + e) * 257.0
                s.add((r, r, b * 257.0, 128 * 257.0), (r + 257.0, r + 514.0, b * 257.0 + 771.0, 100 * 257.0))
                s.add((r + 257.0, r + 514.0, b * 257.0 + 771.0, 5000.0), (r, r, b * 257.0, 60000.0))
    # a tie of the contest: identical endpoints (every encoding reproduces them exactly at QUANT_256)
    for v in (0.0, 257.0 * 64, 257.0 * 200, 65535.0):
        s.add((v, v, v, v), (v, v, v, v), (v, v, v, 1.0), (v, v, v, 0.0))
    # lum1 < lum0 (luminance averages the pair)
    for a, b in ((40000.0, 20000.0), (300.0, 299.0), (65535.0, 0.0)):
        s.add((a, a, a, a), (b, b, b, b))
    # the scale of RGBS: 0, 1, beyond, and colours whose sum quantises away
    for sc in (0.0, 1e-6, 0.5, 0.998, 1.0, 1.001, 3.0, -0.5):
        for c in ((0.0, 0.0, 0.0), (128.5 * 257, 0.2, 64.5 * 257), (65535.0, 65535.0, 65535.0), (100.0, 200.0, 300.0)):
            s.add(c + (sc,), c + (1.0,), c + (sc,), c + (sc,))


def _ldr_random(s, rng, n):
    for _ in range(n):
        kind = rng.integers(0, 4)
        c0 = rng.uniform(0, 65535, 4)
        if kind == 0:      # a close pair (the offset encodings)
            c1 = np.clip(c0 + rng.uniform(-40, 40, 4) * 257.0, -300, 66000)
        elif kind == 1:    # a close pair in a blue-contractible region (r, g near (b .. b + 255) / 2)
            b0 = rng.uniform(0, 255)
            c0 = np.array([rng.uniform(b0 / 2, (b0 + 255) / 2), rng.uniform(b0 / 2, (b0 + 255) / 2), b0, rng.uniform(0, 255)]) * 257.0
            c1 = np.clip(c0 + rng.uniform(-30, 30, 4) * 257.0, 0, 65535)
        elif kind == 2:    # a grey pair (luminance formats)
            l0, l1 = rng.uniform(0, 65535, 2)
            c0 = np.array([l0, l0, l0, rng.uniform(0, 65535)]) + rng.uniform(-300, 300, 4)
            c1 = np.array([l1, l1, l1, rng.uniform(0, 65535)]) + rng.uniform(-300, 300, 4)
        else:
            c1 = rng.uniform(0, 65535, 4)
        rgbs = list(rng.uniform(0, 65535, 3)) + [rng.uniform(0, 1.0)]
        s.add(c0, c1, rgbs, (0, 0, 0, 0), boundary=False)


def _rgbo_vec(s, major, m, d1, d2, off, boundary):
    """An HDR RGB + offset input with the major component value m (after the offset is added), differences d1, d2, offset off."""
    col = _perm((m, m - d1, m - d2), major)
    s.add((0, 0, 0, 0), (0, 0, 0, 0), (0, 0, 0, 0), (col[0] - off, col[1] - off, col[2] - off, off), boundary)


def _hdr_rgbo(s, rng, n):
    for mode, (sh, gb, sb, cut0, cut1) in enumerate(RGBO_MODES):
        dlim, slim = min(1 << cut0, (1 << (sh + gb)) - 1), min(1 << cut1, (1 << (sh + sb)) - 1)
        for major in range(3):
            for d in ((1 << cut0) - 1, 1 << cut0, (1 << cut0) + 0.5, (1 << cut0) + 1,
                      (1 << (sh + gb)) - (1 << (sh - 1)) - 1, (1 << (sh + gb)) - (1 << (sh - 1)), (1 << (sh + gb)) - (1 << (sh - 1)) + 1):
                for m in (60000.0, 65535.0, 40000.0 + 17 * (1 << sh) + (1 << (sh - 1))):
                    _rgbo_vec(s, major, m, d, d / 2, 3.0, True)
                    _rgbo_vec(s, major, m, d / 3, d, 3.0, True)
            for off in ((1 << cut1) - 1, 1 << cut1, (1 << cut1) + 1, (1 << (sh + sb)) - (1 << (sh - 1)), (1 << (sh + sb)) - (1 << (sh - 1)) - 1):
                _rgbo_vec(s, major, 50000.0, dlim / 4, dlim / 8, off, True)
        for _ in range(n // 6):
            major = int(rng.integers(0, 3))
            _rgbo_vec(s, major, rng.uniform(dlim, 65535), rng.uniform(0, dlim), rng.uniform(0, dlim), rng.uniform(0, slim), False)
    # tied components (majcomp selection), the flat form, values beyond the range
    for m in (1000.0, 30000.0, 65535.0):
        for col in ((m, m, m - 10), (m - 10, m, m), (m, m - 10, m), (m, m, m)):
            s.add((0,) * 4, (0,) * 4, (0,) * 4, col + (5.0,))
    for col in ((65535.0, 0.0, 0.0, 0.0), (65535.0, 1.0, 30000.0, 40000.0), (-5.0, 70000.0, 1e6, -1e6), (512.0 * 100 + 256, 256.0, 768.0, 512.0 * 3 + 256)):
        s.add((0,) * 4, (0,) * 4, (0,) * 4, col)
    for _ in range(n // 6):
        s.add((0,) * 4, (0,) * 4, (0,) * 4, list(rng.uniform(-1000, 70000, 3)) + [rng.uniform(0, 70000)], False)


def _rgb_vec(s, major, a, b0, b1, c, d0, d1, alpha, boundary):
    """An HDR RGB input from the format's quantities: a = major of endpoint 1, b = its distances to endpoint 1's other
    components, c = distance to endpoint 0's major, d = what is left for endpoint 0's other components."""
    e1 = _perm((a, a - b0, a - b1), major)
    e0 = _perm((a - c, a - b0 - c - d0, a - b1 - c - d1), major)
    s.add(tuple(e0) + (alpha[0],), tuple(e1) + (alpha[1],), (0, 0, 0, 0), (0, 0, 0, 0), boundary)


def _alpha_pairs():
    """HDR alpha pairs at each precision level's edges: differences at +-cutoff in units of 1 << (8 - i), .5 ties of the shift."""
    out = [(0.0, 0.0), (65280.0, 65280.0), (65535.0, 0.0), (0.0, 65535.0), (-5.0, 70000.0), (1e6, -1e6)]
    for i in range(3):
        unit, cutoff = 1 << (8 - i), 32 >> i
        for base in (1000.0, 30000.0, 60000.0):
            for k in (-cutoff - 1, -cutoff, -cutoff + 1, cutoff - 1, cutoff, cutoff + 1):
                for e in (0.0, unit / 2.0, -unit / 2.0 - 0.5):
                    out.append((base, base + k * unit + e))
    return out


def _hdr_rgb(s, rng, n, fmt):
    alphas = _alpha_pairs()
    ai = 0
    for mode, (sh, bb, cb, db, cutb, cutc, cutd) in enumerate(RGB_MODES):
        bl, cl, dl = min(1 << cutb, (1 << (sh + bb)) - 1), min(1 << cutc, (1 << (sh + cb)) - 1), min(1 << cutd, (1 << (sh + db - 1)) - 1)
        for major in range(3):
            edges = []
            for cut, lim in ((cutb, bb), (cutc, cb)):
                edges.append([(1 << cut) - 1, 1 << cut, (1 << cut) + 1, (1 << (sh + lim)) - (1 << (sh - 1)), (1 << (sh + lim)) - (1 << (sh - 1)) - 1])
            dedge = [(1 << cutd) - 1, 1 << cutd, (1 << cutd) + 1, (1 << (sh + db - 1)) - (1 << (sh - 1)), (1 << (sh + db - 1)) - (1 << (sh - 1)) - 1]
            for a in (65535.0, 50000.0 + 3 * (1 << sh) + (1 << (sh - 1))):
                for b in edges[0]:
                    _rgb_vec(s, major, a, b, bl / 3, cl / 3, 0, 0, alphas[ai % len(alphas)], True)
                    ai += 1
                for c in edges[1]:
                    _rgb_vec(s, major, a, bl / 3, bl / 5, c, 0, 0, alphas[ai % len(alphas)], True)
                    ai += 1
                for d in dedge:
                    for sg in (1, -1):
                        _rgb_vec(s, major, a, bl / 3, bl / 5, cl / 3, sg * d, -sg * d / 2, alphas[ai % len(alphas)], True)
                        ai += 1
        for _ in range(n // 9):
            major = int(rng.integers(0, 3))
            a = rng.uniform(bl + cl + dl, 65535)
            _rgb_vec(s, major, a, rng.uniform(0, bl), rng.uniform(0, bl), rng.uniform(0, cl), rng.uniform(-dl, dl), rng.uniform(-dl, dl),
                     (rng.uniform(0, 65535), rng.uniform(0, 65535)), False)
    # tied majors, the flat form (/256 and /512 ties), values beyond the range
    for m in (2000.0, 40000.0, 65535.0):
        for col in ((m, m, m - 10), (m - 10, m, m), (m, m - 10, m), (m, m, m)):
            s.add((m - 600, m - 700, m - 800, 100.0), col + (200.0,))
    for c0, c1 in (((0.0, 65535.0, 0.0, 0.0), (65535.0, 0.0, 65535.0, 65535.0)), ((256.0 * 7 + 128, 512.0 * 9 + 256, 512.0 * 3 + 256, 1.0), (256.0 * 200 + 128, 256.0 * 3 + 128, 512.0 * 90 + 256, 2.0)),
                   ((-5.0, 70000.0, 1e6, -1e6), (1e6, -1e6, 3.0, 70000.0)), ((65535.0,) * 4, (0.0,) * 4)):
        s.add(c0, c1)
    for a0, a1 in alphas:
        s.add((1000.0, 2000.0, 3000.0, a0), (40000.0, 41000.0, 42000.0, a1))
    for _ in range(n // 9):
        s.add(list(rng.uniform(-1000, 70000, 4)), list(rng.uniform(-1000, 70000, 4)), boundary=False)
    if fmt == 14:      # LDR alpha beside the HDR colour: the /257 ties
        for kk in (0, 1, 100, 254, 255):
            for e in (0.0, 128.5, -128.5, -25.7):
                s.add((1000.0, 2000.0, 3000.0, 257.0 * kk + e), (40000.0, 41000.0, 42000.0, 257.0 * (255 - kk) - e))


def _lum_vec(s, l0, l1, boundary=True, spread=0.0):
    s.add((l0 - spread, l0, l0 + spread, 0.0), (l1 + spread, l1, l1 - spread, 0.0), (0, 0, 0, 0), (0, 0, 0, 0), boundary)


def _hdr_lum(s, rng, n):
    for l0 in (0.0, 1000.0, 16.0 * 7, 32.0 * 100 + 16, 30000.0, 64000.0, 65535.0 - 2049):
        for d in (0, 15, 16, 31, 32 * 15 - 1, 32 * 15, 32 * 15 + 16, 64 * 31 - 1, 64 * 31, 64 * 31 + 32, 2047, 2048, 2049, 2050, 5000):
            _lum_vec(s, l0, l0 + d)
        _lum_vec(s, l0 + 500, l0)     # lum1 < lum0: both take the average
    for l0, l1 in ((65535.0, 65535.0), (-50.0, 80000.0), (1e6, -1e6), (65280.0, 65535.0), (127.5, 128.5), (255.5, 256.5), (65407.5, 65535.0)):
        _lum_vec(s, l0, l1)
    for i in range(n):
        l0 = rng.uniform(0, 65535)
        d = [rng.uniform(0, 480), rng.uniform(0, 1984), rng.uniform(0, 2100), rng.uniform(-2000, 30000)][i % 4]
        _lum_vec(s, l0, l0 + d, False, rng.uniform(0, 200))


def sweep():
    """The input vectors: (colors float32 (n, 16), fmt_quant int32 (n, 2), boundary bool (n,))."""
    colors, fq, boundary = [], [], []
    for fmt in FORMATS:
        for q in QUANT_LEVELS:
            rng = np.random.default_rng(1000 * fmt + q)
            s = _Set()
            if fmt in LDR_FORMATS:
                _ldr_boundary(s)
                _ldr_random(s, rng, N_RANDOM)
            elif fmt == 7:
                _hdr_rgbo(s, rng, N_RANDOM * 2)
            elif fmt in (2, 3):
                _hdr_lum(s, rng, N_RANDOM)
            else:
                _hdr_rgb(s, rng, N_RANDOM * 2, fmt)
            colors.append(np.array(s.rows, dtype=np.float32))
            fq.append(np.tile(np.array([[fmt, q]], dtype=np.int32), (len(s.rows), 1)))
            boundary.append(np.array(s.boundary, dtype=bool))
    colors = np.ascontiguousarray(np.concatenate(colors))
    assert np.isfinite(colors).all()
    return colors, np.ascontiguousarray(np.concatenate(fq)), np.concatenate(boundary)


def inputs_sha256(colors, fmt_quant):
    h = hashlib.sha256()
    h.update(np.ascontiguousarray(colors, dtype="<f4").tobytes())
    h.update(np.ascontiguousarray(fmt_quant, dtype="<i4").tobytes())
    return h.hexdigest()


def run_packer(fn, colors, fmt_quant):
    """Call one of the C entry points with the signature fn(n, colors, fmt_quant, out, out_format) -> (formats, bytes (n, 8))."""
    n = len(colors)
    out = np.full((n, 8), SENTINEL, dtype=np.uint8)
    fmts = np.zeros(n, dtype=np.uint8)
    fn(n, colors.ctypes.data, fmt_quant.ctypes.data, out.ctypes.data, fmts.ctypes.data)
    return fmts, out


def main():
    colors, fq, _ = sweep()
    fmts, out = run_packer(ref_pack_color_endpoints(), colors, fq)
    np.savez_compressed(OUT, formats=fmts, bytes=out, inputs_sha256=np.array(inputs_sha256(colors, fq)))
    print(len(colors), "vectors ->", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    sys.exit(main())
