"""Endpoint packing: every form of the device's pack_color_endpoints against the reference's, vector by vector.

The encoder's last step for every candidate turns two float endpoints into the colour bytes of the block, and the search
scores the decoded bytes, so a wrong packer also changes which candidate wins. The device restates the reference's serial
code in four forms (astc_dev_color.cuh, astc_dev_color_hdr_pack.cuh), each reading color_unquant_to_uquant from global
memory or from a copy staged in shared memory:
    serial     pack_color_endpoints, one vector per lane (LDR formats of multi-partition candidates)
    coop       pack_rgb_endpoints_coop: the RGB / RGBA contest of four encodings on four lanes
    coop_inl   pack_rgb_endpoints_coop_t<true>, the same inlined (one-partition LDR set-up and refinement)
    hdr        pack_hdr_endpoints: the HDR sub-mode ladders, one attempt per lane
The inputs are tests/golden/make_golden_endpoints.sweep(); the reference's answers are stored in golden_endpoints.npz.

CPU: the oracle's restatement, the device source on the host (tests/hostsim/hostsim_endpoints.cpp, one simulated lane and
32 lanes) and - where oracle/_ref was built - the live reference, all against the fixture; the sweep's coverage of the
encodings and HDR sub-modes; the harnesses refuse inputs the packers do not define.
GPU: the device source on the H100 (tests/devunit/pack_endpoints.cu, libastc_devunit.so) against the fixture."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_endpoints as G  # noqa: E402
import astc_blockgen as B  # noqa: E402
from astc_ref import ORACLE_SO, have_ref_pack, ref_pack_color_endpoints  # noqa: E402
from hostsim_build import host_sim  # noqa: E402

VARIANTS = {"serial": 0, "coop": 1, "coop_inl": 2, "hdr": 3}
VARIANT_FORMATS = {"serial": G.LDR_FORMATS, "coop": (8, 12), "coop_inl": (8, 12), "hdr": G.HDR_FORMATS}
PLACEMENTS = {"global": 0, "staged": 1}
DEVUNIT_SO = os.path.join(ROOT, "astc-encoder_b200", "libastc_devunit.so")
_ARGS = [C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]


@pytest.fixture(scope="module")
def sweep():
    colors, fq, boundary = G.sweep()
    z = np.load(G.OUT)
    assert str(z["inputs_sha256"]) == G.inputs_sha256(colors, fq), \
        "inputs changed: make_golden_endpoints.sweep() no longer generates the inputs golden_endpoints.npz was recorded from"
    return colors, fq, boundary, z["formats"], z["bytes"]


def _compare(got_fmt, got_bytes, want_fmt, want_bytes, colors, fq, what):
    bad = np.nonzero((got_fmt != want_fmt) | (got_bytes != want_bytes).any(axis=1))[0]
    if len(bad):
        lines = []
        for i in bad[:8]:
            lines.append("format %d quant %d in %s: got format %d %s, reference format %d %s" % (
                fq[i, 0], fq[i, 1], np.array2string(colors[i], precision=9, max_line_width=400), got_fmt[i], got_bytes[i].tolist(),
                want_fmt[i], want_bytes[i].tolist()))
        pytest.fail("%s: %d of %d vectors differ from the reference\n%s" % (what, len(bad), len(want_fmt), "\n".join(lines)))


def _select(sweep, variant, subset=None):
    colors, fq, boundary, want_fmt, want_bytes = sweep
    sel = np.isin(fq[:, 0], VARIANT_FORMATS[variant])
    if subset is not None:
        sel &= subset
    return (np.ascontiguousarray(colors[sel]), np.ascontiguousarray(fq[sel]), want_fmt[sel], want_bytes[sel])


def test_fixture_sentinel(sweep):
    """The reference writes exactly the bytes of the format it returns: 2, 4, 6 or 8 by the format's class."""
    _, fq, _, fmts, out = sweep
    assert len(fmts) == len(fq)
    n_defined = 2 * ((fmts.astype(int) >> 2) + 1)
    for nb in (2, 4, 6, 8):
        rows = out[n_defined == nb]
        assert (rows[:, nb:] == G.SENTINEL).all()


# ---- oracle (oracle/astc_color.h, astc_color_hdr_pack.inl) ---------------------------------------------------------------
def test_oracle_vs_fixture(sweep):
    colors, fq, _, want_fmt, want_bytes = sweep
    lib = C.CDLL(ORACLE_SO)
    lib.oracle_pack_color_endpoints.argtypes = _ARGS
    lib.oracle_pack_color_endpoints.restype = None
    got_fmt, got_bytes = G.run_packer(lib.oracle_pack_color_endpoints, colors, fq)
    _compare(got_fmt, got_bytes, want_fmt, want_bytes, colors, fq, "oracle")


@pytest.mark.skipif(not have_ref_pack(), reason="oracle/_ref/libastcenc_ref_pack.so not built (no reference sources)")
def test_live_reference_vs_fixture(sweep):
    colors, fq, _, want_fmt, want_bytes = sweep
    got_fmt, got_bytes = G.run_packer(ref_pack_color_endpoints(), colors, fq)
    _compare(got_fmt, got_bytes, want_fmt, want_bytes, colors, fq, "reference build")


# ---- the device source on the host ---------------------------------------------------------------------------------------
_SIMS = {}


def endpoints_sim(lanes32=False):
    """tests/hostsim/hostsim_endpoints.cpp compiled for the host (one simulated lane, or 32 lanes on 32 threads)."""
    if lanes32 in _SIMS:
        return _SIMS[lanes32]
    lib = host_sim("hostsim_endpoints", lanes32)
    lib.hostsim_pack_endpoints.argtypes = [C.c_int, C.c_int] + _ARGS
    lib.hostsim_pack_endpoints.restype = C.c_int
    _SIMS[lanes32] = lib
    return lib


def _run(fn, variant, placement, colors, fq):
    n = len(colors)
    out = np.full((n, 8), G.SENTINEL, dtype=np.uint8)
    fmts = np.zeros(n, dtype=np.uint8)
    rc = fn(VARIANTS[variant], PLACEMENTS[placement], n, colors.ctypes.data, fq.ctypes.data, out.ctypes.data, fmts.ctypes.data)
    return rc, fmts, out


def _lanes32_subset(boundary):
    """The 32-lane build runs every boundary vector and every 8th random one (it is slow: a collective is a thread barrier)."""
    return boundary | (np.cumsum(~boundary) % 8 == 0)


@pytest.mark.parametrize("placement", sorted(PLACEMENTS))
@pytest.mark.parametrize("variant", sorted(VARIANTS))
@pytest.mark.parametrize("lanes32", [False, True], ids=["lanes1", "lanes32"])
def test_hostsim_vs_fixture(sweep, lanes32, variant, placement):
    colors, fq, want_fmt, want_bytes = _select(sweep, variant, _lanes32_subset(sweep[2]) if lanes32 else None)
    rc, got_fmt, got_bytes = _run(endpoints_sim(lanes32).hostsim_pack_endpoints, variant, placement, colors, fq)
    assert rc == 0
    _compare(got_fmt, got_bytes, want_fmt, want_bytes, colors, fq, "host simulation (%s lanes) %s, %s table" % (32 if lanes32 else 1, variant, placement))


# ---- the harnesses refuse what the packers do not define -----------------------------------------------------------------
def _bad_inputs():
    ok_c = np.full((1, 16), 1000.0, dtype=np.float32)
    cases = []
    for bad in (np.nan, np.inf, -np.inf):
        c = ok_c.copy()
        c[0, 5] = bad
        cases.append(("serial", c, (8, 10)))
        cases.append(("hdr", c, (11, 10)))
    cases += [("serial", ok_c, (8, 3)), ("serial", ok_c, (8, 21)), ("coop", ok_c, (12, -1)), ("hdr", ok_c, (7, 21)),
              ("serial", ok_c, (1, 10)), ("serial", ok_c, (11, 10)), ("coop", ok_c, (4, 10)), ("coop_inl", ok_c, (13, 10)),
              ("hdr", ok_c, (8, 10)), ("hdr", ok_c, (16, 10))]
    return cases


def _check_refusals(fn):
    for variant, c, (fmt, q) in _bad_inputs():
        fq = np.array([[fmt, q]], dtype=np.int32)
        rc, fmts, out = _run(fn, variant, "staged", np.ascontiguousarray(c), fq)
        assert rc == 1, (variant, c, fmt, q)
        assert (out == G.SENTINEL).all() and (fmts == 0).all()
    # one bad vector refuses the whole call
    colors, fq = np.full((3, 16), 1000.0, dtype=np.float32), np.array([[8, 10], [8, 10], [8, 10]], dtype=np.int32)
    colors[2, 0] = np.nan
    assert _run(fn, "coop", "global", colors, fq)[0] == 1
    assert fn(7, 0, 1, colors.ctypes.data, fq.ctypes.data, None, None) == 1


@pytest.mark.parametrize("lanes32", [False, True], ids=["lanes1", "lanes32"])
def test_hostsim_refuses_undefined_inputs(lanes32):
    _check_refusals(endpoints_sim(lanes32).hostsim_pack_endpoints)


# ---- coverage of the sweep -----------------------------------------------------------------------------------------------
RGB_ENCODINGS = ("delta_bc", "delta", "bc", "plain")


def ldr_rgb_encoding(fmt, ev):
    """Which of the four RGB / RGBA encodings the bytes ev of returned format fmt (8, 9, 12, 13) are: the decoder's test."""
    if fmt in (9, 13):
        d = [(ev[2 * i + 1] >> 1) & 0x3F for i in range(3)]
        d = [x - 0x40 if x & 0x20 else x for x in d]
        return "delta_bc" if sum(d) < 0 else "delta"
    return "bc" if ev[0] + ev[2] + ev[4] > ev[1] + ev[3] + ev[5] else "plain"


def coverage(fq, fmts, out):
    """{(input format, quant level): set of labels reached}. HDR: hdr_submode() of the returned format ("<cem>:<label>";
    format 15 also as its RGB and alpha parts); RGB / RGBA: the encoding; LA: "delta" when the delta form was returned."""
    cov = {}
    for (fin, q), f, ev in zip(fq.tolist(), fmts.tolist(), out.tolist()):
        labels = cov.setdefault((fin, q), set())
        if f in (2, 3, 7, 11, 14, 15):
            lab = B.hdr_submode(f, ev)
            labels.add("%d:%s" % (f, lab))
            if f == 15:
                rgb, alpha = lab.rsplit(".", 1)
                labels.add("15:" + rgb)
                labels.add("15:" + alpha)
        elif f in (8, 9, 12, 13):
            labels.add(ldr_rgb_encoding(f, ev))
        elif f == 5:
            labels.add("delta")
    return cov


# Labels the packers cannot produce, with the reason
UNREACHABLE = {}


def test_sweep_coverage(sweep):
    _, fq, _, fmts, out = sweep
    cov = coverage(fq, fmts, out)
    missing = []

    def need(key, labels):
        for lab in labels:
            if lab not in cov.get(key, ()) and (key, lab) not in UNREACHABLE:
                missing.append("%s: %s" % (key, lab))

    top = G.QUANT_256
    need((2, top), ["2:%s" % l for l in B.hdr_submodes(2)] + ["3:%s" % l for l in B.hdr_submodes(3)])
    need((3, top), ["2:%s" % l for l in B.hdr_submodes(2)] + ["3:%s" % l for l in B.hdr_submodes(3)])
    for cem in (7, 11, 14):
        need((cem, top), ["%d:%s" % (cem, l) for l in B.hdr_submodes(cem)])
    need((15, top), ["15:%s" % l for l in B.hdr_submodes(11)] + ["15:alpha%d" % a for a in range(4)])
    for q in range(G.QUANT_6, G.QUANT_160 + 1):
        need((8, q), RGB_ENCODINGS)
        need((12, q), RGB_ENCODINGS)
        need((4, q), ["delta"])
    assert not missing, "labels the sweep does not reach:\n" + "\n".join(missing)
    # above QUANT_160 the offset forms are not tried, at QUANT_256 the blue-contracted plain form is not either
    for q in (G.QUANT_160 + 1, G.QUANT_256):
        for f in (8, 12):
            assert not cov[(f, q)] & {"delta", "delta_bc"}
        assert "delta" not in cov[(4, q)]
    assert not cov[(8, G.QUANT_256)] & {"bc"}


# ---- the device source on the GPU ----------------------------------------------------------------------------------------
def devunit():
    """libastc_devunit.so, rebuilt when it is older than its sources (make decides)."""
    r = subprocess.run(["make", "-C", os.path.join(ROOT, "astc-encoder_b200"), "devunit"], capture_output=True, text=True)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    lib = C.CDLL(DEVUNIT_SO, mode=os.RTLD_LOCAL)
    lib.devunit_pack_endpoints.argtypes = [C.c_int, C.c_int] + _ARGS
    lib.devunit_pack_endpoints.restype = C.c_int
    lib.devunit_last_error.restype = C.c_char_p
    return lib


def test_devunit_refuses_undefined_inputs():
    """The GPU harness checks its inputs on the host, before any CUDA call: no GPU needed."""
    _check_refusals(devunit().devunit_pack_endpoints)


@pytest.mark.gpu
@pytest.mark.parametrize("placement", sorted(PLACEMENTS))
@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_gpu_vs_fixture(sweep, variant, placement):
    lib = devunit()
    colors, fq, want_fmt, want_bytes = _select(sweep, variant)
    rc, got_fmt, got_bytes = _run(lib.devunit_pack_endpoints, variant, placement, colors, fq)
    assert rc == 0, lib.devunit_last_error().decode()
    _compare(got_fmt, got_bytes, want_fmt, want_bytes, colors, fq, "GPU %s, %s table" % (variant, placement))
