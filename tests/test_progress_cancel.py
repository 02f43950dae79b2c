"""Progress reporting and cancellation of astcenc_compress_image.

CPU: the device source on the host simulation (one lane and 32 lanes, tests/hostsim/hostsim_progress.cpp) with the pass's two
device words - the cancel flag, looked at wherever a warp takes new work, and the done counter, one add per block whose search
has ended.
GPU: the progress callback and astcenc_compress_cancel through the C ABI, against passes of the same context without them."""
import ctypes as C
import threading
import time

import numpy as np
import pytest

import astc_images as I
from astc_ref import *  # noqa: F401,F403
from hostsim_build import host_sim
from golden.make_golden import CASES, make_image

S = FLG_SELF_DECOMPRESS_ONLY
_DT = {np.dtype(np.uint8): TYPE_U8, np.dtype(np.float16): TYPE_F16, np.dtype(np.float32): TYPE_F32}
GOLDEN = {c[0]: c for c in CASES}

_SIMS = {}


def progress_sim(lanes32):
    """tests/hostsim/hostsim_progress.cpp compiled for the host (one simulated lane, or 32 lanes on 32 threads)."""
    if lanes32 in _SIMS:
        return _SIMS[lanes32]
    lib = host_sim("hostsim_progress", lanes32)
    lib.hostsim_set_cancel.argtypes = [C.c_int]
    lib.hostsim_done.restype = C.c_uint
    lib.hostsim_set_a_scale_radius.argtypes = [C.c_uint]
    lib.hostsim_progress_volume.argtypes = [C.c_int, C.c_uint, C.c_uint, C.c_uint, C.c_float, C.c_uint, C.c_void_p, C.c_int, C.c_uint, C.c_uint, C.c_uint,
                                            C.POINTER(C.c_int), C.c_void_p]
    _SIMS[lanes32] = lib
    return lib


@pytest.fixture(params=["1 lane", "32 lanes"])
def sim(request):
    lib = progress_sim(request.param == "32 lanes")
    lib.hostsim_set_cancel(-1)
    yield lib
    lib.hostsim_set_cancel(-1)


def sim_run(lib, vol, prof, fp, q, fl, out=None):
    """Compress a (D, H, W, 4) volume (D = 1 for 2D footprints); returns (blocks, done counter)."""
    vol = np.ascontiguousarray(vol)
    d, h, w = vol.shape[:3]
    bx, by, bz = fp
    n = ((w + bx - 1) // bx) * ((h + by - 1) // by) * ((d + bz - 1) // bz)
    if out is None:
        out = np.full(n * 16, 0xA5, np.uint8)
    rc = lib.hostsim_progress_volume(prof, bx, by, bz, q, fl, vol.ctypes.data, _DT[vol.dtype], w, h, d, None, out.ctypes.data)
    assert rc == 0
    return out, int(lib.hostsim_done()), n


def _constant_blocks(img, bx, by):
    h, w = img.shape[:2]
    return sum(int(np.all(img[y:y + by, x:x + bx] == img[y, x])) for y in range(0, h, by) for x in range(0, w, bx))


# ---- CPU: the host simulation ----

def test_counter_counts_every_block_of_a_2d_image_with_constant_blocks(sim):
    img = I.photo_like(18, 24, seed=31)
    img[:12, :12] = (40, 90, 200, 255)      # four constant blocks: emitted by wave 0 without a search
    assert _constant_blocks(img, 6, 6) >= 4
    _, done, n = sim_run(sim, img[None], PRF_LDR, (6, 6, 1), PRE_MEDIUM, S)
    assert done == n


def test_counter_counts_alpha_scale_rdo_blocks(sim):
    img = I.alpha_mask(24, 24, seed=13)
    assert any(np.all(img[y:y + 6, x:x + 6, 3] == 0) for y in range(0, 24, 6) for x in range(0, 24, 6))
    sim.hostsim_set_a_scale_radius(2)
    try:
        _, done, n = sim_run(sim, img[None], PRF_LDR, (6, 6, 1), PRE_MEDIUM, S | FLG_USE_ALPHA_WEIGHT)
    finally:
        sim.hostsim_set_a_scale_radius(0)
    assert done == n


def test_counter_counts_every_block_of_a_3d_footprint(sim):
    vol = np.stack([I.photo_like(8, 8, seed=40 + z) for z in range(4)])
    _, done, n = sim_run(sim, vol, PRF_LDR, (4, 4, 4), PRE_FAST, S)
    assert n == 4 and done == n


def test_counter_and_flag_in_the_lockstep_driver(monkeypatch):
    """The phase-aligned single-kernel driver (compress_blocks_lockstep) shares the ticket feed and counts its blocks. (The
    simulation's per-warp driver walks the blocks itself; that driver is covered on the GPU.)"""
    lib = progress_sim(False)
    monkeypatch.setenv("HOSTSIM_DRIVER", "lockstep")
    img = I.photo_like(12, 18, seed=12)
    img[:6, :6] = 9
    lib.hostsim_set_cancel(-1)
    _, done, n = sim_run(lib, img[None], PRF_LDR, (6, 6, 1), PRE_MEDIUM, S)
    assert done == n
    lib.hostsim_set_cancel(0)
    try:
        out, done, n = sim_run(lib, img[None], PRF_LDR, (6, 6, 1), PRE_MEDIUM, S)
    finally:
        lib.hostsim_set_cancel(-1)
    assert done == 0 and np.all(out == 0xA5)


def test_flag_raised_before_the_pass_searches_nothing(sim):
    img = I.photo_like(18, 24, seed=31)
    img[:6, :6] = 7      # (a constant block would be emitted at once if wave 0 took it)
    sim.hostsim_set_cancel(0)
    out, done, n = sim_run(sim, img[None], PRF_LDR, (6, 6, 1), PRE_MEDIUM, S)
    assert done == 0
    assert np.all(out == 0xA5)      # no block was emitted, packed or written


def test_flag_raised_mid_pass_then_a_clean_pass_equals_golden(sim, golden):
    name = "photo_6x6_medium" if sim.hostsim_lanes() == 1 else "photo_5x4_fastest"
    _, gen, size, dtype, prof, bx, by, q, fl, swz = GOLDEN[name]
    assert swz == (0, 1, 2, 3)
    img = np.ascontiguousarray(make_image(gen, size, dtype))
    golden = golden[name]
    n = ((size[1] + bx - 1) // bx) * ((size[0] + by - 1) // by)
    sim.hostsim_set_cancel(4 * n)      # raised at the 4n-th pop / ticket of the pass: in the first waves after wave 0
    out, done, _ = sim_run(sim, img[None], prof, (bx, by, 1), q, fl)
    assert done < n
    assert not np.array_equal(out, golden)
    sim.hostsim_set_cancel(-1)
    out, done, n = sim_run(sim, img[None], prof, (bx, by, 1), q, fl, out=out)      # the same buffers, the flag down
    assert done == n
    assert len(block_diff(out, golden)) == 0


# ---- GPU: astcenc_compress_image ----

def min_diff(total):
    return max(4096.0 / total * 100.0, 1.0)


def check_progress(values, total):
    """The reference's reporting rule: increasing by more than the min-diff step, 100 exactly once and last."""
    assert values and values[-1] == 100.0
    assert values.count(100.0) == 1
    last = 0.0
    for v in values[:-1]:
        assert 0.0 < v < 100.0
        assert v - last > min_diff(total), (last, v)
        last = v


@pytest.fixture(scope="module")
def gpu(pkg):
    import torch
    assert torch.cuda.is_available(), "these tests need a CUDA device"
    return pkg


@pytest.fixture(scope="module")
def long_pass(gpu):
    """4096 x 4096 RGBA8 at 8x8 -thorough: a pass of about 300 ms on an H100; its payload and wall time without a callback."""
    img = I.photo_like(4096, 4096, seed=77)
    cfg = gpu.config_init(PRF_LDR, 8, 8, PRE_THOROUGH, S)
    ctx = gpu.Context(cfg)
    ctx.compress_image(img)      # (warm-up: buffers, modules)
    t0 = time.perf_counter()
    want = ctx.compress_image(img)
    wall = time.perf_counter() - t0
    ctx.close()
    return img, cfg, want, wall


def run_with_progress(gpu, cfg, img, on_value=None, thread_count=1):
    got = []
    holder = {}

    def cb(v):
        got.append((v, time.perf_counter()))
        if on_value is not None:
            on_value(holder["ctx"], v)

    ctx = gpu.Context(cfg, thread_count=thread_count, progress=cb)
    holder["ctx"] = ctx
    return ctx, got


@pytest.mark.gpu
def test_progress_on_a_long_pass(gpu, long_pass):
    img, cfg, want, wall = long_pass
    ctx, got = run_with_progress(gpu, cfg, img)
    ctx.compress_image(img)
    got.clear()
    t0 = time.perf_counter()
    out = ctx.compress_image(img)
    ctx.close()
    total = (4096 // 8) ** 2
    values = [v for v, _ in got]
    print("progress: %d calls below 100 in %.1f ms (first %s, last %s); pass without a callback %.1f ms"
          % (len(values) - 1, (time.perf_counter() - t0) * 1e3, values[:3], values[-4:], wall * 1e3))
    print("progress curve (ms, %%): %s" % [(round((t - t0) * 1e3, 1), round(v, 1)) for v, t in got[::max(1, len(got) // 20)]])
    check_progress(values, total)
    assert len(values) - 1 >= 20
    assert np.array_equal(out, want)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["2d footprint, dim_z 4", "3d footprint"])
def test_progress_over_a_volume(gpu, shape):
    if shape == "3d footprint":
        vol = np.stack([I.photo_like(256, 256, seed=90 + z) for z in range(16)])
        cfg = gpu.config_init(PRF_LDR, 4, 4, PRE_THOROUGH, S, block_z=4)
        total = 64 * 64 * 4
    else:
        vol = np.stack([I.photo_like(2048, 2048, seed=80 + z) for z in range(4)])
        cfg = gpu.config_init(PRF_LDR, 8, 8, PRE_THOROUGH, S)
        total = 256 * 256 * 4
    ref = gpu.Context(cfg)
    want = ref.compress_image(vol)
    ref.close()
    ctx, got = run_with_progress(gpu, cfg, vol)
    out = ctx.compress_image(vol)
    ctx.close()
    values = [v for v, _ in got]
    print("%s: %d calls below 100" % (shape, len(values) - 1))
    check_progress(values, total)
    assert np.array_equal(out, want)


@pytest.mark.gpu
def test_cancel_from_the_callback(gpu, long_pass):
    img, cfg, want, wall = long_pass
    state = {"cancelled_at": None}

    def on_value(ctx, v):
        if v >= 20.0 and state["cancelled_at"] is None:
            state["cancelled_at"] = v
            state["t_cancel"] = time.perf_counter()
            ctx.cancel()

    ctx, got = run_with_progress(gpu, cfg, img, on_value)
    out = np.full(want.size, 0x5A, np.uint8)
    t0 = time.perf_counter()
    ctx.compress_image(img, out=out)      # (raises on anything but ASTCENC_SUCCESS)
    t1 = time.perf_counter()
    took = t1 - t0
    values = [v for v, _ in got]
    print("cancelled at %.2f %%: call %.1f ms against %.1f ms uncancelled, %.2f ms from the cancel to the return"
          % (state["cancelled_at"], took * 1e3, wall * 1e3, (t1 - state["t_cancel"]) * 1e3))
    assert state["cancelled_at"] is not None
    assert 100.0 not in values
    assert np.all(out == 0x5A)
    # The counter counts finished searches, and few blocks finish in the first waves: on this image the first value >= 20 %
    # comes at 27-35 % of the pass's time (H100 80GB HBM3), depending on where a wave boundary falls. What the cancel itself
    # costs is the time from the cancel to the return: about 2 ms measured.
    assert t1 - state["t_cancel"] < 0.02
    assert took < 0.5 * wall
    ctx.reset()
    got.clear()
    state["cancelled_at"] = -1.0      # (no cancel this time)
    assert np.array_equal(ctx.compress_image(img), want)
    assert [v for v, _ in got][-1] == 100.0
    ctx.close()


@pytest.mark.gpu
def test_cancel_from_another_thread_without_a_callback(gpu, long_pass):
    img, cfg, want, wall = long_pass
    ctx = gpu.Context(cfg)
    ctx.compress_image(img)
    out = np.full(want.size, 0x5A, np.uint8)
    timer = threading.Timer(0.2 * wall, ctx.cancel)
    t0 = time.perf_counter()
    timer.start()
    ctx.compress_image(img, out=out)
    took = time.perf_counter() - t0
    timer.join()
    print("cancel from a thread after %.1f ms: call %.1f ms against %.1f ms" % (0.2 * wall * 1e3, took * 1e3, wall * 1e3))
    assert took < 0.6 * wall
    assert np.all(out == 0x5A)
    ctx.reset()
    assert np.array_equal(ctx.compress_image(img), want)
    ctx.close()


@pytest.mark.gpu
def test_cancel_before_the_call_with_two_caller_threads(gpu, long_pass):
    img, cfg, want, wall = long_pass
    ctx = gpu.Context(cfg, thread_count=2)
    ctx.cancel()
    outs = [np.full(want.size, 0x5A, np.uint8) for _ in range(2)]
    errors = []

    def caller(i, o):
        try:
            ctx.compress_image(img, out=o, thread_index=i)
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    t0 = time.perf_counter()
    ts = [threading.Thread(target=caller, args=(i, outs[i])) for i in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    took = time.perf_counter() - t0
    assert not errors
    assert took < 0.25 * wall
    assert all(np.all(o == 0x5A) for o in outs)
    ctx.reset()
    out = np.full(want.size, 0x5A, np.uint8)
    ts = [threading.Thread(target=caller, args=(i, out)) for i in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors
    assert np.array_equal(out, want)
    ctx.close()


@pytest.mark.gpu
def test_a_raised_flag_affects_nothing_else(gpu, long_pass):
    import torch
    img, cfg, want, wall = long_pass
    parent = gpu.Context(cfg)
    child = gpu.Context(parent=parent)
    child_out = {}

    def child_call():
        child_out["blocks"] = child.compress_image(img)

    th = threading.Thread(target=child_call)
    th.start()
    time.sleep(0.1 * wall)
    parent.cancel()      # raised while the child's pass runs
    th.join()
    assert np.array_equal(child_out["blocks"], want)
    # the device-resident path ignores the context's flag: no reset in between
    d_img = torch.from_numpy(np.ascontiguousarray(img)).cuda()
    d_out = torch.empty(want.size, dtype=torch.uint8, device="cuda")
    parent.compress_device(d_img.data_ptr(), TYPE_U8, img.shape[1], img.shape[0], d_out.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(d_out.cpu().numpy(), want)
    child.close()
    parent.close()


@pytest.mark.gpu
@pytest.mark.parametrize("driver", ["lockstep", "warp"])
def test_progress_and_cancel_in_the_single_kernel_drivers(gpu, monkeypatch, driver):
    """ASTCENC_B200_DRIVER=lockstep|warp: one kernel per pass; its blocks are counted and its ticket feed honours the flag."""
    img = I.photo_like(2048, 2048, seed=66)
    cfg = gpu.config_init(PRF_LDR, 8, 8, PRE_THOROUGH, S)
    want = gpu.Context(cfg).compress_image(img)      # (the wave pipeline)
    monkeypatch.setenv("ASTCENC_B200_DRIVER", driver)
    ctx, got = run_with_progress(gpu, cfg, img)
    out = ctx.compress_image(img)
    values = [v for v, _ in got]
    print("%s driver: %d calls below 100" % (driver, len(values) - 1))
    check_progress(values, 256 * 256)
    assert len(values) >= 6 and values[-2] >= 50.0
    assert np.array_equal(out, want)
    state = {}

    def on_value(c, v):
        if "t" not in state:
            state["t"] = time.perf_counter()
            c.cancel()

    ctx2, got2 = run_with_progress(gpu, cfg, img, on_value)
    sentinel = np.full(want.size, 0x5A, np.uint8)
    ctx2.compress_image(img, out=sentinel)
    t1 = time.perf_counter()
    assert 100.0 not in [v for v, _ in got2]
    assert np.all(sentinel == 0x5A)
    assert t1 - state["t"] < 0.02
    ctx.close()
    ctx2.close()
