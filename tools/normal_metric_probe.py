#!/usr/bin/env python
"""Normal-map block metrics (ASTCENC_B200_BLOCK_ANGULAR_ERROR, ASTCENC_B200_BLOCK_WORST_ANGULAR_ERROR): call times, and what
selecting by angle buys a keep-the-better round on a normal map (needs a GPU).

  python tools/normal_metric_probe.py [--reps 7] [--out FILE.json]

Workload: a seeded 4096^2 U8 normal map (two octaves of tests/astc_images.py's _value_noise as a height field, central
differences, normalised, packed as (n + 1) / 2, alpha 255), resident in device memory, 6x6, the CLI's normal-map settings:
ASTCENC_FLG_MAP_NORMAL, encode swizzle rrrg, decode swizzle (R, A, Z, 1) into U8; maps and figures over input_components 3.
  calls:   one whole map call (figures with normal=1 and a map) and one list refresh of a sorted random 1 % list, for SQUARED,
           ANGULAR and WORST
  rounds:  from the same -fast payload, a map of metric M, select_blocks of the worst 1 %, 5 % and 10 %, and one -thorough
           refine_device_block_lists measured in M (keep the better under M), for M = SQUARED, ANGULAR, WORST; the final
           mean_angular_error and worst_angular_error and the round's time (map, select and refine)
  target:  "no texel beyond T degrees" for two T: from the -fast payload, three rounds of select_blocks on the WORST map with
           threshold T and a capacity of 10 % of the blocks, each followed by a -thorough WORST refine; per round the blocks
           still above T and the worst angle
Times: ms (CUDA events on the stream; median of --reps after one warm-up). The card's name and power limit are read in the
same run and printed with the numbers."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

FRACTIONS = (0.01, 0.05, 0.10)
RRRG, RAZ1 = (0, 0, 0, 1), (0, 3, 6, 5)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi unavailable)"


def normal_map(size, seed):
    """The seeded U8 normal map of the module docstring."""
    from astc_images import _value_noise
    rng = np.random.default_rng(seed)
    ht = 48.0 * _value_noise(rng, size, size, 64, 1)[..., 0] + 6.0 * _value_noise(rng, size, size, 12, 1)[..., 0]
    dy, dx = np.gradient(ht.astype(np.float64))
    n = np.stack([-dx, -dy, np.ones_like(ht, dtype=np.float64)], axis=-1)
    n /= np.linalg.norm(n, axis=-1, keepdims=True)
    out = np.full((size, size, 4), 255, np.uint8)
    out[..., :3] = np.clip(np.rint((n + 1.0) * 0.5 * 255.0), 0, 255).astype(np.uint8)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--size", type=int, default=4096)
    ap.add_argument("--out")
    args = ap.parse_args()
    assert args.reps >= 5, "at least 5 timed repetitions"
    import torch
    import __graft_entry__ as g
    assert torch.cuda.is_available(), "normal_metric_probe.py needs a GPU"
    pkg = g.load_package()
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream(device=dev)
    s = st.cuda_stream
    gpu = card()
    print("card: %s" % gpu)
    names = {pkg.BLOCK_SQUARED_ERROR: "SQUARED", pkg.BLOCK_ANGULAR_ERROR: "ANGULAR", pkg.BLOCK_WORST_ANGULAR_ERROR: "WORST"}
    mb = C.sizeof(pkg.ErrorMetrics)
    U8 = pkg.TYPE_U8

    def timed(fn):
        fn()
        st.synchronize()
        ts = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            fn()
            e1.record(st)
            e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        return float(np.median(ts))

    W = H = args.size
    img = normal_map(W, 7)
    fast = pkg.Context(pkg.config_init(pkg.PRF_LDR, 6, 6, pkg.PRE_FAST, pkg.FLG_MAP_NORMAL))
    thorough = pkg.Context(pkg.config_init(pkg.PRF_LDR, 6, 6, pkg.PRE_THOROUGH, pkg.FLG_MAP_NORMAL))
    dec_ctx = pkg.Context(pkg.config_init(pkg.PRF_LDR, 6, 6, pkg.PRE_FAST, pkg.FLG_DECOMPRESS_ONLY))
    bx, by = fast.blocks(W, H)
    n = bx * by
    d_img = torch.from_numpy(img.reshape(-1).view(np.uint8)).to(dev)
    fast_pay = torch.zeros(n * 16, dtype=torch.uint8, device=dev)
    fast_dec = torch.zeros(W * H * 4, dtype=torch.uint8, device=dev)
    pay, dec = torch.zeros_like(fast_pay), torch.zeros_like(fast_dec)
    mp = torch.zeros(n, dtype=torch.float32, device=dev)
    met = torch.zeros(mb, dtype=torch.uint8, device=dev)
    idx = torch.zeros(n, dtype=torch.int32, device=dev)
    cnt = torch.zeros(1, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    fast.compress_device_images([(d_img.data_ptr(), W, H, 1, fast_pay.data_ptr())], U8, swizzle=RRRG, stream=s)
    dec_ctx.decompress_device_images([(fast_pay.data_ptr(), fast_dec.data_ptr(), W, H, 1)], U8, swizzle=RAZ1, stream=s)

    def whole(metric, d=None, m=None):
        dec_ctx.compute_block_metric_device_images([(d_img.data_ptr(), (d if d is not None else dec).data_ptr(), U8, U8, W, H, 1, met.data_ptr(),
                                                     (m if m is not None else mp).data_ptr())], metric, normal=True, input_components=3, stream=s)

    def figures():
        st.synchronize()
        f = pkg.ErrorMetrics.from_buffer_copy(met.cpu().numpy().tobytes())
        return f.mean_angular_error, f.worst_angular_error, f.psnr

    def reset():
        pay.copy_(fast_pay)
        dec.copy_(fast_dec)

    with torch.cuda.stream(st):
        reset()
    whole(pkg.BLOCK_SQUARED_ERROR)
    fast_mean, fast_worst, fast_psnr = figures()
    print("%d^2 normal map, %d blocks of 6x6; -fast: mean angle %.4f deg, worst %.3f deg, PSNR %.3f dB" % (W, n, fast_mean, fast_worst, fast_psnr))
    result = dict(card=gpu, size=W, blocks=n, fast=dict(mean_angular_error=fast_mean, worst_angular_error=fast_worst, psnr=fast_psnr))

    # calls
    k = n // 100
    lst = np.sort(np.random.default_rng(1).choice(n, k, replace=False)).astype(np.int32)
    d_lst = torch.from_numpy(lst).to(dev)
    d_k = torch.tensor([k], dtype=torch.int32, device=dev)
    calls = {}
    for m, name in names.items():
        t_whole = timed(lambda: whole(m))
        t_list = timed(lambda: dec_ctx.compute_block_metric_device_block_lists([(d_img.data_ptr(), dec.data_ptr(), U8, U8, W, H, 1, mp.data_ptr(),
                                                                                  d_lst.data_ptr(), d_k.data_ptr(), k)], m, input_components=3, stream=s))
        calls[name] = dict(whole_ms=t_whole, list_1pct_ms=t_list)
        print("calls  %-8s whole map %.3f ms   1 %% list refresh (%d blocks) %.4f ms" % (name, t_whole, k, t_list))
    result["calls"] = calls

    # rounds
    def one_round(m, cap):
        whole(m)
        thorough.select_blocks([(mp.data_ptr(), n, -np.inf, cap, idx.data_ptr(), cnt.data_ptr())], stream=s)
        thorough.refine_device_block_lists([(d_img.data_ptr(), W, H, 1, pay.data_ptr(), dec.data_ptr(), mp.data_ptr(), idx.data_ptr(), cnt.data_ptr(), cap)],
                                           U8, U8, m, swizzle=RRRG, decode_swizzle=RAZ1, input_components=3, stream=s)

    rounds = []
    for f in FRACTIONS:
        cap = int(n * f)
        for m, name in names.items():
            times = []
            for rep in range(3):
                with torch.cuda.stream(st):
                    reset()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                one_round(m, cap)
                e1.record(st)
                e1.synchronize()
                times.append(e0.elapsed_time(e1))
            whole(pkg.BLOCK_SQUARED_ERROR)
            mean, worst, psnr = figures()
            r = dict(fraction=f, select_by=name, mean_angular_error=mean, worst_angular_error=worst, psnr=psnr, round_ms=float(np.median(times[1:])))
            rounds.append(r)
            print("round  %4.0f %% by %-8s mean %.4f deg  worst %.3f deg  PSNR %.3f dB  %.1f ms" % (100 * f, name, mean, worst, psnr, r["round_ms"]))
    result["rounds"] = rounds

    # "no texel beyond T degrees"
    targets = []
    cap = n // 10
    with torch.cuda.stream(st):
        reset()
    whole(pkg.BLOCK_WORST_ANGULAR_ERROR)
    st.synchronize()
    w0 = mp.cpu().numpy()
    for T in (float(np.percentile(w0, 90)), float(np.percentile(w0, 99))):
        with torch.cuda.stream(st):
            reset()
        whole(pkg.BLOCK_WORST_ANGULAR_ERROR)
        st.synchronize()
        per = [dict(round=0, above=int(np.sum(mp.cpu().numpy() > T)), worst=float(mp.max()))]
        for r in range(1, 4):
            thorough.select_blocks([(mp.data_ptr(), n, T, cap, idx.data_ptr(), cnt.data_ptr())], stream=s)
            thorough.refine_device_block_lists([(d_img.data_ptr(), W, H, 1, pay.data_ptr(), dec.data_ptr(), mp.data_ptr(), idx.data_ptr(), cnt.data_ptr(),
                                                 cap)], U8, U8, pkg.BLOCK_WORST_ANGULAR_ERROR, swizzle=RRRG, decode_swizzle=RAZ1, input_components=3,
                                               stream=s)
            st.synchronize()
            m = mp.cpu().numpy()
            per.append(dict(round=r, listed=int(cnt.cpu()[0]), above=int(np.sum(m > T)), worst=float(m.max())))
        targets.append(dict(T=T, rounds=per))
        print("target T = %.3f deg (capacity %d): %s" % (T, cap, "; ".join("round %d: %d above, worst %.3f" % (p["round"], p["above"], p["worst"])
                                                                          for p in per)))
    result["targets"] = targets
    for c in (fast, thorough, dec_ctx):
        c.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
