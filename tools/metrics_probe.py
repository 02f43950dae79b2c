#!/usr/bin/env python
"""Metrics throughput: one astcenc_b200_compute_error_metrics_device_images call against astcenc_b200_compute_error_metrics once
per image (host pointers, end to end) on the same image pairs (needs a GPU).

  python tools/metrics_probe.py [--reps 7] [--out FILE.json]

Workloads, each image compressed and decoded on the device (compress_device_images, decompress_device_images) and left there:
  config1     bench.py's config 1 image (4096^2 LDR RGBA8, 6x6 -medium) against its decode into U8, and into F16
  set128      256 seeded 128^2 RGBA8 textures at 4x4 -fast against their decodes into U8
  chain_tail  the 12 levels below the base of config 1's mip chain (2048^2 down to 1 x 1), 6x6 -medium, decoded into U8
The device call measures every pair with a per-block error map; the host entry gets host copies of the same pairs. Per workload
and path: ms per call (median of --reps after one warm-up; CUDA events on the launching stream for the device call, a host clock
for the host entry, which returns with the figures in host memory) and GB/s of algorithmic bytes: both images read plus the map
written, against the H100 SXM data sheet's 3.35 TB/s. The sums of the two paths are compared bit for bit. The card's name and
power limit are read in the same run and printed with the numbers."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

HBM_BYTES_PER_S = 3.35e12


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi unavailable)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    import __graft_entry__ as g
    import astc_images
    from decode_probe import mip_chain
    assert torch.cuda.is_available(), "metrics_probe.py needs a GPU"
    pkg = g.load_package()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    gpu = card()
    print("card: %s" % gpu)
    base = astc_images.photo_like(4096, 4096, seed=2024)
    set128 = [astc_images.photo_like(128, 128, seed=k) for k in range(256)]
    np_types = {pkg.TYPE_U8: np.uint8, pkg.TYPE_F16: np.float16}
    mbytes = C.sizeof(pkg.ErrorMetrics)
    workloads = [("config1", [base], 6, 60.0, pkg.TYPE_U8), ("config1", [base], 6, 60.0, pkg.TYPE_F16), ("set128", set128, 4, 10.0, pkg.TYPE_U8),
                 ("chain_tail", mip_chain(base)[1:], 6, 60.0, pkg.TYPE_U8)]
    results = []
    for name, imgs, b, q, dec_type in workloads:
        ctx = pkg.Context(pkg.config_init(pkg.PRF_LDR, b, b, q, 0))
        dec_texel = 4 * np.dtype(np_types[dec_type]).itemsize
        sizes = [ctx.blocks(im.shape[1], im.shape[0]) for im in imgs]
        d_imgs = [torch.from_numpy(im.reshape(-1)).to(dev) for im in imgs]
        d_pays = [torch.zeros(nx * ny * 16, dtype=torch.uint8, device=dev) for nx, ny in sizes]
        d_decs = [torch.zeros(im.shape[0] * im.shape[1] * dec_texel, dtype=torch.uint8, device=dev) for im in imgs]
        ctx.compress_device_images([(d.data_ptr(), im.shape[1], im.shape[0], 1, p.data_ptr()) for d, im, p in zip(d_imgs, imgs, d_pays)], pkg.TYPE_U8,
                                   stream=stream.cuda_stream)
        ctx.decompress_device_images([(p.data_ptr(), o.data_ptr(), im.shape[1], im.shape[0], 1) for p, o, im in zip(d_pays, d_decs, imgs)], dec_type,
                                     stream=stream.cuda_stream)
        stream.synchronize()
        h_decs = [o.cpu().numpy().view(np_types[dec_type]).reshape(im.shape) for o, im in zip(d_decs, imgs)]
        d_met = torch.zeros(len(imgs) * mbytes, dtype=torch.uint8, device=dev)
        d_maps = [torch.zeros(nx * ny, dtype=torch.float32, device=dev) for nx, ny in sizes]
        table = [(i.data_ptr(), o.data_ptr(), pkg.TYPE_U8, dec_type, im.shape[1], im.shape[0], 1, d_met.data_ptr() + k * mbytes, m.data_ptr())
                 for k, (i, o, im, m) in enumerate(zip(d_imgs, d_decs, imgs, d_maps))]
        host_out = []

        def device():
            ctx.compute_error_metrics_device_images(table, stream=stream.cuda_stream)

        def host():
            host_out[:] = [ctx.compute_error_metrics(im, h) for im, h in zip(imgs, h_decs)]

        blocks = int(sum(nx * ny for nx, ny in sizes))
        texels = int(sum(im.shape[0] * im.shape[1] for im in imgs))
        nbytes = texels * (4 + dec_texel) + 4 * blocks
        row = {"workload": name, "images": len(imgs), "blocks": blocks, "block": "%dx%d" % (b, b), "decoded": "U8" if dec_type == pkg.TYPE_U8 else "F16",
               "bytes": nbytes}
        for path, fn in (("device_call", device), ("host_entry", host)):
            fn()
            torch.cuda.synchronize()
            times, launches = [], 0
            for _ in range(args.reps):
                n0 = ctx.launch_count()
                if path == "host_entry":
                    t0 = time.perf_counter()
                    fn()
                    times.append((time.perf_counter() - t0) * 1e3)
                else:
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(stream)
                    fn()
                    e1.record(stream)
                    e1.synchronize()
                    times.append(e0.elapsed_time(e1))
                launches = ctx.launch_count() - n0
            ms = float(np.median(times))
            row[path + "_ms"] = round(ms, 3)
            row[path + "_GBps"] = round(nbytes / ms / 1e6, 1)
            row[path + "_share_of_hbm"] = round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 4)
            row[path + "_launches"] = int(launches)
        torch.cuda.synchronize()
        got = d_met.cpu().numpy()
        dev_mets = [pkg.ErrorMetrics.from_buffer_copy(got[k * mbytes:(k + 1) * mbytes].tobytes()) for k in range(len(imgs))]
        row["sums_equal"] = all(list(d.sum_squared_error) == h["sum_squared_error"] and d.rgb_peak == h["rgb_peak"] for d, h in zip(dev_mets, host_out))
        print(json.dumps(row), flush=True)
        assert row["sums_equal"], "the paths differ on %s" % name
        results.append(row)
        ctx.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": gpu, "reps": args.reps, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
