#!/usr/bin/env python
"""Many small images: one astcenc_b200_compress_device_images call against a compress_device call per image (needs a GPU).

  python tools/multi_image_probe.py [--reps 5] [--out FILE.json]

Workloads, every image resident in device memory:
  chain       the mip chain of bench.py's config 1 image (4096^2 LDR RGBA8, 6x6 -medium) down to 1 x 1 (13 levels)
  chain_tail  the same chain without its base level (12 levels, the largest 2048^2)
  set128      256 seeded 128^2 RGBA8 textures, at 4x4 -fast and at 6x6 -medium
  set512      64 seeded 512^2 RGBA8 textures at 4x4 -fast (config 0's shape)
Per workload and path: ms per call (CUDA events on the launching stream around the whole loop or the one call, median of --reps
after one warm-up) and kernel launches per call. The payloads of the two paths are compared byte for byte. The card's name and
power limit are read in the same run and printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi unavailable)"


def mip_chain(img):
    levels = [np.ascontiguousarray(img)]
    while levels[-1].shape[0] > 1 or levels[-1].shape[1] > 1:
        a = levels[-1].astype(np.float32)
        h, w = a.shape[:2]
        h2, w2 = max(1, h // 2), max(1, w // 2)
        a = a[:h2 * 2 if h > 1 else 1, :w2 * 2 if w > 1 else 1]
        a = a.reshape(h2, a.shape[0] // h2, w2, a.shape[1] // w2, 4).mean(axis=(1, 3))
        levels.append(np.ascontiguousarray(np.round(a).astype(np.uint8)))
    return levels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    import __graft_entry__ as g
    import astc_images
    assert torch.cuda.is_available(), "multi_image_probe.py needs a GPU"
    pkg = g.load_package()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    gpu = card()
    print("card: %s" % gpu)
    chain = mip_chain(astc_images.photo_like(4096, 4096, seed=2024))
    set128 = [astc_images.photo_like(128, 128, seed=k) for k in range(256)]
    set512 = [astc_images.photo_like(512, 512, seed=1000 + k) for k in range(64)]
    workloads = [("chain", chain, 6, 60.0), ("chain_tail", chain[1:], 6, 60.0), ("set128", set128, 4, 10.0), ("set128", set128, 6, 60.0),
                 ("set512", set512, 4, 10.0)]
    results = []
    for name, imgs, b, q in workloads:
        ctx = pkg.Context(pkg.config_init(pkg.PRF_LDR, b, b, q, pkg.FLG_SELF_DECOMPRESS_ONLY))
        d_imgs = [torch.from_numpy(im).to(dev) for im in imgs]
        sizes = [ctx.blocks(im.shape[1], im.shape[0]) for im in imgs]
        d_loop = [torch.zeros(nx * ny * 16, dtype=torch.uint8, device=dev) for nx, ny in sizes]
        d_one = [torch.zeros_like(p) for p in d_loop]
        table = [(d.data_ptr(), im.shape[1], im.shape[0], 1, p.data_ptr()) for d, im, p in zip(d_imgs, imgs, d_one)]

        def loop():
            for d, im, p in zip(d_imgs, imgs, d_loop):
                ctx.compress_device(d.data_ptr(), pkg.TYPE_U8, im.shape[1], im.shape[0], p.data_ptr(), stream=stream.cuda_stream)

        def one():
            ctx.compress_device_images(table, pkg.TYPE_U8, stream=stream.cuda_stream)

        row = {"workload": name, "images": len(imgs), "blocks": int(sum(nx * ny for nx, ny in sizes)), "block": "%dx%d" % (b, b),
               "preset": "fast" if q < 50 else "medium"}
        for path, fn in (("per_image", loop), ("one_call", one)):
            fn()
            torch.cuda.synchronize()
            times, launches = [], 0
            for _ in range(args.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                n0 = ctx.launch_count()
                e0.record(stream)
                fn()
                e1.record(stream)
                e1.synchronize()
                launches = ctx.launch_count() - n0
                times.append(e0.elapsed_time(e1))
            row[path + "_ms"] = round(float(np.median(times)), 3)
            row[path + "_launches"] = int(launches)
        torch.cuda.synchronize()
        row["bytes_equal"] = all(torch.equal(a, b_) for a, b_ in zip(d_loop, d_one))
        row["speedup"] = round(row["per_image_ms"] / row["one_call_ms"], 2)
        print(json.dumps(row), flush=True)
        assert row["bytes_equal"], "the two paths differ on %s" % name
        results.append(row)
        ctx.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": gpu, "reps": args.reps, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
