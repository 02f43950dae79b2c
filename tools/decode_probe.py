#!/usr/bin/env python
"""Decoder throughput: astcenc_b200_decompress_device_images against one device call per image and against
astcenc_decompress_image (host pointers, end to end) on the same payloads (needs a GPU).

  python tools/decode_probe.py [--reps 7] [--out FILE.json]

Workloads, payloads made on the device by compress_device_images and left there:
  config1     bench.py's config 1 image (4096^2 LDR RGBA8, 6x6 -medium), decoded into U8 and into F16
  set128      256 seeded 128^2 RGBA8 textures at 4x4 -fast, decoded into U8
  chain_tail  the 12 levels below the base of config 1's mip chain (2048^2 down to 1 x 1), 6x6 -medium, decoded into U8
Per workload and path: ms per call (median of --reps after one warm-up; CUDA events on the launching stream for the device paths,
a host clock for astcenc_decompress_image, which returns with the image in host memory) and GB/s of algorithmic bytes: 16 per
block read plus 4 * texels * (1 | 2 | 4) written. The outputs of the three paths are compared byte for byte. The card's name and
power limit are read in the same run and printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time

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
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    import __graft_entry__ as g
    import astc_images
    assert torch.cuda.is_available(), "decode_probe.py needs a GPU"
    pkg = g.load_package()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    gpu = card()
    print("card: %s" % gpu)
    base = astc_images.photo_like(4096, 4096, seed=2024)
    set128 = [astc_images.photo_like(128, 128, seed=k) for k in range(256)]
    np_types = {pkg.TYPE_U8: np.uint8, pkg.TYPE_F16: np.float16}
    workloads = [("config1", [base], 6, 60.0, pkg.TYPE_U8), ("config1", [base], 6, 60.0, pkg.TYPE_F16), ("set128", set128, 4, 10.0, pkg.TYPE_U8),
                 ("chain_tail", mip_chain(base)[1:], 6, 60.0, pkg.TYPE_U8)]
    results = []
    for name, imgs, b, q, out_type in workloads:
        ctx = pkg.Context(pkg.config_init(pkg.PRF_LDR, b, b, q, 0))
        texel_bytes = 4 * np.dtype(np_types[out_type]).itemsize
        sizes = [ctx.blocks(im.shape[1], im.shape[0]) for im in imgs]
        d_imgs = [torch.from_numpy(im).to(dev) for im in imgs]
        d_pays = [torch.zeros(nx * ny * 16, dtype=torch.uint8, device=dev) for nx, ny in sizes]
        ctx.compress_device_images([(d.data_ptr(), im.shape[1], im.shape[0], 1, p.data_ptr()) for d, im, p in zip(d_imgs, imgs, d_pays)], pkg.TYPE_U8,
                                   stream=stream.cuda_stream)
        stream.synchronize()
        del d_imgs
        h_pays = [p.cpu().numpy() for p in d_pays]
        d_one = [torch.zeros(im.shape[0] * im.shape[1] * texel_bytes, dtype=torch.uint8, device=dev) for im in imgs]
        d_each = [torch.zeros_like(o) for o in d_one]
        table = [(p.data_ptr(), o.data_ptr(), im.shape[1], im.shape[0], 1) for p, o, im in zip(d_pays, d_one, imgs)]
        tables = [[(p.data_ptr(), o.data_ptr(), im.shape[1], im.shape[0], 1)] for p, o, im in zip(d_pays, d_each, imgs)]
        host_out = []

        def one():
            ctx.decompress_device_images(table, out_type, stream=stream.cuda_stream)

        def each():
            for t in tables:
                ctx.decompress_device_images(t, out_type, stream=stream.cuda_stream)

        def host():
            host_out[:] = [ctx.decompress_image(p, im.shape[1], im.shape[0], dtype=np_types[out_type]) for p, im in zip(h_pays, imgs)]

        blocks = int(sum(nx * ny for nx, ny in sizes))
        texels = int(sum(im.shape[0] * im.shape[1] for im in imgs))
        nbytes = 16 * blocks + texels * texel_bytes
        row = {"workload": name, "images": len(imgs), "blocks": blocks, "block": "%dx%d" % (b, b), "output": "U8" if out_type == pkg.TYPE_U8 else "F16",
               "bytes": nbytes}
        for path, fn in (("one_call", one), ("per_image", each), ("decompress_image", host)):
            fn()
            torch.cuda.synchronize()
            times, launches = [], 0
            for _ in range(args.reps):
                n0 = ctx.launch_count()
                if path == "decompress_image":
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
            row[path + "_launches"] = int(launches)
        torch.cuda.synchronize()
        row["outputs_equal"] = all(torch.equal(a, c) for a, c in zip(d_one, d_each)) and \
            all(np.array_equal(a.cpu().numpy(), h.view(np.uint8).reshape(-1)) for a, h in zip(d_one, host_out))
        print(json.dumps(row), flush=True)
        assert row["outputs_equal"], "the paths differ on %s" % name
        results.append(row)
        ctx.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": gpu, "reps": args.reps, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
