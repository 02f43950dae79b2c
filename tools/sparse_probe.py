#!/usr/bin/env python
"""Block lists against whole-image and block-row passes (astcenc_b200_compress_device_blocks; needs a GPU).

  python tools/sparse_probe.py [--configs 0 1] [--reps 5] [--out FILE.json]

For bench.py's configs 0 (512^2 LDR 4x4 -fast) and 1 (4096^2 LDR 6x6 -medium), on the workload image resident in device memory:
  whole        one compress_device pass over every block row
  rows:<k>     compress_device over the block rows that cover the square of k blocks
  list:<k>     a seeded random scattered list of k blocks
  square:<k>   the blocks of one square of about k blocks in the middle of the image
with k = 1, 121 (a 64 x 64 texel square at 6x6), 1 %, 10 % and 100 % of the blocks. Per case: ms per call (CUDA events on the
launching stream, median of --reps calls after two warm-up calls) and kernel launches per call. Every payload is checked against
the whole-image pass (a list rewrites its blocks in a copy of it: the copy must come out unchanged). The card's name and power
limit are read in the same run and printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

CONFIGS = {0: (512, 4, 10.0, "512x512 LDR RGBA8 4x4 -fast"), 1: (4096, 6, 60.0, "4096x4096 LDR RGBA8 6x6 -medium")}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi unavailable)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", type=int, nargs="+", default=[0, 1])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    import __graft_entry__ as g
    import astc_images
    assert torch.cuda.is_available(), "sparse_probe.py needs a GPU"
    pkg = g.load_package()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    gpu = card()
    print("card: %s" % gpu)
    results = []
    for c in args.configs:
        dim, b, q, name = CONFIGS[c]
        img = np.ascontiguousarray(astc_images.photo_like(dim, dim, seed=2024))
        ctx = pkg.Context(pkg.config_init(pkg.PRF_LDR, b, b, q, pkg.FLG_SELF_DECOMPRESS_ONLY))
        nbx, nby = ctx.blocks(dim, dim)
        total = nbx * nby
        d_img = torch.from_numpy(img).to(dev)
        d_whole = torch.zeros(total * 16, dtype=torch.uint8, device=dev)
        d_work = torch.zeros_like(d_whole)

        def timed(call):
            for _ in range(2):
                call()
            torch.cuda.synchronize()
            ms = []
            n0 = ctx.launch_count()
            for _ in range(args.reps):
                a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(stream)
                call()
                e.record(stream)
                torch.cuda.synchronize()
                ms.append(a.elapsed_time(e))
            return float(np.median(ms)), (ctx.launch_count() - n0) / args.reps

        whole_call = lambda: ctx.compress_device(d_img.data_ptr(), pkg.TYPE_U8, dim, dim, d_whole.data_ptr(), stream=stream.cuda_stream)
        ms, launches = timed(whole_call)
        whole = d_whole.cpu().numpy()
        results.append(dict(config=c, workload=name, case="whole", blocks=total, ms=ms, launches=launches, equal=True))
        rng = np.random.default_rng(2024)
        for k in (1, 121, max(1, total // 100), total // 10, total):
            side = max(1, int(round(k ** 0.5)))
            sx, sy = min(side, nbx), min(-(-k // side), nby)
            x0, y0 = (nbx - sx) // 2, (nby - sy) // 2
            square = ((y0 + np.arange(sy))[:, None] * nbx + (x0 + np.arange(sx))[None, :]).reshape(-1)
            # the block rows that cover the square, through compress_device
            d_rows = torch.zeros(sy * nbx * 16, dtype=torch.uint8, device=dev)
            ms, launches = timed(lambda: ctx.compress_device(d_img.data_ptr(), pkg.TYPE_U8, dim, dim, d_rows.data_ptr(), block_row0=y0, block_rows=sy,
                                                             stream=stream.cuda_stream))
            eq = np.array_equal(d_rows.cpu().numpy(), whole[y0 * nbx * 16:(y0 + sy) * nbx * 16])
            results.append(dict(config=c, workload=name, case="rows:%d" % k, blocks=sy * nbx, ms=ms, launches=launches, equal=bool(eq)))
            for kind, idx in (("list", rng.permutation(total)[:k]), ("square", square)):
                d_work.copy_(d_whole)
                idx = np.ascontiguousarray(idx, dtype=np.uint32)
                ms, launches = timed(lambda: ctx.compress_device_blocks(d_img.data_ptr(), pkg.TYPE_U8, dim, dim, 1, idx, d_work.data_ptr(), stream=stream.cuda_stream))
                eq = np.array_equal(d_work.cpu().numpy(), whole)
                results.append(dict(config=c, workload=name, case="%s:%d" % (kind, k), blocks=len(idx), ms=ms, launches=launches, equal=bool(eq)))
        ctx.close()
    for r in results:
        r["card"] = gpu
        print("config %d  %-14s %8d blocks  %9.3f ms/call  %6.1f launches/call  payload %s" % (r["config"], r["case"], r["blocks"], r["ms"], r["launches"],
                                                                                           "equal" if r["equal"] else "DIFFERS"))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)
    if not all(r["equal"] for r in results):
        sys.exit(1)


if __name__ == "__main__":
    main()
