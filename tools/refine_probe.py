#!/usr/bin/env python
"""Refining the worst blocks on the device: the closed loop against the host round trip, select_blocks alone, and what the
padding slots of a device block list cost (needs a GPU).

  python tools/refine_probe.py [--reps 3] [--out FILE.json]

Workloads, every image resident in device memory, LDR RGBA8 at 6x6:
  loop_config1  bench.py's config 1 image (4096^2, seed 2024)
  loop_set128   256 seeded 128^2 textures
    device: compress_device_images (-fast) -> decompress_device_images -> compute_error_metrics_device_images with maps ->
            select_blocks (threshold -inf, capacity max(1, blocks // 100)) -> compress_device_block_lists (-thorough), all on
            one stream, one synchronise at the end
    host:   the same first three calls, then a synchronise, every map copied down, a numpy argsort per image and one
            compress_device_blocks (-thorough) per image with the host list
  select        select_blocks alone on config 1's map (466,489 values), capacity 1 %
  padding       compress_device_block_lists on the config 1 image at -medium with capacity 1 %, 10 % and 100 % of its blocks,
                with *count == 0 and with *count == capacity, against compress_device_blocks with a host list of `capacity` blocks
Times: ms per call or chain (CUDA events on the stream around it; median of --reps after one warm-up). The final payloads of the
two loops are compared byte for byte. The card's name and power limit are read in the same run and printed with the numbers."""
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


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi unavailable)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    import __graft_entry__ as g
    import astc_images
    assert torch.cuda.is_available(), "refine_probe.py needs a GPU"
    pkg = g.load_package()
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream(device=dev)
    s = st.cuda_stream
    gpu = card()
    print("card: %s" % gpu)
    S = pkg.FLG_SELF_DECOMPRESS_ONLY
    fast = pkg.Context(pkg.config_init(pkg.PRF_LDR, 6, 6, pkg.PRE_FAST, S))
    thorough = pkg.Context(pkg.config_init(pkg.PRF_LDR, 6, 6, pkg.PRE_THOROUGH, S))
    medium = pkg.Context(pkg.config_init(pkg.PRF_LDR, 6, 6, pkg.PRE_MEDIUM, S))
    mb = C.sizeof(pkg.ErrorMetrics)

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

    class Set:
        def __init__(self, imgs):
            self.dims = [(im.shape[1], im.shape[0]) for im in imgs]
            self.nb = [fast.blocks(w, h)[0] * fast.blocks(w, h)[1] for w, h in self.dims]
            self.caps = [max(1, n // 100) for n in self.nb]
            self.img = [torch.from_numpy(im.reshape(-1)).to(dev) for im in imgs]
            self.pay = [torch.zeros(n * 16, dtype=torch.uint8, device=dev) for n in self.nb]
            self.dec = [torch.zeros(im.size, dtype=torch.uint8, device=dev) for im in imgs]
            self.met = torch.zeros(len(imgs) * mb, dtype=torch.uint8, device=dev)
            self.map = [torch.zeros(n, dtype=torch.float32, device=dev) for n in self.nb]
            self.idx = [torch.zeros(c, dtype=torch.int32, device=dev) for c in self.caps]
            self.cnt = torch.zeros(len(imgs), dtype=torch.int32, device=dev)

        def measure(self):
            fast.compress_device_images([(d.data_ptr(), w, h, 1, p.data_ptr()) for d, (w, h), p in zip(self.img, self.dims, self.pay)], pkg.TYPE_U8, stream=s)
            fast.decompress_device_images([(p.data_ptr(), o.data_ptr(), w, h, 1) for p, o, (w, h) in zip(self.pay, self.dec, self.dims)], pkg.TYPE_U8, stream=s)
            fast.compute_error_metrics_device_images([(d.data_ptr(), o.data_ptr(), pkg.TYPE_U8, pkg.TYPE_U8, w, h, 1, self.met.data_ptr() + k * mb, m.data_ptr())
                                                      for k, (d, o, (w, h), m) in enumerate(zip(self.img, self.dec, self.dims, self.map))], stream=s)

        def device_loop(self):
            self.measure()
            fast.select_blocks([(m.data_ptr(), n, -np.inf, c, ix.data_ptr(), self.cnt.data_ptr() + 4 * k)
                                for k, (m, n, c, ix) in enumerate(zip(self.map, self.nb, self.caps, self.idx))], stream=s)
            thorough.compress_device_block_lists([(d.data_ptr(), w, h, 1, p.data_ptr(), ix.data_ptr(), self.cnt.data_ptr() + 4 * k, c)
                                                  for k, (d, (w, h), p, ix, c) in enumerate(zip(self.img, self.dims, self.pay, self.idx, self.caps))],
                                                 pkg.TYPE_U8, stream=s)

        def host_loop(self):
            self.measure()
            st.synchronize()
            maps = [m.cpu().numpy() for m in self.map]
            for d, (w, h), p, m, c in zip(self.img, self.dims, self.pay, maps, self.caps):
                thorough.compress_device_blocks(d.data_ptr(), pkg.TYPE_U8, w, h, 1, np.argsort(-m, kind="stable")[:c], p.data_ptr(), stream=s)

    res = {"card": gpu}
    config1 = astc_images.photo_like(4096, 4096, seed=2024)
    sets = {"loop_config1": [config1], "loop_set128": [astc_images.photo_like(128, 128, seed=k) for k in range(256)]}
    for name, imgs in sets.items():
        w = Set(imgs)
        dev_ms = timed(w.device_loop)
        st.synchronize()
        got = [p.cpu().numpy() for p in w.pay]
        host_ms = timed(w.host_loop)
        st.synchronize()
        same = all(np.array_equal(a, p.cpu().numpy()) for a, p in zip(got, w.pay))
        res[name] = dict(device_ms=dev_ms, host_ms=host_ms, images=len(imgs), same_bytes=same)
        print("%-13s device chain %9.2f ms   host round trip %9.2f ms   (%d images, payloads equal: %s)" % (name, dev_ms, host_ms, len(imgs), same))
        if name == "loop_config1":
            big = w
    # select_blocks alone on config 1's map
    sel_ms = timed(lambda: fast.select_blocks([(big.map[0].data_ptr(), big.nb[0], -np.inf, big.caps[0], big.idx[0].data_ptr(), big.cnt.data_ptr())], stream=s))
    res["select"] = dict(ms=sel_ms, values=big.nb[0], capacity=big.caps[0])
    print("select_blocks alone: %d values, capacity %d: %.3f ms" % (big.nb[0], big.caps[0], sel_ms))
    # padding
    n = big.nb[0]
    W, H = big.dims[0]
    rng = np.random.default_rng(7)
    perm = np.sort(rng.permutation(n)).astype(np.uint32)
    res["padding"] = []
    for frac in (0.01, 0.10, 1.0):
        cap = max(1, int(n * frac))
        lst = np.sort(rng.choice(n, size=cap, replace=False)).astype(np.uint32) if frac < 1.0 else perm
        d_idx = torch.from_numpy(lst.view(np.int32)).to(dev)
        d_cnt = torch.tensor([0, cap], dtype=torch.int32, device=dev)
        row = {"capacity": cap}
        for label, off in (("count0", 0), ("full", 4)):
            row[label + "_ms"] = timed(lambda: medium.compress_device_block_lists(
                [(big.img[0].data_ptr(), W, H, 1, big.pay[0].data_ptr(), d_idx.data_ptr(), d_cnt.data_ptr() + off, cap)], pkg.TYPE_U8, stream=s))
        row["host_list_ms"] = timed(lambda: medium.compress_device_blocks(big.img[0].data_ptr(), pkg.TYPE_U8, W, H, 1, lst, big.pay[0].data_ptr(), stream=s))
        res["padding"].append(row)
        print("padding, capacity %7d (%3d %%): *count == 0 %8.2f ms   *count == capacity %8.2f ms   host list %8.2f ms"
              % (cap, round(frac * 100), row["count0_ms"], row["full_ms"], row["host_list_ms"]))
    for c in (fast, thorough, medium):
        c.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
