#!/usr/bin/env python
"""List refreshes against whole-image refreshes: decode and map calls over device block lists, and a refine ladder that
re-decodes and re-measures through them (needs a GPU).

  python tools/list_refresh_probe.py [--reps 3] [--out FILE.json]

Workloads, every image resident in device memory, LDR RGBA8 at 6x6, payloads compressed at -fast:
  config1   bench.py's config 1 image (4096^2, seed 2024)
  set128    256 seeded 128^2 textures
    whole:  decompress_device_images of every payload; compute_error_metrics_device_images with maps (figures included)
    lists:  decompress_device_block_lists and compute_block_errors_device_block_lists over sorted random lists of 0.1 %, 1 %,
            10 % and 100 % of each image's blocks (at least one), *count == capacity
  ladder    on both workloads: -fast, decode, maps, then three rounds of select_blocks (threshold -inf) ->
            compress_device_block_lists -> refresh: -medium on the worst 10 %, -thorough on the worst 1 %, -exhaustive on the
            worst 0.1 %. The refresh is a list decode and a list map, or a whole decode and a whole map. All on one stream, one
            synchronise at the end; the final payloads, decodes and maps of the two ladders are compared byte for byte.
Times: ms per call or ladder (CUDA events on the stream around it; median of --reps after one warm-up). The card's name and power
limit are read in the same run and printed with the numbers."""
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

FRACTIONS = (0.001, 0.01, 0.10, 1.0)


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
    assert torch.cuda.is_available(), "list_refresh_probe.py needs a GPU"
    pkg = g.load_package()
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream(device=dev)
    s = st.cuda_stream
    gpu = card()
    print("card: %s" % gpu)
    S = pkg.FLG_SELF_DECOMPRESS_ONLY
    ctx = {q: pkg.Context(pkg.config_init(pkg.PRF_LDR, 6, 6, q, S)) for q in (pkg.PRE_FAST, pkg.PRE_MEDIUM, pkg.PRE_THOROUGH, pkg.PRE_EXHAUSTIVE)}
    fast = ctx[pkg.PRE_FAST]
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

    class Set:
        def __init__(self, imgs):
            self.dims = [(im.shape[1], im.shape[0]) for im in imgs]
            self.nb = [fast.blocks(w, h)[0] * fast.blocks(w, h)[1] for w, h in self.dims]
            self.img = [torch.from_numpy(im.reshape(-1)).to(dev) for im in imgs]
            self.pay = [torch.zeros(n * 16, dtype=torch.uint8, device=dev) for n in self.nb]
            self.dec = [torch.zeros(im.size, dtype=torch.uint8, device=dev) for im in imgs]
            self.met = torch.zeros(len(imgs) * mb, dtype=torch.uint8, device=dev)
            self.map = [torch.zeros(n, dtype=torch.float32, device=dev) for n in self.nb]
            self.idx = [torch.zeros(n, dtype=torch.int32, device=dev) for n in self.nb]
            self.cnt = torch.zeros(len(imgs), dtype=torch.int32, device=dev)

        def compress_fast(self):
            fast.compress_device_images([(d.data_ptr(), w, h, 1, p.data_ptr()) for d, (w, h), p in zip(self.img, self.dims, self.pay)], U8, stream=s)

        def whole_decode(self):
            fast.decompress_device_images([(p.data_ptr(), o.data_ptr(), w, h, 1) for p, o, (w, h) in zip(self.pay, self.dec, self.dims)], U8, stream=s)

        def whole_map(self):
            fast.compute_error_metrics_device_images([(d.data_ptr(), o.data_ptr(), U8, U8, w, h, 1, self.met.data_ptr() + k * mb, m.data_ptr())
                                                      for k, (d, o, (w, h), m) in enumerate(zip(self.img, self.dec, self.dims, self.map))], stream=s)

        def list_decode(self, caps):
            fast.decompress_device_block_lists([(p.data_ptr(), o.data_ptr(), w, h, 1, ix.data_ptr(), self.cnt.data_ptr() + 4 * k, c)
                                                for k, (p, o, (w, h), ix, c) in enumerate(zip(self.pay, self.dec, self.dims, self.idx, caps))], U8, stream=s)

        def list_map(self, caps):
            fast.compute_block_errors_device_block_lists([(d.data_ptr(), o.data_ptr(), U8, U8, w, h, 1, m.data_ptr(), ix.data_ptr(), self.cnt.data_ptr() + 4 * k, c)
                                                          for k, (d, o, (w, h), m, ix, c) in enumerate(zip(self.img, self.dec, self.dims, self.map, self.idx, caps))],
                                                         stream=s)

        def ladder(self, lists):
            self.compress_fast()
            self.whole_decode()
            self.whole_map()
            for q, frac in ((pkg.PRE_MEDIUM, 0.10), (pkg.PRE_THOROUGH, 0.01), (pkg.PRE_EXHAUSTIVE, 0.001)):
                caps = [max(1, int(n * frac)) for n in self.nb]
                fast.select_blocks([(m.data_ptr(), n, -np.inf, c, ix.data_ptr(), self.cnt.data_ptr() + 4 * k)
                                    for k, (m, n, c, ix) in enumerate(zip(self.map, self.nb, caps, self.idx))], stream=s)
                ctx[q].compress_device_block_lists([(d.data_ptr(), w, h, 1, p.data_ptr(), ix.data_ptr(), self.cnt.data_ptr() + 4 * k, c)
                                                    for k, (d, (w, h), p, ix, c) in enumerate(zip(self.img, self.dims, self.pay, self.idx, caps))], U8, stream=s)
                if lists:
                    self.list_decode(caps)
                    self.list_map(caps)
                else:
                    self.whole_decode()
                    self.whole_map()

        def outputs(self):
            st.synchronize()
            return [t.cpu().numpy().copy() for t in self.pay + self.dec + self.map]

    res = {"card": gpu}
    sets = {"config1": [astc_images.photo_like(4096, 4096, seed=2024)], "set128": [astc_images.photo_like(128, 128, seed=k) for k in range(256)]}
    rng = np.random.default_rng(7)
    for name, imgs in sets.items():
        w = Set(imgs)
        w.compress_fast()
        st.synchronize()
        row = {"images": len(imgs), "blocks": int(sum(w.nb))}
        row["whole_decode_ms"] = timed(w.whole_decode)
        row["whole_map_ms"] = timed(w.whole_map)
        print("%-8s %d images, %d blocks: whole decode %8.3f ms   whole map (with figures) %8.3f ms"
              % (name, len(imgs), row["blocks"], row["whole_decode_ms"], row["whole_map_ms"]))
        row["lists"] = []
        for frac in FRACTIONS:
            caps = [max(1, int(n * frac)) for n in w.nb]
            for ix, n, c in zip(w.idx, w.nb, caps):
                ix[:c].copy_(torch.from_numpy(np.sort(rng.choice(n, size=c, replace=False)).astype(np.int32)))
            w.cnt.copy_(torch.tensor(caps, dtype=torch.int32))
            st.synchronize()
            r = {"fraction": frac, "slots": int(sum(caps))}
            r["list_decode_ms"] = timed(lambda: w.list_decode(caps))
            r["list_map_ms"] = timed(lambda: w.list_map(caps))
            row["lists"].append(r)
            print("%-8s %6.1f %% (%7d slots): list decode %8.3f ms (%5.2fx of whole)   list map %8.3f ms (%5.2fx of whole)"
                  % (name, frac * 100, r["slots"], r["list_decode_ms"], r["list_decode_ms"] / row["whole_decode_ms"], r["list_map_ms"],
                     r["list_map_ms"] / row["whole_map_ms"]))
        list_ms = timed(lambda: w.ladder(True))
        got_lists = w.outputs()
        whole_ms = timed(lambda: w.ladder(False))
        got_whole = w.outputs()
        same = all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for a, b in zip(got_lists, got_whole))
        row["ladder"] = dict(list_refresh_ms=list_ms, whole_refresh_ms=whole_ms, same_bytes=same)
        print("%-8s ladder (fast -> medium 10 %% -> thorough 1 %% -> exhaustive 0.1 %%): list refreshes %8.2f ms   whole refreshes %8.2f ms   "
              "(payloads, decodes and maps equal: %s)" % (name, list_ms, whole_ms, same))
        res[name] = row
    for c in ctx.values():
        c.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
