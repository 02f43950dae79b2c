#!/usr/bin/env python
"""Keep-the-better rounds against three-call rounds in a device refinement ladder (needs a GPU).

  python tools/refine_keep_probe.py [--reps 3] [--out FILE.json]

Workloads, every image resident in device memory, 6x6 blocks:
  config1   bench.py's config 1 image (4096^2 photo_like, RGBA8, seed 2024), LDR profile, decoded to U8, SQUARED_ERROR over RGBA
  config3   bench.py's config 3 image (2048^2 hdr_noise, F16, seed 2024), HDR profile, decoded to F16, LOG2_ERROR over RGB
  set128    256 seeded 128^2 photo_like textures, as config1
The ladder: -fast, a whole decode and a whole map, then three rounds of select_blocks (threshold -inf) on the map: -medium on the
worst 10 %, -thorough on the worst 1 %, -exhaustive on the worst 0.1 % of each image's blocks. A round is either
  three     compress_device_block_lists, decompress_device_block_lists, compute_block_metric_device_block_lists (the round's
            context does all three), or
  keep      refine_device_block_lists on the round's context.
All on one stream. Times: ms per ladder (CUDA events around it; median of --reps after one warm-up). Then one more run of each
ladder with a synchronise after every round gives, per round, the share of re-encoded blocks whose map value went up (three) or
that were kept (keep), and the final figure: PSNR (LDR, the mean over the images of set128) or log RMSE (HDR) of the whole decode.
The card's name and power limit are read in the same run and printed with the numbers."""
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

ROUNDS = (("medium", 0.10), ("thorough", 0.01), ("exhaustive", 0.001))


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
    assert torch.cuda.is_available(), "refine_keep_probe.py needs a GPU"
    pkg = g.load_package()
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream(device=dev)
    s = st.cuda_stream
    gpu = card()
    print("card: %s" % gpu)
    mb = C.sizeof(pkg.ErrorMetrics)
    presets = {"fast": pkg.PRE_FAST, "medium": pkg.PRE_MEDIUM, "thorough": pkg.PRE_THOROUGH, "exhaustive": pkg.PRE_EXHAUSTIVE}

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

    class Work:
        def __init__(self, imgs, profile, in_type, out_type, comps, metric):
            self.ctx = {k: pkg.Context(pkg.config_init(profile, 6, 6, q)) for k, q in presets.items()}
            self.in_type, self.out_type, self.comps, self.metric, self.hdr = in_type, out_type, comps, metric, profile == pkg.PRF_HDR
            fast = self.ctx["fast"]
            self.dims = [(im.shape[1], im.shape[0]) for im in imgs]
            self.nb = [fast.blocks(w, h)[0] * fast.blocks(w, h)[1] for w, h in self.dims]
            self.img = [torch.from_numpy(np.ascontiguousarray(im).reshape(-1).view(np.uint8)).to(dev) for im in imgs]
            self.pay = [torch.zeros(n * 16, dtype=torch.uint8, device=dev) for n in self.nb]
            self.dec = [torch.zeros(im.nbytes, dtype=torch.uint8, device=dev) for im in imgs]
            self.met = torch.zeros(len(imgs) * mb, dtype=torch.uint8, device=dev)
            self.map = [torch.zeros(n, dtype=torch.float32, device=dev) for n in self.nb]
            self.idx = [torch.zeros(n, dtype=torch.int32, device=dev) for n in self.nb]
            self.cnt = torch.zeros(len(imgs), dtype=torch.int32, device=dev)

        def close(self):
            for c in self.ctx.values():
                c.close()

        def start(self):
            fast = self.ctx["fast"]
            fast.compress_device_images([(d.data_ptr(), w, h, 1, p.data_ptr()) for d, (w, h), p in zip(self.img, self.dims, self.pay)], self.in_type, stream=s)
            fast.decompress_device_images([(p.data_ptr(), o.data_ptr(), w, h, 1) for p, o, (w, h) in zip(self.pay, self.dec, self.dims)], self.out_type,
                                          stream=s)
            self.whole_map(fast)

        def whole_map(self, ctx):
            ctx.compute_block_metric_device_images([(d.data_ptr(), o.data_ptr(), self.in_type, self.out_type, w, h, 1, self.met.data_ptr() + k * mb,
                                                     m.data_ptr()) for k, (d, o, (w, h), m) in enumerate(zip(self.img, self.dec, self.dims, self.map))],
                                                   self.metric, hdr=self.hdr, input_components=self.comps, stream=s)

        def round(self, name, frac, keep):
            ctx = self.ctx[name]
            caps = [max(1, int(n * frac)) for n in self.nb]
            ctx.select_blocks([(m.data_ptr(), n, -np.inf, c, ix.data_ptr(), self.cnt.data_ptr() + 4 * k)
                               for k, (m, n, c, ix) in enumerate(zip(self.map, self.nb, caps, self.idx))], stream=s)
            lists = list(enumerate(zip(self.img, self.dims, self.pay, self.dec, self.map, self.idx, caps)))
            if keep:
                ctx.refine_device_block_lists([(d.data_ptr(), w, h, 1, p.data_ptr(), o.data_ptr(), m.data_ptr(), ix.data_ptr(), self.cnt.data_ptr() + 4 * k, c)
                                               for k, (d, (w, h), p, o, m, ix, c) in lists], self.in_type, self.out_type, self.metric,
                                              input_components=self.comps, stream=s)
            else:
                ctx.compress_device_block_lists([(d.data_ptr(), w, h, 1, p.data_ptr(), ix.data_ptr(), self.cnt.data_ptr() + 4 * k, c)
                                                 for k, (d, (w, h), p, o, m, ix, c) in lists], self.in_type, stream=s)
                ctx.decompress_device_block_lists([(p.data_ptr(), o.data_ptr(), w, h, 1, ix.data_ptr(), self.cnt.data_ptr() + 4 * k, c)
                                                   for k, (d, (w, h), p, o, m, ix, c) in lists], self.out_type, stream=s)
                ctx.compute_block_metric_device_block_lists([(d.data_ptr(), o.data_ptr(), self.in_type, self.out_type, w, h, 1, m.data_ptr(), ix.data_ptr(),
                                                              self.cnt.data_ptr() + 4 * k, c) for k, (d, (w, h), p, o, m, ix, c) in lists],
                                                            self.metric, input_components=self.comps, stream=s)
            return sum(caps)

        def ladder(self, keep):
            self.start()
            for name, frac in ROUNDS:
                self.round(name, frac, keep)

        def counted(self, keep):
            """The ladder with a synchronise after each round: per round (re-encoded blocks, values that went down, up), then the
            final figure."""
            self.start()
            out = []
            for name, frac in ROUNDS:
                st.synchronize()
                before = torch.cat(self.map).clone()
                n = self.round(name, frac, keep)
                st.synchronize()
                after = torch.cat(self.map)
                out.append(dict(round=name, reencoded=n, lower=int((after < before).sum()), higher=int((after > before).sum())))
            self.ctx["fast"].compute_error_metrics_device_images([(d.data_ptr(), o.data_ptr(), self.in_type, self.out_type, w, h, 1,
                                                                   self.met.data_ptr() + k * mb, 0)
                                                                  for k, (d, o, (w, h)) in enumerate(zip(self.img, self.dec, self.dims))],
                                                                 hdr=self.hdr, input_components=self.comps, stream=s)
            st.synchronize()
            raw = self.met.cpu().numpy()
            figs = [pkg.ErrorMetrics.from_buffer_copy(raw[k * mb:(k + 1) * mb].tobytes()) for k in range(len(self.dims))]
            fig = float(np.mean([f.log_rmse if self.hdr else f.psnr for f in figs]))
            return out, fig

    res = {"card": gpu}
    works = {
        "config1": lambda: Work([astc_images.photo_like(4096, 4096, seed=2024)], pkg.PRF_LDR, pkg.TYPE_U8, pkg.TYPE_U8, 4, pkg.BLOCK_SQUARED_ERROR),
        "config3": lambda: Work([astc_images.hdr_noise(2048, 2048, seed=2024, dtype=np.float16)], pkg.PRF_HDR, pkg.TYPE_F16, pkg.TYPE_F16, 3,
                                pkg.BLOCK_LOG2_ERROR),
        "set128": lambda: Work([astc_images.photo_like(128, 128, seed=k) for k in range(256)], pkg.PRF_LDR, pkg.TYPE_U8, pkg.TYPE_U8, 4,
                               pkg.BLOCK_SQUARED_ERROR),
    }
    for name, make in works.items():
        w = make()
        row = {"images": len(w.dims), "blocks": int(sum(w.nb))}
        for way, keep in (("three", False), ("keep", True)):
            ms = timed(lambda: w.ladder(keep))
            rounds, fig = w.counted(keep)
            row[way] = dict(ladder_ms=ms, rounds=rounds, figure=fig)
            shares = "  ".join("%s %d: %5.1f %% lower, %5.1f %% higher" % (r["round"], r["reencoded"], 100.0 * r["lower"] / r["reencoded"],
                                                                       100.0 * r["higher"] / r["reencoded"]) for r in rounds)
            print("%-8s %-5s ladder %8.2f ms   final %s %.5f   %s" % (name, way, ms, "log RMSE" if w.hdr else "PSNR", fig, shares))
        res[name] = row
        w.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
