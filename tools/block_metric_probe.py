#!/usr/bin/env python
"""Per-block error maps of each metric (astcenc_b200_compute_block_metric_device_images and
astcenc_b200_compute_block_metric_device_block_lists): call times, and what LOG2 selection buys an HDR refine loop (needs a GPU).

  python tools/block_metric_probe.py [--reps 7] [--out FILE.json]

Workloads, every image resident in device memory, 6x6, payloads compressed at -fast and decoded on the device:
  config3   bench.py's config 3 image (2048^2 hdr_noise, F16, seed 2024), HDR profile, decoded to F16; maps over RGB
            (input_components 3), figures with hdr=1 (fstop -10..10)
  config1   bench.py's config 1 image (4096^2 photo_like, RGBA8, seed 2024), LDR profile, decoded to U8; maps over RGBA
    whole:  one whole call with figures and a map, per metric
    list:   one list refresh over a sorted random list of 1 % of the blocks (*count == capacity), per metric
  loop      on config3, selecting by SQUARED_ERROR and by LOG2_ERROR: -fast, decode, map, select_blocks (threshold -inf) of the
            worst 1 %, 5 % and 10 %, -thorough compress_device_block_lists, list decode, list refresh; all on one stream. The final
            log_rmse and mpsnr, the loop's time, and whether its payload equals the host round trip's (synchronise, map down,
            numpy argsort, compress_device_blocks). -fast and whole -thorough figures frame the gap.
Times: ms per call or loop (CUDA events on the stream around it; median of --reps after one warm-up). The card's name and power
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

FRACTIONS = (0.01, 0.05, 0.10)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi unavailable)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out")
    args = ap.parse_args()
    assert args.reps >= 5, "at least 5 timed repetitions"
    import torch
    import __graft_entry__ as g
    import astc_images
    assert torch.cuda.is_available(), "block_metric_probe.py needs a GPU"
    pkg = g.load_package()
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream(device=dev)
    s = st.cuda_stream
    gpu = card()
    print("card: %s" % gpu)
    S = pkg.FLG_SELF_DECOMPRESS_ONLY
    mb = C.sizeof(pkg.ErrorMetrics)
    names = {pkg.BLOCK_SQUARED_ERROR: "SQUARED_ERROR", pkg.BLOCK_ALPHA_WEIGHTED_ERROR: "ALPHA_WEIGHTED_ERROR", pkg.BLOCK_LOG2_ERROR: "LOG2_ERROR"}

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
        def __init__(self, img, profile, in_type, out_type, comps, hdr):
            self.h, self.w = img.shape[:2]
            self.in_type, self.out_type, self.comps, self.hdr = in_type, out_type, comps, hdr
            self.fast = pkg.Context(pkg.config_init(profile, 6, 6, pkg.PRE_FAST, S))
            self.thorough = pkg.Context(pkg.config_init(profile, 6, 6, pkg.PRE_THOROUGH, S))
            # decodes and measures: a decompress-only context decodes every block mode (a SELF_DECOMPRESS_ONLY -fast context
            # decodes only the modes its own preset emits, not the -thorough blocks)
            self.dec_ctx = pkg.Context(pkg.config_init(profile, 6, 6, pkg.PRE_FAST, pkg.FLG_DECOMPRESS_ONLY))
            bx, by = self.fast.blocks(self.w, self.h)
            self.n = bx * by
            self.img = torch.from_numpy(img.reshape(-1).view(np.uint8)).to(dev)
            self.pay = torch.zeros(self.n * 16, dtype=torch.uint8, device=dev)
            self.dec = torch.zeros(self.h * self.w * 4 * (2 if out_type == pkg.TYPE_F16 else 1), dtype=torch.uint8, device=dev)
            self.met = torch.zeros(mb, dtype=torch.uint8, device=dev)
            self.map = torch.zeros(self.n, dtype=torch.float32, device=dev)
            self.idx = torch.zeros(self.n, dtype=torch.int32, device=dev)
            self.cnt = torch.zeros(1, dtype=torch.int32, device=dev)

        def compress_fast(self, pay=None):
            self.fast.compress_device_images([(self.img.data_ptr(), self.w, self.h, 1, (pay if pay is not None else self.pay).data_ptr())], self.in_type, stream=s)

        def decode(self, pay=None, dec=None):
            self.dec_ctx.decompress_device_images([((pay if pay is not None else self.pay).data_ptr(), (dec if dec is not None else self.dec).data_ptr(),
                                                 self.w, self.h, 1)], self.out_type, stream=s)

        def whole(self, metric, dec=None, mp=None):
            self.dec_ctx.compute_block_metric_device_images([(self.img.data_ptr(), (dec if dec is not None else self.dec).data_ptr(), self.in_type, self.out_type,
                                                           self.w, self.h, 1, self.met.data_ptr(), (mp if mp is not None else self.map).data_ptr())],
                                                         metric, hdr=self.hdr, input_components=self.comps, stream=s)

        def refresh(self, metric, cap):
            self.dec_ctx.compute_block_metric_device_block_lists([(self.img.data_ptr(), self.dec.data_ptr(), self.in_type, self.out_type, self.w, self.h, 1,
                                                                self.map.data_ptr(), self.idx.data_ptr(), self.cnt.data_ptr(), cap)], metric,
                                                              input_components=self.comps, stream=s)

        def loop(self, metric, cap):
            self.compress_fast()
            self.decode()
            self.whole(metric)
            self.dec_ctx.select_blocks([(self.map.data_ptr(), self.n, -np.inf, cap, self.idx.data_ptr(), self.cnt.data_ptr())], stream=s)
            self.thorough.compress_device_block_lists([(self.img.data_ptr(), self.w, self.h, 1, self.pay.data_ptr(), self.idx.data_ptr(), self.cnt.data_ptr(),
                                                        cap)], self.in_type, stream=s)
            self.dec_ctx.decompress_device_block_lists([(self.pay.data_ptr(), self.dec.data_ptr(), self.w, self.h, 1, self.idx.data_ptr(), self.cnt.data_ptr(),
                                                      cap)], self.out_type, stream=s)
            self.refresh(metric, cap)

        def figures(self, pay):
            """log_rmse and mpsnr (hdr=1, RGB) of a payload's decode."""
            dec = torch.zeros_like(self.dec)
            torch.cuda.synchronize()      # (the zero fill runs on the current stream, the decode on s)
            self.decode(pay, dec)
            self.dec_ctx.compute_error_metrics_device_images([(self.img.data_ptr(), dec.data_ptr(), self.in_type, self.out_type, self.w, self.h, 1,
                                                            self.met.data_ptr(), 0)], hdr=True, input_components=3, stream=s)
            st.synchronize()
            m = pkg.ErrorMetrics.from_buffer_copy(self.met.cpu().numpy().tobytes())
            return dict(log_rmse=m.log_rmse, mpsnr=m.mpsnr)

        def host_round_trip(self, metric, cap):
            pay = torch.zeros_like(self.pay)
            mp = torch.zeros_like(self.map)
            dec = torch.zeros_like(self.dec)
            torch.cuda.synchronize()
            self.compress_fast(pay)
            self.decode(pay, dec)
            self.whole(metric, dec, mp)
            st.synchronize()
            worst = np.sort(np.argsort(-mp.cpu().numpy(), kind="stable")[:cap]).astype(np.uint32)
            self.thorough.compress_device_blocks(self.img.data_ptr(), self.in_type, self.w, self.h, 1, worst, pay.data_ptr(), stream=s)
            st.synchronize()
            return pay

        def close(self):
            self.fast.close()
            self.thorough.close()
            self.dec_ctx.close()

    res = {"card": gpu, "reps": args.reps}
    hdr = np.ascontiguousarray(astc_images.hdr_noise(2048, 2048, seed=2024, dtype=np.float16))
    ldr = np.ascontiguousarray(astc_images.photo_like(4096, 4096, seed=2024))
    works = {"config3": Work(hdr, pkg.PRF_HDR, pkg.TYPE_F16, pkg.TYPE_F16, 3, True),
             "config1": Work(ldr, pkg.PRF_LDR, pkg.TYPE_U8, pkg.TYPE_U8, 4, False)}
    torch.cuda.synchronize()      # (uploads and zero fills run on the current stream; every call below runs on s)
    rng = np.random.default_rng(7)
    for name, w in works.items():
        w.compress_fast()
        w.decode()
        cap = max(1, w.n // 100)
        w.idx[:cap].copy_(torch.from_numpy(np.sort(rng.choice(w.n, size=cap, replace=False)).astype(np.int32)))
        w.cnt.fill_(cap)
        torch.cuda.synchronize()
        row = {"blocks": w.n, "list_slots": cap}
        for metric in sorted(names):
            row["whole_ms_" + names[metric]] = timed(lambda: w.whole(metric))
            row["list_1pct_ms_" + names[metric]] = timed(lambda: w.refresh(metric, cap))
            print("%-8s %-21s whole call (figures + map, %d blocks) %7.3f ms   1 %% list refresh (%d slots) %7.3f ms"
                  % (name, names[metric], w.n, row["whole_ms_" + names[metric]], cap, row["list_1pct_ms_" + names[metric]]))
        res[name] = row

    w = works["config3"]
    fast_pay = torch.zeros_like(w.pay)
    thorough_pay = torch.zeros_like(w.pay)
    torch.cuda.synchronize()
    w.compress_fast(fast_pay)
    w.thorough.compress_device_images([(w.img.data_ptr(), w.w, w.h, 1, thorough_pay.data_ptr())], w.in_type, stream=s)
    st.synchronize()
    loop = {"fast": w.figures(fast_pay), "thorough": w.figures(thorough_pay), "runs": []}
    print("config3  -fast      log_rmse %.5f  mpsnr %.3f dB" % (loop["fast"]["log_rmse"], loop["fast"]["mpsnr"]))
    print("config3  -thorough  log_rmse %.5f  mpsnr %.3f dB" % (loop["thorough"]["log_rmse"], loop["thorough"]["mpsnr"]))
    for frac in FRACTIONS:
        cap = max(1, int(w.n * frac))
        for metric in (pkg.BLOCK_SQUARED_ERROR, pkg.BLOCK_LOG2_ERROR):
            ms = timed(lambda: w.loop(metric, cap))
            st.synchronize()
            fig = w.figures(w.pay)
            same = bool(torch.equal(w.pay, w.host_round_trip(metric, cap)))
            gap = loop["fast"]["log_rmse"] - loop["thorough"]["log_rmse"]
            closed = (loop["fast"]["log_rmse"] - fig["log_rmse"]) / gap if gap > 0 else float("nan")
            r = dict(fraction=frac, metric=names[metric], blocks=cap, loop_ms=ms, same_as_host_round_trip=same, log_gap_closed=closed, **fig)
            loop["runs"].append(r)
            print("config3  worst %4.1f %% by %-13s log_rmse %.5f (%5.1f %% of the -fast/-thorough gap)  mpsnr %.3f dB  loop %7.2f ms  "
                  "payload equals the host round trip: %s" % (frac * 100, names[metric], fig["log_rmse"], closed * 100, fig["mpsnr"], ms, same))
    res["loop_config3"] = loop
    for x in works.values():
        x.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
