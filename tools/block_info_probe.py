#!/usr/bin/env python
"""Block info of device payloads: astcenc_b200_get_block_summaries_device_images and astcenc_b200_get_block_info_device_block_lists
against astcenc_get_block_info per block (needs a GPU).

  python tools/block_info_probe.py [--reps 9] [--out FILE.json]

Workloads, payloads made on the device at 6x6 -fast (LDR) and left there:
  config1     bench.py's config 1 image (4096^2 photo_like, seed 2024): 466,489 blocks
  set128      256 seeded 128^2 textures
  chain_tail  the 12 levels below the base of config 1's mip chain (2048^2 down to 1 x 1), one call
Reported: the summary call's time from a prebuilt descriptor table (CUDA events on the launching stream around the call: its
host checks, table copy and launch; median of --reps after a warm-up, with min and max) and achieved bytes/s over 32 bytes per block (16 read, 16 written); the list call on config 1 at 1 % and 10 % of its
blocks (random sorted indices, device count); astcenc_get_block_info per call over 1,000 blocks of config 1 (host clock: each
call returns with the struct in host memory); astcenc_b200_decompress_device_images of config 1 into U8, for scale. Then the
motivating use: the partition-count and dual-plane histograms of config 1 after -fast and after one -thorough keep-the-better
round over its worst 1 % (select_blocks, refine_device_block_lists), read from the summaries. The card's name and power
limit are read in the same run."""
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
sys.path.insert(0, os.path.join(ROOT, "tools"))


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi unavailable)"


def timed(torch, st, fn, reps):
    """Median, min and max ms of fn() enqueued on st, CUDA events, after one warm-up."""
    ts = []
    for r in range(reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        fn()
        e1.record(st)
        e1.synchronize()
        if r:
            ts.append(e0.elapsed_time(e1))
    return {"ms": float(np.median(ts)), "min_ms": float(min(ts)), "max_ms": float(max(ts))}


def probe(args):
    import ctypes as C
    import torch
    import __graft_entry__ as g
    import astc_images as I
    from decode_probe import mip_chain
    assert torch.cuda.is_available(), "block_info_probe.py needs a GPU"
    pkg = g.load_package()
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream(device=dev)
    s = st.cuda_stream
    res = {"card": card()}
    print("card: %s" % res["card"], flush=True)
    fast = pkg.Context(pkg.config_init(pkg.PRF_LDR, 6, 6, pkg.PRE_FAST))
    thorough = pkg.Context(pkg.config_init(pkg.PRF_LDR, 6, 6, pkg.PRE_THOROUGH))
    nblk = lambda w, h: -(-w // 6) * -(-h // 6)

    def check(err):
        assert err == 0, err

    def upload(imgs):
        dims = [(im.shape[1], im.shape[0]) for im in imgs]
        d_img = [torch.from_numpy(np.ascontiguousarray(im).reshape(-1)).to(dev) for im in imgs]
        pay = [torch.zeros(nblk(w, h) * 16, dtype=torch.uint8, device=dev) for w, h in dims]
        fast.compress_device_images([(d.data_ptr(), w, h, 1, p.data_ptr()) for d, (w, h), p in zip(d_img, dims, pay)], pkg.TYPE_U8, stream=s)
        st.synchronize()
        return dims, d_img, pay

    base = np.ascontiguousarray(I.photo_like(4096, 4096, seed=2024))
    work = {"config1": [base], "set128": [I.photo_like(128, 128, seed=1000 + k) for k in range(256)], "chain_tail": mip_chain(base)[1:]}
    res["summaries"] = {}
    keep = {}
    for name, imgs in work.items():
        dims, d_img, pay = upload(imgs)
        nb = [nblk(w, h) for w, h in dims]
        summ = [torch.zeros(n * 16, dtype=torch.uint8, device=dev) for n in nb]
        # (the descriptor table is built once: the timed window holds the call itself, not the Python that builds its table)
        table = (pkg.DeviceBlockSummaryImage * len(pay))(*[pkg.DeviceBlockSummaryImage(C.c_void_p(p.data_ptr()), w, h, 1, C.c_void_p(o.data_ptr()))
                                                            for p, (w, h), o in zip(pay, dims, summ)])
        call = lambda: check(pkg.lib().astcenc_b200_get_block_summaries_device_images(fast.handle, table, len(pay), C.c_void_p(s)))
        t = timed(torch, st, call, args.reps)
        t.update(images=len(imgs), blocks=int(sum(nb)), GBps=32.0 * sum(nb) / (t["ms"] * 1e-3) / 1e9)
        res["summaries"][name] = t
        print(json.dumps({"summaries_" + name: t}), flush=True)
        if name == "config1":
            keep = dict(dims=dims, d_img=d_img, pay=pay, summ=summ, n=nb[0])
        else:
            del d_img, pay, summ

    # the list call on config 1
    (w, h), n = keep["dims"][0], keep["n"]
    pay, d_img = keep["pay"][0], keep["d_img"][0]
    rng = np.random.default_rng(1)
    res["lists"] = {}
    for f in (0.01, 0.10):
        k = int(n * f)
        idx = torch.from_numpy(np.sort(rng.choice(n, k, replace=False)).astype(np.int32)).to(dev)
        cnt = torch.tensor([k], dtype=torch.int32, device=dev)
        infos = torch.zeros(k * pkg.BLOCK_INFO_BYTES, dtype=torch.uint8, device=dev)
        t = timed(torch, st, lambda: fast.get_block_info_device_block_lists([(pay.data_ptr(), w, h, 1, idx.data_ptr(), cnt.data_ptr(), k, infos.data_ptr())],
                                                                            stream=s), args.reps)
        t.update(slots=k, us_per_slot=t["ms"] * 1e3 / k)
        res["lists"]["%d%%" % round(f * 100)] = t
        print(json.dumps({"list_%d%%" % round(f * 100): t}), flush=True)
        del infos

    # astcenc_get_block_info, one call per block
    host = pay.cpu().numpy().reshape(-1, 16)
    info = pkg.lib()
    buf = (C.c_uint8 * pkg.BLOCK_INFO_BYTES)()
    info.astcenc_get_block_info.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    blocks = [np.ascontiguousarray(host[i]) for i in rng.choice(n, 1000, replace=False)]
    info.astcenc_get_block_info(fast.handle, blocks[0].ctypes.data, buf)
    t0 = time.perf_counter()
    for b in blocks:
        assert info.astcenc_get_block_info(fast.handle, b.ctypes.data, buf) == 0
    per = (time.perf_counter() - t0) / len(blocks)
    res["get_block_info"] = {"calls": len(blocks), "us_per_call": per * 1e6, "config1_s_extrapolated": per * n}
    print(json.dumps({"get_block_info": res["get_block_info"]}), flush=True)

    # the whole-payload decode, for scale
    dec = torch.zeros(w * h * 4, dtype=torch.uint8, device=dev)
    t = timed(torch, st, lambda: fast.decompress_device_images([(pay.data_ptr(), dec.data_ptr(), w, h, 1)], pkg.TYPE_U8, stream=s), args.reps)
    res["decode_config1_u8"] = t
    print(json.dumps({"decode_config1_u8": t}), flush=True)

    # the motivating use: what one -thorough round over the worst 1 % did to the encoding
    def histograms():
        fast.get_block_summaries_device_images([(pay.data_ptr(), w, h, 1, keep["summ"][0].data_ptr())], stream=s)
        st.synchronize()
        sm = keep["summ"][0].cpu().numpy().view(pkg.BLOCK_SUMMARY_DTYPE)
        return {"partition_count": {str(p): int((sm["partition_count"] == p).sum()) for p in range(5)},
                "dual_plane": int(((sm["flags"] & pkg.BLOCK_IS_DUAL_PLANE) != 0).sum()),
                "constant": int(((sm["flags"] & pkg.BLOCK_IS_CONSTANT) != 0).sum()), "error": int(((sm["flags"] & pkg.BLOCK_IS_ERROR) != 0).sum())}

    res["histograms"] = {"fast": histograms()}
    fast.decompress_device_images([(pay.data_ptr(), dec.data_ptr(), w, h, 1)], pkg.TYPE_U8, stream=s)
    mp = torch.zeros(n, dtype=torch.float32, device=dev)
    met = torch.zeros(128, dtype=torch.uint8, device=dev)
    fast.compute_block_metric_device_images([(d_img.data_ptr(), dec.data_ptr(), pkg.TYPE_U8, pkg.TYPE_U8, w, h, 1, met.data_ptr(), mp.data_ptr())],
                                            pkg.BLOCK_SQUARED_ERROR, stream=s)
    cap = n // 100
    idx = torch.zeros(cap, dtype=torch.int32, device=dev)
    cnt = torch.zeros(1, dtype=torch.int32, device=dev)
    fast.select_blocks([(mp.data_ptr(), n, -np.inf, cap, idx.data_ptr(), cnt.data_ptr())], stream=s)
    thorough.refine_device_block_lists([(d_img.data_ptr(), w, h, 1, pay.data_ptr(), dec.data_ptr(), mp.data_ptr(), idx.data_ptr(), cnt.data_ptr(), cap)],
                                       pkg.TYPE_U8, pkg.TYPE_U8, pkg.BLOCK_SQUARED_ERROR, stream=s)
    res["histograms"]["after_thorough_1pct_keep_round"] = histograms()
    print(json.dumps({"histograms": res["histograms"]}), flush=True)
    fast.close()
    thorough.close()
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--out")
    probe(ap.parse_args())


if __name__ == "__main__":
    main()
