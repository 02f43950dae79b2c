#!/usr/bin/env python
"""Budget rules for a -fast -> -thorough keep-the-better round over a whole texture set (needs a GPU).

  python tools/pooled_select_probe.py [--reps 5] [--out FILE.json]
  python tools/pooled_select_probe.py --select-ab PARENT_TREE [--rounds 3]

Workloads, every image resident in device memory, LDR, 6x6 blocks, SQUARED_ERROR maps over RGBA:
  set128   256 seeded 128^2 photo_like textures (484 blocks each)
  chain    the 13 levels of bench.py's config 1 image (4096^2 photo_like, seed 2024), tools/multi_image_probe.py's mip_chain
  mixed    64 textures from 32^2 to 512^2, content cycling through photo_like, uniform_noise, smooth_gradient, voronoi_flat and
           alpha_mask
Each workload is compressed at -fast, decoded and mapped once. A round is then one selection on the maps and one
refine_device_block_lists call at -thorough, at total budgets of 1 % and 10 % of the set's blocks, under four rules:
  a  select_blocks per image with capacity max(1, int(n_j * f)) (the budget K is the sum of these)
  b  select_blocks_pooled, one pool of every image with capacity K, no weight
  c  the same with weight 1 / texels_j
  d  the same with weight 1 / E_j, E_j the image's -fast map total, computed on the device
Pooled lists have capacity min(K, n_j) per image: the refine call pays for those padding slots. Reported per rule: the set's total
squared error after the round (the map's unit), mean and worst PSNR over the images (RGBA, 8-bit), the round's time (select +
refine, CUDA events on one stream, median of --reps after a warm-up, with min and max) and the select call's time alone.
--select-ab times select_blocks alone on the config 1 -fast map (0.5 % worst blocks), running this tree and PARENT_TREE (a
checkout of the parent commit with its library built) alternately in child processes. The card's name and power limit are read in the same run and printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

FRACS = (0.01, 0.10)
RULES = ("a", "b", "c", "d")


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi unavailable)"


def workloads():
    import astc_images as I
    from multi_image_probe import mip_chain
    kinds = (I.photo_like, I.uniform_noise, I.smooth_gradient, I.voronoi_flat, I.alpha_mask)
    sizes = (32, 64, 128, 256, 512)
    rng = np.random.default_rng(7)
    mixed = []
    for k in range(64):
        h, w = int(rng.choice(sizes)), int(rng.choice(sizes))
        mixed.append(np.ascontiguousarray(kinds[k % len(kinds)](h, w, seed=500 + k)))
    return {"set128": [np.ascontiguousarray(I.photo_like(128, 128, seed=1000 + k)) for k in range(256)],
            "chain": mip_chain(I.photo_like(4096, 4096, seed=2024)),
            "mixed": mixed}


def events(torch, st, fn, reps):
    fn()
    st.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        fn()
        e1.record(st)
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return {"median_ms": float(np.median(ts)), "min_ms": float(min(ts)), "max_ms": float(max(ts))}


def psnr(img, dec):
    mse = np.mean((img.astype(np.float64) - dec.astype(np.float64)) ** 2)
    return float("inf") if mse == 0 else float(10 * np.log10(255.0 ** 2 / mse))


def probe(args):
    import torch
    import __graft_entry__ as g
    assert torch.cuda.is_available(), "pooled_select_probe.py needs a GPU"
    pkg = g.load_package()
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream(device=dev)
    s = st.cuda_stream
    res = {"card": card(), "workloads": {}}
    print("card: %s" % res["card"], flush=True)
    fast = pkg.Context(pkg.config_init(pkg.PRF_LDR, 6, 6, pkg.PRE_FAST))
    thorough = pkg.Context(pkg.config_init(pkg.PRF_LDR, 6, 6, pkg.PRE_THOROUGH))
    for name, imgs in workloads().items():
        dims = [(im.shape[1], im.shape[0]) for im in imgs]
        nb = [-(-w // 6) * -(-h // 6) for w, h in dims]
        d_img = [torch.from_numpy(im.reshape(-1)).to(dev) for im in imgs]
        pay0 = [torch.zeros(n * 16, dtype=torch.uint8, device=dev) for n in nb]
        dec0 = [torch.zeros(im.size, dtype=torch.uint8, device=dev) for im in imgs]
        map0 = [torch.zeros(n, dtype=torch.float32, device=dev) for n in nb]
        met = torch.zeros(len(imgs) * 128, dtype=torch.uint8, device=dev)
        fast.compress_device_images([(d.data_ptr(), w, h, 1, p.data_ptr()) for d, (w, h), p in zip(d_img, dims, pay0)], pkg.TYPE_U8, stream=s)
        fast.decompress_device_images([(p.data_ptr(), o.data_ptr(), w, h, 1) for p, o, (w, h) in zip(pay0, dec0, dims)], pkg.TYPE_U8, stream=s)
        fast.compute_block_metric_device_images([(d.data_ptr(), o.data_ptr(), pkg.TYPE_U8, pkg.TYPE_U8, w, h, 1, met.data_ptr() + 128 * k, m.data_ptr())
                                                 for k, (d, o, (w, h), m) in enumerate(zip(d_img, dec0, dims, map0))], pkg.BLOCK_SQUARED_ERROR, stream=s)
        st.synchronize()
        fast_psnr = [psnr(im, o.cpu().numpy().reshape(im.shape)) for im, o in zip(imgs, dec0)]
        out = {"images": len(imgs), "blocks": int(sum(nb)), "fast": {"sse": float(sum(float(m.double().sum()) for m in map0)),
                                                                    "mean_psnr": float(np.mean(fast_psnr)), "worst_psnr": float(min(fast_psnr))}}
        print(json.dumps({name: out["fast"], "images": len(imgs), "blocks": out["blocks"]}), flush=True)
        pay = [p.clone() for p in pay0]
        dec = [o.clone() for o in dec0]
        mp = [m.clone() for m in map0]
        texels = torch.tensor([float(w * h) for w, h in dims], dtype=torch.float32, device=dev)
        w_tex = 1.0 / texels
        w_err = torch.zeros(len(imgs), dtype=torch.float32, device=dev)
        for f in FRACS:
            caps_a = [max(1, int(n * f)) for n in nb]
            K = sum(caps_a)
            caps_p = [min(K, n) for n in nb]
            idx = [torch.zeros(max(a, p), dtype=torch.int32, device=dev) for a, p in zip(caps_a, caps_p)]
            cnt = torch.zeros(len(imgs), dtype=torch.int32, device=dev)
            for rule in RULES:
                caps = caps_a if rule == "a" else caps_p

                def select():
                    if rule == "a":
                        fast.select_blocks([(m.data_ptr(), n, -np.inf, c, ix.data_ptr(), cnt.data_ptr() + 4 * k)
                                            for k, (m, n, c, ix) in enumerate(zip(mp, nb, caps, idx))], stream=s)
                        return
                    if rule == "d":
                        with torch.cuda.stream(st):      # 1 / E_j from the maps, on the device, on the round's stream
                            torch.reciprocal(torch.stack([m.sum() for m in mp]), out=w_err)
                    wp = {"b": None, "c": w_tex, "d": w_err}[rule]
                    fast.select_blocks_pooled([(len(imgs), -np.inf, K)],
                                              [(m.data_ptr(), n, wp.data_ptr() + 4 * k if wp is not None else 0, ix.data_ptr(), cnt.data_ptr() + 4 * k)
                                               for k, (m, n, ix) in enumerate(zip(mp, nb, idx))], stream=s)

                def refine():
                    thorough.refine_device_block_lists([(d.data_ptr(), w, h, 1, p.data_ptr(), o.data_ptr(), m.data_ptr(), ix.data_ptr(),
                                                         cnt.data_ptr() + 4 * k, c)
                                                        for k, (d, (w, h), p, o, m, ix, c) in enumerate(zip(d_img, dims, pay, dec, mp, idx, caps))],
                                                       pkg.TYPE_U8, pkg.TYPE_U8, pkg.BLOCK_SQUARED_ERROR, stream=s)

                def restore():
                    with torch.cuda.stream(st):
                        for a, b in zip(pay + dec + mp, pay0 + dec0 + map0):
                            a.copy_(b)

                ts, tsel = [], []
                for r in range(args.reps + 1):
                    restore()
                    e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
                    e0.record(st)
                    select()
                    e1.record(st)
                    refine()
                    e2.record(st)
                    e2.synchronize()
                    if r:      # (the first is the warm-up)
                        ts.append(e0.elapsed_time(e2))
                        tsel.append(e0.elapsed_time(e1))
                p = [psnr(im, o.cpu().numpy().reshape(im.shape)) for im, o in zip(imgs, dec)]
                kept = int(cnt.cpu().numpy().sum())
                row = {"frac": f, "rule": rule, "K": K, "listed": kept, "slots": int(sum(caps)),
                       "sse": float(sum(float(m.double().sum()) for m in mp)), "mean_psnr": float(np.mean(p)), "worst_psnr": float(min(p)),
                       "round_ms": float(np.median(ts)), "round_min_ms": float(min(ts)), "round_max_ms": float(max(ts)),
                       "select_ms": float(np.median(tsel)), "select_min_ms": float(min(tsel)), "select_max_ms": float(max(tsel))}
                out.setdefault("rounds", []).append(row)
                print(json.dumps({name: row}), flush=True)
        res["workloads"][name] = out
        del pay0, dec0, map0, pay, dec, mp, d_img
        torch.cuda.empty_cache()
    fast.close()
    thorough.close()
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


def select_only(args):
    """select_blocks alone on the config 1 -fast map, CUDA events, median of --reps after a warm-up; the package of --root."""
    import torch
    sys.path.insert(0, args.root)
    import __graft_entry__ as g
    import astc_images as I
    pkg = g.load_package()
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream(device=dev)
    s = st.cuda_stream
    img = np.ascontiguousarray(I.photo_like(4096, 4096, seed=2024))
    fast = pkg.Context(pkg.config_init(pkg.PRF_LDR, 6, 6, pkg.PRE_FAST))
    n = fast.blocks(4096, 4096)[0] * fast.blocks(4096, 4096)[1]
    d_img = torch.from_numpy(img.reshape(-1)).to(dev)
    pay = torch.zeros(n * 16, dtype=torch.uint8, device=dev)
    dec = torch.zeros(img.size, dtype=torch.uint8, device=dev)
    mp = torch.zeros(n, dtype=torch.float32, device=dev)
    met = torch.zeros(128, dtype=torch.uint8, device=dev)
    fast.compress_device_images([(d_img.data_ptr(), 4096, 4096, 1, pay.data_ptr())], pkg.TYPE_U8, stream=s)
    fast.decompress_device_images([(pay.data_ptr(), dec.data_ptr(), 4096, 4096, 1)], pkg.TYPE_U8, stream=s)
    fast.compute_error_metrics_device_images([(d_img.data_ptr(), dec.data_ptr(), pkg.TYPE_U8, pkg.TYPE_U8, 4096, 4096, 1, met.data_ptr(), mp.data_ptr())],
                                             stream=s)
    cap = n // 200
    idx = torch.zeros(cap, dtype=torch.int32, device=dev)
    cnt = torch.zeros(1, dtype=torch.int32, device=dev)
    t = events(torch, st, lambda: fast.select_blocks([(mp.data_ptr(), n, -np.inf, cap, idx.data_ptr(), cnt.data_ptr())], stream=s), args.reps)
    st.synchronize()
    print(json.dumps({"select_blocks_config1": t, "blocks": n, "capacity": cap, "list_crc": int(np.bitwise_xor.reduce(idx.cpu().numpy()))}), flush=True)
    fast.close()


def select_ab(args):
    print("card: %s" % card(), flush=True)
    for r in range(args.rounds):
        for name, root in (("parent", os.path.abspath(args.select_ab)), ("this", ROOT)):
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--select-only", "--root", root, "--reps", "50"], capture_output=True, text=True)
            line = [l for l in p.stdout.splitlines() if l.startswith("{")]
            assert p.returncode == 0 and line, p.stderr[-2000:]
            print(json.dumps({"round": r, "build": name, **json.loads(line[-1])}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    ap.add_argument("--select-ab", metavar="PARENT_TREE")
    ap.add_argument("--root", default=ROOT)
    ap.add_argument("--select-only", action="store_true")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if args.select_only:
        select_only(args)
    elif args.select_ab:
        select_ab(args)
    else:
        probe(args)


if __name__ == "__main__":
    main()
