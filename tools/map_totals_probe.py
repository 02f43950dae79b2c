#!/usr/bin/env python
"""Map totals on the device (astcenc_b200_total_block_maps) in the refinement loop (needs a GPU).

  python tools/map_totals_probe.py [--reps 20] [--out FILE.json]
  python tools/map_totals_probe.py --bench-ab PARENT_TREE [--rounds 2]

Workloads, LDR, 6x6, SQUARED_ERROR maps over RGBA, as tools/pooled_select_probe.py builds them: set128 (256 textures of 128²),
mixed (64 textures of 32² to 512²) and chain (the 13 levels of bench.py's config 1 image). Each is compressed at -fast, decoded
and mapped once. Then:
  select  the rule (d) select step, weights 1 / E_j then select_blocks_pooled (one pool, -inf threshold, K = 1 % of the set's
          blocks): weights from torch (a sum per map and a reciprocal, pooled_select_probe.py's path) against this call
          (ASTCENC_B200_WEIGHT_INVERSE_TOTAL); and the totals call alone. CUDA-event medians of --reps after a warm-up, with
          min and max; whether both paths select the same blocks.
  ladder  (mixed set) three rounds of select + refine_device_block_lists at -thorough with K = 2 % of the set's blocks per
          round: gated (total_block_maps(ONE) -> select_blocks_pooled with those weights and threshold 0) against ungated
          (select_blocks_pooled, no weight, -inf threshold), for two kinds of per-image PSNR target: 40 dB for every texture,
          and each texture's -fast PSNR + 1 dB. Reported: images at their target after the ladder, mean and worst PSNR (RGBA,
          from the final map totals), blocks listed, and the ladder's time (median of 5 after a warm-up, state restored
          between runs).
--bench-ab runs bench.py configs 0-3 for this tree and PARENT_TREE (a checkout of the parent commit with its library built)
alternately. The card's name and power limit are read in the same run and printed with the numbers."""
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

from pooled_select_probe import card, events, workloads  # noqa: E402


def setup(pkg, torch, fast, imgs, st):
    dev = torch.device("cuda", 0)
    s = st.cuda_stream
    dims = [(im.shape[1], im.shape[0]) for im in imgs]
    nb = [-(-w // 6) * -(-h // 6) for w, h in dims]
    d_img = [torch.from_numpy(im.reshape(-1)).to(dev) for im in imgs]
    pay = [torch.zeros(n * 16, dtype=torch.uint8, device=dev) for n in nb]
    dec = [torch.zeros(im.size, dtype=torch.uint8, device=dev) for im in imgs]
    mp = [torch.zeros(n, dtype=torch.float32, device=dev) for n in nb]
    met = torch.zeros(len(imgs) * 128, dtype=torch.uint8, device=dev)
    fast.compress_device_images([(d.data_ptr(), w, h, 1, p.data_ptr()) for d, (w, h), p in zip(d_img, dims, pay)], pkg.TYPE_U8, stream=s)
    fast.decompress_device_images([(p.data_ptr(), o.data_ptr(), w, h, 1) for p, o, (w, h) in zip(pay, dec, dims)], pkg.TYPE_U8, stream=s)
    fast.compute_block_metric_device_images([(d.data_ptr(), o.data_ptr(), pkg.TYPE_U8, pkg.TYPE_U8, w, h, 1, met.data_ptr() + 128 * k, m.data_ptr())
                                             for k, (d, o, (w, h), m) in enumerate(zip(d_img, dec, dims, mp))], pkg.BLOCK_SQUARED_ERROR, stream=s)
    st.synchronize()
    return dims, nb, d_img, pay, dec, mp


def select_step(pkg, torch, fast, name, imgs, st, reps):
    dev = torch.device("cuda", 0)
    s = st.cuda_stream
    dims, nb, d_img, pay, dec, mp = setup(pkg, torch, fast, imgs, st)
    N = len(imgs)
    K = max(1, int(sum(nb) * 0.01))
    w_torch = torch.zeros(N, dtype=torch.float32, device=dev)
    w_call = torch.zeros(N, dtype=torch.float32, device=dev)
    idx = [[torch.zeros(min(K, n), dtype=torch.int32, device=dev) for n in nb] for _ in range(2)]
    cnt = torch.zeros((2, N), dtype=torch.int32, device=dev)

    def pooled(w, k):
        fast.select_blocks_pooled([(N, -np.inf, K)], [(m.data_ptr(), n, w.data_ptr() + 4 * j, ix.data_ptr(), cnt[k].data_ptr() + 4 * j)
                                                      for j, (m, n, ix) in enumerate(zip(mp, nb, idx[k]))], stream=s)

    def torch_path():
        with torch.cuda.stream(st):
            torch.reciprocal(torch.stack([m.sum() for m in mp]), out=w_torch)
        pooled(w_torch, 0)

    def totals():
        fast.total_block_maps([(m.data_ptr(), n, -np.inf, 0, w_call.data_ptr() + 4 * j) for j, (m, n) in enumerate(zip(mp, nb))],
                              pkg.WEIGHT_INVERSE_TOTAL, stream=s)

    def call_path():
        totals()
        pooled(w_call, 1)

    row = {"workload": name, "images": N, "blocks": int(sum(nb)), "K": K}
    # alternate the two paths, several times, so that neither gets a quieter stretch of the card
    ta, tb, tt = [], [], []
    for _ in range(3):
        ta.append(events(torch, st, torch_path, reps)["median_ms"])
        tb.append(events(torch, st, call_path, reps)["median_ms"])
        tt.append(events(torch, st, totals, reps)["median_ms"])
    st.synchronize()
    row.update({"torch_select_ms": ta, "call_select_ms": tb, "totals_alone_ms": tt})
    same = all(np.array_equal(a.cpu().numpy()[:int(c0)], b.cpu().numpy()[:int(c1)])
               for a, b, c0, c1 in zip(idx[0], idx[1], cnt[0].cpu().numpy(), cnt[1].cpu().numpy()))
    wt, wc = w_torch.cpu().numpy(), w_call.cpu().numpy()
    row.update({"same_selection": bool(same), "max_weight_rel_diff": float(np.max(np.abs(wt - wc) / np.maximum(wc, 1e-30)))})
    print(json.dumps(row), flush=True)
    return row


def ladder(pkg, torch, fast, thorough, imgs, st, target_kind, rounds=3, frac=0.02, reps=5):
    dev = torch.device("cuda", 0)
    s = st.cuda_stream
    dims, nb, d_img, pay0, dec0, map0 = setup(pkg, torch, fast, imgs, st)
    N = len(imgs)
    K = max(1, int(sum(nb) * frac))
    samples = np.array([4.0 * w * h for w, h in dims])
    t0 = np.array([float(m.double().sum()) for m in map0])
    fast_psnr = np.where(t0 > 0, 10 * np.log10(samples / np.maximum(t0, 1e-300)), 999.0)
    target = np.full(N, 40.0) if target_kind == "40dB" else fast_psnr + 1.0
    limits = samples * 10 ** (-target / 10)
    pay, dec, mp = [p.clone() for p in pay0], [o.clone() for o in dec0], [m.clone() for m in map0]
    w = torch.zeros(N, dtype=torch.float32, device=dev)
    idx = [torch.zeros(min(K, n), dtype=torch.int32, device=dev) for n in nb]
    cnt = torch.zeros((rounds, N), dtype=torch.int32, device=dev)
    out = {}
    for gated in (True, False):
        def run():
            for r in range(rounds):
                if gated:
                    fast.total_block_maps([(m.data_ptr(), n, float(lim), 0, w.data_ptr() + 4 * j) for j, (m, n, lim) in enumerate(zip(mp, nb, limits))],
                                          pkg.WEIGHT_ONE, stream=s)
                fast.select_blocks_pooled([(N, 0.0 if gated else -np.inf, K)],
                                          [(m.data_ptr(), n, w.data_ptr() + 4 * j if gated else 0, ix.data_ptr(), cnt[r].data_ptr() + 4 * j)
                                           for j, (m, n, ix) in enumerate(zip(mp, nb, idx))], stream=s)
                thorough.refine_device_block_lists([(d.data_ptr(), x, y, 1, p.data_ptr(), o.data_ptr(), m.data_ptr(), ix.data_ptr(),
                                                     cnt[r].data_ptr() + 4 * j, ix.numel())
                                                    for j, (d, (x, y), p, o, m, ix) in enumerate(zip(d_img, dims, pay, dec, mp, idx))],
                                                   pkg.TYPE_U8, pkg.TYPE_U8, pkg.BLOCK_SQUARED_ERROR, stream=s)

        ts = []
        for rep in range(reps + 1):
            with torch.cuda.stream(st):
                for a, b in zip(pay + dec + mp, pay0 + dec0 + map0):
                    a.copy_(b)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            run()
            e1.record(st)
            e1.synchronize()
            if rep:
                ts.append(e0.elapsed_time(e1))
        tot = np.array([float(m.double().sum()) for m in mp])
        psnr = np.where(tot > 0, 10 * np.log10(samples / np.maximum(tot, 1e-300)), 999.0)
        out["gated" if gated else "ungated_b"] = {
            "at_target": int(np.sum(tot <= limits)), "mean_psnr": float(np.mean(psnr)), "worst_psnr": float(np.min(psnr)),
            "listed": int(cnt.cpu().numpy().sum()), "ladder_ms": float(np.median(ts)), "ladder_min_ms": float(min(ts)), "ladder_max_ms": float(max(ts))}
    row = {"target": target_kind, "images": N, "K_per_round": K, "rounds": rounds, "at_target_after_fast": int(np.sum(t0 <= limits)),
           "fast_mean_psnr": float(np.mean(fast_psnr)), "fast_worst_psnr": float(np.min(fast_psnr)), **out}
    print(json.dumps(row), flush=True)
    return row


def probe(args):
    import torch
    import __graft_entry__ as g
    assert torch.cuda.is_available(), "map_totals_probe.py needs a GPU"
    pkg = g.load_package()
    st = torch.cuda.Stream(device=torch.device("cuda", 0))
    res = {"card": card(), "select": [], "ladder": []}
    print("card: %s" % res["card"], flush=True)
    fast = pkg.Context(pkg.config_init(pkg.PRF_LDR, 6, 6, pkg.PRE_FAST))
    thorough = pkg.Context(pkg.config_init(pkg.PRF_LDR, 6, 6, pkg.PRE_THOROUGH))
    wl = workloads()
    for name in ("set128", "mixed", "chain"):
        res["select"].append(select_step(pkg, torch, fast, name, wl[name], st, args.reps))
        torch.cuda.empty_cache()
    for kind in ("40dB", "fast+1dB"):
        res["ladder"].append(ladder(pkg, torch, fast, thorough, wl["mixed"], st, kind))
    fast.close()
    thorough.close()
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


def bench_ab(args):
    print("card: %s" % card(), flush=True)
    for r in range(args.rounds):
        for name, root in ((("parent", os.path.abspath(args.bench_ab)), ("this", ROOT)) if r % 2 == 0 else (("this", ROOT), ("parent", os.path.abspath(args.bench_ab)))):
            for cfg in range(4):
                p = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--gpus", "1", "--steps", "10", "--warmup", "3", "--config", str(cfg), "--no-cpu-baseline"],
                                   capture_output=True, text=True, cwd=root)
                line = [l for l in p.stdout.splitlines() if l.startswith("{")]
                assert p.returncode == 0 and line, p.stderr[-2000:]
                print(json.dumps({"round": r, "build": name, "config": cfg, "result": json.loads(line[-1])}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out")
    ap.add_argument("--bench-ab", metavar="PARENT_TREE")
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    if args.bench_ab:
        bench_ab(args)
    else:
        probe(args)


if __name__ == "__main__":
    main()
