#!/usr/bin/env python
"""Packed against unpacked block lists in a -fast -> -thorough keep-the-better round over a whole texture set (needs a GPU).

  python tools/packed_lists_probe.py [--reps 7] [--out FILE.json]

Workloads: those of tools/pooled_select_probe.py (set128: 256 textures of 128^2; chain: the config 1 mip chain; mixed: 64 mixed
textures), LDR, 6x6 blocks, SQUARED_ERROR maps over RGBA. Each is compressed at -fast, decoded and mapped once. A round is then
one selection and one refine call at -thorough, at budgets K of 1 % and 10 % of the set's blocks, three ways:
  a  select_blocks per image with capacity max(1, int(n_j * f)) and refine_device_block_lists (K is the sum of the capacities)
  u  select_blocks_pooled (one pool of capacity K) and refine_device_block_lists with capacities min(K, n_j)
  p  select_blocks_pooled the same way and refine_device_block_lists_packed with budget K
Reported per path: slots staged by the refine call, the round's time (select + refine, CUDA events on one stream, median of
--reps after a warm-up, with min and max; the three paths alternate rep by rep, each from the same -fast state). u and p are
checked to leave identical payloads, decodes and maps. The card's name and power limit are read in the same run."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from pooled_select_probe import card, workloads  # noqa: E402

FRACS = (0.01, 0.10)
PATHS = ("a", "u", "p")


def probe(args):
    import torch
    import __graft_entry__ as g
    assert torch.cuda.is_available(), "packed_lists_probe.py needs a GPU"
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
        out = {"images": len(imgs), "blocks": int(sum(nb)), "rounds": []}
        state = {k: ([p.clone() for p in pay0], [o.clone() for o in dec0], [m.clone() for m in map0]) for k in PATHS}
        ovf = torch.zeros(1, dtype=torch.int32, device=dev)
        for f in FRACS:
            caps_a = [max(1, int(n * f)) for n in nb]
            K = sum(caps_a)
            caps_p = [min(K, n) for n in nb]
            idx = [torch.zeros(max(a, p), dtype=torch.int32, device=dev) for a, p in zip(caps_a, caps_p)]
            cnt = torch.zeros(len(imgs), dtype=torch.int32, device=dev)
            slots = {"a": sum(caps_a), "u": sum(caps_p), "p": min(K, sum(caps_p))}

            def round_(path):
                pay, dec, mp = state[path]
                if path == "a":
                    fast.select_blocks([(m.data_ptr(), n, -np.inf, c, ix.data_ptr(), cnt.data_ptr() + 4 * k)
                                        for k, (m, n, c, ix) in enumerate(zip(mp, nb, caps_a, idx))], stream=s)
                else:
                    fast.select_blocks_pooled([(len(imgs), -np.inf, K)], [(m.data_ptr(), n, 0, ix.data_ptr(), cnt.data_ptr() + 4 * k)
                                                                         for k, (m, n, ix) in enumerate(zip(mp, nb, idx))], stream=s)
                caps = caps_a if path == "a" else caps_p
                table = [(d.data_ptr(), w, h, 1, p.data_ptr(), o.data_ptr(), m.data_ptr(), ix.data_ptr(), cnt.data_ptr() + 4 * k, c)
                         for k, (d, (w, h), p, o, m, ix, c) in enumerate(zip(d_img, dims, pay, dec, mp, idx, caps))]
                if path == "p":
                    thorough.refine_device_block_lists_packed(table, K, pkg.TYPE_U8, pkg.TYPE_U8, pkg.BLOCK_SQUARED_ERROR, overflow=ovf.data_ptr(), stream=s)
                else:
                    thorough.refine_device_block_lists(table, pkg.TYPE_U8, pkg.TYPE_U8, pkg.BLOCK_SQUARED_ERROR, stream=s)

            def restore(path):
                with torch.cuda.stream(st):
                    for a, b in zip(sum(state[path], []), pay0 + dec0 + map0):
                        a.copy_(b)

            ts = {k: [] for k in PATHS}
            for r in range(args.reps + 1):
                for path in PATHS:
                    restore(path)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(st)
                    round_(path)
                    e1.record(st)
                    e1.synchronize()
                    if r:      # (the first is the warm-up)
                        ts[path].append(e0.elapsed_time(e1))
            same = all(torch.equal(a, b) for a, b in zip(sum(state["u"], []), sum(state["p"], [])))
            row = {"frac": f, "K": K, "identical_u_p": same, "overflow": int(ovf.item())}
            for k in PATHS:
                row[k] = {"slots": slots[k], "round_ms": float(np.median(ts[k])), "min_ms": float(min(ts[k])), "max_ms": float(max(ts[k]))}
            out["rounds"].append(row)
            print(json.dumps({name: row}), flush=True)
            assert same, "packed and unpacked rounds left different bytes"
        res["workloads"][name] = out
        del pay0, dec0, map0, d_img, state
        torch.cuda.empty_cache()
    fast.close()
    thorough.close()
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out")
    probe(ap.parse_args())


if __name__ == "__main__":
    main()
