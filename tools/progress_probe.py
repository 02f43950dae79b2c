"""Cost of progress reporting and cancellation in astcenc_compress_image, in one run on one GPU.

  python tools/progress_probe.py [--parent-lib PATH] [--rounds N] [--out DIR]

1. No regression without a callback: bench.py --config 0..3 for the library of the parent commit (--parent-lib, built from
   that commit's tree) and for this tree's library, alternating, --rounds times each; value and e2e (Mtexels/s) per run.
2. Polling overhead: configs 1 and 2 through astcenc_compress_image (host pointers), with a no-op progress callback and without
   one, alternating; wall time per call.
3. Cancel latency: the time from astcenc_compress_cancel (called from the progress callback at the first value >= 10, 50 and
   90 %) to the return of astcenc_compress_image, on configs 1 and 2; median and maximum.
Prints one JSON line per measurement and a summary; the card's name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def bench(lib, config, steps, warmup):
    env = dict(os.environ)
    if lib:
        env["ASTCENC_B200_LIB"] = lib
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup),
                        "--config", str(config), "--no-cpu-baseline"], capture_output=True, text=True, env=env, cwd=ROOT)
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    if r.returncode != 0 or not lines:
        raise RuntimeError("bench.py --config %d failed:\n%s\n%s" % (config, r.stdout[-2000:], r.stderr[-2000:]))
    d = json.loads(lines[-1])
    return d["value"], d["e2e"]["value"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib", default=os.path.join(ROOT, "tools", "_build", "parent", "libastcenc_b200.so"))
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the results as JSON to DIR/progress_probe.json")
    args = ap.parse_args()
    import numpy as np
    import bench as B
    import __graft_entry__ as g
    pkg = g.load_package()
    res = {"card": card(), "bench": {}, "overhead": {}, "cancel": {}}
    print(json.dumps({"card": res["card"]}), flush=True)

    # 1. bench.py, parent and this build alternating
    libs = [("parent", args.parent_lib), ("this", None)] if os.path.exists(args.parent_lib) else [("this", None)]
    for c in (0, 1, 2, 3):
        runs = {name: [] for name, _ in libs}
        for _ in range(args.rounds):
            for name, lib in libs:
                v, e = bench(lib, c, 10 if c != 2 else 5, 3)
                runs[name].append((v, e))
                print(json.dumps({"bench": c, "build": name, "value": v, "e2e": e}), flush=True)
        res["bench"][c] = runs

    # 2. and 3. through astcenc_compress_image
    for c in (1, 2):
        cfg_d = B.CONFIGS[c]
        img = B.make_image(c, 1)
        cfg = pkg.config_init(cfg_d["profile"], cfg_d["block"], cfg_d["block"], cfg_d["quality"], B.FLAGS)
        plain = pkg.Context(cfg)
        noop = pkg.Context(cfg, progress=lambda v: None)
        out = np.empty(((img.shape[1] + cfg.block_x - 1) // cfg.block_x) * ((img.shape[0] + cfg.block_y - 1) // cfg.block_y) * 16, np.uint8)
        plain.compress_image(img, out=out)
        noop.compress_image(img, out=out)
        t = {"none": [], "noop": []}
        for _ in range(5):
            for name, ctx in (("none", plain), ("noop", noop)):
                t0 = time.perf_counter()
                ctx.compress_image(img, out=out)
                t[name].append((time.perf_counter() - t0) * 1e3)
        res["overhead"][c] = {k: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v)} for k, v in t.items()}
        print(json.dumps({"overhead": c, **res["overhead"][c]}), flush=True)
        plain.close()
        noop.close()
        res["cancel"][c] = {}
        for at in (10.0, 50.0, 90.0):
            lat = []
            state = {}

            def cb(v):
                if "t" not in state and v >= at:
                    state["t"] = time.perf_counter()
                    state["at"] = v
                    ctx.cancel()

            ctx = pkg.Context(cfg, progress=cb)
            ctx.compress_image(img, out=out)      # (warm-up, cancelled too)
            for _ in range(5):
                state.clear()
                ctx.compress_image(img, out=out)
                lat.append((time.perf_counter() - state["t"]) * 1e3)
            ctx.close()
            res["cancel"][c][at] = {"median_ms": statistics.median(lat), "max_ms": max(lat), "runs": lat}
            print(json.dumps({"cancel": c, "at": at, **res["cancel"][c][at]}), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "progress_probe.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
