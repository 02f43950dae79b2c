"""dev tool (GPU box): how the set-up stage of one config 1 pass (4096^2 RGBA8, 6x6 -medium, device-resident) splits over its
launches. One warm pass, then one pass under torch.profiler (CUDA activities only, in a run of its own); the trace is read back
and every astc_wave_setup_kernel launch is printed with its wave (= refinement launches before it), threads per CTA and duration.
   python tools/setup_split.py [--lib path.so] [--dim 4096]"""
import json, os, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
args = sys.argv[1:]
dim = 4096
if "--dim" in args:
    i = args.index("--dim"); dim = int(args[i + 1]); del args[i:i + 2]
if "--lib" in args:
    i = args.index("--lib"); os.environ["ASTCENC_B200_LIB"] = os.path.abspath(args[i + 1]); del args[i:i + 2]
import numpy as np, torch
from torch.profiler import ProfilerActivity, profile
import astc_images as I
import __graft_entry__ as g
pkg = g.load_package()
pkg.LIB_PATH = os.environ.get("ASTCENC_B200_LIB", pkg.LIB_PATH)

dev = torch.device("cuda", 0)
img = np.ascontiguousarray(I.photo_like(dim, dim, seed=2024))
d_img = torch.from_numpy(img).to(dev)
st = torch.cuda.Stream(device=dev)
ctx = pkg.Context(pkg.config_init(pkg.PRF_LDR, 6, 6, pkg.PRE_MEDIUM, 32))
nbx, nby = ctx.blocks(dim, dim)
d_out = torch.zeros(nbx * nby * 16, dtype=torch.uint8, device=dev)


def one_pass():
    with torch.cuda.stream(st):
        ctx.compress_device(d_img.data_ptr(), 0, dim, dim, d_out.data_ptr(), stream=st.cuda_stream)
    torch.cuda.synchronize()


one_pass()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    one_pass()
ctx.close()
with tempfile.TemporaryDirectory() as td:
    path = os.path.join(td, "trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        trace = json.load(f)
kernels = sorted((e for e in trace["traceEvents"] if e.get("cat") == "kernel"), key=lambda e: e["ts"])
print("card: %s" % torch.cuda.get_device_name(0))
wave = 0
seen_refine = False
rows = []
for e in kernels:
    name = e["name"]
    if "astc_wave_refine_kernel" in name:
        seen_refine = True
    elif "astc_wave_setup_kernel" in name:
        if seen_refine:
            wave += 1
            seen_refine = False
        block = e.get("args", {}).get("block", [0])
        rows.append((wave, name.split("(")[0], block[0], e["dur"] / 1e3))
total = sum(r[3] for r in rows)
print("%-5s %-42s %8s %10s" % ("wave", "kernel", "threads", "ms"))
for r in rows:
    print("%-5d %-42s %8d %10.3f" % r)
w0 = sum(r[3] for r in rows if r[0] == 0)
print("set-up: %.3f ms in %d launches; wave 0 %.3f ms (%.1f %%), later waves %.3f ms" % (total, len(rows), w0, 100.0 * w0 / max(total, 1e-9), total - w0))
