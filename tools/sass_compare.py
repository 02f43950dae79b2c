#!/usr/bin/env python
"""Compare the SASS of chosen kernels between two builds of libastcenc_b200.so (cuobjdump -sass, no GPU needed).

  python tools/sass_compare.py OLD.so NEW.so [kernel-name-substring ...]

Default kernels: the four stage kernels of the wave pipeline (every instantiation) and the single-kernel driver. Addresses,
comments and the /*offset*/ column are dropped; the instruction text itself must match line for line. Prints one line per
kernel (instruction count, identical or not) and exits 1 when any differs."""
import re
import subprocess
import sys

DEFAULT = ["astc_wave_setup_kernel", "astc_wave_refine_kernel", "astc_wave_prepare_kernel", "astc_wave_emit_kernel", "astc_compress_kernel"]


def kernels(so):
    out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs[name] = []
            continue
        if name is None:
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line)
        if m:
            funcs[name].append(m.group(1))
    return funcs


def main():
    old, new = kernels(sys.argv[1]), kernels(sys.argv[2])
    wanted = sys.argv[3:] or DEFAULT
    bad = 0
    for name in sorted(old):
        if not any(w in name for w in wanted):
            continue
        a, b = old[name], new.get(name)
        same = b is not None and a == b
        bad += not same
        print("%-80s %6d instructions  %s" % (name, len(a), "identical" if same else "DIFFERS (%s)" % ("missing" if b is None else "%d instructions" % len(b))))
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
