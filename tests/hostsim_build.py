"""Host builds of the device source: tests/hostsim/<name>.cpp compiled with g++, cached under tests/_build by mtime."""
import ctypes as C
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "astc-encoder_b200", "csrc")
# what a host build includes: the device source, the host simulation and the argument layouts of tests/devunit
_WATCHED = (CSRC, os.path.join(HERE, "hostsim"), os.path.join(HERE, "devunit"))


def host_sim(name, lanes32=False):
    """tests/hostsim/<name>.cpp compiled for the host (one simulated lane, or 32 lanes on 32 threads), linked with the library's
    table construction and configuration."""
    so = os.path.join(HERE, "_build", "lib%s%s.so" % (name, "32" if lanes32 else ""))
    newest = max(os.path.getmtime(os.path.join(d, f)) for d in _WATCHED for f in os.listdir(d))
    if not os.path.exists(so) or os.path.getmtime(so) < newest:
        os.makedirs(os.path.dirname(so), exist_ok=True)
        cmd = ["g++", "-std=c++14", "-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-shared"] + \
              (["-pthread", "-DASTC_HOSTSIM_LANES32=1"] if lanes32 else []) + \
              ["-x", "c++", os.path.join(HERE, "hostsim", name + ".cpp"), os.path.join(CSRC, "astc_host_tables.cpp"),
               os.path.join(CSRC, "astc_host_config.cpp"), "-o", so]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(so)
    assert lib.hostsim_lanes() == (32 if lanes32 else 1)
    return lib
