"""Build libspo.so (sm_90a, H100) in-tree with nvcc.  Cross-compiles without a GPU.

    python safe-policy-optimization_b200/build.py [--force]

Output: safe-policy-optimization_b200/safepo/lib/libspo.so (git-ignored build product)."""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OUT_DIR = os.path.join(HERE, "safepo", "lib")
OUT = os.path.join(OUT_DIR, "libspo.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "include"), "-I", CSRC]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def up_to_date():
    if not os.path.exists(OUT):
        return False
    t = os.path.getmtime(OUT)
    deps = sources() + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")] + \
        [os.path.join(ROOT, "include", "spo.h"), os.path.abspath(__file__)]
    return all(os.path.getmtime(d) <= t for d in deps)


def build(force=False, verbose=False, timers=False):
    """timers=True: a second library tools/libspo_timers.so with -DSPO_PHASE_TIMERS (clock64 phase marks in the
    update kernel, read back with spo_debug_phase_cycles; tools/phase_timers.py)."""
    out = os.path.join(ROOT, "tools", "libspo_timers.so") if timers else OUT
    if not timers and not force and up_to_date():
        return OUT
    os.makedirs(OUT_DIR, exist_ok=True)
    objdir = os.path.join(OUT_DIR, "obj_timers" if timers else "obj")
    os.makedirs(objdir, exist_ok=True)

    def cc(src):
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        cmd = [NVCC] + FLAGS + (["-DSPO_PHASE_TIMERS"] if timers else []) + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=8) as ex:
        objs = list(ex.map(cc, sources()))
    cmd = [NVCC, "-shared"] + ARCH + ["-o", out] + objs
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv, timers="--timers" in sys.argv))
