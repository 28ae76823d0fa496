"""In-tree build of libga_b200.so (sm_90a only) with nvcc.

`python -m gaussiananything_b200.build` or `build()`; the .so is written next
to this file so it travels to the GPU box with the repo snapshot.
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libga_b200.so")
OBJ = os.path.join(HERE, "csrc", "_obj")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]

# per-file extra flags.  raster_preprocess.cu: no FMA contraction, so tile
# rectangles / radii / depth keys are bit-exact with the C oracle.
EXTRA = {
    "raster_preprocess.cu": ["--fmad=false"],
    # TSDF weights / tsdf / colours and marching-cubes vertices: bit-exact with oracle/tsdf_oracle.py
    "mesh_tsdf.cu": ["--fmad=false"],
    "mesh_extract.cu": ["--fmad=false"],
}


def _nvcc():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def build(force: bool = False, verbose: bool = False, variant: str = "", extra_flags=()) -> str:
    """variant != "": a tuning build libga_b200_<variant>.so with `extra_flags` (e.g. -DGA_TILE_REPLICAS=4) in its own object
    directory; load it with GA_B200_LIB=<path> (gaussiananything_b200/_lib.py).  The default build is the product."""
    nvcc = _nvcc()
    OUT = os.path.join(HERE, "libga_b200%s.so" % (("_" + variant) if variant else ""))
    OBJ = os.path.join(HERE, "csrc", "_obj" + (("_" + variant) if variant else ""))
    os.makedirs(OBJ, exist_ok=True)
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hdrs.append(os.path.join(HERE, "..", "include", "ga_b200.h"))
    hdr_m = max(os.path.getmtime(h) for h in hdrs)
    objs, rebuilt = [], False
    for f in sources():
        src = os.path.join(CSRC, f)
        obj = os.path.join(OBJ, f[:-3] + ".o")
        objs.append(obj)
        if (not force and os.path.exists(obj)
                and os.path.getmtime(obj) >= max(os.path.getmtime(src), hdr_m)):
            continue
        # GA_B200_NVCC_EXTRA="-DFOO=1 ...": extra flags for every file (tuning experiments; use with --force)
        cmd = [nvcc] + ARCH + COMMON + EXTRA.get(f, []) + os.environ.get("GA_B200_NVCC_EXTRA", "").split() + list(extra_flags) + ["-c", src, "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (f, r.stdout, r.stderr))
        if verbose:
            print(r.stderr)
        rebuilt = True
    if rebuilt or force or not os.path.exists(OUT):
        cmd = [nvcc] + ARCH + ["-shared", "-cudart", "shared", "-o", OUT] + objs
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return OUT


if __name__ == "__main__":
    # python -m gaussiananything_b200.build [--force] [-v] [--variant NAME -DFLAG=1 ...]
    var, flags = "", []
    if "--variant" in sys.argv:
        i = sys.argv.index("--variant")
        var = sys.argv[i + 1]
        flags = [a for a in sys.argv[i + 2:] if a.startswith("-D")]
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv, variant=var, extra_flags=flags))
