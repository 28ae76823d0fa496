"""Builds baseline/libga_standin.so (the GPU comparison baseline of bench.py; not the product)."""
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "raster_standin.cu")
OUT = os.path.join(HERE, "libga_standin.so")


def build(force=False):
    if not force and os.path.exists(OUT) and os.path.getmtime(OUT) >= os.path.getmtime(SRC):
        return OUT
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
           "-shared", "-cudart", "shared", "-o", OUT, SRC]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("stand-in build failed:\n" + r.stdout + r.stderr)
    return OUT


if __name__ == "__main__":
    print(build(force=True))
