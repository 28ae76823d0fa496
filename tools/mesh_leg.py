"""Mesh export timing on the GPU: writes profiles/mesh_h100.md (or --out).

Stage times: CUDA events recorded by the host between the stages (the batched 50-view render at 512^2, prepare,
touch, integrate, marching cubes, clusters + compaction), so they include the host work of each stage (setup copies,
allocations, status waits); then the device-to-host copy and the OBJ write.  Kernel times: torch.profiler over one
fusion + post-processing of the same maps, per kernel.  The algorithmic bytes of prepare and integrate are divided
by their kernel times.  Also the unit / voxel / vertex / triangle counts and the numpy oracle's time for the same fusion.
Open3D cannot be timed: it is not installed on any machine available to this project.
python tools/mesh_leg.py [--out PATH] [--reps N]
"""
import argparse
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gaussiananything_b200 import mesh  # noqa: E402
from tests import mesh_scenes as ms  # noqa: E402


def gpu_name():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else torch.cuda.get_device_name(0)


def one_run(g, cams, setup):
    ev = {}

    def mark(name):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        ev[name] = e
    mark("start")
    _, out = mesh.render_orbit(g, cams, 512)
    mark("render")
    rgb, depth, alpha = out["image"][0], out["depth"][0, :, 0], out["alpha"][0, :, 0]
    mark("stack")
    m, st = mesh.fuse(rgb, depth, alpha, setup, stages=mark)
    post = mesh.post_process_mesh(m)
    mark("clusters_compaction")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    v, t, c = post.vertices, post.triangles, post.vertex_colors
    d2h = time.perf_counter() - t0
    with tempfile.TemporaryDirectory() as d:
        t0 = time.perf_counter()
        mesh.write_triangle_mesh(os.path.join(d, "m.obj"), post)
        obj = time.perf_counter() - t0
    names = ["render", "stack", "prepare", "touch", "integrate", "marching_cubes", "clusters_compaction"]
    ms_ = {}
    prev = "start"
    for n in names:
        ms_[n] = ev[prev].elapsed_time(ev[n])
        prev = n
    ms_["d2h_copy"] = d2h * 1e3
    ms_["obj_write"] = obj * 1e3
    counts = dict(units=st["n_units"], voxels=st["n_units"] * 4096, vertices=m.tensors()[0].shape[0],
                  triangles=m.tensors()[1].shape[0], kept_vertices=len(v), kept_triangles=len(t))
    return ms_, counts, (rgb, depth, alpha)


STAGE_OF = (("prepare_kernel", "prepare"), ("touch_kernel", "touch"), ("unit_flag_kernel", "touch"),
            ("unit_pool_kernel", "touch"), ("integrate_kernel", "integrate"), ("cube_case_kernel", "marching_cubes"),
            ("edge_flag_kernel", "marching_cubes"), ("emit_kernel", "marching_cubes"), ("cluster_", "clusters"),
            ("edge_insert_kernel", "clusters"), ("edge_union_kernel", "clusters"), ("filter_", "compaction"),
            ("copy_flags_kernel", "compaction"), ("scan_", "scans (all stages)"))


def kernel_times(rgb, depth, alpha, setup):
    """{kernel name: (stage, total ms, launches)} of one fusion + post-processing, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m, _ = mesh.fuse(rgb, depth, alpha, setup)
        mesh.post_process_mesh(m)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "self_device_time_total", None)
        if t is None:
            t = e.self_cuda_time_total
        for key, stage in STAGE_OF:
            if key in e.key and t > 0:
                hit = re.search(r"(\w+)\(", e.key)
                name = hit.group(1) if hit else e.key
                st, ms_, n = out.get(name, (stage, 0.0, 0))
                out[name] = (stage, ms_ + t / 1e3, n + e.count)
                break
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "mesh_h100.md"))
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "mesh_leg.py measures on the GPU"
    g = torch.tensor(ms.surface_surfels(73728, 0), device="cuda")
    cams = mesh.uni_mesh_path(10)
    setup = mesh.view_setup(cams, 512, 512)
    one_run(g, cams, setup)                                        # warm-up
    runs = [one_run(g, cams, setup) for _ in range(a.reps)]
    med = {k: float(np.median([r[0][k] for r in runs])) for k in runs[0][0]}
    counts = runs[0][1]
    rgb, depth, alpha = runs[0][2]
    V, H, W = depth.shape
    prep_bytes = V * H * W * (5 * 4 + 8)                           # rgb3 + depth + alpha in, one 8-byte texel out
    # integrate: per unit and view it touched, every voxel reads one texel (upper bound) and the state is written once
    integ_bytes = counts["voxels"] * 5 * 4 + counts["voxels"] * 8 * V
    kt = kernel_times(rgb, depth, alpha, setup)
    stage_kernel = {}
    for stage, ms_, _ in kt.values():
        stage_kernel[stage] = stage_kernel.get(stage, 0.0) + ms_
    from oracle import tsdf_oracle as to
    t0 = time.perf_counter()
    to.fuse(rgb.cpu().numpy(), depth.cpu().numpy(), alpha.cpu().numpy(), setup)
    oracle_s = time.perf_counter() - t0
    name = gpu_name()
    lines = ["# Mesh export on the GPU (TSDF fusion, marching cubes, floater filter)", "",
             "Measured by `tools/mesh_leg.py` on: %s (name, power limit from nvidia-smi)." % name, "",
             "Workload: 73 728 opaque surfels on a sphere and a torus (tests/mesh_scenes.surface_surfels), the 50",
             "uni_mesh_path(10) views rendered at 512^2 in one batched call, then fused. Median of %d runs after one" % a.reps,
             "warm-up.", "",
             "Stage times: CUDA events recorded by the host between stages, so each includes that stage's host work",
             "(setup copies, allocations, status waits).", "",
             "| stage | ms |", "|---|---|"]
    lines += ["| %s | %.3f |" % (k, v) for k, v in med.items()]
    lines += ["", "Kernel times: torch.profiler over one fusion + post-processing of the same maps.", "",
              "| kernel | stage | launches | ms |", "|---|---|---|---|"]
    lines += ["| %s | %s | %d | %.3f |" % (k, st, n, t) for k, (st, t, n) in sorted(kt.items(), key=lambda x: x[1][0])]
    lines += ["", "| stage | kernel ms |", "|---|---|"] + ["| %s | %.3f |" % kv for kv in stage_kernel.items()]
    lines += ["", "| count | value |", "|---|---|"] + ["| %s | %d |" % kv for kv in counts.items()]
    lines += ["", "Algorithmic bytes over kernel time: prepare_kernel moves %.1f MB (%.0f GB/s); integrate_kernel writes"
              " %.1f MB of voxel state and reads at most one 8-byte texel per voxel and view it integrates, %.1f MB in"
              " all (%.0f GB/s upper bound)." % (
                  prep_bytes / 1e6, prep_bytes / stage_kernel.get("prepare", float("nan")) / 1e6, counts["voxels"] * 20 / 1e6,
                  integ_bytes / 1e6, integ_bytes / stage_kernel.get("integrate", float("nan")) / 1e6),
              "", "numpy oracle (oracle/tsdf_oracle.py) for the same fusion on this host's CPU cores: %.1f s." % oracle_s,
              "Open3D, which the reference uses, could not be timed: it is not installed on any machine available to"
              " this project.", ""]
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        f.write("\n".join(lines))
    print("\n".join(lines))


if __name__ == "__main__":
    main()
