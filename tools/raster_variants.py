"""Times the five raster stages of the C2 workload (100k surfels, 512^2, 6 views, fwd+bwd) for the library /
tuning build selected by the environment (GA_B200_LIB, LISTK, STEPS) and prints one JSON line with the stage
times and checksums of the outputs, so that several builds can be compared in one run:
    GA_B200_LIB=gaussiananything_b200/libga_b200_parent.so python tools/raster_variants.py parent"""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from gaussiananything_b200 import _lib, raster  # noqa: E402
from tests.helpers import cameras, scene  # noqa: E402


def main():
    tag = sys.argv[1] if len(sys.argv) > 1 else "default"
    steps = int(os.environ.get("STEPS", "30"))
    P, H, W, V = 100000, 512, 512, 6
    dev = torch.device("cuda:0")
    lib = _lib.lib()
    g = scene(P, 40)
    vs, ps, _, _ = cameras(V)
    g13 = torch.tensor(g, device=dev)[None].contiguous()
    vm = torch.tensor(vs, device=dev)[None].contiguous()
    pm = torch.tensor(ps, device=dev)[None].contiguous()
    bg = torch.ones(3, device=dev)
    torch.manual_seed(0)
    dc = torch.randn(1, V, 3, H, W, device=dev)
    da = torch.randn(1, V, 7, H, W, device=dev)
    flush = torch.empty(256 << 20, device=dev, dtype=torch.uint8)
    LK = int(os.environ.get("LISTK", str(raster.LIST_K)))
    c, a, r, st = raster.forward_raw(g13, vm, pm, bg, H, W, list_k=LK)
    grad = raster.backward_raw(st, dc, da)
    for _ in range(3):
        c, a, r, st = raster.forward_raw(g13, vm, pm, bg, H, W, max_instances=st["max_instances"], list_k=LK)
        grad = raster.backward_raw(st, dc, da)
    torch.cuda.synchronize()
    lib.ga_profile_enable(1)
    acc = np.zeros(5)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    tot = 0.0
    for _ in range(steps):
        flush.zero_()
        e0.record()
        c, a, r, st = raster.forward_raw(g13, vm, pm, bg, H, W, max_instances=st["max_instances"], list_k=LK)
        grad = raster.backward_raw(st, dc, da)
        e1.record()
        e1.synchronize()
        tot += e0.elapsed_time(e1)
        buf = (C.c_float * 8)()
        n = lib.ga_profile_read(buf, 8)
        acc += np.array(buf[:5])
    lib.ga_profile_enable(0)
    acc /= steps
    wsv = raster.workspace_views(st["ws"], st["L"], 1, P, V, H, W, st["max_instances"])
    out = {"tag": tag, "lib": os.path.basename(_lib.LIB_PATH), "env": {k: v for k, v in os.environ.items() if k.startswith("GA_B200_")},
           "stage_us": dict(zip(["preprocess", "binning", "render_fwd", "render_bwd", "preprocess_bwd"], [round(1e3 * x, 1) for x in acc])),
           "sum_us": round(1e3 * acc.sum(), 1), "step_ms_incl_host": tot / steps,
           "check": {"color": float(c.double().sum()), "allmap": float(a.double().abs().sum()),
                     "n_contrib": int(wsv["n_contrib"].long().sum()), "list_k": LK,
                     "flagged_tiles": (int(st["ws"][st["L"].tile_flag:st["L"].tile_flag + 4 * 6 * 1024].view(torch.int32).sum()) if LK else None), "grad_abs": float(grad.double().abs().sum()),
                     "grad_sum": float(grad.double().sum())}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
