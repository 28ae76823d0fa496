"""Per-kernel device time of the C2 raster step (100k surfels, 512^2, 6 views, forward + backward) under
torch.profiler with CUDA activities.  Run it on its own: tracing slows the host, so take end-to-end numbers from
bench.py.  Prints one JSON line {kernel name: mean us per step, launches per step}; the library is the one
GA_B200_LIB selects (gaussiananything_b200/_lib.py).
    python tools/profile_raster_kernels.py [tag] [steps]"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from gaussiananything_b200 import _lib, raster  # noqa: E402
from tests.helpers import cameras, scene  # noqa: E402


def main():
    tag = sys.argv[1] if len(sys.argv) > 1 else "default"
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    P, H, W, V = 100000, 512, 512, 6
    dev = torch.device("cuda:0")
    g13 = torch.tensor(scene(P, 40), device=dev)[None].contiguous()
    vs, ps, _, _ = cameras(V)
    vm = torch.tensor(vs, device=dev)[None].contiguous()
    pm = torch.tensor(ps, device=dev)[None].contiguous()
    bg = torch.ones(3, device=dev)
    torch.manual_seed(0)
    dc = torch.randn(1, V, 3, H, W, device=dev)
    da = torch.randn(1, V, 7, H, W, device=dev)
    c, a, r, st = raster.forward_raw(g13, vm, pm, bg, H, W, list_k=raster.LIST_K)
    for _ in range(3):
        c, a, r, st = raster.forward_raw(g13, vm, pm, bg, H, W, max_instances=st["max_instances"], list_k=raster.LIST_K)
        raster.backward_raw(st, dc, da)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            c, a, r, st = raster.forward_raw(g13, vm, pm, bg, H, W, max_instances=st["max_instances"],
                                             list_k=raster.LIST_K)
            raster.backward_raw(st, dc, da)
        torch.cuda.synchronize()
    kernels = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0:
            kernels[ev.key] = {"us_per_step": round(t / steps, 1), "calls_per_step": ev.count / steps}
    kernels = dict(sorted(kernels.items(), key=lambda kv: -kv[1]["us_per_step"]))
    print(json.dumps({"tag": tag, "lib": os.path.basename(_lib.LIB_PATH), "steps": steps, "kernels": kernels}))


if __name__ == "__main__":
    main()
