"""Time the surface point cloud kernels on the GPU:

    python tools/pcd_leg.py [--json out.json]

Cases: fusion and compaction of the 16-view test chunk (ga_chunk_surface_points); FPS 254 899 -> 4096 (that chunk's
fused cloud), 4 194 304 -> 4096 (synthetic), 73 728 -> 4096 (a surfel cloud with 30 % of the surfels below the
opacity cut, passed with lengths); and both FPS paths at the encoder's sizes (B = 1 and 2, N = 4096, K = 768): the
one-CTA ga_fps and the cooperative kernel (ga_fps_ex with lengths).
Yardsticks, on the same inputs: the oracle's loop in torch (four launches per round) captured in one CUDA graph, and
the single-CTA design pytorch3d uses (one 1024-thread block per cloud streaming its points and distances from global
memory each round), compiled here from the source below into a temporary directory.  Every FPS result is checked
against the library's before it is timed.
Device events around >= 1 s of back-to-back calls after a warm-up.  The card's name, power limit and maximum SM clock
are read in the same run.  Needs a CUDA device.
"""
import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SECONDS = 1.0
CHUNK = os.path.join(ROOT, "tests", "golden", "gbuffer_chunk")

STREAM_FPS = r"""
#include <cuda_runtime.h>
#include <stdint.h>
__global__ void __launch_bounds__(1024) fps_stream(const float *pcd, int N, int K, float *md, int32_t *idx)
{
    __shared__ float wd[32];
    __shared__ int wi[32];
    __shared__ int sel;
    const int b = blockIdx.x, t = threadIdx.x;
    const float *P = pcd + (size_t)b * N * 3;
    float *M = md + (size_t)b * N;
    for (int p = t; p < N; p += 1024) M[p] = INFINITY;
    int cur = 0;
    for (int k = 0; k < K; k++) {
        if (t == 0) idx[(size_t)b * K + k] = cur;
        if (k + 1 == K) break;
        const float sx = P[3 * cur], sy = P[3 * cur + 1], sz = P[3 * cur + 2];
        float best = -1.f;
        int bi = 0x7fffffff;
        for (int p = t; p < N; p += 1024) {
            const float dx = __fsub_rn(P[3 * p], sx), dy = __fsub_rn(P[3 * p + 1], sy), dz = __fsub_rn(P[3 * p + 2], sz);
            const float d = fminf(M[p], __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
            M[p] = d;
            if (d > best) { best = d; bi = p; }
        }
        for (int o = 16; o; o >>= 1) {
            const float d2 = __shfl_xor_sync(0xffffffffu, best, o);
            const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
            if (d2 > best || (d2 == best && i2 < bi)) { best = d2; bi = i2; }
        }
        if ((t & 31) == 0) { wd[t >> 5] = best; wi[t >> 5] = bi; }
        __syncthreads();
        if (t < 32) {
            best = wd[t]; bi = wi[t];
            for (int o = 16; o; o >>= 1) {
                const float d2 = __shfl_xor_sync(0xffffffffu, best, o);
                const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
                if (d2 > best || (d2 == best && i2 < bi)) { best = d2; bi = i2; }
            }
            if (t == 0) sel = bi;
        }
        __syncthreads();
        cur = sel;
    }
}
extern "C" int fps_stream_launch(const float *pcd, int B, int N, int K, float *md, int32_t *idx, void *stream)
{
    fps_stream<<<B, 1024, 0, (cudaStream_t)stream>>>(pcd, N, K, md, idx);
    return (int)cudaGetLastError();
}
"""


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", "0"], capture_output=True, text=True, timeout=30)
        watts, mhz = (float(v) for v in r.stdout.strip().splitlines()[0].split(","))
    except Exception:
        watts = mhz = None
    return name, watts, mhz


def time_ms(fn, seconds=SECONDS):
    for _ in range(2):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    reps = max(3, math.ceil(seconds / max(e0.elapsed_time(e1) * 1e-3, 1e-6)))
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def stream_fps_lib(tmp):
    src, so = os.path.join(tmp, "fps_stream.cu"), os.path.join(tmp, "fps_stream.so")
    with open(src, "w") as f:
        f.write(STREAM_FPS)
    nvcc = os.environ.get("NVCC") or "/usr/local/cuda/bin/nvcc"
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-Xcompiler", "-fPIC", "-shared",
                    "-cudart", "shared", "-o", so, src], check=True, capture_output=True)
    L = C.CDLL(so)
    L.fps_stream_launch.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def torch_graph_fps(pts, K):
    """The oracle's loop (vae_encoder_oracle.fps) on the GPU for one cloud, captured once; returns (replay, idx)."""
    from gaussiananything_b200._launch import no_cyclic_gc
    N = pts.shape[0]
    md = torch.empty(N, device=pts.device)
    idx = torch.zeros(K, dtype=torch.int64, device=pts.device)

    def body():
        md.fill_(float("inf"))
        cur = idx[0:1]
        for k in range(1, K):
            d = pts - pts[cur]
            torch.minimum(md, ((d[:, 0] * d[:, 0]) + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2], out=md)
            torch.argmax(md, 0, keepdim=True, out=idx[k:k + 1])
            cur = idx[k:k + 1]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        body()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with no_cyclic_gc(), torch.cuda.graph(g):
        body()
    return g.replay, idx


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    ap.add_argument("--skip-torch-4m", action="store_true", help="leave out the torch loop on 4M points")
    args = ap.parse_args()
    from gaussiananything_b200 import _lib, gbuffer, pcd
    from gaussiananything_b200._launch import ptr as _p, stream as _stream
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    name, watts, mhz = card()
    res = {"card": name, "power_limit_w": watts, "max_sm_clock_mhz": mhz, "seconds_per_case": SECONDS, "cases": {}}
    L = _lib.lib()
    st = _stream(dev)
    tmp = tempfile.mkdtemp(prefix="pcd_leg_")
    SL = stream_fps_lib(tmp)

    # ---- fusion
    chunk = gbuffer.to_device(gbuffer.read_chunk(CHUNK), dev)
    fused = pcd.chunk_surface_points(chunk, device=dev)
    ms = time_ms(lambda: pcd.chunk_surface_points(chunk, device=dev))
    n, h, w = chunk["depth"].shape
    V = n
    vi = torch.arange(V, dtype=torch.int32, device=dev)
    out = torch.empty(V * h * w, 3, device=dev)
    cnt = torch.empty(1, dtype=torch.int32, device=dev)
    scr = torch.empty(L.ga_chunk_surface_points_scratch_bytes(V, h, w), dtype=torch.uint8, device=dev)
    kern = lambda: L.ga_chunk_surface_points(_p(chunk["alpha"]), _p(chunk["depth"]), _p(chunk["c"]), n, h, w, _p(vi), V,
                                             255, 1.05, _p(out), _p(cnt), _p(scr), scr.numel(), st)
    ms_k = time_ms(kern)
    byts = V * h * w * (4 + 1) + int(fused.shape[0]) * 12
    res["cases"]["fusion_16x512"] = {"points": int(fused.shape[0]), "python_call_ms": round(ms, 4),
                                     "kernels_ms": round(ms_k, 4), "min_bytes": byts,
                                     "hbm_share": round(byts / 3.35e12 / (ms_k * 1e-3), 3)}

    # ---- FPS cases
    g = torch.Generator(device=dev).manual_seed(0)
    big = torch.rand(1, 4194304, 3, device=dev, generator=g) - 0.5
    surf = torch.rand(1, 73728, 3, device=dev, generator=g) - 0.5
    surf_len = 51610                                                  # 70 % of the surfels kept
    cases = [("fps_254899_to_4096", fused[None].contiguous(), None, 4096),
             ("fps_4194304_to_4096", big, None, 4096),
             ("fps_surfels_73728_to_4096", surf, surf_len, 4096)]
    for key, pts, length, K in cases:
        B, N, _ = pts.shape
        ln = torch.full((B,), N if length is None else length, dtype=torch.int32, device=dev)
        start = torch.zeros(B, dtype=torch.int32, device=dev)
        idx = torch.empty(B, K, dtype=torch.int32, device=dev)
        xyz = torch.empty(B, K, 3, device=dev)
        ws = torch.empty(L.ga_fps_ex_workspace_bytes(B, N, K), dtype=torch.uint8, device=dev)
        call = lambda: _lib.check(L.ga_fps_ex(_p(pts), _p(ln), B, N, K, _p(start), _p(idx), _p(xyz), _p(ws),
                                              ws.numel(), st), "ga_fps_ex")
        ms = time_ms(call)
        r = {"N": N if length is None else length, "K": K, "fps_ex_ms": round(ms, 3),
             "us_per_round": round(ms * 1e3 / (K - 1), 3)}
        n_eff = r["N"]
        cloud = pts[0, :n_eff].contiguous()
        md = torch.empty(n_eff, device=dev)
        sidx = torch.empty(1, K, dtype=torch.int32, device=dev)
        scall = lambda: SL.fps_stream_launch(_p(cloud), 1, n_eff, K, _p(md), _p(sidx), st)
        scall()
        torch.cuda.synchronize()
        r["one_cta_stream_matches"] = bool(torch.equal(sidx, idx))
        r["one_cta_stream_ms"] = round(time_ms(scall), 3)
        if not (key.startswith("fps_4194304") and args.skip_torch_4m):
            replay, tidx = torch_graph_fps(cloud, K)
            replay()
            torch.cuda.synchronize()
            r["torch_graph_matches"] = bool(torch.equal(tidx.int(), idx[0]))
            r["torch_graph_ms"] = round(time_ms(replay), 3)
            del replay
        res["cases"][key] = r
        print(key, r, flush=True)

    # ---- encoder sizes: both paths
    for B in (1, 2):
        N, K = 4096, 768
        pts = torch.rand(B, N, 3, device=dev, generator=g) - 0.5
        start = torch.zeros(B, dtype=torch.int32, device=dev)
        ln = torch.full((B,), N, dtype=torch.int32, device=dev)
        i1, i2 = (torch.empty(B, K, dtype=torch.int32, device=dev) for _ in range(2))
        x1, x2 = (torch.empty(B, K, 3, device=dev) for _ in range(2))
        ws = torch.empty(L.ga_fps_ex_workspace_bytes(B, N, K), dtype=torch.uint8, device=dev)
        old = lambda: L.ga_fps(_p(pts), B, N, K, _p(start), _p(i1), _p(x1), st)
        new = lambda: L.ga_fps_ex(_p(pts), _p(ln), B, N, K, _p(start), _p(i2), _p(x2), _p(ws), ws.numel(), st)
        old(), new()
        torch.cuda.synchronize()
        same = bool(torch.equal(i1, i2))
        t_old, t_new = [], []
        for _ in range(3):                                            # alternate the two
            t_old.append(time_ms(old, SECONDS / 3))
            t_new.append(time_ms(new, SECONDS / 3))
        res["cases"]["encoder_B%d_4096_to_768" % B] = {
            "same_indices": same, "one_cta_ga_fps_ms": [round(t, 4) for t in t_old],
            "cooperative_ms": [round(t, 4) for t in t_new]}
        print("encoder B=%d" % B, res["cases"]["encoder_B%d_4096_to_768" % B], flush=True)

    line = json.dumps(res)
    print(line)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
