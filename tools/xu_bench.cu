// Micro-benchmark: sustained MUFU.EX2 rate per SM for the softmax instruction mix (build + run on the GPU box:
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o /tmp/xu_bench tools/xu_bench.cu && /tmp/xu_bench)
#include <cstdio>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

__device__ __forceinline__ float ex2f(float x) { float r; asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }

template <int MODE>
__global__ void k(float *out, long long *cyc, int iters, float a, float b)
{
    float x[32];
#pragma unroll
    for (int i = 0; i < 32; i++) x[i] = -1.0f - 0.01f * (threadIdx.x + i);
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    unsigned acc = 0;
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int i = 0; i < 32; i++) {
            float v = x[i];
            if (MODE >= 1) v = fmaf(v, a, b);
            v = ex2f(v);
            x[i] = v - 2.0f * (MODE == 0);      // keep the chain alive without extra work in modes >= 1 (fma does it)
            if (MODE == 0) x[i] = v;
        }
        if (MODE >= 2) {
#pragma unroll
            for (int i = 0; i < 32; i += 4) { s0 += x[i]; s1 += x[i + 1]; s2 += x[i + 2]; s3 += x[i + 3]; }
        }
        if (MODE >= 3) {
#pragma unroll
            for (int i = 0; i < 32; i += 2) {
                __nv_bfloat162 h = __floats2bfloat162_rn(x[i], x[i + 1]);
                acc ^= *reinterpret_cast<unsigned *>(&h);
            }
        }
    }
    const long long t1 = clock64();
    float s = s0 + s1 + s2 + s3;
#pragma unroll
    for (int i = 0; i < 32; i++) s += x[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s + (float)acc;
    if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

template <int MODE>
void run(int threads, int blocks_per_sm)
{
    const int sms = 148, iters = 200;
    float *out; long long *cyc;
    cudaMalloc(&out, sizeof(float) * sms * blocks_per_sm * threads);
    cudaMalloc(&cyc, sizeof(long long) * sms * blocks_per_sm);
    k<MODE><<<sms * blocks_per_sm, threads>>>(out, cyc, iters, -0.9f, -0.5f);
    k<MODE><<<sms * blocks_per_sm, threads>>>(out, cyc, iters, -0.9f, -0.5f);
    cudaDeviceSynchronize();
    long long h[148 * 8];
    cudaMemcpy(h, cyc, sizeof(long long) * sms * blocks_per_sm, cudaMemcpyDeviceToHost);
    double avg = 0;
    for (int i = 0; i < sms * blocks_per_sm; i++) avg += (double)h[i];
    avg /= sms * blocks_per_sm;
    const double mufu_per_sm = (double)iters * 32 * threads * blocks_per_sm;
    printf("mode %d  warps/SM %2d : %.2f MUFU/clk/SM\n", MODE, threads * blocks_per_sm / 32, mufu_per_sm / avg);
    cudaFree(out); cudaFree(cyc);
}

int main()
{
    for (int w : {4, 8, 12, 16, 24, 32}) {
        run<0>(w * 32 / 1 > 1024 ? 1024 : w * 32, w * 32 > 1024 ? 1 : 1);
    }
    for (int w : {4, 8, 12, 16, 24, 32}) run<1>(w * 32, 1);
    for (int w : {4, 8, 12, 16, 24, 32}) run<2>(w * 32, 1);
    for (int w : {4, 8, 12, 16, 24, 32}) run<3>(w * 32, 1);
    return 0;
}
