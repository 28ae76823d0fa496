// Per-device one-time initialisation flags.  cudaFuncSetAttribute(MaxDynamicSharedMemorySize) and the SM count
// are per device / context, not per process: a process that drives several GPUs (dit.py rebuilds its engine when
// x.device changes) must repeat them on every device it launches on.
#pragma once
#include <cuda_runtime.h>

struct GaPerDevice {
    bool done[64] = {};
    int value[64] = {};
};

// true exactly once per (flag, current device)
static inline bool ga_first_use_on_device(GaPerDevice &f, int *dev_out = nullptr)
{
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev_out) *dev_out = dev;
    if (dev < 0 || dev >= 64) return true;      // unknown ordinal: always (re)initialise
    if (f.done[dev]) return false;
    f.done[dev] = true;
    return true;
}

static inline int ga_sm_count()
{
    static GaPerDevice f;
    int dev = 0;
    if (ga_first_use_on_device(f, &dev) || dev < 0 || dev >= 64) {
        int n = 0;
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 132;
        if (dev < 0 || dev >= 64) return n;
        f.value[dev] = n;
    }
    return f.value[dev];
}
