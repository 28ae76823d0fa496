// K2: tile binning.
//
// Upstream (rasterizer_impl.cu) builds one global list of 64-bit keys
// (tile<<32 | depth bits), runs a device-wide radix sort and reads the
// instance count back to the host.  Here: K1 has already counted instances
// per tile; (a) one block scans the per-tile counts into tile ranges,
// (b) every surfel scatters (depth bits<<32 | surfel) into its tiles' ranges,
// unordered.  Each tile's range is sorted by the forward's CTA for that tile
// before it composites (raster_render.cu).  Because the keys are unique, the
// sorted order equals upstream's stable sort of the duplication order
// (ascending surfel index) -- bit-exact -- without a global sort and without a
// host read-back.
#include "raster_common.cuh"

#define SCAN_THREADS 1024
#define SCAN_TILES_PER_THREAD 8    // tiles per thread and pass: one pass covers 8192 tiles (C2: 6144)
#define BIG_TILE_INSTANCES 512     // tiles above this many instances are listed in ws.big_tiles

// One CTA.  Thread t owns tiles base + j * SCAN_THREADS + t (j < SCAN_TILES_PER_THREAD), so every load and store
// instruction is coalesced.  A pass loads all the replica counters of its tiles in one wave, scans the tile sums
// round by round in shared memory, then reads the counters again (from cache) and writes the tile starts and
// cursors in one wave.  Tiles above BIG_TILE_INSTANCES are appended to ws.big_tiles (in no particular order) and
// counted in status[3]; nothing on the device reads that list, it is a diagnostic of the tile size distribution.
__global__ void __launch_bounds__(SCAN_THREADS)
scan_tiles_kernel(RasterDims d, RasterWs ws)
{
    __shared__ uint32_t s_warp[32];
    __shared__ uint32_t s_carry;
    __shared__ int s_big;
    const int n = d.NV * d.T;
    if (threadIdx.x == 0) { s_carry = 0; s_big = 0; }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint4 *cnt4 = reinterpret_cast<const uint4 *>(ws.tile_count);
    for (int base = 0; base < n; base += SCAN_THREADS * SCAN_TILES_PER_THREAD) {
        uint32_t v[SCAN_TILES_PER_THREAD];
#pragma unroll
        for (int j = 0; j < SCAN_TILES_PER_THREAD; j++) {
            const int i = base + j * SCAN_THREADS + threadIdx.x;
            v[j] = 0u;
#pragma unroll
            for (int q = 0; q < GA_TILE_REPLICAS / 4; q++) {
                const uint4 c = i < n ? cnt4[(size_t)i * (GA_TILE_REPLICAS / 4) + q] : make_uint4(0u, 0u, 0u, 0u);
                v[j] += ((c.x + c.y) + c.z) + c.w;
            }
        }
        uint32_t excl[SCAN_TILES_PER_THREAD];
#pragma unroll
        for (int j = 0; j < SCAN_TILES_PER_THREAD; j++) {
            if (base + j * SCAN_THREADS >= n) { excl[j] = 0u; continue; }        // block-uniform
            if (v[j] > BIG_TILE_INSTANCES) ws.big_tiles[atomicAdd(&s_big, 1)] = (uint32_t)(base + j * SCAN_THREADS + threadIdx.x);
            uint32_t x = v[j];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
                if (lane >= o) x += y;
            }
            if (lane == 31) s_warp[warp] = x;
            __syncthreads();
            if (warp == 0) {
                uint32_t wv = s_warp[lane], wx = wv;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    uint32_t y = __shfl_up_sync(0xffffffffu, wx, o);
                    if (lane >= o) wx += y;
                }
                s_warp[lane] = wx - wv;   // exclusive warp offsets
            }
            __syncthreads();
            excl[j] = s_carry + s_warp[warp] + x - v[j];
            __syncthreads();
            if (threadIdx.x == SCAN_THREADS - 1) s_carry = excl[j] + v[j];
            __syncthreads();
        }
#pragma unroll
        for (int j = 0; j < SCAN_TILES_PER_THREAD; j++) {
            const int i = base + j * SCAN_THREADS + threadIdx.x;
            if (i >= n) continue;
            ws.tile_start[i] = excl[j];
            // every replica becomes the absolute fill cursor of its own sub-range of the tile's slots
            uint32_t run = excl[j];
            uint4 *dst = reinterpret_cast<uint4 *>(ws.tile_count) + (size_t)i * (GA_TILE_REPLICAS / 4);
#pragma unroll
            for (int q = 0; q < GA_TILE_REPLICAS / 4; q++) {
                const uint4 c = cnt4[(size_t)i * (GA_TILE_REPLICAS / 4) + q];
                uint4 cur;
                cur.x = run; run += c.x;
                cur.y = run; run += c.y;
                cur.z = run; run += c.z;
                cur.w = run; run += c.w;
                dst[q] = cur;
            }
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const uint32_t total = s_carry;
        ws.tile_start[n] = total;
        ws.status[0] = (int32_t)total;
        ws.status[1] = ((int64_t)total > d.max_instances) ? 1 : 0;
        ws.status[3] = s_big;                      // entries of ws.big_tiles
    }
}

__global__ void __launch_bounds__(256)
scatter_kernel(RasterDims d, RasterWs ws)
{
    const int view = blockIdx.y;
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= d.P || ws.status[1]) return;
    const size_t vi = (size_t)view * d.P + i;
    const uint32_t r = ws.rect[vi];
    if (r == 0) return;
    const int x0 = r & 255, y0 = (r >> 8) & 255, x1 = (r >> 16) & 255, y1 = r >> 24;
    const unsigned long long key =
        ((unsigned long long)__float_as_uint(ws.depth[vi]) << 32) | (unsigned long long)(uint32_t)i;
    // same replica as in K1 (same launch geometry: 256 threads, surfel i -> thread i % 256), so every replica
    // receives exactly the instances it counted
    const int rep = (threadIdx.x >> 5) & (GA_TILE_REPLICAS - 1);
    for (int y = y0; y < y1; y++)
        for (int x = x0; x < x1; x++) {
            const size_t t = (size_t)view * d.T + y * d.gx + x;
            const uint32_t slot = atomicAdd(&ws.tile_count[t * GA_TILE_REPLICAS + rep], 1u);
            ws.keys[slot] = key;
        }
}

cudaError_t ga_launch_binning(const RasterDims &d, const RasterWs &w, cudaStream_t s, int32_t *status_host,
                              cudaEvent_t status_event)
{
    scan_tiles_kernel<<<1, SCAN_THREADS, 0, s>>>(d, w);
    if (status_host) {
        cudaError_t e = cudaMemcpyAsync(status_host, w.status, 4 * sizeof(int32_t), cudaMemcpyDeviceToHost, s);
        if (e != cudaSuccess) return e;
    }
    if (status_event) {
        cudaError_t e = cudaEventRecord(status_event, s);
        if (e != cudaSuccess) return e;
    }
    dim3 grid((d.P + 255) / 256, d.NV);
    scatter_kernel<<<grid, 256, 0, s>>>(d, w);
    return cudaGetLastError();
}
