// K2: tile binning and per-tile depth sort.
//
// Upstream (rasterizer_impl.cu) builds one global list of 64-bit keys
// (tile<<32 | depth bits), runs a device-wide radix sort and reads the
// instance count back to the host.  Here: K1 has already counted instances
// per tile; (a) one block scans the per-tile counts into tile ranges,
// (b) every surfel scatters (depth bits<<32 | surfel) into its tiles' ranges,
// (c) one warp per tile sorts its range in registers (tiles above 512 instances: one block, shared memory).  Because the keys
// are unique, the sorted order equals upstream's stable sort of the
// duplication order (ascending surfel index) -- bit-exact -- without a global
// sort, without a host read-back and with ~3 passes over 8-byte keys instead
// of ~10 over 12-byte pairs.
#include "raster_common.cuh"
#include "device_once.cuh"

#define SCAN_THREADS 1024
#define SCAN_TILES_PER_THREAD 8    // tiles per thread and pass: one pass covers 8192 tiles (C2: 6144)
#define SORT_WARP_MAX 512          // tiles up to this many instances are sorted by a single warp in registers

// One CTA.  Thread t owns tiles base + j * SCAN_THREADS + t (j < SCAN_TILES_PER_THREAD), so every load and store
// instruction is coalesced.  A pass loads all the replica counters of its tiles in one wave, scans the tile sums
// round by round in shared memory, then reads the counters again (from cache) and writes the tile starts and
// cursors in one wave.  Tiles above SORT_WARP_MAX are appended to ws.big_tiles (in no particular order) and counted
// in status[3].
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
            if (v[j] > SORT_WARP_MAX) ws.big_tiles[atomicAdd(&s_big, 1)] = (uint32_t)(base + j * SCAN_THREADS + threadIdx.x);
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

// Ascending-only bitonic network (flip + half-cleaners): every compare-exchange
// moves the minimum to the lower index, so virtual +inf padding beyond n never
// moves and n need not be a power of two.  Works on shared or global memory.
__device__ __forceinline__ void block_bitonic_sort(unsigned long long *a, int n)
{
    int n2 = 1;
    while (n2 < n) n2 <<= 1;
    for (int k = 2; k <= n2; k <<= 1) {
        // flip step: partner = mirror inside the k-block
        for (int t = threadIdx.x; t < n2 / 2; t += blockDim.x) {
            const int blk = t / (k / 2), off = t % (k / 2);
            const int i = blk * k + off, p = blk * k + k - 1 - off;
            if (p < n) {
                unsigned long long x = a[i], y = a[p];
                if (x > y) { a[i] = y; a[p] = x; }
            }
        }
        __syncthreads();
        for (int j = k / 4; j >= 1; j >>= 1) {
            for (int t = threadIdx.x; t < n2 / 2; t += blockDim.x) {
                const int i = (t / j) * 2 * j + (t % j), p = i + j;
                if (p < n) {
                    unsigned long long x = a[i], y = a[p];
                    if (x > y) { a[i] = y; a[p] = x; }
                }
            }
            __syncthreads();
        }
    }
}

#define SORT_SMEM_KEYS 4096

// Warp-level bitonic sort of up to 32*KPL keys held in registers, element i = r*32 + lane (striped, so global
// loads/stores are coalesced): partner distances < 32 are shuffles, distances >= 32 stay inside the lane.
// No shared memory and no block barrier.  Only the in-lane stages (static register indices) are unrolled; the
// shuffle stages run as a loop over the distance -- fully unrolled, the four instantiations came to 27k
// instructions and the kernel spent half its time on instruction-cache misses (profiles/r01_raster_small.md).
template <int KPL>
__device__ __forceinline__ void warp_shuffle_stages(unsigned long long (&v)[KPL], int lane, int k, int jstart)
{
#pragma unroll 1
    for (int j = jstart; j >= 1; j >>= 1) {
        const bool lower = (lane & j) == 0;
#pragma unroll
        for (int r = 0; r < KPL; r++) {
            const bool asc = ((((r << 5) | lane) & k) == 0);
            const unsigned long long mine = v[r];
            const unsigned long long other = __shfl_xor_sync(0xffffffffu, mine, j);
            const bool keep_min = (lower == asc);
            v[r] = keep_min ? (mine < other ? mine : other) : (mine > other ? mine : other);
        }
    }
}

template <int KPL>
__device__ __forceinline__ void warp_bitonic_sort(unsigned long long (&v)[KPL], int lane)
{
    constexpr int N = 32 * KPL;
#pragma unroll 1
    for (int k = 2; k <= 32; k <<= 1) warp_shuffle_stages<KPL>(v, lane, k, k >> 1);
#pragma unroll
    for (int k = 64; k <= N; k <<= 1) {
#pragma unroll
        for (int j = k >> 1; j >= 32; j >>= 1) {
            const int jr = j >> 5;
#pragma unroll
            for (int r = 0; r < KPL; r++) {
                if ((r & jr) == 0) {
                    const bool asc = (((r << 5) & k) == 0);              // k >= 64 here: decided by r alone
                    unsigned long long a = v[r], b = v[r | jr];
                    const bool sw = asc ? (a > b) : (a < b);
                    v[r] = sw ? b : a;
                    v[r | jr] = sw ? a : b;
                }
            }
        }
        warp_shuffle_stages<KPL>(v, lane, k, 16);
    }
}

template <int KPL>
__device__ __forceinline__ void warp_sort_tile(unsigned long long *gk, uint32_t *gid, int n, int lane)
{
    unsigned long long v[KPL];
#pragma unroll
    for (int r = 0; r < KPL; r++) {
        const int i = r * 32 + lane;
        v[r] = i < n ? gk[i] : 0xffffffffffffffffull;
    }
    warp_bitonic_sort<KPL>(v, lane);
#pragma unroll
    for (int r = 0; r < KPL; r++) {
        const int i = r * 32 + lane;
        if (i < n) {
            gk[i] = v[r];
            gid[i] = (uint32_t)(v[r] & 0xffffffffull);
        }
    }
}

// One launch sorts every tile.  CTAs [0, big_ctas) take the tiles above SORT_WARP_MAX from ws.big_tiles, one block per
// tile in shared memory (global memory above SORT_SMEM_KEYS); they are dispatched first, so their long tail runs
// beside the warp-per-tile CTAs that follow, one warp per tile in registers.
#define SORT_THREADS 256
__global__ void __launch_bounds__(SORT_THREADS, 3)
sort_tiles_kernel(RasterDims d, RasterWs ws, int big_ctas)
{
    __shared__ unsigned long long s_keys[SORT_SMEM_KEYS];
    if (ws.status[1]) return;
    if ((int)blockIdx.x < big_ctas) {
        const int nbig = ws.status[3];
        for (int b = blockIdx.x; b < nbig; b += big_ctas) {
            const uint32_t t = ws.big_tiles[b];
            const uint32_t start = ws.tile_start[t], end = ws.tile_start[t + 1];
            const int n = (int)(end - start);
            unsigned long long *gk = ws.keys + start;
            if (n <= SORT_SMEM_KEYS) {
                for (int i = threadIdx.x; i < n; i += blockDim.x) s_keys[i] = gk[i];
                __syncthreads();
                block_bitonic_sort(s_keys, n);
                for (int i = threadIdx.x; i < n; i += blockDim.x) {
                    const unsigned long long k = s_keys[i];
                    gk[i] = k;
                    ws.ids[start + i] = (uint32_t)(k & 0xffffffffull);
                }
                __syncthreads();                            // s_keys is reused by the next tile
            } else {
                // rare: a tile with more instances than fit in shared memory is sorted
                // in place in global memory (L2 resident) by the same network.
                if (threadIdx.x == 0) atomicAdd(&ws.status[2], 1);
                block_bitonic_sort(gk, n);
                for (int i = threadIdx.x; i < n; i += blockDim.x)
                    ws.ids[start + i] = (uint32_t)(gk[i] & 0xffffffffull);
                __syncthreads();
            }
        }
        return;
    }
    const size_t t = (size_t)(blockIdx.x - big_ctas) * (SORT_THREADS / 32) + (threadIdx.x >> 5);
    if (t >= (size_t)d.NV * d.T) return;
    const int lane = threadIdx.x & 31;
    const uint32_t start = ws.tile_start[t], end = ws.tile_start[t + 1];
    const int n = (int)(end - start);
    if (n == 0 || n > SORT_WARP_MAX) return;
    unsigned long long *gk = ws.keys + start;
    uint32_t *gid = ws.ids + start;
    if (n <= 32) warp_sort_tile<1>(gk, gid, n, lane);
    else if (n <= 128) warp_sort_tile<4>(gk, gid, n, lane);
    else if (n <= 256) warp_sort_tile<8>(gk, gid, n, lane);
    else warp_sort_tile<16>(gk, gid, n, lane);
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
    const int tiles = d.NV * d.T;
    const int big_ctas = tiles < ga_sm_count() ? tiles : ga_sm_count();     // at most one big-tile CTA per SM
    sort_tiles_kernel<<<big_ctas + (tiles + SORT_THREADS / 32 - 1) / (SORT_THREADS / 32), SORT_THREADS, 0, s>>>(d, w, big_ctas);
    return cudaGetLastError();
}
