// K3 / K4: forward and backward alpha compositing of surfels, one CTA per
// 16x16 tile of one image, all images of the batch in one launch.
//
// Restates upstream forward.cu / backward.cu renderCUDA
// (github.com/hbb1/diff-surfel-rasterization; called from
// /root/reference/nsr/gs_surfel.py:100-114).  Differences in HOW, not WHAT:
//  * the binning leaves each tile's keys unordered; the forward's CTA for a
//    tile sorts them by depth in shared memory before it composites, and
//    writes the sorted keys and ids back for the backward.
//  * the forward evaluates only the (pixel, surfel) pairs inside each surfel's
//    conservative cull box (computed in K1), all of them in parallel, and then
//    composites every pixel from shared memory.  The cull box contains every
//    pixel that can reach alpha >= 1/255, so results are identical to
//    evaluating every (pixel, surfel) pair.
//  * the backward walks each tile back to front, keeps the per-(pixel, surfel)
//    records in shared memory, accumulates each surfel's gradient in registers
//    and issues one global atomic per (tile, surfel, component).
#include "raster_common.cuh"
#include "device_once.cuh"

#define CHUNK 256

// single-instruction approximations (MUFU.RCP / MUFU.EX2, <= 2 ulp): the IEEE division and the range-checked
// __expf cost ~10 instructions each in the inner loop; parity with the oracle stays ~1e-6 relative.
__device__ __forceinline__ float fast_rcp(float x)
{
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float fast_ex2(float x)
{
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
#define GA_M_C0 (GA_FAR_N / (GA_FAR_N - GA_NEAR_N))              /* m = C0 - C1 / depth */
#define GA_M_C1 (GA_FAR_N * GA_NEAR_N / (GA_FAR_N - GA_NEAR_N))
#define GA_NEG_HALF_LOG2E (-0.72134752044448170368f)              /* exp(-0.5 rho) = 2^(rho * this) */

struct PixelGeom {
    float s0, s1, p2, rho3d, rho2d, dx, dy, depth, G, alpha;
    bool use3d;
};

// Evaluates one (pixel, surfel) pair up to alpha; returns false when the pair
// is skipped (upstream's `continue` conditions).
__device__ __forceinline__ bool eval_pair(const float4 a, const float4 b, const float4 c,
                                          float pfx, float pfy, PixelGeom &o,
                                          float &k0, float &k1, float &k2,
                                          float &l0, float &l1, float &l2)
{
    // Tu = a.xyz, Tv = (a.w, b.x, b.y), Tw = (b.z, b.w, c.x), xy = (c.y, c.z), opacity = c.w
    k0 = pfx * b.z - a.x; k1 = pfx * b.w - a.y; k2 = pfx * c.x - a.z;
    l0 = pfy * b.z - a.w; l1 = pfy * b.w - b.x; l2 = pfy * c.x - b.y;
    const float p0 = k1 * l2 - k2 * l1, p1 = k2 * l0 - k0 * l2, p2 = k0 * l1 - k1 * l0;
    if (p2 == 0.0f) return false;
    const float ip = fast_rcp(p2);
    o.p2 = p2;
    o.s0 = p0 * ip; o.s1 = p1 * ip;
    o.rho3d = o.s0 * o.s0 + o.s1 * o.s1;
    o.dx = c.y - pfx; o.dy = c.z - pfy;
    o.rho2d = GA_FILTER_INV_SQUARE * (o.dx * o.dx + o.dy * o.dy);
    o.use3d = o.rho3d <= o.rho2d;
    const float rho = fminf(o.rho3d, o.rho2d);
    o.depth = o.use3d ? (o.s0 * b.z + o.s1 * b.w) + c.x : c.x;
    if (o.depth < GA_NEAR_N) return false;
    o.G = fast_ex2(rho * GA_NEG_HALF_LOG2E);         // rho >= 0, so upstream's `power > 0` never fires
    o.alpha = fminf(0.99f, c.w * o.G);
    return o.alpha >= 1.0f / 255.0f;
}

// A surfel's cull box clipped to the pixels [ox, xmax] x [oy, ymax] of a tile, as tile-local integers.  A pixel
// (px, py) of that range lies in the box exactly when bb.x <= px <= bb.y and bb.z <= py <= bb.w.  w = h = 0 when the
// box misses the range (also for the empty box +-1e30 of a surfel that can never reach alpha >= 1/255).
struct TileBox { int x0, y0, w, h; };
__device__ __forceinline__ TileBox clip_box(const float4 bb, int ox, int oy, int xmax, int ymax)
{
    const float x0 = ceilf(fmaxf(bb.x, (float)ox)), x1 = floorf(fminf(bb.y, (float)xmax));
    const float y0 = ceilf(fmaxf(bb.z, (float)oy)), y1 = floorf(fminf(bb.w, (float)ymax));
    if (!(x1 >= x0 && y1 >= y0)) return {0, 0, 0, 0};
    return {(int)x0 - ox, (int)y0 - oy, (int)(x1 - x0) + 1, (int)(y1 - y0) + 1};
}

// Forward staging record (tile-local, computed once per (tile, surfel) by the
// staging thread): with o = tile origin, k_o = o.x*Tw - Tu, l_o = o.y*Tw - Tv,
//   p(dx,dy) = (k_o + dx*Tw) x (l_o + dy*Tw) = C + dx*A + dy*B,
//   C = k_o x l_o, A = Tw x l_o, B = k_o x Tw            (Tw x Tw = 0)
// which is upstream's cross(k, l) re-associated around the tile origin (all
// terms stay O(tile size), so no precision is lost) and costs 6 FMAs per pixel.
//  rec[0] = C.x C.y C.z A.x | rec[1] = A.y A.z B.x B.y | rec[2] = B.z Tw.x Tw.y Tw.z
//  rec[3] = xy.x-o.x xy.y-o.y opacity - | rec[4] = n.x n.y n.z r | rec[5] = g b - -
//
// The tile's instances are staged in chunks of 256 list positions.  Each slot also gets its cull box clipped to the
// tile's pixels inside the image (origin, width, a reciprocal for the division by the width) and its pair count
// w * h; an exclusive scan of the counts gives each slot's pair base.  The chunk is cut into WINDOWS of consecutive
// slots whose pairs fit FWD_PAIRS.  A box holds at most 256 pixels, so every window holds at least one slot.  Per
// window:
//   phase 1 (pair-parallel): the threads take consecutive pairs of the window's (slot, pixel of the clipped box)
//     enumeration, find the slot by a binary search over the pair bases and evaluate the pair.  A pair that reaches
//     alpha >= 1/255 stores {alpha, depth} at its pair index and sets the slot's bit in its pixel's slot mask.
//     Pixels outside a box never reach alpha >= 1/255 (the box is conservative), so nothing else is evaluated.
//   phase 2 (pixel-parallel): every thread composites its pixel's set bits in ascending slot order, i.e. list order,
//     reading {alpha, depth} back from the pair buffer.  The compositing state stays in registers across windows.
// C2 scene (tools/raster_rounds.py): phase 1 needs about half the warp rounds of evaluating every surfel whose box
// meets a 4x2 pixel group, and no compositing round waits on an evaluation.
//
// LISTS: the kernel also records, per pixel, every surfel that contributed -- {position in the tile list, alpha,
// depth} -- into a tile-major array (entry k of the tile's 256 pixels is one contiguous 4 KB row, so a warp's store is
// four full 128-byte lines).  The backward then walks exactly these entries: no cull tests, no pair re-evaluation for
// pairs that do not contribute, and the contribution decisions are the forward's own bits.  It also counts every
// instance's contributions (inst_cnt), which sizes that instance's records in the backward exactly.
// Three CTAs per SM: FwdSmem is about 67 KB.  A 2048-pair buffer fits four CTAs per SM, but on C2 it measured slower
// (render_fwd 0.343 against 0.318 ms, H100 SXM at 400 W): more chunks need a second window, and each window costs
// barriers and a pass over the masks.
#define FWD_PAIRS 4096              /* window pair buffer, 32 KB */

struct FwdSmem {
    float4 rec[6][CHUNK];           // the chunk's staged records, see above
    float2 pair[FWD_PAIRS];         // {alpha, depth} of the window's passing pairs, by pair index; before the first
                                    // window: the tile's keys, sorted (FWD_PAIRS keys of 8 bytes fit)
    uint32_t mask[CHUNK / 32][256]; // per pixel: the window's slots whose pair passed, slot t at bit t & 31 of word t >> 5
    int base[CHUNK + 1];            // pair base of every slot relative to the chunk; base[CHUNK] = the chunk's pairs
    uint32_t box[CHUNK];            // clipped box: x0 | y0 << 4 | w << 8 | (65536 / w + 1) << 13
    int cnt[CHUNK];                 // LISTS: contributions of each staged instance
    int wsum[8];
};

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

// Warp-level bitonic sort of 32*KPL keys held in registers, element i = r*32 + lane: partner distances < 32 are
// shuffles, distances >= 32 stay inside the lane.  Fully unrolled (KPL <= 2 here): every stage is one 64-bit shuffle,
// one 64-bit compare and a select, since the compiler can work out each stage's direction bits once per lane.
template <int KPL>
__device__ __forceinline__ void warp_shuffle_stages(unsigned long long (&v)[KPL], int lane, int k, int jstart)
{
#pragma unroll
    for (int j = jstart; j >= 1; j >>= 1) {
        const bool lower = (lane & j) == 0;
#pragma unroll
        for (int r = 0; r < KPL; r++) {
            const bool asc = ((((r << 5) | lane) & k) == 0);
            const unsigned long long mine = v[r];
            const unsigned long long other = __shfl_xor_sync(0xffffffffu, mine, j);
            const bool keep_min = (lower == asc);
            v[r] = ((other < mine) == keep_min) ? other : mine;
        }
    }
}

template <int KPL>
__device__ __forceinline__ void warp_bitonic_sort(unsigned long long (&v)[KPL], int lane)
{
    constexpr int N = 32 * KPL;
#pragma unroll
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

// Sorts n <= 256 * KPL keys from src into a: warp w sorts keys [w * 32 * KPL, (w + 1) * 32 * KPL) in registers and
// stores that run to a (padded with ~0); then every key's rank is its position in its own run plus, for every other
// run, a binary search for the keys below it.  Keys are unique, so the ranks are a permutation of [0, n).
template <int KPL>
__device__ __forceinline__ void block_merge_sort(const unsigned long long *src, unsigned long long *a, int n,
                                                 const float *rec)
{
    constexpr int SEG = 32 * KPL;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nseg = (n + SEG - 1) / SEG;
    unsigned long long v[KPL];
    int rank[KPL];
    if (warp < nseg) {
#pragma unroll
        for (int r = 0; r < KPL; r++) {
            const int i = warp * SEG + r * 32 + lane;
            v[r] = i < n ? src[i] : ~0ull;
            // the first chunk's staging loads these records right after the sort
            if (i < n) asm volatile("prefetch.global.L2 [%0];" ::"l"(rec + (size_t)(uint32_t)v[r] * GA_REC_F));
        }
        warp_bitonic_sort<KPL>(v, lane);
#pragma unroll
        for (int r = 0; r < KPL; r++) a[warp * SEG + r * 32 + lane] = v[r];
    }
    __syncthreads();
    if (warp < nseg) {
#pragma unroll
        for (int r = 0; r < KPL; r++) rank[r] = r * 32 + lane;
        for (int sg = 0; sg < nseg; sg++) {
            if (sg == warp) continue;
            const unsigned long long *run = a + sg * SEG;
#pragma unroll
            for (int r = 0; r < KPL; r++) {
                int lo = 0;                 // largest lo <= SEG - 1 with run[lo - 1] < v[r], then one more test
#pragma unroll
                for (int step = SEG / 2; step >= 1; step >>= 1)
                    if (run[lo + step - 1] < v[r]) lo += step;
                rank[r] += lo + (run[lo] < v[r] ? 1 : 0);
            }
        }
    }
    __syncthreads();
    if (warp < nseg) {
#pragma unroll
        for (int r = 0; r < KPL; r++)
            if (warp * SEG + r * 32 + lane < n) a[rank[r]] = v[r];
    }
    __syncthreads();
}

// Sorts the tile's n keys [start, start + n) ascending (the scatter wrote them unordered) and writes them back to
// ws.keys, with their surfel ids to ws.ids.  The whole tile is sorted even when compositing stops early: the backward
// reads the ids of every position up to the tile's deepest contributor.  Tiles up to FWD_PAIRS keys are sorted in s
// (the pair buffer, idle until the first window), where they stay for the first chunk's staging; larger tiles are
// sorted in place in global memory (L2 resident) by the bitonic network and counted in status[2].
// The forward is bound by instruction issue, so the sort's cost is its instruction count.  On C2 (H100 80GB HBM3)
// it made render_fwd 18 us longer per step with unrolled warp runs + binary-search ranks and the record prefetch (700 W
// power limit); at 400 W: 25 us with the warp stages as a loop, 31 us without the prefetch, 56 us with a rank sort
// (every key against every key) and 94 us with the bitonic network for every tile.
__device__ __forceinline__ void sort_tile(const RasterWs &ws, uint32_t start, int n, unsigned long long *s, const float *rec)
{
    unsigned long long *gk = ws.keys + start;
    if (n > FWD_PAIRS) {
        if (threadIdx.x == 0) atomicAdd(&ws.status[2], 1);
        block_bitonic_sort(gk, n);
        for (int i = threadIdx.x; i < n; i += 256) ws.ids[start + i] = (uint32_t)(gk[i] & 0xffffffffull);
        return;
    }
    if (n <= 256) block_merge_sort<1>(gk, s, n, rec);
    else if (n <= 512) block_merge_sort<2>(gk, s, n, rec);
    else {
        for (int i = threadIdx.x; i < n; i += 256) s[i] = gk[i];
        __syncthreads();
        block_bitonic_sort(s, n);
    }
    for (int i = threadIdx.x; i < n; i += 256) {
        const unsigned long long k = s[i];
        gk[i] = k;
        ws.ids[start + i] = (uint32_t)(k & 0xffffffffull);
    }
}

template <bool LISTS>
__global__ void __launch_bounds__(256, 3)
render_fwd_kernel(RasterDims d, RasterWs ws, const float *__restrict__ bg,
                  float *__restrict__ out_color, float *__restrict__ out_allmap)
{
    extern __shared__ __align__(16) uint8_t fwd_smem_raw[];
    FwdSmem &sm = *reinterpret_cast<FwdSmem *>(fwd_smem_raw);
    if (ws.status[1]) return;
    const int view = blockIdx.z;
    const int tile = blockIdx.y * d.gx + blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ox = blockIdx.x * GA_BLOCK_X, oy = blockIdx.y * GA_BLOCK_Y;
    const int lxi = (warp & 1) * 8 + (lane & 7), lyi = (warp >> 1) * 4 + (lane >> 3);   // a warp owns an 8x4 block
    const int pix_local = lyi * 16 + lxi;
    const int pxi = ox + lxi, pyi = oy + lyi;
    const bool inside = pxi < d.W && pyi < d.H;
    const float oxf = (float)ox, oyf = (float)oy;

    const uint32_t start = ws.tile_start[(size_t)view * d.T + tile];
    const uint32_t end = ws.tile_start[(size_t)view * d.T + tile + 1];
    const int total = (int)(end - start);
    const float *rec_base = ws.rec + (size_t)view * d.P * GA_REC_F;

    bool done = !inside;
    float T = 1.0f, C0 = 0, C1 = 0, C2 = 0, N0 = 0, N1 = 0, N2 = 0;
    float Dacc = 0, M1 = 0, M2 = 0, dist = 0, median_depth = 0;
    int last_contributor = 0, median_contributor = -1;
    int nl = 0;                                                    // LISTS: contributions of this pixel so far
    uint4 *my_list = nullptr;
    if (LISTS) my_list = ws.lists + ((size_t)view * d.T + tile) * (size_t)d.list_k * 256 + pix_local;

    const unsigned long long *skeys = reinterpret_cast<const unsigned long long *>(sm.pair);
    sort_tile(ws, start, total, reinterpret_cast<unsigned long long *>(sm.pair), rec_base);

    for (int c0 = 0; c0 < total; c0 += CHUNK) {
        if (__syncthreads_count(done) == 256) break;
        const int cnt = min(CHUNK, total - c0);
        if (LISTS) sm.cnt[threadIdx.x] = 0;
        int npairs = 0;
        if ((int)threadIdx.x < cnt) {
            // the first window overwrites the sorted keys in sm.pair; later chunks read the ids back from global memory
            const uint32_t id = (c0 == 0 && total <= FWD_PAIRS) ? (uint32_t)(skeys[threadIdx.x] & 0xffffffffull)
                                                                : ws.ids[start + c0 + threadIdx.x];
            const float4 *src = reinterpret_cast<const float4 *>(rec_base + (size_t)id * GA_REC_F);
            const float4 a = __ldg(src), b = __ldg(src + 1), c = __ldg(src + 2);
            const float4 nr = __ldg(src + 3), bb = __ldg(src + 4), gb = __ldg(src + 5);
            // Tu = a.xyz, Tv = (a.w,b.x,b.y), Tw = (b.z,b.w,c.x), xy = (c.y,c.z), opacity = c.w
            const float k0 = oxf * b.z - a.x, k1 = oxf * b.w - a.y, k2 = oxf * c.x - a.z;
            const float l0 = oyf * b.z - a.w, l1 = oyf * b.w - b.x, l2 = oyf * c.x - b.y;
            const float Cx = k1 * l2 - k2 * l1, Cy = k2 * l0 - k0 * l2, Cz = k0 * l1 - k1 * l0;
            const float Ax = b.w * l2 - c.x * l1, Ay = c.x * l0 - b.z * l2, Az = b.z * l1 - b.w * l0;
            const float Bx = k1 * c.x - k2 * b.w, By = k2 * b.z - k0 * c.x, Bz = k0 * b.w - k1 * b.z;
            sm.rec[0][threadIdx.x] = make_float4(Cx, Cy, Cz, Ax);
            sm.rec[1][threadIdx.x] = make_float4(Ay, Az, Bx, By);
            sm.rec[2][threadIdx.x] = make_float4(Bz, b.z, b.w, c.x);
            sm.rec[3][threadIdx.x] = make_float4(c.y - oxf, c.z - oyf, c.w, 0.f);
            sm.rec[4][threadIdx.x] = nr;
            sm.rec[5][threadIdx.x] = gb;
            const TileBox q = clip_box(bb, ox, oy, min(ox + 15, d.W - 1), min(oy + 15, d.H - 1));
            npairs = q.w * q.h;
            sm.box[threadIdx.x] = npairs ? (uint32_t)(q.x0 | q.y0 << 4 | q.w << 8 | (65536 / q.w + 1) << 13) : 0u;
        }
        int incl = npairs;              // inclusive scan of the pair counts over the slots
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += y;
        }
        if (lane == 31) sm.wsum[warp] = incl;
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 8; k++) incl += k < warp ? sm.wsum[k] : 0;
        sm.base[threadIdx.x] = incl - npairs;
        if (threadIdx.x == CHUNK - 1) sm.base[CHUNK] = incl;

        int t0 = 0, base = 0;           // window = slots [t0, t1); base = pair base of slot t0
        while (t0 < cnt) {
#pragma unroll
            for (int k = 0; k < CHUNK / 32; k++) sm.mask[k][threadIdx.x] = 0u;
            const int t1 = t0 + __syncthreads_count((int)threadIdx.x >= t0 && (int)threadIdx.x < cnt &&
                                                    incl - base <= FWD_PAIRS);
            // ---------------- phase 1: one thread per (slot, pixel) pair of the window
            const int wpairs = sm.base[t1] - base;
            for (int q = threadIdx.x; q < wpairs; q += 256) {
                const int Q = base + q;
                int jj = t0;            // the last slot whose base is <= Q: it has pairs, and Q is one of them
#pragma unroll
                for (int step = CHUNK / 2; step > 0; step >>= 1)
                    if (jj + step < t1 && sm.base[jj + step] <= Q) jj += step;
                const uint32_t bx = sm.box[jj];
                const int k = Q - sm.base[jj], w = (bx >> 8) & 31;
                const int ry = (k * (int)(bx >> 13)) >> 16;               // k / w for k < 256, w <= 16
                const int lx = (int)(bx & 15) + k - ry * w, ly = (int)((bx >> 4) & 15) + ry;
                const float dxf = (float)lx, dyf = (float)ly;
                const float4 f0 = sm.rec[0][jj], f1 = sm.rec[1][jj], f2 = sm.rec[2][jj], f3 = sm.rec[3][jj];
                const float p0 = f0.x + dxf * f0.w + dyf * f1.z;
                const float p1 = f0.y + dxf * f1.x + dyf * f1.w;
                const float p2 = f0.z + dxf * f1.y + dyf * f2.x;
                const float ip = fast_rcp(p2);
                const float s0 = p0 * ip, s1 = p1 * ip;
                const float rho3d = s0 * s0 + s1 * s1;
                const float ddx = f3.x - dxf, ddy = f3.y - dyf;
                // contracted explicitly: which of the two products the compiler fuses otherwise depends on the
                // surrounding code, and the images' last bits depend on it
                const float rho2d = GA_FILTER_INV_SQUARE * __fmaf_rn(ddx, ddx, __fmul_rn(ddy, ddy));
                const float rho = fminf(rho3d, rho2d);
                const float depth = (rho3d <= rho2d) ? (s0 * f2.y + s1 * f2.z) + f2.w : f2.w;
                // power = -0.5*rho > 0 never happens for rho >= 0; NaN rho (p2 == 0) fails the alpha test
                const float alpha = fminf(0.99f, f3.z * fast_ex2(rho * GA_NEG_HALF_LOG2E));
                if (p2 != 0.0f && depth >= GA_NEAR_N && alpha >= 1.0f / 255.0f) {
                    sm.pair[q] = make_float2(alpha, depth);
                    atomicOr(&sm.mask[jj >> 5][ly * 16 + lx], 1u << (jj & 31));
                }
            }
            __syncthreads();
            // ---------------- phase 2: one thread per pixel, its passing pairs in list order
            if (!done) {
                int wi = t0 >> 5;
                const int wlast = (t1 - 1) >> 5;
                uint32_t m = sm.mask[wi][pix_local];
                while (true) {
                    while (m == 0u && wi < wlast) m = sm.mask[++wi][pix_local];
                    if (m == 0u) break;
                    const int jj = wi * 32 + __ffs(m) - 1;
                    m &= m - 1;
                    const uint32_t bx = sm.box[jj];
                    const int k = (lyi - (int)((bx >> 4) & 15)) * (int)((bx >> 8) & 31) + (lxi - (int)(bx & 15));
                    const float2 ad = sm.pair[sm.base[jj] - base + k];
                    const float alpha = ad.x, depth = ad.y;
                    const float test_T = T * (1 - alpha);
                    if (test_T < 0.0001f) { done = true; break; }
                    const float4 nr = sm.rec[4][jj], gb = sm.rec[5][jj];
                    const int contributor = c0 + jj + 1;
                    const float w = alpha * T;
                    const float A = 1 - T;
                    const float mm = GA_M_C0 - GA_M_C1 * fast_rcp(depth);
                    dist += (mm * mm * A + M2 - 2 * mm * M1) * w;
                    Dacc += depth * w;
                    M1 += mm * w;
                    M2 += mm * mm * w;
                    if (T > 0.5f) { median_depth = depth; median_contributor = contributor; }
                    N0 += nr.x * w; N1 += nr.y * w; N2 += nr.z * w;
                    C0 += nr.w * w; C1 += gb.x * w; C2 += gb.y * w;
                    T = test_T;
                    last_contributor = contributor;
                    if (LISTS) {
                        atomicAdd(&sm.cnt[jj], 1);
                        if (nl < d.list_k)
                            my_list[(size_t)nl * 256] = make_uint4((uint32_t)(contributor - 1), __float_as_uint(alpha),
                                                                   __float_as_uint(depth), 0u);
                        nl++;
                    }
                }
            }
            t0 = t1;
            if (t0 < cnt) base = sm.base[t0];
            // the next window rewrites the masks and pairs; once every pixel is saturated the chunk ends here
            if (__syncthreads_count(done) == 256) break;
        }
        // every chunk holding a position below the tile's deepest contributor is staged here, so the backward finds
        // the exact record count of every instance it reads
        if (LISTS && (int)threadIdx.x < cnt) ws.inst_cnt[start + c0 + threadIdx.x] = (uint32_t)sm.cnt[threadIdx.x];
    }
    if (LISTS) {
        if (inside) ws.n_list[(size_t)view * d.H * d.W + (size_t)pyi * d.W + pxi] = nl;
        if (nl > d.list_k) ws.tile_flag[(size_t)view * d.T + tile] = 1u;      // this tile's backward recomputes
    }
    if (inside) {
        const size_t HW = (size_t)d.H * d.W;
        const size_t pix = (size_t)pyi * d.W + pxi;
        float *fT = ws.final_T + (size_t)view * 3 * HW;
        int32_t *nc = ws.n_contrib + (size_t)view * 2 * HW;
        fT[pix] = T; fT[pix + HW] = M1; fT[pix + 2 * HW] = M2;
        nc[pix] = last_contributor; nc[pix + HW] = median_contributor;
        float *oc = out_color + (size_t)view * 3 * HW;
        oc[pix] = C0 + T * bg[0]; oc[pix + HW] = C1 + T * bg[1]; oc[pix + 2 * HW] = C2 + T * bg[2];
        float *oa = out_allmap + (size_t)view * 7 * HW;
        oa[pix] = Dacc;
        oa[pix + HW] = 1 - T;
        oa[pix + 2 * HW] = N0; oa[pix + 3 * HW] = N1; oa[pix + 4 * HW] = N2;
        oa[pix + 5 * HW] = median_depth;
        oa[pix + 6 * HW] = dist;
    }
}

cudaError_t ga_launch_render_fwd(const RasterDims &d, const RasterWs &w, const float *bg,
                                 float *out_color, float *out_allmap, cudaStream_t s)
{
    static GaPerDevice attr_set;
    if (ga_first_use_on_device(attr_set)) {
        cudaError_t e = cudaFuncSetAttribute(render_fwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)sizeof(FwdSmem));
        if (e == cudaSuccess)
            e = cudaFuncSetAttribute(render_fwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)sizeof(FwdSmem));
        if (e != cudaSuccess) return e;
    }
    dim3 grid(d.gx, d.gy, d.NV);
    if (d.list_k > 0) render_fwd_kernel<true><<<grid, 256, sizeof(FwdSmem), s>>>(d, w, bg, out_color, out_allmap);
    else render_fwd_kernel<false><<<grid, 256, sizeof(FwdSmem), s>>>(d, w, bg, out_color, out_allmap);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------
// K4 backward: one CTA of 256 threads per tile; each thread owns one pixel of the tile (a warp an 8x4 block).
//
// The tile's instances are staged back to front in chunks of 256 list positions (slot t = position hi-1-t) and each
// chunk is cut into WINDOWS of consecutive slots whose records fit BWD_RECORDS 16-byte records in shared memory.  An
// instance's record bound is its exact contribution count from the forward (LISTS) or the pixels of its cull box
// inside the tile (recompute); both are <= 256 <= BWD_RECORDS, so every window holds at least one instance.  Per
// window:
//   phase A (pixel-parallel, back to front): every thread runs its pixel's compositing recurrences over the window's
//     contributions -- from the per-pixel lists the forward recorded (LISTS), or by culling and re-evaluating the
//     staged surfels -- and appends the record (pixel, dL/dalpha, dL/dz, w) to the instance's slice of the window's
//     record buffer.  The recurrence state stays in registers from one window to the next.
//   phase B (instance-parallel): the window's non-empty instances, sorted by record count so that the lane pairs of a
//     warp get instances of similar length, are walked by BWD_TPI lanes each; they re-derive the ray-splat geometry
//     of every record with eval_pair() (upstream's cross(k, l) at the pixel; the forward's phase 1 evaluates the
//     tile-origin form instead, so the bits can differ in the last place), accumulate the 18 gradient components in
//     registers, reduce-scatter them over the lanes and add them to grad_acc: one global atomic per (tile, instance,
//     non-zero component).
// The records never leave the SM.  Tiles whose lists overflowed (and callers with list_k == 0) take the recompute
// path of the same launch.
// ---------------------------------------------------------------------------
// Two CTAs per SM: ~104 KB of shared memory and up to 128 registers each.  Three (2048 records, 80 registers) were
// measured slower on C2, 0.465 against 0.407 ms: the recurrence state that phase A carries across phase B does not
// fit next to phase B's accumulators in 80 registers (176 B of spills).
#define BWD_RECORDS 4096            /* window record buffer, 64 KB */
#define BWD_TPI 2                   /* lanes per instance in phase B */

struct BwdSmem {
    float4 rec[6][CHUNK];           // the chunk's staged surfel records, slot t = list position hi-1-t
    uint4 recs[BWD_RECORDS];        // the window's records, instance by instance
    // per pixel: {dL/dcolor (3), dL/dnormal.x}, {dL/dnormal.yz, dL/ddepth, dL/dalpha_acc}, {dL/ddist, dL/dmedian, M1, M2};
    // phase A reads its pixel's constants from here, which keeps them out of the registers phase B needs
    float4 up[3][256];
    uint32_t id[CHUNK];             // surfel of every slot
    int off[CHUNK];                 // start of every slot's record slice, relative to the chunk
    int cnt[CHUNK];                 // records appended to it so far
    int bin[64];                    // phase-B counting sort by record count
    uint16_t perm[CHUNK];
    int wsum[8];
    int maxc, m;
};

// reduce-scatter of 18 components over TPI (2/4/8/16) consecutive lanes by recursive halving: after level l a lane
// is responsible for half of the components it held before; the fully reduced leftovers are added to dst.
template <int TPI>
__device__ __forceinline__ void reduce_scatter18(const float (&g)[GA_GRAD_F], int lane, float *__restrict__ dst)
{
    int off = 0, size = 9;
    float a9[10];
    {
        const bool u = lane & (TPI >> 1);
#pragma unroll
        for (int i = 0; i < 9; i++) {
            const float keep = u ? g[9 + i] : g[i], send = u ? g[i] : g[9 + i];
            a9[i] = keep + __shfl_xor_sync(0xffffffffu, send, TPI >> 1);
        }
        a9[9] = 0.f;
        off += u ? 9 : 0;
    }
    if constexpr (TPI == 2) {
#pragma unroll
        for (int i = 0; i < 9; i++)
            if (a9[i] != 0.f) atomicAdd(dst + off + i, a9[i]);
        return;
    } else {
        float b5[6];
        {
            const bool u = lane & (TPI >> 2);
#pragma unroll
            for (int i = 0; i < 5; i++) {
                const float keep = u ? a9[5 + i] : a9[i], send = u ? a9[i] : a9[5 + i];
                b5[i] = keep + __shfl_xor_sync(0xffffffffu, send, TPI >> 2);
            }
            b5[5] = 0.f;
            off += u ? 5 : 0; size = u ? 4 : 5;
        }
        if constexpr (TPI == 4) {
#pragma unroll
            for (int i = 0; i < 5; i++)
                if (i < size && b5[i] != 0.f) atomicAdd(dst + off + i, b5[i]);
            return;
        } else {
            float c3[4];
            {
                const bool u = lane & (TPI >> 3);
#pragma unroll
                for (int i = 0; i < 3; i++) {
                    const float keep = u ? b5[3 + i] : b5[i], send = u ? b5[i] : b5[3 + i];
                    c3[i] = keep + __shfl_xor_sync(0xffffffffu, send, TPI >> 3);
                }
                c3[3] = 0.f;
                off += u ? 3 : 0; size = u ? size - 3 : 3;
            }
            if constexpr (TPI == 8) {
#pragma unroll
                for (int i = 0; i < 3; i++)
                    if (i < size && c3[i] != 0.f) atomicAdd(dst + off + i, c3[i]);
                return;
            } else {
                const bool u = lane & (TPI >> 4);
                float d2[2];
#pragma unroll
                for (int i = 0; i < 2; i++) {
                    const float keep = u ? c3[2 + i] : c3[i], send = u ? c3[i] : c3[2 + i];
                    d2[i] = keep + __shfl_xor_sync(0xffffffffu, send, TPI >> 4);
                }
                off += u ? 2 : 0; size = u ? max(size - 2, 0) : min(size, 2);
#pragma unroll
                for (int i = 0; i < 2; i++)
                    if (i < size && d2[i] != 0.f) atomicAdd(dst + off + i, d2[i]);
            }
        }
    }
}

__device__ __forceinline__ int clipped_box_area(const float4 bb, int ox, int oy)
{
    const TileBox q = clip_box(bb, ox, oy, ox + 15, oy + 15);
    return q.w * q.h;
}

// LISTS = true: every thread walks ITS pixel's list entries -- {list position, alpha, depth}, the forward's own bits --
// back to front with three entries in flight in registers, so there is no cull test and no pair evaluation for
// surfels that do not reach alpha >= 1/255 at the pixel.  LISTS = false culls and re-evaluates every staged surfel.
template <bool LISTS>
__device__ __forceinline__ void bwd_tile(const RasterDims &d, const RasterWs &ws, BwdSmem &sm, const float *__restrict__ bg,
                                         const float *__restrict__ dL_dcolor, const float *__restrict__ dL_dallmap,
                                         float *__restrict__ grad_acc)
{
    const int view = blockIdx.z;
    const int tile = blockIdx.y * d.gx + blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ox = blockIdx.x * GA_BLOCK_X, oy = blockIdx.y * GA_BLOCK_Y;
    const int lx0 = (warp & 1) * 8, ly0 = (warp >> 1) * 4;
    const int lxi = lx0 + (lane & 7), lyi = ly0 + (lane >> 3);
    const int pxi = ox + lxi, pyi = oy + lyi;
    const int pix_local = lyi * 16 + lxi;
    const bool inside = pxi < d.W && pyi < d.H;
    const float pfx = (float)pxi, pfy = (float)pyi;

    const uint32_t start = ws.tile_start[(size_t)view * d.T + tile];
    const size_t HW = (size_t)d.H * d.W;
    const size_t pix = inside ? (size_t)pyi * d.W + pxi : 0;
    const float *fT = ws.final_T + (size_t)view * 3 * HW;
    const int32_t *nc = ws.n_contrib + (size_t)view * 2 * HW;
    const float *rec_base = ws.rec + (size_t)view * d.P * GA_REC_F;
    float *acc_base = grad_acc + (size_t)view * d.P * GA_GRAD_F;

    const float T_final = inside ? fT[pix] : 0.f;
    float T = T_final;
    const int last_contributor = inside ? nc[pix] : 0;
    const int median_contributor = inside ? nc[pix + HW] : 0;
    float bg_dot_dpixel = 0.f;
    {
        float4 u0 = make_float4(0.f, 0.f, 0.f, 0.f), u1 = u0, u2 = u0;
        if (inside) {
            const float *gc = dL_dcolor + (size_t)view * 3 * HW;
            const float *ga = dL_dallmap + (size_t)view * 7 * HW;
            u0 = make_float4(gc[pix], gc[pix + HW], gc[pix + 2 * HW], ga[pix + 2 * HW]);
            u1 = make_float4(ga[pix + 3 * HW], ga[pix + 4 * HW], ga[pix], ga[pix + HW]);
            u2 = make_float4(ga[pix + 6 * HW], ga[pix + 5 * HW], fT[pix + HW], fT[pix + 2 * HW]);
        }
        sm.up[0][pix_local] = u0;
        sm.up[1][pix_local] = u1;
        sm.up[2][pix_local] = u2;
        bg_dot_dpixel = bg[0] * u0.x + bg[1] * u0.y + bg[2] * u0.z;
    }
    const float final_A = 1 - T_final;
    // Upstream keeps one suffix accumulator per output channel (colour 3, depth, alpha, normal 3), all with the same
    // recurrence acc = last_alpha * last_value + (1 - last_alpha) * acc, and adds (value - acc) * dL/dchannel to
    // dL/dalpha.  The sum over channels is linear, so ONE scalar recurrence on v = sum_ch value_ch * dL/dchannel does
    // the same work (8 recurrences and ~20 registers less per pair).
    float last_alpha = 0, v_last = 0, v_acc = 0, last_dL_dT = 0;

    const uint4 *my_list = nullptr;
    int kk = -1;                        // LISTS: this pixel's next entry, counting down
    if (LISTS) {
        my_list = ws.lists + ((size_t)view * d.T + tile) * (size_t)d.list_k * 256 + pix_local;
        kk = (inside ? ws.n_list[(size_t)view * HW + pix] : 0) - 1;
#pragma unroll
        for (int q = 0; q < 8; q++)
            if (kk >= q) asm volatile("prefetch.global.L2 [%0];" ::"l"(my_list + (size_t)(kk - q) * 256));
    }

    // nothing behind the deepest contributor of the tile can receive gradient
    if (threadIdx.x == 0) sm.maxc = 0;
    __syncthreads();
    {
        int mc = last_contributor;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mc = max(mc, __shfl_xor_sync(0xffffffffu, mc, o));
        if (lane == 0) atomicMax(&sm.maxc, mc);
    }
    __syncthreads();
    const int total = sm.maxc;          // list positions [0,total) matter

    for (int hi = total; hi > 0; hi -= CHUNK) {
        const int cnt = min(CHUNK, hi);
        // stage positions hi-cnt..hi-1, slot t = position hi-1-t, with the record bound of every slot
        int bound = 0;
        if ((int)threadIdx.x < cnt) {
            const int pos = hi - 1 - (int)threadIdx.x;
            const uint32_t id = ws.ids[start + pos];
            sm.id[threadIdx.x] = id;
            const float4 *src = reinterpret_cast<const float4 *>(rec_base + (size_t)id * GA_REC_F);
            float4 q[6];
#pragma unroll
            for (int k = 0; k < 6; k++) { q[k] = __ldg(src + k); sm.rec[k][threadIdx.x] = q[k]; }
            bound = LISTS ? (int)ws.inst_cnt[start + pos] : clipped_box_area(q[4], ox, oy);
        }
        int incl = bound;               // inclusive scan of the bounds over the slots
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += y;
        }
        if (lane == 31) sm.wsum[warp] = incl;
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 8; k++) incl += k < warp ? sm.wsum[k] : 0;
        sm.off[threadIdx.x] = incl - bound;
        sm.cnt[threadIdx.x] = 0;

        int t0 = 0, base = 0;           // window = slots [t0, t1); base = offset of slot t0's slice
        while (t0 < cnt) {
            if (threadIdx.x < 64) sm.bin[threadIdx.x] = 0;
            const int t1 = t0 + __syncthreads_count((int)threadIdx.x >= t0 && (int)threadIdx.x < cnt &&
                                                    incl - base <= BWD_RECORDS);

            // ---------------- phase A: one (pixel, surfel) contribution = the recurrences backwards + one record
            auto contribute = [&](const int jj, const int contributor, const float alpha, const float c_d) {
                const float4 nr = sm.rec[3][jj], gb = sm.rec[5][jj];
                const float4 u0 = sm.up[0][pix_local], u1 = sm.up[1][pix_local], u2 = sm.up[2][pix_local];
                const float dL_ddepth = u1.z, dL_dreg = u2.x, final_D = u2.z, final_D2 = u2.w;
                const float inv1ma = fast_rcp(1.f - alpha);
                T = T * inv1ma;
                const float w = alpha * T;
                float dL_dz = 0.0f;
                const float inv_cd = fast_rcp(c_d);
                const float m_d = GA_M_C0 - GA_M_C1 * inv_cd;
                const float dmd_dd = GA_M_C1 * inv_cd * inv_cd;
                if (contributor == median_contributor - 1) dL_dz += u2.y;
                const float dL_dweight = (final_D2 + m_d * m_d * final_A - 2 * m_d * final_D) * dL_dreg;
                const float dL_dmd = 2.0f * (T * alpha) * (m_d * final_A - final_D) * dL_dreg;
                dL_dz += dL_dmd * dmd_dd;
                // v = (colour . dL/dcolour) + depth dL/ddepth + 1 dL/dalpha_acc + (normal . dL/dnormal)
                const float v = ((nr.w * u0.x + gb.x * u0.y) + (gb.y * u0.z + c_d * dL_ddepth)) +
                                ((nr.x * u0.w + nr.y * u1.x) + (nr.z * u1.y + u1.w));
                v_acc = last_alpha * v_last + (1.f - last_alpha) * v_acc;
                v_last = v;
                float dL_dalpha = (v - v_acc) + (dL_dweight - last_dL_dT);
                last_dL_dT = dL_dweight * alpha + (1 - alpha) * last_dL_dT;
                dL_dalpha *= T;
                last_alpha = alpha;
                dL_dalpha += (-T_final * inv1ma) * bg_dot_dpixel;
                dL_dz += w * dL_ddepth;
                const int slot = atomicAdd(&sm.cnt[jj], 1);          // < the slot's record bound
                sm.recs[sm.off[jj] - base + slot] =
                    make_uint4((uint32_t)pix_local, __float_as_uint(dL_dalpha), __float_as_uint(dL_dz), __float_as_uint(w));
            };
            if constexpr (LISTS) {
                const int pos_lo = hi - t1;     // the window holds positions [hi - t1, hi - t0)
                // three entries in flight; they are reloaded (from L1 / L2) per window rather than held through phase B
                uint4 e = make_uint4(0u, 0u, 0u, 0u), e1 = e, e2 = e;
                if (kk >= 0) e = __ldg(my_list + (size_t)kk * 256);
                if (kk >= 1) e1 = __ldg(my_list + (size_t)(kk - 1) * 256);
                if (kk >= 2) e2 = __ldg(my_list + (size_t)(kk - 2) * 256);
                while (true) {
                    const bool active = kk >= 0 && (int)e.x >= pos_lo;      // entries are in descending list position
                    if (!__any_sync(0xffffffffu, active)) break;
                    if (active) {
                        const uint4 cur = e;
                        e = e1; e1 = e2;
                        if (kk >= 3) e2 = __ldg(my_list + (size_t)(kk - 3) * 256);   // entries kk-1, kk-2, kk-3 are in flight
                        // ... and the row 8 below is asked into L2 (the list rows stream from HBM exactly once)
                        if (kk >= 8) asm volatile("prefetch.global.L2 [%0];" ::"l"(my_list + (size_t)(kk - 8) * 256));
                        kk--;
                        contribute(hi - 1 - (int)cur.x, (int)cur.x, __uint_as_float(cur.y), __uint_as_float(cur.z));
                    }
                }
            } else {
                const float bx_lo = (float)(ox + lx0), bx_hi = (float)(ox + lx0 + 7);
                const float by_lo = (float)(oy + ly0), by_hi = (float)(oy + ly0 + 3);
                for (int sb = t0; sb < t1; sb += 32) {
                    bool hit = false;
                    if (sb + lane < t1) {
                        const float4 bb = sm.rec[4][sb + lane];
                        hit = !(bb.y < bx_lo || bb.x > bx_hi || bb.w < by_lo || bb.z > by_hi);
                    }
                    unsigned mask = __ballot_sync(0xffffffffu, hit);
                    unsigned mine = 0;
                    while (mask) {
                        const int b = __ffs(mask) - 1;
                        mask &= mask - 1;
                        const float4 bb = sm.rec[4][sb + b];
                        if (pfx >= bb.x && pfx <= bb.y && pfy >= bb.z && pfy <= bb.w && (hi - 1 - (sb + b)) < last_contributor)
                            mine |= 1u << b;
                    }
                    if (!inside) mine = 0;
                    while (__any_sync(0xffffffffu, mine != 0)) {
                        const bool active = mine != 0;
                        const int bsel = active ? __ffs(mine) - 1 : 0;
                        mine &= mine - 1;
                        const int jj = sb + bsel;
                        const float4 a = sm.rec[0][jj], b = sm.rec[1][jj], c = sm.rec[2][jj];
                        PixelGeom pg;
                        float k0, k1, k2, l0, l1, l2;
                        const bool ok = active && eval_pair(a, b, c, pfx, pfy, pg, k0, k1, k2, l0, l1, l2);
                        if (ok) contribute(jj, hi - 1 - jj, pg.alpha, pg.depth);
                    }
                }
            }
            __syncthreads();

            // ---------------- phase B: counting sort of the window's non-empty slots by record count, descending
            const int myc = ((int)threadIdx.x >= t0 && (int)threadIdx.x < t1) ? sm.cnt[threadIdx.x] : 0;
            if (myc > 0) atomicAdd(&sm.bin[min(myc, 63)], 1);
            __syncthreads();
            if (threadIdx.x < 32) {
                // exclusive prefix over the bins in descending count order (bin 63 first); bin 0 is unused
                const int hi_bin = 63 - 2 * (int)threadIdx.x, lo_bin = hi_bin - 1;
                const int vh = sm.bin[hi_bin], vl = lo_bin >= 1 ? sm.bin[lo_bin] : 0;
                int x = vh + vl;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int y = __shfl_up_sync(0xffffffffu, x, o);
                    if ((int)threadIdx.x >= o) x += y;
                }
                const int excl = x - (vh + vl);
                sm.bin[hi_bin] = excl;
                if (lo_bin >= 1) sm.bin[lo_bin] = excl + vh;
                if (threadIdx.x == 31) sm.m = x;
            }
            __syncthreads();
            if (myc > 0) sm.perm[atomicAdd(&sm.bin[min(myc, 63)], 1)] = (uint16_t)threadIdx.x;
            __syncthreads();
            const int m = sm.m, sub = threadIdx.x % BWD_TPI;
            for (int b0 = 0; b0 < m; b0 += 256 / BWD_TPI) {
                const int slot = b0 + (int)threadIdx.x / BWD_TPI;
                const int jj = slot < m ? (int)sm.perm[slot] : 0;
                const int n = slot < m ? sm.cnt[jj] : 0;
                float g[GA_GRAD_F];
#pragma unroll
                for (int f = 0; f < GA_GRAD_F; f++) g[f] = 0.f;
                if (n > 0) {
                    const float4 a = sm.rec[0][jj], b = sm.rec[1][jj], c = sm.rec[2][jj];
                    const float opa = c.w;
                    const uint4 *lst = sm.recs + (sm.off[jj] - base);
                    for (int r = sub; r < n; r += BWD_TPI) {
                        const uint4 rc = lst[r];
                        const int p = (int)rc.x;
                        const float dL_dalpha = __uint_as_float(rc.y), dL_dz = __uint_as_float(rc.z), w = __uint_as_float(rc.w);
                        const float qx = (float)(ox + (p & 15)), qy = (float)(oy + (p >> 4));
                        PixelGeom pg;
                        float k0, k1, k2, l0, l1, l2;
                        eval_pair(a, b, c, qx, qy, pg, k0, k1, k2, l0, l1, l2);      // same code path as phase A: same bits
                        const float G = pg.G;
                        const float dL_dG = opa * dL_dalpha;                         // 0.99 clamp passed through (upstream)
                        if (pg.use3d) {
                            const float dL_ds0 = dL_dG * -G * pg.s0 + dL_dz * b.z;
                            const float dL_ds1 = dL_dG * -G * pg.s1 + dL_dz * b.w;
                            const float ip = fast_rcp(pg.p2);
                            const float q0 = dL_ds0 * ip, q1 = dL_ds1 * ip;
                            const float q2 = -(q0 * pg.s0 + q1 * pg.s1);
                            const float dk0 = l1 * q2 - l2 * q1, dk1 = l2 * q0 - l0 * q2, dk2 = l0 * q1 - l1 * q0;
                            const float dl0 = q1 * k2 - q2 * k1, dl1 = q2 * k0 - q0 * k2, dl2 = q0 * k1 - q1 * k0;
                            g[0] -= dk0; g[1] -= dk1; g[2] -= dk2;
                            g[3] -= dl0; g[4] -= dl1; g[5] -= dl2;
                            g[6] += qx * dk0 + qy * dl0 + dL_dz * pg.s0;
                            g[7] += qx * dk1 + qy * dl1 + dL_dz * pg.s1;
                            g[8] += qx * dk2 + qy * dl2 + dL_dz;
                        } else {
                            g[9] += dL_dG * (-G * GA_FILTER_INV_SQUARE * pg.dx);
                            g[10] += dL_dG * (-G * GA_FILTER_INV_SQUARE * pg.dy);
                            g[8] += dL_dz;
                        }
                        g[14] += G * dL_dalpha;
                        const float4 ua = sm.up[0][p], ub = sm.up[1][p];
                        g[15] += w * ua.x; g[16] += w * ua.y; g[17] += w * ua.z;
                        g[11] += w * ua.w; g[12] += w * ub.x; g[13] += w * ub.y;
                    }
                }
                // all lanes of the warp take part in the shuffles; lanes without records carry zeros (adds skipped)
                if (__any_sync(0xffffffffu, n > 0))
                    reduce_scatter18<BWD_TPI>(g, lane, acc_base + (size_t)(n > 0 ? sm.id[jj] : 0) * GA_GRAD_F);
            }
            t0 = t1;
            if (t0 < cnt) base = sm.off[t0];
            __syncthreads();            // the next window's phase A rewrites recs and bin; the next chunk rewrites the rest
        }
    }
}

__global__ void __launch_bounds__(256, 2)
render_bwd_kernel(RasterDims d, RasterWs ws, const float *__restrict__ bg, const float *__restrict__ dL_dcolor,
                  const float *__restrict__ dL_dallmap, float *__restrict__ grad_acc)
{
    extern __shared__ __align__(16) uint8_t bwd_smem_raw[];
    BwdSmem &sm = *reinterpret_cast<BwdSmem *>(bwd_smem_raw);
    if (ws.status[1]) return;
    if (d.list_k > 0 && ws.tile_flag[(size_t)blockIdx.z * d.T + blockIdx.y * d.gx + blockIdx.x] == 0)
        bwd_tile<true>(d, ws, sm, bg, dL_dcolor, dL_dallmap, grad_acc);
    else
        bwd_tile<false>(d, ws, sm, bg, dL_dcolor, dL_dallmap, grad_acc);
}

cudaError_t ga_launch_render_bwd(const RasterDims &d, const RasterWs &w, const float *bg,
                                 const float *dL_dcolor, const float *dL_dallmap, float *grad_acc, cudaStream_t s)
{
    static GaPerDevice attr_set;
    if (ga_first_use_on_device(attr_set)) {
        cudaError_t e = cudaFuncSetAttribute(render_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)sizeof(BwdSmem));
        if (e != cudaSuccess) return e;
    }
    dim3 grid(d.gx, d.gy, d.NV);
    render_bwd_kernel<<<grid, 256, sizeof(BwdSmem), s>>>(d, w, bg, dL_dcolor, dL_dallmap, grad_acc);
    return cudaGetLastError();
}
