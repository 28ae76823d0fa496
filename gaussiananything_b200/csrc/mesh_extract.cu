// Triangle mesh from the fused TSDF units (include/ga_b200.h Part 4): marching cubes in two passes (count, emit) and
// the floater filter of utils/mesh_util.post_process_mesh (cluster triangles through shared edges, keep the large
// clusters, drop unreferenced vertices, drop degenerate triangles).
//
// Marching cubes restates Open3D's ScalableTSDFVolume::ExtractTriangleMesh: a cube is skipped when a corner's unit is
// missing or a corner has weight 0; corner k is set when tsdf < 0; a vertex sits on its grid edge at
// 0.5 vl + vl e (+ f0 vl / (f0 + f1) along the edge), in double.  Each voxel owns the edges on its +x, +y, +z axes, so
// a vertex is created exactly once without a hash map: when the edge changes sign and one of the <= 4 cubes around
// it is valid.  Built with --fmad=false (build.py) so vertices match the oracle's double arithmetic.
#include "mesh_common.cuh"

namespace {

using namespace ga_mesh;

constexpr unsigned long long EMPTY_KEY = ~0ull;

// corner k of a cube and edge i's origin corner / axis (numbering of gaussiananything_b200/mc_table.py)
__constant__ int8_t c_corner[8][3] = {{0, 0, 0}, {1, 0, 0}, {1, 1, 0}, {0, 1, 0},
                                      {0, 0, 1}, {1, 0, 1}, {1, 1, 1}, {0, 1, 1}};
__constant__ int8_t c_edge_org[12][3] = {{0, 0, 0}, {1, 0, 0}, {0, 1, 0}, {0, 0, 0}, {0, 0, 1}, {1, 0, 1},
                                         {0, 1, 1}, {0, 0, 1}, {0, 0, 0}, {1, 0, 0}, {1, 1, 0}, {0, 1, 0}};
__constant__ int8_t c_edge_axis[12] = {0, 1, 0, 1, 0, 1, 0, 1, 2, 2, 2, 2};

struct Grid {
    const int32_t *unit_slot;
    int nx, ny, nz;
};

__device__ __forceinline__ Grid load_grid(const int32_t *unit_slot, const int32_t *box)
{
    return Grid{unit_slot, box[3], box[4], box[5]};
}

__device__ __forceinline__ void unit_coords(const Grid &g, int u, int *c)
{
    c[0] = u / (g.ny * g.nz);
    c[1] = (u / g.nz) % g.ny;
    c[2] = u % g.nz;
}

// voxel index (slot * 4096 + local) of box-relative voxel coordinates, or -1 when its unit is not pooled
__device__ __forceinline__ int64_t voxel_at(const Grid &g, int vx, int vy, int vz)
{
    if (vx < 0 || vy < 0 || vz < 0) return -1;
    const int ux = vx >> 4, uy = vy >> 4, uz = vz >> 4;
    if (ux >= g.nx || uy >= g.ny || uz >= g.nz) return -1;
    const int s = g.unit_slot[((size_t)ux * g.ny + uy) * g.nz + uz];
    if (s < 0) return -1;
    return (int64_t)s * 4096 + (((vx & 15) * 16 + (vy & 15)) * 16 + (vz & 15));
}

// case index of the cube whose corner 0 is at box-relative voxel (vx, vy, vz); 0 when invalid
__device__ int cube_case(const Grid &g, const float *tsdf, const float *weight, int vx, int vy, int vz)
{
    int c = 0;
    for (int k = 0; k < 8; k++) {
        const int64_t i = voxel_at(g, vx + c_corner[k][0], vy + c_corner[k][1], vz + c_corner[k][2]);
        if (i < 0 || weight[i] == 0.f) return 0;
        if (tsdf[i] < 0.f) c |= 1 << k;
    }
    return c;
}

__device__ __forceinline__ int tri_count(const int8_t *tri_table, int c)
{
    int n = 0;
    while (n < 5 && tri_table[c * GA_MESH_TRI_ROW + 3 * n] >= 0) n++;
    return n;
}

// voxel i of pooled unit slot i >> 12, as box-relative voxel coordinates
__device__ __forceinline__ void voxel_coords(const Grid &g, const int32_t *pool, int64_t i, int *p)
{
    int uc[3];
    unit_coords(g, pool[i >> 12], uc);
    const int l = (int)(i & 4095);
    p[0] = uc[0] * 16 + (l >> 8);
    p[1] = uc[1] * 16 + ((l >> 4) & 15);
    p[2] = uc[2] * 16 + (l & 15);
}

__global__ void __launch_bounds__(256)
cube_case_kernel(const float *__restrict__ voxels, int64_t nvox, const int32_t *__restrict__ pool,
                 const int32_t *__restrict__ unit_slot, const int32_t *__restrict__ box,
                 const int8_t *__restrict__ tri_table, uint8_t *__restrict__ cube, int32_t *__restrict__ tri_off)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nvox) return;
    const Grid g = load_grid(unit_slot, box);
    int p[3];
    voxel_coords(g, pool, i, p);
    const int c = cube_case(g, voxels, voxels + nvox, p[0], p[1], p[2]);
    cube[i] = (uint8_t)c;
    tri_off[i] = tri_count(tri_table, c);
}

__global__ void __launch_bounds__(256)
edge_flag_kernel(const float *__restrict__ voxels, int64_t nvox, const int32_t *__restrict__ pool,
                 const int32_t *__restrict__ unit_slot, const int32_t *__restrict__ box, uint8_t *__restrict__ cube,
                 int32_t *__restrict__ vert_off)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nvox) return;
    const Grid g = load_grid(unit_slot, box);
    const float *tsdf = voxels, *weight = voxels + nvox;
    int p[3];
    voxel_coords(g, pool, i, p);
    int flags = 0;
    if (weight[i] != 0.f) {
        const bool neg = tsdf[i] < 0.f;
        for (int a = 0; a < 3; a++) {
            int q[3] = {p[0], p[1], p[2]};
            q[a] += 1;
            const int64_t j = voxel_at(g, q[0], q[1], q[2]);
            if (j < 0 || weight[j] == 0.f || (tsdf[j] < 0.f) == neg) continue;
            const int b = (a + 1) % 3, c = (a + 2) % 3;
            bool any = false;
            for (int k = 0; k < 4 && !any; k++) {
                int o[3] = {p[0], p[1], p[2]};
                o[b] -= k & 1;
                o[c] -= k >> 1;
                const int64_t m = voxel_at(g, o[0], o[1], o[2]);
                if (m >= 0) {
                    const int cc = cube[m];
                    any = cc != 0 && cc != 255;
                }
            }
            if (any) flags |= 1 << a;
        }
    }
    cube[nvox + i] = (uint8_t)flags;
    vert_off[i] = __popc(flags);
}

__global__ void __launch_bounds__(256)
emit_kernel(const float *__restrict__ voxels, int64_t nvox, const int32_t *__restrict__ pool,
            const int32_t *__restrict__ unit_slot, const int32_t *__restrict__ box, const double *__restrict__ volume,
            const int8_t *__restrict__ tri_table, const uint8_t *__restrict__ cube,
            const int32_t *__restrict__ vert_off, const int32_t *__restrict__ tri_off, double *__restrict__ vertices,
            double *__restrict__ colors, int32_t *__restrict__ triangles)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nvox) return;
    const Grid g = load_grid(unit_slot, box);
    const float *tsdf = voxels, *rgb = voxels + 2 * nvox;
    int p[3];
    voxel_coords(g, pool, i, p);
    const int flags = cube[nvox + i];
    if (flags) {
        const double vl = volume[0], half = vl * 0.5;
        double e[3];
        for (int a = 0; a < 3; a++) e[a] = half + vl * (double)(box[a] * 16 + p[a]);
        int out = vert_off[i];
        for (int a = 0; a < 3; a++) {
            if (!((flags >> a) & 1)) continue;
            int q[3] = {p[0], p[1], p[2]};
            q[a] += 1;
            const int64_t j = voxel_at(g, q[0], q[1], q[2]);
            const double f0 = fabs((double)tsdf[i]), f1 = fabs((double)tsdf[j]);
            double pt[3] = {e[0], e[1], e[2]};
            pt[a] += f0 * vl / (f0 + f1);
            for (int k = 0; k < 3; k++) {
                vertices[(size_t)out * 3 + k] = pt[k];
                const double c0 = (double)rgb[k * nvox + i] / 255.0, c1 = (double)rgb[k * nvox + j] / 255.0;
                colors[(size_t)out * 3 + k] = (f1 * c0 + f0 * c1) / (f0 + f1);
            }
            out++;
        }
    }
    const int c = cube[i];
    const int nt = tri_count(tri_table, c);
    for (int t = 0; t < nt; t++) {
        for (int k = 0; k < 3; k++) {
            const int ei = tri_table[c * GA_MESH_TRI_ROW + 3 * t + k];
            const int a = c_edge_axis[ei];
            const int64_t m = voxel_at(g, p[0] + c_edge_org[ei][0], p[1] + c_edge_org[ei][1], p[2] + c_edge_org[ei][2]);
            const int fl = cube[nvox + m];
            triangles[((size_t)tri_off[i] + t) * 3 + k] = vert_off[m] + __popc(fl & ((1 << a) - 1));
        }
    }
}

// ---- clusters of triangles connected through shared edges: lock-free union-find, roots are the smallest index ----

__device__ __forceinline__ unsigned long long edge_key(int a, int b)
{
    const unsigned lo = (unsigned)min(a, b), hi = (unsigned)max(a, b);
    return ((unsigned long long)lo << 32) | hi;
}

__device__ __forceinline__ unsigned long long mix(unsigned long long k)
{
    k ^= k >> 33;
    k *= 0xff51afd7ed558ccdull;
    k ^= k >> 33;
    return k;
}

__device__ __forceinline__ int find_root(int *parent, int x)
{
    while (true) {
        const int y = __ldcg(parent + x);
        if (y == x) return x;
        const int z = __ldcg(parent + y);
        if (z != y) parent[x] = z;                     // path halving: z is an ancestor of x
        x = y;
    }
}

__global__ void __launch_bounds__(256)
cluster_init_kernel(int n_tri, int64_t slots, unsigned long long *keys, int *vals, int *parent, int *count)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < slots) {
        keys[i] = EMPTY_KEY;
        vals[i] = 0x7fffffff;
    }
    if (i < n_tri) {
        parent[i] = (int)i;
        count[i] = 0;
    }
}

__global__ void __launch_bounds__(256)
edge_insert_kernel(const int32_t *__restrict__ tri, int n_tri, int64_t slots, unsigned long long *keys, int *vals)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)n_tri * 3) return;
    const int t = (int)(i / 3), k = (int)(i % 3);
    const unsigned long long key = edge_key(tri[3 * t + k], tri[3 * t + (k + 1) % 3]);
    const unsigned long long mask = (unsigned long long)slots - 1;
    for (unsigned long long h = mix(key) & mask;; h = (h + 1) & mask) {
        const unsigned long long prev = atomicCAS(keys + h, EMPTY_KEY, key);
        if (prev == EMPTY_KEY || prev == key) {
            atomicMin(vals + h, t);
            return;
        }
    }
}

__global__ void __launch_bounds__(256)
edge_union_kernel(const int32_t *__restrict__ tri, int n_tri, int64_t slots, const unsigned long long *keys,
                  const int *vals, int *parent)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)n_tri * 3) return;
    const int t = (int)(i / 3), k = (int)(i % 3);
    const unsigned long long key = edge_key(tri[3 * t + k], tri[3 * t + (k + 1) % 3]);
    const unsigned long long mask = (unsigned long long)slots - 1;
    unsigned long long h = mix(key) & mask;
    while (keys[h] != key) h = (h + 1) & mask;
    int a = t, b = vals[h];
    while (true) {
        a = find_root(parent, a);
        b = find_root(parent, b);
        if (a == b) return;
        if (a < b) { const int x = a; a = b; b = x; }
        if (atomicCAS(parent + a, a, b) == a) return;   // link the larger root under the smaller
    }
}

__global__ void __launch_bounds__(256)
cluster_count_kernel(int n_tri, int *parent, int *count, int *is_root, int *root_of)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_tri) return;
    const int r = find_root(parent, t);
    root_of[t] = r;
    atomicAdd(count + r, 1);
    is_root[t] = r == t;
}

__global__ void __launch_bounds__(256)
cluster_label_kernel(int n_tri, const int *root_of, const int *count, const int *root_off, int32_t *label,
                     int32_t *cluster_size)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_tri) return;
    const int r = root_of[t];
    label[t] = root_off[r];
    if (r == t) cluster_size[root_off[t]] = count[t];
}

// ---- filter ----

__global__ void __launch_bounds__(256)
filter_mark_kernel(const int32_t *__restrict__ tri, int n_tri, const int32_t *__restrict__ label,
                   const int32_t *__restrict__ cluster_size, int min_size, int *vflag, int *tflag, int *toff)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_tri) return;
    const int a = tri[3 * t], b = tri[3 * t + 1], c = tri[3 * t + 2];
    const bool keep = cluster_size[label[t]] >= min_size;
    if (keep) vflag[a] = vflag[b] = vflag[c] = 1;
    const int k = keep && a != b && b != c && a != c;
    tflag[t] = k;
    toff[t] = k;
}

__global__ void __launch_bounds__(256)
copy_flags_kernel(const int *src, int *dst, int n)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = src[i];
}

__global__ void __launch_bounds__(256)
filter_vertex_kernel(const double *__restrict__ v, const double *__restrict__ c, int n_vert, const int *vflag,
                     const int *voff, double *out_v, double *out_c)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_vert || !vflag[i]) return;
    for (int k = 0; k < 3; k++) {
        out_v[(size_t)voff[i] * 3 + k] = v[(size_t)i * 3 + k];
        out_c[(size_t)voff[i] * 3 + k] = c[(size_t)i * 3 + k];
    }
}

__global__ void __launch_bounds__(256)
filter_tri_kernel(const int32_t *__restrict__ tri, int n_tri, const int *tflag, const int *toff, const int *voff,
                  int32_t *out)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_tri || !tflag[t]) return;
    for (int k = 0; k < 3; k++) out[(size_t)toff[t] * 3 + k] = voff[tri[3 * t + k]];
}

inline unsigned blocks(int64_t n) { return (unsigned)((n + 255) / 256); }

}  // namespace

extern "C" int ga_mesh_cubes_count(const float *voxels, int n_units, const int32_t *pool, const int32_t *unit_slot,
                                   const int32_t *box, const int8_t *tri_table, uint8_t *cube, int32_t *vert_off,
                                   int32_t *tri_off, void *work, int32_t *status, int32_t *status_host,
                                   void *status_event, void *stream)
{
    if (!pool || !unit_slot || !box || !tri_table || !work || !status || n_units < 0) return GA_ERR_BADARG;
    if ((status_host == nullptr) != (status_event == nullptr)) return GA_ERR_BADARG;
    if ((int64_t)n_units * 4096 > 0x7fffffff / 8) return GA_ERR_SIZE;
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t nvox = (int64_t)n_units * 4096;
    cudaError_t e;
    if (nvox > 0) {
        if (!voxels || !cube || !vert_off || !tri_off) return GA_ERR_BADARG;
        cube_case_kernel<<<blocks(nvox), 256, 0, s>>>(voxels, nvox, pool, unit_slot, box, tri_table, cube, tri_off);
        edge_flag_kernel<<<blocks(nvox), 256, 0, s>>>(voxels, nvox, pool, unit_slot, box, cube, vert_off);
        if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
    }
    int *partials = (int *)work;
    if ((e = scan_exclusive(vert_off, nvox, partials, &status[2], s)) != cudaSuccess) return (int)e;
    if ((e = scan_exclusive(tri_off, nvox, partials, &status[3], s)) != cudaSuccess) return (int)e;
    return (int)publish_status(status, status_host, status_event, s);
}

extern "C" int ga_mesh_cubes_emit(const float *voxels, int n_units, const int32_t *pool, const int32_t *unit_slot,
                                  const int32_t *box, const double *volume, const int8_t *tri_table,
                                  const uint8_t *cube, const int32_t *vert_off, const int32_t *tri_off,
                                  double *vertices, double *colors, int32_t *triangles, void *stream)
{
    if (!pool || !unit_slot || !box || !volume || !tri_table || n_units < 0) return GA_ERR_BADARG;
    if (n_units == 0) return 0;
    if (!voxels || !cube || !vert_off || !tri_off) return GA_ERR_BADARG;
    const int64_t nvox = (int64_t)n_units * 4096;
    emit_kernel<<<blocks(nvox), 256, 0, (cudaStream_t)stream>>>(voxels, nvox, pool, unit_slot, box, volume,
                                                                tri_table, cube, vert_off, tri_off, vertices,
                                                                colors, triangles);
    return (int)cudaGetLastError();
}

extern "C" int ga_mesh_clusters(const int32_t *triangles, int n_tri, void *hash, int64_t hash_slots, int32_t *label,
                                int32_t *cluster_size, void *work, int32_t *status, int32_t *status_host,
                                void *status_event, void *stream)
{
    if (n_tri < 0 || !work || !status) return GA_ERR_BADARG;
    if ((status_host == nullptr) != (status_event == nullptr)) return GA_ERR_BADARG;
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e;
    if (n_tri > 0) {
        if (!triangles || !hash || !label || !cluster_size) return GA_ERR_BADARG;
        if (hash_slots < 6 * (int64_t)n_tri || (hash_slots & (hash_slots - 1))) return GA_ERR_WORKSPACE;
        unsigned long long *keys = (unsigned long long *)hash;
        int *vals = (int *)(keys + hash_slots);
        int *parent = label;                                     // the forest; overwritten by the labels at the end
        int *count = (int *)work, *root = count + n_tri, *root_of = root + n_tri, *partials = root_of + n_tri;
        cluster_init_kernel<<<blocks(hash_slots), 256, 0, s>>>(n_tri, hash_slots, keys, vals, parent, count);
        edge_insert_kernel<<<blocks((int64_t)n_tri * 3), 256, 0, s>>>(triangles, n_tri, hash_slots, keys, vals);
        edge_union_kernel<<<blocks((int64_t)n_tri * 3), 256, 0, s>>>(triangles, n_tri, hash_slots, keys, vals, parent);
        cluster_count_kernel<<<blocks(n_tri), 256, 0, s>>>(n_tri, parent, count, root, root_of);
        if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
        if ((e = scan_exclusive(root, n_tri, partials, &status[4], s)) != cudaSuccess) return (int)e;
        cluster_label_kernel<<<blocks(n_tri), 256, 0, s>>>(n_tri, root_of, count, root, label, cluster_size);
        if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
    } else if ((e = cudaMemsetAsync(&status[4], 0, sizeof(int32_t), s)) != cudaSuccess) {
        return (int)e;
    }
    return (int)publish_status(status, status_host, status_event, s);
}

extern "C" int ga_mesh_filter(const double *vertices, const double *colors, int n_vert, const int32_t *triangles,
                              int n_tri, const int32_t *label, const int32_t *cluster_size, int min_size,
                              double *out_vertices, double *out_colors, int32_t *out_triangles, void *work,
                              int32_t *status, int32_t *status_host, void *status_event, void *stream)
{
    if (n_vert < 0 || n_tri < 0 || !work || !status) return GA_ERR_BADARG;
    if ((status_host == nullptr) != (status_event == nullptr)) return GA_ERR_BADARG;
    if (n_tri > 0 && (!triangles || !label || !cluster_size || !out_triangles)) return GA_ERR_BADARG;
    if (n_vert > 0 && (!vertices || !colors || !out_vertices || !out_colors)) return GA_ERR_BADARG;
    cudaStream_t s = (cudaStream_t)stream;
    int *vflag = (int *)work, *tflag = vflag + n_vert, *voff = tflag + n_tri, *toff = voff + n_vert;
    int *partials = toff + n_tri;
    cudaError_t e;
    if ((e = cudaMemsetAsync(vflag, 0, (size_t)n_vert * sizeof(int), s)) != cudaSuccess) return (int)e;
    if (n_tri > 0)
        filter_mark_kernel<<<blocks(n_tri), 256, 0, s>>>(triangles, n_tri, label, cluster_size, min_size, vflag, tflag,
                                                         toff);
    if (n_vert > 0) copy_flags_kernel<<<blocks(n_vert), 256, 0, s>>>(vflag, voff, n_vert);
    if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
    if ((e = scan_exclusive(voff, n_vert, partials, &status[5], s)) != cudaSuccess) return (int)e;
    if ((e = scan_exclusive(toff, n_tri, partials, &status[6], s)) != cudaSuccess) return (int)e;
    if (n_vert > 0)
        filter_vertex_kernel<<<blocks(n_vert), 256, 0, s>>>(vertices, colors, n_vert, vflag, voff, out_vertices,
                                                            out_colors);
    if (n_tri > 0)
        filter_tri_kernel<<<blocks(n_tri), 256, 0, s>>>(triangles, n_tri, tflag, toff, voff, out_triangles);
    if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
    return (int)publish_status(status, status_host, status_event, s);
}
