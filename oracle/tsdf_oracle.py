"""numpy oracle of the GPU mesh export (gaussiananything_b200/mesh.py, csrc/mesh_tsdf.cu, csrc/mesh_extract.cu).

PARITY UNPINNED.  It restates Open3D 0.17's legacy ScalableTSDFVolume / TriangleMesh code as
FlowMatchingEngine.extract_mesh_bounded and utils/mesh_util.post_process_mesh call it.  Open3D is not vendored and
cannot be run here, so these points are written from memory of upstream and could not be checked against it:
  - depth >= depth_trunc becomes 0, compared in fp64 (ConvertDepthToFloatImage);
  - touched units: every 4th pixel in x and y with d > 0, unprojected in fp64 with inverse(extrinsic), and every unit
    in floor((p +- sdf_trunc) / unit_length) is touched, per view; a view integrates only the units it touched;
  - integration order and rounding: voxel centre (0.5f vl + vl x) + float(origin); p_cam = ((E0 X + E1 Y) + E2 Z) + E3
    per row, evaluated for every voxel (Open3D steps along z by adding the scaled third column instead; this form is
    the one restated here); u = ((px fx) / pz + cx) + 0.5f; the window 0.0001f <= u < W - 0.0001f;
    mult = sqrtf((xx^2 + yy^2) + 1) with xx = (u - cx) (1/fx); sdf = (d - pz) mult; tsdf = min(1, sdf (1/sdf_trunc));
    T = (T w + tsdf) / (w + 1), C likewise, w += 1;
  - marching cubes: a missing unit or a zero weight skips the cube; bit k when tsdf_k < 0; vertex
    0.5 vl + vl e, + f0 vl / (f0 + f1) along the edge, colour (f1 c0 + f0 c1) / (f0 + f1), c = C / 255, in fp64;
  - cluster_connected_triangles connects triangles through shared edges.
The triangle table is gaussiananything_b200/mc_table.py (generated, not the classic table; it is data both sides
read).  Clustering uses scipy's connected_components on the triangle-edge graph, not a union-find.  Vertex order:
pool order (units by box index), then voxel order, then x, y, z edge.
"""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

from gaussiananything_b200.mc_table import EDGE_AXIS, EDGE_ORIGIN, TRI_COUNT, TRI_TABLE

f32 = np.float32
UNIT = 16


def prepare(rgb, depth, alpha, depth_trunc, alpha_thres=0.08):
    """rgb [V,3,H,W], depth / alpha [V,H,W] fp32 -> (depth fp32 [V,H,W] with 0 where invalid, rgb8 uint8 [V,H,W,3])."""
    d = depth.astype(f32).copy()
    d[alpha < f32(alpha_thres)] = 0
    d[d.astype(np.float64) >= np.asarray(depth_trunc)[:, None, None]] = 0
    c = (np.clip(rgb, f32(0), f32(1)) * f32(255)).astype(f32).astype(np.uint8)
    return d, np.ascontiguousarray(c.transpose(0, 2, 3, 1))


def texels(depth, rgb8):
    """The packed layout of ga_mesh_prepare: int32 [V,H,W,2] = depth bits | r | g << 8 | b << 16."""
    c = rgb8.astype(np.uint32)
    word = c[..., 0] | (c[..., 1] << 8) | (c[..., 2] << 16)
    return np.stack([depth.view(np.int32), word.view(np.int32)], -1)


def touch(depth, setup):
    """bool [V, nx*ny*nz]: units each view touches; raises when a unit leaves the box."""
    box = setup["box"].astype(np.int64)
    V, H, W = depth.shape
    st, ul = setup["sdf_trunc"], setup["voxel_length"] * UNIT
    out = np.zeros((V, int(np.prod(box[3:]))), bool)
    ii, jj = np.meshgrid(np.arange(0, H, 4), np.arange(0, W, 4), indexing="ij")
    for v in range(V):
        M = setup["cams_d"][v]
        d = depth[v, ii, jj]
        ok = d > 0
        z = d[ok].astype(np.float64)
        x = (jj[ok].astype(np.float64) - M[18]) * z / M[16]
        y = (ii[ok].astype(np.float64) - M[19]) * z / M[17]
        lo, n = [], []
        for r in range(3):
            p = M[4 * r] * x + M[4 * r + 1] * y + M[4 * r + 2] * z + M[4 * r + 3]
            a, b = np.floor((p - st) / ul), np.floor((p + st) / ul)
            if (a < box[r]).any() or (b >= box[r] + box[3 + r]).any():
                raise RuntimeError("a depth point lies outside the volume box")
            lo.append(a.astype(np.int64) - box[r])
            n.append((b - a).astype(np.int64) + 1)
        for da in range(int(max(n[0].max(initial=0), 0))):
            for db in range(int(max(n[1].max(initial=0), 0))):
                for dc in range(int(max(n[2].max(initial=0), 0))):
                    m = (da < n[0]) & (db < n[1]) & (dc < n[2])
                    u = ((lo[0][m] + da) * box[4] + lo[1][m] + db) * box[5] + lo[2][m] + dc
                    out[v, u] = True
    return out


def integrate(depth, rgb8, setup, touched):
    """(pool int64 [Nu] box indices, state fp32 [5, Nu*4096] = tsdf | weight | r | g | b)."""
    box = setup["box"].astype(np.int64)
    V, H, W = depth.shape
    pool = np.flatnonzero(touched.any(0))
    Nu = len(pool)
    state = np.zeros((5, Nu, 4096), f32)
    vl = setup["voxel_length"]
    vl_f, st_f = f32(vl), f32(setup["sdf_trunc"])
    half_f, inv_st = vl_f * f32(0.5), f32(1) / st_f
    ny, nz = box[4], box[5]
    g = np.stack([box[0] + pool // (ny * nz), box[1] + (pool // nz) % ny, box[2] + pool % nz], 1)
    org = (g.astype(np.float64) * (vl * UNIT)).astype(f32)                       # [Nu, 3]
    lin = np.arange(4096)
    loc = np.stack([lin >> 8, (lin >> 4) & 15, lin & 15], 1).astype(f32)       # [4096, 3]
    P = [(half_f + vl_f * loc[None, :, a]) + org[:, a:a + 1] for a in range(3)]  # each [Nu, 4096]
    Wf, Hf = f32(W) - f32(0.0001), f32(H) - f32(0.0001)
    for v in range(V):
        sel = np.flatnonzero(touched[v, pool])
        if len(sel) == 0:
            continue
        E = setup["cams_f"][v]
        X, Y, Z = P[0][sel], P[1][sel], P[2][sel]
        row = [E[4 * r] * X + E[4 * r + 1] * Y + E[4 * r + 2] * Z + E[4 * r + 3] for r in range(3)]
        px, py, pz = row
        fx, fy, cx, cy = E[16], E[17], E[18], E[19]
        with np.errstate(divide="ignore", invalid="ignore"):
            uf = px * fx / pz + cx + f32(0.5)
            vf = py * fy / pz + cy + f32(0.5)
        ok = (pz > 0) & (uf >= f32(0.0001)) & (uf < Wf) & (vf >= f32(0.0001)) & (vf < Hf)
        iu = np.where(ok, uf, 0).astype(np.int64)
        iv = np.where(ok, vf, 0).astype(np.int64)
        d = depth[v][iv, iu]
        ok &= d > 0
        xx = (iu.astype(f32) - cx) * (f32(1) / fx)
        yy = (iv.astype(f32) - cy) * (f32(1) / fy)
        sdf = (d - pz) * np.sqrt(xx * xx + yy * yy + f32(1))
        ok &= sdf > -st_f
        tsdf = np.minimum(f32(1), sdf * inv_st)
        s = state[:, sel]
        w = s[1]
        w1 = w + f32(1)
        col = rgb8[v][iv, iu].astype(f32)
        new = [(s[0] * w + tsdf) / w1, w1] + [(s[2 + k] * w + col[..., k]) / w1 for k in range(3)]
        for k in range(5):
            s[k] = np.where(ok, new[k], s[k])
        state[:, sel] = s
    return pool, state.reshape(5, Nu * 4096)


def _padded(pool, state, box):
    """tsdf / weight / rgb of every pooled unit with a one-voxel border from its 26 neighbours: [Nu, 18, 18, 18]
    arrays for local coordinates -1..16 (weight 0 where the neighbour unit is missing)."""
    Nu = len(pool)
    slot = -np.ones(int(np.prod(box[3:])), np.int64)
    slot[pool] = np.arange(Nu)
    ny, nz = box[4], box[5]
    uc = np.stack([pool // (ny * nz), (pool // nz) % ny, pool % nz], 1)
    s = state.reshape(5, Nu, 16, 16, 16)
    out = np.zeros((5, Nu, 18, 18, 18), f32)
    rng = {-1: (slice(15, 16), slice(0, 1)), 0: (slice(0, 16), slice(1, 17)), 1: (slice(0, 1), slice(17, 18))}
    for dx in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dz in (-1, 0, 1):
                n = uc + np.array([dx, dy, dz])
                ok = ((n >= 0) & (n < box[3:])).all(1)
                nb = np.full(Nu, -1)
                nb[ok] = slot[(n[ok, 0] * ny + n[ok, 1]) * nz + n[ok, 2]]
                has = nb >= 0
                (sx, tx), (sy, ty), (sz, tz) = rng[dx], rng[dy], rng[dz]
                out[:, has, tx, ty, tz] = s[:, nb[has]][:, :, sx, sy, sz]
    return out


def marching_cubes(pool, state, setup):
    """(vertices fp64 [Nv,3], colours fp64 [Nv,3], triangles int32 [Nt,3], cube uint8 [Nu*4096], edge key int64 [Nv])."""
    box = setup["box"].astype(np.int64)
    vl = setup["voxel_length"]
    Nu = len(pool)
    if Nu == 0:
        z = np.zeros((0, 3))
        return z, z, np.zeros((0, 3), np.int32), np.zeros(0, np.uint8), np.zeros(0, np.int64)
    P = _padded(pool, state, box)
    T, Wt = P[0], P[1]
    # cube case for cube origins at local -1..15 (index 0..16 of the padded arrays)
    cube = np.zeros((Nu, 17, 17, 17), np.int64)
    valid = np.ones((Nu, 17, 17, 17), bool)
    for k, (cx, cy, cz) in enumerate(((0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1))):
        t = T[:, cx:cx + 17, cy:cy + 17, cz:cz + 17]
        valid &= Wt[:, cx:cx + 17, cy:cy + 17, cz:cz + 17] != 0
        cube |= (t < 0).astype(np.int64) << k
    cube[~valid] = 0
    own_cube = cube[:, 1:, 1:, 1:].reshape(Nu, 4096)
    # vertex flags of each voxel's +x, +y, +z edges
    t0, w0 = T[:, 1:17, 1:17, 1:17], Wt[:, 1:17, 1:17, 1:17]
    flags = np.zeros((Nu, 16, 16, 16), np.int64)
    for a in range(3):
        sl = [slice(1, 17)] * 3
        sl[a] = slice(2, 18)
        t1, w1 = T[(slice(None),) + tuple(sl)], Wt[(slice(None),) + tuple(sl)]
        change = (w0 != 0) & (w1 != 0) & ((t0 < 0) != (t1 < 0))
        b, c = (a + 1) % 3, (a + 2) % 3
        anyc = np.zeros_like(change)
        for k in range(4):
            o = [1, 1, 1]
            o[b] -= k & 1
            o[c] -= k >> 1
            cc = cube[:, o[0]:o[0] + 16, o[1]:o[1] + 16, o[2]:o[2] + 16]
            anyc |= (cc != 0) & (cc != 255)
        flags |= (change & anyc).astype(np.int64) << a
    flags = flags.reshape(Nu, 4096)
    ny, nz = box[4], box[5]
    uc = np.stack([pool // (ny * nz), (pool // nz) % ny, pool % nz], 1)
    lin = np.arange(4096)
    loc = np.stack([lin >> 8, (lin >> 4) & 15, lin & 15], 1)
    gv = uc[:, None, :] * 16 + loc[None]                                # box-relative voxel coords [Nu, 4096, 3]
    NX, NY, NZ = box[3] * 16, box[4] * 16, box[5] * 16
    tsd = state[0].reshape(Nu, 4096)
    rgb = state[2:].reshape(3, Nu, 4096)
    verts, cols, keys = [], [], []
    # emission order: unit, voxel, axis -> sort by (unit, voxel, axis)
    for a in range(3):
        u_i, l_i = np.nonzero((flags >> a) & 1)
        p = gv[u_i, l_i]
        q = p.copy()
        q[:, a] += 1
        qu, ql = q // 16, q % 16
        qs = np.searchsorted(pool, (qu[:, 0] * ny + qu[:, 1]) * nz + qu[:, 2])
        qi = (ql[:, 0] * 16 + ql[:, 1]) * 16 + ql[:, 2]
        f0 = np.abs(tsd[u_i, l_i].astype(np.float64))
        f1 = np.abs(tsd[qs, qi].astype(np.float64))
        pt = 0.5 * vl + vl * (p + box[:3] * 16).astype(np.float64)
        pt[:, a] += f0 * vl / (f0 + f1)
        c0 = rgb[:, u_i, l_i].T.astype(np.float64) / 255.0
        c1 = rgb[:, qs, qi].T.astype(np.float64) / 255.0
        col = (f1[:, None] * c0 + f0[:, None] * c1) / (f0 + f1)[:, None]
        order_key = (u_i * 4096 + l_i) * 3 + a
        verts.append(pt)
        cols.append(col)
        keys.append(np.stack([order_key, ((p[:, 0] * NY + p[:, 1]) * NZ + p[:, 2]) * 3 + a], 1))
    verts, cols, keys = np.concatenate(verts), np.concatenate(cols), np.concatenate(keys)
    o = np.argsort(keys[:, 0], kind="stable")
    verts, cols, ekey = verts[o], cols[o], keys[o, 1]
    ek_sorted = np.argsort(ekey)
    # triangles: unit, voxel, table order
    cu = own_cube.reshape(-1)
    cnt = TRI_COUNT[cu].astype(np.int64)
    vox = np.repeat(np.arange(Nu * 4096), cnt)
    first = np.repeat(np.cumsum(cnt) - cnt, cnt)
    t_in = np.arange(len(vox)) - first
    tris = np.zeros((len(vox), 3), np.int64)
    for k in range(3):
        ei = TRI_TABLE[cu[vox], 3 * t_in + k].astype(np.int64)
        org = np.asarray(EDGE_ORIGIN)[ei]
        ax = np.asarray(EDGE_AXIS)[ei]
        p = gv.reshape(-1, 3)[vox] + org
        key = ((p[:, 0] * NY + p[:, 1]) * NZ + p[:, 2]) * 3 + ax
        pos = np.searchsorted(ekey, key, sorter=ek_sorted)
        tris[:, k] = ek_sorted[pos]
        assert (ekey[tris[:, k]] == key).all()
    return verts, cols, tris.astype(np.int32), own_cube.reshape(-1).astype(np.uint8), ekey


def fuse(rgb, depth, alpha, setup, alpha_thres=0.08):
    """The whole fusion: dict of every stage's result."""
    d, c8 = prepare(rgb, depth, alpha, setup["depth_trunc"], alpha_thres)
    touched = touch(d, setup)
    pool, state = integrate(d, c8, setup, touched)
    v, c, t, cube, ekey = marching_cubes(pool, state, setup)
    return dict(depth=d, rgb8=c8, touched=touched, pool=pool, state=state, vertices=v, colors=c, triangles=t,
                cube=cube, edge_key=ekey)


def clusters(triangles):
    """(label [Nt], sizes [n]) of triangles connected through shared edges; clusters numbered by smallest triangle."""
    t = np.asarray(triangles, np.int64).reshape(-1, 3)
    nt = len(t)
    if nt == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    e = np.stack([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]], 1).reshape(-1, 2)
    e.sort(1)
    _, eid = np.unique(e, axis=0, return_inverse=True)
    eid = eid.reshape(-1)
    ne = eid.max() + 1
    rows = np.repeat(np.arange(nt), 3)
    g = coo_matrix((np.ones(len(rows)), (rows, nt + eid)), shape=(nt + ne, nt + ne))
    _, lab = connected_components(g, directed=False)
    lab = lab[:nt]
    first = np.full(lab.max() + 1, nt)
    np.minimum.at(first, lab, np.arange(nt))
    order = np.argsort(first)
    rank = np.empty_like(order)
    rank[order] = np.arange(len(order))
    label = rank[lab]
    return label, np.bincount(label)


def post_process(vertices, colors, triangles):
    """utils/mesh_util.post_process_mesh -> (vertices, colours, triangles, label, sizes, threshold)."""
    t = np.asarray(triangles, np.int64).reshape(-1, 3)
    if len(t) == 0:
        return vertices[:0], colors[:0], t.astype(np.int32), np.zeros(0, np.int64), np.zeros(0, np.int64), None
    label, sizes = clusters(t)
    k = min(len(sizes), 10)
    n = max(int(np.sort(sizes)[-k]), 50)
    keep = sizes[label] >= n
    t = t[keep]
    used = np.zeros(len(vertices), bool)
    used[t.reshape(-1)] = True
    remap = np.cumsum(used) - 1
    t = remap[t]
    t = t[(t[:, 0] != t[:, 1]) & (t[:, 1] != t[:, 2]) & (t[:, 0] != t[:, 2])]
    return vertices[used], colors[used], t.astype(np.int32), label, sizes, n
