"""Scenes of the mesh-export tests: an analytic sphere rendered in numpy (independent of the rasteriser and of both
fusion implementations), surfels laid on a sphere and a torus for the batched renderer, and mesh checks."""
import numpy as np

SPHERE_R = 0.3


def sphere_maps(cam_pathes, size, r=SPHERE_R, colour=0.5):
    """rgb [V,3,H,W], depth [V,H,W] (camera z of the hit, 0 on a miss), alpha [V,H,W] of a sphere at the origin, from
    the pixel-centre ray of each pixel: direction ((j - cx) / fx, (i - cy) / fy, 1) in camera space with
    fx = (W/2) / tan(fov/2) and cx = (W - 1) / 2."""
    from tools.synth import camera_from_pose25
    V, H, W = len(cam_pathes), size, size
    rgb = np.full((V, 3, H, W), colour, np.float32)
    depth = np.zeros((V, H, W), np.float32)
    alpha = np.zeros((V, H, W), np.float32)
    ii, jj = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    for v, pose in enumerate(cam_pathes):
        world_view, _, _, tanfov = camera_from_pose25(pose)
        w2c = world_view.T.astype(np.float64)
        c2w = np.linalg.inv(w2c)
        f = (W / 2) / tanfov
        d_cam = np.stack([(jj - (W - 1) / 2) / f, (ii - (H - 1) / 2) / f, np.ones_like(ii)], -1)
        d = d_cam @ c2w[:3, :3].T
        o = c2w[:3, 3]
        a = (d * d).sum(-1)
        b = 2 * (d @ o)
        c = o @ o - r * r
        disc = b * b - 4 * a * c
        hit = disc > 0
        t = (-b - np.sqrt(np.where(hit, disc, 0))) / (2 * a)
        depth[v] = np.where(hit, t, 0)
        alpha[v] = hit
    return rgb, depth, alpha


def surface_surfels(P=73728, seed=0):
    """[P,13] opaque surfels tangent to a sphere (r 0.22, centre (-0.12,0,0)) and a torus (R 0.2, r 0.07, centre
    (0.17,0,0)), sized to cover them; colours vary smoothly with position."""
    rng = np.random.default_rng(seed)
    n1 = P // 2
    n2 = P - n1
    u = rng.normal(size=(n1, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    c1 = np.array([-0.12, 0.0, 0.0])
    p1, nrm1 = c1 + 0.22 * u, u
    th, ph = rng.uniform(0, 2 * np.pi, n2), rng.uniform(0, 2 * np.pi, n2)
    c2 = np.array([0.17, 0.0, 0.0])
    ring = np.stack([np.cos(th), np.sin(th), np.zeros(n2)], 1)
    nrm2 = np.cos(ph)[:, None] * ring + np.sin(ph)[:, None] * np.array([0, 0, 1.0])
    p2 = c2 + 0.2 * ring + 0.07 * nrm2
    xyz = np.concatenate([p1, p2])
    n = np.concatenate([nrm1, nrm2])
    # quaternion (w, x, y, z) rotating +z onto the normal: the surfel's tangent plane is its local xy plane
    z = np.array([0, 0, 1.0])
    axis = np.cross(z, n)
    s = np.linalg.norm(axis, axis=1)
    cosang = n[:, 2]
    ang = np.arctan2(s, cosang)
    axis = np.where(s[:, None] > 1e-9, axis / np.maximum(s, 1e-12)[:, None], np.array([1.0, 0, 0]))
    q = np.concatenate([np.cos(ang / 2)[:, None], axis * np.sin(ang / 2)[:, None]], 1)
    scale = np.full((P, 2), 0.006)
    rgb = 0.5 + 0.4 * np.sin(3 * xyz + np.array([0, 2, 4]))
    op = np.full((P, 1), 0.99)
    return np.concatenate([xyz, op, scale, q, rgb], 1).astype(np.float32)


def edge_use(triangles):
    """{(a, b): number of triangles using the undirected edge}."""
    t = np.asarray(triangles, np.int64)
    e = np.sort(np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]]), 1)
    keys, counts = np.unique(e, axis=0, return_counts=True)
    return keys, counts


def check_sphere_mesh(vertices, triangles, colors, voxel_length, r=SPHERE_R, within_half=0.99):
    """The known answer of the sphere: closed, `within_half` of the vertices within half a voxel of it and all within
    1.5, positive volume of 4/3 pi r^3 (3 %), colour 127/255."""
    v, t = np.asarray(vertices), np.asarray(triangles, np.int64)
    assert len(t) > 0
    keys, counts = edge_use(t)
    assert (counts == 2).all(), np.bincount(counts)
    assert len(v) - len(keys) + len(t) == 2
    dist = np.abs(np.linalg.norm(v, axis=1) - r) / voxel_length
    assert (dist <= 0.5).mean() >= within_half, (dist <= 0.5).mean()
    assert dist.max() <= 1.5, dist.max()
    a, b, c = v[t[:, 0]], v[t[:, 1]], v[t[:, 2]]
    vol = np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6
    want = 4 / 3 * np.pi * r ** 3
    assert vol > 0 and abs(vol - want) <= 0.03 * want, (vol, want)
    assert np.abs(np.asarray(colors) - 127 / 255).max() <= 1e-12


def strip(n_tri, offset):
    """A strip of n_tri triangles connected through edges, vertex ids from offset."""
    return np.array([[offset + k, offset + k + 1, offset + k + 2] for k in range(n_tri)], np.int64)


def mesh_arrays(tris, n_vert=None):
    """(vertices, colours, triangles) of a hand-built triangle list; vertex i at (3i, 3i+1, 3i+2)."""
    tris = np.asarray(tris, np.int64).reshape(-1, 3)
    nv = n_vert if n_vert is not None else (int(tris.max()) + 1 if len(tris) else 0)
    v = np.arange(nv * 3, dtype=np.float64).reshape(nv, 3)
    return v, v / max(nv * 3, 1), tris


def _strips(sizes, gap=2):
    out, off = [], 0
    for s in sizes:
        out.append(strip(s, off))
        off += s + gap
    return np.concatenate(out)


def post_process_cases():
    """{name: (vertices, colours, triangles)} of hand-built meshes for the floater filter."""
    ten_largest = _strips([60, 70, 80, 90, 100, 110, 120, 130, 140, 150, 55, 52, 40])
    degenerate = strip(60, 0)
    degenerate = np.concatenate([degenerate, [[5, 5, 6], [7, 8, 8]]])   # repeated index, connected to the strip
    return {
        "ten_largest": mesh_arrays(ten_largest),
        "ties": mesh_arrays(_strips([70] * 12)),
        "few_clusters": mesh_arrays(_strips([60, 80], gap=40)),
        "bow_ties": mesh_arrays(np.concatenate([strip(60, 0), [[70, 71, 72], [72, 73, 74]]])),
        "vertex_order": mesh_arrays(np.concatenate([strip(60, 0)[:, ::-1] + 3, strip(5, 100)])),
        "degenerate": mesh_arrays(degenerate),
    }


def dense_marching_cubes(neg, tri_table, tri_count, corners, edge_origin, edge_axis):
    """Triangles (vertex = global grid edge key) of a dense sign field neg [N,N,N] (True where tsdf < 0)."""
    N = neg.shape[0]
    o = np.stack(np.meshgrid(*[np.arange(N - 1)] * 3, indexing="ij"), -1).reshape(-1, 3)
    case = np.zeros(len(o), np.int64)
    for k, c in enumerate(corners):
        p = o + c
        case |= neg[p[:, 0], p[:, 1], p[:, 2]].astype(np.int64) << k
    cnt = np.asarray(tri_count, np.int64)[case]
    cube = np.repeat(np.arange(len(o)), cnt)
    t_in = np.arange(len(cube)) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    tris = np.zeros((len(cube), 3), np.int64)
    for k in range(3):
        e = np.asarray(tri_table)[case[cube], 3 * t_in + k].astype(np.int64)
        q = o[cube] + np.asarray(edge_origin)[e]
        tris[:, k] = ((q[:, 0] * N + q[:, 1]) * N + q[:, 2]) * 3 + np.asarray(edge_axis)[e]
    return tris


def check_closed_oriented(tris):
    """Every edge used by exactly two triangles, once in each direction; no triangle twice; none degenerate."""
    t = np.asarray(tris, np.int64)
    d = np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]])
    _, dcount = np.unique(d, axis=0, return_counts=True)
    assert (dcount == 1).all(), "a directed edge is used twice"
    _, ucount = np.unique(np.sort(d, 1), axis=0, return_counts=True)
    assert (ucount == 2).all(), np.bincount(ucount)
    assert len(np.unique(np.sort(t, 1), axis=0)) == len(t), "duplicate triangle"
    assert ((t[:, 0] != t[:, 1]) & (t[:, 1] != t[:, 2]) & (t[:, 0] != t[:, 2])).all()
