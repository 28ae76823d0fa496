"""TSDF mesh export on the GPU: the third output of the reference's image-to-3D demo.

Mirrors FlowMatchingEngine.export_mesh_from_2dgs / extract_mesh_bounded (nsr/lsgm/flow_matching_trainer.py:1244-1395),
utils/mesh_util.post_process_mesh (:22-44) and nsr/camera_utils.uni_mesh_path (:233-264).  The reference fuses the
rendered views into Open3D's ScalableTSDFVolume on the CPU, one view at a time; here prepare, touch, integrate,
marching cubes and the floater filter are CUDA kernels of libga_b200.so (include/ga_b200.h Part 4) working on the
device maps the batched renderer produced.  Only counts (and the cluster sizes the keep rule is applied to) come back
to the host before the mesh itself.

Deviations from the reference, all documented in INTEGRATION.md: the marching-cubes triangle table is generated
(gaussiananything_b200/mc_table.py), vertex order is pool order then voxel order (Open3D's follows its hash map), an
empty mesh is returned empty instead of raising, and the caller's depth maps are not modified.
"""
import ctypes as C
import math
import os

import numpy as np
import torch

from . import _lib
from ._launch import ptr, stream
from .mc_table import TRI_TABLE

AABB = np.array([-0.45, -0.45, -0.45, 0.45, 0.45, 0.45]).reshape(2, 3) * 1.1
ALPHA_THRES = 0.08
UNIT = 16
STATUS_INTS = 8


def volume_settings():
    """(center, radius, voxel_length, sdf_trunc) of extract_mesh_bounded (:1338-1342), whatever its arguments say."""
    center = AABB.mean(0)
    radius = np.linalg.norm(AABB[1] - AABB[0]) * 0.5
    voxel_length = radius / 160
    return center, radius, voxel_length, voxel_length * 12


def uni_mesh_path(frame_number=10, radius=1.8):
    """nsr/camera_utils.uni_mesh_path: elevations 60, 30, 0, -30, -60 x `frame_number` azimuths, look-at-origin
    cameras at `radius` (generate_input_camera, fp32 torch), K = normalised fx 1.3889.  Returns [5 * frame_number, 25]
    float32 (c2w row-major | K)."""
    el, az = [], []
    for e in (60, 30, 0, -30, -60):
        for i in range(frame_number):
            el.append(e)
            az.append(i / frame_number * 360)
    poses = torch.tensor(np.deg2rad(np.stack([el, az], 1))).float()
    pitch, yaw = poses[:, 0], poses[:, 1]
    z = radius * torch.sin(pitch)
    x = radius * torch.cos(pitch) * torch.cos(yaw)
    y = radius * torch.cos(pitch) * torch.sin(yaw)
    cam_pos = torch.stack([x, y, z], dim=-1)

    def normalize(v):
        return v / torch.norm(v, dim=-1, keepdim=True)
    forward = normalize(-cam_pos)
    up = torch.tensor([0, 0, -1], dtype=torch.float).expand_as(forward)
    left = normalize(torch.cross(up, forward, dim=-1))
    up = normalize(torch.cross(forward, left, dim=-1))
    n = forward.shape[0]
    rot = torch.eye(4).unsqueeze(0).repeat(n, 1, 1)
    rot[:, :3, :3] = torch.stack((left, up, forward), dim=-1)
    trans = torch.eye(4).unsqueeze(0).repeat(n, 1, 1)
    trans[:, :3, 3] = cam_pos
    c2w = trans @ rot
    K = torch.tensor([1.3889, 0.0, 0.5, 0.0, 1.3889, 0.5, 0.0, 0.0, 0.0039])
    return torch.cat([c2w.reshape(n, -1), K.unsqueeze(0).repeat(n, 1)], dim=-1).numpy()


def view_setup(cam_pathes, H, W):
    """Host-side camera data of every view, shared by the kernels and oracle/tsdf_oracle.py.

    Per view: the extrinsic world_view_transform.T (fp32 w2c), fx = fy = fp32((W/2) P00) and cx = cy = (W-1)/2 of
    utils/mesh_util.to_cam_open3d_compat, its inverse in fp64, depth_trunc = |campos - center| + radius, and the box
    of volume units every point can touch (each frustum out to depth_trunc, widened by sdf_trunc, plus one unit)."""
    from tools.synth import camera_from_pose25
    center, radius, vl, st = volume_settings()
    ul = vl * UNIT
    V = len(cam_pathes)
    cams_f = np.zeros((V, 20), np.float32)
    cams_d = np.zeros((V, 20), np.float64)
    trunc = np.zeros(V, np.float64)
    lo, hi = np.full(3, np.inf), np.full(3, -np.inf)
    for v, pose in enumerate(cam_pathes):
        world_view, _, cam_pos, tanfov = camera_from_pose25(np.asarray(pose, np.float32))
        p00 = np.float32(2.0 * 0.01 / (2 * (tanfov * 0.01)))          # getProjectionMatrix P[0,0], znear 0.01
        fx = np.float32(np.float32(W / 2) * p00)
        fy = np.float32(np.float32(H / 2) * p00)
        cx, cy = (W - 1) / 2, (H - 1) / 2
        ext = world_view.T.astype(np.float32)
        c2w = np.linalg.inv(ext.astype(np.float64))
        cams_f[v, :16] = ext.reshape(-1)
        cams_f[v, 16:] = (fx, fy, cx, cy)
        cams_d[v, :16] = c2w.reshape(-1)
        cams_d[v, 16:] = (float(fx), float(fy), cx, cy)
        trunc[v] = np.linalg.norm(cam_pos - center, axis=-1) + radius
        far = [c2w @ np.array([sx * cx * trunc[v] / float(fx), sy * cy * trunc[v] / float(fy), trunc[v], 1.0])
               for sx in (-1, 1) for sy in (-1, 1)]
        pts = np.stack([c2w[:3, 3]] + [f[:3] for f in far])
        lo, hi = np.minimum(lo, pts.min(0)), np.maximum(hi, pts.max(0))
    b0 = np.floor((lo - st) / ul).astype(np.int64) - 1
    b1 = np.floor((hi + st) / ul).astype(np.int64) + 1
    box = np.concatenate([b0, b1 - b0 + 1]).astype(np.int32)
    return dict(cams_f=cams_f, cams_d=cams_d, depth_trunc=trunc, box=box, voxel_length=vl, sdf_trunc=st, H=H, W=W)


class TriangleMesh:
    """Triangle mesh with Open3D's attribute names.  The arrays may live on the GPU; `vertices`, `triangles` and
    `vertex_colors` return host numpy arrays (fp64 [Nv,3], int32 [Nt,3], fp64 [Nv,3]), copied once."""

    def __init__(self, vertices, triangles, vertex_colors):
        self._v = torch.as_tensor(vertices, dtype=torch.float64)
        self._t = torch.as_tensor(triangles, dtype=torch.int32)
        self._c = torch.as_tensor(vertex_colors, dtype=torch.float64)
        self._host = {}

    def _np(self, name, t):
        if name not in self._host:
            self._host[name] = t.cpu().numpy()
        return self._host[name]

    @property
    def vertices(self):
        return self._np("v", self._v)

    @vertices.setter
    def vertices(self, value):
        self._v = torch.as_tensor(np.asarray(value, np.float64), device=self._v.device)
        self._host.pop("v", None)

    @property
    def triangles(self):
        return self._np("t", self._t)

    @property
    def vertex_colors(self):
        return self._np("c", self._c)

    def tensors(self):
        """(vertices, triangles, vertex_colors) as torch tensors where they live."""
        return self._v, self._t, self._c


def _check_cuda(x, name, dtype, dev=None):
    if not isinstance(x, torch.Tensor) or not x.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor (no CPU fallback)" % name)
    if x.dtype != dtype:
        raise TypeError("%s must be %s, got %s" % (name, dtype, x.dtype))
    if dev is not None and x.device != dev:
        raise ValueError("%s is on %s, expected %s" % (name, x.device, dev))
    return x


class _Status:
    """Pinned status words + event of one call sequence."""

    def __init__(self, dev):
        self.dev_words = torch.zeros(STATUS_INTS, dtype=torch.int32, device=dev)
        self.host = torch.zeros(STATUS_INTS, dtype=torch.int32).pin_memory()
        self.event = torch.cuda.Event()
        self.event.record(torch.cuda.current_stream(dev))

    def args(self):
        return ptr(self.dev_words), C.c_void_p(self.host.data_ptr()), C.c_void_p(self.event.cuda_event)

    def read(self):
        self.event.synchronize()
        return [int(x) for x in self.host]


def _work(n, dev):
    return torch.empty(max(int(_lib.lib().ga_mesh_work_bytes(int(n))), 4), dtype=torch.uint8, device=dev)


def fuse(rgb, depth, alpha, setup, alpha_thres=ALPHA_THRES, stages=None):
    """TSDF fusion + marching cubes of stacked device maps rgb [V,3,H,W], depth / alpha [V,H,W] (CUDA fp32, one
    device).  Returns (TriangleMesh on the device, dict of intermediate device buffers).  `stages`: optional callback
    stages(name) called after each stage is enqueued (measurement)."""
    lib = _lib.lib()
    _check_cuda(rgb, "fuse: rgb", torch.float32)
    dev = rgb.device
    _check_cuda(depth, "fuse: depth", torch.float32, dev)
    _check_cuda(alpha, "fuse: alpha", torch.float32, dev)
    if rgb.dim() != 4 or rgb.shape[1] != 3:
        raise ValueError("fuse: rgb [V,3,H,W] expected, got %s" % (tuple(rgb.shape),))
    V, _, H, W = rgb.shape
    if tuple(depth.shape) != (V, H, W) or tuple(alpha.shape) != (V, H, W):
        raise ValueError("fuse: rgb [V,3,H,W], depth and alpha [V,H,W] expected, got %s %s %s"
                         % (tuple(rgb.shape), tuple(depth.shape), tuple(alpha.shape)))
    if V > 256:
        raise ValueError("fuse: at most 256 views")
    if setup["cams_f"].shape != (V, 20) or (setup["H"], setup["W"]) != (H, W):
        raise ValueError("fuse: the setup was made for %d views of %dx%d" % (len(setup["cams_f"]), setup["H"],
                                                                           setup["W"]))
    rgb, depth, alpha = rgb.contiguous(), depth.contiguous(), alpha.contiguous()
    s = stream(dev)
    mark = stages or (lambda name: None)
    f64 = dict(dtype=torch.float64, device=dev)
    trunc = torch.tensor(setup["depth_trunc"], **f64)
    cams_d = torch.tensor(setup["cams_d"], **f64)
    cams_f = torch.tensor(setup["cams_f"], dtype=torch.float32, device=dev)
    volume = torch.tensor([setup["voxel_length"], setup["sdf_trunc"]], **f64)
    box_h = setup["box"]
    box = torch.tensor(box_h, dtype=torch.int32, device=dev)
    n_box = int(np.prod(box_h[3:].astype(np.int64)))
    st = _Status(dev)
    texels = torch.empty(V, H, W, 2, dtype=torch.int32, device=dev)
    _lib.check(lib.ga_mesh_prepare(ptr(rgb), ptr(depth), ptr(alpha), V, H, W, ptr(trunc), float(alpha_thres),
                                   ptr(texels), s), "ga_mesh_prepare")
    mark("prepare")
    table = torch.empty(n_box, (V + 31) // 32, dtype=torch.int32, device=dev)
    pool = torch.empty(n_box, dtype=torch.int32, device=dev)
    slot = torch.empty(n_box, dtype=torch.int32, device=dev)
    work = _work(n_box, dev)
    _lib.check(lib.ga_mesh_touch(ptr(texels), V, H, W, ptr(cams_d), ptr(volume), ptr(box), n_box, ptr(table),
                                 ptr(pool), ptr(slot), ptr(work), *st.args(), s), "ga_mesh_touch")
    words = st.read()
    if words[1]:
        raise RuntimeError("extract_mesh_bounded: a depth point lies outside the volume box %s" % (box_h.tolist(),))
    n_units = words[0]
    mark("touch")
    nvox = n_units * 4096
    voxels = torch.empty(5, max(nvox, 1), dtype=torch.float32, device=dev)
    _lib.check(lib.ga_mesh_integrate(ptr(texels), V, H, W, ptr(cams_f), ptr(volume), ptr(box), ptr(table),
                                     ptr(pool), n_units, ptr(voxels), s), "ga_mesh_integrate")
    mark("integrate")
    tri_table = torch.tensor(TRI_TABLE, device=dev)
    cube = torch.empty(2, max(nvox, 1), dtype=torch.uint8, device=dev)
    vert_off = torch.empty(max(nvox, 1), dtype=torch.int32, device=dev)
    tri_off = torch.empty(max(nvox, 1), dtype=torch.int32, device=dev)
    work = _work(nvox, dev)
    _lib.check(lib.ga_mesh_cubes_count(ptr(voxels), n_units, ptr(pool), ptr(slot), ptr(box), ptr(tri_table),
                                       ptr(cube), ptr(vert_off), ptr(tri_off), ptr(work), *st.args(), s),
               "ga_mesh_cubes_count")
    words = st.read()
    nv, nt = words[2], words[3]
    verts = torch.empty(nv, 3, **f64)
    cols = torch.empty(nv, 3, **f64)
    tris = torch.empty(nt, 3, dtype=torch.int32, device=dev)
    _lib.check(lib.ga_mesh_cubes_emit(ptr(voxels), n_units, ptr(pool), ptr(slot), ptr(box), ptr(volume),
                                      ptr(tri_table), ptr(cube), ptr(vert_off), ptr(tri_off), ptr(verts),
                                      ptr(cols), ptr(tris), s), "ga_mesh_cubes_emit")
    mark("marching_cubes")
    state = dict(texels=texels, table=table, pool=pool[:n_units], slot=slot, voxels=voxels[:, :nvox],
                 cube=cube[:, :nvox], n_units=n_units)
    return TriangleMesh(verts, tris, cols), state


def _device_mesh(mesh, dev=None):
    """(vertices fp64, triangles int32, colours fp64) of `mesh` as contiguous CUDA tensors, checked: [N,3] shapes,
    as many colours as vertices, every triangle index in [0, Nv)."""
    v, t, c = mesh.tensors()
    if dev is None:
        dev = v.device if v.is_cuda else torch.device("cuda")
    v = v.to(device=dev, dtype=torch.float64).contiguous()
    t = t.to(device=dev, dtype=torch.int32).contiguous()
    c = c.to(device=dev, dtype=torch.float64).contiguous()
    if v.dim() != 2 or v.shape[1] != 3 or t.dim() != 2 or t.shape[1] != 3 or tuple(c.shape) != tuple(v.shape):
        raise ValueError("mesh: vertices / vertex_colors [Nv,3] and triangles [Nt,3] expected, got %s %s %s"
                         % (tuple(v.shape), tuple(c.shape), tuple(t.shape)))
    if t.shape[0] and (int(t.min()) < 0 or int(t.max()) >= v.shape[0]):
        raise ValueError("mesh: a triangle index is outside [0, %d)" % v.shape[0])
    return v, t, c


def keep_threshold(cluster_sizes):
    """utils/mesh_util.post_process_mesh: k = min(#clusters, 10), n = max(sort(sizes)[-k], 50)."""
    k = min(len(cluster_sizes), 10)
    return max(int(np.sort(np.asarray(cluster_sizes))[-k]), 50)


def clusters(mesh):
    """(label int32 [Nt], cluster sizes int32 [n_clusters]) on the device; clusters numbered by smallest triangle."""
    return _clusters(*_device_mesh(mesh)[:2])


def _clusters(v, t):
    lib = _lib.lib()
    dev = t.device
    nt = t.shape[0]
    slots = 1 << max(4, math.ceil(math.log2(max(6 * nt, 1))))
    hash_ = torch.empty(slots * 12, dtype=torch.uint8, device=dev)
    label = torch.empty(max(nt, 1), dtype=torch.int32, device=dev)
    sizes = torch.empty(max(nt, 1), dtype=torch.int32, device=dev)
    work = _work(nt, dev)
    st = _Status(dev)
    s = stream(dev)
    _lib.check(lib.ga_mesh_clusters(ptr(t), nt, ptr(hash_), slots, ptr(label), ptr(sizes), ptr(work),
                                    *st.args(), s), "ga_mesh_clusters")
    nc = st.read()[4]
    return label[:nt], sizes[:nc]


def post_process_mesh(mesh, cluster_to_keep=None):
    """utils/mesh_util.post_process_mesh on the GPU: keep the triangles of clusters (connected through shared edges)
    with at least max(10th largest size, 50) triangles, then the vertices they use (order kept), then drop degenerate
    triangles.  Any TriangleMesh (host or device arrays) is accepted and checked (shapes, index range); the result is
    on the GPU.  An empty mesh gives an empty mesh (the reference raises)."""
    lib = _lib.lib()
    v, t, c = _device_mesh(mesh)
    dev = v.device
    nv, nt = v.shape[0], t.shape[0]
    if nt == 0:
        return TriangleMesh(v[:0], t[:0], c[:0])
    label, sizes = _clusters(v, t)
    n_min = keep_threshold(sizes.cpu().numpy())
    out_v = torch.empty_like(v)
    out_c = torch.empty_like(c)
    out_t = torch.empty_like(t)
    work = _work(nv + nt, dev)
    st = _Status(dev)
    s = stream(dev)
    _lib.check(lib.ga_mesh_filter(ptr(v), ptr(c), nv, ptr(t), nt, ptr(label), ptr(sizes), n_min, ptr(out_v),
                                  ptr(out_c), ptr(out_t), ptr(work), *st.args(), s), "ga_mesh_filter")
    w = st.read()
    return TriangleMesh(out_v[:w[5]], out_t[:w[6]], out_c[:w[5]])


def stack_maps(rgbmaps, depthmaps, alpha_maps):
    """[i][0] indexing of the reference: rgb [V,3,H,W], depth / alpha [V,H,W], on the device, caller's tensors untouched."""
    V = len(rgbmaps)
    if not (len(depthmaps) == len(alpha_maps) == V) or V == 0:
        raise ValueError("extract_mesh_bounded: rgbmaps, depthmaps and alpha_maps need the same (non-zero) length")
    dev = _check_cuda(rgbmaps[0][0], "extract_mesh_bounded: rgbmaps", torch.float32).device
    rgb = torch.stack([_check_cuda(rgbmaps[i][0], "extract_mesh_bounded: rgbmaps", torch.float32, dev)
                       for i in range(V)])
    depth = torch.stack([_check_cuda(depthmaps[i][0], "extract_mesh_bounded: depthmaps", torch.float32, dev)
                         for i in range(V)])
    alpha = torch.stack([_check_cuda(alpha_maps[i][0], "extract_mesh_bounded: alpha_maps", torch.float32, dev)
                         for i in range(V)])
    if depth.dim() == 4:
        depth = depth[:, 0]
    if alpha.dim() == 4:
        alpha = alpha[:, 0]
    if rgb.dim() != 4:
        raise ValueError("extract_mesh_bounded: rgbmaps[i][0] must be [3,H,W], got %s" % (tuple(rgb.shape[1:]),))
    return rgb, depth, alpha


def extract_mesh_bounded(rgbmaps, depthmaps, alpha_maps, cam_pathes, voxel_size=0.004, sdf_trunc=0.02,
                         depth_trunc=3, alpha_thres=0.08, mask_backgrond=False):
    """FlowMatchingEngine.extract_mesh_bounded on the GPU.  rgbmaps[i][0] [3,H,W], depthmaps[i][0] / alpha_maps[i][0]
    [1,H,W] CUDA fp32; cam_pathes [V,25] (uni_mesh_path).  As in the reference, voxel_size / sdf_trunc / depth_trunc
    are replaced by the values derived from the fixed box (volume_settings); depth where alpha < alpha_thres is
    ignored.  The reference zeroes those depths in place; here the caller's maps are left as they are."""
    rgb, depth, alpha = stack_maps(rgbmaps, depthmaps, alpha_maps)
    setup = view_setup(cam_pathes, rgb.shape[2], rgb.shape[3])
    with torch.cuda.device(rgb.device):
        mesh, _ = fuse(rgb, depth, alpha, setup, alpha_thres=alpha_thres)
    return mesh


def rotation_matrix_x(theta_degrees):
    t = np.radians(theta_degrees)
    return np.array([[1, 0, 0], [0, np.cos(t), -np.sin(t)], [0, np.sin(t), np.cos(t)]])


def rotation_matrix_y(theta):
    return np.array([[np.cos(theta), 0, np.sin(theta)], [0, 1, 0], [-np.sin(theta), 0, np.cos(theta)]])


def write_triangle_mesh(path, mesh):
    """OBJ: `v x y z r g b` (colours in [0,1]) then 1-based `f i j k`."""
    v, t, c = mesh.vertices, mesh.triangles, mesh.vertex_colors
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    with open(path, "w") as f:
        vc = np.concatenate([v, c], 1) if len(v) else np.zeros((0, 6))
        f.write("".join("v %.17g %.17g %.17g %.17g %.17g %.17g\n" % tuple(r) for r in vc.tolist()))
        f.write("".join("f %d %d %d\n" % tuple(r) for r in (t.astype(np.int64) + 1).tolist()))
    return True


def read_triangle_mesh(path):
    """Reads what write_triangle_mesh writes."""
    v, f = [], []
    with open(path) as fh:
        for line in fh:
            if line.startswith("v "):
                v.append([float(x) for x in line.split()[1:7]])
            elif line.startswith("f "):
                f.append([int(x.split("/")[0]) - 1 for x in line.split()[1:4]])
    v = np.asarray(v, np.float64).reshape(-1, 6)
    return TriangleMesh(v[:, :3].copy(), np.asarray(f, np.int32).reshape(-1, 3), v[:, 3:].copy())


def export_mesh_from_2dgs(all_rgbs, all_depths, all_alphas, cam_pathes, idx, i, video_path=None, output_dir=None):
    """FlowMatchingEngine.export_mesh_from_2dgs: writes `<...>-mesh_raw.obj` (raw fused mesh) and `<...>-mesh.obj`
    (post-processed, vertices rotated by Rx(-90) then Ry(pi)); returns the second path.  Naming: video_path
    '-gs.mp4' -> '-mesh_raw.obj', else `output_dir/idx/i-mesh_raw.obj` (output_dir defaults to the working
    directory; the reference uses its logger's directory)."""
    if video_path is not None:
        raw_path = video_path.replace("-gs.mp4", "-mesh_raw.obj")
    else:
        raw_path = os.path.join(output_dir or os.getcwd(), f"{idx}/{i}-mesh_raw.obj")
    mesh = extract_mesh_bounded(all_rgbs, all_depths, all_alphas, cam_pathes)
    write_triangle_mesh(raw_path, mesh)
    post = post_process_mesh(mesh)
    post.vertices = np.asarray(post.vertices) @ rotation_matrix_x(-90).T @ rotation_matrix_y(np.pi).T
    post_path = raw_path.replace("_raw.obj", ".obj")
    write_triangle_mesh(post_path, post)
    return post_path


def orbit_cameras(cam_pathes):
    """cam_view, cam_view_proj [1,V,4,4], cam_pos [1,V,3] (reference row-vector layout) of the 25-float poses."""
    from tools.synth import camera_from_pose25
    cams = [camera_from_pose25(np.asarray(p, np.float32)) for p in cam_pathes]
    view = torch.tensor(np.stack([c[0] for c in cams]))[None]
    proj = torch.tensor(np.stack([c[1] for c in cams]))[None]
    pos = torch.tensor(np.stack([c[2] for c in cams]))[None]
    return view, proj, pos, cams[0][3]


def render_orbit(gauss13, cam_pathes=None, size=512):
    """One batched render of the orbit views: (cam_pathes, render dict with [1,V,...] maps), white background."""
    from .gs_surfel import GaussianRenderer2DGS
    if cam_pathes is None:
        cam_pathes = uni_mesh_path(10)
    g = gauss13 if gauss13.dim() == 3 else gauss13[None]
    dev = g.device
    view, proj, pos, tanfov = orbit_cameras(cam_pathes)
    r = GaussianRenderer2DGS(size, 3, {})
    with torch.no_grad():
        out = r.render(g, view.to(dev), proj.to(dev), pos.to(dev), tanfov,
                       bg_color=torch.ones(3, device=dev), output_size=size)
    return cam_pathes, out


def mesh_from_surfels(gauss13, size=512):
    """Surfels [P,13] or [1,P,13] (CUDA) -> (all_rgbs, all_depths, all_alphas, cam_pathes, mesh): one batched render of
    the 50 uni_mesh_path(10) views at size^2, then GPU fusion.  The first four feed export_mesh_from_2dgs."""
    cam_pathes, out = render_orbit(gauss13, None, size)
    V = len(cam_pathes)
    all_rgbs = [out["image"][:, v] for v in range(V)]             # [i][0] -> [3,H,W]
    all_depths = [out["depth"][:, v] for v in range(V)]           # [i][0] -> [1,H,W]
    all_alphas = [out["alpha"][:, v] for v in range(V)]
    mesh = extract_mesh_bounded(all_rgbs, all_depths, all_alphas, cam_pathes)
    return all_rgbs, all_depths, all_alphas, cam_pathes, mesh


def _engine_extract_mesh_bounded(self, rgbmaps, depthmaps, alpha_maps, cam_pathes, *args, **kwargs):
    return extract_mesh_bounded(rgbmaps, depthmaps, alpha_maps, cam_pathes, *args, **kwargs)


def _engine_export_mesh_from_2dgs(self, all_rgbs, all_depths, all_alphas, cam_pathes, idx, i, video_path=None):
    return export_mesh_from_2dgs(all_rgbs, all_depths, all_alphas, cam_pathes, idx, i, video_path=video_path)
