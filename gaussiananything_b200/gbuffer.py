"""3D VAE reconstruction from a G-buffer chunk folder: the reference's third inference entry point
(shell_scripts/release/inference/vae-3d.sh) from its real input.

A chunk folder holds 16 posed views of one object as the reference's dataset stores them
(datasets/g_buffer_objaverse.py read_chunk :3225-3302): raw_img.jpg and normal.png with the views side by side,
alpha.jpg likewise, depth.npz ['depth'] fp32 [16, h, w], c.npy fp32 [16, 25] (c2w 16 | normalised K 9), bbox.npy,
caption.txt, ins.txt; the object's surface samples are a separate fps-4096.ply, or are made from the depth maps by
pcd.chunk_surface_pcd.

  read_chunk / read_fps_pcd   decode the files on the host (PIL and numpy; the PLY is parsed here)
  pack                        one launch of ga_gbuffer_pack: img_to_encoder [V, 15, H, W] and the render targets
  cameras                     the chunk's c rows in the renderer's camera format (mesh.orbit_cameras)
  metrics                     ga_recon_metrics on rendered maps against the targets -> per-view numbers
  perceptual_metrics          per-view LPIPS (VGG) and SSIM of the rendered images against the targets (lpips.py)
  reconstruct_chunk           (surface cloud, pcd.py, when none is given) -> pack -> encode -> decode -> render at the chunk's own cameras -> metrics
                              (SurfelAE behaviour 'reconstruct_chunk')

Deployed configuration only: the files' size == reso_encoder == reso == 512, cameras used as stored
(frame_0_as_canonical=False), ImageNet Normalize, Pluecker rays, normals, unprojected xyz.  The view split is the
reference's (PostProcess.paired_post_process_chunk with split_chunk_size 16: no shuffle, the first 8 views go to the
encoder, the last 8 are the held-out ones).
"""
import os

import numpy as np
import torch

from . import _lib
from ._launch import ptr, stream

SIZE = 512
CHUNK_FILES = ("raw_img.jpg", "normal.png", "alpha.jpg", "depth.npz", "c.npy")
PSNR_CAP = 100.0                         # dB reported where the squared error is exactly zero
METRIC_BLOCKS = 64                       # GA_RECON_METRICS_BLOCKS of include/ga_b200.h


def read_chunk(path):
    """Decodes one chunk folder.  Returns host arrays, the views still side by side (the kernel de-tiles):
    raw_img, normal uint8 [h, n * w, 3]; alpha uint8 [h, n * w]; depth fp32 [n, h, w]; c fp32 [n, 25];
    bbox uint8 [n, 4], caption, ins (None when their optional files are absent)."""
    from PIL import Image
    missing = [f for f in CHUNK_FILES if not os.path.isfile(os.path.join(path, f))]
    if missing:
        raise FileNotFoundError("chunk folder %s lacks %s" % (path, ", ".join(missing)))
    c = np.load(os.path.join(path, "c.npy")).astype(np.float32)
    with np.load(os.path.join(path, "depth.npz")) as z:
        depth = np.ascontiguousarray(z["depth"], dtype=np.float32)
    if c.ndim != 2 or c.shape[1] != 25 or depth.ndim != 3 or depth.shape[0] != c.shape[0]:
        raise ValueError("chunk %s: c.npy %s and depth %s are not [n, 25] and [n, h, w]" % (path, c.shape, depth.shape))
    n, h, w = depth.shape

    def image(name, mode, shape):
        a = np.array(Image.open(os.path.join(path, name)).convert(mode))
        if a.shape != shape:
            raise ValueError("chunk %s: %s is %s, expected %s (%d views of %d x %d side by side)"
                             % (path, name, a.shape, shape, n, h, w))
        return a
    out = {"raw_img": image("raw_img.jpg", "RGB", (h, n * w, 3)), "normal": image("normal.png", "RGB", (h, n * w, 3)),
           "alpha": image("alpha.jpg", "L", (h, n * w)), "depth": depth, "c": c, "bbox": None, "caption": None, "ins": None}
    if os.path.isfile(os.path.join(path, "bbox.npy")):
        out["bbox"] = np.load(os.path.join(path, "bbox.npy")).astype(np.uint8)
    for key in ("caption", "ins"):
        f = os.path.join(path, key + ".txt")
        if os.path.isfile(f):
            with open(f, encoding="utf-8") as fh:
                out[key] = fh.read()
    return out


_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2",
              "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4",
              "double": "f8", "float64": "f8"}


def read_fps_pcd(path):
    """Vertex positions of a PLY file (binary_little_endian or ascii), fp32 [N, 3]: the x, y, z properties of the
    `vertex` element, which must be the file's first element; other vertex properties are skipped."""
    with open(path, "rb") as f:
        data = f.read()
    end = data.find(b"end_header")
    if not data.startswith(b"ply") or end < 0:
        raise ValueError("%s is not a PLY file" % path)
    body = data[data.index(b"\n", end) + 1:]
    fmt, count, props, elements = None, None, [], []
    for line in data[:end].decode("ascii", "replace").splitlines():
        t = line.split()
        if not t:
            continue
        if t[0] == "format":
            fmt = t[1]
        elif t[0] == "element":
            elements.append(t[1])
            if t[1] == "vertex":
                if len(elements) != 1:
                    raise ValueError("%s: the vertex element is not the first one" % path)
                count = int(t[2])
        elif t[0] == "property" and elements == ["vertex"]:
            if t[1] == "list" or t[1] not in _PLY_TYPES:
                raise ValueError("%s: unsupported vertex property %r" % (path, line))
            props.append((t[2], _PLY_TYPES[t[1]]))
    names = [p[0] for p in props]
    if count is None or not all(k in names for k in "xyz"):
        raise ValueError("%s: no vertex element with x, y, z" % path)
    if fmt == "binary_little_endian":
        dt = np.dtype([(nm, "<" + ty) for nm, ty in props])
        if len(body) < count * dt.itemsize:
            raise ValueError("%s: %d vertices declared, the data holds fewer" % (path, count))
        v = np.frombuffer(body, dtype=dt, count=count)
        return np.stack([v["x"], v["y"], v["z"]], 1).astype(np.float32)
    if fmt == "ascii":
        rows = body.decode("ascii").split("\n")[:count]
        v = np.array([r.split() for r in rows], dtype=np.float64)
        if v.shape != (count, len(props)):
            raise ValueError("%s: %d vertices declared, the data holds fewer" % (path, count))
        return np.stack([v[:, names.index(k)] for k in "xyz"], 1).astype(np.float32)
    raise ValueError("%s: PLY format %r is not supported (binary_little_endian and ascii are)" % (path, fmt))


_ARRAYS = ("raw_img", "normal", "alpha", "depth", "c")


def to_device(chunk, device):
    """The chunk's five arrays as device tensors (a chunk that already holds them there is returned as it is)."""
    return {k: (v if isinstance(v, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(v))).to(device)
            if k in _ARRAYS else v for k, v in chunk.items()}


def pack(chunk, views=None, device="cuda", with_targets=True):
    """Builds the encoder input of the chosen views on the GPU, in one launch, from the chunk as read (host arrays,
    or to_device's tensors: then nothing is copied).

    Returns (img_to_encoder fp32 [V, 15, H, W], targets, c fp32 [V, 25] on the device).  targets: img [V, 3, H, W] in
    [-1, 1], alpha, depth, mask (depth > 0) [V, 1, H, W] and normal = img_to_encoder[:, 3:6] (a view, Blender frame);
    None when with_targets is False."""
    n, h, w = chunk["depth"].shape
    if h != SIZE or w != SIZE:
        raise NotImplementedError("gbuffer.pack: chunk views are %d x %d; only %d x %d (reso == reso_encoder == the "
                                  "files' size) is built, other sizes need the reference's resizes" % (h, w, SIZE, SIZE))
    views = list(range(n)) if views is None else [int(v) for v in views]
    if not views or min(views) < 0 or max(views) >= n:
        raise IndexError("gbuffer.pack: views %r outside the chunk's %d views" % (views, n))
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError("gbuffer.pack runs on a CUDA device (there is no CPU fallback)")
    V = len(views)
    raw, normal, alpha, depth, c = (to_device(chunk, dev)[k] for k in _ARRAYS)
    vi = torch.tensor(views, dtype=torch.int32, device=dev)
    enc = torch.empty(V, 15, h, w, device=dev)
    t = None
    if with_targets:
        t = {"img": torch.empty(V, 3, h, w, device=dev), "alpha": torch.empty(V, 1, h, w, device=dev),
             "depth": torch.empty(V, 1, h, w, device=dev), "mask": torch.empty(V, 1, h, w, device=dev)}
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().ga_gbuffer_pack(
            ptr(raw), ptr(normal), ptr(alpha), ptr(depth), ptr(c), n, h, w, ptr(vi), V, ptr(enc),
            *[ptr(t[k] if t else None) for k in ("img", "alpha", "depth", "mask")], stream(dev)), "ga_gbuffer_pack")
    if t is not None:
        t["normal"] = enc[:, 3:6]
    return enc, t, c[vi.long()]


def cameras(c):
    """The chunk's c rows [V, 25] -> {'cam_view', 'cam_view_proj' [1, V, 4, 4], 'cam_pos' [1, V, 3], 'tanfov'} on c's
    device: what GaussianRenderer2DGS.render and SurfelAE's 'triplane_dec' take."""
    from .mesh import orbit_cameras
    dev = c.device if isinstance(c, torch.Tensor) else torch.device("cpu")
    rows = c.detach().cpu().numpy() if isinstance(c, torch.Tensor) else np.asarray(c)
    view, proj, pos, tanfov = orbit_cameras(rows)
    return {"cam_view": view.to(dev), "cam_view_proj": proj.to(dev), "cam_pos": pos.to(dev), "tanfov": tanfov}


def metric_table(render_out, targets):
    """ga_recon_metrics: fp32 [V, 8] sums (include/ga_b200.h Part 7) of rendered maps against targets.  render_out:
    the dict GaussianRenderer2DGS.render returns, [1, V, ...] or [V, ...]; targets: pack's."""
    sq = lambda x: (x[0] if x.dim() == 5 else x).float().contiguous()
    img, dep, alp, nrm = (sq(render_out[k]) for k in ("image", "depth", "alpha", "rend_normal"))
    V, _, H, W = img.shape
    tn = targets["normal"]
    if tuple(targets["img"].shape) != (V, 3, H, W) or tuple(tn.shape) != (V, 3, H, W):
        raise ValueError("gbuffer.metrics: render %s and targets %s differ in shape" % (tuple(img.shape),
                                                                                        tuple(targets["img"].shape)))
    if tn.stride()[1:] != (H * W, W, 1):
        tn = tn.contiguous()
    dev = img.device
    partial = torch.empty(V, METRIC_BLOCKS, 8, device=dev)
    table = torch.empty(V, 8, device=dev)
    ti, td, ta, tm = (targets[k].contiguous() for k in ("img", "depth", "alpha", "mask"))
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().ga_recon_metrics(ptr(img), ptr(dep), ptr(alp), ptr(nrm), ptr(ti), ptr(td), ptr(ta), ptr(tm), ptr(tn),
                                               tn.stride(0) if V > 1 else 3 * H * W, V, H, W, ptr(partial), ptr(table),
                                               stream(dev)), "ga_recon_metrics")
    return table


def derive(table):
    """Per-view numbers from the [V, 8] table (fp64, on the host): psnr on [0, 1] (PSNR_CAP dB where the error is
    exactly zero), depth_l1 and normal_error averaged over the target's foreground (0 for a view without any),
    alpha_l1, iou of the alpha maps at 0.5 (1 where both are empty), fg_pixels."""
    t = table.detach().double().cpu()
    mse = t[:, 0] / (3 * t[:, 7])
    fg = t[:, 2].clamp_min(1)
    zero, has_fg = torch.zeros_like(mse), t[:, 2] > 0
    return {"psnr": torch.where(mse > 0, (-10 * torch.log10(mse.clamp_min(1e-300))).clamp_max(PSNR_CAP),
                                torch.full_like(mse, PSNR_CAP)),
            "depth_l1": torch.where(has_fg, t[:, 1] / fg, zero),
            "normal_error": torch.where(has_fg, t[:, 3] / fg, zero),
            "alpha_l1": t[:, 4] / t[:, 7],
            "iou": torch.where(t[:, 6] > 0, t[:, 5] / t[:, 6].clamp_min(1), torch.ones_like(mse)),
            "fg_pixels": t[:, 2]}


def metrics(render_out, targets):
    return derive(metric_table(render_out, targets))


def perceptual_metrics(render_out, targets, lpips_model):
    """Per-view {'lpips' [V], 'ssim' [V]} (fp32, on the device) of the rendered images against the targets, over
    the whole frame (no mask): LPIPS compares render_out['image'] * 2 - 1 with targets['img'], both in [-1, 1];
    SSIM compares render_out['image'] with (targets['img'] + 1) / 2, both in [0, 1].  render_out: [1, V, ...] or
    [V, ...]; lpips_model: an lpips.LPIPS."""
    from .lpips import ssim
    img = render_out["image"]
    img = (img[0] if img.dim() == 5 else img).float()
    t = targets["img"].float()
    if tuple(img.shape) != tuple(t.shape):
        raise ValueError("gbuffer.perceptual_metrics: render %s and targets %s differ in shape"
                         % (tuple(img.shape), tuple(t.shape)))
    return {"lpips": lpips_model(img * 2 - 1, t).reshape(-1), "ssim": ssim(img, (t + 1) / 2)}


def reconstruct_chunk(ae, chunk, pcd=None, input_views=range(8), eval_views=range(8, 16), fps_start=None, generator=None,
                      bg_color=None, lpips=None):
    """The VAE round trip on one chunk: the encoder sees `input_views`, the finest level of detail (73 728 surfels
    at the deployed sizes) is rendered at the chunk's own cameras for `input_views` and `eval_views`, and each render
    is scored against the chunk's files.  chunk: a folder or read_chunk's dict; pcd: a PLY path or [N, 3], or None:
    the chunk's own surface cloud, pcd.chunk_surface_pcd of all its views (what the reference's save_pcd.py writes).

    Returns the 'enc_dec_wo_triplane' dict (latent, the four gaussians_* levels) plus 'input' and 'eval', each
    {'views', 'c', 'render' (GaussianRenderer2DGS.render's dict, [1, V, ...]), 'targets', 'table' [V, 8],
    'metrics'}; with `lpips` (an lpips.LPIPS) each also holds 'perceptual' (perceptual_metrics)."""
    if ae.encoder is None:
        raise NotImplementedError("SurfelAE(behaviour='reconstruct_chunk') needs encoder= (vae_encoder.SurfelEncoder)")
    if isinstance(chunk, (str, os.PathLike)):
        chunk = read_chunk(chunk)
    if isinstance(pcd, (str, os.PathLike)):
        pcd = read_fps_pcd(pcd)
    input_views, eval_views = list(input_views), list(eval_views)
    if len(input_views) != ae.encoder.V:
        raise ValueError("reconstruct_chunk: %d input views, the encoder was built for %d" % (len(input_views), ae.encoder.V))
    dev = torch.device("cuda", torch.cuda.current_device())
    if pcd is None:
        from .pcd import chunk_surface_pcd
        pcd = chunk_surface_pcd(chunk, device=dev)
    pcd = torch.as_tensor(pcd, dtype=torch.float32).to(dev).reshape(1, -1, 3)
    enc_in, t_all, c_all = pack(chunk, input_views + eval_views, dev)
    nin = len(input_views)
    out = ae(img=enc_in[:nin], behaviour="enc_dec_wo_triplane", pcd=pcd, fps_start=fps_start, generator=generator)
    bg = torch.ones(3, device=dev) if bg_color is None else bg_color
    cam = cameras(c_all)
    with torch.no_grad():
        r = ae.gs.render(out["gaussians_upsampled_3"], cam["cam_view"], cam["cam_view_proj"], cam["cam_pos"],
                         tanfov=cam["tanfov"], bg_color=bg, output_size=enc_in.shape[-1])
    table = metric_table(r, t_all)
    perc = perceptual_metrics(r, t_all, lpips) if lpips is not None else None
    for name, lo, hi, views in (("input", 0, nin, input_views), ("eval", nin, len(c_all), eval_views)):
        if hi > lo:
            out[name] = {"views": views, "c": c_all[lo:hi], "render": {k: v[:, lo:hi] for k, v in r.items()},
                         "targets": {k: v[lo:hi] for k, v in t_all.items()}, "table": table[lo:hi],
                         "metrics": derive(table[lo:hi])}
            if perc is not None:
                out[name]["perceptual"] = {k: v[lo:hi] for k, v in perc.items()}
    return out
