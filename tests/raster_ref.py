"""fp64 reference tile walker of the surfel rasteriser (numpy, host only).

Restates the maths of oracle/surfel_torch.py (itself a restatement of upstream diff-surfel-rasterization) in binary64,
tile by tile, for a given per-tile instance order (normally the one the CUDA binning produced).  Per tile the
(instance, pixel) pairs are evaluated as arrays of instances x 256 pixels, a chunk of instances at a time, and the
transmittance is a cumulative product over the instances.

Besides the fp64 result it marks the pairs whose outcome is NEAR A DECISION: a pair is flagged when one of the
algorithm's discrete decisions could go the other way in binary32 --
  alpha >= 1/255, T (1 - alpha) < 1e-4, depth >= 0.2, rho3d <= rho2d, p2 == 0, T > 0.5 (median) --
i.e. when the fp64 decision differs from the one taken by a binary32 evaluation of the same formula in either of
two associations (upstream's cross(k, l), and the tile-origin form C + dx A + dy B of csrc/raster_render.cu), or when
the fp64 value lies within REL (relative) plus four times the larger binary32 deviation of the threshold.  A pixel
is AMBIGUOUS from its first flagged pair on; everything before that pair is decided the same way in any precision.
"""
import numpy as np

NEAR_N, FAR_N = 0.2, 100.0
FILTER_SIZE, FILTER_INV_SQUARE = 0.707106, 2.0
A_MIN = 1.0 / 255.0
T_STOP = 1e-4
REL = 1e-5                 # relative margin on top of the measured binary32 deviation
EPS32 = 2.0 ** -24         # binary32 unit roundoff
CHUNK = 512                # instances evaluated at once (memory: CHUNK x 256 pairs x ~40 arrays)
# Per-pixel max-abs deviation of the fp32 C oracle from this walker on unambiguous pixels, per channel (colour 3,
# then allmap: depth, alpha, normal 3, median depth, distortion), over the scenes of tests/raster_scenes.py; measured
# on the host (tests/test_raster_ref.py::test_calibration_against_c_oracle):
#   1.4e-5 8.1e-6 8.7e-6 | 5.2e-6 2.9e-6 3.6e-5 1.9e-5 3.5e-5 5.4e-6 2.6e-6
# These are the measured values rounded up; the GPU per-pixel bars add the kernel's approximations to them.
CAL_ORACLE = (2e-5, 1e-5, 1e-5, 1e-5, 5e-6, 4e-5, 2e-5, 4e-5, 1e-5, 5e-6)


def _quat_R(q):
    q = q / np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    R = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                  2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                  2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], 1)
    return R.reshape(-1, 3, 3)


def geometry(g13, view, proj, H, W, scale_modifier=1.0):
    """Per-surfel quantities of one view in binary64: the ray-splat transform (Tu, Tv, Tw), the 2-D centre, radius,
    tile rectangle, view depth, normal (dual-visible sign applied), opacity and colour."""
    g = np.asarray(g13, np.float64)
    vm = np.asarray(view, np.float64).reshape(4, 4)
    pm = np.asarray(proj, np.float64).reshape(4, 4)
    P = g.shape[0]
    ones = np.ones((P, 1))
    mean = g[:, 0:3]
    pv = np.concatenate([mean, ones], 1) @ vm
    vz = pv[:, 2]
    R = _quat_R(g[:, 6:10])
    L0 = R[:, :, 0] * (scale_modifier * g[:, 4:5])
    L1 = R[:, :, 1] * (scale_modifier * g[:, 5:6])
    Mt = np.stack([np.concatenate([L0, 0 * ones], 1), np.concatenate([L1, 0 * ones], 1),
                   np.concatenate([mean, ones], 1)], 1)
    B = Mt @ pm
    Tu = B[:, :, 0] * (0.5 * W) + B[:, :, 3] * (0.5 * (W - 1))
    Tv = B[:, :, 1] * (0.5 * H) + B[:, :, 3] * (0.5 * (H - 1))
    Tw = B[:, :, 3]
    normal = R[:, :, 2] @ vm[:3, :3]
    cosv = -(pv[:, :3] * normal).sum(1)
    normal = normal * np.where(cosv > 0, 1.0, -1.0)[:, None]
    t = np.array([9.0, 9.0, -1.0])
    d = (t * Tw * Tw).sum(1)
    ds = np.where(d == 0, 1.0, d)
    f = t[None] / ds[:, None]
    cx = (f * Tu * Tw).sum(1)
    cy = (f * Tv * Tw).sum(1)
    ex = np.sqrt(np.maximum(cx * cx - (f * Tu * Tu).sum(1), 1e-4))
    ey = np.sqrt(np.maximum(cy * cy - (f * Tv * Tv).sum(1), 1e-4))
    radius = np.ceil(np.maximum(np.maximum(ex, ey), 3.0 * FILTER_SIZE))
    gx, gy = (W + 15) // 16, (H + 15) // 16
    with np.errstate(invalid="ignore"):
        x0 = np.clip(np.trunc((cx - radius) / 16.0), 0, gx).astype(np.int64)
        y0 = np.clip(np.trunc((cy - radius) / 16.0), 0, gy).astype(np.int64)
        x1 = np.clip(np.trunc((cx + radius + 15.0) / 16.0), 0, gx).astype(np.int64)
        y1 = np.clip(np.trunc((cy + radius + 15.0) / 16.0), 0, gy).astype(np.int64)
    ok = (vz > NEAR_N) & (cosv != 0) & (d != 0) & ((x1 - x0) * (y1 - y0) > 0)
    return dict(Tu=Tu, Tv=Tv, Tw=Tw, cx=cx, cy=cy, vz=vz, opacity=g[:, 3], normal=normal, color=g[:, 10:13],
                radii=np.where(ok, radius, 0).astype(np.int32),
                rect=np.where(ok[:, None], np.stack([x0, y0, x1, y1], 1), 0).astype(np.int64), H=H, W=W)


def bin_tiles(geo):
    """(tile_start [T+1], ids) of one view: every visible surfel in each tile of its rectangle, sorted by (binary32
    view depth, surfel id) -- the order upstream's stable radix sort of (tile, depth bits) gives."""
    W, H = geo["W"], geo["H"]
    gx, gy = (W + 15) // 16, (H + 15) // 16
    tiles, ids = [], []
    for i in np.nonzero(geo["radii"] > 0)[0]:
        x0, y0, x1, y1 = geo["rect"][i]
        tt = (np.arange(y0, y1)[:, None] * gx + np.arange(x0, x1)[None]).ravel()
        tiles.append(tt); ids.append(np.full(tt.size, i))
    tiles = np.concatenate(tiles) if tiles else np.zeros(0, np.int64)
    ids = np.concatenate(ids) if ids else np.zeros(0, np.int64)
    dbits = geo["vz"].astype(np.float32).view(np.uint32)[ids]
    o = np.lexsort((ids, dbits, tiles))
    ts = np.zeros(gx * gy + 1, np.int64)
    np.add.at(ts, tiles + 1, 1)
    return np.cumsum(ts), ids[o]


def _pairs(geo, sid, px, py, ox, oy, fp32=True):
    """fp64 and the two binary32 evaluations of every (surfel, pixel) pair: dicts of [n, m] arrays (the binary32 ones
    are None with fp32=False)."""
    Tu, Tv, Tw = geo["Tu"][sid], geo["Tv"][sid], geo["Tw"][sid]
    cx, cy, op = geo["cx"][sid], geo["cy"][sid], geo["opacity"][sid]
    X, Y = px[None, :], py[None, :]

    def finish(p0, p1, p2, cxx, cyy, tw, opa, X, Y, dt):
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            s0, s1 = p0 / p2, p1 / p2
            rho3d = s0 * s0 + s1 * s1
            dx, dy = cxx - X, cyy - Y
            rho2d = dt(FILTER_INV_SQUARE) * (dx * dx + dy * dy)
            use3d = rho3d <= rho2d
            rho = np.minimum(rho3d, rho2d)
            depth = np.where(use3d, (s0 * tw[0] + s1 * tw[1]) + tw[2], tw[2])
            alpha = np.minimum(dt(0.99), opa * np.exp(dt(-0.5) * rho))
        return dict(p2=p2, rho3d=rho3d, rho2d=rho2d, depth=depth, alpha=alpha)

    col = lambda a: a[:, None]
    # binary64, upstream association
    k = [X * col(Tw[:, c]) - col(Tu[:, c]) for c in range(3)]
    l_ = [Y * col(Tw[:, c]) - col(Tv[:, c]) for c in range(3)]
    p = (k[1] * l_[2] - k[2] * l_[1], k[2] * l_[0] - k[0] * l_[2], k[0] * l_[1] - k[1] * l_[0])
    tw = [col(Tw[:, c]) for c in range(3)]
    r64 = finish(*p, col(cx), col(cy), tw, col(op), X, Y, np.float64)
    # first-order bound of the alpha error of any binary32 evaluation, in either association: every intermediate of
    # p = k x l is at most Pm in magnitude (k, l, and the tile-local terms dx A, dy B with dx, dy < 16), so each p_i is
    # off by O(eps Pm_i); that moves s = (p0, p1) / p2 and hence rho, and alpha = o exp(-rho / 2) moves by alpha drho / 2
    Km = [np.abs(X * col(Tw[:, c])) + col(np.abs(Tu[:, c]) + 16 * np.abs(Tw[:, c])) for c in range(3)]
    Lm = [np.abs(Y * col(Tw[:, c])) + col(np.abs(Tv[:, c]) + 16 * np.abs(Tw[:, c])) for c in range(3)]
    Pm = (Km[1] * Lm[2] + Km[2] * Lm[1], Km[2] * Lm[0] + Km[0] * Lm[2], Km[0] * Lm[1] + Km[1] * Lm[0])
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        a0, a1 = np.abs(p[0] / p[2]), np.abs(p[1] / p[2])
        drho3d = 2 * (a0 * (Pm[0] + a0 * Pm[2]) + a1 * (Pm[1] + a1 * Pm[2])) / np.abs(p[2]) + r64["rho3d"]
    ddx, ddy = np.abs(col(cx) - X), np.abs(col(cy) - Y)
    drho2d = 4 * (ddx * (col(np.abs(cx)) + X) + ddy * (col(np.abs(cy)) + Y)) + r64["rho2d"]
    drho = np.where(r64["rho3d"] <= r64["rho2d"], drho3d, drho2d)
    r64["alpha_cond"] = EPS32 * r64["alpha"] * (0.5 * drho + 4)
    if not fp32:
        return r64, None, None
    f = np.float32
    Tu32, Tv32, Tw32 = Tu.astype(f), Tv.astype(f), Tw.astype(f)
    cx32, cy32, op32 = col(cx.astype(f)), col(cy.astype(f)), col(op.astype(f))
    tw32 = [col(Tw32[:, c]) for c in range(3)]
    X32, Y32 = X.astype(f), Y.astype(f)
    # binary32, upstream association: p = cross(x Tw - Tu, y Tw - Tv)
    k = [X32 * tw32[c] - col(Tu32[:, c]) for c in range(3)]
    l_ = [Y32 * tw32[c] - col(Tv32[:, c]) for c in range(3)]
    p = (k[1] * l_[2] - k[2] * l_[1], k[2] * l_[0] - k[0] * l_[2], k[0] * l_[1] - k[1] * l_[0])
    ra = finish(*p, cx32, cy32, tw32, op32, X32, Y32, f)
    # binary32, tile-origin association: p = C + dx A + dy B around the tile origin
    ko = [f(ox) * Tw32[:, c] - Tu32[:, c] for c in range(3)]
    lo = [f(oy) * Tw32[:, c] - Tv32[:, c] for c in range(3)]
    C = (ko[1] * lo[2] - ko[2] * lo[1], ko[2] * lo[0] - ko[0] * lo[2], ko[0] * lo[1] - ko[1] * lo[0])
    A = (Tw32[:, 1] * lo[2] - Tw32[:, 2] * lo[1], Tw32[:, 2] * lo[0] - Tw32[:, 0] * lo[2],
         Tw32[:, 0] * lo[1] - Tw32[:, 1] * lo[0])
    Bv = (ko[1] * Tw32[:, 2] - ko[2] * Tw32[:, 1], ko[2] * Tw32[:, 0] - ko[0] * Tw32[:, 2],
          ko[0] * Tw32[:, 1] - ko[1] * Tw32[:, 0])
    DX, DY = (X32 - f(ox)), (Y32 - f(oy))
    p = tuple((col(C[c]) + DX * col(A[c])) + DY * col(Bv[c]) for c in range(3))
    DXc, DYc = cx32 - f(ox), cy32 - f(oy)
    rb = finish(*p, DXc, DYc, tw32, op32, DX, DY, f)
    return r64, ra, rb


def _near(x64, xa, xb, thr, scale):
    """True where the decision x >= thr is not the same in every precision, or lies within the margin."""
    xa, xb = xa.astype(np.float64), xb.astype(np.float64)
    d64 = x64 >= thr
    with np.errstate(invalid="ignore"):
        err = np.maximum(np.nan_to_num(np.abs(xa - x64), nan=np.inf), np.nan_to_num(np.abs(xb - x64), nan=np.inf))
        return (d64 != (xa >= thr)) | (d64 != (xb >= thr)) | (np.abs(x64 - thr) <= REL * scale + 4.0 * err)


def walk(geo, tile_start, ids, bg):
    """Walks every tile of one view in the given order (tile_start [T+1] and ids, offsets relative to ids).

    Returns a dict:
      color [3,H,W], allmap [7,H,W], final_T [H,W] (binary64)
      n_list, last, median [H,W]: contributions, last contributor and median contributor (1-based list positions,
        median -1 when none), as the forward counts them
      amb_from [H,W]: list position of the pixel's first flagged pair (a large value when there is none);
        ambiguous = amb_from < that value
      pairs: per contribution, sorted by (pixel, position): pix (y*W + x), pos, id, alpha, depth, and alpha_dev32 /
        depth_dev32, the larger deviation of the two binary32 evaluations from the fp64 value, and alpha_cond, a
        first-order bound (in units of the binary32 rounding) of the alpha error of any binary32 evaluation
      flagged_ids: ids of the surfels that own a flagged pair."""
    H, W = geo["H"], geo["W"]
    gx, gy = (W + 15) // 16, (H + 15) // 16
    bg = np.asarray(bg, np.float64)
    BIG = np.iinfo(np.int64).max
    out = dict(color=np.zeros((3, H, W)), allmap=np.zeros((7, H, W)), final_T=np.ones((H, W)),
               n_list=np.zeros((H, W), np.int64), last=np.zeros((H, W), np.int64),
               median=np.full((H, W), -1, np.int64), amb_from=np.full((H, W), BIG, np.int64))
    pair_parts = []
    flagged = set()
    ly, lx = np.divmod(np.arange(256), 16)
    m_c0, m_c1 = FAR_N / (FAR_N - NEAR_N), FAR_N * NEAR_N / (FAR_N - NEAR_N)
    for ty in range(gy):
        for tx in range(gx):
            t = ty * gx + tx
            ox, oy = tx * 16, ty * 16
            inside = (ox + lx < W) & (oy + ly < H)
            px, py = (ox + lx[inside]).astype(np.float64), (oy + ly[inside]).astype(np.float64)
            pix = ((oy + ly[inside]) * W + ox + lx[inside]).astype(np.int64)
            m = pix.size
            sids = np.asarray(ids[tile_start[t]:tile_start[t + 1]], np.int64)
            T = np.ones(m); T32 = np.ones(m, np.float32)
            done = np.zeros(m, bool)
            Cc = np.zeros((3, m)); Nn = np.zeros((3, m)); D = np.zeros(m); M1 = np.zeros(m); M2 = np.zeros(m)
            dist = np.zeros(m); med_d = np.zeros(m); med = np.full(m, -1, np.int64); last = np.zeros(m, np.int64)
            nl = np.zeros(m, np.int64); amb = np.full(m, BIG, np.int64)
            for c0 in range(0, len(sids), CHUNK):
                if done.all():
                    break
                sid = sids[c0:c0 + CHUNK]
                n = sid.size
                pos = c0 + np.arange(n)[:, None]
                r, ra, rb = _pairs(geo, sid, px, py, ox, oy)
                with np.errstate(invalid="ignore"):
                    valid = (r["p2"] != 0) & (r["depth"] >= NEAR_N) & (r["alpha"] >= A_MIN)
                    valid32 = (ra["p2"] != 0) & (ra["depth"] >= NEAR_N) & (ra["alpha"] >= A_MIN)
                a = np.where(valid, r["alpha"], 0.0)
                a32 = np.where(valid, np.nan_to_num(ra["alpha"]), np.float32(0))
                Tinc = T[None] * np.cumprod(1.0 - a, 0)
                Tex = np.concatenate([T[None], Tinc[:-1]], 0)
                Tinc32 = T32[None] * np.cumprod(np.float32(1) - a32, 0, dtype=np.float32)
                Tex32 = np.concatenate([T32[None], Tinc32[:-1]], 0)
                stop = valid & (Tinc < T_STOP) & ~done[None]
                first_stop = np.where(stop.any(0), stop.argmax(0), n)
                idx = np.arange(n)[:, None]
                live = (idx <= first_stop[None]) & ~done[None]             # pairs whose decisions matter
                contrib = valid & (idx < first_stop[None]) & ~done[None]
                # ---- decisions near a flip
                fa = _near(r["alpha"], ra["alpha"], rb["alpha"], A_MIN, A_MIN)
                passing = valid | fa | valid32
                fl = fa.copy()
                fl |= passing & _near(r["depth"], ra["depth"], rb["depth"], NEAR_N, NEAR_N)
                fl |= passing & _near(r["rho2d"] - r["rho3d"], ra["rho2d"] - ra["rho3d"], rb["rho2d"] - rb["rho3d"],
                                      0.0, np.abs(r["rho2d"]) + np.abs(r["rho3d"]))
                fl |= (r["p2"] == 0) | (ra["p2"] == 0) | (rb["p2"] == 0)
                fl |= valid & _near(Tinc, Tinc32, Tinc32, T_STOP, T_STOP)
                fl |= contrib & _near(Tex, Tex32, Tex32, 0.5, 0.5)
                fl &= live
                if fl.any():
                    amb = np.minimum(amb, np.where(fl.any(0), c0 + fl.argmax(0), BIG))
                    flagged.update(np.unique(np.broadcast_to(sid[:, None], fl.shape)[fl]).tolist())
                # ---- compositing of the contributions
                w = np.where(contrib, a * Tex, 0.0)
                with np.errstate(divide="ignore"):
                    mm = np.where(contrib, m_c0 - m_c1 / np.where(contrib, r["depth"], 1.0), 0.0)
                A_b = 1.0 - Tex
                M1b = M1[None] + np.cumsum(mm * w, 0) - mm * w
                M2b = M2[None] + np.cumsum(mm * mm * w, 0) - mm * mm * w
                dist += ((mm * mm * A_b + M2b - 2 * mm * M1b) * w).sum(0)
                M1 += (mm * w).sum(0); M2 += (mm * mm * w).sum(0)
                D += (np.where(contrib, r["depth"], 0.0) * w).sum(0)
                Nn += np.einsum("jc,jp->cp", geo["normal"][sid], w)
                Cc += np.einsum("jc,jp->cp", geo["color"][sid], w)
                mmask = contrib & (Tex > 0.5)
                has_m = mmask.any(0)
                jm = n - 1 - mmask[::-1].argmax(0)
                med = np.where(has_m, c0 + jm + 1, med)
                med_d = np.where(has_m, r["depth"][jm, np.arange(m)], med_d)
                has_c = contrib.any(0)
                jl = n - 1 - contrib[::-1].argmax(0)
                last = np.where(has_c, c0 + jl + 1, last)
                nl += contrib.sum(0)
                jj, pp = np.nonzero(contrib)
                if jj.size:
                    dev32 = lambda q: np.maximum(np.abs(ra[q][jj, pp] - r[q][jj, pp]), np.abs(rb[q][jj, pp] - r[q][jj, pp]))
                    pair_parts.append(np.stack([pix[pp].astype(np.float64), (c0 + jj).astype(np.float64),
                                                sid[jj].astype(np.float64), r["alpha"][jj, pp], r["depth"][jj, pp],
                                                dev32("alpha"), dev32("depth"), r["alpha_cond"][jj, pp]], 1))
                # state after the chunk: T after the last contribution, or the T the pixel stopped at
                T_new = np.where(first_stop < n, Tex[np.minimum(first_stop, n - 1), np.arange(m)], Tinc[-1])
                T32_new = np.where(first_stop < n, Tex32[np.minimum(first_stop, n - 1), np.arange(m)], Tinc32[-1])
                T = np.where(done, T, T_new); T32 = np.where(done, T32, T32_new)
                done |= first_stop < n
            yy, xx = pix // W, pix % W
            out["final_T"][yy, xx] = T
            for c in range(3):
                out["color"][c, yy, xx] = Cc[c] + T * bg[c]
                out["allmap"][2 + c, yy, xx] = Nn[c]
            out["allmap"][0, yy, xx] = D
            out["allmap"][1, yy, xx] = 1.0 - T
            out["allmap"][5, yy, xx] = med_d
            out["allmap"][6, yy, xx] = dist
            out["n_list"][yy, xx] = nl; out["last"][yy, xx] = last; out["median"][yy, xx] = med
            out["amb_from"][yy, xx] = amb
    pr = np.concatenate(pair_parts, 0) if pair_parts else np.zeros((0, 8))
    o = np.lexsort((pr[:, 1], pr[:, 0]))
    pr = pr[o]
    out["pairs"] = dict(pix=pr[:, 0].astype(np.int64), pos=pr[:, 1].astype(np.int64), id=pr[:, 2].astype(np.int64),
                        alpha=pr[:, 3], depth=pr[:, 4], alpha_dev32=pr[:, 5], depth_dev32=pr[:, 6],
                        alpha_cond=pr[:, 7])
    out["ambiguous"] = out["amb_from"] < BIG
    out["flagged_ids"] = np.array(sorted(flagged), np.int64)
    return out


def clear_pass_boxes(geo, eps=1e-3):
    """Per surfel, the pixels of its tile rectangle (inside the image) where the binary64 alpha is at least
    (1/255)(1 + eps) with depth >= near: returns (count [P], xmin, xmax, ymin, ymax [P]) of those pixels; an
    axis-aligned box holds them all exactly when it holds this bounding box."""
    H, W = geo["H"], geo["W"]
    P = geo["radii"].shape[0]
    cnt = np.zeros(P, np.int64)
    bb = np.zeros((4, P))
    for i in np.nonzero(geo["radii"] > 0)[0]:
        x0, y0, x1, y1 = geo["rect"][i]
        xs = np.arange(16 * x0, min(16 * x1, W), dtype=np.float64)
        ys = np.arange(16 * y0, min(16 * y1, H), dtype=np.float64)
        X, Y = np.meshgrid(xs, ys)
        r, _, _ = _pairs(geo, np.array([i]), X.ravel(), Y.ravel(), 0, 0, fp32=False)
        with np.errstate(invalid="ignore"):
            ok = (r["p2"][0] != 0) & (r["depth"][0] >= NEAR_N) & (r["alpha"][0] >= A_MIN * (1 + eps))
        cnt[i] = ok.sum()
        if cnt[i]:
            bb[:, i] = X.ravel()[ok].min(), X.ravel()[ok].max(), Y.ravel()[ok].min(), Y.ravel()[ok].max()
    return cnt, bb[0], bb[1], bb[2], bb[3]
