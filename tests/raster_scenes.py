"""Scene builders for the rasteriser edge tests (numpy only): shared by the GPU tests and the CPU calibration of the
fp64 walker (tests/raster_ref.py) against the C oracle, so both look at the same scenes."""
import numpy as np

from tests.helpers import cameras, scene


def _quat_from_frame(t1, t2, n):
    """Unit quaternion (w, x, y, z) of the rotation whose columns are t1, t2, n (rows of the arrays)."""
    R = np.stack([t1, t2, n], -1)                                    # [P, 3, 3], columns
    w = np.sqrt(np.maximum(0.0, 1.0 + R[:, 0, 0] + R[:, 1, 1] + R[:, 2, 2])) / 2
    x = np.sqrt(np.maximum(0.0, 1.0 + R[:, 0, 0] - R[:, 1, 1] - R[:, 2, 2])) / 2
    y = np.sqrt(np.maximum(0.0, 1.0 - R[:, 0, 0] + R[:, 1, 1] - R[:, 2, 2])) / 2
    z = np.sqrt(np.maximum(0.0, 1.0 - R[:, 0, 0] - R[:, 1, 1] + R[:, 2, 2])) / 2
    x = np.copysign(x, R[:, 2, 1] - R[:, 1, 2])
    y = np.copysign(y, R[:, 0, 2] - R[:, 2, 0])
    z = np.copysign(z, R[:, 1, 0] - R[:, 0, 1])
    q = np.stack([w, x, y, z], 1)
    return q / np.linalg.norm(q, axis=1, keepdims=True)


def _frame_for_normal(n, rng):
    n = n / np.linalg.norm(n, axis=1, keepdims=True)
    a = rng.standard_normal(n.shape)
    t1 = a - (a * n).sum(1, keepdims=True) * n
    t1 /= np.linalg.norm(t1, axis=1, keepdims=True)
    return t1, np.cross(n, t1), n


CULL_SM = 1.3               # scale_modifier the cull-box scene is built for and rendered with


def _switch_ratio(g, view, proj, H, W):
    """dt / Tw_z^2 of K1's cull box in one view (binary64): dt = tau (Tw_x^2 + Tw_y^2) - Tw_z^2 with
    tau = 2 ln(255 opacity) 1.001 + 1e-3; the box is a bounded ellipse below -1e-3 and unbounded above."""
    from tests import raster_ref as rr
    geo = rr.geometry(g, view, proj, H, W, CULL_SM)
    tau = 2.0 * np.log(255.0 * g[:, 3].astype(np.float64)) * 1.001 + 1e-3
    Tw = geo["Tw"]
    return (tau * (Tw[:, 0] ** 2 + Tw[:, 1] ** 2) - Tw[:, 2] ** 2) / Tw[:, 2] ** 2, geo


def cull_box_scene(seed=0):
    """Adversarial surfels for the cull box, placed in the frame of view 0 of three views at 120 x 100:
    opacities at float32(1/255) and its neighbours, 0.0045, 0.5, 0.99, 1; grazing surfels; sizes swept across the
    bounded-ellipse / unbounded-box switch; centres just beyond the near plane; ellipses reaching the camera plane;
    sub-pixel surfels; surfels larger than the image; centres outside the image with the footprint entering it.
    A last group is placed densely on both sides of the switch in view 0 (SWITCH_TARGETS), where 1/dt is large and
    the half-axes cancel in fp32.  Rendered at scale_modifier CULL_SM.
    Returns (g [P, 13] float32, views [3, 4, 4], projs [3, 4, 4], H, W)."""
    rng = np.random.default_rng(seed)
    H, W = 100, 120
    vs, ps, cs, tf = cameras(3, start=11)
    vm = vs[0].astype(np.float64)
    ax, ay, az = vm[:3, 0], vm[:3, 1], vm[:3, 2]
    cam = cs[0].astype(np.float64)

    def at(x, y, z):                                  # view-space coordinates -> world
        return cam + x[:, None] * ax + y[:, None] * ay + z[:, None] * az

    def lateral(z, spread=1.0):                       # points inside the view frustum at depth z
        return (rng.uniform(-spread, spread, z.size) * tf * z, rng.uniform(-spread, spread, z.size) * tf * z)

    parts = []

    def add(pos, scale, normal, opacity):
        n = pos.shape[0]
        t1, t2, nn = _frame_for_normal(normal, rng)
        g = np.zeros((n, 13))
        g[:, 0:3] = pos
        g[:, 3] = opacity
        g[:, 4:6] = scale
        g[:, 6:10] = _quat_from_frame(t1, t2, nn)
        g[:, 10:13] = rng.uniform(0, 1, (n, 3))
        parts.append(g)

    f32 = np.float32
    a255 = f32(1) / f32(255)
    ops = [np.nextafter(np.nextafter(a255, f32(0)), f32(0)), np.nextafter(a255, f32(0)), a255,
           np.nextafter(a255, f32(1)), np.nextafter(np.nextafter(a255, f32(1)), f32(1)), f32(0.0045), f32(0.5),
           f32(0.99), f32(1.0)]
    for o in ops:                                     # ordinary surfels at every opacity of interest
        n = 40
        z = rng.uniform(1.0, 2.5, n)
        x, y = lateral(z)
        add(at(x, y, z), rng.uniform(0.005, 0.06, (n, 2)), rng.standard_normal((n, 3)), float(o))
    n = 120                                           # grazing: normal nearly perpendicular to the view ray
    z = rng.uniform(0.8, 2.5, n)
    x, y = lateral(z)
    p = at(x, y, z)
    ray = (p - cam) / np.linalg.norm(p - cam, axis=1, keepdims=True)
    perp = np.cross(ray, rng.standard_normal((n, 3)))
    perp /= np.linalg.norm(perp, axis=1, keepdims=True)
    nrm = perp + ray * rng.uniform(-3e-3, 3e-3, (n, 1))
    add(p, rng.uniform(0.01, 0.3, (n, 2)), nrm, rng.choice([0.05, 0.5, 0.99], n))
    n = 400                                           # sizes swept across dt = tau |Tw_xy|^2 - Tw_z^2 = 0
    z = rng.uniform(0.6, 2.0, n)
    x, y = lateral(z, 0.8)
    tilt = rng.uniform(0.2, 1.0, n)
    nrm = np.stack([tilt * rng.choice([-1, 1], n), rng.uniform(-0.3, 0.3, n), -np.ones(n)], 1)
    nrm = nrm[:, 0:1] * ax + nrm[:, 1:2] * ay + nrm[:, 2:3] * az
    add(at(x, y, z), z[:, None] * rng.uniform(0.03, 0.6, (n, 2)), nrm, rng.choice([0.02, 0.3, 0.9, 1.0], n))
    n = 60                                            # centres just beyond the near plane
    z = 0.2 + rng.uniform(1e-4, 0.05, n)
    x, y = lateral(z)
    add(at(x, y, z), rng.uniform(0.001, 0.05, (n, 2)), rng.standard_normal((n, 3)), rng.choice([0.1, 0.9], n))
    n = 60                                            # ellipses reaching the camera plane
    z = rng.uniform(0.25, 0.6, n)
    x, y = lateral(z)
    add(at(x, y, z), rng.uniform(0.2, 0.8, (n, 2)), rng.standard_normal((n, 3)), rng.choice([0.05, 0.6, 1.0], n))
    n = 150                                           # sub-pixel: the low-pass disc dominates
    z = rng.uniform(0.5, 3.0, n)
    x, y = lateral(z)
    add(at(x, y, z), rng.uniform(1e-5, 2e-4, (n, 2)), rng.standard_normal((n, 3)), rng.choice([a255, 0.0045, 0.5, 1.0], n))
    n = 30                                            # larger than the image
    z = rng.uniform(1.0, 2.5, n)
    x, y = lateral(z, 0.3)
    nrm = np.stack([rng.uniform(-0.5, 0.5, n), rng.uniform(-0.5, 0.5, n), -np.ones(n)], 1)
    nrm = nrm[:, 0:1] * ax + nrm[:, 1:2] * ay + nrm[:, 2:3] * az
    add(at(x, y, z), rng.uniform(1.5, 4.0, (n, 2)) * z[:, None] * tf, nrm, rng.choice([0.02, 0.3], n))
    n = 200                                           # centres outside the image, footprint entering it
    z = rng.uniform(0.8, 2.5, n)
    side = rng.uniform(1.05, 1.5, n) * rng.choice([-1, 1], n)
    other = rng.uniform(-1.2, 1.2, n)
    swap = rng.uniform(size=n) < 0.5
    x = np.where(swap, side, other) * tf * z
    y = np.where(swap, other, side) * tf * z
    add(at(x, y, z), rng.uniform(0.02, 0.3, (n, 2)) * z[:, None], rng.standard_normal((n, 3)), rng.choice([0.1, 0.9], n))
    g = np.concatenate(parts, 0)
    q = g[:, 6:10]
    g[:, 6:10] = q * rng.uniform(0.7, 1.4, (q.shape[0], 1))         # non-unit quaternions are normalised
    g = g.astype(np.float32)
    # the switch: copies of tilted surfels with both half-axes scaled by k = sqrt((target + 1) / (r0 + 1)), which moves
    # dt / Tw_z^2 from r0 to the target (Tw_x and Tw_y are linear in the scales, Tw_z does not depend on them)
    n = 150
    z = rng.uniform(0.6, 2.0, n)
    x, y = lateral(z, 0.6)
    tilt = rng.uniform(0.3, 1.0, n)
    nrm = np.stack([tilt * rng.choice([-1, 1], n), rng.uniform(-0.3, 0.3, n), -np.ones(n)], 1)
    nrm = nrm[:, 0:1] * ax + nrm[:, 1:2] * ay + nrm[:, 2:3] * az
    parts = []
    add(at(x, y, z), z[:, None] * rng.uniform(0.1, 0.3, (n, 2)), nrm, rng.choice([0.05, 0.3, 0.9, 1.0], n))
    base = parts[0].astype(np.float32)
    r0, _ = _switch_ratio(base, vs[0], ps[0], H, W)
    sw = []
    for t in SWITCH_TARGETS:
        c = base.copy()
        c[:, 4:6] = base[:, 4:6] * np.sqrt((t + 1.0) / (r0 + 1.0))[:, None]
        sw.append(c)
    return np.concatenate([g] + sw, 0).astype(np.float32), vs, ps, H, W


# dt / Tw_z^2 targets of the switch group: 30 log-spaced from -1e-1 to just below the switch at -1e-3, and 6 above it
SWITCH_TARGETS = np.concatenate([-np.logspace(-1, np.log10(1.05e-3), 30), -np.logspace(np.log10(0.95e-3), -4, 6)])


def translucent_scene(seed=0):
    """Large translucent surfels crowded in front of two views of a ragged 120 x 104 image: tiles of several hundred
    instances whose 256-instance chunks need three or more windows of the forward's pair buffer, contributions on
    both sides of chunk boundaries, and backward chunks of more than 4096 records, with no pixel above 256
    contributions.  Returns (g, views [2, 4, 4], projs [2, 4, 4], H, W)."""
    rng = np.random.default_rng(seed)
    P = 2500
    g = scene(P, 300 + seed, 4.0)
    g[:, 0:3] *= 0.5
    g[:, 3] = rng.uniform(0.1, 0.4, P)
    g[:, 4:6] = rng.uniform(0.02, 0.08, (P, 2))
    vs, ps, _, _ = cameras(2, start=5)
    return g, vs, ps, 104, 120


def tiny_scene(seed=0):
    """At most 64 surfels at 32 x 48 for fp64 autograd."""
    g = scene(48, 500 + seed, 30.0)
    vs, ps, _, _ = cameras(1, start=seed)
    return g, vs, ps, 32, 48
