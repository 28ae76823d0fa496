"""The backward's per-surfel gradient rows, in fp64 numpy: mapping every (tile, instance) partial sum through its view's
chain rule and then summing (render_bwd_kernel's grad_row, then preprocess_bwd_kernel) gives what summing the partials
per view and then applying each view's chain rule gives (the per-(view, surfel) accumulator the backward used
before).  The map is linear, so the two orders agree to rounding."""
import numpy as np
import pytest

T9 = np.array([9.0, 9.0, -1.0])          # K1's weights of the mean-2D denominator: cutoff^2, cutoff^2, -1


def view_A(pm, W, H):
    """A[k][c]: dL/dM[r][k] = sum_c A[k][c] dL/dT_c[r], T_c = Tu, Tv, Tw (pm: the 16 floats of the projection)."""
    hw, hh, cw, ch = 0.5 * W, 0.5 * H, 0.5 * (W - 1), 0.5 * (H - 1)
    return np.array([[pm[4 * k] * hw + pm[4 * k + 3] * cw, pm[4 * k + 1] * hh + pm[4 * k + 3] * ch, pm[4 * k + 3]]
                     for k in range(3)])


def normal_sign(vm, p, R):
    """K5's sign of the view-space normal, cosv > 0 ? 1 : -1 (so -1 at cosv == 0)."""
    V = vm.reshape(4, 4)
    pv = p @ V[:3, :3] + V[3, :3]
    n = R[:, 2] @ V[:3, :3]
    cosv = -(pv @ n)
    return 1.0 if cosv > 0 else -1.0


def fold_mean2d(g, T):
    """dL/dT (as G[c][r]) with the mean-2D gradient g[9:11] folded in."""
    Tu, Tv, Tw = T
    G = g[0:9].reshape(3, 3).copy()
    gmx, gmy = g[9], g[10]
    if gmx != 0 or gmy != 0:
        dd = (T9 * Tw * Tw).sum()
        f = T9 / dd
        G[0] += gmx * f * Tw
        G[1] += gmy * f * Tw
        G[2] += gmx * f * Tu + gmy * f * Tv
        dL_dd = ((gmx * Tu * Tw + gmy * Tv * Tw) * f).sum() * (-1.0 / dd)
        G[2] += dL_dd * T9 * Tw * 2.0
    return G


def per_view_then_sum(partials, Ts, As, Rs, signs):
    """The parent's order: one 18-float sum per view, then each view's chain rule, summed over the views."""
    dM, dtn, gop, gcol = np.zeros((3, 3)), np.zeros(3), 0.0, np.zeros(3)
    for v, parts in enumerate(partials):
        ga = np.sum(parts, axis=0)
        dM += (As[v] @ fold_mean2d(ga, Ts[v])).T          # dM[r][k] = sum_c A[k][c] G[c][r]
        dtn += signs[v] * (Rs[v] @ ga[11:14])
        gop += ga[14]
        gcol += ga[15:18]
    return np.concatenate([dM.reshape(9), dtn, [gop], gcol])


def grad_row(g, T, A, R, sign):
    """render_bwd_kernel's grad_row(): one partial's 16-float contribution to the surfel's row."""
    return np.concatenate([(A @ fold_mean2d(g, T)).T.reshape(9), sign * (R @ g[11:14]), g[14:18]])


def rows_then_tail(row, q, sx, sy, scale_modifier, quat_norm_grad):
    """preprocess_bwd_kernel: the 13 gradient columns from the surfel's row."""
    dM = row[0:9].reshape(3, 3)
    dtn = row[9:12]
    nq = np.linalg.norm(q)
    w, x, y, z = q / nq
    Rm = quat_R(q)
    dR = np.stack([dM[0] * sx, dM[1] * sy, dtn], axis=1)    # dR[k][c]
    gs = [(dM[0] * Rm[:, 0]).sum(), (dM[1] * Rm[:, 1]).sum()]
    gq = np.array([
        2 * (z * (dR[1, 0] - dR[0, 1]) + y * (dR[0, 2] - dR[2, 0]) + x * (dR[2, 1] - dR[1, 2])),
        2 * (-2 * x * (dR[1, 1] + dR[2, 2]) + y * (dR[1, 0] + dR[0, 1]) + z * (dR[2, 0] + dR[0, 2]) + w * (dR[2, 1] - dR[1, 2])),
        2 * (x * (dR[1, 0] + dR[0, 1]) - 2 * y * (dR[0, 0] + dR[2, 2]) + z * (dR[2, 1] + dR[1, 2]) + w * (dR[0, 2] - dR[2, 0])),
        2 * (x * (dR[2, 0] + dR[0, 2]) + y * (dR[2, 1] + dR[1, 2]) - 2 * z * (dR[0, 0] + dR[1, 1]) + w * (dR[1, 0] - dR[0, 1]))])
    if quat_norm_grad:
        qh = q / nq
        gq = (gq - qh * (qh @ gq)) / nq
    return np.concatenate([dM[2], [row[12]], scale_modifier * np.array(gs), gq, row[13:16]])


def quat_R(q):
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def _view(rng):
    """A random view matrix (row-vector convention: rotation in [:3,:3], translation in row 3) and projection."""
    Q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
    V = np.eye(4)
    V[:3, :3] = Q
    V[3, :3] = rng.standard_normal(3) * 0.2 + [0.0, 0.0, 2.0]
    return V.reshape(16), rng.standard_normal(16)


@pytest.mark.parametrize("quat_norm_grad", [0, 1])
@pytest.mark.parametrize("seed", range(4))
def test_transform_then_sum_equals_sum_then_transform(seed, quat_norm_grad):
    rng = np.random.default_rng(seed)
    W, H, sm = 112, 96, 1.3
    q = rng.standard_normal(4) * 1.5
    sx, sy = sm * rng.uniform(0.01, 0.05, 2)
    R = quat_R(q)
    p = rng.uniform(-0.4, 0.4, 3)
    n_views = 4
    Ts, As, Rs, signs, partials = [], [], [], [], []
    for v in range(n_views):
        vm, pm = _view(rng)
        if v != 2:
            # camera-space position = c * normal: c = -1 faces the camera, +1 faces away, 0 gives cosv == 0 exactly
            c = {0: -1.0, 1: 1.0, 3: 0.0}[v]
            V = vm.reshape(4, 4)
            V[3, :3] = -(p @ V[:3, :3]) + c * (R[:, 2] @ V[:3, :3])
            vm = V.reshape(16)
        T = rng.standard_normal((3, 3)) * [[50.0], [50.0], [1.0]]
        T[2, 2] = 2.0 + rng.uniform()          # Tw = (x, y, depth): 9 Tw0^2 + 9 Tw1^2 - Tw2^2 away from 0
        n_tiles = 5
        parts = rng.standard_normal((n_tiles, 18))
        parts[::2, 9:11] = 0.0                 # tiles whose records all took the 3-D branch: no mean-2D term
        partials.append(parts)
        Ts.append(T)
        As.append(view_A(pm, W, H))
        Rs.append(vm.reshape(4, 4)[:3, :3])
        signs.append(normal_sign(vm, p, R))
    assert signs[0] == 1.0 and signs[1] == -1.0 and signs[3] == -1.0
    row_old = per_view_then_sum(partials, Ts, As, Rs, signs)
    row_new = np.zeros(16)
    for v in range(n_views):
        for g in partials[v]:
            row_new += grad_row(g, Ts[v], As[v], Rs[v], signs[v])
    scale = np.abs(row_old).max()
    assert np.abs(row_new - row_old).max() <= 1e-12 * scale
    out_old = rows_then_tail(row_old, q, sx, sy, sm, quat_norm_grad)
    out_new = rows_then_tail(row_new, q, sx, sy, sm, quat_norm_grad)
    assert np.abs(out_new - out_old).max() <= 1e-12 * np.abs(out_old).max()
