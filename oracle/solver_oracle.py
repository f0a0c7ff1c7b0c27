"""float64 restatement of the solver's relaxation (bs_solve_tiles, PARITY_GAPS S2/S6): weighted translation / rigid
(Horn quaternion) / affine fits and their interpolation with a regularizer, the multicolour Gauss-Seidel sweep, the
per-match distances, tile and link errors and the stopping rule.  Every fit is taken from the per-match sums over the
tile's matches with its partners' current models applied, not from link moments, so comparing it with the device also
checks the device's moment factorisation.  Test oracle only."""
import numpy as np

MIN_MATCHES = {"IDENTITY": 0, "TRANSLATION": 1, "RIGID": 3, "AFFINE": 4}


def fit(kind, x, y, w):
    """Weighted fit of y ~ M x ((n, 3) each, weights (n,)): (3 x 4 model, ok)."""
    W = w.sum()
    M = np.eye(3, 4)
    if kind == "IDENTITY":
        return M, True
    if not W > 0:
        return M, False
    cx, cy = (w[:, None] * x).sum(0) / W, (w[:, None] * y).sum(0) / W
    if kind == "TRANSLATION":
        M[:, 3] = cy - cx
        return M, True
    xc, yc = x - cx, y - cy
    P = (w[:, None, None] * xc[:, :, None] * xc[:, None, :]).sum(0)
    S = (w[:, None, None] * xc[:, :, None] * yc[:, None, :]).sum(0)
    tr = np.trace(P)
    if kind == "RIGID":
        i2 = P[0, 0] * P[1, 1] - P[0, 1] ** 2 + P[0, 0] * P[2, 2] - P[0, 2] ** 2 + P[1, 1] * P[2, 2] - P[1, 2] ** 2
        (xx, xy, xz), (yx, yy, yz), (zx, zy, zz) = S
        N = np.array([[xx + yy + zz, yz - zy, zx - xz, xy - yx],
                      [yz - zy, xx - yy - zz, xy + yx, zx + xz],
                      [zx - xz, xy + yx, -xx + yy - zz, yz + zy],
                      [xy - yx, zx + xz, yz + zy, -xx - yy + zz]])
        q0, q1, q2, q3 = np.linalg.eigh(N)[1][:, -1]
        A = np.array([[q0 * q0 + q1 * q1 - q2 * q2 - q3 * q3, 2 * (q1 * q2 - q0 * q3), 2 * (q1 * q3 + q0 * q2)],
                      [2 * (q2 * q1 + q0 * q3), q0 * q0 - q1 * q1 + q2 * q2 - q3 * q3, 2 * (q2 * q3 - q0 * q1)],
                      [2 * (q3 * q1 - q0 * q2), 2 * (q3 * q2 + q0 * q1), q0 * q0 - q1 * q1 - q2 * q2 + q3 * q3]])
        ok = i2 > 1e-12 * tr * tr
    else:
        det = np.linalg.det(P)
        ok = bool(np.isfinite(det) and det > 1e-12 * (tr / 3.0) ** 3)
        if not ok:
            return M, False
        A = np.linalg.solve(P, S).T
    M[:, :3] = A
    M[:, 3] = cy - A @ cx
    return M, bool(ok)


def fit_model(tm, rm, lam, x, y, w):
    """createModelInstance: the transformation model, or (1 - lam) M_tm + lam M_rm; too few matches fail."""
    need = MIN_MATCHES[tm] if rm == "NONE" else max(MIN_MATCHES[tm], MIN_MATCHES[rm])
    if len(x) < max(need, 1):
        return None
    M, ok = fit(tm, x, y, w)
    if rm != "NONE":
        R, okr = fit(rm, x, y, w)
        M, ok = (1.0 - lam) * M + lam * R, ok and okr
    return M if ok else None


def proceed(errors, max_error, width):
    i = len(errors)
    if i <= width:
        return True
    go = errors[-1] > max_error
    d = width
    while d >= 1:
        go = go or abs((errors[-1] - errors[-1 - d]) / d) > 1e-4
        d //= 2
    return go


def apply(M, x):
    return x @ M[:, :3].T + M[:, 3]


def solve_tiles(colour_offsets, colour_tiles, fixed, links, match_offsets, p, q, w, models, transformation="AFFINE",
                regularization="RIGID", lam=0.1, max_error=5.0, max_iterations=10000, max_plateau_width=200):
    """Same arguments and results as bsgpu.Context.solve_tiles: (models (T, 3, 4), stats, tile_error (T,),
    link_mean (L,), link_max (L,))."""
    tm, rm = transformation.upper(), regularization.upper()
    M = np.array(models, dtype=np.float64).reshape(-1, 3, 4).copy()
    T, L = len(M), len(links)
    links = np.asarray(links).reshape(-1, 2)
    off = np.asarray(match_offsets)
    link_of = np.repeat(np.arange(L), np.diff(off))
    ma, mb = links[link_of, 0], links[link_of, 1]
    own = []
    for t in range(T):
        sa, sb = ma == t, mb == t
        own.append((np.concatenate([p[sa], q[sb]]), np.concatenate([mb[sa], ma[sb]]), np.concatenate([q[sa], p[sb]]),
                    np.concatenate([w[sa], w[sb]])))
    errors, skipped, stopped = [], 0, False
    tile_err = np.zeros(T)
    link_mean, link_max = np.zeros(L), np.zeros(L)
    for it in range(1, int(max_iterations) + 1):
        for c in range(len(colour_offsets) - 1):
            for t in colour_tiles[colour_offsets[c]:colour_offsets[c + 1]]:
                if fixed[t]:
                    continue
                x, u, z, ww = own[t]
                y = np.einsum("nij,nj->ni", M[u][:, :, :3], z) + M[u][:, :, 3]
                F = fit_model(tm, rm, lam, x, y, ww)
                if F is None:
                    skipped += 1
                else:
                    M[t] = F
        d = np.linalg.norm(np.einsum("nij,nj->ni", M[ma][:, :, :3], p) + M[ma][:, :, 3] -
                           np.einsum("nij,nj->ni", M[mb][:, :, :3], q) - M[mb][:, :, 3], axis=1)
        swd, sw = np.bincount(link_of, w * d, L), np.bincount(link_of, w, L)
        link_mean = np.where(sw > 0, swd / np.where(sw > 0, sw, 1), 0.0)
        link_max = np.zeros(L)
        np.maximum.at(link_max, link_of, d)
        tswd, tsw = np.bincount(links.ravel(), np.repeat(swd, 2), T), np.bincount(links.ravel(), np.repeat(sw, 2), T)
        tile_err = np.where(tsw > 0, tswd / np.where(tsw > 0, tsw, 1), 0.0)
        errors.append(float(tile_err.mean()))
        if not proceed(errors, max_error, max_plateau_width):
            stopped = True
            break
    stats = dict(iterations=len(errors), error=errors[-1] if errors else 0.0, skipped_fits=skipped, stopped=stopped)
    return M, stats, tile_err, link_mean, link_max
