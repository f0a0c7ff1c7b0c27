"""float64 loop-level restatement of match-interestpoints (PARITY_GAPS M1-M9): local descriptors by sorting, the
descriptor distance by explicit subset enumeration, RANSAC drawing the same samples as the product, and the
translation / rigid (Horn quaternion) / affine (centred normal equations) / interpolated fits.  Test oracle only.

Distances are spelled ((dx*dx + dy*dy) + dz*dz) and subset sums left to right, the operations the device performs, so
indices and values compare exactly."""
import itertools

import numpy as np

FLOAT_MAX = float(np.finfo(np.float32).max)
RANSAC_SEED = 69997
MIN_MATCHES = {"IDENTITY": 0, "TRANSLATION": 1, "RIGID": 3, "AFFINE": 4}


def sq3(d):
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def knn(xyz, k, chunk=256):
    """M4: (idx (n, k), d2 (n, k)) -- for every point the first k of the OTHER points sorted by (squared distance,
    index).  Rows are taken from the candidates within the k-th smallest distance (all of its ties), then sorted."""
    xyz = np.asarray(xyz, dtype=np.float64).reshape(-1, 3)
    n = len(xyz)
    idx = np.full((n, k), -1, dtype=np.int64)
    d2 = np.full((n, k), np.inf)
    if n <= k:
        return idx, d2
    for r0 in range(0, n, chunk):
        rows = np.arange(r0, min(n, r0 + chunk))
        D = sq3(xyz[None, :, :] - xyz[rows, None, :])
        D[np.arange(len(rows)), rows] = np.inf
        kth = np.partition(D, k - 1, axis=1)[:, k - 1]
        for i, r in enumerate(rows):
            cand = np.nonzero(D[i] <= kth[i])[0]
            order = np.lexsort((cand, D[i, cand]))[:k]
            idx[r], d2[r] = cand[order], D[i, cand[order]]
    return idx, d2


def knn_full_sort(xyz, k):
    """M4 by a full sort of every row (small sets)."""
    xyz = np.asarray(xyz, dtype=np.float64).reshape(-1, 3)
    n = len(xyz)
    idx = np.full((n, k), -1, dtype=np.int64)
    d2 = np.full((n, k), np.inf)
    if n <= k:
        return idx, d2
    for p in range(n):
        rows = sorted((float(sq3(xyz[q] - xyz[p])), q) for q in range(n) if q != p)[:k]
        idx[p] = [q for _, q in rows]
        d2[p] = [d for d, _ in rows]
    return idx, d2


def descriptors(xyz, idx):
    """The relative vectors q_j - p, (n, k, 3)."""
    xyz = np.asarray(xyz, dtype=np.float64).reshape(-1, 3)
    return xyz[idx] - xyz[:, None, :]


def subsets(n, k):
    """The C(k, n) neighbour subsets in lexicographic order of rank."""
    return list(itertools.combinations(range(k), n))


def descriptor_distance(u, v, n):
    """M5 for one pair: min over subset pairs (s of u, t of v) of sum_j |u_{s_j} - v_{t_j}|^2."""
    k = len(u)
    best = np.inf
    for s in subsets(n, k):
        for t in subsets(n, k):
            acc = sq3(u[s[0]] - v[t[0]])
            for j in range(1, n):
                acc = acc + sq3(u[s[j]] - v[t[j]])
            best = min(best, acc)
    return best


def match(xyz_a, xyz_b, num_neighbors=3, redundancy=1, search_radius=None, chunk=64):
    """The exhaustive search A -> B: (best_b (nA,), best, second) as bs_descriptors_match defines them."""
    k = num_neighbors + redundancy
    xa = np.asarray(xyz_a, dtype=np.float64).reshape(-1, 3)
    xb = np.asarray(xyz_b, dtype=np.float64).reshape(-1, 3)
    na = len(xa)
    best_b = np.full(na, -1, dtype=np.int64)
    best = np.full(na, np.inf)
    second = np.full(na, np.inf)
    if na <= k or len(xb) <= k:
        return best_b, best, second
    u = descriptors(xa, knn(xa, k)[0])
    v = descriptors(xb, knn(xb, k)[0])
    subs = subsets(num_neighbors, k)
    for a0 in range(0, na, chunk):
        ua = u[a0:a0 + chunk]
        # d[a, b, i, j] = |u_i - v_j|^2
        d = sq3(ua[:, None, :, None, :] - v[None, :, None, :, :])
        D = np.full(d.shape[:2], np.inf)
        for s in subs:
            for t in subs:
                acc = d[:, :, s[0], t[0]]
                for j in range(1, num_neighbors):
                    acc = acc + d[:, :, s[j], t[j]]
                D = np.minimum(D, acc)
        if search_radius is not None:
            inside = sq3(xb[None, :, :] - xa[a0:a0 + chunk, None, :]) <= search_radius * search_radius
            D = np.where(inside, D, np.inf)
        for i in range(len(ua)):
            row = D[i]
            if not np.isfinite(row).any():
                continue
            bi = int(np.argmin(row))
            best_b[a0 + i], best[a0 + i] = bi, row[bi]
            rest = np.delete(row, bi)
            second[a0 + i] = rest.min() if len(rest) else np.inf
    return best_b, best, second


def ratio_test(best_b, best, second, significance=3.0):
    """M6: the a whose (a, best_b[a]) is kept."""
    return [a for a in range(len(best_b))
            if best_b[a] >= 0 and best[a] < FLOAT_MAX and second[a] > significance * best[a]]


# ------------------------------------------------------------------------------------------ model fits
def fit_translation(a, b):
    M = np.hstack([np.eye(3), (b.mean(axis=0) - a.mean(axis=0))[:, None]])
    return M


def fit_rigid(a, b):
    """Horn's quaternion solution: the eigenvector of the largest eigenvalue of the symmetric 4 x 4 matrix N."""
    ca, cb = a.mean(axis=0), b.mean(axis=0)
    ac, bc = a - ca, b - cb
    sv = np.linalg.svd(ac, compute_uv=False)
    if not sv[1] > 1e-12 * max(sv[0], 1e-300):
        return None
    S = ac.T @ bc
    (xx, xy, xz), (yx, yy, yz), (zx, zy, zz) = S
    N = np.array([[xx + yy + zz, yz - zy, zx - xz, xy - yx],
                  [yz - zy, xx - yy - zz, xy + yx, zx + xz],
                  [zx - xz, xy + yx, -xx + yy - zz, yz + zy],
                  [xy - yx, zx + xz, yz + zy, -xx - yy + zz]])
    w, V = np.linalg.eigh(N)
    q0, q1, q2, q3 = V[:, np.argmax(w)]
    R = np.array([[q0 * q0 + q1 * q1 - q2 * q2 - q3 * q3, 2 * (q1 * q2 - q0 * q3), 2 * (q1 * q3 + q0 * q2)],
                  [2 * (q2 * q1 + q0 * q3), q0 * q0 - q1 * q1 + q2 * q2 - q3 * q3, 2 * (q2 * q3 - q0 * q1)],
                  [2 * (q3 * q1 - q0 * q2), 2 * (q3 * q2 + q0 * q1), q0 * q0 - q1 * q1 - q2 * q2 + q3 * q3]])
    return np.hstack([R, (cb - R @ ca)[:, None]])


def fit_affine(a, b):
    """Centred normal equations: P = sum a_c a_c^T, Q = sum a_c b_c^T, A = (P^-1 Q)^T; None when P is singular."""
    ca, cb = a.mean(axis=0), b.mean(axis=0)
    ac, bc = a - ca, b - cb
    P, Q = ac.T @ ac, ac.T @ bc
    det = np.linalg.det(P)
    if not (np.isfinite(det) and det > 1e-12 * (np.trace(P) / 3.0) ** 3):
        return None
    A = np.linalg.solve(P, Q).T
    return np.hstack([A, (cb - A @ ca)[:, None]])


def fit(kind, a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    if kind == "IDENTITY":
        return np.hstack([np.eye(3), np.zeros((3, 1))])
    return {"TRANSLATION": fit_translation, "RIGID": fit_rigid, "AFFINE": fit_affine}[kind](a, b)


def fit_model(tm, rm, lam, a, b):
    """createModelInstance: tm alone (rm NONE) or the interpolated (1 - lam) M_tm + lam M_rm."""
    M = fit(tm, a, b)
    if rm == "NONE" or M is None:
        return M
    R = fit(rm, a, b)
    return None if R is None else (1.0 - lam) * M + lam * R


def min_matches(tm, rm):
    return MIN_MATCHES[tm] if rm == "NONE" else max(MIN_MATCHES[tm], MIN_MATCHES[rm])


def residuals(M, a, b):
    return np.linalg.norm(a @ M[:, :3].T + M[:, 3] - b, axis=1)


def ransac(a, b, tm="AFFINE", rm="RIGID", lam=0.1, iterations=10000, max_error=5.0, min_inlier_ratio=0.1,
           min_num_inliers=12, seed=RANSAC_SEED):
    """M7 + M8, one hypothesis at a time: row h of the key stream is rng.random((1, M)); the sample is the m smallest
    keys.  Returns (sorted inlier indices, model) or ([], None)."""
    a, b = np.asarray(a, dtype=np.float64).reshape(-1, 3), np.asarray(b, dtype=np.float64).reshape(-1, 3)
    n = len(a)
    m = max(min_matches(tm, rm), 1)
    if n < m:
        return [], None
    rng = np.random.default_rng(seed)
    best_n, best_in = -1, None
    for _ in range(iterations):
        keys = rng.random((1, n))[0]
        s = np.argsort(keys, kind="stable")[:m]
        M = fit_model(tm, rm, lam, a[s], b[s])
        if M is None:
            continue
        inl = np.nonzero(residuals(M, a, b) < max_error)[0]
        if len(inl) > best_n:
            best_n, best_in = len(inl), inl
    if best_in is None or best_n < m:
        return [], None
    inl = best_in
    while True:
        n0 = len(inl)
        M = fit_model(tm, rm, lam, a[inl], b[inl])
        if M is None:
            return [], None
        r = residuals(M, a[inl], b[inl])
        inl = inl[r <= 4.0 * np.median(r)]
        if len(inl) == n0 or len(inl) < m:
            break
    if len(inl) < m or len(inl) < min_num_inliers or len(inl) < min_inlier_ratio * n:
        return [], None
    M = fit_model(tm, rm, lam, a[inl], b[inl])
    if M is None:
        return [], None
    return sorted(int(i) for i in inl), M
