"""Host side of `match-interestpoints` (PRECISE_TRANSLATION): the ratio test on the device's descriptor search, RANSAC
and its filter, and the model fits of createModelInstance (J/abstractcmdline/AbstractRegistration.java:110-140), in
vectorised float64 numpy.  PARITY_GAPS M6-M8 state the choices.

A model is a 3 x 4 matrix [A | t] mapping a point of view A (world) to its partner in view B (world)."""
from __future__ import annotations

import numpy as np

#: RGLDMParameters.differenceThreshold: a best descriptor distance must be below Float.MAX_VALUE
FLOAT_MAX = float(np.finfo(np.float32).max)
#: seed of the RANSAC sampler, one generator per matching task (M7)
RANSAC_SEED = 69997
#: mpicbg filterRansac maxTrust: keep residuals <= 4 * median
FILTER_MAX_TRUST = 4.0
#: hypotheses per vectorised RANSAC chunk (rows of rng.random((rows, M)); the stream does not depend on it)
RANSAC_CHUNK = 256

MIN_MATCHES = {"IDENTITY": 0, "TRANSLATION": 1, "RIGID": 3, "AFFINE": 4}
TRANSFORMATION_MODELS = ("TRANSLATION", "RIGID", "AFFINE")
REGULARIZATION_MODELS = ("NONE", "IDENTITY", "TRANSLATION", "RIGID", "AFFINE")


class Model:
    """createModelInstance: the transformation model alone (regularization NONE), or the interpolated model
    (1 - lambda) M_tm + lambda M_rm fitted to the same matches."""

    def __init__(self, transformation="AFFINE", regularization="RIGID", lam=0.1):
        transformation, regularization = transformation.upper(), regularization.upper()
        if transformation not in TRANSFORMATION_MODELS:
            raise ValueError(f"-tm {transformation}")
        if regularization not in REGULARIZATION_MODELS:
            raise ValueError(f"-rm {regularization}")
        self.tm, self.rm, self.lam = transformation, regularization, float(lam)
        self.min_matches = MIN_MATCHES[self.tm] if self.rm == "NONE" else max(MIN_MATCHES[self.tm],
                                                                             MIN_MATCHES[self.rm])

    def fit(self, a, b, w=None):
        """Batched fit: a, b (H, m, 3) -> (models (H, 3, 4), ok (H,) bool; False = singular / ill-defined).
        ``w`` (H, m): match weights (the solver's fits); None fits every match with weight 1."""
        M, ok = _fit(self.tm, a, b, w)
        if self.rm == "NONE":
            return M, ok
        R, okr = _fit(self.rm, a, b, w)
        return (1.0 - self.lam) * M + self.lam * R, ok & okr


def _fit(kind, a, b, w=None):
    if w is not None:
        return _fit_weighted(kind, a, b, np.asarray(w, dtype=np.float64))
    H = a.shape[0]
    ca, cb = a.mean(axis=1), b.mean(axis=1)
    M = np.zeros((H, 3, 4))
    ok = np.ones(H, dtype=bool)
    if kind == "IDENTITY":
        M[:, :, :3] = np.eye(3)
    elif kind == "TRANSLATION":
        M[:, :, :3] = np.eye(3)
        M[:, :, 3] = cb - ca
    elif kind == "RIGID":
        M[:] = _fit_rigid(a - ca[:, None], b - cb[:, None], ca, cb)
        sv = np.linalg.svd(a - ca[:, None], compute_uv=False)
        ok = sv[:, 1] > 1e-12 * np.maximum(sv[:, 0], 1e-300)            # collinear points do not fix a rotation
    else:
        ac, bc = a - ca[:, None], b - cb[:, None]
        P = np.einsum("hmi,hmj->hij", ac, ac)
        Q = np.einsum("hmi,hmj->hij", ac, bc)
        det = np.linalg.det(P)
        tr = np.trace(P, axis1=1, axis2=2) / 3.0
        ok = np.isfinite(det) & (det > 1e-12 * tr ** 3)
        Ps = np.where(ok[:, None, None], P, np.eye(3))
        A = np.swapaxes(np.linalg.solve(Ps, Q), 1, 2)                 # b_c = A a_c
        M[:, :, :3] = A
        M[:, :, 3] = cb - np.einsum("hij,hj->hi", A, ca)
    return M, ok


def _fit_weighted(kind, a, b, w):
    """The fits of _fit with weighted centroids and moments, as the solver's tiles fit them.  Singular: total weight
    <= 0; RIGID when the centred points are (numerically) collinear, i.e. the second invariant of P = sum w a_c a_c^T is
    <= 1e-12 (trace P)^2; AFFINE with _fit's determinant test on P."""
    H = a.shape[0]
    W = w.sum(axis=1)
    ok = W > 0
    Ws = np.where(ok, W, 1.0)
    ca = np.einsum("hm,hmi->hi", w, a) / Ws[:, None]
    cb = np.einsum("hm,hmi->hi", w, b) / Ws[:, None]
    M = np.zeros((H, 3, 4))
    if kind in ("IDENTITY", "TRANSLATION"):
        M[:, :, :3] = np.eye(3)
        if kind == "TRANSLATION":
            M[:, :, 3] = cb - ca
        return M, ok if kind == "TRANSLATION" else np.ones(H, dtype=bool)
    ac, bc = a - ca[:, None], b - cb[:, None]
    P = np.einsum("hm,hmi,hmj->hij", w, ac, ac)
    S = np.einsum("hm,hmi,hmj->hij", w, ac, bc)
    tr = np.trace(P, axis1=1, axis2=2)
    if kind == "RIGID":
        i2 = (P[:, 0, 0] * P[:, 1, 1] - P[:, 0, 1] * P[:, 1, 0] + P[:, 0, 0] * P[:, 2, 2] - P[:, 0, 2] * P[:, 2, 0] +
              P[:, 1, 1] * P[:, 2, 2] - P[:, 1, 2] * P[:, 2, 1])
        ok &= i2 > 1e-12 * tr * tr
        return _rigid_from_cov(S, ca, cb), ok
    det = np.linalg.det(P)
    ok &= np.isfinite(det) & (det > 1e-12 * (tr / 3.0) ** 3)
    Ps = np.where(ok[:, None, None], P, np.eye(3))
    A = np.swapaxes(np.linalg.solve(Ps, S), 1, 2)
    M[:, :, :3] = A
    M[:, :, 3] = cb - np.einsum("hij,hj->hi", A, ca)
    return M, ok


def _fit_rigid(ac, bc, ca, cb):
    """Horn's closed form: the rotation is the quaternion of the largest eigenvalue of the 4 x 4 matrix N of the
    centred cross-covariance S = sum a b^T."""
    return _rigid_from_cov(np.einsum("hmi,hmj->hij", ac, bc), ca, cb)


def _rigid_from_cov(S, ca, cb):
    xx, xy, xz = S[:, 0, 0], S[:, 0, 1], S[:, 0, 2]
    yx, yy, yz = S[:, 1, 0], S[:, 1, 1], S[:, 1, 2]
    zx, zy, zz = S[:, 2, 0], S[:, 2, 1], S[:, 2, 2]
    N = np.stack([np.stack([xx + yy + zz, yz - zy, zx - xz, xy - yx], -1),
                  np.stack([yz - zy, xx - yy - zz, xy + yx, zx + xz], -1),
                  np.stack([zx - xz, xy + yx, -xx + yy - zz, yz + zy], -1),
                  np.stack([xy - yx, zx + xz, yz + zy, -xx - yy + zz], -1)], -2)
    _, vec = np.linalg.eigh(N)
    q0, q1, q2, q3 = (vec[:, i, -1] for i in range(4))
    R = np.stack([np.stack([q0 * q0 + q1 * q1 - q2 * q2 - q3 * q3, 2 * (q1 * q2 - q0 * q3), 2 * (q1 * q3 + q0 * q2)], -1),
                  np.stack([2 * (q2 * q1 + q0 * q3), q0 * q0 - q1 * q1 + q2 * q2 - q3 * q3, 2 * (q2 * q3 - q0 * q1)], -1),
                  np.stack([2 * (q3 * q1 - q0 * q2), 2 * (q3 * q2 + q0 * q1), q0 * q0 - q1 * q1 - q2 * q2 + q3 * q3], -1)],
                 -2)
    M = np.zeros((len(R), 3, 4))
    M[:, :, :3] = R
    M[:, :, 3] = cb - np.einsum("hij,hj->hi", R, ca)
    return M


def apply(M, p):
    """Model(s) (..., 3, 4) applied to points (n, 3)."""
    return np.einsum("...ij,nj->...ni", M[..., :3], p) + M[..., None, :, 3]


def ratio_test(best_b, best, second, significance):
    """M6: indices a whose match (a, best_b[a]) survives RGLDM's ratio test."""
    best_b = np.asarray(best_b)
    keep = (best_b >= 0) & (np.asarray(best) < FLOAT_MAX) & (np.asarray(second) > significance * np.asarray(best))
    return np.nonzero(keep)[0]


def ransac(a, b, model: Model, iterations=10000, max_error=5.0, min_inlier_ratio=0.1, min_num_inliers=12,
           seed=RANSAC_SEED, chunk=RANSAC_CHUNK):
    """M7 + M8 on candidate matches a[i] <-> b[i] ((M, 3) each).  Returns (sorted inlier indices, model 3 x 4) or
    (empty, None) when the pair is rejected."""
    a = np.asarray(a, dtype=np.float64).reshape(-1, 3)
    b = np.asarray(b, dtype=np.float64).reshape(-1, 3)
    M, m = len(a), model.min_matches
    none = (np.zeros(0, dtype=np.int64), None)
    if M < max(m, 1):
        return none
    rng = np.random.default_rng(seed)
    best_n, best_in = -1, None
    for h0 in range(0, iterations, chunk):
        rows = min(chunk, iterations - h0)
        keys = rng.random((rows, M))
        idx = np.argsort(keys, axis=1, kind="stable")[:, :max(m, 1)]
        Ms, ok = model.fit(a[idx], b[idx])
        if not ok.any():
            continue
        res = np.linalg.norm(apply(Ms, a) - b[None], axis=2)
        cnt = np.where(ok, (res < max_error).sum(axis=1), -1)
        h = int(np.argmax(cnt))                                   # the first hypothesis with most inliers
        if cnt[h] > best_n:
            best_n, best_in = int(cnt[h]), np.nonzero(res[h] < max_error)[0]
    if best_in is None or best_n < max(m, 1):
        return none
    inl = best_in
    while True:                                                   # M8: filterRansac
        n0 = len(inl)
        Mf, ok = model.fit(a[inl][None], b[inl][None])
        if not ok[0]:
            return none
        r = np.linalg.norm(apply(Mf[0], a[inl]) - b[inl], axis=1)
        inl = inl[r <= FILTER_MAX_TRUST * np.median(r)]
        if len(inl) == n0 or len(inl) < max(m, 1):
            break
    if len(inl) < max(m, 1) or len(inl) < min_num_inliers or len(inl) < min_inlier_ratio * M:
        return none
    Mf, ok = model.fit(a[inl][None], b[inl][None])
    if not ok[0]:
        return none
    return np.sort(inl), Mf[0]
