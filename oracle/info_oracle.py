"""numpy restatement of SIVO's information-based map-point selection: the loop of Tracking::StereoInitialization (Tracking.cc:470-520,
threshold 0) and Tracking::CreateNewKeyFrame (Tracking.cc:953-1000, threshold mThEntropyReduction) with the helpers it calls
(sivo_helpers.cpp:64-88 computeStereoJacobianPose, :160-181 computeStereoCovariance, :199-218 computeStereoMutualInformation).

The rule, for semantic key j with keypoint k, depth z = depth[j], entropy H and s2 = sigma2[k.octave] (GetScaleSigmaSquares):
1. valid iff z > 0 (NaN is invalid, as the reference's `!(z > 0)`) and 0 <= octave < nlevels; an invalid key gets world = NaN x 3
   and reduction = NaN and is never selected.
2. world = Frame::UnprojectStereo (Frame.cc:631-645) in float32: x = ((u - cx) * z) * invfx, y = ((v - cy) * z) * invfy,
   w_r = ((Rwc[r,0] * x + Rwc[r,1] * y) + Rwc[r,2] * z) + Ow[r] -- what cv::gemm(Rwc, xc, 1, Ow, 1) computes (tests pin it).
3. J = computeStereoJacobianPose(fx, fy, mb, wX, wY, wZ) in float64, each expression left to right; all zeros when wZ == 0.  The
   reference passes the WORLD point where the helper expects camera coordinates; the two agree only at the identity pose.
4. M (9 x 9) = [[S, S J^T], [J S, (J S) J^T + s2 I]] with S = Sigma_cw; each product entry summed over k ascending, starting from
   the first product.
5. MI = 0.5 * log2((det S * det M33) / det M): the 3 x 3 det by cofactors along the first row, the 6 x 6 / 9 x 9 by LU with partial
   pivoting (first row with the largest |a|; a zero pivot column is skipped; product of the diagonal in order, times the sign).
6. reduction = MI - H; selected iff reduction > threshold (IEEE: NaN never), listed in ascending j.
Every operation is one IEEE float32 / float64 operation (numpy elementwise arithmetic, no fused multiply-add); the loops run over
the matrix entries and are vectorised over the keys only.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

F32, F64 = np.float32, np.float64


@dataclass
class Camera:
    """The Frame members the loop reads (Frame.cc:166-172: fx, fy, cx, cy, invfx = 1 / fx, invfy, mb = mbf / fx; mRwc, mOw,
    mSigmacw)."""
    fx: float
    fy: float
    cx: float
    cy: float
    mb: float
    Rwc: np.ndarray
    Ow: np.ndarray
    sigma_cw: np.ndarray

    def __post_init__(self):
        self.fx, self.fy, self.cx, self.cy, self.mb = (F32(v) for v in (self.fx, self.fy, self.cx, self.cy, self.mb))
        self.invfx, self.invfy = F32(1) / self.fx, F32(1) / self.fy
        self.Rwc = np.asarray(self.Rwc, F32).reshape(3, 3)
        self.Ow = np.asarray(self.Ow, F32).reshape(3)
        self.sigma_cw = np.asarray(self.sigma_cw, F64).reshape(6, 6)


def unproject(u, v, z, cam: Camera) -> np.ndarray:
    """Frame::UnprojectStereo for arrays of keys (float32 throughout) -> (n, 3)."""
    u, v, z = (np.asarray(a, F32) for a in (u, v, z))
    x = ((u - cam.cx) * z) * cam.invfx
    y = ((v - cam.cy) * z) * cam.invfy
    xc = (x, y, z)
    R, o = cam.Rwc, cam.Ow
    return np.stack([((R[r, 0] * xc[0] + R[r, 1] * xc[1]) + R[r, 2] * xc[2]) + o[r] for r in range(3)], axis=1)


def stereo_jacobian_pose(fx, fy, bl, X, Y, Z) -> np.ndarray:
    """computeStereoJacobianPose (sivo_helpers.cpp:64-88) -> (n, 3, 6) float64, zero rows where Z == 0."""
    fx, fy, bl = F64(fx), F64(fy), F64(bl)
    X, Y, Z = (np.asarray(a, F64) for a in (X, Y, Z))
    J = np.zeros(X.shape + (3, 6), F64)
    nz = Z != 0
    X, Y, Z = X[nz], Y[nz], Z[nz]
    ZZ = Z * Z
    J[nz, 0, 0] = fx / Z
    J[nz, 0, 2] = -fx * X / ZZ
    J[nz, 0, 3] = -fx * X * Y / ZZ
    J[nz, 0, 4] = fx * (1.0 + (X * X) / ZZ)
    J[nz, 0, 5] = -fx * Y / Z
    J[nz, 1, 1] = fy / Z
    J[nz, 1, 2] = -fy * Y / ZZ
    J[nz, 1, 3] = -fy * (1 + (Y * Y) / ZZ)
    J[nz, 1, 4] = fy * X * Y / ZZ
    J[nz, 1, 5] = fy * X / Z
    J[nz, 2, 0] = fx / Z
    J[nz, 2, 2] = -fx * (X - bl) / ZZ
    J[nz, 2, 3] = -fx * (X - bl) * Y / ZZ
    J[nz, 2, 4] = fx * (1.0 + (X * (X - bl)) / ZZ)
    J[nz, 2, 5] = -fx * Y / Z
    return J


def _matmul(A, B) -> np.ndarray:
    """(n, r, m) x (n, m, c) with each entry summed over k ascending, starting from the first product."""
    out = A[:, :, :1] * B[:, :1, :]
    for k in range(1, A.shape[2]):
        out = out + A[:, :, k:k + 1] * B[:, k:k + 1, :]
    return out


def stereo_covariance(S, J, sigma2) -> np.ndarray:
    """computeStereoCovariance (sivo_helpers.cpp:160-181) -> (n, 9, 9); R = sigma2 * I (sigma2 per key)."""
    n = len(J)
    Sn = np.broadcast_to(np.asarray(S, F64), (n, 6, 6))
    Jt = np.swapaxes(J, 1, 2)
    JS = _matmul(J, Sn)
    R = np.asarray(sigma2, F64)[:, None, None] * np.eye(3)[None]
    M = np.empty((n, 9, 9), F64)
    M[:, :6, :6] = Sn
    M[:, 6:, 6:] = _matmul(JS, Jt) + R
    M[:, :6, 6:] = _matmul(Sn, Jt)
    M[:, 6:, :6] = JS
    return M


def det3_cofactor(A) -> np.ndarray:
    """(n, 3, 3) -> det by cofactor expansion along the first row."""
    a = np.asarray(A, F64)
    return (a[:, 0, 0] * (a[:, 1, 1] * a[:, 2, 2] - a[:, 1, 2] * a[:, 2, 1]) - a[:, 0, 1] * (a[:, 1, 0] * a[:, 2, 2] - a[:, 1, 2] * a[:, 2, 0])
            + a[:, 0, 2] * (a[:, 1, 0] * a[:, 2, 1] - a[:, 1, 1] * a[:, 2, 0]))


def det_lu(A) -> np.ndarray:
    """(n, N, N) -> det by LU with partial pivoting: in column c the pivot is the first row r >= c with the largest |a[r, c]| (a NaN
    is never preferred to the row already held, so a NaN diagonal keeps its row); a zero pivot column is skipped; rows below are
    divided by the pivot and the trailing block gets the rank-1 update; det = product of the diagonal in order, times the sign."""
    a = np.array(A, F64, copy=True)
    n, N, _ = a.shape
    neg = np.zeros(n, bool)
    rows = np.arange(n)
    for c in range(N):
        col = np.abs(a[:, c:, c])
        col = np.where(np.isnan(col), -np.inf, col)
        p = c + np.argmax(col, axis=1)
        p = np.where(np.isnan(a[:, c, c]), c, p)
        best = np.abs(a[rows, p, c])
        act = best != 0.0
        sw = act & (p != c)
        if sw.any():
            top = a[rows[sw], c, c:].copy()
            a[rows[sw], c, c:] = a[rows[sw], p[sw], c:]
            a[rows[sw], p[sw], c:] = top
            neg ^= sw
        piv = a[:, c, c]
        for r in range(c + 1, N):
            with np.errstate(all="ignore"):  # skipped columns (act False) divide by their zero pivot; the result is dropped
                l = a[:, r, c] / piv
                upd = a[:, r, c + 1:] - l[:, None] * a[:, c, c + 1:]
            a[act, r, c + 1:] = upd[act]
    d = a[:, 0, 0]
    for i in range(1, N):
        d = d * a[:, i, i]
    return np.where(neg, d * -1.0, d)


def info_terms(kps, depth, sigma2_table, cam: Camera):
    """Per key: (world (n, 3) float32, det S, det M33, det M, valid); NaN for invalid keys."""
    kps = np.asarray(kps)
    z = np.asarray(depth, F32)
    n = len(z)
    octave = kps["octave"].astype(np.int64)
    sigma2_table = np.asarray(sigma2_table, F32)
    valid = (z > 0) & (octave >= 0) & (octave < len(sigma2_table))
    world = np.full((n, 3), np.nan, F32)
    dets = [np.full(n, np.nan, F64) for _ in range(3)]
    if valid.any():
        w = unproject(kps["x"][valid], kps["y"][valid], z[valid], cam)
        world[valid] = w
        J = stereo_jacobian_pose(cam.fx, cam.fy, cam.mb, w[:, 0].astype(F64), w[:, 1].astype(F64), w[:, 2].astype(F64))
        s2 = sigma2_table[octave[valid]].astype(F64)
        M = stereo_covariance(cam.sigma_cw, J, s2)
        dets[0][valid] = det_lu(np.broadcast_to(cam.sigma_cw, (1, 6, 6)))[0]
        dets[1][valid] = det3_cofactor(M[:, 6:, 6:])
        dets[2][valid] = det_lu(M)
    return world, dets[0], dets[1], dets[2], valid


def mutual_information(det_state, det_meas, det_joint) -> np.ndarray:
    """computeStereoMutualInformation (sivo_helpers.cpp:199-218)."""
    with np.errstate(all="ignore"):
        return 0.5 * np.log2(det_state * det_meas / det_joint)


def select(kps, depth, entropy, sigma2_table, cam: Camera, threshold: float):
    """The Tracking.cc loop -> (world (n, 3) float32, reduction float64, selected int32 ascending)."""
    world, ds, dm, dj, valid = info_terms(kps, depth, sigma2_table, cam)
    red = np.full(len(world), np.nan, F64)
    red[valid] = mutual_information(ds[valid], dm[valid], dj[valid]) - np.asarray(entropy, F64)[valid]
    with np.errstate(invalid="ignore"):
        sel = np.flatnonzero(red > F64(threshold)).astype(np.int32)
    return world, red, sel


def update_state_covariance_motion(prev, R, t) -> np.ndarray:
    """updateStateCovarianceMotion (sivo_helpers.cpp:244-268): F = I + [[R, [t]x R], [0, R]]; F P F^T + 0.01 I.  Used to make
    realistic pose covariances for the tests (numpy matmul: its summation order is not part of any rule)."""
    R = np.asarray(R, F64)
    t = np.asarray(t, F64)
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]], F64)
    adj = np.zeros((6, 6), F64)
    adj[:3, :3] = R
    adj[:3, 3:] = tx @ R
    adj[3:, 3:] = R
    F = np.eye(6) + adj
    return F @ np.asarray(prev, F64) @ F.T + np.eye(6) * 0.01
