"""CPU: the information-selection oracle (oracle/info_oracle.py) against OpenCV's gemm, numpy's determinant and the closed form
of the stereo mutual information."""
import cv2
import numpy as np

from oracle import info_oracle as I
from oracle.mapping_scene import rotation

KITTI_FX, KITTI_CX, KITTI_CY, KITTI_MBF = 718.856, 607.1928, 185.2157, 386.1448


def random_spd(rng, n, scale=1.0):
    a = rng.standard_normal((n, n))
    return scale * (a @ a.T + n * np.eye(n))


def camera(R=np.eye(3), Ow=(0, 0, 0), sigma=1e-6 * np.eye(6)):
    return I.Camera(KITTI_FX, KITTI_FX, KITTI_CX, KITTI_CY, KITTI_MBF / KITTI_FX, R, Ow, sigma)


def test_unprojection_equals_cv2_gemm():
    rng = np.random.default_rng(0)
    n_random, n_kitti = 6000, 6000
    mismatches = 0
    for case in range(n_random + n_kitti):
        if case < n_random:  # arbitrary rotations, translations, intrinsics and keys
            cam = I.Camera(rng.uniform(100, 2000), rng.uniform(100, 2000), rng.uniform(0, 1300), rng.uniform(0, 400), 0.5,
                           rotation(*rng.uniform(-np.pi, np.pi, 3)), rng.uniform(-100, 100, 3), np.eye(6))
            u, v, z = rng.uniform(-10, 1300), rng.uniform(-10, 400), rng.uniform(0.01, 200)
        else:  # KITTI intrinsics, key on the crop, depth mbf / disparity, a drive-like pose
            cam = camera(rotation(*rng.uniform(-0.05, 0.05, 2), rng.uniform(-np.pi, np.pi)), rng.uniform(-300, 300, 3) * (1, 0.02, 1))
            u, v = rng.uniform(109, 1133), rng.uniform(11, 363)
            z = np.float32(KITTI_MBF) / np.float32(rng.uniform(0.5, 120))
        got = I.unproject(np.array([u]), np.array([v]), np.array([z]), cam)[0]
        u32, v32, z32 = np.float32(u), np.float32(v), np.float32(z)
        x = (u32 - cam.cx) * z32 * cam.invfx
        y = (v32 - cam.cy) * z32 * cam.invfy
        xc = np.array([[x], [y], [z32]], np.float32)
        want = cv2.gemm(cam.Rwc, xc, 1, cam.Ow.reshape(3, 1), 1)[:, 0]
        assert want.dtype == np.float32
        mismatches += got.tobytes() != want.tobytes()
    assert mismatches == 0


def test_lu_determinant_against_numpy_and_zero_pivots():
    rng = np.random.default_rng(1)
    for n in (6, 9):
        A = np.stack([random_spd(rng, n, 10.0 ** rng.uniform(-6, 2)) for _ in range(300)])
        got, want = I.det_lu(A), np.linalg.det(A)
        assert np.all(np.abs(got - want) <= 1e-13 * np.abs(want))
        # general (non-symmetric, sometimes ill-conditioned) matrices exercise the row swaps
        B = rng.standard_normal((300, n, n))
        got, want = I.det_lu(B), np.linalg.det(B)
        assert np.all(np.abs(got - want) <= 1e-10 * np.abs(want))
        # a zero column skips its pivot and gives 0; a zero leading column is skipped without a division by zero
        Z = A[:5].copy()
        Z[:, :, 2] = 0
        assert np.all(I.det_lu(Z) == 0)
        Z[:, :, 0] = 0
        assert np.all(I.det_lu(Z) == 0)
    C = rng.standard_normal((50, 3, 3))
    assert np.allclose(I.det3_cofactor(C), np.linalg.det(C), rtol=1e-13, atol=1e-15)


def keys(rng, n):
    k = np.zeros(n, [("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"), ("octave", "<i4"),
                     ("class_id", "<i4")])
    k["x"] = rng.uniform(109, 1133, n)
    k["y"] = rng.uniform(11, 363, n)
    k["octave"] = rng.integers(0, 8, n)
    return k


SIGMA2 = (np.float32(1.2) ** (2 * np.arange(8))).astype(np.float32)


def test_mutual_information_matches_the_closed_form():
    """MI(pose; z) of z = J x + v with x ~ N(0, S), v ~ N(0, R) is 0.5 log2(det(J S J^T + R) / det R): checks the block assembly."""
    rng = np.random.default_rng(2)
    k = keys(rng, 400)
    z = rng.uniform(2, 60, len(k)).astype(np.float32)
    for S in (1e-6 * np.eye(6), random_spd(rng, 6, 1e-4), random_spd(rng, 6, 1e-2)):
        for R, Ow in ((np.eye(3), (0, 0, 0)), (rotation(0.1, -0.3, 0.2), (1.5, -0.4, 7.0))):
            cam = camera(R, Ow, S)
            world, ds, dm, dj, valid = I.info_terms(k, z, SIGMA2, cam)
            assert valid.all()
            mi = I.mutual_information(ds, dm, dj)
            J = I.stereo_jacobian_pose(cam.fx, cam.fy, cam.mb, *world.astype(np.float64).T)
            s2 = SIGMA2[k["octave"]].astype(np.float64)
            P = J @ S @ np.swapaxes(J, 1, 2) + s2[:, None, None] * np.eye(3)
            closed = 0.5 * np.log2(np.linalg.det(P) / s2 ** 3)
            assert np.abs(mi - closed).max() <= 1e-9
            assert (mi > 0).all()


def test_zero_world_depth_gives_zero_information_and_invalid_keys_give_nan():
    rng = np.random.default_rng(3)
    k = keys(rng, 64)
    z = np.full(len(k), 5.0, np.float32)
    cam = camera(np.eye(3), (0, 0, -5.0), random_spd(rng, 6, 1e-3))  # wZ = 5 + (-5) = 0 exactly
    world, ds, dm, dj, valid = I.info_terms(k, z, SIGMA2, cam)
    assert (world[:, 2] == 0).all() and valid.all()
    assert np.abs(I.mutual_information(ds, dm, dj)).max() <= 1e-12
    bad = k.copy()
    bad["octave"][:3] = (-1, 8, 99)
    z2 = z.copy()
    z2[3:6] = (0.0, -1.0, np.nan)
    world, red, sel = I.select(bad, z2, np.zeros(len(k)), SIGMA2, camera(), -1e300)
    assert np.isnan(red[:6]).all() and np.isnan(world[:6]).all() and np.array_equal(sel, np.arange(6, len(k)))


def test_world_coordinate_jacobian_differs_from_the_camera_frame_one_away_from_identity():
    """The reference feeds the world point to a helper written for camera coordinates; only the identity pose hides it."""
    rng = np.random.default_rng(4)
    k = keys(rng, 32)
    z = rng.uniform(2, 60, len(k)).astype(np.float32)
    for R, Ow, same in ((np.eye(3), (0, 0, 0), True), (rotation(0.05, 0.4, -0.1), (2.0, 0.1, 12.0), False)):
        cam = camera(R, Ow)
        world = I.unproject(k["x"], k["y"], z, cam).astype(np.float64)
        xc = np.stack([((k["x"] - cam.cx) * z) * cam.invfx, ((k["y"] - cam.cy) * z) * cam.invfy, z], 1).astype(np.float64)
        Jw = I.stereo_jacobian_pose(cam.fx, cam.fy, cam.mb, *world.T)
        Jc = I.stereo_jacobian_pose(cam.fx, cam.fy, cam.mb, *xc.T)
        assert np.array_equal(Jw, Jc) == same


def test_motion_update_keeps_the_covariance_symmetric_positive_definite():
    S = 1e-6 * np.eye(6)
    for i in range(4):
        S = I.update_state_covariance_motion(S, rotation(0.01 * i, 0.02, -0.01), (0.1, 0.0, 1.0 + i))
        assert np.allclose(S, S.T) and np.linalg.eigvalsh(0.5 * (S + S.T)).min() > 0
