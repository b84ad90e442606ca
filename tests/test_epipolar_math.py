"""csrc/epipolar_math.cuh compiled for the host (tests/cpp/epipolar_math_host.cpp): the numerics behind the two-view
kernels (SURVEY.md §8f-1) against numpy and, where the reference's arithmetic is an OpenCV routine, against cv2:
cv::decomposeEssentialMat (recoverPose, reference src/geometry/epipolar_geometry.cpp:53) and cv::triangulatePoints (:154)."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def epi(tmp_path_factory):
    so = tmp_path_factory.mktemp("epi") / "libepi_host.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off", "-I",
                    str(ROOT / "monocular-visual-odometry_b200" / "csrc"), str(ROOT / "tests" / "cpp" / "epipolar_math_host.cpp"),
                    "-o", str(so)], check=True)
    lib = C.CDLL(str(so))
    lib.epi_sampson.restype = C.c_double
    lib.epi_sampson.argtypes = [C.c_void_p] + [C.c_double] * 4
    lib.epi_triangulate.argtypes = [C.c_void_p, C.c_void_p] + [C.c_double] * 4 + [C.c_void_p]
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _rodrigues(r):
    th = np.linalg.norm(r)
    if th < 1e-12:
        return np.eye(3)
    k = r / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def _two_view(rng, n):
    """Points in front of both cameras; x2 = R x1 + t (OpenCV's recoverPose convention)."""
    R = _rodrigues(rng.normal(0, 0.15, 3))
    t = rng.normal(0, 1, 3)
    t /= np.linalg.norm(t)
    X1 = np.stack([rng.uniform(-2, 2, n), rng.uniform(-1.5, 1.5, n), rng.uniform(3, 9, n)], 1)
    X2 = X1 @ R.T + 0.4 * t
    return R, t, X1, X2, X1[:, :2] / X1[:, 2:3], X2[:, :2] / X2[:, 2:3]


def test_svd3_and_null_vector(epi):
    rng = np.random.default_rng(0)
    for k in range(200):
        M = rng.normal(0, 1, (3, 3))
        if k % 5 == 0:
            M[:, 2] = M[:, 0] * 0.3 - M[:, 1]                 # rank 2, like an essential matrix estimate
        U, s, V = np.zeros((3, 3)), np.zeros(3), np.zeros((3, 3))
        epi.epi_svd3(_p(M), _p(U), _p(s), _p(V))
        assert np.allclose(U @ np.diag(s) @ V.T, M, atol=1e-10)
        assert np.allclose(U.T @ U, np.eye(3), atol=1e-10) and np.allclose(V.T @ V, np.eye(3), atol=1e-10)
        assert np.allclose(s, np.linalg.svd(M, compute_uv=False), atol=1e-7) and s[0] >= s[1] >= s[2] >= 0
    for k in range(100):
        A = rng.normal(0, 1, (8, 9))
        x = np.zeros(9)
        assert epi.epi_null_8x9(_p(A), _p(x)) == 1
        assert abs(np.linalg.norm(x) - 1) < 1e-12 and np.abs(A @ x).max() < 1e-10
    A = rng.normal(0, 1, (8, 9))
    A[7] = A[0] + A[1]                                        # rank 7: two-dimensional null space -> rejected
    assert epi.epi_null_8x9(_p(A), _p(np.zeros(9))) == 0


def test_essential_from_8_and_sampson(epi):
    rng = np.random.default_rng(1)
    for k in range(100):
        R, t, X1, X2, x1, x2 = _two_view(rng, 8)
        E = np.zeros((3, 3))
        assert epi.epi_essential_from_8(_p(np.ascontiguousarray(x1)), _p(np.ascontiguousarray(x2)), _p(E)) == 1
        tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
        Et = tx @ R
        Et /= np.linalg.norm(Et)
        En = E / np.linalg.norm(E)
        assert min(np.abs(En - Et).max(), np.abs(En + Et).max()) < 1e-7, k
        assert np.allclose(np.linalg.svd(E, compute_uv=False), [1, 1, 0], atol=1e-9)
        for i in range(8):
            assert epi.epi_sampson(_p(E), x1[i, 0], x1[i, 1], x2[i, 0], x2[i, 1]) < 1e-20
        # a point moved off its epipolar line: Sampson distance ~ squared distance to the line (first order)
        d = 1e-3
        l = E @ np.array([x1[0, 0], x1[0, 1], 1.0])
        nrm = l[:2] / np.linalg.norm(l[:2])
        s = epi.epi_sampson(_p(E), x1[0, 0], x1[0, 1], x2[0, 0] + d * nrm[0], x2[0, 1] + d * nrm[1])
        lt = E.T @ np.array([x2[0, 0], x2[0, 1], 1.0])
        expect = (d * np.linalg.norm(l[:2])) ** 2 / (l[0] ** 2 + l[1] ** 2 + lt[0] ** 2 + lt[1] ** 2)
        assert abs(s - expect) < 0.05 * expect
    # degenerate sample: the same point eight times
    x = np.tile([[0.1, 0.2]], (8, 1))
    assert epi.epi_essential_from_8(_p(x), _p(x.copy()), _p(np.zeros((3, 3)))) == 0


def test_decompose_and_triangulate_vs_cv2(epi):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(2)
    for k in range(50):
        R, t, X1, X2, x1, x2 = _two_view(rng, 40)
        tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
        E = tx @ R
        R1, R2, tt = np.zeros((3, 3)), np.zeros((3, 3)), np.zeros(3)
        epi.epi_decompose(_p(np.ascontiguousarray(E)), _p(R1), _p(R2), _p(tt))
        c1, c2, ct = cv2.decomposeEssentialMat(E)
        for Rm in (R1, R2):
            assert abs(np.linalg.det(Rm) - 1) < 1e-9 and np.allclose(Rm @ Rm.T, np.eye(3), atol=1e-9)
        # the same two rotations as OpenCV (in either order) and the same translation up to sign; the truth among them
        assert min(max(np.abs(R1 - c1).max(), np.abs(R2 - c2).max()), max(np.abs(R1 - c2).max(), np.abs(R2 - c1).max())) < 1e-8
        assert min(np.abs(tt - ct.ravel()).max(), np.abs(tt + ct.ravel()).max()) < 1e-8
        assert min(np.abs(R1 - R).max(), np.abs(R2 - R).max()) < 1e-8 and min(np.abs(tt - t).max(), np.abs(tt + t).max()) < 1e-8
        # cv::triangulatePoints with the reference's projection matrices [I|0], [R|t] (epipolar_geometry.cpp:146-154)
        P1 = np.hstack([np.eye(3), np.zeros((3, 1))])
        P2 = np.hstack([R, 0.4 * t[:, None]])
        noise = rng.normal(0, 1e-3, x2.shape)
        ref = cv2.triangulatePoints(P1.astype(np.float32), P2.astype(np.float32), x1.T.astype(np.float32), (x2 + noise).T.astype(np.float32))
        ref = (ref[:3] / ref[3]).T
        for i in range(len(x1)):
            X = np.zeros(4)
            a, b = x1[i].astype(np.float32), (x2[i] + noise[i]).astype(np.float32)
            epi.epi_triangulate(_p(P1.astype(np.float32).astype(np.float64)), _p(P2.astype(np.float32).astype(np.float64)),
                                float(a[0]), float(a[1]), float(b[0]), float(b[1]), _p(X))
            assert np.abs(X[:3] / X[3] - ref[i]).max() < 2e-4 * max(1.0, np.abs(ref[i]).max()), (k, i)


def _plane_scene(rng, n=60):
    """Points on a plane n.X = d seen from two cameras: x2 ~ (R + t n^T / d) x1."""
    R = _rodrigues(rng.normal(0, 0.08, 3))
    t = rng.normal(0, 0.15, 3)
    nrm = np.array([rng.normal(0, 0.2), rng.normal(0, 0.2), 1.0])
    nrm /= np.linalg.norm(nrm)
    d = rng.uniform(3, 6)
    P = np.stack([rng.uniform(-2, 2, n), rng.uniform(-1.5, 1.5, n), np.zeros(n)], 1)
    P[:, 2] = (d - P[:, :2] @ nrm[:2]) / nrm[2]
    P2 = P @ R.T + t
    return R, t / d, nrm, P[:, :2] / P[:, 2:3], P2[:, :2] / P2[:, 2:3]


def test_homography_from_4_and_transfer_error(epi):
    epi.epi_transfer_err.restype = C.c_double
    epi.epi_transfer_err.argtypes = [C.c_void_p] + [C.c_double] * 4
    rng = np.random.default_rng(4)
    for k in range(100):
        R, td, nrm, x1, x2 = _plane_scene(rng, 12)
        H = np.zeros((3, 3))
        assert epi.epi_homography_from_4(_p(np.ascontiguousarray(x1[:4])), _p(np.ascontiguousarray(x2[:4])), _p(H)) == 1
        Ht = R + np.outer(td, nrm)
        Hn, Htn = H / np.linalg.norm(H), Ht / np.linalg.norm(Ht)
        assert min(np.abs(Hn - Htn).max(), np.abs(Hn + Htn).max()) < 1e-8
        for i in range(12):                                   # the other points of the plane obey the same homography
            assert epi.epi_transfer_err(_p(H), x1[i, 0], x1[i, 1], x2[i, 0], x2[i, 1]) < 1e-18
        assert abs(epi.epi_transfer_err(_p(H), x1[5, 0], x1[5, 1], x2[5, 0] + 3e-3, x2[5, 1] - 4e-3) - 25e-6) < 1e-9
    x = np.array([[0, 0], [1, 1], [2, 2], [0.5, 0.1]], float)  # three collinear points
    assert epi.epi_homography_from_4(_p(x), _p(x.copy()), _p(np.zeros((3, 3)))) == 0


def test_homography_local_optimisation(epi):
    """The Gauss-Newton refinement k_homo_finish_batch applies to the best four-point model (same header functions, run serially):
    from a minimal model fitted to NOISY points it reaches the least-squares homography of the consensus set — as good as
    cv2.findHomography's own refinement on the noise-free plane — and stops by itself."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(12)
    f = 615.0
    thr2 = (3.0 / f) ** 2
    for k in range(20):
        R, td, nrm, x1, x2 = _plane_scene(rng, 400)
        a = x1 + rng.normal(0, 0.4 / f, x1.shape)               # 0.4 px of noise in scaled coordinates
        b = x2 + rng.normal(0, 0.4 / f, x2.shape)
        bad = rng.random(len(a)) < 0.2
        b[bad] += rng.uniform(-0.1, 0.1, (bad.sum(), 2))
        # the RANSAC front end in miniature: 64 four-point samples, the one with the largest consensus is refined
        H, best = np.zeros((3, 3)), -1
        for s_ in range(64):
            idx = rng.choice(len(a), 4, replace=False)
            Hs = np.zeros((3, 3))
            if epi.epi_homography_from_4(_p(np.ascontiguousarray(a[idx])), _p(np.ascontiguousarray(b[idx])), _p(Hs)) != 1:
                continue
            m = np.c_[a, np.ones(len(a))] @ Hs.T
            with np.errstate(divide="ignore", invalid="ignore"):
                cnt = int((np.sum((m[:, :2] / m[:, 2:3] - b) ** 2, 1) <= thr2).sum())
            if cnt > best:
                best, H = cnt, Hs
        assert best > 200

        def plane_err(Hm):                                      # RMS transfer error on the noise-free points, pixels
            m = np.c_[x1, np.ones(len(x1))] @ Hm.T
            return f * np.sqrt(np.mean(np.sum((m[:, :2] / m[:, 2:3] - x2) ** 2, 1)))
        e_min = plane_err(H)
        a_c, b_c = np.ascontiguousarray(a), np.ascontiguousarray(b)
        steps = epi.epi_homography_lo(_p(a_c), _p(b_c), len(a), C.c_double(thr2), 3, 8, _p(H))
        e_lo = plane_err(H)
        assert abs(np.linalg.norm(H) - 1) < 1e-12 and 3 <= steps <= 24
        Hcv, _ = cv2.findHomography((a * f).astype(np.float32), (b * f).astype(np.float32), cv2.RANSAC, 3.0)
        S = np.diag([1 / f, 1 / f, 1.0])
        e_cv = plane_err(S @ Hcv @ np.linalg.inv(S))
        assert e_lo < 0.15 and e_lo < e_cv + 0.02, (k, e_min, e_lo, e_cv)
        assert e_lo <= e_min + 1e-9
        # a second run from the optimum is a fixed point: the first step already reports convergence
        H2 = H.copy()
        assert epi.epi_homography_lo(_p(a_c), _p(b_c), len(a), C.c_double(thr2), 1, 8, _p(H2)) <= 2 and np.abs(H2 - H).max() < 1e-9


def test_decompose_homography_and_filter_vs_cv2(epi):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(5)
    K = np.array([[615.0, 0, 320], [0, 615, 240], [0, 0, 1]])
    for k in range(60):
        R, td, nrm, x1, x2 = _plane_scene(rng, 40)
        Hn = (R + np.outer(td, nrm)) * rng.choice([1.0, -3.7, 0.2])         # scale and sign are irrelevant
        Rs, ts, ns = np.zeros((4, 9)), np.zeros((4, 3)), np.zeros((4, 3))
        m = epi.epi_decompose_homography(_p(np.ascontiguousarray(Hn)), _p(Rs), _p(ts), _p(ns))
        num, cR, ct, cn = cv2.decomposeHomographyMat(K @ Hn @ np.linalg.inv(K), K)
        assert m == num == 4
        used = set()
        for i in range(4):                                                    # same solution SET as OpenCV
            assert abs(np.linalg.det(Rs[i].reshape(3, 3)) - 1) < 1e-8
            best = min(range(4), key=lambda j: np.abs(Rs[i].reshape(3, 3) - cR[j]).max() + np.abs(ts[i] - ct[j].ravel()).max() + np.abs(ns[i] - cn[j].ravel()).max())
            err = max(np.abs(Rs[i].reshape(3, 3) - cR[best]).max(), np.abs(ts[i] - ct[best].ravel()).max(), np.abs(ns[i] - cn[best].ravel()).max())
            assert err < 1e-6, (k, i, err)
            used.add(best)
        assert used == {0, 1, 2, 3}
        assert min(max(np.abs(Rs[i].reshape(3, 3) - R).max(), np.abs(ts[i] - td).max(), np.abs(ns[i] - nrm).max()) for i in range(4)) < 1e-8
        # removeWrongRtOfHomography: the same surviving solutions as cv2.filterHomographyDecompByVisibleRefpoints
        keep = np.zeros(4, np.int32)
        a, b = np.ascontiguousarray(x1, np.float32), np.ascontiguousarray(x2, np.float32)
        kept = epi.epi_filter_homography(_p(Rs), _p(ns), 4, _p(a), _p(b), None, len(a), _p(keep))
        ref = cv2.filterHomographyDecompByVisibleRefpoints([r.reshape(3, 3) for r in Rs], [v.reshape(3, 1) for v in ns], a.reshape(-1, 1, 2), b.reshape(-1, 1, 2))
        ref = set() if ref is None else set(ref.ravel().tolist())
        assert set(np.nonzero(keep)[0].tolist()) == ref and kept == len(ref) and kept >= 1
    # pure rotation: one solution, no translation
    Rr = _rodrigues(np.array([0.02, -0.05, 0.01]))
    Rs, ts, ns = np.zeros((4, 9)), np.zeros((4, 3)), np.zeros((4, 3))
    assert epi.epi_decompose_homography(_p(np.ascontiguousarray(2.0 * Rr)), _p(Rs), _p(ts), _p(ns)) == 1
    assert np.abs(Rs[0].reshape(3, 3) - Rr).max() < 1e-9 and np.abs(ts[0]).max() == 0
