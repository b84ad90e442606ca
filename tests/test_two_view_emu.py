"""The two-view CUDA kernels (csrc/epipolar_kernels.cuh) EXECUTED ON THE CPU through tests/cpp/cuda_emu.h, launched as
csrc/epipolar.cu launches them, against the reference's arithmetic (oracle/epipolar_oracle.py = the OpenCV calls of
reference src/geometry/epipolar_geometry.cpp:17-175) with the acceptance bars of the hardware tests
(tests/test_epipolar_gpu.py, tests/test_homography_gpu.py).  For the homography kernels, which have not run on a GPU yet,
this is the first execution of any kind; for the essential-matrix kernels, which have, it shows that the emulation carries
the kernels' numerics.  Fewer hypotheses and points than on the GPU: one OS thread plays one CUDA thread."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

import mvo_synth
from conftest import have_cv2

ROOT = Path(__file__).resolve().parent.parent
pytestmark = pytest.mark.skipif(not have_cv2(), reason="cv2 (the reference's third-party code) not importable")
K = mvo_synth.K_DEFAULT
HYP = 512


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = tmp_path_factory.mktemp("twoview") / "libtwo_view_emu.so"
    subprocess.run(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-I", str(ROOT / "include"),
                    "-I", str(ROOT / "monocular-visual-odometry_b200" / "csrc"), "-I", str(ROOT / "tests" / "cpp"), "-I", "/usr/local/cuda/include",
                    str(ROOT / "tests" / "cpp" / "two_view_emu.cpp"), "-o", str(so)], check=True)
    lib = C.CDLL(str(so))
    vp, i, d, u64 = C.c_void_p, C.c_int, C.c_double, C.c_uint64
    lib.emu_essential.argtypes = [vp, vp, i, vp, d, i, u64, vp, vp, vp, vp, vp]
    lib.emu_homography.argtypes = [vp, vp, i, vp, d, i, u64, vp, vp, vp]
    lib.emu_triangulate.argtypes = [vp, vp, vp, i, vp, vp, vp]
    return lib


def _rod(r):
    th = np.linalg.norm(r)
    k = r / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def _general_scene(seed, n=360, noise=0.5, outliers=0.2):
    rng = np.random.default_rng(seed)
    R = _rod(rng.normal(0, 0.06, 3) + 1e-9)
    t = np.array([0.25, 0.02, 0.05]) + rng.normal(0, 0.02, 3)
    X1 = np.stack([rng.uniform(-2.2, 2.2, n), rng.uniform(-1.6, 1.6, n), rng.uniform(2.5, 9, n)], 1)
    X2 = X1 @ R.T + t
    p1 = X1[:, :2] / X1[:, 2:3] * K[0, 0] + K[:2, 2] + rng.normal(0, noise, (n, 2))
    p2 = X2[:, :2] / X2[:, 2:3] * K[0, 0] + K[:2, 2] + rng.normal(0, noise, (n, 2))
    bad = rng.random(n) < outliers
    p2[bad] = rng.uniform([0, 0], [640, 480], (bad.sum(), 2))
    return p1.astype(np.float32), p2.astype(np.float32), R, t / np.linalg.norm(t), ~bad, X1


def _rot_err(Ra, Rb):
    return np.arccos(np.clip((np.trace(Ra.T @ Rb) - 1) / 2, -1, 1))


def _dir_err(a, b):
    return np.arccos(np.clip(np.dot(a, b) / (np.linalg.norm(a) * np.linalg.norm(b)), -1, 1))


@pytest.mark.parametrize("seed", [0, 1])
def test_essential_kernels_as_a_batch_of_one(emu, seed):
    from oracle import epipolar_oracle
    p1, p2, R_true, t_true, good, X1 = _general_scene(seed)
    n = len(p1)
    E, R, t, inl, oi = np.zeros((3, 3)), np.zeros((3, 3)), np.zeros(3), np.zeros(n, np.int32), np.zeros(8, np.int32)
    Kc = np.ascontiguousarray(K, np.float64)
    ni = emu.emu_essential(p1.ctypes.data, p2.ctypes.data, n, Kc.ctypes.data, 1.0, HYP, 12345, E.ctypes.data, R.ctypes.data, t.ctypes.data,
                           inl.ctypes.data, oi.ctypes.data)
    inl = inl[:ni]
    Eo, Ro, to, inlo = epipolar_oracle.esti_motion_by_essential(p1, p2, K, 0.999, 1.0)
    assert ni >= 8 and oi[4] >= oi[3]                               # the local optimisation did not lose support
    assert abs(E[2, 2] - 1) < 1e-12 and abs(np.linalg.norm(t) - 1) < 1e-12 and abs(np.linalg.det(R) - 1) < 1e-9
    er, ero, et, eto = _rot_err(R, R_true), _rot_err(Ro, R_true), _dir_err(t, t_true), _dir_err(to, t_true)
    assert er < max(2 * ero, 3e-3) and et < max(2 * eto, 0.035), (er, ero, et, eto)      # the bars of tests/test_epipolar_gpu.py
    assert np.all(np.diff(inl) > 0) and good[inl].mean() > 0.97
    assert len(set(inl.tolist()) & set(inlo.tolist())) / len(inlo) > 0.9
    # triangulation kernel with this motion against cv2.triangulatePoints
    Ki = np.linalg.inv(K)
    np1 = ((np.c_[p1, np.ones(n)] @ Ki.T)[:, :2]).astype(np.float32)
    np2 = ((np.c_[p2, np.ones(n)] @ Ki.T)[:, :2]).astype(np.float32)
    X = np.zeros((ni, 3), np.float32)
    assert emu.emu_triangulate(np1.ctypes.data, np2.ctypes.data, inl.ctypes.data, ni, np.ascontiguousarray(R).ctypes.data, t.ctypes.data, X.ctypes.data) == 0
    Xo = epipolar_oracle.do_triangulation(np1, np2, R, t, inl)
    rel = np.linalg.norm(X - Xo, axis=1) / np.linalg.norm(Xo, axis=1)
    assert np.median(rel) < 2e-4 and (rel < 2e-2).mean() > 0.98, (np.median(rel), rel.max())


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_homography_kernels_as_a_batch_of_one(emu, seed):
    from oracle import epipolar_oracle
    rng = np.random.default_rng(seed)
    n = 320
    R = _rod(rng.normal(0, 0.05, 3) + 1e-9)
    t = np.array([0.3, 0.03, 0.08]) + rng.normal(0, 0.02, 3)
    nrm = np.array([rng.normal(0, 0.15), rng.normal(0, 0.15), 1.0])
    nrm /= np.linalg.norm(nrm)
    P = np.stack([rng.uniform(-2, 2, n), rng.uniform(-1.5, 1.5, n), np.zeros(n)], 1)
    P[:, 2] = (4.0 - P[:, :2] @ nrm[:2]) / nrm[2]
    P2 = P @ R.T + t
    q1 = P[:, :2] / P[:, 2:3] * K[0, 0] + K[:2, 2]
    q2 = P2[:, :2] / P2[:, 2:3] * K[0, 0] + K[:2, 2]
    p1 = (q1 + rng.normal(0, 0.4, (n, 2))).astype(np.float32)
    p2 = q2 + rng.normal(0, 0.4, (n, 2))
    bad = rng.random(n) < 0.2
    p2[bad] = rng.uniform([0, 0], [640, 480], (bad.sum(), 2))
    p2 = p2.astype(np.float32)
    H, inl, oi = np.zeros((3, 3)), np.zeros(n, np.int32), np.zeros(8, np.int32)
    Kc = np.ascontiguousarray(K, np.float64)
    ni = emu.emu_homography(p1.ctypes.data, p2.ctypes.data, n, Kc.ctypes.data, 3.0, HYP, 777, H.ctypes.data, inl.ctypes.data, oi.ctypes.data)
    inl = inl[:ni]
    Ho, _, _, _, inlo = epipolar_oracle.esti_motion_by_homography(p1, p2, K, 3.0)
    assert ni >= 4 and oi[4] >= oi[3] and abs(H[2, 2] - 1) < 1e-12

    def terr(Hm):                                                   # transfer error of the noise-free plane points, pixels RMS
        m = np.c_[q1, np.ones(n)] @ Hm.T
        return np.sqrt(np.mean(np.sum((m[:, :2] / m[:, 2:3] - q2) ** 2, 1)))
    assert terr(H) < terr(Ho) + 0.1, (terr(H), terr(Ho))            # the bars of tests/test_homography_gpu.py
    a, b = set(inl.tolist()), set(inlo.tolist())
    assert np.all(np.diff(inl) > 0) and len(a & b) / len(b) > 0.9 and (~bad)[inl].mean() > 0.97
    # every reported inlier is within the threshold of the reported H, every other point is not
    m = np.c_[p1.astype(np.float64), np.ones(n)] @ H.T
    err = np.sqrt(np.sum((m[:, :2] / m[:, 2:3] - p2) ** 2, 1))
    inside = np.zeros(n, bool)
    inside[inl] = True
    assert (err[inside] <= 3.0 + 1e-6).all() and (err[~inside] > 3.0 - 1e-6).all()


def test_homography_kernels_on_six_exact_points(emu):
    """Six correspondences of an exactly planar scene: fewer than the essential matrix needs, enough for a homography, which
    mvo_esti_motion_by_homography accepts from 4 correspondences on."""
    rng = np.random.default_rng(6)
    n = 6
    R, t = _rod(np.array([0.02, -0.03, 0.01])), np.array([0.3, 0.02, 0.05])
    nrm = np.array([0.1, -0.05, 1.0]) / np.linalg.norm([0.1, -0.05, 1.0])
    P = np.stack([rng.uniform(-2, 2, n), rng.uniform(-1.5, 1.5, n), np.zeros(n)], 1)
    P[:, 2] = (4.0 - P[:, :2] @ nrm[:2]) / nrm[2]
    P2 = P @ R.T + t
    p1 = (P[:, :2] / P[:, 2:3] * K[0, 0] + K[:2, 2]).astype(np.float32)
    p2 = (P2[:, :2] / P2[:, 2:3] * K[0, 0] + K[:2, 2]).astype(np.float32)
    H, inl, oi = np.zeros((3, 3)), np.zeros(n, np.int32), np.zeros(8, np.int32)
    Kc = np.ascontiguousarray(K, np.float64)
    ni = emu.emu_homography(p1.ctypes.data, p2.ctypes.data, n, Kc.ctypes.data, 3.0, HYP, 777, H.ctypes.data, inl.ctypes.data, oi.ctypes.data)
    assert ni >= 4                                                  # mvo_esti_motion_by_homography returns MVO_OK
    assert ni == 6 and inl.tolist() == list(range(6)) and abs(H[2, 2] - 1) < 1e-12
    m = np.c_[p1.astype(np.float64), np.ones(n)] @ H.T
    assert np.abs(m[:, :2] / m[:, 2:3] - p2).max() < 1e-3
