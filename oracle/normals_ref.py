"""fp64 numpy restatement of the reference's scripts/depth_normal_consistency.py (DepthNormalConsistency) and
scripts/depth_to_normal.py (DepthToNormal), and of the Open3D call they make.

Quirks kept (each pinned by tests/golden/dn_depth_normals.npz):
- depth files: a PNG read as 16 bit and a .npy (channel 0 of a 3-D array) are both multiplied by 0.001, then cast to f32;
- the camera coordinates (u + 0.5 - cx) * d / fx are formed in f32 (numpy's weak Python scalars), then `@ inv(R) + t` in
  f64, so every depth-0 pixel lands exactly on the camera centre and joins the cloud;
- a normal is negated where (p - t) . n > 0;
- DepthNormalConsistency decodes the mono normal as 2 m - 1 (dsine: then diag(1, -1, -1)), tests degrees > angle_treshold
  and names its outputs with png -> jpg; DepthToNormal decodes (m - 0.5) * 2, takes the angle between the *encoded*
  vectors (n + 1) / 2 and m * 0.5 + 0.5, tests > 10 and keeps the frame's own file name.

Open3D's PointCloud.estimate_normals(KDTreeSearchParamKNN(k)) with fast_normal_computation=True [EXT, restated from
Open3D's EstimateNormals.cpp, not installed here]: the min(k, N) nearest points of each point, itself included; fewer than
3 -> identity covariance; else E[x x^T] - E[x] E[x]^T from fp64 cumulants summed in neighbour order and divided by the
count; FastEigen3x3 (Geometric Tools' robust symmetric solver); a zero vector becomes (0, 0, 1).  nanoflann's order among
equidistant points cannot be reproduced; this project's tie rule: distinct positions in (squared distance, smallest point
index) order, all copies of a position before the next.  Squared distances are ((dx dx + dy dy) + dz dz) with
d = p - q, as the kernel computes them.
"""
from __future__ import annotations

import math

import numpy as np

SCALE_FACTOR = 0.001
OPENGL_TO_OPENCV = np.array([[1, 0, 0, 0], [0, -1, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]])


def backproject(depth: np.ndarray, fx, fy, cx, cy, w: int, h: int, c2w: np.ndarray):
    """(world points [h*w,3] f64, camera coordinates [h*w,3] f32) exactly as the scripts' backproject forms them."""
    coords = np.stack(np.meshgrid(np.arange(w), np.arange(h), indexing="xy"), axis=-1) + 0.5
    coords = coords.reshape(-1, 2).astype(np.float32)
    d = depth.reshape(-1, 1)
    cam = np.zeros([w, h, 3], dtype=np.float32).reshape(-1, 3)
    cam[:, 0] = (coords[:, 0] - cx) * d[:, 0] / fx
    cam[:, 1] = (coords[:, 1] - cy) * d[:, 0] / fy
    cam[:, 2] = d[:, 0]
    return cam @ np.linalg.inv(c2w[..., :3, :3]) + c2w[..., :3, 3], cam


def unique_positions(points: np.ndarray):
    """(positions [U,3], smallest index [U], multiplicity [U], position of each point [N]); -0.0 equals +0.0."""
    p = np.asarray(points, np.float64) + 0.0
    uniq, first, inv, counts = np.unique(p, axis=0, return_index=True, return_inverse=True, return_counts=True)
    return uniq, first, counts, inv.reshape(-1)


def sq_dist(q: np.ndarray, pts: np.ndarray) -> np.ndarray:
    d = pts - q
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def knn(points: np.ndarray, k: int, queries=None):
    """Per query point (default: every point), the neighbour positions' smallest indices, one entry per copy taken, in
    the tie rule's order: a list of int arrays of length min(k, N)."""
    uniq, first, counts, inv = unique_positions(points)
    n = len(points)
    kk = min(k, n)
    qs = range(n) if queries is None else queries
    cache, out = {}, []
    for i in qs:
        u = inv[i]
        if u not in cache:
            d2 = sq_dist(uniq[u], uniq)
            order = np.lexsort((first, d2))
            c = np.cumsum(counts[order])
            last = int(np.searchsorted(c, kk))
            take = counts[order[: last + 1]].copy()
            take[-1] -= c[last] - kk
            cache[u] = np.repeat(first[order[: last + 1]], take)
        out.append(cache[u])
    return out


def covariance(points: np.ndarray, nbr: np.ndarray) -> np.ndarray:
    """Open3D's ComputeCovariance over points[nbr] in order (sequential fp64 cumulants)."""
    if len(nbr) < 3:
        return np.eye(3)
    p = np.asarray(points, np.float64)[nbr]
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    cum = np.array([np.cumsum(v)[-1] for v in (x, y, z, x * x, x * y, x * z, y * y, y * z, z * z)]) / float(len(nbr))
    c = np.empty((3, 3))
    c[0, 0] = cum[3] - cum[0] * cum[0]
    c[1, 1] = cum[6] - cum[1] * cum[1]
    c[2, 2] = cum[8] - cum[2] * cum[2]
    c[0, 1] = c[1, 0] = cum[4] - cum[0] * cum[1]
    c[0, 2] = c[2, 0] = cum[5] - cum[0] * cum[2]
    c[1, 2] = c[2, 1] = cum[7] - cum[1] * cum[2]
    return c


def _cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _eigvec0(A, e):
    r0 = (A[0][0] - e, A[0][1], A[0][2])
    r1 = (A[0][1], A[1][1] - e, A[1][2])
    r2 = (A[0][2], A[1][2], A[2][2] - e)
    c = [_cross(r0, r1), _cross(r0, r2), _cross(r1, r2)]
    d = [_dot(v, v) for v in c]
    imax, dmax = 0, d[0]
    if d[1] > dmax:
        imax, dmax = 1, d[1]
    if d[2] > dmax:
        imax = 2
    s = math.sqrt(d[imax])
    return tuple(v / s for v in c[imax])


def _eigvec1(A, e0, e1):
    if abs(e0[0]) > abs(e0[1]):
        il = 1 / math.sqrt(e0[0] * e0[0] + e0[2] * e0[2])
        U = (-e0[2] * il, 0.0, e0[0] * il)
    else:
        il = 1 / math.sqrt(e0[1] * e0[1] + e0[2] * e0[2])
        U = (0.0, e0[2] * il, -e0[1] * il)
    V = _cross(e0, U)
    AU = tuple(A[r][0] * U[0] + A[r][1] * U[1] + A[r][2] * U[2] for r in range(3))
    AV = tuple(A[r][0] * V[0] + A[r][1] * V[1] + A[r][2] * V[2] for r in range(3))
    m00 = U[0] * AU[0] + U[1] * AU[1] + U[2] * AU[2] - e1
    m01 = U[0] * AV[0] + U[1] * AV[1] + U[2] * AV[2]
    m11 = V[0] * AV[0] + V[1] * AV[1] + V[2] * AV[2] - e1
    a00, a01, a11 = abs(m00), abs(m01), abs(m11)
    if a00 >= a11:
        if max(a00, a01) > 0:
            if a00 >= a01:
                m01 /= m00
                m00 = 1 / math.sqrt(1 + m01 * m01)
                m01 *= m00
            else:
                m00 /= m01
                m01 = 1 / math.sqrt(1 + m00 * m00)
                m00 *= m01
            return tuple(m01 * U[i] - m00 * V[i] for i in range(3))
        return U
    if max(a11, a01) > 0:
        if a11 >= a01:
            m01 /= m11
            m11 = 1 / math.sqrt(1 + m01 * m01)
            m01 *= m11
        else:
            m11 /= m01
            m01 = 1 / math.sqrt(1 + m11 * m11)
            m11 *= m01
        return tuple(m11 * U[i] - m01 * V[i] for i in range(3))
    return U


def fast_eigen3x3(cov: np.ndarray, branch: list | None = None) -> np.ndarray:
    """Open3D's FastEigen3x3: the unit eigenvector of the smallest eigenvalue of a symmetric 3x3 (zero for a zero matrix).
    `branch`, if given, receives the name of the path taken."""
    C = [[float(cov[r][c]) for c in range(3)] for r in range(3)]
    mx = max(C[0][0], C[0][1], C[0][2], C[1][1], C[1][2], C[2][2])
    note = branch.append if branch is not None else (lambda _: None)
    if mx == 0:
        note("zero")
        return np.zeros(3)
    A = [[v / mx for v in row] for row in C]
    norm = A[0][1] * A[0][1] + A[0][2] * A[0][2] + A[1][2] * A[1][2]
    if norm > 0:
        q = (A[0][0] + A[1][1] + A[2][2]) / 3
        b00, b11, b22 = A[0][0] - q, A[1][1] - q, A[2][2] - q
        p = math.sqrt((b00 * b00 + b11 * b11 + b22 * b22 + norm * 2) / 6)
        c00 = b11 * b22 - A[1][2] * A[1][2]
        c01 = A[0][1] * b22 - A[1][2] * A[0][2]
        c02 = A[0][1] * A[1][2] - b11 * A[0][2]
        det = (b00 * c00 - A[0][1] * c01 + A[0][2] * c02) / (p * p * p)
        half_det = min(max(det * 0.5, -1.0), 1.0)
        angle = math.acos(half_det) / 3.0
        beta2 = math.cos(angle) * 2
        beta0 = math.cos(angle + 2.09439510239319549) * 2
        beta1 = -(beta0 + beta2)
        ev = (q + p * beta0, q + p * beta1, q + p * beta2)
        if half_det >= 0:
            v2 = _eigvec0(A, ev[2])
            if ev[2] < ev[0] and ev[2] < ev[1]:
                note("pos/2")
                return np.array(v2)
            v1 = _eigvec1(A, v2, ev[1])
            if ev[1] < ev[0] and ev[1] < ev[2]:
                note("pos/1")
                return np.array(v1)
            note("pos/0")
            return np.array(_cross(v1, v2))
        v0 = _eigvec0(A, ev[0])
        if ev[0] < ev[1] and ev[0] < ev[2]:
            note("neg/0")
            return np.array(v0)
        v1 = _eigvec1(A, v0, ev[1])
        if ev[1] < ev[0] and ev[1] < ev[2]:
            note("neg/1")
            return np.array(v1)
        note("neg/2")
        return np.array(_cross(v0, v1))
    note("diagonal")
    if C[0][0] < C[1][1] and C[0][0] < C[2][2]:
        return np.array([1.0, 0.0, 0.0])
    if C[1][1] < C[0][0] and C[1][1] < C[2][2]:
        return np.array([0.0, 1.0, 0.0])
    return np.array([0.0, 0.0, 1.0])


def estimate_normals(points: np.ndarray, k: int = 200, nbrs=None):
    """(normals [N,3], covariances [N,3,3]) as Open3D's estimate_normals(KDTreeSearchParamKNN(k)) under the tie rule.
    nbrs: precomputed knn(points, k)."""
    pts = np.asarray(points, np.float64)
    nbrs = knn(pts, k) if nbrs is None else nbrs
    normals = np.empty((len(pts), 3))
    covs = np.empty((len(pts), 3, 3))
    done = {}
    for i, nb in enumerate(nbrs):
        key = (pts[i] + 0.0).tobytes()
        if key not in done:
            c = covariance(pts, nb)
            n = fast_eigen3x3(c)
            if np.linalg.norm(n) == 0.0:
                n = np.array([0.0, 0.0, 1.0])
            done[key] = (n, c)
        normals[i], covs[i] = done[key]
    return normals, covs


def orient(points: np.ndarray, normals: np.ndarray, center: np.ndarray) -> np.ndarray:
    n = normals.copy()
    flip = ((points - center.reshape(1, 3)) * n).sum(axis=-1) > 0
    n[flip] = -n[flip]
    return n


def angle_between(n1: np.ndarray, n2: np.ndarray) -> np.ndarray:
    """compute_angle_between_normals of the scripts ([..., 3] each)."""
    a = n1 / np.linalg.norm(n1, axis=-1, keepdims=True)
    b = n2 / np.linalg.norm(n2, axis=-1, keepdims=True)
    return np.degrees(np.arccos(np.clip(np.sum(a * b, axis=-1), -1.0, 1.0)))


def mono_rotation(c2w: np.ndarray) -> np.ndarray:
    return np.transpose(np.linalg.inv(c2w)[:3, :3])


def consistency(normals: np.ndarray, mono_u8: np.ndarray, c2w: np.ndarray, mode: str, threshold: float):
    """(degrees [N], mask [N] bool, normals image [N,3] u8) of one frame; mode "omnidata" / "dsine"
    (DepthNormalConsistency) or "depth_to_normal" (DepthToNormal, whose threshold is 10)."""
    R = mono_rotation(c2w)
    m = mono_u8.reshape(-1, 3) / 255.0
    enc = ((normals + 1) / 2 * 255).astype(np.uint8)
    if mode == "depth_to_normal":
        m = (m.T - 0.5) * 2
        m = (R @ m).T
        m = m / np.linalg.norm(m, axis=1, keepdims=True)
        deg = angle_between((normals + 1) / 2, m * 0.5 + 0.5)
    else:
        m = 2 * m - 1
        if mode == "dsine":
            m = m @ np.diag([1, -1, -1])
        m = (R @ m.T).T
        m = m / np.linalg.norm(m, axis=1, keepdims=True)
        deg = angle_between(normals, m)
    return deg, deg > threshold, enc
