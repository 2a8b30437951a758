"""CPU checks of the screened Poisson reconstruction: the fp64 oracle's discrete operators and surfaces
(oracle/poisson_ref.py), the exporters' host logic (depth edges, the surface-normal conversion, samples per frame)
against independent per-pixel restatements, the point-cloud helpers against brute-force loops, the point-cloud PLY,
and the argument checks of the new C entry points (no GPU touched)."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from dn_splatter_b200 import _lib as L
from oracle import mesh_ref as M
from oracle import poisson_ref as P


# ------------------------------------------------------------------------------------------------ oracle self-checks
def test_div_grad_is_the_neumann_laplacian():
    R = 6
    g = np.random.default_rng(0)
    x = g.normal(size=(R, R, R))
    G = P.gradient(R)
    faces = np.zeros((3, R, R, R))
    for a in range(3):
        faces[a].reshape(-1)[P._face_rows(R, a)] = G[a] @ x.reshape(-1)
    lap = np.zeros_like(x)  # 7-point, neighbours outside the box dropped (zero flux)
    for i, j, k in np.ndindex(R, R, R):
        for d in ((1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)):
            q = (i + d[0], j + d[1], k + d[2])
            if all(0 <= c < R for c in q):
                lap[i, j, k] += x[q] - x[i, j, k]
    np.testing.assert_allclose(P.divergence(faces), lap, atol=1e-12)
    np.testing.assert_allclose((P.laplacian(R) @ x.reshape(-1)).reshape(R, R, R), -lap, atol=1e-12)


def test_linear_chi_is_reproduced_from_its_gradient():
    R = 8
    i, j, k = np.meshgrid(*[np.arange(R)] * 3, indexing="ij")
    chi = 0.3 * i - 1.1 * j + 0.7 * k
    faces = np.zeros((3, R, R, R))
    for a, c in enumerate((0.3, -1.1, 0.7)):
        sl = [slice(None)] * 3
        sl[a] = slice(0, R - 1)
        faces[a][tuple(sl)] = c
    got = P.solve(np.zeros((R, R, R)), faces, 0.0)
    np.testing.assert_allclose(got, chi - chi.mean(), atol=1e-9)


def _sphere(n, r=0.6, seed=0):
    v = np.random.default_rng(seed).normal(size=(n, 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    return (r * v).astype(np.float32), v.astype(np.float32)


def _torus(n, R=0.5, r=0.2, seed=0):
    g = np.random.default_rng(seed)
    th = g.uniform(0, 2 * np.pi, 4 * n)
    th = th[g.uniform(0, 1, th.shape[0]) < (R + r * np.cos(th)) / (R + r)][:n]
    ph = g.uniform(0, 2 * np.pi, th.shape[0])
    nrm = np.stack([np.cos(th) * np.cos(ph), np.cos(th) * np.sin(ph), np.sin(th)], axis=1)
    p = np.stack([R * np.cos(ph), R * np.sin(ph), np.zeros_like(ph)], axis=1) + r * nrm
    return p.astype(np.float32), nrm.astype(np.float32)


@pytest.mark.parametrize("shape", ["sphere", "torus"])
def test_oracle_surface_within_one_cell(shape):
    p, n = (_sphere if shape == "sphere" else _torus)(40000)
    chi, iso, origin, h, _ = P.reconstruct_field(p, n, 6, 4.0)
    v, f, _ = M.marching_cubes(chi.astype(np.float32), iso, origin + 0.5 * h, h)
    if shape == "sphere":
        d = np.abs(np.linalg.norm(v, axis=1) - 0.6)
    else:
        q = np.linalg.norm(v[:, :2], axis=1) - 0.5
        d = np.abs(np.sqrt(q * q + v[:, 2] ** 2) - 0.2)
    assert f.shape[0] > 1000 and d.max() <= h


# ------------------------------------------------------------------------------------------------ host logic, restated
def _edges_loop(depth, threshold, dilation_itr):
    """The depth-edge rule of the `dn` exporter restated pixel by pixel: the 5-point Laplacian of 1 / (depth + 1e-6)
    with zeros outside the image, > threshold, then dilation_itr dilations by the 3x3 box (zeros outside)."""
    d = depth[..., 0].astype(np.float32)
    H, W = d.shape
    inv = (1.0 / (d + np.float32(1e-6))).astype(np.float32)
    pad = np.zeros((H + 2, W + 2), np.float32)
    pad[1:-1, 1:-1] = inv
    edges = np.zeros((H, W), bool)
    for i in range(H):
        for j in range(W):
            lap = pad[i, j + 1] + pad[i + 2, j + 1] + pad[i + 1, j] + pad[i + 1, j + 2] - 4 * pad[i + 1, j + 1]
            edges[i, j] = lap > threshold
    for _ in range(dilation_itr):
        grown = edges.copy()
        for i in range(H):
            for j in range(W):
                grown[i, j] = edges[max(i - 1, 0):i + 2, max(j - 1, 0):j + 2].any()
        edges = grown
    return edges


def test_find_depth_edges_matches_loop():
    from dn_splatter_b200.poisson import find_depth_edges

    g = torch.Generator().manual_seed(0)
    d = 1 + 3 * torch.rand(40, 56, 1, generator=g)
    d[10:20, 5:30] = 0.5
    d[30:33, 40:44] = 9.0
    for thr, it in ((0.004, 10), (0.01, 3), (0.5, 0), (0.3, 1)):
        got = find_depth_edges(d, thr, it)
        assert got.shape == (40, 56, 1) and set(got.unique().tolist()) <= {0.0, 1.0}
        want = _edges_loop(d.numpy(), thr, it)
        # the sums of the restated Laplacian may round differently from a convolution's; ignore pixels at the threshold
        inv = 1.0 / (d[..., 0].numpy().astype(np.float64) + 1e-6)
        assert (got[..., 0].numpy() == want).mean() > 0.999, (thr, it)
        if it == 0:
            pad = np.pad(inv, 1)
            lap = pad[:-2, 1:-1] + pad[2:, 1:-1] + pad[1:-1, :-2] + pad[1:-1, 2:] - 4 * inv
            sure = np.abs(lap - thr) > 1e-4 * np.abs(inv).max()
            assert np.array_equal(got[..., 0].numpy()[sure] > 0, want[sure])


def test_surface_normal_conversion_matches_per_pixel_restatement():
    """The `dn` exporter's normal rule, restated per pixel in fp64: a surface-normal pixel s in [0,1]^3 is the camera
    normal 2s - 1 with y and z flipped (OpenCV -> OpenGL), normalised, and rotated by the flipped camera-to-world."""
    from dn_splatter_b200.cameras import Cameras
    from dn_splatter_b200.poisson import flipped_c2w, surface_normals_to_world
    from dn_splatter_b200.synthetic import look_at_c2w

    cam = Cameras(look_at_c2w(torch.tensor([0.3, -1.0, 0.5]), torch.zeros(3), torch.tensor([0.0, 0.0, 1.0]))[None],
                  50.0, 50.0, 16.0, 12.0, 32, 24)
    c2w_gl = cam.camera_to_worlds.reshape(3, 4).double().numpy()
    flip = np.diag([1.0, -1.0, -1.0])
    want_c2w = np.concatenate([c2w_gl[:, :3] @ flip, c2w_gl[:, 3:]], axis=1)
    c2w = flipped_c2w(cam)
    np.testing.assert_allclose(c2w.double().numpy(), want_c2w, atol=1e-7)
    sn = torch.rand(24, 32, 3, generator=torch.Generator().manual_seed(1))
    sn[0, 0] = 0.5  # the zero normal of the image border stays zero
    got = surface_normals_to_world(sn, c2w).double().numpy()
    rot = c2w.double().numpy()[:, :3]
    for k, s in enumerate(sn.reshape(-1, 3).double().numpy()):
        n = flip @ (2 * s - 1)
        n = n / max(np.linalg.norm(n), 1e-12)
        np.testing.assert_allclose(got[k], rot @ n, atol=1e-6)
    assert np.abs(got[0]).max() < 1e-6


def test_samples_per_frame():
    from dn_splatter_b200.poisson import samples_per_frame

    for total, n in ((2_000_000, 200), (2_000_000, 7), (10, 3), (1, 1)):
        assert samples_per_frame(total, n) * n >= total  # every view gets its share, rounded up
        assert samples_per_frame(total, n) == total // n + 1


def test_density_grad_is_refused():
    from dn_splatter_b200.poisson import export_dn_poisson_mesh

    with pytest.raises(NotImplementedError, match="density_grad"):
        export_dn_poisson_mesh(None, [], "/nonexistent", normal_method="density_grad")


# ------------------------------------------------------------------------------------------------ point-cloud helpers
def test_voxel_down_sample_matches_loop():
    from dn_splatter_b200.poisson import voxel_down_sample

    g = np.random.default_rng(3)
    p = g.uniform(-1, 1, (3000, 3)).astype(np.float32)
    n, c = g.normal(size=p.shape).astype(np.float32), g.uniform(0, 1, p.shape).astype(np.float32)
    vp, vn, vc = voxel_down_sample(torch.from_numpy(p), torch.from_numpy(n), torch.from_numpy(c), 0.3)
    key = np.floor((p.astype(np.float64) - (p.min(0).astype(np.float64) - 0.15)) / 0.3).astype(np.int64)  # Open3D [EXT]
    groups = {}
    for i, k in enumerate(map(tuple, key)):
        groups.setdefault(k, []).append(i)
    want = sorted(groups)
    assert vp.shape[0] == len(want)
    for r, k in enumerate(want):
        ids = groups[k]
        np.testing.assert_allclose(vp[r].numpy(), p[ids].astype(np.float64).mean(0), atol=1e-6)
        np.testing.assert_allclose(vn[r].numpy(), n[ids].astype(np.float64).mean(0), atol=1e-6)
        np.testing.assert_allclose(vc[r].numpy(), c[ids].astype(np.float64).mean(0), atol=1e-6)


def test_filter_smooth_laplacian_matches_loop():
    from dn_splatter_b200.mesh import TriangleMesh
    from dn_splatter_b200.poisson import filter_smooth_laplacian

    v, f, _ = M.marching_cubes(np.fromfunction(lambda i, j, k: np.sqrt((i - 5.2) ** 2 + (j - 4.9) ** 2 + (k - 5.1) ** 2),
                                               (11, 11, 11)).astype(np.float32), 3.7, (0, 0, 0), 0.1)
    col = np.random.default_rng(6).uniform(0, 1, v.shape).astype(np.float32)
    out = filter_smooth_laplacian(TriangleMesh(torch.from_numpy(v), torch.from_numpy(f.astype(np.int32)), torch.from_numpy(col)))
    got, got_c = out.vertices.numpy(), out.colors.numpy()
    nb = [set() for _ in range(v.shape[0])]
    for a, b, c in f:
        for x, y in ((a, b), (b, c), (c, a)):
            nb[x].add(y)
            nb[y].add(x)
    vd = v.astype(np.float64)
    cd = col.astype(np.float64)
    want, want_c = vd.copy(), cd.copy()
    for i in range(v.shape[0]):
        w = np.array([1.0 / np.linalg.norm(vd[i] - vd[j]) for j in nb[i]])
        for x, y in ((vd, want), (cd, want_c)):  # Open3D's default scope smooths the colours with the same weights [EXT]
            avg = (w[:, None] * x[list(nb[i])]).sum(0) / w.sum()
            y[i] = x[i] + 0.5 * (avg - x[i])
    np.testing.assert_allclose(got, want, atol=1e-6)
    np.testing.assert_allclose(got_c, want_c, atol=1e-6)


def test_statistical_outlier_rule_matches_loop():
    """The selection rule of remove_statistical_outlier (k-NN from the device index) on a brute-force k-NN."""
    g = np.random.default_rng(4)
    p = np.concatenate([g.normal(size=(400, 3)) * 0.1, g.uniform(-3, 3, (8, 3))])
    k, ratio = 20, 2.0
    d = np.linalg.norm(p[:, None] - p[None], axis=-1)
    avg = np.sort(d, axis=1)[:, :k].mean(1)  # the point itself (distance 0) included
    keep = np.nonzero(avg <= avg.mean() + ratio * avg.std(ddof=1))[0]
    assert set(range(400, 408)) - set(keep.tolist())  # the far points go
    if not torch.cuda.is_available():
        return
    from dn_splatter_b200.poisson import remove_statistical_outlier

    got = remove_statistical_outlier(torch.from_numpy(p).float().cuda(), k, ratio).cpu().numpy()
    assert np.array_equal(got, keep)


def test_point_cloud_ply_round_trip(tmp_path):
    from dn_splatter_b200.poisson import read_point_cloud_ply, write_point_cloud_ply

    g = torch.Generator().manual_seed(5)
    p, n, c = torch.randn(77, 3, generator=g), torch.randn(77, 3, generator=g), torch.rand(77, 3, generator=g) * 1.2 - 0.1
    path = str(tmp_path / "pcd.ply")
    write_point_cloud_ply(path, p, n, c)
    bp, bn, bc = read_point_cloud_ply(path)
    assert torch.equal(bp, p) and torch.equal(bn, n)
    np.testing.assert_allclose(bc.numpy(), np.round(np.clip(c.numpy(), 0, 1) * 255) / 255, atol=1e-7)
    head = open(path, "rb").read(400).split(b"end_header")[0].decode()
    assert [l.split()[-1] for l in head.splitlines() if l.startswith("property")] == \
        ["x", "y", "z", "nx", "ny", "nz", "red", "green", "blue"]


def test_trim_low_density_drops_faces_of_removed_vertices():
    from dn_splatter_b200.mesh import TriangleMesh
    from dn_splatter_b200.poisson import trim_low_density

    v = torch.arange(30, dtype=torch.float32).reshape(10, 3)
    f = torch.tensor([[0, 1, 2], [2, 3, 4], [5, 6, 7], [7, 8, 9], [0, 9, 5]], dtype=torch.int32)
    dens = torch.tensor([5.0, 0.1, 4, 4, 4, 4, 4, 4, 4, 4])
    out = trim_low_density(TriangleMesh(v, f, v * 0.01), dens)
    thr = np.quantile(dens.numpy().astype(np.float64), 0.01)
    keep = dens.numpy() >= thr
    assert out.vertices.shape[0] == keep.sum() == 9
    assert out.faces.tolist() == [[1, 2, 3], [4, 5, 6], [6, 7, 8], [0, 8, 4]]
    assert torch.equal(out.colors, v[torch.from_numpy(keep)] * 0.01)


# ------------------------------------------------------------------------------------------------ C entry points
@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(L.LIB_PATH):
        from dn_splatter_b200.build import build

        build()
    return L.load()


def test_argument_errors_are_negative_codes(lib):
    one = C.c_void_p(16)  # non-NULL dummy: checks come first, nothing is dereferenced
    g = L.DnrPoissonGrid()
    assert lib.dnr_poisson_splat_workspace_bytes(None, 10) == -1
    assert lib.dnr_poisson_splat_workspace_bytes(C.byref(g), 10) == -2  # depth 0
    g.depth, g.cell = 11, 0.1
    assert lib.dnr_poisson_splat_workspace_bytes(C.byref(g), 10) == -2  # depth > 10
    g.depth = 6
    assert lib.dnr_poisson_splat_workspace_bytes(C.byref(g), 0) == -2
    ws = lib.dnr_poisson_splat_workspace_bytes(C.byref(g), 1000)
    assert ws >= 4 * 64 ** 3 * 2 + 1000 * 48
    args = [one] * 7
    assert lib.dnr_poisson_splat(C.byref(g), None, one, None, 1000, one, ws, *args[:3], None, one, one, None) == -1
    assert lib.dnr_poisson_splat(C.byref(g), one, one, one, 1000, one, ws, *args[:3], None, one, one, None) == -1  # colours
    assert lib.dnr_poisson_splat(C.byref(g), one, one, None, 1000, one, ws - 1, *args[:3], None, one, one, None) == -5
    assert lib.dnr_poisson_solve_workspace_bytes(C.byref(g), 0) == -2
    assert lib.dnr_poisson_solve_workspace_bytes(C.byref(g), 101) == -2
    sws = lib.dnr_poisson_solve_workspace_bytes(C.byref(g), 10)
    assert sws >= 4 * 64 ** 3
    hist, cyc = (C.c_float * 11)(), C.c_int32()
    assert lib.dnr_poisson_solve(C.byref(g), one, one, -1.0, 1e-5, 10, one, sws, one, hist, C.byref(cyc), None) == -2
    assert lib.dnr_poisson_solve(C.byref(g), one, None, 4.0, 1e-5, 10, one, sws, one, hist, C.byref(cyc), None) == -1
    assert lib.dnr_poisson_solve(C.byref(g), one, one, 4.0, 1e-5, 10, one, sws - 1, one, hist, C.byref(cyc), None) == -5
    d = L.DnrGridDesc()
    assert lib.dnr_grid_sample(None, one, one, 5, one, None) == -1
    assert lib.dnr_grid_sample(C.byref(d), one, one, 5, one, None) == -2
    d.dims[0] = d.dims[1] = d.dims[2] = 4
    d.cell, d.channels = 0.5, 1
    assert lib.dnr_grid_sample(C.byref(d), None, one, 5, one, None) == -1
    assert lib.dnr_grid_sample(C.byref(d), None, None, 0, None, None) == 0  # nothing to do


def test_grid_budget_names_the_bytes(lib):
    from dn_splatter_b200.poisson import DEFAULT_MAX_BYTES, required_bytes

    assert required_bytes(10, 2_000_000) <= DEFAULT_MAX_BYTES
    assert required_bytes(9, 2_000_000) < required_bytes(10, 2_000_000) / 6
    assert math.isclose(required_bytes(8, 1) / 256 ** 3, 4 * 6, rel_tol=0.25)
