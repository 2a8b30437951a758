"""Screened Poisson reconstruction (csrc/poisson.cu, dn_splatter_b200.poisson) against the fp64 oracle
(oracle/poisson_ref.py), its solver and geometry on analytic shapes, and the three Poisson exporters on the closed room
of flat Gaussians of tests/test_gpu_mesh.py."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import poisson_ref as P

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]


def _sphere(n, dense_half=1, seed=0, r=0.6):
    """n oriented samples on a sphere; the z > 0 hemisphere sampled dense_half times denser."""
    g = np.random.default_rng(seed)
    v = g.normal(size=(n * (dense_half + 1), 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    keep = (v[:, 2] > 0) | (np.arange(v.shape[0]) % dense_half == 0)
    v = v[keep][: n if dense_half == 1 else None]
    return (r * v + np.array([0.03, -0.02, 0.01])).astype(np.float32), v.astype(np.float32)


def _torus(n, dense_half=1, seed=0, R=0.5, r=0.2):
    g = np.random.default_rng(seed)
    m = n * (dense_half + 1)
    # area-uniform: accept theta with probability (R + r cos(theta)) / (R + r)
    th = g.uniform(0, 2 * np.pi, 4 * m)
    th = th[g.uniform(0, 1, th.shape[0]) < (R + r * np.cos(th)) / (R + r)][:m]
    ph = g.uniform(0, 2 * np.pi, th.shape[0])
    nrm = np.stack([np.cos(th) * np.cos(ph), np.cos(th) * np.sin(ph), np.sin(th)], axis=1)
    c = np.stack([R * np.cos(ph), R * np.sin(ph), np.zeros_like(ph)], axis=1)
    p = c + r * nrm
    keep = (p[:, 2] > 0) | (np.arange(p.shape[0]) % dense_half == 0)
    p, nrm = p[keep], nrm[keep]
    if dense_half == 1:
        p, nrm = p[:n], nrm[:n]
    return p.astype(np.float32), nrm.astype(np.float32)


def _dist_sphere(v, r=0.6):
    return np.abs(np.linalg.norm(v - np.array([0.03, -0.02, 0.01]), axis=1) - r)


def _dist_torus(v, R=0.5, r=0.2):
    q = np.linalg.norm(v[:, :2], axis=1) - R
    return np.abs(np.sqrt(q * q + v[:, 2] ** 2) - r)


def _cuda(*a):
    return [None if x is None else torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in a]


def _rel(got, want):
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-30))


@pytest.mark.parametrize("depth", [5, 6])
def test_splat_matches_oracle(depth):
    from dn_splatter_b200.poisson import poisson_grid, poisson_splat

    p, n = _sphere(30000, dense_half=10, seed=depth)
    col = np.random.default_rng(1).uniform(0, 1, p.shape).astype(np.float32)
    pt, nt, ct = _cuda(p, n, col)
    grid = poisson_grid(pt, depth)
    got = poisson_splat(pt, nt, ct, grid)
    want = P.splat(p, n, col, np.array(grid.origin), grid.cell, depth)
    R = 1 << depth
    assert _rel(got["screen"].cpu().numpy().reshape(R, R, R), want["screen"]) <= 1e-6
    assert _rel(got["faces"].cpu().numpy().reshape(3, R, R, R), want["faces"]) <= 1e-6
    assert _rel(got["density"].cpu().numpy().reshape(R // 4, R // 4, R // 4), want["density"]) <= 1e-6
    assert _rel(got["colors"].cpu().numpy().reshape(R // 4, R // 4, R // 4, 4), want["colors"]) <= 1e-6
    assert _rel(got["weights"].cpu().numpy(), want["weights"]) <= 1e-6
    assert abs(float(got["area_scale"]) / want["area_scale"] - 1) <= 1e-6
    assert want["weights"].max() > 3 * want["weights"].min()  # the dense hemisphere is down-weighted


def test_grid_sample_matches_oracle():
    """Six point sets, each from the same seed: random points around the grid, points on node centres, points whose
    floor(x) is the last node (the clamp), an axis with one node, 4 channels, and no points; every grid is also read
    one channel at a time."""
    from dn_splatter_b200.poisson import grid_sample

    for case in ("random", "centres", "clamp", "dims1", "channels4", "empty"):
        g = np.random.default_rng(2)
        dims = np.array([9, 1, 7] if case == "dims1" else [9, 13, 7])
        vals = g.normal(size=(*dims, 4 if case == "channels4" else 3)).astype(np.float32)
        origin, cell = (-0.3, 0.2, -1.0), 0.17
        n = 0 if case == "empty" else 5000
        if case == "centres":
            x = g.integers(0, dims, (n, 3)) + 0.5
        elif case == "clamp":  # floor(x - 0.5) == dims - 1 on one axis, exactly at the last centre for some
            x = g.uniform(-0.3, 1.2, (n, 3)) * dims
            ax = g.integers(0, 3, n)
            x[np.arange(n), ax] = dims[ax] - 0.5 + np.where(np.arange(n) % 4 == 0, 0.0, g.uniform(0, 1, n))
        else:
            x = g.uniform(-0.3, 1.2, (n, 3)) * dims
        pts = (np.array(origin) + x * cell).astype(np.float32)
        vt, pt = _cuda(vals, pts)
        for v, w in ((vt, vals), (vt[..., 1].contiguous(), vals[..., 1])):
            got = grid_sample(v, origin, cell, pt).cpu().numpy()
            assert got.shape == (n,) + w.shape[3:], case
            want = P.sample(w, origin, cell, pts)
            assert np.abs(got - want).max(initial=0.0) <= 1e-6 * np.abs(w).max(), case


@pytest.mark.parametrize("depth", [4, 5, 6])
@pytest.mark.parametrize("alpha", [0.0, 4.0])
def test_multigrid_matches_direct_solve(depth, alpha):
    from dn_splatter_b200.poisson import poisson_grid, poisson_solve, poisson_splat

    p, n = _torus(30000, seed=depth)
    pt, nt = _cuda(p, n)
    grid = poisson_grid(pt, depth)
    sp = poisson_splat(pt, nt, None, grid)
    sigma = alpha * float(sp["area_scale"])
    chi, hist = poisson_solve(grid, sp["screen"], sp["faces"], sigma, tol=1e-7, max_cycles=40)
    R = 1 << depth
    got = chi.cpu().numpy().reshape(R, R, R).astype(np.float64)
    want = P.solve(sp["screen"].cpu().numpy().astype(np.float64).reshape(R, R, R),
                   sp["faces"].cpu().numpy().astype(np.float64).reshape(3, R, R, R), np.float32(sigma))
    if alpha == 0:
        got, want = got - got.mean(), want - want.mean()
    err = np.abs(got - want).max() / (want.max() - want.min())
    print(f"depth {depth} alpha {alpha}: cycles {len(hist) - 1} residual {hist[-1]:.2e} chi err / range {err:.2e}")
    assert err <= 1e-4


@pytest.mark.parametrize("depth", [7, 8])
def test_residual_history(depth):
    from dn_splatter_b200.poisson import DEFAULT_POINT_WEIGHT, poisson_grid, poisson_solve, poisson_splat

    p, n = _sphere(400000, seed=depth)
    pt, nt = _cuda(p, n)
    grid = poisson_grid(pt, depth)
    sp = poisson_splat(pt, nt, None, grid)
    for alpha in (0.0, DEFAULT_POINT_WEIGHT):
        _, hist = poisson_solve(grid, sp["screen"], sp["faces"], alpha * float(sp["area_scale"]), tol=1e-5, max_cycles=30)
        rates = [hist[i + 1] / hist[i] for i in range(len(hist) - 1)]
        print(f"depth {depth} alpha {alpha}: cycles {len(hist) - 1}, residuals {['%.2e' % h for h in hist]}")
        assert hist[-1] <= 1e-5
        if alpha == 0:
            assert max(rates) <= 0.2, rates
        else:
            # screened: the coarse levels carry the row-sum (lumped) restriction of S, not the Galerkin product, and a
            # thin shell of strong screening is what lumping represents worst; the rate settles near 0.5 (DESIGN.md §2)
            assert rates[0] <= 0.2 and max(rates) <= 0.6, rates


def _manifold(v, f):
    """(closed 2-manifold with consistent orientation, Euler characteristic)."""
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]).astype(np.int64)
    directed = np.unique(e[:, 0] * v.shape[0] + e[:, 1])
    und, cnt = np.unique(np.sort(e, axis=1)[:, 0] * v.shape[0] + np.sort(e, axis=1)[:, 1], return_counts=True)
    closed = directed.shape[0] == e.shape[0] and (cnt == 2).all()
    return closed, v.shape[0] - und.shape[0] + f.shape[0]


def _face_normal_agreement(v, f, p, n):
    from scipy.spatial import cKDTree

    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    fn = np.cross(b - a, c - a)
    fn /= np.maximum(np.linalg.norm(fn, axis=1, keepdims=True), 1e-30)
    _, nearest = cKDTree(p).query((a + b + c) / 3)
    return float(((fn * n[nearest]).sum(1) >= math.cos(math.radians(30))).mean())


@pytest.mark.parametrize("depth", [7, 8])
@pytest.mark.parametrize("shape", ["sphere", "torus"])
@pytest.mark.parametrize("dense_half", [1, 10])
def test_geometry(depth, shape, dense_half):
    from dn_splatter_b200.poisson import poisson_solve_points

    make, dist, euler = (_sphere, _dist_sphere, 2) if shape == "sphere" else (_torus, _dist_torus, 0)
    p, n = make(200000, dense_half=dense_half, seed=depth)
    pt, nt = _cuda(p, n)
    r = poisson_solve_points(pt, nt, depth=depth)
    v, f = r.mesh.vertices.cpu().numpy(), r.mesh.faces.cpu().numpy()
    closed, chi_e = _manifold(v, f)
    err = dist(v).max() / r.grid.cell
    agree = _face_normal_agreement(v, f, p, n)
    print(f"{shape} depth {depth} dense {dense_half}: V {v.shape[0]} F {f.shape[0]} euler {chi_e} max err {err:.3f} cells, "
          f"normals {agree:.4f}, cycles {len(r.residuals) - 1}")
    assert closed and chi_e == euler
    assert err <= 1.0
    assert agree >= 0.99


def test_deterministic():
    from dn_splatter_b200.poisson import poisson_reconstruct

    p, n = _torus(300000, dense_half=4, seed=3)
    col = np.random.default_rng(3).uniform(0, 1, p.shape).astype(np.float32)
    pt, nt, ct = _cuda(p, n, col)
    a = poisson_reconstruct(pt, nt, ct, depth=8)
    b = poisson_reconstruct(pt, nt, ct, depth=8)
    for x, y in ((a[0].vertices, b[0].vertices), (a[0].faces, b[0].faces), (a[0].colors, b[0].colors), (a[1], b[1])):
        assert torch.equal(x, y)


def test_depth_10_fits_and_completes():
    from dn_splatter_b200.poisson import DEFAULT_MAX_BYTES, poisson_solve_points, required_bytes

    p, n = _sphere(2_000_000, seed=10)
    assert required_bytes(10, p.shape[0]) <= DEFAULT_MAX_BYTES
    pt, nt = _cuda(p, n)
    r = poisson_solve_points(pt, nt, depth=10)
    err = _dist_sphere(r.mesh.vertices.cpu().numpy()).max() / r.grid.cell
    print(f"depth 10: cycles {len(r.residuals) - 1} residual {r.residuals[-1]:.2e} faces {r.mesh.faces.shape[0]} err {err:.3f}")
    assert r.mesh.faces.shape[0] > 1_000_000 and r.residuals[-1] <= 1e-5
    with pytest.raises(ValueError, match="GiB"):
        poisson_solve_points(pt, nt, depth=10, max_bytes=1 << 30)


# ------------------------------------------------------------------------------------------------ the room
@pytest.fixture(scope="module")
def room():
    from dn_splatter_b200.dn_model import DNSplatterModelConfig
    from tests.test_gpu_mesh import _room

    params, cams = _room()
    m = DNSplatterModelConfig(random_init=True, num_random=16, background_color="black").setup(device="cuda")
    m.load_gaussians(params)
    m.step = 30000
    m.eval()
    m.get_outputs(cams[0])  # sets model.normals
    return m, cams


def _observed(v, samples, radius):
    """Vertices with a sample within radius."""
    from scipy.spatial import cKDTree

    return cKDTree(samples).query(v, distance_upper_bound=radius)[0] <= radius


def _largest_component_share(f, nv):
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components

    adj = coo_matrix((np.ones(3 * f.shape[0]), (np.repeat(f[:, 0], 3), f.reshape(-1))), shape=(nv, nv))
    _, lab = connected_components(adj, directed=False)
    return np.bincount(lab[f[:, 0]]).max() / f.shape[0]


def test_dn_exporter_on_the_room(room, tmp_path):
    from dn_splatter_b200.mesh import read_ply
    from dn_splatter_b200.poisson import DN_MESH_NAME, DN_PCD_NAME, export_dn_poisson_mesh, read_point_cloud_ply
    from tests.test_gpu_mesh import WALL_RGB, _wall_distance

    m, cams = room
    mesh, (pts, nrm, col) = export_dn_poisson_mesh(m, cams, str(tmp_path), total_points=1_000_000, poisson_depth=8)
    p, n = pts.cpu().numpy(), nrm.cpu().numpy()
    assert (np.abs(_wall_distance(p)) <= 0.02).mean() >= 0.99
    # the depth-derived normal map is undefined (0.5, i.e. a zero normal) on the 1-pixel image border, as upstream:
    # those samples add no flux; every other normal must face the inside of the room, where the cameras are
    defined = np.linalg.norm(n, axis=1) > 0.5
    assert (~defined).mean() <= 1.5 * 2 * (320 + 240) / (320 * 240)  # the border's share of the pixels, with slack
    assert ((n[defined] * -p[defined]).sum(axis=1) > 0).mean() >= 0.99
    # the rendered depth of a wall of opaque Gaussians 0.01 thick lies about 0.01 in front of the wall's plane, so the
    # samples, and the surface through them, are a box that much smaller: distances are measured from that offset
    offset = float(np.median(_wall_distance(p)))
    assert 0.005 < offset < 0.015
    v, f, c = mesh.vertices.cpu().numpy(), mesh.faces.cpu().numpy(), mesh.colors.cpu().numpy()
    h = 2.0 * 1.1 / 256
    inner = np.sort(np.abs(v), axis=1)[:, 1] < 0.85  # away from the box's edges, where depth blends two walls
    near = np.abs(_wall_distance(v) - offset) <= 1.5 * h
    # 48 random views from near the centre leave wall patches no view sees; Poisson closes them with a smooth membrane
    # that bows off the wall and that no sample colours.  The bounds hold where a sample lies within 2 cells.
    observed = _observed(v, p, 2 * h)
    print(f"dn: offset {offset:.4f}; observed inner vertices within 1.5 cells of it {near[inner & observed].mean():.4f}, "
          f"unobserved {near[inner & ~observed].mean():.4f} of {(inner & ~observed).sum()}; all {near.mean():.4f}")
    assert inner.mean() > 0.5 and (inner & observed).mean() > 0.5 and near[inner & observed].mean() >= 0.99
    assert _largest_component_share(f, v.shape[0]) >= 0.95
    vax = np.argmin(1.0 - np.abs(v), axis=1)
    face = 2 * vax + (v[np.arange(v.shape[0]), vax] > 0)
    sel = inner & near & observed
    err = np.abs(c[sel] - np.asarray(WALL_RGB, np.float32)[face[sel]]).max(axis=1)
    bad = inner & near & ~observed
    print(f"dn: colour error of observed inner vertices max {err.max():.2e}; unobserved ones within 3/255: "
          f"{(np.abs(c[bad] - np.asarray(WALL_RGB, np.float32)[face[bad]]).max(axis=1) <= 3 / 255).mean():.4f}")
    assert sel.sum() > 1000 and (err <= 3 / 255).all(), float(err.max())
    back = read_ply(str(tmp_path / DN_MESH_NAME))
    assert torch.equal(back.vertices, mesh.vertices.cpu()) and torch.equal(back.faces, mesh.faces.cpu())
    bp, bn, bc = read_point_cloud_ply(str(tmp_path / DN_PCD_NAME))
    assert torch.equal(bp, pts.cpu()) and torch.equal(bn, nrm.cpu())
    np.testing.assert_allclose(bc.numpy(), np.round(np.clip(col.cpu().numpy(), 0, 1) * 255) / 255, atol=1e-6)


def test_gaussians_exporter_on_the_room(room, tmp_path):
    from dn_splatter_b200.poisson import GAUSSIANS_MESH_NAME, GAUSSIANS_PCD_NAME, export_gaussians_poisson_mesh
    from tests.test_gpu_mesh import _wall_distance

    m, _ = room
    mesh, _ = export_gaussians_poisson_mesh(m, str(tmp_path), poisson_depth=8)
    v, f = mesh.vertices.cpu().numpy(), mesh.faces.cpu().numpy()
    h = 2.0 * 1.1 / 256
    assert f.shape[0] > 10000
    assert (np.abs(_wall_distance(v)) <= 1.5 * h).mean() >= 0.99
    assert _largest_component_share(f, v.shape[0]) >= 0.95
    assert os.path.exists(tmp_path / GAUSSIANS_MESH_NAME) and os.path.exists(tmp_path / GAUSSIANS_PCD_NAME)


def test_level_set_exporter_on_the_room(room, tmp_path):
    from dn_splatter_b200.poisson import export_level_set_poisson_mesh, read_point_cloud_ply
    from tests.test_gpu_mesh import _wall_distance

    m, cams = room
    levels = (0.1, 0.3, 0.5)
    meshes = export_level_set_poisson_mesh(m, cams[:12], str(tmp_path), total_points=600_000, surface_levels=levels,
                                           poisson_depth=8)
    h = 2.0 * 1.1 / 256
    for lv in levels:
        tag = f"surface_level_{lv}_closest_gaussian.ply"
        for name in (f"before_clean_points_{tag}", f"after_clean_points_{tag}", f"poisson_mesh_{tag}",
                     f"smoothed_1_poisson_mesh_{tag}", f"smoothed_2_poisson_mesh_{tag}"):
            assert os.path.exists(tmp_path / name), name
        v, f = meshes[lv].vertices.cpu().numpy(), meshes[lv].faces.cpu().numpy()
        assert f.shape[0] > 10000
        assert _largest_component_share(f, v.shape[0]) >= 0.95
        # a level set of the 0.01-thick walls lies in front of them by a distance set by the level; with 12 views many
        # wall patches are unseen and closed by a membrane that bows off the wall (see the dn test)
        p = read_point_cloud_ply(str(tmp_path / f"after_clean_points_{tag}"))[0].numpy()
        offset = float(np.median(_wall_distance(p)))
        inner = np.sort(np.abs(v), axis=1)[:, 1] < 0.85
        near = np.abs(_wall_distance(v) - offset) <= 1.5 * h
        observed = _observed(v, p, 2 * h)
        print(f"level {lv}: sample offset {offset:.4f} (q1-q99 {np.quantile(_wall_distance(p), [0.01, 0.99])}); observed "
              f"inner vertices within 1.5 cells of it {near[inner & observed].mean():.4f}, unobserved "
              f"{near[inner & ~observed].mean():.4f} of {(inner & ~observed).sum()}; all {near.mean():.4f}")
        assert (inner & observed).mean() > 0.3 and near[inner & observed].mean() >= 0.99
