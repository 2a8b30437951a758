"""Mesh export without a GPU: the generated marching-cubes tables, the numpy oracle (oracle/mesh_ref.py) on analytic
fields and depth maps, the host logic of dn_splatter_b200.mesh, and the argument checks of the new C ABI."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from dn_splatter_b200 import _lib as L
from dn_splatter_b200 import mc_tables as T
from dn_splatter_b200 import mesh as M
from oracle import mesh_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------------------------- tables
def test_generator_reproduces_committed_header():
    with open(os.path.join(ROOT, "dn_splatter_b200", "csrc", "mc_tables.cuh")) as fh:
        assert fh.read() == T.header()


def test_triangles_use_exactly_the_crossed_edges():
    ntri, tris = T.tables()
    for case in range(256):
        t = np.array(tris[case]).reshape(-1, 3)
        assert t.shape[0] == ntri[case]
        assert set(t.reshape(-1).tolist()) == set(T.crossed_edges(case)), case
        assert all(len(set(row)) == 3 for row in t.tolist()), case
    assert ntri[0] == ntri[255] == 0


def _face_edges(axis, side):
    return {e for e in range(12) if T.EDGE_AXIS[e] != axis and ((T.EDGE_C0[e] >> axis) & 1) == side}


def test_face_segments_match_every_neighbour_configuration():
    """The cube across face (axis, 1) sees the same four corners on its face (axis, 0): whatever its other corners, it
    draws the same segments there, in the opposite direction."""
    for case in range(256):
        segs = T.face_segments(case)
        for a in range(3):
            ours = sorted((e0, e1) for e0, e1 in segs if {e0, e1} <= _face_edges(a, 1))
            shared = [c for c in range(8) if (c >> a) & 1]
            for other in range(16):  # the neighbour's four corners away from the shared face
                nb = 0
                for c in shared:  # our corner c is the neighbour's corner c ^ (1 << a)
                    nb |= ((case >> c) & 1) << (c ^ (1 << a))
                far = [c for c in range(8) if (c >> a) & 1]
                for bit, c in enumerate(far):
                    nb |= ((other >> bit) & 1) << c
                mapped = []
                for e0, e1 in T.face_segments(nb):
                    if {e0, e1} <= _face_edges(a, 0):
                        up = [T._EDGE_OF[frozenset((T.EDGE_C0[e] | (1 << a), T.EDGE_C0[e] | (1 << a) | (1 << T.EDGE_AXIS[e])))]
                              for e in (e0, e1)]
                        mapped.append((up[1], up[0]))
                assert sorted(mapped) == ours, (case, a, other)


# ------------------------------------------------------------------------------------------- oracle marching cubes
def _grid(n, lo=-1.0, hi=1.0):
    s = (hi - lo) / (n - 1)
    x = lo + s * np.arange(n)
    return np.meshgrid(x, x, x, indexing="ij"), s


def _closed_manifold(verts, faces):
    """Every edge in exactly two faces with opposite orientation; returns the Euler characteristic."""
    V = verts.shape[0]
    assert np.unique(faces.reshape(-1)).shape[0] == V  # welded: every vertex used
    d = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]]).astype(np.int64)
    fwd, rev = d[:, 0] * V + d[:, 1], d[:, 1] * V + d[:, 0]
    assert np.unique(fwd).shape[0] == fwd.shape[0], "a directed edge is used twice"
    assert np.array_equal(np.sort(fwd), np.sort(rev)), "an edge lacks its opposite half"
    return V - fwd.shape[0] // 2 + faces.shape[0]


def _sphere(x, y, z):
    return np.sqrt(x * x + y * y + z * z) - 0.6


def _sphere_grad(p):
    return p


def _torus(x, y, z):
    return np.sqrt((np.sqrt(x * x + y * y) - 0.55) ** 2 + z * z) - 0.25


def _torus_grad(p):
    q = np.sqrt(p[:, 0] ** 2 + p[:, 1] ** 2)
    c = np.stack([p[:, 0] / q * 0.55, p[:, 1] / q * 0.55, np.zeros_like(q)], axis=1)
    return p - c


@pytest.mark.parametrize("fn,grad,chi", [(_sphere, _sphere_grad, 2), (_torus, _torus_grad, 0)])
def test_oracle_marching_cubes_on_analytic_fields(fn, grad, chi):
    (x, y, z), s = _grid(48)
    verts, faces, _ = R.marching_cubes(fn(x, y, z).astype(np.float32), 0.0, (-1.0, -1.0, -1.0), s)
    assert faces.shape[0] > 1000
    assert _closed_manifold(verts, faces) == chi
    v = verts.astype(np.float64)
    assert np.abs(fn(v[:, 0], v[:, 1], v[:, 2])).max() < 0.05 * s  # linear interpolation of a smooth SDF
    tri = v[faces]
    n = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    dots = (n * grad(tri.mean(axis=1))).sum(axis=1)
    assert (dots > 0).all()  # counter-clockwise seen from f > iso


@pytest.mark.parametrize("seed", range(6))
def test_oracle_marching_cubes_random_fields_are_closed(seed):
    rng = np.random.default_rng(seed)
    f = rng.uniform(-1, 1, (11, 9, 13)).astype(np.float32)
    f[[0, -1]], f[:, [0, -1]], f[:, :, [0, -1]] = 1.0, 1.0, 1.0
    verts, faces, _ = R.marching_cubes(f, 0.0, (0.0, 0.0, 0.0), 1.0)
    assert faces.shape[0] > 0
    _closed_manifold(verts, faces)


def test_oracle_marching_cubes_skips_invalid_cubes():
    (x, y, z), s = _grid(20)
    f = _sphere(x, y, z).astype(np.float32)
    valid = np.ones(f.shape, bool)
    valid[10, 10, 3] = False
    v_all, f_all, _ = R.marching_cubes(f, 0.0, (-1.0,) * 3, s)
    v_cut, f_cut, _ = R.marching_cubes(f, 0.0, (-1.0,) * 3, s, valid=valid)
    assert 0 < f_all.shape[0] - f_cut.shape[0] <= 8 * T.max_triangles()


# ------------------------------------------------------------------------------------------ oracle integration
W_, H_ = 64, 48


def _cam_block(c2w_gl, fx, fy, cx, cy):
    c2w = np.eye(4)
    c2w[:3, :4] = c2w_gl
    E = np.linalg.inv(c2w @ np.diag([1.0, -1.0, -1.0, 1.0]))[:3]
    return np.array([fx, fy, cx, cy, *E.reshape(-1)], np.float64)


def _look_at(pos, target=(0.0, 0.0, 0.0), up=(0.0, 0.0, 1.0)):
    pos, target, up = (np.asarray(v, np.float64) for v in (pos, target, up))
    f = target - pos
    f /= np.linalg.norm(f)
    r = np.cross(f, up)
    r /= np.linalg.norm(r)
    u = np.cross(r, f)
    return np.stack([r, u, -f, pos], axis=1)


def _pixel_rays(cam):
    fx, fy, cx, cy = cam[:4]
    u, v = np.meshgrid(np.arange(W_), np.arange(H_))  # pixel u spans fx x / z + cx in [u - 0.5, u + 0.5)
    return (u - cx) / fx, (v - cy) / fy  # camera-frame ray (a, b, 1) through the pixel's centre


def _sphere_depth(cam, radius=0.5):
    """z-depth of the sphere at the origin along every pixel-centre ray (0 where the ray misses)."""
    E = cam[4:].reshape(3, 4)
    Rm, t = E[:, :3], E[:, 3]
    centre = t  # the world origin in the camera frame
    a, b = _pixel_rays(cam)
    d = np.stack([a, b, np.ones_like(a)], axis=-1)
    dd = (d * d).sum(-1)
    bc = (d * centre).sum(-1)
    disc = bc * bc - dd * ((centre * centre).sum() - radius * radius)
    z = (bc - np.sqrt(np.maximum(disc, 0))) / dd
    return np.where(disc > 0, z, 0.0).astype(np.float32)


def _volume(n=40, ext=0.8):
    vox = 2 * ext / n
    return R.empty_volume((n, n, n)), (-ext, -ext, -ext), vox


def test_oracle_integration_plane_matches_along_ray_distance():
    cam = _cam_block(_look_at((0.0, -2.0, 0.0)), 50.0, 50.0, W_ / 2, H_ / 2)
    depth = np.full((H_, W_), 2.0, np.float32)  # the plane y = 0, facing the camera
    rgb = np.full((H_, W_, 3), 0.5, np.float32)
    (tsdf, w, col), origin, vox = _volume()
    trunc = 0.06
    u, v = R.integrate(tsdf, w, col, origin, vox, trunc, depth, rgb, None, cam, 20.0)
    n = tsdf.shape[0]
    idx = np.stack(np.meshgrid(*[np.arange(n)] * 3, indexing="ij"), -1)
    p = np.asarray(origin) + (idx + 0.5) * vox
    pc = p @ cam[4:].reshape(3, 4)[:, :3].T + cam[4:].reshape(3, 4)[:, 3]
    along = (2.0 - pc[..., 2]) * np.linalg.norm(pc, axis=-1) / pc[..., 2]  # the voxel's own ray
    band = (w > 0) & (tsdf < 1)
    assert band.sum() > 1000
    np.testing.assert_allclose(tsdf[band] * trunc, along[band], atol=2e-3)
    assert (col[w > 0].astype(np.float32) == 127).all()  # (uint8)(0.5 * 255)
    # voxels more than sdf_trunc behind the plane are never touched
    assert not (w[pc[..., 2] > 2.0 + trunc * 1.01] > 0).any()


def test_oracle_integration_sphere_weights_count_views():
    cams = [_cam_block(_look_at((3 * np.cos(t), 3 * np.sin(t), 0.5)), 60.0, 60.0, W_ / 2, H_ / 2)
            for t in np.linspace(0, 2 * np.pi, 5)[:-1]]
    rgb = np.full((H_, W_, 3), 0.25, np.float32)
    (tsdf, w, col), origin, vox = _volume()
    trunc = 0.1
    seen = np.zeros(w.shape, np.int64)
    for cam in cams:
        depth = _sphere_depth(cam)
        (t1, w1, c1), _, _ = _volume()
        R.integrate(t1, w1, c1, origin, vox, trunc, depth, rgb, None, cam, 20.0)
        seen += w1 > 0
        R.integrate(tsdf, w, col, origin, vox, trunc, depth, rgb, None, cam, 20.0)
    assert (w == seen).all() and w.max() == len(cams)
    # the fused surface is the sphere: observed voxels inside it are negative, outside it positive
    n = w.shape[0]
    idx = np.stack(np.meshgrid(*[np.arange(n)] * 3, indexing="ij"), -1)
    r = np.linalg.norm(np.asarray(origin) + (idx + 0.5) * vox, axis=-1)
    obs = w > 0
    assert (tsdf[obs & (r < 0.5 - 0.03)] < 0).mean() > 0.95 and (tsdf[obs & (r > 0.5 + 0.03)] > 0).mean() > 0.9
    # fp32 restatement against fp64
    t64, w64, c64 = R.empty_volume(w.shape, np.float64)
    for cam in cams:
        R.integrate(t64, w64, c64, origin, vox, trunc, _sphere_depth(cam), rgb, None, cam, 20.0, dtype=np.float64)
    same = w64 == w
    assert same.mean() > 0.999
    np.testing.assert_allclose(tsdf[same & (w > 0)], t64[same & (w > 0)], atol=1e-4)


def test_oracle_integration_depth_trunc_mask_and_half_pixel():
    cam = _cam_block(_look_at((0.0, -2.0, 0.0)), 50.0, 50.0, W_ / 2, H_ / 2)
    depth = np.full((H_, W_), 2.0, np.float32)
    depth[:, W_ // 2:] = 2.3
    rgb = np.full((H_, W_, 3), 0.5, np.float32)
    trunc = 0.1

    def run(depth_trunc=20.0, mask=None):
        (tsdf, w, col), origin, vox = _volume()
        u, v = R.integrate(tsdf, w, col, origin, vox, trunc, depth, rgb, mask, cam, depth_trunc)
        return w > 0, u, v, (origin, vox)

    base, u, v, (origin, vox) = run()
    cut, _, _, _ = run(depth_trunc=2.1)
    assert np.array_equal(cut, base & (u < W_ // 2))  # only the pixels beyond depth_trunc drop out
    mask = np.zeros((H_, W_), np.uint8)
    mask[: H_ // 2] = 1
    masked, _, _, _ = run(mask=mask)
    assert np.array_equal(masked, base & (v < H_ // 2))
    # the pixel is int(fx x / z + cx + 0.5): a projection whose fraction is >= 0.5 reads the next pixel
    n = base.shape[0]
    idx = np.stack(np.meshgrid(*[np.arange(n)] * 3, indexing="ij"), -1)
    p = np.asarray(origin) + (idx + 0.5) * vox
    E = cam[4:].reshape(3, 4)
    pc = p @ E[:, :3].T + E[:, 3]
    uu = cam[0] * pc[..., 0] / pc[..., 2] + cam[2]
    frac = uu - np.floor(uu)
    clear = base & (np.abs(frac - 0.5) > 1e-3) & (frac > 1e-3) & (frac < 1 - 1e-3)
    want = np.floor(uu).astype(np.int64) + (frac >= 0.5)
    assert clear.sum() > 1000 and ((frac >= 0.5) & clear).sum() > 100
    assert np.array_equal(u[clear], want[clear])


# -------------------------------------------------------------------------------------------------- host logic
def test_bounds_snap_outward_to_the_voxel_lattice():
    origin, dims = M.snap_bounds(((-0.013, 0.0, 0.21), (0.5, 0.02, 0.3)), 0.02)
    np.testing.assert_allclose(origin, [-0.02, 0.0, 0.2])
    assert dims == [26, 1, 5]
    # voxel centres on (k + 0.5) * voxel
    c = np.asarray(origin) + 0.5 * 0.02
    np.testing.assert_allclose(np.round(c / 0.02 - 0.5), c / 0.02 - 0.5, atol=1e-9)


def test_max_bytes_guard_names_the_voxel_count():
    with pytest.raises(ValueError, match=r"1000000 voxels.*coarser voxel_size or tighter bounds"):
        M.TSDFVolume(((0, 0, 0), (1, 1, 1)), voxel_size=0.01, max_bytes=1 << 20, device="cpu")


def _mesh(verts, faces, colors=None):
    return M.TriangleMesh(torch.as_tensor(np.asarray(verts, np.float32)), torch.as_tensor(np.asarray(faces, np.int32)),
                          None if colors is None else torch.as_tensor(np.asarray(colors, np.float32)))


def test_ply_round_trip(tmp_path):
    rng = np.random.default_rng(0)
    m = _mesh(rng.normal(size=(30, 3)), rng.integers(0, 30, (50, 3)), rng.uniform(-0.2, 1.2, (30, 3)))
    p = str(tmp_path / "m.ply")
    M.write_ply(p, m)
    with open(p, "rb") as fh:
        assert fh.read(64).startswith(b"ply\nformat binary_little_endian 1.0\nelement vertex 30\n")
    back = M.read_ply(p)
    assert torch.equal(back.vertices, m.vertices) and torch.equal(back.faces, m.faces)
    want = np.round(np.clip(m.colors.numpy(), 0, 1) * 255) / 255
    np.testing.assert_allclose(back.colors.numpy(), want, atol=1e-7)


def _strip(n_tri, offset):
    """A triangle strip of n_tri edge-connected triangles on n_tri + 2 fresh vertices."""
    verts = [(offset + i // 2, i % 2, 0.0) for i in range(n_tri + 2)]
    faces = [(i, i + 1, i + 2) if i % 2 == 0 else (i + 1, i, i + 2) for i in range(n_tri)]
    return verts, faces


def _components(sizes):
    verts, faces = [], []
    for k, s in enumerate(sizes):
        v, f = _strip(s, 10 * k)
        faces += [tuple(i + len(verts) for i in t) for t in f]
        verts += v
    return verts, faces


def test_filter_small_clusters_keeps_the_50_largest_and_at_least_50():
    sizes = [60 + k for k in range(55)] + [3, 7]  # 57 clusters: threshold = the 50th largest (65)
    verts, faces = _components(sizes)
    out = M.filter_small_clusters(_mesh(verts, faces, np.zeros((len(verts), 3))))
    assert out.faces.shape[0] == sum(s for s in sizes if s >= 65)
    assert out.vertices.shape[0] == sum(s + 2 for s in sizes if s >= 65)  # unreferenced vertices removed
    assert int(out.faces.max()) == out.vertices.shape[0] - 1 and out.colors.shape == out.vertices.shape


def test_filter_small_clusters_with_fewer_than_50_clusters():
    sizes = [200, 49, 50, 10]  # the reference would raise IndexError; the threshold is 50
    verts, faces = _components(sizes)
    faces.append((0, 0, 1))  # degenerate triangle in the kept cluster: removed
    out = M.filter_small_clusters(_mesh(verts, faces))
    assert out.faces.shape[0] == 250 and out.vertices.shape[0] == 202 + 52


def test_abi_argument_errors_of_the_mesh_entry_points():
    lib = L.load() if os.path.exists(L.LIB_PATH) else None
    if lib is None:
        from dn_splatter_b200.build import build

        build()
        lib = L.load()
    one = C.c_void_p(16)  # never dereferenced: the checks come first
    cam = (C.c_float * 16)()
    g = L.DnrTsdfGrid()
    g.voxels = 16
    assert lib.dnr_tsdf_integrate(None, one, one, None, 8, 8, cam, 1.0, None) == -1
    assert lib.dnr_tsdf_integrate(C.byref(g), None, one, None, 8, 8, cam, 1.0, None) == -1
    assert lib.dnr_tsdf_integrate(C.byref(g), one, one, None, 8, 8, cam, 1.0, None) == -2  # dims 0
    g.dims[0], g.dims[1], g.dims[2] = 4, 4, 4
    assert lib.dnr_tsdf_integrate(C.byref(g), one, one, None, 8, 8, cam, 1.0, None) == -2  # voxel 0
    g.voxel = 0.1
    assert lib.dnr_tsdf_integrate(C.byref(g), one, one, None, 8, 8, cam, 1.0, None) == -2  # sdf_trunc 0
    g.sdf_trunc = 0.3
    assert lib.dnr_tsdf_integrate(C.byref(g), one, one, None, 0, 8, cam, 1.0, None) == -2
    f = L.DnrMcField()
    assert lib.dnr_mc_count_workspace_bytes(None) == -1
    assert lib.dnr_mc_count_workspace_bytes(C.byref(f)) == -1  # neither values nor tsdf
    f.values = 16
    assert lib.dnr_mc_count_workspace_bytes(C.byref(f)) == -2
    f.dims[0], f.dims[1], f.dims[2] = 8, 8, 8
    assert lib.dnr_mc_count_workspace_bytes(C.byref(f)) == -2  # spacing 0
    f.spacing = 0.5
    nbytes = lib.dnr_mc_count_workspace_bytes(C.byref(f))
    assert nbytes >= 2 * 3 * 65 * 8
    counts = (C.c_int64 * 3)(5, 10, 7)
    assert lib.dnr_mc_count(C.byref(f), one, nbytes - 1, counts, None) == -5
    assert lib.dnr_mc_count(C.byref(f), None, nbytes, counts, None) == -1
    assert lib.dnr_mc_emit_workspace_bytes(counts) >= 5 * 16 + 7 * 8
    assert lib.dnr_mc_emit(C.byref(f), one, counts, one, 8, one, one, None, None) == -5
    assert lib.dnr_mc_emit(C.byref(f), one, counts, one, 1 << 20, None, one, None, None) == -1
    f.tsdf = 16
    assert lib.dnr_mc_count(C.byref(f), one, nbytes, counts, None) == -1  # both values and tsdf
