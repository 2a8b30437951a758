"""Mesh-export kernels (csrc/mesh.cu) against oracle/mesh_ref.py, and the two exporters end to end on a closed room of
flat Gaussians."""
import math

import numpy as np
import pytest
import torch

from oracle import mesh_ref as R

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]

W, H = 64, 48  # <= 256: the test colour encodes the pixel each voxel read


def _look_at(pos, target, up=(0.0, 0.0, 1.0)):
    from dn_splatter_b200.synthetic import look_at_c2w

    return look_at_c2w(torch.tensor(pos, dtype=torch.float32), torch.tensor(target, dtype=torch.float32),
                       torch.tensor(up, dtype=torch.float32))


def _camera(c2w, w=W, h=H, f=60.0):
    from dn_splatter_b200.cameras import Cameras

    return Cameras(c2w[None], f, f, w / 2, h / 2, w, h)


def _sphere_depth(cam_block, radius=0.5):
    E = np.asarray(cam_block, np.float64)[4:].reshape(3, 4)
    fx, fy, cx, cy = np.asarray(cam_block, np.float64)[:4]
    u, v = np.meshgrid(np.arange(W), np.arange(H))
    d = np.stack([(u - cx) / fx, (v - cy) / fy, np.ones((H, W))], axis=-1)
    c = E[:, 3]
    dd, bc = (d * d).sum(-1), (d * c).sum(-1)
    disc = bc * bc - dd * ((c * c).sum() - radius * radius)
    return np.where(disc > 0, (bc - np.sqrt(np.maximum(disc, 0))) / dd, 0.0).astype(np.float32)


def _voxels(vol):
    """tsdf, weight and colour (levels, decoded from the voxel's fixed point) of the volume, as [X,Y,Z] grids."""
    shape = tuple(vol.dims)
    tsdf, w, col = R.unpack_voxels(vol.voxels.cpu().numpy())
    return tsdf.reshape(shape), w.reshape(shape), col.reshape(shape + (3,))


def _views():
    """(camera, cam block, depth, rgb, mask, depth_trunc) of 5 views of a sphere: one masked, one with depth_trunc hits."""
    from dn_splatter_b200.mesh import TSDFVolume

    u, v = np.meshgrid(np.arange(W), np.arange(H))
    rgb = np.stack([(u + 0.5) / 255, (v + 0.5) / 255, np.full(u.shape, 0.3)], axis=-1).astype(np.float32)
    out = []
    for n, th in enumerate(np.linspace(0, 2 * math.pi, 6)[:-1]):
        cam = _camera(_look_at((2.2 * math.cos(th), 2.2 * math.sin(th), 0.4 * n - 0.6), (0.1, 0.0, 0.0)))
        block = np.array(TSDFVolume.camera_block(cam)[:], np.float32)
        depth = _sphere_depth(block)
        mask = None
        if n == 2:
            mask = np.zeros((H, W), np.uint8)
            mask[:, : W // 2] = 1
        trunc = 1.75 if n == 3 else 20.0
        out.append((cam, block, depth, rgb, mask, trunc))
    return out


def _integrate_both(bounds=((-0.71, -0.63, -0.77), (0.69, 0.55, 0.83)), voxel=0.037, sdf_trunc=0.11):
    from dn_splatter_b200.mesh import TSDFVolume

    vol = TSDFVolume(bounds, voxel_size=voxel, sdf_trunc=sdf_trunc)
    tsdf, w, col = R.empty_volume(tuple(vol.dims))
    first_uv = None
    for k, (cam, block, depth, rgb, mask, trunc) in enumerate(_views()):
        vol.depth_trunc = trunc
        vol.integrate(torch.from_numpy(depth)[..., None].cuda(), torch.from_numpy(rgb).cuda(), cam,
                      None if mask is None else torch.from_numpy(mask).cuda())
        uv = R.integrate(tsdf, w, col, vol.origin, voxel, sdf_trunc, depth, rgb, mask, block, trunc)
        if k == 0:
            first_uv = uv
            first = _voxels(vol)
    return vol, (tsdf, w, col), first, first_uv


def test_tsdf_integrate_matches_fp32_oracle_fixed_point_colour():
    vol, (tsdf, w, col), first, (u, v) = _integrate_both()
    assert all(d % 128 for d in vol.dims)
    # after the first view the colour is the pixel the voxel read: (u, v) encoded in red / green
    g_tsdf, g_w, g_col = first
    seen = u >= 0
    assert seen.sum() > 1000 and not seen.all()  # some voxels are out of the frustum or occluded
    assert np.array_equal(g_w > 0, seen)
    assert np.array_equal(g_col[seen][:, 0].astype(np.int64), u[seen]) and np.array_equal(g_col[seen][:, 1].astype(np.int64), v[seen])
    g_tsdf, g_w, g_col = _voxels(vol)
    assert np.array_equal(g_w, w) and w.max() >= 3
    np.testing.assert_allclose(g_tsdf, tsdf, rtol=0, atol=1e-6)
    np.testing.assert_allclose(g_col.astype(np.float32), col.astype(np.float32), rtol=0, atol=1e-6)
    untouched = w == 0
    assert (g_tsdf[untouched] == 0).all() and (g_col[untouched] == 0).all()


def _sphere_field(dims, s, origin):
    i, j, k = np.meshgrid(*[np.arange(d) for d in dims], indexing="ij")
    p = [origin[a] + s * idx for a, idx in enumerate((i, j, k))]
    return (np.sqrt(p[0] ** 2 + p[1] ** 2 + p[2] ** 2) - 0.55 + 0.05 * np.sin(7 * p[0]) * np.cos(5 * p[1])).astype(np.float32)


def test_marching_cubes_matches_oracle_and_is_deterministic():
    from dn_splatter_b200.mesh import marching_cubes

    dims, s, origin = (45, 38, 261), 0.031, (-0.7, -0.6, -0.8)
    f = _sphere_field(dims, s, origin)
    valid = np.ones(dims, bool)
    valid[20:26, 10:30, :] = False  # a hole of invalid samples
    for val in (None, valid):
        got = marching_cubes(torch.from_numpy(f).cuda(), 0.0, origin, s,
                             None if val is None else torch.from_numpy(val).cuda())
        again = marching_cubes(torch.from_numpy(f).cuda(), 0.0, origin, s,
                               None if val is None else torch.from_numpy(val).cuda())
        assert torch.equal(got.vertices, again.vertices) and torch.equal(got.faces, again.faces)
        rv, rf, _ = R.marching_cubes(f, 0.0, origin, s, valid=val)
        assert rf.shape[0] > 1000
        assert np.array_equal(got.faces.cpu().numpy(), rf)
        np.testing.assert_allclose(got.vertices.cpu().numpy(), rv, rtol=1e-6, atol=1e-7)


def test_tsdf_extraction_matches_oracle_fixed_point_colour():
    vol, (tsdf, w, col), _, _ = _integrate_both()
    got = vol.extract_mesh()
    again = vol.extract_mesh()
    assert torch.equal(got.faces, again.faces) and torch.equal(got.vertices, again.vertices)
    assert torch.equal(got.colors, again.colors)
    origin = [o + 0.5 * vol.voxel_size for o in vol.origin]
    g_tsdf, g_w, g_col = _voxels(vol)
    rv, rf, rc = R.marching_cubes(g_tsdf, 0.0, origin, vol.voxel_size, valid=g_w > 0, colors=g_col)
    assert rf.shape[0] > 500 and (g_w == 0).any()
    assert np.array_equal(got.faces.cpu().numpy(), rf)
    np.testing.assert_allclose(got.vertices.cpu().numpy(), rv, rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(got.colors.cpu().numpy(), rc, rtol=1e-6, atol=1e-7)


# ------------------------------------------------------------------------------------------------ the room
WALL_RGB = [(0.8, 0.2, 0.2), (0.2, 0.8, 0.2), (0.2, 0.2, 0.8), (0.8, 0.8, 0.2), (0.2, 0.8, 0.8), (0.8, 0.2, 0.8)]
THICK = 0.01  # normal sigma of the flat Gaussians


def _room(n_side=182):
    """Closed box [-1,1]^3: n_side^2 flat opaque Gaussians on each inner face, one colour per face (-x, +x, -y, ...)."""
    from dn_splatter_b200.cameras import Cameras

    g = torch.Generator().manual_seed(0)
    t = (torch.arange(n_side) + 0.5) / n_side * 2 - 1
    a, b = torch.meshgrid(t, t, indexing="ij")
    a, b = a.reshape(-1), b.reshape(-1)
    s45 = math.sqrt(0.5)
    rot = {0: (s45, 0.0, s45, 0.0), 1: (s45, s45, 0.0, 0.0), 2: (1.0, 0.0, 0.0, 0.0)}  # local z -> the face normal
    means, quats, dc = [], [], []
    for face in range(6):
        axis, side = face // 2, (1.0 if face % 2 else -1.0)
        p = torch.zeros(a.shape[0], 3)
        others = [x for x in range(3) if x != axis]
        p[:, axis] = side
        p[:, others[0]], p[:, others[1]] = a, b
        means.append(p)
        quats.append(torch.tensor(rot[axis]).expand(a.shape[0], 4))
        dc.append(((torch.tensor(WALL_RGB[face]) - 0.5) / 0.28209479177387814).expand(a.shape[0], 3))
    n = 6 * a.shape[0]
    sig = 2.0 / n_side
    scales = torch.log(torch.tensor([sig, sig, THICK])).expand(n, 3).clone()
    params = {"means": torch.cat(means), "quats": torch.cat(quats).clone(), "scales": scales,
              "opacities": torch.full((n, 1), math.log(0.99 / 0.01)), "features_dc": torch.cat(dc).clone(),
              "features_rest": torch.zeros(n, 15, 3)}
    cams = []  # near the centre, 53 degree field of view: few grazing views, which shift a TSDF surface by ~a voxel
    for _ in range(48):
        pos = (torch.rand(3, generator=g) - 0.5) * 0.4
        d = torch.randn(3, generator=g)
        d = d / d.norm()
        up = (0.0, 1.0, 0.0) if abs(float(d[2])) > 0.9 else (0.0, 0.0, 1.0)
        from dn_splatter_b200.synthetic import look_at_c2w

        c2w = look_at_c2w(pos, pos + d, torch.tensor(up))
        cams.append(Cameras(c2w[None], 320.0, 320.0, 160.0, 120.0, 320, 240))
    return params, cams


@pytest.fixture(scope="module")
def room():
    from dn_splatter_b200.dn_model import DNSplatterModelConfig

    params, cams = _room()
    m = DNSplatterModelConfig(random_init=True, num_random=16, background_color="black").setup(device="cuda")
    m.load_gaussians(params)
    m.step = 30000
    m.eval()
    return m, cams


def _wall_distance(v):
    return (1.0 - np.abs(v)).min(axis=1)


def test_export_tsdf_mesh_on_the_room(room, tmp_path):
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components

    from dn_splatter_b200.mesh import TSDF_MESH_NAME, export_tsdf_mesh, read_ply

    m, cams = room
    mesh = export_tsdf_mesh(m, cams, str(tmp_path), voxel_size=0.02, sdf_trunc=0.06)
    v, f, c = mesh.vertices.numpy(), mesh.faces.numpy(), mesh.colors.numpy()
    assert f.shape[0] > 10000
    assert (np.abs(_wall_distance(v)) <= 0.02).mean() >= 0.99
    adj = coo_matrix((np.ones(3 * f.shape[0]), (np.repeat(f[:, 0], 3), f.reshape(-1))), shape=(v.shape[0],) * 2)
    _, lab = connected_components(adj, directed=False)
    tri_lab = lab[f[:, 0]]
    assert np.bincount(tri_lab).max() >= 0.95 * f.shape[0]
    # away from the box's edges every vertex carries its wall's colour
    axis = np.argmin(1.0 - np.abs(v), axis=1)
    face = 2 * axis + (v[np.arange(v.shape[0]), axis] > 0)
    inner = np.sort(np.abs(v), axis=1)[:, 1] < 0.85
    want = np.floor(np.asarray(WALL_RGB, np.float32) * 255) / 255
    err = np.abs(c[inner] - want[face[inner]]).max(axis=1)
    assert inner.sum() > 1000 and (err <= 3 / 255).all(), float(err.max())
    back = read_ply(str(tmp_path / TSDF_MESH_NAME))
    assert torch.equal(back.vertices, mesh.vertices) and torch.equal(back.faces, mesh.faces)
    np.testing.assert_allclose(back.colors.numpy(), np.round(np.clip(c, 0, 1) * 255) / 255, atol=1e-6)


def test_export_marching_cubes_mesh_on_the_room(room, tmp_path):
    from dn_splatter_b200.mesh import export_marching_cubes_mesh, read_ply

    from dn_splatter_b200.cameras import Cameras
    from dn_splatter_b200.synthetic import look_at_c2w

    m, _ = room
    res = 128
    # cameras at the corners of [-0.6, 0.6]^3: the exporter's grid, 2 * 0.6 * sqrt(3) wide, covers the room
    cams = [Cameras(look_at_c2w(0.6 * torch.tensor([sx, sy, sz]), torch.zeros(3), torch.tensor([0.0, 0.0, 1.0]))[None],
                    320.0, 320.0, 160.0, 120.0, 320, 240) for sx in (-1.0, 1.0) for sy in (-1.0, 1.0) for sz in (-1.0, 1.0)]
    mesh = export_marching_cubes_mesh(m, cams, str(tmp_path), resolution=res)
    centres = torch.stack([c.camera_to_worlds[0, :, 3] for c in cams])
    radius = 2 * float((centres - centres.mean(0)).norm(dim=-1).max())
    spacing = 2 * radius / (res - 1)
    v = mesh.vertices.cpu().numpy()
    assert v.shape[0] > 10000
    assert (np.abs(_wall_distance(v)) <= spacing + 3 * THICK).all()
    back = read_ply(str(tmp_path / f"marching_cubes_raw_{res}.ply"))
    assert torch.equal(back.faces, mesh.faces.cpu())
