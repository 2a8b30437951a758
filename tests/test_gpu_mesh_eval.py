"""Mesh evaluation on the device (csrc/mesh_eval.cu, dn_splatter_b200/mesh_eval.py) against the fp64 oracle
(oracle/mesh_eval_ref.py), analytic boxes, and the room model's exported meshes."""
import json
import math

import numpy as np
import pytest
import torch

from oracle import mesh_eval_ref as R
from tests import mesh_eval_cases as C
from tests.mesh_eval_cases import box, sphere

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]


def _look_at(pos, target, up=(0.0, 0.0, 1.0)):
    from dn_splatter_b200.synthetic import look_at_c2w

    return look_at_c2w(torch.tensor(pos, dtype=torch.float32), torch.tensor(target, dtype=torch.float32),
                       torch.tensor(up, dtype=torch.float32))


def _cam(c2w, W, H, fx, fy=None, cx=None, cy=None):
    from dn_splatter_b200.cameras import Cameras

    return Cameras(torch.as_tensor(c2w, dtype=torch.float32).reshape(-1, 3, 4)[:1], fx, fy or fx,
                   W / 2 if cx is None else cx, H / 2 if cy is None else cy, W, H)


def _block(cam):
    return R.camera_block(cam.camera_to_worlds[0].double().numpy(), float(cam.fx[0, 0]), float(cam.fy[0, 0]),
                          float(cam.cx[0, 0]), float(cam.cy[0, 0]))


def _mesh(v, f):
    from dn_splatter_b200.mesh import TriangleMesh

    return TriangleMesh(torch.as_tensor(np.asarray(v), dtype=torch.float32), torch.as_tensor(np.asarray(f), dtype=torch.int32), None)


def _scenes(W, H):
    return [(name, v, f, _cam(c2w, W, H, fx, fy, cx, cy)) for name, v, f, c2w, fx, fy, cx, cy in C.legacy_scenes(W, H)]


def _compare_depth(name, v, f, cam, W, H, chunk=64):
    """The kernel's depth against the oracle's restatement of its rule on the fp32 camera block it reads: every pixel's
    bits equal.  The independent ray cast (fp64 Moller-Trumbore) agrees on hits away from triangle edges, to 1 fp32 ulp.
    Returns (kernel depth, ray-cast depth, near-edge pixel count, the rule's decision counts)."""
    from dn_splatter_b200.mesh_eval import camera_blocks, render_mesh_depth

    got = render_mesh_depth(_mesh(v, f), [cam])[0]
    again = render_mesh_depth(_mesh(v, f), [cam])[0]
    assert torch.equal(got, again), name
    got = got.cpu().numpy()
    blk = camera_blocks([cam], torch.float32).cpu().numpy()[0]
    assert np.array_equal(blk, _block(cam).astype(np.float32)), name
    v32 = np.asarray(v, np.float32)  # the kernel reads float32 vertices
    want, stats = R.depth_kernel_rule(v32, f, blk, W, H)
    n_diff = int((got.view(np.uint32) != want.view(np.uint32)).sum())
    assert n_diff == 0, (name, n_diff)
    rc = R.ray_cast_depth(v32.astype(np.float64), f, blk.astype(np.float64), W, H, chunk=chunk)
    amb = R.near_edge_pixels(v32.astype(np.float64), f, blk.astype(np.float64), W, H, chunk=chunk)
    assert np.array_equal((got > 0)[~amb], (rc > 0)[~amb]), name
    both = (got > 0) & (rc > 0) & ~amb
    ulp = np.abs(got[both].view(np.int32).astype(np.int64) - rc[both].astype(np.float32).view(np.int32).astype(np.int64))
    assert ulp.max(initial=0) <= 1, (name, int(ulp.max()))
    return got, rc, int(amb.sum()), stats


@pytest.mark.parametrize("W,H", [(81, 49), (75, 53)])
def test_mesh_depth_matches_the_oracle_ray_cast(W, H):
    report = {}
    for name, v, f, cam in _scenes(W, H):
        got, rc, n_amb, stats = _compare_depth(name, v, f, cam, W, H)
        report[name] = (n_amb, stats)
        if name == "box_inside":
            assert (got > 0).all()  # a closed box seen from inside has no empty pixel
        if name == "edges":
            # pixels the independent ray cast hits along with their 4 neighbours: away from the grid's outer boundary
            inner = C.interior_hits(v, f, _block(cam).astype(np.float32), W, H)
            assert inner.sum() > 0.5 * W * H and (got[inner] > 0).all()  # no pixel centre on a shared edge is lost
        if name == "odd":
            assert (got > 0).all() and (got < 5.0).any()  # the full-screen triangle behind the nearer ones
    print("near-edge pixels / pixels per decision of the rule", report)


def test_mesh_depth_full_hd():
    W, H = 1920, 1080
    v, f, c2w, fx, fy, cx, cy = C.full_hd_scene()
    cam = _cam(c2w, W, H, fx, fy, cx, cy)
    got, rc, n_amb, stats = _compare_depth("full_hd", v, f, cam, W, H, chunk=2)
    assert (got > 0).mean() > 0.99
    print("1080p near-edge pixels", n_amb, "pixels per decision", stats)


def test_mesh_depth_batches_views():
    from dn_splatter_b200.mesh_eval import render_mesh_depth

    W, H = 64, 40
    v, f = box()
    cams = [_cam(_look_at((0.2 * math.cos(a), 0.2 * math.sin(a), 0.1), (math.cos(a + 1), math.sin(a + 1), 0.0)), W, H, 40.0)
            for a in np.linspace(0, 6, 5)]
    batch = render_mesh_depth(_mesh(v, f), cams)
    for k, c in enumerate(cams):
        assert torch.equal(batch[k], render_mesh_depth(_mesh(v, f), [c])[0])


# ------------------------------------------------------------------------------------------------ visibility
def test_visibility_counts_equal_the_oracle():
    from dn_splatter_b200.mesh_eval import visibility_counts

    W, H, n = 81, 49, 56
    rng = np.random.default_rng(0)
    cams = [_cam(_look_at(tuple(rng.uniform(-0.3, 0.3, 3)), tuple(rng.uniform(-0.3, 0.3, 3) + np.array([math.cos(a), math.sin(a), 0.0]) * 2)),
                 W, H, 50.0, 52.0, 40.3, 24.1) for a in np.linspace(0, 2 * np.pi, n, endpoint=False)]
    blocks = [_block(c) for c in cams]
    pts = rng.uniform(-1.2, 1.2, (20000, 3))
    # points exactly on px = W - 1 and py = 0 of view 0, behind view 0, and at its camera centre
    fx, fy, cx, cy = blocks[0][:4]
    E = blocks[0][4:].reshape(3, 4)
    Rinv, t = np.linalg.inv(E[:, :3]), E[:, 3]
    z = rng.uniform(0.5, 2.0, 300)
    u = np.where(np.arange(300) % 2 == 0, W - 1, rng.uniform(0, W - 1, 300))
    vv = np.where(np.arange(300) % 3 == 0, 0.0, rng.uniform(0, H - 1, 300))
    pc = np.stack([(u - cx) * z / fx, (vv - cy) * z / fy, z], 1)
    on_edge = (pc - t) @ Rinv.T
    behind = (np.stack([pc[:, 0], pc[:, 1], -pc[:, 2]], 1) - t) @ Rinv.T
    pts = np.concatenate([pts, on_edge, behind, (-Rinv @ t)[None]])
    rendered = np.stack([(0.5 + 2.0 * rng.random((H, W))).astype(np.float32) for _ in range(n)])
    gt = np.stack([np.where(rng.random((H, W)) < 0.25, 0.0, 1.0).astype(np.float32) for _ in range(n)])
    gt[:, :, -1] = 0.0  # zero gt depth on the last column
    first = None
    for rend, g in ((rendered, gt), (None, gt), (rendered, None)):
        obs, inv = visibility_counts(torch.from_numpy(pts).cuda(), cams, None if rend is None else torch.from_numpy(rend).cuda(),
                                     None if g is None else torch.from_numpy(g).cuda(), chunk=16)
        ro, ri = R.visibility_counts(pts, blocks, W, H, rend, g)
        assert np.array_equal(obs.cpu().numpy(), ro) and np.array_equal(inv.cpu().numpy(), ri)
        first = (ro, ri) if first is None else first
    ro, ri = first
    assert ro.max() > 3 and (ri > 0).any() and (ro == 0).any()
    ro0, _ = R.visibility_counts(on_edge, blocks[:1], W, H)
    assert ro0.sum() > 100  # most points of the border set count as in the frustum


# ------------------------------------------------------------------------------------------------ culling
def _room_views(n=24, W=64, H=48, f=30.0, seed=1):
    rng = np.random.default_rng(seed)
    return [_cam(_look_at(tuple(rng.uniform(-0.3, 0.3, 3)), tuple(rng.uniform(-0.3, 0.3, 3) + np.array([math.cos(a), math.sin(a), 0.2 * math.sin(3 * a)]) * 2)),
                 W, H, f) for a in np.linspace(0, 2 * np.pi, n, endpoint=False)]


def test_device_subdivision_equals_the_oracle():
    from dn_splatter_b200.mesh_eval import subdivide_to_size

    v, f = sphere(6, 0.7)
    v = np.concatenate([v, box((-1, -1, -1), (1, 1, 1))[0]])
    f = np.concatenate([f, box()[1] + sphere(6, 0.7)[0].shape[0]])
    for me in (0.05, 0.3):
        got = subdivide_to_size(_mesh(v, f), me)
        sv, sf, _ = R.subdivide_to_size(np.asarray(v, np.float32).astype(np.float64), f, me)
        assert got.vertices.dtype == torch.float64
        assert np.array_equal(R.triangle_multiset(got.vertices.cpu().numpy(), got.faces.cpu().numpy()), R.triangle_multiset(sv, sf))


def test_cull_mesh_keeps_the_oracle_faces():
    from dn_splatter_b200.mesh_eval import cull_mesh, render_mesh_depth

    W, H = 64, 48
    cams = _room_views(W=W, H=H)
    bv, bf = box()
    ov, of = box((-0.2, -0.3, -0.2), (0.2, 0.1, 0.2))
    v = np.concatenate([bv, ov + np.array([0.3, 0.2, -0.5])])
    f = np.concatenate([bf, of[:, [0, 2, 1]] + 8])
    mesh = _mesh(v, f)
    gt = render_mesh_depth(_mesh(bv, bf), cams).cpu().numpy()
    gt[:, : H // 3, : W // 2] = 0.0
    got = cull_mesh(mesh, cams, torch.from_numpy(gt).cuda(), max_edge=0.2)
    depths = render_mesh_depth(mesh, cams).cpu().numpy()
    blocks = [_block(c) for c in cams]
    rv, rf, _, _ = R.cull_mesh(np.asarray(v, np.float32).astype(np.float64), f, blocks, W, H, gt_depths=gt, max_edge=0.2,
                               depths=list(depths))
    assert rf.shape[0] > 100
    assert np.array_equal(R.triangle_multiset(got.vertices.cpu().numpy(), got.faces.cpu().numpy()), R.triangle_multiset(rv, rf))


# ------------------------------------------------------------------------------------------------ sampling and metrics
def test_sample_surface():
    from scipy.stats import chisquare

    from dn_splatter_b200.mesh_eval import compute_metrics, mesh_area, sample_surface

    v, f = sphere(5, 0.4)
    v = v * np.array([1.0, 0.5, 2.0])
    mesh = _mesh(v, f)
    area = mesh_area(mesh)
    n = int(area * 1e4)
    g = torch.Generator(device="cuda").manual_seed(3)
    p, nrm, idx = sample_surface(mesh, n, g, return_index=True)
    g2 = torch.Generator(device="cuda").manual_seed(3)
    p2, nrm2 = sample_surface(mesh, n, g2)
    assert p.shape == (n, 3) and torch.equal(p, p2) and torch.equal(nrm, nrm2)
    v32 = np.asarray(v, np.float32).astype(np.float64)
    tri = v32[f[idx.cpu().numpy()]]
    pp = p.double().cpu().numpy()
    # barycentrics by least squares in the face plane
    e1, e2, d = tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0], pp - tri[:, 0]
    a11, a12, a22 = (e1 * e1).sum(1), (e1 * e2).sum(1), (e2 * e2).sum(1)
    b1, b2 = (d * e1).sum(1), (d * e2).sum(1)
    det = a11 * a22 - a12 * a12
    l1, l2 = (a22 * b1 - a12 * b2) / det, (a11 * b2 - a12 * b1) / det
    plane = np.abs((d * np.cross(e1, e2)).sum(1)) / np.linalg.norm(np.cross(e1, e2), axis=1)
    assert (l1 >= -1e-6).all() and (l2 >= -1e-6).all() and (l1 + l2 <= 1 + 1e-6).all() and plane.max() < 1e-6
    areas = R.triangle_areas(v32, f)
    counts = np.bincount(idx.cpu().numpy(), minlength=f.shape[0])
    pos = areas > 1e-12  # the pole fans of the sphere have zero-area faces, which are never drawn
    assert counts[~pos].sum() == 0
    assert chisquare(counts[pos], areas[pos] / areas[pos].sum() * n).pvalue > 1e-3
    fn = R.face_normals(v32, f)[idx.cpu().numpy()]
    assert np.abs(nrm.double().cpu().numpy() - fn).max() < 1e-6
    assert n == int(R.triangle_areas(v32, f).sum() * 1e4)
    m1 = compute_metrics(mesh, mesh, generator=torch.Generator(device="cuda").manual_seed(1))
    m2 = compute_metrics(mesh, mesh, generator=torch.Generator(device="cuda").manual_seed(1))
    assert m1 == m2


def _check_metrics(got, want, pd, gd, thr=0.05):
    for k in ("Acc", "Comp", "C-L1", "NC"):
        assert abs(got[k] - want[k]) <= 1e-6 * abs(want[k]), (k, got[k], want[k])
    close = (np.abs(pd - thr) < 1e-6).any() or (np.abs(gd - thr) < 1e-6).any()
    if np.isnan(want["F-score"]):
        assert np.isnan(got["F-score"])
    elif not close:
        p, r = float((pd <= thr).mean()), float((gd <= thr).mean())
        assert got["F-score"] == pytest.approx(2 * p * r / (p + r), rel=1e-15)
        assert abs(got["F-score"] - want["F-score"]) <= 1e-6 * want["F-score"]


def test_metrics_on_injected_samples_match_the_oracle():
    from scipy.spatial import cKDTree

    from dn_splatter_b200.mesh_eval import metrics_from_samples, point_cloud_metrics

    rng = np.random.default_rng(4)
    for shift in (0.0, 0.03, 0.2):
        gp = rng.uniform(-1, 1, (30000, 3)).astype(np.float32) * np.array([1, 1, 0.05], np.float32)
        pp = (rng.uniform(-1, 1, (25000, 3)) * np.array([1, 1, 0.05]) + np.array([0, 0, shift])).astype(np.float32)
        gn = rng.normal(size=gp.shape)
        pn = rng.normal(size=pp.shape)
        got = metrics_from_samples(torch.from_numpy(pp).cuda(), torch.from_numpy(pn).cuda(), torch.from_numpy(gp).cuda(),
                                   torch.from_numpy(gn).cuda())
        want = R.mesh_metrics(pp, pn, gp, gn)
        pd = cKDTree(gp).query(pp)[0]
        gd = cKDTree(pp).query(gp)[0]
        _check_metrics(got, want, pd, gd)
        acc, comp = point_cloud_metrics(torch.from_numpy(pp).cuda(), torch.from_numpy(gp).cuda())
        assert acc == pytest.approx(R.pd_accuracy(pp, gp), rel=1e-6)
        assert comp == pytest.approx(R.pd_completeness(pp, gp), rel=1e-6, abs=1e-4)


# ------------------------------------------------------------------------------------------------ end to end
def _room_cameras():
    """The 48 cameras of test_gpu_mesh.py's room."""
    from dn_splatter_b200.cameras import Cameras
    from dn_splatter_b200.synthetic import look_at_c2w

    g = torch.Generator().manual_seed(0)
    cams = []
    for _ in range(48):
        pos = (torch.rand(3, generator=g) - 0.5) * 0.4
        d = torch.randn(3, generator=g)
        d = d / d.norm()
        up = (0.0, 1.0, 0.0) if abs(float(d[2])) > 0.9 else (0.0, 0.0, 1.0)
        cams.append(Cameras(look_at_c2w(pos, pos + d, torch.tensor(up))[None], 320.0, 320.0, 160.0, 120.0, 320, 240))
    return cams


def test_end_to_end_on_the_box_room(tmp_path):
    from dn_splatter_b200.mesh_eval import evaluate_mesh, render_mesh_depth

    cams = _room_cameras()
    bv, bf = box()
    gt = _mesh(bv, bf)
    gt_depth = render_mesh_depth(gt, cams)
    g = lambda: torch.Generator(device="cuda").manual_seed(0)  # noqa: E731
    same = evaluate_mesh(gt, gt, cams, str(tmp_path / "same"), gt_depth, generator=g())
    # samples within a few mm of the box's 12 edges find their neighbour on the perpendicular wall: NC 0.996 at 1e4
    # samples per m^2 (measured on an H100), the reference's rule on the same samples gives the same
    # the mean nearest-neighbour distance of independent samples at 1e4 per m^2 is 0.5 / sqrt(1e4) = 0.005
    assert same["F-score"] == 1.0 and same["NC"] >= 0.99 and abs(same["Acc"] - 0.005) < 0.0015 and abs(same["Comp"] - 0.005) < 0.0015
    out2 = evaluate_mesh(_mesh(bv * 1.02, bf), gt, cams, str(tmp_path / "o2"), gt_depth, generator=g())
    # a few subdivided faces near the corners survive the culling in one mesh only (measured F = 0.999975)
    assert out2["F-score"] >= 0.9999 and abs(out2["Acc"] - 0.02) < 0.004 and abs(out2["Comp"] - 0.02) < 0.004
    out8 = evaluate_mesh(_mesh(bv * 1.08, bf), gt, cams, str(tmp_path / "o8"), gt_depth, generator=g())
    assert math.isnan(out8["F-score"])  # precision = recall = 0: F is 0 / 0, NaN as the reference's rule gives it
    # an object behind a wall (outside the room), in pred only: culled, metrics unchanged
    ov, of = box((1.3, -0.2, -0.2), (1.6, 0.2, 0.2))
    pv, pf = np.concatenate([bv, ov]), np.concatenate([bf, of + 8])
    hidden = evaluate_mesh(_mesh(pv, pf), gt, cams, str(tmp_path / "hid"), gt_depth, generator=g())
    assert all(hidden[k] == pytest.approx(same[k], rel=1e-12) for k in same)
    # gt depth zeroed over the left third of every view: the 0.7 rule removes the same faces as the oracle
    from dn_splatter_b200.mesh_eval import cull_mesh

    holes = gt_depth.clone()
    holes[:, :, : 320 // 3] = 0.0
    got = cull_mesh(gt, cams, holes, max_edge=0.1)
    full = cull_mesh(gt, cams, gt_depth, max_edge=0.1)
    blocks = [_block(c) for c in cams]
    rv, rf, _, _ = R.cull_mesh(bv, bf, blocks, 320, 240, gt_depths=list(holes.cpu().numpy()), max_edge=0.1,
                               depths=list(gt_depth.cpu().numpy()))
    assert got.faces.shape[0] < full.faces.shape[0]
    assert np.array_equal(R.triangle_multiset(got.vertices.cpu().numpy(), got.faces.cpu().numpy()), R.triangle_multiset(rv, rf))
    print("box room:", same, out2, out8)


@pytest.fixture(scope="module")
def room():
    from dn_splatter_b200.dn_model import DNSplatterModelConfig

    from tests.test_gpu_mesh import _room

    params, cams = _room()
    m = DNSplatterModelConfig(random_init=True, num_random=16, background_color="black").setup(device="cuda")
    m.load_gaussians(params)
    m.step = 30000
    m.eval()
    return m, cams


def test_exported_room_meshes_against_the_box(room, tmp_path):
    from dn_splatter_b200.mesh import export_tsdf_mesh
    from dn_splatter_b200.mesh_eval import evaluate_mesh, render_mesh_depth
    from dn_splatter_b200.poisson import export_dn_poisson_mesh

    m, cams = room
    bv, bf = box()
    gt = _mesh(bv, bf)
    gt_depth = render_mesh_depth(gt, cams)
    tsdf = export_tsdf_mesh(m, cams, str(tmp_path / "tsdf"), voxel_size=0.02, sdf_trunc=0.06)
    dn = export_dn_poisson_mesh(m, cams, str(tmp_path / "dn"), total_points=400_000, poisson_depth=8)[0]
    res = {}
    for name, mesh in (("tsdf", tsdf), ("dn", dn)):
        res[name] = evaluate_mesh(mesh, gt, cams, str(tmp_path / name), gt_depth,
                                  generator=torch.Generator(device="cuda").manual_seed(0))
    print("room meshes vs the box:", json.dumps(res))
    for name, r in res.items():
        # measured on an H100: Acc / Comp 0.0113-0.0119 (the rendered depth of the 0.01-thick walls lies ~0.01 in front
        # of them), NC 0.983-0.990, F-score 0.99995
        assert r["F-score"] >= 0.999 and r["Acc"] <= 0.015 and r["Comp"] <= 0.015 and r["NC"] >= 0.97, (name, r)


def test_evaluate_mesh_files_on_a_replica_layout(tmp_path):
    from PIL import Image

    from dn_splatter_b200.mesh import write_ply
    from dn_splatter_b200.mesh_eval import evaluate_mesh, evaluate_mesh_files, load_dataset_views, read_triangle_mesh
    from dn_splatter_b200.mesh_eval import render_mesh_depth

    cams = _room_views(n=16, W=64, H=48)
    bv, bf = box()
    gt = _mesh(bv, bf)
    pred = _mesh(bv * 1.01 + 0.003, bf)
    depth = render_mesh_depth(gt, cams).cpu().numpy()
    (tmp_path / "data" / "depth").mkdir(parents=True)
    frames = []
    for k, c in enumerate(cams):
        png = np.round(depth[k] * 6553.5).astype(np.uint16)
        Image.fromarray(png).save(tmp_path / "data" / "depth" / f"{k}.png")
        c2w = np.eye(4)
        c2w[:3] = c.camera_to_worlds[0].double().numpy()
        c2w[0:3, 1:3] *= -1  # replica stores OpenCV poses
        frames.append({"depth_file_path": f"depth/{k}.png", "transform_matrix": c2w.tolist()})
    tf = tmp_path / "data" / "transforms.json"
    tf.write_text(json.dumps({"h": 48, "w": 64, "fl_x": 30.0, "fl_y": 30.0, "cx": 32.0, "cy": 24.0, "frames": frames}))
    (tmp_path / "meshes").mkdir()
    write_ply(str(tmp_path / "meshes" / "gt.ply"), gt)
    write_ply(str(tmp_path / "meshes" / "pred.ply"), pred)
    g = lambda: torch.Generator(device="cuda").manual_seed(5)  # noqa: E731
    rst = evaluate_mesh_files(tmp_path / "meshes" / "gt.ply", tmp_path / "meshes" / "pred.ply", tf, tmp_path / "data",
                              dataset="replica", generator=g())
    back = json.loads((tmp_path / "meshes" / "mesh_metrics.json").read_text())
    assert back == rst and set(back) == {"Acc", "Comp", "C-L1", "NC", "F-score"}
    culled = read_triangle_mesh(str(tmp_path / "meshes" / "mesh_cull.ply"))
    assert culled.faces.shape[0] > 100
    views, depths = load_dataset_views(str(tf), str(tmp_path / "data"), "replica")
    same = evaluate_mesh(read_triangle_mesh(str(tmp_path / "meshes" / "pred.ply")), read_triangle_mesh(str(tmp_path / "meshes" / "gt.ply")),
                         views, str(tmp_path / "mem"), depths, generator=g())
    assert same == rst
    assert rst["F-score"] == 1.0 and rst["Acc"] < 0.03
