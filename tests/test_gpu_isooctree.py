"""The isooctree kernels (csrc/isooctree.cu) against oracle/isooctree_ref.py, and the extractor end to end: on the
reference-golden render folder, and on the closed room of test_gpu_mesh.py through export_isooctree_mesh."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import isooctree_ref as O
from tests import isooctree_scene as S
from tests.test_isooctree_cpu import golden, golden_frames

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]


def frameset(frames):
    """A device FrameSet holding the oracle frames' file values."""
    from dn_splatter_b200 import isooctree as I

    cam = frames[0].camera
    fs = I.FrameSet(I.CameraModel({"w": cam.resolution[0], "h": cam.resolution[1], "fl_x": cam.camera_matrix[0, 0],
                                   "fl_y": cam.camera_matrix[1, 1], "cx": cam.camera_matrix[0, 2], "cy": cam.camera_matrix[1, 2]}),
                    len(frames), frames[0].cam_coordinate_normals)
    for i, f in enumerate(frames):
        fs.depth[i] = torch.from_numpy(np.asarray(f.depth_raw, np.float32))
        fs.normals[i] = torch.from_numpy(np.asarray(f.normal_raw, np.float32))
        fs.set_pose(i, f.pose_c2w, f.pose_w2c)
    return fs


def room_frames(n, w=S.W, h=S.H, f=S.F, cam_normals=False, seed=0):
    """n frames of the analytic room from random poses inside it."""
    g = np.random.default_rng(seed)
    cam = O.CameraModel({"w": w, "h": h, "fl_x": f, "fl_y": f, "cx": w / 2, "cy": h / 2})
    out = []
    for _ in range(n):
        pos = g.uniform(S.ROOM[0] + 0.4, S.ROOM[1] - 0.4)
        c2w = S.look_at_opencv(pos, pos + np.append(g.normal(size=2), g.normal() * 0.3))
        d, nw, png = S.frame_files(c2w, w, h, f)
        out.append(O.Frame(cam, S.transform_matrix(c2w), d[..., 0], png if cam_normals else nw, cam_normals))
    return out


# ------------------------------------------------------------------------------------------------ hint cloud
@pytest.mark.parametrize("cam", [False, True])
def test_samples_equal_oracle_on_golden_folder(cam):
    from dn_splatter_b200.isooctree import hint_samples

    frames = golden_frames(golden(), cam)
    fs = frameset(frames)
    for stride in (1, 2, 6):
        want_p, want_n = O.hint_cloud(frames, stride)
        got_p, got_n = hint_samples(fs, stride, with_normals=True)
        assert want_p.shape[0] > 20
        assert np.array_equal(got_p.cpu().numpy(), want_p) and np.array_equal(got_n.cpu().numpy(), want_n)


@pytest.mark.parametrize("w,h", [(61, 37), (1, 9), (130, 1)])
def test_samples_equal_oracle_on_ragged_sizes(w, h):
    from dn_splatter_b200.isooctree import hint_samples

    for cam in (False, True):
        frames = room_frames(5, w, h, f=3.0 * max(w, h), cam_normals=cam, seed=w)
        fs = frameset(frames)
        for stride in (1, 3, 7):
            want_p, _ = O.hint_cloud(frames, stride)
            got_p, got_n = hint_samples(fs, stride)
            assert got_n is None and np.array_equal(got_p.cpu().numpy(), want_p)


# ------------------------------------------------------------------------------------------------ isoFunc
MODES = {"two_pass": {}, "best_frame": dict(choose_best_frame=True), "no_normals": dict(use_normals=False),
         "one_pass": dict(two_pass=False), "tsdf_abs": dict(max_tsdf_abs=0.04)}


def _check_eval(frames, points, kw, what):
    from dn_splatter_b200.isooctree import iso_eval

    fs = frameset(frames)
    pts = torch.from_numpy(points).cuda()
    got = iso_eval(fs, pts, **kw)
    again = iso_eval(fs, pts, **kw)
    assert torch.equal(got, again), f"{what}: not bit-identical between runs"
    want = O.iso_func(frames, points, **kw)
    err = np.abs(got.cpu().numpy().astype(np.float64) - want)
    bad = err > S.eval_tolerance(want)
    # fp64 throughout: no decision can flip at fp32 resolution, so no value is accepted for a flipped decision
    print(f"{what}: {points.shape[0]} points, {int(bad.sum())} outside the bound, max err {err.max():.3e}, "
          f"0 accepted as flipped decisions")
    assert not bad.any(), f"{what}: {int(bad.sum())} points, max err {err.max():.3e}"
    return want


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("cam", [False, True])
def test_eval_matches_oracle_on_golden_queries(mode, cam):
    z = golden()
    want = _check_eval(golden_frames(z, cam), z["queries"], MODES[mode], f"golden {mode} cam={cam}")
    assert (np.abs(want) != 1).sum() > 50 and (want == 1).any() and (want == -1).any()


@pytest.mark.parametrize("n_frames", [1, 2, 7, 64, 300])
def test_eval_matches_oracle_over_frame_counts(n_frames):
    frames = room_frames(n_frames, seed=n_frames)
    pts = S.query_points(seed=n_frames)[:: max(1, n_frames // 30)]
    for mode in ("two_pass", "no_normals"):
        _check_eval(frames, pts, MODES[mode], f"{n_frames} frames {mode}")


@pytest.mark.parametrize("cam", [False, True])
def test_eval_frame_order_ties(cam):
    z = golden()
    frames = S.tie_frames(golden_frames(z, cam))
    for mode in ("two_pass", "best_frame"):
        _check_eval(frames, z["queries"], MODES[mode], f"ties {mode} cam={cam}")
    # the tie decides: swapping each pair changes the result
    swapped = [frames[i ^ 1] for i in range(len(frames))]
    assert not np.array_equal(O.iso_func(frames, z["queries"]), O.iso_func(swapped, z["queries"]))


# ------------------------------------------------------------------------------------------------ octree and fill
def _hint():
    z = golden()
    return O.hint_cloud(golden_frames(z, False), 1)[0]


@pytest.mark.parametrize("threshold", [1, 50, 10 ** 6])
@pytest.mark.parametrize("max_depth", [4, 5, 6, 7, 8, 9, 10])
def test_octree_leaves_and_corners_equal_oracle(threshold, max_depth):
    from dn_splatter_b200.isooctree import build_octree

    hint = _hint()
    tree = build_octree(torch.from_numpy(hint).cuda(), max_depth, threshold)
    leaves, origin, cell = O.octree(hint, max_depth, threshold)
    assert np.array_equal(np.asarray(tree.origin), origin) and tree.cell == cell
    assert np.array_equal(tree.leaves.cpu().numpy(), leaves)
    level = leaves >> 58
    assert tree.level_counts == tuple(int((level == lv).sum()) for lv in range(max_depth + 1))
    keys = O.leaf_corners(leaves, max_depth)
    assert np.array_equal(tree.corner_keys.cpu().numpy(), keys)
    assert np.array_equal(tree.corner_points.cpu().numpy(), O.corner_points(keys, origin, cell, max_depth))
    lc = tree.leaf_corners.cpu().numpy().astype(np.int64)
    R1 = (1 << max_depth) + 1
    _, lo, size = O.leaf_boxes(leaves, max_depth)
    q = np.arange(8)
    want = ((lo[:, None, 0] + ((q >> 2) & 1) * size[:, None]) * R1 + lo[:, None, 1] + ((q >> 1) & 1) * size[:, None]) * R1 \
        + lo[:, None, 2] + (q & 1) * size[:, None]
    assert np.array_equal(keys[lc], want)
    if threshold == 10 ** 6:
        assert leaves.tolist() == [0]
    elif threshold == 1:
        assert level.max() == max_depth


@pytest.mark.parametrize("max_depth,threshold", [(5, 1), (6, 20), (7, 50)])
def test_fill_equals_oracle_grid(max_depth, threshold):
    from dn_splatter_b200.isooctree import build_octree, fill_grid

    hint = _hint()
    tree = build_octree(torch.from_numpy(hint).cuda(), max_depth, threshold)
    vals = torch.from_numpy(np.random.default_rng(max_depth).normal(size=tree.corner_keys.shape[0]).astype(np.float32)).cuda()
    field = fill_grid(tree, vals)
    again = fill_grid(tree, vals)
    assert torch.equal(field, again)
    leaves, _, _ = O.octree(hint, max_depth, threshold)
    want = O.fill(leaves, tree.corner_keys.cpu().numpy(), vals.cpu().numpy(), max_depth)
    assert not np.isnan(want).any()
    assert np.array_equal(field.cpu().numpy(), want)


# ------------------------------------------------------------------------------------------------ end to end
def test_mesh_files_on_golden_folder_equal_oracle_pipeline(tmp_path):
    from dn_splatter_b200.isooctree import isooctree_mesh_files
    from dn_splatter_b200.mesh import read_obj, read_ply

    z = golden()
    js = S.write_folder(str(tmp_path), json.loads(str(z["camera"])), z["transforms"], z["depth_mm"], z["normal_npy"],
                        z["normal_png"])
    for cam in (False, True):
        frames = O.load_frames(str(tmp_path), js, camera_coordinate_normals=cam)
        rv, rf, _ = O.mesh_pipeline(frames, 10, 1, 7)
        mesh = isooctree_mesh_files(str(tmp_path), js, camera_coordinate_normals=cam, pixel_stride=1, max_depth=7,
                                    subdivision_threshold=10)
        assert rf.shape[0] > 1000
        assert np.array_equal(mesh.faces.cpu().numpy(), rf)
        np.testing.assert_allclose(mesh.vertices.cpu().numpy(), rv, rtol=0, atol=1e-5)
        back = read_obj(str(tmp_path / "mesh.obj"))
        assert torch.equal(back.faces, mesh.faces.cpu()) and (back.vertices - mesh.vertices.cpu()).abs().max() <= 1e-6
    ply = str(tmp_path / "m.ply")
    mesh = isooctree_mesh_files(str(tmp_path), js, pixel_stride=1, max_depth=7, subdivision_threshold=10, output_mesh_file=ply,
                                debug_ply_file=str(tmp_path / "hint.ply"))
    assert torch.equal(read_ply(ply).vertices, mesh.vertices.cpu())
    from dn_splatter_b200.poisson import read_point_cloud_ply

    assert read_point_cloud_ply(str(tmp_path / "hint.ply"))[0].shape[0] == O.hint_cloud(frames, 1)[0].shape[0]


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


def test_export_isooctree_mesh_on_the_room(room, tmp_path):
    """The walls are found to within 1.5 finest cells.  Behind them, where the back mask (points up to 25 % of the depth
    behind an observed surface read -1) stops and unobserved samples read 1, the field crosses 0 again inside the root
    cube's 2.5 % margin: that outer shell is part of what isoFunc defines (in -cam mode get_depth_values tests the
    camera-frame normals against world rays, so many frames drop out and the band is patchy), and is counted apart."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components

    from dn_splatter_b200.isooctree import build_octree, export_isooctree_mesh, hint_samples, render_frames
    from dn_splatter_b200.mesh import read_obj, read_ply

    m, cams = room
    D, stride = 8, 2
    mesh = export_isooctree_mesh(m, cams, str(tmp_path), max_depth=D, pixel_stride=stride)
    v, f = mesh.vertices.cpu().numpy(), mesh.faces.cpu().numpy()
    assert f.shape[0] > 10000 and np.isfinite(v).all()
    hint = hint_samples(render_frames(m, cams), stride)[0]
    tree = build_octree(hint, D, 50)
    hint = hint.cpu().numpy()

    def wall(p):  # the wall each point is nearest to, and its |coordinate| along that wall's axis
        a = np.argmax(np.abs(p), axis=1)
        return 2 * a + (p[np.arange(p.shape[0]), a] > 0), np.abs(p[np.arange(p.shape[0]), a])

    hw, hd = wall(hint)
    plane = np.array([np.median(hd[hw == k]) for k in range(6)])  # the rendered depth lies ~0.01 inside the walls
    vw, vd = wall(v)
    off = vd - plane[vw]
    near = np.abs(off) <= 1.5 * tree.cell
    shell = off > 1.5 * tree.cell
    margin = 0.025 * (hint.max(0) - hint.min(0)).max() + (plane.max() - plane.min())
    print(f"room: {v.shape[0]} vertices, {near.mean():.4f} within 1.5 cells of a wall plane, {shell.mean():.4f} on the "
          f"outer shell, cell {tree.cell:.5f}")
    assert (off[shell] <= margin + tree.cell).all()  # the shell stays inside the root cube's margin
    assert near[~shell].mean() >= 0.99 and shell.mean() <= 0.25
    wall_faces = f[near[f].all(axis=1)]
    adj = coo_matrix((np.ones(3 * wall_faces.shape[0]), (np.repeat(wall_faces[:, 0], 3), wall_faces.reshape(-1))),
                     shape=(v.shape[0],) * 2)
    _, lab = connected_components(adj, directed=False)
    assert np.bincount(lab[wall_faces[:, 0]]).max() >= 0.95 * wall_faces.shape[0]
    back = read_obj(str(tmp_path / "mesh.obj"))
    assert torch.equal(back.faces, mesh.faces.cpu()) and (back.vertices - mesh.vertices.cpu()).abs().max() <= 1e-6
    ply = export_isooctree_mesh(m, cams, str(tmp_path), max_depth=7, pixel_stride=4, mesh_file="mesh.ply")
    back = read_ply(str(tmp_path / "mesh.ply"))
    assert torch.equal(back.faces, ply.faces.cpu()) and torch.equal(back.vertices, ply.vertices.cpu())


def test_model_route_equals_file_route(room, tmp_path):
    """The renders written as render_model.py writes them (depth / 0.001 as .npy, uint8(normal * 255) as .png), read back
    with -cam, give the mesh the model route builds without the files."""
    from PIL import Image

    from dn_splatter_b200.isooctree import export_isooctree_mesh, isooctree_mesh_files
    from dn_splatter_b200.render_service import ViewRenderer

    m, cams = room
    cams = cams[:12]
    os.makedirs(tmp_path / "depth" / "raw")
    os.makedirs(tmp_path / "normal")
    frames = []
    for idx, maps in ViewRenderer(m, keys=("depth", "normal"), to_host=False).render(cams):
        iid = f"{idx:05d}"
        np.save(tmp_path / "depth" / "raw" / f"frame_{iid}.npy", (maps["depth"].float() / 0.001).cpu().numpy())
        nrm = maps["normal"].float().cpu().numpy() * 255
        Image.fromarray(nrm.astype(np.uint8)).save(tmp_path / "normal" / f"frame_{iid}.png")
        frames.append({"file_path": f"images/frame_{iid}.png",
                       "transform_matrix": cams[idx].camera_to_worlds[0].cpu().double().numpy().tolist()})
    c = cams[0]
    data = {"w": int(c.width), "h": int(c.height), "fl_x": float(c.fx), "fl_y": float(c.fy), "cx": float(c.cx),
            "cy": float(c.cy), "frames": frames}
    js = str(tmp_path / "transforms.json")
    with open(js, "w") as fh:
        json.dump(data, fh)
    a = isooctree_mesh_files(str(tmp_path), js, camera_coordinate_normals=True, max_depth=7)
    b = export_isooctree_mesh(m, cams, str(tmp_path / "model"), max_depth=7)
    assert a.faces.shape[0] > 1000
    assert torch.equal(a.faces, b.faces) and torch.equal(a.vertices, b.vertices)
