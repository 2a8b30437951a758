"""CPU checks of the mesh evaluation: oracle/mesh_eval_ref.py against goldens from the reference's own
eval_mesh_vis_cull.py / metrics.py (tests/golden/make_golden_mesh_eval.py), the oracle's subdivision and ray cast against
independent restatements and analytic scenes, the PLY reader, and the argument checks of the C ABI entry points."""
import ctypes as C
import io
import os

import numpy as np
import pytest
import torch

from dn_splatter_b200 import _lib as L
from oracle import mesh_eval_ref as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dn_mesh_eval.npz")


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLDEN)


def _cams(poses, K):
    return [R.camera_block(p, K[0, 0], K[1, 1], K[0, 2], K[1, 2]) for p in poses]


def test_visibility_counts_equal_the_reference(gold):
    H, W = (int(x) for x in gold["vis_hw"])
    cams = _cams(gold["vis_poses"], gold["vis_K"])
    for tag, rend, g in (("both", gold["vis_rendered"], gold["vis_gt"]), ("noocc", None, gold["vis_gt"]),
                         ("nomiss", gold["vis_rendered"], None)):
        obs, inv = R.visibility_counts(gold["vis_points"], cams, W, H, rend, g)
        assert np.array_equal(obs, gold[f"vis_{tag}_obs"].astype(np.int64)), tag
        assert np.array_equal(inv, gold[f"vis_{tag}_invalid"].astype(np.int64)), tag
    assert gold["vis_both_obs"].max() >= 3 and gold["vis_both_invalid"].max() >= 2 and (gold["vis_both_obs"] == 0).any()
    obs, inv = R.visibility_counts(gold["vis_points"], cams[:1], W, H, gold["vis_rendered"][:1], gold["vis_gt"][:1])
    assert np.array_equal(obs, gold["vis_one_obs"]) and np.array_equal(inv, gold["vis_one_invalid"])


def test_cull_mesh_equals_the_reference(gold):
    W, H, fx, fy, cx, cy, max_edge = gold["cull_params"]
    W, H = int(W), int(H)
    cams = [R.camera_block(p, fx, fy, cx, cy) for p in gold["cull_room_poses"]]
    depths = gold["cull_depth_png"] / 6553.5
    depths = depths.astype(np.float32)
    v, f, obs, inv = R.cull_mesh(gold["cull_room_in_vertices"], gold["cull_room_in_faces"], cams, W, H, gt_depths=depths,
                                 max_edge=max_edge)
    assert np.array_equal(obs, gold["cull_room_obs"].astype(np.int64))
    assert np.array_equal(inv, gold["cull_room_invalid"].astype(np.int64))
    assert np.array_equal(f, gold["cull_room_faces"]) and np.array_equal(v, gold["cull_room_vertices"])
    n_sub = R.subdivide_to_size(gold["cull_room_in_vertices"], gold["cull_room_in_faces"], max_edge)[1].shape[0]
    assert 0 < f.shape[0] < n_sub  # the missing-depth corner and the unseen faces go
    # the ray cast the golden used for pyrender's depth is the oracle's own
    d0 = R.ray_cast_depth(*R.remove_unreferenced(gold["cull_room_in_vertices"], gold["cull_room_in_faces"]), cams[0], W, H)
    assert np.array_equal(d0.astype(np.float32), gold["cull_room_rendered"][0])


@pytest.mark.parametrize("tag", ["near", "mixed", "far"])
def test_metrics_equal_the_reference(gold, tag):
    f = gold[f"met_{tag}_faces"]
    pn = R.face_normals(gold[f"met_{tag}_pred_vertices"], f)[gold[f"met_{tag}_pred_idx"]]
    gn = R.face_normals(gold[f"met_{tag}_gt_vertices"], f)[gold[f"met_{tag}_gt_idx"]]
    got = R.mesh_metrics(gold[f"met_{tag}_pred_samples"], pn, gold[f"met_{tag}_gt_samples"], gn)
    want = gold[f"met_{tag}_values"]
    for k, w in zip(("Acc", "Comp", "C-L1", "NC", "F-score"), want):
        if np.isnan(w):
            assert np.isnan(got[k]), k
        else:
            assert abs(got[k] - w) <= 1e-12 * abs(w), (k, got[k], w)
    assert len(gold[f"met_{tag}_pred_samples"]) == int(R.triangle_areas(gold[f"met_{tag}_pred_vertices"], f).sum() * 1e4)


def test_point_cloud_metrics_equal_the_reference(gold):
    p, g = gold["pd_pred"], gold["pd_gt"]
    assert abs(R.pd_accuracy(p, g) - gold["pd_acc"][0]) <= 1e-12 * gold["pd_acc"][0]
    assert abs(R.pd_accuracy(p, g, 50) - gold["pd_acc"][1]) <= 1e-12 * gold["pd_acc"][1]
    assert abs(R.pd_completeness(p, g) - gold["pd_comp"][0]) <= 1e-12 * gold["pd_comp"][0]
    assert abs(R.pd_completeness(p, g, 0.02) - gold["pd_comp"][1]) <= 1e-12 * gold["pd_comp"][1]


# ------------------------------------------------------------------------------------------------ subdivision
def _brute_subdivide(tri, max_edge, depth=0, max_iter=10):
    """Recursive restatement: a triangle (3 corners) is final when no edge exceeds max_edge, else its 4 children."""
    e = [np.sqrt(((tri[(k + 1) % 3] - tri[k]) ** 2).sum()) for k in range(3)]
    if max(e) <= max_edge:
        return [tri]
    if depth == max_iter:
        return []
    a, b, c = tri
    ab, bc, ca = (a + b) / 2, (b + c) / 2, (c + a) / 2
    out = []
    for t in ([a, ab, ca], [ab, b, bc], [ca, bc, c], [ab, bc, ca]):
        out += _brute_subdivide(np.array(t), max_edge, depth + 1, max_iter)
    return out


def _random_mesh(seed):
    rng = np.random.default_rng(seed)
    v = rng.normal(size=(9, 3)) * np.array([0.3, 0.2, 0.1])
    f = np.array([[0, 1, 2], [1, 3, 2], [2, 3, 4], [4, 5, 6], [6, 7, 8], [0, 8, 7], [1, 5, 7]])
    return v, f


@pytest.mark.parametrize("max_edge", [0.05, 0.11, 1.0])
def test_subdivision_matches_the_recursive_rule(max_edge):
    v, f = _random_mesh(3)
    sv, sf, dropped = R.subdivide_to_size(v, f, max_edge)
    assert dropped == 0
    assert (R.edge_lengths(sv, sf) <= max_edge).all()
    assert abs(R.triangle_areas(sv, sf).sum() - R.triangle_areas(v, f).sum()) <= 1e-12 * R.triangle_areas(v, f).sum()
    brute = np.array([t for tri in v[f] for t in _brute_subdivide(tri, max_edge)])
    bf = np.arange(3 * len(brute)).reshape(-1, 3)
    assert np.array_equal(R.triangle_multiset(sv, sf), R.triangle_multiset(brute.reshape(-1, 3), bf))
    # midpoints are welded: every vertex is distinct
    assert np.unique(sv, axis=0).shape[0] == sv.shape[0]


def test_subdivision_drops_faces_beyond_max_iter():
    v = np.array([[0.0, 0, 0], [1.0, 0, 0], [0, 1.0, 0], [0.0, 0, 0.01], [0.01, 0, 0.01], [0, 0.01, 0.01]])
    f = np.array([[0, 1, 2], [3, 4, 5]])
    sv, sf, dropped = R.subdivide_to_size(v, f, max_edge=0.1, max_iter=2)  # the big face needs 4 rounds
    assert dropped == 16 and sf.shape[0] == 1
    sv, sf, dropped = R.subdivide_to_size(v, f, max_edge=0.1, max_iter=4)
    assert dropped == 0 and sf.shape[0] == 1 + 256


# ------------------------------------------------------------------------------------------------ ray cast
def _cam(W, H, f=40.0, c2w=None):
    return R.camera_block(np.eye(4)[:3] if c2w is None else c2w, f, f * 1.1, W / 2 + 0.3, H / 2 - 0.2)


def test_ray_cast_plane_with_clips_and_back_faces():
    W, H = 31, 23
    cam = _cam(W, H)
    # plane z = -2 in world (in front of an identity OpenGL camera), both windings
    v = np.array([[-50.0, -50, -2], [50, -50, -2], [0, 50, -2]])
    for f in (np.array([[0, 1, 2]]), np.array([[0, 2, 1]])):
        d = R.ray_cast_depth(v, f, cam, W, H)
        assert np.allclose(d, 2.0, rtol=1e-14)
        assert (R.ray_cast_depth(v, f, cam, W, H, far=1.9) == 0).all()
        assert (R.ray_cast_depth(v, f, cam, W, H, near=2.1) == 0).all()
    # behind the camera: nothing
    assert (R.ray_cast_depth(v * np.array([1, 1, -1]), np.array([[0, 1, 2]]), cam, W, H) == 0).all()
    # a tilted plane z = -(2 + 5 x) straddling the near plane: depth is analytic where in [near, far]
    t = np.array([[-50.0, -50, 0], [50, -50, 0], [0, 50, 0]])
    t[:, 2] = -(2 + 5.0 * t[:, 0])
    d = R.ray_cast_depth(t, np.array([[0, 1, 2]]), cam, W, H, near=1.0)
    fx, fy, cx, cy = cam[:4]
    xs = (np.arange(W) + 0.5 - cx) / fx
    want = 2.0 / (1.0 - 5.0 * xs)  # z = 2 + 5 * (x_n z)  (camera x = world x, camera z = -world z)
    want = np.where((want >= 1.0) & (want <= 10.0) & (want > 0), want, 0.0)
    assert np.allclose(d, np.broadcast_to(want, (H, W)), rtol=1e-12)
    assert (d == 0).any() and (d > 0).any()


def _sphere(n=24, r=0.5, centre=(0.0, 0.0, -2.0)):
    th, ph = np.meshgrid(np.linspace(0, np.pi, n + 1), np.linspace(0, 2 * np.pi, 2 * n + 1), indexing="ij")
    v = np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], -1).reshape(-1, 3) * r + np.array(centre)
    idx = np.arange(v.shape[0]).reshape(n + 1, 2 * n + 1)
    a, b, c, d = idx[:-1, :-1], idx[:-1, 1:], idx[1:, :-1], idx[1:, 1:]
    f = np.concatenate([np.stack([a, c, b], -1).reshape(-1, 3), np.stack([b, c, d], -1).reshape(-1, 3)])
    return v, f


def test_ray_cast_sphere_is_close_to_the_analytic_sphere():
    W, H = 41, 37
    cam = _cam(W, H, f=30.0)
    v, f = _sphere(48)
    d = R.ray_cast_depth(v, f, cam, W, H)
    fx, fy, cx, cy = cam[:4]
    i, j = np.meshgrid(np.arange(W), np.arange(H))
    ray = np.stack([(i + 0.5 - cx) / fx, -(j + 0.5 - cy) / fy, -np.ones((H, W))], -1)  # world directions (OpenGL camera)
    c = np.array([0.0, 0.0, -2.0])
    dd, bc = (ray * ray).sum(-1), (ray * c).sum(-1)
    disc = bc * bc - dd * ((c * c).sum() - 0.25)
    t = np.where(disc > 0, (bc - np.sqrt(np.maximum(disc, 0))) / dd, 0.0)
    inner = disc > 0.05 * dd
    assert inner.sum() > 100
    assert np.allclose(d[inner], t[inner], rtol=2e-3)  # a 48-segment sphere sags by < 0.2 % of its radius
    assert (d[disc < 0] == 0).all()


def test_near_edge_marks_pixels_on_edges():
    W, H = 8, 6
    cam = R.camera_block(np.eye(4)[:3], 10.0, 10.0, 4.0, 3.0)  # pixel (4, 3) centre is on the ray x_n = 0.05, y_n = 0.05
    v = np.array([[0.05 * 2, -0.05 * 2, -2], [5, -0.05 * 2, -2], [0.05 * 2, 5, -2]])  # edge through pixel centre column 4
    m = R.near_edge_pixels(v, np.array([[0, 1, 2]]), cam, W, H)
    assert m[:, 4].sum() >= 1 and not m[:, :3].any()


# ------------------------------------------------------------------------------------------------ PLY
def _ply_bytes(fmt, verts, faces, vprops=("x", "y", "z"), vtype="float", extra=True, list_spelling="vertex_indices",
               count_type="uchar", index_type="int"):
    n = len(verts)
    head = [f"ply", f"format {fmt} 1.0", "comment test", f"element vertex {n}"]
    for p in vprops:
        head.append(f"property {vtype} {p}")
    if extra:
        head += ["property uchar red", "property uchar green", "property uchar blue", "property float quality"]
    head += [f"element face {len(faces)}", f"property list {count_type} {index_type} {list_spelling}", "property int flags",
             "end_header"]
    out = io.BytesIO()
    out.write(("\n".join(head) + "\n").encode())
    rng = np.random.default_rng(0)
    cols = rng.integers(0, 256, (n, 3))
    if fmt == "ascii":
        for k, p in enumerate(verts):
            row = [repr(float(x)) for x in p] + ([str(int(c)) for c in cols[k]] + ["0.5"] if extra else [])
            out.write((" ".join(row) + "\n").encode())
        for fc in faces:
            out.write((" ".join([str(len(fc))] + [str(i) for i in fc] + ["7"]) + "\n").encode())
    else:
        e = "<" if fmt == "binary_little_endian" else ">"
        ft = {"float": "f4", "double": "f8"}[vtype]
        ct = {"uchar": "u1", "int": "i4"}[count_type]
        it = {"int": "i4", "uint": "u4"}[index_type]
        for k, p in enumerate(verts):
            out.write(np.asarray(p, e + ft).tobytes())
            if extra:
                out.write(np.asarray(cols[k], "u1").tobytes() + np.asarray([0.5], e + "f4").tobytes())
        for fc in faces:
            out.write(np.asarray([len(fc)], e + ct).tobytes() + np.asarray(fc, e + it).tobytes() + np.asarray([7], e + "i4").tobytes())
    return out.getvalue(), cols


@pytest.mark.parametrize("fmt", ["ascii", "binary_little_endian", "binary_big_endian"])
@pytest.mark.parametrize("spelling", ["vertex_indices", "vertex_index"])
def test_read_triangle_mesh_formats(tmp_path, fmt, spelling):
    from dn_splatter_b200.mesh_eval import read_triangle_mesh

    verts = np.random.default_rng(1).normal(size=(7, 3)).astype(np.float32)
    for faces, want in (([[0, 1, 2], [2, 3, 4], [4, 5, 6]], [[0, 1, 2], [2, 3, 4], [4, 5, 6]]),
                        ([[0, 1, 2, 3], [3, 4, 5], [1, 2, 5, 6, 0]], [[0, 1, 2], [0, 2, 3], [3, 4, 5], [1, 2, 5], [1, 5, 6], [1, 6, 0]])):
        for kw in (dict(), dict(vtype="double"), dict(count_type="int", index_type="uint", extra=False)):
            if fmt == "ascii" and kw.get("count_type"):
                kw = dict(extra=False)
            data, cols = _ply_bytes(fmt, verts, faces, list_spelling=spelling, **kw)
            p = tmp_path / "m.ply"
            p.write_bytes(data)
            m = read_triangle_mesh(str(p))
            assert np.array_equal(m.faces.numpy(), np.asarray(want, np.int32))
            assert m.vertices.dtype == (torch.float64 if kw.get("vtype") == "double" else torch.float32)
            assert np.allclose(m.vertices.numpy(), verts, atol=0 if fmt != "ascii" else 1e-7)
            if kw.get("extra", True):
                assert np.allclose(m.colors.numpy(), cols / 255.0)
            else:
                assert m.colors is None


def test_read_triangle_mesh_round_trips_write_ply(tmp_path):
    from dn_splatter_b200.mesh import TriangleMesh, read_ply, write_ply
    from dn_splatter_b200.mesh_eval import read_triangle_mesh

    rng = np.random.default_rng(2)
    mesh = TriangleMesh(torch.from_numpy(rng.normal(size=(50, 3)).astype(np.float32)),
                        torch.from_numpy(rng.integers(0, 50, (80, 3)).astype(np.int32)),
                        torch.from_numpy(rng.random((50, 3)).astype(np.float32)))
    write_ply(str(tmp_path / "a.ply"), mesh)
    got, old = read_triangle_mesh(str(tmp_path / "a.ply")), read_ply(str(tmp_path / "a.ply"))
    assert torch.equal(got.vertices, mesh.vertices) and torch.equal(got.faces, mesh.faces)
    assert torch.equal(got.colors, old.colors)


def test_read_triangle_mesh_errors(tmp_path):
    from dn_splatter_b200.mesh_eval import read_triangle_mesh

    p = tmp_path / "bad.ply"
    cases = [
        (b"OFF\n3 1 0\n", "not a PLY"),
        (b"ply\nformat binary_middle_endian 1.0\nelement vertex 0\nend_header\n", "unsupported PLY format"),
        (b"ply\nformat ascii 1.0\nelement vertex 1\nproperty float128 x\nend_header\n1\n", "unsupported PLY property type"),
        (b"ply\nformat ascii 1.0\nelement face 0\nproperty list uchar int vertex_indices\nend_header\n", "no vertex element"),
        (b"ply\nformat ascii 1.0\nelement vertex 3\nproperty float x\nproperty float y\nproperty float z\nend_header\n0 0 0\n",
         "ends inside"),
        (b"ply\nformat binary_little_endian 1.0\nelement vertex 3\nproperty float x\nproperty float y\nproperty float z\n"
         b"end_header\n" + b"\0" * 20, "ends inside"),
        (b"ply\nformat ascii 1.0\nelement vertex 1\nproperty float x\nproperty float y\nproperty float z\nelement face 1\n"
         b"property list uchar int vertex_indices\nend_header\n0 0 0\n3 0 1 2\n", "out of range"),
        (b"ply\nformat ascii 1.0\nelement vertex 1\nproperty float x\nproperty float y\nend_header\n0 0\n", "x, y and z"),
        (b"ply\nformat ascii 1.0\nelement vertex 1\nproperty float x\n", "end_header"),
    ]
    for data, msg in cases:
        p.write_bytes(data)
        with pytest.raises(ValueError, match=msg):
            read_triangle_mesh(str(p))


# ------------------------------------------------------------------------------------------------ C ABI
@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(L.LIB_PATH):
        from dn_splatter_b200.build import build

        build()
    return L.load()


def test_mesh_eval_argument_errors_are_negative_codes(lib):
    one = C.c_void_p(16)  # a non-NULL dummy: the checks come first, nothing is dereferenced
    assert lib.dnr_mesh_depth_workspace_bytes(0) == -2
    assert lib.dnr_mesh_depth_workspace_bytes(1000) >= 1000 * (16 + 8 + 8)
    ws = lib.dnr_mesh_depth_workspace_bytes(10)
    assert lib.dnr_mesh_depth(None, 3, one, 10, one, 1, 8, 8, 0.01, 10.0, one, ws, one, None) == -1
    assert lib.dnr_mesh_depth(one, 3, one, 10, one, 1, 8, 8, 0.01, 10.0, one, ws, None, None) == -1
    assert lib.dnr_mesh_depth(one, 0, one, 10, one, 1, 8, 8, 0.01, 10.0, one, ws, one, None) == -2
    assert lib.dnr_mesh_depth(one, 3, one, 10, one, 0, 8, 8, 0.01, 10.0, one, ws, one, None) == -2
    assert lib.dnr_mesh_depth(one, 3, one, 10, one, 1, 0, 8, 0.01, 10.0, one, ws, one, None) == -2
    assert lib.dnr_mesh_depth(one, 3, one, 10, one, 1, 8, 8, 0.0, 10.0, one, ws, one, None) == -3  # near must be > 0
    assert lib.dnr_mesh_depth(one, 3, one, 10, one, 1, 8, 8, 1.0, 0.5, one, ws, one, None) == -3  # far < near
    assert lib.dnr_mesh_depth(one, 3, one, 10, one, 1, 8, 8, 0.01, 10.0, one, ws - 1, one, None) == -5
    assert lib.dnr_mesh_visibility(None, 5, one, None, None, 1, 8, 8, 0.02, one, one, None) == -1
    assert lib.dnr_mesh_visibility(one, 5, one, None, one, 1, 8, 8, 0.02, one, None, None) == -1  # gt without invalid
    assert lib.dnr_mesh_visibility(one, 0, one, None, None, 1, 8, 8, 0.02, one, one, None) == -2
    assert lib.dnr_mesh_visibility(one, 5, one, None, None, 0, 8, 8, 0.02, one, one, None) == -2
    assert lib.dnr_mesh_visibility(one, 5, one, None, None, 1, 8, -1, 0.02, one, one, None) == -2


def test_product_path_fails_loudly_without_cuda():
    from dn_splatter_b200 import mesh_eval

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(L.DnrError):
        mesh_eval.sample_surface(mesh_eval.TriangleMesh(torch.zeros(3, 3), torch.tensor([[0, 1, 2]]), None), 10)


def test_cull_mesh_without_gt_depths_needs_remove_missing_depth_false():
    from dn_splatter_b200 import mesh_eval

    with pytest.raises(ValueError, match="remove_missing_depth"):
        mesh_eval.cull_mesh(mesh_eval.TriangleMesh(torch.zeros(3, 3), torch.tensor([[0, 1, 2]]), None), [], None)


def test_align_is_not_implemented(tmp_path):
    from dn_splatter_b200 import mesh_eval

    with pytest.raises(NotImplementedError):
        mesh_eval.evaluate_mesh_files("gt.ply", "pred.ply", "t.json", str(tmp_path), align=True)
