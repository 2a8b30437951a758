"""CPU checks of the isooctree extractor: oracle/isooctree_ref.py against the reference's own outputs
(tests/golden/dn_isooctree.npz), the octree and fill rules against brute force, the OBJ writer, the C ABI's argument
errors and the device-memory budget, and that the GPU test's acceptance rule detects each restated slip."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from oracle import isooctree_ref as O
from tests import isooctree_scene as S
from tests.golden.make_golden_isooctree import SETTINGS

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dn_isooctree.npz")


def golden():
    return np.load(GOLDEN)


def golden_frames(z, cam_normals):
    cam = O.CameraModel(json.loads(str(z["camera"])))
    return [O.Frame(cam, z["transforms"][i], z["depth_mm"][i][..., 0], z["normal_png"][i] if cam_normals else z["normal_npy"][i],
                    cam_normals) for i in range(z["transforms"].shape[0])]


@pytest.mark.parametrize("name", list(SETTINGS))
def test_oracle_reproduces_reference_golden(name):
    z = golden()
    cam, kw = SETTINGS[name]
    kw = dict(kw)
    stride = kw.pop("pixel_stride")
    frames = golden_frames(z, cam)
    hint, _ = O.hint_cloud(frames, stride)
    assert np.array_equal(hint, z[f"{name}/hint"]) and hint.shape[0] > 50
    want = z[f"{name}/values"]
    got = O.iso_func(frames, z["queries"], **kw)
    assert np.abs(got - want).max() <= 1e-12
    assert ((want > -1) & (want < 1)).sum() > 100 and (want == -1).any() and (want == 1).any()


def test_golden_folder_round_trip(tmp_path):
    z = golden()
    js = S.write_folder(str(tmp_path), json.loads(str(z["camera"])), z["transforms"], z["depth_mm"], z["normal_npy"],
                        z["normal_png"])
    for cam in (False, True):
        a = O.load_frames(str(tmp_path), js, camera_coordinate_normals=cam)
        b = golden_frames(z, cam)
        assert len(a) == len(b) == 6
        for fa, fb in zip(a, b):
            assert np.array_equal(fa.depth_raw, fb.depth_raw) and np.array_equal(fa.normal_raw, fb.normal_raw)
            assert np.array_equal(fa.pose_c2w, fb.pose_c2w)
    assert len(O.load_frames(str(tmp_path), js, max_frames=2, frame_stride=2)) == 2


def _clustered_cloud(n=3000, seed=1):
    g = np.random.default_rng(seed)
    centres = g.uniform(-1, 1, (6, 3))
    pts = centres[g.integers(0, 6, n)] + g.normal(0, 0.08, (n, 3))
    return np.concatenate([pts, g.uniform(-1.2, 1.2, (n // 10, 3))])


@pytest.mark.parametrize("threshold", [1, 7, 50, 10 ** 6])
def test_octree_rule_matches_brute_force_counts(threshold):
    pts = _clustered_cloud()
    D = 5
    leaves, origin, cell = O.octree(pts, D, threshold)
    level, lo, size = O.leaf_boxes(leaves, D)
    fine = O.finest_cells(pts, origin, cell, D)
    # every leaf: its parent split (count >= threshold) and it does not (count < threshold or level == D)
    for lv, c, s in zip(level, lo, size):
        inside = np.all((fine >= c) & (fine < c + s), axis=1).sum()
        assert lv == D or inside < threshold
        if lv > 0:
            ps = 2 * s
            pc = (c // ps) * ps
            assert np.all((fine >= pc) & (fine < pc + ps), axis=1).sum() >= threshold
    # the leaves tile the root cube exactly once
    R = 1 << D
    cover = np.zeros((R, R, R), np.int64)
    for c, s in zip(lo, size):
        cover[c[0]:c[0] + s, c[1]:c[1] + s, c[2]:c[2] + s] += 1
    assert (cover == 1).all()
    assert np.array_equal(leaves, np.sort(leaves))
    if threshold == 10 ** 6:
        assert leaves.tolist() == [0]


def test_root_cube():
    pts = _clustered_cloud()
    origin, side = O.root_cube(pts)
    lo, hi = pts.min(0), pts.max(0)
    assert np.isclose(side, 1.05 * (hi - lo).max())
    assert np.allclose(origin + side / 2, (lo + hi) / 2)


def test_fill_matches_scalar_loop():
    D = 4
    pts = _clustered_cloud(800)
    leaves, origin, cell = O.octree(pts, D, 20)
    level, lo, size = O.leaf_boxes(leaves, D)
    assert len(set(level.tolist())) >= 3
    keys = O.leaf_corners(leaves, D)
    vals = np.random.default_rng(3).normal(size=keys.shape[0]).astype(np.float32)
    field = O.fill(leaves, keys, vals, D)
    R1 = (1 << D) + 1
    lookup = dict(zip(keys.tolist(), vals.tolist()))
    f32 = np.float32
    for i in range(R1):
        for j in range(R1):
            for k in range(R1):
                hold = [n for n in range(leaves.shape[0])
                        if all(lo[n][a] <= p <= lo[n][a] + size[n] for a, p in enumerate((i, j, k)))]
                n = min(hold, key=lambda q: size[q])  # the smallest leaf holding the sample
                s = int(size[n])
                cv = [[[f32(lookup[((lo[n][0] + dx * s) * R1 + lo[n][1] + dy * s) * R1 + lo[n][2] + dz * s])
                        for dz in (0, 1)] for dy in (0, 1)] for dx in (0, 1)]
                t = [f32(p - lo[n][a]) / f32(s) for a, p in enumerate((i, j, k))]
                lerp = lambda a, b, u: (f32(1) - u) * a + u * b  # noqa: E731
                c0 = lerp(lerp(cv[0][0][0], cv[1][0][0], t[0]), lerp(cv[0][1][0], cv[1][1][0], t[0]), t[1])
                c1 = lerp(lerp(cv[0][0][1], cv[1][0][1], t[0]), lerp(cv[0][1][1], cv[1][1][1], t[0]), t[1])
                want = lerp(c0, c1, t[2])
                assert field[i, j, k] == want, (i, j, k)
                key = (i * R1 + j) * R1 + k
                if key in lookup:  # a corner sample keeps its evaluated value
                    assert field[i, j, k] == f32(lookup[key])


def test_obj_round_trip(tmp_path):
    from dn_splatter_b200.mesh import TriangleMesh, read_obj, write_obj

    g = torch.Generator().manual_seed(0)
    v = (torch.rand(50, 3, generator=g) - 0.5) * 4
    f = torch.randint(0, 50, (80, 3), generator=g, dtype=torch.int32)
    p = str(tmp_path / "m.obj")
    write_obj(p, TriangleMesh(v, f, None))
    lines = open(p).read().splitlines()
    assert lines[0].startswith("v ") and lines[50].startswith("f ") and len(lines) == 130
    back = read_obj(p)
    assert torch.equal(back.faces, f)
    assert (back.vertices - v).abs().max() <= 1e-6  # "%f": 6 decimals
    write_obj(p, TriangleMesh(torch.zeros(0, 3), torch.zeros(0, 3, dtype=torch.int32), None))
    assert read_obj(p).faces.shape == (0, 3)


def test_cli_matches_script_flags():
    from dn_splatter_b200 import isooctree as I

    seen = {}
    orig = I.isooctree_mesh_files
    try:
        I.isooctree_mesh_files = lambda root, **kw: seen.update(root=root, **kw)
        I.main(["room", "-cam", "--pixel_stride", "3", "--max_depth", "7", "--tsdf_abs", "0.1", "-o", "x.ply"])
    finally:
        I.isooctree_mesh_files = orig
    assert seen["root"] == "room" and seen["camera_coordinate_normals"] and seen["pixel_stride"] == 3
    assert seen["max_depth"] == 7 and seen["tsdf_abs"] == 0.1 and seen["output_mesh_file"] == "x.ply"
    assert seen["subdivision_threshold"] == 50 and seen["tsdf_rel"] == 0.05 and not seen["disable_normals"]


# ------------------------------------------------------------------------------------------------ C ABI
@pytest.fixture(scope="module")
def lib():
    from dn_splatter_b200 import _lib as L

    if not os.path.exists(L.LIB_PATH):
        from dn_splatter_b200.build import build

        build()
    return L.load()


def test_abi_argument_errors(lib):
    from dn_splatter_b200 import _lib as L

    fr = L.DnrIsoFrames()
    assert lib.dnr_iso_samples_workspace_bytes(None, 1) == -1
    assert lib.dnr_iso_samples_workspace_bytes(C.byref(fr), 1) == -1  # no buffers
    fr.depth, fr.normals, fr.poses = 16, 16, 16
    assert lib.dnr_iso_samples_workspace_bytes(C.byref(fr), 1) == -2  # no frames
    fr.n_frames, fr.width, fr.height = 2, 8, 6
    assert lib.dnr_iso_samples_workspace_bytes(C.byref(fr), 0) == -2
    cnt = C.c_int64()
    assert lib.dnr_iso_samples(C.byref(fr), 1, None, 0, None, None, C.byref(cnt), None) == -1
    ws = lib.dnr_iso_samples_workspace_bytes(C.byref(fr), 1)
    assert lib.dnr_iso_samples(C.byref(fr), 1, 16, ws - 1, 16, None, C.byref(cnt), None) == -5
    p = L.DnrIsoParams()
    assert lib.dnr_iso_eval(C.byref(fr), None, None, 1, None, None) == -1
    assert lib.dnr_iso_eval(C.byref(fr), C.byref(p), None, 1, None, None) == -2  # no pass
    p.passes = 1
    assert lib.dnr_iso_eval(C.byref(fr), C.byref(p), None, 1, None, None) == -3  # a normal pass without normals
    p.use_normals = 1
    assert lib.dnr_iso_eval(C.byref(fr), C.byref(p), None, 1, None, None) == -1
    assert lib.dnr_iso_eval(C.byref(fr), C.byref(p), None, 0, None, None) == 0
    g = L.DnrIsoGrid()
    g.cell, g.threshold, g.max_depth = 0.1, 50, 11
    assert lib.dnr_iso_octree_workspace_bytes(C.byref(g), 10) == -2  # past DNR_ISO_MAX_DEPTH
    g.max_depth, g.threshold = 10, 0
    assert lib.dnr_iso_octree_workspace_bytes(C.byref(g), 10) == -2
    g.threshold, g.cell = 50, 0.0
    assert lib.dnr_iso_octree_workspace_bytes(C.byref(g), 10) == -2
    g.cell = 0.1
    counts = (C.c_int64 * 11)()
    assert lib.dnr_iso_octree(C.byref(g), None, 10, None, 0, counts, None) == -1
    ws = lib.dnr_iso_octree_workspace_bytes(C.byref(g), 10)
    assert lib.dnr_iso_octree(C.byref(g), 16, 10, 16, ws - 1, counts, None) == -5
    assert lib.dnr_iso_corners_workspace_bytes(C.byref(g), 0) == -2
    counts[0] = 1
    ws, n_corners = lib.dnr_iso_corners_workspace_bytes(C.byref(g), 1), C.c_int64()
    assert lib.dnr_iso_corners(C.byref(g), 16, counts, 16, ws - 1, 16, 16, 16, 16, C.byref(n_corners), None) == -5
    assert lib.dnr_iso_fill(C.byref(g), None, counts, None, None, None, None) == -1


def test_python_argument_errors_and_budget(lib):
    from dn_splatter_b200 import isooctree as I

    with pytest.raises(ValueError, match="max_depth"):
        I.iso_grid((0, 0, 0), 1.0, 11, 50)
    with pytest.raises(ValueError, match="subdivision_threshold"):
        I.iso_grid((0, 0, 0), 1.0, 8, 0)
    need = I.required_bytes(200, 1920, 1080, 6, 10, 50)
    assert need > 4 * 1025 ** 3 + 200 * 1920 * 1080 * 16  # the dense grid and the frames at least
    assert I.required_bytes(200, 1920, 1080, 6, 9, 50) < need
    I.check_budget(200, 1920, 1080, 6, 10, 50, need)
    with pytest.raises(ValueError, match="max_bytes"):
        I.check_budget(200, 1920, 1080, 6, 10, 50, need - 1)


# ------------------------------------------------------------------------------------------------ slips
@pytest.mark.parametrize("slip", ["floor", "tie", "cut4", "no_back", "norm_ray"])
def test_acceptance_rule_detects_each_slip(slip):
    """The GPU eval test accepts |gpu - oracle| <= S.eval_tolerance(oracle) on these cases (the golden folder's queries
    in every mode, and the frame-order tie set); each slip moves some value by >= 10x that."""
    z = golden()
    worst = 0.0
    for name, (cam, kw) in SETTINGS.items():
        kw = {k: v for k, v in kw.items() if k != "pixel_stride"}
        frames = golden_frames(z, cam)
        if slip == "tie":
            frames = S.tie_frames(frames)
        want = O.iso_func(frames, z["queries"], **kw)
        got = O.iso_func(frames, z["queries"], slip=slip, **kw)
        worst = max(worst, float((np.abs(got - want) / S.eval_tolerance(want)).max()))
    assert worst >= 10, worst
