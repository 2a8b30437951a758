"""CPU checks of the depth-normal pipeline (dn_splatter_b200/depth_normals.py, oracle/normals_ref.py): the oracle against
the golden the reference scripts wrote (tests/golden/make_golden_normals.py), the FastEigen3x3 restatement, the host I/O
helpers, the C-ABI argument errors and the memory budget, and five restated slips that the golden must catch."""
import ctypes as C
import io
import os

import numpy as np
import pytest

from dn_splatter_b200 import _lib as L
from dn_splatter_b200 import depth_normals as DN
from oracle import normals_ref as R
from tests import depth_normals_scene as D

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "dn_depth_normals.npz"))
RUNS = {"omnidata": ("omnidata", 20.0, True, {}), "dsine": ("dsine", 15.0, True, dict(dsine=True, intrinsics_in_frames=True)),
        "depth_to_normal": ("depth_to_normal", 10.0, False, {}),
        # angle_treshold equal to an angle frame_1's pixels attain: pins the strict > of the mask
        "omnidata_tie": ("omnidata", float(GOLDEN["omnidata_tie/threshold"]), True, {})}


def golden_points(run):
    return GOLDEN[f"{'omnidata' if run == 'omnidata_tie' else run}/points"]


def oracle_run(root, mode, threshold, rename_png, slip=None):
    """The oracle's pipeline over a capture folder: (points per frame, {relative path: bytes})."""
    frames, (fx, fy, cx, cy, w, h) = DN.load_transforms(root, "transforms.json")
    pts_all, files = [], {}
    for f in frames:
        name = f["file_path"].split("/")[-1]
        depth = DN.resize_nearest(DN.load_depth(os.path.join(root, f["depth_file_path"])), w, h)
        if slip == "npy_unscaled" and f["depth_file_path"].endswith(".npy"):
            depth = depth / np.float32(0.001)
        c2w = DN.c2w_of(f)
        if slip == "fp64_camera":
            pts, _ = R.backproject(depth.astype(np.float64), np.float64(fx), fy, cx, cy, w, h, c2w)
        else:
            pts, _ = R.backproject(depth, fx, fy, cx, cy, w, h, c2w)
        pts_all.append(pts)
        if slip in ("fp64_camera", "npy_unscaled"):
            continue
        n = R.estimate_normals(pts)[0]
        if slip != "unoriented":
            n = R.orient(pts, n, c2w[:3, 3])
        mono = DN.read_mono(os.path.join(root, "normals_from_pretrain", name.replace("jpg", "png")), w, h)
        deg, mask, enc = R.consistency(n, mono, c2w, mode, threshold)
        if slip == "ge":
            mask = deg >= threshold
        if slip == "decoded_angle":  # DepthToNormal's angle taken between the decoded unit vectors
            mask = R.consistency(n, mono, c2w, "omnidata", threshold)[1]
        save = name.replace("png", "jpg") if rename_png else name
        for sub, img in (("depth_normals", enc.reshape(h, w, 3)), ("depth_normals_mask", (mask * 255).astype(np.uint8).reshape(h, w))):
            buf = os.path.join(root, sub)
            os.makedirs(buf, exist_ok=True)
            DN.write_image(os.path.join(buf, save), img)
    return pts_all, (D.list_outputs(root) if slip not in ("fp64_camera", "npy_unscaled") else {})


def golden_files(run):
    return {f: GOLDEN[f"{run}/file/{f}"].tobytes() for f in GOLDEN[f"{run}/files"]}


def decoded(b):
    from PIL import Image

    return np.array(Image.open(io.BytesIO(b)))


@pytest.fixture(scope="module")
def oracle_outputs(tmp_path_factory):
    out = {}
    for run, (mode, thr, rename, folder) in RUNS.items():
        root = str(tmp_path_factory.mktemp(run))
        D.build(root, **folder)
        out[run] = (root,) + oracle_run(root, mode, thr, rename)
    return out


@pytest.mark.parametrize("run", list(RUNS))
def test_oracle_equals_golden(oracle_outputs, run):
    _, pts, files = oracle_outputs[run]
    np.testing.assert_array_equal(np.stack(pts), golden_points(run))  # bit for bit
    want = golden_files(run)
    assert list(files) == list(want)
    for f, b in want.items():
        if f.endswith(".jpg"):
            assert files[f] == b, f
        else:
            np.testing.assert_array_equal(decoded(files[f]), decoded(b), err_msg=f)
    masks = np.concatenate([decoded(b).reshape(-1) for f, b in want.items() if f.startswith("depth_normals_mask")])
    assert (masks < 128).any() and (masks >= 128).any()  # both mask values occur


def test_golden_folder_shape():
    assert sorted(D.NAMES, key=DN.natural_key) == ["frame_1.jpg", "frame_2.png", "frame_3.png", "frame_10.jpg", "frame_11.jpg",
                                                    "frame_20.jpg"]
    assert sorted(D.NAMES) != sorted(D.NAMES, key=DN.natural_key)
    holes = (GOLDEN["depth_mm"] == 0).reshape(6, -1).sum(1)
    assert holes.min() == 0 and 0 < sorted(holes)[-2] < 200 < holes.max()


@pytest.mark.parametrize("slip", ["fp64_camera", "npy_unscaled", "ge", "decoded_angle", "unoriented"])
def test_each_slip_changes_the_golden(tmp_path, slip):
    run = {"fp64_camera": "omnidata", "npy_unscaled": "omnidata", "ge": "omnidata_tie", "decoded_angle": "depth_to_normal",
           "unoriented": "omnidata"}[slip]
    mode, thr, rename, folder = RUNS[run]
    D.build(str(tmp_path), **folder)
    if slip in ("fp64_camera", "npy_unscaled"):
        pts, _ = oracle_run(str(tmp_path), mode, thr, rename, slip)
        assert not np.array_equal(np.stack(pts), golden_points(run))
        return
    _, files = oracle_run(str(tmp_path), mode, thr, rename, slip)
    want = golden_files(run)
    assert any(not np.array_equal(decoded(files[f]), decoded(b)) for f, b in want.items())


def _branch_cases():
    g = np.random.default_rng(3)
    plane = np.c_[g.normal(size=(50, 2)), np.zeros(50)] @ np.linalg.qr(g.normal(size=(3, 3)))[0]
    line = np.outer(g.normal(size=40), [1.0, 2.0, -0.5])
    return {
        "zero": np.zeros((3, 3)),
        "diagonal_ties": np.diag([2.0, 1.0, 1.0]),
        "diagonal": np.diag([3.0, 0.5, 1.0]),
        "planar": np.cov(plane.T, bias=True),
        "collinear": np.cov(line.T, bias=True),
        "negative_half_det": np.array([[2.0, 0.9, 0.0], [0.9, 2.0, 0.0], [0.0, 0.0, 0.3]]) * -1 + 3 * np.eye(3),
    }


@pytest.mark.parametrize("name", list(_branch_cases()))
def test_fast_eigen_branches(name):
    A = _branch_cases()[name]
    taken = []
    v = R.fast_eigen3x3(A, taken)
    if name == "zero":
        assert taken == ["zero"] and not v.any()
        return
    if name == "diagonal_ties":  # strict comparisons: a tie for the smallest falls through to z
        assert taken == ["diagonal"] and v.tolist() == [0.0, 0.0, 1.0]
        return
    w = np.linalg.eigvalsh(A)  # v spans the smallest eigenvalue's space (two-dimensional for the line)
    assert abs(np.linalg.norm(v) - 1) < 1e-12 and np.linalg.norm(A @ v - w[0] * v) < 1e-9 * w[2], (taken, v)
    if name == "negative_half_det":
        assert taken[0].startswith("neg")


def test_fast_eigen_matches_eigh():
    g = np.random.default_rng(7)
    branches = set()
    for _ in range(2000):
        X = g.normal(size=(30, 3)) * g.uniform(0.01, 3, 3)
        A = np.cov((X @ np.linalg.qr(g.normal(size=(3, 3)))[0]).T, bias=True)
        w, V = np.linalg.eigh(A)
        taken = []
        v = R.fast_eigen3x3(A, taken)
        branches.add(taken[0])
        if w[1] - w[0] > 1e-6 * w[2]:
            assert abs(abs(v @ V[:, 0]) - 1) < 1e-8
    assert len(branches) >= 2, branches


def test_natural_sort():
    names = ["f10.png", "f2.png", "f1.png", "a/f02b.png", "f2a.png", "10x", "9x"]
    assert sorted(names, key=DN.natural_key) == ["9x", "10x", "a/f02b.png", "f1.png", "f2.png", "f2a.png", "f10.png"]


def test_resize_nearest_matches_cv2():
    cv2 = pytest.importorskip("cv2")
    img = np.random.default_rng(0).uniform(0, 5, (37, 53)).astype(np.float32)
    for w, h in ((64, 48), (20, 15), (53, 37), (100, 11), (7, 90)):
        np.testing.assert_array_equal(DN.resize_nearest(img, w, h), cv2.resize(img, (w, h), interpolation=cv2.INTER_NEAREST))


def test_pil_jpeg_equals_cv2(tmp_path):
    cv2 = pytest.importorskip("cv2")
    g = np.random.default_rng(1)
    grey = (g.uniform(size=(48, 64)) > 0.5).astype(np.uint8) * 255
    bgr = g.integers(0, 256, (48, 64, 3)).astype(np.uint8)
    for img in (grey, bgr):
        p = str(tmp_path / "x.jpg")
        DN.write_image(p, img)
        assert open(p, "rb").read() == cv2.imencode(".jpg", img)[1].tobytes()


def test_mono_size_mismatch_raises(tmp_path):
    from PIL import Image

    D.build(str(tmp_path))
    Image.fromarray(np.zeros((10, 12, 3), np.uint8)).save(tmp_path / "normals_from_pretrain" / "frame_10.png")
    frames, (_, _, _, _, w, h) = DN.load_transforms(str(tmp_path), "transforms.json")
    with pytest.raises(ValueError, match="frame_10.png"):
        for f in frames:
            DN._frame_job(str(tmp_path), f, str(tmp_path / "normals_from_pretrain"), w, h)


def test_nonfinite_depth_raises(tmp_path):
    p = tmp_path / "d.npy"
    np.save(p, np.array([[1.0, np.nan]], np.float32))
    with pytest.raises(ValueError, match="d.npy"):
        DN.load_depth(p)


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(L.LIB_PATH):
        from dn_splatter_b200.build import build

        build()
    return L.load()


def test_abi_argument_errors(lib):
    s = L.DnrDnSearch()
    s.cell, s.k = 1.0, 200
    pose = L.DnrDnPose()
    intr = (C.c_float * 4)(1, 1, 0, 0)
    fake = C.c_void_p(16)
    assert lib.dnr_dn_normals_workspace_bytes(0) < 0
    assert lib.dnr_dn_normals_workspace_bytes(1 << 31) < 0
    ws = lib.dnr_dn_normals_workspace_bytes(1000)
    assert ws > 0 and lib.dnr_dn_normals_workspace_bytes(2000) > ws
    assert lib.dnr_dn_normals(None, 10, C.byref(s), fake, ws, fake, None, None, None, None, None) == -1
    assert lib.dnr_dn_normals(fake, 0, C.byref(s), fake, ws, fake, None, None, None, None, None) == -2
    s.k = 257
    assert lib.dnr_dn_normals(fake, 1000, C.byref(s), fake, ws, fake, None, None, None, None, None) == -3
    s.k, s.cell = 200, 0.0
    assert lib.dnr_dn_normals(fake, 1000, C.byref(s), fake, ws, fake, None, None, None, None, None) == -2
    s.cell = 1.0
    assert lib.dnr_dn_normals(fake, 1000, C.byref(s), fake, ws - 1, fake, None, None, None, None, None) == -5
    assert lib.dnr_dn_backproject(None, 4, 4, intr, C.byref(pose), None, fake, None) == -1
    assert lib.dnr_dn_backproject(fake, 0, 4, intr, C.byref(pose), None, fake, None) == -2
    assert lib.dnr_dn_consistency(fake, fake, 10, C.byref(pose), 3, 20.0, fake, fake, fake, None) == -3
    assert lib.dnr_dn_consistency(fake, fake, 0, C.byref(pose), 0, 20.0, fake, fake, fake, None) == -2
    assert lib.dnr_dn_consistency(fake, None, 10, C.byref(pose), 0, 20.0, fake, fake, fake, None) == -1


def test_max_bytes(lib):
    need = DN.required_bytes(1920 * 1440)
    assert need < DN.DEFAULT_MAX_BYTES
    DN.check_budget(1920 * 1440, need)
    with pytest.raises(ValueError, match="max_bytes"):
        DN.check_budget(1920 * 1440, need - 1)
