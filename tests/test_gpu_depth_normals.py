"""GPU checks of dn_splatter_b200/depth_normals.py against oracle/normals_ref.py: back-projection, the neighbour search
per query (multisets under the tie rule), covariances and normals, the consistency pass, work per query against the hole
share, run-to-run identity, and both scripts end to end on the golden folder."""
import os

import numpy as np
import pytest
import torch

from dn_splatter_b200 import depth_normals as DN
from oracle import normals_ref as R
from tests import depth_normals_scene as D
from tests.test_depth_normals_cpu import RUNS, decoded, golden_files

pytestmark = pytest.mark.gpu
EPS = 2.0 ** -52


@pytest.fixture(scope="module")
def folder(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("dn"))
    D.build(root)
    return root


def test_backproject(folder):
    frames, (fx, fy, cx, cy, w, h) = DN.load_transforms(folder, "transforms.json")
    for f in frames:
        depth = DN.resize_nearest(DN.load_depth(os.path.join(folder, f["depth_file_path"])), w, h)
        c2w = DN.c2w_of(f)
        pts, cam = DN.backproject_depth(depth, fx, fy, cx, cy, c2w, with_camera=True)
        want, want_cam = R.backproject(depth, fx, fy, cx, cy, w, h, c2w)
        np.testing.assert_array_equal(cam.cpu().numpy(), want_cam)
        terms = np.abs(want_cam.astype(np.float64)[:, :, None] * np.linalg.inv(c2w[:3, :3])[None]).sum(1) + np.abs(c2w[:3, 3])
        assert (np.abs(pts.cpu().numpy() - want) <= 2 * EPS * terms).all()


def clouds():
    g = np.random.default_rng(5)
    surf = np.c_[g.uniform(0, 1, (1500, 2)), 0.02 * g.normal(size=1500)]
    out = {"surface": surf}
    for m in (0, 199, 200):
        out[f"centre_dups_{m}"] = np.r_[surf[:800] + [0, 0, 1.0], np.zeros((m, 3))]
    out["centre_dups_1e5"] = np.r_[surf[:600] + [0, 0, 1.0], np.zeros((100000, 3))]
    ii, jj = np.meshgrid(np.arange(40), np.arange(40))
    out["lattice_plane"] = np.c_[ii.ravel() * 0.1, jj.ravel() * 0.1, np.zeros(1600)]
    out["line"] = np.outer(np.arange(500), [0.01, 0.02, -0.005])
    out["single"] = np.array([[1.0, 2.0, 3.0]])
    out["outliers"] = np.r_[surf[:1000], g.uniform(-1e4, 1e4, (5, 3))]
    out["few"] = surf[:150]
    return out


@pytest.mark.parametrize("name", list(clouds()))
@pytest.mark.parametrize("k", [1, 3, 30, 200, 256])
def test_neighbours_covariance_normals(name, k):
    pts = clouds()[name]
    n = len(pts)
    normals, cov, nbr = DN.estimate_normals(torch.from_numpy(pts).cuda(), k, debug=True)
    normals, cov, nbr = normals.cpu().numpy(), cov.cpu().numpy().reshape(-1, 3, 3), nbr.cpu().numpy()
    kk = min(k, n)
    assert (nbr[:, kk:] == -1).all()
    uniq, first, counts, inv = R.unique_positions(pts)
    rows = np.unique(inv, return_index=True)[1]  # one query per distinct position, every one of them
    assert (counts > 1).sum() == (name.startswith("centre_dups_") and not name.endswith("_0"))
    want = R.knn(pts, k, queries=rows)
    scale = np.abs(pts).max() ** 2 + 1e-300
    for r, wn in zip(rows, want):
        got = nbr[r, :kk]
        np.testing.assert_array_equal(np.sort(got), np.sort(wn), err_msg=f"row {r}")
        c = R.covariance(pts, wn)
        bound = 8 * kk * EPS * scale
        assert np.abs(cov[r] - c).max() <= bound, (r, np.abs(cov[r] - c).max(), bound)
        v = R.fast_eigen3x3(c)
        if np.linalg.norm(v) == 0:
            v = np.array([0.0, 0.0, 1.0])
        w = np.linalg.eigvalsh(c)
        gap = w[1] - w[0]
        if gap > 1e-6 * max(w[2], 1e-300) and kk >= 3:
            err = min(np.abs(normals[r] - v).max(), np.abs(normals[r] + v).max())
            assert err <= 1e3 * bound / gap + 1e-9, (r, err, gap)


def test_orientation_and_consistency(folder):
    frames, (fx, fy, cx, cy, w, h) = DN.load_transforms(folder, "transforms.json")
    for mode, thr in (("omnidata", 20.0), ("dsine", 15.0), ("depth_to_normal", 10.0)):
        for f in frames[:3]:
            depth = DN.resize_nearest(DN.load_depth(os.path.join(folder, f["depth_file_path"])), w, h)
            c2w = DN.c2w_of(f)
            pts = DN.backproject_depth(depth, fx, fy, cx, cy, c2w)
            n_gpu = DN.estimate_normals(pts, 200, center=c2w[:3, 3]).cpu().numpy()
            p = pts.cpu().numpy()
            n_ref = R.orient(p, R.estimate_normals(p)[0], c2w[:3, 3])
            ray = p - c2w[:3, 3]
            flip = (n_gpu * n_ref).sum(1)
            band = np.abs((ray * n_ref).sum(1)) <= 1e-9 * np.linalg.norm(ray, axis=1)
            assert ((flip > 0) | band).all()
            mono = DN.read_mono(os.path.join(folder, "normals_from_pretrain", f["file_path"].split("/")[-1].replace("jpg", "png")), w, h)
            enc, deg, mask = DN.depth_normal_consistency(torch.from_numpy(n_ref).cuda(), mono, c2w, mode, thr)
            d_ref, m_ref, e_ref = R.consistency(n_ref, mono, c2w, mode, thr)
            deg = deg.cpu().numpy()
            assert np.abs(deg - d_ref).max() <= 1e-9
            near = np.abs(d_ref - thr) <= 1e-9
            assert ((mask.cpu().numpy() == 255) == m_ref)[~near].all()
            assert (np.abs(enc.cpu().numpy().astype(int) - e_ref.astype(int)) <= 1).all()
            np.testing.assert_array_equal(enc.cpu().numpy()[np.abs(n_ref * 127.5 % 1 - 0.5).min(1) > 1e-6],
                                          e_ref[np.abs(n_ref * 127.5 % 1 - 0.5).min(1) > 1e-6])


def _room_depth(w, h, hole_share, seed=0):
    """A 0.3-8 m room frame (ramp of planes) with hole_share of the pixels zeroed in blobs."""
    g = np.random.default_rng(seed)
    u, v = np.meshgrid(np.arange(w), np.arange(h))
    z = 0.3 + 7.7 * (u / w) ** 2 + 0.3 * np.sin(v / h * 6)
    holes = np.zeros((h, w), bool)
    while holes.mean() < hole_share:
        cx, cy, r = g.integers(0, w), g.integers(0, h), g.integers(4, 30)
        holes |= (u - cx) ** 2 + (v - cy) ** 2 < r * r
    return np.where(holes, 0, z).astype(np.float32)


def test_work_per_query_independent_of_holes_and_rerun_identical():
    w, h = 320, 240
    intr = (250.0, 250.0, w / 2, h / 2)
    per_query = []
    for share in (0.01, 0.4):
        stats = torch.zeros(2, dtype=torch.int64, device="cuda")
        depth = _room_depth(w, h, share)
        a = DN.estimate_normals(depth, 200, intrinsics=intr, c2w=np.eye(4), stats=stats)
        b = DN.estimate_normals(depth, 200, intrinsics=intr, c2w=np.eye(4))
        assert torch.equal(a, b)
        s = stats.cpu().numpy()
        per_query.append(s[0] / s[1])
    assert max(per_query) <= 2 * min(per_query), per_query


def test_mask_is_strict(folder):
    """mask = 255 where the angle exceeds the threshold, never where it equals it (the golden's omnidata_tie run pins the
    oracle; here the kernel is run at thresholds equal to its own angles)."""
    frames, (fx, fy, cx, cy, w, h) = DN.load_transforms(folder, "transforms.json")
    f = frames[0]
    depth = DN.load_depth(os.path.join(folder, f["depth_file_path"]))
    c2w = DN.c2w_of(f)
    normals = DN.estimate_normals(depth, 200, intrinsics=(fx, fy, cx, cy), c2w=c2w)
    mono = DN.read_mono(os.path.join(folder, "normals_from_pretrain", "frame_1.png"), w, h)
    for mode in ("omnidata", "dsine", "depth_to_normal"):
        deg = DN.depth_normal_consistency(normals, mono, c2w, mode, 20.0)[1].cpu().numpy()
        for t in np.quantile(deg, [0.1, 0.5, 0.9], method="nearest"):
            mask = DN.depth_normal_consistency(normals, mono, c2w, mode, float(t))[2].cpu().numpy()
            assert mask[deg == t].max() == 0
            np.testing.assert_array_equal(mask, np.where(deg > t, 255, 0))


@pytest.mark.parametrize("run", [r for r in RUNS if r != "omnidata_tie"])  # ties at the threshold: test_mask_is_strict
def test_scripts_write_the_golden_files(tmp_path, run):
    mode, thr, rename, folder = RUNS[run]
    name = D.build(str(tmp_path), **folder)
    if run == "depth_to_normal":
        DN.DepthToNormal(tmp_path, name).main()
    else:
        DN.DepthNormalConsistency(tmp_path, name, mode, thr).main()
    files = D.list_outputs(str(tmp_path))
    want = golden_files(run)
    assert list(files) == list(want)
    for f, b in want.items():
        if f.endswith(".jpg"):
            assert files[f] == b, f
        else:
            np.testing.assert_array_equal(decoded(files[f]), decoded(b), err_msg=f)


def test_full_size_frame_within_budget():
    w, h = 1920, 1440
    depth = _room_depth(w, h, 0.05)
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    n = DN.estimate_normals(depth, 200, intrinsics=(1400.0, 1400.0, w / 2, h / 2), c2w=np.eye(4))
    torch.cuda.synchronize()
    assert n.shape == (w * h, 3) and torch.isfinite(n).all()
    assert torch.cuda.max_memory_allocated() - base <= DN.required_bytes(w * h) + (1 << 20)
