"""oracle/mesh_ref.py, the TSDF rule tests/test_gpu_mesh_kernels.py holds `dnr_tsdf_integrate` to.

  * its fp64 rule equals a scalar loop over the voxels, one Python float operation at a time, on random scenes;
  * the fixed-point colour round trips through the voxel layout and rounds half up;
  * the correct fp32 restatement passes the GPU test's fp64 acceptance rules on that test's own cases;
  * each kernel mistake the oracle can restate (mesh_ref.SLIPS, and the fp16 colour of the voxel layout before the fixed
    point) leaves those rules on those cases by at least 10x: a bound used 10 times over, a weight, update decision or
    pixel that differs outside the band, or a decision placement whose voxel changes by 10x the per-view tsdf bound.
"""
import math

import numpy as np
import pytest

from oracle import mesh_ref as R
from tests import test_gpu_mesh_kernels as T


def scalar_integrate(tsdf, weight, color, g, v):
    """One view, one voxel at a time, in Python floats: Open3D's legacy integration rule as DESIGN.md §2 (5) states it."""
    X, Y, Z = g["dims"]
    H, W = v["depth"].shape
    fx, fy, cx, cy = (float(c) for c in v["cam"][:4])
    E = [float(e) for e in v["cam"][4:]]
    o, vx, tr = [float(a) for a in g["origin"]], float(g["voxel"]), float(g["sdf_trunc"])
    dtr = float(np.float32(v["depth_trunc"]))
    for i in range(X):
        for j in range(Y):
            for k in range(Z):
                p = [o[0] + (i + 0.5) * vx, o[1] + (j + 0.5) * vx, o[2] + (k + 0.5) * vx]
                cam = [E[4 * r] * p[0] + E[4 * r + 1] * p[1] + E[4 * r + 2] * p[2] + E[4 * r + 3] for r in range(3)]
                z = cam[2]
                if not z > 0:
                    continue
                uf = fx * cam[0] / z + cx + 0.5
                vf = fy * cam[1] / z + cy + 0.5
                if not (uf >= 1e-4 and uf < W - 1e-4 and vf >= 1e-4 and vf < H - 1e-4):
                    continue
                u, w_ = int(uf), int(vf)
                d = float(v["depth"][w_, u])
                if (v["mask"] is not None and v["mask"][w_, u] == 0) or d > dtr or d < 0:
                    d = 0.0
                if not d > 0:
                    continue
                a, b = (u - cx) / fx, (w_ - cy) / fy
                sdf = (d - z) * math.sqrt(1 + a * a + b * b)
                if not sdf > -tr:
                    continue
                t = min(1.0, sdf / tr)
                c = []
                for ch in range(3):
                    x = float(v["rgb"][w_, u, ch]) * 255
                    c.append(0 if math.isnan(x) else int(min(max(x, 0.0), 255.0)))
                wt = weight[i, j, k]
                tsdf[i, j, k] = (tsdf[i, j, k] * wt + t) / (wt + 1)
                for ch in range(3):
                    color[i, j, k, ch] = (color[i, j, k, ch] * wt + c[ch]) / (wt + 1)
                weight[i, j, k] = wt + 1


@pytest.mark.parametrize("seed", range(2))
def test_fp64_rule_equals_a_scalar_loop(seed):
    g, views = T.scene_views(seed, n_views=4, dims=(9, 11, 7))
    want = R.empty_volume(g["dims"], np.float64)
    got = R.empty_volume(g["dims"], np.float64)
    for v in views:
        scalar_integrate(*want, g, v)
        R.integrate(*got, g["origin"], g["voxel"], g["sdf_trunc"], v["depth"], v["rgb"], v["mask"], v["cam"], v["depth_trunc"],
                    dtype=np.float64)
    assert want[1].max() >= 3 and (want[1] == 0).any()
    for a, b in zip(got, want):
        assert np.array_equal(a, b)


def test_fixed_point_colour_layout_and_rounding():
    rng = np.random.default_rng(0)
    col = (rng.integers(0, 255 << R.COLOR_FRAC_BITS, (1000, 3), endpoint=True) * 2.0 ** -R.COLOR_FRAC_BITS).astype(np.float32)
    t, w = rng.normal(size=1000).astype(np.float32), rng.integers(0, 9, 1000).astype(np.float32)
    t2, w2, c2 = R.unpack_voxels(R.pack_voxels(t, w, col))
    assert np.array_equal(t2, t) and np.array_equal(w2, w) and np.array_equal(c2, col)
    # one voxel, weight 1, colour 1 level + 1 unit, fused with colour 0: the mean (2^13 + 1) / 2 units ends in a half, up
    g = T.grid((1, 1, 1), (-1 / 32, -1 / 32, 1.0), 1 / 16, 0.25)
    v = T.view(T._cam(), np.full((12, 16), 1.25, np.float32), np.zeros((12, 16, 3), np.float32))
    tsdf, wt, c = R.empty_volume(g["dims"])
    wt[...] = 1
    c[...] = 1 + 2.0 ** -R.COLOR_FRAC_BITS
    R.integrate(tsdf, wt, c, g["origin"], g["voxel"], g["sdf_trunc"], v["depth"], v["rgb"], v["mask"], v["cam"], v["depth_trunc"])
    assert wt[0, 0, 0] == 2 and (c == 0.5 + 2.0 ** -R.COLOR_FRAC_BITS).all()


def test_placements_straddle_their_decisions():
    for name, (cases, target, outcome, flip, hit) in T._placements().items():
        assert len(cases) == 6 and (hit or name.endswith("1e-4")), name


# ----------------------------------------------------------------------------------------------------- slips
@pytest.mark.parametrize("seed", range(3))
def test_the_correct_result_passes_the_scene_rule(seed):
    g, views = T.scene_views(seed)
    fails, worst, band, n = T.check_scene(T.oracle_runner(), g, views)
    assert not fails and band < 0.01 and n > 2000, (fails, worst, band, n)
    assert max(worst.values()) <= 0.5  # fp32 itself uses at most half of each bound


@pytest.mark.parametrize("n", [1000, 5000])
def test_the_correct_result_passes_the_long_sequence_rule(n):
    fails, worst = T.check_long(T.oracle_runner(), n)
    assert not fails and worst["colour"] <= 0.5, worst


@pytest.mark.parametrize("n", [1000, 5000])
def test_fp16_colour_fails_the_long_sequence_rule(n):
    fails, worst = T.check_long(T.oracle_runner(color_dtype=np.float16), n)
    assert fails and worst["colour"] >= 10 * 100, worst  # tens of levels off: the mean stops following the views


@pytest.mark.parametrize("slip", ["round_uf", "ray_from_uf", "round_color"])
def test_slip_leaves_the_scene_rule(slip):
    g, views = T.scene_views(0)
    fails, worst, _, _ = T.check_scene(T.oracle_runner(slip), g, views)
    assert fails and max(worst.values()) >= 10, (slip, worst)


@pytest.mark.parametrize("slip,name", [("sdf_ge", "sdf_gt_-trunc"), ("depth_trunc_ge", "d_le_depth_trunc")])
def test_slip_leaves_the_decision_placement(slip, name):
    """The GPU test asserts bit equality at each placement; the slip changes the target voxel's weight, and its tsdf by
    more than 10x the per-view bound."""
    cases, target, _, _, _ = T._placements()[name]
    changed = 0
    for g, v in cases:
        ok_t, ok_w, _ = T.oracle_runner()(g, [v])
        bad_t, bad_w, _ = T.oracle_runner(slip)(g, [v])
        _, _, _, _, err_t = T._bounds(g, v)
        lin = np.ravel_multi_index(target, g["dims"])
        if ok_w[lin] != bad_w[lin]:
            changed += 1
            assert abs(float(ok_t[lin]) - float(bad_t[lin])) >= 10 * float(np.nanmax(err_t))
    assert changed == 1  # exactly the placement on the threshold


def test_slips_are_named():
    assert set(R.SLIPS) == {"round_uf", "sdf_ge", "depth_trunc_ge", "ray_from_uf", "round_color"}
