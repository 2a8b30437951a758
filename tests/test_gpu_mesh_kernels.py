"""TSDF fusion (`dnr_tsdf_integrate`) per voxel and marching cubes (`dnr_mc_count` / `dnr_mc_emit`) per vertex, against
oracle/mesh_ref.py: bit for bit against its fp32 restatement where a voxel sits on a decision of the integration rule, and
against its fp64 rule on random scenes, long view sequences and fields with ties, plateaus, invalid corners and the
largest dimensions.

The case builders and acceptance rules below need no GPU: tests/test_mesh_ref_cpu.py runs them on the oracle, to show
that the correct fp32 result passes them and that each restated kernel mistake (mesh_ref.SLIPS, fp16 colour) fails them.

Bounds (fp32 unit roundoff EPS = 2^-24):
  * one view's t = min(1, sdf / sdf_trunc): BOUND_T_FACTOR times twice the first-order error of z, the ray multiplier
    and the division (`_bounds`);
  * a fused tsdf: the largest per-view bound plus 2 EPS per fused view (each running-mean update rounds three times);
  * colour: COLOR_TOL = 0.01 level of the exact mean;
  * a marching-cubes vertex: `vertex_bound`, twice the error of t = (iso - f0) / (f1 - f0) and of
    origin + spacing * (p + t); a vertex colour: 1e-6.
A voxel whose fp64 margin to a decision of one view is below that decision's fp32 error (`band`) may take either side.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import mesh_ref as R

F32 = np.float32
EPS = 2.0 ** -24
COLOR_TOL = 0.01
BOUND_T_FACTOR = 2.0
WORST = {}  # bound name -> largest fraction used, printed by the last test


def _used(name, frac):
    WORST[name] = max(WORST.get(name, 0.0), float(frac))


# ------------------------------------------------------------------------------------------------- runners
def grid(dims, origin, voxel, sdf_trunc):
    return dict(dims=tuple(int(d) for d in dims), origin=np.asarray(origin, F32), voxel=F32(voxel), sdf_trunc=F32(sdf_trunc))


def view(cam, depth, rgb, mask=None, depth_trunc=20.0):
    return dict(cam=np.asarray(cam, F32), depth=np.ascontiguousarray(depth, F32), rgb=np.ascontiguousarray(rgb, F32),
                mask=None if mask is None else np.ascontiguousarray(mask, np.uint8), depth_trunc=float(F32(depth_trunc)))


def oracle_runner(slip=None, color_dtype=None):
    """fuse(g, views, state=None) -> (tsdf, weight, colour levels) flattened, by the fp32 restatement with `slip`."""
    def fuse(g, views, state=None):
        tsdf, w, col = R.empty_volume(g["dims"], np.float32, color_dtype)
        if state is not None:
            t0, w0, c0 = R.unpack_voxels(state)
            tsdf[...], w[...], col[...] = t0.reshape(tsdf.shape), w0.reshape(w.shape), c0.reshape(col.shape)
        for v in views:
            R.integrate(tsdf, w, col, g["origin"], g["voxel"], g["sdf_trunc"], v["depth"], v["rgb"], v["mask"], v["cam"],
                        v["depth_trunc"], slip=slip)
        return tsdf.reshape(-1), w.reshape(-1), R.color_levels(col).reshape(-1, 3)
    return fuse


def gpu_voxels(g, views, state=None):
    """The kernel's [N,4] voxels after fusing `views` in order into `state` (zeros when None)."""
    from dn_splatter_b200 import _lib as L
    from dn_splatter_b200.sugar import _stream

    lib = L.load()
    n = int(np.prod(g["dims"]))
    q = torch.zeros((n, 4), dtype=torch.float32, device="cuda") if state is None else torch.from_numpy(state.copy()).cuda()
    s = L.DnrTsdfGrid()
    for a in range(3):
        s.origin[a], s.dims[a] = float(g["origin"][a]), g["dims"][a]
    s.voxel, s.sdf_trunc, s.voxels = float(g["voxel"]), float(g["sdf_trunc"]), q.data_ptr()
    keep = []
    for v in views:
        H, W = v["depth"].shape
        d, c = torch.from_numpy(v["depth"]).cuda(), torch.from_numpy(v["rgb"]).cuda()
        m = None if v["mask"] is None else torch.from_numpy(v["mask"]).cuda()
        keep.append((d, c, m))
        L.check(lib.dnr_tsdf_integrate(C.byref(s), d.data_ptr(), c.data_ptr(), None if m is None else m.data_ptr(), W, H,
                                       (C.c_float * 16)(*v["cam"].tolist()), v["depth_trunc"], _stream()), "dnr_tsdf_integrate")
    return q.cpu().numpy()


def gpu_runner(g, views, state=None):
    tsdf, w, col = R.unpack_voxels(gpu_voxels(g, views, state))
    return tsdf, w, R.color_levels(col)


def pixel_rgb(H, W, blue=0.5):
    """rgb whose truncated uint8 colour is (u, v, .): a voxel fused once from empty carries the pixel it read."""
    u, v = np.meshgrid(np.arange(W), np.arange(H))
    return np.stack([(u + 0.5) / 255, (v + 0.5) / 255, np.full(u.shape, blue)], -1).astype(F32)


# ------------------------------------------------------------------------------------- decisions, bit for bit
AXIS_CAM = [64.0, 64.0, 0.0, 0.0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0]  # world = camera frame: z, x / z exact
BASE_GRID = grid((4, 4, 4), (-0.125, -0.125, 1.0), 1 / 16, 0.25)  # centres +-1/32, +-3/32; z 1 + 1/32 .. 1 + 7/32
TARGET = (1, 2, 1)  # x = -1/32, y = 1/32, z = 1 + 3/32


def _placement(make, knob0, qty, thr, span=64):
    """The knob (knob0 stepped by fp32 ulps) at which the fp32 quantity qty(make(knob)) first reaches thr, the three
    knobs below it and the two above.  Returns (knobs, hit): hit when the quantity equals thr exactly there."""
    knobs = [F32(knob0)]
    for _ in range(span):
        knobs.insert(0, np.nextafter(knobs[0], F32(-np.inf), dtype=F32))
        knobs.append(np.nextafter(knobs[-1], F32(np.inf), dtype=F32))
    q = np.array([qty(make(k)) for k in knobs])
    assert (np.diff(q) >= 0).all() and q[0] < thr <= q[-1]
    n = int(np.argmax(q >= thr))
    assert 3 <= n <= len(knobs) - 3
    return knobs[n - 3:n + 3], bool(q[n] == F32(thr))


def _at(name, g, v, target):
    return R.project(g["dims"], g["origin"], g["voxel"], g["sdf_trunc"], v["depth"], v["rgb"], v["mask"], v["cam"],
                     v["depth_trunc"])[name][target]


def _cam(cx=8.0, cy=6.0, tz=0.0):
    c = list(AXIS_CAM)
    c[2], c[3], c[15] = cx, cy, tz
    return c


def placements():
    """name -> (six (grid, view) cases, target voxel, outcome name, flip, exact hit).  The six straddle one decision at the
    target voxel: its outcome (branch, pixel u / v, or whether t is clamped to 1) takes one value on cases [:flip] and
    another on [flip:].  The
    threshold is at case 3; a strict comparison (z > 0, d <= trunc, sdf > -trunc) flips one case later."""
    W, H = 16, 12
    rgb = pixel_rgb(H, W)
    depth = np.full((H, W), 1.25, F32)
    out = {}

    def add(name, make, knob0, qty, thr, outcome, flip, exact, target=TARGET):
        qf = qty if callable(qty) else (lambda gv: _at(qty, *gv, target))
        knobs, hit = _placement(make, knob0, qf, thr)
        assert hit or not exact, name
        out[name] = ([make(k) for k in knobs], target, outcome, flip, hit)

    s_u = F32(F32(64 * -1 / 32) / F32(1 + 3 / 32))  # fx x / z at TARGET, exact inputs
    s_v = F32(F32(64 * 1 / 32) / F32(1 + 3 / 32))
    mk_u = lambda cx: (BASE_GRID, view(_cam(cx=cx), depth, rgb))  # noqa: E731
    mk_v = lambda cy: (BASE_GRID, view(_cam(cy=cy), depth, rgb))  # noqa: E731
    # 1e-4f is not a multiple of the ulp of uf = B + 0.5 with B ~ -0.5: no placement is on it, six straddle it
    add("u_ge_1e-4", mk_u, F32(1e-4) - 0.5 - s_u, "uf", F32(1e-4), "branch", 3, False)
    # for W - 1e-4f, cx must lie in uf's binade [8, 16) to reach every uf there: the voxel at x = +1/32
    add("u_lt_W-1e-4", mk_u, F32(W - 1e-4) - 0.5 + s_u, "uf", F32(W) - F32(1e-4), "branch", 3, True, (2, 2, 1))
    add("u_integer", mk_u, F32(5.0) - 0.5 - s_u, "uf", F32(5.0), "u", 3, True)
    add("v_ge_1e-4", mk_v, F32(1e-4) - 0.5 - s_v, "vf", F32(1e-4), "branch", 3, False)
    add("v_lt_H-1e-4", mk_v, F32(H - 1e-4) - 0.5 - s_v, "vf", F32(H) - F32(1e-4), "branch", 3, True)
    add("v_integer", mk_v, F32(7.0) - 0.5 - s_v, "vf", F32(7.0), "v", 3, True)
    add("z_gt_0", lambda tz: (BASE_GRID, view(_cam(tz=tz), depth, rgb)), -F32(1 + 3 / 32), "z", F32(0), "branch", 4, True)
    add("d_le_depth_trunc", lambda d: (BASE_GRID, view(_cam(), np.full((H, W), d, F32), rgb, depth_trunc=1.25)),
        F32(1.25), lambda gv: gv[1]["depth"][0, 0], F32(1.25), "branch", 4, True)
    # the principal point: the voxel at x = y = 0 reads pixel (cx, cy) = (8, 6) and its ray multiplier is exactly 1
    pp = grid((4, 4, 4), (-0.09375, -0.09375, 1.0), 1 / 16, 0.25)

    def mk_d(d):
        dm = depth.copy()
        dm[6, 8] = d
        return pp, view(_cam(), dm, rgb)

    z_pp = F32(1 + 3 / 32)
    add("sdf_gt_-trunc", mk_d, z_pp - F32(0.25), "sdf", F32(-0.25), "branch", 4, True, (1, 1, 1))
    add("sdf_eq_+trunc", mk_d, z_pp + F32(0.25), "sdf", F32(0.25), "t", 3, True, (1, 1, 1))
    return out


PLACEMENTS = None


def _placements():
    global PLACEMENTS
    if PLACEMENTS is None:
        PLACEMENTS = placements()
    return PLACEMENTS


def special_depth_cases():
    """Depth values at the pixels: 0, -0, the smallest subnormals, negative, NaN, +-inf, and a zero mask byte."""
    W, H = 16, 12
    rgb = pixel_rgb(H, W)
    out = []
    for d in (0.0, -0.0, 1.4e-45, -1.4e-45, -1.0, np.nan, np.inf, -np.inf, 1.25):
        out.append((BASE_GRID, view(_cam(), np.full((H, W), d, F32), rgb)))
    for m in (0, 1, 255):
        out.append((BASE_GRID, view(_cam(), np.full((H, W), 1.25, F32), rgb, np.full((H, W), m, np.uint8))))
    return out


def color_values():
    """rgb channel values: k / 255 for every k (fp32), their neighbours, negative, above 1, NaN and +-inf."""
    k = np.arange(256)
    vals = (k / 255).astype(F32)
    extra = np.array([-0.1, -0.0, 1.0 + 2 ** -23, 1.5, np.nan, np.inf, -np.inf], F32)
    return np.concatenate([vals, np.nextafter(vals, F32(2)), np.nextafter(vals, F32(-1)), extra])


def color_cases():
    """One view per triple of color_values() over a 2x2x2 grid all of whose voxels read pixels of that colour."""
    vals = color_values()
    g = grid((2, 2, 2), (-1 / 16, -1 / 16, 1.0), 1 / 16, 0.25)
    out = []
    for n in range(0, vals.shape[0], 3):
        trip = np.resize(vals[n:n + 3], 3)
        out.append((g, view(_cam(), np.full((12, 16), 1.25, F32), np.broadcast_to(trip, (12, 16, 3)))))
    return out


def prior_state(g, seed):
    """Random voxels: tsdf in (-1, 1], integer weights up to 5000 (and 0), fixed-point colours anywhere in 0..255."""
    rng = np.random.default_rng(seed)
    n = int(np.prod(g["dims"]))
    w = rng.integers(0, 5000, n).astype(F32)
    w[::7] = 0
    tsdf = np.where(w > 0, rng.uniform(-1, 1, n), 0).astype(F32)
    col = np.where(w[:, None] > 0, rng.integers(0, 255 << R.COLOR_FRAC_BITS, (n, 3), endpoint=True), 0)
    return R.pack_voxels(tsdf, w, col * 2.0 ** -R.COLOR_FRAC_BITS)


def _assert_bitwise(g, views, state=None):
    got = gpu_voxels(g, views, state)
    tsdf, w, col = R.empty_volume(g["dims"])
    if state is not None:
        t0, w0, c0 = R.unpack_voxels(state)
        tsdf[...], w[...], col[...] = t0.reshape(tsdf.shape), w0.reshape(w.shape), c0.reshape(col.shape)
    for v in views:
        R.integrate(tsdf, w, col, g["origin"], g["voxel"], g["sdf_trunc"], v["depth"], v["rgb"], v["mask"], v["cam"], v["depth_trunc"])
    want = R.pack_voxels(tsdf, w, col)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.argwhere(got.view(np.uint32) != want.view(np.uint32))[:5]
    return got


PLACEMENT_NAMES = ["u_ge_1e-4", "u_lt_W-1e-4", "u_integer", "v_ge_1e-4", "v_lt_H-1e-4", "v_integer", "z_gt_0",
                   "d_le_depth_trunc", "sdf_gt_-trunc", "sdf_eq_+trunc"]


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
@pytest.mark.parametrize("name", PLACEMENT_NAMES)
def test_decision_placements_bit_for_bit(name):
    cases, target, outcome, flip, _ = _placements()[name]
    seen = []
    for g, v in cases:
        got = _assert_bitwise(g, [v])
        r = R.project(g["dims"], g["origin"], g["voxel"], g["sdf_trunc"], v["depth"], v["rgb"], v["mask"], v["cam"], v["depth_trunc"])
        lin = np.ravel_multi_index(target, g["dims"])
        updated = got[lin, 1] > 0
        assert updated == (r["branch"][target] == R.UPDATED)
        if outcome == "branch":
            seen.append(int(r["branch"][target]))
        else:
            assert updated
            _, _, col = R.unpack_voxels(got[lin:lin + 1])
            seen.append({"u": int(col[0, 0]), "v": int(col[0, 1]),
                         "t": bool(got[lin, 0] == 1)}[outcome])
    # the decision is straddled, and it flips exactly where the fp32 comparison does
    assert seen[:flip] == [seen[0]] * flip and seen[flip:] == [seen[-1]] * (6 - flip) and seen[0] != seen[-1], (name, seen)


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_special_depths_and_mask_bit_for_bit():
    want = [R.NO_DEPTH, R.NO_DEPTH, R.TOO_FAR, R.NO_DEPTH, R.NO_DEPTH, R.NO_DEPTH, R.NO_DEPTH, R.NO_DEPTH, R.UPDATED,
            R.NO_DEPTH, R.UPDATED, R.UPDATED]
    for (g, v), br in zip(special_depth_cases(), want):
        got = _assert_bitwise(g, [v])
        r = R.project(g["dims"], g["origin"], g["voxel"], g["sdf_trunc"], v["depth"], v["rgb"], v["mask"], v["cam"], v["depth_trunc"])
        assert r["branch"][TARGET] == br and (got[np.ravel_multi_index(TARGET, g["dims"]), 1] > 0) == (br == R.UPDATED)


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_colour_truncation_bit_for_bit():
    below = 0
    for g, v in color_cases():
        got = _assert_bitwise(g, [v])  # from empty: the colour is c levels exactly
        c = R.unpack_voxels(got)[2]
        trip = v["rgb"][0, 0]
        with np.errstate(invalid="ignore"):
            want = np.clip(np.nan_to_num(trip * F32(255), nan=0.0), 0, 255).astype(np.int64)
        assert (c == want[None]).all()
        with np.errstate(invalid="ignore"):
            p = trip * F32(255)
            below += int(((p < np.round(p)) & (np.round(p) - p < 1e-3)).sum())
    assert below > 0  # some fp32(k / 255) * 255 fall below k and truncate to k - 1


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
@pytest.mark.parametrize("seed", range(3))
def test_update_from_prior_state_bit_for_bit(seed):
    """Running means from random weights and colours, including exact halves of the fixed-point rounding."""
    g, views = scene_views(seed, n_views=2, dims=(15, 16, 17))
    state = prior_state(g, seed)
    got = _assert_bitwise(g, views, state)
    assert (got[:, 1] > state[:, 1]).sum() > 500


# ------------------------------------------------------------------------------------------ random scenes, fp64
def _look_at(pos, target, rng):
    f = target - pos
    f /= np.linalg.norm(f)
    up = rng.normal(size=3)
    r = np.cross(f, up)
    r /= np.linalg.norm(r)
    u = np.cross(r, f)
    c2w = np.eye(4)
    c2w[:3, :4] = np.stack([r, u, -f, pos], axis=1)
    return np.linalg.inv(c2w @ np.diag([1.0, -1.0, -1.0, 1.0]))[:3]


def scene_views(seed, n_views=16, dims=(23, 31, 19)):
    """(grid, views): random cameras around the grid, ragged image sizes, a smooth depth surface with holes, negative,
    NaN, infinite and beyond-depth_trunc pixels, masks on some views, colours a fraction 0.02..0.98 from an integer."""
    rng = np.random.default_rng(1000 + seed)
    vox = 0.05
    ext = np.asarray(dims) * vox
    g = grid(dims, -ext / 2 + rng.uniform(-0.02, 0.02, 3), vox, 0.15)
    views = []
    for n in range(n_views):
        W, H = (int(x) for x in rng.integers(17, 140, 2))
        f = rng.uniform(0.6, 1.6) * W
        cam_pos = rng.normal(size=3)
        cam_pos = cam_pos / np.linalg.norm(cam_pos) * rng.uniform(1.2, 2.5)
        E = _look_at(cam_pos, rng.normal(scale=0.1, size=3), rng)
        cx, cy = W / 2 + rng.uniform(-3, 3), H / 2 + rng.uniform(-3, 3)
        u, v = np.meshgrid(np.arange(W), np.arange(H))
        centre = np.linalg.norm(cam_pos)
        depth = centre - 0.3 + 0.25 * np.sin(u / W * rng.uniform(2, 6) + rng.uniform(0, 6)) * np.cos(v / H * rng.uniform(2, 6))
        depth += rng.normal(scale=0.01, size=depth.shape)
        bad = rng.uniform(size=depth.shape)
        depth[bad < 0.03] = 0
        depth[(bad >= 0.03) & (bad < 0.04)] = -0.5
        depth[(bad >= 0.04) & (bad < 0.045)] = np.nan
        depth[(bad >= 0.045) & (bad < 0.05)] = np.inf
        rgb = ((rng.integers(0, 256, (H, W, 3)) + rng.uniform(0.02, 0.98, (H, W, 3))) / 255).astype(F32)
        mask = (rng.uniform(size=(H, W)) > 0.2).astype(np.uint8) * rng.integers(1, 256) if n % 3 == 1 else None
        trunc = float(F32(centre + rng.uniform(-0.2, 0.4)))
        views.append(view([f, f * rng.uniform(0.9, 1.1), cx, cy, *E.reshape(-1)], depth, rgb, mask, trunc))
    return g, views


def _bounds(g, v):
    """fp64 project of one view, and the fp32 error of z, uf / vf, sdf and t per voxel (first order, times 2)."""
    r = R.project(g["dims"], g["origin"], g["voxel"], g["sdf_trunc"], v["depth"], v["rgb"], v["mask"], v["cam"], v["depth_trunc"],
                  dtype=np.float64)
    cam = v["cam"].astype(np.float64)
    fx, fy, cx, cy, E = cam[0], cam[1], cam[2], cam[3], cam[4:].reshape(3, 4)
    i, j, k = np.meshgrid(*[np.arange(d) for d in g["dims"]], indexing="ij")
    p = [float(g["origin"][a]) + (idx + 0.5) * float(g["voxel"]) for a, idx in enumerate((i, j, k))]
    # a camera coordinate E p + e: p rounded once, three products and three sums
    S = [5 * EPS * (sum(np.abs(E[rr, a] * p[a]) for a in range(3)) + abs(E[rr, 3])) for rr in range(3)]
    z = r["z"]
    err_z = 2 * S[2]
    err = {}
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for name, fq, c0, e_x, q in (("u", fx, cx, S[0], r["uf"]), ("v", fy, cy, S[1], r["vf"])):
            proj = np.abs(q - c0 - 0.5)  # |f x / z|
            err[name] = 2 * (abs(fq) * (e_x + proj / abs(fq) * S[2]) / np.abs(z) + 3 * EPS * proj + EPS * (abs(c0) + np.abs(q)))
        ray = np.sqrt(1 + ((r["u"] - cx) / fx) ** 2 + ((r["v"] - cy) / fy) ** 2)
        err_sdf = 2 * (ray * (S[2] + EPS * np.abs(r["d"] - z)) + 5 * EPS * np.abs(r["sdf"]))
        err_t = BOUND_T_FACTOR * (err_sdf / float(g["sdf_trunc"]) + EPS * np.abs(r["t"]))
    return r, err_z, err, err_sdf, err_t


def _band(g, v, r, err_z, err, err_sdf):
    """Voxels with a decision of this view within its fp32 error in fp64."""
    H, W = v["depth"].shape
    with np.errstate(invalid="ignore"):
        band = np.abs(r["z"]) <= err_z
        front = r["z"] > err_z
        for q, e, n in ((r["uf"], err["u"], W), (r["vf"], err["v"], H)):
            band |= front & ((np.abs(q - 1e-4) <= e) | (np.abs(q - (n - 1e-4)) <= e) | (np.abs(q - np.round(q)) <= e))
        upd = r["branch"] == R.UPDATED
        band |= (upd | (r["branch"] == R.TOO_FAR)) & (np.abs(r["sdf"] + float(g["sdf_trunc"])) <= err_sdf)
        c = np.nan_to_num(v["rgb"].astype(np.float64)[np.maximum(r["v"], 0), np.maximum(r["u"], 0)] * 255)
        band |= upd & (np.abs(c - np.round(c)) <= 1e-3).any(-1)
    return band


def _t_at_pixel(g, v, z, u, w):
    """fp64 t of voxels at camera depth z that read pixel (u, w)."""
    cam = v["cam"].astype(np.float64)
    d = v["depth"].astype(np.float64)[w, u]
    with np.errstate(invalid="ignore"):
        sdf = (d - z) * np.sqrt(1 + ((u - cam[2]) / cam[0]) ** 2 + ((w - cam[3]) / cam[1]) ** 2)
    return np.minimum(1, sdf / float(g["sdf_trunc"]))


def check_scene(fuse, g, views):
    """The acceptance rule against fp64 on one random scene, for a runner fuse(g, views) -> (tsdf, weight, levels).
    Returns (failures, {bound: worst fraction used}, band fraction)."""
    fails, worst = [], {"t": 0.0, "tsdf": 0.0, "colour": 0.0}
    n_band = np.zeros(g["dims"], bool)
    t64, w64, c64 = R.empty_volume(g["dims"], np.float64)
    acc_bound = np.zeros(g["dims"])
    for n, v in enumerate(views):
        r, err_z, err, err_sdf, err_t = _bounds(g, v)
        band = _band(g, v, r, err_z, err, err_sdf)
        n_band |= band
        H, W = v["depth"].shape
        enc = dict(v, rgb=pixel_rgb(H, W))
        tsdf, w, lev = (a.reshape(tuple(g["dims"]) + a.shape[1:]) for a in fuse(g, [enc]))
        upd, want = w > 0, r["branch"] == R.UPDATED
        gu, gv = np.floor(lev[..., 0]).astype(np.int64), np.floor(lev[..., 1]).astype(np.int64)
        out = ~band
        if (upd != want)[out].any():
            fails.append(f"view {n}: {int((upd != want)[out].sum())} update decisions differ outside the band")
        both = out & upd & want
        if ((gu != r["u"]) | (gv != r["v"]))[both].any():
            fails.append(f"view {n}: {int(((gu != r['u']) | (gv != r['v']))[both].sum())} pixels differ outside the band")
        same = both & (gu == r["u"]) & (gv == r["v"])
        frac = np.abs(tsdf - r["t"]) / err_t
        if same.any():
            worst["t"] = max(worst["t"], float(frac[same].max()))
        # in the band: an update must read a pixel within the fp32 error of fp64's projection, and hold fp64's t there
        ib = band & upd
        if ib.any():
            with np.errstate(invalid="ignore"):
                ok = ((gu >= np.floor(r["uf"] - err["u"])) & (gu <= np.floor(r["uf"] + err["u"]))
                      & (gv >= np.floor(r["vf"] - err["v"])) & (gv <= np.floor(r["vf"] + err["v"])))[ib]
            if not ok.all():
                fails.append(f"view {n}: {int((~ok).sum())} voxels in the band read a pixel fp64 does not reach")
            t_alt = _t_at_pixel(g, v, r["z"][ib], gu[ib], gv[ib])
            frac_b = np.abs(tsdf[ib] - t_alt) / err_t[ib]
            if not (frac_b <= 1).all():
                fails.append(f"view {n}: a voxel in the band holds no t of its pixel ({float(np.nanmax(frac_b)):.3g} of the bound)")
        acc_bound = np.maximum(acc_bound, np.where(want, err_t, 0))
        R.integrate(t64, w64, c64, g["origin"], g["voxel"], g["sdf_trunc"], v["depth"], v["rgb"], v["mask"], v["cam"],
                    v["depth_trunc"], dtype=np.float64)
    tsdf, w, lev = (a.reshape(tuple(g["dims"]) + a.shape[1:]) for a in fuse(g, views))
    out = ~n_band
    if (w != w64)[out].any():
        fails.append(f"fused: {int((w != w64)[out].sum())} weights differ outside the band")
    seen = out & (w64 > 0) & (w == w64)
    bound = acc_bound + 2 * EPS * w64
    worst["tsdf"] = float((np.abs(tsdf - t64)[seen] / bound[seen]).max())
    worst["colour"] = float((np.abs(lev - c64).max(-1)[seen] / COLOR_TOL).max())
    if worst["t"] > 1 or worst["tsdf"] > 1 or worst["colour"] > 1:
        fails.append(f"bounds exceeded: {worst}")
    return fails, worst, float(n_band.mean()), int(seen.sum())


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
@pytest.mark.parametrize("seed", range(3))
def test_random_scenes_against_fp64(seed):
    g, views = scene_views(seed)
    fails, worst, band, n = check_scene(gpu_runner, g, views)
    assert not fails, fails
    assert band < 0.01 and n > 2000, (band, n)
    for k, val in worst.items():
        _used(k, val)


# ------------------------------------------------------------------------------------------------ long sequences
LONG_GRID = grid((4, 4, 4), (-0.125, -0.125, 1.0), 1 / 16, 0.25)


def long_colours(n):
    """The integer colour of each view: a ramp 140 -> 200 (r), a step 100 -> 180 halfway (g), seeded noise (b)."""
    k = np.arange(n)
    ramp = np.floor(140 + 60 * k / (n - 1)).astype(np.int64)
    step = np.where(k < n // 2, 100, 180)
    noise = np.random.default_rng(n).integers(0, 256, n)
    return np.stack([ramp, step, noise], 1)


def long_views(n):
    """n views of one camera, each a plane at depth 1.4 + 0.05 sin(0.37 k) painted one constant colour."""
    cols = long_colours(n)
    out = []
    for k in range(n):
        rgb = np.broadcast_to(((cols[k] + 0.5) / 255).astype(F32), (16, 16, 3))
        out.append(view(_cam(cy=8.0), np.full((16, 16), 1.4 + 0.05 * np.sin(0.37 * k), F32), rgb))
    return out


def check_long(fuse, n):
    """(failures, {bound: worst fraction}) of a runner on the n-view sequence: weights exact, colour within COLOR_TOL of
    the closed-form mean, tsdf within the fp32 bound of the fp64 running mean."""
    g, views = LONG_GRID, long_views(n)
    tsdf, w, lev = fuse(g, views)
    t64 = np.zeros(int(np.prod(g["dims"])))
    bound = np.zeros_like(t64)
    for v in views:
        r, err_z, err, err_sdf, err_t = _bounds(g, v)
        assert (r["branch"] == R.UPDATED).all() and not _band(g, v, r, err_z, err, err_sdf).any()
        t64 += r["t"].reshape(-1)
        bound = np.maximum(bound, err_t.reshape(-1))
    t64 /= n
    bound += 2 * EPS * n
    want = long_colours(n).mean(0)
    worst = {"colour": float(np.abs(lev - want[None]).max() / COLOR_TOL), "tsdf": float((np.abs(tsdf - t64) / bound).max())}
    fails = [] if (w == n).all() else [f"weights {np.unique(w)} != {n}"]
    fails += [f"{k}: {x:.3g} of its bound" for k, x in worst.items() if x > 1]
    return fails, worst


def gpu_long_runner(g, views):
    """gpu_runner for many views of one size: all images uploaded once."""
    from dn_splatter_b200 import _lib as L
    from dn_splatter_b200.sugar import _stream

    lib = L.load()
    q = torch.zeros((int(np.prod(g["dims"])), 4), dtype=torch.float32, device="cuda")
    s = L.DnrTsdfGrid()
    for a in range(3):
        s.origin[a], s.dims[a] = float(g["origin"][a]), g["dims"][a]
    s.voxel, s.sdf_trunc, s.voxels = float(g["voxel"]), float(g["sdf_trunc"]), q.data_ptr()
    d = torch.from_numpy(np.stack([v["depth"] for v in views])).cuda()
    c = torch.from_numpy(np.stack([v["rgb"] for v in views])).cuda()
    H, W = views[0]["depth"].shape
    for k, v in enumerate(views):
        L.check(lib.dnr_tsdf_integrate(C.byref(s), d[k].data_ptr(), c[k].data_ptr(), None, W, H,
                                       (C.c_float * 16)(*v["cam"].tolist()), v["depth_trunc"], _stream()), "dnr_tsdf_integrate")
    tsdf, w, col = R.unpack_voxels(q.cpu().numpy())
    return tsdf, w, R.color_levels(col)


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
@pytest.mark.parametrize("n", [1000, 5000])
def test_long_sequences_keep_the_colour_mean(n):
    fails, worst = check_long(gpu_long_runner, n)
    assert not fails, (fails, worst)
    for k, val in worst.items():
        _used(f"long {k}", val)


# ---------------------------------------------------------------------------------------------- marching cubes
def vertex_bound(verts64, origin, spacing):
    """Twice the fp32 error of origin + spacing * (p + t) with t = (iso - f0) / (f1 - f0) (three roundings, |t| <= 1), per
    coordinate of the fp64 vertex."""
    o = np.asarray(origin, np.float64)
    return 2 * EPS * (3 * float(spacing) + 2 * np.abs(verts64 - o) + np.abs(verts64) + np.abs(o))


def _mc_gpu(values=None, valid=None, tsdf_voxels=None, dims=None, iso=0.0, origin=(0.0, 0.0, 0.0), spacing=1.0):
    from dn_splatter_b200 import _lib as L
    from dn_splatter_b200.mesh import _mc

    s = L.DnrMcField()
    keep = []
    if tsdf_voxels is not None:
        s.tsdf = tsdf_voxels.data_ptr()
    else:
        s.values = values.data_ptr()
        dims = values.shape
        if valid is not None:
            keep.append(valid.to(torch.uint8).contiguous())
            s.valid = keep[-1].data_ptr()
    s.dims[0], s.dims[1], s.dims[2] = dims
    s.iso, s.spacing = float(iso), float(spacing)
    s.origin[0], s.origin[1], s.origin[2] = [float(o) for o in origin]
    return _mc(s, "cuda", with_colors=tsdf_voxels is not None)


def check_mc(f, iso, origin, spacing, valid=None, colors=None, tsdf_voxels=None):
    """GPU marching cubes twice (bit-identical), faces equal to the oracle's, vertices and colours within their bounds
    of fp64.  Returns the mesh and the fp64 interpolation parameters."""
    f = np.ascontiguousarray(f, F32)
    if tsdf_voxels is not None:
        run = lambda: _mc_gpu(tsdf_voxels=tsdf_voxels, dims=f.shape, iso=iso, origin=origin, spacing=spacing)  # noqa: E731
    else:
        ft = torch.from_numpy(f).cuda()
        vt = None if valid is None else torch.from_numpy(valid).cuda()
        run = lambda: _mc_gpu(ft, vt, iso=iso, origin=origin, spacing=spacing)  # noqa: E731
    got, again = run(), run()
    assert torch.equal(got.vertices, again.vertices) and torch.equal(got.faces, again.faces)
    if got.colors is not None:
        assert torch.equal(got.colors, again.colors)
    o32 = np.asarray(origin, F32)
    rv, rf, rc = R.marching_cubes(f, iso, o32, F32(spacing), valid=valid, colors=colors, dtype=np.float64)
    assert np.array_equal(got.faces.cpu().numpy().astype(np.int64), rf)
    v = got.vertices.cpu().numpy().astype(np.float64)
    assert v.shape == rv.shape
    if v.shape[0]:
        frac = (np.abs(v - rv) / vertex_bound(rv, o32, F32(spacing))).max()
        assert frac <= 1, frac
        _used("vertex", frac)
        if rc is not None:
            cerr = np.abs(got.colors.cpu().numpy() - rc).max()
            assert cerr <= 1e-6, cerr
            _used("vertex colour", cerr / 1e-6)
    return got, rv, rf


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
@pytest.mark.parametrize("with_valid", [False, True])
def test_marching_cubes_ties_at_iso(with_valid):
    """Samples exactly at iso count as outside: vertices on corners (t = 0 or 1) and zero-area faces."""
    rng = np.random.default_rng(7)
    iso = 0.25
    f = (iso + rng.integers(-1, 2, (9, 11, 13))).astype(F32)
    valid = (rng.uniform(size=f.shape) > 0.05) if with_valid else None
    got, rv, rf = check_mc(f, iso, (-0.5, 0.25, 1.0), 0.125, valid=valid)
    on_corner = (np.abs((rv - np.asarray([-0.5, 0.25, 1.0])) / 0.125 - np.round((rv - np.asarray([-0.5, 0.25, 1.0])) / 0.125)) == 0).all(1)
    tri = rv[rf]
    area = np.linalg.norm(np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]), axis=1)
    assert on_corner.sum() > 50 and (area == 0).sum() > 10 and rf.shape[0] > 500


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_marching_cubes_on_a_fused_tsdf_with_plateaus():
    g, views = scene_views(0)
    q = torch.from_numpy(gpu_voxels(g, views)).cuda()
    tsdf, w, col = R.unpack_voxels(q.cpu().numpy())
    shape = g["dims"]
    assert (tsdf == 1).sum() > 500 and (w == 0).sum() > 50  # the +1 plateau and unobserved voxels
    origin = g["origin"].astype(np.float64) + 0.5 * float(g["voxel"])
    got, _, rf = check_mc(tsdf.reshape(shape), 0.0, origin.astype(F32), g["voxel"], valid=(w > 0).reshape(shape),
                          colors=R.color_levels(col).reshape(shape + (3,)), tsdf_voxels=q)
    assert rf.shape[0] > 500


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_marching_cubes_one_invalid_corner_emits_nothing():
    n = 20
    x = np.linspace(-1, 1, n)
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    f = (np.sqrt(X * X + Y * Y + Z * Z) - 0.6).astype(F32)
    s = 2 / (n - 1)
    _, _, f_all = check_mc(f, 0.0, (-1.0,) * 3, s)
    def cases_around(h):
        out = []
        for c in range(8):
            lo = tuple(x - ((c >> a) & 1) for a, x in enumerate(h))
            out.append(sum(int(f[lo[0] + (k & 1), lo[1] + ((k >> 1) & 1), lo[2] + ((k >> 2) & 1)] < 0) << k for k in range(8)))
        return out

    # a sample next to the surface: the crossed cubes around it lose their triangles, each has one invalid corner
    hole = next((i, 10, 10) for i in range(10, n - 1) if sum(0 < c < 255 for c in cases_around((i, 10, 10))) >= 4)
    valid = np.ones(f.shape, bool)
    valid[hole] = False
    _, _, f_cut = check_mc(f, 0.0, (-1.0,) * 3, s, valid=valid)
    lost = sum(int(R._NTRI[c]) for c in cases_around(hole))
    assert lost > 0
    assert f_all.shape[0] - f_cut.shape[0] == lost


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
@pytest.mark.parametrize("dims", [(2, 17, 19), (13, 2, 11), (9, 7, 2), (2, 2, 2), (1, 5, 6), (5, 1, 6), (5, 6, 1)])
def test_marching_cubes_thin_grids(dims):
    f = np.random.default_rng(sum(dims)).uniform(-1, 1, dims).astype(F32)
    got, _, rf = check_mc(f, 0.0, (0.5, -0.25, 2.0), 0.0625)
    assert (rf.shape[0] > 0) == (min(dims) >= 2)


def checkerboard(dims):
    i, j, k = np.meshgrid(*[np.arange(d) for d in dims], indexing="ij")
    return np.where((i + j + k) % 2 == 0, 1.0, -1.0).astype(F32)


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_marching_cubes_at_max_dim_and_rejects_max_dim_plus_one(axis):
    """MAX_DIM = 65535 samples along one axis of a checkerboard: every cube is active, the widest rows (axis 2) carry
    the largest packed per-row counts.  65536 is rejected before any launch."""
    from dn_splatter_b200 import _lib as L

    dims = [2, 2, 2]
    dims[axis] = 65535
    f = checkerboard(dims)
    got, rv, rf = check_mc(f, 0.0, (0.0, 0.0, 0.0), 1.0 / 1024)
    assert rf.shape[0] >= 65534 * 2
    lib = L.load()
    s = L.DnrMcField()
    s.values = 16
    s.dims[0], s.dims[1], s.dims[2] = dims
    s.spacing = 1.0
    assert lib.dnr_mc_count_workspace_bytes(C.byref(s)) > 0
    s.dims[axis] = 65536
    assert lib.dnr_mc_count_workspace_bytes(C.byref(s)) == -2  # DNR_E_SIZE


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_tsdf_integrate_at_max_dim_and_rejects_max_dim_plus_one(axis):
    dims = [1, 1, 1]
    dims[axis] = 65535
    origin = [-1 / 32, -1 / 32, 1.0]
    origin[axis] = -65535 / 2 / 1024 + (1.0 if axis == 2 else 0.0)
    g = grid(dims, origin, 1 / 1024, 0.25)
    v = view(_cam(cx=32.0, cy=24.0), np.full((48, 64), 1.2, F32), pixel_rgb(48, 64))
    v["cam"][0] = v["cam"][1] = 16.0
    got = _assert_bitwise(g, [v])
    assert (got[:, 1] > 0).sum() > 100
    from dn_splatter_b200 import _lib as L
    from dn_splatter_b200.sugar import _stream

    s = L.DnrTsdfGrid()
    s.dims[0], s.dims[1], s.dims[2] = dims
    s.dims[axis] = 65536
    s.voxel, s.sdf_trunc, s.voxels = 1 / 1024, 0.25, 16
    one = C.c_void_p(16)
    assert L.load().dnr_tsdf_integrate(C.byref(s), one, one, None, 64, 48, (C.c_float * 16)(*_cam()), 1.0, _stream()) == -2


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_zz_report_worst_fraction_of_each_bound():
    """Prints the largest fraction of each bound the tests before this one used (pytest -s shows it)."""
    print("\nworst fraction of each bound used:", {k: round(v, 4) for k, v in sorted(WORST.items())})
