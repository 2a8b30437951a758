"""oracle/raster_ref.py, the fp64 per-pixel compositor that tests/test_gpu_raster_forward.py holds `raster_fwd_kernel` to.

  * it equals oracle/gsplat_ref.rasterize_tiles (pinned to the reference project by the goldens) in fp64 on the three
    parity scenes: images, last_ids, the normal pass with its white background, the depth fill value;
  * a scalar loop over one pixel agrees on constructed lists (stop at the second / last entry, everything skipped, sigma < 0
    from an indefinite conic);
  * an alpha one fp64 step either side of each threshold gives the expected margin and the expected alternative;
  * supertile lists with the tile box give what per-tile lists give;
  * each kernel mistake that can be restated in fp64 (raster_ref.SLIPS) leaves the GPU test's acceptance rule on that
    test's own cases, by the factor stated here.  One of them cannot: D / (alpha + 1e-10) differs from
    D / max(alpha, 1e-10) by at most 2.6e-8 relative on any composited pixel (alpha >= 1/255) and not at all on an
    uncovered one (0 / 1e-10), which is below fp32 resolution.
"""
import math

import numpy as np
import pytest
import torch

from oracle import dn_ref
from oracle import gsplat_ref as G
from oracle import raster_ref as R
from tests import test_gpu_raster_forward as T
from tests.helpers import oracle_outputs, scene_and_camera
from tests.test_gpu_parity import CASES

F64 = torch.float64


@pytest.mark.parametrize("case", CASES, ids=["1000@128x128", "3000@200x136", "400@75x53"])
def test_equals_gsplat_ref_on_the_parity_scenes(case):
    params, cam = scene_and_camera(**case)
    p, out = oracle_outputs(params, cam, dtype=F64, predict_normals=True)
    info = out["info"]
    _, ncam = dn_ref.gaussian_normals(p["quats"], p["scales"], p["means"], cam["c2w"].double())
    W, H = cam["width"], cam["height"]
    offs = torch.cat([info["isect_offsets"], torch.tensor([info["flatten_ids"].shape[0]], dtype=torch.int32)])
    ref = R.composite(info["means2d"], info["conics"], info["opacities"], info["colors"], info["depths"], ncam, info["radii"],
                      info["flatten_ids"], offs, 0, W, H, out["background"])
    # gsplat_ref compares with the fp64 constants 1/255, 0.999, 1e-4, this oracle with the kernel's fp32 ones: pixels with a
    # decision between the two are not comparable
    far = ref.margin > 1e-6
    assert far.mean() > 0.999
    close = lambda a, b, tol=1e-12: np.abs(a - b.detach().numpy())[far].max() <= tol  # noqa: E731
    assert close(ref.rgb, out["rgb"]) and close(ref.alpha, out["accumulation"][..., 0])
    assert np.array_equal(ref.last_ids[far], info["last_ids"].numpy().astype(np.int64)[far])
    assert close(ref.normal, out["normal"])
    covered = far & (ref.alpha > 0)
    assert np.abs(ref.depth - out["depth"][..., 0].detach().numpy())[covered].max() <= 1e-11
    fill = out["depth"][..., 0].detach().numpy()[ref.alpha == 0]
    assert abs(float(out["depth"].max()) - ref.depth_max) <= 1e-11 and (fill.size == 0 or np.abs(fill - ref.depth_max).max() <= 1e-11)


def scalar_pixel(px, py, entries, bg, amin=R.ALPHA_MIN, amax=R.ALPHA_MAX, tstop=R.T_STOP):
    """One pixel, one entry at a time: entries = [(mx, my, A, B, C, op, feats[7])]."""
    T, acc, last = 1.0, [0.0] * 7, 0
    for k, (mx, my, A, B, Cc, op, f) in enumerate(entries):
        dx, dy = mx - px, my - py
        sigma = 0.5 * (A * dx * dx + Cc * dy * dy) + B * dx * dy
        alpha = min(op * math.exp(-sigma), amax)
        if sigma < 0 or alpha < amin:
            continue
        if T * (1 - alpha) <= tstop:
            break
        acc = [a + f_ * alpha * T for a, f_ in zip(acc, f)]
        T, last = T * (1 - alpha), k
    n = [a + T for a in acc[4:7]]
    nn = math.sqrt(sum(v * v for v in n))
    return dict(rgb=[min(max(acc[k] + T * bg[k], 0.0), 1.0) for k in range(3)], alpha=1 - T, depth=acc[3] / max(1 - T, 1e-10),
                normal=[(v / nn + 1) / 2 for v in n], last=last)


def _one_tile(entries, bg=(0.2, 0.4, 0.9), radius=40, **kw):
    n = len(entries)
    t = lambda i: torch.tensor([[e[j] for j in i] for e in entries], dtype=F64)  # noqa: E731
    feats = torch.tensor([e[6] for e in entries], dtype=F64)
    return R.composite(t((0, 1)), t((2, 3, 4)), t((5,)).reshape(-1), feats[:, 0:3], feats[:, 3], feats[:, 4:7],
                       torch.full((n,), radius, dtype=torch.int32), torch.arange(n, dtype=torch.int32),
                       torch.tensor([0, n], dtype=torch.int32), 0, 16, 16, bg, **kw)


LISTS = {
    # the earliest possible stop: alpha <= 0.999 leaves T >= 1e-3 after one entry, so no pixel can stop at its first
    "stop_at_second": [(8.5, 8.5, 1e-6, 0.0, 1e-6, 0.99995, None)] + [(6.0, 7.0, 1e-6, 0.0, 1e-6, 0.95, None)] * 3,
    "stop_at_last": [(6.0, 7.0, 1e-3, 0.0, 1e-3, 0.9, None)] * 4 + [(8.0, 8.0, 1e-4, 0.0, 1e-4, 0.9999, None)],
    "all_skipped": [(40.0, 40.0, 0.5, 0.0, 0.5, 0.9, None), (8.0, 8.0, 0.1, 0.0, 0.1, 0.0039, None), (3.0, 3.0, 0.2, 0.0, 0.2, 0.0, None)],
    "indefinite": [(8.2, 7.9, 0.05, 0.2, 0.05, 0.8, None), (5.0, 9.0, 0.02, 0.01, 0.03, 0.4, None)],
    "generic": [(3.0 + 0.7 * k, 12.0 - 0.6 * k, 0.02 + 0.003 * k, 0.004 * (k % 3 - 1), 0.03, 0.1 + 0.05 * (k % 7), None) for k in range(20)],
}


@pytest.mark.parametrize("name", list(LISTS))
def test_scalar_loop_agrees(name):
    g = torch.Generator().manual_seed(7)
    entries = [e[:6] + ((2 * torch.rand(7, generator=g, dtype=F64) - 0.5).tolist(),) for e in LISTS[name]]
    bg = (0.2, 0.4, 0.9)
    ref = _one_tile(entries, bg)
    for i in range(16):
        for j in range(16):
            want = scalar_pixel(j + 0.5, i + 0.5, entries, bg)
            got = np.concatenate([ref.rgb[i, j], [ref.alpha[i, j], ref.depth[i, j]], ref.normal[i, j]])
            exp = np.array(want["rgb"] + [want["alpha"], want["depth"]] + want["normal"])
            assert np.abs(got - exp).max() <= 1e-12 and ref.last_ids[i, j] == want["last"], (name, i, j)
    if name == "stop_at_second":
        assert ref.stopped.all() and (ref.ncomp == 1).all() and (ref.last_ids == 0).all() and ref.clamped.all()
    if name == "stop_at_last":
        assert ref.stopped.all() and (ref.last_ids == 3).all()
    if name == "all_skipped":
        assert ref.ncomp.max() == 0 and not ref.stopped.any()
    if name == "indefinite":
        assert (ref.margin_kind == R.KIND_SIGMA).any() and ((ref.ncomp < 2) & (ref.alpha > 0)).any()


def _feat():
    return [0.3, 0.6, 0.9, 2.0, 0.0, 0.6, 0.8]


@pytest.mark.parametrize("side", [+1, -1])
def test_alpha_threshold_margin_and_alternative(side):
    op = float(np.nextafter(R.ALPHA_MIN, side * math.inf))  # vis = 1 at the pixel centre (8, 8)
    ref = _one_tile([(8.5, 8.5, 3.0, 0.0, 3.0, op, _feat())], eps=1e-9, radius=4)
    assert ref.margin[8, 8] < 1e-15 and ref.margin_kind[8, 8] == R.KIND_ALPHA and ref.margin_pos[8, 8] == 0
    assert ref.ncomp[8, 8] == (1 if side > 0 else 0)
    alts = ref.alts[(8, 8)]
    assert len(alts) == 2 and sorted(int(a["ncomp"]) for a in alts) == [0, 1]
    assert int(alts[0]["ncomp"]) == ref.ncomp[8, 8] and abs(float(alts[side < 0]["alpha"]) - op) < 1e-15
    assert list(ref.alts) == [(8, 8)] and ref.margin[8, 9] > 0.1


@pytest.mark.parametrize("side", [+1, -1])
def test_stop_threshold_margin_and_alternative(side):
    a1 = 0.99
    a2 = 1.0 - R.T_STOP / (1.0 - a1)
    a2 = float(np.nextafter(a2, side * math.inf))  # +: T (1 - a2) just below 1e-4 -> stop
    ents = [(8.5, 8.5, 3.0, 0.0, 3.0, a1, _feat()), (8.5, 8.5, 3.0, 0.0, 3.0, a2, _feat())]
    ref = _one_tile(ents, eps=1e-9, radius=4)
    assert ref.margin_kind[8, 8] == R.KIND_STOP and ref.margin[8, 8] < 1e-12 and ref.margin_pos[8, 8] == 1
    assert bool(ref.stopped[8, 8]) == (side > 0) and ref.last_ids[8, 8] == (0 if side > 0 else 1)
    alts = ref.alts[(8, 8)]
    assert [int(a["last_ids"]) for a in alts] == ([0, 1] if side > 0 else [1, 0])


def test_clamp_margin_is_reported_but_not_ambiguous():
    ref = _one_tile([(8.5, 8.5, 3.0, 0.0, 3.0, float(np.nextafter(R.ALPHA_MAX, 2.0)), _feat())], eps=1e-9, radius=4)
    assert ref.clamp_margin[8, 8] < 1e-15 and ref.clamped[8, 8] and not ref.alts and ref.alpha[8, 8] == R.ALPHA_MAX


def test_too_many_alternatives_are_unresolved():
    op = float(np.nextafter(R.ALPHA_MIN, 1.0))
    ref = _one_tile([(8.5, 8.5, 3.0, 0.0, 3.0, op, _feat())] * 5, eps=1e-6, radius=4, max_alts=8)
    assert ref.unresolved == [(8, 8)] and not ref.alts


@pytest.mark.parametrize("shift", [1, 2, 3])
def test_supertile_lists_with_the_tile_box_equal_per_tile_lists(shift):
    W, H = 81, 49
    f = T.splats(300, W, H, seed=3)
    k = 75
    f["means2d"][:k] = (f["means2d"][:k] / 8).round() * 8
    f["radii"][:k] = (f["radii"][:k] // 8 + 1) * 8
    a, b = T.binned(f, W, H, 0).oracle(eps=0.0), T.binned(f, W, H, shift).oracle(eps=0.0)
    assert a.box_margin == 0.0 and b.n_listed > 1.2 * a.n_listed and a.n_contrib == b.n_contrib
    for k in ("rgb", "alpha", "depth", "normal", "normal_norm", "ncomp", "clamp_mask", "margin"):
        assert np.array_equal(getattr(a, k), getattr(b, k)), k
    # last_ids index each one's own list: the Gaussian they name is the same
    ga = a.last_ids * 0 + T.binned(f, W, H, 0).flatten_ids.numpy()[a.last_ids]
    gb = T.binned(f, W, H, shift).flatten_ids.numpy()[b.last_ids]
    assert np.array_equal(ga[a.ncomp > 0], gb[a.ncomp > 0])


# ----------------------------------------------------------------------------------------------------- slips
def _as_kernel_output(ref):
    f = np.float32
    return dict(rgb=ref.rgb.astype(f), depth=ref.depth.astype(f), alpha=ref.alpha.astype(f), normal=ref.normal.astype(f),
                normal_norm=ref.normal_norm.astype(f), last_ids=ref.last_ids, clamp_mask=ref.clamp_mask)


def _frames_case():
    return T.generic(200, 136, seed=200)  # test_frames[200x136]


def test_the_correct_result_passes_its_own_rule():
    c = _frames_case()
    ref = c.oracle()
    v = R.judge(ref, _as_kernel_output(ref), T.EPS, T.RTOL, T.ATOL)
    assert v.ok and v.worst < 0.1 and v.n_decided > 0.99 * 200 * 136


# slip -> (smallest number of failing pixels, smallest factor by which the worst decided pixel leaves the bound)
EXPECT = {"pretest_slack": (10, 50.0), "stop_after": (50, 1.0), "last_partner": (5000, 0.0), "no_white": (5000, 100.0)}


@pytest.mark.parametrize("slip", list(EXPECT))
def test_slip_leaves_the_acceptance_rule(slip):
    c = _frames_case()
    ref = c.oracle()
    bad = c.oracle(slip=slip, eps=0.0)
    v = R.judge(ref, _as_kernel_output(bad), T.EPS, T.RTOL, T.ATOL)
    n_min, factor = EXPECT[slip]
    assert v.n_fail >= n_min and v.worst >= factor, f"{slip}: {v.n_fail} pixels fail, worst ratio {v.worst:.3g}"


def test_stop_after_fails_every_tile_that_saturates():
    c = T.listed([L for L in T.LENGTHS if L > 128] + [129], seed=2, kind="opaque", stop_at=128)  # test_whole_tile_saturates[128]
    ref = c.oracle()
    bad = c.oracle(slip="stop_after", eps=0.0)
    v = R.judge(ref, _as_kernel_output(bad), T.EPS, T.RTOL, T.ATOL)
    assert v.n_fail >= 0.95 * c.width * c.height


def test_depth_eps_slip_is_below_fp32_resolution():
    c = _frames_case()
    ref, bad = c.oracle(), c.oracle(slip="depth_eps", eps=0.0)
    assert np.abs(bad.depth - ref.depth).max() <= 2.6e-8 * ref.depth.max() and (bad.depth[ref.alpha == 0] == 0).all()
    v = R.judge(ref, _as_kernel_output(bad), T.EPS, T.RTOL, T.ATOL)
    assert v.ok and v.worst < 0.1


def test_stale_depth_max_is_seen():
    """test_depth_max_reset_and_last_tile: the second, shallower frame must report its own maximum."""
    deep = T.generic(81, 49, seed=31)
    shallow = T.generic(81, 49, seed=31)
    shallow.depths = deep.depths * 0.25
    stale = deep.oracle(eps=0.0).depth_max
    ref = shallow.oracle(eps=0.0)
    bad = shallow.oracle(eps=0.0, slip="stale_depth_max", stale_depth_max=stale)
    assert ref.depth_max == float(ref.depth.max()) and bad.depth_max >= 3.9 * ref.depth_max
    assert T.bits(bad.depth_max) != T.bits(float(np.float32(ref.depth).max()))
