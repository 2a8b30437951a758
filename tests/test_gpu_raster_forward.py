"""GPU tests of the rasterizer forward (`raster_fwd_kernel`, csrc/raster.cu) per pixel against the fp64 compositor of
oracle/raster_ref.py, which tests/test_raster_ref_cpu.py pins on the CPU.

Two layers.  A: `dnr_raster_fwd` through the C ABI on constructed records and lists (both record layouts), reading every
output: list lengths around the 128-entry chunks, tiles that saturate inside a chunk / at a chunk's edge, pixel pairs of
one lane that disagree, ragged frames, supertile lists with the tile box and the tile-hit filter, the three thresholds hit
exactly in fp32, colours and backgrounds outside [0, 1], `depth_max` and its reset, run-to-run bit identity.  B: through
`dn_rasterize` on scenes, the oracle fed the CUDA side's own per-Gaussian outputs and lists.

How a pixel is judged (raster_ref.judge).  The oracle reports, per pixel, the margin of the closest decision it took.
Pixels with margin >= EPS: every output within sqrt(1 + composited) (RTOL mass + ATOL) of fp64 (mass = sum of w_i |feat_i|,
the absolute composited mass), `last_ids` equal, clamp mask equal unless the pre-clamp value is within the bound of 0 or 1.
No share of the pixels is exempt.  Pixels under EPS must match one of the outcomes the oracle obtains by taking each
near-threshold decision either way.  Each scene asserts that such pixels are few and each constructed case that it
reaches the branch it is named for.

Set DNR_RASTER_REPORT=<file> to append one JSON line per check (worst ratio to the bound, pixel counts): that is how the
constants below are re-measured.
"""
import json
import os

import numpy as np
import pytest
import torch

from oracle import raster_ref as R
from tests.raster_cases import (EPS, F32, TILE, Buffers, Case, binned, bits, generic, listed, pack_records, run_fwd,  # noqa: F401
                                scene, scene_run, splats)

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]

# Bound per output: sqrt(1 + composited) (RTOL mass + ATOL).  Measured on an H100 80GB HBM3 (700 W limit) over the 98 checks
# of this file: the worst decided pixel uses 0.25 of the bound (a clamp-scene pixel 1.7e-2 from sigma = 0; constructed
# cases at most 0.19), 1270 pixels in all sit under the band (at most 1.04 % of a frame), 2 of them match an alternative
# other than the oracle's primary outcome, none has too many alternatives.
RTOL, ATOL = 2e-6, 2.4e-7
MAX_AMBIGUOUS = 0.01  # share of a scene's pixels that may sit under the band (measured: 0.1 % on the scenes)




def check(name, ref: R.RasterRef, got, regions=None, max_ambiguous=MAX_AMBIGUOUS):
    """Judges the whole frame (and every named region on its own); returns the frame's verdict."""
    v = R.judge(ref, got, EPS, RTOL, ATOL)
    path = os.environ.get("DNR_RASTER_REPORT")
    if path:
        with open(path, "a") as fh:
            fh.write(json.dumps(dict(check=name, worst=v.worst, decided=v.n_decided, ambiguous=v.n_ambiguous,
                                     alt_used=v.n_alt_used, unresolved=v.n_unresolved, fail=v.n_fail, what=v.worst_what)) + "\n")
    assert v.ok, f"{name}: {v.n_fail} pixels fail (worst decided ratio {v.worst:.3g}):\n" + "\n".join(v.failures)
    total = int(ref.done.sum())
    assert v.n_ambiguous + v.n_unresolved <= max(3, max_ambiguous * total), \
        f"{name}: {v.n_ambiguous} + {v.n_unresolved} of {total} pixels are under the decision band"
    assert v.n_unresolved <= max(1, 1e-3 * total), f"{name}: {v.n_unresolved} pixels have too many alternatives"
    for rname, mask in (regions or {}).items():
        assert mask.any(), f"{name}: region {rname} is empty"
        vr = R.judge(ref, got, EPS, RTOL, ATOL, region=mask)
        assert vr.ok, f"{name} / {rname}: {vr.n_fail} pixels fail:\n" + "\n".join(vr.failures)
    dm = float(np.max(got["depth"])) if got["depth"].size else 0.0
    assert got["depth_max_bits"] == bits(max(dm, 0.0)), f"{name}: depth_max is not the maximum of out_depth"
    assert abs(dm - ref.depth_max) <= 1e-4 * max(ref.depth_max, 1.0) or v.n_ambiguous > 0, f"{name}: depth_max {dm} vs {ref.depth_max}"
    walked, kept = got["stats"][0], got["stats"][1]
    assert kept <= walked <= ref.n_listed, f"{name}: kept {kept}, walked {walked}, listed {ref.n_listed}"
    if not ref.stopped.any():  # no early exit: every entry some pixel composites must have survived the tile filter
        assert walked == ref.n_listed and kept >= ref.n_contrib, f"{name}: kept {kept} < {ref.n_contrib} contributing entries"
    return v


def last_tile_regions(W, H):
    out = {}
    if H % TILE:
        m = np.zeros((H, W), bool)
        m[H // TILE * TILE:] = True
        out["last_tile_row"] = m
    if W % TILE:
        m = np.zeros((H, W), bool)
        m[:, W // TILE * TILE:] = True
        out["last_tile_col"] = m
    return out


# ----------------------------------------------------------------------------------------------------- A: constructed
LENGTHS = (0, 1, 3, 4, 5, 127, 128, 129, 255, 256, 257, 640, 1100)


@pytest.mark.parametrize("normals", [True, False], ids=["rec16", "rec12"])
def test_list_lengths_faint(normals):
    """Every chunk count up to nine, both mbarrier phases several times, survivor counts of every residue mod 4."""
    c = listed(LENGTHS, seed=1)
    ref = c.oracle(normals)
    assert not ref.stopped.any(), "no pixel may saturate"
    for t, L in enumerate(LENGTHS):  # every list is composited from its first chunk to its last
        sl = (slice(None), slice(t * TILE, (t + 1) * TILE))
        assert int(ref.ncomp[sl].max()) >= min(L, max(3, L // 5)), (L, int(ref.ncomp[sl].max()))
        assert L == 0 or int(ref.last_ids[sl].max()) >= int(c.tile_offsets[t]) + L - 1 - L // 10
    got, _ = run_fwd(c, normals)
    check(f"lengths-{normals}", ref, got)
    for t, L in enumerate(LENGTHS):
        assert got["last_ids"][:, t * TILE:(t + 1) * TILE].max() <= max(int(c.tile_offsets[t]) + L - 1, 0)


STOPS = (5, 127, 128, 129, 200, 255, 256, 383)


@pytest.mark.parametrize("normals", [True, False], ids=["rec16", "rec12"])
@pytest.mark.parametrize("stop_at", STOPS)
def test_whole_tile_saturates(stop_at, normals):
    """Opaque splats take every pixel of the tile to the stop rule at list entry `stop_at` (inside chunk 0, at the last
    entry of a chunk, at the first of the next, ...) while the following chunk's copy is in flight: nothing after it may be
    composited and `last_ids` stay at the entry before it."""
    c = listed([L for L in LENGTHS if L > stop_at] + [stop_at + 1], seed=2, kind="opaque", stop_at=stop_at)
    ref = c.oracle(normals)
    assert ref.stopped.all(), "every pixel must stop"
    got, _ = run_fwd(c, normals)
    check(f"saturate-{stop_at}-{normals}", ref, got)
    for t in range(c.width // TILE):
        sl = (slice(None), slice(t * TILE, (t + 1) * TILE))
        assert (got["last_ids"][sl] == int(c.tile_offsets[t]) + stop_at - 1).all(), "last_ids moved past the stop"
    if stop_at < 128:
        assert got["stats"][0] <= 128 * (c.width // TILE), "a saturated tile fetched more than its first chunk"


@pytest.mark.parametrize("normals", [True, False], ids=["rec16", "rec12"])
@pytest.mark.parametrize("kind,stop_at", [("half", 60), ("half", 128), ("rows", 10), ("rows", 120)])
def test_pixel_pairs_disagree(kind, stop_at, normals):
    """Half of the tile stops and half goes on; and rows r stop while rows r + 4 — the other pixel of the same lane — skip
    the opaque splats and composite the rest of the list."""
    c = listed((300, 640, 257), seed=3, kind=kind, stop_at=stop_at)
    ref = c.oracle(normals)
    if kind == "rows":
        rows = np.arange(TILE)
        upper, lower = (rows % 8) < 4, (rows % 8) >= 4
        assert ref.stopped[upper].all() and not ref.stopped[lower].any(), "rows r must stop and rows r + 4 must not"
        for t in range(c.width // TILE):
            tile = ref.last_ids[:, t * TILE:(t + 1) * TILE]
            assert tile[lower].min() > tile[upper].max()
    else:
        assert ref.stopped[:, :4].all() and not ref.stopped[:, 12:16].any(), "left columns stop, right ones do not"
    got, _ = run_fwd(c, normals)
    # a third of these pixels stop behind four splats of alpha ~0.85: kappa ~ 25 widens the band of the stop test
    check(f"pairs-{kind}-{stop_at}-{normals}", ref, got, max_ambiguous=0.05)


FRAMES = [(1, 1), (13, 7), (16, 16), (17, 17), (81, 49), (75, 53), (200, 136)]


@pytest.mark.parametrize("normals", [True, False], ids=["rec16", "rec12"])
@pytest.mark.parametrize("wh", FRAMES, ids=[f"{w}x{h}" for w, h in FRAMES])
def test_frames(wh, normals):
    """Pixels of a lane's pair outside the frame; the last partial tile row and column judged on their own."""
    W, H = wh
    c = generic(W, H, seed=W)
    ref = c.oracle(normals)
    got, _ = run_fwd(c, normals)
    v = check(f"frame-{W}x{H}-{normals}", ref, got, regions=last_tile_regions(W, H))
    if W * H >= 3000:
        assert ref.stopped.any() and ref.clamped.any() and v.n_decided > 0.98 * W * H


@pytest.mark.parametrize("normals", [True, False], ids=["rec16", "rec12"])
@pytest.mark.parametrize("shift,exact", [(0, False), (0, True), (1, False), (2, False), (3, False)])
@pytest.mark.parametrize("wh", [(81, 49), (200, 136)], ids=["81x49", "200x136"])
def test_supertile_lists(wh, shift, exact, normals):
    """Supertiles cut by the frame edge; splats whose tile box ends exactly on a tile boundary; splats centred in another
    tile of the same supertile.  An entry the oracle composites in a tile must survive the tile-box and tile-hit filters
    there (`check` compares the kept count with the oracle's contributing entries when no tile exits early)."""
    W, H = wh
    f = splats(max(8, W * H // 40), W, H, seed=11, opaque=0.0, faint=0.5)
    k = f["means2d"].shape[0] // 4
    f["means2d"][:k] = (f["means2d"][:k] / 8).round() * 8  # centres on multiples of 8 ...
    f["radii"][:k] = (f["radii"][:k] // 8 + 1) * 8          # ... and radii too: m +- r on tile boundaries
    c = binned(f, W, H, shift)
    ref = c.oracle(normals)
    assert ref.box_margin == 0.0, "no tile box ends on a tile boundary"
    if shift:
        assert ref.n_contrib < 0.8 * ref.n_listed, "the supertile lists must hold entries their tiles do not composite"
    got, _ = run_fwd(c, normals, exact_flag=exact)
    check(f"lists-{W}x{H}-{shift}-{exact}-{normals}", ref, got, regions=last_tile_regions(W, H))


def _at_centres(ops, second=None, W=None):
    """Tile t holds one tiny splat of opacity ops[t] exactly on the centre of its pixel (5, 8) (vis = 2^0 = 1 exactly), and
    after it, if given, one of opacity second[t] at the same place."""
    n = len(ops)
    m = torch.tensor([[t * TILE + 8.5, 5.5] for t in range(n)])
    two = second is not None
    f = dict(means2d=torch.cat([m, m]) if two else m, opac=torch.tensor(list(ops) + (list(second) if two else []), dtype=F32))
    N = f["means2d"].shape[0]
    ids = torch.tensor([[t, n + t] for t in range(n)] if two else [[t] for t in range(n)], dtype=torch.int32).reshape(-1)
    offs = torch.arange(n + 1, dtype=torch.int32) * (2 if two else 1)
    g = torch.Generator().manual_seed(5)
    return Case(conics=torch.tensor([[0.5, 0.1, 0.7]]).repeat(N, 1), colors=torch.rand(N, 3, generator=g), depths=1 + torch.rand(N, generator=g),
                normals_cam=torch.nn.functional.normalize(torch.randn(N, 3, generator=g), dim=1), radii=torch.full((N,), 6, dtype=torch.int32),
                flatten_ids=ids, tile_offsets=offs, list_shift=0, width=TILE * n, height=TILE, **f)


def _steps(x, ks):
    """fp32 x moved by k units in the last place for k in ks."""
    b = np.float32(x).view(np.int32)
    return [float((b + np.int32(k)).view(np.float32)) for k in ks]


KS = (-3, -2, -1, 0, 1, 2, 3)


@pytest.mark.parametrize("normals", [True, False], ids=["rec16", "rec12"])
def test_alpha_threshold_exact(normals):
    """alpha = op exactly at a pixel centre: composited iff op >= fp32(1/255); op = 0 (nthr = +inf) never."""
    amin = np.float32(1.0) / np.float32(255.0)
    ops = _steps(amin, KS) + [0.0]
    c = _at_centres(ops)
    got, _ = run_fwd(c, normals)
    for t, op in enumerate(ops):
        a = got["alpha"][5, t * TILE + 8]
        want = np.float32(1) - (np.float32(1) - np.float32(op)) if np.float32(op) >= amin else np.float32(0)
        assert a == want, f"op = 1/255 {KS[t] if t < len(KS) else 'zero'} ulp: alpha {a} != {want}"
    check(f"alpha-threshold-{normals}", c.oracle(normals), got, max_ambiguous=1.0)


@pytest.mark.parametrize("normals", [True, False], ids=["rec16", "rec12"])
def test_alpha_clamp_exact(normals):
    """op * vis = op around 0.999 at a pixel centre: alpha = min(op, 0.999f), so T = 1 - that, exactly."""
    ops = _steps(0.999, KS)
    c = _at_centres(ops)
    ref = c.oracle(normals)
    assert (ref.clamp_margin < 1e-6).sum() == len(ops)
    got, _ = run_fwd(c, normals)
    for t, op in enumerate(ops):
        a = got["alpha"][5, t * TILE + 8]
        want = np.float32(1) - (np.float32(1) - min(np.float32(op), np.float32(0.999)))
        assert a == want, f"op = 0.999 {KS[t]:+d} ulp: alpha {a} != {want}"
    check(f"alpha-clamp-{normals}", ref, got, max_ambiguous=1.0)


@pytest.mark.parametrize("normals", [True, False], ids=["rec16", "rec12"])
def test_stop_threshold_exact(normals):
    """Two splats on one pixel centre: T = 1 - a1 after the first, and the second is composited iff
    fp32(T * (1 - a2)) > 1e-4f.  a2 is stepped across that point one fp32 value at a time."""
    one = np.float32(1)
    a1 = np.float32(0.99)
    T1 = one - a1
    lo, hi = np.float32(0.98), np.float32(0.995)  # bisect for the smallest a2 that stops
    while np.nextafter(lo, hi) < hi:
        mid = np.float32((np.float64(lo) + np.float64(hi)) / 2)
        if T1 * (one - mid) <= np.float32(1e-4):
            hi = mid
        else:
            lo = mid
    a2s = _steps(hi, KS)
    c = _at_centres([float(a1)] * len(a2s), second=a2s)
    got, _ = run_fwd(c, normals)
    stops = 0
    for t, a2 in enumerate(a2s):
        nT = T1 * (one - np.float32(a2))
        stop = nT <= np.float32(1e-4)
        stops += int(stop)
        want = one - (T1 if stop else nT)
        x = t * TILE + 8
        assert got["alpha"][5, x] == want and got["last_ids"][5, x] == 2 * t + (0 if stop else 1), \
            f"a2 {KS[t]:+d} ulp from the stop point: alpha {got['alpha'][5, x]} last {got['last_ids'][5, x]}, stop expected {stop}"
    assert 0 < stops < len(a2s)
    check(f"stop-threshold-{normals}", c.oracle(normals), got, max_ambiguous=1.0)


@pytest.mark.parametrize("normals", [True, False], ids=["rec16", "rec12"])
@pytest.mark.parametrize("bg", [(1.0, 1.0, 1.0), (0.0, 0.0, 0.0), (-0.2, 0.5, 1.3)])
def test_clamp_mask_and_backgrounds(bg, normals):
    """Colours in [-0.5, 1.5] and backgrounds in and outside [0, 1]: the clamped value and the mask bit per channel."""
    c = generic(75, 53, seed=21, color=(-0.5, 1.5), background=bg)
    ref = c.oracle(normals)
    for k in range(3):
        bit = (ref.clamp_mask >> k) & 1
        assert bit.min() == 0 and bit.max() == 1, f"channel {k}: the mask bit never changes"
    got, _ = run_fwd(c, normals)
    check(f"clamp-{bg}-{normals}", ref, got)


@pytest.mark.parametrize("normals", [True, False], ids=["rec16", "rec12"])
def test_empty_frame(normals):
    """No list at all: rgb = clamp(bg), alpha = 0, depth = 0, depth_max = 0, the white-background normal."""
    c = listed((0, 0, 0))
    c.background = (0.25, -1.0, 2.0)
    got, _ = run_fwd(c, normals)
    assert (got["rgb"] == np.array([0.25, 0.0, 1.0], np.float32)).all() and (got["clamp_mask"] == 1).all()
    assert (got["alpha"] == 0).all() and (got["depth"] == 0).all() and (got["last_ids"] == 0).all()
    assert got["depth_max_bits"] == 0 and got["stats"][:2] == [0, 0]
    if normals:
        s3 = np.sqrt(np.float32(3))
        assert (got["normal_norm"] == s3).all() and (got["normal"] == (np.float32(1) / s3 + np.float32(1)) * np.float32(0.5)).all()
    check(f"empty-{normals}", c.oracle(normals), got)


@pytest.mark.parametrize("normals", [True, False], ids=["rec16", "rec12"])
def test_depth_max_reset_and_last_tile(normals):
    """A second call on the same buffers with a shallower scene reports the smaller maximum; a frame whose only covered
    pixels are in the last partial tile still reports theirs."""
    deep, shallow = generic(81, 49, seed=31), generic(81, 49, seed=31)
    shallow.depths = deep.depths * 0.25
    got_deep, buf = run_fwd(deep, normals)
    got_shallow, _ = run_fwd(shallow, normals, buf=buf)
    check(f"depthmax-deep-{normals}", deep.oracle(normals), got_deep)
    check(f"depthmax-shallow-{normals}", shallow.oracle(normals), got_shallow)  # holds depth_max to max(out_depth)
    assert 0 < got_shallow["depth_max_bits"] < got_deep["depth_max_bits"]
    f = splats(1, 81, 49, seed=1)
    f["means2d"][0] = torch.tensor([80.5, 48.5])
    f["conics"][0] = torch.tensor([20.0, 0.0, 20.0])
    f["radii"][0], f["opac"][0], f["depths"][0] = 3, 0.75, 3.25  # 1 - (1 - 0.75) and 3.25 * 0.75 / 0.75 are exact
    corner = binned(f, 81, 49, 0)
    ref = corner.oracle(normals)
    assert ref.ncomp[:48, :80].max() == 0 and ref.ncomp[48, 80] == 1
    got, _ = run_fwd(corner, normals)
    check(f"depthmax-corner-{normals}", ref, got)
    assert got["depth_max_bits"] == bits(3.25)


@pytest.mark.parametrize("normals", [True, False], ids=["rec16", "rec12"])
def test_two_calls_bit_identical(normals):
    c = generic(200, 136, shift=2, seed=41)
    a, _ = run_fwd(c, normals)
    b, _ = run_fwd(c, normals)
    for k in a:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k]), equal_nan=True), f"{k} differs between two calls"


# ----------------------------------------------------------------------------------------------------- B: scenes
SCENES = ("parity0", "parity1", "parity2", "deep", "clamp", "inside", "antialiased", "sh0")
# every scene with normals on both list kinds (gsplat's exact per-tile lists; the default 64-pixel supertile lists), and
# the 12-float record layout on a few
SCENE_RUNS = [(n, True, l) for n in SCENES for l in ("exact", "2")] + \
    [("parity0", False, "exact"), ("parity2", False, "exact"), ("deep", False, "exact"), ("parity1", False, "2")]


@pytest.mark.parametrize("name,normals,lists", SCENE_RUNS, ids=[f"{n}-{'rec16' if m else 'rec12'}-{l}" for n, m, l in SCENE_RUNS])
def test_scene(name, normals, lists):
    out, c, ref = scene_run(name, normals, lists)
    H, W = c.height, c.width
    depth_max = out.info["depth_max"].cpu().view(F32).item()
    filled = out.depth.cpu().numpy()[..., 0]
    alpha = out.alpha.cpu().numpy()[..., 0]
    # finalize_fwd's fill: uncovered pixels equal depth_max bit for bit; covered ones are the raster kernel's own
    assert (filled[alpha == 0] == np.float32(depth_max)).all(), "uncovered pixels are not filled with depth_max"
    raw = np.where(alpha > 0, filled, 0.0)
    assert np.float32(raw.max()) == np.float32(depth_max)
    # the maps dn_rasterize does not return are not judged here (layer A reads them): give the oracle's own
    got = dict(rgb=out.rgb.cpu().numpy(), depth=raw, alpha=alpha, last_ids=out.info["last_ids"].cpu().numpy().astype(np.int64),
               normal=out.normal.cpu().numpy() if normals else np.zeros((H, W, 3)),
               normal_norm=ref.normal_norm, clamp_mask=ref.clamp_mask)
    v = R.judge(ref, got, EPS, RTOL, ATOL)
    path = os.environ.get("DNR_RASTER_REPORT")
    if path:
        with open(path, "a") as fh:
            fh.write(json.dumps(dict(check=f"scene-{name}-{normals}-{lists}", worst=v.worst, decided=v.n_decided,
                                     ambiguous=v.n_ambiguous, alt_used=v.n_alt_used, unresolved=v.n_unresolved, fail=v.n_fail,
                                     what=v.worst_what)) + "\n")
    assert v.ok, f"{v.n_fail} pixels fail (worst decided ratio {v.worst:.3g}):\n" + "\n".join(v.failures)
    assert v.n_decided >= (1 - MAX_AMBIGUOUS) * H * W and v.n_unresolved <= 1e-3 * H * W, (v.n_decided, v.n_unresolved)
    assert int(ref.ncomp.max()) > 0
    if name == "deep":
        offs = c.tile_offsets.long()
        assert int((offs[1:] - offs[:-1]).max()) > 3 * 128 and ref.stopped.sum() > 100
    if name == "clamp":
        assert ref.clamped.sum() >= 50, "pixels must composite a clamped alpha"
