"""GPU tests of the rasterizer backward (`raster_bwd_kernel`, csrc/raster.cu) per Gaussian against the fp64 backward of
oracle/raster_ref.py, which tests/test_raster_bwd_ref_cpu.py pins on the CPU (torch autograd, finite differences, gsplat_ref's
means2d hooks).

`dnr_raster_bwd` is called through the C ABI with the forward state that `dnr_raster_fwd` itself wrote for the same case
(out_alpha, out_depth, out_normal, normal_norm, clamp_mask, last_ids) and seeded upstream images, and every one of the 16
floats of every `grad_records` row is read, with the `touched` flags.  Layer A: constructed records and lists (both record
layouts), each asserting the branch it is named for.  Layer B: the forward test's scenes, and a 256 x 192 window of the
1M-Gaussian 1080p frame of tests/test_gpu_fullsize.py at its real list depths (upstream non-zero in the window only, the
reference run on the window's tiles).

Ambiguity without exemptions.  Every gradient term of a pixel is proportional to its upstream gradients, so the upstream
images are zeroed on the pixels the forward oracle puts under its decision band (EPS), and on those where an entry sits
within EPS of the 0.999 clamp (the sigma / opacity gradient jumps to 0 there): those pixels contribute exactly nothing,
and every Gaussian is judged.  As a precondition the forward's last_ids must equal the oracle's on every other
pixel, so that a forward fault is not reported as a backward one.

How a Gaussian is judged (raster_ref.judge_bwd), per slot k:
    |got - want| <= RTOL sum_p sqrt(1 + n_p) mass_pgk + ATOL max_g' mass_g'k
with n_p the entries pixel p composited and mass the same expression with every term replaced by its absolute value
(so cancellation in v_alpha = T dot - S' / (1 - alpha) widens the bound instead of failing).  The reference replays the
state the kernel starts from (T_final = 1 - out_alpha); each scene is also held to the unreplayed fp64 state with the
T_final term |(1 - out_alpha) - T64| / T64 x mass as the only extra allowance.  Exact: `touched` is the set of Gaussians
some decided pixel composited (a Gaussian composited only under the band may go either way), untouched rows and slot 15
are bit-zero, a slot without mass (slots 0-3 with only v_normal, 12-14 without it) is exactly 0.

Set DNR_RASTER_REPORT=<file> to append one JSON line per check (worst ratio to the bound, the T_final term): that is how
the constants (tests/raster_cases.py) are re-measured.
"""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from oracle import raster_ref as R
from tests.raster_cases import (BWD_ATOL, BWD_RTOL, EPS, FULLSIZE_WINDOW, TILE, UPSTREAM, Case, binned, generic, listed,
                                pack_records, run_fwd, scene_run, splats, undecided, upstream)

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]

RTOL, ATOL = BWD_RTOL, BWD_ATOL  # measured: tests/raster_cases.py


# ----------------------------------------------------------------------------------------------------- helpers
def state_of(got: dict) -> dict:
    return {k: got[k] for k in ("alpha", "depth", "normal", "normal_norm", "clamp_mask")}


def run_bwd(c: Case, buf, normals: bool, up: dict, exact_flag=False, persistent=False, grads=None, touched=None):
    """dnr_raster_bwd (loss_flags 0) on the forward buffers `buf` of run_fwd for the same case.  Without `persistent` the
    workspace is handed over full of garbage, which the call must clear.  Returns (grad_records, touched) as numpy."""
    from dn_splatter_b200 import _lib as L

    lib = L.load()
    n = c.means2d.shape[0]
    rec = pack_records(c, normals).cuda()
    ids = c.flatten_ids.cuda() if c.flatten_ids.numel() else torch.zeros(1, dtype=torch.int32, device="cuda")
    offs = c.tile_offsets.cuda()
    if grads is None:
        grads = torch.zeros(n, L.GRAD_FLOATS, device="cuda") if persistent else torch.full((n, L.GRAD_FLOATS), 7.25, device="cuda")
    if touched is None:
        touched = torch.zeros(n, dtype=torch.uint8, device="cuda") if persistent else torch.full((n,), 0xAB, dtype=torch.uint8, device="cuda")
    a = L.DnrArgs()
    a.n_gauss, a.width, a.height, a.tile_size = n, c.width, c.height, TILE
    a.flags = (L.FLAG_NORMALS if normals else 0) | (L.FLAG_EXACT_LISTS if exact_flag else 0) | (L.FLAG_PERSISTENT_WS if persistent else 0)
    a.list_shift = c.list_shift
    a.n_isects = int(c.flatten_ids.numel())
    a.background[0], a.background[1], a.background[2] = c.background
    a.loss_flags = 0
    dev = {k: torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32)).cuda() for k, v in up.items()}
    ptrs = dict(records=rec, flatten_ids=ids, tile_offsets=offs, out_rgb=buf.rgb, out_depth=buf.depth, out_alpha=buf.alpha,
                last_ids=buf.last_ids, clamp_mask=buf.clamp_mask, grad_records=grads, touched=touched)
    if normals:
        ptrs.update(out_normal=buf.normal, normal_norm=buf.normal_norm)
    for k, name in (("rgb", "v_rgb"), ("depth", "v_depth"), ("normal", "v_normal"), ("alpha", "v_alpha")):
        if k in dev and (k != "normal" or normals):
            ptrs[name] = dev[k]
    for k, t in ptrs.items():
        setattr(a, k, t.data_ptr())
    L.check(lib.dnr_raster_bwd(C.byref(a), C.c_void_p(torch.cuda.current_stream().cuda_stream)), "dnr_raster_bwd")
    torch.cuda.synchronize()
    return grads.cpu().numpy(), touched.cpu().numpy(), grads, touched


def report(**kw):
    path = os.environ.get("DNR_RASTER_REPORT")
    if path:
        with open(path, "a") as fh:
            fh.write(json.dumps(kw) + "\n")


def touched_sets(bref: R.RasterBwd, n: int, decided: np.ndarray):
    """(Gaussians some decided pixel composited, Gaussians some pixel composited)."""
    sure, any_ = np.zeros(n, bool), np.zeros(n, bool)
    any_[bref.gid] = True
    dec = decided.reshape(-1)[bref.pix]
    sure[bref.gid[dec]] = True
    return sure, any_


def check(name, c: Case, normals: bool, which=UPSTREAM, seed=0, exact_flag=False, unreplayed=False, zero_band=True, only=None,
          tiles=None):
    """Forward, backward and the fp64 reference on case `c`; asserts the rule and the exact properties.  `tiles`: the
    reference composites only those tiles (the upstream images must be zero elsewhere: `only`), and Gaussians touched
    outside them are not questioned.  Returns (reference, grads, touched, forward outputs)."""
    keep: dict = {}
    fref = c.oracle(normals, eps=0.0, keep=keep, tiles=tiles)
    up = upstream(c, fref, which, seed, zero_band, only)
    got_f, buf = run_fwd(c, normals, exact_flag=exact_flag)
    decided = fref.done & (fref.margin >= EPS) if zero_band else fref.done
    bad = decided & (got_f["last_ids"] != fref.last_ids)
    assert not bad.any(), f"{name}: the forward's last_ids differ from the oracle's on {int(bad.sum())} decided pixels"
    grads, touched, _, _ = run_bwd(c, buf, normals, up, exact_flag=exact_flag)
    bref = c.backward(up, state_of(got_f), normals, pre=(fref, keep))
    v = R.judge_bwd(bref, grads, RTOL, ATOL)
    rec = dict(check=name, worst=v.worst, judged=v.n_judged, fail=v.n_fail, what=v.worst_what,
               composited=int(bref.gid.size), undecided=int((fref.done & (~decided | undecided(fref))).sum()))
    if unreplayed:
        uref = c.backward(up, state_of(got_f), normals, pre=(fref, keep), replay=False)
        vu = R.judge_bwd(uref, grads, RTOL, ATOL, extra=1.0)
        b = R.bwd_bound(bref, RTOL, ATOL)
        with np.errstate(invalid="ignore", divide="ignore"):
            term = np.where(uref.tmass > 0, uref.tmass / b, 0.0)
            moved = np.where(b > 0, np.abs(uref.grads - bref.grads) / b, 0.0)
        err_u = np.abs(grads - uref.grads)
        with np.errstate(invalid="ignore", divide="ignore"):  # how much of the unreplayed error the T_final term explains
            share = np.where(err_u > 0, np.abs(uref.grads - bref.grads) / err_u, 0.0)
            g_w, k_w = np.unravel_index(int(np.argmax(np.where(b > 0, err_u / b, 0.0))), err_u.shape)
        rec.update(worst_unreplayed=vu.worst, tfinal_term=float(term.max()), tfinal_moved=float(moved.max()),
                   tfinal_share_at_worst=float(share[g_w, k_w]))
    report(**rec)
    assert v.ok, f"{name}: {v.n_fail} (Gaussian, slot) pairs fail (worst ratio {v.worst:.3g}):\n" + "\n".join(v.failures)
    if unreplayed:
        assert vu.ok, f"{name} (unreplayed): {vu.n_fail} fail (worst {vu.worst:.3g}):\n" + "\n".join(vu.failures)
    n = c.means2d.shape[0]
    assert set(np.unique(touched).tolist()) <= {0, 1}, f"{name}: touched holds values other than 0 / 1"
    # which entries a pixel composited does not depend on the 0.999 clamp (alpha >= 1/255 on both sides of it), so the
    # pixels under the band alone may go either way here
    sure, any_ = touched_sets(bref, n, decided)
    miss, extra = np.nonzero(sure & (touched == 0))[0], np.nonzero(~any_ & (touched != 0))[0]
    assert miss.size == 0, f"{name}: Gaussians {miss[:10].tolist()} were composited but are not touched"
    assert tiles is not None or extra.size == 0, f"{name}: Gaussians {extra[:10].tolist()} were composited by no pixel but are touched"
    assert (grads[touched == 0] == 0).all(), f"{name}: an untouched Gaussian has a non-zero row"
    assert (grads[:, 15] == 0).all(), f"{name}: slot 15 is not zero"
    return bref, grads, touched, got_f


# ----------------------------------------------------------------------------------------------------- A: constructed
LENGTHS = (0, 1, 3, 4, 5, 127, 128, 129, 255, 256, 257, 640, 1100)


@pytest.mark.parametrize("normals", [True, False], ids=["rec16", "rec12"])
def test_list_lengths(normals):
    """Every chunk count up to nine, walked back to front from each tile's deepest last_id, and an empty list."""
    c = listed(LENGTHS, seed=1)
    bref, grads, _, _ = check(f"lengths-{normals}", c, normals)
    assert not bref.fwd.stopped.any() and int(bref.fwd.ncomp.max()) > 200


STOPS = (5, 127, 128, 129, 256, 383)


@pytest.mark.parametrize("normals", [True, False], ids=["rec16", "rec12"])
@pytest.mark.parametrize("stop_at", STOPS)
def test_whole_tile_saturates(stop_at, normals):
    """Every pixel of a tile stops at list entry `stop_at`, so the CTA walks the stop_at entries before it back to front
    from its deepest last_id: a part of one chunk, exactly one or two chunks (the list start on a chunk edge), or one past
    it; and lists up to 1100 entries deep are cut more than a chunk before their end."""
    c = listed([L for L in LENGTHS if L > stop_at] + [stop_at + 1], seed=2, kind="opaque", stop_at=stop_at)
    bref, _, _, got = check(f"saturate-{stop_at}-{normals}", c, normals)
    assert bref.fwd.stopped.all()
    for t in range(c.width // TILE):
        deepest = int(got["last_ids"][:, t * TILE:(t + 1) * TILE].max()) - int(c.tile_offsets[t])
        assert deepest == stop_at - 1
    lens = np.diff(c.tile_offsets.numpy())
    assert lens.max() > 3 * 128 and (lens - stop_at > 128).any()


@pytest.mark.parametrize("normals", [True, False], ids=["rec16", "rec12"])
@pytest.mark.parametrize("kind,stop_at", [("half", 60), ("rows", 10), ("rows", 120), ("warp", 10), ("warp", 130)])
def test_pixels_disagree(kind, stop_at, normals):
    """rows: rows r stop while rows r + 4 of the same lane go on; warp: the lower 8-row half of every tile (one warp)
    stops early and its entries deeper than its own last_id are skipped (pos > wl) while the upper warp walks them."""
    c = listed((300, 640, 257), seed=3, kind=kind, stop_at=stop_at)
    bref, _, _, got = check(f"pairs-{kind}-{stop_at}-{normals}", c, normals)
    ref = bref.fwd
    if kind == "warp":
        assert ref.stopped[8:].all() and not ref.stopped[:8].any()
        gap = 0
        for t in range(c.width // TILE):
            sl = slice(t * TILE, (t + 1) * TILE)
            top, bottom = got["last_ids"][:8, sl], got["last_ids"][8:, sl]
            assert int(top.min()) > int(bottom.max())
            gap = max(gap, int(top.max()) - int(bottom.max()))
        assert gap > 128, "the upper warp must walk more than a chunk past the lower warp's deepest entry"
    if kind == "rows":
        rows = np.arange(TILE)
        assert ref.stopped[(rows % 8) < 4].all() and not ref.stopped[(rows % 8) >= 4].any()


FRAMES = [(13, 7), (17, 17), (81, 49), (75, 53)]


@pytest.mark.parametrize("normals", [True, False], ids=["rec16", "rec12"])
@pytest.mark.parametrize("wh", FRAMES, ids=[f"{w}x{h}" for w, h in FRAMES])
def test_frames(wh, normals):
    """Ragged frames whose last tile row holds an odd number of rows (a lane's pixel pair split by the frame edge),
    alpha-clamped splats (opacity 0.9995 on pixel centres) in warps with unclamped pixels."""
    W, H = wh
    c = generic(W, H, seed=W)
    bref, _, _, _ = check(f"frame-{W}x{H}-{normals}", c, normals)
    ref = bref.fwd
    assert (H % TILE) % 2 == 1, "the last tile row must hold an odd number of rows"
    if W * H >= 3000:
        assert ref.clamped.any() and (~ref.clamped & (ref.ncomp > 0)).any()


@pytest.mark.parametrize("normals", [True, False], ids=["rec16", "rec12"])
@pytest.mark.parametrize("shift,exact", [(0, True), (1, False), (2, False), (3, False)])
def test_supertile_lists(shift, exact, normals):
    """list_shift 1-3 (supertile lists walked with the tile box and the tile-hit filter) and DNR_FLAG_EXACT_LISTS."""
    W, H = 81, 49
    f = splats(max(8, W * H // 40), W, H, seed=11, opaque=0.0, faint=0.5)
    c = binned(f, W, H, shift)
    bref, _, _, _ = check(f"lists-{shift}-{exact}-{normals}", c, normals, exact_flag=exact)
    if shift:
        assert bref.fwd.n_contrib < 0.8 * bref.fwd.n_listed


@pytest.mark.parametrize("normals", [True, False], ids=["rec16", "rec12"])
@pytest.mark.parametrize("bg", [(1.0, 1.0, 1.0), (-0.2, 0.5, 1.3)])
def test_clamp_mask_and_backgrounds(bg, normals):
    """Colours in [-0.5, 1.5] and backgrounds in and outside [0, 1]: a channel outside [0, 1] passes nothing."""
    c = generic(75, 53, seed=21, color=(-0.5, 1.5), background=bg)
    bref, _, _, got = check(f"clamp-{bg}-{normals}", c, normals)
    for k in range(3):
        bit = (got["clamp_mask"] >> k) & 1
        assert bit.min() == 0 and bit.max() == 1


@pytest.mark.parametrize("normals", [True, False], ids=["rec16", "rec12"])
@pytest.mark.parametrize("which", ["rgb", "depth", "normal", "alpha", "all"])
def test_each_upstream_image(which, normals):
    """Each upstream image alone (the others NULL) and all four: only v_normal leaves slots 0-3 exactly 0, and without it
    slots 12-14 are exactly 0."""
    if which == "normal" and not normals:
        pytest.skip("the 12-float layout has no normal image")
    c = generic(81, 49, seed=7)
    sel = UPSTREAM if which == "all" else (which,)
    _, grads, touched, _ = check(f"upstream-{which}-{normals}", c, normals, which=sel)
    assert (grads[touched == 1, 4:8] != 0).any()
    if which == "normal":
        assert (grads[:, 0:4] == 0).all()
    elif which == "all":
        assert (grads[:, 0:4] != 0).any() and (not normals or (grads[:, 12:15] != 0).any())
    else:
        assert (grads[:, 12:15] == 0).all()


def test_empty_tiles_and_the_first_list():
    """Tile 0 holds one small splat at list position 0: its pixels either composited entry 0 (last_id 0) or nothing
    (last_id 0 as well), and the kernel must re-decide which; the latter have alpha = 0 and a non-zero v_depth.  Tile 1's list is all below 1/255 (no pixel composites: the
    CTA returns early); tile 2's list is empty."""
    from tests.test_gpu_raster_forward import _at_centres

    c = _at_centres([0.6, 0.002, 0.5])
    ids = c.flatten_ids.tolist()
    c.flatten_ids = torch.tensor([ids[0], ids[1]], dtype=torch.int32)
    c.tile_offsets = torch.tensor([0, 1, 2, 2], dtype=torch.int32)
    for normals in (True, False):
        bref, grads, touched, got = check(f"first-list-{normals}", c, normals)
        t0 = got["last_ids"][:, :TILE]
        assert (t0 == 0).all() and (bref.fwd.ncomp[:, :TILE] == 1).any() and (got["alpha"][:, :TILE] == 0).any()
        assert touched.tolist() == [1, 0, 0] and (grads[0, 4:15] != 0).any()


@pytest.mark.parametrize("normals", [True, False], ids=["rec16", "rec12"])
def test_no_intersections(normals):
    """n_isects = 0: the call returns after clearing the workspace."""
    c = listed((0, 0, 0))
    keep: dict = {}
    fref = c.oracle(normals, eps=0.0, keep=keep)
    got, buf = run_fwd(c, normals)
    grads, touched, _, _ = run_bwd(c, buf, normals, upstream(c, fref))
    assert c.flatten_ids.numel() == 0 and (grads == 0).all() and (touched == 0).all()


KS = (-3, -2, -1, 0, 1, 2, 3)


@pytest.mark.parametrize("normals", [True, False], ids=["rec16", "rec12"])
@pytest.mark.parametrize("where", ["alpha_min", "alpha_max"])
def test_thresholds_as_the_forward_decided(where, normals):
    """Splats on a pixel centre (sigma = 0 exactly, vis = 1) with opacity 1/255 (resp. 0.999) stepped +-3 ulp in fp32:
    the backward re-decides alpha < 1/255 itself; a splat is touched and has a non-zero row exactly when the forward
    composited it, and its opacity gradient is exactly 0 exactly when op * vis > 0.999f (the clamp fix-up; for that
    check the upstream images are non-zero only on the splats' centre pixels)."""
    from tests.test_gpu_raster_forward import _at_centres, _steps

    x = np.float32(1.0) / np.float32(255.0) if where == "alpha_min" else np.float32(0.999)
    ops = _steps(x, KS)
    c = _at_centres(ops)
    centres = np.zeros((c.height, c.width), bool)
    centres[5, 8::TILE] = True
    _, grads, touched, got = check(f"threshold-{where}-{normals}", c, normals, zero_band=False,
                                   only=centres if where == "alpha_max" else None)
    for t, op in enumerate(ops):
        composited = bool(got["alpha"][5, t * TILE + 8] > 0)
        assert composited == (np.float32(op) >= x if where == "alpha_min" else True)
        assert bool(touched[t]) == composited and bool((grads[t] != 0).any()) == composited, (KS[t], composited)
        if where == "alpha_max":
            assert (grads[t, 7] == 0) == (np.float32(op) > x), f"{KS[t]:+d} ulp: v_opacity {grads[t, 7]}"


def test_persistent_workspace_accumulates():
    """DNR_FLAG_PERSISTENT_WS: two calls add into the same rows (within the sum of the bounds) and the flags are the
    union; each call alone is what the default mode gives."""
    c1 = generic(81, 49, seed=51)
    f = {k: getattr(c1, k) for k in ("conics", "opac", "colors", "depths", "normals_cam", "radii")}
    c2 = binned(dict(f, means2d=c1.means2d + torch.tensor([37.0, -11.0])), 81, 49, 0, background=c1.background)  # other ones visible
    refs, flags = [], []
    grads = touched = None
    for k, c in enumerate((c1, c2)):
        keep: dict = {}
        fref = c.oracle(True, eps=0.0, keep=keep)
        up = upstream(c, fref, seed=k)
        got, buf = run_fwd(c, True)
        g_np, t_np, grads, touched = run_bwd(c, buf, True, up, persistent=True, grads=grads, touched=touched)
        bref = c.backward(up, state_of(got), True, pre=(fref, keep))
        refs.append(bref)
        sure, any_ = touched_sets(bref, c.means2d.shape[0], fref.done & (fref.margin >= EPS))
        flags.append((sure, any_))
    want = refs[0].grads + refs[1].grads
    bound = R.bwd_bound(refs[0], RTOL, ATOL) + R.bwd_bound(refs[1], RTOL, ATOL)
    err = np.abs(g_np - want)
    assert (err <= bound).all(), f"accumulated rows leave the bound: worst {float(np.max(np.where(bound > 0, err / bound, np.where(err > 0, np.inf, 0)))):.3g}"
    sure = flags[0][0] | flags[1][0]
    any_ = flags[0][1] | flags[1][1]
    assert (t_np[sure] == 1).all() and (t_np[~any_] == 0).all()
    assert (flags[0][0] & ~flags[1][1]).any() and (flags[1][0] & ~flags[0][1]).any(), "each call must touch Gaussians the other does not"


# ----------------------------------------------------------------------------------------------------- B: scenes
SCENES = ("parity0", "parity1", "parity2", "deep", "clamp", "inside", "antialiased", "sh0")
# every scene on gsplat's exact per-tile lists and on the default 64-pixel supertile lists, except the two largest parity
# scenes (one kind each: the file stays within its minute), and two in the 12-float layout
SCENE_RUNS = [(n, True, l) for n in SCENES for l in ("exact", "2") if (n, l) not in (("parity0", "2"), ("parity1", "exact"))] + \
    [("parity2", False, "exact"), ("sh0", False, "2")]


@pytest.mark.parametrize("name,normals,lists", SCENE_RUNS, ids=[f"{n}-{'rec16' if m else 'rec12'}-{l}" for n, m, l in SCENE_RUNS])
def test_scene(name, normals, lists):
    """The forward test's scenes (the CUDA side's own per-Gaussian outputs and lists), seeded upstream images, and the
    unreplayed fp64 state with the T_final term as its only extra allowance."""
    _, c, _ = scene_run(name, normals, lists, oracle=False)
    bref, grads, touched, _ = check(f"scene-{name}-{normals}-{lists}", c, normals, exact_flag=lists == "exact", unreplayed=True)
    assert int(touched.sum()) > 20
    if name == "deep":
        offs = c.tile_offsets.long()
        assert int((offs[1:] - offs[:-1]).max()) > 3 * 128 and bref.fwd.stopped.sum() > 100
    if name == "clamp":
        assert bref.fwd.clamped.sum() >= 50


def test_fullsize_window():
    """The 1M-Gaussian 1080p frame of tests/test_gpu_fullsize.py on exact lists: the kernel runs on the whole frame with
    upstream images non-zero only in a 256 x 192 window of whole tiles, and the reference composites only the window's
    tiles, at the frame's real list depths.  Every Gaussian is judged: those the window does not reach must have rows of
    exact zeros (they may still be touched by pixels outside it)."""
    _, c, _ = scene_run("fullsize", True, "exact", oracle=False)
    x0, y0, ww, wh = FULLSIZE_WINDOW
    only = np.zeros((c.height, c.width), bool)
    only[y0:y0 + wh, x0:x0 + ww] = True
    tiles = [(tx, ty) for ty in range(y0 // TILE, (y0 + wh) // TILE) for tx in range(x0 // TILE, (x0 + ww) // TILE)]
    bref, grads, touched, _ = check("fullsize-window", c, True, exact_flag=True, only=only, tiles=tiles)
    tiles_x = -(-c.width // TILE)
    offs = c.tile_offsets.numpy().astype(np.int64)
    lens = np.array([offs[ty * tiles_x + tx + 1] - offs[ty * tiles_x + tx] for tx, ty in tiles])
    reached = np.unique(bref.gid)
    assert lens.max() > 3 * 128 and int(bref.fwd.stopped[only].sum()) >= 100, (int(lens.max()), int(bref.fwd.stopped[only].sum()))
    assert reached.size > 100 and int(touched.sum()) > reached.size, "Gaussians outside the window must be touched too"
    assert (grads[np.setdiff1d(np.nonzero(touched)[0], reached)] == 0).all()

