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
import ctypes as C
import json
import os
from dataclasses import dataclass
from typing import Optional

import numpy as np
import pytest
import torch

from oracle import gsplat_ref as G
from oracle import raster_ref as R

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]

F32 = torch.float32
TILE = 16
# The decision band.  It must stay well below 7e-4, the relative width of the slack 2^-1e-3 of the in-loop pre-test
# `pw < nthr`: a pre-test with the slack on the wrong side drops alphas up to 7e-4 above 1/255, and would hide in a wider band.
EPS = 2e-5
# Bound per output: sqrt(1 + composited) (RTOL mass + ATOL).  Measured on an H100 80GB HBM3 (700 W limit) over the 98 checks
# of this file: the worst decided pixel uses 0.25 of the bound (a clamp-scene pixel 1.7e-2 from sigma = 0; constructed
# cases at most 0.19), 1270 pixels in all sit under the band (at most 1.04 % of a frame), 2 of them match an alternative
# other than the oracle's primary outcome, none has too many alternatives.
RTOL, ATOL = 2e-6, 2.4e-7
MAX_AMBIGUOUS = 0.01  # share of a scene's pixels that may sit under the band (measured: 0.1 % on the scenes)


# ----------------------------------------------------------------------------------------------------- cases (CPU)
@dataclass
class Case:
    """What the kernel reads, as fp32 / int32 CPU tensors."""

    means2d: torch.Tensor
    conics: torch.Tensor
    opac: torch.Tensor
    colors: torch.Tensor
    depths: torch.Tensor
    normals_cam: torch.Tensor
    radii: torch.Tensor
    flatten_ids: torch.Tensor
    tile_offsets: torch.Tensor
    list_shift: int
    width: int
    height: int
    background: tuple = (0.1, 0.2, 0.3)

    def oracle(self, normals=True, eps=EPS, **kw) -> R.RasterRef:
        return R.composite(self.means2d, self.conics, self.opac, self.colors, self.depths,
                           self.normals_cam if normals else None, self.radii, self.flatten_ids, self.tile_offsets,
                           self.list_shift, self.width, self.height, self.background, eps=eps, **kw)


def splats(n, W, H, seed, faint=0.3, opaque=0.2, color=(0.0, 1.0), snap=0.2):
    """n generic 2-D Gaussians around a W x H frame: std 1.5 to 11.5 px, correlation up to 0.8, opacities a mixture of
    faint (0.004 to 0.03), middling and nearly opaque (0.9 to 1, a third of them 0.9995: above the clamp); a share `snap`
    sits exactly on a pixel centre.  Returns the per-Gaussian fields of Case as a dict."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.rand(*s, generator=g)  # noqa: E731
    m = r(n, 2) * torch.tensor([W + 16.0, H + 16.0]) - 8.0
    sn = r(n) < snap
    m = torch.where(sn[:, None], m.floor() + 0.5, m)
    sx, sy, rho = 1.5 + 10 * r(n), 1.5 + 10 * r(n), 0.8 * (2 * r(n) - 1)
    a, c, b = sx * sx, sy * sy, rho * sx * sy
    det = a * c - b * b
    conics = torch.stack([c / det, -b / det, a / det], 1)
    mid = 0.5 * (a + c)
    radii = torch.ceil(3 * torch.sqrt(mid + torch.sqrt(torch.clamp(mid * mid - det, min=0.01)))).to(torch.int32)
    u = r(n)
    op = torch.where(u < faint, 0.004 + 0.026 * r(n), torch.where(u > 1 - opaque, 0.9 + 0.1 * r(n), 0.05 + 0.55 * r(n)))
    op = torch.where((u > 1 - opaque) & (r(n) < 1 / 3), torch.tensor(0.9995), op)
    nrm = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=1)
    return dict(means2d=m.float(), conics=conics.float(), opac=op.float(), colors=color[0] + (color[1] - color[0]) * r(n, 3),
                depths=0.5 + 9.5 * r(n), normals_cam=nrm.float(), radii=radii)


def binned(f, W, H, shift, **kw) -> Case:
    """Lists per supertile of (16 << shift)^2 pixels from the splats' tile boxes, sorted by depth."""
    _, _, flat, offs, _ = G.isect_tiles(f["means2d"], f["radii"], f["depths"], TILE << shift, W, H)
    to = torch.cat([offs, torch.tensor([flat.shape[0]], dtype=torch.int32)])
    return Case(flatten_ids=flat, tile_offsets=to, list_shift=shift, width=W, height=H, **f, **kw)


def generic(W, H, shift=0, n=None, seed=0, **kw) -> Case:
    bg = kw.pop("background", (0.1, 0.2, 0.3))
    n = n if n is not None else max(8, W * H // 12)
    return binned(splats(n, W, H, seed, **kw), W, H, shift, background=bg)


def listed(lengths, seed=0, kind="faint", stop_at=None) -> Case:
    """One row of 16 x 16 tiles, tile t with a hand-made list of lengths[t] entries in shuffled id order (list_shift 0).
    faint: opacities 0.006 to 0.02, std 6 px (the first 8 entries of a list 0.02 and inside the tile): no pixel saturates.
    opaque run (stop_at = s): entries s-4 .. s-1 of every list are wide splats of opacity 0.8 and entry s one of opacity
    0.999: every pixel composites s-4 .. s-1 (T stays above 1e-4) and stops at entry s.
    half: the same run at opacity 0.9, narrow in x around column 2: the left columns stop there, the right ones go on.
    rows: the run is replaced by 4 thin horizontal lines on each of the rows 0..3 of both 8-row bands: rows r stop,
    rows r + 4 (the other pixel of the same lane) skip every line."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.rand(*s, generator=g)  # noqa: E731
    f = {k: [] for k in ("means2d", "conics", "opac")}
    offs = [0]
    n = 0
    for t, L in enumerate(lengths):
        x0 = t * TILE
        m = torch.stack([x0 - 4 + 24 * r(L), -4 + 24 * r(L)], 1)
        con = torch.stack([torch.full((L,), 1 / 36.0), 0.01 * (2 * r(L) - 1), torch.full((L,), 1 / 36.0)], 1)
        op = 0.006 + 0.014 * r(L)
        m[:8] = torch.stack([x0 + 2 + 12 * r(L), 2 + 12 * r(L)], 1)[:8]
        op[:8] = 0.02
        if kind in ("opaque", "half") and stop_at is not None and L > stop_at:
            run = torch.arange(stop_at - 4, stop_at + 1)
            m[run] = torch.tensor([x0 + (2.3 if kind == "half" else 8.2), 7.7])
            con[run] = torch.tensor([0.02 if kind == "half" else 1e-4, 0.0, 1e-4])
            op[run] = 0.9 if kind == "half" else 0.8
            op[stop_at] = 0.999
        if kind == "rows" and stop_at is not None and L >= stop_at + 32:
            k = 0
            for band in (0, 8):
                for row in range(4):
                    for _ in range(4):
                        m[stop_at + k] = torch.tensor([x0 + 8.0, band + row + 0.5])
                        con[stop_at + k] = torch.tensor([1e-4, 0.0, 2.0])
                        op[stop_at + k] = 0.95
                        k += 1
        f["means2d"].append(m)
        f["conics"].append(con)
        f["opac"].append(op)
        n += L
        offs.append(n)
    perm = torch.randperm(max(n, 1), generator=g)[:n]
    inv = torch.empty_like(perm)
    inv[perm] = torch.arange(n)
    cat = lambda k, w: (torch.cat(f[k]) if n else torch.zeros((0,) + w))  # noqa: E731
    pick = lambda t: t[inv] if n else t  # noqa: E731  Gaussian perm[q] holds entry q: row i of the tables is entry inv[i]
    nn = max(n, 1)
    out = dict(means2d=pick(cat("means2d", (2,))), conics=pick(cat("conics", (3,))), opac=pick(cat("opac", ())))
    if n == 0:  # the kernel still wants a records table
        out = dict(means2d=torch.zeros(1, 2), conics=torch.ones(1, 3), opac=torch.zeros(1))
    return Case(colors=r(nn, 3), depths=0.5 + 9.5 * r(nn), normals_cam=torch.nn.functional.normalize(torch.randn(nn, 3, generator=g), dim=1),
                radii=torch.full((nn,), 64, dtype=torch.int32), flatten_ids=perm.to(torch.int32),
                tile_offsets=torch.tensor(offs, dtype=torch.int32), list_shift=0, width=TILE * len(lengths), height=TILE,
                **{k: v.float() for k, v in out.items()})


# ----------------------------------------------------------------------------------------------------- the kernel
LOG2E = torch.tensor(1.4426950408889634, dtype=F32)


def pack_records(c: Case, normals: bool) -> torch.Tensor:
    """The packed records as project_fwd writes them (tests/test_gpu_projection.py pins that packing bit for bit)."""
    n = c.means2d.shape[0]
    rec = torch.zeros(n, 16 if normals else 12, dtype=F32)
    rec[:, 0:2] = c.means2d
    rec[:, 2] = (-0.5 * LOG2E) * c.conics[:, 0]
    rec[:, 3] = (-LOG2E) * c.conics[:, 1]
    rec[:, 4] = (-0.5 * LOG2E) * c.conics[:, 2]
    rec[:, 5] = c.opac
    rec[:, 6] = -torch.log2(255.0 * c.opac) - torch.tensor(1e-3, dtype=F32)
    rec[:, 7] = c.radii.float()
    rec[:, 8:11] = c.colors
    rec[:, 11] = c.depths
    if normals:
        rec[:, 12:15] = c.normals_cam
    return rec


class Buffers:
    """Device outputs of dnr_raster_fwd, pre-filled so that a pixel the kernel does not write fails."""

    def __init__(self, H, W):
        nan = float("nan")
        d = "cuda"
        self.rgb = torch.full((H, W, 3), nan, dtype=F32, device=d)
        self.depth = torch.full((H, W), nan, dtype=F32, device=d)
        self.alpha = torch.full((H, W), nan, dtype=F32, device=d)
        self.normal = torch.full((H, W, 3), nan, dtype=F32, device=d)
        self.normal_norm = torch.full((H, W), nan, dtype=F32, device=d)
        self.last_ids = torch.full((H, W), -7, dtype=torch.int32, device=d)
        self.clamp_mask = torch.full((H, W), 0xAA, dtype=torch.uint8, device=d)
        self.depth_max = torch.full((1,), 0x7F000000, dtype=torch.int32, device=d)  # a huge stale maximum
        self.stats = torch.zeros(4, dtype=torch.int64, device=d)

    def numpy(self, normals):
        torch.cuda.synchronize()
        out = dict(rgb=self.rgb, depth=self.depth, alpha=self.alpha, last_ids=self.last_ids, clamp_mask=self.clamp_mask)
        out = {k: v.cpu().numpy() for k, v in out.items()}
        H, W = self.depth.shape
        out["normal"] = self.normal.cpu().numpy() if normals else np.zeros((H, W, 3))
        out["normal_norm"] = self.normal_norm.cpu().numpy() if normals else np.zeros((H, W))
        out["last_ids"] = out["last_ids"].astype(np.int64)
        out["depth_max_bits"] = int(self.depth_max.cpu()[0])
        out["stats"] = self.stats.cpu().tolist()
        return out


def run_fwd(c: Case, normals=True, exact_flag=False, buf: Optional[Buffers] = None):
    """dnr_raster_fwd on the case; returns (numpy outputs, buffers)."""
    from dn_splatter_b200 import _lib as L

    lib = L.load()
    buf = buf or Buffers(c.height, c.width)
    buf.stats.zero_()  # the kernel adds to them
    rec = pack_records(c, normals).cuda()
    ids = c.flatten_ids.cuda() if c.flatten_ids.numel() else torch.zeros(1, dtype=torch.int32, device="cuda")
    offs = c.tile_offsets.cuda()
    a = L.DnrArgs()
    a.n_gauss, a.width, a.height, a.tile_size = rec.shape[0], c.width, c.height, TILE
    a.flags = (L.FLAG_NORMALS if normals else 0) | (L.FLAG_EXACT_LISTS if exact_flag else 0)
    a.list_shift = c.list_shift
    a.n_isects = int(c.flatten_ids.numel())
    a.background[0], a.background[1], a.background[2] = c.background
    for k, t in dict(records=rec, flatten_ids=ids, tile_offsets=offs, out_rgb=buf.rgb, out_depth=buf.depth, out_alpha=buf.alpha,
                     last_ids=buf.last_ids, clamp_mask=buf.clamp_mask, depth_max=buf.depth_max, stats=buf.stats).items():
        setattr(a, k, t.data_ptr())
    if normals:
        a.out_normal, a.normal_norm = buf.normal.data_ptr(), buf.normal_norm.data_ptr()
    L.check(lib.dnr_raster_fwd(C.byref(a), C.c_void_p(torch.cuda.current_stream().cuda_stream)), "dnr_raster_fwd")
    return buf.numpy(normals), buf


def bits(x: float) -> int:
    return int(np.float32(x).view(np.int32))


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
def scene(name):
    """(params, cam, dn_rasterize kwargs)."""
    from tests.helpers import scene_and_camera
    from tests.test_gpu_backward_edges import clamp_scene, inside_camera

    if name.startswith("parity"):
        from tests.test_gpu_parity import CASES

        return (*scene_and_camera(**CASES[int(name[-1])]), {})
    if name == "deep":
        return (*scene_and_camera(8000, 96, 80, view=1), {})
    if name == "clamp":
        p, cam, _ = clamp_scene()
        return p, cam, {}
    if name == "inside":
        from dn_splatter_b200.synthetic import make_scene

        return make_scene(3000, seed=1), inside_camera(), {}
    if name == "antialiased":
        return (*scene_and_camera(1000, 96, 80, view=1), dict(antialiased=True))
    if name == "sh0":
        return (*scene_and_camera(1000, 128, 80, view=2), dict(sh_degree=0))
    raise ValueError(name)


SCENES = ("parity0", "parity1", "parity2", "deep", "clamp", "inside", "antialiased", "sh0")
# every scene with normals on both list kinds (gsplat's exact per-tile lists; the default 64-pixel supertile lists), and
# the 12-float record layout on a few
SCENE_RUNS = [(n, True, l) for n in SCENES for l in ("exact", "2")] + \
    [("parity0", False, "exact"), ("parity2", False, "exact"), ("deep", False, "exact"), ("parity1", False, "2")]


def scene_run(name, normals, lists):
    """dn_rasterize on the scene, and the oracle on the CUDA side's own per-Gaussian outputs and lists."""
    from tests.helpers import cuda_outputs

    params, cam, kw = scene(name)
    kw = dict(kw, render_normals=normals, **(dict(exact_lists=True) if lists == "exact" else dict(list_shift=int(lists))))
    _, out = cuda_outputs(params, cam, **kw)
    info = out.info
    ncam = (out.normals_world @ cam["c2w"][:3, :3].cuda()).cpu() if normals else None
    c = Case(means2d=out.means2d.cpu(), conics=out.conics.cpu(), opac=info["opacities"].cpu(), colors=info["colors"].cpu(),
             depths=out.depths.cpu(), normals_cam=ncam, radii=out.radii.cpu(), flatten_ids=info["flatten_ids"].cpu(),
             tile_offsets=info["tile_offsets"].cpu(), list_shift=0 if lists == "exact" else int(lists), width=cam["width"],
             height=cam["height"], background=tuple(float(b) for b in _background()))
    return out, c, c.oracle(normals)


def _background():
    from dn_splatter_b200.synthetic import BACKGROUND

    return BACKGROUND


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
