"""Cases for the rasterizer tests (tests/test_gpu_raster_forward.py, tests/test_gpu_raster_backward.py and the CPU pins
of oracle/raster_ref.py): what `raster_fwd_kernel` / `raster_bwd_kernel` read, built on the CPU, and the C-ABI calls
that run the forward on them."""
import ctypes as C
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from oracle import gsplat_ref as G
from oracle import raster_ref as R

F32 = torch.float32
TILE = 16

# The decision band.  It must stay well below 7e-4, the relative width of the slack 2^-1e-3 of the in-loop pre-test
# `pw < nthr`: a pre-test with the slack on the wrong side drops alphas up to 7e-4 above 1/255, and would hide in a wider band.
EPS = 2e-5
# The backward's acceptance rule (raster_ref.judge_bwd), per Gaussian and grad_records slot k:
#     |got - want| <= BWD_RTOL sum_p sqrt(1 + n_p) mass_pgk + BWD_ATOL max_g' mass_g'k.
# Measured on an H100 80GB HBM3 (700 W limit) over the checks of tests/test_gpu_raster_backward.py: the worst (Gaussian,
# slot) uses 0.26 of the bound (a colour slot of the `rows` pairs case; scenes at most 0.23, the clamp scene; the 1080p
# window 0.020).  Against the unreplayed fp64 state the T_final term moves the reference by up to 15x this bound (clamp
# scene) and explains >= 99.5 % of the kernel's difference at the worst Gaussian of every scene.
BWD_RTOL, BWD_ATOL = 5e-7, 5e-8
UPSTREAM = ("rgb", "depth", "normal", "alpha")


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

    def backward(self, up: dict, state: dict, normals=True, **kw) -> R.RasterBwd:
        """raster_ref.backward on upstream images up = {rgb, depth, normal, alpha} (missing: zero) at forward `state`."""
        return R.backward(self.means2d, self.conics, self.opac, self.colors, self.depths,
                          self.normals_cam if normals else None, self.radii, self.flatten_ids, self.tile_offsets,
                          self.list_shift, self.width, self.height, self.background, up.get("rgb"), up.get("depth"),
                          up.get("normal") if normals else None, up.get("alpha"), state, **kw)


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
    rows r + 4 (the other pixel of the same lane) skip every line.
    warp: the same lines on each of the rows 8..15 only: the lower 8-row half of the tile stops there, the upper half goes
    on to the end of the list."""
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
        if kind in ("rows", "warp") and stop_at is not None and L >= stop_at + 32:
            k = 0
            lines = [band + row for band in (0, 8) for row in range(4)] if kind == "rows" else list(range(8, 16))
            for row in lines:
                for _ in range(4):
                    m[stop_at + k] = torch.tensor([x0 + 8.0, row + 0.5])
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


FULLSIZE = (1_000_000, 1920, 1080)  # BASELINE.json's C2 size, as tests/test_gpu_fullsize.py renders it
FULLSIZE_WINDOW = (832, 448, 256, 192)  # x0, y0, width, height: whole 16 x 16 tiles around the principal point


def scene(name):
    """(params, cam, dn_rasterize kwargs)."""
    from tests.helpers import scene_and_camera
    from tests.test_gpu_backward_edges import clamp_scene, inside_camera

    if name == "fullsize":
        from dn_splatter_b200.synthetic import make_scene, ring_cameras

        n, W, H = FULLSIZE
        return make_scene(n, seed=0), ring_cameras(200, W, H)[17], {}
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


def scene_run(name, normals, lists, oracle=True):
    """dn_rasterize on the scene, and the oracle on the CUDA side's own per-Gaussian outputs and lists (None without
    `oracle`)."""
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
    return out, c, (c.oracle(normals) if oracle else None)


def upstream(c: Case, fref: R.RasterRef, which=UPSTREAM, seed=0, zero_band=True, only=None) -> dict:
    """Seeded upstream images in [-1, 1) (fp32) for the images in `which`, zero on the pixels `undecided` puts under the
    decision band (and outside the bool [H,W] `only`)."""
    g = torch.Generator().manual_seed(seed)
    H, W = c.height, c.width
    shapes = dict(rgb=(H, W, 3), depth=(H, W), normal=(H, W, 3), alpha=(H, W))
    out = {}
    for k in UPSTREAM:
        x = (2 * torch.rand(*shapes[k], generator=g) - 1).numpy()
        if zero_band:
            x[undecided(fref)] = 0.0
        if only is not None:
            x[~only] = 0.0
        if k in which:
            out[k] = x
    return out


def undecided(fref: R.RasterRef) -> np.ndarray:
    """Pixels whose backward the kernel and fp64 may take differently: a compositing decision within EPS of its threshold
    (margin), or an entry within EPS of the 0.999 clamp, where the sigma / opacity gradient jumps from -op vis to 0."""
    return (fref.margin < EPS) | (fref.clamp_margin < EPS)


def _background():
    from dn_splatter_b200.synthetic import BACKGROUND

    return BACKGROUND
