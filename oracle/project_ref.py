"""ORACLE (test infrastructure, NOT product code): the per-Gaussian projection of csrc/project.cu in float64 and its
vector-Jacobian product, the reference of tests/test_gpu_projection.py.

`forward64` evaluates, per Gaussian, every output dnr_project_fwd hands to the rasterizer: means2d, the conic (A, B, C),
the opacity the raster sees (x compensation when antialiased), the clamped SH colour, the camera depth and the
camera-frame normal.  The formulas are those of gsplat_ref.project_gaussians, gsplat_ref.eval_sh and
dn_ref.gaussian_normals (tests/test_project_ref_cpu.py checks that, away from ties, its autograd equals theirs), with the
kernel's conventions at the points where the derivative is not defined taken explicitly from `Branches`:

  * the 1.3 tan(fov) Jacobian clamp: |x/z| = lim counts as unclamped (the kernel clamps when !(xr <= lim && xr >= -lim));
  * clamp_min(colour + 0.5, 0): colour + 0.5 = 0 passes the gradient;
  * the compensation sqrt(det_orig / det): no gradient where it is 0;
  * the normal's sign: the one the forward rendered (its normals_world), never recomputed from float64.

`Branches.from_fp32` decides these the way the kernel does, in float32 and in its operation order.  `vjp64` is autograd
of sum(grad_records . outputs) over the rows of the given Gaussians: what dnr_project_bwd computes from a
raster-gradient record.

`SLIPS` are plausible mistakes in the backward, applied to the reference; tests/test_project_ref_cpu.py shows each moves
some Gaussian of the GPU test's data far outside the per-Gaussian tolerance.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional

import torch
from torch import Tensor

from oracle import gsplat_ref as G
from oracle.dn_ref import get_viewmat

F32, F64 = torch.float32, torch.float64
PARAM_KEYS = ("means", "quats", "scales", "opacities", "sh_dc", "sh_rest")
LOG2E = 1.4426950408889634
SLIPS = ("clamp_z", "comp", "inorm", "abs_swap", "flip_bwd")


# ----------------------------------------------------------------------------------------------------- cases
@dataclass
class Case:
    """One projection problem: fp32 parameters (raw or activated), an fp32 camera and the launch options."""

    params: Dict[str, Tensor]  # means [N,3], quats [N,4], scales [N,3], opacities [N], sh_dc [N,3], sh_rest [N,B-1,3]
    viewmat: Tensor  # [4,4] world -> OpenCV camera
    K: Tensor  # [3,3]
    c2w: Tensor  # [3,4] OpenGL camera -> world (normals)
    width: int
    height: int
    activated: bool = False
    antialiased: bool = False
    normals: bool = True
    sh_degree: int = 3
    eps2d: float = 0.3
    near_plane: float = 0.01
    far_plane: float = 50.0
    radius_clip: float = 0.0
    cov_noise: Optional[Tensor] = None  # [N,3,3] symmetric, relative to max|Sc| per Gaussian (see `perturbed`)

    @property
    def n(self) -> int:
        return self.params["means"].shape[0]

    @property
    def sh_bases(self) -> int:
        return 1 + self.params["sh_rest"].shape[1]


def _rotation(g: torch.Generator) -> Tensor:
    q, r = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=F64))
    q = q * torch.sign(torch.diagonal(r))[None, :]
    return q if torch.det(q) > 0 else -q


def camera(seed: int, width: int = 96, height: int = 72):
    """(viewmat [4,4], K [3,3], c2w [3,4]) fp32: a randomly oriented camera, fx != fy, an off-centre principal point."""
    g = torch.Generator().manual_seed(seed)
    c2w = torch.cat([_rotation(g), 2 * torch.randn(3, 1, generator=g, dtype=F64)], 1).float()
    vm = get_viewmat(c2w.double()).float()
    K = torch.tensor([[0.9 * width, 0, width / 2 + 3.25], [0, 1.05 * height, height / 2 - 2.5], [0, 0, 1]], dtype=F32)
    return vm, K, c2w


def _to_world(vm: Tensor, pc: Tensor) -> Tensor:
    Wm, t = vm[:3, :3].double(), vm[:3, 3].double()
    return ((pc - t) @ Wm).float()  # W^T (p - t), row by row


def _lims(K: Tensor, width: int, height: int):
    """The kernel's fp32 1.3 tan(fov) limits."""
    tx = torch.tensor(0.5 * width, dtype=F32) / K[0, 0].float()
    ty = torch.tensor(0.5 * height, dtype=F32) / K[1, 1].float()
    return float(tx * 1.3), float(ty * 1.3)


def random_case(n: int, seed: int, sh_bases: int = 16, sh_degree: int = 3, kind: str = "random", **kw) -> Case:
    """Gaussians for the per-Gaussian comparisons.

    random   depth 0.3-8 (3 % behind the near plane, 3 % beyond the far plane), x/z and y/z up to 1.5 x the clamp limit,
             log-scales N(-3.5, 1) with 15 % needles (one axis e^5 x the other two), un-normalised quaternions (norm
             0.5-2), raw opacities N(0, 2), SH coefficients with a third of the colours clamped at 0
    clamped  every Gaussian past the Jacobian clamp in x, in y or in both (alternating), large enough to reach the frame
    rank1    activated scales (s, 0, 0): a rank-1 covariance, compensation 0 (det_orig <= 0) on many of them
    """
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.rand(*s, generator=g, dtype=F64)  # noqa: E731
    nrm = lambda *s: torch.randn(*s, generator=g, dtype=F64)  # noqa: E731
    W, H = kw.pop("width", 96), kw.pop("height", 72)
    vm, K, c2w = camera(seed, W, H)
    lx, ly = _lims(K, W, H)
    z = 0.3 + 7.7 * r(n)
    xr, yr = (2 * r(n) - 1) * 1.5 * lx, (2 * r(n) - 1) * 1.5 * ly
    logs = nrm(n, 3) - 3.5
    needle = r(n) < 0.15
    logs[needle] = torch.stack([logs[needle, 0] + 5, logs[needle, 0], logs[needle, 0]], 1)
    if kind == "random":
        u = r(n)
        z = torch.where(u < 0.03, -0.5 + 0.5 * r(n), torch.where(u > 0.97, 50 + 10 * r(n), z))
    elif kind == "clamped":
        which = torch.arange(n) % 3  # 0: x, 1: y, 2: both
        sx = torch.where(r(n) < 0.5, -1.0, 1.0)
        sy = torch.where(r(n) < 0.5, -1.0, 1.0)
        cx_, cy_ = float(K[0, 2]), float(K[1, 2])
        fx, fy = float(K[0, 0]), float(K[1, 1])
        xr = torch.where(which != 1, sx * lx * (1.02 + 0.2 * r(n)), xr / 1.5 * 0.9)
        yr = torch.where(which != 0, sy * ly * (1.02 + 0.2 * r(n)), yr / 1.5 * 0.9)
        # radius ~ 3 f s / z must reach back into the frame from mx ~ c + f x/z
        need = torch.maximum((fx * xr.abs() + abs(cx_) + W) / fx, (fy * yr.abs() + abs(cy_) + H) / fy)
        logs = torch.log(z * need * (0.25 + 0.2 * r(n)))[:, None] + 0.3 * nrm(n, 3)
    elif kind == "rank1":
        pass
    else:
        raise ValueError(kind)
    pc = torch.stack([xr * z, yr * z, z], 1)
    means = _to_world(vm, pc)
    quats = nrm(n, 4)
    quats = (quats / quats.norm(dim=1, keepdim=True) * (0.5 + 1.5 * r(n, 1))).float()
    opac = (2 * nrm(n)).float()
    dc = 0.5 * nrm(n, 3)
    dc[r(n) < 0.33] -= 4.0
    rest = (0.3 * nrm(n, sh_bases - 1, 3)).float()
    scales = logs.float()
    activated = kw.pop("activated", False)
    if kind == "rank1":
        activated = True
        scales = torch.exp(logs).float()
        scales[:, 1:] = 0.0
    if activated:
        if kind != "rank1":
            scales = torch.exp(logs).float()
        opac = torch.sigmoid(opac.double()).float()
    params = dict(means=means, quats=quats, scales=scales.contiguous(), opacities=opac, sh_dc=dc.float(),
                  sh_rest=rest.contiguous())
    return Case(params, vm, K, c2w, W, H, activated=activated, sh_degree=sh_degree, **kw)


def edge_on_case(n: int, seed: int, **kw) -> Case:
    """Gaussians seen edge-on: the normal (the R(q) column at the smallest scale, evaluated in fp32 as the kernel does)
    is perpendicular to the direction to the camera up to a cosine of 1e-7 (signed, random), and the Gaussian is in
    view.  The forward's flip decision is then a matter of the last bits of its float expression."""
    case = random_case(n, seed, kind="random", **kw)
    g = torch.Generator().manual_seed(seed + 1)
    vm, c2w = case.viewmat, case.c2w
    W, H = case.width, case.height
    fx, fy, cx, cy = (float(case.K[i, j]) for i, j in ((0, 0), (1, 1), (0, 2), (1, 2)))
    z = 1.0 + 4.0 * torch.rand(n, generator=g, dtype=F64)
    u = (torch.rand(n, 2, generator=g, dtype=F64) * 0.8 + 0.1) * torch.tensor([W, H], dtype=F64)
    pc = torch.stack([(u[:, 0] - cx) / fx * z, (u[:, 1] - cy) / fy * z, z], 1)
    m0 = _to_world(vm, pc).double()
    cam = c2w[:, 3].double()
    v0 = cam - m0
    # a rotation whose column `idx` is perpendicular to v0; `idx` is the smallest scale
    idx = torch.randint(0, 3, (n,), generator=g)
    a = torch.nn.functional.normalize(torch.linalg.cross(v0, torch.randn(n, 3, generator=g, dtype=F64)), dim=1)
    b = torch.nn.functional.normalize(torch.linalg.cross(a, torch.randn(n, 3, generator=g, dtype=F64)), dim=1)
    c = torch.linalg.cross(a, b)
    cols = [a, b, c]
    R = torch.empty(n, 3, 3, dtype=F64)
    for k in range(3):
        R[torch.arange(n), :, (idx + k) % 3] = cols[k]
    bad = torch.det(R) < 0
    R[bad] = -R[bad]  # keeps column idx perpendicular
    quats = _rotmat_to_quat(R) * (0.5 + 1.5 * torch.rand(n, 1, generator=g, dtype=F64))
    quats = quats.float()
    s = case.params["scales"].double()
    lo = s.min(1).values
    scales = s.clone()
    for k in range(3):
        scales[:, k] = torch.where(idx == k, lo - 1.0, torch.maximum(s[:, k], lo - 0.5))
    # move the mean along the fp32 normal so that the view direction is perpendicular to it, up to 1e-7
    n32 = _normal32(quats, scales.float()).double()
    cosine = 1e-7 * (2 * torch.rand(n, generator=g, dtype=F64) - 1)
    vn = v0.norm(dim=1, keepdim=True)
    v = v0 - (v0 * n32).sum(1, keepdim=True) * n32 + cosine[:, None] * vn * n32
    means = (cam - v).float()
    case.params.update(means=means, quats=quats, scales=scales.float())
    return case


# ----------------------------------------------------------------------------------------------------- boundaries
BOUNDARY_KINDS = ("depth", "lim", "outside", "radius_clip", "eps2d0", "colour_tie")
BW, BH = 100, 70  # ragged against the 16-pixel tile in both axes


def _up(x: float) -> float:
    return float(torch.nextafter(torch.tensor(x, dtype=F32), torch.tensor(math.inf, dtype=F32)))


def _down(x: float) -> float:
    return float(torch.nextafter(torch.tensor(x, dtype=F32), torch.tensor(-math.inf, dtype=F32)))


def _f32(x: float) -> float:
    return float(torch.tensor(x, dtype=F32))


def _axis_camera(cx: float, cy: float):
    """Rotation I, zero translation, fx = fy = 64, integer principal point: the camera-space mean is the world mean bit
    for bit and mx = 64 x / z + cx is exact for power-of-two z."""
    vm = torch.eye(4, dtype=F32)
    K = torch.tensor([[64.0, 0, cx], [0, 64.0, cy], [0, 0, 1]], dtype=F32)
    c2w = torch.tensor([[1.0, 0, 0, 0], [0, -1.0, 0, 0], [0, 0, -1.0, 0]], dtype=F32)  # get_viewmat(c2w) == I
    return vm, K, c2w


def _radius32(case: Case, means: Tensor, scales: Tensor) -> Tensor:
    """Radii of the fp32 oracle (activated scales, identity rotation) for the case's camera and options, culling by
    the frame and radius_clip ignored: the radius the kernel computes before it decides."""
    q = torch.tensor([[1.0, 0, 0, 0]], dtype=F32).expand(means.shape[0], 4).contiguous()
    K = case.K.clone()
    K[0, 2] += 5e5  # the radius does not depend on the principal point: keep the mean inside a huge frame
    K[1, 2] += 5e5
    p = G.project_gaussians(means, q, scales, case.viewmat, K, 10 ** 6, 10 ** 6, eps2d=case.eps2d,
                            near_plane=case.near_plane, far_plane=case.far_plane, fov_size=(case.width, case.height))
    return p["radii"]


def boundary_case(kind: str) -> tuple:
    """(Case, expect) with Gaussians placed exactly on a branch point of the projection and one fp32 ulp to either side.
    `expect` maps a label to (index, visible, extra) where extra is the branch the placement must take (for "lim": the
    Jacobian clamp flag; for "colour_tie": the channels at colour + 0.5 = 0).  Activated parameters, identity rotations
    unless the branch does not depend on them.

    depth        z = near_plane and far_plane, exactly and one ulp to either side (visible iff near <= z <= far)
    lim          x/z and y/z = +-1.3 tan(fov) exactly (unclamped) and one ulp either side (clamped past it)
    outside      mx + r = 0, mx - r = W, my + r = 0, my - r = H exactly (culled) and one ulp either side; the radius is
                 iterated until it is stable at the placement; the boxes clamp to the frame and end in ragged tiles
    radius_clip  radius = radius_clip (culled) and radius_clip + 1 (visible)
    eps2d0       eps2d = 0: rank-1 covariances (det = 0 exactly: culled) next to full-rank ones (visible)
    colour_tie   SH degree 0 colours at fp32(C0 dc) = -0.5 exactly (colour + 0.5 = 0: the gradient passes)
    """
    expect = {}
    means, scales = [], []

    def add(label, m, s, visible, extra=None):
        expect[label] = (len(means), visible, extra)
        means.append(m)
        scales.append(s)

    cx, cy = (0.0, 0.0) if kind == "outside" else (50.0, 35.0)
    vm, K, c2w = _axis_camera(cx, cy)
    kw = dict(activated=True, normals=True, sh_degree=3, near_plane=0.25, far_plane=8.0)
    if kind == "radius_clip":
        kw["radius_clip"] = 6.0
    if kind == "eps2d0":
        kw["eps2d"] = 0.0
    if kind == "colour_tie":
        kw["sh_degree"] = 0
    probe = Case({}, vm, K, c2w, BW, BH, **kw)
    if kind == "depth":
        for name, zb in (("near", 0.25), ("far", 8.0)):
            for tag, z, vis in (("at", zb, True), ("below", _down(zb), name == "far"), ("above", _up(zb), name == "near")):
                add(f"{name} {tag}", (0.0, 0.0, z), (0.0125 * z,) * 3, vis)
    elif kind == "lim":
        lx, ly = _lims(K, BW, BH)
        for axis, lim in ((0, lx), (1, ly)):
            for sign in (1.0, -1.0):
                for tag, v, clamped in (("at", lim, False), ("past", _up(lim), True), ("inside", _down(lim), False)):
                    m = [0.0, 0.0, 2.0]
                    m[axis] = sign * 2.0 * v  # z = 2: x * (1/z) is v exactly
                    add(f"{'xy'[axis]}{'+' if sign > 0 else '-'} {tag}", tuple(m), (0.35,) * 3, True, clamped)
    elif kind == "outside":
        s = 0.1
        for edge in ("left", "right", "top", "bottom"):
            axis = 0 if edge in ("left", "right") else 1
            size = BW if axis == 0 else BH
            other = (BH if axis == 0 else BW) / 2 / 32.0  # the other coordinate at the frame centre (z = 2)
            r = 0
            for _ in range(8):  # the radius depends on the placement through the Jacobian
                target = -r if edge in ("left", "top") else size + r
                m = [0.0, 0.0, 2.0]
                m[axis], m[1 - axis] = target / 32.0, other
                r_new = int(_radius32(probe, torch.tensor([m], dtype=F32), torch.full((1, 3), s))[0])
                if r_new == r:
                    break
                r = r_new
            target = float(-r if edge in ("left", "top") else size + r)
            inward = _up if edge in ("left", "top") else _down
            outward = _down if edge in ("left", "top") else _up
            for tag, t, vis in (("at", target, False), ("inward", inward(target), True), ("outward", outward(target), False)):
                m = [0.0, 0.0, 2.0]
                m[axis], m[1 - axis] = t / 32.0, other  # 64 (t / 32) * 0.5 + 0 == t exactly
                add(f"{edge} {tag}", tuple(m), (s,) * 3, vis, r)
    elif kind == "radius_clip":
        zs = torch.full((4000, 1), 2.0)
        ss = torch.linspace(0.005, 0.1, 4000)[:, None]
        r = _radius32(probe, torch.cat([torch.zeros(4000, 2), zs], 1), ss.expand(4000, 3).contiguous())
        clip = int(kw["radius_clip"])
        for tag, want, vis in (("at", clip, False), ("above", clip + 1, True), ("below", clip - 1, False)):
            i = int(torch.nonzero(r == want)[0])
            add(f"radius {tag}", (0.0, 0.0, 2.0), (float(ss[i]),) * 3, vis, want)
    elif kind == "eps2d0":
        # identity rotation, one non-zero scale: two of a, b, c are exactly 0 (along z the mean has y = 0, so J12 = 0),
        # hence det = a c - b^2 = 0 exactly
        for j, s in enumerate(((0.1, 0.0, 0.0), (0.0, 0.1, 0.0), (0.0, 0.0, 0.1))):
            add(f"rank1 axis {j}", (0.1 * j, 0.0, 2.0), s, False)
        add("full rank", (0.0, 0.1, 2.0), (0.1, 0.05, 0.02), True)
    elif kind == "colour_tie":
        for j in range(6):
            add(f"tie {j}", (0.1 * (j - 3), 0.05 * j - 0.1, 2.0), (0.05, 0.04, 0.03), True, (j % 3,))
    else:
        raise ValueError(kind)
    n = len(means)
    g = torch.Generator().manual_seed(BOUNDARY_KINDS.index(kind))
    quats = torch.tensor([[1.0, 0, 0, 0]]).repeat(n, 1)
    if kind in ("depth", "lim"):  # the branch does not depend on the rotation
        quats = torch.randn(n, 4, generator=g)
    dc = 0.5 * torch.randn(n, 3, generator=g)
    if kind == "colour_tie":
        c0 = torch.tensor(SH_C0_F32, dtype=F32)
        tie = _colour_tie_dc()
        for i, _, chans in expect.values():
            for c in chans:
                dc[i, c] = tie
                assert float(c0 * dc[i, c].float()) == -0.5
    params = dict(means=torch.tensor(means, dtype=F32), quats=quats.float().contiguous(),
                  scales=torch.tensor(scales, dtype=F32), opacities=torch.full((n,), 0.7),
                  sh_dc=dc.float(), sh_rest=(0.3 * torch.randn(n, 15, 3, generator=g)).float())
    return Case(params, vm, K, c2w, BW, BH, **kw), expect


SH_C0_F32 = 0.2820947917738781


def _colour_tie_dc() -> float:
    """An fp32 dc with fp32(C0 * dc) == -0.5 exactly (C0 rounded to fp32, as the kernel's literal)."""
    c0 = torch.tensor(SH_C0_F32, dtype=F32)
    x = torch.tensor(-0.5 / SH_C0_F32, dtype=F32)
    for _ in range(64):
        p = float(c0 * x)
        if p == -0.5:
            return float(x)
        x = torch.nextafter(x, torch.tensor(0.0 if p < -0.5 else -1.0, dtype=F32))
    raise AssertionError("no fp32 dc ties the colour at -0.5")


def _rotmat_to_quat(R: Tensor) -> Tensor:
    """wxyz unit quaternions of rotation matrices [N,3,3] (float64): the dominant eigenvector of Bar-Itzhack's
    symmetric 4 x 4 matrix, which is exact for a rotation and needs no case split."""
    r = lambda i, j: R[:, i, j]  # noqa: E731
    Km = torch.stack([
        torch.stack([r(0, 0) - r(1, 1) - r(2, 2), r(1, 0) + r(0, 1), r(2, 0) + r(0, 2), r(2, 1) - r(1, 2)], 1),
        torch.stack([r(1, 0) + r(0, 1), r(1, 1) - r(0, 0) - r(2, 2), r(2, 1) + r(1, 2), r(0, 2) - r(2, 0)], 1),
        torch.stack([r(2, 0) + r(0, 2), r(2, 1) + r(1, 2), r(2, 2) - r(0, 0) - r(1, 1), r(1, 0) - r(0, 1)], 1),
        torch.stack([r(2, 1) - r(1, 2), r(0, 2) - r(2, 0), r(1, 0) - r(0, 1), r(0, 0) + r(1, 1) + r(2, 2)], 1)], 1) / 3
    xyzw = torch.linalg.eigh(Km)[1][:, :, -1]
    q = torch.cat([xyzw[:, 3:], xyzw[:, :3]], 1)
    assert float((G.quat_to_rotmat(q) - R).abs().max()) < 1e-9, "not a rotation"
    return q


def _normal32(quats: Tensor, scales: Tensor) -> Tensor:
    """The kernel's unit normal before the flip, in fp32 and its operation order."""
    R = G.quat_to_rotmat_entries(quats.float())
    idx = _argmin3(scales.float())
    n = [torch.where(idx == 0, R[r][0], torch.where(idx == 1, R[r][1], R[r][2])) for r in range(3)]
    nn = torch.clamp(torch.sqrt((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2]), min=1e-12)
    return torch.stack([n[k] / nn for k in range(3)], 1)


def _argmin3(s: Tensor) -> Tensor:
    """argmin3 of project.cu: the first index of the smallest value (strict <), like torch.argmin."""
    idx = torch.zeros(s.shape[0], dtype=torch.long)
    m = s[:, 0].clone()
    lt1 = s[:, 1] < m
    idx[lt1] = 1
    m = torch.where(lt1, s[:, 1], m)
    idx[s[:, 2] < m] = 2
    return idx


# ----------------------------------------------------------------------------------------------------- branches
@dataclass
class Branches:
    """Per-Gaussian decisions the kernel takes in fp32 where the projection is not differentiable."""

    clamp_x: Tensor  # bool [N]
    clamp_y: Tensor
    color_pass: Tensor  # bool [N,3]: colour + 0.5 >= 0
    comp_pos: Tensor  # bool [N]: compensation > 0
    flip: Tensor  # bool [N]: the forward negates the normal
    flip_bwd: Tensor  # bool [N]: the decision the backward took before it shared the forward's expression
    lim_x: float
    lim_y: float

    @staticmethod
    def from_fp32(case: Case, flip: Optional[Tensor] = None, comp_pos: Optional[Tensor] = None) -> "Branches":
        """The kernel's decisions, emulated in fp32 in its operation order (torch on the CPU rounds each operation
        like the kernel built with -fmad=false).  `flip` / `comp_pos` override the emulation with the kernel's own
        outputs (its normals_world and compensations)."""
        p = {k: v.float() for k, v in case.params.items()}
        vm = case.viewmat.float()
        Wm = [[vm[i, j] for j in range(3)] for i in range(3)]
        t = [vm[i, 3] for i in range(3)]
        px, py, pz = p["means"].unbind(1)
        x = G._dot3(Wm[0][0], px, Wm[0][1], py, Wm[0][2], pz) + t[0]
        y = G._dot3(Wm[1][0], px, Wm[1][1], py, Wm[1][2], pz) + t[1]
        z = G._dot3(Wm[2][0], px, Wm[2][1], py, Wm[2][2], pz) + t[2]
        ok = (z >= case.near_plane) & (z <= case.far_plane)
        zs = torch.where(ok, z, torch.ones_like(z))
        rz = 1.0 / zs
        lx, ly = _lims(case.K, case.width, case.height)
        xr, yr = x * rz, y * rz
        clamp_x = ~((xr <= lx) & (xr >= -lx))
        clamp_y = ~((yr <= ly) & (yr >= -ly))
        col = colors32(case)
        if comp_pos is None:
            s = p["scales"] if case.activated else torch.exp(p["scales"])
            proj = G.project_gaussians(p["means"], p["quats"], s, vm, case.K.float(), case.width, case.height,
                                       eps2d=case.eps2d, near_plane=case.near_plane, far_plane=case.far_plane)
            comp_pos = proj["compensations"] > 0
        nu = _normal32(p["quats"], p["scales"])
        c2wT = case.c2w[:, 3].float()
        vd = [c2wT[k] - p["means"][:, k] for k in range(3)]
        vn = torch.sqrt((vd[0] * vd[0] + vd[1] * vd[1]) + vd[2] * vd[2])
        d_fwd = (nu[:, 0] * (vd[0] / vn) + nu[:, 1] * (vd[1] / vn)) + nu[:, 2] * (vd[2] / vn)
        d_bwd = (nu[:, 0] * vd[0] + nu[:, 1] * vd[1]) + nu[:, 2] * vd[2]
        return Branches(clamp_x, clamp_y, col + 0.5 >= 0, comp_pos.bool(), d_fwd < 0 if flip is None else flip.bool(),
                        d_bwd < 0, lx, ly)


def _sh_basis32(deg: int, x: Tensor, y: Tensor, z: Tensor):
    """sh_basis of project.cu in fp32: the 16 basis values (zeros above `deg`)."""
    f = lambda c: float(torch.tensor(c, dtype=F32))  # noqa: E731  the kernel's fp32 literals
    zero = torch.zeros_like(x)
    b = [torch.full_like(x, f(0.2820947917738781))] + [zero] * 15
    if deg < 1:
        return b
    b[1] = f(-0.48860251190292) * y
    b[2] = f(0.48860251190292) * z
    b[3] = f(-0.48860251190292) * x
    if deg < 2:
        return b
    z2 = z * z
    t0b = f(-1.092548430592079) * z
    fc1 = x * x - y * y
    fs1 = 2.0 * x * y
    b[6] = f(0.9461746957575601) * z2 - f(0.3153915652525201)
    b[7] = t0b * x
    b[5] = t0b * y
    b[8] = f(0.5462742152960395) * fc1
    b[4] = f(0.5462742152960395) * fs1
    if deg < 3:
        return b
    t0c = f(-2.285228997322329) * z2 + f(0.4570457994644658)
    t1b = f(1.445305721320277) * z
    fc2 = x * fc1 - y * fs1
    fs2 = x * fs1 + y * fc1
    b[12] = z * (f(1.865881662950577) * z2 - f(1.119528997770346))
    b[13] = t0c * x
    b[11] = t0c * y
    b[14] = t1b * fc1
    b[10] = t1b * fs1
    b[15] = f(-0.5900435899266435) * fc2
    b[9] = f(-0.5900435899266435) * fs2
    return b


def colors32(case: Case) -> Tensor:
    """The kernel's pre-clamp SH colour [N,3] in fp32 and its operation order."""
    p = {k: v.float() for k, v in case.params.items()}
    vm = case.viewmat.float()
    Wm = [[vm[i, j] for j in range(3)] for i in range(3)]
    t = [vm[i, 3] for i in range(3)]
    campos = [-((Wm[0][j] * t[0] + Wm[1][j] * t[1]) + Wm[2][j] * t[2]) for j in range(3)]
    d = [p["means"][:, k] - campos[k] for k in range(3)]
    deg = case.sh_degree
    if deg > 0:
        inorm = 1.0 / torch.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])
        b = _sh_basis32(deg, d[0] * inorm, d[1] * inorm, d[2] * inorm)
    else:
        b = _sh_basis32(0, d[0], d[1], d[2])
    col = b[0][:, None] * p["sh_dc"]
    for k in range(1, (deg + 1) ** 2):
        col = col + b[k][:, None] * p["sh_rest"][:, k - 1]
    return col


# ----------------------------------------------------------------------------------------------------- float64
def forward64(case: Case, br: Branches, p: Optional[Dict[str, Tensor]] = None, viewmat: Optional[Tensor] = None,
              slip: Optional[str] = None) -> Dict[str, Tensor]:
    """The projection's float outputs per Gaussian in float64 (of `p` / `viewmat` when given, e.g. leaves that require
    grad): means2d [N,2], conics [N,3], opac [N], rgb [N,3], depth [N], comp [N], normals_world / ncam [N,3]."""
    if p is None:
        p = {k: v.double() for k, v in case.params.items()}
    vm = case.viewmat.double() if viewmat is None else viewmat
    s = p["scales"] if case.activated else torch.exp(p["scales"])
    o = p["opacities"] if case.activated else torch.sigmoid(p["opacities"])
    Wm, t = vm[:3, :3], vm[:3, 3]
    mc = p["means"] @ Wm.T + t
    x, y, z = mc.unbind(1)
    M = G.quat_to_rotmat(p["quats"]) * s[:, None, :]
    Sc = Wm @ (M @ M.transpose(1, 2)) @ Wm.T
    if case.cov_noise is not None:
        Sc = Sc + case.cov_noise * Sc.abs().amax((1, 2), keepdim=True)
    K = case.K.double()
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    tx_c = z * torch.clamp(x / z, -br.lim_x, br.lim_x)
    ty_c = z * torch.clamp(y / z, -br.lim_y, br.lim_y)
    if slip == "clamp_z":  # the clamped branch's dependence of J on z dropped
        tx_c = torch.where(br.clamp_x, z.detach() * torch.sign(x) * br.lim_x, tx_c)
        ty_c = torch.where(br.clamp_y, z.detach() * torch.sign(y) * br.lim_y, ty_c)
    tx = torch.where(br.clamp_x, tx_c, x)
    ty = torch.where(br.clamp_y, ty_c, y)
    zero = torch.zeros_like(z)
    J = torch.stack([torch.stack([fx / z, zero, -fx * tx / (z * z)], 1),
                     torch.stack([zero, fy / z, -fy * ty / (z * z)], 1)], 1)
    cov = J @ Sc @ J.transpose(1, 2)
    a, b, c = cov[:, 0, 0], cov[:, 0, 1], cov[:, 1, 1]
    det_orig = a * c - b * b
    ab, cb = a + case.eps2d, c + case.eps2d
    det = ab * cb - b * b
    # a rank-deficient covariance has det_orig of rounding size: fp32 may find it > 0 where fp64 does not (and vice
    # versa); the reference then has no compensation (and no gradient) there, and the caller compares no such Gaussian
    pos = br.comp_pos & (det_orig > 0)
    ratio = torch.where(pos, det_orig / det, torch.ones_like(det))
    comp = torch.where(pos, torch.sqrt(ratio), zero)
    if slip == "comp":  # the compensation's gradient dropped
        comp = comp.detach()
    op = o * comp if case.antialiased else o
    conics = torch.stack([cb / det, -b / det, ab / det], 1)
    means2d = torch.stack([fx * x / z + cx, fy * y / z + cy], 1)
    campos = -(Wm.T @ t)
    dirs = p["means"] - campos
    u = dirs / dirs.norm(dim=1, keepdim=True)
    if slip == "inorm":  # d(dir/|dir|)/d(dir) without its 1/|dir|
        dd = dirs - dirs.detach()
        ud = u.detach()
        u = ud + (dd - ud * (dd * ud).sum(1, keepdim=True))
    deg = case.sh_degree
    coeffs = torch.cat([p["sh_dc"][:, None], p["sh_rest"][:, :(deg + 1) ** 2 - 1]], 1)
    col = G.eval_sh(deg, u, coeffs) + 0.5
    rgb = torch.where(br.color_pass, col, torch.zeros_like(col))
    out = dict(means2d=means2d, conics=conics, opac=op, rgb=rgb, depth=z, comp=comp)
    if case.normals:
        q = p["quats"] / p["quats"].norm(dim=1, keepdim=True)
        R = G.quat_to_rotmat(q)
        idx = _argmin3(case.params["scales"].float())
        n = R[torch.arange(R.shape[0]), :, idx]
        n = n / n.norm(dim=1, keepdim=True).clamp(min=1e-12)
        flip = br.flip_bwd if slip == "flip_bwd" else br.flip
        nw = torch.where(flip[:, None], -n, n)
        out["normals_world"] = nw
        out["ncam"] = nw @ case.c2w[:, :3].double()
    return out


def vjp64(case: Case, br: Branches, grad_records: Tensor, rows: Tensor, viewmat: bool = False,
          slip: Optional[str] = None) -> Dict[str, Tensor]:
    """d/d(params) of sum over `rows` (bool [N]) of grad_records . outputs, in float64, with the record layout
    dnr_project_bwd reads: g0 = (v_mx, v_my, abs_x, abs_y), g1 = (v_A, v_B, v_C, v_opac), g2 = (v_rgb, v_z),
    g3 = (v_ncam, unused).  Also v_means2d / v_means2d_abs (the record's slots, on `rows`) and, with `viewmat`,
    v_viewmat [4,4]."""
    p = {k: v.detach().double().requires_grad_(True) for k, v in case.params.items()}
    vm = case.viewmat.detach().double().requires_grad_(viewmat)
    out = forward64(case, br, p, vm, slip=slip)
    g = torch.where(rows[:, None], grad_records.double(), torch.zeros((), dtype=F64))
    loss = (g[:, 0:2] * out["means2d"]).sum() + (g[:, 4:7] * out["conics"]).sum() + (g[:, 7] * out["opac"]).sum()
    loss = loss + (g[:, 8:11] * out["rgb"]).sum() + (g[:, 11] * out["depth"]).sum()
    if case.normals:
        loss = loss + (g[:, 12:15] * out["ncam"]).sum()
    leaves = [p[k] for k in PARAM_KEYS] + ([vm] if viewmat else [])
    gs = torch.autograd.grad(loss, leaves, allow_unused=True)
    res = {k: torch.zeros_like(p[k]) if gg is None else gg for k, gg in zip(PARAM_KEYS, gs)}
    if viewmat:
        res["viewmat"] = gs[-1]
    m2, m2a = g[:, 0:2], g[:, 2:4]
    if slip == "abs_swap":
        m2, m2a = m2a, m2
    res["means2d"], res["means2d_abs"] = m2, m2a
    return res


# ----------------------------------------------------------------------------------------------------- tolerances
# Per Gaussian and parameter group (a row):
#   max |g - g64| <= RTOL max|g64 row| + ATOL max|g64 of the group| + SENS max|spread row|
# where `spread` is how far the fp64 result itself moves when every input (parameters and camera) is perturbed by a
# relative DELTA (three random draws): the part of the error an fp32 evaluation cannot avoid.  It is large only where
# the problem is ill-conditioned (needles, compensation near 1, cancelling terms) and ~RTOL-sized elsewhere, so a wrong
# term that reaches a well-conditioned Gaussian fails.  The perturbation includes the camera covariance itself (see
# `perturbed`).  SENS is per kind (gradients / forward floats), mode (classic / antialiased) and output group, with
# needles (cond(cov2d) > 1e3) apart.  The factors each row needed over every case of tests/test_gpu_projection.py are
# in the comments; the bounds keep 3.7x or more headroom.
DELTA = 1e-5
GRAD_RTOL, GRAD_ATOL, FWD_RTOL = 2e-5, 1e-7, 2e-5
_ALL = ("means", "quats", "scales", "opacities", "sh_dc", "sh_rest", "viewmat", "means2d", "depth", "rgb", "ncam",
        "normals_world", "conics", "opac", "comp")
SENS = {  # (kind, mode) -> group -> factor; needed on an H100 80GB HBM3 (700 W limit) over every case:
    # gradients, classic: < 0.7 everywhere
    ("grad", "classic"): dict.fromkeys(_ALL, 4.0),
    # gradients, antialiased: v_scales 104 (Jacobian-clamped scene), every other group < 0.5
    ("grad", "antialiased"): {**dict.fromkeys(_ALL, 4.0), "scales": 400.0},
    # forward floats: < 0.5 everywhere, both modes
    ("fwd", "classic"): dict.fromkeys(_ALL, 4.0),
    ("fwd", "antialiased"): dict.fromkeys(_ALL, 4.0),
}
NEEDLE_SENS = {  # needles, every group: needed 0.64 / 24.5 (v_scales, v_opacities) / < 0.5 / 10.7 (compensation)
    ("grad", "classic"): 4.0, ("grad", "antialiased"): 100.0, ("fwd", "classic"): 4.0, ("fwd", "antialiased"): 40.0}


def _mode(case: Case) -> str:
    return "antialiased" if case.antialiased else "classic"


def sens(kind: str, case: Case) -> Dict[str, float]:
    return SENS[(kind, _mode(case))]


def needle_sens(kind: str, case: Case) -> float:
    return NEEDLE_SENS[(kind, _mode(case))]


def perturbed(case: Case, seed: int, delta: float = DELTA) -> Case:
    """The case with every float input scaled by 1 + delta u, u ~ U(-1, 1), in float64, and the camera covariance Sc
    moved by delta max|Sc| U(-1, 1) (symmetric): an fp32 evaluation rounds Sc's entries on the scale of its largest,
    which no relative change of the inputs reproduces where Sc is (near) rank-deficient."""
    g = torch.Generator().manual_seed(seed)
    u = lambda *s: 2 * torch.rand(*s, generator=g, dtype=F64) - 1  # noqa: E731
    f = lambda t: t.double() * (1 + delta * u(*t.shape))  # noqa: E731
    e = delta * u(case.n, 3, 3)
    return Case({k: f(v) for k, v in case.params.items()}, f(case.viewmat), f(case.K), f(case.c2w), case.width,
                case.height, case.activated, case.antialiased, case.normals, case.sh_degree, case.eps2d,
                case.near_plane, case.far_plane, case.radius_clip, (e + e.transpose(1, 2)) / 2)


def spread(fn, case: Case, trials: int = 3) -> Dict[str, Tensor]:
    """Elementwise max over `trials` perturbed cases of |fn(perturbed) - fn(case)| for a dict-valued fn."""
    base = fn(case)
    out = {k: torch.zeros_like(v) for k, v in base.items()}
    for s in range(trials):
        other = fn(perturbed(case, seed=1000 + s))
        for k in out:
            out[k] = torch.maximum(out[k], (other[k] - base[k]).abs().nan_to_num(nan=math.inf))
    return out


def row_ratio(got: Tensor, want: Tensor, spr: Tensor, rows: Tensor, rtol: float, atol: float, sens: float) -> Tensor:
    """Per row: max |got - want| / (rtol max|want row| + atol max|want over rows| + sens max|spread row|); 0 outside
    `rows`, inf for a non-finite kernel value."""
    n = got.shape[0]
    g, w, s = got.double().reshape(n, -1), want.double().reshape(n, -1), spr.double().reshape(n, -1)
    if w.shape[1] == 0:  # an empty group (sh_rest with one stored basis)
        return torch.zeros(n, dtype=F64)
    gmax = float(w[rows].abs().max()) if bool(rows.any()) else 0.0
    bound = rtol * w.abs().amax(1) + atol * gmax + sens * s.amax(1)
    err = (g - w).abs().amax(1)
    r = torch.where(err == 0, torch.zeros_like(err), err / bound.clamp(min=1e-300))
    r = torch.where(torch.isfinite(g).all(1), r, torch.full_like(r, math.inf))
    return torch.where(rows, r, torch.zeros_like(r))


def needles(case: Case) -> Tensor:
    """bool [N]: the 2-D covariance (before the blur) has a condition number above 1e3."""
    br = Branches.from_fp32(case)
    with torch.no_grad():
        out = forward64(case, br)
        A, B, C = out["conics"].unbind(1)
    ev = torch.stack([(A + C) / 2 - torch.sqrt(((A - C) / 2) ** 2 + B * B), (A + C) / 2 + torch.sqrt(((A - C) / 2) ** 2 + B * B)], 1)
    cond = (ev[:, 1] / ev[:, 0].clamp(min=1e-300)).abs()
    return cond > 1e3
