"""ORACLE (test infrastructure, NOT product code): fp64 per-pixel compositor for `raster_fwd_kernel` (csrc/raster.cu) that
reports the margins of its own decisions.

Written from the rules stated in oracle/gsplat_ref.py and DESIGN.md, not from any source: front to back over a tile's
list, an entry is skipped when sigma < 0 or alpha = min(op * exp(-sigma), 0.999) < 1/255, the pixel stops BEFORE
accumulating the entry that would take T * (1 - alpha) to 1e-4 or below; seven channels (rgb, depth, camera-space
normal); `last_id` is the position in `flatten_ids` of the last composited entry (0 when none); then the kernel's
epilogue: rgb = clamp(C + T bg), the clamp mask, expected depth D / max(alpha, 1e-10), the normal image with its white
background term + T normalised into [0, 1], |n|, and the frame-wide maximum of the expected depth.

The inputs are what the kernel reads (per-Gaussian 2-D means, conics, opacities, colours, depths, camera-space normals,
radii, and the sorted lists), so a comparison with the kernel does not go through projection or binning.  Every 16 x 16
tile walks the list of its supertile of (16 << list_shift)^2 pixels and composites an entry only if the tile lies in
the entry's gsplat tile box (`dnr_tile_box` of the 3-sigma radius), which is evaluated in fp32 with the kernel's
operations; the kernel's precise tile-hit filter is NOT restated: it may only drop entries no pixel of the tile
composites, and a comparison against this oracle is what checks that.

The three thresholds are the kernel's fp32 constants (0.999f is 1.3e-8 above 0.999, which is 1.3e-5 of 1 - alpha).

Margins.  For every pixel, `margin` is the smallest relative distance to its threshold of any decision taken on the way
(entries up to and including the one the pixel stopped at): sigma against 0 (relative to the sum of the absolute
terms of the quadratic form), alpha against 1/255, and T (1 - alpha) against 1e-4, the last divided by 1 + kappa with
kappa = sum alpha_i / (1 - alpha_i) over the entries composited so far: a relative error d in every alpha moves T by
kappa d, which is far more than d behind a nearly opaque splat.  `margin_pos` / `margin_kind` say which entry and which
test.  The clamp min(., 0.999) is continuous and the tile box is evaluated exactly as the kernel does, so neither makes
a pixel ambiguous; their distances are reported on their own (`clamp_margin`, `box_margin`) for tests that must show
they reach those branches.  With eps > 0, every pixel with margin < eps gets the list of outcomes obtained by taking
each decision within eps of its threshold either way (`alts[(i, j)]`, primary outcome first), found by a scalar walk that
branches at such decisions; pixels with more than `max_alts` outcomes are listed in `unresolved` instead.

`slip=` restates, in fp64, mistakes a kernel could make (SLIPS); tests/test_raster_ref_cpu.py uses them to show that the
acceptance rule `judge` separates each of them from the correct result.

`backward` differentiates `composite` at its own decisions with the conventions of `raster_bwd_kernel` and returns, per
Gaussian, the 16 floats of a `grad_records` row with their absolute mass; `judge_bwd` is the per-Gaussian acceptance rule
of tests/test_gpu_raster_backward.py, and BWD_SLIPS the backward mistakes tests/test_raster_bwd_ref_cpu.py holds it to.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

TILE = 16
F32 = np.float32
ALPHA_MIN = float(F32(1.0) / F32(255.0))
ALPHA_MAX = float(F32(0.999))
T_STOP = float(F32(1e-4))
KIND_SIGMA, KIND_ALPHA, KIND_STOP = 0, 1, 2
KINDS = ("sigma vs 0", "alpha vs 1/255", "T (1 - alpha) vs 1e-4")

# kernel mistakes restated in fp64 (what each one would be in raster.cu / project.cu is in the docstrings below)
SLIPS = (
    "pretest_slack",    # record slot nthr = -log2(255 op) + 1e-3: entries with alpha in [1/255, 2^1e-3 / 255) are dropped
    "stop_after",       # the stop rule tests T instead of T (1 - alpha): the stopping entry is accumulated first
    "last_partner",     # the lower pixel of a lane's pair (row + 4 of an 8 x 8 patch) records the upper pixel's last_id
    "no_white",         # the + T white-background term of the normal image is dropped
    "depth_eps",        # expected depth D / (alpha + 1e-10) instead of D / max(alpha, 1e-10)
    "stale_depth_max",  # depth_max is not reset: it keeps the maximum of an earlier, deeper frame (`stale_depth_max=`)
)


def _np64(t) -> np.ndarray:
    if isinstance(t, torch.Tensor):
        t = t.detach().cpu().numpy()
    return np.asarray(t, dtype=np.float64)


@dataclass
class RasterRef:
    """Outputs of `composite`: images as numpy arrays over the frame (pixels of tiles that were not requested are zero)."""

    rgb: np.ndarray          # [H,W,3] clamped
    rgb_pre: np.ndarray      # [H,W,3] before the clamp
    clamp_mask: np.ndarray   # [H,W] uint8, bit k: channel k lies in [0, 1] before the clamp
    depth: np.ndarray        # [H,W] expected depth (not filled)
    alpha: np.ndarray        # [H,W]
    normal: np.ndarray       # [H,W,3] (n / |n| + 1) / 2, zeros without normals
    normal_norm: np.ndarray  # [H,W]
    last_ids: np.ndarray     # [H,W] int64
    depth_max: float
    sums: np.ndarray         # [H,W,7] premultiplied sums C, D, N (before background terms)
    T: np.ndarray            # [H,W]
    mass: np.ndarray         # [H,W,7] sum_i w_i |feat_i| (+ T |bg| for rgb, + T for the normal): the scale of the sums
    ncomp: np.ndarray        # [H,W] entries composited
    margin: np.ndarray       # [H,W]
    margin_pos: np.ndarray   # [H,W] list position of the decision closest to its threshold (-1: no decision taken)
    margin_kind: np.ndarray  # [H,W] KIND_*
    clamp_margin: np.ndarray  # [H,W] min |op vis / 0.999 - 1| over composited entries
    box_margin: float        # min distance (in tiles) of a listed entry's m +- r to a tile boundary
    stopped: np.ndarray      # [H,W] bool: the pixel stopped under the T rule
    clamped: np.ndarray      # [H,W] bool: the pixel composited an entry with op vis > 0.999
    n_contrib: int           # (tile, entry) pairs composited by at least one pixel of the tile
    n_listed: int            # (tile, entry) pairs walked
    done: np.ndarray         # [H,W] bool: pixels of requested tiles
    normals: bool
    alts: Dict[Tuple[int, int], List[dict]] = field(default_factory=dict)
    unresolved: List[Tuple[int, int]] = field(default_factory=list)

    def report(self, i: int, j: int) -> str:
        k = int(self.margin_kind[i, j])
        return (f"pixel ({i}, {j}): margin {self.margin[i, j]:.3e} ({KINDS[k]} at list position {int(self.margin_pos[i, j])}), "
                f"{int(self.ncomp[i, j])} composited, last_id {int(self.last_ids[i, j])}, alpha {self.alpha[i, j]:.9g}, "
                f"stopped {bool(self.stopped[i, j])}, alternatives {len(self.alts.get((i, j), []))}")


def epilogue(T, sums, background, normals: bool, slip: Optional[str] = None) -> dict:
    """The kernel's epilogue on arrays [..., ] T and [..., 7] sums."""
    bg = np.asarray(background, dtype=np.float64)
    alpha = 1.0 - T
    pre = sums[..., 0:3] + T[..., None] * bg
    mask = np.zeros(T.shape, dtype=np.uint8)
    for k in range(3):
        mask |= (((pre[..., k] >= 0.0) & (pre[..., k] <= 1.0)).astype(np.uint8) << k)
    den = alpha + 1e-10 if slip == "depth_eps" else np.maximum(alpha, 1e-10)
    out = dict(rgb=np.clip(pre, 0.0, 1.0), rgb_pre=pre, clamp_mask=mask, depth=sums[..., 3] / den, alpha=alpha)
    if normals:
        n = sums[..., 4:7] + (0.0 if slip == "no_white" else T[..., None])
        nn = np.sqrt((n * n).sum(-1))
        with np.errstate(invalid="ignore", divide="ignore"):
            out["normal"] = (n / nn[..., None] + 1.0) * 0.5
        out["normal_norm"] = nn
    else:
        out["normal"] = np.zeros(T.shape + (3,))
        out["normal_norm"] = np.zeros(T.shape)
    return out


def tile_box(means2d, radii):
    """gsplat's tile box per Gaussian in fp32, before the clamp to the frame: (x0, y0, x1, y1), max exclusive, and the
    distance of each of the four m +- r (in tiles) to the nearest integer."""
    m = np.asarray(means2d.detach().cpu().numpy() if isinstance(means2d, torch.Tensor) else means2d).astype(F32)
    rad = np.asarray(radii.detach().cpu().numpy() if isinstance(radii, torch.Tensor) else radii).astype(F32)
    s = F32(1.0 / TILE)
    r, tcx, tcy = rad * s, m[:, 0] * s, m[:, 1] * s
    lo_x, hi_x, lo_y, hi_y = tcx - r, tcx + r, tcy - r, tcy + r  # fp32 roundings, as dnr_in_tile_box
    edges = np.stack([lo_x, hi_x, lo_y, hi_y], 1).astype(np.float64)
    dist = np.abs(edges - np.round(edges)).min(1)
    return np.floor(lo_x), np.floor(lo_y), np.ceil(hi_x), np.ceil(hi_y), dist


def composite(means2d, conics, opacities, colors, depths, normals_cam, radii, flatten_ids, tile_offsets, list_shift: int,
              width: int, height: int, background: Sequence[float], *, eps: float = 0.0, max_alts: int = 8,
              slip: Optional[str] = None, stale_depth_max: float = 0.0, tiles: Optional[Sequence[Tuple[int, int]]] = None,
              chunk: int = 512, keep: Optional[dict] = None) -> RasterRef:
    """See the module docstring.  `tiles`: [(tx, ty)] restricts the work to those 16 x 16 tiles.  `keep`: a dict that
    receives, per walked tile (tx, ty), (y0, y1, x0, x1, g, pos, live[P,K], alpha[P,K], vis[P,K], dx[P,K], dy[P,K]) over
    the K entries some pixel of the tile composited, in list order (`backward` differentiates exactly these)."""
    if slip is not None and slip not in SLIPS:
        raise ValueError(slip)
    m2, con, op = _np64(means2d), _np64(conics), _np64(opacities).reshape(-1)
    normals = normals_cam is not None
    feats = np.concatenate([_np64(colors), _np64(depths).reshape(-1, 1),
                            _np64(normals_cam) if normals else np.zeros((m2.shape[0], 3))], 1)
    ids = np.asarray(flatten_ids.detach().cpu().numpy() if isinstance(flatten_ids, torch.Tensor) else flatten_ids).astype(np.int64)
    offs = np.asarray(tile_offsets.detach().cpu().numpy() if isinstance(tile_offsets, torch.Tensor) else tile_offsets).astype(np.int64)
    bx0, by0, bx1, by1, bdist = tile_box(means2d, radii)
    H, W = height, width
    tiles_x, tiles_y = -(-W // TILE), -(-H // TILE)
    stiles_x = -(-W // (TILE << list_shift))
    ref = RasterRef(rgb=None, rgb_pre=None, clamp_mask=None, depth=None, alpha=None, normal=None, normal_norm=None,
                    last_ids=np.zeros((H, W), np.int64), depth_max=0.0, sums=np.zeros((H, W, 7)), T=np.ones((H, W)),
                    mass=np.zeros((H, W, 7)), ncomp=np.zeros((H, W), np.int64), margin=np.full((H, W), np.inf),
                    margin_pos=np.full((H, W), -1, np.int64), margin_kind=np.zeros((H, W), np.int64),
                    clamp_margin=np.full((H, W), np.inf), box_margin=math.inf, stopped=np.zeros((H, W), bool),
                    clamped=np.zeros((H, W), bool), n_contrib=0,
                    n_listed=0, done=np.zeros((H, W), bool), normals=normals)
    alpha_min = ALPHA_MIN * 2.0 ** 1e-3 if slip == "pretest_slack" else ALPHA_MIN
    ambiguous = []  # (i, j, tx, ty)
    for ty in range(tiles_y):
        for tx in range(tiles_x):
            if tiles is not None and (tx, ty) not in tiles:
                continue
            y0, x0 = ty * TILE, tx * TILE
            y1, x1 = min(y0 + TILE, H), min(x0 + TILE, W)
            ref.done[y0:y1, x0:x1] = True
            st = (ty >> list_shift) * stiles_x + (tx >> list_shift)
            lo, hi = int(offs[st]), int(offs[st + 1])
            if hi <= lo:
                continue
            g_all = ids[lo:hi]
            ref.n_listed += hi - lo
            ref.box_margin = min(ref.box_margin, float(bdist[g_all].min()))
            inbox = (tx >= bx0[g_all]) & (tx < bx1[g_all]) & (ty >= by0[g_all]) & (ty < by1[g_all])
            pos_all = np.arange(lo, hi)[inbox]
            g_all = g_all[inbox]
            h, w_ = y1 - y0, x1 - x0
            P = h * w_
            py = np.repeat(np.arange(y0, y1) + 0.5, w_)
            px = np.tile(np.arange(x0, x1) + 0.5, h)
            T = np.ones(P)
            kap = np.zeros(P)
            fin = np.zeros(P, bool)  # stopped
            acc, mass = np.zeros((P, 7)), np.zeros((P, 7))
            last, ncomp = np.zeros(P, np.int64), np.zeros(P, np.int64)
            marg, mpos, mkind = np.full(P, np.inf), np.full(P, -1, np.int64), np.zeros(P, np.int64)
            cmarg = np.full(P, np.inf)
            clamped = np.zeros(P, bool)
            used = np.zeros(g_all.shape[0], bool)
            kept = []
            for s in range(0, g_all.shape[0], chunk):
                if fin.all():
                    break
                g = g_all[s:s + chunk]
                pos = pos_all[s:s + chunk]
                dx = m2[g, 0][None, :] - px[:, None]
                dy = m2[g, 1][None, :] - py[:, None]
                t0, t1, t2 = 0.5 * con[g, 0][None] * dx * dx, 0.5 * con[g, 2][None] * dy * dy, con[g, 1][None] * dx * dy
                sigma = (t0 + t1) + t2
                vis = np.exp(-sigma)
                ov = op[g][None, :] * vis
                alpha = np.minimum(ov, ALPHA_MAX)
                valid = (sigma >= 0) & (alpha >= alpha_min)
                a_eff = np.where(valid, alpha, 0.0)
                cp = np.cumprod(np.concatenate([T[:, None], 1.0 - a_eff], 1), 1)
                T_before, T_after = cp[:, :-1], cp[:, 1:]
                kap_after = kap[:, None] + np.cumsum(a_eff / (1.0 - a_eff), 1)
                stop = valid & ((T_before if slip == "stop_after" else T_after) <= T_STOP)
                stopped_incl = np.maximum.accumulate(stop, 1)
                stopped_excl = np.concatenate([np.zeros((P, 1), bool), stopped_incl[:, :-1]], 1)
                reached = ~stopped_excl & ~fin[:, None]
                live = valid & ~stopped_incl & ~fin[:, None]
                wgt = np.where(live, a_eff * T_before, 0.0)
                acc += wgt @ feats[g]
                mass += wgt @ np.abs(feats[g])
                ncomp += live.sum(1)
                cand = np.where(live, pos[None, :], -1).max(1)
                last = np.where(cand >= 0, cand, last)
                used[s:s + chunk] |= live.any(0)
                if keep is not None:
                    cols = live.any(0)
                    kept.append((g[cols], pos[cols], live[:, cols], alpha[:, cols], vis[:, cols], dx[:, cols], dy[:, cols]))
                # margins of the decisions taken on the entries the pixel reached
                den = np.abs(t0) + np.abs(t1) + np.abs(t2)
                with np.errstate(invalid="ignore", divide="ignore"):
                    m_sig = np.where(den > 0, np.abs(sigma) / den, np.inf)
                    m_alp = np.where(sigma >= 0, np.abs(alpha / ALPHA_MIN - 1.0), np.inf)
                    m_stp = np.where(valid, np.abs(T_after / T_STOP - 1.0) / (1.0 + kap_after), np.inf)
                    m_clp = np.where(live, np.abs(ov / ALPHA_MAX - 1.0), np.inf)
                allm = np.where(reached[None], np.stack([m_sig, m_alp, m_stp]), np.inf)  # [3,P,G]
                flat = allm.transpose(1, 0, 2).reshape(P, -1)
                am = flat.argmin(1)
                mv = flat[np.arange(P), am]
                better = mv < marg
                marg = np.where(better, mv, marg)
                mkind = np.where(better, am // g.shape[0], mkind)
                mpos = np.where(better, pos[am % g.shape[0]], mpos)
                cmarg = np.minimum(cmarg, m_clp.min(1))
                clamped |= (live & (ov > ALPHA_MAX)).any(1)
                # state leaving the chunk
                any_stop = stopped_incl[:, -1] & ~fin
                first = np.argmax(stop, 1)
                rows = np.arange(P)
                T_new = np.where(any_stop, T_before[rows, first], T_after[:, -1])  # the stopping entry is not composited
                kap_new = np.where(any_stop, (kap_after - a_eff / (1.0 - a_eff))[rows, first], kap_after[:, -1])
                T = np.where(fin, T, T_new)
                kap = np.where(fin, kap, kap_new)
                fin = fin | any_stop
            ref.n_contrib += int(used.sum())
            if keep is not None and kept:
                keep[(tx, ty)] = (y0, y1, x0, x1) + tuple(np.concatenate(k, axis=-1) for k in zip(*kept))
            sl = (slice(y0, y1), slice(x0, x1))
            ref.T[sl] = T.reshape(h, w_)
            ref.sums[sl] = acc.reshape(h, w_, 7)
            ref.mass[sl] = mass.reshape(h, w_, 7)
            ref.ncomp[sl] = ncomp.reshape(h, w_)
            ref.last_ids[sl] = last.reshape(h, w_)
            ref.margin[sl] = marg.reshape(h, w_)
            ref.margin_pos[sl] = mpos.reshape(h, w_)
            ref.margin_kind[sl] = mkind.reshape(h, w_)
            ref.clamp_margin[sl] = cmarg.reshape(h, w_)
            ref.stopped[sl] = fin.reshape(h, w_)
            ref.clamped[sl] = clamped.reshape(h, w_)
            if eps > 0:
                for p in np.nonzero(marg < eps)[0]:
                    ambiguous.append((y0 + int(p) // w_, x0 + int(p) % w_, g_all, pos_all))
    if slip == "last_partner":
        rows = np.arange(H)
        lower = (rows % 8) >= 4
        ref.last_ids[lower] = ref.last_ids[rows[lower] - 4]
    bg = np.asarray(background, dtype=np.float64)
    ref.mass[..., 0:3] += ref.T[..., None] * np.abs(bg)
    if normals:
        ref.mass[..., 4:7] += ref.T[..., None]
    for k, v in epilogue(ref.T, ref.sums, bg, normals, slip).items():
        setattr(ref, k, v)
    covered = ref.depth[ref.done]
    ref.depth_max = max(float(covered.max()) if covered.size else 0.0, 0.0)
    if slip == "stale_depth_max":
        ref.depth_max = max(ref.depth_max, float(stale_depth_max))
    for i, j, g, pos in ambiguous:
        paths = _pixel_paths(m2, con, op, feats, g, pos, j + 0.5, i + 0.5, eps, max_alts)
        if paths is None:
            ref.unresolved.append((i, j))
            continue
        alts = []
        for T, acc, mass, last, ncomp in paths:
            mass = mass.copy()
            mass[0:3] += T * np.abs(bg)
            if normals:
                mass[4:7] += T
            o = epilogue(np.asarray(T), acc, bg, normals)
            o.update(mass=mass, last_ids=last, ncomp=ncomp)
            alts.append(o)
        ref.alts[(i, j)] = alts
    return ref


def _pixel_paths(m2, con, op, feats, g, pos, px, py, eps, cap):
    """Every outcome of one pixel when each decision within eps of its threshold is taken either way (primary first):
    [(T, sums[7], mass[7], last_id, composited)], or None when there are more than `cap`."""
    dx, dy = m2[g, 0] - px, m2[g, 1] - py
    t0, t1, t2 = 0.5 * con[g, 0] * dx * dx, 0.5 * con[g, 2] * dy * dy, con[g, 1] * dx * dy
    sigma = (t0 + t1) + t2
    den = np.abs(t0) + np.abs(t1) + np.abs(t2)
    alpha = np.minimum(op[g] * np.exp(-sigma), ALPHA_MAX)
    valid = (sigma >= 0) & (alpha >= ALPHA_MIN)
    with np.errstate(invalid="ignore", divide="ignore"):
        near = (np.where(den > 0, np.abs(sigma) / den, np.inf) < eps) | ((sigma >= 0) & (np.abs(alpha / ALPHA_MIN - 1.0) < eps))
    cands = [int(e) for e in np.nonzero(valid | near)[0]]
    leaves = []

    class TooMany(Exception):
        pass

    def leaf(state):
        T, _, acc, mass, last, n = state
        leaves.append((T, acc, mass, last, n))
        if len(leaves) > cap:
            raise TooMany

    def take(e, state):
        """Entry e passes the skip tests: (stops, stop test within eps, state after compositing it)."""
        T, kap, acc, mass, _, n = state
        a = float(alpha[e])
        nT = T * (1.0 - a)
        k2 = kap + a / (1.0 - a)
        w = a * T
        f = feats[g[e]]
        return (nT <= T_STOP, abs(nT / T_STOP - 1.0) / (1.0 + k2) < eps,
                (nT, k2, acc + w * f, mass + w * np.abs(f), int(pos[e]), n + 1))

    def taken(c, e, state):
        stops, near_stop, after = take(e, state)
        for s in ((stops, not stops) if near_stop else (stops,)):
            if s:
                leaf(state)
            else:
                walk(c, after)

    def walk(c, state):  # iterative along the unbranched stretch: lists are longer than the recursion limit
        while c < len(cands):
            e = cands[c]
            c += 1
            v = bool(valid[e])
            if near[e]:
                for t in (v, not v):
                    if t:
                        taken(c, e, state)
                    else:
                        walk(c, state)
                return
            stops, near_stop, after = take(e, state)
            if near_stop:
                for s in (stops, not stops):
                    if s:
                        leaf(state)
                    else:
                        walk(c, after)
                return
            if stops:
                break
            state = after
        leaf(state)

    try:
        walk(0, (1.0, 0.0, np.zeros(7), np.zeros(7), 0, 0))
    except TooMany:
        return None
    return leaves


# ------------------------------------------------------------------------------------------------------ acceptance rule
@dataclass
class Verdict:
    worst: float          # largest |got - want| / bound over decided pixels and outputs
    worst_what: str
    failures: List[str]   # reports of the pixels that fail (at most 10)
    n_fail: int
    n_decided: int
    n_ambiguous: int      # pixels under the decision band (judged against their alternatives)
    n_alt_used: int       # of those, pixels that match an alternative other than the primary outcome
    n_unresolved: int     # pixels with too many alternatives (not judged)

    @property
    def ok(self) -> bool:
        return self.n_fail == 0


def _ratios(got: dict, want: dict, mass, ncomp, rtol, atol, normals):
    """Per pixel: the largest |got - want| / bound over the float outputs, and whether last_ids and the clamp mask agree.
    With r = sqrt(1 + composited): sums within r (rtol mass + atol); alpha within r (rtol alpha + atol); the expected depth
    and the normalised normal within the bound their quotient inherits."""
    r = np.sqrt(1.0 + ncomp)
    b = r[..., None] * (rtol * mass + atol)  # [.., 7]
    alpha = want["alpha"]
    b_alpha = r * (rtol * alpha + atol)
    out = np.abs(got["rgb"] - want["rgb"]) / b[..., 0:3]
    ratio = out.max(-1)
    ratio = np.maximum(ratio, np.abs(got["alpha"] - alpha) / b_alpha)
    b_depth = np.where(alpha > 0, (b[..., 3] + np.abs(want["depth"]) * b_alpha) / np.maximum(alpha, 1e-10), 0.0)
    dd = np.abs(got["depth"] - want["depth"])
    with np.errstate(invalid="ignore", divide="ignore"):
        ratio = np.maximum(ratio, np.where(dd == 0, 0.0, dd / b_depth))
        if normals:
            bn = b[..., 4:7].sum(-1)
            ratio = np.maximum(ratio, np.abs(got["normal_norm"] - want["normal_norm"]) / bn)
            ratio = np.maximum(ratio, (np.abs(got["normal"] - want["normal"]) / (bn / want["normal_norm"])[..., None]).max(-1))
    ratio = np.where(np.isnan(ratio), np.inf, ratio)
    ok = got["last_ids"] == want["last_ids"]
    diff = (got["clamp_mask"] ^ want["clamp_mask"]).astype(np.uint8)
    for k in range(3):
        pre = want["rgb_pre"][..., k]
        near = (np.abs(pre) <= b[..., k]) | (np.abs(pre - 1.0) <= b[..., k])
        ok = ok & ((((diff >> k) & 1) == 0) | near)
    return ratio, ok


def judge(ref: RasterRef, got: dict, eps: float, rtol: float, atol: float, region=None) -> Verdict:
    """Holds the kernel's outputs `got` (numpy arrays rgb [H,W,3], depth, alpha, normal, normal_norm, last_ids, clamp_mask)
    to `ref`, which must have been computed with the same eps.  Decided pixels (margin >= eps): every output within its
    bound, last_ids equal, clamp mask equal unless the pre-clamp value is within the bound of 0 or 1.  Pixels under the
    band: the same against any one of their alternatives.  `region`: bool [H,W] restricts the pixels judged."""
    sel = ref.done if region is None else (ref.done & region)
    want = dict(rgb=ref.rgb, rgb_pre=ref.rgb_pre, alpha=ref.alpha, depth=ref.depth, normal=ref.normal,
                normal_norm=ref.normal_norm, last_ids=ref.last_ids, clamp_mask=ref.clamp_mask)
    ratio, ok = _ratios(got, want, ref.mass, ref.ncomp, rtol, atol, ref.normals)
    decided = sel & (ref.margin >= eps)
    bad = decided & ((ratio > 1.0) | ~ok)
    failures = []
    worst, what = 0.0, ""
    if decided.any():
        rr = np.where(decided, ratio, -1.0)
        i, j = np.unravel_index(int(rr.argmax()), rr.shape)
        worst, what = float(rr[i, j]), ref.report(int(i), int(j))
    n_fail = int(bad.sum())
    for i, j in zip(*np.nonzero(bad)):
        if len(failures) < 10:
            failures.append(f"{ref.report(int(i), int(j))}; ratio {ratio[i, j]:.3g}, got last_id {int(got['last_ids'][i, j])} "
                            f"alpha {got['alpha'][i, j]:.9g} mask {int(got['clamp_mask'][i, j])} vs {int(ref.clamp_mask[i, j])}")
    unresolved = {p for p in ref.unresolved if sel[p]}
    n_amb = n_used = 0
    for i, j in zip(*np.nonzero(sel & (ref.margin < eps))):
        p = (int(i), int(j))
        if p in unresolved:
            continue
        n_amb += 1
        g1 = {k: np.asarray(got[k][i, j]) for k in ("rgb", "alpha", "depth", "normal", "normal_norm", "last_ids", "clamp_mask")}
        hit = -1
        for a_i, alt in enumerate(ref.alts[p]):
            r1, ok1 = _ratios(g1, alt, alt["mass"], np.asarray(alt["ncomp"]), rtol, atol, ref.normals)
            if float(r1) <= 1.0 and bool(ok1):
                hit = a_i
                break
        if hit < 0:
            n_fail += 1
            if len(failures) < 10:
                failures.append(f"{ref.report(*p)}; matches none of its alternatives (got last_id {int(got['last_ids'][i, j])}, "
                                f"alpha {got['alpha'][i, j]:.9g})")
        elif hit > 0:
            n_used += 1
    return Verdict(worst=worst, worst_what=what, failures=failures, n_fail=n_fail, n_decided=int(decided.sum()),
                   n_ambiguous=n_amb, n_alt_used=n_used, n_unresolved=len(unresolved))


# ------------------------------------------------------------------------------------------------------------ backward
# kernel mistakes of `raster_bwd_kernel` restated in fp64 (`backward(slip=)`)
BWD_SLIPS = (
    "normal_to_means",  # the normal route's v_alpha reaches means2d (the normal pass sees detached means, quirk B3)
    "abs_after_pair",   # |d/d means2d| taken after a lane's pixel pair (rows r and r + 2 of one column) is summed
    "clamp_warp",       # the clamp fix-up zeroes the sigma / opacity gradient of every pixel of the warp (8-row half tile)
    "clamp_missing",    # no clamp fix-up: a clamped pixel passes -op vis to sigma and vis to the opacity
    "last_excluded",    # pos < last_id instead of pos <= last_id: the entry at last_id is skipped (gradient and T)
    "no_bg",            # the -sum_k bg_k v_rgb_k term of v_alpha is dropped
    "no_white_va",      # the white-background term -sum_c v_n_c of the normal image's v_alpha is dropped
    "mask_ignored",     # the clamp mask is ignored: clamped rgb channels pass their upstream gradient
    "no_depth_quot",    # the -v_depth D / alpha^2 term of v_alpha is dropped
    "T_unclamped",      # T recovered back to front with 1 - op vis instead of 1 - min(op vis, 0.999)
)
SLOTS = ("x", "y", "|x|", "|y|", "A", "B", "C", "opacity", "r", "g", "b", "depth", "n0", "n1", "n2", "pad")


@dataclass
class RasterBwd:
    """Outputs of `backward`: per Gaussian, the 16 floats of a `grad_records` row (include/dnr.h) and their scales."""

    grads: np.ndarray  # [N,16] v_x, v_y, |v_x|, |v_y|, v_A, v_B, v_C, v_opacity, v_rgb, v_depth, v_n, 0
    mass: np.ndarray   # [N,16] sum over pixels of the same expression with every term replaced by its absolute value
    wmass: np.ndarray  # [N,16] the same sum, pixel p weighted by sqrt(1 + entries p composited)
    tmass: np.ndarray  # [N,16] the same sum, pixel p weighted by |(1 - out_alpha) - T64_final| / T64_final
    pix: np.ndarray    # [M] pixel index i * W + j of every (pixel, Gaussian) pair the forward composited
    gid: np.ndarray    # [M] the Gaussian of that pair
    fwd: RasterRef     # the forward oracle whose decisions were differentiated


def backward(means2d, conics, opacities, colors, depths, normals_cam, radii, flatten_ids, tile_offsets, list_shift: int,
             width: int, height: int, background: Sequence[float], v_rgb, v_depth, v_normal, v_alpha, state: dict, *,
             replay: bool = True, slip: Optional[str] = None, tiles: Optional[Sequence[Tuple[int, int]]] = None,
             pre: Optional[Tuple[RasterRef, dict]] = None) -> RasterBwd:
    """fp64 gradient of sum(v_rgb rgb + v_depth depth + v_normal normal + v_alpha alpha) at the forward oracle's own
    decisions (`composite`: which entries each pixel composited, where it stopped, the fp32 tile box), with the
    conventions of `raster_bwd_kernel`:
      * no gradient through sigma or opacity on a pixel where op vis > 0.999 (alpha is clamped there);
      * an rgb channel outside [0, 1] before the clamp (clamp mask bit clear) passes nothing;
      * the expected depth D / max(alpha, 1e-10) passes v_depth / alpha to D where alpha > 0 and -v_depth D / alpha^2
        to alpha, with D / alpha read as the stored expected depth;
      * the normal image (n / |n| + 1) / 2 of n = N + T (white background) is differentiated at the stored normal and
        |n|; its route reaches conics and opacities but not means2d;
      * |v_x|, |v_y| are sums over pixels of the absolute per-pixel derivative.
    `state` holds the forward state the kernel reads: alpha, depth, normal, normal_norm, clamp_mask ([H,W(,3)]).
    replay: the transmittances of each pixel are scaled so that T_final = 1 - state alpha, the value the kernel starts
    its back-to-front recovery from; the result is then the exact derivative at that state.  Without it, the fp64 T.
    Upstream images may be None (zero).  Slips: BWD_SLIPS.  `pre`: (ref, keep) of an earlier
    `composite(..., keep=keep)` on the same inputs, reused instead of compositing again."""
    if slip is not None and slip not in BWD_SLIPS:
        raise ValueError(slip)
    if pre is None:
        keep: dict = {}
        fwd = composite(means2d, conics, opacities, colors, depths, normals_cam, radii, flatten_ids, tile_offsets,
                        list_shift, width, height, background, tiles=tiles, keep=keep)
    else:
        fwd, keep = pre
    H, W = height, width
    con, op = _np64(conics), _np64(opacities).reshape(-1)
    N = con.shape[0]
    normals = normals_cam is not None
    feats = np.concatenate([_np64(colors), _np64(depths).reshape(-1, 1),
                            _np64(normals_cam) if normals else np.zeros((N, 3))], 1)
    bg = np.asarray(background, dtype=np.float64)
    img = lambda x, s: np.zeros((H, W) + s) if x is None else _np64(x).reshape((H, W) + s)  # noqa: E731
    g_rgb, g_d, g_a = img(v_rgb, (3,)), img(v_depth, ()), img(v_alpha, ())
    g_n = img(v_normal if normals else None, (3,))
    oa, od = img(state["alpha"], ()), img(state["depth"], ())
    cmask = np.asarray(state["clamp_mask"]).astype(np.uint8).reshape(H, W)

    # per pixel: the upstream gradient of the composited sums and of T_final (the kernel's prologue), and its mass
    bit = (cmask[..., None] >> np.arange(3, dtype=np.uint8)) & 1
    vC = g_rgb if slip == "mask_ignored" else np.where(bit == 1, g_rgb, 0.0)
    ac = np.maximum(oa, 1e-10)
    vD = np.where(oa > 0, g_d / ac, 0.0)
    quot = np.where(oa >= 1e-10, g_d * od / ac, 0.0)
    va_cd = g_a - (0.0 if slip == "no_bg" else (vC * bg).sum(-1)) - (0.0 if slip == "no_depth_quot" else quot)
    mva_cd = np.abs(g_a) + (np.abs(vC) * np.abs(bg)).sum(-1) + np.abs(quot)
    vN, mvN = np.zeros((H, W, 3)), np.zeros((H, W, 3))
    va_n, mva_n = np.zeros((H, W)), np.zeros((H, W))
    if normals:
        nh = 2.0 * img(state["normal"], (3,)) - 1.0
        nn = img(state["normal_norm"], ())[..., None]
        gh = 0.5 * g_n
        with np.errstate(invalid="ignore", divide="ignore"):
            vN = (gh - nh * (nh * gh).sum(-1, keepdims=True)) / nn
            mvN = (np.abs(gh) + np.abs(nh) * (np.abs(nh) * np.abs(gh)).sum(-1, keepdims=True)) / nn
        if slip != "no_white_va":
            va_n = -vN.sum(-1)
        mva_n = mvN.sum(-1)
    Tk = 1.0 - oa if replay else fwd.T
    dT = np.abs((1.0 - oa) - fwd.T) / fwd.T
    rw = np.sqrt(1.0 + fwd.ncomp)

    out = {k: np.zeros((N, 16)) for k in ("grads", "mass", "wmass", "tmass")}
    pix_l, gid_l = [], []

    def later(x):  # sum over the entries after each one, along axis 1
        c = np.flip(np.cumsum(np.flip(x, 1), 1), 1)
        return np.concatenate([c[:, 1:], np.zeros((x.shape[0], 1))], 1)

    for (y0, y1, x0, x1, g, pos, live, alpha, vis, dx, dy) in keep.values():
        if g.shape[0] == 0:
            continue
        h, w_ = y1 - y0, x1 - x0
        P = h * w_
        sl = (slice(y0, y1), slice(x0, x1))
        px = lambda a: a[sl].reshape((P,) + a.shape[2:])  # noqa: E731
        p_idx = np.nonzero(live)
        pix_l.append((y0 + p_idx[0] // w_) * W + x0 + p_idx[0] % w_)
        gid_l.append(g[p_idx[1]])
        if slip == "last_excluded":
            live = live & (pos[None, :] != px(fwd.last_ids)[:, None])
        a = np.where(live, alpha, 0.0)
        ov = op[g][None, :] * vis
        fac = np.where(live, 1.0 - ov, 1.0) if slip == "T_unclamped" else 1.0 - a
        Tf = px(Tk)[:, None]
        Tb = Tf / np.flip(np.cumprod(np.flip(fac, 1), 1), 1)  # T before each entry, recovered from T_final
        wgt = a * Tb
        inv = 1.0 / fac
        f, af = feats[g], np.abs(feats[g])
        vCp, vDp, vNp, mvNp = px(vC), px(vD), px(vN), px(mvN)
        dot1 = vCp @ f[:, 0:3].T + vDp[:, None] * f[None, :, 3]
        mdot1 = np.abs(vCp) @ af[:, 0:3].T + np.abs(vDp)[:, None] * af[None, :, 3]
        dot2, mdot2 = vNp @ f[:, 4:7].T, mvNp @ af[:, 4:7].T
        # d out / d alpha_i = T_i dot_i - (sum_{j>i} w_j dot_j - T_final va) / (1 - alpha_i), per route
        va1 = Tb * dot1 - (later(wgt * dot1) - Tf * px(va_cd)[:, None]) * inv
        mva1 = Tb * mdot1 + (later(wgt * mdot1) + Tf * px(mva_cd)[:, None]) * inv
        va2 = Tb * dot2 - (later(wgt * dot2) - Tf * px(va_n)[:, None]) * inv
        mva2 = Tb * mdot2 + (later(wgt * mdot2) + Tf * px(mva_n)[:, None]) * inv
        clamped = live & (ov > ALPHA_MAX)
        if slip == "clamp_missing":
            zero = np.zeros_like(live)
        elif slip == "clamp_warp":
            half = (np.arange(P) // w_) >= 8
            zero = np.where(half[:, None], clamped[half].any(0)[None, :], clamped[~half].any(0)[None, :])
        else:
            zero = clamped
        nov = np.where(live & ~zero, -ov, 0.0)  # d alpha / d sigma
        visg = np.where(live & ~zero, vis, 0.0)  # d alpha / d opacity
        va, mva = va1 + va2, mva1 + mva2
        vs, mvs = nov * va, -nov * mva
        vs1, mvs1 = (vs, mvs) if slip == "normal_to_means" else (nov * va1, -nov * mva1)
        A, B, Cc = con[g, 0][None, :], con[g, 1][None, :], con[g, 2][None, :]
        gx, gy = vs1 * (A * dx + B * dy), vs1 * (B * dx + Cc * dy)
        mgx, mgy = mvs1 * (np.abs(A * dx) + np.abs(B * dy)), mvs1 * (np.abs(B * dx) + np.abs(Cc * dy))
        if slip == "abs_after_pair":  # rows r and r + 2 (r & 2 == 0) of a column share a lane's f32x2 pair
            rows = np.arange(P) // w_
            partner = np.where((rows & 2) == 0, np.arange(P) + 2 * w_, -1)
            has = (partner >= 0) & (partner < P)
            agx, agy = np.abs(gx), np.abs(gy)
            for arr, gg in ((agx, gx), (agy, gy)):
                arr[has] = np.abs(gg[has] + gg[partner[has]])
                arr[partner[has]] = 0.0
        else:
            agx, agy = np.abs(gx), np.abs(gy)
        vals = [gx, gy, agx, agy, 0.5 * vs * dx * dx, vs * dx * dy, 0.5 * vs * dy * dy, visg * va]
        masses = [mgx, mgy, mgx, mgy, 0.5 * mvs * dx * dx, mvs * np.abs(dx * dy), 0.5 * mvs * dy * dy, visg * mva]
        for k in range(3):
            vals.append(wgt * vCp[:, k:k + 1])
            masses.append(wgt * np.abs(vCp[:, k:k + 1]))
        vals.append(wgt * vDp[:, None])
        masses.append(wgt * np.abs(vDp)[:, None])
        for k in range(3):
            vals.append(wgt * vNp[:, k:k + 1])
            masses.append(wgt * mvNp[:, k:k + 1])
        r, t = px(rw)[:, None], px(dT)[:, None]
        for k, (v, m) in enumerate(zip(vals, masses)):
            m = np.where(live, m, 0.0)
            np.add.at(out["grads"][:, k], g, np.where(live, v, 0.0).sum(0))
            np.add.at(out["mass"][:, k], g, m.sum(0))
            np.add.at(out["wmass"][:, k], g, (r * m).sum(0))
            np.add.at(out["tmass"][:, k], g, (t * m).sum(0))
    cat = lambda xs: np.concatenate(xs) if xs else np.zeros(0, np.int64)  # noqa: E731
    return RasterBwd(pix=cat(pix_l), gid=cat(gid_l), fwd=fwd, **out)


@dataclass
class BwdVerdict:
    worst: float         # largest |got - want| / bound over the judged Gaussians and slots
    worst_what: str
    failures: List[str]  # the first 10 failing (Gaussian, slot) reports
    n_fail: int
    n_judged: int        # Gaussians judged

    @property
    def ok(self) -> bool:
        return self.n_fail == 0


def bwd_bound(ref: RasterBwd, rtol: float, atol: float, extra: float = 0.0) -> np.ndarray:
    """RTOL sum_p sqrt(1 + n_p) mass_pgk + ATOL max_g' mass_g'k (+ extra tmass: the T_final term of an unreplayed
    reference)."""
    return rtol * ref.wmass + atol * ref.mass.max(0, initial=0.0)[None, :] + extra * ref.tmass


def judge_bwd(ref: RasterBwd, got: np.ndarray, rtol: float, atol: float, rows=None, extra: float = 0.0) -> BwdVerdict:
    """Holds the kernel's grad_records `got` [N,16] to `ref` per Gaussian and slot.  A slot whose bound is 0 (no mass:
    slot 15, the normal slots without v_normal, ...) must be exactly 0.  `rows`: bool [N] restricts the Gaussians."""
    got = np.asarray(got, dtype=np.float64)
    b = bwd_bound(ref, rtol, atol, extra)
    err = np.abs(got - ref.grads)
    with np.errstate(invalid="ignore", divide="ignore"):
        ratio = np.where(err == 0, 0.0, err / b)
    ratio = np.where(np.isnan(ratio), np.inf, ratio)
    sel = np.ones(ratio.shape[0], bool) if rows is None else np.asarray(rows, bool)
    rr = np.where(sel[:, None], ratio, -1.0)
    bad = np.argwhere(rr > 1.0)
    worst, what = 0.0, ""
    if sel.any():
        g, k = np.unravel_index(int(rr.argmax()), rr.shape)
        worst = float(rr[g, k])
        what = f"Gaussian {g} slot {k} ({SLOTS[k]}): got {got[g, k]:.9g}, want {ref.grads[g, k]:.9g}, bound {b[g, k]:.3g}"
    fails = [f"Gaussian {g} slot {k} ({SLOTS[k]}): got {got[g, k]:.9g}, want {ref.grads[g, k]:.9g}, ratio {ratio[g, k]:.3g}"
             for g, k in bad[:10]]
    return BwdVerdict(worst=worst, worst_what=what, failures=fails, n_fail=int(bad.shape[0]), n_judged=int(sel.sum()))
