"""`dn_rasterize`: the Python operator surface of the H100 depth+normal rasterizer (SURVEY.md §8b).

One autograd.Function replaces, inside DNSplatterModel.get_outputs of the reference
(/root/reference/dn_splatter/dn_model.py):
    :495-516  gsplat.rendering.rasterization(..., render_mode="RGB+ED", absgrad=True)
    :526-537  background blend / clamp / depth fill
    :543-575  per-Gaussian normals + gsplat.rasterize_gaussians (legacy, white background)
    :577-578  normalise / remap of the normal image
    :589-603  normal_from_depth_image on the detached depth
All arithmetic runs in libdnr_b200.so (hand-written sm_90a CUDA) through the C ABI of include/dnr.h;
torch only owns the device buffers and the stream.  There is no CPU / PyTorch fallback.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import NamedTuple, Optional, Sequence, Tuple

import torch
from torch import Tensor

from . import _lib as L

TILE = 16


class DnrCapacityError(L.DnrError):
    """A view needed more intersection slots than its (sync-free / fixed) buffers had: its render and gradients are
    truncated and must not be used.  The capacity has already been raised; render the view again."""


class CountWatch:
    """Host-side overflow check of fixed-capacity intersection buffers, whose binning kernels silently drop the entries
    past the capacity.  Each view's count is copied to a pinned ring asynchronously (`observe`); `check` raises
    DnrCapacityError for a truncated view, and a truncated view nobody checked is kept for `raise_unreported`."""

    SLOTS = 256

    def __init__(self, remedy: str = ""):
        self.remedy = remedy  # what the error message tells the user to do
        self.max_seen, self.overflows, self.pending, self.seeds = 0, 0, [], 0
        self.host, self.slot = torch.zeros(self.SLOTS, dtype=torch.int64).pin_memory(), 0
        self.unreported = None  # (needed, capacity) of a truncated view whose ticket nobody has checked

    def seed(self, count: int) -> None:
        """Records a count that was read back synchronously."""
        self.max_seen = max(self.max_seen, count)
        self.seeds += 1

    def observe(self, count_dev: Tensor, cap: int) -> dict:
        """Queues the async read-back of `count_dev` (int64[1]) on the current stream; returns its ticket."""
        if len(self.pending) >= self.SLOTS - 1:
            self.poll(wait=True)
        host = self.host[self.slot:self.slot + 1]
        self.slot = (self.slot + 1) % self.SLOTS
        host.copy_(count_dev, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        ticket = {"host": host, "event": ev, "cap": cap, "count": None, "checked": False}
        self.pending.append(ticket)
        return ticket

    def _resolve(self, t) -> None:
        if t["count"] is None:
            t["count"] = int(t["host"].item())
            self.max_seen = max(self.max_seen, t["count"])
            if t["count"] > t["cap"]:
                self.overflows += 1
                if not t["checked"]:
                    self.unreported = (t["count"], t["cap"])

    def poll(self, wait: bool = False) -> None:
        """Resolves the tickets whose copies have landed (all pending tickets with wait=True)."""
        keep = []
        for t in self.pending:
            if wait:
                t["event"].synchronize()
            if t["event"].query():
                self._resolve(t)
            else:
                keep.append(t)
        self.pending = keep

    def check(self, ticket) -> None:
        """Waits for this ticket's count and raises DnrCapacityError if its view was truncated."""
        ticket["checked"] = True
        ticket["event"].synchronize()
        self._resolve(ticket)
        if self.unreported == (ticket["count"], ticket["cap"]):
            self.unreported = None
        if ticket["count"] > ticket["cap"]:
            raise DnrCapacityError(f"this view needs {ticket['count']} intersection slots but was rendered with "
                                   f"{ticket['cap']}: its outputs and gradients are truncated.  {self.remedy}")

    def raise_unreported(self) -> None:
        if self.unreported is not None:
            (need, cap), self.unreported = self.unreported, None
            raise DnrCapacityError(f"an earlier view needed {need} intersection slots but was rendered with {cap}: its "
                                   f"outputs and gradients are truncated.  {self.remedy}")


GROWTH = 1.15  # headroom over the largest count seen: sync-free sizing and training-graph re-capture


def round_capacity(need: int) -> int:
    """Rounds up keeping 4 significant bits (steps of 1/16 .. 1/8 of the value, at least 4096 entries): few distinct buffer
    sizes for the caching allocator without over-allocating small scenes."""
    need = max(int(need), 4096)
    step = max(4096, 1 << max(need.bit_length() - 4, 0))
    return (need + step - 1) // step * step


def grow(count: int, factor: float) -> int:
    """Intersection capacity with room for `count` times `factor`, plus a fixed margin, rounded up."""
    return round_capacity(int(count * factor) + 4096)


# Sync-free sizing: one CountWatch per (device, n, W, H, normals, exact lists, list tile).  After two synchronous views a
# view gets grow(max count seen, GROWTH) slots; if truncated, its backward (no-grad: the next forward) raises.
_CAPACITY: dict = {}


def suggested_capacity(n_gauss: int, width: int, height: int, render_normals: bool = True, exact_lists: bool = False,
                       device_index: Optional[int] = None, list_shift: Optional[int] = None) -> int:
    """Capacity for graph capture: grow(largest count seen in sync-free mode, GROWTH), 0 without statistics.
    `list_shift` is ignored with exact_lists, which always bins per 16-pixel tile."""
    best = 0
    for (di, n, w, h, rn, ex, lt), t in _CAPACITY.items():
        if (n, w, h, rn, ex) == (n_gauss, width, height, render_normals, exact_lists) and (device_index in (None, di)) \
                and (list_shift is None or exact_lists or lt == TILE << list_shift):
            t.poll(wait=True)
            best = max(best, grow(t.max_seen, GROWTH))
    return best


def capacity_report() -> dict:
    """{key: (max intersections seen, truncated views)} for the sync-free mode; waits for pending counts."""
    out = {}
    for k, t in _CAPACITY.items():
        t.poll(wait=True)
        out[k] = (t.max_seen, t.overflows)
    return out


# Optional per-stage device timing (bench.py's roofline pass): when STAGE_EVENTS is a list, every C-ABI
# stage call is bracketed by CUDA events on the launching stream and (name, start, end) is appended.
STAGE_EVENTS = None


def _timed(name, fn, *args):
    if STAGE_EVENTS is None:
        return fn(*args)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    rc = fn(*args)
    e1.record()
    STAGE_EVENTS.append((name, e0, e1))
    return rc


@dataclass(frozen=True)
class RasterSettings:
    width: int
    height: int
    sh_degree: int = 3
    near_plane: float = 0.01  # dn_model.py:507
    far_plane: float = 1e10  # dn_model.py:508
    eps2d: float = 0.3
    antialiased: bool = False  # rasterize_mode == "antialiased" (dn_model.py:513)
    render_normals: bool = True  # config.predict_normals
    activated: bool = False  # inputs already exp()/sigmoid()-activated (gsplat's own signature)
    background: Tuple[float, float, float] = (0.0, 0.0, 0.0)
    surface_normal: bool = True
    exact_lists: bool = False  # parity mode: gsplat's full bbox intersection lists instead of the precise-hit lists
    sync_free: bool = False  # size the intersection buffers from past views instead of reading the count back
    fixed_capacity: int = 0  # > 0: use exactly this many intersection slots, no host bookkeeping (CUDA-graph capture)
    list_shift: int = 2  # intersection lists per (16 << list_shift)-pixel supertile; forced to 0 by exact_lists


class RasterOutput(NamedTuple):
    rgb: Tensor  # [H,W,3]
    depth: Tensor  # [H,W,1]
    normal: Tensor  # [H,W,3] in [0,1] (zeros when render_normals is False)
    alpha: Tensor  # [H,W,1]
    surface_normal: Tensor  # [H,W,3] in [0,1]
    means2d: Tensor  # [N,2]; after backward carries .grad and .absgrad (dn_model.py:517-519)
    radii: Tensor  # [N] int32
    depths: Tensor  # [N]
    conics: Tensor  # [N,3]
    tiles_per_gauss: Tensor  # [N] int32
    normals_world: Tensor  # [N,3] (gauss_params["normals"], dn_model.py:558)
    info: dict


def _ptr(t: Optional[Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _require_cuda(*ts: Tensor) -> torch.device:
    dev = ts[0].device
    if dev.type != "cuda":
        raise L.DnrError("dn_rasterize needs CUDA tensors: this library has no CPU path")
    for t in ts:
        if t is not None and t.device != dev:
            raise L.DnrError("all tensors must live on the same CUDA device")
    if dev.index is not None and dev.index != torch.cuda.current_device():
        # kernels are enqueued on torch's CURRENT stream, which belongs to the current device
        raise L.DnrError(f"tensors are on {dev} but the current device is cuda:{torch.cuda.current_device()}: "
                         "call torch.cuda.set_device / use torch.cuda.device(...)")
    return dev


def _base_args(s: RasterSettings, n: int, sh_bases: int, accumulate: bool = False) -> L.DnrArgs:
    a = L.DnrArgs()
    a.n_gauss, a.width, a.height, a.tile_size = n, s.width, s.height, TILE
    a.sh_degree, a.sh_bases = s.sh_degree, sh_bases
    flags = 0
    if s.activated:
        flags |= L.FLAG_ACTIVATED
    if s.antialiased:
        flags |= L.FLAG_ANTIALIASED
    if s.render_normals:
        flags |= L.FLAG_NORMALS
    if accumulate:
        flags |= L.FLAG_ACCUMULATE
    if s.exact_lists:
        flags |= L.FLAG_EXACT_LISTS
    a.flags = flags
    a.list_shift = 0 if s.exact_lists else int(s.list_shift)
    a.near_plane, a.far_plane, a.eps2d, a.radius_clip = s.near_plane, s.far_plane, s.eps2d, 0.0
    a.background[0], a.background[1], a.background[2] = s.background
    return a


def _set_host_cam(a: L.DnrArgs, host_cam) -> None:
    if host_cam is not None:
        a.flags |= L.FLAG_HOST_CAMERA
        a.host_cam[:] = host_cam


def _set(a: L.DnrArgs, **tensors: Optional[Tensor]) -> None:
    for k, t in tensors.items():
        setattr(a, k, _ptr(t))


class _DnRasterize(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means, quats, scales, opacities, sh_dc, sh_rest, viewmat, K, c2w, settings: RasterSettings, holder: dict):
        lib = L.load()
        s = settings
        ctx.set_materialize_grads(False)  # unused output gradients arrive as None instead of freshly filled zero tensors
        dev = _require_cuda(means, quats, scales, opacities, sh_dc, sh_rest)
        ctx.viewmat_meta = (viewmat.shape, viewmat.device)
        # camera on the host (CPU tensors) -> passed by value, no device traffic; on the device -> read by the kernels
        host_cam = None
        if viewmat.device.type == "cpu":
            host_cam = viewmat.detach().float().reshape(16).tolist()
            Kc = K.detach().float().cpu().reshape(3, 3)
            host_cam += [float(Kc[0, 0]), float(Kc[1, 1]), float(Kc[0, 2]), float(Kc[1, 2])]
            host_cam += c2w.detach().float().cpu().reshape(12).tolist() if c2w is not None else [0.0] * 12
        else:
            _require_cuda(means, viewmat, K)
        f32 = dict(dtype=torch.float32, device=dev)
        i32 = dict(dtype=torch.int32, device=dev)
        means, quats, scales = means.contiguous().float(), quats.contiguous().float(), scales.contiguous().float()
        opac = opacities.contiguous().float().view(-1)
        sh_dc, sh_rest = sh_dc.contiguous().float(), sh_rest.contiguous().float()
        if host_cam is None:
            viewmat, K = viewmat.contiguous().float().view(4, 4), K.contiguous().float().view(3, 3)
        else:
            viewmat = K = None
        n = means.shape[0]
        sh_bases = 1 + sh_rest.shape[1]
        if n == 0:
            raise L.DnrError("dn_rasterize: empty Gaussian set")
        if s.render_normals:
            if c2w is None:
                raise L.DnrError("render_normals=True needs the camera_to_world matrix")
            c2w = None if host_cam is not None else c2w.contiguous().float().view(3, 4)
        H, W = s.height, s.width
        tiles_x, tiles_y = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
        list_tile = TILE << (0 if s.exact_lists else int(s.list_shift))  # one sorted list per list_tile^2 pixels
        lists_x, lists_y = (W + list_tile - 1) // list_tile, (H + list_tile - 1) // list_tile
        n_tiles = lists_x * lists_y
        rec_f = L.REC_FLOATS_N if s.render_normals else L.REC_FLOATS
        st = L.stream()
        ctx.fwd_stream = torch.cuda.current_stream()
        ctx.capacity_ticket = None

        radii = torch.empty(n, **i32)
        means2d = torch.empty(n, 2, **f32)
        depths = torch.empty(n, **f32)
        conics = torch.empty(n, 3, **f32)
        opac_act = torch.empty(n, **f32)
        comp = torch.empty(n, **f32) if s.antialiased else None
        colors = torch.empty(n, 3, **f32)
        normals_world = torch.empty(n, 3, **f32) if s.render_normals else torch.zeros(n, 3, **f32)
        tiles_per_gauss = torch.empty(n, **i32)
        depth_keys = torch.empty(n, **i32)
        records = torch.empty(n, rec_f, **f32)
        cull_lim = torch.empty(n, **f32)
        n_isects_dev = torch.empty(1, dtype=torch.int64, device=dev)

        a = _base_args(s, n, sh_bases)
        _set_host_cam(a, host_cam)
        _set(a, viewmat=viewmat, K=K, c2w=c2w, means=means, quats=quats, scales=scales, opacities=opac, sh_dc=sh_dc,
             sh_rest=sh_rest if sh_bases > 1 else None, radii=radii, means2d=means2d, depths=depths, conics=conics,
             opac_act=opac_act, compensations=comp, colors=colors,
             normals_world=normals_world if s.render_normals else None, tiles_per_gauss=tiles_per_gauss,
             depth_keys=depth_keys, records=records, cull_lim=cull_lim, n_isects_dev=n_isects_dev)
        L.check(_timed("project_fwd", lib.dnr_project_fwd, C.byref(a), st), "dnr_project_fwd")

        ws_scan = torch.empty(lib.dnr_bin_scan_workspace_bytes(n), dtype=torch.uint8, device=dev)
        _set(a, ws_scan=ws_scan)
        cap_key = (dev.index, n, W, H, s.render_normals, s.exact_lists, list_tile)
        watch = _CAPACITY.get(cap_key) if s.sync_free else None
        if s.fixed_capacity > 0:
            # graph-capturable: no read-back, no events, no host state; the owner of the graph (graph_step.py,
            # render_service.py) gives the replay's info["n_isects_dev"] to a CountWatch
            L.check(_timed("bin_scan", lib.dnr_bin_scan, C.byref(a), st, None), "dnr_bin_scan")
            n_isects = int(s.fixed_capacity)
        elif watch is not None and watch.seeds >= 2:
            # sync-free: nothing is read back on this stream; capacity comes from the counts of earlier views
            watch.poll()
            watch.raise_unreported()
            L.check(_timed("bin_scan", lib.dnr_bin_scan, C.byref(a), st, None), "dnr_bin_scan")
            n_isects = grow(watch.max_seen, GROWTH)
            ctx.capacity_ticket = (watch, watch.observe(n_isects_dev, n_isects))
        else:
            total = C.c_int64(0)
            L.check(_timed("bin_scan", lib.dnr_bin_scan, C.byref(a), st, C.byref(total)), "dnr_bin_scan")
            n_isects = int(total.value)
            if s.sync_free:
                if cap_key not in _CAPACITY:
                    # the Gaussian count changed (densification): drop the watches of the old counts for this
                    # device / resolution instead of keeping one pinned buffer per count ever seen
                    for stale in [k for k in _CAPACITY if k[0] == cap_key[0] and k[2:] == cap_key[2:] and k[1] != n]:
                        del _CAPACITY[stale]
                    _CAPACITY[cap_key] = CountWatch("The capacity has been raised — render the view again "
                                                    "(or use sync_free=False).")
                _CAPACITY[cap_key].seed(n_isects)
        a.n_isects = n_isects
        ws_sort = torch.empty(lib.dnr_bin_sort_workspace_bytes(n, n_isects, n_tiles), dtype=torch.uint8, device=dev)
        flatten_ids = torch.empty(max(n_isects, 1), **i32)
        tile_offsets = torch.empty(n_tiles + 1, **i32)
        _set(a, ws_sort=ws_sort, flatten_ids=flatten_ids, tile_offsets=tile_offsets)
        L.check(_timed("bin_sort", lib.dnr_bin_sort, C.byref(a), st), "dnr_bin_sort")

        out_rgb = torch.empty(H, W, 3, **f32)
        out_depth = torch.empty(H, W, 1, **f32)
        out_alpha = torch.empty(H, W, 1, **f32)
        out_normal = torch.empty(H, W, 3, **f32) if s.render_normals else None
        normal_norm = torch.empty(H, W, **f32) if s.render_normals else None
        out_sn = torch.empty(H, W, 3, **f32) if s.surface_normal else None
        last_ids = torch.empty(H, W, **i32)
        clamp_mask = torch.empty(H, W, dtype=torch.uint8, device=dev)
        depth_max = torch.empty(1, **i32)
        stats = holder.get("stats")  # optional uint64[4] device counters (list entries walked / kept by the tile filter)
        _set(a, out_rgb=out_rgb, out_depth=out_depth, out_alpha=out_alpha, out_normal=out_normal,
             out_surface_normal=out_sn, last_ids=last_ids, normal_norm=normal_norm, clamp_mask=clamp_mask,
             depth_max=depth_max, stats=stats)
        L.check(_timed("raster_fwd", lib.dnr_raster_fwd, C.byref(a), st), "dnr_raster_fwd")
        L.check(_timed("finalize_fwd", lib.dnr_finalize_fwd, C.byref(a), st), "dnr_finalize_fwd")

        ctx.settings, ctx.n, ctx.sh_bases, ctx.n_isects, ctx.host_cam = s, n, sh_bases, n_isects, host_cam
        ctx.save_for_backward(means, quats, scales, opac, sh_dc, sh_rest, viewmat, K, c2w if s.render_normals else None)
        ctx.state = dict(radii=radii, records=records, flatten_ids=flatten_ids, tile_offsets=tile_offsets,
                         out_rgb=out_rgb, out_depth=out_depth, out_alpha=out_alpha, out_normal=out_normal, last_ids=last_ids,
                         normal_norm=normal_norm, clamp_mask=clamp_mask, means2d=means2d)
        ctx.holder = holder
        ctx.opac_shape = opacities.shape
        normal_ret = out_normal if s.render_normals else torch.zeros(H, W, 3, **f32)
        sn_ret = out_sn if s.surface_normal else torch.zeros(H, W, 3, **f32)
        info = dict(flatten_ids=flatten_ids[:n_isects], tile_offsets=tile_offsets, last_ids=last_ids, n_isects=n_isects,
                    n_isects_dev=n_isects_dev,
                    colors=colors, opacities=opac_act, compensations=comp, tile_width=tiles_x, tile_height=tiles_y,
                    list_tile=list_tile, lists_x=lists_x, lists_y=lists_y, depth_max=depth_max)
        ctx.grad_sink = holder.pop("grad_sink", None)
        holder.update(info)
        ctx.mark_non_differentiable(sn_ret, means2d, radii, depths, conics, tiles_per_gauss, normals_world)
        return (out_rgb, out_depth, normal_ret, out_alpha, sn_ret, means2d, radii, depths, conics, tiles_per_gauss,
                normals_world)

    @staticmethod
    def backward(ctx, v_rgb, v_depth, v_normal, v_alpha, *_unused):
        # run on the forward's stream explicitly (the autograd worker thread's current stream is not guaranteed to be
        # it for foreign launches, and under CUDA-graph capture anything on another stream invalidates the capture)
        with torch.cuda.stream(ctx.fwd_stream):
            return _DnRasterize._backward(ctx, v_rgb, v_depth, v_normal, v_alpha)

    @staticmethod
    def _backward(ctx, v_rgb, v_depth, v_normal, v_alpha):
        lib = L.load()
        s: RasterSettings = ctx.settings
        if ctx.capacity_ticket is not None:  # sync-free sizing: never produce gradients from a truncated render
            watch, ticket = ctx.capacity_ticket
            watch.check(ticket)
        means, quats, scales, opac, sh_dc, sh_rest, viewmat, K, c2w = ctx.saved_tensors
        S = ctx.state
        n, dev = ctx.n, means.device
        f32 = dict(dtype=torch.float32, device=dev)
        st = L.stream()

        def prep(g):
            # zero-stride tokens stand for "this gradient is evaluated inside dnr_raster_bwd" (deferred losses, below)
            if g is None or _is_zero_token(g):
                return None
            return g.contiguous().float()

        v_rgb, v_depth, v_alpha = prep(v_rgb), prep(v_depth), prep(v_alpha)
        v_normal = prep(v_normal) if s.render_normals else None
        sink = ctx.grad_sink
        touched = grad_records = None
        if sink is not None:
            # the caller's buffers: a FlatGradBucket keeps the flags across backwards and grad_records always zero
            # (DNR_FLAG_PERSISTENT_WS); parallel.PeerGradBucket's peers read its flags over NVLink
            touched, grad_records = sink.get("touched"), sink.get("grad_records")
        if touched is None:
            touched, grad_records = torch.empty(n, dtype=torch.uint8, device=dev), None
        persistent = grad_records is not None
        if grad_records is None:
            grad_records = torch.empty(n, L.GRAD_FLOATS, **f32)
        a = _base_args(s, n, ctx.sh_bases)
        _set_host_cam(a, ctx.host_cam)
        a.n_isects = ctx.n_isects
        _set(a, viewmat=viewmat, K=K, c2w=c2w, means=means, quats=quats, scales=scales, opacities=opac, sh_dc=sh_dc,
             sh_rest=sh_rest if ctx.sh_bases > 1 else None, radii=S["radii"], records=S["records"],
             flatten_ids=S["flatten_ids"], tile_offsets=S["tile_offsets"], out_rgb=S["out_rgb"], out_depth=S["out_depth"],
             out_alpha=S["out_alpha"], out_normal=S["out_normal"], last_ids=S["last_ids"],
             normal_norm=S["normal_norm"], clamp_mask=S["clamp_mask"], v_rgb=v_rgb, v_depth=v_depth,
             v_normal=v_normal, v_alpha=v_alpha, grad_records=grad_records, stats=ctx.holder.get("stats"))
        # losses whose backward asked to be evaluated in the raster kernel's prologue (regularization_strategy.py)
        keep = _apply_deferred_losses(a, ctx.holder.pop("deferred", None))
        _set(a, touched=touched)
        if persistent:
            a.flags |= L.FLAG_PERSISTENT_WS
        L.check(_timed("raster_bwd", lib.dnr_raster_bwd, C.byref(a), st), "dnr_raster_bwd")
        del keep
        # project_bwd visits only the flagged Gaussians and accumulates: every gradient buffer starts at zero
        a.flags |= L.FLAG_ACCUMULATE
        if sink is not None:
            # write straight into the caller's (pre-zeroed, e.g. flat all-reduce bucket) gradient buffers
            v_means, v_quats, v_scales = sink["means"], sink["quats"], sink["scales"]
            v_opac, v_sh_dc, v_sh_rest = sink["opacities"], sink["features_dc"], sink["features_rest"]
        else:
            v_means = torch.zeros_like(means)
            v_quats = torch.zeros_like(quats)
            v_scales = torch.zeros_like(scales)
            v_opac = torch.zeros_like(opac)
            v_sh_dc = torch.zeros_like(sh_dc)
            v_sh_rest = torch.zeros_like(sh_rest)
        v_m2d = torch.zeros(n, 2, **f32)
        v_m2d_abs = torch.zeros(n, 2, **f32)
        # camera optimisation: d(loss)/d(viewmat) only when the viewmat asks for it (otherwise the launch is unchanged)
        v_viewmat = torch.zeros(4, 4, **f32) if ctx.needs_input_grad[6] else None
        _set(a, v_means=v_means, v_quats=v_quats, v_scales=v_scales, v_opacities=v_opac, v_sh_dc=v_sh_dc,
             v_sh_rest=v_sh_rest if ctx.sh_bases > 1 else None, v_means2d=v_m2d, v_means2d_abs=v_m2d_abs,
             v_viewmat=v_viewmat)
        L.check(_timed("project_bwd", lib.dnr_project_bwd, C.byref(a), st), "dnr_project_bwd")
        # what nerfstudio's after_train reads: self.xys.grad / self.xys.absgrad (dn_model.py:517-519)
        S["means2d"].grad = v_m2d
        S["means2d"].absgrad = v_m2d_abs
        if v_viewmat is not None:
            shape, vdev = ctx.viewmat_meta
            v_viewmat = v_viewmat.to(vdev).view(shape)
        if sink is not None:
            if sink.get("bucket") is not None:
                sink["bucket"].note_backward()
            return (None,) * 6 + (v_viewmat,) + (None,) * 4
        return (v_means, v_quats, v_scales, v_opac.view(ctx.opac_shape), v_sh_dc, v_sh_rest, v_viewmat, None, None, None,
                None)


def _apply_deferred_losses(a: L.DnrArgs, deferred: Optional[dict]):
    """Fills the DNR_LOSS_FUSED_BWD fields of `a` from the specs the loss Functions left in the raster holder; returns
    the tensors that must stay alive until the launch."""
    if not deferred:
        return None
    keep = []
    flags = L.LOSS_FUSED_BWD
    l1 = deferred.get("l1")
    if l1 is not None:
        gt, v = l1["gt"], l1["v"]
        if gt.dtype == torch.uint8:
            flags |= L.LOSS_IMG_U8
        a.gt_image, a.v_l1 = gt.data_ptr(), v.data_ptr()
        keep += [gt, v]
    reg = deferred.get("reg")
    if reg is not None:
        a.depth_loss_type, a.use_normal_loss = reg["depth_type"], reg["use_normal"]
        a.depth_lambda, a.depth_tolerance = reg["depth_lambda"], reg["depth_tolerance"]
        for k in ("gt_depth", "gt_normal", "gt_rgb", "loss_partials"):
            t = reg.get(k)
            setattr(a, k, None if t is None else t.data_ptr())
            keep.append(t)
        a.v_loss = reg["v"].data_ptr()
        keep.append(reg["v"])
        if reg.get("gt_normal") is not None and reg["gt_normal"].dtype == torch.uint8:
            flags |= L.LOSS_NORMAL_U8
        if reg.get("edge_image") is not None:  # EdgeAwareLogL1 weights straight from the uint8 image
            img = reg["edge_image"]
            if l1 is not None and l1["gt"].data_ptr() != img.data_ptr():
                raise L.DnrError("fused losses: the photometric target and the edge image must be the same uint8 tensor")
            a.gt_image = img.data_ptr()
            flags |= L.LOSS_EDGE_FROM_IMAGE | L.LOSS_IMG_U8
            keep.append(img)
    a.loss_flags = flags
    return keep


def raster_holder(t: Tensor) -> Optional[dict]:
    """The holder dict of the dn_rasterize call that produced `t` (a RasterOutput map), or None.  Loss Functions use it
    to hand their backward to dnr_raster_bwd: they store a spec under holder["deferred"] and return zero_token(...)."""
    return getattr(t, "_dnr_holder", None)


def zero_token(like: Tensor) -> Tensor:
    """A zero gradient without memory: zero-stride view of a cached scalar 0 (adds exactly nothing if autograd sums it
    with a real gradient; recognised and skipped by _DnRasterize.backward)."""
    z = _ZERO.get(like.device)
    if z is None:
        z = _ZERO[like.device] = torch.zeros((), dtype=torch.float32, device=like.device)
    return z.expand(like.shape)


_ZERO: dict = {}


def _is_zero_token(g: Tensor) -> bool:
    # identity, not just shape: `x.sum().backward()` also yields zero-stride gradients (of ones)
    z = _ZERO.get(g.device)
    return z is not None and g.data_ptr() == z.data_ptr() and all(sd == 0 for sd in g.stride())


def dn_rasterize(
    means: Tensor, quats: Tensor, scales: Tensor, opacities: Tensor, sh_dc: Tensor, sh_rest: Tensor,
    viewmat: Tensor, K: Tensor, width: int, height: int, *, sh_degree: int = 3, near_plane: float = 0.01,
    far_plane: float = 1e10, eps2d: float = 0.3, antialiased: bool = False,
    background: Sequence[float] = (0.0, 0.0, 0.0), render_normals: bool = True, c2w: Optional[Tensor] = None,
    activated: bool = False, surface_normal: bool = True, grad_sink: Optional[dict] = None,
    exact_lists: bool = False, sync_free: bool = False, fixed_capacity: int = 0, list_shift: int = 2,
    stats: Optional[Tensor] = None,
) -> RasterOutput:
    """Renders one view.  Inputs are the reference's RAW gauss_params (log-scales, opacity logits,
    un-normalised wxyz quats, SH coefficients split as features_dc / features_rest) unless
    ``activated=True``.  `viewmat` is the OpenCV world->camera matrix of nerfstudio's get_viewmat,
    `c2w` the un-optimised nerfstudio camera_to_world [3,4] (only used for normals)."""
    if isinstance(background, Tensor):
        background = background.detach().flatten().tolist()
    bg = tuple(float(b) for b in background)
    settings = RasterSettings(width=int(width), height=int(height), sh_degree=int(sh_degree), near_plane=near_plane,
                              far_plane=far_plane, eps2d=eps2d, antialiased=antialiased, render_normals=render_normals,
                              activated=activated, background=bg, surface_normal=surface_normal, exact_lists=exact_lists,
                              sync_free=sync_free, fixed_capacity=int(fixed_capacity), list_shift=int(list_shift))
    info: dict = {}
    if stats is not None:
        info["stats"] = stats
    if grad_sink is not None:
        # dict with fp32 contiguous buffers shaped like the six parameters (keys: means, quats, scales, opacities,
        # features_dc, features_rest); the backward ACCUMULATES into them and autograd sees no gradient.
        info["grad_sink"] = grad_sink
    outs = _DnRasterize.apply(means, quats, scales, opacities, sh_dc, sh_rest, viewmat, K, c2w, settings, info)
    if torch.is_grad_enabled():
        for t in outs[:4]:  # rgb, depth, normal, alpha: losses may defer their backward to dnr_raster_bwd through this
            t._dnr_holder = info
    return RasterOutput(*outs, info)


def get_viewmat(c2w: Tensor) -> Tensor:
    """nerfstudio `get_viewmat` [EXT] (SURVEY A7): OpenGL camera_to_world [..,3,4] -> OpenCV world->camera [4,4].
    Device-only ops (no host constants): building it must not trigger a blocking H2D copy."""
    c2w = c2w.reshape(3, 4)
    Rinv = torch.cat([c2w[:, :1], -c2w[:, 1:3]], dim=1).T  # (R * diag(1,-1,-1))^T
    t = -(Rinv @ c2w[:, 3:4])
    bottom = torch.zeros(1, 4, dtype=c2w.dtype, device=c2w.device)
    bottom[:, 3:].fill_(1.0)  # a fill kernel: `bottom[0, 3] = 1.0` copies a host scalar (not capturable)
    return torch.cat([torch.cat([Rinv, t], dim=1), bottom], dim=0)


def to_device_async(t: Tensor, device) -> Tensor:
    """Small host tensor -> device without blocking the host (pinned staging + non_blocking copy)."""
    if t.device == torch.device(device):
        return t
    if t.device.type == "cpu" and torch.device(device).type == "cuda":
        return t.pin_memory().to(device, non_blocking=True)
    return t.to(device)
