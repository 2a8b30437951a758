"""Render-all-views forward service (SURVEY.md §8f-1): what `gs-mesh`, `ns-eval` and `render_model.py` do with the model
— `for camera in views: model.get_outputs_for_camera(camera)` (reference export_mesh.py:360-367, 863-905, 965-1017;
dn_pipeline.py:194-214; scripts/render_model.py:47-69; utils/utils.py:331-443) — as a service that keeps the device busy.

CUDA path (`graph=True`, the default on a GPU): the forward of one view (project -> bin/sort -> composite -> depth fill +
surface normal, ~20 launches and ~1 ms of Python) is captured ONCE per resolution as a CUDA graph in `n_slots` copies
that write into their own static output maps; a view is then one 148-byte camera upload + one graph launch.  With
`to_host=True` the selected maps of slot s are copied to pinned host buffers on a side stream while slot s+1 renders, and
a view is handed out when its copy has landed.  The intersection buffers have a fixed capacity inside a graph: every
replay's count goes to a rasterize.CountWatch on the copy stream, and a view that needed more is rendered again after
re-capturing with a larger capacity — the consumer never sees a truncated render.  The static camera block and the
capture recipe are graph_step.py's.

`graph=False` is the plain loop (also what non-CUDA models, i.e. the CPU-proxy tests, use).
"""
from __future__ import annotations

from typing import Dict, Iterable, Iterator, List, Optional, Sequence, Tuple

import torch
from torch import Tensor

from .graph_step import StaticCamera, capture_slots
from .rasterize import CountWatch, DnrCapacityError, grow, suggested_capacity

DEFAULT_KEYS = ("rgb", "depth", "normal", "surface_normal", "accumulation")
RENDER_GROWTH = 1.3  # headroom over the count of an overflowing view (or, without statistics, of the first view)


class _ForwardGraphs:
    """`n_slots` captured copies of model.get_outputs for one resolution."""

    def __init__(self, model, camera, keys: Sequence[str], n_slots: int, capacity: int):
        self.model, self.keys, self.n_slots = model, tuple(keys), n_slots
        self.cam = StaticCamera((int(camera.width.flatten()[0]), int(camera.height.flatten()[0])), model.device, capacity)
        self._camera = camera
        self._capture()

    def _eager(self, slot: int) -> Tuple[Dict[str, Tensor], Tensor]:
        m = self.model
        m.__dict__["_graph_cam"] = self.cam
        try:
            out = m.get_outputs(self._camera)
            return {k: out[k] for k in self.keys if k in out}, m.raster_out.info["n_isects_dev"]
        finally:
            m.__dict__["_graph_cam"] = None

    @torch.no_grad()
    def _capture(self) -> None:
        self.cam.load(self._camera)
        self.graphs = self.maps = self.counts = ()  # release the old graphs and their maps before capturing new ones
        self.graphs, outs = capture_slots(self._eager, self.n_slots, 2, self.model.device)
        self.maps, self.counts = zip(*outs)  # per slot: the static output maps and the intersection count


class ViewRenderer:
    def __init__(self, model, keys: Sequence[str] = DEFAULT_KEYS, to_host: bool = False, n_host_buffers: int = 2,
                 graph: Optional[bool] = None, n_slots: int = 2):
        self.model, self.keys, self.to_host = model, tuple(keys), to_host
        self._host: list = [None] * n_host_buffers
        self._events: list = [None] * n_host_buffers
        self.graph = (model.device.type == "cuda") if graph is None else bool(graph)
        self.n_slots = max(2, n_slots) if to_host else max(1, n_slots)
        self._graphs: Dict[Tuple[int, int], _ForwardGraphs] = {}
        self.recaptures = 0

    # ------------------------------------------------------------------ plain loop
    @torch.no_grad()
    def _render_eager(self, cameras: Iterable) -> Iterator[Tuple[int, Dict[str, Tensor]]]:
        m = self.model
        pending: Optional[Tuple[int, int]] = None
        for idx, cam in enumerate(cameras):
            out = m.get_outputs(cam)
            maps = {k: out[k] for k in self.keys if k in out}
            if not self.to_host:
                yield idx, maps
                continue
            slot = idx % len(self._host)
            if self._host[slot] is None:
                self._host[slot] = {k: torch.empty(v.shape, dtype=v.dtype).pin_memory() if torch.cuda.is_available()
                                    else torch.empty(v.shape, dtype=v.dtype) for k, v in maps.items()}
            for k, v in maps.items():
                self._host[slot][k].copy_(v, non_blocking=True)
            ev = torch.cuda.Event() if torch.cuda.is_available() else None
            if ev is not None:
                ev.record()
            self._events[slot] = ev
            if pending is not None:  # hand out the previous view while this one renders / copies
                yield self._finish(*pending)
            pending = (idx, slot)
        if pending is not None:
            yield self._finish(*pending)

    def _finish(self, idx: int, slot: int):
        ev = self._events[slot]
        if ev is not None:
            ev.synchronize()
        return idx, self._host[slot]

    # ------------------------------------------------------------------ captured forward
    def _graphs_for(self, cam) -> _ForwardGraphs:
        m = self.model
        key = (int(cam.width.flatten()[0]), int(cam.height.flatten()[0]))
        fg = self._graphs.get(key)
        if fg is None or fg.model.num_points != m.num_points:
            cfg = m.config
            with torch.no_grad():  # without sync-free statistics for this size, one synchronous view sizes the capacity
                cap = suggested_capacity(m.num_points, key[0], key[1], cfg.predict_normals, cfg.exact_isect_lists, m.device.index,
                                         cfg.list_shift)
                if cap <= 0:
                    m.get_outputs(cam)
                    cap = grow(int(m.raster_out.info["n_isects_dev"]), RENDER_GROWTH)
            fg = self._graphs[key] = _ForwardGraphs(m, cam, self.keys, self.n_slots, cap)
        return fg

    @torch.no_grad()
    def _render_graphed(self, cameras: Iterable) -> Iterator[Tuple[int, Dict[str, Tensor]]]:
        cams = list(cameras)
        if not cams:
            return
        dev = self.model.device
        copy_stream = torch.cuda.Stream(device=dev)
        compute = torch.cuda.current_stream()
        n_slots = self.n_slots
        watch = CountWatch()
        host = [None] * n_slots            # pinned {key: tensor} per slot (to_host)
        rendered = [torch.cuda.Event() for _ in range(n_slots)]
        copied = [torch.cuda.Event() for _ in range(n_slots)]
        busy = [False] * n_slots
        inflight: List[Tuple[int, int, _ForwardGraphs, dict]] = []  # (view index, slot, graphs, count ticket) in order

        def submit(idx):
            cam = cams[idx]
            fg = self._graphs_for(cam)
            slot = idx % n_slots
            if busy[slot]:
                compute.wait_event(copied[slot])  # the copy that still reads this slot's static maps
            fg.cam.load(cam)
            fg.graphs[slot].replay()
            rendered[slot].record(compute)
            if self.to_host and (host[slot] is None or any(host[slot][k].shape != v.shape for k, v in fg.maps[slot].items())):
                host[slot] = {k: torch.empty(v.shape, dtype=v.dtype).pin_memory() for k, v in fg.maps[slot].items()}
            with torch.cuda.stream(copy_stream):
                copy_stream.wait_event(rendered[slot])
                ticket = watch.observe(fg.counts[slot], fg.cam.capacity)
                if self.to_host:
                    for k, v in fg.maps[slot].items():
                        host[slot][k].copy_(v, non_blocking=True)
                copied[slot].record(copy_stream)
            busy[slot] = True
            inflight.append((idx, slot, fg, ticket))

        def collect():
            idx, slot, fg, ticket = inflight.pop(0)
            copied[slot].synchronize()
            try:
                watch.check(ticket)
            except DnrCapacityError:  # truncated: grow, re-capture, and submit this view and those in flight again
                for _, s2, _, _ in inflight:  # drain what is in flight on the old graphs first
                    copied[s2].synchronize()
                fg.cam.capacity = grow(ticket["count"], RENDER_GROWTH)
                fg._capture()
                self.recaptures += 1
                redo = [idx] + [i for i, _, _, _ in inflight]
                inflight.clear()
                busy[:] = [False] * n_slots
                for j in redo:  # back in flight in order; collect() checks each of them again
                    submit(j)
                return None
            return idx, (host[slot] if self.to_host else fg.maps[slot])

        depth = n_slots - 1 if self.to_host else 0  # views in flight while the caller consumes one
        nxt = 0
        while nxt < len(cams) or inflight:
            while nxt < len(cams) and len(inflight) <= depth:
                submit(nxt)
                nxt += 1
            item = collect()
            if item is not None:
                yield item

    @torch.no_grad()
    def render(self, cameras: Iterable) -> Iterator[Tuple[int, Dict[str, Tensor]]]:
        """Yields (view index, {key: map}) in order.  With to_host=True the maps are pinned host tensors whose copy has
        completed when they are yielded; the next view is already rendering while the caller consumes them.  The buffers
        (host buffers, or the graph's static device maps with to_host=False) are reused round-robin: consume (or copy) a
        view's maps before asking for the next one."""
        m = self.model
        was_training = m.training
        m.eval()
        try:
            it = self._render_graphed(cameras) if (self.graph and m.device.type == "cuda") else self._render_eager(cameras)
            for item in it:
                yield item
        finally:
            m.train(was_training)
