"""oracle/raster_ref.backward, the fp64 per-Gaussian backward that tests/test_gpu_raster_backward.py holds
`raster_bwd_kernel` to.

  * its 13 signed slots equal torch fp64 autograd through a differentiable restatement of `composite` with the decisions
    frozen (the colour / depth route from means2d, the normal route from detached means2d, quirk B3), on the GPU test's
    constructed cases;
  * on the parity scenes with exact lists, v_means2d and |v_means2d| equal what oracle/gsplat_ref gives through autograd
    and its absgrad hooks;
  * central finite differences of `composite` agree on a tile whose decisions are far from every threshold;
  * each kernel mistake of BWD_SLIPS, restated in fp64, leaves the GPU test's acceptance rule on that test's own cases by
    10x or more; and the norm-wise relative change each one makes per slot on the scenes of
    tests/test_gpu_backward_edges.py is printed: four of them stay below those tests' 1e-3 on some or all of the scenes.
"""
import numpy as np
import pytest
import torch

from oracle import dn_ref
from oracle import gsplat_ref as G
from oracle import raster_ref as R
from tests.helpers import oracle_outputs, scene_and_camera
from tests.raster_cases import BWD_ATOL, BWD_RTOL, Case, generic, listed, upstream
from tests.test_gpu_parity import CASES

F64 = torch.float64
SIGNED = [0, 1, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14]


def _state(ref: R.RasterRef, f32: bool) -> dict:
    st = dict(alpha=ref.alpha, depth=ref.depth, normal=ref.normal, normal_norm=ref.normal_norm, clamp_mask=ref.clamp_mask)
    return {k: (v.astype(np.float32) if f32 and k != "clamp_mask" else v) for k, v in st.items()}


def _upstream(H, W, seed=0, dtype=F64):
    g = torch.Generator().manual_seed(seed)
    return dict(rgb=2 * torch.rand(H, W, 3, generator=g, dtype=dtype) - 1, depth=2 * torch.rand(H, W, generator=g, dtype=dtype) - 1,
                normal=2 * torch.rand(H, W, 3, generator=g, dtype=dtype) - 1, alpha=2 * torch.rand(H, W, generator=g, dtype=dtype) - 1)


def autograd_slots(c: Case, up: dict, keep: dict) -> np.ndarray:
    """[N, 13] gradients of sum(up * outputs) by torch autograd, per tile over the entries `keep` says were composited."""
    names = ("means2d", "conics", "opac", "colors", "depths", "normals_cam")
    P = {k: torch.tensor(np.asarray(getattr(c, k), np.float64), requires_grad=True) for k in names}
    bg = torch.tensor(c.background, dtype=F64)
    zero = torch.zeros((), dtype=F64)
    loss = zero
    for (y0, y1, x0, x1, g, _pos, live, _a, _v, _dx, _dy) in keep.values():
        if g.size == 0:
            continue
        gi, lv = torch.from_numpy(g), torch.from_numpy(live)
        h, w_ = y1 - y0, x1 - x0
        py = (torch.arange(y0, y1, dtype=F64) + 0.5).repeat_interleave(w_)
        px = (torch.arange(x0, x1, dtype=F64) + 0.5).repeat(h)

        def walk(m2):
            dx, dy = m2[gi, 0][None] - px[:, None], m2[gi, 1][None] - py[:, None]
            con = P["conics"][gi]
            sig = 0.5 * (con[:, 0][None] * dx * dx + con[:, 2][None] * dy * dy) + con[:, 1][None] * dx * dy
            a = torch.where(lv, torch.clamp(P["opac"][gi][None] * torch.exp(-sig), max=R.ALPHA_MAX), zero)
            om = 1.0 - a
            Tb = torch.cumprod(torch.cat([torch.ones(om.shape[0], 1, dtype=F64), om[:, :-1]], 1), 1)
            return a * Tb, torch.prod(om, 1)

        tile = lambda x: x[y0:y1, x0:x1].reshape((h * w_,) + x.shape[2:])  # noqa: E731
        w1, T1 = walk(P["means2d"])
        S = w1 @ torch.cat([P["colors"], P["depths"][:, None]], 1)[gi]
        ao = 1.0 - T1
        loss = loss + (tile(up["rgb"]) * torch.clamp(S[:, :3] + T1[:, None] * bg, 0.0, 1.0)).sum()
        loss = loss + (tile(up["depth"]) * (S[:, 3] / torch.clamp(ao, min=1e-10))).sum() + (tile(up["alpha"]) * ao).sum()
        w2, T2 = walk(P["means2d"].detach())
        n = w2 @ P["normals_cam"][gi] + T2[:, None]
        loss = loss + (tile(up["normal"]) * (n / n.norm(dim=-1, keepdim=True) + 1.0) * 0.5).sum()
    loss.backward()
    gr = lambda k: P[k].grad if P[k].grad is not None else torch.zeros_like(P[k])  # noqa: E731
    return torch.cat([gr("means2d"), gr("conics"), gr("opac")[:, None], gr("colors"), gr("depths")[:, None],
                      gr("normals_cam")], 1).numpy()


CONSTRUCTED = {
    "frame-81x49": lambda: generic(81, 49, seed=81),                                   # test_frames
    "clamp-bg": lambda: generic(75, 53, seed=21, color=(-0.5, 1.5), background=(-0.2, 0.5, 1.3)),  # clamp mask
    "saturate-129": lambda: listed((300, 640, 130), seed=2, kind="opaque", stop_at=129),  # test_whole_tile_saturates
    "shift2": lambda: generic(81, 49, shift=2, seed=5),
}


@pytest.mark.parametrize("name", list(CONSTRUCTED))
def test_equals_autograd_with_frozen_decisions(name):
    c = CONSTRUCTED[name]()
    keep: dict = {}
    ref = c.oracle(eps=0.0, keep=keep)
    up = _upstream(c.height, c.width)
    b = c.backward({k: v.numpy() for k, v in up.items()}, _state(ref, f32=False), pre=(ref, keep))
    ag = autograd_slots(c, up, keep)
    scale = b.mass[:, SIGNED].max(0)
    assert (scale > 0).all()
    err = np.abs(b.grads[:, SIGNED] - ag).max(0) / scale
    assert err.max() <= 1e-12, f"{name}: relative error per slot {err}"
    assert (b.grads[:, 15] == 0).all() and (b.grads[:, 2:4] >= np.abs(b.grads[:, 0:2]) * (1 - 1e-12)).all()


@pytest.mark.parametrize("case", CASES, ids=["1000@128x128", "3000@200x136", "400@75x53"])
def test_means2d_and_absgrad_equal_gsplat_ref_hooks(case):
    params, cam = scene_and_camera(**case)
    p, out = oracle_outputs(params, cam, dtype=F64, requires_grad=True, predict_normals=True, collect_absgrad=True)
    info = out["info"]
    info["means2d"].retain_grad()
    _, ncam = dn_ref.gaussian_normals(p["quats"], p["scales"], p["means"], cam["c2w"].double())
    W, H = cam["width"], cam["height"]
    offs = torch.cat([info["isect_offsets"], torch.tensor([info["flatten_ids"].shape[0]], dtype=torch.int32)])
    c = Case(means2d=info["means2d"].detach(), conics=info["conics"].detach(), opac=info["opacities"].detach(),
             colors=info["colors"].detach(), depths=info["depths"].detach(), normals_cam=ncam.detach(), radii=info["radii"],
             flatten_ids=info["flatten_ids"], tile_offsets=offs, list_shift=0, width=W, height=H,
             background=tuple(float(x) for x in out["background"]))
    keep: dict = {}
    ref = c.oracle(eps=0.0, keep=keep)
    up = _upstream(H, W, seed=3)
    far = torch.from_numpy(ref.margin > 1e-6)  # gsplat_ref decides with the fp64 thresholds, this oracle with fp32 ones
    up = {k: torch.where(far.reshape(far.shape + (1,) * (v.dim() - 2)), v, torch.zeros((), dtype=F64)) for k, v in up.items()}
    assert float(far.double().mean()) > 0.999
    loss = (up["rgb"] * out["rgb"]).sum() + (up["depth"] * out["depth"][..., 0]).sum() + \
        (up["normal"] * out["normal"]).sum() + (up["alpha"] * out["accumulation"][..., 0]).sum()
    loss.backward()
    b = c.backward({k: v.numpy() for k, v in up.items()}, _state(ref, f32=False), pre=(ref, keep))
    want = info["means2d"].grad.numpy()
    absg = G.absgrad_from_hooks(info["hooks"], info["conics"], info["opacities"], want.shape[0]).numpy()
    for got, w, what in ((b.grads[:, 0:2], want, "v_means2d"), (b.grads[:, 2:4], absg, "|v_means2d|")):
        assert np.abs(w).max() > 0
        assert np.abs(got - w).max() <= 1e-11 * np.abs(w).max(), f"{what}: {np.abs(got - w).max():.3e}"


def test_finite_differences_far_from_thresholds():
    g = torch.Generator().manual_seed(17)
    n = 12
    m = 3.0 + 10.0 * torch.rand(n, 2, generator=g, dtype=F64)
    c = Case(means2d=m, conics=torch.stack([0.02 + 0.02 * torch.rand(n, generator=g, dtype=F64), 0.004 * (2 * torch.rand(n, generator=g, dtype=F64) - 1),
                                            0.02 + 0.02 * torch.rand(n, generator=g, dtype=F64)], 1),
             opac=0.2 + 0.5 * torch.rand(n, generator=g, dtype=F64), colors=0.2 + 0.3 * torch.rand(n, 3, generator=g, dtype=F64),
             depths=1.0 + torch.rand(n, generator=g, dtype=F64), normals_cam=torch.nn.functional.normalize(torch.randn(n, 3, generator=g, dtype=F64), dim=1),
             radii=torch.full((n,), 40, dtype=torch.int32), flatten_ids=torch.arange(n, dtype=torch.int32),
             tile_offsets=torch.tensor([0, n], dtype=torch.int32), list_shift=0, width=16, height=16, background=(0.2, 0.3, 0.4))
    keep: dict = {}
    ref = c.oracle(eps=0.0, keep=keep)
    assert ref.margin.min() > 1e-3 and not ref.clamped.any() and (ref.clamp_mask == 7).all() and ref.ncomp.min() == n
    up = {k: v.numpy() for k, v in _upstream(16, 16, seed=5).items()}

    def loss(cc, normal=True):
        r = cc.oracle(eps=0.0)
        s = (up["rgb"] * r.rgb).sum() + (up["depth"] * r.depth).sum() + (up["alpha"] * r.alpha).sum()
        return s + ((up["normal"] * r.normal).sum() if normal else 0.0)

    b = c.backward(up, _state(ref, f32=False), pre=(ref, keep))
    b_nn = c.backward(dict(up, normal=np.zeros_like(up["normal"])), _state(ref, f32=False))
    fields = [("means2d", 0, 0), ("means2d", 1, 1), ("conics", 0, 4), ("conics", 1, 5), ("conics", 2, 6), ("opac", None, 7),
              ("colors", 0, 8), ("colors", 1, 9), ("colors", 2, 10), ("depths", None, 11), ("normals_cam", 0, 12),
              ("normals_cam", 1, 13), ("normals_cam", 2, 14)]
    for name, col, slot in fields:
        normal = slot >= 4  # the normal route does not reach means2d (B3): compare those without v_normal
        want = (b if normal else b_nn).grads[:, slot]
        for gi in range(n):
            x = getattr(c, name)
            hstep = 1e-6 * max(1.0, float(x[gi].abs().max()))
            fd = []
            for sgn in (1, -1):
                y = x.clone()
                if col is None:
                    y[gi] += sgn * hstep
                else:
                    y[gi, col] += sgn * hstep
                fd.append(loss(Case(**{**c.__dict__, name: y}), normal))
            d = (fd[0] - fd[1]) / (2 * hstep)
            assert abs(d - want[gi]) <= 1e-6 * max(1.0, np.abs(want).max()), (name, col, gi, d, want[gi])


# ----------------------------------------------------------------------------------------------------- slips
def _gpu_case_refs(c: Case, normals=True):
    """The GPU test's reference on case c: fp32 forward state, seeded upstream zero under the band."""
    keep: dict = {}
    ref = c.oracle(normals, eps=0.0, keep=keep)
    up = upstream(c, ref)
    st = _state(ref, f32=True)
    return ref, keep, up, st, c.backward(up, st, normals, pre=(ref, keep))


_SLIP_CACHE: dict = {}


def _slip_worst(slip):
    worst = 0.0
    for name in ("frame-81x49", "clamp-bg", "saturate-129"):
        if name not in _SLIP_CACHE:
            c = CONSTRUCTED[name]()
            _SLIP_CACHE[name] = (c,) + _gpu_case_refs(c)
        c, ref, keep, up, st, good = _SLIP_CACHE[name]
        bad = c.backward(up, st, pre=(ref, keep), slip=slip)
        worst = max(worst, R.judge_bwd(good, bad.grads, BWD_RTOL, BWD_ATOL).worst)
    return worst


def test_the_correct_result_passes_its_own_rule():
    for name in ("frame-81x49", "clamp-bg"):
        c = CONSTRUCTED[name]()
        _, _, _, _, good = _gpu_case_refs(c)
        v = R.judge_bwd(good, good.grads.astype(np.float32), BWD_RTOL, BWD_ATOL)
        assert v.ok and v.worst < 0.1, v.worst_what


@pytest.mark.parametrize("slip", R.BWD_SLIPS)
def test_slip_leaves_the_acceptance_rule(slip):
    w = _slip_worst(slip)
    assert w >= 10.0, f"{slip}: worst ratio to the bound {w:.3g}"


def _edges_scenes():
    """(name, Case, upstream) of tests/test_gpu_backward_edges.py's scenes, from the fp64 oracle's projection, with the
    upstream images of its route "all" (rgb, 0.1 depth, normal, alpha with seeded weights)."""
    from tests.test_gpu_backward_edges import clamp_scene

    out = []
    scenes = [("ragged-81x49", scene_and_camera(400, 81, 49, view=0)), ("ragged-75x53", scene_and_camera(400, 75, 53, view=0)),
              ("clamp", clamp_scene()[:2])]
    for name, (params, cam) in scenes:
        p, o = oracle_outputs(params, cam, dtype=F64, predict_normals=True)
        info = o["info"]
        _, ncam = dn_ref.gaussian_normals(p["quats"], p["scales"], p["means"], cam["c2w"].double())
        W, H = cam["width"], cam["height"]
        offs = torch.cat([info["isect_offsets"], torch.tensor([info["flatten_ids"].shape[0]], dtype=torch.int32)])
        c = Case(means2d=info["means2d"], conics=info["conics"], opac=info["opacities"], colors=info["colors"],
                 depths=info["depths"], normals_cam=ncam, radii=info["radii"], flatten_ids=info["flatten_ids"], tile_offsets=offs,
                 list_shift=0, width=W, height=H, background=tuple(float(x) for x in o["background"]))
        g = torch.Generator().manual_seed(0)
        w = dict(rgb=torch.rand(H, W, 3, generator=g), depth=torch.rand(H, W, 1, generator=g),
                 normal=torch.rand(H, W, 3, generator=g), alpha=torch.rand(H, W, 1, generator=g))
        up = dict(rgb=w["rgb"].numpy(), depth=0.1 * w["depth"][..., 0].numpy(), normal=w["normal"].numpy(), alpha=w["alpha"][..., 0].numpy())
        out.append((name, c, up))
    return out


GROUPS = {"means2d": [0, 1], "|means2d|": [2, 3], "conics": [4, 5, 6], "opacity": [7], "rgb": [8, 9, 10], "depth": [11],
          "normal": [12, 13, 14]}


def test_norm_wise_visibility_of_each_slip(capsys):
    """Prints, per slip, the largest and smallest over the scenes of the norm-wise relative change of each slot group:
    a slip whose change stays under 1e-3 in a group on some scene is invisible to a 1e-3 norm-wise test there."""
    rows = {}
    for name, c, up in _edges_scenes():
        keep: dict = {}
        ref = c.oracle(eps=0.0, keep=keep)
        st = _state(ref, f32=False)
        good = c.backward(up, st, pre=(ref, keep))
        for slip in R.BWD_SLIPS:
            bad = c.backward(up, st, pre=(ref, keep), slip=slip)
            for gname, cols in GROUPS.items():
                den = np.linalg.norm(good.grads[:, cols])
                rel = np.linalg.norm(bad.grads[:, cols] - good.grads[:, cols]) / den if den > 0 else 0.0
                rows.setdefault((slip, gname), []).append(rel)
    with capsys.disabled():
        print("\nnorm-wise relative change per slot group, min .. max over the test_gpu_backward_edges scenes")
        print(f"{'slip':16s}" + "".join(f"{g:>22s}" for g in GROUPS))
        for slip in R.BWD_SLIPS:
            print(f"{slip:16s}" + "".join(f"{min(rows[(slip, g)]):>10.1e} ..{max(rows[(slip, g)]):>8.1e}" for g in GROUPS))
    assert all(np.isfinite(v).all() for v in rows.values())
