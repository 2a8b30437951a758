"""GPU tests of the projection kernels (csrc/project.cu) per Gaussian, against the fp32 oracle and an fp64 reference.

dnr_project_fwd and dnr_project_bwd are driven directly through the C ABI.  The references:
  * integer outputs (radii, tiles per Gaussian, depth sort keys) against gsplat_ref.project_gaussians / tile_bounds in
    fp32, bit for bit: the kernel is built with -fmad=false in the oracle's operation order.  The raw-parameter path
    gets the oracle exp(scales) evaluated by torch on the device, which calls the same expf as the kernel;
  * float outputs against oracle/project_ref.forward64 (fp64) per Gaussian;
  * the packed raster records against the kernel's own outputs, bit for bit, and the log-domain culling thresholds
    within 2 ulp;
  * gradients against oracle/project_ref.vjp64, the fp64 VJP of the same outputs, per Gaussian and parameter group,
    with the kernel's conventions where the projection is not differentiable (project_ref.Branches);
  * the flag compaction and the buffer contract of dnr_project_bwd (accumulate once per flagged Gaussian, consume its
    record, leave everything else alone) bit for bit against a run with every Gaussian flagged.
Nothing here compares one norm over all Gaussians: a wrong term that reaches only a few Gaussians fails its rows.
"""
import ctypes as C
import math

import pytest
import torch

from oracle import gsplat_ref as G
from oracle import project_ref as P

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]

F32, F64 = torch.float32, torch.float64
TILE = 16
# Per Gaussian and parameter group, project_ref's bound: RTOL of the row's largest |g64|, ATOL of the group's, and SENS
# times how far fp64 itself moves under a 1e-5 relative perturbation of the inputs (large only where the problem is
# ill-conditioned).  Needles (cond(cov2d) > 1e3) are reported in their own bucket.
VIEWMAT_RTOL = 1e-4  # v_viewmat (a sum over all Gaussians) per entry, relative to its largest entry
SH_SETS = [(0, 1), (1, 4), (2, 9), (3, 16), (1, 16), (0, 9)]  # (active degree, stored bases)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _lib():
    from dn_splatter_b200 import _lib as L

    return L, L.load()


def _case(kind="random", n=2000, seed=0, deg=3, bases=16, **kw):
    if kind == "edge_on":
        return P.edge_on_case(n, seed, sh_bases=bases, sh_degree=deg, **kw)
    return P.random_case(n, seed, sh_bases=bases, sh_degree=deg, kind=kind, **kw)


# ----------------------------------------------------------------------------------------------------- ABI
class Run:
    """One dnr_project_fwd on a Case; keeps the device tensors for the backward."""

    def __init__(self, case: P.Case, host=False):
        L, lib = _lib()
        self.case, self.host = case, host
        n = case.n
        dev = {k: v.contiguous().cuda() for k, v in case.params.items()}
        self.dev = dev
        nan = lambda *s: torch.full(s, float("nan"), dtype=F32, device="cuda")  # noqa: E731
        ones = lambda *s: torch.full(s, -7, dtype=torch.int32, device="cuda")  # noqa: E731
        rec_f = L.REC_FLOATS_N if case.normals else L.REC_FLOATS
        self.out = dict(radii=ones(n), means2d=nan(n, 2), depths=nan(n), conics=nan(n, 3), opac_act=nan(n),
                        compensations=nan(n), colors=nan(n, 3), normals_world=nan(n, 3), tiles_per_gauss=ones(n),
                        depth_keys=ones(n), records=nan(n, rec_f), cull_lim=nan(n))
        self.cam = dict(viewmat=case.viewmat.contiguous().cuda(), K=case.K.contiguous().cuda(),
                        c2w=case.c2w.contiguous().cuda())
        a = self.args(L)
        for k, t in self.out.items():
            if k == "normals_world" and not case.normals:
                continue
            if k == "compensations" and not case.antialiased:
                continue
            setattr(a, k, t.data_ptr())
        L.check(lib.dnr_project_fwd(C.byref(a), _stream()), "dnr_project_fwd")
        torch.cuda.synchronize()
        self.host_out = {k: v.cpu() for k, v in self.out.items()}

    def args(self, L):
        c = self.case
        a = L.DnrArgs()
        a.n_gauss, a.width, a.height, a.tile_size = c.n, c.width, c.height, TILE
        a.sh_degree, a.sh_bases = c.sh_degree, c.sh_bases
        flags = 0
        if c.activated:
            flags |= L.FLAG_ACTIVATED
        if c.antialiased:
            flags |= L.FLAG_ANTIALIASED
        if c.normals:
            flags |= L.FLAG_NORMALS
        a.near_plane, a.far_plane, a.eps2d, a.radius_clip = c.near_plane, c.far_plane, c.eps2d, c.radius_clip
        if self.host:
            flags |= L.FLAG_HOST_CAMERA
            a.host_cam[:] = (c.viewmat.reshape(16).tolist() + [float(c.K[0, 0]), float(c.K[1, 1]), float(c.K[0, 2]),
                                                               float(c.K[1, 2])] + c.c2w.reshape(12).tolist())
        else:
            a.viewmat, a.K = self.cam["viewmat"].data_ptr(), self.cam["K"].data_ptr()
            if c.normals:
                a.c2w = self.cam["c2w"].data_ptr()
        a.flags = flags
        d = self.dev
        a.means, a.quats, a.scales, a.opacities, a.sh_dc = (d[k].data_ptr() for k in
                                                            ("means", "quats", "scales", "opacities", "sh_dc"))
        if c.sh_bases > 1:
            a.sh_rest = d["sh_rest"].data_ptr()
        a.radii = self.out["radii"].data_ptr()
        return a

    def backward(self, grad_records, touched, prefill=None, viewmat=False, m2d_prefill=None):
        """dnr_project_bwd with FLAG_ACCUMULATE into buffers that start at `prefill` (zeros by default): the gradient
        buffers, v_means2d / v_means2d_abs, the grad_records after the call and v_viewmat (or None)."""
        L, lib = _lib()
        n = self.case.n
        a = self.args(L)
        a.flags |= L.FLAG_ACCUMULATE
        gr = grad_records.contiguous().cuda()
        tc = touched.contiguous().cuda()
        bufs = {k: (torch.zeros_like(v) if prefill is None else prefill[k].clone().cuda()) for k, v in self.dev.items()}
        m2 = torch.zeros(n, 2, dtype=F32) if m2d_prefill is None else m2d_prefill[0]
        m2a = torch.zeros(n, 2, dtype=F32) if m2d_prefill is None else m2d_prefill[1]
        bufs["means2d"], bufs["means2d_abs"] = m2.clone().cuda(), m2a.clone().cuda()
        vv = torch.zeros(4, 4, dtype=F32, device="cuda") if viewmat else None
        a.grad_records, a.touched = gr.data_ptr(), tc.data_ptr()
        a.v_means, a.v_quats, a.v_scales, a.v_opacities, a.v_sh_dc = (
            bufs[k].data_ptr() for k in ("means", "quats", "scales", "opacities", "sh_dc"))
        if self.case.sh_bases > 1:
            a.v_sh_rest = bufs["sh_rest"].data_ptr()
        a.v_means2d, a.v_means2d_abs = bufs["means2d"].data_ptr(), bufs["means2d_abs"].data_ptr()
        if vv is not None:
            a.v_viewmat = vv.data_ptr()
        L.check(lib.dnr_project_bwd(C.byref(a), _stream()), "dnr_project_bwd")
        torch.cuda.synchronize()
        return {k: v.cpu() for k, v in bufs.items()}, gr.cpu(), None if vv is None else vv.cpu()


def _seeded_records(n, seed, only_normal=False):
    g = torch.Generator().manual_seed(seed)
    gr = torch.randn(n, 16, generator=g)
    gr[:, 15] = 0.0
    if only_normal:
        gr[:, :12] = 0.0
    return gr


# ----------------------------------------------------------------------------------------------------- error measures
def check_rows(got, want, spr, rows, case, what, keys, kind="grad"):
    """Every row of `rows` within project_ref's per-Gaussian bound, with the factors of `kind` ("grad" / "fwd") and
    of the case's mode (classic / antialiased); needles, with their own factor, and the rest are reported apart."""
    rtol, atol = (P.GRAD_RTOL, P.GRAD_ATOL) if kind == "grad" else (P.FWD_RTOL, 0.0)
    sens, needle = P.sens(kind, case), P.needles(case)
    for k in keys:
        for name, sel, f in (("regular", rows & ~needle, sens[k]), ("needle", rows & needle, P.needle_sens(kind, case))):
            rr = P.row_ratio(got[k], want[k], spr[k], sel, rtol, atol, f)
            worst = int(rr.argmax())
            assert float(rr[worst]) <= 1.0, (
                f"{what} {kind} {k} [{name}] Gaussian {worst}: {float(rr[worst]):.2f} x the bound; "
                f"kernel {got[k][worst].flatten()[:6].tolist()} fp64 {want[k][worst].flatten()[:6].tolist()}")


# ----------------------------------------------------------------------------------------------------- forward
def _oracle32(case, run):
    """gsplat_ref fp32 projection + tile boxes of the case, with the kernel's activations."""
    s = case.params["scales"]
    if not case.activated:
        s = torch.exp(s.cuda()).cpu()  # the kernel's expf
    proj = G.project_gaussians(case.params["means"], case.params["quats"], s, case.viewmat, case.K, case.width,
                               case.height, eps2d=case.eps2d, near_plane=case.near_plane, far_plane=case.far_plane,
                               radius_clip=case.radius_clip)
    tw, th = -(-case.width // TILE), -(-case.height // TILE)
    x0, y0, x1, y1 = G.tile_bounds(proj["means2d"], proj["radii"], TILE, tw, th)
    return proj, ((x1 - x0) * (y1 - y0)).to(torch.int32)


def _sigmoid32(case):
    o = case.params["opacities"]
    if case.activated:
        return o
    return (1.0 / (1.0 + torch.exp(-o.cuda()))).cpu()  # the kernel's 1 / (1 + expf(-o))


def _ulps(got, want):
    """|got - want| in units of the fp32 spacing at |want| (fp64 want)."""
    sp = torch.nextafter(want.float().abs(), torch.tensor(math.inf)).double() - want.float().abs().double()
    return ((got.double() - want).abs() / sp).nan_to_num(nan=0.0)


def check_forward(run: Run, what: str):
    case, o = run.case, run.host_out
    n = case.n
    proj, tpg = _oracle32(case, run)
    assert torch.equal(o["radii"], proj["radii"]), f"{what}: radii differ at {torch.nonzero(o['radii'] != proj['radii'])[:5].flatten().tolist()}"
    assert torch.equal(o["tiles_per_gauss"], tpg), f"{what}: tiles_per_gauss"
    vis = o["radii"] > 0
    keys = torch.where(vis, proj["depths"].view(torch.int32), torch.tensor(-1, dtype=torch.int32))  # 0xFFFFFFFF culled
    assert torch.equal(o["depth_keys"], keys), f"{what}: depth_keys"
    if case.activated:  # the oracle's fp32 floats, bit for bit (its conics differ in the last bits: fp64 below)
        for k, w in (("means2d", proj["means2d"]), ("depths", proj["depths"])):
            assert torch.equal(o[k], w), f"{what}: {k} differs from the fp32 oracle"
    # culled rows: all zero, but depth_keys, cull_lim = -1 and normals_world
    cul = ~vis
    for k in ("means2d", "depths", "conics", "opac_act", "colors", "records"):
        assert bool((o[k][cul] == 0).all()), f"{what}: culled {k} not zero"
    assert bool((o["cull_lim"][cul] == -1).all()), f"{what}: culled cull_lim"
    if case.antialiased:
        assert bool((o["compensations"][cul] == 0).all()), f"{what}: culled compensations"
    # float outputs against fp64 per Gaussian; the normal's sign is the one the kernel rendered
    flip = _kernel_flip(case, o) if case.normals else None
    br = P.Branches.from_fp32(case, flip=flip, comp_pos=o["compensations"] > 0 if case.antialiased else None)
    fn = lambda c: P.forward64(c, br)  # noqa: E731
    with torch.no_grad():
        ref, spr = fn(case), P.spread(fn, case)
    ref["depth"], spr["depth"] = ref["depth"][:, None], spr["depth"][:, None]
    got = dict(means2d=o["means2d"], depth=o["depths"], conics=o["conics"], opac=o["opac_act"], rgb=o["colors"])
    keys = ["means2d", "depth", "conics", "opac", "rgb"]
    if case.antialiased:
        got["comp"] = o["compensations"]
        keys.append("comp")
    rows = vis
    if case.antialiased:  # rank-deficient covariances: compensation of rounding size, compared where it is 0
        rows = vis & ((o["compensations"] == 0) | (ref["comp"] > 1e-3))
    if case.normals:
        got.update(normals_world=o["normals_world"], ncam=o["records"][:, 12:15])
        keys += ["ncam"]
        check_rows(got, ref, spr, torch.ones(n, dtype=torch.bool), case, what, ["normals_world"], kind="fwd")
        assert bool((o["records"][vis, 15] == 0).all())
        # away from ties (|cos| > 1e-5) the kernel flips where fp64 does
        cam = case.c2w[:, 3].double()
        v = torch.nn.functional.normalize(cam - case.params["means"].double(), dim=1)
        n64 = P.forward64(case, P.Branches.from_fp32(case, flip=torch.zeros(n, dtype=torch.bool)))["normals_world"]
        cos = (n64 * v).sum(1)
        clear = cos.abs() > 1e-5
        assert torch.equal(flip[clear], (cos < 0)[clear]), f"{what}: the forward's normal flip"
    check_rows(got, ref, spr, rows, case, what, keys, kind="fwd")
    # packed records against the outputs, bit for bit (nthr, cull_lim within 2 ulp)
    rec = o["records"][vis]
    l2e = torch.tensor(P.LOG2E, dtype=F32)
    hl2e = torch.tensor(-0.5, dtype=F32) * l2e
    A, B, Cc = o["conics"][vis].unbind(1)
    op = o["opac_act"][vis]
    assert torch.equal(rec[:, 0], o["means2d"][vis, 0]) and torch.equal(rec[:, 1], o["means2d"][vis, 1]), what
    assert torch.equal(rec[:, 2], hl2e * A) and torch.equal(rec[:, 3], -l2e * B), f"{what}: rec0 conic"
    assert torch.equal(rec[:, 4], hl2e * Cc) and torch.equal(rec[:, 5], op), f"{what}: rec1"
    assert torch.equal(rec[:, 7], o["radii"][vis].float()), f"{what}: rec1 radius"
    assert torch.equal(rec[:, 8:11], o["colors"][vis]) and torch.equal(rec[:, 11], o["depths"][vis]), f"{what}: rec2"
    zero_op = op == 0
    assert bool(torch.isinf(rec[zero_op, 6]).all() & (rec[zero_op, 6] > 0).all()), f"{what}: nthr at op = 0"
    # -log2(255 op) - 1e-3 and ln(255 op) + 0.1: 2 ulp of the log term (the sum may cancel to far below it)
    lg = -torch.log2((torch.tensor(255.0, dtype=F32) * op).double())
    _check_ulps(rec[~zero_op, 6], lg[~zero_op], -1e-3, f"{what}: nthr")
    op_pre = _sigmoid32(case)[vis]
    ln = torch.log((torch.tensor(255.0, dtype=F32) * op_pre).double())
    _check_ulps(o["cull_lim"][vis], ln, 0.1, f"{what}: cull_lim")
    return vis


def _check_ulps(got, log_term, add, what):
    """fp32(log term) + fp32(add) within 2 ulp of the log term (plus the final rounding)."""
    if got.numel() == 0:
        return
    want = log_term.float() + torch.tensor(add, dtype=F32)
    err = (got.double() - want.double()).abs()
    a = torch.maximum(log_term.abs(), want.double().abs()).float()
    ulp = (torch.nextafter(a, torch.tensor(math.inf)) - a).double()
    u = float((err / ulp).max())
    assert u <= 2.0, f"{what}: {u:.1f} ulp"


def _kernel_flip(case, o):
    """bool [N]: the kernel's forward negated the normal (its normals_world against the unflipped fp64 normal)."""
    n64 = P.forward64(case, P.Branches.from_fp32(case, flip=torch.zeros(case.n, dtype=torch.bool)))["normals_world"]
    return (o["normals_world"].double() * n64).sum(1) < 0


FWD_CASES = [(kind, act, aa, sh) for kind in ("random",) for act in (False, True) for aa in (False, True)
             for sh in SH_SETS] + [("clamped", False, False, (3, 16)), ("rank1", True, True, (1, 4)),
                                   ("edge_on", False, False, (3, 16))]


@pytest.mark.parametrize("kind,act,aa,sh", FWD_CASES,
                         ids=[f"{k}-{'act' if a else 'raw'}-{'aa' if aa else 'classic'}-deg{s[0]}b{s[1]}"
                              for k, a, aa, s in FWD_CASES])
def test_forward_matches_oracle_per_gaussian(kind, act, aa, sh):
    case = _case(kind, seed=FWD_CASES.index((kind, act, aa, sh)), deg=sh[0], bases=sh[1], activated=act,
                 antialiased=aa)
    vis = check_forward(Run(case), f"{kind} act={act} aa={aa} sh={sh}")
    assert 0 < int(vis.sum()) < case.n or kind != "random", "the random scene must have culled and visible Gaussians"


def check_expect(case, expect, o):
    """Each constructed placement took the branch it was placed for (the kernel's outputs and, for branches the kernel
    does not report, its fp32 decision emulated in its operation order)."""
    br = P.Branches.from_fp32(case)
    col32 = P.colors32(case)
    tx = -(-case.width // TILE)
    ty = -(-case.height // TILE)
    for label, (i, visible, extra) in expect.items():
        r = int(o["radii"][i])
        assert (r > 0) == visible, f"{label}: radius {r}, expected {'visible' if visible else 'culled'}"
        if extra is None:
            continue
        if isinstance(extra, bool):  # lim: the Jacobian clamp flag
            assert bool(br.clamp_x[i] | br.clamp_y[i]) == extra, f"{label}: clamp"
        elif isinstance(extra, tuple):  # colour_tie: colour + 0.5 == 0 exactly, and the gradient passes
            for c in extra:
                assert float(col32[i, c]) + 0.5 == 0.0 and bool(br.color_pass[i, c]), f"{label}: colour tie"
                assert float(o["colors"][i, c]) == 0.0, label
        elif visible:  # outside / radius_clip: the radius the placement was built for
            assert r == extra, f"{label}: radius {r} != {extra}"
    if "right inward" in expect:  # boxes clamped to the frame, ending in the ragged last tile column / row
        mx, my = o["means2d"].unbind(1)
        for label, axis, lim in (("left inward", 0, 0), ("top inward", 1, 0), ("right inward", 0, tx),
                                 ("bottom inward", 1, ty)):
            i, _, r = expect[label]
            m = float((mx, my)[axis][i])
            lo, hi = math.floor((m - r) / TILE), math.ceil((m + r) / TILE)
            assert lo < 0 if lim == 0 else hi > lim, f"{label}: the box is not clamped ({lo}, {hi})"
        assert case.width % TILE and case.height % TILE


@pytest.mark.parametrize("kind", P.BOUNDARY_KINDS)
def test_forward_constructed_boundaries(kind):
    """Axis-aligned camera (rotation I, fx = fy = 64, integer principal point, 100 x 70: ragged last tiles), Gaussians
    placed exactly on each branch point of the projection and one fp32 ulp to either side: z = near / far plane,
    |x/z| = 1.3 tan(fov) in x and y, mx +- r = 0 / W and my +- r = 0 / H, radius = radius_clip and radius_clip + 1,
    eps2d = 0 with rank-1 covariances (det = 0: culled), colours at exactly -0.5 + 0.5 = 0.  Every output is held to
    the fp32 oracle and fp64 as in the generic cases, and each placement asserts its branch."""
    case, expect = P.boundary_case(kind)
    run = Run(case)
    check_forward(run, f"boundary {kind}")
    check_expect(case, expect, run.host_out)


@pytest.mark.parametrize("kind", ["lim", "colour_tie"])
def test_backward_at_ties(kind):
    """The backward at the two ties whose convention the reference states: |x/z| = lim exactly counts as unclamped
    (one ulp past it is clamped, one ulp inside is not), and colour + 0.5 = 0 passes the gradient.  Per Gaussian
    against fp64 with those conventions."""
    case, expect = P.boundary_case(kind)
    _, br, got, want, rows = check_backward(case, f"tie {kind}")
    check_expect(case, expect, Run(case).host_out)
    assert bool(rows.all()), "every placement is visible and compared"
    if kind == "colour_tie":
        for i, _, chans in expect.values():
            for c in chans:
                assert float(got["sh_dc"][i, c]) != 0.0, "the tied channel's gradient passes"


# ----------------------------------------------------------------------------------------------------- backward
BWD_CASES = [(act, aa, normals, sh) for act in (False, True) for aa in (False, True) for normals in (True, False)
             for sh in SH_SETS[:5]]


def bwd_case(act, aa, normals, sh):
    """The scene of test_backward_matches_fp64_per_gaussian for one parameter set (its records: `records(case)`)."""
    return _case("random", seed=100 + BWD_CASES.index((act, aa, normals, sh)), deg=sh[0], bases=sh[1], activated=act,
                 antialiased=aa, normals=normals)


def records(case, only_normal=False):
    """The grad_records check_backward feeds the kernel for `case`."""
    return _seeded_records(case.n, seed=case.n + case.sh_bases, only_normal=only_normal)


def check_backward(case, what, only_normal=False, host=False, viewmat=False, compare=None):
    """Every Gaussian flagged; `compare` (bool [N] or None) narrows the rows compared with fp64."""
    run = Run(case, host=host)
    o = run.host_out
    n = case.n
    vis = o["radii"] > 0
    gr = records(case, only_normal)
    touched = torch.ones(n, dtype=torch.uint8)
    got, gr_after, vv = run.backward(gr, touched, viewmat=viewmat)
    flip = _kernel_flip(case, o) if case.normals else None
    br = P.Branches.from_fp32(case, flip=flip, comp_pos=o["compensations"] > 0 if case.antialiased else None)
    fn = lambda c: P.vjp64(c, br, gr, vis, viewmat=viewmat)  # noqa: E731
    want, spr = fn(case), P.spread(fn, case)
    assert bool((gr_after == 0).all()), f"{what}: grad_records not cleared"
    # means2d slots: the records' values of the visible Gaussians, bit for bit; zero elsewhere
    assert torch.equal(got["means2d"], torch.where(vis[:, None], gr[:, 0:2], torch.zeros(()))), f"{what}: v_means2d"
    assert torch.equal(got["means2d_abs"], torch.where(vis[:, None], gr[:, 2:4], torch.zeros(()))), f"{what}: abs"
    for k in P.PARAM_KEYS:  # radius 0: no gradient at all
        assert bool((got[k][~vis] == 0).all()), f"{what}: v_{k} of a culled Gaussian"
        assert bool(torch.isfinite(got[k]).all()), f"{what}: v_{k} not finite"
    rows = vis
    if case.antialiased:  # rank-deficient covariances: compensation of rounding size, compared where it is 0
        with torch.no_grad():
            comp64 = P.forward64(case, br)["comp"]
        rows = vis & ((o["compensations"] == 0) | (comp64 > 1e-3))
    keys = P.PARAM_KEYS if case.sh_bases > 1 else P.PARAM_KEYS[:-1]
    if compare is not None:
        rows = rows & compare
    check_rows(got, want, spr, rows, case, what, keys)
    if viewmat:
        assert float(vv[3].abs().max()) == 0.0, f"{what}: v_viewmat row 3"
        w, s = want["viewmat"], spr["viewmat"]
        r = float(((vv.double() - w).abs() / (VIEWMAT_RTOL * w.abs().max() + P.sens("grad", case)["viewmat"] * s)).max())
        assert r <= 1.0, f"{what}: v_viewmat {r:.2f} x the bound"
    return run, br, got, want, rows


@pytest.mark.parametrize("act,aa,normals,sh", BWD_CASES,
                         ids=[f"{'act' if a else 'raw'}-{'aa' if aa else 'classic'}-{'n' if nm else 'nonormal'}-deg{s[0]}b{s[1]}"
                              for a, aa, nm, s in BWD_CASES])
def test_backward_matches_fp64_per_gaussian(act, aa, normals, sh):
    """Every Gaussian flagged, culled ones included (zero gradient, record still cleared)."""
    case = bwd_case(act, aa, normals, sh)
    _, br, _, _, vis = check_backward(case, f"act={act} aa={aa} normals={normals} sh={sh}")
    assert 0 < int(vis.sum()) < case.n
    assert bool((~br.color_pass[vis]).any()), "premise: some colours are clamped at 0"


@pytest.mark.parametrize("aa", [False, True], ids=["classic", "aa"])
def test_backward_clamped_jacobian(aa):
    """Past the 1.3 tan(fov) limit in x, in y and in both: the z-term of the clamped Jacobian."""
    case = _case("clamped", n=900, seed=7, antialiased=aa)
    _, br, _, _, vis = check_backward(case, f"clamped aa={aa}")
    for name, sel in (("x", br.clamp_x & ~br.clamp_y), ("y", br.clamp_y & ~br.clamp_x), ("xy", br.clamp_x & br.clamp_y)):
        assert int((sel & vis).sum()) >= 50, f"premise: visible Gaussians clamped in {name} only"


def test_backward_zero_compensation():
    """Antialiased, rank-1 covariances: compensation 0 next to compensation of rounding size.  Where it is 0 the
    opacity the raster sees is 0 and v_opacities is exactly 0, and the conic and means2d routes (v_means, v_quats,
    v_scales) are compared with fp64 per Gaussian.  A rank-1 compensation > 0 is rounding noise in fp32 and in fp64
    alike: those rows are held to the buffer contract only."""
    case = _case("rank1", n=900, seed=8, deg=1, bases=4, antialiased=True)
    run = Run(case)
    comp, vis = run.host_out["compensations"], run.host_out["radii"] > 0
    zero = (comp == 0) & vis
    assert int(zero.sum()) >= 20 and int(((comp > 0) & vis).sum()) >= 20, "premise: both branches"
    _, _, got, _, rows = check_backward(case, "rank1", compare=comp == 0)
    assert torch.equal(rows, zero), "the comp = 0 rows are the ones compared"
    assert bool((run.host_out["opac_act"][zero] == 0).all())
    assert bool((got["opacities"][zero] == 0).all()), "v_opacities where the compensation is 0"
    assert bool((got["means"][zero] != 0).any(1).all()), "premise: the other routes reach the comp = 0 Gaussians"


@pytest.mark.parametrize("host", [False, True], ids=["device_camera", "host_camera"])
def test_backward_viewmat(host):
    """d(loss)/d(viewmat) with the camera on the device and passed by value."""
    case = _case("random", n=3000, seed=9, antialiased=True)
    check_backward(case, f"viewmat host={host}", host=host, viewmat=True)


def test_backward_edge_on_normals():
    """~2000 Gaussians seen edge-on (|cos(view, normal)| <= 1e-7) with only the normal slot of the record non-zero: the
    backward must differentiate the normal with the sign the forward rendered.  The old backward recomputed the flip
    from an un-normalised view vector and disagreed with the forward on several percent of these."""
    case = _case("edge_on", n=2000, seed=11)
    run = Run(case)
    o = run.host_out
    vis = o["radii"] > 0
    kernel_flip = _kernel_flip(case, o)
    br = P.Branches.from_fp32(case, flip=kernel_flip)
    disagree = vis & (kernel_flip != br.flip_bwd)
    assert int(disagree.sum()) >= 20, f"premise: the backward's old expression disagrees on {int(disagree.sum())}"
    gr = _seeded_records(case.n, seed=11, only_normal=True)
    got, _, _ = run.backward(gr, torch.ones(case.n, dtype=torch.uint8))
    fn = lambda c: P.vjp64(c, br, gr, vis)  # noqa: E731
    want, spr = fn(case), P.spread(fn, case)
    gq, wq = got["quats"].double(), want["quats"]
    cos = (gq * wq).sum(1) / (gq.norm(dim=1) * wq.norm(dim=1)).clamp(min=1e-300)
    flipped = vis & (cos < -0.99)
    assert not bool(flipped.any()), (
        f"{int(flipped.sum())} of {int(vis.sum())} edge-on Gaussians get the normal gradient with the opposite sign "
        f"(v_quats . fp64 / |.||.| = -1), e.g. Gaussian {int(torch.nonzero(flipped)[0])}: kernel "
        f"{gq[flipped][0].tolist()} fp64 {wq[flipped][0].tolist()}")
    check_rows(got, want, spr, vis, case, "edge-on", P.PARAM_KEYS)


# ----------------------------------------------------------------------------------------------------- compaction
NS = [1, 7, 8, 9, 1023, 1024, 1025, 2051, 5003]
PATTERNS = ["none", "all", "every_other", "last", "chunk_first", "random10"]


def _flags(n, pattern, value, seed):
    t = torch.zeros(n, dtype=torch.uint8)
    if pattern == "all":
        t[:] = value
    elif pattern == "every_other":
        t[::2] = value
    elif pattern == "last":
        t[-1] = value
    elif pattern == "chunk_first":
        t[::1024] = value
    elif pattern == "random10":
        g = torch.Generator().manual_seed(seed)
        t[torch.rand(n, generator=g) < 0.1] = value
    elif pattern != "none":
        raise ValueError(pattern)
    return t


def _prefill(run, seed):
    """Random buffers without zeros (so without -0.0: the kernel adds +0.0 to inactive SH rows)."""
    g = torch.Generator().manual_seed(seed)
    r = lambda t: (torch.rand(t.shape, generator=g) + 0.5) * torch.where(torch.rand(t.shape, generator=g) < 0.5, -1.0, 1.0)  # noqa
    pre = {k: r(v) for k, v in run.case.params.items()}
    n = run.case.n
    return pre, (r(torch.zeros(n, 2)), r(torch.zeros(n, 2)))


@pytest.mark.parametrize("n", NS)
def test_compaction_and_buffer_contract(n):
    """For every flag pattern and flag value 1 / 255: flagged rows end at exactly prefill + the gradient of a zero-prefill
    run with every Gaussian flagged (each Gaussian is written once), their records are consumed; unflagged rows,
    records and v_means2d / v_means2d_abs keep their bytes.  Two runs are bit-identical (v_viewmat aside: atomics)."""
    case = _case("random", n=n, seed=n, deg=1, bases=16, antialiased=True)
    run = Run(case)
    vis = run.host_out["radii"] > 0
    gr = _seeded_records(n, seed=n)
    fresh, _, _ = run.backward(gr, torch.ones(n, dtype=torch.uint8))
    pre, m2d = _prefill(run, seed=n + 1)
    for value in (1, 255):
        for pattern in PATTERNS:
            what = f"n={n} pattern={pattern} flag={value}"
            fl = _flags(n, pattern, value, seed=n + value)
            sel = fl != 0
            res = [run.backward(gr, fl, prefill=pre, viewmat=True, m2d_prefill=m2d) for _ in range(2)]
            (got, gr_after, vv), (got2, gr_after2, _) = res
            for k in list(P.PARAM_KEYS) + ["means2d", "means2d_abs"]:
                assert torch.equal(got[k], got2[k]), f"{what}: v_{k} differs between two runs"
            assert torch.equal(gr_after, gr_after2)
            want_rec = torch.where(sel[:, None], torch.zeros(()), gr)
            assert torch.equal(gr_after, want_rec), f"{what}: grad_records"
            for k in P.PARAM_KEYS:
                shape = (-1,) + (1,) * (pre[k].dim() - 1)
                want = torch.where(sel.view(shape), pre[k] + fresh[k], pre[k])
                bad = torch.nonzero((got[k] != want).reshape(n, -1).any(1)).flatten()
                assert bad.numel() == 0, f"{what}: v_{k} rows {bad[:5].tolist()}"
            for k, src, p in (("means2d", gr[:, 0:2], m2d[0]), ("means2d_abs", gr[:, 2:4], m2d[1])):
                want = torch.where((sel & vis)[:, None], src, p)
                assert torch.equal(got[k], want), f"{what}: v_{k}"
            if not bool(sel.any()):
                assert float(vv.abs().max()) == 0.0, f"{what}: v_viewmat without a flagged Gaussian"
    # inactive SH rows (degree 1 of 16 stored bases) of a flagged Gaussian keep their prefill exactly
    assert torch.equal(fresh["sh_rest"][:, 3:], torch.zeros_like(fresh["sh_rest"][:, 3:]))
