"""oracle/project_ref.py: the fp64 projection VJP that tests/test_gpu_projection.py holds dnr_project_bwd to.

  * away from its branch points it is autograd of the existing oracle (gsplat_ref.project_gaussians, gsplat_ref.eval_sh,
    dn_ref.gaussian_normals), and it matches fp64 central differences;
  * each plausible slip in the backward moves at least one Gaussian of the GPU test's own data (the same builders and
    seeds) outside the per-Gaussian tolerance by 10x or more.  Several of them move the norm-wise relative error over
    all Gaussians, the measure of test_gpu_parity.py and test_gpu_backward_edges.py, by less than their 1e-3.
"""
import pytest
import torch

from oracle import dn_ref
from oracle import gsplat_ref as G
from oracle import project_ref as P
from tests.test_gpu_projection import _case, _seeded_records, bwd_case, records

F64 = torch.float64
NORMWISE = 1e-3  # the norm-wise gradient bound of the whole-render tests


def _oracle_loss(case, p, vm, gr, rows):
    """sum(grad_records . outputs) through the existing oracle, fp64."""
    s = p["scales"] if case.activated else torch.exp(p["scales"])
    o = p["opacities"] if case.activated else torch.sigmoid(p["opacities"])
    proj = G.project_gaussians(p["means"], p["quats"], s, vm, case.K.double(), case.width, case.height, eps2d=case.eps2d,
                               near_plane=case.near_plane, far_plane=case.far_plane)
    campos = -(vm[:3, :3].T @ vm[:3, 3])
    deg = case.sh_degree
    coeffs = torch.cat([p["sh_dc"][:, None], p["sh_rest"][:, :(deg + 1) ** 2 - 1]], 1)
    rgb = torch.clamp_min(G.eval_sh(deg, p["means"] - campos, coeffs) + 0.5, 0.0)
    op = o * proj["compensations"] if case.antialiased else o
    g = torch.where(rows[:, None], gr.double(), torch.zeros((), dtype=F64))
    loss = (g[:, 0:2] * proj["means2d"]).sum() + (g[:, 4:7] * proj["conics"]).sum() + (g[:, 7] * op).sum()
    loss = loss + (g[:, 8:11] * rgb).sum() + (g[:, 11] * proj["depths"]).sum()
    if case.normals:
        _, ncam = dn_ref.gaussian_normals(p["quats"], p["scales"], p["means"], case.c2w.double())
        loss = loss + (g[:, 12:15] * ncam).sum()
    return loss


def _away_from_ties(case, br):
    """Visible Gaussians at least 1e-4 (relative) from every branch point of the projection."""
    with torch.no_grad():
        out = P.forward64(case, br)
        proj = G.project_gaussians(*(case.params[k].double() for k in ("means", "quats")),
                                   case.params["scales"].double() if case.activated else torch.exp(case.params["scales"].double()),
                                   case.viewmat.double(), case.K.double(), case.width, case.height, eps2d=case.eps2d,
                                   near_plane=case.near_plane, far_plane=case.far_plane)
        x, y, z = proj["mean_cam"].unbind(1)
        vis = proj["radii"] > 0
        far = ((x / z).abs() - br.lim_x).abs() > 1e-4 * br.lim_x
        far &= ((y / z).abs() - br.lim_y).abs() > 1e-4 * br.lim_y
        col = P.colors32(case).double() + 0.5
        far &= (col.abs() > 1e-4).all(1)
        far &= out["comp"] > 1e-3 if case.antialiased else torch.ones_like(far)
        if case.normals:
            cam = case.c2w[:, 3].double()
            v = torch.nn.functional.normalize(cam - case.params["means"].double(), dim=1)
            far &= ((out["normals_world"] * v).sum(1)).abs() > 1e-4
            s = case.params["scales"].double()
            srt = s.sort(1).values
            far &= (srt[:, 1] - srt[:, 0]) > 1e-4
    return vis & far


@pytest.mark.parametrize("kind,act,aa,deg,bases", [("random", False, False, 3, 16), ("random", True, True, 2, 9),
                                                  ("random", False, True, 1, 16), ("clamped", False, True, 3, 16),
                                                  ("random", True, False, 0, 4)])
def test_reference_is_autograd_of_the_oracle(kind, act, aa, deg, bases):
    case = _case(kind, n=400, seed=5, deg=deg, bases=bases, activated=act, antialiased=aa)
    br = P.Branches.from_fp32(case)
    rows = _away_from_ties(case, br)
    assert int(rows.sum()) >= 100
    gr = _seeded_records(case.n, seed=3)
    want = P.vjp64(case, br, gr, rows, viewmat=True)
    p = {k: v.double().requires_grad_(True) for k, v in case.params.items()}
    vm = case.viewmat.double().requires_grad_(True)
    gs = torch.autograd.grad(_oracle_loss(case, p, vm, gr, rows), [p[k] for k in P.PARAM_KEYS] + [vm], allow_unused=True)
    for k, g in zip(list(P.PARAM_KEYS) + ["viewmat"], gs):
        g = torch.zeros_like(want[k]) if g is None else g
        # two fp64 evaluations in different operation orders: needles' conics lose up to ~1e-8 of the group's scale
        torch.testing.assert_close(want[k], g, rtol=1e-7, atol=1e-7 * float(g.abs().max()), msg=k)


def test_reference_matches_finite_differences():
    case = _case("random", n=60, seed=6, deg=3, bases=16, antialiased=True)
    br = P.Branches.from_fp32(case)
    rows = _away_from_ties(case, br)
    idx = torch.nonzero(rows).flatten()[:6]
    assert idx.numel() == 6
    gr = _seeded_records(case.n, seed=4)
    want = P.vjp64(case, br, gr, rows, viewmat=True)

    def loss(p, vm):
        out = P.forward64(case, br, p, vm)
        g = torch.where(rows[:, None], gr.double(), torch.zeros((), dtype=F64))
        return float((g[:, 0:2] * out["means2d"]).sum() + (g[:, 4:7] * out["conics"]).sum() + (g[:, 7] * out["opac"]).sum()
                     + (g[:, 8:11] * out["rgb"]).sum() + (g[:, 11] * out["depth"]).sum() + (g[:, 12:15] * out["ncam"]).sum())

    base = {k: v.double() for k, v in case.params.items()}
    vm0 = case.viewmat.double()
    h = 1e-6
    for k in P.PARAM_KEYS:
        for i in idx.tolist():
            for j in range(base[k][i].numel()):
                pp, pm = {kk: v.clone() for kk, v in base.items()}, {kk: v.clone() for kk, v in base.items()}
                pp[k][i].view(-1)[j] += h
                pm[k][i].view(-1)[j] -= h
                fd = (loss(pp, vm0) - loss(pm, vm0)) / (2 * h)
                an = float(want[k][i].reshape(-1)[j])
                assert abs(fd - an) <= 1e-5 * max(1.0, abs(an)), (k, i, j, fd, an)
    for r in range(3):
        for c in range(4):
            vp, vmm = vm0.clone(), vm0.clone()
            vp[r, c] += h
            vmm[r, c] -= h
            fd = (loss(base, vp) - loss(base, vmm)) / (2 * h)
            an = float(want["viewmat"][r, c])
            assert abs(fd - an) <= 1e-5 * max(1.0, abs(an)), ("viewmat", r, c, fd, an)


# The GPU test's data for each slip: a scene of test_backward_matches_fp64_per_gaussian (act, aa, normals, (degree,
# bases)), or the edge-on set of test_backward_edge_on_normals; and whether the slip stays below the whole-render tests'
# 1e-3 norm-wise bound on it.  Over all 40 scenes of that test the clamp slip moves the norm-wise error by 7.4e-4 to
# 2.9e-3 (below 1e-3 on 11 of them) and leaves the per-Gaussian bound by 29x or more on every one.
SLIP_DATA = {
    "clamp_z": ((False, False, True, (0, 1)), True),
    "comp": ((False, True, True, (3, 16)), False),
    "inorm": ((False, False, True, (3, 16)), False),
    "abs_swap": ((False, False, True, (3, 16)), False),
    "flip_bwd": ("edge_on", False),
}


def _slip_errors(slip):
    data, _ = SLIP_DATA[slip]
    if data == "edge_on":  # as test_backward_edge_on_normals builds it
        case = _case("edge_on", n=2000, seed=11)
        gr = _seeded_records(case.n, seed=11, only_normal=True)
    else:
        case = bwd_case(*data)
        gr = records(case)
    br = P.Branches.from_fp32(case)
    proj = G.project_gaussians(case.params["means"], case.params["quats"],
                               case.params["scales"] if case.activated else torch.exp(case.params["scales"]),
                               case.viewmat, case.K, case.width, case.height, eps2d=case.eps2d,
                               near_plane=case.near_plane, far_plane=case.far_plane)
    vis = proj["radii"] > 0
    fn = lambda c: P.vjp64(c, br, gr, vis)  # noqa: E731
    good, spr = fn(case), P.spread(fn, case)
    bad = P.vjp64(case, br, gr, vis, slip=slip)
    spr.update(means2d=torch.zeros_like(good["means2d"]), means2d_abs=torch.zeros_like(good["means2d"]))
    worst, normwise = 0.0, 0.0
    needle = P.needles(case)
    sens = P.sens("grad", case)
    for k in list(P.PARAM_KEYS) + ["means2d", "means2d_abs"]:
        for sel, f in ((vis & ~needle, sens.get(k, 0.0)), (vis & needle, P.needle_sens("grad", case))):
            worst = max(worst, float(P.row_ratio(bad[k], good[k], spr[k], sel, P.GRAD_RTOL, P.GRAD_ATOL, f).max()))
        nw = float(good[k].norm())
        if nw > 0:
            normwise = max(normwise, float((bad[k] - good[k]).norm()) / nw)
    return worst, normwise


@pytest.mark.parametrize("slip", P.SLIPS)
def test_slip_leaves_the_per_gaussian_bound(slip):
    worst, normwise = _slip_errors(slip)
    assert worst >= 10, f"{slip}: the worst Gaussian is only {worst:.2f} x the per-Gaussian tolerance"
    # where the slip hides from the whole-render tests' measure, say so
    assert (normwise < NORMWISE) == SLIP_DATA[slip][1], f"{slip}: norm-wise relative error {normwise:.3e}"
