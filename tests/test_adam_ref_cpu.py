"""oracle/adam_ref.py: the fp64 Adam step and its fp32 error bound.  The unmutated fp32 restatement of csrc/adam.cu
(numpy, operation for operation) stays inside the bound and equals FusedAdam.reference_step bit for bit; each of six
plausible slips in the update rule leaves the bound by at least 100x on the data tests/test_gpu_adam.py feeds the kernel.

The case builders here (`SIXTEEN`, `segment_state`) are shared with the GPU test, so the teeth shown here are the teeth
that test has."""
from collections import namedtuple

import numpy as np
import pytest
import torch

from dn_splatter_b200.optim import FusedAdam, bias_corrections
from oracle.adam_ref import adam_bound, adam_step_fp64, fp32_scalars

BETAS = (0.9, 0.999)
STEPS = 3

Seg = namedtuple("Seg", "n lr eps t seed init")

# one dnr_adam_step launch with DNR_ADAM_MAX_SEGS segments: own lengths, lr, eps and step count (so own bc1 / bc2)
_TS = (1, 2, 10, 1000, 100000)
SIXTEEN = [Seg(n, lr, eps, _TS[i % 5], 100 + i, "zero" if i % 3 == 0 else "random")
           for i, (n, lr, eps) in enumerate(zip(
               (1, 2, 3, 4, 5, 7, 8, 1023, 4097, 33, 64, 100, 257, 999, 2048, 5000),
               (1.6e-4, 5e-3, 1e-3, 2.5e-3, 1.25e-4, 5e-2, 1e-2, 3e-4, 7e-3, 1e-1, 2e-5, 1e-3, 4e-2, 6e-4, 8e-3, 1.5e-3),
               (1e-15, 1e-8) * 8))]


def segment_state(seg: Seg):
    """fp32 (p, m, v, [g for each of STEPS steps]) of one segment from its seed.  Gradients mix magnitudes from 1e-12 to
    1e3 with exact zeros (the rows must still decay), |g| ~ 1e-25 (w2 g^2 underflows to 0) and ~ 1e-21 (w2 g^2 is
    subnormal); half of the elements flip sign every step.  m, v start at zero or at random values (v >= 0)."""
    rng = np.random.default_rng(seg.seed)
    n = seg.n
    p = (rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 2, n)).astype(np.float32)
    if seg.init == "zero":
        m, v = np.zeros(n, np.float32), np.zeros(n, np.float32)
    else:
        m = (rng.standard_normal(n) * 10.0 ** rng.uniform(-8, 1, n)).astype(np.float32)
        v = ((rng.standard_normal(n) * 10.0 ** rng.uniform(-8, 1, n)) ** 2).astype(np.float32)
    sign = np.where(rng.random(n) < 0.5, -1.0, 1.0)
    base = sign * 10.0 ** rng.uniform(-12, 3, n)
    kind = rng.permutation(n) % 10
    base[kind == 0] = 0.0
    base[kind == 1] = sign[kind == 1] * 1e-25 * rng.uniform(1, 2, int((kind == 1).sum()))
    base[kind == 2] = sign[kind == 2] * 1e-21 * rng.uniform(1, 2, int((kind == 2).sum()))
    flip = rng.random(n) < 0.5
    grads = [(base * np.where(flip, (-1.0) ** s, 1.0) * rng.uniform(0.5, 2.0, n)).astype(np.float32)
             for s in range(STEPS)]
    return p, m, v, grads


def scalars(seg: Seg, t: int, betas=BETAS):
    return fp32_scalars(seg.lr, seg.eps, *bias_corrections(t, *betas), *betas)


def reference_step(segs, states, ts):
    """FusedAdam.reference_step (torch fp32 on the CPU) from the given (p, g, m, v) at step counts `ts`: new (p, m, v)."""
    params = [torch.nn.Parameter(torch.from_numpy(p.copy())) for p, _, _, _ in states]
    opt = FusedAdam([{"params": [q], "lr": s.lr, "eps": s.eps} for q, s in zip(params, segs)], betas=BETAS)
    for q, (_, g, m, v), t in zip(params, states, ts):
        q.grad = torch.from_numpy(g.copy())
        opt.state[q] = {"step": t - 1, "exp_avg": torch.from_numpy(m.copy()), "exp_avg_sq": torch.from_numpy(v.copy())}
    opt.reference_step()
    return [(q.detach().numpy(), opt.state[q]["exp_avg"].numpy(), opt.state[q]["exp_avg_sq"].numpy()) for q in params]


def check_step(got, p, g, m, v, sc, what=""):
    """got = (p', m', v') of one fp32 step from (p, g, m, v): asserts it lies within adam_bound of adam_step_fp64."""
    want = adam_step_fp64(p, g, m, v, **sc)
    tols = adam_bound(p, g, m, v, **sc)
    for name, x, y, tol in zip("pmv", got, want, tols):
        assert np.isfinite(tol).all() and np.isfinite(y).all(), (what, name)
        err = np.abs(np.asarray(x, np.float64) - y)
        bad = np.flatnonzero(err > tol)
        assert bad.size == 0, (what, name, bad[:5], err[bad[:5]], tol[bad[:5]])


def _fp32_step(p, g, m, v, sc, mutation=None, seg=None, t=None):
    """csrc/adam.cu adam_one in numpy fp32, operation for operation; `mutation` names a slip to make instead."""
    f = np.float32
    if mutation == "bias_correction_of_step_t_minus_1":
        sc = scalars(seg, max(t - 1, 1))  # bc1(0) = 0: the t = 1 segments keep their own step
    w1, b2, w2, S, c, e = f(sc["w1"]), f(sc["beta2"]), f(sc["w2"]), f(sc["step_size"]), f(sc["bc2_sqrt"]), f(sc["eps"])
    if mutation == "betas_swapped":
        w1, b2, w2 = f(1.0 - BETAS[1]), f(BETAS[0]), f(1.0 - BETAS[0])
    if mutation == "bc2_where_sqrt_bc2_belongs":
        c = f(bias_corrections(t, *BETAS)[1] ** 2)
    if mutation == "w1_m_plus_beta1_g":
        m2 = w1 * m + f(BETAS[0]) * g
    else:
        m2 = m + w1 * (g - m)
    v2 = b2 * v + w2 * g * g
    if mutation == "eps_inside_the_sqrt":
        denom = np.sqrt(v2 + e) / c
    else:
        denom = np.sqrt(v2) / c + e
    p2 = p - S * ((m if mutation == "update_with_the_previous_m" else m2) / denom)
    return p2, m2, v2


def test_unmutated_fp32_restatement_is_within_the_bound_and_equals_reference_step():
    for s in range(STEPS):
        states, got = [], []
        for seg in SIXTEEN:
            p, m, v, grads = segment_state(seg)
            sc = scalars(seg, seg.t + s)
            states.append((p, grads[s], m, v))
            got.append(_fp32_step(p, grads[s], m, v, sc))
            check_step(got[-1], p, grads[s], m, v, sc, seg)
        ref = reference_step(SIXTEEN, states, [seg.t + s for seg in SIXTEEN])
        for seg, a, b in zip(SIXTEEN, got, ref):
            for x, y in zip(a, b):
                assert np.array_equal(x.view(np.int32), y.view(np.int32)), seg


MUTATIONS = ["bias_correction_of_step_t_minus_1", "eps_inside_the_sqrt", "betas_swapped", "bc2_where_sqrt_bc2_belongs",
             "update_with_the_previous_m", "w1_m_plus_beta1_g"]


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_each_slip_leaves_the_bound_by_100x(mutation):
    worst = 0.0
    for seg in SIXTEEN:
        p, m, v, grads = segment_state(seg)
        g = grads[0]
        sc = scalars(seg, seg.t)
        got = _fp32_step(p, g, m, v, sc, mutation, seg, seg.t)
        want = adam_step_fp64(p, g, m, v, **sc)
        tols = adam_bound(p, g, m, v, **sc)
        for x, y, tol in zip(got, want, tols):
            err = np.abs(np.asarray(x, np.float64) - y)
            ok = np.isfinite(err) & (tol > 0)  # only finite violations count (a NaN would be a slip as well)
            worst = max(worst, float((err[ok] / tol[ok]).max(initial=0.0)))
    assert worst >= 100.0, (mutation, worst)
