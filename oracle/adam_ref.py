"""fp64 numpy restatement of one step of the fused Adam update (dn_splatter_b200/csrc/adam.cu: adam_one), and a
per-element bound on how far the kernel's fp32 arithmetic may lie from it.

The kernel's rule, from fp32 state p, g, m, v and fp32 scalars (fill_adam_launch rounds them from the host's doubles):

    m' = m + w1 (g - m)            w1 = fl(1 - beta1)
    v' = beta2 v + w2 g g          beta2 = fl(beta2), w2 = fl(1 - beta2)
    D  = sqrt(v') / c + e          c = fl(sqrt(1 - beta2^t)), e = fl(eps)
    p' = p - S m' / D              S = fl(lr / (1 - beta1^t))

`adam_step_fp64` evaluates it in float64 from exactly those fp32 values, so the rounding of the scalars is part of the
contract and not of the error budget.  One comparison covers one step taken from one fp32 state; callers check every
step from the kernel's own previous state, so errors never compound.

Error bound (`adam_bound`), u = 2^-24, each fp32 operation fl(x) = x (1 + d) + z with |d| <= u, |z| <= 2^-150 and
d z = 0 (z only when the result is subnormal; adam.cu is compiled without flush-to-zero):

m: three roundings.  fl(m + fl(w1 fl(g - m))) - m' = m d3 + w1 (g - m) ((1 + d1)(1 + d2)(1 + d3) - 1), so
   |m32 - m'| <= u |m| + 3.0000003 u w1 (|g| + |m|) <= 4u (|m| + |g|) for w1 <= 0.99.  This assumes the
   intermediates of m stay normal (|w1 (g - m)| >= 2^-126 or zero), which every input here satisfies down to
   |g| = 1e-25.
v: four roundings; both summands are non-negative, so no cancellation:
   |v32 - v'| <= 2.0000001 u beta2 v + 3.0000003 u w2 g^2 + (three subnormal z, and the addition of a subnormal
   result is exact) <= 4u (beta2 v + w2 g^2) + 4 * 2^-149.  The extra 2^-149 terms cover w2 g^2 falling into (or
   under) the subnormal range, e.g. |g| ~ 1e-21 (w2 g^2 ~ 1e-45) or 1e-25 (w2 g^2 underflows to 0).
D: with sq = a bound on |sqrt(v32) - sqrt(v')| for |v32 - v'| <= tol_v,
   sq = min(tol_v / (sqrt(v') + sqrt(max(v' - tol_v, 0))), sqrt(tol_v))
   (|sqrt(a) - sqrt(b)| = |a - b| / (sqrt(a) + sqrt(b)) and <= sqrt(|a - b|); to first order sq = tol_v / (2 sqrt(v')),
   but the exact form stays valid where v' is subnormal or 0).  Three roundings (sqrt, /c, +e) then give
   rho = |D32 - D| / D <= u + (1 + u)^3 (sq / c + 2.0000001 u sqrt(v') / c) / D <= 4u + (1 + 4u) sq / (c D).
p: the update U = S m' / D takes two more roundings (m32 / D32, then S *).  With |1/D32 - 1/D| <= rho / (D (1 - rho)),
   |U32 - U| <= (S / D) (1 + 2.0000001 u) (tol_m + |m'| (rho + 2.0000001 u)) / (1 - rho),
   and rho + 2.0000001 u <= 8u + (1 + 4u) sq / (c D) (6u spent, 2u slack).  The final subtraction adds
   u |p - U32| <= u |p'| + u |U32 - U|, so
   |p32 - p'| <= 2u |p'| + (1 + 4u) (S / D) (tol_m + |m'| (8u + (1 + 4u) sq / (c D))) / (1 - rho),
   where the second u |p'| and the 2u of slack in 8u cover the float64 evaluation of p' itself (a few 2^-53 of |p'|
   and of |U|).
No constant exceeds 8u.  Where rho >= 1 the bound is infinite; callers assert that it is finite everywhere, so no case
passes vacuously.
"""
from __future__ import annotations

import numpy as np

U = 2.0 ** -24
SUBNORMAL = 2.0 ** -149


def fp32_scalars(lr: float, eps: float, bc1: float, bc2_sqrt: float, beta1: float, beta2: float) -> dict:
    """The scalars of one segment as fill_adam_launch rounds them to fp32 (returned as the float64 values of those
    fp32 numbers): S = fl(lr / bc1), c = fl(bc2_sqrt), e = fl(eps), beta2, w1 = fl(1 - beta1), w2 = fl(1 - beta2)."""
    f = lambda x: float(np.float32(x))
    return dict(step_size=f(lr / bc1), bc2_sqrt=f(bc2_sqrt), eps=f(eps), beta2=f(beta2), w1=f(1.0 - beta1),
                w2=f(1.0 - beta2))


def adam_step_fp64(p, g, m, v, step_size, bc2_sqrt, eps, beta2, w1, w2):
    """One Adam step in float64 from fp32 inputs and fp32-rounded scalars: returns (p', m', v') as float64 arrays."""
    p, g, m, v = (np.asarray(x, np.float32).astype(np.float64) for x in (p, g, m, v))
    m2 = m + w1 * (g - m)
    v2 = beta2 * v + w2 * g * g
    p2 = p - step_size * (m2 / (np.sqrt(v2) / bc2_sqrt + eps))
    return p2, m2, v2


def adam_bound(p, g, m, v, step_size, bc2_sqrt, eps, beta2, w1, w2):
    """Per-element bounds (tol_p, tol_m, tol_v) on |fp32 kernel - adam_step_fp64| for one step (module docstring)."""
    g, m, v = (np.asarray(x, np.float32).astype(np.float64) for x in (g, m, v))
    p2, m2, v2 = adam_step_fp64(p, g, m, v, step_size, bc2_sqrt, eps, beta2, w1, w2)
    tol_m = 4 * U * (np.abs(m) + np.abs(g))
    tol_v = 4 * U * (beta2 * v + w2 * g * g) + 4 * SUBNORMAL
    with np.errstate(divide="ignore", invalid="ignore"):
        sq = np.minimum(tol_v / (np.sqrt(v2) + np.sqrt(np.maximum(v2 - tol_v, 0.0))), np.sqrt(tol_v))
        D = np.sqrt(v2) / bc2_sqrt + eps
        rel_sqrt = sq / (bc2_sqrt * D)
        rho = 4 * U + (1 + 4 * U) * rel_sqrt
        upd = (1 + 4 * U) * (step_size / D) * (tol_m + np.abs(m2) * (8 * U + (1 + 4 * U) * rel_sqrt))
        tol_p = np.where(rho < 1.0, 2 * U * np.abs(p2) + upd / (1.0 - rho), np.inf)
    return tol_p, tol_m, tol_v
