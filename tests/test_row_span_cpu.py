"""Conservativeness of the precise-hit emission formula (csrc/binning.cu: load_hit_gauss + row_span), restated in numpy
float32 and checked against brute force: every list tile that contains a pixel centre with sigma <= lim must lie inside
the emitted span of its row — for ordinary, needle-like, huge and off-screen splats, at every list tile the kernel uses
(16 << list_shift, list_shift 0..3).  (The CUDA kernels themselves are held to the same contract per pair on the GPU by
tests/test_gpu_binning.py.)"""
import numpy as np
import pytest

f32 = np.float32
LIST_TILES = [16, 32, 64, 128]


def fma32(a, b, c):
    """fmaf: the fp64 product of two floats is exact."""
    return f32(np.float64(a) * np.float64(b) + np.float64(c))


def det32(A, B, C):
    """The kernel's A C - B^2 of the fp32 conic: Kahan's difference of products, exact but for the last rounding."""
    bb = f32(B * B)
    return f32(fma32(A, C, -bb) + fma32(-B, B, bb))


def spans(mx, my, A, B, C, L, x0, y0, nx, ny, ts=16):
    """Mirror of load_hit_gauss + row_span for one Gaussian at list tile `ts`; returns [(lo, hi)] per tile row of the box."""
    mx, my, A, B, C, L = map(f32, (mx, my, A, B, C, L))
    det = det32(A, B, C)
    if not (L > 0) or not (det > 0):
        return [(x0, x0)] * ny
    invA, bac, twoAL = f32(1) / A, -det, f32(2) * A * L
    ex_max = np.sqrt(f32(2) * L * C / det, dtype=f32) * f32(1.0001) + f32(0.01)
    ey_max = np.sqrt(f32(2) * L * A / det, dtype=f32) * f32(1.0001) + f32(0.01)
    ey_star = -B * ex_max / C
    out = []
    for r in range(ny):
        ty = y0 + r
        lo, hi = x0, x0 + nx
        e0 = f32(ty * ts + 0.5) - my - f32(0.01)
        e1 = f32(ty * ts + ts - 1 + 0.5) - my + f32(0.01)
        if e0 > ey_max or e1 < -ey_max:
            out.append((lo, lo))
            continue
        e0, e1 = max(e0, -ey_max), min(e1, ey_max)
        s0 = np.sqrt(max(f32(bac * e0 * e0 + twoAL), f32(0)), dtype=f32)
        s1 = np.sqrt(max(f32(bac * e1 * e1 + twoAL), f32(0)), dtype=f32)
        xmax = max((-B * e0 + s0) * invA, (-B * e1 + s1) * invA)
        xmin = min((-B * e0 - s0) * invA, (-B * e1 - s1) * invA)
        if e0 <= ey_star <= e1:
            xmax = ex_max
        if e0 <= -ey_star <= e1:
            xmin = -ex_max
        xmax = xmax + f32(0.01) + f32(1e-5) * abs(xmax)
        xmin = xmin - f32(0.01) - f32(1e-5) * abs(xmin)
        t_lo = int(np.ceil((mx + xmin - f32(ts - 0.5)) * f32(1.0 / ts)))  # tile tx holds centres [ts tx + 0.5, ts tx + ts - 0.5]
        t_hi = int(np.floor((mx + xmax - f32(0.5)) * f32(1.0 / ts))) + 1
        out.append((max(lo, t_lo), min(hi, t_hi)))
    return out


def brute_force_tiles(mx, my, A, B, C, L, tiles_x, tiles_y, ts=16):
    xs = np.arange(tiles_x * ts, dtype=np.float64) + 0.5
    ys = np.arange(tiles_y * ts, dtype=np.float64) + 0.5
    dx, dy = mx - xs[None, :], my - ys[:, None]
    sigma = 0.5 * (A * dx * dx + C * dy * dy) + B * dx * dy
    hit = sigma <= L
    return hit.reshape(tiles_y, ts, tiles_x, ts).any(axis=(1, 3))


def check_spans(mx, my, A, B, C, opac, tiles_x, tiles_y, ts, what):
    """Asserts the mirror's spans cover the brute-force reach; returns (tiles kept, tiles reachable)."""
    L = np.log(255.0 * opac) + 0.1  # cull_lim of project_fwd
    want = brute_force_tiles(mx, my, A, B, C, np.log(255.0 * opac), tiles_x, tiles_y, ts)  # true reach (no margin)
    got = spans(mx, my, A, B, C, L, 0, 0, tiles_x, tiles_y, ts)
    kept = 0
    for ty in range(tiles_y):
        lo, hi = got[ty]
        need = np.nonzero(want[ty])[0]
        if need.size:
            assert lo <= need.min() and hi > need.max(), (what, ts, mx, my, A, B, C, opac, ty, (lo, hi), need)
        kept += max(hi - lo, 0)
    return kept, int(want.sum())


@pytest.mark.parametrize("seed", range(6))
def test_row_spans_cover_every_reachable_tile(seed):
    """A 320 x 192 frame at every list tile: ordinary, needle-like (axis ratio up to 1:200), huge and off-screen splats."""
    W, H = 320, 192
    for ts in LIST_TILES:
        rng = np.random.default_rng(seed)
        tiles_x, tiles_y = -(-W // ts), -(-H // ts)
        kept = total = 0
        for _ in range(300):
            # covariance from random axes; every third splat is a needle (axis ratio up to 1:200)
            s1 = rng.uniform(0.6, 60.0)
            s2 = s1 / rng.uniform(1.0, 200.0 if rng.random() < 0.33 else 6.0)
            s2 = max(s2, 0.55)
            th = rng.uniform(0, np.pi)
            c, s = np.cos(th), np.sin(th)
            cov = np.array([[c * c * s1 * s1 + s * s * s2 * s2, c * s * (s1 * s1 - s2 * s2)],
                            [c * s * (s1 * s1 - s2 * s2), s * s * s1 * s1 + c * c * s2 * s2]])
            con = np.linalg.inv(cov)
            mx, my = rng.uniform(-40, W + 40), rng.uniform(-40, H + 40)
            k, t = check_spans(mx, my, con[0, 0], con[0, 1], con[1, 1], rng.uniform(0.005, 1.0), tiles_x, tiles_y, ts,
                               f"seed {seed}")
            kept, total = kept + k, total + t
        # and the spans are tight: not more than ~1.6x the truly reachable tiles on this mix
        assert kept <= 1.6 * total + 50, (ts, kept, total)


@pytest.mark.parametrize("ts", LIST_TILES)
@pytest.mark.parametrize("seed", range(3))
def test_row_spans_cover_needles(ts, seed):
    """Needles up to 3000 px sigma along the long axis, down to no width at all but the eps2d blur (1e-4 .. 0.3), in a
    640 x 360 frame, centres on and off it.  The conic is what the kernel sees, the fp32 inverse of cov + eps2d I;
    one whose fp32 entries are no longer positive definite (A C - B^2 <= 0 in fp64) is not an ellipse the spans could
    describe and is left out (the kernel drops it: det <= 0)."""
    rng = np.random.default_rng(100 + seed)
    W, H = 640, 360
    tiles_x, tiles_y = -(-W // ts), -(-H // ts)
    tested = 0
    for _ in range(200):
        s1 = float(np.exp(rng.uniform(np.log(5.0), np.log(3000.0))))
        s2 = s1 * float(np.exp(rng.uniform(np.log(1e-6), np.log(0.05)))) if rng.random() < 0.8 else 0.0
        eps2d = float(np.exp(rng.uniform(np.log(1e-4), np.log(0.3))))
        th = rng.uniform(0, np.pi)
        c, s = np.cos(th), np.sin(th)
        cov = np.array([[c * c * s1 * s1 + s * s * s2 * s2 + eps2d, c * s * (s1 * s1 - s2 * s2)],
                        [c * s * (s1 * s1 - s2 * s2), s * s * s1 * s1 + c * c * s2 * s2 + eps2d]])
        con = np.linalg.inv(cov).astype(f32).astype(np.float64)
        if not con[0, 0] * con[1, 1] - con[0, 1] ** 2 > 0:
            continue
        mx, my = rng.uniform(-0.3 * W, 1.3 * W), rng.uniform(-0.3 * H, 1.3 * H)
        check_spans(mx, my, con[0, 0], con[0, 1], con[1, 1], rng.uniform(0.005, 1.0), tiles_x, tiles_y, ts,
                    f"needle s1={s1:.1f} s2={s2:.3g} eps2d={eps2d:.2g}")
        tested += 1
    assert tested >= 150, f"premise: {tested} positive-definite needles"
