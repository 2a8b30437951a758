"""GPU tests of the tile binning (csrc/binning.cu: dnr_bin_scan + dnr_bin_sort) per (Gaussian, list) pair, through the C
ABI and independent of the rasterizer, against oracle/binning_ref.py.

The contract: which pairs, in which order, with which offsets.
  1. superset  every pair the raster can composite (binning_ref.needed, fp64) is emitted; a miss is reported per Gaussian
               once brute force over its pixel centres confirms it;
  2. subset    every pair lies in the Gaussian's list box; the exact lists (DNR_FLAG_EXACT_LISTS) equal
               binning_ref.expected_lists bit for bit; the precise-hit lists emit at most R_s times the needed pairs;
  3. order     each list strictly increasing in (depth key, index), no culled Gaussian, offsets from 0 to the count,
               the count equal to dnr_bin_scan's host count and n_isects_dev, two runs bit-identical;
  4. the uint16 / uint32 key switch and the padding key's extra bit, at list counts on both sides of each boundary;
  5. capacities above the count (padded) and below it (truncated: binning_ref.truncated), and none at all.
Inputs are dnr_project_fwd's own outputs on project_ref's cases and a synthetic 1080p scene, and hand-made arrays for
the edges the projection never produces.
"""
import ctypes as C
import time

import numpy as np
import pytest
import torch

from oracle import binning_ref as BR
from oracle import project_ref as P

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]

MODES = [(0, True), (0, False), (1, False), (2, False), (3, False)]  # (list_shift, exact)
MODE_IDS = ["exact", "s0", "s1", "s2", "s3"]
# Precise-hit pairs emitted / needed pairs, the needed ones at the opacity the binning is given (cull_lim; without the
# antialiasing compensation, which it never sees).  The CPU mirror of row_span (tests/test_row_span_cpu.py) on the
# projected random case of test_projected_outputs (20k Gaussians, 640 x 480) gives 1.013 / 1.010 / 1.023 / 1.025 at
# list_shift 0..3 (the whole list boxes: 7.1 / 5.8 / 4.4 / 2.9); the bound leaves about 10 %.  The kernels measured
# 1.013 / 1.010 / 1.023 / 1.025 on that case, 1.018 / 1.017 / 1.014 / 1.025 over every input of this file, and at most
# 1.026 / 1.058 / 1.097 / 1.125 on one input set of more than a few Gaussians (the rank-1 antialiased case).
RATIO = {0: 1.12, 1: 1.12, 2: 1.15, 3: 1.15}
RATIO_SLACK = 64  # pairs: small input sets, where a few Gaussians whose reach ends right past a list edge weigh more
RATIOS_SEEN = {}


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _lib():
    from dn_splatter_b200 import _lib as L

    return L, L.load()


class Inputs:
    """The binning's inputs, host arrays: means2d f32 [N,2], radii i32, conics f32 [N,3], opac f32 (the opacity the raster
    sees), cull_lim f32, depth_keys i32 (the bits of a positive fp32 depth, -1 when culled).  `compensated`: opac holds
    the antialiasing compensation, which cull_lim does not."""

    def __init__(self, W, H, means2d, radii, conics, opac, cull_lim, depth_keys, what, compensated=False):
        self.W, self.H, self.what, self.compensated = W, H, what, compensated
        self.means2d = np.ascontiguousarray(means2d, dtype=np.float32).reshape(-1, 2)
        self.radii = np.ascontiguousarray(radii, dtype=np.int32)
        self.conics = np.ascontiguousarray(conics, dtype=np.float32).reshape(-1, 3)
        self.opac = np.ascontiguousarray(opac, dtype=np.float32)
        self.cull_lim = np.ascontiguousarray(cull_lim, dtype=np.float32)
        self.depth_keys = np.ascontiguousarray(depth_keys).astype(np.uint32).view(np.int32)
        self.n = self.radii.size

    @staticmethod
    def projected(case: P.Case, what):
        from tests.test_gpu_projection import Run

        o = Run(case).host_out
        return Inputs(case.width, case.height, o["means2d"].numpy(), o["radii"].numpy(), o["conics"].numpy(),
                      o["opac_act"].numpy(), o["cull_lim"].numpy(), o["depth_keys"].numpy(), what,
                      compensated=case.antialiased)


class Binner:
    """dnr_bin_scan once, then dnr_bin_sort at any capacity, on the device copies of `inp`."""

    def __init__(self, inp: Inputs, shift: int, exact: bool):
        L, lib = _lib()
        self.inp, self.shift, self.exact = inp, shift, exact
        self.ts = 16 << shift
        self.lx, self.ly = BR.lists_xy(inp.W, inp.H, self.ts)
        self.n_lists = self.lx * self.ly
        cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
        self.dev = dict(means2d=cuda(inp.means2d), radii=cuda(inp.radii), conics=cuda(inp.conics),
                        cull_lim=cuda(inp.cull_lim), depth_keys=cuda(inp.depth_keys),
                        tiles_per_gauss=torch.zeros(inp.n, dtype=torch.int32, device="cuda"),
                        n_isects_dev=torch.full((1,), -7, dtype=torch.int64, device="cuda"),
                        ws_scan=torch.empty(lib.dnr_bin_scan_workspace_bytes(inp.n), dtype=torch.uint8, device="cuda"))
        self.count = None

    def args(self, L):
        a = L.DnrArgs()
        a.n_gauss, a.width, a.height, a.tile_size = self.inp.n, self.inp.W, self.inp.H, 16
        a.flags = L.FLAG_EXACT_LISTS if self.exact else 0
        a.list_shift = self.shift
        for k, t in self.dev.items():
            setattr(a, k, t.data_ptr())
        return a

    def scan(self):
        """The host count, checked against n_isects_dev."""
        L, lib = _lib()
        a = self.args(L)
        total = C.c_int64(-1)
        L.check(lib.dnr_bin_scan(C.byref(a), _stream(), C.byref(total)), "dnr_bin_scan")
        torch.cuda.synchronize()
        self.count = int(total.value)
        assert int(self.dev["n_isects_dev"].item()) == self.count, f"{self.inp.what}: n_isects_dev != the host count"
        return self.count

    def sort(self, cap, ids=True):
        """(flatten_ids [cap] or None, offsets int64 [n_lists + 1], n_isects_dev) after dnr_bin_sort at capacity `cap`."""
        L, lib = _lib()
        a = self.args(L)
        a.n_isects = cap
        ws = torch.empty(lib.dnr_bin_sort_workspace_bytes(self.inp.n, cap, self.n_lists), dtype=torch.uint8, device="cuda")
        flat = torch.full((max(cap, 1),), -7, dtype=torch.int32, device="cuda") if ids else None
        offs = torch.full((self.n_lists + 1,), -7, dtype=torch.int32, device="cuda")
        a.ws_sort, a.tile_offsets = ws.data_ptr(), offs.data_ptr()
        if flat is not None:
            a.flatten_ids = flat.data_ptr()
        L.check(lib.dnr_bin_sort(C.byref(a), _stream()), "dnr_bin_sort")
        torch.cuda.synchronize()
        return (None if flat is None else flat[:cap].cpu().numpy(), offs.cpu().numpy().astype(np.int64),
                int(self.dev["n_isects_dev"].item()))


def _describe(inp, g, lid, lx):
    return (f"Gaussian {g}: mean {inp.means2d[g].tolist()} conic {inp.conics[g].tolist()} opacity {float(inp.opac[g])} "
            f"cull_lim {float(inp.cull_lim[g])} radius {int(inp.radii[g])}, list {lid} = ({lid % lx}, {lid // lx})")


def check_layout(b: Binner, ids, offs, count, what):
    """Checks 2 (box) and 3 (order, offsets) on one complete layout; returns its (gid, list id) pairs."""
    inp = b.inp
    assert offs[0] == 0 and offs[-1] == count, f"{what}: offsets run from {offs[0]} to {offs[-1]}, count {count}"
    assert bool((np.diff(offs) >= 0).all()), f"{what}: offsets decrease"
    assert ids.size == count
    gid, lid = BR.pairs_of(ids, offs)
    assert bool(((gid >= 0) & (gid < inp.n)).all()), f"{what}: Gaussian id out of range"
    culled = inp.radii[gid] <= 0
    assert not culled.any(), f"{what}: culled Gaussian {gid[culled][:5]} in the lists"
    x0, y0, x1, y1 = BR.list_box(inp.means2d, inp.radii, b.ts, b.lx, b.ly)
    lx, ly = lid % b.lx, lid // b.lx
    out = ~((lx >= x0[gid]) & (lx < x1[gid]) & (ly >= y0[gid]) & (ly < y1[gid]))
    assert not out.any(), f"{what}: pair outside the list box: {_describe(inp, int(gid[out][0]), int(lid[out][0]), b.lx)}"
    key = (inp.depth_keys.view(np.uint32)[gid].astype(np.uint64) << np.uint64(32)) | gid.astype(np.uint64)
    same = lid[1:] == lid[:-1]
    bad = same & ~(key[1:] > key[:-1])
    assert not bad.any(), (f"{what}: list {int(lid[1:][bad][0])} not strictly increasing in (depth key, index) at "
                           f"Gaussians {int(gid[:-1][bad][0])}, {int(gid[1:][bad][0])}")
    return gid, lid


def check_superset(b: Binner, gid, lid, what):
    """Check 1, and the precise-hit bound of check 2.  Returns (emitted, needed)."""
    inp = b.inp
    need_g, need_l = BR.needed(inp.means2d, inp.conics, inp.opac, inp.radii, b.ts, inp.W, inp.H)
    have = np.sort(lid * np.int64(inp.n) + gid)
    want = need_l * np.int64(inp.n) + need_g
    missing = have[np.minimum(np.searchsorted(have, want), have.size - 1)] != want if have.size else np.ones(want.size, bool)
    if missing.any():
        mg, ml = need_g[missing], need_l[missing]
        real = BR.needed_discrete(inp.means2d, inp.conics, inp.opac, inp.radii, mg, ml, b.ts, inp.W, inp.H)
        lines = [_describe(inp, int(g), int(l), b.lx) for g, l in zip(mg[real][:8], ml[real][:8])]
        assert not real.any(), (f"{what}: {int(real.sum())} reachable pairs not emitted, e.g.\n  " + "\n  ".join(lines))
    if inp.compensated:  # cull_lim = ln(255 op) + 0.1 of the opacity before the compensation
        op_bin = (np.exp(inp.cull_lim.astype(np.float64) - 0.1) / 255.0).astype(np.float32)
        need_g, _ = BR.needed(inp.means2d, inp.conics, np.maximum(op_bin, inp.opac), inp.radii, b.ts, inp.W, inp.H)
    return gid.size, need_g.size


def check_mode(inp: Inputs, shift, exact, caps=True):
    """Every check of one mode on one input set; returns the Binner and the complete layout."""
    what = f"{inp.what} {'exact' if exact else f'list_shift {shift}'}"
    b = Binner(inp, shift, exact)
    count = b.scan()
    ids, offs, dev = b.sort(count)
    assert dev == count
    gid, lid = check_layout(b, ids, offs, count, what)
    if exact:
        want_ids, want_offs = BR.expected_lists(inp.means2d, inp.radii, inp.depth_keys, b.ts, inp.W, inp.H)
        assert np.array_equal(offs, want_offs), f"{what}: offsets differ from the exact reference"
        assert np.array_equal(ids, want_ids), f"{what}: flatten_ids differ from the exact reference"
    else:
        emitted, needed = check_superset(b, gid, lid, what)
        RATIOS_SEEN.setdefault(shift, []).append((inp.what, emitted, needed))
        assert emitted <= RATIO[shift] * needed + RATIO_SLACK, f"{what}: {emitted} pairs emitted for {needed} needed"
    # bit-identical on a second scan + sort
    b2 = Binner(inp, shift, exact)
    assert b2.scan() == count
    ids2, offs2, _ = b2.sort(count)
    assert np.array_equal(ids, ids2) and np.array_equal(offs, offs2), f"{what}: two runs differ"
    if caps:
        check_capacities(b, ids, offs, what)
    return b, ids, offs


def _mid_gaussian_cap(b: Binner, ids, offs):
    """A capacity that cuts through the pairs of a Gaussian spanning two or more list rows (0 if there is none)."""
    gid, lid = BR.pairs_of(ids, offs)
    rank = BR.emission_rank(gid, lid, b.inp.depth_keys)
    order = np.argsort(rank)
    g, row = gid[order], (lid // b.lx)[order]
    multi = np.nonzero((g[1:] == g[:-1]) & (row[1:] != row[:-1]))[0]
    return int(multi[len(multi) // 2]) + 1 if multi.size else 0


def check_capacities(b: Binner, ids, offs, what):
    """Check 5 around the complete layout (ids, offs) of capacity = count."""
    c = b.count
    for cap in (c + 1, c + 4096):
        got, got_offs, dev = b.sort(cap)
        assert dev == c, f"{what} cap {cap}: n_isects_dev"
        assert np.array_equal(got_offs, offs), f"{what} cap {cap}: padded offsets differ"
        assert np.array_equal(got[:c], ids), f"{what} cap {cap}: padded ids differ"
    for cap in sorted({c - 1, c // 2, 1, _mid_gaussian_cap(b, ids, offs)}):
        if not 0 < cap < c:
            continue
        got, got_offs, dev = b.sort(cap)
        want_ids, want_offs = BR.truncated(ids, offs, b.inp.depth_keys, cap)
        assert dev == c, f"{what} cap {cap}: n_isects_dev must keep the count"
        assert got_offs[-1] == cap and np.array_equal(got_offs, want_offs), f"{what} cap {cap}: truncated offsets"
        assert np.array_equal(got, want_ids), f"{what} cap {cap}: truncated ids"
    _, got_offs, dev = b.sort(0, ids=False)
    assert dev == c and not got_offs.any(), f"{what}: cap 0 offsets"


def _report():
    for s, rows in sorted(RATIOS_SEEN.items()):
        e, n = sum(r[1] for r in rows), sum(r[2] for r in rows)
        print(f"list_shift {s}: emitted / needed = {e} / {n} = {e / max(n, 1):.3f}  "
              + ", ".join(f"{w}: {x / max(y, 1):.3f}" for w, x, y in rows))


# ----------------------------------------------------------------------------------------------------- (a) projected
def _projected(name):
    if name == "random":
        return Inputs.projected(P.random_case(20000, 1, width=640, height=480), name)
    if name == "random_aa":
        return Inputs.projected(P.random_case(8000, 2, width=333, height=250, antialiased=True), name)
    if name == "edge_on":
        return Inputs.projected(P.edge_on_case(5000, 3, width=320, height=240), name)
    if name == "rank1":
        return Inputs.projected(P.random_case(5000, 4, kind="rank1", sh_bases=4, sh_degree=1, width=320, height=200,
                                              antialiased=True), name)
    if name == "scene_200k":
        return Inputs.projected(_scene_case(200_000, 1920, 1080), name)
    raise ValueError(name)


def _scene_case(n, W, H):
    from dn_splatter_b200.synthetic import make_scene, ring_cameras
    from oracle.dn_ref import get_viewmat

    p = make_scene(n, seed=0)
    cam = ring_cameras(200, W, H)[17]
    K = torch.tensor([[cam["fx"], 0, cam["cx"]], [0, cam["fy"], cam["cy"]], [0, 0, 1]], dtype=torch.float32)
    params = dict(means=p["means"], quats=p["quats"], scales=p["scales"], opacities=p["opacities"].reshape(-1),
                  sh_dc=p["features_dc"], sh_rest=p["features_rest"])
    return P.Case(params, get_viewmat(cam["c2w"].double()).float(), K, cam["c2w"], W, H)


PROJECTED = ["random", "random_aa", "edge_on", "rank1", "scene_200k"]
_CACHE = {}


def _cached(key, fn):
    if key not in _CACHE:
        _CACHE[key] = fn()
    return _CACHE[key]


@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("name", PROJECTED)
def test_projected_outputs(name, mode):
    inp = _cached(name, lambda: _projected(name))
    assert int((inp.radii > 0).sum()) > 0.2 * inp.n, "premise: visible Gaussians"
    check_mode(inp, *mode, caps=name != "scene_200k")


# ----------------------------------------------------------------------------------------------------- (b) hand-made
def _iso(n, rng, sig_lo=0.6, sig_hi=6.0):
    """Isotropic / mildly elongated conics with their 3-sigma radius (as project_fwd rounds it)."""
    s1 = rng.uniform(sig_lo, sig_hi, n)
    s2 = s1 / rng.uniform(1.0, 3.0, n)
    th = rng.uniform(0, np.pi, n)
    c, s = np.cos(th), np.sin(th)
    a = c * c * s1 * s1 + s * s * s2 * s2
    b = c * s * (s1 * s1 - s2 * s2)
    cc = s * s * s1 * s1 + c * c * s2 * s2
    det = a * cc - b * b
    con = np.stack([cc / det, -b / det, a / det], 1)
    lam = 0.5 * (a + cc) + np.sqrt(np.maximum(0.25 * (a - cc) ** 2 + b * b, 0.01))
    return con, np.ceil(3 * np.sqrt(lam)).astype(np.int32)


def _depth_bits(d):
    return np.asarray(d, dtype=np.float32).view(np.int32)


def handmade(n, W, H, seed, what, keys="random", sig=(0.6, 6.0)):
    """n Gaussians scattered over and just around a W x H frame (the first two on its corners)."""
    rng = np.random.default_rng(seed)
    con, r = _iso(n, rng, *sig)
    m = np.stack([rng.uniform(-10, W + 10, n), rng.uniform(-10, H + 10, n)], 1)
    m[0] = (0.5, 0.5)
    if n > 1:
        m[1] = (W - 0.5, H - 0.5)
    op = rng.uniform(0.05, 1.0, n).astype(np.float32)
    cull = (np.log(255.0 * op.astype(np.float64)) + 0.1).astype(np.float32)
    if keys == "random":
        dk = _depth_bits(rng.uniform(0.2, 40.0, n))
    elif keys == "equal":
        dk = _depth_bits(np.full(n, 3.0))
    elif keys == "last_bit":  # 0x40400000 / 0x40400001
        dk = _depth_bits(np.full(n, 3.0)) + rng.integers(0, 2, n).astype(np.int32)
    else:
        raise ValueError(keys)
    return Inputs(W, H, m, r, con, op, cull, dk, what)


# list counts around 2^8 and 2^16 (uint16 / uint32 keys; the padding key n_lists needs one bit more at a power of two)
SIZES = [(1, 1, 0), (16, 16, 0), (4080, 16, 0), (256, 256, 0), (4112, 16, 0), (4112, 4080, 0), (4096, 4096, 0),
         (8192, 8192, 1)]


@pytest.mark.parametrize("W,H,shift", SIZES, ids=[f"{w}x{h}-s{s}" for w, h, s in SIZES])
def test_list_counts_and_key_widths(W, H, shift):
    ts = 16 << shift
    lx, ly = BR.lists_xy(W, H, ts)
    n = 3000 if lx * ly > 1 else 50
    inp = handmade(n, W, H, seed=W + H + shift, what=f"{W}x{H} ({lx * ly} lists)")
    for exact in ((False, True) if shift == 0 else (False,)):
        b, ids, offs = check_mode(inp, shift, exact)
        assert offs[1] > 0 and offs[-1] > offs[-2], f"{inp.what}: list 0 and the last list must be populated"


def _specials(W, H):
    """Gaussians at the edges the projection never produces, appended after a random set: (arrays, index groups)."""
    rows, groups = [], {}

    def add(group, mx, my, con, radius, op=None, cull=None, key=3.0):
        """`op` or `cull` (cull_lim = ln(255 op) + 0.1, as project_fwd pairs them)."""
        groups.setdefault(group, []).append(len(rows))
        op = float(np.exp(cull - 0.1) / 255.0) if op is None else op
        c = np.log(255.0 * op) + 0.1 if cull is None else cull
        rows.append((mx, my, *con, radius, op, c, key))

    iso = lambda s: (1 / (s * s), 0.0, 1 / (s * s))  # noqa: E731
    for i in range(4):  # radius > 0, but no pixel can reach 1/255: cull_lim <= 0
        add("no_reach", W * 0.3 + 7 * i, H * 0.4, iso(4.0), 12, 0.003, key=1.0 + i)
    add("no_reach", W * 0.5, H * 0.5, iso(4.0), 12, cull=0.0)
    add("no_reach", W * 0.5, H * 0.5, iso(4.0), 12, cull=-1.0)
    for mx, my in ((W + 5000.0, H * 0.5), (-5000.0, H * 0.5), (W * 0.5, H + 5000.0), (W * 0.5, -5000.0)):
        add("off_box", mx, my, iso(4.0), 12, 0.8)  # box entirely off-screen (beyond every list)
    for mx, my, s in ((-20.0, H * 0.5, 10.0), (W + 20.0, H * 0.3, 10.0), (W * 0.6, -25.0, 12.0), (W * 0.2, H + 25.0, 12.0),
                      (-30.0, -30.0, 15.0), (W + 30.0, H + 30.0, 15.0)):
        add("off_centre", mx, my, iso(s), int(np.ceil(3 * s)), 0.9)  # centre off-screen, splat reaching in
    # needles (eps2d 2e-4 .. 9e-4, 550 - 1500 px long) whose fp32 conic is an ellipse, but the plain fp32 A C - B^2 of
    # it, with or without a fused multiply-add, is <= 0: load_hit_gauss took them for unreachable and dropped every pair
    for A, B, Cc, r in ((94.84357452392578, 608.4221801757812, 3903.032470703125, 4446),
                        (172.5365753173828, -254.3012237548828, 374.8139343261719, 1651),
                        (255.6551513671875, 589.6783447265625, 1360.1156005859375, 2210),
                        (1181.9344482421875, -170.58506774902344, 24.620033264160156, 3669)):
        add("needle", W * 0.5 + 0.25, H * 0.5 - 0.25, (A, B, Cc), r, 0.9, key=2.0)
    for k in range(3):  # identical Gaussians at different indices
        add("twins", W * 0.45, H * 0.55, (0.02, 0.005, 0.03), 25, 0.7, key=2.5)
    add("culled", W * 0.5, H * 0.5, iso(3.0), 0, 0.8, key=np.float32(np.nan))
    return rows, groups


def handmade_edges(n, W, H, seed, keys="random"):
    base = handmade(n, W, H, seed, f"edges {W}x{H} n={n} keys={keys}", keys=keys)
    rows, groups = _specials(W, H)
    a = np.array(rows, dtype=np.float64)
    k = a[:, 8].astype(np.float32).view(np.int32).copy()
    k[groups["culled"]] = -1
    inp = Inputs(W, H, np.concatenate([base.means2d, a[:, 0:2]]), np.concatenate([base.radii, a[:, 5]]),
                 np.concatenate([base.conics, a[:, 2:5]]), np.concatenate([base.opac, a[:, 6]]),
                 np.concatenate([base.cull_lim, a[:, 7]]), np.concatenate([base.depth_keys, k]), base.what)
    return inp, {g: np.array(v) + base.n for g, v in groups.items()}


@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("keys", ["random", "equal", "last_bit"])
def test_handmade_edges(keys, mode):
    """Ragged frame (not a multiple of any list tile); depth keys all equal / differing in the last bit only (the order
    is then the index order); the special Gaussians of _specials."""
    shift, exact = mode
    W, H = 333, 201
    inp, groups = handmade_edges(4000, W, H, seed=7, keys=keys)
    b, ids, offs = check_mode(inp, shift, exact)
    gid, lid = BR.pairs_of(ids, offs)
    what = f"{inp.what} {MODE_IDS[MODES.index(mode)]}"
    assert not np.isin(gid, groups["off_box"]).any(), f"{what}: a box off the frame emitted a pair"
    if not exact:  # (the exact lists keep the whole box: the exact reference has held them to it)
        assert not np.isin(gid, groups["no_reach"]).any(), f"{what}: a Gaussian that reaches no pixel emitted a pair"
    for g in groups["off_centre"]:
        assert (gid == g).any(), f"{what}: off-screen centre {g} reaching into the frame has no list"
    for g in groups["needle"]:
        assert (gid == g).any(), f"{what}: the needle {g} through the frame's centre emits no pair"
    tw = [set(lid[gid == g].tolist()) for g in groups["twins"]]
    assert tw[0] and tw[0] == tw[1] == tw[2], f"{what}: identical Gaussians get different lists"
    if exact:
        x0, y0, x1, y1 = BR.list_box(inp.means2d, inp.radii, b.ts, b.lx, b.ly)
        g = groups["no_reach"]
        assert int((gid[:, None] == g[None, :]).sum()) == int(((x1 - x0) * (y1 - y0))[g].sum()) > 0


@pytest.mark.parametrize("n", [1, 255, 256, 257])
@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
def test_gaussian_counts(n, mode):
    """count_kernel runs n + 1 lanes: the Gaussian counts around a block of 256."""
    inp = handmade(n, 200, 120, seed=n, what=f"n={n}", sig=(2.0, 20.0))
    check_mode(inp, *mode)


@pytest.mark.parametrize("mode", [(2, False), (0, True)], ids=["s2", "exact"])
def test_million_gaussians_1080p(mode):
    """About 1M Gaussians at 1920 x 1080, the benchmark's size: the production lists (list_shift 2) and the exact ones."""
    inp = _cached("scene_1m", lambda: Inputs.projected(_scene_case(1_000_000, 1920, 1080), "scene_1m"))
    t = time.perf_counter()
    check_mode(inp, *mode, caps=False)
    print(f"1M Gaussians {MODE_IDS[MODES.index(mode)]}: {time.perf_counter() - t:.1f} s")


def test_zz_report_ratios():
    """Prints the emitted / needed pair ratios the precise-hit tests above measured (run with -s)."""
    _report()
