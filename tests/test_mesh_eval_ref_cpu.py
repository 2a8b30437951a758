"""CPU checks of the fp64 restatement of dnr_mesh_depth / dnr_mesh_visibility in oracle/mesh_eval_ref.py: the kernel's
rule against the independent Moller-Trumbore ray cast and a scalar loop, the kernel's box pass and item search against
the rule's wider boxes, the reach of every case of tests/test_gpu_mesh_eval_kernels.py, and that each restated kernel
slip changes some pixel or count on those cases."""
import numpy as np
import pytest

from oracle import mesh_eval_ref as R
from tests import mesh_eval_cases as C


@pytest.fixture(scope="module")
def cases():
    return C.depth_cases()


def _legacy(W, H):
    return [(n, v, f, C.block32(c2w, fx, fy, cx, cy)) for n, v, f, c2w, fx, fy, cx, cy in C.legacy_scenes(W, H)]


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("W,H", [(81, 49), (75, 53)])
def test_rule_equals_the_ray_cast_away_from_edges(W, H):
    for name, v, f, blk in _legacy(W, H):
        v32 = np.asarray(v, np.float32)
        rule, _ = R.depth_kernel_rule(v32, f, blk, W, H)
        cam = blk.astype(np.float64)
        rc = R.ray_cast_depth(v32.astype(np.float64), f, cam, W, H)
        amb = R.near_edge_pixels(v32.astype(np.float64), f, cam, W, H)
        assert np.array_equal((rule > 0)[~amb], (rc > 0)[~amb]), name
        both = (rule > 0) & (rc > 0) & ~amb
        ulp = np.abs(_bits(rule[both]).astype(np.int64) - _bits(rc[both]).astype(np.int64))
        assert ulp.max(initial=0) <= 1, (name, int(ulp.max()))
        assert ((rule > 0) & (rc > 0)).sum() > 0.2 * W * H, name


def test_rule_equals_a_scalar_loop(cases):
    small = [c for c in cases if c["name"] in ("near_far", "bad_faces", "duplicates")]
    for name, v, f, blk in _legacy(31, 23):
        small.append(C._case(name, v, f, blk, 31, 23))
    for c in small:
        for cam in c["cams"]:
            rule, _ = R.depth_kernel_rule(c["verts"], c["faces"], cam, c["W"], c["H"], c["near"], c["far"])
            ref = R.depth_scalar(c["verts"], c["faces"], cam, c["W"], c["H"], c["near"], c["far"])
            assert np.array_equal(_bits(rule), _bits(ref)), c["name"]


def _reached(c, cam):
    rule, stats = R.depth_kernel_rule(c["verts"], c["faces"], cam, c["W"], c["H"], c["near"], c["far"])
    mirror, mstats, boxes, counts = R.depth_kernel_mirror(c["verts"], c["faces"], cam, c["W"], c["H"], c["near"], c["far"])
    live = counts > 0
    bw, bh = boxes[live, 1] - boxes[live, 0] + 1, boxes[live, 3] - boxes[live, 2] + 1
    got = {k for k, n in stats.items() if n > 0} | {f"area:{a}" for a in (bw * bh).tolist()}
    got |= {"1xN"} if ((bw == 1) & (bh > 1)).any() else set()
    got |= {"Nx1"} if ((bh == 1) & (bw > 1)).any() else set()
    return rule, mirror, stats, mstats, got


def test_each_case_reaches_its_branches_and_the_kernel_boxes_hold_every_hit(cases):
    for c in cases:
        reached = set()
        for cam in c["cams"]:
            rule, mirror, stats, mstats, got = _reached(c, cam)
            assert np.array_equal(_bits(rule), _bits(mirror)), c["name"]  # the kernel's boxes lose no pixel of the rule
            assert (stats["hit"], stats["tie"]) == (mstats["hit"], mstats["tie"]), c["name"]
            reached |= got
            if c["name"].startswith("closed"):
                assert (rule > 0).all(), c["name"]  # seen from inside, every pixel hits
        assert set(c["reach"]) <= reached, (c["name"], set(c["reach"]) - reached)
        print(c["name"], {k: v for k, v in stats.items()})


def _watertight(cases):
    out = [c for c in cases if c["watertight"]]
    for W, H in ((81, 49), (75, 53)):
        out += [C._case(n, v, f, blk, W, H, watertight=True) for n, v, f, blk in _legacy(W, H) if n == "edges"]
    return out


def test_rule_loses_no_pixel_on_shared_edges_and_a_strict_inside_test_would(cases):
    """Watertightness against the independent ray cast: every pixel the ray cast hits along with its 4 neighbours is hit
    by the rule; the strict-inside slip leaves holes at pixel centres on shared edges there, so the check bites."""
    holes = {}
    for c in _watertight(cases):
        for cam in c["cams"]:
            inner = C.interior_hits(c["verts"], c["faces"], cam, c["W"], c["H"], c["near"], c["far"])
            rule, _ = R.depth_kernel_rule(c["verts"], c["faces"], cam, c["W"], c["H"], c["near"], c["far"])
            assert inner.sum() > 0.5 * c["W"] * c["H"] and (rule[inner] > 0).all(), c["name"]
            bad = R.depth_kernel_mirror(c["verts"], c["faces"], cam, c["W"], c["H"], c["near"], c["far"], slip="strict_inside")[0]
            holes[f"{c['name']} {c['W']}x{c['H']}"] = int((bad[inner] == 0).sum())
    print("holes the strict-inside slip leaves on shared edges:", holes)
    assert holes["grid_rot90 96x96"] > 0 and holes["edges 81x49"] > 0 and holes["edges 75x53"] > 0


def test_many_views_case_differs_per_view():
    c = C.many_views_case(64, 32, 24)
    outs = [R.depth_kernel_rule(c["verts"], c["faces"], cam, c["W"], c["H"])[0] for cam in c["cams"]]
    assert len({o.tobytes() for o in outs}) == len(outs)
    assert min(int((o > 0).sum()) for o in outs) == c["W"] * c["H"]  # from inside the room


def _slip_changes(cases, slip):
    """{case: (pixels changed, faces whose box or item count changed)} where the slip changes something."""
    changed = {}
    for c in cases:
        for cam in c["cams"]:
            base, _, bb, bc = R.depth_kernel_mirror(c["verts"], c["faces"], cam, c["W"], c["H"], c["near"], c["far"])
            bad, _, sb, sc = R.depth_kernel_mirror(c["verts"], c["faces"], cam, c["W"], c["H"], c["near"], c["far"], slip=slip)
            n = int((_bits(base) != _bits(bad)).sum())
            m = int(((bb != sb).any(1) | (bc != sc)).sum())
            if n or m:
                p, q = changed.get(c["name"], (0, 0))
                changed[c["name"]] = (p + n, q + m)
    return changed


# the kernel's 1-px box margin guards against fp64 rounding at pixel centres on a vertex's ray, which no case reaches:
# that slip shows in the boxes and item counts the GPU test reads back from the workspace, not in any pixel
BOX_ONLY_SLIPS = ("no_box_margin",)


@pytest.mark.parametrize("slip", R.DEPTH_SLIPS)
def test_each_depth_slip_changes_some_pixel(cases, slip):
    legacy = [C._case(n, v, f, blk, 81, 49) for n, v, f, blk in _legacy(81, 49)]
    changed = _slip_changes(cases + legacy, slip)
    print(f"slip {slip} caught: (pixels, boxes) changed per case {changed}")
    assert changed, slip
    if slip not in BOX_ONLY_SLIPS:
        assert any(n for n, _ in changed.values()), slip


def test_visibility_case_reaches_its_edges():
    pts, blocks, rendered, gt, eps = C.visibility_case()
    W, H = C.VIS_W, C.VIS_H
    px, py, pz = R.project_points(pts, blocks[0])
    for name, m in (("px=0", px == 0), ("px=W-1", px == W - 1), ("py=0", py == 0), ("py=H-1", py == H - 1),
                    ("pz=0", pz == 0), ("pz<0", (pz < 0) & (pz > -1e-7)), ("pz>0 tiny", (pz > 0) & (pz < 1e-7)),
                    ("nan", np.isnan(px) & np.isnan(pts).any(1))):
        assert m.sum() > 0, name
    inside = (px >= 0) & (px <= W - 1) & (py >= 0) & (py <= H - 1) & (pz > 0)
    u, v = np.clip(np.nan_to_num(px), 0, W - 1).astype(np.int64), np.clip(np.nan_to_num(py), 0, H - 1).astype(np.int64)
    lim = (rendered[0][v, u] + np.float32(eps)).astype(np.float64)
    assert (inside & (pz == lim)).sum() > 100  # pz exactly on the occlusion threshold
    assert (inside & (rendered[0][v, u] == 0)).sum() > 0
    obs, inv = R.visibility_counts(pts, blocks, W, H, rendered, gt, eps)
    assert obs.max() > 3 and (inv > 0).any() and (obs == 0).any()


@pytest.mark.parametrize("slip", R.VIS_SLIPS)
def test_each_visibility_slip_changes_some_count(slip):
    pts, blocks, rendered, gt, eps = C.visibility_case()
    base = R.visibility_counts(pts, blocks, C.VIS_W, C.VIS_H, rendered, gt, eps)
    bad = R.visibility_counts(pts, blocks, C.VIS_W, C.VIS_H, rendered, gt, eps, slip=slip)
    n = int(((base[0] != bad[0]) | (base[1] != bad[1])).sum())
    print(f"slip {slip} caught: {n} points change count")
    assert n > 0, slip


def test_stratified_pixels_cover_item_boundaries():
    c = C.item_boundary_case()
    cam = c["cams"][0]
    _, _, _, _, E = R.kernel_camera(cam)
    T = R.triangle_setup(c["verts"], c["faces"], E)
    boxes, counts = R.kernel_boxes(T, cam, c["W"], c["H"], c["near"], c["far"])
    pix = C.stratified_pixels(c["W"], c["H"], boxes, counts, np.random.default_rng(0))
    f = int(np.nonzero(counts == 2)[0][0])  # a box of 257..512 pixels: pixels 255 and 256 of its raster order
    b = boxes[f]
    bw = b[1] - b[0] + 1
    for p in (255, 256):
        assert (b[2] + p // bw) * c["W"] + b[0] + p % bw in set(pix.tolist())
    assert set(range(c["W"])) <= set(pix.tolist())
