"""dnr_mesh_depth and dnr_mesh_visibility per pixel and per point against the kernel's own fp64 rule
(oracle/mesh_eval_ref.py): depth bits equal on every pixel, the box pass's boxes, item counts and scan equal to its
restatement, two runs bit-identical, counts equal.  Cases: tests/mesh_eval_cases.py, plus the eval script's workload
(1200 x 680, 20 views, about 6.5e5 faces) on a stratified pixel set.  Prints, per case, the pixels that reached each
decision of the rule (near / far rejects and equalities, an edge function exactly 0, den = 0, ties)."""
import time

import numpy as np
import pytest
import torch

from oracle import mesh_eval_ref as R
from tests import mesh_eval_cases as C

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]


def _a256(x):
    return (x + 255) & ~255


def render(verts, faces, cams, W, H, near=C.NEAR, far=C.FAR):
    """dnr_mesh_depth on the device: (depth [V,H,W] float32, the workspace's boxes [F,4], item counts and inclusive scan
    of the last view; the kernel leaves them there: boxes int4 at 0, counts and scan int64 at the next 256-B
    boundaries)."""
    from dn_splatter_b200 import _lib as L
    from dn_splatter_b200.sugar import _stream

    lib = L.load()
    v = torch.from_numpy(np.ascontiguousarray(verts, np.float32)).cuda()
    f = torch.from_numpy(np.ascontiguousarray(faces, np.int32)).cuda()
    c = torch.from_numpy(np.ascontiguousarray(np.asarray(cams, np.float32).reshape(-1, 16))).cuda()
    F, V = f.shape[0], c.shape[0]
    nbytes = lib.dnr_mesh_depth_workspace_bytes(F)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    out = torch.empty((V, H, W), dtype=torch.float32, device="cuda")
    L.check(lib.dnr_mesh_depth(v.data_ptr(), v.shape[0], f.data_ptr(), F, c.data_ptr(), V, W, H, float(near), float(far),
                               ws.data_ptr(), nbytes, out.data_ptr(), _stream()), "dnr_mesh_depth")
    w = ws.cpu().numpy()
    o_cnt = _a256(16 * F)
    o_scan = _a256(o_cnt + 8 * F)
    boxes = w[:16 * F].view(np.int32).reshape(F, 4).astype(np.int64)
    counts = w[o_cnt:o_cnt + 8 * F].view(np.int64)
    scan = w[o_scan:o_scan + 8 * F].view(np.int64)
    return out.cpu().numpy(), boxes, counts, scan


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def _check_boxes(verts, faces, cam, W, H, near, far, boxes, counts, scan, name):
    _, _, _, _, E = R.kernel_camera(cam)
    T = R.triangle_setup(verts, faces, E)
    rb, rc = R.kernel_boxes(T, cam, W, H, near, far)
    assert np.array_equal(boxes, rb), (name, int((boxes != rb).any(1).sum()))
    assert np.array_equal(counts, rc) and np.array_equal(scan, np.cumsum(rc)), name


CASES = {c["name"]: c for c in C.depth_cases()}


@pytest.mark.parametrize("name", list(CASES))
def test_depth_bits_equal_the_rule(name):
    c = CASES[name]
    W, H, near, far = c["W"], c["H"], c["near"], c["far"]
    total = {k: 0 for k in R.DECISIONS}
    for k, cam in enumerate(c["cams"]):
        got, boxes, counts, scan = render(c["verts"], c["faces"], cam, W, H, near, far)
        again = render(c["verts"], c["faces"], cam, W, H, near, far)[0]
        assert np.array_equal(_bits(got), _bits(again)), name
        want, stats = R.depth_kernel_rule(c["verts"], c["faces"], cam, W, H, near, far)
        bad = _bits(got[0]) != _bits(want)
        assert not bad.any(), (name, k, int(bad.sum()), np.argwhere(bad)[:5].tolist())
        _check_boxes(c["verts"], c["faces"], cam, W, H, near, far, boxes, counts, scan, name)
        if name.startswith("closed"):
            assert (got > 0).all(), name
        if c["watertight"]:  # against the independent ray cast: no pixel centre on a shared edge is lost by both faces
            inner = C.interior_hits(c["verts"], c["faces"], cam, W, H, near, far)
            assert inner.sum() > 0.5 * W * H and (got[0][inner] > 0).all(), (name, int((got[0][inner] == 0).sum()))
        for d in total:
            total[d] += stats[d]
    print(f"{name}: pixels per decision {total}, items {int(counts.sum())}")


@pytest.mark.parametrize("W,H", [(81, 49), (75, 53)])
def test_legacy_scenes_bits_equal_the_rule(W, H):
    for name, v, f, c2w, fx, fy, cx, cy in C.legacy_scenes(W, H):
        cam = C.block32(c2w, fx, fy, cx, cy)
        got = render(np.asarray(v, np.float32), f, cam, W, H)[0][0]
        want, stats = R.depth_kernel_rule(np.asarray(v, np.float32), f, cam, W, H)
        assert np.array_equal(_bits(got), _bits(want)), (name, int((_bits(got) != _bits(want)).sum()))
        if name == "edges":
            inner = C.interior_hits(v, f, cam, W, H)
            assert inner.sum() > 0.5 * W * H and (got[inner] > 0).all(), (name, int((got[inner] == 0).sum()))
        print(f"{name} {W}x{H}: pixels per decision {stats}")


@pytest.mark.parametrize("n", [64, 200])
def test_many_views_in_one_call_equal_their_single_view_calls(n):
    c = C.many_views_case(n)
    W, H = c["W"], c["H"]
    batch = render(c["verts"], c["faces"], c["cams"], W, H)[0]
    assert len({b.tobytes() for b in batch}) == n  # every view differs
    for k, cam in enumerate(c["cams"]):
        one = render(c["verts"], c["faces"], cam, W, H)[0][0]
        assert np.array_equal(_bits(batch[k]), _bits(one)), k
        if k % 8 == 0:
            want, _ = R.depth_kernel_rule(c["verts"], c["faces"], cam, W, H)
            assert np.array_equal(_bits(one), _bits(want)), k
    assert (batch > 0).all()  # from inside the room


# ------------------------------------------------------------------------------------------------ production size
@pytest.fixture(scope="module")
def production():
    v, f = C.production_mesh()
    cams = C.production_blocks()
    v32 = v.astype(np.float32)
    t = time.time()
    got, boxes, counts, scan = render(v32, f, cams, C.PROD_W, C.PROD_H)
    torch.cuda.synchronize()
    print(f"production: {f.shape[0]} faces, {len(cams)} views at {C.PROD_W}x{C.PROD_H} rendered in {time.time() - t:.2f} s "
          "(one call, first launch included)")
    return v, f, v32, cams, got, boxes, counts, scan


def test_production_depth_equals_the_rule_on_stratified_pixels(production):
    v, f, v32, cams, got, boxes, counts, scan = production
    W, H = C.PROD_W, C.PROD_H
    assert 4e5 < f.shape[0] < 1e6
    _check_boxes(v32, f, cams[-1], W, H, C.NEAR, C.FAR, boxes, counts, scan, "production")
    again = render(v32, f, cams, W, H)[0]
    assert np.array_equal(_bits(got), _bits(again))
    rng = np.random.default_rng(3)
    total = {k: 0 for k in R.DECISIONS}
    n_pix = 0
    t = time.time()
    for k, cam in enumerate(cams):
        _, _, _, _, E = R.kernel_camera(cam)
        kb, kc = R.kernel_boxes(R.triangle_setup(v32, f, E), cam, W, H, C.NEAR, C.FAR)
        pix = C.stratified_pixels(W, H, kb, kc, rng)
        want, stats = R.depth_kernel_rule(v32, f, cam, W, H, pixels=pix, whole_frame_straddlers=False)
        g = got[k].reshape(-1)[pix]
        bad = _bits(g) != _bits(want)
        assert not bad.any(), (k, int(bad.sum()), pix[bad][:5].tolist())
        assert (got[k] > 0).all(), k  # inside the closed room
        n_pix += pix.size
        for d in total:
            total[d] += stats[d]
    print(f"production: {n_pix} stratified pixels over {len(cams)} views equal the rule ({time.time() - t:.1f} s on the "
          f"host); pixels per decision {total}; items in the last view {int(counts.sum())}, faces with more than one "
          f"item {int((counts > 1).sum())}")


def test_production_cull_mesh_equals_the_oracle(production):
    from dn_splatter_b200.mesh import TriangleMesh
    from dn_splatter_b200.mesh_eval import cull_mesh

    v, f, v32, cams, got, _, _, _ = production
    W, H = C.PROD_W, C.PROD_H
    views = _cameras(cams, W, H)
    gt = got.copy()
    gt[:, : H // 4, : W // 3] = 0.0  # missing sensor depth in a corner of every view
    t = time.time()
    culled = cull_mesh(TriangleMesh(torch.from_numpy(v32), torch.from_numpy(f.astype(np.int32)), None), views,
                       torch.from_numpy(gt).cuda(), max_edge=0.03, chunk=16)
    torch.cuda.synchronize()
    dt = time.time() - t
    blocks = [R.camera_block(c.camera_to_worlds[0].double().numpy(), float(c.fx[0, 0]), float(c.fy[0, 0]),
                             float(c.cx[0, 0]), float(c.cy[0, 0])) for c in views]
    # max_edge 0.03 splits the 0.05 room faces once (about 2.6e6 subdivided faces) and keeps the numpy oracle in reach
    rv, rf, _, _ = R.cull_mesh(v32.astype(np.float64), f, blocks, W, H, gt_depths=list(gt), depths=list(got), max_edge=0.03)
    assert 0 < rf.shape[0]
    assert np.array_equal(R.triangle_multiset(culled.vertices.cpu().numpy(), culled.faces.cpu().numpy()),
                          R.triangle_multiset(rv, rf))
    print(f"production cull_mesh: {rf.shape[0]} faces kept, {dt:.2f} s on the device")


def _cameras(blocks32, W, H):
    """Cameras of the production views; their fp32 blocks are the ones rendered."""
    from dn_splatter_b200.cameras import Cameras
    from dn_splatter_b200.mesh_eval import camera_blocks

    views = [Cameras(torch.from_numpy(c2w)[None], *C.PROD_INTRINSICS, W, H) for c2w in C.production_poses()]
    assert np.array_equal(camera_blocks(views, torch.float32).cpu().numpy(), blocks32)
    return views


# ------------------------------------------------------------------------------------------------ visibility
@pytest.mark.parametrize("chunk", [1, 5, 16, 64])
def test_visibility_counts_equal_the_oracle_per_chunk(chunk):
    from dn_splatter_b200 import _lib as L
    from dn_splatter_b200.sugar import _stream

    pts, blocks, rendered, gt, eps = C.visibility_case()
    W, H, V = C.VIS_W, C.VIS_H, len(blocks)
    assert V % chunk != 0 or chunk == 1
    p = torch.from_numpy(pts).cuda()
    cams = torch.from_numpy(blocks).cuda()
    rd, gd = torch.from_numpy(rendered).cuda(), torch.from_numpy(gt).cuda()
    for tag, use_r, use_g in (("both", True, True), ("no_occlusion", False, True), ("no_missing", True, False)):
        obs = torch.zeros(len(pts), dtype=torch.int32, device="cuda")
        inv = torch.zeros_like(obs)
        for c0 in range(0, V, chunk):
            c1 = min(c0 + chunk, V)
            L.check(L.load().dnr_mesh_visibility(p.data_ptr(), len(pts), cams[c0:c1].contiguous().data_ptr(),
                                                 rd[c0:c1].contiguous().data_ptr() if use_r else None,
                                                 gd[c0:c1].contiguous().data_ptr() if use_g else None, c1 - c0, W, H,
                                                 float(eps), obs.data_ptr(), inv.data_ptr(), _stream()), "dnr_mesh_visibility")
        ro, ri = R.visibility_counts(pts, blocks, W, H, rendered if use_r else None, gt if use_g else None, eps)
        o, i = obs.cpu().numpy(), inv.cpu().numpy()
        assert np.array_equal(o, ro), (tag, int((o != ro).sum()))
        assert np.array_equal(i, ri), (tag, int((i != ri).sum()))


def test_visibility_counts_through_the_python_surface():
    from dn_splatter_b200.cameras import Cameras
    from dn_splatter_b200.mesh_eval import camera_blocks, visibility_counts

    W, H = C.VIS_W, C.VIS_H
    g = np.random.default_rng(2)
    views = []
    for k in range(23):
        pos = tuple(g.uniform(-0.3, 0.3, 3))
        a = 2 * np.pi * k / 23
        c2w = C.look_at(pos, tuple(np.asarray(pos) + np.array([np.cos(a), np.sin(a), 0.1])))
        views.append(Cameras(torch.from_numpy(c2w)[None], 50.0, 51.0, 31.6, 23.7, W, H))
    blocks = camera_blocks(views, torch.float64).cpu().numpy()
    pts = g.uniform(-1.5, 1.5, (20000, 3))
    rendered = (0.3 + 2.0 * g.random((23, H, W))).astype(np.float32)
    gt = np.where(g.random((23, H, W)) < 0.3, 0.0, 1.0).astype(np.float32)
    ro, ri = R.visibility_counts(pts, blocks, W, H, rendered, gt)
    for chunk in (1, 4, 16, 23, 50):
        obs, inv = visibility_counts(torch.from_numpy(pts).cuda(), views, torch.from_numpy(rendered).cuda(),
                                     torch.from_numpy(gt).cuda(), chunk=chunk)
        assert np.array_equal(obs.cpu().numpy(), ro) and np.array_equal(inv.cpu().numpy(), ri), chunk
    assert ro.max() > 3 and (ri > 0).any()
