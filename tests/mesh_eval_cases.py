"""Meshes and fp32 camera blocks for the per-pixel tests of dnr_mesh_depth and dnr_mesh_visibility
(tests/test_gpu_mesh_eval_kernels.py runs them on the device, tests/test_mesh_eval_ref_cpu.py checks the oracle's rule on
them).  Every case is built from constants or a seed.  A depth case is a dict: name, verts [n,3] float32, faces [F,3]
int32, cams [V,16] float32 (the block the kernel reads), W, H, near, far, and `reach`: the decisions of
oracle.mesh_eval_ref.DECISIONS (or box areas, "area:<n>", and box shapes "1xN" / "Nx1") the case exists to reach."""
from __future__ import annotations

import math

import numpy as np

from oracle import mesh_eval_ref as R

NEAR, FAR = 0.01, 10.0
EYE = np.eye(4)[:3]  # OpenGL camera at the origin looking down -z: camera (X, Y, Z) = (x, -y, -z), exactly
NEAR32 = float(np.float32(NEAR))  # the near plane the kernel compares against


def block32(c2w, fx, fy, cx, cy) -> np.ndarray:
    """The fp32 camera block of mesh_eval.camera_blocks(..., torch.float32): fp64 inverse, rounded once."""
    return R.camera_block(np.asarray(c2w, np.float64), fx, fy, cx, cy).astype(np.float32)


def look_at(pos, target, up=(0.0, 0.0, 1.0)) -> np.ndarray:
    """synthetic.look_at_c2w in float32 torch, as the GPU tests' Cameras hold it."""
    import torch

    from dn_splatter_b200.synthetic import look_at_c2w

    return look_at_c2w(torch.tensor(pos, dtype=torch.float32), torch.tensor(target, dtype=torch.float32),
                       torch.tensor(up, dtype=torch.float32)).numpy()


def _rz(a):
    c, s = math.cos(a), math.sin(a)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


# ---- meshes -------------------------------------------------------------------------------------------------------
def box(lo=(-1.0, -1.0, -1.0), hi=(1.0, 1.0, 1.0)):
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    v = np.array([[hi[0] if i & 1 else lo[0], hi[1] if i & 2 else lo[1], hi[2] if i & 4 else lo[2]] for i in range(8)])
    f = np.array([[0, 2, 1], [1, 2, 3], [4, 5, 6], [5, 7, 6], [0, 1, 4], [1, 5, 4], [2, 6, 3], [3, 6, 7],
                  [0, 4, 2], [2, 4, 6], [1, 3, 5], [3, 7, 5]])
    return v, f


def sphere(n=16, r=0.6, c=(0.0, 0.0, 0.0)):
    th, ph = np.meshgrid(np.linspace(0, np.pi, n + 1), np.linspace(0, 2 * np.pi, 2 * n + 1), indexing="ij")
    v = np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], -1).reshape(-1, 3) * r + np.asarray(c)
    idx = np.arange(v.shape[0]).reshape(n + 1, 2 * n + 1)
    a, b, cc, d = idx[:-1, :-1], idx[:-1, 1:], idx[1:, :-1], idx[1:, 1:]
    return v, np.concatenate([np.stack([a, cc, b], -1).reshape(-1, 3), np.stack([b, cc, d], -1).reshape(-1, 3)])


def odd_triangles():
    """Seen from an identity OpenGL camera (looking down -z): triangles straddling the near plane, beyond far, behind the
    camera, back-facing, full-screen, sub-pixel and degenerate."""
    tris = [
        [[-0.5, -0.4, -0.005], [0.6, -0.3, -3.0], [0.1, 0.7, -2.5]],      # straddles near = 0.01
        [[-0.3, -0.3, -12.0], [0.3, -0.3, -12.0], [0.0, 0.3, -12.0]],     # beyond far
        [[-0.3, -0.3, -9.0], [0.3, -0.3, -11.0], [0.0, 0.3, -9.5]],       # straddles far
        [[-0.5, -0.5, 2.0], [0.5, -0.5, 2.0], [0.0, 0.5, 2.0]],           # behind the camera
        [[0.2, 0.1, -1.5], [0.1, 0.4, -1.5], [0.4, 0.3, -1.6]],           # back-facing winding
        [[-40.0, -40.0, -6.0], [40.0, -40.0, -6.5], [0.0, 60.0, -6.2]],   # full screen
        [[0.0101, 0.0102, -1.0], [0.0104, 0.0101, -1.0], [0.0102, 0.0105, -1.0]],  # sub-pixel
        [[0.1, 0.1, -2.0], [0.2, 0.2, -2.0], [0.3, 0.3, -2.0]],           # degenerate (collinear)
        [[-0.2, 0.0, -1.0], [-0.2, 0.0, -1.0], [-0.1, 0.2, -1.0]],        # degenerate (repeated vertex)
        [[-0.9, -0.9, -3.0], [-0.1, -0.8, -0.5], [-0.5, 0.2, 3.0]],       # reaches behind the camera
    ]
    v = np.asarray(tris, np.float64).reshape(-1, 3)
    return v, np.arange(v.shape[0]).reshape(-1, 3)


def edge_grid(W, H, f, cx=None, cy=None, z=2.0):
    """A triangulated grid at depth z whose vertices project onto pixel centres (camera space, identity camera), so its
    edges pass through them."""
    cx = W / 2 if cx is None else cx
    cy = H / 2 if cy is None else cy
    xs = ((np.arange(2, W - 2, 3) + 0.5 - cx) / f) * z
    ys = ((np.arange(2, H - 2, 3) + 0.5 - cy) / f) * z
    X, Y = np.meshgrid(xs, ys)
    v = np.stack([X.reshape(-1), -Y.reshape(-1), np.full(X.size, -z)], 1)  # image y points down, world y up
    nx = xs.shape[0]
    idx = np.arange(v.shape[0]).reshape(ys.shape[0], nx)
    a, b, c, d = idx[:-1, :-1], idx[:-1, 1:], idx[1:, :-1], idx[1:, 1:]
    fl = np.concatenate([np.stack([a, c, b], -1).reshape(-1, 3), np.stack([b, c, d], -1).reshape(-1, 3)])
    return v, fl


def legacy_scenes(W, H):
    """The four scenes of test_gpu_mesh_eval.py: (name, verts, faces, c2w [3,4] float32, fx, fy, cx, cy)."""
    out = [("box_inside", *box(), look_at((0.1, -0.2, 0.05), (1.0, 0.3, 0.2)), 0.6 * W, 0.6 * W, W / 2, H / 2),
           ("sphere", *sphere(), look_at((0.3, -2.0, 0.4), (0.0, 0.0, 0.0)), 1.1 * W, 1.0 * W, W / 2 - 1.3, H / 2 + 0.7),
           ("odd", *odd_triangles(), EYE.astype(np.float32), 0.8 * W, 0.8 * W, W / 2, H / 2)]
    gv, gf = edge_grid(W, H, 0.7 * W)
    out.append(("edges", gv, gf, EYE.astype(np.float32), 0.7 * W, 0.7 * W, W / 2, H / 2))
    return out


def interior_hits(verts, faces, cam32, W, H, near=NEAR, far=FAR):
    """[H,W] bool: pixels the independent ray cast (fp64 Moller-Trumbore on the same fp32 inputs) hits, together with
    their 4 neighbours, off the frame border.  On a mesh without gaps every such pixel must be hit; a pixel centre on a
    shared edge that both faces miss shows up here as a hole."""
    rc = R.ray_cast_depth(np.asarray(verts, np.float32).astype(np.float64), faces, np.asarray(cam32, np.float32).astype(np.float64),
                          W, H, near, far)
    hit = rc > 0
    inner = hit.copy()
    inner[1:-1, 1:-1] &= hit[:-2, 1:-1] & hit[2:, 1:-1] & hit[1:-1, :-2] & hit[1:-1, 2:]
    inner[[0, -1], :] = False
    inner[:, [0, -1]] = False
    return inner


def full_hd_scene():
    v1, f1 = odd_triangles()
    v2, f2 = box((-3.0, -3.0, -8.0), (3.0, 3.0, 1.0))
    return np.concatenate([v1, v2]), np.concatenate([f1, f2 + v1.shape[0]]), EYE.astype(np.float32), 1100.0, 1090.0, 961.3, 538.9


def _case(name, v, f, cams, W, H, reach=(), near=NEAR, far=FAR, watertight=False):
    """watertight: the mesh has no gaps in view, so every pixel of `interior_hits` must be hit."""
    return {"name": name, "verts": np.asarray(v, np.float32).reshape(-1, 3), "faces": np.asarray(f, np.int32).reshape(-1, 3),
            "cams": np.asarray(cams, np.float32).reshape(-1, 16), "W": W, "H": H, "near": near, "far": far,
            "reach": tuple(reach), "watertight": watertight}


def _px_tri(u0, u1, v0, v1, z, fx, fy, cx, cy):
    """World corners (identity camera) of a right triangle whose projection spans pixel coordinates [u0, u1] x [v0, v1]."""
    pts = [(u0, v0), (u1, v0), (u0, v1)]
    return [[(u - cx) * z / fx, -(v - cy) * z / fy, -z] for u, v in pts]


# ---- depth cases ----------------------------------------------------------------------------------------------------
def item_boundary_case():
    """Triangles whose kernel boxes hold 255, 256, 257, 511 and 513 pixels (one pixel of margin each side: a projected
    span [a + 0.25, b + 0.75] gives b - a + 3 pixels), and boxes one pixel wide or tall, clamped at the frame's edges."""
    W, H, fx, fy, cx, cy = 320, 300, 280.0, 280.0, 160.0, 150.0
    tris = []
    spans = [(15, 17), (16, 16), (7, 73), (19, 27), (11, 47)]  # 255, 256, 511, 513, 517
    x = 4
    for k, (w, h) in enumerate(spans):
        tris.append(_px_tri(x + 0.25, x + w - 3 + 0.75, 4 + 0.25, 4 + h - 3 + 0.75, 1.0 + 0.1 * k, fx, fy, cx, cy))
        x += w + 4
    tris.append(_px_tri(-9.0, 0.3, 100.25, 354.0, 1.5, fx, fy, cx, cy))        # 1 x 200 at the left edge
    tris.append(_px_tri(W - 0.3, W + 9.0, 40.25, 298.0, 1.6, fx, fy, cx, cy))  # 1 x N at the right edge
    tris.append(_px_tri(40.25, 400.0, -9.0, 0.3, 1.7, fx, fy, cx, cy))         # N x 1 at the top, 281 px
    tris.append(_px_tri(60.25, 314.75, H - 0.3, H + 9.0, 1.8, fx, fy, cx, cy))  # 257 x 1 at the bottom
    v = np.asarray(tris, np.float64).reshape(-1, 3)
    reach = ("area:255", "area:256", "area:257", "area:511", "area:513", "1xN", "Nx1", "hit")
    return _case("item_boundaries", v, np.arange(v.shape[0]).reshape(-1, 3), block32(EYE, fx, fy, cx, cy), W, H, reach)


def full_wall_case():
    """1200 x 680: a full-frame wall (two faces, thousands of items each) behind a slanted full-frame plane."""
    W, H, fx, fy, cx, cy = 1200, 680, 600.0, 600.0, 600.3, 339.8
    v = np.array([[-50, -50, -5.0], [50, -50, -5.0], [50, 50, -5.0], [-50, 50, -5.0],
                  [-30, -30, -3.0], [30, -30, -7.0], [30, 30, -7.0], [-30, 30, -3.0]])
    f = np.array([[0, 1, 2], [0, 2, 3], [4, 5, 6], [4, 6, 7]])
    return _case("full_wall", v, f, block32(EYE, fx, fy, cx, cy), W, H, ("hit", "area:816000"))


def near_far_case():
    """Faces in the planes z = near (the fp32 near the kernel compares with) and z = far with dyadic corners, so z is
    exactly near / far; corners exactly on those planes; faces straddling either plane; faces reaching behind the
    camera whose clipped polygon leaves the frame."""
    W, H, fx, fy, cx, cy = 96, 64, 64.0, 64.0, 48.0, 32.0
    s = 2.0 ** -9
    n = NEAR32
    tris = [
        [[-s, -s, -n], [s, -s, -n], [-s, s, -n]],                 # in the near plane: z == near exactly
        [[-4.0, -2.0, -10.0], [4.0, -2.0, -10.0], [4.0, 2.0, -10.0]],  # in the far plane: z == far exactly
        [[0.0, 0.0, -n], [0.3, -0.1, -2.0], [0.1, 0.3, -2.5]],    # one corner on the near plane
        [[0.0, 0.0, -10.0], [-1.0, -0.5, -9.0], [-1.2, 0.4, -9.5]],  # one corner on the far plane
        [[-0.02, -0.02, -0.004], [0.3, -0.2, -0.5], [-0.2, 0.25, -0.6]],  # straddles near
        [[-1.0, -1.0, -9.0], [1.0, -1.0, -11.0], [0.0, 1.5, -10.5]],  # straddles far
        [[-0.5, -0.5, 1.0], [0.5, -0.4, -0.5], [0.2, 0.6, -0.3]],    # behind the camera, clipped polygon leaves the frame
        [[-3.0, 0.5, 2.0], [-0.3, -0.2, -1.2], [-0.4, 0.1, -0.02]],  # behind the camera on another side
    ]
    v = np.asarray(tris, np.float64).reshape(-1, 3)
    return _case("near_far", v, np.arange(v.shape[0]).reshape(-1, 3), block32(EYE, fx, fy, cx, cy), W, H,
                 ("hit", "near", "near_equal", "far", "far_equal"))


def bad_faces_case():
    """Faces with index -1 and n_vertices, degenerate faces (repeated index, repeated point, collinear), slivers, and
    edge-on faces whose plane passes through the camera centre, on a row whose rays lie in that plane (cy = j + 0.5)."""
    W, H, fx, fy, cx, cy = 80, 60, 64.0, 64.0, 40.0, 30.5
    v = np.array([
        [-0.3, -0.2, -1.0], [0.3, -0.25, -1.1], [0.0, 0.3, -0.9],    # 0-2 a plain face
        [0.0, 0.0, -1.0], [0.0, 0.0, -2.0], [0.3, 0.0, -1.5],        # 3-5 edge-on: the plane y = 0 holds the camera
        [-0.2, -0.1, -1.0], [0.2, 0.1, -2.0], [0.1, 0.05, -1.5],     # 6-8 edge-on, tilted: plane through the origin
        [-0.1, -0.1, -1.3], [0.1, 0.1, -1.3], [0.3, 0.3, -1.3],      # 9-11 collinear
        [-0.4, 0.2, -1.2], [0.4, 0.2001, -1.2], [0.4, 0.2, -1.2],    # 12-14 a sliver across the frame
        [-0.35, -0.3, -0.8], [0.35, -0.3, -0.8],                     # 15-16
        [0.0, -0.3, -0.8],                                           # 17 repeated point of 15-16's line
    ])
    nv = v.shape[0]
    f = np.array([[0, 1, 2], [3, 4, 5], [6, 7, 8], [9, 10, 11], [12, 13, 14], [15, 16, 17], [0, 0, 1], [0, 1, -1],
                  [nv, 1, 2], [2, nv, 0], [-1, -1, -1], [5, 4, 3]])
    return _case("bad_faces", v, f, block32(EYE, fx, fy, cx, cy), W, H, ("hit", "den_zero", "edge_zero"))


def duplicates_case():
    """Duplicate faces with reversed winding (and reversed index order), and coplanar overlapping faces: ties in the
    depth minimum."""
    W, H, fx, fy, cx, cy = 72, 56, 64.0, 64.0, 36.0, 28.0
    v = np.array([[-0.5, -0.4, -1.5], [0.5, -0.3, -1.7], [0.0, 0.5, -1.2],
                  [-0.3, -0.3, -1.0], [0.3, -0.3, -1.0], [0.3, 0.3, -1.0], [-0.3, 0.3, -1.0],
                  [-0.45, -0.35, -1.0], [0.2, -0.35, -1.0], [0.0, 0.35, -1.0]])
    f = np.array([[0, 1, 2], [2, 1, 0], [1, 0, 2], [3, 4, 5], [3, 5, 6], [7, 8, 9], [5, 4, 3]])
    return _case("duplicates", v, f, block32(EYE, fx, fy, cx, cy), W, H, ("hit", "tie", "edge_zero"))


def rotated_grid_cases():
    """The edge grid seen through cameras rotated about the optical axis, with non-integer cx, cy: by 90 degrees (the
    block stays exact, so grid edges pass exactly through pixel centres) and by 0.3 rad."""
    W, H, f = 96, 96, 64.0
    cx, cy = W / 2 + 0.25, H / 2 - 0.375
    out = []
    for name, a in (("grid_rot90", math.pi / 2), ("grid_rot0.3", 0.3)):
        v, fl = edge_grid(W, H, f, cx, cy)
        Rz = np.round(_rz(a), 15) if a == math.pi / 2 else _rz(a)
        Rz[np.abs(Rz) < 1e-12] = 0.0
        c2w = np.concatenate([Rz, np.zeros((3, 1))], 1)
        wv = np.asarray(v, np.float64) @ Rz.T  # world = R @ camera-frame grid, so the rotated camera sees the grid
        out.append(_case(name, wv, fl, block32(c2w, f, f, cx, cy), W, H, ("hit", "edge_zero") if a == math.pi / 2 else ("hit",),
                         watertight=True))
    return out


def closed_inside_cases():
    """Closed subdivided meshes seen from inside: a box room and a sphere (whose pole fans hold zero-area faces)."""
    bv, bf = box((-1.5, -1.0, -1.2), (1.5, 1.0, 1.3))
    sv, sf, _ = R.subdivide_to_size(bv, bf, 0.4)
    W, H = 128, 96
    cams = [block32(look_at((0.1, -0.2, 0.05), (1.0, 0.3, 0.2)), 70.0, 70.0, 64.3, 47.6),
            block32(look_at((-1.2, 0.7, 1.0), (1.0, -0.8, -1.0)), 50.0, 55.0, 63.0, 49.1)]
    pv, pf = sphere(24, 0.8, (0.05, -0.02, 0.1))
    return [_case("closed_box", sv, sf, cams[0], W, H, ("hit",)), _case("closed_box_corner", sv, sf, cams[1], W, H, ("hit",)),
            _case("closed_sphere", pv, pf, block32(look_at((0.1, 0.0, 0.2), (0.5, 0.7, -0.3)), 80.0, 80.0, 64.0, 48.0), W, H,
                  ("hit",))]


def depth_cases():
    return [item_boundary_case(), full_wall_case(), near_far_case(), bad_faces_case(), duplicates_case(),
            *rotated_grid_cases(), *closed_inside_cases()]


def scene_mesh(n_sphere=24):
    """A 3 x 2.4 x 2.5 room (box subdivided to 0.3) around a sphere and a small box: the geometry of the many-view case."""
    bv, bf = box((-1.5, -1.2, -1.0), (1.5, 1.2, 1.5))
    rv, rf, _ = R.subdivide_to_size(bv, bf, 0.3)
    sv, sf = sphere(n_sphere, 0.5, (0.4, 0.2, 0.0))
    ov, of = box((-0.9, -0.6, -0.8), (-0.5, -0.2, -0.3))
    v = np.concatenate([rv, sv, ov])
    f = np.concatenate([rf, sf + rv.shape[0], of + rv.shape[0] + sv.shape[0]])
    return v, f


def ring_blocks(n, W, H, seed=0, radius=0.9):
    """n distinct views from inside the scene room: positions, headings, focal lengths and principal points all vary."""
    g = np.random.default_rng(seed)
    out = []
    for k in range(n):
        a = 2 * np.pi * k / n
        pos = (radius * math.cos(a) * g.uniform(0.2, 1.0), radius * math.sin(a) * g.uniform(0.2, 1.0), g.uniform(-0.5, 0.8))
        tgt = np.asarray(pos) + np.array([math.cos(a + 2.0), math.sin(a + 2.0), g.uniform(-0.6, 0.6)])
        f = float(g.uniform(0.5, 1.3) * W)
        out.append(block32(look_at(pos, tuple(tgt)), f, f * g.uniform(0.95, 1.05), W / 2 + g.uniform(-3, 3), H / 2 + g.uniform(-3, 3)))
    return np.stack(out)


def many_views_case(n=128, W=48, H=32):
    v, f = scene_mesh()
    return _case(f"many_views_{n}", v, f, ring_blocks(n, W, H, seed=5), W, H, ("hit",))


# ---- production: the eval script's workload -------------------------------------------------------------------------
PROD_W, PROD_H, PROD_VIEWS = 1200, 680, 20


def production_mesh():
    """A 6 x 4 x 2.6 box room subdivided to 0.05 (7-8 rounds) around a 128-ring sphere: about 6.5e5 faces."""
    bv, bf = box((-3.0, -2.0, -1.0), (3.0, 2.0, 1.6))
    rv, rf, _ = R.subdivide_to_size(bv, bf, 0.05)
    sv, sf = sphere(128, 0.6, (1.0, 0.5, 0.0))
    return np.concatenate([rv, sv]), np.concatenate([rf, sf + rv.shape[0]])


def production_poses():
    """Replica-like views from inside the room: c2w [3,4] float32 per view; fx = fy = 600, cx = 599.5, cy = 339.5."""
    g = np.random.default_rng(11)
    out = []
    for k in range(PROD_VIEWS):
        a = 2 * np.pi * k / PROD_VIEWS
        pos = (g.uniform(-2.2, 2.2), g.uniform(-1.4, 1.4), g.uniform(-0.5, 1.2))
        tgt = np.asarray(pos) + np.array([math.cos(a), math.sin(a), g.uniform(-0.5, 0.5)])
        out.append(look_at(pos, tuple(tgt)))
    return out


PROD_INTRINSICS = (600.0, 600.0, 599.5, 339.5)


def production_blocks():
    return np.stack([block32(c2w, *PROD_INTRINSICS) for c2w in production_poses()])


def stratified_pixels(W, H, boxes, counts, rng, random_share=0.01, n_lines=8):
    """Flat pixel indices: every pixel of the border rows and columns, the pixels on both sides of every work-item
    boundary of the kernel's boxes, the full row and column through n_lines of those boundaries, and random_share of
    the frame at random."""
    sel = [np.arange(W), (H - 1) * W + np.arange(W), np.arange(H) * W, np.arange(H) * W + W - 1]
    multi = np.nonzero(counts > 1)[0]
    bnd = []
    if multi.size:
        rep = counts[multi] - 1
        f = np.repeat(multi, rep)
        k = np.arange(rep.sum()) - np.repeat(np.cumsum(rep) - rep, rep) + 1
        b = boxes[f]
        bw = b[:, 1] - b[:, 0] + 1
        for p in (k * R.PIX_PER_ITEM - 1, k * R.PIX_PER_ITEM):
            bnd.append((b[:, 2] + p // bw) * W + b[:, 0] + p % bw)
        bnd = np.concatenate(bnd)
        sel.append(bnd)
        for p in rng.choice(bnd, size=min(n_lines, bnd.size), replace=False):
            sel += [(p // W) * W + np.arange(W), np.arange(H) * W + p % W]
    sel.append(rng.choice(W * H, size=int(random_share * W * H), replace=False))
    return np.unique(np.concatenate(sel))


# ---- visibility cases -----------------------------------------------------------------------------------------------
VIS_W, VIS_H = 64, 48


def visibility_case(seed=0):
    """(points [n,3] f64, fp64 camera blocks [V,16], rendered [V,H,W] f32, gt [V,H,W] f32, eps, expectations): random
    points plus points projected exactly onto px = 0 / W - 1 and py = 0 / H - 1, points with Z + 1e-8 around 0, NaN
    points, points with pz == rendered + eps in fp32, and zero rendered depth under some points.  View 0 has the
    identity rotation, so camera coordinates are exact."""
    W, H = VIS_W, VIS_H
    g = np.random.default_rng(seed)
    fx, fy, cx, cy = 64.0, 64.0, 32.0, 24.0
    blocks = [R.camera_block(EYE, fx, fy, cx, cy)]  # E = diag(1, -1, -1): (X, Y, Z) = (x, -y, -z)
    for k in range(36):
        pos = tuple(g.uniform(-0.3, 0.3, 3))
        a = 2 * np.pi * k / 36
        blocks.append(R.camera_block(look_at(pos, tuple(np.asarray(pos) + np.array([math.cos(a), math.sin(a), 0.3 * math.sin(2 * a)]))),
                                     50.0, 52.0, 31.7, 23.4))
    blocks = np.stack(blocks)
    eps = 0.02
    pts = [g.uniform(-1.5, 1.5, (6000, 3))]

    def world(X, Y, Z):  # view 0's camera coordinates -> world
        return np.stack([X, -Y, -Z], 1)

    # px exactly 0 / W - 1, py exactly 0 / H - 1 (and one ulp either side), found by nudging X / Y
    Z = g.uniform(0.5, 3.0, 400)
    pz = Z + 1e-8
    edge = []
    for target, axis in ((0.0, 0), (W - 1.0, 0), (0.0, 1), (H - 1.0, 1)):
        f_, c_ = (fx, cx) if axis == 0 else (fy, cy)
        A = (target * pz - c_ * Z) / f_
        other = g.uniform(2, (W if axis else H) - 3, Z.size)
        B = ((other * pz) - ((cy if axis == 0 else cx) * Z)) / (fy if axis == 0 else fx)
        for step in range(-3, 4):
            A2 = A.copy()
            for _ in range(abs(step)):
                A2 = np.nextafter(A2, np.inf if step > 0 else -np.inf)
            edge.append(world(A2, B, Z) if axis == 0 else world(B, A2, Z))
    pts += edge
    # Z + 1e-8 around 0
    Zs = np.concatenate([np.array([-1e-8, -1e-8 * (1 + 1e-15), 0.0, 1e-300, -1e-300]),
                         np.nextafter(-1e-8, 0.0) * np.ones(1), np.nextafter(-1e-8, -1.0) * np.ones(1),
                         g.uniform(-3e-8, 3e-8, 40)])
    pts.append(world(np.zeros_like(Zs), np.zeros_like(Zs), Zs))
    pts.append(world(np.full_like(Zs, 1e-9), np.full_like(Zs, -2e-9), Zs))
    # NaN points
    pts.append(np.array([[np.nan, 0.0, -1.0], [0.0, np.nan, -1.0], [0.0, 0.0, np.nan], [np.nan] * 3]))
    # rendered maps; a block of zero rendered depth
    rendered = (0.3 + 2.5 * g.random((len(blocks), H, W))).astype(np.float32)
    rendered[:, 10:20, 5:15] = 0.0
    gt = np.where(g.random((len(blocks), H, W)) < 0.3, 0.0, 1.0).astype(np.float32)
    # pz == rendered + eps in fp32 at view 0: points at pixel centres (i + 0.5, j + 0.5) of view 0, at that depth
    ii, jj = g.integers(0, W, 300), g.integers(0, H, 300)
    lim = (rendered[0, jj, ii] + np.float32(eps)).astype(np.float64)
    Zt = lim - 1e-8
    for _ in range(3):  # land Z + 1e-8 exactly on the fp32 sum
        Zt = np.where(Zt + 1e-8 > lim, np.nextafter(Zt, -np.inf), np.where(Zt + 1e-8 < lim, np.nextafter(Zt, np.inf), Zt))
    Xt, Yt = (ii + 0.5 - cx) * Zt / fx, (jj + 0.5 - cy) * Zt / fy
    pts.append(world(Xt, Yt, Zt))
    # points under the zero-depth block of view 0, in front of and behind eps
    zz = np.array([0.005, 0.0199, 0.02, 0.0201, 0.5])
    pts.append(world((9.5 - cx) * zz / fx, (14.5 - cy) * zz / fy, zz))
    return np.concatenate(pts), blocks, rendered, gt, eps
