"""Generates tests/golden/dn_mesh_eval.npz by executing the REFERENCE's own mesh evaluation
(/root/reference/dn_splatter/eval/eval_mesh_vis_cull.py and dn_splatter/metrics.py), unmodified, with its absent imports
(open3d, trimesh, pyrender, matplotlib, torchmetrics) stubbed:

- get_grid_culling_pattern / cull_from_one_pose (:68-149) on random points, with and without the occlusion and
  missing-depth tests;
- cull_mesh (:176-266), replica branch, on a temporary dataset directory (transforms json + 16-bit depth PNGs).  Its
  render_depth_maps_doublesided calls .cuda() and pyrender, so it is replaced by the oracle's ray cast; trimesh.Trimesh and
  trimesh.remesh.subdivide_to_size are replaced by stand-ins (the subdivision is the oracle's);
- compute_metrics (:333-397, with distance_p2p and get_threshold_percentage) on stand-in meshes whose `sample` returns
  recorded samples;
- metrics.calculate_accuracy / calculate_completeness.

tests/test_mesh_eval_cpu.py checks oracle/mesh_eval_ref.py against the file.

Run only where /root/reference exists:   python tests/golden/make_golden_mesh_eval.py
"""
import importlib.util
import json
import os
import sys
import tempfile
import types

import numpy as np

OUT = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(OUT))
sys.path.insert(0, ROOT)
from oracle import mesh_eval_ref as R  # noqa: E402

REF = "/root/reference/dn_splatter"


class StandInMesh:
    """trimesh.Trimesh as cull_mesh / compute_metrics use it."""

    def __init__(self, vertices, faces, process=False, samples=None):
        self.vertices = np.asarray(vertices, np.float64)
        self.faces = np.asarray(faces, np.int64)
        self._samples = samples

    def remove_unreferenced_vertices(self):
        self.vertices, self.faces = R.remove_unreferenced(self.vertices, self.faces)

    @property
    def area(self):
        return float(R.triangle_areas(self.vertices, self.faces).sum())

    @property
    def face_normals(self):
        return R.face_normals(self.vertices, self.faces)

    def sample(self, count, return_index=False):
        pts, idx = self._samples
        assert count == pts.shape[0], (count, pts.shape)
        return (pts, idx) if return_index else pts


def install_stubs():
    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    class PointCloud:
        pass

    o3d = mod("open3d", geometry=types.SimpleNamespace(PointCloud=PointCloud, TriangleMesh=object),
              utility=types.SimpleNamespace(Vector3dVector=lambda x: np.asarray(x)))
    mod("open3d.core")
    remesh = types.SimpleNamespace(subdivide_to_size=lambda v, f, max_edge, max_iter: R.subdivide_to_size(v, f, max_edge, max_iter)[:2])
    mod("trimesh", Trimesh=StandInMesh, remesh=remesh)
    mod("pyrender")
    cm = types.SimpleNamespace(get_cmap=lambda name: (lambda x: np.zeros(np.shape(x) + (4,))))
    plt = types.SimpleNamespace(cm=cm)
    mpl = mod("matplotlib", pyplot=plt)
    mod("matplotlib.pyplot", cm=cm)
    mpl.pyplot = sys.modules["matplotlib.pyplot"]
    tm = mod("torchmetrics")
    mod("torchmetrics.image", PeakSignalNoiseRatio=object, StructuralSimilarityIndexMeasure=object)
    mod("torchmetrics.image.lpip", LearnedPerceptualImagePatchSimilarity=object)
    tm.image = sys.modules["torchmetrics.image"]
    return o3d


def load(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def look_at(pos, target, up=(0.0, 0.0, 1.0)):
    """OpenGL c2w [4,4]: camera looks down -z."""
    pos, target, up = (np.asarray(a, np.float64) for a in (pos, target, up))
    fwd = target - pos
    fwd /= np.linalg.norm(fwd)
    right = np.cross(fwd, up)
    right /= np.linalg.norm(right)
    cup = np.cross(right, fwd)
    m = np.eye(4)
    m[:3, 0], m[:3, 1], m[:3, 2], m[:3, 3] = right, cup, -fwd, pos
    return m


def box_mesh(lo, hi, inward=True):
    """The 12-triangle box, faces wound towards the inside when inward."""
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    v = np.array([[lo[0] if i & 1 == 0 else hi[0], lo[1] if i & 2 == 0 else hi[1], lo[2] if i & 4 == 0 else hi[2]]
                  for i in range(8)])
    f = np.array([[0, 2, 1], [1, 2, 3], [4, 5, 6], [5, 7, 6], [0, 1, 4], [1, 5, 4], [2, 6, 3], [3, 6, 7],
                  [0, 4, 2], [2, 4, 6], [1, 3, 5], [3, 7, 5]])
    return v, (f if inward else f[:, [0, 2, 1]])


def sample_mesh(verts, faces, count, rng):
    """Area-weighted samples with parallelogram folding (the recorded samples of the stand-in meshes)."""
    a = R.triangle_areas(verts, faces)
    cum = np.cumsum(a)
    idx = np.searchsorted(cum, rng.random(count) * cum[-1])
    t = np.asarray(verts)[np.asarray(faces)[idx]]
    r = rng.random((count, 2, 1))
    fold = r.sum(axis=1).reshape(-1) > 1.0
    r[fold] -= 1.0
    r = np.abs(r)
    return (t[:, 0] + ((t[:, 1:] - t[:, :1]) * r).sum(axis=1)), idx


def main():
    install_stubs()
    E = load(os.path.join(REF, "eval", "eval_mesh_vis_cull.py"), "ref_eval_mesh_vis_cull")
    M = load(os.path.join(REF, "metrics.py"), "ref_metrics")
    rng = np.random.default_rng(7)
    z = {}

    # --- get_grid_culling_pattern / cull_from_one_pose
    W, H, n_views = 37, 29, 6
    K = np.array([[30.0, 0, 18.3], [0, 31.0, 14.1], [0, 0, 1]]).astype(np.float32)
    poses = [look_at(rng.normal(size=3) * 0.3 + np.array([0, 0, 0.2 * k]), rng.normal(size=3) * 0.2 + np.array([0, 0, -3.0]),
                     up=(0.0, 1.0, 0.0)) for k in range(n_views)]
    pts = np.concatenate([rng.normal(size=(3000, 3)) * np.array([1.5, 1.2, 1.0]) + np.array([0, 0, -3.0]),
                          rng.normal(size=(200, 3)) + np.array([0, 0, 2.0])])  # the last ones mostly behind the cameras
    rendered = [(2.0 + 2.0 * rng.random((H, W))).astype(np.float32) for _ in range(n_views)]
    gt = [np.where(rng.random((H, W)) < 0.3, 0.0, 1.0 + rng.random((H, W))).astype(np.float32) for _ in range(n_views)]
    z["vis_points"], z["vis_poses"], z["vis_K"] = pts, np.stack(poses), K
    z["vis_rendered"], z["vis_gt"], z["vis_hw"] = np.stack(rendered), np.stack(gt), np.array([H, W])
    for tag, rmd, ro in (("both", True, True), ("noocc", True, False), ("nomiss", False, True)):
        obs, inv = E.get_grid_culling_pattern(pts, poses, H, W, K, rendered_depth_list=rendered, depth_gt_list=gt,
                                              remove_missing_depth=rmd, remove_occlusion=ro)
        z[f"vis_{tag}_obs"], z[f"vis_{tag}_invalid"] = obs, inv
    o1, i1 = E.cull_from_one_pose(pts, poses[0], H, W, K, rendered_depth=rendered[0], depth_gt=gt[0])
    z["vis_one_obs"], z["vis_one_invalid"] = o1, i1

    # --- cull_mesh, replica branch: a room (inward box) with an object, 24 views, depth holes
    W2, H2, n2 = 48, 36, 24
    fl, cx2, cy2 = 22.0, 24.0, 18.0
    bv, bf = box_mesh((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0))
    ov, of = box_mesh((-0.2, -0.3, -0.2), (0.2, 0.1, 0.2), inward=False)
    extra = np.array([[5.0, 5.0, 5.0]])  # an unreferenced vertex
    mv = np.concatenate([bv, ov + np.array([0.3, 0.2, -0.5]), extra])
    mf = np.concatenate([bf, of + 8])
    c2w_gl = [look_at(rng.uniform(-0.3, 0.3, 3), rng.uniform(-0.3, 0.3, 3) + np.array([np.cos(a), np.sin(a), 0.1]) * 2)
              for a in np.linspace(0, 2 * np.pi, n2, endpoint=False)]
    with tempfile.TemporaryDirectory() as d:
        frames = []
        os.makedirs(os.path.join(d, "depth"))
        from PIL import Image

        Kf = np.array([[fl, 0, cx2], [0, fl, cy2], [0, 0, 1]], np.float32)
        for k, m in enumerate(c2w_gl):
            cam = R.camera_block(m.astype(np.float32).astype(np.float64), fl, fl, cx2, cy2)
            dep = R.ray_cast_depth(bv, bf, cam, W2, H2)
            png = np.round(dep * 6553.5).astype(np.uint16)
            png[: H2 // 3, : W2 // 2] = 0  # missing sensor depth
            Image.fromarray(png).save(os.path.join(d, "depth", f"{k:04d}.png"))
            stored = m.copy()
            stored[0:3, 1:3] *= -1  # replica stores OpenCV c2w; the branch flips it back
            frames.append({"depth_file_path": f"depth/{k:04d}.png", "transform_matrix": stored[:3].tolist() + [[0, 0, 0, 1]]})
        tf = os.path.join(d, "transforms.json")
        with open(tf, "w") as fh:
            json.dump({"h": H2, "w": W2, "fl_x": fl, "fl_y": fl, "cx": cx2, "cy": cy2, "frames": frames}, fh)
        z["cull_depth_png"] = np.stack([np.asarray(Image.open(os.path.join(d, "depth", f"{k:04d}.png"))) for k in range(n2)])
        z["cull_transforms"] = np.frombuffer(open(tf, "rb").read(), np.uint8)

        rendered_by_ref = []

        def render_stand_in(mesh, poses, H_, W_, K_, far=10.0):
            out = []
            for p in poses:
                cam = R.camera_block(np.asarray(p, np.float64), float(K_[0, 0]), float(K_[1, 1]), float(K_[0, 2]), float(K_[1, 2]))
                out.append(R.ray_cast_depth(mesh.vertices, mesh.faces, cam, W_, H_, far=far).astype(np.float32))
            rendered_by_ref.append(np.stack(out))
            return out

        spy = {}
        real_pattern = E.get_grid_culling_pattern

        def pattern_spy(points, poses, *a, **kw):
            obs, inv = real_pattern(points, poses, *a, **kw)
            spy["points"], spy["obs"], spy["invalid"] = np.array(points), obs, inv
            spy["poses"] = np.stack(poses)
            return obs, inv

        E.render_depth_maps_doublesided = render_stand_in
        E.get_grid_culling_pattern = pattern_spy
        from pathlib import Path

        for tag, me in (("room", StandInMesh(mv, mf)),):
            out = E.cull_mesh(Path(d), "replica", me, tf, max_edge=0.25)
            z[f"cull_{tag}_in_vertices"], z[f"cull_{tag}_in_faces"] = mv, mf
            z[f"cull_{tag}_vertices"], z[f"cull_{tag}_faces"] = out.vertices, out.faces
            z[f"cull_{tag}_sub_points"], z[f"cull_{tag}_obs"], z[f"cull_{tag}_invalid"] = spy["points"], spy["obs"], spy["invalid"]
            z[f"cull_{tag}_poses"], z[f"cull_{tag}_rendered"] = spy["poses"], rendered_by_ref[-1]
        z["cull_params"] = np.array([W2, H2, fl, fl, cx2, cy2, 0.25])
        E.get_grid_culling_pattern = real_pattern

    # --- compute_metrics on recorded samples
    gv, gf = box_mesh((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0))
    gv = gv * 0.12
    for tag, shift in (("near", 0.02), ("mixed", 0.05), ("far", 0.5)):
        pv = (gv * (1.0 + shift / 0.12) if shift < 0.1 else gv + shift) + rng.normal(size=gv.shape) * 0.004
        gm = StandInMesh(gv, gf)
        pm = StandInMesh(pv, gf)
        ns_p, ns_g = int(pm.area * 1e4), int(gm.area * 1e4)
        sp, ip = sample_mesh(pv, gf, ns_p, rng)
        sg, ig = sample_mesh(gv, gf, ns_g, rng)
        pm._samples, gm._samples = (sp, ip), (sg, ig)
        with np.errstate(invalid="ignore", divide="ignore"):
            rst = E.compute_metrics(pm, gm)
        z[f"met_{tag}_pred_vertices"], z[f"met_{tag}_gt_vertices"], z[f"met_{tag}_faces"] = pv, gv, gf
        z[f"met_{tag}_pred_samples"], z[f"met_{tag}_pred_idx"] = sp, ip
        z[f"met_{tag}_gt_samples"], z[f"met_{tag}_gt_idx"] = sg, ig
        z[f"met_{tag}_values"] = np.array([float(rst[k]) for k in ("Acc", "Comp", "C-L1", "NC", "F-score")])
        print(tag, {k: float(v) for k, v in rst.items()})

    # --- PDMetrics
    a = rng.normal(size=(4000, 3)).astype(np.float32)
    b = (a[:3000] + 0.04 * rng.normal(size=(3000, 3))).astype(np.float32)
    z["pd_pred"], z["pd_gt"] = b, a
    z["pd_acc"] = np.array([M.calculate_accuracy(b, a), M.calculate_accuracy(b, a, percentile=50)])
    z["pd_comp"] = np.array([M.calculate_completeness(b, a), M.calculate_completeness(b, a, threshold=0.02)])
    np.savez_compressed(os.path.join(OUT, "dn_mesh_eval.npz"), **z)
    print("culled faces", z["cull_room_faces"].shape[0], "of", mf.shape[0], "-> sub", z["cull_room_obs"].shape[0], "vertices")


if __name__ == "__main__":
    main()
