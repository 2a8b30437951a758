"""Generates tests/golden/dn_depth_normals.npz by executing the REFERENCE's own scripts/depth_normal_consistency.py and
scripts/depth_to_normal.py, unmodified, on the capture folder of tests/depth_normals_scene.py.  Open3D, natsort and
nerfstudio are absent: stub modules stand in.  The stub PointCloud records the points each estimate_normals call receives
and computes the normals with oracle/normals_ref.py (Open3D's semantics restated, with this project's tie rule), so the
golden pins everything the scripts do around that call: sorting, depth loading, back-projection, orientation, the mono
decode, the angle, the mask and the bytes of every file written.

Runs: DepthNormalConsistency (omnidata, angle_treshold 20; dsine, 15, intrinsics in the frames; omnidata with
angle_treshold equal to an angle the oracle attains on frame_1, so the strict `>` of the mask is pinned), DepthToNormal.

Run only where /root/reference exists:   python tests/golden/make_golden_normals.py
"""
import importlib.util
import os
import sys
import tempfile
import types
from pathlib import Path

import numpy as np

OUT = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(OUT))
sys.path.insert(0, ROOT)
from dn_splatter_b200.depth_normals import c2w_of, load_depth, natural_key, read_mono  # noqa: E402
from dn_splatter_b200.depth_normals import load_transforms as natural_frames  # noqa: E402
from oracle import normals_ref as R  # noqa: E402
from tests import depth_normals_scene as D  # noqa: E402

SCRIPTS = "/root/reference/dn_splatter/scripts"
RUNS = {
    "omnidata": ("depth_normal_consistency.py", "DepthNormalConsistency", dict(normal_format="omnidata", angle_treshold=20.0),
                 dict(dsine=False)),
    "dsine": ("depth_normal_consistency.py", "DepthNormalConsistency", dict(normal_format="dsine", angle_treshold=15.0),
              dict(dsine=True, intrinsics_in_frames=True)),
    "depth_to_normal": ("depth_to_normal.py", "DepthToNormal", {}, dict(dsine=False)),
    "omnidata_tie": ("depth_normal_consistency.py", "DepthNormalConsistency", dict(normal_format="omnidata"), dict(dsine=False)),
}


def tie_threshold():
    """An angle that pixels of frame_1 attain exactly (the most frequent one above 20 degrees), from the oracle."""
    with tempfile.TemporaryDirectory() as tmp:
        name = D.build(tmp)
        frames, (fx, fy, cx, cy, w, h) = natural_frames(tmp, name)
        f = frames[0]
        depth = load_depth(os.path.join(tmp, f["depth_file_path"]))
        c2w = c2w_of(f)
        pts, _ = R.backproject(depth, fx, fy, cx, cy, w, h, c2w)
        n = R.orient(pts, R.estimate_normals(pts)[0], c2w[:3, 3])
        mono = read_mono(os.path.join(tmp, "normals_from_pretrain", "frame_1.png"), w, h)
        deg = R.consistency(n, mono, c2w, "omnidata", 20.0)[0]
    vals, counts = np.unique(deg[deg > 20], return_counts=True)
    return float(vals[np.argmax(counts)])


def stubs(record):
    class PointCloud:
        def __init__(self):
            self.points = None
            self.normals = None

        def estimate_normals(self, search_param):
            pts = np.asarray(self.points, np.float64)
            record.append(pts.copy())
            self.normals = R.estimate_normals(pts, search_param.knn)[0]

    o3d = types.ModuleType("open3d")
    o3d.geometry = types.SimpleNamespace(PointCloud=PointCloud, KDTreeSearchParamKNN=lambda knn: types.SimpleNamespace(knn=knn))
    o3d.utility = types.SimpleNamespace(Vector3dVector=lambda a: a)
    sys.modules["open3d"] = o3d
    sys.modules["natsort"] = types.SimpleNamespace(natsorted=lambda xs, key: sorted(xs, key=lambda x: natural_key(key(x))))
    import json

    def load_from_json(p):
        with open(p, encoding="UTF-8") as fh:
            return json.load(fh)

    io = types.SimpleNamespace(load_from_json=load_from_json)
    sys.modules["nerfstudio"] = types.SimpleNamespace(utils=types.SimpleNamespace(io=io))
    sys.modules["nerfstudio.utils"] = sys.modules["nerfstudio"].utils
    sys.modules["nerfstudio.utils.io"] = io


def main():
    record = []
    stubs(record)
    depth, normals, transforms = D.scene_arrays()
    z = {"depth_mm": depth, "world_normals": normals, "transforms": transforms}
    z["omnidata_tie/threshold"] = np.float64(tie_threshold())
    RUNS["omnidata_tie"][2]["angle_treshold"] = float(z["omnidata_tie/threshold"])
    for run, (script, cls, kw, folder) in RUNS.items():
        spec = importlib.util.spec_from_file_location(f"ref_{run}", os.path.join(SCRIPTS, script))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        with tempfile.TemporaryDirectory() as tmp:
            name = D.build(tmp, **folder)
            record.clear()
            getattr(mod, cls)(data_dir=Path(tmp), transforms_name=name, **kw).main()
            if run != "omnidata_tie":  # the same folder and poses as "omnidata": the same points
                z[f"{run}/points"] = np.stack(record)
            files = D.list_outputs(tmp)
            z[f"{run}/files"] = np.array(list(files))
            for f, b in files.items():
                z[f"{run}/file/{f}"] = np.frombuffer(b, np.uint8)
            print(run, len(record), list(files))
    np.savez_compressed(os.path.join(OUT, "dn_depth_normals.npz"), **z)


if __name__ == "__main__":
    main()
