"""Generates tests/golden/dn_isooctree.npz by executing the REFERENCE's own mesh extractor
(/root/reference/dn_splatter/scripts/isooctree_dn.py), unmodified, on a small render folder (tests/isooctree_scene.py: a
box room with a block, 6 frames at 64x48, analytic depth and normals, both file layouts).  IsoOctree is absent, so a
stub module stands in for it: its buildMeshWithPointCloudHint records the hint cloud and calls the captured isoFunc on
fixed query points (pixel edges, (-1, 0) projections, points behind the cameras and in the back-mask band).

Settings: the default; use_normals=False; max_tsdf_abs; -cam (PNG normals in camera coordinates) on and off;
pixel_stride 1 and 6; choose_best_frame; two_pass=False with normals.  The folder's arrays are stored too, so tests
rebuild it without the reference (tests/test_isooctree_cpu.py).

Run only where /root/reference exists:   python tests/golden/make_golden_isooctree.py
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
from tests import isooctree_scene as S  # noqa: E402

REF = "/root/reference/dn_splatter/scripts/isooctree_dn.py"

# name -> (camera_coordinate_normals, build_mesh_projection kwargs)
SETTINGS = {
    "default": (False, dict(pixel_stride=6)),
    "no_normals": (False, dict(pixel_stride=6, use_normals=False)),
    "tsdf_abs": (False, dict(pixel_stride=6, max_tsdf_abs=0.04)),
    "cam": (True, dict(pixel_stride=6)),
    "cam_stride1": (True, dict(pixel_stride=1)),
    "stride1": (False, dict(pixel_stride=1)),
    "best_frame": (False, dict(pixel_stride=6, choose_best_frame=True)),
    "one_pass": (False, dict(pixel_stride=6, two_pass=False)),
}


def main():
    record = {}

    def build(iso_func, hint, maxDepth, subdivisionThreshold):
        record["hint"] = np.array(hint)
        record["values"] = np.array(iso_func(record["queries"]))
        return types.SimpleNamespace(vertices=np.zeros((0, 3)), triangles=np.zeros((0, 3), int))

    sys.modules["IsoOctree"] = types.SimpleNamespace(buildMeshWithPointCloudHint=build)
    spec = importlib.util.spec_from_file_location("ref_isooctree_dn", REF)
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)

    files = [S.frame_files(p) for p in S.POSES]
    z = {
        "depth_mm": np.stack([f[0] for f in files]), "normal_npy": np.stack([f[1] for f in files]),
        "normal_png": np.stack([f[2] for f in files]),
        "transforms": np.stack([S.transform_matrix(p) for p in S.POSES]),
        "camera": np.array(json.dumps(S.camera_json())), "queries": S.query_points(),
    }
    record["queries"] = z["queries"]
    with tempfile.TemporaryDirectory() as tmp:
        js = S.write_folder(tmp, S.camera_json(), z["transforms"], z["depth_mm"], z["normal_npy"], z["normal_png"])
        for name, (cam, kw) in SETTINGS.items():
            frames = ref.load_frame_metadata(tmp, js, camera_coordinate_normals=cam)
            assert len(frames) == len(S.POSES)
            ref.build_mesh_projection(frames, subdivision_threshold=50, max_depth=8, **kw)
            z[f"{name}/hint"] = record["hint"]
            z[f"{name}/values"] = record["values"]
            print(name, record["hint"].shape, np.unique(np.round(record["values"], 6)).shape)
    np.savez_compressed(os.path.join(OUT, "dn_isooctree.npz"), **z)


if __name__ == "__main__":
    main()
