"""CPU-side checks of the drop-in boundary: the C-ABI library builds/loads, exports every symbol that
include/dnr.h declares, the ctypes mirror of DnrArgs matches the header field for field, and argument
errors are reported as negative codes without touching a GPU."""
import ctypes as C
import os
import re

import pytest

from dn_splatter_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "dnr.h")


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(L.LIB_PATH):
        from dn_splatter_b200.build import build

        build()
    return L.load()


def _declared_functions():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(dnr_[a-z_0-9]+)\s*\(", src)))


def _header_fields():
    src = open(HEADER).read()
    body = src[src.index("typedef struct DnrArgs {"):src.index("} DnrArgs;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for stmt in body.split(";"):
        stmt = stmt.replace("typedef struct DnrArgs {", "").strip()
        if not stmt:
            continue
        m = re.match(r"(const\s+)?(\w+)\s*(\**)\s*(.*)", stmt.strip())
        base, star, names = m.group(2), m.group(3), m.group(4)
        for nm in names.split(","):
            nm = nm.strip()
            is_ptr = bool(star) or nm.startswith("*")
            nm = nm.lstrip("*").strip()
            arr = re.match(r"(\w+)\[(\d+)\]", nm)
            if arr:
                fields.append((arr.group(1), f"{base}[{arr.group(2)}]"))
            else:
                fields.append((nm, "ptr" if is_ptr else base))
    return fields


def test_library_exports_every_declared_symbol(lib):
    declared = _declared_functions()
    assert set(declared) == set(L.EXPORTS)
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in dnr.h but not exported"
    assert lib.dnr_version() == 100


def test_ctypes_struct_matches_header():
    want = _header_fields()
    ctype_name = {C.c_int32: "int32_t", C.c_uint32: "uint32_t", C.c_float: "float", C.c_int64: "int64_t",
                  C.c_void_p: "ptr"}
    got = []
    for name, t in L.DnrArgs._fields_:
        if t in ctype_name:
            got.append((name, ctype_name[t]))
        else:
            got.append((name, f"float[{t._length_}]"))
    assert got == want


def test_argument_errors_are_negative_codes(lib):
    a = L.DnrArgs()
    assert lib.dnr_project_fwd(None, None) == -1
    assert lib.dnr_project_fwd(C.byref(a), None) == -2  # n_gauss == 0
    a.n_gauss, a.width, a.height, a.tile_size, a.sh_degree, a.sh_bases = 10, 32, 32, 8, 3, 16
    assert lib.dnr_project_fwd(C.byref(a), None) == -3  # tile size must be 16
    a.tile_size = 16
    assert lib.dnr_project_fwd(C.byref(a), None) == -1  # NULL buffers
    a.sh_degree = 4
    assert lib.dnr_project_fwd(C.byref(a), None) == -3
    assert lib.dnr_raster_fwd(C.byref(a), None) == -1
    assert lib.dnr_bin_scan(C.byref(a), None, None) == -1
    assert b"NULL" in lib.dnr_error_string(-1)
    assert lib.dnr_bin_scan_workspace_bytes(1000) > 1000 * 20
    assert lib.dnr_bin_sort_workspace_bytes(1000, 5000, 64) > 5000 * 8


def test_argument_errors_of_the_8f_entry_points(lib):
    """SSIM / Adam / k-NN / density validate their arguments before touching the GPU."""
    one = C.c_void_p(16)  # a non-NULL dummy: the size checks come first, nothing is dereferenced
    assert lib.dnr_ssim_fwd(None, one, 32, 32, 3, one, one, None) == -1
    assert lib.dnr_ssim_fwd(one, one, 10, 32, 3, one, one, None) == -2  # an 11x11 window needs H, W > 10
    assert lib.dnr_ssim_bwd(one, one, 32, 32, 3, None, None, one, None) == -1
    assert lib.dnr_adam_step(None, 1, 0.9, 0.999, None) == -1
    seg = (L.DnrAdamSeg * 1)()
    assert lib.dnr_adam_step(C.cast(seg, C.c_void_p), 0, 0.9, 0.999, None) == -2
    assert lib.dnr_adam_step(C.cast(seg, C.c_void_p), 17, 0.9, 0.999, None) == -2  # DNR_ADAM_MAX_SEGS = 16
    assert lib.dnr_adam_step(C.cast(seg, C.c_void_p), 1, 0.9, 0.999, None) == -1  # NULL tensors in the segment
    g = L.DnrKnnGrid()
    assert lib.dnr_knn_workspace_bytes(100, C.byref(g)) == -1  # zero dims
    g.cell, g.inv_cell = 0.5, 2.0
    g.dims[0], g.dims[1], g.dims[2] = 8, 8, 8
    assert lib.dnr_knn_workspace_bytes(100, C.byref(g)) >= 100 * (4 + 4 + 4 + 4 + 16) + 2 * 512 * 4
    assert lib.dnr_knn_build(None, 100, C.byref(g), one, 1 << 20, None) == -1
    assert lib.dnr_knn_build(one, 100, C.byref(g), one, 8, None) == -5  # workspace too small
    assert lib.dnr_knn_query(100, C.byref(g), one, one, 5, 40, 1, one, None, None) == -3  # k + 1 > 33
    assert lib.dnr_density(one, 0, one, 16, 1, one, one, one, one, 10, 0.0, one, None) == -2
    assert lib.dnr_ray_densities(one, 5, one, 16, one, one, one, one, one, 10, 20, 3.0, one, one, one, None) == -3  # 21 samples only


def _reduce_call(lib, break_one):
    """dnr_adam_step_reduce on fake 16-byte-aligned addresses (never dereferenced): a valid call at world 3, rank 1 with
    one field broken by `break_one(segs, widths, peers)`, which returns the arguments to pass instead when it replaces
    one (n_segs).  Every case must fail a host check, so nothing is launched."""
    segs = (L.DnrAdamSeg * 2)()
    widths = (C.c_int32 * 2)(3, 45)
    pr = L.DnrPeerReduce()
    pr.world, pr.rank, pr.n_gauss = 3, 1, 8
    for k in range(3):
        pr.peer_flat[k], pr.peer_touched[k] = 0x1000000 * (k + 1), 0x1000000 * (k + 1) + 0x800000
    pr.mask = 0x9000000
    for i, (off, w) in enumerate(((0, 3), (24, 45))):  # segment offsets in floats, multiples of 4
        segs[i].p, segs[i].m, segs[i].v = 0x10000000 + 0x100000 * i, 0x20000000 + 0x100000 * i, 0x30000000 + 0x100000 * i
        segs[i].g = pr.peer_flat[1] + 4 * off
        segs[i].n, segs[i].lr, segs[i].eps, segs[i].bc1, segs[i].bc2_sqrt = 8 * w, 1e-3, 1e-15, 0.1, 0.03
    n_segs = break_one(segs, widths, pr)
    return lib.dnr_adam_step_reduce(C.cast(segs, C.c_void_p), C.cast(widths, C.c_void_p), 2 if n_segs is None else n_segs,
                                    0.9, 0.999, C.byref(pr), None)


def _set(obj, **kw):
    for k, v in kw.items():
        setattr(obj, k, v)


REDUCE_ARGUMENT_ERRORS = {
    "null_segs": (-1, None),
    "null_widths": (-1, None),
    "null_peers": (-1, None),
    "n_segs_0": (-2, lambda s, w, p: 0),
    "n_segs_17": (-2, lambda s, w, p: 17),
    "world_0": (-2, lambda s, w, p: _set(p, world=0)),
    "world_9": (-2, lambda s, w, p: _set(p, world=9)),
    "rank_-1": (-2, lambda s, w, p: _set(p, rank=-1)),
    "rank_eq_world": (-2, lambda s, w, p: _set(p, rank=3)),
    "n_gauss_0": (-2, lambda s, w, p: _set(p, n_gauss=0)),
    "null_mask_at_world_3": (-1, lambda s, w, p: _set(p, mask=None)),
    "null_peer_flat_0": (-1, lambda s, w, p: p.peer_flat.__setitem__(0, None)),
    "null_peer_flat_2": (-1, lambda s, w, p: p.peer_flat.__setitem__(2, None)),
    "null_peer_touched_2": (-1, lambda s, w, p: p.peer_touched.__setitem__(2, None)),
    "null_p": (-1, lambda s, w, p: _set(s[1], p=None)),
    "width_0": (-2, lambda s, w, p: w.__setitem__(1, 0)),
    "n_not_a_multiple_of_width": (-2, lambda s, w, p: _set(s[1], n=8 * 45 + 1)),
    "n_over_width_is_not_n_gauss": (-2, lambda s, w, p: _set(s[1], n=9 * 45)),
    "n_at_2_pow_32": (-2, lambda s, w, p: (_set(p, n_gauss=1 << 30), _set(s[0], n=3 << 30), w.__setitem__(1, 4),
                                           _set(s[1], n=1 << 32)) and None),
    "g_below_peer_flat_rank": (-2, lambda s, w, p: _set(s[0], g=p.peer_flat[1] - 16)),
    "g_offset_1_float": (-2, lambda s, w, p: _set(s[1], g=s[1].g + 4)),
    "g_offset_2_floats": (-2, lambda s, w, p: _set(s[1], g=s[1].g + 8)),
    "g_offset_3_floats": (-2, lambda s, w, p: _set(s[1], g=s[1].g + 12)),
    "p_misaligned": (-2, lambda s, w, p: _set(s[1], p=s[1].p + 4)),
    "m_misaligned": (-2, lambda s, w, p: _set(s[1], m=s[1].m + 8)),
    "v_misaligned": (-2, lambda s, w, p: _set(s[0], v=s[0].v + 12)),
    "bc1_0": (-2, lambda s, w, p: _set(s[1], bc1=0.0)),
    "bc1_negative": (-2, lambda s, w, p: _set(s[0], bc1=-0.5)),
    "bc1_nan": (-2, lambda s, w, p: _set(s[0], bc1=float("nan"))),
}


@pytest.mark.parametrize("case", list(REDUCE_ARGUMENT_ERRORS))
def test_argument_errors_of_adam_step_reduce(lib, case):
    """Host checks of dnr_adam_step_reduce, each from a valid call with exactly one field broken: a negative code before
    any CUDA call."""
    want, brk = REDUCE_ARGUMENT_ERRORS[case]
    if brk is None:  # a NULL array or struct
        segs, widths, pr = (L.DnrAdamSeg * 1)(), (C.c_int32 * 1)(3), L.DnrPeerReduce()
        args = [C.cast(segs, C.c_void_p), C.cast(widths, C.c_void_p), 1, 0.9, 0.999, C.byref(pr), None]
        args[{"null_segs": 0, "null_widths": 1, "null_peers": 5}[case]] = None
        assert lib.dnr_adam_step_reduce(*args) == want
        return
    assert _reduce_call(lib, brk) == want


def test_product_path_fails_loudly_without_cuda():
    import torch

    from dn_splatter_b200 import dn_rasterize

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    z = torch.zeros
    with pytest.raises(L.DnrError):
        dn_rasterize(z(4, 3), z(4, 4), z(4, 3), z(4, 1), z(4, 3), z(4, 15, 3), torch.eye(4), torch.eye(3), 32, 32,
                     render_normals=False)
