"""CPU checks of the flat gradient bucket's sparse mode: the host-side rule that decides when its `touched` flags cover
every non-zero row, the argument checks of dnr_grad_zero, and numpy mirrors of what the sparse kernels read and write."""
import ctypes as C

import numpy as np
import pytest
import torch

from dn_splatter_b200 import _lib as L
from dn_splatter_b200.parallel import FlatGradBucket, bucket_of
from tests.test_fused_adam_cpu import _peer_gather_mirror


def _bucket(n=50):
    shapes = {"means": (n, 3), "scales": (n, 3), "quats": (n, 4), "features_dc": (n, 3), "features_rest": (n, 15, 3),
              "opacities": (n, 1)}
    return FlatGradBucket({k: torch.nn.Parameter(torch.zeros(*s)) for k, s in shapes.items()})


def test_flags_are_valid_only_after_backwards_since_a_zero():
    b = _bucket()
    assert not b.flags_valid  # a fresh bucket may be filled by other means (flat.copy_)
    b.note_backward()
    assert not b.flags_valid  # ... so a backward without a zero_() first does not validate it
    b.zero_()  # dense while the flags are not valid (no kernel: runs on the CPU)
    b.note_backward()
    b.note_backward()  # the antialiased + normals model: two flagged passes per step
    assert b.flags_valid
    b = _bucket()
    b.zero_()
    b.sparse_ok = False  # parameter-only loss terms besides min-scale (dn_model.enable_flat_grads)
    b.note_backward()
    assert not b.flags_valid
    assert b.dense_params == {"scales"} and b.n_gauss == 50
    assert b.grad_records.shape == (50, L.GRAD_FLOATS) and b.touched.dtype == torch.uint8
    assert set(b.sink()) == set(b.names) | {"touched", "grad_records", "bucket"}


def test_bucket_of_finds_the_bucket_of_a_view_only():
    b = _bucket()
    for v in b.views.values():
        assert bucket_of(v) is b
    assert bucket_of(b.views["means"].clone()) is None
    assert bucket_of(torch.zeros(4)) is None


def test_grad_zero_argument_errors():
    lib = L.load()
    one = C.c_void_p(16)
    seg = (L.DnrGradSeg * 1)()
    assert lib.dnr_grad_zero(None, 1, one, 10, None) == -1
    assert lib.dnr_grad_zero(C.cast(seg, C.c_void_p), 1, None, 10, None) == -1
    assert lib.dnr_grad_zero(C.cast(seg, C.c_void_p), 0, one, 10, None) == -2
    assert lib.dnr_grad_zero(C.cast(seg, C.c_void_p), 17, one, 10, None) == -2  # DNR_ADAM_MAX_SEGS
    assert lib.dnr_grad_zero(C.cast(seg, C.c_void_p), 1, one, 0, None) == -2
    assert lib.dnr_grad_zero(C.cast(seg, C.c_void_p), 1, one, 10, None) == -1  # NULL segment
    seg[0].g, seg[0].width = 20, 3
    assert lib.dnr_grad_zero(C.cast(seg, C.c_void_p), 1, one, 10, None) == -2  # not 16-byte aligned
    seg[0].g, seg[0].width = 16, 0
    assert lib.dnr_grad_zero(C.cast(seg, C.c_void_p), 1, one, 10, None) == -2
    assert L.FLAG_PERSISTENT_WS == 256


@pytest.mark.parametrize("width", [1, 3, 4, 45])
def test_single_rank_gather_reads_exactly_the_bucket(width):
    """dnr_adam_step_reduce at world 1 (the single-GPU sparse step): the bucket's own flags as the mask select rows that
    reproduce the dense gradient bit for bit, because untouched rows are zero."""
    rng = np.random.default_rng(width)
    n_gauss = 37
    touched = (rng.random(n_gauss) < 0.35).astype(np.uint8)
    rows = (rng.standard_normal((n_gauss, width)).astype(np.float32) * touched[:, None]).reshape(-1)
    assert np.array_equal(_peer_gather_mirror([rows], [touched], width), rows)


def _grad_zero_mirror(seg, flags, width, dense, chunk=256):
    """numpy mirror of csrc/adam.cu grad_zero_kernel on one padded segment: returns the segment after the call and the
    number of float4 stores."""
    out, n, stores = seg.copy(), flags.size, 0
    for g0 in range(0, n, chunk):
        ng = min(chunk, n - g0)
        f = flags[g0:g0 + ng]
        if not dense and not f.any():
            continue
        for i in range((ng * width + 3) // 4):
            hit = dense or any(f[j] for j in range(4 * i // width, min((4 * i + 3) // width, ng - 1) + 1))
            if hit:
                base = g0 * width + 4 * i
                out[base:base + 4] = 0.0
                stores += 1
    return out, stores


def grad_zero_mirror_vec(seg, flags, width, dense):
    """_grad_zero_mirror without the per-float4 Python loop (for segments of millions of floats): chunks of 256 Gaussians
    start on float4 boundaries, so float4 q of the padded segment is stored iff the segment is dense or a Gaussian among
    those of its four elements (the last one standing in for the padding) is flagged."""
    n = flags.size
    q4 = np.arange((n * width + 3) // 4, dtype=np.int64) * 4
    hit = np.full(q4.size, bool(dense))
    if not dense:
        for r in range(4):
            hit |= flags[np.minimum((q4 + r) // width, n - 1)] != 0
    out = seg.copy()
    out[:4 * q4.size].reshape(-1, 4)[hit] = 0.0
    return out, int(hit.sum())


@pytest.mark.parametrize("width", [1, 2, 3, 4, 45, 4096])
@pytest.mark.parametrize("n_gauss", [1, 255, 256, 257, 600])
def test_vectorised_grad_zero_mirror_equals_the_loop(width, n_gauss):
    rng = np.random.default_rng(width * 7 + n_gauss)
    flags = (rng.random(n_gauss) < 0.02).astype(np.uint8) * rng.choice(np.array([1, 0x80, 0xff], np.uint8), n_gauss)
    flags[-1] = 2
    if n_gauss == 600:
        flags[256:512] = 0  # a chunk without flags
    seg = rng.uniform(1, 2, (n_gauss * width + 3) & ~3).astype(np.float32)
    for dense in (False, True):
        a, b = _grad_zero_mirror(seg, flags, width, dense), grad_zero_mirror_vec(seg, flags, width, dense)
        assert np.array_equal(a[0], b[0]) and a[1] == b[1]


@pytest.mark.parametrize("width", [1, 3, 4, 45])
@pytest.mark.parametrize("n_gauss", [37, 600])
def test_grad_zero_clears_every_flagged_row_and_stays_in_the_padded_segment(width, n_gauss):
    rng = np.random.default_rng(width * 1000 + n_gauss)
    flags = (rng.random(n_gauss) < 0.1).astype(np.uint8)
    padded = (n_gauss * width + 3) & ~3
    seg = np.zeros(padded, dtype=np.float32)
    seg[:n_gauss * width] = (rng.standard_normal((n_gauss, width)).astype(np.float32) * flags[:, None]).reshape(-1)
    out, stores = _grad_zero_mirror(seg, flags, width, dense=False)  # an out-of-range store raises in numpy slicing
    assert not out.any()
    assert stores * 4 <= padded
    touched_f4 = {(g * width + k) // 4 for g in np.flatnonzero(flags) for k in range(width)}
    assert stores == len(touched_f4)  # only float4s that hold a flagged row are written
    dense_seg = rng.standard_normal(padded).astype(np.float32)
    dense_seg[n_gauss * width:] = 0.0
    out, stores = _grad_zero_mirror(dense_seg, flags, width, dense=True)
    assert not out.any() and stores * 4 == padded
