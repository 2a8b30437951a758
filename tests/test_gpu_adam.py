"""csrc/adam.cu on one GPU: dnr_adam_step (float4 and scalar paths, grid-stride passes, 16 segments with their own lr /
eps / step count), dnr_adam_step_reduce at every rank count 1-8 with the W "ranks" as W buckets on the same device
(it only dereferences the pointers in DnrPeerReduce), and dnr_grad_zero.

Every step is checked from the kernel's own previous state: within oracle/adam_ref.py's fp32 bound of the fp64 step, and
bit for bit against FusedAdam.reference_step on the CPU (adam.cu is built with -fmad=false and IEEE division and sqrt).
The reduce path must give bit-identical replicas, equal to dnr_adam_step on the rank-ordered dense sum of the
gradients; grad_zero must store exactly the float4s its numpy mirror stores."""
import ctypes as C

import numpy as np
import pytest
import torch

from dn_splatter_b200 import _lib as L
from dn_splatter_b200.optim import FusedAdam, bias_corrections
from oracle.adam_ref import fp32_scalars
from tests.test_adam_ref_cpu import BETAS, SIXTEEN, STEPS, Seg, check_step, reference_step, scalars, segment_state
from tests.test_sparse_grads_cpu import _grad_zero_mirror, grad_zero_mirror_vec

pytestmark = pytest.mark.gpu
needs_cuda = pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")

GUARD = 8  # sentinel floats before and after every buffer (a multiple of 4: the buffer itself stays 16-byte aligned)
SENTINEL = 0x7FA5A5A5  # a NaN bit pattern no step can produce


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _guarded(x: np.ndarray, offset: int = 0):
    """(whole buffer, view): `x` on the device at float GUARD + offset of a buffer framed by sentinels."""
    buf = torch.full((GUARD + offset + x.size + GUARD,), SENTINEL, dtype=torch.int32).view(torch.float32)
    buf[GUARD + offset:GUARD + offset + x.size] = torch.from_numpy(x)
    buf = buf.cuda()
    return buf, buf[GUARD + offset:GUARD + offset + x.size]


def _assert_guards(buf, n, offset, what):
    g = _bits(buf).cpu().numpy()
    assert (g[:GUARD + offset] == SENTINEL).all() and (g[GUARD + offset + n:] == SENTINEL).all(), what


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _run_adam_step(segs, offsets=None):
    """STEPS launches of dnr_adam_step over `segs` (Seg tuples); `offsets`: {"p" | "g" | "m" | "v": floats} shifts that
    pointer of every segment off 16 bytes."""
    offsets = offsets or {}
    host = [segment_state(s) for s in segs]
    dev = []
    for (p, m, v, grads) in host:
        d = {}
        for name, x in (("p", p), ("g", grads[0]), ("m", m), ("v", v)):
            d[name] = _guarded(x, offsets.get(name, 0))
        dev.append(d)
    arr = (L.DnrAdamSeg * len(segs))()
    for i, d in enumerate(dev):
        arr[i].p, arr[i].g, arr[i].m, arr[i].v = (d[k][1].data_ptr() for k in "pgmv")
        for k in "pgmv":
            assert (d[k][1].data_ptr() % 16 == 0) == (offsets.get(k, 0) == 0)
    for s in range(STEPS):
        cur = []
        for i, (seg, d) in enumerate(zip(segs, dev)):
            g = host[i][3][s]
            d["g"][1].copy_(torch.from_numpy(g))
            bc1, bc2s = bias_corrections(seg.t + s, *BETAS)
            arr[i].n, arr[i].lr, arr[i].eps, arr[i].bc1, arr[i].bc2_sqrt = seg.n, seg.lr, seg.eps, bc1, bc2s
            cur.append(tuple(d[k][1].cpu().numpy() for k in "pgmv"))  # the kernel's own state before this step
        L.check(L.load().dnr_adam_step(C.cast(arr, C.c_void_p), len(segs), BETAS[0], BETAS[1], _stream()), "dnr_adam_step")
        torch.cuda.synchronize()
        ref = reference_step(segs, [(p, g, m, v) for p, g, m, v in cur], [seg.t + s for seg in segs])
        for i, (seg, d) in enumerate(zip(segs, dev)):
            got = tuple(d[k][1].cpu().numpy() for k in "pmv")
            p, g, m, v = cur[i]
            check_step(got, p, g, m, v, scalars(seg, seg.t + s), (s, seg))
            for name, x, y in zip("pmv", got, ref[i]):
                assert np.array_equal(x.view(np.int32), y.view(np.int32)), ("reference_step", s, seg, name,
                                                                            np.flatnonzero(x != y)[:5])
            for k in "pgmv":
                _assert_guards(d[k][0], seg.n, offsets.get(k, 0), (s, seg, k))


LENGTHS = [1, 2, 3, 4, 5, 7, 8, 1023, 4097, 3_000_001]  # 3 000 001: 2.8 grid-stride passes of float4s, then the tail


@needs_cuda
@pytest.mark.parametrize("init", ["zero", "random"])
@pytest.mark.parametrize("n", LENGTHS)
def test_adam_step_one_segment(n, init):
    _run_adam_step([Seg(n, 1e-3, 1e-15, 1, 11 + n % 1000, init)])


@needs_cuda
def test_adam_step_largest_and_smallest_segment_in_one_launch():
    _run_adam_step([Seg(3_000_001, 5e-3, 1e-15, 10, 3, "random"), Seg(1, 1.6e-4, 1e-8, 1000, 4, "random")])


@needs_cuda
def test_adam_step_sixteen_segments_with_their_own_lr_eps_and_step():
    assert len(SIXTEEN) == 16 and len({(s.lr, s.eps, s.t) for s in SIXTEEN}) == 16
    _run_adam_step(SIXTEEN)


@needs_cuda
@pytest.mark.parametrize("offset", [1, 2, 3])
@pytest.mark.parametrize("which", ["p", "g", "m", "v"])
def test_adam_step_unaligned_pointer_takes_the_scalar_path(which, offset):
    _run_adam_step([Seg(4097, 2e-3, 1e-15, 2, 21, "random"), Seg(6, 1e-2, 1e-8, 1, 22, "zero")], {which: offset})


@needs_cuda
def test_adam_step_unaligned_over_several_grid_stride_passes():
    _run_adam_step([Seg(3_000_001, 1e-3, 1e-15, 1000, 23, "random")], {"v": 1})


# ---- dnr_adam_step_reduce: W buckets on one device ----

PRODUCT = {"means": (3,), "scales": (3,), "quats": (4,), "features_dc": (3,), "features_rest": (15, 3), "opacities": (1,)}
PRODUCT_LR = {"means": 1.6e-4, "scales": 5e-3, "quats": 1e-3, "features_dc": 2.5e-3, "features_rest": 1.25e-4,
              "opacities": 5e-2}
# 16 groups of widths 1-16; the width-3 one is named `scales`, so it is the dense segment
SIXTEEN_GROUPS = {("scales" if w == 3 else f"w{w:02d}"): (w,) for w in range(1, 17)}
FLAG_BYTES = np.array([1, 2, 0x7F, 0x80, 0xFF], np.uint8)


def _replica(groups, lrs, n, seed):
    """Parameters, and a FusedAdam whose state starts at random moments and per-group step counts."""
    rng = np.random.default_rng(seed)
    params, pg, state = {}, [], {}
    for i, (name, shape) in enumerate(groups.items()):
        full = (n, *shape)
        params[name] = torch.nn.Parameter(torch.from_numpy(rng.standard_normal(full).astype(np.float32)).cuda())
        pg.append({"params": [params[name]], "lr": lrs.get(name, 1e-3 * (1 + i)), "eps": (1e-15, 1e-8)[i % 2], "name": name})
        m = (rng.standard_normal(full) * 1e-2).astype(np.float32)
        v = ((rng.standard_normal(full) * 1e-2) ** 2).astype(np.float32)
        state[name] = ((0, 1, 9, 999, 99999)[i % 5], m, v)
    opt = FusedAdam(pg, betas=BETAS)
    for name, (t, m, v) in state.items():
        opt.state[params[name]] = {"step": t, "exp_avg": torch.from_numpy(m).cuda(), "exp_avg_sq": torch.from_numpy(v).cuda()}
    return params, opt


def _fill_ranks(rng, buckets, groups, n):
    """Per rank: flags at 10-35 % with bytes from FLAG_BYTES (Gaussians i % 5 == 1 touched by every rank, i % 5 == 3 by
    none), random rows for flagged Gaussians, exactly zero rows for the others; the dense `scales` rows non-zero
    everywhere.  Returns the flags."""
    idx = np.arange(n)
    flags = []
    for b in buckets:
        sel = rng.random(n) < rng.uniform(0.10, 0.35)
        sel[idx % 5 == 1], sel[idx % 5 == 3] = True, False
        f = rng.choice(FLAG_BYTES, n) * sel
        for name, shape in groups.items():
            rows = rng.standard_normal((n, *shape)) * 10.0 ** rng.uniform(-6, 2, (n,) + (1,) * len(shape))
            if name in b.dense_params:
                rows = np.where(rows == 0, 1.0, rows)
            else:
                rows = rows * sel.reshape((n,) + (1,) * len(shape))
            b.views[name].copy_(torch.from_numpy(rows.astype(np.float32)))
        b.touched.copy_(torch.from_numpy(f.astype(np.uint8)))
        flags.append(f)
    return flags


def _run_reduce(groups, lrs, world, n, seed):
    from dn_splatter_b200.parallel import FlatGradBucket

    replicas = [_replica(groups, lrs, n, seed) for _ in range(world)]
    twin, twin_opt = _replica(groups, lrs, n, seed)
    buckets = [FlatGradBucket(params, names=list(groups)) for params, _ in replicas]
    for b in buckets:
        assert b.dense_params == {"scales"} and b.n_gauss == n
    pad = (n + 15) // 16 * 16
    all_ranks = (1 << world) - 1
    masks = [torch.full((pad,), all_ranks, dtype=torch.uint8, device="cuda") for _ in range(world)]
    for mk in masks:
        mk[:n] = 0
    rng = np.random.default_rng(seed + 1)
    for s in range(STEPS):
        flags = _fill_ranks(rng, buckets, groups, n)
        flat0 = [b.flat.clone() for b in buckets]
        touched0 = [b.touched.clone() for b in buckets]
        for r, ((params, opt), b) in enumerate(zip(replicas, buckets)):
            pr = L.DnrPeerReduce()
            pr.world, pr.rank, pr.n_gauss = world, r, n
            for k in range(world):
                pr.peer_flat[k], pr.peer_touched[k] = buckets[k].flat.data_ptr(), buckets[k].touched.data_ptr()
            pr.mask = masks[r].data_ptr()
            FusedAdam._launch_reduce(opt._segments(), b, pr)
        # the dense twin: dnr_adam_step on the fp32 rank-ordered sum ((g0 + g1) + g2) + ...
        before = {}
        for name in groups:
            acc = buckets[0].views[name].clone()
            for k in range(1, world):
                acc = acc + buckets[k].views[name]
            twin[name].grad = acc
            st = twin_opt.state[twin[name]]
            before[name] = (twin[name].detach().cpu().numpy().ravel(), acc.cpu().numpy().ravel(),
                            st["exp_avg"].cpu().numpy().ravel(), st["exp_avg_sq"].cpu().numpy().ravel(), int(st["step"]) + 1)
        twin_opt.step()
        torch.cuda.synchronize()
        for k, b in enumerate(buckets):  # every peer's bucket and flags are read, never written
            assert torch.equal(_bits(b.flat), _bits(flat0[k])) and torch.equal(b.touched, touched0[k]), (s, k)
        want_mask = np.zeros(n, np.int64)
        for k, f in enumerate(flags):
            want_mask |= (f != 0).astype(np.int64) << k
        assert (want_mask == all_ranks).any() and (want_mask == 0).any()
        for r, mk in enumerate(masks):
            got = mk.cpu().numpy()
            if world > 1:
                assert np.array_equal(got[:n], want_mask), (s, r, np.flatnonzero(got[:n] != want_mask)[:5])
            else:  # world 1 reads the bucket's own flags; the scratch is not touched
                assert not got[:n].any()
            assert (got[n:] == all_ranks).all(), (s, r)
        for name in groups:
            tp = twin[name]
            tst = twin_opt.state[tp]
            for r, (params, opt) in enumerate(replicas):
                q = params[name]
                st = opt.state[q]
                assert int(st["step"]) == int(tst["step"])
                for x, y, what in ((q.detach(), tp.detach(), "p"), (st["exp_avg"], tst["exp_avg"], "m"),
                                   (st["exp_avg_sq"], tst["exp_avg_sq"], "v")):
                    assert torch.equal(_bits(x), _bits(y)), (s, name, r, what, int((x != y).sum()))
            p, g, m, v, t = before[name]
            grp = next(gr for gr in twin_opt.param_groups if gr["name"] == name)
            bc1, bc2s = bias_corrections(t, *BETAS)
            sc = fp32_scalars(grp["lr"], grp["eps"], bc1, bc2s, *BETAS)
            got = tuple(x.detach().cpu().numpy().ravel() for x in (tp, tst["exp_avg"], tst["exp_avg_sq"]))
            check_step(got, p, g, m, v, sc, (s, name))


WORLDS = [1, 2, 3, 4, 5, 7, 8]


@needs_cuda
@pytest.mark.parametrize("n_gauss", [5, 16, 37, 4099, 30001])  # 16, 4099: peer_mask's vector and tail paths
@pytest.mark.parametrize("world", WORLDS)
def test_adam_step_reduce_product_groups(world, n_gauss):
    _run_reduce(PRODUCT, PRODUCT_LR, world, n_gauss, seed=world * 100003 + n_gauss)


@needs_cuda
@pytest.mark.parametrize("world", WORLDS)
def test_adam_step_reduce_sixteen_groups_of_widths_1_to_16(world):
    _run_reduce(SIXTEEN_GROUPS, {}, world, 4099, seed=world)


# ---- dnr_grad_zero ----

def _run_grad_zero(specs, n, seed):
    """specs: [(width, dense)]; every segment (padding included) filled with non-zero values, sentinels between the
    padded segments and after the flags."""
    rng = np.random.default_rng(seed)
    flags = (rng.random(n) < 0.2) * rng.choice(FLAG_BYTES, n)
    flags[-1] = 0x80  # the last chunk's last row is flagged: its float4 may reach into the padding
    if n > 512:
        flags[256:512] = 0  # a chunk without flags
    flags = flags.astype(np.uint8)
    sizes = [(n * w + 3) & ~3 for w, _ in specs]
    host = np.full(GUARD + sum(s + GUARD for s in sizes), 0, np.float32)
    host.view(np.int32)[:] = SENTINEL
    offs, o = [], GUARD
    for size in sizes:
        host[o:o + size] = rng.uniform(0.5, 2.0, size).astype(np.float32) * np.where(rng.random(size) < 0.5, -1, 1)
        offs.append(o)
        o += size + GUARD
    buf = torch.from_numpy(host).cuda()
    touched = torch.from_numpy(np.concatenate([flags, np.full(16, 0x5A, np.uint8)])).cuda()
    segs = (L.DnrGradSeg * len(specs))()
    for i, ((w, dense), off) in enumerate(zip(specs, offs)):
        segs[i].g, segs[i].width, segs[i].dense = buf.data_ptr() + 4 * off, w, int(dense)
    L.check(L.load().dnr_grad_zero(C.cast(segs, C.c_void_p), len(specs), touched.data_ptr(), n, _stream()), "dnr_grad_zero")
    torch.cuda.synchronize()
    got = buf.cpu().numpy()
    t = touched.cpu().numpy()
    assert not t[:n].any() and (t[n:] == 0x5A).all()
    expect = host.copy()
    for (w, dense), off, size in zip(specs, offs, sizes):
        seg = host[off:off + size]
        mirror = _grad_zero_mirror if size <= 300_000 else grad_zero_mirror_vec
        expect[off:off + size] = mirror(seg, flags, w, dense)[0]
    bad = np.flatnonzero(got.view(np.int32) != expect.view(np.int32))
    assert bad.size == 0, (bad[:8], got[bad[:8]], expect[bad[:8]])


# widths up to 4096 (the maximum) x counts around the 256-Gaussian chunk; width 4096 stops at 600 Gaussians (three
# chunks, 2.5 M floats) rather than 100003 (1.6 GB per segment)
GZ_CASES = [(w, n) for w in (1, 2, 3, 4, 45, 4096) for n in (1, 255, 256, 257, 600, 100003) if w * n < 5_000_000]


@needs_cuda
@pytest.mark.parametrize("width,n_gauss", GZ_CASES)
def test_grad_zero_sparse_and_dense_segment_in_one_call(width, n_gauss):
    _run_grad_zero([(width, False), (width, True)], n_gauss, seed=width * 1000003 + n_gauss)


@needs_cuda
@pytest.mark.parametrize("n_gauss", [257, 600])
def test_grad_zero_sixteen_segments_in_one_call(n_gauss):
    widths = [1, 2, 3, 4, 5, 7, 8, 13, 16, 45, 64, 100, 1, 3, 4096, 45]
    _run_grad_zero([(w, i % 4 == 1) for i, w in enumerate(widths)], n_gauss, seed=n_gauss)
