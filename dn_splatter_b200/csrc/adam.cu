// One-launch Adam over every Gaussian parameter group (SURVEY.md §8f-3, "next" row).  The reference builds one
// torch.optim.Adam per group (/root/reference/dn_splatter/dn_config.py:29-68: lr per group, eps 1e-15, no weight decay,
// no amsgrad) and nerfstudio steps them one after the other [EXT Optimizers.optimizer_step]; at 1M Gaussians that is
// 59M parameters x 28 B = 1.65 GB of HBM traffic (at least 0.49 ms at the H100 SXM data sheet's 3.35 TB/s), but
// 7 optimizers x several elementwise passes each in torch.  Here: one kernel, blockIdx.y = group, float4 grid-stride
// over the group.  A single-GPU bucket whose `touched` flags are valid is stepped by adam_reduce_kernel<1> instead, which
// reads only the touched gradient rows (28 B -> ~24.4 B per float).
//
// Update rule — torch.optim.Adam [EXT torch 2.x, _single_tensor_adam], dense (zero-gradient rows still decay):
//   m = m + (1-b1)(g - m)  [lerp];  v = b2 v + (1-b2) g g;  p -= (lr / bc1) * m / (sqrt(v) / sqrt(bc2) + eps)
// with bc1 = 1 - b1^t, bc2 = 1 - b2^t computed by the host in double precision and passed per group.
//
// dnr_adam_step_reduce (round 2) fuses the multi-GPU gradient reduction into the same pass: every rank keeps its flat
// gradient bucket and its per-Gaussian `touched` flags in NVLink-mapped symmetric memory; a Gaussian's gradient rows are
// non-zero only on the ranks whose view composited it (~10 % per view), so instead of an all-reduce of the dense bucket
// (236 MB in and out per rank and step) each element's gradient is gathered straight from the peers that touched it —
// sum over ranks in rank order, so every replica computes bit-identical updates — and consumed by the Adam update in the
// same thread.  Inbound NVLink traffic is the touched rows only (~24 MB per peer at 1 M Gaussians / 1080p), plus the few
// segments flagged dense (the min-scale regulariser makes `scales` non-zero everywhere: 12 MB per peer).
#include "common.cuh"

namespace {

struct AdamSegDev {
  float* p; const float* g; float* m; float* v;
  int64_t n;
  float step_size, bc2_sqrt, eps;  // rounded from the host's doubles, as torch rounds its python scalars
};

struct AdamLaunch {
  AdamSegDev seg[DNR_ADAM_MAX_SEGS];
  float beta2, w1, w2;  // w = 1 - beta, rounded from double as torch does
};

__device__ __forceinline__ void adam_one(float& p, float g, float& m, float& v, float w1, float b2, float w2, float step_size,
                                         float bc2_sqrt, float eps) {
  m = m + w1 * (g - m);
  v = b2 * v + w2 * g * g;
  const float denom = sqrtf(v) / bc2_sqrt + eps;  // division, as torch does
  p = p - step_size * (m / denom);
}

__global__ void __launch_bounds__(256) adam_kernel(const AdamLaunch L) {
  const AdamSegDev& s = L.seg[blockIdx.y];
  const float w1 = L.w1, b2 = L.beta2, w2 = L.w2;
  const float step_size = s.step_size, bc2_sqrt = s.bc2_sqrt, eps = s.eps;
  const int64_t n = s.n;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
  const bool vec = ((((uintptr_t)s.p | (uintptr_t)s.g | (uintptr_t)s.m | (uintptr_t)s.v) & 15) == 0);
  const int64_t n4 = vec ? (n >> 2) : 0;
  float4* p4 = reinterpret_cast<float4*>(s.p);
  const float4* g4 = reinterpret_cast<const float4*>(s.g);
  float4* m4 = reinterpret_cast<float4*>(s.m);
  float4* v4 = reinterpret_cast<float4*>(s.v);
  for (int64_t i = tid; i < n4; i += stride) {
    float4 p = p4[i], m = m4[i], v = v4[i];
    const float4 g = g4[i];
    adam_one(p.x, g.x, m.x, v.x, w1, b2, w2, step_size, bc2_sqrt, eps);
    adam_one(p.y, g.y, m.y, v.y, w1, b2, w2, step_size, bc2_sqrt, eps);
    adam_one(p.z, g.z, m.z, v.z, w1, b2, w2, step_size, bc2_sqrt, eps);
    adam_one(p.w, g.w, m.w, v.w, w1, b2, w2, step_size, bc2_sqrt, eps);
    p4[i] = p; m4[i] = m; v4[i] = v;
  }
  for (int64_t i = (n4 << 2) + tid; i < n; i += stride) {  // tail (or everything when a pointer is unaligned)
    float p = s.p[i], m = s.m[i], v = s.v[i];
    adam_one(p, s.g[i], m, v, w1, b2, w2, step_size, bc2_sqrt, eps);
    s.p[i] = p; s.m[i] = m; s.v[i] = v;
  }
}

struct PeerDev {
  const float* flat[DNR_PEER_MAX];
  const uint8_t* touched[DNR_PEER_MAX];
  int world;
};

// mask[id] = bit k set <=> rank k's view touched Gaussian id.  16 Gaussians per thread (one 16-byte load per peer).
__global__ void __launch_bounds__(256) peer_mask_kernel(const PeerDev P, int n, uint8_t* __restrict__ mask) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) * 16;
  if (i >= n) return;
  if (i + 16 <= n) {
    uint32_t m[4] = {0u, 0u, 0u, 0u};
    for (int k = 0; k < P.world; ++k) {
      const uint4 t = *reinterpret_cast<const uint4*>(P.touched[k] + i);
      const uint32_t w[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        // per byte: non-zero -> bit k
        const uint32_t nz = ((w[j] | ((w[j] & 0x7f7f7f7fu) + 0x7f7f7f7fu)) >> 7) & 0x01010101u;
        m[j] |= nz << k;
      }
    }
    *reinterpret_cast<uint4*>(mask + i) = make_uint4(m[0], m[1], m[2], m[3]);
  } else {
    for (int j = i; j < n; ++j) {
      uint32_t m = 0;
      for (int k = 0; k < P.world; ++k) m |= (P.touched[k][j] ? 1u : 0u) << k;
      mask[j] = (uint8_t)m;
    }
  }
}

struct AdamReduceLaunch {
  AdamLaunch adam;
  int dense[DNR_ADAM_MAX_SEGS];  // != 0: gather the segment's rows from every rank (see DnrAdamSeg.dense)
  int64_t off[DNR_ADAM_MAX_SEGS];  // segment offset (floats) inside every rank's flat bucket
  int32_t width[DNR_ADAM_MAX_SEGS];  // floats per Gaussian in the segment
};

// WORLD = the rank count rounded up to 2 / 4 / 8: the peer loop unrolls completely, every peer's float4 is requested with
// a predicated load BEFORE the first one is consumed (a thread otherwise pays one NVLink round trip, ~2 us, per touching
// rank in turn), and the local p / m / v loads are already in flight behind them.  Bits of ranks >= world are never set.
// WORLD = 1 is the single-GPU step over a bucket with valid flags: the mask is the bucket's own `touched` array, so the
// gradient rows of untouched Gaussians (~90 % of the bucket) are never read; p / m / v are still read and written for
// every element, and g = 0 rows still decay, exactly as in adam_kernel.
template <int WORLD>
__global__ void __launch_bounds__(256, WORLD > 4 ? 3 : (WORLD > 1 ? 4 : 5)) adam_reduce_kernel(const AdamReduceLaunch L, const PeerDev P, const uint8_t* __restrict__ mask) {
  const AdamSegDev& s = L.adam.seg[blockIdx.y];
  const float w1 = L.adam.w1, b2 = L.adam.beta2, w2 = L.adam.w2;
  const float step_size = s.step_size, bc2_sqrt = s.bc2_sqrt, eps = s.eps;
  const int64_t n = s.n, off = L.off[blockIdx.y];
  const uint32_t width = (uint32_t)L.width[blockIdx.y];
  const uint32_t all_ranks = L.dense[blockIdx.y] ? ((1u << P.world) - 1u) : 0u;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t n4 = n >> 2;  // segments start on 16-byte boundaries in every bucket (FlatGradBucket._padded)
  float4* p4 = reinterpret_cast<float4*>(s.p);
  float4* m4 = reinterpret_cast<float4*>(s.m);
  float4* v4 = reinterpret_cast<float4*>(s.v);
  for (int64_t i = tid; i < n4; i += stride) {
    // rows that a rank did not touch are exactly zero in its bucket, so the union mask of the Gaussians this float4
    // covers (up to four of them when width == 1) only decides which peers are worth reading; the sum runs in rank order
    // on every replica.  n < 2^32 (checked by the host): 32-bit divisions.
    const uint32_t e = (uint32_t)(i << 2);
    uint32_t mk = all_ranks | (uint32_t)mask[e / width] | (uint32_t)mask[(e + 1u) / width] |
                  (uint32_t)mask[(e + 2u) / width] | (uint32_t)mask[(e + 3u) / width];
    if (WORLD == 1) mk = mk != 0u;  // touched flags: any non-zero byte
    float4 p = p4[i], m = m4[i], v = v4[i];
    float4 t[WORLD];
#pragma unroll
    for (int k = 0; k < WORLD; ++k) {
      t[k] = make_float4(0.f, 0.f, 0.f, 0.f);
      if ((mk >> k) & 1u) t[k] = reinterpret_cast<const float4*>(P.flat[k] + off)[i];
    }
    float4 g = t[0];
#pragma unroll
    for (int k = 1; k < WORLD; ++k) {  // x + 0 == x: the zeros of untouched ranks do not change the rank-ordered sum
      g.x += t[k].x; g.y += t[k].y; g.z += t[k].z; g.w += t[k].w;
    }
    adam_one(p.x, g.x, m.x, v.x, w1, b2, w2, step_size, bc2_sqrt, eps);
    adam_one(p.y, g.y, m.y, v.y, w1, b2, w2, step_size, bc2_sqrt, eps);
    adam_one(p.z, g.z, m.z, v.z, w1, b2, w2, step_size, bc2_sqrt, eps);
    adam_one(p.w, g.w, m.w, v.w, w1, b2, w2, step_size, bc2_sqrt, eps);
    p4[i] = p; m4[i] = m; v4[i] = v;
  }
  for (int64_t i = (n4 << 2) + tid; i < n; i += stride) {  // tail
    uint32_t mk = all_ranks | (uint32_t)mask[(uint32_t)i / width];
    if (WORLD == 1) mk = mk != 0u;
    float g = 0.f;
    for (int k = 0; k < P.world; ++k)
      if ((mk >> k) & 1u) g += P.flat[k][off + i];
    float p = s.p[i], m = s.m[i], v = s.v[i];
    adam_one(p, g, m, v, w1, b2, w2, step_size, bc2_sqrt, eps);
    s.p[i] = p; s.m[i] = m; s.v[i] = v;
  }
}

struct GradZeroLaunch {
  float* g[DNR_ADAM_MAX_SEGS];
  int32_t width[DNR_ADAM_MAX_SEGS];
  int32_t dense[DNR_ADAM_MAX_SEGS];
  int n_segs;
};

// dnr_grad_zero: a CTA owns GZ_CHUNK consecutive Gaussians.  It reads their flags once, zeroes the float4s of each segment
// that hold a flagged Gaussian's row (all of them in a dense segment; the untouched elements a float4 shares with a flagged
// row are zero already), and only then clears the flags it read: no other CTA reads them, so there is no race.
// GZ_CHUNK is a multiple of 4, so every chunk of every segment starts on a float4.
constexpr int GZ_CHUNK = 256;

__global__ void __launch_bounds__(GZ_CHUNK) grad_zero_kernel(const GradZeroLaunch L, uint8_t* __restrict__ touched, int n) {
  __shared__ uint8_t s_f[GZ_CHUNK];
  const int tid = threadIdx.x;
  const int g0 = blockIdx.x * GZ_CHUNK;
  const int ng = min(GZ_CHUNK, n - g0);
  const uint8_t f = tid < ng ? touched[g0 + tid] : 0;
  s_f[tid] = f;
  const bool any = __syncthreads_or(f != 0);
  const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int s = 0; s < L.n_segs; ++s) {
    const bool dense = L.dense[s] != 0;
    if (!dense && !any) continue;
    const uint32_t w = (uint32_t)L.width[s];
    float4* out = reinterpret_cast<float4*>(L.g[s] + (size_t)g0 * w);
    const uint32_t n4 = ((uint32_t)ng * w + 3u) >> 2;  // the last chunk may write into the segment's zero padding
    for (uint32_t i = tid; i < n4; i += GZ_CHUNK) {
      bool hit = dense;
      if (!dense) {
        const uint32_t last = min((4u * i + 3u) / w, (uint32_t)ng - 1u);
        for (uint32_t j = (4u * i) / w; j <= last; ++j) hit |= s_f[j] != 0;
      }
      if (hit) out[i] = z;
    }
  }
  if (f) touched[g0 + tid] = 0;
}

}  // namespace

static int fill_adam_launch(const DnrAdamSeg* segs, int32_t n_segs, double beta1, double beta2, AdamLaunch& L, int64_t& longest) {
  longest = 0;
  for (int i = 0; i < n_segs; ++i) {
    const DnrAdamSeg& s = segs[i];
    if (!s.p || !s.g || !s.m || !s.v) return DNR_E_NULL;
    if (s.n <= 0 || !(s.bc1 > 0.0) || !(s.bc2_sqrt > 0.0)) return DNR_E_SIZE;
    L.seg[i] = AdamSegDev{s.p, s.g, s.m, s.v, s.n, (float)(s.lr / s.bc1), (float)s.bc2_sqrt, (float)s.eps};
    longest = s.n > longest ? s.n : longest;
  }
  L.beta2 = (float)beta2;
  L.w1 = (float)(1.0 - beta1);
  L.w2 = (float)(1.0 - beta2);
  return 0;
}

extern "C" int dnr_adam_step_reduce(const DnrAdamSeg* segs, const int32_t* widths, int32_t n_segs, double beta1, double beta2,
                                    const DnrPeerReduce* peers, void* stream) {
  if (!segs || !widths || !peers) return DNR_E_NULL;
  if (n_segs <= 0 || n_segs > DNR_ADAM_MAX_SEGS) return DNR_E_SIZE;
  if (peers->world < 1 || peers->world > DNR_PEER_MAX || peers->rank < 0 || peers->rank >= peers->world || peers->n_gauss <= 0)
    return DNR_E_SIZE;
  if (!peers->mask && peers->world > 1) return DNR_E_NULL;
  AdamReduceLaunch L;
  int64_t longest = 0;
  if (const int rc = fill_adam_launch(segs, n_segs, beta1, beta2, L.adam, longest)) return rc;
  PeerDev P;
  P.world = peers->world;
  for (int k = 0; k < peers->world; ++k) {
    if (!peers->peer_flat[k] || !peers->peer_touched[k]) return DNR_E_NULL;
    P.flat[k] = peers->peer_flat[k];
    P.touched[k] = peers->peer_touched[k];
  }
  const float* mine = peers->peer_flat[peers->rank];
  for (int i = 0; i < n_segs; ++i) {
    if (widths[i] <= 0 || segs[i].n % widths[i] != 0 || segs[i].n / widths[i] != peers->n_gauss) return DNR_E_SIZE;
    if (segs[i].n >= ((int64_t)1 << 32)) return DNR_E_SIZE;  // the kernel indexes a segment's elements with 32 bits
    L.off[i] = segs[i].g - mine;  // the gradient segment lives at the same offset in every rank's bucket
    if (L.off[i] < 0 || (L.off[i] & 3) != 0) return DNR_E_SIZE;
    if (((uintptr_t)segs[i].p | (uintptr_t)segs[i].m | (uintptr_t)segs[i].v) & 15) return DNR_E_SIZE;
    L.width[i] = widths[i];
    L.dense[i] = segs[i].dense != 0;
  }
  cudaStream_t s = (cudaStream_t)stream;
  const int n = peers->n_gauss;
  if (peers->world > 1) {
    peer_mask_kernel<<<(n / 16 + 256) / 256, 256, 0, s>>>(P, n, peers->mask);
    DNR_CHECK_LAUNCH();
  }
  int64_t blocks = (longest / 4 + 255) / 256;
  if (blocks > DNR_NUM_SMS * 8) blocks = DNR_NUM_SMS * 8;
  if (blocks < 1) blocks = 1;
  const dim3 grid((unsigned)blocks, (unsigned)n_segs);
  if (peers->world == 1) adam_reduce_kernel<1><<<grid, 256, 0, s>>>(L, P, P.touched[0]);
  else if (peers->world <= 2) adam_reduce_kernel<2><<<grid, 256, 0, s>>>(L, P, peers->mask);
  else if (peers->world <= 4) adam_reduce_kernel<4><<<grid, 256, 0, s>>>(L, P, peers->mask);
  else adam_reduce_kernel<8><<<grid, 256, 0, s>>>(L, P, peers->mask);
  DNR_CHECK_LAUNCH();
  return 0;
}

extern "C" int dnr_adam_step(const DnrAdamSeg* segs, int32_t n_segs, double beta1, double beta2, void* stream) {
  if (!segs) return DNR_E_NULL;
  if (n_segs <= 0 || n_segs > DNR_ADAM_MAX_SEGS) return DNR_E_SIZE;
  AdamLaunch L;
  int64_t longest = 0;
  if (const int rc = fill_adam_launch(segs, n_segs, beta1, beta2, L, longest)) return rc;
  // 8 resident CTAs of 256 threads per SM; short groups leave their extra CTAs idle after one bounds check
  int64_t blocks = (longest / 4 + 255) / 256;
  if (blocks > DNR_NUM_SMS * 8) blocks = DNR_NUM_SMS * 8;
  if (blocks < 1) blocks = 1;
  adam_kernel<<<dim3((unsigned)blocks, (unsigned)n_segs), 256, 0, (cudaStream_t)stream>>>(L);
  DNR_CHECK_LAUNCH();
  return 0;
}

extern "C" int dnr_grad_zero(const DnrGradSeg* segs, int32_t n_segs, uint8_t* touched, int32_t n_gauss, void* stream) {
  if (!segs || !touched) return DNR_E_NULL;
  if (n_segs <= 0 || n_segs > DNR_ADAM_MAX_SEGS || n_gauss <= 0) return DNR_E_SIZE;
  GradZeroLaunch L;
  L.n_segs = n_segs;
  for (int i = 0; i < n_segs; ++i) {
    if (!segs[i].g) return DNR_E_NULL;
    if (segs[i].width <= 0 || segs[i].width > 4096 || ((uintptr_t)segs[i].g & 15)) return DNR_E_SIZE;
    L.g[i] = segs[i].g;
    L.width[i] = segs[i].width;
    L.dense[i] = segs[i].dense;
  }
  grad_zero_kernel<<<(n_gauss + GZ_CHUNK - 1) / GZ_CHUNK, GZ_CHUNK, 0, (cudaStream_t)stream>>>(L, touched, n_gauss);
  DNR_CHECK_LAUNCH();
  return 0;
}
