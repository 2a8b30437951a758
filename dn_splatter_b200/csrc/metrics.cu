// Evaluation metrics of renders (DNSplatterModel.get_metrics_dict / get_image_metrics_and_images): the depth and normal
// reductions of dn_splatter/metrics.py's DepthMetrics and NormalMetrics.  PSNR / SSIM live in ssim.cu (dnr_rgb_metrics).
//
// Compiled with -fmad=false: every per-element fp32 value a decision rests on (the depth ratio, the clamped normal dot,
// |g - p| that the median selects) is the plain IEEE sequence the fp64 oracle restates (oracle/metrics_ref.py).  The
// sums themselves are formed in fp64 from the fp32 inputs and added with one fp64 atomic per CTA per quantity.
#include "common.cuh"

namespace {

constexpr int MT_NT = 256;
constexpr int MT_RADIX_BITS = 8;
constexpr int MT_BINS = 1 << MT_RADIX_BITS;

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Sums NQ per-thread values over the CTA and adds each non-zero total to out[q * stride] (one fp64 atomic per quantity).
template <int NQ>
__device__ __forceinline__ void block_add(double (&v)[NQ], double* out, int stride) {
  __shared__ double red[NQ][MT_NT / 32];
  const int tid = threadIdx.x;
#pragma unroll
  for (int q = 0; q < NQ; ++q) {
    const double w = warp_sum_d(v[q]);
    if ((tid & 31) == 0) red[q][tid >> 5] = w;
  }
  __syncthreads();
  if (tid < NQ) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < MT_NT / 32; ++w) t += red[tid][w];
    if (t != 0.0) atomicAdd(out + tid * stride, t);
  }
}

// DepthMetrics over n pooled elements; out[9] as documented at dnr_depth_metrics.
__global__ void __launch_bounds__(MT_NT) depth_metrics_kernel(const float* __restrict__ pred, const float* __restrict__ gt,
                                                              int64_t n, float tol, double* __restrict__ out) {
  double v[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int64_t i = (int64_t)blockIdx.x * MT_NT + threadIdx.x; i < n; i += (int64_t)gridDim.x * MT_NT) {
    const float g = gt[i], p = pred[i];
    if (!(g > tol)) continue;
    // torch.max propagates NaN; fmaxf would not
    const float r0 = g / p, r1 = p / g;
    const float t = (r0 != r0 || r1 != r1) ? __int_as_float(0x7fc00000) : fmaxf(r0, r1);
    v[0] += 1.0;
    v[1] += (t < 1.25f) ? 1.0 : 0.0;
    v[2] += (t < 1.5625f) ? 1.0 : 0.0;
    v[3] += (t < 1.953125f) ? 1.0 : 0.0;
    const double gd = g, d = gd - (double)p;
    v[4] += d * d;
    v[5] += fabs(d) / gd;
    v[6] += d * d / gd;
    const double l = fabs(log(gd) - log((double)p));  // sqrt((log g - log p)^2)
    if (l == l) { v[7] += l; v[8] += 1.0; }
  }
  block_add<9>(v, out, 1);
}

// Median state after the header: hist[MT_BINS] (counts of the current digit among the keys that match the prefix),
// then {prefix of the selected key, rank still to skip inside the prefix}.
struct MedianState {
  unsigned long long hist[MT_BINS];
  unsigned long long rank;
  unsigned int prefix;
  unsigned int pad;
};

template <bool U8>
__device__ __forceinline__ float ld_target(const void* img, size_t idx) {
  return U8 ? __fmul_rn((float)((const uint8_t*)img)[idx], 1.0f / 255.0f) : ((const float*)img)[idx];
}

// One pass of the radix select over key = bits(|g - p|) (order-preserving: the values are >= 0), recomputed from the
// inputs.  Pass 0 also adds the per-image sums: out[3b] sum acos(clamp(dot)), out[3b+1] sum (g-p)^2, out[3b+2] sum |g-p|.
template <bool U8, bool FIRST>
__global__ void __launch_bounds__(MT_NT) normal_pass_kernel(const float* __restrict__ pred, const void* __restrict__ gt, int HW,
                                                            int shift, MedianState* __restrict__ st, double* __restrict__ out) {
  __shared__ unsigned int hist[MT_BINS];
  for (int b = threadIdx.x; b < MT_BINS; b += MT_NT) hist[b] = 0u;
  __syncthreads();
  const unsigned int prefix = FIRST ? 0u : st->prefix;
  const size_t img = (size_t)blockIdx.y * HW;
  double v[3] = {0.0, 0.0, 0.0};
  for (int i = blockIdx.x * MT_NT + threadIdx.x; i < HW; i += gridDim.x * MT_NT) {
    const size_t e = (img + i) * 3;
    float g[3], p[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) { g[c] = ld_target<U8>(gt, e + c); p[c] = pred[e + c]; }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const unsigned int key = __float_as_uint(fabsf(g[c] - p[c]));
      if (FIRST || (key >> (shift + MT_RADIX_BITS)) == prefix) atomicAdd(&hist[(key >> shift) & (MT_BINS - 1)], 1u);
    }
    if (FIRST) {
      const float dot = (g[0] * p[0] + g[1] * p[1]) + g[2] * p[2];
      v[0] += acos((double)fminf(fmaxf(dot, -1.0f), 1.0f));
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const double d = (double)g[c] - (double)p[c];
        v[1] += d * d;
        v[2] += fabs(d);
      }
    }
  }
  __syncthreads();
  for (int b = threadIdx.x; b < MT_BINS; b += MT_NT)
    if (hist[b]) atomicAdd(&st->hist[b], (unsigned long long)hist[b]);
  if (FIRST) block_add<3>(v, out + 3 * blockIdx.y, 1);
}

// Narrows the selection to the bin that holds the remaining rank and clears the histogram for the next pass; after the
// last pass the prefix is the key of the selected element.
__global__ void median_select_kernel(MedianState* st, unsigned long long first_rank, int last, double* median_out) {
  __shared__ unsigned int sel;
  if (threadIdx.x == 0) {
    unsigned long long k = first_rank != ~0ull ? first_rank : st->rank, below = 0;
    int b = 0;
    for (; b < MT_BINS - 1 && below + st->hist[b] <= k; ++b) below += st->hist[b];
    st->rank = k - below;
    sel = (first_rank != ~0ull ? 0u : st->prefix << MT_RADIX_BITS) | (unsigned int)b;
    st->prefix = sel;
    if (last) *median_out = (double)__uint_as_float(sel);
  }
  __syncthreads();
  for (int b = threadIdx.x; b < MT_BINS; b += blockDim.x) st->hist[b] = 0ull;
}

int stream_grid(int64_t work, int cap) {
  const int64_t g = (work + MT_NT - 1) / MT_NT;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace

// Sums of DepthMetrics over n pooled elements, out[9] double (zeroed by the call), over the elements with gt > tolerance:
// [0] count, [1..3] count of thresh < 1.25, 1.25^2, 1.25^3 with thresh = max(gt/pred, pred/gt) in fp32 (NaN if either
// ratio is), [4] sum (gt-pred)^2, [5] sum |gt-pred|/gt, [6] sum (gt-pred)^2/gt, [7] sum |log gt - log pred| over the
// non-NaN terms, [8] the number of those terms.
extern "C" int dnr_depth_metrics(const float* pred, const float* gt, int64_t n, float tolerance, double* out, void* stream) {
  if (!pred || !gt || !out) return DNR_E_NULL;
  if (n <= 0) return DNR_E_SIZE;
  cudaStream_t s = (cudaStream_t)stream;
  DNR_CUDA(cudaMemsetAsync(out, 0, 9 * sizeof(double), s));
  depth_metrics_kernel<<<stream_grid(n, 4 * DNR_NUM_SMS), MT_NT, 0, s>>>(pred, gt, n, tolerance, out);
  DNR_CHECK_LAUNCH();
  return 0;
}

extern "C" int64_t dnr_normal_metrics_workspace_bytes(int32_t B, int32_t H, int32_t W) {
  if (B <= 0 || H <= 0 || W <= 0) return DNR_E_SIZE;
  return (int64_t)sizeof(MedianState);
}

// pred, gt: [B,H,W,3] (gt fp32, or uint8 read as value / 255 when gt_is_u8 != 0).  out[3B+1] double (zeroed by the call):
// per image b, [3b] sum acos(clamp((g0 p0 + g1 p1) + g2 p2, -1, 1)), [3b+1] sum (g-p)^2, [3b+2] sum |g-p|; [3B] the lower
// median of |g - p| over all B*3*H*W values (the element of rank (N-1)/2, as torch.median returns it).
extern "C" int dnr_normal_metrics(const float* pred, const void* gt, int32_t gt_is_u8, int32_t B, int32_t H, int32_t W, void* ws,
                                  int64_t ws_bytes, double* out, void* stream) {
  if (!pred || !gt || !ws || !out) return DNR_E_NULL;
  if (B <= 0 || B > 65535 || H <= 0 || W <= 0 || (int64_t)H * W > INT32_MAX / 3) return DNR_E_SIZE;
  if (ws_bytes < (int64_t)sizeof(MedianState)) return DNR_E_WORKSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  MedianState* st = (MedianState*)ws;
  DNR_CUDA(cudaMemsetAsync(out, 0, (3 * (size_t)B + 1) * sizeof(double), s));
  DNR_CUDA(cudaMemsetAsync(st, 0, sizeof(MedianState), s));
  const int HW = H * W;
  const int bx = stream_grid(HW, (8 * DNR_NUM_SMS + B - 1) / B);
  const dim3 grid(bx, B);
  const unsigned long long n = 3ull * B * HW;
  for (int pass = 0; pass < 32 / MT_RADIX_BITS; ++pass) {
    const int shift = 32 - MT_RADIX_BITS * (pass + 1);
    if (pass == 0) {
      if (gt_is_u8) normal_pass_kernel<true, true><<<grid, MT_NT, 0, s>>>(pred, gt, HW, shift, st, out);
      else normal_pass_kernel<false, true><<<grid, MT_NT, 0, s>>>(pred, gt, HW, shift, st, out);
    } else {
      if (gt_is_u8) normal_pass_kernel<true, false><<<grid, MT_NT, 0, s>>>(pred, gt, HW, shift, st, out);
      else normal_pass_kernel<false, false><<<grid, MT_NT, 0, s>>>(pred, gt, HW, shift, st, out);
    }
    DNR_CHECK_LAUNCH();
    median_select_kernel<<<1, MT_BINS, 0, s>>>(st, pass == 0 ? (n - 1) / 2 : ~0ull, shift == 0, out + 3 * (size_t)B);
    DNR_CHECK_LAUNCH();
  }
  return 0;
}
