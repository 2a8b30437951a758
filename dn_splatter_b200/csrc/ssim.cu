// Fused SSIM (value + gradient) for the photometric term of SplatfactoModel.get_loss_dict [EXT nerfstudio 1.1.3], which
// dn-splatter evaluates with torchmetrics' StructuralSimilarityIndexMeasure(data_range=1.0, kernel_size=11)
// (/root/reference/dn_splatter/dn_model.py:180, loss assembled at :624-628).  SURVEY.md §8f-3.
//
// torchmetrics pads by reflection, filters with an 11x11 Gaussian (sigma 1.5) and then CROPS the padding away before
// taking the mean, so only windows that lie fully inside the image contribute: mean over the (H-10)x(W-10) interior of
//   S = ((2 mx my + C1)(2 sxy + C2)) / ((mx^2 + my^2 + C1)(sx + sy + C2)),   C1 = 0.01^2, C2 = 0.03^2.
// Forward: a separable 11-tap filter (horizontal, then vertical) of {x, y, x^2, y^2, xy} over the zero-padded image;
// writes the three partial-derivative maps dS/dmx, dS/dExx, dS/dExy and reduces the SSIM sum.  Backward: the same
// separable filter applied to those maps (the transposed correlation of a symmetric kernel),
//   v_x = v * (F[dS/dmx] + 2 x F[dS/dExx] + y F[dS/dExy]) / count.
// gt may be uint8 (/255).
//
// Decomposition (both passes): a CTA owns a column strip of SS_TW = 32 output columns x one band of output rows x the <= 3
// channels of its launch; warp w is channel c0 + w and lane l is output column j0 + l.  The warp walks its strip top to
// bottom, one input row per step: the row's 42 columns (the strip plus the 5-column halo on each side) go through a
// per-warp shared row, are filtered horizontally once, and the filtered values enter an 11-row register ring; the
// vertical 11-tap filter of the ring emits one output row per step.  Every input row is read once per strip (plus the
// 10-row halo of the band), every thread works in both passes, and a CTA needs at most 1.5 KB of shared memory.  Each
// output value is the same fp32 sequence of operations as a plain per-pixel evaluation of the formulas above (taps in
// order k = 0..10, horizontal first), so the values do not depend on the decomposition; only the order of the block
// sums does.
//
// The derivative maps are scratch private to the forward / backward pair: 3 H W C floats, stored planar as
// dmaps[(q C + c) H W + i W + j] for map q in {dS/dmx, dS/dExx, dS/dExy}, so that the row walks read and write them
// coalesced.  They are zero outside the interior.
#include "common.cuh"

namespace {

constexpr int SS_R = 5;                 // window radius
constexpr int SS_K = 2 * SS_R + 1;      // taps (11): also the length of the register ring
constexpr int SS_TW = 32;               // output columns per strip: one per lane
constexpr int SS_IW = SS_TW + 2 * SS_R; // input columns per strip row (42)
// Output rows per CTA.  A band costs its 10 halo rows again, so it should be tall; and at 1920x1080 on the 132 SMs of an
// H100 the CTAs should fit on the card in one wave (a second, partial wave runs at a fraction of the occupancy and costs
// nearly as long as the first).  Both kernels are held to 80 registers, 8 CTAs (24 warps) per SM: 60 strips x 17 bands
// of 64 rows = 1020 CTAs <= 1056 resident.  (The forward's 55-value ring then spills a few loop invariants; measured,
// that is faster than 6 CTAs per SM without spills.)
constexpr int SS_BAND = 64;
constexpr int SS_MIN_CTAS = 8;
constexpr int SS_C = 3;                 // channels (warps) per CTA

// normalised 1-D Gaussian, sigma 1.5: exp(-d^2 / 4.5) / sum, evaluated in fp32 exactly as torchmetrics' _gaussian does
__constant__ float c_win[11] = {1.028380357e-03f, 7.598758209e-03f, 3.600077331e-02f, 1.093606874e-01f, 2.130055279e-01f,
                                2.660117149e-01f, 2.130055279e-01f, 1.093606874e-01f, 3.600077331e-02f, 7.598758209e-03f,
                                1.028380357e-03f};

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <bool U8>
__device__ __forceinline__ float ld_gt(const void* img, size_t idx) {
  return U8 ? __fmul_rn((float)((const uint8_t*)img)[idx], 1.0f / 255.0f) : ((const float*)img)[idx];
}

// The strip geometry of one lane: output column j, and the two input columns it stages into the shared row (ja for
// every lane, jb = ja + 32 for lanes 0..9), with validity (outside the image the input is zero).
struct StripLane {
  int j, ja, jb;
  bool va, vb;
  __device__ StripLane(int W) {
    const int lane = threadIdx.x & 31;
    j = blockIdx.x * SS_TW + lane;
    ja = j - SS_R;
    jb = ja + SS_TW;
    va = ja >= 0 && ja < W;
    vb = lane < 2 * SS_R && jb < W;
  }
};

// sum_out[0] += SSIM over the interior; with L1: sum_out[1] += |x - y| over all pixels (the parent's photometric L1 shares
// the pass: both values come from the same loads).
// NC = channels this launch handles per CTA (one warp each); c0 = first channel; band = output rows per CTA.
// METRIC (evaluation, no gradient): blockIdx.z is the image of a [B,H,W,C] batch, no dmaps are written, the second sum is
// (x - y)^2 instead of |x - y|, and sum_out is double [B,2] that receives one fp64 atomic per CTA per quantity.
template <bool U8, bool L1, int NC, bool METRIC = false>
__global__ void __launch_bounds__(32 * SS_C, SS_MIN_CTAS)
    ssim_fwd_kernel(const float* __restrict__ x, const void* __restrict__ y, int H, int W, int C, int c0, int band,
                    float* __restrict__ dmaps, float* __restrict__ sum_out) {
  __shared__ float2 s_row[NC][SS_IW];  // (x, y) of the current input row
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, c = c0 + w;
  const StripLane sl(W);
  const int i0 = blockIdx.y * band;
  const int rows = min(band, H - i0);
  const int n_in = rows + 2 * SS_R;  // input rows i0 - 5 .. i0 + rows + 4
  const long long rs = (long long)W * C, oa = (long long)sl.ja * C + c, ob = (long long)sl.jb * C + c;
  if constexpr (METRIC) {
    const size_t img = (size_t)blockIdx.z * H * W * C;
    x += img;
    y = U8 ? (const void*)((const uint8_t*)y + img) : (const void*)((const float*)y + img);
  }
  const size_t n = (size_t)H * W;
  float2 va, vb;  // the next input row's staged (x, y)
  auto load = [&](int r) {
    va = vb = make_float2(0.f, 0.f);
    if (r >= 0 && r < H) {
      const long long row = r * rs;
      if (sl.va) va = make_float2(x[row + oa], ld_gt<U8>(y, row + oa));
      if (sl.vb) vb = make_float2(x[row + ob], ld_gt<U8>(y, row + ob));
    }
  };
  float2* sw = s_row[w];
  float ring[5][SS_K];  // horizontally filtered x, y, x^2, y^2, xy of the last 11 input rows
  float ssum = 0.f, lsum = 0.f;
  load(i0 - SS_R);
  for (int t0 = 0; t0 < n_in; t0 += SS_K) {
#pragma unroll
    for (int u = 0; u < SS_K; ++u) {  // t = t0 + u: input row i0 - 5 + t goes to ring slot u
      const int t = t0 + u;
      if (t >= n_in) break;
      __syncwarp();
      sw[lane] = va;
      if (lane < 2 * SS_R) sw[SS_TW + lane] = vb;
      __syncwarp();
      if (t + 1 < n_in) load(i0 - SS_R + t + 1);
      float acc[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int k = 0; k < SS_K; ++k) {
        const float2 in = sw[lane + k];
        const float xs = in.x, ys = in.y;
        const float v[5] = {xs, ys, xs * xs, ys * ys, xs * ys};
#pragma unroll
        for (int q = 0; q < 5; ++q) acc[q] += c_win[k] * v[q];
      }
#pragma unroll
      for (int q = 0; q < 5; ++q) ring[q][u] = acc[q];
      if (t >= SS_R && t < SS_R + rows && sl.j < W) {  // the centre tap of a row of the band: the L1 / squared error
        const float2 in = sw[lane + SS_R];
        const float d = in.x - in.y;
        if constexpr (METRIC) lsum += d * d;
        else if (L1) lsum += fabsf(d);
      }
      if (t >= 2 * SS_R) {  // output row i = i0 + t - 10 from input rows t - 10 .. t = ring slots (u + 1 + k) mod 11
        float f[5];
#pragma unroll
        for (int q = 0; q < 5; ++q) {
          float a = 0.f;
#pragma unroll
          for (int k = 0; k < SS_K; ++k) a += c_win[k] * ring[q][(u + 1 + k) % SS_K];
          f[q] = a;
        }
        const int i = i0 + t - 2 * SS_R, j = sl.j;
        const bool interior = (i >= SS_R) && (i < H - SS_R) && (j >= SS_R) && (j < W - SS_R);
        float s = 0.f, d_mu = 0.f, d_xx = 0.f, d_xy = 0.f;
        if (interior) {
          const float C1 = 0.0001f, C2 = 0.0009f;
          const float mx = f[0], my = f[1];
          const float sx = f[2] - mx * mx, sy = f[3] - my * my, sxy = f[4] - mx * my;
          const float A1 = 2.f * mx * my + C1, A2 = 2.f * sxy + C2, B1 = mx * mx + my * my + C1, B2 = sx + sy + C2;
          const float inv = 1.0f / (B1 * B2);
          s = A1 * A2 * inv;
          d_xx = -s / B2;
          d_xy = 2.f * A1 * inv;
          d_mu = 2.f * my * (A2 - A1) * inv - 2.f * mx * s / B1 + 2.f * mx * s / B2;
        }
        if constexpr (!METRIC) {
          if (j < W) {
            const size_t p = (size_t)c * n + (size_t)i * W + j, plane = (size_t)C * n;
            dmaps[p] = d_mu; dmaps[plane + p] = d_xx; dmaps[2 * plane + p] = d_xy;
          }
        }
        ssum += s;
      }
    }
  }
  if constexpr (METRIC) {
    __shared__ double red_d[2][SS_C];
    const double ds = warp_sum_f64(ssum), dl = warp_sum_f64(lsum);
    if (lane == 0) { red_d[0][w] = ds; red_d[1][w] = dl; }
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = 0.0, tl = 0.0;
#pragma unroll
      for (int v = 0; v < NC; ++v) { t += red_d[0][v]; tl += red_d[1][v]; }
      double* out = reinterpret_cast<double*>(sum_out) + 2 * blockIdx.z;
      if (t != 0.0) atomicAdd(out, t);
      if (tl != 0.0) atomicAdd(out + 1, tl);
    }
    return;
  }
  __shared__ float red[2][SS_C];
  ssum = warp_sum(ssum);
  if (L1) lsum = warp_sum(lsum);
  if (lane == 0) { red[0][w] = ssum; red[1][w] = lsum; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f, tl = 0.f;
#pragma unroll
    for (int v = 0; v < NC; ++v) { t += red[0][v]; if (L1) tl += red[1][v]; }
    if (t != 0.f) atomicAdd(sum_out, t);
    if (L1 && tl != 0.f) atomicAdd(sum_out + 1, tl);
  }
}

// out[2] = (1 - lambda) * mean|x - y| + lambda * (1 - mean SSIM): SplatfactoModel.get_loss_dict's main_loss [EXT]
__global__ void photometric_finish_kernel(float* out, float lambda, float inv_count_ssim, float inv_count_l1) {
  out[2] = (1.0f - lambda) * (out[1] * inv_count_l1) + lambda * (1.0f - out[0] * inv_count_ssim);
}

// v_x = (*v_mean or 1) * (w_ssim * d(mean SSIM)/dx + w_l1 * d(mean |x - y|)/dx); the same strip walk over the maps
template <bool U8, int NC>
__global__ void __launch_bounds__(32 * SS_C, SS_MIN_CTAS)
    ssim_bwd_kernel(const float* __restrict__ x, const void* __restrict__ y, int H, int W, int C, int c0, int band,
                    const float* __restrict__ dmaps, const float* v_mean, float w_ssim, float w_l1, float* __restrict__ v_x) {
  __shared__ float s_row[NC][3][SS_IW];  // the three maps of the current input row
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, c = c0 + w;
  const StripLane sl(W);
  const int i0 = blockIdx.y * band;
  const int rows = min(band, H - i0);
  const int n_in = rows + 2 * SS_R;
  const size_t n = (size_t)H * W;
  const float* maps[3] = {dmaps + (size_t)c * n, dmaps + ((size_t)C + c) * n, dmaps + ((size_t)2 * C + c) * n};
  float ma[3], mb[3];
  auto load = [&](int r) {  // outside the image: zero (inside, the forward wrote zeros outside the interior)
#pragma unroll
    for (int q = 0; q < 3; ++q) ma[q] = mb[q] = 0.f;
    if (r >= 0 && r < H) {
      const size_t row = (size_t)r * W;
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        if (sl.va) ma[q] = maps[q][row + sl.ja];
        if (sl.vb) mb[q] = maps[q][row + sl.jb];
      }
    }
  };
  const float count = (float)(H - 2 * SS_R) * (float)(W - 2 * SS_R) * (float)C;
  const float vm = v_mean ? __ldg(v_mean) : 1.0f;
  const float gsc = vm * w_ssim / count;
  const float gl1 = vm * w_l1 / ((float)H * (float)W * (float)C);
  float ring[3][SS_K];
  load(i0 - SS_R);
  for (int t0 = 0; t0 < n_in; t0 += SS_K) {
#pragma unroll
    for (int u = 0; u < SS_K; ++u) {
      const int t = t0 + u;
      if (t >= n_in) break;
      const int i = i0 + t - 2 * SS_R, j = sl.j;
      const bool emit = t >= 2 * SS_R && j < W;
      float xv = 0.f, yv = 0.f;
      size_t p = 0;
      if (emit) {  // issued before the filter so that its latency hides under it
        p = ((size_t)i * W + j) * C + c;
        xv = x[p];
        yv = ld_gt<U8>(y, p);
      }
      __syncwarp();
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        s_row[w][q][lane] = ma[q];
        if (lane < 2 * SS_R) s_row[w][q][SS_TW + lane] = mb[q];
      }
      __syncwarp();
      if (t + 1 < n_in) load(i0 - SS_R + t + 1);
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        float a = 0.f;
#pragma unroll
        for (int k = 0; k < SS_K; ++k) a += c_win[k] * s_row[w][q][lane + k];
        ring[q][u] = a;
      }
      if (t >= 2 * SS_R) {
        float f[3];
#pragma unroll
        for (int q = 0; q < 3; ++q) {
          float a = 0.f;
#pragma unroll
          for (int k = 0; k < SS_K; ++k) a += c_win[k] * ring[q][(u + 1 + k) % SS_K];
          f[q] = a;
        }
        if (emit) {
          const float d = xv - yv;
          v_x[p] = gsc * (f[0] + 2.f * xv * f[1] + yv * f[2]) + gl1 * ((d > 0.f) ? 1.f : ((d < 0.f) ? -1.f : 0.f));
        }
      }
    }
  }
}

}  // namespace

// One launch per group of up to three channels (C = 3: a single launch).
template <bool L1>
static int launch_ssim_fwd(const float* pred, const void* gt, int gt_is_u8, int H, int W, int C, float* dmaps, float* out, cudaStream_t s) {
  const dim3 grid((W + SS_TW - 1) / SS_TW, (H + SS_BAND - 1) / SS_BAND, 1);
  for (int c0 = 0; c0 < C; c0 += SS_C) {
    const int nc = C - c0 < SS_C ? C - c0 : SS_C;
#define DNR_SSIM_FWD(U8, NC) ssim_fwd_kernel<U8, L1, NC><<<grid, 32 * NC, 0, s>>>(pred, gt, H, W, C, c0, SS_BAND, dmaps, out)
    if (gt_is_u8) { if (nc == 3) DNR_SSIM_FWD(true, 3); else if (nc == 2) DNR_SSIM_FWD(true, 2); else DNR_SSIM_FWD(true, 1); }
    else { if (nc == 3) DNR_SSIM_FWD(false, 3); else if (nc == 2) DNR_SSIM_FWD(false, 2); else DNR_SSIM_FWD(false, 1); }
#undef DNR_SSIM_FWD
    DNR_CHECK_LAUNCH();
  }
  return 0;
}

static int launch_ssim_bwd(const float* pred, const void* gt, int gt_is_u8, int H, int W, int C, const float* dmaps, const float* v,
                           float w_ssim, float w_l1, float* v_pred, cudaStream_t s) {
  const dim3 grid((W + SS_TW - 1) / SS_TW, (H + SS_BAND - 1) / SS_BAND, 1);
  for (int c0 = 0; c0 < C; c0 += SS_C) {
    const int nc = C - c0 < SS_C ? C - c0 : SS_C;
#define DNR_SSIM_BWD(U8, NC) ssim_bwd_kernel<U8, NC><<<grid, 32 * NC, 0, s>>>(pred, gt, H, W, C, c0, SS_BAND, dmaps, v, w_ssim, w_l1, \
                                                                              v_pred)
    if (gt_is_u8) { if (nc == 3) DNR_SSIM_BWD(true, 3); else if (nc == 2) DNR_SSIM_BWD(true, 2); else DNR_SSIM_BWD(true, 1); }
    else { if (nc == 3) DNR_SSIM_BWD(false, 3); else if (nc == 2) DNR_SSIM_BWD(false, 2); else DNR_SSIM_BWD(false, 1); }
#undef DNR_SSIM_BWD
    DNR_CHECK_LAUNCH();
  }
  return 0;
}

// pred: [B,H,W,C] fp32; gt: [B,H,W,C] fp32, or uint8 read as value / 255 when gt_is_u8 != 0.  out [B,2] double, zeroed by
// the call: per image the SSIM sum over the (H-10)(W-10)C interior and the sum of squared errors over all H W C values.
extern "C" int dnr_rgb_metrics(const float* pred, const void* gt, int32_t gt_is_u8, int32_t B, int32_t H, int32_t W, int32_t C,
                               double* out, void* stream) {
  if (!pred || !gt || !out) return DNR_E_NULL;
  if (B <= 0 || B > 65535 || H <= 2 * SS_R || W <= 2 * SS_R || C <= 0) return DNR_E_SIZE;
  cudaStream_t s = (cudaStream_t)stream;
  DNR_CUDA(cudaMemsetAsync(out, 0, 2 * (size_t)B * sizeof(double), s));
  const dim3 grid((W + SS_TW - 1) / SS_TW, (H + SS_BAND - 1) / SS_BAND, B);
  float* o = reinterpret_cast<float*>(out);
  for (int c0 = 0; c0 < C; c0 += SS_C) {
    const int nc = C - c0 < SS_C ? C - c0 : SS_C;
#define DNR_SSIM_MET(U8, NC) ssim_fwd_kernel<U8, false, NC, true><<<grid, 32 * NC, 0, s>>>(pred, gt, H, W, C, c0, SS_BAND, nullptr, o)
    if (gt_is_u8) { if (nc == 3) DNR_SSIM_MET(true, 3); else if (nc == 2) DNR_SSIM_MET(true, 2); else DNR_SSIM_MET(true, 1); }
    else { if (nc == 3) DNR_SSIM_MET(false, 3); else if (nc == 2) DNR_SSIM_MET(false, 2); else DNR_SSIM_MET(false, 1); }
#undef DNR_SSIM_MET
    DNR_CHECK_LAUNCH();
  }
  return 0;
}

// pred: [H,W,C] fp32; gt: [H,W,C] fp32, or uint8 scaled by 1/255 when gt_is_u8 != 0.  dmaps: 3 H W C floats of scratch
// kept for the backward (layout: the header of this file).  *sum_out (zeroed by the call) receives the SUM of the SSIM map over the interior; the caller divides by
// (H-10)(W-10)C.
extern "C" int dnr_ssim_fwd_ex(const float* pred, const void* gt, int32_t gt_is_u8, int32_t H, int32_t W, int32_t C, float* dmaps,
                               float* sum_out, void* stream) {
  if (!pred || !gt || !dmaps || !sum_out) return DNR_E_NULL;
  if (H <= 2 * SS_R || W <= 2 * SS_R || C <= 0) return DNR_E_SIZE;
  cudaStream_t s = (cudaStream_t)stream;
  DNR_CUDA(cudaMemsetAsync(sum_out, 0, sizeof(float), s));
  return launch_ssim_fwd<false>(pred, gt, gt_is_u8, H, W, C, dmaps, sum_out, s);
}

// The whole photometric term of SplatfactoModel.get_loss_dict in one pass each way:
//   main = (1 - ssim_lambda) * mean|pred - gt| + ssim_lambda * (1 - mean SSIM)        (dn_model.py:624-628 -> parent [EXT])
// out (3 floats, zeroed by the call): [0] SSIM sum over the interior, [1] sum |pred - gt|, [2] main.
extern "C" int dnr_photometric_fwd(const float* pred, const void* gt, int32_t gt_is_u8, int32_t H, int32_t W, int32_t C,
                                   float ssim_lambda, float* dmaps, float* out, void* stream) {
  if (!pred || !gt || !dmaps || !out) return DNR_E_NULL;
  if (H <= 2 * SS_R || W <= 2 * SS_R || C <= 0) return DNR_E_SIZE;
  cudaStream_t s = (cudaStream_t)stream;
  DNR_CUDA(cudaMemsetAsync(out, 0, 3 * sizeof(float), s));
  if (const int rc = launch_ssim_fwd<true>(pred, gt, gt_is_u8, H, W, C, dmaps, out, s)) return rc;
  photometric_finish_kernel<<<1, 1, 0, s>>>(out, ssim_lambda, 1.0f / ((float)(H - 2 * SS_R) * (float)(W - 2 * SS_R) * (float)C),
                                            1.0f / ((float)H * (float)W * (float)C));
  DNR_CHECK_LAUNCH();
  return 0;
}

// v_pred[H,W,C] = (*v_main or 1) * d(main)/d(pred): the SSIM and the L1 gradient written by one kernel.
extern "C" int dnr_photometric_bwd(const float* pred, const void* gt, int32_t gt_is_u8, int32_t H, int32_t W, int32_t C,
                                   float ssim_lambda, const float* dmaps, const float* v_main, float* v_pred, void* stream) {
  if (!pred || !gt || !dmaps || !v_pred) return DNR_E_NULL;
  if (H <= 2 * SS_R || W <= 2 * SS_R || C <= 0) return DNR_E_SIZE;
  return launch_ssim_bwd(pred, gt, gt_is_u8, H, W, C, dmaps, v_main, -ssim_lambda, 1.0f - ssim_lambda, v_pred, (cudaStream_t)stream);
}

// v_pred[H,W,C] = (*v_mean or 1) * d(mean SSIM)/d(pred).
extern "C" int dnr_ssim_bwd_ex(const float* pred, const void* gt, int32_t gt_is_u8, int32_t H, int32_t W, int32_t C,
                               const float* dmaps, const float* v_mean, float* v_pred, void* stream) {
  if (!pred || !gt || !dmaps || !v_pred) return DNR_E_NULL;
  if (H <= 2 * SS_R || W <= 2 * SS_R || C <= 0) return DNR_E_SIZE;
  return launch_ssim_bwd(pred, gt, gt_is_u8, H, W, C, dmaps, v_mean, 1.0f, 0.0f, v_pred, (cudaStream_t)stream);
}

extern "C" int dnr_ssim_fwd(const float* pred, const float* gt, int32_t H, int32_t W, int32_t C, float* dmaps, float* sum_out,
                            void* stream) {
  return dnr_ssim_fwd_ex(pred, gt, 0, H, W, C, dmaps, sum_out, stream);
}

extern "C" int dnr_ssim_bwd(const float* pred, const float* gt, int32_t H, int32_t W, int32_t C, const float* dmaps,
                            const float* v_mean, float* v_pred, void* stream) {
  return dnr_ssim_bwd_ex(pred, gt, 0, H, W, C, dmaps, v_mean, v_pred, stream);
}
