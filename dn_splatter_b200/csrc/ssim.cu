// Fused SSIM (value + gradient) for the photometric term of SplatfactoModel.get_loss_dict [EXT nerfstudio 1.1.3], which
// dn-splatter evaluates with torchmetrics' StructuralSimilarityIndexMeasure(data_range=1.0, kernel_size=11)
// (/root/reference/dn_splatter/dn_model.py:180, loss assembled at :624-628).  SURVEY.md §8f-3.
//
// torchmetrics pads by reflection, filters with an 11x11 Gaussian (sigma 1.5) and then CROPS the padding away before
// taking the mean, so only windows that lie fully inside the image contribute: mean over the (H-10)x(W-10) interior of
//   S = ((2 mx my + C1)(2 sxy + C2)) / ((mx^2 + my^2 + C1)(sx + sy + C2)),   C1 = 0.01^2, C2 = 0.03^2.
// Forward: one CTA per 16x16 output tile and up to three channels; the 26x26 halo of pred / gt goes to shared memory
// (rows of the interleaved [H,W,C] image are read contiguously), then a separable 11-tap filter of {x, y, x^2, y^2, xy};
// writes the three partial-derivative maps dS/dmx, dS/dExx, dS/dExy and block-reduces the SSIM sum.  Backward: the same
// separable filter applied to those maps (the transposed correlation of a symmetric kernel),
//   v_x = v * (F[dS/dmx] + 2 x F[dS/dExx] + y F[dS/dExy]) / count.
// Round 2: both passes are register-blocked (a thread filters 2 adjacent columns / 4 adjacent rows from one sliding
// window of loaded values), which cuts the shared-memory instructions per output 3.5x — the round-1 kernel issued one
// LDS per FMA and was bound by the load/store unit, not by arithmetic or HBM.  gt may be uint8 (/255).
#include "common.cuh"

namespace {

constexpr int SS_R = 5;                 // window radius
constexpr int SS_T = 16;                // output tile
constexpr int SS_H = SS_T + 2 * SS_R;   // halo tile edge (26)
constexpr int SS_P = 28;                // padded halo row (floats): 8-byte aligned pairs
constexpr int SS_C = 3;                 // channels per CTA
constexpr int SS_NT = 256;

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

// Horizontal pass: s_in[q][c][r][0..25] -> s_mid[q][c][r][0..15] for the NQ_OUT quantities `make` derives from the NQ_IN
// loaded ones.  One work item = (channel, halo row, pair of adjacent output columns): 12 loaded values per input quantity.
template <int NQ_IN, int NQ_OUT, int NC, typename Make>
__device__ __forceinline__ void hpass(float (*s_in)[SS_C][SS_H][SS_P], float (*s_mid)[SS_C][SS_H][SS_T], int tid, Make make) {
  constexpr int items = NC * SS_H * (SS_T / 2);
  for (int it = tid; it < items; it += SS_NT) {
    const int seg = it % (SS_T / 2), r = (it / (SS_T / 2)) % SS_H, c = it / ((SS_T / 2) * SS_H);
    float in[NQ_IN][12];
#pragma unroll
    for (int q = 0; q < NQ_IN; ++q) {
      const float2* p = reinterpret_cast<const float2*>(&s_in[q][c][r][2 * seg]);
#pragma unroll
      for (int k = 0; k < 6; ++k) { const float2 v = p[k]; in[q][2 * k] = v.x; in[q][2 * k + 1] = v.y; }
    }
    float acc[NQ_OUT][2];
#pragma unroll
    for (int q = 0; q < NQ_OUT; ++q) acc[q][0] = acc[q][1] = 0.f;
#pragma unroll
    for (int k = 0; k < 12; ++k) {
      float v[NQ_OUT];
      float src[NQ_IN];
#pragma unroll
      for (int q = 0; q < NQ_IN; ++q) src[q] = in[q][k];
      make(src, v);
#pragma unroll
      for (int q = 0; q < NQ_OUT; ++q) {
        if (k < 11) acc[q][0] += c_win[k] * v[q];
        if (k > 0) acc[q][1] += c_win[k - 1] * v[q];
      }
    }
#pragma unroll
    for (int q = 0; q < NQ_OUT; ++q) *reinterpret_cast<float2*>(&s_mid[q][c][r][2 * seg]) = make_float2(acc[q][0], acc[q][1]);
  }
}

// Vertical pass for one work item (channel c, column col, rows 4g .. 4g+3): out[q][o].
template <int NQ>
__device__ __forceinline__ void vpass(float (*s_mid)[SS_C][SS_H][SS_T], int c, int col, int g, float out[NQ][4]) {
#pragma unroll
  for (int q = 0; q < NQ; ++q) {
    float v[14];
#pragma unroll
    for (int j = 0; j < 14; ++j) v[j] = s_mid[q][c][4 * g + j][col];
#pragma unroll
    for (int o = 0; o < 4; ++o) {
      float acc = 0.f;
#pragma unroll
      for (int k = 0; k < 11; ++k) acc += c_win[k] * v[o + k];
      out[q][o] = acc;
    }
  }
}

// sum_out[0] += SSIM over the interior; with L1: sum_out[1] += |x - y| over all pixels (the parent's photometric L1 shares
// the pass: both values come from the same loads)
// NC = channels this launch handles per CTA (compile time: the index arithmetic of the halo load and of the work-item
// loops is mul-shift instead of runtime integer division, which cost a third of the round-2a kernel's instructions);
// c0 = first channel.
// METRIC (evaluation, no gradient): blockIdx.z is the image of a [B,H,W,C] batch, no dmaps are written, the second sum is
// (x - y)^2 instead of |x - y|, and sum_out is double [B,2] that receives one fp64 atomic per CTA per quantity.
template <bool U8, bool L1, int NC, bool METRIC = false>
__global__ void __launch_bounds__(SS_NT) ssim_fwd_kernel(const float* __restrict__ x, const void* __restrict__ y, int H, int W,
                                                        int C, int c0, float* __restrict__ dmaps, float* __restrict__ sum_out) {
  __shared__ __align__(16) float s_in[2][SS_C][SS_H][SS_P];
  __shared__ __align__(16) float s_mid[5][SS_C][SS_H][SS_T];
  __shared__ float red[SS_NT / 32];
  __shared__ float red_l1[SS_NT / 32];
  const int tid = threadIdx.x;
  constexpr int nc = NC;
  const int i0 = blockIdx.y * SS_T - SS_R, j0 = blockIdx.x * SS_T - SS_R;
  if constexpr (METRIC) {
    const size_t img = (size_t)blockIdx.z * H * W * C;
    x += img;
    y = U8 ? (const void*)((const uint8_t*)y + img) : (const void*)((const float*)y + img);
  }
  // halo load: consecutive threads walk (column, channel) of one image row -> contiguous global addresses
  for (int e = tid; e < SS_H * SS_H * NC; e += SS_NT) {
    const int c = e % NC, q = (e / NC) % SS_H, r = e / (NC * SS_H);
    const int i = i0 + r, j = j0 + q;
    float xv = 0.f, yv = 0.f;
    if (i >= 0 && i < H && j >= 0 && j < W) {
      const size_t p = ((size_t)i * W + j) * C + c0 + c;
      xv = x[p];
      yv = ld_gt<U8>(y, p);
    }
    s_in[0][c][r][q] = xv;
    s_in[1][c][r][q] = yv;
  }
  __syncthreads();
  hpass<2, 5, NC>(s_in, s_mid, tid, [](const float* s, float* v) {
    v[0] = s[0]; v[1] = s[1]; v[2] = s[0] * s[0]; v[3] = s[1] * s[1]; v[4] = s[0] * s[1];
  });
  __syncthreads();
  float ssum = 0.f, lsum = 0.f;
  if (tid < nc * SS_T * 4) {
    const int col = tid % SS_T, g = (tid / SS_T) % 4, c = tid / (SS_T * 4);
    float f[5][4];
    vpass<5>(s_mid, c, col, g, f);
    const int j = blockIdx.x * SS_T + col;
    const size_t n = (size_t)H * W * C;
#pragma unroll
    for (int o = 0; o < 4; ++o) {
      const int i = blockIdx.y * SS_T + 4 * g + o;
      const bool interior = (i >= SS_R) && (i < H - SS_R) && (j >= SS_R) && (j < W - SS_R);
      float s = 0.f, d_mu = 0.f, d_xx = 0.f, d_xy = 0.f;
      if (interior) {
        const float C1 = 0.0001f, C2 = 0.0009f;
        const float mx = f[0][o], my = f[1][o];
        const float sx = f[2][o] - mx * mx, sy = f[3][o] - my * my, sxy = f[4][o] - mx * my;
        const float A1 = 2.f * mx * my + C1, A2 = 2.f * sxy + C2, B1 = mx * mx + my * my + C1, B2 = sx + sy + C2;
        const float inv = 1.0f / (B1 * B2);
        s = A1 * A2 * inv;
        d_xx = -s / B2;
        d_xy = 2.f * A1 * inv;
        d_mu = 2.f * my * (A2 - A1) * inv - 2.f * mx * s / B1 + 2.f * mx * s / B2;
      }
      if (i < H && j < W) {
        const size_t p = ((size_t)i * W + j) * C + c0 + c;
        if constexpr (METRIC) {
          const float d = s_in[0][c][4 * g + o + SS_R][col + SS_R] - s_in[1][c][4 * g + o + SS_R][col + SS_R];
          lsum += d * d;
        } else {
          dmaps[p] = d_mu; dmaps[n + p] = d_xx; dmaps[2 * n + p] = d_xy;
          if (L1) lsum += fabsf(s_in[0][c][4 * g + o + SS_R][col + SS_R] - s_in[1][c][4 * g + o + SS_R][col + SS_R]);
        }
      }
      ssum += s;
    }
  }
  if constexpr (METRIC) {
    __shared__ double red_d[2][SS_NT / 32];
    const double ds = warp_sum_f64(ssum), dl = warp_sum_f64(lsum);
    if ((tid & 31) == 0) { red_d[0][tid >> 5] = ds; red_d[1][tid >> 5] = dl; }
    __syncthreads();
    if (tid == 0) {
      double t = 0.0, tl = 0.0;
#pragma unroll
      for (int w = 0; w < SS_NT / 32; ++w) { t += red_d[0][w]; tl += red_d[1][w]; }
      double* out = reinterpret_cast<double*>(sum_out) + 2 * blockIdx.z;
      if (t != 0.0) atomicAdd(out, t);
      if (tl != 0.0) atomicAdd(out + 1, tl);
    }
    return;
  }
  ssum = warp_sum(ssum);
  if (L1) lsum = warp_sum(lsum);
  if ((tid & 31) == 0) { red[tid >> 5] = ssum; if (L1) red_l1[tid >> 5] = lsum; }
  __syncthreads();
  if (tid == 0) {
    float t = 0.f, tl = 0.f;
#pragma unroll
    for (int w = 0; w < SS_NT / 32; ++w) { t += red[w]; if (L1) tl += red_l1[w]; }
    if (t != 0.f) atomicAdd(sum_out, t);
    if (L1 && tl != 0.f) atomicAdd(sum_out + 1, tl);
  }
}

// out[2] = (1 - lambda) * mean|x - y| + lambda * (1 - mean SSIM): SplatfactoModel.get_loss_dict's main_loss [EXT]
__global__ void photometric_finish_kernel(float* out, float lambda, float inv_count_ssim, float inv_count_l1) {
  out[2] = (1.0f - lambda) * (out[1] * inv_count_l1) + lambda * (1.0f - out[0] * inv_count_ssim);
}

// v_x = (*v_mean or 1) * (w_ssim * d(mean SSIM)/dx + w_l1 * d(mean |x - y|)/dx)
template <bool U8, int NC>
__global__ void __launch_bounds__(SS_NT) ssim_bwd_kernel(const float* __restrict__ x, const void* __restrict__ y, int H, int W,
                                                        int C, int c0, const float* __restrict__ dmaps, const float* v_mean,
                                                        float w_ssim, float w_l1, float* __restrict__ v_x) {
  __shared__ __align__(16) float s_in[3][SS_C][SS_H][SS_P];
  __shared__ __align__(16) float s_mid[3][SS_C][SS_H][SS_T];
  const int tid = threadIdx.x;
  constexpr int nc = NC;
  const int i0 = blockIdx.y * SS_T - SS_R, j0 = blockIdx.x * SS_T - SS_R;
  const size_t n = (size_t)H * W * C;
  for (int e = tid; e < SS_H * SS_H * NC; e += SS_NT) {
    const int c = e % NC, q = (e / NC) % SS_H, r = e / (NC * SS_H);
    const int i = i0 + r, j = j0 + q;
    // the maps are zero outside the interior by construction (forward wrote zeros there); outside the image: zero
    float a = 0.f, b = 0.f, d = 0.f;
    if (i >= 0 && i < H && j >= 0 && j < W) {
      const size_t p = ((size_t)i * W + j) * C + c0 + c;
      a = dmaps[p]; b = dmaps[n + p]; d = dmaps[2 * n + p];
    }
    s_in[0][c][r][q] = a; s_in[1][c][r][q] = b; s_in[2][c][r][q] = d;
  }
  __syncthreads();
  hpass<3, 3, NC>(s_in, s_mid, tid, [](const float* s, float* v) { v[0] = s[0]; v[1] = s[1]; v[2] = s[2]; });
  __syncthreads();
  if (tid < nc * SS_T * 4) {
    const int col = tid % SS_T, g = (tid / SS_T) % 4, c = tid / (SS_T * 4);
    float f[3][4];
    vpass<3>(s_mid, c, col, g, f);
    const int j = blockIdx.x * SS_T + col;
    const float count = (float)(H - 2 * SS_R) * (float)(W - 2 * SS_R) * (float)C;
    const float vm = v_mean ? __ldg(v_mean) : 1.0f;
    const float gsc = vm * w_ssim / count;
    const float gl1 = vm * w_l1 / ((float)H * (float)W * (float)C);
#pragma unroll
    for (int o = 0; o < 4; ++o) {
      const int i = blockIdx.y * SS_T + 4 * g + o;
      if (i < H && j < W) {
        const size_t p = ((size_t)i * W + j) * C + c0 + c;
        const float xv = x[p], yv = ld_gt<U8>(y, p);
        const float d = xv - yv;
        v_x[p] = gsc * (f[0][o] + 2.f * xv * f[1][o] + yv * f[2][o]) + gl1 * ((d > 0.f) ? 1.f : ((d < 0.f) ? -1.f : 0.f));
      }
    }
  }
}

}  // namespace

// One launch per group of up to three channels (C = 3: a single launch).
template <bool L1>
static int launch_ssim_fwd(const float* pred, const void* gt, int gt_is_u8, int H, int W, int C, float* dmaps, float* out, cudaStream_t s) {
  const dim3 grid((W + SS_T - 1) / SS_T, (H + SS_T - 1) / SS_T, 1);
  for (int c0 = 0; c0 < C; c0 += SS_C) {
    const int nc = C - c0 < SS_C ? C - c0 : SS_C;
#define DNR_SSIM_FWD(U8, NC) ssim_fwd_kernel<U8, L1, NC><<<grid, SS_NT, 0, s>>>(pred, gt, H, W, C, c0, dmaps, out)
    if (gt_is_u8) { if (nc == 3) DNR_SSIM_FWD(true, 3); else if (nc == 2) DNR_SSIM_FWD(true, 2); else DNR_SSIM_FWD(true, 1); }
    else { if (nc == 3) DNR_SSIM_FWD(false, 3); else if (nc == 2) DNR_SSIM_FWD(false, 2); else DNR_SSIM_FWD(false, 1); }
#undef DNR_SSIM_FWD
    DNR_CHECK_LAUNCH();
  }
  return 0;
}

static int launch_ssim_bwd(const float* pred, const void* gt, int gt_is_u8, int H, int W, int C, const float* dmaps, const float* v,
                           float w_ssim, float w_l1, float* v_pred, cudaStream_t s) {
  const dim3 grid((W + SS_T - 1) / SS_T, (H + SS_T - 1) / SS_T, 1);
  for (int c0 = 0; c0 < C; c0 += SS_C) {
    const int nc = C - c0 < SS_C ? C - c0 : SS_C;
#define DNR_SSIM_BWD(U8, NC) ssim_bwd_kernel<U8, NC><<<grid, SS_NT, 0, s>>>(pred, gt, H, W, C, c0, dmaps, v, w_ssim, w_l1, v_pred)
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
  const dim3 grid((W + SS_T - 1) / SS_T, (H + SS_T - 1) / SS_T, B);
  float* o = reinterpret_cast<float*>(out);
  for (int c0 = 0; c0 < C; c0 += SS_C) {
    const int nc = C - c0 < SS_C ? C - c0 : SS_C;
#define DNR_SSIM_MET(U8, NC) ssim_fwd_kernel<U8, false, NC, true><<<grid, SS_NT, 0, s>>>(pred, gt, H, W, C, c0, nullptr, o)
    if (gt_is_u8) { if (nc == 3) DNR_SSIM_MET(true, 3); else if (nc == 2) DNR_SSIM_MET(true, 2); else DNR_SSIM_MET(true, 1); }
    else { if (nc == 3) DNR_SSIM_MET(false, 3); else if (nc == 2) DNR_SSIM_MET(false, 2); else DNR_SSIM_MET(false, 1); }
#undef DNR_SSIM_MET
    DNR_CHECK_LAUNCH();
  }
  return 0;
}

// pred: [H,W,C] fp32; gt: [H,W,C] fp32, or uint8 scaled by 1/255 when gt_is_u8 != 0.  dmaps: [3,H,W,C] scratch kept for
// the backward.  *sum_out (zeroed by the call) receives the SUM of the SSIM map over the interior; the caller divides by
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
