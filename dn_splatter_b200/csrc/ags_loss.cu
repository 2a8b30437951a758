// AGSMeshRegularization (depth + normal terms, regularization_strategy.py:202-321) on rendered maps: one pass over the
// frame forward plus a one-thread finish, one pass backward.  Compiled with -fmad=false: products and sums round as
// torch's separate element-wise kernels round them.
//
// Per pixel p and channel c, with s, g, n the signed surface / gt / predicted normals (2x - 1 of the [0,1] maps, in
// fp32, or the signed [3,H,W] maps as given with DNR_AGS_SIGNED_CHW):
//   depth      the configured DepthLoss over gt > tol, gt first zeroed where the confidence is not positive
//              (DNR_AGS_CONF_GATE), weighted by depth_lambda;
//   surface    lam * mean |s - g| over the kept elements: per element, not on a dilated edge of g (edge mask), or per
//              pixel, acos(clip(sum_c s g, -1, 1)) not above 0.1 (DNR_AGS_ANGLE_MASK);
//   predicted  lam * mean |n - g| over all 3HW elements.
// The edge mask needs the Laplacian of r = 1 / (g + 1e-6) at the 3x3 neighbours of p, so each CTA stages r for its
// 32 x 8 tile with a 2-pixel halo (zero outside the image, as conv2d's padding of r), then the 3-bit edge code of the
// tile with a 1-pixel halo (no edge outside the image: the dilation is clipped to it).
#include "common.cuh"

namespace {

constexpr int TW = 32, TH = 8;

__device__ __forceinline__ float sgn_ags(float x) { return (x > 0.f) ? 1.f : ((x < 0.f) ? -1.f : 0.f); }

__device__ __forceinline__ float u8f(uint8_t v) { return __fmul_rn((float)v, 1.0f / 255.0f); }

// signed normal component (channel c of pixel p) of a [0,1] [H,W,3] map (fp32 or uint8) or a signed [3,H,W] map
__device__ __forceinline__ float normal_at(const void* m, bool u8, bool chw, int p, int c, int HW) {
  if (chw) return ((const float*)m)[c * HW + p];
  const float x = u8 ? u8f(((const uint8_t*)m)[p * 3 + c]) : ((const float*)m)[p * 3 + c];
  return __fsub_rn(__fmul_rn(2.0f, x), 1.0f);
}

__device__ __forceinline__ float ags_edge_weight(const DnrAgsLoss& a, int p, int q) {
  float g = 0.f;
  if (a.flags & DNR_AGS_IMG_U8) {
    const uint8_t* im = (const uint8_t*)a.image;
    const float lo = 10.0f / 255.0f;
#pragma unroll
    for (int c = 0; c < 3; ++c) g += fabsf(fmaxf(u8f(im[p * 3 + c]), lo) - fmaxf(u8f(im[q * 3 + c]), lo));
  } else {
    const float* im = (const float*)a.image;
#pragma unroll
    for (int c = 0; c < 3; ++c) g += fabsf(im[p * 3 + c] - im[q * 3 + c]);
  }
  return expf(-(g / 3.0f));
}

// gt depth after the confidence gate: torch.where(conf > 0, gt, 0), conf = 1 - get_gt_img(c) / 255 for a raw map
__device__ __forceinline__ float gated_gt_depth(const DnrAgsLoss& a, int p) {
  const float gd = a.gt_depth[p];
  if (!(a.flags & DNR_AGS_CONF_GATE)) return gd;
  float conf;
  if (a.flags & DNR_AGS_CONF_RAW) {
    const float c = (a.flags & DNR_AGS_CONF_U8) ? u8f(((const uint8_t*)a.confidence)[p]) : ((const float*)a.confidence)[p];
    conf = __fsub_rn(1.0f, __fmul_rn(c, 1.0f / 255.0f));
  } else {
    conf = ((const float*)a.confidence)[p];
  }
  return conf > 0.f ? gd : 0.f;
}

__device__ __forceinline__ void depth_piece(int type, float d, float g, float& val, float& dval) {
  const float e = d - g;
  if (type == 1 || type == 2) { val = logf(1.0f + fabsf(e)); dval = sgn_ags(e) / (1.0f + fabsf(e)); }
  else if (type == 3) { val = fabsf(e); dval = sgn_ags(e); }
  else { val = e * e; dval = 2.0f * e; }
}

// bit c set: element (c, p) is kept by the surface-normal selection.  `edges` is the CTA's edge-code tile (edge mode).
__device__ __forceinline__ uint32_t keep_bits(const DnrAgsLoss& a, const uint8_t (*edges)[TW + 2], int ti, int tj, int p,
                                              const float s[3], const float g[3]) {
  if (a.flags & DNR_AGS_ANGLE_MASK) {
    const float dot = (s[0] * g[0] + s[1] * g[1]) + s[2] * g[2];
    const float cl = isnan(dot) ? dot : fminf(fmaxf(dot, -1.0f), 1.0f);  // torch.clip keeps a nan (kept: nan > 0.1 is false)
    return (acosf(cl) > 0.1f) ? 0u : 7u;
  }
  uint32_t e = 0;
#pragma unroll
  for (int dy = 0; dy < 3; ++dy)
#pragma unroll
    for (int dx = 0; dx < 3; ++dx) e |= edges[ti + dy][tj + dx];
  return (~e) & 7u;
}

// Stages the edge codes of the CTA's tile plus a 1-pixel halo (edge mode only; a uniform branch).
__device__ void stage_edges(const DnrAgsLoss& a, int i0, int j0, float (*r)[TH + 4][TW + 4], uint8_t (*edges)[TW + 2]) {
  const int W = a.width, H = a.height, HW = W * H;
  const bool u8 = a.flags & DNR_AGS_NORMAL_U8, chw = a.flags & DNR_AGS_SIGNED_CHW;
  for (int k = threadIdx.x; k < (TH + 4) * (TW + 4); k += blockDim.x) {
    const int y = k / (TW + 4), x = k % (TW + 4);
    const int i = i0 + y - 2, j = j0 + x - 2;
    const bool in = i >= 0 && i < H && j >= 0 && j < W;
#pragma unroll
    for (int c = 0; c < 3; ++c)  // 1.0 / (g + 1e-6): IEEE reciprocal, as torch's reciprocal (inf at 0, nan stays nan)
      r[c][y][x] = in ? __frcp_rn(__fadd_rn(normal_at(a.gt_normal, u8, chw, i * W + j, c, HW), 1e-6f)) : 0.f;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < (TH + 2) * (TW + 2); k += blockDim.x) {
    const int y = k / (TW + 2), x = k % (TW + 2);
    const int i = i0 + y - 1, j = j0 + x - 1;
    uint8_t e = 0;
    if (i >= 0 && i < H && j >= 0 && j < W) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float (*rc)[TW + 4] = r[c];
        const int yy = y + 1, xx = x + 1;
        // conv2d's nine products in row-major order: the zero corners matter only to a non-finite r (0 * inf = nan)
        float lap = 0.0f * rc[yy - 1][xx - 1];
        lap = lap + rc[yy - 1][xx];
        lap = lap + 0.0f * rc[yy - 1][xx + 1];
        lap = lap + rc[yy][xx - 1];
        lap = lap + (-4.0f) * rc[yy][xx];
        lap = lap + rc[yy][xx + 1];
        lap = lap + 0.0f * rc[yy + 1][xx - 1];
        lap = lap + rc[yy + 1][xx];
        lap = lap + 0.0f * rc[yy + 1][xx + 1];
        if (lap > 0.01f) e |= (uint8_t)(1u << c);
      }
    }
    edges[y][x] = e;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(256) ags_loss_fwd_kernel(const DnrAgsLoss a) {
  __shared__ float r[3][TH + 4][TW + 4];
  __shared__ uint8_t edges[TH + 2][TW + 2];
  __shared__ float red[7][8];
  const int tj = threadIdx.x & 31, ti = threadIdx.x >> 5;
  const int i0 = blockIdx.y * TH, j0 = blockIdx.x * TW;
  const int j = j0 + tj, i = i0 + ti;
  const int W = a.width, H = a.height, HW = W * H;
  if (!(a.flags & DNR_AGS_ANGLE_MASK)) stage_edges(a, i0, j0, r, edges);
  float acc[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (i < H && j < W) {
    const int p = i * W + j;
    if (a.depth_loss_type != 0) {
      const float gd = gated_gt_depth(a, p);
      if (gd > a.depth_tolerance) {
        float val, dval;
        depth_piece(a.depth_loss_type, a.pred_depth[p], gd, val, dval);
        if (a.depth_loss_type == 1) {
          if (j < W - 1) { acc[0] = ags_edge_weight(a, p, p + 1) * val; acc[1] = 1.f; }
          if (i < H - 1) { acc[2] = ags_edge_weight(a, p, p + W) * val; acc[3] = 1.f; }
        } else {
          acc[0] = val; acc[1] = 1.f;
        }
      }
    }
    const bool u8 = a.flags & DNR_AGS_NORMAL_U8, chw = a.flags & DNR_AGS_SIGNED_CHW;
    float s[3], g[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      g[c] = normal_at(a.gt_normal, u8, chw, p, c, HW);
      s[c] = normal_at(a.surf_normal, false, chw, p, c, HW);
      acc[4] += fabsf(normal_at(a.pred_normal, false, chw, p, c, HW) - g[c]);
    }
    const uint32_t keep = keep_bits(a, edges, ti, tj, p, s, g);
#pragma unroll
    for (int c = 0; c < 3; ++c)
      if (keep & (1u << c)) { acc[5] += fabsf(s[c] - g[c]); acc[6] += 1.f; }
    if (a.keep_mask) a.keep_mask[p] = (uint8_t)keep;
  }
#pragma unroll
  for (int k = 0; k < 7; ++k) {
    const float w = warp_sum(acc[k]);
    if (tj == 0) red[k][ti] = w;
  }
  __syncthreads();
  if (threadIdx.x < 7) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[threadIdx.x][w];
    if (t != 0.f) atomicAdd(a.partials + threadIdx.x, t);
  }
}

__global__ void ags_loss_finish_kernel(const DnrAgsLoss a) {
  float* p = a.partials;
  const float HW3 = 3.0f * (float)a.height * (float)a.width;
  float depth = 0.f;
  if (a.depth_loss_type == 1) depth = p[0] / p[1] + p[2] / p[3];  // 0/0 = nan for an empty mask, as torch's mean
  else if (a.depth_loss_type != 0) depth = p[0] / p[1];
  depth = depth * a.depth_lambda;
  const float surf = (p[5] / p[6]) * a.normal_lambda;  // an empty selection is nan, and 0 * nan stays nan
  const float pred = (p[4] / HW3) * a.normal_lambda;
  p[8] = depth; p[9] = surf; p[10] = pred; p[11] = depth + (surf + pred);
}

__global__ void __launch_bounds__(256) ags_loss_bwd_kernel(const DnrAgsLoss a, float* __restrict__ v_depth,
                                                          float* __restrict__ v_normal) {
  const int j = blockIdx.x * TW + (threadIdx.x & 31);
  const int i = blockIdx.y * TH + (threadIdx.x >> 5);
  const int W = a.width, H = a.height, HW = W * H;
  if (i >= H || j >= W) return;
  const int p = i * W + j;
  const float vl = a.v_loss ? __ldg(a.v_loss) : 1.0f;
  if (v_depth) {
    float gr = 0.f;
    if (a.depth_loss_type != 0) {
      const float gd = gated_gt_depth(a, p);
      if (gd > a.depth_tolerance) {
        float val, dval;
        depth_piece(a.depth_loss_type, a.pred_depth[p], gd, val, dval);
        const float scale = vl * a.depth_lambda;
        if (a.depth_loss_type == 1) {
          float w = 0.f;
          if (j < W - 1) w += ags_edge_weight(a, p, p + 1) / a.partials[1];
          if (i < H - 1) w += ags_edge_weight(a, p, p + W) / a.partials[3];
          gr = scale * dval * w;
        } else {
          gr = scale * dval / a.partials[1];
        }
      }
    }
    v_depth[p] = gr;
  }
  if (v_normal) {
    const bool u8 = a.flags & DNR_AGS_NORMAL_U8, chw = a.flags & DNR_AGS_SIGNED_CHW;
    // d/dn of lam * mean |(2n - 1) - g|: the factor 2 of 2n - 1 unless the map is given signed
    const float k = chw ? (vl * a.normal_lambda) / (3.0f * (float)HW) : ((vl * a.normal_lambda) * 2.0f) / (3.0f * (float)HW);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float d = normal_at(a.pred_normal, false, chw, p, c, HW) - normal_at(a.gt_normal, u8, chw, p, c, HW);
      v_normal[chw ? c * HW + p : p * 3 + c] = sgn_ags(d) * k;
    }
  }
}

inline dim3 ags_grid(const DnrAgsLoss* a) { return dim3((a->width + TW - 1) / TW, (a->height + TH - 1) / TH); }

int check_ags(const DnrAgsLoss* a) {
  if (!a) return DNR_E_NULL;
  if (a->width <= 0 || a->height <= 0 || (int64_t)a->width * a->height * 3 > INT32_MAX) return DNR_E_SIZE;
  if (a->depth_loss_type < 0 || a->depth_loss_type > 4) return DNR_E_OPTION;
  if ((a->flags & ~DNR_AGS_ALL_FLAGS) != 0) return DNR_E_OPTION;
  if ((a->flags & DNR_AGS_SIGNED_CHW) && (a->flags & DNR_AGS_NORMAL_U8)) return DNR_E_OPTION;
  if ((a->flags & DNR_AGS_CONF_U8) && !(a->flags & DNR_AGS_CONF_RAW)) return DNR_E_OPTION;
  if (!a->partials || !a->gt_normal || !a->pred_normal) return DNR_E_NULL;
  if (a->depth_loss_type != 0) {
    if (!a->pred_depth || !a->gt_depth) return DNR_E_NULL;
    if ((a->flags & DNR_AGS_CONF_GATE) && !a->confidence) return DNR_E_NULL;
    if (a->depth_loss_type == 1 && !a->image) return DNR_E_NULL;
  }
  return 0;
}

}  // namespace

extern "C" int dnr_ags_loss_fwd(const DnrAgsLoss* a, void* stream) {
  if (const int rc = check_ags(a)) return rc;
  if (!a->surf_normal) return DNR_E_NULL;
  cudaStream_t s = (cudaStream_t)stream;
  DNR_CUDA(cudaMemsetAsync(a->partials, 0, 12 * sizeof(float), s));
  ags_loss_fwd_kernel<<<ags_grid(a), 256, 0, s>>>(*a);
  DNR_CHECK_LAUNCH();
  ags_loss_finish_kernel<<<1, 1, 0, s>>>(*a);
  DNR_CHECK_LAUNCH();
  return 0;
}

extern "C" int dnr_ags_loss_bwd(const DnrAgsLoss* a, float* v_depth_out, float* v_normal_out, void* stream) {
  if (const int rc = check_ags(a)) return rc;
  if (!v_depth_out && !v_normal_out) return 0;
  ags_loss_bwd_kernel<<<ags_grid(a), 256, 0, (cudaStream_t)stream>>>(*a, v_depth_out, v_normal_out);
  DNR_CHECK_LAUNCH();
  return 0;
}
