// Full-image stencils around the rasterizer, each one pass over HBM instead of the reference's chains of
// torch element-wise kernels.  Compiled with -fmad=false (cheap kernels; keeps results close to torch's).
//
//   finalize_fwd          dn_model.py:534-537 depth fill with the global max  +  :589-603 surface normal
//                         (utils/normal_utils.py:9-48, utils/camera_utils.py:70-144 with c2w = I)
//   normal_from_depth     the same stencil for an arbitrary depth map (normal_supervision == "depth",
//                         dn_model.py:669-686)
//   loss_fwd / loss_bwd   DNRegularization depth + normal terms (regularization_strategy.py:146-193;
//                         losses.py:155-224 L1/LogL1/EdgeAwareLogL1, :279-295 TVLoss)
#include "common.cuh"
#include "loss_common.cuh"

namespace {

struct Intr { float fx, fy, cx, cy; };

__device__ __forceinline__ Intr load_intr(const DnrArgs& a) {
  Intr k;
  if (a.flags & DNR_FLAG_HOST_CAMERA) {
    k.fx = a.host_cam[16]; k.fy = a.host_cam[17]; k.cx = a.host_cam[18]; k.cy = a.host_cam[19];
  } else {
    k.fx = __ldg(a.K + 0); k.fy = __ldg(a.K + 4); k.cx = __ldg(a.K + 2); k.cy = __ldg(a.K + 5);
  }
  return k;
}

__device__ __forceinline__ void backproject(const Intr& k, int u, int v, float d, float p[3]) {
  p[0] = (((float)u + 0.5f) - k.cx) * d / k.fx;
  p[1] = (((float)v + 0.5f) - k.cy) * d / k.fy;
  p[2] = d;
}

// normal at interior pixel (i,j) from the 4-neighbourhood; `depth_at` returns the (filled) depth.
template <typename F>
__device__ __forceinline__ void stencil_normal(const Intr& k, int i, int j, F depth_at, float n[3]) {
  float r[3], l[3], t[3], b[3];
  backproject(k, j + 1, i, depth_at(i, j + 1), r);
  backproject(k, j - 1, i, depth_at(i, j - 1), l);
  backproject(k, j, i - 1, depth_at(i - 1, j), t);
  backproject(k, j, i + 1, depth_at(i + 1, j), b);
  const float a0 = r[0] - l[0], a1 = r[1] - l[1], a2 = r[2] - l[2];  // left -> right
  const float c0 = t[0] - b[0], c1 = t[1] - b[1], c2 = t[2] - b[2];  // bottom -> top
  n[0] = a1 * c2 - a2 * c1;
  n[1] = a2 * c0 - a0 * c2;
  n[2] = a0 * c1 - a1 * c0;
  const float nn = fmaxf(sqrtf((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2]), 1e-12f);
  n[0] /= nn; n[1] /= nn; n[2] /= nn;
}

__global__ void __launch_bounds__(256) finalize_fwd_kernel(const DnrArgs a) {
  const int j = blockIdx.x * 32 + (threadIdx.x & 31);
  const int i = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (i >= a.height || j >= a.width) return;
  const float maxd = __int_as_float(*a.depth_max);
  const int W = a.width, H = a.height;
  auto depth_at = [&](int y, int x) -> float {
    const int p = y * W + x;
    return a.out_alpha[p] > 0.f ? a.out_depth[p] : maxd;
  };
  const int pix = i * W + j;
  if (!(a.out_alpha[pix] > 0.f)) a.out_depth[pix] = maxd;  // neighbours ignore the stored value when alpha == 0
  if (a.out_surface_normal) {
    float n[3] = {0.f, 0.f, 0.f};
    if (i > 0 && j > 0 && i < H - 1 && j < W - 1) {
      const Intr k = load_intr(a);
      stencil_normal(k, i, j, depth_at, n);
    }
    // flip y,z (dn_model.py:600-602) and map to [0,1] (:603); border stays exactly 0.5
    a.out_surface_normal[pix * 3 + 0] = (1.0f + n[0]) * 0.5f;
    a.out_surface_normal[pix * 3 + 1] = (1.0f - n[1]) * 0.5f;
    a.out_surface_normal[pix * 3 + 2] = (1.0f - n[2]) * 0.5f;
  }
}

__global__ void __launch_bounds__(256) normal_from_depth_kernel(const DnrArgs a) {
  const int j = blockIdx.x * 32 + (threadIdx.x & 31);
  const int i = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (i >= a.height || j >= a.width) return;
  const int W = a.width, H = a.height;
  auto depth_at = [&](int y, int x) -> float { return a.out_depth[y * W + x]; };
  float n[3] = {0.f, 0.f, 0.f};
  if (i > 0 && j > 0 && i < H - 1 && j < W - 1) {
    const Intr k = load_intr(a);
    stencil_normal(k, i, j, depth_at, n);
  }
  const int pix = i * W + j;
  a.out_surface_normal[pix * 3 + 0] = n[0];
  a.out_surface_normal[pix * 3 + 1] = n[1];
  a.out_surface_normal[pix * 3 + 2] = n[2];
}

__device__ __forceinline__ float sgn(float x) { return sgnf(x); }

// per-pixel depth-term pieces: value (for the type) and d(value)/d(pred)
__device__ __forceinline__ void depth_term(int type, float d, float g, float& val, float& dval) {
  const float e = d - g;
  if (type == 1 || type == 2) { val = logf(1.0f + fabsf(e)); dval = sgn(e) / (1.0f + fabsf(e)); }
  else if (type == 3) { val = fabsf(e); dval = sgn(e); }
  else { val = e * e; dval = 2.0f * e; }
}

__global__ void __launch_bounds__(256) loss_fwd_kernel(const DnrArgs a) {
  __shared__ float red[7][8];
  const int j = blockIdx.x * 32 + (threadIdx.x & 31);
  const int i = blockIdx.y * 8 + (threadIdx.x >> 5);
  const int W = a.width, H = a.height;
  float s[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (i < H && j < W) {
    const int p = i * W + j;
    if (a.depth_loss_type != 0 && a.gt_depth[p] > a.depth_tolerance) {
      float val, dval;
      depth_term(a.depth_loss_type, a.out_depth[p], a.gt_depth[p], val, dval);
      if (a.depth_loss_type == 1) {
        if (j < W - 1) { s[0] = edge_weight(a, p, p + 1) * val; s[1] = 1.f; }
        if (i < H - 1) { s[2] = edge_weight(a, p, p + W) * val; s[3] = 1.f; }
      } else {
        s[0] = val; s[1] = 1.f;
      }
    }
    if (a.use_normal_loss) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float n = a.out_normal[p * 3 + c];
        s[4] += fabsf(n - gt_normal_at(a, p * 3 + c));
        if (j < W - 1) s[5] += fabsf(n - a.out_normal[(p + 1) * 3 + c]);
        if (i < H - 1) s[6] += fabsf(n - a.out_normal[(p + W) * 3 + c]);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 7; ++k) {
    const float w = warp_sum(s[k]);
    if ((threadIdx.x & 31) == 0) red[k][threadIdx.x >> 5] = w;
  }
  __syncthreads();
  if (threadIdx.x < 7) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[threadIdx.x][w];
    if (t != 0.f) atomicAdd(a.loss_partials + threadIdx.x, t);
  }
}

__global__ void __launch_bounds__(256) loss_bwd_kernel(const DnrArgs a, float* __restrict__ v_depth, float* __restrict__ v_normal) {
  const int j = blockIdx.x * 32 + (threadIdx.x & 31);
  const int i = blockIdx.y * 8 + (threadIdx.x >> 5);
  const int W = a.width, H = a.height;
  if (i >= H || j >= W) return;
  const int p = i * W + j;
  const float vl = a.v_loss ? __ldg(a.v_loss) : 1.0f;
  if (v_depth) {
    float g = 0.f;
    if (a.depth_loss_type != 0 && a.gt_depth[p] > a.depth_tolerance) {
      float val, dval;
      depth_term(a.depth_loss_type, a.out_depth[p], a.gt_depth[p], val, dval);
      const float scale = vl * (1.0f + a.depth_lambda);  // quirk B6: depth_loss += lambda * depth_loss
      if (a.depth_loss_type == 1) {
        float w = 0.f;
        if (j < W - 1) w += edge_weight(a, p, p + 1) / a.loss_partials[1];
        if (i < H - 1) w += edge_weight(a, p, p + W) / a.loss_partials[3];
        g = scale * dval * w;
      } else {
        g = scale * dval / a.loss_partials[1];
      }
    }
    v_depth[p] = g;
  }
  if (v_normal) {
    const float inv_l1 = vl / (3.0f * (float)H * (float)W);
    const float inv_tx = (W > 1) ? vl / (3.0f * (float)H * (float)(W - 1)) : 0.f;
    const float inv_ty = (H > 1) ? vl / (3.0f * (float)(H - 1) * (float)W) : 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float g = 0.f;
      if (a.use_normal_loss) {
        const float n = a.out_normal[p * 3 + c];
        g = sgn(n - gt_normal_at(a, p * 3 + c)) * inv_l1;
        if (j < W - 1) g += sgn(n - a.out_normal[(p + 1) * 3 + c]) * inv_tx;
        if (j > 0) g -= sgn(a.out_normal[(p - 1) * 3 + c] - n) * inv_tx;
        if (i < H - 1) g += sgn(n - a.out_normal[(p + W) * 3 + c]) * inv_ty;
        if (i > 0) g -= sgn(a.out_normal[(p - W) * 3 + c] - n) * inv_ty;
      }
      v_normal[p * 3 + c] = g;
    }
  }
}

__global__ void loss_finish_kernel(const DnrArgs a) {
  float* p = a.loss_partials;
  const int W = a.width, H = a.height;
  float depth = 0.f;
  if (a.depth_loss_type == 1) depth = p[0] / p[1] + p[2] / p[3];  // 0/0 = nan when nothing is valid, as torch's mean of empty
  else if (a.depth_loss_type != 0) depth = p[0] / p[1];
  depth = depth + a.depth_lambda * depth;  // quirk B6
  float l1 = 0.f, tv = 0.f;
  if (a.use_normal_loss) {
    l1 = p[4] / (3.0f * (float)H * (float)W);
    tv = p[5] / (3.0f * (float)H * (float)(W - 1)) + p[6] / (3.0f * (float)(H - 1) * (float)W);
  }
  p[8] = depth; p[9] = l1; p[10] = tv; p[11] = depth + (l1 + tv);
}

__global__ void __launch_bounds__(256) scale_loss_fwd_kernel(const float* __restrict__ scales, int n, float* out) {
  __shared__ float red[8];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  float v = 0.f;
  if (i < n) v = expf(fminf(fminf(scales[i * 3], scales[i * 3 + 1]), scales[i * 3 + 2]));
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[w];
    atomicAdd(out, t / (float)n);
  }
}

__global__ void __launch_bounds__(256) scale_loss_bwd_kernel(const float* __restrict__ scales, int n, const float* v_loss,
                                                            float* __restrict__ v_scales) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float vl = v_loss ? __ldg(v_loss) : 1.0f;
  // torch.exp(scales).min(1) picks the FIRST index of the smallest exp: distinct log-scales whose exp rounds to one fp32
  // value are a tie there, so the argmin is taken over the exps, not over the log-scales
  const float e0 = expf(scales[i * 3]), e1 = expf(scales[i * 3 + 1]), e2 = expf(scales[i * 3 + 2]);
  int idx = 0;
  float m = e0;
  if (e1 < m) { m = e1; idx = 1; }
  if (e2 < m) { m = e2; idx = 2; }
  const float g = vl * m / (float)n;
  v_scales[i * 3 + 0] = idx == 0 ? g : 0.f;
  v_scales[i * 3 + 1] = idx == 1 ? g : 0.f;
  v_scales[i * 3 + 2] = idx == 2 ? g : 0.f;
}

template <bool U8>
__device__ __forceinline__ float gt_at(const void* gt, int64_t i) {
  return U8 ? (float)((const uint8_t*)gt)[i] * (1.0f / 255.0f) : ((const float*)gt)[i];
}

template <bool U8>
__global__ void __launch_bounds__(256) l1_fwd_kernel(const float* __restrict__ pred, const void* __restrict__ gt, int64_t n,
                                                    float* out) {
  __shared__ float red[8];
  float acc = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    acc += fabsf(pred[i] - gt_at<U8>(gt, i));
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[w];
    atomicAdd(out, t / (float)n);
  }
}

template <bool U8>
__global__ void __launch_bounds__(256) l1_bwd_kernel(const float* __restrict__ pred, const void* __restrict__ gt, int64_t n,
                                                    const float* v_loss, float* __restrict__ v_pred) {
  const float s = (v_loss ? __ldg(v_loss) : 1.0f) / (float)n;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    v_pred[i] = sgn(pred[i] - gt_at<U8>(gt, i)) * s;
}

__global__ void __launch_bounds__(256) u8_to_f32_kernel(const uint8_t* __restrict__ src, int64_t n, float divisor, float lo,
                                                       float* __restrict__ dst) {
  const float inv = 1.0f / divisor;  // torch's CUDA `x / scalar` multiplies by the fp32 reciprocal: match it bit for bit
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    dst[i] = fmaxf((float)src[i] * inv, lo);
}

inline int stream_grid(int64_t n) {
  const int64_t b = (n + 256 * 4 - 1) / (256 * 4);
  return (int)(b < DNR_NUM_SMS * 8 ? (b > 0 ? b : 1) : DNR_NUM_SMS * 8);
}

inline dim3 img_grid(const DnrArgs* a) { return dim3((a->width + 31) / 32, (a->height + 7) / 8); }

}  // namespace

extern "C" int dnr_finalize_fwd(const DnrArgs* a, void* stream) {
  if (!a) return DNR_E_NULL;
  if (a->width <= 0 || a->height <= 0) return DNR_E_SIZE;
  if (!a->out_depth || !a->out_alpha || !a->depth_max) return DNR_E_NULL;
  if (a->out_surface_normal && !a->K && !(a->flags & DNR_FLAG_HOST_CAMERA)) return DNR_E_NULL;
  finalize_fwd_kernel<<<img_grid(a), 256, 0, (cudaStream_t)stream>>>(*a);
  DNR_CHECK_LAUNCH();
  return 0;
}

extern "C" int dnr_normal_from_depth(const DnrArgs* a, void* stream) {
  if (!a) return DNR_E_NULL;
  if (a->width <= 0 || a->height <= 0) return DNR_E_SIZE;
  if (!a->out_depth || !a->out_surface_normal) return DNR_E_NULL;
  if (!a->K && !(a->flags & DNR_FLAG_HOST_CAMERA)) return DNR_E_NULL;
  normal_from_depth_kernel<<<img_grid(a), 256, 0, (cudaStream_t)stream>>>(*a);
  DNR_CHECK_LAUNCH();
  return 0;
}

extern "C" int dnr_loss_fwd(const DnrArgs* a, void* stream) {
  if (!a) return DNR_E_NULL;
  if (a->width <= 0 || a->height <= 0) return DNR_E_SIZE;
  if (a->depth_loss_type < 0 || a->depth_loss_type > 4) return DNR_E_OPTION;
  if (!a->loss_partials) return DNR_E_NULL;
  if (a->depth_loss_type != 0 && (!a->out_depth || !a->gt_depth)) return DNR_E_NULL;
  if (a->depth_loss_type == 1 && !((a->loss_flags & DNR_LOSS_EDGE_FROM_IMAGE) ? a->gt_image : (const void*)a->gt_rgb)) return DNR_E_NULL;
  if ((a->loss_flags & DNR_LOSS_EDGE_FROM_IMAGE) && !(a->loss_flags & DNR_LOSS_IMG_U8)) return DNR_E_OPTION;
  if (a->use_normal_loss && (!a->out_normal || !a->gt_normal)) return DNR_E_NULL;
  cudaStream_t s = (cudaStream_t)stream;
  DNR_CUDA(cudaMemsetAsync(a->loss_partials, 0, 12 * sizeof(float), s));
  loss_fwd_kernel<<<img_grid(a), 256, 0, s>>>(*a);
  DNR_CHECK_LAUNCH();
  loss_finish_kernel<<<1, 1, 0, s>>>(*a);
  DNR_CHECK_LAUNCH();
  return 0;
}

extern "C" int dnr_loss_bwd(const DnrArgs* a, float* v_depth_out, float* v_normal_out, void* stream) {
  if (!a) return DNR_E_NULL;
  if (a->width <= 0 || a->height <= 0) return DNR_E_SIZE;
  if (a->depth_loss_type < 0 || a->depth_loss_type > 4) return DNR_E_OPTION;
  if (!a->loss_partials) return DNR_E_NULL;
  if (v_depth_out && a->depth_loss_type != 0 && (!a->out_depth || !a->gt_depth)) return DNR_E_NULL;
  if (v_depth_out && a->depth_loss_type == 1 && !((a->loss_flags & DNR_LOSS_EDGE_FROM_IMAGE) ? a->gt_image : (const void*)a->gt_rgb)) return DNR_E_NULL;
  if (v_normal_out && a->use_normal_loss && (!a->out_normal || !a->gt_normal)) return DNR_E_NULL;
  loss_bwd_kernel<<<img_grid(a), 256, 0, (cudaStream_t)stream>>>(*a, v_depth_out, v_normal_out);
  DNR_CHECK_LAUNCH();
  return 0;
}

extern "C" int dnr_scale_loss_fwd(const float* scales, int32_t n_gauss, float* loss_out, void* stream) {
  if (!scales || !loss_out) return DNR_E_NULL;
  if (n_gauss <= 0) return DNR_E_SIZE;
  cudaStream_t s = (cudaStream_t)stream;
  DNR_CUDA(cudaMemsetAsync(loss_out, 0, sizeof(float), s));
  scale_loss_fwd_kernel<<<(n_gauss + 255) / 256, 256, 0, s>>>(scales, n_gauss, loss_out);
  DNR_CHECK_LAUNCH();
  return 0;
}

extern "C" int dnr_scale_loss_bwd(const float* scales, int32_t n_gauss, const float* v_loss, float* v_scales, void* stream) {
  if (!scales || !v_scales) return DNR_E_NULL;
  if (n_gauss <= 0) return DNR_E_SIZE;
  scale_loss_bwd_kernel<<<(n_gauss + 255) / 256, 256, 0, (cudaStream_t)stream>>>(scales, n_gauss, v_loss, v_scales);
  DNR_CHECK_LAUNCH();
  return 0;
}

extern "C" int dnr_l1_fwd(const float* pred, const void* gt, int64_t n, int32_t gt_is_u8, float* loss_out, void* stream) {
  if (!pred || !gt || !loss_out) return DNR_E_NULL;
  if (n <= 0) return DNR_E_SIZE;
  cudaStream_t s = (cudaStream_t)stream;
  DNR_CUDA(cudaMemsetAsync(loss_out, 0, sizeof(float), s));
  if (gt_is_u8) l1_fwd_kernel<true><<<stream_grid(n), 256, 0, s>>>(pred, gt, n, loss_out);
  else l1_fwd_kernel<false><<<stream_grid(n), 256, 0, s>>>(pred, gt, n, loss_out);
  DNR_CHECK_LAUNCH();
  return 0;
}

extern "C" int dnr_l1_bwd(const float* pred, const void* gt, int64_t n, int32_t gt_is_u8, const float* v_loss, float* v_pred,
                          void* stream) {
  if (!pred || !gt || !v_pred) return DNR_E_NULL;
  if (n <= 0) return DNR_E_SIZE;
  cudaStream_t s = (cudaStream_t)stream;
  if (gt_is_u8) l1_bwd_kernel<true><<<stream_grid(n), 256, 0, s>>>(pred, gt, n, v_loss, v_pred);
  else l1_bwd_kernel<false><<<stream_grid(n), 256, 0, s>>>(pred, gt, n, v_loss, v_pred);
  DNR_CHECK_LAUNCH();
  return 0;
}

extern "C" int dnr_u8_to_f32(const uint8_t* src, int64_t n, float divisor, float clamp_min, float* dst, void* stream) {
  if (!src || !dst) return DNR_E_NULL;
  if (n <= 0) return DNR_E_SIZE;
  u8_to_f32_kernel<<<stream_grid(n), 256, 0, (cudaStream_t)stream>>>(src, n, divisor, clamp_min, dst);
  DNR_CHECK_LAUNCH();
  return 0;
}
