// SuGaR-style density of a Gaussian set at sample points, given each sample's neighbour list (SURVEY.md §8f-4).
// Replaces the torch passes of /root/reference/dn_splatter/dn_model.py:
//   get_density                    :1077-1135  (one sample per neighbour row, clamp(min=1e-4) at the end)
//   compute_level_surface_points   :1264-1345  (21 samples along every pixel ray sharing the pixel's 16 neighbours,
//                                               processed by the reference in 2M-sample chunks that materialise
//                                               [2M,16,3,3] tensors)
// density(x) = sum_k sigmoid(o_k) exp(-1/2 clamp(|M_k^T (x - mu_k)|^2, 0, 1e8)),  M_k = R(q_k/|q_k|) diag(1/max(exp(s_k),1e-3))
// and, as in the reference, a density >= 1 is replaced by d / (d + 1e-5).
// One thread per sample (dnr_density) or per pixel ray (dnr_ray_densities: the 16 neighbours are gathered once and
// reused for the 21 samples).  Precise expf / division: this is an export-time path compared value by value.
//
// The algorithm is pinned on the CPU (oracle/sugar_ref.py vs goldens from the reference's own functions) and the kernel
// against that restatement on the GPU (tests/test_gpu_sugar.py), and per sample / per ray against an fp64 sum with a
// per-term error bound (tests/test_gpu_knn_density.py).
#include "common.cuh"

namespace {

constexpr int RAY_SAMPLES = 21;

struct Nbr {
  float mx, my, mz;        // centre
  float r[9];              // R(q_hat), row-major
  float is0, is1, is2;     // 1 / max(exp(s), 1e-3)
  float op;                // sigmoid(opacity)
};

__device__ __forceinline__ void rotmat(const float* __restrict__ q4, float r[9]) {
  float w = q4[0], x = q4[1], y = q4[2], z = q4[3];
  const float inv = 1.0f / sqrtf(w * w + x * x + y * y + z * z);
  w *= inv; x *= inv; y *= inv; z *= inv;
  r[0] = 1.f - 2.f * (y * y + z * z); r[1] = 2.f * (x * y - w * z); r[2] = 2.f * (x * z + w * y);
  r[3] = 2.f * (x * y + w * z); r[4] = 1.f - 2.f * (x * x + z * z); r[5] = 2.f * (y * z - w * x);
  r[6] = 2.f * (x * z - w * y); r[7] = 2.f * (y * z + w * x); r[8] = 1.f - 2.f * (x * x + y * y);
}

__device__ __forceinline__ Nbr load_nbr(int64_t g, const float* __restrict__ means, const float* __restrict__ scales,
                                        const float* __restrict__ quats, const float* __restrict__ opac) {
  Nbr n;
  n.mx = means[3 * g]; n.my = means[3 * g + 1]; n.mz = means[3 * g + 2];
  rotmat(quats + 4 * g, n.r);
  n.is0 = 1.0f / fmaxf(expf(scales[3 * g]), 1e-3f);
  n.is1 = 1.0f / fmaxf(expf(scales[3 * g + 1]), 1e-3f);
  n.is2 = 1.0f / fmaxf(expf(scales[3 * g + 2]), 1e-3f);
  n.op = 1.0f / (1.0f + expf(-opac[g]));
  return n;
}

// sigmoid(o) exp(-1/2 clamp(|M^T (x - mu)|^2)): (M^T d)_c = is_c * (column c of R) . d
__device__ __forceinline__ float nbr_weight(const Nbr& n, float x, float y, float z) {
  const float dx = x - n.mx, dy = y - n.my, dz = z - n.mz;
  const float a = n.is0 * (n.r[0] * dx + n.r[3] * dy + n.r[6] * dz);
  const float b = n.is1 * (n.r[1] * dx + n.r[4] * dy + n.r[7] * dz);
  const float c = n.is2 * (n.r[2] * dx + n.r[5] * dy + n.r[8] * dz);
  const float d2 = fminf(fmaxf(a * a + b * b + c * c, 0.0f), 1e8f);
  return n.op * expf(-0.5f * d2);
}

__device__ __forceinline__ float squash(float d) { return d >= 1.0f ? d / (d + 1e-5f) : d; }

__global__ void __launch_bounds__(256) density_kernel(const float* __restrict__ samples, int64_t m, const int64_t* __restrict__ idx, int k,
                                                      int per_row, const float* __restrict__ means, const float* __restrict__ scales,
                                                      const float* __restrict__ quats, const float* __restrict__ opac, int n_gauss,
                                                      float clamp_min, float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const float x = samples[3 * i], y = samples[3 * i + 1], z = samples[3 * i + 2];
  const int64_t* row = idx + (i / per_row) * k;
  float d = 0.f;
  for (int j = 0; j < k; ++j) {
    const int64_t g = row[j];
    if (g < 0 || g >= n_gauss) continue;  // -1: fewer than k Gaussians exist
    d += nbr_weight(load_nbr(g, means, scales, quats, opac), x, y, z);
  }
  out[i] = fmaxf(squash(d), clamp_min);
}

// torch.linspace(-R, R, 21) in fp32: start + i*step below the midpoint, end - (20-i)*step from it on, each rounded once
// as torch's fused multiply-add does (this file is built with -fmad=false, so the fma is spelled out: two roundings
// differ from torch at 5 of the 21 samples for R = 3)
__device__ __forceinline__ float linspace21(int i, float range) {
  const float step = (range - (-range)) / 20.0f;
  return i < RAY_SAMPLES / 2 ? fmaf(step, (float)i, -range) : fmaf(-step, (float)(RAY_SAMPLES - 1 - i), range);
}

__global__ void __launch_bounds__(128) ray_density_kernel(const float* __restrict__ points, int64_t P, const int64_t* __restrict__ idx, int k,
                                                          float cx, float cy, float cz, const float* __restrict__ means,
                                                          const float* __restrict__ scales, const float* __restrict__ quats,
                                                          const float* __restrict__ opac, int n_gauss, float range,
                                                          float* __restrict__ out_dens, float* __restrict__ out_t, float* __restrict__ out_dirs) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const float px = points[3 * p], py = points[3 * p + 1], pz = points[3 * p + 2];
  // unit ray direction camera -> point (F.normalize: eps 1e-12)
  float dx = px - cx, dy = py - cy, dz = pz - cz;
  const float dn = fmaxf(sqrtf(dx * dx + dy * dy + dz * dz), 1e-12f);
  dx /= dn; dy /= dn; dz /= dn;
  out_dirs[3 * p] = dx; out_dirs[3 * p + 1] = dy; out_dirs[3 * p + 2] = dz;
  // standard deviation of the FIRST neighbour along ITS OWN view direction (dn_model.py:1264-1274):
  // || exp(s) * (R^T v) ||, v = normalize(cam - mu)
  const int64_t* row = idx + p * k;
  float std = 0.f;
  {
    const int64_t g = row[0];
    if (g >= 0 && g < n_gauss) {
      float r[9];
      rotmat(quats + 4 * g, r);
      float vx = cx - means[3 * g], vy = cy - means[3 * g + 1], vz = cz - means[3 * g + 2];
      const float vn = sqrtf(vx * vx + vy * vy + vz * vz);
      vx /= vn; vy /= vn; vz /= vn;
      const float a = expf(scales[3 * g]) * (r[0] * vx + r[3] * vy + r[6] * vz);
      const float b = expf(scales[3 * g + 1]) * (r[1] * vx + r[4] * vy + r[7] * vz);
      const float c = expf(scales[3 * g + 2]) * (r[2] * vx + r[5] * vy + r[8] * vz);
      std = sqrtf(a * a + b * b + c * c);
    }
  }
  float t[RAY_SAMPLES], dens[RAY_SAMPLES];
#pragma unroll
  for (int s = 0; s < RAY_SAMPLES; ++s) {
    t[s] = linspace21(s, range) * std;
    dens[s] = 0.f;
  }
  for (int j = 0; j < k; ++j) {
    const int64_t g = row[j];
    if (g < 0 || g >= n_gauss) continue;
    const Nbr n = load_nbr(g, means, scales, quats, opac);
#pragma unroll
    for (int s = 0; s < RAY_SAMPLES; ++s) dens[s] += nbr_weight(n, px + t[s] * dx, py + t[s] * dy, pz + t[s] * dz);
  }
#pragma unroll
  for (int s = 0; s < RAY_SAMPLES; ++s) {
    out_dens[p * RAY_SAMPLES + s] = squash(dens[s]);
    out_t[p * RAY_SAMPLES + s] = t[s];
  }
}

}  // namespace

extern "C" int dnr_density(const float* samples, int64_t n_samples, const int64_t* nbr_idx, int32_t k, int32_t samples_per_row,
                           const float* means, const float* scales, const float* quats, const float* opacities, int32_t n_gauss,
                           float clamp_min, float* out, void* stream) {
  if (!samples || !nbr_idx || !means || !scales || !quats || !opacities || !out) return DNR_E_NULL;
  if (n_samples <= 0 || k <= 0 || samples_per_row <= 0 || n_gauss <= 0) return DNR_E_SIZE;
  const int64_t blocks = (n_samples + 255) / 256;
  if (blocks > 0x7fffffff) return DNR_E_SIZE;
  density_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(samples, n_samples, nbr_idx, k, samples_per_row, means, scales, quats,
                                                                     opacities, n_gauss, clamp_min, out);
  DNR_CHECK_LAUNCH();
  return 0;
}

extern "C" int dnr_ray_densities(const float* points, int64_t n_points, const int64_t* nbr_idx, int32_t k, const float* cam_pos_host,
                                 const float* means, const float* scales, const float* quats, const float* opacities, int32_t n_gauss,
                                 int32_t n_range, float range_size, float* out_dens, float* out_t, float* out_dirs, void* stream) {
  if (!points || !nbr_idx || !cam_pos_host || !means || !scales || !quats || !opacities || !out_dens || !out_t || !out_dirs)
    return DNR_E_NULL;
  if (n_points <= 0 || k <= 0 || n_gauss <= 0) return DNR_E_SIZE;
  if (n_range != RAY_SAMPLES) return DNR_E_OPTION;  // the reference hard-codes 21 samples in [-3, 3] sigma
  const int64_t blocks = (n_points + 127) / 128;
  if (blocks > 0x7fffffff) return DNR_E_SIZE;
  ray_density_kernel<<<(unsigned)blocks, 128, 0, (cudaStream_t)stream>>>(points, n_points, nbr_idx, k, cam_pos_host[0], cam_pos_host[1],
                                                                         cam_pos_host[2], means, scales, quats, opacities, n_gauss,
                                                                         range_size, out_dens, out_t, out_dirs);
  DNR_CHECK_LAUNCH();
  return 0;
}
