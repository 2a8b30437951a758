// Screened Poisson surface reconstruction on a dense grid (Python surface: dn_splatter_b200.poisson).  Replaces
// Open3D's TriangleMesh.create_from_point_cloud_poisson behind the reference's `gs-mesh dn / gaussians / sugar-coarse`
// exporters.  The discrete system (DESIGN.md §2 (6), restated in fp64 by oracle/poisson_ref.py):
//
//   grid    R = 2^depth cells per axis, chi at the cell centres; node n = (i * R + j) * R + k.  u = (p - origin) / h.
//   faces   V_a[n] lives on the face between cell n and its +a neighbour (MAC layout; the last face per axis is the
//           boundary and stays 0): V_a = sum_p a_p w_pf n_p,a with trilinear (tent) weights w.  G chi = forward
//           difference onto the faces, so G^T G = -Laplacian (7-point, Neumann) and G^T V = -div V exactly.
//   weights a_p = (1 / rho_p) / mean(1 / rho): rho_p = the trilinear splat of sample counts, sum-restricted two levels
//           (R/4 per axis) and interpolated at p.  S_n = sum_p a_p w_pn.
//   system  (-Lap + sigma S) chi = -div V, in units of the finest cell; sigma = point_weight * area_scale, where
//           area_scale = 16 mean(1 / rho) is the surface area per unit weight in cells^2, so a surface node gets about
//           point_weight of screening at every depth.
//
// Determinism: samples are sorted by the Morton code of their finest cell (cub radix sort, stable), every grid node
// gathers from the sorted runs of its 27 neighbouring cells in a fixed order, all sums are in a fixed order (block
// partials + one finishing block), red-black Gauss-Seidel is order-free.  No float atomics: two runs are bit-identical.
//
// Multigrid: level l has R >> l cells per axis, operator 2^l (-Lap_unit) + sigma S_l, S_l = the 8-child sum of S_(l-1),
// right-hand side = the 8-child sum of the finer residual, trilinear prolongation (clamped at the walls), 2 + 2 red-black
// sweeps, the 4^3 coarsest level solved by sweeps in one CTA.  V-cycles until ||b - A chi|| / ||b|| <= tol or the cap;
// one host read of the residual per cycle.  At sigma = 0 the constant is fixed by removing chi's mean.
#include <algorithm>

#include <cub/cub.cuh>

#include "common.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int RED_BLOCKS = 1024;  // fixed block count of the deterministic reductions
constexpr int COARSE_SWEEPS = 400;
constexpr int PRE_SWEEPS = 2, POST_SWEEPS = 2;

__host__ __device__ __forceinline__ uint32_t spread3(uint32_t v) {  // 10 bits -> every third bit
  v &= 0x3ff;
  v = (v | (v << 16)) & 0x030000ff;
  v = (v | (v << 8)) & 0x0300f00f;
  v = (v | (v << 4)) & 0x030c30c3;
  v = (v | (v << 2)) & 0x09249249;
  return v;
}
__host__ __device__ __forceinline__ uint32_t morton(uint32_t i, uint32_t j, uint32_t k) {
  return (spread3(i) << 2) | (spread3(j) << 1) | spread3(k);
}
__device__ __forceinline__ float tent(float d) { return fmaxf(0.f, 1.f - fabsf(d)); }
__host__ __device__ __forceinline__ int64_t lin(int i, int j, int k, int R) { return ((int64_t)i * R + j) * R + k; }

// ---- splat ----------------------------------------------------------------------------------------------------------
struct Geo {
  double origin[3];
  double inv_h;
  int R, depth;
};

__global__ void keys_kernel(Geo g, const float* __restrict__ pts, int n, uint32_t* __restrict__ keys, int32_t* __restrict__ idx) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  int c[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double u = ((double)pts[3 * p + a] - g.origin[a]) * g.inv_h;
    c[a] = (int)fmin(fmax(floor(u), 0.0), (double)(g.R - 1));
  }
  keys[p] = morton(c[0], c[1], c[2]);
  idx[p] = p;
}

// sorted copies: {frac in [0,1]^3 of the finest cell, a_p (filled later)}, {normal, 0}, {colour, 0}
__global__ void gather_kernel(Geo g, const float* __restrict__ pts, const float* __restrict__ nrm, const float* __restrict__ col,
                              const int32_t* __restrict__ order, int n, float4* __restrict__ sf, float4* __restrict__ sn,
                              float4* __restrict__ sc) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  const int p = order[q];
  float f[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double u = ((double)pts[3 * p + a] - g.origin[a]) * g.inv_h;
    const double c = fmin(fmax(floor(u), 0.0), (double)(g.R - 1));
    f[a] = (float)(u - c);  // in [0, 1) except for points clamped into a border cell
  }
  sf[q] = make_float4(f[0], f[1], f[2], 1.f);
  sn[q] = make_float4(nrm[3 * p], nrm[3 * p + 1], nrm[3 * p + 2], 0.f);
  if (col) sc[q] = make_float4(col[3 * p], col[3 * p + 1], col[3 * p + 2], 0.f);
}

// start[c] = first sorted sample whose Morton key is >= c, for c in [0, R^3]
__global__ void cell_start_kernel(const uint32_t* __restrict__ keys, int n, int64_t ncell, int32_t* __restrict__ start) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c > ncell) return;
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if ((int64_t)keys[mid] < c) lo = mid + 1; else hi = mid;
  }
  start[c] = lo;
}

__device__ __forceinline__ void decode(int64_t n, int R, int* i, int* j, int* k) {
  *k = (int)(n % R);
  *j = (int)((n / R) % R);
  *i = (int)(n / ((int64_t)R * R));
}

// One thread per finest node: gathers the samples of the 27 neighbouring cells.  FULL = false: the count splat
// (out0 = sum_p w_pn).  FULL = true: out0 = S, out1[0..2] = the three face grids (weights a_p = sf.w).
template <bool FULL>
__global__ void __launch_bounds__(THREADS) splat_kernel(int R, const int32_t* __restrict__ start, const float4* __restrict__ sf,
                                                        const float4* __restrict__ sn, float* __restrict__ out0,
                                                        float* __restrict__ faces) {
  const int64_t N = (int64_t)R * R * R;
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  int i, j, k;
  decode(n, R, &i, &j, &k);
  float s = 0.f, vx = 0.f, vy = 0.f, vz = 0.f;
  for (int ci = max(i - 1, 0); ci <= min(i + 1, R - 1); ++ci)
    for (int cj = max(j - 1, 0); cj <= min(j + 1, R - 1); ++cj)
      for (int ck = max(k - 1, 0); ck <= min(k + 1, R - 1); ++ck) {
        const uint32_t m = morton(ci, cj, ck);
        const int e = start[m + 1];
        for (int q = start[m]; q < e; ++q) {
          const float4 f = sf[q];
          const float dx = (float)(ci - i) + f.x, dy = (float)(cj - j) + f.y, dz = (float)(ck - k) + f.z;
          const float nx = tent(dx - 0.5f), ny = tent(dy - 0.5f), nz = tent(dz - 0.5f);
          if (!FULL) {
            s += nx * ny * nz;
          } else {
            const float a = f.w;
            const float4 nv = sn[q];
            s += a * (nx * ny * nz);
            vx += a * (tent(dx - 1.f) * ny * nz) * nv.x;
            vy += a * (nx * tent(dy - 1.f) * nz) * nv.y;
            vz += a * (nx * ny * tent(dz - 1.f)) * nv.z;
          }
        }
      }
  out0[n] = s;
  if (FULL) {
    faces[n] = i < R - 1 ? vx : 0.f;  // the face past the last cell is the box wall: zero flux
    faces[N + n] = j < R - 1 ? vy : 0.f;
    faces[2 * N + n] = k < R - 1 ? vz : 0.f;
  }
}

// coarse[n] = sum of the 8 children (Rc = R / 2 cells per axis on the coarse side)
__global__ void restrict_sum_kernel(int Rc, const float* __restrict__ fine, float* __restrict__ coarse) {
  const int64_t Nc = (int64_t)Rc * Rc * Rc;
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= Nc) return;
  int I, J, K;
  decode(n, Rc, &I, &J, &K);
  const int R = 2 * Rc;
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < 8; ++c) s += fine[lin(2 * I + (c >> 2), 2 * J + ((c >> 1) & 1), 2 * K + (c & 1), R)];
  coarse[n] = s;
}

// trilinear weights of a cell-centred grid with Rc nodes per axis at coordinate x (in that grid's cell units), clamped
__device__ __forceinline__ void lerp_axis(float x, int Rc, int* i0, int* i1, float* t) {
  const float y = x - 0.5f;
  int a = (int)floorf(y);
  float tt = y - (float)a;
  if (a < 0) { a = 0; tt = 0.f; }
  if (a >= Rc - 1) { a = Rc - 1; tt = 0.f; }
  *i0 = a;
  *i1 = min(a + 1, Rc - 1);
  *t = tt;
}

// rho_p: the level-2 count grid interpolated at the sample; sf.w = 1 / rho_p (normalised later)
__global__ void rho_kernel(int R, const uint32_t* __restrict__ keys, const float* __restrict__ count2, int n,
                           float4* __restrict__ sf) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  const uint32_t key = keys[q];
  int c[3] = {0, 0, 0};
  for (int b = 0; b < 10; ++b) {
    c[0] |= ((key >> (3 * b + 2)) & 1) << b;
    c[1] |= ((key >> (3 * b + 1)) & 1) << b;
    c[2] |= ((key >> (3 * b)) & 1) << b;
  }
  const float4 f = sf[q];
  const float fr[3] = {f.x, f.y, f.z};
  const int R2 = R >> 2;
  int i0[3], i1[3];
  float t[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const int base = c[a] >> 2;  // level-2 cell; coordinate = base + ((c & 3) + frac) / 4, exact in fp32
    const float x = (float)base + ((float)(c[a] & 3) + fr[a]) * 0.25f;
    lerp_axis(x, R2, &i0[a], &i1[a], &t[a]);
  }
  float rho = 0.f;
#pragma unroll
  for (int cc = 0; cc < 8; ++cc) {
    const int ia = (cc >> 2) ? i1[0] : i0[0], ja = ((cc >> 1) & 1) ? i1[1] : i0[1], ka = (cc & 1) ? i1[2] : i0[2];
    const float w = ((cc >> 2) ? t[0] : 1.f - t[0]) * (((cc >> 1) & 1) ? t[1] : 1.f - t[1]) * ((cc & 1) ? t[2] : 1.f - t[2]);
    rho += w * count2[lin(ia, ja, ka, R2)];
  }
  sf[q].w = 1.f / fmaxf(rho, 1e-20f);
}

// deterministic sums: block partials over a fixed block count, then one block finishes in a fixed order
__device__ __forceinline__ double block_sum(double v) {
  __shared__ double sh[THREADS];
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int s = THREADS / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  const double r = sh[0];
  __syncthreads();
  return r;
}

__global__ void __launch_bounds__(THREADS) sum_w_partials(const float4* __restrict__ sf, int n, double* __restrict__ part) {
  double s = 0.0;
  for (int q = blockIdx.x * THREADS + threadIdx.x; q < n; q += gridDim.x * THREADS) s += sf[q].w;
  s = block_sum(s);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}

__global__ void __launch_bounds__(THREADS) finish_sum(const double* __restrict__ part, int nparts, double* __restrict__ out) {
  double s = 0.0;
  for (int q = threadIdx.x; q < nparts; q += THREADS) s += part[q];
  s = block_sum(s);
  if (threadIdx.x == 0) *out = s;
}

// a_p = (1 / rho_p) / mean(1 / rho); area_scale = 16 mean(1 / rho); weights_out[original index] = a_p
__global__ void normalise_kernel(float4* __restrict__ sf, const int32_t* __restrict__ order, int n, const double* __restrict__ sum,
                                 float* __restrict__ weights_out, float* __restrict__ area_scale) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  const double mean = *sum / (double)n;
  if (q == 0 && area_scale) *area_scale = (float)(16.0 * mean);
  if (q >= n) return;
  const float a = (float)((double)sf[q].w / mean);
  sf[q].w = a;
  if (weights_out) weights_out[order[q]] = a;
}

// colour grid at level 2: {sum a w c (3 channels), sum a w} over the samples of the 27 neighbouring level-2 cells (each
// a Morton run of 64 finest cells).  The weighted mean is taken after interpolation, so that nodes no sample reaches
// do not darken the vertices next to them.
__global__ void __launch_bounds__(THREADS) color_kernel(int R, const int32_t* __restrict__ start, const uint32_t* __restrict__ keys,
                                                        const float4* __restrict__ sf, const float4* __restrict__ sc,
                                                        float* __restrict__ out) {
  const int R2 = R >> 2;
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= (int64_t)R2 * R2 * R2) return;
  int I, J, K;
  decode(n, R2, &I, &J, &K);
  double w = 0.0, r = 0.0, gg = 0.0, b = 0.0;  // a level-2 node sums ~64x more samples than a finest one
  for (int ci = max(I - 1, 0); ci <= min(I + 1, R2 - 1); ++ci)
    for (int cj = max(J - 1, 0); cj <= min(J + 1, R2 - 1); ++cj)
      for (int ck = max(K - 1, 0); ck <= min(K + 1, R2 - 1); ++ck) {
        const uint32_t m = morton(ci, cj, ck);
        const int e = start[(m + 1) << 6];
        for (int q = start[m << 6]; q < e; ++q) {
          const uint32_t key = keys[q];
          const float4 f = sf[q];
          // position in level-2 units relative to node I: ((fine cell & 3) + frac) / 4 + (ci - I) - 0.5
          const float dx = (float)(ci - I) + ((float)(((key >> 2) & 1) | (((key >> 5) & 1) << 1)) + f.x) * 0.25f;
          const float dy = (float)(cj - J) + ((float)(((key >> 1) & 1) | (((key >> 4) & 1) << 1)) + f.y) * 0.25f;
          const float dz = (float)(ck - K) + ((float)((key & 1) | (((key >> 3) & 1) << 1)) + f.z) * 0.25f;
          const float ww = f.w * (tent(dx - 0.5f) * tent(dy - 0.5f) * tent(dz - 0.5f));
          const float4 c = sc[q];
          w += ww;
          r += ww * c.x;
          gg += ww * c.y;
          b += ww * c.z;
        }
      }
  out[4 * n] = (float)r;
  out[4 * n + 1] = (float)gg;
  out[4 * n + 2] = (float)b;
  out[4 * n + 3] = (float)w;
}

struct SplatLayout {
  DnrCarver carve;
  uint32_t *keys_in, *keys_out;
  int32_t *idx_in, *idx_out, *start;
  void* cub_temp;
  size_t cub_bytes = 0;
  float4 *sf, *sn, *sc;
  float *count0, *count1;
  double *part, *sum;
  SplatLayout(void* base, int depth, int64_t n) : carve(base) {
    const int64_t R = 1ll << depth, N = R * R * R;
    keys_in = carve.take<uint32_t>(n);
    keys_out = carve.take<uint32_t>(n);
    idx_in = carve.take<int32_t>(n);
    idx_out = carve.take<int32_t>(n);
    const cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                                          (const int32_t*)nullptr, (int32_t*)nullptr, (int)n, 0, 3 * depth);
    cub_temp = carve.cub_scratch(e, cub_bytes);
    sf = carve.take<float4>(n);
    sn = carve.take<float4>(n);
    sc = carve.take<float4>(n);
    start = carve.take<int32_t>(N + 1);
    count0 = carve.take<float>(N);
    count1 = carve.take<float>(N / 8);
    part = carve.take<double>(RED_BLOCKS);
    sum = carve.take<double>(1);
  }
};

int check_grid(const DnrPoissonGrid* g, Geo* geo) {
  if (!g) return DNR_E_NULL;
  if (g->depth < DNR_POISSON_MIN_DEPTH || g->depth > DNR_POISSON_MAX_DEPTH) return DNR_E_SIZE;
  if (!(g->cell > 0.f)) return DNR_E_SIZE;
  for (int a = 0; a < 3; ++a) geo->origin[a] = g->origin[a];
  geo->inv_h = 1.0 / (double)g->cell;
  geo->depth = g->depth;
  geo->R = 1 << g->depth;
  return 0;
}

unsigned blocks_for(int64_t n) { return (unsigned)((n + THREADS - 1) / THREADS); }

// ---- multigrid ------------------------------------------------------------------------------------------------------
struct Level {
  int R;
  float c;  // Laplacian coefficient 2^l
  float* x;
  float* b;
  const float* S;
};

// residual at node (i, j, k): b - c sum_nb (x_n - x_nb) - sigma S_n x_n (difference form: exact for smooth x)
__device__ __forceinline__ float node_residual(const Level& L, float sigma, int i, int j, int k, float* diag) {
  const int R = L.R;
  const int64_t n = lin(i, j, k, R);
  const float xn = L.x[n];
  float acc = 0.f;
  int nb = 0;
  const int64_t RR = (int64_t)R * R;
  if (i > 0) { acc += xn - L.x[n - RR]; ++nb; }
  if (i < R - 1) { acc += xn - L.x[n + RR]; ++nb; }
  if (j > 0) { acc += xn - L.x[n - R]; ++nb; }
  if (j < R - 1) { acc += xn - L.x[n + R]; ++nb; }
  if (k > 0) { acc += xn - L.x[n - 1]; ++nb; }
  if (k < R - 1) { acc += xn - L.x[n + 1]; ++nb; }
  const float s = sigma * L.S[n];
  *diag = L.c * (float)nb + s;
  return L.b[n] - L.c * acc - s * xn;
}

__global__ void __launch_bounds__(THREADS) rbgs_kernel(Level L, float sigma, int color) {
  const int R = L.R, half = R >> 1;
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)R * R * half) return;
  const int k2 = (int)(t % half);
  const int j = (int)((t / half) % R);
  const int i = (int)(t / ((int64_t)half * R));
  const int k = 2 * k2 + ((i + j + color) & 1);
  float diag;
  const float r = node_residual(L, sigma, i, j, k, &diag);
  if (diag > 0.f) L.x[lin(i, j, k, R)] += r / diag;
}

// coarse b = 8-child sum of the fine residual
__global__ void __launch_bounds__(THREADS) restrict_residual_kernel(Level F, float sigma, float* __restrict__ bc) {
  const int Rc = F.R >> 1;
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= (int64_t)Rc * Rc * Rc) return;
  int I, J, K;
  decode(n, Rc, &I, &J, &K);
  float s = 0.f, d;
#pragma unroll
  for (int c = 0; c < 8; ++c) s += node_residual(F, sigma, 2 * I + (c >> 2), 2 * J + ((c >> 1) & 1), 2 * K + (c & 1), &d);
  bc[n] = s;
}

// fine x += trilinear interpolation of the coarse correction (cell-centred; clamped at the walls)
__global__ void __launch_bounds__(THREADS) prolong_kernel(int R, float* __restrict__ x, const float* __restrict__ xc) {
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= (int64_t)R * R * R) return;
  int i, j, k;
  decode(n, R, &i, &j, &k);
  const int Rc = R >> 1;
  int a0[3], a1[3];
  float t[3];
  const int p[3] = {i, j, k};
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const int q = p[a] >> 1;
    if (p[a] & 1) { a0[a] = q; a1[a] = min(q + 1, Rc - 1); t[a] = 0.25f; }
    else { a0[a] = max(q - 1, 0); a1[a] = q; t[a] = 0.75f; }
  }
  float v = 0.f;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const float w = ((c >> 2) ? t[0] : 1.f - t[0]) * (((c >> 1) & 1) ? t[1] : 1.f - t[1]) * ((c & 1) ? t[2] : 1.f - t[2]);
    v += w * xc[lin((c >> 2) ? a1[0] : a0[0], ((c >> 1) & 1) ? a1[1] : a0[1], (c & 1) ? a1[2] : a0[2], Rc)];
  }
  x[n] += v;
}

// coarsest level (R^3 <= 4096 nodes) in one CTA: b's mean removed when sigma == 0 (the Neumann problem is singular),
// COARSE_SWEEPS red-black sweeps from zero, mean of x removed again
__global__ void __launch_bounds__(1024) coarse_solve_kernel(Level L, float sigma) {
  const int R = L.R, N = R * R * R;
  __shared__ double red[1024];
  if (sigma == 0.f) {
    double s = 0.0;
    for (int n = threadIdx.x; n < N; n += blockDim.x) s += L.b[n];
    red[threadIdx.x] = s;
    __syncthreads();
    for (int h = blockDim.x / 2; h > 0; h >>= 1) {
      if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
      __syncthreads();
    }
    const float mean = (float)(red[0] / N);
    __syncthreads();
    for (int n = threadIdx.x; n < N; n += blockDim.x) L.b[n] -= mean;
  }
  for (int n = threadIdx.x; n < N; n += blockDim.x) L.x[n] = 0.f;
  __syncthreads();
  for (int sweep = 0; sweep < COARSE_SWEEPS; ++sweep)
    for (int color = 0; color < 2; ++color) {
      for (int n = threadIdx.x; n < N; n += blockDim.x) {
        const int k = n % R, j = (n / R) % R, i = n / (R * R);
        if (((i + j + k) & 1) != color) continue;
        float diag;
        const float r = node_residual(L, sigma, i, j, k, &diag);
        if (diag > 0.f) L.x[n] += r / diag;
      }
      __syncthreads();
    }
  if (sigma == 0.f) {
    double s = 0.0;
    for (int n = threadIdx.x; n < N; n += blockDim.x) s += L.x[n];
    red[threadIdx.x] = s;
    __syncthreads();
    for (int h = blockDim.x / 2; h > 0; h >>= 1) {
      if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
      __syncthreads();
    }
    const float mean = (float)(red[0] / N);
    for (int n = threadIdx.x; n < N; n += blockDim.x) L.x[n] -= mean;
  }
}

// b = -div V (faces [3, N]; the face below the first cell is the wall)
__global__ void __launch_bounds__(THREADS) rhs_kernel(int R, const float* __restrict__ V, float* __restrict__ b) {
  const int64_t N = (int64_t)R * R * R;
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  int i, j, k;
  decode(n, R, &i, &j, &k);
  float d = V[n] - (i > 0 ? V[n - (int64_t)R * R] : 0.f);
  d += V[N + n] - (j > 0 ? V[N + n - R] : 0.f);
  d += V[2 * N + n] - (k > 0 ? V[2 * N + n - 1] : 0.f);
  b[n] = -d;
}

// MODE 0: partials of sum r^2 (residual); 1: sum b^2; 2: sum x
template <int MODE>
__global__ void __launch_bounds__(THREADS) norm_partials(Level L, float sigma, double* __restrict__ part) {
  const int R = L.R;
  const int64_t N = (int64_t)R * R * R;
  double s = 0.0;
  for (int64_t n = (int64_t)blockIdx.x * THREADS + threadIdx.x; n < N; n += (int64_t)gridDim.x * THREADS) {
    if (MODE == 0) {
      int i, j, k;
      decode(n, R, &i, &j, &k);
      float d;
      const float r = node_residual(L, sigma, i, j, k, &d);
      s += (double)r * r;
    } else if (MODE == 1) {
      s += (double)L.b[n] * L.b[n];
    } else {
      s += L.x[n];
    }
  }
  s = block_sum(s);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}

__global__ void subtract_mean_kernel(float* __restrict__ x, int64_t N, const double* __restrict__ sum) {
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n < N) x[n] -= (float)(*sum / (double)N);
}

struct SolveLayout {
  DnrCarver carve;
  float* b0;
  float* lvl[DNR_POISSON_MAX_DEPTH][3];  // lvl[l] = {x, b, S} for l >= 1
  double *part, *hist;
  int levels;  // number of levels incl. the finest
  SolveLayout(void* base, int depth, int max_cycles) : carve(base) {
    const int64_t R = 1ll << depth;
    b0 = carve.take<float>(R * R * R);
    levels = depth - 1;  // down to 4^3
    for (int l = 1; l < levels; ++l) {
      const int64_t Rl = R >> l, Nl = Rl * Rl * Rl;
      for (int q = 0; q < 3; ++q) lvl[l][q] = carve.take<float>(Nl);
    }
    part = carve.take<double>(RED_BLOCKS);
    hist = carve.take<double>(max_cycles + 2);
  }
};

unsigned red_blocks(int64_t N) { return (unsigned)std::min<int64_t>(RED_BLOCKS, (N + THREADS - 1) / THREADS); }

template <int MODE>
int reduce(const Level& L, float sigma, double* part, double* out, cudaStream_t s) {
  const int64_t N = (int64_t)L.R * L.R * L.R;
  const unsigned nb = red_blocks(N);
  norm_partials<MODE><<<nb, THREADS, 0, s>>>(L, sigma, part);
  DNR_CHECK_LAUNCH();
  finish_sum<<<1, THREADS, 0, s>>>(part, (int)nb, out);
  DNR_CHECK_LAUNCH();
  return 0;
}

int smooth(const Level& L, float sigma, int sweeps, cudaStream_t s) {
  const int64_t half = (int64_t)L.R * L.R * (L.R / 2);
  for (int it = 0; it < sweeps; ++it)
    for (int color = 0; color < 2; ++color) {
      rbgs_kernel<<<blocks_for(half), THREADS, 0, s>>>(L, sigma, color);
      DNR_CHECK_LAUNCH();
    }
  return 0;
}

int vcycle(Level* lv, int l, int levels, float sigma, cudaStream_t s) {
  if (l == levels - 1) {
    coarse_solve_kernel<<<1, 1024, 0, s>>>(lv[l], sigma);
    DNR_CHECK_LAUNCH();
    return 0;
  }
  int rc = smooth(lv[l], sigma, PRE_SWEEPS, s);
  if (rc) return rc;
  const int64_t Nc = (int64_t)lv[l + 1].R * lv[l + 1].R * lv[l + 1].R;
  restrict_residual_kernel<<<blocks_for(Nc), THREADS, 0, s>>>(lv[l], sigma, lv[l + 1].b);
  DNR_CHECK_LAUNCH();
  if (l + 1 < levels - 1) DNR_CUDA(cudaMemsetAsync(lv[l + 1].x, 0, 4 * (size_t)Nc, s));
  rc = vcycle(lv, l + 1, levels, sigma, s);
  if (rc) return rc;
  const int64_t N = (int64_t)lv[l].R * lv[l].R * lv[l].R;
  prolong_kernel<<<blocks_for(N), THREADS, 0, s>>>(lv[l].R, lv[l].x, lv[l + 1].x);
  DNR_CHECK_LAUNCH();
  return smooth(lv[l], sigma, POST_SWEEPS, s);
}

// ---- trilinear sampling ---------------------------------------------------------------------------------------------
__global__ void grid_sample_kernel(DnrGridDesc d, const float* __restrict__ grid, const float* __restrict__ pts, int64_t n,
                                   float* __restrict__ out) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  int i0[3], i1[3];
  float t[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double x = ((double)pts[3 * q + a] - (double)d.origin[a]) / (double)d.cell - 0.5;
    double fl = floor(x);
    double tt = x - fl;
    int lo = (int)fl;
    if (fl < 0.0) { lo = 0; tt = 0.0; }
    if (fl >= (double)(d.dims[a] - 1)) { lo = d.dims[a] - 1; tt = 0.0; }
    i0[a] = lo;
    i1[a] = min(lo + 1, d.dims[a] - 1);
    t[a] = (float)tt;
  }
  const int C = d.channels;
  for (int ch = 0; ch < C; ++ch) {
    float v = 0.f;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const float w = ((c >> 2) ? t[0] : 1.f - t[0]) * (((c >> 1) & 1) ? t[1] : 1.f - t[1]) * ((c & 1) ? t[2] : 1.f - t[2]);
      const int64_t node = ((int64_t)((c >> 2) ? i1[0] : i0[0]) * d.dims[1] + (((c >> 1) & 1) ? i1[1] : i0[1])) * d.dims[2] +
                           ((c & 1) ? i1[2] : i0[2]);
      v += w * grid[node * C + ch];
    }
    out[q * C + ch] = v;
  }
}

}  // namespace

extern "C" int64_t dnr_poisson_splat_workspace_bytes(const DnrPoissonGrid* grid, int64_t n_points) {
  Geo g;
  const int rc = check_grid(grid, &g);
  if (rc) return rc;
  if (n_points <= 0 || n_points > INT32_MAX) return DNR_E_SIZE;
  return (int64_t)SplatLayout(nullptr, g.depth, n_points).carve.total();
}

extern "C" int dnr_poisson_splat(const DnrPoissonGrid* grid, const float* points, const float* normals, const float* colors,
                                 int64_t n_points, void* ws, int64_t ws_bytes, float* screen, float* faces, float* density,
                                 float* color_grid, float* weights, float* area_scale, void* stream) {
  Geo g;
  const int rc = check_grid(grid, &g);
  if (rc) return rc;
  if (n_points <= 0 || n_points > INT32_MAX) return DNR_E_SIZE;
  if (!points || !normals || !ws || !screen || !faces || !density || !area_scale) return DNR_E_NULL;
  if ((colors == nullptr) != (color_grid == nullptr)) return DNR_E_NULL;
  const SplatLayout L(ws, g.depth, n_points);
  if (const int e = L.carve.check(ws_bytes)) return e;
  cudaStream_t s = (cudaStream_t)stream;
  const int n = (int)n_points, R = g.R;
  const int64_t N = (int64_t)R * R * R;
  uint32_t *keys_in = L.keys_in, *keys = L.keys_out;
  int32_t *idx_in = L.idx_in, *order = L.idx_out, *start = L.start;
  float4 *sf = L.sf, *sn = L.sn, *sc = L.sc;
  float *count0 = L.count0, *count1 = L.count1;
  double *part = L.part, *sum = L.sum;

  keys_kernel<<<blocks_for(n), THREADS, 0, s>>>(g, points, n, keys_in, idx_in);
  DNR_CHECK_LAUNCH();
  size_t temp = L.cub_bytes;
  DNR_CUDA(cub::DeviceRadixSort::SortPairs(L.cub_temp, temp, keys_in, keys, idx_in, order, n, 0, 3 * g.depth, s));
  gather_kernel<<<blocks_for(n), THREADS, 0, s>>>(g, points, normals, colors, order, n, sf, sn, sc);
  DNR_CHECK_LAUNCH();
  cell_start_kernel<<<blocks_for(N + 1), THREADS, 0, s>>>(keys, n, N, start);
  DNR_CHECK_LAUNCH();
  splat_kernel<false><<<blocks_for(N), THREADS, 0, s>>>(R, start, sf, sn, count0, nullptr);
  DNR_CHECK_LAUNCH();
  restrict_sum_kernel<<<blocks_for(N / 8), THREADS, 0, s>>>(R / 2, count0, count1);
  DNR_CHECK_LAUNCH();
  restrict_sum_kernel<<<blocks_for(N / 64), THREADS, 0, s>>>(R / 4, count1, density);
  DNR_CHECK_LAUNCH();
  rho_kernel<<<blocks_for(n), THREADS, 0, s>>>(R, keys, density, n, sf);
  DNR_CHECK_LAUNCH();
  const unsigned nb = red_blocks(n);
  sum_w_partials<<<nb, THREADS, 0, s>>>(sf, n, part);
  DNR_CHECK_LAUNCH();
  finish_sum<<<1, THREADS, 0, s>>>(part, (int)nb, sum);
  DNR_CHECK_LAUNCH();
  normalise_kernel<<<blocks_for(n), THREADS, 0, s>>>(sf, order, n, sum, weights, area_scale);
  DNR_CHECK_LAUNCH();
  splat_kernel<true><<<blocks_for(N), THREADS, 0, s>>>(R, start, sf, sn, screen, faces);
  DNR_CHECK_LAUNCH();
  if (colors) {
    color_kernel<<<blocks_for(N / 64), THREADS, 0, s>>>(R, start, keys, sf, sc, color_grid);
    DNR_CHECK_LAUNCH();
  }
  return 0;
}

extern "C" int64_t dnr_poisson_solve_workspace_bytes(const DnrPoissonGrid* grid, int32_t max_cycles) {
  Geo g;
  const int rc = check_grid(grid, &g);
  if (rc) return rc;
  if (max_cycles < 1 || max_cycles > DNR_POISSON_MAX_CYCLES) return DNR_E_SIZE;
  return (int64_t)SolveLayout(nullptr, g.depth, max_cycles).carve.total();
}

extern "C" int dnr_poisson_solve(const DnrPoissonGrid* grid, const float* screen, const float* faces, float screen_weight,
                                 float tol, int32_t max_cycles, void* ws, int64_t ws_bytes, float* chi, float* residual_host,
                                 int32_t* cycles_host, void* stream) {
  Geo g;
  const int rc0 = check_grid(grid, &g);
  if (rc0) return rc0;
  if (max_cycles < 1 || max_cycles > DNR_POISSON_MAX_CYCLES) return DNR_E_SIZE;
  if (!(screen_weight >= 0.f) || !(tol >= 0.f)) return DNR_E_SIZE;
  if (!screen || !faces || !ws || !chi || !residual_host || !cycles_host) return DNR_E_NULL;
  const SolveLayout SL(ws, g.depth, max_cycles);
  if (const int e = SL.carve.check(ws_bytes)) return e;
  cudaStream_t s = (cudaStream_t)stream;
  const int R = g.R;
  const int64_t N = (int64_t)R * R * R;
  Level lv[DNR_POISSON_MAX_DEPTH];
  lv[0] = Level{R, 1.f, chi, SL.b0, screen};
  for (int l = 1; l < SL.levels; ++l) lv[l] = Level{R >> l, (float)(1 << l), SL.lvl[l][0], SL.lvl[l][1], SL.lvl[l][2]};
  double *part = SL.part, *hist = SL.hist;  // hist[0] = ||b||^2, [c] = ||r||^2 after cycle c

  rhs_kernel<<<blocks_for(N), THREADS, 0, s>>>(R, faces, lv[0].b);
  DNR_CHECK_LAUNCH();
  for (int l = 1; l < SL.levels; ++l) {
    const int64_t Nl = (int64_t)lv[l].R * lv[l].R * lv[l].R;
    restrict_sum_kernel<<<blocks_for(Nl), THREADS, 0, s>>>(lv[l].R, lv[l - 1].S, (float*)lv[l].S);
    DNR_CHECK_LAUNCH();
  }
  DNR_CUDA(cudaMemsetAsync(chi, 0, 4 * (size_t)N, s));
  int rc = reduce<1>(lv[0], screen_weight, part, hist, s);
  if (rc) return rc;
  double b2 = 0.0;
  DNR_CUDA(cudaMemcpyAsync(&b2, hist, 8, cudaMemcpyDeviceToHost, s));
  DNR_CUDA(cudaStreamSynchronize(s));
  residual_host[0] = b2 > 0.0 ? 1.f : 0.f;
  int cycles = 0;
  while (b2 > 0.0 && cycles < max_cycles) {
    rc = vcycle(lv, 0, SL.levels, screen_weight, s);
    if (rc) return rc;
    ++cycles;
    rc = reduce<0>(lv[0], screen_weight, part, hist + cycles, s);
    if (rc) return rc;
    double r2 = 0.0;
    DNR_CUDA(cudaMemcpyAsync(&r2, hist + cycles, 8, cudaMemcpyDeviceToHost, s));
    DNR_CUDA(cudaStreamSynchronize(s));  // the one host read per cycle
    const float rel = (float)sqrt(r2 / b2);
    residual_host[cycles] = rel;
    if (rel <= tol) break;
  }
  if (screen_weight == 0.f && cycles > 0) {
    rc = reduce<2>(lv[0], 0.f, part, hist + max_cycles + 1, s);
    if (rc) return rc;
    subtract_mean_kernel<<<blocks_for(N), THREADS, 0, s>>>(chi, N, hist + max_cycles + 1);
    DNR_CHECK_LAUNCH();
  }
  *cycles_host = cycles;
  return 0;
}

extern "C" int dnr_grid_sample(const DnrGridDesc* grid, const float* values, const float* points, int64_t n_points,
                               float* out, void* stream) {
  if (!grid) return DNR_E_NULL;
  for (int a = 0; a < 3; ++a)
    if (grid->dims[a] <= 0) return DNR_E_SIZE;
  if (!(grid->cell > 0.f) || grid->channels <= 0 || n_points < 0) return DNR_E_SIZE;
  if (n_points == 0) return 0;
  if (!values || !points || !out) return DNR_E_NULL;
  grid_sample_kernel<<<blocks_for(n_points), THREADS, 0, (cudaStream_t)stream>>>(*grid, values, points, n_points, out);
  DNR_CHECK_LAUNCH();
  return 0;
}
