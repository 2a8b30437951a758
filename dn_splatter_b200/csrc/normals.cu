// AGS-Mesh depth confidence masks on the device: the reference's scripts/depth_normal_consistency.py and
// scripts/depth_to_normal.py (DESIGN.md §2, deviation 9).  Three calls:
//
// dnr_dn_backproject   a depth frame -> world points [h*w,3] f64.  The camera coordinates are formed in fp32 exactly as
//                      numpy forms them ((u + 0.5 - cx) * d / fx, one rounding per operation: built with -fmad=false),
//                      then rotated by inv(R) (computed on the host) and offset by t in fp64.
// dnr_dn_normals       Open3D's estimate_normals(KDTreeSearchParamKNN(k)) with fast_normal_computation [EXT]: the k
//                      nearest points of every point (itself included), their covariance from fp64 cumulants, the
//                      eigenvector of its smallest eigenvalue by FastEigen3x3, (0, 0, 1) for a zero vector; then the
//                      scripts' orientation (negated where (p - centre) . n > 0).
// dnr_dn_consistency   the mono-normal decode, rotation and angle test of either script, and the uint8 encodings.
//
// Neighbour search.  Exact duplicates are collapsed first (every hole pixel of a depth map lands on the camera centre):
// the points are sorted stably by their coordinate bits and then by a 63-bit Morton key of a 2^21-per-axis grid over
// their bounding box, so equal points are adjacent, each distinct position gets one entry with its multiplicity and its
// smallest point index, and every Morton cell of every level is one contiguous range of entries.  Neighbours are taken
// in (fp64 squared distance, smallest index) order, all copies of a position before the next position, which fixes the
// result where nanoflann's order among equidistant points cannot be reproduced.  One warp per distinct position:
//   1. a position with multiplicity >= k is its own k neighbours (no search);
//   2. the window of k entries on either side in Morton order holds >= k points, so the k-th smallest key over it bounds
//      the true k-th distance R (if the window is every entry, it is the answer);
//   3. every cell of the level whose cell edge is >= R/2 that the box [q - R, q + R] touches is scanned; candidates whose
//      key exceeds the running k-th key are dropped, and the shared-memory buffer is cut back to its k best by a
//      weighted radix select whenever it fills.
// The cell of a coordinate is floor((x - lo) / cell) clamped to the grid, a monotone function of x, so a point within
// R of the query along every axis lies in a visited cell (R carries a 2^-40 relative margin over the rounded distance and
// is at least 2^-510, which covers squared distances that underflowed).
// Work per query therefore depends on the local density only, not on how many points coincide.
#include <cub/cub.cuh>

#include "common.cuh"

namespace {

constexpr int MORTON_BITS = 21;
constexpr int CAP = 768;          // candidate buffer entries per warp (>= 2 * DNR_DN_MAX_K + 1 + 32)
constexpr int QWARPS = 2;         // warps per block of the query kernel (32 KB of static shared memory)
constexpr int LEVEL_DIV = 2;      // scan cells of edge >= R / LEVEL_DIV

struct NrmLayout {
  DnrCarver carve;
  uint64_t *keys_a, *keys_b, *ukey;
  int32_t *vals_a, *vals_b, *scan, *ustart, *umin, *ucount;
  double *upts, *unormal;
  void* cub_temp;
  size_t cub_bytes;
  NrmLayout(void* base, int64_t n) : carve(base) {
    const size_t N = (size_t)n;
    keys_a = carve.take<uint64_t>(N);
    keys_b = carve.take<uint64_t>(N);
    vals_a = carve.take<int32_t>(N);
    vals_b = carve.take<int32_t>(N);
    scan = carve.take<int32_t>(N);
    ustart = carve.take<int32_t>(N + 1);
    upts = carve.take<double>(3 * N);
    ukey = carve.take<uint64_t>(N);
    umin = carve.take<int32_t>(N);
    unormal = carve.take<double>(3 * N);
    ucount = carve.take<int32_t>(N);
    size_t t1 = 0, t2 = 0;
    const cudaError_t e1 = cub::DeviceRadixSort::SortPairs(nullptr, t1, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                                                           (const int32_t*)nullptr, (int32_t*)nullptr, (int)n, 0, 64);
    const cudaError_t e2 = cub::DeviceScan::InclusiveSum(nullptr, t2, (const int32_t*)nullptr, (int32_t*)nullptr, (int)n);
    cub_bytes = t1 > t2 ? t1 : t2;
    cub_temp = carve.cub_scratch(e1 != cudaSuccess ? e1 : e2, cub_bytes);
  }
};

struct GridP {
  double lo[3], inv_cell;
};

__device__ __forceinline__ uint32_t cell_of(double x, double lo, double inv) {
  const double c = floor((x - lo) * inv);
  return (uint32_t)fmin(fmax(c, 0.0), (double)((1 << MORTON_BITS) - 1));
}

__device__ __forceinline__ uint64_t spread3(uint32_t v) {
  uint64_t x = v & 0x1fffff;
  x = (x | x << 32) & 0x1f00000000ffffull;
  x = (x | x << 16) & 0x1f0000ff0000ffull;
  x = (x | x << 8) & 0x100f00f00f00f00full;
  x = (x | x << 4) & 0x10c30c30c30c30c3ull;
  x = (x | x << 2) & 0x1249249249249249ull;
  return x;
}

__device__ __forceinline__ uint64_t morton(uint32_t cx, uint32_t cy, uint32_t cz) {
  return spread3(cx) | spread3(cy) << 1 | spread3(cz) << 2;
}

// pass 0..2: the bits of coordinate 2 - pass (+0.0 folds -0.0 into +0.0); pass 3: the Morton key
__global__ void nrm_keys_kernel(const double* __restrict__ pts, int n, int pass, GridP g, const int32_t* __restrict__ vals,
                                uint64_t* __restrict__ keys, int32_t* __restrict__ vals_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int src = pass == 0 ? i : vals[i];
  if (pass == 0) vals_out[i] = i;
  const double* p = pts + 3 * (size_t)src;
  if (pass < 3) {
    keys[i] = (uint64_t)__double_as_longlong(p[2 - pass] + 0.0);
  } else {
    keys[i] = morton(cell_of(p[0], g.lo[0], g.inv_cell), cell_of(p[1], g.lo[1], g.inv_cell), cell_of(p[2], g.lo[2], g.inv_cell));
  }
}

__device__ __forceinline__ bool same_point(const double* a, const double* b) {
  return a[0] == b[0] && a[1] == b[1] && a[2] == b[2];
}

__global__ void nrm_heads_kernel(const double* __restrict__ pts, int n, const int32_t* __restrict__ order, int32_t* __restrict__ head) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  head[i] = (i == 0 || !same_point(pts + 3 * (size_t)order[i], pts + 3 * (size_t)order[i - 1])) ? 1 : 0;
}

__global__ void nrm_unique_kernel(const double* __restrict__ pts, int n, const int32_t* __restrict__ order,
                                  const uint64_t* __restrict__ keys, const int32_t* __restrict__ scan, int32_t* __restrict__ ustart,
                                  double* __restrict__ upts, uint64_t* __restrict__ ukey, int32_t* __restrict__ umin) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int u = scan[i] - 1;
  const int src = order[i];
  if (i == 0 || scan[i - 1] != scan[i]) {  // the first (smallest-index: the sorts are stable) copy of a position
    ustart[u] = i;
    for (int a = 0; a < 3; ++a) upts[3 * (size_t)u + a] = pts[3 * (size_t)src + a];
    ukey[u] = keys[i];
    umin[u] = src;
  }
  if (i == n - 1) ustart[u + 1] = n;
}

struct WarpBuf {
  double d2[CAP];
  int32_t mi[CAP];
  int32_t w[CAP];
  int32_t u[CAP];
  uint32_t hist[256];
};

__device__ __forceinline__ unsigned lanemask_lt() {
  unsigned m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}

struct Key {
  uint64_t hi;  // bits of the squared distance (non-negative doubles order as unsigned integers)
  uint32_t lo;  // smallest point index of the position
};

__device__ __forceinline__ bool key_le(uint64_t h, uint32_t l, const Key& t) { return h < t.hi || (h == t.hi && l <= t.lo); }

// The key T of the kk-th point (by weight) among buf[0, cnt) in (d2, index) order, and rem: how many copies of T's position
// complete the kk (1 <= rem <= its weight).  Keys are distinct, so W(< T) = kk - rem.  Twelve 8-bit passes, MSB first.
__device__ Key weighted_select(WarpBuf& b, int cnt, uint32_t kk, uint32_t& rem_out) {
  const int lane = threadIdx.x & 31;
  uint64_t pref_hi = 0, mask_hi = 0;
  uint32_t pref_lo = 0, mask_lo = 0;
  uint32_t rem = kk;
  for (int pass = 0; pass < 12; ++pass) {
    for (int j = lane; j < 256; j += 32) b.hist[j] = 0;
    __syncwarp();
    const bool in_hi = pass < 8;
    const int shift = in_hi ? 56 - 8 * pass : 24 - 8 * (pass - 8);
    for (int i = lane; i < cnt; i += 32) {
      const uint64_t h = (uint64_t)__double_as_longlong(b.d2[i]);
      const uint32_t l = (uint32_t)b.mi[i];
      if ((h & mask_hi) != pref_hi || (l & mask_lo) != pref_lo) continue;
      const uint32_t digit = in_hi ? (uint32_t)(h >> shift) & 255u : (l >> shift) & 255u;
      atomicAdd(&b.hist[digit], (uint32_t)b.w[i]);
    }
    __syncwarp();
    uint32_t loc[8], s = 0;
    for (int j = 0; j < 8; ++j) {
      loc[j] = b.hist[8 * lane + j];
      s += loc[j];
    }
    uint32_t incl = s;
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    const uint32_t excl = incl - s;
    const bool mine = excl < rem && rem <= incl;
    const unsigned who = __ballot_sync(0xffffffffu, mine);
    int digit = 0;
    uint32_t new_rem = 0;
    if (mine) {
      uint32_t acc = excl;
      int j = 0;
      while (acc + loc[j] < rem) acc += loc[j++];
      digit = 8 * lane + j;
      new_rem = rem - acc;
    }
    const int src = __ffs(who) - 1;
    digit = __shfl_sync(0xffffffffu, digit, src);
    rem = __shfl_sync(0xffffffffu, new_rem, src);
    if (in_hi) {
      pref_hi |= (uint64_t)digit << shift;
      mask_hi |= (uint64_t)255 << shift;
    } else {
      pref_lo |= (uint32_t)digit << shift;
      mask_lo |= 255u << shift;
    }
    __syncwarp();
  }
  rem_out = rem;
  return Key{pref_hi, pref_lo};
}

// keeps the entries with key <= t, in order
__device__ int compact(WarpBuf& b, int cnt, const Key& t) {
  const int lane = threadIdx.x & 31;
  int out = 0;
  for (int base = 0; base < cnt; base += 32) {
    const int i = base + lane;
    double d2 = 0;
    int32_t mi = 0, w = 0, u = 0;
    bool keep = false;
    if (i < cnt) {
      d2 = b.d2[i]; mi = b.mi[i]; w = b.w[i]; u = b.u[i];
      keep = key_le((uint64_t)__double_as_longlong(d2), (uint32_t)mi, t);
    }
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    __syncwarp();
    if (keep) {
      const int p = out + __popc(m & lanemask_lt());
      b.d2[p] = d2; b.mi[p] = mi; b.w[p] = w; b.u[p] = u;
    }
    out += __popc(m);
    __syncwarp();
  }
  return out;
}

__device__ __forceinline__ double dist2(const double* q, const double* p) {
  const double dx = p[0] - q[0], dy = p[1] - q[1], dz = p[2] - q[2];
  return dx * dx + dy * dy + dz * dz;
}

// --- Open3D's FastEigen3x3 (Geometric Tools' robust symmetric 3x3 solver), restated [EXT] ---
struct V3 {
  double x, y, z;
};
__device__ __forceinline__ V3 cross(V3 a, V3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
__device__ __forceinline__ double dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

__device__ V3 eigvec0(const double A[6], double e) {  // A: a00 a01 a02 a11 a12 a22
  const V3 r0 = {A[0] - e, A[1], A[2]}, r1 = {A[1], A[3] - e, A[4]}, r2 = {A[2], A[4], A[5] - e};
  const V3 c01 = cross(r0, r1), c02 = cross(r0, r2), c12 = cross(r1, r2);
  const double d0 = dot(c01, c01), d1 = dot(c02, c02), d2 = dot(c12, c12);
  double dmax = d0;
  int imax = 0;
  if (d1 > dmax) { dmax = d1; imax = 1; }
  if (d2 > dmax) imax = 2;
  if (imax == 0) { const double s = sqrt(d0); return {c01.x / s, c01.y / s, c01.z / s}; }
  if (imax == 1) { const double s = sqrt(d1); return {c02.x / s, c02.y / s, c02.z / s}; }
  const double s = sqrt(d2);
  return {c12.x / s, c12.y / s, c12.z / s};
}

__device__ V3 eigvec1(const double A[6], V3 e0, double e1) {
  V3 U;
  if (fabs(e0.x) > fabs(e0.y)) {
    const double il = 1 / sqrt(e0.x * e0.x + e0.z * e0.z);
    U = {-e0.z * il, 0, e0.x * il};
  } else {
    const double il = 1 / sqrt(e0.y * e0.y + e0.z * e0.z);
    U = {0, e0.z * il, -e0.y * il};
  }
  const V3 V = cross(e0, U);
  const V3 AU = {A[0] * U.x + A[1] * U.y + A[2] * U.z, A[1] * U.x + A[3] * U.y + A[4] * U.z, A[2] * U.x + A[4] * U.y + A[5] * U.z};
  const V3 AV = {A[0] * V.x + A[1] * V.y + A[2] * V.z, A[1] * V.x + A[3] * V.y + A[4] * V.z, A[2] * V.x + A[4] * V.y + A[5] * V.z};
  double m00 = U.x * AU.x + U.y * AU.y + U.z * AU.z - e1;
  double m01 = U.x * AV.x + U.y * AV.y + U.z * AV.z;
  double m11 = V.x * AV.x + V.y * AV.y + V.z * AV.z - e1;
  const double a00 = fabs(m00), a01 = fabs(m01), a11 = fabs(m11);
  if (a00 >= a11) {
    if (fmax(a00, a01) > 0) {
      if (a00 >= a01) { m01 /= m00; m00 = 1 / sqrt(1 + m01 * m01); m01 *= m00; }
      else { m00 /= m01; m01 = 1 / sqrt(1 + m00 * m00); m00 *= m01; }
      return {m01 * U.x - m00 * V.x, m01 * U.y - m00 * V.y, m01 * U.z - m00 * V.z};
    }
    return U;
  }
  if (fmax(a11, a01) > 0) {
    if (a11 >= a01) { m01 /= m11; m11 = 1 / sqrt(1 + m01 * m01); m01 *= m11; }
    else { m11 /= m01; m01 = 1 / sqrt(1 + m11 * m11); m11 *= m01; }
    return {m11 * U.x - m01 * V.x, m11 * U.y - m01 * V.y, m11 * U.z - m01 * V.z};
  }
  return U;
}

__device__ V3 fast_eigen3x3(const double C[6]) {
  double mx = C[0];
  for (int i = 1; i < 6; ++i) mx = fmax(mx, C[i]);
  if (mx == 0) return {0, 0, 0};
  double A[6];
  for (int i = 0; i < 6; ++i) A[i] = C[i] / mx;
  const double norm = A[1] * A[1] + A[2] * A[2] + A[4] * A[4];
  if (norm > 0) {
    const double q = (A[0] + A[3] + A[5]) / 3;
    const double b00 = A[0] - q, b11 = A[3] - q, b22 = A[5] - q;
    const double p = sqrt((b00 * b00 + b11 * b11 + b22 * b22 + norm * 2) / 6);
    const double c00 = b11 * b22 - A[4] * A[4];
    const double c01 = A[1] * b22 - A[4] * A[2];
    const double c02 = A[1] * A[4] - b11 * A[2];
    const double det = (b00 * c00 - A[1] * c01 + A[2] * c02) / (p * p * p);
    const double half_det = fmin(fmax(det * 0.5, -1.0), 1.0);
    const double angle = acos(half_det) / 3.0;
    const double two_thirds_pi = 2.09439510239319549;
    const double beta2 = cos(angle) * 2;
    const double beta0 = cos(angle + two_thirds_pi) * 2;
    const double beta1 = -(beta0 + beta2);
    const double ev0 = q + p * beta0, ev1 = q + p * beta1, ev2 = q + p * beta2;
    if (half_det >= 0) {
      const V3 v2 = eigvec0(A, ev2);
      if (ev2 < ev0 && ev2 < ev1) return v2;
      const V3 v1 = eigvec1(A, v2, ev1);
      if (ev1 < ev0 && ev1 < ev2) return v1;
      return cross(v1, v2);
    }
    const V3 v0 = eigvec0(A, ev0);
    if (ev0 < ev1 && ev0 < ev2) return v0;
    const V3 v1 = eigvec1(A, v0, ev1);
    if (ev1 < ev0 && ev1 < ev2) return v1;
    return cross(v0, v1);
  }
  if (C[0] < C[3] && C[0] < C[5]) return {1, 0, 0};
  if (C[3] < C[0] && C[3] < C[5]) return {0, 1, 0};
  return {0, 0, 1};
}

struct QueryArgs {
  const double* upts;
  const uint64_t* ukey;
  const int32_t* umin;
  const int32_t* ustart;
  const int32_t* order;     // sorted position -> point index: the copies of position u are order[ustart[u], ustart[u+1])
  const int32_t* n_unique;  // device scalar: scan[n - 1]
  double* unormal;          // [U,3] the normal of each position
  int32_t* ucount;          // [U] candidates its search examined
  double* cov;              // [n,9] or null: written at each position's first copy (nrm_scatter_kernel copies it)
  int32_t* nbr;             // [n,k] or null: likewise
  unsigned long long* stats;
  GridP g;
  double cell;
  double center[3];
  int32_t orient, k, n;
};

__device__ __forceinline__ int lower_bound(const uint64_t* a, int n, uint64_t v) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < v) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// appends entry j (already known to be a candidate of this lane when ok) to the buffer
__device__ __forceinline__ void push(WarpBuf& b, int& cnt, bool ok, double d2, int32_t mi, int32_t w, int32_t j) {
  const unsigned m = __ballot_sync(0xffffffffu, ok);
  if (ok) {
    const int p = cnt + __popc(m & lanemask_lt());
    b.d2[p] = d2; b.mi[p] = mi; b.w[p] = w; b.u[p] = j;
  }
  cnt += __popc(m);
  __syncwarp();
}

__global__ void __launch_bounds__(32 * QWARPS) nrm_query_kernel(QueryArgs a) {
  __shared__ WarpBuf bufs[QWARPS];
  WarpBuf& b = bufs[threadIdx.x >> 5];
  const int lane = threadIdx.x & 31;
  const int u = blockIdx.x * QWARPS + (threadIdx.x >> 5);
  const int U = *a.n_unique;
  if (u >= U) return;
  const uint32_t kk = (uint32_t)min(a.k, a.n);
  const double q[3] = {a.upts[3 * (size_t)u], a.upts[3 * (size_t)u + 1], a.upts[3 * (size_t)u + 2]};
  int cnt = 0;
  unsigned long long examined = 0;
  const int own = a.ustart[u + 1] - a.ustart[u];
  if ((uint32_t)own >= kk) {  // its own copies are its kk nearest
    if (lane == 0) { b.d2[0] = 0; b.mi[0] = a.umin[u]; b.w[0] = own; b.u[0] = u; }
    cnt = 1;
    __syncwarp();
  } else {
    const int wlo = max(u - (int)kk, 0), whi = min(u + (int)kk + 1, U);
    for (int base = wlo; base < whi; base += 32) {
      const int j = base + lane;
      const bool ok = j < whi;
      double d2 = 0;
      int32_t mi = 0, w = 0;
      if (ok) { d2 = dist2(q, a.upts + 3 * (size_t)j); mi = a.umin[j]; w = a.ustart[j + 1] - a.ustart[j]; }
      push(b, cnt, ok, d2, mi, w, j);
    }
    examined += (unsigned long long)(whi - wlo);
    if (wlo > 0 || whi < U) {  // the window is not everything: search the grid within its k-th distance
      uint32_t rem;
      Key t = weighted_select(b, cnt, kk, rem);
      cnt = compact(b, cnt, t);
      // the floor: a d2 below 2^-1022 carries an absolute rounding error (dx * dx may underflow to 0), so the true
      // distance is only known to lie below 2^-511
      const double R = fmax(sqrt(__longlong_as_double((long long)t.hi)) * (1.0 + 0x1p-40), 0x1p-510);
      int level = 0;
      while (level < MORTON_BITS && a.cell * (double)(1 << level) * LEVEL_DIV < R) ++level;
      uint32_t c0[3], c1[3];
      for (int ax = 0; ax < 3; ++ax) {
        c0[ax] = cell_of(q[ax] - R, a.g.lo[ax], a.g.inv_cell) >> level;
        c1[ax] = cell_of(q[ax] + R, a.g.lo[ax], a.g.inv_cell) >> level;
      }
      const int nx = c1[0] - c0[0] + 1, ny = c1[1] - c0[1] + 1, nz = c1[2] - c0[2] + 1;
      const int ncell = nx * ny * nz;
      for (int cb = 0; cb < ncell; cb += 32) {
        int s = 0, e = 0;
        const int c = cb + lane;
        if (c < ncell) {
          const uint32_t cx = c0[0] + c % nx, cy = c0[1] + (c / nx) % ny, cz = c0[2] + c / (nx * ny);
          const uint64_t k0 = morton(cx << level, cy << level, cz << level);
          s = lower_bound(a.ukey, U, k0);
          e = lower_bound(a.ukey, U, k0 + ((uint64_t)1 << (3 * level)));
        }
        const int nc = min(32, ncell - cb);
        for (int ci = 0; ci < nc; ++ci) {
          const int cs = __shfl_sync(0xffffffffu, s, ci), ce = __shfl_sync(0xffffffffu, e, ci);
          examined += (unsigned long long)(ce - cs);
          for (int base = cs; base < ce; base += 32) {
            if (cnt > CAP - 32) {
              t = weighted_select(b, cnt, kk, rem);
              cnt = compact(b, cnt, t);
            }
            const int j = base + lane;
            bool ok = j < ce && (j < wlo || j >= whi);
            double d2 = 0;
            int32_t mi = 0, w = 0;
            if (ok) {
              d2 = dist2(q, a.upts + 3 * (size_t)j);
              mi = a.umin[j];
              ok = key_le((uint64_t)__double_as_longlong(d2), (uint32_t)mi, t);
              if (ok) w = a.ustart[j + 1] - a.ustart[j];
            }
            push(b, cnt, ok, d2, mi, w, j);
          }
        }
      }
    }
  }
  uint32_t rem = (uint32_t)b.w[0];
  Key t = {0, (uint32_t)b.mi[0]};
  if (cnt > 1) t = weighted_select(b, cnt, kk, rem);
  else rem = kk;
  double s[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int i = lane; i < cnt; i += 32) {
    const uint64_t h = (uint64_t)__double_as_longlong(b.d2[i]);
    const uint32_t l = (uint32_t)b.mi[i];
    if (!key_le(h, l, t)) continue;
    const double w = (h == t.hi && l == t.lo) ? (double)rem : (double)b.w[i];
    const double* p = a.upts + 3 * (size_t)b.u[i];
    s[0] += w * p[0]; s[1] += w * p[1]; s[2] += w * p[2];
    s[3] += w * (p[0] * p[0]); s[4] += w * (p[0] * p[1]); s[5] += w * (p[0] * p[2]);
    s[6] += w * (p[1] * p[1]); s[7] += w * (p[1] * p[2]); s[8] += w * (p[2] * p[2]);
  }
  for (int o = 16; o > 0; o >>= 1)
    for (int j = 0; j < 9; ++j) s[j] += __shfl_xor_sync(0xffffffffu, s[j], o);
  const int c0 = a.ustart[u];
  if (a.nbr) {  // test output: the neighbours' smallest indices, one per copy taken, in the first copy's row
    int32_t* row = a.nbr + (size_t)a.order[c0] * a.k;
    if (lane == 0) {
      int o = 0;
      for (int i = 0; i < cnt; ++i) {
        const uint64_t h = (uint64_t)__double_as_longlong(b.d2[i]);
        const uint32_t l = (uint32_t)b.mi[i];
        if (!key_le(h, l, t)) continue;
        const int w = (h == t.hi && l == t.lo) ? (int)rem : b.w[i];
        for (int c = 0; c < w; ++c) row[o++] = b.mi[i];
      }
      for (; o < a.k; ++o) row[o] = -1;
    }
  }
  if (lane == 0 && a.stats) {
    atomicAdd(a.stats, examined);
    atomicAdd(a.stats + 1, 1ull);
  }
  double C[6];
  if (kk < 3) {
    C[0] = 1; C[1] = 0; C[2] = 0; C[3] = 1; C[4] = 0; C[5] = 1;
  } else {
    for (int j = 0; j < 9; ++j) s[j] /= (double)kk;
    C[0] = s[3] - s[0] * s[0];
    C[3] = s[6] - s[1] * s[1];
    C[5] = s[8] - s[2] * s[2];
    C[1] = s[4] - s[0] * s[1];
    C[2] = s[5] - s[0] * s[2];
    C[4] = s[7] - s[1] * s[2];
  }
  V3 nrm = fast_eigen3x3(C);
  if (sqrt(dot(nrm, nrm)) == 0.0) nrm = {0, 0, 1};
  if (a.orient) {
    const double r0 = q[0] - a.center[0], r1 = q[1] - a.center[1], r2 = q[2] - a.center[2];
    if ((r0 * nrm.x + r1 * nrm.y) + r2 * nrm.z > 0) nrm = {-nrm.x, -nrm.y, -nrm.z};
  }
  if (lane == 0) {
    a.unormal[3 * (size_t)u] = nrm.x;
    a.unormal[3 * (size_t)u + 1] = nrm.y;
    a.unormal[3 * (size_t)u + 2] = nrm.z;
    a.ucount[u] = (int32_t)min(examined, (unsigned long long)INT32_MAX);
    if (a.cov) {
      const double full[9] = {C[0], C[1], C[2], C[1], C[3], C[4], C[2], C[4], C[5]};
      for (int j = 0; j < 9; ++j) a.cov[9 * (size_t)a.order[c0] + j] = full[j];
    }
  }
}

// one thread per point (in sorted order): the result of its position; the test outputs are copied from the first copy
__global__ void nrm_scatter_kernel(int n, int k, const int32_t* __restrict__ order, const int32_t* __restrict__ scan,
                                   const int32_t* __restrict__ ustart, const double* __restrict__ unormal,
                                   const int32_t* __restrict__ ucount, double* __restrict__ normals, int32_t* __restrict__ examined,
                                   double* __restrict__ cov, int32_t* __restrict__ nbr) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const size_t i = (size_t)order[s];
  const int u = scan[s] - 1;
  for (int a = 0; a < 3; ++a) normals[3 * i + a] = unormal[3 * (size_t)u + a];
  if (examined) examined[i] = ucount[u];
  const int first = ustart[u];
  if (s == first) return;
  const size_t f = (size_t)order[first];
  if (cov)
    for (int a = 0; a < 9; ++a) cov[9 * i + a] = cov[9 * f + a];
  if (nbr)
    for (int a = 0; a < k; ++a) nbr[i * k + a] = nbr[f * k + a];
}

__global__ void backproject_kernel(const float* __restrict__ depth, int w, int h, float fx, float fy, float cx, float cy, DnrDnPose P,
                                   float* __restrict__ cam, double* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= w * h) return;
  const float u = (float)(i % w) + 0.5f, v = (float)(i / w) + 0.5f;
  const float d = depth[i];
  const float x = __fdiv_rn(__fmul_rn(__fsub_rn(u, cx), d), fx);
  const float y = __fdiv_rn(__fmul_rn(__fsub_rn(v, cy), d), fy);
  if (cam) {
    cam[3 * (size_t)i] = x;
    cam[3 * (size_t)i + 1] = y;
    cam[3 * (size_t)i + 2] = d;
  }
  const double p[3] = {x, y, d};
  for (int j = 0; j < 3; ++j)
    out[3 * (size_t)i + j] = ((p[0] * P.rinv[j] + p[1] * P.rinv[3 + j]) + p[2] * P.rinv[6 + j]) + P.t[j];
}

__global__ void consistency_kernel(const double* __restrict__ normals, const uint8_t* __restrict__ mono, int64_t n, DnrDnPose P,
                                   int mode, double threshold, double* __restrict__ degrees, uint8_t* __restrict__ mask,
                                   uint8_t* __restrict__ normals_u8) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double nd[3], m[3];
  for (int a = 0; a < 3; ++a) {
    nd[a] = normals[3 * i + a];
    const double e = (nd[a] + 1) / 2;
    normals_u8[3 * i + a] = (uint8_t)(int)(e * 255);
    const double c = (double)mono[3 * i + a] / 255.0;
    m[a] = mode == DNR_DN_DEPTH_TO_NORMAL ? (c - 0.5) * 2 : 2 * c - 1;
  }
  if (mode == DNR_DN_DSINE) { m[1] = -m[1]; m[2] = -m[2]; }
  double r[3];  // R @ m with R = transpose(inv(c2w)[:3, :3]) (row-major in P.rinv)
  for (int j = 0; j < 3; ++j) r[j] = (P.rinv[3 * j] * m[0] + P.rinv[3 * j + 1] * m[1]) + P.rinv[3 * j + 2] * m[2];
  const double rn = sqrt((r[0] * r[0] + r[1] * r[1]) + r[2] * r[2]);
  for (int j = 0; j < 3; ++j) r[j] = r[j] / rn;
  if (mode == DNR_DN_DEPTH_TO_NORMAL) {  // the angle between the encoded vectors
    for (int j = 0; j < 3; ++j) {
      nd[j] = (nd[j] + 1) / 2;
      r[j] = r[j] * 0.5 + 0.5;
    }
  }
  const double a1 = sqrt((nd[0] * nd[0] + nd[1] * nd[1]) + nd[2] * nd[2]);
  const double a2 = sqrt((r[0] * r[0] + r[1] * r[1]) + r[2] * r[2]);
  const double dp = (nd[0] / a1 * (r[0] / a2) + nd[1] / a1 * (r[1] / a2)) + nd[2] / a1 * (r[2] / a2);
  const double deg = acos(fmin(fmax(dp, -1.0), 1.0)) * (180.0 / 3.14159265358979323846);
  degrees[i] = deg;
  mask[i] = deg > threshold ? 255 : 0;
}

}  // namespace

extern "C" int dnr_dn_backproject(const float* depth, int32_t width, int32_t height, const float* intrinsics_host,
                                  const DnrDnPose* pose, float* cam_points, double* points, void* stream) {
  if (!depth || !intrinsics_host || !pose || !points) return DNR_E_NULL;
  if (width <= 0 || height <= 0 || (int64_t)width * height > INT32_MAX) return DNR_E_SIZE;
  const int n = width * height;
  backproject_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(depth, width, height, intrinsics_host[0], intrinsics_host[1],
                                                                         intrinsics_host[2], intrinsics_host[3], *pose, cam_points,
                                                                         points);
  DNR_CHECK_LAUNCH();
  return 0;
}

extern "C" int64_t dnr_dn_normals_workspace_bytes(int64_t n_points) {
  if (n_points <= 0 || n_points > INT32_MAX - 1) return DNR_E_SIZE;
  return (int64_t)NrmLayout(nullptr, n_points).carve.total();
}

extern "C" int dnr_dn_normals(const double* points, int64_t n_points, const DnrDnSearch* search, void* ws, int64_t ws_bytes,
                              double* normals, int32_t* examined, double* cov, int32_t* neighbours, unsigned long long* stats,
                              void* stream) {
  if (!points || !search || !ws || !normals) return DNR_E_NULL;
  if (n_points <= 0 || n_points > INT32_MAX - 1) return DNR_E_SIZE;
  if (search->k <= 0 || search->k > DNR_DN_MAX_K) return DNR_E_OPTION;
  if (!(search->cell > 0.0) || !(search->cell < INFINITY)) return DNR_E_SIZE;
  const NrmLayout L(ws, n_points);
  if (const int e = L.carve.check(ws_bytes)) return e;
  const int n = (int)n_points;
  cudaStream_t s = (cudaStream_t)stream;
  uint64_t *ka = L.keys_a, *kb = L.keys_b;
  int32_t *va = L.vals_a, *vb = L.vals_b, *scan = L.scan;
  GridP g;
  for (int a = 0; a < 3; ++a) g.lo[a] = search->lo[a];
  g.inv_cell = 1.0 / search->cell;
  const int blocks = (n + 255) / 256;
  for (int pass = 0; pass < 4; ++pass) {  // stable LSD: z, y, x bits, then the Morton key
    nrm_keys_kernel<<<blocks, 256, 0, s>>>(points, n, pass, g, va, ka, va);
    DNR_CHECK_LAUNCH();
    size_t temp = L.cub_bytes;
    DNR_CUDA(cub::DeviceRadixSort::SortPairs(L.cub_temp, temp, ka, kb, va, vb, n, 0, pass < 3 ? 64 : 3 * MORTON_BITS, s));
    DNR_CUDA(cudaMemcpyAsync(va, vb, 4 * (size_t)n, cudaMemcpyDeviceToDevice, s));
  }
  nrm_heads_kernel<<<blocks, 256, 0, s>>>(points, n, va, vb);
  DNR_CHECK_LAUNCH();
  size_t temp = L.cub_bytes;
  DNR_CUDA(cub::DeviceScan::InclusiveSum(L.cub_temp, temp, vb, scan, n, s));
  nrm_unique_kernel<<<blocks, 256, 0, s>>>(points, n, va, kb, scan, L.ustart, L.upts, L.ukey, L.umin);
  DNR_CHECK_LAUNCH();
  QueryArgs a;
  a.upts = L.upts; a.ukey = L.ukey; a.umin = L.umin; a.ustart = L.ustart; a.order = va; a.n_unique = scan + (n - 1);
  a.unormal = L.unormal; a.ucount = L.ucount; a.cov = cov; a.nbr = neighbours; a.stats = stats; a.g = g; a.cell = search->cell;
  for (int j = 0; j < 3; ++j) a.center[j] = search->center[j];
  a.orient = search->orient; a.k = search->k; a.n = n;
  nrm_query_kernel<<<(n + QWARPS - 1) / QWARPS, 32 * QWARPS, 0, s>>>(a);
  DNR_CHECK_LAUNCH();
  nrm_scatter_kernel<<<blocks, 256, 0, s>>>(n, search->k, va, scan, L.ustart, a.unormal, a.ucount, normals, examined, cov, neighbours);
  DNR_CHECK_LAUNCH();
  return 0;
}

extern "C" int dnr_dn_consistency(const double* normals, const uint8_t* mono, int64_t n, const DnrDnPose* rotation, int32_t mode,
                                  double threshold, double* degrees, uint8_t* mask, uint8_t* normals_u8, void* stream) {
  if (!normals || !mono || !rotation || !degrees || !mask || !normals_u8) return DNR_E_NULL;
  if (n <= 0) return DNR_E_SIZE;
  if (mode < DNR_DN_OMNIDATA || mode > DNR_DN_DEPTH_TO_NORMAL) return DNR_E_OPTION;
  consistency_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(normals, mono, n, *rotation, mode, threshold,
                                                                                     degrees, mask, normals_u8);
  DNR_CHECK_LAUNCH();
  return 0;
}
