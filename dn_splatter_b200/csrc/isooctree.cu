// AGS-Mesh's mesh extractor (the reference's dn_splatter/scripts/isooctree_dn.py) on the device (Python surface:
// dn_splatter_b200.isooctree; fp64 restatement: oracle/isooctree_ref.py, whose quirk list Q1..Q12 the comments cite).
//
// dnr_iso_samples  Frame.get_samples of every frame: one thread per strided pixel flags the survivors (4 m cut, validity
//                  mask on the strided image with rel_delta * stride, normal sign test), cub compacts their indices in
//                  (frame, row, column) order, a second kernel writes their points.
// dnr_iso_eval     isoFunc: one thread per point walks the frames in order for each pass, keeping the best-frame normal,
//                  value, weight and the valid / back flags in registers; nothing per frame goes to memory.
// dnr_iso_octree   Morton keys of the hint samples at max_depth, sorted with cub; per level, the 8 children of every
//                  split node count their samples by two binary searches in the sorted keys, and cub selects the
//                  children that split (next level) and those that are leaves, in code order.
// dnr_iso_corners  the 8 lattice keys of every leaf, sorted and made unique with cub, and each leaf's 8 corner indices.
// dnr_iso_fill     per level, coarse to fine, every leaf writes its closed cube of samples: a finer leaf overwrites a
//                  coarser one on shared faces, and equal-size neighbours write equal values there (lerp endpoints are
//                  exact), so the grid does not depend on scheduling.
//
// Precision: every operation that feeds a decision (pixel truncation, validity mask, the 4 m and MIN_DEPTH cuts, the
// normal sign test, tv > -1, the strict w > weight of the normal pass, the back-mask band) or a value is fp64, in the
// oracle's order, and the file is compiled with -fmad=false, so the kernels equal the fp64 oracle bit for bit.  An fp32
// evaluation would flip pixel truncations and the strict weight comparison near their thresholds (the golden folder puts
// query points exactly on pixel edges), and each flip changes a value by up to the full TSDF range.
#include <cub/cub.cuh>
#include <math.h>
#include <thrust/iterator/counting_iterator.h>

#include "common.cuh"

namespace {

constexpr double EPS = 1e-6;
constexpr double MIN_DEPTH = 1e-3;
constexpr double BACK_MASK_COEFF = 0.25;
constexpr int LEVEL_SHIFT = 58;
constexpr int64_t CODE_MASK = (int64_t(1) << LEVEL_SHIFT) - 1;


struct Pose {  // one row of DnrIsoFrames::poses
  const double* p;
  __device__ __forceinline__ double w2c(int r, int c) const { return p[4 * r + c]; }
  __device__ __forceinline__ double rot(int r, int c) const { return p[12 + 3 * r + c]; }
  __device__ __forceinline__ double pos(int a) const { return p[21 + a]; }
  __device__ __forceinline__ double nrot(int r, int c) const { return p[24 + 3 * r + c]; }
};

__device__ __forceinline__ double dot3(const double* a, const double* b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }

__device__ __forceinline__ double depth_at(const DnrIsoFrames& fr, const float* d, int y, int x) {
  return (double)d[(int64_t)y * fr.width + x] * fr.depth_scale;
}

// compute_depth_validity_mask at (y, x) of an image given by depth(y, x), h x w
template <class D>
__device__ bool valid_depth(const D& depth, int y, int x, int h, int w, double rel) {
  const double d0 = depth(y, x);
  const int ny[4] = {y, y, y - 1, y + 1}, nx[4] = {x - 1, x + 1, x, x};
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    if (nx[q] < 0 || nx[q] >= w || ny[q] < 0 || ny[q] >= h) continue;
    const double d1 = depth(ny[q], nx[q]);
    if (!(fabs(d1 - d0) < fmin(d1, d0) * rel)) return false;  // fmin: both finite here
  }
  return true;
}

__device__ __forceinline__ void load_normal(const DnrIsoFrames& fr, const float* nrm, int64_t pix, double n[3]) {
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double v = (double)nrm[3 * pix + a];
    n[a] = fr.cam_normals ? v / 255.0 * 2.0 - 1.0 : v;  // Q10
  }
}

// ---- hint cloud ---------------------------------------------------------------------------------------------------
struct Strided {  // the stride-subsampled depth with the 4 m cut (Q4)
  const DnrIsoFrames* fr;
  const float* d;
  int s;
  __device__ double operator()(int y, int x) const {
    const double v = depth_at(*fr, d, y * s, x * s);
    return v <= 4.0 ? v : 0.0;
  }
};

__device__ void sample_at(const DnrIsoFrames& fr, int64_t i, int s, int ws_, int hs, bool* keep, double pt[3], double nw[3]) {
  const int64_t per = (int64_t)ws_ * hs;
  const int f = (int)(i / per);
  const int r = (int)(i % per), ys = r / ws_, xs = r % ws_;
  const float* d = fr.depth + (int64_t)f * fr.height * fr.width;
  const Pose P{fr.poses + (int64_t)f * DNR_ISO_POSE};
  const double px[3] = {(double)(xs * s) + 0.5, (double)(ys * s) + 0.5, 1.0};
  double h[3], ray[3];
  for (int a = 0; a < 3; ++a) h[a] = dot3(fr.inv_K + 3 * a, px);
  for (int a = 0; a < 3; ++a) ray[a] = (h[0] * P.rot(a, 0) + h[1] * P.rot(a, 1)) + h[2] * P.rot(a, 2);  // Q5
  const Strided depth{&fr, d, s};
  const double dep = depth(ys, xs);
  const bool ok = valid_depth(depth, ys, xs, hs, ws_, fr.rel_delta * s);
  double n[3];
  load_normal(fr, fr.normals + (int64_t)f * fr.height * fr.width * 3, (int64_t)(ys * s) * fr.width + xs * s, n);
  if (fr.cam_normals) {  // Q10
    double m[3];
    for (int a = 0; a < 3; ++a) m[a] = (n[0] * P.nrot(a, 0) + n[1] * P.nrot(a, 1)) + n[2] * P.nrot(a, 2);
    const double len = sqrt(dot3(m, m));
    for (int a = 0; a < 3; ++a) n[a] = m[a] / len;
  }
  *keep = (dot3(n, ray) < 0.0) && ok;
  for (int a = 0; a < 3; ++a) {
    pt[a] = P.pos(a) + ray[a] * dep;
    nw[a] = n[a];
  }
}

__global__ void iso_sample_flags_kernel(DnrIsoFrames fr, int s, int ws_, int hs, int64_t total, uint8_t* __restrict__ flags) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  bool keep;
  double pt[3], n[3];
  sample_at(fr, i, s, ws_, hs, &keep, pt, n);
  flags[i] = keep;
}

__global__ void iso_sample_write_kernel(DnrIsoFrames fr, int s, int ws_, int hs, const int64_t* __restrict__ idx, int64_t count,
                                        double* __restrict__ points, double* __restrict__ normals) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= count) return;
  bool keep;
  double pt[3], n[3];
  sample_at(fr, idx[q], s, ws_, hs, &keep, pt, n);
  for (int a = 0; a < 3; ++a) points[3 * q + a] = pt[a];
  if (normals)
    for (int a = 0; a < 3; ++a) normals[3 * q + a] = n[a];
}

// ---- isoFunc ------------------------------------------------------------------------------------------------------
struct Full {
  const DnrIsoFrames* fr;
  const float* d;
  __device__ double operator()(int y, int x) const { return depth_at(*fr, d, y, x); }
};

// Frame.get_depth_values at p: false when the frame does not see p; else pd (interpolated depth), zc (camera z) and n.
__device__ bool depth_value(const DnrIsoFrames& fr, int f, const double p[3], bool with_normals, double* pd, double* zc,
                            double n[3]) {
  const Pose P{fr.poses + (int64_t)f * DNR_ISO_POSE};
  double c[3];
  for (int r = 0; r < 3; ++r) c[r] = ((p[0] * P.w2c(r, 0) + p[1] * P.w2c(r, 1)) + p[2] * P.w2c(r, 2)) + P.w2c(r, 3);
  *zc = c[2];
  if (!(c[2] > EPS)) return false;
  double h[3];
  for (int r = 0; r < 3; ++r) h[r] = dot3(fr.K + 3 * r, c);
  const double x = h[0] / h[2], y = h[1] / h[2];
  if (!(x > -1.0 && y > -1.0 && x < (double)fr.width && y < (double)fr.height)) return false;  // Q1: (int) truncates
  const int ix = (int)x, iy = (int)y;
  const double tx = x - ix, ty = y - iy;
  const int ix1 = min(ix + 1, fr.width - 1), iy1 = min(iy + 1, fr.height - 1);  // Q3
  const float* d = fr.depth + (int64_t)f * fr.height * fr.width;
  const Full depth{&fr, d};
  const double dd = depth(iy, ix) * (1 - tx) * (1 - ty) + depth(iy, ix1) * tx * (1 - ty) + depth(iy1, ix) * (1 - tx) * ty +
                    depth(iy1, ix1) * tx * ty;
  *pd = dd;
  if (!(valid_depth(depth, iy, ix, fr.height, fr.width, fr.rel_delta) && dd > MIN_DEPTH)) return false;  // Q2, Q4
  if (with_normals) {
    load_normal(fr, fr.normals + (int64_t)f * fr.height * fr.width * 3, (int64_t)iy * fr.width + ix, n);
    double ray[3];
    for (int a = 0; a < 3; ++a) ray[a] = p[a] - P.pos(a);
    if (!(dot3(n, ray) < 0.0)) return false;  // Q6
  }
  return true;
}

__global__ void __launch_bounds__(128) iso_eval_kernel(DnrIsoFrames fr, DnrIsoParams prm, const double* __restrict__ points,
                                                       int64_t n, float* __restrict__ values) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double p[3] = {points[3 * i], points[3 * i + 1], points[3 * i + 2]};
  const bool use_normals = prm.use_normals != 0;
  double mwn[3] = {0.0, 0.0, 0.0};
  bool valid_mask = false, back = false;
  double value = 0.0, weight = 0.0;
  for (int pass = 0; pass < 2; ++pass) {
    if (!((prm.passes >> pass) & 1)) continue;
    const bool normal_pass = pass == 0;
    valid_mask = false;
    back = false;
    value = 0.0;
    weight = 0.0;
    for (int f = 0; f < fr.n_frames; ++f) {
      double pd, zc, nrm[3] = {0.0, 0.0, 0.0};
      if (!depth_value(fr, f, p, use_normals, &pd, &zc, nrm)) continue;
      double max_tsdf = prm.max_tsdf_rel * pd;
      max_tsdf = fmin(max_tsdf, prm.max_tsdf_abs);
      double tv = (pd - zc) / max_tsdf;
      if (tv * prm.max_tsdf_rel > -BACK_MASK_COEFF && tv < 0.0) back = true;  // Q8
      if (!(tv > -1.0)) continue;
      tv = fmin(tv, 1.0);
      const Pose P{fr.poses + (int64_t)f * DNR_ISO_POSE};
      double ray[3];
      for (int a = 0; a < 3; ++a) ray[a] = p[a] - P.pos(a);
      const double len = fmax(EPS, sqrt(dot3(ray, ray)));
      for (int a = 0; a < 3; ++a) ray[a] = ray[a] / len;
      const double dir_weight = (normal_pass || !use_normals) ? 1.0 : -dot3(nrm, ray);
      tv = tv * dir_weight;
      double w = dir_weight / fmax(EPS, pd);
      if (normal_pass) {
        w = w * fmax(0.0, fmin(tv + 0.5, 1.0));
        if (!(w > weight)) continue;  // Q7: strict, the earlier frame wins a tie
        weight = w;
        for (int a = 0; a < 3; ++a) mwn[a] = nrm[a];
        value = tv;
      } else {
        if (use_normals && dot3(mwn, mwn) > 0.0) {
          const double mnw = fmax(dot3(mwn, nrm) - prm.min_dot, 0.0) / (1 - prm.min_dot);
          const double neg = 1 - fmax(0.0, fmin(tv + 0.5, 1.0));
          w *= mnw * neg + (1 - neg);
        }
        value += tv * w;
        weight += w;
      }
      valid_mask = true;
    }
    if (normal_pass) {
      valid_mask = valid_mask && dot3(mwn, mwn) > 0.0;
      if (valid_mask) {
        const double len = sqrt(dot3(mwn, mwn));
        for (int a = 0; a < 3; ++a) mwn[a] = mwn[a] / len;
      }
    }
  }
  valid_mask = valid_mask && weight > 0.0;
  double v = valid_mask ? value / weight : 1.0;  // Q9, Q12
  if (!valid_mask && back) v = -1.0;             // Q8
  values[i] = (float)v;
}

// ---- octree -------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int64_t spread3(int64_t v, int bits) {
  int64_t r = 0;
  for (int b = 0; b < bits; ++b) r |= ((v >> b) & 1) << (3 * b);
  return r;
}
__device__ __forceinline__ int64_t compact3(int64_t v, int bits) {
  int64_t r = 0;
  for (int b = 0; b < bits; ++b) r |= ((v >> (3 * b)) & 1) << b;
  return r;
}

__global__ void iso_keys_kernel(DnrIsoGrid g, const double* __restrict__ pts, int64_t n, int64_t* __restrict__ keys) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t R = int64_t(1) << g.max_depth;
  int64_t key = 0;
  for (int a = 0; a < 3; ++a) {
    const double c = floor((pts[3 * i + a] - g.origin[a]) / g.cell);
    const int64_t ci = c < 0.0 ? 0 : (c > (double)(R - 1) ? R - 1 : (int64_t)c);  // NaN -> R - 1
    key |= spread3(ci, g.max_depth) << (2 - a);
  }
  keys[i] = key;
}

__device__ __forceinline__ int64_t lower_bound(const int64_t* a, int64_t n, int64_t key) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (a[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__global__ void iso_children_kernel(DnrIsoGrid g, int level, const int64_t* __restrict__ parents, int64_t n_parents,
                                    const int64_t* __restrict__ keys, int64_t n_keys, int64_t* __restrict__ children,
                                    uint8_t* __restrict__ split, uint8_t* __restrict__ leaf) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 8 * n_parents) return;
  const int64_t code = (parents[t >> 3] & CODE_MASK) * 8 + (t & 7);
  const int shift = 3 * (g.max_depth - level);
  const int64_t count = lower_bound(keys, n_keys, (code + 1) << shift) - lower_bound(keys, n_keys, code << shift);
  const bool s = count >= g.threshold && level < g.max_depth;
  children[t] = ((int64_t)level << LEVEL_SHIFT) | code;
  split[t] = s;
  leaf[t] = !s;
}

struct OctLayout {
  DnrCarver carve;
  int64_t bound;  // split nodes of one level, at most
  int64_t *leaves, *keys, *sorted, *lists, *children, *num;
  uint8_t *split, *leaf;
  void* cub_temp;
  size_t cub_bytes;
  OctLayout(const void* base, const DnrIsoGrid* g, int64_t n) : carve(base) {
    const int64_t by_count = n / g->threshold;
    int64_t b = 1, pw = 1;
    for (int l = 1; l < g->max_depth; ++l) {
      pw = pw < (int64_t(1) << 40) ? pw * 8 : pw;
      b = std::max(b, std::min(pw, by_count));
    }
    bound = std::max<int64_t>(b, 1);
    // first, so that their place does not depend on n: dnr_iso_corners reads them from the octree's workspace
    leaves = carve.take<int64_t>((int64_t)g->max_depth * 8 * bound + 1);  // leaves of all levels
    keys = carve.take<int64_t>(std::max<int64_t>(n, 1));
    sorted = carve.take<int64_t>(std::max<int64_t>(n, 1));
    lists = carve.take<int64_t>(2 * bound);  // this level's split nodes and the next's
    children = carve.take<int64_t>(8 * bound);
    split = carve.take<uint8_t>(8 * bound);
    leaf = carve.take<uint8_t>(8 * bound);
    num = carve.take<int64_t>(2);
    size_t t_sort = 0, t_sel = 0;
    const cudaError_t e1 = cub::DeviceRadixSort::SortKeys(nullptr, t_sort, (const int64_t*)nullptr, (int64_t*)nullptr,
                                                          (int64_t)std::max<int64_t>(n, 1));
    const cudaError_t e2 = cub::DeviceSelect::Flagged(nullptr, t_sel, (const int64_t*)nullptr, (const uint8_t*)nullptr,
                                                      (int64_t*)nullptr, (int64_t*)nullptr, (int64_t)(8 * bound));
    cub_bytes = std::max(t_sort, t_sel);
    cub_temp = carve.cub_scratch(e1 != cudaSuccess ? e1 : e2, cub_bytes);
  }
};

int check_grid(const DnrIsoGrid* g) {
  if (!g) return DNR_E_NULL;
  if (g->max_depth < 0 || g->max_depth > DNR_ISO_MAX_DEPTH || g->threshold < 1 || !(g->cell > 0.0)) return DNR_E_SIZE;
  return 0;
}

int check_frames(const DnrIsoFrames* fr) {
  if (!fr) return DNR_E_NULL;
  if (!fr->depth || !fr->normals || !fr->poses) return DNR_E_NULL;
  if (fr->n_frames <= 0 || fr->width <= 0 || fr->height <= 0) return DNR_E_SIZE;
  return 0;
}

constexpr int THREADS = 256;
unsigned blocks_for(int64_t n, int t = THREADS) { return (unsigned)((n + t - 1) / t); }

struct SampleLayout {
  DnrCarver carve;
  uint8_t* flags;
  int64_t *idx, *num;
  void* cub_temp;
  size_t cub_bytes = 0;
  SampleLayout(void* base, int64_t total) : carve(base) {
    flags = carve.take<uint8_t>(total);
    idx = carve.take<int64_t>(total);
    num = carve.take<int64_t>(1);
    const cudaError_t e = cub::DeviceSelect::Flagged(nullptr, cub_bytes, thrust::counting_iterator<int64_t>(0), (const uint8_t*)nullptr,
                                                     (int64_t*)nullptr, (int64_t*)nullptr, total);
    cub_temp = carve.cub_scratch(e, cub_bytes);
  }
};

int64_t sample_total(const DnrIsoFrames* fr, int stride) {
  return (int64_t)fr->n_frames * ((fr->height + stride - 1) / stride) * ((fr->width + stride - 1) / stride);
}

struct CornerLayout {
  DnrCarver carve;
  int64_t *keys8, *sorted, *num;
  void* cub_temp;
  size_t cub_bytes;
  CornerLayout(void* base, int64_t n_leaves) : carve(base) {
    const int64_t m = std::max<int64_t>(8 * n_leaves, 1);
    keys8 = carve.take<int64_t>(m);
    sorted = carve.take<int64_t>(m);
    num = carve.take<int64_t>(1);
    size_t t_sort = 0, t_uni = 0;
    const cudaError_t e1 = cub::DeviceRadixSort::SortKeys(nullptr, t_sort, (const int64_t*)nullptr, (int64_t*)nullptr, m);
    const cudaError_t e2 = cub::DeviceSelect::Unique(nullptr, t_uni, (const int64_t*)nullptr, (int64_t*)nullptr, (int64_t*)nullptr, m);
    cub_bytes = std::max(t_sort, t_uni);
    cub_temp = carve.cub_scratch(e1 != cudaSuccess ? e1 : e2, cub_bytes);
  }
};

__device__ __forceinline__ void leaf_box(int64_t leaf, int D, int64_t* lo, int64_t* size) {
  const int level = (int)(leaf >> LEVEL_SHIFT);
  const int64_t code = leaf & CODE_MASK;
  *size = int64_t(1) << (D - level);
  for (int a = 0; a < 3; ++a) lo[a] = compact3(code >> (2 - a), level) * *size;
}

__global__ void iso_corner_keys_kernel(int D, const int64_t* __restrict__ leaves, int64_t n_leaves, int64_t* __restrict__ keys8) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 8 * n_leaves) return;
  int64_t lo[3], s;
  leaf_box(leaves[t >> 3], D, lo, &s);
  const int q = (int)(t & 7);
  const int64_t R1 = (int64_t(1) << D) + 1;
  keys8[t] = ((lo[0] + ((q >> 2) & 1) * s) * R1 + (lo[1] + ((q >> 1) & 1) * s)) * R1 + (lo[2] + (q & 1) * s);
}

__global__ void iso_corner_index_kernel(const int64_t* __restrict__ keys8, int64_t m, const int64_t* __restrict__ corners,
                                        const int64_t* __restrict__ n_corners, int32_t* __restrict__ leaf_corners) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= m) return;
  leaf_corners[t] = (int32_t)lower_bound(corners, *n_corners, keys8[t]);
}

__global__ void iso_corner_points_kernel(DnrIsoGrid g, const int64_t* __restrict__ corners, const int64_t* __restrict__ n_corners,
                                         double* __restrict__ points) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= *n_corners) return;
  const int64_t R1 = (int64_t(1) << g.max_depth) + 1, k = corners[t];
  const int64_t ijk[3] = {k / (R1 * R1), (k / R1) % R1, k % R1};
  for (int a = 0; a < 3; ++a) points[3 * t + a] = g.origin[a] + (double)ijk[a] * g.cell;
}

__device__ __forceinline__ float lerpf_exact(float a, float b, float t) { return (1.f - t) * a + t * b; }

__global__ void iso_fill_kernel(int D, const int64_t* __restrict__ leaves, int64_t n_leaves, int64_t side,
                                const int32_t* __restrict__ leaf_corners, const float* __restrict__ vals, float* __restrict__ field) {
  const int64_t per = side * side * side, total = n_leaves * per, R1 = (int64_t(1) << D) + 1;
  const float inv = 1.f / (float)(side - 1);  // side - 1 is a power of two: t = k * inv is exact
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t leaf = t / per, r = t % per;
    const int64_t a = r / (side * side), b = (r / side) % side, c = r % side;
    int64_t lo[3], s;
    leaf_box(leaves[leaf], D, lo, &s);
    const int32_t* ci = leaf_corners + 8 * leaf;
    float v[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) v[q] = vals[ci[q]];
    const float tx = (float)a * inv, ty = (float)b * inv, tz = (float)c * inv;
    // corner q = dx << 2 | dy << 1 | dz; the oracle's order: x, then y, then z
    const float c00 = lerpf_exact(v[0], v[4], tx), c01 = lerpf_exact(v[1], v[5], tx);
    const float c10 = lerpf_exact(v[2], v[6], tx), c11 = lerpf_exact(v[3], v[7], tx);
    const float c0 = lerpf_exact(c00, c10, ty), c1 = lerpf_exact(c01, c11, ty);
    field[((lo[0] + a) * R1 + (lo[1] + b)) * R1 + (lo[2] + c)] = lerpf_exact(c0, c1, tz);
  }
}

}  // namespace

extern "C" int64_t dnr_iso_samples_workspace_bytes(const DnrIsoFrames* fr, int32_t stride) {
  const int rc = check_frames(fr);
  if (rc) return rc;
  if (stride <= 0) return DNR_E_SIZE;
  return (int64_t)SampleLayout(nullptr, sample_total(fr, stride)).carve.total();
}

extern "C" int dnr_iso_samples(const DnrIsoFrames* fr, int32_t stride, void* ws, int64_t ws_bytes, double* points, double* normals,
                               int64_t* count_host, void* stream) {
  const int rc = check_frames(fr);
  if (rc) return rc;
  if (stride <= 0) return DNR_E_SIZE;
  if (!ws || !points || !count_host) return DNR_E_NULL;
  const int64_t total = sample_total(fr, stride);
  const SampleLayout L(ws, total);
  if (const int e = L.carve.check(ws_bytes)) return e;
  cudaStream_t s = (cudaStream_t)stream;
  uint8_t* flags = L.flags;
  int64_t *idx = L.idx, *num = L.num;
  const int ws_ = (fr->width + stride - 1) / stride, hs = (fr->height + stride - 1) / stride;
  iso_sample_flags_kernel<<<blocks_for(total), THREADS, 0, s>>>(*fr, stride, ws_, hs, total, flags);
  DNR_CHECK_LAUNCH();
  size_t t = L.cub_bytes;
  DNR_CUDA(cub::DeviceSelect::Flagged(L.cub_temp, t, thrust::counting_iterator<int64_t>(0), flags, idx, num, total, s));
  DNR_CUDA(cudaMemcpyAsync(count_host, num, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  DNR_CUDA(cudaStreamSynchronize(s));
  if (*count_host > 0) {
    iso_sample_write_kernel<<<blocks_for(*count_host), THREADS, 0, s>>>(*fr, stride, ws_, hs, idx, *count_host, points, normals);
    DNR_CHECK_LAUNCH();
  }
  return 0;
}

extern "C" int dnr_iso_eval(const DnrIsoFrames* fr, const DnrIsoParams* prm, const double* points, int64_t n, float* values,
                            void* stream) {
  const int rc = check_frames(fr);
  if (rc) return rc;
  if (!prm) return DNR_E_NULL;
  if (n < 0 || (prm->passes & 3) == 0 || (prm->passes & ~3) != 0) return DNR_E_SIZE;
  if ((prm->passes & 1) && !prm->use_normals) return DNR_E_OPTION;
  if (n == 0) return 0;
  if (!points || !values) return DNR_E_NULL;
  iso_eval_kernel<<<blocks_for(n, 128), 128, 0, (cudaStream_t)stream>>>(*fr, *prm, points, n, values);
  DNR_CHECK_LAUNCH();
  return 0;
}

extern "C" int64_t dnr_iso_octree_workspace_bytes(const DnrIsoGrid* g, int64_t n) {
  const int rc = check_grid(g);
  if (rc) return rc;
  if (n < 0) return DNR_E_SIZE;
  return (int64_t)OctLayout(nullptr, g, n).carve.total();
}

extern "C" int dnr_iso_octree(const DnrIsoGrid* g, const double* points, int64_t n, void* ws, int64_t ws_bytes,
                              int64_t* level_counts_host, void* stream) {
  const int rc = check_grid(g);
  if (rc) return rc;
  if (n < 0) return DNR_E_SIZE;
  if (!ws || !level_counts_host || (n > 0 && !points)) return DNR_E_NULL;
  const OctLayout L(ws, g, n);
  if (const int e = L.carve.check(ws_bytes)) return e;
  cudaStream_t s = (cudaStream_t)stream;
  int64_t *keys = L.keys, *sorted = L.sorted, *children = L.children, *leaves = L.leaves, *num = L.num;
  int64_t* lists[2] = {L.lists, L.lists + L.bound};
  uint8_t *split = L.split, *leaf = L.leaf;
  const int D = g->max_depth;
  for (int l = 0; l <= D; ++l) level_counts_host[l] = 0;
  if (!(n >= g->threshold && D > 0)) {  // the root is the only leaf
    DNR_CUDA(cudaMemsetAsync(leaves, 0, sizeof(int64_t), s));
    level_counts_host[0] = 1;
    return 0;
  }
  iso_keys_kernel<<<blocks_for(n), THREADS, 0, s>>>(*g, points, n, keys);
  DNR_CHECK_LAUNCH();
  size_t t = L.cub_bytes;
  DNR_CUDA(cub::DeviceRadixSort::SortKeys(L.cub_temp, t, keys, sorted, n, 0, 3 * D, s));
  DNR_CUDA(cudaMemsetAsync(lists[0], 0, sizeof(int64_t), s));  // the root, level 0, code 0
  int64_t n_parents = 1, n_leaves = 0;
  for (int l = 1; l <= D; ++l) {
    const int64_t m = 8 * n_parents;
    iso_children_kernel<<<blocks_for(m), THREADS, 0, s>>>(*g, l, lists[(l - 1) & 1], n_parents, sorted, n, children, split, leaf);
    DNR_CHECK_LAUNCH();
    t = L.cub_bytes;
    DNR_CUDA(cub::DeviceSelect::Flagged(L.cub_temp, t, children, split, lists[l & 1], num, m, s));
    t = L.cub_bytes;
    DNR_CUDA(cub::DeviceSelect::Flagged(L.cub_temp, t, children, leaf, leaves + n_leaves, num + 1, m, s));
    int64_t got[2];
    DNR_CUDA(cudaMemcpyAsync(got, num, sizeof(got), cudaMemcpyDeviceToHost, s));
    DNR_CUDA(cudaStreamSynchronize(s));
    level_counts_host[l] = got[1];
    n_leaves += got[1];
    n_parents = got[0];
    if (n_parents > L.bound) return DNR_E_OVERFLOW;  // cannot happen: each split node holds >= threshold samples
    if (n_parents == 0) break;
  }
  return 0;
}

extern "C" int64_t dnr_iso_corners_workspace_bytes(const DnrIsoGrid* g, int64_t n_leaves) {
  const int rc = check_grid(g);
  if (rc) return rc;
  if (n_leaves <= 0) return DNR_E_SIZE;
  return (int64_t)CornerLayout(nullptr, n_leaves).carve.total();
}

extern "C" int dnr_iso_corners(const DnrIsoGrid* g, const void* octree_ws, const int64_t* level_counts_host, void* ws,
                               int64_t ws_bytes, int64_t* leaves, int64_t* corner_keys, double* corner_points,
                               int32_t* leaf_corners, int64_t* n_corners_host, void* stream) {
  const int rc = check_grid(g);
  if (rc) return rc;
  if (!octree_ws || !level_counts_host || !ws || !leaves || !corner_keys || !corner_points || !leaf_corners || !n_corners_host)
    return DNR_E_NULL;
  int64_t n_leaves = 0;
  for (int l = 0; l <= g->max_depth; ++l) n_leaves += level_counts_host[l];
  if (n_leaves <= 0) return DNR_E_SIZE;
  const CornerLayout L(ws, n_leaves);
  if (const int e = L.carve.check(ws_bytes)) return e;
  if (8 * n_leaves > INT32_MAX) return DNR_E_OVERFLOW;
  cudaStream_t s = (cudaStream_t)stream;
  int64_t *keys8 = L.keys8, *sorted = L.sorted, *num = L.num;
  const int64_t* octree_leaves = OctLayout(octree_ws, g, 0).leaves;
  DNR_CUDA(cudaMemcpyAsync(leaves, octree_leaves, sizeof(int64_t) * n_leaves, cudaMemcpyDeviceToDevice, s));
  const int D = g->max_depth;
  const int64_t m = 8 * n_leaves;
  iso_corner_keys_kernel<<<blocks_for(m), THREADS, 0, s>>>(D, leaves, n_leaves, keys8);
  DNR_CHECK_LAUNCH();
  int bits = 1;
  while (bits < 63 && (int64_t(1) << bits) < ((int64_t(1) << D) + 1) * ((int64_t(1) << D) + 1) * ((int64_t(1) << D) + 1)) ++bits;
  size_t t = L.cub_bytes;
  DNR_CUDA(cub::DeviceRadixSort::SortKeys(L.cub_temp, t, keys8, sorted, m, 0, bits, s));
  t = L.cub_bytes;
  DNR_CUDA(cub::DeviceSelect::Unique(L.cub_temp, t, sorted, corner_keys, num, m, s));
  iso_corner_index_kernel<<<blocks_for(m), THREADS, 0, s>>>(keys8, m, corner_keys, num, leaf_corners);
  DNR_CHECK_LAUNCH();
  iso_corner_points_kernel<<<blocks_for(m), THREADS, 0, s>>>(*g, corner_keys, num, corner_points);
  DNR_CHECK_LAUNCH();
  DNR_CUDA(cudaMemcpyAsync(n_corners_host, num, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  DNR_CUDA(cudaStreamSynchronize(s));
  return 0;
}

extern "C" int dnr_iso_fill(const DnrIsoGrid* g, const int64_t* leaves, const int64_t* level_counts_host, const int32_t* leaf_corners,
                            const float* corner_values, float* field, void* stream) {
  const int rc = check_grid(g);
  if (rc) return rc;
  if (!leaves || !level_counts_host || !leaf_corners || !corner_values || !field) return DNR_E_NULL;
  cudaStream_t s = (cudaStream_t)stream;
  const int D = g->max_depth;
  int64_t off = 0;
  for (int l = 0; l <= D; ++l) {  // coarse to fine: the smallest leaf holding a sample writes it last
    const int64_t cnt = level_counts_host[l];
    if (cnt < 0) return DNR_E_SIZE;
    if (cnt == 0) continue;
    const int64_t side = (int64_t(1) << (D - l)) + 1;
    const int64_t total = cnt * side * side * side;
    const unsigned nb = (unsigned)std::min<int64_t>((total + THREADS - 1) / THREADS, (int64_t)DNR_NUM_SMS * 16);
    iso_fill_kernel<<<nb, THREADS, 0, s>>>(D, leaves + off, cnt, side, leaf_corners + 8 * off, corner_values, field);
    DNR_CHECK_LAUNCH();
    off += cnt;
  }
  return 0;
}
