// Tile binning: one binning shared by the colour/depth and the normal channels.
//
// Replaces gsplat isect_tiles + cub radix sort of 64-bit (tile|depth) keys + isect_offset_encode
// (reference call sites /root/reference/dn_splatter/dn_model.py:495-516 and the second, redundant
// binning hidden in the legacy rasterize_gaussians call at :564-575).
//
// Formulation (same result, ~4x less sort traffic than sorting I 64-bit keys):
//   1. sort the N Gaussians once by depth bits (32-bit keys, N items; culled = 0xFFFFFFFF go last);
//      a stable sort keeps equal depths in ascending Gaussian index;
//   2. count, per Gaussian (one warp each, lanes over its tile box), the tiles it can really reach:
//      a conservative exact ellipse/rectangle test (dnr_rect_hit) drops the ~55 % of bbox tiles in which no
//      pixel can reach alpha >= 1/255 — those pairs would be skipped by every pixel anyway, so the rendered
//      images are bit-identical; DNR_FLAG_EXACT_LISTS keeps gsplat's full bbox lists for parity checks;
//      exclusive-scan the counts in depth order -> where each Gaussian emits;
//   3. emit (tile_id, gaussian_id) pairs in depth order — one warp per Gaussian, ballot-compacted, coalesced;
//   4. STABLE radix sort of the I pairs on the tile-id bits only (13-15 bits, 16-bit keys): within a
//      tile the depth order of step 1 survives, so the list equals gsplat's sort by (tile, depth, id);
//   5. tile offsets from the sorted tile ids.
//
// Granularity (round 2): the lists are kept per SUPERTILE of (16 << list_shift)^2 pixels.  Only ~7 % of the pairs of a
// per-tile list are ever composited (pixels saturate long before the list ends), so emitting and sorting per-tile pairs
// was the largest waste of the step (11.5 M pairs at 1 M Gaussians / 1080p).  With 64-pixel supertiles 4-5x fewer pairs
// are emitted and sorted; each 16x16 tile then filters the chunks of its supertile's list that it actually walks
// (dnr_tile_hit in csrc/raster.cu).  list_shift = 0 keeps one list per tile (gsplat's lists with DNR_FLAG_EXACT_LISTS).
#include <cub/cub.cuh>
#include <thrust/iterator/transform_iterator.h>

#include "common.cuh"

namespace {

struct ToI64 {
  __host__ __device__ __forceinline__ int64_t operator()(int32_t v) const { return (int64_t)v; }
};

__global__ void iota_kernel(int32_t* out, int32_t n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = i;
}

struct ScanWs {
  DnrCarver carve;
  uint32_t* keys_sorted;
  int32_t* order;
  int32_t* iota;
  int32_t* counts;       // [N+1] tiles really touched, in depth order (last = 0)
  int64_t* isect_start;  // [N+1]
  void* cub_temp;
  size_t cub_bytes;
  ScanWs(void* base, int32_t n) : carve(base) {
    keys_sorted = carve.take<uint32_t>(n);
    order = carve.take<int32_t>(n);
    iota = carve.take<int32_t>(n);
    counts = carve.take<int32_t>((size_t)n + 1);
    isect_start = carve.take<int64_t>((size_t)n + 1);
    size_t sort_bytes = 0, scan_bytes = 0;
    const cudaError_t e1 = cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                                           (const int32_t*)nullptr, (int32_t*)nullptr, n, 0, 32);
    auto it = thrust::make_transform_iterator((const int32_t*)nullptr, ToI64());
    const cudaError_t e2 = cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, it, (int64_t*)nullptr, n + 1);
    cub_bytes = sort_bytes > scan_bytes ? sort_bytes : scan_bytes;
    cub_temp = carve.cub_scratch(e1 != cudaSuccess ? e1 : e2, cub_bytes);
  }
};

// the padding key is n_tiles (one past the last list id), so `tile_bits` = bits of the value n_tiles
template <typename KeyT>
inline int sort_end_bit(int tile_bits) {
  const int full = (int)(8 * sizeof(KeyT));
  return tile_bits < full ? tile_bits : full;
}

template <typename KeyT>
struct SortWs {
  DnrCarver carve;
  KeyT* keys_in;
  KeyT* keys_out;
  int32_t* gids_in;
  void* cub_temp;
  size_t cub_bytes = 0;
  SortWs(void* base, int64_t n_isects, int tile_bits) : carve(base) {
    const size_t n = (size_t)(n_isects > 0 ? n_isects : 1);
    keys_in = carve.template take<KeyT>(n);
    keys_out = carve.template take<KeyT>(n);
    gids_in = carve.template take<int32_t>(n);
    const cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const KeyT*)nullptr, (KeyT*)nullptr, (const int32_t*)nullptr,
                                                          (int32_t*)nullptr, (int64_t)n, 0, sort_end_bit<KeyT>(tile_bits));
    cub_temp = carve.cub_scratch(e, cub_bytes);
  }
};

inline int tile_bits_for(int n_tiles) {  // bits needed to represent the values 0..n_tiles (n_tiles = the padding key)
  int b = 1;
  while ((1 << b) <= n_tiles) ++b;
  return b;
}

// ---- precise-hit emission -------------------------------------------------------------------------------------
// For a Gaussian (centre m, conic A,B,C) and the largest sigma `lim` at which a pixel can still reach alpha >= 1/255,
// the reachable region is the ellipse q(e) = 0.5 (A ex^2 + C ey^2) + B ex ey <= lim (e = pixel - m).  For one row of
// tiles (pixel centres ey in [e0,e1]) the ellipse slice is convex, so the tiles it touches form ONE span: those
// whose centre range overlaps [xmin,xmax], the x-extent of the slice.  With D(ey) = (B^2-AC) ey^2 + 2 A lim the
// slice at height ey is ex in [(-B ey -+ sqrt D)/A]; the upper root is concave in ey (max at the ellipse's right-most
// point or at an end of the interval), the lower root convex.  Everything is widened by small slacks: the span may
// only err on the keeping side (kept-but-unreachable pairs are skipped per pixel anyway; images are bit-identical).
struct HitGauss {
  int g, radius, x0, y0, nx, ny;
  float mx, my, A, B, invA, bac, twoAL, ex_max, ey_max, ey_star;
};

// box of list tiles (edge `ts` pixels) a projected Gaussian overlaps; ts = 16 reproduces dnr_tile_box bit for bit
__device__ __forceinline__ void list_box(float mx, float my, int radius, int ts, int tiles_x, int tiles_y, int& x0, int& y0,
                                         int& x1, int& y1) {
  if (ts == DNR_TILE) { dnr_tile_box(mx, my, radius, tiles_x, tiles_y, x0, y0, x1, y1); return; }
  const float inv = 1.0f / (float)ts;  // power of two: exact
  const float r = (float)radius * inv, tcx = mx * inv, tcy = my * inv;
  x0 = min(max((int)floorf(tcx - r), 0), tiles_x);
  y0 = min(max((int)floorf(tcy - r), 0), tiles_y);
  x1 = min(max((int)ceilf(tcx + r), 0), tiles_x);
  y1 = min(max((int)ceilf(tcy + r), 0), tiles_y);
}

__device__ __forceinline__ HitGauss load_hit_gauss(const DnrArgs& a, const int32_t* __restrict__ order, int i, int tiles_x,
                                                   int tiles_y) {
  HitGauss h;
  h.g = 0; h.radius = 0; h.x0 = h.y0 = h.nx = h.ny = 0;
  h.mx = h.my = h.A = h.B = h.invA = h.bac = h.twoAL = h.ex_max = h.ey_max = h.ey_star = 0.f;
  if (i < a.n_gauss) {
    h.g = order[i];
    h.radius = a.radii[h.g];
    if (h.radius > 0) {
      h.mx = a.means2d[h.g * 2 + 0]; h.my = a.means2d[h.g * 2 + 1];
      int x1, y1;
      list_box(h.mx, h.my, h.radius, DNR_TILE << a.list_shift, tiles_x, tiles_y, h.x0, h.y0, x1, y1);
      h.nx = x1 - h.x0;
      h.ny = y1 - h.y0;
      if (!(a.flags & DNR_FLAG_EXACT_LISTS)) {
        const float A = a.conics[h.g * 3 + 0], B = a.conics[h.g * 3 + 1], C = a.conics[h.g * 3 + 2];
        const float L = a.cull_lim[h.g];
        // A C - B^2 by Kahan's difference of products: for a needle (eps2d well below 0.3) the two products agree in
        // all but their last bits, and the plain difference comes out <= 0 for a conic that is an ellipse
        const float bb = B * B;
        const float det = fmaf(A, C, -bb) + fmaf(-B, B, bb);
        if (!(L > 0.f) || !(det > 0.f)) {
          h.ny = 0;  // cannot reach alpha >= 1/255 anywhere
        } else {
          h.A = A; h.B = B; h.invA = 1.0f / A; h.bac = -det; h.twoAL = 2.0f * A * L;
          h.ex_max = sqrtf(2.0f * L * C / det) * 1.0001f + 0.01f;
          h.ey_max = sqrtf(2.0f * L * A / det) * 1.0001f + 0.01f;
          h.ey_star = -B * h.ex_max / C;  // height of the right-most point; the left-most one sits at -ey_star
        }
      }
    }
  }
  return h;
}

// Tiles [lo, hi) of tile-row `ty` that the Gaussian can reach (empty when hi <= lo); `exact` keeps the whole box row.
__device__ __forceinline__ void row_span(const HitGauss& h, int ty, bool exact, int ts, int& lo, int& hi) {
  lo = h.x0; hi = h.x0 + h.nx;
  if (exact) return;
  float e0 = ((float)(ty * ts) + 0.5f) - h.my - 0.01f;
  float e1 = ((float)(ty * ts + ts - 1) + 0.5f) - h.my + 0.01f;
  if (e0 > h.ey_max || e1 < -h.ey_max) { hi = lo; return; }
  e0 = fmaxf(e0, -h.ey_max); e1 = fminf(e1, h.ey_max);
  const float s0 = sqrtf(fmaxf(fmaf(h.bac, e0 * e0, h.twoAL), 0.f)), s1 = sqrtf(fmaxf(fmaf(h.bac, e1 * e1, h.twoAL), 0.f));
  float xmax = fmaxf((-h.B * e0 + s0) * h.invA, (-h.B * e1 + s1) * h.invA);
  float xmin = fminf((-h.B * e0 - s0) * h.invA, (-h.B * e1 - s1) * h.invA);
  if (h.ey_star >= e0 && h.ey_star <= e1) xmax = h.ex_max;
  if (-h.ey_star >= e0 && -h.ey_star <= e1) xmin = -h.ex_max;
  xmax = xmax + 0.01f + 1e-5f * fabsf(xmax);
  xmin = xmin - 0.01f - 1e-5f * fabsf(xmin);
  // tile tx holds pixel centres [ts tx + 0.5, ts tx + ts - 0.5]
  const float inv = 1.0f / (float)ts;
  const int t_lo = (int)ceilf((h.mx + xmin - ((float)ts - 0.5f)) * inv);
  const int t_hi = (int)floorf((h.mx + xmax - 0.5f) * inv) + 1;
  lo = max(lo, t_lo); hi = min(hi, t_hi);
}

// One lane per depth-sorted Gaussian: counts[i] = number of tiles of its box that it can really reach.
__global__ void __launch_bounds__(256) count_kernel(const DnrArgs a, const int32_t* __restrict__ order,
                                                   int32_t* __restrict__ counts, int tiles_x, int tiles_y) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > a.n_gauss) return;
  const HitGauss h = load_hit_gauss(a, order, i, tiles_x, tiles_y);
  const bool exact = (a.flags & DNR_FLAG_EXACT_LISTS) != 0;
  const int ts = DNR_TILE << a.list_shift;
  int cnt = 0;
  for (int r = 0; r < h.ny; ++r) {
    int lo, hi;
    row_span(h, h.y0 + r, exact, ts, lo, hi);
    cnt += max(hi - lo, 0);
  }
  counts[i] = (i < a.n_gauss) ? cnt : 0;
}

// One lane per depth-sorted Gaussian (like count_kernel): it recomputes its row spans and writes its (list id, Gaussian
// id) pairs at [isect_start[i], isect_start[i+1]) — row-major, ascending x: the order gsplat emits.  At supertile
// granularity a Gaussian emits ~4-5 pairs, and neighbouring lanes (consecutive in depth order) own neighbouring output
// ranges, so the small per-lane stores of a warp land in a few contiguous sectors.  (Round 1 walked 8 Gaussians per warp
// with lanes over tile rows: 149 us at 1.8 M pairs, dominated by the per-Gaussian shuffle / ballot choreography.)
// Entries past the capacity are dropped; n_isects_dev keeps the true count and the caller raises (DnrCapacityError).
template <typename KeyT>
__global__ void __launch_bounds__(256) emit_kernel(const DnrArgs a, const int32_t* __restrict__ order,
                                                  const int64_t* __restrict__ isect_start, KeyT* __restrict__ keys,
                                                  int32_t* __restrict__ gids, int tiles_x, int tiles_y) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n_gauss) return;
  int64_t dst = isect_start[i];
  const int64_t dst_end = isect_start[i + 1];
  if (dst_end <= dst) return;
  const HitGauss h = load_hit_gauss(a, order, i, tiles_x, tiles_y);
  const int64_t cap = a.n_isects;
  const bool exact = (a.flags & DNR_FLAG_EXACT_LISTS) != 0;
  const int ts = DNR_TILE << a.list_shift;
  for (int r = 0; r < h.ny; ++r) {
    int lo, hi;
    row_span(h, h.y0 + r, exact, ts, lo, hi);
    const int row_key = (h.y0 + r) * tiles_x;
    for (int x = lo; x < hi; ++x, ++dst) {
      if (dst < cap) {
        keys[dst] = (KeyT)(row_key + x);
        gids[dst] = h.g;
      }
    }
  }
}

// Pads [count, capacity) with the maximal key so a fixed-size sort leaves them at the end.
template <typename KeyT>
__global__ void __launch_bounds__(256) pad_kernel(KeyT* __restrict__ keys, int32_t* __restrict__ gids,
                                                 const int64_t* __restrict__ n_isects_dev, int64_t cap, KeyT pad_key) {
  // only the tail [count, capacity) is touched: a small fixed grid strides over it
  for (int64_t i = *n_isects_dev + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (int64_t)gridDim.x * blockDim.x) {
    keys[i] = pad_key;
    gids[i] = 0;
  }
}

template <typename KeyT>
__global__ void __launch_bounds__(256) offsets_kernel(const KeyT* __restrict__ keys, const int64_t* __restrict__ n_isects_dev,
                                                     int64_t cap, int n_tiles, int32_t* __restrict__ offsets) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t n_isects = min(*n_isects_dev, cap);
  if (n_isects == 0) {
    if (i <= n_tiles) offsets[i] = 0;
    return;
  }
  if (i >= n_isects) return;
  const int cur = (int)keys[i];
  if (i == 0) {
    for (int t = 0; t <= cur; ++t) offsets[t] = 0;
  } else {
    const int prev = (int)keys[i - 1];
    for (int t = prev + 1; t <= cur; ++t) offsets[t] = (int32_t)i;
  }
  if (i == n_isects - 1) {
    for (int t = cur + 1; t <= n_tiles; ++t) offsets[t] = (int32_t)n_isects;
  }
}

template <typename KeyT>
int bin_sort_impl(const DnrArgs* a, cudaStream_t s, int n_tiles, int tile_bits) {
  const int tiles_x = dnr_stiles_x(a), tiles_y = dnr_stiles_y(a);
  const ScanWs sw(a->ws_scan, a->n_gauss);
  const int64_t cap = a->n_isects;
  const SortWs<KeyT> w(a->ws_sort, cap, tile_bits);
  if (const int e = w.carve.cub_error()) return e;
  if (cap > 0) {
    emit_kernel<KeyT><<<(unsigned)((a->n_gauss + 255) / 256), 256, 0, s>>>(*a, sw.order, sw.isect_start, w.keys_in, w.gids_in,
                                                                          tiles_x, tiles_y);
    DNR_CHECK_LAUNCH();
    pad_kernel<KeyT><<<DNR_NUM_SMS * 2, 256, 0, s>>>(w.keys_in, w.gids_in, a->n_isects_dev, cap, (KeyT)n_tiles);
    DNR_CHECK_LAUNCH();
    size_t bytes = w.cub_bytes;
    const int end_bit = sort_end_bit<KeyT>(tile_bits);
    DNR_CUDA(cub::DeviceRadixSort::SortPairs(w.cub_temp, bytes, (const KeyT*)w.keys_in, w.keys_out,
                                             (const int32_t*)w.gids_in, a->flatten_ids, cap, 0, end_bit, s));
  }
  const int64_t n = cap > (int64_t)n_tiles + 1 ? cap : (int64_t)n_tiles + 1;
  offsets_kernel<KeyT><<<(unsigned)((n + 255) / 256), 256, 0, s>>>(w.keys_out, a->n_isects_dev, cap, n_tiles, a->tile_offsets);
  DNR_CHECK_LAUNCH();
  return 0;
}

}  // namespace

extern "C" size_t dnr_bin_scan_workspace_bytes(int32_t n_gauss) {
  if (n_gauss <= 0) return 0;
  return ScanWs(nullptr, n_gauss).carve.total();
}

extern "C" int dnr_bin_scan(const DnrArgs* a, void* stream, int64_t* n_isects_host) {
  if (!a) return DNR_E_NULL;
  if (a->n_gauss <= 0 || a->width <= 0 || a->height <= 0) return DNR_E_SIZE;
  if (a->list_shift < 0 || a->list_shift > 3) return DNR_E_OPTION;
  if ((a->flags & DNR_FLAG_EXACT_LISTS) && a->list_shift != 0) return DNR_E_OPTION;
  if (!a->ws_scan || !a->depth_keys || !a->tiles_per_gauss || !a->n_isects_dev || !a->radii || !a->means2d) return DNR_E_NULL;
  if (!(a->flags & DNR_FLAG_EXACT_LISTS) && (!a->conics || !a->cull_lim)) return DNR_E_NULL;
  cudaStream_t s = (cudaStream_t)stream;
  const int32_t n = a->n_gauss;
  const ScanWs w(a->ws_scan, n);
  if (const int e = w.carve.cub_error()) return e;
  iota_kernel<<<(n + 255) / 256, 256, 0, s>>>(w.iota, n);
  DNR_CHECK_LAUNCH();
  size_t bytes = w.cub_bytes;
  DNR_CUDA(cub::DeviceRadixSort::SortPairs(w.cub_temp, bytes, (const uint32_t*)a->depth_keys, w.keys_sorted,
                                           (const int32_t*)w.iota, w.order, n, 0, 32, s));
  {
    const int64_t threads = (int64_t)n + 1;  // one lane per Gaussian (+ the terminating zero)
    count_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(*a, w.order, w.counts, dnr_stiles_x(a), dnr_stiles_y(a));
    DNR_CHECK_LAUNCH();
  }
  auto it = thrust::make_transform_iterator((const int32_t*)w.counts, ToI64());
  bytes = w.cub_bytes;
  DNR_CUDA(cub::DeviceScan::ExclusiveSum(w.cub_temp, bytes, it, w.isect_start, n + 1, s));
  DNR_CUDA(cudaMemcpyAsync(a->n_isects_dev, w.isect_start + n, sizeof(int64_t), cudaMemcpyDeviceToDevice, s));
  if (n_isects_host) {
    int64_t total = 0;
    DNR_CUDA(cudaMemcpyAsync(&total, w.isect_start + n, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    DNR_CUDA(cudaStreamSynchronize(s));
    *n_isects_host = total;
    if (total > 0x7FFFFFFFLL) return DNR_E_OVERFLOW;
  }
  return 0;
}

extern "C" size_t dnr_bin_sort_workspace_bytes(int32_t n_gauss, int64_t n_isects, int32_t n_tiles) {
  (void)n_gauss;
  if (n_isects < 0 || n_tiles <= 0) return 0;
  const int bits = tile_bits_for(n_tiles);
  if (n_tiles < 65536) return SortWs<uint16_t>(nullptr, n_isects, bits).carve.total();
  return SortWs<uint32_t>(nullptr, n_isects, bits).carve.total();
}

extern "C" int dnr_bin_sort(const DnrArgs* a, void* stream) {
  if (!a) return DNR_E_NULL;
  if (a->n_gauss <= 0 || a->n_isects < 0 || a->width <= 0 || a->height <= 0) return DNR_E_SIZE;
  if (a->n_isects > 0x7FFFFFFFLL) return DNR_E_OVERFLOW;
  if (!a->ws_scan || !a->ws_sort || !a->tile_offsets || !a->means2d || !a->radii || !a->n_isects_dev) return DNR_E_NULL;
  if (!(a->flags & DNR_FLAG_EXACT_LISTS) && (!a->conics || !a->cull_lim)) return DNR_E_NULL;
  if (a->n_isects > 0 && !a->flatten_ids) return DNR_E_NULL;
  if (a->list_shift < 0 || a->list_shift > 3) return DNR_E_OPTION;
  if ((a->flags & DNR_FLAG_EXACT_LISTS) && a->list_shift != 0) return DNR_E_OPTION;
  const int n_tiles = dnr_stiles_x(a) * dnr_stiles_y(a);  // number of lists
  const int bits = tile_bits_for(n_tiles);
  cudaStream_t s = (cudaStream_t)stream;
  if (n_tiles < 65536) return bin_sort_impl<uint16_t>(a, s, n_tiles, bits);
  return bin_sort_impl<uint32_t>(a, s, n_tiles, bits);
}
