// Grid-hash k-nearest-neighbour search on the device (SURVEY.md §8f-4, "next" row).  Replaces the CPU sklearn search
// behind /root/reference/dn_splatter/utils/knn.py:29-43 (knn_sk: k+1 neighbours, first column dropped) that
// get_closest_gaussians (dn_model.py:1061-1075) and compute_level_surface_points (:1262) call, and nerfstudio's
// k_nearest_sklearn used by populate_modules (dn_model.py:187) [EXT].
//
// Build: points are binned into a uniform grid (origin / cell size / dims chosen by the host from the point statistics;
// points outside the box are clamped into the border cells, which keeps the bound below valid), sorted by cell with cub,
// and each cell's [start, end) range recorded.  Query: one thread per query walks cube shells of growing Chebyshev radius
// r around its own (clamped) cell, keeping the K best in a sorted per-thread list.
//
// Stop rule.  In exact arithmetic the coordinate -> cell map u = (x - lo) / cell is monotone per axis, so two points whose
// cells differ by D along an axis are more than (D-1) cells apart and, after shell r, everything unvisited is > r * cell
// away.  The kernel bins by fl(fl(x - lo) * inv_cell) in fp32: three roundings (the difference, inv_cell = fl(1 / cell),
// the product), so u is off by at most 4 eps |u| (eps = 2^-24, one more for a host that rounds 1 / cell twice).  Along
// the axis where the cells differ by r+1 the computed gap exceeds r, the larger u is >= 1 and the smaller one < dim, so
// the true gap exceeds r (1 - 4 eps) - 8 eps dim >= r - 12 eps max_dim cells (r < dim).  The search
// therefore stops only once the K-th distance <= (r - delta) * cell with delta = 2^-18 max_dim, 5.3x that bound (about
// 1e-3 cells at the 256-cell cap of choose_grid; measured binning errors reach 2.4e-5 cells there).  What remains is the
// fp32 rounding of the distances themselves: a returned neighbour is farther than an unreturned one only when their
// squared distances agree to about 10 eps relative, the band inside which fp32 cannot order them anyway.
//
// Pinned on the CPU by a numpy mirror against sklearn (tests/test_knn_grid_cpu.py) and on the GPU per query against
// brute-force fp64 distances (tests/test_gpu_knn_density.py).
#include <cub/cub.cuh>

#include "common.cuh"

namespace {

constexpr int KNN_MAX = 33;  // k <= 32 plus the dropped self / nearest column

// dnr_knn_query reads the grid (pts_sorted, cell_start, cell_end) that dnr_knn_build left in the same workspace
struct KnnLayout {
  DnrCarver carve;
  uint32_t *cell_ids, *cell_ids_sorted;
  int32_t *order, *order_sorted, *cell_start, *cell_end;
  float4* pts_sorted;
  void* cub_temp;
  size_t cub_bytes = 0;
  KnnLayout(const void* base, int32_t n, int64_t n_cells) : carve(base) {
    cell_ids = carve.take<uint32_t>(n);
    cell_ids_sorted = carve.take<uint32_t>(n);
    order = carve.take<int32_t>(n);
    order_sorted = carve.take<int32_t>(n);
    pts_sorted = carve.take<float4>(n);
    cell_start = carve.take<int32_t>(n_cells);
    cell_end = carve.take<int32_t>(n_cells);
    const cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                                          (const int32_t*)nullptr, (int32_t*)nullptr, n, 0, 32);
    cub_temp = carve.cub_scratch(e, cub_bytes);
  }
};

__device__ __forceinline__ int cell_coord(float x, float lo, float inv_cell, int dim) {
  const int c = (int)floorf((x - lo) * inv_cell);
  return min(max(c, 0), dim - 1);
}

__global__ void knn_bin_kernel(const float* __restrict__ pts, int n, DnrKnnGrid g, uint32_t* __restrict__ cell_ids,
                               int32_t* __restrict__ order) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int cx = cell_coord(pts[3 * i + 0], g.lo[0], g.inv_cell, g.dims[0]);
  const int cy = cell_coord(pts[3 * i + 1], g.lo[1], g.inv_cell, g.dims[1]);
  const int cz = cell_coord(pts[3 * i + 2], g.lo[2], g.inv_cell, g.dims[2]);
  cell_ids[i] = (uint32_t)((cz * g.dims[1] + cy) * g.dims[0] + cx);
  order[i] = i;
}

__global__ void knn_ranges_kernel(const float* __restrict__ pts, int n, const uint32_t* __restrict__ cell_sorted,
                                  const int32_t* __restrict__ order_sorted, float4* __restrict__ pts_sorted,
                                  int32_t* __restrict__ cell_start, int32_t* __restrict__ cell_end) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int src = order_sorted[i];
  pts_sorted[i] = make_float4(pts[3 * src], pts[3 * src + 1], pts[3 * src + 2], __int_as_float(src));
  const uint32_t c = cell_sorted[i];
  if (i == 0 || cell_sorted[i - 1] != c) cell_start[c] = i;
  if (i == n - 1 || cell_sorted[i + 1] != c) cell_end[c] = i + 1;
}

struct TopK {
  float d[KNN_MAX];
  int id[KNN_MAX];
  int count;
};

__device__ __forceinline__ void topk_insert(TopK& t, int K, float d2, int id) {
  if (t.count == K && !(d2 < t.d[K - 1])) return;
  int pos = t.count < K ? t.count : K - 1;
  while (pos > 0 && t.d[pos - 1] > d2) {  // strict: an equal distance keeps the candidate seen first
    t.d[pos] = t.d[pos - 1];
    t.id[pos] = t.id[pos - 1];
    --pos;
  }
  t.d[pos] = d2;
  t.id[pos] = id;
  if (t.count < K) ++t.count;
}

__device__ __forceinline__ void scan_cell(TopK& t, int K, float qx, float qy, float qz, int cell, const float4* __restrict__ pts_sorted,
                                          const int32_t* __restrict__ cell_start, const int32_t* __restrict__ cell_end) {
  const int e = cell_end[cell];
  for (int j = cell_start[cell]; j < e; ++j) {
    const float4 p = pts_sorted[j];
    const float dx = p.x - qx, dy = p.y - qy, dz = p.z - qz;
    topk_insert(t, K, dx * dx + dy * dy + dz * dz, __float_as_int(p.w));
  }
}

__global__ void __launch_bounds__(128) knn_query_kernel(const float* __restrict__ queries, int m, DnrKnnGrid g, int K, int skip,
                                                        const float4* __restrict__ pts_sorted, const int32_t* __restrict__ cell_start,
                                                        const int32_t* __restrict__ cell_end, int64_t* __restrict__ out_idx,
                                                        float* __restrict__ out_dist) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= m) return;
  const float qx = queries[3 * q], qy = queries[3 * q + 1], qz = queries[3 * q + 2];
  const int cx = cell_coord(qx, g.lo[0], g.inv_cell, g.dims[0]);
  const int cy = cell_coord(qy, g.lo[1], g.inv_cell, g.dims[1]);
  const int cz = cell_coord(qz, g.lo[2], g.inv_cell, g.dims[2]);
  const int r_max = max(max(max(cx, g.dims[0] - 1 - cx), max(cy, g.dims[1] - 1 - cy)), max(cz, g.dims[2] - 1 - cz));
  const float delta = (float)max(max(g.dims[0], g.dims[1]), g.dims[2]) * 0x1p-18f;  // binning slack in cells (see top)
  TopK t;
  t.count = 0;
  for (int r = 0; r <= r_max; ++r) {
    const int z0 = max(cz - r, 0), z1 = min(cz + r, g.dims[2] - 1);
    const int y0 = max(cy - r, 0), y1 = min(cy + r, g.dims[1] - 1);
    for (int z = z0; z <= z1; ++z) {
      const bool z_face = (z == cz - r) || (z == cz + r);
      for (int y = y0; y <= y1; ++y) {
        const bool face = z_face || (y == cy - r) || (y == cy + r);
        const int row = (z * g.dims[1] + y) * g.dims[0];
        if (face) {  // the whole x-run of this row belongs to the shell
          const int x1 = min(cx + r, g.dims[0] - 1);
          for (int x = max(cx - r, 0); x <= x1; ++x) scan_cell(t, K, qx, qy, qz, row + x, pts_sorted, cell_start, cell_end);
        } else {  // only the two end caps
          if (cx - r >= 0) scan_cell(t, K, qx, qy, qz, row + cx - r, pts_sorted, cell_start, cell_end);
          if (cx + r < g.dims[0]) scan_cell(t, K, qx, qy, qz, row + cx + r, pts_sorted, cell_start, cell_end);
        }
      }
    }
    const float reach = fmaxf((float)r - delta, 0.f) * g.cell;
    if (t.count == K && t.d[K - 1] <= reach * reach) break;
  }
  const int k_out = K - skip;
  for (int j = 0; j < k_out; ++j) {
    const bool have = (j + skip) < t.count;
    out_idx[(size_t)q * k_out + j] = have ? (int64_t)t.id[j + skip] : (int64_t)-1;
    if (out_dist) out_dist[(size_t)q * k_out + j] = have ? sqrtf(t.d[j + skip]) : INFINITY;
  }
}

int check_grid(const DnrKnnGrid* g, int64_t* n_cells) {
  if (!g) return DNR_E_NULL;
  if (g->dims[0] <= 0 || g->dims[1] <= 0 || g->dims[2] <= 0 || !(g->cell > 0.f) || !(g->inv_cell > 0.f)) return DNR_E_SIZE;
  *n_cells = (int64_t)g->dims[0] * g->dims[1] * g->dims[2];
  if (*n_cells > (int64_t)1 << 26) return DNR_E_SIZE;
  return 0;
}

}  // namespace

extern "C" int64_t dnr_knn_workspace_bytes(int32_t n_points, const DnrKnnGrid* grid) {
  int64_t n_cells = 0;
  if (n_points <= 0 || check_grid(grid, &n_cells)) return -1;
  return (int64_t)KnnLayout(nullptr, n_points, n_cells).carve.total();
}

extern "C" int dnr_knn_build(const float* points, int32_t n_points, const DnrKnnGrid* grid, void* ws, int64_t ws_bytes, void* stream) {
  if (!points || !ws) return DNR_E_NULL;
  if (n_points <= 0) return DNR_E_SIZE;
  int64_t n_cells = 0;
  const int rc = check_grid(grid, &n_cells);
  if (rc) return rc;
  const KnnLayout L(ws, n_points, n_cells);
  if (const int e = L.carve.check(ws_bytes)) return e;
  cudaStream_t s = (cudaStream_t)stream;
  const int blocks = (n_points + 255) / 256;
  knn_bin_kernel<<<blocks, 256, 0, s>>>(points, n_points, *grid, L.cell_ids, L.order);
  DNR_CHECK_LAUNCH();
  size_t temp = L.cub_bytes;
  int bits = 1;
  while (((int64_t)1 << bits) < n_cells) ++bits;
  DNR_CUDA(cub::DeviceRadixSort::SortPairs(L.cub_temp, temp, L.cell_ids, L.cell_ids_sorted, L.order, L.order_sorted, n_points, 0,
                                           bits, s));
  DNR_CUDA(cudaMemsetAsync(L.cell_start, 0, sizeof(int32_t) * (size_t)n_cells, s));
  DNR_CUDA(cudaMemsetAsync(L.cell_end, 0, sizeof(int32_t) * (size_t)n_cells, s));
  knn_ranges_kernel<<<blocks, 256, 0, s>>>(points, n_points, L.cell_ids_sorted, L.order_sorted, L.pts_sorted, L.cell_start,
                                           L.cell_end);
  DNR_CHECK_LAUNCH();
  return 0;
}

extern "C" int dnr_knn_query(int32_t n_points, const DnrKnnGrid* grid, const void* ws, const float* queries, int32_t n_queries, int32_t k,
                             int32_t skip_first, int64_t* out_idx, float* out_dist, void* stream) {
  if (!ws || !queries || !out_idx) return DNR_E_NULL;
  if (n_points <= 0 || n_queries <= 0 || k <= 0) return DNR_E_SIZE;
  const int K = k + (skip_first ? 1 : 0);
  if (K > KNN_MAX) return DNR_E_OPTION;
  int64_t n_cells = 0;
  const int rc = check_grid(grid, &n_cells);
  if (rc) return rc;
  const KnnLayout L(ws, n_points, n_cells);
  knn_query_kernel<<<(n_queries + 127) / 128, 128, 0, (cudaStream_t)stream>>>(queries, n_queries, *grid, K, skip_first ? 1 : 0,
                                                                              L.pts_sorted, L.cell_start, L.cell_end, out_idx, out_dist);
  DNR_CHECK_LAUNCH();
  return 0;
}
