// Mesh export on the device: TSDF fusion of rendered depth maps into a dense voxel grid, and marching cubes with welded,
// deterministic output (Python surface: dn_splatter_b200.mesh).  Replaces the open3d / PyMCubes calls of the reference's
// `gs-mesh o3dtsdf` and `gs-mesh marching` exporters (/root/reference/dn_splatter/export_mesh.py:714-820, 942-1044).
//
// dnr_tsdf_integrate: one thread per voxel (x = the grid's fastest axis z, grid = (z blocks, y, x)), so the 64-bit linear
// voxel index is built from three small coordinates without a division.  A voxel is read and written only where the
// view updates it (Open3D's legacy ScalableTSDFVolume.integrate rule, restated in DESIGN.md §2 and oracle/mesh_ref.py).
//
// Marching cubes, sized in two phases with one host read:
//   count   one CTA per grid row (i, j): every voxel classifies the cube whose lower corner it is, and counts the crossed
//           edges it owns (the three edges leaving it) that some valid cube uses.  Per-row totals of cubes, triangles
//           and vertices are scanned with cub; the three grand totals go to the host (the one synchronisation).
//   emit    the same per-row pass again, now with a block scan: it writes the ids and triangle offsets of the active
//           cubes and the vertices (ascending (voxel, axis) key, so the row offsets of the count phase place them);
//           then one thread per active cube writes its triangles, finding each corner's vertex by a binary search in
//           its row's few keys.  No atomics decide any position, so two runs are bit-identical.
// Workspace: 48 B per grid row in the count phase, 16 B per active cube + 8 B per vertex in the emit phase.
#include <cub/cub.cuh>

#include "common.cuh"
#include "mc_tables.cuh"

namespace {

constexpr int MC_THREADS = 256;
constexpr int MAX_DIM = 65535;  // grid rows are launched as (y, x) blocks
constexpr long long FIELD_MASK = (1ll << 21) - 1;  // packed per-row counts: cubes | tris << 21 | verts << 42

struct Cam {
  float fx, fy, cx, cy;
  float E[12];  // world -> camera (OpenCV), row-major [3,4]
};

// Voxel colour: the running means of r, g, b as three 21-bit unsigned fixed-point numbers in units of 2^-13 of a level
// (255 * 2^13 < 2^21), packed r | g << 21 | b << 42 into the 64 bits of q.z (low word) and q.w.  fp16 (0.125-level spacing
// above 128) rounds away every update smaller than 0.0625 level, so a mean over many views stops following them.
constexpr int COLOR_FRAC_BITS = 13;
constexpr uint64_t COLOR_MASK = (1ull << 21) - 1;

__device__ __forceinline__ uint64_t color_bits(const float4& q) {
  return (uint64_t)__float_as_uint(q.z) | ((uint64_t)__float_as_uint(q.w) << 32);
}

__global__ void __launch_bounds__(128) tsdf_integrate_kernel(DnrTsdfGrid g, Cam cam, const float* __restrict__ depth,
                                                             const float* __restrict__ rgb, const uint8_t* __restrict__ mask,
                                                             int W, int H, float depth_trunc) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= g.dims[2]) return;
  const int j = blockIdx.y, i = blockIdx.z;
  const float px = g.origin[0] + ((float)i + 0.5f) * g.voxel;
  const float py = g.origin[1] + ((float)j + 0.5f) * g.voxel;
  const float pz = g.origin[2] + ((float)k + 0.5f) * g.voxel;
  const float* E = cam.E;
  const float z = E[8] * px + E[9] * py + E[10] * pz + E[11];
  if (!(z > 0.f)) return;
  const float x = E[0] * px + E[1] * py + E[2] * pz + E[3];
  const float y = E[4] * px + E[5] * py + E[6] * pz + E[7];
  const float uf = cam.fx * x / z + cam.cx + 0.5f;
  const float vf = cam.fy * y / z + cam.cy + 0.5f;
  if (!(uf >= 1e-4f && uf < (float)W - 1e-4f && vf >= 1e-4f && vf < (float)H - 1e-4f)) return;
  const int u = (int)uf, v = (int)vf;
  const int64_t pix = (int64_t)v * W + u;
  float d = depth[pix];
  if ((mask != nullptr && mask[pix] == 0) || d > depth_trunc || d < 0.f) d = 0.f;
  if (!(d > 0.f)) return;
  const float a = ((float)u - cam.cx) / cam.fx, b = ((float)v - cam.cy) / cam.fy;
  const float sdf = (d - z) * sqrtf(1.f + a * a + b * b);
  if (!(sdf > -g.sdf_trunc)) return;
  const float t = fminf(1.f, sdf / g.sdf_trunc);
  // the reference's uint8 colour: np.asarray(rgb * 255, dtype=np.uint8) truncates (clamped here, NaN -> 0)
  int c[3];
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) c[ch] = (int)fminf(fmaxf(rgb[3 * pix + ch] * 255.f, 0.f), 255.f);
  float4* vox = reinterpret_cast<float4*>(g.voxels) + (((int64_t)i * g.dims[1] + j) * g.dims[2] + k);
  float4 q = *vox;  // {tsdf, weight, packed fixed-point r g b}
  const float w = q.y, w1 = w + 1.f;
  // colour mean (m * w + c) / (w + 1) in integers, rounded half up; the weight is an integer count (exact below 2^24)
  const uint64_t wi = (uint64_t)w, den2 = 2 * (wi + 1), cin = color_bits(q);
  uint64_t cout = 0;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const uint64_t m = (cin >> (21 * ch)) & COLOR_MASK;
    const uint64_t num = m * wi + ((uint64_t)c[ch] << COLOR_FRAC_BITS);
    cout |= ((2 * num + (wi + 1)) / den2) << (21 * ch);
  }
  q.x = (q.x * w + t) / w1;
  q.y = w1;
  q.z = __uint_as_float((uint32_t)cout);
  q.w = __uint_as_float((uint32_t)(cout >> 32));
  *vox = q;
}

// ---- marching cubes ------------------------------------------------------------------------------------------------
struct Geo {
  int X, Y, Z;
  float iso;
  float origin[3];
  float spacing;
  __device__ __forceinline__ int64_t lin(int i, int j, int k) const { return ((int64_t)i * Y + j) * Z + k; }
};

struct ScalarField {  // f[X,Y,Z], optional validity mask
  const float* f;
  const uint8_t* m;
  static constexpr bool has_color = false;
  __device__ __forceinline__ float val(int64_t i) const { return f[i]; }
  __device__ __forceinline__ bool ok(int64_t i) const { return m == nullptr || m[i] != 0; }
  __device__ __forceinline__ float3 color(int64_t) const { return make_float3(0.f, 0.f, 0.f); }
};

struct TsdfField {  // 16-byte TSDF voxels: valid where weight > 0
  const float4* v;
  static constexpr bool has_color = true;
  __device__ __forceinline__ float val(int64_t i) const { return reinterpret_cast<const float2*>(v + i)->x; }
  __device__ __forceinline__ bool ok(int64_t i) const { return reinterpret_cast<const float2*>(v + i)->y > 0.f; }
  __device__ __forceinline__ float3 color(int64_t i) const {
    const uint64_t u = color_bits(v[i]);  // exact in fp32: below 2^21 units
    constexpr float unit = 1.f / (1 << COLOR_FRAC_BITS);
    return make_float3((float)(u & COLOR_MASK) * unit, (float)((u >> 21) & COLOR_MASK) * unit,
                       (float)((u >> 42) & COLOR_MASK) * unit);
  }
};

// case of the cube with lower corner (i, j, k) (bit c: corner c inside, f < iso), or -1 when a corner is invalid
template <class F>
__device__ int cube_case(const F& f, const Geo& g, int i, int j, int k) {
  int cs = 0;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int64_t idx = g.lin(i + (c & 1), j + ((c >> 1) & 1), k + ((c >> 2) & 1));
    if (!f.ok(idx)) return -1;
    if (f.val(idx) < g.iso) cs |= 1 << c;
  }
  return cs;
}

template <class F>
__device__ bool cube_valid(const F& f, const Geo& g, int i, int j, int k) {
  if (i < 0 || j < 0 || k < 0 || i >= g.X - 1 || j >= g.Y - 1 || k >= g.Z - 1) return false;
#pragma unroll
  for (int c = 0; c < 8; ++c)
    if (!f.ok(g.lin(i + (c & 1), j + ((c >> 1) & 1), k + ((c >> 2) & 1)))) return false;
  return true;
}

// Bit a set: the edge along axis a leaving voxel (i, j, k) is crossed and used by a valid cube (so it is a vertex).
template <class F>
__device__ int owned_vertices(const F& f, const Geo& g, int i, int j, int k) {
  const int64_t idx = g.lin(i, j, k);
  if (!f.ok(idx)) return 0;
  const bool in0 = f.val(idx) < g.iso;
  const int p[3] = {i, j, k}, dim[3] = {g.X, g.Y, g.Z};
  const int64_t stride[3] = {(int64_t)g.Y * g.Z, (int64_t)g.Z, 1};
  int bits = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    if (p[a] + 1 >= dim[a]) continue;
    const int64_t n = idx + stride[a];
    if (!f.ok(n) || (f.val(n) < g.iso) == in0) continue;
    const int b = (a + 1) % 3, c = (a + 2) % 3;
    bool used = false;
    for (int q = 0; q < 4 && !used; ++q) {
      int lo[3] = {i, j, k};
      lo[b] -= q & 1;
      lo[c] -= q >> 1;
      used = cube_valid(f, g, lo[0], lo[1], lo[2]);
    }
    if (used) bits |= 1 << a;
  }
  return bits;
}

// packed {active cube, its triangles, owned vertices} of voxel (i, j, k); *case_out / *vbits_out for the emit pass
template <class F>
__device__ long long voxel_counts(const F& f, const Geo& g, int i, int j, int k, int* case_out, int* vbits_out) {
  int cs = -1;
  if (i < g.X - 1 && j < g.Y - 1 && k < g.Z - 1) cs = cube_case(f, g, i, j, k);
  const int nt = cs >= 0 ? (int)dnr_mc_ntri[cs] : 0;
  const int vb = owned_vertices(f, g, i, j, k);
  *case_out = cs;
  *vbits_out = vb;
  const int nv = (vb & 1) + ((vb >> 1) & 1) + ((vb >> 2) & 1);
  return (long long)(nt > 0) | ((long long)nt << 21) | ((long long)nv << 42);
}

template <class F>
__global__ void __launch_bounds__(MC_THREADS) mc_count_kernel(F f, Geo g, int64_t* __restrict__ cnt, int64_t R) {
  using Reduce = cub::BlockReduce<long long, MC_THREADS>;
  __shared__ typename Reduce::TempStorage tmp;
  const int i = blockIdx.y, j = blockIdx.x;
  const int64_t row = (int64_t)i * g.Y + j;
  long long sum = 0;
  for (int k = threadIdx.x; k < g.Z; k += MC_THREADS) {
    int cs, vb;
    sum += voxel_counts(f, g, i, j, k, &cs, &vb);
  }
  sum = Reduce(tmp).Sum(sum);
  if (threadIdx.x == 0) {
    cnt[row] = sum & FIELD_MASK;
    cnt[(R + 1) + row] = (sum >> 21) & FIELD_MASK;
    cnt[2 * (R + 1) + row] = sum >> 42;
    if (row == 0) cnt[R] = cnt[2 * R + 1] = cnt[3 * R + 2] = 0;  // the scans' tail entries: offsets [R] = totals
  }
}

template <class F>
__device__ void write_vertex(const F& f, const Geo& g, int i, int j, int k, int a, int64_t out, int64_t* __restrict__ vkeys,
                             float* __restrict__ verts, float* __restrict__ colors) {
  const int64_t idx = g.lin(i, j, k);
  const int64_t n = a == 0 ? g.lin(i + 1, j, k) : a == 1 ? g.lin(i, j + 1, k) : g.lin(i, j, k + 1);
  const float f0 = f.val(idx), f1 = f.val(n);
  const float t = (g.iso - f0) / (f1 - f0);
  const int p[3] = {i, j, k};
  vkeys[out] = idx * 3 + a;
#pragma unroll
  for (int c = 0; c < 3; ++c) verts[3 * out + c] = g.origin[c] + g.spacing * (c == a ? (float)p[c] + t : (float)p[c]);
  if (F::has_color && colors != nullptr) {
    const float3 c0 = f.color(idx), c1 = f.color(n);
    colors[3 * out + 0] = (c0.x + t * (c1.x - c0.x)) / 255.f;
    colors[3 * out + 1] = (c0.y + t * (c1.y - c0.y)) / 255.f;
    colors[3 * out + 2] = (c0.z + t * (c1.z - c0.z)) / 255.f;
  }
}

template <class F>
__global__ void __launch_bounds__(MC_THREADS) mc_compact_kernel(F f, Geo g, const int64_t* __restrict__ off, int64_t R,
                                                                int64_t* __restrict__ cube_ids, int64_t* __restrict__ tri_start,
                                                                int64_t* __restrict__ vkeys, float* __restrict__ verts,
                                                                float* __restrict__ colors) {
  using Scan = cub::BlockScan<long long, MC_THREADS>;
  __shared__ typename Scan::TempStorage tmp;
  const int i = blockIdx.y, j = blockIdx.x;
  const int64_t row = (int64_t)i * g.Y + j;
  int64_t base_c = off[row], base_t = off[(R + 1) + row], base_v = off[2 * (R + 1) + row];
  for (int k0 = 0; k0 < g.Z; k0 += MC_THREADS) {
    const int k = k0 + threadIdx.x;
    int cs = -1, vb = 0;
    long long packed = 0, prefix, total;
    if (k < g.Z) packed = voxel_counts(f, g, i, j, k, &cs, &vb);
    Scan(tmp).ExclusiveSum(packed, prefix, total);
    if (packed & FIELD_MASK) {
      const int64_t pos = base_c + (prefix & FIELD_MASK);
      cube_ids[pos] = g.lin(i, j, k);
      tri_start[pos] = base_t + ((prefix >> 21) & FIELD_MASK);
    }
    int64_t vpos = base_v + (prefix >> 42);
    for (int a = 0; a < 3; ++a)
      if ((vb >> a) & 1) write_vertex(f, g, i, j, k, a, vpos++, vkeys, verts, colors);
    base_c += total & FIELD_MASK;
    base_t += (total >> 21) & FIELD_MASK;
    base_v += total >> 42;
    __syncthreads();  // tmp is reused by the next chunk's scan
  }
}

template <class F>
__global__ void __launch_bounds__(MC_THREADS) mc_faces_kernel(F f, Geo g, const int64_t* __restrict__ cube_ids,
                                                              const int64_t* __restrict__ tri_start, int64_t n_cubes,
                                                              const int64_t* __restrict__ voff, const int64_t* __restrict__ vkeys,
                                                              int32_t* __restrict__ faces) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n_cubes) return;
  const int64_t lin = cube_ids[q], plane = (int64_t)g.Y * g.Z;
  const int i = (int)(lin / plane), j = (int)((lin % plane) / g.Z), k = (int)(lin % g.Z);
  const int cs = cube_case(f, g, i, j, k);
  const int nt = dnr_mc_ntri[cs];
  int32_t* out = faces + 3 * tri_start[q];
  for (int e3 = 0; e3 < 3 * nt; ++e3) {
    const int e = dnr_mc_tri[cs][e3], c0 = dnr_mc_edge_c0[e];
    const int vi = i + (c0 & 1), vj = j + ((c0 >> 1) & 1), vk = k + ((c0 >> 2) & 1);
    const int64_t key = g.lin(vi, vj, vk) * 3 + dnr_mc_edge_axis[e];
    const int64_t row = (int64_t)vi * g.Y + vj;
    int64_t lo = voff[row], hi = voff[row + 1];
    while (lo < hi) {  // lower bound of key among the row's vertices
      const int64_t mid = (lo + hi) >> 1;
      if (vkeys[mid] < key) lo = mid + 1; else hi = mid;
    }
    out[e3] = (int32_t)lo;
  }
}

int check_field(const DnrMcField* f, Geo* g) {
  if (!f) return DNR_E_NULL;
  if ((f->values == nullptr) == (f->tsdf == nullptr)) return DNR_E_NULL;  // exactly one of them
  for (int a = 0; a < 3; ++a)
    if (f->dims[a] <= 0 || f->dims[a] > MAX_DIM) return DNR_E_SIZE;
  if (!(f->spacing > 0.f)) return DNR_E_SIZE;
  g->X = f->dims[0];
  g->Y = f->dims[1];
  g->Z = f->dims[2];
  g->iso = f->iso;
  for (int a = 0; a < 3; ++a) g->origin[a] = f->origin[a];
  g->spacing = f->spacing;
  return 0;
}

// dnr_mc_emit reads the exclusive scans `off` that dnr_mc_count left in its workspace
struct CountLayout {
  DnrCarver carve;
  int64_t *cnt, *off;
  void* cub_temp;
  size_t cub_bytes = 0;
  CountLayout(const void* base, int64_t R) : carve(base) {
    cnt = carve.take<int64_t>(3 * (size_t)(R + 1));
    off = carve.take<int64_t>(3 * (size_t)(R + 1));
    const cudaError_t e = cub::DeviceScan::ExclusiveSum(nullptr, cub_bytes, (const int64_t*)nullptr, (int64_t*)nullptr, (int64_t)(R + 1));
    cub_temp = carve.cub_scratch(e, cub_bytes);
  }
};

struct EmitLayout {
  DnrCarver carve;
  int64_t *cube_ids, *tri_start, *vkeys;
  EmitLayout(void* base, int64_t n_cubes, int64_t n_verts) : carve(base) {
    cube_ids = carve.take<int64_t>(n_cubes);
    tri_start = carve.take<int64_t>(n_cubes);
    vkeys = carve.take<int64_t>(n_verts);
  }
};

template <class F>
int mc_count(const F& f, const Geo& g, const CountLayout& L, int64_t* counts_host, cudaStream_t s) {
  const int64_t R = (int64_t)g.X * g.Y;
  int64_t *cnt = L.cnt, *off = L.off;
  mc_count_kernel<F><<<dim3(g.Y, g.X), MC_THREADS, 0, s>>>(f, g, cnt, R);
  DNR_CHECK_LAUNCH();
  for (int a = 0; a < 3; ++a) {
    size_t temp = L.cub_bytes;
    DNR_CUDA(cub::DeviceScan::ExclusiveSum(L.cub_temp, temp, cnt + a * (R + 1), off + a * (R + 1), (int64_t)(R + 1), s));
  }
  for (int a = 0; a < 3; ++a)
    DNR_CUDA(cudaMemcpyAsync(counts_host + a, off + a * (R + 1) + R, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  DNR_CUDA(cudaStreamSynchronize(s));  // the one documented host read
  return 0;
}

template <class F>
int mc_emit(const F& f, const Geo& g, const int64_t* off, const int64_t* counts, const EmitLayout& L, float* verts, int32_t* faces,
            float* colors, cudaStream_t s) {
  const int64_t R = (int64_t)g.X * g.Y;
  mc_compact_kernel<F><<<dim3(g.Y, g.X), MC_THREADS, 0, s>>>(f, g, off, R, L.cube_ids, L.tri_start, L.vkeys, verts, colors);
  DNR_CHECK_LAUNCH();
  if (counts[0] > 0) {
    mc_faces_kernel<F><<<(unsigned)((counts[0] + 127) / 128), 128, 0, s>>>(f, g, L.cube_ids, L.tri_start, counts[0],
                                                                          off + 2 * (R + 1), L.vkeys, faces);
    DNR_CHECK_LAUNCH();
  }
  return 0;
}

}  // namespace

extern "C" int dnr_tsdf_integrate(const DnrTsdfGrid* grid, const float* depth, const float* rgb, const uint8_t* mask,
                                  int32_t width, int32_t height, const float* cam_host, float depth_trunc, void* stream) {
  if (!grid || !depth || !rgb || !cam_host || !grid->voxels) return DNR_E_NULL;
  for (int a = 0; a < 3; ++a)
    if (grid->dims[a] <= 0 || grid->dims[a] > MAX_DIM) return DNR_E_SIZE;
  if (!(grid->voxel > 0.f) || !(grid->sdf_trunc > 0.f) || width <= 0 || height <= 0) return DNR_E_SIZE;
  Cam cam;
  cam.fx = cam_host[0];
  cam.fy = cam_host[1];
  cam.cx = cam_host[2];
  cam.cy = cam_host[3];
  for (int r = 0; r < 12; ++r) cam.E[r] = cam_host[4 + r];
  const dim3 blocks((grid->dims[2] + 127) / 128, grid->dims[1], grid->dims[0]);
  tsdf_integrate_kernel<<<blocks, 128, 0, (cudaStream_t)stream>>>(*grid, cam, depth, rgb, mask, width, height, depth_trunc);
  DNR_CHECK_LAUNCH();
  return 0;
}

extern "C" int64_t dnr_mc_count_workspace_bytes(const DnrMcField* field) {
  Geo g;
  const int rc = check_field(field, &g);
  if (rc) return rc;
  return (int64_t)CountLayout(nullptr, (int64_t)g.X * g.Y).carve.total();
}

extern "C" int dnr_mc_count(const DnrMcField* field, void* ws, int64_t ws_bytes, int64_t* counts_host, void* stream) {
  Geo g;
  const int rc = check_field(field, &g);
  if (rc) return rc;
  if (!ws || !counts_host) return DNR_E_NULL;
  const CountLayout L(ws, (int64_t)g.X * g.Y);
  if (const int e = L.carve.check(ws_bytes)) return e;
  cudaStream_t s = (cudaStream_t)stream;
  if (field->tsdf) return mc_count(TsdfField{(const float4*)field->tsdf}, g, L, counts_host, s);
  return mc_count(ScalarField{field->values, field->valid}, g, L, counts_host, s);
}

extern "C" int64_t dnr_mc_emit_workspace_bytes(const int64_t* counts_host) {
  if (!counts_host) return DNR_E_NULL;
  if (counts_host[0] < 0 || counts_host[1] < 0 || counts_host[2] < 0) return DNR_E_SIZE;
  return (int64_t)EmitLayout(nullptr, counts_host[0], counts_host[2]).carve.total();
}

extern "C" int dnr_mc_emit(const DnrMcField* field, const void* count_ws, const int64_t* counts_host, void* ws, int64_t ws_bytes,
                           float* vertices, int32_t* faces, float* colors, void* stream) {
  Geo g;
  const int rc = check_field(field, &g);
  if (rc) return rc;
  if (!count_ws || !counts_host || !ws) return DNR_E_NULL;
  if (counts_host[0] < 0 || counts_host[1] < 0 || counts_host[2] < 0) return DNR_E_SIZE;
  if (counts_host[1] > INT32_MAX || counts_host[2] > INT32_MAX) return DNR_E_OVERFLOW;
  if ((counts_host[1] > 0 && !faces) || (counts_host[2] > 0 && !vertices)) return DNR_E_NULL;
  const EmitLayout L(ws, counts_host[0], counts_host[2]);
  if (const int e = L.carve.check(ws_bytes)) return e;
  const int64_t* off = CountLayout(count_ws, (int64_t)g.X * g.Y).off;
  cudaStream_t s = (cudaStream_t)stream;
  if (field->tsdf) return mc_emit(TsdfField{(const float4*)field->tsdf}, g, off, counts_host, L, vertices, faces, colors, s);
  return mc_emit(ScalarField{field->values, field->valid}, g, off, counts_host, L, vertices, faces, nullptr, s);
}
