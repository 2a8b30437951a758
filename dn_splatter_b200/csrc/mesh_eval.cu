// Mesh evaluation on the device (Python surface: dn_splatter_b200.mesh_eval): the depth rendering and the per-vertex
// visibility counts of the reference's mesh culling (/root/reference/dn_splatter/eval/eval_mesh_vis_cull.py:68-172).
//
// dnr_mesh_depth: camera-space z of the nearest triangle hit by the ray through every pixel centre (i + 0.5, j + 0.5),
// no back-face culling, hits outside [near, far] ignored, 0 where nothing is hit.  Per view, three passes:
//   box     one thread per face: camera-space vertices (fp64), the triangle clipped against the near plane only to bound
//           its pixel box; the box's pixel count is cut into work items of at most PIX_PER_ITEM pixels.
//   scan    cub inclusive scan of the per-face item counts.
//   raster  a fixed grid strides over the items (the total is read on the device, no host synchronisation); an item finds
//           its face by binary search in the scan and tests its pixels by exact ray-triangle intersection.  A full-screen
//           wall triangle is thousands of items, so it does not serialise on one thread.
// Watertightness: the edge function of the ray d against edge (P, Q) is d . (P x Q), evaluated from the endpoints in
// ascending vertex-index order and negated when the face runs the other way; a pixel is inside when its three edge
// functions share a sign (zero counts as either).  Two faces sharing an edge see the same value with opposite signs, so a
// pixel centre on the edge cannot be missed by both.  Hits are resolved with atomicMin on the bits of the positive fp32
// depth (the output buffer doubles as the z-buffer, initialised to 0xFFFFFFFF): the min commutes, so two runs are
// bit-identical.
//
// dnr_mesh_visibility: one thread per point, looping over a chunk of views: the obs / invalid counts of cull_from_one_pose
// and get_grid_culling_pattern, projection in fp64 with the reference's operation order (the file is built with
// -fmad=false), so the counts equal the fp64 numpy restatement in oracle/mesh_eval_ref.py.
#include <cub/cub.cuh>

#include "common.cuh"

namespace {

constexpr int PIX_PER_ITEM = 256;
constexpr int BOX_THREADS = 256;
constexpr int RASTER_THREADS = 256;
constexpr int VIS_THREADS = 128;

// Workspace of dnr_mesh_depth.  tests/test_gpu_mesh_eval_kernels.py reads the last view's boxes, counts and scan back
// from it at these offsets (int4 boxes at 0, then the int64 arrays at 256-B boundaries): change both together.
// Workspace of dnr_mesh_depth.  tests/test_gpu_mesh_eval_kernels.py reads the last view's boxes, counts and scan back
// from it at these offsets (int4 boxes at 0, then the int64 arrays at 256-B boundaries): change both together.
struct DepthLayout {
  DnrCarver carve;
  int4* boxes;
  int64_t *counts, *scan;
  void* cub_temp;
  size_t cub_bytes = 0;
  DepthLayout(void* base, int64_t n_faces) : carve(base) {
    boxes = carve.take<int4>(n_faces);
    counts = carve.take<int64_t>(n_faces);
    scan = carve.take<int64_t>(n_faces);
    const cudaError_t e = cub::DeviceScan::InclusiveSum(nullptr, cub_bytes, (const int64_t*)nullptr, (int64_t*)nullptr, n_faces);
    cub_temp = carve.cub_scratch(e, cub_bytes);
  }
};

__device__ __forceinline__ double3 to_camera(const float* __restrict__ cam, const float* __restrict__ verts, int v) {
  const double x = verts[3 * v], y = verts[3 * v + 1], z = verts[3 * v + 2];
  const float* E = cam + 4;
  return make_double3((double)E[0] * x + (double)E[1] * y + (double)E[2] * z + (double)E[3],
                      (double)E[4] * x + (double)E[5] * y + (double)E[6] * z + (double)E[7],
                      (double)E[8] * x + (double)E[9] * y + (double)E[10] * z + (double)E[11]);
}

__device__ __forceinline__ double3 cross(double3 a, double3 b) {
  return make_double3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}
__device__ __forceinline__ double3 sub(double3 a, double3 b) { return make_double3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ double dot(double3 a, double3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

struct Tri {
  double3 e[3];  // oriented edge planes: inside when d . e[k] share a sign
  double3 n;     // (B - A) x (C - A)
  double num;    // n . A: the hit at ray d lies at z = num / (n . d)
};

// false for faces with an index out of range or zero area
__device__ bool tri_setup(const float* __restrict__ cam, const float* __restrict__ verts, int n_verts, const int32_t* __restrict__ face,
                          double3 P[3], Tri& t) {
  int id[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    id[k] = face[k];
    if (id[k] < 0 || id[k] >= n_verts) return false;
    P[k] = to_camera(cam, verts, id[k]);
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int a = k, b = (k + 1) % 3;
    if (id[a] <= id[b]) {
      t.e[k] = cross(P[a], P[b]);
    } else {
      const double3 c = cross(P[b], P[a]);
      t.e[k] = make_double3(-c.x, -c.y, -c.z);
    }
  }
  t.n = cross(sub(P[1], P[0]), sub(P[2], P[0]));
  t.num = dot(t.n, P[0]);
  return t.n.x != 0.0 || t.n.y != 0.0 || t.n.z != 0.0;
}

__global__ void __launch_bounds__(BOX_THREADS) depth_box_kernel(const float* __restrict__ verts, int n_verts, const int32_t* __restrict__ faces,
                                                                int64_t n_faces, const float* __restrict__ cam, int W, int H, float near,
                                                                float far, int4* __restrict__ boxes, int64_t* __restrict__ counts) {
  const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n_faces) return;
  double3 P[3];
  Tri t;
  int64_t items = 0;
  int4 box = make_int4(0, -1, 0, -1);
  const bool ok = tri_setup(cam, verts, n_verts, faces + 3 * f, P, t);
  const bool all_near = P[0].z < near && P[1].z < near && P[2].z < near;
  const bool all_far = P[0].z > far && P[1].z > far && P[2].z > far;
  if (ok && !all_near && !all_far) {
    const double fx = cam[0], fy = cam[1], cx = cam[2], cy = cam[3];
    double x0 = INFINITY, x1 = -INFINITY, y0 = INFINITY, y1 = -INFINITY;
    auto add = [&](double X, double Y, double Z) {
      const double u = fx * X / Z + cx, v = fy * Y / Z + cy;
      x0 = fmin(x0, u); x1 = fmax(x1, u);
      y0 = fmin(y0, v); y1 = fmax(y1, v);
    };
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double3 a = P[k], b = P[(k + 1) % 3];
      if (a.z >= near) add(a.x, a.y, a.z);
      if ((a.z < near) != (b.z < near)) {  // the edge crosses the near plane
        const double s = ((double)near - a.z) / (b.z - a.z);
        add(a.x + s * (b.x - a.x), a.y + s * (b.y - a.y), (double)near);
      }
    }
    // pixel i is sampled at i + 0.5; one pixel of margin, the exact test decides
    const double lo_x = fmax(ceil(x0 - 0.5) - 1.0, 0.0), hi_x = fmin(floor(x1 - 0.5) + 1.0, (double)(W - 1));
    const double lo_y = fmax(ceil(y0 - 0.5) - 1.0, 0.0), hi_y = fmin(floor(y1 - 0.5) + 1.0, (double)(H - 1));
    if (lo_x <= hi_x && lo_y <= hi_y) {
      box = make_int4((int)lo_x, (int)hi_x, (int)lo_y, (int)hi_y);
      const int64_t area = (int64_t)(box.y - box.x + 1) * (box.w - box.z + 1);
      items = (area + PIX_PER_ITEM - 1) / PIX_PER_ITEM;
    }
  }
  boxes[f] = box;
  counts[f] = items;
}

__global__ void __launch_bounds__(RASTER_THREADS) depth_raster_kernel(const float* __restrict__ verts, int n_verts,
                                                                      const int32_t* __restrict__ faces, int64_t n_faces,
                                                                      const float* __restrict__ cam, int W, float near, float far,
                                                                      const int4* __restrict__ boxes, const int64_t* __restrict__ scan,
                                                                      uint32_t* __restrict__ zbuf) {
  const int64_t total = scan[n_faces - 1];
  const double fx = cam[0], fy = cam[1], cx = cam[2], cy = cam[3];
  for (int64_t item = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; item < total; item += (int64_t)gridDim.x * blockDim.x) {
    int64_t lo = 0, hi = n_faces - 1;  // first face whose inclusive scan exceeds item
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (scan[mid] > item) hi = mid; else lo = mid + 1;
    }
    const int64_t f = lo;
    const int64_t first = (f == 0 ? 0 : scan[f - 1]);
    const int4 box = boxes[f];
    double3 P[3];
    Tri t;
    tri_setup(cam, verts, n_verts, faces + 3 * f, P, t);  // succeeded in the box pass, or the face has no items
    const int bw = box.y - box.x + 1;
    const int64_t area = (int64_t)bw * (box.w - box.z + 1);
    const int64_t p0 = (item - first) * PIX_PER_ITEM;
    const int64_t p1 = min(p0 + PIX_PER_ITEM, area);
    for (int64_t p = p0; p < p1; ++p) {
      const int i = box.x + (int)(p % bw), j = box.z + (int)(p / bw);
      const double dx = ((double)i + 0.5 - cx) / fx, dy = ((double)j + 0.5 - cy) / fy;
      const double e0 = dx * t.e[0].x + dy * t.e[0].y + t.e[0].z;
      const double e1 = dx * t.e[1].x + dy * t.e[1].y + t.e[1].z;
      const double e2 = dx * t.e[2].x + dy * t.e[2].y + t.e[2].z;
      const bool inside = (e0 >= 0.0 && e1 >= 0.0 && e2 >= 0.0) || (e0 <= 0.0 && e1 <= 0.0 && e2 <= 0.0);
      if (!inside) continue;
      const double den = dx * t.n.x + dy * t.n.y + t.n.z;
      if (den == 0.0) continue;
      const double z = t.num / den;
      if (!(z >= (double)near && z <= (double)far)) continue;
      atomicMin(zbuf + (int64_t)j * W + i, __float_as_uint((float)z));
    }
  }
}

__global__ void depth_resolve_kernel(uint32_t* __restrict__ zbuf, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    if (zbuf[i] == 0xFFFFFFFFu) zbuf[i] = 0u;  // the bits of +0.0f
  }
}

__global__ void __launch_bounds__(VIS_THREADS) visibility_kernel(const double* __restrict__ pts, int64_t n, const double* __restrict__ cams,
                                                                 const float* __restrict__ rendered, const float* __restrict__ gt,
                                                                 int n_views, int W, int H, float eps, int32_t* __restrict__ obs,
                                                                 int32_t* __restrict__ invalid) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
  const double Wm = (double)(W - 1), Hm = (double)(H - 1);
  int32_t n_obs = 0, n_inv = 0;
  for (int v = 0; v < n_views; ++v) {
    const double* c = cams + 16 * v;
    const double* E = c + 4;
    // rotation @ p + t, then K @ (X, Y, Z): ((fx X + 0 Y) + cx Z), ((0 X + fy Y) + cy Z), Z
    const double X = E[0] * x + E[1] * y + E[2] * z + E[3];
    const double Y = E[4] * x + E[5] * y + E[6] * z + E[7];
    const double Z = E[8] * x + E[9] * y + E[10] * z + E[11];
    const double pz = Z + 1e-8;
    const double px = (c[0] * X + c[2] * Z) / pz;
    const double py = (c[1] * Y + c[3] * Z) / pz;
    if (!(0.0 <= px && px <= Wm && 0.0 <= py && py <= Hm && pz > 0.0)) continue;
    const int64_t pix = (int64_t)v * W * H + (int64_t)(int)py * W + (int)px;  // in the frustum: clip is a no-op, astype truncates
    if (rendered == nullptr || pz < (double)(rendered[pix] + eps)) ++n_obs;
    if (gt != nullptr && gt[pix] <= 0.f) ++n_inv;
  }
  obs[i] += n_obs;
  if (invalid != nullptr) invalid[i] += n_inv;
}

}  // namespace

extern "C" int64_t dnr_mesh_depth_workspace_bytes(int64_t n_faces) {
  if (n_faces <= 0) return DNR_E_SIZE;
  return (int64_t)DepthLayout(nullptr, n_faces).carve.total();
}

extern "C" int dnr_mesh_depth(const float* vertices, int32_t n_vertices, const int32_t* faces, int64_t n_faces, const float* cams,
                              int32_t n_views, int32_t width, int32_t height, float near, float far, void* ws, int64_t ws_bytes,
                              float* depth, void* stream) {
  if (!vertices || !faces || !cams || !ws || !depth) return DNR_E_NULL;
  if (n_vertices <= 0 || n_faces <= 0 || n_views <= 0 || width <= 0 || height <= 0) return DNR_E_SIZE;
  if (!(near > 0.f) || !(far >= near)) return DNR_E_OPTION;
  const DepthLayout L(ws, n_faces);
  if (const int e = L.carve.check(ws_bytes)) return e;
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t pixels = (int64_t)width * height;
  uint32_t* zbuf = reinterpret_cast<uint32_t*>(depth);
  DNR_CUDA(cudaMemsetAsync(zbuf, 0xFF, sizeof(uint32_t) * (size_t)(pixels * n_views), s));
  const int64_t box_blocks = (n_faces + BOX_THREADS - 1) / BOX_THREADS;
  if (box_blocks > INT32_MAX) return DNR_E_SIZE;
  for (int v = 0; v < n_views; ++v) {
    const float* cam = cams + 16 * (int64_t)v;
    depth_box_kernel<<<(unsigned)box_blocks, BOX_THREADS, 0, s>>>(vertices, n_vertices, faces, n_faces, cam, width, height, near, far,
                                                                  L.boxes, L.counts);
    DNR_CHECK_LAUNCH();
    size_t temp = L.cub_bytes;
    DNR_CUDA(cub::DeviceScan::InclusiveSum(L.cub_temp, temp, L.counts, L.scan, n_faces, s));
    depth_raster_kernel<<<DNR_NUM_SMS * 16, RASTER_THREADS, 0, s>>>(vertices, n_vertices, faces, n_faces, cam, width, near, far,
                                                                    L.boxes, L.scan, zbuf + pixels * v);
    DNR_CHECK_LAUNCH();
  }
  depth_resolve_kernel<<<DNR_NUM_SMS * 8, 256, 0, s>>>(zbuf, pixels * n_views);
  DNR_CHECK_LAUNCH();
  return 0;
}

extern "C" int dnr_mesh_visibility(const double* points, int64_t n_points, const double* cams, const float* rendered, const float* gt,
                                   int32_t n_views, int32_t width, int32_t height, float eps, int32_t* obs, int32_t* invalid,
                                   void* stream) {
  if (!points || !cams || !obs || (gt != nullptr && invalid == nullptr)) return DNR_E_NULL;
  if (n_points <= 0 || n_views <= 0 || width <= 0 || height <= 0) return DNR_E_SIZE;
  const int64_t blocks = (n_points + VIS_THREADS - 1) / VIS_THREADS;
  if (blocks > INT32_MAX) return DNR_E_SIZE;
  visibility_kernel<<<(unsigned)blocks, VIS_THREADS, 0, (cudaStream_t)stream>>>(points, n_points, cams, rendered, gt, n_views, width,
                                                                                height, eps, obs, invalid);
  DNR_CHECK_LAUNCH();
  return 0;
}
