// Shared device helpers for libdnr_b200 (sm_90a, H100).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/dnr.h"

#define DNR_TILE 16
#define DNR_ALPHA_MIN (1.0f / 255.0f)
#define DNR_ALPHA_MAX 0.999f
#define DNR_T_STOP 1e-4f
// streaming kernels cap their grid at a few resident CTAs per SM of an H100 SXM
#define DNR_NUM_SMS 132

#define DNR_CHECK_LAUNCH()                         \
  do {                                             \
    cudaError_t e__ = cudaGetLastError();          \
    if (e__ != cudaSuccess) return (int)e__;       \
  } while (0)

#define DNR_CUDA(expr)                             \
  do {                                             \
    cudaError_t e__ = (expr);                      \
    if (e__ != cudaSuccess) return (int)e__;       \
  } while (0)

// Carves a caller-owned workspace into regions, each at the next 256-byte boundary, in the order they are taken.  On a
// null base it only sizes the workspace.  cub's scratch is taken with the status of its size query: when a query fails
// the workspace has no room for cub, so check() makes the entry point refuse to run rather than launch cub without it.
class DnrCarver {
 public:
  explicit DnrCarver(const void* base) : base_((uintptr_t)base) {}
  template <class T>
  T* take(size_t count) {
    T* p = base_ ? (T*)(base_ + off_) : nullptr;
    off_ += (sizeof(T) * count + 255) & ~(size_t)255;
    return p;
  }
  void* cub_scratch(cudaError_t query, size_t bytes) {
    if (err_ == cudaSuccess) err_ = query;
    return take<char>(bytes);
  }
  size_t total() const { return off_; }
  int cub_error() const { return (int)err_; }
  // DNR_E_WORKSPACE when ws_bytes is short of total(), else the first failed cub size query, else 0
  int check(int64_t ws_bytes) const { return (int64_t)off_ > ws_bytes ? DNR_E_WORKSPACE : cub_error(); }

 private:
  uintptr_t base_;
  size_t off_ = 0;
  cudaError_t err_ = cudaSuccess;
};

static inline int dnr_tiles_x(const DnrArgs* a) { return (a->width + DNR_TILE - 1) / DNR_TILE; }
static inline int dnr_tiles_y(const DnrArgs* a) { return (a->height + DNR_TILE - 1) / DNR_TILE; }
// supertiles: the intersection lists are kept per (16 << list_shift)^2-pixel block
static inline int dnr_list_tile(const DnrArgs* a) { return DNR_TILE << a->list_shift; }
static inline int dnr_stiles_x(const DnrArgs* a) { return (a->width + dnr_list_tile(a) - 1) / dnr_list_tile(a); }
static inline int dnr_stiles_y(const DnrArgs* a) { return (a->height + dnr_list_tile(a) - 1) / dnr_list_tile(a); }

// Tile box of a projected Gaussian: tile_min inclusive, tile_max exclusive (gsplat isect_tiles, SURVEY A3).
// Shared by the count (project_fwd) and emit (bin_sort) kernels so both see the same integers.
__device__ __forceinline__ void dnr_tile_box(float mx, float my, int radius, int tiles_x, int tiles_y,
                                             int& x0, int& y0, int& x1, int& y1) {
  const float r = (float)radius * (1.0f / DNR_TILE);
  const float tcx = mx * (1.0f / DNR_TILE);
  const float tcy = my * (1.0f / DNR_TILE);
  // (uint32_t)floor(negative) saturates to 0 on the GPU
  x0 = min(max((int)floorf(tcx - r), 0), tiles_x);
  y0 = min(max((int)floorf(tcy - r), 0), tiles_y);
  x1 = min(max((int)ceilf(tcx + r), 0), tiles_x);
  y1 = min(max((int)ceilf(tcy + r), 0), tiles_y);
}

// log2-domain exponent of a splat at offset (dx,dy): records hold a' = -0.5*log2(e)*A, b' = -log2(e)*B,
// c' = -0.5*log2(e)*C, so alpha = opac * 2^power.  Fixed rounding order, shared by the forward and backward
// kernels so that both take the same skip/stop branches for every (pixel, Gaussian) pair.
__device__ __forceinline__ float dnr_power2(float a, float b, float c, float dx, float dy) {
  const float t1 = __fmaf_rn(a, dx, __fmul_rn(b, dy));
  const float t2 = __fmul_rn(c, dy);
  return __fmaf_rn(dx, t1, __fmul_rn(dy, t2));
}
__device__ __forceinline__ float dnr_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
#define DNR_LOG2E 1.4426950408889634f
#define DNR_LN2 0.6931471805599453f
#define DNR_CULL_MARGIN 0.1f /* in sigma units: a tile is dropped only if alpha_max < e^-0.1 / 255 */

// ---- mbarrier / bulk-copy (TMA, 1-D) primitives -------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// global -> shared bulk async copy (SASS: UBLKCP), completes `bytes` on the mbarrier's tx-count.
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ---- two fp32 lanes per value: the two pixels a raster thread owns ---------------------------------------------------
// Plain scalar IEEE fp32 operations with explicit rounding (no contraction), so the forward and backward kernels take
// the same branches for every (pixel, Gaussian) pair.  A scalar operand is written v2(s) (broadcast).
struct V2 { float x, y; };

__device__ __forceinline__ V2 v2(float a, float b) { return V2{a, b}; }
__device__ __forceinline__ V2 v2(float a) { return V2{a, a}; }
__device__ __forceinline__ float lo(const V2& a) { return a.x; }
__device__ __forceinline__ float hi(const V2& a) { return a.y; }
__device__ __forceinline__ V2 fma2(const V2& a, const V2& b, const V2& c) {
  return V2{__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)};
}
__device__ __forceinline__ V2 mul2(const V2& a, const V2& b) { return V2{__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)}; }
__device__ __forceinline__ V2 add2(const V2& a, const V2& b) { return V2{__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)}; }
__device__ __forceinline__ V2 sub2(const V2& a, const V2& b) { return V2{__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)}; }
// dnr_power2 for two pixels that share dx (same column): identical roundings per half.
__device__ __forceinline__ V2 dnr_power2x2(float a, float b, float c, float dx, const V2& dy) {
  const V2 t1 = fma2(v2(a), v2(dx), mul2(v2(b), dy));
  const V2 t2 = mul2(v2(c), dy);
  return fma2(v2(dx), t1, mul2(dy, t2));
}

// Does tile (tx, ty) belong to the splat's gsplat tile box (dnr_tile_box of its 3-sigma radius, same float operations)?
// gsplat composites a splat only in the tiles of that box — also where a pixel just outside it would still pass the
// alpha test — so a 16x16 tile that walks a coarser supertile list has to apply the box itself to stay bit-identical.
__device__ __forceinline__ bool dnr_in_tile_box(const float4& q0, const float4& q1, int tx, int ty) {
  const float r = q1.w * (1.0f / DNR_TILE), tcx = q0.x * (1.0f / DNR_TILE), tcy = q0.y * (1.0f / DNR_TILE);
  const float fx = (float)tx, fy = (float)ty;
  return fx >= floorf(tcx - r) && fx < ceilf(tcx + r) && fy >= floorf(tcy - r) && fy < ceilf(tcy + r);
}

// Can the splat (record head q0 = {x, y, a', b'}, q1 = {c', opac, nthr, radius}) reach alpha >= 1/255 at any pixel centre of
// the rectangle [cx0, cx1] x [cy0, cy1]?  The log2-domain exponent p(dx,dy) = a' dx^2 + b' dx dy + c' dy^2 is concave
// with its maximum 0 at the centre, so its maximum over the rectangle is 0 when the centre lies inside and otherwise
// sits on one of the four edges, where it is a 1-D parabola.  Conservative: slack on the threshold, and anything
// degenerate (NaN, non-negative a' or c') is kept.  Dropped entries would be skipped by every pixel of the tile
// anyway (alpha < 1/255 everywhere), so the images do not depend on this test.
#define DNR_TILE_HIT_SLACK 0.05f
__device__ __forceinline__ bool dnr_tile_hit(const float4& q0, const float4& q1, float cx0, float cx1, float cy0, float cy1) {
  const float a = q0.z, b = q0.w, c = q1.x;
  const float d0 = q0.x - cx1, d1 = q0.x - cx0;  // dx = X - px over the rectangle: [d0, d1]
  const float e0 = q0.y - cy1, e1 = q0.y - cy0;
  if (d0 <= 0.f && d1 >= 0.f && e0 <= 0.f && e1 >= 0.f) return true;
  if (!(a < 0.f) || !(c < 0.f)) return true;
  const float hb_c = -0.5f * b / c, hb_a = -0.5f * b / a;  // argmax of the parabola along e for fixed d is hb_c * d, ...
  float best;
  {
    const float e = fminf(fmaxf(hb_c * d0, e0), e1);
    best = dnr_power2(a, b, c, d0, e);
  }
  {
    const float e = fminf(fmaxf(hb_c * d1, e0), e1);
    best = fmaxf(best, dnr_power2(a, b, c, d1, e));
  }
  {
    const float d = fminf(fmaxf(hb_a * e0, d0), d1);
    best = fmaxf(best, dnr_power2(a, b, c, d, e0));
  }
  {
    const float d = fminf(fmaxf(hb_a * e1, d0), d1);
    best = fmaxf(best, dnr_power2(a, b, c, d, e1));
  }
  return !(best < q1.z - DNR_TILE_HIT_SLACK);
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
