// Per-tile front-to-back alpha compositing of RGB + expected depth + per-Gaussian normal in ONE pass,
// forward and backward, with the loss gradients evaluated in the backward kernel's prologue.
//
// Replaces (reference /root/reference/dn_splatter/dn_model.py):
//   :495-516  gsplat rasterize_to_pixels fwd (RGB+ED)  and its autograd backward      [EXT gsplat 1.0.0]
//   :564-575  gsplat legacy rasterize_gaussians on normals (white background) + bwd   [EXT]
//   :526-537  rgb = clamp(render + (1-alpha) bg), depth = where(alpha>0, ED, max)     (max: finalize)
//   :577-578  normal = (n/|n| + 1)/2
// and, in dnr_raster_bwd's prologue (DNR_LOSS_FUSED_BWD), the backward of
//   dn_splatter/regularization_strategy.py:158-193, dn_splatter/losses.py:197-224,285-295 (EdgeAwareLogL1 / LogL1 /
//   L1 / MSE depth term, normal L1 + TV) and of the parent's photometric L1 (dn_model.py:624-628).
// The two reference passes share alpha/T exactly (same means2d, conics, opacities, order), so one
// compositing loop with 7 channels reproduces both; only the gradient routing differs (the normal pass
// sees detached xys: its alpha-gradient reaches conics/opacity but not means2d — quirk B3).
//
// Lists and data movement.  The sorted intersection lists are kept per SUPERTILE of (16 << list_shift)^2 pixels (5-14x
// fewer pairs to emit and sort than per-tile lists).  A CTA owns one 16x16 tile and walks its supertile's list in
// chunks of 128 entries: the packed 64 B records are gathered by id straight into shared memory by per-thread 1-D bulk
// async copies (cp.async.bulk -> UBLKCP, TMA engine) completing on an mbarrier, double-buffered; one thread per entry
// then tests whether the splat can reach the tile at all (dnr_tile_hit) and the survivors are ballot-compacted into an
// index list that the compositing loop walks.  Only the chunks a tile consumes before all of its pixels saturate are
// ever fetched.  `last_ids` are positions in the supertile list, so the backward replays exactly the same entries.
//
// Arithmetic.  A thread owns 2 (forward) / 4 (backward) pixels of one column and evaluates them as pairs of scalar fp32
// operations with explicit rounding (V2 in common.cuh).  The backward's per-record warp reduction of its 16 gradient
// values goes through a padded shared-memory transpose (4 STS.128 + 16 LDS.32 per lane, no SEL: fewer instructions than
// a 16-SHFL / 30-SEL shuffle reduction), and is paid once per 128 pixels.
//
// Tests.  The forward is pinned per pixel (every output, last_ids, clamp_mask, depth_max) to the fp64 compositor of
// oracle/raster_ref.py by tests/test_gpu_raster_forward.py; the backward per Gaussian (every grad_records slot, the
// touched flags) to the fp64 backward of the same oracle by tests/test_gpu_raster_backward.py, and end to end by
// tests/test_gpu_backward_edges.py.
#include "common.cuh"
#include "loss_common.cuh"

namespace {

constexpr int CH = 128;   // list entries per chunk
constexpr int STAGES = 2;
constexpr int FWD_THREADS = 128;  // 4 warps x (8x8 pixels), 2 pixels per thread
constexpr int BWD_THREADS = 64;   // 2 warps x (16x8 pixels), 4 pixels per thread
constexpr int RED_STRIDE = 20;    // floats per lane row of the reduction scratch (80 B: 16 B aligned, conflict-free)
constexpr int RED_WARP_FLOATS = 32 * RED_STRIDE + 16;  // per-warp scratch (the upper half-warp's rows are shifted by 16)

__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// One chunk of the list: entry t of the chunk lives at list position `first + t * step` (step = +1 forward, -1 backward).
template <int REC, int NT>
__device__ __forceinline__ void issue_chunk(const float* __restrict__ records, const int32_t* __restrict__ ids, int first,
                                            int step, int n_c, float* stage_smem, int* ids_smem, uint64_t* bar, int tid) {
  if (tid == 0) mbar_arrive_expect_tx(bar, (uint32_t)(n_c * REC * 4));
  for (int t = tid; t < n_c; t += NT) {
    const int g = ids[first + t * step];
    if (ids_smem) ids_smem[t] = g;
    bulk_g2s(stage_smem + t * REC, records + (size_t)g * REC, REC * 4, bar);
  }
}

// Tile filter over a landed chunk: survivors' chunk slots, in list order, into sidx[0..total).  Called by all NT
// threads; contains two __syncthreads().
template <int REC, int NT>
__device__ __forceinline__ int filter_chunk(const float* stage_smem, int n_c, int tile_x, int tile_y, unsigned char* sidx,
                                            int* scnt, int tid) {
  const float cx0 = (float)(tile_x * DNR_TILE) + 0.5f, cy0 = (float)(tile_y * DNR_TILE) + 0.5f;
  const float cx1 = cx0 + (float)(DNR_TILE - 1), cy1 = cy0 + (float)(DNR_TILE - 1);
  constexpr int PER = CH / NT;  // entries per thread
  constexpr int NW = NT / 32;
  const int lane = tid & 31, warp = tid >> 5;
  const float4* r4 = reinterpret_cast<const float4*>(stage_smem);
  unsigned m[PER];
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    // warp w tests entries [w*32*PER, (w+1)*32*PER), 32 at a time: ascending slot order within and across warps
    const int t = (warp * PER + k) * 32 + lane;
    bool hit = false;
    if (t < n_c) {
      const float4 q0 = r4[t * (REC / 4) + 0], q1 = r4[t * (REC / 4) + 1];
      hit = dnr_in_tile_box(q0, q1, tile_x, tile_y) && dnr_tile_hit(q0, q1, cx0, cx1, cy0, cy1);
    }
    m[k] = __ballot_sync(0xffffffffu, hit);
  }
  if (lane == 0) {
    int c = 0;
#pragma unroll
    for (int k = 0; k < PER; ++k) c += __popc(m[k]);
    scnt[warp] = c;
  }
  __syncthreads();
  int base = 0, total = 0;
#pragma unroll
  for (int w = 0; w < NW; ++w) {
    const int c = scnt[w];
    if (w < warp) base += c;
    total += c;
  }
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    if (m[k] & (1u << lane)) sidx[base + __popc(m[k] & ((1u << lane) - 1u))] = (unsigned char)((warp * PER + k) * 32 + lane);
    base += __popc(m[k]);
  }
  __syncthreads();
  return total;
}

// ------------------------------------------------------------------------------------------------ forward
template <bool NORMALS>
__global__ void __launch_bounds__(FWD_THREADS) raster_fwd_kernel(const DnrArgs a, int stiles_x) {
  constexpr int REC = NORMALS ? DNR_REC_FLOATS_N : DNR_REC_FLOATS;
  constexpr int RQ = REC / 4;
  __shared__ __align__(128) float recs[STAGES][CH * REC];
  __shared__ __align__(8) uint64_t bars[STAGES];
  __shared__ __align__(4) unsigned char sidx[CH];
  __shared__ int scnt[FWD_THREADS / 32];
  __shared__ float red_max[FWD_THREADS / 32];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int shift = a.list_shift;
  const int stile = (blockIdx.y >> shift) * stiles_x + (blockIdx.x >> shift);
  // warp -> 8x8 pixel patch, lane -> column (lane & 7), rows (lane >> 3) and (lane >> 3) + 4
  const int lx = ((warp & 1) << 3) + (lane & 7);
  const int ly = ((warp >> 1) << 3) + (lane >> 3);
  const int j = blockIdx.x * DNR_TILE + lx, i0 = blockIdx.y * DNR_TILE + ly, i1 = i0 + 4;
  const bool in0 = (i0 < a.height) && (j < a.width), in1 = (i1 < a.height) && (j < a.width);
  const float px = (float)j + 0.5f;
  const V2 npy = v2(-((float)i0 + 0.5f), -((float)i1 + 0.5f));
  const int start = a.tile_offsets[stile], end = a.tile_offsets[stile + 1];
  const int n = end - start;
  const int nchunks = (n + CH - 1) / CH;

  if (tid == 0) {
    mbar_init(&bars[0], 1);
    mbar_init(&bars[1], 1);
    mbar_fence_init();
  }
  __syncthreads();

  const V2 zero = v2(0.f);
  V2 T = v2(1.0f);
  V2 C0 = zero, C1 = zero, C2 = zero, D = zero, N0 = zero, N1 = zero, N2 = zero;
  int last0 = 0, last1 = 0;
  bool done0 = !in0, done1 = !in1;
  unsigned long long walked = 0, kept = 0;

  int issued = 0, consumed = 0;
  if (nchunks > 0) {
    issue_chunk<REC, FWD_THREADS>(a.records, a.flatten_ids, start, 1, min(CH, n), recs[0], nullptr, &bars[0], tid);
    issued = 1;
  }
  for (int c = 0; c < nchunks; ++c) {
    const int stage = c & 1;
    if (c + 1 < nchunks) {  // stage (c+1)&1 was released by the barrier that closed iteration c-1
      issue_chunk<REC, FWD_THREADS>(a.records, a.flatten_ids, start + (c + 1) * CH, 1, min(CH, n - (c + 1) * CH),
                                    recs[stage ^ 1], nullptr, &bars[stage ^ 1], tid);
      issued = c + 2;
    }
    mbar_wait(&bars[stage], (uint32_t)((c >> 1) & 1));
    consumed = c + 1;
    const int n_c = min(CH, n - c * CH);
    const int total = filter_chunk<REC, FWD_THREADS>(recs[stage], n_c, blockIdx.x, blockIdx.y, sidx, scnt, tid);
    walked += n_c; kept += total;
    const float4* r4 = reinterpret_cast<const float4*>(recs[stage]);
    const int base = start + c * CH;
    // Warp-uniform loop: every lane walks the survivors in lockstep (predicated), so the warp issues each record once.
    for (int s0 = 0; s0 < total; s0 += 4) {
      if (__all_sync(0xffffffffu, done0 && done1)) break;
      const unsigned slots = *reinterpret_cast<const unsigned*>(sidx + s0);  // 4 survivor slots in one LDS
      const int s1 = min(s0 + 4, total);
#pragma unroll 4
      for (int s = s0; s < s1; ++s) {
        const int t = (slots >> (8 * (s - s0))) & 0xff;
        const float4 q0 = r4[t * RQ + 0];  // x, y, a', b'
        const float4 q1 = r4[t * RQ + 1];  // c', opacity, -log2(255 opacity) - slack, -
        const float dx = q0.x - px;
        const V2 dy = add2(v2(q0.y), npy);
        const V2 pw = dnr_power2x2(q0.z, q0.w, q1.x, dx, dy);  // = -sigma * log2(e)
        const float pw0 = lo(pw), pw1 = hi(pw);
        int ok0 = !done0 & !(pw0 > 0.f) & !(pw0 < q1.z);  // else: sigma < 0, or alpha certainly < 1/255
        int ok1 = !done1 & !(pw1 > 0.f) & !(pw1 < q1.z);
        if (ok0 | ok1) {
          const V2 vis = v2(dnr_ex2(pw0), dnr_ex2(pw1));
          const V2 araw = mul2(v2(q1.y), vis);
          const float a0 = fminf(DNR_ALPHA_MAX, lo(araw)), a1 = fminf(DNR_ALPHA_MAX, hi(araw));
          ok0 &= !(a0 < DNR_ALPHA_MIN);
          ok1 &= !(a1 < DNR_ALPHA_MIN);
          const V2 nT = mul2(T, sub2(v2(1.0f), v2(a0, a1)));
          const int stop0 = ok0 & (lo(nT) <= DNR_T_STOP), stop1 = ok1 & (hi(nT) <= DNR_T_STOP);
          done0 = done0 | (stop0 != 0);
          done1 = done1 | (stop1 != 0);
          ok0 &= !stop0;
          ok1 &= !stop1;
          if (ok0 | ok1) {
            // masked alpha: a pixel that skips this splat composites it with alpha = 0 (T and the sums stay bit-exact)
            const V2 al = v2(ok0 ? a0 : 0.f, ok1 ? a1 : 0.f);
            const V2 w = mul2(al, T);
            const float4 q2 = r4[t * RQ + 2];  // r, g, b, depth
            C0 = fma2(v2(q2.x), w, C0);
            C1 = fma2(v2(q2.y), w, C1);
            C2 = fma2(v2(q2.z), w, C2);
            D = fma2(v2(q2.w), w, D);
            if (NORMALS) {
              const float4 q3 = r4[t * RQ + 3];  // camera-space normal
              N0 = fma2(v2(q3.x), w, N0);
              N1 = fma2(v2(q3.y), w, N1);
              N2 = fma2(v2(q3.z), w, N2);
            }
            T = v2(ok0 ? lo(nT) : lo(T), ok1 ? hi(nT) : hi(T));
            last0 = ok0 ? base + t : last0;
            last1 = ok1 ? base + t : last1;
          }
        }
      }
    }
    if (__syncthreads_count(done0 && done1) == FWD_THREADS) break;
  }
  // never leave the CTA with a bulk copy still in flight into its shared memory
  if (issued > consumed) mbar_wait(&bars[(issued - 1) & 1], (uint32_t)(((issued - 1) >> 1) & 1));
  if (a.stats != nullptr && tid == 0) {
    atomicAdd((unsigned long long*)a.stats + 0, walked);
    atomicAdd((unsigned long long*)a.stats + 1, kept);
  }

  float ed_for_max = 0.f;
#pragma unroll
  for (int p = 0; p < 2; ++p) {
    const bool inside = p ? in1 : in0;
    if (!inside) continue;
    const int pix = (p ? i1 : i0) * a.width + j;
    const float Tp = p ? hi(T) : lo(T);
    const float c0 = p ? hi(C0) : lo(C0), c1 = p ? hi(C1) : lo(C1), c2 = p ? hi(C2) : lo(C2), d = p ? hi(D) : lo(D);
    const float alpha = 1.0f - Tp;
    const float om = 1.0f - alpha;
    const float pre[3] = {c0 + om * a.background[0], c1 + om * a.background[1], c2 + om * a.background[2]};
    uint8_t mask = 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      if (pre[k] >= 0.f && pre[k] <= 1.f) mask |= (uint8_t)(1u << k);
      a.out_rgb[pix * 3 + k] = fminf(fmaxf(pre[k], 0.f), 1.f);
    }
    a.clamp_mask[pix] = mask;
    const float ed = d / fmaxf(alpha, 1e-10f);
    a.out_depth[pix] = ed;
    a.out_alpha[pix] = alpha;
    a.last_ids[pix] = p ? last1 : last0;
    ed_for_max = fmaxf(ed_for_max, ed);
    if (NORMALS) {
      const float n0 = (p ? hi(N0) : lo(N0)) + Tp, n1 = (p ? hi(N1) : lo(N1)) + Tp, n2 = (p ? hi(N2) : lo(N2)) + Tp;  // white bg (B1)
      const float nn = sqrtf(__fmaf_rn(n2, n2, __fmaf_rn(n1, n1, __fmul_rn(n0, n0))));  // explicit: identical in every instantiation
      a.normal_norm[pix] = nn;
      a.out_normal[pix * 3 + 0] = (n0 / nn + 1.0f) * 0.5f;
      a.out_normal[pix * 3 + 1] = (n1 / nn + 1.0f) * 0.5f;
      a.out_normal[pix * 3 + 2] = (n2 / nn + 1.0f) * 0.5f;
    }
  }
  // global max of the expected depth (dn_model.py:536: depth_im.detach().max())
  const float wm = warp_max(ed_for_max);
  if (lane == 0) red_max[warp] = wm;
  __syncthreads();
  if (tid == 0) {
    float m = red_max[0];
#pragma unroll
    for (int w = 1; w < FWD_THREADS / 32; ++w) m = fmaxf(m, red_max[w]);
    if (m > 0.f) atomicMax(a.depth_max, __float_as_int(m));
  }
}

// ------------------------------------------------------------------------------------------------ loss gradients
// d(loss)/d(rgb, depth, normal) at pixel (i, j) of the losses listed in include/dnr.h under DNR_LOSS_FUSED_BWD; the same
// formulas as loss_bwd_kernel / l1_bwd_kernel (csrc/image_ops.cu), which remain the unfused path.  Written for memory-
// level parallelism: a CTA has only 64 threads, so every load is unconditional (neighbour indices are clamped into the
// image: a clamped neighbour is the pixel itself and contributes sgn(0) = 0 to the TV term; the edge weights carry an
// explicit 0/1 factor) and only warp-uniform configuration tests remain as branches — the loads of a pixel issue back
// to back instead of one round trip per `if`.
__device__ __forceinline__ void fused_loss_grads(const DnrArgs& a, int i, int j, float v_rgb[3], float& v_depth, float v_n[3]) {
  const int W = a.width, H = a.height;
  const int p = i * W + j;
  const int jr = min(j + 1, W - 1), jl = max(j - 1, 0), id = min(i + 1, H - 1), iu = max(i - 1, 0);
  const int pr = i * W + jr, pl = i * W + jl, pd = id * W + j, pu = iu * W + j;
  const float vl = a.v_loss ? __ldg(a.v_loss) : 1.0f;
  if (a.v_l1 != nullptr) {
    const float s = __ldg(a.v_l1) / (3.0f * (float)H * (float)W);
    float gt[3], pred[3];
    if (a.loss_flags & DNR_LOSS_IMG_U8) {
      const uint8_t* im = (const uint8_t*)a.gt_image;
#pragma unroll
      for (int c = 0; c < 3; ++c) gt[c] = __fmul_rn((float)__ldg(im + p * 3 + c), 1.0f / 255.0f);
    } else {
#pragma unroll
      for (int c = 0; c < 3; ++c) gt[c] = __ldg((const float*)a.gt_image + p * 3 + c);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) pred[c] = __ldg(a.out_rgb + p * 3 + c);
#pragma unroll
    for (int c = 0; c < 3; ++c) v_rgb[c] += sgnf(pred[c] - gt[c]) * s;
  }
  if (a.depth_loss_type != 0) {
    const float gd = __ldg(a.gt_depth + p), od = __ldg(a.out_depth + p);
    float w = 1.0f / __ldg(a.loss_partials + 1);
    if (a.depth_loss_type == 1) {
      const float wx = edge_weight(a, p, pr), wy = edge_weight(a, p, pd);  // exp(0) = 1 at the clamped border: masked below
      // select, not multiply: a count is 0 when no valid pixel has that neighbour, and 0 / 0 would poison the pixel
      w = (j < W - 1 ? wx / __ldg(a.loss_partials + 1) : 0.f) + (i < H - 1 ? wy / __ldg(a.loss_partials + 3) : 0.f);
    }
    const float e = od - gd;
    float dval;
    if (a.depth_loss_type == 1 || a.depth_loss_type == 2) dval = sgnf(e) / (1.0f + fabsf(e));
    else if (a.depth_loss_type == 3) dval = sgnf(e);
    else dval = 2.0f * e;
    const float scale = vl * (1.0f + a.depth_lambda);  // quirk B6: depth_loss += lambda * depth_loss
    v_depth += (gd > a.depth_tolerance) ? scale * dval * w : 0.f;
  }
  if (a.use_normal_loss) {
    const float inv_l1 = vl / (3.0f * (float)H * (float)W);
    const float inv_tx = (W > 1) ? vl / (3.0f * (float)H * (float)(W - 1)) : 0.f;
    const float inv_ty = (H > 1) ? vl / (3.0f * (float)(H - 1) * (float)W) : 0.f;
    float n[3], nr[3], nl[3], nd[3], nu[3], gn[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      n[c] = __ldg(a.out_normal + p * 3 + c);
      nr[c] = __ldg(a.out_normal + pr * 3 + c);
      nl[c] = __ldg(a.out_normal + pl * 3 + c);
      nd[c] = __ldg(a.out_normal + pd * 3 + c);
      nu[c] = __ldg(a.out_normal + pu * 3 + c);
      gn[c] = gt_normal_at(a, p * 3 + c);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float g = sgnf(n[c] - gn[c]) * inv_l1;
      g += sgnf(n[c] - nr[c]) * inv_tx;   // clamped neighbour == the pixel itself -> sgn(0) = 0
      g -= sgnf(nl[c] - n[c]) * inv_tx;
      g += sgnf(n[c] - nd[c]) * inv_ty;
      g -= sgnf(nu[c] - n[c]) * inv_ty;
      v_n[c] += g;
    }
  }
}

// ------------------------------------------------------------------------------------------------ backward
// 16 per-lane values -> per-value warp totals through a padded shared-memory transpose: no SEL, 4 STS.128 + 16 LDS.32
// per lane.  Lane L returns the total of value index L & 15 (both half-warps hold it).  `scr` is the warp's private
// [32][RED_STRIDE] scratch.
__device__ __forceinline__ float transpose_reduce16(const float (&v)[16], float* scr, int lane) {
  __syncwarp();  // previous reads of the scratch are done
  float4* row = reinterpret_cast<float4*>(scr + lane * RED_STRIDE + (lane >> 4) * 16);
  row[0] = make_float4(v[0], v[1], v[2], v[3]);
  row[1] = make_float4(v[4], v[5], v[6], v[7]);
  row[2] = make_float4(v[8], v[9], v[10], v[11]);
  row[3] = make_float4(v[12], v[13], v[14], v[15]);
  __syncwarp();
  // the rows of the upper half-warp sit 16 floats further: at step r the two half-warps read rows r and 16 + r whose
  // bank offsets differ by 16, so the 32 lanes hit 32 distinct banks, and every offset below is an immediate
  const float* col = scr + (lane & 15) + (lane >> 4) * (16 * RED_STRIDE + 16);
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;  // four chains: the adds do not wait on each other's latency
#pragma unroll
  for (int r = 0; r < 16; r += 4) {
    s0 += col[r * RED_STRIDE];
    s1 += col[(r + 1) * RED_STRIDE];
    s2 += col[(r + 2) * RED_STRIDE];
    s3 += col[(r + 3) * RED_STRIDE];
  }
  const float s = (s0 + s1) + (s2 + s3);
  return s + __shfl_xor_sync(0xffffffffu, s, 16);
}

template <bool NORMALS>
__global__ void __launch_bounds__(BWD_THREADS, 9) raster_bwd_kernel(const DnrArgs a, int stiles_x) {
  constexpr int REC = NORMALS ? DNR_REC_FLOATS_N : DNR_REC_FLOATS;
  constexpr int RQ = REC / 4;
  constexpr int NW = BWD_THREADS / 32;
  __shared__ __align__(128) float recs[STAGES][CH * REC];
  __shared__ int ids_s[STAGES][CH];
  __shared__ __align__(8) uint64_t bars[STAGES];
  __shared__ __align__(4) unsigned char sidx[CH];
  __shared__ int scnt[NW];
  __shared__ int red_last[NW];
  __shared__ __align__(16) float red_scr[NW * RED_WARP_FLOATS];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int shift = a.list_shift;
  const int stile = (blockIdx.y >> shift) * stiles_x + (blockIdx.x >> shift);
  const int start = a.tile_offsets[stile], end = a.tile_offsets[stile + 1];

  // ---- per-pixel state and the gradient of the glue (P1/P3 backward) ----
  // warp -> 16 wide x 8 tall strip; lane -> column lane & 15, rows (lane >> 4) + {0, 2, 4, 6}: pixel pairs A = rows
  // {0, 2}, B = rows {4, 6} of the lane share dx and are evaluated as f32x2 halves
  const int lx = lane & 15;
  const int ly = warp * 8 + (lane >> 4);
  const int j = blockIdx.x * DNR_TILE + lx;
  const float px = (float)j + 0.5f;
  float Tp[4], Scd[4], Sn[4], vC0[4], vC1[4], vC2[4], vD[4], vN0[4], vN1[4], vN2[4];
  int last_id[4];
  int wl = -1;
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    const int i_raw = blockIdx.y * DNR_TILE + ly + 2 * p;
    const bool inside = (i_raw < a.height) && (j < a.width);
    // pixels past the image edge read a valid pixel (clamped) and are masked out at the end: no load hides behind a branch
    const int i = min(i_raw, a.height - 1), jc = min(j, a.width - 1);
    const int pix = i * a.width + jc;
    const int li = __ldg(a.last_ids + pix);
    const float alpha = __ldg(a.out_alpha + pix);
    const float odepth = __ldg(a.out_depth + pix);
    const uint8_t m = __ldg(a.clamp_mask + pix);
    float nn = 1.f, on0 = 0.f, on1 = 0.f, on2 = 0.f;
    if (NORMALS) {
      nn = __ldg(a.normal_norm + pix);
      on0 = __ldg(a.out_normal + pix * 3 + 0); on1 = __ldg(a.out_normal + pix * 3 + 1); on2 = __ldg(a.out_normal + pix * 3 + 2);
    }
    float g_rgb[3] = {0.f, 0.f, 0.f}, g_d = 0.f, g_n[3] = {0.f, 0.f, 0.f};
    if (a.v_rgb) { g_rgb[0] = __ldg(a.v_rgb + pix * 3 + 0); g_rgb[1] = __ldg(a.v_rgb + pix * 3 + 1); g_rgb[2] = __ldg(a.v_rgb + pix * 3 + 2); }
    if (a.v_depth) g_d = __ldg(a.v_depth + pix);
    if (NORMALS && a.v_normal) { g_n[0] = __ldg(a.v_normal + pix * 3 + 0); g_n[1] = __ldg(a.v_normal + pix * 3 + 1); g_n[2] = __ldg(a.v_normal + pix * 3 + 2); }
    const float g_a = a.v_alpha ? __ldg(a.v_alpha + pix) : 0.f;
    if (a.loss_flags & DNR_LOSS_FUSED_BWD) fused_loss_grads(a, i, jc, g_rgb, g_d, g_n);

    last_id[p] = inside ? li : -1;
    wl = max(wl, last_id[p]);
    const float T_final = inside ? 1.0f - alpha : 1.0f;
    vC0[p] = (inside && (m & 1)) ? g_rgb[0] : 0.f;
    vC1[p] = (inside && (m & 2)) ? g_rgb[1] : 0.f;
    vC2[p] = (inside && (m & 4)) ? g_rgb[2] : 0.f;
    float va_cd = g_a - (a.background[0] * vC0[p] + a.background[1] * vC1[p] + a.background[2] * vC2[p]);
    const float ac = fmaxf(alpha, 1e-10f);
    vD[p] = (inside && alpha > 0.f) ? g_d / ac : 0.f;
    if (alpha >= 1e-10f) va_cd -= g_d * odepth / ac;
    float va_n = 0.f;
    vN0[p] = vN1[p] = vN2[p] = 0.f;
    if (NORMALS) {
      const float n0 = 2.0f * on0 - 1.0f, n1 = 2.0f * on1 - 1.0f, n2 = 2.0f * on2 - 1.0f;
      const float g0 = 0.5f * g_n[0], g1 = 0.5f * g_n[1], g2 = 0.5f * g_n[2];
      const float dp = n0 * g0 + n1 * g1 + n2 * g2;
      vN0[p] = inside ? (g0 - n0 * dp) / nn : 0.f;
      vN1[p] = inside ? (g1 - n1 * dp) / nn : 0.f;
      vN2[p] = inside ? (g2 - n2 * dp) / nn : 0.f;
      va_n = -(vN0[p] + vN1[p] + vN2[p]);
    }
    if (!inside) va_cd = 0.f;
    // d(out)/d(alpha_i) = sum_k (c_k T - B_k ra) v_k + T_final ra v_a, B_k = sum_{j>i} c_jk fac_j.  Only the contraction
    // S = sum_k B_k v_k is needed, and it is carried as S' = S - T_final v_a: one running scalar per gradient route.
    Tp[p] = T_final;
    Scd[p] = -T_final * va_cd;
    Sn[p] = -T_final * va_n;
  }

  // ---- range actually composited by this tile ----
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) wl = max(wl, __shfl_xor_sync(0xffffffffu, wl, o));
  if (lane == 0) red_last[warp] = wl;  // wl: deepest list position any pixel of this warp composited
  if (tid == 0) {
    mbar_init(&bars[0], 1);
    mbar_init(&bars[1], 1);
    mbar_fence_init();
  }
  __syncthreads();
  int hi_ = red_last[0];
#pragma unroll
  for (int w = 1; w < NW; ++w) hi_ = max(hi_, red_last[w]);
  hi_ = min(hi_ + 1, end);  // exclusive
  const int n = hi_ - start;
  if (n <= 0) return;
  const int nchunks = (n + CH - 1) / CH;

  V2 T[2], S1[2], S2[2], gC0[2], gC1[2], gC2[2], gD[2], gN0[2], gN1[2], gN2[2], npy[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    T[h] = v2(Tp[2 * h], Tp[2 * h + 1]);
    S1[h] = v2(Scd[2 * h], Scd[2 * h + 1]);
    S2[h] = v2(Sn[2 * h], Sn[2 * h + 1]);
    gC0[h] = v2(vC0[2 * h], vC0[2 * h + 1]); gC1[h] = v2(vC1[2 * h], vC1[2 * h + 1]);
    gC2[h] = v2(vC2[2 * h], vC2[2 * h + 1]); gD[h] = v2(vD[2 * h], vD[2 * h + 1]);
    gN0[h] = v2(vN0[2 * h], vN0[2 * h + 1]); gN1[h] = v2(vN1[2 * h], vN1[2 * h + 1]);
    gN2[h] = v2(vN2[2 * h], vN2[2 * h + 1]);
    const float y0 = (float)(blockIdx.y * DNR_TILE + ly + 4 * h) + 0.5f;
    npy[h] = v2(-y0, -(y0 + 2.0f));
  }
  // per-lane post-scale of the reduced totals (lane k & 15 owns value k): conic rows 0.5, mean rows -ln2 / ln2 (abs)
  const int vk = lane & 15;
  const float post = (vk == 0 || vk == 1) ? -DNR_LN2 : ((vk == 2 || vk == 3) ? DNR_LN2 : ((vk == 4 || vk == 6) ? 0.5f : 1.0f));
  float* scr = red_scr + warp * RED_WARP_FLOATS;
  unsigned long long walked = 0, kept = 0;

  // chunk c covers list positions [chi - n_c, chi), chi = hi - c*CH; slot t <-> position chi-1-t
  issue_chunk<REC, BWD_THREADS>(a.records, a.flatten_ids, hi_ - 1, -1, min(CH, n), recs[0], ids_s[0], &bars[0], tid);
  for (int c = 0; c < nchunks; ++c) {
    const int stage = c & 1;
    const int chi = hi_ - c * CH;
    const int n_c = min(CH, chi - start);
    if (c + 1 < nchunks)
      issue_chunk<REC, BWD_THREADS>(a.records, a.flatten_ids, chi - CH - 1, -1, min(CH, chi - CH - start), recs[stage ^ 1],
                                    ids_s[stage ^ 1], &bars[stage ^ 1], tid);
    mbar_wait(&bars[stage], (uint32_t)((c >> 1) & 1));
    const int total = filter_chunk<REC, BWD_THREADS>(recs[stage], n_c, blockIdx.x, blockIdx.y, sidx, scnt, tid);
    walked += n_c; kept += total;
    const float4* r4 = reinterpret_cast<const float4*>(recs[stage]);
    int t_next = total > 0 ? (int)sidx[0] : 0;
    for (int s = 0; s < total; ++s) {
      const int t = t_next;
      if (s + 1 < total) t_next = sidx[s + 1];  // next survivor's slot: off the critical path of the next iteration
      const int pos = chi - 1 - t;
      if (pos > wl) continue;  // deeper than anything this warp composited (warp-uniform)
      const int gid = ids_s[stage][t];  // for the RED at the end: loaded now, needed ~300 instructions later
      const float4 q0 = r4[t * RQ + 0];
      const float4 q1 = r4[t * RQ + 1];
      const float dx = q0.x - px;
      V2 dy[2], vis[2], al[2], t1[2], cdy[2];
      int any = 0, clamped = 0;  // ints and bitwise ops on purpose: && / || compile to divergent branches here
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        dy[h] = add2(v2(q0.y), npy[h]);
        // dnr_power2x2 spelled out (same roundings): its intermediates give d(power)/d(dx, dy) below for one FMA each
        const V2 bdy = mul2(v2(q0.w), dy[h]);
        cdy[h] = mul2(v2(q1.x), dy[h]);
        t1[h] = fma2(v2(q0.z), v2(dx), bdy);
        const V2 pw = fma2(v2(dx), t1[h], mul2(dy[h], cdy[h]));
        const float pw0 = lo(pw), pw1 = hi(pw);
        int ok0 = (pos <= last_id[2 * h]) & !(pw0 > 0.f) & !(pw0 < q1.z);
        int ok1 = (pos <= last_id[2 * h + 1]) & !(pw1 > 0.f) & !(pw1 < q1.z);
        const float e0 = dnr_ex2(pw0), e1 = dnr_ex2(pw1);
        const V2 araw = mul2(v2(q1.y), v2(e0, e1));
        const float a0 = fminf(DNR_ALPHA_MAX, lo(araw)), a1 = fminf(DNR_ALPHA_MAX, hi(araw));
        ok0 &= !(a0 < DNR_ALPHA_MIN);
        ok1 &= !(a1 < DNR_ALPHA_MIN);
        // a pixel that did not composite this splat carries vis = alpha = 0: every contribution below is then exactly
        // zero and its T / S state is unchanged (rcp.approx(1) == 1)
        vis[h] = v2(ok0 ? e0 : 0.f, ok1 ? e1 : 0.f);
        al[h] = v2(ok0 ? a0 : 0.f, ok1 ? a1 : 0.f);
        any |= ok0 | ok1;
        clamped |= (ok0 & (lo(araw) > DNR_ALPHA_MAX)) | (ok1 & (hi(araw) > DNR_ALPHA_MAX));
      }
      if (!__any_sync(0xffffffffu, any)) continue;
      const float4 q2 = r4[t * RQ + 2];
      float4 q3 = make_float4(0.f, 0.f, 0.f, 0.f);
      if (NORMALS) q3 = r4[t * RQ + 3];
      const bool slow = __any_sync(0xffffffffu, clamped);  // some alpha hit the 0.999 clamp: no gradient through sigma / opacity
      const V2 zero = v2(0.f);
      V2 acc[16];
#pragma unroll
      for (int k = 0; k < 16; ++k) acc[k] = zero;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const V2 om = sub2(v2(1.0f), al[h]);
        const V2 ra = v2(rcp_approx(lo(om)), rcp_approx(hi(om)));
        T[h] = mul2(T[h], ra);
        const V2 fac = mul2(al[h], T[h]);
        const V2 dot_cd = fma2(v2(q2.x), gC0[h], fma2(v2(q2.y), gC1[h], fma2(v2(q2.z), gC2[h], mul2(v2(q2.w), gD[h]))));
        // v_alpha = T dot - ra S'
        const V2 va_cd = sub2(mul2(T[h], dot_cd), mul2(ra, S1[h]));
        S1[h] = fma2(fac, dot_cd, S1[h]);
        acc[8] = fma2(fac, gC0[h], acc[8]); acc[9] = fma2(fac, gC1[h], acc[9]);
        acc[10] = fma2(fac, gC2[h], acc[10]); acc[11] = fma2(fac, gD[h], acc[11]);
        V2 va_all = va_cd;
        if (NORMALS) {
          const V2 dot_n = fma2(v2(q3.x), gN0[h], fma2(v2(q3.y), gN1[h], mul2(v2(q3.z), gN2[h])));
          const V2 va_n = sub2(mul2(T[h], dot_n), mul2(ra, S2[h]));
          S2[h] = fma2(fac, dot_n, S2[h]);
          acc[12] = fma2(fac, gN0[h], acc[12]); acc[13] = fma2(fac, gN1[h], acc[13]); acc[14] = fma2(fac, gN2[h], acc[14]);
          va_all = add2(va_cd, va_n);
        }
        V2 nov = mul2(v2(-q1.y), vis[h]);  // -opacity * vis
        V2 visg = vis[h];
        if (slow) {
          const bool c0 = lo(nov) < -DNR_ALPHA_MAX, c1 = hi(nov) < -DNR_ALPHA_MAX;
          nov = v2(c0 ? 0.f : lo(nov), c1 ? 0.f : hi(nov));
          visg = v2(c0 ? 0.f : lo(visg), c1 ? 0.f : hi(visg));
        }
        // d/d sigma; the constant factors 0.5 (conic rows) and -+ln2 (mean rows) are applied to the reduced totals (`post`)
        const V2 vs_cd = mul2(nov, va_cd);    // colour / depth route only (the normal pass sees detached xys, B3)
        const V2 vs_all = mul2(nov, va_all);
        const V2 tx = mul2(vs_all, v2(dx));
        acc[4] = fma2(tx, v2(dx), acc[4]);
        acc[5] = fma2(tx, dy[h], acc[5]);
        acc[6] = fma2(mul2(vs_all, dy[h]), dy[h], acc[6]);
        // d sigma / d mean2d = -ln2 (2 a' dx + b' dy, b' dx + 2 c' dy)
        const V2 u = fma2(v2(q0.z), v2(dx), t1[h]);           // t1 = a' dx + b' dy
        const V2 w = fma2(v2(2.0f), cdy[h], v2(q0.w * dx));  // cdy = c' dy
        const V2 gx = mul2(vs_cd, u);
        const V2 gy = mul2(vs_cd, w);
        acc[0] = add2(acc[0], gx);
        acc[1] = add2(acc[1], gy);
        acc[2] = add2(acc[2], v2(fabsf(lo(gx)), fabsf(hi(gx))));
        acc[3] = add2(acc[3], v2(fabsf(lo(gy)), fabsf(hi(gy))));
        acc[7] = fma2(visg, va_all, acc[7]);
      }
      float v[16];
#pragma unroll
      for (int k = 0; k < 16; ++k) v[k] = lo(acc[k]) + hi(acc[k]);
      const float tot = transpose_reduce16(v, scr, lane) * post;
      if (lane < 16 && tot != 0.f) atomicAdd(a.grad_records + (size_t)gid * DNR_GRAD_FLOATS + lane, tot);
      if (a.touched != nullptr && lane == 0) a.touched[gid] = 1;
    }
    __syncthreads();  // stage, sidx and ids_s free for the chunk after next
  }
  if (a.stats != nullptr && tid == 0) {
    atomicAdd((unsigned long long*)a.stats + 2, walked);
    atomicAdd((unsigned long long*)a.stats + 3, kept);
  }
}

}  // namespace

static int raster_common_checks(const DnrArgs* a) {
  if (!a) return DNR_E_NULL;
  if (a->width <= 0 || a->height <= 0 || a->n_isects < 0) return DNR_E_SIZE;
  if (a->tile_size != DNR_TILE) return DNR_E_OPTION;
  if (a->list_shift < 0 || a->list_shift > 3) return DNR_E_OPTION;
  if ((a->flags & DNR_FLAG_EXACT_LISTS) && a->list_shift != 0) return DNR_E_OPTION;
  return 0;
}

extern "C" int dnr_raster_fwd(const DnrArgs* a, void* stream) {
  if (const int rc = raster_common_checks(a)) return rc;
  if (!a->records || !a->tile_offsets || !a->out_rgb || !a->out_depth || !a->out_alpha || !a->last_ids ||
      !a->clamp_mask || !a->depth_max)
    return DNR_E_NULL;
  if (a->n_isects > 0 && !a->flatten_ids) return DNR_E_NULL;
  const bool normals = (a->flags & DNR_FLAG_NORMALS) != 0;
  if (normals && (!a->out_normal || !a->normal_norm)) return DNR_E_NULL;
  cudaStream_t s = (cudaStream_t)stream;
  DNR_CUDA(cudaMemsetAsync(a->depth_max, 0, sizeof(int32_t), s));
  const dim3 grid(dnr_tiles_x(a), dnr_tiles_y(a));
  const int sx = dnr_stiles_x(a);
  if (normals) raster_fwd_kernel<true><<<grid, FWD_THREADS, 0, s>>>(*a, sx);
  else raster_fwd_kernel<false><<<grid, FWD_THREADS, 0, s>>>(*a, sx);
  DNR_CHECK_LAUNCH();
  return 0;
}

extern "C" int dnr_raster_bwd(const DnrArgs* a, void* stream) {
  if (const int rc = raster_common_checks(a)) return rc;
  if (a->n_gauss <= 0) return DNR_E_SIZE;
  if (!a->records || !a->tile_offsets || !a->out_depth || !a->out_alpha || !a->last_ids || !a->clamp_mask ||
      !a->grad_records)
    return DNR_E_NULL;
  if (a->n_isects > 0 && !a->flatten_ids) return DNR_E_NULL;
  const bool normals = (a->flags & DNR_FLAG_NORMALS) != 0;
  if (normals && (!a->out_normal || !a->normal_norm)) return DNR_E_NULL;
  if (a->loss_flags & DNR_LOSS_FUSED_BWD) {
    if (a->v_l1 && (!a->gt_image || !a->out_rgb)) return DNR_E_NULL;
    if (a->depth_loss_type < 0 || a->depth_loss_type > 4) return DNR_E_OPTION;
    if (a->depth_loss_type != 0 && (!a->gt_depth || !a->loss_partials)) return DNR_E_NULL;
    if (a->depth_loss_type == 1 && !((a->loss_flags & DNR_LOSS_EDGE_FROM_IMAGE) ? a->gt_image : (const void*)a->gt_rgb)) return DNR_E_NULL;
    if ((a->loss_flags & DNR_LOSS_EDGE_FROM_IMAGE) && !(a->loss_flags & DNR_LOSS_IMG_U8)) return DNR_E_OPTION;
    if (a->use_normal_loss && (!normals || !a->gt_normal)) return DNR_E_NULL;
  }
  cudaStream_t s = (cudaStream_t)stream;
  if (a->flags & DNR_FLAG_PERSISTENT_WS) {
    if (!a->touched) return DNR_E_NULL;  // the flags are what lets the next project_bwd restore grad_records to zero
  } else {
    DNR_CUDA(cudaMemsetAsync(a->grad_records, 0, (size_t)a->n_gauss * DNR_GRAD_FLOATS * sizeof(float), s));
    if (a->touched) DNR_CUDA(cudaMemsetAsync(a->touched, 0, (size_t)a->n_gauss, s));
  }
  if (a->n_isects == 0) return 0;
  const dim3 grid(dnr_tiles_x(a), dnr_tiles_y(a));
  const int sx = dnr_stiles_x(a);
  if (normals) raster_bwd_kernel<true><<<grid, BWD_THREADS, 0, s>>>(*a, sx);
  else raster_bwd_kernel<false><<<grid, BWD_THREADS, 0, s>>>(*a, sx);
  DNR_CHECK_LAUNCH();
  return 0;
}
