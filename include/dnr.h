/*
 * dnr.h — C ABI of libdnr_b200.so: the H100 (sm_90a) depth+normal Gaussian rasterizer that
 * replaces the two gsplat calls (and the torch glue between them) inside
 * DNSplatterModel.get_outputs of maturk/dn-splatter.
 *
 * Reference interfaces replaced (paths relative to /root/reference/):
 *   dnr_project_fwd    gsplat fully_fused_projection + spherical_harmonics + param activations
 *                      (dn_splatter/dn_model.py:495-500 arguments of rasterization();
 *                      :543-560 per-Gaussian normals)
 *   dnr_bin_scan/sort  gsplat isect_tiles + radix sort + isect_offset_encode, shared by the colour and
 *                      the normal pass (dn_model.py:495-516 and the second binning hidden in :564-575)
 *   dnr_raster_fwd     gsplat rasterize_to_pixels (RGB+ED, dn_model.py:495-516) + legacy
 *                      rasterize_gaussians on normals (:564-575) + blend/clamp/normalise (:526-537,:577-578)
 *   dnr_finalize_fwd   depth fill with the global max (dn_model.py:534-537) + normal_from_depth_image
 *                      (dn_splatter/utils/normal_utils.py:25-48, called at dn_model.py:589-603)
 *   dnr_raster_bwd     autograd backward of the two rasterizations and of the glue above
 *   dnr_project_bwd    autograd backward of projection / SH / activations / normals
 *   dnr_loss_*         DNRegularization depth + normal terms (dn_splatter/regularization_strategy.py:146-193,
 *                      dn_splatter/losses.py:155-224,279-295) fused: value + per-pixel gradient
 *
 * Conventions: plain C, POD only, every pointer is a DEVICE pointer unless named *_host, row-major
 * contiguous fp32, images [H,W,C], quaternions wxyz, viewmat = world->camera (OpenCV), pixel centres
 * at +0.5, tile size 16.  The caller owns every buffer (including workspaces sized by the *_bytes
 * queries).  All work is enqueued on the stream passed in (a cudaStream_t cast to void*); the only
 * host synchronisation is the documented n_isects read-back inside dnr_bin_scan.
 * Return value: 0 = ok, <0 = DNR_E_* argument error, >0 = cudaError_t of a failed launch.
 * Workspaces: the cub scratch in a workspace is sized by cub's queries, which need a device; without one they fail and
 * the size a *_workspace_bytes query returns lacks that scratch.  Every entry point that runs cub repeats the queries and,
 * after DNR_E_WORKSPACE for a workspace that is too small, returns the first failed query's cudaError_t (> 0) rather
 * than run without the scratch.
 * No global state, re-entrant, never throws, never prints.
 */
#ifndef DNR_H_
#define DNR_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DNR_VERSION 100 /* 0.1.0 */

#define DNR_E_NULL (-1)     /* a required pointer is NULL */
#define DNR_E_SIZE (-2)     /* non-positive / inconsistent sizes */
#define DNR_E_OPTION (-3)   /* unsupported option (tile size, sh degree, ...) */
#define DNR_E_OVERFLOW (-4) /* more than 2^31-1 tile intersections */
#define DNR_E_WORKSPACE (-5)/* workspace too small */

/* flags */
#define DNR_FLAG_ACTIVATED 1u   /* scales/opacities are already exp()/sigmoid()-activated (gsplat's signature) */
#define DNR_FLAG_ANTIALIASED 2u /* rasterize_mode == "antialiased": opacity *= compensation */
#define DNR_FLAG_NORMALS 4u     /* predict_normals: render the per-Gaussian normal channels */
#define DNR_FLAG_ACCUMULATE 8u  /* project_bwd adds into the parameter-gradient buffers (required by dnr_project_bwd) */
#define DNR_FLAG_HOST_CAMERA 32u /* camera passed by value in host_cam[] (no device reads, no H2D copy) */
#define DNR_FLAG_EXACT_LISTS 16u /* parity mode: emit gsplat's full bbox intersection lists (no precise-hit cull) */
/* 64u and 128u are retired (they selected project_bwd kernels that no longer exist) and are not to be reused */
#define DNR_FLAG_PERSISTENT_WS 256u /* raster_bwd: touched and grad_records are the caller's persistent buffers and are not
                                       cleared.  grad_records must be all zero on entry (the project_bwd that follows
                                       leaves it so); the flags accumulate over calls until the caller clears them
                                       (dnr_grad_zero) */

/* floats per packed per-Gaussian raster record, without / with normals */
#define DNR_REC_FLOATS 12
#define DNR_REC_FLOATS_N 16
/* floats per per-Gaussian raster-gradient record (always) */
#define DNR_GRAD_FLOATS 16

typedef struct DnrArgs {
  /* ---- sizes and options (host scalars) ---- */
  int32_t n_gauss;   /* N */
  int32_t width, height;
  int32_t tile_size; /* must be 16 (dn_model.py:470-472) */
  int32_t sh_degree; /* active degree 0..3 (dn_model.py:487-490) */
  int32_t sh_bases;  /* bases stored per Gaussian: sh_rest is [N, sh_bases-1, 3] */
  uint32_t flags;    /* DNR_FLAG_* */
  int32_t list_shift; /* intersection lists are kept per SUPERTILE of (16 << list_shift)^2 pixels (0..3); every 16x16 tile
                         walks its supertile's list and drops, inside the raster kernels, the entries that cannot reach it.
                         0 = one list per tile (required with DNR_FLAG_EXACT_LISTS: gsplat's lists) */
  float near_plane, far_plane, eps2d, radius_clip;
  float background[3];
  float reserved1;
  int64_t n_isects; /* capacity of flatten_ids / ws_sort in intersections (>= the count dnr_bin_scan reports, or an
                       estimate when running sync-free: see n_isects_dev) */

  /* ---- camera (device) ---- */
  const float* viewmat; /* [4,4] */
  const float* K;       /* [3,3] */
  const float* c2w;     /* [3,4] nerfstudio camera_to_world (OpenGL, un-optimised); normals only */

  /* ---- Gaussian parameters (device, the reference's gauss_params layout, dn_model.py:227-237) ---- */
  const float* means;     /* [N,3] */
  const float* quats;     /* [N,4] */
  const float* scales;    /* [N,3] log-scales (or activated with DNR_FLAG_ACTIVATED) */
  const float* opacities; /* [N]   logits     (or activated) */
  const float* sh_dc;     /* [N,3] */
  const float* sh_rest;   /* [N,sh_bases-1,3] (may be NULL when sh_bases==1) */

  /* ---- projection outputs (info dict of gsplat.rasterization, dn_model.py:517-524) ---- */
  int32_t* radii;           /* [N] */
  float* means2d;           /* [N,2] */
  float* depths;            /* [N] */
  float* conics;            /* [N,3] */
  float* opac_act;          /* [N] activated (x compensation) opacity */
  float* compensations;     /* [N] or NULL */
  float* colors;            /* [N,3] clamp_min(SH+0.5,0) */
  float* normals_world;     /* [N,3] flipped world normals (gauss_params["normals"], dn_model.py:558) or NULL */
  int32_t* tiles_per_gauss; /* [N] */
  uint32_t* depth_keys;     /* [N] bit pattern of depth, 0xFFFFFFFF when culled */
  float* records;           /* [N, DNR_REC_FLOATS(_N)] packed raster records */
  float* cull_lim;          /* [N] ln(255 * sigmoid opacity) + margin: largest sigma that can still reach alpha >= 1/255 */

  /* ---- binning ---- */
  void* ws_scan;         /* dnr_bin_scan_workspace_bytes(N) */
  void* ws_sort;         /* dnr_bin_sort_workspace_bytes(N, I, n_tiles) */
  int32_t* flatten_ids;  /* [I] Gaussian ids sorted by (tile, depth, id) */
  int32_t* tile_offsets; /* [n_tiles+1] */
  int64_t* n_isects_dev; /* [1] device copy of the intersection count (may exceed the capacity: then the render is
                            truncated and the caller must retry with a larger n_isects) */

  /* ---- raster forward outputs / backward state ---- */
  float* out_rgb;      /* [H,W,3] clamp(C + (1-alpha) bg, 0, 1) */
  float* out_depth;    /* [H,W]   D/alpha, then filled by dnr_finalize_fwd */
  float* out_alpha;    /* [H,W] */
  float* out_normal;   /* [H,W,3] (n/|n|+1)/2 or NULL */
  float* out_surface_normal; /* [H,W,3] or NULL */
  int32_t* last_ids;   /* [H,W] */
  float* normal_norm;  /* [H,W] |n_raw| (backward state) or NULL */
  uint8_t* clamp_mask; /* [H,W] bit k set: rgb channel k passes gradient */
  int32_t* depth_max;  /* [1] bit pattern of max expected depth */

  /* ---- raster backward ---- */
  const float* v_rgb;    /* [H,W,3] or NULL */
  const float* v_depth;  /* [H,W]   or NULL */
  const float* v_normal; /* [H,W,3] or NULL */
  const float* v_alpha;  /* [H,W]   or NULL */
  float* grad_records;   /* [N, DNR_GRAD_FLOATS] zeroed by dnr_raster_bwd (unless DNR_FLAG_PERSISTENT_WS);
                            dnr_project_bwd writes zeros back to every row it consumes */

  /* ---- projection backward outputs ---- */
  float* v_means;       /* [N,3] */
  float* v_quats;       /* [N,4] */
  float* v_scales;      /* [N,3] */
  float* v_opacities;   /* [N] */
  float* v_sh_dc;       /* [N,3] */
  float* v_sh_rest;     /* [N,sh_bases-1,3] */
  float* v_means2d;     /* [N,2] or NULL  (info["means2d"].grad) */
  float* v_means2d_abs; /* [N,2] or NULL  (info["means2d"].absgrad) */

  /* ---- fused regularisers (DNRegularization) ---- */
  const float* gt_depth;  /* [H,W] */
  const float* gt_normal; /* [H,W,3] */
  const float* gt_rgb;    /* [H,W,3] */
  float* loss_partials;   /* [12] fp32 accumulators + results, see dnr_loss_fwd */
  const float* v_loss;    /* [1] device scalar: upstream gradient of the regulariser (NULL = 1) */
  float depth_lambda, depth_tolerance;
  int32_t depth_loss_type; /* 0 none, 1 EdgeAwareLogL1, 2 LogL1, 3 L1, 4 MSE */
  int32_t use_normal_loss;
  /* with DNR_FLAG_HOST_CAMERA: [0..15] viewmat, [16..19] fx fy cx cy, [20..31] c2w[3,4]; viewmat/K/c2w pointers unused */
  float host_cam[32];
  const void* reserved2; /* unused; keeps the layout (and so the kernels' parameter offsets) stable */

  /* ---- loss gradients evaluated inside dnr_raster_bwd (BASELINE north_star: regularisers fused into the backward) ----
   * With DNR_LOSS_FUSED_BWD the per-pixel gradients of
   *   *v_l1  * mean|rgb - gt_image|                     (parent photometric L1; term off when v_l1 == NULL)
   *   *v_loss * DNRegularization(depth, normal)         (dnr_loss_fwd's terms; uses gt_depth, gt_normal, gt_rgb /
   *                                                      gt_image, loss_partials, depth_* fields, use_normal_loss)
   * are computed in the kernel's prologue from the rendered maps instead of being read from v_rgb / v_depth / v_normal
   * images; non-NULL v_rgb / v_depth / v_normal / v_alpha are ADDED (e.g. the SSIM gradient). */
  uint32_t loss_flags;   /* DNR_LOSS_* */
  int32_t reserved3;     /* unused, as reserved2 */
  const void* gt_image;  /* [H,W,3] photometric target: uint8 (DNR_LOSS_IMG_U8, scaled by 1/255) or fp32 */
  const float* v_l1;     /* [1] device scalar */
  uint8_t* touched;      /* [N]: dnr_raster_bwd sets touched[g] = 1 for every Gaussian that received a gradient
                            (zeroed by the call unless DNR_FLAG_PERSISTENT_WS); dnr_project_bwd processes only the
                            flagged Gaussians.  Required by dnr_project_bwd; dnr_raster_bwd alone accepts NULL (without
                            DNR_FLAG_PERSISTENT_WS) */
  uint64_t* stats; /* [4] or NULL: += {list entries walked, entries kept by the tile filter} (fwd: [0],[1]; bwd: [2],[3]) */
  float* v_viewmat; /* [4,4] or NULL: dnr_project_bwd ADDS d(loss)/d(viewmat) (camera optimisation; the caller zeroes it
                       first; row 3 is left alone).  Works with DNR_FLAG_HOST_CAMERA too.  The normals' c2w is treated
                       as a separate constant. */
} DnrArgs;

/* loss_flags */
#define DNR_LOSS_FUSED_BWD 1u  /* dnr_raster_bwd evaluates the loss gradients itself (see above) */
#define DNR_LOSS_IMG_U8 2u     /* gt_image is uint8 */
#define DNR_LOSS_NORMAL_U8 4u  /* gt_normal is uint8 [H,W,3] (value / 255, as get_gt_img does) */
#define DNR_LOSS_EDGE_FROM_IMAGE 8u /* EdgeAwareLogL1 edge weights from gt_image clamped below at 10/255 (dn_model.py:633)
                                       instead of the fp32 gt_rgb map */

int dnr_version(void);
const char* dnr_error_string(int code);

int dnr_project_fwd(const DnrArgs* a, void* stream);

size_t dnr_bin_scan_workspace_bytes(int32_t n_gauss);
/* Sorts visible Gaussians by depth, counts the tiles each one really touches (or its whole bbox with
 * DNR_FLAG_EXACT_LISTS), scans the counts and stores the total in *a->n_isects_dev.  If n_isects_host is not
 * NULL the total is also copied there and the stream is synchronised (the one documented host sync);
 * pass NULL to stay asynchronous and size by capacity. */
int dnr_bin_scan(const DnrArgs* a, void* stream, int64_t* n_isects_host);
size_t dnr_bin_sort_workspace_bytes(int32_t n_gauss, int64_t n_isects, int32_t n_tiles);
int dnr_bin_sort(const DnrArgs* a, void* stream);

int dnr_raster_fwd(const DnrArgs* a, void* stream);
int dnr_finalize_fwd(const DnrArgs* a, void* stream);
/* normal_from_depth_image for an arbitrary depth map: depth in a->out_depth, result (un-flipped,
 * un-remapped, zero border) in a->out_surface_normal; intrinsics from a->K. */
int dnr_normal_from_depth(const DnrArgs* a, void* stream);

int dnr_raster_bwd(const DnrArgs* a, void* stream);
int dnr_project_bwd(const DnrArgs* a, void* stream);

/* DNRegularization depth + normal terms on rendered maps: pred depth in a->out_depth, pred normal in
 * a->out_normal.  loss_partials (zeroed by the call):
 * [0] sum_x  [1] count_x  [2] sum_y  [3] count_y  (depth term; for non edge-aware types only x is used)
 * [4] sum |n - n_gt|   [5] sum |dW n|   [6] sum |dH n|
 * [8] depth term incl. the (1 + depth_lambda) factor  [9] normal L1  [10] normal TV  [11] [8]+[9]+[10].
 * dnr_loss_bwd writes d(loss)/d(depth) [H,W] and d(loss)/d(normal) [H,W,3] (either may be NULL). */
int dnr_loss_fwd(const DnrArgs* a, void* stream);
int dnr_loss_bwd(const DnrArgs* a, float* v_depth_out, float* v_normal_out, void* stream);

/* AGSMeshRegularization depth + normal terms (dn_splatter/regularization_strategy.py:202-321) on rendered maps.
 * The step-dependent choices are host flags: DNR_AGS_CONF_GATE (step >= 7000), DNR_AGS_ANGLE_MASK (step >=
 * normal_mask_steps; else the dilated-edge mask of the gt normal) and normal_lambda, which the caller passes as 0 while
 * step <= 7000.  Normal maps are [H,W,3] in the [0,1] encoding (the kernels form 2x - 1 in fp32; gt_normal may be uint8,
 * read as value / 255 with DNR_AGS_NORMAL_U8), or, with DNR_AGS_SIGNED_CHW, fp32 [3,H,W] already signed.
 * partials (16 floats; [0..11] zeroed by the forward):
 * [0] sum_x  [1] count_x  [2] sum_y  [3] count_y  (depth term; for non edge-aware types only x is used)
 * [4] sum |n - g| over all elements  [5] sum |s - g| over the kept elements  [6] their count
 * [8] depth_lambda * depth term  [9] normal_lambda * surface term  [10] normal_lambda * predicted-normal term
 * [11] [8] + ([9] + [10]).  An empty depth mask or surface selection makes its term nan, as torch's mean of nothing.
 * keep_mask (optional, [H,W] uint8): bit c set where element (c, pixel) is in the surface-term selection.
 * dnr_ags_loss_bwd writes d(loss)/d(pred_depth) [H,W] and d(loss)/d(pred_normal) ([H,W,3], or [3,H,W] with
 * DNR_AGS_SIGNED_CHW); either may be NULL.  The surface normal gets no gradient (it comes from detached depth). */
typedef struct DnrAgsLoss {
  int32_t width, height;
  int32_t depth_loss_type;  /* 0 none, 1 EdgeAwareLogL1, 2 LogL1, 3 L1, 4 MSE */
  uint32_t flags;           /* DNR_AGS_* */
  float depth_lambda, depth_tolerance;
  float normal_lambda;      /* already gated by the step */
  int32_t reserved;
  const float* pred_depth;  /* [H,W] */
  const float* gt_depth;    /* [H,W] */
  const void* confidence;   /* [H,W]: the gate map (fp32), or the raw map (DNR_AGS_CONF_RAW: fp32, or uint8 with
                               DNR_AGS_CONF_U8) gated on conf = 1 - get_gt_img(c) / 255 */
  const void* image;        /* [H,W,3] edge image of EdgeAwareLogL1: fp32 as given, or uint8 (DNR_AGS_IMG_U8) scaled
                               by 1/255 and clamped below at 10/255 */
  const float* surf_normal; /* surface normal of the rendered depth */
  const void* gt_normal;
  const float* pred_normal;
  float* partials;
  const float* v_loss;      /* upstream gradient of [11] (NULL: 1) */
  uint8_t* keep_mask;
} DnrAgsLoss;

#define DNR_AGS_CONF_GATE 1u
#define DNR_AGS_ANGLE_MASK 2u
#define DNR_AGS_NORMAL_U8 4u
#define DNR_AGS_IMG_U8 8u
#define DNR_AGS_CONF_RAW 16u
#define DNR_AGS_CONF_U8 32u
#define DNR_AGS_SIGNED_CHW 64u
#define DNR_AGS_ALL_FLAGS 127u

int dnr_ags_loss_fwd(const DnrAgsLoss* a, void* stream);
int dnr_ags_loss_bwd(const DnrAgsLoss* a, float* v_depth_out, float* v_normal_out, void* stream);

/* DNRegularization.get_scale_loss (regularization_strategy.py:195-199): mean_i min_k exp(scales[i,k]).
 * fwd: *loss_out (zeroed by the call) = the mean.  bwd: v_scales[N,3] = v * d(loss)/d(scales) (dense). */
int dnr_scale_loss_fwd(const float* scales, int32_t n_gauss, float* loss_out, void* stream);
int dnr_scale_loss_bwd(const float* scales, int32_t n_gauss, const float* v_loss, float* v_scales, void* stream);

/* Photometric L1 of the parent SplatfactoModel.get_loss_dict [EXT] (dn_splatter/dn_model.py:624-628 calls it):
 * mean |pred - gt| over n floats; gt is fp32, or uint8 (gt_is_u8 != 0, scaled by 1/255 as get_gt_img does).
 * fwd: *loss_out (zeroed by the call) = the mean.  bwd: v_pred[n] = (*v_loss or 1) * sign(pred - gt) / n. */
int dnr_l1_fwd(const float* pred, const void* gt, int64_t n, int32_t gt_is_u8, float* loss_out, void* stream);
int dnr_l1_bwd(const float* pred, const void* gt, int64_t n, int32_t gt_is_u8, const float* v_loss, float* v_pred,
               void* stream);
/* get_gt_img's uint8 -> float conversion in one pass: dst[i] = max(src[i] / divisor, clamp_min). */
int dnr_u8_to_f32(const uint8_t* src, int64_t n, float divisor, float clamp_min, float* dst, void* stream);

/* SSIM term of the same photometric loss: torchmetrics StructuralSimilarityIndexMeasure(data_range=1.0,
 * kernel_size=11) (dn_splatter/dn_model.py:180), i.e. an 11x11 Gaussian window (sigma 1.5), mean over the
 * (H-10)x(W-10) interior.  pred / gt: [H,W,C] fp32.  fwd: *sum_out (zeroed by the call) = SUM of the SSIM map over
 * the interior and all channels (divide by (H-10)(W-10)C for the mean); dmaps: 3·H·W·C floats of scratch whose
 * layout is private to the pair, written by the forward and read by the backward.
 * bwd: v_pred[H,W,C] = (*v_mean or 1) * d(mean SSIM)/d(pred).
 * Default since round 2 (DNSplatterModelConfig.fused_ssim). */
int dnr_ssim_fwd(const float* pred, const float* gt, int32_t H, int32_t W, int32_t C, float* dmaps, float* sum_out,
                 void* stream);
int dnr_ssim_bwd(const float* pred, const float* gt, int32_t H, int32_t W, int32_t C, const float* dmaps,
                 const float* v_mean, float* v_pred, void* stream);
/* The same with the target read as stored: gt is uint8 (value / 255, as get_gt_img does) when gt_is_u8 != 0, else fp32. */
int dnr_ssim_fwd_ex(const float* pred, const void* gt, int32_t gt_is_u8, int32_t H, int32_t W, int32_t C, float* dmaps,
                    float* sum_out, void* stream);
int dnr_ssim_bwd_ex(const float* pred, const void* gt, int32_t gt_is_u8, int32_t H, int32_t W, int32_t C, const float* dmaps,
                    const float* v_mean, float* v_pred, void* stream);

/* Evaluation (no gradient) of the same SSIM for a batch, with the squared error for PSNR / MSE, as torchmetrics'
 * StructuralSimilarityIndexMeasure(data_range=1.0, kernel_size=11) and PeakSignalNoiseRatio(data_range=1.0) need them
 * (Python surface: dn_splatter_b200.metrics.RGBMetrics).  pred: [B,H,W,C] fp32; gt: [B,H,W,C] fp32, or uint8 read as
 * value / 255 when gt_is_u8 != 0.  out [B,2] double (zeroed by the call): per image the SUM of the SSIM map over the
 * (H-10)x(W-10) interior and all channels, and the sum of (pred - gt)^2 over all H*W*C values.  H, W >= 11; B <= 65535. */
int dnr_rgb_metrics(const float* pred, const void* gt, int32_t gt_is_u8, int32_t B, int32_t H, int32_t W, int32_t C,
                    double* out, void* stream);

/* The whole photometric term of the parent SplatfactoModel.get_loss_dict [EXT] (dn_splatter/dn_model.py:624-628 calls it):
 *   main = (1 - ssim_lambda) * mean|pred - gt| + ssim_lambda * (1 - mean SSIM)
 * in one pass each way (the L1 sum shares the SSIM kernel's loads; its sign gradient is added by the SSIM backward).
 * out (3 floats, zeroed by the call): [0] SSIM sum over the interior, [1] sum |pred - gt|, [2] main.
 * bwd: v_pred[H,W,C] = (*v_main or 1) * d(main)/d(pred). */
int dnr_photometric_fwd(const float* pred, const void* gt, int32_t gt_is_u8, int32_t H, int32_t W, int32_t C,
                        float ssim_lambda, float* dmaps, float* out, void* stream);
int dnr_photometric_bwd(const float* pred, const void* gt, int32_t gt_is_u8, int32_t H, int32_t W, int32_t C,
                        float ssim_lambda, const float* dmaps, const float* v_main, float* v_pred, void* stream);

/* One-launch Adam over all Gaussian parameter groups: replaces the per-group torch.optim.Adam instances of
 * dn_splatter/dn_config.py:29-68 (lr per group, eps 1e-15; betas (0.9, 0.999), no weight decay, no amsgrad).
 * bc1 = 1 - beta1^t and bc2_sqrt = sqrt(1 - beta2^t) are computed by the host for each group's own step count t.
 * Python surface: optim.FusedAdam. */
#define DNR_ADAM_MAX_SEGS 16
typedef struct DnrAdamSeg {
  float* p;       /* [n] parameters, updated in place */
  const float* g; /* [n] gradients */
  float* m;       /* [n] exp_avg, updated in place */
  float* v;       /* [n] exp_avg_sq, updated in place */
  int64_t n;
  double lr, eps, bc1, bc2_sqrt; /* doubles: rounded to fp32 exactly where torch.optim.Adam rounds them */
  int64_t dense; /* dnr_adam_step_reduce only: != 0 -> every rank's rows of this segment are gathered, not just the rows of
                    the ranks that touched the Gaussian (a gradient term that depends on the parameters alone, e.g. the
                    min-scale regulariser, makes the whole segment non-zero on every rank) */
} DnrAdamSeg;
int dnr_adam_step(const DnrAdamSeg* segs /* HOST array */, int32_t n_segs, double beta1, double beta2, void* stream);

/* Multi-GPU: the gradient reduction fused into the Adam pass over NVLink peer memory (replaces the
 * bucket.all_reduce() + optimizer.step() pair that stands in for the reference's DDP wrapper, dn_pipeline.py:123-128).
 * Every rank keeps its flat gradient bucket and its `touched` flags (DnrArgs.touched, written by dnr_raster_bwd) in
 * peer-mapped memory at the same offsets; rows of untouched Gaussians are exactly zero.  For each element the gradient
 * is the sum, in rank order, of the rows of the ranks that touched the Gaussian (read straight from their memory), so
 * all replicas apply bit-identical updates.  segs[i].g must point into THIS rank's bucket (peer_flat[rank]); widths[i] =
 * floats per Gaussian of segment i.  The caller brackets the call with cross-rank barriers (all buckets final before,
 * all reads done before anyone zeroes its bucket again).
 * world == 1 is the single-GPU sparse step: peer_touched[0] (the bucket's own flags, which must cover every non-zero row
 * of the segments not marked dense) is the mask, `mask` is unused and no barrier is needed. */
#define DNR_PEER_MAX 8
typedef struct DnrPeerReduce {
  int32_t world, rank;
  int32_t n_gauss, reserved;
  const float* peer_flat[DNR_PEER_MAX];      /* device pointers valid on THIS device: rank k's flat bucket */
  const uint8_t* peer_touched[DNR_PEER_MAX]; /* rank k's touched flags [n_gauss] */
  uint8_t* mask;                             /* [n_gauss] local scratch (bit k: rank k touched the Gaussian) */
} DnrPeerReduce;
int dnr_adam_step_reduce(const DnrAdamSeg* segs /* HOST array */, const int32_t* widths /* HOST array */, int32_t n_segs,
                         double beta1, double beta2, const DnrPeerReduce* peers /* HOST struct */, void* stream);

/* Clears a flat gradient bucket whose `touched` flags cover every non-zero row (DNR_FLAG_PERSISTENT_WS): the rows of
 * flagged Gaussians in each segment, every segment marked dense, and the flags themselves.  Each g starts on a 16-byte
 * boundary and its segment is padded with zeros to a multiple of 4 floats (the padding may be written). */
typedef struct DnrGradSeg {
  float* g;      /* [n_gauss * width] */
  int32_t width; /* floats per Gaussian */
  int32_t dense; /* != 0: zero the whole segment (a gradient term that depends on the parameters alone) */
} DnrGradSeg;
int dnr_grad_zero(const DnrGradSeg* segs /* HOST array, at most DNR_ADAM_MAX_SEGS */, int32_t n_segs, uint8_t* touched,
                  int32_t n_gauss, void* stream);

/* ---- SuGaR-style queries (SURVEY 8f-4; Python surface: dn_splatter_b200.sugar) ----
 * Grid-hash k-NN: replaces sklearn behind dn_splatter/utils/knn.py:29-43 (knn_sk) and nerfstudio's k_nearest_sklearn
 * (dn_model.py:187).  The host chooses the grid; points outside it are clamped into the border cells (still exact). */
typedef struct DnrKnnGrid {
  float lo[3];     /* origin of cell (0,0,0) */
  float cell;      /* cell edge */
  float inv_cell;  /* 1 / cell */
  int32_t dims[3]; /* cells per axis; product <= 2^26 */
} DnrKnnGrid;
int64_t dnr_knn_workspace_bytes(int32_t n_points, const DnrKnnGrid* grid);
int dnr_knn_build(const float* points /* [n,3] */, int32_t n_points, const DnrKnnGrid* grid, void* ws, int64_t ws_bytes,
                  void* stream);
/* out_idx [n_queries,k] int64 (-1 where fewer than k points exist), out_dist [n_queries,k] Euclidean or NULL.
 * skip_first != 0 reproduces knn_sk: search k+1 and drop the nearest (the query itself when it is a data point). */
int dnr_knn_query(int32_t n_points, const DnrKnnGrid* grid, const void* ws, const float* queries /* [m,3] */,
                  int32_t n_queries, int32_t k, int32_t skip_first, int64_t* out_idx, float* out_dist, void* stream);
/* Density of the Gaussian set at samples [n,3] given neighbour lists nbr_idx [n / samples_per_row, k] (int64, -1 =
 * none): get_density (dn_model.py:1077-1135) with clamp_min = 1e-4.  Raw parameters (log-scales, opacity logits,
 * un-normalised wxyz quats). */
int dnr_density(const float* samples, int64_t n_samples, const int64_t* nbr_idx, int32_t k, int32_t samples_per_row,
                const float* means, const float* scales, const float* quats, const float* opacities, int32_t n_gauss,
                float clamp_min, float* out, void* stream);
/* The ray sampling of compute_level_surface_points (dn_model.py:1264-1345): for each point p (a back-projected
 * pixel) 21 samples p + t_j d, t_j = linspace(-range, range, 21) * std(first neighbour), d = normalize(p - cam).
 * out_dens / out_t [n_points,21], out_dirs [n_points,3].  cam_pos_host: 3 floats on the HOST. */
int dnr_ray_densities(const float* points, int64_t n_points, const int64_t* nbr_idx, int32_t k, const float* cam_pos_host,
                      const float* means, const float* scales, const float* quats, const float* opacities,
                      int32_t n_gauss, int32_t n_range, float range_size, float* out_dens, float* out_t, float* out_dirs,
                      void* stream);

/* ---- Mesh export (Python surface: dn_splatter_b200.mesh) ----
 * Dense TSDF volume: voxel (i, j, k) is voxels[(i * dims[1] + j) * dims[2] + k] (64-bit index), 16 bytes
 * {float tsdf, float weight, uint64 rgb}; colour is the weighted mean of the reference's uint8 colours (0..255), kept as
 * three 21-bit fixed-point numbers in units of 2^-13 of a level, r | g << 21 | b << 42, rounded half up on each update.
 * Voxel centres are origin + (index + 0.5) * voxel.  All zero is an empty volume. */
typedef struct DnrTsdfGrid {
  float origin[3];
  float voxel;     /* voxel edge */
  float sdf_trunc; /* truncation distance */
  int32_t dims[3]; /* voxels per axis, each <= 65535 */
  void* voxels;
} DnrTsdfGrid;
/* Fuses one view, Open3D legacy ScalableTSDFVolume.integrate semantics (DESIGN.md §2) [EXT]: depth [H,W] f32,
 * rgb [H,W,3] f32 in [0,1], mask [H,W] uint8 or NULL (0 = no depth), depth <= 0 or > depth_trunc is no depth.
 * cam_host: 16 HOST floats {fx, fy, cx, cy, world->camera [3,4] row-major (OpenCV)}.  Only updated voxels are written. */
int dnr_tsdf_integrate(const DnrTsdfGrid* grid, const float* depth, const float* rgb, const uint8_t* mask, int32_t width,
                       int32_t height, const float* cam_host, float depth_trunc, void* stream);

/* Marching cubes over samples (i, j, k) at origin + (i, j, k) * spacing, index (i * dims[1] + j) * dims[2] + k.  Exactly
 * one of values / tsdf is set.  "Inside" is value < iso; a cube with an invalid corner emits nothing.  Vertices are welded
 * (one per crossed grid edge), ordered by (sample index, edge axis); faces by cube index, then table order
 * (csrc/mc_tables.cuh), counter-clockwise seen from the value > iso side. */
typedef struct DnrMcField {
  const float* values;  /* [X,Y,Z] scalar field, or NULL */
  const uint8_t* valid; /* [X,Y,Z] or NULL (all valid); with values only */
  const void* tsdf;     /* [X,Y,Z] DnrTsdfGrid voxels, or NULL: value = tsdf, valid where weight > 0, with colour */
  int32_t dims[3];      /* samples per axis, each <= 65535 */
  float iso;
  float origin[3];
  float spacing;
} DnrMcField;
/* Phase 1: counts_host[3] = {active cubes, triangles, vertices}; synchronises the stream (the one host read). */
int64_t dnr_mc_count_workspace_bytes(const DnrMcField* field);
int dnr_mc_count(const DnrMcField* field, void* ws, int64_t ws_bytes, int64_t* counts_host, void* stream);
/* Phase 2, with the count workspace as phase 1 left it: vertices [V,3], faces [F,3] int32, colors [V,3] in [0,1] (tsdf
 * only; may be NULL).  DNR_E_OVERFLOW past 2^31-1 vertices or faces. */
int64_t dnr_mc_emit_workspace_bytes(const int64_t* counts_host);
int dnr_mc_emit(const DnrMcField* field, const void* count_ws, const int64_t* counts_host, void* ws, int64_t ws_bytes,
                float* vertices, int32_t* faces, float* colors, void* stream);

/* ---- Screened Poisson reconstruction (Python surface: dn_splatter_b200.poisson; the discrete system is stated in
 * csrc/poisson.cu and DESIGN.md §2 (6)).  Dense grid of R = 2^depth cells per axis over a cube; chi lives at the cell
 * centres origin + (index + 0.5) * cell, node (i, j, k) at (i * R + j) * R + k. */
#define DNR_POISSON_MIN_DEPTH 4
#define DNR_POISSON_MAX_DEPTH 10
#define DNR_POISSON_MAX_CYCLES 100
typedef struct DnrPoissonGrid {
  float origin[3]; /* corner of cell (0, 0, 0) */
  float cell;      /* finest cell edge */
  int32_t depth;   /* DNR_POISSON_MIN_DEPTH..DNR_POISSON_MAX_DEPTH */
  int32_t reserved;
} DnrPoissonGrid;
/* Sorts the n oriented samples (points, normals [n,3]; colors [n,3] or NULL) by finest cell and gathers, per node:
 * screen [R^3] = S (sum of a_p * trilinear weight), faces [3,R^3] = the MAC face grids of the weighted normals (x, y,
 * z; face n lies between cell n and its +axis neighbour, the last one per axis is the wall and is 0), density
 * [(R/4)^3] = the count splat sum-restricted two levels, color_grid [(R/4)^3,4] = {sum a_p w c_p (rgb), sum a_p w} at
 * that level (NULL iff colors is NULL; the colour at a point is the ratio of the interpolated sums), weights [n] = a_p in input order (or NULL), area_scale [1] = 16 * mean(1 / rho).
 * Deterministic, no host synchronisation.  n <= 2^31-1. */
int64_t dnr_poisson_splat_workspace_bytes(const DnrPoissonGrid* grid, int64_t n_points);
int dnr_poisson_splat(const DnrPoissonGrid* grid, const float* points, const float* normals, const float* colors,
                      int64_t n_points, void* ws, int64_t ws_bytes, float* screen, float* faces, float* density,
                      float* color_grid, float* weights, float* area_scale, void* stream);
/* Solves (-Lap + screen_weight * S) chi = -div V (Neumann walls; mean(chi) = 0 when screen_weight == 0) by multigrid
 * V-cycles until ||b - A chi|| / ||b|| <= tol or max_cycles.  residual_host[0..cycles] (HOST) receives the relative
 * residual before the first and after every cycle, *cycles_host the cycle count; one host read per cycle. */
int64_t dnr_poisson_solve_workspace_bytes(const DnrPoissonGrid* grid, int32_t max_cycles);
int dnr_poisson_solve(const DnrPoissonGrid* grid, const float* screen, const float* faces, float screen_weight, float tol,
                      int32_t max_cycles, void* ws, int64_t ws_bytes, float* chi, float* residual_host,
                      int32_t* cycles_host, void* stream);
/* Cell-centred grid [dims[0], dims[1], dims[2], channels]: node (i, j, k) sits at origin + (index + 0.5) * cell. */
typedef struct DnrGridDesc {
  float origin[3];
  float cell;
  int32_t dims[3];
  int32_t channels;
} DnrGridDesc;
/* out[n, channels] = trilinear interpolation of the grid at points [n,3]; coordinates past the outer node centres are
 * clamped to them. */
int dnr_grid_sample(const DnrGridDesc* grid, const float* values, const float* points, int64_t n_points, float* out,
                    void* stream);

/* ---- Mesh evaluation (Python surface: dn_splatter_b200.mesh_eval; rules in csrc/mesh_eval.cu and DESIGN.md §2) ----
 * Camera blocks are the 16 numbers of dnr_tsdf_integrate's cam_host, {fx, fy, cx, cy, world->camera [3,4] row-major
 * (OpenCV)}, one per view, in DEVICE memory: float for dnr_mesh_depth, double for dnr_mesh_visibility.
 *
 * depth [n_views,H,W] = camera-space z of the nearest hit of the ray through pixel centre (i + 0.5, j + 0.5) with
 * near <= z <= far, both faces of every triangle, 0 where there is none.  Watertight on shared edges, bit-identical
 * between runs, no host synchronisation.  Faces with an out-of-range index are skipped. */
int64_t dnr_mesh_depth_workspace_bytes(int64_t n_faces);
int dnr_mesh_depth(const float* vertices /* [V,3] */, int32_t n_vertices, const int32_t* faces /* [F,3] */, int64_t n_faces,
                   const float* cams /* [n_views,16] */, int32_t n_views, int32_t width, int32_t height, float near, float far,
                   void* ws, int64_t ws_bytes, float* depth, void* stream);
/* Adds to obs / invalid [n] (int32) the counts of cull_from_one_pose over n_views views, projected in fp64: pz = z + 1e-8,
 * in frustum = 0 <= px <= W-1, 0 <= py <= H-1, pz > 0; observed = in frustum and pz < rendered + eps (fp32 sum), or in
 * frustum when rendered is NULL; invalid = in frustum and gt <= 0 (not counted when gt is NULL; invalid may then be NULL).
 * rendered / gt: [n_views,H,W] float. */
int dnr_mesh_visibility(const double* points /* [n,3] */, int64_t n_points, const double* cams /* [n_views,16] */,
                        const float* rendered, const float* gt, int32_t n_views, int32_t width, int32_t height, float eps,
                        int32_t* obs, int32_t* invalid, void* stream);

/* ---- Render evaluation (Python surface: dn_splatter_b200.metrics; rules in csrc/metrics.cu and DESIGN.md) ----
 * DepthMetrics (dn_splatter/metrics.py) over n pooled fp32 elements.  out[9] double (zeroed by the call), over the
 * elements with gt > tolerance: [0] their count; [1], [2], [3] the counts of thresh < 1.25, 1.25^2, 1.25^3, where
 * thresh = max(gt/pred, pred/gt) is formed in fp32 (NaN when either ratio is); [4] sum (gt-pred)^2; [5] sum |gt-pred|/gt;
 * [6] sum (gt-pred)^2/gt; [7] sum |log gt - log pred| over the terms that are not NaN; [8] the number of those terms.
 * Everything but the ratio test is evaluated in fp64. */
int dnr_depth_metrics(const float* pred, const float* gt, int64_t n, float tolerance, double* out, void* stream);
/* NormalMetrics (dn_splatter/metrics.py) of [B,H,W,3] maps: gt fp32, or uint8 read as value / 255 when gt_is_u8 != 0.
 * out[3B+1] double (zeroed by the call): per image b, [3b] sum acos(clamp(dot, -1, 1)) with the fp32
 * dot = (g0 p0 + g1 p1) + g2 p2, [3b+1] sum (g-p)^2, [3b+2] sum |g-p|; [3B] the lower median of the fp32 |g - p| over all
 * N = 3BHW values (the element of rank (N-1)/2, as torch.median returns it), found by a radix select over the fp32 bit
 * patterns without a host synchronisation.  ws: dnr_normal_metrics_workspace_bytes(B, H, W) bytes of device memory. */
int64_t dnr_normal_metrics_workspace_bytes(int32_t B, int32_t H, int32_t W);
int dnr_normal_metrics(const float* pred, const void* gt, int32_t gt_is_u8, int32_t B, int32_t H, int32_t W, void* ws,
                       int64_t ws_bytes, double* out, void* stream);

/* ---- AGS-Mesh isooctree extraction (Python surface: dn_splatter_b200.isooctree; rules in csrc/isooctree.cu and
 * DESIGN.md §2).  Everything that decides a sample or a value is evaluated in fp64.
 *
 * Frames: the depth and normal files of F views of one camera model (w x h, intrinsics K).  poses [F,DNR_ISO_POSE]
 * (DEVICE doubles) per view: world->camera [3,4], camera->world rotation [3,3], camera position [3], normal rotation
 * [3,3] (c2w rotation . diag(1, -1, -1), used when cam_normals != 0), all row-major, then 3 doubles of padding.  depth = file value * depth_scale;
 * normals are the file values: uint8 PNG values of camera-frame normals (cam_normals != 0) or world-frame floats. */
#define DNR_ISO_POSE 36
#define DNR_ISO_MAX_DEPTH 10
typedef struct DnrIsoFrames {
  const float* depth;   /* [F,h,w] */
  const float* normals; /* [F,h,w,3] */
  const double* poses;  /* [F,DNR_ISO_POSE] */
  int32_t n_frames, width, height, cam_normals;
  double K[9], inv_K[9]; /* row-major */
  double depth_scale;    /* 1/1000: millimetre files */
  double rel_delta;      /* max_valid_depth_rel_delta (0.005) */
} DnrIsoFrames;
typedef struct DnrIsoParams {
  double max_tsdf_rel;
  double max_tsdf_abs; /* +inf: no absolute cap */
  double min_dot;      /* cos(max_angle_to_max_weight_normal) */
  int32_t use_normals;
  int32_t passes; /* bit 0: a best-frame normal pass, bit 1: a fusion pass (3 = two-pass, 1 = choose_best_frame) */
} DnrIsoParams;
/* Octree over the hint cloud: root cube [origin, origin + cell * 2^max_depth)^3; a node splits iff it holds >= threshold
 * samples and its level < max_depth.  Leaves: int64 level << 58 | Morton code of the node at its level (bit 3b + 2 - a
 * is bit b of the axis-a coordinate), ordered by level, then code.  Lattice keys: (i * (R+1) + j) * (R+1) + k,
 * R = 2^max_depth, sample (i, j, k) at origin + (i, j, k) * cell. */
typedef struct DnrIsoGrid {
  double origin[3];
  double cell; /* finest cell edge */
  int32_t max_depth; /* 0..DNR_ISO_MAX_DEPTH */
  int32_t threshold; /* subdivision_threshold >= 1 */
} DnrIsoGrid;
/* The hint cloud (Frame.get_samples over all frames, in frame then row-major pixel order): points / normals (normals
 * may be NULL) [capacity,3] with capacity = F * ceil(h/stride) * ceil(w/stride); *count_host = the survivors.
 * Synchronises the stream (the one host read). */
int64_t dnr_iso_samples_workspace_bytes(const DnrIsoFrames* frames, int32_t stride);
int dnr_iso_samples(const DnrIsoFrames* frames, int32_t stride, void* ws, int64_t ws_bytes, double* points, double* normals,
                    int64_t* count_host, void* stream);
/* isoFunc at points [n,3]: values [n] (fp64 evaluation rounded to f32).  One thread per point, no host read. */
int dnr_iso_eval(const DnrIsoFrames* frames, const DnrIsoParams* params, const double* points, int64_t n, float* values,
                 void* stream);
/* Leaves of the octree of points [n,3], kept in ws; level_counts_host[max_depth + 1] = leaves per level.  One host read
 * per level. */
int64_t dnr_iso_octree_workspace_bytes(const DnrIsoGrid* grid, int64_t n_points);
int dnr_iso_octree(const DnrIsoGrid* grid, const double* points, int64_t n_points, void* ws, int64_t ws_bytes,
                   int64_t* level_counts_host, void* stream);
/* From dnr_iso_octree's workspace: leaves [L], the sorted unique corner lattice keys and their points (capacity 8L;
 * *n_corners_host are written), leaf_corners [L,8] = the index of corner (dx << 2 | dy << 1 | dz) of each leaf. */
int64_t dnr_iso_corners_workspace_bytes(const DnrIsoGrid* grid, int64_t n_leaves);
int dnr_iso_corners(const DnrIsoGrid* grid, const void* octree_ws, const int64_t* level_counts_host, void* ws, int64_t ws_bytes,
                    int64_t* leaves, int64_t* corner_keys, double* corner_points, int32_t* leaf_corners,
                    int64_t* n_corners_host, void* stream);
/* field [(R+1)^3] f32: every sample takes the value of the smallest leaf whose closed cube holds it, the lerp of lerps
 * (x, then y, then z) of that leaf's corner values, which a corner sample reproduces exactly. */
int dnr_iso_fill(const DnrIsoGrid* grid, const int64_t* leaves, const int64_t* level_counts_host, const int32_t* leaf_corners,
                 const float* corner_values, float* field, void* stream);

/* ---- AGS-Mesh depth confidence masks: scripts/depth_normal_consistency.py and depth_to_normal.py (DESIGN.md §2 (9)) ---- */
#define DNR_DN_MAX_K 256
#define DNR_DN_OMNIDATA 0         /* DepthNormalConsistency, normal_format "omnidata" */
#define DNR_DN_DSINE 1            /* DepthNormalConsistency, normal_format "dsine" */
#define DNR_DN_DEPTH_TO_NORMAL 2  /* DepthToNormal: the angle between the encoded vectors */
/* A 3x3 matrix (row-major) and a translation.  dnr_dn_backproject: world = cam @ rinv + t with rinv = inv(c2w[:3,:3]);
 * dnr_dn_consistency: rinv holds R = transpose(inv(c2w)[:3,:3]), the mono normal's rotation, and t is unused. */
typedef struct DnrDnPose {
  double rinv[9];
  double t[3];
} DnrDnPose;
/* The neighbour search: k in [1, DNR_DN_MAX_K]; the Morton grid spans lo + [0, 2^21 cell) per axis (points outside are
 * clamped into the border cells); with orient != 0 a normal n of point p is negated where (p - center) . n > 0. */
typedef struct DnrDnSearch {
  double lo[3];
  double cell;
  double center[3];
  int32_t k;
  int32_t orient;
} DnrDnSearch;
/* points [w*h,3] f64 of a depth frame [h,w] f32 (intrinsics_host = fx, fy, cx, cy as f32); cam_points [w*h,3] f32, the
 * camera coordinates, may be NULL. */
int dnr_dn_backproject(const float* depth, int32_t width, int32_t height, const float* intrinsics_host, const DnrDnPose* pose,
                       float* cam_points, double* points, void* stream);
/* normals [n,3] f64 of points [n,3] f64 (Open3D's estimate_normals, KNN k, fast_normal_computation) [EXT].  Optional
 * outputs (NULL: not written): examined [n] the candidates the search of each point's position examined; stats (device,
 * 2 x u64) += (candidates examined, searches run), one search per distinct position; for tests, cov [n,9] the covariance of
 * each point's neighbours and neighbours [n,k] the smallest point index of each neighbour's position, one entry per copy
 * taken, -1 past min(k, n). */
int64_t dnr_dn_normals_workspace_bytes(int64_t n_points);
int dnr_dn_normals(const double* points, int64_t n_points, const DnrDnSearch* search, void* ws, int64_t ws_bytes, double* normals,
                   int32_t* examined, double* cov, int32_t* neighbours, unsigned long long* stats, void* stream);
/* Per pixel of oriented normals [n,3] and the mono-normal PNG values mono [n,3] u8: the angle in degrees, mask = 255 where it
 * exceeds threshold else 0, and normals_u8 [n,3] = uint8((n + 1) / 2 * 255). */
int dnr_dn_consistency(const double* normals, const uint8_t* mono, int64_t n, const DnrDnPose* rotation, int32_t mode,
                       double threshold, double* degrees, uint8_t* mask, uint8_t* normals_u8, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DNR_H_ */
