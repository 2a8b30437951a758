// Per-Gaussian projection, forward and backward.  Compiled with -fmad=false: the forward's float
// operation order is the contract that makes radii / tile boxes / sort keys bit-identical to the
// oracle (oracle/gsplat_ref.py::project_gaussians).  One thread per Gaussian; the kernel is a pure
// HBM stream (44 B in, ~130 B out per Gaussian forward; ~300 B out backward at 16 SH bases).
//
// Replaces (reference, /root/reference/dn_splatter/dn_model.py):
//   :496-500  quats/|quats|, exp(scales), sigmoid(opacities)            (activations)
//   :495-516  gsplat fully_fused_projection + spherical_harmonics       [EXT gsplat 1.0.0]
//   :543-560  per-Gaussian normal: column argmin(scale) of R(q), flip toward camera, rotate to camera
#include "common.cuh"

namespace {

struct Cam {
  float W[3][3];
  float t[3];
  float fx, fy, cx, cy;
  float campos[3];   // -R^T t  (== inverse(viewmat)[:3,3])
  float c2wR[3][3];  // nerfstudio c2w rotation (normals)
  float c2wT[3];
};

__device__ __forceinline__ void load_cam(const DnrArgs& a, Cam& c) {
  const bool host = (a.flags & DNR_FLAG_HOST_CAMERA) != 0;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int j = 0; j < 3; ++j) c.W[i][j] = host ? a.host_cam[i * 4 + j] : __ldg(a.viewmat + i * 4 + j);
    c.t[i] = host ? a.host_cam[i * 4 + 3] : __ldg(a.viewmat + i * 4 + 3);
  }
  c.fx = host ? a.host_cam[16] : __ldg(a.K + 0);
  c.fy = host ? a.host_cam[17] : __ldg(a.K + 4);
  c.cx = host ? a.host_cam[18] : __ldg(a.K + 2);
  c.cy = host ? a.host_cam[19] : __ldg(a.K + 5);
#pragma unroll
  for (int j = 0; j < 3; ++j) c.campos[j] = -((c.W[0][j] * c.t[0] + c.W[1][j] * c.t[1]) + c.W[2][j] * c.t[2]);
  if (host || a.c2w != nullptr) {
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
      for (int j = 0; j < 3; ++j) c.c2wR[i][j] = host ? a.host_cam[20 + i * 4 + j] : __ldg(a.c2w + i * 4 + j);
      c.c2wT[i] = host ? a.host_cam[20 + i * 4 + 3] : __ldg(a.c2w + i * 4 + 3);
    }
  }
}

__device__ __forceinline__ float dot3(float a0, float b0, float a1, float b1, float a2, float b2) {
  return (a0 * b0 + a1 * b1) + a2 * b2;
}

__device__ __forceinline__ void quat_rot(const float q[4], float R[3][3], float qn[4], float& inv_norm) {
  const float n2 = ((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3];
  inv_norm = 1.0f / sqrtf(n2);
  const float w = q[0] * inv_norm, x = q[1] * inv_norm, y = q[2] * inv_norm, z = q[3] * inv_norm;
  qn[0] = w; qn[1] = x; qn[2] = y; qn[3] = z;
  const float x2 = x * x, y2 = y * y, z2 = z * z;
  const float xy = x * y, xz = x * z, yz = y * z, wx = w * x, wy = w * y, wz = w * z;
  R[0][0] = 1.0f - 2.0f * (y2 + z2); R[0][1] = 2.0f * (xy - wz);        R[0][2] = 2.0f * (xz + wy);
  R[1][0] = 2.0f * (xy + wz);        R[1][1] = 1.0f - 2.0f * (x2 + z2); R[1][2] = 2.0f * (yz - wx);
  R[2][0] = 2.0f * (xz - wy);        R[2][1] = 2.0f * (yz + wx);        R[2][2] = 1.0f - 2.0f * (x2 + y2);
}

// SH basis values for a unit direction (Sloan's polynomial form; gsplat spherical_harmonics [EXT]).
__device__ __forceinline__ void sh_basis(int degree, float x, float y, float z, float b[16]) {
#pragma unroll
  for (int k = 1; k < 16; ++k) b[k] = 0.f;
  b[0] = 0.2820947917738781f;
  if (degree < 1) return;
  b[1] = -0.48860251190292f * y;
  b[2] = 0.48860251190292f * z;
  b[3] = -0.48860251190292f * x;
  if (degree < 2) return;
  const float z2 = z * z;
  const float fTmp0B = -1.092548430592079f * z;
  const float fC1 = x * x - y * y;
  const float fS1 = 2.0f * x * y;
  b[6] = 0.9461746957575601f * z2 - 0.3153915652525201f;
  b[7] = fTmp0B * x;
  b[5] = fTmp0B * y;
  b[8] = 0.5462742152960395f * fC1;
  b[4] = 0.5462742152960395f * fS1;
  if (degree < 3) return;
  const float fTmp0C = -2.285228997322329f * z2 + 0.4570457994644658f;
  const float fTmp1B = 1.445305721320277f * z;
  const float fC2 = x * fC1 - y * fS1;
  const float fS2 = x * fS1 + y * fC1;
  b[12] = z * (1.865881662950577f * z2 - 1.119528997770346f);
  b[13] = fTmp0C * x;
  b[11] = fTmp0C * y;
  b[14] = fTmp1B * fC1;
  b[10] = fTmp1B * fS1;
  b[15] = -0.5900435899266435f * fC2;
  b[9] = -0.5900435899266435f * fS2;
}

// d(basis_k)/d(x,y,z) contracted with per-basis weights g[k] = sum_c coeff[k][c] * v_c.
__device__ __forceinline__ void sh_basis_vjp(int degree, float x, float y, float z, const float g[16], float v[3]) {
  v[0] = v[1] = v[2] = 0.f;
  if (degree < 1) return;
  v[1] += -0.48860251190292f * g[1];
  v[2] += 0.48860251190292f * g[2];
  v[0] += -0.48860251190292f * g[3];
  if (degree < 2) return;
  const float z2 = z * z;
  const float fTmp0B = -1.092548430592079f * z;
  const float fC1 = x * x - y * y;
  const float fS1 = 2.0f * x * y;
  // b4 = c*fS1, b5 = fTmp0B*y, b6 = a z2 - k, b7 = fTmp0B*x, b8 = c*fC1
  v[0] += 0.5462742152960395f * 2.0f * y * g[4] + fTmp0B * g[7] + 0.5462742152960395f * 2.0f * x * g[8];
  v[1] += 0.5462742152960395f * 2.0f * x * g[4] + fTmp0B * g[5] - 0.5462742152960395f * 2.0f * y * g[8];
  v[2] += -1.092548430592079f * y * g[5] + 2.0f * 0.9461746957575601f * z * g[6] - 1.092548430592079f * x * g[7];
  if (degree < 3) return;
  const float fTmp0C = -2.285228997322329f * z2 + 0.4570457994644658f;
  const float fTmp1B = 1.445305721320277f * z;
  const float fC2 = x * fC1 - y * fS1;
  const float fS2 = x * fS1 + y * fC1;
  (void)fC2; (void)fS2;
  // dfC1 = (2x,-2y,0) dfS1 = (2y,2x,0); dfC2 = (fC1 + x*2x - y*2y, -2xy - fS1 ... )
  const float dC2x = fC1 + x * 2.0f * x - y * 2.0f * y;   // 3(x^2-y^2)
  const float dC2y = -x * 2.0f * y - fS1 - y * 2.0f * x;   // -6xy
  const float dS2x = fS1 + x * 2.0f * y + y * 2.0f * x;    // 6xy
  const float dS2y = x * 2.0f * x + fC1 - y * 2.0f * y;    // 3(x^2-y^2)
  const float dT0Cz = -2.285228997322329f * 2.0f * z;
  // b9 = k*fS2, b10 = fTmp1B*fS1, b11 = fTmp0C*y, b12 = z(a z2 - b), b13 = fTmp0C*x, b14 = fTmp1B*fC1, b15 = k*fC2
  const float k = -0.5900435899266435f;
  v[0] += k * dS2x * g[9] + fTmp1B * 2.0f * y * g[10] + fTmp0C * g[13] + fTmp1B * 2.0f * x * g[14] + k * dC2x * g[15];
  v[1] += k * dS2y * g[9] + fTmp1B * 2.0f * x * g[10] + fTmp0C * g[11] - fTmp1B * 2.0f * y * g[14] + k * dC2y * g[15];
  v[2] += 1.445305721320277f * fS1 * g[10] + dT0Cz * y * g[11] +
          (3.0f * 1.865881662950577f * z2 - 1.119528997770346f) * g[12] + dT0Cz * x * g[13] +
          1.445305721320277f * fC1 * g[14];
}

struct Geo {  // forward intermediates reused by the backward
  float R[3][3];   // R(q)
  float qn[4];
  float inv_qnorm;
  float s[3];      // activated scales
  float mc[3];     // camera-space mean
  float Sc[3][3];  // camera covariance
  float M[3][3];   // R diag(s)
  float rz, rz2, tx, ty;
  bool clamp_x, clamp_y;  // x*rz outside [-lim,lim]
  float a, b, c;   // blurred 2-D covariance
  float det, det_orig, comp;
  float mx, my;
  int radius;
  bool ok;
};

__device__ __forceinline__ void forward_geo(const DnrArgs& a, const Cam& cam, int i, Geo& g) {
  const float px = a.means[i * 3 + 0], py = a.means[i * 3 + 1], pz = a.means[i * 3 + 2];
  const float4 q4 = reinterpret_cast<const float4*>(a.quats)[i];
  const float q[4] = {q4.x, q4.y, q4.z, q4.w};
  const bool act = (a.flags & DNR_FLAG_ACTIVATED) != 0;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float s = a.scales[i * 3 + k];
    g.s[k] = act ? s : expf(s);
  }
  g.mc[0] = dot3(cam.W[0][0], px, cam.W[0][1], py, cam.W[0][2], pz) + cam.t[0];
  g.mc[1] = dot3(cam.W[1][0], px, cam.W[1][1], py, cam.W[1][2], pz) + cam.t[1];
  g.mc[2] = dot3(cam.W[2][0], px, cam.W[2][1], py, cam.W[2][2], pz) + cam.t[2];
  const float x = g.mc[0], y = g.mc[1], z = g.mc[2];
  g.ok = (z >= a.near_plane) && (z <= a.far_plane);
  quat_rot(q, g.R, g.qn, g.inv_qnorm);
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) g.M[r][c] = g.R[r][c] * g.s[c];
  float S[3][3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = r; c < 3; ++c) {
      S[r][c] = dot3(g.M[r][0], g.M[c][0], g.M[r][1], g.M[c][1], g.M[r][2], g.M[c][2]);
      S[c][r] = S[r][c];
    }
  float A[3][3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) A[r][c] = dot3(cam.W[r][0], S[0][c], cam.W[r][1], S[1][c], cam.W[r][2], S[2][c]);
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = r; c < 3; ++c) {
      g.Sc[r][c] = dot3(A[r][0], cam.W[c][0], A[r][1], cam.W[c][1], A[r][2], cam.W[c][2]);
      g.Sc[c][r] = g.Sc[r][c];
    }
  const float tan_fovx = (0.5f * (float)a.width) / cam.fx;
  const float tan_fovy = (0.5f * (float)a.height) / cam.fy;
  const float lim_x = 1.3f * tan_fovx, lim_y = 1.3f * tan_fovy;
  const float zs = g.ok ? z : 1.0f;
  g.rz = 1.0f / zs;
  g.rz2 = g.rz * g.rz;
  const float xr = x * g.rz, yr = y * g.rz;
  g.clamp_x = !(xr <= lim_x && xr >= -lim_x);
  g.clamp_y = !(yr <= lim_y && yr >= -lim_y);
  g.tx = zs * fminf(lim_x, fmaxf(-lim_x, xr));
  g.ty = zs * fminf(lim_y, fmaxf(-lim_y, yr));
  const float J00 = cam.fx * g.rz, J02 = -(cam.fx * g.tx) * g.rz2;
  const float J11 = cam.fy * g.rz, J12 = -(cam.fy * g.ty) * g.rz2;
  const float B00 = J00 * g.Sc[0][0] + J02 * g.Sc[2][0];
  const float B01 = J00 * g.Sc[0][1] + J02 * g.Sc[2][1];
  const float B02 = J00 * g.Sc[0][2] + J02 * g.Sc[2][2];
  const float B11 = J11 * g.Sc[1][1] + J12 * g.Sc[2][1];
  const float B12 = J11 * g.Sc[1][2] + J12 * g.Sc[2][2];
  float ca = B00 * J00 + B02 * J02;
  const float cb = B01 * J11 + B02 * J12;
  float cc = B11 * J11 + B12 * J12;
  g.mx = (cam.fx * x) * g.rz + cam.cx;
  g.my = (cam.fy * y) * g.rz + cam.cy;
  g.det_orig = ca * cc - cb * cb;
  ca = ca + a.eps2d;
  cc = cc + a.eps2d;
  g.det = ca * cc - cb * cb;
  g.a = ca; g.b = cb; g.c = cc;
  const bool ok_det = g.det > 0.f;
  const float dets = ok_det ? g.det : 1.0f;
  g.comp = sqrtf(fmaxf(g.det_orig / dets, 0.0f));
  g.det = dets;
  const float mid = 0.5f * (ca + cc);
  const float lam = mid + sqrtf(fmaxf(mid * mid - dets, 0.01f));
  const float radius = ceilf(3.0f * sqrtf(lam));
  g.ok = g.ok && ok_det && (radius > a.radius_clip);
  const bool outside = (g.mx + radius <= 0.f) || (g.mx - radius >= (float)a.width) || (g.my + radius <= 0.f) ||
                       (g.my - radius >= (float)a.height);
  g.ok = g.ok && !outside;
  g.radius = g.ok ? (int)radius : 0;
}

__device__ __forceinline__ int argmin3(float s0, float s1, float s2) {
  int idx = 0;
  float m = s0;
  if (s1 < m) { m = s1; idx = 1; }
  if (s2 < m) { idx = 2; }
  return idx;
}

// Sign of the per-Gaussian normal: -1 when the unit normal n faces away from the camera (its dot product with the
// normalised view vector vd = campos - mean is negative).  The forward and the backward both take it from here: for a
// Gaussian seen edge-on the dot product is ~0, and a differently rounded expression in the backward would differentiate
// the normal with the opposite sign from the one that was rendered.
__device__ __forceinline__ float normal_sign(const float n[3], const float vd[3]) {
  const float vn = sqrtf((vd[0] * vd[0] + vd[1] * vd[1]) + vd[2] * vd[2]);
  const float d = (n[0] * (vd[0] / vn) + n[1] * (vd[1] / vn)) + n[2] * (vd[2] / vn);
  return d < 0.f ? -1.0f : 1.0f;
}

template <bool NORMALS>
__global__ void __launch_bounds__(256) project_fwd_kernel(const DnrArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n_gauss) return;
  Cam cam;
  load_cam(a, cam);
  Geo g;
  forward_geo(a, cam, i, g);
  constexpr int REC = NORMALS ? DNR_REC_FLOATS_N : DNR_REC_FLOATS;
  float4* rec = reinterpret_cast<float4*>(a.records + (size_t)i * REC);

  // world normal (side output even for culled Gaussians: gauss_params["normals"], dn_model.py:558)
  float nw[3] = {0.f, 0.f, 0.f}, nc[3] = {0.f, 0.f, 0.f};
  if (NORMALS) {
    const int idx = argmin3(a.scales[i * 3 + 0], a.scales[i * 3 + 1], a.scales[i * 3 + 2]);
    float n[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) n[r] = idx == 0 ? g.R[r][0] : (idx == 1 ? g.R[r][1] : g.R[r][2]);
    const float nn = fmaxf(sqrtf((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2]), 1e-12f);
    float vd[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      n[k] = n[k] / nn;
      vd[k] = cam.c2wT[k] - a.means[i * 3 + k];
    }
    const float sgn = normal_sign(n, vd);
#pragma unroll
    for (int k = 0; k < 3; ++k) nw[k] = sgn * n[k];
#pragma unroll
    for (int j = 0; j < 3; ++j) nc[j] = (nw[0] * cam.c2wR[0][j] + nw[1] * cam.c2wR[1][j]) + nw[2] * cam.c2wR[2][j];
    if (a.normals_world != nullptr) {
      a.normals_world[i * 3 + 0] = nw[0];
      a.normals_world[i * 3 + 1] = nw[1];
      a.normals_world[i * 3 + 2] = nw[2];
    }
  }

  if (!g.ok) {
    a.radii[i] = 0;
    a.tiles_per_gauss[i] = 0;
    a.depth_keys[i] = 0xFFFFFFFFu;
    a.means2d[i * 2 + 0] = 0.f; a.means2d[i * 2 + 1] = 0.f;
    a.depths[i] = 0.f;
    a.conics[i * 3 + 0] = 0.f; a.conics[i * 3 + 1] = 0.f; a.conics[i * 3 + 2] = 0.f;
    a.opac_act[i] = 0.f;
    if (a.cull_lim) a.cull_lim[i] = -1.0f;
    if (a.compensations) a.compensations[i] = 0.f;
    a.colors[i * 3 + 0] = 0.f; a.colors[i * 3 + 1] = 0.f; a.colors[i * 3 + 2] = 0.f;
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    rec[0] = z4; rec[1] = z4; rec[2] = z4;
    if (NORMALS) rec[3] = z4;
    return;
  }
  const float inv_det = 1.0f / g.det;
  const float conA = g.c * inv_det, conB = -(g.b * inv_det), conC = g.a * inv_det;
  float op = a.opacities[i];
  if (!(a.flags & DNR_FLAG_ACTIVATED)) op = 1.0f / (1.0f + expf(-op));
  // largest sigma at which a pixel can still pass alpha >= 1/255 (pre-compensation opacity: conservative for both modes)
  if (a.cull_lim) a.cull_lim[i] = logf(255.0f * op) + DNR_CULL_MARGIN;
  if (a.flags & DNR_FLAG_ANTIALIASED) op = op * g.comp;

  // SH colour: clamp_min(SH(dir) + 0.5, 0)
  float dir[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) dir[k] = a.means[i * 3 + k] - cam.campos[k];
  float basis[16];
  const int deg = a.sh_degree;
  if (deg > 0) {
    const float inorm = 1.0f / sqrtf((dir[0] * dir[0] + dir[1] * dir[1]) + dir[2] * dir[2]);
    sh_basis(deg, dir[0] * inorm, dir[1] * inorm, dir[2] * inorm, basis);
  } else {
    sh_basis(0, 0.f, 0.f, 1.f, basis);
  }
  const int nb = (deg + 1) * (deg + 1);
  float col[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) col[c] = basis[0] * a.sh_dc[i * 3 + c];
  const float* rest = a.sh_rest + (size_t)i * (a.sh_bases - 1) * 3;
#pragma unroll
  for (int k = 1; k < 16; ++k) {
    if (k < nb) {
#pragma unroll
      for (int c = 0; c < 3; ++c) col[c] += basis[k] * rest[(k - 1) * 3 + c];
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) col[c] = fmaxf(col[c] + 0.5f, 0.0f);

  int x0, y0, x1, y1;
  dnr_tile_box(g.mx, g.my, g.radius, (a.width + DNR_TILE - 1) / DNR_TILE, (a.height + DNR_TILE - 1) / DNR_TILE, x0, y0, x1, y1);
  a.radii[i] = g.radius;
  a.tiles_per_gauss[i] = (x1 - x0) * (y1 - y0);
  a.depth_keys[i] = __float_as_uint(g.mc[2]);
  a.means2d[i * 2 + 0] = g.mx; a.means2d[i * 2 + 1] = g.my;
  a.depths[i] = g.mc[2];
  a.conics[i * 3 + 0] = conA; a.conics[i * 3 + 1] = conB; a.conics[i * 3 + 2] = conC;
  a.opac_act[i] = op;
  if (a.compensations) a.compensations[i] = g.comp;
  a.colors[i * 3 + 0] = col[0]; a.colors[i * 3 + 1] = col[1]; a.colors[i * 3 + 2] = col[2];
  // raster record: log2-domain conic (see dnr_power2), opacity, and -log2(255*op) - slack: the cheap in-loop
  // pre-test "power < nthr => alpha < 1/255" (the exact alpha test still decides; 1e-3 slack keeps it conservative)
  const float nthr = -log2f(255.0f * op) - 1e-3f;
  rec[0] = make_float4(g.mx, g.my, (-0.5f * DNR_LOG2E) * conA, (-DNR_LOG2E) * conB);
  rec[1] = make_float4((-0.5f * DNR_LOG2E) * conC, op, nthr, (float)g.radius);  // radius: the raster kernels' tile-box test
  rec[2] = make_float4(col[0], col[1], col[2], g.mc[2]);
  if (NORMALS) rec[3] = make_float4(nc[0], nc[1], nc[2], 0.f);
}

// ------------------------------------------------------------------------------------------------
// backward: raster-gradient record -> parameter gradients (gsplat fully_fused_projection_bwd +
// spherical_harmonics bwd + activation / normal chain rules).
// ------------------------------------------------------------------------------------------------
constexpr int PB_THREADS = 128;   // Gaussians per CTA in project_bwd
constexpr int PB_REST_MAX = 45;    // (16 - 1) * 3 floats of higher-order SH gradient per Gaussian

// Parameter gradients of ONE visible Gaussian from its raster-gradient record: gsplat fully_fused_projection_bwd +
// spherical_harmonics bwd + activation / normal chain rules.  The 3*(sh_bases-1) higher-order SH gradients go to `srow`
// (shared memory staging, written out by the caller); the rest is returned in registers.
// VIEWMAT: also ADDS this Gaussian's d(loss)/d(viewmat) to pv[k * PB_THREADS], k over {v_W row-major [9], v_t [3]} (the
// thread's column of a shared-memory accumulator: keeps 12 sums out of the register budget).  With mc = W p + t,
// Sc = W S W^T and dir = p - campos = p + W^T t:
//   v_W += vmc p^T + 2 vSc W S + t vdir^T,   v_t += vmc + W vdir
// (vSc is symmetric; the normals' c2w is a separate, un-optimised input and contributes nothing).
template <bool NORMALS, bool VIEWMAT = false>
__device__ __forceinline__ void project_bwd_gauss(const DnrArgs& a, int i, int nrest, float* srow, float vm[3], float vq[4],
                                                  float vs[3], float& vo, float vdc[3], float* pv = nullptr) {
  Cam cam;
  load_cam(a, cam);
  Geo g;
  forward_geo(a, cam, i, g);
  const float4* gr = reinterpret_cast<const float4*>(a.grad_records + (size_t)i * DNR_GRAD_FLOATS);
  const float4 g0 = gr[0], g1 = gr[1], g2 = gr[2], g3 = gr[3];
  const float v_mx = g0.x, v_my = g0.y;
  const float v_conA = g1.x, v_conB = g1.y, v_conC = g1.z, v_op = g1.w;
  const float v_col[3] = {g2.x, g2.y, g2.z};
  const float v_depth = g2.w;
  if (a.v_means2d) { a.v_means2d[i * 2] = v_mx; a.v_means2d[i * 2 + 1] = v_my; }
  if (a.v_means2d_abs) { a.v_means2d_abs[i * 2] = g0.z; a.v_means2d_abs[i * 2 + 1] = g0.w; }

  // ---- opacity ----
  const bool act = (a.flags & DNR_FLAG_ACTIVATED) != 0;
  const float o_in = a.opacities[i];
  const float sig = act ? o_in : 1.0f / (1.0f + expf(-o_in));
  float v_comp = 0.f;
  float v_sig = v_op;
  if (a.flags & DNR_FLAG_ANTIALIASED) { v_comp = v_op * sig; v_sig = v_op * g.comp; }
  vo = act ? v_sig : v_sig * sig * (1.0f - sig);

  // ---- conic -> blurred 2-D covariance:  V2 = -Q G Q ----
  const float inv_det = 1.0f / g.det;
  const float qa = g.c * inv_det, qb = -(g.b * inv_det), qc = g.a * inv_det;  // Q = [[qa,qb],[qb,qc]]
  const float Ga = v_conA, Gb = 0.5f * v_conB, Gc = v_conC;
  // T = G Q
  const float t00 = Ga * qa + Gb * qb, t01 = Ga * qb + Gb * qc, t10 = Gb * qa + Gc * qb, t11 = Gb * qb + Gc * qc;
  float V00 = -(qa * t00 + qb * t10), V01 = -(qa * t01 + qb * t11), V11 = -(qb * t01 + qc * t11);
  if ((a.flags & DNR_FLAG_ANTIALIASED) && g.comp > 0.f) {
    // comp^2 = det_orig/det_blur ; d(comp^2)/dS2 = (1-comp^2) Q - eps det(Q) I
    const float v_c2 = v_comp * 0.5f / g.comp;
    const float om = 1.0f - g.comp * g.comp;
    const float detQ = qa * qc - qb * qb;
    V00 += v_c2 * (om * qa - a.eps2d * detQ);
    V01 += v_c2 * (om * qb);
    V11 += v_c2 * (om * qc - a.eps2d * detQ);
  }
  // ---- cov2d = J Sc J^T ----
  const float x = g.mc[0], y = g.mc[1];
  const float fx = cam.fx, fy = cam.fy;
  const float J[2][3] = {{fx * g.rz, 0.f, -(fx * g.tx) * g.rz2}, {0.f, fy * g.rz, -(fy * g.ty) * g.rz2}};
  const float V[2][2] = {{V00, V01}, {V01, V11}};
  // v_Sc = J^T V J
  float VJ[2][3];
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) VJ[r][c] = V[r][0] * J[0][c] + V[r][1] * J[1][c];
  float vSc[3][3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) vSc[r][c] = J[0][r] * VJ[0][c] + J[1][r] * VJ[1][c];
  // v_J = 2 V J Sc
  float vJ[2][3];
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c)
      vJ[r][c] = 2.0f * (VJ[r][0] * g.Sc[0][c] + VJ[r][1] * g.Sc[1][c] + VJ[r][2] * g.Sc[2][c]);
  float vmc[3];
  const float rz3 = g.rz2 * g.rz;
  vmc[0] = fx * g.rz * v_mx;
  vmc[1] = fy * g.rz * v_my;
  vmc[2] = -(fx * x * v_mx + fy * y * v_my) * g.rz2;
  vmc[2] += -fx * g.rz2 * vJ[0][0] - fy * g.rz2 * vJ[1][1] + 2.0f * fx * g.tx * rz3 * vJ[0][2] + 2.0f * fy * g.ty * rz3 * vJ[1][2];
  if (!g.clamp_x) vmc[0] += -fx * g.rz2 * vJ[0][2]; else vmc[2] += -fx * rz3 * vJ[0][2] * g.tx;
  if (!g.clamp_y) vmc[1] += -fy * g.rz2 * vJ[1][2]; else vmc[2] += -fy * rz3 * vJ[1][2] * g.ty;
  vmc[2] += v_depth;
  // ---- world <- camera ----
#pragma unroll
  for (int k = 0; k < 3; ++k) vm[k] = cam.W[0][k] * vmc[0] + cam.W[1][k] * vmc[1] + cam.W[2][k] * vmc[2];
  // v_S = W^T vSc W
  float tmp[3][3], vS[3][3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) tmp[r][c] = vSc[r][0] * cam.W[0][c] + vSc[r][1] * cam.W[1][c] + vSc[r][2] * cam.W[2][c];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) vS[r][c] = cam.W[0][r] * tmp[0][c] + cam.W[1][r] * tmp[1][c] + cam.W[2][r] * tmp[2][c];
  if constexpr (VIEWMAT) {
    // v_W += vmc p^T + 2 (vSc W) M M^T ;  v_t += vmc
    const float p[3] = {a.means[i * 3 + 0], a.means[i * 3 + 1], a.means[i * 3 + 2]};
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      float u[3];
#pragma unroll
      for (int j = 0; j < 3; ++j) u[j] = tmp[r][0] * g.M[0][j] + tmp[r][1] * g.M[1][j] + tmp[r][2] * g.M[2][j];
#pragma unroll
      for (int c = 0; c < 3; ++c)
        pv[(r * 3 + c) * PB_THREADS] += vmc[r] * p[c] + 2.0f * (u[0] * g.M[c][0] + u[1] * g.M[c][1] + u[2] * g.M[c][2]);
      pv[(9 + r) * PB_THREADS] += vmc[r];
    }
  }
  // v_M = (vS + vS^T) M
  float vM[3][3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c)
      vM[r][c] = (vS[r][0] + vS[0][r]) * g.M[0][c] + (vS[r][1] + vS[1][r]) * g.M[1][c] + (vS[r][2] + vS[2][r]) * g.M[2][c];
  float vR[3][3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) vR[r][c] = vM[r][c] * g.s[c];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float v_s = g.R[0][c] * vM[0][c] + g.R[1][c] * vM[1][c] + g.R[2][c] * vM[2][c];
    vs[c] = act ? v_s : v_s * g.s[c];
  }
  // ---- per-Gaussian normal -> R column ----
  if (NORMALS) {
    const float v_nc[3] = {g3.x, g3.y, g3.z};
    const int idx = argmin3(a.scales[i * 3 + 0], a.scales[i * 3 + 1], a.scales[i * 3 + 2]);
    float n[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) n[r] = idx == 0 ? g.R[r][0] : (idx == 1 ? g.R[r][1] : g.R[r][2]);
    const float nn = fmaxf(sqrtf(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]), 1e-12f);
    float vd[3], nu[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) { nu[k] = n[k] / nn; vd[k] = cam.c2wT[k] - a.means[i * 3 + k]; }
    const float sgn = normal_sign(nu, vd);
    float vnw[3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
      vnw[r] = sgn * (cam.c2wR[r][0] * v_nc[0] + cam.c2wR[r][1] * v_nc[1] + cam.c2wR[r][2] * v_nc[2]);
    const float dp = nu[0] * vnw[0] + nu[1] * vnw[1] + nu[2] * vnw[2];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const float vcol = (vnw[r] - nu[r] * dp) / nn;
      if (idx == 0) vR[r][0] += vcol; else if (idx == 1) vR[r][1] += vcol; else vR[r][2] += vcol;
    }
  }
  // ---- R(q) -> q (normalised) -> raw q ----
  {
    const float w = g.qn[0], qx = g.qn[1], qy = g.qn[2], qz = g.qn[3];
    float vqn[4];
    vqn[0] = 2.0f * (qx * (vR[2][1] - vR[1][2]) + qy * (vR[0][2] - vR[2][0]) + qz * (vR[1][0] - vR[0][1]));
    vqn[1] = 2.0f * (-2.0f * qx * (vR[1][1] + vR[2][2]) + qy * (vR[1][0] + vR[0][1]) + qz * (vR[2][0] + vR[0][2]) + w * (vR[2][1] - vR[1][2]));
    vqn[2] = 2.0f * (qx * (vR[1][0] + vR[0][1]) - 2.0f * qy * (vR[0][0] + vR[2][2]) + qz * (vR[2][1] + vR[1][2]) + w * (vR[0][2] - vR[2][0]));
    vqn[3] = 2.0f * (qx * (vR[2][0] + vR[0][2]) + qy * (vR[2][1] + vR[1][2]) - 2.0f * qz * (vR[0][0] + vR[1][1]) + w * (vR[1][0] - vR[0][1]));
    const float dp = g.qn[0] * vqn[0] + g.qn[1] * vqn[1] + g.qn[2] * vqn[2] + g.qn[3] * vqn[3];
#pragma unroll
    for (int k = 0; k < 4; ++k) vq[k] = (vqn[k] - g.qn[k] * dp) * g.inv_qnorm;
  }
  // ---- SH ----
  {
    float dir[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) dir[k] = a.means[i * 3 + k] - cam.campos[k];
    const int deg = a.sh_degree;
    const int nb = (deg + 1) * (deg + 1);
    float basis[16];
    float inorm = 1.f, ux = 0.f, uy = 0.f, uz = 1.f;
    if (deg > 0) {
      inorm = 1.0f / sqrtf(dir[0] * dir[0] + dir[1] * dir[1] + dir[2] * dir[2]);
      ux = dir[0] * inorm; uy = dir[1] * inorm; uz = dir[2] * inorm;
    }
    sh_basis(deg, ux, uy, uz, basis);
    const float* rest = a.sh_rest + (size_t)i * nrest * 3;
    // clamp mask: recompute the pre-clamp colour
    float col[3], gk[16];
#pragma unroll
    for (int c = 0; c < 3; ++c) col[c] = basis[0] * a.sh_dc[i * 3 + c];
#pragma unroll
    for (int k = 1; k < 16; ++k) {
      if (k < nb) {
#pragma unroll
        for (int c = 0; c < 3; ++c) col[c] += basis[k] * rest[(k - 1) * 3 + c];
      }
    }
    float vc[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) vc[c] = (col[c] + 0.5f >= 0.0f) ? v_col[c] : 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) vdc[c] = basis[0] * vc[c];
    gk[0] = 0.f;
#pragma unroll
    for (int k = 1; k < 16; ++k) {
      gk[k] = 0.f;
      if (k < nb) gk[k] = rest[(k - 1) * 3 + 0] * vc[0] + rest[(k - 1) * 3 + 1] * vc[1] + rest[(k - 1) * 3 + 2] * vc[2];  // L1 hit
      if (k <= nrest) {
        srow[(k - 1) * 3 + 0] = basis[k] * vc[0];
        srow[(k - 1) * 3 + 1] = basis[k] * vc[1];
        srow[(k - 1) * 3 + 2] = basis[k] * vc[2];
      }
    }
    if (deg > 0) {
      float vu[3];
      sh_basis_vjp(deg, ux, uy, uz, gk, vu);
      const float dp = ux * vu[0] + uy * vu[1] + uz * vu[2];
      vm[0] += (vu[0] - ux * dp) * inorm;
      vm[1] += (vu[1] - uy * dp) * inorm;
      vm[2] += (vu[2] - uz * dp) * inorm;
      if constexpr (VIEWMAT) {
        // campos = -W^T t:  v_W += t vdir^T ;  v_t += W vdir
        const float vdir[3] = {(vu[0] - ux * dp) * inorm, (vu[1] - uy * dp) * inorm, (vu[2] - uz * dp) * inorm};
#pragma unroll
        for (int r = 0; r < 3; ++r) {
#pragma unroll
          for (int c = 0; c < 3; ++c) pv[(r * 3 + c) * PB_THREADS] += cam.t[r] * vdir[c];
          pv[(9 + r) * PB_THREADS] += cam.W[r][0] * vdir[0] + cam.W[r][1] * vdir[1] + cam.W[r][2] * vdir[2];
        }
      }
    }
  }
}

// Adds the CTA's per-thread viewmat partials into v_viewmat[4,4] with 12 float atomics per CTA: s_pv[k * PB_THREADS +
// tid] holds thread tid's sum of component k (v_W row-major [9], v_t [3]); warp shuffles, then one 12-float row per
// warp in shared memory.  Every thread of the CTA must call it.
__device__ __forceinline__ void cta_add_viewmat(const float* s_pv, float* v_viewmat) {
  __shared__ float s_red[PB_THREADS / 32][12];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 12; ++k) {
    float v = s_pv[k * PB_THREADS + threadIdx.x];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    if (lane == 0) s_red[warp][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < 12) {
    const int k = threadIdx.x;
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < PB_THREADS / 32; ++w) s += s_red[w][k];
    atomicAdd(v_viewmat + (k < 9 ? (k / 3) * 4 + k % 3 : (k - 9) * 4 + 3), s);
  }
}

// Only Gaussians that received a raster gradient are processed (touched[g] != 0, written by dnr_raster_bwd).  On the
// 1 M-Gaussian / 1080p scene ~40 % are visible but only ~10 % are ever composited before the pixels saturate, so a pass
// with one lane per Gaussian would leave most lanes idle.  Here a CTA scans the flags of PB_SCAN consecutive Gaussians
// (coalesced bytes), compacts the touched ids in shared memory and then runs the per-Gaussian backward with every lane
// busy; the 180 B SH rows are staged in shared memory (stride 45 words: conflict-free) and accumulated row by row (each
// row is a contiguous span).  Accumulate-only: the caller pre-zeroes the gradient buffers (and v_means2d /
// v_means2d_abs).
constexpr int PB_SCAN = 1024;

// VIEWMAT: each thread sums its Gaussians' d(loss)/d(viewmat) over the loop; one CTA reduction adds it to a.v_viewmat.
template <bool NORMALS, bool VIEWMAT = false>
__global__ void __launch_bounds__(PB_THREADS, 8) project_bwd_touched_kernel(const DnrArgs a) {
  __shared__ float s_rest[PB_THREADS * PB_REST_MAX];
  __shared__ int s_ids[PB_SCAN];
  __shared__ int s_n;
  const int tid = threadIdx.x;
  const int base = blockIdx.x * PB_SCAN;
  if (tid == 0) s_n = 0;
  __syncthreads();
  {
    const int n_here = min(PB_SCAN, a.n_gauss - base);
    const uint8_t* fl = a.touched + base;
    // 8 flags per thread and step; `base` is a multiple of 1024, so the 8-byte loads are aligned
    for (int k = tid * 8; k < n_here; k += PB_THREADS * 8) {
      unsigned long long w = 0;
      if (k + 8 <= n_here) {
        w = *reinterpret_cast<const unsigned long long*>(fl + k);
      } else {
        for (int b = 0; k + b < n_here; ++b) w |= (unsigned long long)fl[k + b] << (8 * b);
      }
      while (w) {
        const int b = (__ffsll((long long)w) - 1) >> 3;
        s_ids[atomicAdd(&s_n, 1)] = base + k + b;
        w &= ~(0xffull << (8 * b));
      }
    }
  }
  __syncthreads();
  const int n_touched = s_n;
  const int nrest = a.sh_bases - 1;
  const int nrow = nrest * 3;
  float* srow = s_rest + tid * PB_REST_MAX;
  __shared__ float s_pv[VIEWMAT ? 12 * PB_THREADS : 1];
  float* pv = VIEWMAT ? s_pv + tid : nullptr;
  if constexpr (VIEWMAT) {
#pragma unroll
    for (int k = 0; k < 12; ++k) pv[k * PB_THREADS] = 0.f;
  }
  for (int off = 0; off < n_touched; off += PB_THREADS) {
    const int slot = off + tid;
    const bool active = slot < n_touched;
    if (active) {
      const int i = s_ids[slot];
      float vm[3] = {0, 0, 0}, vq[4] = {0, 0, 0, 0}, vs[3] = {0, 0, 0}, vo = 0.f, vdc[3] = {0, 0, 0};
      if (a.radii[i] > 0) {
        project_bwd_gauss<NORMALS, VIEWMAT>(a, i, nrest, srow, vm, vq, vs, vo, vdc, pv);
      } else {
        for (int k = 0; k < nrow; ++k) srow[k] = 0.f;
      }
      for (int k = 0; k < 3; ++k) { a.v_means[i * 3 + k] += vm[k]; a.v_scales[i * 3 + k] += vs[k]; a.v_sh_dc[i * 3 + k] += vdc[k]; }
      for (int k = 0; k < 4; ++k) a.v_quats[i * 4 + k] += vq[k];
      a.v_opacities[i] += vo;
      // the record is consumed: leave grad_records all zero for the next dnr_raster_bwd (DNR_FLAG_PERSISTENT_WS), 64 B
      // per touched Gaussian instead of a memset of the whole buffer
      float4* gr = reinterpret_cast<float4*>(a.grad_records + (size_t)i * DNR_GRAD_FLOATS);
      const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
      gr[0] = z; gr[1] = z; gr[2] = z; gr[3] = z;
    }
    __syncthreads();
    if (nrest > 0) {
      const int rows = min(PB_THREADS, n_touched - off);
      const int total = rows * nrow;
      for (int e = tid; e < total; e += PB_THREADS) {
        const int r = e / nrow, k = e - r * nrow;
        a.v_sh_rest[(size_t)s_ids[off + r] * nrow + k] += s_rest[r * PB_REST_MAX + k];
      }
    }
    __syncthreads();
  }
  if constexpr (VIEWMAT) {
    if (n_touched > 0) cta_add_viewmat(s_pv, a.v_viewmat);
  }
}

}  // namespace

extern "C" int dnr_project_fwd(const DnrArgs* a, void* stream) {
  if (!a) return DNR_E_NULL;
  if (a->n_gauss <= 0 || a->width <= 0 || a->height <= 0) return DNR_E_SIZE;
  if (a->tile_size != DNR_TILE || a->sh_degree < 0 || a->sh_degree > 3 || (a->sh_degree + 1) * (a->sh_degree + 1) > a->sh_bases)
    return DNR_E_OPTION;
  const bool hostcam = (a->flags & DNR_FLAG_HOST_CAMERA) != 0;
  if (!hostcam && (!a->viewmat || !a->K)) return DNR_E_NULL;
  if (!a->means || !a->quats || !a->scales || !a->opacities || !a->sh_dc || !a->radii ||
      !a->means2d || !a->depths || !a->conics || !a->opac_act || !a->colors || !a->tiles_per_gauss || !a->depth_keys ||
      !a->records)
    return DNR_E_NULL;
  if (a->sh_bases > 1 && !a->sh_rest) return DNR_E_NULL;
  const bool normals = (a->flags & DNR_FLAG_NORMALS) != 0;
  if (normals && !hostcam && !a->c2w) return DNR_E_NULL;
  const int block = 256, grid = (a->n_gauss + block - 1) / block;
  cudaStream_t s = (cudaStream_t)stream;
  if (normals) project_fwd_kernel<true><<<grid, block, 0, s>>>(*a);
  else project_fwd_kernel<false><<<grid, block, 0, s>>>(*a);
  DNR_CHECK_LAUNCH();
  return 0;
}

extern "C" int dnr_project_bwd(const DnrArgs* a, void* stream) {
  if (!a) return DNR_E_NULL;
  if (a->n_gauss <= 0) return DNR_E_SIZE;
  const bool hostcam = (a->flags & DNR_FLAG_HOST_CAMERA) != 0;
  if (!hostcam && (!a->viewmat || !a->K)) return DNR_E_NULL;
  if (!a->means || !a->quats || !a->scales || !a->opacities || !a->sh_dc || !a->radii ||
      !a->grad_records || !a->v_means || !a->v_quats || !a->v_scales || !a->v_opacities || !a->v_sh_dc)
    return DNR_E_NULL;
  if (a->sh_bases > 1 && (!a->sh_rest || !a->v_sh_rest)) return DNR_E_NULL;
  const bool normals = (a->flags & DNR_FLAG_NORMALS) != 0;
  if (normals && !hostcam && !a->c2w) return DNR_E_NULL;
  if (a->sh_bases > 16) return DNR_E_OPTION;
  if (!a->touched) return DNR_E_NULL;
  if (!(a->flags & DNR_FLAG_ACCUMULATE)) return DNR_E_OPTION;  // scattered rows: the caller pre-zeroes and accumulates
  const int grid = (a->n_gauss + PB_SCAN - 1) / PB_SCAN;
  cudaStream_t s = (cudaStream_t)stream;
  if (a->v_viewmat != nullptr) {
    if (normals) project_bwd_touched_kernel<true, true><<<grid, PB_THREADS, 0, s>>>(*a);
    else project_bwd_touched_kernel<false, true><<<grid, PB_THREADS, 0, s>>>(*a);
  } else {
    if (normals) project_bwd_touched_kernel<true><<<grid, PB_THREADS, 0, s>>>(*a);
    else project_bwd_touched_kernel<false><<<grid, PB_THREADS, 0, s>>>(*a);
  }
  DNR_CHECK_LAUNCH();
  return 0;
}
