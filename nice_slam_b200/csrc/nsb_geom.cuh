// nsb_geom.cuh -- ray sampling, point generation, normalisation and trilinear set-up.
//
// Everything that decides WHICH voxels a sample touches is computed with explicit round-to-nearest
// intrinsics (no FMA contraction) in the same dtype flow as the reference, so that sample order and
// voxel-corner indices are bit-exact (north_star):  near f32; far, z, p, normalised coords f64
// (slam.bound is a float64 tensor, src/NICE_SLAM.py:145-146); grid coordinates f32
// (src/utils/Renderer.py:82-174, src/common.py:269-284, ATen/native/GridSampler.h:27-33,58-60).
#pragma once
#include "nsb_common.cuh"

namespace nsb {

__device__ __forceinline__ double nanmax(double a, double b) { return (a > b || a != a) ? a : b; }  // torch.max semantics
__device__ __forceinline__ double nanmin(double a, double b) { return (a < b || a != a) ? a : b; }

// t_exit of the ray through the (f64) bound box: min over axes of max over (lo,hi) of (bound - o)/d
// (src/utils/Renderer.py:98-105, src/Tracker.py:97-101)
__device__ __forceinline__ double ray_far_bb(const double* __restrict__ bound, const float o[3], const float d[3]) {
  double far = 0.0;
#pragma unroll
  for (int a = 0; a < 3; a++) {
    const double oo = (double)o[a], dd = (double)d[a];
    const double t0 = __ddiv_rn(__dsub_rn(bound[2 * a], oo), dd);
    const double t1 = __ddiv_rn(__dsub_rn(bound[2 * a + 1], oo), dd);
    const double m = nanmax(t0, t1);
    far = a == 0 ? m : nanmin(far, m);
  }
  return far;
}

struct RaySampler {       // per-ray constants of the stratified + near-surface sampler
  float near;             // f32
  double far;             // f64
  float gt;               // sensor depth of this ray (0 if none)
  int has_gt;
};

__device__ __forceinline__ RaySampler make_sampler(const double* bound, const float o[3], const float d[3],
                                                   int has_gt, float gt, float gtmax12) {
  RaySampler rs;
  const double far_bb = __dadd_rn(ray_far_bb(bound, o, d), 0.01);
  rs.has_gt = has_gt; rs.gt = gt;
  if (has_gt) {
    rs.near = __fmul_rn(gt, 0.01f);                                  // Renderer.py:96
    rs.far = nanmin(nanmax(far_bb, 0.0), (double)gtmax12);           // clamp(far_bb, 0, max(gt*1.2)), :109
  } else { rs.near = 0.01f; rs.far = far_bb; }
  return rs;
}
// stratified sample at t = linspace value (Renderer.py:154-157).  lindisp: 1/near is the f32 reciprocal (near = gt*0.01 f32; the
// Python 0.01 without sensor depth gives the same 100.0f), 1/far and the rest f64; gt = 0 gives 1/near = inf -> z = 0, and NaN at t = 1.
__device__ __forceinline__ double uniform_z(const RaySampler& rs, float t, int lindisp) {
  if (!lindisp) {
    const float a = __fmul_rn(rs.near, __fsub_rn(1.0f, t));        // f32 (Renderer.py:155)
    return __dadd_rn((double)a, __dmul_rn(rs.far, (double)t));     // f64
  }
  const float a = __fmul_rn(__frcp_rn(rs.near), __fsub_rn(1.0f, t));                       // f32 (:157)
  return __drcp_rn(__dadd_rn((double)a, __dmul_rn(__drcp_rn(rs.far), (double)t)));          // f64
}
// unsorted sample i of the concatenation [uniform(n_samples) | surface(n_surface)] (perturb: jitter_z afterwards)
__device__ __forceinline__ double sample_z(const RaySampler& rs, int i, int n_samples,
                                           const float* __restrict__ t_uniform, const double* __restrict__ t_surface,
                                           float gtmax, int lindisp) {
  if (i < n_samples) return uniform_z(rs, t_uniform[i], lindisp);
  const double ts = t_surface[i - n_samples];
  const double omt = __dsub_rn(1.0, ts);
  if (rs.gt > 0.0f)                                                  // Renderer.py:128-140
    return __dadd_rn(__dmul_rn((double)__fmul_rn(0.95f, rs.gt), omt), __dmul_rn((double)__fmul_rn(1.05f, rs.gt), ts));
  return __dadd_rn(__dmul_rn(0.001, omt), __dmul_rn((double)gtmax, ts));   // :143-150
}
// perturb (Renderer.py:159-166): stratified sample i of z [n] moves to lower + (upper - lower) t_rand, lower / upper = the mid-points
// .5 (z[i-1] + z[i]) and .5 (z[i] + z[i+1]) (z[0] / z[n-1] at the ends); t_rand is promoted to f64
__device__ __forceinline__ double jitter_z(const double* z, int i, int n, float t_rand) {
  const double lo = i > 0 ? __dmul_rn(0.5, __dadd_rn(z[i], z[i - 1])) : z[i];
  const double hi = i + 1 < n ? __dmul_rn(0.5, __dadd_rn(z[i + 1], z[i])) : z[i];
  return __dadd_rn(lo, __dmul_rn(__dsub_rn(hi, lo), (double)t_rand));
}
// strict-weak order used by the rank sort: ascending, NaN last (torch.sort)
__device__ __forceinline__ bool z_less(double a, double b) { return (a < b) || (b != b && a == a); }

struct PointGeom {
  double p[3];
  float pf[3];        // p.float(): input of the Fourier embedding (un-normalised world coordinates)
  float xn[3];        // normalised to the scene bound, f32
  float xnc[3];       // normalised to the coarse (enlarged) bound
  int inb;            // strictly inside the scene bound (Renderer.py:43-46)
};

__device__ __forceinline__ void make_point(const double* __restrict__ bound, const double* __restrict__ cbound,
                                           const float o[3], const float d[3], double z, PointGeom& P) {
  P.inb = 1;
#pragma unroll
  for (int a = 0; a < 3; a++) {
    const double p = __dadd_rn((double)o[a], __dmul_rn((double)d[a], z));        // Renderer.py:172-174
    P.p[a] = p; P.pf[a] = (float)p;
    const double lo = bound[2 * a], hi = bound[2 * a + 1];
    if (!(p < hi && p > lo)) P.inb = 0;
    P.xn[a] = (float)__dsub_rn(__dmul_rn(__ddiv_rn(__dsub_rn(p, lo), __dsub_rn(hi, lo)), 2.0), 1.0);   // common.py:280-282
    const double clo = cbound[2 * a], chi = cbound[2 * a + 1];
    P.xnc[a] = (float)__dsub_rn(__dmul_rn(__ddiv_rn(__dsub_rn(p, clo), __dsub_rn(chi, clo)), 2.0), 1.0);
  }
}
__device__ __forceinline__ void make_point_from_p(const double* __restrict__ bound, const double* __restrict__ cbound,
                                                  const double pin[3], PointGeom& P) {
  P.inb = 1;
#pragma unroll
  for (int a = 0; a < 3; a++) {
    const double p = pin[a];
    P.p[a] = p; P.pf[a] = (float)p;
    const double lo = bound[2 * a], hi = bound[2 * a + 1];
    if (!(p < hi && p > lo)) P.inb = 0;
    P.xn[a] = (float)__dsub_rn(__dmul_rn(__ddiv_rn(__dsub_rn(p, lo), __dsub_rn(hi, lo)), 2.0), 1.0);
    const double clo = cbound[2 * a], chi = cbound[2 * a + 1];
    P.xnc[a] = (float)__dsub_rn(__dmul_rn(__ddiv_rn(__dsub_rn(p, clo), __dsub_rn(chi, clo)), 2.0), 1.0);
  }
}

// F.grid_sample(align_corners=True, padding_mode='border') coordinate set-up for one axis.
// u = ((x+1)/2)*(size-1) clipped to [0,size-1]; i0 = floor(u); clipg = 0 where the clip is active.
__device__ __forceinline__ void tri_axis(float xn, int size, float& u, int& i0, float& clipg) {
  const float mx = (float)(size - 1);
  u = __fmul_rn(__fmul_rn(__fadd_rn(xn, 1.0f), 0.5f), mx);
  if (u <= 0.0f) { u = 0.0f; clipg = 0.0f; }
  else if (u >= mx) { u = mx; clipg = 0.0f; }
  else clipg = 1.0f;
  i0 = (int)floorf(u);
}

struct Tri {              // trilinear cell of one point in one grid
  int i0[3];              // x (W), y (H), z (D) lower corner
  float w0[3], w1[3];     // per-axis weights: w0 = (i0+1) - u, w1 = u - i0
  float clipg[3];
};
__device__ __forceinline__ Tri make_tri(const float xn[3], int W, int H, int D) {
  Tri t; const int size[3] = {W, H, D};
#pragma unroll
  for (int a = 0; a < 3; a++) {
    float u; tri_axis(xn[a], size[a], u, t.i0[a], t.clipg[a]);
    const float f0 = (float)t.i0[a];
    t.w0[a] = __fsub_rn(__fadd_rn(f0, 1.0f), u);
    t.w1[a] = __fsub_rn(u, f0);
  }
  return t;
}
__device__ __forceinline__ float tri_weight(const Tri& t, int k) {   // corner k: bit0 +x, bit1 +y, bit2 +z
  const float wx = (k & 1) ? t.w1[0] : t.w0[0];
  const float wy = (k & 2) ? t.w1[1] : t.w0[1];
  const float wz = (k & 4) ? t.w1[2] : t.w0[2];
  return __fmul_rn(__fmul_rn(wx, wy), wz);
}
// Branch-free corner addressing: the upper corner index is clamped to the grid; when the clamp is active the sample sits
// exactly on the last voxel (u == size-1) so that corner's weight w1 is exactly 0 -- same result as grid_sample skipping it.
__device__ __forceinline__ void tri_corner_clamped(const Tri& t, int k, int W, int H, int D, int& x, int& y, int& z) {
  x = min(t.i0[0] + (k & 1), W - 1); y = min(t.i0[1] + ((k >> 1) & 1), H - 1); z = min(t.i0[2] + ((k >> 2) & 1), D - 1);
}
__device__ __forceinline__ bool tri_corner(const Tri& t, int k, int W, int H, int D, int& x, int& y, int& z) {
  x = t.i0[0] + (k & 1); y = t.i0[1] + ((k >> 1) & 1); z = t.i0[2] + ((k >> 2) & 1);
  return x < W && y < H && z < D;      // lower bounds hold by construction (border clip)
}

}  // namespace nsb
