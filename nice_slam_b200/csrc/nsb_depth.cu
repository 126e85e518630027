// nsb_depth.cu -- the 2D reconstruction metric (calc_2d_metric, src/tools/eval_recon.py:120-209): a watertight depth rasterizer for
// triangle meshes, the unseen-region test of the view sampler (check_proj, :60-87) and the per-view depth L1.  Declarations and rules:
// include/nice_slam_b200.h, "2D reconstruction metric".
#include <cmath>
#include "nsb_common.cuh"
#include "nsb_geom.cuh"

namespace nsb {
namespace {

constexpr int kThreads = 256;
constexpr int kCams = 64;                        // camera rows staged in shared memory per pass of the face kernel
constexpr long long kSmallPixels = 128;          // pixel boxes up to this size are walked by the face's own thread
constexpr unsigned kEmptyBits = 0x7f800000u;     // +inf: no hit yet
constexpr int kLargeBlocks = 132 * 8;            // blocks of the cooperative kernel (grid-stride over the queue)
unsigned blocks_for(long long n) { return (unsigned)((n + kThreads - 1) / kThreads); }

// float64 without contraction, so that every thread computes the same bits for the same inputs
__device__ __forceinline__ void cross3(const double a[3], const double b[3], double r[3]) {
  r[0] = __dsub_rn(__dmul_rn(a[1], b[2]), __dmul_rn(a[2], b[1]));
  r[1] = __dsub_rn(__dmul_rn(a[2], b[0]), __dmul_rn(a[0], b[2]));
  r[2] = __dsub_rn(__dmul_rn(a[0], b[1]), __dmul_rn(a[1], b[0]));
}
__device__ __forceinline__ double dot3(const double a[3], const double b[3]) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a[0], b[0]), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]));
}
// camera space of world point p under c2w rows 0-2 (c: 12 doubles, row-major [R | t]): q = R^T (p - t)
__device__ __forceinline__ void to_camera(const double* c, const double p[3], double q[3]) {
  const double d0 = __dsub_rn(p[0], c[3]), d1 = __dsub_rn(p[1], c[7]), d2 = __dsub_rn(p[2], c[11]);
#pragma unroll
  for (int k = 0; k < 3; k++) q[k] = __dadd_rn(__dadd_rn(__dmul_rn(c[k], d0), __dmul_rn(c[4 + k], d1)), __dmul_rn(c[8 + k], d2));
}

struct Intr { double fx, fy, cx, cy, zn, zf; int H, W; };

// One face under one camera.  m[k] = sgn(D) (v_k x v_k+1): the pixel ray d is inside edge k iff m[k].d > 0, or == 0 and tie bit k is
// set.  The plane v_k x v_k+1 and its twin v_k+1 x v_k of a neighbouring face are exact negations of each other, so both faces see the
// same |m.d| bits.  The tie bit says whether the face lies on the positive side of the edge plane with its normal's sign chosen
// lexicographically (first non-zero component > 0): a ray exactly on a shared edge goes to the face on the positive side, and a ray
// exactly through a vertex to the one face of its fan that the same half-plane rule selects.  Depth: z = D / (N.d), N = (b - a) x (c - a),
// D = N.a, the ray's intersection with the face's plane.
struct FaceRast {
  double m[3][3];
  double N[3];
  double D;
  int tie;
};

__device__ __forceinline__ bool lex_negative(const double n[3]) {
  return n[0] < 0.0 || (n[0] == 0.0 && (n[1] < 0.0 || (n[1] == 0.0 && n[2] < 0.0)));
}

// -> false if the face covers no pixel of the image in [zn, ...): D == 0 (its plane holds the camera centre), every vertex in front of
// zn or behind zf, or its box (of the part with z >= zn, one pixel of margin) misses the image.
__device__ __forceinline__ bool face_setup(const double v[3][3], const Intr& I, FaceRast& r, int& i0, int& i1, int& j0, int& j1) {
  const bool front0 = v[0][2] >= I.zn, front1 = v[1][2] >= I.zn, front2 = v[2][2] >= I.zn;
  if (!front0 && !front1 && !front2) return false;
  if (v[0][2] > I.zf && v[1][2] > I.zf && v[2][2] > I.zf) return false;
  const double e1[3] = {__dsub_rn(v[1][0], v[0][0]), __dsub_rn(v[1][1], v[0][1]), __dsub_rn(v[1][2], v[0][2])};
  const double e2[3] = {__dsub_rn(v[2][0], v[0][0]), __dsub_rn(v[2][1], v[0][1]), __dsub_rn(v[2][2], v[0][2])};
  cross3(e1, e2, r.N);
  r.D = dot3(r.N, v[0]);
  if (!(r.D != 0.0)) return false;
  const bool dneg = r.D < 0.0;
  r.tie = 0;
#pragma unroll
  for (int k = 0; k < 3; k++) {
    double c[3];
    cross3(v[k], v[(k + 1) % 3], c);
    r.tie |= (lex_negative(c) == dneg) << k;
#pragma unroll
    for (int a = 0; a < 3; a++) r.m[k][a] = dneg ? -c[a] : c[a];
  }
  // pixel box of the polygon {face} cut to z >= zn: its vertices in front and the crossings of its edges with z = zn
  double umin = INFINITY, umax = -INFINITY, vmin = INFINITY, vmax = -INFINITY;
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const int l = (k + 1) % 3;
    const bool fk = v[k][2] >= I.zn, fl = v[l][2] >= I.zn;
    if (fk) {
      const double u = __dadd_rn(__ddiv_rn(__dmul_rn(I.fx, v[k][0]), v[k][2]), I.cx), w = __dadd_rn(__ddiv_rn(__dmul_rn(I.fy, v[k][1]), v[k][2]), I.cy);
      umin = fmin(umin, u); umax = fmax(umax, u); vmin = fmin(vmin, w); vmax = fmax(vmax, w);
    }
    if (fk != fl) {
      const double t = __ddiv_rn(__dsub_rn(I.zn, v[k][2]), __dsub_rn(v[l][2], v[k][2]));
      const double x = __dadd_rn(v[k][0], __dmul_rn(t, __dsub_rn(v[l][0], v[k][0])));
      const double y = __dadd_rn(v[k][1], __dmul_rn(t, __dsub_rn(v[l][1], v[k][1])));
      const double u = __dadd_rn(__ddiv_rn(__dmul_rn(I.fx, x), I.zn), I.cx), w = __dadd_rn(__ddiv_rn(__dmul_rn(I.fy, y), I.zn), I.cy);
      umin = fmin(umin, u); umax = fmax(umax, u); vmin = fmin(vmin, w); vmax = fmax(vmax, w);
    }
  }
  umin = fmax(umin - 1.0, 0.0); vmin = fmax(vmin - 1.0, 0.0);
  umax = fmin(umax + 1.0, (double)(I.W - 1)); vmax = fmin(vmax + 1.0, (double)(I.H - 1));
  if (!(umin <= umax && vmin <= vmax)) return false;
  j0 = (int)ceil(umin); j1 = (int)floor(umax); i0 = (int)ceil(vmin); i1 = (int)floor(vmax);
  return j0 <= j1 && i0 <= i1;
}

// the pixel (row i, column j): the face's depth there if it covers it within [zn, zf], folded into the pixel by atomicMin on the bits
__device__ __forceinline__ void shade(const FaceRast& r, const Intr& I, int i, int j, unsigned* __restrict__ depth) {
  const double d[3] = {__ddiv_rn(__dsub_rn((double)j, I.cx), I.fx), __ddiv_rn(__dsub_rn((double)i, I.cy), I.fy), 1.0};
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const double e = dot3(r.m[k], d);
    if (!(e > 0.0 || (e == 0.0 && ((r.tie >> k) & 1)))) return;
  }
  const double z = __ddiv_rn(r.D, dot3(r.N, d));
  if (!(z >= I.zn && z <= I.zf)) return;
  atomicMin(depth + (long long)i * I.W + j, __float_as_uint(__double2float_rn(z)));
}

__device__ __forceinline__ void load_face(const double* __restrict__ verts, const int* __restrict__ faces, int f, double w[3][3]) {
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const double* p = verts + 3ll * faces[3 * f + k];
    w[k][0] = p[0]; w[k][1] = p[1]; w[k][2] = p[2];
  }
}

__global__ void depth_fill_kernel(unsigned* depth, long long n, unsigned value) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) depth[i] = value;
}
__global__ void depth_finish_kernel(unsigned* depth, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && depth[i] == kEmptyBits) depth[i] = 0u;
}

// One thread per face over every camera (rows 0-2 staged kCams at a time).  Small pixel boxes are walked here; larger ones are queued
// as (face, camera) for raster_large_kernel.
__global__ void __launch_bounds__(kThreads) raster_faces_kernel(const double* __restrict__ verts, const int* __restrict__ faces, int F,
                                                                const double* __restrict__ c2w, int P, Intr I, unsigned* __restrict__ depth,
                                                                int2* __restrict__ queue, unsigned long long* __restrict__ n_queued) {
  __shared__ double s_c[kCams * 12];
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  double w[3][3] = {};
  if (f < F) load_face(verts, faces, f, w);
  const long long hw = (long long)I.H * I.W;
  for (int base = 0; base < P; base += kCams) {
    const int np = P - base < kCams ? P - base : kCams;
    __syncthreads();
    for (int i = threadIdx.x; i < 12 * np; i += blockDim.x) s_c[i] = c2w[16ll * base + 16 * (i / 12) + i % 12];
    __syncthreads();
    if (f >= F) continue;
    for (int m = 0; m < np; m++) {
      double v[3][3];
#pragma unroll
      for (int k = 0; k < 3; k++) to_camera(s_c + 12 * m, w[k], v[k]);
      FaceRast r;
      int i0, i1, j0, j1;
      if (!face_setup(v, I, r, i0, i1, j0, j1)) continue;
      const long long area = (long long)(i1 - i0 + 1) * (j1 - j0 + 1);
      if (area > kSmallPixels) {
        queue[atomicAdd(n_queued, 1ull)] = make_int2(f, base + m);
        continue;
      }
      unsigned* out = depth + (long long)(base + m) * hw;
      for (int i = i0; i <= i1; i++)
        for (int j = j0; j <= j1; j++) shade(r, I, i, j, out);
    }
  }
}

// A block per queued (face, camera): every thread sets the face up (the same bits), then the block walks its pixel box.
__global__ void __launch_bounds__(kThreads) raster_large_kernel(const double* __restrict__ verts, const int* __restrict__ faces,
                                                                const double* __restrict__ c2w, Intr I, unsigned* __restrict__ depth,
                                                                const int2* __restrict__ queue, const unsigned long long* __restrict__ n_queued) {
  const unsigned long long n = *n_queued;
  const long long hw = (long long)I.H * I.W;
  for (unsigned long long q = blockIdx.x; q < n; q += gridDim.x) {
    const int2 e = queue[q];
    double w[3][3], v[3][3], c[12];
    load_face(verts, faces, e.x, w);
#pragma unroll
    for (int k = 0; k < 12; k++) c[k] = c2w[16ll * e.y + k];
#pragma unroll
    for (int k = 0; k < 3; k++) to_camera(c, w[k], v[k]);
    FaceRast r;
    int i0, i1, j0, j1;
    if (!face_setup(v, I, r, i0, i1, j0, j1)) continue;
    const int bw = j1 - j0 + 1;
    const long long area = (long long)(i1 - i0 + 1) * bw;
    unsigned* out = depth + (long long)e.y * hw;
    for (long long p = threadIdx.x; p < area; p += blockDim.x) shade(r, I, i0 + (int)(p / bw), j0 + (int)(p % bw), out);
  }
}

// view errors: out[p] = mean |a - b| over the view's pixels in float64; each thread sums a fixed strided set in order, then a fixed tree
__global__ void __launch_bounds__(kThreads) depth_l1_kernel(const float* __restrict__ a, const float* __restrict__ b, long long hw,
                                                            double* __restrict__ out) {
  __shared__ double s[kThreads];
  const float* pa = a + (long long)blockIdx.x * hw;
  const float* pb = b + (long long)blockIdx.x * hw;
  double acc = 0.0;
  for (long long i = threadIdx.x; i < hw; i += kThreads) acc = __dadd_rn(acc, fabs(__dsub_rn((double)pa[i], (double)pb[i])));
  s[threadIdx.x] = acc;
  __syncthreads();
  for (int h = kThreads / 2; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h) s[threadIdx.x] = __dadd_rn(s[threadIdx.x], s[threadIdx.x + h]);
    __syncthreads();
  }
  if (threadIdx.x == 0) out[blockIdx.x] = __ddiv_rn(s[0], (double)hw);
}

// check_proj over a batch of poses: blockIdx.y = pose; a thread stops at its first point inside, a block skips a pose already seen
__global__ void __launch_bounds__(kThreads) views_see_any_kernel(const double* __restrict__ pts, int n, const float* __restrict__ w2c,
                                                                 float fx, float fy, float cx, float cy, float H, float W,
                                                                 uint8_t* any) {
  const int p = blockIdx.y;
  if (*(volatile uint8_t*)(any + p)) return;
  const float* T = w2c + 16ll * p;
  bool s = false;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n && !s; i += (long long)gridDim.x * blockDim.x) {
    const float q[3] = {(float)pts[3 * i], (float)pts[3 * i + 1], (float)pts[3 * i + 2]};
    float cz;
    s = in_frustum(T, q, fx, fy, cx, cy, H, W, 1e-5f, cz);
  }
  if (s) any[p] = 1;
}
__global__ void zero_u8_kernel(uint8_t* p, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = 0;
}

}  // namespace
}  // namespace nsb

using namespace nsb;

extern "C" size_t nsb_depth_render_workspace(int F, int P) {
  return F < 0 || P < 0 ? 0 : 16 + 8ull * (unsigned long long)F * (unsigned long long)P;
}
extern "C" int nsb_depth_render(const double* vertices, int V, const int32_t* faces, int F, const double* c2w, int P, double fx, double fy,
                                double cx, double cy, int H, int W, double z_near, double z_far, void* ws, size_t ws_bytes, float* depth,
                                void* stream) {
  if (V < 0 || F < 0 || P < 0 || (P > 0 && (!c2w || !depth || !ws)) || (F > 0 && (!vertices || !faces))) {
    set_error("nsb_depth_render: NULL pointer or negative count"); return NSB_ERR_ARG; }
  if (H < 1 || W < 1 || !(fx != 0.0) || !(fy != 0.0) || !std::isfinite(fx) || !std::isfinite(fy) || !std::isfinite(cx) || !std::isfinite(cy)) {
    set_error("nsb_depth_render: H and W must be >= 1 and fx, fy finite and non-zero, cx, cy finite (H %d, W %d)", H, W); return NSB_ERR_ARG; }
  if (!(z_near > 0.0) || !(z_far >= z_near) || !std::isfinite(z_far)) {
    set_error("nsb_depth_render: need 0 < z_near <= z_far < inf (z_near %g, z_far %g)", z_near, z_far); return NSB_ERR_ARG; }
  if (P == 0) return NSB_OK;
  if (ws_bytes < nsb_depth_render_workspace(F, P)) {
    set_error("nsb_depth_render: workspace %zu < %zu bytes", ws_bytes, nsb_depth_render_workspace(F, P)); return NSB_ERR_ARG; }
  const cudaStream_t st = (cudaStream_t)stream;
  const long long n = (long long)P * H * W;
  unsigned* d = reinterpret_cast<unsigned*>(depth);
  unsigned long long* n_queued = static_cast<unsigned long long*>(ws);
  int2* queue = reinterpret_cast<int2*>(static_cast<char*>(ws) + 16);
  depth_fill_kernel<<<blocks_for(n), kThreads, 0, st>>>(d, n, kEmptyBits);
  int rc = check_cuda(cudaGetLastError(), "depth_fill_kernel launch"); if (rc) return rc;
  if (F > 0) {
    if ((rc = check_cuda(cudaMemsetAsync(n_queued, 0, 8, st), "nsb_depth_render: queue reset"))) return rc;
    const Intr I{fx, fy, cx, cy, z_near, z_far, H, W};
    raster_faces_kernel<<<blocks_for(F), kThreads, 0, st>>>(vertices, faces, F, c2w, P, I, d, queue, n_queued);
    if ((rc = check_cuda(cudaGetLastError(), "raster_faces_kernel launch"))) return rc;
    raster_large_kernel<<<kLargeBlocks, kThreads, 0, st>>>(vertices, faces, c2w, I, d, queue, n_queued);
    if ((rc = check_cuda(cudaGetLastError(), "raster_large_kernel launch"))) return rc;
  }
  depth_finish_kernel<<<blocks_for(n), kThreads, 0, st>>>(d, n);
  return check_cuda(cudaGetLastError(), "depth_finish_kernel launch");
}

extern "C" int nsb_depth_l1(const float* depth_a, const float* depth_b, int P, long long hw, double* errors, void* stream) {
  if (P < 0 || hw < 1 || (P > 0 && (!depth_a || !depth_b || !errors))) { set_error("nsb_depth_l1: NULL pointer or bad size"); return NSB_ERR_ARG; }
  if (P == 0) return NSB_OK;
  depth_l1_kernel<<<P, kThreads, 0, (cudaStream_t)stream>>>(depth_a, depth_b, hw, errors);
  return check_cuda(cudaGetLastError(), "depth_l1_kernel launch");
}

extern "C" int nsb_views_see_any(const double* points, int n, const float* w2c, int P, double fx, double fy, double cx, double cy, int H,
                                 int W, uint8_t* any, void* stream) {
  if (n < 0 || P < 0 || (P > 0 && (!w2c || !any)) || (n > 0 && !points)) { set_error("nsb_views_see_any: NULL pointer or negative count"); return NSB_ERR_ARG; }
  if (H < 1 || W < 1 || !std::isfinite(fx) || !std::isfinite(fy) || !std::isfinite(cx) || !std::isfinite(cy)) {
    set_error("nsb_views_see_any: H and W must be >= 1 and the intrinsics finite (H %d, W %d)", H, W); return NSB_ERR_ARG; }
  if (P == 0) return NSB_OK;
  const cudaStream_t st = (cudaStream_t)stream;
  zero_u8_kernel<<<blocks_for(P), kThreads, 0, st>>>(any, P);
  int rc = check_cuda(cudaGetLastError(), "zero_u8_kernel launch"); if (rc) return rc;
  if (n == 0) return NSB_OK;
  const unsigned bx = blocks_for(n) < 64u ? blocks_for(n) : 64u;
  for (int p0 = 0; p0 < P; p0 += 65535) {
    const int np = P - p0 < 65535 ? P - p0 : 65535;
    views_see_any_kernel<<<dim3(bx, np), kThreads, 0, st>>>(points, n, w2c + 16ll * p0, (float)fx, (float)fy, (float)cx, (float)cy, (float)H,
                                                           (float)W, any + p0);
    if ((rc = check_cuda(cudaGetLastError(), "views_see_any_kernel launch"))) return rc;
  }
  return NSB_OK;
}
