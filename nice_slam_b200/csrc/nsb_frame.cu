// nsb_frame.cu -- frame preparation (BaseDataset.__getitem__, src/utils/datasets.py:77-113): the raw decoded bytes of one RGB-D frame in,
// the frame the tracker and mapper read out.  One pass per reference operation, in its order; declarations and the exact rules:
// include/nice_slam_b200.h, "frame preparation".  Every float64 operation is written with an explicit rounding intrinsic, so nvcc's
// default -fmad=true cannot fuse one the reference rounds twice (or split the one fused multiply-add the reference's build makes).
#include <cmath>
#include <cstdint>
#include "nsb_common.cuh"

namespace nsb {
namespace {

constexpr int kThreads = 256;
unsigned blocks_for(long long n) { return (unsigned)((n + kThreads - 1) / kThreads); }

__device__ __forceinline__ double dm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double da(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ds(double a, double b) { return __dsub_rn(a, b); }

// cv::invert's closed form for a 3x3 float64 matrix (DECOMP_LU, n <= 3): cofactors times 1/det
__device__ void inv3(const double S[9], double t[9]) {
  const double det = da(ds(dm(S[0], ds(dm(S[4], S[8]), dm(S[5], S[7]))), dm(S[1], ds(dm(S[3], S[8]), dm(S[5], S[6])))),
                        dm(S[2], ds(dm(S[3], S[7]), dm(S[4], S[6]))));
  const double d = __ddiv_rn(1.0, det);
  t[0] = dm(ds(dm(S[4], S[8]), dm(S[5], S[7])), d);
  t[1] = dm(ds(dm(S[2], S[7]), dm(S[1], S[8])), d);
  t[2] = dm(ds(dm(S[1], S[5]), dm(S[2], S[4])), d);
  t[3] = dm(ds(dm(S[5], S[6]), dm(S[3], S[8])), d);
  t[4] = dm(ds(dm(S[0], S[8]), dm(S[2], S[6])), d);
  t[5] = dm(ds(dm(S[2], S[3]), dm(S[0], S[5])), d);
  t[6] = dm(ds(dm(S[3], S[7]), dm(S[4], S[6])), d);
  t[7] = dm(ds(dm(S[1], S[6]), dm(S[0], S[7])), d);
  t[8] = dm(ds(dm(S[0], S[4]), dm(S[1], S[3])), d);
}

// cvRound + saturate_cast<int> of a double: round half to even; out of range and NaN give INT_MIN, as cvRound's cvtsd2si does
__device__ __forceinline__ int round_sat(double v) {
  if (!(v >= -2147483648.0 && v < 2147483647.5)) return INT32_MIN;
  return __double2int_rn(v);
}

// ---- stage 1: cv2.undistort(colour, K, dist) ----------------------------------------------------------------------------------------
// cv::undistort maps the image in stripes of max(1, 4096 / W) rows, each with the new camera matrix's cy shifted by the stripe's first
// row; initUndistortRectifyMap then walks a row in chunks of 8 columns (its AVX2 double path), accumulating the chunk start, and the
// columns after the last whole chunk one by one.  The map is rounded to 1/32 pixel; remap blends the 4 neighbours with 15-bit weights.
__global__ void undistort_kernel(const uint8_t* __restrict__ src, int H, int W, double fx, double fy, double cx, double cy,
                                 double k1, double k2, double p1, double p2, double k3, uint8_t* __restrict__ dst) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= (long long)H * W) return;
  const int row = (int)(p / W), j = (int)(p % W);
  int s0 = 4096 / (W > 1 ? W : 1);
  s0 = s0 < 1 ? 1 : (s0 > H ? H : s0);
  const int y0 = row - row % s0;
  const double Ar[9] = {fx, 0.0, cx, 0.0, fy, ds(cy, (double)y0), 0.0, 0.0, 1.0};
  double ir[9];
  inv3(Ar, ir);
  const double i = (double)(row - y0);
  double bx = da(dm(i, ir[1]), ir[2]), by = da(dm(i, ir[4]), ir[5]), bw = da(dm(i, ir[7]), ir[8]);
  const int chunks = W / 8, c = j / 8;
  double X, Y, Wt;
  if (c < chunks) {
    for (int n = 0; n < c; ++n) { bx = da(bx, dm(8.0, ir[0])); by = da(by, dm(8.0, ir[3])); bw = da(bw, dm(8.0, ir[6])); }
    const double s = (double)(j - 8 * c);
    X = da(bx, dm(ir[0], s)); Y = da(by, dm(ir[3], s)); Wt = da(bw, dm(ir[6], s));
  } else {
    for (int n = 0; n < chunks; ++n) { bx = da(bx, dm(8.0, ir[0])); by = da(by, dm(8.0, ir[3])); bw = da(bw, dm(8.0, ir[6])); }
    for (int n = 8 * chunks; n < j; ++n) { bx = da(bx, ir[0]); by = da(by, ir[3]); bw = da(bw, ir[6]); }
    X = bx; Y = by; Wt = bw;
  }
  const double w = __ddiv_rn(1.0, Wt);
  const double x = dm(X, w), y = dm(Y, w);
  const double x2 = dm(x, x), y2 = dm(y, y), r2 = da(x2, y2), xy2 = dm(dm(2.0, x), y);
  const double kr = da(1.0, dm(da(dm(da(dm(k3, r2), k2), r2), k1), r2));
  const double xd = da(da(dm(x, kr), dm(p1, xy2)), dm(p2, da(r2, dm(2.0, x2))));
  const double yd = da(da(dm(y, kr), dm(p1, da(r2, dm(2.0, y2)))), dm(p2, xy2));
  const int iu = round_sat(dm(__fma_rn(fx, xd, cx), 32.0));
  const int iv = round_sat(dm(__fma_rn(fy, yd, cy), 32.0));
  const int sx = (int)(short)(iu >> 5), sy = (int)(short)(iv >> 5);      // the CV_16SC2 map stores the cell as shorts
  const int a = iu & 31, b = iv & 31;
  const int wt[4] = {32 * (32 - a) * (32 - b), 32 * a * (32 - b), 32 * (32 - a) * b, 32 * a * b};
  int acc[3] = {0, 0, 0};
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int X0 = sx + (q & 1), Y0 = sy + (q >> 1);
    if (X0 < 0 || X0 >= W || Y0 < 0 || Y0 >= H) continue;             // BORDER_CONSTANT 0
    const uint8_t* s = src + 3ll * ((long long)Y0 * W + X0);
    for (int ch = 0; ch < 3; ++ch) acc[ch] += (int)s[ch] * wt[q];
  }
  for (int ch = 0; ch < 3; ++ch) {
    const int v = (acc[ch] + (1 << 14)) >> 15;
    dst[3 * p + ch] = (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
  }
}

// ---- stages 2-3: BGR -> RGB, / 255. in float64, cv2.resize(colour, (Wd, Hd)) INTER_LINEAR ---------------------------------------------
// resize's float64 path: float64 coefficients (fx = (dx + 0.5) * scale_x - 0.5, floor, 1 - fx), a horizontal pass with the columns
// whose right neighbour falls outside copied, and a vertical pass whose rows are clamped to the image with the weights kept.  At an exact
// 2x2 downscale cv::resize averages 4 pixels (INTER_AREA) instead; the bilinear weights there are all 1/2, so only rounding differs.
// Only the pixels that survive crop_edge are written (a crop selects; it computes nothing); out has row stride out_w.
__device__ __forceinline__ double rgb01(const uint8_t* src, long long pix, int c) { return __ddiv_rn((double)src[3 * pix + 2 - c], 255.0); }

__global__ void colour_kernel(const uint8_t* __restrict__ src, int Hs, int Ws, int Hd, int Wd, double scale_x, double scale_y,
                              int y_off, int x_off, int out_h, int out_w, double* __restrict__ out) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= (long long)out_h * out_w) return;
  const int oy = (int)(p / out_w), ox = (int)(p % out_w);
  const int dy = oy + y_off, dx = ox + x_off;
  double* o = out + 3 * p;
  if (Hs == Hd && Ws == Wd) {                                           // cv::resize returns a copy at the same size
    const long long s = (long long)dy * Ws + dx;
    for (int c = 0; c < 3; ++c) o[c] = rgb01(src, s, c);
    return;
  }
  const double fxr = ds(dm(da((double)dx, 0.5), scale_x), 0.5);
  int sx = (int)floor(fxr);
  double fxd = ds(fxr, (double)sx);
  const bool copy = sx + 1 >= Ws;
  if (sx < 0) { fxd = 0.0; sx = 0; }
  if (sx >= Ws - 1) { fxd = 0.0; sx = Ws - 1; }
  const double a0 = ds(1.0, fxd), a1 = fxd;
  const double fyr = ds(dm(da((double)dy, 0.5), scale_y), 0.5);
  const int sy = (int)floor(fyr);
  const double b1 = ds(fyr, (double)sy), b0 = ds(1.0, b1);
  const int r0 = sy < 0 ? 0 : (sy > Hs - 1 ? Hs - 1 : sy);
  const int r1 = sy + 1 < 0 ? 0 : (sy + 1 > Hs - 1 ? Hs - 1 : sy + 1);
  for (int c = 0; c < 3; ++c) {
    double h[2];
    const int rows[2] = {r0, r1};
    for (int k = 0; k < 2; ++k) {
      const long long base = (long long)rows[k] * Ws;
      h[k] = copy ? dm(rgb01(src, base + sx, c), 1.0) : da(dm(rgb01(src, base + sx, c), a0), dm(rgb01(src, base + sx + 1, c), a1));
    }
    o[c] = da(dm(h[0], b0), dm(h[1], b1));
  }
}

// ---- stage 5 (colour): F.interpolate(mode='bilinear', align_corners=True) on CPU float64, channels-last input ----------------------
// torch's compute_source_index_and_lambda: same size -> the index itself with weights (1, 0); else real = ratio * i, index =
// floorf(real) (through float), lambda = clamp(real - index, 0, 1); the four products h*w, summed left to right.
__device__ __forceinline__ void torch_linear(int i, int in, int outn, double ratio, int& i0, int& i1, double& l0, double& l1) {
  if (outn == in) { i0 = i1 = i; l0 = 1.0; l1 = 0.0; return; }
  const double real = dm(ratio, (double)i);
  long long idx = (long long)floorf((float)real);
  if (idx > in - 1) idx = in - 1;
  i0 = (int)idx;
  double lam = ds(real, (double)idx);
  lam = lam < 0.0 ? 0.0 : (lam > 1.0 ? 1.0 : lam);
  i1 = i0 + (i0 < in - 1 ? 1 : 0);
  l1 = lam;
  l0 = ds(1.0, lam);
}

__global__ void bilinear_kernel(const double* __restrict__ src, int Hs, int Ws, int Ho, int Wo, double ratio_h, double ratio_w,
                                int edge, int out_h, int out_w, double* __restrict__ out) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= (long long)out_h * out_w) return;
  const int oy = (int)(p / out_w) + edge, ox = (int)(p % out_w) + edge;
  int h0, h1, w0, w1;
  double hl0, hl1, wl0, wl1;
  torch_linear(oy, Hs, Ho, ratio_h, h0, h1, hl0, hl1);
  torch_linear(ox, Ws, Wo, ratio_w, w0, w1, wl0, wl1);
  const double w00 = dm(hl0, wl0), w01 = dm(hl0, wl1), w10 = dm(hl1, wl0), w11 = dm(hl1, wl1);
  const double* i00 = src + 3ll * ((long long)h0 * Ws + w0);
  const double* i01 = src + 3ll * ((long long)h0 * Ws + w1);
  const double* i10 = src + 3ll * ((long long)h1 * Ws + w0);
  const double* i11 = src + 3ll * ((long long)h1 * Ws + w1);
  for (int c = 0; c < 3; ++c)
    out[3 * p + c] = da(da(da(dm(i00[c], w00), dm(i01[c], w01)), dm(i10[c], w10)), dm(i11[c], w11));
}

// ---- stages 4-6 (depth): float32(raw) / float32(png_depth_scale) * float32(scale), F.interpolate(mode='nearest'), crop_edge -----------
// torch's nearest_idx: same size -> i; twice the size -> i >> 1; else min(floorf(i * (float)in / out), in - 1), all in float32
__device__ __forceinline__ int torch_nearest(int i, int in, int outn) {
  if (outn == in) return i;
  if (outn == 2 * in) return i >> 1;
  const float scale = __fdiv_rn((float)in, (float)outn);
  const long long s = (long long)floorf(__fmul_rn((float)i, scale));
  return (int)(s < in - 1 ? s : in - 1);
}

__global__ void depth_kernel(const uint16_t* __restrict__ raw, int Hs, int Ws, int Ho, int Wo, float png_scale, float scale, int edge,
                             int out_h, int out_w, float* __restrict__ out) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= (long long)out_h * out_w) return;
  const int sy = torch_nearest((int)(p / out_w) + edge, Hs, Ho), sx = torch_nearest((int)(p % out_w) + edge, Ws, Wo);
  out[p] = __fmul_rn(__fdiv_rn((float)raw[(long long)sy * Ws + sx], png_scale), scale);
}

}  // namespace
}  // namespace nsb

using namespace nsb;

namespace {
bool bad_params(const nsb_frame_params* f) {
  if (!f || f->color_h < 1 || f->color_w < 1 || f->depth_h < 1 || f->depth_w < 1 || f->crop_edge < 0) return true;
  if ((f->crop_h != 0) != (f->crop_w != 0) || f->crop_h < 0 || f->crop_w < 0) return true;
  const int h = f->crop_h ? f->crop_h : f->depth_h, w = f->crop_w ? f->crop_w : f->depth_w;
  return h - 2 * f->crop_edge < 1 || w - 2 * f->crop_edge < 1 || !(f->png_depth_scale > 0.0);
}
size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }
}  // namespace

extern "C" void nsb_frame_output_size(const nsb_frame_params* f, int* H, int* W) {
  const int h = f->crop_h ? f->crop_h : f->depth_h, w = f->crop_w ? f->crop_w : f->depth_w;
  *H = h - 2 * f->crop_edge;
  *W = w - 2 * f->crop_edge;
}

extern "C" size_t nsb_frame_workspace(const nsb_frame_params* f) {
  if (bad_params(f)) return 0;
  size_t n = 0;
  if (f->undistort) n += align256(3ull * f->color_h * f->color_w);
  if (f->crop_h) n += 8ull * 3 * f->depth_h * f->depth_w;
  return n;
}

extern "C" int nsb_frame_prepare(const nsb_frame_params* f, const uint8_t* color_bgr, const uint16_t* depth_raw, void* ws, size_t ws_bytes,
                                 double* color_out, float* depth_out, void* stream) {
  if (bad_params(f) || !color_bgr || !depth_raw || !color_out || !depth_out) {
    set_error("nsb_frame_prepare: bad argument (positive sizes, crop_size both or neither, crop_edge leaving a pixel, png_depth_scale > 0)");
    return NSB_ERR_ARG;
  }
  const size_t need = nsb_frame_workspace(f);
  if (need && (!ws || ws_bytes < need)) { set_error("nsb_frame_prepare: workspace too small (%zu bytes needed)", need); return NSB_ERR_ARG; }
  cudaStream_t s = (cudaStream_t)stream;
  int rc;
  int Ho, Wo;
  nsb_frame_output_size(f, &Ho, &Wo);
  const long long n_out = (long long)Ho * Wo;
  const uint8_t* col = color_bgr;
  char* w = (char*)ws;
  if (f->undistort) {
    uint8_t* und = (uint8_t*)w;
    w += align256(3ull * f->color_h * f->color_w);
    const long long n = (long long)f->color_h * f->color_w;
    undistort_kernel<<<blocks_for(n), kThreads, 0, s>>>(color_bgr, f->color_h, f->color_w, f->fx, f->fy, f->cx, f->cy, f->dist[0], f->dist[1],
                                                        f->dist[2], f->dist[3], f->dist[4], und);
    if ((rc = check_cuda(cudaGetLastError(), "undistort_kernel launch"))) return rc;
    col = und;
  }
  // cv::resize: inv_scale = (double)dsize / ssize, scale = 1. / inv_scale
  const double scale_x = 1.0 / ((double)f->depth_w / f->color_w), scale_y = 1.0 / ((double)f->depth_h / f->color_h);
  if (f->crop_h) {
    double* full = (double*)w;
    const long long n = (long long)f->depth_h * f->depth_w;
    colour_kernel<<<blocks_for(n), kThreads, 0, s>>>(col, f->color_h, f->color_w, f->depth_h, f->depth_w, scale_x, scale_y, 0, 0, f->depth_h,
                                                     f->depth_w, full);
    if ((rc = check_cuda(cudaGetLastError(), "colour_kernel launch"))) return rc;
    const double rh = f->crop_h > 1 ? (double)(f->depth_h - 1) / (double)(f->crop_h - 1) : 0.0;
    const double rw = f->crop_w > 1 ? (double)(f->depth_w - 1) / (double)(f->crop_w - 1) : 0.0;
    bilinear_kernel<<<blocks_for(n_out), kThreads, 0, s>>>(full, f->depth_h, f->depth_w, f->crop_h, f->crop_w, rh, rw, f->crop_edge, Ho, Wo,
                                                          color_out);
    if ((rc = check_cuda(cudaGetLastError(), "bilinear_kernel launch"))) return rc;
  } else {
    colour_kernel<<<blocks_for(n_out), kThreads, 0, s>>>(col, f->color_h, f->color_w, f->depth_h, f->depth_w, scale_x, scale_y, f->crop_edge,
                                                         f->crop_edge, Ho, Wo, color_out);
    if ((rc = check_cuda(cudaGetLastError(), "colour_kernel launch"))) return rc;
  }
  depth_kernel<<<blocks_for(n_out), kThreads, 0, s>>>(depth_raw, f->depth_h, f->depth_w, f->crop_h ? f->crop_h : f->depth_h,
                                                      f->crop_w ? f->crop_w : f->depth_w, (float)f->png_depth_scale, (float)f->scale,
                                                      f->crop_edge, Ho, Wo, depth_out);
  return check_cuda(cudaGetLastError(), "depth_kernel launch");
}
