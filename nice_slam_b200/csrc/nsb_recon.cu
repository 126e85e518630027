// nsb_recon.cu -- reconstruction metrics (calc_3d_metric, src/tools/eval_recon.py:91-117): area-weighted surface sampling, exact nearest
// neighbours on a uniform grid, and the correspondence pass of point-to-point ICP.  Declarations and rules: include/nice_slam_b200.h,
// "reconstruction metrics".
#include <cfloat>
#include <cmath>
#include "nsb_common.cuh"
#include "nsb_scan.cuh"

namespace nsb {
namespace {

constexpr int kThreads = 256;
constexpr int kMaxPartials = 1024;                  // per-block partials of the two-stage reductions
constexpr int kIcpSums = 17;                        // count, sum d^2, sum p [3], sum q [3], sum p q^T [9]
unsigned blocks_for(long long n) { return (unsigned)((n + kThreads - 1) / kThreads); }
unsigned partial_blocks(long long n) { const unsigned b = blocks_for(n); return b < 1u ? 1u : (b > (unsigned)kMaxPartials ? (unsigned)kMaxPartials : b); }

// ---- surface sampling (trimesh.sample.sample_surface, trimesh 3.10.7) ----------------------------------------------------------------
// area[f] = |(v1 - v0) x (v2 - v0)| / 2 in numpy's order (trimesh.triangles.area); area[F] = 0 so that the exclusive scan ends in the total
__global__ void face_area_kernel(const double* __restrict__ v, const int* __restrict__ faces, int F, double* area) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > F) return;
  if (f == F) { area[F] = 0.0; return; }
  const double* A = v + 3ll * faces[3 * f];
  const double* B = v + 3ll * faces[3 * f + 1];
  const double* Cc = v + 3ll * faces[3 * f + 2];
  const double u[3] = {__dsub_rn(B[0], A[0]), __dsub_rn(B[1], A[1]), __dsub_rn(B[2], A[2])};
  const double w[3] = {__dsub_rn(Cc[0], A[0]), __dsub_rn(Cc[1], A[1]), __dsub_rn(Cc[2], A[2])};
  const double c0 = __dsub_rn(__dmul_rn(u[1], w[2]), __dmul_rn(u[2], w[1]));
  const double c1 = __dsub_rn(__dmul_rn(u[2], w[0]), __dmul_rn(u[0], w[2]));
  const double c2 = __dsub_rn(__dmul_rn(u[0], w[1]), __dmul_rn(u[1], w[0]));
  area[f] = __ddiv_rn(__dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(c0, c0), __dmul_rn(c1, c1)), __dmul_rn(c2, c2))), 2.0);
}
// excl[f + 1] is the inclusive cumulative area of face f; face = searchsorted(cum, u0 * cum[F-1], 'left')
__global__ void sample_kernel(const double* __restrict__ v, const int* __restrict__ faces, int F, const double* __restrict__ excl,
                              const double* __restrict__ u, long long count, double* pts, long long* face_index) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= count) return;
  const double pick = __dmul_rn(u[3 * s], excl[F]);
  int lo = 0, hi = F;                                   // first f in [0, F) with cum[f] >= pick, F if none
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (excl[mid + 1] < pick) lo = mid + 1; else hi = mid; }
  const int f = lo < F ? lo : F - 1;
  double a = u[3 * s + 1], b = u[3 * s + 2];
  if (__dadd_rn(a, b) > 1.0) { a = fabs(__dsub_rn(a, 1.0)); b = fabs(__dsub_rn(b, 1.0)); }
  const double* A = v + 3ll * faces[3 * f];
  const double* B = v + 3ll * faces[3 * f + 1];
  const double* Cc = v + 3ll * faces[3 * f + 2];
  for (int k = 0; k < 3; k++)                            // (a (v1 - v0) + b (v2 - v0)) + v0, as trimesh sums it
    pts[3 * s + k] = __dadd_rn(__dadd_rn(__dmul_rn(__dsub_rn(B[k], A[k]), a), __dmul_rn(__dsub_rn(Cc[k], A[k]), b)), A[k]);
  face_index[s] = f;
}

// ---- uniform grid ----------------------------------------------------------------------------------------------------------------
// bounds: per-block min / max, then one block over the partials (min and max do not depend on the order)
__global__ void bounds_partial_kernel(const double* __restrict__ p, int n, double* partial) {
  __shared__ double s[kThreads / 32][6];
  double m[6] = {INFINITY, INFINITY, INFINITY, -INFINITY, -INFINITY, -INFINITY};
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    for (int a = 0; a < 3; a++) { const double x = p[3 * i + a]; m[a] = fmin(m[a], x); m[3 + a] = fmax(m[3 + a], x); }
  for (int o = 16; o > 0; o >>= 1)
    for (int a = 0; a < 3; a++) {
      m[a] = fmin(m[a], __shfl_xor_sync(0xffffffffu, m[a], o));
      m[3 + a] = fmax(m[3 + a], __shfl_xor_sync(0xffffffffu, m[3 + a], o));
    }
  if ((threadIdx.x & 31) == 0) for (int k = 0; k < 6; k++) s[threadIdx.x >> 5][k] = m[k];
  __syncthreads();
  if (threadIdx.x < 6) {
    double r = s[0][threadIdx.x];
    for (int w = 1; w < kThreads / 32; w++) r = threadIdx.x < 3 ? fmin(r, s[w][threadIdx.x]) : fmax(r, s[w][threadIdx.x]);
    partial[6 * blockIdx.x + threadIdx.x] = r;
  }
}
__global__ void bounds_final_kernel(const double* partial, int nb, double* box) {
  if (threadIdx.x >= 6) return;
  double r = partial[threadIdx.x];
  for (int b = 1; b < nb; b++) r = threadIdx.x < 3 ? fmin(r, partial[6 * b + threadIdx.x]) : fmax(r, partial[6 * b + threadIdx.x]);
  box[threadIdx.x] = r;
}

struct GridView {
  double o[3], cell, slack;
  int dims[3];
  const unsigned long long* start;
  const double* pts;
  const int* idx;
};
GridView view_of(const nsb_nn_grid* g) {
  GridView v;
  for (int a = 0; a < 3; a++) { v.o[a] = g->origin[a]; v.dims[a] = g->dims[a]; }
  v.cell = g->cell; v.slack = g->slack; v.start = g->cell_start; v.pts = g->points; v.idx = g->index;
  return v;
}
// cell coordinate along axis a, clamped to the grid (the same rule for targets and queries)
__device__ __forceinline__ int cell_coord(const GridView& g, int a, double x) {
  const double f = floor(__ddiv_rn(__dsub_rn(x, g.o[a]), g.cell));
  return f < 0.0 ? 0 : (f >= (double)(g.dims[a] - 1) ? g.dims[a] - 1 : (int)f);
}
__device__ __forceinline__ long long cell_linear(const GridView& g, int i, int j, int k) {
  return ((long long)i * g.dims[1] + j) * g.dims[2] + k;
}
__global__ void grid_count_kernel(const double* __restrict__ p, int n, GridView g, unsigned long long* counts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long c = cell_linear(g, cell_coord(g, 0, p[3ll * i]), cell_coord(g, 1, p[3ll * i + 1]), cell_coord(g, 2, p[3ll * i + 2]));
  atomicAdd(&counts[c], 1ull);
}
__global__ void grid_scatter_kernel(const double* __restrict__ p, int n, GridView g, unsigned long long* cursor, double* sorted, int* index) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double x = p[3ll * i], y = p[3ll * i + 1], z = p[3ll * i + 2];
  const long long c = cell_linear(g, cell_coord(g, 0, x), cell_coord(g, 1, y), cell_coord(g, 2, z));
  const unsigned long long s = atomicAdd(&cursor[c], 1ull);
  sorted[3 * s] = x; sorted[3 * s + 1] = y; sorted[3 * s + 2] = z;
  index[s] = i;
}

// squared distance from q to the box [lo, hi] along the axes, each face moved out by slack
__device__ __forceinline__ double gap2(const double q[3], const double lo[3], const double hi[3], double slack) {
  double s = 0.0;
  for (int a = 0; a < 3; a++) {
    const double d = fmax(0.0, fmax(lo[a] - slack - q[a], q[a] - hi[a] - slack));
    s += d * d;
  }
  return s;
}
// exact nearest target of q: d2 < best (best = radius^2, or +inf) or an equal d2 with a smaller index wins; shell by shell around q's
// clamped cell, skipping cells whose box is farther than the best so far, until no cell outside the visited block can hold a point at
// d2 <= best.  -> target index (its sorted slot in slot), or -1 with best unchanged.
__device__ int nn_search(const GridView& g, const double q[3], double& best, unsigned long long& slot) {
  int bi = -1;
  const int c[3] = {cell_coord(g, 0, q[0]), cell_coord(g, 1, q[1]), cell_coord(g, 2, q[2])};
  double glo[3], ghi[3];
  int maxr = 0;
  for (int a = 0; a < 3; a++) {
    glo[a] = g.o[a]; ghi[a] = g.o[a] + g.dims[a] * g.cell;
    maxr = max(maxr, max(c[a], g.dims[a] - 1 - c[a]));
  }
  for (int r = 0; r <= maxr; r++) {
    const int x0 = max(c[0] - r, 0), x1 = min(c[0] + r, g.dims[0] - 1);
    const int y0 = max(c[1] - r, 0), y1 = min(c[1] + r, g.dims[1] - 1);
    for (int i = x0; i <= x1; i++)
      for (int j = y0; j <= y1; j++) {
        const bool edge = abs(i - c[0]) == r || abs(j - c[1]) == r;
        const int kstep = edge ? 1 : (r > 0 ? 2 * r : 1);
        for (int k = edge ? max(c[2] - r, 0) : c[2] - r; k <= (edge ? min(c[2] + r, g.dims[2] - 1) : c[2] + r); k += kstep) {
          if (k < 0 || k >= g.dims[2]) continue;
          const double lo[3] = {g.o[0] + i * g.cell, g.o[1] + j * g.cell, g.o[2] + k * g.cell};
          const double hi[3] = {lo[0] + g.cell, lo[1] + g.cell, lo[2] + g.cell};
          if (gap2(q, lo, hi, g.slack) > best) continue;
          const long long cl = cell_linear(g, i, j, k);
          const unsigned long long e = g.start[cl + 1];
          for (unsigned long long s = g.start[cl]; s < e; s++) {
            const double dx = __dsub_rn(q[0], g.pts[3 * s]), dy = __dsub_rn(q[1], g.pts[3 * s + 1]), dz = __dsub_rn(q[2], g.pts[3 * s + 2]);
            const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
            const int id = g.idx[s];
            if (d2 < best || (d2 == best && bi >= 0 && id < bi)) { best = d2; bi = id; slot = s; }
          }
        }
      }
    if (r == maxr) break;
    // lower bound over every cell at Chebyshev distance > r: the six slabs beyond the visited block, each with the grid's full extent
    // along the other two axes
    double bound = INFINITY;
    for (int a = 0; a < 3; a++)
      for (int side = 0; side < 2; side++) {
        const int ci = side ? c[a] + r + 1 : c[a] - r - 1;
        if (ci < 0 || ci >= g.dims[a]) continue;
        double lo[3], hi[3];
        for (int b = 0; b < 3; b++) { lo[b] = glo[b]; hi[b] = ghi[b]; }
        if (side) lo[a] = g.o[a] + ci * g.cell; else hi[a] = g.o[a] + (ci + 1) * g.cell;
        bound = fmin(bound, gap2(q, lo, hi, g.slack));
      }
    if (bound > best) break;
  }
  return bi;
}

__global__ void nn_query_kernel(GridView g, const double* __restrict__ q, int m, double r2, double* dist2, int* index) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const double p[3] = {q[3ll * i], q[3ll * i + 1], q[3ll * i + 2]};
  double best = r2;
  unsigned long long slot;
  const int bi = nn_search(g, p, best, slot);
  dist2[i] = bi >= 0 ? best : INFINITY;
  index[i] = bi;
}

// ---- ICP correspondences + sums ------------------------------------------------------------------------------------------------
struct Rigid { double m[12]; };                         // rows of T[:3, :4]
__device__ __forceinline__ void warp_sum(double* v) {
  for (int o = 16; o > 0; o >>= 1)
    for (int k = 0; k < kIcpSums; k++) v[k] = __dadd_rn(v[k], __shfl_down_sync(0xffffffffu, v[k], o));
}
// per-block partial sums over the source points, in a fixed order: each thread sums its grid-stride points in turn, then a shuffle tree
// per warp and the warps in turn
__global__ void icp_partial_kernel(GridView g, const double* __restrict__ src, int m, Rigid T, double r2, double* partial) {
  __shared__ double s[kThreads / 32][kIcpSums];
  double acc[kIcpSums];
  for (int k = 0; k < kIcpSums; k++) acc[k] = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (long long)gridDim.x * blockDim.x) {
    const double x = src[3 * i], y = src[3 * i + 1], z = src[3 * i + 2];
    double p[3];
    for (int a = 0; a < 3; a++)
      p[a] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T.m[4 * a], x), __dmul_rn(T.m[4 * a + 1], y)), __dmul_rn(T.m[4 * a + 2], z)), T.m[4 * a + 3]);
    double best = r2;
    unsigned long long slot;
    if (nn_search(g, p, best, slot) < 0) continue;
    const double q[3] = {g.pts[3 * slot], g.pts[3 * slot + 1], g.pts[3 * slot + 2]};
    acc[0] = __dadd_rn(acc[0], 1.0);
    acc[1] = __dadd_rn(acc[1], best);
    for (int a = 0; a < 3; a++) { acc[2 + a] = __dadd_rn(acc[2 + a], p[a]); acc[5 + a] = __dadd_rn(acc[5 + a], q[a]); }
    for (int a = 0; a < 3; a++)
      for (int b = 0; b < 3; b++) acc[8 + 3 * a + b] = __dadd_rn(acc[8 + 3 * a + b], __dmul_rn(p[a], q[b]));
  }
  warp_sum(acc);
  if ((threadIdx.x & 31) == 0) for (int k = 0; k < kIcpSums; k++) s[threadIdx.x >> 5][k] = acc[k];
  __syncthreads();
  if (threadIdx.x < kIcpSums) {
    double r = s[0][threadIdx.x];
    for (int w = 1; w < kThreads / 32; w++) r = __dadd_rn(r, s[w][threadIdx.x]);
    partial[kIcpSums * blockIdx.x + threadIdx.x] = r;
  }
}
__global__ void icp_final_kernel(const double* partial, int nb, double* sums) {
  if (threadIdx.x >= kIcpSums) return;
  double r = 0.0;
  for (int b = 0; b < nb; b++) r = __dadd_rn(r, partial[kIcpSums * b + threadIdx.x]);
  sums[threadIdx.x] = r;
}

bool bad_grid(const nsb_nn_grid* g) {
  return !g || g->n_points < 0 || g->cell <= 0.0 || !(g->slack >= 0.0) || g->dims[0] < 1 || g->dims[1] < 1 || g->dims[2] < 1 ||
         g->n_cells != (long long)g->dims[0] * g->dims[1] * g->dims[2] || !g->cell_start || (g->n_points > 0 && (!g->points || !g->index));
}

}  // namespace
}  // namespace nsb

using namespace nsb;

// trimesh.sample.sample_surface (trimesh 3.10.7) with the caller's uniforms
extern "C" size_t nsb_sample_surface_workspace(int n_faces) {
  return align16(8ull * (n_faces + 1)) + 8ull * scan_ws_elems((long long)n_faces + 1);
}
extern "C" int nsb_sample_surface(const double* vertices, const int32_t* faces, int n_faces, const double* uniforms, long long count,
                                  void* ws, size_t ws_bytes, double* points, long long* face_index, void* stream) {
  if (n_faces < 1 || count < 0 || !vertices || !faces || !ws || (count > 0 && (!uniforms || !points || !face_index))) {
    set_error("nsb_sample_surface: bad argument (n_faces >= 1, count >= 0)"); return NSB_ERR_ARG; }
  if (ws_bytes < nsb_sample_surface_workspace(n_faces)) { set_error("nsb_sample_surface: workspace too small"); return NSB_ERR_ARG; }
  const cudaStream_t st = (cudaStream_t)stream;
  double* area = static_cast<double*>(ws);
  double* scan_ws = reinterpret_cast<double*>(static_cast<char*>(ws) + align16(8ull * (n_faces + 1)));
  face_area_kernel<<<blocks_for((long long)n_faces + 1), kThreads, 0, st>>>(vertices, faces, n_faces, area);
  int rc = check_cuda(cudaGetLastError(), "face_area_kernel launch"); if (rc) return rc;
  if ((rc = excl_scan(area, (long long)n_faces + 1, scan_ws, st))) return rc;
  if (count == 0) return NSB_OK;
  sample_kernel<<<blocks_for(count), kThreads, 0, st>>>(vertices, faces, n_faces, area, uniforms, count, points, face_index);
  return check_cuda(cudaGetLastError(), "sample_kernel launch");
}

// the targets' bounding box
extern "C" size_t nsb_nn_bounds_workspace(int n_points) { return 8ull * 6 * partial_blocks(n_points); }
extern "C" int nsb_nn_bounds(const double* points, int n_points, void* ws, size_t ws_bytes, double* box, void* stream) {
  if (n_points < 1 || !points || !ws || !box) { set_error("nsb_nn_bounds: bad argument (n_points >= 1)"); return NSB_ERR_ARG; }
  if (ws_bytes < nsb_nn_bounds_workspace(n_points)) { set_error("nsb_nn_bounds: workspace too small"); return NSB_ERR_ARG; }
  const unsigned nb = partial_blocks(n_points);
  bounds_partial_kernel<<<nb, kThreads, 0, (cudaStream_t)stream>>>(points, n_points, static_cast<double*>(ws));
  bounds_final_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(static_cast<const double*>(ws), (int)nb, box);
  return check_cuda(cudaGetLastError(), "nsb_nn_bounds launch");
}

// the cell rule of the header, on the host
extern "C" int nsb_nn_plan(const double box[6], int n_points, nsb_nn_grid* g) {
  if (!box || !g || n_points < 1) { set_error("nsb_nn_plan: bad argument (n_points >= 1)"); return NSB_ERR_ARG; }
  double e[3], E = 0.0, mag = 0.0;
  for (int a = 0; a < 3; a++) {
    if (!std::isfinite(box[a]) || !std::isfinite(box[3 + a]) || box[3 + a] < box[a]) { set_error("nsb_nn_plan: box is not finite"); return NSB_ERR_ARG; }
    e[a] = box[3 + a] - box[a]; E = std::fmax(E, e[a]);
    mag = std::fmax(mag, std::fmax(std::fabs(box[a]), std::fabs(box[3 + a])));
  }
  const double cap = 2.0 * n_points;
  double cell = 1.0, dims[3] = {1.0, 1.0, 1.0};
  if (E > 0.0) {
    double vol = 1.0;
    for (int a = 0; a < 3; a++) vol *= std::fmax(e[a], E / 64.0);
    cell = std::cbrt(vol / n_points);
    for (;;) {
      for (int a = 0; a < 3; a++) dims[a] = std::floor(e[a] / cell) + 1.0;
      if (dims[0] * dims[1] * dims[2] <= cap) break;
      cell *= 1.0905077326652577;                     // 2^(1/8)
    }
  }
  for (int a = 0; a < 3; a++) { g->origin[a] = box[a]; g->dims[a] = (int32_t)dims[a]; }
  g->cell = cell;
  g->slack = 16.0 * DBL_EPSILON * (mag + E + cell);
  g->n_cells = (long long)dims[0] * (long long)dims[1] * (long long)dims[2];
  g->n_points = n_points;
  return NSB_OK;
}

// counting sort of the targets into the cells of a planned grid
extern "C" size_t nsb_nn_build_workspace(long long n_cells) {
  return align16(8ull * (n_cells + 1)) + 8ull * scan_ws_elems(n_cells + 1);
}
extern "C" int nsb_nn_build(const double* targets, const nsb_nn_grid* g, void* ws, size_t ws_bytes, void* stream) {
  if (!targets || bad_grid(g) || g->n_points < 1 || !ws) { set_error("nsb_nn_build: bad argument (plan the grid with nsb_nn_plan)"); return NSB_ERR_ARG; }
  if (ws_bytes < nsb_nn_build_workspace(g->n_cells)) { set_error("nsb_nn_build: workspace too small"); return NSB_ERR_ARG; }
  const cudaStream_t st = (cudaStream_t)stream;
  const GridView v = view_of(g);
  unsigned long long* start = g->cell_start;
  unsigned long long* cursor = static_cast<unsigned long long*>(ws);
  unsigned long long* scan_ws = reinterpret_cast<unsigned long long*>(static_cast<char*>(ws) + align16(8ull * (g->n_cells + 1)));
  int rc = check_cuda(cudaMemsetAsync(start, 0, 8ull * (g->n_cells + 1), st), "nsb_nn_build memset"); if (rc) return rc;
  grid_count_kernel<<<blocks_for(g->n_points), kThreads, 0, st>>>(targets, g->n_points, v, start);
  if ((rc = check_cuda(cudaGetLastError(), "grid_count_kernel launch"))) return rc;
  if ((rc = excl_scan(start, g->n_cells + 1, scan_ws, st))) return rc;
  if ((rc = check_cuda(cudaMemcpyAsync(cursor, start, 8ull * (g->n_cells + 1), cudaMemcpyDeviceToDevice, st), "nsb_nn_build copy"))) return rc;
  grid_scatter_kernel<<<blocks_for(g->n_points), kThreads, 0, st>>>(targets, g->n_points, v, cursor, g->points, g->index);
  return check_cuda(cudaGetLastError(), "grid_scatter_kernel launch");
}

// exact nearest target of every query, optionally within a radius
extern "C" int nsb_nn_query(const nsb_nn_grid* g, const double* queries, int n_queries, double radius, double* dist2, int32_t* index,
                            void* stream) {
  if (bad_grid(g) || n_queries < 0 || (n_queries > 0 && (!queries || !dist2 || !index))) { set_error("nsb_nn_query: bad argument"); return NSB_ERR_ARG; }
  if (n_queries == 0) return NSB_OK;
  const double r2 = radius >= 0.0 && std::isfinite(radius) ? radius * radius : INFINITY;
  nn_query_kernel<<<blocks_for(n_queries), kThreads, 0, (cudaStream_t)stream>>>(view_of(g), queries, n_queries, r2, dist2, index);
  return check_cuda(cudaGetLastError(), "nn_query_kernel launch");
}

// one ICP correspondence pass and its sums
extern "C" size_t nsb_icp_workspace(int n_source) { return 8ull * kIcpSums * partial_blocks(n_source); }
extern "C" int nsb_icp_sums(const nsb_nn_grid* g, const double* source, int n_source, const double transform[16], double max_distance,
                            void* ws, size_t ws_bytes, double* sums, void* stream) {
  if (bad_grid(g) || n_source < 0 || !transform || !ws || !sums || (n_source > 0 && !source) || !(max_distance >= 0.0)) {
    set_error("nsb_icp_sums: bad argument"); return NSB_ERR_ARG; }
  if (ws_bytes < nsb_icp_workspace(n_source)) { set_error("nsb_icp_sums: workspace too small"); return NSB_ERR_ARG; }
  Rigid T;
  for (int k = 0; k < 12; k++) T.m[k] = transform[k];
  const unsigned nb = partial_blocks(n_source);
  const cudaStream_t st = (cudaStream_t)stream;
  icp_partial_kernel<<<nb, kThreads, 0, st>>>(view_of(g), source, n_source, T, max_distance * max_distance, static_cast<double*>(ws));
  icp_final_kernel<<<1, 32, 0, st>>>(static_cast<const double*>(ws), (int)nb, sums);
  return check_cuda(cudaGetLastError(), "nsb_icp_sums launch");
}
