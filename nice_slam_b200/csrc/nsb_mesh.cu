// nsb_mesh.cu -- mesh extraction of a fused run's state (Mesher.get_mesh, src/utils/Mesher.py:349-574): the lattice decode (through the
// points mode of the render forward), marching cubes, the scene-hull candidates, the seen masks, culling / components / compaction and the
// vertex colours.  Declarations, rules and the deviations from the reference: include/nice_slam_b200.h, "mesh extraction".
#include <cstdio>
#include <cstring>
#include "nsb_common.cuh"
#include "nsb_geom.cuh"
#include "nsb_mc_table.h"
#include "nsb_scan.cuh"

namespace nsb {
namespace {

constexpr int kThreads = 256;
__constant__ unsigned char c_mc_edge[12][2];
__constant__ unsigned char c_mc_count[256];
__constant__ signed char c_mc_tri[256][3 * NSB_MC_MAX_TRI];

int upload_table() {
  static bool done[64] = {false};
  int dev = 0; cudaGetDevice(&dev);
  if (dev < 64 && done[dev]) return NSB_OK;
  if (check_cuda(cudaMemcpyToSymbol(c_mc_edge, kMcEdge, sizeof(kMcEdge)), "mc table") ||
      check_cuda(cudaMemcpyToSymbol(c_mc_count, kMcTriCount, sizeof(kMcTriCount)), "mc table") ||
      check_cuda(cudaMemcpyToSymbol(c_mc_tri, kMcTri, sizeof(kMcTri)), "mc table")) return NSB_ERR_CUDA;
  if (dev < 64) done[dev] = true;
  return NSB_OK;
}
unsigned blocks_for(long long n) { return (unsigned)((n + kThreads - 1) / kThreads); }

// ---- marching cubes ----------------------------------------------------------------------------------------------------------------
struct Lat { int nx, ny, nz; long long N; };
__device__ __forceinline__ void unravel(const Lat& L, long long p, int& i, int& j, int& k) {
  const long long nyz = (long long)L.ny * L.nz;
  i = (int)(p / nyz); const long long r = p - i * nyz; j = (int)(r / L.nz); k = (int)(r - (long long)j * L.nz);
}
__device__ __forceinline__ long long stride_of(const Lat& L, int a) { return a == 0 ? (long long)L.ny * L.nz : a == 1 ? (long long)L.nz : 1ll; }
// crossed edges owned by point p (its +x, +y, +z edges): bit a
__device__ __forceinline__ int cross_mask(const float* z, const Lat& L, long long p, int i, int j, int k, double level) {
  const bool in0 = (double)z[p] > level;
  const int idx[3] = {i, j, k}, lim[3] = {L.nx, L.ny, L.nz};
  int m = 0;
  for (int a = 0; a < 3; a++)
    if (idx[a] + 1 < lim[a] && (((double)z[p + stride_of(L, a)] > level) != in0)) m |= 1 << a;
  return m;
}
__device__ __forceinline__ int cell_case(const float* z, const Lat& L, long long p, int i, int j, int k, double level) {
  if (i + 1 >= L.nx || j + 1 >= L.ny || k + 1 >= L.nz) return 0;
  int c = 0;
  for (int b = 0; b < 8; b++) {
    const long long q = p + (b & 1) * stride_of(L, 0) + ((b >> 1) & 1) * stride_of(L, 1) + ((b >> 2) & 1);
    if ((double)z[q] > level) c |= 1 << b;
  }
  return c;
}
// counts[p] = (triangles of cell p) << 32 | (crossed edges of point p); counts[N] = 0 (its scan is the total)
__global__ void mc_count_kernel(const float* __restrict__ z, Lat L, double level, unsigned long long* counts) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p > L.N) return;
  if (p == L.N) { counts[p] = 0; return; }
  int i, j, k; unravel(L, p, i, j, k);
  const int m = cross_mask(z, L, p, i, j, k, level);
  counts[p] = ((unsigned long long)c_mc_count[cell_case(z, L, p, i, j, k, level)] << 32) | (unsigned long long)__popc(m);
}
__global__ void mc_totals_kernel(const unsigned long long* scanned, long long N, long long* totals) {
  totals[0] = (long long)(scanned[N] & 0xffffffffull); totals[1] = (long long)(scanned[N] >> 32);
}
__global__ void mc_emit_kernel(const float* __restrict__ z, Lat L, double level, double3 origin, double3 spacing,
                               const unsigned long long* __restrict__ off, double* verts, int* faces, long long* edge_ids) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= L.N) return;
  int i, j, k; unravel(L, p, i, j, k);
  const unsigned long long o = off[p];
  long long v = (long long)(o & 0xffffffffull);
  const int m = cross_mask(z, L, p, i, j, k, level);
  const double org[3] = {origin.x, origin.y, origin.z}, sp[3] = {spacing.x, spacing.y, spacing.z};
  const int idx[3] = {i, j, k};
  for (int a = 0; a < 3; a++) {
    if (!(m >> a & 1)) continue;
    const double z0 = (double)z[p], z1 = (double)z[p + stride_of(L, a)];
    const double t = __ddiv_rn(__dsub_rn(level, z0), __dsub_rn(z1, z0));
    for (int b = 0; b < 3; b++) {
      const double c = b == a ? __dadd_rn((double)idx[b], t) : (double)idx[b];
      verts[3 * v + b] = __dadd_rn(__dmul_rn(c, sp[b]), org[b]);
    }
    if (edge_ids) edge_ids[v] = a * L.N + p;
    v++;
  }
  const int cs = cell_case(z, L, p, i, j, k, level);
  const int nt = c_mc_count[cs];
  if (nt == 0) return;
  long long f = (long long)(o >> 32);
  for (int t = 0; t < nt; t++, f++) {
    for (int c = 0; c < 3; c++) {
      const int e = c_mc_tri[cs][3 * t + c], a = e >> 2, c0 = c_mc_edge[e][0];
      const long long q = p + (c0 & 1) * stride_of(L, 0) + ((c0 >> 1) & 1) * stride_of(L, 1) + ((c0 >> 2) & 1);
      int qi, qj, qk; unravel(L, q, qi, qj, qk);
      const int qm = cross_mask(z, L, q, qi, qj, qk, level);
      faces[3 * f + c] = (int)((off[q] & 0xffffffffull) + __popc(qm & ((1 << a) - 1)));
    }
  }
}

// ---- scene hull --------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool pixel_point(const float* depth, int H, int W, const double* c2w, double fx, double fy, double cx, double cy,
                                            long long id, double p[3]) {
  const long long hw = (long long)H * W;
  const int m = (int)(id / hw); const long long r = id - m * hw;
  const int v = (int)(r / W), u = (int)(r - (long long)v * W);
  const float d = depth[id];
  if (!(d > 0.0f)) return false;
  const double dd = (double)d;
  const double cam[3] = {__dmul_rn(__ddiv_rn((double)u - cx, fx), dd), -__dmul_rn(__ddiv_rn((double)v - cy, fy), dd), -dd};
  const double* T = c2w + 12 * m;
  for (int a = 0; a < 3; a++)
    p[a] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[4 * a], cam[0]), __dmul_rn(T[4 * a + 1], cam[1])), __dmul_rn(T[4 * a + 2], cam[2])), T[4 * a + 3]);
  return true;
}
__device__ __forceinline__ unsigned int ordered_bits(float f) {
  const unsigned int u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
constexpr int kMaxDirs = 256;
__global__ void hull_support_kernel(const float* depth, long long n, int H, int W, const double* c2w, double fx, double fy, double cx, double cy,
                                    const double* dirs, int K, unsigned long long* best) {
  __shared__ unsigned long long s_best[kMaxDirs];
  for (int d = threadIdx.x; d < K; d += blockDim.x) s_best[d] = 0ull;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  for (long long base = (long long)blockIdx.x * blockDim.x; base < n; base += (long long)gridDim.x * blockDim.x) {
    const long long id = base + threadIdx.x;
    double p[3];
    const bool ok = id < n && pixel_point(depth, H, W, c2w, fx, fy, cx, cy, id, p);
    if (!__any_sync(0xffffffffu, ok)) continue;
    for (int d = 0; d < K; d++) {
      unsigned long long key = 0ull;
      if (ok) {
        const float s = (float)__dadd_rn(__dadd_rn(__dmul_rn(dirs[3 * d], p[0]), __dmul_rn(dirs[3 * d + 1], p[1])), __dmul_rn(dirs[3 * d + 2], p[2]));
        key = ((unsigned long long)ordered_bits(s) << 32) | (unsigned long long)(unsigned int)id;
      }
      for (int o = 16; o > 0; o >>= 1) { const unsigned long long t = __shfl_xor_sync(0xffffffffu, key, o); key = t > key ? t : key; }
      if (lane == 0 && key) atomicMax(&s_best[d], key);
    }
  }
  __syncthreads();
  for (int d = threadIdx.x; d < K; d += blockDim.x) if (s_best[d]) atomicMax(&best[d], s_best[d]);
}
__global__ void hull_outside_kernel(const float* depth, long long n, int H, int W, const double* c2w, double fx, double fy, double cx, double cy,
                                    const double* planes, int np, double tol, uint8_t* flag) {
  const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= n) return;
  double p[3];
  uint8_t out = 0;
  if (pixel_point(depth, H, W, c2w, fx, fy, cx, cy, id, p))
    for (int k = 0; k < np && !out; k++) {
      const double* h = planes + 4 * k;
      if (__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(h[0], p[0]), __dmul_rn(h[1], p[1])), __dmul_rn(h[2], p[2])), h[3]) > -tol) out = 1;
    }
  flag[id] = out;
}
__global__ void hull_points_kernel(const float* depth, int H, int W, const double* c2w, double fx, double fy, double cx, double cy,
                                   const long long* ids, int n, double* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double p[3] = {0.0, 0.0, 0.0};
  pixel_point(depth, H, W, c2w, fx, fy, cx, cy, ids[i], p);
  out[3 * i] = p[0]; out[3 * i + 1] = p[1]; out[3 * i + 2] = p[2];
}

// ---- seen masks --------------------------------------------------------------------------------------------------------------------
__global__ void depth_limits_kernel(const float* depth, long long hw, float* out) {
  __shared__ float s_m[kThreads / 32];
  const float* d = depth + (long long)blockIdx.x * hw;
  float m = -INFINITY;
  for (long long i = threadIdx.x; i < hw; i += blockDim.x) m = fmaxf(m, d[i]);
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) s_m[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    m = s_m[0];
    for (int w = 1; w < kThreads / 32; w++) m = fmaxf(m, s_m[w]);
    out[blockIdx.x] = __fmul_rn(m, 1.1f);                                   // torch.max(depth) * 1.1 (Mesher.py:179)
  }
}
// in_frustum (nsb_geom.cuh) is the projection of point_masks and cull_mesh.py
__global__ void seen_kernel(const double* verts, int n, const float* w2c, int M, const float* lim, float fx, float fy, float cx, float cy,
                            float H, float W, uint8_t* seen) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  const float p[3] = {(float)verts[3 * v], (float)verts[3 * v + 1], (float)verts[3 * v + 2]};
  uint8_t s = 0;
  for (int m = 0; m < M && !s; m++) {
    float cz;
    bool ok = in_frustum(w2c + 16 * m, p, fx, fy, cx, cy, H, W, 1e-8f, cz);
    if (lim != nullptr) ok = ok && (-cz < lim[m]);
    s = ok;
  }
  seen[v] = s;
}

// ---- cull_mesh.py -------------------------------------------------------------------------------------------------------------------
// One thread per vertex over P poses.  Rows 0-2 of the poses are staged in shared memory kCullPoses at a time; a thread stops at the
// first pose that sees its vertex, the block at the first tile boundary where all its vertices are seen (threads past V count as seen).
constexpr int kCullPoses = 256;
__global__ void __launch_bounds__(kThreads) cull_seen_kernel(const double* verts, int n, const float* w2c, int P, float fx, float fy,
                                                             float cx, float cy, float H, float W, uint8_t* seen) {
  __shared__ float s_T[kCullPoses * 12];
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  float p[3] = {0.0f, 0.0f, 0.0f};
  if (v < n) { p[0] = (float)verts[3 * v]; p[1] = (float)verts[3 * v + 1]; p[2] = (float)verts[3 * v + 2]; }
  bool s = v >= n;
  for (int base = 0; base < P; base += kCullPoses) {
    if (__syncthreads_and(s)) break;                                        // also: every thread is done with the previous tile
    const int np = P - base < kCullPoses ? P - base : kCullPoses;
    for (int i = threadIdx.x; i < 12 * np; i += blockDim.x) s_T[i] = w2c[16ll * base + 16 * (i / 12) + i % 12];
    __syncthreads();
    for (int m = 0; m < np && !s; m++) { float cz; s = in_frustum(s_T + 12 * m, p, fx, fy, cx, cy, H, W, 1e-5f, cz); }
  }
  if (v < n) seen[v] = s;
}
// keep[f] = 1 iff a vertex of face f is seen (f < F); keep[F] = 0, so that the exclusive scan ends in the total
__global__ void cull_flag_kernel(const int* faces, int F, const uint8_t* seen, unsigned long long* keep) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > F) return;
  keep[f] = f < F && (seen[faces[3 * f]] || seen[faces[3 * f + 1]] || seen[faces[3 * f + 2]]);
}
__global__ void cull_totals_kernel(const unsigned long long* scanned, int F, long long* totals) { totals[0] = (long long)scanned[F]; }
__global__ void cull_emit_kernel(const unsigned long long* scanned, int F, int* kept) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f < F && scanned[f + 1] != scanned[f]) kept[scanned[f]] = f;
}

// ---- culling, components, compaction ----------------------------------------------------------------------------------------------
struct CleanWs {
  int* parent;                   // [F] union-find over faces
  unsigned long long* keys;      // [T] edge hash table
  int* vals;                     // [T]
  double* area;                  // [F] component area at its root
  unsigned long long* fkeep;     // [F+1] -> exclusive scan = new face index
  unsigned long long* vused;     // [V+1] -> exclusive scan = new vertex index
  unsigned long long* best;      // [2] largest component: max area bits, root
  unsigned long long* scan_ws;
  long long T;
};
long long table_size(int F) { long long t = 64; while (t < 6ll * F) t <<= 1; return t; }
size_t clean_layout(int V, int F, void* base, CleanWs* w) {
  const long long T = table_size(F);
  const size_t sws = scan_ws_elems((long long)(V > F ? V : F) + 1);
  const size_t sizes[] = {align16(4ull * F), align16(8ull * T), align16(4ull * T), align16(8ull * F), align16(8ull * (F + 1)),
                          align16(8ull * (V + 1)), 16, align16(8 * sws)};
  size_t off = 0, offs[8];
  for (int i = 0; i < 8; i++) { offs[i] = off; off += sizes[i]; }
  if (w) {
    char* b = static_cast<char*>(base);
    w->parent = reinterpret_cast<int*>(b + offs[0]); w->keys = reinterpret_cast<unsigned long long*>(b + offs[1]);
    w->vals = reinterpret_cast<int*>(b + offs[2]); w->area = reinterpret_cast<double*>(b + offs[3]);
    w->fkeep = reinterpret_cast<unsigned long long*>(b + offs[4]); w->vused = reinterpret_cast<unsigned long long*>(b + offs[5]);
    w->best = reinterpret_cast<unsigned long long*>(b + offs[6]); w->scan_ws = reinterpret_cast<unsigned long long*>(b + offs[7]); w->T = T;
  }
  return off;
}
__global__ void clean_init_kernel(CleanWs w, int F, int V) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < F) { w.parent[i] = (int)i; w.area[i] = 0.0; }
  if (i < w.T) { w.keys[i] = ~0ull; w.vals[i] = -1; }
  if (i <= V) w.vused[i] = 0ull;
  if (i <= F) w.fkeep[i] = 0ull;
  if (i < 2) w.best[i] = i == 0 ? 0ull : ~0ull;
}
__device__ __forceinline__ bool face_seen(const int* f, const uint8_t* seen) { return seen[f[0]] || seen[f[1]] || seen[f[2]]; }
__device__ __forceinline__ int uf_find(int* parent, int x) {
  while (true) { const int p = parent[x]; if (p == x) return x; x = p; }
}
__device__ __forceinline__ void uf_union(int* parent, int a, int b) {
  while (true) {
    a = uf_find(parent, a); b = uf_find(parent, b);
    if (a == b) return;
    if (a < b) { const int t = a; a = b; b = t; }                          // the larger root goes under the smaller: root = smallest face
    if (atomicCAS(&parent[a], a, b) == a) return;
  }
}
__device__ __forceinline__ unsigned long long mix64(unsigned long long k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33; return k;
}
__global__ void edge_union_kernel(const int* faces, int F, const uint8_t* seen, CleanWs w) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3ll * F) return;
  const int f = (int)(i / 3), e = (int)(i - 3ll * f);
  const int* fv = faces + 3 * f;
  if (!face_seen(fv, seen)) return;
  const int a = fv[e], b = fv[e == 2 ? 0 : e + 1];
  const unsigned long long key = ((unsigned long long)(unsigned)min(a, b) << 32) | (unsigned)max(a, b);
  for (long long h = (long long)(mix64(key) & (unsigned long long)(w.T - 1));; h = (h + 1) & (w.T - 1)) {
    const unsigned long long prev = atomicCAS(&w.keys[h], ~0ull, key);
    if (prev == ~0ull || prev == key) {
      const int other = atomicExch(&w.vals[h], f);
      if (other >= 0) uf_union(w.parent, f, other);
      return;
    }
  }
}
__global__ void area_kernel(const double* verts, const int* faces, int F, const uint8_t* seen, CleanWs w) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const int* fv = faces + 3 * f;
  if (!face_seen(fv, seen)) return;
  const int r = uf_find(w.parent, f);
  w.parent[f] = r;
  const double* A = verts + 3 * fv[0]; const double* B = verts + 3 * fv[1]; const double* C = verts + 3 * fv[2];
  const double u[3] = {B[0] - A[0], B[1] - A[1], B[2] - A[2]}, v[3] = {C[0] - A[0], C[1] - A[1], C[2] - A[2]};
  const double c0 = u[1] * v[2] - u[2] * v[1], c1 = u[2] * v[0] - u[0] * v[2], c2 = u[0] * v[1] - u[1] * v[0];
  atomicAdd(&w.area[r], sqrt(c0 * c0 + c1 * c1 + c2 * c2) * 0.5);
}
__global__ void largest_kernel(int F, CleanWs w, int pass) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F || w.parent[f] != f) return;
  const unsigned long long bits = (unsigned long long)__double_as_longlong(w.area[f]);      // areas >= 0: the bits order as the values
  if (pass == 0) atomicMax(&w.best[0], bits);
  else if (bits == w.best[0]) atomicMin(&w.best[1], (unsigned long long)f);
}
__global__ void keep_kernel(const int* faces, int F, const uint8_t* seen, double threshold, int largest, CleanWs w) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const int* fv = faces + 3 * f;
  if (!face_seen(fv, seen)) return;
  const int r = w.parent[f];
  const bool keep = largest ? (unsigned long long)r == w.best[1] : w.area[r] > threshold;
  if (!keep) return;
  w.fkeep[f] = 1ull;
  w.vused[fv[0]] = 1ull; w.vused[fv[1]] = 1ull; w.vused[fv[2]] = 1ull;
}
__global__ void clean_totals_kernel(CleanWs w, int V, int F, long long* totals) {
  totals[0] = (long long)w.vused[V]; totals[1] = (long long)w.fkeep[F];
}
__global__ void compact_kernel(const double* verts, int V, const int* faces, int F, CleanWs w, double* ov, int* of) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < V && w.vused[i + 1] != w.vused[i]) {
    const long long j = (long long)w.vused[i];
    ov[3 * j] = verts[3 * i]; ov[3 * j + 1] = verts[3 * i + 1]; ov[3 * j + 2] = verts[3 * i + 2];
  }
  if (i < F && w.fkeep[i + 1] != w.fkeep[i]) {
    const long long j = (long long)w.fkeep[i];
    for (int c = 0; c < 3; c++) of[3 * j + c] = (int)w.vused[faces[3 * i + c]];
  }
}

__global__ void colors_kernel(const float* raw, int n, uint8_t* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3 * n) return;
  const int v = i / 3, c = i - 3 * v;
  const float x = fminf(fmaxf(raw[4 * v + c], 0.0f), 1.0f);               // np.clip(rgb, 0, 1) * 255, astype(np.uint8)
  out[i] = (uint8_t)(int)__fmul_rn(x, 255.0f);
}

Lat make_lat(const int32_t n[3]) { Lat L; L.nx = n[0]; L.ny = n[1]; L.nz = n[2]; L.N = (long long)n[0] * n[1] * n[2]; return L; }
bool bad_lattice(const int32_t* n) {
  if (!n || n[0] < 2 || n[1] < 2 || n[2] < 2 || (long long)n[0] * n[1] * n[2] >= (1ll << 31)) {
    set_error("mesh lattice: every axis needs >= 2 points and the lattice < 2^31 points"); return true; }
  return false;
}

}  // namespace
}  // namespace nsb

using namespace nsb;

// Mesher.get_grid_uniform + eval_points at stage 'fine' + the hull mask (Mesher.py:321-347, 281-319, 421-433)
extern "C" int nsb_mesh_lattice_eval(const nsb_render_inputs* in, const nsb_mesh_lattice* lat, float* z, void* stream) {
  if (!in || !lat || !z) { set_error("nsb_mesh_lattice_eval: NULL argument"); return NSB_ERR_ARG; }
  if (bad_lattice(lat->n)) return NSB_ERR_ARG;
  if (in->stage != NSB_STAGE_FINE) { set_error("nsb_mesh_lattice_eval: stage must be fine (Mesher.py:429)"); return NSB_ERR_ARG; }
  if (lat->n_planes < 0 || (lat->n_planes > 0 && !lat->planes)) { set_error("nsb_mesh_lattice_eval: planes missing"); return NSB_ERR_ARG; }
  return eval_points_mesh(in, nullptr, lat, lat->n[0] * lat->n[1] * lat->n[2], nullptr, z, stream);
}

// direct_point_query (Mesher.py:513-524, 555-556)
extern "C" int nsb_mesh_colors(const nsb_render_inputs* in, const double* vertices, int n, float* raw, uint8_t* colors, void* stream) {
  if (n < 0 || (n > 0 && (!vertices || !raw || !colors))) { set_error("nsb_mesh_colors: NULL argument"); return NSB_ERR_ARG; }
  if (in && in->stage != NSB_STAGE_COLOR) { set_error("nsb_mesh_colors: stage must be color (Mesher.py:520)"); return NSB_ERR_ARG; }
  if (n == 0) return NSB_OK;
  int rc = eval_points_mesh(in, vertices, nullptr, n, raw, nullptr, stream); if (rc) return rc;
  colors_kernel<<<blocks_for(3ll * n), kThreads, 0, (cudaStream_t)stream>>>(raw, n, colors);
  return check_cuda(cudaGetLastError(), "colors_kernel launch");
}

// skimage.measure.marching_cubes (Mesher.py:437-467): per-point counts + scan, then emit
extern "C" size_t nsb_mc_workspace(long long n_points) { return align16(8ull * (n_points + 1)) + 8ull * scan_ws_elems(n_points + 1); }
extern "C" int nsb_mc_count(const float* z, const int32_t n[3], double level, void* ws, size_t ws_bytes, long long* totals, void* stream) {
  if (!z || !ws || !totals) { set_error("nsb_mc_count: NULL argument"); return NSB_ERR_ARG; }
  if (bad_lattice(n)) return NSB_ERR_ARG;
  const Lat L = make_lat(n);
  if (ws_bytes < nsb_mc_workspace(L.N)) { set_error("nsb_mc_count: workspace %zu < %zu bytes", ws_bytes, nsb_mc_workspace(L.N)); return NSB_ERR_ARG; }
  int rc = upload_table(); if (rc) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* counts = static_cast<unsigned long long*>(ws);
  mc_count_kernel<<<blocks_for(L.N + 1), kThreads, 0, st>>>(z, L, level, counts);
  if ((rc = check_cuda(cudaGetLastError(), "mc_count_kernel launch"))) return rc;
  if ((rc = excl_scan(counts, L.N + 1, reinterpret_cast<unsigned long long*>(static_cast<char*>(ws) + align16(8ull * (L.N + 1))), st))) return rc;
  mc_totals_kernel<<<1, 1, 0, st>>>(counts, L.N, totals);
  return check_cuda(cudaGetLastError(), "mc_totals_kernel launch");
}
extern "C" int nsb_mc_emit(const float* z, const int32_t n[3], double level, const double origin[3], const double spacing[3], const void* ws,
                           double* vertices, int32_t* faces, long long* edge_ids, void* stream) {
  if (!z || !ws || !origin || !spacing || !vertices || !faces) { set_error("nsb_mc_emit: NULL argument"); return NSB_ERR_ARG; }
  if (bad_lattice(n)) return NSB_ERR_ARG;
  int rc = upload_table(); if (rc) return rc;
  const Lat L = make_lat(n);
  mc_emit_kernel<<<blocks_for(L.N), kThreads, 0, (cudaStream_t)stream>>>(z, L, level, make_double3(origin[0], origin[1], origin[2]),
      make_double3(spacing[0], spacing[1], spacing[2]), static_cast<const unsigned long long*>(ws), vertices, faces, edge_ids);
  return check_cuda(cudaGetLastError(), "mc_emit_kernel launch");
}

// get_bound_from_frames' candidates (Mesher.py:214-279)
extern "C" int nsb_mesh_hull_support(const float* depth, int M, int H, int W, const double* c2w, double fx, double fy, double cx, double cy,
                                     const double* dirs, int K, unsigned long long* best, void* stream) {
  if (!depth || !c2w || !dirs || !best || M < 1 || H < 1 || W < 1 || K < 1 || K > kMaxDirs || (long long)M * H * W >= (1ll << 32)) {
    set_error("nsb_mesh_hull_support: bad argument (1 <= K <= %d, M*H*W < 2^32)", kMaxDirs); return NSB_ERR_ARG; }
  const long long n = (long long)M * H * W;
  const unsigned grid = (unsigned)(blocks_for(n) < 1056u ? blocks_for(n) : 1056u);
  hull_support_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(depth, n, H, W, c2w, fx, fy, cx, cy, dirs, K, best);
  return check_cuda(cudaGetLastError(), "hull_support_kernel launch");
}
extern "C" int nsb_mesh_hull_outside(const float* depth, int M, int H, int W, const double* c2w, double fx, double fy, double cx, double cy,
                                     const double* planes, int n_planes, double tol, uint8_t* flag, void* stream) {
  if (!depth || !c2w || !flag || M < 1 || H < 1 || W < 1 || n_planes < 0 || (n_planes > 0 && !planes)) {
    set_error("nsb_mesh_hull_outside: bad argument"); return NSB_ERR_ARG; }
  const long long n = (long long)M * H * W;
  hull_outside_kernel<<<blocks_for(n), kThreads, 0, (cudaStream_t)stream>>>(depth, n, H, W, c2w, fx, fy, cx, cy, planes, n_planes, tol, flag);
  return check_cuda(cudaGetLastError(), "hull_outside_kernel launch");
}
extern "C" int nsb_mesh_hull_points(const float* depth, int H, int W, const double* c2w, double fx, double fy, double cx, double cy,
                                    const long long* ids, int n, double* points, void* stream) {
  if (n < 0 || (n > 0 && (!depth || !c2w || !ids || !points))) { set_error("nsb_mesh_hull_points: bad argument"); return NSB_ERR_ARG; }
  if (n == 0) return NSB_OK;
  hull_points_kernel<<<blocks_for(n), kThreads, 0, (cudaStream_t)stream>>>(depth, H, W, c2w, fx, fy, cx, cy, ids, n, points);
  return check_cuda(cudaGetLastError(), "hull_points_kernel launch");
}

// point_masks (Mesher.py:53-212), the seen output
extern "C" int nsb_mesh_depth_limits(const float* depth, int M, long long hw, float* out, void* stream) {
  if (M < 0 || hw < 1 || (M > 0 && (!depth || !out))) { set_error("nsb_mesh_depth_limits: bad argument"); return NSB_ERR_ARG; }
  if (M == 0) return NSB_OK;
  depth_limits_kernel<<<M, kThreads, 0, (cudaStream_t)stream>>>(depth, hw, out);
  return check_cuda(cudaGetLastError(), "depth_limits_kernel launch");
}
extern "C" int nsb_mesh_seen(const double* vertices, int n, const float* w2c, int M, const float* lim, double fx, double fy, double cx, double cy,
                             int H, int W, uint8_t* seen, void* stream) {
  if (n < 0 || M < 0 || (n > 0 && (!vertices || !seen || (M > 0 && !w2c)))) { set_error("nsb_mesh_seen: bad argument"); return NSB_ERR_ARG; }
  if (n == 0) return NSB_OK;
  seen_kernel<<<blocks_for(n), kThreads, 0, (cudaStream_t)stream>>>(vertices, n, w2c, M, lim, (float)fx, (float)fy, (float)cx, (float)cy,
                                                                     (float)H, (float)W, seen);
  return check_cuda(cudaGetLastError(), "seen_kernel launch");
}

// cull_mesh.py:47-75: the seen mask over every pose, then the faces with a seen vertex
extern "C" int nsb_cull_seen(const double* vertices, int n, const float* w2c, int P, double fx, double fy, double cx, double cy, int H, int W,
                             uint8_t* seen, void* stream) {
  if (n < 0 || P < 0 || (n > 0 && (!vertices || !seen || (P > 0 && !w2c)))) { set_error("nsb_cull_seen: NULL pointer or negative count"); return NSB_ERR_ARG; }
  if (H < 1 || W < 1 || !isfinite(fx) || !isfinite(fy) || !isfinite(cx) || !isfinite(cy)) {
    set_error("nsb_cull_seen: H and W must be >= 1 and the intrinsics finite (H %d, W %d)", H, W); return NSB_ERR_ARG; }
  if (n == 0) return NSB_OK;
  cull_seen_kernel<<<blocks_for(n), kThreads, 0, (cudaStream_t)stream>>>(vertices, n, w2c, P, (float)fx, (float)fy, (float)cx, (float)cy,
                                                                         (float)H, (float)W, seen);
  return check_cuda(cudaGetLastError(), "cull_seen_kernel launch");
}
extern "C" size_t nsb_cull_faces_workspace(int F) { return F < 0 ? 0 : align16(8ull * (F + 1)) + 8ull * scan_ws_elems((long long)F + 1); }
extern "C" int nsb_cull_faces(const int32_t* faces, int F, const uint8_t* seen, void* ws, size_t ws_bytes, long long* totals, void* stream) {
  if (F < 0 || !ws || !totals || (F > 0 && (!faces || !seen))) { set_error("nsb_cull_faces: NULL pointer or negative count"); return NSB_ERR_ARG; }
  if (ws_bytes < nsb_cull_faces_workspace(F)) { set_error("nsb_cull_faces: workspace %zu < %zu bytes", ws_bytes, nsb_cull_faces_workspace(F)); return NSB_ERR_ARG; }
  const cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* keep = static_cast<unsigned long long*>(ws);
  cull_flag_kernel<<<blocks_for((long long)F + 1), kThreads, 0, st>>>(faces, F, seen, keep);
  int rc = check_cuda(cudaGetLastError(), "cull_flag_kernel launch"); if (rc) return rc;
  if ((rc = excl_scan(keep, (long long)F + 1, reinterpret_cast<unsigned long long*>(static_cast<char*>(ws) + align16(8ull * (F + 1))), st))) return rc;
  cull_totals_kernel<<<1, 1, 0, st>>>(keep, F, totals);
  return check_cuda(cudaGetLastError(), "cull_totals_kernel launch");
}
extern "C" int nsb_cull_faces_emit(int F, const void* ws, int32_t* kept, void* stream) {
  if (F < 0 || !ws || (F > 0 && !kept)) { set_error("nsb_cull_faces_emit: NULL pointer or negative count"); return NSB_ERR_ARG; }
  if (F == 0) return NSB_OK;
  cull_emit_kernel<<<blocks_for(F), kThreads, 0, (cudaStream_t)stream>>>(static_cast<const unsigned long long*>(ws), F, kept);
  return check_cuda(cudaGetLastError(), "cull_emit_kernel launch");
}

// culling + trimesh's split + the area filter + compaction (Mesher.py:469-511)
extern "C" size_t nsb_mesh_clean_workspace(int V, int F) { return clean_layout(V, F, nullptr, nullptr); }
extern "C" int nsb_mesh_clean(const double* verts, int V, const int32_t* faces, int F, const uint8_t* seen, double threshold, int largest,
                              void* ws, size_t ws_bytes, long long* totals, void* stream) {
  if (V < 0 || F < 0 || !ws || !totals || (F > 0 && (!verts || !faces || !seen))) { set_error("nsb_mesh_clean: bad argument"); return NSB_ERR_ARG; }
  if (ws_bytes < nsb_mesh_clean_workspace(V, F)) { set_error("nsb_mesh_clean: workspace too small"); return NSB_ERR_ARG; }
  const cudaStream_t st = (cudaStream_t)stream;
  CleanWs w; clean_layout(V, F, ws, &w);
  const long long n0 = w.T > (long long)V + 1 ? w.T : (long long)V + 1;
  clean_init_kernel<<<blocks_for(n0), kThreads, 0, st>>>(w, F, V);
  if (F > 0) {
    edge_union_kernel<<<blocks_for(3ll * F), kThreads, 0, st>>>(faces, F, seen, w);
    area_kernel<<<blocks_for(F), kThreads, 0, st>>>(verts, faces, F, seen, w);
    if (largest) {
      largest_kernel<<<blocks_for(F), kThreads, 0, st>>>(F, w, 0);
      largest_kernel<<<blocks_for(F), kThreads, 0, st>>>(F, w, 1);
    }
    keep_kernel<<<blocks_for(F), kThreads, 0, st>>>(faces, F, seen, threshold, largest, w);
  }
  int rc = check_cuda(cudaGetLastError(), "mesh clean launch"); if (rc) return rc;
  if ((rc = excl_scan(w.fkeep, (long long)F + 1, w.scan_ws, st))) return rc;
  if ((rc = excl_scan(w.vused, (long long)V + 1, w.scan_ws, st))) return rc;
  clean_totals_kernel<<<1, 1, 0, st>>>(w, V, F, totals);
  return check_cuda(cudaGetLastError(), "clean_totals_kernel launch");
}
extern "C" int nsb_mesh_compact(const double* verts, int V, const int32_t* faces, int F, const void* ws, double* ov, int32_t* of, void* stream) {
  if (V < 0 || F < 0 || !ws) { set_error("nsb_mesh_compact: bad argument"); return NSB_ERR_ARG; }
  CleanWs w; clean_layout(V, F, const_cast<void*>(ws), &w);
  const int n = V > F ? V : F;
  if (n == 0) return NSB_OK;
  compact_kernel<<<blocks_for(n), kThreads, 0, (cudaStream_t)stream>>>(verts, V, faces, F, w, ov, of);
  return check_cuda(cudaGetLastError(), "compact_kernel launch");
}
