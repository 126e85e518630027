// nsb_det.cu -- the ordered reductions of the deterministic mode (option "deterministic"; DESIGN.md "Deterministic mode").
//
// With the option on, the tile backward (nsb_tile.cuh, kDet instantiations) does not add into the voxel and decoder-weight gradients: it
// writes each point's dL/dc and normalised coordinate, and each tile's weight-gradient partial image, to the split workspace.  The passes
// here then sum them in an order fixed by the data alone:
//   voxel gradients: the (voxel key, point, corner) list of every in-grid corner, sorted stably by key (CUB radix sort; the list is built in
//     ascending (point, corner) order, so that order survives inside a key), one sequential float32 sum per voxel and channel, starting
//     from the gradient's current value and adding fl(w * dc) -- the product the default scatter adds -- in ascending (point, corner) order;
//   weight gradients: for every element of a decoder's packed gradient image, the per-tile partials added in ascending tile order.
#include <cub/cub.cuh>
#include "nsb_common.cuh"
#include "nsb_geom.cuh"

namespace nsb {
namespace det {

constexpr int kThreads = 256;
constexpr int kUnroll = 8;                      // contributions whose loads are in flight together in the per-voxel sum

// entry i = 8 p + k: key of corner k of point p (the slot, or the linear voxel of a dense grid), `invalid` for a corner outside the grid or
// a voxel with slot -1 -- the corners the default scatter skips
__global__ void __launch_bounds__(kThreads) build_kernel(const float* __restrict__ xn, long long n_entries, int W, int H, int D,
                                                         const int32_t* __restrict__ slots, uint32_t invalid, uint32_t* __restrict__ keys,
                                                         uint32_t* __restrict__ vals) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= n_entries) return;
  const long long p = i >> 3;
  const int k = (int)(i & 7);
  const float x[3] = {xn[3 * p], xn[3 * p + 1], xn[3 * p + 2]};
  const Tri t = make_tri(x, W, H, D);
  int cx, cy, cz;
  uint32_t key = invalid;
  if (tri_corner(t, k, W, H, D, cx, cy, cz)) {
    const long long v = ((long long)cz * H + cy) * W + cx;
    if (slots == nullptr) key = (uint32_t)v;
    else { const int s = __ldg(slots + v); if (s >= 0) key = (uint32_t)s; }
  }
  keys[i] = key;
  vals[i] = (uint32_t)i;
}

// one warp per run of equal keys, lane = channel: d_grid[voxel][lane] += fl(w * dc[p][lane]) over the run's entries in their (sorted) order
__global__ void __launch_bounds__(kThreads) segment_kernel(const uint32_t* __restrict__ ukeys, const uint32_t* __restrict__ counts,
                                                           const uint32_t* __restrict__ offs, const int* __restrict__ num_runs, uint32_t invalid,
                                                           const uint32_t* __restrict__ vals, const float* __restrict__ xn,
                                                           const float* __restrict__ dc, nsb_grid g, int compact, float* __restrict__ dgrid) {
  const int lane = threadIdx.x & 31;
  const int nw = gridDim.x * (kThreads / 32);
  const int runs = *num_runs;
  for (int r = blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5); r < runs; r += nw) {
    const uint32_t key = ukeys[r];
    if (key == invalid) continue;
    long long addr;
    if (compact) addr = (long long)key * 32 + lane;
    else {
      const int cx = (int)(key % (uint32_t)g.W), cy = (int)((key / (uint32_t)g.W) % (uint32_t)g.H), cz = (int)(key / ((uint32_t)g.W * (uint32_t)g.H));
      addr = cz * g.stride_d + cy * g.stride_h + cx * g.stride_w + (long long)lane * g.stride_c;
    }
    const uint32_t j0 = offs[r], n = counts[r];
    float acc = dgrid[addr];
    for (uint32_t j = 0; j < n; j += kUnroll) {
      float pr[kUnroll];
#pragma unroll
      for (int u = 0; u < kUnroll; u++) {
        pr[u] = 0.0f;
        if (j + u < n) {
          const uint32_t e = vals[j0 + j + u];
          const uint32_t p = e >> 3;
          const float x[3] = {xn[3 * (size_t)p], xn[3 * (size_t)p + 1], xn[3 * (size_t)p + 2]};
          const Tri t = make_tri(x, g.W, g.H, g.D);
          pr[u] = __fmul_rn(tri_weight(t, (int)(e & 7)), dc[(size_t)p * 32 + lane]);
        }
      }
#pragma unroll
      for (int u = 0; u < kUnroll; u++)
        if (j + u < n) acc = __fadd_rn(acc, pr[u]);
    }
    dgrid[addr] = acc;
  }
}

// out[e] = sum over tiles t = 0, 1, ... of part[t][e] (float32, in that order)
__global__ void __launch_bounds__(kThreads) tile_sum_kernel(const float* __restrict__ part, int tiles, int nf, float* __restrict__ out) {
  const int e = blockIdx.x * kThreads + threadIdx.x;
  if (e >= nf) return;
  float acc = 0.0f;
  for (int t = 0; t < tiles; t += kUnroll) {
    float v[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; u++) v[u] = t + u < tiles ? __ldcs(part + (size_t)(t + u) * nf + e) : 0.0f;
#pragma unroll
    for (int u = 0; u < kUnroll; u++)
      if (t + u < tiles) acc = __fadd_rn(acc, v[u]);
  }
  out[e] = acc;
}

static int key_bits(long long n_voxels) {       // bits of the keys 0 .. n_voxels (n_voxels = the invalid key)
  int b = 1;
  while (b < 32 && (1ll << b) <= n_voxels) b++;
  return b;
}

struct VoxelWs { uint32_t *keys_in, *vals_in, *keys_out, *vals_out, *offs; int* num_runs; void* temp; size_t temp_bytes; };
static size_t temp_bytes(long long m, int end_bit) {
  size_t a = 0, b = 0, c = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, a, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)m, 0, end_bit);
  cub::DeviceRunLengthEncode::Encode(nullptr, b, (const uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr, (int*)nullptr, (int)m);
  cub::DeviceScan::ExclusiveSum(nullptr, c, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)m);
  return a > b ? (a > c ? a : c) : (b > c ? b : c);
}
// workspace: keys / values before and after the sort, run offsets (m entries each), the run count, CUB's scratch
static size_t carve(void* base, long long n_points, VoxelWs* w) {
  const long long m = 8 * n_points;
  size_t o = 0;
  auto take = [&](size_t bytes) { const size_t r = o; o = align16(o + bytes); return r; };
  const size_t o_ki = take(4 * m), o_vi = take(4 * m), o_ko = take(4 * m), o_vo = take(4 * m), o_of = take(4 * m), o_nr = take(16);
  const size_t tb = temp_bytes(m, 32);
  const size_t o_t = take(tb);
  if (w != nullptr) {
    char* b = static_cast<char*>(base);
    w->keys_in = (uint32_t*)(b + o_ki); w->vals_in = (uint32_t*)(b + o_vi); w->keys_out = (uint32_t*)(b + o_ko); w->vals_out = (uint32_t*)(b + o_vo);
    w->offs = (uint32_t*)(b + o_of); w->num_runs = (int*)(b + o_nr); w->temp = b + o_t; w->temp_bytes = tb;
  }
  return o;
}

}  // namespace det

size_t det_voxel_workspace_bytes(long long n_points) { return n_points < 1 ? 0 : det::carve(nullptr, n_points, nullptr); }

int det_voxel_reduce(const nsb_grid& g, const int32_t* slot_map, const float* xn, const float* dc, long long n_points, float* d_grid,
                     void* workspace, size_t workspace_bytes, cudaStream_t st) {
  using namespace det;
  if (n_points == 0) return NSB_OK;
  const long long n_vox = (long long)g.D * g.H * g.W;
  if (n_points < 0 || n_points >= (1ll << 28) || n_vox >= 0xffffffffll) {
    set_error("ordered voxel gradient: %lld points / %lld voxels exceed the 32-bit (point, corner) and voxel keys", n_points, n_vox); return NSB_ERR_ARG; }
  if (workspace == nullptr || (reinterpret_cast<uintptr_t>(workspace) & 15) || workspace_bytes < det_voxel_workspace_bytes(n_points)) {
    set_error("ordered voxel gradient: workspace missing, unaligned or smaller than %zu bytes", det_voxel_workspace_bytes(n_points)); return NSB_ERR_ARG; }
  VoxelWs w; carve(workspace, n_points, &w);
  const long long m = 8 * n_points;
  const uint32_t invalid = (uint32_t)n_vox;
  const int end_bit = key_bits(n_vox);
  build_kernel<<<(unsigned)((m + kThreads - 1) / kThreads), kThreads, 0, st>>>(xn, m, g.W, g.H, g.D, slot_map, invalid, w.keys_in, w.vals_in);
  if (check_cuda(cudaGetLastError(), "ordered voxel gradient: build_kernel launch")) return NSB_ERR_CUDA;
  size_t tb = w.temp_bytes;
  if (check_cuda(cub::DeviceRadixSort::SortPairs(w.temp, tb, w.keys_in, w.keys_out, w.vals_in, w.vals_out, (int)m, 0, end_bit, st), "cub SortPairs"))
    return NSB_ERR_CUDA;
  // (the sort's inputs are dead: the run keys and lengths go there)
  tb = w.temp_bytes;
  if (check_cuda(cub::DeviceRunLengthEncode::Encode(w.temp, tb, w.keys_out, w.keys_in, w.vals_in, w.num_runs, (int)m, st), "cub Encode"))
    return NSB_ERR_CUDA;
  tb = w.temp_bytes;
  if (check_cuda(cub::DeviceScan::ExclusiveSum(w.temp, tb, w.vals_in, w.offs, (int)m, st), "cub ExclusiveSum")) return NSB_ERR_CUDA;
  int dev = 0, sms = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); if (sms <= 0) sms = 132;
  const long long want = (m + (kThreads / 32) - 1) / (kThreads / 32);
  const unsigned blocks = (unsigned)(want < 16ll * sms ? want : 16ll * sms);
  segment_kernel<<<blocks, kThreads, 0, st>>>(w.keys_in, w.vals_in, w.offs, w.num_runs, invalid, w.vals_out, xn, dc, g, slot_map != nullptr ? 1 : 0, d_grid);
  return check_cuda(cudaGetLastError(), "ordered voxel gradient: segment_kernel launch");
}

int det_tile_sum(const float* part, int tiles, int n_floats, float* out, cudaStream_t st) {
  if (tiles < 1 || n_floats < 1) return NSB_OK;
  det::tile_sum_kernel<<<(n_floats + det::kThreads - 1) / det::kThreads, det::kThreads, 0, st>>>(part, tiles, n_floats, out);
  return check_cuda(cudaGetLastError(), "ordered weight gradient: tile_sum_kernel launch");
}

}  // namespace nsb

using namespace nsb;

extern "C" size_t nsb_voxel_grad_ordered_workspace(int n_points) { return det_voxel_workspace_bytes(n_points); }

extern "C" int nsb_voxel_grad_ordered(const nsb_grid* grid, const int32_t* slot_map, const float* xn, const float* dc, int n_points, float* d_grid,
                                      void* workspace, size_t workspace_bytes, void* stream) {
  if (grid == nullptr || grid->D < 1 || grid->H < 1 || grid->W < 1) { set_error("nsb_voxel_grad_ordered: grid shape missing"); return NSB_ERR_ARG; }
  if (n_points < 0) { set_error("nsb_voxel_grad_ordered: n_points < 0"); return NSB_ERR_ARG; }
  if (n_points > 0 && (!xn || !dc || !d_grid)) { set_error("nsb_voxel_grad_ordered: xn / dc / d_grid missing"); return NSB_ERR_ARG; }
  return det_voxel_reduce(*grid, slot_map, xn, dc, n_points, d_grid, workspace, workspace_bytes, (cudaStream_t)stream);
}
