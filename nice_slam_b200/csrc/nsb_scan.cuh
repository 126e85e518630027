// nsb_scan.cuh -- exclusive scan in place, x[i] <- sum_{j<i} x[j], shared by the mesh (u64 counts) and reconstruction-metric (f64 face
// areas, u64 cell counts) code: three kernels per level, the block sums scanned recursively.  The order of the additions depends on n
// alone, so a float scan gives the same bits on every call.
#pragma once
#include <cuda_runtime.h>
#include "nsb_common.cuh"

namespace nsb {
namespace {

constexpr int kScanThreads = 256;
constexpr int kScanItems = 4;                       // per thread
constexpr long long kScanBlock = (long long)kScanThreads * kScanItems;
template <typename T>
__device__ __forceinline__ T block_excl_scan(T v, T* total) {
  __shared__ T s_w[kScanThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T inc = v;
  for (int o = 1; o < 32; o <<= 1) { const T t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
  if (lane == 31) s_w[warp] = inc;
  __syncthreads();
  T base = 0, all = 0;
  for (int w = 0; w < kScanThreads / 32; w++) { if (w < warp) base += s_w[w]; all += s_w[w]; }
  __syncthreads();
  *total = all;
  return base + inc - v;
}
template <typename T>
__global__ void scan_blocks_kernel(T* x, long long n, T* sums) {
  const long long b0 = (long long)blockIdx.x * kScanBlock + (long long)threadIdx.x * kScanItems;
  T v[kScanItems], s = 0;
#pragma unroll
  for (int i = 0; i < kScanItems; i++) { v[i] = b0 + i < n ? x[b0 + i] : T(0); s += v[i]; }
  T total;
  T run = block_excl_scan(s, &total);
#pragma unroll
  for (int i = 0; i < kScanItems; i++) { if (b0 + i < n) x[b0 + i] = run; run += v[i]; }
  if (threadIdx.x == 0) sums[blockIdx.x] = total;
}
template <typename T>
__global__ void scan_add_kernel(T* x, long long n, const T* sums) {
  const long long i = (long long)blockIdx.x * kScanBlock + threadIdx.x;
  for (int k = 0; k < kScanItems; k++) { const long long j = i + (long long)k * kScanThreads; if (j < n) x[j] += sums[blockIdx.x]; }
}
// workspace of excl_scan over n elements, in elements of T
size_t scan_ws_elems(long long n) {
  size_t t = 0;
  for (long long m = n; m > 1; m = (m + kScanBlock - 1) / kScanBlock) t += (size_t)((m + kScanBlock - 1) / kScanBlock);
  return t + 1;
}
template <typename T>
int excl_scan(T* x, long long n, T* ws, cudaStream_t st) {
  if (n <= 0) return NSB_OK;
  const long long nb = (n + kScanBlock - 1) / kScanBlock;
  scan_blocks_kernel<T><<<(unsigned)nb, kScanThreads, 0, st>>>(x, n, ws);
  if (nb > 1) {
    int rc = excl_scan(ws, nb, ws + nb, st); if (rc) return rc;
    scan_add_kernel<T><<<(unsigned)nb, kScanThreads, 0, st>>>(x, n, ws);
  }
  return check_cuda(cudaGetLastError(), "scan");
}

}  // namespace
}  // namespace nsb
