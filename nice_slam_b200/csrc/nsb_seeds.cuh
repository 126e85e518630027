// nsb_seeds.cuh -- device bodies of the loss-seed computations (Tracker.py:108-123, Mapper.py:487-493), the d c2w sums and the peer-memory
// exchange helpers.  Used by the stand-alone single-CTA kernels of nsb_aux.cu and, fused, by the LAST CTA of the render kernels
// (nsb_render.cu): for small batches the loss seeds are produced by the forward launch itself.
#pragma once
// NOTE: no __restrict__ in this header.  These bodies communicate between threads through `scratch` / `res` across __syncthreads() and, in the
// fused form, read depth / var / rgb that OTHER CTAs of the same launch have just written.  With noalias pointers the compiler may treat a
// barrier as not touching that memory: it forwarded `sel[]` across the barrier of the radix select (loading it BEFORE the writer's store in the
// other threads) -- found with n > 512 in the stand-alone kernel -- and it may route const noalias loads through the non-coherent path.
#include <cstdio>
#include "nsb_common.cuh"

namespace nsb {

// ------------------------------------------------------------------------------------------------ in-kernel exchanges over peer memory
// A ray-sharded tracking iteration needs three tiny batch-global quantities (SURVEY.md 8e).  Instead of three NCCL launches the
// single-CTA kernels that produce them exchange them themselves through NVLink peer memory (symmetric buffers, one per rank, mapped
// on every rank): push the local value into slot [parity][my rank] of EVERY peer's buffer, each 8-byte word carrying the exchange's
// sequence number next to 4 bytes of payload ("LL" words, below), and poll the own buffer until every rank's words show that number.
// Parity double-buffering + one sequence counter per channel make the buffers reusable without any reset; a rank cannot run two
// exchanges of a channel ahead because the other channels of the same iteration need everybody.
constexpr long long kPeerWaitCycles = 20000000000ll;        // ~10 s at 1.9 GHz
// buffer: [depth maxima: 2 x 8 x one LL word (16-byte stride) | sums: 2 x 8 x 16 LL pairs | residual pool: 2 x 8 x max_n LL pairs | this rank's plain copy of
// the gathered pool: 8 x max_n f64]
constexpr size_t kXMaxOff = 0, kXSumOff = 256, kXSumStride = 256, kXPoolOff = kXSumOff + 2 * NSB_MAX_PEERS * kXSumStride;
__host__ __device__ inline size_t peer_pool_plain_off(int max_n) { return kXPoolOff + (size_t)2 * NSB_MAX_PEERS * (size_t)max_n * 16; }
__host__ __device__ inline size_t peer_buffer_bytes(int max_n) { return peer_pool_plain_off(max_n) + (size_t)NSB_MAX_PEERS * (size_t)max_n * sizeof(double); }
// "LL" pairs (the low-latency protocol of the collective libraries): a double travels as two 8-byte words {32 bits of payload | the exchange's 32-bit
// sequence number}, written with ONE 16-byte store.  An aligned 8-byte word is single-copy atomic, so data and "it has arrived" are the same
// word: no system-scope fence on the sender (a membar.sys costs microseconds on a path that is all latency), no separate flag, and the receiver
// polls exactly the words it consumes.  Used by the two exchanges of a ray-sharded tracking iteration (residual pool, [loss | d c2w] sum).
__device__ __forceinline__ void ll_put(unsigned char* slot16, double v, uint32_t seq) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(v);
  const unsigned long long w0 = ((unsigned long long)seq << 32) | (b & 0xffffffffull), w1 = ((unsigned long long)seq << 32) | (b >> 32);
  asm volatile("st.relaxed.sys.global.v2.u64 [%0], {%1, %2};" ::"l"(slot16), "l"(w0), "l"(w1) : "memory");
}
__device__ __forceinline__ double ll_get(const unsigned char* slot16, uint32_t seq) {
  unsigned long long w0, w1;
  const long long t0 = clock64();
  for (;;) {
    asm volatile("ld.relaxed.sys.global.v2.u64 {%0, %1}, [%2];" : "=l"(w0), "=l"(w1) : "l"(slot16) : "memory");
    if ((uint32_t)(w0 >> 32) == seq && (uint32_t)(w1 >> 32) == seq) break;
    // a rank that never arrives (crashed process, mismatched call sequence) must not hang the device: fail the launch instead (no printf:
    // these waits run inside wgmma kernels, see nsb_tile.cuh mbar_wait_b)
    if (clock64() - t0 > kPeerWaitCycles) __trap();
  }
  return __longlong_as_double((long long)((w1 << 32) | (w0 & 0xffffffffull)));
}
// one float as a single LL word
__device__ __forceinline__ void ll_put_f32(unsigned char* slot8, float v, uint32_t seq) {
  const unsigned long long w = ((unsigned long long)seq << 32) | (unsigned long long)__float_as_uint(v);
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(slot8), "l"(w) : "memory");
}
__device__ __forceinline__ float ll_get_f32(const unsigned char* slot8, uint32_t seq) {
  unsigned long long w;
  const long long t0 = clock64();
  for (;;) {
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(w) : "l"(slot8) : "memory");
    if ((uint32_t)(w >> 32) == seq) break;
    if (clock64() - t0 > kPeerWaitCycles) __trap();
  }
  return __uint_as_float((uint32_t)w);
}
// close an LL exchange: every thread has consumed its words -> remember the sequence number
__device__ __forceinline__ void peer_end(const PeerX& px, int c, uint32_t seq) {
  __syncthreads();
  if (threadIdx.x == 0) px.counter[c] = (unsigned long long)seq;
}
// sequence number of this launch on channel c (CTA-uniform)
__device__ __forceinline__ uint32_t peer_begin(const PeerX& px, int c, uint32_t* s_seq) {
  if (threadIdx.x == 0) *s_seq = (uint32_t)(px.counter[c] + 1ull);
  __syncthreads();
  return *s_seq;
}

// ---- exchanges fused into multi-CTA kernels (tile kernels, nsb_tile.cuh) ----------------------------------------------------------------
// MAX over ranks of one float, needed by EVERY CTA of the grid before it can sample (channel 0): CTA 0 pushes this rank's value to every
// peer and raises the flags; all CTAs spin on this rank's own buffer.  The sequence number is read, not advanced: the grid's last CTA
// advances the channel with peer_advance() once every CTA has passed this point.
__device__ __forceinline__ float peer_max_all_ctas(const PeerX& px, float local, uint32_t* s_seq) {
  if (threadIdx.x == 0) *s_seq = (uint32_t)(px.counter[0] + 1ull);
  __syncthreads();
  const uint32_t seq = *s_seq;
  const int par = seq & 1u;
  __syncthreads();                                           // (*s_seq is reused for the result below)
  if (blockIdx.x == 0 && (int)threadIdx.x < px.world)
    ll_put_f32(px.peer[threadIdx.x] + kXMaxOff + ((size_t)par * NSB_MAX_PEERS + px.rank) * 16, local, seq);
  float m = -INFINITY;
  if (threadIdx.x < 32) {                                    // warp 0: lane r polls rank r's word, then the maximum over the lanes
    if ((int)threadIdx.x < px.world) m = ll_get_f32(px.peer[px.rank] + kXMaxOff + ((size_t)par * NSB_MAX_PEERS + threadIdx.x) * 16, seq);
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (threadIdx.x == 0) *reinterpret_cast<float*>(s_seq) = m;
  }
  __syncthreads();
  m = *reinterpret_cast<const float*>(s_seq);
  __syncthreads();
  return m;
}
__device__ __forceinline__ void peer_advance(const PeerX& px, int c) {      // one thread of the grid's last CTA
  px.counter[c] = px.counter[c] + 1ull;
}
// SUM over ranks of `n_val` (<= 13) doubles held in shared memory `tot` (channel 2), rank order -> identical bits on every rank.  Single CTA.
__device__ __forceinline__ void peer_sum13(const PeerX& px, const double* tot, int n_val, double* out, uint32_t* s_seq) {
  const uint32_t seq = peer_begin(px, 2, s_seq);
  const int par = seq & 1u;
  for (int i = threadIdx.x; i < n_val * px.world; i += blockDim.x) {
    const int r = i / n_val, k = i - n_val * r;
    ll_put(px.peer[r] + kXSumOff + ((size_t)par * NSB_MAX_PEERS + px.rank) * kXSumStride + (size_t)k * 16, tot[k], seq);
  }
  if ((int)threadIdx.x < n_val) {
    double v = 0.0;
    for (int r = 0; r < px.world; r++) v += ll_get(px.peer[px.rank] + kXSumOff + ((size_t)par * NSB_MAX_PEERS + r) * kXSumStride + (size_t)threadIdx.x * 16, seq);
    out[threadIdx.x] = v;
  }
  peer_end(px, 2, seq);
}

constexpr int kMedianDirect = 512;       // larger pools: 8-pass radix select (the direct count is O(n^2))
constexpr int kSeedsScratchBytes = 34 * 8 + kMedianDirect * 8 + (256 + 8 + 2 + 2) * 4;

// ------------------------------------------------------------------------------------------------ loss seeds
__device__ __forceinline__ double block_sum(double v, double* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  if (threadIdx.x < 32) {
    t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.0;
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  }
  __syncthreads();
  return t;   // valid in thread 0
}
// This thread's share of d c2w = [sum_r d_rays_d[r] (x) dirs[r] | sum_r d_rays_o[r]] over rows lo + threadIdx.x, step blockDim.x, below hi:
// acc[4 i + j] (j < 3) and acc[4 i + 3].  The ray gradients are read through L2 (__ldcg): in the fused form other CTAs of the launch wrote them.
__device__ __forceinline__ void pose_grad_partial(const float* dirs, const float* d_rays_o, const float* d_rays_d, int lo, int hi, double acc[12]) {
#pragma unroll
  for (int k = 0; k < 12; k++) acc[k] = 0.0;
  for (int r = lo + threadIdx.x; r < hi; r += blockDim.x) {
#pragma unroll
    for (int i = 0; i < 3; i++) {
      const double g = (double)__ldcg(d_rays_d + 3 * r + i);
#pragma unroll
      for (int j = 0; j < 3; j++) acc[4 * i + j] += g * (double)__ldg(dirs + 3 * r + j);
      acc[4 * i + 3] += (double)__ldcg(d_rays_o + 3 * r + i);
    }
  }
}
__device__ __forceinline__ double sgn(double x) { return (x > 0.0) - (x < 0.0); }

// Tracker.optimize_cam_in_batch loss (src/Tracker.py:108-123); single CTA, residuals staged in `res`.
__device__ __forceinline__ void tracking_seeds_body(const double* depth, const double* var, const float* rgb,
                                      const float* gt, const double* gt_rgb, int n, double w_color,
                                      int handle_dynamic, int use_color, const double* pool, int n_pool,
                                      double* g_depth, float* g_rgb,
                                      double* loss, double* res, const PeerX& px, unsigned char* scratch) {
  // scratch (kSeedsScratchBytes, 16-byte aligned shared memory): red[32] f64 | med_s f64 | med_key u64 | keys[kMedianDirect] u64 | hist[256] | wtot[8] | sel[2] | seq
  double* red = reinterpret_cast<double*>(scratch);
  double& med_s = red[32];
  unsigned long long& med_key = *reinterpret_cast<unsigned long long*>(red + 33);
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(red + 34);
  int* hist = reinterpret_cast<int*>(keys + kMedianDirect);
  int* wtot = hist + 256;
  int* sel = wtot + 8;
  uint32_t* s_seq_p = reinterpret_cast<uint32_t*>(sel + 2);
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    res[i] = fabs((double)gt[i] - depth[i]) / sqrt(var[i] + 1e-10);
  __syncthreads();
  if (handle_dynamic) {
    // torch.median = lower median = the element of rank (n-1)/2 of the IEEE bit patterns (residuals are non-negative, so the unsigned
    // 64-bit pattern is order preserving).  torch.median of a pool that holds a NaN IS NaN -- the mask r < 10 * NaN then keeps no ray and
    // the loss is 0 --, so the loops that read the pool also look for one and the selected key is replaced by NaN at the end.
    const double* mp = pool != nullptr ? pool : res;       // sharded batches: median over the all-gathered residuals
    int np = pool != nullptr ? n_pool : n;
    int pool_pitch = 0;                                    // > 0: the pool is [world][pool_pitch] with n valid entries per rank
    if (px.world > 1) {
      // all-gather of the residuals through peer memory (channel 1): push this shard into block [parity][rank] of every peer's pool
      const uint32_t seq = peer_begin(px, 1, s_seq_p);
      const int par = seq & 1u;
      for (int i = threadIdx.x; i < n * px.world; i += blockDim.x) {
        const int r = i / n, j = i - r * n;
        ll_put(px.peer[r] + kXPoolOff + (((size_t)par * NSB_MAX_PEERS + px.rank) * px.max_n + j) * 16, res[j], seq);
      }
      // receive: each thread polls the words it owns and leaves the value in this rank's plain copy of the pool
      double* plain = reinterpret_cast<double*>(px.peer[px.rank] + peer_pool_plain_off(px.max_n));
      for (int i = threadIdx.x; i < n * px.world; i += blockDim.x) {
        const int r = i / n, j = i - r * n;
        plain[(size_t)r * px.max_n + j] = ll_get(px.peer[px.rank] + kXPoolOff + (((size_t)par * NSB_MAX_PEERS + r) * px.max_n + j) * 16, seq);
      }
      peer_end(px, 1, seq);                                  // (its barrier also makes `plain` visible to the whole CTA)
      mp = plain;
      np = n * px.world; pool_pitch = px.max_n;
    }
    auto pool_at = [&](int i) { return pool_pitch ? mp[(size_t)(i / n) * pool_pitch + (i % n)] : mp[i]; };
    const int k = (np - 1) / 2;
    int saw_nan = 0, pool_nan = 0;                         // this thread met a NaN in the pool / some thread did (CTA-uniform)
    // the key of rank `want` among keys[0 .. cnt), cnt <= kMedianDirect: direct rank counting from shared memory (no serial passes) or a sort
    auto select_direct = [&](int cnt, int want) {
      if (cnt > 256) {
        // more than one key per thread: bitonic sort in shared memory (45 compare-exchange stages for 512 keys) beats cnt^2 / 256 comparisons.
        // Padding with ~0 sorts behind every key, so the key of rank `want` is simply keys[want].
        int m = 512;                                             // == kMedianDirect (capacity of keys[])
        for (int i = cnt + threadIdx.x; i < m; i += blockDim.x) keys[i] = ~0ull;
        __syncthreads();
        for (int k2 = 2; k2 <= m; k2 <<= 1)
          for (int j = k2 >> 1; j > 0; j >>= 1) {
            for (int t = threadIdx.x; t < m / 2; t += blockDim.x) {
              const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
              const unsigned long long x = keys[i], y = keys[i | j];
              if ((x > y) == ((i & k2) == 0)) { keys[i] = y; keys[i | j] = x; }
            }
            __syncthreads();
          }
        if (threadIdx.x == 0) med_key = keys[want];
        __syncthreads();
        return;
      }
      for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
        const unsigned long long key = keys[i];
        int less = 0, eq = 0;
        for (int j = 0; j < cnt; j++) { const unsigned long long o = keys[j]; less += o < key ? 1 : 0; eq += o == key ? 1 : 0; }
        if (less <= want && want < less + eq) med_key = key;     // every thread that qualifies writes the same value
      }
      __syncthreads();
    };
    if (np <= kMedianDirect) {
      // small pools (a tracking batch is 200 rays)
      for (int i = threadIdx.x; i < np; i += blockDim.x) {
        const double v = pool_at(i);
        saw_nan |= v != v;
        keys[i] = (unsigned long long)__double_as_longlong(v);
      }
      pool_nan = __syncthreads_or(saw_nan);
      select_direct(np, k);
    } else {
      // radix select, 8 bits per pass over a 256-bin shared histogram -- until the bin that holds the wanted rank is small enough for the direct
      // count (residuals spread over many exponents: normally after the second pass), at most 8 passes
      unsigned long long prefix = 0ull;
      int kk = k;
      bool direct = false;
      for (int shift = 56; shift >= 0; shift -= 8) {
        for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
        __syncthreads();
        const unsigned long long maskhi = shift == 56 ? 0ull : (~0ull << (shift + 8));
        for (int i = threadIdx.x; i < np; i += blockDim.x) {
          const double v = pool_at(i);
          saw_nan |= v != v;
          const unsigned long long key = (unsigned long long)__double_as_longlong(v);
          if ((key & maskhi) == prefix) atomicAdd(&hist[(int)((key >> shift) & 0xffull)], 1);
        }
        pool_nan = __syncthreads_or(saw_nan);              // (every pass reads the whole pool)
        // digit of the k-th key = the bin whose [exclusive, inclusive) prefix-count range contains kk (256 bins: 8 warps scan them)
        {
          const int v = threadIdx.x < 256 ? hist[threadIdx.x] : 0;
          int incl = v;
          for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if ((threadIdx.x & 31) >= o) incl += t; }
          if (threadIdx.x < 256 && (threadIdx.x & 31) == 31) wtot[threadIdx.x >> 5] = incl;
          __syncthreads();
          int before = 0;
          for (int w = 0; w < (int)(threadIdx.x >> 5) && w < 8; w++) before += wtot[w];
          incl += before;
          if (threadIdx.x < 256 && incl - v <= kk && kk < incl) { sel[0] = (int)threadIdx.x; sel[1] = incl - v; }
          __syncthreads();
        }
        prefix |= (unsigned long long)sel[0] << shift;
        kk -= sel[1];
        const int cnt = hist[sel[0]];                        // keys that share the prefix (CTA-uniform)
        __syncthreads();
        if (shift > 0 && cnt <= kMedianDirect) {
          if (threadIdx.x == 0) sel[0] = 0;
          __syncthreads();
          const unsigned long long maskall = ~0ull << shift;
          for (int i = threadIdx.x; i < np; i += blockDim.x) {
            const unsigned long long key = (unsigned long long)__double_as_longlong(pool_at(i));
            if ((key & maskall) == prefix) keys[atomicAdd(&sel[0], 1)] = key;
          }
          __syncthreads();
          select_direct(cnt, kk);
          direct = true;
          break;
        }
      }
      if (!direct) {
        if (threadIdx.x == 0) med_key = prefix;
        __syncthreads();
      }
    }
    if (threadIdx.x == 0) med_s = pool_nan ? __longlong_as_double(0x7ff8000000000000ll) : __longlong_as_double((long long)med_key);
    __syncthreads();
  }
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const double r = res[i];
    bool m = gt[i] > 0.0f;
    if (handle_dynamic) m = m && (r < 10.0 * med_s);
    double gd = 0.0; float gc[3] = {0.f, 0.f, 0.f};
    if (m) {
      acc += r;
      gd = -sgn((double)gt[i] - depth[i]) / sqrt(var[i] + 1e-10);
      if (use_color) {
#pragma unroll
        for (int a = 0; a < 3; a++) { const double df = gt_rgb[3 * i + a] - (double)rgb[3 * i + a]; acc += w_color * fabs(df); gc[a] = (float)(-w_color * sgn(df)); }
      }
    }
    g_depth[i] = gd; g_rgb[3 * i] = gc[0]; g_rgb[3 * i + 1] = gc[1]; g_rgb[3 * i + 2] = gc[2];
  }
  const double tot = block_sum(acc, red);
  if (threadIdx.x == 0) loss[0] = tot;
}

// Mapper.optimize_map loss (src/Mapper.py:487-493); single CTA (deterministic sum)
__device__ __forceinline__ void mapping_seeds_body(const double* depth, const float* rgb, const float* gt,
                                     const float* gt_rgb, int n, double w_color, int use_color,
                                     double* g_depth, float* g_rgb, double* loss,
                                     unsigned char* scratch) {
  double* red = reinterpret_cast<double*>(scratch);
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    double gd = 0.0;
    if (gt[i] > 0.0f) { const double df = (double)gt[i] - depth[i]; acc += fabs(df); gd = -sgn(df); }
    g_depth[i] = gd;
#pragma unroll
    for (int a = 0; a < 3; a++) {
      float g = 0.0f;
      if (use_color) { const float df = gt_rgb[3 * i + a] - rgb[3 * i + a]; acc += w_color * (double)fabsf(df); g = (float)(-w_color * sgn((double)df)); }
      g_rgb[3 * i + a] = g;
    }
  }
  const double tot = block_sum(acc, red);
  if (threadIdx.x == 0) loss[0] = tot;
}


// Grid-wide "last CTA" election: every participating CTA calls it once after its global writes; returns true in exactly one CTA (all of
// its threads), after every other participant's writes are visible.  counter: zero between launches (the winner resets it).
__device__ __forceinline__ bool grid_last_arrival(int* counter, int n_participants, int* s_flag) {
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const int old = atomicAdd(counter, 1);
    *s_flag = old == n_participants - 1;
    if (*s_flag) *counter = 0;
  }
  __syncthreads();
  const bool last = *s_flag != 0;
  if (last) __threadfence();
  return last;
}

}  // namespace nsb
