// nsb_tile.cuh -- tile-centric tensor-core kernels (round 2): two co-resident CTAs per SM.
//
// Work item = (128-point TILE of the batch's global (ray, sample) order, decoder).  A tile is independent of ray boundaries, so every
// tile is full (no padding rows for S = 48), small batches spread over all SMs (200 rays x 48 x 3 decoders = 225 items, all resident
// at once at two CTAs per SM) and the shared-memory footprint no longer grows with the number of samples per ray.  What needs whole
// rays -- compositing in the forward, the ray-gradient sums in the backward -- is done by the CTA that COMPLETES a ray: every item
// bumps the counters of the rays it touches after publishing its per-point results, the CTA that brings a counter to its target value
// composites / reduces that ray from global (L2) scratch in a fixed order (bit-reproducible), and resets the counter.
//
// CTA = 256 threads = two warpgroups; warpgroup g issues and waits for the MMAs of tile rows [64 g, 64 g + 64) (wgmma).  In the forward
// and the backward the accumulators stay in registers and the epilogues work on the wgmma fragments ("register accumulators of the
// forward", "backward (input gradients)"); the point state (gather, embedding, scatter) is owned row-wise: thread tid owns row tid & 127
// and the 16-column half tid >> 7.  Thread 0 is also the TMA producer:
//   * weights stream through a 4-slot ring of operand UNITS (pre-split hi|lo canonical tiles, consumption order, nsb_common.cuh) with full
//     (TMA -> MMA) and empty (MMA done -> producer, one arrival per warpgroup) mbarriers: three units of prefetch, no thread touches a weight;
//   * tiles that both warpgroups write (forward: gather, embedding) ping-pong between two 32 KB operand buffers; warps publish them by
//     fence.proxy.async + one mbarrier.arrive per warp (A_ready), and each warpgroup signals the buffer's `done` barrier when its MMAs on it
//     have completed.  Tiles a warpgroup writes from its own fragments (H, G, DU) are published by a barrier of its 128 threads.
// Shared memory: 64 KB activations + 40 KB ring + 6 KB headers + < 6 KB state <= 113 KB -> two CTAs per SM.
//
// Arithmetic is that of nsb_tc.cuh (3xTF32 split, same operand order), so results match the round-1 kernels to rounding of the output
// layer's partial sums.  Sampling and the sort, compositing and its backward, the trilinear scatter, the ray-gradient store and the
// loss-seed / pose tails are the functions every kernel family calls from nsb_render.cu; this file keeps only the tile's mapping of
// threads and scratch around them.
#pragma once

namespace nsb {
namespace tl {

using tc::TM;
constexpr int kThreads = 256;                 // 8 warps = two warpgroups
constexpr int kEpiThreads = kThreads;
constexpr int kCG = 2, kCW = 16, kKQ = 4;      // column halves per row, columns per thread, 16-byte chunks per thread
constexpr int kSlots = 4;
constexpr int kSlotFloatsFwd = 2560;          // 10 KB: the largest forward unit (fc_c: [160 x 8] hi|lo)
constexpr int kSlotFloatsBwd = 2048;          //  8 KB: every backward unit is [32 x 32] hi|lo
constexpr int kABufFloats = 2 * TM * 32;      // one [128 x 32] operand tile, hi|lo = 32 KB
constexpr int kMaxTileRays = 18;              // rays one tile can touch (S >= 8)
constexpr int kMinSamples = 8;
constexpr long long kWaitCycles = 4000000000ll;      // ~2 s: a wait that long is a protocol bug -> trap instead of hanging the GPU

// barrier indices
enum { B_FULL = 0, B_EMPTY = 4, B_HDR = 8, B_AREADY = 10, B_DONE = 12, kNumBars = 14 };

__device__ __forceinline__ bool mbar_try(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}"
               : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
// non-blocking poll (try_wait may suspend the thread for a hardware-defined time before it answers "not yet")
__device__ __forceinline__ bool mbar_test(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}"
               : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
// bounded wait: a protocol error traps (the launch fails with an error) instead of hanging the device.  No printf here or anywhere else in
// a wgmma kernel: a call to it makes ptxas serialize every wgmma of the kernel (C7510).
__device__ __forceinline__ void mbar_wait_b(uint64_t* bar, uint32_t parity) {
  if (mbar_try(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try(bar, parity)) {
    if (clock64() - t0 > kWaitCycles) __trap();
  }
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void epi_sync() { __syncthreads(); }

// ---- shared memory -------------------------------------------------------------------------------------------------------------
struct TileSmem {
  float* a[2];        // operand buffers
  float* ring;        // kSlots x slot_floats
  int slot_floats;
  float* hdr;         // 2 x kHdrFloats
  uint64_t* bars;
  uint32_t* tmem;
  unsigned char* extra;      // kernel-specific state behind the common part
};
__host__ __device__ constexpr size_t common_bytes(bool bwd) {     // + barriers (14 x 8) + accumulator slot index
  return (2 * (size_t)kABufFloats + (size_t)kSlots * (bwd ? kSlotFloatsBwd : kSlotFloatsFwd) + 2 * kHdrFloats) * 4 + 128;
}
__device__ __forceinline__ void carve(unsigned char* base, TileSmem& t, bool bwd) {
  float* f = reinterpret_cast<float*>(base);
  t.a[0] = f; f += kABufFloats; t.a[1] = f; f += kABufFloats;
  t.slot_floats = bwd ? kSlotFloatsBwd : kSlotFloatsFwd;
  t.ring = f; f += kSlots * t.slot_floats;
  t.hdr = f; f += 2 * kHdrFloats;
  t.bars = reinterpret_cast<uint64_t*>(f);
  t.tmem = reinterpret_cast<uint32_t*>(f + 2 * kNumBars);
  t.extra = base + common_bytes(bwd);
}

// ---- unit sequences of the v2 operand images (nsb_common.cuh: op2_*) ---------------------------------------------------------------
__device__ __forceinline__ int fwd_units(int lv) { return op2_fwd_units(lv); }
__device__ __forceinline__ int bwd_units(int lv) { return op2_bwd_units(lv); }

// Producer cursor: walks the units of the decoders this CTA evaluates, in consumption order.
struct Loader {
  const KParams* P;
  int q, q1;          // current / end decoder slot
  int k;              // unit index inside decoder q
  uint32_t loaded;    // units issued so far (global sequence number of the next one)
  int mode;           // 0 = forward (3xTF32 units), 1 = backward, 2 = forward with FP16 hi|lo units (op3_*)
};
__device__ __forceinline__ bool loader_done(const Loader& L) { return L.q >= L.q1; }
__device__ __forceinline__ void loader_issue(Loader& L, const TileSmem& t) {
  const int lv = L.P->dec[L.q];
  const float* img = L.P->in.packed[lv] + (L.mode == 1 ? op2_bwd_offset(lv) : L.mode == 2 ? op3_fwd_offset(lv) : op2_fwd_offset(lv));
  int off, floats, n_units;
  if (L.mode == 1) { off = L.k * 2048; floats = 2048; n_units = bwd_units(lv); }
  else if (L.mode == 2) {
    const int nfc = op3_fc_units(lv), nl0 = op_nblk(lv);
    if (L.k < nfc) { off = L.k * 2560; floats = 2560; }
    else if (L.k < nfc + nl0) { off = nfc * 2560 + (L.k - nfc) * 2048; floats = 2048; }
    else { off = nfc * 2560 + nl0 * 2048 + (L.k - nfc - nl0) * 1024; floats = 1024; }
    n_units = op3_fwd_units(lv);
  } else {
    const int nfc = op2_fc_units(lv);
    if (L.k < nfc) { off = L.k * 2560; floats = 2560; } else { off = nfc * 2560 + (L.k - nfc) * 2048; floats = 2048; }
    n_units = fwd_units(lv);
  }
  const int slot = L.loaded & (kSlots - 1);
  uint64_t* bar = t.bars + B_FULL + slot;
  mbar_expect_tx(bar, (uint32_t)floats * 4u);
  tma_bulk_g2s(t.ring + slot * t.slot_floats, img + off, (uint32_t)floats * 4u, bar);
  L.loaded++;
  if (++L.k == n_units) { L.k = 0; L.q++; }
}
// refill one slot if a unit is pending and its slot's previous occupant has been issued (blocking on that unit's MMAs)
__device__ __forceinline__ bool loader_refill(Loader& L, const TileSmem& t, uint32_t issued) {
  if (loader_done(L) || L.loaded >= issued + kSlots) return false;
  if (L.loaded >= kSlots) { const uint32_t prev = L.loaded - kSlots; mbar_wait_b(t.bars + B_EMPTY + (prev & (kSlots - 1)), (prev >> 2) & 1u); }
  loader_issue(L, t);
  return true;
}
// request every unit whose slot is already free (non-blocking)
__device__ __forceinline__ void loader_top_up(Loader& L, const TileSmem& t, uint32_t issued) {
  while (!loader_done(L) && L.loaded < issued + kSlots) {
    if (L.loaded >= kSlots) { const uint32_t prev = L.loaded - kSlots; if (!mbar_test(t.bars + B_EMPTY + (prev & (kSlots - 1)), (prev >> 2) & 1u)) return; }
    loader_issue(L, t);
  }
}
__device__ __forceinline__ void load_header(const KParams& P, const TileSmem& t, int lv, int hb) {
  uint64_t* bar = t.bars + B_HDR + hb;
  mbar_expect_tx(bar, kHdrFloats * 4u);
  tma_bulk_g2s(t.hdr + hb * kHdrFloats, P.in.packed[lv] + op_fwd_offset(lv), kHdrFloats * 4u, bar);
}

// Issuer state (control thread)
struct Issuer {
  Loader L;
  uint32_t issued;    // units consumed so far
  uint32_t g;         // operand groups consumed so far (forward: buffer = g & 1)
};
// The issue path is executed by EVERY thread of the CTA (wgmma is a warpgroup instruction; the two warpgroups compute rows [0, 64) and
// [64, 128)): the counters `issued` / `g` advance identically in every thread.  Only the TMA producer bookkeeping (Loader) is thread 0's private state.
// wait for the operands of group `g` on A_ready[b]; while they are not there, thread 0 keeps the ring full
__device__ __forceinline__ void issuer_wait_operands(Issuer& I, const TileSmem& t, int b, uint32_t parity) {
  uint64_t* bar = t.bars + B_AREADY + b;
  const long long t0 = clock64();
  while (!mbar_test(bar, parity)) {                              // poll: the ring is topped up between polls
    if (threadIdx.x == 0) loader_top_up(I.L, t, I.issued);
    if (clock64() - t0 > kWaitCycles) __trap();
  }
}
// unit I.issued + k (k < kSlots) of the consumption order: make sure it was requested (thread 0), wait for it (all threads), return its slot base
__device__ __forceinline__ const float* issuer_unit(Issuer& I, const TileSmem& t, uint32_t k = 0) {
  if (threadIdx.x == 0) {
    loader_top_up(I.L, t, I.issued);
    while (I.L.loaded <= I.issued + k) loader_refill(I.L, t, I.issued);
  }
  const uint32_t u = I.issued + k;
  const int slot = u & (kSlots - 1);
  mbar_wait_b(t.bars + B_FULL + slot, (u >> 2) & 1u);
  return t.ring + slot * t.slot_floats;
}
// slot base of unit I.issued + k (already waited for)
__device__ __forceinline__ const float* issued_unit(const Issuer& I, const TileSmem& t, uint32_t k) { return t.ring + ((I.issued + k) & (kSlots - 1)) * t.slot_floats; }

// ---- FP16 hi|lo forward (option fwd_f16) ------------------------------------------------------------------------------------------------------
// x = hi + lo with hi = fp16(x), lo = fp16(x - hi): 22 significant bits for |x| in [2^-3, 65504], an absolute error <= 2^-25 below (lo goes
// subnormal) -- the forward's operands (features, sin embedding, ReLU outputs, weights) are O(1) values, far inside the 1e-4 tolerance of the
// path.  wgmma f16 contracts K = 16 per instruction: half the MMAs and half the shared-memory operand traffic of the 3xTF32 forward (which is
// what bounds the MMA phases: every N <= 64 MMA re-reads its [128 x K] A slice).  Conversions saturate (cvt.rn.satfinite): an operand beyond
// the fp16 range degrades instead of producing Inf/NaN.  The backward keeps 3xTF32 (gradients span far more than fp16's exponent range).
// 16-bit canonical K-major tile of width K halves: [row/8][k/8][row%8][k%8]; hi tile, then lo tile.
__device__ __forceinline__ uint32_t cvt_h2(float lo_elem, float hi_elem) {          // {fp16(lo_elem), fp16(hi_elem)} packed, saturating
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi_elem), "f"(lo_elem));
  return r;
}
__device__ __forceinline__ void split_h2(float x, float y, uint32_t& h, uint32_t& l) {
  h = cvt_h2(x, y);
  const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&h));
  l = cvt_h2(x - f.x, y - f.y);
}
// four consecutive features (4-wide chunk kq of a 32-wide tile) of row r: 8 bytes in the hi tile, 8 in the lo tile
__device__ __forceinline__ void put4_h(float* tile, int r, int kq, const float4 v) {
  unsigned char* hi = reinterpret_cast<unsigned char*>(tile) + (((r >> 3) * 4 + (kq >> 1)) * 128 + (r & 7) * 16 + (kq & 1) * 8);
  uint2 h, l;
  split_h2(v.x, v.y, h.x, l.x); split_h2(v.z, v.w, h.y, l.y);
  *reinterpret_cast<uint2*>(hi) = h;
  *reinterpret_cast<uint2*>(hi + TM * 32 * 2) = l;
}
// this thread's 16 features (column group cg) of row r: two 16-byte chunks per tile
__device__ __forceinline__ void put16_h(float* tile, int r, int cg, const float (&v)[kCW]) {
#pragma unroll
  for (int c = 0; c < 2; c++) {
    unsigned char* hi = reinterpret_cast<unsigned char*>(tile) + (((r >> 3) * 4 + 2 * cg + c) * 128 + (r & 7) * 16);
    uint4 h, l;
    split_h2(v[8 * c], v[8 * c + 1], h.x, l.x); split_h2(v[8 * c + 2], v[8 * c + 3], h.y, l.y);
    split_h2(v[8 * c + 4], v[8 * c + 5], h.z, l.z); split_h2(v[8 * c + 6], v[8 * c + 7], h.w, l.w);
    *reinterpret_cast<uint4*>(hi) = h;
    *reinterpret_cast<uint4*>(hi + TM * 32 * 2) = l;
  }
}
// ---- register accumulators of the forward ------------------------------------------------------------------------------------------
// Warpgroup g issues the MMAs of its own rows [64 g, 64 g + 64) and waits for them itself, so an accumulator stays in the registers of the
// threads that hold its wgmma m64n32 fragment (tc::frag_rc) from the first MMA to the epilogue.  A warpgroup only ever reads its own rows of
// an A tile: tiles that the warpgroup writes from its fragments (H) need a barrier of its 128 threads only.
// d += A[rows of this warpgroup, ka0 .. ka0 + ksteps k-steps) * B[32 c .. 32 c + 32, first ksteps k-steps]^T with the split-operand scheme (lo*hi + hi*lo + hi*hi),
// tf32 (k-step 8) or fp16 (k-step 16, offsets in halves).  A: [128 x 32] hi|lo tile; B: unit [N x KB] hi|lo.  Issues only: the caller fences,
// commits and waits.
// MMA groups are kept in a form ptxas can pipeline (otherwise it waits for every wgmma before issuing the next, C7517-C7520): between
// wgmma.fence and commit_group a straight run of wgmma with compile-time unit and k-step counts, reached by every thread of the warpgroup;
// accumulators initialised just before the fence (a constant zero kept in the open, as in the coarse layer 0, is materialised by ptxas
// inside the group, hence zero16_opaque); producer work and mbarrier waits before them; every group waited for on every path that leads
// to a read of its accumulators.  A group may stay in flight across other code (the layer-0 chain) if that code has no branch or predicated
// instruction ptxas may take as divergent (C7518) and every wait follows a whole group in the code.
struct RowsDesc { uint64_t ah, al, bh, bl; };      // hi / lo descriptors of this warpgroup's A rows and of B from row 32 c
template <bool H16>
__device__ __forceinline__ RowsDesc rows_desc(const float* a, int ka0, const float* b, int N, int KB, int c) {
  const uint32_t g = (threadIdx.x >> 7) & 1u;
  const int esz = H16 ? 2 : 4, kcm = H16 ? 8 : 4;               // bytes per element, elements per 16-byte core-matrix row
  const uint32_t sbo_a = (32u / kcm) * 128u, sbo_b = (uint32_t)(KB / kcm) * 128u;
  RowsDesc r;
  r.ah = tc::make_desc(a + (ka0 / kcm) * 32, 128u, sbo_a) + (uint64_t)((8u * sbo_a * g) >> 4);
  r.bh = tc::make_desc(b, 128u, sbo_b) + (uint64_t)((4u * sbo_b * (uint32_t)c) >> 4);
  r.al = r.ah + (uint64_t)((TM * 32 * esz) >> 4); r.bl = r.bh + (uint64_t)((N * KB * esz) >> 4);
  return r;
}
template <bool H16, int ksteps>
__device__ __forceinline__ void mma_rows(float (&d)[16], const float* a, int ka0, const float* b, int N, int KB, int c) {
  const RowsDesc r = rows_desc<H16>(a, ka0, b, N, KB, c);
#pragma unroll
  for (int ks = 0; ks < ksteps; ks++) {
    const uint64_t o = 16u * (uint64_t)ks;
    if (H16) { tc::wgmma_f16_n32(d, r.al + o, r.bh + o); tc::wgmma_f16_n32(d, r.ah + o, r.bl + o); tc::wgmma_f16_n32(d, r.ah + o, r.bh + o); }
    else { tc::wgmma_tf32_n32(d, r.al + o, r.bh + o); tc::wgmma_tf32_n32(d, r.ah + o, r.bl + o); tc::wgmma_tf32_n32(d, r.ah + o, r.bh + o); }
  }
}
// the same for B rows [32 c, 32 c + 64) into [d0 | d1] with m64n64 instructions: every element sees the products of mma_rows on d0 (c) and
// d1 (c + 1) in the same order, with half the instructions and one read of the A slice instead of two
template <bool H16, int ksteps>
__device__ __forceinline__ void mma_rows64(float (&d0)[16], float (&d1)[16], const float* a, int ka0, const float* b, int N, int KB, int c) {
  const RowsDesc r = rows_desc<H16>(a, ka0, b, N, KB, c);
#pragma unroll
  for (int ks = 0; ks < ksteps; ks++) {
    const uint64_t o = 16u * (uint64_t)ks;
    if (H16) { tc::wgmma_f16_n64(d0, d1, r.al + o, r.bh + o); tc::wgmma_f16_n64(d0, d1, r.ah + o, r.bl + o); tc::wgmma_f16_n64(d0, d1, r.ah + o, r.bh + o); }
    else { tc::wgmma_tf32_n64(d0, d1, r.al + o, r.bh + o); tc::wgmma_tf32_n64(d0, d1, r.ah + o, r.bl + o); tc::wgmma_tf32_n64(d0, d1, r.ah + o, r.bh + o); }
  }
}
// this warpgroup's MMAs on units [first, first + count) of the consumption order have completed: one arrival per warpgroup on each unit's
// `empty` barrier (and on `done`)
__device__ __forceinline__ void arrive_units(const TileSmem& t, uint32_t first, uint32_t count, uint64_t* done = nullptr) {
  if ((threadIdx.x & 127) == 0) {
    for (uint32_t k = 0; k < count; k++) mbar_arrive(t.bars + B_EMPTY + ((first + k) & (kSlots - 1)));
    if (done != nullptr) mbar_arrive(done);
  }
}
// ... on the next `count` units
__device__ __forceinline__ void release_units(Issuer& I, const TileSmem& t, uint32_t count, uint64_t* done = nullptr) {
  arrive_units(t, I.issued, count, done);
  I.issued += count;
}
__device__ __forceinline__ void wg_bar_sync() {                 // named barrier of this warpgroup's 128 threads (ids 1, 2; 0 is __syncthreads)
  if (threadIdx.x >> 7) asm volatile("bar.sync 2, 128;" ::: "memory");
  else asm volatile("bar.sync 1, 128;" ::: "memory");
}
__device__ __forceinline__ void zero16(float (&d)[16]) {
#pragma unroll
  for (int e = 0; e < 16; e++) d[e] = 0.0f;
}
__device__ __forceinline__ void zero16_opaque(float (&d)[16]) {
#pragma unroll
  for (int e = 0; e < 16; e++) asm volatile("mov.b32 %0, 0;" : "=f"(d[e])::"memory");
}
// columns c, c + 1 (c even) of row r of a [128 x 32] tf32 operand tile (canonical K-major, hi | lo): one 8-byte store per tile
__device__ __forceinline__ void put2(float* hi, int r, int c, float a, float b) {
  float* hp = hi + tc::canon_q(r, c >> 2, 32) + (c & 3);
  const float h0 = tc::to_tf32(a), h1 = tc::to_tf32(b);
  *reinterpret_cast<float2*>(hp) = make_float2(h0, h1);
  *reinterpret_cast<float2*>(hp + TM * 32) = make_float2(a - h0, b - h1);
}

// ---- epilogue-side helpers -------------------------------------------------------------------------------------------------------
// operands of this thread are written: make them visible to the async proxy, arrive
__device__ __forceinline__ void publish(const TileSmem& t, int b) {
  fence_proxy_async();
  __syncwarp();                                                 // one arrival per warp (256 arrivals on one barrier word serialise)
  if ((threadIdx.x & 31) == 0) mbar_arrive(t.bars + B_AREADY + b);
}
__device__ __forceinline__ void wait_group(const TileSmem& t, uint32_t m) {      // MMAs of operand group m (and all earlier ones) have completed
  mbar_wait_b(t.bars + B_DONE + (m & 1u), (m >> 1) & 1u);
}

// 8 lanes per point, 4 points per pass: 32 channels of grid `g` -> [128 x 32] tile.  Warp w serves the rows of its lane quadrant (w & 3);
// the eight passes of a quadrant are split over the two warps that share it.  The loads of pass i+1 are issued before pass i is consumed
// (16 x 16-byte loads in flight per lane), corner offsets come from per-axis offsets (two adds per corner).
struct GatherPass {
  float4 v[8];
  float w[8];
  int src_lane;
};
template <bool FAST>
__device__ __forceinline__ void gather_issue(const nsb_grid& g, const float xn[3], int it, int lane, GatherPass& gp) {
  const int q = lane & 7;
  gp.src_lane = it * 4 + (lane >> 3);
  float x[3];
  x[0] = __shfl_sync(0xffffffffu, xn[0], gp.src_lane); x[1] = __shfl_sync(0xffffffffu, xn[1], gp.src_lane); x[2] = __shfl_sync(0xffffffffu, xn[2], gp.src_lane);
  const Tri t = make_tri(x, g.W, g.H, g.D);
  // branch-free clamped corners (tri_corner_clamped): the clamped upper corner carries weight exactly 0
  const long long ox[2] = {(long long)t.i0[0] * g.stride_w, (long long)min(t.i0[0] + 1, g.W - 1) * g.stride_w};
  const long long oy[2] = {(long long)t.i0[1] * g.stride_h, (long long)min(t.i0[1] + 1, g.H - 1) * g.stride_h};
  const long long oz[2] = {(long long)t.i0[2] * g.stride_d, (long long)min(t.i0[2] + 1, g.D - 1) * g.stride_d};
#pragma unroll
  for (int k = 0; k < 8; k++) gp.v[k] = grid_load4(g, oz[k >> 2] + oy[(k >> 1) & 1] + ox[k & 1], 4 * q, FAST);
  const float wxy[4] = {__fmul_rn(t.w0[0], t.w0[1]), __fmul_rn(t.w1[0], t.w0[1]), __fmul_rn(t.w0[0], t.w1[1]), __fmul_rn(t.w1[0], t.w1[1])};
#pragma unroll
  for (int k = 0; k < 8; k++) gp.w[k] = __fmul_rn(wxy[k & 3], (k & 4) ? t.w1[2] : t.w0[2]);      // == tri_weight(t, k)
}
template <bool H16 = false>
__device__ __forceinline__ void gather_consume(float* c_hi, float* c_lo, int qd, int lane, const GatherPass& gp) {
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const float w = gp.w[k];
    acc.x = fmaf(gp.v[k].x, w, acc.x); acc.y = fmaf(gp.v[k].y, w, acc.y); acc.z = fmaf(gp.v[k].z, w, acc.z); acc.w = fmaf(gp.v[k].w, w, acc.w);
  }
  if (H16) put4_h(c_hi, qd * 32 + gp.src_lane, lane & 7, acc);
  else tc::put4(c_hi, c_lo, qd * 32 + gp.src_lane, lane & 7, 32, acc);
}
// (the strided NCDHW form -- four scalar loads with 64-bit strides per corner -- is a separate, out-of-line copy: inlined next to the channels-last
// form at every unrolled corner it made up a third of the forward kernel's 19 k instructions, and instruction fetch shows up in the stall samples)
template <bool FAST, bool H16 = false>
__device__ __forceinline__ void gather_tile_t(const nsb_grid& g, float* c_hi, const float xn[3], int warp, int lane) {
  float* c_lo = c_hi + TM * 32;
  const int qd = warp & 3, it0 = (warp >> 2) * 4;
  if (FAST) {
    GatherPass A, B;
    gather_issue<true>(g, xn, it0, lane, A);
    gather_issue<true>(g, xn, it0 + 1, lane, B);
    gather_consume<H16>(c_hi, c_lo, qd, lane, A);
    gather_issue<true>(g, xn, it0 + 2, lane, A);
    gather_consume<H16>(c_hi, c_lo, qd, lane, B);
    gather_issue<true>(g, xn, it0 + 3, lane, B);
    gather_consume<H16>(c_hi, c_lo, qd, lane, A);
    gather_consume<H16>(c_hi, c_lo, qd, lane, B);
  } else {
#pragma unroll 1
    for (int it = it0; it < it0 + 4; it++) { GatherPass A; gather_issue<false>(g, xn, it, lane, A); gather_consume<H16>(c_hi, c_lo, qd, lane, A); }
  }
}
template <bool H16>
static __device__ __noinline__ void gather_tile_strided(const nsb_grid& g, float* c_hi, float x0, float x1, float x2, int warp, int lane) {
  const float xn[3] = {x0, x1, x2};
  gather_tile_t<false, H16>(g, c_hi, xn, warp, lane);
}
template <bool H16 = false>
__device__ __forceinline__ void gather_tile(const nsb_grid& g, float* c_hi, const float xn[3], int warp, int lane) {
  if (grid_fast(g)) gather_tile_t<true, H16>(g, c_hi, xn, warp, lane);
  else gather_tile_strided<H16>(g, c_hi, xn[0], xn[1], xn[2], warp, lane);
}
// this thread's 16 features of embedding block `blk` of its point -> [128 x 32] tile
template <bool H16 = false>
__device__ __forceinline__ void embed_tile(float* e_hi, const float* B, const float pf[3], int row, int cg, int blk) {
  float* e_lo = e_hi + TM * 32;
#pragma unroll
  for (int kq = kKQ * cg; kq < kKQ * cg + kKQ; kq++) {
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int f = 32 * blk + 4 * kq + j;
      float x = pf[0] * B[f]; x = fmaf(pf[1], B[kEmbPad + f], x); x = fmaf(pf[2], B[2 * kEmbPad + f], x);
      v[j] = f < kEmb ? __sinf(reduce_2pi(x)) : 0.0f;
    }
    if (H16) put4_h(e_hi, row, kq, make_float4(v[0], v[1], v[2], v[3]));
    else tc::put4(e_hi, e_lo, row, kq, 32, make_float4(v[0], v[1], v[2], v[3]));
  }
}

// ---- forward: the MMA groups of one decoder, executed by every thread (each warpgroup for its own rows) ---------------------------------
// Register accumulators: D1 (layers 0, 1, 2, 4) and D3 (layer 3: its skip part E * W3E^T is accumulated while the embedding blocks are live).
// D2 = fc_c of the five layers is computed one 32-column chunk at a time over a whole C half and stored once, in fragment order, to this
// thread's region of the accumulator slot (tc::s_acc): chunk i of thread tid at floats (i * kThreads + tid) * 16.  Only the thread that
// stored a fragment reads it back (at layer i's epilogue), so the store needs no barrier.  Chunk 5 holds D3 between layer 0 and layer 3.
__device__ __forceinline__ float4* d2_frag(int i) { return reinterpret_cast<float4*>(tc::s_acc + ((size_t)i * kThreads + threadIdx.x) * 16); }
__device__ __forceinline__ void ld_frag(const float4* p, float (&d)[16]) {
#pragma unroll
  for (int k = 0; k < 4; k++) { const float4 v = p[k]; d[4 * k] = v.x; d[4 * k + 1] = v.y; d[4 * k + 2] = v.z; d[4 * k + 3] = v.w; }
}
__device__ __forceinline__ void st_frag(float4* p, const float (&d)[16]) {
#pragma unroll
  for (int k = 0; k < 4; k++) p[k] = make_float4(d[4 * k], d[4 * k + 1], d[4 * k + 2], d[4 * k + 3]);
}
// C tile `half` -> D2 (+)= C * Wc^T in three MMA groups: chunks (0, 1) and (2, 3) as one 64-column group each into [d1 | d3] (dead until
// layer 0), chunk 4 as a 32-column group into d1; each group is waited for and stored before the next one reuses the registers.  The half's
// units and operand buffer are released after the last group.  kAccumulate: C half 1 adds onto the chunks of half 0 (a template argument:
// each group's accumulators are set up by straight-line code).  Per element the products come in the order of one m64n32 group per chunk.
template <bool H16, bool kAccumulate>
__device__ __forceinline__ void issue_fc(Issuer& I, const TileSmem& t, float (&d1)[16], float (&d3)[16]) {
  constexpr int nu = H16 ? 2 : 4;                                // units of one C half: [160 x 16] FP16 / [160 x 8] tf32 (all in the ring at once)
  const int b = I.g & 1;
  issuer_wait_operands(I, t, b, (I.g >> 1) & 1u);
  NSB_PH(5);
#pragma unroll 1
  for (int u = 0; u < nu; u++) issuer_unit(I, t, u);
  NSB_PH(11);
#pragma unroll
  for (int c = 0; c < 5; c += 2) {                               // chunk c = fc_c of layer c
    const bool pair = c < 4;
    if (kAccumulate) { ld_frag(d2_frag(c), d1); if (pair) ld_frag(d2_frag(c + 1), d3); }
    else { zero16_opaque(d1); if (pair) zero16_opaque(d3); }
    tc::wg_fence();
#pragma unroll
    for (int u = 0; u < nu; u++) {
      if (pair) mma_rows64<H16, 1>(d1, d3, t.a[b], H16 ? 16 * u : 8 * u, issued_unit(I, t, u), 160, H16 ? 16 : 8, c);
      else mma_rows<H16, 1>(d1, t.a[b], H16 ? 16 * u : 8 * u, issued_unit(I, t, u), 160, H16 ? 16 : 8, c);
    }
    tc::wg_commit(); tc::wg_wait0(); tc::fence_acc(d1);
    st_frag(d2_frag(c), d1);
    if (pair) { tc::fence_acc(d3); st_frag(d2_frag(c + 1), d3); }
  }
  release_units(I, t, nu, t.bars + B_DONE + b);
  I.g++;
}
// [D1 | D3] += E_blk * [W0_blk; W3E_blk]^T  (coarse: E = C).  The blocks of layer 0 are one chain of groups on the same accumulators, committed
// without a wait: the next block's embedding is computed while this block's MMAs run.  The caller retires the groups (wait_group) and then
// releases their units and operand buffers (release_l0).
template <bool H16 = false>
__device__ __forceinline__ void issue_l0(Issuer& I, const TileSmem& t, float (&d1)[16], float (&d3)[16]) {
  constexpr int nu = H16 ? 1 : 2;                                // one [64 x 32] FP16 unit / two [64 x 16] tf32 units
  const int b = I.g & 1;
  issuer_wait_operands(I, t, b, (I.g >> 1) & 1u);
  NSB_PH(10);
#pragma unroll 1
  for (int u = 0; u < nu; u++) issuer_unit(I, t, u);             // (the ring holds this block's and the previous block's units)
  tc::wg_fence();
#pragma unroll
  for (int u = 0; u < nu; u++) mma_rows64<H16, 2>(d1, d3, t.a[b], 16 * u, issued_unit(I, t, u), 64, H16 ? 32 : 16, 0);
  tc::wg_commit();
  I.issued += nu;
  I.g++;
}
// layer-0 groups I.g - back .. I.g - back + count - 1 have completed in this warpgroup: release their units and operand buffers
template <bool H16 = false>
__device__ __forceinline__ void release_l0(const Issuer& I, const TileSmem& t, uint32_t back, uint32_t count) {
  constexpr uint32_t nu = H16 ? 1 : 2;
  for (uint32_t j = back; j > back - count; j--) arrive_units(t, I.issued - j * nu, nu, t.bars + B_DONE + ((I.g - j) & 1u));
}
// layer i (1..4) of this warpgroup's rows from its rows of the H tile of layer i-1 into d1 (layer 3 accumulates onto D3); committed, not waited for
template <bool H16 = false>
__device__ __forceinline__ void issue_h(Issuer& I, const TileSmem& t, float (&d1)[16], const float (&d3)[16], const float* hbuf, int i) {
  const float* w = issuer_unit(I, t);
  if (i == 3) {
#pragma unroll
    for (int e = 0; e < 16; e++) d1[e] = d3[e];
  } else {
    zero16(d1);
  }
  tc::wg_fence();
  mma_rows<H16, H16 ? 2 : 4>(d1, hbuf, 0, w, 32, 32, 0);
  tc::wg_commit();
}

// ---- forward of one decoder.  n = operand-group counter of the groups that both warpgroups write (gather, embedding).  out[] = decoder
// outputs of this thread's row.  masks / acts: this decoder's ReLU-mask words / layer outputs of the tile's point 0 (point stride 15 / 160), or nullptr.
template <bool H16 = false>
__device__ __forceinline__ void epi_forward(const KParams& P, const TileSmem& t, Issuer& I, int lv, const PointGeom& G, uint32_t& n, int hb, uint32_t hdr_parity,
                                            float (&out)[4], uint32_t* __restrict__ masks, float* __restrict__ acts, int npts) {
  const int row = threadIdx.x & (TM - 1), cg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool xyz = lv != 0;
  const int cd = op_cd(lv), no = lv == 3 ? 4 : 1;
  const float* hdr = t.hdr + hb * kHdrFloats;
  float d1[16], d3[16];                                          // (the fc_c chunks pass through them before layer 0)
  if (xyz) {
    for (int half = 0; half < cd / 32; half++) {
      if (n >= 2) wait_group(t, n - 2);
      if (threadIdx.x == 0) loader_top_up(I.L, t, I.issued);     // request whatever fits the ring before the long gather
      gather_tile<H16>(P.in.grid[half == 0 ? lv : 1], t.a[n & 1], G.xn, warp, lane);
      NSB_PH(1);
      publish(t, n & 1); n++;
      if (half == 0) issue_fc<H16, false>(I, t, d1, d3); else issue_fc<H16, true>(I, t, d1, d3);
      NSB_PH(2);
    }
    mbar_wait_b(t.bars + B_HDR + hb, hdr_parity);
    zero16_opaque(d1); zero16_opaque(d3);                        // (straight-line zeros would be materialised inside the MMA group)
#pragma unroll
    for (int blk = 0; blk < 3; blk++) {                          // (unrolled: every wait below follows a whole MMA group in the code)
      if (n >= 2) wait_group(t, n - 2);
      if (threadIdx.x == 0) loader_top_up(I.L, t, I.issued);
      NSB_PH(6);
      embed_tile<H16>(t.a[n & 1], hdr + 464, G.pf, row, cg, blk);
      NSB_PH(3);
      publish(t, n & 1); n++;
      issue_l0<H16>(I, t, d1, d3);
      // the ring holds two blocks' units: block 0 is retired here to make room for block 2's
      if (blk == 1) { tc::wg_wait<1>(); release_l0<H16>(I, t, 2, 1); }
      NSB_PH(4);
    }
  } else {
    if (n >= 2) wait_group(t, n - 2);
    gather_tile<H16>(P.in.grid[0], t.a[n & 1], G.xnc, warp, lane);
    publish(t, n & 1); n++;
    zero16_opaque(d1); zero16_opaque(d3);
    issue_l0<H16>(I, t, d1, d3);
    mbar_wait_b(t.bars + B_HDR + hb, hdr_parity);
  }
  tc::wg_wait0(); tc::fence_acc(d1); tc::fence_acc(d3);          // layer 0 has completed
  release_l0<H16>(I, t, xyz ? 2 : 1, xyz ? 2 : 1);
  st_frag(d2_frag(5), d3);                                       // D3 waits for layer 3 in the slot (fewer live registers in layers 1, 2)
  // Hidden layers.  H tiles go to buffer n & 1: every group of this warpgroup has completed (the wait above), and each warpgroup writes and reads
  // only its own rows of it.
  float* hbuf = t.a[n & 1];
  const int wg = threadIdx.x >> 7, q = lane & 3;
  const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);        // rows of this thread's fragment: r0 (elements e with bit 1 clear) and r0 + 8
  float v2[16];
  if (xyz) ld_frag(d2_frag(0), v2);
#pragma unroll 1
  for (int i = 0; i < 5; i++) {
    if (threadIdx.x == 0) loader_top_up(I.L, t, I.issued);       // the layer's weight slot is free: request the next units now, under the epilogue
    NSB_PH(7);
    // epilogue of layer i on the fragment: h = relu(D + b_i) + (D2_i + bc_i)
    uint32_t m0 = 0, m1 = 0;                                     // ReLU bits of rows r0 / r0 + 8, this thread's columns
#pragma unroll
    for (int e = 0; e < 16; e++) {
      const int c = 8 * (e >> 2) + 2 * q + (e & 1);
      const float u = d1[e] + hdr[i * 32 + c];
      const uint32_t bit = u > 0.0f ? 1u << (8 * (e >> 2) + (e & 1)) : 0u;
      if (e & 2) m1 |= bit; else m0 |= bit;
      float h = u > 0.0f ? u : 0.0f;
      if (xyz) h += v2[e] + hdr[160 + i * 32 + c];
      d1[e] = h;
    }
    if (masks != nullptr) {                                      // one 32-bit word per point and layer, bit j = column j
      m0 <<= 2 * q; m1 <<= 2 * q;
      m0 |= __shfl_xor_sync(0xffffffffu, m0, 1); m1 |= __shfl_xor_sync(0xffffffffu, m1, 1);
      m0 |= __shfl_xor_sync(0xffffffffu, m0, 2); m1 |= __shfl_xor_sync(0xffffffffu, m1, 2);
      if (q == 0 && r0 < npts) masks[(size_t)r0 * 15 + i] = m0;
      if (q == 1 && r0 + 8 < npts) masks[(size_t)(r0 + 8) * 15 + i] = m1;
    }
    if (acts != nullptr) {                                       // layer outputs kept for the tensor-core weight gradients of the backward
#pragma unroll
      for (int e = 0; e < 16; e += 2) {
        const int r = r0 + 8 * ((e >> 1) & 1), c = 8 * (e >> 2) + 2 * q;
        if (r < npts) __stcg(reinterpret_cast<float2*>(acts + (size_t)r * 160 + i * 32 + c), make_float2(d1[e], d1[e + 1]));
      }
    }
    if (i == 4) break;
    if (i == 2) ld_frag(d2_frag(5), d3);
    // H tile (canonical K-major, hi | lo): two adjacent columns of a row per 8-byte (tf32) / 4-byte (fp16) store
#pragma unroll
    for (int e = 0; e < 16; e += 2) {
      const int r = r0 + 8 * ((e >> 1) & 1), c = 8 * (e >> 2) + 2 * q;
      if (H16) {
        unsigned char* hp = reinterpret_cast<unsigned char*>(hbuf) + (((r >> 3) * 4 + (c >> 3)) * 128 + (r & 7) * 16 + (c & 7) * 2);
        uint32_t hh, ll;
        split_h2(d1[e], d1[e + 1], hh, ll);
        *reinterpret_cast<uint32_t*>(hp) = hh;
        *reinterpret_cast<uint32_t*>(hp + TM * 32 * 2) = ll;
      } else {
        put2(hbuf, r, c, d1[e], d1[e + 1]);
      }
    }
    NSB_PH(8);
    fence_proxy_async();
    wg_bar_sync();                                               // this warpgroup's rows of H are written -> its MMA
    issue_h<H16>(I, t, d1, d3, hbuf, i + 1);
    NSB_PH(9);
    // layer i + 1 is waited for here, on the path that issued it (a wait under `i > 0` at the top of the loop left ptxas a path on
    // which the epilogue reads an accumulator in flight)
    if (xyz) ld_frag(d2_frag(i + 1), v2);                        // (issued before the wait: the load latency hides under the MMA)
    tc::wg_wait0(); tc::fence_acc(d1); release_units(I, t, 1);
  }
  NSB_PH(8);
  // output layer: per-row dot products over the fragment, summed over the four lanes of a row; handed to the row owners through this
  // warpgroup's rows of the H tile (its last MMA has completed)
  float s0[4], s1[4];
#pragma unroll
  for (int o = 0; o < 4; o++) {
    s0[o] = s1[o] = 0.0f;
    if (o < no) {
#pragma unroll
      for (int e = 0; e < 16; e++) {
        const float w = hdr[336 + o * 32 + 8 * (e >> 2) + 2 * q + (e & 1)];
        if (e & 2) s1[o] = fmaf(d1[e], w, s1[o]); else s0[o] = fmaf(d1[e], w, s0[o]);
      }
    }
    s0[o] += __shfl_xor_sync(0xffffffffu, s0[o], 1); s1[o] += __shfl_xor_sync(0xffffffffu, s1[o], 1);
    s0[o] += __shfl_xor_sync(0xffffffffu, s0[o], 2); s1[o] += __shfl_xor_sync(0xffffffffu, s1[o], 2);
  }
  constexpr int kWgHiFloats = 64 * 32 / (H16 ? 2 : 1);          // one warpgroup's rows of the hi tile
  auto part = [&](int r) { return reinterpret_cast<float4*>(hbuf + (r >> 6) * kWgHiFloats + (r & 63) * 4); };
  if (q == 0) *part(r0) = make_float4(s0[0], s0[1], s0[2], s0[3]);
  if (q == 1) *part(r0 + 8) = make_float4(s1[0], s1[1], s1[2], s1[3]);
  epi_sync();
  {
    const float4 v = *part(row);
    out[0] = hdr[320] + v.x; out[1] = hdr[321] + v.y; out[2] = hdr[322] + v.z; out[3] = hdr[323] + v.w;
  }
  epi_sync();                                                    // partials consumed before the next decoder's gather reuses the buffer
  NSB_PH(12);
}

// ---- tensor-core weight gradients (the colour decoder in the mapper's colour stage, src/Mapper.py:339-341,503, the fine decoder with ---------
// fix_fine = False; with option wgrad_all also the middle and coarse decoders, which the tracker's and mapper's autograd ask for) -----------
// dW_i = DU_i^T X_i, dWc_i = G_i^T C, dWo = g_out^T H_4, dB = P^T DX are contractions over the POINTS of a tile: both operands of the MMA have the
// points as K.  wgmma takes tf32 operands K-major only, so the epilogue threads write the rows they own a second time, transposed, into
// [feature][point] tiles (the canonical no-swizzle layout with K = 128 points): DU_i and G_i form the A operand (M = 64 = [DU | G], hi tiles
// adjacent, then the lo tiles), the layer inputs X_i come back from the forward's `acts`, C and the embedding blocks are recomputed.  One MMA
// group = 16 k-steps x 3 (3xTF32) with N = 32, issued by warpgroup 0; rows 0..31 (DU part) or 32..63 (G part) of its fragments are reduced
// into the packed gradient image with 8-byte vector reductions.
constexpr int kMnTile = TM * 32;                               // floats of one tile (16 KB)
constexpr size_t kWgBytes = (size_t)6 * kMnTile * 4;           // A: DU hi, G hi, DU lo, G lo (64 KB)  B: one tile hi|lo (32 KB)
constexpr int kWgALo = 2 * kMnTile, kWgBLo = kMnTile;          // offsets of the lo tiles
struct WgSmem { float* du; float* g; float* b; float* dpk; };
// block of decoder lv in fo.acts / bw.acts (levels of `mask` in level order), -1 if its layer outputs are not kept
__host__ __device__ __forceinline__ int acts_slot(int mask, int lv) { return (mask >> lv) & 1 ? __builtin_popcount(mask & ((1 << lv) - 1)) : -1; }
// packed-gradient offsets of a weight-gradient decoder: fine (fc_c input [c_fine | c_middle], 64 wide; one output), colour (32; four), middle
// (32; one) and coarse (no embedding, no fc_c: layer 0 and the skip part of layer 3 read the coarse features, 32 wide; one output)
struct WgDec { int o_W0, o_W1, o_W2, o_W3E, o_W3H, o_W4, o_WC, PC, o_WO, no, o_b, o_bc, o_bo; };
template <int LV>
__device__ __forceinline__ WgDec wg_dec() {
  using D = Dec<LV>;
  return WgDec{D::o_W0, D::o_W1, D::o_W2, D::o_W3E, D::o_W3H, D::o_W4, D::o_WC, D::PC, D::o_WO, D::NO, D::o_b, D::o_bc, D::o_bo};
}
static_assert(Dec<0>::PH == Dec<3>::PH && Dec<1>::PH == Dec<3>::PH && Dec<2>::PH == Dec<3>::PH, "shared hidden pitch of the WG decoders");
static_assert(Dec<1>::PF == Dec<3>::PF && Dec<2>::PF == Dec<3>::PF && Dec<1>::o_B == Dec<3>::o_B && Dec<2>::o_B == Dec<3>::o_B,
              "shared first-input pitch and embedding block of the xyz WG decoders");
static_assert(Dec<1>::o_WO == Dec<3>::o_WO && Dec<1>::o_bo == Dec<3>::o_bo && Dec<1>::TOTAL == Dec<3>::TOTAL, "middle decoder = colour layout");
__device__ __forceinline__ void split4(const float4 v, float4& h, float4& l) {
  h = make_float4(tc::to_tf32(v.x), tc::to_tf32(v.y), tc::to_tf32(v.z), tc::to_tf32(v.w));
  l = make_float4(v.x - h.x, v.y - h.y, v.z - h.z, v.w - h.w);
}
// element (feature f, point p) of a [32 x 128] K-major tile
__device__ __forceinline__ int kt_idx(int f, int p) { return ((f >> 3) * (TM / 4) + (p >> 2)) * 32 + (f & 7) * 4 + (p & 3); }
// features [16 cg, 16 cg + 16) of point p -> hi | lo tiles
__device__ __forceinline__ void put_kt16(float* hi, int lo_off, int p, int cg, const float (&v)[kCW]) {
#pragma unroll
  for (int j = 0; j < kCW; j++) {
    const float h = tc::to_tf32(v[j]);
    const int o = kt_idx(kCW * cg + j, p);
    hi[o] = h; hi[lo_off + o] = v[j] - h;
  }
}
// element (feature f, point p) -> hi | lo tiles
__device__ __forceinline__ void put_kt1(float* hi, int lo_off, int f, int p, float v) {
  const float h = tc::to_tf32(v);
  const int o = kt_idx(f, p);
  hi[o] = h; hi[lo_off + o] = v - h;
}
__device__ __forceinline__ void get_kt16(const float* hi, int lo_off, int p, int cg, float (&v)[kCW]) {      // hi + lo = the value that was split
#pragma unroll
  for (int j = 0; j < kCW; j++) { const int o = kt_idx(kCW * cg + j, p); v[j] = hi[o] + hi[lo_off + o]; }
}
// gather_tile with the transposed destination (lane q of a point holds channels [4 q, 4 q + 4))
__device__ __forceinline__ void gather_tile_kt(const nsb_grid& g, float* c_hi, int lo_off, const float xn[3], int warp, int lane) {
  const bool fast = grid_fast(g);
  const int qd = warp & 3, it0 = (warp >> 2) * 4, q = lane & 7;
#pragma unroll 1
  for (int it = it0; it < it0 + 4; it++) {
    GatherPass A;
    if (fast) gather_issue<true>(g, xn, it, lane, A); else gather_issue<false>(g, xn, it, lane, A);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int k = 0; k < 8; k++) {
      const float w = A.w[k];
      acc.x = fmaf(A.v[k].x, w, acc.x); acc.y = fmaf(A.v[k].y, w, acc.y); acc.z = fmaf(A.v[k].z, w, acc.z); acc.w = fmaf(A.v[k].w, w, acc.w);
    }
    const int p = qd * 32 + A.src_lane;
    float4 xh, xl; split4(acc, xh, xl);
    const float hv[4] = {xh.x, xh.y, xh.z, xh.w}, lv[4] = {xl.x, xl.y, xl.z, xl.w};
#pragma unroll
    for (int c = 0; c < 4; c++) { const int o = kt_idx(4 * q + c, p); c_hi[o] = hv[c]; c_hi[lo_off + o] = lv[c]; }
  }
}
// One group, called by every thread: the B tile (and, the first time in a layer, the A tiles) have been written by all threads.  part 0 = rows of
// the DU block (D rows 0..31), part 1 = rows of the G block (32..63); dst = packed-image address of element (out 0, in 0), pitch in floats;
// n_rows <= 32 rows are reduced.
__device__ __forceinline__ void wg_group(WgSmem& w, int part, float* dst, int pitch, int n_rows, bool transposed3 = false) {
  fence_proxy_async();
  __syncthreads();
  // warpgroup 0: D[64 x 32] = [DU | G] . B^T over the 128 points (the index comes through a shuffle: ptxas then knows the branch is
  // warp-uniform and does not serialize the group, see mma_rows)
  if (__shfl_sync(0xffffffffu, threadIdx.x >> 7, 0) == 0) {
    const uint64_t ah = tc::make_desc(w.du, 128u, 4096u), al = ah + (uint64_t)((kWgALo * 4) >> 4);
    const uint64_t bh = tc::make_desc(w.b, 128u, 4096u), bl = bh + (uint64_t)((kWgBLo * 4) >> 4);
    float d[16];
    zero16_opaque(d);
    tc::wg_fence();
#pragma unroll
    for (int ks = 0; ks < TM / 8; ks++) {                       // 8 points per k-step = two core matrices = 256 bytes
      const uint64_t o = 16u * (uint64_t)ks;
      tc::wgmma_tf32_n32(d, al + o, bh + o); tc::wgmma_tf32_n32(d, ah + o, bl + o); tc::wgmma_tf32_n32(d, ah + o, bh + o);
    }
    tc::wg_commit_wait();
    if ((threadIdx.x >> 6) == part) {                            // warps 2 part, 2 part + 1 hold the rows of this part
#pragma unroll
      for (int e = 0; e < 16; e += 2) {
        int r, c; tc::frag_rc(e, r, c); r -= 32 * part;
        if (r >= n_rows) continue;
        if (transposed3) {                                       // dB[a][f] = D[f][a], a < 3 (the B tile held the three coordinates in columns 0..2)
          if (c < 3) atomicAdd(dst + (size_t)c * pitch + r, d[e]);
          if (c + 1 < 3) atomicAdd(dst + (size_t)(c + 1) * pitch + r, d[e + 1]);
        } else {
          red_add_v2(dst + (size_t)r * pitch + c, d[e], d[e + 1]);
        }
      }
    }
  }
  __syncthreads();                                               // the tiles may be rewritten
}
// column sums of a [32 rows (lanes)][16] register tile: lane l returns the sum of column ((l >> 4) & 1) * 8 + ((l >> 3) & 1) * 4 + ((l >> 2) & 1) * 2 + ((l >> 1) & 1)
__device__ __forceinline__ float warp_colsum16(const float (&v)[kCW], int lane) {
  float a[8];
#pragma unroll
  for (int j = 0; j < 8; j++) { const float give = (lane & 16) ? v[j] : v[j + 8], keep = (lane & 16) ? v[j + 8] : v[j]; a[j] = keep + __shfl_xor_sync(0xffffffffu, give, 16); }
  float b[4];
#pragma unroll
  for (int j = 0; j < 4; j++) { const float give = (lane & 8) ? a[j] : a[j + 4], keep = (lane & 8) ? a[j + 4] : a[j]; b[j] = keep + __shfl_xor_sync(0xffffffffu, give, 8); }
  float c[2];
#pragma unroll
  for (int j = 0; j < 2; j++) { const float give = (lane & 4) ? b[j] : b[j + 2], keep = (lane & 4) ? b[j + 2] : b[j]; c[j] = keep + __shfl_xor_sync(0xffffffffu, give, 4); }
  const float give = (lane & 2) ? c[0] : c[1], keep = (lane & 2) ? c[1] : c[0];
  float d = keep + __shfl_xor_sync(0xffffffffu, give, 2);
  d += __shfl_xor_sync(0xffffffffu, d, 1);
  return d;
}
__device__ __forceinline__ int colsum_col(int lane) { return ((lane >> 4) & 1) * 8 + ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1); }
// column sums of a warp's 16 rows of an m64n32 fragment: lane l returns the sum of column frag_colsum_col(l) (the eight lanes with the same
// l & 3 hold the same columns: reduce-scatter over lane bits 4, 3, 2)
__device__ __forceinline__ float frag_colsum(const float (&v)[16], int lane) {
  float a[8];                                                    // a[2 j + k] = column 8 j + 2 (l & 3) + k, both rows
#pragma unroll
  for (int j = 0; j < 8; j++) a[j] = v[4 * (j >> 1) + (j & 1)] + v[4 * (j >> 1) + (j & 1) + 2];
  float b[4];
#pragma unroll
  for (int j = 0; j < 4; j++) { const float give = (lane & 16) ? a[j] : a[j + 4], keep = (lane & 16) ? a[j + 4] : a[j]; b[j] = keep + __shfl_xor_sync(0xffffffffu, give, 16); }
  float c[2];
#pragma unroll
  for (int j = 0; j < 2; j++) { const float give = (lane & 8) ? b[j] : b[j + 2], keep = (lane & 8) ? b[j + 2] : b[j]; c[j] = keep + __shfl_xor_sync(0xffffffffu, give, 8); }
  const float give = (lane & 4) ? c[0] : c[1], keep = (lane & 4) ? c[1] : c[0];
  return keep + __shfl_xor_sync(0xffffffffu, give, 4);
}
__device__ __forceinline__ int frag_colsum_col(int lane) {
  const int j = ((lane >> 4) & 1) * 4 + ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1);
  return 8 * (j >> 1) + 2 * (lane & 3) + (j & 1);
}

// ---- backward (input gradients) ------------------------------------------------------------------------------------------------------
// Register accumulators, as in the forward: warpgroup g issues and waits for the MMAs of its rows [64 g, 64 g + 64), and every accumulator
// is a wgmma m64n32 fragment (tc::frag_rc) in the registers of the threads that run the epilogue on it:
//   D1 = DU_i * W_i[:, hidden]   (dL/dh_{i-1}: from layer i's MMA to layer i-1's epilogue)
//   DC = sum_i G_i * Wc_i        (dL/dc, accumulated over the five layers)
//   DF = DU_3 * W_3[:, first] + DU_0 * W_0   (dL/d first input; 96 columns, the coarse decoder's 32 are dL/dc)
// DF does not fit beside the others: its 32-column chunks live in this thread's fragment-order region of the slot (d2_frag) between layer 3
// and layer 0, and are read back by the same thread only (no barrier).  DC keeps only the first 32 columns: the scatter reads no others (the
// fine decoder's middle-grid features are detached), so the units of its second DC chunk are consumed without an MMA.
struct BwdExtra {            // behind the common shared-memory part
  double dp[TM * 3];
  double z[TM];
  float gocc[TM];
  float wgt[TM];
  float gc[kMaxTileRays * 3];
};
// dL/d(decoder output) of tile row r (zero beyond npts): colour decoder = compositing weight x dL/d rgb of its ray, else dL/d occupancy logit.
// off0 = index of the tile's first point within its first ray.
__device__ __forceinline__ void bwd_gout(const BwdExtra& X, int lv, int r, int npts, int off0, int S, float (&go)[4]) {
  go[0] = go[1] = go[2] = go[3] = 0.0f;
  if (r >= npts) return;
  if (lv == 3) { const float w = X.wgt[r]; const float* gc = X.gc + 3 * ((off0 + r) / S); go[0] = w * gc[0]; go[1] = w * gc[1]; go[2] = w * gc[2]; }
  else go[0] = X.gocc[r];
}

// Layer i of this warpgroup's rows, from its rows of the G (a[0]) and DU (a[1]) tiles: DC += G * Wc_i, D1 = DU * W_i[:, hidden] (i >= 1),
// DF += DU * W_i[:, first input] (i = 3, 0).  A layer has up to six units (fine decoder, layer 3) for the four ring slots: they go out in waves
// of at most kSlots units, each wave committed, waited for and released at once.  A wave carries one DF chunk (accumulator fa), two at layer 0,
// where D1 is free to take the second: more would not fit in the registers beside D1 and DC.
// Which MMAs a wave issues is fixed at compile time (DC: the decoder has a DC chain; NDF DF chunks; L0 = layer 0), so that every wave is one
// straight-line MMA group (see mma_rows); only the number of DC units, ndc, which shifts the others in the ring, is a run-time value.
template <bool DC, int NDF, bool L0>
__device__ __forceinline__ void issue_bwd_layer_t(Issuer& I, const TileSmem& t, int ndc, float (&d1)[16], float (&dc)[16], float (&fa)[16]) {
  constexpr int ND1 = L0 ? 0 : 1, FMAX = L0 ? 2 : 1;             // D1 units, DF chunks per wave
  constexpr int kWaves = NDF > FMAX ? (NDF + FMAX - 1) / FMAX : 1;
#pragma unroll
  for (int wave = 0; wave < kWaves; wave++) {
    const int f0 = wave * FMAX;                                  // first DF chunk of the wave
    const int nf = NDF - f0 < FMAX ? NDF - f0 : FMAX;
    const int k = wave == 0 ? ndc + ND1 : 0;                     // unit of the wave's first DF chunk
    const int nu = k + nf;
#pragma unroll 1
    for (int u = 0; u < nu; u++) issuer_unit(I, t, u);
    if (nf > 0) { if (L0) ld_frag(d2_frag(f0), fa); else zero16_opaque(fa); }
    if (nf > 1) ld_frag(d2_frag(f0 + 1), d1);
    if (wave == 0 && ND1) zero16_opaque(d1);
    tc::wg_fence();
    if (wave == 0) {
      if (DC) mma_rows<false, 4>(dc, t.a[0], 0, issued_unit(I, t, 0), 32, 32, 0);
      if (ND1) mma_rows<false, 4>(d1, t.a[1], 0, issued_unit(I, t, ndc), 32, 32, 0);
    }
    if (nf > 0) mma_rows<false, 4>(fa, t.a[1], 0, issued_unit(I, t, k), 32, 32, 0);
    if (nf > 1) mma_rows<false, 4>(d1, t.a[1], 0, issued_unit(I, t, k + 1), 32, 32, 0);
    tc::wg_commit(); tc::wg_wait0();
    tc::fence_acc(dc); tc::fence_acc(d1); tc::fence_acc(fa);
    if (nf > 0) st_frag(d2_frag(f0), fa);
    if (nf > 1) st_frag(d2_frag(f0 + 1), d1);
    release_units(I, t, nu);
  }
}
template <bool XYZ>
__device__ __forceinline__ void issue_bwd_layer_x(Issuer& I, const TileSmem& t, int ndc, int i, float (&d1)[16], float (&dc)[16], float (&fa)[16]) {
  constexpr int NDF = op_firstp(XYZ ? 1 : 0) / 32;               // (the same for every xyz decoder)
  if (XYZ && i == 4) zero16_opaque(dc);
  if (i == 3) issue_bwd_layer_t<XYZ, NDF, false>(I, t, ndc, d1, dc, fa);
  else if (i == 0) issue_bwd_layer_t<XYZ, NDF, true>(I, t, ndc, d1, dc, fa);
  else issue_bwd_layer_t<XYZ, 0, false>(I, t, ndc, d1, dc, fa);
}
__device__ __forceinline__ void issue_bwd_layer(Issuer& I, const TileSmem& t, int lv, int i, float (&d1)[16], float (&dc)[16], float (&fa)[16]) {
  if (lv != 0) issue_bwd_layer_x<true>(I, t, op_cd(lv) / 32, i, d1, dc, fa);
  else issue_bwd_layer_x<false>(I, t, 0, i, d1, dc, fa);
}

// ---- backward of one decoder.  Leaves dL/dc rows ([128][32] fp32) in a[0] and the embedding-chain part of dL/dp ([128][4] fp32, row r at
// a[1] + bwd_dpe_off(r)) in a[1]; the caller scatters after an epi_sync().  Each warpgroup writes both into its own rows of the operand tiles,
// which only its own (completed) MMAs read.  masks = this decoder's ReLU-mask words of the tile's point 0 (point stride 15).
// WG = which weight gradients the instantiation computes: none (input gradients only, any decoder), those of the xyz decoders (middle, fine,
// colour) or those of the coarse decoder (no embedding, no fc_c).  The coarse decoder has its own instantiation: its branches compiled into
// the xyz one took that kernel past 255 registers (spills).
enum { kWgNone = 0, kWgXyz = 1, kWgCoarse = 2 };
__device__ __forceinline__ int bwd_dpe_off(int r) { return (r >> 6) * (64 * 32) + (r & 63) * 4; }
// Bias gradients: the per-warp column sums are added in warp order through shared memory, so a tile contributes one sum per element.  The
// default kernels add that sum to w->dpk with one atomic (the order of the atomics is then the order of the tiles alone, not of the tiles'
// eight warps); kDet (deterministic mode) stores it, w->dpk being this tile's own zeroed partial image, which every other element of receives
// exactly one reduction per tile.
__device__ __forceinline__ float* det_bias_smem() { __shared__ float s[8 * 64]; return s; }
template <int WG, bool kDet = false>
__device__ __forceinline__ void epi_backward(const KParams& P, const TileSmem& t, Issuer& I, const BwdExtra& X, int lv, const PointGeom& G, int hb, uint32_t hdr_parity,
                                             const uint32_t* __restrict__ masks, int npts, int off0, long long gp0, WgSmem* w = nullptr, const float* acts_row = nullptr) {
  const int row = threadIdx.x & (TM - 1), cg = threadIdx.x >> 7, warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31, q = lane & 3;
  const int r0 = 64 * (threadIdx.x >> 7) + 16 * (warp & 3) + (lane >> 2);      // rows of this thread's fragment: r0 (elements e with bit 1 clear) and r0 + 8
  const int S = P.S;
  constexpr bool kWg = WG != kWgNone;
  constexpr int PH = Dec<3>::PH, PF = WG == kWgCoarse ? Dec<0>::PF : Dec<3>::PF;      // (PH: the same for every WG decoder)
  // packed gradient image of this WG decoder.  The middle decoder's is the colour decoder's layout with one output: rows 1..3 of dWo and
  // dbo[1..3], padding of its image that the unpack does not read, receive the zero columns 1..3 of its g_out.
  const WgDec DW = WG == kWgCoarse ? wg_dec<0>() : lv == 2 ? wg_dec<2>() : wg_dec<3>();
  float creg[kCW], cmid[kCW];                                    // WG: this thread's 16 grid features of its point (fine: + the middle grid's)
  const bool xyz = WG == kWgCoarse ? false : lv != 0;
  const float* hdr = t.hdr + hb * kHdrFloats;
  // ReLU bits of this thread's elements: word i of a row shifted right by 2 q puts column 8 j + 2 q + k on bit 8 j + k; row r0 + 8 goes to bits
  // 8 j + 2 + k, and layers (0, 1) / (2, 3) share m01 / m23 (odd layer in the high nibble of each byte)
  uint32_t m01 = 0, m23 = 0, m4 = 0;
  {
    const uint32_t* w0 = masks + (size_t)(r0 < npts ? r0 : npts - 1) * 15;
    const uint32_t* w1 = masks + (size_t)(r0 + 8 < npts ? r0 + 8 : npts - 1) * 15;
#pragma unroll
    for (int i = 0; i < 5; i++) {
      const uint32_t v = ((w0[i] >> (2 * q)) & 0x03030303u) | (((w1[i] >> (2 * q)) & 0x03030303u) << 2);
      if (i == 4) m4 = v; else if (i & 2) m23 |= v << (4 * (i & 1)); else m01 |= v << (4 * (i & 1));
    }
  }
  mbar_wait_b(t.bars + B_HDR + hb, hdr_parity);
  float d1[16], dc[16], fa[16];
  {
    float go0[4], go1[4];
    bwd_gout(X, lv, r0, npts, off0, S, go0); bwd_gout(X, lv, r0 + 8, npts, off0, S, go1);
#pragma unroll
    for (int e = 0; e < 16; e++) {
      float v = 0.0f;
#pragma unroll
      for (int o = 0; o < 4; o++) v = fmaf(hdr[336 + o * 32 + 8 * (e >> 2) + 2 * q + (e & 1)], (e & 2) ? go1[o] : go0[o], v);      // rows >= NO are zero
      d1[e] = v;
    }
  }
  if constexpr (kWg) {
    float g_out[4];
    bwd_gout(X, lv, row, npts, off0, S, g_out);
    // grid features of this point -> registers (gathered once through the B tile; the coarse grid at the enlarged coarse bound)
    gather_tile_kt(P.in.grid[lv], w->b, kWgBLo, WG == kWgCoarse ? G.xnc : G.xn, warp, lane);
    __syncthreads();
    get_kt16(w->b, kWgBLo, row, cg, creg);
    __syncthreads();
    if (lv == 2) {                                               // the fine decoder's fc_c also reads the middle features (no gradient into them)
      gather_tile_kt(P.in.grid[NSB_MIDDLE], w->b, kWgBLo, G.xn, warp, lane);
      __syncthreads();
      get_kt16(w->b, kWgBLo, row, cg, cmid);
      __syncthreads();
    }
    // output layer: dWo = g_out^T H_4 (A block 0 = g_out in columns 0..3), dbo = column sums of g_out
    float go[kCW];
#pragma unroll
    for (int j = 0; j < kCW; j++) go[j] = (cg == 0 && j < 4) ? g_out[j] : 0.0f;
    put_kt16(w->du, kWgALo, row, cg, go);
    float h4[kCW];
#pragma unroll
    for (int k = 0; k < kKQ; k++) {
      const float4 v = acts_row != nullptr ? __ldcg(reinterpret_cast<const float4*>(acts_row + 4 * 32 + 4 * k)) : make_float4(0.f, 0.f, 0.f, 0.f);
      h4[4 * k] = v.x; h4[4 * k + 1] = v.y; h4[4 * k + 2] = v.z; h4[4 * k + 3] = v.w;
    }
    put_kt16(w->b, kWgBLo, row, cg, h4);
    wg_group(*w, 0, w->dpk + DW.o_WO, PH, DW.no);
    if (cg == 0) {
      const float sb = warp_colsum16(go, lane);
      const int col = colsum_col(lane);
      if ((lane & 1) == 0 && col < DW.no) det_bias_smem()[warp * 64 + col] = sb;
    }
    __syncthreads();
    if ((int)threadIdx.x < DW.no) {
      float s = 0.0f;
      for (int wp = 0; wp < 4; wp++) s = __fadd_rn(s, det_bias_smem()[wp * 64 + threadIdx.x]);
      if constexpr (kDet) w->dpk[DW.o_bo + threadIdx.x] = s;
      else atomicAdd(w->dpk + DW.o_bo + threadIdx.x, s);
    }
    __syncthreads();
  }
#pragma unroll 1
  for (int i = 4; i >= 0; i--) {
    const uint32_t m = (i == 4 ? m4 : (i & 2) ? m23 : m01) >> (4 * (i & 1));
    // epilogue of layer i on the fragment: g = d1, du = relu'(u_i) g -> this warpgroup's rows of the G (xyz) and DU tiles
    float du[16];
#pragma unroll
    for (int e = 0; e < 16; e++) du[e] = (m >> (8 * (e >> 2) + 2 * ((e >> 1) & 1) + (e & 1))) & 1u ? d1[e] : 0.0f;
#pragma unroll
    for (int e = 0; e < 16; e += 2) {
      const int r = r0 + 8 * ((e >> 1) & 1), c = 8 * (e >> 2) + 2 * q;
      if (xyz) put2(t.a[0], r, c, d1[e], d1[e + 1]);
      put2(t.a[1], r, c, du[e], du[e + 1]);
    }
    if constexpr (kWg) {                                         // the same values transposed ([feature][point]) and their column sums: db_i, dbc_i
#pragma unroll
      for (int e = 0; e < 16; e++) {
        const int r = r0 + 8 * ((e >> 1) & 1), c = 8 * (e >> 2) + 2 * q + (e & 1);
        put_kt1(w->du, kWgALo, c, r, du[e]);
        if constexpr (WG != kWgCoarse) put_kt1(w->g, kWgALo, c, r, d1[e]);      // (the coarse decoder has no fc_c: no G block, no dbc)
      }
      const float sb = frag_colsum(du, lane);
      float sc = 0.0f;
      if constexpr (WG != kWgCoarse) sc = frag_colsum(d1, lane);
      const int col = frag_colsum_col(lane);
      float* sbias = det_bias_smem();
      sbias[warp * 64 + col] = sb;
      if constexpr (WG != kWgCoarse) sbias[warp * 64 + 32 + col] = sc;
      __syncthreads();
      if ((int)threadIdx.x < (WG != kWgCoarse ? 64 : 32)) {
        const int c = threadIdx.x & 31;
        float s = 0.0f;
        for (int wp = 0; wp < kThreads / 32; wp++) s = __fadd_rn(s, sbias[wp * 64 + threadIdx.x]);
        float* const dst = w->dpk + (threadIdx.x < 32 ? DW.o_b : DW.o_bc) + 32 * i + c;
        if constexpr (kDet) *dst = s;
        else atomicAdd(dst, s);
      }
      __syncthreads();
    }
    fence_proxy_async();
    wg_bar_sync();                                               // this warpgroup's rows of G / DU are written -> its MMAs
    NSB_PH(22);
    issue_bwd_layer(I, t, WG == kWgCoarse ? 0 : lv, i, d1, dc, fa);
    if (threadIdx.x == 0) loader_top_up(I.L, t, I.issued);       // slots of this layer are free: fetch the next layer's units under the epilogue
    NSB_PH(23);
    if constexpr (kWg) {                                         // weight gradients of layer i
      if (i >= 1) {                                              // hidden input H_{i-1}
        float xr[kCW];
#pragma unroll
        for (int k = 0; k < kKQ; k++) {
          const float4 v = acts_row != nullptr ? __ldcg(reinterpret_cast<const float4*>(acts_row + (i - 1) * 32 + 4 * k)) : make_float4(0.f, 0.f, 0.f, 0.f);
          xr[4 * k] = v.x; xr[4 * k + 1] = v.y; xr[4 * k + 2] = v.z; xr[4 * k + 3] = v.w;
        }
        put_kt16(w->b, kWgBLo, row, cg, xr);
        const int o_wh = i == 1 ? DW.o_W1 : i == 2 ? DW.o_W2 : i == 3 ? DW.o_W3H : DW.o_W4;
        wg_group(*w, 0, w->dpk + o_wh, PH, 32);
      }
      if constexpr (WG != kWgCoarse) {
        put_kt16(w->b, kWgBLo, row, cg, creg);                           // dWc_i = G_i^T C
        wg_group(*w, 1, w->dpk + DW.o_WC + 32 * i * DW.PC, DW.PC, 32);
        if (lv == 2) {                                           // fine: columns 32..63 of dWc_i = G_i^T C_middle (a second pass over the B tile)
          put_kt16(w->b, kWgBLo, row, cg, cmid);
          wg_group(*w, 1, w->dpk + DW.o_WC + 32 * i * DW.PC + 32, DW.PC, 32);
        }
      }
      if (i == 3 || i == 0) {                                    // first-input part of W_0 / W_3: the embedding, or the coarse features
        if constexpr (WG != kWgCoarse) {
          const float* B = hdr + 464;
          for (int blk = 0; blk < 3; blk++) {
            float e[kCW];
#pragma unroll
            for (int j = 0; j < kCW; j++) {
              const int f = 32 * blk + kCW * cg + j;
              float x = G.pf[0] * B[f]; x = fmaf(G.pf[1], B[kEmbPad + f], x); x = fmaf(G.pf[2], B[2 * kEmbPad + f], x);
              e[j] = f < kEmb ? __sinf(reduce_2pi(x)) : 0.0f;
            }
            put_kt16(w->b, kWgBLo, row, cg, e);
            wg_group(*w, 0, w->dpk + (i == 0 ? DW.o_W0 : DW.o_W3E) + 32 * blk, PF, 32);
          }
        } else {                                                 // coarse: dW_0 = DU_0^T C, dW_3[:, :32] = DU_3^T C
          put_kt16(w->b, kWgBLo, row, cg, creg);
          wg_group(*w, 0, w->dpk + (i == 0 ? DW.o_W0 : DW.o_W3E), PF, 32);
        }
      }
      NSB_PH(24);
    }
  }
  // dL/dc rows -> a[0] (plain fp32 [128][32]): DC, or the coarse decoder's DF
  if (!xyz) ld_frag(d2_frag(0), dc);
#pragma unroll
  for (int e = 0; e < 16; e += 2) {
    const int r = r0 + 8 * ((e >> 1) & 1), c = 8 * (e >> 2) + 2 * q;
    *reinterpret_cast<float2*>(t.a[0] + r * 32 + c) = make_float2(dc[e], dc[e + 1]);
  }
  float dpe0[3] = {0.0f, 0.0f, 0.0f}, dpe1[3] = {0.0f, 0.0f, 0.0f};          // rows r0, r0 + 8
  if (xyz) {
    const float* B = hdr + 464;
    if constexpr (kWg) {                                         // B tile of the dB groups: the point's coordinates in columns 0..2
      float pv[kCW];
#pragma unroll
      for (int j = 0; j < kCW; j++) pv[j] = (cg == 0 && j < 3) ? G.pf[j] : 0.0f;
      put_kt16(w->b, kWgBLo, row, cg, pv);
    }
    float pf0[3], pf1[3];                                        // embedding inputs of the fragment's rows (make_point, as the row owners did)
    {
      float o[3], d[3];
      PointGeom Gr;
      const int l0 = r0 < npts ? r0 : npts - 1, l1 = r0 + 8 < npts ? r0 + 8 : npts - 1;
      const int ray0 = (int)((gp0 + l0) / S), ray1 = (int)((gp0 + l1) / S);
#pragma unroll
      for (int a = 0; a < 3; a++) { o[a] = P.in.rays_o[3 * ray0 + a]; d[a] = P.in.rays_d[3 * ray0 + a]; }
      make_point(P.in.bound, P.in.coarse_bound, o, d, X.z[r0], Gr);
      pf0[0] = Gr.pf[0]; pf0[1] = Gr.pf[1]; pf0[2] = Gr.pf[2];
#pragma unroll
      for (int a = 0; a < 3; a++) { o[a] = P.in.rays_o[3 * ray1 + a]; d[a] = P.in.rays_d[3 * ray1 + a]; }
      make_point(P.in.bound, P.in.coarse_bound, o, d, X.z[r0 + 8], Gr);
      pf1[0] = Gr.pf[0]; pf1[1] = Gr.pf[1]; pf1[2] = Gr.pf[2];
    }
    for (int c = 0; c < 3; c++) {
      ld_frag(d2_frag(c), fa);
#pragma unroll
      for (int e = 0; e < 16; e++) {
        const int f = 32 * c + 8 * (e >> 2) + 2 * q + (e & 1);
        float dx = 0.0f;
        if (f < kEmb) {
          const float* pf = (e & 2) ? pf1 : pf0;
          float* dpe = (e & 2) ? dpe1 : dpe0;
          const float b0 = B[f], b1 = B[kEmbPad + f], b2 = B[2 * kEmbPad + f];
          float x = pf[0] * b0; x = fmaf(pf[1], b1, x); x = fmaf(pf[2], b2, x);
          dx = __cosf(reduce_2pi(x)) * fa[e];
          dpe[0] = fmaf(b0, dx, dpe[0]); dpe[1] = fmaf(b1, dx, dpe[1]); dpe[2] = fmaf(b2, dx, dpe[2]);
        }
        if constexpr (kWg) put_kt1(w->du, kWgALo, f - 32 * c, r0 + 8 * ((e >> 1) & 1), dx);
      }
      if constexpr (kWg) {                                       // dB[a][f] = sum_p p_a cos(.) dE_f  (embedder._B is a parameter of the decoder)
        const int nf = kEmb - 32 * c < 32 ? kEmb - 32 * c : 32;
        wg_group(*w, 0, w->dpk + Dec<3>::o_B + 32 * c, kEmbPad, nf, true);
      }
    }
  }
  // per-row sums over the four lanes of a row
#pragma unroll
  for (int a = 0; a < 3; a++) {
    dpe0[a] += __shfl_xor_sync(0xffffffffu, dpe0[a], 1); dpe1[a] += __shfl_xor_sync(0xffffffffu, dpe1[a], 1);
    dpe0[a] += __shfl_xor_sync(0xffffffffu, dpe0[a], 2); dpe1[a] += __shfl_xor_sync(0xffffffffu, dpe1[a], 2);
  }
  if (q == 0) *reinterpret_cast<float4*>(t.a[1] + bwd_dpe_off(r0)) = make_float4(dpe0[0], dpe0[1], dpe0[2], 0.0f);
  if (q == 1) *reinterpret_cast<float4*>(t.a[1] + bwd_dpe_off(r0 + 8)) = make_float4(dpe1[0], dpe1[1], dpe1[2], 0.0f);
  NSB_PH(27);
}

// Backward of gather_tile (same warp -> rows mapping).  dcs = [128][32] fp32.  emit(row, gx) once per point.
// kStore (deterministic mode, dgrid NULL): rows < npts of dcs and their coordinates also go to dc_out [rows][32] / xn_out [rows][3], if non-NULL.
template <bool kStore = false, typename F>
__device__ __forceinline__ void scatter_tile(const nsb_grid& g, float* __restrict__ dgrid, const int32_t* __restrict__ slots,
                                             const float* dcs, const float xn[3], int warp, int lane, F&& emit,
                                             float* dc_out = nullptr, float* xn_out = nullptr, int npts = 0) {
  const int q = lane & 7, qd = warp & 3, it0 = (warp >> 2) * 4;
#pragma unroll 1
  for (int it = it0; it < it0 + 4; it++) {
    const int src_lane = it * 4 + (lane >> 3);
    const int row = qd * 32 + src_lane;
    float x[3];
    x[0] = __shfl_sync(0xffffffffu, xn[0], src_lane); x[1] = __shfl_sync(0xffffffffu, xn[1], src_lane); x[2] = __shfl_sync(0xffffffffu, xn[2], src_lane);
    const float4 d4 = *reinterpret_cast<const float4*>(dcs + row * 32 + 4 * q);
    const float dc[4] = {d4.x, d4.y, d4.z, d4.w};
    if constexpr (kStore) {
      if (dc_out != nullptr && row < npts) {
        __stcg(reinterpret_cast<float4*>(dc_out + row * 32 + 4 * q), d4);
        if (q < 3) xn_out[3 * row + q] = x[q];
      }
    }
    float gx[3];
    scatter_pass(g, dgrid, slots, x, dc, q, gx);
    if (q == 0) emit(row, gx);
  }
}

// ---- block -> item -----------------------------------------------------------------------------------------------------------------
// Block b of a launch of tiles x split items runs item (tile, my): decoder-major (P.kind_major, item_order in nsb_render.cu) b = my * tiles +
// tile, so the decoders come in their evaluation order, the fine decoder -- the slowest item: two grids, eight fc_c units -- first;
// tile-major b = tile * split + my.  split == 1: block = tile either way.  Results do not depend on the order: the forward composites from
// the per-decoder parts in decoder order, the backward adds the ray parts in (tile, decoder) order.  kShared = false: kernels of one CTA per
// SM, which share no SM and so run tile-major (item_order never picks decoder-major for them).
struct Item { int tile, my; };
template <bool kShared = true>
__device__ __forceinline__ Item item_of_block(const KParams& P, int b) {
  if constexpr (!kShared) {
    const int tile = b / P.split;
    return {tile, b - tile * P.split};
  }
  const int d = P.kind_major ? (int)gridDim.x / P.split : P.split;
  const int q = b / d, r = b - q * d;
  return P.kind_major ? Item{r, q} : Item{q, r};
}

// Optional item timing (make ../libnsb_items.so, tools/item_timing.py): thread 0 of every tile CTA records its SM, its item and the global
// timer at start, at the end of its decoder chain and at exit, per launch kind (0 forward, 1 backward, 2 weight-gradient backward); read
// back with nsb_debug_items().  Compiled out of the product library.
#ifdef NSB_ITEM_TIMING
constexpr int kItemRecords = 16384;
struct ItemRecord { int sm, tile, my, level; unsigned long long t[3]; };
__device__ ItemRecord g_items[3][kItemRecords];
__device__ __forceinline__ void item_mark(int launch, int k, const KParams& P, const Item& it) {
  if (threadIdx.x != 0 || blockIdx.x >= kItemRecords) return;
  ItemRecord& r = g_items[launch][blockIdx.x];
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t) :: "memory");
  r.t[k] = t;
  if (k == 0) {
    int sm; asm volatile("mov.u32 %0, %%smid;" : "=r"(sm));
    r.sm = sm; r.tile = it.tile; r.my = it.my; r.level = P.split > 1 ? P.dec[it.my] : -1;
  }
}
#define NSB_ITEM_MARK(launch, k, P, it) ::nsb::tl::item_mark(launch, k, P, it)
#else
#define NSB_ITEM_MARK(launch, k, P, it) do { } while (0)
#endif

// ---- tile <-> ray bookkeeping ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int tiles_of_ray(int ray, int S) {
  const long long p0 = (long long)ray * S;
  return (int)((p0 + S - 1) / TM - p0 / TM) + 1;
}
// Bump the completion counters of the rays [ray_lo, ray_lo + nr) this item touched; returns (CTA-uniform) how many of them this CTA
// completed, their indices in s_done[].  Every thread must call it, after its global writes.  target = items per tile (split).
__device__ __forceinline__ int complete_rays(int* ray_cnt, int ray_lo, int nr, int S, int per_tile, int* s_done, int* s_ndone) {
  __threadfence();
  if (threadIdx.x == 0) *s_ndone = 0;
  __syncthreads();
  if ((int)threadIdx.x < nr) {
    const int ray = ray_lo + threadIdx.x;
    const int target = tiles_of_ray(ray, S) * per_tile;
    const int old = atomicAdd(ray_cnt + ray, 1);
    if (old == target - 1) { ray_cnt[ray] = 0; s_done[atomicAdd(s_ndone, 1)] = ray; }
  }
  __syncthreads();
  const int nd = *s_ndone;
  if (nd > 0) __threadfence();
  return nd;
}

// raw2outputs_nerf_color of one completed ray by one warp (common.py:204-245 incl. the out-of-bound override of Renderer.py:57).
// scratch: per-warp shared memory, composite_scratch_bytes(S) bytes, 16-byte aligned: raw [S] float4 | z [S] f64 | w [S] f32.
__host__ __device__ inline size_t composite_scratch_bytes(int S) { return ((size_t)28 * S + 15) & ~size_t(15); }
__device__ __forceinline__ void composite_ray(const KParams& P, int ray, int lane, unsigned char* scratch) {
  const int S = P.S;
  float* rw = reinterpret_cast<float*>(scratch);
  double* zz = reinterpret_cast<double*>(rw + 4 * S);
  float* wq = reinterpret_cast<float*>(zz + S);
  float o[3], d[3];
#pragma unroll
  for (int a = 0; a < 3; a++) { o[a] = P.in.rays_o[3 * ray + a]; d[a] = P.in.rays_d[3 * ray + a]; }
  const long long g0 = (long long)ray * S, NS = (long long)P.in.n_rays * S;
  for (int s = lane; s < S; s += 32) {
    // (all loads of the sample first: with a run-time trip count they were issued one L2 round trip after the other)
    float4 pq[3];
#pragma unroll
    for (int q = 0; q < 3; q++) pq[q] = q < P.split ? __ldcg(P.tile_parts + q * NS + g0 + s) : make_float4(0.f, 0.f, 0.f, 0.f);
    const double z = __ldcg(P.fo.z_vals + g0 + s);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int q = 0; q < 3; q++) { v.x += pq[q].x; v.y += pq[q].y; v.z += pq[q].z; v.w += pq[q].w; }       // decoder order: occ = fine + middle, rgb = colour decoder (zeros elsewhere)
    PointGeom G; make_point(P.in.bound, P.in.coarse_bound, o, d, z, G);
    if (!G.inb) v.w = 100.0f;
    zz[s] = z;
    *reinterpret_cast<float4*>(rw + 4 * s) = v;
    *reinterpret_cast<float4*>(P.fo.raw + 4 * (g0 + s)) = v;
  }
  __syncwarp();
  composite_ray_outputs(P, ray, rw, zz, wq, lane);
  __syncwarp();
}

}  // namespace tl

// ================================================================================================================================
// forward kernel
// ================================================================================================================================
template <bool H16, bool kSampled = false, bool kMesh = false>
__device__ __forceinline__ void render_fwd_tile_body(const KParams& P, const MeshPoints* M = nullptr) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  using namespace tl;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int row = tid & (TM - 1), cg = tid >> 7;            // (control warp: row/cg unused)
  TileSmem t; carve(smem_raw, t, false);
  __shared__ int s_ndone, s_done[kMaxTileRays];
  __shared__ float s_max[16];
  __shared__ uint32_t s_seq;

  const bool points = kMesh || P.points != nullptr;
  const int nsplit = P.split;
  const Item item = item_of_block(P, blockIdx.x);
  const int tile = item.tile, my = item.my;
  NSB_ITEM_MARK(0, 0, P, item);
  const int q0 = nsplit > 1 ? my : 0, q1 = nsplit > 1 ? my + 1 : P.n_dec;
  const long long NP = points ? (long long)P.n_points : (long long)P.in.n_rays * P.S;
  const long long gp0 = (long long)tile * TM;
  const int npts = (int)(NP - gp0 < TM ? NP - gp0 : TM);
  const int S = P.S;
  int ray_lo = 0, nr = 0;
  if (!points) { ray_lo = (int)(gp0 / S); nr = (int)((gp0 + npts - 1) / S) - ray_lo + 1; }

  if (threadIdx.x == 0) *t.tmem = tc::acc_acquire();             // this CTA's accumulator slot (visible after the next barrier)
  NSB_PH_RESET();
  Issuer I; I.L.P = &P; I.L.q = q0; I.L.q1 = q1; I.L.k = 0; I.L.loaded = 0; I.L.mode = H16 ? 2 : 0; I.issued = 0; I.g = 0;
  if (tid == 0) {
    // A_ready: one arrival per warp; empty / done: one per warpgroup (release_units)
    for (int i = 0; i < kNumBars; i++)
      mbar_init(t.bars + i, (i == B_AREADY || i == B_AREADY + 1) ? kEpiThreads / 32 : ((i >= B_EMPTY && i < B_EMPTY + kSlots) || i >= B_DONE) ? 2 : 1);
    mbar_fence_init();
    load_header(P, t, P.dec[q0], 0);
    for (int i = 0; i < kSlots; i++) loader_issue(I.L, t);      // (every decoder has >= 6 units)
  }

  // ---- prologue: this tile's rays -> sorted sample depths -> this row's point
  PointGeom G;
  const int lp = row < npts ? row : npts - 1;
  if (points) {
    const long long gp = gp0 + lp;
    if constexpr (kMesh) {
      mesh_point_geom(P, *M, gp, G);
    } else {
      const double pin[3] = {P.points[3 * gp], P.points[3 * gp + 1], P.points[3 * gp + 2]};
      make_point_from_p(P.in.bound, P.in.coarse_bound, pin, G);
    }
    __syncthreads();
  } else {
    float gtmax, gtmax12;
    batch_depth_max(P, s_max, &s_seq, gtmax, gtmax12);
    NSB_PH(40);
    // scratch in the (still unused) operand buffers: ray table [nr][8] f32 + far [nr] f64 | unsorted z [nr*S] | sorted z [nr*S] | flags [nr]
    float* rays = t.a[0];
    double* far = reinterpret_cast<double*>(t.a[0] + 8 * kMaxTileRays);
    double* zu = far + kMaxTileRays;
    double* zs = zu + (size_t)nr * S;
    block_setup_rays(P, rays, far, ray_lo, nr, gtmax12);
    __syncthreads();
    NSB_PH(41);
    block_sample_sort<kSampled>(P, rays, far, ray_lo, nr, gtmax, zu, zs, reinterpret_cast<int*>(zs + (size_t)nr * S));
    __syncthreads();
    NSB_PH(43);
    {
      const long long gp = gp0 + lp;
      const int r = (int)(gp / S) - ray_lo, s = (int)(gp - (long long)(ray_lo + r) * S);
      const double z = zs[r * S + s];
      const float o[3] = {rays[8 * r], rays[8 * r + 1], rays[8 * r + 2]}, dd[3] = {rays[8 * r + 3], rays[8 * r + 4], rays[8 * r + 5]};
      make_point(P.in.bound, P.in.coarse_bound, o, dd, z, G);
      if (cg == 0 && row < npts && my == 0) P.fo.z_vals[gp] = z;
    }
    __syncthreads();                                              // the scratch is dead: the operand buffers may be written
  }
  __syncthreads();                                                // accumulator slot + barrier initialisation visible
  const uint32_t acc_slot = *t.tmem;                              // (the slot holds the fc_c fragments, d2_frag)
  NSB_PH(44);

  float occ = 0.0f, c0 = 0.0f, c1 = 0.0f, c2 = 0.0f;
  {
    uint32_t n = 0;
    for (int qd = q0; qd < q1; qd++) {
      const int lv = P.dec[qd];
      float out[4];
      uint32_t* gm = P.fo.masks != nullptr ? P.fo.masks + (gp0 * 15 + qd * 5) : nullptr;
      const int dq = qd - q0;
      if (tid == 0 && qd + 1 < q1) load_header(P, t, P.dec[qd + 1], (dq + 1) & 1);      // (decoder qd-1 ended with CTA barriers: its buffer is free)
      const int as = acts_slot(P.acts_mask, lv);
      float* acts = (P.fo.acts != nullptr && as >= 0) ? P.fo.acts + (as * NP + gp0) * 5 * 32 : nullptr;
      epi_forward<H16>(P, t, I, lv, G, n, dq & 1, (dq >> 1) & 1u, out, gm, acts, npts);
      if (lv == 3) { c0 = out[0]; c1 = out[1]; c2 = out[2]; } else occ += out[0];
      if (qd == 0 && cg == 0 && row < npts && P.fo.corner_idx != nullptr) {
        const nsb_grid& g = P.in.grid[lv];
        const Tri tr = make_tri(lv == 0 ? G.xnc : G.xn, g.W, g.H, g.D);
        const long long gp = gp0 + row;
        P.fo.corner_idx[3 * gp] = tr.i0[0]; P.fo.corner_idx[3 * gp + 1] = tr.i0[1]; P.fo.corner_idx[3 * gp + 2] = tr.i0[2];
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) tc::acc_release(acc_slot);
  // the decoder chain of this item is done: a backward launched as a programmatic dependent may take the slots that free up from here on and
  // set up under the ray compositing / loss-seed tail (triggering at kernel start made the early backward CTAs compete with the chain: slower)
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  NSB_PH(14);
  NSB_ITEM_MARK(0, 1, P, item);

  if (points) {                                                   // Renderer.eval_points: raw with the out-of-bound override
    if (cg == 0 && row < npts) {
      if (kMesh && M->z != nullptr) M->z[gp0 + row] = G.inb ? occ : 100.0f;
      else *reinterpret_cast<float4*>(P.points_raw + 4 * (gp0 + row)) = make_float4(c0, c1, c2, G.inb ? occ : 100.0f);
    }
    return;
  }
  if (cg == 0 && row < npts) P.tile_parts[(long long)my * NP + gp0 + row] = make_float4(c0, c1, c2, occ);
  const int nd = complete_rays(P.ray_cnt, ray_lo, nr, S, nsplit, s_done, &s_ndone);
  NSB_PH(15);
  for (int k = warp; k < nd; k += kThreads / 32) composite_ray(P, s_done[k], lane, smem_raw + (size_t)warp * composite_scratch_bytes(S));
  NSB_PH(16);
  fused_seeds_tail(P, gridDim.x, smem_raw);                       // the last CTA of the grid to get here sees every ray composited
  NSB_ITEM_MARK(0, 2, P, item);
}
__global__ void __launch_bounds__(tl::kThreads, 2) render_fwd_tile_kernel(const __grid_constant__ KParams P) { render_fwd_tile_body<false>(P); }
// forward with FP16 hi|lo operands (option fwd_f16; see mma_rows)
__global__ void __launch_bounds__(tl::kThreads, 2) render_fwd_tile_h16_kernel(const __grid_constant__ KParams P) { render_fwd_tile_body<true>(P); }
// lindisp / perturb / a given sample list (KParams::smp, nsb_render_forward_sampled)
__global__ void __launch_bounds__(tl::kThreads, 2) render_fwd_tile_sampled_kernel(const __grid_constant__ KParams P) { render_fwd_tile_body<false, true>(P); }
// mesh extraction's points (MeshPoints): the 3xTF32 forward
__global__ void __launch_bounds__(tl::kThreads, 2) render_fwd_tile_mesh_kernel(const __grid_constant__ KParams P, const __grid_constant__ MeshPoints M) {
  render_fwd_tile_body<false, false, true>(P, &M);
}

// ================================================================================================================================
// backward kernel (input gradients: rays + grid voxels)
// ================================================================================================================================
// WG != kWgNone: the item's decoder also gets its WEIGHT gradients (tensor-core contraction over the tile's points, see the "tensor-core weight
// gradients" helpers; kWgXyz: the middle, fine and colour decoders, kWgCoarse: the coarse decoder): 96 KB more shared memory in front of the
// common part -> one CTA per SM.
// kDet: the deterministic-mode instantiation (DetParams D): dL/dc rows and coordinates go to D->dc / D->xn instead of the voxel scatter (which
// still yields the coordinate gradients), weight gradients to this tile's partial image in D->wpart.
template <int WG, bool kDet = false>
__device__ __forceinline__ void render_bwd_tile_body(const KParams& P, const DetParams* D = nullptr) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  using namespace tl;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int row = tid & (TM - 1), cg = tid >> 7;
  // (WG: the MN-major tiles need the 1024-byte alignment of their swizzle pattern: aligned by hand, 1 KB of slack in the launch size)
  unsigned char* sbase = WG ? smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u) : smem_raw;
  TileSmem t; carve(sbase + (WG ? kWgBytes : 0), t, true);
  BwdExtra& X = *reinterpret_cast<BwdExtra*>(t.extra);
  __shared__ int s_ndone, s_done[kMaxTileRays];
  WgSmem wg;
  wg.du = reinterpret_cast<float*>(sbase); wg.g = wg.du + kMnTile; wg.b = wg.du + 4 * kMnTile;
  wg.dpk = nullptr;

  const int nsplit = P.split;
  const Item item = item_of_block<WG == kWgNone>(P, blockIdx.x);
  const int tile = item.tile, my = item.my;
  NSB_ITEM_MARK(WG ? 2 : 1, 0, P, item);
  const int q0 = nsplit > 1 ? my : 0, q1 = nsplit > 1 ? my + 1 : P.n_dec;
  const int S = P.S;
  const long long NP = (long long)P.in.n_rays * S;
  const long long gp0 = (long long)tile * TM;
  const int npts = (int)(NP - gp0 < TM ? NP - gp0 : TM);
  const int ray_lo = (int)(gp0 / S), nr = (int)((gp0 + npts - 1) / S) - ray_lo + 1;

  if (threadIdx.x == 0) *t.tmem = tc::acc_acquire();             // this CTA's accumulator slot (visible after the next barrier)
  NSB_PH_RESET();
  Issuer I; I.L.P = &P; I.L.q = q0; I.L.q1 = q1; I.L.k = 0; I.L.loaded = 0; I.L.mode = 1; I.issued = 0; I.g = 0;
  if (tid == 0) {
    // empty: one arrival per warpgroup (release_units); A_ready / done are not used by the backward
    for (int i = 0; i < kNumBars; i++) mbar_init(t.bars + i, (i >= B_EMPTY && i < B_EMPTY + kSlots) ? 2 : 1);
    mbar_fence_init();
    load_header(P, t, P.dec[q0], 0);
    for (int i = 0; i < kSlots; i++) loader_issue(I.L, t);
  }

  for (int i = tid; i < TM * 3; i += kThreads) X.dp[i] = 0.0;
  // Launched as a programmatic dependent of the forward (nsb_render.cu): everything above ran under the forward's tail; nothing the forward
  // produces (raw, z_vals, ReLU bits, loss seeds, completion counters) is touched before the forward grid has completed.  (No-op otherwise.)
  asm volatile("griddepcontrol.wait;" ::: "memory");
  // ---- prologue: per ray of this tile, compositing weights and dL/d(occupancy logit) (SURVEY.md 8.1); scratch in the operand buffers
  for (int r = warp; r < nr; r += kThreads / 32) {
    const int ray = ray_lo + r;
    float* rw = t.a[0] + (size_t)warp * ((6 * S + 3) & ~3);       // per warp (16-byte aligned): raw [4S] | w [S] | go [S]
    float* wq = rw + 4 * S; float* go = wq + S;
    const long long g0 = (long long)ray * S;
    float o[3], d[3];
#pragma unroll
    for (int a = 0; a < 3; a++) { o[a] = P.in.rays_o[3 * ray + a]; d[a] = P.in.rays_d[3 * ray + a]; }
    for (int s = lane; s < S; s += 32) *reinterpret_cast<float4*>(rw + 4 * s) = *reinterpret_cast<const float4*>(P.bw.raw + 4 * (g0 + s));
    __syncwarp();
    float g3[3] = {0.f, 0.f, 0.f};
    if (P.bw.g_rgb != nullptr) { g3[0] = P.bw.g_rgb[3 * ray]; g3[1] = P.bw.g_rgb[3 * ray + 1]; g3[2] = P.bw.g_rgb[3 * ray + 2]; }
    if (lane == 0) { X.gc[3 * r] = g3[0]; X.gc[3 * r + 1] = g3[1]; X.gc[3 * r + 2] = g3[2]; }
    const double* z = P.bw.z_vals + g0;
    composite_ray_backward(rw, z, S, P.bw.g_depth != nullptr ? P.bw.g_depth[ray] : 0.0, P.bw.g_var != nullptr ? P.bw.g_var[ray] : 0.0, g3,
                           wq, go, lane, [&](int s, float w, float al, float ga) {
      const long long gp = g0 + s;
      if (gp >= gp0 && gp < gp0 + npts) {                          // only the samples of this tile are needed
        PointGeom Gs; make_point(P.in.bound, P.in.coarse_bound, o, d, z[s], Gs);
        X.gocc[gp - gp0] = Gs.inb ? 10.0f * al * (1.0f - al) * ga : 0.0f;
        X.wgt[gp - gp0] = w;
      }
    });
  }
  NSB_PH(20);
  PointGeom G;
  const int lp = row < npts ? row : npts - 1;
  const long long gpr = gp0 + lp;
  const int rayr = (int)(gpr / S);
  {
    float o[3], d[3];
#pragma unroll
    for (int a = 0; a < 3; a++) { o[a] = P.in.rays_o[3 * rayr + a]; d[a] = P.in.rays_d[3 * rayr + a]; }
    const double z = P.bw.z_vals[gpr];
    make_point(P.in.bound, P.in.coarse_bound, o, d, z, G);
    if (cg == 0) X.z[row] = z;
  }
  __syncthreads();                                                // prologue scratch dead, gocc / wgt / gc visible, accumulator slot + barriers visible
  const uint32_t acc_slot = *t.tmem;                              // (the slot holds the DF fragments between layers 3 and 0, d2_frag)
  NSB_PH(21);

  {
    const int off0 = (int)(gp0 - (long long)ray_lo * S);
    for (int qd = q0; qd < q1; qd++) {
      const int lv = P.dec[qd];
      const uint32_t* gm = P.bw.masks + (gp0 * 15 + P.dec_pos[qd] * 5);
      const int dq = qd - q0;
      if (tid == 0 && qd + 1 < q1) load_header(P, t, P.dec[qd + 1], (dq + 1) & 1);      // (the previous decoder ended with CTA barriers: its buffer is free)
      if constexpr (kDet) { if (WG) wg.dpk = D->wpart[lv] + (size_t)tile * packed_floats(lv); }
      else if (WG) wg.dpk = P.d_packed[lv];
      const float* acts_row = (WG && row < npts) ? P.bw.acts + ((acts_slot(P.acts_mask, lv) * NP + gp0 + row) * 5) * 32 + kCW * cg : nullptr;
      epi_backward<WG, kDet>(P, t, I, X, lv, G, dq & 1, (dq >> 1) & 1u, gm, npts, off0, gp0, WG ? &wg : nullptr, acts_row);
      epi_sync();                                                 // dL/dc rows + embedding partials visible
      const double* bb = lv == 0 ? P.in.coarse_bound : P.in.bound;
      const double sc[3] = {2.0 / (bb[1] - bb[0]), 2.0 / (bb[3] - bb[2]), 2.0 / (bb[5] - bb[4])};      // d(normalised)/dp, common.py:280-282
      const float* xn = lv == 0 ? G.xnc : G.xn;
      // (kDet: this tile's rows of dL/dc and coordinates go to D for nsb_det.cu's ordered sum instead of the voxel scatter)
      float* const dc_out = kDet && D->dc[lv] != nullptr ? D->dc[lv] + gp0 * 32 : nullptr;
      float* const xn_out = kDet && D->dc[lv] != nullptr ? D->xn[lv] + gp0 * 3 : nullptr;
      scatter_tile<kDet>(P.in.grid[lv], kDet ? nullptr : P.bw.d_grid[lv], P.bw.slot_map[lv], t.a[0], xn, warp, lane, [&](int prow, const float gx[3]) {
        if (prow < npts) {
          const float4 p = *reinterpret_cast<const float4*>(t.a[1] + bwd_dpe_off(prow));
          const float dpe[3] = {p.x, p.y, p.z};
#pragma unroll
          for (int a = 0; a < 3; a++) X.dp[3 * prow + a] += (double)dpe[a] + (double)gx[a] * sc[a];
        }
      }, dc_out, xn_out, npts);
      epi_sync();                                                 // reads of a[0] / a[1] done before the next decoder overwrites them
      NSB_PH(29);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) tc::acc_release(acc_slot);
  NSB_ITEM_MARK(WG ? 2 : 1, 1, P, item);

  // per-ray sums of this item: d rays_o = sum_s dp, d rays_d = sum_s z_s dp (pts = o + d z, Renderer.py:172-174) -> global scratch
  const int RT = P.tile_rays;                                     // rays a tile can touch: stride of the per-item parts
  double* parts = P.ray_parts + ((long long)tile * nsplit + my) * RT * 6;
  for (int i = tid; i < nr * 3; i += kThreads) {
    const int r = i / 3, a = i - 3 * r;
    const long long g0 = (long long)(ray_lo + r) * S;
    const int s0 = (int)(g0 > gp0 ? g0 - gp0 : 0), s1 = (int)(g0 + S - gp0 < npts ? g0 + S - gp0 : npts);
    double so = 0.0, sd = 0.0;
    for (int p = s0; p < s1; p++) { const double v = X.dp[3 * p + a]; so += v; sd += v * X.z[p]; }
    parts[r * 6 + a] = so; parts[r * 6 + 3 + a] = sd;
  }
  NSB_PH(30);
  const int nd = complete_rays(P.ray_cnt, ray_lo, nr, S, nsplit, s_done, &s_ndone);
  NSB_PH(31);
  for (int i = tid; i < nd * 3; i += kThreads) {                  // the completing CTA adds the parts in (tile, decoder) order
    const int ray = s_done[i / 3], a = i % 3;
    const long long p0 = (long long)ray * S;
    const int t0 = (int)(p0 / TM), t1 = (int)((p0 + S - 1) / TM);
    double so = 0.0, sd = 0.0;
    for (int tt = t0; tt <= t1; tt++) {
      const int rl = (int)(((long long)tt * TM) / S);
      for (int q = 0; q < nsplit; q++) {
        const double* pp = P.ray_parts + (((long long)tt * nsplit + q) * RT + (ray - rl)) * 6;
        so += __ldcg(pp + a); sd += __ldcg(pp + 3 + a);
      }
    }
    store_ray_grad(P, ray, a, so, sd);
  }
  NSB_PH(32);
  if (fused_pose_grad(P, gridDim.x, reinterpret_cast<double*>(smem_raw))) pose_tail_peers(P);
  NSB_ITEM_MARK(WG ? 2 : 1, 2, P, item);
}
__global__ void __launch_bounds__(tl::kThreads, 2) render_bwd_tile_kernel(const __grid_constant__ KParams P) { render_bwd_tile_body<tl::kWgNone>(P); }
__global__ void __launch_bounds__(tl::kThreads, 1) render_bwd_wg_tile_kernel(const __grid_constant__ KParams P) { render_bwd_tile_body<tl::kWgXyz>(P); }
// the coarse decoder's weight gradients (stage coarse, option wgrad_all)
__global__ void __launch_bounds__(tl::kThreads, 1) render_bwd_wg_coarse_tile_kernel(const __grid_constant__ KParams P) {
  render_bwd_tile_body<tl::kWgCoarse>(P);
}
// the deterministic-mode instantiations of the three (option "deterministic", DetParams)
__global__ void __launch_bounds__(tl::kThreads, 2) render_bwd_tile_det_kernel(const __grid_constant__ KParams P, const __grid_constant__ DetParams D) {
  render_bwd_tile_body<tl::kWgNone, true>(P, &D);
}
__global__ void __launch_bounds__(tl::kThreads, 1) render_bwd_wg_tile_det_kernel(const __grid_constant__ KParams P, const __grid_constant__ DetParams D) {
  render_bwd_tile_body<tl::kWgXyz, true>(P, &D);
}
__global__ void __launch_bounds__(tl::kThreads, 1) render_bwd_wg_coarse_tile_det_kernel(const __grid_constant__ KParams P,
                                                                                        const __grid_constant__ DetParams D) {
  render_bwd_tile_body<tl::kWgCoarse, true>(P, &D);
}

}  // namespace nsb
