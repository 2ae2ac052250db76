// wgmma / mbarrier / bulk-copy PTX wrappers and the operand-format helpers of the tensor-core path (sm_90a).
//
// Numerics: every contraction is accumulated in fp32 registers by wgmma, in one of three operand formats (TcFormat):
//   3xTF32 (tf32 operands, 4 B/operand element, 8-bit exponent: range-robust), or
//   3xFP16 (f16 operands,  2 B/operand element: half the shared-memory operand traffic and twice the MMA rate; operands are
//           pre-scaled by powers of two so residuals stay in fp16's normal range; |x| > 65504 -> inf -> NaN flag of the output),
//   1xFP16 (the single product a_hi.b_hi of the 3xFP16 operands: a third of the wgmmas, no residual tile and no low weight
//           image; fp16-grade accuracy, 2^-11 relative per operand; same range limit as 3xFP16).
// 3xTF32:
//     a = a_hi + a_lo,  a_hi = cvt.rna.tf32(a),  a_lo = a - a_hi   (exact; the MMA truncates a_lo to 11 bits: 2^-23 |a|)
//     a.b ~= a_lo.b_hi + a_hi.b_lo + a_hi.b_hi                       (dropped a_lo.b_lo ~ 2^-24 |a||b|)
// which keeps fp32-grade accuracy (the parity tolerance is atol 1e-5 / rtol 1e-4; plain TF32 would be ~1e-3).
//
// Operand layout (both operands K-major, SWIZZLE_128B): a tile of R rows x 128 bytes of k-values; 8-row groups are
// 1024 B apart (SBO); inside a row the 16-byte chunk c sits at position c ^ (row & 7).  One wgmma consumes 32 bytes of
// every row (K=8 tf32 or K=16 fp16); stepping K inside the swizzled row = advancing the descriptor start address by 32 bytes.
#pragma once
#include <cuda_fp16.h>

#include "dsb_internal.cuh"
#include "dsb_wgmma.cuh"

namespace dsb {
namespace tc {

constexpr int TM = 128;            // rows (edges / nodes) per tile: two warpgroups of 64 rows
constexpr int WG_ROWS = 64;        // rows per warpgroup = M of one wgmma
constexpr int TKC = 32;            // k-values per 128-byte swizzle row with 4-byte (TF32) operands
constexpr int TKC16 = 64;          // ... with 2-byte (FP16) operands
constexpr float X_SCALE = 1.0f;    // 3xFP16 activation scale (1: |x| < 0.25 has a subnormal fp16 residual, abs. error <= 3e-8)
constexpr int A_CHUNK_BYTES = TM * 128;        // 16 KB
constexpr int NSTAGE = 2;
constexpr int MMA_THREADS = 256;   // two warpgroups: each builds the A operand of its 64 rows, issues its wgmmas and runs the epilogue
constexpr int TC_THREADS = MMA_THREADS + 128;  // + a third warpgroup whose lane 0 streams the weight chunks (keeps the MMA
                                               //   warpgroups free of single-thread branches while their wgmmas are in flight)
// register split (setmaxnreg): the weight warpgroup gives its registers to the two MMA warpgroups, which hold H/2
// accumulators per thread: 128 x 40 + 256 x 232 <= 64 K registers
constexpr int WEIGHT_WG_REGS = 40, MMA_WG_REGS = 232;
template <int R> __device__ __forceinline__ void regs_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void regs_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// Geometry that depends on the width H = hidden_nf of the network (128, 192 or 256): the accumulator tile is TM x H, a weight
// chunk image is H rows x 128 B.
template <int H>
struct Geo {
  static_assert(H == 128 || H == 192 || H == 256, "tensor-core kernels are built for hidden_nf 128, 192, 256");
  static constexpr int TN = H;                                  // accumulator columns per tile = N of one wgmma
  static constexpr int ACC = H / 2;                             // fp32 accumulator registers per thread
  static constexpr int B_CHUNK_BYTES = H * 128;                 // 16 / 24 / 32 KB
  static constexpr int B_CHUNK_FLOATS = H * TKC;                // 32-bit words per chunk image
  static constexpr int STAGE_BYTES = 2 * A_CHUNK_BYTES + 2 * B_CHUNK_BYTES;   // Xhi, Xlo, Whi, Wlo = 64 / 80 / 96 KB
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P1;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2, %3;\n\t"
      "selp.b32 %0, 1, 0, P1;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(20000u)
      : "memory");
  return ok != 0;
}
// Bounded spin: a protocol bug must trap (CUDA error) instead of hanging the GPU.  The trap is a predicated instruction,
// not a branch, and there is no printf (a call): either would put a divergent path between a wgmma and its wait, which
// makes ptxas serialise the wgmma pipeline.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    ++spins;
    asm volatile("{\n\t.reg .pred p;\n\tsetp.gt.u32 p, %0, %1;\n\t@p trap;\n\t}" ::"r"(spins), "r"(1u << 17));
  }
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// barrier over the 128 threads of warpgroup wg (ids 1, 2; 0 is __syncthreads)
__device__ __forceinline__ void wg_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(wg + 1) : "memory"); }

// ---- bulk copy global -> shared, completion on an mbarrier -------------------------------------------------------------
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// ---- wgmma ---------------------------------------------------------------------------------------------------------
// K-major SWIZZLE_128B shared-memory descriptor: start>>4 | LBO (unused for this layout, 1) <<16 | SBO (1024>>4) <<32 |
// layout SWIZZLE_128B (1) <<62.  Tiles start 1024-byte aligned, so the base offset field stays 0.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFFu) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous wgmma window
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// The 12 wgmmas of one K-chunk held in stage memory `st` (A_hi | A_lo | W_hi | W_lo) for the 64 rows of warpgroup wg:
// 4 k-steps x 3 split products into d (1xFP16: 4 k-steps x the A_hi.W_hi product); the first product of a tile's first
// chunk overwrites d.  first_chunk only sets the scale-d predicate of one instruction: no branch around the wgmmas (a
// divergent path between a wgmma and its wait makes ptxas serialise the pipeline).
template <TcFormat FMT, int H>
__device__ __forceinline__ void mma_chunk(float (&d)[H / 2], const char* st, int wg, bool first_chunk) {
  using G = Geo<H>;
  const uint32_t xhi = smem_u32(st) + (uint32_t)(wg * WG_ROWS * 128), xlo = xhi + A_CHUNK_BYTES;
  const uint32_t whi = smem_u32(st) + 2 * A_CHUNK_BYTES, wlo = whi + G::B_CHUNK_BYTES;
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {       // 4 k-steps of 32 bytes per 128-byte row (K=8 tf32 or K=16 fp16 each)
    const uint32_t ko = ks * 32;
    const uint32_t acc = (first_chunk && ks == 0) ? 0u : 1u;
    if constexpr (FMT == TcFormat::F16x1) {
      Wgmma<H>::f16(d, wgmma_desc_sw128(xhi + ko), wgmma_desc_sw128(whi + ko), acc);
    } else if constexpr (FMT == TcFormat::F16x3) {
      Wgmma<H>::f16(d, wgmma_desc_sw128(xlo + ko), wgmma_desc_sw128(whi + ko), acc);
      Wgmma<H>::f16(d, wgmma_desc_sw128(xhi + ko), wgmma_desc_sw128(wlo + ko), 1u);
      Wgmma<H>::f16(d, wgmma_desc_sw128(xhi + ko), wgmma_desc_sw128(whi + ko), 1u);
    } else {
      Wgmma<H>::tf32(d, wgmma_desc_sw128(xlo + ko), wgmma_desc_sw128(whi + ko), acc);
      Wgmma<H>::tf32(d, wgmma_desc_sw128(xhi + ko), wgmma_desc_sw128(wlo + ko), 1u);
      Wgmma<H>::tf32(d, wgmma_desc_sw128(xhi + ko), wgmma_desc_sw128(whi + ko), 1u);
    }
  }
}

// round-to-nearest (ties away) to the 19-bit TF32 container with two integer-pipe instructions
__device__ __forceinline__ float tf32_hi(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u); }

// byte offset of (row r, 16-byte chunk c) inside a [rows][128 B] SWIZZLE_128B tile
__device__ __host__ __forceinline__ uint32_t sw128_offset(int r, int c) {
  return (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((c ^ (r & 7)) << 4));
}

// Residual of the 3xFP16 split, x - float(hi), for a packed pair of fp16 hi parts (exact: the difference is
// representable in fp32).
__device__ __forceinline__ void residual_f16(uint32_t hi2, float x0, float x1, float& r0, float& r1) {
  const __half2 h = *reinterpret_cast<const __half2*>(&hi2);
  r0 = x0 - __low2float(h);
  r1 = x1 - __high2float(h);
}
__device__ __forceinline__ uint32_t h2_bits(__half2 h) { return *reinterpret_cast<const uint32_t*>(&h); }

// Producer-side store of 4 consecutive k-values of one tile row at `dst` (stage base + swizzled offset of the row piece):
//   TF32: 16-byte stores (hi tile, lo tile A_CHUNK_BYTES further)
//   FP16: 8-byte stores (1xFP16: the hi tile only, no residual)
// An FP16 activation beyond the fp16 range becomes inf here and reaches the output as NaN -> the NaN guard of the
// denoiser raises; 3xTF32 has no such limit.
template <TcFormat FMT>
__device__ __forceinline__ void store_pair(char* dst, f32x2 u01, f32x2 u23) {
  float x0, x1, x2, x3;
  upk2(u01, x0, x1); upk2(u23, x2, x3);
  if constexpr (FMT == TcFormat::F16x1) {
    uint2 hv;
    hv.x = h2_bits(__floats2half2_rn(x0, x1)); hv.y = h2_bits(__floats2half2_rn(x2, x3));
    *reinterpret_cast<uint2*>(dst) = hv;
  } else if constexpr (FMT == TcFormat::F16x3) {
    const __half2 h0 = __floats2half2_rn(x0, x1), h1 = __floats2half2_rn(x2, x3);
    float l0, l1, l2, l3;
    residual_f16(h2_bits(h0), x0, x1, l0, l1); residual_f16(h2_bits(h1), x2, x3, l2, l3);
    const __half2 q0 = __floats2half2_rn(l0, l1), q1 = __floats2half2_rn(l2, l3);
    uint2 hv, lv;
    hv.x = h2_bits(h0); hv.y = h2_bits(h1);
    lv.x = h2_bits(q0); lv.y = h2_bits(q1);
    *reinterpret_cast<uint2*>(dst) = hv;
    *reinterpret_cast<uint2*>(dst + A_CHUNK_BYTES) = lv;
  } else {
    const float4 h = make_float4(tf32_hi(x0), tf32_hi(x1), tf32_hi(x2), tf32_hi(x3));
    *reinterpret_cast<float4*>(dst) = h;
    *reinterpret_cast<float4*>(dst + A_CHUNK_BYTES) = make_float4(x0 - h.x, x1 - h.y, x2 - h.z, x3 - h.w);
  }
}
// byte offset of row r's piece p (4 k-values, p in 0..7) of 32-k half hf inside a stage's A tile
template <bool F16>
__device__ __forceinline__ uint32_t piece_offset(int r, int hf, int p) {
  return F16 ? sw128_offset(r, (hf & 1) * 4 + (p >> 1)) + (uint32_t)(p & 1) * 8u : sw128_offset(r, p);
}

// ---- weight pipeline --------------------------------------------------------------------------------------------------
// Stage s holds one K-chunk: A_hi | A_lo (built by the warpgroups, each its own 64 rows) | W_hi | W_lo (bulk copies);
// 1xFP16 leaves A_lo and W_lo unused.
// full_w[s]: the weight chunk has landed (1 arrive + tx bytes).  empty[s]: the wgmmas that read the stage have completed
// in all 8 warps of both warpgroups (one arrive per warp), so the next weight chunk may be copied in.
struct Control {
  uint64_t full_w[NSTAGE];
  uint64_t empty[NSTAGE];
};

__device__ __forceinline__ void control_init(Control* c) {
  for (int s = 0; s < NSTAGE; ++s) { mbar_init(&c->full_w[s], 1); mbar_init(&c->empty[s], 8); }
  fence_barrier_init();
}

// Sequence of K-chunks g = 0, 1, ... of a CTA (all tiles in order), issued by lane 0 of the weight warp: chunk g goes into
// stage g % 2 once chunk g - 2 (same stage) has been consumed by both warpgroups.
template <TcFormat FMT, int H>
struct WeightStream {
  Control* ctl;
  char* stages;
  __device__ void issue(uint32_t g, const float* hi, const float* lo) const {
    using G = Geo<H>;
    const int s = g & 1;
    if (g >= NSTAGE) mbar_wait(&ctl->empty[s], ((g >> 1) - 1) & 1);
    char* st = stages + (size_t)s * G::STAGE_BYTES + 2 * A_CHUNK_BYTES;
    if constexpr (FMT == TcFormat::F16x1) {       // W_hi only
      mbar_arrive_expect_tx(&ctl->full_w[s], G::B_CHUNK_BYTES);
      bulk_g2s(st, hi, G::B_CHUNK_BYTES, &ctl->full_w[s]);
    } else {
      mbar_arrive_expect_tx(&ctl->full_w[s], 2 * G::B_CHUNK_BYTES);
      bulk_g2s(st, hi, G::B_CHUNK_BYTES, &ctl->full_w[s]);
      bulk_g2s(st + G::B_CHUNK_BYTES, lo, G::B_CHUNK_BYTES, &ctl->full_w[s]);
    }
  }
};

// Per-warpgroup bookkeeping of the asynchronous wgmma groups: every chunk's stage is released (one arrive on empty) once
// its wgmmas are known to be complete (lane 0 of every warp arrives).  At most one group stays in flight while the next
// chunk's operand is built (in the edge kernels also across unit boundaries: the next unit's first chunk is built under
// the last chunk of the current one); the accumulators are read only after drain().
struct MmaTracker {
  int pend = -1;
  // after committing chunk g: wait for the previous chunk's group and release its stage
  __device__ __forceinline__ void release_prev(Control* ctl, int g, bool leader) {
    wgmma_wait<1>();
    if (leader && pend >= 0) mbar_arrive(&ctl->empty[pend & 1]);
    pend = g;
  }
  // wait for the last committed group, release its stage; the accumulators are final
  template <int H>
  __device__ __forceinline__ void drain(Control* ctl, float (&d)[H / 2], bool leader) {
    wgmma_wait<0>();
    acc_fence(d);
    if (leader && pend >= 0) mbar_arrive(&ctl->empty[pend & 1]);
    pend = -1;
  }
};

}  // namespace tc
}  // namespace dsb
