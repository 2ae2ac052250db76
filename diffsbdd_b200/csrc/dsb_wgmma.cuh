// wgmma.mma_async wrappers (sm_90a) for the accumulator widths of the tensor-core kernels: one warpgroup, M = 64,
// N = hidden_nf, both operands K-major in shared memory (descriptors), fp32 accumulators in registers:
// D (+)= A . B^T, accumulate == 0 overwrites D.
// Layout of d[] per thread t of the warpgroup: d[4j + 2h + b] = D[16 (t / 32) + (t % 32) / 4 + 8h][8j + 2 (t % 4) + b].
#pragma once
#include <stdint.h>

// operand lists: "%a0, ..., %a9, " (a = leading decimal digits) and eight accumulator registers from d[i]
#define DSB_P10(a) "%" #a "0, %" #a "1, %" #a "2, %" #a "3, %" #a "4, %" #a "5, %" #a "6, %" #a "7, %" #a "8, %" #a "9, "
#define DSB_O8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), \
                  "+f"(d[i + 6]), "+f"(d[i + 7])

namespace dsb {
namespace tc {

template <int N> struct Wgmma;

template <> struct Wgmma<128> {
  static __device__ __forceinline__ void f16(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {" DSB_P10() DSB_P10(1) DSB_P10(2) DSB_P10(3) DSB_P10(4) DSB_P10(5) "%60, %61, %62, %63"
                 "}, %64, %65, p, 1, 1, 0, 0;\n\t}"
                 : DSB_O8(0), DSB_O8(8), DSB_O8(16), DSB_O8(24), DSB_O8(32), DSB_O8(40), DSB_O8(48), DSB_O8(56)
                 : "l"(da), "l"(db), "r"(accumulate));
  }
  static __device__ __forceinline__ void tf32(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {" DSB_P10() DSB_P10(1) DSB_P10(2) DSB_P10(3) DSB_P10(4) DSB_P10(5) "%60, %61, %62, %63"
                 "}, %64, %65, p, 1, 1;\n\t}"
                 : DSB_O8(0), DSB_O8(8), DSB_O8(16), DSB_O8(24), DSB_O8(32), DSB_O8(40), DSB_O8(48), DSB_O8(56)
                 : "l"(da), "l"(db), "r"(accumulate));
  }
};

template <> struct Wgmma<192> {
  static __device__ __forceinline__ void f16(float (&d)[96], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %98, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n192k16.f32.f16.f16 {" DSB_P10() DSB_P10(1) DSB_P10(2) DSB_P10(3) DSB_P10(4) DSB_P10(5) DSB_P10(6) DSB_P10(7) DSB_P10(8) "%90, %91, %92, %93, %94, %95"
                 "}, %96, %97, p, 1, 1, 0, 0;\n\t}"
                 : DSB_O8(0), DSB_O8(8), DSB_O8(16), DSB_O8(24), DSB_O8(32), DSB_O8(40), DSB_O8(48), DSB_O8(56), DSB_O8(64), DSB_O8(72), DSB_O8(80), DSB_O8(88)
                 : "l"(da), "l"(db), "r"(accumulate));
  }
  static __device__ __forceinline__ void tf32(float (&d)[96], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %98, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n192k8.f32.tf32.tf32 {" DSB_P10() DSB_P10(1) DSB_P10(2) DSB_P10(3) DSB_P10(4) DSB_P10(5) DSB_P10(6) DSB_P10(7) DSB_P10(8) "%90, %91, %92, %93, %94, %95"
                 "}, %96, %97, p, 1, 1;\n\t}"
                 : DSB_O8(0), DSB_O8(8), DSB_O8(16), DSB_O8(24), DSB_O8(32), DSB_O8(40), DSB_O8(48), DSB_O8(56), DSB_O8(64), DSB_O8(72), DSB_O8(80), DSB_O8(88)
                 : "l"(da), "l"(db), "r"(accumulate));
  }
};

template <> struct Wgmma<256> {
  static __device__ __forceinline__ void f16(float (&d)[128], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {" DSB_P10() DSB_P10(1) DSB_P10(2) DSB_P10(3) DSB_P10(4) DSB_P10(5) DSB_P10(6) DSB_P10(7) DSB_P10(8) DSB_P10(9) DSB_P10(10) DSB_P10(11) "%120, %121, %122, %123, %124, %125, %126, %127"
                 "}, %128, %129, p, 1, 1, 0, 0;\n\t}"
                 : DSB_O8(0), DSB_O8(8), DSB_O8(16), DSB_O8(24), DSB_O8(32), DSB_O8(40), DSB_O8(48), DSB_O8(56), DSB_O8(64), DSB_O8(72), DSB_O8(80), DSB_O8(88), DSB_O8(96), DSB_O8(104), DSB_O8(112), DSB_O8(120)
                 : "l"(da), "l"(db), "r"(accumulate));
  }
  static __device__ __forceinline__ void tf32(float (&d)[128], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {" DSB_P10() DSB_P10(1) DSB_P10(2) DSB_P10(3) DSB_P10(4) DSB_P10(5) DSB_P10(6) DSB_P10(7) DSB_P10(8) DSB_P10(9) DSB_P10(10) DSB_P10(11) "%120, %121, %122, %123, %124, %125, %126, %127"
                 "}, %128, %129, p, 1, 1;\n\t}"
                 : DSB_O8(0), DSB_O8(8), DSB_O8(16), DSB_O8(24), DSB_O8(32), DSB_O8(40), DSB_O8(48), DSB_O8(56), DSB_O8(64), DSB_O8(72), DSB_O8(80), DSB_O8(88), DSB_O8(96), DSB_O8(104), DSB_O8(112), DSB_O8(120)
                 : "l"(da), "l"(db), "r"(accumulate));
  }
};
}  // namespace tc
}  // namespace dsb

#undef DSB_P10
#undef DSB_O8
