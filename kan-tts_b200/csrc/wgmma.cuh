// wgmma.mma_async m64nNk16, bf16 x bf16 -> fp32 (register accumulators of one warpgroup), A and B from shared-memory
// descriptors; TA / TB = 1: the operand is MN-major (transposed).  wgmma_nN uses the accumulators d[O, O + N / 2);
// scale_d = 0 overwrites them.  N = 16, 32, ..., 128: 8 accumulator registers per 16 columns.
#pragma once
#include <stdint.h>

namespace kt {
namespace tc {

constexpr int kWgmmaMaxN = 128;
constexpr int kWgmmaMaxRegs = kWgmmaMaxN / 2;   // fp32 accumulators per thread at N = 128

// asm operand names of accumulator registers 8c .. 8c + 7, and the matching "+f" operands
#define KT_R0 "%0, %1, %2, %3, %4, %5, %6, %7"
#define KT_R1 "%8, %9, %10, %11, %12, %13, %14, %15"
#define KT_R2 "%16, %17, %18, %19, %20, %21, %22, %23"
#define KT_R3 "%24, %25, %26, %27, %28, %29, %30, %31"
#define KT_R4 "%32, %33, %34, %35, %36, %37, %38, %39"
#define KT_R5 "%40, %41, %42, %43, %44, %45, %46, %47"
#define KT_R6 "%48, %49, %50, %51, %52, %53, %54, %55"
#define KT_R7 "%56, %57, %58, %59, %60, %61, %62, %63"
#define KT_D(c) "+f"(d[O + 8 * c]), "+f"(d[O + 8 * c + 1]), "+f"(d[O + 8 * c + 2]), "+f"(d[O + 8 * c + 3]), \
                "+f"(d[O + 8 * c + 4]), "+f"(d[O + 8 * c + 5]), "+f"(d[O + 8 * c + 6]), "+f"(d[O + 8 * c + 7])

// IA .. ITB: asm operand numbers of the descriptors, scale_d and the transpose immediates (they follow the accumulators)
#define KT_WGMMA_FN(N, REGS, IA, IB, IS, ITA, ITB, ...)                                                                \
  template <int TA, int TB, int O = 0>                                                                                 \
  __device__ __forceinline__ void wgmma_n##N(float (&d)[kWgmmaMaxRegs], uint64_t da, uint64_t db, uint32_t scale_d) { \
    static_assert(O + N / 2 <= kWgmmaMaxRegs, "wgmma_n" #N ": accumulator offset out of range");                     \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" IS ", 0;\n\t"                                              \
                 "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.bf16.bf16 {" REGS "}, %" IA ", %" IB               \
                 ", p, 1, 1, %" ITA ", %" ITB ";\n\t}"                                                                 \
                 : __VA_ARGS__                                                                                         \
                 : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));                                                 \
  }

KT_WGMMA_FN(16, KT_R0, "8", "9", "10", "11", "12", KT_D(0))
KT_WGMMA_FN(32, KT_R0 ", " KT_R1, "16", "17", "18", "19", "20", KT_D(0), KT_D(1))
KT_WGMMA_FN(48, KT_R0 ", " KT_R1 ", " KT_R2, "24", "25", "26", "27", "28", KT_D(0), KT_D(1), KT_D(2))
KT_WGMMA_FN(64, KT_R0 ", " KT_R1 ", " KT_R2 ", " KT_R3, "32", "33", "34", "35", "36", KT_D(0), KT_D(1), KT_D(2), KT_D(3))
KT_WGMMA_FN(80, KT_R0 ", " KT_R1 ", " KT_R2 ", " KT_R3 ", " KT_R4, "40", "41", "42", "43", "44", KT_D(0), KT_D(1), KT_D(2), KT_D(3),
            KT_D(4))
KT_WGMMA_FN(96, KT_R0 ", " KT_R1 ", " KT_R2 ", " KT_R3 ", " KT_R4 ", " KT_R5, "48", "49", "50", "51", "52", KT_D(0), KT_D(1), KT_D(2),
            KT_D(3), KT_D(4), KT_D(5))
KT_WGMMA_FN(112, KT_R0 ", " KT_R1 ", " KT_R2 ", " KT_R3 ", " KT_R4 ", " KT_R5 ", " KT_R6, "56", "57", "58", "59", "60", KT_D(0), KT_D(1),
            KT_D(2), KT_D(3), KT_D(4), KT_D(5), KT_D(6))
KT_WGMMA_FN(128, KT_R0 ", " KT_R1 ", " KT_R2 ", " KT_R3 ", " KT_R4 ", " KT_R5 ", " KT_R6 ", " KT_R7, "64", "65", "66", "67", "68", KT_D(0),
            KT_D(1), KT_D(2), KT_D(3), KT_D(4), KT_D(5), KT_D(6), KT_D(7))

#undef KT_WGMMA_FN
#undef KT_D
#undef KT_R0
#undef KT_R1
#undef KT_R2
#undef KT_R3
#undef KT_R4
#undef KT_R5
#undef KT_R6
#undef KT_R7

// N fixed at compile time
template <int N, int TA, int TB, int O = 0>
__device__ __forceinline__ void wgmma_bf16_n(float (&d)[kWgmmaMaxRegs], uint64_t da, uint64_t db, uint32_t scale_d) {
  static_assert(N % 16 == 0 && N >= 16 && N <= kWgmmaMaxN, "wgmma_bf16_n: N out of range");
  if constexpr (N == 16) wgmma_n16<TA, TB, O>(d, da, db, scale_d);
  else if constexpr (N == 32) wgmma_n32<TA, TB, O>(d, da, db, scale_d);
  else if constexpr (N == 48) wgmma_n48<TA, TB, O>(d, da, db, scale_d);
  else if constexpr (N == 64) wgmma_n64<TA, TB, O>(d, da, db, scale_d);
  else if constexpr (N == 80) wgmma_n80<TA, TB, O>(d, da, db, scale_d);
  else if constexpr (N == 96) wgmma_n96<TA, TB, O>(d, da, db, scale_d);
  else if constexpr (N == 112) wgmma_n112<TA, TB, O>(d, da, db, scale_d);
  else wgmma_n128<TA, TB, O>(d, da, db, scale_d);
}

// N = 16, 32, ..., 128 chosen at run time; the accumulator array is always indexed with constants (registers)
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16(int n, float (&d)[kWgmmaMaxRegs], uint64_t da, uint64_t db, uint32_t scale_d) {
  switch (n) {
    case 16: wgmma_n16<TA, TB>(d, da, db, scale_d); break;
    case 32: wgmma_n32<TA, TB>(d, da, db, scale_d); break;
    case 48: wgmma_n48<TA, TB>(d, da, db, scale_d); break;
    case 64: wgmma_n64<TA, TB>(d, da, db, scale_d); break;
    case 80: wgmma_n80<TA, TB>(d, da, db, scale_d); break;
    case 96: wgmma_n96<TA, TB>(d, da, db, scale_d); break;
    case 112: wgmma_n112<TA, TB>(d, da, db, scale_d); break;
    case 128: wgmma_n128<TA, TB>(d, da, db, scale_d); break;
    default: __trap();
  }
}

}  // namespace tc
}  // namespace kt
