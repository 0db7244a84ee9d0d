// wgmma.mma_async m64nNk16, fp16 A and B both K-major from shared memory, fp32 accumulators in registers.
// Inline assembly cannot loop over an operand list, so the register lists are spelled out by macros, one wrapper per
// tile width N (multiples of 32): N / 2 accumulators per thread, operands %0 .. %(N/2 - 1), then desc A, desc B, scale-d.
#pragma once
#include <stdint.h>

#define PE_D8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), \
    "+f"(d[i + 6]), "+f"(d[i + 7])
#define PE_D16(i) PE_D8(i), PE_D8(i + 8)

#define PE_R16 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
#define PE_R32 PE_R16 ", %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
#define PE_R48 PE_R32 ", %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47"
#define PE_R64 PE_R48 ", %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
#define PE_R80 PE_R64 ", %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79"
#define PE_R96 PE_R80 ", %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95"
#define PE_R112 PE_R96 ", %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111"
#define PE_R128 PE_R112 ", %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"

#define PE_WGMMA(N, R, RA, RB, RS, ...)                                                                                     \
  template <>                                                                                                   \
  struct Wgmma<N> {                                                                                             \
    __device__ __forceinline__ static void mma(float (&d)[R], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) { \
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #RS ", 0;\n\t"                                   \
                   "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.f16.f16 {" PE_R##R "}, %" #RA ", %" #RB ", p, 1, 1, 0, 0;\n\t}" \
                   : __VA_ARGS__                                                                                    \
                   : "l"(desc_a), "l"(desc_b), "r"(scale_d));                                                   \
    }                                                                                                           \
  };

namespace pe {

template <int N>
struct Wgmma;

PE_WGMMA(32, 16, 16, 17, 18, PE_D16(0))
PE_WGMMA(64, 32, 32, 33, 34, PE_D16(0), PE_D16(16))
PE_WGMMA(96, 48, 48, 49, 50, PE_D16(0), PE_D16(16), PE_D16(32))
PE_WGMMA(128, 64, 64, 65, 66, PE_D16(0), PE_D16(16), PE_D16(32), PE_D16(48))
PE_WGMMA(160, 80, 80, 81, 82, PE_D16(0), PE_D16(16), PE_D16(32), PE_D16(48), PE_D16(64))
PE_WGMMA(192, 96, 96, 97, 98, PE_D16(0), PE_D16(16), PE_D16(32), PE_D16(48), PE_D16(64), PE_D16(80))
PE_WGMMA(224, 112, 112, 113, 114, PE_D16(0), PE_D16(16), PE_D16(32), PE_D16(48), PE_D16(64), PE_D16(80), PE_D16(96))
PE_WGMMA(256, 128, 128, 129, 130, PE_D16(0), PE_D16(16), PE_D16(32), PE_D16(48), PE_D16(64), PE_D16(80), PE_D16(96), PE_D16(112))

}  // namespace pe
