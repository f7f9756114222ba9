// deflate.cuh -- zlib / RFC 1950-1951 pieces shared by the PNG encoder (png.cu) and decoder (png_decode.cu).
#pragma once
#include <stdint.h>

namespace gab {
namespace {

constexpr uint32_t ADLER_BASE = 65521;

// zlib's adler32_combine: the Adler-32 of A || B from those of A and B and B's length
__device__ __forceinline__ uint32_t adler_combine(uint32_t a1, uint32_t a2, uint32_t len2) {
  const uint32_t rem = len2 % ADLER_BASE;
  uint32_t sum1 = a1 & 0xffff;
  uint32_t sum2 = (uint32_t)(((uint64_t)rem * sum1) % ADLER_BASE);
  sum1 += (a2 & 0xffff) + ADLER_BASE - 1;
  sum2 += ((a1 >> 16) & 0xffff) + ((a2 >> 16) & 0xffff) + ADLER_BASE - rem;
  if (sum1 >= ADLER_BASE) sum1 -= ADLER_BASE;
  if (sum1 >= ADLER_BASE) sum1 -= ADLER_BASE;
  if (sum2 >= (ADLER_BASE << 1)) sum2 -= (ADLER_BASE << 1);
  if (sum2 >= ADLER_BASE) sum2 -= ADLER_BASE;
  return sum1 | (sum2 << 16);
}

// the order in which a dynamic block header lists the code-length code's lengths (RFC 1951 3.2.7)
__constant__ uint8_t CL_ORDER[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

}  // namespace
}  // namespace gab
