// Shared device helpers: exact dyadic requantisation, PTX wrappers (cp.async, ldmatrix, IMMA), nibble packing.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/hawq_b200.h"

namespace hawq {

// ---------------------------------------------------------------------------------------------------------
// q = RHE(v * m / 2^e)  (round-half-to-even), exact in 64-bit integers.
// Reference semantics: torch.round(f64(v) * f64(m) / 2^e), utils/quantization_utils/quant_utils.py:406-408;
// identical while |v*m| < 2^53 (the reference's own exactness envelope, SURVEY.md A.6), exact beyond it.
// Preconditions: m <= 2^31, 1 <= e <= 62.  Result saturated to int32.
// ---------------------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ long long rhe_requant64(int32_t v, uint32_t m, int32_t e) {   // unsaturated
  const long long p = (long long)v * (long long)(unsigned long long)m;  // |p| <= 2^62
  long long q = p >> e;                                                  // floor
  const unsigned long long rem = (unsigned long long)p & ((1ull << e) - 1ull);
  const unsigned long long half = 1ull << (e - 1);
  q += (long long)((rem > half) | ((rem == half) & (unsigned long long)(q & 1)));
  return q;
}
__host__ __device__ __forceinline__ int32_t sat_i32(long long q) {
  q = q > 2147483647ll ? 2147483647ll : q;
  q = q < -2147483648ll ? -2147483648ll : q;
  return (int32_t)q;
}
__host__ __device__ __forceinline__ int32_t rhe_requant(int32_t v, uint32_t m, int32_t e) { return sat_i32(rhe_requant64(v, m, e)); }

__device__ __forceinline__ int32_t clampi(int32_t v, int32_t lo, int32_t hi) { return max(lo, min(v, hi)); }

__device__ __forceinline__ int32_t sat_add(int32_t a, int32_t b) {
  int32_t r;
  asm("add.sat.s32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
  return r;
}

// ---------------------------------------------------------------------------------------------------------
// Fast exact path for the common case ratio = m * 2^-e <= 1 (every HAWQ ResNet layer):
//   q = RHE(v * M),  M = m * 2^-e held as a double (exact: m <= 2^31, power-of-two scaling).
// double(v) is built without a conversion instruction: bits(2^52 + 2^31 + v) = {0x43300000, v ^ 0x80000000}, minus
// (2^52 + 2^31) is exact.  fma(double(v), M, 1.5 * 2^52) forms the exact product and rounds ONCE, to an integer
// (ulp = 1 in [2^52, 2^53)), ties-to-even; the low mantissa word is q in two's complement (|q| <= |v| < 2^31).
// = the reference's round(f64(v) * f64(m) / 2^e) whenever that product is exact in fp64, and the exact integer
// result otherwise.  2 FP64 instructions + 1 LOP per value.
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double dyadic_to_double(uint32_t m, int32_t e) {
  return (double)m * __hiloint2double((1023 - e) << 20, 0);   // m * 2^-e, exact
}
__host__ __device__ __forceinline__ bool dyadic_is_fast(uint32_t m, int32_t e) { return m == 0u || e >= 31; }
// ratio m * 2^-e <= 2^20: |v| < 2^32 times M stays below 2^52, so the one-FMA form is exact whenever its result fits int32
__host__ __device__ __forceinline__ bool dyadic_is_wide(uint32_t m, int32_t e) { return m == 0u || e >= 11; }

__device__ __forceinline__ int32_t rhe_requant_fast(int32_t v, double M) {
  const double dv = __hiloint2double(0x43300000, (int)((uint32_t)v ^ 0x80000000u)) - 4503601774854144.0;
  return __double2loint(__fma_rn(dv, M, 6755399441055744.0));
}

// QuantAveragePool2d integer rule (quant_modules.py:585-602, quant_utils.py:324-341): trunc(sum/kk + 0.01).
__host__ __device__ __forceinline__ int32_t trunc_avg(long long s, int kk) {
  if (s >= 0) return (int32_t)(s / kk);
  const long long a = -s;
  const long long q = a / kk;
  return (int32_t)((a % kk == 0) ? (-q + 1) : -q);
}

// ---------------------------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void cp_async_16(uint32_t dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

__device__ __forceinline__ void ldmatrix_x2(uint32_t& r0, uint32_t& r1, uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0,%1}, [%2];\n" : "=r"(r0), "=r"(r1) : "r"(addr));
}

// D(16x8,s32) += A(16x32, s8 row) * B(32x8, s8 col)
__device__ __forceinline__ void mma_16832(int32_t (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// hawq nibble order: 8 channels c0..c7 -> 4 bytes, byte j = c_j | c_{j+4} << 4.
// lo_word holds c0..c3 as bytes, hi_word holds c4..c7 as bytes (all values 0..15).
__host__ __device__ __forceinline__ uint32_t pack_nibbles8(uint32_t lo_word, uint32_t hi_word) {
  return (lo_word & 0x0F0F0F0Fu) | ((hi_word & 0x0F0F0F0Fu) << 4);
}

}  // namespace hawq
