// rbk_f16.cuh — the storage rule of RBK_INDEX_SCAN_F16 indexes (DESIGN.md §3), shared by the ingest kernels (rows)
// and the query preparation (queries), so that both sides of the scan are rounded the same way:
//   e   = 15 - E, where max_i |x_i| over the finite elements = m * 2^E, m in [0.5, 1) (frexp): max|x| * 2^e lies in
//         [2^14, 2^15), so every finite element scales into fp16's normal range or below it;
//   h_i = RNE_f16(x_i * 2^e), ONE rounding from float64 (what numpy's astype(np.float16) does), and a result that
//         would be subnormal is stored as a zero of the same sign: no stored value is subnormal.
// All-zero rows give zeros, non-finite elements stay non-finite.  The scale is not stored: cosine does not depend on
// it, and 1/||h|| carries it wherever a raw score meets a cosine.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

namespace rbk {

// e of the rule above for amax = max |x_i| over the finite elements (0 for an all-zero / all-non-finite row).
__device__ __forceinline__ int f16_scale_exp(double amax) {
  if (!(amax > 0.0)) return 0;
  int E;
  frexp(amax, &E);
  return 15 - E;
}

// x * 2^e, e in [-1009, 1089] (the range f16_scale_exp yields): exact unless the result is below the smallest normal
// double, which only happens to elements far below the fp16 range (they round to zero either way).
__device__ __forceinline__ double scale_pow2(double x, int e) {
  if (e > 1000) {   // rows below 2^-985: scale up in two exact steps
    x *= 0x1p600;
    e -= 600;
  }
  return x * __longlong_as_double(static_cast<long long>(e + 1023) << 52);
}

// RNE of y to fp16 in one step from float64, subnormal results flushed to a signed zero.  |y| < 2^15 for finite y
// (a scaled element), so nothing overflows.
__device__ __forceinline__ uint16_t f16_bits_flush(double y) {
  const double a = fabs(y);
  if (!(a < INFINITY)) return __half_as_ushort(__float2half_rn(static_cast<float>(y)));   // inf / nan stay so
  const uint16_t sign = signbit(y) ? 0x8000u : 0u;
  if (a < 0x1p-15) return sign;   // rounds below 2^-14 (the smallest normal fp16): flushed
  int E;
  frexp(a, &E);                                   // a in [2^(E-1), 2^E)
  const int ulp_exp = E - 11 > -24 ? E - 11 : -24;   // fp16 keeps 11 significant bits; subnormal spacing 2^-24
  const double r = ldexp(rint(ldexp(a, -ulp_exp)), ulp_exp);   // exact scalings around one RNE
  if (r < 0x1p-14) return sign;
  return sign | __half_as_ushort(__float2half_rn(static_cast<float>(r)));   // r is an fp16 value: exact
}

__device__ __forceinline__ double f16_bits_to_f64(uint32_t h) {
  return static_cast<double>(__half2float(__ushort_as_half(static_cast<unsigned short>(h))));
}

}  // namespace rbk
