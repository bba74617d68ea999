// rbk_gather.cu — the gather kernel of rbk_index_search_slots_f64: stored rows of named slots as float64 queries.
#include "rbk_internal.h"

namespace rbk {

namespace {

// The stored value of element j of a row as float64: the exact element widened, the split's float32 joined from its
// low half and the scan copy's high half hi[j], or (uint16_t: an index without exact rows) the bf16 scan copy widened.
__device__ __forceinline__ double stored_f64(double x, const uint16_t*, int) { return x; }
__device__ __forceinline__ double stored_f64(float x, const uint16_t*, int) { return static_cast<double>(x); }
__device__ __forceinline__ double stored_f64(F32Lo x, const uint16_t* hi, int j) { return split_f64(hi[j], x.bits); }
__device__ __forceinline__ double stored_f64(uint16_t x, const uint16_t*, int) {
  return static_cast<double>(__uint_as_float(static_cast<uint32_t>(x) << 16));
}

constexpr int kGatherThreads = 256;

// One block per query: row sel[b]'s stored values into dst row b (pitch d), read with 16-byte loads from the row's
// first 16-byte boundary on (a row of x starts wherever d * sizeof(XT) puts it); a tombstoned row adds 1 to *n_dead.
// x: the exact rows (pitch d; mapped host memory under RBK_INDEX_ROWS_ON_HOST) or, uint16_t, the scan copy itself.
template <typename XT>
__global__ void __launch_bounds__(kGatherThreads) gather_rows_kernel(const XT* __restrict__ x, int64_t x_pitch,
                                                                     const uint16_t* __restrict__ rows, int dpad,
                                                                     const unsigned int* __restrict__ dead_bits,
                                                                     const int64_t* __restrict__ sel, int d,
                                                                     double* __restrict__ dst, int* __restrict__ n_dead) {
  const int64_t r = sel[blockIdx.x];
  double* out = dst + static_cast<int64_t>(blockIdx.x) * d;
  if ((dead_bits[r >> 5] >> (r & 31)) & 1u) {   // uniform over the block
    if (threadIdx.x == 0) atomicAdd(n_dead, 1);
    for (int j = threadIdx.x; j < d; j += kGatherThreads) out[j] = 0.0;
    return;
  }
  const XT* src = x + r * x_pitch;
  const uint16_t* hi = rows + r * dpad;
  constexpr int V = 16 / sizeof(XT);
  const int head = min(d, static_cast<int>(((16 - (reinterpret_cast<uintptr_t>(src) & 15)) & 15) / sizeof(XT)));
  const int nvec = (d - head) / V;
  for (int j = threadIdx.x; j < head; j += kGatherThreads) out[j] = stored_f64(src[j], hi, j);
  const uint4* vsrc = reinterpret_cast<const uint4*>(src + head);
  for (int v = threadIdx.x; v < nvec; v += kGatherThreads) {
    const uint4 w = vsrc[v];
    const XT* e = reinterpret_cast<const XT*>(&w);
#pragma unroll
    for (int i = 0; i < V; ++i) out[head + v * V + i] = stored_f64(e[i], hi, head + v * V + i);
  }
  for (int j = head + nvec * V + threadIdx.x; j < d; j += kGatherThreads) out[j] = stored_f64(src[j], hi, j);
}

}  // namespace

cudaError_t launch_gather_rows(const uint16_t* rows, const void* rows_x, int x_elem, const unsigned int* dead_bits,
                               const int64_t* sel, int B, int d, int dpad, double* dst, int* n_dead,
                               cudaStream_t stream) {
  if (B <= 0) return cudaSuccess;
  if (x_elem == 8)
    gather_rows_kernel<double><<<B, kGatherThreads, 0, stream>>>(static_cast<const double*>(rows_x), d, rows, dpad,
                                                                 dead_bits, sel, d, dst, n_dead);
  else if (x_elem == 4)
    gather_rows_kernel<float><<<B, kGatherThreads, 0, stream>>>(static_cast<const float*>(rows_x), d, rows, dpad,
                                                                dead_bits, sel, d, dst, n_dead);
  else if (x_elem == 2)
    gather_rows_kernel<F32Lo><<<B, kGatherThreads, 0, stream>>>(static_cast<const F32Lo*>(rows_x), d, rows, dpad,
                                                                dead_bits, sel, d, dst, n_dead);
  else
    gather_rows_kernel<uint16_t><<<B, kGatherThreads, 0, stream>>>(rows, dpad, rows, dpad, dead_bits, sel, d, dst,
                                                                   n_dead);
  return cudaGetLastError();
}

}  // namespace rbk
