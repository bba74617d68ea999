// rbk_compact.cu — K8: compaction.  Reclaims the slots of tombstoned rows (rbk_index_compact): the live rows move
// down to local slots 0 .. count()-1 in their current order.  Three small kernels turn the liveness bits of the
// 32-row words of dead_bits into old_to_new (an exclusive prefix count of live rows), and one gather kernel per
// staging chunk copies the live rows of that chunk, packed, into the staging buffer; the host then places each staged
// chunk with plain device-to-device copies (rbk_capi.cu).  All of it is an HBM stream with no reuse.
#include <type_traits>

#include "rbk_internal.h"

namespace rbk {

namespace {

constexpr int kScanBlock = 1024;   // words per block of the first scan level (and threads per block)

// live bits of word w of a corpus of n_rows rows: the complement of the tombstone bits, cut at n_rows
__device__ __forceinline__ unsigned int live_word(const unsigned int* __restrict__ dead_bits, int64_t w, int64_t n_rows) {
  unsigned int live = ~dead_bits[w];
  const int64_t left = n_rows - w * 32;
  if (left < 32) live &= (1u << left) - 1u;
  return live;
}

// exclusive scan of v over the block (blockDim.x == kScanBlock); *total receives the block's sum
__device__ __forceinline__ int block_exclusive_scan(int v, int* total) {
  __shared__ int s_warp[kScanBlock / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xFFFFFFFFu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) s_warp[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int t = s_warp[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xFFFFFFFFu, t, o);
      if (lane >= o) t += y;
    }
    s_warp[lane] = t;   // inclusive over warps
  }
  __syncthreads();
  const int before = (warp > 0 ? s_warp[warp - 1] : 0) + x - v;
  *total = s_warp[kScanBlock / 32 - 1];
  __syncthreads();      // s_warp is reused by the next call
  return before;
}

// Level 1: per word, the live rows of the earlier words of its block; per block, its live rows.
__global__ void __launch_bounds__(kScanBlock) compact_word_scan_kernel(const unsigned int* __restrict__ dead_bits,
                                                                      int64_t n_rows, int64_t n_words,
                                                                      int* __restrict__ word_pref,
                                                                      int* __restrict__ block_sum) {
  const int64_t w = static_cast<int64_t>(blockIdx.x) * kScanBlock + threadIdx.x;
  const int c = w < n_words ? __popc(live_word(dead_bits, w, n_rows)) : 0;
  int total;
  const int ex = block_exclusive_scan(c, &total);
  if (w < n_words) word_pref[w] = ex;
  if (threadIdx.x == 0) block_sum[blockIdx.x] = total;
}

// Level 2 (one block): exclusive scan of the block sums in place; the grand total goes to *n_live_out.
__global__ void __launch_bounds__(kScanBlock) compact_block_scan_kernel(int* __restrict__ block_sum, int n_blocks,
                                                                       int* __restrict__ n_live_out) {
  int carry = 0;
  for (int b0 = 0; b0 < n_blocks; b0 += kScanBlock) {
    const int b = b0 + threadIdx.x;
    const int v = b < n_blocks ? block_sum[b] : 0;
    int total;
    const int ex = block_exclusive_scan(v, &total);
    if (b < n_blocks) block_sum[b] = carry + ex;
    carry += total;
  }
  if (threadIdx.x == 0) *n_live_out = carry;
}

// Level 3: old_to_new of every row, and the live rows before each staging chunk (chunk_rows is a multiple of 32).
__global__ void compact_map_kernel(const unsigned int* __restrict__ dead_bits, int64_t n_rows,
                                   const int* __restrict__ word_pref, const int* __restrict__ block_sum,
                                   int64_t chunk_rows, long long* __restrict__ old_to_new,
                                   int* __restrict__ chunk_pref) {
  const int64_t s = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (s >= n_rows) return;
  const int64_t w = s >> 5;
  const unsigned int live = live_word(dead_bits, w, n_rows);
  const int bit = static_cast<int>(s & 31);
  const long long before = static_cast<long long>(block_sum[w / kScanBlock]) + word_pref[w];
  old_to_new[s] = ((live >> bit) & 1u) ? before + __popc(live & ((1u << bit) - 1u)) : -1ll;
  if (s % chunk_rows == 0) chunk_pref[s / chunk_rows] = static_cast<int>(before);
}

// Every live row of source rows [s0, s0 + n) goes to staging row old_to_new[s] - d0: its bf16 row (16-byte pieces),
// its exact row (when the index keeps one; XT = double or float, moved as is), norm2 and inv_norm.
template <typename XT>
__global__ void __launch_bounds__(256) compact_gather_kernel(const uint16_t* __restrict__ rows,
                                                             const XT* __restrict__ rows_f64,
                                                             const double* __restrict__ norm2,
                                                             const float* __restrict__ inv_norm,
                                                             const long long* __restrict__ old_to_new, int64_t s0,
                                                             int64_t n, long long d0, int d, int dpad,
                                                             uint16_t* __restrict__ st_rows,
                                                             XT* __restrict__ st_f64,
                                                             double* __restrict__ st_norm2,
                                                             float* __restrict__ st_inv) {
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  const int64_t t0 = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int u16 = dpad >> 3;   // 16-byte pieces per bf16 row
  for (int64_t g = t0; g < n * u16; g += stride) {
    const int64_t r = g / u16;
    const int u = static_cast<int>(g - r * u16);
    const long long j = old_to_new[s0 + r];
    if (j < 0) continue;
    reinterpret_cast<uint4*>(st_rows + (j - d0) * dpad)[u] =
        __ldg(reinterpret_cast<const uint4*>(rows + (s0 + r) * dpad) + u);
  }
  // two elements per move: 16 bytes (double2), 8 (float2) or 4 (the split's low halves, ushort2; their high halves
  // moved with the scan copy above)
  using X2 = typename std::conditional<sizeof(XT) == 8, double2,
                                       typename std::conditional<sizeof(XT) == 4, float2, ushort2>::type>::type;
  if (rows_f64 != nullptr) {
    if ((d & 1) == 0) {   // rows start aligned to two elements
      const int u2 = d >> 1;
      for (int64_t g = t0; g < n * u2; g += stride) {
        const int64_t r = g / u2;
        const int u = static_cast<int>(g - r * u2);
        const long long j = old_to_new[s0 + r];
        if (j < 0) continue;
        reinterpret_cast<X2*>(st_f64 + (j - d0) * d)[u] = __ldg(reinterpret_cast<const X2*>(rows_f64 + (s0 + r) * d) + u);
      }
    } else {
      for (int64_t g = t0; g < n * d; g += stride) {
        const int64_t r = g / d;
        const int u = static_cast<int>(g - r * d);
        const long long j = old_to_new[s0 + r];
        if (j < 0) continue;
        if constexpr (kIsSplit<XT>) st_f64[(j - d0) * d + u].bits = __ldg(&rows_f64[(s0 + r) * d + u].bits);
        else st_f64[(j - d0) * d + u] = __ldg(rows_f64 + (s0 + r) * d + u);
      }
    }
  }
  for (int64_t r = t0; r < n; r += stride) {
    const long long j = old_to_new[s0 + r];
    if (j < 0) continue;
    st_norm2[j - d0] = norm2[s0 + r];
    st_inv[j - d0] = inv_norm[s0 + r];
  }
}

}  // namespace

cudaError_t launch_compact_map(const unsigned int* dead_bits, int64_t n_rows, int64_t chunk_rows, int* word_pref,
                               int* block_sum, long long* old_to_new, int* chunk_pref, cudaStream_t stream) {
  if (n_rows <= 0) return cudaSuccess;
  const int64_t n_words = (n_rows + 31) / 32;
  const int n_blocks = static_cast<int>((n_words + kScanBlock - 1) / kScanBlock);
  const int64_t n_chunks = (n_rows + chunk_rows - 1) / chunk_rows;
  compact_word_scan_kernel<<<n_blocks, kScanBlock, 0, stream>>>(dead_bits, n_rows, n_words, word_pref, block_sum);
  compact_block_scan_kernel<<<1, kScanBlock, 0, stream>>>(block_sum, n_blocks, chunk_pref + n_chunks);
  compact_map_kernel<<<static_cast<unsigned>((n_rows + 255) / 256), 256, 0, stream>>>(
      dead_bits, n_rows, word_pref, block_sum, chunk_rows, old_to_new, chunk_pref);
  return cudaGetLastError();
}

cudaError_t launch_compact_gather(const uint16_t* rows, const void* rows_x, int x_elem, const double* norm2,
                                  const float* inv_norm, const long long* old_to_new, int64_t s0, int64_t n,
                                  long long d0, int d, int dpad, uint16_t* st_rows, void* st_x, double* st_norm2,
                                  float* st_inv, int sm_count, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  const int64_t work = n * (dpad >> 3);
  int64_t blocks = (work + 255) / 256;
  if (blocks > static_cast<int64_t>(sm_count) * 16) blocks = static_cast<int64_t>(sm_count) * 16;   // grid-stride
  if (x_elem == 4)
    compact_gather_kernel<float><<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
        rows, static_cast<const float*>(rows_x), norm2, inv_norm, old_to_new, s0, n, d0, d, dpad, st_rows,
        static_cast<float*>(st_x), st_norm2, st_inv);
  else if (x_elem == 2)
    compact_gather_kernel<F32Lo><<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
        rows, static_cast<const F32Lo*>(rows_x), norm2, inv_norm, old_to_new, s0, n, d0, d, dpad, st_rows,
        static_cast<F32Lo*>(st_x), st_norm2, st_inv);
  else
    compact_gather_kernel<double><<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
        rows, static_cast<const double*>(rows_x), norm2, inv_norm, old_to_new, s0, n, d0, d, dpad, st_rows,
        static_cast<double*>(st_x), st_norm2, st_inv);
  return cudaGetLastError();
}

}  // namespace rbk
