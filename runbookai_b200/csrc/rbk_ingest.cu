// rbk_ingest.cu — K3: corpus ingest.  Replaces VectorStore.loadEmbeddings /
// bufferToFloatArray (reference src/knowledge/store/vector-store.ts:56-88): rows arrive as
// little-endian float64 (the SQLite BLOB layout), float32 or bf16 and are stored as bf16
// rows of pitch dpad (= dim rounded up to 8 elements, zero padded) - or, for RBK_INDEX_SCAN_F16
// indexes, as per-row scaled fp16 rows (rbk_f16.cuh) - plus, per row,
//   inv_norm (fp32)  1/||row||           for the approximate scan (NaN = never matches)
//   norm2    (fp64)  sum of squares accumulated in index order, multiply-then-add — the
//                    reference's `normB` (embedder.ts:175-181) bit for bit, reused by the
//                    exact re-rank so it is not recomputed per query.
// Both kernels are HBM-bound streams: 16-byte vector loads/stores, no reuse.
#include <cuda_bf16.h>

#include "rbk_f16.cuh"
#include "rbk_internal.h"

namespace rbk {

namespace {

__device__ __forceinline__ uint16_t f64_to_bf16_bits(double x) {
  // f64 -> f32 (RNE) -> bf16 (RNE); documented in DESIGN.md §3.
  return __bfloat16_as_ushort(__float2bfloat16_rn(__double2float_rn(x)));
}
__device__ __forceinline__ uint16_t f32_to_bf16_bits(float x) {
  return __bfloat16_as_ushort(__float2bfloat16_rn(x));
}

// One thread produces 8 consecutive output elements (one 16-byte store).  XT: element type of the exact rows (double,
// or float for RBK_INDEX_KEEP_F32, whose sources hold float32-exact values: the scan copy is derived from the source
// value, which equals the stored one).
template <typename SrcT, typename XT>
__global__ void __launch_bounds__(256) convert_rows_kernel(const SrcT* __restrict__ src, int64_t n_rows, int d,
                                                           int dpad, uint16_t* __restrict__ dst,
                                                           XT* __restrict__ dst_f64, bool aligned,
                                                           const int64_t* __restrict__ slot_map,
                                                           const unsigned int* __restrict__ dead_bits,
                                                           int* __restrict__ n_dead) {
  // slot_map == nullptr: source row r -> destination row r of dst (an append).  slot_map != nullptr (bulk
  // overwrite): dst/dst_f64 are the index's row 0 and source row r goes to row slot_map[r]; tombstoned slots are
  // skipped and counted (once per row) in *n_dead.
  const int groups = dpad >> 3;
  const int64_t total = n_rows * groups;
  for (int64_t g = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; g < total;
       g += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t srow = g / groups;
    const int c0 = static_cast<int>(g - srow * groups) << 3;
    const SrcT* s = src + srow * d + c0;
    int64_t row = srow;
    if (slot_map != nullptr) {
      row = slot_map[srow];
      if ((dead_bits[row >> 5] >> (row & 31)) & 1u) {
        if (c0 == 0) atomicAdd(n_dead, 1);
        continue;
      }
    }
    uint16_t o[8];
    if (c0 >= d) {
      // pad columns (the row pitch is a whole number of 128-byte lines): zeros, and nothing to read
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = 0;
    } else if constexpr (kIsSplit<XT>) {
      // RBK_INDEX_KEEP_F32_SPLIT: the scan copy by the split rule (rbk_internal.h) and the low half beside it; a bf16
      // source is its own scan copy, with a zero low half.  dst_f64 null: only the scan copy (a tier change into the
      // split re-derives it from float32-exact rows).
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        o[j] = 0;
        if (c0 + j < d) {
          uint32_t u;
          if constexpr (sizeof(SrcT) == 8) u = __float_as_uint(__double2float_rn(static_cast<double>(s[j])));
          else if constexpr (sizeof(SrcT) == 4) u = __float_as_uint(static_cast<float>(s[j]));
          else u = static_cast<uint32_t>(s[j]) << 16;
          o[j] = sizeof(SrcT) == 2 ? static_cast<uint16_t>(s[j]) : split_hi(u);
          if (dst_f64 != nullptr) dst_f64[row * d + c0 + j].bits = static_cast<uint16_t>(u & 0xFFFFu);
        }
      }
    } else if (aligned) {
      if constexpr (sizeof(SrcT) == 8) {
        const double2* s2 = reinterpret_cast<const double2*>(s);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const double2 v = __ldg(s2 + j);
          o[2 * j] = f64_to_bf16_bits(v.x);
          o[2 * j + 1] = f64_to_bf16_bits(v.y);
        }
      } else if constexpr (sizeof(SrcT) == 4) {
        const float4* s4 = reinterpret_cast<const float4*>(s);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const float4 v = __ldg(s4 + j);
          o[4 * j] = f32_to_bf16_bits(v.x);
          o[4 * j + 1] = f32_to_bf16_bits(v.y);
          o[4 * j + 2] = f32_to_bf16_bits(v.z);
          o[4 * j + 3] = f32_to_bf16_bits(v.w);
        }
      } else {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(s));
        *reinterpret_cast<uint4*>(o) = v;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        uint16_t b = 0;
        if (c0 + j < d) {
          if constexpr (sizeof(SrcT) == 8) b = f64_to_bf16_bits(static_cast<double>(s[j]));
          else if constexpr (sizeof(SrcT) == 4) b = f32_to_bf16_bits(static_cast<float>(s[j]));
          else b = static_cast<uint16_t>(s[j]);
        }
        o[j] = b;
      }
    }
    if constexpr (!kIsSplit<XT>) {
      if (dst_f64 != nullptr) {   // exact-source sidecar: the original values, widened to f64 (pitch d)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (c0 + j < d) {
            double x;
            if constexpr (sizeof(SrcT) == 8) x = static_cast<double>(s[j]);
            else if constexpr (sizeof(SrcT) == 4) x = static_cast<double>(static_cast<float>(s[j]));
            else x = static_cast<double>(__uint_as_float(static_cast<uint32_t>(s[j]) << 16));
            dst_f64[row * d + c0 + j] = static_cast<XT>(x);
          }
        }
      }
    }
    uint4 out;
    out.x = o[0] | (static_cast<uint32_t>(o[1]) << 16);
    out.y = o[2] | (static_cast<uint32_t>(o[3]) << 16);
    out.z = o[4] | (static_cast<uint32_t>(o[5]) << 16);
    out.w = o[6] | (static_cast<uint32_t>(o[7]) << 16);
    *reinterpret_cast<uint4*>(dst + row * dpad + c0) = out;
  }
}

template <typename SrcT>
__device__ __forceinline__ double src_to_f64(SrcT v) {   // exact widening of every source type
  if constexpr (sizeof(SrcT) == 8) return static_cast<double>(v);
  else if constexpr (sizeof(SrcT) == 4) return static_cast<double>(static_cast<float>(v));
  else return static_cast<double>(__uint_as_float(static_cast<uint32_t>(v) << 16));
}

// RBK_INDEX_SCAN_F16 rows (rbk_f16.cuh): the scale needs the row's largest finite magnitude before any element is
// converted, so one WARP owns a row - pass 1 reduces max |x| over the row (coalesced reads), pass 2 re-reads it (from
// L1 / L2) and writes the scaled fp16 row in 16-byte stores, plus the f64 sidecar, which such an index always keeps
// (dst_f64 null: the source IS the sidecar, when a tier change re-derives the scan copy from it).
// Same slot_map / dead_bits / n_dead contract as convert_rows_kernel.
constexpr int kF16ConvThreads = 256;
template <typename SrcT, typename XT>
__global__ void __launch_bounds__(kF16ConvThreads) convert_rows_f16_kernel(
    const SrcT* __restrict__ src, int64_t n_rows, int d, int dpad, uint16_t* __restrict__ dst,
    XT* __restrict__ dst_f64, const int64_t* __restrict__ slot_map, const unsigned int* __restrict__ dead_bits,
    int* __restrict__ n_dead) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = static_cast<int64_t>(gridDim.x) * (kF16ConvThreads / 32);
  for (int64_t srow = blockIdx.x * static_cast<int64_t>(kF16ConvThreads / 32) + (threadIdx.x >> 5); srow < n_rows;
       srow += warps) {
    int64_t row = srow;
    if (slot_map != nullptr) {
      row = slot_map[srow];
      if ((dead_bits[row >> 5] >> (row & 31)) & 1u) {
        if (lane == 0) atomicAdd(n_dead, 1);
        continue;
      }
    }
    const SrcT* s = src + srow * d;
    double amax = 0.0;
    for (int i = lane; i < d; i += 32) {
      const double a = fabs(src_to_f64(s[i]));
      if (a < INFINITY) amax = fmax(amax, a);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmax(amax, __shfl_xor_sync(0xFFFFFFFFu, amax, o));
    const int e = f16_scale_exp(amax);
    for (int c0 = lane * 8; c0 < dpad; c0 += 32 * 8) {
      uint16_t o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        o[j] = 0;
        if (c0 + j < d) {
          const double x = src_to_f64(s[c0 + j]);
          if (dst_f64 != nullptr) dst_f64[row * d + c0 + j] = static_cast<XT>(x);
          o[j] = f16_bits_flush(scale_pow2(x, e));
        }
      }
      uint4 out;
      out.x = o[0] | (static_cast<uint32_t>(o[1]) << 16);
      out.y = o[2] | (static_cast<uint32_t>(o[3]) << 16);
      out.z = o[4] | (static_cast<uint32_t>(o[5]) << 16);
      out.w = o[6] | (static_cast<uint32_t>(o[7]) << 16);
      *reinterpret_cast<uint4*>(dst + row * dpad + c0) = out;
    }
  }
}

__device__ __forceinline__ double bf16_bits_to_f64(uint32_t h) {
  return static_cast<double>(__uint_as_float(h << 16));
}

// ---- K3b: per-row norms.  The accumulation ORDER is part of the parity contract (norm2 must be the reference's
// normB, embedder.ts:180: index order, multiply then add), so each row is one sequential fp64 chain owned by one
// thread - but the chain must not wait on memory, and the loads must be coalesced.  A block of kNormRows threads
// (= rows) therefore stages a K-chunk of all its rows in shared memory with 16-byte loads in which consecutive
// lanes read consecutive 16-byte pieces of the SAME row (full 128-byte lines, every byte of the chunk requested
// exactly once, many loads in flight per thread), and only then does every thread walk its own row's chunk out
// of shared memory (row pitch = an odd number of 16-byte units: conflict-free).  Several blocks per SM overlap
// one block's staging with the others' arithmetic.  (Round 1 had one thread read its row straight from global
// memory: adjacent threads 2*dpad bytes apart, one dependent 16-byte load per 8 elements of the chain.)
// slot_map == nullptr: item i is row first_row + i.  slot_map != nullptr (bulk overwrite): item i is row
// slot_map[i]; items whose slot is tombstoned are skipped.
constexpr int kNormRows = 128;          // rows (= threads) per block
constexpr int kNormChunk = 128;         // bf16 elements per staged chunk (256 B per row)
constexpr int kNormPitch16 = kNormChunk / 8 + 1;   // 17 x 16 B per row in smem: odd -> conflict-free walks

// kF16: the rows are RBK_INDEX_SCAN_F16 fp16 bits (inv_norm is that of the stored, scaled values).
template <bool kF16>
__global__ void __launch_bounds__(kNormRows) row_norms_kernel(const uint16_t* __restrict__ rows_base,
                                                              const double* __restrict__ rows_f64_base,
                                                              const int64_t* __restrict__ slot_map,
                                                              const unsigned int* __restrict__ dead_bits,
                                                              int64_t first_row, int64_t n_items, int d, int dpad,
                                                              float* __restrict__ inv_norm_base,
                                                              double* __restrict__ norm2_base,
                                                              int* __restrict__ eps_c_max) {
  __shared__ uint4 s_chunk[kNormRows * kNormPitch16];
  __shared__ long long s_row[kNormRows];
  const int tid = threadIdx.x;
  const int64_t item0 = static_cast<int64_t>(blockIdx.x) * kNormRows;
  {
    const int64_t item = item0 + tid;
    long long row = -1;
    if (item < n_items) {
      row = slot_map ? slot_map[item] : first_row + item;
      if (dead_bits && ((dead_bits[row >> 5] >> (row & 31)) & 1u)) row = -1;   // tombstoned slots stay dead
    }
    s_row[tid] = row;
  }
  __syncthreads();
  const long long my_row = s_row[tid];
  double acc = 0.0, amax = 0.0;   // amax: largest |element| (a bf16 index's scan band, DESIGN.md §6)
  const int n16 = dpad >> 3;                         // 16-byte pieces per row
  constexpr int kPieces = kNormChunk / 8;            // 16-byte pieces per row and chunk; = pieces per thread and chunk
  // piece index i of a chunk -> (row i / len16, unit i % len16): consecutive lanes = consecutive units of a row;
  // all of a thread's 16 loads are in flight before the first is stored.  The sequential fp64 chain per row, which
  // the parity contract imposes, is what bounds this kernel.
  uint4 v[kPieces];
  auto load_chunk = [&](int c0) {
    const int len16 = n16 - c0 < kPieces ? n16 - c0 : kPieces;
#pragma unroll
    for (int u = 0; u < kPieces; ++u) {
      const int i = tid + u * kNormRows;
      v[u] = make_uint4(0u, 0u, 0u, 0u);
      if (i < kNormRows * len16) {
        const int rr = i / len16, un = i - rr * len16;
        const long long row = s_row[rr];
        if (row >= 0) v[u] = __ldg(reinterpret_cast<const uint4*>(rows_base + row * dpad) + c0 + un);
      }
    }
  };
  for (int c0 = 0; c0 < n16; c0 += kPieces) {
    const int len16 = n16 - c0 < kPieces ? n16 - c0 : kPieces;
    load_chunk(c0);
#pragma unroll
    for (int u = 0; u < kPieces; ++u) {
      const int i = tid + u * kNormRows;
      if (i < kNormRows * len16) {
        const int rr = i / len16, un = i - rr * len16;
        s_chunk[rr * kNormPitch16 + un] = v[u];
      }
    }
    __syncthreads();
    if (my_row >= 0) {
      const uint4* mine = s_chunk + tid * kNormPitch16;
      for (int g = 0; g < len16; ++g) {   // pad columns are zero: adding 0*0 is exact
        const uint4 w4 = mine[g];
        const uint32_t w[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const double lo = kF16 ? f16_bits_to_f64(w[j] & 0xFFFFu) : bf16_bits_to_f64(w[j] & 0xFFFFu);
          const double hi = kF16 ? f16_bits_to_f64(w[j] >> 16) : bf16_bits_to_f64(w[j] >> 16);
          acc = __dadd_rn(acc, __dmul_rn(lo, lo));
          acc = __dadd_rn(acc, __dmul_rn(hi, hi));
          if (!kF16) amax = fmax(amax, fmax(fabs(lo), fabs(hi)));
        }
      }
    }
    __syncthreads();
  }
  if (my_row < 0) return;
  const bool ok = acc > 0.0 && acc < INFINITY;
  inv_norm_base[my_row] = ok ? static_cast<float>(1.0 / sqrt(acc)) : __uint_as_float(0x7FC00000u);
  if (rows_f64_base == nullptr) {
    norm2_base[my_row] = acc;
    // a bf16 row the reference scores but the scan's bound does not cover: no first pass proves anything any more
    if (!kF16 && ok && !in_scan_band(amax)) atomicMax(eps_c_max, __float_as_int(kEpsOffBand));
  }
}

// Exact-source sidecar indexes (RBK_INDEX_KEEP_F64): norm2 comes from the f64 row (the reference's normB for
// the values it really stores), again as one sequential chain per row fed from shared memory, and the angle
// between the f64 row and its bf16 rounding - an upper bound on how far the scan's approximate cosine of this
// row can be from its true cosine, on top of the other error terms - is folded into *eps_c_max.
// kF16 (RBK_INDEX_SCAN_F16): the stored rows are fp16 scaled by 2^e, with e recomputed here from the f64 row (a first
// walk over it for max |x|); the angle folded in is that between x and h * 2^-e, measured in the scaled domain
// (x * 2^e - h: the same angle).  The row's liveness in the scan must stay what a bf16 index gives it, so that both
// tiers answer alike: a row whose bf16 rounding has a zero or non-finite norm (elements past float32's range, or all of
// them below bf16's) gets the NaN inv_norm and the corpus angle such a row gets in a bf16 index.
// XT: element type of the exact rows (float for RBK_INDEX_KEEP_F32), widened to double as it is staged.
constexpr int kNorm64Chunk = 32;        // doubles per staged chunk (256 B per row)
constexpr int kNorm64Pitch = kNorm64Chunk + 1;

__device__ __forceinline__ float angle_bound(double diff2, double n2) {
  float eps = 0.f;
  if (diff2 > 0.0) {
    const double ratio = (n2 > 0.0 && n2 < INFINITY) ? sqrt(diff2 / n2) * (1.0 + 1e-9) : 2.0;
    eps = static_cast<float>((ratio < 1.0 ? asin(ratio) : 3.2) * (1.0 + 1e-6));
    eps = nextafterf(eps, INFINITY);
  }
  return eps;
}

template <bool kF16, typename XT>
__global__ void __launch_bounds__(kNormRows) row_norms_f64_kernel(const uint16_t* __restrict__ rows_base,
                                                                  const XT* __restrict__ rows_f64_base,
                                                                  const int64_t* __restrict__ slot_map,
                                                                  const unsigned int* __restrict__ dead_bits,
                                                                  int64_t first_row, int64_t n_items, int d, int dpad,
                                                                  double* __restrict__ norm2_base,
                                                                  float* __restrict__ inv_norm_base,
                                                                  int* __restrict__ eps_c_max) {
  __shared__ double s_x[kNormRows * kNorm64Pitch];
  __shared__ uint16_t s_b[kNormRows * (kNorm64Chunk + 2)];
  __shared__ long long s_row[kNormRows];
  const int tid = threadIdx.x;
  const int64_t item0 = static_cast<int64_t>(blockIdx.x) * kNormRows;
  {
    const int64_t item = item0 + tid;
    long long row = -1;
    if (item < n_items) {
      row = slot_map ? slot_map[item] : first_row + item;
      if (slot_map && ((dead_bits[row >> 5] >> (row & 31)) & 1u)) row = -1;
    }
    s_row[tid] = row;
  }
  __syncthreads();
  const long long my_row = s_row[tid];
  int e = 0;
  if constexpr (kF16) {   // the row's scale: max |x| over the finite elements, staged like the walk below
    double amax = 0.0;
    for (int c0 = 0; c0 < d; c0 += kNorm64Chunk) {
      const int len = d - c0 < kNorm64Chunk ? d - c0 : kNorm64Chunk;
      for (int i = tid; i < kNormRows * len; i += kNormRows) {
        const int rr = i / len, el = i - rr * len;
        const long long row = s_row[rr];
        s_x[rr * kNorm64Pitch + el] = row >= 0 ? static_cast<double>(__ldg(rows_f64_base + row * d + c0 + el)) : 0.0;
      }
      __syncthreads();
      if (my_row >= 0)
        for (int i = 0; i < len; ++i) {
          const double a = fabs(s_x[tid * kNorm64Pitch + i]);
          if (a < INFINITY) amax = fmax(amax, a);
        }
      __syncthreads();
    }
    e = f16_scale_exp(amax);
  }
  double n2 = 0.0, diff2 = 0.0;
  double xmax = 0.0, bad = 0.0;     // largest finite |x|; 1 if some element is not finite
  double h2 = 0.0, hdiff2 = 0.0;    // kF16: ||x 2^e||^2 and ||x 2^e - h||^2 (any order: bounds only)
  bool b_nonzero = false, b_finite = true;   // kF16: the bf16 rounding of the row has a nonzero / finite norm
  for (int c0 = 0; c0 < d; c0 += kNorm64Chunk) {
    const int len = d - c0 < kNorm64Chunk ? d - c0 : kNorm64Chunk;
    for (int i = tid; i < kNormRows * len; i += kNormRows) {   // consecutive lanes = consecutive elements of a row
      const int rr = i / len, el = i - rr * len;
      const long long row = s_row[rr];
      double x = 0.0;
      uint16_t bq = 0;
      if (row >= 0) {
        if constexpr (kIsSplit<XT>) {   // the float32 row joined from its scan copy and its low half
          bq = __ldg(rows_base + row * dpad + c0 + el);
          x = split_f64(bq, __ldg(&rows_f64_base[row * d + c0 + el].bits));
        } else {
          x = static_cast<double>(__ldg(rows_f64_base + row * d + c0 + el));
          bq = __ldg(rows_base + row * dpad + c0 + el);
        }
      }
      s_x[rr * kNorm64Pitch + el] = x;
      s_b[rr * (kNorm64Chunk + 2) + el] = bq;
    }
    __syncthreads();
    if (my_row >= 0) {
      const double* mine = s_x + tid * kNorm64Pitch;
      const uint16_t* mb = s_b + tid * (kNorm64Chunk + 2);
      for (int i = 0; i < len; ++i) {
        const double v = mine[i];
        n2 = __dadd_rn(n2, __dmul_rn(v, v));   // the reference's normB for the f64 row
        if (fabs(v) < INFINITY) xmax = fmax(xmax, fabs(v));
        else bad = 1.0;
        if constexpr (kF16) {
          const double y = scale_pow2(v, e), t = y - f16_bits_to_f64(mb[i]);
          h2 += y * y;
          hdiff2 += t * t;
          const float vb = __bfloat162float(__float2bfloat16_rn(__double2float_rn(v)));   // what a bf16 index stores
          b_nonzero |= vb != 0.f;
          b_finite &= fabsf(vb) < INFINITY;
          const double eb = v - static_cast<double>(vb);
          diff2 += eb * eb;
        } else {
          const double eb = v - bf16_bits_to_f64(mb[i]);
          diff2 += eb * eb;
        }
      }
    }
    __syncthreads();
  }
  if (my_row < 0) return;
  norm2_base[my_row] = n2;
  float eps;
  if constexpr (kF16) {
    const bool bf16_live = b_nonzero && b_finite;
    if (!bf16_live) inv_norm_base[my_row] = __uint_as_float(0x7FC00000u);
    eps = bf16_live ? angle_bound(hdiff2, h2) : angle_bound(diff2, n2);
  } else {
    eps = angle_bound(diff2, n2);
  }
  // a row the reference scores (finite, not all zero) outside the scan band: its scan copy may be dead or its normB
  // may underflow or overflow, so no first pass on this index proves anything any more (DESIGN.md §6)
  if (bad == 0.0 && xmax > 0.0 && !in_scan_band(xmax)) eps = fmaxf(eps, kEpsOffBand);
  if (eps > 0.f) atomicMax(eps_c_max, __float_as_int(eps));   // non-negative floats order like ints
}

__global__ void tombstone_kernel(const int64_t* __restrict__ slots, int64_t n, int64_t n_rows,
                                 float* __restrict__ inv_norm, unsigned int* __restrict__ dead_bits,
                                 int* __restrict__ n_killed) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const int64_t s = slots[i];
  if (s < 0 || s >= n_rows) return;
  const unsigned int bit = 1u << (s & 31);
  const unsigned int old = atomicOr(dead_bits + (s >> 5), bit);
  if (!(old & bit)) {
    inv_norm[s] = __uint_as_float(0x7FC00000u);
    atomicAdd(n_killed, 1);
  }
}

__global__ void __launch_bounds__(256) find_not_f32_kernel(const double* __restrict__ src, int64_t n,
                                                           int* __restrict__ found) {
  bool bad = false;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const double x = src[i];
    bad |= x == x && static_cast<double>(__double2float_rn(x)) != x;
  }
  if (__any_sync(0xFFFFFFFFu, bad) && (threadIdx.x & 31) == 0) *found = 1;
}

template <typename SrcT, typename DstT>
__global__ void __launch_bounds__(256) convert_exact_kernel(const SrcT* __restrict__ src, DstT* __restrict__ dst,
                                                            int64_t n) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    dst[i] = static_cast<DstT>(src[i]);
}

// Out of the split: element i of row i / d is the float32 joined from its scan copy (pitch dpad) and its low half.
template <typename DstT>
__global__ void __launch_bounds__(256) join_exact_kernel(const F32Lo* __restrict__ src,
                                                         const uint16_t* __restrict__ rows, int d, int dpad,
                                                         DstT* __restrict__ dst, int64_t n) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t row = i / d;
    const float x = __uint_as_float(split_join(__ldg(rows + row * dpad + (i - row * d)), __ldg(&src[i].bits)));
    dst[i] = static_cast<DstT>(x);
  }
}

int grid_for(int64_t items, int threads, int max_blocks) {
  int64_t b = (items + threads - 1) / threads;
  if (b < 1) b = 1;
  if (b > max_blocks) b = max_blocks;
  return static_cast<int>(b);
}

}  // namespace

namespace {
template <typename XT>
cudaError_t convert_rows_typed(const void* src, int src_type, int64_t n_rows, int d, int dpad, uint16_t* dst_rows,
                               XT* dst_x, cudaStream_t stream, const int64_t* slot_map, const unsigned int* dead_bits,
                               int* n_dead, bool f16) {
  if constexpr (kIsSplit<XT>) {
    if (f16) return cudaErrorInvalidValue;   // the split's scan copy is bf16 by construction
  } else if (f16) {
    constexpr int rows_per_block = kF16ConvThreads / 32;
    int dev = 0, sms = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return e;
    const int grid = grid_for(n_rows, rows_per_block, sms * 8);
    if (src_type == 0)
      convert_rows_f16_kernel<double, XT><<<grid, kF16ConvThreads, 0, stream>>>(
          static_cast<const double*>(src), n_rows, d, dpad, dst_rows, dst_x, slot_map, dead_bits, n_dead);
    else if (src_type == 1)
      convert_rows_f16_kernel<float, XT><<<grid, kF16ConvThreads, 0, stream>>>(
          static_cast<const float*>(src), n_rows, d, dpad, dst_rows, dst_x, slot_map, dead_bits, n_dead);
    else
      convert_rows_f16_kernel<uint16_t, XT><<<grid, kF16ConvThreads, 0, stream>>>(
          static_cast<const uint16_t*>(src), n_rows, d, dpad, dst_rows, dst_x, slot_map, dead_bits, n_dead);
    return cudaGetLastError();
  }
  const int64_t total = n_rows * (dpad >> 3);
  int dev = 0, sms = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (e != cudaSuccess) return e;
  const int grid = grid_for(total, 256, sms * 16);   // grid-stride loop: 16 blocks per SM
  // vector loads need d % 8 == 0 (every 8-group starts 16-byte aligned) and an aligned base
  const bool aligned = (d & 7) == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0;
  if (src_type == 0)
    convert_rows_kernel<double, XT><<<grid, 256, 0, stream>>>(static_cast<const double*>(src), n_rows, d, dpad,
                                                              dst_rows, dst_x, aligned, slot_map, dead_bits, n_dead);
  else if (src_type == 1)
    convert_rows_kernel<float, XT><<<grid, 256, 0, stream>>>(static_cast<const float*>(src), n_rows, d, dpad,
                                                             dst_rows, dst_x, aligned, slot_map, dead_bits, n_dead);
  else
    convert_rows_kernel<uint16_t, XT><<<grid, 256, 0, stream>>>(static_cast<const uint16_t*>(src), n_rows, d, dpad,
                                                                dst_rows, dst_x, aligned, slot_map, dead_bits, n_dead);
  return cudaGetLastError();
}
}  // namespace

cudaError_t launch_convert_rows(const void* src, int src_type, int64_t n_rows, int d, int dpad, uint16_t* dst_rows,
                                void* dst_x, int x_elem, cudaStream_t stream, const int64_t* slot_map,
                                const unsigned int* dead_bits, int* n_dead, bool f16) {
  if (n_rows <= 0) return cudaSuccess;
  if (x_elem == 4)
    return convert_rows_typed(src, src_type, n_rows, d, dpad, dst_rows, static_cast<float*>(dst_x), stream, slot_map,
                              dead_bits, n_dead, f16);
  if (x_elem == 2)
    return convert_rows_typed(src, src_type, n_rows, d, dpad, dst_rows, static_cast<F32Lo*>(dst_x), stream, slot_map,
                              dead_bits, n_dead, f16);
  return convert_rows_typed(src, src_type, n_rows, d, dpad, dst_rows, static_cast<double*>(dst_x), stream, slot_map,
                            dead_bits, n_dead, f16);
}

cudaError_t launch_row_norms(const uint16_t* rows_base, const void* rows_x_base, int x_elem, int64_t first_row,
                             int64_t n_items, int d, int dpad, float* inv_norm_base, double* norm2_base, int* eps_c_max,
                             cudaStream_t stream, const int64_t* slot_map, const unsigned int* dead_bits, bool f16) {
  if (n_items <= 0) return cudaSuccess;
  if (f16 && rows_x_base == nullptr) return cudaErrorInvalidValue;   // the fp16 tier always keeps the exact rows
  // dead_bits without slot_map (a tier change): the exact-row kernel folds every row's angle in, tombstoned or not
  if (!slot_map && dead_bits && rows_x_base == nullptr) return cudaErrorInvalidValue;
  const unsigned blocks = static_cast<unsigned>((n_items + kNormRows - 1) / kNormRows);
  // the bf16 kernel only tests rows_f64_base for null
  const double* rows_f64_base = static_cast<const double*>(rows_x_base);
  if (f16)
    row_norms_kernel<true><<<blocks, kNormRows, 0, stream>>>(rows_base, rows_f64_base, slot_map, dead_bits, first_row,
                                                             n_items, d, dpad, inv_norm_base, norm2_base, eps_c_max);
  else
    row_norms_kernel<false><<<blocks, kNormRows, 0, stream>>>(rows_base, rows_f64_base, slot_map, dead_bits, first_row,
                                                              n_items, d, dpad, inv_norm_base, norm2_base, eps_c_max);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess || rows_x_base == nullptr) return e;
  const float* rows_f32_base = static_cast<const float*>(rows_x_base);
  if (x_elem == 2) {
    if (f16) return cudaErrorInvalidValue;
    row_norms_f64_kernel<false, F32Lo><<<blocks, kNormRows, 0, stream>>>(
        rows_base, static_cast<const F32Lo*>(rows_x_base), slot_map, dead_bits, first_row, n_items, d, dpad,
        norm2_base, inv_norm_base, eps_c_max);
  } else if (f16 && x_elem == 4)
    row_norms_f64_kernel<true, float><<<blocks, kNormRows, 0, stream>>>(rows_base, rows_f32_base, slot_map, dead_bits,
                                                                        first_row, n_items, d, dpad, norm2_base,
                                                                        inv_norm_base, eps_c_max);
  else if (f16)
    row_norms_f64_kernel<true, double><<<blocks, kNormRows, 0, stream>>>(rows_base, rows_f64_base, slot_map, dead_bits,
                                                                         first_row, n_items, d, dpad, norm2_base,
                                                                         inv_norm_base, eps_c_max);
  else if (x_elem == 4)
    row_norms_f64_kernel<false, float><<<blocks, kNormRows, 0, stream>>>(rows_base, rows_f32_base, slot_map, dead_bits,
                                                                         first_row, n_items, d, dpad, norm2_base,
                                                                         inv_norm_base, eps_c_max);
  else
    row_norms_f64_kernel<false, double><<<blocks, kNormRows, 0, stream>>>(rows_base, rows_f64_base, slot_map,
                                                                          dead_bits, first_row, n_items, d, dpad,
                                                                          norm2_base, inv_norm_base, eps_c_max);
  return cudaGetLastError();
}

cudaError_t launch_find_not_f32(const double* src, int64_t n, int* found, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  int dev = 0, sms = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (e != cudaSuccess) return e;
  find_not_f32_kernel<<<grid_for(n, 256, sms * 16), 256, 0, stream>>>(src, n, found);
  return cudaGetLastError();
}

cudaError_t launch_convert_exact(const void* src, int src_elem, void* dst, int dst_elem, int64_t n,
                                 cudaStream_t stream, const uint16_t* rows, int d, int dpad) {
  if (n <= 0) return cudaSuccess;
  int dev = 0, sms = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (e != cudaSuccess) return e;
  const int grid = grid_for(n, 256, sms * 16);
  if (src_elem == 2 && (rows == nullptr || d <= 0))
    return cudaErrorInvalidValue;
  else if (src_elem == 2 && dst_elem == 4)
    join_exact_kernel<float><<<grid, 256, 0, stream>>>(static_cast<const F32Lo*>(src), rows, d, dpad,
                                                       static_cast<float*>(dst), n);
  else if (src_elem == 2 && dst_elem == 8)
    join_exact_kernel<double><<<grid, 256, 0, stream>>>(static_cast<const F32Lo*>(src), rows, d, dpad,
                                                        static_cast<double*>(dst), n);
  else if (src_elem == 8 && dst_elem == 4)
    convert_exact_kernel<double, float><<<grid, 256, 0, stream>>>(static_cast<const double*>(src),
                                                                  static_cast<float*>(dst), n);
  else if (src_elem == 4 && dst_elem == 8)
    convert_exact_kernel<float, double><<<grid, 256, 0, stream>>>(static_cast<const float*>(src),
                                                                  static_cast<double*>(dst), n);
  else
    return cudaErrorInvalidValue;
  return cudaGetLastError();
}

cudaError_t launch_tombstone(const int64_t* dev_slots, int64_t n, int64_t n_rows, float* inv_norm,
                             unsigned int* dead_bits, int* n_killed, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  tombstone_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(dev_slots, n, n_rows, inv_norm,
                                                                              dead_bits, n_killed);
  return cudaGetLastError();
}

}  // namespace rbk
