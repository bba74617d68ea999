// rbk_finalize.cu — everything around the fused scan that makes the result EXACT:
//   prep_queries   : per query  bf16 copy for the scan, fp64 copy + exact ||q||^2 (the
//                    reference's `normA`, embedder.ts:175-180), error bound, start threshold
//   finalize       : K2 (select the k' best approximate candidates of a query across the
//                    per-CTA lists) + K4 (re-score them in fp64 in the reference's exact
//                    operation order, embedder.ts:173-183) + the final ordering of
//                    VectorStore.search (score desc, stable = slot asc; `>= minScore`;
//                    vector-store.ts:212,218,221) + the proof that no other row can belong
//                    to the answer
//   exact fallback : K0, exhaustive fp64 scan for the (rare) queries whose proof failed
//   merge_shards   : merge of per-GPU result lists after the all-gather (SURVEY.md §8e)
#include <cuda_bf16.h>
#include <limits.h>

#include <type_traits>

#include "rbk_f16.cuh"
#include "rbk_internal.h"
#include "rbk_ptx.cuh"

namespace rbk {

namespace {

constexpr uint32_t kFull = 0xFFFFFFFFu;

__device__ __forceinline__ double bf16_to_f64(uint32_t h) { return static_cast<double>(__uint_as_float(h << 16)); }

// dot(q, row) accumulated in index order, multiply then add, no FMA (embedder.ts:177-178).
__device__ __forceinline__ double exact_dot(const double* __restrict__ q, const uint16_t* __restrict__ row, int d) {
  double dot = 0.0;
  const uint4* p = reinterpret_cast<const uint4*>(row);
  int i = 0;
  for (; i + 8 <= d; i += 8) {
    const uint4 v = __ldg(p + (i >> 3));
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      dot = __dadd_rn(dot, __dmul_rn(__ldg(q + i + 2 * j), bf16_to_f64(w[j] & 0xFFFFu)));
      dot = __dadd_rn(dot, __dmul_rn(__ldg(q + i + 2 * j + 1), bf16_to_f64(w[j] >> 16)));
    }
  }
  for (; i < d; ++i) dot = __dadd_rn(dot, __dmul_rn(__ldg(q + i), bf16_to_f64(row[i])));
  return dot;
}
// One exact-row element widened to double.  x: the element; hi: the same element of the scan copy, which only the split
// (F32Lo, x_elem 2) reads - it holds the high half of the float32.
template <typename XT>
__device__ __forceinline__ double ldx(const XT* x, const uint16_t* hi) {
  return static_cast<double>(__ldg(x));
}
__device__ __forceinline__ double ldx(const F32Lo* x, const uint16_t* hi) {
  return split_f64(__ldg(hi), __ldg(&x->bits));
}
// same, exact-source row of float64, float32 or split float32 elements (widened on load: the same operands either way);
// hi: the row of the scan copy
template <typename XT>
__device__ __forceinline__ double exact_dot_f64(const double* __restrict__ q, const XT* __restrict__ row, int d,
                                                const uint16_t* __restrict__ hi) {
  double dot = 0.0;
  for (int i = 0; i < d; ++i) dot = __dadd_rn(dot, __dmul_rn(__ldg(q + i), ldx(row + i, hi + i)));
  return dot;
}
// The split's rows are read eight elements at a time, one 16-byte load from each half (the rows start 16-byte aligned
// when d % 8 == 0; the scan copy's always do): a thread walking its own row issues an eighth of the loads.  Same chain.
__device__ __forceinline__ double exact_dot_f64(const double* __restrict__ q, const F32Lo* __restrict__ row, int d,
                                                const uint16_t* __restrict__ hi) {
  double dot = 0.0;
  int i = 0;
  if ((d & 7) == 0) {
    const uint4* lp = reinterpret_cast<const uint4*>(row);
    const uint4* hp = reinterpret_cast<const uint4*>(hi);
    for (; i < d; i += 8) {
      const uint4 l = __ldg(lp + (i >> 3)), h = __ldg(hp + (i >> 3));
      const uint32_t lw[4] = {l.x, l.y, l.z, l.w}, hw[4] = {h.x, h.y, h.z, h.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        dot = __dadd_rn(dot, __dmul_rn(__ldg(q + i + 2 * j), split_f64(hw[j] & 0xFFFFu, lw[j] & 0xFFFFu)));
        dot = __dadd_rn(dot, __dmul_rn(__ldg(q + i + 2 * j + 1), split_f64(hw[j] >> 16, lw[j] >> 16)));
      }
    }
  }
  for (; i < d; ++i) dot = __dadd_rn(dot, __dmul_rn(__ldg(q + i), ldx(row + i, hi + i)));
  return dot;
}
// two exact-row elements per load: 16 bytes of float64, 8 of float32, 4 of low halves (plus 4 of the scan copy)
template <typename XT>
using Pair = typename std::conditional<sizeof(XT) == 8, double2,
                                       typename std::conditional<sizeof(XT) == 4, float2, ushort2>::type>::type;
__device__ __forceinline__ double2 widen2(double2 v) { return v; }
__device__ __forceinline__ double2 widen2(float2 v) { return make_double2(v.x, v.y); }
__device__ __forceinline__ double2 ldx2(const double2* x, const uint16_t*) { return widen2(__ldg(x)); }
__device__ __forceinline__ double2 ldx2(const float2* x, const uint16_t*) { return widen2(__ldg(x)); }
__device__ __forceinline__ double2 ldx2(const ushort2* x, const uint16_t* hi) {
  const ushort2 r = __ldg(x), s = __ldg(reinterpret_cast<const ushort2*>(hi));
  return make_double2(split_f64(s.x, r.x), split_f64(s.y, r.y));
}
// embedder.ts:183  dotProduct / (Math.sqrt(normA) * Math.sqrt(normB))
__device__ __forceinline__ double exact_cosine(double dot, double na, double nb) {
  return __ddiv_rn(dot, __dmul_rn(__dsqrt_rn(na), __dsqrt_rn(nb)));
}

// --------------------------------------------------------------------------- prep
// kNorm2: also compute the reference's normA (one SEQUENTIAL fp64 chain over d elements, ~30 cycles each: 12 us
// at d = 768).  A search does not need it here: only the finalize kernel reads it, and computes it itself on an
// otherwise idle thread beside the candidates' dot chains - so the chain left the critical path of every search.
// The exact-scores path, which has no finalize, asks for it.
// scratch (nullable): the per-launch scan scratch of the FIRST sub-batch - hist [Bs][kHistBins] | maxbin [Bs] |
// gthr [Bs] | progress [n_progress] - zeroed here, one row per query block, instead of by a separate memset node.
// kF16 (RBK_INDEX_SCAN_F16): the scan's copy is the query scaled by its own power of two and rounded to fp16 (the rule
// of rbk_f16.cuh, applied to the f64 query, or to the f32 one widened exactly); q_inv_norm = 1/||h|| (so it carries
// the scale) and the angle in q_eps is that of h.  The query stays live or dead (q_inv_norm NaN, thr_init +inf) exactly
// as in a bf16 index, so that the two tiers take the same decisions on zero, tiny or huge queries.
// kEach: the start threshold comes from the query's own min_each[q] (rbk_index_search_each_f64) instead of min_score.
template <typename SrcT, bool kNorm2, bool kF16, bool kEach = false>
__global__ void __launch_bounds__(128) prep_queries_kernel(const SrcT* __restrict__ src, int d, int dpad,
                                                           double min_score, double acc_eps,
                                                           const float* __restrict__ eps_c, QueryBuffers qb,
                                                           unsigned int* __restrict__ scratch, int Bs, int n_progress,
                                                           const double* __restrict__ min_each) {
  const int q = blockIdx.x;
  const int tid = threadIdx.x;
  if (scratch != nullptr && q < Bs) {
    uint4* row = reinterpret_cast<uint4*>(scratch + static_cast<size_t>(q) * kHistBins);
    for (int i = tid; i < kHistBins / 4; i += blockDim.x) row[i] = make_uint4(0u, 0u, 0u, 0u);
    unsigned int* tail = scratch + static_cast<size_t>(Bs) * kHistBins;
    if (tid == 0) {
      tail[q] = 0u;        // maxbin
      tail[Bs + q] = 0u;   // gthr
    }
    if (q == 0)
      for (int i = tid; i < n_progress; i += blockDim.x) tail[2 * Bs + i] = 0u;
  }
  const SrcT* s = src + static_cast<size_t>(q) * d;
  int e = 0;   // kF16: the query's scale exponent
  if constexpr (kF16) {
    __shared__ double red_m[4];
    double amax = 0.0;
    for (int i = tid; i < d; i += blockDim.x) {
      const double a = fabs(static_cast<double>(__ldg(s + i)));
      if (a < INFINITY) amax = fmax(amax, a);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmax(amax, __shfl_xor_sync(kFull, amax, o));
    if ((tid & 31) == 0) red_m[tid >> 5] = amax;
    __syncthreads();
    e = f16_scale_exp(fmax(fmax(red_m[0], red_m[1]), fmax(red_m[2], red_m[3])));
  }
  double sb = 0.0, sd = 0.0, sq = 0.0;  // ||bf16(q)||^2, ||q - bf16(q)||^2, ||q||^2 (any order: bounds only)
  double fmx = 0.0, bad = 0.0;           // max |x| over the finite elements; 1 if any element is not finite
  double sh = 0.0, shd = 0.0, sx = 0.0; // kF16: ||h||^2, ||q 2^e - h||^2, ||q 2^e||^2 (any order: bounds only)
  // 8 elements per thread and pass, ALL loads first: the stores below may alias the source as far as the compiler
  // knows, so a load -> store loop exposed one global round trip per element (the kernel took 7.8 us for this)
  for (int i0 = tid; i0 < dpad; i0 += 8 * blockDim.x) {
    double xs[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int i = i0 + u * blockDim.x;
      xs[u] = i < d ? static_cast<double>(__ldg(s + i)) : 0.0;
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int i = i0 + u * blockDim.x;
      if (i >= dpad) continue;
      uint16_t b = 0;
      if (i < d) {
        const double x = xs[u];
        qb.q_f64[static_cast<size_t>(q) * d + i] = x;
        if (fabs(x) < INFINITY) fmx = fmax(fmx, fabs(x));
        else bad = 1.0;
        const __nv_bfloat16 h = __float2bfloat16_rn(__double2float_rn(x));
        b = __bfloat16_as_ushort(h);
        const double xb = static_cast<double>(__bfloat162float(h));
        sb += xb * xb;
        sd += (x - xb) * (x - xb);
        sq += x * x;
        if constexpr (kF16) {
          const double y = scale_pow2(x, e);
          b = f16_bits_flush(y);
          const double yh = f16_bits_to_f64(b);
          sh += yh * yh;
          shd += (y - yh) * (y - yh);
          sx += y * y;
        }
      }
      qb.q_bf16[static_cast<size_t>(q) * dpad + i] = b;
    }
  }
  __shared__ double red_b[4], red_d[4], red_m2[4], red_bad[4];
  __shared__ double red_h[4], red_hd[4], red_x[4];
  __shared__ double s_na;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sb += __shfl_xor_sync(kFull, sb, o);
    sd += __shfl_xor_sync(kFull, sd, o);
    fmx = fmax(fmx, __shfl_xor_sync(kFull, fmx, o));
    bad = fmax(bad, __shfl_xor_sync(kFull, bad, o));
    if constexpr (kF16) {
      sh += __shfl_xor_sync(kFull, sh, o);
      shd += __shfl_xor_sync(kFull, shd, o);
      sx += __shfl_xor_sync(kFull, sx, o);
    }
  }
  if ((tid & 31) == 0) {
    red_b[tid >> 5] = sb;
    red_d[tid >> 5] = sd;
    red_m2[tid >> 5] = fmx;
    red_bad[tid >> 5] = bad;
    if constexpr (kF16) {
      red_h[tid >> 5] = sh;
      red_hd[tid >> 5] = shd;
      red_x[tid >> 5] = sx;
    }
  }
  // the reference's normA: index order, multiply then add.  The chain is sequential by contract, so its
  // operands are staged in smem first (a dependent global load per element cost ~23 ns each).
  __shared__ double s_x[512];
  double na = 0.0;
  if (kNorm2) {
    for (int c0 = 0; c0 < d; c0 += 512) {
      const int len = d - c0 < 512 ? d - c0 : 512;
      __syncthreads();
      for (int i = tid; i < len; i += blockDim.x) s_x[i] = static_cast<double>(s[c0 + i]);
      __syncthreads();
      if (tid == 0)
        for (int i = 0; i < len; ++i) na = __dadd_rn(na, __dmul_rn(s_x[i], s_x[i]));
    }
  } else {
    // any-order sum of squares of the f64 query (accumulated above): only its sign/finiteness and the ratio below
    // (bounds) are used
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(kFull, sq, o);
    __shared__ double red_q[4];
    if ((tid & 31) == 0) red_q[tid >> 5] = sq;
    __syncthreads();
    na = red_q[0] + red_q[1] + red_q[2] + red_q[3];
  }
  if (tid == 0) s_na = na;
  __syncthreads();
  if (tid == 0) {
    const double na = s_na;
    const double nb2 = red_b[0] + red_b[1] + red_b[2] + red_b[3];
    const double nd2 = red_d[0] + red_d[1] + red_d[2] + red_d[3];
    const bool ok = nb2 > 0.0 && nb2 < INFINITY && na > 0.0 && na < INFINITY;
    // A query the reference scores (finite, not all zero) whose largest element lies outside the scan band is left
    // to the exhaustive kernel (DESIGN.md §6): its bf16 copy may be zero or infinite, its fp32 products may leave
    // fp32's range, its normA may underflow or overflow.  Inside the band none of that happens, and ok holds.
    const double qmax = fmax(fmax(red_m2[0], red_m2[1]), fmax(red_m2[2], red_m2[3]));
    const bool ref_live = fmax(fmax(red_bad[0], red_bad[1]), fmax(red_bad[2], red_bad[3])) == 0.0 && qmax > 0.0;
    const bool off_band = ref_live && !in_scan_band(qmax);
    double inv = ok ? 1.0 / sqrt(nb2) : 0.0;
    // angle(q, bf16(q)) <= asin(||q - bf16(q)|| / ||q||); cosine is 1-Lipschitz in the angle
    double ang = 0.0;
    if (ok && nd2 > 0.0) {
      const double ratio = sqrt(nd2 / na) * (1.0 + 1e-9) * (kNorm2 ? 1.0 : 1.0 + 1e-12 * d);   // any-order sum: widen

      ang = ratio < 1.0 ? asin(ratio) * (1.0 + 1e-9) : 3.2;
    }
    if constexpr (kF16) {
      // the same bound for h * 2^-e, measured in the scaled domain (the angle does not depend on the scale); a live
      // query has a finite nonzero bf16 norm, so its h (the largest element in [2^14, 2^15]) has one too
      const double nh2 = red_h[0] + red_h[1] + red_h[2] + red_h[3];
      const double nhd2 = red_hd[0] + red_hd[1] + red_hd[2] + red_hd[3];
      const double nx2 = red_x[0] + red_x[1] + red_x[2] + red_x[3];
      inv = ok ? 1.0 / sqrt(nh2) : 0.0;
      ang = 0.0;
      if (ok && nhd2 > 0.0) {
        const double ratio = sqrt(nhd2 / nx2) * (1.0 + 1e-9) * (1.0 + 1e-12 * d);   // any-order sums: widen
        ang = ratio < 1.0 ? asin(ratio) * (1.0 + 1e-9) : 3.2;
      }
    }
    // + corpus-side quantisation angle when the exact source is an f64 sidecar (0 for bf16-exact corpora)
    const double eps = off_band ? INFINITY
                                : acc_eps + ang + (eps_c != nullptr ? static_cast<double>(*eps_c) * (1.0 + 1e-6) : 0.0);
    if (kNorm2) qb.q_norm2[q] = na;   // (else: written by the finalize kernel, bit-exact)
    qb.q_eps[q] = eps;
    const float invf = ok ? static_cast<float>(inv) : __uint_as_float(0x7FC00000u);
    qb.q_inv_norm[q] = invf;
    const double min_q = kEach ? min_each[q] : min_score;
    float thr;
    if (!ok || !(eps < kEpsNone)) {
      // zero / non-finite query: cosine is NaN for every row (S3) -> nothing matches; or a bound that proves
      // nothing: the scan is skipped and the query is answered exactly (finalize flags it, large_select emits all)
      thr = INFINITY;
    } else if (min_q == -INFINITY) {
      thr = -INFINITY;
    } else {
      // a row can only reach min_score if approx > min_score - eps; go to the raw domain
      // (divide by inv_norm_q) and step two ulps down so rounding never hides a row.
      const double raw = (min_q - eps) / static_cast<double>(invf);
      float t = static_cast<float>(raw);
      t = nextafterf(nextafterf(t, -INFINITY), -INFINITY);
      thr = t;
    }
    qb.thr_init[q] = thr;
  }
}

// --------------------------------------------------------------------------- finalize
constexpr int kFinThreads = 256;

constexpr int kQChunk = 512;    // query elements staged per re-rank chunk
// Candidate keys of one query are staged in dynamic smem (key_cap keys, chosen per launch: large for few
// queries, small for many so that 8 blocks fit an SM); a query with more keys streams them from L2.

// Visit every candidate key of one query: from the smem staging buffer when it holds them all,
// else straight from the per-unit lists (qb, r, qrow), r in [0, R), in L2.
template <typename F>
__device__ __forceinline__ void for_each_key(const unsigned long long* __restrict__ cand, const int* s_cnt,
                                             const unsigned long long* s_keys, int M, bool staged, int R, int qb,
                                             int qrow, int block_m, F&& f) {
  if (staged) {
    for (int i = threadIdx.x; i < M; i += kFinThreads) f(s_keys[i]);
    return;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r = warp; r < R; r += kFinThreads / 32) {
    const unsigned long long* l =
        cand + (static_cast<size_t>(qb * R + r) * block_m + qrow) * static_cast<size_t>(kListCap);
    const int c = s_cnt[r];
    for (int i = lane; i < c; i += 32) f(__ldcg(l + i));
  }
}

// Host-row staging (kHostRows): row pieces each thread keeps in flight.  A mapped host read waits a PCIe round trip,
// so a block needs many bytes in flight to stream: 256 threads x 8 x 16 B = 32 KB.
constexpr int kHostLoads = 8;

// kHostRows: rows_x is mapped host memory (RBK_INDEX_ROWS_ON_HOST).  Only the exact-row staging differs; the device-tier
// instantiation compiles to the same code as before the host tier existed.  XT: the exact rows' element type (float
// for RBK_INDEX_KEEP_F32), widened to double as it is staged, so the chains below see the same operands.
// kEach: the query's cut and threshold come from p.k_each / p.min_each (rbk_index_search_each_f64); p.k_fetch is the
// row stride.  The scalar instantiations read neither array.
template <bool kHostRows, typename XT, bool kEach>
__device__ __forceinline__ void finalize_rows(const FinalizeParams& p) {
  const int ql = blockIdx.x;  // query index inside this launch
  const int tid = threadIdx.x;
  const int qb = ql / p.block_m, qrow = ql % p.block_m;

  __shared__ int s_cnt[160];
  __shared__ int s_off[161];
  extern __shared__ __align__(16) unsigned long long s_keys[];   // p.key_cap keys; later the re-rank's row chunks
  __shared__ unsigned int s_hist[256];
  __shared__ unsigned long long s_sel[kMaxKPrime];
  __shared__ double s_score[kMaxKPrime];
  __shared__ int s_row[kMaxKPrime];
  __shared__ int s_valid[kMaxKPrime];
  __shared__ int s_total, s_nsel, s_nvalid, s_bin, s_want, s_done;
  __shared__ unsigned long long s_prefix, s_minkey;
  __shared__ double s_ekth;

  if (tid == 0) {
    s_total = 0;
    s_nsel = 0;
    s_nvalid = 0;
    s_ekth = 0.0;
    s_done = 0;
    s_minkey = ~0ull;
  }
  __syncthreads();
  int local = 0;
  for (int r = tid; r < p.R; r += kFinThreads) {
    const int c = p.cand_cnt[(qb * p.R + r) * p.block_m + qrow];
    s_cnt[r] = c;
    local += c;
  }
  if (local) atomicAdd(&s_total, local);
  __syncthreads();
  const int M = s_total;
  const int kprime = p.kprime;
  // Stage the query's keys in smem with every load in flight at once: flat key index ->
  // (list, offset) by binary search in the prefix sums.  (Walking the lists one after the
  // other costs one L2 round trip per list and pass: 60-125 us per block, measured.)
  const bool staged = M <= p.key_cap;
  if (staged) {
    if (tid < 32) {   // exclusive scan of up to 160 counts, 5 per lane
      int v[5], sum = 0;
#pragma unroll
      for (int j = 0; j < 5; ++j) {
        const int r = tid * 5 + j;
        v[j] = r < p.R ? s_cnt[r] : 0;
        sum += v[j];
      }
      int incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(kFull, incl, o);
        if (tid >= o) incl += t;
      }
      int run = incl - sum;
#pragma unroll
      for (int j = 0; j < 5; ++j) {
        const int r = tid * 5 + j;
        if (r <= p.R) s_off[r] = run;
        run += v[j];
      }
    }
    __syncthreads();
    // four independent loads in flight per thread (a load -> store loop exposes one L2 round trip per key)
    for (int i0 = tid; i0 < M; i0 += 4 * kFinThreads) {
      unsigned long long kv[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + u * kFinThreads;
        kv[u] = 0ull;
        if (i < M) {
          int lo = 0, hi = p.R - 1;   // last r with s_off[r] <= i
          while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (s_off[mid] <= i) lo = mid;
            else hi = mid - 1;
          }
          const unsigned long long* l =
              p.cand + (static_cast<size_t>(qb * p.R + lo) * p.block_m + qrow) * static_cast<size_t>(kListCap);
          kv[u] = __ldcg(l + (i - s_off[lo]));
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + u * kFinThreads;
        if (i < M) s_keys[i] = kv[u];
      }
    }
    __syncthreads();
  }

  // ---- K2: radix select of the k'-th largest 64-bit key (keys are unique) ----
  unsigned long long pivot = 0ull;
  if (M >= kprime) {
    if (tid == 0) {
      s_prefix = 0ull;
      s_want = kprime;
    }
    unsigned long long mask = 0ull;
    for (int pass = 7; pass >= 0; --pass) {
      const int shift = pass * 8;
      s_hist[tid] = 0u;
      __syncthreads();
      const unsigned long long prefix = s_prefix;
      for_each_key(p.cand, s_cnt, s_keys, M, staged, p.R, qb, qrow, p.block_m, [&](unsigned long long k) {
        if ((k & mask) == prefix) atomicAdd(&s_hist[static_cast<unsigned>(k >> shift) & 255u], 1u);
      });
      __syncthreads();
      if (tid < 32) {
        // lane L owns bins [255-8L-7, 255-8L]; scan from the top bin down
        const int top = 255 - 8 * tid;
        unsigned int mine = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) mine += s_hist[top - j];
        unsigned int incl = mine;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const unsigned int v = __shfl_up_sync(kFull, incl, o);
          if (tid >= o) incl += v;
        }
        const unsigned int want = static_cast<unsigned int>(s_want);
        const bool crosses = (incl >= want) && (incl - mine < want);
        if (crosses) {
          unsigned int cum = incl - mine;
          int b = top;
          for (int j = 0; j < 8; ++j, --b) {
            const unsigned int h = s_hist[b];
            if (cum + h >= want) break;
            cum += h;
          }
          s_bin = b;
          s_want = static_cast<int>(want - cum);
          // every key left in this bin is wanted: the bin's lower edge is already a valid pivot
          s_done = (s_hist[b] == want - cum) ? 1 : 0;
        }
      }
      __syncthreads();
      if (tid == 0) s_prefix = prefix | (static_cast<unsigned long long>(s_bin) << shift);
      mask |= 0xFFull << shift;
      __syncthreads();
      if (s_done) break;   // uniform: read after the barrier
    }
    pivot = s_prefix;
  }
  for_each_key(p.cand, s_cnt, s_keys, M, staged, p.R, qb, qrow, p.block_m, [&](unsigned long long k) {
    if (k >= pivot) {
      const int pos = atomicAdd(&s_nsel, 1);
      if (pos < kMaxKPrime) s_sel[pos] = k;
      atomicMin(&s_minkey, k);   // the k'-th best key itself (the pivot may be only a bin edge after an early exit)
    }
  });
  __syncthreads();
  const int nsel = s_nsel < kMaxKPrime ? s_nsel : kMaxKPrime;
  // every row that is NOT a candidate has raw score <= tau_raw (or was cut by thr_init)
  const float tau_raw = M >= kprime ? key_score(s_minkey) : -INFINITY;

  // ---- K4: exact fp64 re-score of the candidates ----
  // The arithmetic is a sequential chain per candidate (parity contract), so global-load latency
  // must not sit inside it: all threads stage a K-chunk of every candidate row (and of the query)
  // into smem with the loads in flight together, then each candidate's thread walks its chunk.
  // The key staging buffer is dead by now (selection is in s_sel) and is reused for the rows.
  // Cycle stamps (a clock64 probe build, round 2; 625k-row shard, B=256, d=768, 32 candidates): this phase is
  // 26 k of the block's 44 k cycles = 34 cycles per element for conversion + DMUL + DADD in one warp.  Three
  // rearrangements of the same operations were measured and ALL lost: widening bf16 -> binary64 with integer
  // instructions instead of F2F (51 k cycles), forming the next group's 8 products ahead of the current group's
  // 8 dependent adds by hand (38 k), and letting all 256 threads form the products into shared memory so that the
  // chain thread only adds (65 k with 16-byte row loads, 110 k element-wise).  Whatever issues them, fp64-pipe
  // instructions cost this kernel 11-27 cycles each; the loop below issues the fewest.
  // The reference's normA (embedder.ts:179: index order, multiply then add) is one more sequential fp64 chain over
  // the query.  The last thread of the block - idle, at most kMaxKPrime threads carry candidates - walks it over the
  // same staged query chunks the candidates' dot chains read, so it costs the search nothing.
  __shared__ double s_na;
  double na_chain = 0.0;
  const double* qv = p.q.q_f64 + static_cast<size_t>(ql) * p.d;
  __shared__ double s_q[kQChunk];
  unsigned char* s_rows = reinterpret_cast<unsigned char*>(s_keys);
  int my_row = 0;
  double dot = 0.0;
  if (tid < nsel) my_row = static_cast<int>(key_row(s_sel[tid]));
  if (p.rows_x == nullptr) {
    int chunk = nsel > 0 ? ((p.key_cap * 8 / nsel - 16) / 2) & ~7 : kQChunk;
    chunk = chunk < kQChunk ? chunk : kQChunk;
    const int chunk16 = chunk >> 3;                                   // 16-byte units per row chunk
    const int row_stride = (chunk16 | 1) << 4;                        // odd number of 16-B units: conflict-free walks
    for (int c0 = 0; c0 < p.d; c0 += chunk) {
      const int len = p.d - c0 < chunk ? p.d - c0 : chunk;            // elements of this chunk
      const int len16 = (len + 7) >> 3;                               // rows are zero padded to dpad (multiple of 8)
      __syncthreads();                                                // previous chunk fully consumed
      for (int i0 = tid; i0 < nsel * len16; i0 += 4 * kFinThreads) {   // 4 row pieces in flight per thread
        uint4 pv[4];
#pragma unroll
        for (int b = 0; b < 4; ++b) {
          const int i = i0 + b * kFinThreads;
          pv[b] = make_uint4(0u, 0u, 0u, 0u);
          if (i < nsel * len16) {
            const int rr = i / len16, u = i - rr * len16;
            const int row = static_cast<int>(key_row(s_sel[rr]));
            pv[b] = __ldg(reinterpret_cast<const uint4*>(p.rows + static_cast<size_t>(row) * p.dpad + c0) + u);
          }
        }
#pragma unroll
        for (int b = 0; b < 4; ++b) {
          const int i = i0 + b * kFinThreads;
          if (i < nsel * len16) {
            const int rr = i / len16, u = i - rr * len16;
            *reinterpret_cast<uint4*>(s_rows + rr * row_stride + u * 16) = pv[b];
          }
        }
      }
      for (int i = tid; i < len; i += kFinThreads) s_q[i] = __ldg(qv + c0 + i);
      __syncthreads();
      if (tid < nsel) {
        const unsigned char* mine = s_rows + tid * row_stride;
        int i = 0;
        for (; i + 8 <= len; i += 8) {
          const uint4 v = *reinterpret_cast<const uint4*>(mine + i * 2);
          const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            dot = __dadd_rn(dot, __dmul_rn(s_q[i + 2 * j], bf16_to_f64(w[j] & 0xFFFFu)));
            dot = __dadd_rn(dot, __dmul_rn(s_q[i + 2 * j + 1], bf16_to_f64(w[j] >> 16)));
          }
        }
        for (; i < len; ++i)
          dot = __dadd_rn(dot, __dmul_rn(s_q[i], bf16_to_f64(reinterpret_cast<const uint16_t*>(mine)[i])));
      }
      if (tid == kFinThreads - 1)
        for (int i = 0; i < len; ++i) na_chain = __dadd_rn(na_chain, __dmul_rn(s_q[i], s_q[i]));
    }
  } else if constexpr (kHostRows) {
    // exact source = f64 rows in mapped host memory: the same chunks walked in the same order, but staged with
    // 16-byte loads, kHostLoads of them in flight per thread (8-byte ones for odd d, whose rows are not all 16-byte
    // aligned).  The chunk is even so that every 16-byte piece of an even-d row starts aligned.
    const XT* rows_x = static_cast<const XT*>(p.rows_x);
    double* s_rows64 = reinterpret_cast<double*>(s_keys);
    int chunk = nsel > 0 ? (p.key_cap / nsel - 1) : kQChunk;
    chunk = (chunk < kQChunk ? chunk : kQChunk) & ~1;
    const int row_stride = chunk | 1;
    const bool wide = (p.d & 1) == 0;
    for (int c0 = 0; c0 < p.d; c0 += chunk) {
      const int len = p.d - c0 < chunk ? p.d - c0 : chunk;
      __syncthreads();
      if (wide) {
        const int len2 = len >> 1;   // even d, even chunk: len is even
        for (int i0 = tid; i0 < nsel * len2; i0 += kHostLoads * kFinThreads) {
          double2 v[kHostLoads];
#pragma unroll
          for (int b = 0; b < kHostLoads; ++b) {
            const int i = i0 + b * kFinThreads;
            if (i < nsel * len2) {
              const int rr = i / len2, u = i - rr * len2;
              const int row = static_cast<int>(key_row(s_sel[rr]));
              v[b] = ldx2(reinterpret_cast<const Pair<XT>*>(rows_x + static_cast<size_t>(row) * p.d + c0) + u,
                          p.rows + static_cast<size_t>(row) * p.dpad + c0 + 2 * u);
            }
          }
#pragma unroll
          for (int b = 0; b < kHostLoads; ++b) {
            const int i = i0 + b * kFinThreads;
            if (i < nsel * len2) {
              const int rr = i / len2, u = i - rr * len2;
              s_rows64[rr * row_stride + 2 * u] = v[b].x;
              s_rows64[rr * row_stride + 2 * u + 1] = v[b].y;
            }
          }
        }
      } else {
        for (int i0 = tid; i0 < nsel * len; i0 += 2 * kHostLoads * kFinThreads) {
          double v[2 * kHostLoads];
#pragma unroll
          for (int b = 0; b < 2 * kHostLoads; ++b) {
            const int i = i0 + b * kFinThreads;
            if (i < nsel * len) {
              const int rr = i / len, u = i - rr * len;
              const int row = static_cast<int>(key_row(s_sel[rr]));
              v[b] = ldx(rows_x + static_cast<size_t>(row) * p.d + c0 + u, p.rows + static_cast<size_t>(row) * p.dpad + c0 + u);
            }
          }
#pragma unroll
          for (int b = 0; b < 2 * kHostLoads; ++b) {
            const int i = i0 + b * kFinThreads;
            if (i < nsel * len) {
              const int rr = i / len, u = i - rr * len;
              s_rows64[rr * row_stride + u] = v[b];
            }
          }
        }
      }
      for (int i = tid; i < len; i += kFinThreads) s_q[i] = __ldg(qv + c0 + i);
      __syncthreads();
      if (tid < nsel) {
        const double* mine = s_rows64 + tid * row_stride;
        for (int i = 0; i < len; ++i) dot = __dadd_rn(dot, __dmul_rn(s_q[i], mine[i]));
      }
      if (tid == kFinThreads - 1)
        for (int i = 0; i < len; ++i) na_chain = __dadd_rn(na_chain, __dmul_rn(s_q[i], s_q[i]));
    }
  } else {
    // exact source = the f64 sidecar: same staging, 8-byte elements (odd stride in doubles: conflict-free)
    const XT* rows_x = static_cast<const XT*>(p.rows_x);
    double* s_rows64 = reinterpret_cast<double*>(s_keys);
    int chunk = nsel > 0 ? (p.key_cap / nsel - 1) : kQChunk;          // doubles per row chunk
    chunk = chunk < kQChunk ? chunk : kQChunk;
    const int row_stride = chunk | 1;
    for (int c0 = 0; c0 < p.d; c0 += chunk) {
      const int len = p.d - c0 < chunk ? p.d - c0 : chunk;
      __syncthreads();
      for (int i = tid; i < nsel * len; i += kFinThreads) {
        const int rr = i / len, u = i - rr * len;
        const int row = static_cast<int>(key_row(s_sel[rr]));
        s_rows64[rr * row_stride + u] =
            ldx(rows_x + static_cast<size_t>(row) * p.d + c0 + u, p.rows + static_cast<size_t>(row) * p.dpad + c0 + u);
      }
      for (int i = tid; i < len; i += kFinThreads) s_q[i] = __ldg(qv + c0 + i);
      __syncthreads();
      if (tid < nsel) {
        const double* mine = s_rows64 + tid * row_stride;
        for (int i = 0; i < len; ++i) dot = __dadd_rn(dot, __dmul_rn(s_q[i], mine[i]));
      }
      if (tid == kFinThreads - 1)
        for (int i = 0; i < len; ++i) na_chain = __dadd_rn(na_chain, __dmul_rn(s_q[i], s_q[i]));
    }
  }
  if (tid == kFinThreads - 1) {
    s_na = na_chain;
    p.q.q_norm2[ql] = na_chain;   // kept for the exhaustive fallback of a flagged query
  }
  __syncthreads();
  const double na = s_na;
  const int k_q = kEach ? p.k_each[ql] : p.k_fetch;             // this query's cut (<= k_fetch, the row stride)
  const double min_q = kEach ? p.min_each[ql] : p.min_score;    // and threshold
  if (tid < nsel) {
    const double sc = exact_cosine(dot, na, p.row_norm2[my_row]);
    s_score[tid] = sc;
    s_row[tid] = my_row;
    const int ok = sc >= min_q ? 1 : 0;  // vector-store.ts:212 (NaN fails; -inf = no threshold)
    s_valid[tid] = ok;
    if (ok) atomicAdd(&s_nvalid, 1);
  }
  __syncthreads();
  const int nvalid = s_nvalid;
  const int count = nvalid < k_q ? nvalid : k_q;
  // ---- final order: score desc, ties -> lower slot (stable sort over insertion order) ----
  if (tid < nsel && s_valid[tid]) {
    const double sc = s_score[tid];
    const int row = s_row[tid];
    int rank = 0;
    for (int j = 0; j < nsel; ++j) {
      if (!s_valid[j]) continue;
      const double sj = s_score[j];
      rank += (sj > sc || (sj == sc && s_row[j] < row)) ? 1 : 0;
    }
    if (rank < k_q) {
      p.out_slots[static_cast<size_t>(ql) * p.k_fetch + rank] = p.slot.global(row);
      p.out_scores[static_cast<size_t>(ql) * p.k_fetch + rank] = sc;
    }
    if (rank == k_q - 1) s_ekth = sc;
  }
  for (int i = count + tid; i < p.k_fetch; i += kFinThreads) {
    p.out_slots[static_cast<size_t>(ql) * p.k_fetch + i] = -1;
    p.out_scores[static_cast<size_t>(ql) * p.k_fetch + i] = __longlong_as_double(0x7FF8000000000000ll);
  }
  __syncthreads();
  if (tid == 0) {
    p.out_counts[ql] = count;
    // ---- proof of exactness (DESIGN.md §6) ----
    bool ok;
    if (!(p.q.q_eps[ql] < kEpsNone)) {
      ok = false;  // the scan's bound proves nothing for this query (prep_queries): the exhaustive kernel answers it
    } else if (tau_raw == -INFINITY) {
      ok = true;  // nothing was ever dropped except by thr_init (provably below min_score)
    } else {
      const double bound = static_cast<double>(tau_raw) * static_cast<double>(p.q.q_inv_norm[ql]) + p.q.q_eps[ql];
      if (count == k_q) ok = s_ekth > bound;             // every outsider scores strictly below the k-th hit
      else ok = bound < min_q;                            // no outsider can pass the threshold
    }
    p.flags[ql] = ok ? 0 : 1;
  }
}

}  // namespace
// The entry points of the three exact-row types (float64, float32, split float32) sit in a named namespace, so that
// their symbols, which the build tests pair up by name across the row types, carry no hash of this file.
namespace entry {
// One kernel per exact-row type: float64 rows (finalize_kernel) and float32 rows (finalize_f32_kernel).
template <bool kHostRows>
__global__ void __launch_bounds__(kFinThreads) finalize_kernel(FinalizeParams p) {
  finalize_rows<kHostRows, double, false>(p);
}
template <bool kHostRows>
__global__ void __launch_bounds__(kFinThreads) finalize_f32_kernel(FinalizeParams p) {
  finalize_rows<kHostRows, float, false>(p);
}
// and split float32 rows (finalize_split_kernel): low halves in rows_x, high halves in rows
template <bool kHostRows>
__global__ void __launch_bounds__(kFinThreads) finalize_split_kernel(FinalizeParams p) {
  finalize_rows<kHostRows, F32Lo, false>(p);
}
}  // namespace entry
namespace {
// The exact-row type of x_elem bytes per element, for the per-query kernels below (named by width, so that their
// symbols stay apart from the scalar kernels' per-type ones).
template <int kXElem>
struct XOf {
  using T = double;
};
template <>
struct XOf<4> {
  using T = float;
};
template <>
struct XOf<2> {
  using T = F32Lo;
};
// rbk_index_search_each_f64: every exact-row type and placement, each query at its own cut and threshold.
template <bool kHostRows, int kXElem>
__global__ void __launch_bounds__(kFinThreads) finalize_each_kernel(FinalizeParams p) {
  finalize_rows<kHostRows, typename XOf<kXElem>::T, true>(p);
}

// --------------------------------------------------------------------------- exact fallback (K0)
constexpr int kExThreads = 256;
constexpr int kExBuf = 1024;

struct ExactTopK {
  double score[kExBuf];
  int row[kExBuf];
  int n;
  int have_thr;
  double thr_score;
  int thr_row;
};

__device__ __forceinline__ bool hit_before(double sa, int ra, double sb, int rb) {
  return sa > sb || (sa == sb && ra < rb);
}

// Block-wide: sort the buffer by (score desc, row asc), keep the best K.
__device__ void exact_compact(ExactTopK& t, int K) {
  const int tid = threadIdx.x;
  __syncthreads();
  const int n = t.n;
  for (int i = n + tid; i < kExBuf; i += kExThreads) {
    t.score[i] = -INFINITY;
    t.row[i] = INT_MAX;
  }
  __syncthreads();
  for (int k2 = 2; k2 <= kExBuf; k2 <<= 1) {
    for (int s = k2 >> 1; s > 0; s >>= 1) {
      for (int i = tid; i < kExBuf; i += kExThreads) {
        const int j = i ^ s;
        if (j > i) {
          const bool desc = (i & k2) == 0;
          const bool j_first = hit_before(t.score[j], t.row[j], t.score[i], t.row[i]);
          if (desc ? j_first : !j_first) {
            const double ts = t.score[i];
            t.score[i] = t.score[j];
            t.score[j] = ts;
            const int tr = t.row[i];
            t.row[i] = t.row[j];
            t.row[j] = tr;
          }
        }
      }
      __syncthreads();
    }
  }
  if (tid == 0) {
    const int keep = n < K ? n : K;
    t.n = keep;
    if (keep == K) {
      t.have_thr = 1;
      t.thr_score = t.score[K - 1];
      t.thr_row = t.row[K - 1];
    }
  }
  __syncthreads();
}

__device__ __forceinline__ void exact_push(ExactTopK& t, double sc, int row) {
  if (t.have_thr && !hit_before(sc, row, t.thr_score, t.thr_row)) return;
  const int pos = atomicAdd(&t.n, 1);
  t.score[pos] = sc;
  t.row[pos] = row;
}

// kEach: each failing query is cut at its own p.k_each[q] and filtered at p.min_each[q]; p.k_fetch stays the stride.
template <typename XT, bool kEach>
__device__ __forceinline__ void exact_scan_rows(const ExactParams& p) {
  __shared__ ExactTopK t;
  const int tid = threadIdx.x;
  const int f = blockIdx.y;
  const int q = p.fail_list[f];
  if (tid == 0) {
    t.n = 0;
    t.have_thr = 0;
  }
  __syncthreads();
  const int64_t chunk = (p.n_rows + p.n_blocks - 1) / p.n_blocks;
  const int64_t r0 = blockIdx.x * chunk;
  const int64_t r1 = r0 + chunk < p.n_rows ? r0 + chunk : p.n_rows;
  const double* qv = p.q_f64 + static_cast<size_t>(q) * p.d;
  const double na = p.q_norm2[q];
  const double min_q = kEach ? p.min_each[q] : p.min_score;
  // the cut is read where a compaction needs it, not held in a register across the scan
  auto k_q = [&]() { return kEach ? __ldg(p.k_each + q) : p.k_fetch; };
  for (int64_t base = r0; base < r1; base += kExThreads) {
    // Every thread reads t.n before any push of this iteration moves it: read after the last barrier alone, a fast
    // thread's push could send a slow one into exact_compact's barriers without the others.
    const int n_now = t.n;
    __syncthreads();
    if (n_now > kExBuf - kExThreads) exact_compact(t, k_q());
    const int64_t row = base + tid;
    if (row < r1) {
      const bool dead = (p.dead_bits[row >> 5] >> (row & 31)) & 1u;
      if (!dead) {   // zero-norm rows give NaN and fail the compare below, like in the reference (S3)
        const XT* rows_x = static_cast<const XT*>(p.rows_x);
        const double dot = rows_x != nullptr ? exact_dot_f64(qv, rows_x + static_cast<size_t>(row) * p.d, p.d,
                                                             p.rows + static_cast<size_t>(row) * p.dpad)
                                             : exact_dot(qv, p.rows + static_cast<size_t>(row) * p.dpad, p.d);
        const double sc = exact_cosine(dot, na, p.row_norm2[row]);
        if (sc >= min_q) exact_push(t, sc, static_cast<int>(row));
      }
    }
    __syncthreads();
  }
  exact_compact(t, k_q());
  const size_t o = (static_cast<size_t>(f) * p.n_blocks + blockIdx.x) * p.k_fetch;
  for (int i = tid; i < t.n; i += kExThreads) {
    p.part_scores[o + i] = t.score[i];
    p.part_rows[o + i] = t.row[i];
  }
  if (tid == 0) p.part_cnt[f * p.n_blocks + blockIdx.x] = t.n;
}
template <typename XT>
__global__ void __launch_bounds__(kExThreads) exact_scan_kernel(ExactParams p) {
  exact_scan_rows<XT, false>(p);
}
template <int kXElem>
__global__ void __launch_bounds__(kExThreads) exact_scan_each_kernel(ExactParams p) {
  exact_scan_rows<typename XOf<kXElem>::T, true>(p);
}

__global__ void __launch_bounds__(kExThreads) exact_merge_kernel(ExactParams p) {
  __shared__ ExactTopK t;
  const int tid = threadIdx.x;
  const int f = blockIdx.x;
  const int q = p.fail_list[f];
  if (tid == 0) {
    t.n = 0;
    t.have_thr = 0;
  }
  __syncthreads();
  const int total = p.n_blocks * p.k_fetch;
  const int k_q = p.k_each != nullptr ? p.k_each[q] : p.k_fetch;
  for (int base = 0; base < total; base += kExThreads) {
    const int n_now = t.n;   // read by every thread before any push moves it (as in exact_scan_kernel)
    __syncthreads();
    if (n_now > kExBuf - kExThreads) exact_compact(t, k_q);
    const int i = base + tid;
    if (i < total) {
      const int b = i / p.k_fetch, e = i % p.k_fetch;
      if (e < p.part_cnt[f * p.n_blocks + b]) {
        const size_t o = (static_cast<size_t>(f) * p.n_blocks + b) * p.k_fetch + e;
        exact_push(t, p.part_scores[o], p.part_rows[o]);
      }
    }
    __syncthreads();
  }
  exact_compact(t, k_q);
  const int n = t.n;
  for (int i = tid; i < p.k_fetch; i += kExThreads) {
    const size_t o = static_cast<size_t>(q) * p.k_fetch + i;
    if (i < n) {
      p.out_slots[o] = p.slot.global(t.row[i]);
      p.out_scores[o] = t.score[i];
    } else {
      p.out_slots[o] = -1;
      p.out_scores[o] = __longlong_as_double(0x7FF8000000000000ll);
    }
  }
  if (tid == 0) p.out_counts[q] = n;
}

// --------------------------------------------------------------------------- large-k search (DESIGN.md §6)
// select: one block per query, between the count pass and the emit pass.  T_q = lower edge of the highest bin j with
// >= k_fetch counted rows in bins >= j; theta_q = max(T_q - 2 eps_q, thr_init) (raw domain, nudged down);
// C_q = counted rows in bins >= bin(theta_q), an upper bound on the rows the emit pass finds at or above theta_q.
__global__ void __launch_bounds__(256) large_select_kernel(const unsigned int* __restrict__ hist,
                                                           const float* __restrict__ thr_init,
                                                           const float* __restrict__ inv_norm_q,
                                                           const double* __restrict__ q_eps, int k_fetch,
                                                           int n_rows, float* __restrict__ theta,
                                                           int* __restrict__ cap, const int* __restrict__ k_each) {
  const int q = blockIdx.x;
  const int tid = threadIdx.x;
  const unsigned int k_q = static_cast<unsigned int>(k_each != nullptr ? k_each[q] : k_fetch);
  __shared__ unsigned int s_grp[256];          // suffix sums over groups of 4 bins
  __shared__ unsigned int s_suf[kHistBins];    // rows counted in bins >= b
  __shared__ int s_top;
  const uint4 h = reinterpret_cast<const uint4*>(hist + static_cast<size_t>(q) * kHistBins)[tid];
  s_grp[tid] = h.x + h.y + h.z + h.w;
  if (tid == 0) s_top = -1;
  __syncthreads();
  for (int o = 1; o < 256; o <<= 1) {
    const unsigned int v = tid + o < 256 ? s_grp[tid + o] : 0u;
    __syncthreads();
    s_grp[tid] += v;
    __syncthreads();
  }
  const unsigned int c[4] = {h.x, h.y, h.z, h.w};
  unsigned int suf = s_grp[tid];
  int best = -1;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    s_suf[4 * tid + j] = suf;
    if (suf >= k_q) best = 4 * tid + j;
    suf -= c[j];
  }
  if (best >= 0) atomicMax(&s_top, best);
  __syncthreads();
  if (tid != 0) return;
  const float ti = thr_init[q];
  if (!(q_eps[q] < kEpsNone)) {   // the bound proves nothing: no scan, every live row is a candidate (large_emit_all)
    theta[q] = INFINITY;
    cap[q] = n_rows;
    return;
  }
  if (!(ti < INFINITY)) {   // zero / non-finite query: nothing matches
    theta[q] = INFINITY;
    cap[q] = 0;
    return;
  }
  float th = ti;
  const float inv = inv_norm_q[q];
  if (s_top >= 0) {
    const double edge = static_cast<double>(s_top) * (2.0 / kHistBins) - 1.0;
    const double raw = (edge - 2.0 * q_eps[q] - 1e-6) / static_cast<double>(inv);
    float t = static_cast<float>(raw);
    t = nextafterf(nextafterf(t, -INFINITY), -INFINITY);
    th = fmaxf(th, t);
  }
  theta[q] = th;
  // the bin of a row with a >= th is >= this one: same float expression as hist_add
  const int b = static_cast<int>((th * inv + 1.0f) * (kHistBins * 0.5f));
  cap[q] = static_cast<int>(s_suf[min(max(b, 0), kHistBins - 1)]);
}

// The candidates of a query whose bound proves nothing (large_select gave it theta = +inf and C_q = n_rows, so the
// emit scan wrote nothing for it): every row that is not tombstoned, in any order - the re-rank sorts them.
__global__ void __launch_bounds__(256) large_emit_all_kernel(const double* __restrict__ q_eps,
                                                             const unsigned int* __restrict__ dead_bits,
                                                             int64_t n_rows, const long long* __restrict__ emit_off,
                                                             int* __restrict__ emit_cnt, int* __restrict__ emit_rows) {
  const int q = blockIdx.y;
  if (q_eps[q] < kEpsNone) return;
  const int64_t row = static_cast<int64_t>(blockIdx.x) * 256 + threadIdx.x;
  const bool take = row < n_rows && !((dead_bits[row >> 5] >> (row & 31)) & 1u);
  const unsigned int m = __ballot_sync(kFull, take);
  const int lane = threadIdx.x & 31;
  int base = 0;
  if (lane == 0 && m != 0u) base = atomicAdd(emit_cnt + q, __popc(m));
  base = __shfl_sync(kFull, base, 0);
  if (take) emit_rows[emit_off[q] + base + __popc(m & ((1u << lane) - 1u))] = static_cast<int>(row);
}

// re-rank, part 1: the reference's fp64 cosine of every emitted row (one thread per candidate).
// kHostRows (rows_f64 in mapped host memory): a thread walking its own row would issue 32 scattered host reads per
// warp load.  Instead the block's 256 candidates stage their rows kLsChunk elements at a time in shared memory -
// consecutive lanes read consecutive 16-byte pieces of one row, kHostLoads pieces in flight per thread - and each
// thread then walks its own chain from there, in the same order as exact_dot_f64.
constexpr int kLsChunk = 16;   // doubles per staged row piece (128 bytes)

template <bool kHostRows, typename XT>
__device__ __forceinline__ void large_score_rows(const LargeRerankParams& p) {
  const XT* rows_x = static_cast<const XT*>(p.rows_x);
  const int q = blockIdx.y;
  const int i = blockIdx.x * 256 + threadIdx.x;
  const int n = min(p.emit_cnt[q], p.emit_cap[q]);
  if constexpr (!kHostRows) {
    if (i >= n) return;
    const size_t o = static_cast<size_t>(p.emit_off[q]) + i;
    const int row = p.emit_rows[o];
    const double* qv = p.q_f64 + static_cast<size_t>(q) * p.d;
    const double dot = rows_x != nullptr ? exact_dot_f64(qv, rows_x + static_cast<size_t>(row) * p.d, p.d,
                                                         p.rows + static_cast<size_t>(row) * p.dpad)
                                         : exact_dot(qv, p.rows + static_cast<size_t>(row) * p.dpad, p.d);
    p.cand_scores[o] = exact_cosine(dot, p.q_norm2[q], p.row_norm2[row]);
  } else {
    __shared__ double s_x[256 * (kLsChunk + 1)];   // odd pitch in doubles: conflict-free walks
    __shared__ double s_q[kLsChunk];
    __shared__ int s_row[256];
    const int tid = threadIdx.x;
    const int first = blockIdx.x * 256;
    if (first >= n) return;   // uniform over the block
    const int m = n - first < 256 ? n - first : 256;   // candidates of this block
    const size_t o = static_cast<size_t>(p.emit_off[q]) + i;
    if (tid < m) s_row[tid] = p.emit_rows[o];
    const double* qv = p.q_f64 + static_cast<size_t>(q) * p.d;
    const bool wide = (p.d & 1) == 0;   // every row and every even column start 16-byte aligned
    double dot = 0.0;
    for (int c0 = 0; c0 < p.d; c0 += kLsChunk) {
      const int len = p.d - c0 < kLsChunk ? p.d - c0 : kLsChunk;
      __syncthreads();   // s_row written / the previous chunk consumed
      if (wide) {
        const int len2 = len >> 1;
        for (int i0 = tid; i0 < m * len2; i0 += kHostLoads * 256) {
          double2 v[kHostLoads];
#pragma unroll
          for (int b = 0; b < kHostLoads; ++b) {
            const int e = i0 + b * 256;
            if (e < m * len2) {
              const int rr = e / len2, u = e - rr * len2;
              v[b] = ldx2(reinterpret_cast<const Pair<XT>*>(rows_x + static_cast<size_t>(s_row[rr]) * p.d + c0) + u,
                          p.rows + static_cast<size_t>(s_row[rr]) * p.dpad + c0 + 2 * u);
            }
          }
#pragma unroll
          for (int b = 0; b < kHostLoads; ++b) {
            const int e = i0 + b * 256;
            if (e < m * len2) {
              const int rr = e / len2, u = e - rr * len2;
              s_x[rr * (kLsChunk + 1) + 2 * u] = v[b].x;
              s_x[rr * (kLsChunk + 1) + 2 * u + 1] = v[b].y;
            }
          }
        }
      } else {
        for (int i0 = tid; i0 < m * len; i0 += 2 * kHostLoads * 256) {
          double v[2 * kHostLoads];
#pragma unroll
          for (int b = 0; b < 2 * kHostLoads; ++b) {
            const int e = i0 + b * 256;
            if (e < m * len) {
              const int rr = e / len, u = e - rr * len;
              v[b] = ldx(rows_x + static_cast<size_t>(s_row[rr]) * p.d + c0 + u,
                         p.rows + static_cast<size_t>(s_row[rr]) * p.dpad + c0 + u);
            }
          }
#pragma unroll
          for (int b = 0; b < 2 * kHostLoads; ++b) {
            const int e = i0 + b * 256;
            if (e < m * len) {
              const int rr = e / len, u = e - rr * len;
              s_x[rr * (kLsChunk + 1) + u] = v[b];
            }
          }
        }
      }
      if (tid < len) s_q[tid] = __ldg(qv + c0 + tid);
      __syncthreads();
      if (tid < m) {
        const double* mine = s_x + tid * (kLsChunk + 1);
        for (int e = 0; e < len; ++e) dot = __dadd_rn(dot, __dmul_rn(s_q[e], mine[e]));
      }
    }
    if (tid < m) p.cand_scores[o] = exact_cosine(dot, p.q_norm2[q], p.row_norm2[s_row[tid]]);
  }
}

}  // namespace
namespace entry {   // (see finalize_kernel)
template <bool kHostRows>
__global__ void __launch_bounds__(256) large_score_kernel(LargeRerankParams p) {
  large_score_rows<kHostRows, double>(p);
}
template <bool kHostRows>
__global__ void __launch_bounds__(256) large_score_f32_kernel(LargeRerankParams p) {
  large_score_rows<kHostRows, float>(p);
}
template <bool kHostRows>
__global__ void __launch_bounds__(256) large_score_split_kernel(LargeRerankParams p) {
  large_score_rows<kHostRows, F32Lo>(p);
}
}  // namespace entry
namespace {

// re-rank, part 2: one block per query keeps the best k_fetch of its candidates by (score desc, row asc) in a
// shared-memory buffer of S >= k_fetch + blockDim entries, compacted (bitonic sort, cut at k_fetch) whenever the next
// round of pushes might not fit - so any number of candidates (every duplicate of the k-th row is one) streams through.
constexpr int kTopThreads = 512;

__device__ void large_compact(double* sc, int* rw, int S, int* s_n, int K, int* s_have, double* s_ts, int* s_tr) {
  const int tid = threadIdx.x;
  __syncthreads();
  const int n = *s_n;
  for (int i = n + tid; i < S; i += kTopThreads) {
    sc[i] = -INFINITY;
    rw[i] = INT_MAX;
  }
  __syncthreads();
  for (int k2 = 2; k2 <= S; k2 <<= 1) {
    for (int s = k2 >> 1; s > 0; s >>= 1) {
      for (int i = tid; i < S; i += kTopThreads) {
        const int j = i ^ s;
        if (j > i) {
          const bool desc = (i & k2) == 0;
          const bool j_first = hit_before(sc[j], rw[j], sc[i], rw[i]);
          if (desc ? j_first : !j_first) {
            const double ts = sc[i];
            sc[i] = sc[j];
            sc[j] = ts;
            const int tr = rw[i];
            rw[i] = rw[j];
            rw[j] = tr;
          }
        }
      }
      __syncthreads();
    }
  }
  if (tid == 0) {
    const int keep = n < K ? n : K;
    *s_n = keep;
    if (keep == K) {
      *s_have = 1;
      *s_ts = sc[K - 1];
      *s_tr = rw[K - 1];
    }
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kTopThreads) large_topk_kernel(LargeRerankParams p, int S) {
  extern __shared__ __align__(16) double s_sc[];
  int* s_rw = reinterpret_cast<int*>(s_sc + S);
  __shared__ int s_n, s_have, s_tr;
  __shared__ double s_ts;
  const int q = blockIdx.x;
  const int tid = threadIdx.x;
  if (tid == 0) {
    s_n = 0;
    s_have = 0;
  }
  __syncthreads();
  const int emitted = p.emit_cnt[q];
  const int n_cand = min(emitted, p.emit_cap[q]);
  const size_t off = static_cast<size_t>(p.emit_off[q]);
  const int k_q = p.k_each != nullptr ? p.k_each[q] : p.k_fetch;   // the query's cut; p.k_fetch is the row stride
  const double min_q = p.min_each != nullptr ? p.min_each[q] : p.min_score;
  for (int base = 0; base < n_cand; base += kTopThreads) {
    if (s_n > S - kTopThreads) large_compact(s_sc, s_rw, S, &s_n, k_q, &s_have, &s_ts, &s_tr);  // uniform
    const int i = base + tid;
    if (i < n_cand) {
      const double sc = p.cand_scores[off + i];
      const int row = p.emit_rows[off + i];
      // vector-store.ts:212 (NaN fails; -inf = no threshold), then only what can still make the cut
      if (sc >= min_q && (!s_have || hit_before(sc, row, s_ts, s_tr))) {
        const int pos = atomicAdd(&s_n, 1);
        s_sc[pos] = sc;
        s_rw[pos] = row;
      }
    }
    __syncthreads();
  }
  large_compact(s_sc, s_rw, S, &s_n, k_q, &s_have, &s_ts, &s_tr);
  const int n = s_n;
  for (int i = tid; i < p.k_fetch; i += kTopThreads) {
    const size_t o = static_cast<size_t>(q) * p.k_fetch + i;
    if (i < n) {
      p.out_slots[o] = p.slot.global(s_rw[i]);
      p.out_scores[o] = s_sc[i];
    } else {
      p.out_slots[o] = -1;
      p.out_scores[o] = __longlong_as_double(0x7FF8000000000000ll);
    }
  }
  if (tid == 0) {
    p.out_counts[q] = n;
    if (emitted > p.emit_cap[q]) atomicAdd(p.overflow, 1);   // the count pass missed rows: the answer is not proven
  }
}

// --------------------------------------------------------------------------- unbounded search: segmented sort
// Replaces large_topk_kernel when k_fetch exceeds what one block's shared memory holds.  After large_score_kernel a
// query's segment holds n_q = min(emit_cnt, emit_cap) candidates (row, exact score).  (1) seg_tile_sort_kernel: one
// block per tile of kSortTile candidates of one query drops what fails `>= min_score` (NaN included), sorts the rest by
// (score desc, row asc) in shared memory, writes the first min(passing, k_eff) back in place and records that length.
// (2) seg_merge_kernel, once per doubling: adjacent runs 2r and 2r+1 of a query become run r of twice the width.  Each
// entry's rank in the merged run is its own index plus the number of entries of the partner run that come before it
// (binary search; rows are unique, so hit_before is a strict total order and the ranks are a permutation); ranks >= k_eff
// are dropped, because nothing past position k_eff of a run can reach the answer.  (3) seg_write_kernel: global slots,
// scores, the -1 / NaN tail and the counts in the [B][k_eff] layout large_topk_kernel writes.
constexpr int kSortThreads = 512;
constexpr int kMergeThreads = 256;

__global__ void __launch_bounds__(kSortThreads) seg_tile_sort_kernel(LargeRerankParams p, SegSortScratch s) {
  extern __shared__ __align__(16) double s_sc[];   // kSortTile scores, then kSortTile rows
  int* s_rw = reinterpret_cast<int*>(s_sc + kSortTile);
  __shared__ int s_pass;
  const int q = blockIdx.y, t = blockIdx.x, tid = threadIdx.x;
  const int n = min(p.emit_cnt[q], p.emit_cap[q]);
  const int i0 = t * kSortTile;
  if (i0 >= n) return;   // uniform: a tile past the segment's end holds nothing and is never read
  const int m = min(kSortTile, n - i0);
  int S = 2;             // the bitonic network's width: a power of two >= m
  while (S < m) S <<= 1;
  const size_t base = static_cast<size_t>(p.emit_off[q]) + i0;
  const double min_q = p.min_each != nullptr ? p.min_each[q] : p.min_score;
  if (tid == 0) s_pass = 0;
  __syncthreads();
  int mine = 0;
  for (int i = tid; i < S; i += kSortThreads) {
    double sc = -INFINITY;
    int rw = INT_MAX;    // after every real row, even one scoring -inf
    if (i < m) {
      const double v = p.cand_scores[base + i];
      if (v >= min_q) {   // vector-store.ts:212 (NaN fails; -inf = no threshold)
        sc = v;
        rw = p.emit_rows[base + i];
        ++mine;
      }
    }
    s_sc[i] = sc;
    s_rw[i] = rw;
  }
  if (mine) atomicAdd(&s_pass, mine);
  __syncthreads();
  for (int k2 = 2; k2 <= S; k2 <<= 1) {
    for (int st = k2 >> 1; st > 0; st >>= 1) {
      for (int i = tid; i < S; i += kSortThreads) {
        const int j = i ^ st;
        if (j > i) {
          const bool desc = (i & k2) == 0;
          const bool j_first = hit_before(s_sc[j], s_rw[j], s_sc[i], s_rw[i]);
          if (desc ? j_first : !j_first) {
            const double ts = s_sc[i];
            s_sc[i] = s_sc[j];
            s_sc[j] = ts;
            const int tr = s_rw[i];
            s_rw[i] = s_rw[j];
            s_rw[j] = tr;
          }
        }
      }
      __syncthreads();
    }
  }
  const int L = min(s_pass, p.k_each != nullptr ? p.k_each[q] : p.k_fetch);   // truncated at the query's own cut
  for (int i = tid; i < L; i += kSortThreads) {
    p.cand_scores[base + i] = s_sc[i];
    p.emit_rows[base + i] = s_rw[i];
  }
  if (tid == 0) s.len[0][s.tile_off[q] + t] = L;
}

// Merge pass `pass` (0-based): runs of 2^pass tiles -> runs of 2^(pass+1) tiles.  One block per input tile.  kEach:
// every run is truncated at its query's own p.k_each[q].
template <bool kEach = false>
__global__ void __launch_bounds__(kMergeThreads) seg_merge_kernel(LargeRerankParams p, SegSortScratch s, int pass) {
  const int q = blockIdx.y, t = blockIdx.x, tid = threadIdx.x;
  const int n = min(p.emit_cnt[q], p.emit_cap[q]);
  const int nt = (n + kSortTile - 1) / kSortTile;
  if (t >= nt) return;
  const int src = pass & 1, dst = src ^ 1;
  const double* sc_in = src ? s.scores : p.cand_scores;
  const int* rw_in = src ? s.rows : p.emit_rows;
  double* sc_out = dst ? s.scores : p.cand_scores;
  int* rw_out = dst ? s.rows : p.emit_rows;
  const int w = 1 << pass;                 // tiles per input run
  const int r = t >> pass, local = t & (w - 1);
  const int partner = r ^ 1;
  // (selects, not s.len[src]: a run-time index into the parameter array would copy it to local memory)
  const int* len_in = (src ? s.len[1] : s.len[0]) + s.tile_off[q];
  int* len_out = (dst ? s.len[1] : s.len[0]) + s.tile_off[q];
  const int La = len_in[r * w];
  const int Lb = partner * w < nt ? len_in[partner * w] : 0;   // the last run of an odd count has no partner: copied
  const int L = min(La + Lb, kEach ? p.k_each[q] : p.k_fetch);
  if (local == 0 && (r & 1) == 0 && tid == 0) len_out[r * w] = L;
  const size_t seg = static_cast<size_t>(p.emit_off[q]);
  const size_t mine = seg + static_cast<size_t>(r) * w * kSortTile;
  const size_t other = seg + static_cast<size_t>(partner) * w * kSortTile;
  const size_t out = seg + static_cast<size_t>(r >> 1) * 2 * w * kSortTile;
  // 64-bit positions: with k_eff (< 2^31) entries a run's last tile may end past INT_MAX
  const long long e1 = min(static_cast<long long>(local + 1) * kSortTile, static_cast<long long>(La));
  for (long long e = static_cast<long long>(local) * kSortTile + tid; e < e1; e += kMergeThreads) {
    const double sc = sc_in[mine + e];
    const int rw = rw_in[mine + e];
    int lo = 0, hi = Lb;                   // entries of the partner run that come before (sc, rw)
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (hit_before(__ldg(sc_in + other + mid), __ldg(rw_in + other + mid), sc, rw)) lo = mid + 1;
      else hi = mid;
    }
    const long long rank = e + lo;   // La <= k_eff: every rank is >= its own index
    if (rank < L) {
      sc_out[out + rank] = sc;
      rw_out[out + rank] = rw;
    }
  }
}

__global__ void __launch_bounds__(256) seg_write_kernel(LargeRerankParams p, SegSortScratch s, int final_buf) {
  const int q = blockIdx.y;
  const int emitted = p.emit_cnt[q];
  const int n = min(emitted, p.emit_cap[q]);
  const int L = n > 0 ? (final_buf ? s.len[1] : s.len[0])[s.tile_off[q]] : 0;
  const double* sc = final_buf ? s.scores : p.cand_scores;
  const int* rw = final_buf ? s.rows : p.emit_rows;
  const size_t seg = static_cast<size_t>(p.emit_off[q]);
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < p.k_fetch; i += gridDim.x * 256ll) {
    const size_t o = static_cast<size_t>(q) * p.k_fetch + i;
    if (i < L) {
      p.out_slots[o] = p.slot.global(rw[seg + i]);
      p.out_scores[o] = sc[seg + i];
    } else {
      p.out_slots[o] = -1;
      p.out_scores[o] = __longlong_as_double(0x7FF8000000000000ll);
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    p.out_counts[q] = L;
    if (emitted > p.emit_cap[q]) atomicAdd(p.overflow, 1);   // the count pass missed rows: the answer is not proven
  }
}

// --------------------------------------------------------------------------- similar pairs (DESIGN.md §6)
// rbk_index_similar_pairs_f64 runs the unbounded search's re-rank with no cut, for queries that are the stored rows of
// consecutive global slots pp.a0 + q and candidates that are rows pp.r0 + emit_rows[i] (p's row pointers start at row
// r0).  (1) pairs_mask_kernel, between the re-score and the tile sort: a candidate whose global slot is not above its
// query's gets the score NaN, which the tile sort drops together with the scores below min_score.  (2)
// pairs_offsets_kernel: each query's exact pair count (the length of its sorted run) and their exclusive scan.  (3)
// pairs_write_kernel: the sorted runs packed end to end as (global slot, score), query after query.
__global__ void __launch_bounds__(256) pairs_mask_kernel(LargeRerankParams p, PairsParams pp) {
  const int q = blockIdx.y;
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= min(p.emit_cnt[q], p.emit_cap[q])) return;
  const size_t o = static_cast<size_t>(p.emit_off[q]) + i;
  if (p.slot.global(pp.r0 + p.emit_rows[o]) <= pp.a0 + q) p.cand_scores[o] = __longlong_as_double(0x7FF8000000000000ll);
}

constexpr int kPairsScanThreads = 1024;   // one thread per query of a launch (B <= kMaxSubBatch)
static_assert(kMaxSubBatch <= kPairsScanThreads, "one thread per query");

__global__ void __launch_bounds__(kPairsScanThreads) pairs_offsets_kernel(LargeRerankParams p, SegSortScratch s,
                                                                          int final_buf, PairsParams pp) {
  __shared__ long long s_sum[kPairsScanThreads];
  const int q = threadIdx.x;
  int L = 0;
  if (q < p.B) {
    const int emitted = p.emit_cnt[q];
    if (min(emitted, p.emit_cap[q]) > 0) L = (final_buf ? s.len[1] : s.len[0])[s.tile_off[q]];
    pp.counts[q] = L;
    if (emitted > p.emit_cap[q]) atomicAdd(p.overflow, 1);   // the count pass missed rows: the answer is not proven
  }
  s_sum[q] = L;
  __syncthreads();
  for (int o = 1; o < kPairsScanThreads; o <<= 1) {   // inclusive scan
    const long long v = q >= o ? s_sum[q - o] : 0;
    __syncthreads();
    s_sum[q] += v;
    __syncthreads();
  }
  if (q < p.B) pp.offsets[q] = s_sum[q] - L;
}

__global__ void __launch_bounds__(256) pairs_write_kernel(LargeRerankParams p, SegSortScratch s, int final_buf,
                                                          PairsParams pp) {
  const int q = blockIdx.y;
  const int L = pp.counts[q];
  const double* sc = final_buf ? s.scores : p.cand_scores;
  const int* rw = final_buf ? s.rows : p.emit_rows;
  const size_t seg = static_cast<size_t>(p.emit_off[q]);
  const long long o = pp.offsets[q];
  for (int i = blockIdx.x * 256 + threadIdx.x; i < L; i += gridDim.x * 256) {
    pp.out_b[o + i] = p.slot.global(pp.r0 + rw[seg + i]);
    pp.out_scores[o + i] = sc[seg + i];
  }
}

// --------------------------------------------------------------------------- all exact scores
// One thread per (row, query): the reference's fp64 cosine of EVERY row, NaN for tombstoned / zero rows, for a host
// that applies `>= minScore`, the stable sort and the cut itself (vector-store.ts:212-221).  Searches for any number of
// hits do not need it: rbk_index_search_unbounded_f64 sorts on the device and copies back only the answer, which is far
// faster than this route's 8 bytes per row and query over PCIe plus a host sort.  Kept simple: one fp64 pass per query.
template <typename XT>
__global__ void __launch_bounds__(256) exact_scores_kernel(const uint16_t* __restrict__ rows,
                                                           const XT* __restrict__ rows_f64,
                                                           const double* __restrict__ row_norm2,
                                                           const unsigned int* __restrict__ dead_bits, int64_t n_rows,
                                                           int d, int dpad, const double* __restrict__ q_f64,
                                                           const double* __restrict__ q_norm2,
                                                           double* __restrict__ out) {
  const int64_t row = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int q = blockIdx.y;
  if (row >= n_rows) return;
  double sc = __longlong_as_double(0x7FF8000000000000ll);
  if (!((dead_bits[row >> 5] >> (row & 31)) & 1u)) {
    const double* qv = q_f64 + static_cast<size_t>(q) * d;
    const double dot = rows_f64 != nullptr ? exact_dot_f64(qv, rows_f64 + static_cast<size_t>(row) * d, d,
                                                           rows + static_cast<size_t>(row) * dpad)
                                           : exact_dot(qv, rows + static_cast<size_t>(row) * dpad, d);
    sc = exact_cosine(dot, q_norm2[q], row_norm2[row]);
  }
  out[static_cast<size_t>(q) * n_rows + row] = sc;
}

// --------------------------------------------------------------------------- shard merge
// Lists are sorted by (score desc, slot asc); slots are globally unique, so the rank of an
// entry in the merged order is its own index plus, for every other list, the number of
// entries of that list that come before it (binary search).
__global__ void __launch_bounds__(128) merge_shards_kernel(int G, int B, int k, const char* __restrict__ slots_base,
                                                           const char* __restrict__ scores_base,
                                                           const char* __restrict__ counts_base,
                                                           const char* __restrict__ flags_base, size_t slots_stride,
                                                           size_t scores_stride, size_t counts_stride,
                                                           size_t flags_stride, long long* out_slots,
                                                           double* out_scores, int* out_counts, int* out_flags,
                                                           const int* __restrict__ k_each) {
  // shard g's arrays start g * stride bytes after shard 0's (dense [G][...] arrays: stride = array size;
  // packed per-rank blocks, e.g. straight out of ONE all-gather: the same block stride for all three)
  auto slots_of = [&](int g) { return reinterpret_cast<const long long*>(slots_base + g * slots_stride); };
  auto scores_of = [&](int g) { return reinterpret_cast<const double*>(scores_base + g * scores_stride); };
  auto count_of = [&](int g, int b) { return reinterpret_cast<const int*>(counts_base + g * counts_stride)[b]; };
  const int b = blockIdx.x;
  int total = 0;
  for (int g = 0; g < G; ++g) total += count_of(g, b);
  const int k_b = k_each != nullptr ? k_each[b] : k;   // query b's cut; k is the row stride of every list
  const int n_out = total < k_b ? total : k_b;
  for (int i = threadIdx.x; i < G * k; i += blockDim.x) {
    const int g = i / k, e = i % k;
    if (e >= count_of(g, b)) continue;
    const size_t o = static_cast<size_t>(b) * k;
    const double sc = scores_of(g)[o + e];
    const long long sl = slots_of(g)[o + e];
    int rank = e;
    for (int g2 = 0; g2 < G; ++g2) {
      if (g2 == g) continue;
      const double* s2p = scores_of(g2) + o;
      const long long* l2p = slots_of(g2) + o;
      int lo = 0, hi = count_of(g2, b);
      while (lo < hi) {  // first index whose entry does NOT come before (sc, sl)
        const int mid = (lo + hi) >> 1;
        const double s2 = s2p[mid];
        const long long l2 = l2p[mid];
        if (s2 > sc || (s2 == sc && l2 < sl)) lo = mid + 1;
        else hi = mid;
      }
      rank += lo;
    }
    if (rank < k_b) {
      out_slots[o + rank] = sl;
      out_scores[o + rank] = sc;
    }
  }
  for (int i = n_out + threadIdx.x; i < k; i += blockDim.x) {
    out_slots[static_cast<size_t>(b) * k + i] = -1;
    out_scores[static_cast<size_t>(b) * k + i] = __longlong_as_double(0x7FF8000000000000ll);
  }
  if (threadIdx.x == 0) {
    out_counts[b] = n_out;
    if (out_flags != nullptr) {
      // "not provably exact" travels with the lists: a query is dirty if any shard's proof failed.  out_flags[B]
      // counts dirty queries across calls (the caller zeroes it), so a pipelined caller can check once at the end.
      int dirty = 0;
      for (int g = 0; g < G; ++g) dirty |= reinterpret_cast<const int*>(flags_base + g * flags_stride)[b];
      out_flags[b] = dirty;
      if (dirty) atomicAdd(out_flags + B, 1);
    }
  }
}

}  // namespace

template <typename SrcT, bool kNorm2, bool kEach = false>
void launch_prep_typed(const SrcT* src, bool f16, int B, int d, int dpad, double min_score, double acc_eps,
                       const float* eps_c, const QueryBuffers& qb, cudaStream_t stream, unsigned int* scratch, int Bs,
                       int n_progress, const double* min_each) {
  if (f16)
    prep_queries_kernel<SrcT, kNorm2, true, kEach><<<B, 128, 0, stream>>>(src, d, dpad, min_score, acc_eps, eps_c, qb,
                                                                          scratch, Bs, n_progress, min_each);
  else
    prep_queries_kernel<SrcT, kNorm2, false, kEach><<<B, 128, 0, stream>>>(src, d, dpad, min_score, acc_eps, eps_c, qb,
                                                                           scratch, Bs, n_progress, min_each);
}

cudaError_t launch_prep_queries(const void* src, int src_type, int B, int d, int dpad, double min_score,
                                const float* eps_c, const QueryBuffers& qb, cudaStream_t stream, bool with_norm2,
                                unsigned int* scratch, int Bs, int n_progress, bool f16, const double* min_each) {
  if (B <= 0) return cudaSuccess;
  const double acc_eps = accumulation_eps(d);
  const double* sd = static_cast<const double*>(src);
  const float* sf = static_cast<const float*>(src);
  if (min_each != nullptr) {   // rbk_index_search_each_f64 takes float64 queries only
    if (src_type != 0) return cudaErrorInvalidValue;
    if (with_norm2)
      launch_prep_typed<double, true, true>(sd, f16, B, d, dpad, min_score, acc_eps, eps_c, qb, stream, scratch, Bs,
                                            n_progress, min_each);
    else
      launch_prep_typed<double, false, true>(sd, f16, B, d, dpad, min_score, acc_eps, eps_c, qb, stream, scratch, Bs,
                                             n_progress, min_each);
  } else if (src_type == 0) {
    if (with_norm2)
      launch_prep_typed<double, true>(sd, f16, B, d, dpad, min_score, acc_eps, eps_c, qb, stream, scratch, Bs, n_progress,
                                      nullptr);
    else
      launch_prep_typed<double, false>(sd, f16, B, d, dpad, min_score, acc_eps, eps_c, qb, stream, scratch, Bs,
                                       n_progress, nullptr);
  } else {
    if (with_norm2)
      launch_prep_typed<float, true>(sf, f16, B, d, dpad, min_score, acc_eps, eps_c, qb, stream, scratch, Bs, n_progress,
                                     nullptr);
    else
      launch_prep_typed<float, false>(sf, f16, B, d, dpad, min_score, acc_eps, eps_c, qb, stream, scratch, Bs,
                                      n_progress, nullptr);
  }
  return cudaGetLastError();
}

cudaError_t launch_finalize(const FinalizeParams& p_in, bool rows_on_host, int x_elem, cudaStream_t stream) {
  if (p_in.B <= 0) return cudaSuccess;
  FinalizeParams p = p_in;
  // >= 2048 keys (16 KB: room for 128 candidate rows x 56 elements per re-rank chunk)
  p.key_cap = p.B <= 160 ? 16384 : (p.B <= 320 ? 8192 : 2048);
  const size_t smem = static_cast<size_t>(p.key_cap) * 8;
  using namespace entry;
  auto kernel = x_elem == 4   ? (rows_on_host ? finalize_f32_kernel<true> : finalize_f32_kernel<false>)
                : x_elem == 2 ? (rows_on_host ? finalize_split_kernel<true> : finalize_split_kernel<false>)
                              : (rows_on_host ? finalize_kernel<true> : finalize_kernel<false>);
  if (p.k_each != nullptr)   // rbk_index_search_each_f64 sets both arrays or neither
    kernel = x_elem == 4   ? (rows_on_host ? finalize_each_kernel<true, 4> : finalize_each_kernel<false, 4>)
             : x_elem == 2 ? (rows_on_host ? finalize_each_kernel<true, 2> : finalize_each_kernel<false, 2>)
                           : (rows_on_host ? finalize_each_kernel<true, 8> : finalize_each_kernel<false, 8>);
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 16384 * 8);
  if (e != cudaSuccess) return e;
  kernel<<<p.B, kFinThreads, smem, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_exact_fallback(const ExactParams& p, int x_elem, cudaStream_t stream) {
  if (p.n_fail <= 0) return cudaSuccess;
  dim3 grid(p.n_blocks, p.n_fail);
  if (p.k_each != nullptr) {   // rbk_index_search_each_f64 sets both arrays or neither
    if (x_elem == 4) exact_scan_each_kernel<4><<<grid, kExThreads, 0, stream>>>(p);
    else if (x_elem == 2) exact_scan_each_kernel<2><<<grid, kExThreads, 0, stream>>>(p);
    else exact_scan_each_kernel<8><<<grid, kExThreads, 0, stream>>>(p);
  } else if (x_elem == 4) {
    exact_scan_kernel<float><<<grid, kExThreads, 0, stream>>>(p);
  } else if (x_elem == 2) {
    exact_scan_kernel<F32Lo><<<grid, kExThreads, 0, stream>>>(p);
  } else {
    exact_scan_kernel<double><<<grid, kExThreads, 0, stream>>>(p);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  exact_merge_kernel<<<p.n_fail, kExThreads, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_exact_scores(const uint16_t* rows, const void* rows_x, int x_elem, const double* row_norm2,
                                const unsigned int* dead_bits, int64_t n_rows, int d, int dpad, const double* q_f64,
                                const double* q_norm2, int B, double* out, cudaStream_t stream) {
  if (B <= 0 || n_rows <= 0) return cudaSuccess;
  dim3 grid(static_cast<unsigned>((n_rows + 255) / 256), static_cast<unsigned>(B));
  if (x_elem == 4)
    exact_scores_kernel<float><<<grid, 256, 0, stream>>>(rows, static_cast<const float*>(rows_x), row_norm2, dead_bits,
                                                         n_rows, d, dpad, q_f64, q_norm2, out);
  else if (x_elem == 2)
    exact_scores_kernel<F32Lo><<<grid, 256, 0, stream>>>(rows, static_cast<const F32Lo*>(rows_x), row_norm2, dead_bits,
                                                         n_rows, d, dpad, q_f64, q_norm2, out);
  else
    exact_scores_kernel<double><<<grid, 256, 0, stream>>>(rows, static_cast<const double*>(rows_x), row_norm2,
                                                          dead_bits, n_rows, d, dpad, q_f64, q_norm2, out);
  return cudaGetLastError();
}

cudaError_t launch_large_select(const unsigned int* hist, const float* thr_init, const float* inv_norm_q,
                                const double* q_eps, int B, int k_fetch, int n_rows, float* theta, int* cap,
                                cudaStream_t stream, const int* k_each) {
  if (B <= 0) return cudaSuccess;
  large_select_kernel<<<B, 256, 0, stream>>>(hist, thr_init, inv_norm_q, q_eps, k_fetch, n_rows, theta, cap, k_each);
  return cudaGetLastError();
}

cudaError_t launch_large_emit_all(const double* q_eps, const unsigned int* dead_bits, int64_t n_rows, int B,
                                  const long long* emit_off, int* emit_cnt, int* emit_rows, cudaStream_t stream) {
  if (B <= 0 || n_rows <= 0) return cudaSuccess;
  dim3 grid(static_cast<unsigned>((n_rows + 255) / 256), static_cast<unsigned>(B));
  large_emit_all_kernel<<<grid, 256, 0, stream>>>(q_eps, dead_bits, n_rows, emit_off, emit_cnt, emit_rows);
  return cudaGetLastError();
}

namespace {
// The exact re-score of every emitted candidate (launch_large_rerank, launch_pairs_rerank).
cudaError_t launch_large_score(const LargeRerankParams& p, int max_cap, bool rows_on_host, int x_elem,
                               cudaStream_t stream, int* launches) {
  using namespace entry;
  if (max_cap <= 0) return cudaSuccess;
  dim3 grid(static_cast<unsigned>((max_cap + 255) / 256), static_cast<unsigned>(p.B));
  if (x_elem == 4) {
    if (rows_on_host) large_score_f32_kernel<true><<<grid, 256, 0, stream>>>(p);
    else large_score_f32_kernel<false><<<grid, 256, 0, stream>>>(p);
  } else if (x_elem == 2) {
    if (rows_on_host) large_score_split_kernel<true><<<grid, 256, 0, stream>>>(p);
    else large_score_split_kernel<false><<<grid, 256, 0, stream>>>(p);
  } else {
    if (rows_on_host) large_score_kernel<true><<<grid, 256, 0, stream>>>(p);
    else large_score_kernel<false><<<grid, 256, 0, stream>>>(p);
  }
  ++*launches;
  return cudaGetLastError();
}

// The segmented sort's tile sort and merge passes; *passes: merge passes run (the sorted runs end in buffer
// passes & 1).
cudaError_t launch_seg_sort(const LargeRerankParams& p, const SegSortScratch& s, cudaStream_t stream, int* launches,
                            int* passes) {
  *passes = 0;
  if (s.max_tiles <= 0) return cudaSuccess;
  const size_t smem = static_cast<size_t>(kSortTile) * (sizeof(double) + sizeof(int));
  cudaError_t e = cudaFuncSetAttribute(seg_tile_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  const dim3 grid(static_cast<unsigned>(s.max_tiles), static_cast<unsigned>(p.B));
  seg_tile_sort_kernel<<<grid, kSortThreads, smem, stream>>>(p, s);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  ++*launches;
  for (; (1 << *passes) < s.max_tiles; ++*passes) {
    if (p.k_each != nullptr) seg_merge_kernel<true><<<grid, kMergeThreads, 0, stream>>>(p, s, *passes);
    else seg_merge_kernel<<<grid, kMergeThreads, 0, stream>>>(p, s, *passes);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    ++*launches;
  }
  return cudaSuccess;
}
}  // namespace

cudaError_t launch_large_rerank(const LargeRerankParams& p, const SegSortScratch* sort, int max_cap,
                                bool rows_on_host, int x_elem, cudaStream_t stream, int* launches) {
  *launches = 0;
  if (p.B <= 0) return cudaSuccess;
  cudaError_t e = launch_large_score(p, max_cap, rows_on_host, x_elem, stream, launches);
  if (e != cudaSuccess) return e;
  if (!sort) {   // the cut in shared memory, one block per query
    int S = 2048;
    while (S < p.k_fetch + kTopThreads) S <<= 1;
    const size_t smem = static_cast<size_t>(S) * (sizeof(double) + sizeof(int));
    e = cudaFuncSetAttribute(large_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    large_topk_kernel<<<p.B, kTopThreads, smem, stream>>>(p, S);
    ++*launches;
    return cudaGetLastError();
  }
  const SegSortScratch& s = *sort;
  int passes = 0;
  if ((e = launch_seg_sort(p, s, stream, launches, &passes)) != cudaSuccess) return e;
  const long long need = (p.k_fetch + 255ll) / 256;
  const int wblocks = need < 1024 ? static_cast<int>(need) : 1024;
  seg_write_kernel<<<dim3(static_cast<unsigned>(wblocks), static_cast<unsigned>(p.B)), 256, 0, stream>>>(p, s,
                                                                                                       passes & 1);
  ++*launches;
  return cudaGetLastError();
}

cudaError_t launch_pairs_rerank(const LargeRerankParams& p_in, const SegSortScratch& s, int max_cap, bool rows_on_host,
                                int x_elem, const PairsParams& pp, cudaStream_t stream, int* launches) {
  *launches = 0;
  if (p_in.B <= 0) return cudaSuccess;
  if (p_in.B > kPairsScanThreads) return cudaErrorInvalidValue;
  LargeRerankParams p = p_in;
  p.k_fetch = INT_MAX;   // no cut: every pair is kept
  p.k_each = nullptr;
  cudaError_t e = launch_large_score(p, max_cap, rows_on_host, x_elem, stream, launches);
  if (e != cudaSuccess) return e;
  const int cap_blocks = (max_cap + 255) / 256;
  const unsigned blocks = static_cast<unsigned>(cap_blocks < 1024 ? cap_blocks : 1024);
  if (max_cap > 0) {
    pairs_mask_kernel<<<dim3(static_cast<unsigned>(cap_blocks), static_cast<unsigned>(p.B)), 256, 0, stream>>>(p, pp);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    ++*launches;
  }
  int passes = 0;
  if ((e = launch_seg_sort(p, s, stream, launches, &passes)) != cudaSuccess) return e;
  pairs_offsets_kernel<<<1, kPairsScanThreads, 0, stream>>>(p, s, passes & 1, pp);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  ++*launches;
  if (max_cap > 0) {
    pairs_write_kernel<<<dim3(blocks, static_cast<unsigned>(p.B)), 256, 0, stream>>>(p, s, passes & 1, pp);
    ++*launches;
  }
  return cudaGetLastError();
}

cudaError_t launch_merge_shards(int G, int B, int k_fetch, const void* slots, const void* scores, const void* counts,
                                const void* flags, size_t slots_stride, size_t scores_stride, size_t counts_stride,
                                size_t flags_stride, long long* out_slots, double* out_scores, int* out_counts,
                                int* out_flags, cudaStream_t stream, const int* k_each) {
  if (B <= 0) return cudaSuccess;
  merge_shards_kernel<<<B, 128, 0, stream>>>(G, B, k_fetch, static_cast<const char*>(slots),
                                             static_cast<const char*>(scores), static_cast<const char*>(counts),
                                             static_cast<const char*>(flags), slots_stride, scores_stride,
                                             counts_stride, flags_stride, out_slots, out_scores, out_counts,
                                             flags ? out_flags : nullptr, k_each);
  return cudaGetLastError();
}

}  // namespace rbk
