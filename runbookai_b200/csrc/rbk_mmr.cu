// rbk_mmr.cu — the greedy selection of rbk_index_search_mmr_f64 (maximal marginal relevance) over candidate rows
// already staged as float64 on the device.
#include "rbk_internal.h"

namespace rbk {

namespace {

constexpr int kMmrThreads = 512;
constexpr int kMmrWarps = kMmrThreads / 32;
constexpr int kTileCols = 16;   // columns of a warp's tile of 32 candidate rows (padded by one against bank conflicts)
constexpr size_t kTileBytes = static_cast<size_t>(kMmrWarps) * 32 * (kTileCols + 1) * sizeof(double);

// Order-preserving bits of an mmr value under the selection's total order: NaN is 0, below every number, and both zeros
// map to +0's key, so that for numbers key(a) > key(b) iff a > b.
__device__ __forceinline__ unsigned long long mmr_key(double v) {
  if (v != v) return 0ull;
  if (v == 0.0) v = 0.0;
  const unsigned long long u = static_cast<unsigned long long>(__double_as_longlong(v));
  return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}

// (key, i) becomes (k2, i2) when that ranks first: the larger key, then the smaller index.
__device__ __forceinline__ void keep_better(unsigned long long& key, int& i, unsigned long long k2, int i2) {
  if (k2 > key || (k2 == key && i2 < i)) {
    key = k2;
    i = i2;
  }
}

// One block per query b: its m = off[b + 1] - off[b] candidates are rows [off[b], off[b + 1]) of x (pitch d), with
// global slots slot[] and relevances rel[] there.  Writes row b of out_slots / out_scores (K entries): the min(k_q[b],
// m) picks in selection order, then slot -1 / quiet NaN.  Shared memory per candidate: r, ||row||^2, red (8 bytes each)
// and a picked byte, after each warp's row tile.  Every dot chain runs sequentially over the row, as the reference's
// cosine does, so the parallelism is over candidates; the picked row, read by every thread, comes from L1 / L2.
__global__ void __launch_bounds__(kMmrThreads, 1)
    mmr_select_kernel(const double* __restrict__ x, int d, const int64_t* __restrict__ off,
                      const int64_t* __restrict__ slot, const double* __restrict__ rel, const int* __restrict__ k_q,
                      const double* __restrict__ lam_q, int K, int64_t* __restrict__ out_slots,
                      double* __restrict__ out_scores) {
  extern __shared__ double smem[];
  __shared__ unsigned long long w_key[kMmrWarps];
  __shared__ int w_idx[kMmrWarps];
  __shared__ int s_pick;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t o = off[b];
  const int m = static_cast<int>(off[b + 1] - o);
  const int k = min(k_q[b], m);
  const double lam = lam_q[b];
  double* tile = smem + static_cast<size_t>(warp) * 32 * (kTileCols + 1);
  double* s_r = smem + kTileBytes / sizeof(double);
  double* s_na = s_r + m;
  double* s_red = s_r + 2 * m;
  unsigned char* s_picked = reinterpret_cast<unsigned char*>(s_r + 3 * m);
  const double* xb = x + o * d;
  int64_t* os = out_slots + static_cast<int64_t>(b) * K;
  double* ov = out_scores + static_cast<int64_t>(b) * K;
  const double qnan = __longlong_as_double(0x7FF8000000000000ll);
  for (int t = k + tid; t < K; t += kMmrThreads) {
    os[t] = -1;
    ov[t] = qnan;
  }
  if (k == 0) return;
  for (int i = tid; i < m; i += kMmrThreads) {
    s_r[i] = rel[o + i];
    s_red[i] = qnan;
    s_picked[i] = i == 0;
  }
  if (tid == 0) {   // the first pick is c_0
    os[0] = slot[o];
    ov[0] = rel[o];
  }
  __syncthreads();
  const double t1 = __dsub_rn(1.0, lam);
  int p = 0;
  for (int step = 1; step < k; ++step) {
    const double* xp = xb + static_cast<int64_t>(p) * d;
    unsigned long long bkey = 0ull;
    int bi = INT_MAX;
    // warp w takes candidates i0 + lane for i0 = 32 w, 32 w + kMmrThreads, ...: the 32 rows come through the warp's
    // shared tile kTileCols columns at a time, read row-contiguously (coalesced), and lane l runs candidate i0 + l's
    // chains over the tile's columns in order
    for (int i0 = warp * 32; i0 < m; i0 += kMmrThreads) {
      const int i = i0 + lane;
      const bool mine = i < m && (step == 1 || !s_picked[i]);
      if (!__any_sync(0xffffffffu, mine)) continue;
      double dot = 0.0, na = 0.0, nb = 0.0;
      for (int c0 = 0; c0 < d; c0 += kTileCols) {
        const int nc = min(kTileCols, d - c0);
#pragma unroll
        for (int rr = 0; rr < 32; rr += 32 / kTileCols) {
          const int r = rr + lane / kTileCols, c = lane % kTileCols;
          if (i0 + r < m && c < nc) tile[r * (kTileCols + 1) + c] = xb[static_cast<int64_t>(i0 + r) * d + c0 + c];
        }
        __syncwarp();
        const double* t = tile + lane * (kTileCols + 1);
        const double* pc = xp + c0;
        if (step == 1) {
          // the reference's cosine with c_0 as it stands: its three chains in one pass; ||row i||^2 is kept for later
          // steps (c_0's own too, which is why the picked row is not skipped here)
          for (int j = 0; j < nc; ++j) {
            const double a = t[j], c = pc[j];
            dot = __dadd_rn(dot, __dmul_rn(a, c));
            na = __dadd_rn(na, __dmul_rn(a, a));
            nb = __dadd_rn(nb, __dmul_rn(c, c));
          }
        } else {
#pragma unroll 4
          for (int j = 0; j < nc; ++j) dot = __dadd_rn(dot, __dmul_rn(t[j], pc[j]));
        }
        __syncwarp();
      }
      if (!mine) continue;
      double s;
      if (step == 1) {
        s_na[i] = na;
        if (i == 0) continue;
        s = __ddiv_rn(dot, __dmul_rn(__dsqrt_rn(na), __dsqrt_rn(nb)));
      } else {
        s = __ddiv_rn(dot, __dmul_rn(__dsqrt_rn(s_na[i]), __dsqrt_rn(s_na[p])));
      }
      double red = s_red[i];
      if (red != red || s > red) {
        red = s;
        s_red[i] = red;
      }
      const double v = __dsub_rn(__dmul_rn(lam, s_r[i]), __dmul_rn(t1, red));
      keep_better(bkey, bi, mmr_key(v), i);
    }
    // the order is total, so any reduction order finds the same pick
#pragma unroll
    for (int sh = 16; sh > 0; sh >>= 1)
      keep_better(bkey, bi, __shfl_xor_sync(0xffffffffu, bkey, sh), __shfl_xor_sync(0xffffffffu, bi, sh));
    if (lane == 0) {
      w_key[warp] = bkey;
      w_idx[warp] = bi;
    }
    __syncthreads();
    if (warp == 0) {
      bkey = lane < kMmrWarps ? w_key[lane] : 0ull;
      bi = lane < kMmrWarps ? w_idx[lane] : INT_MAX;
#pragma unroll
      for (int sh = 16; sh > 0; sh >>= 1)
        keep_better(bkey, bi, __shfl_xor_sync(0xffffffffu, bkey, sh), __shfl_xor_sync(0xffffffffu, bi, sh));
      if (lane == 0) {
        s_pick = bi;
        s_picked[bi] = 1;
        os[step] = slot[o + bi];
        ov[step] = s_r[bi];
      }
    }
    __syncthreads();
    p = s_pick;
  }
}

}  // namespace

size_t mmr_smem_bytes(int max_m) { return kTileBytes + static_cast<size_t>(max_m) * (3 * sizeof(double) + 1); }

cudaError_t launch_mmr_select(const double* x, int d, const int64_t* off, const int64_t* slot, const double* rel,
                              const int* k, const double* lambda_mult, int B, int max_m, int K, int64_t* out_slots,
                              double* out_scores, cudaStream_t stream) {
  if (B <= 0) return cudaSuccess;
  const size_t smem = mmr_smem_bytes(max_m);
  cudaError_t e = cudaFuncSetAttribute(mmr_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(smem));
  if (e != cudaSuccess) return e;
  mmr_select_kernel<<<B, kMmrThreads, smem, stream>>>(x, d, off, slot, rel, k, lambda_mult, K, out_slots, out_scores);
  return cudaGetLastError();
}

}  // namespace rbk
