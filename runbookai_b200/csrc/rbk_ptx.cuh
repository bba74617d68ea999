// rbk_ptx.cuh — thin inline-PTX wrappers for the sm_90a features the scan kernel uses:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (fence / mma_async / commit / wait) and the
// shared-memory matrix descriptor.  Hand-written for this engine; bit layouts follow the
// PTX ISA tables for wgmma descriptors (see DESIGN.md §5).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace rbk {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must surface as a trapped kernel (cudaErrorLaunchFailure
// -> RBK_ECUDA), never as a hung GPU.  ~2^31 cycles is seconds; real waits are micro-
// seconds.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (((++spins) & 0x3FFu) == 0 && (clock64() - t0) > (1ll << 31)) __trap();
  }
}

// Adds 1 to a shared-memory counter and returns its old value.  acq_rel at CTA scope: the add releases what this thread
// did or observed before it and acquires what every earlier adder had released, as an mbarrier arrive + wait pair does.
__device__ __forceinline__ uint32_t smem_inc_acq_rel(uint32_t addr) {
  uint32_t old;
  asm volatile("atom.acq_rel.cta.shared::cta.add.u32 %0, [%1], 1;" : "=r"(old) : "r"(addr) : "memory");
  return old;
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
// 2D tiled load global -> shared, completion on an mbarrier (complete_tx::bytes).
// crd0 = innermost (element) coordinate, crd1 = row coordinate.
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const void* tmap, uint32_t bar, int32_t crd0,
                                            int32_t crd1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      :
      : "r"(smem_dst), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(bar), "r"(crd0), "r"(crd1)
      : "memory");
}

// 1D bulk copy global -> shared (bytes and both addresses multiples of 16), completion on an mbarrier.
__device__ __forceinline__ void bulk_load(uint32_t smem_dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :
               : "r"(smem_dst), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(bar)
               : "memory");
}

// ---------------------------------------------------------------- wgmma
// Orders earlier register / shared-memory writes before the wgmma that follow (required before the first
// wgmma of a batch that accumulates into registers).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// Wait until at most N committed groups of this warpgroup are pending.  The accumulator registers are in/out
// operands so that no read of them is scheduled before the wait.
template <int N>
__device__ __forceinline__ void wgmma_wait(float (&d)[128]) {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
#pragma unroll
  for (int i = 0; i < 128; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor, K-major operand, 128-byte swizzle, rows of 64 bf16 (128 B) packed
// densely: 8-row groups are 1024 B apart (SBO); LBO is unused for swizzled K-major layouts (encoded 1);
// layout type [62,64) = 1 (SWIZZLE_128B).  Advancing K by 16 elements = +32 B = +2 in the address field.
__device__ __forceinline__ uint64_t make_sw128_kmajor_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);  // [0,14)  start address >> 4
  d |= static_cast<uint64_t>(1) << 16;                      // [16,30) leading byte offset >> 4
  d |= static_cast<uint64_t>(1024 >> 4) << 32;              // [32,46) stride byte offset >> 4
  d |= static_cast<uint64_t>(1) << 62;                      // [62,64) SWIZZLE_128B
  return d;
}

// The 128 accumulator operands of an m64n256 wgmma: "{%0, ..., %127}" and their "+f" constraints.
#define RBK_WGMMA_D128                                                                                              \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "                                         \
  "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "                                \
  "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "                                \
  "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "                                \
  "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "                                \
  "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "                                \
  "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "                    \
  "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}"
#define RBK_WGMMA_D128_OUT(d)                                                                                         \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),      \
      "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),         \
      "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),        \
      "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),        \
      "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),        \
      "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),        \
      "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),        \
      "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]),        \
      "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]),        \
      "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]),        \
      "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]),        \
      "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]),        \
      "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]),   \
      "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),              \
      "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]),              \
      "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]),              \
      "+f"(d[126]), "+f"(d[127])

// D[64 x 256] (+)= A[smem, 64 x 16] * B[smem, 256 x 16]^T, bf16 x bf16 -> fp32 in registers; warpgroup-collective
// and asynchronous (wgmma_commit / wgmma_wait).  Thread t of the warpgroup holds d[4j + 2h + e] = D[16 * (t / 32) +
// (t % 32) / 4 + 8h][8j + 2 * (t % 4) + e].
__device__ __forceinline__ void wgmma_m64n256k16_bf16(float (&d)[128], uint64_t desc_a, uint64_t desc_b,
                                                      uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 " RBK_WGMMA_D128 ", %128, %129, p, 1, 1, 0, 0;\n\t}"
      : RBK_WGMMA_D128_OUT(d)
      : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}
// The same with fp16 operands (RBK_INDEX_SCAN_F16): same shapes, descriptors, fragment layout and fp32 accumulation.
__device__ __forceinline__ void wgmma_m64n256k16_f16(float (&d)[128], uint64_t desc_a, uint64_t desc_b,
                                                     uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 " RBK_WGMMA_D128 ", %128, %129, p, 1, 1, 0, 0;\n\t}"
      : RBK_WGMMA_D128_OUT(d)
      : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}

// One lane of a converged warp: the TMA issue runs with the WHOLE warp (uniform control flow, operands in
// uniform registers) and elects a lane only around the asynchronous instruction itself.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xFFFFFFFF;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- misc
// Per-warp register budget of the executing warpgroup (warpgroup-collective; N a multiple of 8 in [24, 256]).  What
// one warpgroup gives back (dec) another can take (inc) as long as the CTA's total stays what it was launched with.
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// Order-preserving map float -> u32 (larger float -> larger integer; NaN never packed).
__device__ __forceinline__ uint32_t f32_ordered(float f) {
  uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float f32_from_ordered(uint32_t o) {
  uint32_t u = (o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o;
  return __uint_as_float(u);
}
// Candidate key: (score desc, row asc) == larger key first.
__device__ __forceinline__ uint64_t pack_key(float score, uint32_t row) {
  return (static_cast<uint64_t>(f32_ordered(score)) << 32) | static_cast<uint64_t>(0xFFFFFFFFu - row);
}
__device__ __forceinline__ uint32_t key_row(uint64_t k) { return 0xFFFFFFFFu - static_cast<uint32_t>(k); }
__device__ __forceinline__ float key_score(uint64_t k) { return f32_from_ordered(static_cast<uint32_t>(k >> 32)); }

}  // namespace rbk
