// Inline-PTX wrappers for the Hopper (sm_90a) async machinery the tensor-core kernels use: mbarrier, TMA
// (cp.async.bulk.tensor), the warp-level tf32 tensor-core MMA (mma.sync m16n8k8) and the warpgroup one (wgmma), and the
// host-side lookup of the driver's tensor-map encoder.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace dv {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier ---------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// Bounded spin: a pipeline bug traps (kernel error) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t done = 0;
  for (uint32_t spin = 0; !done; ++spin) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
    if (spin > (1u << 24)) __trap();
  }
}

// ---- named barriers -----------------------------------------------------------------
// Barrier `id` completes once `count` threads (whole warps) have reached it: bar.sync counts this warp and waits,
// bar.arrive counts it and goes on (the signalling side of a producer / consumer hand-off).
__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(int id, int count) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// one 32-bit word of shared memory (explicit ld.shared: 32-bit address arithmetic)
__device__ __forceinline__ uint32_t lds32(uint32_t smem_addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(smem_addr) : "memory");
  return v;
}

// four consecutive 32-bit words of shared memory (16-byte aligned address)
__device__ __forceinline__ void sts128(uint32_t smem_addr, const uint32_t (&v)[4]) {
  asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(smem_addr), "r"(v[0]), "r"(v[1]), "r"(v[2]), "r"(v[3]) : "memory");
}
// Orders this thread's earlier shared-memory stores (generic proxy) before later reads of the async proxy: a wgmma
// whose descriptor points at a tile that threads wrote themselves, not TMA.  Followed by a barrier among the writers.
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// Byte offset of fp32 element (row r, column c < 32) in a tile of 128-byte rows written by TMA with
// CU_TENSOR_MAP_SWIZZLE_128B into a 1024-byte aligned buffer: the 16-byte chunk index is XOR-ed with (r & 7).
__device__ __forceinline__ uint32_t swz128(int r, int c) {
  return (uint32_t)(r * 128 + ((((c >> 2) ^ (r & 7)) << 4) | ((c & 3) << 2)));
}

// ---- TMA ------------------------------------------------------------------------------
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// L2 prefetch of a tensor-map box (no shared-memory destination, no completion tracking): hides the HBM leg of
// the latency of a TMA load that will be issued a tile later.
__device__ __forceinline__ void tma_prefetch_4d(const CUtensorMap* m, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.prefetch.tensor.4d.L2.global.tile [%0, {%1, %2, %3, %4}];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}

// Host side: the driver's cuTensorMapEncodeTiled, looked up once per process through the runtime (no -lcuda);
// nullptr if the driver does not provide it.
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline EncodeTiledFn get_encode() {
  static const EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    const bool ok = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
                    qres == cudaDriverEntryPointSuccess;
    return ok ? reinterpret_cast<EncodeTiledFn>(p) : nullptr;
  }();
  return fn;
}

// ---- tf32 tensor-core MMA -----------------------------------------------------------------
// Error-compensated 3xTF32: x = hi + lo with hi = x rounded to the nearest tf32 and lo = x - hi (exact in fp32,
// |lo| <= 2^-11 |x|), itself rounded to the nearest tf32; a*b ~ a_hi*b_hi + (a_hi*b_lo + a_lo*b_hi), the lo*lo term is
// below fp32 rounding.  Rounding both planes to nearest (not truncating) keeps the residual error of a product near
// 2^-22 of it and unbiased: a truncated split leaves an error of one sign in every product, which accumulates over
// long reductions.
// Nearest tf32, ties away from zero (what cvt.rna.tf32.f32 computes), as two full-rate integer operations on the
// sign-magnitude bit pattern: add half a tf32 ulp, clear the 13 low mantissa bits.
__device__ __forceinline__ float tf32_round(float x) {
  return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
}
__device__ __forceinline__ void split_tf32(uint32_t x, uint32_t& hi, uint32_t& lo) {
  const float h = tf32_round(__uint_as_float(x));
  hi = __float_as_uint(h);
  lo = __float_as_uint(tf32_round(__uint_as_float(x) - h));
}

// D[16x8] += A[16x8] * B[8x8] (tf32 operands, fp32 accumulate).  With g = lane >> 2, t = lane & 3:
//   a = {A[g][t], A[g+8][t], A[g][t+4], A[g+8][t+4]},  b = {B[t][g], B[t+4][g]},
//   d = {D[g][2t], D[g][2t+1], D[g+8][2t], D[g+8][2t+1]}.
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// main += a_hi * b_hi;  corr += a_hi * b_lo + a_lo * b_hi.  The correction products accumulate apart from the main
// one, so they are not rounded at its magnitude.
__device__ __forceinline__ void mma_3xtf32(float (&main)[4], float (&corr)[4], const uint32_t (&a_hi)[4],
                                           const uint32_t (&a_lo)[4], const uint32_t (&b_hi)[2], const uint32_t (&b_lo)[2]) {
  mma_tf32(main, a_hi, b_hi);
  mma_tf32(corr, a_hi, b_lo);
  mma_tf32(corr, a_lo, b_hi);
}

// ---- warpgroup tf32 MMA (wgmma), A from registers -------------------------------------------
// Shared-memory descriptor of a K-major operand tile in the 128-byte swizzle layout (as TMA writes it): rows of 128 B (32 fp32
// of K), 8-row swizzle atoms 1024 B apart (stride byte offset), leading byte offset unused for a swizzled K-major tile.
// The k8 slice ks of a tile starts 32*ks bytes into the tile (the hardware applies the swizzle to the full address).
__device__ __forceinline__ uint64_t wgmma_desc_k128(uint32_t smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Pins the order of register accesses around the asynchronous MMAs (the compiler does not know that the registers of
// an issued wgmma change until its wait_group).
template <int N>
__device__ __forceinline__ void fence_regs(float (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}

// D[64 x 32] (+)= A[64 x 8] * B[8 x 32], tf32 operands, fp32 accumulate, issued by a whole warpgroup.  A per warp
// (rows 16*(warp%4) + ...) in the m16n8k8 layout of mma_tf32; D per warp in the m16n8 layout repeated along N:
// d[4j + e] = D[g + 8(e>>1)][8j + 2t + (e&1)].  B: descriptor of the 32 x 8 K-major slice.  accumulate == 0 overwrites D.
__device__ __forceinline__ void wgmma_m64n32k8_rs(float (&d)[16], const uint32_t* a, uint64_t b_desc, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "{%16, %17, %18, %19}, %20, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate));
}

}  // namespace ptx
}  // namespace dv
