// Thin inline-PTX layer for sm_90a (Hopper): mbarrier, TMA (cp.async.bulk.tensor), warpgroup MMA (wgmma.mma_async)
// with shared-memory matrix descriptors or a register A operand, stmatrix, setmaxnreg, the row view of a wgmma
// accumulator used by the epilogues, system-scope
// release/acquire for the peer-memory (NVLink) kernels, and the GELU math shared by the kernels.
//
// Descriptor encodings follow the PTX ISA ("Matrix Descriptor Format" of wgmma): canonical SWIZZLE_128B layouts,
// K-major "Swizzle<3,4,3> o ((8,m),(T,2k)):((8T,SBO),(1,T))" and MN-major "((T,8,m),(8,k)):((1,T,LBO),(8T,SBO))"
// in 16-byte units.  Nothing here depends on CUTLASS at compile time.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace dfno {

// ------------------------------------------------------------------------------------------
// generic helpers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ------------------------------------------------------------------------------------------
// mbarrier
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// one lane polls, the warp follows: 128 threads spinning on try_wait slow every other mbarrier operation down
__device__ __forceinline__ void mbar_wait_warp(uint64_t* bar, uint32_t parity) {
  if ((threadIdx.x & 31) == 0) mbar_wait(bar, parity);
  __syncwarp();
}

// ------------------------------------------------------------------------------------------
// TMA
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];\n" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2-D tiled load: coordinates are (c0 = innermost element index, c1 = row index)
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar,
                                            int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];\n" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// 3-D tiled load: coordinates innermost first
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar,
                                            int32_t c0, int32_t c1, int32_t c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];\n" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// tiled stores (shared -> global, bulk async-group completion); out-of-range parts of the box are clipped
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];\n" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, const void* smem_src, int32_t c0, int32_t c1,
                                             int32_t c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];\n" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;\n" ::: "memory"); }
// the issuing thread's committed stores have finished READING shared memory (it may be overwritten)
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;\n" ::: "memory"); }
// ... and are complete (globally performed)
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;\n" ::: "memory"); }

// ------------------------------------------------------------------------------------------
// wgmma: shared-memory matrix descriptors (SWIZZLE_128B)
// ------------------------------------------------------------------------------------------
// start address [0,14), leading byte offset [16,30), stride byte offset [32,46) (all in 16-byte units),
// base offset [49,52) = 0 (every operand block is 1024-byte aligned), layout type [62,64) = 1 (SWIZZLE_128B).
__device__ __forceinline__ uint64_t gdesc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4) |
         (static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16) |
         (static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32) | (1ull << 62);
}
// K-major operand: rows of 128 bytes (64 16-bit elements along K), 8-row swizzle atoms stacked every 1024 bytes
// along M/N; LBO is unused by swizzled K-major layouts.  A k16 step inside the row advances the start by 32 bytes.
__device__ __forceinline__ uint64_t gdesc_k128(uint32_t smem_addr) { return gdesc(smem_addr, 16, 1024); }
// MN-major operand (the M/N index contiguous): an atom is 64 MN elements (128 B) x 8 K rows (1024 B); atoms repeat
// every SBO bytes along K and every LBO bytes along MN.
__device__ __forceinline__ uint64_t gdesc_mn128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return gdesc(smem_addr, lbo_bytes, sbo_bytes);
}

// ------------------------------------------------------------------------------------------
// wgmma: issue / ordering.  A warpgroup is four consecutive warps starting at a multiple of four; all 128 threads
// execute every call below with identical operands.
// ------------------------------------------------------------------------------------------
// Per-warpgroup register budget (all 128 threads execute it): a TMA producer warpgroup gives registers back so
// that the consumer warpgroups can hold fragments beyond the uniform per-thread limit of the launch.
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(N)); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }

// The accumulator of one warpgroup: R <= 128 fp32 registers per thread, i.e. a 128 x N tile (two m64 halves in
// acc[0, R/2) and acc[R/2, R), N <= R) or a 64 x N tile (N <= 2R).  Fragment of an m64nN instruction (PTX ISA, wgmma D layout): register
// 4j + e of thread (warp w, lane l) holds row 16w + l/4 + 8(e/2), column 8j + 2(l%4) + e%2.
constexpr int kAccRegs = 128;

// Keeps the compiler from moving accesses of the accumulator across wgmma_fence / wgmma_wait.
template <int R>
__device__ __forceinline__ void acc_fence(float (&acc)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(acc[i])::"memory");
}

// wgmma.mma_async m64nNk16, fp32 accumulators, both operands from shared memory
// DFNO_F<g>: the first 8g accumulator registers d[0 .. 8g) as asm operands; DFNO_R<g>: their asm names %0 .. %8g-1
#define DFNO_OP8(o) "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), \
                    "+f"(d[o + 6]), "+f"(d[o + 7])
#define DFNO_F1 DFNO_OP8(0)
#define DFNO_F2 DFNO_F1, DFNO_OP8(8)
#define DFNO_F3 DFNO_F2, DFNO_OP8(16)
#define DFNO_F4 DFNO_F3, DFNO_OP8(24)
#define DFNO_F5 DFNO_F4, DFNO_OP8(32)
#define DFNO_F6 DFNO_F5, DFNO_OP8(40)
#define DFNO_F7 DFNO_F6, DFNO_OP8(48)
#define DFNO_F8 DFNO_F7, DFNO_OP8(56)
#define DFNO_F9 DFNO_F8, DFNO_OP8(64)
#define DFNO_F10 DFNO_F9, DFNO_OP8(72)
#define DFNO_F11 DFNO_F10, DFNO_OP8(80)
#define DFNO_F12 DFNO_F11, DFNO_OP8(88)
#define DFNO_F13 DFNO_F12, DFNO_OP8(96)
#define DFNO_F14 DFNO_F13, DFNO_OP8(104)
#define DFNO_F15 DFNO_F14, DFNO_OP8(112)
#define DFNO_F16 DFNO_F15, DFNO_OP8(120)
#define DFNO_R1 "%0,%1,%2,%3,%4,%5,%6,%7"
#define DFNO_R2 DFNO_R1 "," "%8,%9,%10,%11,%12,%13,%14,%15"
#define DFNO_R3 DFNO_R2 "," "%16,%17,%18,%19,%20,%21,%22,%23"
#define DFNO_R4 DFNO_R3 "," "%24,%25,%26,%27,%28,%29,%30,%31"
#define DFNO_R5 DFNO_R4 "," "%32,%33,%34,%35,%36,%37,%38,%39"
#define DFNO_R6 DFNO_R5 "," "%40,%41,%42,%43,%44,%45,%46,%47"
#define DFNO_R7 DFNO_R6 "," "%48,%49,%50,%51,%52,%53,%54,%55"
#define DFNO_R8 DFNO_R7 "," "%56,%57,%58,%59,%60,%61,%62,%63"
#define DFNO_R9 DFNO_R8 "," "%64,%65,%66,%67,%68,%69,%70,%71"
#define DFNO_R10 DFNO_R9 "," "%72,%73,%74,%75,%76,%77,%78,%79"
#define DFNO_R11 DFNO_R10 "," "%80,%81,%82,%83,%84,%85,%86,%87"
#define DFNO_R12 DFNO_R11 "," "%88,%89,%90,%91,%92,%93,%94,%95"
#define DFNO_R13 DFNO_R12 "," "%96,%97,%98,%99,%100,%101,%102,%103"
#define DFNO_R14 DFNO_R13 "," "%104,%105,%106,%107,%108,%109,%110,%111"
#define DFNO_R15 DFNO_R14 "," "%112,%113,%114,%115,%116,%117,%118,%119"
#define DFNO_R16 DFNO_R15 "," "%120,%121,%122,%123,%124,%125,%126,%127"
// wgmma_m64n<N>k16_<TY>(d, da, db, scale_d): d = the N/2 accumulator registers; A, B, S, TA, TB are the asm
// operand numbers of the two descriptors, scale-d and the two transpose immediates (N/2 .. N/2 + 4)
#define DFNO_WGMMA(N, TY, REGS, A, B, S, TA, TB, ...)                                                        \
  template <int kTA, int kTB>                                                                               \
  __device__ __forceinline__ void wgmma_m64n##N##k16_##TY(float* d, uint64_t da, uint64_t db, uint32_t scale_d) { \
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %" #S ", 0;\nwgmma.mma_async.sync.aligned.m64n" #N "k16.f32." #TY  \
                 "." #TY " {" REGS "}, %" #A ", %" #B ", p, 1, 1, %" #TA ", %" #TB ";\n}\n"                        \
                 : __VA_ARGS__                                                                              \
                 : "l"(da), "l"(db), "r"(scale_d), "n"(kTA), "n"(kTB));                                  \
  }
DFNO_WGMMA(16, bf16, DFNO_R1, 8, 9, 10, 11, 12, DFNO_F1)
DFNO_WGMMA(16, f16, DFNO_R1, 8, 9, 10, 11, 12, DFNO_F1)
DFNO_WGMMA(32, bf16, DFNO_R2, 16, 17, 18, 19, 20, DFNO_F2)
DFNO_WGMMA(32, f16, DFNO_R2, 16, 17, 18, 19, 20, DFNO_F2)
DFNO_WGMMA(48, bf16, DFNO_R3, 24, 25, 26, 27, 28, DFNO_F3)
DFNO_WGMMA(48, f16, DFNO_R3, 24, 25, 26, 27, 28, DFNO_F3)
DFNO_WGMMA(64, bf16, DFNO_R4, 32, 33, 34, 35, 36, DFNO_F4)
DFNO_WGMMA(64, f16, DFNO_R4, 32, 33, 34, 35, 36, DFNO_F4)
DFNO_WGMMA(80, bf16, DFNO_R5, 40, 41, 42, 43, 44, DFNO_F5)
DFNO_WGMMA(80, f16, DFNO_R5, 40, 41, 42, 43, 44, DFNO_F5)
DFNO_WGMMA(96, bf16, DFNO_R6, 48, 49, 50, 51, 52, DFNO_F6)
DFNO_WGMMA(112, bf16, DFNO_R7, 56, 57, 58, 59, 60, DFNO_F7)
DFNO_WGMMA(128, bf16, DFNO_R8, 64, 65, 66, 67, 68, DFNO_F8)
DFNO_WGMMA(128, f16, DFNO_R8, 64, 65, 66, 67, 68, DFNO_F8)
DFNO_WGMMA(144, bf16, DFNO_R9, 72, 73, 74, 75, 76, DFNO_F9)
DFNO_WGMMA(160, bf16, DFNO_R10, 80, 81, 82, 83, 84, DFNO_F10)
DFNO_WGMMA(176, bf16, DFNO_R11, 88, 89, 90, 91, 92, DFNO_F11)
DFNO_WGMMA(192, bf16, DFNO_R12, 96, 97, 98, 99, 100, DFNO_F12)
DFNO_WGMMA(208, bf16, DFNO_R13, 104, 105, 106, 107, 108, DFNO_F13)
DFNO_WGMMA(224, bf16, DFNO_R14, 112, 113, 114, 115, 116, DFNO_F14)
DFNO_WGMMA(240, bf16, DFNO_R15, 120, 121, 122, 123, 124, DFNO_F15)
DFNO_WGMMA(256, bf16, DFNO_R16, 128, 129, 130, 131, 132, DFNO_F16)
#undef DFNO_WGMMA
#undef DFNO_OP8
#undef DFNO_F1
#undef DFNO_R1
#undef DFNO_F2
#undef DFNO_R2
#undef DFNO_F3
#undef DFNO_R3
#undef DFNO_F4
#undef DFNO_R4
#undef DFNO_F5
#undef DFNO_R5
#undef DFNO_F6
#undef DFNO_R6
#undef DFNO_F7
#undef DFNO_R7
#undef DFNO_F8
#undef DFNO_R8
#undef DFNO_F9
#undef DFNO_R9
#undef DFNO_F10
#undef DFNO_R10
#undef DFNO_F11
#undef DFNO_R11
#undef DFNO_F12
#undef DFNO_R12
#undef DFNO_F13
#undef DFNO_R13
#undef DFNO_F14
#undef DFNO_R14
#undef DFNO_F15
#undef DFNO_R15
#undef DFNO_F16
#undef DFNO_R16

// acc[OFF .. OFF + n/2) (+)= A[64 x 16] . B[16 x n] for a run-time n (a multiple of 16); widths whose registers would
// not fit between OFF and R are not instantiated.  kF16: fp16 inputs (the fp16 variants exist for n = 16, 32, 48, 64, 80
// and 128).
#define DFNO_WG_CASE(N)                                                                    \
  case N:                                                                                  \
    if constexpr (OFF + N / 2 <= R) wgmma_m64n##N##k16_bf16<TA, TB>(acc + OFF, da, db, scale_d); \
    break;
#define DFNO_WG_CASE16(N)                                                                  \
  case N:                                                                                  \
    if constexpr (OFF + N / 2 <= R) wgmma_m64n##N##k16_f16<TA, TB>(acc + OFF, da, db, scale_d); \
    break;
template <bool kF16, int TA, int TB, int OFF, int R>
__device__ __forceinline__ void wg_mma64(float (&acc)[R], int n, uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (kF16) {
    switch (n) {
      DFNO_WG_CASE16(16) DFNO_WG_CASE16(32) DFNO_WG_CASE16(48) DFNO_WG_CASE16(64) DFNO_WG_CASE16(80)
      DFNO_WG_CASE16(128) default: break;
    }
  } else {
    switch (n) {
      DFNO_WG_CASE(16) DFNO_WG_CASE(32) DFNO_WG_CASE(48) DFNO_WG_CASE(64) DFNO_WG_CASE(80) DFNO_WG_CASE(96)
      DFNO_WG_CASE(112) DFNO_WG_CASE(128) DFNO_WG_CASE(144) DFNO_WG_CASE(160) DFNO_WG_CASE(176) DFNO_WG_CASE(192)
      DFNO_WG_CASE(208) DFNO_WG_CASE(224) DFNO_WG_CASE(240) DFNO_WG_CASE(256)
      default: break;
    }
  }
}
#undef DFNO_WG_CASE
#undef DFNO_WG_CASE16

// D = A . B^T over `kblocks` >= 1 K blocks of 64 (four k16 steps each), both operands K-major (a_blk / b_blk bytes
// per block), N columns and kHalves m64 halves (rows 64..127 into acc[R/2, R)).  N and kHalves are compile-time
// constants and the k16 steps of a block are unrolled, so that the chain's wgmmas issue back to back with one commit
// and one wait: a width chosen per instruction makes ptxas serialise every wgmma (C7511), and a fully unrolled
// K loop runs out of (uniform) registers for the descriptors and is serialised too.  The block loop is a run-time
// loop with a fence per block; ptxas closes it with one extra arrive before the wait (C7519).
// `accumulate`: add to the accumulator instead of overwriting it (the second and later K chunks of one tile).
template <int N, int kHalves, int R>
__device__ __forceinline__ void mma_chain(float (&acc)[R], uint32_t a, uint32_t a_blk, uint32_t b, uint32_t b_blk,
                                          int kblocks, bool accumulate = false) {
  int kb = 0;
#pragma unroll 1
  do {
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const uint64_t da = gdesc_k128(a + kb * a_blk + kk * 32), db = gdesc_k128(b + kb * b_blk + kk * 32);
      const uint32_t scale_d = accumulate || kb > 0 || kk > 0 ? 1u : 0u;
      wg_mma64<false, 0, 0, 0>(acc, N, da, db, scale_d);
      if constexpr (kHalves == 2) wg_mma64<false, 0, 0, R / 2>(acc, N, da + (8192 >> 4), db, scale_d);
    }
  } while (++kb < kblocks);
  wgmma_commit();
  wgmma_wait<0>();
  acc_fence(acc);
}

// m64n8k16, fp16 inputs, both operands from shared memory: d = the 4 accumulator registers of an m64n8 tile
template <int kTA, int kTB>
__device__ __forceinline__ void wgmma_m64n8k16_f16(float (&d)[4], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %6, 0;\nwgmma.mma_async.sync.aligned.m64n8k16.f32.f16.f16 "
               "{%0,%1,%2,%3}, %4, %5, p, 1, 1, %7, %8;\n}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "l"(da), "l"(db), "r"(scale_d), "n"(kTA), "n"(kTB));
}

// One k16 step of a 128 x n tile (n <= R): rows 0..63 into acc[0, R/2), rows 64..127 into acc[R/2, R).
// `a_half_bytes` is the step to the second half of A (8192 B for a K-major block, LBO for an MN-major one).
template <bool kF16, int TA, int TB, int R>
__device__ __forceinline__ void wg_mma128(float (&acc)[R], int n, uint64_t da, uint32_t a_half_bytes, uint64_t db,
                                          uint32_t scale_d) {
  wg_mma64<kF16, TA, TB, 0>(acc, n, da, db, scale_d);
  wg_mma64<kF16, TA, TB, R / 2>(acc, n, da + (a_half_bytes >> 4), db, scale_d);
}

// wgmma.mma_async m64nNk16, fp16 inputs, fp32 accumulators, A from REGISTERS (a[4]: the m64k16 A fragment of this
// thread, see afrag_from_acc), B from shared memory.  N = 16 / 32 / 48.
#define DFNO_WGMMA_RS(N, REGS, A, B, S, TB, ...)                                                                \
  template <int kTB>                                                                                             \
  __device__ __forceinline__ void wgmma_m64n##N##k16_f16_rs(float* d, const uint32_t (&a)[4], uint64_t db,       \
                                                            uint32_t scale_d) {                                  \
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %" #S ", 0;\nwgmma.mma_async.sync.aligned.m64n" #N            \
                 "k16.f32.f16.f16 {" REGS "}, {" A "}, %" #B ", p, 1, 1, %" #TB ";\n}\n"                         \
                 : __VA_ARGS__                                                                                   \
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d), "n"(kTB));                 \
  }
DFNO_WGMMA_RS(16, "%0,%1,%2,%3,%4,%5,%6,%7", "%8,%9,%10,%11", 12, 13, 14,
              "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]))
DFNO_WGMMA_RS(32, "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15", "%16,%17,%18,%19", 20, 21, 22,
              "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]))
DFNO_WGMMA_RS(48,
              "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23",
              "%24,%25,%26,%27", 28, 29, 30,
              "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]))
#undef DFNO_WGMMA_RS

// acc[OFF .. OFF + N/2) (+)= A[64 x 16] (registers) . B[16 x N] (shared memory), N = 16, 32 or 48
template <int N, int TB, int OFF, int R>
__device__ __forceinline__ void wg_mma64_rs(float (&acc)[R], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  static_assert(OFF + N / 2 <= R, "accumulator too small");
  if constexpr (N == 16) wgmma_m64n16k16_f16_rs<TB>(acc + OFF, a, db, scale_d);
  else if constexpr (N == 32) wgmma_m64n32k16_f16_rs<TB>(acc + OFF, a, db, scale_d);
  else { static_assert(N == 48, "N = 16, 32 or 48"); wgmma_m64n48k16_f16_rs<TB>(acc + OFF, a, db, scale_d); }
}

// The accumulator fragment of an m64nN wgmma is the A fragment of the next k16 step: register 4j + e holds row
// l/4 + 8(e/2), column 8j + 2(l%4) + e%2 (per warp), and A register i of k16 step ks holds row l/4 + 8(i%2),
// columns 16ks + 8(i/2) + 2(l%4) + {0, 1}.  So A register i of step ks is the packed pair acc[8ks + 2i, 8ks + 2i + 1]:
// a[i] = f(acc[8ks + 2i], acc[8ks + 2i + 1], i), where f returns the f16x2 bits of the (transformed) pair.
template <typename F>
__device__ __forceinline__ void afrag_from_acc(const float* acc, int ks, uint32_t (&a)[4], F&& f) {
#pragma unroll
  for (int i = 0; i < 4; ++i) a[i] = f(acc[8 * ks + 2 * i], acc[8 * ks + 2 * i + 1], i);
}

// stmatrix: four 8 x 8 b16 matrices, matrix i from register r[i] of every lane (lane l holds row l/4, columns
// 2(l%4), 2(l%4) + 1: the fragment layout above); lane 8i + k gives the shared address of row k of matrix i
// (16 contiguous bytes).  The .trans form stores each matrix transposed: memory row k receives column k.
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, const uint32_t (&r)[4]) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};\n" ::"r"(addr), "r"(r[0]),
               "r"(r[1]), "r"(r[2]), "r"(r[3])
               : "memory");
}
__device__ __forceinline__ void stmatrix_x4_trans(uint32_t addr, const uint32_t (&r)[4]) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};\n" ::"r"(addr), "r"(r[0]),
               "r"(r[1]), "r"(r[2]), "r"(r[3])
               : "memory");
}

// ------------------------------------------------------------------------------------------
// Row view of an accumulator: the epilogues are written for "one thread owns one tile row".  Thread (warp q of the
// warpgroup, lane l) owns row wg_row128(q, l) of a 128-row tile, or row 16q + l (l < 16) of a 64-row tile.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ int wg_row128(int q, int lane) { return (lane < 16 ? 0 : 48) + 16 * q + lane; }
constexpr int kRowScratchFloats = 32 * 17;        // per warp: 32 rows x 16 columns, padded against bank conflicts

// Columns [c0, c0 + 16) of this thread's row into v (fp32 bits).  c0 must be a compile-time constant after unrolling
// (the accumulator lives in registers).  kHalves = 2 for a 128-row tile, 1 for a 64-row tile.  Whole warp.
template <int kHalves, int R>
__device__ __forceinline__ void wg_row16(const float (&acc)[R], int c0, float* scratch, uint32_t (&v)[16]) {
  const int lane = threadIdx.x & 31;
  const int r = lane >> 2, c = 2 * (lane & 3), j0 = c0 >> 3;
#pragma unroll
  for (int h = 0; h < kHalves; ++h) {
#pragma unroll
    for (int jj = 0; jj < 2; ++jj) {
      const float* a = acc + h * (R / 2) + 4 * (j0 + jj);
      float* s = scratch + (h * 16 + r) * 17 + 8 * jj + c;
      s[0] = a[0];
      s[1] = a[1];
      s[8 * 17] = a[2];
      s[8 * 17 + 1] = a[3];
    }
  }
  __syncwarp();
#pragma unroll
  for (int i = 0; i < 16; ++i) v[i] = __float_as_uint(scratch[lane * 17 + i]);
  __syncwarp();
}

// lane l ends up with the sum over the 32 lanes of v[l % 16]  (v is destroyed)
__device__ __forceinline__ float warp_transpose_reduce16(float (&v)[16], int lane) {
#pragma unroll
  for (int half = 8; half >= 1; half >>= 1) {
    const bool up = (lane & half) != 0;
#pragma unroll
    for (int i = 0; i < half; ++i) {
      const float send = up ? v[i] : v[i + half];
      const float keep = up ? v[i + half] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, half);
    }
  }
  return v[0] + __shfl_xor_sync(0xffffffffu, v[0], 16);
}

// ------------------------------------------------------------------------------------------
// system-scope synchronisation for peer (NVLink) memory
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;\n" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];\n" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];\n" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void fence_acq_rel_sys() {
  asm volatile("fence.acq_rel.sys;\n" ::: "memory");
}

// ------------------------------------------------------------------------------------------
// math
// ------------------------------------------------------------------------------------------
// erf-GELU and its derivative (the reference uses F.gelu's default, exact erf form).
// erf via Abramowitz-Stegun 7.1.26 (|abs err| <= 1.5e-7, i.e. below fp32 round-off of the
// surrounding arithmetic and far below bf16 resolution): one MUFU.RCP, one MUFU.EX2 and a
// degree-5 Horner polynomial.  cdf and pdf share the same exponential exp(-x^2/2), so
// value + derivative cost ~16 instructions instead of two libm calls.
__device__ __forceinline__ float rcp_approx(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float ex2_approx(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
struct GeluParts { float cdf; float pdf; };
__device__ __forceinline__ GeluParts gelu_parts(float x) {
  const float u = fabsf(x) * 0.70710678118654752f;
  const float t = rcp_approx(fmaf(0.3275911f, u, 1.0f));
  const float e = ex2_approx(-1.44269504088896341f * u * u);           // exp(-x^2 / 2)
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float half_tail = 0.5f * p * t * e;                           // 0.5 * erfc(|u|)
  GeluParts r;
  r.cdf = x >= 0.f ? 1.0f - half_tail : half_tail;
  r.pdf = 0.3989422804014327f * e;
  return r;
}
struct GeluVG { float value; float grad; };                 // gelu(x) and d gelu / dx from one evaluation
__device__ __forceinline__ float gelu_erf(float x) { return x * gelu_parts(x).cdf; }
__device__ __forceinline__ float gelu_erf_grad(float x) {
  const GeluParts g = gelu_parts(x);
  return fmaf(x, g.pdf, g.cdf);
}
__device__ __forceinline__ GeluVG gelu_value_grad(float x) {
  const GeluParts g = gelu_parts(x);
  return GeluVG{x * g.cdf, fmaf(x, g.pdf, g.cdf)};
}
// ------------------------------------------------------------------------------------------
// packed fp16 GELU: two values per instruction (HFMA2; the tanh is one tanh.approx.f16x2 per PAIR, which sm_90
// executes as two scalar MUFU.TANH.F16)
// ------------------------------------------------------------------------------------------
// The pointwise epilogues evaluate 10^9..10^10 GELUs per step and were issue bound with the fp32
// erf form (~17 instr + 2 MUFU per value).  This is the tanh form fitted to the *erf* GELU
//     Phi(x) ~ 0.5 (1 + tanh(x (a + b x^2 + c x^4))),  x^2 clamped at 64   (|gelu err| <= 2.6e-5 in exact
// arithmetic) evaluated in fp16x2: 7 instr + 2 MUFU per PAIR for the value, 14 + 2 for value and
// derivative.  fp16 (11-bit significand) keeps the absolute error of gelu / gelu' near 1e-3 * max(1,|x|),
// below the bf16 rounding (2^-9 relative) applied to every stored activation.
// Inputs beyond the fp16 range are handled by the clamp (x^2 = inf -> 64; tanh saturates).
#define DFNO_H2C(v) __float2half2_rn(v)
// saturating: |x| beyond the fp16 range becomes +-65504 instead of inf, so x * cdf(x) stays finite (0 or x)
__device__ __forceinline__ __half2 h2_from_f32(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return *reinterpret_cast<__half2*>(&r);
}
// DFNO_HEAD_PROBE (timing builds only, their outputs are wrong; RESULTS "Projection head on H100"): 1
// replaces the packed GELU by the identity, 2 replaces the tanh by one HFMA2, so a kernel's time splits into the
// MUFU, the rest of the GELU, and everything else.  It applies to every kernel that uses these helpers.
__device__ __forceinline__ __half2 h2_tanh(__half2 x) {
#if DFNO_HEAD_PROBE == 2
  return __hfma2(x, x, x);
#else
  uint32_t r, xi = *reinterpret_cast<uint32_t*>(&x);
  asm("tanh.approx.f16x2 %0, %1;" : "=r"(r) : "r"(xi));
  return *reinterpret_cast<__half2*>(&r);
#endif
}
struct GeluH2 { __half2 value; __half2 grad; };
__device__ __forceinline__ __half2 gelu_h2(__half2 x) {
#if DFNO_HEAD_PROBE == 1
  return x;
#endif
  const __half2 x2 = __hmin2(__hmul2(x, x), DFNO_H2C(64.0f));
  __half2 g = __hfma2(DFNO_H2C(-3.51519787e-4f), x2, DFNO_H2C(3.70056658e-2f));
  g = __hfma2(g, x2, DFNO_H2C(7.97507861e-1f));
  const __half2 t = h2_tanh(__hmul2(x, g));
  return __hmul2(x, __hfma2(DFNO_H2C(0.5f), t, DFNO_H2C(0.5f)));
}
__device__ __forceinline__ GeluH2 gelu_vg_h2(__half2 x) {
#if DFNO_HEAD_PROBE == 1
  return GeluH2{x, DFNO_H2C(1.0f)};
#endif
  const __half2 x2 = __hmin2(__hmul2(x, x), DFNO_H2C(64.0f));
  __half2 g = __hfma2(DFNO_H2C(-3.51519787e-4f), x2, DFNO_H2C(3.70056658e-2f));
  g = __hfma2(g, x2, DFNO_H2C(7.97507861e-1f));
  const __half2 t = h2_tanh(__hmul2(x, g));
  const __half2 cdf = __hfma2(DFNO_H2C(0.5f), t, DFNO_H2C(0.5f));
  __half2 gp = __hfma2(DFNO_H2C(5.0f * -3.51519787e-4f), x2, DFNO_H2C(3.0f * 3.70056658e-2f));
  gp = __hfma2(gp, x2, DFNO_H2C(7.97507861e-1f));                 // d/dx [x g(x^2)]
  const __half2 s = __hfma2(__hneg2(t), t, DFNO_H2C(1.0f));       // sech^2
  const __half2 xs = __hmul2(__hmul2(x, s), DFNO_H2C(0.5f));
  GeluH2 r;
  r.value = __hmul2(x, cdf);
  r.grad = __hfma2(xs, gp, cdf);
  return r;
}
__device__ __forceinline__ uint32_t h2_bits(__half2 v) { return *reinterpret_cast<uint32_t*>(&v); }
__device__ __forceinline__ __half2 h2_of_bits(uint32_t u) { return *reinterpret_cast<__half2*>(&u); }
// fp16x2 <-> bf16x2 (through fp32; values outside the fp16 range saturate to inf and are clamped by the GELU)
__device__ __forceinline__ uint32_t h2_to_bf16x2(__half2 v) {
  const float2 f = __half22float2(v);
  __nv_bfloat162 b = __floats2bfloat162_rn(f.x, f.y);
  return *reinterpret_cast<uint32_t*>(&b);
}
__device__ __forceinline__ __half2 bf16x2_to_h2(uint32_t u) {
  __nv_bfloat162 b = *reinterpret_cast<__nv_bfloat162*>(&u);
  const float2 f = __bfloat1622float2(b);
  return h2_from_f32(f.x, f.y);
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}

}  // namespace dfno
