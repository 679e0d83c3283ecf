// kreduce_gemm_sm90.cu -- long-K reduction GEMM on wgmma:  D[i, j] += sum_k A[i, k] * B[j, k]
//
// A: [Ma <= 128, K], B: [Nb <= 256, K], both bf16 with the *reduced* index contiguous, K in
// the millions (all field positions).  Used for the weight gradients of the 1x1 convolutions
// (dW[o, i] = sum_pos dpre[o, pos] * h[i, pos], the SumReduce side of BroadcastedLinear,
// SURVEY.md K18): the activations are already stored channel-major with positions
// contiguous, so both operands are K-major as they are -- no transpose, no im2col.
//
// Split-K over persistent CTAs: each CTA streams a contiguous range of 64-wide K blocks
// through a TMA/mbarrier ring (rows beyond Ma/Nb are zero-filled by TMA and cost no HBM
// traffic).  Two consumer warpgroups own rows 0..63 and 64..127 of the result and keep their
// 64 x Nb_pad partial sums in registers (m64nNk16, N up to 256) over the CTA's whole K range,
// then add them to the fp32 result with atomics.  Memory bound: ~ (Ma + Nb) * 128 B per 64 K-steps.
#include "sm90_ptx.cuh"
#include "kernels.h"
#include "tma_host.h"

namespace dfno {

namespace {
constexpr int kMaxStages = 8;
constexpr int kThreads = 256 + 32;       // two consumer warpgroups, one TMA warp

struct KrParams {
  int Ma, Nb, nb_pad;
  int a_rows;              // rows of the A box (32 / 64 when Ma is small: the m64 instruction still reads 64
                           // rows, the extra ones hold don't-care values that are never stored)
  int nwg;                 // consumer warpgroups with rows to compute (1 when Ma <= 64)
  int stages;
  long long kblocks;       // total 64-wide K blocks
  float* D;
  long long ldd;
};

__global__ void __launch_bounds__(kThreads, 1)
kreduce_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const KrParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t a_bytes = p.a_rows * 128, b_bytes = p.nb_pad * 128;
  const uint32_t stage_bytes = a_bytes + b_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + p.stages * stage_bytes + 16384);
  uint64_t* full = bars;
  uint64_t* empty = bars + kMaxStages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // contiguous K range of this CTA
  const long long per = (p.kblocks + gridDim.x - 1) / gridDim.x;
  const long long kb0 = per * blockIdx.x;
  const long long kb1 = kb0 + per < p.kblocks ? kb0 + per : p.kblocks;
  const bool has_work = kb0 < kb1;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < p.stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], p.nwg); }
    fence_barrier_init();
  }
  __syncthreads();
  if (!has_work) return;

  if (warp == 8) {
    if (lane == 0) {
      uint32_t s = 0, ph = 0;
      for (long long kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&empty[s], ph ^ 1);
        mbar_arrive_expect_tx(&full[s], stage_bytes);
        uint8_t* dst = smem + s * stage_bytes;
        tma_load_2d(dst, &tmA, &full[s], static_cast<int32_t>(kb * 64), 0);
        tma_load_2d(dst + a_bytes, &tmB, &full[s], static_cast<int32_t>(kb * 64), 0);
        if (++s == static_cast<uint32_t>(p.stages)) { s = 0; ph ^= 1; }
      }
    }
    return;
  }
  const int wg = warp >> 2;
  if (wg >= p.nwg) return;
  float acc[kAccRegs];
  uint32_t s = 0, ph = 0;
  for (long long kb = kb0; kb < kb1; ++kb) {
    mbar_wait(&full[s], ph);
    const uint32_t a_base = smem_u32(smem + s * stage_bytes) + wg * 8192;
    const uint32_t b_base = smem_u32(smem + s * stage_bytes) + a_bytes;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
      wg_mma64<false, 0, 0, 0>(acc, p.nb_pad, gdesc_k128(a_base + kk * 32), gdesc_k128(b_base + kk * 32),
                               (kb > kb0 || kk > 0) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(acc);
    if ((threadIdx.x & 127) == 0) mbar_arrive(&empty[s]);
    if (++s == static_cast<uint32_t>(p.stages)) { s = 0; ph ^= 1; }
  }
  const int r0 = wg * 64 + 16 * (warp & 3) + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < kAccRegs / 4; ++j) {
    if (8 * j < p.nb_pad) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int row = r0 + 8 * (e >> 1), col = 8 * j + c + (e & 1);
        if (row < p.Ma && col < p.Nb) atomicAdd(p.D + row * p.ldd + col, acc[4 * j + e]);
      }
    }
  }
}
}  // namespace

const char* kreduce_gemm(const void* A, long long lda, int Ma, const void* Bm, long long ldb, int Nb, long long K,
                         float* D, long long ldd, int num_sms, cudaStream_t stream) {
  if (Ma < 1 || Ma > 128 || Nb < 1 || Nb > 256) return "kreduce: Ma<=128, Nb<=256";
  if ((lda * 2) % 16 || (ldb * 2) % 16) return "kreduce: row pitches must be multiples of 16 bytes";
  if (K > (1ll << 31) - 64) return "kreduce: K too large for one launch";
  KrParams p;
  p.Ma = Ma; p.Nb = Nb; p.nb_pad = (Nb + 15) / 16 * 16;
  p.a_rows = Ma <= 32 ? 32 : (Ma <= 64 ? 64 : 128);
  p.nwg = Ma <= 64 ? 1 : 2;
  p.kblocks = (K + 63) / 64;
  p.D = D; p.ldd = ldd;
  // + 16 KB slack: the m64 descriptor of the last stage reads past a 32-row box
  const uint32_t stage_bytes = p.a_rows * 128 + p.nb_pad * 128;
  p.stages = (227 * 1024 - 16384 - 1024) / stage_bytes;
  if (p.stages > kMaxStages) p.stages = kMaxStages;
  if (p.stages < 2) return "kreduce: tiles do not fit shared memory";
  CUtensorMap tmA, tmB;
  if (make_map_2d(&tmA, A, static_cast<uint64_t>(K), static_cast<uint64_t>(Ma), static_cast<uint64_t>(lda), 64,
                  static_cast<uint32_t>(p.a_rows)))
    return "cuTensorMapEncodeTiled(A) failed";
  if (make_map_2d(&tmB, Bm, static_cast<uint64_t>(K), static_cast<uint64_t>(Nb), static_cast<uint64_t>(ldb), 64,
                  static_cast<uint32_t>(p.nb_pad)))
    return "cuTensorMapEncodeTiled(B) failed";
  const uint32_t smem_bytes = p.stages * stage_bytes + 16384 + 256;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(kreduce_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess)
      return "cudaFuncSetAttribute failed";
    attr_set = true;
  }
  // at least ~64 K-blocks per CTA so the per-CTA atomics stay negligible
  long long ctas = (p.kblocks + 63) / 64;
  if (ctas > num_sms) ctas = num_sms;
  if (ctas < 1) ctas = 1;
  kreduce_kernel<<<static_cast<int>(ctas), kThreads, smem_bytes, stream>>>(tmA, tmB, p);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

}  // namespace dfno
