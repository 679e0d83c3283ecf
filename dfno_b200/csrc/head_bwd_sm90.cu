// head_bwd_sm90.cu -- backward of the projection head  out = W4 . gelu(W3 h + b3) + b4 on the channels-last
// activation (reference dfno.py:348-351; SURVEY.md K17), one wgmma kernel per step, per tile of 128 positions:
//
//   MMA1   pre[pos, j]  = h[pos, :] . W3[j, :]
//   epi A  g[pos, j]    = dout[pos] * W4[j] * gelu'(pre + b3)  -> bf16 tile P;  db3 / dW4 by warp reductions
//   MMA2   dh[pos, i]   = sum_j g[pos, j] * W3[j, i]           -> channels-last global (epi B)
//   MMA3   dW3[j, i]   += sum_pos g[pos, j] * h[pos, i]        (P and the h tile read MN-major; K = positions),
//          kept in registers across the CTA's tiles and flushed once with atomics.
#include "sm90_ptx.cuh"
#include "kernels.h"
#include "tma_host.h"

namespace dfno {
namespace {

constexpr int kStagesH = 3;
constexpr int kThreadsH = 128 + 32;      // one consumer warpgroup (128 x 128 pre-activation in registers), TMA warp

struct HeadBwdParams {
  long long npos;
  int C, CP;
  const float* dout;          // fp32, addressed through the row digits below (public layout)
  int nrl; int R[4]; long long SR[4];
  const float* b3; const float* W4;
  __nv_bfloat16* gcl;         // [npos, CP]
  float* gW3; float* gb3; float* gW4; float* gb4;
};

__global__ void __launch_bounds__(kThreadsH, 1)
head_bwd_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW3,
                const __grid_constant__ CUtensorMap tmW3T, const HeadBwdParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* smem_w3 = smem;                          // [128 hid][64 c]   K-major (K = c)      16 KB
  uint8_t* smem_w3t = smem + 16384;                 // 2 x [32 c][64 hid] K-major (K = hid)    8 KB
  uint8_t* smem_p = smem + 24576;                   // 2 x [128 pos][64 hid]                  32 KB
  uint8_t* smem_a = smem + 57344;                   // stages x [128 pos][64 c]               48 KB
  float* s_scratch = reinterpret_cast<float*>(smem_a + kStagesH * 16384);
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_scratch + 4 * kRowScratchFloats);
  uint64_t* a_full = bars;            // [3]
  uint64_t* a_empty = bars + 3;       // [3]
  uint64_t* w_full = bars + 6;
  float* s_b3 = reinterpret_cast<float*>(bars + 8);    // [128]
  float* s_w4 = s_b3 + 128;                            // [128]
  float* s_gb3 = s_w4 + 128;                           // [128] CTA partial sums
  float* s_gw4 = s_gb3 + 128;                          // [128]
  float* s_gb4 = s_gw4 + 128;                          // [1]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_tiles = static_cast<int>((p.npos + 127) / 128);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA); tma_prefetch_desc(&tmW3); tma_prefetch_desc(&tmW3T);
    for (int s = 0; s < kStagesH; ++s) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], 1); }
    mbar_init(w_full, 1);
    fence_barrier_init();
  }
  for (int i = threadIdx.x; i < 128; i += kThreadsH) {
    s_b3[i] = p.b3[i]; s_w4[i] = p.W4[i]; s_gb3[i] = 0.f; s_gw4[i] = 0.f;
  }
  if (threadIdx.x == 0) s_gb4[0] = 0.f;
  __syncthreads();

  if (warp == 4) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      mbar_arrive_expect_tx(w_full, 16384 + 8192);
      tma_load_2d(smem_w3, &tmW3, w_full, 0, 0);
      tma_load_2d(smem_w3t, &tmW3T, w_full, 0, 0);
      tma_load_2d(smem_w3t + 4096, &tmW3T, w_full, 64, 0);
      uint32_t s = 0, ph = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        mbar_wait(&a_empty[s], ph ^ 1);
        mbar_arrive_expect_tx(&a_full[s], 16384);
        tma_load_2d(smem_a + s * 16384, &tmA, &a_full[s], 0, tile * 128);
        if (++s == kStagesH) { s = 0; ph ^= 1; }
      }
    }
    return;
  }
  // ===================== consumer warpgroup (thread = field position in the row view) ==========
  const int q = warp & 3;
  const int r_in_tile = wg_row128(q, lane);
  float* scratch = s_scratch + warp * kRowScratchFloats;
  const int k1steps = (p.C + 15) / 16;
  const uint32_t wbase = smem_u32(smem_w3), wtbase = smem_u32(smem_w3t), pbase = smem_u32(smem_p);
  float acc_gb4 = 0.f;
  float d3[32];                                 // dW3 [hid rows, c]: 128 x 32 over all tiles of the CTA
  mbar_wait(w_full, 0);
  uint32_t s = 0, ph = 0;
  int n = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++n) {
    const long long row = static_cast<long long>(tile) * 128 + r_in_tile;
    const bool row_ok = row < p.npos;
    float dout = 0.f;
    if (row_ok) {
      long long roff = 0;
      uint32_t r = static_cast<uint32_t>(row);
#pragma unroll
      for (int l = 0; l < 4; ++l) {
        if (l < p.nrl) {
          uint32_t d = r;
          if (l != p.nrl - 1) { const uint32_t qq = r / static_cast<uint32_t>(p.R[l]); d = r - qq * p.R[l]; r = qq; }
          roff += static_cast<long long>(d) * p.SR[l];
        }
      }
      dout = p.dout[roff];
    }
    acc_gb4 += dout;
    mbar_wait(&a_full[s], ph);
    const uint32_t abase = smem_u32(smem_a + s * 16384);
    float acc[128];
    // ---- MMA1: pre = h . W3^T  (128 positions x 128 hidden units)
    wgmma_fence();
    for (int ks = 0; ks < k1steps; ++ks)
      wg_mma128<false, 0, 0>(acc, 128, gdesc_k128(abase + ks * 32), 8192, gdesc_k128(wbase + ks * 32), ks > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(acc);
    // ---- epi A: g = dout * W4 * gelu'(pre + b3) -> bf16 tile P; db3 / dW4 partial sums
    uint8_t* prow = smem_p + r_in_tile * 128;
#pragma unroll
    for (int ch = 0; ch < 8; ++ch) {
      const int jbase = ch * 16;
      uint32_t v[16];
      wg_row16<2>(acc, jbase, scratch, v);
      float gsum[16], wsum[16];
      uint32_t packed[8];
#pragma unroll
      for (int i = 0; i < 16; i += 2) {
        float g2[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int j = jbase + i + e;
          const float pre = __uint_as_float(v[i + e]) + s_b3[j];
          const GeluVG gv = gelu_value_grad(pre);
          const float g = dout * s_w4[j] * gv.grad;
          wsum[i + e] = dout * gv.value;            // -> dW4[j]
          gsum[i + e] = g;                          // -> db3[j]
          g2[e] = g;
        }
        packed[i >> 1] = pack_bf16x2(g2[0], g2[1]);
      }
      // 16 bf16 = two 16-byte chunks of this row in the 64-wide hid block, SWIZZLE_128B
      const int kb = jbase >> 6;
      const int chunk = (jbase & 63) >> 3;
      uint8_t* blk = prow + kb * 16384;
      *reinterpret_cast<uint4*>(blk + (((chunk) ^ (r_in_tile & 7)) << 4)) = make_uint4(packed[0], packed[1], packed[2], packed[3]);
      *reinterpret_cast<uint4*>(blk + (((chunk + 1) ^ (r_in_tile & 7)) << 4)) = make_uint4(packed[4], packed[5], packed[6], packed[7]);
      const float sg = warp_transpose_reduce16(gsum, lane);
      const float sw = warp_transpose_reduce16(wsum, lane);
      if (lane < 16) {
        atomicAdd(&s_gb3[jbase + lane], sg);
        atomicAdd(&s_gw4[jbase + lane], sw);
      }
    }
    // P is complete: publish to the async proxy
    fence_proxy_async_smem();
    asm volatile("bar.sync 1, 128;" ::: "memory");
    // ---- MMA2: dh = P . W3T^T  (K = hid);  MMA3: dW3 += P^T . h  (K = positions, both MN-major)
    float acc2[32];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const int kb = ks >> 2, kk = ks & 3;
      wg_mma128<false, 0, 0>(acc2, 32, gdesc_k128(pbase + kb * 16384 + kk * 32), 8192,
                             gdesc_k128(wtbase + kb * 4096 + kk * 32), ks > 0 ? 1u : 0u);
    }
#pragma unroll
    for (int ks = 0; ks < 8; ++ks)
      wg_mma128<false, 1, 1>(d3, 32, gdesc_mn128(pbase + ks * 2048, 16384, 1024), 16384,
                             gdesc_mn128(abase + ks * 2048, 16384, 1024), (n > 0 || ks > 0) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(acc2);
    acc_fence(d3);
    if (threadIdx.x == 0) mbar_arrive(&a_empty[s]);
    if (++s == kStagesH) { s = 0; ph ^= 1; }
    // ---- epi B: dh tile -> channels-last global
    {
      uint32_t v[16], w[16];
      wg_row16<2>(acc2, 0, scratch, v);
      wg_row16<2>(acc2, 16, scratch, w);
      if (row_ok) {
        __nv_bfloat16* o = p.gcl + row * p.CP;
#pragma unroll
        for (int c = 0; c < 64; c += 8) {
          if (c >= p.CP) break;
          uint32_t u[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int cc = c + 2 * i;
            const float a = cc < 16 ? __uint_as_float(v[cc & 15]) : __uint_as_float(w[cc & 15]);
            const float b = cc + 1 < 16 ? __uint_as_float(v[(cc + 1) & 15]) : __uint_as_float(w[(cc + 1) & 15]);
            u[i] = pack_bf16x2(cc < p.C ? a : 0.f, cc + 1 < p.C ? b : 0.f);
          }
          *reinterpret_cast<uint4*>(o + c) = make_uint4(u[0], u[1], u[2], u[3]);
        }
      }
    }
  }
  // ---- per-CTA flush of the weight gradients
  acc_gb4 += __shfl_xor_sync(0xffffffffu, acc_gb4, 16);
  acc_gb4 += __shfl_xor_sync(0xffffffffu, acc_gb4, 8);
  acc_gb4 += __shfl_xor_sync(0xffffffffu, acc_gb4, 4);
  acc_gb4 += __shfl_xor_sync(0xffffffffu, acc_gb4, 2);
  acc_gb4 += __shfl_xor_sync(0xffffffffu, acc_gb4, 1);
  if (lane == 0) atomicAdd(s_gb4, acc_gb4);
  asm volatile("bar.sync 1, 128;" ::: "memory");
  if (n > 0) {
    // fragment of the 128 x 32 dW3 accumulator: register 16h + 4j + e holds hidden unit 64h + 16q + lane/4 + 8(e/2),
    // channel 8j + 2(lane%4) + e%2
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int hid = 64 * h + 16 * q + (lane >> 2) + 8 * (e >> 1), c = 8 * j + 2 * (lane & 3) + (e & 1);
          if (c < p.C) atomicAdd(p.gW3 + hid * p.C + c, d3[16 * h + 4 * j + e]);
        }
    const int j = threadIdx.x;
    atomicAdd(p.gb3 + j, s_gb3[j]);
    atomicAdd(p.gW4 + j, s_gw4[j]);
    if (j == 0) atomicAdd(p.gb4, s_gb4[0]);
  }
}

}  // namespace

const char* head_bwd(const void* hcl, long long npos, int C, int CP, const void* W3pad, const void* W3Tpad,
                     const float* b3, const float* W4, const float* dout, int nrl, const int* R, const long long* SR,
                     void* gcl, float* gW3, float* gb3, float* gW4, float* gb4, int num_sms, cudaStream_t stream) {
  if (C > 32 || CP % 8 || CP < C || CP > 64) return "head_bwd: need C <= 32 and an 8-aligned channels-last pitch <= 64";
  if (npos > (1ll << 31) - 256) return "head_bwd: too many positions for one launch";
  HeadBwdParams p;
  p.npos = npos; p.C = C; p.CP = CP; p.dout = dout; p.nrl = nrl;
  for (int i = 0; i < 4; ++i) { p.R[i] = i < nrl ? R[i] : 1; p.SR[i] = i < nrl ? SR[i] : 0; }
  p.b3 = b3; p.W4 = W4; p.gcl = static_cast<__nv_bfloat16*>(gcl);
  p.gW3 = gW3; p.gb3 = gb3; p.gW4 = gW4; p.gb4 = gb4;
  CUtensorMap tmA, tmW3, tmW3T;
  if (make_map_2d(&tmA, hcl, static_cast<uint64_t>(C), static_cast<uint64_t>(npos), static_cast<uint64_t>(CP), 64, 128))
    return "cuTensorMapEncodeTiled(h) failed";
  if (make_map_2d(&tmW3, W3pad, 64, 128, 64, 64, 128)) return "cuTensorMapEncodeTiled(W3) failed";
  if (make_map_2d(&tmW3T, W3Tpad, 128, 32, 128, 64, 32)) return "cuTensorMapEncodeTiled(W3T) failed";
  const uint32_t smem_bytes = 57344 + kStagesH * 16384 + 4 * kRowScratchFloats * 4 + 4096;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(head_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess)
      return "cudaFuncSetAttribute failed";
    attr_set = true;
  }
  const int num_tiles = static_cast<int>((npos + 127) / 128);
  const int grid = num_tiles < num_sms ? num_tiles : num_sms;
  head_bwd_kernel<<<grid, kThreadsH, smem_bytes, stream>>>(tmA, tmW3, tmW3T, p);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

}  // namespace dfno
