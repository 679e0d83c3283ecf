// bypass_sm90.cu -- the 1x1 "bypass" convolution of a Fourier layer fused with the GELU
// (forward: SURVEY.md K2 + K14, reference dfno.py:244,291; backward: its adjoint plus the weight
// gradient) on wgmma, TMA in *and* out.
//
//   forward   pre[o, pos] = spec[o, pos] + sum_i W[o, i] h[i, pos];   out = gelu(pre)
//   backward  g[o, pos]   = dout[o, pos] * gelu'(pre[o, pos])          (written over pre)
//             dhb[i, pos] = sum_o W[o, i] g[o, pos]
//             dW[o, i]   += sum_pos g[o, pos] h[i, pos]                (accumulated in registers)
//
// Activations are channel-major ([b*C + c][S positions], positions contiguous).  A tile is
// 128 consecutive positions of all C channels of one batch element: TMA drops it into
// shared memory as two SWIZZLE_128B boxes of [C rows][64 positions].  That single image is
// used three ways without ever being transposed:
//   * as an MN-major A operand (M = positions, K = channels)   -> channel mixing, positions on
//     the accumulator rows, so the epilogue thread of a position owns all its channels;
//   * as a K-major operand (rows = channels, K = positions)     -> the weight gradient, a
//     K-reduction over every position a warpgroup visits, accumulated in its registers;
//   * as the source of a TMA store after the epilogue rewrote it in place.
// Rows C..31 of every box are zeroed once and never touched again (boxes have exactly C rows),
// so the padded K range contributes exact zeros.
#include "sm90_ptx.cuh"
#include "kernels.h"
#include "tma_host.h"

namespace dfno {
namespace {

constexpr int kGroups = 4;                     // consumer warpgroups: tile n belongs to warpgroup n % kGroups
constexpr int kThreadsB = 128 * kGroups + 32;  // + the TMA warp
constexpr int kProducerWarp = 4 * kGroups;
constexpr uint32_t kTile = 8192;               // one tensor tile: 2 boxes x 32 rows x 128 B
constexpr uint32_t kScratchB = 4 * kGroups * kRowScratchFloats * 4;

__device__ __forceinline__ void tma_store_commit_and_wait() {
  tma_store_commit();
  tma_store_wait_read();
}
// byte offset of element (channel c, position t in [0,128)) inside a tile image
__device__ __forceinline__ uint32_t tile_off(int c, int t) {
  const int j = t >> 6, cp = t & 63;
  return j * 4096 + c * 128 + ((((cp >> 3) ^ (c & 7)) << 4) | ((cp & 7) << 1));
}

struct BypassParams {
  int B, C;
  long long S;              // positions per (b, c) slab; multiple of 128
  int save_pre;
  int cl_pitch;
  __nv_bfloat16* out_cl;    // forward: optional channels-last output (instead of the TMA-stored `out`)
  const __nv_bfloat16* dout_cl;   // backward: optional channels-last incoming gradient
  float* dW;                // backward: [C, C] fp32, accumulated with atomics
};

// ================================================================================ forward
constexpr int kStagesF = 8;                    // 16 KB each: h tile + spec tile (a multiple of kGroups: see below)
static_assert(kStagesF % kGroups == 0, "every ring stage must belong to one consumer warpgroup");

__global__ void __launch_bounds__(kThreadsB, 1)
bypass_fwd_tc_kernel(const __grid_constant__ CUtensorMap tmH, const __grid_constant__ CUtensorMap tmS,
                     const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmW,
                     const BypassParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* smem_w = smem;                                   // [32 o][64 i] K-major, 4 KB
  uint8_t* stage0 = smem + 4096;                            // kStagesF x {h tile 8 KB, spec tile 8 KB}
  float* s_scratch = reinterpret_cast<float*>(stage0 + kStagesF * 2 * kTile);
  uint64_t* bars = reinterpret_cast<uint64_t*>(stage0 + kStagesF * 2 * kTile + kScratchB);
  uint64_t* full = bars;                 // [kStagesF]
  uint64_t* empty = bars + kStagesF;     // [kStagesF]   arrived by the epilogue after its TMA stores drained
  uint64_t* wfull = bars + 2 * kStagesF;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long tiles_per_b = p.S / 128;
  const long long num_tiles = tiles_per_b * p.B;

  // zero the padding rows of every tile image once
  for (uint32_t i = threadIdx.x; i < kStagesF * 2 * kTile / 16; i += blockDim.x)
    reinterpret_cast<uint4*>(stage0)[i] = make_uint4(0, 0, 0, 0);
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmH); tma_prefetch_desc(&tmS); tma_prefetch_desc(&tmO); tma_prefetch_desc(&tmW);
    for (int s = 0; s < kStagesF; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 1); }
    mbar_init(wfull, 1);
    fence_barrier_init();
  }
  fence_proxy_async_smem();
  __syncthreads();

  if (warp == kProducerWarp) {
    if (lane == 0) {
      mbar_arrive_expect_tx(wfull, 4096);
      tma_load_2d(smem_w, &tmW, wfull, 0, 0);
      uint32_t s = 0, ph = 0;
      for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int b = static_cast<int>(tile / tiles_per_b);
        const int p0 = static_cast<int>((tile % tiles_per_b) * 128);
        mbar_wait(&empty[s], ph ^ 1);
        mbar_arrive_expect_tx(&full[s], 4u * p.C * 128);
        uint8_t* st = stage0 + s * 2 * kTile;
        tma_load_2d(st, &tmH, &full[s], p0, b * p.C);
        tma_load_2d(st + 4096, &tmH, &full[s], p0 + 64, b * p.C);
        tma_load_2d(st + kTile, &tmS, &full[s], p0, b * p.C);
        tma_load_2d(st + kTile + 4096, &tmS, &full[s], p0 + 64, b * p.C);
        if (++s == kStagesF) { s = 0; ph ^= 1; }
      }
    }
  } else {
    // consumer warpgroup g: channel mixing of its tiles on the tensor core, then the epilogue (thread = position).
    // kStagesF is a multiple of kGroups, so stage s = n % kStagesF is only ever used by warpgroup s % kGroups: every
    // stage has one producer and one consumer, both in order, and a parity wait cannot pass on a stale phase.
    const int q = warp & 3, g = warp >> 2;
    const int t = wg_row128(q, lane);                       // position inside the tile
    float* scratch = s_scratch + warp * kRowScratchFloats;
    mbar_wait(wfull, 0);
    const uint32_t wbase = smem_u32(smem_w);
    long long n = 0;
    for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++n) {
      if (n % kGroups != g) continue;
      const uint32_t s = static_cast<uint32_t>(n % kStagesF);
      const int b = static_cast<int>(tile / tiles_per_b);
      const int p0 = static_cast<int>((tile % tiles_per_b) * 128);
      uint8_t* ht = stage0 + s * 2 * kTile;
      uint8_t* st = ht + kTile;
      mbar_wait(&full[s], (n / kStagesF) & 1);              // TMA data visible to this thread
      float acc[32];
      {
        const uint32_t hbase = smem_u32(ht);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 2; ++ks)            // K = 32 channels, 16 (= two 8-row groups) per MMA; A MN-major
          wg_mma128<false, 1, 0>(acc, 32, gdesc_mn128(hbase + ks * 2048, 4096, 1024), 4096,
                                 gdesc_k128(wbase + ks * 32), ks > 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        acc_fence(acc);
      }
      uint32_t v[32];
      {
        uint32_t v0[16], v1[16];
        wg_row16<2>(acc, 0, scratch, v0);
        wg_row16<2>(acc, 16, scratch, v1);
#pragma unroll
        for (int i = 0; i < 16; ++i) { v[i] = v0[i]; v[16 + i] = v1[i]; }
      }
      __nv_bfloat16* clrow = p.out_cl ? p.out_cl + (static_cast<long long>(b) * p.S + p0 + t) * p.cl_pitch : nullptr;
      uint32_t pk[16];                                      // channels-last row, two channels per word
#pragma unroll
      for (int o = 0; o < 32; ++o) {
        if (o < p.C) {
          const uint32_t off = tile_off(o, t);
          const float pre = __uint_as_float(v[o]) + __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(st + off));
          *reinterpret_cast<__nv_bfloat16*>(st + off) = __float2bfloat16(pre);
          const __nv_bfloat16 y = __float2bfloat16(gelu_erf(pre));
          if (clrow) {
            const uint32_t bits = __bfloat16_as_ushort(y);
            if (o & 1) pk[o >> 1] |= bits << 16; else pk[o >> 1] = bits;
          } else {
            *reinterpret_cast<__nv_bfloat16*>(ht + off) = y;
          }
        } else if ((o & 1) == 0) {
          pk[o >> 1] = 0;
        }
      }
      if (clrow) {                                          // 16-byte vectors; the pitch is a multiple of 8 channels
#pragma unroll
        for (int w = 0; w < 4; ++w)
          if (8 * w < p.cl_pitch)
            reinterpret_cast<uint4*>(clrow)[w] = make_uint4(pk[4 * w], pk[4 * w + 1], pk[4 * w + 2], pk[4 * w + 3]);
      }
      fence_proxy_async_smem();
      asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");
      if (t == 0) {
        if (p.save_pre) {
          tma_store_2d(&tmS, st, p0, b * p.C);
          tma_store_2d(&tmS, st + 4096, p0 + 64, b * p.C);
        }
        if (!p.out_cl) {
          tma_store_2d(&tmO, ht, p0, b * p.C);
          tma_store_2d(&tmO, ht + 4096, p0 + 64, b * p.C);
        }
        tma_store_commit_and_wait();                        // smem may be refilled
        mbar_arrive(&empty[s]);
      }
    }
  }
}

// ================================================================================ backward
constexpr int kStagesBw = 4;                   // 24 KB each: pre tile, dout tile, h tile (a multiple of kGroups)
static_assert(kStagesBw % kGroups == 0, "every ring stage must belong to one consumer warpgroup");

__global__ void __launch_bounds__(kThreadsB, 1)
bypass_bwd_tc_kernel(const __grid_constant__ CUtensorMap tmP, const __grid_constant__ CUtensorMap tmG,
                     const __grid_constant__ CUtensorMap tmH, const __grid_constant__ CUtensorMap tmD,
                     const __grid_constant__ CUtensorMap tmWT, const BypassParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* smem_wt = smem;                                  // [32 i][64 o] K-major, 4 KB
  uint8_t* stage0 = smem + 4096;                            // kStagesBw x {pre, dout, h} tiles
  float* s_scratch = reinterpret_cast<float*>(stage0 + kStagesBw * 3 * kTile + 16384 /*m64 over-read slack*/);
  uint64_t* bars = reinterpret_cast<uint64_t*>(stage0 + kStagesBw * 3 * kTile + 16384 + kScratchB);
  uint64_t* full = bars;                 // [4]
  uint64_t* empty = bars + 4;            // [4]
  uint64_t* wfull = bars + 8;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long tiles_per_b = p.S / 128;
  const long long num_tiles = tiles_per_b * p.B;

  for (uint32_t i = threadIdx.x; i < (kStagesBw * 3 * kTile + 16384) / 16; i += blockDim.x)
    reinterpret_cast<uint4*>(stage0)[i] = make_uint4(0, 0, 0, 0);
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmP); tma_prefetch_desc(&tmG); tma_prefetch_desc(&tmH); tma_prefetch_desc(&tmD);
    tma_prefetch_desc(&tmWT);
    for (int s = 0; s < kStagesBw; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 1); }
    mbar_init(wfull, 1);
    fence_barrier_init();
  }
  fence_proxy_async_smem();
  __syncthreads();
  const bool cl_in = p.dout_cl != nullptr;

  if (warp == kProducerWarp) {
    if (lane == 0) {
      mbar_arrive_expect_tx(wfull, 4096);
      tma_load_2d(smem_wt, &tmWT, wfull, 0, 0);
      uint32_t s = 0, ph = 0;
      for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int b = static_cast<int>(tile / tiles_per_b);
        const int p0 = static_cast<int>((tile % tiles_per_b) * 128);
        mbar_wait(&empty[s], ph ^ 1);
        mbar_arrive_expect_tx(&full[s], (cl_in ? 4u : 6u) * p.C * 128);
        uint8_t* st = stage0 + s * 3 * kTile;
        tma_load_2d(st, &tmP, &full[s], p0, b * p.C);
        tma_load_2d(st + 4096, &tmP, &full[s], p0 + 64, b * p.C);
        if (!cl_in) {
          tma_load_2d(st + kTile, &tmG, &full[s], p0, b * p.C);
          tma_load_2d(st + kTile + 4096, &tmG, &full[s], p0 + 64, b * p.C);
        }
        tma_load_2d(st + 2 * kTile, &tmH, &full[s], p0, b * p.C);
        tma_load_2d(st + 2 * kTile + 4096, &tmH, &full[s], p0 + 64, b * p.C);
        if (++s == kStagesBw) { s = 0; ph ^= 1; }
      }
    }
  } else {
    // consumer warpgroup g: g tile -> (tensor core) dhb tile and its share of dW, kept in registers until the end
    const int q = warp & 3, g = warp >> 2;
    const int t = wg_row128(q, lane);
    float* scratch = s_scratch + warp * kRowScratchFloats;
    float dw[16];                                           // dW rows o (<= 64), columns i (32): m64n32
    long long n = 0, mine = 0;
    mbar_wait(wfull, 0);
    const uint32_t wbase = smem_u32(smem_wt);
    for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++n) {
      if (n % kGroups != g) continue;
      const uint32_t s = static_cast<uint32_t>(n % kStagesBw);
      const int b = static_cast<int>(tile / tiles_per_b);
      const int p0 = static_cast<int>((tile % tiles_per_b) * 128);
      uint8_t* pt = stage0 + s * 3 * kTile;
      uint8_t* gt = pt + kTile;
      mbar_wait(&full[s], (n / kStagesBw) & 1);
      uint32_t pk[16];
      if (cl_in) {                                          // this position's channels-last gradient row
        const uint4* clrow = reinterpret_cast<const uint4*>(p.dout_cl + (static_cast<long long>(b) * p.S + p0 + t) * p.cl_pitch);
#pragma unroll
        for (int w = 0; w < 4; ++w) {
          uint4 u = make_uint4(0, 0, 0, 0);
          if (8 * w < p.cl_pitch) u = clrow[w];
          pk[4 * w] = u.x; pk[4 * w + 1] = u.y; pk[4 * w + 2] = u.z; pk[4 * w + 3] = u.w;
        }
      }
#pragma unroll
      for (int o = 0; o < 32; ++o) {
        if (o < p.C) {
          const uint32_t off = tile_off(o, t);
          const float pre = __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(pt + off));
          const float dy = cl_in ? __uint_as_float((o & 1) ? (pk[o >> 1] & 0xffff0000u) : (pk[o >> 1] << 16))
                                 : __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(gt + off));
          *reinterpret_cast<__nv_bfloat16*>(pt + off) = __float2bfloat16(dy * gelu_erf_grad(pre));
        }
      }
      fence_proxy_async_smem();                             // the g tile is an MMA operand
      asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");
      float acc[32];
      {
        const uint32_t gbase = smem_u32(pt);                // g tile (over the pre tile)
        const uint32_t hbase = gbase + 2 * kTile;
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 2; ++ks)            // dhb = g^T-view . WT: K = 32 output channels o, A MN-major
          wg_mma128<false, 1, 0>(acc, 32, gdesc_mn128(gbase + ks * 2048, 4096, 1024), 4096,
                                 gdesc_k128(wbase + ks * 32), ks > 0 ? 1u : 0u);
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) {          // dW += g . h^T: K = 128 positions, 2 boxes x 4 steps of 16
          const int j = ks >> 2, kk = ks & 3;
          wg_mma64<false, 0, 0, 0>(dw, 32, gdesc_k128(gbase + j * 4096 + kk * 32), gdesc_k128(hbase + j * 4096 + kk * 32),
                                   (mine > 0 || ks > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        acc_fence(acc);
        acc_fence(dw);
        ++mine;
      }
      {
        uint32_t v0[16], v1[16];
        wg_row16<2>(acc, 0, scratch, v0);
        wg_row16<2>(acc, 16, scratch, v1);
#pragma unroll
        for (int i = 0; i < 32; ++i)
          if (i < p.C)
            *reinterpret_cast<__nv_bfloat16*>(gt + tile_off(i, t)) =
                __float2bfloat16(__uint_as_float(i < 16 ? v0[i & 15] : v1[i & 15]));
      }
      fence_proxy_async_smem();
      asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");
      if (t == 0) {
        tma_store_2d(&tmP, pt, p0, b * p.C);                // dpre over pre
        tma_store_2d(&tmP, pt + 4096, p0 + 64, b * p.C);
        tma_store_2d(&tmD, gt, p0, b * p.C);                // dhb
        tma_store_2d(&tmD, gt + 4096, p0 + 64, b * p.C);
        tma_store_commit_and_wait();
        mbar_arrive(&empty[s]);
      }
    }
    if (mine > 0) {
      // fragment of the m64n32 accumulator: row o = 16q + lane/4 (+8), column i = 8j + 2(lane%4) (+1)
      const int o0 = 16 * q + (lane >> 2), i0 = 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int o = o0 + 8 * (e >> 1), i = 8 * j + i0 + (e & 1);
          if (o < p.C && i < p.C) atomicAdd(p.dW + o * p.C + i, dw[4 * j + e]);
        }
    }
  }
}

const char* set_attr_once(const void* fn, bool* flag) {
  if (!*flag) {
    if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess)
      return "cudaFuncSetAttribute failed";
    *flag = true;
  }
  return nullptr;
}

}  // namespace

const char* bypass_fwd_tc(const void* h, void* spec_pre, const void* Wpad, void* out, void* out_cl, int cl_pitch,
                          int B, int C, long long S, int save_pre, int num_sms, cudaStream_t stream) {
  if (C > 32 || S % 128) return "bypass_fwd_tc: need C <= 32 and S % 128 == 0";
  if (S > (1ll << 31) - 256) return "bypass_fwd_tc: slab too large";
  if (!out && !out_cl) return "bypass_fwd_tc: no output";
  BypassParams p{};
  p.B = B; p.C = C; p.S = S; p.save_pre = save_pre; p.cl_pitch = cl_pitch;
  p.out_cl = static_cast<__nv_bfloat16*>(out_cl);
  CUtensorMap tmH, tmS, tmO, tmW;
  const uint64_t rows = static_cast<uint64_t>(B) * C;
  if (make_map_2d(&tmH, h, S, rows, S, 64, C)) return "tensor map (h) failed";
  if (make_map_2d(&tmS, spec_pre, S, rows, S, 64, C)) return "tensor map (spec) failed";
  if (make_map_2d(&tmO, out ? out : spec_pre, S, rows, S, 64, C)) return "tensor map (out) failed";
  if (make_map_2d(&tmW, Wpad, 64, 32, 64, 64, 32)) return "tensor map (W) failed";
  static bool attr = false;
  if (const char* e = set_attr_once(reinterpret_cast<const void*>(bypass_fwd_tc_kernel), &attr)) return e;
  const long long tiles = S / 128 * B;
  const int grid = static_cast<int>(tiles < num_sms ? tiles : num_sms);
  const uint32_t smem_bytes = 4096 + kStagesF * 2 * kTile + kScratchB + 1024;
  bypass_fwd_tc_kernel<<<grid, kThreadsB, smem_bytes, stream>>>(tmH, tmS, tmO, tmW, p);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

const char* bypass_bwd_tc(const void* dout, const void* dout_cl, int cl_pitch, void* pre_dpre, const void* h,
                          const void* WTpad, void* dhb, float* dW, int B, int C, long long S, int num_sms,
                          cudaStream_t stream) {
  if (C > 32 || S % 128) return "bypass_bwd_tc: need C <= 32 and S % 128 == 0";
  if (S > (1ll << 31) - 256) return "bypass_bwd_tc: slab too large";
  BypassParams p{};
  p.B = B; p.C = C; p.S = S; p.cl_pitch = cl_pitch;
  p.dout_cl = static_cast<const __nv_bfloat16*>(dout_cl);
  p.dW = dW;
  CUtensorMap tmP, tmG, tmH, tmD, tmWT;
  const uint64_t rows = static_cast<uint64_t>(B) * C;
  if (make_map_2d(&tmP, pre_dpre, S, rows, S, 64, C)) return "tensor map (pre) failed";
  if (make_map_2d(&tmG, dout ? dout : pre_dpre, S, rows, S, 64, C)) return "tensor map (dout) failed";
  if (make_map_2d(&tmH, h, S, rows, S, 64, C)) return "tensor map (h) failed";
  if (make_map_2d(&tmD, dhb, S, rows, S, 64, C)) return "tensor map (dhb) failed";
  if (make_map_2d(&tmWT, WTpad, 64, 32, 64, 64, 32)) return "tensor map (WT) failed";
  static bool attr = false;
  if (const char* e = set_attr_once(reinterpret_cast<const void*>(bypass_bwd_tc_kernel), &attr)) return e;
  const long long tiles = S / 128 * B;
  const int grid = static_cast<int>(tiles < num_sms ? tiles : num_sms);
  const uint32_t smem_bytes = 4096 + kStagesBw * 3 * kTile + 16384 + kScratchB + 1024;
  bypass_bwd_tc_kernel<<<grid, kThreadsB, smem_bytes, stream>>>(tmP, tmG, tmH, tmD, tmWT, p);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

}  // namespace dfno
