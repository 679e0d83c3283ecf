// head_multi_sm90.cu -- projection head with O = 1..4 output channels,  out[o] = W4[o] . gelu(W3 h + b3) + b4[o]
// (SURVEY.md K17 with linear4 widened to O outputs), forward and backward.  Tiling, operands and pipeline are those of
// head_sm90.cu: 128-position tiles of all C channels of the channel-major activation h[b*C + c][S], dropped by TMA
// into SWIZZLE_128B boxes and used as an MN-major A operand, a row of ones that carries b3 through the MMA, TMA rings
// whose depth is a multiple of the consumer warpgroups, and a setmaxnreg producer warpgroup in the backward.
//
//   forward   MMA   pre[pos, j] = sum_c h[c, pos] W3[j, c] + b3[j]
//             epi   out[pos, o] = b4[o] + sum_j W4[o, j] gelu(pre[pos, j])   (packed fp16 GELU once per fragment,
//                                 then one HFMA2 dot per output finished across the 4 lanes of a quad)
//
//   backward  the per-position dout can no longer be factored out of P (head_sm90.cu), so it moves into it:
//             MMA1  pre (as above), in two 64-unit hidden halves
//             epi A P'[pos, j]  = gelu'(pre) sum_o ds[pos, o] W4[o, j]   (ds = s dout, s = 2^k from one |dout| max
//                                 over all O planes keeps it inside the fp16 range; undone when the sums are flushed)
//                   G[pos, j]   = gelu(pre)  (fp16, this half only)
//             MMA4  D4[j, o]   += sum_pos G[pos, j] ds[pos, o]            -> dW4: O column sums per hidden unit do
//                                 not fit in registers next to D3, so they are reduced on the tensor core (N = 8)
//             MMA2  dh0[pos, i] = sum_j P'[pos, j] W3[j, i]               epi B: g[i, pos] = dh0[pos, i] / s
//             MMA3  D3[j, i]   += sum_pos P'[pos, j] hs[i, pos]           -> dW3 (i < C), db3 (i = C)
//             with hs the fp16 copy of the h tile and its row of ones; db4[o] = sum_pos dout[pos, o].
#include "head_common.cuh"
#include "kernels.h"
#include "tma_host.h"

namespace dfno {
namespace {

constexpr int kMaxOut = 4;

// ================================================================================ forward
constexpr int kStagesMF = 6;
constexpr int kGroupsMF = 2;                    // consumer warpgroups (kStagesMF a multiple of it: see bypass_sm90.cu)
static_assert(kStagesMF % kGroupsMF == 0, "every ring stage must belong to one consumer warpgroup");
constexpr int kThreadsMF = 128 * kGroupsMF + 32;

struct HeadMultiFwdParams {
  int B, C;
  long long S, tiles_per_b;
  long long plane;            // element stride between output channels of the public layout
  const float* w4b4;          // [O x 128 weights, O biases]
  float* out;
  RowMap map;
};

// KR: channels + the ones row, padded to 16 (the K of the MMA); O: output channels.  kPad: as head_fwd_kernel.
template <int KR, int O, bool kPad>
__device__ __forceinline__ void head_fwd_multi_body(const CUtensorMap& tmH, const CUtensorMap& tmW3,
                                                    const HeadMultiFwdParams p, const PadRowMap pm) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* s_w3 = smem;                                    // [128 hid][64] K-major, column C = b3
  uint8_t* s_a = smem + 16384;                             // stages x 2 halves x [KR rows][64 pos]
  constexpr uint32_t half_bytes = KR * 128;
  constexpr uint32_t stage_bytes = 2 * half_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_a + kStagesMF * stage_bytes);
  uint64_t* full = bars;              // [6]
  uint64_t* empty = bars + 6;         // [6]
  uint64_t* wfull = bars + 12;
  // [O][4 lanes of a quad][16] fp16x2 pairs of W4: entry j of lane group cq = hidden units 8j + 2cq + {0, 1}
  uint32_t* s_w4 = reinterpret_cast<uint32_t*>(bars + 14);
  float* s_b4 = reinterpret_cast<float*>(s_w4 + 64 * O);

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const long long num_tiles = p.tiles_per_b * p.B;

  for (uint32_t i = threadIdx.x; i < kStagesMF * stage_bytes / 16; i += blockDim.x)
    reinterpret_cast<uint4*>(s_a)[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < kStagesMF * 2 * 16; i += blockDim.x) {      // the ones row (row C) of every half
    const uint32_t hb = i >> 4, ch = i & 15;
    reinterpret_cast<uint2*>(s_a + hb * half_bytes + p.C * 128)[ch] = make_uint2(0x3F803F80u, 0x3F803F80u);
  }
  for (int i = threadIdx.x; i < 64 * O; i += blockDim.x) {
    const int o = i >> 6, cq = (i >> 4) & 3, j = i & 15;
    const float* w = p.w4b4 + o * kHidH + 8 * j + 2 * cq;
    s_w4[i] = h2_bits(h2_from_f32(w[0], w[1]));
  }
  if (threadIdx.x < O) s_b4[threadIdx.x] = p.w4b4[O * kHidH + threadIdx.x];
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmH); tma_prefetch_desc(&tmW3);
    for (int s = 0; s < kStagesMF; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 1); }
    mbar_init(wfull, 1);
    fence_barrier_init();
  }
  fence_proxy_async_smem();
  __syncthreads();

  if (warp == 4 * kGroupsMF) {
    if (lane == 0) {
      mbar_arrive_expect_tx(wfull, 16384);
      tma_load_2d(s_w3, &tmW3, wfull, 0, 0);
      uint32_t s = 0, ph = 0;
      for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int b = static_cast<int>(tile / p.tiles_per_b);
        const int p0 = static_cast<int>((tile % p.tiles_per_b) * 128);
        mbar_wait(&empty[s], ph ^ 1);
        mbar_arrive_expect_tx(&full[s], 2u * p.C * 128);
        uint8_t* st = s_a + s * stage_bytes;
        tma_load_2d(st, &tmH, &full[s], p0, b * p.C);
        tma_load_2d(st + half_bytes, &tmH, &full[s], p0 + 64, b * p.C);
        if (++s == kStagesMF) { s = 0; ph ^= 1; }
      }
    }
    return;
  }
  const int q = warp & 3, g = warp >> 2, cq = lane & 3;
  const int my_row = frag_row(q, lane, cq);          // the row this lane stores (each lane of a quad stores one)
  const uint32_t w_addr = smem_u32(s_w3);
  const uint4* w4q = reinterpret_cast<const uint4*>(s_w4) + 4 * cq;   // + 16 per output channel
  mbar_wait(wfull, 0);
  float acc[128];
  long long n = 0;
  for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++n) {
    if (n % kGroupsMF != g) continue;
    const uint32_t s = static_cast<uint32_t>(n % kStagesMF);
    const int b = static_cast<int>(tile / p.tiles_per_b);
    const long long pos = (tile % p.tiles_per_b) * 128 + my_row;
    mbar_wait(&full[s], (n / kStagesMF) & 1);
    const uint32_t abase = smem_u32(s_a + s * stage_bytes);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < KR / 16; ++ks)
      wg_mma128<false, 1, 0>(acc, kHidH, gdesc_mn128(abase + ks * 2048, half_bytes, 1024), half_bytes,
                             gdesc_k128(w_addr + ks * 32), ks > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(acc);
    if (q == 0 && lane == 0) mbar_arrive(&empty[s]);
    // gelu of row k of the thread (registers 64(k/2) + 4j + 2(k%2) + {0, 1}) as 16 fp16 pairs, once for all outputs
    uint32_t gh[4][16];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float* a = acc + 64 * (k >> 1) + 2 * (k & 1);
#pragma unroll
      for (int j = 0; j < 16; ++j) gh[k][j] = h2_bits(gelu_h2(h2_from_f32(a[4 * j], a[4 * j + 1])));
    }
    long long base;
    if constexpr (kPad) base = pos < p.S ? pad_row_to_offset(pm, static_cast<uint32_t>(b * p.S + pos)) : -1;
    else base = pos < p.S ? row_to_offset(p.map, static_cast<uint32_t>(b * p.S + pos)) : 0;
#pragma unroll
    for (int o = 0; o < O; ++o) {
      uint32_t w4[16];
#pragma unroll
      for (int v = 0; v < 4; ++v) {
        const uint4 u = w4q[16 * o + v];
        w4[4 * v] = u.x; w4[4 * v + 1] = u.y; w4[4 * v + 2] = u.z; w4[4 * v + 3] = u.w;
      }
      float out[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {                  // two fp16 dot chains of 8 pairs each, as in head_sm90.cu
        float sum = 0.f;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          __half2 part = __float2half2_rn(0.f);
#pragma unroll
          for (int j = 8 * half; j < 8 * half + 8; ++j) part = __hfma2(h2_of_bits(gh[k][j]), h2_of_bits(w4[j]), part);
          const float2 f = __half22float2(part);
          sum += f.x + f.y;
        }
        sum += __shfl_xor_sync(0xffffffffu, sum, 1);
        sum += __shfl_xor_sync(0xffffffffu, sum, 2);
        out[k] = sum;
      }
      if (kPad ? base >= 0 : pos < p.S) p.out[base + o * p.plane] = s_b4[o] + pick4(out, cq);
    }
  }
}

template <int KR, int O>
__global__ void __launch_bounds__(kThreadsMF, 1)
head_fwd_multi_kernel(const __grid_constant__ CUtensorMap tmH, const __grid_constant__ CUtensorMap tmW3,
                      const HeadMultiFwdParams p) {
  head_fwd_multi_body<KR, O, false>(tmH, tmW3, p, PadRowMap{});
}

template <int KR, int O>
__global__ void __launch_bounds__(kThreadsMF, 1)
head_fwd_multi_pad_kernel(const __grid_constant__ CUtensorMap tmH, const __grid_constant__ CUtensorMap tmW3,
                          const HeadMultiFwdParams p, const __grid_constant__ PadRowMap pm) {
  head_fwd_multi_body<KR, O, true>(tmH, tmW3, p, pm);
}

// ================================================================================ backward
constexpr int kMaxStagesMB = 6;
constexpr int kGroupsMB = 2;                    // consumer warpgroups (stages a multiple of it: see bypass_sm90.cu)
constexpr int kThreadsMB = 128 * kGroupsMB + 128;
constexpr int kProducerRegsMB = 24, kConsumerRegsMB = 240;
static_assert(128 * kProducerRegsMB + 128 * kGroupsMB * kConsumerRegsMB <= 65536, "register file");
// per consumer warpgroup besides the h-sized buffers: P' (2 x 16 KB), the G half (16 KB), the ds operand (2 KB)
constexpr uint32_t kWgBytesMB = 32768 + 16384 + 2048;

struct HeadMultiBwdParams {
  int B, C, stages;
  long long S, tiles_per_b, plane;
  const float* dout;          // fp32, public layout (plane stride between output channels)
  const float* amax;          // max |dout| over all planes (device scalar)
  const float* W4;            // [O, 128]
  float* gW3; float* gb3; float* gW4; float* gb4;
  RowMap map;
};

// One consumer warpgroup per tile of 128 positions, as head_bwd2_kernel.  Per 64-unit hidden half, epilogue A turns
// the MMA1 accumulator into P' (register A operand of MMA2, stored with stmatrix for MMA3) and G (stored with stmatrix
// for MMA4); epilogue B stages g as bf16 [C][128 positions] with stmatrix.trans for two TMA stores.
// KR: channels + the ones row, padded to 16 (the N of MMA2 / MMA3 and the accumulator width); O: output channels.
// kPad: as head_bwd2_kernel (pad rows read dout as 0).
template <int KR, int O, bool kPad>
__device__ __forceinline__ void head_bwd_multi_body(const CUtensorMap& tmH, const CUtensorMap& tmW3,
                                                    const CUtensorMap& tmW3T, const CUtensorMap& tmG,
                                                    const HeadMultiBwdParams p, const PadRowMap pm) {
  extern __shared__ __align__(1024) uint8_t smem[];
  constexpr uint32_t half_bytes = KR * 128;
  constexpr uint32_t tile_bytes = 2 * half_bytes;
  uint8_t* s_w3 = smem;                                   // 16 KB
  uint8_t* s_w3t = s_w3 + 16384;                          // 2 k-blocks x [KR c rows][64 hid] fp16
  uint8_t* s_wg = s_w3t + tile_bytes;                     // per warpgroup: P' [2][128 pos][64 hid], G [128][64],
                                                          //   ds [2 pos blocks][8 outputs][64 pos] (fp16)
  uint8_t* s_a = s_wg + kGroupsMB * kWgBytesMB;           // stages x h tile
  uint8_t* s_hs = s_a + p.stages * tile_bytes;            // per warpgroup: fp16 copy of the h tile + ones row
  uint8_t* s_g = s_hs + kGroupsMB * tile_bytes;           // per warpgroup: bf16 g staging, 2 x [KR c rows][64 pos]
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_g + kGroupsMB * tile_bytes);
  uint64_t* a_full = bars;            // [8]
  uint64_t* a_empty = bars + 8;       // [8]
  uint64_t* w_full = bars + 16;
  float* s_gb4 = reinterpret_cast<float*>(bars + 18);          // [4] CTA partial sums of db4
  uint32_t* s_w4h = reinterpret_cast<uint32_t*>(bars + 20);    // [O][64] fp16x2 pairs of W4
  float* s_gw4 = reinterpret_cast<float*>(s_w4h + 64 * kMaxOut);   // [O][128] CTA partial sums of s dW4

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const long long num_tiles = p.tiles_per_b * p.B;

  for (uint32_t i = threadIdx.x; i < p.stages * tile_bytes / 16; i += blockDim.x)
    reinterpret_cast<uint4*>(s_a)[i] = make_uint4(0, 0, 0, 0);
  for (uint32_t i = threadIdx.x; i < kGroupsMB * tile_bytes / 16; i += blockDim.x)
    reinterpret_cast<uint4*>(s_hs)[i] = make_uint4(0, 0, 0, 0);
  for (uint32_t i = threadIdx.x; i < kGroupsMB * kWgBytesMB / 16; i += blockDim.x)
    reinterpret_cast<uint4*>(s_wg)[i] = make_uint4(0, 0, 0, 0);              // ds rows O..7 stay zero
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < static_cast<uint32_t>(p.stages) * 2 * 16; i += blockDim.x) {
    const uint32_t hb = i >> 4, ch = i & 15;
    reinterpret_cast<uint2*>(s_a + hb * half_bytes + p.C * 128)[ch] = make_uint2(0x3F803F80u, 0x3F803F80u);
  }
  // the ones row of hs (row C, fp16 1.0 at every position; the swizzle only permutes 16-byte chunks of a row)
  for (uint32_t i = threadIdx.x; i < kGroupsMB * 2 * 16; i += blockDim.x) {
    const uint32_t hb = i >> 4, ch = i & 15;
    reinterpret_cast<uint2*>(s_hs + hb * half_bytes + p.C * 128)[ch] = make_uint2(0x3C003C00u, 0x3C003C00u);
  }
  if (threadIdx.x < kMaxOut) s_gb4[threadIdx.x] = 0.f;
  for (int i = threadIdx.x; i < O * kHidH; i += blockDim.x) s_gw4[i] = 0.f;
  for (int i = threadIdx.x; i < 64 * O; i += blockDim.x)
    s_w4h[i] = h2_bits(h2_from_f32(p.W4[2 * i], p.W4[2 * i + 1]));
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmH); tma_prefetch_desc(&tmW3); tma_prefetch_desc(&tmW3T); tma_prefetch_desc(&tmG);
    for (int s = 0; s < p.stages; ++s) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], 1); }
    mbar_init(w_full, 1);
    fence_barrier_init();
  }
  fence_proxy_async_smem();
  __syncthreads();
  const float amax = *p.amax;
  const float scale = amax > 0.f ? exp2f(-ceilf(log2f(amax))) : 1.0f;      // |scale * dout| <= 1

  if (warp >= 4 * kGroupsMB) {
    setmaxnreg_dec<kProducerRegsMB>();
    if (warp == 4 * kGroupsMB && lane == 0) {
      mbar_arrive_expect_tx(w_full, 16384 + tile_bytes);
      tma_load_2d(s_w3, &tmW3, w_full, 0, 0);
      tma_load_2d(s_w3t, &tmW3T, w_full, 0, 0);
      tma_load_2d(s_w3t + half_bytes, &tmW3T, w_full, 64, 0);
      uint32_t s = 0, ph = 0;
      for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int b = static_cast<int>(tile / p.tiles_per_b);
        const int p0 = static_cast<int>((tile % p.tiles_per_b) * 128);
        mbar_wait(&a_empty[s], ph ^ 1);
        mbar_arrive_expect_tx(&a_full[s], 2u * p.C * 128);
        uint8_t* st = s_a + s * tile_bytes;
        tma_load_2d(st, &tmH, &a_full[s], p0, b * p.C);
        tma_load_2d(st + half_bytes, &tmH, &a_full[s], p0 + 64, b * p.C);
        if (++s == static_cast<uint32_t>(p.stages)) { s = 0; ph ^= 1; }
      }
    }
    return;
  }

  setmaxnreg_inc<kConsumerRegsMB>();
  const int q = warp & 3, g = warp >> 2, cq = lane & 3;
  const int my_row = frag_row(q, lane, cq);          // the row whose dout this lane loads
  const uint32_t barid = 1 + g;
  const bool leader = q == 0 && lane == 0;           // releases ring stages and issues this warpgroup's g stores
  uint8_t* pbuf = s_wg + g * kWgBytesMB;
  uint8_t* gtbuf = pbuf + 32768;
  uint8_t* dsbuf = gtbuf + 16384;
  uint8_t* hsbuf = s_hs + g * tile_bytes;
  uint8_t* gbuf = s_g + g * tile_bytes;
  const uint32_t w3_addr = smem_u32(s_w3), w3t_addr = smem_u32(s_w3t);
  const uint32_t p_addr = smem_u32(pbuf), gt_addr = smem_u32(gtbuf), ds_addr = smem_u32(dsbuf);
  const uint32_t hs_addr = smem_u32(hsbuf), g_addr = smem_u32(gbuf);
  // stmatrix addressing as in head_bwd2_kernel: P' / G matrix i = positions 16q + 8(i%2) + k of an m64 half, hidden
  // units 8(i/2).. of a k16 step; g (transposed) memory row k of matrix i = channel 8(i/2) + k of a 16-channel group
  const int mi = lane >> 3, mk = lane & 7;
  const uint32_t p_row = 16 * q + 8 * (mi & 1) + mk;
  const uint32_t g_chunk = 2 * q + (mi & 1);
  // this lane's slot of the ds operand (K-major, 128-byte swizzle): row o, position my_row, in 16-byte chunk
  // ds_chunk ^ o of the row
  const uint32_t ds_off = (my_row >> 6) * 1024 + ((my_row & 7) << 1);
  const uint32_t ds_chunk = (my_row & 63) >> 3;
  constexpr int NG = KR;                             // dh0 columns (C <= 31 here, so KR = ceil16(C + 1) >= C)
  float d3[KR];                                      // [hid, c] over this warpgroup's tiles: 128 x KR
  uint32_t pa[2][4][4];                              // P' of one 64-unit hidden half: [m64 half][k16 step][A register]
  auto mma2 = [&](float (&acc2)[NG], int kb) {       // dh0 (+)= P' . W3 over hidden units [64 kb, 64 kb + 64)
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const uint64_t db = gdesc_k128(w3t_addr + kb * half_bytes + ks * 32);
      const uint32_t sc = (kb > 0 || ks > 0) ? 1u : 0u;
      wg_mma64_rs<NG, 0, 0>(acc2, pa[0][ks], db, sc);
      wg_mma64_rs<NG, 0, NG / 2>(acc2, pa[1][ks], db, sc);
    }
  };
  auto mma4 = [&](float (&d)[4]) {                   // D4 = G^T . ds over the tile's 128 positions
#pragma unroll
    for (int ks = 0; ks < 8; ++ks)
      wgmma_m64n8k16_f16<1, 0>(d, gdesc_mn128(gt_addr + ks * 2048, 16384, 1024),
                               gdesc_k128(ds_addr + (ks >> 2) * 1024 + (ks & 3) * 32), ks > 0 ? 1u : 0u);
  };
  // D4 of hidden half h into the CTA sums: register e holds hidden unit 64h + 16q + lane/4 + 8(e/2), output
  // 2(lane%4) + e%2.  Flushed per tile so that no D4 registers are live across the epilogues.
  auto add_d4 = [&](const float (&d)[4], int h) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int hid = 64 * h + 16 * q + (lane >> 2) + 8 * (e >> 1), o = 2 * (lane & 3) + (e & 1);
      if (o < O) atomicAdd(s_gw4 + o * kHidH + hid, d[e]);
    }
  };
  long long n = 0;
  bool mine = false;                                 // this warpgroup took a tile (D3 holds sums)
  mbar_wait(w_full, 0);
  for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++n) {
    if (n % kGroupsMB != g) continue;
    const uint32_t s = static_cast<uint32_t>(n % p.stages);
    const int b = static_cast<int>(tile / p.tiles_per_b);
    const long long p0 = (tile % p.tiles_per_b) * 128;
    const long long pos = p0 + my_row;
    long long base;
    if constexpr (kPad) base = pos < p.S ? pad_row_to_offset(pm, static_cast<uint32_t>(b * p.S + pos)) : -1;
    else base = pos < p.S ? row_to_offset(p.map, static_cast<uint32_t>(b * p.S + pos)) : 0;
    __half2 dsh[O][2];                               // s dout[row, o] of the thread's rows frag_row(q, lane, 2m + {0, 1})
#pragma unroll
    for (int o = 0; o < O; ++o) {
      const float dl = (kPad ? base >= 0 : pos < p.S) ? p.dout[base + o * p.plane] : 0.f;
      float sum = dl;                                // db4: this warp's 32 rows, one shared-memory add per warp
#pragma unroll
      for (int m = 16; m > 0; m >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, m);
      if (lane == 0) atomicAdd(s_gb4 + o, sum);
      const float ds = dl * scale;
      *reinterpret_cast<__half*>(dsbuf + ds_off + o * 128 + ((ds_chunk ^ o) << 4)) = __float2half_rn(ds);
#pragma unroll
      for (int m = 0; m < 2; ++m)
        dsh[o][m] = __floats2half2_rn(__shfl_sync(0xffffffffu, ds, (lane & ~3) | (2 * m)),
                                      __shfl_sync(0xffffffffu, ds, (lane & ~3) | (2 * m + 1)));
    }
    mbar_wait(&a_full[s], (n / p.stages) & 1);
    const uint32_t abase = smem_u32(s_a + s * tile_bytes);
    float acc2[NG];                                  // dh0 [pos, c]: 128 x NG
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {                 // hidden units [64 hh, 64 hh + 64)
      float acc[64];
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < KR / 16; ++ks)
        wg_mma128<false, 1, 0>(acc, 64, gdesc_mn128(abase + ks * 2048, half_bytes, 1024), half_bytes,
                               gdesc_k128(w3_addr + hh * 8192 + ks * 32), ks > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(acc);
      // ---- epi A: P' = gelu'(pre) sum_o ds W4[o] into the A registers and the smem tile; G = gelu(pre)
#pragma unroll
      for (int mh = 0; mh < 2; ++mh) {
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          uint32_t gv[4];                            // A register i of step ks: the pair acc[8ks + 2i, + 1] (afrag_from_acc)
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float* a = acc + 32 * mh + 8 * ks + 2 * i;
            const int j = 2 * ks + (i >> 1);
            const GeluH2 vg = gelu_vg_h2(h2_from_f32(a[0], a[1]));
            gv[i] = h2_bits(vg.value);
            // s dout of the pair's row (row 2mh + i%2 of the thread) in both halves
            __half2 w = __hmul2((i & 1) ? __high2half2(dsh[0][mh]) : __low2half2(dsh[0][mh]),
                                h2_of_bits(s_w4h[32 * hh + 4 * j + cq]));
#pragma unroll
            for (int o = 1; o < O; ++o)
              w = __hfma2((i & 1) ? __high2half2(dsh[o][mh]) : __low2half2(dsh[o][mh]),
                          h2_of_bits(s_w4h[64 * o + 32 * hh + 4 * j + cq]), w);
            pa[mh][ks][i] = h2_bits(__hmul2(vg.grad, w));
          }
          const uint32_t row = 64 * mh + p_row, chunk = 2 * ks + (mi >> 1);
          const uint32_t sw = row * 128 + ((chunk ^ (row & 7)) << 4);
          stmatrix_x4(p_addr + hh * 16384 + sw, pa[mh][ks]);
          stmatrix_x4(gt_addr + sw, gv);
        }
      }
      fence_proxy_async_smem();
      asm volatile("bar.sync %0, 128;" ::"r"(barid) : "memory");     // G (and, on the first half, ds) complete
      float d4[4];
      wgmma_fence();
      if (hh == 0) mma2(acc2, 0);                    // MMA2 over the first half, before the second half's MMA1
      mma4(d4);
      wgmma_commit();
      wgmma_wait<0>();                               // the G buffer is free for the next half
      acc_fence(d4);
      add_d4(d4, hh);
    }
    {
      // ---- hs: fp16 copy of the h tile at the thread's rows, channels c = l%4 (mod 4) below C (row C: ones)
      const uint8_t* src = s_a + s * tile_bytes;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int row = frag_row(q, lane, k);
        const uint32_t colo = (row >> 6) * half_bytes + ((row & 7) << 1);
        const uint32_t ch = (row & 63) >> 3;
#pragma unroll
        for (int cc = 0; cc < KR / 4; ++cc) {
          const int c = 4 * cc + cq;
          const uint32_t off = colo + c * 128 + ((ch ^ (c & 7)) << 4);
          if (c < p.C) {
            const uint16_t hv = *reinterpret_cast<const uint16_t*>(src + off);
            *reinterpret_cast<__half*>(hsbuf + off) = __float2half_rn(__uint_as_float(static_cast<uint32_t>(hv) << 16));
          }
        }
      }
    }
    if (leader) tma_store_wait_read();               // the previous tile's g staging is free after the barrier
    fence_proxy_async_smem();
    asm volatile("bar.sync %0, 128;" ::"r"(barid) : "memory");
    wgmma_fence();
    mma2(acc2, 1);
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {                 // MMA3: K = positions; A = P' read MN-major (hid contiguous)
      const uint32_t kb = ks >> 2, kk = ks & 3;
      wg_mma128<true, 1, 0>(d3, KR, gdesc_mn128(p_addr + ks * 2048, 16384, 1024), 16384,
                            gdesc_k128(hs_addr + kb * half_bytes + kk * 32), (mine || ks > 0) ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(acc2);
    acc_fence(d3);
    mine = true;
    if (leader) mbar_arrive(&a_empty[s]);
    // ---- epi B: g[c, pos] = dh0[pos, c] / s, staged as bf16 [c][64 pos] x 2 (the TMA box layout)
    const float inv = 1.0f / scale;
#pragma unroll
    for (int mh = 0; mh < 2; ++mh) {
#pragma unroll
      for (int t = 0; t < NG / 16; ++t) {
        uint32_t r[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float* a = acc2 + (NG / 2) * mh + 4 * (2 * t + (i >> 1)) + 2 * (i & 1);
          r[i] = pack_bf16x2(inv * a[0], inv * a[1]);
        }
        const uint32_t c = 16 * t + 8 * (mi >> 1) + mk;
        stmatrix_x4_trans(g_addr + mh * half_bytes + c * 128 + ((g_chunk ^ (c & 7)) << 4), r);
      }
    }
    fence_proxy_async_smem();
    asm volatile("bar.sync %0, 128;" ::"r"(barid) : "memory");
    if (leader) {
      const int row0 = b * p.C;
      tma_store_2d(&tmG, gbuf, static_cast<int32_t>(p0), row0);
      if (p0 + 64 < p.S) tma_store_2d(&tmG, gbuf + half_bytes, static_cast<int32_t>(p0 + 64), row0);
      tma_store_commit();
    }
  }
  if (leader) tma_store_wait_all();
  // ---- per-CTA flush of the weight gradients
  if (mine) {
    const float inv = 1.0f / scale;
    // fragment of the 128 x KR accumulator: register (KR/2)h + 4j + e holds hidden unit 64h + 16q + lane/4 + 8(e/2),
    // column 8j + 2(lane%4) + e%2
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < KR / 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int hid = 64 * h + 16 * q + (lane >> 2) + 8 * (e >> 1), c = 8 * j + 2 * (lane & 3) + (e & 1);
          const float v = d3[(KR / 2) * h + 4 * j + e] * inv;
          if (c < p.C) atomicAdd(p.gW3 + hid * p.C + c, v);
          else if (c == p.C) atomicAdd(p.gb3 + hid, v);
        }
  }
  asm volatile("bar.sync 3, %0;" ::"n"(128 * kGroupsMB) : "memory");
  if (num_tiles > blockIdx.x) {
    const float inv = 1.0f / scale;
    for (int i = threadIdx.x; i < O * kHidH; i += 128 * kGroupsMB) atomicAdd(p.gW4 + i, s_gw4[i] * inv);
    if (threadIdx.x < O) atomicAdd(p.gb4 + threadIdx.x, s_gb4[threadIdx.x]);
  }
}

template <int KR, int O>
__global__ void __launch_bounds__(kThreadsMB, 1)
head_bwd_multi_kernel(const __grid_constant__ CUtensorMap tmH, const __grid_constant__ CUtensorMap tmW3,
                      const __grid_constant__ CUtensorMap tmW3T, const __grid_constant__ CUtensorMap tmG,
                      const HeadMultiBwdParams p) {
  head_bwd_multi_body<KR, O, false>(tmH, tmW3, tmW3T, tmG, p, PadRowMap{});
}

template <int KR, int O>
__global__ void __launch_bounds__(kThreadsMB, 1)
head_bwd_multi_pad_kernel(const __grid_constant__ CUtensorMap tmH, const __grid_constant__ CUtensorMap tmW3,
                          const __grid_constant__ CUtensorMap tmW3T, const __grid_constant__ CUtensorMap tmG,
                          const HeadMultiBwdParams p, const __grid_constant__ PadRowMap pm) {
  head_bwd_multi_body<KR, O, true>(tmH, tmW3, tmW3T, tmG, p, pm);
}

// ================================================================================ dispatch over (KR, O)
template <int KR, int O, bool kPad>
void launch_fwd(int grid, uint32_t smem, cudaStream_t st, const CUtensorMap& a, const CUtensorMap& b,
                const HeadMultiFwdParams p, const PadRowMap pm) {
  if constexpr (kPad) head_fwd_multi_pad_kernel<KR, O><<<grid, kThreadsMF, smem, st>>>(a, b, p, pm);
  else head_fwd_multi_kernel<KR, O><<<grid, kThreadsMF, smem, st>>>(a, b, p);
}
template <int KR, int O, bool kPad>
void launch_bwd(int grid, uint32_t smem, cudaStream_t st, const CUtensorMap& a, const CUtensorMap& b,
                const CUtensorMap& c, const CUtensorMap& d, const HeadMultiBwdParams p, const PadRowMap pm) {
  if constexpr (kPad) head_bwd_multi_pad_kernel<KR, O><<<grid, kThreadsMB, smem, st>>>(a, b, c, d, p, pm);
  else head_bwd_multi_kernel<KR, O><<<grid, kThreadsMB, smem, st>>>(a, b, c, d, p);
}

template <int KR, bool kPad>
const void* fwd_fn(int O) {
  return O == 1 ? (kPad ? reinterpret_cast<const void*>(head_fwd_multi_pad_kernel<KR, 1>)
                      : reinterpret_cast<const void*>(head_fwd_multi_kernel<KR, 1>))
       : O == 2 ? (kPad ? reinterpret_cast<const void*>(head_fwd_multi_pad_kernel<KR, 2>)
                      : reinterpret_cast<const void*>(head_fwd_multi_kernel<KR, 2>))
       : O == 3 ? (kPad ? reinterpret_cast<const void*>(head_fwd_multi_pad_kernel<KR, 3>)
                      : reinterpret_cast<const void*>(head_fwd_multi_kernel<KR, 3>))
                : (kPad ? reinterpret_cast<const void*>(head_fwd_multi_pad_kernel<KR, 4>)
                      : reinterpret_cast<const void*>(head_fwd_multi_kernel<KR, 4>));
}
template <int KR, bool kPad>
const void* bwd_fn(int O) {
  return O == 1 ? (kPad ? reinterpret_cast<const void*>(head_bwd_multi_pad_kernel<KR, 1>)
                      : reinterpret_cast<const void*>(head_bwd_multi_kernel<KR, 1>))
       : O == 2 ? (kPad ? reinterpret_cast<const void*>(head_bwd_multi_pad_kernel<KR, 2>)
                      : reinterpret_cast<const void*>(head_bwd_multi_kernel<KR, 2>))
       : O == 3 ? (kPad ? reinterpret_cast<const void*>(head_bwd_multi_pad_kernel<KR, 3>)
                      : reinterpret_cast<const void*>(head_bwd_multi_kernel<KR, 3>))
                : (kPad ? reinterpret_cast<const void*>(head_bwd_multi_pad_kernel<KR, 4>)
                      : reinterpret_cast<const void*>(head_bwd_multi_kernel<KR, 4>));
}

template <int KR, bool kPad>
void launch_fwd_o(int O, int grid, uint32_t smem, cudaStream_t st, const CUtensorMap& a, const CUtensorMap& b,
                  const HeadMultiFwdParams p, const PadRowMap pm) {
  if (O == 1) launch_fwd<KR, 1, kPad>(grid, smem, st, a, b, p, pm);
  else if (O == 2) launch_fwd<KR, 2, kPad>(grid, smem, st, a, b, p, pm);
  else if (O == 3) launch_fwd<KR, 3, kPad>(grid, smem, st, a, b, p, pm);
  else launch_fwd<KR, 4, kPad>(grid, smem, st, a, b, p, pm);
}
template <int KR, bool kPad>
void launch_bwd_o(int O, int grid, uint32_t smem, cudaStream_t st, const CUtensorMap& a, const CUtensorMap& b,
                  const CUtensorMap& c, const CUtensorMap& d, const HeadMultiBwdParams p, const PadRowMap pm) {
  if (O == 1) launch_bwd<KR, 1, kPad>(grid, smem, st, a, b, c, d, p, pm);
  else if (O == 2) launch_bwd<KR, 2, kPad>(grid, smem, st, a, b, c, d, p, pm);
  else if (O == 3) launch_bwd<KR, 3, kPad>(grid, smem, st, a, b, c, d, p, pm);
  else launch_bwd<KR, 4, kPad>(grid, smem, st, a, b, c, d, p, pm);
}

const char* set_max_smem(const void* fn, bool* done) {
  if (*done) return nullptr;
  if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess)
    return "cudaFuncSetAttribute failed";
  *done = true;
  return nullptr;
}

}  // namespace

// h: bf16 [B*C, S] channel-major; W3aug: bf16 [128, 64] with column C = b3; w4b4: fp32 [O*128 + O] (W4 [O, 128] then
// b4 [O]); out: fp32, row addressed through the row digits (row = b*S + position), output channel o at + o*plane.
const char* head_fwd_multi(const void* h, const void* W3aug, const float* w4b4, float* out, int B, int C, long long S,
                           int O, long long plane, int nrl, const int* R, const long long* SR, const int* lim,
                           int num_sms, cudaStream_t stream) {
  if (C < 1 || C > 47) return "head_fwd_multi: 1 <= C <= 47";
  if (O < 1 || O > kMaxOut) return "head_fwd_multi: 1 <= O <= 4";
  if (S % 8 || S > (1ll << 31) - 256 || static_cast<long long>(B) * S > (1ll << 31) - 256)
    return "head_fwd_multi: bad slab size";
  HeadMultiFwdParams p{};
  p.B = B; p.C = C; p.S = S; p.tiles_per_b = (S + 127) / 128; p.plane = plane;
  p.w4b4 = w4b4; p.out = out;
  PadRowMap pm{};
  if (lim ? set_padrowmap(&pm, nrl, R, SR, lim) : set_rowmap(&p.map, nrl, R, SR))
    return lim ? "head_fwd_multi: 1..5 row digits, each bound within its radix" : "head_fwd_multi: 1..4 row digits";
  CUtensorMap tmH, tmW3;
  if (make_map_2d(&tmH, h, S, static_cast<uint64_t>(B) * C, S, 64, C)) return "tensor map (h) failed";
  if (make_map_2d(&tmW3, W3aug, 64, 128, 64, 64, 128)) return "tensor map (W3) failed";
  const int KR = (C + 1 + 15) / 16 * 16, kr_i = KR / 16 - 1;
  static bool attr[2][3][kMaxOut] = {};
  const int pd = lim ? 1 : 0;
  const void* fn = pd ? (kr_i == 0 ? fwd_fn<16, true>(O) : kr_i == 1 ? fwd_fn<32, true>(O) : fwd_fn<48, true>(O))
                      : (kr_i == 0 ? fwd_fn<16, false>(O) : kr_i == 1 ? fwd_fn<32, false>(O) : fwd_fn<48, false>(O));
  if (const char* e = set_max_smem(fn, &attr[pd][kr_i][O - 1])) return e;
  const uint32_t smem_bytes = 16384 + kStagesMF * 2 * KR * 128 + 2048 + 1024;
  const long long tiles = p.tiles_per_b * B;
  const int grid = static_cast<int>(tiles < num_sms ? tiles : num_sms);
#define DFNO_HEAD_FWD_MULTI(P_)                                                          \
  if (kr_i == 0) launch_fwd_o<16, P_>(O, grid, smem_bytes, stream, tmH, tmW3, p, pm);      \
  else if (kr_i == 1) launch_fwd_o<32, P_>(O, grid, smem_bytes, stream, tmH, tmW3, p, pm); \
  else launch_fwd_o<48, P_>(O, grid, smem_bytes, stream, tmH, tmW3, p, pm);
  if (pd) { DFNO_HEAD_FWD_MULTI(true) } else { DFNO_HEAD_FWD_MULTI(false) }
#undef DFNO_HEAD_FWD_MULTI
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

// W3T16: fp16 [KR, 128] (rows = input channel, zero padded); W4: fp32 [O, 128]; dout: fp32 public layout of n_dout
// elements (all O planes); amax_ws: one uint of scratch (receives max |dout|); g: bf16 [B*C, S]; gradients gW4 [O, 128]
// and gb4 [O] as well as gW3 / gb3 are accumulated with atomics.
const char* head_bwd_multi(const void* h, const void* W3aug, const void* W3T16, const float* W4, const float* dout,
                           long long n_dout, unsigned* amax_ws, void* g, float* gW3, float* gb3, float* gW4, float* gb4,
                           int B, int C, long long S, int O, long long plane, int nrl, const int* R,
                           const long long* SR, const int* lim, int num_sms, cudaStream_t stream) {
  // C = 32 (KR = 48) would need more than the 240 consumer registers (ptxas keeps a stack frame): not instantiated
  if (C < 1 || C > 31) return "head_bwd_multi: 1 <= C <= 31";
  if (O < 1 || O > kMaxOut) return "head_bwd_multi: 1 <= O <= 4";
  if (S % 8 || S > (1ll << 31) - 256 || static_cast<long long>(B) * S > (1ll << 31) - 256)
    return "head_bwd_multi: bad slab size";
  HeadMultiBwdParams p{};
  p.B = B; p.C = C; p.S = S; p.tiles_per_b = (S + 127) / 128; p.plane = plane;
  p.dout = dout; p.amax = reinterpret_cast<const float*>(amax_ws); p.W4 = W4;
  p.gW3 = gW3; p.gb3 = gb3; p.gW4 = gW4; p.gb4 = gb4;
  PadRowMap pm{};
  if (lim ? set_padrowmap(&pm, nrl, R, SR, lim) : set_rowmap(&p.map, nrl, R, SR))
    return lim ? "head_bwd_multi: 1..5 row digits, each bound within its radix" : "head_bwd_multi: 1..4 row digits";
  const int KR = (C + 1 + 15) / 16 * 16, kr_i = KR / 16 - 1;
  CUtensorMap tmH, tmW3, tmW3T, tmG;
  if (make_map_2d(&tmH, h, S, static_cast<uint64_t>(B) * C, S, 64, C)) return "tensor map (h) failed";
  if (make_map_2d(&tmW3, W3aug, 64, 128, 64, 64, 128)) return "tensor map (W3) failed";
  if (make_map_2d(&tmW3T, W3T16, 128, KR, 128, 64, KR)) return "tensor map (W3T) failed";
  if (make_map_2d(&tmG, g, S, static_cast<uint64_t>(B) * C, S, 64, C)) return "tensor map (g) failed";
  static bool attr[2][2][kMaxOut] = {};
  const int pd = lim ? 1 : 0;
  const void* fn = pd ? (kr_i == 0 ? bwd_fn<16, true>(O) : bwd_fn<32, true>(O))
                      : (kr_i == 0 ? bwd_fn<16, false>(O) : bwd_fn<32, false>(O));
  if (const char* e = set_max_smem(fn, &attr[pd][kr_i][O - 1])) return e;
  if (cudaMemsetAsync(amax_ws, 0, 4, stream) != cudaSuccess) return "head_bwd_multi: memset failed";
  absmax_kernel<<<num_sms * 4, 256, 0, stream>>>(dout, n_dout, amax_ws);
  const uint32_t tile_bytes = 2u * KR * 128;
  // + barriers, W4 pairs and the CTA sums of dW4 / db4 (4 KB), + 1 KB slack
  const uint32_t fixed = 16384 + tile_bytes + kGroupsMB * (kWgBytesMB + 2 * tile_bytes) + 4096 + 1024;
  p.stages = kMaxStagesMB;
  while (p.stages > kGroupsMB && fixed + p.stages * tile_bytes > 227 * 1024) p.stages -= kGroupsMB;
  const uint32_t smem_bytes = fixed + p.stages * tile_bytes;
  if (smem_bytes > 227 * 1024) return "head_bwd_multi: shared memory";
  const long long tiles = p.tiles_per_b * B;
  const int grid = static_cast<int>(tiles < num_sms ? tiles : num_sms);
  if (pd) {
    if (kr_i == 0) launch_bwd_o<16, true>(O, grid, smem_bytes, stream, tmH, tmW3, tmW3T, tmG, p, pm);
    else launch_bwd_o<32, true>(O, grid, smem_bytes, stream, tmH, tmW3, tmW3T, tmG, p, pm);
  } else {
    if (kr_i == 0) launch_bwd_o<16, false>(O, grid, smem_bytes, stream, tmH, tmW3, tmW3T, tmG, p, pm);
    else launch_bwd_o<32, false>(O, grid, smem_bytes, stream, tmH, tmW3, tmW3T, tmG, p, pm);
  }
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

}  // namespace dfno
