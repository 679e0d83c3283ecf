// head_sm90.cu -- projection head  out = W4 . gelu(W3 h + b3) + b4  (reference linear3 -> gelu -> linear4,
// dfno.py:348-351; SURVEY.md K17), forward and backward, straight from the engine's CHANNEL-MAJOR activation
// h[b*C + c][S positions] (no channels-last copy): a tile is 128 consecutive positions of all C channels,
// dropped into shared memory by TMA as two SWIZZLE_128B boxes of [C rows][64 positions] and used as an
// MN-major A operand (M = positions, K = channels).  Row C of every tile image is a constant row of ones and
// column C of the W3 operand holds b3, so the hidden bias rides through the MMA -- and, in the backward, the
// same ones row turns the tensor core into the reducer for db3.  The 128-channel hidden layer never exists in
// memory.
//
//   forward   MMA   pre[pos, j] = sum_c h[c, pos] W3[j, c] + b3[j]
//             epi   out[pos]    = b4 + sum_j W4[j] gelu(pre[pos, j])      (packed fp16 GELU, HFMA2 dot)
//
//   backward  MMA1  pre (as above)
//             epi A P[pos, j]   = W4[j] gelu'(pre)  (fp16 tile in smem);  dW4[j] += sum_pos dout gelu(pre)
//                   hs[c, pos]  = s dout[pos] h[c, pos],  hs[C, pos] = s dout[pos]   (fp16, s = 2^k keeps the
//                                 loss gradient inside the fp16 range; undone when the sums are flushed)
//             MMA2  dh0[pos, i]    = sum_j P[pos, j] W3[j, i]          epi B: g[i, pos] = dout[pos] dh0[pos, i]
//             MMA3  D3[j, i]      += sum_pos P[pos, j] hs[i, pos]      -> dW3 (i < C), db3 (i = C)
//
// Widths 48 and 64 (KR = 64, 80): W3aug spans KR columns, so at KR = 80 it is two 64-column swizzle blocks ([H, 128]
// in memory, b3 in column 64).  The backward cannot hold dh0 (KR registers), D3 (KR) and an MMA1 half (64) at once in
// the 240 registers of a consumer: it runs MMA2 after both MMA1 halves, from the P tile in shared memory, in two
// channel-column groups (32 + 32 or 48 + 32) whose epilogue B runs in turn.  MMA1 runs in 32-unit quarters, the hs
// copy walks its four rows in a loop (unrolled, ptxas keeps all 4 KR of its shared addresses live across tiles), the
// dW4 sums stay in shared memory as at KR = 48 (24 of the 32 at KR = 80), and g is staged in the warpgroup's hs buffer
// (free once MMA3 has read it), which keeps KR = 80 inside shared memory.
#include <type_traits>

#include "head_common.cuh"
#include "kernels.h"
#include "tma_host.h"

namespace dfno {
namespace {

// ================================================================================ forward
// The epilogue is latency bound (each GELU pair is a dependent chain of about ten steps), so the warps a scheduler can
// switch between set its speed.  KR <= 48 runs MMA1 in two 64-unit hidden halves, each followed by its share of the
// epilogue: the accumulator is 64 registers, which lets 4 consumer warpgroups and the TMA warp share the register file
// (17 warps, at most 120 registers each).  KR = 64, 80 keep one 128-unit pass in 2 warpgroups.
template <int KR>
constexpr bool kWideHF = KR > 48;
template <int KR>
constexpr int kGroupsHF = kWideHF<KR> ? 2 : 4;  // consumer warpgroups (kStagesHF a multiple of it: see bypass_sm90.cu)
template <int KR>
constexpr int kStagesHF = kWideHF<KR> ? 6 : 8;
static_assert(kStagesHF<16> % kGroupsHF<16> == 0 && kStagesHF<80> % kGroupsHF<80> == 0,
              "every ring stage must belong to one consumer warpgroup");
template <int KR>
constexpr int kThreadsHF = 128 * kGroupsHF<KR> + 32;

struct HeadFwdParams {
  int B, C, KR;
  long long S, tiles_per_b;
  const float* w4b4;          // [128 weights, 1 bias]
  float* out;
  RowMap map;
};

// The epilogue works on the accumulator fragment (frag_row); the W4 dot is finished across the 4 lanes of a quad.

// KR: channels + the ones row, padded to 16 (the K of the MMA).  kPad: h is a zero-padded activation whose rows map
// through pm; pad rows store nothing (p.map is not read).
template <int KR, bool kPad>
__device__ __forceinline__ void head_fwd_body(const CUtensorMap& tmH, const CUtensorMap& tmW3, const HeadFwdParams p,
                                              const PadRowMap pm) {
  extern __shared__ __align__(1024) uint8_t smem[];
  constexpr int kStages = kStagesHF<KR>, kGroups = kGroupsHF<KR>;
  constexpr int kN = kWideHF<KR> ? kHidH : 64;             // hidden units per MMA1 pass
  constexpr uint32_t w3_bytes = KR > 64 ? 32768u : 16384u;  // one or two [128 hid][64] blocks
  uint8_t* s_w3 = smem;                                    // [128 hid][64] K-major block(s), column C = b3
  uint8_t* s_a = smem + w3_bytes;                          // stages x 2 halves x [KR rows][64 pos]
  constexpr uint32_t half_bytes = KR * 128;
  constexpr uint32_t stage_bytes = 2 * half_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_a + kStages * stage_bytes);
  uint64_t* full = bars;                    // [kStages]
  uint64_t* empty = bars + kStages;         // [kStages]
  uint64_t* wfull = bars + 2 * kStages;
  uint32_t* s_w4 = reinterpret_cast<uint32_t*>(bars + 2 * kStages + 2);   // [64] fp16x2 pairs of W4 (16-byte aligned)
  float* s_b4 = reinterpret_cast<float*>(s_w4 + 64);

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const long long num_tiles = p.tiles_per_b * p.B;

  for (uint32_t i = threadIdx.x; i < kStages * stage_bytes / 16; i += blockDim.x)
    reinterpret_cast<uint4*>(s_a)[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < kStages * 2 * 16; i += blockDim.x) {        // the ones row (row C) of every half
    const uint32_t hb = i >> 4, ch = i & 15;
    reinterpret_cast<uint2*>(s_a + hb * half_bytes + p.C * 128)[ch] = make_uint2(0x3F803F80u, 0x3F803F80u);
  }
  for (int i = threadIdx.x; i < 64; i += blockDim.x)
    s_w4[i] = h2_bits(h2_from_f32(p.w4b4[2 * i], p.w4b4[2 * i + 1]));
  if (threadIdx.x == 0) s_b4[0] = p.w4b4[kHidH];
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmH); tma_prefetch_desc(&tmW3);
    for (int s = 0; s < kStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 1); }
    mbar_init(wfull, 1);
    fence_barrier_init();
  }
  fence_proxy_async_smem();
  __syncthreads();

  if (warp == 4 * kGroups) {
    if (lane == 0) {
      mbar_arrive_expect_tx(wfull, w3_bytes);
      tma_load_2d(s_w3, &tmW3, wfull, 0, 0);
      if constexpr (KR > 64) tma_load_2d(s_w3 + 16384, &tmW3, wfull, 64, 0);
      uint32_t s = 0, ph = 0;
      for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int b = static_cast<int>(tile / p.tiles_per_b);
        const int p0 = static_cast<int>((tile % p.tiles_per_b) * 128);
        mbar_wait(&empty[s], ph ^ 1);
        mbar_arrive_expect_tx(&full[s], 2u * p.C * 128);
        uint8_t* st = s_a + s * stage_bytes;
        tma_load_2d(st, &tmH, &full[s], p0, b * p.C);
        tma_load_2d(st + half_bytes, &tmH, &full[s], p0 + 64, b * p.C);
        if (++s == kStages) { s = 0; ph ^= 1; }
      }
    }
    return;
  }
  const int q = warp & 3, g = warp >> 2, cq = lane & 3;
  const int my_row = frag_row(q, lane, cq);          // the row this lane stores (each lane of a quad stores one)
  const float b4 = s_b4[0];
  const uint32_t w_addr = smem_u32(s_w3);
  uint32_t w4[16];                                   // W4 pairs of this thread's hidden units 8j + 2(l%4) + {0, 1}
#pragma unroll
  for (int j = 0; j < 16; ++j) w4[j] = s_w4[4 * j + cq];
  mbar_wait(wfull, 0);
  float acc[kN];
  long long n = 0;
  for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++n) {
    if (n % kGroups != g) continue;
    const uint32_t s = static_cast<uint32_t>(n % kStages);
    const int b = static_cast<int>(tile / p.tiles_per_b);
    const long long pos = (tile % p.tiles_per_b) * 128 + my_row;
    mbar_wait(&full[s], (n / kStages) & 1);
    // pre[pos, j] = sum_c h[c, pos] W3aug[j, c]: A MN-major (positions contiguous, 64-position halves half_bytes apart)
    const uint32_t abase = smem_u32(s_a + s * stage_bytes);
    // row k of the thread: registers (kN/2)(k/2) + 4j + 2(k%2) + {0, 1} of a pass; one fp16 dot chain of 8 pairs per
    // 64 hidden units, each chain's sum added to out[k] in hidden-unit order
    float out[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int hh = 0; hh < kHidH / kN; ++hh) {        // hidden units [kN hh, kN hh + kN): W3 rows 128 bytes apart
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < KR / 16; ++ks) {
        // k16 step ks of W3aug: 64-column block ks / 4 (a second block only at KR = 80)
        const uint32_t w_k = KR > 64 ? (ks >> 2) * 16384 + (ks & 3) * 32 : ks * 32;
        wg_mma128<false, 1, 0>(acc, kN, gdesc_mn128(abase + ks * 2048, half_bytes, 1024), half_bytes,
                               gdesc_k128(w_addr + hh * kN * 128 + w_k), ks > 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(acc);
      if (hh == kHidH / kN - 1 && q == 0 && lane == 0) mbar_arrive(&empty[s]);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float* a = acc + (kN / 2) * (k >> 1) + 2 * (k & 1);
#pragma unroll
        for (int half = 0; half < kN / 64; ++half) {
          __half2 part = __float2half2_rn(0.f);
#pragma unroll
          for (int j = 8 * half; j < 8 * half + 8; ++j)
            part = __hfma2(gelu_h2(h2_from_f32(a[4 * j], a[4 * j + 1])), h2_of_bits(w4[(kN / 8) * hh + j]), part);
          const float2 f = __half22float2(part);
          out[k] += f.x + f.y;
        }
        if (hh == kHidH / kN - 1) {
          out[k] += __shfl_xor_sync(0xffffffffu, out[k], 1);
          out[k] += __shfl_xor_sync(0xffffffffu, out[k], 2);
        }
      }
    }
    if constexpr (kPad) {
      const long long o = pos < p.S ? pad_row_to_offset(pm, static_cast<uint32_t>(b * p.S + pos)) : -1;
      if (o >= 0) p.out[o] = b4 + pick4(out, cq);
    } else {
      if (pos < p.S) p.out[row_to_offset(p.map, static_cast<uint32_t>(b * p.S + pos))] = b4 + pick4(out, cq);
    }
  }
}

template <int KR>
__global__ void __launch_bounds__(kThreadsHF<KR>, 1)
head_fwd_kernel(const __grid_constant__ CUtensorMap tmH, const __grid_constant__ CUtensorMap tmW3,
                const HeadFwdParams p) {
  head_fwd_body<KR, false>(tmH, tmW3, p, PadRowMap{});
}

template <int KR>
__global__ void __launch_bounds__(kThreadsHF<KR>, 1)
head_fwd_pad_kernel(const __grid_constant__ CUtensorMap tmH, const __grid_constant__ CUtensorMap tmW3,
                    const HeadFwdParams p, const __grid_constant__ PadRowMap pm) {
  head_fwd_body<KR, true>(tmH, tmW3, p, pm);
}

// ================================================================================ backward
constexpr int kMaxStagesHB = 6;                 // h tiles are small: deep prefetch keeps TMA latency off the consumers
constexpr int kGroupsHB = 2;                    // consumer warpgroups (stages a multiple of it: see bypass_sm90.cu)
// One producer WARPGROUP (one warp issues TMA): setmaxnreg moves its registers to the consumers, whose fragment
// epilogues need more than the uniform 168 per thread of a 384-thread block.
constexpr int kThreadsHB = 128 * kGroupsHB + 128;
constexpr int kProducerRegsHB = 24, kConsumerRegsHB = 240;
static_assert(128 * kProducerRegsHB + 128 * kGroupsHB * kConsumerRegsHB <= 65536, "register file");
// KR = 64, 80 (widths 48, 64): MMA2 from shared memory in channel groups, g staged over hs (see the file header)
template <int KR>
constexpr bool kWideHB = KR > 48;
template <int KR>
constexpr bool kWsumSmem = KR > 32 && !kWideHB<KR>;
// KR = 64, 80: the first kWsumSmemW dW4 column sums live in shared memory, the rest in registers (all 32 do not fit the
// shared memory of KR = 80)
template <int KR>
constexpr int kWsumSmemW = !kWideHB<KR> ? 0 : KR > 64 ? 24 : 32;

struct HeadBwdParams {
  int B, C, KR, stages;
  long long S, tiles_per_b;
  const float* dout;          // fp32, public layout
  const float* amax;          // max |dout| (device scalar)
  const float* W4;
  float* gW3; float* gb3; float* gW4; float* gb4;
  RowMap map;
};

// Per tile of 128 positions, one consumer warpgroup runs the backward of the file header; MMA1 in two
// 64-column halves so that the D3 accumulator fits next to it.  Both epilogues work on the accumulator fragments
// (frag_row): epilogue A turns each MMA1 half into P in registers, which feeds MMA2 as its register A operand and is
// stored once with stmatrix for MMA3; dW4 stays in per-thread column registers until the flush; epilogue B stages
// g as bf16 [C][128 positions] with stmatrix.trans and writes it with two TMA stores.
// KR: channels + the ones row, padded to 16 (the N of MMA2 / MMA3 and the accumulator width).  kPad: rows map through
// pm and pad rows read dout as 0, so g is exactly 0 there and they add nothing to dW3, db3, dW4, db4.
template <int KR, bool kPad>
__device__ __forceinline__ void head_bwd2_body(const CUtensorMap& tmH, const CUtensorMap& tmW3, const CUtensorMap& tmW3T,
                                               const CUtensorMap& tmG, const HeadBwdParams p, const PadRowMap pm) {
  extern __shared__ __align__(1024) uint8_t smem[];
  constexpr uint32_t half_bytes = KR * 128;
  constexpr uint32_t tile_bytes = 2 * half_bytes;
  constexpr uint32_t w3_bytes = KR > 64 ? 32768u : 16384u;
  uint8_t* s_w3 = smem;                                   // 16 KB (32 KB at KR = 80)
  uint8_t* s_w3t = s_w3 + w3_bytes;                       // 2 k-blocks x [KR c rows][64 hid] fp16
  uint8_t* s_p = s_w3t + tile_bytes;                      // per warpgroup: 2 x [128 pos][64 hid] fp16
  uint8_t* s_a = s_p + kGroupsHB * 32768;                 // stages x h tile
  uint8_t* s_hs = s_a + p.stages * tile_bytes;            // per warpgroup: scaled fp16 copy of the h tile
  // per warpgroup: bf16 g staging, 2 x [KR c rows][64 pos] (the hs buffer itself at KR >= 64)
  uint8_t* s_g = kWideHB<KR> ? s_hs : s_hs + kGroupsHB * tile_bytes;
  // KR = 48 leaves no registers for the dW4 column sums: they live in [32][consumer threads] floats instead
  float* s_wsum = reinterpret_cast<float*>(s_g + kGroupsHB * tile_bytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_wsum + (kWsumSmem<KR> ? 32 * 128 * kGroupsHB : 0) +
                                               kWsumSmemW<KR> * 128 * kGroupsHB);
  uint64_t* a_full = bars;            // [8]
  uint64_t* a_empty = bars + 8;       // [8]
  uint64_t* w_full = bars + 16;
  float* s_gb4 = reinterpret_cast<float*>(bars + 18);
  uint32_t* s_w4h = reinterpret_cast<uint32_t*>(bars + 20);   // [64] fp16x2 pairs of W4 (16-byte aligned)
  float* s_gw4 = reinterpret_cast<float*>(s_w4h + 64);       // [128] CTA partial sums of dW4
  float* s_ds = s_gw4 + kHidH;                                // KR <= 48, per warpgroup: [128 positions] s dout

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const long long num_tiles = p.tiles_per_b * p.B;

  for (uint32_t i = threadIdx.x; i < p.stages * tile_bytes / 16; i += blockDim.x)
    reinterpret_cast<uint4*>(s_a)[i] = make_uint4(0, 0, 0, 0);
  for (uint32_t i = threadIdx.x; i < kGroupsHB * tile_bytes / 16; i += blockDim.x)
    reinterpret_cast<uint4*>(s_hs)[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < static_cast<uint32_t>(p.stages) * 2 * 16; i += blockDim.x) {
    const uint32_t hb = i >> 4, ch = i & 15;
    reinterpret_cast<uint2*>(s_a + hb * half_bytes + p.C * 128)[ch] = make_uint2(0x3F803F80u, 0x3F803F80u);
  }
  if (threadIdx.x == 0) s_gb4[0] = 0.f;
  for (int i = threadIdx.x; i < 64; i += blockDim.x) s_w4h[i] = h2_bits(h2_from_f32(p.W4[2 * i], p.W4[2 * i + 1]));
  for (int i = threadIdx.x; i < kHidH; i += blockDim.x) s_gw4[i] = 0.f;
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

  if (warp >= 4 * kGroupsHB) {
    setmaxnreg_dec<kProducerRegsHB>();
    if (warp == 4 * kGroupsHB && lane == 0) {
      mbar_arrive_expect_tx(w_full, w3_bytes + tile_bytes);
      tma_load_2d(s_w3, &tmW3, w_full, 0, 0);
      if constexpr (KR > 64) tma_load_2d(s_w3 + 16384, &tmW3, w_full, 64, 0);
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

  setmaxnreg_inc<kConsumerRegsHB>();
  const int q = warp & 3, g = warp >> 2, cq = lane & 3;
  const int my_row = frag_row(q, lane, cq);          // the row whose dout this lane loads
  const uint32_t barid = 1 + g;
  const bool leader = q == 0 && lane == 0;           // releases ring stages and issues this warpgroup's g stores
  uint8_t* pbuf = s_p + g * 32768;
  uint8_t* hsbuf = s_hs + g * tile_bytes;
  uint8_t* gbuf = s_g + g * tile_bytes;
  const uint32_t w3_addr = smem_u32(s_w3), w3t_addr = smem_u32(s_w3t);
  const uint32_t p_addr = smem_u32(pbuf), hs_addr = smem_u32(hsbuf), g_addr = smem_u32(gbuf);
  // stmatrix: lane 8i + k addresses row k of matrix i.  P (epilogue A): matrix i = positions 16q + 8(i%2) + k of an
  // m64 half, hidden units 8(i/2).. of a k16 step.  g (epilogue B, transposed): memory row k of matrix i = channel
  // 8(i/2) + k of a 16-channel group, holding positions 16q + 8(i%2) .. + 7 (16-byte chunk 2q + i%2 of the row).
  const int mi = lane >> 3, mk = lane & 7;
  const uint32_t p_row = 16 * q + 8 * (mi & 1) + mk;
  const uint32_t g_chunk = 2 * q + (mi & 1);
  float acc_gb4 = 0.f;
  float wsum[32];                                    // [16 hh + 2 j + e]: dW4 of hidden unit 64 hh + 8 j + 2(l%4) + e
  float* my_wsum = s_wsum + (threadIdx.x & (128 * kGroupsHB - 1));   // its shared slots (stride 128 kGroupsHB)
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    if constexpr (kWsumSmem<KR>) my_wsum[i * 128 * kGroupsHB] = 0.f;
    else if constexpr (kWideHB<KR>) { if (i < kWsumSmemW<KR>) my_wsum[i * 128 * kGroupsHB] = 0.f; else wsum[i] = 0.f; }
    else wsum[i] = 0.f;
  }
  // dW4 column sum i += v
  auto wsum_add = [&](int i, float d, float v) {
    if constexpr (kWsumSmem<KR>) my_wsum[i * 128 * kGroupsHB] = fmaf(d, v, my_wsum[i * 128 * kGroupsHB]);
    else if constexpr (kWideHB<KR>) {
      if (i < kWsumSmemW<KR>) my_wsum[i * 128 * kGroupsHB] = fmaf(d, v, my_wsum[i * 128 * kGroupsHB]);
      else wsum[i] = fmaf(d, v, wsum[i]);
    } else wsum[i] = fmaf(d, v, wsum[i]);
  };
  float d3[KR];                                      // [hid, c] over this warpgroup's tiles: 128 x KR
  uint32_t pa[2][4][4];                              // P of one 64-unit hidden half: [m64 half][k16 step][A register]
  // MMA2, hidden units [64 kb, 64 kb + 64): dh0 (+)= P . W3, A = the P registers
  auto mma2 = [&](float (&acc2)[KR], int kb) {
    if constexpr (!kWideHB<KR>) {
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const uint64_t db = gdesc_k128(w3t_addr + kb * half_bytes + ks * 32);
        const uint32_t sc = (kb > 0 || ks > 0) ? 1u : 0u;
        wg_mma64_rs<KR, 0, 0>(acc2, pa[0][ks], db, sc);
        wg_mma64_rs<KR, 0, KR / 2>(acc2, pa[1][ks], db, sc);
      }
    }
  };
  // KR >= 64: MMA2 for the channel columns [c0, c0 + NG), A = the P tile in shared memory (K-major, hidden units
  // contiguous), then epilogue B of those columns into the g staging
  auto mma2_group = [&](auto c0_, auto ng_, const float (&dk)[4]) {
    constexpr int c0 = decltype(c0_)::value, NG = decltype(ng_)::value;
    float a2[NG];                                    // dh0 [pos, c0 + n]: 128 x NG
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const uint32_t kb = ks >> 2, kk = ks & 3;
      wg_mma128<true, 0, 0>(a2, NG, gdesc_k128(p_addr + kb * 16384 + kk * 32), 8192,
                            gdesc_k128(w3t_addr + kb * half_bytes + c0 * 128 + kk * 32), ks > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(a2);
#pragma unroll
    for (int mh = 0; mh < 2; ++mh) {
#pragma unroll
      for (int t = 0; t < NG / 16; ++t) {
        uint32_t r[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float* a = a2 + (NG / 2) * mh + 4 * (2 * t + (i >> 1)) + 2 * (i & 1);
          const float d = dk[2 * mh + (i & 1)];
          r[i] = pack_bf16x2(d * a[0], d * a[1]);
        }
        const uint32_t c = c0 + 16 * t + 8 * (mi >> 1) + mk;
        stmatrix_x4_trans(g_addr + mh * half_bytes + c * 128 + ((g_chunk ^ (c & 7)) << 4), r);
      }
    }
  };
  long long n = 0, mine = 0;
  mbar_wait(w_full, 0);
  for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++n) {
    if (n % kGroupsHB != g) continue;
    const uint32_t s = static_cast<uint32_t>(n % p.stages);
    const int b = static_cast<int>(tile / p.tiles_per_b);
    const long long p0 = (tile % p.tiles_per_b) * 128;
    const long long pos = p0 + my_row;
    float dl;
    if constexpr (kPad) {
      const long long o = pos < p.S ? pad_row_to_offset(pm, static_cast<uint32_t>(b * p.S + pos)) : -1;
      dl = o >= 0 ? p.dout[o] : 0.f;
    } else {
      dl = pos < p.S ? p.dout[row_to_offset(p.map, static_cast<uint32_t>(b * p.S + pos))] : 0.f;
    }
    float dk[4];                                     // dout of the thread's rows frag_row(q, lane, k)
    auto take_dout = [&]() {
      acc_gb4 += dl;
      if constexpr (!kWideHB<KR>) s_ds[128 * g + my_row] = dl * scale;   // the lanes' rows cover the tile once
#pragma unroll
      for (int k = 0; k < 4; ++k) dk[k] = __shfl_sync(0xffffffffu, dl, (lane & ~3) | k);
    };
    // KR <= 48 first uses dout after the first MMA1 half, so the load's latency hides behind the ring wait and MMA1
    if constexpr (kWideHB<KR>) take_dout();
    mbar_wait(&a_full[s], (n / p.stages) & 1);
    const uint32_t abase = smem_u32(s_a + s * tile_bytes);
    float acc2[KR];                                  // dh0 [pos, c]: 128 x KR (KR <= 48)
    if constexpr (kWideHB<KR>) {
      // MMA1 in four 32-unit quarters (the registers of a 64-unit half are taken by D3); P goes to shared memory only
#pragma unroll
      for (int hq = 0; hq < 4; ++hq) {               // hidden units [32 hq, 32 hq + 32)
        float acc[32];
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < KR / 16; ++ks) {
          const uint32_t w_k = KR > 64 ? (ks >> 2) * 16384 + (ks & 3) * 32 : ks * 32;
          wg_mma128<false, 1, 0>(acc, 32, gdesc_mn128(abase + ks * 2048, half_bytes, 1024), half_bytes,
                                 gdesc_k128(w3_addr + hq * 4096 + w_k), ks > 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        acc_fence(acc);
        const int hh = hq >> 1;
#pragma unroll
        for (int mh = 0; mh < 2; ++mh) {
#pragma unroll
          for (int kq = 0; kq < 2; ++kq) {
            const int ks = 2 * (hq & 1) + kq;            // k16 step inside the 64-unit half hh (epi A as below)
            uint32_t pr[4];
            afrag_from_acc(acc + 16 * mh, kq, pr, [&](float lo, float hi, int i) {
              const int j = 2 * ks + (i >> 1);
              const GeluH2 vg = gelu_vg_h2(h2_from_f32(lo, hi));
              const float2 a = __half22float2(vg.value);
              const float d = dk[2 * mh + (i & 1)];
              wsum_add(16 * hh + 2 * j, d, a.x);
              wsum_add(16 * hh + 2 * j + 1, d, a.y);
              return h2_bits(__hmul2(vg.grad, h2_of_bits(s_w4h[32 * hh + 4 * j + cq])));
            });
            const uint32_t row = 64 * mh + p_row, chunk = 2 * ks + (mi >> 1);
            stmatrix_x4(p_addr + hh * 16384 + row * 128 + ((chunk ^ (row & 7)) << 4), pr);
          }
        }
      }
    } else {
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
        if (hh == 0) take_dout();
        // ---- epi A: P = W4 gelu'(pre) into the A registers and the smem tile; dW4 += dout gelu(pre)
#pragma unroll
        for (int mh = 0; mh < 2; ++mh) {
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) {
            afrag_from_acc(acc + 32 * mh, ks, pa[mh][ks], [&](float lo, float hi, int i) {
              const int j = 2 * ks + (i >> 1);
              const GeluH2 vg = gelu_vg_h2(h2_from_f32(lo, hi));
              const float2 a = __half22float2(vg.value);
              const float d = dk[2 * mh + (i & 1)];
              wsum_add(16 * hh + 2 * j, d, a.x);
              wsum_add(16 * hh + 2 * j + 1, d, a.y);
              return h2_bits(__hmul2(vg.grad, h2_of_bits(s_w4h[32 * hh + 4 * j + cq])));
            });
            const uint32_t row = 64 * mh + p_row, chunk = 2 * ks + (mi >> 1);
            stmatrix_x4(p_addr + hh * 16384 + row * 128 + ((chunk ^ (row & 7)) << 4), pa[mh][ks]);
          }
        }
        if (hh == 0) {                                 // MMA2 over the first half, before the second half's MMA1
          wgmma_fence();
          mma2(acc2, 0);
          wgmma_commit();
          wgmma_wait<0>();
        }
      }
    }
    if constexpr (kWideHB<KR>) {
      if (leader) tma_store_wait_read();             // hs doubles as the g staging: the previous g stores must be out
      asm volatile("bar.sync %0, 128;" ::"r"(barid) : "memory");
      const uint8_t* src = s_a + s * tile_bytes;     // hs as below, one row per iteration
#pragma unroll 1
      for (int k = 0; k < 4; ++k) {
        const int row = frag_row(q, lane, k);
        const float ds = dk[k] * scale;
        const uint32_t colo = (row >> 6) * half_bytes + ((row & 7) << 1);
        const uint32_t ch = (row & 63) >> 3;
#pragma unroll
        for (int cc = 0; cc < KR / 4; ++cc) {
          const int c = 4 * cc + cq;
          const uint32_t off = colo + c * 128 + ((ch ^ (c & 7)) << 4);
          if (c < p.C) {
            const uint16_t hv = *reinterpret_cast<const uint16_t*>(src + off);
            *reinterpret_cast<__half*>(hsbuf + off) = __float2half_rn(__uint_as_float(static_cast<uint32_t>(hv) << 16) * ds);
          } else if (c == p.C) {
            *reinterpret_cast<__half*>(hsbuf + off) = __float2half_rn(ds);
          }
        }
      }

      fence_proxy_async_smem();
      asm volatile("bar.sync %0, 128;" ::"r"(barid) : "memory");
      if (leader) mbar_arrive(&a_empty[s]);          // the h tile has been read for the last time
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
        const uint32_t kb = ks >> 2, kk = ks & 3;
        wg_mma128<true, 1, 0>(d3, KR, gdesc_mn128(p_addr + ks * 2048, 16384, 1024), 16384,
                              gdesc_k128(hs_addr + kb * half_bytes + kk * 32), (mine > 0 || ks > 0) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();                               // MMA3 has read hs before g is staged over it
      acc_fence(d3);
      ++mine;
      constexpr int kG0 = KR > 64 ? 48 : 32;         // channel columns of the first MMA2 group
      mma2_group(std::integral_constant<int, 0>{}, std::integral_constant<int, kG0>{}, dk);
      mma2_group(std::integral_constant<int, kG0>{}, std::integral_constant<int, KR - kG0>{}, dk);
      fence_proxy_async_smem();
      asm volatile("bar.sync %0, 128;" ::"r"(barid) : "memory");
      if (leader) {
        const int row0 = b * p.C;
        tma_store_2d(&tmG, gbuf, static_cast<int32_t>(p0), row0);
        if (p0 + 64 < p.S) tma_store_2d(&tmG, gbuf + half_bytes, static_cast<int32_t>(p0 + 64), row0);
        tma_store_commit();
      }
      continue;
    }
    {
      // ---- hs: scaled fp16 copy of rows 0..C of the h tile, one 16-byte chunk (8 positions of one channel) per
      // thread and step; row C = the scaled gradient itself.  Chunk pc of row r holds positions 8 (pc ^ (r % 8)).. of
      // its 64-position half (the 128-byte swizzle); rows above C stay zero from the start.
      asm volatile("bar.sync %0, 128;" ::"r"(barid) : "memory");      // s_ds of this tile complete
      const uint8_t* src = s_a + s * tile_bytes;
      const float* ds_t = s_ds + 128 * g;
      const int nh = (p.C + 1) * 8;                  // chunks per half
      for (int i = threadIdx.x & 127; i < 2 * nh; i += 128) {
        const int mh = i >= nh ? 1 : 0, r = (i - mh * nh) >> 3, pc = i & 7;
        const uint32_t off = mh * half_bytes + r * 128 + pc * 16;
        const float* d = ds_t + 64 * mh + 8 * (pc ^ (r & 7));
        const float4 d0 = *reinterpret_cast<const float4*>(d), d1 = *reinterpret_cast<const float4*>(d + 4);
        const float dv[8] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
        uint32_t o[4];
        if (r < p.C) {
          const uint4 v = *reinterpret_cast<const uint4*>(src + off);
          const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int e = 0; e < 4; ++e)
            o[e] = h2_bits(__floats2half2_rn(__uint_as_float(w[e] << 16) * dv[2 * e],
                                             __uint_as_float(w[e] & 0xffff0000u) * dv[2 * e + 1]));
        } else {
#pragma unroll
          for (int e = 0; e < 4; ++e) o[e] = h2_bits(__floats2half2_rn(dv[2 * e], dv[2 * e + 1]));
        }
        *reinterpret_cast<uint4*>(hsbuf + off) = make_uint4(o[0], o[1], o[2], o[3]);
      }
    }
    if (leader) tma_store_wait_read();               // the previous tile's g staging is free after the barrier
    fence_proxy_async_smem();
    asm volatile("bar.sync %0, 128;" ::"r"(barid) : "memory");
    wgmma_fence();
    mma2(acc2, 1);
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {                 // K = positions; A = P read MN-major (hid contiguous)
      const uint32_t kb = ks >> 2, kk = ks & 3;
      wg_mma128<true, 1, 0>(d3, KR, gdesc_mn128(p_addr + ks * 2048, 16384, 1024), 16384,
                            gdesc_k128(hs_addr + kb * half_bytes + kk * 32), (mine > 0 || ks > 0) ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(acc2);
    acc_fence(d3);
    ++mine;
    if (leader) mbar_arrive(&a_empty[s]);
    // ---- epi B: g[c, pos] = dout * dh0[pos, c], staged as bf16 [c][64 pos] x 2 (the TMA box layout)
#pragma unroll
    for (int mh = 0; mh < 2; ++mh) {
#pragma unroll
      for (int t = 0; t < KR / 16; ++t) {
        uint32_t r[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float* a = acc2 + (KR / 2) * mh + 4 * (2 * t + (i >> 1)) + 2 * (i & 1);
          const float d = dk[2 * mh + (i & 1)];
          r[i] = pack_bf16x2(d * a[0], d * a[1]);
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
  acc_gb4 += __shfl_xor_sync(0xffffffffu, acc_gb4, 16);
  acc_gb4 += __shfl_xor_sync(0xffffffffu, acc_gb4, 8);
  acc_gb4 += __shfl_xor_sync(0xffffffffu, acc_gb4, 4);
  acc_gb4 += __shfl_xor_sync(0xffffffffu, acc_gb4, 2);
  acc_gb4 += __shfl_xor_sync(0xffffffffu, acc_gb4, 1);
  if (lane == 0) atomicAdd(s_gb4, acc_gb4);
#pragma unroll
  for (int i = 0; i < 32; ++i) {                     // lanes with equal l%4 hold the same hidden units
    float v = kWsumSmem<KR> || i < kWsumSmemW<KR> ? my_wsum[i * 128 * kGroupsHB] : wsum[i];
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 8);
    v += __shfl_xor_sync(0xffffffffu, v, 16);
    if (lane < 4) atomicAdd(&s_gw4[64 * (i >> 4) + 8 * ((i & 15) >> 1) + 2 * cq + (i & 1)], v);
  }
  if (mine > 0) {
    // fragment of the 128 x KR accumulator: register (KR/2)h + 4j + e holds hidden unit 64h + 16q + lane/4 + 8(e/2),
    // column 8j + 2(lane%4) + e%2
    const float inv = 1.0f / scale;
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < KR / 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int hid = 64 * h + 16 * q + (lane >> 2) + 8 * (e >> 1), c = 8 * j + 2 * (lane & 3) + (e & 1);
          const float v = d3[(KR / 2) * h + 4 * j + e] * inv;
          {
            if (c < p.C) atomicAdd(p.gW3 + hid * p.C + c, v);
            else if (c == p.C) atomicAdd(p.gb3 + hid, v);
          }
        }
  }
  asm volatile("bar.sync 3, %0;" ::"n"(128 * kGroupsHB) : "memory");
  if (num_tiles > blockIdx.x && threadIdx.x < kHidH) {
    atomicAdd(p.gW4 + threadIdx.x, s_gw4[threadIdx.x]);
    if (threadIdx.x == 0) atomicAdd(p.gb4, s_gb4[0]);
  }
}

template <int KR>
__global__ void __launch_bounds__(kThreadsHB, 1)
head_bwd2_kernel(const __grid_constant__ CUtensorMap tmH, const __grid_constant__ CUtensorMap tmW3,
                 const __grid_constant__ CUtensorMap tmW3T, const __grid_constant__ CUtensorMap tmG,
                 const HeadBwdParams p) {
  head_bwd2_body<KR, false>(tmH, tmW3, tmW3T, tmG, p, PadRowMap{});
}

template <int KR>
__global__ void __launch_bounds__(kThreadsHB, 1)
head_bwd2_pad_kernel(const __grid_constant__ CUtensorMap tmH, const __grid_constant__ CUtensorMap tmW3,
                     const __grid_constant__ CUtensorMap tmW3T, const __grid_constant__ CUtensorMap tmG,
                     const HeadBwdParams p, const __grid_constant__ PadRowMap pm) {
  head_bwd2_body<KR, true>(tmH, tmW3, tmW3T, tmG, p, pm);
}

}  // namespace

// h: bf16 [B*C, S] channel-major; W3aug: bf16 [128, 64] with column C = b3 ([128, 128] when C = 64); w4b4: fp32 [129]; out: fp32, addressed
// through the row digits (row = b*S + position).  lim (may be null): per-digit interior bounds of a zero-padded h
// (up to 5 digits); rows beyond them are not stored.
const char* head_fwd(const void* h, const void* W3aug, const float* w4b4, float* out, int B, int C, long long S,
                     int nrl, const int* R, const long long* SR, const int* lim, int num_sms, cudaStream_t stream) {
  if (C < 1 || C > 64) return "head_fwd: 1 <= C <= 64";
  if (S % 8 || S > (1ll << 31) - 256 || static_cast<long long>(B) * S > (1ll << 31) - 256) return "head_fwd: bad slab size";
  HeadFwdParams p{};
  p.B = B; p.C = C; p.KR = (C + 1 + 15) / 16 * 16; p.S = S; p.tiles_per_b = (S + 127) / 128;
  p.w4b4 = w4b4; p.out = out;
  PadRowMap pm{};
  if (lim ? set_padrowmap(&pm, nrl, R, SR, lim) : set_rowmap(&p.map, nrl, R, SR))
    return lim ? "head_fwd: 1..5 row digits, each bound within its radix" : "head_fwd: 1..4 row digits";
  CUtensorMap tmH, tmW3;
  if (make_map_2d(&tmH, h, S, static_cast<uint64_t>(B) * C, S, 64, C)) return "tensor map (h) failed";
  const int w3_cols = p.KR > 64 ? 128 : 64;
  if (make_map_2d(&tmW3, W3aug, w3_cols, 128, w3_cols, 64, 128)) return "tensor map (W3) failed";
  static bool attr[2][5] = {};
  const int kr_i = p.KR / 16 - 1, pd = lim ? 1 : 0;
  const void* fns[2][5] = {{reinterpret_cast<const void*>(head_fwd_kernel<16>),
                            reinterpret_cast<const void*>(head_fwd_kernel<32>),
                            reinterpret_cast<const void*>(head_fwd_kernel<48>),
                            reinterpret_cast<const void*>(head_fwd_kernel<64>),
                            reinterpret_cast<const void*>(head_fwd_kernel<80>)},
                           {reinterpret_cast<const void*>(head_fwd_pad_kernel<16>),
                            reinterpret_cast<const void*>(head_fwd_pad_kernel<32>),
                            reinterpret_cast<const void*>(head_fwd_pad_kernel<48>),
                            reinterpret_cast<const void*>(head_fwd_pad_kernel<64>),
                            reinterpret_cast<const void*>(head_fwd_pad_kernel<80>)}};
  const void* fn = fns[pd][kr_i];
  if (!attr[pd][kr_i]) {
    if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess)
      return "cudaFuncSetAttribute failed";
    attr[pd][kr_i] = true;
  }
  const int stages = p.KR > 48 ? kStagesHF<64> : kStagesHF<48>;
  const uint32_t smem_bytes = (p.KR > 64 ? 32768 : 16384) + stages * 2 * p.KR * 128 + 2048 + 1024;
  const long long tiles = p.tiles_per_b * B;
  const int grid = static_cast<int>(tiles < num_sms ? tiles : num_sms);
#define DFNO_HEAD_FWD(K_, ...)                                                                         \
  if (kr_i == 0) K_<16><<<grid, kThreadsHF<16>, smem_bytes, stream>>>(__VA_ARGS__);                      \
  else if (kr_i == 1) K_<32><<<grid, kThreadsHF<32>, smem_bytes, stream>>>(__VA_ARGS__);                 \
  else if (kr_i == 2) K_<48><<<grid, kThreadsHF<48>, smem_bytes, stream>>>(__VA_ARGS__);                 \
  else if (kr_i == 3) K_<64><<<grid, kThreadsHF<64>, smem_bytes, stream>>>(__VA_ARGS__);                 \
  else K_<80><<<grid, kThreadsHF<80>, smem_bytes, stream>>>(__VA_ARGS__);
  if (pd) { DFNO_HEAD_FWD(head_fwd_pad_kernel, tmH, tmW3, p, pm) } else { DFNO_HEAD_FWD(head_fwd_kernel, tmH, tmW3, p) }
#undef DFNO_HEAD_FWD
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

// W3T16: fp16 [KR, 128] (rows = input channel, zero padded); dout: fp32 public layout; amax_ws: one uint of scratch
// (receives max |dout|); g: bf16 [B*C, S]; gradients are accumulated with atomics.
const char* head_bwd2(const void* h, const void* W3aug, const void* W3T16, const float* W4, const float* dout,
                      long long n_dout, unsigned* amax_ws, void* g, float* gW3, float* gb3, float* gW4, float* gb4,
                      int B, int C, long long S, int nrl, const int* R, const long long* SR, const int* lim,
                      int num_sms, cudaStream_t stream) {
  if (C < 1 || C > 64) return "head_bwd: 1 <= C <= 64";
  if (S % 8 || S > (1ll << 31) - 256 || static_cast<long long>(B) * S > (1ll << 31) - 256) return "head_bwd: bad slab size";
  HeadBwdParams p{};
  p.B = B; p.C = C; p.KR = (C + 1 + 15) / 16 * 16; p.S = S; p.tiles_per_b = (S + 127) / 128;
  p.dout = dout; p.amax = reinterpret_cast<const float*>(amax_ws); p.W4 = W4;
  p.gW3 = gW3; p.gb3 = gb3; p.gW4 = gW4; p.gb4 = gb4;
  PadRowMap pm{};
  if (lim ? set_padrowmap(&pm, nrl, R, SR, lim) : set_rowmap(&p.map, nrl, R, SR))
    return lim ? "head_bwd: 1..5 row digits, each bound within its radix" : "head_bwd: 1..4 row digits";
  CUtensorMap tmH, tmW3, tmW3T, tmG;
  if (make_map_2d(&tmH, h, S, static_cast<uint64_t>(B) * C, S, 64, C)) return "tensor map (h) failed";
  const int w3_cols = p.KR > 64 ? 128 : 64;
  if (make_map_2d(&tmW3, W3aug, w3_cols, 128, w3_cols, 64, 128)) return "tensor map (W3) failed";
  if (make_map_2d(&tmW3T, W3T16, 128, p.KR, 128, 64, p.KR)) return "tensor map (W3T) failed";
  if (make_map_2d(&tmG, g, S, static_cast<uint64_t>(B) * C, S, 64, C)) return "tensor map (g) failed";
  static bool attr[2][5] = {};
  const int kr_i = p.KR / 16 - 1, pd = lim ? 1 : 0;
  const void* fns[2][5] = {{reinterpret_cast<const void*>(head_bwd2_kernel<16>),
                            reinterpret_cast<const void*>(head_bwd2_kernel<32>),
                            reinterpret_cast<const void*>(head_bwd2_kernel<48>),
                            reinterpret_cast<const void*>(head_bwd2_kernel<64>),
                            reinterpret_cast<const void*>(head_bwd2_kernel<80>)},
                           {reinterpret_cast<const void*>(head_bwd2_pad_kernel<16>),
                            reinterpret_cast<const void*>(head_bwd2_pad_kernel<32>),
                            reinterpret_cast<const void*>(head_bwd2_pad_kernel<48>),
                            reinterpret_cast<const void*>(head_bwd2_pad_kernel<64>),
                            reinterpret_cast<const void*>(head_bwd2_pad_kernel<80>)}};
  const void* fn = fns[pd][kr_i];
  if (!attr[pd][kr_i]) {
    if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess)
      return "cudaFuncSetAttribute failed";
    attr[pd][kr_i] = true;
  }
  if (cudaMemsetAsync(amax_ws, 0, 4, stream) != cudaSuccess) return "head_bwd: memset failed";
  absmax_kernel<<<num_sms * 4, 256, 0, stream>>>(dout, n_dout, amax_ws);
  const uint32_t tile_bytes = 2u * p.KR * 128;
  const bool wide = p.KR > 48;                                     // g staged over hs
  const uint32_t wsum_n = !wide ? (p.KR > 32 ? 32 : 0) : p.KR > 64 ? 24 : 32;   // dW4 sums in shared memory
  const uint32_t fixed = (p.KR > 64 ? 32768 : 16384) + tile_bytes + kGroupsHB * (32768 + (wide ? 1 : 2) * tile_bytes) +
                         2048 + 1024 + wsum_n * 128 * kGroupsHB * 4;
  p.stages = kMaxStagesHB;
  while (p.stages > kGroupsHB && fixed + p.stages * tile_bytes > 227 * 1024) p.stages -= kGroupsHB;
  if (fixed + p.stages * tile_bytes > 227 * 1024) return "head_bwd: tile does not fit shared memory";
  const uint32_t smem_bytes = fixed + p.stages * tile_bytes;
  const long long tiles = p.tiles_per_b * B;
  const int grid = static_cast<int>(tiles < num_sms ? tiles : num_sms);
#define DFNO_HEAD_BWD(K_, ...)                                                                         \
  if (kr_i == 0) K_<16><<<grid, kThreadsHB, smem_bytes, stream>>>(__VA_ARGS__);                          \
  else if (kr_i == 1) K_<32><<<grid, kThreadsHB, smem_bytes, stream>>>(__VA_ARGS__);                     \
  else if (kr_i == 2) K_<48><<<grid, kThreadsHB, smem_bytes, stream>>>(__VA_ARGS__);                     \
  else if (kr_i == 3) K_<64><<<grid, kThreadsHB, smem_bytes, stream>>>(__VA_ARGS__);                     \
  else K_<80><<<grid, kThreadsHB, smem_bytes, stream>>>(__VA_ARGS__);
  if (pd) { DFNO_HEAD_BWD(head_bwd2_pad_kernel, tmH, tmW3, tmW3T, tmG, p, pm) }
  else { DFNO_HEAD_BWD(head_bwd2_kernel, tmH, tmW3, tmW3T, tmG, p) }
#undef DFNO_HEAD_BWD
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

}  // namespace dfno
