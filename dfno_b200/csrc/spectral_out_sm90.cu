// spectral_out_sm90.cu -- the LAST stage of a Fourier layer fused with everything that follows it.
//
//   forward   pre[c, l, z] = sum_k U[c, l, k] F[z, k]            inverse real z-DFT  (SURVEY.md K13)
//                          + sum_i W[c, i] h[i, l, z]            bypass 1x1 conv     (K2)
//             out          = gelu(pre)                           (K14, reference dfno.py:244,285-291)
//   adjoint   g[c, l, z]   = sum_k U[c, l, k] F'[z, k] + sum_o W[o, c] dpre[o, l, z]
//
// One wgmma kernel, two chained MMAs per tile into the same register accumulator.  A tile is R = floor(128/C)
// field lines l = (x, y, t) of ALL C channels of one batch element: rows m = c*R + r, columns z.
//
//   MMA1   D[m, z]  = A1[m, k] . B1[z, k]^T     A1 = U tile, 3-D TMA box (k, R lines, C channels), K-major;
//                                               B1 = the resident DFT operator
//   MMA2   D[m, z] += A2[m, m'] . B2[m', z]     A2 = W (x) I_R  (128 x 128, built once per CTA from the fp32
//                                               weights), B2 = the h tile -- the SAME 3-D box geometry as the
//                                               output, used as an MN-major operand (z contiguous), so the
//                                               channel mixing is a contraction over the tile's own rows
//
// The epilogue thread of row m owns a whole z-line: it rounds the accumulator to bf16 (pre-activation,
// kept for the backward), evaluates the GELU in packed fp16 and hands both tiles to TMA stores through a
// swizzled staging buffer.  The activation is therefore read once (as B2) and written once per layer; the
// separate bypass+GELU pass of round 1 (4 more activation passes per block) is gone.
#include "sm90_ptx.cuh"
#include "kernels.h"
#include "tma_host.h"

namespace dfno {
namespace {

constexpr uint32_t kBlk = 16384;          // one [128 rows][64 bf16] SWIZZLE_128B block
constexpr int kMaxStagesS = 4;
constexpr int kMaxE = 2;                  // consumer warpgroups (stages a multiple of E: see bypass_sm90.cu)

struct SpecOutParams {
  int B, C, R, RC;
  long long L;              // lines per (b, c)
  long long tiles_per_b;    // ceil(L / R)
  int Z, nzt;               // row length; column tiles of up to 128 columns
  int K1, k1blocks, n_pad;  // DFT operator: reduction length, 64-wide K blocks, rows in memory
  int transpose_w;
  const float* W;           // [C, C] fp32
  int stages, E;
  uint32_t stage_bytes, zbt;
};

template <bool kGelu, bool kPre>
__global__ void __launch_bounds__(128 * kMaxE + 32, 1)
spectral_out_kernel(const __grid_constant__ CUtensorMap tmU, const __grid_constant__ CUtensorMap tmH,
                    const __grid_constant__ CUtensorMap tmB1, const __grid_constant__ CUtensorMap tmP,
                    const __grid_constant__ CUtensorMap tmO, const SpecOutParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* s_b1 = smem;
  uint8_t* s_a2 = s_b1 + static_cast<uint32_t>(p.k1blocks) * p.n_pad * 128;
  uint8_t* s_ring = s_a2 + 2 * kBlk;
  uint8_t* s_stage = s_ring + p.stages * p.stage_bytes;
  float* s_scratch = reinterpret_cast<float*>(s_stage + p.E * p.zbt * kBlk);
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_scratch + 4 * p.E * kRowScratchFloats);
  uint64_t* full = bars;              // [4] TMA -> consumer
  uint64_t* empty = bars + 4;         // [4] consumer -> TMA
  uint64_t* bfull = bars + 8;

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const long long num_tiles = p.tiles_per_b * p.B * p.nzt;

  // rows >= R*C of every operand block are never written by TMA: zero them once; build A2 = W (x) I_R
  {
    uint4* z0 = reinterpret_cast<uint4*>(s_a2);
    const uint32_t nz = (2 * kBlk + p.stages * p.stage_bytes) / 16;
    for (uint32_t i = threadIdx.x; i < nz; i += blockDim.x) z0[i] = make_uint4(0, 0, 0, 0);
  }
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmU); tma_prefetch_desc(&tmH); tma_prefetch_desc(&tmB1);
    tma_prefetch_desc(&tmP); tma_prefetch_desc(&tmO);
    for (int s = 0; s < p.stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 1); }
    mbar_init(bfull, 1);
    fence_barrier_init();
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < p.C * p.C * p.R; idx += blockDim.x) {
    const int a = idx / (p.C * p.R);                  // output channel (row block)
    const int rem = idx - a * (p.C * p.R);
    const int b = rem / p.R, r = rem - b * p.R;       // input channel (column block), line inside the tile
    const float w = p.transpose_w ? p.W[b * p.C + a] : p.W[a * p.C + b];
    const int m = a * p.R + r, k = b * p.R + r;
    const uint32_t off = (k >> 6) * kBlk + m * 128 + (((((k & 63) >> 3) ^ (m & 7)) << 4) | ((k & 7) << 1));
    *reinterpret_cast<__nv_bfloat16*>(s_a2 + off) = __float2bfloat16(w);
  }
  fence_proxy_async_smem();
  __syncthreads();

  if (warp == 4 * p.E) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      mbar_arrive_expect_tx(bfull, static_cast<uint32_t>(p.k1blocks) * p.n_pad * 128);
      for (int kb = 0; kb < p.k1blocks; ++kb) tma_load_2d(s_b1 + kb * p.n_pad * 128, &tmB1, bfull, kb * 64, 0);
      uint32_t s = 0, ph = 0;
      for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int zt = static_cast<int>(tile % p.nzt);
        const long long lt = (tile / p.nzt) % p.tiles_per_b;
        const int b = static_cast<int>(tile / (p.nzt * p.tiles_per_b));
        const int ncols = min(128, p.Z - zt * 128);
        const int zbn = (ncols + 63) >> 6;
        mbar_wait(&empty[s], ph ^ 1);
        mbar_arrive_expect_tx(&full[s], static_cast<uint32_t>(p.k1blocks + zbn) * p.RC * 128);
        uint8_t* dst = s_ring + s * p.stage_bytes;
        const int l0 = static_cast<int>(lt * p.R);
        for (int kb = 0; kb < p.k1blocks; ++kb) tma_load_3d(dst + kb * kBlk, &tmU, &full[s], kb * 64, l0, b * p.C);
        for (int zb = 0; zb < zbn; ++zb)
          tma_load_3d(dst + (p.k1blocks + zb) * kBlk, &tmH, &full[s], zt * 128 + zb * 64, l0, b * p.C);
        if (++s == static_cast<uint32_t>(p.stages)) { s = 0; ph ^= 1; }
      }
    }
    return;
  }

  // ===================== consumer warpgroups: both MMAs, then the epilogue (one thread per row (c, r)) =========
  const int q = warp & 3, g = warp >> 2;
  const int m = wg_row128(q, lane);
  const bool t0 = q == 0 && lane == 0;
  uint8_t* stg = s_stage + g * p.zbt * kBlk;
  uint8_t* myrow = stg + m * 128;
  float* scratch = s_scratch + warp * kRowScratchFloats;
  const uint32_t sw = m & 7;
  const uint32_t barid = 1 + g;
  const int k1steps = (p.K1 + 15) >> 4;
  const int k2steps = (p.RC + 15) >> 4;
  const uint32_t b1_addr = smem_u32(s_b1), a2_addr = smem_u32(s_a2);
  mbar_wait(bfull, 0);
  float acc[128];
  long long n = 0;
  for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++n) {
    if (n % p.E != g) continue;
    const uint32_t s = static_cast<uint32_t>(n % p.stages);
    const int zt = static_cast<int>(tile % p.nzt);
    const long long lt = (tile / p.nzt) % p.tiles_per_b;
    const int b = static_cast<int>(tile / (p.nzt * p.tiles_per_b));
    const int ncols = min(128, p.Z - zt * 128);
    const int ntp = (ncols + 15) & ~15;
    const int zbn = (ncols + 63) >> 6;
    const int l0 = static_cast<int>(lt * p.R);
    mbar_wait(&full[s], (n / p.stages) & 1);
    {
      //   MMA1   D  = U tile . F^T          (both K-major)
      //   MMA2   D += (W (x) I_R) . h tile   (B MN-major: z contiguous, atoms every kBlk bytes along z)
      const uint32_t a1 = smem_u32(s_ring + s * p.stage_bytes);
      const uint32_t b2 = a1 + p.k1blocks * kBlk;
      const uint32_t b1 = b1_addr + zt * 128 * 128;
      wgmma_fence();
      for (int ks = 0; ks < k1steps; ++ks) {
        const uint32_t kb = ks >> 2, kk = ks & 3;
        wg_mma128<false, 0, 0>(acc, ntp, gdesc_k128(a1 + kb * kBlk + kk * 32), 8192,
                               gdesc_k128(b1 + kb * (p.n_pad * 128) + kk * 32), ks > 0 ? 1u : 0u);
      }
      for (int ks = 0; ks < k2steps; ++ks) {       // K = the tile's own rows (c, r): 16 rows per instruction
        const uint32_t kb = ks >> 2, kk = ks & 3;
        wg_mma128<false, 0, 1>(acc, ntp, gdesc_k128(a2_addr + kb * kBlk + kk * 32), 8192,
                               gdesc_mn128(b2 + ks * 2048, kBlk, 1024), 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(acc);
      if (t0) mbar_arrive(&empty[s]);                  // the ring stage may be refilled
    }
    if (t0) tma_store_wait_read();                     // the previous tile's stores have left the staging buffer
    asm volatile("bar.sync %0, 128;" ::"r"(barid) : "memory");
    // accumulator -> bf16 (the pre-activation, or the GELU of it when `act`) -> swizzled staging rows
    auto stage_rows = [&](bool act) {
#pragma unroll
      for (int ch = 0; ch < 8; ++ch) {
        const int c0 = ch * 16;
        if (c0 < ncols) {
          uint32_t v[16], pk[8];
          wg_row16<2>(acc, c0, scratch, v);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float x0 = __uint_as_float(v[2 * i]), x1 = __uint_as_float(v[2 * i + 1]);
            pk[i] = act ? h2_to_bf16x2(gelu_h2(h2_from_f32(x0, x1))) : pack_bf16x2(x0, x1);
          }
          uint8_t* rowp = myrow + (c0 >> 6) * kBlk;
          const uint32_t j0 = (c0 & 63) >> 3;
          *reinterpret_cast<uint4*>(rowp + ((j0 ^ sw) << 4)) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
          *reinterpret_cast<uint4*>(rowp + (((j0 + 1) ^ sw) << 4)) = make_uint4(pk[4], pk[5], pk[6], pk[7]);
        }
      }
      fence_proxy_async_smem();
      asm volatile("bar.sync %0, 128;" ::"r"(barid) : "memory");
    };
    stage_rows(kGelu && !kPre);
    if (t0) {
      const CUtensorMap* mp = kPre ? &tmP : &tmO;
      for (int zb = 0; zb < zbn; ++zb) tma_store_3d(mp, stg + zb * kBlk, zt * 128 + zb * 64, l0, b * p.C);
      tma_store_commit();
    }
    if (kPre) {                                      // the GELU of the same accumulator, after the pre store left
      if (t0) tma_store_wait_read();
      asm volatile("bar.sync %0, 128;" ::"r"(barid) : "memory");
      stage_rows(true);
      if (t0) {
        for (int zb = 0; zb < zbn; ++zb) tma_store_3d(&tmO, stg + zb * kBlk, zt * 128 + zb * 64, l0, b * p.C);
        tma_store_commit();
      }
    }
  }
  if (t0) tma_store_wait_all();
}

// ---------------------------------------------------------------------------------------------------------------
// Adjoint with the pointwise backward of the neighbouring blocks folded in (block k of the backward, see the
// launcher spectral_out_adj below):
//
//   g            = sum_k U F'[z, k] + W^T dpre_k          (as the plain adjoint, rounded to bf16)
//   kDpre        dpre_{k-1} = g * gelu'(pre_{k-1})         (written over pre_{k-1}; g itself is not stored)
//   kDw          dW_k      += sum_{l, z} dpre_k h_k^T      (the bypass weight gradient of block k)
//
// Tiles are 64 columns (one swizzle block) of R lines x C channels, so every operand is one 16 KB box and a stage is
// {U (k1blocks boxes), dpre_k, pre_{k-1} (kDpre), h_k (kDw)}.  The owner warpgroup of a tile (tiles alternate) runs
// MMA1 + MMA2 into an m128 x n64 accumulator and the epilogue directly on its fragments: each thread reads and writes
// 4-byte pairs of the swizzled tile (conflict-free), dpre_{k-1} in place over the pre slot (or g over the first U
// block), from where the TMA store reads it.  The weight gradient D[(o, r), (i, r')] = dpre_k . h_k^T (both K-major
// over z, as in dpre_dw_sm90.cu) is split by rows: warpgroup g accumulates rows 64g .. 64g + 63 of D for EVERY tile,
// so a stage is released by both warpgroups (empty count 2) and each keeps 64 + 64 accumulator registers.  With
// kDpre the other warpgroup also evaluates gelu'(pre_{k-1}) in place over the pre slot while the owner runs its MMAs
// (handed over through named barrier 3), so the owner's epilogue only rounds and multiplies.  Every consumer passes
// every stage, so the ring depth is free of E (3 stages of 48 KB for the top-block and block-0 variants, 2 of 64 KB
// for the middle one at K1 <= 64, Z <= 128).
// ---------------------------------------------------------------------------------------------------------------
constexpr int kAdjE = 2;

template <bool kDpre, bool kDw>
__global__ void __launch_bounds__(128 * kAdjE + 32, 1)
spectral_out_adj_kernel(const __grid_constant__ CUtensorMap tmU, const __grid_constant__ CUtensorMap tmD,
                        const __grid_constant__ CUtensorMap tmB1, const __grid_constant__ CUtensorMap tmO,
                        const __grid_constant__ CUtensorMap tmHw, const SpecOutParams p, float* dW) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* s_b1 = smem;
  uint8_t* s_a2 = s_b1 + static_cast<uint32_t>(p.k1blocks) * p.n_pad * 128;
  uint8_t* s_ring = s_a2 + 2 * kBlk;
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_ring + p.stages * p.stage_bytes);
  uint64_t* full = bars;              // [4] TMA -> consumers
  uint64_t* empty = bars + 4;         // [4] consumers -> TMA
  uint64_t* bfull = bars + 8;
  // stage slots: U blocks, then dpre_k, pre_{k-1}, h_k
  const uint32_t o_d = p.k1blocks * kBlk, o_p = o_d + kBlk, o_h = o_p + (kDpre ? kBlk : 0);

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const long long num_tiles = p.tiles_per_b * p.B * p.nzt;       // nzt: 64-column blocks here

  {
    uint4* z0 = reinterpret_cast<uint4*>(s_a2);
    const uint32_t nz = (2 * kBlk + p.stages * p.stage_bytes) / 16;
    for (uint32_t i = threadIdx.x; i < nz; i += blockDim.x) z0[i] = make_uint4(0, 0, 0, 0);
  }
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmU); tma_prefetch_desc(&tmD); tma_prefetch_desc(&tmB1);
    tma_prefetch_desc(&tmO); if (kDw) tma_prefetch_desc(&tmHw);
    for (int s = 0; s < p.stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kAdjE); }
    mbar_init(bfull, 1);
    fence_barrier_init();
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < p.C * p.C * p.R; idx += blockDim.x) {   // A2 = W^T (x) I_R
    const int a = idx / (p.C * p.R);
    const int rem = idx - a * (p.C * p.R);
    const int b = rem / p.R, r = rem - b * p.R;
    const float w = p.W[b * p.C + a];
    const int m = a * p.R + r, k = b * p.R + r;
    const uint32_t off = (k >> 6) * kBlk + m * 128 + (((((k & 63) >> 3) ^ (m & 7)) << 4) | ((k & 7) << 1));
    *reinterpret_cast<__nv_bfloat16*>(s_a2 + off) = __float2bfloat16(w);
  }
  fence_proxy_async_smem();
  __syncthreads();

  if (warp == 4 * kAdjE) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      mbar_arrive_expect_tx(bfull, static_cast<uint32_t>(p.k1blocks) * p.n_pad * 128);
      for (int kb = 0; kb < p.k1blocks; ++kb) tma_load_2d(s_b1 + kb * p.n_pad * 128, &tmB1, bfull, kb * 64, 0);
      const uint32_t boxes = p.k1blocks + 1 + (kDpre ? 1 : 0) + (kDw ? 1 : 0);
      uint32_t s = 0, ph = 0;
      for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int zb = static_cast<int>(tile % p.nzt);
        const long long lt = (tile / p.nzt) % p.tiles_per_b;
        const int b = static_cast<int>(tile / (p.nzt * p.tiles_per_b));
        const int l0 = static_cast<int>(lt * p.R);
        mbar_wait(&empty[s], ph ^ 1);
        mbar_arrive_expect_tx(&full[s], boxes * p.RC * 128);
        uint8_t* dst = s_ring + s * p.stage_bytes;
        for (int kb = 0; kb < p.k1blocks; ++kb) tma_load_3d(dst + kb * kBlk, &tmU, &full[s], kb * 64, l0, b * p.C);
        tma_load_3d(dst + o_d, &tmD, &full[s], zb * 64, l0, b * p.C);
        if (kDpre) tma_load_3d(dst + o_p, &tmO, &full[s], zb * 64, l0, b * p.C);
        if (kDw) tma_load_3d(dst + o_h, &tmHw, &full[s], zb * 64, l0, b * p.C);
        if (++s == static_cast<uint32_t>(p.stages)) { s = 0; ph ^= 1; }
      }
    }
    return;
  }

  // ===================== consumer warpgroups =====================
  const int q = warp & 3, g = warp >> 2;
  const bool t0 = q == 0 && lane == 0;
  const uint32_t barid = 1 + g;
  const int k1steps = (p.K1 + 15) >> 4;
  const int k2steps = (p.RC + 15) >> 4;
  const uint32_t b1_addr = smem_u32(s_b1), a2_addr = smem_u32(s_a2);
  mbar_wait(bfull, 0);
  float acc[64];                      // D[m, z] of the tiles this warpgroup owns (m128 x n64)
  float accw[kDw ? 64 : 1];           // rows 64g .. 64g + 63 of the weight-gradient D over every tile
  long long n = 0;
  for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++n) {
    const bool own = n % kAdjE == g;
    const uint32_t s = static_cast<uint32_t>(n % p.stages);
    const int zb = static_cast<int>(tile % p.nzt);
    const long long lt = (tile / p.nzt) % p.tiles_per_b;
    const int b = static_cast<int>(tile / (p.nzt * p.tiles_per_b));
    const int ncols = min(64, p.Z - zb * 64);
    const int ntp = (ncols + 15) & ~15;
    const int l0 = static_cast<int>(lt * p.R);
    uint8_t* st = s_ring + s * p.stage_bytes;
    const uint32_t a1 = smem_u32(st);
    mbar_wait(&full[s], (n / p.stages) & 1);
    if (!own) {
      // the other warpgroup's tile: its rows of dW (kDw), and gelu'(pre_{k-1}) written in place over the pre slot as
      // fp16 pairs (kDpre), while the owner runs its MMAs -- the owner's epilogue then only multiplies
      if constexpr (kDw) {
        wgmma_fence();
        const int ksteps = ntp >> 4;
        for (int kk = 0; kk < ksteps; ++kk)
          wgmma_m64n128k16_bf16<0, 0>(accw, gdesc_k128(a1 + o_d + g * 8192 + kk * 32), gdesc_k128(a1 + o_h + kk * 32),
                                      (n > 0 || kk > 0) ? 1u : 0u);
        wgmma_commit();
      }
      if constexpr (kDpre) {
        uint8_t* pt = st + o_p;
        const int t = threadIdx.x & 127;
        for (int i0 = t; i0 < p.RC * 8; i0 += 2 * 128) {      // 16-byte chunks, element-wise: position is irrelevant
          uint4 P[2];
#pragma unroll
          for (int u = 0; u < 2; ++u)
            if (i0 + u * 128 < p.RC * 8) P[u] = *reinterpret_cast<const uint4*>(pt + (i0 + u * 128) * 16);
#pragma unroll
          for (int u = 0; u < 2; ++u)
            if (i0 + u * 128 < p.RC * 8) {
              uint4 G;
              G.x = h2_bits(gelu_vg_h2(bf16x2_to_h2(P[u].x)).grad);
              G.y = h2_bits(gelu_vg_h2(bf16x2_to_h2(P[u].y)).grad);
              G.z = h2_bits(gelu_vg_h2(bf16x2_to_h2(P[u].z)).grad);
              G.w = h2_bits(gelu_vg_h2(bf16x2_to_h2(P[u].w)).grad);
              *reinterpret_cast<uint4*>(pt + (i0 + u * 128) * 16) = G;
            }
        }
        asm volatile("bar.sync 3, %0;" ::"n"(128 * kAdjE) : "memory");   // the owner may read gelu'
      }
      if constexpr (kDw) {
        wgmma_wait<0>();
        acc_fence(accw);
      }
      if (t0) mbar_arrive(&empty[s]);
      continue;
    }
    {
      //   MMA1   D  = U tile . F'^T        (both K-major)
      //   MMA2   D += (W^T (x) I_R) . dpre_k tile   (B MN-major, z contiguous)
      //   (kDw)  D[64g + (o, r), (i, r')] += dpre_k[(o, r), z] . h_k[(i, r'), z]   (K = z; columns beyond Z zero-filled)
      wgmma_fence();
      const uint32_t b1 = b1_addr + zb * 64 * 128;
      for (int ks = 0; ks < k1steps; ++ks) {
        const uint32_t kb = ks >> 2, kk = ks & 3;
        wg_mma128<false, 0, 0>(acc, ntp, gdesc_k128(a1 + kb * kBlk + kk * 32), 8192,
                               gdesc_k128(b1 + kb * (p.n_pad * 128) + kk * 32), ks > 0 ? 1u : 0u);
      }
      for (int ks = 0; ks < k2steps; ++ks) {
        const uint32_t kb = ks >> 2, kk = ks & 3;
        wg_mma128<false, 0, 1>(acc, ntp, gdesc_k128(a2_addr + kb * kBlk + kk * 32), 8192,
                               gdesc_mn128(a1 + o_d + ks * 2048, kBlk, 1024), 1u);
      }
      if constexpr (kDw) {
        const int ksteps = ntp >> 4;
        for (int kk = 0; kk < ksteps; ++kk)
          wgmma_m64n128k16_bf16<0, 0>(accw, gdesc_k128(a1 + o_d + g * 8192 + kk * 32), gdesc_k128(a1 + o_h + kk * 32),
                                      (n > 0 || kk > 0) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(acc);
      if constexpr (kDw) acc_fence(accw);
    }
    if (kDpre)   // the other warpgroup has put gelu'(pre) over the pre slot
      asm volatile("bar.sync 3, %0;" ::"n"(128 * kAdjE) : "memory");
    else         // every warp's MMAs have read the U slot before it is overwritten with g
      asm volatile("bar.sync %0, 128;" ::"r"(barid) : "memory");
    // epilogue on the fragments: register h*32 + 4j + e holds row 64h + 16q + lane/4 + 8(e/2), columns 8j + 2(lane%4)
    // + {0, 1}; g rounds to bf16 exactly as the plain adjoint stores it, dpre = bf16(g) * gelu' as dpre_dw forms it
    {
      uint8_t* ot = st + (kDpre ? o_p : 0);
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int eh = 0; eh < 2; ++eh) {
          const int m = 64 * h + 16 * q + (lane >> 2) + 8 * eh;
          uint8_t* row = ot + m * 128 + 4 * (lane & 3);
          uint32_t gw[8];
          if (kDpre) {        // all 8 words before any store, which would otherwise order the loads behind it
#pragma unroll
            for (int j = 0; j < 8; ++j)
              gw[j] = 8 * j < ncols ? *reinterpret_cast<const uint32_t*>(row + ((j ^ (m & 7)) << 4)) : 0u;
          }
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            if (8 * j < ncols) {
              const float* a = acc + 32 * h + 4 * j + 2 * eh;
              uint32_t v = pack_bf16x2(a[0], a[1]);
              if (kDpre) {
                const float2 gr = __half22float2(h2_of_bits(gw[j]));
                const float2 gg = unpack_bf16x2(v);
                v = pack_bf16x2(gg.x * gr.x, gg.y * gr.y);
              }
              *reinterpret_cast<uint32_t*>(row + ((j ^ (m & 7)) << 4)) = v;
            }
          }
        }
    }
    fence_proxy_async_smem();
    asm volatile("bar.sync %0, 128;" ::"r"(barid) : "memory");
    if (t0) {
      tma_store_3d(&tmO, st + (kDpre ? o_p : 0), zb * 64, l0, b * p.C);
      tma_store_commit();
      tma_store_wait_read();
      mbar_arrive(&empty[s]);
    }
  }
  if (t0) tma_store_wait_all();
  if constexpr (kDw) {
    // weight gradient: the r == r' entries of D summed over r, through shared memory (the idle ring) into dW
    float* s_dw = reinterpret_cast<float*>(s_ring);
    asm volatile("bar.sync 3, %0;" ::"n"(128 * kAdjE) : "memory");
    for (int i = threadIdx.x; i < p.C * p.C; i += 128 * kAdjE) s_dw[i] = 0.f;
    asm volatile("bar.sync 3, %0;" ::"n"(128 * kAdjE) : "memory");
    if (n > 0) {
      const int m0 = 64 * g + 16 * q + (lane >> 2), k0 = 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int m = m0 + 8 * (e >> 1), k = 8 * j + k0 + (e & 1);
          if (m < p.RC && k < p.RC) {
            const int o = m / p.R, i = k / p.R;
            if (m - o * p.R == k - i * p.R) atomicAdd(&s_dw[o * p.C + i], accw[4 * j + e]);
          }
        }
    }
    asm volatile("bar.sync 3, %0;" ::"n"(128 * kAdjE) : "memory");
    if (num_tiles > blockIdx.x)
      for (int i = threadIdx.x; i < p.C * p.C; i += 128 * kAdjE) atomicAdd(dW + i, s_dw[i]);
  }
}

// Shared memory of spectral_out_adj_kernel (stages chosen from 4 down to 2), 0 when it does not fit
uint32_t spectral_out_adj_smem(int k1blocks, int n_pad, bool dpre, bool dw, int* stages_out, uint32_t* stage_bytes_out) {
  const uint32_t stage_bytes = (k1blocks + 1 + (dpre ? 1 : 0) + (dw ? 1 : 0)) * kBlk;
  const uint32_t fixed = static_cast<uint32_t>(k1blocks) * n_pad * 128 + 2 * kBlk + 1024 /*barriers*/ + 1024 /*align*/;
  for (int st = kMaxStagesS; st >= 2; --st) {
    if (fixed + st * stage_bytes <= 227u * 1024) {
      if (stages_out) *stages_out = st;
      if (stage_bytes_out) *stage_bytes_out = stage_bytes;
      return fixed + st * stage_bytes;
    }
  }
  return 0;
}

}  // namespace

// U: bf16 [B*C, L, K1]; h / pre / out: bf16 [B*C, L, Z]; Bop: padded DFT operator bf16 [n_pad >= Z, k_pad];
// W: fp32 [C, C].  gelu = 1: out = gelu(pre) (+ pre stored when save_pre); gelu = 0: out = accumulator.
const char* spectral_out(const void* U, const void* h, const void* Bop, int n_pad, int k_pad, const float* W,
                         int transpose_w, void* pre, void* out, int B, int C, long long L, int Z, int K1, int gelu,
                         int save_pre, int num_sms, cudaStream_t stream) {
  if (C < 1 || C > 64) return "spectral_out: 1 <= C <= 64";
  if (Z % 8 || Z > 256 || K1 % 8) return "spectral_out: need Z % 8 == 0, Z <= 256 and K1 % 8 == 0";
  if (k_pad % 64 || k_pad > 128 || K1 > k_pad || n_pad % 16 || n_pad < Z || n_pad > 256) return "spectral_out: bad operator padding";
  if (L > (1ll << 31) - 256 || static_cast<long long>(B) * C > (1 << 30)) return "spectral_out: tensor too large";
  SpecOutParams p{};
  p.B = B; p.C = C; p.R = 128 / C; p.RC = p.R * C; p.L = L;
  p.tiles_per_b = (L + p.R - 1) / p.R;
  p.Z = Z; p.nzt = (Z + 127) / 128;
  p.K1 = K1; p.k1blocks = k_pad / 64; p.n_pad = n_pad;
  p.transpose_w = transpose_w; p.W = W;
  p.zbt = Z > 64 ? 2 : 1;
  p.stage_bytes = (p.k1blocks + p.zbt) * kBlk;
  const uint32_t fixed = static_cast<uint32_t>(p.k1blocks) * n_pad * 128 + 2 * kBlk + 1024 /*barriers*/ + 1024 /*align*/;
  const uint32_t budget = 227 * 1024;
  auto scratch_bytes = [](int E) { return static_cast<uint32_t>(4 * E * kRowScratchFloats * 4); };
  p.E = kMaxE; p.stages = 0;
  for (int E = kMaxE; E >= 1 && !p.stages; --E)
    for (int st = kMaxStagesS; st >= 2; --st)
      if (st % E == 0 && fixed + st * p.stage_bytes + E * p.zbt * kBlk + scratch_bytes(E) <= budget) {
        p.E = E; p.stages = st; break;
      }
  if (!p.stages) return "spectral_out: tile does not fit shared memory";
  CUtensorMap tmU, tmH, tmB1, tmP, tmO;
  const uint64_t BC = static_cast<uint64_t>(B) * C;
  if (make_map_3d(&tmU, U, K1, L, BC, K1, static_cast<uint64_t>(L) * K1, 64, p.R, C)) return "tensor map (U) failed";
  if (make_map_3d(&tmH, h, Z, L, BC, Z, static_cast<uint64_t>(L) * Z, 64, p.R, C)) return "tensor map (h) failed";
  if (make_map_2d(&tmB1, Bop, k_pad, n_pad, k_pad, 64, n_pad)) return "tensor map (operator) failed";
  if (make_map_3d(&tmP, pre ? pre : out, Z, L, BC, Z, static_cast<uint64_t>(L) * Z, 64, p.R, C)) return "tensor map (pre) failed";
  if (make_map_3d(&tmO, out, Z, L, BC, Z, static_cast<uint64_t>(L) * Z, 64, p.R, C)) return "tensor map (out) failed";
  const uint32_t smem_bytes = fixed + p.stages * p.stage_bytes + p.E * p.zbt * kBlk + scratch_bytes(p.E);
  const long long tiles = p.tiles_per_b * B * p.nzt;
  const int grid = static_cast<int>(tiles < num_sms ? tiles : num_sms);
  const int threads = 128 * p.E + 32;
  const uint32_t dyn = smem_bytes;
  const bool want_pre = gelu && save_pre && pre != nullptr;
#define DFNO_SO_LAUNCH(G, P)                                                                                         \
  do {                                                                                                               \
    static bool attr = false;                                                                                        \
    if (!attr) {                                                                                                     \
      if (cudaFuncSetAttribute(spectral_out_kernel<G, P>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != \
          cudaSuccess)                                                                                               \
        return "cudaFuncSetAttribute failed";                                                                        \
      attr = true;                                                                                                   \
    }                                                                                                                \
    spectral_out_kernel<G, P><<<grid, threads, dyn, stream>>>(tmU, tmH, tmB1, tmP, tmO, p);                          \
  } while (0)
  if (gelu && want_pre) DFNO_SO_LAUNCH(true, true);
  else if (gelu) DFNO_SO_LAUNCH(true, false);
  else DFNO_SO_LAUNCH(false, false);
#undef DFNO_SO_LAUNCH
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

const char* spectral_out_adj_check(int n_pad, int k_pad, int C, int Z, int K1, int dpre, int dw) {
  if (C < 1 || C > 64) return "spectral_out_adj: 1 <= C <= 64";
  if (Z % 8 || Z > 256 || K1 % 8) return "spectral_out_adj: need Z % 8 == 0, Z <= 256 and K1 % 8 == 0";
  if (k_pad % 64 || k_pad > 128 || K1 > k_pad || n_pad % 16 || n_pad < Z || n_pad > 256)
    return "spectral_out_adj: bad operator padding";
  if (!dpre && !dw) return "spectral_out_adj: nothing to fold (use spectral_out)";
  if (!spectral_out_adj_smem(k_pad / 64, n_pad, dpre != 0, dw != 0, nullptr, nullptr))
    return "spectral_out_adj: two ring stages do not fit shared memory";
  return nullptr;
}

// Adjoint spectral_out with the neighbouring pointwise backward folded in: U: bf16 [B*C, L, K1]; dpre: bf16
// [B*C, L, Z] (the MMA2 operand); pre_prev (may be null): pre_{k-1} in, dpre_{k-1} = g * gelu'(pre_{k-1}) out, else
// g goes to `g`; h / dW (both or neither): dW[o, i] += sum dpre[o] h[i]^T.  W: fp32 [C, C], applied transposed.
const char* spectral_out_adj(const void* U, const void* dpre, const void* Bop, int n_pad, int k_pad, const float* W,
                             void* pre_prev, void* g, const void* h, float* dW, int B, int C, long long L, int Z, int K1,
                             int num_sms, cudaStream_t stream) {
  const bool kd = pre_prev != nullptr, kw = dW != nullptr;
  if (kw != (h != nullptr)) return "spectral_out_adj: h and dW go together";
  if (const char* e = spectral_out_adj_check(n_pad, k_pad, C, Z, K1, kd, kw)) return e;
  if (!kd && !g) return "spectral_out_adj: no output";
  if (L > (1ll << 31) - 256 || static_cast<long long>(B) * C > (1 << 30)) return "spectral_out_adj: tensor too large";
  SpecOutParams p{};
  p.B = B; p.C = C; p.R = 128 / C; p.RC = p.R * C; p.L = L;
  p.tiles_per_b = (L + p.R - 1) / p.R;
  p.Z = Z; p.nzt = (Z + 63) / 64;
  p.K1 = K1; p.k1blocks = k_pad / 64; p.n_pad = n_pad;
  p.transpose_w = 1; p.W = W;
  p.E = kAdjE;
  const uint32_t smem_bytes = spectral_out_adj_smem(p.k1blocks, n_pad, kd, kw, &p.stages, &p.stage_bytes);
  CUtensorMap tmU, tmD, tmB1, tmO, tmHw;
  const uint64_t BC = static_cast<uint64_t>(B) * C;
  const uint64_t LZ = static_cast<uint64_t>(L) * Z;
  if (make_map_3d(&tmU, U, K1, L, BC, K1, static_cast<uint64_t>(L) * K1, 64, p.R, C)) return "tensor map (U) failed";
  if (make_map_3d(&tmD, dpre, Z, L, BC, Z, LZ, 64, p.R, C)) return "tensor map (dpre) failed";
  if (make_map_2d(&tmB1, Bop, k_pad, n_pad, k_pad, 64, n_pad)) return "tensor map (operator) failed";
  if (make_map_3d(&tmO, kd ? pre_prev : g, Z, L, BC, Z, LZ, 64, p.R, C)) return "tensor map (out) failed";
  if (make_map_3d(&tmHw, kw ? h : dpre, Z, L, BC, Z, LZ, 64, p.R, C)) return "tensor map (h) failed";
  const long long tiles = p.tiles_per_b * B * p.nzt;
  const int grid = static_cast<int>(tiles < num_sms ? tiles : num_sms);
  const int threads = 128 * kAdjE + 32;
#define DFNO_SOA_LAUNCH(D, WW)                                                                                        \
  do {                                                                                                               \
    static bool attr = false;                                                                                        \
    if (!attr) {                                                                                                     \
      if (cudaFuncSetAttribute(spectral_out_adj_kernel<D, WW>, cudaFuncAttributeMaxDynamicSharedMemorySize,          \
                               227 * 1024) != cudaSuccess)                                                           \
        return "cudaFuncSetAttribute failed";                                                                        \
      attr = true;                                                                                                   \
    }                                                                                                                \
    spectral_out_adj_kernel<D, WW><<<grid, threads, smem_bytes, stream>>>(tmU, tmD, tmB1, tmO, tmHw, p, dW);         \
  } while (0)
  if (kd && kw) DFNO_SOA_LAUNCH(true, true);
  else if (kd) DFNO_SOA_LAUNCH(true, false);
  else DFNO_SOA_LAUNCH(false, true);
#undef DFNO_SOA_LAUNCH
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

}  // namespace dfno
