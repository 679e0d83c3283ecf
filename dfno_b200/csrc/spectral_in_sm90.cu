// spectral_in_sm90.cu -- the FIRST two stages of a Fourier layer in one kernel (SURVEY.md K4 + K5 + K6,
// reference dfno.py:247-259: rfft over the last axis, fft over the next, then the pencil transpose R2).
//
//   Z1[(p, t), (kz, ri)]  = sum_z  h[(p, t), z] . F1[(kz, ri), z]          truncated real z-DFT       (G1a)
//   S1[(kz, p), (kt, ri)] = sum_(t, ri') Z1[(p, t), (kz, ri')] . F2[(kt, ri), (t, ri')]   truncated t-DFT (G1b)
//
// p = one (x, y) position of one (batch, channel) row, Rp positions per tile.  The round-2 chain ran the two
// GEMMs as separate launches with Z1 (0.63 GB per pass at 128^3 x 20) written to and re-read from HBM, the
// second one with K = 2T = 40, i.e. 80-byte operand rows.  Here Z1 never leaves the SM:
//
//   MMA1   D1[m1 = p*T + t, n = 2 kz + ri]   A1 = the h tile (TMA, Rp*T lines of Z samples, K-major), B1 = F1
//   epi-1  D1 -> bf16 -> A2[m2 = kz*Rp + p, k = 2 t + ri]   (registers -> swizzled shared memory: the
//          transpose that turns MMA1's rows (t) into MMA2's reduction index)
//   MMA2   D2[m2, n2 = 2 kt + ri] = A2 . F2^T
//   epi-2  D2 -> bf16 pairs -> staging[kz][kt][y] for a run of Yc consecutive y of the same (b, c, x) row
//   flush  one 5-D TMA store per DESTINATION RANK: box (y-run, kt, kz-slab of that rank) straight into the
//          owner's S1 (or its staging block S1s) over NVLink -- the pencil transpose R2 rides on the store.
//
// Warp roles: 0 .. 4E-1 = E consumer warpgroups (MMA1, epi-1, MMA2, epi-2 of their tiles; warpgroup g owns tiles
// i = g (mod E) and the A2 buffer of that slot), 4E = TMA producer, 4E+1 = store warp.
#include <algorithm>

#include "sm90_ptx.cuh"
#include "kernels.h"
#include "tma_host.h"

namespace dfno {
namespace {

constexpr int kMaxPeersIn = 8;
// consumer warpgroups: two while the accumulator takes at most 64 registers, one beyond (two would spill)
constexpr int max_groups(int acc_regs) { return acc_regs <= 64 ? 2 : 1; }
// MMA2 widths beyond 80 (mt > 40, not an FNO truncation of T <= 64 steps) run as N = 128: the extra operator rows
// the wgmma reads are never stored
constexpr int mma2_width(int n2_pad) { return n2_pad <= 80 ? n2_pad : 128; }
constexpr int kMaxStagesIn = 6;

struct alignas(64) PeerMaps {
  CUtensorMap m[kMaxPeersIn];
};

struct SpecInParams {
  long long rows;            // (b, c, x) rows
  int X;
  int T, Rp, RT, RK;         // lines per position, positions per tile, Rp*T, Rp*KZ
  int KZ, mt, kzl, P;
  int Yc, tpc, ncy;          // positions per chunk, tiles per chunk, chunks per row
  int k1blocks, n1_pad;      // operator 1: 64-wide K blocks, padded rows (= MMA1 N)
  int k2blocks, n2_pad;      // operator 2: 64-wide K blocks (MMA2 runs all of them), padded rows (= MMA2 N)
  int stages, E;
  uint32_t blk1, stage_bytes, a2blk, a2_bytes, stg_bytes, peer_bytes;
  uint32_t smem_bytes;
  uint32_t swz;              // staging swizzle: Yc / 4 - 1 (the 16-byte chunks of a 128-byte line that are XORed)
};

__device__ __forceinline__ void tma_store_5d(const CUtensorMap* m, const void* smem_src, int32_t c0, int32_t c1,
                                             int32_t c2, int32_t c3, int32_t c4) {
  asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];\n" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
               : "memory");
}

// One dispatch per chain (never per instruction) on the tile rows; the second m64 half is skipped when the tile has
// at most 64 rows (its A rows would lie past the operand block).
template <int N, int R>
__device__ __forceinline__ void mma_kmajor(float (&acc)[R], int rows, uint32_t a, uint32_t a_blk, uint32_t b,
                                           uint32_t b_blk, int kblocks) {
  if (rows > 64) mma_chain<N, 2>(acc, a, a_blk, b, b_blk, kblocks);
  else mma_chain<N, 1>(acc, a, a_blk, b, b_blk, kblocks);
}

// Byte offset of word y of staging row `row` (rows of Yc words, one per (kz, kt)); the chunks of 16 bytes are XORed with
// the 128-byte line index as the destination map's swizzle mode (128 / 64 / 32 B for Yc = 32 / 16 / 8) does it, so
// that epi-2's stores (8 rows x 4 positions per warp) spread over the banks.  swz_mask = Yc / 4 - 1.
__device__ __forceinline__ uint32_t stg_offset(uint32_t row, uint32_t y, int Yc, uint32_t swz_mask) {
  const uint32_t b = (row * Yc + y) * 4;
  return b ^ (((b >> 7) & swz_mask) << 4);
}

// N1 / N2: the operator widths n1_pad / n2_pad (MMA1 / MMA2 N), chosen per launch; the accumulator holds the wider
template <int N1, int N2>
__global__ void __launch_bounds__(128 * max_groups(N1 > N2 ? N1 : N2) + 64, 1)
spectral_in_kernel(const __grid_constant__ CUtensorMap tmH, const __grid_constant__ CUtensorMap tmB1,
                   const __grid_constant__ CUtensorMap tmB2, const __grid_constant__ PeerMaps pm,
                   const SpecInParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* s_b1 = smem;
  uint8_t* s_b2 = s_b1 + static_cast<uint32_t>(p.k1blocks) * p.n1_pad * 128;
  uint8_t* s_ring = s_b2 + static_cast<uint32_t>(p.k2blocks) * p.n2_pad * 128;   // both operator sizes are multiples of 1024
  uint8_t* s_a2 = s_ring + p.stages * p.stage_bytes;
  uint8_t* s_stg = s_a2 + p.E * p.a2_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_stg + 2 * p.stg_bytes);
  uint64_t* full = bars;                       // [kMaxStagesIn] TMA -> consumer
  uint64_t* empty = full + kMaxStagesIn;       // [kMaxStagesIn] consumer -> TMA
  uint64_t* stg_done = empty + kMaxStagesIn;   // [2] consumers -> store warp
  uint64_t* stg_free = stg_done + 2;           // [2] store warp -> consumers
  uint64_t* bfull = stg_free + 2;

  // broadcast through a shuffle so that the compiler knows the role index is warp-uniform (uniform datapath)
  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const long long n_chunks = p.rows * p.ncy;

  // the K padding of A2 (columns 2T .. 64*k2blocks) is never written by the epilogue: zero the buffers once
  {
    uint4* z0 = reinterpret_cast<uint4*>(s_a2);
    const uint32_t nz = p.E * p.a2_bytes / 16;
    for (uint32_t i = threadIdx.x; i < nz; i += blockDim.x) z0[i] = make_uint4(0, 0, 0, 0);
  }
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmH); tma_prefetch_desc(&tmB1); tma_prefetch_desc(&tmB2);
    for (int j = 0; j < p.P; ++j) tma_prefetch_desc(&pm.m[j]);
    for (int s = 0; s < p.stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 1); }
    for (int b = 0; b < 2; ++b) { mbar_init(&stg_done[b], p.tpc); mbar_init(&stg_free[b], 1); }
    mbar_init(bfull, 1);
    fence_barrier_init();
  }
  fence_proxy_async_smem();
  __syncthreads();

  if (warp == 4 * p.E) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      mbar_arrive_expect_tx(bfull, (static_cast<uint32_t>(p.k1blocks) * p.n1_pad + static_cast<uint32_t>(p.k2blocks) * p.n2_pad) * 128);
      for (int kb = 0; kb < p.k1blocks; ++kb) tma_load_2d(s_b1 + kb * p.n1_pad * 128, &tmB1, bfull, kb * 64, 0);
      for (int kb = 0; kb < p.k2blocks; ++kb) tma_load_2d(s_b2 + kb * p.n2_pad * 128, &tmB2, bfull, kb * 64, 0);
      uint32_t s = 0, ph = 0;
      for (long long chunk = blockIdx.x; chunk < n_chunks; chunk += gridDim.x) {
        const int row = static_cast<int>(chunk / p.ncy);
        const int cy = static_cast<int>(chunk - static_cast<long long>(row) * p.ncy);
        for (int tt = 0; tt < p.tpc; ++tt) {
          const int line0 = (cy * p.Yc + tt * p.Rp) * p.T;
          mbar_wait(&empty[s], ph ^ 1);
          mbar_arrive_expect_tx(&full[s], static_cast<uint32_t>(p.k1blocks) * p.RT * 128);
          uint8_t* dst = s_ring + s * p.stage_bytes;
          for (int kb = 0; kb < p.k1blocks; ++kb) tma_load_3d(dst + kb * p.blk1, &tmH, &full[s], kb * 64, line0, row);
          if (++s == static_cast<uint32_t>(p.stages)) { s = 0; ph ^= 1; }
        }
      }
    }
  } else if (warp == 4 * p.E + 1) {
    // ===================== store warp: one TMA store per destination rank and chunk =====================
    if (lane == 0) {
      uint32_t cn = 0;
      for (long long chunk = blockIdx.x; chunk < n_chunks; chunk += gridDim.x, ++cn) {
        const int row = static_cast<int>(chunk / p.ncy);
        const int cy = static_cast<int>(chunk - static_cast<long long>(row) * p.ncy);
        const int bc = row / p.X, x = row - bc * p.X;
        const uint32_t b = cn & 1;
        mbar_wait(&stg_done[b], (cn >> 1) & 1);
        const uint8_t* src = s_stg + b * p.stg_bytes;
        for (int j = 0; j < p.P; ++j) tma_store_5d(&pm.m[j], src + j * p.peer_bytes, cy * p.Yc * 2, x, 0, 0, bc);
        tma_store_commit();
        tma_store_wait_read();
        mbar_arrive(&stg_free[b]);
      }
      tma_store_wait_all();
      __threadfence_system();
    }
  } else if (warp < 4 * p.E) {
    // ===================== consumer warpgroups: MMA1 -> epi-1 -> MMA2 -> epi-2 per tile =====================
    // warpgroup g owns tiles j = g (mod E) of this CTA and the A2 buffer of that slot; the ring stage of tile j is
    // j mod stages (stages is a multiple of E, so every stage has one consumer and a parity wait never passes on a
    // stale phase)
    const int q = warp & 3, g = warp >> 2;
    const bool elected = q == 0 && lane == 0;
    const uint32_t barid = 1 + g;
    // Both epilogues work on the wgmma fragment: this thread holds rows m = 64 h + 16 q + lane/4 + 8 s (row slot
    // i = 2 h + s), and registers acc[h R/2 + 4 j + 2 s + {0, 1}] are columns 8 j + 2 (lane % 4) + {0, 1}, i.e. the
    // (re, im) pair of mode 4 j + lane % 4 (kz in D1, kt in D2): one 32-bit store each.
    const int kc = lane & 3;
    uint8_t* a2 = s_a2 + g * p.a2_bytes;
    uint32_t act1 = 0, act2 = 0;                          // row slots inside the tile (m < RT for D1, m < RK for D2)
    int p1[4], p2[4], row2[4];
    uint32_t off1[4], c16[4], blk2[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int m = 64 * (i >> 1) + 16 * q + (lane >> 2) + 8 * (i & 1);
      // epi-1: row m = p1*T + t  ->  A2[kz*Rp + p1, 2t .. 2t+1] (K block and word inside the 16-byte chunk, the chunk)
      if (m < p.RT) act1 |= 1u << i;
      p1[i] = m / p.T;
      const uint32_t k0 = 2 * (m - p1[i] * p.T);
      off1[i] = (k0 >> 6) * p.a2blk + ((k0 & 7) >> 1) * 4;
      c16[i] = (k0 & 63) >> 3;
      // epi-2: row m = kz*Rp + p2  ->  staging block of rank kz / kzl, row (kz mod kzl)*mt + kt, word tt*Rp + p2
      if (m < p.RK) act2 |= 1u << i;
      const int kz = m / p.Rp, jr = kz / p.kzl;
      p2[i] = m - kz * p.Rp;
      blk2[i] = jr * p.peer_bytes;
      row2[i] = (kz - jr * p.kzl) * p.mt;
    }
    const uint32_t ring_addr = smem_u32(s_ring), b1_addr = smem_u32(s_b1), b2_addr = smem_u32(s_b2);
    const uint32_t a2_addr = smem_u32(a2);
    constexpr int R = N1 > N2 ? N1 : N2;
    int gi = 0;                                           // group of the current tile (tiles rotate over the groups)
    uint32_t cn = 0, s = 0, ph = 0;                       // chunk counter; ring stage and phase of the current tile
    mbar_wait(bfull, 0);
    float acc[R];
    for (long long chunk = blockIdx.x; chunk < n_chunks; chunk += gridDim.x, ++cn) {
      uint8_t* stg = s_stg + (cn & 1) * p.stg_bytes;
      for (int tt = 0; tt < p.tpc; ++tt) {
        const bool mine = gi == g;
        if (++gi == p.E) gi = 0;
        const uint32_t st = s, sph = ph;
        if (++s == static_cast<uint32_t>(p.stages)) { s = 0; ph ^= 1; }
        if (!mine) continue;
        // ---------------- MMA1: D1 = h tile . F1^T ----------------
        mbar_wait(&full[st], sph);
        mma_kmajor<N1>(acc, p.RT, ring_addr + st * p.stage_bytes, p.blk1, b1_addr, p.n1_pad * 128, p.k1blocks);
        if (elected) mbar_arrive(&empty[st]);
        // ---------------- epi-1 ----------------
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          if (!((act1 >> i) & 1)) continue;
          const float* d = acc + (i >> 1) * (R / 2) + 2 * (i & 1);
#pragma unroll
          for (int j = 0; j < N1 / 8; ++j) {
            const int kz = 4 * j + kc;
            if (kz < p.KZ) {
              const uint32_t r = static_cast<uint32_t>(kz * p.Rp + p1[i]);
              *reinterpret_cast<uint32_t*>(a2 + off1[i] + r * 128 + ((c16[i] ^ (r & 7)) << 4)) =
                  pack_bf16x2(d[4 * j], d[4 * j + 1]);
            }
          }
        }
        fence_proxy_async_smem();
        asm volatile("bar.sync %0, 128;" ::"r"(barid) : "memory");
        // ---------------- MMA2: D2 = A2 . F2^T ----------------
        mma_kmajor<N2>(acc, p.RK, a2_addr, p.a2blk, b2_addr, p.n2_pad * 128, p.k2blocks);
        // ---------------- epi-2 ----------------
        mbar_wait_warp(&stg_free[cn & 1], ((cn >> 1) & 1) ^ 1);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          if (!((act2 >> i) & 1)) continue;
          const float* d = acc + (i >> 1) * (R / 2) + 2 * (i & 1);
          uint8_t* blk = stg + blk2[i];
          const uint32_t y = static_cast<uint32_t>(tt * p.Rp + p2[i]);
#pragma unroll
          for (int j = 0; j < N2 / 8; ++j) {
            const int kt = 4 * j + kc;
            if (kt < p.mt)
              *reinterpret_cast<uint32_t*>(blk + stg_offset(row2[i] + kt, y, p.Yc, p.swz)) =
                  pack_bf16x2(d[4 * j], d[4 * j + 1]);
          }
        }
        fence_proxy_async_smem();
        asm volatile("bar.sync %0, 128;" ::"r"(barid) : "memory");
        if (elected) mbar_arrive(&stg_done[cn & 1]);
      }
    }
  }
}

template <int N1, int N2>
cudaError_t launch_spectral_in(int grid, int threads, uint32_t smem_bytes, cudaStream_t stream, const CUtensorMap& tmH,
                               const CUtensorMap& tmB1, const CUtensorMap& tmB2, const PeerMaps& pm, const SpecInParams& p) {
  static bool attr = false;
  if (!attr) {
    const cudaError_t e = cudaFuncSetAttribute(spectral_in_kernel<N1, N2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return e;
    attr = true;
  }
  spectral_in_kernel<N1, N2><<<grid, threads, smem_bytes, stream>>>(tmH, tmB1, tmB2, pm, p);
  return cudaGetLastError();
}

// one instantiation per (n1_pad, MMA2 width class): n1_pad = 16 .. 128, N2 = 16, 32, 48, 64, 80, 128
using SpecInLaunch = decltype(&launch_spectral_in<16, 16>);
#define DFNO_ROW(N1)                                                                                            \
  {&launch_spectral_in<N1, 16>, &launch_spectral_in<N1, 32>, &launch_spectral_in<N1, 48>,                      \
   &launch_spectral_in<N1, 64>, &launch_spectral_in<N1, 80>, &launch_spectral_in<N1, 128>}
constexpr SpecInLaunch kLaunch[8][6] = {DFNO_ROW(16), DFNO_ROW(32), DFNO_ROW(48), DFNO_ROW(64),
                                        DFNO_ROW(80), DFNO_ROW(96), DFNO_ROW(112), DFNO_ROW(128)};
#undef DFNO_ROW

inline uint32_t align_up_u32(uint32_t v, uint32_t a) { return (v + a - 1) / a * a; }

// Tile configuration for one problem shape (shared by the launcher and by the eligibility query).
const char* plan_spectral_in(SpecInParams& p, int n1_pad, int k1_pad, int n2_pad, int k2_pad, int P, long long dst_off,
                             const long long* dstr, int BC, int X, int Yl, int T, int Z, int KZ, int mt) {
  if (P < 1 || P > kMaxPeersIn || KZ % P) return "spectral_in: 1..8 destination ranks, KZ divisible by their number";
  if (Z % 8 || Z > 256 || k1_pad % 64 || k1_pad < Z || k1_pad > 256) return "spectral_in: need Z % 8 == 0, Z <= 256";
  if (T < 1 || T > 64 || k2_pad % 64 || k2_pad < 2 * T) return "spectral_in: need T <= 64";
  if (n1_pad % 16 || n1_pad < 2 * KZ || n1_pad > 128 || n2_pad % 16 || n2_pad < 2 * mt || n2_pad > 128)
    return "spectral_in: operator padding";
  if (KZ > 128 || mt < 1) return "spectral_in: mode counts";
  if (Yl % 4) return "spectral_in: the local y extent must be a multiple of 4 (stores are clipped in 16-byte units)";
  if (dst_off % 8 || dstr[0] % 8 || dstr[1] % 8 || dstr[2] % 8 || dstr[3] % 8)
    return "spectral_in: destination offset / strides must be multiples of 8 elements (16-byte TMA alignment)";
  p = SpecInParams{};
  p.rows = static_cast<long long>(BC) * X;
  if (p.rows > (1ll << 30)) return "spectral_in: tensor too large";
  p.X = X; p.T = T; p.KZ = KZ; p.mt = mt; p.P = P; p.kzl = KZ / P;
  p.k1blocks = k1_pad / 64; p.n1_pad = n1_pad;
  p.k2blocks = (2 * T + 63) / 64; p.n2_pad = n2_pad;
  if (p.k2blocks * 64 > k2_pad) return "spectral_in: operator 2 is narrower than its reduction";
  const uint32_t ops_bytes = static_cast<uint32_t>(p.k1blocks) * n1_pad * 128 + static_cast<uint32_t>(p.k2blocks) * n2_pad * 128;
  if ((static_cast<uint32_t>(p.k1blocks) * n1_pad * 128) % 1024 || ops_bytes % 1024) return "spectral_in: operator rows must be a multiple of 8";
  const int rmax = (128 / T) < (128 / KZ) ? (128 / T) : (128 / KZ);
  const int max_e = max_groups(n1_pad > mma2_width(n2_pad) ? n1_pad : mma2_width(n2_pad));
  bool ok = false;
  for (int min_st = 3; min_st >= 2 && !ok; --min_st)       // prefer a deep TMA ring and two epilogue groups
  for (int Rp = 4; Rp >= 1 && !ok; Rp >>= 1) {
    if (Rp > rmax) continue;
    int yc = 32;
    while (yc > 4 && yc / 2 >= Yl) yc >>= 1;                   // the smallest of {4, 8, 16, 32} covering Yl, 32 beyond
    for (; yc >= 4 && !ok; yc >>= 1) {
      if (yc % Rp) continue;
      const uint32_t peer_dense = static_cast<uint32_t>(p.kzl) * mt * yc * 4;
      if (peer_dense % 128) continue;
      // swizzled staging (yc >= 8) starts every rank's block on a 1024-byte boundary, where the swizzle pattern starts
      const uint32_t peer_swz = yc >= 8 ? align_up_u32(peer_dense, 1024) : peer_dense;
      const uint32_t blk1 = align_up_u32(static_cast<uint32_t>(Rp) * T * 128, 1024);
      const uint32_t a2blk = align_up_u32(static_cast<uint32_t>(Rp) * KZ * 128, 1024);
      for (int E = max_e; E >= 1 && !ok; --E) {
        for (int st = kMaxStagesIn; st >= 2; --st) {
          if (st % E) continue;                                  // every ring stage belongs to one warpgroup
          const uint32_t ring_end = ops_bytes + st * p.k1blocks * blk1, a2_end = ring_end + E * p.k2blocks * a2blk;
          // a wgmma reads whole m64 halves, i.e. up to 64 (128) rows from the last K block of the last ring stage
          // and A2 buffer, past the rows a tile fills: those reads have to stay inside the allocation
          const uint32_t reach = std::max(ring_end - blk1 + (Rp * T > 64 ? 128u : 64u) * 128,
                                          a2_end - a2blk + (Rp * KZ > 64 ? 128u : 64u) * 128);
          auto smem_for = [&](uint32_t stg) { return std::max(a2_end + 2 * stg + 512 /*barriers*/, reach) + 1024 /*align*/; };
          // dense (bank-conflicted) staging only where the padding of the swizzled one does not fit
          const bool swizzled = smem_for(align_up_u32(peer_swz * P, 1024)) <= 227u * 1024;
          const uint32_t peer_bytes = swizzled ? peer_swz : peer_dense;
          const uint32_t stg_bytes = align_up_u32(peer_bytes * P, 1024);
          if (smem_for(stg_bytes) <= 227u * 1024 && st >= min_st && (E >= 2 || min_st == 2)) {
            p.smem_bytes = smem_for(stg_bytes);
            p.Rp = Rp; p.Yc = yc; p.E = E; p.stages = st; p.blk1 = blk1; p.a2blk = a2blk;
            p.stage_bytes = p.k1blocks * blk1; p.a2_bytes = p.k2blocks * a2blk; p.stg_bytes = stg_bytes;
            p.peer_bytes = peer_bytes;
            p.swz = swizzled ? static_cast<uint32_t>(yc / 4 - 1) : 0u;
            ok = true;
            break;
          }
        }
      }
    }
  }
  if (!ok) return "spectral_in: no tile configuration fits shared memory";
  p.RT = p.Rp * T; p.RK = p.Rp * KZ;
  p.tpc = p.Yc / p.Rp; p.ncy = (Yl + p.Yc - 1) / p.Yc;
  return nullptr;
}

}  // namespace

// nullptr when spectral_in supports the shape (no launch): the engine asks before it drops G1a + G1b from its chain.
const char* spectral_in_check(int n1_pad, int k1_pad, int n2_pad, int k2_pad, int P, long long dst_off, const long long* dstr,
                              int BC, int X, int Yl, int T, int Z, int KZ, int mt, int* cfg) {
  SpecInParams p;
  const char* e = plan_spectral_in(p, n1_pad, k1_pad, n2_pad, k2_pad, P, dst_off, dstr, BC, X, Yl, T, Z, KZ, mt);
  if (!e && cfg) { cfg[0] = p.Rp; cfg[1] = p.Yc; cfg[2] = p.E; cfg[3] = p.stages; }
  return e;
}

// h: bf16 [rows = B*C*X, Yl, T, Z] (the engine layout of one activation).  op1: padded bf16 [n1_pad >= 2 KZ, k1_pad >= Z],
// op2: padded bf16 [n2_pad >= 2 mt, k2_pad >= 2 T] (reduction index 2 t + ri).  Destination: for rank j the bf16
// tensor at dst_ptrs[j] + dst_off viewed as [B*C, kzl, mt, X, Yl*2] with element strides dstr = {x, kt, kz, bc}
// (the y / (re, im) run is contiguous); rank j receives the modes kz in [j*kzl, (j+1)*kzl).
const char* spectral_in(const void* h, const void* op1, int n1_pad, int k1_pad, const void* op2, int n2_pad, int k2_pad,
                        const long long* dst_ptrs, int P, long long dst_off, const long long* dstr, int BC, int X,
                        int Yl, int T, int Z, int KZ, int mt, int num_sms, cudaStream_t stream) {
  SpecInParams p;
  if (const char* err = plan_spectral_in(p, n1_pad, k1_pad, n2_pad, k2_pad, P, dst_off, dstr, BC, X, Yl, T, Z, KZ, mt)) return err;
  CUtensorMap tmH, tmB1, tmB2;
  PeerMaps pm;
  if (make_map_3d(&tmH, h, Z, static_cast<uint64_t>(Yl) * T, p.rows, Z, static_cast<uint64_t>(Yl) * T * Z, 64, p.RT, 1))
    return "tensor map (h) failed";
  if (make_map_2d(&tmB1, op1, k1_pad, n1_pad, k1_pad, 64, n1_pad)) return "tensor map (operator 1) failed";
  if (make_map_2d(&tmB2, op2, k2_pad, n2_pad, k2_pad, 64, n2_pad)) return "tensor map (operator 2) failed";
  for (int j = 0; j < kMaxPeersIn; ++j) {
    const int jj = j < P ? j : 0;
    const uint64_t dims[5] = {static_cast<uint64_t>(Yl) * 2, static_cast<uint64_t>(X), static_cast<uint64_t>(mt),
                              static_cast<uint64_t>(p.kzl), static_cast<uint64_t>(BC)};
    const uint64_t str[4] = {static_cast<uint64_t>(dstr[0]), static_cast<uint64_t>(dstr[1]), static_cast<uint64_t>(dstr[2]),
                             static_cast<uint64_t>(dstr[3])};
    const uint32_t box[5] = {static_cast<uint32_t>(p.Yc) * 2, 1, static_cast<uint32_t>(mt), static_cast<uint32_t>(p.kzl), 1};
    const void* base = reinterpret_cast<const void*>(static_cast<uintptr_t>(dst_ptrs[jj]) + static_cast<uintptr_t>(dst_off) * 2);
    const CUtensorMapSwizzle swz = p.swz == 7 ? CU_TENSOR_MAP_SWIZZLE_128B : p.swz == 3 ? CU_TENSOR_MAP_SWIZZLE_64B
                                 : p.swz == 1 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE;
    if (make_map_nd(&pm.m[j], base, 5, dims, str, box, swz)) return "tensor map (destination) failed";
  }
  const long long chunks = p.rows * p.ncy;
  const int grid = static_cast<int>(chunks < num_sms ? chunks : num_sms);
  const int threads = 128 * p.E + 64;
  const int i1 = n1_pad / 16 - 1, i2 = mma2_width(n2_pad) / 16 - 1 - (n2_pad > 80 ? 2 : 0);
  const cudaError_t e = kLaunch[i1][i2](grid, threads, p.smem_bytes, stream, tmH, tmB1, tmB2, pm, p);
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

}  // namespace dfno
