// dft_gemm_sm90.cu -- "skinny" GEMM with a resident operator matrix on wgmma / TMA (DESIGN.md §3, "The kernel").
//
//     C[M, N] = A[M, K] * B[N, K]^T        A, B bf16 (K-major), fp32 accumulation in registers
//
// Every truncated (inverse) DFT stage of SURVEY.md §2.5 is such a product: M = millions of field lines,
// K = the transformed axis, N = the retained modes -- a tiny operator B applied to a huge streamed A.  B stays
// resident in shared memory; A tiles stream through one TMA/mbarrier ring per consumer warpgroup; a consumer
// warpgroup issues the wgmma chain of a whole tile (128 rows for N <= 128, 64 rows for N <= 256) and runs its
// epilogue on the accumulator fragments: a row-major tile (optionally adding a bf16 tensor) or a scattered, transposed
// layout through a mixed-radix address table, possibly into a peer GPU's symmetric buffer (the fused pencil
// transposes).  Memory bound by construction (AI ~ N flop/byte): the tensor core only has to stay off the critical
// path.  The kernel is instantiated per padded operator width, so that each chain's wgmmas issue back to back.
#include "sm90_ptx.cuh"
#include "dft_gemm.h"
#include "tma_host.h"

namespace dfno {

static constexpr int kBlockK = 64;                 // bf16 elements per 128-byte swizzle row
static constexpr int kMaxStagesPerGroup = 4;       // A-tile ring depth of one consumer: bytes in flight per SM must
                                                   // cover HBM latency x bandwidth share (~40 KB)
static constexpr int kMaxStages = 16;              // ring stages of all consumer warpgroups (mbarrier pairs)

// Tile geometry of the instantiation for padded width n_pad: 128-row tiles (two m64 halves) up to 128 columns, 64-row
// tiles beyond; the accumulator holds kHalves * n_pad / 2 registers.  Consumer warpgroups: four while the
// accumulator takes at most 64 registers, two beyond (the register file of one CTA per SM).
constexpr int dft_halves(int n_pad) { return n_pad <= 128 ? 2 : 1; }
constexpr int dft_acc_regs(int n_pad) { return dft_halves(n_pad) * n_pad / 2; }
constexpr int dft_max_groups(int n_pad) { return dft_acc_regs(n_pad) <= 64 ? 3 : 2; }

struct SmemLayout {
  uint32_t b_bytes;       // kblocks * n_pad * 128
  uint32_t a_tile_bytes;  // bytes of one ring stage = kbs * MT * 128
  uint32_t kbs;           // 64-wide K blocks per ring stage (= kblocks unless the whole-K tile is too large)
  uint32_t spg;           // ring stages per consumer warpgroup
  uint32_t stage_off;     // byte offset of the epilogue staging area
  uint32_t stage_pitch;   // bytes per staged row (+16 B pad); 0 = direct stores
};

// EPI_BOX_STORE (dft_gemm.h, BoxGeom): per-launch state of the T1 box stores.  The other instantiations take a
// 4-byte placeholder in its place and compile to the SASS they had without it (an empty, 1-byte-aligned parameter
// made ptxas load the SmemLayout before it byte by byte).
static constexpr int kMaxBoxPeers = 8;
template <bool kBox> struct BoxArgs { int unused; };
template <> struct alignas(64) BoxArgs<true> {
  CUtensorMap m[kMaxBoxPeers];   // per destination, 4-byte words: dims {kzl mtp, Yl, bcx}, box {G mtp, ybox, 1}
  int mt, mtp, G, kzl;
  int tpb;                       // tiles per bcx: ceil(kzl / G)
  int tiles;                     // bcx * tpb
  int npeers, ybox, y0;
  uint32_t peer_bytes;           // staging bytes of one destination: ybox * G * mtp words, rounded up to 128 B
  uint32_t group_bytes;          // staging bytes of one consumer warpgroup: npeers * peer_bytes
};

// floor(n / d) for n < 2^31 with a host-computed magic number
__device__ __forceinline__ uint32_t fast_div(uint32_t n, unsigned long long magic, int shift) {
  return static_cast<uint32_t>((static_cast<unsigned long long>(n) * magic) >> shift);
}

// mixed-radix row address (shared by the scatter and head epilogues)
__device__ __forceinline__ long long row_offset(const EpiParams& e, uint32_t r, int& peer) {
  long long off = e.base_off;
  peer = 0;
#pragma unroll
  for (int l = 0; l < 4; ++l) {
    if (l < e.nrl) {
      uint32_t d = r;
      if (l != e.nrl - 1) {
        const uint32_t q = fast_div(r, e.Rm[l], e.Rs[l]);
        d = r - q * static_cast<uint32_t>(e.R[l]);
        r = q;
      }
      if (e.peer_sel == PEER_BY_ROW && l == e.peer_lvl) {
        const uint32_t pq = fast_div(d, e.Pm, e.Ps);
        peer = static_cast<int>(pq);
        d -= pq * static_cast<uint32_t>(e.peer_div);
      }
      off += static_cast<long long>(d) * e.SR[l];
    }
  }
  return off;
}

// Accumulator fragment (sm90_ptx.cuh, wgmma D layout): thread (warp q of its warpgroup, lane l) holds, in m64 half h
// and for i = 0, 1, the tile row 64h + 16q + l/4 + 8i; register h * kN/2 + 4j + 2i + {0, 1} is column 8j + 2(l%4) + {0, 1}
// of that row, i.e. the (re, im) pair 4j + l%4.
// kBox: the EPI_BOX_STORE instantiation (tiles of whole kz groups, box-stored from a staging tile); the others run
// every other epilogue on 64 * kHalves-row tiles.
template <int kN, bool kBox>
__global__ void __launch_bounds__(128 * dft_max_groups(kN) + 32, 1)
dft_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const GemmParams p, const SmemLayout L, const __grid_constant__ BoxArgs<kBox> bx) {
  constexpr int kHalves = dft_halves(kN);
  constexpr int kTileM = 64 * kHalves;
  constexpr int kAcc = dft_acc_regs(kN);
  constexpr int kHalfRegs = kN / 2;                  // registers of one m64 half
  constexpr int kRows = 2 * kHalves;                 // tile rows held by one thread
  extern __shared__ __align__(1024) uint8_t smem[];
  const int E = (static_cast<int>(blockDim.x) - 32) >> 7;     // consumer warpgroups
  const int spg = static_cast<int>(L.spg);
  uint8_t* smem_b = smem;
  uint8_t* smem_a = smem + L.b_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_a + E * spg * L.a_tile_bytes);
  uint64_t* full = bars;                              // [E * spg]   TMA -> consumer
  uint64_t* empty = bars + kMaxStages;                // [E * spg]   consumer -> TMA
  uint64_t* bfull = bars + 2 * kMaxStages;            // [1]   B resident
  long long* s_coloff = reinterpret_cast<long long*>(bars + 2 * kMaxStages + 8);   // [128] pair -> element offset
  float* s_vec = reinterpret_cast<float*>(s_coloff + 128);              // [512] EPI_HEAD vectors
  uint8_t* s_colpeer = reinterpret_cast<uint8_t*>(s_vec + 512);         // [128] pair -> peer

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);   // warp-uniform for the compiler
  const int lane = threadIdx.x & 31;
  const int kblocks = p.k_pad / kBlockK;
  const int kbs = static_cast<int>(L.kbs);
  int num_tiles;
  if constexpr (kBox) num_tiles = bx.tiles;
  else num_tiles = static_cast<int>((p.M + kTileM - 1) / kTileM);
  // first A row of a tile: G whole kz groups of one bcx (box store), else 64 * kHalves consecutive rows
  auto tile_row0 = [&](int tile) -> int {
    if constexpr (kBox) {
      const int bcx = tile / bx.tpb;
      return (bcx * bx.kzl + (tile - bcx * bx.tpb) * bx.G) * bx.mt;
    } else {
      return tile * kTileM;
    }
  };

  if constexpr (kBox) {
    // the staging tiles' pad words (kt = mt .. mtp-1) are never written by the fragments: zero them once
    uint4* z = reinterpret_cast<uint4*>(smem + L.stage_off);
    for (uint32_t i = threadIdx.x; i < E * bx.group_bytes / 16; i += blockDim.x) z[i] = make_uint4(0, 0, 0, 0);
    fence_proxy_async_smem();
  }
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if constexpr (kBox)
      for (int j = 0; j < bx.npeers; ++j) tma_prefetch_desc(&bx.m[j]);
    for (int s = 0; s < E * spg; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 1);
    }
    mbar_init(bfull, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4 * E) {
    // ===================== TMA producer (one lane) =====================
    // the n-th tile of this CTA goes to warpgroup n % E, through that warpgroup's own ring as its (n / E)-th tile
    // (each ring is filled and drained in order, so a parity wait can never pass on a phase two fills ahead)
    if (lane == 0) {
      mbar_arrive_expect_tx(bfull, L.b_bytes);
      for (int kb = 0; kb < kblocks; ++kb)
        tma_load_2d(smem_b + kb * p.n_pad * 128, &tmB, bfull, kb * kBlockK, 0);
      const uint32_t chunks = static_cast<uint32_t>(kblocks / kbs);   // ring stages per tile
      uint32_t n = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++n) {
        const uint32_t g = n % static_cast<uint32_t>(E);
        uint32_t fill = (n / static_cast<uint32_t>(E)) * chunks;      // this warpgroup's ring fills so far
        for (int kb0 = 0; kb0 < kblocks; kb0 += kbs, ++fill) {       // one ring stage per K chunk (usually the whole K)
          const uint32_t s = g * spg + fill % spg, ph = (fill / spg) & 1;
          mbar_wait(&empty[s], ph ^ 1);
          mbar_arrive_expect_tx(&full[s], L.a_tile_bytes);
          uint8_t* dst = smem_a + s * L.a_tile_bytes;
          for (int kb = 0; kb < kbs; ++kb)
            tma_load_2d(dst + kb * (kTileM * 128), &tmA, &full[s], (kb0 + kb) * kBlockK, tile_row0(tile));
        }
      }
    }
    return;
  }

  // ===================== consumer warpgroups: wgmma chain + epilogue =====================
  const int g = warp >> 2;                                     // warpgroup
  const int q = warp & 3;                                      // warp inside the warpgroup
  const int npairs = p.N >> 1;
  {
    // per-CTA lookup tables (all consumer threads; named barrier 1)
    const int et = threadIdx.x;
    const int nthr = 128 * E;
    if constexpr (kBox) {
      // pair -> word offset of its y block in the staging tile (one 128-byte aligned part per destination)
      for (int j = et; j < npairs && j < 128; j += nthr)
        s_coloff[j] = (j / bx.ybox) * (bx.peer_bytes / 4) + (j % bx.ybox) * bx.G * bx.mtp;
    } else if (p.epi.mode == EPI_PAIR_SCATTER) {
      for (int j = et; j < npairs && j < 128; j += nthr) {
        int jj = j, peer = 0;
        if (p.epi.peer_sel == PEER_BY_COL) { peer = jj / p.epi.peer_div; jj -= peer * p.epi.peer_div; }
        const int j0 = jj % p.epi.J[0], j1 = jj / p.epi.J[0];
        s_coloff[j] = j0 * p.epi.SJ[0] + j1 * p.epi.SJ[1];
        s_colpeer[j] = static_cast<uint8_t>(peer);
      }
    } else if (p.epi.mode == EPI_HEAD) {
      for (int j = et; j < p.N; j += nthr) { s_vec[j] = p.epi.v0[j]; s_vec[256 + j] = p.epi.v1[j]; }
      if (et == 0) s_vec[511] = p.epi.v1[p.N];          // output bias stored right after the weights
    }
    asm volatile("bar.sync 1, %0;" ::"r"(nthr) : "memory");
  }
  mbar_wait(bfull, 0);
  const uint32_t b_addr = smem_u32(smem_b);
  const int quad = lane & 3;
  float acc[kAcc];
  // box store: word offset of this thread's fragment rows (kz, kt) inside a y block of the staging tile; rows past
  // the tile's G kz groups are computed and dropped (-1)
  int box_roff[kRows];
  if constexpr (kBox) {
#pragma unroll
    for (int r = 0; r < kRows; ++r) {
      const int rl = 64 * (r >> 1) + 16 * q + (lane >> 2) + 8 * (r & 1);
      box_roff[r] = rl < bx.G * bx.mt ? (rl / bx.mt) * bx.mtp + rl % bx.mt : -1;
    }
  }
  uint32_t slot = 0, ph = 0;
  for (int tile = blockIdx.x + g * gridDim.x; tile < num_tiles; tile += E * gridDim.x) {
    for (int kb0 = 0; kb0 < kblocks; kb0 += kbs) {
      const uint32_t s = g * spg + slot;
      mbar_wait_warp(&full[s], ph);
      // whole K blocks: the zero K tail inside the last block (TMA zero-fills A past K) costs no memory traffic
      mma_chain<kN, kHalves>(acc, smem_u32(smem_a + s * L.a_tile_bytes), kTileM * 128, b_addr + kb0 * kN * 128,
                             kN * 128, kbs, kb0 > 0);
      if ((threadIdx.x & 127) == 0) mbar_arrive(&empty[s]);       // the ring stage may be refilled
      if (++slot == static_cast<uint32_t>(spg)) { slot = 0; ph ^= 1; }
    }
    const long long tile0 = static_cast<long long>(tile) * kTileM;
    // tile row of this thread's fragment row r = 2h + i, and its row in the warp's staging slab
    auto frag_row = [&](int r) { return 64 * (r >> 1) + 16 * q + (lane >> 2) + 8 * (r & 1); };

    if constexpr (kBox) {
      // ---- box store: fragments -> staging [y][kz][kt] (4-byte (re, im) words) -> one TMA box per destination,
      // clipped at kzl and Yl; every global run is G * mtp whole words of T1
      uint8_t* stg = smem + L.stage_off + g * bx.group_bytes;
      const bool leader = (threadIdx.x & 127) == 0;
      if (leader) tma_store_wait_read();                      // the previous tile's boxes have left the staging
      asm volatile("bar.sync %0, 128;" ::"r"(2 + g) : "memory");
#pragma unroll
      for (int j = 0; j < kN / 8; ++j) {
        const int jp = 4 * j + quad;
        if (jp >= npairs) continue;
        uint32_t* col = reinterpret_cast<uint32_t*>(stg) + s_coloff[jp];
#pragma unroll
        for (int r = 0; r < kRows; ++r) {
          if (box_roff[r] < 0) continue;
          const float* a = acc + (r >> 1) * kHalfRegs + 4 * j + 2 * (r & 1);
          col[box_roff[r]] = pack_bf16x2(a[0], a[1]);
        }
      }
      fence_proxy_async_smem();
      asm volatile("bar.sync %0, 128;" ::"r"(2 + g) : "memory");
      if (leader) {
        const int bcx = tile / bx.tpb;
        const int kz0 = (tile - bcx * bx.tpb) * bx.G;
        for (int pj = 0; pj < bx.npeers; ++pj)
          tma_store_3d(&bx.m[pj], stg + pj * bx.peer_bytes, kz0 * bx.mtp, bx.y0, bcx);
        tma_store_commit();
      }
    } else if (p.epi.mode == EPI_ROWMAJOR && L.stage_pitch != 0) {
      // ---- coalesced row-major store: fragments -> staging rows in smem (a private slab per warp holding its
      // 16 * kHalves rows: slab row 16h + r' = tile row 64h + 16q + r') -> groups of lanes write whole rows contiguously
      uint8_t* slab = smem + L.stage_off + (warp * 32) * L.stage_pitch;
      const bool st16 = !p.epi.out_fp32;                       // bf16 output: stage packed bf16
      const uint32_t slab_addr = smem_u32(slab);
#pragma unroll
      for (int h = 0; h < kHalves; ++h) {
#pragma unroll
        for (int c = 0; c < kN / 16; ++c) {
          if (16 * c >= p.N) continue;
          const float* a = acc + h * kHalfRegs + 8 * c;
          if (st16) {
            // four 8 x 8 matrices: rows 0-7 / 8-15 x columns 16c .. +7 / 16c + 8 .. +15
            const uint32_t r[4] = {pack_bf16x2(a[0], a[1]), pack_bf16x2(a[2], a[3]), pack_bf16x2(a[4], a[5]),
                                   pack_bf16x2(a[6], a[7])};
            const int mi = lane >> 3;
            const uint32_t row = 16 * h + (lane & 7) + 8 * (mi & 1);
            stmatrix_x4(slab_addr + row * L.stage_pitch + (16 * c + 8 * (mi >> 1)) * 2, r);
          } else {
#pragma unroll
            for (int jj = 0; jj < 2; ++jj)
#pragma unroll
              for (int i = 0; i < 2; ++i) {
                const int row = 16 * h + (lane >> 2) + 8 * i;
                *reinterpret_cast<float2*>(slab + row * L.stage_pitch + (16 * c + 8 * jj + 2 * quad) * 4) =
                    make_float2(a[4 * jj + 2 * i], a[4 * jj + 2 * i + 1]);
              }
          }
        }
      }
      __syncwarp();
      constexpr int kWarpRows = 16 * kHalves;                 // rows of a tile held by one warp
      const int vec_per_row = p.N >> 3;                       // 8 outputs per lane
      const int rows_per_it = 32 / vec_per_row;               // N = 128 -> 16 lanes per row, 2 rows / instr
      const int lr = lane / vec_per_row, lc = lane % vec_per_row;
      for (int rb = lr; rb < kWarpRows; rb += 4 * rows_per_it) {
        uint4 addv[4];
        bool okv[4];
        long long growv[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {                          // issue all global loads first
          const int rr = rb + u * rows_per_it;
          growv[u] = tile0 + 64 * (rr >> 4) + 16 * q + (rr & 15);
          okv[u] = rr < kWarpRows && growv[u] < p.M;
          addv[u] = make_uint4(0, 0, 0, 0);
          if (okv[u] && p.epi.add_src != nullptr)
            addv[u] = *reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(p.epi.add_src) +
                                                      growv[u] * p.epi.ld_add + lc * 8);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          if (!okv[u]) continue;
          const int rr = rb + u * rows_per_it;
          const long long grow = growv[u];
          const uint8_t* srow = slab + rr * L.stage_pitch;
          if (st16) {
            uint4 sv = *reinterpret_cast<const uint4*>(srow + lc * 16);
            if (p.epi.add_src != nullptr) {
              float2 a, b;
              a = unpack_bf16x2(sv.x); b = unpack_bf16x2(addv[u].x); sv.x = pack_bf16x2(a.x + b.x, a.y + b.y);
              a = unpack_bf16x2(sv.y); b = unpack_bf16x2(addv[u].y); sv.y = pack_bf16x2(a.x + b.x, a.y + b.y);
              a = unpack_bf16x2(sv.z); b = unpack_bf16x2(addv[u].z); sv.z = pack_bf16x2(a.x + b.x, a.y + b.y);
              a = unpack_bf16x2(sv.w); b = unpack_bf16x2(addv[u].w); sv.w = pack_bf16x2(a.x + b.x, a.y + b.y);
            }
            *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.epi.peers[0]) + grow * p.epi.ldc + lc * 8) = sv;
          } else {
            float4 f0 = reinterpret_cast<const float4*>(srow + lc * 32)[0];
            float4 f1 = reinterpret_cast<const float4*>(srow + lc * 32)[1];
            float2 t;
            t = unpack_bf16x2(addv[u].x); f0.x += t.x; f0.y += t.y;
            t = unpack_bf16x2(addv[u].y); f0.z += t.x; f0.w += t.y;
            t = unpack_bf16x2(addv[u].z); f1.x += t.x; f1.y += t.y;
            t = unpack_bf16x2(addv[u].w); f1.z += t.x; f1.w += t.y;
            float* o = reinterpret_cast<float*>(p.epi.peers[0]) + grow * p.epi.ldc + lc * 8;
            reinterpret_cast<float4*>(o)[0] = f0;
            reinterpret_cast<float4*>(o)[1] = f1;
          }
        }
      }
      __syncwarp();                                            // slab reusable by this warp's next tile
    } else if (p.epi.mode == EPI_ROWMAJOR) {
      // ---- direct row-major store: each (re, im)-adjacent register pair is two consecutive columns of one row
#pragma unroll
      for (int r = 0; r < kRows; ++r) {
        const long long row = tile0 + frag_row(r);
        if (row >= p.M) continue;
        const float* a = acc + (r >> 1) * kHalfRegs + 2 * (r & 1);
#pragma unroll
        for (int j = 0; j < kN / 8; ++j) {
          const int col = 8 * j + 2 * quad;
          if (col >= p.N) continue;
          float f0 = a[4 * j], f1 = a[4 * j + 1];
          const bool two = col + 1 < p.N;
          const bool vec = p.epi.vec_ok && two;               // 8 / 4-byte aligned: ldc, ld_add and bases are 16 B
          if (p.epi.add_src != nullptr) {
            const __nv_bfloat16* ap = reinterpret_cast<const __nv_bfloat16*>(p.epi.add_src) + row * p.epi.ld_add + col;
            if (vec) {
              const float2 t = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(ap));
              f0 += t.x; f1 += t.y;
            } else {
              f0 += __bfloat162float(ap[0]);
              if (two) f1 += __bfloat162float(ap[1]);
            }
          }
          if (p.epi.out_fp32) {
            float* o = reinterpret_cast<float*>(p.epi.peers[0]) + row * p.epi.ldc + col;
            if (vec) {
              *reinterpret_cast<float2*>(o) = make_float2(f0, f1);
            } else {
              o[0] = f0;
              if (two) o[1] = f1;
            }
          } else {
            __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.epi.peers[0]) + row * p.epi.ldc + col;
            if (vec) {
              *reinterpret_cast<uint32_t*>(o) = pack_bf16x2(f0, f1);
            } else {
              o[0] = __float2bfloat16(f0);
              if (two) o[1] = __float2bfloat16(f1);
            }
          }
        }
      }
    } else if (p.epi.mode == EPI_PAIR_SCATTER) {
      // ---- pair scatter: each register pair is one (re, im) pair, stored as one 32-bit word at a mixed-radix
      // address, possibly on a peer GPU.  A warp's store covers 8 consecutive rows x 4 pairs.
      // Byte address = row part + column part; the peer buffer's base goes with the digit that selects it.
      const bool by_col = p.epi.peer_sel == PEER_BY_COL;
      uint64_t rbase[kRows];
      bool rok[kRows];
#ifdef DFNO_IG2_PROBE
      const int probe_gap = p.epi.nrl >= 2 && p.epi.SR[0] == 2 ? static_cast<int>(p.epi.SR[1] / 2) - p.epi.R[0] : 0;
      const int probe_pad = probe_gap >= 1 && probe_gap <= 3 ? probe_gap : 0;
      bool probe_last[kRows];
#endif
#pragma unroll
      for (int r = 0; r < kRows; ++r) {
        const long long row = tile0 + frag_row(r);
        int rpeer;
        rok[r] = row < p.M;
#ifdef DFNO_IG2_PROBE
        probe_last[r] = row % p.epi.R[0] == p.epi.R[0] - 1;
#endif
        const long long roff = row_offset(p.epi, static_cast<uint32_t>(rok[r] ? row : 0), rpeer);
        rbase[r] = (by_col ? 0ull : reinterpret_cast<uint64_t>(p.epi.peers[rpeer])) + 2ull * roff;
      }
#pragma unroll
      for (int j = 0; j < kN / 8; ++j) {
        const int jp = 4 * j + quad;
        if (jp >= npairs) continue;
        const uint64_t cadd = (by_col ? reinterpret_cast<uint64_t>(p.epi.peers[s_colpeer[jp]]) : 0ull) +
                              2ull * s_coloff[jp];
#pragma unroll
        for (int r = 0; r < kRows; ++r) {
          if (!rok[r]) continue;
          const float* a = acc + (r >> 1) * kHalfRegs + 4 * j + 2 * (r & 1);
          *reinterpret_cast<uint32_t*>(rbase[r] + cadd) = pack_bf16x2(a[0], a[1]);
#ifdef DFNO_IG2_PROBE
          // timing builds only: the row of the last kt of a kt-padded T1 run (1..3 pad words between the row digit
          // of radix mt and that of pitch mtp) also writes the pad words as zeros, so that every run is written whole
          if (probe_pad > 0 && probe_last[r])
            for (int k = 1; k <= probe_pad; ++k) *reinterpret_cast<uint32_t*>(rbase[r] + cadd + 4ull * k) = 0u;
#endif
        }
      }
    } else {
      // ---- projection head: out = b4 + sum_j W4[j] * gelu(acc[j] + b3[j]); the four lanes of a quad hold the
      // columns of the same rows and are reduced with shuffles
#pragma unroll
      for (int r = 0; r < kRows; ++r) {
        const float* a = acc + (r >> 1) * kHalfRegs + 2 * (r & 1);
        float part = 0.f;
#pragma unroll
        for (int j = 0; j < kN / 8; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = 8 * j + 2 * quad + e;
            if (col < p.N) part = fmaf(s_vec[256 + col], gelu_erf(a[4 * j + e] + s_vec[col]), part);
          }
        }
        part += __shfl_xor_sync(0xffffffffu, part, 1);
        part += __shfl_xor_sync(0xffffffffu, part, 2);
        const long long row = tile0 + frag_row(r);
        if (quad == 0 && row < p.M) {
          int unused;
          reinterpret_cast<float*>(p.epi.peers[0])[row_offset(p.epi, static_cast<uint32_t>(row), unused)] =
              s_vec[511] + part;
        }
      }
    }
  }
  if constexpr (kBox) {
    // the boxes must be written, not only read out of shared memory, before the fence that publishes them
    if ((threadIdx.x & 127) == 0) {
      tma_store_wait_all();
      __threadfence_system();
    }
  } else if (p.epi.peer_sel != PEER_NONE) {
    __threadfence_system();   // publish peer stores
  }
}

// -------------------------------------------------------------------------------------------
// host side
// -------------------------------------------------------------------------------------------
static void magic_for(unsigned d, unsigned long long* magic, int* shift) {
  int s = 0;
  while ((1ull << s) < d) ++s;
  *magic = ((1ull << (31 + s)) / d) + 1;
  *shift = 31 + s;
}

// one instantiation per padded operator width (the host dispatches once per launch)
template <int kN, bool kBox>
static const char* launch(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, const SmemLayout& L,
                          const BoxArgs<kBox>& bx, int grid, int E, uint32_t smem_bytes, cudaStream_t stream) {
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(dft_gemm_kernel<kN, kBox>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) !=
        cudaSuccess)
      return "cudaFuncSetAttribute(max dynamic smem) failed";
    attr_set = true;
  }
  dft_gemm_kernel<kN, kBox><<<grid, 128 * E + 32, smem_bytes, stream>>>(tmA, tmB, p, L, bx);
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

template <bool kBox>
static const char* dispatch(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, const SmemLayout& L,
                            const BoxArgs<kBox>& bx, int grid, int E, uint32_t smem_bytes, cudaStream_t stream) {
  switch (p.n_pad) {
    case 16: return launch<16>(tmA, tmB, p, L, bx, grid, E, smem_bytes, stream);
    case 32: return launch<32>(tmA, tmB, p, L, bx, grid, E, smem_bytes, stream);
    case 48: return launch<48>(tmA, tmB, p, L, bx, grid, E, smem_bytes, stream);
    case 64: return launch<64>(tmA, tmB, p, L, bx, grid, E, smem_bytes, stream);
    case 80: return launch<80>(tmA, tmB, p, L, bx, grid, E, smem_bytes, stream);
    case 96: return launch<96>(tmA, tmB, p, L, bx, grid, E, smem_bytes, stream);
    case 112: return launch<112>(tmA, tmB, p, L, bx, grid, E, smem_bytes, stream);
    case 128: return launch<128>(tmA, tmB, p, L, bx, grid, E, smem_bytes, stream);
    case 144: return launch<144>(tmA, tmB, p, L, bx, grid, E, smem_bytes, stream);
    case 160: return launch<160>(tmA, tmB, p, L, bx, grid, E, smem_bytes, stream);
    case 176: return launch<176>(tmA, tmB, p, L, bx, grid, E, smem_bytes, stream);
    case 192: return launch<192>(tmA, tmB, p, L, bx, grid, E, smem_bytes, stream);
    case 208: return launch<208>(tmA, tmB, p, L, bx, grid, E, smem_bytes, stream);
    case 224: return launch<224>(tmA, tmB, p, L, bx, grid, E, smem_bytes, stream);
    case 240: return launch<240>(tmA, tmB, p, L, bx, grid, E, smem_bytes, stream);
    default: return launch<256>(tmA, tmB, p, L, bx, grid, E, smem_bytes, stream);
  }
}

// Box-store geometry of one launch (dft_gemm.h, BoxGeom) and its destination maps; nullptr or an error string.
static const char* box_setup(const GemmParams& p, const BoxGeom& b, uint32_t tile_m, BoxArgs<true>* bx) {
  const int npairs = p.N / 2;
  if (b.mt < 1 || b.kzl < 1 || b.KZ < b.kzl || b.Yl < 1 || b.bcx < 1 || b.y0 < 0 || b.base_off < 0)
    return "box store: bad geometry";
  if (b.bcx * b.kzl * b.mt != p.M) return "box store: M must be bcx * kzl * mt rows";
  if (b.mtp % 4 || b.mtp < b.mt) return "box store: the kt pitch must be a multiple of 4, at least mt";
  bx->mt = b.mt; bx->mtp = b.mtp; bx->kzl = b.kzl;
  bx->G = static_cast<int>(tile_m) / b.mt;
  if (bx->G < 1) return "box store: a kz group is longer than a tile";
  bx->tpb = (b.kzl + bx->G - 1) / bx->G;
  if (b.bcx * bx->tpb > (1ll << 31) - 1) return "box store: too many tiles for one launch";
  bx->tiles = static_cast<int>(b.bcx * bx->tpb);
  bx->ybox = npairs < b.Yl ? npairs : b.Yl;
  bx->npeers = npairs / bx->ybox;
  bx->y0 = b.y0;
  if (npairs % bx->ybox || bx->npeers > kMaxBoxPeers || bx->ybox > 256 || b.y0 + bx->ybox > b.Yl)
    return "box store: the pairs must be whole destinations, or lie inside one";
  bx->peer_bytes = (static_cast<uint32_t>(bx->ybox) * bx->G * b.mtp * 4 + 127) / 128 * 128;
  bx->group_bytes = bx->npeers * bx->peer_bytes;
  // the G kz groups of one (bcx, y) are one contiguous run of G * mtp words: the box's inner row
  if (bx->G * b.mtp > 256) return "box store: more than 256 words per y in a tile";
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return "cuTensorMapEncodeTiled not available";
  cuuint64_t dims[3] = {static_cast<cuuint64_t>(b.kzl) * b.mtp, static_cast<cuuint64_t>(b.Yl),
                        static_cast<cuuint64_t>(b.bcx)};
  cuuint64_t str[2] = {static_cast<cuuint64_t>(b.KZ) * b.mtp * 4, static_cast<cuuint64_t>(b.Yl) * b.KZ * b.mtp * 4};
  cuuint32_t box[3] = {static_cast<cuuint32_t>(bx->G * b.mtp), static_cast<cuuint32_t>(bx->ybox), 1};
  cuuint32_t estr[3] = {1, 1, 1};
  for (int j = 0; j < bx->npeers; ++j) {
    uint8_t* base = reinterpret_cast<uint8_t*>(p.epi.peers[j]) + 2 * b.base_off;
    if (reinterpret_cast<uintptr_t>(base) % 16) return "box store: destination must be 16B aligned";
    if (enc(&bx->m[j], CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, base, dims, str, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) !=
        CUDA_SUCCESS)
      return "cuTensorMapEncodeTiled(box store) failed";
  }
  return nullptr;
}

const char* dft_gemm_launch(const void* A, long long lda, const void* Bmat, GemmParams p, int num_sms,
                            cudaStream_t stream, const BoxGeom* box) {
  if (p.M <= 0) return nullptr;
  if (p.a_f16) return "fp16 A with a bf16 operator needs a mixed-format MMA, which sm_90 does not have";
  if (p.n_pad % 16 || p.n_pad < 16 || p.n_pad > 256) return "n_pad must be a multiple of 16 in [16,256]";
  if (p.k_pad % kBlockK || p.k_pad < kBlockK || p.k_pad > 512) return "k_pad must be a multiple of 64 in [64,512]";
  if (p.K > p.k_pad || p.N > p.n_pad) return "K/N exceed padded operator";
  if ((lda * 2) % 16) return "A row pitch must be a multiple of 16 bytes";
  if (reinterpret_cast<uintptr_t>(A) % 16 || reinterpret_cast<uintptr_t>(Bmat) % 16) return "A/B base must be 16B aligned";
  if (p.M > (1ll << 31) - 256) return "M too large for one launch";

  if (p.epi.mode == EPI_ROWMAJOR) {
    const long long esz = p.epi.out_fp32 ? 4 : 2;
    bool ok = (p.epi.ldc * esz) % 16 == 0 && reinterpret_cast<uintptr_t>(p.epi.peers[0]) % 16 == 0;
    if (p.epi.add_src)
      ok = ok && (p.epi.ld_add * 2) % 16 == 0 && reinterpret_cast<uintptr_t>(p.epi.add_src) % 16 == 0;
    p.epi.vec_ok = ok ? 1 : 0;
  }
  const int halves = p.n_pad <= 128 ? 2 : 1;
  const uint32_t tile_m = 64u * halves;
  const bool boxed = p.epi.mode == EPI_BOX_STORE;
  BoxArgs<true> bx{};
  if (boxed) {
    if (box == nullptr) return "box store without its geometry";
    if (const char* err = box_setup(p, *box, tile_m, &bx)) return err;
  }
  SmemLayout L;
  const int kblocks = p.k_pad / kBlockK;
  L.b_bytes = static_cast<uint32_t>(kblocks) * p.n_pad * 128;
  const uint32_t fixed = L.b_bytes + 4096 /*barriers + tables*/ + 1024 /*align slack*/;
  // coalesced row-major epilogue: needs N to be a multiple of 8 dividing 256 and aligned rows
  uint32_t pitch = 0;
  if (p.epi.mode == EPI_ROWMAJOR && p.epi.vec_ok && p.N % 8 == 0 && (p.N == 8 || p.N == 16 || p.N == 32 ||
      p.N == 64 || p.N == 128 || p.N == 256))
    pitch = ((p.N + 15) / 16 * 16) * (p.epi.out_fp32 ? 4 : 2) + 16;   // whole 16-column chunks are staged
  // consumer warpgroups, staging, ring depth and K chunk: as many warpgroups as the accumulator allows with >= 2
  // stages each, whole-K stages if possible, else the largest divisor of the K blocks that leaves room for two.  The
  // box store cannot run without its staging tiles (one per warpgroup).
  bool ok = false;
  int E = dft_max_groups(p.n_pad);
  for (; E >= 1 && !ok; --E) {
    for (int with_stage = (pitch || boxed) ? 1 : 0; with_stage >= (boxed ? 1 : 0) && !ok; --with_stage) {
      const uint32_t stg = with_stage ? E * (boxed ? bx.group_bytes : 4u * 32 * pitch) : 0;
      if (fixed + stg > 227 * 1024) continue;
      const uint32_t avail = 227 * 1024 - fixed - stg;
      for (int dv = kblocks; dv >= 1 && !ok; --dv) {
        if (kblocks % dv) continue;
        const uint32_t a_tile = static_cast<uint32_t>(dv) * tile_m * 128;
        uint32_t spg = avail / (E * a_tile);
        if (spg > kMaxStagesPerGroup) spg = kMaxStagesPerGroup;
        if (spg >= 2) {
          L.kbs = static_cast<uint32_t>(dv); L.a_tile_bytes = a_tile; L.spg = spg;
          L.stage_pitch = with_stage ? pitch : 0;
          L.stage_off = L.b_bytes + E * spg * a_tile + 4096;
          ok = true;
        }
      }
      if (ok) break;
    }
    if (ok) break;
  }
  if (!ok) return "operator too large for shared memory";
  for (int l = 0; l < 4; ++l) magic_for(static_cast<unsigned>(p.epi.R[l] > 0 ? p.epi.R[l] : 1), &p.epi.Rm[l], &p.epi.Rs[l]);
  magic_for(static_cast<unsigned>(p.epi.peer_div > 0 ? p.epi.peer_div : 1), &p.epi.Pm, &p.epi.Ps);
  const uint32_t smem_bytes =
      L.stage_off + (boxed ? E * bx.group_bytes : L.stage_pitch ? 4u * E * 32 * L.stage_pitch : 0);

  CUtensorMap tmA, tmB;
  // A: the K tail beyond p.K (up to k_pad) and the M tail are zero-filled by TMA
  if (make_map_2d(&tmA, A, static_cast<uint64_t>(p.K), static_cast<uint64_t>(p.M), static_cast<uint64_t>(lda),
                  kBlockK, tile_m))
    return "cuTensorMapEncodeTiled(A) failed";
  if (make_map_2d(&tmB, Bmat, static_cast<uint64_t>(p.k_pad), static_cast<uint64_t>(p.n_pad),
                  static_cast<uint64_t>(p.k_pad), kBlockK, static_cast<uint32_t>(p.n_pad)))
    return "cuTensorMapEncodeTiled(B) failed";

  const int num_tiles = boxed ? bx.tiles : static_cast<int>((p.M + tile_m - 1) / tile_m);
  const int grid = num_tiles < num_sms ? num_tiles : num_sms;
  if (boxed) return dispatch<true>(tmA, tmB, p, L, bx, grid, E, smem_bytes, stream);
  return dispatch<false>(tmA, tmB, p, L, BoxArgs<false>{}, grid, E, smem_bytes, stream);
}

}  // namespace dfno
