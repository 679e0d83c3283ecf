// dft_gemm_sm90.cu -- "skinny" GEMM with a resident operator matrix on wgmma / TMA (DESIGN.md §3, "The kernel").
//
//     C[M, N] = A[M, K] * B[N, K]^T        A, B bf16 (K-major), fp32 accumulation in registers
//
// Every truncated (inverse) DFT stage of SURVEY.md §2.5 is such a product: M = millions of field lines,
// K = the transformed axis, N = the retained modes -- a tiny operator B applied to a huge streamed A.  B stays
// resident in shared memory; A tiles stream through one TMA/mbarrier ring per consumer warpgroup; a consumer
// warpgroup issues the wgmma chain of a whole tile (128 rows for N <= 128, 64 rows for N <= 256) and runs its
// epilogue: a row-major tile (optionally adding a bf16 tensor) or a scattered, transposed layout through a
// mixed-radix address table, possibly into a peer GPU's symmetric buffer (the fused pencil transposes).
// Memory bound by construction (AI ~ N flop/byte): the tensor core only has to stay off the critical path.
#include "sm90_ptx.cuh"
#include "dft_gemm.h"
#include "tma_host.h"

namespace dfno {

static constexpr int kBlockK = 64;                 // bf16 elements per 128-byte swizzle row
static constexpr int kMaxGroups = 2;               // consumer warpgroups (128 accumulator registers each)
static constexpr int kMaxThreads = 128 * kMaxGroups + 32;
static constexpr int kMaxStagesPerGroup = 4;       // A-tile ring depth of one consumer: bytes in flight per SM must
                                                   // cover HBM latency x bandwidth share (~40 KB)

struct SmemLayout {
  uint32_t b_bytes;       // kblocks * n_pad * 128
  uint32_t a_tile_bytes;  // bytes of one ring stage = kbs * MT * 128
  uint32_t kbs;           // 64-wide K blocks per ring stage (= kblocks unless the whole-K tile is too large)
  uint32_t spg;           // ring stages per consumer warpgroup
  uint32_t scratch_off;   // byte offset of the per-warp row-view scratch
  uint32_t stage_off;     // byte offset of the epilogue staging area
  uint32_t stage_pitch;   // bytes per staged row (+16 B pad); 0 = direct stores
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

// kHalves = 2: 128-row tiles (n_pad <= 128); 1: 64-row tiles (n_pad <= 256)
template <int kHalves>
__global__ void __launch_bounds__(kMaxThreads, 1)
dft_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const GemmParams p, const SmemLayout L) {
  constexpr int kTileM = 64 * kHalves;
  constexpr int kWarpRows = 16 * kHalves;            // rows of a tile held by one warp
  extern __shared__ __align__(1024) uint8_t smem[];
  const int E = (static_cast<int>(blockDim.x) - 32) >> 7;     // consumer warpgroups
  const int spg = static_cast<int>(L.spg);
  uint8_t* smem_b = smem;
  uint8_t* smem_a = smem + L.b_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_a + E * spg * L.a_tile_bytes);
  uint64_t* full = bars;                      // [E * spg]   TMA -> consumer
  uint64_t* empty = bars + 8;                 // [E * spg]   consumer -> TMA
  uint64_t* bfull = bars + 16;                // [1]   B resident
  long long* s_coloff = reinterpret_cast<long long*>(bars + 24);        // [128] pair -> element offset
  float* s_vec = reinterpret_cast<float*>(s_coloff + 128);              // [512] EPI_HEAD vectors
  uint8_t* s_colpeer = reinterpret_cast<uint8_t*>(s_vec + 512);         // [128] pair -> peer

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);   // warp-uniform for the compiler
  const int lane = threadIdx.x & 31;
  const int kblocks = p.k_pad / kBlockK;
  const int kbs = static_cast<int>(L.kbs);
  const int num_tiles = static_cast<int>((p.M + kTileM - 1) / kTileM);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
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
    // tile n of this CTA goes to warpgroup n % E, through that warpgroup's own ring (each ring is filled and
    // drained in order, so a parity wait can never pass on a phase two fills ahead)
    if (lane == 0) {
      mbar_arrive_expect_tx(bfull, L.b_bytes);
      for (int kb = 0; kb < kblocks; ++kb)
        tma_load_2d(smem_b + kb * p.n_pad * 128, &tmB, bfull, kb * kBlockK, 0);
      uint32_t slot = 0, ph = 0, slot_o = 0, ph_o = 0;         // ring position of this / the other warpgroup
      int g = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        for (int kb0 = 0; kb0 < kblocks; kb0 += kbs) {          // one ring stage per K chunk (usually the whole K)
          const uint32_t s = g * spg + slot;
          mbar_wait(&empty[s], ph ^ 1);
          mbar_arrive_expect_tx(&full[s], L.a_tile_bytes);
          uint8_t* dst = smem_a + s * L.a_tile_bytes;
          for (int kb = 0; kb < kbs; ++kb)
            tma_load_2d(dst + kb * (kTileM * 128), &tmA, &full[s], (kb0 + kb) * kBlockK, tile * kTileM);
          if (++slot == static_cast<uint32_t>(spg)) { slot = 0; ph ^= 1; }
        }
        if (E == 2) {
          g ^= 1;
          const uint32_t ts = slot, tp = ph;
          slot = slot_o; ph = ph_o; slot_o = ts; ph_o = tp;
        }
      }
    }
    return;
  }

  // ===================== consumer warpgroups: wgmma chain + epilogue =====================
  const int g = warp >> 2;                                     // warpgroup
  const int q = warp & 3;                                      // warp inside the warpgroup
  const int r_in_tile = kHalves == 2 ? wg_row128(q, lane) : 16 * q + lane;
  const bool lane_has_row = kHalves == 2 || lane < 16;
  float* scratch = reinterpret_cast<float*>(smem + L.scratch_off) + warp * kRowScratchFloats;
  const int npairs = p.N >> 1;
  {
    // per-CTA lookup tables (all consumer threads; named barrier 1)
    const int et = threadIdx.x;
    const int nthr = 128 * E;
    if (p.epi.mode == EPI_PAIR_SCATTER) {
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
  const int ksteps = (p.K + 15) / 16;                          // K=16 per instruction; zero tail needs no MMA
  const uint32_t b_addr = smem_u32(smem_b);
  float acc[kAccRegs];
  uint32_t slot = 0, ph = 0;
  for (int tile = blockIdx.x + g * gridDim.x; tile < num_tiles; tile += E * gridDim.x) {
    for (int kb0 = 0; kb0 < kblocks; kb0 += kbs) {
      const uint32_t s = g * spg + slot;
      mbar_wait(&full[s], ph);
      const uint32_t a_addr = smem_u32(smem_a + s * L.a_tile_bytes);
      const int ks_end = min(ksteps, (kb0 + kbs) * 4);
      wgmma_fence();
      for (int ks = kb0 * 4; ks < ks_end; ++ks) {
        const uint32_t kb = ks >> 2, kk = ks & 3;
        const uint64_t da = gdesc_k128(a_addr + (kb - kb0) * (kTileM * 128) + kk * 32);
        const uint64_t db = gdesc_k128(b_addr + kb * p.n_pad * 128 + kk * 32);
        if (kHalves == 2) wg_mma128<false, 0, 0>(acc, p.n_pad, da, 8192, db, ks > 0 ? 1u : 0u);
        else wg_mma64<false, 0, 0, 0>(acc, p.n_pad, da, db, ks > 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(acc);
      if ((threadIdx.x & 127) == 0) mbar_arrive(&empty[s]);       // the ring stage may be refilled
      if (++slot == static_cast<uint32_t>(spg)) { slot = 0; ph ^= 1; }
    }
    const long long row = static_cast<long long>(tile) * kTileM + r_in_tile;
    const bool row_ok = lane_has_row && row < p.M;

    if (p.epi.mode == EPI_ROWMAJOR && L.stage_pitch != 0) {
      // ---- coalesced row-major store: accumulator -> staging rows in smem (a private slab per warp holding its
      // kWarpRows rows, lane r = row r of the warp) -> groups of lanes write whole rows contiguously
      uint8_t* slab = smem + L.stage_off + (warp * 32) * L.stage_pitch;
      uint8_t* myrow = slab + lane * L.stage_pitch;
      const bool st16 = !p.epi.out_fp32;                       // bf16 output: stage packed bf16
#pragma unroll
      for (int ch = 0; ch < 8 * (3 - kHalves); ++ch) {
        const int c0 = ch * 16;
        if (c0 < p.N) {
          uint32_t v[16];
          wg_row16<kHalves>(acc, c0, scratch, v);
          if (st16) {
            uint4 u0, u1;
            u0.x = pack_bf16x2(__uint_as_float(v[0]), __uint_as_float(v[1]));
            u0.y = pack_bf16x2(__uint_as_float(v[2]), __uint_as_float(v[3]));
            u0.z = pack_bf16x2(__uint_as_float(v[4]), __uint_as_float(v[5]));
            u0.w = pack_bf16x2(__uint_as_float(v[6]), __uint_as_float(v[7]));
            u1.x = pack_bf16x2(__uint_as_float(v[8]), __uint_as_float(v[9]));
            u1.y = pack_bf16x2(__uint_as_float(v[10]), __uint_as_float(v[11]));
            u1.z = pack_bf16x2(__uint_as_float(v[12]), __uint_as_float(v[13]));
            u1.w = pack_bf16x2(__uint_as_float(v[14]), __uint_as_float(v[15]));
            reinterpret_cast<uint4*>(myrow + c0 * 2)[0] = u0;
            reinterpret_cast<uint4*>(myrow + c0 * 2)[1] = u1;
          } else {
#pragma unroll
            for (int i = 0; i < 4; ++i)
              reinterpret_cast<uint4*>(myrow + c0 * 4)[i] = make_uint4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
          }
        }
      }
      __syncwarp();
      const int vec_per_row = p.N >> 3;                       // 8 outputs per lane
      const int rows_per_it = 32 / vec_per_row;               // N = 128 -> 16 lanes per row, 2 rows / instr
      const int lr = lane / vec_per_row, lc = lane % vec_per_row;
      const long long tile0 = static_cast<long long>(tile) * kTileM;
      for (int rb = lr; rb < kWarpRows; rb += 4 * rows_per_it) {
        uint4 addv[4];
        bool okv[4];
        long long growv[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {                          // issue all global loads first
          const int rr = rb + u * rows_per_it;
          growv[u] = tile0 + (kHalves == 2 ? wg_row128(q, rr) : 16 * q + rr);
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
#pragma unroll
      for (int ch = 0; ch < 8 * (3 - kHalves); ++ch) {
        const int c0 = ch * 16;
        if (c0 >= p.N) continue;
        uint32_t v[16];
        wg_row16<kHalves>(acc, c0, scratch, v);
        if (!row_ok) continue;
        float f[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) f[i] = __uint_as_float(v[i]);
        const int ncol = min(16, p.N - c0);
        const bool vec = p.epi.vec_ok && ncol == 16;
        if (p.epi.add_src != nullptr) {
          const __nv_bfloat16* ap = reinterpret_cast<const __nv_bfloat16*>(p.epi.add_src) + row * p.epi.ld_add + c0;
          for (int i = 0; i < ncol; ++i) f[i] += __bfloat162float(ap[i]);
        }
        if (p.epi.out_fp32) {
          float* o = reinterpret_cast<float*>(p.epi.peers[0]) + row * p.epi.ldc + c0;
          if (vec) {
#pragma unroll
            for (int i = 0; i < 4; ++i)
              reinterpret_cast<float4*>(o)[i] = make_float4(f[4 * i], f[4 * i + 1], f[4 * i + 2], f[4 * i + 3]);
          } else {
            for (int i = 0; i < ncol; ++i) o[i] = f[i];
          }
        } else {
          __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.epi.peers[0]) + row * p.epi.ldc + c0;
          if (vec) {
            uint4 u0, u1;
            u0.x = pack_bf16x2(f[0], f[1]);   u0.y = pack_bf16x2(f[2], f[3]);
            u0.z = pack_bf16x2(f[4], f[5]);   u0.w = pack_bf16x2(f[6], f[7]);
            u1.x = pack_bf16x2(f[8], f[9]);   u1.y = pack_bf16x2(f[10], f[11]);
            u1.z = pack_bf16x2(f[12], f[13]); u1.w = pack_bf16x2(f[14], f[15]);
            reinterpret_cast<uint4*>(o)[0] = u0;
            reinterpret_cast<uint4*>(o)[1] = u1;
          } else {
            for (int i = 0; i < ncol; ++i) o[i] = __float2bfloat16(f[i]);
          }
        }
      }
    } else if (p.epi.mode == EPI_PAIR_SCATTER) {
      // ---- pair scatter: (re, im) pairs to a mixed-radix address, possibly on a peer GPU
      int rpeer;
      const long long roff = row_offset(p.epi, static_cast<uint32_t>(row_ok ? row : 0), rpeer);
      __nv_bfloat16* const rbase = reinterpret_cast<__nv_bfloat16*>(p.epi.peers[rpeer]) + roff;
#pragma unroll
      for (int ch = 0; ch < 8 * (3 - kHalves); ++ch) {
        const int c0 = ch * 16;
        if (c0 >= p.N) continue;
        uint32_t v[16];
        wg_row16<kHalves>(acc, c0, scratch, v);
        if (!row_ok) continue;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int j = (c0 >> 1) + i;
          if (j < npairs) {
            __nv_bfloat16* base = rbase;
            if (p.epi.peer_sel == PEER_BY_COL)
              base = reinterpret_cast<__nv_bfloat16*>(p.epi.peers[s_colpeer[j]]) + roff;
            *reinterpret_cast<uint32_t*>(base + s_coloff[j]) =
                pack_bf16x2(__uint_as_float(v[2 * i]), __uint_as_float(v[2 * i + 1]));
          }
        }
      }
    } else {
      // ---- projection head: out = b4 + sum_j W4[j] * gelu(acc[j] + b3[j])
      float part = s_vec[511];
#pragma unroll
      for (int ch = 0; ch < 8 * (3 - kHalves); ++ch) {
        const int c0 = ch * 16;
        if (c0 >= p.N) continue;
        uint32_t v[16];
        wg_row16<kHalves>(acc, c0, scratch, v);
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          if (c0 + i < p.N) {
            const float pre = __uint_as_float(v[i]) + s_vec[c0 + i];
            part = fmaf(s_vec[256 + c0 + i], gelu_erf(pre), part);
          }
        }
      }
      if (row_ok) {
        int unused;
        reinterpret_cast<float*>(p.epi.peers[0])[row_offset(p.epi, static_cast<uint32_t>(row), unused)] = part;
      }
    }
  }
  if (p.epi.peer_sel != PEER_NONE) __threadfence_system();   // publish peer stores
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

const char* dft_gemm_launch(const void* A, long long lda, const void* Bmat, GemmParams p, int num_sms,
                            cudaStream_t stream) {
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
  SmemLayout L;
  const int kblocks = p.k_pad / kBlockK;
  L.b_bytes = static_cast<uint32_t>(kblocks) * p.n_pad * 128;
  const uint32_t fixed = L.b_bytes + 4096 /*barriers + tables*/ + 1024 /*align slack*/;
  // coalesced row-major epilogue: needs N to be a multiple of 8 dividing 256 and aligned rows
  uint32_t pitch = 0;
  if (p.epi.mode == EPI_ROWMAJOR && p.epi.vec_ok && p.N % 8 == 0 && (p.N == 8 || p.N == 16 || p.N == 32 ||
      p.N == 64 || p.N == 128 || p.N == 256))
    pitch = ((p.N + 15) / 16 * 16) * (p.epi.out_fp32 ? 4 : 2) + 16;   // whole 16-column chunks are staged
  // consumer warpgroups, staging, ring depth and K chunk: two warpgroups with >= 2 whole-K stages each if possible;
  // for long K the largest divisor of the K blocks that leaves room for two stages
  bool ok = false;
  int E = kMaxGroups;
  for (; E >= 1 && !ok; --E) {
    for (int with_stage = pitch ? 1 : 0; with_stage >= 0 && !ok; --with_stage) {
      const uint32_t scratch = 4u * E * kRowScratchFloats * 4;
      const uint32_t stg = with_stage ? 4u * E * 32 * pitch : 0;
      if (fixed + scratch + stg > 227 * 1024) continue;
      const uint32_t avail = 227 * 1024 - fixed - scratch - stg;
      for (int dv = kblocks; dv >= 1 && !ok; --dv) {
        if (kblocks % dv) continue;
        const uint32_t a_tile = static_cast<uint32_t>(dv) * tile_m * 128;
        uint32_t spg = avail / (E * a_tile);
        if (spg > kMaxStagesPerGroup) spg = kMaxStagesPerGroup;
        if (spg >= 2) {
          L.kbs = static_cast<uint32_t>(dv); L.a_tile_bytes = a_tile; L.spg = spg;
          L.stage_pitch = with_stage ? pitch : 0;
          L.scratch_off = L.b_bytes + E * spg * a_tile + 4096;
          L.stage_off = L.scratch_off + scratch;
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
  const uint32_t smem_bytes = L.stage_off + (L.stage_pitch ? 4u * E * 32 * L.stage_pitch : 0);

  CUtensorMap tmA, tmB;
  // A: the K tail beyond p.K (up to k_pad) and the M tail are zero-filled by TMA
  if (make_map_2d(&tmA, A, static_cast<uint64_t>(p.K), static_cast<uint64_t>(p.M), static_cast<uint64_t>(lda),
                  kBlockK, tile_m))
    return "cuTensorMapEncodeTiled(A) failed";
  if (make_map_2d(&tmB, Bmat, static_cast<uint64_t>(p.k_pad), static_cast<uint64_t>(p.n_pad),
                  static_cast<uint64_t>(p.k_pad), kBlockK, static_cast<uint32_t>(p.n_pad)))
    return "cuTensorMapEncodeTiled(B) failed";

  static bool attr_set[2] = {false, false};
  const void* fn = halves == 2 ? reinterpret_cast<const void*>(dft_gemm_kernel<2>) : reinterpret_cast<const void*>(dft_gemm_kernel<1>);
  if (!attr_set[halves - 1]) {
    if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess)
      return "cudaFuncSetAttribute(max dynamic smem) failed";
    attr_set[halves - 1] = true;
  }
  const int num_tiles = static_cast<int>((p.M + tile_m - 1) / tile_m);
  const int grid = num_tiles < num_sms ? num_tiles : num_sms;
  if (halves == 2) dft_gemm_kernel<2><<<grid, 128 * E + 32, smem_bytes, stream>>>(tmA, tmB, p, L);
  else dft_gemm_kernel<1><<<grid, 128 * E + 32, smem_bytes, stream>>>(tmA, tmB, p, L);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

}  // namespace dfno
