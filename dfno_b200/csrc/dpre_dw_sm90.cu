// dpre_dw_sm90.cu -- backward of the pointwise part of a Fourier layer:
//
//   dpre[c, l, z] = g[c, l, z] * gelu'(pre[c, l, z])               (written over pre)
//   dW[o, i]     += sum_{l, z} dpre[o, l, z] * h[i, l, z]          (bypass weight gradient, reference
//                                                                   BroadcastedLinear backward, dfno.py:57-62)
//
// Same tile geometry as spectral_out_sm90.cu: R = floor(128/C) lines of all C channels, here 64 columns
// (one swizzle block) at a time, so g, pre and h tiles are 16 KB TMA boxes.  The element-wise part works on
// 16-byte chunks (8 values, packed fp16 GELU'); the weight gradient is a K-reduction over z on the tensor core:
//
//   D[(o, r), (i, r')] += sum_z dpre_tile[(o, r), z] * h_tile[(i, r'), z]      (both operands K-major as loaded)
//
// accumulated in the registers of each consumer warpgroup over every tile it visits; dW[o, i] is the sum of
// its r = r' entries, extracted once per CTA.  The input-gradient half of the bypass (W^T dpre) is not computed here: it
// is the second MMA of the adjoint chain's last stage (spectral_out with transpose_w).
#include "sm90_ptx.cuh"
#include "kernels.h"
#include "tma_host.h"

namespace dfno {
namespace {

constexpr uint32_t kBlkD = 16384;
constexpr int kStagesD = 4;
constexpr int kGroupsD = 2;                    // consumer warpgroups (kStagesD a multiple of it: see bypass_sm90.cu)
static_assert(kStagesD % kGroupsD == 0, "every ring stage must belong to one consumer warpgroup");
constexpr int kThreadsD = 128 * kGroupsD + 32;

struct DpreParams {
  int B, C, R, RC;
  long long L, tiles_per_b;
  int Z, nzb;               // 64-column blocks per line
  float* dW;                // [C, C] fp32, accumulated with atomics
};

__global__ void __launch_bounds__(kThreadsD, 1)
dpre_dw_kernel(const __grid_constant__ CUtensorMap tmG, const __grid_constant__ CUtensorMap tmP,
               const __grid_constant__ CUtensorMap tmH, const DpreParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* ring = smem;                                        // stages x {g, pre, h}
  uint64_t* bars = reinterpret_cast<uint64_t*>(ring + kStagesD * 3 * kBlkD);
  uint64_t* full = bars;              // [4] TMA -> compute
  uint64_t* empty = bars + 4;         // [4] compute -> TMA (after the dpre store has been read and the MMA retired)
  float* s_dw = reinterpret_cast<float*>(bars + 8);            // [C * C]

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const long long num_tiles = p.tiles_per_b * p.B * p.nzb;

  for (uint32_t i = threadIdx.x; i < kStagesD * 3 * kBlkD / 16; i += blockDim.x)
    reinterpret_cast<uint4*>(ring)[i] = make_uint4(0, 0, 0, 0);
  for (int i = threadIdx.x; i < p.C * p.C; i += blockDim.x) s_dw[i] = 0.f;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmG); tma_prefetch_desc(&tmP); tma_prefetch_desc(&tmH);
    for (int s = 0; s < kStagesD; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 1); }
    fence_barrier_init();
  }
  fence_proxy_async_smem();
  __syncthreads();

  if (warp == 4 * kGroupsD) {
    if (lane == 0) {
      uint32_t s = 0, ph = 0;
      for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int zb = static_cast<int>(tile % p.nzb);
        const long long lt = (tile / p.nzb) % p.tiles_per_b;
        const int b = static_cast<int>(tile / (p.nzb * p.tiles_per_b));
        const int l0 = static_cast<int>(lt * p.R);
        mbar_wait(&empty[s], ph ^ 1);
        mbar_arrive_expect_tx(&full[s], 3u * p.RC * 128);
        uint8_t* st = ring + s * 3 * kBlkD;
        tma_load_3d(st, &tmG, &full[s], zb * 64, l0, b * p.C);
        tma_load_3d(st + kBlkD, &tmP, &full[s], zb * 64, l0, b * p.C);
        tma_load_3d(st + 2 * kBlkD, &tmH, &full[s], zb * 64, l0, b * p.C);
        if (++s == kStagesD) { s = 0; ph ^= 1; }
      }
    }
    return;
  }
  const int g = warp >> 2;
  const int t = threadIdx.x & 127;                                  // 0..127 inside the warpgroup
  const uint32_t barid = 1 + g;
  float acc[128];                                                   // D[(o, r), (i, r')] of this warpgroup's tiles
  long long n = 0, mine = 0;
  for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++n) {
    if (n % kGroupsD != g) continue;
    const uint32_t s = static_cast<uint32_t>(n % kStagesD);
    const uint32_t par = (n / kStagesD) & 1;
    const int zb = static_cast<int>(tile % p.nzb);
    const long long lt = (tile / p.nzb) % p.tiles_per_b;
    const int b = static_cast<int>(tile / (p.nzb * p.tiles_per_b));
    uint8_t* gt = ring + s * 3 * kBlkD;
    uint8_t* pt = gt + kBlkD;
    mbar_wait(&full[s], par);
    for (int idx = t; idx < p.RC * 8; idx += 128) {
      const uint32_t off = static_cast<uint32_t>(idx) << 4;       // chunk position is irrelevant: element-wise
      const uint4 G = *reinterpret_cast<const uint4*>(gt + off);
      const uint4 P = *reinterpret_cast<const uint4*>(pt + off);
      uint4 D;
      const uint32_t gw[4] = {G.x, G.y, G.z, G.w}, pw[4] = {P.x, P.y, P.z, P.w};
      uint32_t dw[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 gr = __half22float2(gelu_vg_h2(bf16x2_to_h2(pw[i])).grad);
        const float2 gg = unpack_bf16x2(gw[i]);
        dw[i] = pack_bf16x2(gg.x * gr.x, gg.y * gr.y);
      }
      D.x = dw[0]; D.y = dw[1]; D.z = dw[2]; D.w = dw[3];
      *reinterpret_cast<uint4*>(pt + off) = D;
    }
    fence_proxy_async_smem();
    asm volatile("bar.sync %0, 128;" ::"r"(barid) : "memory");
    if (t == 0) {
      tma_store_3d(&tmP, pt, zb * 64, static_cast<int>(lt * p.R), b * p.C);
      tma_store_commit();
    }
    {
      // weight gradient on the tensor core: D += dpre_tile . h_tile^T, K = z (columns beyond Z are zero-filled by TMA)
      const int ksteps = (min(64, p.Z - zb * 64) + 15) >> 4;
      const uint32_t dp = smem_u32(pt), hh = dp + kBlkD;
      wgmma_fence();
      for (int kk = 0; kk < ksteps; ++kk)
        wg_mma128<false, 0, 0>(acc, 128, gdesc_k128(dp + kk * 32), 8192, gdesc_k128(hh + kk * 32),
                               (mine > 0 || kk > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(acc);
      ++mine;
    }
    if (t == 0) {
      tma_store_wait_read();
      mbar_arrive(&empty[s]);
    }
  }
  if (t == 0) tma_store_wait_all();
  // ---- weight gradient: diagonal (r == r') entries of the accumulator, summed over r.  Fragment: register
  // h*64 + 4j + e holds row m = 64h + 16(warp%4) + lane/4 + 8(e/2), column k = 8j + 2(lane%4) + e%2.
  if (mine > 0) {
    const int m0 = 16 * (warp & 3) + (lane >> 2), k0 = 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int m = 64 * h + m0 + 8 * (e >> 1), k = 8 * j + k0 + (e & 1);
          if (m < p.RC && k < p.RC) {
            const int o = m / p.R, i = k / p.R;
            if (m - o * p.R == k - i * p.R) atomicAdd(&s_dw[o * p.C + i], acc[64 * h + 4 * j + e]);
          }
        }
  }
  asm volatile("bar.sync 3, %0;" ::"n"(128 * kGroupsD) : "memory");
  if (num_tiles > blockIdx.x)
    for (int i = threadIdx.x; i < p.C * p.C; i += 128 * kGroupsD) atomicAdd(p.dW + i, s_dw[i]);
}

}  // namespace

// g, h: bf16 [B*C, L, Z]; pre_dpre: bf16 [B*C, L, Z], pre-activation in, dpre out; dW: fp32 [C, C] (accumulated)
const char* dpre_dw(const void* g, void* pre_dpre, const void* h, float* dW, int B, int C, long long L, int Z,
                    int num_sms, cudaStream_t stream) {
  if (C < 1 || C > 64) return "dpre_dw: 1 <= C <= 64";
  if (Z % 8) return "dpre_dw: Z % 8 != 0";
  if (L > (1ll << 31) - 256) return "dpre_dw: tensor too large";
  DpreParams p{};
  p.B = B; p.C = C; p.R = 128 / C; p.RC = p.R * C; p.L = L; p.tiles_per_b = (L + p.R - 1) / p.R;
  p.Z = Z; p.nzb = (Z + 63) / 64; p.dW = dW;
  CUtensorMap tmG, tmP, tmH;
  const uint64_t BC = static_cast<uint64_t>(B) * C;
  if (make_map_3d(&tmG, g, Z, L, BC, Z, static_cast<uint64_t>(L) * Z, 64, p.R, C)) return "tensor map (g) failed";
  if (make_map_3d(&tmP, pre_dpre, Z, L, BC, Z, static_cast<uint64_t>(L) * Z, 64, p.R, C)) return "tensor map (pre) failed";
  if (make_map_3d(&tmH, h, Z, L, BC, Z, static_cast<uint64_t>(L) * Z, 64, p.R, C)) return "tensor map (h) failed";
  static bool attr = false;
  if (!attr) {
    if (cudaFuncSetAttribute(dpre_dw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess)
      return "cudaFuncSetAttribute failed";
    attr = true;
  }
  const uint32_t smem_bytes = kStagesD * 3 * kBlkD + 64 + 4 * 64 * 64 + 1024;
  const long long tiles = p.tiles_per_b * B * p.nzb;
  const int grid = static_cast<int>(tiles < num_sms ? tiles : num_sms);
  dpre_dw_kernel<<<grid, kThreadsD, smem_bytes, stream>>>(tmG, tmP, tmH, p);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

}  // namespace dfno
