// pointwise.cu -- channel/time mixing kernels around the Fourier layers (sm_90a, CUDA cores).
//
// Internal activation layout of the fused engine: h[bc = b*C + c][x][y_local][t][z], bf16,
// z contiguous (so that every DFT stage is a K-major GEMM, see dft_gemm_sm90.cu).  The
// public tensors keep the reference layout [B, C, X, Y, Z, T] (t contiguous); the lift and
// the projection head are where the two layouts meet, so no transpose pass ever runs.
//
//   lift_fwd        : x[B,Cin,X,Y,Z,Tin] -> h = gelu(W2 ._c gelu(W1 ._t x + b1) + b2)
//                     (reference: linear1 -> gelu -> linear2 -> gelu, dfno.py:333-338; K15+K16)
//   lift_bwd        : dh -> dW1, db1, dW2, db2 (recomputes the tiny activations), optionally dx
//   bypass_gelu_fwd : pre = spec + W ._c h ; out = gelu(pre)         (K2 + K14, dfno.py:244,291)
//   bypass_gelu_bwd : dpre = dout * gelu'(pre) ; dhb = W^T ._c dpre  (weight grad: kreduce GEMM)
//   to_channels_last / from_channels_last : layout bridges for the projection head
#include "sm90_ptx.cuh"
#include "kernels.h"

namespace dfno {

namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <typename T>
__device__ __forceinline__ float ldf(const T* p);
template <>
__device__ __forceinline__ float ldf<float>(const float* p) { return *p; }
template <>
__device__ __forceinline__ float ldf<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }

// ------------------------------------------------------------------------------------------
// lift
// ------------------------------------------------------------------------------------------
// One thread owns 8 consecutive z of one (b, x, y) -- a 16-byte bf16 vector of every output row it produces,
// so a warp writes whole 256-byte z-lines -- and walks t and c.  Both GELUs run in packed fp16 (sm90_ptx.cuh):
// the outer one is evaluated B*C*X*Y*Z*T times per step.  The few input values a thread needs stay in
// registers when Tin == 1 (the benchmark / two-phase case) and are re-read through L1 otherwise (Cin <= 4, Tin <= 64;
// more input channels run the one-warp-per-item kernels below).
constexpr int kLiftMaxTin = 64;
constexpr int kLiftMaxW = 4096;    // floats of shared memory for W1, b1 (+ packed W2, b2)

template <typename TIn>
__device__ __forceinline__ void lift_load8(const TIn* __restrict__ src, int Tin, int ti, float (&v)[8]) {
#pragma unroll
  for (int z = 0; z < 8; ++z) v[z] = ldf(src + z * Tin + ti);
}
template <>
__device__ __forceinline__ void lift_load8<float>(const float* __restrict__ src, int Tin, int ti, float (&v)[8]) {
  if (Tin == 1) {
    const float4 a = reinterpret_cast<const float4*>(src)[0], b = reinterpret_cast<const float4*>(src)[1];
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
#pragma unroll
    for (int z = 0; z < 8; ++z) v[z] = src[z * Tin + ti];
  }
}

// v1[z] = b1[t] + sum_ti W1[t, ti] x[ci, z, ti]
template <typename TIn, bool kRegs>
__device__ __forceinline__ void lift_inner(const TIn* __restrict__ xci, const float (*xr)[8], int ci, int Tin,
                                           const float* sW1t, float b1t, float (&v)[8]) {
#pragma unroll
  for (int z = 0; z < 8; ++z) v[z] = b1t;
  for (int ti = 0; ti < Tin; ++ti) {
    float xv[8];
    if (kRegs) {                        // Tin == 1
#pragma unroll
      for (int z = 0; z < 8; ++z) xv[z] = xr[ci][z];
    } else {
      lift_load8<TIn>(xci, Tin, ti, xv);
    }
    const float w = sW1t[ti];
#pragma unroll
    for (int z = 0; z < 8; ++z) v[z] = fmaf(w, xv[z], v[z]);
  }
}

template <typename TIn, int CIN, bool kRegs>
__global__ void __launch_bounds__(256)
lift_fwd_kernel(const TIn* __restrict__ x, const float* __restrict__ W1, const float* __restrict__ b1,
                const float* __restrict__ W2, const float* __restrict__ b2, __nv_bfloat16* __restrict__ h,
                LiftDims d) {
  __shared__ float sw[kLiftMaxW];
  float* sW1 = sw;                                          // [T][Tin]
  float* sb1 = sW1 + d.T * d.Tin;                           // [T]
  __half2* sW2 = reinterpret_cast<__half2*>(sb1 + d.T);     // [C][CIN] (value duplicated in both halves)
  __half2* sb2 = sW2 + d.C * CIN;                           // [C]
  for (int i = threadIdx.x; i < d.T * d.Tin; i += blockDim.x) sW1[i] = W1[i];
  for (int i = threadIdx.x; i < d.T; i += blockDim.x) sb1[i] = b1[i];
  for (int i = threadIdx.x; i < d.C * CIN; i += blockDim.x) sW2[i] = __float2half2_rn(W2[i]);
  for (int i = threadIdx.x; i < d.C; i += blockDim.x) sb2[i] = __float2half2_rn(b2[i]);
  __syncthreads();

  const int zv = d.Z >> 3;
  const long long plane = static_cast<long long>(d.X) * d.Y;
  const long long nitems = static_cast<long long>(d.B) * plane * zv;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < nitems;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int z0 = static_cast<int>(idx % zv) * 8;
    const long long xy = (idx / zv) % plane;
    const int b = static_cast<int>(idx / (zv * plane));
    const TIn* xb = x + (((static_cast<long long>(b) * CIN) * plane + xy) * d.Z + z0) * d.Tin;
    const long long xci_stride = plane * d.Z * d.Tin;
    float xr[kRegs ? CIN : 1][8];
    if (kRegs) {
#pragma unroll
      for (int ci = 0; ci < CIN; ++ci) lift_load8<TIn>(xb + ci * xci_stride, 1, 0, xr[ci]);
    }
    __nv_bfloat16* hb = h + ((static_cast<long long>(b) * d.C * plane + xy) * d.T) * d.Z + z0;
    const long long hc_stride = plane * d.T * d.Z;
    for (int t = 0; t < d.T; ++t) {
      __half2 a1[CIN][4];
#pragma unroll
      for (int ci = 0; ci < CIN; ++ci) {
        float v[8];
        lift_inner<TIn, kRegs>(xb + ci * xci_stride, xr, ci, d.Tin, sW1 + t * d.Tin, sb1[t], v);
#pragma unroll
        for (int k = 0; k < 4; ++k) a1[ci][k] = gelu_h2(h2_from_f32(v[2 * k], v[2 * k + 1]));
      }
      for (int c = 0; c < d.C; ++c) {
        uint32_t o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          __half2 acc = sb2[c];
#pragma unroll
          for (int ci = 0; ci < CIN; ++ci) acc = __hfma2(sW2[c * CIN + ci], a1[ci][k], acc);
          o[k] = h2_to_bf16x2(gelu_h2(acc));
        }
        *reinterpret_cast<uint4*>(hb + c * hc_stride + static_cast<long long>(t) * d.Z) = make_uint4(o[0], o[1], o[2], o[3]);
      }
    }
  }
}

// dW1[T][Tin], db1[T], dW2[C][Cin], db2[C] accumulated with atomics into fp32 buffers.  Four adjacent lanes share
// one item (8 consecutive z of one (b, x, y)) and split the C channels between them: a thread keeps C/4 channel
// sums in registers over the whole grid-stride loop (with all C channels per thread the kernel needs about twice
// the registers and far lower occupancy), the input-gradient
// partials of the four quarters meet in two shuffles per value, and time-indexed sums are warp-reduced once per
// t.  The loss gradient can be far below the fp16 range, so everything it multiplies is fp32; only the GELU'
// evaluations are packed fp16.
//
// kDx: also the input gradient dx[b, ci, x, y, z, ti] = sum_t W1[t, ti] e[ci, z, t] (fp32, same layout as x), with
// e = dL/d(linear1 pre-activation).  After the quad shuffles every lane of the quad holds all 8 e[ci][z]; lane cg
// owns z0 + 2cg and z0 + 2cg + 1, whose 2 * Tin values are contiguous in x's layout and written by this lane alone:
// no atomics, no memset.  Tin == 1 keeps the 2 * CIN sums in registers over t; otherwise the first t stores and
// later t add (read-modify-write of the lane's own run, which stays in L1 / L2).
//
// Widths above 32 (48, 64) split the channels over eight lanes instead (kSplit): each lane keeps C/8 channel sums, the
// per-thread register cost of width 32.  The input gradient is then written by the first four lanes of the eight.
template <typename TIn, int C, int CIN, bool kRegs, bool kDx>
__global__ void __launch_bounds__(128, (CIN == 1 ? 4 : 2))      // several input channels: more live values, no spills
lift_bwd_kernel(const TIn* __restrict__ x, const float* __restrict__ W1, const float* __restrict__ b1,
                const float* __restrict__ W2, const float* __restrict__ b2,
                const __nv_bfloat16* __restrict__ dh, float* __restrict__ gW1, float* __restrict__ gb1,
                float* __restrict__ gW2, float* __restrict__ gb2, LiftDims d, float* __restrict__ dx) {
  constexpr int kSplitLog = C > 32 ? 3 : 2;
  constexpr int kSplit = 1 << kSplitLog;                     // lanes per item
  static_assert(C % kSplit == 0, "the channels are split evenly over the lanes of an item");
  constexpr int CG = C / kSplit;
  __shared__ float sw[kLiftMaxW];
  __shared__ float sg[kLiftMaxW];
  float* sW1 = sw;
  float* sb1 = sW1 + d.T * d.Tin;
  float* sW2f = sb1 + d.T;                                   // [C][CIN] fp32 (input-gradient path)
  __half2* sW2 = reinterpret_cast<__half2*>(sW2f + C * CIN); // [C][CIN] packed fp16 (recomputation)
  __half2* sb2 = sW2 + C * CIN;
  float* gsW1 = sg;
  float* gsb1 = gsW1 + d.T * d.Tin;
  for (int i = threadIdx.x; i < d.T * d.Tin; i += blockDim.x) { sW1[i] = W1[i]; gsW1[i] = 0.f; }
  for (int i = threadIdx.x; i < d.T; i += blockDim.x) { sb1[i] = b1[i]; gsb1[i] = 0.f; }
  for (int i = threadIdx.x; i < C * CIN; i += blockDim.x) { sW2f[i] = W2[i]; sW2[i] = __float2half2_rn(W2[i]); }
  for (int i = threadIdx.x; i < C; i += blockDim.x) sb2[i] = __float2half2_rn(b2[i]);
  __syncthreads();

  float accb2[CG], accW2[CG][CIN];
#pragma unroll
  for (int u = 0; u < CG; ++u) {
    accb2[u] = 0.f;
#pragma unroll
    for (int ci = 0; ci < CIN; ++ci) accW2[u][ci] = 0.f;
  }
  const int lane = threadIdx.x & 31;
  const int cg = lane & (kSplit - 1), c0 = cg * CG;          // this lane's channels: [c0, c0 + CG)
  const bool dx_lane = kSplit == 4 || cg < 4;                // lanes 0..3 of the item own its 8 z of dx
  const int zv = d.Z >> 3;
  const long long plane = static_cast<long long>(d.X) * d.Y;
  const long long nitems = static_cast<long long>(d.B) * plane * zv;
  const long long per_it = (static_cast<long long>(gridDim.x) * blockDim.x) >> kSplitLog;
  const long long nloop = (nitems + per_it - 1) / per_it;
  const long long item0 = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> kSplitLog;
  for (long long it = 0; it < nloop; ++it) {
    const long long idx = it * per_it + item0;
    const bool ok = idx < nitems;                           // whole warps stay in the loop (shuffles)
    const long long id = ok ? idx : 0;
    const int z0 = static_cast<int>(id % zv) * 8;
    const long long xy = (id / zv) % plane;
    const int b = static_cast<int>(id / (zv * plane));
    const TIn* xb = x + (((static_cast<long long>(b) * CIN) * plane + xy) * d.Z + z0) * d.Tin;
    const long long xci_stride = plane * d.Z * d.Tin;
    float xr[kRegs ? CIN : 1][8];
    if (kRegs) {
#pragma unroll
      for (int ci = 0; ci < CIN; ++ci) lift_load8<TIn>(xb + ci * xci_stride, 1, 0, xr[ci]);
    }
    const long long hc_stride = plane * d.T * d.Z;
    const __nv_bfloat16* gb = dh + ((static_cast<long long>(b) * C * plane + xy) * d.T) * d.Z + z0 + c0 * hc_stride;
    float* dxl = kDx ? dx + (xb - x) + 2 * cg * d.Tin : nullptr;     // this lane's run [2 z][Tin] of ci = 0
    float dxr[kDx && kRegs ? CIN : 1][2];
    if (kDx && kRegs) {
#pragma unroll
      for (int ci = 0; ci < CIN; ++ci) dxr[ci][0] = dxr[ci][1] = 0.f;
    }
    for (int t = 0; t < d.T; ++t) {
      __half2 a1[CIN][4];
      float a1f[CIN][8], g1f[CIN][8], da1[CIN][8];
#pragma unroll
      for (int ci = 0; ci < CIN; ++ci) {
        float v[8];
        lift_inner<TIn, kRegs>(xb + ci * xci_stride, xr, ci, d.Tin, sW1 + t * d.Tin, sb1[t], v);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const GeluH2 vg = gelu_vg_h2(h2_from_f32(v[2 * k], v[2 * k + 1]));
          a1[ci][k] = vg.value;
          const float2 av = __half22float2(vg.value), gv = __half22float2(vg.grad);
          a1f[ci][2 * k] = av.x; a1f[ci][2 * k + 1] = av.y;
          g1f[ci][2 * k] = gv.x; g1f[ci][2 * k + 1] = gv.y;
          da1[ci][2 * k] = 0.f; da1[ci][2 * k + 1] = 0.f;
        }
      }
      uint4 gv[CG];                                         // this lane's channel loads, all in flight together
#pragma unroll
      for (int u = 0; u < CG; ++u)
        gv[u] = ok ? *reinterpret_cast<const uint4*>(gb + u * hc_stride + static_cast<long long>(t) * d.Z)
                   : make_uint4(0, 0, 0, 0);
#pragma unroll
      for (int u = 0; u < CG; ++u) {
        const int c = c0 + u;
        const uint32_t gw[4] = {gv[u].x, gv[u].y, gv[u].z, gv[u].w};
        float dv[8];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          __half2 acc = sb2[c];
#pragma unroll
          for (int ci = 0; ci < CIN; ++ci) acc = __hfma2(sW2[c * CIN + ci], a1[ci][k], acc);
          const float2 gr = __half22float2(gelu_vg_h2(acc).grad);
          const float2 g = unpack_bf16x2(gw[k]);
          dv[2 * k] = g.x * gr.x; dv[2 * k + 1] = g.y * gr.y;
        }
        float sb = 0.f;
#pragma unroll
        for (int z = 0; z < 8; ++z) sb += dv[z];
        accb2[u] += sb;
#pragma unroll
        for (int ci = 0; ci < CIN; ++ci) {
          const float w = sW2f[c * CIN + ci];
          float sacc = 0.f;
#pragma unroll
          for (int z = 0; z < 8; ++z) {
            sacc = fmaf(dv[z], a1f[ci][z], sacc);
            da1[ci][z] = fmaf(w, dv[z], da1[ci][z]);
          }
          accW2[u][ci] += sacc;
        }
      }
      // input-gradient partials of the four channel quarters -> every lane of the quad holds the full sum
#pragma unroll
      for (int ci = 0; ci < CIN; ++ci) {
#pragma unroll
        for (int z = 0; z < 8; ++z) {
          float v = da1[ci][z];
          v += __shfl_xor_sync(0xffffffffu, v, 1);
          v += __shfl_xor_sync(0xffffffffu, v, 2);
          if constexpr (kSplit == 8) v += __shfl_xor_sync(0xffffffffu, v, 4);
          da1[ci][z] = v;
        }
      }
      const bool own = ok && cg == 0;                       // one lane of the quad feeds the time-indexed sums
      float sb1v = 0.f;
#pragma unroll
      for (int ci = 0; ci < CIN; ++ci) {
        float e[8];
#pragma unroll
        for (int z = 0; z < 8; ++z) { e[z] = da1[ci][z] * g1f[ci][z]; sb1v += e[z]; }
        float e0 = e[0], e1 = e[1];                           // e at this lane's two z (kDx)
        if (kDx) {
#pragma unroll
          for (int k = 1; k < 4; ++k)
            if (cg == k) { e0 = e[2 * k]; e1 = e[2 * k + 1]; }
          if (kRegs) {
            const float w = sW1[t];
            dxr[ci][0] = fmaf(w, e0, dxr[ci][0]);
            dxr[ci][1] = fmaf(w, e1, dxr[ci][1]);
          }
        }
        for (int ti = 0; ti < d.Tin; ++ti) {
          float xv[8];
          if (kRegs) {
#pragma unroll
            for (int z = 0; z < 8; ++z) xv[z] = xr[ci][z];
          } else {
            lift_load8<TIn>(xb + ci * xci_stride, d.Tin, ti, xv);
          }
          float sres = 0.f;
#pragma unroll
          for (int z = 0; z < 8; ++z) sres = fmaf(e[z], xv[z], sres);
          sres = warp_sum(own ? sres : 0.f);
          if (lane == 0) atomicAdd(&gsW1[t * d.Tin + ti], sres);
          if (kDx && !kRegs && ok && dx_lane) {
            float* p = dxl + ci * xci_stride + ti;
            const float w = sW1[t * d.Tin + ti];
            if (t == 0) {
              p[0] = w * e0;
              p[d.Tin] = w * e1;
            } else {
              p[0] = fmaf(w, e0, p[0]);
              p[d.Tin] = fmaf(w, e1, p[d.Tin]);
            }
          }
        }
      }
      sb1v = warp_sum(own ? sb1v : 0.f);
      if (lane == 0) atomicAdd(&gsb1[t], sb1v);
    }
    if (kDx && kRegs && ok && dx_lane) {
#pragma unroll
      for (int ci = 0; ci < CIN; ++ci)
        *reinterpret_cast<float2*>(dxl + ci * xci_stride) = make_float2(dxr[ci][0], dxr[ci][1]);
    }
  }
  __shared__ float gsW2[64 * 4 + 64];
  for (int i = threadIdx.x; i < C * CIN + C; i += blockDim.x) gsW2[i] = 0.f;
  __syncthreads();
  // channel sums: lanes with the same share (lane % kSplit) hold partials of the same channels
  auto quarter_sum = [](float v) {
    if constexpr (kSplit == 4) v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 8);
    v += __shfl_xor_sync(0xffffffffu, v, 16);
    return v;
  };
#pragma unroll
  for (int u = 0; u < CG; ++u) {
    const float sres = quarter_sum(accb2[u]);
    if (lane < kSplit) atomicAdd(&gsW2[C * CIN + c0 + u], sres);
#pragma unroll
    for (int ci = 0; ci < CIN; ++ci) {
      const float sw2 = quarter_sum(accW2[u][ci]);
      if (lane < kSplit) atomicAdd(&gsW2[(c0 + u) * CIN + ci], sw2);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < d.T * d.Tin; i += blockDim.x) atomicAdd(&gW1[i], gsW1[i]);
  for (int i = threadIdx.x; i < d.T; i += blockDim.x) atomicAdd(&gb1[i], gsb1[i]);
  for (int i = threadIdx.x; i < C * CIN; i += blockDim.x) atomicAdd(&gW2[i], gsW2[i]);
  for (int i = threadIdx.x; i < C; i += blockDim.x) atomicAdd(&gb2[i], gsW2[C * CIN + i]);
}

// ------------------------------------------------------------------------------------------
// lift, 5 <= Cin <= 16
// ------------------------------------------------------------------------------------------
// One warp owns one item (8 consecutive z of one (b, x, y)) and walks t.  Per t it runs in phases that map the lanes
// differently, with a per-warp tile in shared memory between them:
//   time lift : lane = (ci, z part of ZL = CINP / 4 values); a1 = gelu(b1 + W1 ._t x) in packed fp16 -> tile
//   channels  : lane = output channel c (c + 32 for widths above 32); all CINP a1 values of the item come from the tile
//   (backward) input side : lane = (ci, z part) again, reading the tile of dv = dh * gelu'(pre2) of every c.
// So no thread ever holds CIN x 8 values.  With Tin > 1 the warp first copies the item's x (Cin runs of 8 * Tin
// values, 5 KB at Cin = 16, Tin = 10 in fp32) into its own shared-memory slice with 16-byte loads; every t then reads
// that copy, so x is read from global memory exactly once per call whatever T is.  (Tin == 1 keeps the lane's few x
// values in registers instead.)  CINP (8 or 16) is the compile-time channel bound; W2 is zero-padded to it, so
// channels ci >= Cin add exact zeros.
constexpr int kLiftManyMaxC = 64;
constexpr int kLiftManyWarps = 4;                      // warps per block (each with its own x slice)

// elements between the shared-memory runs of two input channels: the run rounded up to 32 bytes, plus 16 bytes, so
// that the lanes of different channels fall on different banks
template <typename TIn>
__host__ __device__ inline int lift_many_xs_stride(int Tin) {
  const int words = 8 * Tin * static_cast<int>(sizeof(TIn)) / 4;
  return ((words + 7) / 8 * 8 + 4) * 4 / static_cast<int>(sizeof(TIn));
}

// the warp's copy of one item's x: xs[ci * stride + z * Tin + ti] = x[b, ci, x, y, z0 + z, ti] (runs are 16-byte
// multiples at 16-byte aligned addresses: Z % 8 == 0)
template <typename TIn>
__device__ __forceinline__ void lift_many_stage(const TIn* __restrict__ xb, long long xci_stride, int Cin, int Tin,
                                                int lane, TIn* xs) {
  const int nv = 8 * Tin * static_cast<int>(sizeof(TIn)) / 16;
  const int sv = lift_many_xs_stride<TIn>(Tin) * static_cast<int>(sizeof(TIn)) / 16;
  for (int j = lane; j < Cin * nv; j += 32) {
    const int ci = j / nv, k = j - ci * nv;
    reinterpret_cast<uint4*>(xs)[ci * sv + k] = reinterpret_cast<const uint4*>(xb + ci * xci_stride)[k];
  }
}

template <int CINP>
struct LiftManyLanes {
  static constexpr int ZL = CINP / 4;                 // z values per lane in the input-side phases
  static constexpr int kParts = 8 / ZL;               // lanes per input channel
};

template <typename TIn, int ZL>
__device__ __forceinline__ void lift_many_load(const TIn* __restrict__ p, int stride, float (&v)[ZL]) {
#pragma unroll
  for (int z = 0; z < ZL; ++z) v[z] = ldf(p + z * stride);
}

// v[z] = b1[t] + sum_ti W1[t, ti] x[ci, z, ti] for this lane's ZL values of z
template <typename TIn, int ZL, bool kRegs>
__device__ __forceinline__ void lift_many_inner(const TIn* __restrict__ xz, const float (&xr)[ZL], int Tin,
                                                const float* sW1t, float b1t, float (&v)[ZL]) {
#pragma unroll
  for (int z = 0; z < ZL; ++z) v[z] = kRegs ? fmaf(sW1t[0], xr[z], b1t) : b1t;
  if (!kRegs) {
    for (int ti = 0; ti < Tin; ++ti) {
      float xv[ZL];
      lift_many_load<TIn, ZL>(xz + ti, Tin, xv);
      const float w = sW1t[ti];
#pragma unroll
      for (int z = 0; z < ZL; ++z) v[z] = fmaf(w, xv[z], v[z]);
    }
  }
}

template <typename TIn, int CINP, bool kRegs>
__global__ void __launch_bounds__(32 * kLiftManyWarps)
lift_fwd_many_kernel(const TIn* __restrict__ x, const float* __restrict__ W1, const float* __restrict__ b1,
                     const float* __restrict__ W2, const float* __restrict__ b2, __nv_bfloat16* __restrict__ h,
                     LiftDims d) {
  using L = LiftManyLanes<CINP>;
  constexpr int ZL = L::ZL, kWarps = kLiftManyWarps;
  extern __shared__ uint4 fxs[];                                       // per warp: Cin runs of x (Tin > 1)
  __shared__ float sw[kLiftMaxW];                                      // W1 [T][Tin], b1 [T]
  __shared__ __half2 sW2[CINP * kLiftManyMaxC];                        // [CINP][C] (lanes = c: no bank conflicts)
  __shared__ __half2 sb2[kLiftManyMaxC];
  __shared__ __align__(16) __half2 sa1[kWarps][CINP][4];              // a1 of the warp's item at one t
  float* sW1 = sw;
  float* sb1 = sW1 + d.T * d.Tin;
  for (int i = threadIdx.x; i < d.T * d.Tin; i += blockDim.x) sW1[i] = W1[i];
  for (int i = threadIdx.x; i < d.T; i += blockDim.x) sb1[i] = b1[i];
  for (int i = threadIdx.x; i < d.C * CINP; i += blockDim.x) {
    const int c = i / CINP, ci = i % CINP;
    sW2[ci * kLiftManyMaxC + c] = __float2half2_rn(ci < d.Cin ? W2[c * d.Cin + ci] : 0.f);  // zero beyond Cin
  }
  for (int i = threadIdx.x; i < d.C; i += blockDim.x) sb2[i] = __float2half2_rn(b2[i]);
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ci = lane / L::kParts, zl = (lane % L::kParts) * ZL;        // input-side role
  const bool live = ci < d.Cin;
  const int zv = d.Z >> 3;
  const long long plane = static_cast<long long>(d.X) * d.Y;
  const long long nitems = static_cast<long long>(d.B) * plane * zv;
  const long long hc_stride = plane * d.T * d.Z;
  for (long long idx = blockIdx.x * static_cast<long long>(kWarps) + warp; idx < nitems;
       idx += static_cast<long long>(gridDim.x) * kWarps) {              // warp-uniform
    const int z0 = static_cast<int>(idx % zv) * 8;
    const long long xy = (idx / zv) % plane;
    const int b = static_cast<int>(idx / (zv * plane));
    const TIn* xb = x + ((static_cast<long long>(b) * d.Cin * plane + xy) * d.Z + z0) * d.Tin;
    const long long xci_stride = plane * d.Z * d.Tin;
    const TIn* xz;
    float xr[ZL];
    if (kRegs) {
      xz = xb + (live ? ci : 0) * xci_stride + zl;
      if (live) lift_many_load<TIn, ZL>(xz, 1, xr);
    } else {
      const int xss = lift_many_xs_stride<TIn>(d.Tin);
      TIn* xs = reinterpret_cast<TIn*>(fxs) + warp * d.Cin * xss;
      lift_many_stage<TIn>(xb, xci_stride, d.Cin, d.Tin, lane, xs);   // the previous item's reads ended at __syncwarp
      __syncwarp();
      xz = xs + (live ? ci : 0) * xss + zl * d.Tin;
    }
    __nv_bfloat16* hb = h + ((static_cast<long long>(b) * d.C * plane + xy) * d.T) * d.Z + z0;
    for (int t = 0; t < d.T; ++t) {
      float v[ZL];
      if (live) lift_many_inner<TIn, ZL, kRegs>(xz, xr, d.Tin, sW1 + t * d.Tin, sb1[t], v);
#pragma unroll
      for (int k = 0; k < ZL / 2; ++k)
        sa1[warp][ci][zl / 2 + k] = live ? gelu_h2(h2_from_f32(v[2 * k], v[2 * k + 1])) : __float2half2_rn(0.f);
      __syncwarp();
      for (int c = lane; c < d.C; c += 32) {
        __half2 acc[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) acc[k] = sb2[c];
#pragma unroll
        for (int j = 0; j < CINP; ++j) {
          const uint4 a = *reinterpret_cast<const uint4*>(&sa1[warp][j][0]);
          const __half2 w = sW2[j * kLiftManyMaxC + c];
          acc[0] = __hfma2(w, h2_of_bits(a.x), acc[0]);
          acc[1] = __hfma2(w, h2_of_bits(a.y), acc[1]);
          acc[2] = __hfma2(w, h2_of_bits(a.z), acc[2]);
          acc[3] = __hfma2(w, h2_of_bits(a.w), acc[3]);
        }
        uint32_t o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) o[k] = h2_to_bf16x2(gelu_h2(acc[k]));
        *reinterpret_cast<uint4*>(hb + c * hc_stride + static_cast<long long>(t) * d.Z) = make_uint4(o[0], o[1], o[2], o[3]);
      }
      __syncwarp();
    }
  }
}

// Backward of lift_fwd_many_kernel: the same outputs as lift_bwd_kernel.  Per t, after the time lift:
//   channels   : lane c recomputes pre2 (packed fp16, as the forward), forms dv = dh * gelu'(pre2) in fp32, adds its
//                db2[c] and dW2[c, :] = sum_z dv a1 partials to registers held over the whole loop (2 x CINP) and
//                writes dv to the warp's [C][8] fp32 tile;
//   input side : lane (ci, z part) forms da1 = W2^T dv from the tile (fp32 W2), e = da1 * gelu'(pre1), the time sums
//                db1[t], dW1[t, :] (warp sums) and, with kDx, its own dx values: Tin == 1 keeps them in registers
//                over t, otherwise the first t stores and later t add (read-modify-write of the lane's own values).
// Everything the loss gradient multiplies is fp32; the GELU' evaluations are packed fp16.  W1 / b1 and their
// gradient sums take dynamic shared memory (2 * (T * Tin + T) floats).
template <typename TIn, int CINP, bool kRegs, bool kDx>
__global__ void __launch_bounds__(32 * kLiftManyWarps, (CINP == 8 ? 4 : 3))        // 16 channels: more live values, no spills
lift_bwd_many_kernel(const TIn* __restrict__ x, const float* __restrict__ W1, const float* __restrict__ b1,
                     const float* __restrict__ W2, const float* __restrict__ b2,
                     const __nv_bfloat16* __restrict__ dh, float* __restrict__ gW1, float* __restrict__ gb1,
                     float* __restrict__ gW2, float* __restrict__ gb2, LiftDims d, float* __restrict__ dx) {
  using L = LiftManyLanes<CINP>;
  constexpr int ZL = L::ZL, kWarps = kLiftManyWarps, kU = kLiftManyMaxC / 32;
  extern __shared__ float dsm[];                                       // W1, b1, their sums; then the x slices
  __shared__ float sW2f[kLiftManyMaxC * CINP];                         // [C][CINP] fp32, zero beyond Cin
  __shared__ __half2 sW2[CINP * kLiftManyMaxC];                        // the same, packed fp16, [CINP][C]
  __shared__ __half2 sb2[kLiftManyMaxC];
  __shared__ __align__(16) __half2 sa1[kWarps][CINP][4];
  __shared__ __align__(16) float sdv[kWarps][kLiftManyMaxC][8];      // dv of the warp's item at one t
  const int nw = d.T * d.Tin + d.T;
  float* sW1 = dsm;
  float* sb1 = sW1 + d.T * d.Tin;
  float* gsW1 = dsm + nw;
  float* gsb1 = gsW1 + d.T * d.Tin;
  for (int i = threadIdx.x; i < nw; i += blockDim.x) { dsm[i] = i < d.T * d.Tin ? W1[i] : b1[i - d.T * d.Tin]; gsW1[i] = 0.f; }
  for (int i = threadIdx.x; i < d.C * CINP; i += blockDim.x) {
    const int c = i / CINP, ci = i % CINP;
    sW2f[i] = ci < d.Cin ? W2[c * d.Cin + ci] : 0.f;
    sW2[ci * kLiftManyMaxC + c] = __float2half2_rn(sW2f[i]);
  }
  for (int i = threadIdx.x; i < d.C; i += blockDim.x) sb2[i] = __float2half2_rn(b2[i]);
  __syncthreads();

  float accb2[kU], accW2[kU][CINP];
#pragma unroll
  for (int u = 0; u < kU; ++u) {
    accb2[u] = 0.f;
#pragma unroll
    for (int j = 0; j < CINP; ++j) accW2[u][j] = 0.f;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ci = lane / L::kParts, zl = (lane % L::kParts) * ZL;
  const bool live = ci < d.Cin;
  const int zv = d.Z >> 3;
  const long long plane = static_cast<long long>(d.X) * d.Y;
  const long long nitems = static_cast<long long>(d.B) * plane * zv;
  const long long hc_stride = plane * d.T * d.Z;
  for (long long idx = blockIdx.x * static_cast<long long>(kWarps) + warp; idx < nitems;
       idx += static_cast<long long>(gridDim.x) * kWarps) {              // warp-uniform
    const int z0 = static_cast<int>(idx % zv) * 8;
    const long long xy = (idx / zv) % plane;
    const int b = static_cast<int>(idx / (zv * plane));
    const long long xoff = ((((static_cast<long long>(b) * d.Cin) + (live ? ci : 0)) * plane + xy) * d.Z + z0 + zl) * d.Tin;
    const TIn* xz;
    float xr[ZL];
    if (kRegs) {
      xz = x + xoff;
      if (live) lift_many_load<TIn, ZL>(xz, 1, xr);
    } else {
      const int xss = lift_many_xs_stride<TIn>(d.Tin);
      TIn* xs = reinterpret_cast<TIn*>(dsm + (2 * nw + 3) / 4 * 4) + warp * d.Cin * xss;
      __syncwarp();                                                    // the previous item's last reads of xs
      lift_many_stage<TIn>(x + (xoff - (live ? ci : 0) * plane * d.Z * d.Tin - zl * d.Tin), plane * d.Z * d.Tin,
                           d.Cin, d.Tin, lane, xs);
      __syncwarp();
      xz = xs + (live ? ci : 0) * xss + zl * d.Tin;
    }
    const __nv_bfloat16* gb = dh + ((static_cast<long long>(b) * d.C * plane + xy) * d.T) * d.Z + z0;
    float dxr[ZL];
#pragma unroll
    for (int z = 0; z < ZL; ++z) dxr[z] = 0.f;
    for (int t = 0; t < d.T; ++t) {
      float g1[ZL];
      {
        float v[ZL];
        if (live) lift_many_inner<TIn, ZL, kRegs>(xz, xr, d.Tin, sW1 + t * d.Tin, sb1[t], v);
#pragma unroll
        for (int k = 0; k < ZL / 2; ++k) {
          GeluH2 vg;
          vg.value = vg.grad = __float2half2_rn(0.f);
          if (live) vg = gelu_vg_h2(h2_from_f32(v[2 * k], v[2 * k + 1]));
          sa1[warp][ci][zl / 2 + k] = vg.value;
          const float2 gv = __half22float2(vg.grad);
          g1[2 * k] = gv.x; g1[2 * k + 1] = gv.y;
        }
      }
      __syncwarp();
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const int c = lane + 32 * u;
        if (c < d.C) {
          const uint4 gw = *reinterpret_cast<const uint4*>(gb + c * hc_stride + static_cast<long long>(t) * d.Z);
          __half2 acc[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) acc[k] = sb2[c];
#pragma unroll
          for (int j = 0; j < CINP; ++j) {
            const uint4 a = *reinterpret_cast<const uint4*>(&sa1[warp][j][0]);
            const __half2 w = sW2[j * kLiftManyMaxC + c];
            acc[0] = __hfma2(w, h2_of_bits(a.x), acc[0]);
            acc[1] = __hfma2(w, h2_of_bits(a.y), acc[1]);
            acc[2] = __hfma2(w, h2_of_bits(a.z), acc[2]);
            acc[3] = __hfma2(w, h2_of_bits(a.w), acc[3]);
          }
          const uint32_t gws[4] = {gw.x, gw.y, gw.z, gw.w};
          float dv[8];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const float2 gr = __half22float2(gelu_vg_h2(acc[k]).grad);
            const float2 g = unpack_bf16x2(gws[k]);
            dv[2 * k] = g.x * gr.x; dv[2 * k + 1] = g.y * gr.y;
          }
          float sb = 0.f;
#pragma unroll
          for (int z = 0; z < 8; ++z) sb += dv[z];
          accb2[u] += sb;
#pragma unroll
          for (int j = 0; j < CINP; ++j) {
            const uint4 a = *reinterpret_cast<const uint4*>(&sa1[warp][j][0]);
            const uint32_t aw[4] = {a.x, a.y, a.z, a.w};
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const float2 af = __half22float2(h2_of_bits(aw[k]));
              s = fmaf(dv[2 * k], af.x, s);
              s = fmaf(dv[2 * k + 1], af.y, s);
            }
            accW2[u][j] += s;
          }
          float4* dst = reinterpret_cast<float4*>(&sdv[warp][c][0]);
          dst[0] = make_float4(dv[0], dv[1], dv[2], dv[3]);
          dst[1] = make_float4(dv[4], dv[5], dv[6], dv[7]);
        }
      }
      __syncwarp();
      float e[ZL];
#pragma unroll
      for (int z = 0; z < ZL; ++z) e[z] = 0.f;
      if (live) {
        for (int c = 0; c < d.C; ++c) {
          const float w = sW2f[c * CINP + ci];
#pragma unroll
          for (int z = 0; z < ZL; ++z) e[z] = fmaf(w, sdv[warp][c][zl + z], e[z]);
        }
      }
      float sb1v = 0.f;
#pragma unroll
      for (int z = 0; z < ZL; ++z) { e[z] *= g1[z]; sb1v += e[z]; }
      sb1v = warp_sum(sb1v);
      if (lane == 0) atomicAdd(&gsb1[t], sb1v);
      if (kRegs) {
        float s = 0.f;
#pragma unroll
        for (int z = 0; z < ZL; ++z) s = fmaf(e[z], live ? xr[z] : 0.f, s);
        s = warp_sum(s);
        if (lane == 0) atomicAdd(&gsW1[t], s);
        if (kDx) {
          const float w = sW1[t];
#pragma unroll
          for (int z = 0; z < ZL; ++z) dxr[z] = fmaf(w, e[z], dxr[z]);
        }
      } else {
        for (int ti = 0; ti < d.Tin; ++ti) {
          float xv[ZL];
          if (live) lift_many_load<TIn, ZL>(xz + ti, d.Tin, xv);
          float s = 0.f;
#pragma unroll
          for (int z = 0; z < ZL; ++z) s = fmaf(e[z], live ? xv[z] : 0.f, s);
          s = warp_sum(s);
          if (lane == 0) atomicAdd(&gsW1[t * d.Tin + ti], s);
          if (kDx && live) {
            const float w = sW1[t * d.Tin + ti];
            float* p = dx + xoff + ti;
#pragma unroll
            for (int z = 0; z < ZL; ++z) p[z * d.Tin] = t == 0 ? w * e[z] : fmaf(w, e[z], p[z * d.Tin]);
          }
        }
      }
    }
    if (kDx && kRegs && live) {
#pragma unroll
      for (int z = 0; z < ZL; z += 2) *reinterpret_cast<float2*>(dx + xoff + z) = make_float2(dxr[z], dxr[z + 1]);
    }
  }
  // channel sums: lane c holds the partials of channels c and c + 32 (no two lanes of a warp share a channel)
  __syncthreads();
  float* gsW2 = &sdv[0][0][0];                                         // [C][CINP] + [C], the dv tiles are done
  for (int i = threadIdx.x; i < d.C * CINP + d.C; i += blockDim.x) gsW2[i] = 0.f;
  __syncthreads();
#pragma unroll
  for (int u = 0; u < kU; ++u) {
    const int c = lane + 32 * u;
    if (c < d.C) {
      atomicAdd(&gsW2[d.C * CINP + c], accb2[u]);
#pragma unroll
      for (int j = 0; j < CINP; ++j) atomicAdd(&gsW2[c * CINP + j], accW2[u][j]);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < d.T * d.Tin; i += blockDim.x) atomicAdd(&gW1[i], gsW1[i]);
  for (int i = threadIdx.x; i < d.T; i += blockDim.x) atomicAdd(&gb1[i], gsb1[i]);
  for (int i = threadIdx.x; i < d.C * d.Cin; i += blockDim.x) atomicAdd(&gW2[i], gsW2[(i / d.Cin) * CINP + i % d.Cin]);
  for (int i = threadIdx.x; i < d.C; i += blockDim.x) atomicAdd(&gb2[i], gsW2[d.C * CINP + i]);
}

// ------------------------------------------------------------------------------------------
// bypass conv + GELU
// ------------------------------------------------------------------------------------------
// Each thread owns 2 consecutive z of one (b, x, y, t) and all C channels.
// spec_pre: in = spectral branch, out (in place) = pre-activation (kept for the backward).
template <int C, bool kCL>
__global__ void __launch_bounds__(128)
bypass_gelu_fwd_kernel(const __nv_bfloat16* __restrict__ h, __nv_bfloat16* __restrict__ spec_pre,
                       const float* __restrict__ W, __nv_bfloat16* __restrict__ out,
                       __nv_bfloat16* __restrict__ out_cl, int cl_pitch, int B, long long S, int save_pre) {
  __shared__ __align__(16) float sW[C * C];
  for (int i = threadIdx.x; i < C * C; i += blockDim.x) sW[i] = W[i];
  __syncthreads();
  const long long S2 = S >> 1;                       // position pairs per channel
  const long long total = static_cast<long long>(B) * S2;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long b = idx / S2, p2 = idx % S2;
    const long long base = b * C * S + 2 * p2;
    float h0[C], h1[C];
#pragma unroll
    for (int i = 0; i < C; ++i) {
      const float2 v = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(h + base + i * S));
      h0[i] = v.x; h1[i] = v.y;
    }
    // channels-last rows (for the projection head) are assembled in registers and written as
    // 8-byte vectors: two rows of cl_pitch bf16 per thread
    uint32_t cl0[kCL ? C / 2 + 1 : 1], cl1[kCL ? C / 2 + 1 : 1];
    // all spectral-branch values are fetched up front: with few resident warps the loads
    // must overlap each other, not the dependent FMA chains
    uint32_t sp[C];
#pragma unroll
    for (int o = 0; o < C; ++o) sp[o] = *reinterpret_cast<const uint32_t*>(spec_pre + base + o * S);
#pragma unroll
    for (int o = 0; o < C; ++o) {
      const float2 s = unpack_bf16x2(sp[o]);
      float a0 = s.x, a1 = s.y;
#pragma unroll
      for (int i = 0; i < C; ++i) {
        const float w = sW[o * C + i];
        a0 = fmaf(w, h0[i], a0);
        a1 = fmaf(w, h1[i], a1);
      }
      if (save_pre) *reinterpret_cast<uint32_t*>(spec_pre + base + o * S) = pack_bf16x2(a0, a1);
      const float y0 = gelu_erf(a0), y1 = gelu_erf(a1);
      if (out) *reinterpret_cast<uint32_t*>(out + base + o * S) = pack_bf16x2(y0, y1);
      if (kCL) {
        // even channel: low half, odd channel: high half of the packed word
        if ((o & 1) == 0) {
          cl0[o >> 1] = __bfloat16_as_ushort(__float2bfloat16(y0));
          cl1[o >> 1] = __bfloat16_as_ushort(__float2bfloat16(y1));
        } else {
          cl0[o >> 1] |= static_cast<uint32_t>(__bfloat16_as_ushort(__float2bfloat16(y0))) << 16;
          cl1[o >> 1] |= static_cast<uint32_t>(__bfloat16_as_ushort(__float2bfloat16(y1))) << 16;
        }
      }
    }
    if (kCL) {
      static_assert(C % 4 == 0, "channels-last rows are written as 8-byte vectors");
      __nv_bfloat16* r0 = out_cl + (b * S + 2 * p2) * cl_pitch;
      __nv_bfloat16* r1 = r0 + cl_pitch;
#pragma unroll
      for (int w2 = 0; w2 < C / 4; ++w2) {
        reinterpret_cast<uint2*>(r0)[w2] = make_uint2(cl0[2 * w2], cl0[2 * w2 + 1]);
        reinterpret_cast<uint2*>(r1)[w2] = make_uint2(cl1[2 * w2], cl1[2 * w2 + 1]);
      }
    }
  }
}

// dpre = dout * gelu'(pre);  dhb = W^T dpre.  dout may come channel-major (internal layout)
// or channels-last (from the projection head).
template <int C>
__global__ void __launch_bounds__(256)
bypass_gelu_bwd_kernel(const __nv_bfloat16* __restrict__ dout, const __nv_bfloat16* __restrict__ dout_cl,
                       int cl_pitch, const __nv_bfloat16* __restrict__ pre, const float* __restrict__ W,
                       __nv_bfloat16* __restrict__ dpre, __nv_bfloat16* __restrict__ dhb, int B, long long S) {
  __shared__ __align__(16) float sW[C * C];
  for (int i = threadIdx.x; i < C * C; i += blockDim.x) sW[i] = W[i];
  __syncthreads();
  const long long S2 = S >> 1;
  const long long total = static_cast<long long>(B) * S2;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long b = idx / S2, p2 = idx % S2;
    const long long base = b * C * S + 2 * p2;
    float g0[C], g1[C];
#pragma unroll
    for (int o = 0; o < C; ++o) {
      float2 g;
      if (dout_cl) {
        const long long r = (b * S + 2 * p2) * cl_pitch + o;
        g.x = __bfloat162float(dout_cl[r]);
        g.y = __bfloat162float(dout_cl[r + cl_pitch]);
      } else {
        g = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(dout + base + o * S));
      }
      const float2 p = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(pre + base + o * S));
      g0[o] = g.x * gelu_erf_grad(p.x);
      g1[o] = g.y * gelu_erf_grad(p.y);
      *reinterpret_cast<uint32_t*>(dpre + base + o * S) = pack_bf16x2(g0[o], g1[o]);
    }
#pragma unroll 4
    for (int i = 0; i < C; ++i) {
      float a0 = 0.f, a1 = 0.f;
#pragma unroll
      for (int o = 0; o < C; ++o) {
        const float w = sW[o * C + i];
        a0 = fmaf(w, g0[o], a0);
        a1 = fmaf(w, g1[o], a1);
      }
      *reinterpret_cast<uint32_t*>(dhb + base + i * S) = pack_bf16x2(a0, a1);
    }
  }
}

__global__ void gelu_probe_kernel(const float* __restrict__ x, float* __restrict__ y, float* __restrict__ dy, long long n) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i < n) { y[i] = gelu_erf(x[i]); dy[i] = gelu_erf_grad(x[i]); }
}

// the packed fp16 GELU the fused kernels use (pairs of adjacent elements)
__global__ void gelu_probe_h2_kernel(const float* __restrict__ x, float* __restrict__ y, float* __restrict__ dy, long long n) {
  const long long i = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) * 2;
  if (i + 1 < n) {
    const GeluH2 r = gelu_vg_h2(h2_from_f32(x[i], x[i + 1]));
    const float2 v = __half22float2(r.value), g = __half22float2(r.grad);
    const float2 v2 = __half22float2(gelu_h2(h2_from_f32(x[i], x[i + 1])));
    y[i] = v.x; y[i + 1] = v2.y; dy[i] = g.x; dy[i + 1] = g.y;
  }
}

// Generic strided permutation of 32-bit words (one (re, im) bf16 pair each): dst is walked in its
// own mixed-radix order (innermost digit first), the same digits address src through src_strides.
// Used on the receiving side of the fused pencil transposes: peers deposit their contribution as
// one long contiguous run per source rank (NVLink-friendly), this kernel interleaves the runs into
// the K-major layout the next GEMM stage reads.  The tensors are the *truncated* spectra, a few MB.
struct PermuteDesc {
  int nd;
  unsigned size[6];
  unsigned long long magic[6];
  int shift[6];
  long long sstr[6];
  long long dstr[6];
};

// V = words per thread access (the innermost digit is contiguous on both sides and a multiple of V);
// digits by magic-number division (n < 2^31); kUnroll independent loads in flight per thread.
template <typename Vec, int kUnroll>
__global__ void __launch_bounds__(256)
permute_vec_kernel(const Vec* __restrict__ src, Vec* __restrict__ dst, unsigned total, PermuteDesc d) {
  const unsigned stride = gridDim.x * blockDim.x;
  for (unsigned i0 = blockIdx.x * blockDim.x + threadIdx.x; i0 < total; i0 += stride * kUnroll) {
    Vec v[kUnroll];
    long long dof[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      unsigned r = i0 + u * stride;
      long long so = 0;
      dof[u] = -1;
      if (r < total) {
        dof[u] = 0;
#pragma unroll
        for (int l = 0; l < 6; ++l) {
          if (l < d.nd) {
            unsigned dig = r;
            if (l != d.nd - 1) {
              const unsigned q = static_cast<unsigned>((static_cast<unsigned long long>(r) * d.magic[l]) >> d.shift[l]);
              dig = r - q * d.size[l];
              r = q;
            }
            so += static_cast<long long>(dig) * d.sstr[l];
            dof[u] += static_cast<long long>(dig) * d.dstr[l];
          }
        }
        v[u] = src[so];
      }
    }
#pragma unroll
    for (int u = 0; u < kUnroll; ++u)
      if (dof[u] >= 0) dst[dof[u]] = v[u];
  }
}

int grid_for(long long work_items, int threads, int num_sms, int per_sm) {
  long long blocks = (work_items + threads - 1) / threads;
  const long long cap = static_cast<long long>(num_sms) * per_sm;
  return static_cast<int>(blocks < cap ? (blocks > 0 ? blocks : 1) : cap);
}

}  // namespace

// ------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------
const char* permute_u32(const void* src, void* dst, int nd, const int* size, const long long* sstr,
                        const long long* dstr, int num_sms, cudaStream_t s) {
  if (nd < 1 || nd > 6) return "permute_u32: 1..6 digits";
  // widest vector the innermost (contiguous) digit allows
  int V = 1;
  if (sstr[0] == 1 && dstr[0] == 1) {
    for (int cand = 4; cand > 1 && V == 1; cand >>= 1) {
      bool ok = size[0] % cand == 0 && reinterpret_cast<uintptr_t>(src) % (4 * cand) == 0 &&
                reinterpret_cast<uintptr_t>(dst) % (4 * cand) == 0;
      for (int i = 1; i < nd; ++i) ok = ok && sstr[i] % cand == 0 && dstr[i] % cand == 0;
      if (ok) V = cand;
    }
  }
  PermuteDesc d;
  d.nd = nd;
  long long total = 1;
  for (int i = 0; i < 6; ++i) {
    long long sz = i < nd ? size[i] : 1;
    if (sz <= 0) return nullptr;
    if (i == 0) sz /= V;
    d.size[i] = static_cast<unsigned>(sz);
    d.sstr[i] = i < nd ? (i == 0 ? sstr[i] : sstr[i] / V) : 0;
    d.dstr[i] = i < nd ? (i == 0 ? dstr[i] : dstr[i] / V) : 0;
    int sh = 0;
    while ((1ull << sh) < static_cast<unsigned long long>(sz)) ++sh;
    d.magic[i] = ((1ull << (31 + sh)) / static_cast<unsigned long long>(sz)) + 1;
    d.shift[i] = 31 + sh;
    total *= sz;
  }
  if (total >= (1ll << 31)) return "permute_u32: tensor too large for one launch";
  constexpr int kUnroll = 4;
  long long blocks = (total + 256 * kUnroll - 1) / (256 * kUnroll);
  const long long cap = static_cast<long long>(num_sms) * 8;
  if (blocks > cap) blocks = cap;
  const unsigned tot = static_cast<unsigned>(total);
  const int g = static_cast<int>(blocks);
  if (V == 4)
    permute_vec_kernel<uint4, kUnroll><<<g, 256, 0, s>>>(static_cast<const uint4*>(src), static_cast<uint4*>(dst), tot, d);
  else if (V == 2)
    permute_vec_kernel<uint2, kUnroll><<<g, 256, 0, s>>>(static_cast<const uint2*>(src), static_cast<uint2*>(dst), tot, d);
  else
    permute_vec_kernel<uint32_t, kUnroll><<<g, 256, 0, s>>>(static_cast<const uint32_t*>(src),
                                                            static_cast<uint32_t*>(dst), tot, d);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

const char* gelu_probe_h2(const float* x, float* y, float* dy, long long n, cudaStream_t s) {
  gelu_probe_h2_kernel<<<static_cast<int>((n / 2 + 255) / 256), 256, 0, s>>>(x, y, dy, n);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

const char* gelu_probe(const float* x, float* y, float* dy, long long n, cudaStream_t s) {
  gelu_probe_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, s>>>(x, y, dy, n);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

static const char* lift_check(const LiftDims& d) {
  if (d.Z % 8) return "lift: Z must be a multiple of 8";
  if (d.Cin < 1 || d.Cin > 16) return "lift: supported input channel counts are 1..16";
  if (d.Tin < 1 || d.Tin > kLiftMaxTin) return "lift: 1 <= Tin <= 64";
  if (d.C > 64) return "lift: C <= 64";
  if (d.T * d.Tin + d.T + 2 * (d.C * d.Cin + d.C) > kLiftMaxW) return "lift: weights exceed shared memory budget";
  return nullptr;
}

// 5 <= Cin <= 16: one warp per item (lift_fwd_many_kernel), channels padded to 8 or 16
// bytes of the per-warp x slices of one block (Tin > 1; up to 129 KB at Cin = 16, Tin = 64 in fp32)
template <typename TIn>
static size_t lift_many_xs_bytes(int Cin, int Tin) {
  return Tin == 1 ? 0 : static_cast<size_t>(kLiftManyWarps) * Cin * lift_many_xs_stride<TIn>(Tin) * sizeof(TIn);
}

// opts a kernel into the largest dynamic shared memory its launches ask for (once per instantiation)
template <typename K>
static const char* lift_many_allow_smem(K kern, bool& done, size_t bytes) {
  if (done) return nullptr;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes));
  if (e != cudaSuccess) return cudaGetErrorString(e);
  done = true;
  return nullptr;
}

template <typename TIn, int CINP, bool kRegs>
static const char* lift_fwd_many_launch(const void* x, const float* W1, const float* b1, const float* W2,
                                        const float* b2, void* h, LiftDims d, int grid, cudaStream_t s) {
  auto kern = lift_fwd_many_kernel<TIn, CINP, kRegs>;
  static bool attr = false;
  if (const char* e = lift_many_allow_smem(kern, attr, lift_many_xs_bytes<TIn>(16, kLiftMaxTin))) return e;
  kern<<<grid, 32 * kLiftManyWarps, lift_many_xs_bytes<TIn>(d.Cin, d.Tin), s>>>(
      static_cast<const TIn*>(x), W1, b1, W2, b2, static_cast<__nv_bfloat16*>(h), d);
  return nullptr;
}

static const char* lift_fwd_many(const void* x, int x_is_bf16, const float* W1, const float* b1, const float* W2,
                                 const float* b2, void* h, LiftDims d, int num_sms, cudaStream_t s) {
  const long long nitems = static_cast<long long>(d.B) * d.X * d.Y * (d.Z / 8);
  const int grid = grid_for(32 * nitems, 32 * kLiftManyWarps, num_sms, 8);
  const bool regs = d.Tin == 1;
#define DFNO_LIFT_FWD_MANY(T_, CINP_)                                                          \
  (regs ? lift_fwd_many_launch<T_, CINP_, true>(x, W1, b1, W2, b2, h, d, grid, s)               \
        : lift_fwd_many_launch<T_, CINP_, false>(x, W1, b1, W2, b2, h, d, grid, s))
  const char* err;
  if (x_is_bf16)
    err = d.Cin <= 8 ? DFNO_LIFT_FWD_MANY(__nv_bfloat16, 8) : DFNO_LIFT_FWD_MANY(__nv_bfloat16, 16);
  else
    err = d.Cin <= 8 ? DFNO_LIFT_FWD_MANY(float, 8) : DFNO_LIFT_FWD_MANY(float, 16);
#undef DFNO_LIFT_FWD_MANY
  if (err) return err;
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

template <typename TIn, int CINP, bool kRegs, bool kDx>
static const char* lift_bwd_many_launch(const void* x, const float* W1, const float* b1, const float* W2,
                                        const float* b2, const void* dh, float* gW1, float* gb1, float* gW2,
                                        float* gb2, float* dx, LiftDims d, int grid, cudaStream_t s) {
  auto kern = lift_bwd_many_kernel<TIn, CINP, kRegs, kDx>;
  static bool attr = false;                     // W1, b1 and their sums (up to 2 * kLiftMaxW floats), then x slices
  if (const char* e = lift_many_allow_smem(kern, attr, 2 * kLiftMaxW * sizeof(float) +
                                                           lift_many_xs_bytes<TIn>(16, kLiftMaxTin)))
    return e;
  const size_t smem = (2 * static_cast<size_t>(d.T * d.Tin + d.T) + 3) / 4 * 4 * sizeof(float) +
                      lift_many_xs_bytes<TIn>(d.Cin, d.Tin);
  kern<<<grid, 32 * kLiftManyWarps, smem, s>>>(static_cast<const TIn*>(x), W1, b1, W2, b2, static_cast<const __nv_bfloat16*>(dh), gW1,
                               gb1, gW2, gb2, d, dx);
  return nullptr;
}

// 5 <= Cin <= 16: one warp per item (lift_bwd_many_kernel)
static const char* lift_bwd_many(const void* x, int x_is_bf16, const float* W1, const float* b1, const float* W2,
                                 const float* b2, const void* dh, float* gW1, float* gb1, float* gW2, float* gb2,
                                 float* dx, LiftDims d, int num_sms, cudaStream_t s) {
  const long long nitems = static_cast<long long>(d.B) * d.X * d.Y * (d.Z / 8);
  const int grid = grid_for(32 * nitems, 32 * kLiftManyWarps, num_sms, 8);
  const bool regs = d.Tin == 1;
#define DFNO_LIFT_BWD_MANY3(T_, CINP_, R_, DX_) \
  lift_bwd_many_launch<T_, CINP_, R_, DX_>(x, W1, b1, W2, b2, dh, gW1, gb1, gW2, gb2, dx, d, grid, s)
#define DFNO_LIFT_BWD_MANY2(T_, CINP_, R_) \
  (dx ? DFNO_LIFT_BWD_MANY3(T_, CINP_, R_, true) : DFNO_LIFT_BWD_MANY3(T_, CINP_, R_, false))
#define DFNO_LIFT_BWD_MANY1(T_, CINP_) \
  (regs ? DFNO_LIFT_BWD_MANY2(T_, CINP_, true) : DFNO_LIFT_BWD_MANY2(T_, CINP_, false))
  const char* err;
  if (x_is_bf16)
    err = d.Cin <= 8 ? DFNO_LIFT_BWD_MANY1(__nv_bfloat16, 8) : DFNO_LIFT_BWD_MANY1(__nv_bfloat16, 16);
  else
    err = d.Cin <= 8 ? DFNO_LIFT_BWD_MANY1(float, 8) : DFNO_LIFT_BWD_MANY1(float, 16);
#undef DFNO_LIFT_BWD_MANY1
#undef DFNO_LIFT_BWD_MANY2
#undef DFNO_LIFT_BWD_MANY3
  if (err) return err;
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

const char* lift_fwd(const void* x, int x_is_bf16, const float* W1, const float* b1, const float* W2,
                     const float* b2, void* h, LiftDims d, int num_sms, cudaStream_t s) {
  if (const char* e = lift_check(d)) return e;
  if (d.Cin > 4) return lift_fwd_many(x, x_is_bf16, W1, b1, W2, b2, h, d, num_sms, s);
  const long long nitems = static_cast<long long>(d.B) * d.X * d.Y * (d.Z / 8);
  const int grid = grid_for(nitems, 256, num_sms, 4);
  const bool regs = d.Tin == 1;
#define DFNO_LIFT_FWD(T_, CIN_, R_) \
  lift_fwd_kernel<T_, CIN_, R_><<<grid, 256, 0, s>>>(static_cast<const T_*>(x), W1, b1, W2, b2, static_cast<__nv_bfloat16*>(h), d)
#define DFNO_LIFT_FWD_T(T_)                                                                         \
  switch (d.Cin) {                                                                                  \
    case 1: if (regs) DFNO_LIFT_FWD(T_, 1, true); else DFNO_LIFT_FWD(T_, 1, false); break;          \
    case 2: if (regs) DFNO_LIFT_FWD(T_, 2, true); else DFNO_LIFT_FWD(T_, 2, false); break;          \
    case 3: if (regs) DFNO_LIFT_FWD(T_, 3, true); else DFNO_LIFT_FWD(T_, 3, false); break;          \
    default: if (regs) DFNO_LIFT_FWD(T_, 4, true); else DFNO_LIFT_FWD(T_, 4, false); break;         \
  }
  if (x_is_bf16) { DFNO_LIFT_FWD_T(__nv_bfloat16) } else { DFNO_LIFT_FWD_T(float) }
#undef DFNO_LIFT_FWD_T
#undef DFNO_LIFT_FWD
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

#define DFNO_DISPATCH_C(C_, BODY)                 \
  switch (C_) {                                   \
    case 4:  { constexpr int kC = 4;  BODY; } break;  \
    case 8:  { constexpr int kC = 8;  BODY; } break;  \
    case 12: { constexpr int kC = 12; BODY; } break;  \
    case 16: { constexpr int kC = 16; BODY; } break;  \
    case 20: { constexpr int kC = 20; BODY; } break;  \
    case 24: { constexpr int kC = 24; BODY; } break;  \
    case 32: { constexpr int kC = 32; BODY; } break;  \
    default: return "unsupported channel width (supported: 4,8,12,16,20,24,32)"; \
  }

// the lift backward's widths: those of every pointwise kernel, and 48 and 64 (the wide widths of the round-2 route)
#define DFNO_LIFT_DISPATCH_C(C_, BODY)                \
  switch (C_) {                                       \
    case 48: { constexpr int kC = 48; BODY; } break;  \
    case 64: { constexpr int kC = 64; BODY; } break;  \
    default: DFNO_DISPATCH_C(C_, BODY)                \
  }

template <int C>
static const char* lift_bwd_cin(const void* x, int x_is_bf16, const float* W1, const float* b1, const float* W2,
                                const float* b2, const void* dh, float* gW1, float* gb1, float* gW2, float* gb2,
                                float* dx, LiftDims d, int grid, bool regs, cudaStream_t s) {
#define DFNO_LIFT_BWD3(T_, CIN_, R_, DX_)                                                                         \
  lift_bwd_kernel<T_, C, CIN_, R_, DX_><<<grid, 128, 0, s>>>(static_cast<const T_*>(x), W1, b1, W2, b2,           \
                                                             static_cast<const __nv_bfloat16*>(dh), gW1, gb1, gW2, \
                                                             gb2, d, dx)
#define DFNO_LIFT_BWD2(T_, CIN_, R_) \
  if (dx) DFNO_LIFT_BWD3(T_, CIN_, R_, true); else DFNO_LIFT_BWD3(T_, CIN_, R_, false)
#define DFNO_LIFT_BWD(CIN_)                                                                    \
  if (x_is_bf16) { if (regs) { DFNO_LIFT_BWD2(__nv_bfloat16, CIN_, true); } else { DFNO_LIFT_BWD2(__nv_bfloat16, CIN_, false); } } \
  else { if (regs) { DFNO_LIFT_BWD2(float, CIN_, true); } else { DFNO_LIFT_BWD2(float, CIN_, false); } }
  switch (d.Cin) {
    case 1: DFNO_LIFT_BWD(1); break;
    case 2: DFNO_LIFT_BWD(2); break;
    case 3: DFNO_LIFT_BWD(3); break;
    case 4: DFNO_LIFT_BWD(4); break;
    default: return "lift_bwd: supported input channel counts are 1..4";
  }
#undef DFNO_LIFT_BWD
#undef DFNO_LIFT_BWD2
#undef DFNO_LIFT_BWD3
  return nullptr;
}

const char* lift_bwd(const void* x, int x_is_bf16, const float* W1, const float* b1, const float* W2,
                     const float* b2, const void* dh, float* gW1, float* gb1, float* gW2, float* gb2, float* dx,
                     LiftDims d, int num_sms, cudaStream_t s) {
  if (const char* e = lift_check(d)) return e;
  if (dx && reinterpret_cast<uintptr_t>(dx) % 8) return "lift_bwd: dx must be 8-byte aligned";
  if (d.Cin > 4) return lift_bwd_many(x, x_is_bf16, W1, b1, W2, b2, dh, gW1, gb1, gW2, gb2, dx, d, num_sms, s);
  const long long nitems = static_cast<long long>(d.B) * d.X * d.Y * (d.Z / 8);
  const int split = d.C > 32 ? 8 : 4;                                 // lanes per item (see lift_bwd_kernel)
  const int grid = grid_for(split * nitems, 128, num_sms, 4);
  const bool regs = d.Tin == 1;
  const char* err = nullptr;
  DFNO_LIFT_DISPATCH_C(d.C, (err = lift_bwd_cin<kC>(x, x_is_bf16, W1, b1, W2, b2, dh, gW1, gb1, gW2, gb2, dx, d, grid, regs,
                                               s)));
  if (err) return err;
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

const char* bypass_gelu_fwd(const void* h, void* spec_pre, const float* W, void* out, void* out_cl, int cl_pitch,
                            int B, int C, long long S, int save_pre, int num_sms, cudaStream_t s) {
  if (S % 2) return "spatial size per channel must be even";
  const int grid = grid_for(static_cast<long long>(B) * (S / 2), 128, num_sms, 16);
  if (out_cl) {
    DFNO_DISPATCH_C(C, (bypass_gelu_fwd_kernel<kC, true><<<grid, 128, 0, s>>>(
                           static_cast<const __nv_bfloat16*>(h), static_cast<__nv_bfloat16*>(spec_pre), W,
                           static_cast<__nv_bfloat16*>(out), static_cast<__nv_bfloat16*>(out_cl), cl_pitch, B, S,
                           save_pre)));
  } else {
    DFNO_DISPATCH_C(C, (bypass_gelu_fwd_kernel<kC, false><<<grid, 128, 0, s>>>(
                           static_cast<const __nv_bfloat16*>(h), static_cast<__nv_bfloat16*>(spec_pre), W,
                           static_cast<__nv_bfloat16*>(out), nullptr, cl_pitch, B, S, save_pre)));
  }
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

const char* bypass_gelu_bwd(const void* dout, const void* dout_cl, int cl_pitch, const void* pre, const float* W,
                            void* dpre, void* dhb, int B, int C, long long S, int num_sms, cudaStream_t s) {
  if (S % 2) return "spatial size per channel must be even";
  const int grid = grid_for(static_cast<long long>(B) * (S / 2), 256, num_sms, 4);
  DFNO_DISPATCH_C(C, (bypass_gelu_bwd_kernel<kC><<<grid, 256, 0, s>>>(
                         static_cast<const __nv_bfloat16*>(dout), static_cast<const __nv_bfloat16*>(dout_cl),
                         cl_pitch, static_cast<const __nv_bfloat16*>(pre), W, static_cast<__nv_bfloat16*>(dpre),
                         static_cast<__nv_bfloat16*>(dhb), B, S)));
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

}  // namespace dfno
