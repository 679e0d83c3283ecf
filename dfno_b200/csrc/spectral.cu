// spectral.cu -- per-mode complex channel mixing of the truncated spectrum (SURVEY.md K8/K9,
// reference dfno.py:269-271):   Y[b, o, q] = sum_i X[b, i, q] * R[i, o, q]
//
// q runs over this rank's slab of retained modes (all corners at once: the low/high corners
// tile the slab, so there is no per-corner loop and no zero-initialised output).  With the
// batch sizes FNOs train at (B = 1..4) every mode owns a distinct C x C matrix that is used
// once: the op is bound by streaming the fp32 weights (113-442 MB per block), i.e. a
// bandwidth problem for plain FMA units with fully coalesced 8-byte loads, not a tensor-core
// problem.  The backward makes ONE pass over R and produces both dX and dR (dX alone for frozen weights).
#include "sm90_ptx.cuh"
#include "kernels.h"

namespace dfno {
namespace {

// Thread (q, g): mode q and the g-th quarter of the output (forward) / input (backward) channels, so a slab of
// Q modes runs 4 Q threads: with the mode slab split over 8 GPUs a rank holds only ~17 k modes, and one thread
// per mode (400 dependent weight loads each) left most of the machine idle.  threadIdx.x walks q: every weight
// load of a warp is one contiguous 256-byte run.
constexpr int kMixSplit = 4;
constexpr int kMixQ = 64;                      // modes per block (blockDim = (64, 4))
constexpr int kMixChunk = 8;                   // channels per chunk of the wide kernels (mix_fwd_wide_kernel)

template <int C>
__global__ void __launch_bounds__(kMixQ * kMixSplit)
mix_fwd_kernel(const uint32_t* __restrict__ x, const float2* __restrict__ w, uint32_t* __restrict__ y, int B,
               long long Q) {
  constexpr int CG = C / kMixSplit;
  const int o0 = threadIdx.y * CG;
  for (long long q = blockIdx.x * static_cast<long long>(kMixQ) + threadIdx.x; q < Q;
       q += static_cast<long long>(gridDim.x) * kMixQ) {
    for (int b = 0; b < B; ++b) {
      float2 xv[C];
#pragma unroll
      for (int i = 0; i < C; ++i) xv[i] = unpack_bf16x2(x[(static_cast<long long>(b) * C + i) * Q + q]);
#pragma unroll
      for (int oo = 0; oo < CG; ++oo) {
        const int o = o0 + oo;
        float2 r[C];
#pragma unroll
        for (int i = 0; i < C; ++i) r[i] = __ldg(&w[(static_cast<long long>(i) * C + o) * Q + q]);   // C loads in flight
        float ar = 0.f, ai = 0.f;
#pragma unroll
        for (int i = 0; i < C; ++i) {
          ar = fmaf(xv[i].x, r[i].x, ar); ar = fmaf(-xv[i].y, r[i].y, ar);
          ai = fmaf(xv[i].x, r[i].y, ai); ai = fmaf(xv[i].y, r[i].x, ai);
        }
        y[(static_cast<long long>(b) * C + o) * Q + q] = pack_bf16x2(ar, ai);
      }
    }
  }
}

// one batch element per launch; dw (+)= conj(x) * dy ; dx = sum_o dy * conj(w)
// kDw = false (frozen weights): dx only -- no x read, no read-modify-write of dw.
template <int C, bool kDw>
__global__ void __launch_bounds__(kMixQ * kMixSplit)
mix_bwd_kernel(const uint32_t* __restrict__ x, const float2* __restrict__ w, const uint32_t* __restrict__ dy,
               uint32_t* __restrict__ dx, float2* __restrict__ dw, int accumulate, long long Q) {
  constexpr int CG = C / kMixSplit;
  const int i0 = threadIdx.y * CG;
  for (long long q = blockIdx.x * static_cast<long long>(kMixQ) + threadIdx.x; q < Q;
       q += static_cast<long long>(gridDim.x) * kMixQ) {
    float2 gv[C];
#pragma unroll
    for (int o = 0; o < C; ++o) gv[o] = unpack_bf16x2(dy[static_cast<long long>(o) * Q + q]);
#pragma unroll
    for (int ii = 0; ii < CG; ++ii) {
      const int i = i0 + ii;
      const float2 xi = kDw ? unpack_bf16x2(x[static_cast<long long>(i) * Q + q]) : make_float2(0.f, 0.f);
      float2 r[C];
#pragma unroll
      for (int o = 0; o < C; ++o) r[o] = __ldg(&w[(static_cast<long long>(i) * C + o) * Q + q]);
      float dr = 0.f, di = 0.f;
#pragma unroll
      for (int o = 0; o < C; ++o) {
        const long long widx = (static_cast<long long>(i) * C + o) * Q + q;
        // dy * conj(r)
        dr = fmaf(gv[o].x, r[o].x, dr); dr = fmaf(gv[o].y, r[o].y, dr);
        di = fmaf(gv[o].y, r[o].x, di); di = fmaf(-gv[o].x, r[o].y, di);
        if (kDw) {
          // conj(x) * dy
          float2 g;
          g.x = xi.x * gv[o].x + xi.y * gv[o].y;
          g.y = xi.x * gv[o].y - xi.y * gv[o].x;
          if (accumulate) { const float2 old = dw[widx]; g.x += old.x; g.y += old.y; }
          dw[widx] = g;
        }
      }
      dx[static_cast<long long>(i) * Q + q] = pack_bf16x2(dr, di);
    }
  }
}

// Widths above 32 (48, 64) do not fit C inputs and C weights in registers at once (4 C floats): the contraction index
// is streamed in chunks of kMixChunk, and the thread's C/4 complex sums stay in registers across chunks.  Same thread
// mapping and summation order as mix_fwd_kernel / mix_bwd_kernel.
template <int C>
__global__ void __launch_bounds__(kMixQ * kMixSplit, 2)
mix_fwd_wide_kernel(const uint32_t* __restrict__ x, const float2* __restrict__ w, uint32_t* __restrict__ y, int B,
                    long long Q) {
  constexpr int CG = C / kMixSplit;
  const int o0 = threadIdx.y * CG;
  static_assert(C % kMixChunk == 0, "whole input-channel chunks");
  for (long long q = blockIdx.x * static_cast<long long>(kMixQ) + threadIdx.x; q < Q;
       q += static_cast<long long>(gridDim.x) * kMixQ) {
    for (int b = 0; b < B; ++b) {
      float2 acc[CG];
#pragma unroll
      for (int oo = 0; oo < CG; ++oo) acc[oo] = make_float2(0.f, 0.f);
#pragma unroll 1
      for (int i0 = 0; i0 < C; i0 += kMixChunk) {
        float2 xv[kMixChunk];
#pragma unroll
        for (int i = 0; i < kMixChunk; ++i)
          xv[i] = unpack_bf16x2(x[(static_cast<long long>(b) * C + i0 + i) * Q + q]);
#pragma unroll
        for (int oo = 0; oo < CG; ++oo) {
          const int o = o0 + oo;
          float2 r[kMixChunk];
#pragma unroll
          for (int i = 0; i < kMixChunk; ++i) r[i] = __ldg(&w[(static_cast<long long>(i0 + i) * C + o) * Q + q]);
          float ar = acc[oo].x, ai = acc[oo].y;
#pragma unroll
          for (int i = 0; i < kMixChunk; ++i) {
            ar = fmaf(xv[i].x, r[i].x, ar); ar = fmaf(-xv[i].y, r[i].y, ar);
            ai = fmaf(xv[i].x, r[i].y, ai); ai = fmaf(xv[i].y, r[i].x, ai);
          }
          acc[oo] = make_float2(ar, ai);
        }
      }
#pragma unroll
      for (int oo = 0; oo < CG; ++oo)
        y[(static_cast<long long>(b) * C + o0 + oo) * Q + q] = pack_bf16x2(acc[oo].x, acc[oo].y);
    }
  }
}

template <int C, bool kDw>
__global__ void __launch_bounds__(kMixQ * kMixSplit)
mix_bwd_wide_kernel(const uint32_t* __restrict__ x, const float2* __restrict__ w, const uint32_t* __restrict__ dy,
                    uint32_t* __restrict__ dx, float2* __restrict__ dw, int accumulate, long long Q) {
  constexpr int CG = C / kMixSplit;
  const int i0 = threadIdx.y * CG;
  static_assert(C % kMixChunk == 0, "whole output-channel chunks");
  for (long long q = blockIdx.x * static_cast<long long>(kMixQ) + threadIdx.x; q < Q;
       q += static_cast<long long>(gridDim.x) * kMixQ) {
    float2 acc[CG];
#pragma unroll
    for (int ii = 0; ii < CG; ++ii) acc[ii] = make_float2(0.f, 0.f);
#pragma unroll 1
    for (int o0 = 0; o0 < C; o0 += kMixChunk) {
      float2 gv[kMixChunk];
#pragma unroll
      for (int o = 0; o < kMixChunk; ++o) gv[o] = unpack_bf16x2(dy[static_cast<long long>(o0 + o) * Q + q]);
#pragma unroll
      for (int ii = 0; ii < CG; ++ii) {
        const int i = i0 + ii;
        const float2 xi = kDw ? unpack_bf16x2(x[static_cast<long long>(i) * Q + q]) : make_float2(0.f, 0.f);
        float2 r[kMixChunk];
#pragma unroll
        for (int o = 0; o < kMixChunk; ++o) r[o] = __ldg(&w[(static_cast<long long>(i) * C + o0 + o) * Q + q]);
        float dr = acc[ii].x, di = acc[ii].y;
#pragma unroll
        for (int o = 0; o < kMixChunk; ++o) {
          const long long widx = (static_cast<long long>(i) * C + o0 + o) * Q + q;
          dr = fmaf(gv[o].x, r[o].x, dr); dr = fmaf(gv[o].y, r[o].y, dr);
          di = fmaf(gv[o].y, r[o].x, di); di = fmaf(-gv[o].x, r[o].y, di);
          if (kDw) {
            float2 g;
            g.x = xi.x * gv[o].x + xi.y * gv[o].y;
            g.y = xi.x * gv[o].y - xi.y * gv[o].x;
            if (accumulate) { const float2 old = dw[widx]; g.x += old.x; g.y += old.y; }
            dw[widx] = g;
          }
        }
        acc[ii] = make_float2(dr, di);
      }
    }
#pragma unroll
    for (int ii = 0; ii < CG; ++ii) dx[static_cast<long long>(i0 + ii) * Q + q] = pack_bf16x2(acc[ii].x, acc[ii].y);
  }
}

// the kernel of width C: the register-resident one up to 32, the streamed one above
template <int C>
void launch_mix_fwd(int grid, dim3 block, cudaStream_t s, const uint32_t* x, const float2* w, uint32_t* y, int B,
                    long long Q) {
  if constexpr (C > 32) mix_fwd_wide_kernel<C><<<grid, block, 0, s>>>(x, w, y, B, Q);
  else mix_fwd_kernel<C><<<grid, block, 0, s>>>(x, w, y, B, Q);
}
template <int C, bool kDw>
void launch_mix_bwd(int grid, dim3 block, cudaStream_t s, const uint32_t* x, const float2* w, const uint32_t* dy,
                    uint32_t* dx, float2* dw, int accumulate, long long Q) {
  if constexpr (C > 32) mix_bwd_wide_kernel<C, kDw><<<grid, block, 0, s>>>(x, w, dy, dx, dw, accumulate, Q);
  else mix_bwd_kernel<C, kDw><<<grid, block, 0, s>>>(x, w, dy, dx, dw, accumulate, Q);
}

}  // namespace

#define DFNO_MIX_DISPATCH(C_, BODY)                  \
  switch (C_) {                                      \
    case 4:  { constexpr int kC = 4;  BODY; } break; \
    case 8:  { constexpr int kC = 8;  BODY; } break; \
    case 12: { constexpr int kC = 12; BODY; } break; \
    case 16: { constexpr int kC = 16; BODY; } break; \
    case 20: { constexpr int kC = 20; BODY; } break; \
    case 24: { constexpr int kC = 24; BODY; } break; \
    case 32: { constexpr int kC = 32; BODY; } break; \
    case 48: { constexpr int kC = 48; BODY; } break; \
    case 64: { constexpr int kC = 64; BODY; } break; \
    default: return "unsupported channel width (supported: 4,8,12,16,20,24,32,48,64)"; \
  }

const char* spectral_mix_fwd(const void* x, const float* w, void* y, int B, int C, long long Q, cudaStream_t s) {
  if (Q <= 0) return nullptr;
  const int grid = static_cast<int>((Q + kMixQ - 1) / kMixQ);
  const dim3 block(kMixQ, kMixSplit);
  DFNO_MIX_DISPATCH(C, (launch_mix_fwd<kC>(grid, block, s, static_cast<const uint32_t*>(x),
                                            reinterpret_cast<const float2*>(w), static_cast<uint32_t*>(y), B, Q)));
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

const char* spectral_mix_bwd(const void* x, const float* w, const void* dy, void* dx, float* dw, int accumulate,
                             int B, int C, long long Q, cudaStream_t s) {
  if (Q <= 0) return nullptr;
  const int grid = static_cast<int>((Q + kMixQ - 1) / kMixQ);
  const dim3 block(kMixQ, kMixSplit);
  for (int b = 0; b < B; ++b) {
    const uint32_t* xb = static_cast<const uint32_t*>(x) + static_cast<long long>(b) * C * Q;
    const uint32_t* gb = static_cast<const uint32_t*>(dy) + static_cast<long long>(b) * C * Q;
    uint32_t* dxb = static_cast<uint32_t*>(dx) + static_cast<long long>(b) * C * Q;
    const int acc = (accumulate || b > 0) ? 1 : 0;
    if (dw) {
      DFNO_MIX_DISPATCH(C, (launch_mix_bwd<kC, true>(grid, block, s, xb, reinterpret_cast<const float2*>(w), gb, dxb,
                                                     reinterpret_cast<float2*>(dw), acc, Q)));
    } else {
      DFNO_MIX_DISPATCH(C, (launch_mix_bwd<kC, false>(grid, block, s, xb, reinterpret_cast<const float2*>(w), gb, dxb,
                                                      nullptr, 0, Q)));
    }
  }
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

}  // namespace dfno
