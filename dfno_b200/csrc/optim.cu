// optim.cu -- fused Adam over the engine's single flat fp32 parameter buffer.
// All parameters of the fused model (pointwise weights and every spectral shard) live in one
// contiguous allocation, so one vectorised launch updates the whole model
// (reference: torch.optim.Adam, train_two_phase.py:82, experiment_navier_stokes.py:120).
//
// Two instantiations of adam_kernel:
//   kDev = false  hyperparameters are kernel arguments (the default path; a captured CUDA graph bakes them in);
//   kDev = true   hyperparameters are read from a device array (AdamHparams layout) that the host rewrites before
//                 every step or graph replay, so learning-rate / momentum schedules run under replay.  Adds decoupled
//                 (AdamW) weight decay and gradient-norm clipping with the coefficient of
//                 torch.nn.utils.clip_grad_norm_, computed in the prologue from the device sum of squares.
// sumsq_kernel gives that sum of squares: block partials, then a fixed-order pass by the last block (an integer
// ticket, no floating-point atomics), accumulated in fp64, so the result is the same on every call.
#include "sm90_ptx.cuh"
#include "kernels.h"

namespace dfno {
namespace {

// device hyperparameter array (fp64, written by adam_hparams_kernel)
enum AdamHp { kHpLr = 0, kHpBeta1, kHpBeta2, kHpEps, kHpWd, kHpDecoupled, kHpMaxNorm, kHpCount };

struct AdamDevArgs {
  const double* hp;        // AdamHp layout
  const double* sumsq;     // sum of squares of the (unscaled) gradient, or nullptr: no clipping
  float* norm_out;         // pre-clip gradient norm (written by block 0 when sumsq != nullptr)
};

template <bool kDev>
__global__ void __launch_bounds__(256)
adam_kernel(float4* __restrict__ p, const float4* __restrict__ g, float4* __restrict__ m, float4* __restrict__ v,
            long long n4, float* __restrict__ ps, const float* __restrict__ gs, float* __restrict__ ms,
            float* __restrict__ vs, int tail, float lr, float b1, float b2, float eps, float wd, float bias1,
            float bias2, float gscale, const float* __restrict__ step_dev, AdamDevArgs dev) {
  if constexpr (!kDev) {
    if (step_dev != nullptr) {                 // step count read from device memory (CUDA-graph replay)
      const float t = *step_dev;
      bias1 = 1.f - powf(b1, t);
      bias2 = 1.f - powf(b2, t);
    }
    const float step = lr / bias1;
    const float inv_sqrt_b2 = rsqrtf(bias2);
    auto upd = [&](float& pp, float gg, float& mm, float& vv) {
      gg = gg * gscale + wd * pp;
      mm = b1 * mm + (1.f - b1) * gg;
      vv = b2 * vv + (1.f - b2) * gg * gg;
      pp -= step * mm / (sqrtf(vv) * inv_sqrt_b2 + eps);
    };
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
      float4 P = p[i], G = g[i], M = m[i], V = v[i];
      upd(P.x, G.x, M.x, V.x); upd(P.y, G.y, M.y, V.y); upd(P.z, G.z, M.z, V.z); upd(P.w, G.w, M.w, V.w);
      p[i] = P; m[i] = M; v[i] = V;
    }
    if (blockIdx.x == 0 && threadIdx.x < tail) {
      const int i = threadIdx.x;
      float P = ps[i], M = ms[i], V = vs[i];
      upd(P, gs[i], M, V);
      ps[i] = P; ms[i] = M; vs[i] = V;
    }
  } else {
    // Prologue, once per block.  Scalars follow torch.optim.Adam's foreach path: bias corrections, lr / bias1,
    // sqrt(bias2), 1 - lr * wd and 1 - beta in fp64, rounded to fp32 for the element loop.  The clip coefficient is
    // clip_grad_norm_'s: max_norm / (norm + 1e-6) clamped to at most 1 (a NaN stays NaN), on the fp32 norm.
    __shared__ float s[11];
    if (threadIdx.x == 0) {
      const double* hp = dev.hp;
      const double t = static_cast<double>(*step_dev);
      const double lr_d = hp[kHpLr], b1_d = hp[kHpBeta1], b2_d = hp[kHpBeta2], wd_d = hp[kHpWd];
      const bool decoupled = hp[kHpDecoupled] != 0.0;
      float coef = 1.f;
      if (dev.sumsq != nullptr) {
        // the sum is rounded to fp32 before the root, as torch's fp32 norm accumulates it: a sum beyond the fp32
        // range gives an infinite norm and a zero coefficient there too
        const float sq = static_cast<float>(*dev.sumsq * (static_cast<double>(gscale) * gscale));
        const float norm = sqrtf(sq);
        const float c = static_cast<float>(hp[kHpMaxNorm]) / (norm + 1e-6f);
        coef = c > 1.f ? 1.f : c;
        if (blockIdx.x == 0) *dev.norm_out = norm;
      }
      s[0] = static_cast<float>(b1_d);
      s[1] = static_cast<float>(1.0 - b1_d);
      s[2] = static_cast<float>(b2_d);
      s[3] = static_cast<float>(1.0 - b2_d);
      s[4] = static_cast<float>(hp[kHpEps]);
      s[5] = decoupled ? 0.f : static_cast<float>(wd_d);                      // L2 term
      s[6] = decoupled ? static_cast<float>(1.0 - lr_d * wd_d) : 1.f;        // decoupled decay factor
      s[7] = static_cast<float>(lr_d / (1.0 - pow(b1_d, t)));                // step size
      s[8] = static_cast<float>(sqrt(1.0 - pow(b2_d, t)));                   // sqrt(bias2)
      s[9] = gscale * coef;
      s[10] = decoupled ? 1.f : 0.f;
    }
    __syncthreads();
    const float B1 = s[0], OMB1 = s[1], B2 = s[2], OMB2 = s[3], EPS = s[4], WD = s[5], DECAY = s[6];
    const float STEP = s[7], BC2S = s[8], GMUL = s[9];
    const bool decoupled = s[10] != 0.f;
    auto upd = [&](float& pp, float gg, float& mm, float& vv) {
      gg = gg * GMUL;
      if (decoupled) pp *= DECAY;
      else gg += WD * pp;
      mm = B1 * mm + OMB1 * gg;
      vv = B2 * vv + OMB2 * gg * gg;
      pp -= STEP * (mm / (sqrtf(vv) / BC2S + EPS));
    };
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
      float4 P = p[i], G = g[i], M = m[i], V = v[i];
      upd(P.x, G.x, M.x, V.x); upd(P.y, G.y, M.y, V.y); upd(P.z, G.z, M.z, V.z); upd(P.w, G.w, M.w, V.w);
      p[i] = P; m[i] = M; v[i] = V;
    }
    if (blockIdx.x == 0 && threadIdx.x < tail) {
      const int i = threadIdx.x;
      float P = ps[i], M = ms[i], V = vs[i];
      upd(P, gs[i], M, V);
      ps[i] = P; ms[i] = M; vs[i] = V;
    }
  }
}

__global__ void adam_hparams_kernel(double* __restrict__ hp, double lr, double b1, double b2, double eps, double wd,
                                    double decoupled, double max_norm) {
  if (threadIdx.x == 0) {
    hp[kHpLr] = lr; hp[kHpBeta1] = b1; hp[kHpBeta2] = b2; hp[kHpEps] = eps; hp[kHpWd] = wd;
    hp[kHpDecoupled] = decoupled; hp[kHpMaxNorm] = max_norm;
  }
}

// fixed-order sum over a 256-thread block; the result is valid in thread 0
__device__ __forceinline__ double block_sum_256(double a, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a += __shfl_down_sync(0xffffffffu, a, o);
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) red[w] = a;
  __syncthreads();
  if (threadIdx.x == 0) {
    a = red[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) a += red[i];
  }
  return a;
}

__global__ void __launch_bounds__(256, 8)
sumsq_kernel(const float4* __restrict__ body, long long n4, const float* __restrict__ head, int nhead,
             const float* __restrict__ tail, int ntail, double* __restrict__ partials, unsigned* __restrict__ ticket,
             double* __restrict__ out) {
  __shared__ double red[8];
  __shared__ bool last;
  double a0 = 0.0, a1 = 0.0;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 x = body[i];
    a0 = fma(static_cast<double>(x.x), static_cast<double>(x.x), a0);
    a1 = fma(static_cast<double>(x.y), static_cast<double>(x.y), a1);
    a0 = fma(static_cast<double>(x.z), static_cast<double>(x.z), a0);
    a1 = fma(static_cast<double>(x.w), static_cast<double>(x.w), a1);
  }
  if (blockIdx.x == 0) {                        // unaligned head and scalar tail
    if (static_cast<int>(threadIdx.x) < nhead) a0 = fma(static_cast<double>(head[threadIdx.x]), head[threadIdx.x], a0);
    if (static_cast<int>(threadIdx.x) < ntail) a1 = fma(static_cast<double>(tail[threadIdx.x]), tail[threadIdx.x], a1);
  }
  const double b = block_sum_256(a0 + a1, red);
  if (threadIdx.x == 0) {
    partials[blockIdx.x] = b;
    __threadfence();                            // the partial is visible before the ticket is taken
    last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  double a = 0.0;                               // last block: partials in index order
  for (int i = threadIdx.x; i < static_cast<int>(gridDim.x); i += 256) a += __ldcg(partials + i);
  __syncthreads();                              // red is reused
  a = block_sum_256(a, red);
  if (threadIdx.x == 0) {
    *out = a;
    *ticket = 0u;                               // ready for the next call (and the next graph replay)
  }
}

long long adam_blocks(long long n4, int num_sms) {
  long long blocks = (n4 + 255) / 256;
  const long long cap = static_cast<long long>(num_sms) * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return blocks;
}
}  // namespace

const char* adam_step(float* p, const float* g, float* m, float* v, long long n, float lr, float beta1, float beta2,
                      float eps, float weight_decay, float bias1, float bias2, float grad_scale, const float* step_dev,
                      int num_sms, cudaStream_t s) {
  if (n <= 0) return nullptr;
  if ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
       reinterpret_cast<uintptr_t>(v)) % 16)
    return "adam: buffers must be 16-byte aligned";
  const long long n4 = n / 4;
  const int tail = static_cast<int>(n - n4 * 4);
  adam_kernel<false><<<static_cast<int>(adam_blocks(n4, num_sms)), 256, 0, s>>>(
      reinterpret_cast<float4*>(p), reinterpret_cast<const float4*>(g), reinterpret_cast<float4*>(m),
      reinterpret_cast<float4*>(v), n4, p + n4 * 4, g + n4 * 4, m + n4 * 4, v + n4 * 4, tail, lr, beta1, beta2, eps,
      weight_decay, bias1, bias2, grad_scale, step_dev, AdamDevArgs{nullptr, nullptr, nullptr});
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

const char* adam_step_dev(float* p, const float* g, float* m, float* v, long long n, const double* hparams,
                          const float* step_dev, float grad_scale, const double* sumsq, float* norm_out, int num_sms,
                          cudaStream_t s) {
  if (n <= 0) return nullptr;
  if ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
       reinterpret_cast<uintptr_t>(v)) % 16)
    return "adam: buffers must be 16-byte aligned";
  if (hparams == nullptr || step_dev == nullptr) return "adam: the device path needs the hyperparameters and step";
  if (sumsq != nullptr && norm_out == nullptr) return "adam: clipping needs a norm output";
  const long long n4 = n / 4;
  const int tail = static_cast<int>(n - n4 * 4);
  adam_kernel<true><<<static_cast<int>(adam_blocks(n4, num_sms)), 256, 0, s>>>(
      reinterpret_cast<float4*>(p), reinterpret_cast<const float4*>(g), reinterpret_cast<float4*>(m),
      reinterpret_cast<float4*>(v), n4, p + n4 * 4, g + n4 * 4, m + n4 * 4, v + n4 * 4, tail, 0.f, 0.f, 0.f, 0.f,
      0.f, 1.f, 1.f, grad_scale, step_dev, AdamDevArgs{hparams, sumsq, norm_out});
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

const char* adam_set_hparams(double* hparams, double lr, double beta1, double beta2, double eps, double weight_decay,
                             bool decoupled, double max_norm, cudaStream_t s) {
  adam_hparams_kernel<<<1, 32, 0, s>>>(hparams, lr, beta1, beta2, eps, weight_decay, decoupled ? 1.0 : 0.0, max_norm);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

const char* sumsq(const float* x, long long n, double* out, double* partials, int max_blocks, unsigned* ticket,
                  int num_sms, cudaStream_t s) {
  if (n < 0) return "sumsq: negative length";
  if (reinterpret_cast<uintptr_t>(x) % 4) return "sumsq: x must be 4-byte aligned";
  if (max_blocks < 1 || partials == nullptr || ticket == nullptr || out == nullptr) return "sumsq: missing workspace";
  const int mis = static_cast<int>((reinterpret_cast<uintptr_t>(x) % 16) / 4);
  const int nhead = static_cast<int>(mis ? (4 - mis < n ? 4 - mis : n) : 0);
  const float* body = x + nhead;
  const long long n4 = (n - nhead) / 4;
  const int ntail = static_cast<int>(n - nhead - n4 * 4);
  long long blocks = adam_blocks(n4, num_sms);
  if (blocks > max_blocks) blocks = max_blocks;
  sumsq_kernel<<<static_cast<int>(blocks), 256, 0, s>>>(reinterpret_cast<const float4*>(body), n4, x, nhead,
                                                        body + n4 * 4, ntail, partials, ticket, out);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}
}  // namespace dfno
