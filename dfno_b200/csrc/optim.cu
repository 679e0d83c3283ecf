// optim.cu -- fused Adam over the engine's single flat fp32 parameter buffer.
// All parameters of the fused model (pointwise weights and every spectral shard) live in one
// contiguous allocation, so one vectorised launch updates the whole model
// (reference: torch.optim.Adam, train_two_phase.py:82, experiment_navier_stokes.py:120).
#include "sm90_ptx.cuh"
#include "kernels.h"

namespace dfno {
namespace {
__global__ void __launch_bounds__(256)
adam_kernel(float4* __restrict__ p, const float4* __restrict__ g, float4* __restrict__ m, float4* __restrict__ v,
            long long n4, float* __restrict__ ps, const float* __restrict__ gs, float* __restrict__ ms,
            float* __restrict__ vs, int tail, float lr, float b1, float b2, float eps, float wd, float bias1,
            float bias2, float gscale, const float* __restrict__ step_dev) {
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
  long long blocks = (n4 + 255) / 256;
  const long long cap = static_cast<long long>(num_sms) * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  adam_kernel<<<static_cast<int>(blocks), 256, 0, s>>>(
      reinterpret_cast<float4*>(p), reinterpret_cast<const float4*>(g), reinterpret_cast<float4*>(m),
      reinterpret_cast<float4*>(v), n4, p + n4 * 4, g + n4 * 4, m + n4 * 4, v + n4 * 4, tail, lr, beta1, beta2, eps,
      weight_decay, bias1, bias2, grad_scale, step_dev);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}
}  // namespace dfno
