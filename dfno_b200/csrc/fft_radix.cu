// fft_radix.cu -- batched 1-D Stockham autosort FFT along the contiguous axis, radix 4 (+ one radix-2 pass),
// entirely in shared memory, with the FNO's mode truncation / zero padding fused into the load and the store.
//
// Role (SURVEY.md section 2.5, K5 note): the fused engine turns a *truncated* DFT into a tensor-core GEMM, which
// moves the same bytes as an FFT as long as few modes are kept (m <= N/4).  For wide spectra (m > N/4), for
// un-truncated transforms and for power-of-two axes longer than the GEMM kernel's 256 samples the O(N log N)
// butterfly network wins; this kernel is that path (reference ops: torch.fft.rfft/fft/ifft/irfft + restrict /
// zeropad, reference dfno/dfno.py:252-258,281-285).
//
//   forward   x[line, N] (real or complex) -> X[line, kept modes]     kept = [0,m) (one-sided) or [0,m) u [N-m,N)
//   inverse   X[line, kept modes] -> x[line, N] (complex, or real via Hermitian completion), scaled 1/N
//
// One line = N complex points ping-ponging between two shared-memory arrays; N/4 threads per line; several lines
// per CTA so that a CTA always has >= 128 threads.  Twiddles come from sincospif (exact argument reduction).
#include "sm90_ptx.cuh"
#include "kernels.h"

namespace dfno {
namespace {

struct FftParams {
  int N, logN;
  long long lines;
  int inverse;
  int in_real;        // forward: input is real
  int out_real;       // inverse: write the real part only
  int one_sided;      // kept modes are [0, m) of a Hermitian spectrum (rfft / irfft axis)
  int m;              // retained modes per side (m == 0: keep everything)
  int n_in, n_out;    // elements (complex or real) per line in the input / output tensors
  int lines_per_cta;
};

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

template <typename T> __device__ __forceinline__ float2 ld_c(const T* p, long long i);
template <> __device__ __forceinline__ float2 ld_c<float>(const float* p, long long i) { return reinterpret_cast<const float2*>(p)[i]; }
template <> __device__ __forceinline__ float2 ld_c<__nv_bfloat16>(const __nv_bfloat16* p, long long i) {
  return unpack_bf16x2(reinterpret_cast<const uint32_t*>(p)[i]);
}
template <typename T> __device__ __forceinline__ float ld_r(const T* p, long long i);
template <> __device__ __forceinline__ float ld_r<float>(const float* p, long long i) { return p[i]; }
template <> __device__ __forceinline__ float ld_r<__nv_bfloat16>(const __nv_bfloat16* p, long long i) { return __bfloat162float(p[i]); }
template <typename T> __device__ __forceinline__ void st_c(T* p, long long i, float2 v);
template <> __device__ __forceinline__ void st_c<float>(float* p, long long i, float2 v) { reinterpret_cast<float2*>(p)[i] = v; }
template <> __device__ __forceinline__ void st_c<__nv_bfloat16>(__nv_bfloat16* p, long long i, float2 v) {
  reinterpret_cast<uint32_t*>(p)[i] = pack_bf16x2(v.x, v.y);
}
template <typename T> __device__ __forceinline__ void st_r(T* p, long long i, float v);
template <> __device__ __forceinline__ void st_r<float>(float* p, long long i, float v) { p[i] = v; }
template <> __device__ __forceinline__ void st_r<__nv_bfloat16>(__nv_bfloat16* p, long long i, float v) { p[i] = __float2bfloat16(v); }

// one Stockham pass of radix R over a line of N points: src -> dst (natural order in, natural order out)
template <int R>
__device__ __forceinline__ void stockham_pass(const float2* __restrict__ src, float2* __restrict__ dst, int N, int Ns,
                                              int t, int nthreads, float sign) {
  const int stride = N / R;
  for (int j = t; j < stride; j += nthreads) {
    const int k = j & (Ns - 1);                       // Ns is a power of two
    float2 v[R];
#pragma unroll
    for (int r = 0; r < R; ++r) v[r] = src[j + r * stride];
    if (Ns > 1) {
      const float base = sign * 2.0f * static_cast<float>(k) / static_cast<float>(Ns * R);   // angle / pi
#pragma unroll
      for (int r = 1; r < R; ++r) {
        float s, c;
        sincospif(base * r, &s, &c);
        v[r] = cmul(v[r], make_float2(c, s));
      }
    }
    if (R == 2) {
      const float2 a = v[0], b = v[1];
      v[0] = make_float2(a.x + b.x, a.y + b.y);
      v[1] = make_float2(a.x - b.x, a.y - b.y);
    } else {                                          // radix-4 butterfly; multiplication by -+i for the odd outputs
      const float2 a = make_float2(v[0].x + v[2].x, v[0].y + v[2].y), b = make_float2(v[0].x - v[2].x, v[0].y - v[2].y);
      const float2 c = make_float2(v[1].x + v[3].x, v[1].y + v[3].y), d = make_float2(v[1].x - v[3].x, v[1].y - v[3].y);
      const float2 id = make_float2(-sign * d.y, sign * d.x);     // sign * i * d   (sign = -1 forward)
      v[0] = make_float2(a.x + c.x, a.y + c.y);
      v[2] = make_float2(a.x - c.x, a.y - c.y);
      v[1] = make_float2(b.x + id.x, b.y + id.y);
      v[3] = make_float2(b.x - id.x, b.y - id.y);
    }
    const int d0 = (j - k) * R + k;                   // expand(j, Ns, R)
#pragma unroll
    for (int r = 0; r < R; ++r) dst[d0 + r * Ns] = v[r];
  }
}

template <typename TIn, typename TOut>
__global__ void __launch_bounds__(1024)
fft_radix_kernel(const TIn* __restrict__ x, TOut* __restrict__ y, const FftParams p) {
  extern __shared__ float2 fft_smem[];
  const int tpl = blockDim.x / p.lines_per_cta;               // threads per line
  const int l_in_cta = threadIdx.x / tpl, t = threadIdx.x - l_in_cta * tpl;
  const int N = p.N, m = p.m;
  float2* A = fft_smem + static_cast<size_t>(l_in_cta) * 2 * N;
  float2* B = A + N;
  const float sign = p.inverse ? 1.0f : -1.0f;
  for (long long line0 = static_cast<long long>(blockIdx.x) * p.lines_per_cta; line0 < p.lines;
       line0 += static_cast<long long>(gridDim.x) * p.lines_per_cta) {
    const long long line = line0 + l_in_cta;
    const bool live = line < p.lines;
    // ---- load (zero padding / Hermitian completion fused)
    if (live) {
      const long long base = line * p.n_in;
      for (int i = t; i < N; i += tpl) {
        float2 v = make_float2(0.f, 0.f);
        if (!p.inverse) {
          v = p.in_real ? make_float2(ld_r<TIn>(x, base + i), 0.f) : ld_c<TIn>(x, base + i);
        } else if (m == 0) {
          if (!p.one_sided) v = ld_c<TIn>(x, base + i);
          else if (i <= N / 2) { v = ld_c<TIn>(x, base + i); if (i == 0 || 2 * i == N) v.y = 0.f; }
          else { v = ld_c<TIn>(x, base + (N - i)); v.y = -v.y; }
        } else if (p.one_sided) {                              // modes [0, m) of a Hermitian spectrum
          if (i < m) { v = ld_c<TIn>(x, base + i); if (i == 0 || 2 * i == N) v.y = 0.f; }
          else if (N - i < m && N - i > 0) { v = ld_c<TIn>(x, base + (N - i)); v.y = -v.y; }
        } else {                                               // [0, m) u [N - m, N), stored back to back
          if (i < m) v = ld_c<TIn>(x, base + i);
          else if (i >= N - m) v = ld_c<TIn>(x, base + (i - (N - 2 * m)));
        }
        A[i] = v;
      }
    }
    __syncthreads();
    // ---- butterflies: radix-4 passes, then one radix-2 pass when log2 N is odd
    float2* src = A;
    float2* dst = B;
    int Ns = 1;
    for (int s = 0; s + 1 < p.logN; s += 2) {
      if (live) stockham_pass<4>(src, dst, N, Ns, t, tpl, sign);
      __syncthreads();
      float2* tmp = src; src = dst; dst = tmp;
      Ns <<= 2;
    }
    if (p.logN & 1) {
      if (live) stockham_pass<2>(src, dst, N, Ns, t, tpl, sign);
      __syncthreads();
      float2* tmp = src; src = dst; dst = tmp;
    }
    // ---- store (mode truncation / real part / 1/N fused)
    if (live) {
      const long long base = line * p.n_out;
      if (p.inverse) {
        const float sc = 1.0f / static_cast<float>(N);
        for (int i = t; i < N; i += tpl) {
          const float2 v = src[i];
          if (p.out_real) st_r<TOut>(y, base + i, v.x * sc);
          else st_c<TOut>(y, base + i, make_float2(v.x * sc, v.y * sc));
        }
      } else {
        for (int i = t; i < p.n_out; i += tpl) {
          int k = i;
          if (m > 0 && !p.one_sided && i >= m) k = N - 2 * m + i;
          st_c<TOut>(y, base + i, src[k]);
        }
      }
    }
    __syncthreads();
  }
}

}  // namespace

// x / y: contiguous lines along the transformed axis.  `bf16` selects bf16 vs fp32 storage for both tensors.
//   forward: n_in = N (real or complex), n_out = kept modes (N, N/2+1, m or 2m)
//   inverse: n_in = kept modes, n_out = N (complex or real)
const char* fft_radix(const void* x, void* y, int bf16, int N, long long lines, int inverse, int in_real, int out_real,
                      int one_sided, int m, int num_sms, cudaStream_t s) {
  if (N < 2 || N > 4096 || (N & (N - 1))) return "fft_radix: N must be a power of two in [2, 4096]";
  if (m < 0 || (one_sided ? m > N / 2 + 1 : 2 * m > N)) return "fft_radix: more modes than the axis has";
  if (in_real && inverse) return "fft_radix: a real input belongs to the forward transform";
  if (out_real && !inverse) return "fft_radix: a real output belongs to the inverse transform";
  if (lines <= 0) return nullptr;
  FftParams p{};
  p.N = N; p.logN = 0;
  while ((1 << p.logN) < N) ++p.logN;
  p.lines = lines; p.inverse = inverse; p.in_real = in_real; p.out_real = out_real; p.one_sided = one_sided; p.m = m;
  const int kept = m > 0 ? (one_sided ? m : 2 * m) : (one_sided ? N / 2 + 1 : N);
  p.n_in = inverse ? kept : N;
  p.n_out = inverse ? N : kept;
  const int tpl = N >= 8 ? N / 4 : 1;
  p.lines_per_cta = tpl >= 128 ? 1 : 128 / tpl;
  const int threads = tpl * p.lines_per_cta;
  const size_t smem = static_cast<size_t>(p.lines_per_cta) * 2 * N * sizeof(float2);
  const long long ctas = (lines + p.lines_per_cta - 1) / p.lines_per_cta;
  const long long cap = static_cast<long long>(num_sms) * (smem > 32768 ? 2 : 8);
  const int grid = static_cast<int>(ctas < cap ? ctas : cap);
#define DFNO_FFT_LAUNCH(TI, TO)                                                                                  \
  do {                                                                                                           \
    if (smem > 48 * 1024) {                                                                                      \
      static bool attr = false;                                                                                  \
      if (!attr) {                                                                                               \
        if (cudaFuncSetAttribute(fft_radix_kernel<TI, TO>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024) != \
            cudaSuccess)                                                                                         \
          return "fft_radix: cudaFuncSetAttribute failed";                                                       \
        attr = true;                                                                                             \
      }                                                                                                          \
    }                                                                                                            \
    fft_radix_kernel<TI, TO><<<grid, threads, smem, s>>>(static_cast<const TI*>(x), static_cast<TO*>(y), p);     \
  } while (0)
  if (bf16) DFNO_FFT_LAUNCH(__nv_bfloat16, __nv_bfloat16);
  else DFNO_FFT_LAUNCH(float, float);
#undef DFNO_FFT_LAUNCH
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

}  // namespace dfno
