// head_common.cuh -- pieces shared by the projection-head kernels (head_sm90.cu, head_multi_sm90.cu): the row map from
// an engine position row to its element offset in the public output layout, the accumulator-fragment row of a
// thread, and the |dout| maximum that sets the fp16 scale of the backward.  Each translation unit gets its own copy.
#pragma once
#include "sm90_ptx.cuh"

namespace dfno {
namespace {

constexpr int kHidH = 128;

struct RowMap {                      // position row -> element offset in the public [B,O,X,Y,Z,T] layout
  int nrl;
  int R[4];
  long long SR[4];
  unsigned long long Rm[4];
  int Rs[4];
};

__device__ __forceinline__ long long row_to_offset(const RowMap& e, uint32_t r) {
  long long off = 0;
#pragma unroll
  for (int l = 0; l < 4; ++l) {
    if (l < e.nrl) {
      uint32_t d = r;
      if (l != e.nrl - 1) {
        const uint32_t q = static_cast<uint32_t>((static_cast<unsigned long long>(r) * e.Rm[l]) >> e.Rs[l]);
        d = r - q * static_cast<uint32_t>(e.R[l]);
        r = q;
      }
      off += static_cast<long long>(d) * e.SR[l];
    }
  }
  return off;
}

void fill_magic(RowMap* m) {
  for (int l = 0; l < 4; ++l) {
    const unsigned d = static_cast<unsigned>(m->R[l] > 0 ? m->R[l] : 1);
    int s = 0;
    while ((1ull << s) < d) ++s;
    m->Rm[l] = ((1ull << (31 + s)) / d) + 1;
    m->Rs[l] = 31 + s;
  }
}

// The epilogues work on the accumulator fragment: thread (warp q of the warpgroup, lane l) holds 4 positions of the
// tile (frag_row) and, for each, the 32 hidden units 8j + 2(l%4) + {0, 1} of a 128-unit row.
__device__ __forceinline__ int frag_row(int q, int lane, int k) {     // k = 0..3: the thread's rows of a 128-row tile
  return 64 * (k >> 1) + 16 * q + (lane >> 2) + 8 * (k & 1);
}
__device__ __forceinline__ float pick4(const float (&v)[4], int k) {   // v[k] for a run-time k, without local memory
  return k == 0 ? v[0] : k == 1 ? v[1] : k == 2 ? v[2] : v[3];
}

__global__ void absmax_kernel(const float* __restrict__ x, long long n, unsigned* __restrict__ out) {
  float mx = 0.f;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i * 4 < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    if (i * 4 + 3 < n) {
      const float4 v = reinterpret_cast<const float4*>(x)[i];
      mx = fmaxf(mx, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
    } else {
      for (long long k = i * 4; k < n; ++k) mx = fmaxf(mx, fabsf(x[k]));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0 && mx > 0.f) atomicMax(out, __float_as_uint(mx));   // non-negative floats order like uints
}

int set_rowmap(RowMap* mp, int nrl, const int* R, const long long* SR) {
  if (nrl < 1 || nrl > 4) return -1;
  mp->nrl = nrl;
  for (int i = 0; i < 4; ++i) { mp->R[i] = i < nrl ? R[i] : 1; mp->SR[i] = i < nrl ? SR[i] : 0; }
  fill_magic(mp);
  return 0;
}

// Row map of a zero-padded activation (the padded-layout head kernels): up to 5 digits (b, x, y, t, z can all be
// separate), each with the extent of its interior; a row with any digit at or beyond its bound lies in the pad region
// and has no output element.
constexpr int kPadDigits = 5;
struct PadRowMap {
  int nrl;
  int R[kPadDigits], lim[kPadDigits];
  long long SR[kPadDigits];
  unsigned long long Rm[kPadDigits];
  int Rs[kPadDigits];
};

// element offset of row r in the public output, or -1 for a pad row
__device__ __forceinline__ long long pad_row_to_offset(const PadRowMap& e, uint32_t r) {
  long long off = 0;
  bool inside = true;
#pragma unroll
  for (int l = 0; l < kPadDigits; ++l) {
    if (l < e.nrl) {
      uint32_t d = r;
      if (l != e.nrl - 1) {
        const uint32_t q = static_cast<uint32_t>((static_cast<unsigned long long>(r) * e.Rm[l]) >> e.Rs[l]);
        d = r - q * static_cast<uint32_t>(e.R[l]);
        r = q;
      }
      inside = inside && d < static_cast<uint32_t>(e.lim[l]);
      off += static_cast<long long>(d) * e.SR[l];
    }
  }
  return inside ? off : -1;
}

int set_padrowmap(PadRowMap* mp, int nrl, const int* R, const long long* SR, const int* lim) {
  if (nrl < 1 || nrl > kPadDigits) return -1;
  mp->nrl = nrl;
  for (int i = 0; i < kPadDigits; ++i) {
    mp->R[i] = i < nrl ? R[i] : 1;
    mp->SR[i] = i < nrl ? SR[i] : 0;
    mp->lim[i] = i < nrl ? lim[i] : 1;
    if (mp->lim[i] > mp->R[i]) return -1;
    const unsigned d = static_cast<unsigned>(mp->R[i] > 0 ? mp->R[i] : 1);      // as fill_magic
    int s = 0;
    while ((1ull << s) < d) ++s;
    mp->Rm[i] = ((1ull << (31 + s)) / d) + 1;
    mp->Rs[i] = 31 + s;
  }
  return 0;
}

}  // namespace
}  // namespace dfno
