// Host/device-shared parameter blocks of the resident-operator GEMM (dft_gemm_sm90.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dfno {

enum EpiMode { EPI_ROWMAJOR = 0, EPI_PAIR_SCATTER = 1, EPI_HEAD = 2, EPI_BOX_STORE = 3 };
enum PeerSel { PEER_NONE = 0, PEER_BY_ROW = 1, PEER_BY_COL = 2 };

// Output addressing of the epilogue.  All strides/offsets are in *elements of the output
// type* (bf16 unless out_fp32).
//   EPI_ROWMAJOR     : out[row * ldc + col] (+ add_src[row * ld_add + col])
//   EPI_PAIR_SCATTER : column pairs (2j, 2j+1) are complex numbers.  The row index is split
//                      mixed-radix, innermost digit first, into nrl digits with radices R[]
//                      and element strides SR[]; the pair index j into (j % J[0], j / J[0])
//                      with strides SJ[].  One digit (a row digit, or j itself) may select the
//                      destination peer: peer = digit / peer_div, and digit % peer_div is used
//                      for addressing inside that peer's buffer.
//   EPI_HEAD         : projection head: out[addr(row)] = s0 + sum_j v1[j] * gelu(acc[row, j] + v0[j])
//                      (fp32 out; addr(row) from the row digits), i.e. linear3 -> gelu -> linear4
//                      without ever materialising the 128-channel intermediate (SURVEY.md K17).
//   EPI_BOX_STORE    : T1 box stores of the inverse y-DFT, addressed by BoxGeom (below); peers[] as above.
struct EpiParams {
  int mode;
  int out_fp32;
  int vec_ok;            // set by the launcher: row-major rows are 16-byte aligned
  long long ldc;
  const void* add_src;
  long long ld_add;
  int nrl;
  int R[4];
  long long SR[4];
  unsigned long long Rm[4];   // filled by the launcher: magic multipliers / shifts for fast division
  int Rs[4];
  unsigned long long Pm;
  int Ps;
  int J[2];
  long long SJ[2];
  int peer_sel;
  int peer_lvl;
  int peer_div;
  long long base_off;
  void* peers[8];
  const float* v0;       // EPI_HEAD: bias of the hidden layer   [N]
  const float* v1;       // EPI_HEAD: weights of the output layer [N]
  float s0;              // EPI_HEAD: output bias
};

struct GemmParams {
  long long M;   // rows of A / C
  int N;         // valid output columns
  int K;         // valid reduction length
  int n_pad;     // operator rows in memory   (multiple of 16, <= 256)
  int k_pad;     // operator row length       (multiple of 64)
  int a_f16;     // A holds IEEE fp16 instead of bf16: refused (wgmma has no mixed fp16 x bf16 form)
  EpiParams epi;
};

// EPI_BOX_STORE (the inverse y-DFT into T1): rows are (bcx, kz, kt), kt fastest, mt rows per kz group and kzl groups
// per bcx (M = bcx * kzl * mt); pair j is y.  A tile holds G = tile rows / mt whole kz groups of one bcx, staged in
// shared memory as [y][kz][kt (pitch mtp, pad words zero)] and stored with one TMA box per destination buffer:
// pair j goes to peers[j / ybox] at T1[bcx, y0 + j % ybox, kz, kt] with T1 = peer + base_off elements,
// [bcx][Yl][KZ][mtp] complex pairs (the rank's own kzl-wide kz slab starts at base_off).  ybox = min(N / 2, Yl).
struct BoxGeom {
  int mt, mtp, kzl, KZ, Yl, y0;
  long long bcx, base_off;
};

// Returns nullptr on success, else a static error string.  `Bmat` is the operator, bf16
// [n_pad, k_pad] row-major with zero padding; A is bf16 [M, K] with row pitch lda elements.
// `box` describes the T1 box store and is read for p.epi.mode == EPI_BOX_STORE only.
const char* dft_gemm_launch(const void* A, long long lda, const void* Bmat, GemmParams p, int num_sms,
                            cudaStream_t stream, const BoxGeom* box = nullptr);

}  // namespace dfno
