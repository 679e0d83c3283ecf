// Launchers of the torch-free CUDA translation units (pointwise / spectral / optimizer / p2p).
// Every launcher returns nullptr on success or a static error string.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dfno {

struct LiftDims {
  int B, Cin, Tin;     // input  [B, Cin, X, Y, Z, Tin]   (reference layout, t contiguous)
  int C, T;            // output [B*C, X, Y, T, Z]        (engine layout, z contiguous)
  int X, Y, Z;         // local spatial extents
};

// Extents of a zero-padded engine activation (each >= the LiftDims one, Z a multiple of 8): h[B*C, X, Y, T, Z] with
// the interior [0, d.X) x [0, d.Y) x [0, d.T) x [0, d.Z) and zeros elsewhere.
struct LiftPad {
  int X, Y, Z, T;
};

// pad (may be null): h has the padded extents; the lift writes its pad positions as exact zeros
const char* lift_fwd(const void* x, int x_is_bf16, const float* W1, const float* b1, const float* W2,
                     const float* b2, void* h, LiftDims d, const LiftPad* pad, int num_sms, cudaStream_t s);
// dx (may be null): fp32 input gradient in x's layout, written (not accumulated).  pad (may be null): dh has the
// padded extents and is read at interior positions only.
const char* lift_bwd(const void* x, int x_is_bf16, const float* W1, const float* b1, const float* W2,
                     const float* b2, const void* dh, float* gW1, float* gb1, float* gW2, float* gb2, float* dx,
                     LiftDims d, const LiftPad* pad, int num_sms, cudaStream_t s);
// strided permutation of 32-bit words: dst walked in mixed-radix order (innermost digit first, strides in words)
const char* permute_u32(const void* src, void* dst, int nd, const int* size, const long long* sstr,
                        const long long* dstr, int num_sms, cudaStream_t s);
// device GELU / GELU' evaluated on a vector (accuracy probe for the tests)
const char* gelu_probe(const float* x, float* y, float* dy, long long n, cudaStream_t s);
const char* gelu_probe_h2(const float* x, float* y, float* dy, long long n, cudaStream_t s);   // packed fp16 variant (n even)
// S = X*Y*T*Z elements per (b, c) slab.  out / out_cl may be null.
const char* bypass_gelu_fwd(const void* h, void* spec_pre, const float* W, void* out, void* out_cl, int cl_pitch,
                            int B, int C, long long S, int save_pre, int num_sms, cudaStream_t s);
const char* bypass_gelu_bwd(const void* dout, const void* dout_cl, int cl_pitch, const void* pre, const float* W,
                            void* dpre, void* dhb, int B, int C, long long S, int num_sms, cudaStream_t s);

// wgmma versions (bypass_sm90.cu): TMA in/out, channel mixing on the tensor core, dW accumulated in registers.
// Wpad / WTpad: bf16 [32, 64] zero-padded W[o, i] / W^T[i, o].  Need C <= 32 and S % 128 == 0.
const char* bypass_fwd_tc(const void* h, void* spec_pre, const void* Wpad, void* out, void* out_cl, int cl_pitch,
                          int B, int C, long long S, int save_pre, int num_sms, cudaStream_t stream);
const char* bypass_bwd_tc(const void* dout, const void* dout_cl, int cl_pitch, void* pre_dpre, const void* h,
                          const void* WTpad, void* dhb, float* dW, int B, int C, long long S, int num_sms,
                          cudaStream_t stream);

// spectral channel mixing over the local mode slab: x,y bf16 [B, C, Q, 2]; w fp32 [C, C, Q, 2]
const char* spectral_mix_fwd(const void* x, const float* w, void* y, int B, int C, long long Q, cudaStream_t s);
// dx = dy * conj(w) ; dw (+)= conj(x) * dy summed over the batch (dw null: dx only, frozen weights)
const char* spectral_mix_bwd(const void* x, const float* w, const void* dy, void* dx, float* dw, int accumulate,
                             int B, int C, long long Q, cudaStream_t s);

// fused Adam over one flat fp32 parameter buffer (decoupled=0: L2 weight decay like torch.optim.Adam)
const char* adam_step(float* p, const float* g, float* m, float* v, long long n, float lr, float beta1, float beta2,
                      float eps, float weight_decay, float bias1, float bias2, float grad_scale, const float* step_dev,
                      int num_sms, cudaStream_t s);
// the same update with its hyperparameters read from a device array (written by adam_set_hparams before every step
// or graph replay): schedules under CUDA-graph replay, decoupled (AdamW) decay, and clipping to a global norm whose
// sum of squares `sumsq` (nullable: no clipping) is on the device; the pre-clip norm goes to norm_out
const char* adam_step_dev(float* p, const float* g, float* m, float* v, long long n, const double* hparams,
                          const float* step_dev, float grad_scale, const double* sumsq, float* norm_out, int num_sms,
                          cudaStream_t s);
const char* adam_set_hparams(double* hparams, double lr, double beta1, double beta2, double eps, double weight_decay,
                             bool decoupled, double max_norm, cudaStream_t s);
// out[0] = sum(x*x) over n fp32 values, in fp64, deterministic (fixed grid and reduction order); partials holds
// max_blocks doubles, ticket one zeroed uint32 that the kernel leaves at zero
const char* sumsq(const float* x, long long n, double* out, double* partials, int max_blocks, unsigned* ticket,
                  int num_sms, cudaStream_t s);

// cross-GPU flag barrier over NVLink-mapped signal pads: every rank bumps its slot on each
// peer to `epoch`, then waits until all of its own slots reached `epoch`.
// timeout_ns > 0 bounds the spin: a late peer makes the kernel record the slot and trap (failure detection).
const char* p2p_barrier(uint32_t* const* peer_flags, uint32_t* my_flags, int rank, int world, uint32_t epoch,
                        unsigned long long timeout_ns, cudaStream_t s);
// sum-all-reduce of a small fp32 vector through peer reads (every rank reads all peers' copies)
const char* p2p_allreduce_small(float* const* peer_bufs, float* out, long long n, int rank, int world,
                                cudaStream_t s);
// out = sum over ranks, in rank order, of the fp64 scalar at each peer pointer
const char* p2p_sum_f64(double* const* peer_bufs, double* out, int world, cudaStream_t s);

// push all-to-all-v over peer memory: segment i of `send` ([send_off[i], send_off[i+1]) bytes) is stored at
// byte offset dst_off[i] of peer i's receive buffer.  Follow with p2p_barrier before reading.
const char* p2p_alltoall(const void* send, const long long* send_off, void* const* peer_recv, const long long* dst_off,
                         int world, int ctas_per_peer, cudaStream_t s);

// K-reduction GEMM: D[i, j] (+)= sum_k A[i, k] * B[j, k]; A: [Ma<=128, K], B: [Nb<=256, K] bf16 K-major.
const char* kreduce_gemm(const void* A, long long lda, int Ma, const void* Bm, long long ldb, int Nb, long long K,
                         float* D, long long ldd, int num_sms, cudaStream_t s);

// backward of the projection head (head_bwd_sm90.cu).  dout is read at the mixed-radix address
// of each row (public [B,1,X,Y,Z,T] layout); gradients are accumulated with atomics.
const char* head_bwd(const void* hcl, long long npos, int C, int CP, const void* W3pad, const void* W3Tpad,
                     const float* b3, const float* W4, const float* dout, int nrl, const int* R, const long long* SR,
                     void* gcl, float* gW3, float* gb3, float* gW4, float* gb4, int num_sms, cudaStream_t stream);

// batched Stockham FFT along the contiguous axis with fused truncation / zero padding (fft_radix.cu)
const char* fft_radix(const void* x, void* y, int bf16, int N, long long lines, int inverse, int in_real, int out_real,
                      int one_sided, int m, int num_sms, cudaStream_t s);

// First two stages of a Fourier layer (truncated z-DFT then t-DFT) + the pencil transpose R2 in one kernel: see
// spectral_in_sm90.cu.  dst_ptrs[j] (+ dst_off elements): rank j's S1 / S1s, viewed [B*C, kzl, mt, X, Yl*2] with
// element strides dstr = {x, kt, kz, bc}.
const char* spectral_in(const void* h, const void* op1, int n1_pad, int k1_pad, const void* op2, int n2_pad, int k2_pad,
                        const long long* dst_ptrs, int P, long long dst_off, const long long* dstr, int BC, int X,
                        int Yl, int T, int Z, int KZ, int mt, int num_sms, cudaStream_t stream);
const char* spectral_in_check(int n1_pad, int k1_pad, int n2_pad, int k2_pad, int P, long long dst_off, const long long* dstr,
                              int BC, int X, int Yl, int T, int Z, int KZ, int mt, int* cfg /* {Rp, Yc, E, stages} or null */);

// Elementwise part of the relative-L2 / MSE losses (loss.cu): per-sample sums of (y_hat - y)^2 and y^2 into
// part[0..B) / part[B..2B), and grad = (y_hat - y) * scale[b].
const char* sq_partials(const float* yh, const float* y, float* part, long long n_per_b, int B, int num_sms, cudaStream_t s);
const char* scaled_diff(const float* yh, const float* y, const float* scale, float* grad, long long n_per_b, int B,
                        int scale_per_b, int num_sms, cudaStream_t s);

// ---- round-2 fused pointwise path (spectral_out_sm90.cu, dpre_dw_sm90.cu, head_sm90.cu) ----
// Last stage of a Fourier layer + bypass conv (+ GELU): see spectral_out_sm90.cu.  U: bf16 [B*C, L, K1];
// h / pre / out: bf16 [B*C, L, Z]; Bop: padded operator bf16 [n_pad, k_pad]; W: fp32 [C, C].
const char* spectral_out(const void* U, const void* h, const void* Bop, int n_pad, int k_pad, const float* W,
                         int transpose_w, void* pre, void* out, int B, int C, long long L, int Z, int K1, int gelu,
                         int save_pre, int num_sms, cudaStream_t stream);
// The adjoint of spectral_out with the pointwise backward of the neighbouring blocks folded in: pre_prev (may be null)
// is pre_{k-1} in and dpre_{k-1} = g * gelu'(pre_{k-1}) out (g is then not stored), h + dW (may be null): dW += dpre . h^T.
// spectral_out_adj_check: null when the kernel takes the shape (dpre / dw: which of the two it folds), the reason otherwise.
const char* spectral_out_adj(const void* U, const void* dpre, const void* Bop, int n_pad, int k_pad, const float* W,
                             void* pre_prev, void* g, const void* h, float* dW, int B, int C, long long L, int Z, int K1,
                             int num_sms, cudaStream_t stream);
const char* spectral_out_adj_check(int n_pad, int k_pad, int C, int Z, int K1, int dpre, int dw);
// dpre = g * gelu'(pre) (in place over pre); dW += dpre . h^T
const char* dpre_dw(const void* g, void* pre_dpre, const void* h, float* dW, int B, int C, long long L, int Z,
                    int num_sms, cudaStream_t stream);
// projection head on the channel-major activation (head_sm90.cu).  lim (may be null): h is zero-padded; the row digits
// (up to 5) come with per-digit interior bounds, pad rows store no output and read dout as 0.
const char* head_fwd(const void* h, const void* W3aug, const float* w4b4, float* out, int B, int C, long long S,
                     int nrl, const int* R, const long long* SR, const int* lim, int num_sms, cudaStream_t stream);
const char* head_bwd2(const void* h, const void* W3aug, const void* W3T16, const float* W4, const float* dout,
                      long long n_dout, unsigned* amax_ws, void* g, float* gW3, float* gb3, float* gW4, float* gb4,
                      int B, int C, long long S, int nrl, const int* R, const long long* SR, const int* lim,
                      int num_sms, cudaStream_t stream);
// projection head with O = 1..4 output channels (head_multi_sm90.cu): output channel o of a row at + o*plane.
// w4b4 = [W4 (O x 128), b4 (O)]; the backward takes C <= 31 and reduces |dout| over all n_dout elements.
const char* head_fwd_multi(const void* h, const void* W3aug, const float* w4b4, float* out, int B, int C, long long S,
                           int O, long long plane, int nrl, const int* R, const long long* SR, const int* lim,
                           int num_sms, cudaStream_t stream);
const char* head_bwd_multi(const void* h, const void* W3aug, const void* W3T16, const float* W4, const float* dout,
                           long long n_dout, unsigned* amax_ws, void* g, float* gW3, float* gb3, float* gW4, float* gb4,
                           int B, int C, long long S, int O, long long plane, int nrl, const int* R,
                           const long long* SR, const int* lim, int num_sms, cudaStream_t stream);

}  // namespace dfno
