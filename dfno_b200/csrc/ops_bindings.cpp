// Bindings for the pointwise / spectral / optimizer / p2p launchers (kernels.h).
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>

#include "kernels.h"

namespace {

int sm_count() {
  static int n = 0;
  if (!n) n = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  return n;
}
cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }
void check(const char* err, const char* what) { TORCH_CHECK(err == nullptr, what, ": ", err ? err : ""); }
const float* fptr(const at::Tensor& t) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kFloat && t.is_contiguous(), "expected contiguous CUDA fp32 tensor");
  return t.data_ptr<float>();
}
float* fptr_mut(at::Tensor& t) { return const_cast<float*>(fptr(t)); }
void* bptr(const at::Tensor& t) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kBFloat16, "expected CUDA bf16 tensor");
  return t.data_ptr();
}

dfno::LiftDims lift_dims(const std::vector<int64_t>& d) {
  TORCH_CHECK(d.size() == 8 || d.size() == 12, "dims = [B, Cin, Tin, C, T, X, Y, Z] (+ padded [X, Y, Z, T])");
  dfno::LiftDims L;
  L.B = d[0]; L.Cin = d[1]; L.Tin = d[2]; L.C = d[3]; L.T = d[4]; L.X = d[5]; L.Y = d[6]; L.Z = d[7];
  return L;
}

// the padded extents of h when dims carries them (12 entries), else none
const dfno::LiftPad* lift_pad(const std::vector<int64_t>& d, dfno::LiftPad* buf) {
  if (d.size() != 12) return nullptr;
  buf->X = d[8]; buf->Y = d[9]; buf->Z = d[10]; buf->T = d[11];
  return buf;
}

void lift_fwd(const at::Tensor& x, const at::Tensor& W1, const at::Tensor& b1, const at::Tensor& W2,
              const at::Tensor& b2, at::Tensor& h, const std::vector<int64_t>& dims) {
  TORCH_CHECK(x.is_cuda() && x.is_contiguous(), "x must be a contiguous CUDA tensor");
  TORCH_CHECK(x.scalar_type() == at::kFloat || x.scalar_type() == at::kBFloat16, "x must be fp32 or bf16");
  c10::cuda::CUDAGuard guard(x.device());
  dfno::LiftPad pad;
  check(dfno::lift_fwd(x.data_ptr(), x.scalar_type() == at::kBFloat16, fptr(W1), fptr(b1), fptr(W2), fptr(b2),
                       bptr(h), lift_dims(dims), lift_pad(dims, &pad), sm_count(), cur_stream()), "lift_fwd");
}

// dx (optional): fp32 tensor of x's size, receives the input gradient
void lift_bwd(const at::Tensor& x, const at::Tensor& W1, const at::Tensor& b1, const at::Tensor& W2,
              const at::Tensor& b2, const at::Tensor& dh, at::Tensor& gW1, at::Tensor& gb1, at::Tensor& gW2,
              at::Tensor& gb2, const std::vector<int64_t>& dims, const c10::optional<at::Tensor>& dx) {
  TORCH_CHECK(x.is_cuda() && x.is_contiguous(), "x must be a contiguous CUDA tensor");
  TORCH_CHECK(x.scalar_type() == at::kFloat || x.scalar_type() == at::kBFloat16, "x must be fp32 or bf16");
  TORCH_CHECK(!dx || dx->numel() == x.numel(), "dx must have as many elements as x");
  c10::cuda::CUDAGuard guard(x.device());
  dfno::LiftPad pad;
  check(dfno::lift_bwd(x.data_ptr(), x.scalar_type() == at::kBFloat16, fptr(W1), fptr(b1), fptr(W2), fptr(b2),
                       bptr(dh), fptr_mut(gW1), fptr_mut(gb1), fptr_mut(gW2), fptr_mut(gb2),
                       dx ? const_cast<float*>(fptr(*dx)) : nullptr, lift_dims(dims), lift_pad(dims, &pad), sm_count(),
                       cur_stream()),
        "lift_bwd");
}

void bypass_gelu_fwd(const at::Tensor& h, at::Tensor& spec_pre, const at::Tensor& W,
                     const c10::optional<at::Tensor>& out, const c10::optional<at::Tensor>& out_cl, int64_t cl_pitch,
                     int64_t B, int64_t C, int64_t S, bool save_pre) {
  c10::cuda::CUDAGuard guard(h.device());
  check(dfno::bypass_gelu_fwd(bptr(h), bptr(spec_pre), fptr(W), out ? bptr(*out) : nullptr,
                              out_cl ? bptr(*out_cl) : nullptr, static_cast<int>(cl_pitch), static_cast<int>(B),
                              static_cast<int>(C), S, save_pre ? 1 : 0, sm_count(), cur_stream()), "bypass_gelu_fwd");
}

void bypass_gelu_bwd(const c10::optional<at::Tensor>& dout, const c10::optional<at::Tensor>& dout_cl, int64_t cl_pitch,
                     const at::Tensor& pre, const at::Tensor& W, at::Tensor& dpre, at::Tensor& dhb, int64_t B,
                     int64_t C, int64_t S) {
  TORCH_CHECK(dout.has_value() != dout_cl.has_value(), "give exactly one of dout / dout_cl");
  c10::cuda::CUDAGuard guard(pre.device());
  check(dfno::bypass_gelu_bwd(dout ? bptr(*dout) : nullptr, dout_cl ? bptr(*dout_cl) : nullptr,
                              static_cast<int>(cl_pitch), bptr(pre), fptr(W), bptr(dpre), bptr(dhb),
                              static_cast<int>(B), static_cast<int>(C), S, sm_count(), cur_stream()), "bypass_gelu_bwd");
}

void bypass_fwd_tc(const at::Tensor& h, at::Tensor& spec_pre, const at::Tensor& Wpad, const c10::optional<at::Tensor>& out,
                   const c10::optional<at::Tensor>& out_cl, int64_t cl_pitch, int64_t B, int64_t C, int64_t S, bool save_pre) {
  TORCH_CHECK(Wpad.dim() == 2 && Wpad.size(0) == 32 && Wpad.size(1) == 64 && Wpad.is_contiguous(), "Wpad [32,64]");
  c10::cuda::CUDAGuard guard(h.device());
  check(dfno::bypass_fwd_tc(bptr(h), bptr(spec_pre), bptr(Wpad), out ? bptr(*out) : nullptr,
                            out_cl ? bptr(*out_cl) : nullptr, static_cast<int>(cl_pitch), static_cast<int>(B),
                            static_cast<int>(C), S, save_pre ? 1 : 0, sm_count(), cur_stream()), "bypass_fwd_tc");
}

void bypass_bwd_tc(const c10::optional<at::Tensor>& dout, const c10::optional<at::Tensor>& dout_cl, int64_t cl_pitch,
                   at::Tensor& pre_dpre, const at::Tensor& h, const at::Tensor& WTpad, at::Tensor& dhb, at::Tensor& dW,
                   int64_t B, int64_t C, int64_t S) {
  TORCH_CHECK(dout.has_value() != dout_cl.has_value(), "give exactly one of dout / dout_cl");
  TORCH_CHECK(WTpad.dim() == 2 && WTpad.size(0) == 32 && WTpad.size(1) == 64 && WTpad.is_contiguous(), "WTpad [32,64]");
  c10::cuda::CUDAGuard guard(h.device());
  check(dfno::bypass_bwd_tc(dout ? bptr(*dout) : nullptr, dout_cl ? bptr(*dout_cl) : nullptr,
                            static_cast<int>(cl_pitch), bptr(pre_dpre), bptr(h), bptr(WTpad), bptr(dhb), fptr_mut(dW),
                            static_cast<int>(B), static_cast<int>(C), S, sm_count(), cur_stream()), "bypass_bwd_tc");
}

void spectral_mix_fwd(const at::Tensor& x, const at::Tensor& w, at::Tensor& y, int64_t B, int64_t C, int64_t Q) {
  c10::cuda::CUDAGuard guard(x.device());
  check(dfno::spectral_mix_fwd(bptr(x), fptr(w), bptr(y), static_cast<int>(B), static_cast<int>(C), Q, cur_stream()),
        "spectral_mix_fwd");
}

// dw None: dx only (frozen weights)
void spectral_mix_bwd(const at::Tensor& x, const at::Tensor& w, const at::Tensor& dy, at::Tensor& dx,
                      const c10::optional<at::Tensor>& dw, bool accumulate, int64_t B, int64_t C, int64_t Q) {
  c10::cuda::CUDAGuard guard(x.device());
  check(dfno::spectral_mix_bwd(bptr(x), fptr(w), bptr(dy), bptr(dx), dw ? const_cast<float*>(fptr(*dw)) : nullptr,
                               accumulate ? 1 : 0, static_cast<int>(B), static_cast<int>(C), Q, cur_stream()),
        "spectral_mix_bwd");
}

void adam_step(at::Tensor& p, const at::Tensor& g, at::Tensor& m, at::Tensor& v, double lr, double beta1, double beta2,
               double eps, double weight_decay, int64_t step, double grad_scale,
               const c10::optional<at::Tensor>& step_dev) {
  TORCH_CHECK(p.numel() == g.numel() && p.numel() == m.numel() && p.numel() == v.numel(), "adam: size mismatch");
  c10::cuda::CUDAGuard guard(p.device());
  if (step < 1) step = 1;
  const double bias1 = 1.0 - std::pow(beta1, static_cast<double>(step));
  const double bias2 = 1.0 - std::pow(beta2, static_cast<double>(step));
  check(dfno::adam_step(fptr_mut(p), fptr(g), fptr_mut(m), fptr_mut(v), p.numel(), static_cast<float>(lr),
                        static_cast<float>(beta1), static_cast<float>(beta2), static_cast<float>(eps),
                        static_cast<float>(weight_decay), static_cast<float>(bias1), static_cast<float>(bias2),
                        static_cast<float>(grad_scale), step_dev ? fptr(*step_dev) : nullptr, sm_count(), cur_stream()),
        "adam_step");
}

double* dptr_mut(at::Tensor& t) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kDouble && t.is_contiguous(), "expected contiguous CUDA fp64 tensor");
  return t.data_ptr<double>();
}

void adam_step_dev(at::Tensor& p, const at::Tensor& g, at::Tensor& m, at::Tensor& v, at::Tensor& hparams,
                   const at::Tensor& step_dev, double grad_scale, const c10::optional<at::Tensor>& sumsq,
                   const c10::optional<at::Tensor>& norm_out) {
  TORCH_CHECK(p.numel() == g.numel() && p.numel() == m.numel() && p.numel() == v.numel(), "adam: size mismatch");
  TORCH_CHECK(hparams.numel() >= 8 && step_dev.numel() >= 1, "adam: hparams holds 8 doubles, step_dev one float");
  TORCH_CHECK(sumsq.has_value() == norm_out.has_value(), "adam: sumsq and norm_out go together");
  TORCH_CHECK(!sumsq || sumsq->numel() >= 1, "adam: empty sumsq");
  c10::cuda::CUDAGuard guard(p.device());
  at::Tensor sq = sumsq ? *sumsq : at::Tensor(), nrm = norm_out ? *norm_out : at::Tensor();
  check(dfno::adam_step_dev(fptr_mut(p), fptr(g), fptr_mut(m), fptr_mut(v), p.numel(), dptr_mut(hparams),
                            fptr(step_dev), static_cast<float>(grad_scale), sumsq ? dptr_mut(sq) : nullptr,
                            norm_out ? fptr_mut(nrm) : nullptr, sm_count(), cur_stream()),
        "adam_step_dev");
}

void adam_set_hparams(at::Tensor& hparams, double lr, double beta1, double beta2, double eps, double weight_decay,
                      bool decoupled, double max_norm) {
  TORCH_CHECK(hparams.numel() >= 8, "adam: hparams holds 8 doubles");
  c10::cuda::CUDAGuard guard(hparams.device());
  check(dfno::adam_set_hparams(dptr_mut(hparams), lr, beta1, beta2, eps, weight_decay, decoupled, max_norm,
                               cur_stream()), "adam_set_hparams");
}

void sumsq(const at::Tensor& x, at::Tensor& out, at::Tensor& partials, at::Tensor& ticket) {
  TORCH_CHECK(x.dim() == 1, "sumsq: x must be a 1-D fp32 vector");
  TORCH_CHECK(out.numel() >= 1, "sumsq: empty out");
  TORCH_CHECK(ticket.is_cuda() && ticket.scalar_type() == at::kInt && ticket.numel() >= 1, "sumsq: int32 ticket");
  TORCH_CHECK(partials.numel() >= 1, "sumsq: partials needs room for at least one block");
  c10::cuda::CUDAGuard guard(x.device());
  check(dfno::sumsq(fptr(x), x.numel(), dptr_mut(out), dptr_mut(partials), static_cast<int>(partials.numel()),
                    reinterpret_cast<unsigned*>(ticket.data_ptr<int>()), sm_count(), cur_stream()), "sumsq");
}

void p2p_sum_f64(const std::vector<int64_t>& buf_ptrs, at::Tensor& out) {
  const int world = static_cast<int>(buf_ptrs.size());
  TORCH_CHECK(world >= 1 && world <= 8, "p2p_sum_f64: 1..8 peer pointers");
  TORCH_CHECK(out.numel() >= 1, "p2p_sum_f64: empty out");
  double* peers[8];
  for (int i = 0; i < 8; ++i) peers[i] = reinterpret_cast<double*>(buf_ptrs[i < world ? i : 0]);
  check(dfno::p2p_sum_f64(peers, dptr_mut(out), world, cur_stream()), "p2p_sum_f64");
}

void p2p_barrier(const std::vector<int64_t>& flag_ptrs, int64_t rank, int64_t epoch, double timeout_s) {
  const int world = static_cast<int>(flag_ptrs.size());
  uint32_t* peers[8];
  for (int i = 0; i < 8; ++i) peers[i] = reinterpret_cast<uint32_t*>(flag_ptrs[i < world ? i : 0]);
  check(dfno::p2p_barrier(peers, peers[rank], static_cast<int>(rank), world, static_cast<uint32_t>(epoch),
                          static_cast<unsigned long long>(timeout_s * 1e9), cur_stream()), "p2p_barrier");
}

void p2p_allreduce_small(const std::vector<int64_t>& buf_ptrs, at::Tensor& out, int64_t n, int64_t rank) {
  const int world = static_cast<int>(buf_ptrs.size());
  float* peers[8];
  for (int i = 0; i < 8; ++i) peers[i] = reinterpret_cast<float*>(buf_ptrs[i < world ? i : 0]);
  check(dfno::p2p_allreduce_small(peers, fptr_mut(out), n, static_cast<int>(rank), world, cur_stream()),
        "p2p_allreduce_small");
}

void p2p_alltoall(const at::Tensor& send, const std::vector<int64_t>& send_off, const std::vector<int64_t>& recv_ptrs,
                  const std::vector<int64_t>& dst_off, int64_t ctas_per_peer) {
  const int world = static_cast<int>(recv_ptrs.size());
  TORCH_CHECK(send.is_cuda() && send.is_contiguous(), "send must be a contiguous CUDA tensor");
  TORCH_CHECK(static_cast<int>(send_off.size()) == world + 1 && static_cast<int>(dst_off.size()) == world,
              "offset tables do not match the world size");
  c10::cuda::CUDAGuard guard(send.device());
  void* peers[8]; long long so[9]; long long doff[8];
  for (int i = 0; i < 8; ++i) { peers[i] = reinterpret_cast<void*>(recv_ptrs[i < world ? i : 0]); doff[i] = i < world ? dst_off[i] : 0; }
  for (int i = 0; i <= 8; ++i) so[i] = send_off[i <= world ? i : world];
  check(dfno::p2p_alltoall(send.data_ptr(), so, peers, doff, world, static_cast<int>(ctas_per_peer), cur_stream()),
        "p2p_alltoall");
}

// D[Ma, Nb] (fp32, pre-zeroed or accumulated) += A[Ma, K] * B[Nb, K]^T, K contiguous
void kreduce_gemm(const at::Tensor& A, int64_t lda, int64_t Ma, const at::Tensor& Bm, int64_t ldb, int64_t Nb,
                  int64_t K, at::Tensor& D) {
  TORCH_CHECK(D.dim() == 2 && D.size(0) >= Ma && D.size(1) >= Nb, "D too small");
  c10::cuda::CUDAGuard guard(A.device());
  check(dfno::kreduce_gemm(bptr(A), lda, static_cast<int>(Ma), bptr(Bm), ldb, static_cast<int>(Nb), K, fptr_mut(D),
                           D.stride(0), sm_count(), cur_stream()), "kreduce_gemm");
}

void permute_u32(const at::Tensor& src, at::Tensor& dst, const std::vector<int64_t>& size,
                 const std::vector<int64_t>& sstr, const std::vector<int64_t>& dstr) {
  TORCH_CHECK(size.size() == sstr.size() && size.size() == dstr.size() && !size.empty() && size.size() <= 6,
              "permute_u32: 1..6 matching digits");
  c10::cuda::CUDAGuard guard(src.device());
  int sz[6]; long long ss[6], ds[6];
  for (size_t i = 0; i < size.size(); ++i) { sz[i] = static_cast<int>(size[i]); ss[i] = sstr[i]; ds[i] = dstr[i]; }
  check(dfno::permute_u32(src.data_ptr(), dst.data_ptr(), static_cast<int>(size.size()), sz, ss, ds, sm_count(),
                          cur_stream()), "permute_u32");
}

std::vector<at::Tensor> gelu_probe(const at::Tensor& x) {
  c10::cuda::CUDAGuard guard(x.device());
  at::Tensor y = at::empty_like(x), dy = at::empty_like(x);
  check(dfno::gelu_probe(fptr(x), y.data_ptr<float>(), dy.data_ptr<float>(), x.numel(), cur_stream()), "gelu_probe");
  return {y, dy};
}

std::vector<at::Tensor> gelu_probe_h2(const at::Tensor& x) {
  TORCH_CHECK(x.numel() % 2 == 0, "even length");
  c10::cuda::CUDAGuard guard(x.device());
  at::Tensor y = at::empty_like(x), dy = at::empty_like(x);
  check(dfno::gelu_probe_h2(fptr(x), y.data_ptr<float>(), dy.data_ptr<float>(), x.numel(), cur_stream()), "gelu_probe_h2");
  return {y, dy};
}

void head_bwd(const at::Tensor& hcl, int64_t npos, int64_t C, int64_t CP, const at::Tensor& W3pad,
              const at::Tensor& W3Tpad, const at::Tensor& b3, const at::Tensor& W4, const at::Tensor& dout,
              const std::vector<int64_t>& radices, const std::vector<int64_t>& strides, at::Tensor& gcl,
              at::Tensor& gW3, at::Tensor& gb3, at::Tensor& gW4, at::Tensor& gb4) {
  TORCH_CHECK(radices.size() == strides.size() && !radices.empty() && radices.size() <= 4, "1..4 row digits");
  TORCH_CHECK(W3pad.dim() == 2 && W3pad.size(0) == 128 && W3pad.size(1) == 64 && W3pad.is_contiguous(), "W3pad [128,64]");
  TORCH_CHECK(W3Tpad.dim() == 2 && W3Tpad.size(0) == 32 && W3Tpad.size(1) == 128 && W3Tpad.is_contiguous(), "W3Tpad [32,128]");
  c10::cuda::CUDAGuard guard(hcl.device());
  int R[4]; long long SR[4];
  for (size_t i = 0; i < 4; ++i) { R[i] = i < radices.size() ? static_cast<int>(radices[i]) : 1; SR[i] = i < strides.size() ? strides[i] : 0; }
  check(dfno::head_bwd(bptr(hcl), npos, static_cast<int>(C), static_cast<int>(CP), bptr(W3pad), bptr(W3Tpad), fptr(b3),
                       fptr(W4), fptr(dout), static_cast<int>(radices.size()), R, SR, bptr(gcl), fptr_mut(gW3),
                       fptr_mut(gb3), fptr_mut(gW4), fptr_mut(gb4), sm_count(), cur_stream()), "head_bwd");
}

void fft_radix(const at::Tensor& x, at::Tensor& y, int64_t N, int64_t lines, bool inverse, bool in_real, bool out_real,
               bool one_sided, int64_t m) {
  TORCH_CHECK(x.is_cuda() && y.is_cuda() && x.is_contiguous() && y.is_contiguous(), "contiguous CUDA tensors");
  TORCH_CHECK(x.scalar_type() == y.scalar_type() && (x.scalar_type() == at::kFloat || x.scalar_type() == at::kBFloat16),
              "fp32 or bf16 (same type in and out)");
  c10::cuda::CUDAGuard guard(x.device());
  check(dfno::fft_radix(x.data_ptr(), y.data_ptr(), x.scalar_type() == at::kBFloat16, static_cast<int>(N), lines,
                        inverse, in_real, out_real, one_sided, static_cast<int>(m), sm_count(), cur_stream()), "fft_radix");
}

// pre_prev / h_dw / dW (adjoint only, optional): fold the neighbouring pointwise backward into the adjoint
// (spectral_out_adj); with pre_prev, `out` is not written
void spectral_out(const at::Tensor& U, const at::Tensor& h, const at::Tensor& Bop, const at::Tensor& W, bool transpose_w,
                  const c10::optional<at::Tensor>& pre, at::Tensor& out, int64_t B, int64_t C, int64_t L, int64_t Z,
                  int64_t K1, bool gelu, bool save_pre, const c10::optional<at::Tensor>& pre_prev,
                  const c10::optional<at::Tensor>& h_dw, const c10::optional<at::Tensor>& dW) {
  TORCH_CHECK(Bop.dim() == 2 && Bop.is_contiguous(), "operator must be a contiguous [n_pad, k_pad] tensor");
  c10::cuda::CUDAGuard guard(U.device());
  if (pre_prev || h_dw || dW) {
    TORCH_CHECK(transpose_w && !gelu, "pre_prev / h_dw / dW: adjoint only");
    TORCH_CHECK(!dW || (dW->scalar_type() == at::kFloat && dW->numel() >= C * C), "dW: fp32 [C, C]");
    check(dfno::spectral_out_adj(bptr(U), bptr(h), bptr(Bop), static_cast<int>(Bop.size(0)),
                                 static_cast<int>(Bop.size(1)), fptr(W), pre_prev ? bptr(*pre_prev) : nullptr, bptr(out),
                                 h_dw ? bptr(*h_dw) : nullptr, dW ? const_cast<float*>(fptr(*dW)) : nullptr, static_cast<int>(B),
                                 static_cast<int>(C), L, static_cast<int>(Z), static_cast<int>(K1), sm_count(),
                                 cur_stream()), "spectral_out_adj");
    return;
  }
  check(dfno::spectral_out(bptr(U), bptr(h), bptr(Bop), static_cast<int>(Bop.size(0)), static_cast<int>(Bop.size(1)),
                           fptr(W), transpose_w ? 1 : 0, pre ? bptr(*pre) : nullptr, bptr(out), static_cast<int>(B),
                           static_cast<int>(C), L, static_cast<int>(Z), static_cast<int>(K1), gelu ? 1 : 0,
                           save_pre ? 1 : 0, sm_count(), cur_stream()), "spectral_out");
}

// "" when the folded adjoint takes the shape, the reason otherwise (no launch, no device needed)
std::string spectral_out_adj_check(int64_t n_pad, int64_t k_pad, int64_t C, int64_t Z, int64_t K1, bool dpre, bool dw) {
  const char* e = dfno::spectral_out_adj_check(static_cast<int>(n_pad), static_cast<int>(k_pad), static_cast<int>(C),
                                               static_cast<int>(Z), static_cast<int>(K1), dpre ? 1 : 0, dw ? 1 : 0);
  return e ? std::string(e) : std::string();
}

void spectral_in(const at::Tensor& h, const at::Tensor& op1, const at::Tensor& op2, const std::vector<int64_t>& dst_ptrs,
                 int64_t dst_off, const std::vector<int64_t>& dstr, int64_t BC, int64_t X, int64_t Yl, int64_t T, int64_t Z,
                 int64_t KZ, int64_t mt) {
  TORCH_CHECK(op1.dim() == 2 && op1.is_contiguous() && op2.dim() == 2 && op2.is_contiguous(), "operators: contiguous [n_pad, k_pad]");
  TORCH_CHECK(!dst_ptrs.empty() && dst_ptrs.size() <= 8 && dstr.size() == 4, "1..8 destinations, 4 strides");
  TORCH_CHECK(h.numel() >= BC * X * Yl * T * Z, "activation smaller than its description");
  c10::cuda::CUDAGuard guard(h.device());
  long long ptrs[8], str[4];
  for (size_t i = 0; i < dst_ptrs.size(); ++i) ptrs[i] = dst_ptrs[i];
  for (size_t i = 0; i < 4; ++i) str[i] = dstr[i];
  check(dfno::spectral_in(bptr(h), bptr(op1), static_cast<int>(op1.size(0)), static_cast<int>(op1.size(1)), bptr(op2),
                          static_cast<int>(op2.size(0)), static_cast<int>(op2.size(1)), ptrs, static_cast<int>(dst_ptrs.size()),
                          dst_off, str, static_cast<int>(BC), static_cast<int>(X), static_cast<int>(Yl), static_cast<int>(T),
                          static_cast<int>(Z), static_cast<int>(KZ), static_cast<int>(mt), sm_count(), cur_stream()),
        "spectral_in");
}

// "" when the fused front stage supports the shape, the reason otherwise (no launch, no device needed)
std::string spectral_in_check(int64_t n1_pad, int64_t k1_pad, int64_t n2_pad, int64_t k2_pad, int64_t P, int64_t dst_off,
                              const std::vector<int64_t>& dstr, int64_t BC, int64_t X, int64_t Yl, int64_t T, int64_t Z,
                              int64_t KZ, int64_t mt) {
  TORCH_CHECK(dstr.size() == 4, "4 strides");
  long long str[4];
  for (size_t i = 0; i < 4; ++i) str[i] = dstr[i];
  const char* e = dfno::spectral_in_check(static_cast<int>(n1_pad), static_cast<int>(k1_pad), static_cast<int>(n2_pad),
                                          static_cast<int>(k2_pad), static_cast<int>(P), dst_off, str, static_cast<int>(BC),
                                          static_cast<int>(X), static_cast<int>(Yl), static_cast<int>(T), static_cast<int>(Z),
                                          static_cast<int>(KZ), static_cast<int>(mt), nullptr);
  return e ? std::string(e) : std::string();
}

// {positions per tile, positions per store chunk, epilogue groups, TMA ring stages} the kernel would use
std::vector<int64_t> spectral_in_config(int64_t n1_pad, int64_t k1_pad, int64_t n2_pad, int64_t k2_pad, int64_t P,
                                        int64_t dst_off, const std::vector<int64_t>& dstr, int64_t BC, int64_t X, int64_t Yl,
                                        int64_t T, int64_t Z, int64_t KZ, int64_t mt) {
  TORCH_CHECK(dstr.size() == 4, "4 strides");
  long long str[4];
  for (size_t i = 0; i < 4; ++i) str[i] = dstr[i];
  int cfg[4] = {0, 0, 0, 0};
  const char* e = dfno::spectral_in_check(static_cast<int>(n1_pad), static_cast<int>(k1_pad), static_cast<int>(n2_pad),
                                          static_cast<int>(k2_pad), static_cast<int>(P), dst_off, str, static_cast<int>(BC),
                                          static_cast<int>(X), static_cast<int>(Yl), static_cast<int>(T), static_cast<int>(Z),
                                          static_cast<int>(KZ), static_cast<int>(mt), cfg);
  TORCH_CHECK(!e, e);
  return {cfg[0], cfg[1], cfg[2], cfg[3]};
}

void sq_partials(const at::Tensor& yh, const at::Tensor& y, at::Tensor& part, int64_t B) {
  TORCH_CHECK(yh.is_cuda() && y.is_cuda() && yh.scalar_type() == at::kFloat && y.scalar_type() == at::kFloat &&
              yh.is_contiguous() && y.is_contiguous() && yh.numel() == y.numel() && yh.numel() % B == 0, "fp32 contiguous fields");
  TORCH_CHECK(part.scalar_type() == at::kFloat && part.numel() >= 2 * B && part.is_contiguous(), "part: 2B floats");
  c10::cuda::CUDAGuard guard(yh.device());
  check(dfno::sq_partials(fptr(yh), fptr(y), fptr_mut(part), yh.numel() / B, static_cast<int>(B), sm_count(), cur_stream()),
        "sq_partials");
}

void scaled_diff(const at::Tensor& yh, const at::Tensor& y, const at::Tensor& scale, at::Tensor& grad, int64_t B) {
  TORCH_CHECK(yh.is_cuda() && yh.scalar_type() == at::kFloat && y.scalar_type() == at::kFloat && grad.scalar_type() == at::kFloat &&
              yh.is_contiguous() && y.is_contiguous() && grad.is_contiguous() && yh.numel() == y.numel() &&
              grad.numel() == yh.numel() && yh.numel() % B == 0, "fp32 contiguous fields");
  TORCH_CHECK(scale.scalar_type() == at::kFloat && (scale.numel() == 1 || scale.numel() == B), "scale: 1 or B floats");
  c10::cuda::CUDAGuard guard(yh.device());
  check(dfno::scaled_diff(fptr(yh), fptr(y), fptr(scale), fptr_mut(grad), yh.numel() / B, static_cast<int>(B),
                          scale.numel() == B ? 1 : 0, sm_count(), cur_stream()), "scaled_diff");
}

void dpre_dw(const at::Tensor& g, at::Tensor& pre_dpre, const at::Tensor& h, at::Tensor& dW, int64_t B, int64_t C,
             int64_t L, int64_t Z) {
  c10::cuda::CUDAGuard guard(g.device());
  check(dfno::dpre_dw(bptr(g), bptr(pre_dpre), bptr(h), fptr_mut(dW), static_cast<int>(B), static_cast<int>(C), L,
                      static_cast<int>(Z), sm_count(), cur_stream()), "dpre_dw");
}

// row digits (+ per-digit interior bounds of a zero-padded activation, `limits`, empty for none) -> launcher arrays
const int* row_digits(const std::vector<int64_t>& radices, const std::vector<int64_t>& strides,
                      const std::vector<int64_t>& limits, int* R, long long* SR, int* lim) {
  const size_t maxd = limits.empty() ? 4 : 5;
  TORCH_CHECK(radices.size() == strides.size() && !radices.empty() && radices.size() <= maxd,
              limits.empty() ? "1..4 row digits" : "1..5 row digits");
  TORCH_CHECK(limits.empty() || limits.size() == radices.size(), "one limit per row digit");
  for (size_t i = 0; i < 5; ++i) {
    R[i] = i < radices.size() ? static_cast<int>(radices[i]) : 1;
    SR[i] = i < strides.size() ? strides[i] : 0;
    lim[i] = i < limits.size() ? static_cast<int>(limits[i]) : 1;
  }
  return limits.empty() ? nullptr : lim;
}

void head_fwd(const at::Tensor& h, const at::Tensor& W3aug, const at::Tensor& w4b4, at::Tensor& out, int64_t B,
              int64_t C, int64_t S, const std::vector<int64_t>& radices, const std::vector<int64_t>& strides,
              const std::vector<int64_t>& limits) {
  TORCH_CHECK(W3aug.dim() == 2 && W3aug.size(0) == 128 && W3aug.size(1) == (C + 1 > 64 ? 128 : 64) &&
              W3aug.is_contiguous(), "W3aug [128, 64] ([128, 128] when C + 1 > 64)");
  TORCH_CHECK(w4b4.numel() >= 129, "w4b4 = [W4 (128), b4]");
  c10::cuda::CUDAGuard guard(h.device());
  int R[5], lim[5]; long long SR[5];
  const int* lp = row_digits(radices, strides, limits, R, SR, lim);
  check(dfno::head_fwd(bptr(h), bptr(W3aug), fptr(w4b4), fptr_mut(out), static_cast<int>(B), static_cast<int>(C), S,
                       static_cast<int>(radices.size()), R, SR, lp, sm_count(), cur_stream()), "head_fwd");
}

void head_bwd2(const at::Tensor& h, const at::Tensor& W3aug, const at::Tensor& W3T16, const at::Tensor& W4,
               const at::Tensor& dout, at::Tensor& amax_ws, at::Tensor& g, at::Tensor& gW3, at::Tensor& gb3,
               at::Tensor& gW4, at::Tensor& gb4, int64_t B, int64_t C, int64_t S, const std::vector<int64_t>& radices,
               const std::vector<int64_t>& strides, const std::vector<int64_t>& limits) {
  TORCH_CHECK(W3aug.dim() == 2 && W3aug.size(0) == 128 && W3aug.size(1) == (C + 1 > 64 ? 128 : 64) &&
              W3aug.is_contiguous(), "W3aug [128, 64] ([128, 128] when C + 1 > 64)");
  TORCH_CHECK(W3T16.is_cuda() && W3T16.scalar_type() == at::kHalf && W3T16.dim() == 2 && W3T16.size(1) == 128 &&
              W3T16.size(0) == (C + 1 + 15) / 16 * 16 && W3T16.is_contiguous(), "W3T16: fp16 [ceil16(C+1), 128]");
  TORCH_CHECK(amax_ws.is_cuda() && amax_ws.numel() >= 1 && amax_ws.element_size() == 4, "amax_ws: one 32-bit word");
  c10::cuda::CUDAGuard guard(h.device());
  int R[5], lim[5]; long long SR[5];
  const int* lp = row_digits(radices, strides, limits, R, SR, lim);
  check(dfno::head_bwd2(bptr(h), bptr(W3aug), W3T16.data_ptr(), fptr(W4), fptr(dout), dout.numel(),
                        reinterpret_cast<unsigned*>(amax_ws.data_ptr()), bptr(g), fptr_mut(gW3), fptr_mut(gb3),
                        fptr_mut(gW4), fptr_mut(gb4), static_cast<int>(B), static_cast<int>(C), S,
                        static_cast<int>(radices.size()), R, SR, lp, sm_count(), cur_stream()), "head_bwd2");
}

// out: fp32 [B, O, ...] addressed through the row digits, output channel o at + o * plane
void head_fwd_multi(const at::Tensor& h, const at::Tensor& W3aug, const at::Tensor& w4b4, at::Tensor& out, int64_t B,
                    int64_t C, int64_t S, int64_t O, int64_t plane, const std::vector<int64_t>& radices,
                    const std::vector<int64_t>& strides, const std::vector<int64_t>& limits) {
  TORCH_CHECK(W3aug.dim() == 2 && W3aug.size(0) == 128 && W3aug.size(1) == 64 && W3aug.is_contiguous(), "W3aug [128,64]");
  TORCH_CHECK(w4b4.numel() >= O * 129, "w4b4 = [W4 (O x 128), b4 (O)]");
  TORCH_CHECK(out.numel() >= B * O * plane, "out smaller than B * O * plane");
  c10::cuda::CUDAGuard guard(h.device());
  int R[5], lim[5]; long long SR[5];
  const int* lp = row_digits(radices, strides, limits, R, SR, lim);
  check(dfno::head_fwd_multi(bptr(h), bptr(W3aug), fptr(w4b4), fptr_mut(out), static_cast<int>(B), static_cast<int>(C),
                             S, static_cast<int>(O), plane, static_cast<int>(radices.size()), R, SR, lp, sm_count(),
                             cur_stream()), "head_fwd_multi");
}

void head_bwd_multi(const at::Tensor& h, const at::Tensor& W3aug, const at::Tensor& W3T16, const at::Tensor& W4,
                    const at::Tensor& dout, at::Tensor& amax_ws, at::Tensor& g, at::Tensor& gW3, at::Tensor& gb3,
                    at::Tensor& gW4, at::Tensor& gb4, int64_t B, int64_t C, int64_t S, int64_t O, int64_t plane,
                    const std::vector<int64_t>& radices, const std::vector<int64_t>& strides,
                    const std::vector<int64_t>& limits) {
  TORCH_CHECK(W3aug.dim() == 2 && W3aug.size(0) == 128 && W3aug.size(1) == 64 && W3aug.is_contiguous(), "W3aug [128,64]");
  TORCH_CHECK(W3T16.is_cuda() && W3T16.scalar_type() == at::kHalf && W3T16.dim() == 2 && W3T16.size(1) == 128 &&
              W3T16.size(0) == (C + 1 + 15) / 16 * 16 && W3T16.is_contiguous(), "W3T16: fp16 [ceil16(C+1), 128]");
  TORCH_CHECK(W4.numel() == O * 128 && gW4.numel() == O * 128 && gb4.numel() == O, "W4 / dW4 [O, 128], db4 [O]");
  TORCH_CHECK(dout.numel() >= B * O * plane, "dout smaller than B * O * plane");
  TORCH_CHECK(amax_ws.is_cuda() && amax_ws.numel() >= 1 && amax_ws.element_size() == 4, "amax_ws: one 32-bit word");
  c10::cuda::CUDAGuard guard(h.device());
  int R[5], lim[5]; long long SR[5];
  const int* lp = row_digits(radices, strides, limits, R, SR, lim);
  check(dfno::head_bwd_multi(bptr(h), bptr(W3aug), W3T16.data_ptr(), fptr(W4), fptr(dout), dout.numel(),
                             reinterpret_cast<unsigned*>(amax_ws.data_ptr()), bptr(g), fptr_mut(gW3), fptr_mut(gb3),
                             fptr_mut(gW4), fptr_mut(gb4), static_cast<int>(B), static_cast<int>(C), S,
                             static_cast<int>(O), plane, static_cast<int>(radices.size()), R, SR, lp, sm_count(),
                             cur_stream()), "head_bwd_multi");
}

}  // namespace

void register_ops(pybind11::module& m) {
  m.def("fft_radix", &fft_radix);
  m.def("sq_partials", &sq_partials);
  m.def("scaled_diff", &scaled_diff);
  m.def("spectral_in", &spectral_in);
  m.def("spectral_in_check", &spectral_in_check);
  m.def("spectral_in_config", &spectral_in_config);
  m.def("spectral_out", &spectral_out, py::arg("U"), py::arg("h"), py::arg("Bop"), py::arg("W"), py::arg("transpose_w"),
        py::arg("pre"), py::arg("out"), py::arg("B"), py::arg("C"), py::arg("L"), py::arg("Z"), py::arg("K1"),
        py::arg("gelu"), py::arg("save_pre"), py::arg("pre_prev") = c10::nullopt, py::arg("h_dw") = c10::nullopt,
        py::arg("dW") = c10::nullopt);
  m.def("spectral_out_adj_check", &spectral_out_adj_check);
  m.def("dpre_dw", &dpre_dw);
  // limits (optional): per-digit interior bounds of a zero-padded h
  m.def("head_fwd", &head_fwd, py::arg("h"), py::arg("W3aug"), py::arg("w4b4"), py::arg("out"), py::arg("B"), py::arg("C"),
        py::arg("S"), py::arg("radices"), py::arg("strides"), py::arg("limits") = std::vector<int64_t>{});
  m.def("head_bwd2", &head_bwd2, py::arg("h"), py::arg("W3aug"), py::arg("W3T16"), py::arg("W4"), py::arg("dout"),
        py::arg("amax_ws"), py::arg("g"), py::arg("gW3"), py::arg("gb3"), py::arg("gW4"), py::arg("gb4"), py::arg("B"),
        py::arg("C"), py::arg("S"), py::arg("radices"), py::arg("strides"), py::arg("limits") = std::vector<int64_t>{});
  m.def("head_fwd_multi", &head_fwd_multi, py::arg("h"), py::arg("W3aug"), py::arg("w4b4"), py::arg("out"), py::arg("B"),
        py::arg("C"), py::arg("S"), py::arg("O"), py::arg("plane"), py::arg("radices"), py::arg("strides"),
        py::arg("limits") = std::vector<int64_t>{});
  m.def("head_bwd_multi", &head_bwd_multi, py::arg("h"), py::arg("W3aug"), py::arg("W3T16"), py::arg("W4"),
        py::arg("dout"), py::arg("amax_ws"), py::arg("g"), py::arg("gW3"), py::arg("gb3"), py::arg("gW4"), py::arg("gb4"),
        py::arg("B"), py::arg("C"), py::arg("S"), py::arg("O"), py::arg("plane"), py::arg("radices"), py::arg("strides"),
        py::arg("limits") = std::vector<int64_t>{});
  m.def("lift_fwd", &lift_fwd);
  m.def("lift_bwd", &lift_bwd, py::arg("x"), py::arg("W1"), py::arg("b1"), py::arg("W2"), py::arg("b2"), py::arg("dh"),
        py::arg("gW1"), py::arg("gb1"), py::arg("gW2"), py::arg("gb2"), py::arg("dims"), py::arg("dx") = c10::nullopt);
  m.def("bypass_gelu_fwd", &bypass_gelu_fwd);
  m.def("bypass_gelu_bwd", &bypass_gelu_bwd);
  m.def("bypass_fwd_tc", &bypass_fwd_tc);
  m.def("bypass_bwd_tc", &bypass_bwd_tc);
  m.def("spectral_mix_fwd", &spectral_mix_fwd);
  m.def("spectral_mix_bwd", &spectral_mix_bwd);
  m.def("adam_step", &adam_step, py::arg("p"), py::arg("g"), py::arg("m"), py::arg("v"), py::arg("lr"), py::arg("beta1"),
        py::arg("beta2"), py::arg("eps"), py::arg("weight_decay"), py::arg("step"), py::arg("grad_scale"),
        py::arg("step_dev") = c10::nullopt);
  m.def("adam_step_dev", &adam_step_dev, py::arg("p"), py::arg("g"), py::arg("m"), py::arg("v"), py::arg("hparams"),
        py::arg("step_dev"), py::arg("grad_scale"), py::arg("sumsq") = c10::nullopt, py::arg("norm_out") = c10::nullopt);
  m.def("adam_set_hparams", &adam_set_hparams, py::arg("hparams"), py::arg("lr"), py::arg("beta1"), py::arg("beta2"),
        py::arg("eps"), py::arg("weight_decay"), py::arg("decoupled"), py::arg("max_norm"));
  m.def("sumsq", &sumsq, py::arg("x"), py::arg("out"), py::arg("partials"), py::arg("ticket"));
  m.def("p2p_sum_f64", &p2p_sum_f64);
  m.def("p2p_barrier", &p2p_barrier);
  m.def("p2p_allreduce_small", &p2p_allreduce_small);
  m.def("p2p_alltoall", &p2p_alltoall);
  m.def("kreduce_gemm", &kreduce_gemm);
  m.def("head_bwd", &head_bwd);
  m.def("gelu_probe", &gelu_probe);
  m.def("gelu_probe_h2", &gelu_probe_h2);
  m.def("permute_u32", &permute_u32);
}
