// Python bindings (torch extension) for the sm_90a kernels.  The kernels themselves are
// torch-free CUDA translation units; this file only unpacks tensors / streams.
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>

#include "dft_gemm.h"
#include "kernels.h"

namespace {

int sm_count() {
  static int n = 0;
  if (!n) n = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  return n;
}

cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }

void check(const char* err, const char* what) {
  TORCH_CHECK(err == nullptr, what, ": ", err ? err : "");
}

// epi = [mode, out_fp32, ldc, nrl, R0..R3, SR0..SR3, J0, J1, SJ0, SJ1, peer_sel, peer_lvl, peer_div, base_off]
// EPI_BOX_STORE appends the box geometry: [..., mt, mtp, kzl, KZ, Yl, y0, bcx, base_off] (dft_gemm.h, BoxGeom)
void dft_gemm(const at::Tensor& A, int64_t M, int64_t K, int64_t lda, const at::Tensor& Bmat, int64_t N,
              const std::vector<int64_t>& epi, const std::vector<int64_t>& peer_ptrs,
              const c10::optional<at::Tensor>& add_src, int64_t ld_add, int64_t max_ctas,
              const c10::optional<at::Tensor>& v0, const c10::optional<at::Tensor>& v1, double s0, bool a_f16) {
  TORCH_CHECK(A.is_cuda() && A.scalar_type() == (a_f16 ? at::kHalf : at::kBFloat16), "A must be a CUDA bf16 (or, with a_f16, fp16) tensor");
  TORCH_CHECK(Bmat.is_cuda() && Bmat.scalar_type() == at::kBFloat16 && Bmat.dim() == 2 && Bmat.is_contiguous(),
              "operator must be a contiguous CUDA bf16 [n_pad, k_pad] tensor");
  const bool boxed = !epi.empty() && epi[0] == dfno::EPI_BOX_STORE;
  TORCH_CHECK(epi.size() == (boxed ? 28u : 20u), "epi descriptor must have 20 entries (28 for the box store)");
  TORCH_CHECK(!peer_ptrs.empty() && peer_ptrs.size() <= 8, "1..8 peer pointers");
  c10::cuda::CUDAGuard guard(A.device());
  dfno::GemmParams p{};
  p.M = M; p.N = static_cast<int>(N); p.K = static_cast<int>(K);
  p.n_pad = static_cast<int>(Bmat.size(0)); p.k_pad = static_cast<int>(Bmat.size(1));
  p.a_f16 = a_f16 ? 1 : 0;
  auto& e = p.epi;
  e.mode = static_cast<int>(epi[0]); e.out_fp32 = static_cast<int>(epi[1]); e.ldc = epi[2];
  e.nrl = static_cast<int>(epi[3]);
  for (int i = 0; i < 4; ++i) { e.R[i] = static_cast<int>(epi[4 + i]); e.SR[i] = epi[8 + i]; }
  e.J[0] = static_cast<int>(epi[12]); e.J[1] = static_cast<int>(epi[13]);
  e.SJ[0] = epi[14]; e.SJ[1] = epi[15];
  e.peer_sel = static_cast<int>(epi[16]); e.peer_lvl = static_cast<int>(epi[17]);
  e.peer_div = static_cast<int>(epi[18]); e.base_off = epi[19];
  for (size_t i = 0; i < 8; ++i)
    e.peers[i] = reinterpret_cast<void*>(i < peer_ptrs.size() ? peer_ptrs[i] : peer_ptrs[0]);
  e.add_src = nullptr; e.ld_add = ld_add;
  if (add_src.has_value()) {
    TORCH_CHECK(add_src->scalar_type() == at::kBFloat16, "add_src must be bf16");
    e.add_src = add_src->data_ptr();
  }
  e.v0 = nullptr; e.v1 = nullptr; e.s0 = static_cast<float>(s0);
  if (e.mode == dfno::EPI_HEAD) {
    TORCH_CHECK(v0.has_value() && v1.has_value(), "EPI_HEAD needs the hidden bias and output weights");
    TORCH_CHECK(v0->scalar_type() == at::kFloat && v1->scalar_type() == at::kFloat && v0->is_contiguous() &&
                v1->is_contiguous() && v0->numel() >= N && v1->numel() >= N + 1 && N < 255, "bad head vectors");
    TORCH_CHECK(e.nrl >= 1 && e.nrl <= 4, "bad head row digits");
    e.v0 = v0->data_ptr<float>(); e.v1 = v1->data_ptr<float>();
  }
  if (e.mode == dfno::EPI_PAIR_SCATTER) {
    TORCH_CHECK(N % 2 == 0 && e.J[0] > 0 && e.nrl >= 1 && e.nrl <= 4, "bad scatter descriptor");
    for (int i = 0; i + 1 < e.nrl; ++i) TORCH_CHECK(e.R[i] > 0, "row radix must be positive");
    if (e.peer_sel != dfno::PEER_NONE) TORCH_CHECK(e.peer_div > 0, "peer_div must be positive");
  }
  dfno::BoxGeom box{};
  if (boxed) {
    box.mt = static_cast<int>(epi[20]); box.mtp = static_cast<int>(epi[21]); box.kzl = static_cast<int>(epi[22]);
    box.KZ = static_cast<int>(epi[23]); box.Yl = static_cast<int>(epi[24]); box.y0 = static_cast<int>(epi[25]);
    box.bcx = epi[26]; box.base_off = epi[27];
  }
  int ctas = sm_count();
  if (max_ctas > 0 && max_ctas < ctas) ctas = static_cast<int>(max_ctas);
  check(dfno::dft_gemm_launch(A.data_ptr(), lda, Bmat.data_ptr(), p, ctas, cur_stream(), boxed ? &box : nullptr),
        "dft_gemm");
}

}  // namespace

void register_ops(pybind11::module& m);    // ops_bindings.cpp
void register_symm(pybind11::module& m);   // symm_mem.cpp

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "dfno_b200 sm_90a kernels";
  m.def("dft_gemm", &dft_gemm, "resident-operator GEMM on wgmma (see dft_gemm_sm90.cu)",
        py::arg("A"), py::arg("M"), py::arg("K"), py::arg("lda"), py::arg("Bmat"), py::arg("N"),
        py::arg("epi"), py::arg("peer_ptrs"), py::arg("add_src") = c10::nullopt, py::arg("ld_add") = 0,
        py::arg("max_ctas") = 0, py::arg("v0") = c10::nullopt, py::arg("v1") = c10::nullopt, py::arg("s0") = 0.0, py::arg("a_f16") = false);
  register_ops(m);
  register_symm(m);
}
