// symm_mem.cpp -- symmetric (peer-mapped) device memory for the NVLink data plane.
//
// Every rank cudaMalloc's a buffer, exports a CUDA IPC handle, and maps the handles of all
// other ranks of the box (handles travel through the torch.distributed control plane).  The
// result is a table of device pointers -- one per rank -- that sm_90a kernels dereference
// directly: stores/loads to a peer pointer are routed over NVLink 5 / NVSwitch by the
// hardware.  This replaces the MPI communicator the reference reaches through DistDL
// (SURVEY.md §5.8) for everything on the hot path.
#include <torch/extension.h>
#include <c10/cuda/CUDAGuard.h>
#include <cuda_runtime.h>

#include <string>

namespace {

void cuda_check(cudaError_t e, const char* what) {
  TORCH_CHECK(e == cudaSuccess, what, ": ", cudaGetErrorString(e));
}

// returns (device pointer, 64-byte IPC handle)
std::pair<int64_t, py::bytes> symm_alloc(int64_t nbytes, int64_t device) {
  c10::cuda::CUDAGuard guard(static_cast<c10::DeviceIndex>(device));
  void* ptr = nullptr;
  cuda_check(cudaMalloc(&ptr, static_cast<size_t>(nbytes)), "cudaMalloc(symmetric buffer)");
  cuda_check(cudaMemset(ptr, 0, static_cast<size_t>(nbytes)), "cudaMemset(symmetric buffer)");
  cuda_check(cudaDeviceSynchronize(), "cudaDeviceSynchronize");
  cudaIpcMemHandle_t h;
  cuda_check(cudaIpcGetMemHandle(&h, ptr), "cudaIpcGetMemHandle");
  return {reinterpret_cast<int64_t>(ptr), py::bytes(reinterpret_cast<const char*>(&h), sizeof(h))};
}

int64_t symm_open(const std::string& handle, int64_t device) {
  TORCH_CHECK(handle.size() == sizeof(cudaIpcMemHandle_t), "bad IPC handle size");
  c10::cuda::CUDAGuard guard(static_cast<c10::DeviceIndex>(device));
  cudaIpcMemHandle_t h;
  memcpy(&h, handle.data(), sizeof(h));
  void* ptr = nullptr;
  cuda_check(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess), "cudaIpcOpenMemHandle");
  return reinterpret_cast<int64_t>(ptr);
}

void symm_close(int64_t ptr) { cudaIpcCloseMemHandle(reinterpret_cast<void*>(ptr)); }
void symm_free(int64_t ptr) { cudaFree(reinterpret_cast<void*>(ptr)); }

// non-owning tensor view of raw device memory (local part of a symmetric buffer)
at::Tensor tensor_from_ptr(int64_t ptr, std::vector<int64_t> shape, at::ScalarType dtype, int64_t device) {
  auto opts = at::TensorOptions().dtype(dtype).device(at::kCUDA, static_cast<c10::DeviceIndex>(device));
  return at::from_blob(reinterpret_cast<void*>(ptr), shape, [](void*) {}, opts);
}

}  // namespace

void register_symm(pybind11::module& m) {
  m.def("symm_alloc", &symm_alloc, "allocate a zeroed symmetric buffer; returns (ptr, ipc_handle)");
  m.def("symm_open", &symm_open, "map a peer's buffer from its IPC handle; returns the local pointer");
  m.def("symm_close", &symm_close);
  m.def("symm_free", &symm_free);
  m.def("tensor_from_ptr", &tensor_from_ptr);
}
