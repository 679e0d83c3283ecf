// p2p.cu -- peer-memory (NVLink 5 / NVSwitch) synchronisation and small collectives.
//
// Symmetric buffers (symm_mem.cpp) give every rank a device pointer to every peer's buffer.
// The fused GEMM epilogues store tiles straight into those; what remains is ordering:
//
//   p2p_barrier        : flag exchange.  Rank r writes `epoch` into slot r of every peer's
//                        flag array (st.release.sys after a system fence, so all peer stores
//                        issued earlier on the stream are visible), then spins until all of
//                        its own slots reached `epoch` (ld.acquire.sys).  ~2 NVLink latencies,
//                        no host involvement, capturable in a CUDA graph.
//   p2p_alltoall       : push-model all-to-all-v (the Repartition data plane for tensors the
//                        fused GEMM epilogues do not cover): each rank stores its per-peer segments
//                        directly into the peers' receive buffers; followed by p2p_barrier.
//   p2p_allreduce_small: sum of a small fp32 vector across ranks by reading every peer's
//                        copy in rank order (bitwise identical result on all ranks).  This is
//                        the gradient reduction of the replicated pointwise weights -- the
//                        Broadcast/SumReduce pair of the reference's BroadcastedLinear
//                        (SURVEY.md K1, K18) collapses to one such call per optimizer step.
//   p2p_sum_f64        : the same for one fp64 scalar per rank (each rank's part of the squared
//                        gradient norm): a fixed rank order, so every rank gets the same bits.
#include "sm90_ptx.cuh"
#include "kernels.h"

namespace dfno {
namespace {

struct PeerFlags { uint32_t* p[8]; };
struct PeerBufs { const float* p[8]; };
struct PeerF64 { const double* p[8]; };

__device__ __forceinline__ unsigned long long global_timer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// Failure detection: a peer that died (or never reached the barrier) would hang every other
// GPU of the box forever -- the reference has exactly this failure mode with MPI (SURVEY.md
// 5.3).  The spin is bounded: after `timeout_ns` the slot that is late is recorded in
// my_flags[16 + r] and the kernel traps, so the hang surfaces as a CUDA error on this rank.
__global__ void p2p_barrier_kernel(PeerFlags peers, uint32_t* my_flags, int rank, int world, uint32_t epoch_arg,
                                   unsigned long long timeout_ns) {
  // The epoch lives in device memory (my_flags[32]) and is bumped by the kernel itself, so the
  // launch carries no step-dependent argument and can be replayed from a CUDA graph.  Every
  // rank executes the same barrier sequence, hence the counters agree.  epoch_arg != 0 overrides.
  __shared__ uint32_t s_epoch;
  if (threadIdx.x == 0) {
    const uint32_t e = epoch_arg ? epoch_arg : my_flags[32] + 1;
    my_flags[32] = e;
    s_epoch = e;
  }
  __syncthreads();
  const uint32_t epoch = s_epoch;
  const int r = threadIdx.x;
  if (r < world) {
    __threadfence_system();
    st_release_sys(peers.p[r] + rank, epoch);
    const unsigned long long t0 = global_timer_ns();
    // epochs only grow; signed difference tolerates wrap-around
    while (static_cast<int32_t>(ld_acquire_sys(my_flags + r) - epoch) < 0) {
      if (timeout_ns && global_timer_ns() - t0 > timeout_ns) {
        my_flags[16 + r] = epoch;                 // which peer / which epoch never arrived
        __threadfence_system();
        asm volatile("trap;");
      }
    }
  }
}

__global__ void __launch_bounds__(256)
p2p_allreduce_kernel(PeerBufs bufs, float* __restrict__ out, long long n, int world) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float acc = 0.f;
    for (int r = 0; r < world; ++r) acc += bufs.p[r][i];
    out[i] = acc;
  }
}

__global__ void p2p_sum_f64_kernel(PeerF64 bufs, double* __restrict__ out, int world) {
  if (threadIdx.x == 0) {
    double acc = 0.0;
    for (int r = 0; r < world; ++r) acc += bufs.p[r][0];
    *out = acc;
  }
}

// push-model all-to-all-v: block (peer, chunk) copies a slice of the segment destined for `peer`
// from the local send buffer into that peer's receive buffer with 16-byte vector stores.
struct A2AParams {
  const uint8_t* send;
  uint8_t* recv[8];              // peers' receive buffers (NVLink-mapped)
  long long send_off[9];         // byte offsets of the per-peer segments in `send`
  long long dst_off[8];          // byte offset inside peer p's receive buffer where *my* data goes
  int world;
};

__global__ void __launch_bounds__(512)
p2p_alltoall_kernel(A2AParams a) {
  const int peer = blockIdx.y;
  const long long n = a.send_off[peer + 1] - a.send_off[peer];
  const uint8_t* src = a.send + a.send_off[peer];
  uint8_t* dst = a.recv[peer] + a.dst_off[peer];
  const long long nvec = n / 16;
  const uint4* s4 = reinterpret_cast<const uint4*>(src);
  uint4* d4 = reinterpret_cast<uint4*>(dst);
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  // 4 independent 16-byte loads in flight per thread before the stores
  for (; i + 3 * stride < nvec; i += 4 * stride) {
    const uint4 v0 = s4[i], v1 = s4[i + stride], v2 = s4[i + 2 * stride], v3 = s4[i + 3 * stride];
    d4[i] = v0; d4[i + stride] = v1; d4[i + 2 * stride] = v2; d4[i + 3 * stride] = v3;
  }
  for (; i < nvec; i += stride) d4[i] = s4[i];
  if (blockIdx.x == 0)
    for (long long b = nvec * 16 + threadIdx.x; b < n; b += blockDim.x) dst[b] = src[b];
  __threadfence_system();
}

}  // namespace

const char* p2p_alltoall(const void* send, const long long* send_off, void* const* peer_recv, const long long* dst_off,
                         int world, int ctas_per_peer, cudaStream_t s) {
  if (world < 1 || world > 8) return "p2p_alltoall: world size must be 1..8";
  A2AParams a;
  a.send = static_cast<const uint8_t*>(send);
  a.world = world;
  for (int i = 0; i < 8; ++i) {
    a.recv[i] = static_cast<uint8_t*>(peer_recv[i < world ? i : 0]);
    a.dst_off[i] = i < world ? dst_off[i] : 0;
  }
  for (int i = 0; i <= 8; ++i) a.send_off[i] = send_off[i <= world ? i : world];
  for (int i = 0; i < world; ++i)
    if ((a.send_off[i] % 16) || (a.dst_off[i] % 16)) return "p2p_alltoall: segments must be 16-byte aligned";
  if (ctas_per_peer < 1) ctas_per_peer = 1;
  p2p_alltoall_kernel<<<dim3(ctas_per_peer, world), 512, 0, s>>>(a);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

const char* p2p_barrier(uint32_t* const* peer_flags, uint32_t* my_flags, int rank, int world, uint32_t epoch,
                        unsigned long long timeout_ns, cudaStream_t s) {
  if (world < 1 || world > 8) return "p2p_barrier: world size must be 1..8";
  PeerFlags pf;
  for (int i = 0; i < 8; ++i) pf.p[i] = peer_flags[i < world ? i : 0];
  p2p_barrier_kernel<<<1, 32, 0, s>>>(pf, my_flags, rank, world, epoch, timeout_ns);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

const char* p2p_allreduce_small(float* const* peer_bufs, float* out, long long n, int rank, int world,
                                cudaStream_t s) {
  if (world < 1 || world > 8) return "p2p_allreduce: world size must be 1..8";
  PeerBufs pb;
  for (int i = 0; i < 8; ++i) pb.p[i] = peer_bufs[i < world ? i : 0];
  long long blocks = (n + 255) / 256;
  if (blocks > 64) blocks = 64;
  if (blocks < 1) blocks = 1;
  p2p_allreduce_kernel<<<static_cast<int>(blocks), 256, 0, s>>>(pb, out, n, world);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

const char* p2p_sum_f64(double* const* peer_bufs, double* out, int world, cudaStream_t s) {
  if (world < 1 || world > 8) return "p2p_sum_f64: world size must be 1..8";
  PeerF64 pb;
  for (int i = 0; i < 8; ++i) pb.p[i] = peer_bufs[i < world ? i : 0];
  p2p_sum_f64_kernel<<<1, 32, 0, s>>>(pb, out, world);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

}  // namespace dfno
