// Peer-to-peer exchange of the token-sharded runs over NVLink 5 / NVSwitch, behind the C ABI (SURVEY §8b / §8e): the B200
// counterpart of the reference's sequence-parallel gather (`dist.all_gather` + `torch.cat`, videosys/core/comm.py:272-292, used
// by eval/magcache/experiments/opensora.py:284-293,356-361). No collective library on the data path:
//   * every rank owns one cudaMalloc'ed window that its peers map through CUDA IPC (mc_p2p_alloc / mc_p2p_open);
//   * the K|V rows a rank has just projected are pushed into every peer's gathered buffer by the COPY ENGINES (mc_p2p_push:
//     one cudaMemcpyAsync per peer on a side stream, followed by a 4-byte flag copy that publishes the segment) — no SM is
//     involved, so the pushes can never starve, or be starved by, the attention kernel that is consuming them;
//   * the attention kernel (mc_attn_fwd_ex) starts on the keys it already has and waits, tile by tile, on the flag of the
//     segment it needs next (ld.acquire.sys in the TMA-issuing warp): the transfer hides behind the math instead of a barrier;
//   * the head kernel stores its rows straight into every peer's output tensor (mc_head_unpatchify_ex, n_out = world), followed
//     by a flag per peer and a one-thread wait kernel (mc_p2p_wait).
//   * Open-Sora's sequence-parallel layout switch (frames <-> positions, videosys/core/comm.py:297-367 `all_to_all_with_pad`) and its
//     output assembly move strided blocks: mc_p2p_push2d issues one cudaMemcpy2DAsync per (sample, peer) block, then the flags.
// Flags carry a monotonically increasing epoch kept in device memory (mc_p2p_bump), so that a captured CUDA graph of a whole
// forward can be replayed: nothing epoch-dependent is baked into a launch.
#include "common.cuh"
#include "ptx.cuh"

namespace mc {

__global__ void p2p_bump_kernel(uint32_t* epoch, uint32_t* own_flag) {
  const uint32_t e = *epoch + 1;
  *epoch = e;
  if (own_flag != nullptr) *own_flag = e;
}

__global__ void p2p_wait_kernel(const uint32_t* flags, int n, const uint32_t* epoch) {
  const uint32_t want = *epoch;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const long long t0 = clock64();
    for (;;) {
      uint32_t v;
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flags + i) : "memory");
      if (static_cast<int32_t>(v - want) >= 0) break;
      __nanosleep(200);
      if (clock64() - t0 > MC_MBAR_TIMEOUT_CYCLES) {
        printf("mc_p2p_wait: peer %d never signalled (flag %u, epoch %u)\n", i, v, want);
        __trap();
      }
    }
  }
}

}  // namespace mc

extern "C" {

int32_t mc_p2p_alloc(int64_t bytes, void** ptr_out, void* handle_out) {
  MC_CHECK_ARG(bytes > 0 && ptr_out != nullptr && handle_out != nullptr, "mc_p2p_alloc: bad arguments");
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, static_cast<size_t>(bytes));
  if (e != cudaSuccess) return mc::cuda_fail(e, "mc_p2p_alloc: cudaMalloc");
  e = cudaMemset(p, 0, static_cast<size_t>(bytes));
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  cudaIpcMemHandle_t h;
  if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) {
    cudaFree(p);
    return mc::cuda_fail(e, "mc_p2p_alloc: cudaIpcGetMemHandle");
  }
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  memcpy(handle_out, &h, sizeof(h));
  *ptr_out = p;
  return MC_OK;
}

int32_t mc_p2p_open(const void* handle, void** ptr_out) {
  MC_CHECK_ARG(handle != nullptr && ptr_out != nullptr, "mc_p2p_open: bad arguments");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, sizeof(h));
  void* p = nullptr;
  cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) return mc::cuda_fail(e, "mc_p2p_open: cudaIpcOpenMemHandle (peer access between the GPUs of this node is required)");
  *ptr_out = p;
  return MC_OK;
}

int32_t mc_p2p_close(void* ptr) {
  if (ptr == nullptr) return MC_OK;
  cudaError_t e = cudaIpcCloseMemHandle(ptr);
  if (e != cudaSuccess) return mc::cuda_fail(e, "mc_p2p_close");
  return MC_OK;
}

int32_t mc_p2p_free(void* ptr) {
  if (ptr == nullptr) return MC_OK;
  cudaError_t e = cudaFree(ptr);
  if (e != cudaSuccess) return mc::cuda_fail(e, "mc_p2p_free");
  return MC_OK;
}

int32_t mc_p2p_bump(uint32_t* epoch, uint32_t* own_flag_or_null, void* stream) {
  MC_CHECK_ARG(epoch != nullptr, "mc_p2p_bump: null epoch");
  mc::p2p_bump_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(epoch, own_flag_or_null);
  MC_CHECK_LAUNCH("p2p_bump_kernel launch");
  return MC_OK;
}

int32_t mc_p2p_push(const void* src, void* const* dst_ptrs, void* const* flag_ptrs, int32_t n_dst, int64_t bytes, const uint32_t* epoch,
                    void* stream) {
  MC_CHECK_ARG(n_dst >= 0 && (n_dst == 0 || (dst_ptrs != nullptr && flag_ptrs != nullptr)) && epoch != nullptr && bytes >= 0,
               "mc_p2p_push: bad arguments");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  for (int i = 0; i < n_dst; ++i) {
    if (bytes > 0) {
      MC_CHECK_ARG(src != nullptr && dst_ptrs[i] != nullptr, "mc_p2p_push: null data pointer");
      cudaError_t e = cudaMemcpyAsync(dst_ptrs[i], src, static_cast<size_t>(bytes), cudaMemcpyDefault, s);
      if (e != cudaSuccess) return mc::cuda_fail(e, "mc_p2p_push: data copy");
    }
    // same stream, after the data: a peer that observes the flag also observes the segment
    cudaError_t e = cudaMemcpyAsync(flag_ptrs[i], epoch, sizeof(uint32_t), cudaMemcpyDefault, s);
    if (e != cudaSuccess) return mc::cuda_fail(e, "mc_p2p_push: flag copy");
  }
  return MC_OK;
}

int32_t mc_p2p_push2d(const mc_copy2d* copies, int32_t n_copies, void* const* flag_ptrs, int32_t n_flags, const uint32_t* epoch,
                      void* stream) {
  MC_CHECK_ARG(n_copies >= 0 && n_flags >= 0 && (n_copies == 0 || copies != nullptr) && (n_flags == 0 || (flag_ptrs != nullptr && epoch != nullptr)),
               "mc_p2p_push2d: bad arguments");
  // every argument is checked before the first copy is issued: a refused call moves nothing
  for (int i = 0; i < n_copies; ++i) {
    const mc_copy2d& c = copies[i];
    MC_CHECK_ARG(c.width >= 0 && c.height >= 0, "mc_p2p_push2d: copy %d has width %lld, height %lld", i, (long long)c.width, (long long)c.height);
    if (c.width == 0 || c.height == 0) continue;
    MC_CHECK_ARG(c.dst != nullptr && c.src != nullptr, "mc_p2p_push2d: copy %d has a null pointer", i);
    MC_CHECK_ARG(c.dpitch >= c.width && c.spitch >= c.width, "mc_p2p_push2d: copy %d has a pitch below its width (%lld, %lld < %lld)", i,
                 (long long)c.dpitch, (long long)c.spitch, (long long)c.width);
  }
  for (int i = 0; i < n_flags; ++i) MC_CHECK_ARG(flag_ptrs[i] != nullptr, "mc_p2p_push2d: flag %d is null", i);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  for (int i = 0; i < n_copies; ++i) {
    const mc_copy2d& c = copies[i];
    if (c.width == 0 || c.height == 0) continue;
    cudaError_t e = cudaMemcpy2DAsync(c.dst, static_cast<size_t>(c.dpitch), c.src, static_cast<size_t>(c.spitch), static_cast<size_t>(c.width),
                                      static_cast<size_t>(c.height), cudaMemcpyDefault, s);
    if (e != cudaSuccess) return mc::cuda_fail(e, "mc_p2p_push2d: data copy");
  }
  // same stream, after every block: a peer that observes its flag also observes the blocks
  for (int i = 0; i < n_flags; ++i) {
    cudaError_t e = cudaMemcpyAsync(flag_ptrs[i], epoch, sizeof(uint32_t), cudaMemcpyDefault, s);
    if (e != cudaSuccess) return mc::cuda_fail(e, "mc_p2p_push2d: flag copy");
  }
  return MC_OK;
}

int32_t mc_p2p_wait(const uint32_t* flags, int32_t n, const uint32_t* epoch, void* stream) {
  MC_CHECK_ARG(flags != nullptr && epoch != nullptr && n >= 1 && n <= 64, "mc_p2p_wait: bad arguments");
  mc::p2p_wait_kernel<<<1, 64, 0, static_cast<cudaStream_t>(stream)>>>(flags, n, epoch);
  MC_CHECK_LAUNCH("p2p_wait_kernel launch");
  return MC_OK;
}

}  // extern "C"
