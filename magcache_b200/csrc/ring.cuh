// Shared-memory staging ring of the HBM-bound row kernels (LayerNorm + modulate, RMSNorm + RoPE, residual statistics): one
// producer thread keeps `stages` chunks of rows in flight with cp.async.bulk, independent of what the consumer warps are doing,
// and the consumer warps read each chunk out of shared memory. Chunk c of the kernel goes to the c-th stage the CTA walks; the
// CTAs stride over the chunks by the grid size.
#pragma once
#include "common.cuh"
#include "ptx.cuh"

namespace mc {

// Dynamic shared memory: `stages` data slots of `stage_bytes`, then a full and an empty mbarrier per stage.
struct StageRing {
  uint8_t* data;
  uint64_t* full;   // one arrival (the producer's expect_tx) + the bytes of the stage's copies
  uint64_t* empty;  // one arrival per consumer warp that reads the stage
  int stages, stage_bytes;

  // Called by every thread of the CTA.
  __device__ __forceinline__ StageRing(uint8_t* smem, int stages_, int stage_bytes_, int consumer_warps)
      : data(smem), stages(stages_), stage_bytes(stage_bytes_) {
    full = reinterpret_cast<uint64_t*>(smem + static_cast<size_t>(stages) * stage_bytes);
    empty = full + stages;
    if (threadIdx.x == 0) {
      for (int s = 0; s < stages; ++s) {
        ptx::mbar_init(&full[s], 1);
        ptx::mbar_init(&empty[s], consumer_warps);
      }
      ptx::fence_mbar_init();
    }
    __syncthreads();
  }
  // First byte past the barriers: room for the kernel's own shared memory.
  __device__ __forceinline__ uint8_t* end() const { return reinterpret_cast<uint8_t*>(empty + stages); }

  // Producer (one thread): for each of this CTA's chunks, wait until its stage is free, arm the full barrier for
  // `bytes(c)`, then let `copy(c, slot, bar)` issue the bulk copies of chunk c into `slot` on `bar`.
  template <typename Bytes, typename Copy>
  __device__ __forceinline__ void produce(int64_t n_chunks, Bytes bytes, Copy copy) const {
    uint32_t it = 0;
    for (int64_t c = blockIdx.x; c < n_chunks; c += gridDim.x, ++it) {
      const int s = it % stages;
      ptx::mbar_wait(&empty[s], ((it / stages) & 1) ^ 1);
      ptx::mbar_expect_tx(&full[s], bytes(c));
      copy(c, data + static_cast<size_t>(s) * stage_bytes, &full[s]);
    }
  }

  // Consumer warps, NG groups of them taking this CTA's chunks in turn (group `grp` takes the CTA's chunks grp, grp + NG, ...):
  // wait until the chunk has landed, then `body(c, slot, release)`; the body calls release() (whole warp) once it no longer
  // reads the slot, which hands the stage back to the producer.
  template <int NG, typename Body>
  __device__ __forceinline__ void consume(int64_t n_chunks, int grp, Body body) const {
    uint32_t it = grp;
    for (int64_t c = blockIdx.x + static_cast<int64_t>(grp) * gridDim.x; c < n_chunks; c += static_cast<int64_t>(NG) * gridDim.x, it += NG) {
      const int s = it % stages;
      ptx::mbar_wait(&full[s], (it / stages) & 1);
      body(c, static_cast<const uint8_t*>(data + static_cast<size_t>(s) * stage_bytes), [&] {
        __syncwarp();
        if ((threadIdx.x & 31) == 0) ptx::mbar_arrive(&empty[s]);
      });
    }
  }
};

// Host: the number of stages of `stage_bytes` that fit the 200 KB budget, at most `max_stages`; 0 when fewer than two fit
// (the staged form does not apply).
inline int ring_stages(int stage_bytes, int max_stages) {
  int stages = (200 * 1024) / stage_bytes;
  if (stages > max_stages) stages = max_stages;
  return stages >= 2 ? stages : 0;
}

// Host: launch a ring kernel over `n_chunks` chunks, one CTA per SM (fewer when there are fewer chunks). Its dynamic shared
// memory is the ring (`stages` x `stage_bytes` and the barriers) plus `extra_smem` bytes of the kernel's own, within the 8 KB
// the limit leaves above the 200 KB budget.
template <auto Kernel, typename... Args>
inline int32_t launch_ring(int stages, int stage_bytes, int extra_smem, int64_t n_chunks, int threads, cudaStream_t s, const char* what,
                           Args... args) {
  static PerDeviceOnce once;
  const int32_t rc = set_max_smem_once(Kernel, 208 * 1024, once, what);
  if (rc) return rc;
  const int smem = stages * stage_bytes + stages * 16 + extra_smem + 64;
  const int grid = static_cast<int>(n_chunks < num_sms() ? n_chunks : num_sms());
  Kernel<<<grid, threads, smem, s>>>(args...);
  MC_CHECK_LAUNCH(what);
  return MC_OK;
}

}  // namespace mc
