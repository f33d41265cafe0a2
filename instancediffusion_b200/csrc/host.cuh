// Host-side helpers shared by the launchers: error reporting and TMA tensor-map encoding.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#ifndef IDIFF_STORAGE_BF16
#define IDIFF_STORAGE_BF16 0  // see common.cuh: 16-bit storage type of this build
#endif

namespace idiff {

int set_error(const char* fmt, ...);  // always returns -1

#define IDIFF_CHECK_CUDA(expr)                                                              \
  do {                                                                                      \
    cudaError_t _e = (expr);                                                                \
    if (_e != cudaSuccess)                                                                  \
      return idiff::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),       \
                              __FILE__, __LINE__);                                          \
  } while (0)

#define IDIFF_REQUIRE(cond, ...)                       \
  do {                                                 \
    if (!(cond)) return idiff::set_error(__VA_ARGS__); \
  } while (0)

// Encode a tiled fp16 tensor map with 128B swizzle and zero OOB fill.
// dims/strides innermost-first; strides[i] (bytes) is the stride of dim i+1 (rank-1 entries).
int encode_tmap_f16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                    const uint64_t* strides_bytes, const uint32_t* box);
// same with an explicit swizzle span (128 / 64 / 32 bytes, 0 = none)
int encode_tmap_f16_sw(CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                       const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes);

// Launch with programmatic stream serialization ("programmatic dependent launch"): the kernel may
// become resident while its predecessor in the stream is still running; every kernel of this library
// calls pdl_wait() (common.cuh) before it touches global memory, so only launch latency and prologues
// (barrier init, descriptor prefetch) overlap.  About 500 dependent launches make one
// UNet forward.  Opt-in with IDIFF_PDL=1: measured neutral inside the CUDA graph (the big kernels fill
// the register file, so a successor cannot become resident before they exit); plain stream order is
// the default.
bool pdl_enabled();
// multiprocessor count of the current device (queried once; grid sizes of the bandwidth-bound kernels)
int num_sms();
// idiff_set_batch_invariant: reduction geometry must not depend on the batch, M or num_sms()
bool batch_invariant();
// Pixel chunks per image of a batch-invariant GroupNorm / ScaleU reduction over hw x channels: about 8K elements
// (16 KB of 16-bit storage) per CTA, 1..max_chunks -- from the per-image shape alone.  At the UNet's 64x64 levels
// this is the cap, as the batch-dependent rule gives up to batch 8; at 8x8 x 1280 it is 10 chunks instead of 1-pixel
// ones; a VAE plane gets the cap.
inline int invariant_chunks(int hw, int channels, int max_chunks) {
  const long c = ((long)hw * channels + 8191) / 8192;
  return c < 1 ? 1 : c > max_chunks ? max_chunks : (int)c;
}
template <typename... KArgs, typename... Args>
cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                       Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// same, launched as thread-block clusters of `cluster_x` CTAs along x (1 = no cluster attribute)
template <typename... KArgs, typename... Args>
cudaError_t launch_pdl_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                               int cluster_x, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (cluster_x > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster_x;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  if (pdl_enabled()) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace idiff
