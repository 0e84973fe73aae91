// Shared internals of libicaf_b200: error reporting, checked launches, device info.
#pragma once
#include <cstdio>
#include <cuda.h>          // CUtensorMap + enums only; the driver entry point is resolved at run time (no -lcuda)
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "../../include/icaf_b200.h"
#include "ptx.cuh"

namespace icaf {

int set_error(int code, const char* msg);
int set_cuda_error(cudaError_t e, const char* where);
const uint32_t* seed_offset_ptr();    // see icaf_set_seed_offset
int sm_count_cached();   // SM count the planners size for: the CURRENT device's (cached per ordinal), or the lower
                         // icaf_set_sm_count_target
int current_device();    // cudaGetDevice; -1 on error
bool pdl_enabled();        // programmatic dependent launch on every kernel (env ICAF_PDL, default on)

void count_launch();   // api.cu: process-wide tally behind icaf_kernel_launches()

// Launch with the programmatic-stream-serialization attribute when PDL is enabled (every kernel of this library
// executes griddepcontrol.wait before it touches memory another kernel may have produced).  Returns ICAF_OK, or the
// launch's own error under `where` (the prefix of icaf_last_error()); never synchronises.  Only launches the runtime
// accepted are counted.
template <typename... KArgs, typename... Args>
inline int launch_kc(const char* where, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                     unsigned cluster_x, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (pdl_enabled()) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  if (cluster_x > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster_x; attr[n].val.clusterDim.y = 1; attr[n].val.clusterDim.z = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();   // the refused launch also set the runtime's last error: clear it so no later check reports it again
    return set_cuda_error(e, where);
  }
  count_launch();
  return ICAF_OK;
}
template <typename... KArgs, typename... Args>
inline int launch_k(const char* where, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  return launch_kc(where, kernel, grid, block, smem, st, 1u, static_cast<Args&&>(args)...);
}

// Blocks of `block` threads that cover n items (a 1-D grid, or the x extent of one)
inline unsigned blocks_for(long long n, int block) { return unsigned((n + block - 1) / block); }

// Opt a kernel into > 48 KB of dynamic shared memory once per device (the attribute is per device and per function):
// `done` is the caller's static per-device flag array.
constexpr int kMaxDevices = 64;
template <typename K>
inline int configure_smem(K kernel, int bytes, bool (&done)[kMaxDevices], const char* where) {
  const int dev = current_device();
  if (dev < 0 || dev >= kMaxDevices) return set_error(ICAF_ERR_CUDA, "no current CUDA device (or ordinal >= 64)");
  if (done[dev]) return ICAF_OK;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) return set_cuda_error(e, where);
  done[dev] = true;      // idempotent attribute; a race between two threads only sets it twice
  return ICAF_OK;
}

// TMA descriptors (host side). fp16 tensors, 128-byte swizzle, zero fill out of bounds.
// 2D: [rows][inner] with a row pitch in bytes; box = box_rows x box_inner (box_inner = 64 / 32 / 16 halfs -> 128B / 64B / 32B swizzle).
int encode_tmap_2d(CUtensorMap* out, const void* base, uint64_t inner, uint64_t rows, uint64_t row_pitch_bytes,
                   uint32_t box_inner, uint32_t box_rows);
// 3D: dims (d0, d1, d2) with d1 / d2 pitches in bytes; box = (box0, box1, box2), box0 = 64 / 32 / 16 halfs as in 2D.  Boxes may
// overhang any dimension (the attention kernel reads a head of d columns as a padded box of up to 2d: the rest is zero-filled).
int encode_tmap_3d(CUtensorMap* out, const void* base, const uint64_t (&dims)[3], uint64_t pitch1_bytes, uint64_t pitch2_bytes,
                   const uint32_t (&box)[3]);
// 4D NHWC activation view (C, W, H, B) with pixel pitch `ld` elements; box = (box_c, box_w, box_h, 1) *input* elements,
// traversal strides (1, sw, sh, 1): loads ceil(box_w/sw) x ceil(box_h/sh) pixels per box.
int encode_tmap_nhwc(CUtensorMap* out, const void* base, int C, int W, int H, int B, int64_t ld, uint32_t box_c,
                     uint32_t box_w, uint32_t box_h, uint32_t sw, uint32_t sh);

}  // namespace icaf
