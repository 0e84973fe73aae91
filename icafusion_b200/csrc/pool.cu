// Pooling and resampling of fp16 NHWC maps, each forward next to its backward: SPPF's chained 5x5 max pools, nearest 2x
// up-sampling, and the channel-slice copy behind Concat; plus the L2 prefetch of the parameters.  Each thread moves 16-byte
// (8-channel) vectors, so every warp access is a run of full 128-byte lines along the channel axis.
#include "icaf_internal.cuh"

namespace icaf {

// SPPF: three chained 5x5/s1/p2 max pools == 5x5, 9x9, 13x13 windows clipped to the map (-inf padding)
__global__ void sppf_pool_kernel(const __half* __restrict__ x, long long x_ld, __half* y1, __half* y2, __half* y3,
                                 long long y_ld, int B, int H, int W, int C8) {
  pdl_launch_dependents();
  pdl_wait();
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  long long total = (long long)B * H * W * C8;
  if (i >= total) return;
  const auto [c, p, px, py, b] = nhwc8(i, H, W, C8);
  const __half ninf = __ushort_as_half(0xFC00);
  __half2 n2 = __halves2half2(ninf, ninf);
  uint4 m5, m9, m13;
  *reinterpret_cast<__half2*>(&m5.x) = n2; m5.y = m5.x; m5.z = m5.x; m5.w = m5.x;
  m9 = m5; m13 = m5;
  for (int dy = -6; dy <= 6; ++dy) {
    int yy = py + dy;
    if ((unsigned)yy >= (unsigned)H) continue;
    for (int dx = -6; dx <= 6; ++dx) {
      int xx = px + dx;
      if ((unsigned)xx >= (unsigned)W) continue;
      uint4 v = ldg16(x + ((long long)(b * H + yy) * W + xx) * x_ld + c * 8);
      m13 = hmax8(m13, v);
      if (dy >= -4 && dy <= 4 && dx >= -4 && dx <= 4) m9 = hmax8(m9, v);
      if (dy >= -2 && dy <= 2 && dx >= -2 && dx <= 2) m5 = hmax8(m5, v);
    }
  }
  long long o = p * y_ld + c * 8;
  *reinterpret_cast<uint4*>(y1 + o) = m5;
  *reinterpret_cast<uint4*>(y2 + o) = m9;
  *reinterpret_cast<uint4*>(y3 + o) = m13;
}

// Fast path for maps of <= 1024 pixels (the P5 map of any input up to 1024x1024): one block per (image, 8-channel
// chunk) keeps the whole map in shared memory and runs the three chained pools as separable 5-tap row / column passes.
__global__ void __launch_bounds__(1024) sppf_pool_smem_kernel(const __half* __restrict__ x, long long x_ld, __half* y1, __half* y2,
                                                              __half* y3, long long y_ld, int H, int W, int C8) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ uint4 sp[];                 // [2][H*W]
  const int HW = H * W;
  uint4* a = sp;
  uint4* t = sp + HW;
  const int b = blockIdx.x / C8, c = blockIdx.x % C8;
  const int p = threadIdx.x;
  const int py = p / W, px = p - py * W;
  const long long pix = (long long)b * HW + p;
  if (p < HW) a[p] = ldg16(x + pix * x_ld + c * 8);
  __syncthreads();
  __half* outs[3] = {y1, y2, y3};
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    if (p < HW) {                                // row pass: max over x-2..x+2 (clipped = -inf padding)
      uint4 m = a[p];
#pragma unroll
      for (int d = 1; d <= 2; ++d) {
        if (px - d >= 0) m = hmax8(m, a[p - d]);
        if (px + d < W) m = hmax8(m, a[p + d]);
      }
      t[p] = m;
    }
    __syncthreads();
    if (p < HW) {                                // column pass
      uint4 m = t[p];
#pragma unroll
      for (int d = 1; d <= 2; ++d) {
        if (py - d >= 0) m = hmax8(m, t[p - d * W]);
        if (py + d < H) m = hmax8(m, t[p + d * W]);
      }
      a[p] = m;                                  // input of the next chained pool (each thread rewrites only its own pixel)
      *reinterpret_cast<uint4*>(outs[k] + pix * y_ld + c * 8) = m;
    }
    __syncthreads();
  }
}

// MaxPool2d(5, 1, 2) backward (one stage of SPPF's chain): dx[q] = sum over the windows w containing q of dy[w] * [argmax_w == q],
// argmax = first maximum in row-major window order (torch's max_pool2d_with_indices).  Two gather kernels, deterministic:
//   1. per window (= per output pixel) and channel: the position code (ky*5 + kx) of its first maximum -> one byte;
//   2. per input pixel q: the <= 25 windows that contain q; those whose code points at q contribute their dy.
__global__ void __launch_bounds__(256) maxpool5_argmax_kernel(const __half* __restrict__ x, uint2* __restrict__ code, int B, int H, int W, int C8) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)B * H * W * C8) return;
  const auto [c, p, wx, wy, b] = nhwc8(i, H, W, C8);
  const __half* xb = x + (size_t(b) * H * W) * (C8 * 8) + c * 8;
  float best[8];
  uint32_t arg[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { best[e] = -INFINITY; arg[e] = 0u; }
  for (int ky = 0; ky < 5; ++ky) {
    const int yy = wy + ky - 2;
    if (yy < 0 || yy >= H) continue;
    for (int kx = 0; kx < 5; ++kx) {
      const int xx = wx + kx - 2;
      if (xx < 0 || xx >= W) continue;
      float v[8];
      unpack8(ldg16(xb + (size_t(yy) * W + xx) * (C8 * 8)), v);
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (v[e] > best[e]) { best[e] = v[e]; arg[e] = uint32_t(ky * 5 + kx); }
    }
  }
  code[i] = pack_argmax8(arg);
}
__global__ void __launch_bounds__(256) maxpool5_bwd_kernel(const uint2* __restrict__ code, const __half* __restrict__ dy, __half* __restrict__ dx, int B, int H, int W,
                                                           int C8) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)B * H * W * C8) return;
  const auto [c, p, qx, qy, b] = nhwc8(i, H, W, C8);
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = 0.f;
  for (int wy = max(qy - 2, 0); wy <= min(qy + 2, H - 1); ++wy)
    for (int wx = max(qx - 2, 0); wx <= min(qx + 2, W - 1); ++wx) {
      const size_t w = ((size_t(b) * H + wy) * W + wx) * C8 + c;
      const uint2 cd = __ldg(code + w);
      const uint32_t mine = uint32_t((qy - wy + 2) * 5 + (qx - wx + 2));      // q's position code inside window w
      float g[8];
      unpack8(ldg16(dy + w * 8), g);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        if (argmax_code(cd, e) == mine) acc[e] += g[e];
      }
    }
  reinterpret_cast<uint4*>(dx)[i] = pack8(acc);
}

// ------------------------------------------------------------------------------------------------
__global__ void upsample2x_kernel(const __half* __restrict__ x, long long x_ld, __half* __restrict__ y, long long y_ld,
                                  int B, int H, int W, int C8) {
  pdl_launch_dependents();
  pdl_wait();
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  long long total = (long long)B * (2 * H) * (2 * W) * C8;
  if (i >= total) return;
  const auto [c, p, ox, oy, b] = nhwc8(i, 2 * H, 2 * W, C8);
  uint4 v = ldg16(x + ((long long)(b * H + (oy >> 1)) * W + (ox >> 1)) * x_ld + c * 8);
  *reinterpret_cast<uint4*>(y + p * y_ld + c * 8) = v;
}

// nearest 2x up-sampling backward: dx[b, y, x] = sum of the 2x2 block of dy
__global__ void upsample2x_bwd_kernel(const __half* __restrict__ dy, __half* __restrict__ dx, int B, int H, int W, int C8) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)B * H * W * C8) return;
  const auto [c, p, x, y, b] = nhwc8(i, H, W, C8);
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int dyy = 0; dyy < 2; ++dyy)
    for (int dxx = 0; dxx < 2; ++dxx) {
      float v[8];
      unpack8(ldg16(dy + ((size_t(b) * 2 * H + 2 * y + dyy) * (2 * W) + 2 * x + dxx) * (C8 * 8) + c * 8), v);
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] += v[e];
    }
  reinterpret_cast<uint4*>(dx)[i] = pack8(acc);
}

// ------------------------------------------------------------------------------------------------
__global__ void copy_channels_kernel(const __half* __restrict__ x, long long x_ld, __half* __restrict__ y,
                                     long long y_ld, long long pixels, int C8) {
  pdl_launch_dependents();
  pdl_wait();
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= pixels * C8) return;
  int c = int(i % C8);
  long long p = i / C8;
  *reinterpret_cast<uint4*>(y + p * y_ld + c * 8) = ldg16(x + p * x_ld + c * 8);
}

__global__ void prefetch_l2_kernel(const char* __restrict__ p, size_t bytes) {
  pdl_launch_dependents();
  // The region holds parameters (no kernel writes it), so the prefetches need not wait for the previous kernel ...
  size_t i = (size_t(blockIdx.x) * blockDim.x + threadIdx.x) * 128;
  const size_t stride = size_t(gridDim.x) * blockDim.x * 128;
  for (; i < bytes; i += stride) prefetch_l2(p + i);
  // ... but this grid must not COMPLETE before its predecessor does: the next kernel's griddepcontrol.wait only covers
  // the grid launched right before it, so an early-finishing prefetch would let a consumer overtake its producer.
  pdl_wait();
}

}  // namespace icaf

using namespace icaf;

extern "C" int icaf_sppf_pool(const void* x, int64_t x_ld, void* y1, void* y2, void* y3, int64_t y_ld, int B, int H,
                              int W, int C, void* stream) {
  if (!x || !y1 || !y2 || !y3 || C % 8 || x_ld % 8 || y_ld % 8) return set_error(ICAF_ERR_BAD_ARG, "sppf_pool: bad argument");
  if (H * W <= 1024) {
    int threads = (H * W + 31) / 32 * 32;
    return launch_k("sppf_pool", sppf_pool_smem_kernel, dim3(B * (C / 8)), dim3(threads), (size_t)(2 * H * W * sizeof(uint4)), (cudaStream_t)stream,
                    (const __half*)x, x_ld, (__half*)y1, (__half*)y2, (__half*)y3, y_ld, H, W, C / 8);
  }
  long long total = (long long)B * H * W * (C / 8);
  return launch_k("sppf_pool", sppf_pool_kernel, dim3(blocks_for(total, 128)), dim3(128), 0, (cudaStream_t)stream, (const __half*)x, x_ld,
                  (__half*)y1, (__half*)y2, (__half*)y3, y_ld, B, H, W, C / 8);
}

extern "C" int icaf_maxpool5_bwd(const void* x, const void* dy, void* dx, int B, int H, int W, int C, void* workspace, size_t workspace_bytes, void* stream) {
  if (!x || !dy || !dx || !workspace || C % 8 || B < 1 || H < 1 || W < 1) return set_error(ICAF_ERR_BAD_ARG, "maxpool5_bwd: null pointer or C % 8");
  if (workspace_bytes < size_t(B) * H * W * C || (reinterpret_cast<uintptr_t>(workspace) & 7)) return set_error(ICAF_ERR_BAD_ARG, "maxpool5_bwd: workspace needs B*H*W*C bytes, 8-byte aligned");
  const long long n8 = (long long)B * H * W * (C / 8);
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = launch_k("maxpool5_bwd(argmax)", maxpool5_argmax_kernel, dim3(blocks_for(n8, 256)), dim3(256), 0, st, (const __half*)x,
                        (uint2*)workspace, B, H, W, C / 8)) return rc;
  return launch_k("maxpool5_bwd", maxpool5_bwd_kernel, dim3(blocks_for(n8, 256)), dim3(256), 0, st, (const uint2*)workspace, (const __half*)dy,
                  (__half*)dx, B, H, W, C / 8);
}

extern "C" int icaf_upsample2x(const void* x, int64_t x_ld, void* y, int64_t y_ld, int B, int H, int W, int C, void* stream) {
  if (!x || !y || C % 8 || x_ld % 8 || y_ld % 8) return set_error(ICAF_ERR_BAD_ARG, "upsample2x: bad argument");
  long long total = (long long)B * 4 * H * W * (C / 8);
  return launch_k("upsample2x", upsample2x_kernel, dim3(blocks_for(total, 256)), dim3(256), 0, (cudaStream_t)stream, (const __half*)x, x_ld,
                  (__half*)y, y_ld, B, H, W, C / 8);
}

extern "C" int icaf_upsample2x_bwd(const void* dy, void* dx, int B, int H, int W, int C, void* stream) {
  if (!dy || !dx || C % 8) return set_error(ICAF_ERR_BAD_ARG, "upsample2x_bwd: bad argument");
  return launch_k("upsample2x_bwd", upsample2x_bwd_kernel, dim3(blocks_for((long long)B * H * W * (C / 8), 256)), dim3(256), 0, (cudaStream_t)stream,
                  (const __half*)dy, (__half*)dx, B, H, W, C / 8);
}

extern "C" int icaf_copy_channels(const void* x, int64_t x_ld, void* y, int64_t y_ld, int64_t pixels, int C, void* stream) {
  if (!x || !y || C % 8 || x_ld % 8 || y_ld % 8) return set_error(ICAF_ERR_BAD_ARG, "copy_channels: bad argument");
  return launch_k("copy_channels", copy_channels_kernel, dim3(blocks_for(pixels * (C / 8), 256)), dim3(256), 0, (cudaStream_t)stream,
                  (const __half*)x, x_ld, (__half*)y, y_ld, pixels, C / 8);
}

extern "C" int icaf_prefetch_l2(const void* ptr, size_t bytes, void* stream) {
  if (!ptr || bytes == 0) return set_error(ICAF_ERR_BAD_ARG, "prefetch_l2: bad argument");
  unsigned blocks = blocks_for((bytes + 127) / 128, 256);
  if (blocks > 148u * 8u) blocks = 148u * 8u;
  return launch_k("prefetch_l2", prefetch_l2_kernel, dim3(blocks), dim3(256), 0, (cudaStream_t)stream, (const char*)ptr, bytes);
}
