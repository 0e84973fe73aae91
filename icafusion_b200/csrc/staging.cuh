// Image staging shared by the letterbox, validation and augmentation kernels: decoded uint8 BGR (H0, W0, 3) frames ->
// planar RGB.  cv2.resize(INTER_LINEAR) on uint8 is fixed-point -- horizontal taps {x0, x1, a0, a1}, vertical taps
// {y0, y1, b0, b1} (weights x 2048, datasets.resize_taps), dst = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2
// over the horizontal sums h0, h1 of the two source rows -- and is reproduced here bit for bit.
#pragma once
#include "icaf_internal.cuh"

namespace icaf {

constexpr int kStagePad = 114;   // the letterbox and mosaic border of the reference loader

// Parameter blocks are laid out in 16-byte aligned regions.
inline size_t align16(size_t n) { return (n + 15) & ~size_t(15); }

// Pixel (x, y) of a frame W0 pixels wide, unresized: v = B, G, R.
__device__ __forceinline__ void copy_pixel(const unsigned char* f, int W0, int x, int y, int* v) {
  const unsigned char* p = f + ((long long)y * W0 + x) * 3;
  v[0] = p[0]; v[1] = p[1]; v[2] = p[2];
}

// Pixel of the cv2.resize INTER_LINEAR result at column taps tx and row taps ty: v = B, G, R.
__device__ __forceinline__ void linear_pixel(const unsigned char* f, int W0, int4 tx, int4 ty, int* v) {
  const unsigned char* r0 = f + (long long)ty.x * W0 * 3;
  const unsigned char* r1 = f + (long long)ty.y * W0 * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int h0 = r0[tx.x * 3 + c] * tx.z + r0[tx.y * 3 + c] * tx.w;
    const int h1 = r1[tx.x * 3 + c] * tx.z + r1[tx.y * 3 + c] * tx.w;
    v[c] = (((ty.z * (h0 >> 4)) >> 16) + ((ty.w * (h1 >> 4)) >> 16) + 2) >> 2;
  }
}

// The same for an RGB/IR pair of one size: v[0..2] = RGB frame B, G, R; v[3..5] = IR frame.
__device__ __forceinline__ void copy_pixel(const unsigned char* const (&fr)[2], int W0, int x, int y, int (&v)[6]) {
  copy_pixel(fr[0], W0, x, y, v);
  copy_pixel(fr[1], W0, x, y, v + 3);
}
__device__ __forceinline__ void linear_pixel(const unsigned char* const (&fr)[2], int W0, int4 tx, int4 ty, int (&v)[6]) {
  linear_pixel(fr[0], W0, tx, ty, v);
  linear_pixel(fr[1], W0, tx, ty, v + 3);
}

// One B, G, R triple into planar RGB at d (planes `plane` bytes apart): channel 0 = R.
__device__ __forceinline__ void store_planar_rgb(unsigned char* d, long long plane, int b, int g, int r) {
  d[0] = (unsigned char)r; d[plane] = (unsigned char)g; d[2 * plane] = (unsigned char)b;
}

}  // namespace icaf
