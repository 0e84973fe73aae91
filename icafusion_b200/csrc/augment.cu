// Training augmentation of RGB/IR pairs (utils/datasets.py:948-1024 with augment=True), one launch per batch, one thread per
// output pixel of both modalities.  Every step restates cv2's own arithmetic so the result is bit-exact:
//   warpAffine (imgwarp.cpp, INTER_LINEAR, BORDER_CONSTANT 114): X = (X0[y] + adelta[x]) >> 5, source X >> 5, fraction X & 31,
//     weights (32-ay)(32-ax)*32 ... (sum 2^15), dst = (sum S*w + 2^14) >> 15, taps off the canvas read 114;
//   mosaic canvas: up to four tile rectangles over a 114 background (load_mosaic_RGB_IR :1233-1253);
//   tile pixel: cv2.resize INTER_LINEAR of the decoded frame (the icaf_letterbox taps), identity when r = 1;
//   augment_hsv: BGR->HSV with cv2's integer tables (hsv_shift 12), the three LUTs, HSV->BGR in float32 as cv2's
//     vectorised path computes it (the two inner products fused, result x 255 truncated);
//   flipud / fliplr (output index only), BGR->RGB, HWC->CHW.
#include "staging.cuh"

namespace icaf {

constexpr int kAugThreads = 256;

struct AugmentParams {
  const icaf_aug_sample* samples; const int* warp; const int4* taps;
  unsigned char* rgb_out; unsigned char* ir_out;
  int s;
};

// Pixel (tx, ty) of the load_image-resized frame, both modalities: v[0..2] = RGB frame B, G, R; v[3..5] = IR frame.
__device__ __forceinline__ void tile_pixel(const icaf_aug_tile& T, const int4* __restrict__ taps, int tx, int ty, int (&v)[6]) {
  const unsigned char* fr[2] = {static_cast<const unsigned char*>(T.rgb), static_cast<const unsigned char*>(T.ir)};
  if (T.h == T.H0 && T.w == T.W0) {
    copy_pixel(fr, T.W0, tx, ty, v);
    return;
  }
  linear_pixel(fr, T.W0, taps[T.xtab + tx], taps[T.ytab + ty], v);
}

// Canvas pixel (cx, cy): the last tile placed over it, or the 114 background (also outside the canvas).
__device__ __forceinline__ void canvas_pixel(const icaf_aug_sample& S, const int4* __restrict__ taps, int cx, int cy, int (&v)[6]) {
  if (cx >= 0 && cy >= 0 && cx < S.canvas && cy < S.canvas) {
    for (int t = S.ntiles - 1; t >= 0; --t) {
      const icaf_aug_tile& T = S.tile[t];
      if (cx >= T.x1a && cx < T.x2a && cy >= T.y1a && cy < T.y2a) {
        tile_pixel(T, taps, cx - T.x1a + T.x1b, cy - T.y1a + T.y1b, v);
        return;
      }
    }
  }
#pragma unroll
  for (int c = 0; c < 6; ++c) v[c] = kStagePad;
}

// cv2 COLOR_BGR2HSV (uint8, hrange 180) -> LUT -> COLOR_HSV2BGR, in place on (b, g, r).
__device__ __forceinline__ void hsv_jitter(int& b, int& g, int& r, const unsigned char* __restrict__ lut, const int* sdiv,
                                           const int* hdiv) {
  const int v = max(b, max(g, r)), vmin = min(b, min(g, r));
  const int diff = v - vmin;
  const int vr = v == r ? -1 : 0, vg = v == g ? -1 : 0;
  const int s = (diff * sdiv[v] + (1 << 11)) >> 12;
  int h = (vr & (g - b)) + (~vr & ((vg & (b - r + 2 * diff)) + ((~vg) & (r - g + 4 * diff))));
  h = (h * hdiv[diff] + (1 << 11)) >> 12;
  h += h < 0 ? 180 : 0;
  const int H = lut[h], Sv = lut[256 + s], V = lut[512 + v];
  // HSV2RGB: hue sector and fraction from h * (6/180); every rounding spelled out (no contraction beyond cv2's own two FMAs).
  const float hs = __fmul_rn((float)H, 6.0f / 180.0f);
  const float sf = __fmul_rn((float)Sv, 1.0f / 255.0f), vf = __fmul_rn((float)V, 1.0f / 255.0f);
  const float sector_f = truncf(hs);
  const float fr = __fsub_rn(hs, sector_f);
  int sector = (int)sector_f;
  if ((unsigned)sector >= 6u) sector = 0;
  float tab[4];
  tab[0] = vf;
  tab[1] = __fmul_rn(vf, __fsub_rn(1.0f, sf));
  tab[2] = __fmul_rn(vf, __fmaf_rn(-sf, fr, 1.0f));
  tab[3] = __fmul_rn(vf, __fmaf_rn(-sf, __fsub_rn(1.0f, fr), 1.0f));
  int ib, ig, ir;                                           // sector -> the (b, g, r) entries of tab
  switch (sector) {
    case 0: ib = 1; ig = 3; ir = 0; break;
    case 1: ib = 1; ig = 0; ir = 2; break;
    case 2: ib = 3; ig = 0; ir = 1; break;
    case 3: ib = 0; ig = 2; ir = 1; break;
    case 4: ib = 0; ig = 1; ir = 3; break;
    default: ib = 2; ig = 1; ir = 0; break;
  }
  b = min(255, (int)__fmul_rn(tab[ib], 255.0f));
  g = min(255, (int)__fmul_rn(tab[ig], 255.0f));
  r = min(255, (int)__fmul_rn(tab[ir], 255.0f));
}

__global__ void __launch_bounds__(kAugThreads) augment_kernel(const AugmentParams P) {
  __shared__ int sdiv[256], hdiv[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {      // cv2's tables: cvRound((255 << 12) / i), cvRound((180 << 12) / (6 i))
    sdiv[i] = i ? __double2int_rn((double)(255 << 12) / (double)i) : 0;
    hdiv[i] = i ? __double2int_rn((double)(180 << 12) / (6.0 * i)) : 0;
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();
  const int s = P.s;
  const int b = blockIdx.y;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= s * s) return;
  const int y = p / s, x = p - y * s;
  const icaf_aug_sample& S = P.samples[b];
  const int yy = S.flipud ? s - 1 - y : y, xx = S.fliplr ? s - 1 - x : x;   // the flips only move the output index
  int v[6];
  if (S.warp) {
    const int* wt = P.warp + (long long)b * 4 * s;
    const int X = (wt[2 * s + yy] + wt[xx]) >> 5, Y = (wt[3 * s + yy] + wt[s + xx]) >> 5;
    const int sx = max(-32768, min(32767, X >> 5)), sy = max(-32768, min(32767, Y >> 5));   // saturate_cast<short>
    const int ax = X & 31, ay = Y & 31;
    const int w00 = (32 - ay) * (32 - ax) * 32, w01 = (32 - ay) * ax * 32, w10 = ay * (32 - ax) * 32, w11 = ay * ax * 32;
    int t00[6], t01[6], t10[6], t11[6];
    canvas_pixel(S, P.taps, sx, sy, t00);
    canvas_pixel(S, P.taps, sx + 1, sy, t01);
    canvas_pixel(S, P.taps, sx, sy + 1, t10);
    canvas_pixel(S, P.taps, sx + 1, sy + 1, t11);
#pragma unroll
    for (int c = 0; c < 6; ++c) v[c] = (t00[c] * w00 + t01[c] * w01 + t10[c] * w10 + t11[c] * w11 + (1 << 14)) >> 15;
  } else {
    canvas_pixel(S, P.taps, xx, yy, v);
  }
  const long long plane = (long long)s * s;
  unsigned char* outs[2] = {P.rgb_out, P.ir_out};
#pragma unroll
  for (int m = 0; m < 2; ++m) {
    int bb = v[3 * m], gg = v[3 * m + 1], rr = v[3 * m + 2];
    hsv_jitter(bb, gg, rr, &S.lut[m][0][0], sdiv, hdiv);
    store_planar_rgb(outs[m] + (long long)b * 3 * plane + p, plane, bb, gg, rr);
  }
}

}  // namespace icaf

using namespace icaf;

extern "C" size_t icaf_augment_params_bytes(int B, int s, int n_taps) {
  if (B < 1 || B > 65535 || s < 1 || s > 8192 || n_taps < 0) return 0;
  return align16((size_t)B * sizeof(icaf_aug_sample)) + (size_t)B * 4 * s * sizeof(int) + (size_t)n_taps * 4 * sizeof(int);
}

extern "C" int icaf_augment(const void* params, size_t params_bytes, int B, int s, int n_taps, void* rgb_out, void* ir_out, void* stream) {
  if (!params || !rgb_out || !ir_out) return set_error(ICAF_ERR_BAD_ARG, "augment: null pointer");
  const size_t need = icaf_augment_params_bytes(B, s, n_taps);
  if (!need || params_bytes < need) return set_error(ICAF_ERR_BAD_ARG, "augment: bad shape or parameter block smaller than icaf_augment_params_bytes");
  if (reinterpret_cast<uintptr_t>(params) & 15) return set_error(ICAF_ERR_BAD_ARG, "augment: parameter block not 16-byte aligned");
  AugmentParams P;
  const char* base = static_cast<const char*>(params);
  const size_t off_warp = align16((size_t)B * sizeof(icaf_aug_sample));
  P.samples = reinterpret_cast<const icaf_aug_sample*>(base);
  P.warp = reinterpret_cast<const int*>(base + off_warp);
  P.taps = reinterpret_cast<const int4*>(base + off_warp + (size_t)B * 4 * s * sizeof(int));
  P.rgb_out = static_cast<unsigned char*>(rgb_out); P.ir_out = static_cast<unsigned char*>(ir_out);
  P.s = s;
  const dim3 grid(blocks_for((long long)s * s, kAugThreads), (unsigned)B);
  return launch_k("augment", augment_kernel, grid, dim3(kAugThreads), 0, (cudaStream_t)stream, P);
}
