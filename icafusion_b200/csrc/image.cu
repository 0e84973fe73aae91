// Image staging of the inference path: planar input frames -> the fp16 NHWC image the stem convolution reads (plain or
// space-to-depth), and the letterbox resize of uint8 frames.
#include "icaf_internal.cuh"

namespace icaf {

// (B,3,H,W) planar -> (B,H,W,4) fp16
template <typename T>
__global__ void pack_image_kernel(const T* __restrict__ src, float scale, long long npix, long long hw, __half* __restrict__ dst) {
  pdl_launch_dependents();
  pdl_wait();
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= npix) return;
  long long b = i / hw, p = i - b * hw;
  const T* s = src + b * 3 * hw + p;
  float r = float(s[0]) * scale, g = float(s[hw]) * scale, bl = float(s[2 * hw]) * scale;
  uint2 o;
  o.x = pack_half2(r, g);
  o.y = pack_half2(bl, 0.f);
  reinterpret_cast<uint2*>(dst)[i] = o;
}

// (B,3,H,W) planar -> (B,H/2,W/2,16) fp16 space-to-depth: one thread per output pixel (2x2 input pixels x 4 channels)
template <typename T>
__global__ void pack_image_s2d_kernel(const T* __restrict__ src, float scale, int B, int H, int W, __half* __restrict__ dst) {
  pdl_launch_dependents();
  pdl_wait();
  const int W2 = W >> 1, H2 = H >> 1;
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)B * H2 * W2) return;
  const int x = int(i % W2);
  long long t = i / W2;
  const int y = int(t % H2), b = int(t / H2);
  const long long hw = (long long)H * W;
  const T* s = src + (long long)b * 3 * hw + (long long)(2 * y) * W + 2 * x;
  uint32_t o[8];
#pragma unroll
  for (int d = 0; d < 4; ++d) {                      // d = dy*2 + dx
    const T* p = s + (d >> 1) * W + (d & 1);
    o[2 * d] = pack_half2(float(p[0]) * scale, float(p[hw]) * scale);
    o[2 * d + 1] = pack_half2(float(p[2 * hw]) * scale, 0.f);
  }
  uint4* out = reinterpret_cast<uint4*>(dst + i * 16);
  out[0] = make_uint4(o[0], o[1], o[2], o[3]);
  out[1] = make_uint4(o[4], o[5], o[6], o[7]);
}

// ------------------------------------------------------------------------------------------------
// Letterbox (utils/datasets.py:1404-1427) + BGR->RGB + HWC->CHW (datasets.py:238) for a batch of frames:
// cv2.resize(INTER_LINEAR) on uint8 is fixed-point -- horizontal taps a0, a1 (x 2048, from the host-built tables), vertical
// dst = (((b0 * (r0 >> 4)) >> 16) + ((b1 * (r1 >> 4)) >> 16) + 2) >> 2 -- reproduced bit for bit; the border is `pad`.
struct LetterboxParams {
  const unsigned char* src; unsigned char* dst;
  const int* xtab; const int* ytab;     // [new_w][4] = {x0, x1, a0, a1}, [new_h][4] = {y0, y1, b0, b1}; NULL = no resize
  int B, H0, W0, H, W, top, left, new_h, new_w, pad;
};
__global__ void letterbox_kernel(const LetterboxParams P) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long hw = (long long)P.H * P.W;
  if (i >= (long long)P.B * hw) return;
  const int b = int(i / hw);
  const long long r = i - b * hw;
  const int y = int(r / P.W), x = int(r - (long long)y * P.W);
  const int yy = y - P.top, xx = x - P.left;
  int v0 = P.pad, v1 = P.pad, v2 = P.pad;               // B, G, R of the source order
  if (yy >= 0 && yy < P.new_h && xx >= 0 && xx < P.new_w) {
    const unsigned char* S = P.src + (long long)b * P.H0 * P.W0 * 3;
    if (!P.xtab) {
      const unsigned char* s = S + ((long long)yy * P.W0 + xx) * 3;
      v0 = s[0]; v1 = s[1]; v2 = s[2];
    } else {
      const int4 tx = reinterpret_cast<const int4*>(P.xtab)[xx], ty = reinterpret_cast<const int4*>(P.ytab)[yy];
      const unsigned char* r0 = S + (long long)ty.x * P.W0 * 3;
      const unsigned char* r1 = S + (long long)ty.y * P.W0 * 3;
      int out[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const int h0 = r0[tx.x * 3 + c] * tx.z + r0[tx.y * 3 + c] * tx.w;
        const int h1 = r1[tx.x * 3 + c] * tx.z + r1[tx.y * 3 + c] * tx.w;
        out[c] = (((ty.z * (h0 >> 4)) >> 16) + ((ty.w * (h1 >> 4)) >> 16) + 2) >> 2;
      }
      v0 = out[0]; v1 = out[1]; v2 = out[2];
    }
  }
  unsigned char* d = P.dst + (long long)b * 3 * hw + r;  // planar RGB: channel 0 = R = source channel 2
  d[0] = (unsigned char)v2; d[hw] = (unsigned char)v1; d[2 * hw] = (unsigned char)v0;
}

}  // namespace icaf

using namespace icaf;

extern "C" int icaf_pack_image(const void* src, int src_dtype, float scale, int B, int H, int W, void* dst, void* stream) {
  if (!src || !dst || B < 1 || H < 1 || W < 1) return set_error(ICAF_ERR_BAD_ARG, "pack_image: bad argument");
  long long hw = (long long)H * W, npix = hw * B;
  cudaStream_t st = (cudaStream_t)stream;
  unsigned g = blocks_for(npix, 256);
  if (src_dtype == 0) return launch_k("pack_image", pack_image_kernel<__half>, dim3(g), dim3(256), 0, st, (const __half*)src, scale, npix, hw,
                                      (__half*)dst);
  if (src_dtype == 1) return launch_k("pack_image", pack_image_kernel<float>, dim3(g), dim3(256), 0, st, (const float*)src, scale, npix, hw,
                                      (__half*)dst);
  if (src_dtype == 2) return launch_k("pack_image", pack_image_kernel<uint8_t>, dim3(g), dim3(256), 0, st, (const uint8_t*)src, scale, npix, hw,
                                      (__half*)dst);
  return set_error(ICAF_ERR_BAD_ARG, "pack_image: src_dtype must be 0 (fp16), 1 (fp32) or 2 (uint8)");
}

extern "C" int icaf_pack_image_s2d(const void* src, int src_dtype, float scale, int B, int H, int W, void* dst, void* stream) {
  if (!src || !dst || B < 1 || H < 2 || W < 2 || (H & 1) || (W & 1)) return set_error(ICAF_ERR_BAD_ARG, "pack_image_s2d: H and W must be even");
  cudaStream_t st = (cudaStream_t)stream;
  unsigned g = blocks_for((long long)B * (H / 2) * (W / 2), 256);
  if (src_dtype == 0) return launch_k("pack_image_s2d", pack_image_s2d_kernel<__half>, dim3(g), dim3(256), 0, st, (const __half*)src, scale, B, H, W,
                                      (__half*)dst);
  if (src_dtype == 1) return launch_k("pack_image_s2d", pack_image_s2d_kernel<float>, dim3(g), dim3(256), 0, st, (const float*)src, scale, B, H, W,
                                      (__half*)dst);
  if (src_dtype == 2) return launch_k("pack_image_s2d", pack_image_s2d_kernel<uint8_t>, dim3(g), dim3(256), 0, st, (const uint8_t*)src, scale, B, H,
                                      W, (__half*)dst);
  return set_error(ICAF_ERR_BAD_ARG, "pack_image_s2d: src_dtype must be 0 (fp16), 1 (fp32) or 2 (uint8)");
}

extern "C" int icaf_letterbox(const void* src, int B, int H0, int W0, void* dst, int H, int W, int top, int left, int new_h, int new_w,
                              const int* xtab, const int* ytab, int pad_value, void* stream) {
  if (!src || !dst || B < 1 || H0 < 1 || W0 < 1 || H < 1 || W < 1 || new_h < 1 || new_w < 1 || top < 0 || left < 0 || top + new_h > H ||
      left + new_w > W || pad_value < 0 || pad_value > 255)
    return set_error(ICAF_ERR_BAD_ARG, "letterbox: bad shape");
  const bool resize = new_h != H0 || new_w != W0;
  if (resize && (!xtab || !ytab || (reinterpret_cast<uintptr_t>(xtab) & 15) || (reinterpret_cast<uintptr_t>(ytab) & 15)))
    return set_error(ICAF_ERR_BAD_ARG, "letterbox: resizing needs the 16-byte aligned tap tables");
  LetterboxParams P;
  P.src = (const unsigned char*)src; P.dst = (unsigned char*)dst; P.xtab = resize ? xtab : nullptr; P.ytab = resize ? ytab : nullptr;
  P.B = B; P.H0 = H0; P.W0 = W0; P.H = H; P.W = W; P.top = top; P.left = left; P.new_h = new_h; P.new_w = new_w; P.pad = pad_value;
  return launch_k("letterbox", letterbox_kernel, dim3(blocks_for((long long)B * H * W, 256)), dim3(256), 0, (cudaStream_t)stream, P);
}
