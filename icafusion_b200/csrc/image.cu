// Image staging of the inference path: planar input frames -> the fp16 NHWC image the stem convolution reads (plain or
// space-to-depth), and the letterbox resize of uint8 frames.
#include "staging.cuh"

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
// Letterbox (utils/datasets.py:1404-1427) + BGR->RGB + HWC->CHW (datasets.py:238) for a batch of frames: the frame, copied or
// through cv2.resize(INTER_LINEAR) (staging.cuh, host-built tables), at (top, left); the border is `pad`.
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
  int v[3] = {P.pad, P.pad, P.pad};                     // B, G, R of the source order
  if (yy >= 0 && yy < P.new_h && xx >= 0 && xx < P.new_w) {
    const unsigned char* S = P.src + (long long)b * P.H0 * P.W0 * 3;
    if (!P.xtab) copy_pixel(S, P.W0, xx, yy, v);
    else linear_pixel(S, P.W0, reinterpret_cast<const int4*>(P.xtab)[xx], reinterpret_cast<const int4*>(P.ytab)[yy], v);
  }
  store_planar_rgb(P.dst + (long long)b * 3 * hw + r, hw, v[0], v[1], v[2]);
}

// ------------------------------------------------------------------------------------------------
// Validation batch staging (utils/datasets.py:948-1024, augment=False, rect=True): one thread per 4 adjacent output pixels of
// one sample, both frames; each of the 6 output planes gets one 32-bit store.  A pixel inside the load_image rectangle is
// cv2.resize of the decoded frame -- copy, INTER_LINEAR (staging.cuh) or INTER_AREA (resizeAreaFast's block sums, or
// resizeArea_'s float taps with every product and sum rounded in cv2's order) -- and 114 outside it.
constexpr int kValThreads = 256;

struct ValStageParams {
  const icaf_val_sample* samples; const int* tab;
  unsigned char* out;
  int H, W;
};

__device__ __forceinline__ unsigned char sat_u8(float v) { return (unsigned char)min(255, max(0, __float2int_rn(v))); }

// Pixel (x, y) of the load_image-resized pair: v[0..2] = RGB frame B, G, R; v[3..5] = IR frame.
__device__ __forceinline__ void val_pixel(const icaf_val_sample& S, const int* __restrict__ tab, int x, int y, int (&v)[6]) {
  const unsigned char* fr[2] = {static_cast<const unsigned char*>(S.rgb), static_cast<const unsigned char*>(S.ir)};
  const long long row = (long long)S.W0 * 3;
  if (S.mode == ICAF_VAL_COPY) {
    copy_pixel(fr, S.W0, x, y, v);
  } else if (S.mode == ICAF_VAL_LINEAR) {
    linear_pixel(fr, S.W0, reinterpret_cast<const int4*>(tab + S.xtab)[x], reinterpret_cast<const int4*>(tab + S.ytab)[y], v);
  } else if (S.mode == ICAF_VAL_AREA_FAST) {
    int sum[6] = {0, 0, 0, 0, 0, 0};
    for (int dy = 0; dy < S.sy; ++dy)
      for (int dx = 0; dx < S.sx; ++dx) {
        const long long o = (long long)(y * S.sy + dy) * row + (x * S.sx + dx) * 3;
#pragma unroll
        for (int m = 0; m < 2; ++m) {
          sum[3 * m] += fr[m][o]; sum[3 * m + 1] += fr[m][o + 1]; sum[3 * m + 2] += fr[m][o + 2];
        }
      }
    if (S.sx == 2 && S.sy == 2) {
#pragma unroll
      for (int c = 0; c < 6; ++c) v[c] = (sum[c] + 2) >> 2;
    } else {
      const float scale = __fdiv_rn(1.0f, (float)(S.sx * S.sy));
#pragma unroll
      for (int c = 0; c < 6; ++c) v[c] = sat_u8(__fmul_rn((float)sum[c], scale));
    }
  } else {
    const int2 hx = reinterpret_cast<const int2*>(tab + S.xtab)[x], hy = reinterpret_cast<const int2*>(tab + S.ytab)[y];
    const int2* tx = reinterpret_cast<const int2*>(tab + S.xtab + hx.x);
    const int2* ty = reinterpret_cast<const int2*>(tab + S.ytab + hy.x);
    float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int j = 0; j < hy.y; ++j) {
      const int2 t = ty[j];
      const float beta = __int_as_float(t.y);
      float buf[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      for (int k = 0; k < hx.y; ++k) {
        const int2 s = tx[k];
        const float alpha = __int_as_float(s.y);
        const long long o = t.x * row + s.x * 3;
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
          for (int c = 0; c < 3; ++c) buf[3 * m + c] = __fadd_rn(buf[3 * m + c], __fmul_rn((float)fr[m][o + c], alpha));
      }
#pragma unroll
      for (int c = 0; c < 6; ++c) acc[c] = __fadd_rn(acc[c], __fmul_rn(beta, buf[c]));
    }
#pragma unroll
    for (int c = 0; c < 6; ++c) v[c] = sat_u8(acc[c]);
  }
}

__global__ void __launch_bounds__(kValThreads) val_stage_kernel(const ValStageParams P) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.y;
  const int W4 = P.W >> 2;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= P.H * W4) return;
  const int y = q / W4, x0 = (q - y * W4) * 4;
  const icaf_val_sample& S = P.samples[b];
  uint32_t word[6] = {0, 0, 0, 0, 0, 0};
  const int yy = y - S.top;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int xx = x0 + i - S.left;
    int v[6] = {kStagePad, kStagePad, kStagePad, kStagePad, kStagePad, kStagePad};
    if (yy >= 0 && yy < S.h && xx >= 0 && xx < S.w) val_pixel(S, P.tab, xx, yy, v);
#pragma unroll
    for (int m = 0; m < 2; ++m) {                           // planar RGB: channel 0 = R = source channel 2
      word[3 * m] |= uint32_t(v[3 * m + 2]) << (8 * i);
      word[3 * m + 1] |= uint32_t(v[3 * m + 1]) << (8 * i);
      word[3 * m + 2] |= uint32_t(v[3 * m]) << (8 * i);
    }
  }
  const long long plane = (long long)P.H * P.W;
  uint32_t* d = reinterpret_cast<uint32_t*>(P.out + (long long)b * 6 * plane + (long long)y * P.W + x0);
#pragma unroll
  for (int c = 0; c < 6; ++c) d[c * (plane >> 2)] = word[c];
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

extern "C" size_t icaf_val_stage_params_bytes(int B, int n_words) {
  if (B < 1 || B > 65535 || n_words < 0 || (n_words & 3)) return 0;
  return align16((size_t)B * sizeof(icaf_val_sample)) + (size_t)n_words * sizeof(int);
}

extern "C" int icaf_val_stage(const void* params, size_t params_bytes, int B, int H, int W, int n_words, void* out, void* stream) {
  if (!params || !out) return set_error(ICAF_ERR_BAD_ARG, "val_stage: null pointer");
  if (H < 1 || W < 4 || (W & 3) || (long long)H * W > (1ll << 30)) return set_error(ICAF_ERR_BAD_ARG, "val_stage: H x W must be positive with W % 4 == 0");
  const size_t need = icaf_val_stage_params_bytes(B, n_words);
  if (!need || params_bytes < need) return set_error(ICAF_ERR_BAD_ARG, "val_stage: bad batch or parameter block smaller than icaf_val_stage_params_bytes");
  if ((reinterpret_cast<uintptr_t>(params) & 15) || (reinterpret_cast<uintptr_t>(out) & 3))
    return set_error(ICAF_ERR_BAD_ARG, "val_stage: parameter block not 16-byte aligned or output not 4-byte aligned");
  ValStageParams P;
  P.samples = static_cast<const icaf_val_sample*>(params);
  P.tab = reinterpret_cast<const int*>(static_cast<const char*>(params) + align16((size_t)B * sizeof(icaf_val_sample)));
  P.out = static_cast<unsigned char*>(out);
  P.H = H; P.W = W;
  const dim3 grid(blocks_for((long long)H * (W / 4), kValThreads), (unsigned)B);
  return launch_k("val_stage", val_stage_kernel, grid, dim3(kValThreads), 0, (cudaStream_t)stream, P);
}
