// Backward of the two DMFF-specific data-movement kernels (aux.cu) and the fp32 -> fp16 filter packing of the training step.
//   dmff_pool_tokens_bwd : gradient of the avg/max adaptive pooling mix (common.py:817-823, AdaptivePool2d :868-891) w.r.t. the
//                          two feature maps; gather form (one thread per pixel x 8 channels, no atomics).
//   dmff_upsample_cat_bwd: gradient of the training-mode tail (nearest resample, common.py:829) w.r.t. the token streams;
//                          gather form over the pixels each token was copied to.  (The residual/concat part of the tail is a
//                          channel slice of the incoming gradient and needs no kernel.)
//   pack_weight          : fp32 master filter (Cout, Cin, kh, kw) -> the fp16 [rows][k_pad] bank of the implicit-GEMM kernel, either
//                          as it is (forward) or flipped and transposed (data-gradient convolution); pad rows/columns written as 0.
#include "icaf_internal.cuh"

namespace icaf {

struct PoolBwdParams {
  const __half* x[2]; const __half* dtok[2]; __half* dx[2];
  uint2* code[2];          // [B][N][C8]: per window and channel, the position code (ky*kw + kx) of its first maximum
  const float* mix;
  long long x_ld;
  int B, H, W, C8, nh, nw, n_pad, kh, kw, sh, sw;
};
// 1 of 2: arg-max position of every pooling window (windows are few: nh*nw per image)
__global__ void __launch_bounds__(128) dmff_pool_argmax_kernel(const PoolBwdParams P) {
  pdl_launch_dependents();
  pdl_wait();
  const int mod = blockIdx.y;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const int N = P.nh * P.nw;
  if (i >= (long long)P.B * N * P.C8) return;
  const int c = int(i % P.C8);
  const long long t = i / P.C8;
  const int n = int(t % N), b = int(t / N);
  const int ty = n / P.nw, tx = n % P.nw;
  const __half* x0 = (mod ? P.x[1] : P.x[0]) + ((long long)(b * P.H + ty * P.sh) * P.W + tx * P.sw) * P.x_ld + c * 8;
  float best[8];
  uint32_t arg[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { best[e] = -INFINITY; arg[e] = 0u; }
  for (int k = 0; k < P.kh * P.kw; ++k) {
    const int ky = k / P.kw, kx = k - ky * P.kw;
    float f[8];
    unpack8(ldg16(x0 + ((long long)ky * P.W + kx) * P.x_ld), f);
#pragma unroll
    for (int e = 0; e < 8; ++e)
      if (f[e] > best[e]) { best[e] = f[e]; arg[e] = uint32_t(k); }       // strict: the first maximum in row-major order wins
  }
  (mod ? P.code[1] : P.code[0])[i] = pack_argmax8(arg);
}
// 2 of 2: every pixel gathers from the windows that contain it
__global__ void __launch_bounds__(128) dmff_pool_tokens_bwd_kernel(const PoolBwdParams P) {
  pdl_launch_dependents();
  pdl_wait();
  const int mod = blockIdx.y;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long total = (long long)P.B * P.H * P.W * P.C8;
  if (i >= total) return;
  const int c = int(i % P.C8);
  long long p = i / P.C8;
  const int w = int(p % P.W);
  long long t = p / P.W;
  const int h = int(t % P.H), b = int(t / P.H);
  const int C = P.C8 * 8, N = P.nh * P.nw;
  const __half* dtok = (mod ? P.dtok[1] : P.dtok[0]) + (long long)b * P.n_pad * C + c * 8;
  const uint2* code = (mod ? P.code[1] : P.code[0]) + (long long)b * N * P.C8 + c;
  const float w1 = P.mix[mod * 2] / float(P.kh * P.kw), w2 = P.mix[mod * 2 + 1];
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = 0.f;
  // windows [ty*sh, ty*sh + kh) that contain row h (likewise columns); kh >= sh, so there is at least one
  const int ty1 = min(h / P.sh, P.nh - 1), tx1 = min(w / P.sw, P.nw - 1);
  const int ty0 = max((h - P.kh + P.sh) / P.sh, 0), tx0 = max((w - P.kw + P.sw) / P.sw, 0);
  for (int ty = ty0; ty <= ty1; ++ty) {
    if (h < ty * P.sh || h >= ty * P.sh + P.kh) continue;
    for (int tx = tx0; tx <= tx1; ++tx) {
      if (w < tx * P.sw || w >= tx * P.sw + P.kw) continue;
      const int n = ty * P.nw + tx;
      float g[8];
      unpack8(ldg16(dtok + (long long)n * C), g);
      const uint2 cd = __ldg(code + (long long)n * P.C8);
      const uint32_t mine = uint32_t((h - ty * P.sh) * P.kw + (w - tx * P.sw));
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        acc[e] += g[e] * (w1 + (argmax_code(cd, e) == mine ? w2 : 0.f));
      }
    }
  }
  *reinterpret_cast<uint4*>((mod ? P.dx[1] : P.dx[0]) + p * C + c * 8) = pack8(acc);
}

struct UpCatBwdParams {
  const __half* dcat; __half* dtok[2];
  long long d_ld;
  int B, H, W, C8, nh, nw, n_pad;
  float sy, sx;
};
__global__ void __launch_bounds__(128) dmff_upsample_cat_bwd_kernel(const UpCatBwdParams P) {
  pdl_launch_dependents();
  pdl_wait();
  const int mod = blockIdx.y;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long total = (long long)P.B * P.n_pad * P.C8;
  if (i >= total) return;
  const int c = int(i % P.C8);
  const long long t = i / P.C8;
  const int n = int(t % P.n_pad), b = int(t / P.n_pad);
  const int C = P.C8 * 8;
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = 0.f;
  if (n < P.nh * P.nw) {
    const int iy = n / P.nw, ix = n % P.nw;
    const __half* d = P.dcat + mod * C + c * 8;
    // destination rows oy with min(floor(oy * sy), nh - 1) == iy -- the forward kernel's own expression decides membership
    const int oy0 = max(int(floorf(iy / P.sy)) - 1, 0), oy1 = min(int(ceilf((iy + 1) / P.sy)) + 1, P.H - 1);
    const int ox0 = max(int(floorf(ix / P.sx)) - 1, 0), ox1 = min(int(ceilf((ix + 1) / P.sx)) + 1, P.W - 1);
    const bool ident = P.nh == P.H && P.nw == P.W;
    for (int oy = oy0; oy <= oy1; ++oy) {
      if ((ident ? oy : min(int(floorf(oy * P.sy)), P.nh - 1)) != iy) continue;
      for (int ox = ox0; ox <= ox1; ++ox) {
        if ((ident ? ox : min(int(floorf(ox * P.sx)), P.nw - 1)) != ix) continue;
        float g[8];
        unpack8(ldg16(d + ((long long)(b * P.H + oy) * P.W + ox) * P.d_ld), g);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] += g[e];
      }
    }
  }
  *reinterpret_cast<uint4*>((mod ? P.dtok[1] : P.dtok[0]) + t * C + c * 8) = pack8(acc);
}

// Element i of a packed [rows][k_pad] filter bank (pad rows / columns are 0):
//   forward:         out[n][(ky*kw + kx)*chan_p + c]                  = w[n][c][ky][kx]      (rows >= Cout, k_pad >= kh*kw*chan_p)
//   flip_transpose:  out[c][((kh-1-ky)*kw + (kw-1-kx))*chan_p + n]    = w[n][c][ky][kx]      (rows >= Cin,  k_pad >= kh*kw*chan_p)
__device__ __forceinline__ __half packed_weight(const float* __restrict__ w, long long i, int k_pad, int chan_p, int Cout, int Cin, int kh,
                                                int kw, bool flip_transpose) {
  const int r = int(i / k_pad), k = int(i - (long long)r * k_pad);
  const int tap = k / chan_p, ch = k - tap * chan_p;
  float v = 0.f;
  if (tap < kh * kw) {
    const int ky = tap / kw, kx = tap - ky * kw;
    if (!flip_transpose) {
      if (r < Cout && ch < Cin) v = w[(((long long)r * Cin + ch) * kh + ky) * kw + kx];
    } else {
      if (r < Cin && ch < Cout) v = w[(((long long)ch * Cin + r) * kh + (kh - 1 - ky)) * kw + (kw - 1 - kx)];
    }
  }
  return __float2half(v);
}

// mode 0: the forward bank; mode 1: the flipped and transposed one
__global__ void __launch_bounds__(256) pack_weight_kernel(const float* __restrict__ w, __half* __restrict__ out, int Cout, int Cin, int kh, int kw,
                                                          int chan_p, int rows, int k_pad, int mode) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = blockIdx.x * 256ll + threadIdx.x;
  if (i >= (long long)rows * k_pad) return;
  out[i] = packed_weight(w, i, k_pad, chan_p, Cout, Cin, kh, kw, mode != 0);
}

// both banks of one filter in one launch (the training step packs every filter once per step, forward and data-gradient form)
__global__ void __launch_bounds__(256) pack_weight_pair_kernel(const float* __restrict__ w, __half* __restrict__ out_f, __half* __restrict__ out_d, int Cout, int Cin,
                                                               int kh, int kw, int rows_f, int kpad_f, int chan_d, int rows_d, int kpad_d) {
  pdl_launch_dependents();
  pdl_wait();
  long long i = blockIdx.x * 256ll + threadIdx.x;
  const long long nf = (long long)rows_f * kpad_f, nd = (long long)rows_d * kpad_d;
  if (i >= nf + nd) return;
  const bool dg = i >= nf;
  if (dg) i -= nf;
  (dg ? out_d : out_f)[i] = packed_weight(w, i, dg ? kpad_d : kpad_f, dg ? chan_d : Cin, Cout, Cin, kh, kw, dg);
}

}  // namespace icaf

using namespace icaf;

extern "C" int icaf_dmff_pool_tokens_bwd(const void* x_vis, const void* x_ir, int64_t x_ld, const void* dtok_vis, const void* dtok_ir, const float* mix,
                                         void* dx_vis, void* dx_ir, int B, int H, int W, int C, int nh, int nw, int n_pad, void* workspace,
                                         size_t workspace_bytes, void* stream) {
  if (!x_vis || !x_ir || !dtok_vis || !dtok_ir || !mix || !dx_vis || !dx_ir || !workspace) return set_error(ICAF_ERR_BAD_ARG, "dmff_pool_tokens_bwd: null pointer");
  if (workspace_bytes < 2 * size_t(B) * nh * nw * C || (reinterpret_cast<uintptr_t>(workspace) & 7))
    return set_error(ICAF_ERR_BAD_ARG, "dmff_pool_tokens_bwd: workspace needs 2*B*nh*nw*C bytes, 8-byte aligned");
  if (C % 8 || x_ld % 8 || B < 1 || nh < 1 || nw < 1 || H < nh || W < nw || n_pad < nh * nw)
    return set_error(ICAF_ERR_BAD_ARG, "dmff_pool_tokens_bwd: bad shape");
  PoolBwdParams P;
  P.x[0] = (const __half*)x_vis; P.x[1] = (const __half*)x_ir; P.dtok[0] = (const __half*)dtok_vis; P.dtok[1] = (const __half*)dtok_ir;
  P.dx[0] = (__half*)dx_vis; P.dx[1] = (__half*)dx_ir; P.mix = mix; P.x_ld = x_ld;
  P.B = B; P.H = H; P.W = W; P.C8 = C / 8; P.nh = nh; P.nw = nw; P.n_pad = n_pad;
  P.sh = H / nh; P.sw = W / nw;                                   // AdaptivePool2d geometry, models/common.py:878-882
  P.kh = H - (nh - 1) * P.sh; P.kw = W - (nw - 1) * P.sw;
  if (P.kh * P.kw > 255) return set_error(ICAF_ERR_UNSUPPORTED, "dmff_pool_tokens_bwd: pooling windows of more than 255 pixels");
  P.code[0] = (uint2*)workspace; P.code[1] = P.code[0] + size_t(B) * nh * nw * P.C8;
  const long long nwin = (long long)B * nh * nw * P.C8;
  if (int rc = launch_k("dmff_pool_tokens_bwd(argmax)", dmff_pool_argmax_kernel, dim3(blocks_for(nwin, 128), 2), dim3(128), 0, (cudaStream_t)stream, P)) return rc;
  const long long total = (long long)B * H * W * P.C8;
  return launch_k("dmff_pool_tokens_bwd", dmff_pool_tokens_bwd_kernel, dim3(blocks_for(total, 128), 2), dim3(128), 0, (cudaStream_t)stream, P);
}

extern "C" int icaf_dmff_upsample_cat_bwd(const void* dcat, int64_t d_ld, void* dtok_vis, void* dtok_ir, int B, int H, int W, int C, int nh, int nw,
                                          int n_pad, int mode, void* stream) {
  if (!dcat || !dtok_vis || !dtok_ir) return set_error(ICAF_ERR_BAD_ARG, "dmff_upsample_cat_bwd: null pointer");
  if (C % 8 || d_ld % 8 || d_ld < 2 * C || n_pad < nh * nw || B < 1) return set_error(ICAF_ERR_BAD_ARG, "dmff_upsample_cat_bwd: bad shape");
  if (mode != 1 && !(nh == H && nw == W))
    return set_error(ICAF_ERR_UNSUPPORTED, "dmff_upsample_cat_bwd: only the training-mode (nearest) tail has a backward (common.py:828-829)");
  UpCatBwdParams P;
  P.dcat = (const __half*)dcat; P.dtok[0] = (__half*)dtok_vis; P.dtok[1] = (__half*)dtok_ir; P.d_ld = d_ld;
  P.B = B; P.H = H; P.W = W; P.C8 = C / 8; P.nh = nh; P.nw = nw; P.n_pad = n_pad;
  P.sy = float(nh) / float(H); P.sx = float(nw) / float(W);
  const long long total = (long long)B * n_pad * P.C8;
  return launch_k("dmff_upsample_cat_bwd", dmff_upsample_cat_bwd_kernel, dim3(blocks_for(total, 128), 2), dim3(128), 0, (cudaStream_t)stream, P);
}

extern "C" int icaf_pack_weight(const float* w, int Cout, int Cin, int kh, int kw, int chan_pad, int rows, int k_pad, int transpose_flip, void* out,
                                void* stream) {
  if (!w || !out || Cout < 1 || Cin < 1 || kh < 1 || kw < 1) return set_error(ICAF_ERR_BAD_ARG, "pack_weight: bad argument");
  const int chan = transpose_flip ? Cout : Cin, need_rows = transpose_flip ? Cin : Cout;
  if (chan_pad < chan || rows < need_rows || k_pad < kh * kw * chan_pad) return set_error(ICAF_ERR_BAD_ARG, "pack_weight: padded sizes smaller than the filter");
  const long long total = (long long)rows * k_pad;
  return launch_k("pack_weight", pack_weight_kernel, dim3(blocks_for(total, 256)), dim3(256), 0, (cudaStream_t)stream, w, (__half*)out, Cout, Cin, kh,
                  kw, chan_pad, rows, k_pad, transpose_flip ? 1 : 0);
}

extern "C" int icaf_pack_weight_pair(const float* w, int Cout, int Cin, int kh, int kw, int rows_f, int kpad_f, void* out_fwd, int chan_pad_d, int rows_d,
                                     int kpad_d, void* out_dgrad, void* stream) {
  if (!w || !out_fwd || !out_dgrad || Cout < 1 || Cin < 1 || kh < 1 || kw < 1) return set_error(ICAF_ERR_BAD_ARG, "pack_weight_pair: bad argument");
  if (rows_f < Cout || kpad_f < kh * kw * Cin || chan_pad_d < Cout || rows_d < Cin || kpad_d < kh * kw * chan_pad_d)
    return set_error(ICAF_ERR_BAD_ARG, "pack_weight_pair: padded sizes smaller than the filter");
  const long long total = (long long)rows_f * kpad_f + (long long)rows_d * kpad_d;
  return launch_k("pack_weight_pair", pack_weight_pair_kernel, dim3(blocks_for(total, 256)), dim3(256), 0, (cudaStream_t)stream, w, (__half*)out_fwd,
                  (__half*)out_dgrad, Cout, Cin, kh, kw, rows_f, kpad_f, chan_pad_d, rows_d, kpad_d);
}
