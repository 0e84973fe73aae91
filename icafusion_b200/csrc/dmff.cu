// The DMFF block's (TransformerFusionBlock, common.py:762-865) kernels that are not GEMMs, each forward next to its backward
// (gather forms, no atomics): token pooling, the tail, LayerNorm (its backward is in train.cu, next to the reductions it
// launches), row statistics and axpby.  fp16 NHWC / token views; each thread moves 16-byte (8-channel) vectors.
#include "icaf_internal.cuh"

namespace icaf {

// Token pooling: token n = (ty, tx) of an nh x nw grid pools the kh x kw window at (ty*sh, tx*sw) of its stream's map.
// The forward and the backward take the same parameters; the buffers each of them reads or writes share slots.
// The *_f32 members are the same slots for an fp32 token stream (TransformerFusionBlock.stream_dtype = float32).
struct PoolTokParams {
  const __half* x[2];
  union {                  // forward: position embeddings; backward: token gradients
    const __half* pos[2]; const __half* dtok[2]; const float* pos_f32[2]; const float* dtok_f32[2];
  };
  union { __half* tok[2]; __half* dx[2]; float* tok_f32[2]; };   // forward: tokens (B,Npad,C); backward: map gradients
  union {
    float2* stats[2];      // forward, optional: (sum, sum of squares) of every token row per 32 channels, [B*Npad][C/32]
    uint2* code[2];        // backward: [B][N][C8] per window and channel, the position code (ky*kw + kx) of its first maximum
  };
  const float* mix;
  long long x_ld;
  int B, H, W, C8, nh, nw, n_pad, kh, kw, sh, sw;
};
// AdaptivePool2d geometry, models/common.py:878-882 (identity when the map is not larger than the grid)
static PoolTokParams pool_tok_params(const void* x_vis, const void* x_ir, int64_t x_ld, const float* mix, int B, int H, int W, int C, int nh,
                                     int nw, int n_pad) {
  PoolTokParams P;
  P.x[0] = (const __half*)x_vis; P.x[1] = (const __half*)x_ir; P.mix = mix; P.x_ld = x_ld;
  P.B = B; P.H = H; P.W = W; P.C8 = C / 8; P.nh = nh; P.nw = nw; P.n_pad = n_pad;
  P.sh = H / nh; P.sw = W / nw;
  P.kh = H - (nh - 1) * P.sh; P.kw = W - (nw - 1) * P.sw;
  return P;
}
// channel chunk c of the first pixel of token n's window in image b of map x
__device__ __forceinline__ const __half* pool_window(const PoolTokParams& P, const __half* x, int b, int n, int c) {
  const int ty = n / P.nw, tx = n % P.nw;
  return x + ((long long)(b * P.H + ty * P.sh) * P.W + tx * P.sw) * P.x_ld + c * 8;
}
// element k (row-major) of the window that starts at x0
__device__ __forceinline__ const __half* pool_tap(const PoolTokParams& P, const __half* x0, int k) {
  const int ky = k / P.kw, kx = k - ky * P.kw;
  return x0 + ((long long)ky * P.W + kx) * P.x_ld;
}
// sum and maximum over the window that starts at x0, 8 channels; window elements are fetched 8 at a time (independent 16-byte
// loads in flight) before they are reduced
__device__ __forceinline__ void pool_window_sum_max(const PoolTokParams& P, const __half* x0, float (&sum)[8], float (&mx)[8]) {
#pragma unroll
  for (int e = 0; e < 8; ++e) { sum[e] = 0.f; mx[e] = -INFINITY; }
  const int wn = P.kh * P.kw;
  for (int w0 = 0; w0 < wn; w0 += 8) {
    uint4 v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (w0 + j < wn) v[j] = ldg16(pool_tap(P, x0, w0 + j));
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (w0 + j < wn) {
        float f[8];
        unpack8(v[j], f);
#pragma unroll
        for (int e = 0; e < 8; ++e) { sum[e] += f[e]; mx[e] = fmaxf(mx[e], f[e]); }
      }
    }
  }
}
// the backward's token gradients of stream `mod`, in the stream's precision
template <typename T> __device__ __forceinline__ const T* pool_dtok(const PoolTokParams& P, int mod);
template <> __device__ __forceinline__ const __half* pool_dtok<__half>(const PoolTokParams& P, int mod) { return mod ? P.dtok[1] : P.dtok[0]; }
template <> __device__ __forceinline__ const float* pool_dtok<float>(const PoolTokParams& P, int mod) { return mod ? P.dtok_f32[1] : P.dtok_f32[0]; }

__global__ void dmff_pool_tokens_kernel(const PoolTokParams P) {
  pdl_launch_dependents();
  pdl_wait();
  const int mod = blockIdx.y;
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  long long total = (long long)P.B * P.n_pad * P.C8;
  const bool live = i < total;            // no early exit: groups of four lanes reduce the row statistics together
  if (!live) i = total - 1;
  int c = int(i % P.C8);
  long long t = i / P.C8;
  int n = int(t % P.n_pad);
  int b = int(t / P.n_pad);
  __half* out = (mod ? P.tok[1] : P.tok[0]) + t * (P.C8 * 8) + c * 8;
  const int N = P.nh * P.nw;
  uint4 packed = make_uint4(0, 0, 0, 0);  // pad rows (n >= N) are zero
  if (n < N) {
    float sum[8], mx[8];
    pool_window_sum_max(P, pool_window(P, mod ? P.x[1] : P.x[0], b, n, c), sum, mx);
    const float w1 = P.mix[mod * 2], w2 = P.mix[mod * 2 + 1];
    const float inv = 1.f / float(P.kh * P.kw);
    float pe[8], o[8];
    unpack8(ldg16((mod ? P.pos[1] : P.pos[0]) + (long long)n * (P.C8 * 8) + c * 8), pe);
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = w1 * (sum[e] * inv) + w2 * mx[e] + pe[e];
    packed = pack8(o);
  }
  if (live) *reinterpret_cast<uint4*>(out) = packed;
  float2* st = mod ? P.stats[1] : P.stats[0];
  if (st) {                               // statistics of the fp16-rounded token row, one partial per 32 channels (4 lanes)
    float f[8], su = 0.f, sq = 0.f;
    unpack8(packed, f);
#pragma unroll
    for (int e = 0; e < 8; ++e) { su += f[e]; sq += f[e] * f[e]; }
    su += __shfl_xor_sync(0xffffffffu, su, 1); sq += __shfl_xor_sync(0xffffffffu, sq, 1);
    su += __shfl_xor_sync(0xffffffffu, su, 2); sq += __shfl_xor_sync(0xffffffffu, sq, 2);
    if (live && (c & 3) == 0) st[t * (P.C8 >> 2) + (c >> 2)] = make_float2(su, sq);
  }
}

// fp32 token stream: common.py:817-823 as the reference evaluates it under autocast.  torch's fp16 pooling returns fp16 (the
// average is rounded), LearnableWeights multiplies by its fp32 weights (two rounded products, a rounded sum) and the fp32
// pos_emb is added (rounded): __fmul_rn / __fadd_rn keep the compiler from contracting any of it into an FMA.
__global__ void __launch_bounds__(128) dmff_pool_tokens_f32_kernel(const PoolTokParams P) {
  pdl_launch_dependents();
  pdl_wait();
  const int mod = blockIdx.y;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)P.B * P.n_pad * P.C8) return;
  const int c = int(i % P.C8);
  const long long t = i / P.C8;
  const int n = int(t % P.n_pad), b = int(t / P.n_pad);
  float o[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) o[e] = 0.f;             // pad rows (n >= N) are zero
  if (n < P.nh * P.nw) {
    float sum[8], mx[8], pe[8];
    pool_window_sum_max(P, pool_window(P, mod ? P.x[1] : P.x[0], b, n, c), sum, mx);
    const float w1 = P.mix[mod * 2], w2 = P.mix[mod * 2 + 1];
    const float k = float(P.kh * P.kw);
    ld8f((mod ? P.pos_f32[1] : P.pos_f32[0]) + (long long)n * (P.C8 * 8) + c * 8, pe);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float avg = __half2float(__float2half_rn(__fdiv_rn(sum[e], k)));      // avg_pool2d: sum / window size
      o[e] = __fadd_rn(__fadd_rn(__fmul_rn(avg, w1), __fmul_rn(mx[e], w2)), pe[e]);
    }
  }
  st8((mod ? P.tok_f32[1] : P.tok_f32[0]) + t * (P.C8 * 8) + c * 8, o);
}

// backward 1 of 2: arg-max position of every pooling window (windows are few: nh*nw per image)
__global__ void __launch_bounds__(128) dmff_pool_argmax_kernel(const PoolTokParams P) {
  pdl_launch_dependents();
  pdl_wait();
  const int mod = blockIdx.y;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const int N = P.nh * P.nw;
  if (i >= (long long)P.B * N * P.C8) return;
  const int c = int(i % P.C8);
  const long long t = i / P.C8;
  const int n = int(t % N), b = int(t / N);
  const __half* x0 = pool_window(P, mod ? P.x[1] : P.x[0], b, n, c);
  float best[8];
  uint32_t arg[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { best[e] = -INFINITY; arg[e] = 0u; }
  for (int k = 0; k < P.kh * P.kw; ++k) {
    float f[8];
    unpack8(ldg16(pool_tap(P, x0, k)), f);
#pragma unroll
    for (int e = 0; e < 8; ++e)
      if (f[e] > best[e]) { best[e] = f[e]; arg[e] = uint32_t(k); }       // strict: the first maximum in row-major order wins
  }
  (mod ? P.code[1] : P.code[0])[i] = pack_argmax8(arg);
}
// backward 2 of 2: every pixel gathers from the windows that contain it (token gradients T: fp16, or fp32 for an fp32 stream)
template <typename T>
__global__ void __launch_bounds__(128) dmff_pool_tokens_bwd_kernel(const PoolTokParams P) {
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
  const T* dtok = pool_dtok<T>(P, mod) + (long long)b * P.n_pad * C + c * 8;
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
      ld8(dtok + (long long)n * C, g);
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

// ------------------------------------------------------------------------------------------------
// DMFF tail: tokens -> (nh,nw) map -> interpolate to (H,W) + stream features -> concat buffer (B,H,W,2C).  The backward
// (training mode: nearest, common.py:829) gathers over the pixels each token was copied to; the residual / concat part of
// the tail is a channel slice of the incoming gradient and needs no kernel.
// Nearest resampling (F.interpolate mode='nearest'): destination index o of an axis of n sources, scale s = n / out
__device__ __forceinline__ int nearest_src(int o, float s, int n) { return min(int(floorf(o * s)), n - 1); }

// An fp32 token stream (tok_f32) is added to the fp16 map in fp32 and the sum rounded once to the fp16 concat, which is where
// the reference's autocast rounds it (the cast at conv1x1_out).
struct UpCatParams {
  union { const __half* tok[2]; const float* tok_f32[2]; };
  const __half* x[2]; __half* y;
  long long x_ld, y_ld;
  int B, H, W, C8, nh, nw, n_pad, mode;
  float sy, sx;   // nh/H, nw/W
};
template <typename T> __device__ __forceinline__ const T* upcat_tok(const UpCatParams& P, int mod);
template <> __device__ __forceinline__ const __half* upcat_tok<__half>(const UpCatParams& P, int mod) { return mod ? P.tok[1] : P.tok[0]; }
template <> __device__ __forceinline__ const float* upcat_tok<float>(const UpCatParams& P, int mod) { return mod ? P.tok_f32[1] : P.tok_f32[0]; }

template <typename T>
__global__ void dmff_upsample_cat_kernel(const UpCatParams P) {
  pdl_launch_dependents();
  pdl_wait();
  const int mod = blockIdx.y;
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  long long total = (long long)P.B * P.H * P.W * P.C8;
  if (i >= total) return;
  const auto [c, p, ox, oy, b] = nhwc8(i, P.H, P.W, P.C8);
  const int C = P.C8 * 8;
  const T* tok = upcat_tok<T>(P, mod) + (long long)b * P.n_pad * C + c * 8;
  float r[8];
  if (P.nh == P.H && P.nw == P.W) {                    // identity resample (un-pooled DMFF)
    ld8(tok + (long long)(oy * P.nw + ox) * C, r);
  } else if (P.mode == 1) {                            // nearest
    int iy = nearest_src(oy, P.sy, P.nh), ix = nearest_src(ox, P.sx, P.nw);
    ld8(tok + (long long)(iy * P.nw + ix) * C, r);
  } else {                                             // bilinear, align_corners=False
    float fy = fmaxf((oy + 0.5f) * P.sy - 0.5f, 0.f), fx = fmaxf((ox + 0.5f) * P.sx - 0.5f, 0.f);
    int y0 = int(fy), x0 = int(fx);
    int y1 = min(y0 + 1, P.nh - 1), x1 = min(x0 + 1, P.nw - 1);
    float ly = fy - y0, lx = fx - x0;
    float a[8], bq[8], cq[8], d[8];
    ld8(tok + (long long)(y0 * P.nw + x0) * C, a);
    ld8(tok + (long long)(y0 * P.nw + x1) * C, bq);
    ld8(tok + (long long)(y1 * P.nw + x0) * C, cq);
    ld8(tok + (long long)(y1 * P.nw + x1) * C, d);
#pragma unroll
    for (int e = 0; e < 8; ++e)
      r[e] = (1.f - ly) * ((1.f - lx) * a[e] + lx * bq[e]) + ly * ((1.f - lx) * cq[e] + lx * d[e]);
  }
  float f[8];
  unpack8(ldg16((mod ? P.x[1] : P.x[0]) + p * P.x_ld + c * 8), f);
#pragma unroll
  for (int e = 0; e < 8; ++e) r[e] += f[e];
  *reinterpret_cast<uint4*>(P.y + p * P.y_ld + mod * C + c * 8) = pack8(r);
}

struct UpCatBwdParams {
  const __half* dcat;
  union { __half* dtok[2]; float* dtok_f32[2]; };     // token gradients: fp16, or fp32 for an fp32 stream
  long long d_ld;
  int B, H, W, C8, nh, nw, n_pad;
  float sy, sx;
};
template <typename T> __device__ __forceinline__ T* upcat_dtok(const UpCatBwdParams& P, int mod);
template <> __device__ __forceinline__ __half* upcat_dtok<__half>(const UpCatBwdParams& P, int mod) { return mod ? P.dtok[1] : P.dtok[0]; }
template <> __device__ __forceinline__ float* upcat_dtok<float>(const UpCatBwdParams& P, int mod) { return mod ? P.dtok_f32[1] : P.dtok_f32[0]; }
template <typename T>
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
    // destination rows oy whose nearest source is iy: a superset from the inverse scale, then the forward's own index decides
    const int oy0 = max(int(floorf(iy / P.sy)) - 1, 0), oy1 = min(int(ceilf((iy + 1) / P.sy)) + 1, P.H - 1);
    const int ox0 = max(int(floorf(ix / P.sx)) - 1, 0), ox1 = min(int(ceilf((ix + 1) / P.sx)) + 1, P.W - 1);
    const bool ident = P.nh == P.H && P.nw == P.W;
    for (int oy = oy0; oy <= oy1; ++oy) {
      if ((ident ? oy : nearest_src(oy, P.sy, P.nh)) != iy) continue;
      for (int ox = ox0; ox <= ox1; ++ox) {
        if ((ident ? ox : nearest_src(ox, P.sx, P.nw)) != ix) continue;
        float g[8];
        unpack8(ldg16(d + ((long long)(b * P.H + oy) * P.W + ox) * P.d_ld), g);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] += g[e];
      }
    }
  }
  st8(upcat_dtok<T>(P, mod) + t * C + c * 8, acc);
}

// ------------------------------------------------------------------------------------------------
// LayerNorm: one warp per row, row cached in registers (C <= 2048).  The output is fp16 for either input: for an fp32 token
// stream it is the reference's fp32 LayerNorm under autocast followed by the fp16 cast at the Linear that consumes it.
struct LnParams {
  union { const __half* x[2]; const float* x_f32[2]; };
  __half* y[2]; const float* g[2]; const float* b[2];
  long long rows; int C; float eps;
};
template <typename T> __device__ __forceinline__ const T* ln_x(const LnParams& P, int prob);
template <> __device__ __forceinline__ const __half* ln_x<__half>(const LnParams& P, int prob) { return prob ? P.x[1] : P.x[0]; }
template <> __device__ __forceinline__ const float* ln_x<float>(const LnParams& P, int prob) { return prob ? P.x_f32[1] : P.x_f32[0]; }
template <typename T>
__global__ void layernorm_kernel(const LnParams P) {
  pdl_launch_dependents();
  pdl_wait();
  const int prob = blockIdx.y;
  const long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= P.rows) return;
  const int lane = threadIdx.x & 31;
  __half* y = (prob ? P.y[1] : P.y[0]) + row * P.C;
  const float* g = prob ? P.g[1] : P.g[0];
  const float* be = prob ? P.b[1] : P.b[0];
  const int nch = P.C >> 3;                 // 16-byte chunks in the row
  float v[8][8], mean, rstd;
  ln_row_moments(ln_x<T>(P, prob), row, P.C, P.eps, v, mean, rstd);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    int ch = lane + 32 * j;
    if (ch < nch) {
      float o[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = (v[j][e] - mean) * rstd * __ldg(g + ch * 8 + e) + __ldg(be + ch * 8 + e);
      *reinterpret_cast<uint4*>(y + ch * 8) = pack8(o);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// (sum, sum of squares) per row of a (rows, C) fp16 matrix: one warp per row, 16-byte loads.
__global__ void row_stats_kernel(const __half* __restrict__ x0, const __half* __restrict__ x1, float2* __restrict__ s0,
                                 float2* __restrict__ s1, long long rows, int C) {
  pdl_launch_dependents();
  pdl_wait();
  const long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const __half* x = (blockIdx.y ? x1 : x0) + row * C;
  float su = 0.f, sq = 0.f;
  for (int ch = lane; ch < (C >> 3); ch += 32) {
    float v[8];
    unpack8(ldg16(x + ch * 8), v);
#pragma unroll
    for (int e = 0; e < 8; ++e) { su += v[e]; sq += v[e] * v[e]; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    su += __shfl_xor_sync(0xffffffffu, su, o);
    sq += __shfl_xor_sync(0xffffffffu, sq, o);
  }
  if (lane == 0) (blockIdx.y ? s1 : s0)[row] = make_float2(su, sq);
}

// ------------------------------------------------------------------------------------------------
// out = a * x (+ b * y): LearnableCoefficient / LearnableWeights called stand-alone (common.py:569-587)
__global__ void axpby_kernel(const __half* __restrict__ x, const __half* __restrict__ y, const float* __restrict__ a,
                             const float* __restrict__ b, __half* __restrict__ out, long long n8) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n8) return;
  const float av = __ldg(a), bv = y ? __ldg(b) : 0.f;
  float fx[8], fy[8];
  unpack8(ldg16(x + i * 8), fx);
  if (y) {
    unpack8(ldg16(y + i * 8), fy);
#pragma unroll
    for (int e = 0; e < 8; ++e) fx[e] = av * fx[e] + bv * fy[e];
  } else {
#pragma unroll
    for (int e = 0; e < 8; ++e) fx[e] = av * fx[e];
  }
  *reinterpret_cast<uint4*>(out + i * 8) = pack8(fx);
}

// The coefficient pairs of an fp32 token stream (common.py:747-750 under autocast): out = a * x (+ b * y), x the fp32 stream,
// y an fp16 branch output, out fp32 or fp16 (TOut).  A one-element fp32 parameter times an fp16 tensor promotes to fp32, so
// the reference forms two rounded fp32 products and a rounded sum: __fmul_rn / __fadd_rn keep the compiler from contracting
// them into an FMA, and the result is torch's `c_a * x + c_b * y`, bit for bit.  An fp16 TOut is the backward's branch
// gradient, rounded once to the branch's dtype.
template <typename TOut>
__global__ void __launch_bounds__(256) axpby_f32_kernel(const float* __restrict__ x, const __half* __restrict__ y, const float* __restrict__ a,
                                                        const float* __restrict__ b, TOut* __restrict__ out, long long n8) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n8) return;
  const float av = __ldg(a), bv = y ? __ldg(b) : 0.f;
  float fx[8];
  ld8f(x + i * 8, fx);
  if (y) {
    float fy[8];
    unpack8(ldg16(y + i * 8), fy);
#pragma unroll
    for (int e = 0; e < 8; ++e) fx[e] = __fadd_rn(__fmul_rn(av, fx[e]), __fmul_rn(bv, fy[e]));
  } else {
#pragma unroll
    for (int e = 0; e < 8; ++e) fx[e] = __fmul_rn(av, fx[e]);
  }
  st8(out + i * 8, fx);
}

}  // namespace icaf

using namespace icaf;

extern "C" int icaf_dmff_pool_tokens(const void* x_vis, const void* x_ir, int64_t x_ld, const void* pos_vis,
                                     const void* pos_ir, const float* mix, void* tok_vis, void* tok_ir, float* stats_vis,
                                     float* stats_ir, int B, int H, int W, int C, int nh, int nw, int n_pad, void* stream) {
  if (!x_vis || !x_ir || !pos_vis || !pos_ir || !mix || !tok_vis || !tok_ir) return set_error(ICAF_ERR_BAD_ARG, "dmff_pool_tokens: null pointer");
  if (C % 8 || x_ld % 8 || nh < 1 || nw < 1 || nh > H || nw > W || n_pad < nh * nw || n_pad % 8)
    return set_error(ICAF_ERR_BAD_ARG, "dmff_pool_tokens: bad shape (token grid must not exceed the map)");
  if ((stats_vis || stats_ir) && (!stats_vis || !stats_ir || C % 32))
    return set_error(ICAF_ERR_BAD_ARG, "dmff_pool_tokens: row statistics need both outputs and C % 32 == 0");
  PoolTokParams P = pool_tok_params(x_vis, x_ir, x_ld, mix, B, H, W, C, nh, nw, n_pad);
  P.pos[0] = (const __half*)pos_vis; P.pos[1] = (const __half*)pos_ir;
  P.tok[0] = (__half*)tok_vis; P.tok[1] = (__half*)tok_ir;
  P.stats[0] = (float2*)stats_vis; P.stats[1] = (float2*)stats_ir;
  long long total = (long long)B * n_pad * P.C8;
  dim3 grid(blocks_for(total, 128), 2);
  return launch_k("dmff_pool_tokens", dmff_pool_tokens_kernel, dim3(grid), dim3(128), 0, (cudaStream_t)stream, P);
}

extern "C" int icaf_dmff_pool_tokens_bwd(const void* x_vis, const void* x_ir, int64_t x_ld, const void* dtok_vis, const void* dtok_ir, const float* mix,
                                         void* dx_vis, void* dx_ir, int B, int H, int W, int C, int nh, int nw, int n_pad, void* workspace,
                                         size_t workspace_bytes, void* stream) {
  if (!x_vis || !x_ir || !dtok_vis || !dtok_ir || !mix || !dx_vis || !dx_ir || !workspace) return set_error(ICAF_ERR_BAD_ARG, "dmff_pool_tokens_bwd: null pointer");
  if (workspace_bytes < 2 * size_t(B) * nh * nw * C || (reinterpret_cast<uintptr_t>(workspace) & 7))
    return set_error(ICAF_ERR_BAD_ARG, "dmff_pool_tokens_bwd: workspace needs 2*B*nh*nw*C bytes, 8-byte aligned");
  if (C % 8 || x_ld % 8 || B < 1 || nh < 1 || nw < 1 || H < nh || W < nw || n_pad < nh * nw)
    return set_error(ICAF_ERR_BAD_ARG, "dmff_pool_tokens_bwd: bad shape");
  PoolTokParams P = pool_tok_params(x_vis, x_ir, x_ld, mix, B, H, W, C, nh, nw, n_pad);
  if (P.kh * P.kw > 255) return set_error(ICAF_ERR_UNSUPPORTED, "dmff_pool_tokens_bwd: pooling windows of more than 255 pixels");
  P.dtok[0] = (const __half*)dtok_vis; P.dtok[1] = (const __half*)dtok_ir;
  P.dx[0] = (__half*)dx_vis; P.dx[1] = (__half*)dx_ir;
  P.code[0] = (uint2*)workspace; P.code[1] = P.code[0] + size_t(B) * nh * nw * P.C8;
  const long long nwin = (long long)B * nh * nw * P.C8;
  if (int rc = launch_k("dmff_pool_tokens_bwd(argmax)", dmff_pool_argmax_kernel, dim3(blocks_for(nwin, 128), 2), dim3(128), 0, (cudaStream_t)stream, P)) return rc;
  const long long total = (long long)B * H * W * P.C8;
  return launch_k("dmff_pool_tokens_bwd", dmff_pool_tokens_bwd_kernel<__half>, dim3(blocks_for(total, 128), 2), dim3(128), 0, (cudaStream_t)stream, P);
}

extern "C" int icaf_dmff_upsample_cat(const void* tok_vis, const void* tok_ir, int n_pad, const void* x_vis,
                                      const void* x_ir, int64_t x_ld, void* y, int64_t y_ld, int B, int H, int W, int C,
                                      int nh, int nw, int mode, void* stream) {
  if (!tok_vis || !tok_ir || !x_vis || !x_ir || !y) return set_error(ICAF_ERR_BAD_ARG, "dmff_upsample_cat: null pointer");
  if (C % 8 || x_ld % 8 || y_ld % 8 || y_ld < 2 * C || n_pad < nh * nw) return set_error(ICAF_ERR_BAD_ARG, "dmff_upsample_cat: bad shape");
  UpCatParams P;
  P.tok[0] = (const __half*)tok_vis; P.tok[1] = (const __half*)tok_ir;
  P.x[0] = (const __half*)x_vis; P.x[1] = (const __half*)x_ir; P.y = (__half*)y;
  P.x_ld = x_ld; P.y_ld = y_ld; P.B = B; P.H = H; P.W = W; P.C8 = C / 8; P.nh = nh; P.nw = nw; P.n_pad = n_pad; P.mode = mode;
  P.sy = float(nh) / float(H); P.sx = float(nw) / float(W);
  long long total = (long long)B * H * W * P.C8;
  dim3 grid(blocks_for(total, 256), 2);
  return launch_k("dmff_upsample_cat", dmff_upsample_cat_kernel<__half>, dim3(grid), dim3(256), 0, (cudaStream_t)stream, P);
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
  return launch_k("dmff_upsample_cat_bwd", dmff_upsample_cat_bwd_kernel<__half>, dim3(blocks_for(total, 128), 2), dim3(128), 0, (cudaStream_t)stream, P);
}

extern "C" int icaf_layernorm(const void* x0, const void* x1, const float* g0, const float* b0, const float* g1,
                              const float* b1, void* y0, void* y1, int64_t rows, int C, float eps, void* stream) {
  if (!x0 || !y0 || !g0 || !b0 || (x1 && (!y1 || !g1 || !b1))) return set_error(ICAF_ERR_BAD_ARG, "layernorm: null pointer");
  if (C % 8 || C > 2048 || rows < 1) return set_error(ICAF_ERR_UNSUPPORTED, "layernorm: C must be a multiple of 8, <= 2048");
  LnParams P;
  P.x[0] = (const __half*)x0; P.x[1] = (const __half*)x1; P.y[0] = (__half*)y0; P.y[1] = (__half*)y1;
  P.g[0] = g0; P.g[1] = g1; P.b[0] = b0; P.b[1] = b1; P.rows = rows; P.C = C; P.eps = eps;
  dim3 grid(blocks_for(rows, 4), x1 ? 2 : 1);
  return launch_k("layernorm", layernorm_kernel<__half>, dim3(grid), dim3(128), 0, (cudaStream_t)stream, P);
}

extern "C" int icaf_row_stats(const void* x0, const void* x1, float* stats0, float* stats1, int64_t rows, int C, void* stream) {
  if (!x0 || !stats0 || (x1 && !stats1) || rows < 1 || C < 8 || C % 8) return set_error(ICAF_ERR_BAD_ARG, "row_stats: bad argument");
  dim3 grid(blocks_for(rows, 4), x1 ? 2 : 1);
  return launch_k("row_stats", row_stats_kernel, dim3(grid), dim3(128), 0, (cudaStream_t)stream, (const __half*)x0, (const __half*)x1,
                  (float2*)stats0, (float2*)stats1, (long long)rows, C);
}

extern "C" int icaf_axpby(const void* x, const void* y, const float* a, const float* b, void* out, int64_t n, void* stream) {
  if (!x || !a || !out || (y && !b) || n < 0 || n % 8) return set_error(ICAF_ERR_BAD_ARG, "axpby: null pointer or element count not a multiple of 8");
  if (n == 0) return ICAF_OK;
  return launch_k("axpby", axpby_kernel, dim3(blocks_for(n / 8, 256)), dim3(256), 0, (cudaStream_t)stream, (const __half*)x, (const __half*)y, a, b,
                  (__half*)out, (long long)(n / 8));
}

// ------------------------------------------------------------------------------------------------
// fp32 DMFF token streams (training, TransformerFusionBlock.stream_dtype = float32): the same operators with fp32 tokens and
// token gradients; maps, map gradients and GEMM operands stay fp16.
extern "C" int icaf_dmff_pool_tokens_f32(const void* x_vis, const void* x_ir, int64_t x_ld, const float* pos_vis, const float* pos_ir,
                                         const float* mix, float* tok_vis, float* tok_ir, int B, int H, int W, int C, int nh, int nw,
                                         int n_pad, void* stream) {
  if (!x_vis || !x_ir || !pos_vis || !pos_ir || !mix || !tok_vis || !tok_ir) return set_error(ICAF_ERR_BAD_ARG, "dmff_pool_tokens_f32: null pointer");
  if (C % 8 || x_ld % 8 || B < 1 || nh < 1 || nw < 1 || nh > H || nw > W || n_pad < nh * nw || n_pad % 8)
    return set_error(ICAF_ERR_BAD_ARG, "dmff_pool_tokens_f32: bad shape (token grid must not exceed the map)");
  PoolTokParams P = pool_tok_params(x_vis, x_ir, x_ld, mix, B, H, W, C, nh, nw, n_pad);
  P.pos_f32[0] = pos_vis; P.pos_f32[1] = pos_ir;
  P.tok_f32[0] = tok_vis; P.tok_f32[1] = tok_ir;
  P.stats[0] = P.stats[1] = nullptr;
  const long long total = (long long)B * n_pad * P.C8;
  return launch_k("dmff_pool_tokens_f32", dmff_pool_tokens_f32_kernel, dim3(blocks_for(total, 128), 2), dim3(128), 0, (cudaStream_t)stream, P);
}

extern "C" int icaf_dmff_pool_tokens_bwd_f32(const void* x_vis, const void* x_ir, int64_t x_ld, const float* dtok_vis, const float* dtok_ir,
                                             const float* mix, void* dx_vis, void* dx_ir, int B, int H, int W, int C, int nh, int nw, int n_pad,
                                             void* workspace, size_t workspace_bytes, void* stream) {
  if (!x_vis || !x_ir || !dtok_vis || !dtok_ir || !mix || !dx_vis || !dx_ir || !workspace) return set_error(ICAF_ERR_BAD_ARG, "dmff_pool_tokens_bwd_f32: null pointer");
  if (workspace_bytes < 2 * size_t(B) * nh * nw * C || (reinterpret_cast<uintptr_t>(workspace) & 7))
    return set_error(ICAF_ERR_BAD_ARG, "dmff_pool_tokens_bwd_f32: workspace needs 2*B*nh*nw*C bytes, 8-byte aligned");
  if (C % 8 || x_ld % 8 || B < 1 || nh < 1 || nw < 1 || H < nh || W < nw || n_pad < nh * nw)
    return set_error(ICAF_ERR_BAD_ARG, "dmff_pool_tokens_bwd_f32: bad shape");
  PoolTokParams P = pool_tok_params(x_vis, x_ir, x_ld, mix, B, H, W, C, nh, nw, n_pad);
  if (P.kh * P.kw > 255) return set_error(ICAF_ERR_UNSUPPORTED, "dmff_pool_tokens_bwd_f32: pooling windows of more than 255 pixels");
  P.dtok_f32[0] = dtok_vis; P.dtok_f32[1] = dtok_ir;
  P.dx[0] = (__half*)dx_vis; P.dx[1] = (__half*)dx_ir;
  P.code[0] = (uint2*)workspace; P.code[1] = P.code[0] + size_t(B) * nh * nw * P.C8;
  const long long nwin = (long long)B * nh * nw * P.C8;
  if (int rc = launch_k("dmff_pool_tokens_bwd_f32(argmax)", dmff_pool_argmax_kernel, dim3(blocks_for(nwin, 128), 2), dim3(128), 0, (cudaStream_t)stream, P)) return rc;
  const long long total = (long long)B * H * W * P.C8;
  return launch_k("dmff_pool_tokens_bwd_f32", dmff_pool_tokens_bwd_kernel<float>, dim3(blocks_for(total, 128), 2), dim3(128), 0, (cudaStream_t)stream, P);
}

extern "C" int icaf_dmff_upsample_cat_f32(const float* tok_vis, const float* tok_ir, int n_pad, const void* x_vis, const void* x_ir, int64_t x_ld,
                                          void* y, int64_t y_ld, int B, int H, int W, int C, int nh, int nw, void* stream) {
  if (!tok_vis || !tok_ir || !x_vis || !x_ir || !y) return set_error(ICAF_ERR_BAD_ARG, "dmff_upsample_cat_f32: null pointer");
  if (C % 8 || x_ld % 8 || y_ld % 8 || y_ld < 2 * C || B < 1 || nh < 1 || nw < 1 || nh > H || nw > W || n_pad < nh * nw)
    return set_error(ICAF_ERR_BAD_ARG, "dmff_upsample_cat_f32: bad shape");
  UpCatParams P;
  P.tok_f32[0] = tok_vis; P.tok_f32[1] = tok_ir;
  P.x[0] = (const __half*)x_vis; P.x[1] = (const __half*)x_ir; P.y = (__half*)y;
  P.x_ld = x_ld; P.y_ld = y_ld; P.B = B; P.H = H; P.W = W; P.C8 = C / 8; P.nh = nh; P.nw = nw; P.n_pad = n_pad; P.mode = 1;   // nearest (training)
  P.sy = float(nh) / float(H); P.sx = float(nw) / float(W);
  const long long total = (long long)B * H * W * P.C8;
  return launch_k("dmff_upsample_cat_f32", dmff_upsample_cat_kernel<float>, dim3(blocks_for(total, 256), 2), dim3(256), 0, (cudaStream_t)stream, P);
}

extern "C" int icaf_dmff_upsample_cat_bwd_f32(const void* dcat, int64_t d_ld, float* dtok_vis, float* dtok_ir, int B, int H, int W, int C, int nh,
                                              int nw, int n_pad, void* stream) {
  if (!dcat || !dtok_vis || !dtok_ir) return set_error(ICAF_ERR_BAD_ARG, "dmff_upsample_cat_bwd_f32: null pointer");
  if (C % 8 || d_ld % 8 || d_ld < 2 * C || B < 1 || nh < 1 || nw < 1 || nh > H || nw > W || n_pad < nh * nw)
    return set_error(ICAF_ERR_BAD_ARG, "dmff_upsample_cat_bwd_f32: bad shape");
  UpCatBwdParams P;
  P.dcat = (const __half*)dcat; P.dtok_f32[0] = dtok_vis; P.dtok_f32[1] = dtok_ir; P.d_ld = d_ld;
  P.B = B; P.H = H; P.W = W; P.C8 = C / 8; P.nh = nh; P.nw = nw; P.n_pad = n_pad;
  P.sy = float(nh) / float(H); P.sx = float(nw) / float(W);
  const long long total = (long long)B * n_pad * P.C8;
  return launch_k("dmff_upsample_cat_bwd_f32", dmff_upsample_cat_bwd_kernel<float>, dim3(blocks_for(total, 128), 2), dim3(128), 0, (cudaStream_t)stream, P);
}

extern "C" int icaf_layernorm_f32(const float* x0, const float* x1, const float* g0, const float* b0, const float* g1, const float* b1, void* y0,
                                  void* y1, int64_t rows, int C, float eps, void* stream) {
  if (!x0 || !y0 || !g0 || !b0 || (x1 && (!y1 || !g1 || !b1))) return set_error(ICAF_ERR_BAD_ARG, "layernorm_f32: null pointer");
  if (C % 8 || C > 2048 || rows < 1) return set_error(ICAF_ERR_UNSUPPORTED, "layernorm_f32: C must be a multiple of 8, <= 2048");
  LnParams P;
  P.x_f32[0] = x0; P.x_f32[1] = x1; P.y[0] = (__half*)y0; P.y[1] = (__half*)y1;
  P.g[0] = g0; P.g[1] = g1; P.b[0] = b0; P.b[1] = b1; P.rows = rows; P.C = C; P.eps = eps;
  return launch_k("layernorm_f32", layernorm_kernel<float>, dim3(blocks_for(rows, 4), x1 ? 2 : 1), dim3(128), 0, (cudaStream_t)stream, P);
}

// out = a * x (+ b * y): x fp32, y fp16 (optional), out fp16 when out_f16 else fp32
extern "C" int icaf_axpby_f32(const float* x, const void* y, const float* a, const float* b, void* out, int out_f16, int64_t n, void* stream) {
  if (!x || !a || !out || (y && !b) || n < 0 || n % 8) return set_error(ICAF_ERR_BAD_ARG, "axpby_f32: null pointer or element count not a multiple of 8");
  if (n == 0) return ICAF_OK;
  const dim3 grid(blocks_for(n / 8, 256));
  if (out_f16)
    return launch_k("axpby_f32", axpby_f32_kernel<__half>, grid, dim3(256), 0, (cudaStream_t)stream, x, (const __half*)y, a, b, (__half*)out, (long long)(n / 8));
  return launch_k("axpby_f32", axpby_f32_kernel<float>, grid, dim3(256), 0, (cudaStream_t)stream, x, (const __half*)y, a, b, (float*)out, (long long)(n / 8));
}
