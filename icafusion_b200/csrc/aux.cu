// HBM-bound helper kernels of the hot path (everything that is not a GEMM): image staging, SPPF pooling,
// nearest up-sampling / concat copies, DMFF token pooling (+pos-emb), LayerNorm, DMFF bilinear tail, Detect decode.
// All work on fp16 NHWC views; each thread moves 16-byte (8-channel) vectors so every warp access is a run of
// full 128-byte lines along the channel axis.
#include <climits>

#include "icaf_internal.cuh"

namespace icaf {

// ------------------------------------------------------------------------------------------------
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
// SPPF: three chained 5x5/s1/p2 max pools == 5x5, 9x9, 13x13 windows clipped to the map (-inf padding)
__global__ void sppf_pool_kernel(const __half* __restrict__ x, long long x_ld, __half* y1, __half* y2, __half* y3,
                                 long long y_ld, int B, int H, int W, int C8) {
  pdl_launch_dependents();
  pdl_wait();
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  long long total = (long long)B * H * W * C8;
  if (i >= total) return;
  int c = int(i % C8);
  long long p = i / C8;
  int px = int(p % W);
  long long t = p / W;
  int py = int(t % H);
  int b = int(t / H);
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

// ------------------------------------------------------------------------------------------------
__global__ void upsample2x_kernel(const __half* __restrict__ x, long long x_ld, __half* __restrict__ y, long long y_ld,
                                  int B, int H, int W, int C8) {
  pdl_launch_dependents();
  pdl_wait();
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  long long total = (long long)B * (2 * H) * (2 * W) * C8;
  if (i >= total) return;
  int c = int(i % C8);
  long long p = i / C8;
  int ox = int(p % (2 * W));
  long long t = p / (2 * W);
  int oy = int(t % (2 * H));
  int b = int(t / (2 * H));
  uint4 v = ldg16(x + ((long long)(b * H + (oy >> 1)) * W + (ox >> 1)) * x_ld + c * 8);
  *reinterpret_cast<uint4*>(y + p * y_ld + c * 8) = v;
}

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

// ------------------------------------------------------------------------------------------------
// DMFF front: avg+max pool with (kh,kw)/(sh,sw) windows, learnable mix, + pos_emb -> tokens (B,Npad,C)
struct PoolTokParams {
  const __half* x[2]; const __half* pos[2]; __half* tok[2];
  float2* stats[2];        // optional: (sum, sum of squares) of every token row per 32 channels, [B*Npad][C/32]
  const float* mix;
  long long x_ld;
  int B, H, W, C8, nh, nw, n_pad, kh, kw, sh, sw;
};
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
    const __half* x = mod ? P.x[1] : P.x[0];
    const int ty = n / P.nw, tx = n % P.nw;
    float sum[8], mx[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) { sum[e] = 0.f; mx[e] = -INFINITY; }
    // window elements are fetched 8 at a time (independent 16-byte loads in flight) before they are reduced
    const __half* x0 = x + ((long long)(b * P.H + ty * P.sh) * P.W + tx * P.sw) * P.x_ld + c * 8;
    const int wn = P.kh * P.kw;
    for (int w0 = 0; w0 < wn; w0 += 8) {
      uint4 v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        int w = w0 + j;
        int ky = w / P.kw, kx = w - ky * P.kw;
        if (w < wn) v[j] = ldg16(x0 + ((long long)ky * P.W + kx) * P.x_ld);
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

// ------------------------------------------------------------------------------------------------
// LayerNorm: one warp per row, row cached in registers (C <= 2048)
struct LnParams {
  const __half* x[2]; __half* y[2]; const float* g[2]; const float* b[2];
  long long rows; int C; float eps;
};
__global__ void layernorm_kernel(const LnParams P) {
  pdl_launch_dependents();
  pdl_wait();
  const int prob = blockIdx.y;
  const long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= P.rows) return;
  const int lane = threadIdx.x & 31;
  const __half* x = (prob ? P.x[1] : P.x[0]) + row * P.C;
  __half* y = (prob ? P.y[1] : P.y[0]) + row * P.C;
  const float* g = prob ? P.g[1] : P.g[0];
  const float* be = prob ? P.b[1] : P.b[0];
  const int nch = P.C >> 3;                 // 16-byte chunks in the row
  float v[8][8];                            // up to 8 chunks per lane -> C <= 2048
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    int ch = lane + 32 * j;
    if (ch < nch) {
      unpack8(ldg16(x + ch * 8), v[j]);
#pragma unroll
      for (int e = 0; e < 8; ++e) s += v[j][e];
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / float(P.C);
  float q = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    int ch = lane + 32 * j;
    if (ch < nch) {
#pragma unroll
      for (int e = 0; e < 8; ++e) { float d = v[j][e] - mean; q += d * d; }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / float(P.C) + P.eps);
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
// DMFF tail: tokens -> (nh,nw) map -> interpolate to (H,W) + stream features -> concat buffer (B,H,W,2C)
struct UpCatParams {
  const __half* tok[2]; const __half* x[2]; __half* y;
  long long x_ld, y_ld;
  int B, H, W, C8, nh, nw, n_pad, mode;
  float sy, sx;   // nh/H, nw/W
};
__global__ void dmff_upsample_cat_kernel(const UpCatParams P) {
  pdl_launch_dependents();
  pdl_wait();
  const int mod = blockIdx.y;
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  long long total = (long long)P.B * P.H * P.W * P.C8;
  if (i >= total) return;
  int c = int(i % P.C8);
  long long p = i / P.C8;
  int ox = int(p % P.W);
  long long t = p / P.W;
  int oy = int(t % P.H);
  int b = int(t / P.H);
  const int C = P.C8 * 8;
  const __half* tok = (mod ? P.tok[1] : P.tok[0]) + (long long)b * P.n_pad * C + c * 8;
  float r[8];
  if (P.nh == P.H && P.nw == P.W) {                    // identity resample (un-pooled DMFF)
    unpack8(ldg16(tok + (long long)(oy * P.nw + ox) * C), r);
  } else if (P.mode == 1) {                            // nearest: src = min(floor(dst*scale), in-1)
    int iy = min(int(floorf(oy * P.sy)), P.nh - 1), ix = min(int(floorf(ox * P.sx)), P.nw - 1);
    unpack8(ldg16(tok + (long long)(iy * P.nw + ix) * C), r);
  } else {                                             // bilinear, align_corners=False
    float fy = fmaxf((oy + 0.5f) * P.sy - 0.5f, 0.f), fx = fmaxf((ox + 0.5f) * P.sx - 0.5f, 0.f);
    int y0 = int(fy), x0 = int(fx);
    int y1 = min(y0 + 1, P.nh - 1), x1 = min(x0 + 1, P.nw - 1);
    float ly = fy - y0, lx = fx - x0;
    float a[8], bq[8], cq[8], d[8];
    unpack8(ldg16(tok + (long long)(y0 * P.nw + x0) * C), a);
    unpack8(ldg16(tok + (long long)(y0 * P.nw + x1) * C), bq);
    unpack8(ldg16(tok + (long long)(y1 * P.nw + x0) * C), cq);
    unpack8(ldg16(tok + (long long)(y1 * P.nw + x1) * C), d);
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

// ------------------------------------------------------------------------------------------------
// Detect decode for one level
struct DetectParams {
  const __half* p; long long p_ld;
  __half* x_out; __half* z; __half* logits;
  int B, ny, nx, na, no, total_rows, row_off;
  float stride;
  float anchors[16];
};
__global__ void detect_decode_kernel(const DetectParams P) {
  pdl_launch_dependents();
  pdl_wait();
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  long long total = (long long)P.B * P.na * P.ny * P.nx;
  if (i >= total) return;
  int gx = int(i % P.nx);
  long long t = i / P.nx;
  int gy = int(t % P.ny); t /= P.ny;
  int a = int(t % P.na);
  int b = int(t / P.na);
  const __half* src = P.p + ((long long)(b * P.ny + gy) * P.nx + gx) * P.p_ld + a * P.no;
  __half* xo = P.x_out + i * P.no;                                      // (B,na,ny,nx,no) contiguous
  long long zr = (long long)b * P.total_rows + P.row_off + ((long long)a * P.ny + gy) * P.nx + gx;
  __half* zo = P.z + zr * P.no;
  __half* lo = P.logits + zr * (P.no - 5);
  for (int o = 0; o < P.no; ++o) {
    __half raw = src[o];
    xo[o] = raw;
    float v = __half2float(raw);
    float s = 1.f / (1.f + __expf(-v));
    float r;
    if (o == 0) r = (s * 2.f - 0.5f + gx) * P.stride;
    else if (o == 1) r = (s * 2.f - 0.5f + gy) * P.stride;
    else if (o == 2) r = (s * 2.f) * (s * 2.f) * P.anchors[a * 2];
    else if (o == 3) r = (s * 2.f) * (s * 2.f) * P.anchors[a * 2 + 1];
    else r = s;
    zo[o] = __float2half_rn(r);
    if (o >= 5) lo[o - 5] = raw;
  }
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

// ------------------------------------------------------------------------------------------------
// Batched non-maximum suppression on the decoded predictions (reference: utils/general.py:518-607, best-class branch +
// torchvision.ops.nms).  Three launches, no host round trip:
//   1. candidates: obj > conf_thres and conf = obj * max_k cls_k > conf_thres (fp32 from the fp16 predictions), class filter;
//      key = (conf bits << 32) | ~row  -> descending key order = descending confidence, ties in row order (= stable sort)
//   2. rank sort: rank[i] = #{j : key_j > key_i} (keys are unique), order[rank] = row
//   3. greedy suppression in confidence order, 16 candidates per round (one per warp against the kept list, then warp 0
//      resolves the round in order); stops after max_det kept boxes.  IoU arithmetic mirrors torchvision's kernel in fp32
//      (no FMA contraction), boxes offset by cls * 4096 unless agnostic (general.py:590-592).
// Multi-label mode (general.py:566-568) reuses the filter and suppression kernels; only the order step differs:
//   1. one candidate per (row r, class j) with obj > conf_thres and cls_j * obj > conf_thres, id = r * nc + j; the filter
//      writes a sort key for every id (a sentinel where there is no candidate), so the key array is in id order
//   2. nms_sort_kernel, one block per image: a stable LSD radix sort (4 passes of 8 bits) of the keys; its first pass also
//      compacts the candidates in id order, so the result is descending confidence with ties in id order.  Work is linear
//      in R * nc, where the rank sort above is quadratic in the candidate count (60 480 candidates at test.py's setting)
//   3. the same greedy suppression; a candidate's box is its row's, its conf and class those of class j
constexpr int kNmsThreads = 512;
constexpr int kNmsMaxDet = 1024;
constexpr int kNmsSortThreads = 1024, kNmsSortItems = 4;
constexpr unsigned kNmsNoKey = 0xffffffffu;      // no candidate (no valid key maps here: see nms_sort_key)
struct NmsParams {
  const __half* z;
  int B, R, no, agnostic, max_det, max_nms, multi_label;
  float conf_thres, iou_thres;
  unsigned long long class_mask;
  float* det; int* count;
  unsigned long long* keys; int* order;
  unsigned* mkeys[2]; int* mids[2];           // multi-label: radix ping-pong buffers, R * nc entries per image each
};
// ascending order of the key = descending order of the float (sign-flip to an ordered integer, then complement)
__device__ __forceinline__ unsigned nms_sort_key(float conf) {
  const unsigned u = __float_as_uint(conf);
  return ~(u ^ ((u >> 31) ? 0xffffffffu : 0x80000000u));
}
struct NmsBox { float x1, y1, x2, y2, conf, cls; };
// cls < 0: the best class (best-class branch); otherwise class `cls` (multi-label branch)
__device__ __forceinline__ NmsBox nms_box(const __half* __restrict__ r, int no, int cls = -1) {
  NmsBox b;
  const float cx = __half2float(r[0]), cy = __half2float(r[1]), w = __half2float(r[2]), h = __half2float(r[3]);
  const float obj = __half2float(r[4]);
  float best;
  int bj;
  if (cls >= 0) {
    best = __fmul_rn(__half2float(r[5 + cls]), obj);
    bj = cls;
  } else {
    best = __fmul_rn(__half2float(r[5]), obj);
    bj = 0;
    for (int k = 1; k < no - 5; ++k) {
      const float c = __fmul_rn(__half2float(r[5 + k]), obj);
      if (c > best) { best = c; bj = k; }
    }
  }
  const float hw = __fmul_rn(w, 0.5f), hh = __fmul_rn(h, 0.5f);       // xywh2xyxy, general.py:332-339
  b.x1 = __fsub_rn(cx, hw); b.y1 = __fsub_rn(cy, hh); b.x2 = __fadd_rn(cx, hw); b.y2 = __fadd_rn(cy, hh);
  b.conf = best; b.cls = float(bj);
  return b;
}
__device__ __forceinline__ bool nms_iou_gt(const float4& a, const float4& b, float thr) {
  const float left = fmaxf(a.x, b.x), right = fminf(a.z, b.z), top = fmaxf(a.y, b.y), bottom = fminf(a.w, b.w);
  const float w = fmaxf(__fsub_rn(right, left), 0.f), h = fmaxf(__fsub_rn(bottom, top), 0.f);
  const float inter = __fmul_rn(w, h);
  const float sa = __fmul_rn(__fsub_rn(a.z, a.x), __fsub_rn(a.w, a.y));
  const float sb = __fmul_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y));
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(sa, sb), inter)) > thr;
}
// the box, confidence and class of candidate `id` (a row, or row * nc + class in multi-label mode) of image z
__device__ __forceinline__ NmsBox nms_candidate(const NmsParams& P, const __half* z, int id) {
  if (!P.multi_label) return nms_box(z + (size_t)id * P.no, P.no);
  const int nc = P.no - 5, r = id / nc;
  return nms_box(z + (size_t)r * P.no, P.no, id - r * nc);
}
// phase 1: grid (ceil(R / 256), B) -- candidate keys, compacted per image through one integer counter (order is irrelevant:
// the keys are unique and the rank sort below orders them).  Multi-label: one key per (row, class), kNmsNoKey where the
// pair is no candidate.
__global__ void __launch_bounds__(256) nms_filter_kernel(const NmsParams P) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.y, r = blockIdx.x * 256 + threadIdx.x;
  if (r >= P.R) return;
  const __half* row = P.z + ((size_t)b * P.R + r) * P.no;
  if (P.multi_label) {
    const int nc = P.no - 5;
    const float obj = __half2float(row[4]);
    const bool obj_ok = obj > P.conf_thres;
    unsigned* keys = P.mkeys[0] + ((size_t)b * P.R + r) * nc;
    for (int j = 0; j < nc; ++j) {
      const float c = __fmul_rn(__half2float(row[5 + j]), obj);
      const bool ok = obj_ok && c > P.conf_thres && (!P.class_mask || ((P.class_mask >> j) & 1ull));
      keys[j] = ok ? nms_sort_key(c) : kNmsNoKey;
    }
    return;
  }
  if (!(__half2float(row[4]) > P.conf_thres)) return;
  const NmsBox bx = nms_box(row, P.no);
  if (!(bx.conf > P.conf_thres)) return;
  if (P.class_mask && !((P.class_mask >> int(bx.cls)) & 1ull)) return;
  const int slot = atomicAdd(P.count + b, 1);                 // `count` doubles as the candidate counter until phase 3 overwrites it
  P.keys[(size_t)b * P.R + slot] = ((unsigned long long)__float_as_uint(bx.conf) << 32) | (unsigned long long)(~(unsigned)r);
}
// phase 2: grid (ceil(R / 256), B) -- rank of each candidate = number of larger keys (all SMs work on the O(n^2) compares)
__global__ void __launch_bounds__(256) nms_rank_kernel(const NmsParams P) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ unsigned long long skeys[256];
  const int b = blockIdx.y;
  const int n = P.count[b];
  if (blockIdx.x * 256 >= n) return;
  const unsigned long long* keys = P.keys + (size_t)b * P.R;
  const int i = blockIdx.x * 256 + threadIdx.x;
  const unsigned long long ki = i < n ? keys[i] : 0ull;
  int rank = 0;
  for (int t0 = 0; t0 < n; t0 += 256) {
    __syncthreads();
    skeys[threadIdx.x] = t0 + threadIdx.x < n ? keys[t0 + threadIdx.x] : 0ull;
    __syncthreads();
    const int m = min(256, n - t0);
    for (int j = 0; j < m; ++j) rank += skeys[j] > ki;
  }
  if (i < n) P.order[(size_t)b * P.R + rank] = int(~(unsigned)(ki & 0xffffffffull));
}
// phase 2, multi-label: one block per image -- stable LSD radix sort of the candidate keys, 8 bits per pass, ping-ponging
// between mkeys/mids[0] and [1].  Pass 0 reads the filter's key array (implicit id = index) and drops the kNmsNoKey
// entries; the sorted ids end in mids[0] (= P.order) and the candidate count in count[b].  Inside a tile of
// kNmsSortThreads * kNmsSortItems keys, each warp ranks its keys among equal digits with __match_any_sync (element order
// within the warp: item-major, lane-minor), then the per-warp digit counts are scanned across warps in tile order.
__global__ void __launch_bounds__(kNmsSortThreads) nms_sort_kernel(const NmsParams P) {
  pdl_launch_dependents();
  pdl_wait();
  constexpr int kWarps = kNmsSortThreads / 32, kTile = kNmsSortThreads * kNmsSortItems;
  __shared__ int hist[4][256];           // per pass: digit histogram, then the running output offset of each digit
  __shared__ int wcnt[kWarps][256];      // per tile: digit counts of each warp, then each warp's output offsets
  __shared__ int s_n;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int S = P.R * (P.no - 5);
  const size_t base = (size_t)b * S;
  for (int i = tid; i < 4 * 256; i += kNmsSortThreads) (&hist[0][0])[i] = 0;
  if (tid == 0) s_n = 0;
  __syncthreads();
  int my_n = 0;
  for (int i = tid; i < S; i += kNmsSortThreads) {
    const unsigned k = P.mkeys[0][base + i];
    if (k == kNmsNoKey) continue;
    ++my_n;
#pragma unroll
    for (int p = 0; p < 4; ++p) atomicAdd(&hist[p][(k >> (8 * p)) & 255], 1);
  }
  my_n = __reduce_add_sync(0xffffffffu, my_n);
  if (lane == 0) atomicAdd(&s_n, my_n);
  __syncthreads();
  if (warp < 4) {                        // exclusive scan of histogram `warp`, 8 bins per lane
    int v[8], s = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) { v[k] = hist[warp][lane * 8 + k]; s += v[k]; }
    int incl = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    int run = incl - s;
#pragma unroll
    for (int k = 0; k < 8; ++k) { hist[warp][lane * 8 + k] = run; run += v[k]; }
  }
  __syncthreads();
  const int n = s_n;
  for (int p = 0; p < 4; ++p) {
    const bool odd = p & 1;              // (select, not index: a run-time index into the parameter arrays goes to the stack)
    const unsigned* ksrc = (odd ? P.mkeys[1] : P.mkeys[0]) + base;
    const int* isrc = (odd ? P.mids[1] : P.mids[0]) + base;
    unsigned* kdst = (odd ? P.mkeys[0] : P.mkeys[1]) + base;
    int* idst = (odd ? P.mids[0] : P.mids[1]) + base;
    const int len = p == 0 ? S : n;
    for (int t0 = 0; t0 < len; t0 += kTile) {
      for (int d = lane; d < 256; d += 32) wcnt[warp][d] = 0;
      __syncwarp();
      unsigned key[kNmsSortItems];
      int id[kNmsSortItems], dig[kNmsSortItems], rank[kNmsSortItems];
#pragma unroll
      for (int i = 0; i < kNmsSortItems; ++i) {
        const int e = t0 + (warp * kNmsSortItems + i) * 32 + lane;
        key[i] = e < len ? ksrc[e] : kNmsNoKey;
        id[i] = p == 0 ? e : (e < len ? isrc[e] : 0);
      }
#pragma unroll
      for (int i = 0; i < kNmsSortItems; ++i) {
        dig[i] = key[i] != kNmsNoKey ? int((key[i] >> (8 * p)) & 255) : 256;
        const unsigned peers = __match_any_sync(0xffffffffu, dig[i]);
        const int below = __popc(peers & ((1u << lane) - 1u));
        rank[i] = dig[i] < 256 ? wcnt[warp][dig[i]] + below : 0;
        __syncwarp();
        if (dig[i] < 256 && below == 0) wcnt[warp][dig[i]] += __popc(peers);
        __syncwarp();
      }
      __syncthreads();
      if (tid < 256) {
        int run = hist[p][tid];
        for (int w = 0; w < kWarps; ++w) {
          const int c = wcnt[w][tid];
          wcnt[w][tid] = run;
          run += c;
        }
        hist[p][tid] = run;
      }
      __syncthreads();
#pragma unroll
      for (int i = 0; i < kNmsSortItems; ++i) {
        if (dig[i] == 256) continue;
        const int pos = wcnt[warp][dig[i]] + rank[i];
        kdst[pos] = key[i];
        idst[pos] = id[i];
      }
      __syncthreads();
    }
  }
  if (tid == 0) P.count[b] = n;
}
// phase 3: one block per image -- greedy suppression in confidence order, 16 candidates per round
__global__ void __launch_bounds__(kNmsThreads) nms_kernel(const NmsParams P) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float4 kept[kNmsMaxDet];        // offset boxes of the kept detections
  __shared__ float4 round_box[16];
  __shared__ int round_sup[16];
  __shared__ int s_kept;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const __half* z = P.z + (size_t)b * P.R * P.no;
  const int* order = P.order + (size_t)b * P.R * (P.multi_label ? P.no - 5 : 1);
  const int n = P.count[b];
  if (tid == 0) s_kept = 0;
  __syncthreads();
  const int n_eff = min(n, P.max_nms);
  float* det = P.det + (size_t)b * P.max_det * 6;
  for (int c0 = 0; c0 < n_eff; c0 += 16) {
    const int nk = s_kept;
    if (nk >= P.max_det) break;
    const int c = c0 + warp;
    NmsBox bx;
    float4 ob = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < n_eff) {
      bx = nms_candidate(P, z, order[c]);
      const float off = P.agnostic ? 0.f : __fmul_rn(bx.cls, 4096.f);
      ob = make_float4(__fadd_rn(bx.x1, off), __fadd_rn(bx.y1, off), __fadd_rn(bx.x2, off), __fadd_rn(bx.y2, off));
      bool sup = false;
      for (int k = lane; k < nk; k += 32) sup |= nms_iou_gt(kept[k], ob, P.iou_thres);
      sup = __any_sync(0xffffffffu, sup);
      if (lane == 0) { round_sup[warp] = sup; round_box[warp] = ob; }
    } else if (lane == 0) {
      round_sup[warp] = 1;
    }
    __syncthreads();
    if (warp == 0) {                       // resolve the round in confidence order against the boxes it adds itself
      int nk2 = nk;
      const int first_new = nk;
      for (int w = 0; w < 16 && nk2 < P.max_det; ++w) {
        if (round_sup[w]) continue;        // uniform across the warp (shared memory)
        const float4 cb = round_box[w];
        bool sup = false;
        if (first_new + lane < nk2) sup = nms_iou_gt(kept[first_new + lane], cb, P.iou_thres);
        if (__any_sync(0xffffffffu, sup)) continue;
        if (lane == 0) {
          kept[nk2] = cb;
          const NmsBox kb = nms_candidate(P, z, order[c0 + w]);
          float* d = det + (size_t)nk2 * 6;
          d[0] = kb.x1; d[1] = kb.y1; d[2] = kb.x2; d[3] = kb.y2; d[4] = kb.conf; d[5] = kb.cls;
        }
        __syncwarp();
        ++nk2;
      }
      if (lane == 0) s_kept = nk2;
    }
    __syncthreads();
  }
  if (tid == 0) P.count[b] = s_kept;
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

extern "C" int icaf_upsample2x(const void* x, int64_t x_ld, void* y, int64_t y_ld, int B, int H, int W, int C, void* stream) {
  if (!x || !y || C % 8 || x_ld % 8 || y_ld % 8) return set_error(ICAF_ERR_BAD_ARG, "upsample2x: bad argument");
  long long total = (long long)B * 4 * H * W * (C / 8);
  return launch_k("upsample2x", upsample2x_kernel, dim3(blocks_for(total, 256)), dim3(256), 0, (cudaStream_t)stream, (const __half*)x, x_ld,
                  (__half*)y, y_ld, B, H, W, C / 8);
}

extern "C" int icaf_prefetch_l2(const void* ptr, size_t bytes, void* stream) {
  if (!ptr || bytes == 0) return set_error(ICAF_ERR_BAD_ARG, "prefetch_l2: bad argument");
  unsigned blocks = blocks_for((bytes + 127) / 128, 256);
  if (blocks > 148u * 8u) blocks = 148u * 8u;
  return launch_k("prefetch_l2", prefetch_l2_kernel, dim3(blocks), dim3(256), 0, (cudaStream_t)stream, (const char*)ptr, bytes);
}

extern "C" int icaf_copy_channels(const void* x, int64_t x_ld, void* y, int64_t y_ld, int64_t pixels, int C, void* stream) {
  if (!x || !y || C % 8 || x_ld % 8 || y_ld % 8) return set_error(ICAF_ERR_BAD_ARG, "copy_channels: bad argument");
  return launch_k("copy_channels", copy_channels_kernel, dim3(blocks_for(pixels * (C / 8), 256)), dim3(256), 0, (cudaStream_t)stream,
                  (const __half*)x, x_ld, (__half*)y, y_ld, pixels, C / 8);
}

extern "C" int icaf_dmff_pool_tokens(const void* x_vis, const void* x_ir, int64_t x_ld, const void* pos_vis,
                                     const void* pos_ir, const float* mix, void* tok_vis, void* tok_ir, float* stats_vis,
                                     float* stats_ir, int B, int H, int W, int C, int nh, int nw, int n_pad, void* stream) {
  if (!x_vis || !x_ir || !pos_vis || !pos_ir || !mix || !tok_vis || !tok_ir) return set_error(ICAF_ERR_BAD_ARG, "dmff_pool_tokens: null pointer");
  if (C % 8 || x_ld % 8 || nh < 1 || nw < 1 || nh > H || nw > W || n_pad < nh * nw || n_pad % 8)
    return set_error(ICAF_ERR_BAD_ARG, "dmff_pool_tokens: bad shape (token grid must not exceed the map)");
  PoolTokParams P;
  P.x[0] = (const __half*)x_vis; P.x[1] = (const __half*)x_ir;
  P.pos[0] = (const __half*)pos_vis; P.pos[1] = (const __half*)pos_ir;
  P.tok[0] = (__half*)tok_vis; P.tok[1] = (__half*)tok_ir;
  if ((stats_vis || stats_ir) && (!stats_vis || !stats_ir || C % 32))
    return set_error(ICAF_ERR_BAD_ARG, "dmff_pool_tokens: row statistics need both outputs and C % 32 == 0");
  P.stats[0] = (float2*)stats_vis; P.stats[1] = (float2*)stats_ir;
  P.mix = mix; P.x_ld = x_ld;
  P.B = B; P.H = H; P.W = W; P.C8 = C / 8; P.nh = nh; P.nw = nw; P.n_pad = n_pad;
  // AdaptivePool2d geometry, models/common.py:878-882 (identity when the map is not larger than the grid)
  P.sh = H / nh; P.sw = W / nw;
  P.kh = H - (nh - 1) * P.sh; P.kw = W - (nw - 1) * P.sw;
  long long total = (long long)B * n_pad * P.C8;
  dim3 grid(blocks_for(total, 128), 2);
  return launch_k("dmff_pool_tokens", dmff_pool_tokens_kernel, dim3(grid), dim3(128), 0, (cudaStream_t)stream, P);
}

extern "C" int icaf_layernorm(const void* x0, const void* x1, const float* g0, const float* b0, const float* g1,
                              const float* b1, void* y0, void* y1, int64_t rows, int C, float eps, void* stream) {
  if (!x0 || !y0 || !g0 || !b0 || (x1 && (!y1 || !g1 || !b1))) return set_error(ICAF_ERR_BAD_ARG, "layernorm: null pointer");
  if (C % 8 || C > 2048 || rows < 1) return set_error(ICAF_ERR_UNSUPPORTED, "layernorm: C must be a multiple of 8, <= 2048");
  LnParams P;
  P.x[0] = (const __half*)x0; P.x[1] = (const __half*)x1; P.y[0] = (__half*)y0; P.y[1] = (__half*)y1;
  P.g[0] = g0; P.g[1] = g1; P.b[0] = b0; P.b[1] = b1; P.rows = rows; P.C = C; P.eps = eps;
  dim3 grid(blocks_for(rows, 4), x1 ? 2 : 1);
  return launch_k("layernorm", layernorm_kernel, dim3(grid), dim3(128), 0, (cudaStream_t)stream, P);
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
  return launch_k("dmff_upsample_cat", dmff_upsample_cat_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream, P);
}

extern "C" int icaf_detect_decode(const void* p, int64_t p_ld, void* x_out, void* z, void* logits, int B, int ny, int nx,
                                  int na, int no, int total_rows, int row_off, float stride, const float* anchors_host,
                                  void* stream) {
  if (!p || !x_out || !z || !logits || !anchors_host || na < 1 || na > 8 || no < 6) return set_error(ICAF_ERR_BAD_ARG, "detect_decode: bad argument");
  if (B < 1 || ny < 1 || nx < 1 || p_ld < (int64_t)na * no || row_off < 0 || (long long)row_off + (long long)na * ny * nx > total_rows)
    return set_error(ICAF_ERR_BAD_ARG, "detect_decode: rows [row_off, row_off + na*ny*nx) must lie inside [0, total_rows) and p_ld >= na*no");
  DetectParams P;
  P.p = (const __half*)p; P.p_ld = p_ld; P.x_out = (__half*)x_out; P.z = (__half*)z; P.logits = (__half*)logits;
  P.B = B; P.ny = ny; P.nx = nx; P.na = na; P.no = no; P.total_rows = total_rows; P.row_off = row_off; P.stride = stride;
  for (int i = 0; i < na * 2; ++i) P.anchors[i] = anchors_host[i];
  long long total = (long long)B * na * ny * nx;
  return launch_k("detect_decode", detect_decode_kernel, dim3(blocks_for(total, 128)), dim3(128), 0, (cudaStream_t)stream, P);
}

extern "C" int icaf_axpby(const void* x, const void* y, const float* a, const float* b, void* out, int64_t n, void* stream) {
  if (!x || !a || !out || (y && !b) || n < 0 || n % 8) return set_error(ICAF_ERR_BAD_ARG, "axpby: null pointer or element count not a multiple of 8");
  if (n == 0) return ICAF_OK;
  return launch_k("axpby", axpby_kernel, dim3(blocks_for(n / 8, 256)), dim3(256), 0, (cudaStream_t)stream, (const __half*)x, (const __half*)y, a, b,
                  (__half*)out, (long long)(n / 8));
}

extern "C" size_t icaf_nms_workspace_bytes(int B, int R) {
  if (B < 1 || R < 1) return 0;
  return (size_t)B * R * (sizeof(unsigned long long) + sizeof(int));
}

extern "C" size_t icaf_nms_multi_label_workspace_bytes(int B, int R, int no) {
  if (B < 1 || R < 1 || no < 6 || (long long)R * (no - 5) > INT_MAX) return 0;
  return (size_t)B * R * (no - 5) * 2 * (sizeof(unsigned) + sizeof(int));
}

static int nms_launch(const void* z, int B, int R, int no, float conf_thres, float iou_thres, int agnostic, uint64_t class_mask,
                      int max_det, float* det, int* count, void* workspace, size_t workspace_bytes, void* stream, bool multi_label) {
  if (!z || !det || !count || !workspace) return set_error(ICAF_ERR_BAD_ARG, "nms: null pointer");
  if (B < 1 || R < 1 || no < 6 || max_det < 1 || max_det > kNmsMaxDet) return set_error(ICAF_ERR_BAD_ARG, "nms: bad shape (max_det <= 1024)");
  if (multi_label && (long long)R * (no - 5) > INT_MAX) return set_error(ICAF_ERR_UNSUPPORTED, "nms: R * nc candidates must fit in int");
  if (class_mask && no - 5 > 64) return set_error(ICAF_ERR_UNSUPPORTED, "nms: the class filter covers at most 64 classes");
  const size_t need = multi_label ? icaf_nms_multi_label_workspace_bytes(B, R, no) : icaf_nms_workspace_bytes(B, R);
  if (workspace_bytes < need || (reinterpret_cast<uintptr_t>(workspace) & 7))
    return set_error(ICAF_ERR_BAD_ARG, multi_label ? "nms: workspace too small (icaf_nms_multi_label_workspace_bytes) or not 8-byte aligned"
                                                   : "nms: workspace too small (icaf_nms_workspace_bytes) or not 8-byte aligned");
  NmsParams P = {};
  P.z = (const __half*)z; P.B = B; P.R = R; P.no = no; P.agnostic = agnostic; P.max_det = max_det; P.max_nms = 30000;   // general.py:531
  P.multi_label = multi_label;
  P.conf_thres = conf_thres; P.iou_thres = iou_thres; P.class_mask = class_mask; P.det = det; P.count = count;
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid(blocks_for(R, 256), (unsigned)B);
  if (multi_label) {
    const size_t slots = (size_t)B * R * (no - 5);
    P.mkeys[0] = (unsigned*)workspace; P.mids[0] = (int*)(P.mkeys[0] + slots);
    P.mkeys[1] = (unsigned*)(P.mids[0] + slots); P.mids[1] = (int*)(P.mkeys[1] + slots);
    P.order = P.mids[0];
    if (int rc = launch_k("nms(filter)", nms_filter_kernel, grid, dim3(256), 0, st, P)) return rc;
    if (int rc = launch_k("nms(sort)", nms_sort_kernel, dim3(B), dim3(kNmsSortThreads), 0, st, P)) return rc;
  } else {
    P.keys = (unsigned long long*)workspace;
    P.order = (int*)((char*)workspace + (size_t)B * R * sizeof(unsigned long long));
    cudaError_t e = cudaMemsetAsync(count, 0, (size_t)B * sizeof(int), st);      // candidate counters
    if (e != cudaSuccess) return set_cuda_error(e, "nms: cudaMemsetAsync");
    if (int rc = launch_k("nms(filter)", nms_filter_kernel, grid, dim3(256), 0, st, P)) return rc;
    if (int rc = launch_k("nms(rank)", nms_rank_kernel, grid, dim3(256), 0, st, P)) return rc;
  }
  return launch_k("nms", nms_kernel, dim3(B), dim3(kNmsThreads), 0, st, P);
}

extern "C" int icaf_nms(const void* z, int B, int R, int no, float conf_thres, float iou_thres, int agnostic, uint64_t class_mask,
                        int max_det, float* det, int* count, void* workspace, size_t workspace_bytes, void* stream) {
  return nms_launch(z, B, R, no, conf_thres, iou_thres, agnostic, class_mask, max_det, det, count, workspace, workspace_bytes,
                    stream, false);
}

extern "C" int icaf_nms_multi_label(const void* z, int B, int R, int no, float conf_thres, float iou_thres, int agnostic,
                                    uint64_t class_mask, int max_det, float* det, int* count, void* workspace,
                                    size_t workspace_bytes, void* stream) {
  return nms_launch(z, B, R, no, conf_thres, iou_thres, agnostic, class_mask, max_det, det, count, workspace, workspace_bytes,
                    stream, true);
}

extern "C" int icaf_row_stats(const void* x0, const void* x1, float* stats0, float* stats1, int64_t rows, int C, void* stream) {
  if (!x0 || !stats0 || (x1 && !stats1) || rows < 1 || C < 8 || C % 8) return set_error(ICAF_ERR_BAD_ARG, "row_stats: bad argument");
  dim3 grid(blocks_for(rows, 4), x1 ? 2 : 1);
  return launch_k("row_stats", row_stats_kernel, dim3(grid), dim3(128), 0, (cudaStream_t)stream, (const __half*)x0, (const __half*)x1,
                  (float2*)stats0, (float2*)stats1, (long long)rows, C);
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
