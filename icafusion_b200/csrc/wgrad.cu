// Convolution / linear weight gradient on the Hopper tensor cores (training step, train.py:344 `scaler.scale(loss).backward()`
// -> the wgrad of every nn.Conv2d / nn.Linear of the hot path):
//     dW[n][ky][kx][c] = sum_{b,oy,ox} dY[b,oy,ox,n] * X[b, oy*s - p + ky, ox*s - p + kx, c]
// As a GEMM the reduction runs over PIXELS, so both operands are "MN-major": a tile of 128 pixels x 64 channels arrives by
// one TMA box exactly as it lies in the NHWC tensor (rows = pixels = the K index, channels contiguous) -- no transpose, no
// im2col: the tap shift and the padding are the box coordinates / out-of-bounds zero fill, the stride is the box traversal
// stride, like in the forward kernels.  wgmma reads both operands transposed (MN-major descriptors).
//   CTA work item = (128-wide n tile, <=128-wide c tile, filter tap, split): it walks its share of the 16 x 8 pixel tiles of
//   the output map (one ring stage = dY box(es) + X box(es) of one tile, 8 MMAs of K = 16 pixels each), accumulates
//   D[128 n][c tile] in registers and writes one fp32 partial; wgrad_reduce_kernel sums the splits in a fixed order into the
//   (Cout, Cin, kh, kw) fp32 gradient (deterministic: no atomics).
// 288 threads: warps 0-7 two consumer warpgroups (n rows 0-63 / 64-127 of the tile), warp 8 TMA producer.
// Also here: the fp32 -> fp16 filter packing and the zero-stuffing the training GEMMs consume, and the bias-gradient column sums.
#include <cstring>

#include "icaf_internal.cuh"

namespace icaf {

constexpr int kWStages = 3;
constexpr int kWTile = 128 * 128;                  // one 64-channel block of a 128-pixel tile (128 rows x 128 B)
constexpr int kWStageBytes = 4 * kWTile;           // dY: two 64-n blocks, X: two 64-c blocks
constexpr int kWSmem = kWStages * kWStageBytes + 256 + 1024;

struct WgradParams {
  float* partial;          // [splits][n_pad][taps][c_pad] fp32
  int B, Ho, Wo, Hi, Wi, Cout, Cin, kh, kw, stride, pad;
  int linear;              // 1: 2-D operands (rows x channels), tiles = 128 rows
  int tiles_x, tiles_y, m_tiles, splits, n_tiles, c_tiles, c_tile, c_blk, taps;
  int n_pad, c_pad;
};
struct WgradMaps { CUtensorMap dy; CUtensorMap x; };

// CW = channels of the tile (16, 32, 64 or 128): the N of the wgmma
template <int CW>
__device__ __forceinline__ void wgrad_consume(const WgradParams& P, uint32_t smem_base, uint32_t bar_base, int mt_begin, int mt_end,
                                              int split, int tap, int n0, int c0) {
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (4 + s); };
  const int warp = threadIdx.x >> 5, g = warp >> 2, w = warp & 3, l = threadIdx.x & 31;
  const uint32_t x_row_bytes = uint32_t(P.c_blk) * 2u;      // 128 B, or 64 / 32 B for 32- / 16-channel maps
  const uint32_t x_blk_bytes = 128u * x_row_bytes;
  float acc[CW / 2];
#pragma unroll
  for (int i = 0; i < CW / 2; ++i) acc[i] = 0.f;
  int s = 0;
  uint32_t ph = 0;
  for (int mt = mt_begin; mt < mt_end; ++mt) {
    mbar_wait(full_bar(s), ph);
    const uint32_t sa = smem_base + s * kWStageBytes;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 8; ++k) {                       // 16 pixels per MMA: two 8-row groups of each operand
      const uint64_t ad = gmma_desc_mnmajor(sa + g * kWTile + k * 16 * 128, 128, kWTile);
      const uint64_t bd = gmma_desc_mnmajor(sa + 2 * kWTile + k * 16 * x_row_bytes, x_row_bytes, x_blk_bytes);
      wgmma_ss<1, 1>(acc, ad, bd, true);
    }
    wgmma_commit();
    wgmma_wait<0>();
    if (l == 0) mbar_arrive(empty_bar(s));
    if (++s == kWStages) { s = 0; ph ^= 1; }
  }
  // ---- epilogue: acc[i] is n row 64g + 16w + l/4 + 8*((i>>1)&1), channel 8*(i>>2) + 2*(l&3) + (i&1) ----
#pragma unroll
  for (int i = 0; i < CW / 2; i += 2) {
    const int n = n0 + 64 * g + 16 * w + (l >> 2) + 8 * ((i >> 1) & 1);
    float* dst = P.partial + ((size_t(split) * P.n_pad + n) * P.taps + tap) * P.c_pad + c0 + 8 * (i >> 2) + 2 * (l & 3);
    *reinterpret_cast<float2*>(dst) = make_float2(acc[i], acc[i + 1]);   // an empty split writes zeros
  }
}

__global__ void __launch_bounds__(288, 1) wgrad_kernel(const WgradParams P, const __grid_constant__ WgradMaps maps) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + kWStages * kWStageBytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (4 + s); };

  pdl_launch_dependents();
  const int warp = threadIdx.x >> 5, tid = threadIdx.x;
  // work item
  int w = blockIdx.x;
  const int split = w % P.splits; w /= P.splits;
  const int tap = w % P.taps; w /= P.taps;
  const int ct = w % P.c_tiles;
  const int nt = w / P.c_tiles;
  const int ky = tap / P.kw, kx = tap - ky * P.kw;
  const int n0 = nt * 128, c0 = ct * P.c_tile;
  const int cw = min(P.c_tile, P.Cin - c0);                 // channels of this tile (multiple of c_blk)
  const int n_cblk = (cw + P.c_blk - 1) / P.c_blk;          // X boxes per stage (1 or 2)
  const int mt_begin = int((long long)P.m_tiles * split / P.splits), mt_end = int((long long)P.m_tiles * (split + 1) / P.splits);

  if (tid == 0) {
    for (int s = 0; s < kWStages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 8); }   // 8 consumer warps
    fence_mbar_init();
  }
  if (warp == 8 && lane_id() == 0) { tma_prefetch_desc(&maps.dy); tma_prefetch_desc(&maps.x); }
  __syncthreads();
  pdl_wait();
  const uint32_t x_row_bytes = uint32_t(P.c_blk) * 2u;
  const uint32_t x_blk_bytes = 128u * x_row_bytes;

  if (warp == 8) {
    if (lane_id() == 0) {
      int s = 0;
      uint32_t ph = 0;
      const uint32_t bytes = 2u * kWTile + uint32_t(n_cblk) * x_blk_bytes;
      for (int mt = mt_begin; mt < mt_end; ++mt) {
        mbar_wait(empty_bar(s), ph ^ 1);
        const uint32_t sa = smem_base + s * kWStageBytes;
        mbar_arrive_expect_tx(full_bar(s), bytes);
        if (P.linear) {
          for (int j = 0; j < 2; ++j) tma_load_2d(sa + j * kWTile, &maps.dy, full_bar(s), n0 + j * 64, mt * 128);
          for (int j = 0; j < n_cblk; ++j) tma_load_2d(sa + 2 * kWTile + j * x_blk_bytes, &maps.x, full_bar(s), c0 + j * P.c_blk, mt * 128);
        } else {
          const int per_img = P.tiles_x * P.tiles_y;
          const int b = mt / per_img, r = mt - b * per_img;
          const int oy0 = (r / P.tiles_x) * 16, ox0 = (r % P.tiles_x) * 8;
          for (int j = 0; j < 2; ++j) tma_load_4d(sa + j * kWTile, &maps.dy, full_bar(s), n0 + j * 64, ox0, oy0, b);
          for (int j = 0; j < n_cblk; ++j)
            tma_load_4d(sa + 2 * kWTile + j * x_blk_bytes, &maps.x, full_bar(s), c0 + j * P.c_blk, ox0 * P.stride - P.pad + kx,
                        oy0 * P.stride - P.pad + ky, b);
        }
        if (++s == kWStages) { s = 0; ph ^= 1; }
      }
    }
  } else {
    switch (cw) {      // multiples of c_blk: 128 / 64 for 64-channel blocks, else the whole (16 / 32 channel) map
      case 128: wgrad_consume<128>(P, smem_base, bar_base, mt_begin, mt_end, split, tap, n0, c0); break;
      case 64: wgrad_consume<64>(P, smem_base, bar_base, mt_begin, mt_end, split, tap, n0, c0); break;
      case 32: wgrad_consume<32>(P, smem_base, bar_base, mt_begin, mt_end, split, tap, n0, c0); break;
      default: wgrad_consume<16>(P, smem_base, bar_base, mt_begin, mt_end, split, tap, n0, c0); break;
    }
  }
}

// dW[n][c][ky][kx] (PyTorch layout, fp32) = (accumulate ? dW : 0) + scale * sum_split partial[split][n][tap][c]
// One block per (n, 128-channel tile): partials are read tap-major (coalesced over c), transposed through shared memory, and
// written as the contiguous [c][tap] run of dW -- both sides of the layout change stay coalesced.
constexpr int kRedC = 128;
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const float* __restrict__ partial, float* __restrict__ dw, int splits, int n_pad, int taps, int c_pad,
                                                           int Cout, int Cin, float scale, int accumulate) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float tile[];                          // [taps][kRedC + 1]
  const int c_tiles = (Cin + kRedC - 1) / kRedC;
  const int n = blockIdx.x / c_tiles, c0 = (blockIdx.x % c_tiles) * kRedC;
  const int cw = min(kRedC, Cin - c0);
  for (int i = threadIdx.x; i < taps * cw; i += 256) {
    const int tap = i / cw, c = i - tap * cw;
    const float* src = partial + (size_t(n) * taps + tap) * c_pad + c0 + c;
    const size_t step = size_t(n_pad) * taps * c_pad;
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;            // four independent chains (loads in flight), combined in a fixed order
    int sp = 0;
    for (; sp + 4 <= splits; sp += 4) {
      s0 += __ldg(src + sp * step); s1 += __ldg(src + (sp + 1) * step); s2 += __ldg(src + (sp + 2) * step); s3 += __ldg(src + (sp + 3) * step);
    }
    for (; sp < splits; ++sp) s0 += __ldg(src + sp * step);
    tile[tap * (kRedC + 1) + c] = (s0 + s1) + (s2 + s3);
  }
  __syncthreads();
  float* d = dw + (size_t(n) * Cin + c0) * taps;
  for (int o = threadIdx.x; o < taps * cw; o += 256) {
    const int c = o / taps, tap = o - c * taps;
    const float v = scale * tile[tap * (kRedC + 1) + c];
    d[o] = accumulate ? d[o] + v : v;
  }
}

// 1x1 filters: the two layouts coincide, one thread per element
__global__ void __launch_bounds__(256) wgrad_reduce_flat_kernel(const float* __restrict__ partial, float* __restrict__ dw, int splits, int n_pad, int c_pad, int Cout,
                                                                int Cin, float scale, int accumulate) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = blockIdx.x * 256ll + threadIdx.x;
  if (i >= (long long)Cout * Cin) return;
  const int c = int(i % Cin), n = int(i / Cin);
  const float* src = partial + size_t(n) * c_pad + c;
  const size_t step = size_t(n_pad) * c_pad;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  int sp = 0;
  for (; sp + 4 <= splits; sp += 4) {
    s0 += __ldg(src + sp * step); s1 += __ldg(src + (sp + 1) * step); s2 += __ldg(src + (sp + 2) * step); s3 += __ldg(src + (sp + 3) * step);
  }
  for (; sp < splits; ++sp) s0 += __ldg(src + sp * step);
  dw[i] = (accumulate ? dw[i] : 0.f) + scale * ((s0 + s1) + (s2 + s3));
}

// zero-stuffed copy: y[b, 2*oy, 2*ox, :] = x[b, oy, ox, :], every other pixel 0 (dgrad of a stride-2 convolution = stride-1
// convolution of the zero-stuffed output gradient with the flipped filter)
__global__ void zero_stuff2_kernel(const __half* __restrict__ x, __half* __restrict__ y, int B, int H, int W, int C8, int H2, int W2) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long total = (long long)B * H2 * W2 * C8;
  if (i >= total) return;
  const int c = int(i % C8);
  long long p = i / C8;
  const int ox = int(p % W2);
  p /= W2;
  const int oy = int(p % H2), b = int(p / H2);
  uint4 v = make_uint4(0, 0, 0, 0);
  if (!(oy & 1) && !(ox & 1) && (oy >> 1) < H && (ox >> 1) < W)
    v = __ldg(reinterpret_cast<const uint4*>(x + ((size_t(b) * H + (oy >> 1)) * W + (ox >> 1)) * (C8 * 8) + c * 8));
  *reinterpret_cast<uint4*>(y + i * 8) = v;
}

// column sums of a (rows, C) fp16 matrix in fp32 (bias gradients): fixed chunks per block, fixed-order second stage
__global__ void colsum_partial_kernel(const __half* __restrict__ x, float* __restrict__ part, long long rows, int C, int chunks) {
  pdl_launch_dependents();
  pdl_wait();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const long long per = (rows + chunks - 1) / chunks;
  const long long r0 = blockIdx.y * per, r1 = min(r0 + per, rows);
  float s = 0.f;
  for (long long r = r0; r < r1; ++r) s += __half2float(x[r * C + c]);
  part[size_t(blockIdx.y) * C + c] = s;
}
__global__ void colsum_final_kernel(const float* __restrict__ part, float* __restrict__ out, int C, int chunks, float scale, int accumulate) {
  pdl_launch_dependents();
  pdl_wait();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float s = 0.f;
  for (int k = 0; k < chunks; ++k) s += part[size_t(k) * C + c];
  out[c] = (accumulate ? out[c] : 0.f) + scale * s;
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

struct WgradPlan { WgradParams P; int grid; size_t ws_bytes; };

static int plan_wgrad(const icaf_conv_geom* g, int sms, WgradPlan& pl) {
  WgradParams& P = pl.P;
  memset(&P, 0, sizeof(P));
  if (!g || g->Cin % 16 || g->Cout % 8 || g->stride < 1 || g->stride > 2) return set_error(ICAF_ERR_UNSUPPORTED, "wgrad: Cin % 16, Cout % 8, stride 1 or 2");
  P.B = g->B; P.Ho = g->Ho; P.Wo = g->Wo; P.Hi = g->Hi; P.Wi = g->Wi; P.Cout = g->Cout; P.Cin = g->Cin;
  P.kh = g->kh; P.kw = g->kw; P.stride = g->stride; P.pad = g->pad; P.taps = g->kh * g->kw;
  P.linear = (g->kh == 1 && g->kw == 1 && g->stride == 1 && g->pad == 0) ? 1 : 0;
  if (P.linear) {
    const long long rows = (long long)g->B * g->Ho * g->Wo;
    P.m_tiles = int((rows + 127) / 128);
  } else {
    P.tiles_x = (g->Wo + 7) / 8; P.tiles_y = (g->Ho + 15) / 16;
    P.m_tiles = g->B * P.tiles_x * P.tiles_y;
  }
  P.c_blk = g->Cin % 64 == 0 ? 64 : (g->Cin % 32 == 0 ? 32 : 16);
  if (P.c_blk < 64 && g->Cin != P.c_blk) return set_error(ICAF_ERR_UNSUPPORTED, "wgrad: Cin must be 16, 32 or a multiple of 64");
  P.c_tile = P.c_blk == 64 ? 128 : P.c_blk;
  P.c_tiles = (g->Cin + P.c_tile - 1) / P.c_tile;
  P.n_tiles = (g->Cout + 127) / 128;
  P.n_pad = P.n_tiles * 128; P.c_pad = P.c_tiles * P.c_tile;
  const long long items = (long long)P.n_tiles * P.c_tiles * P.taps;
  // one CTA per SM is resident (192 KB of staging): the grid must not spill a few CTAs into an extra wave -> floor, not ceil
  long long splits = (2LL * sms) / items;
  if (splits > P.m_tiles) splits = P.m_tiles;
  if (splits < 1) splits = 1;
  if (splits > 64) splits = 64;
  P.splits = int(splits);
  pl.grid = int(items * splits);
  pl.ws_bytes = size_t(P.splits) * P.n_pad * P.taps * P.c_pad * sizeof(float);
  return ICAF_OK;
}

}  // namespace icaf

using namespace icaf;

extern "C" size_t icaf_conv2d_wgrad_workspace_bytes(const icaf_conv_geom* g) {
  WgradPlan pl;
  if (plan_wgrad(g, sm_count_cached(), pl)) return 0;
  return pl.ws_bytes;
}

extern "C" int icaf_conv2d_wgrad(const icaf_conv_geom* g, const void* x, int64_t x_ld, const void* dy, int64_t dy_ld, float* dw, float scale,
                                 int accumulate, void* workspace, size_t workspace_bytes, void* stream) {
  if (!g || !x || !dy || !dw || !workspace) return set_error(ICAF_ERR_BAD_ARG, "wgrad: null pointer");
  WgradPlan pl;
  if (int rc = plan_wgrad(g, sm_count_cached(), pl)) return rc;
  if (workspace_bytes < pl.ws_bytes || (reinterpret_cast<uintptr_t>(workspace) & 15)) return set_error(ICAF_ERR_BAD_ARG, "wgrad: workspace too small or misaligned");
  if (x_ld % 8 || dy_ld % 8 || (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(dy) & 15))
    return set_error(ICAF_ERR_BAD_ARG, "wgrad: operands must be 16-byte aligned views");
  WgradParams& P = pl.P;
  P.partial = (float*)workspace;
  WgradMaps maps;
  memset(&maps, 0, sizeof(maps));
  int rc;
  if (P.linear) {
    const uint64_t rows = uint64_t(g->B) * g->Ho * g->Wo;
    rc = encode_tmap_2d(&maps.dy, dy, uint64_t(g->Cout), rows, uint64_t(dy_ld) * 2, 64, 128);
    if (!rc) rc = encode_tmap_2d(&maps.x, x, uint64_t(g->Cin), rows, uint64_t(x_ld) * 2, uint32_t(P.c_blk), 128);
  } else {
    rc = encode_tmap_nhwc(&maps.dy, dy, g->Cout, g->Wo, g->Ho, g->B, dy_ld, 64, 8, 16, 1, 1);
    if (!rc) rc = encode_tmap_nhwc(&maps.x, x, g->Cin, g->Wi, g->Hi, g->B, x_ld, uint32_t(P.c_blk), 8 * g->stride, 16 * g->stride, g->stride, g->stride);
  }
  if (rc) return rc;
  static bool configured[kMaxDevices] = {false};
  if (int r2 = configure_smem(wgrad_kernel, kWSmem, configured, "wgrad: cudaFuncSetAttribute")) return r2;
  cudaStream_t st = (cudaStream_t)stream;
  if (int r3 = launch_k("conv2d_wgrad", wgrad_kernel, dim3(pl.grid), dim3(288), (size_t)kWSmem, st, P, maps)) return r3;
  if (P.taps == 1) {
    return launch_k("conv2d_wgrad(reduce)", wgrad_reduce_flat_kernel, dim3(blocks_for((long long)g->Cout * g->Cin, 256)), dim3(256), 0, st,
                    (const float*)P.partial, dw, P.splits, P.n_pad, P.c_pad, g->Cout, g->Cin, scale, accumulate);
  }
  const unsigned red_blocks = (unsigned)g->Cout * (unsigned)((g->Cin + kRedC - 1) / kRedC);
  return launch_k("conv2d_wgrad(reduce)", wgrad_reduce_kernel, dim3(red_blocks), dim3(256), size_t(P.taps) * (kRedC + 1) * sizeof(float), st,
                  (const float*)P.partial, dw, P.splits, P.n_pad, P.taps, P.c_pad, g->Cout, g->Cin, scale, accumulate);
}

extern "C" int icaf_zero_stuff2(const void* x, void* y, int B, int H, int W, int C, int H2, int W2, void* stream) {
  if (!x || !y || C % 8 || B < 1 || H2 < 2 * H - 1 || W2 < 2 * W - 1) return set_error(ICAF_ERR_BAD_ARG, "zero_stuff2: bad argument");
  const long long total = (long long)B * H2 * W2 * (C / 8);
  return launch_k("zero_stuff2", zero_stuff2_kernel, dim3(blocks_for(total, 256)), dim3(256), 0, (cudaStream_t)stream, (const __half*)x, (__half*)y,
                  B, H, W, C / 8, H2, W2);
}

extern "C" int icaf_colsum(const void* x, int64_t rows, int C, float* out, float scale, int accumulate, float* workspace, size_t workspace_bytes,
                           void* stream) {
  constexpr int kChunks = 64;
  if (!x || !out || !workspace || rows < 1 || C < 1) return set_error(ICAF_ERR_BAD_ARG, "colsum: bad argument");
  if (workspace_bytes < size_t(kChunks) * C * sizeof(float)) return set_error(ICAF_ERR_BAD_ARG, "colsum: workspace needs 64 * C floats");
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = launch_k("colsum(partial)", colsum_partial_kernel, dim3(blocks_for(C, 128), kChunks), dim3(128), 0, st, (const __half*)x, workspace,
                        (long long)rows, C, kChunks)) return rc;
  return launch_k("colsum", colsum_final_kernel, dim3(blocks_for(C, 128)), dim3(128), 0, st, (const float*)workspace, out, C, kChunks, scale,
                  accumulate);
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
