// Fused Bottleneck (models/common.py:184-194 with shortcut, Cin = C_ = 64, BN folded):
//
//   y = x + SiLU(conv3x3(h) + b2),   h = SiLU(conv1x1(x) + b1)        fp16 maps, fp32 accumulation
//
// The two-launch path (conv_gemm.cu: cv1, then cv2 with the residual in its epilogue) writes h to HBM and reads it back,
// and reads x twice.  Here the hidden map never leaves the SM: each output patch of 4 x 32 pixels recomputes h on its
// (6 x 34)-pixel halo from the x halo in shared memory, and the residual comes from the centre of that same halo.
//
// bottleneck_kernel: one persistent CTA per SM; CTA k of problem z (z = blockIdx.x % n_io) walks the patches k, k + G, ...
// of problem z (G = CTAs per problem).  384 threads:
//   warpgroup 0    : TMA producer (one elected thread): both filters once, then the x halo of every patch
//   warpgroups 1, 2: consumers; warpgroup 1 + (j % 2) owns the CTA's j-th patch, so one consumer's epilogues run while
//                    the other's MMAs do.  Per patch:
//     phase 1  the 1x1 over the 204 halo pixels: wgmma SS (A = x halo, 128B-swizzled by TMA; B = resident W1) on four
//              64-row blocks (rows 0, 64, 128, 144: the last two overlap so that no block reads past the 208-row buffer);
//              + b1, SiLU, fp16 (epi_value, so h rounds exactly as cv1's output does), 0 for halo pixels outside the image
//              (the 3x3 pads h, and SiLU(b1) != 0), into an unswizzled h patch of kHPitch-byte rows
//     then     the x halo centre is copied into the consumer's output tile as the residual tile (128B-swizzled, the
//              layout of the 4-D TMA box of the patch) and the x buffer is handed back, so the next halo load overlaps
//              phase 2
//     phase 2  the 3x3: 9 taps x 64 channels, K order tap-major as pack_conv_weight lays it out (k = tap * 64 + channel),
//              wgmma RS with A fragments from the h patch by ldmatrix (output pixel (r, c) reads h pixel (r + ky, c + kx))
//              and B = resident W3
//     epilogue + b2, SiLU, + residual on the accumulator registers, in place in the output tile (epi_value at the
//              stmatrix addressing of epi_fragments, as the one-tile conv kernel runs it), one 4-D TMA store that clips
//              the patch at the map's right and bottom edges
// Both epilogues are bound by the latency of their SiLU chains (two consumer warps per SM sub-partition), so each
// computes all 64 values of a thread before it stores any.
// The MMAs run in the order cv1 and cv2 of the two-launch path run theirs (4 K steps; 9 taps x 4 K steps on one
// accumulator), so the outputs are bit-identical to it.
#include <cstring>

#include "conv_common.cuh"

namespace icaf {
namespace {

constexpr int kThreadsBn = 384;
constexpr int kC = 64;                          // input, hidden and output channels
constexpr int kPH = 4, kPW = 32;                // output patch: 4 rows x 32 columns = 128 pixels
constexpr int kHaloH = kPH + 2, kHaloW = kPW + 2;
constexpr int kHaloPix = kHaloH * kHaloW;       // 204
constexpr int kHPitch = 144;                    // bytes per h pixel: 128 + 16 spreads 8 consecutive pixels over all banks
constexpr int kFilterTile = kC * kC * 2;        // one 64 x 64 fp16 filter box (8 KB)
// Registers: ptxas gives each of the 384 threads 168; the producer warpgroup hands its surplus to the consumers, and the
// CTA's total must stay what it was launched with (setmaxnreg.inc waits for registers that would never come free).
constexpr int kRegsProducer = 40, kRegsConsumer = 232;
static_assert(128 * kRegsProducer + 256 * kRegsConsumer == kThreadsBn * 168, "register rebalance exceeds the launch budget");

struct BnLayout {                               // byte offsets from the 1024-aligned base
  static constexpr int kW1 = 0;
  static constexpr int kW3 = kW1 + kFilterTile;                              // 9 taps
  static constexpr int kXBytes = 208 * 128;                                  // 204 halo rows (+4 that phase 1 reads past)
  static constexpr int kX = kW3 + 9 * kFilterTile;                           // per consumer
  static constexpr int kHBytes = (kHaloPix * kHPitch + 1023) / 1024 * 1024;
  static constexpr int kH = kX + 2 * kXBytes;                                // h patch, per consumer
  static constexpr int kOut = kH + 2 * kHBytes;                              // output tile, per consumer
  static constexpr int kBias = kOut + 2 * kOutHalfBytes;                     // b1[64] | b2[64] fp32
  static constexpr int kBar = kBias + 2 * kC * 4;
  static constexpr int kTotal = kBar + 64 + 1024;                            // + alignment slack
  static_assert(kX % 1024 == 0 && kXBytes % 1024 == 0 && kOut % 1024 == 0, "swizzled tiles need 1024-byte alignment");
  static_assert(kTotal <= 227 * 1024, "shared memory");
};

struct BnParams {
  const float* b1[2];
  const float* b2[2];
  int H, W, tiles_x, patches_per_img, patches;  // patches per problem
  int n_io;
};
struct BnMaps {
  CUtensorMap w1[2], w3[2], x[2], y[2];
};

__device__ __forceinline__ void patch_origin(const BnParams& P, int p, int& b, int& oy0, int& ox0) {
  b = p / P.patches_per_img;
  const int t = p - b * P.patches_per_img;
  const int ty = t / P.tiles_x;
  oy0 = ty * kPH;
  ox0 = (t - ty * P.tiles_x) * kPW;
}

__device__ __forceinline__ void st_shared_u32(uint32_t a, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}

// Phase-1 epilogue of two 64-row accumulator blocks, from halo rows r0 (a0) and r1 (a1): + b1, SiLU, fp16, 0 for halo
// pixels outside the image, into the h patch.  Rows of a1 below r1_min (computed by a0 already) and past the halo are
// not stored.  Every value is computed before any store, without branches, so that the 64 SiLU chains of a thread
// overlap.  Accumulator layout: see ptx.cuh.
__device__ __forceinline__ void epi_hidden(const float (&a0)[32], const float (&a1)[32], int r0, int r1, int r1_min, uint32_t sh,
                                           const float* sb1, int oy0, int ox0, int H, int W, int w, int l) {
  float2 b[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) b[j] = *reinterpret_cast<const float2*>(sb1 + 8 * j + 2 * (l & 3));
  uint32_t v[4][8];                            // [2 * block + hh][j]
  auto pack_row = [&](const float (&a)[32], int hh, uint32_t (&o)[8]) {
#pragma unroll
    for (int j = 0; j < 8; ++j)
      o[j] = pack_half2(epi_value<ICAF_ACT_SILU, 0>(a[4 * j + 2 * hh], b[j].x, 0.f, 0.f, 0.f, 1.f),
                        epi_value<ICAF_ACT_SILU, 0>(a[4 * j + 2 * hh + 1], b[j].y, 0.f, 0.f, 0.f, 1.f));
  };
  pack_row(a0, 0, v[0]);
  pack_row(a0, 1, v[1]);
  pack_row(a1, 0, v[2]);
  pack_row(a1, 1, v[3]);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int row = (q < 2 ? r0 : r1) + 16 * w + (l >> 2) + 8 * (q & 1);
    const int hy = row / kHaloW, hx = row - hy * kHaloW;
    const int iy = oy0 - 1 + hy, ix = ox0 - 1 + hx;
    const bool inside = (unsigned)iy < (unsigned)H && (unsigned)ix < (unsigned)W;
    const uint32_t dst = sh + uint32_t(row * kHPitch) + 4u * (l & 3);
    if (row >= (q < 2 ? 0 : r1_min) && row < kHaloPix) {
#pragma unroll
      for (int j = 0; j < 8; ++j) st_shared_u32(dst + 16u * j, inside ? v[q][j] : 0u);
    }
  }
}

// Epilogue of the 3x3: + b2, SiLU, + residual (the residual tile in sout, overwritten in place), per element the
// epi_value of epi_fragments (conv_common.cuh) at its stmatrix addressing, so the tile rounds exactly as the one-tile
// conv kernel's.  All residual fragments are loaded first and all results stored last, so that the 64 SiLU chains of a
// thread overlap.
__device__ __forceinline__ void epi_out(const float (&acc0)[32], const float (&acc1)[32], uint32_t sout, const float* sb2, int w,
                                        int l) {
  const uint32_t sa = sout + uint32_t(16 * w + (l & 7) + 8 * ((l >> 3) & 1)) * 128u;   // stmatrix row of this lane
  const float* sb = sb2 + 2 * (l & 3);
  uint32_t r[4][2][4];                         // [16-column group p][rows 64 h ...][matrix k]
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int h = 0; h < 2; ++h) ldmatrix_x4(r[p][h], sa + 8192u * h + (uint32_t((2 * p + (l >> 4)) ^ (l & 7)) << 4));
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 b = *reinterpret_cast<const float2*>(sb + 16 * p + 8 * (k >> 1));
      const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&r[p][0][k]));
      const float2 f1 = __half22float2(*reinterpret_cast<const __half2*>(&r[p][1][k]));
      r[p][0][k] = pack_half2(epi_value<ICAF_ACT_SILU, 1>(acc0[8 * p + 2 * k], b.x, 0.f, f0.x, 0.f, 1.f),
                              epi_value<ICAF_ACT_SILU, 1>(acc0[8 * p + 2 * k + 1], b.y, 0.f, f0.y, 0.f, 1.f));
      r[p][1][k] = pack_half2(epi_value<ICAF_ACT_SILU, 1>(acc1[8 * p + 2 * k], b.x, 0.f, f1.x, 0.f, 1.f),
                              epi_value<ICAF_ACT_SILU, 1>(acc1[8 * p + 2 * k + 1], b.y, 0.f, f1.y, 0.f, 1.f));
    }
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int h = 0; h < 2; ++h) stmatrix_x4(sa + 8192u * h + (uint32_t((2 * p + (l >> 4)) ^ (l & 7)) << 4), r[p][h]);
}

// The residual tile: output pixel m = 32 r + c of the patch is halo pixel (r + 1, c + 1).  Both tiles are 128B-swizzled
// (16-byte chunk k of row m sits at chunk k ^ (m % 8)); thread t copies chunks t, t + 128, ...
__device__ __forceinline__ void copy_residual(uint32_t sout, uint32_t sx, int t) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int e = t + 128 * i, m = e >> 3, k = e & 7;
    const int hp = ((m >> 5) + 1) * kHaloW + (m & 31) + 1;
    uint32_t v0, v1, v2, v3;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v0), "=r"(v1), "=r"(v2), "=r"(v3)
                 : "r"(sx + uint32_t(hp * 128) + (uint32_t(k ^ (hp & 7)) << 4)) : "memory");
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(sout + uint32_t(m * 128) + (uint32_t(k ^ (m & 7)) << 4)),
                 "r"(v0), "r"(v1), "r"(v2), "r"(v3) : "memory");
  }
}

__global__ void __launch_bounds__(kThreadsBn, 1) bottleneck_kernel(const BnParams P, const __grid_constant__ BnMaps maps) {
  extern __shared__ uint8_t smem_raw[];
  using L = BnLayout;
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* gen = smem_raw + (base - smem_u32(smem_raw));
  const uint32_t bar = base + L::kBar;
  const uint32_t w_bar = bar;                                      // both filters resident
  auto full_bar = [&](int c) { return bar + 8u + 8u * c; };        // consumer c's x halo has landed
  auto empty_bar = [&](int c) { return bar + 24u + 8u * c; };      // consumer c has read its x halo
  float* sb = reinterpret_cast<float*>(gen + L::kBias);

  pdl_launch_dependents();
  const int tid = threadIdx.x;
  const int wg = tid >> 7;
  const int z = int(blockIdx.x) % P.n_io;
  const int per = int(gridDim.x) / P.n_io;                         // CTAs per problem
  const int k0 = int(blockIdx.x) / P.n_io;
  if (tid == 0) {
    mbar_init(w_bar, 1);
    for (int c = 0; c < 2; ++c) { mbar_init(full_bar(c), 1); mbar_init(empty_bar(c), 4); }   // one arrival per consumer warp
    fence_mbar_init();
  }
  const CUtensorMap* mx = z ? &maps.x[1] : &maps.x[0];
  const CUtensorMap* my = z ? &maps.y[1] : &maps.y[0];
  if (tid == 32) {
    tma_prefetch_desc(mx);
    tma_prefetch_desc(my);
  }
  __syncthreads();
  pdl_wait();   // prologue (barriers, descriptor prefetch) overlapped the previous kernel
  if (tid < 2 * kC) sb[tid] = __ldg(tid < kC ? (z ? P.b1[1] : P.b1[0]) + tid : (z ? P.b2[1] : P.b2[0]) + tid - kC);
  __syncthreads();

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer (warp 0, one thread)
    setmaxnreg_dec<kRegsProducer>();
    if (tid < 32 && elect_one()) {
      mbar_arrive_expect_tx(w_bar, 10u * kFilterTile);
      tma_load_2d(base + L::kW1, z ? &maps.w1[1] : &maps.w1[0], w_bar, 0, 0);
      for (int t = 0; t < 9; ++t) tma_load_2d(base + L::kW3 + t * kFilterTile, z ? &maps.w3[1] : &maps.w3[0], w_bar, t * kC, 0);
      for (int j = 0, p = k0; p < P.patches; ++j, p += per) {
        const int c = j & 1;
        mbar_wait_quiet(empty_bar(c), (uint32_t(j >> 1) & 1u) ^ 1u);
        int b, oy0, ox0;
        patch_origin(P, p, b, oy0, ox0);
        mbar_arrive_expect_tx(full_bar(c), uint32_t(kHaloPix * 128));
        tma_load_4d(base + L::kX + c * L::kXBytes, mx, full_bar(c), 0, ox0 - 1, oy0 - 1, b);
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroups
  setmaxnreg_inc<kRegsConsumer>();
  const int c = wg - 1;
  const int t = tid & 127, w = t >> 5, l = t & 31;
  const int bar_id = 2 + c;                                        // warpgroup-local named barrier
  const uint32_t sx = base + L::kX + c * L::kXBytes;
  const uint32_t sh = base + L::kH + c * L::kHBytes;
  const uint32_t sout = base + L::kOut + c * kOutHalfBytes;
  const uint32_t sw1 = base + L::kW1, sw3 = base + L::kW3;
  // ldmatrix row address of this lane in the h patch for accumulator block hm (tile rows 64 hm ...), tap (0, 0): matrix
  // q = l / 8 of the x4 covers tile rows 8 (q % 2) ... and channels 8 (q / 2) ... of the 16-channel K step
  uint32_t lane_h[2];
#pragma unroll
  for (int hm = 0; hm < 2; ++hm) {
    const int q = l >> 3;
    const int m = 64 * hm + 16 * w + (l & 7) + 8 * (q & 1);
    lane_h[hm] = sh + uint32_t(((m >> 5) * kHaloW + (m & 31)) * kHPitch + 16 * (q >> 1));
  }
  mbar_wait_quiet(w_bar, 0);

  int j = c;
  for (int p = k0 + c * per; p < P.patches; p += 2 * per, j += 2) {
    const int u = j >> 1;                                          // ordinal of the patch among this consumer's
    int b, oy0, ox0;
    patch_origin(P, p, b, oy0, ox0);
    if (t == 0) bulk_wait_group_read<0>();                         // the previous output tile has been read out
    named_bar_sync(bar_id, 128);                                   // (and every warp is done with the previous h patch)
    mbar_wait_quiet(full_bar(c), uint32_t(u) & 1u);

    // ---- phase 1: h = SiLU(x W1^T + b1) on the halo, two 64-row blocks at a time
    float acc0[32], acc1[32];
#pragma unroll
    for (int pass = 0; pass < 2; ++pass) {
      const int r0 = pass ? 128 : 0, r1 = pass ? 144 : 64;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint64_t bd = gmma_desc_sw128(sw1 + 32 * k);
        wgmma_ss<0, 0>(acc0, gmma_desc_sw128(sx + r0 * 128 + 32 * k), bd, k != 0);
        wgmma_ss<0, 0>(acc1, gmma_desc_sw128(sx + r1 * 128 + 32 * k), bd, k != 0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      epi_hidden(acc0, acc1, r0, r1, pass ? 192 : 0, sh, sb, oy0, ox0, P.H, P.W, w, l);
    }
    copy_residual(sout, sx, t);
    __syncwarp();
    if (l == 0) mbar_arrive(empty_bar(c));                         // x halo read: the producer may refill it
    named_bar_sync(bar_id, 128);                                   // the h patch and the residual tile are complete

    // ---- phase 2: the 3x3 over h, one (tap, 64-row block) group of four K steps at a time; the fragments of group g + 1
    // are loaded while group g runs (group g - 1, which used the same registers, has retired)
    uint32_t fa[2][4][4];
#pragma unroll
    for (int g = 0; g < 18; ++g) {
      const int tap = g >> 1, hm = g & 1;
      const uint32_t a0 = lane_h[hm] + uint32_t(((tap / 3) * kHaloW + tap % 3) * kHPitch);
#pragma unroll
      for (int kc = 0; kc < 4; ++kc) ldmatrix_x4(fa[g & 1][kc], a0 + 32u * kc);
      wgmma_fence();
#pragma unroll
      for (int kc = 0; kc < 4; ++kc) {
        const uint64_t bd = gmma_desc_sw128(sw3 + tap * kFilterTile + 32 * kc);
        if (hm == 0) wgmma_rs<0>(acc0, fa[g & 1][kc], bd, (tap | kc) != 0);
        else wgmma_rs<0>(acc1, fa[g & 1][kc], bd, (tap | kc) != 0);
      }
      wgmma_commit();
      wgmma_wait<1>();
    }
    wgmma_wait<0>();

    // ---- epilogue: + b2, SiLU, + x in place in the output tile, TMA store clipped to the map
    epi_out(acc0, acc1, sout, sb + kC, w, l);
    fence_proxy_async_smem();                                      // the tile is visible to the TMA unit ...
    named_bar_sync(bar_id, 128);                                   // ... once every thread of the warpgroup has written its part
    if (t == 0) {
      tma_store_4d(my, sout, 0, ox0, oy0, b);
      bulk_commit_group();
    }
  }
  if (t == 0) bulk_wait_group<0>();                                // complete before the grid is (PDL dependents read it)
}

// [x, x + extent) of an NHWC view
bool views_overlap(const void* a, long long a_ld, const void* b, long long b_ld, long long pixels) {
  const uintptr_t a0 = reinterpret_cast<uintptr_t>(a), b0 = reinterpret_cast<uintptr_t>(b);
  const uintptr_t a1 = a0 + uintptr_t(((pixels - 1) * a_ld + kC) * 2), b1 = b0 + uintptr_t(((pixels - 1) * b_ld + kC) * 2);
  return a0 < b1 && b0 < a1;
}

}  // namespace
}  // namespace icaf

using namespace icaf;

extern "C" int icaf_bottleneck_fwd(int B, int H, int W, const icaf_bottleneck_io* io, int n_io, void* stream) {
  if (!io || n_io < 1 || n_io > 2) return set_error(ICAF_ERR_BAD_ARG, "bottleneck: need 1 or 2 problems");
  const long long pixels = (long long)B * H * W;
  if (B < 1 || H < 1 || W < 1 || pixels > 0x7fffffffLL) return set_error(ICAF_ERR_BAD_ARG, "bottleneck: size out of range");
  BnParams P;
  memset(&P, 0, sizeof(P));
  BnMaps maps;
  memset(&maps, 0, sizeof(maps));
  for (int i = 0; i < n_io; ++i) {
    const icaf_bottleneck_io& s = io[i];
    if (!s.x || !s.w1 || !s.b1 || !s.w3 || !s.b2 || !s.y) return set_error(ICAF_ERR_BAD_ARG, "bottleneck: null pointer");
    if ((reinterpret_cast<uintptr_t>(s.x) | reinterpret_cast<uintptr_t>(s.y) | reinterpret_cast<uintptr_t>(s.w1) |
         reinterpret_cast<uintptr_t>(s.w3)) & 15 || s.x_ld % 8 || s.y_ld % 8 || s.x_ld < kC || s.y_ld < kC)
      return set_error(ICAF_ERR_BAD_ARG, "bottleneck: x / y / filters must be 16-byte aligned, pixel pitches multiples of 8 and >= 64");
    for (int k = 0; k < n_io; ++k)
      if (views_overlap(s.y, s.y_ld, io[k].x, io[k].x_ld, pixels))
        return set_error(ICAF_ERR_BAD_ARG, "bottleneck: the output must not overlap an input (patches read x halos other CTAs overwrite)");
    P.b1[i] = s.b1;
    P.b2[i] = s.b2;
    int rc = encode_tmap_2d(&maps.w1[i], s.w1, kC, kC, kC * 2, kC, kC);
    if (!rc) rc = encode_tmap_2d(&maps.w3[i], s.w3, 9 * kC, kC, 9 * kC * 2, kC, kC);
    if (!rc) rc = encode_tmap_nhwc(&maps.x[i], s.x, kC, W, H, B, s.x_ld, kC, kHaloW, kHaloH, 1, 1);
    if (!rc) rc = encode_tmap_nhwc(&maps.y[i], s.y, kC, W, H, B, s.y_ld, kC, kPW, kPH, 1, 1);
    if (rc) return rc;
  }
  P.H = H; P.W = W;
  P.tiles_x = (W + kPW - 1) / kPW;
  P.patches_per_img = P.tiles_x * ((H + kPH - 1) / kPH);
  P.patches = B * P.patches_per_img;
  P.n_io = n_io;
  // one CTA per SM, split evenly between the problems (each CTA keeps one problem's filters resident)
  int per = sm_count_cached() / n_io;
  if (per > (P.patches + 1) / 2) per = (P.patches + 1) / 2;
  if (per < 1) per = 1;
  static bool configured[kMaxDevices] = {};
  if (int rc = configure_smem(bottleneck_kernel, BnLayout::kTotal, configured, "bottleneck: cudaFuncSetAttribute")) return rc;
  return launch_k("bottleneck_fwd", bottleneck_kernel, dim3(unsigned(per * n_io)), dim3(kThreadsBn), size_t(BnLayout::kTotal), (cudaStream_t)stream,
                  P, maps);
}
