// Shared pieces of the implicit-GEMM conv kernels (conv_gemm.cu): problem descriptors, TMA descriptor bundle, tile origin,
// and the epilogues (staged rows: row set-up, load, chunk dispatch; accumulator registers: row bias, fragments into an
// output tile, its TMA store and the residual tile's TMA load).
#pragma once
#include "icaf_internal.cuh"

namespace icaf {

constexpr int BM = 128;
constexpr int BK = 64;              // 64 halfs = one 128-byte swizzle atom row
constexpr int kLag = 2;             // cp.async groups kept in flight per gather thread
constexpr int kThreads = 288;     // epilogue / gather warpgroup, consumer warpgroup, TMA warp

enum AMode { A_GATHER = 0, A_TMA2D = 1, A_TMA4D = 2 };

struct ConvProblem {
  const __half* x; const float* bias; const __half* res; __half* y;
  const float* alpha; const float* beta;
  long long x_ld, res_ld, y_ld;
  const float2* ln_stats;   // LN fold: (sum, sum of squares) partials of every INPUT row, [M][ln_parts]
  const float* ln_s;        // LN fold: column sums of the gamma-folded filter, fp32 [Cout]
  float2* stats_out;        // EMIT_STATS: (sum, sum of squares) partials of every OUTPUT row, [M][ceil(N/32)]
};
struct ConvParams {
  ConvProblem p[2];
  int M, N, K, k_pad;
  int B, Hi, Wi, Cin, Ho, Wo, kh, kw, stride, pad;
  int act, epi;
  int a_mode, tw, th, tiles_x, tiles_y;   // A_TMA4D: tile = th x tw output pixels (tw*th <= 128), tiles per image
  int stages;                             // smem ring depth (runtime: deep rings for small grids, 2 CTAs/SM for BN <= 64)
  int splits;                             // split-K factor = cluster size along x (1 = no cluster); partial sums meet in DSMEM
  int cblk;                               // A_TMA4D: channels per TMA box (64)
  int ln_parts;                           // LN fold: partials per input row (0 = no fold)
  float ln_eps, ln_inv_k;                 // LN fold: epsilon, 1 / (normalised features = K)
  int m_tiles, n_tiles, tiles;            // persistent kernel: tile grid (m, n, problem) and its product
  int tma_epi;                            // register epilogue + TMA-stored output tile (else staged rows), set by plan_conv
  int halo_bytes;                         // persistent stride-1 3x3: bytes of one input-halo slot (0: a shifted box per tap)
};
struct ConvMaps {          // TMA descriptors, passed by value as a __grid_constant__ kernel parameter
  CUtensorMap w[2];
  CUtensorMap a[2];
  CUtensorMap y[2];        // register epilogue (both kernels): output (and residual) tiles, 64-column boxes
  CUtensorMap res[2];
};

__device__ __forceinline__ ConvProblem pick_problem(const ConvParams& P, unsigned z) {
  ConvProblem r;
  r.x = z ? P.p[1].x : P.p[0].x;          r.bias = z ? P.p[1].bias : P.p[0].bias;
  r.res = z ? P.p[1].res : P.p[0].res;    r.y = z ? P.p[1].y : P.p[0].y;
  r.alpha = z ? P.p[1].alpha : P.p[0].alpha; r.beta = z ? P.p[1].beta : P.p[0].beta;
  r.x_ld = z ? P.p[1].x_ld : P.p[0].x_ld; r.res_ld = z ? P.p[1].res_ld : P.p[0].res_ld;
  r.y_ld = z ? P.p[1].y_ld : P.p[0].y_ld;
  r.ln_stats = z ? P.p[1].ln_stats : P.p[0].ln_stats; r.ln_s = z ? P.p[1].ln_s : P.p[0].ln_s;
  r.stats_out = z ? P.p[1].stats_out : P.p[0].stats_out;
  return r;
}

// Origin of an output tile: linear rows from m0 (gather / 2-D), or a th x tw patch at (oy0, ox0) of image tb (4-D).
struct TileOrigin { int m0, tb, oy0, ox0; };
// The origin of m-tile `mtile`, into four scalars rather than a TileOrigin: the one-tile kernel keeps them apart, and
// ptxas allocates its registers differently when they start out as one struct.
__device__ __forceinline__ void tile_origin(const ConvParams& P, int mtile, int& m0, int& tb, int& oy0, int& ox0) {
  m0 = mtile * BM; tb = 0; oy0 = 0; ox0 = 0;
  if (P.a_mode == A_TMA4D) {
    const int per_img = P.tiles_x * P.tiles_y;
    m0 = 0;
    tb = mtile / per_img;
    const int t = mtile - tb * per_img;
    oy0 = (t / P.tiles_x) * P.th;
    ox0 = (t % P.tiles_x) * P.tw;
  }
}

// Tile row -> output row m; valid: inside the output (4-D: tw divides Wo; the last tile row of an image may hang over).
__device__ __forceinline__ void tile_row(const ConvParams& P, const TileOrigin& o, int row, int& m, bool& valid) {
  if (P.a_mode == A_TMA4D) {
    const int ry = row / P.tw, rx = row - ry * P.tw;
    m = (o.tb * P.Ho + o.oy0 + ry) * P.Wo + o.ox0 + rx;
    valid = ry < P.th && o.oy0 + ry < P.Ho;
  } else {
    m = o.m0 + row;
    valid = m < P.M;
  }
}

// Per-row extras of an epilogue thread.  XM = 1 (LayerNorm folded into this GEMM, common.py:660,665,749-750): the filter
// carries gamma, the bias carries beta . W, and the row is normalised after the fact:
//     LN(x) . W^T + b  =  rstd * (x . W'^T  -  mean * s)  +  b'          W' = W diag(gamma), s_n = sum_k W'[n][k]
// XM = 2 (EMIT_STATS): sum and sum of squares of the fp16-rounded outputs of this row, for the LN fold of the NEXT GEMM.
struct EpiRow {
  float ln_a, ln_mu;     // rstd, mean of this thread's input row
  const float* ln_s;     // s, offset to the first column of the current pass
  float sum, sumsq;
};
__device__ __forceinline__ void epi_row_ln(EpiRow& ex, const ConvParams& P, const ConvProblem& pr, int m, bool mvalid) {
  float su = 0.f, sq = 0.f;
  if (mvalid) {
    const float2* sp = pr.ln_stats + size_t(m) * P.ln_parts;
    for (int i = 0; i < P.ln_parts; ++i) { const float2 v = __ldg(sp + i); su += v.x; sq += v.y; }
  }
  const float mu = su * P.ln_inv_k;
  ex.ln_mu = mu;
  ex.ln_a = rsqrtf(fmaxf(sq * P.ln_inv_k - mu * mu, 0.f) + P.ln_eps);
}

// The output row of an epilogue thread that owns tile row `row` (staged-row epilogue): output row m (mvalid: inside the
// output), its row bias (ICAF_EPI_BIAS_ROW), output and residual row pointers, and the XM extras.  Everything here is
// independent of the main loop, so it is set up (and the residual row prefetched into L2) while the main loop still runs.
struct StagedRow {
  int m;
  bool mvalid;
  float rbias;
  __half* yrow;
  const __half* rrow;
  EpiRow ex;
};
template <int BN, bool XM>
__device__ __forceinline__ void staged_row(StagedRow& r, const ConvParams& P, const ConvProblem& pr, const TileOrigin& o, int row, int n0) {
  tile_row(P, o, row, r.m, r.mvalid);
  r.rbias = ((P.epi & ICAF_EPI_BIAS_ROW) && pr.bias && r.mvalid) ? __ldg(pr.bias + r.m) : 0.f;
  r.yrow = pr.y + size_t(r.mvalid ? r.m : 0) * pr.y_ld;
  r.rrow = pr.res ? pr.res + size_t(r.mvalid ? r.m : 0) * pr.res_ld : nullptr;
  if (r.rrow && r.mvalid) {
    for (int cb = 0; cb < BN && n0 + cb < P.N; cb += 64) prefetch_l2(r.rrow + n0 + cb);   // 128-byte lines of the residual row
  }
  r.ex.sum = r.ex.sumsq = 0.f; r.ex.ln_a = 1.f; r.ex.ln_mu = 0.f; r.ex.ln_s = nullptr;
  if (XM) {
    r.ex.ln_s = pr.ln_s ? pr.ln_s + n0 : nullptr;
    if (P.ln_parts > 0) epi_row_ln(r.ex, P, pr, r.m, r.mvalid);   // row statistics
  }
}

// slots [n_begin/32, n_end/32) of this row's partials: the first one carries the sums, the others zero
__device__ __forceinline__ void epi_row_emit(const EpiRow& ex, const ConvParams& P, const ConvProblem& pr, int m, int n_begin, int n_end) {
  const int slots = (P.N + 31) >> 5;
  float2* sp = pr.stats_out + size_t(m) * slots;
  const int s0 = n_begin >> 5, s1 = min((n_end + 31) >> 5, slots);
  for (int i = s0; i < s1; ++i) sp[i] = i == s0 ? make_float2(ex.sum, ex.sumsq) : make_float2(0.f, 0.f);
}

// One output element before its fp16 rounding: accumulator a + column bias b + row bias, activation, residual rf.
// ACT: 0 none, 1 SiLU, 2 GELU(erf).  RES: 0 none, 1 y = act(v) + res, 2 y = alpha*res + beta*v.
// Both epilogues (epi_chunk on staged rows, epi_fragments on the accumulator registers) compute every element with it,
// so they round identically.
template <int ACT, int RES>
__device__ __forceinline__ float epi_value(float a, float b, float rbias, float rf, float alpha, float beta) {
  float t = a + b + rbias;
  if (ACT == ICAF_ACT_SILU) t = silu_f(t);
  if (ACT == ICAF_ACT_GELU) t = gelu_erf_f(t);
  if (RES == 1) t = t + rf;
  if (RES == 2) t = alpha * rf + beta * t;
  return t;
}

// One 32-column chunk of one output row: + bias, activation, residual, fp16 store (see epi_value).
template <int ACT, int RES, int XM = 0>
__device__ __forceinline__ void epi_chunk(const uint32_t (&acc)[32], const float* __restrict__ sb, float rbias,
                                          float alpha, float beta, const __half* __restrict__ rp,
                                          __half* __restrict__ yp, bool vec, int ncols, EpiRow& ex, int cb, bool do_store = true) {
  auto f = [&](int j, float rf) {
    float a = __uint_as_float(acc[j]);
    if (XM == 1) a = ex.ln_a * (a - ex.ln_mu * __ldg(ex.ln_s + cb + j));
    return epi_value<ACT, RES>(a, sb[j], rbias, rf, alpha, beta);
  };
  if (vec) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      float rf[8];
      if (RES != 0) {
        uint4 rr = *reinterpret_cast<const uint4*>(rp + q * 8);
        const __half2* rh = reinterpret_cast<const __half2*>(&rr);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 r2 = __half22float2(rh[e]);
          rf[2 * e] = r2.x; rf[2 * e + 1] = r2.y;
        }
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) rf[e] = 0.f;
      }
      float v[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = f(q * 8 + e, rf[e]);
      uint4 o;
      o.x = pack_half2(v[0], v[1]); o.y = pack_half2(v[2], v[3]);
      o.z = pack_half2(v[4], v[5]); o.w = pack_half2(v[6], v[7]);
      if (XM == 2) {
        const __half2* oh = reinterpret_cast<const __half2*>(&o);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 w = __half22float2(oh[e]);
          ex.sum += w.x + w.y;
          ex.sumsq += w.x * w.x + w.y * w.y;
        }
      }
      if (do_store) *reinterpret_cast<uint4*>(yp + q * 8) = o;
    }
  } else {
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      if (j < ncols) {
        const float t = f(j, RES != 0 ? __half2float(rp[j]) : 0.f);
        const __half h = __float2half_rn(t);
        if (XM == 2) { const float w = __half2float(h); ex.sum += w; ex.sumsq += w * w; }
        yp[j] = h;
      }
    }
  }
}

// 32 staged fp32 accumulators of one row (16-byte aligned) as the bit patterns epi_chunk takes
__device__ __forceinline__ void load_staged(uint32_t (&acc)[32], const float* p) {
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const float4 v = *reinterpret_cast<const float4*>(p + 4 * q);
    acc[4 * q] = __float_as_uint(v.x); acc[4 * q + 1] = __float_as_uint(v.y);
    acc[4 * q + 2] = __float_as_uint(v.z); acc[4 * q + 3] = __float_as_uint(v.w);
  }
}

// One chunk through the epi_chunk specialisation of the row's mode.  The activation / residual mode is warp-uniform, so
// it is dispatched once per chunk to straight-line code.  mode_act = 3 * ACT + RES; XM: 9 / 10 = LayerNorm folded into
// this GEMM (no activation / GELU), 11 = scaled residual + statistics of the output rows.
template <bool XM>
__device__ __forceinline__ void epi_dispatch(int mode_act, const uint32_t (&acc)[32], const float* sb, float rbias, float alpha,
                                             float beta, const __half* rp, __half* yp, bool vec, int ncols, EpiRow& ex, int cb) {
  if (XM) {
    switch (mode_act) {
      case 9: epi_chunk<0, 0, 1>(acc, sb, rbias, alpha, beta, rp, yp, vec, ncols, ex, cb); break;
      case 10: epi_chunk<2, 0, 1>(acc, sb, rbias, alpha, beta, rp, yp, vec, ncols, ex, cb); break;
      default: epi_chunk<0, 2, 2>(acc, sb, rbias, alpha, beta, rp, yp, vec, ncols, ex, cb); break;
    }
  } else {
    switch (mode_act) {
      case 0: epi_chunk<0, 0>(acc, sb, rbias, alpha, beta, rp, yp, vec, ncols, ex, cb); break;
      case 1: epi_chunk<0, 1>(acc, sb, rbias, alpha, beta, rp, yp, vec, ncols, ex, cb); break;
      case 2: epi_chunk<0, 2>(acc, sb, rbias, alpha, beta, rp, yp, vec, ncols, ex, cb); break;
      case 3: epi_chunk<1, 0>(acc, sb, rbias, alpha, beta, rp, yp, vec, ncols, ex, cb); break;
      case 4: epi_chunk<1, 1>(acc, sb, rbias, alpha, beta, rp, yp, vec, ncols, ex, cb); break;
      case 5: epi_chunk<1, 2>(acc, sb, rbias, alpha, beta, rp, yp, vec, ncols, ex, cb); break;
      case 6: epi_chunk<2, 0>(acc, sb, rbias, alpha, beta, rp, yp, vec, ncols, ex, cb); break;
      case 7: epi_chunk<2, 1>(acc, sb, rbias, alpha, beta, rp, yp, vec, ncols, ex, cb); break;
      default: epi_chunk<2, 2>(acc, sb, rbias, alpha, beta, rp, yp, vec, ncols, ex, cb); break;
    }
  }
}

// The launch's mode_act (see epi_dispatch) for both epilogues: 3 * ACT + RES (has_res: the launch adds a residual), or
// the XM modes.
template <bool XM>
__device__ __forceinline__ int epi_mode_act(const ConvParams& P, bool has_res) {
  if (XM) return P.ln_parts > 0 ? (P.act == ICAF_ACT_GELU ? 10 : 9) : 11;
  return P.act * 3 + ((P.epi & ICAF_EPI_SCALED_RES) ? 2 : (has_res ? 1 : 0));
}

// Staged-row epilogue of tile columns [cb, cb + 32) of row r, output columns from nb = n0 + cb < N: the 32 staged
// accumulators acc, sbias = the tile's column bias.  16-byte vectors when all 32 columns are inside the output and aligned.
template <bool XM>
__device__ __forceinline__ void epi_staged_chunk(int mode_act, const uint32_t (&acc)[32], StagedRow& r, const float* sbias,
                                                 float alpha, float beta, int cb, int nb, int N) {
  const int ncols = min(32, N - nb);
  const bool vec = ncols == 32 && ((reinterpret_cast<uintptr_t>(r.yrow + nb) & 15) == 0) &&
                   (!r.rrow || (reinterpret_cast<uintptr_t>(r.rrow + nb) & 15) == 0);
  epi_dispatch<XM>(mode_act, acc, sbias + cb, r.rbias, alpha, beta, r.rrow ? r.rrow + nb : nullptr, r.yrow + nb, vec, ncols,
                   r.ex, cb);
}

// ---------------------------------------------------------------------------------------------------
// Epilogue on the accumulator registers of a consumer warpgroup (tile rows 0-63 in acc0, 64-127 in acc1, NA = BN / 2 each),
// written as fp16 into an output tile of 64-column halves: 128 rows of 128 bytes each, 128B-swizzled (the layout of a TMA
// box of 64 columns x 128 rows, or of tw x th pixels), the halves kOutHalfBytes apart.  One thread then stores each half
// with a TMA store, which clips the rows and columns outside the output.
constexpr int kOutHalfBytes = BM * 64 * 2;

// columns [16 PP, 16 PP + 16) of the warpgroup's accumulators: v[0..7] from rows 0-63 (acc0), v[8..15] from rows 64-127
template <int PP, int NA>
__device__ __forceinline__ void take_cols16(const float (&acc0)[NA], const float (&acc1)[NA], float (&v)[16]) {
  constexpr int Q = PP < NA / 8 ? PP : NA / 8 - 1;   // the groups past a narrow tile are never taken
#pragma unroll
  for (int e = 0; e < 8; ++e) { v[e] = acc0[8 * Q + e]; v[8 + e] = acc1[8 * Q + e]; }
}

// Epilogue of 16 columns (take_cols16) on the accumulator registers: epi_value per element, fp16 pairs into the output
// tile with stmatrix.  Register pair k of v[8h ...] is tile row 16w + l/4 + 8 (k % 2) + 64h, columns 8 (k / 2) + 2 (l % 4)
// (+0, +1) of the 16: exactly one register of matrix k of an m8n8.x4 stmatrix.  sa: this lane's stmatrix row address for
// rows 0-63 (rows 64-127 are 8 KB further); RES != 0 reads the residual pairs from the same place with ldmatrix first.
// sb: column bias at the lane's column 2 (l % 4); rb: row bias of the lane's rows l/4 + {0, 8, 64, 72}.
template <int ACT, int RES>
__device__ __forceinline__ void epi_fragments(const float (&v)[16], uint32_t sa, const float* sb, const float (&rb)[4],
                                              float alpha, float beta) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    uint32_t r[4];
    if (RES != 0) ldmatrix_x4(r, sa + 8192u * h);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 b = *reinterpret_cast<const float2*>(sb + 8 * (k >> 1));
      const float rbias = rb[2 * h + (k & 1)];
      float2 rf = make_float2(0.f, 0.f);
      if (RES != 0) rf = __half22float2(*reinterpret_cast<const __half2*>(&r[k]));
      r[k] = pack_half2(epi_value<ACT, RES>(v[8 * h + 2 * k], b.x, rbias, rf.x, alpha, beta),
                        epi_value<ACT, RES>(v[8 * h + 2 * k + 1], b.y, rbias, rf.y, alpha, beta));
    }
    stmatrix_x4(sa + 8192u * h, r);
  }
}

// mode_act = 3 * ACT + RES, warp-uniform: dispatched once per 16 columns to straight-line code
__device__ __forceinline__ void epi_fragments_dispatch(int mode_act, const float (&v)[16], uint32_t sa, const float* sb,
                                                       const float (&rb)[4], float alpha, float beta) {
  switch (mode_act) {
    case 0: epi_fragments<0, 0>(v, sa, sb, rb, alpha, beta); break;
    case 1: epi_fragments<0, 1>(v, sa, sb, rb, alpha, beta); break;
    case 2: epi_fragments<0, 2>(v, sa, sb, rb, alpha, beta); break;
    case 3: epi_fragments<1, 0>(v, sa, sb, rb, alpha, beta); break;
    case 4: epi_fragments<1, 1>(v, sa, sb, rb, alpha, beta); break;
    case 5: epi_fragments<1, 2>(v, sa, sb, rb, alpha, beta); break;
    case 6: epi_fragments<2, 0>(v, sa, sb, rb, alpha, beta); break;
    case 7: epi_fragments<2, 1>(v, sa, sb, rb, alpha, beta); break;
    default: epi_fragments<2, 2>(v, sa, sb, rb, alpha, beta); break;
  }
}

// The whole tile, 16 columns at a time: sout = the output tile (1024-byte aligned), sbias = the tile's column bias,
// w / l = warp of the warpgroup / lane.
template <int NA>
__device__ __forceinline__ void epi_tile_fragments(int mode_act, const float (&acc0)[NA], const float (&acc1)[NA], uint32_t sout,
                                                   const float* sbias, const float (&rb)[4], float alpha, float beta, int w, int l) {
  const uint32_t sa = sout + uint32_t(16 * w + (l & 7) + 8 * ((l >> 3) & 1)) * 128u;   // stmatrix row of this lane
  const float* sb = sbias + 2 * (l & 3);
#pragma unroll 1
  for (int p = 0; p < NA / 8; ++p) {
    float v[16];
    switch (p) {
      case 0: take_cols16<0>(acc0, acc1, v); break;
      case 1: take_cols16<1>(acc0, acc1, v); break;
      case 2: take_cols16<2>(acc0, acc1, v); break;
      case 3: take_cols16<3>(acc0, acc1, v); break;
      case 4: take_cols16<4>(acc0, acc1, v); break;
      case 5: take_cols16<5>(acc0, acc1, v); break;
      case 6: take_cols16<6>(acc0, acc1, v); break;
      default: take_cols16<7>(acc0, acc1, v); break;
    }
    // half p / 4 of the tile; 16-byte chunk 2 (p % 4) + l / 16 of the 128-byte row, 128B-swizzled by the row
    const uint32_t a = sa + uint32_t(p >> 2) * uint32_t(kOutHalfBytes) + (uint32_t((2 * (p & 3) + (l >> 4)) ^ (l & 7)) << 4);
    epi_fragments_dispatch(mode_act, v, a, sb + 16 * p, rb, alpha, beta);
  }
}

// rb of epi_tile_fragments (zero-initialised by the caller): the row bias (ICAF_EPI_BIAS_ROW) of this lane's accumulator
// rows l/4 + {0, 8, 64, 72} of warp w
__device__ __forceinline__ void fragment_row_bias(float (&rb)[4], const ConvParams& P, const ConvProblem& pr, const TileOrigin& o,
                                                  int w, int l) {
  if ((P.epi & ICAF_EPI_BIAS_ROW) && pr.bias) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      int mq;
      bool vq;
      tile_row(P, o, 16 * w + (l >> 2) + 8 * (q & 1) + 64 * (q >> 1), mq, vq);
      rb[q] = vq ? __ldg(pr.bias + mq) : 0.f;
    }
  }
}

// The 64-column halves of a BN-wide tile from column n0 that lie inside the output, each one TMA box of the output or
// residual map: 128 rows from m0 (2-D map: A_TMA2D and A_GATHER launches) or the tw x th patch (4-D map: A_TMA4D).  In
// shared memory the halves are kOutHalfBytes apart from `s`.  The store commits one bulk group; the load completes on `bar`.
template <int BN>
__device__ __forceinline__ void tma_store_tile(const ConvParams& P, const CUtensorMap* map, uint32_t s, int n0, const TileOrigin& o) {
  const int halves = (BN == 128 && n0 + 64 < P.N) ? 2 : 1;
  for (int hh = 0; hh < halves; ++hh) {
    const uint32_t src = s + uint32_t(hh * kOutHalfBytes);
    if (P.a_mode == A_TMA4D) tma_store_4d(map, src, n0 + 64 * hh, o.ox0, o.oy0, o.tb);
    else tma_store_2d(map, src, n0 + 64 * hh, o.m0);
  }
  bulk_commit_group();
}

template <int BN>
__device__ __forceinline__ void tma_load_tile(const ConvParams& P, const CUtensorMap* map, uint32_t s, uint32_t bar, int n0,
                                              const TileOrigin& o) {
  const int halves = (BN == 128 && n0 + 64 < P.N) ? 2 : 1;
  const uint32_t half_bytes = P.a_mode == A_TMA4D ? uint32_t(P.tw * P.th) * 128u : uint32_t(kOutHalfBytes);
  mbar_arrive_expect_tx(bar, uint32_t(halves) * half_bytes);
  for (int hh = 0; hh < halves; ++hh) {
    const uint32_t dst = s + uint32_t(hh * kOutHalfBytes);
    if (P.a_mode == A_TMA4D) tma_load_4d(dst, map, bar, n0 + 64 * hh, o.ox0, o.oy0, o.tb);
    else tma_load_2d(dst, map, bar, n0 + 64 * hh, o.m0);
  }
}

// Host-side launch plan: everything the dispatcher decides before it touches CUDA.  icaf_conv2d_plan (host only, no
// device needed) exposes it so that a CPU test can walk every layer geometry through the dispatcher's invariants.
struct ConvPlan {
  int kernel;                     // ICAF_KERNEL_TC
  int bn;                         // output-channel tile width
  unsigned grid_x, grid_y, grid_z, cluster;
  int smem;                       // dynamic shared memory per CTA (bytes)
  int tiles, m_tiles, n_tiles;    // output tiles of the launch (icaf_conv_plan.work_items) = m_tiles * n_tiles * problems
  int sms;                        // SM count the plan was made for
  bool persist;                   // conv_gemm_persist_kernel: `ctas` CTAs walk the grid_x * grid_y * grid_z tiles
  bool stem;                      // conv_stem_kernel: one tile per CTA, 16-channel 3x3 stride-1 gather launches at BN = 64
  bool xm;                        // LayerNorm-fold / row-statistics epilogue: the XM instantiation of either kernel
  int ctas;                       // CTAs the launch starts
};

}  // namespace icaf
