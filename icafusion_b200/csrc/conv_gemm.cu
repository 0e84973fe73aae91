// Implicit-GEMM Conv(+folded BN)+bias+activation(+residual) / Linear on the Hopper tensor cores (wgmma).
//
//   C[M=B*Ho*Wo, N=Cout] = A[M, K=kh*kw*Cin] * W[N, K]^T           fp16 operands, fp32 accumulate in registers
//
// A is never materialised (no im2col).  Three ways to stage the A tile (128 rows x 64 K) into the 128B-swizzled
// K-major shared-memory layout the wgmma descriptors expect, picked per layer on the host:
//   A_TMA2D  : 1x1 conv / linear -- A is a plain [M][Cin] matrix: one 2-D TMA box per stage.
//   A_TMA4D  : kxk conv whose 128-row tile is a TH x TW patch of one image and Cin % 64 == 0: one 4-D TMA box
//              (64 ch, TW*s, TH*s, 1) of the NHWC input per stage at coordinates shifted by the filter tap;
//              out-of-bounds (= padding) is zero-filled by the TMA unit, the stride is the box traversal stride.
//   A_GATHER : anything else (Cin = 4 / 8 / 16 / 32 / odd multiples of 8): producer warps gather 16-byte channel runs
//              with cp.async (zero-fill), 4 rows x 128 B per warp instruction.
// The filter tile (BN rows x 64 K) always arrives by 2-D TMA.
// conv_gemm_tc_kernel: CTA = one 128 x BN output tile (BN = 32 / 64 / 128), 288 threads:
//   warps 0-3 : A_GATHER producers, then (staged-row epilogue) the epilogue: thread t owns output row t
//   warps 4-7 : one consumer warpgroup: two m64nBNk16 wgmma per 16 K (rows 0-63, 64-127), accumulators in registers;
//               then either the register epilogue (as in the persistent kernel) into an idle ring stage and a TMA store,
//               or the accumulators as fp32 rows into the idle ring for warps 0-3
//   warp  8   : TMA producer (one elected thread); with the register epilogue also the residual tile's TMA load
// Pipelines: smem ring full[]/empty[] (producers <-> consumer), named barrier (staged accumulator -> epilogue).  Small
// tiles (BN <= 64) let two CTAs share an SM so that one CTA's epilogue overlaps the other's main loop.  Split-K: the
// CTAs of a cluster take a K range each; the leader adds the others' staged tiles through distributed shared memory.
// The register epilogue serves BN >= 64 launches that are not XM or split-K and whose output TMA can write; the others
// keep the staged rows.  plan_conv makes that choice for both kernels (ConvParams::tma_epi).
// conv_gemm_persist_kernel: BN = 128 grids of more than one wave with TMA-staged A -- one persistent CTA per SM, a TMA
// producer warpgroup and two consumer warpgroups that take turns on the main loop; each consumer runs the epilogue on its
// accumulator registers and writes the tile with TMA stores (see its own comment below).  Its stride-1 3x3 launches
// (pad 1, A_TMA4D) stage A differently: one (64 ch, tw+2, th+2) input halo per 64-channel block feeds all nine taps, with
// the A fragments read from it by ldmatrix (wgmma RS, halo_mma_loop), instead of nine shifted boxes that each bring the
// same pixels in again from L2.
// The two kernels share the TMA producer stage (load_stage), the main loop (mma_loop), the tile origin, the per-element
// epilogue expression (epi_value), so they compute bit-identical tiles (the halo launches sum K in another order: equal up
// to fp32 summation order), and every other epilogue piece (conv_common.cuh):
// register epilogue (fragment_row_bias, epi_tile_fragments, tma_store_tile, tma_load_tile), staged rows (staged_row,
// epi_staged_chunk) and the mode selection (epi_mode_act).
// conv_stem_kernel: the gather launches with 16 input channels, 3x3, stride 1, pad 1 and BN = 64 (the yolov5m/l image
// stems over the space-to-depth frame): one 128-row tile per CTA as above, but its input pixels are gathered once into a
// halo that feeds all nine taps, and only the nine k16 steps that carry data are issued (see its own comment below).
#include <cstdlib>
#include <cstring>

#include "conv_common.cuh"

namespace icaf {

constexpr int kMaxStages = 10;
template <int BN>
struct SmemLayout {
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kPitch = BN + 4;                       // floats per staged accumulator row (spreads rows over banks)
  static constexpr int kAccBytes = BM * kPitch * 4;
  // [ring: stages x (A|B), at least the staged accumulator] [barriers 256 B] [bias BN fp32] ; + 1024 B alignment slack
  static constexpr int kTailBytes = 256 + BN * 4 + 1024;
  __host__ __device__ static int region(int stages) { return stages * kStageBytes > kAccBytes ? stages * kStageBytes : kAccBytes; }
  static int total(int stages) { return region(stages) + kTailBytes; }
};

// ---------------------------------------------------------------------------------------------------
// Producer and main-loop pieces of both wgmma kernels (the epilogue pieces are in conv_common.cuh).

// TMA producer, one K block `kb` of the tile into the ring stage at `sa`: the filter box (BN rows from n0) and, unless the
// gather producers fill A, the A box -- 2-D rows from m0, or the 4-D box of the tile's patch shifted by the block's filter
// tap.  kTmaA: the launch never gathers A, so an A that is not 2-D is 4-D.
template <int BN, bool kTmaA>
__device__ __forceinline__ void load_stage(const ConvParams& P, int a_mode, uint32_t sa, uint32_t bar, uint32_t bytes,
                                           const CUtensorMap* mw, const CUtensorMap* ma, int kb, int n0, const TileOrigin& o) {
  mbar_arrive_expect_tx(bar, bytes);
  tma_load_2d(sa + SmemLayout<BN>::kABytes, mw, bar, kb * BK, n0);
  if (a_mode == A_TMA2D) {
    tma_load_2d(sa, ma, bar, kb * BK, o.m0);
  } else if (kTmaA || a_mode == A_TMA4D) {
    const int k0 = kb * BK;
    const int tap = k0 / P.Cin;
    const int ch = k0 - tap * P.Cin;
    const int ky = tap / P.kw, kx = tap - ky * P.kw;
    tma_load_4d(sa, ma, bar, ch, o.ox0 * P.stride - P.pad + kx, o.oy0 * P.stride - P.pad + ky, o.tb);
  }
}

// Consumer warpgroup main loop over the tile's nkb K blocks, from ring stage s0 at phase ph0: per stage, wait for it to
// fill, issue two m64nBNk16 wgmma per 16 K (tile rows 0-63 into acc0, 64-127 into acc1), then hand back the previous
// stage, whose MMAs are done once this stage's are the only ones in flight.  Returns the last stage, which is still in
// use until the caller's final wgmma_wait.  It waits without the printf report (see mbar_wait_quiet), and so do the
// producers of both kernels: a printf reachable anywhere in the kernel makes ptxas serialise every wgmma (warning C7510).
template <int BN, class FullBar, class HandBack>
__device__ __forceinline__ int mma_loop(float (&acc0)[BN / 2], float (&acc1)[BN / 2], uint32_t smem_base, int kStages, int nkb,
                                        int s0, uint32_t ph0, FullBar full_bar, HandBack hand_back) {
  int s = s0, s_prev = s0;
  uint32_t ph = ph0;
  for (int kb = 0; kb < nkb; ++kb) {
    mbar_wait_quiet(full_bar(s), ph);
    const uint32_t sa = smem_base + s * SmemLayout<BN>::kStageBytes;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) {
      const uint64_t bd = gmma_desc_sw128(sa + SmemLayout<BN>::kABytes + 32 * k);
      wgmma_ss<0, 0>(acc0, gmma_desc_sw128(sa + 32 * k), bd, (kb | k) != 0);
      wgmma_ss<0, 0>(acc1, gmma_desc_sw128(sa + 64 * 128 + 32 * k), bd, (kb | k) != 0);
    }
    wgmma_commit();
    wgmma_wait<1>();
    if (kb > 0) hand_back(s_prev);
    s_prev = s;
    if (++s == kStages) { s = 0; ph ^= 1; }
  }
  return s_prev;
}

// Register budget of the BN <= 64 instantiations (two CTAs per SM: 96 registers per thread at launch).  Warps 0-3 give
// some to the consumer warpgroup, whose epilogue runs on its accumulators; warp 8 (not a whole warpgroup) keeps the launch
// count, so the CTA's total stays 288 x 96.  BN = 64 XM keeps 96 everywhere: its consumer only stages rows, and the row
// epilogue of warps 0-3 needs them.  (ptxas -v: no spills in any instantiation with this split.)
constexpr int kRegsLow = 80, kRegsHigh = 112;
static_assert(128 * kRegsLow + 128 * kRegsHigh + 32 * 96 <= kThreads * 96, "register rebalance exceeds the launch budget");
template <int BN, bool XM>
__host__ __device__ constexpr bool rebalance_regs() { return BN == 32 || (BN == 64 && !XM); }

// XM: the LayerNorm-fold / row-statistics epilogues (DMFF linears) live in their own instantiation so that the epilogue
// of every other layer stays small (the hot loops are instruction-cache sensitive).
template <int BN, bool XM>
__global__ void __launch_bounds__(kThreads, (BN <= 64 ? 2 : 1))
conv_gemm_tc_kernel(const ConvParams P, const __grid_constant__ ConvMaps maps) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  using L = SmemLayout<BN>;
  const int kStages = P.stages;
  const uint32_t bar_off = uint32_t(L::region(kStages));
  const uint32_t bar_base = smem_base + bar_off;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (kMaxStages + s); };
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));

  pdl_launch_dependents();
  const int warp = threadIdx.x >> 5;
  const int tid = threadIdx.x;
  // split-K: the `splits` CTAs of a cluster (consecutive blockIdx.x) share one output tile and take a K range each
  const int splits = P.splits;
  const int mtile = splits > 1 ? blockIdx.x / splits : blockIdx.x;
  const int ntile = blockIdx.y, bz = blockIdx.z;
  const ConvProblem pr = pick_problem(P, bz);           // by value: a dynamic param index would spill to local
  const int n0 = ntile * BN;
  const int a_mode = P.a_mode;
  const uint32_t crank = splits > 1 ? cluster_ctarank() : 0u;
  const int nkb_all = P.k_pad / BK;
  const int kb_begin = (nkb_all * int(crank)) / splits;
  const int nkb = (nkb_all * (int(crank) + 1)) / splits - kb_begin;
  int m0, tb, oy0, ox0;
  tile_origin(P, mtile, m0, tb, oy0, ox0);
  const TileOrigin o{m0, tb, oy0, ox0};
  // Register epilogue (P.tma_epi, see plan_conv; the XM and BN = 32 instantiations leave its code out): the consumer
  // warpgroup applies the epilogue to its accumulators and stores the tile by TMA from ring stage s_out -- the stage the K
  // block after the last one would take.  It is free once block nkb - stages has been consumed, so a residual tile is
  // TMA-loaded into it (on res_bar) while the last blocks of the main loop still run.
  const bool tma_epi = !XM && BN >= 64 && P.tma_epi != 0;
  const bool has_res = (P.epi & (ICAF_EPI_ADD_RES | ICAF_EPI_SCALED_RES)) != 0;
  const int s_out = nkb % kStages;
  const uint32_t res_bar = bar_base + 8u * (2 * kMaxStages);

  if (tid == 0) {
    const uint32_t nfull = a_mode == A_GATHER ? 129u : 1u;    // 128 gather threads + the TMA thread
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full_bar(s), nfull);
      mbar_init(empty_bar(s), 4);                             // one arrival per consumer warp
    }
    mbar_init(res_bar, 1);
    fence_mbar_init();
  }
  if (warp == 8 && lane_id() == 0) {
    tma_prefetch_desc(bz ? &maps.w[1] : &maps.w[0]);
    if (a_mode != A_GATHER) tma_prefetch_desc(bz ? &maps.a[1] : &maps.a[0]);
    if (tma_epi) {
      tma_prefetch_desc(bz ? &maps.y[1] : &maps.y[0]);
      if (has_res) tma_prefetch_desc(bz ? &maps.res[1] : &maps.res[0]);
    }
  }
  float* sbias = reinterpret_cast<float*>(smem_gen + bar_off + 256);
  float* sacc = reinterpret_cast<float*>(smem_gen);           // staged accumulator [BM][kPitch], reuses the idle ring
  __syncthreads();
  pdl_wait();   // prologue (barriers, descriptor prefetch) overlapped the previous kernel

  if (warp < 4) {
    if constexpr (rebalance_regs<BN, XM>()) setmaxnreg_dec<kRegsLow>();
    // Epilogue operands that do not depend on the main loop are fetched now so their DRAM latency hides behind it:
    // bias slice and (alpha, beta) into registers, this thread's residual row into L2.
    float bias_r[(BN + 127) / 128];
#pragma unroll
    for (int i = 0; i < (BN + 127) / 128; ++i) {
      const int col = tid + 128 * i;
      bias_r[i] = (!tma_epi && col < BN && pr.bias && !(P.epi & ICAF_EPI_BIAS_ROW) && n0 + col < P.N) ? __ldg(pr.bias + n0 + col) : 0.f;
    }
    float alpha = 0.f, beta = 1.f;
    if (!tma_epi && (P.epi & ICAF_EPI_SCALED_RES)) { alpha = __ldg(pr.alpha); beta = __ldg(pr.beta); }
    if (a_mode == A_GATHER) {
      // ---------------------------------------------------------------- cp.async gather producers
      // A stage is handed over once this thread's copies of it have landed and been made visible to the async proxy
      // (wait_group + fence.proxy.async): `lag` stages stay in flight per thread.  The consumer frees stage j only once
      // it holds stage j + 1, so the lag must stay below stages - 1.
      const int lag = kStages - 2 < kLag ? kStages - 2 : kLag;
      const int c = tid & 7;          // 16-byte chunk within the 128-byte K row
      const int r0 = tid >> 3;        // rows r0 + 16*i
      const uint32_t sw = uint32_t(c ^ (r0 & 7)) << 4;
      uint32_t base[8];
      int iy0[8], ix0[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        int m = o.m0 + r0 + 16 * i;
        bool mv = m < P.M;
        int mm = mv ? m : 0;
        int ox = mm % P.Wo;
        int t = mm / P.Wo;
        int oy = t % P.Ho;
        int b = t / P.Ho;
        base[i] = uint32_t(b) * uint32_t(P.Hi * P.Wi);
        iy0[i] = mv ? oy * P.stride - P.pad : -100000;   // invalid rows fall out of bounds -> zero fill
        ix0[i] = ox * P.stride - P.pad;
      }
      int s = 0, s_done = 0;
      uint32_t ph = 0;
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait_quiet(empty_bar(s), ph ^ 1);
        const uint32_t sa = smem_base + s * L::kStageBytes;
        const int k0 = (kb_begin + kb) * BK + c * 8;
        const bool kvalid = k0 < P.K;
        const int tap = k0 / P.Cin;
        const int ch = k0 - tap * P.Cin;
        const int ky = tap / P.kw;
        const int kx = tap - ky * P.kw;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          int iy = iy0[i] + ky, ix = ix0[i] + kx;
          bool ok = kvalid && (unsigned)iy < (unsigned)P.Hi && (unsigned)ix < (unsigned)P.Wi;
          size_t off = ok ? (size_t(base[i] + uint32_t(iy * P.Wi + ix)) * size_t(pr.x_ld) + ch) : 0;
          cp_async16(sa + uint32_t(r0 + 16 * i) * 128u + sw, pr.x + off, ok);
        }
        cp_async_commit();
        if (kb >= lag) {
          if (lag == 2) cp_async_wait<2>(); else if (lag == 1) cp_async_wait<1>(); else cp_async_wait<0>();
          fence_proxy_async_smem();
          mbar_arrive(full_bar(s_done));
          if (++s_done == kStages) s_done = 0;
        }
        if (++s == kStages) { s = 0; ph ^= 1; }
      }
      cp_async_wait<0>();
      fence_proxy_async_smem();
      for (int kb = nkb - lag < 0 ? 0 : nkb - lag; kb < nkb; ++kb) {
        mbar_arrive(full_bar(s_done));
        if (++s_done == kStages) s_done = 0;
      }
    }
    if (tma_epi) return;                   // the consumer warpgroup runs the epilogue

    // ------------------------------------------------------------------ epilogue
    const int row = tid;                   // staged accumulator row == tile row
    StagedRow sr;
    staged_row<BN, XM>(sr, P, pr, o, row, n0);
#pragma unroll
    for (int i = 0; i < (BN + 127) / 128; ++i)
      if (tid + 128 * i < BN) sbias[tid + 128 * i] = bias_r[i];
    // the staged accumulators (of every CTA of the cluster) and the bias tile are complete
    if (splits > 1) { cluster_arrive(); cluster_wait(); } else { named_bar_sync(1, 256); }
    const int mode_act = epi_mode_act<XM>(P, sr.rrow != nullptr);
    if (crank == 0) {
      const float* arow = sacc + size_t(row) * L::kPitch;
      const uint32_t arow_s = smem_u32(arow);
#pragma unroll 1
      for (int cb = 0; cb < BN; cb += 32) {
        uint32_t acc[32];
        load_staged(acc, arow + cb);
        // ---- split-K reduction: the other CTAs' staged partial tiles, read through distributed shared memory ----
        for (int r = 1; r < splits; ++r) {
          const uint32_t peer = map_to_cta(arow_s, uint32_t(r)) + uint32_t(cb) * 4u;
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            float4 v;
            ld_cluster_v4(peer + 16u * q, v);
            acc[4 * q] = __float_as_uint(__uint_as_float(acc[4 * q]) + v.x);
            acc[4 * q + 1] = __float_as_uint(__uint_as_float(acc[4 * q + 1]) + v.y);
            acc[4 * q + 2] = __float_as_uint(__uint_as_float(acc[4 * q + 2]) + v.z);
            acc[4 * q + 3] = __float_as_uint(__uint_as_float(acc[4 * q + 3]) + v.w);
          }
        }
        if (sr.mvalid && n0 + cb < P.N) epi_staged_chunk<XM>(mode_act, acc, sr, sbias, alpha, beta, cb, n0 + cb, P.N);
      }
      if (XM && mode_act == 11 && sr.mvalid && n0 < P.N) epi_row_emit(sr.ex, P, pr, sr.m, n0, min(n0 + BN, P.N));
    }
    if (splits > 1) { cluster_arrive(); cluster_wait(); }   // the peers' staged tiles stay alive until the leader has read them
  } else if (warp < 8) {
    // ------------------------------------------------------------------ consumer warpgroup (wgmma)
    if constexpr (rebalance_regs<BN, XM>()) setmaxnreg_inc<kRegsHigh>();
    const int t = tid - 128, w = t >> 5, l = t & 31;
    float alpha = 0.f, beta = 1.f;
    float rb[4] = {0.f, 0.f, 0.f, 0.f};      // tma_epi: row bias of the accumulator fragments
    if (tma_epi) {
      // epilogue operands that do not depend on the main loop: bias slice, (alpha, beta), row bias
      if (t < BN) sbias[t] = (pr.bias && !(P.epi & ICAF_EPI_BIAS_ROW) && n0 + t < P.N) ? __ldg(pr.bias + n0 + t) : 0.f;
      if (P.epi & ICAF_EPI_SCALED_RES) { alpha = __ldg(pr.alpha); beta = __ldg(pr.beta); }
      fragment_row_bias(rb, P, pr, o, w, l);
      named_bar_sync(2, 128);                                 // bias slice complete
    }
    float acc0[BN / 2], acc1[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
    mma_loop<BN>(acc0, acc1, smem_base, kStages, nkb, 0, 0u, full_bar,
                 [&](int s) { if (lane_id() == 0) mbar_arrive(empty_bar(s)); });   // one arrival per consumer warp
    wgmma_wait<0>();
    if constexpr (!XM && BN >= 64) {
      if (tma_epi) {
        // ---- epilogue on the accumulator registers into ring stage s_out (every stage is consumed now), TMA store
        const uint32_t sout = smem_base + uint32_t(s_out) * L::kStageBytes;
        if (has_res) mbar_wait_quiet(res_bar, 0);
        epi_tile_fragments<BN / 2>(epi_mode_act<false>(P, has_res), acc0, acc1, sout, sbias, rb, alpha, beta, w, l);
        fence_proxy_async_smem();                             // the tile is visible to the TMA unit ...
        named_bar_sync(2, 128);                               // ... once every thread of the warpgroup has written its part
        if (t == 0) {
          tma_store_tile<BN>(P, bz ? &maps.y[1] : &maps.y[0], sout, n0, o);
          bulk_wait_group<0>();                               // complete before the grid is (PDL dependents read it)
        }
        return;
      }
    }
    // the ring is idle now (every stage consumed): stage the accumulator tile as rows for the epilogue warps
#pragma unroll
    for (int i = 0; i < BN / 2; i += 2) {
      const int r = 16 * w + (l >> 2) + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + 2 * (l & 3);
      *reinterpret_cast<float2*>(sacc + size_t(r) * L::kPitch + col) = make_float2(acc0[i], acc0[i + 1]);
      *reinterpret_cast<float2*>(sacc + size_t(r + 64) * L::kPitch + col) = make_float2(acc1[i], acc1[i + 1]);
    }
    if (splits > 1) { cluster_arrive(); cluster_wait(); cluster_arrive(); cluster_wait(); } else { named_bar_sync(1, 256); }
  } else {
    // ------------------------------------------------------------------ TMA producer (warp 8, one thread)
    if (elect_one()) {
      const CUtensorMap* mw = bz ? &maps.w[1] : &maps.w[0];
      const CUtensorMap* ma = bz ? &maps.a[1] : &maps.a[0];
      const uint32_t a_bytes = a_mode == A_TMA2D ? L::kABytes : (a_mode == A_TMA4D ? uint32_t(P.tw * P.th) * 128u : 0u);
      const uint32_t bytes = L::kBBytes + a_bytes;
      int s = 0;
      uint32_t ph = 0;
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait_quiet(empty_bar(s), ph ^ 1);
        load_stage<BN, false>(P, a_mode, smem_base + s * L::kStageBytes, full_bar(s), bytes, mw, ma, kb_begin + kb, n0, o);
        if (++s == kStages) { s = 0; ph ^= 1; }
      }
      if (tma_epi && has_res) {
        // the residual tile into stage s_out (== s) once block nkb - stages has left it
        mbar_wait_quiet(empty_bar(s), ph ^ 1);
        tma_load_tile<BN>(P, bz ? &maps.res[1] : &maps.res[0], smem_base + uint32_t(s) * L::kStageBytes, res_bar, n0, o);
      }
    }
    __syncwarp();
    if (splits > 1) { cluster_arrive(); cluster_wait(); cluster_arrive(); cluster_wait(); }
  }
}

// ---------------------------------------------------------------------------------------------------
// conv_gemm_persist_kernel: the 128 x 128 tile of grids that take more than one wave (TMA-staged A, no split-K).
// grid = min(tiles, SMs) CTAs; CTA c walks the tiles c, c + G, c + 2G, ... of the whole launch, n-tile fastest, then
// m-tile, then problem, so that the CTAs resident at the same time read the same A rows.  384 threads:
//   warpgroup 0    : TMA producer (one elected thread), running straight on from one tile's K blocks into the next one's
//   warpgroups 1, 2: consumers; warpgroup 1 + (j % 2) owns the CTA's j-th tile.  An ordering barrier hands the main loop
//                    from one consumer to the other, so one warpgroup's epilogue runs while the other's MMAs run.
// Each consumer owns a 128 x 128 fp16 output tile in shared memory: two 64-column halves of 128-byte rows, 128B-swizzled
// (the layout a TMA box of 64 columns x 128 rows has).  The epilogue runs on the accumulator registers (epi_fragments),
// writes fp16 pairs into the tile with stmatrix and one thread stores each half with a TMA store, which clips the rows and
// columns outside the output and completes while the warpgroup goes on to its next tile.  A residual tile is TMA-loaded
// into the same buffer when the tile starts and overwritten in place.  XM (LayerNorm fold / row statistics) keeps the
// row epilogue of epi_chunk: the accumulators are staged 32 columns at a time through the first 18 KB of the buffer
// (thread t owns tile row t).
// Halo launches (P.halo_bytes != 0, stride-1 3x3): the ring holds filter boxes only, and beside it kHaloSlots input halos
// take turns, one per (tile, 64-channel block).  A tile's K order is channel-block-major (cb outer, tap inner), so only
// the current block's halo has to be resident; a tile's halos are ring blocks of their own ring, j*ncb ... j*ncb + ncb - 1.
constexpr int kPersistThreads = 384;
constexpr int kHaloSlots = 2;
struct PersistLayout {
  static constexpr int kStageBytes = SmemLayout<128>::kStageBytes;
  static constexpr int kFilterBytes = SmemLayout<128>::kBBytes; // halo launches: a ring stage is the filter box alone
  static constexpr int kOutBytes = 2 * kOutHalfBytes;          // per consumer, 1024-byte aligned (TMA 128B swizzle)
  static constexpr int kPitch = 32 + 4;                        // XM: floats per staged row of a 32-column chunk
  static constexpr int kChunkBytes = BM * kPitch * 4;
  static_assert(kChunkBytes <= kOutBytes, "the XM staged chunk lives in the output tile");
  // [ring: stages x (A|B), or stages x B + kHaloSlots x halo] [2 x output tile] [barriers 256 B] [2 x bias 128 fp32]
  // ; + 1024 B alignment slack
  __host__ __device__ static int ring_bytes(int stages, int halo_bytes) {
    return halo_bytes ? stages * kFilterBytes + kHaloSlots * halo_bytes : stages * kStageBytes;
  }
  __host__ __device__ static int bar_off(int stages, int halo_bytes) { return ring_bytes(stages, halo_bytes) + 2 * kOutBytes; }
  static int total(int stages, int halo_bytes) { return bar_off(stages, halo_bytes) + 256 + 2 * 128 * 4 + 1024; }
};

// Consumer main loop of a halo launch over one tile: per 64-channel block cb, wait for its halo (ring block h0 + cb),
// then per tap wait for the filter stage (ring block g0 + 9 cb + tap) and issue two groups of four m64n128k16 wgmma RS,
// one per 64-row accumulator block hm.  Tile row m = (py, px) of tap (ky, kx) reads halo pixel r = (py + ky)(tw + 2) +
// px + kx, whose 16-byte chunk k sits at chunk k ^ (r % 8) (128B swizzle of the TMA box); lane_px[hm] is r at tap (0, 0)
// for the row this lane addresses in ldmatrix.  Fragments rotate through three register sets, so the two groups before
// a group stay in flight while its fragments load: a group's set is free once the group three back has retired.  A filter
// stage goes back once both groups of its tap have retired, a halo once its ninth tap's have.  Returns the last filter
// stage and halo slot, which the caller's final wgmma_wait frees.
template <class FullBar, class HaloFull, class HandBack, class HaloBack>
__device__ __forceinline__ void halo_mma_loop(float (&acc0)[64], float (&acc1)[64], const ConvParams& P, uint32_t smem_base,
                                              int kStages, int g0, int h0, const int (&lane_px)[2], int l, FullBar full_bar,
                                              HaloFull halo_full, HandBack hand_back, HaloBack halo_back, int& s_last, int& h_last) {
  const int ncb = P.Cin / BK, hw = P.tw + 2;
  const uint32_t halo_base = smem_base + uint32_t(kStages * PersistLayout::kFilterBytes);
  int s = g0 % kStages, h = h0 % kHaloSlots;
  uint32_t ph = uint32_t(g0 / kStages) & 1u, hph = uint32_t(h0 / kHaloSlots) & 1u;
  int s_prev = s, h_prev = h;
  uint32_t fa[3][4][4];
  for (int cb = 0; cb < ncb; ++cb) {
    mbar_wait_quiet(halo_full(h), hph);
    const uint32_t sh = halo_base + uint32_t(h * P.halo_bytes);
#pragma unroll 1
    for (int ky = 0; ky < 3; ++ky) {
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int tap = 3 * ky + kx;
        mbar_wait_quiet(full_bar(s), ph);
        const uint32_t sb = smem_base + uint32_t(s * PersistLayout::kFilterBytes);
#pragma unroll
        for (int hm = 0; hm < 2; ++hm) {
          const int f = (2 * kx + hm) % 3;          // group 2 tap + hm of the block, mod 3 (6 groups per filter row)
          const int r = lane_px[hm] + ky * hw + kx;
          const uint32_t a = sh + uint32_t(r) * 128u;
#pragma unroll
          for (int kc = 0; kc < 4; ++kc) ldmatrix_x4(fa[f][kc], a + (uint32_t((2 * kc + (l >> 4)) ^ (r & 7)) << 4));
          wgmma_fence();
#pragma unroll
          for (int kc = 0; kc < 4; ++kc) {
            const uint64_t bd = gmma_desc_sw128(sb + 32 * kc);
            if (hm == 0) wgmma_rs<0>(acc0, fa[f][kc], bd, (cb | tap | kc) != 0);
            else wgmma_rs<0>(acc1, fa[f][kc], bd, (cb | tap | kc) != 0);
          }
          wgmma_commit();
          wgmma_wait<2>();
          if (hm == 1 && (cb | tap) != 0) {   // group (previous tap, hm 1) has retired, and with it every MMA of that tap
            hand_back(s_prev);
            if (tap == 0) halo_back(h_prev);
          }
        }
        s_prev = s;
        if (++s == kStages) { s = 0; ph ^= 1; }
      }
    }
    h_prev = h;
    if (++h == kHaloSlots) { h = 0; hph ^= 1; }
  }
  s_last = s_prev;
  h_last = h_prev;
}

// tile t of the launch: n-tile fastest, then m-tile, then problem z
struct PersistTile { int z, n0; TileOrigin o; };
__device__ __forceinline__ PersistTile persist_tile(const ConvParams& P, int t) {
  PersistTile pt;
  const int r = t / P.n_tiles;
  const int mtile = r % P.m_tiles;
  pt.n0 = (t - r * P.n_tiles) * 128;
  pt.z = r / P.m_tiles;
  tile_origin(P, mtile, pt.o.m0, pt.o.tb, pt.o.oy0, pt.o.ox0);
  return pt;
}

// columns [32 CC, 32 CC + 32) of the warpgroup's accumulators -> staged rows (accumulator layout: see ptx.cuh)
template <int CC>
__device__ __forceinline__ void stage_chunk(const float (&acc0)[64], const float (&acc1)[64], float* sacc, int w, int l) {
#pragma unroll
  for (int i = 16 * CC; i < 16 * CC + 16; i += 2) {
    const int r = 16 * w + (l >> 2) + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) - 32 * CC + 2 * (l & 3);
    *reinterpret_cast<float2*>(sacc + r * PersistLayout::kPitch + col) = make_float2(acc0[i], acc0[i + 1]);
    *reinterpret_cast<float2*>(sacc + (r + 64) * PersistLayout::kPitch + col) = make_float2(acc1[i], acc1[i + 1]);
  }
}

template <bool XM>
__global__ void __launch_bounds__(kPersistThreads, 1)
conv_gemm_persist_kernel(const ConvParams P, const __grid_constant__ ConvMaps maps) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  using L = SmemLayout<128>;
  using PL = PersistLayout;
  const int kStages = P.stages;
  const bool halo = !XM && P.halo_bytes != 0;                 // stride-1 3x3: one input halo per 64-channel block
  const uint32_t ring_bytes = uint32_t(PL::ring_bytes(kStages, P.halo_bytes));
  const uint32_t bar_off = uint32_t(PL::bar_off(kStages, P.halo_bytes));
  const uint32_t bar_base = smem_base + bar_off;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (kMaxStages + s); };
  auto order_bar = [&](int c) { return bar_base + 8u * (2 * kMaxStages + c); };   // consumer c may start its main loop
  auto res_bar = [&](int c) { return bar_base + 8u * (2 * kMaxStages + 2 + c); }; // consumer c's residual tile has landed
  auto halo_full = [&](int h) { return bar_base + 8u * (2 * kMaxStages + 4 + h); };
  auto halo_empty = [&](int h) { return bar_base + 8u * (2 * kMaxStages + 4 + kHaloSlots + h); };
  static_assert(8 * (2 * kMaxStages + 4 + 2 * kHaloSlots) <= 256, "barriers");
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));

  pdl_launch_dependents();
  const int tid = threadIdx.x;
  const int wg = tid >> 7;
  const int ncb = P.Cin / BK;                                 // halo: 64-channel blocks, 9 filter blocks each
  const int nkb = halo ? 9 * ncb : P.k_pad / BK;
  const int a_mode = P.a_mode;
  const bool has_res = (P.epi & (ICAF_EPI_ADD_RES | ICAF_EPI_SCALED_RES)) != 0;
  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 4);                             // one arrival per warp of the consuming warpgroup
    }
    mbar_init(order_bar(0), 4);
    mbar_init(order_bar(1), 4);
    mbar_init(res_bar(0), 1);
    mbar_init(res_bar(1), 1);
    for (int h = 0; h < kHaloSlots; ++h) {
      mbar_init(halo_full(h), 1);
      mbar_init(halo_empty(h), 4);
    }
    fence_mbar_init();
  }
  if (tid == 32) {
    tma_prefetch_desc(&maps.w[0]);
    tma_prefetch_desc(&maps.a[0]);
    if (P.tiles > P.m_tiles * P.n_tiles) { tma_prefetch_desc(&maps.w[1]); tma_prefetch_desc(&maps.a[1]); }
    if (!XM) {
      tma_prefetch_desc(&maps.y[0]);
      if (has_res) tma_prefetch_desc(&maps.res[0]);
    }
  }
  __syncthreads();
  pdl_wait();   // prologue (barriers, descriptor prefetch) overlapped the previous kernel

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer (warp 0, one thread)
    setmaxnreg_dec<40>();
    if (tid < 32 && elect_one()) {
      const uint32_t a_bytes = a_mode == A_TMA2D ? L::kABytes : uint32_t(P.tw * P.th) * 128u;
      const uint32_t bytes = L::kBBytes + a_bytes;
      int s = 0, h = 0;
      uint32_t ph = 0, hph = 0;
      for (int tile = blockIdx.x; tile < P.tiles; tile += gridDim.x) {
        const PersistTile pt = persist_tile(P, tile);
        const CUtensorMap* mw = pt.z ? &maps.w[1] : &maps.w[0];
        const CUtensorMap* ma = pt.z ? &maps.a[1] : &maps.a[0];
        if (halo) {
          // per 64-channel block: the (64, tw+2, th+2) halo around the tile (zero-filled outside the map), then the
          // block's nine filter boxes at K column tap * Cin + cb * 64 (pack_conv_weight's tap-major K)
          const uint32_t halo_tx = uint32_t((P.tw + 2) * (P.th + 2)) * 128u;
          for (int cb = 0; cb < ncb; ++cb) {
            mbar_wait_quiet(halo_empty(h), hph ^ 1);
            mbar_arrive_expect_tx(halo_full(h), halo_tx);
            tma_load_4d(smem_base + uint32_t(kStages * PL::kFilterBytes + h * P.halo_bytes), ma, halo_full(h), cb * BK,
                        pt.o.ox0 - 1, pt.o.oy0 - 1, pt.o.tb);
            if (++h == kHaloSlots) { h = 0; hph ^= 1; }
            for (int tap = 0; tap < 9; ++tap) {
              mbar_wait_quiet(empty_bar(s), ph ^ 1);
              mbar_arrive_expect_tx(full_bar(s), PL::kFilterBytes);
              tma_load_2d(smem_base + uint32_t(s * PL::kFilterBytes), mw, full_bar(s), tap * P.Cin + cb * BK, pt.n0);
              if (++s == kStages) { s = 0; ph ^= 1; }
            }
          }
          continue;
        }
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait_quiet(empty_bar(s), ph ^ 1);
          load_stage<128, true>(P, a_mode, smem_base + s * L::kStageBytes, full_bar(s), bytes, mw, ma, kb, pt.n0, pt.o);
          if (++s == kStages) { s = 0; ph ^= 1; }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroups (wgmma + epilogue)
  setmaxnreg_inc<232>();
  const int c = wg - 1;
  const int t = tid & 127, w = t >> 5, l = t & 31;
  const int bar_id = 2 + c;                                   // warpgroup-local named barrier
  const uint32_t sout = smem_base + ring_bytes + uint32_t(c * PL::kOutBytes);                  // this consumer's output tile
  float* sacc = reinterpret_cast<float*>(smem_gen + ring_bytes + c * PL::kOutBytes);           // XM: staged chunk
  float* sbias = reinterpret_cast<float*>(smem_gen + bar_off + 256 + c * 128 * 4);
  // halo: the halo pixel at tap (0, 0) of the tile row this lane addresses in ldmatrix (matrix l / 8 of an x4 covers rows
  // 8 ((l / 8) % 2) ... of the 16-row group, chunk (l / 16) of the 16-channel K step) for the accumulator blocks 0-63 and
  // 64-127.  Rows past the tw x th patch (20 x 6 tiles) read the patch's last pixel: they are never stored.
  int lane_px[2];
#pragma unroll
  for (int hm = 0; hm < 2; ++hm) {
    int m = 64 * hm + 16 * w + (l & 7) + 8 * ((l >> 3) & 1);
    if (m > P.tw * P.th - 1) m = P.tw * P.th - 1;
    const int py = P.tw ? m / P.tw : 0;
    lane_px[hm] = py * (P.tw + 2) + m - py * P.tw;
  }
  for (int tile = blockIdx.x + c * gridDim.x; tile < P.tiles; tile += 2 * gridDim.x) {
    const int j = (tile - int(blockIdx.x)) / int(gridDim.x);  // ordinal of the tile among this CTA's tiles
    const PersistTile pt = persist_tile(P, tile);
    const ConvProblem pr = pick_problem(P, pt.z);
    const int n0 = pt.n0;
    const TileOrigin& o = pt.o;
    // Epilogue operands that do not depend on the main loop are fetched now so their DRAM latency hides behind it:
    // bias slice and (alpha, beta) into registers; XM: this thread's output row (residual row into L2); otherwise the
    // row bias of the accumulator fragments and the residual tile.
    const float bias_r = (pr.bias && !(P.epi & ICAF_EPI_BIAS_ROW) && n0 + t < P.N) ? __ldg(pr.bias + n0 + t) : 0.f;
    float alpha = 0.f, beta = 1.f;
    if (P.epi & ICAF_EPI_SCALED_RES) { alpha = __ldg(pr.alpha); beta = __ldg(pr.beta); }
    StagedRow sr;                                             // XM
    float rb[4] = {0.f, 0.f, 0.f, 0.f};                       // !XM: row bias of the accumulator fragments
    if (XM) {
      staged_row<128, XM>(sr, P, pr, o, t, n0);
    } else {
      fragment_row_bias(rb, P, pr, o, w, l);
      if (t == 0) {
        bulk_wait_group_read<0>();                            // the previous tile's TMA store has read the buffer
        if (has_res) tma_load_tile<128>(P, pt.z ? &maps.res[1] : &maps.res[0], sout, res_bar(c), n0, o);
      }
      sbias[t] = bias_r;
      named_bar_sync(bar_id, 128);                            // bias slice complete, output tile free
    }

    // ---- main loop.  Tile j's K blocks are ring blocks j*nkb ... j*nkb + nkb - 1.  Waiting for the other consumer's
    // turn also guarantees that every earlier ring block has been seen full, so the parity waits below cannot alias.
    float acc0[64], acc1[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
    auto hand_back = [&](int s) { if (l == 0) mbar_arrive(empty_bar(s)); };   // one arrival per consumer warp
    auto halo_back = [&](int h) { if (l == 0) mbar_arrive(halo_empty(h)); };
    const int g0 = j * nkb;
    if (j > 0) mbar_wait_quiet(order_bar(c), uint32_t((j >> 1) - (1 - c)) & 1u);
    int s_last, h_last = 0;
    if (halo) {
      halo_mma_loop(acc0, acc1, P, smem_base, kStages, g0, j * ncb, lane_px, l, full_bar, halo_full, hand_back, halo_back,
                    s_last, h_last);
    } else {
      s_last = mma_loop<128>(acc0, acc1, smem_base, kStages, nkb, g0 % kStages, uint32_t(g0 / kStages) & 1u, full_bar,
                             hand_back);
    }
    if (l == 0) mbar_arrive(order_bar(c ^ 1));          // every MMA of this tile is issued: the other consumer's turn
    wgmma_wait<0>();
    hand_back(s_last);
    if (halo) halo_back(h_last);

    if constexpr (!XM) {
      // ---- epilogue on the accumulator registers, 16 columns at a time, then the TMA store of the tile
      if (has_res) mbar_wait_quiet(res_bar(c), uint32_t(j >> 1) & 1u);
      epi_tile_fragments<64>(epi_mode_act<false>(P, has_res), acc0, acc1, sout, sbias, rb, alpha, beta, w, l);
      fence_proxy_async_smem();                             // the tile is visible to the TMA unit ...
      named_bar_sync(bar_id, 128);                          // ... once every thread of the warpgroup has written its part
      if (t == 0) {
        tma_store_tile<128>(P, pt.z ? &maps.y[1] : &maps.y[0], sout, n0, o);
        // this consumer's last tile: its writes complete before the grid does (dependent launches read them after
        // griddepcontrol.wait).  Waiting inside the loop keeps the consumer's code one setmaxnreg region for ptxas.
        if (tile + 2 * int(gridDim.x) >= P.tiles) bulk_wait_group<0>();
      }
      continue;
    }

    // ---- XM epilogue, 32 columns at a time
    const int mode_act = epi_mode_act<XM>(P, has_res);
    const float* arow = sacc + size_t(t) * PL::kPitch;
#pragma unroll 1
    for (int cc = 0; cc < 4; ++cc) {
      named_bar_sync(bar_id, 128);                      // the previous chunk (or tile) has been read out
      if (cc == 0) sbias[t] = bias_r;
      switch (cc) {
        case 0: stage_chunk<0>(acc0, acc1, sacc, w, l); break;
        case 1: stage_chunk<1>(acc0, acc1, sacc, w, l); break;
        case 2: stage_chunk<2>(acc0, acc1, sacc, w, l); break;
        default: stage_chunk<3>(acc0, acc1, sacc, w, l); break;
      }
      named_bar_sync(bar_id, 128);
      const int cb = 32 * cc;
      if (sr.mvalid && n0 + cb < P.N) {
        uint32_t acc[32];
        load_staged(acc, arow);
        epi_staged_chunk<XM>(mode_act, acc, sr, sbias, alpha, beta, cb, n0 + cb, P.N);
      }
    }
    if (mode_act == 11 && sr.mvalid && n0 < P.N) epi_row_emit(sr.ex, P, pr, sr.m, n0, min(n0 + 128, P.N));
  }
}

// ---------------------------------------------------------------------------------------------------
// conv_stem_kernel: 16 input channels, 3x3, stride 1, pad 1, one 128 x 64 output tile per CTA (plan_conv sends the BN = 64
// gather launches of that geometry here when TMA can store the output and there is no residual).  On the one-tile
// kernel such a launch gathers A once per tap, so every input pixel crosses from L2 nine times, and pads K from 144 to
// 192, so three of its twelve k16 steps multiply zeros.  Here one warpgroup does everything:
//   filter : the packed filter's first three 64-column K blocks by TMA, 128B-swizzled as on the one-tile kernel (24 KB,
//            one mbarrier); K columns 144-191 are loaded but never read;
//   halo   : the tile's 128 consecutive output rows (b, y, x) fall into runs of one output row each -- at most two when
//            Wo >= 128, up to StemLayout::runs(Wo) on narrow maps.  Run j (from output pixel (g0 + j, xs), len pixels)
//            needs the input rows y - 1 ... y + 1, pixels xs - 1 ... xs + len, cp.async'd (zero-filled outside the map:
//            the padding; and past M) into halo rows 3 j + ty of `pitch` pixels each, the same pitch for every run, so
//            tile row (j, p) at tap (ty, tx) is halo pixel (3 j + ty) pitch + p + tx.  A pixel is 32 bytes (two 16-byte
//            chunks); chunk c of halo pixel h sits at chunk c ^ ((h >> 2) & 1), so the eight rows of an ldmatrix phase
//            (consecutive pixels) hit eight distinct bank groups;
//   MMA    : per tap, the two 64-row blocks' A fragments by ldmatrix and two m64n64k16 wgmma RS: 18 MMAs, tap-major like
//            the one-tile kernel's K order, so each accumulator sums the same nine products in the same order (the one-tile
//            kernel's three padded steps add +0).  Fragments rotate through three register sets, two taps in flight;
//   output : the halo becomes the output tile: epi_tile_fragments and a TMA store of the 2-D [M][N] box, as on the
//            one-tile kernel's register epilogue.
// Shared memory (51 KB at Wo >= 128) and registers (at most 128 per thread) let four CTAs share an SM, so one CTA's
// filter load and gather overlap the others' MMAs, epilogues and stores.
constexpr int kStemThreads = 128;
struct StemLayout {
  static constexpr int kFilterBytes = 3 * SmemLayout<64>::kBBytes;   // three 64 x 64 K filter boxes
  static constexpr int kBiasOff = kFilterBytes;                // 64 fp32
  static constexpr int kBarOff = kBiasOff + 64 * 4;
  static constexpr int kHaloOff = kFilterBytes + 1024;         // 1024-byte aligned: the output tile (128B swizzle) reuses it
  __host__ __device__ static int pitch(int Wo) { return (Wo < BM ? Wo : BM) + 2; }   // pixels per halo row
  __host__ __device__ static int runs(int Wo) { return 1 + (BM - 1 + Wo - 1) / Wo; }  // most runs a tile can span
  // [filter][bias, mbarrier][halo, or the output tile] ; + 1024 B alignment slack
  static int total(int Wo) {
    const int halo = runs(Wo) * 3 * pitch(Wo) * 32;
    return kHaloOff + (halo > kOutHalfBytes ? halo : kOutHalfBytes) + 1024;
  }
};

__global__ void __launch_bounds__(kStemThreads, 4)
conv_stem_kernel(const ConvParams P, const __grid_constant__ ConvMaps maps) {
  extern __shared__ uint8_t smem_raw[];
  using SL = StemLayout;
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  const uint32_t bar = smem_base + SL::kBarOff;
  const uint32_t halo = smem_base + SL::kHaloOff;
  float* sbias = reinterpret_cast<float*>(smem_gen + SL::kBiasOff);

  pdl_launch_dependents();
  const int t = threadIdx.x, w = t >> 5, l = t & 31;
  const int bz = blockIdx.z, n0 = blockIdx.y * 64;
  const ConvProblem pr = pick_problem(P, bz);
  const TileOrigin o{int(blockIdx.x) * BM, 0, 0, 0};
  // the tile's runs: the first from output pixel (g0, ox0) of the (b, y) row index g0, the others from x = 0
  const int g0 = o.m0 / P.Wo, ox0 = o.m0 - g0 * P.Wo;
  const int len0 = min(P.Wo - ox0, BM);
  const int nruns = 1 + (BM - len0 + P.Wo - 1) / P.Wo;
  const int pitch = SL::pitch(P.Wo);
  // halo pixel at tap (0, 0) of the tile row this lane addresses in ldmatrix, for the 64-row blocks 0 and 1 (matrix l / 8
  // of an x4 covers rows 8 ((l / 8) % 2) ... of the warp's 16, chunk l / 16 of the tap's 16 channels)
  int lane_hp[2];
#pragma unroll
  for (int hm = 0; hm < 2; ++hm) {
    const int r = 64 * hm + 16 * w + (l & 7) + 8 * ((l >> 3) & 1);
    int j = 0, p = r;
    if (r >= len0) {
      const int q = (r - len0) / P.Wo;
      j = 1 + q;
      p = r - len0 - q * P.Wo;
    }
    lane_hp[hm] = 3 * j * pitch + p;
  }
  if (t == 0) {
    mbar_init(bar, 1);
    fence_mbar_init();
  }
  if (t == 32) {
    tma_prefetch_desc(bz ? &maps.w[1] : &maps.w[0]);
    tma_prefetch_desc(bz ? &maps.y[1] : &maps.y[0]);
  }
  __syncthreads();
  pdl_wait();   // prologue (barrier, descriptor prefetch, lane addresses) overlapped the previous kernel

  if (t == 0) {
    // K blocks 0-2 of the packed filter (K = tap * 16 + channel), output channels n0 ... n0 + 63
    const CUtensorMap* mw = bz ? &maps.w[1] : &maps.w[0];
    mbar_arrive_expect_tx(bar, SL::kFilterBytes);
#pragma unroll 1
    for (int kb = 0; kb < 3; ++kb) tma_load_2d(smem_base + uint32_t(kb * SmemLayout<64>::kBBytes), mw, bar, kb * BK, n0);
  }
  if (t < 64) sbias[t] = (pr.bias && !(P.epi & ICAF_EPI_BIAS_ROW) && n0 + t < P.N) ? __ldg(pr.bias + n0 + t) : 0.f;
  float rb[4] = {0.f, 0.f, 0.f, 0.f};
  fragment_row_bias(rb, P, pr, o, w, l);

  // ---- halo: thread t copies chunk t % 2 of pixels t / 2, t / 2 + 64, ... of every halo row
  const int c = t & 1;
#pragma unroll 1
  for (int j = 0; j < nruns; ++j) {
    const int g = g0 + j;
    const int xs = j ? 0 : ox0;
    const int len = j ? min(P.Wo, BM - len0 - (j - 1) * P.Wo) : len0;
    const int b = g / P.Ho, oy = g - b * P.Ho;
    const bool gv = g < P.B * P.Ho;
#pragma unroll
    for (int ty = 0; ty < 3; ++ty) {
      const int iy = oy + ty - 1;
      const bool rv = gv && (unsigned)iy < (unsigned)P.Hi;
      const __half* src = pr.x + (rv ? (size_t(b) * P.Hi + iy) * P.Wi * pr.x_ld : 0) + 8 * c;
      const int h0 = (3 * j + ty) * pitch;
      for (int px = t >> 1; px < len + 2; px += kStemThreads / 2) {
        const int ix = xs - 1 + px, h = h0 + px;
        const bool ok = rv && (unsigned)ix < (unsigned)P.Wi;
        cp_async16(halo + uint32_t(h) * 32u + (uint32_t(c ^ ((h >> 2) & 1)) << 4), ok ? src + size_t(ix) * pr.x_ld : pr.x, ok);
      }
    }
  }
  cp_async_commit();
  cp_async_wait<0>();
  __syncthreads();                                            // halo and bias complete
  mbar_wait_quiet(bar, 0);                                    // filter landed

  // ---- nine taps x two 64-row blocks of m64n64k16 wgmma RS
  float acc0[32], acc1[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
  uint32_t fa[3][2][4];
#pragma unroll
  for (int tap = 0; tap < 9; ++tap) {
    const int f = tap % 3;                                    // free once the group of tap - 3 has retired
    const int off = (tap / 3) * pitch + tap % 3;
#pragma unroll
    for (int hm = 0; hm < 2; ++hm) {
      const int h = lane_hp[hm] + off;
      ldmatrix_x4(fa[f][hm], halo + uint32_t(h) * 32u + (uint32_t((l >> 4) ^ ((h >> 2) & 1)) << 4));
    }
    wgmma_fence();
    const uint64_t bd = gmma_desc_sw128(smem_base + uint32_t((tap >> 2) * SmemLayout<64>::kBBytes + 32 * (tap & 3)));
    wgmma_rs<0>(acc0, fa[f][0], bd, tap != 0);
    wgmma_rs<0>(acc1, fa[f][1], bd, tap != 0);
    wgmma_commit();
    wgmma_wait<2>();
  }
  wgmma_wait<0>();
  __syncthreads();                                            // every warp's fragments are in: the halo is free

  // ---- epilogue on the accumulators into the output tile (where the halo was), TMA store
  epi_tile_fragments<32>(epi_mode_act<false>(P, false), acc0, acc1, halo, sbias, rb, 0.f, 1.f, w, l);
  fence_proxy_async_smem();                                   // the tile is visible to the TMA unit ...
  __syncthreads();                                            // ... once every thread has written its part
  if (t == 0) {
    tma_store_tile<64>(P, bz ? &maps.y[1] : &maps.y[0], halo, n0, o);
    bulk_wait_group<0>();                                     // complete before the grid is (PDL dependents read it)
  }
}

// ---------------------------------------------------------------------------------------------------
// CUDA-core reference with the identical contract (tests only).
struct SimtParams { ConvParams P; const __half* w[2]; };
__global__ void conv_gemm_simt_kernel(const SimtParams S) {
  pdl_launch_dependents();
  pdl_wait();
  const ConvParams& P = S.P;
  const ConvProblem pr = pick_problem(P, blockIdx.z);
  const __half* w = blockIdx.z ? S.w[1] : S.w[0];
  long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= (long long)P.M * P.N) return;
  int n = int(idx % P.N);
  int m = int(idx / P.N);
  int ox = m % P.Wo, t = m / P.Wo, oy = t % P.Ho, b = t / P.Ho;
  float acc = 0.f;
  for (int ky = 0; ky < P.kh; ++ky)
    for (int kx = 0; kx < P.kw; ++kx) {
      int iy = oy * P.stride - P.pad + ky, ix = ox * P.stride - P.pad + kx;
      if ((unsigned)iy >= (unsigned)P.Hi || (unsigned)ix >= (unsigned)P.Wi) continue;
      const __half* xp = pr.x + (size_t(b) * P.Hi * P.Wi + size_t(iy) * P.Wi + ix) * pr.x_ld;
      const __half* wp = w + size_t(n) * P.k_pad + (ky * P.kw + kx) * P.Cin;
      for (int c = 0; c < P.Cin; ++c) acc += __half2float(xp[c]) * __half2float(wp[c]);
    }
  if (pr.bias) acc += (P.epi & ICAF_EPI_BIAS_ROW) ? pr.bias[m] : pr.bias[n];
  if (P.act == ICAF_ACT_SILU) acc = acc / (1.0f + expf(-acc));
  else if (P.act == ICAF_ACT_GELU) acc = gelu_erf_f(acc);
  if (pr.res) {
    float rf = __half2float(pr.res[size_t(m) * pr.res_ld + n]);
    acc = (P.epi & ICAF_EPI_SCALED_RES) ? (*pr.alpha) * rf + (*pr.beta) * acc : acc + rf;
  }
  pr.y[size_t(m) * pr.y_ld + n] = __float2half_rn(acc);
}

// Geometry half of the argument check (host only): everything the planner needs, no pointers.
static int fill_geom(const icaf_conv_geom* g, int n_io, ConvParams& P) {
  if (!g || n_io < 1 || n_io > 2) return set_error(ICAF_ERR_BAD_ARG, "conv2d: need 1 or 2 problems");
  if (!(g->Cin == 4 || g->Cin % 8 == 0)) return set_error(ICAF_ERR_UNSUPPORTED, "conv2d: Cin must be 4 or a multiple of 8");
  if (g->Cin == 4 && (g->Wi % 2 || g->stride % 2 || g->pad % 2 || g->kw % 2))
    return set_error(ICAF_ERR_UNSUPPORTED, "conv2d: packed-image (Cin=4) path needs even Wi, stride, pad, kw");
  if (g->k_pad % 64 || g->k_pad < g->kh * g->kw * g->Cin) return set_error(ICAF_ERR_BAD_ARG, "conv2d: bad k_pad");
  if (g->w_rows < g->Cout) return set_error(ICAF_ERR_BAD_ARG, "conv2d: w_rows < Cout");
  long long M = (long long)g->B * g->Ho * g->Wo;
  if (M <= 0 || M > 0x7fffffffLL || (long long)g->B * g->Hi * g->Wi > 0x7fffffffLL)
    return set_error(ICAF_ERR_BAD_ARG, "conv2d: size out of range");
  if ((g->epi & (ICAF_EPI_ADD_RES | ICAF_EPI_SCALED_RES)) == (ICAF_EPI_ADD_RES | ICAF_EPI_SCALED_RES))
    return set_error(ICAF_ERR_BAD_ARG, "conv2d: ADD_RES and SCALED_RES are exclusive");
  if ((g->epi & ICAF_EPI_LN_FOLD) && ((g->epi & ~ICAF_EPI_LN_FOLD) != 0 || !(g->act == ICAF_ACT_NONE || g->act == ICAF_ACT_GELU) ||
                                      g->kh != 1 || g->kw != 1 || g->stride != 1 || g->pad != 0))
    return set_error(ICAF_ERR_UNSUPPORTED, "conv2d: LN_FOLD is a linear-layer (1x1) epilogue without residual, activation none / GELU");
  if ((g->epi & ICAF_EPI_EMIT_STATS) && ((g->epi & ~ICAF_EPI_EMIT_STATS) != ICAF_EPI_SCALED_RES || g->act != ICAF_ACT_NONE))
    return set_error(ICAF_ERR_UNSUPPORTED, "conv2d: EMIT_STATS rides on the SCALED_RES epilogue without activation");
  P.M = int(M); P.N = g->Cout; P.K = g->kh * g->kw * g->Cin; P.k_pad = g->k_pad;
  P.B = g->B; P.Hi = g->Hi; P.Wi = g->Wi; P.Cin = g->Cin; P.Ho = g->Ho; P.Wo = g->Wo;
  P.kh = g->kh; P.kw = g->kw; P.stride = g->stride; P.pad = g->pad; P.act = g->act; P.epi = g->epi;
  P.a_mode = A_GATHER; P.tw = P.th = P.tiles_x = P.tiles_y = 0; P.stages = 2; P.splits = 1; P.cblk = 64;
  P.ln_parts = 0; P.ln_eps = 0.f; P.ln_inv_k = 0.f;
  P.m_tiles = P.n_tiles = P.tiles = 0;
  P.tma_epi = 0;
  P.halo_bytes = 0;
  memset(P.p, 0, sizeof(P.p));
  return ICAF_OK;
}

static int fill_params(const icaf_conv_geom* g, const icaf_conv_io* io, int n_io, ConvParams& P, const __half* (&w)[2]) {
  if (!io) return set_error(ICAF_ERR_BAD_ARG, "conv2d: null io");
  if (int rc = fill_geom(g, n_io, P)) return rc;
  for (int i = 0; i < 2; ++i) {
    const icaf_conv_io& s = io[i < n_io ? i : 0];
    bool need_res = g->epi & (ICAF_EPI_ADD_RES | ICAF_EPI_SCALED_RES);
    if (!s.x || !s.w || !s.y || (need_res && !s.res) || ((g->epi & ICAF_EPI_SCALED_RES) && (!s.alpha || !s.beta)))
      return set_error(ICAF_ERR_BAD_ARG, "conv2d: null pointer");
    if ((reinterpret_cast<uintptr_t>(s.x) & 15) || (reinterpret_cast<uintptr_t>(s.w) & 15) || (s.x_ld % 8 && g->Cin != 4) ||
        (g->Cin == 4 && s.x_ld != 4))
      return set_error(ICAF_ERR_BAD_ARG, "conv2d: x / w must be 16-byte aligned with x_ld a multiple of 8");
    if ((g->epi & ICAF_EPI_LN_FOLD) && (!s.ln_stats || !s.ln_colsum || s.ln_parts < 1 || s.ln_parts > 64))
      return set_error(ICAF_ERR_BAD_ARG, "conv2d: LN_FOLD needs ln_stats, ln_colsum and 1..64 partials per row");
    if ((g->epi & ICAF_EPI_EMIT_STATS) && !s.stats_out) return set_error(ICAF_ERR_BAD_ARG, "conv2d: EMIT_STATS needs stats_out");
    if (i > 0 && (g->epi & ICAF_EPI_LN_FOLD) && (s.ln_parts != io[0].ln_parts || s.ln_eps != io[0].ln_eps))
      return set_error(ICAF_ERR_BAD_ARG, "conv2d: grouped problems must share ln_parts / ln_eps");
    P.p[i] = ConvProblem{(const __half*)s.x, s.bias, need_res ? (const __half*)s.res : nullptr, (__half*)s.y, s.alpha, s.beta,
                         s.x_ld, s.res_ld, s.y_ld,
                         (g->epi & ICAF_EPI_LN_FOLD) ? (const float2*)s.ln_stats : nullptr,
                         (g->epi & ICAF_EPI_LN_FOLD) ? s.ln_colsum : nullptr,
                         (g->epi & ICAF_EPI_EMIT_STATS) ? (float2*)s.stats_out : nullptr};
    if (i == 0 && (g->epi & ICAF_EPI_LN_FOLD)) { P.ln_parts = s.ln_parts; P.ln_eps = s.ln_eps; P.ln_inv_k = 1.0f / float(P.K); }
    w[i] = (const __half*)s.w;
  }
  return ICAF_OK;
}

// Pick how the A tile is staged (see the header comment) and, for A_TMA4D, the tile shape.
static void plan_a_mode(const icaf_conv_geom* g, ConvParams& P) {
  if (g->kh == 1 && g->kw == 1 && g->stride == 1 && g->pad == 0 && g->Cin % 8 == 0) {
    P.a_mode = A_TMA2D;
    return;
  }
  if (g->Cin % 64 == 0 && g->stride <= 2) {
    // tile = th x tw output pixels of one image, tw | Wo, tw*th <= 128: maximise the fraction of useful MMA rows
    int best_tw = 0, best_th = 0;
    double best_u = 0.0;
    for (int tw = 1; tw <= 128 && tw <= g->Wo; ++tw) {
      if (g->Wo % tw || tw * g->stride > 256) continue;
      int th = 128 / tw;
      if (th > g->Ho) th = g->Ho;
      if (th * g->stride > 256) th = 256 / g->stride;
      int ty = (g->Ho + th - 1) / th;
      double u = double(g->Wo) * g->Ho / (double(g->Wo / tw) * ty * 128.0);
      if (u > best_u + 1e-9 || (u > best_u - 1e-9 && tw > best_tw)) { best_u = u; best_tw = tw; best_th = th; }
    }
    if (best_u >= 0.6) {
      P.a_mode = A_TMA4D; P.tw = best_tw; P.th = best_th; P.tiles_x = g->Wo / best_tw; P.tiles_y = (g->Ho + best_th - 1) / best_th;
    }
  }
}

template <int BN>
static int plan_tc(ConvParams& P, int n_io, ConvPlan& pl) {
  using L = SmemLayout<BN>;
  constexpr int kSmemCap = 227 * 1024;
  const int mt = P.a_mode == A_TMA4D ? P.B * P.tiles_x * P.tiles_y : (P.M + BM - 1) / BM;
  if (P.a_mode == A_TMA4D && !(P.tw >= 1 && P.th >= 1 && P.tw * P.th <= BM && P.tiles_x * P.tw >= P.Wo && P.tiles_y * P.th >= P.Ho &&
                               P.cblk == 64 && P.Cin % 64 == 0))
    return set_error(ICAF_ERR_BAD_ARG, "conv2d(tc): 4-D tiles must cover the map with at most 128 pixels each, 64-channel blocks");
  unsigned gx = unsigned(mt), gy = unsigned((P.N + BN - 1) / BN), gz = unsigned(n_io);
  // Ring depth: a grid that fits in one wave gets the whole SM (deep ring: the K loop is latency-bound at small M);
  // otherwise two CTAs of the narrow tiles share an SM so that one CTA's epilogue overlaps the other's main loop (BN = 128
  // keeps one CTA per SM: its 128 accumulator registers per consumer thread leave no room for a second one).
  const long long tiles = (long long)gx * gy * gz;
  const int budget = (tiles <= pl.sms || BN > 64) ? kSmemCap : (kSmemCap / 2 - 1024);
  int stages = (budget - L::kTailBytes) / L::kStageBytes;
  const int nkb = P.k_pad / BK;
  if (stages > nkb) stages = nkb;
  if (stages > kMaxStages) stages = kMaxStages;
  if (stages < 2) stages = 2;
  // Split-K: a grid that leaves most SMs idle on a deep K loop is spread over clusters of `splits` CTAs per tile.
  int splits = 1;
  if (tiles * 2 <= pl.sms && nkb >= 8) {
    splits = int(pl.sms / tiles);
    if (splits > 8) splits = 8;                    // portable cluster size
    if (splits > nkb / 4) splits = nkb / 4;        // >= 4 K blocks per CTA
    if (splits < 1) splits = 1;
  }
  if (splits > 1) {
    const int per = (nkb + splits - 1) / splits;
    if (stages > per) stages = per < 2 ? 2 : per;
    gx *= splits;
  }
  if (stages > kMaxStages || L::total(stages) > kSmemCap)
    return set_error(ICAF_ERR_BAD_ARG, "conv2d(tc): shared-memory plan exceeds the ring / 227 KB");
  P.stages = stages;
  P.splits = splits;
  pl.kernel = ICAF_KERNEL_TC; pl.bn = BN;
  pl.grid_x = gx; pl.grid_y = gy; pl.grid_z = gz; pl.cluster = unsigned(splits);
  pl.smem = L::total(stages);
  pl.tiles = int(tiles); pl.m_tiles = mt; pl.n_tiles = int(gy);
  pl.persist = false; pl.ctas = int(gx * gy * gz);
  return ICAF_OK;
}

// A 128 x 128 plan with TMA-staged A, no split-K and more tiles than SMs runs on conv_gemm_persist_kernel: one CTA per SM
// walks the tiles, so the ring fill and the epilogue of one tile overlap the main loop of the next.  The ring takes what
// the output tiles (and, for stride-1 3x3 patch tiles, the input halos) leave of the 227 KB (it is not clamped to the K
// loop: it runs on across tiles).  A halo slot holds (tw+2)(th+2) pixels of 128 B, rounded up to the 1 KB the 128B
// swizzle needs (23 KB for 16 x 8 and 8 x 16 tiles, 22 KB for 20 x 6), which leaves 7 filter stages.
static int plan_persist(ConvParams& P, ConvPlan& pl) {
  constexpr int kSmemCap = 227 * 1024;
  const bool halo = !pl.xm && P.a_mode == A_TMA4D && P.kh == 3 && P.kw == 3 && P.stride == 1 && P.pad == 1;
  P.halo_bytes = halo ? ((P.tw + 2) * (P.th + 2) * 128 + 1023) / 1024 * 1024 : 0;
  int stages = kMaxStages;
  while (stages > 2 && PersistLayout::total(stages, P.halo_bytes) > kSmemCap) --stages;
  if (PersistLayout::total(stages, P.halo_bytes) > kSmemCap)
    return set_error(ICAF_ERR_BAD_ARG, "conv2d(persist): shared-memory plan exceeds 227 KB");
  P.stages = stages;
  P.m_tiles = pl.m_tiles; P.n_tiles = pl.n_tiles; P.tiles = pl.tiles;
  pl.persist = true;
  pl.ctas = pl.tiles < pl.sms ? pl.tiles : pl.sms;
  pl.smem = PersistLayout::total(stages, P.halo_bytes);
  return ICAF_OK;
}

// out_maps: the output (and residual) maps of the register epilogue's TMA stores, 64-column boxes of the tile's rows
// (2-D: 128 rows of [M][N], for A_TMA2D and A_GATHER; 4-D: the tw x th patch of the (N, Wo, Ho, B) view).  They span N
// columns, so a tile never writes the channels next to a slice of a wider buffer.
template <int BN>
static int encode_maps(const ConvParams& P, const __half* const (&w)[2], const icaf_conv_geom* g, int n_io, bool out_maps,
                       ConvMaps& maps) {
  memset(&maps, 0, sizeof(maps));
  for (int i = 0; i < n_io; ++i) {
    int rc = encode_tmap_2d(&maps.w[i], w[i], (uint64_t)P.k_pad, (uint64_t)g->w_rows, (uint64_t)P.k_pad * 2, BK, BN);
    if (rc) return rc;
    const ConvProblem& pr = P.p[i];
    if (P.a_mode == A_TMA2D)
      rc = encode_tmap_2d(&maps.a[i], pr.x, (uint64_t)P.Cin, (uint64_t)P.M, (uint64_t)pr.x_ld * 2, BK, BM);
    else if (P.a_mode == A_TMA4D && P.halo_bytes)       // persistent stride-1 3x3: the tile's input halo
      rc = encode_tmap_nhwc(&maps.a[i], pr.x, P.Cin, P.Wi, P.Hi, P.B, pr.x_ld, BK, P.tw + 2, P.th + 2, 1, 1);
    else if (P.a_mode == A_TMA4D)
      rc = encode_tmap_nhwc(&maps.a[i], pr.x, P.Cin, P.Wi, P.Hi, P.B, pr.x_ld, BK, P.tw * P.stride, P.th * P.stride, P.stride,
                            P.stride);
    if (rc) return rc;
    if (out_maps) {
      auto out_map = [&](CUtensorMap* m, const __half* base, long long ld) {
        return P.a_mode != A_TMA4D ? encode_tmap_2d(m, base, (uint64_t)P.N, (uint64_t)P.M, (uint64_t)ld * 2, 64, BM)
                                   : encode_tmap_nhwc(m, base, P.N, P.Wo, P.Ho, P.B, ld, 64, P.tw, P.th, 1, 1);
      };
      if ((rc = out_map(&maps.y[i], pr.y, pr.y_ld))) return rc;
      if (pr.res && (rc = out_map(&maps.res[i], pr.res, pr.res_ld))) return rc;
    }
  }
  if (n_io == 1) { maps.w[1] = maps.w[0]; maps.a[1] = maps.a[0]; maps.y[1] = maps.y[0]; maps.res[1] = maps.res[0]; }
  return ICAF_OK;
}

// Launch a planned conv on the kernel the plan picked (XM: the LayerNorm-fold / row-statistics instantiation).  Its
// shared-memory limit is raised once per device; the filter maps are encoded for the plan's tile width, and the output
// maps when the launch stores its tiles by TMA (P.tma_epi).
template <int BN>
static int launch_conv(const ConvParams& P, const ConvPlan& pl, const __half* const (&w)[2], const icaf_conv_geom* g, int n_io,
                       cudaStream_t st) {
  void (*kernel)(ConvParams, ConvMaps) = pl.xm ? conv_gemm_tc_kernel<BN, true> : conv_gemm_tc_kernel<BN, false>;
  if (pl.persist) kernel = pl.xm ? conv_gemm_persist_kernel<true> : conv_gemm_persist_kernel<false>;
  if (pl.stem) kernel = conv_stem_kernel;
  static bool configured[3][2][kMaxDevices] = {};
  const int family = pl.stem ? 2 : (pl.persist ? 1 : 0);
  if (int rc = configure_smem(kernel, 227 * 1024, configured[family][pl.xm], "conv2d: cudaFuncSetAttribute")) return rc;
  ConvMaps maps;
  if (int rc = encode_maps<BN>(P, w, g, n_io, P.tma_epi != 0, maps)) return rc;
  // the one-tile kernels take the tile grid (split-K: in clusters along x); the persistent one `ctas` CTAs
  const dim3 grid = pl.persist ? dim3(unsigned(pl.ctas)) : dim3(pl.grid_x, pl.grid_y, pl.grid_z);
  const int threads = pl.persist ? kPersistThreads : (pl.stem ? kStemThreads : kThreads);
  return launch_kc("conv2d_fwd", kernel, grid, dim3(threads), (size_t)pl.smem, st, pl.cluster, P, maps);
}

// ---------------------------------------------------------------------------------------------------
// The dispatcher, host only: staging mode, tile shape and tile width for one layer geometry.  No CUDA call.
// (`pair_mode` of icaf_conv2d_plan selects CTA-pair kernels on architectures that have them; sm_90a has none.)
// It also picks the epilogue (P.tma_epi): tma_out says whether TMA can write the outputs and read the residuals
// (16-byte aligned bases and row pitches).
static int plan_conv(const icaf_conv_geom* g, int n_io, int sms, bool tma_out, ConvParams& P, ConvPlan& pl) {
  memset(&pl, 0, sizeof(pl));
  pl.sms = sms;
  if (sms < 1) return set_error(ICAF_ERR_BAD_ARG, "conv2d: SM count must be positive");
  pl.xm = (P.epi & (ICAF_EPI_LN_FOLD | ICAF_EPI_EMIT_STATS)) != 0;
  plan_a_mode(g, P);
  // Tile width: the widest BN that still yields at least ~one CTA per SM; small problems take BN = 32 so that more SMs
  // share the K loop (and split it over clusters when even that leaves most SMs idle).
  const long long mt = P.a_mode == A_TMA4D ? (long long)P.B * P.tiles_x * P.tiles_y : (P.M + BM - 1) / BM;
  auto ctas = [&](int bn) { return mt * ((P.N + bn - 1) / bn) * n_io; };
  int bn = 32;
  if (P.N > 64 && ctas(128) >= sms) bn = 128;
  else if (P.N > 32 && ctas(64) >= sms) bn = 64;
  int rc;
  switch (bn) {
    case 128:
      rc = plan_tc<128>(P, n_io, pl);
      // the persistent kernel stores its non-XM tiles by TMA; a launch whose outputs TMA cannot write stays one-tile
      if (!rc && (pl.xm || tma_out) && P.a_mode != A_GATHER && P.splits == 1 && pl.tiles > sms) rc = plan_persist(P, pl);
      break;
    case 64:
      rc = plan_tc<64>(P, n_io, pl);
      // 16-channel stride-1 3x3 gather launches (the yolov5m/l image stems) run on conv_stem_kernel, whose epilogue is
      // the register one with a TMA store and has no residual
      if (!rc && !pl.xm && tma_out && P.a_mode == A_GATHER && P.splits == 1 && P.Cin == 16 && P.kh == 3 && P.kw == 3 &&
          P.stride == 1 && P.pad == 1 && !(P.epi & (ICAF_EPI_ADD_RES | ICAF_EPI_SCALED_RES))) {
        P.stages = 1;                                   // one filter load and one halo per tile, no ring
        pl.stem = true;
        pl.smem = StemLayout::total(P.Wo);
      }
      break;
    default: rc = plan_tc<32>(P, n_io, pl); break;
  }
  if (rc) return rc;
  // Register epilogue with TMA-stored output tiles: every persistent launch but XM; on the one-tile kernel also BN >= 64
  // without split-K (the leader reduces the cluster's staged rows).  The others keep the staged-row epilogue.
  P.tma_epi = !pl.xm && (pl.persist || (tma_out && P.splits == 1 && pl.bn >= 64)) ? 1 : 0;
  return ICAF_OK;
}

}  // namespace icaf

using namespace icaf;


extern "C" int icaf_conv2d_plan(const icaf_conv_geom* g, int n_io, int sm_count, int pair_mode, icaf_conv_plan* out) {
  if (!out) return set_error(ICAF_ERR_BAD_ARG, "conv2d_plan: null output");
  ConvParams P;
  int rc = fill_geom(g, n_io, P);
  if (rc) return rc;
  ConvPlan pl;
  (void)pair_mode;
  rc = plan_conv(g, n_io, sm_count, true, P, pl);
  if (rc) return rc;
  out->kernel = pl.kernel; out->bn = pl.bn; out->a_mode = P.a_mode;
  out->tile_w = P.tw; out->tile_h = P.th; out->tiles_x = P.tiles_x; out->tiles_y = P.tiles_y;
  out->cblk = P.cblk; out->halo = 0; out->stages = P.stages; out->splits = P.splits;
  out->grid_x = int(pl.grid_x); out->grid_y = int(pl.grid_y); out->grid_z = int(pl.grid_z); out->cluster = int(pl.cluster);
  out->smem_bytes = pl.smem; out->work_items = pl.tiles; out->ctas = pl.ctas;
  return ICAF_OK;
}

extern "C" int icaf_conv2d_fwd(const icaf_conv_geom* g, const icaf_conv_io* io, int n_io, void* stream) {
  ConvParams P;
  const __half* w[2];
  int rc = fill_params(g, io, n_io, P, w);
  if (rc) return rc;
  // TMA stores outputs (and loads residuals) from 16-byte aligned bases with 16-byte aligned row pitches
  bool tma_out = true;
  for (int i = 0; i < n_io; ++i) {
    const ConvProblem& pr = P.p[i];
    tma_out = tma_out && (reinterpret_cast<uintptr_t>(pr.y) & 15) == 0 && pr.y_ld % 8 == 0 &&
              (!pr.res || ((reinterpret_cast<uintptr_t>(pr.res) & 15) == 0 && pr.res_ld % 8 == 0));
  }
  ConvPlan pl;
  rc = plan_conv(g, n_io, sm_count_cached(), tma_out, P, pl);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  switch (pl.bn) {
    case 128: return launch_conv<128>(P, pl, w, g, n_io, st);
    case 64: return launch_conv<64>(P, pl, w, g, n_io, st);
    case 32: return launch_conv<32>(P, pl, w, g, n_io, st);
    default: return set_error(ICAF_ERR_BAD_ARG, "conv2d: the planner produced an unknown tile width");
  }
}

extern "C" int icaf_conv2d_fwd_simt(const icaf_conv_geom* g, const icaf_conv_io* io, int n_io, void* stream) {
  SimtParams S;
  int rc = fill_params(g, io, n_io, S.P, S.w);
  if (rc) return rc;
  long long total = (long long)S.P.M * S.P.N;
  dim3 grid(blocks_for(total, 256), 1, n_io);
  return launch_k("conv2d_fwd_simt", conv_gemm_simt_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream, S);
}
