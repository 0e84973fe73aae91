// Bidirectional DMFF cross-attention core (models/common.py:670-684) as a flash-style wgmma kernel:
//   out_vis = softmax(q_ir k_vis^T / sqrt(d)) v_vis        out_ir = softmax(q_vis k_ir^T / sqrt(d)) v_ir
// The N x N score matrix never leaves the SM: each of two consumer warpgroups owns 64 query rows, computes S = Q K^T
// into registers (wgmma, both operands in shared memory), runs the online softmax on the accumulator fragments, packs P
// to fp16 in registers and feeds it straight back as the A operand of O += P V (wgmma with a register A operand); running
// (max, sum, O) live in registers.  Q / K / V tiles are staged by TMA (cp.async.bulk.tensor) from a producer warp, K / V
// double-buffered.
//
// Layouts (see include/icaf_b200.h): either qkv (B, Npad, 3C) = [q | k | v] rows as ONE fused projection emits them (V is
// then consumed as an MN-major operand straight from its token-major tile), or qk (B, Npad, 2C) + vt (C, B*Npad) = V^T
// (K-major); out (B, Npad, C).
// CTA = (128-query tile, batch*head, direction).
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "icaf_internal.cuh"

namespace icaf {

constexpr int kQT = 128;    // queries per CTA (two warpgroups x 64 rows)

struct AttnParams {
  const __half* qk[2];   // [0]=vis, [1]=ir
  const __half* vt[2];   // NULL in the fused-qkv form
  __half* out[2];
  int B, N, n_pad, C, heads;
  int d;                 // head dim C / heads (the kernel runs width D >= d)
  int ld;                // row pitch of qk: 2C, or 3C in the fused-qkv form ([q | k | v])
  float p_drop;          // training forward only (TRAIN instantiation): dropout on the probabilities (common.py:677,680)
  uint32_t seed;
  const uint32_t* seed_off;   // optional device-side offset (icaf_set_seed_offset)
  float scale_log2;      // log2(e) / sqrt(d)
};

// ---------------------------------------------------------------------------------------------------
// 288 threads: warps 0-7 two consumer warpgroups (queries 0-63 / 64-127 of the tile), warp 8 TMA producer.
// A head dim d (any multiple of 8 up to 128) runs the kernel of width D = 16 / 32 / 64 / 128, the smallest >= d; d = 160
// runs its own width D = 160.  Every tile comes through a 3-D map that gives each head its own extent of d columns:
//   Q / K tiles: (d, k*heads, B*Npad) view of the projection matrix (k = 2 split, 3 fused), box (W, 1, rows) with
//                W = min(D, 64), or 32 at D = 160 -> K-major rows of 32 / 64 / 128 bytes with the matching swizzle, D / W
//                column blocks (D = 128: two 64-column blocks; D = 160: five 32-column blocks, 64-byte rows)
//   V tiles    : (VF, fused [q|k|v] rows) boxes like K's at projection 2 -> rows = keys, i.e. an MN-major B operand
//   V^T tiles  : (B*Npad, d, heads) view of the (C, B*Npad) matrix, box (64, D, 1) -> K-major SW128 (keys are the K dim
//                of PV)
// Columns d .. D-1, rows past the tensor and keys past the tensor are zero-filled by the TMA unit; keys in [N, ...) are
// masked in the softmax.  The zero columns add exactly 0 to S = Q K^T and produce zero columns of O = P V, which are not
// stored.
struct AttnMaps {
  CUtensorMap qk[2];   // [0] = vis, [1] = ir : box (W, 1, 128) -- Q tiles
  CUtensorMap kv[2];   // same views, box (W, 1, KV) -- K tiles (and V tiles in the fused form)
  CUtensorMap vt[2];   // split form: V^T view, box (64, D, 1)
};

// KV = keys per tile (N of S, K of PV).  Head dims up to 32 run 64-key tiles (less masked work at the DMFF token counts).
// The dropout kernel at D = 128 spills 48 bytes with 128-key tiles; 64-key tiles would change the rounding of yolov5l's
// P5 training attention (d = 128).  D = 160 runs 64-key tiles: with 128 its 80 accumulator registers, S and P spill
// 256 bytes under the 168-register cap of 288 threads.
template <int D>
struct AttnCfg {
  static constexpr int kKV = D <= 32 || D == 160 ? 64 : 128;
};

template <int D, int KV>
struct AttnSmemT {
  // head-dim columns per TMA box and staged row: 160 = 5 x 32 keeps one swizzle mode (64 B) across the whole head, so
  // P V runs as one N = 160 wgmma on a uniform MN-major V tile
  static constexpr int kBoxW = D % 64 == 0 ? 64 : (D >= 32 ? 32 : D);
  static constexpr int kKB = D / kBoxW;                     // column blocks of the head dim
  static constexpr int kRowB = kBoxW * 2;                   // bytes per staged Q / K row (= swizzle span)
  static constexpr int kKS = kRowB / 32;                    // k16 steps per column block
  static constexpr int kQBytes = kKB * kQT * kRowB;
  static constexpr int kKBytes = kKB * KV * kRowB;          // per buffer
  static constexpr int kVBytes = (KV / 64) * D * 128;       // per buffer: 64-key blocks of D rows (= KV rows of D halfs)
  static constexpr int kQOff = 0;
  static constexpr int kKOff = kQOff + kQBytes;
  static constexpr int kVOff = kKOff + 2 * kKBytes;
  static constexpr int kBarOff = kVOff + 2 * kVBytes;
  static constexpr int kTotal = kBarOff + 128 + 1024;       // + alignment slack
  static_assert(D % kBoxW == 0 && kBoxW % 16 == 0, "the head dim must split into whole column blocks of k16 steps");
  static_assert(kQBytes % 1024 == 0 && kKBytes % 1024 == 0 && kVBytes % 1024 == 0, "tiles must keep 1024-byte alignment");
};

__device__ __forceinline__ float fast_exp2_t(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Barrier waits of the width-D kernel.  D = 160 waits without the deadlock report (mbar_wait_quiet): a printf reachable
// anywhere in a kernel makes ptxas serialise all of its wgmmas (warning C7510).  The other widths keep the reporting wait.
template <int D>
__device__ __forceinline__ void attn_wait(uint32_t bar, uint32_t parity) {
  if constexpr (D == 160) mbar_wait_quiet(bar, parity);
  else mbar_wait(bar, parity);
}

// TRAIN: dropout on the attention probabilities (the row sum still runs over the un-dropped values, like
// `att = softmax(..); att = attn_drop(att)`); its own instantiation, so the inference kernels keep their size.
template <int D, bool VF, bool TRAIN = false>
__global__ void __launch_bounds__(288, 1) cross_attn_tma_kernel(const AttnParams P, const __grid_constant__ AttnMaps M) {
  constexpr int kKV = AttnCfg<D>::kKV;
  using L = AttnSmemT<D, kKV>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar = sbase + L::kBarOff;
  const uint32_t q_full = bar;
  auto kv_full = [&](int i) { return bar + 32u + 8u * i; };
  auto kv_empty = [&](int i) { return bar + 48u + 8u * i; };

  pdl_launch_dependents();
  const int tid = threadIdx.x, warp = tid >> 5;
  const int dir = blockIdx.z;                 // 0: out_vis (q_ir, k_vis, v_vis)   1: out_ir (q_vis, k_ir, v_ir)
  const int b = blockIdx.y / P.heads, head = blockIdx.y % P.heads;
  const int q0 = blockIdx.x * kQT;
  const int C = P.C, N = P.N, n_pad = P.n_pad;
  const int nkv = (N + kKV - 1) / kKV;

  if (tid == 0) {
    mbar_init(q_full, 1);
    mbar_init(kv_full(0), 1); mbar_init(kv_full(1), 1);
    mbar_init(kv_empty(0), 8); mbar_init(kv_empty(1), 8);      // one arrival per consumer warp
    fence_mbar_init();
  }
  if (warp == 8 && lane_id() == 0) {
    tma_prefetch_desc(dir == 0 ? &M.qk[1] : &M.qk[0]);
    tma_prefetch_desc(dir == 0 ? &M.kv[0] : &M.kv[1]);
    if (!VF) tma_prefetch_desc(dir == 0 ? &M.vt[0] : &M.vt[1]);
  }
  __syncthreads();
  pdl_wait();           // everything above overlapped the previous kernel's tail; q/k/v are its outputs

  if (warp < 8) {
    // ------------------------------------------------------------------ consumer warpgroup g: query rows 64g .. 64g+63
    const int g = warp >> 2, w = warp & 3, l = tid & 31;
    const int r_lo = 64 * g + 16 * w + (l >> 2);              // this thread's two rows: r_lo, r_lo + 8
    const int qn0 = q0 + r_lo, qn1 = qn0 + 8;
    const float sl2 = P.scale_log2;
    const uint32_t seed = TRAIN ? P.seed + (P.seed_off ? __ldg(P.seed_off) : 0u) : 0u;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    float o[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
    attn_wait<D>(q_full, 0);
    for (int j = 0; j < nkv; ++j) {
      const int buf = j & 1;
      const int kv0 = j * kKV;
      attn_wait<D>(kv_full(buf), (j >> 1) & 1);
      // ---- S = Q K^T (64 x KV per warpgroup) ----
      float s[kKV / 2];
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < D / 16; ++k) {
        const int kb = k / L::kKS, ko = (k % L::kKS) * 32;    // column block, byte offset of the k16 step in its rows
        const uint64_t ad = gmma_desc_kmajor(sbase + L::kQOff + kb * (kQT * L::kRowB) + 64 * g * L::kRowB + ko, L::kRowB);
        const uint64_t bd = gmma_desc_kmajor(sbase + L::kKOff + buf * L::kKBytes + kb * (kKV * L::kRowB) + ko, L::kRowB);
        wgmma_ss<0, 0>(s, ad, bd, k != 0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      // ---- online softmax on the fragments: s[i] is row r_lo + 8*((i>>1)&1), key kv0 + 8*(i>>2) + 2*(l&3) + (i&1) ----
      const bool full = kv0 + kKV <= N;       // every key of the tile is valid: no masking
      if (!full) {
#pragma unroll
        for (int i = 0; i < kKV / 2; ++i)
          if (kv0 + 8 * (i >> 2) + 2 * (l & 3) + (i & 1) >= N) s[i] = -INFINITY;
      }
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int i = 0; i < kKV / 2; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], s[i]);
      float corr[2], moff[2], rs[2] = {0.f, 0.f};
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));   // the four threads of a row agree
        const float m_new = fmaxf(m_run[h], mx[h]);                      // finite: every tile has >= 1 valid key
        corr[h] = fast_exp2_t((m_run[h] - m_new) * sl2);
        moff[h] = m_new * sl2;
        m_run[h] = m_new;
      }
      uint32_t pa[kKV / 16][4];                 // P as the register A operand of the PV wgmma, one set per 16 keys
#pragma unroll
      for (int i = 0; i < kKV / 2; i += 2) {
        const int h = (i >> 1) & 1;
        const float p0 = fast_exp2_t(fmaf(s[i], sl2, -moff[h]));       // exp2(-inf) = 0 for the masked keys
        const float p1 = fast_exp2_t(fmaf(s[i + 1], sl2, -moff[h]));
        __half2 hp = __floats2half2_rn(p0, p1);
        const float2 hf = __half22float2(hp);            // sum what the PV MMA will actually see
        rs[h] += hf.x + hf.y;
        if (TRAIN) {
          const float ks = 1.f / (1.f - P.p_drop);
          const int qn = h ? qn1 : qn0, key = kv0 + 8 * (i >> 2) + 2 * (l & 3);
          const bool k0 = attn_keep(seed, dir, blockIdx.y, qn, key, P.p_drop), k1 = attn_keep(seed, dir, blockIdx.y, qn, key + 1, P.p_drop);
          hp = __floats2half2_rn(k0 ? hf.x * ks : 0.f, k1 ? hf.y * ks : 0.f);
        }
        pa[i >> 3][(i >> 1) & 3] = *reinterpret_cast<const uint32_t*>(&hp);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) l_run[h] = l_run[h] * corr[h] + rs[h];   // per-thread partial sums; reduced at the end
#pragma unroll
      for (int i = 0; i < D / 2; ++i) o[i] *= corr[(i >> 1) & 1];
      // ---- O += P V ----
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kKV / 16; ++k) {
        if (VF) {
          wgmma_rs<1>(o, pa[k], gmma_desc_mnmajor(sbase + L::kVOff + buf * L::kVBytes + k * 16 * L::kRowB, L::kRowB, kKV * L::kRowB), true);
        } else {
          wgmma_rs<0>(o, pa[k], gmma_desc_sw128(sbase + L::kVOff + buf * L::kVBytes + (k >> 2) * (D * 128) + (k & 3) * 32), true);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      if (l == 0) mbar_arrive(kv_empty(buf));
    }
    // ---- normalise and store (heads merged: column head*d) ; zero the pad rows ----
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 1);
      l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 2);
    }
    const int d = P.d;                        // true head dim: columns d .. D-1 of o are the zero padding
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int qn = h ? qn1 : qn0;
      if (qn < n_pad) {
        const float inv = qn < N ? 1.f / l_run[h] : 0.f;
        __half* op = (dir == 0 ? P.out[0] : P.out[1]) + (size_t(b) * n_pad + qn) * C + head * d + 2 * (l & 3);
#pragma unroll
        for (int i = 2 * h; i < D / 2; i += 4)
          if (8 * (i >> 2) < d)
            *reinterpret_cast<uint32_t*>(op + 8 * (i >> 2)) = pack_half2(o[i] * inv, o[i + 1] * inv);
      }
    }
  } else if (lane_id() == 0) {
    // ------------------------------------------------------------------ TMA producer (one thread)
    const CUtensorMap* mq = dir == 0 ? &M.qk[1] : &M.qk[0];
    const CUtensorMap* mk = dir == 0 ? &M.kv[0] : &M.kv[1];
    const CUtensorMap* mv = dir == 0 ? &M.vt[0] : &M.vt[1];
    const int row_b = b * n_pad;
    // a tile = (column block kb of projection k's head `head`, rows r0 ..)
    auto load_tile = [&](uint32_t dst, const CUtensorMap* m, uint32_t bar, int k, int kb, int r0) {
      tma_load_3d(dst, m, bar, kb * L::kBoxW, k * P.heads + head, r0);
    };
    mbar_arrive_expect_tx(q_full, L::kQBytes);      // overhanging boxes count in full: the zero fill arrives as bytes too
#pragma unroll
    for (int kb = 0; kb < L::kKB; ++kb)
      load_tile(sbase + L::kQOff + kb * (kQT * L::kRowB), mq, q_full, 0, kb, row_b + q0);
    for (int j = 0; j < nkv; ++j) {
      const int buf = j & 1;
      if (j >= 2) attn_wait<D>(kv_empty(buf), ((j >> 1) & 1) ^ 1);     // PV(j-2) has drained this buffer
      mbar_arrive_expect_tx(kv_full(buf), L::kKBytes + L::kVBytes);
#pragma unroll
      for (int kb = 0; kb < L::kKB; ++kb)
        load_tile(sbase + L::kKOff + buf * L::kKBytes + kb * (kKV * L::kRowB), mk, kv_full(buf), 1, kb, row_b + j * kKV);
      if (VF) {
#pragma unroll
        for (int kb = 0; kb < L::kKB; ++kb)
          load_tile(sbase + L::kVOff + buf * L::kVBytes + kb * (kKV * L::kRowB), mk, kv_full(buf), 2, kb, row_b + j * kKV);
      } else {
#pragma unroll
        for (int kb = 0; kb < kKV / 64; ++kb)
          tma_load_3d(sbase + L::kVOff + buf * L::kVBytes + kb * (D * 128), mv, kv_full(buf), row_b + j * kKV + kb * 64, 0, head);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// CUDA-core reference, one thread per (query, head, batch, direction). Tests only.
__global__ void cross_attn_simt_kernel(const AttnParams P) {
  pdl_launch_dependents();
  pdl_wait();
  const int d = P.C / P.heads;
  long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  long long total = 2LL * P.B * P.heads * P.n_pad;
  if (idx >= total) return;
  int qn = int(idx % P.n_pad);
  long long t = idx / P.n_pad;
  int head = int(t % P.heads); t /= P.heads;
  int b = int(t % P.B);
  int dir = int(t / P.B);
  const __half* qsrc = dir == 0 ? P.qk[1] : P.qk[0];
  const __half* ksrc = dir == 0 ? P.qk[0] : P.qk[1];
  const __half* vsrc = dir == 0 ? P.vt[0] : P.vt[1];
  __half* o = (dir == 0 ? P.out[0] : P.out[1]) + (size_t(b) * P.n_pad + qn) * P.C + head * d;
  if (qn >= P.N) {
    for (int i = 0; i < d; ++i) o[i] = __float2half(0.f);
    return;
  }
  const __half* q = qsrc + (size_t(b) * P.n_pad + qn) * P.ld + head * d;
  float mx = -INFINITY;
  for (int k = 0; k < P.N; ++k) {
    const __half* kp = ksrc + (size_t(b) * P.n_pad + k) * P.ld + P.C + head * d;
    float s = 0.f;
    for (int i = 0; i < d; ++i) s += __half2float(q[i]) * __half2float(kp[i]);
    mx = fmaxf(mx, s);
  }
  float l = 0.f;
  float acc[128];
  for (int i = 0; i < d; ++i) acc[i] = 0.f;
  for (int k = 0; k < P.N; ++k) {
    const __half* kp = ksrc + (size_t(b) * P.n_pad + k) * P.ld + P.C + head * d;
    float s = 0.f;
    for (int i = 0; i < d; ++i) s += __half2float(q[i]) * __half2float(kp[i]);
    float p = exp2f((s - mx) * P.scale_log2);
    l += p;
    for (int i = 0; i < d; ++i)
      acc[i] += p * __half2float(vsrc ? vsrc[size_t(head * d + i) * (size_t(P.B) * P.n_pad) + size_t(b) * P.n_pad + k]
                                      : kp[P.C + i]);                     // fused form: v sits one C further in the key's row
  }
  for (int i = 0; i < d; ++i) o[i] = __float2half_rn(acc[i] / l);
}

// d160: the caller has a kernel for head dim 160 (the tensor-core forward; not the CUDA-core or dropout kernels)
static int fill_attn(const void* qk_vis, const void* qk_ir, const void* vt_vis, const void* vt_ir, void* out_vis,
                     void* out_ir, int B, int N, int n_pad, int C, int heads, AttnParams& P, bool d160 = false) {
  // vt_* both NULL: the fused form, qk_* are (B, Npad, 3C) [q | k | v] matrices
  if (!qk_vis || !qk_ir || (!vt_vis != !vt_ir) || !out_vis || !out_ir) return set_error(ICAF_ERR_BAD_ARG, "cross_attention: null pointer");
  if (B < 1 || N < 1 || n_pad < N || n_pad % 8 || heads < 1 || C % heads) return set_error(ICAF_ERR_BAD_ARG, "cross_attention: bad shape");
  int d = C / heads;
  if (d % 8 || d < 8 || (d > 128 && !(d160 && d == 160)))
    return set_error(ICAF_ERR_UNSUPPORTED, d160 ? "cross_attention: head dim must be a multiple of 8 in [8, 128], or 160"
                                                : "cross_attention: head dim must be a multiple of 8 in [8, 128]");
  P.qk[0] = (const __half*)qk_vis; P.qk[1] = (const __half*)qk_ir;
  P.vt[0] = (const __half*)vt_vis; P.vt[1] = (const __half*)vt_ir;
  P.out[0] = (__half*)out_vis; P.out[1] = (__half*)out_ir;
  P.B = B; P.N = N; P.n_pad = n_pad; P.C = C; P.heads = heads; P.d = d;
  P.ld = vt_vis ? 2 * C : 3 * C;
  P.p_drop = 0.f; P.seed = 0u; P.seed_off = nullptr;
  P.scale_log2 = 1.4426950408889634f / sqrtf(float(d));   // 1/sqrt(d_k), common.py:670
  return ICAF_OK;
}

template <int D, bool VF, bool TRAIN = false>
static int launch_attn_tma(const AttnParams& P, cudaStream_t st) {
  constexpr int kKV = AttnCfg<D>::kKV;
  using L = AttnSmemT<D, kKV>;
  static bool configured[kMaxDevices] = {false};
  if (int rc = configure_smem(cross_attn_tma_kernel<D, VF, TRAIN>, L::kTotal, configured, "cross_attention: cudaFuncSetAttribute")) return rc;
  AttnMaps maps;
  memset(&maps, 0, sizeof(maps));
  const uint64_t rows = uint64_t(P.B) * P.n_pad;
  const uint64_t d = uint64_t(P.d);
  const uint32_t bw = L::kBoxW;
  const uint64_t dims[3] = {d, uint64_t(P.ld / d), rows};       // (head column, projection * heads + head, token)
  const uint64_t vdims[3] = {rows, d, uint64_t(P.heads)};       // (token, head row, head)
  for (int i = 0; i < 2; ++i) {
    int rc = encode_tmap_3d(&maps.qk[i], P.qk[i], dims, d * 2, uint64_t(P.ld) * 2, {bw, 1u, uint32_t(kQT)});
    if (!rc) rc = encode_tmap_3d(&maps.kv[i], P.qk[i], dims, d * 2, uint64_t(P.ld) * 2, {bw, 1u, uint32_t(kKV)});
    if (!rc && !VF) rc = encode_tmap_3d(&maps.vt[i], P.vt[i], vdims, rows * 2, rows * 2 * d, {64u, uint32_t(D), 1u});
    if (rc) return rc;
  }
  dim3 grid(blocks_for(P.n_pad, kQT), P.B * P.heads, 2);
  return launch_k("cross_attention", cross_attn_tma_kernel<D, VF, TRAIN>, dim3(grid), dim3(288), L::kTotal, st, P, maps);
}

// A head dim d up to 128 runs the kernel of the smallest width D >= d; columns d .. D-1 are zero-filled (see AttnMaps).
// d = 160 (yolov5x's P5 block) runs at its exact width: padded to 256 it would cost 60 % more MMA work and a 128-register
// accumulator.  It has no dropout instantiation: the training entry point refuses it (there is no backward either).
template <bool VF, bool TRAIN = false>
static int dispatch_attn(const AttnParams& P, cudaStream_t st) {
  const int d = P.d;
  if (d <= 16) return launch_attn_tma<16, VF, TRAIN>(P, st);
  if (d <= 32) return launch_attn_tma<32, VF, TRAIN>(P, st);
  if (d <= 64) return launch_attn_tma<64, VF, TRAIN>(P, st);
  if (d <= 128) return launch_attn_tma<128, VF, TRAIN>(P, st);
  if constexpr (!TRAIN) {
    if (d == 160) return launch_attn_tma<160, VF>(P, st);
  }
  return set_error(ICAF_ERR_UNSUPPORTED, "cross_attention: no kernel for this head dim");
}

}  // namespace icaf

using namespace icaf;

extern "C" int icaf_cross_attention(const void* qk_vis, const void* qk_ir, const void* vt_vis, const void* vt_ir,
                                    void* out_vis, void* out_ir, int B, int N, int n_pad, int C, int heads, void* stream) {
  AttnParams P;
  int rc = fill_attn(qk_vis, qk_ir, vt_vis, vt_ir, out_vis, out_ir, B, N, n_pad, C, heads, P, true);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if ((uint64_t(B) * n_pad * 2) % 16 || (reinterpret_cast<uintptr_t>(vt_vis) & 15) || (reinterpret_cast<uintptr_t>(qk_vis) & 15) ||
      (reinterpret_cast<uintptr_t>(vt_ir) & 15) || (reinterpret_cast<uintptr_t>(qk_ir) & 15))
    return set_error(ICAF_ERR_BAD_ARG, "cross_attention: TMA needs 16-byte aligned tensors and row pitches");
  return vt_vis ? dispatch_attn<false>(P, st) : dispatch_attn<true>(P, st);
}

extern "C" int icaf_cross_attention_train(const void* qkv_vis, const void* qkv_ir, void* out_vis, void* out_ir, int B, int N, int n_pad, int C, int heads,
                                          float p_drop, uint32_t seed, void* stream) {
  AttnParams P;
  int rc = fill_attn(qkv_vis, qkv_ir, nullptr, nullptr, out_vis, out_ir, B, N, n_pad, C, heads, P);
  if (rc) return rc;
  if (!(p_drop >= 0.f && p_drop < 1.f)) return set_error(ICAF_ERR_BAD_ARG, "cross_attention_train: dropout probability must be in [0, 1)");
  if ((uint64_t(B) * n_pad * 2) % 16 || (reinterpret_cast<uintptr_t>(qkv_vis) & 15) || (reinterpret_cast<uintptr_t>(qkv_ir) & 15))
    return set_error(ICAF_ERR_BAD_ARG, "cross_attention_train: TMA needs 16-byte aligned tensors and row pitches");
  P.p_drop = p_drop; P.seed = seed; P.seed_off = seed_offset_ptr();
  cudaStream_t st = (cudaStream_t)stream;
  return p_drop == 0.f ? dispatch_attn<true>(P, st) : dispatch_attn<true, true>(P, st);
}

extern "C" int icaf_cross_attention_simt(const void* qk_vis, const void* qk_ir, const void* vt_vis, const void* vt_ir,
                                         void* out_vis, void* out_ir, int B, int N, int n_pad, int C, int heads,
                                         void* stream) {
  AttnParams P;
  int rc = fill_attn(qk_vis, qk_ir, vt_vis, vt_ir, out_vis, out_ir, B, N, n_pad, C, heads, P);
  if (rc) return rc;
  long long total = 2LL * B * heads * n_pad;
  return launch_k("cross_attention_simt", cross_attn_simt_kernel, dim3(blocks_for(total, 128)), dim3(128), 0, (cudaStream_t)stream, P);
}
