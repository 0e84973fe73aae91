// Backward of the bidirectional DMFF cross-attention (models/common.py:670-684) with recompute, CUDA cores.
//   P = softmax(scale Q K^T), Pd = dropout(P), O = Pd V          (Q from the OTHER modality: common.py:670)
//   dV = Pd^T dO;  dPd = dO V^T;  dS = P o (mask/(1-p) o dPd - delta), delta_i = dO_i . O_i;  dQ = scale dS K;  dK = scale dS^T Q
// Two kernels per call, both tiled through shared memory, one thread per query (kernel Q) / per key (kernel KV); head dims
// <= 64 take the register-resident variants further down, 128 the shared-memory ones:
//   attn_bwd_q_kernel : row max / sum (recomputed, written to `stats` for the second kernel), dQ
//   attn_bwd_kv_kernel: dK, dV (channel accumulators in registers, 64 channels per pass)
// Inputs are the fused projection rows [q | k | v] (B, Npad, 3C) of both modalities, the forward outputs O and their
// gradients dO (B, Npad, C); outputs are d[q|k|v] in the same layout.  No atomics: deterministic.
// This is the pooled-token regime's kernel (N <= a few hundred); a tensor-core version is the next step.
#include "icaf_internal.cuh"

namespace icaf {

struct AttnBwdParams {
  const __half* qkv[2]; const __half* o[2]; const __half* dout[2];
  __half* dqkv[2];
  float* stats;            // [2 dir][B][heads][Npad][2] = (row max of scale*S in log2 units, 1 / row sum)
  int B, N, n_pad, C, heads;
  float scale_log2, scale, p_drop;
  uint32_t seed;
  const uint32_t* seed_off;   // optional device-side offset (icaf_set_seed_offset)
};

constexpr int kBT = 128;   // rows (queries or keys) per block
constexpr int kTT = 32;    // rows of the other side staged per tile

template <int D>
__global__ void __launch_bounds__(kBT) attn_bwd_q_kernel(const AttnBwdParams P) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ __half sm_h[];
  __half* qT = sm_h;                  // [D][kBT]
  __half* dT = qT + D * kBT;          // [D][kBT]  dO
  __half* kt = dT + D * kBT;          // [kTT][D]
  __half* vt = kt + kTT * D;          // [kTT][D]
  const int dir = blockIdx.z, bh = blockIdx.y, b = bh / P.heads, head = bh % P.heads;
  const int i = blockIdx.x * kBT + threadIdx.x;
  const int ld = 3 * P.C;
  const __half* qsrc = (dir == 0 ? P.qkv[1] : P.qkv[0]) + size_t(b) * P.n_pad * ld + head * D;          // queries of the other modality
  const __half* ksrc = (dir == 0 ? P.qkv[0] : P.qkv[1]) + size_t(b) * P.n_pad * ld + P.C + head * D;
  const __half* vsrc = ksrc + P.C;
  const __half* osrc = (dir == 0 ? P.o[0] : P.o[1]) + size_t(b) * P.n_pad * P.C + head * D;
  const __half* dsrc = (dir == 0 ? P.dout[0] : P.dout[1]) + size_t(b) * P.n_pad * P.C + head * D;
  const bool valid = i < P.N;
  float delta = 0.f;
  for (int c = 0; c < D; ++c) {
    const __half qv = valid ? qsrc[size_t(i) * ld + c] : __float2half(0.f);
    const __half dv = valid ? dsrc[size_t(i) * P.C + c] : __float2half(0.f);
    qT[c * kBT + threadIdx.x] = qv;
    dT[c * kBT + threadIdx.x] = dv;
    if (valid) delta += __half2float(dv) * __half2float(osrc[size_t(i) * P.C + c]);
  }
  // pass 1: row max and sum
  float m = -INFINITY, l = 0.f;
  for (int j0 = 0; j0 < P.N; j0 += kTT) {
    __syncthreads();
    for (int e = threadIdx.x; e < kTT * D; e += kBT) {
      const int j = j0 + e / D, c = e % D;
      kt[e] = j < P.N ? ksrc[size_t(j) * ld + c] : __float2half(0.f);
    }
    __syncthreads();
    const int jn = min(kTT, P.N - j0);
    for (int j = 0; j < jn; ++j) {
      float s = 0.f;
#pragma unroll 8
      for (int c = 0; c < D; ++c) s += __half2float(qT[c * kBT + threadIdx.x]) * __half2float(kt[j * D + c]);
      s *= P.scale_log2;
      const float mn = fmaxf(m, s);
      l = l * exp2f(m - mn) + exp2f(s - mn);
      m = mn;
    }
  }
  const float inv_l = 1.f / l;
  if (valid) {
    float* st = P.stats + ((size_t(dir) * P.B * P.heads + bh) * P.n_pad + i) * 2;
    st[0] = m; st[1] = inv_l;
  }
  // pass 2: dQ
  float dq[D];
#pragma unroll
  for (int c = 0; c < D; ++c) dq[c] = 0.f;
  const float keep_scale = 1.f / (1.f - P.p_drop);
  for (int j0 = 0; j0 < P.N; j0 += kTT) {
    __syncthreads();
    for (int e = threadIdx.x; e < kTT * D; e += kBT) {
      const int j = j0 + e / D, c = e % D;
      kt[e] = j < P.N ? ksrc[size_t(j) * ld + c] : __float2half(0.f);
      vt[e] = j < P.N ? vsrc[size_t(j) * ld + c] : __float2half(0.f);
    }
    __syncthreads();
    const int jn = min(kTT, P.N - j0);
    for (int j = 0; j < jn; ++j) {
      float s = 0.f, dp = 0.f;
#pragma unroll 8
      for (int c = 0; c < D; ++c) {
        s += __half2float(qT[c * kBT + threadIdx.x]) * __half2float(kt[j * D + c]);
        dp += __half2float(dT[c * kBT + threadIdx.x]) * __half2float(vt[j * D + c]);
      }
      const float p = exp2f(s * P.scale_log2 - m) * inv_l;
      if (P.p_drop > 0.f) dp = attn_keep(P.seed + (P.seed_off ? __ldg(P.seed_off) : 0u), dir, bh, i, j0 + j, P.p_drop) ? dp * keep_scale : 0.f;
      const float ds = p * (dp - delta) * P.scale;
#pragma unroll
      for (int c = 0; c < D; ++c) dq[c] += ds * __half2float(kt[j * D + c]);
    }
  }
  if (i < P.n_pad) {
    __half* dst = (dir == 0 ? P.dqkv[1] : P.dqkv[0]) + (size_t(b) * P.n_pad + i) * ld + head * D;
#pragma unroll
    for (int c = 0; c < D; c += 2) *reinterpret_cast<__half2*>(dst + c) = valid ? __floats2half2_rn(dq[c], dq[c + 1]) : __floats2half2_rn(0.f, 0.f);
  }
}

template <int D>
__global__ void __launch_bounds__(kBT) attn_bwd_kv_kernel(const AttnBwdParams P) {
  pdl_launch_dependents();
  pdl_wait();
  constexpr int DH = D < 64 ? D : 64;       // channel accumulators per pass
  extern __shared__ __half sm_h[];
  __half* kT = sm_h;                  // [D][kBT]
  __half* vT = kT + D * kBT;          // [D][kBT]
  __half* qt = vT + D * kBT;          // [kTT][D]
  __half* dt = qt + kTT * D;          // [kTT][D]  dO
  float* st = reinterpret_cast<float*>(dt + kTT * D);      // [kTT][3] = m, 1/l, delta
  const int dir = blockIdx.z, bh = blockIdx.y, b = bh / P.heads, head = bh % P.heads;
  const int j = blockIdx.x * kBT + threadIdx.x;
  const int ld = 3 * P.C;
  const __half* qsrc = (dir == 0 ? P.qkv[1] : P.qkv[0]) + size_t(b) * P.n_pad * ld + head * D;
  const __half* ksrc = (dir == 0 ? P.qkv[0] : P.qkv[1]) + size_t(b) * P.n_pad * ld + P.C + head * D;
  const __half* vsrc = ksrc + P.C;
  const __half* osrc = (dir == 0 ? P.o[0] : P.o[1]) + size_t(b) * P.n_pad * P.C + head * D;
  const __half* dsrc = (dir == 0 ? P.dout[0] : P.dout[1]) + size_t(b) * P.n_pad * P.C + head * D;
  const float* stats = P.stats + (size_t(dir) * P.B * P.heads + bh) * P.n_pad * 2;
  const bool valid = j < P.N;
  for (int c = 0; c < D; ++c) {
    kT[c * kBT + threadIdx.x] = valid ? ksrc[size_t(j) * ld + c] : __float2half(0.f);
    vT[c * kBT + threadIdx.x] = valid ? vsrc[size_t(j) * ld + c] : __float2half(0.f);
  }
  const float keep_scale = 1.f / (1.f - P.p_drop);
  __half* dstk = (dir == 0 ? P.dqkv[0] : P.dqkv[1]) + (size_t(b) * P.n_pad + j) * ld + P.C + head * D;
  __half* dstv = dstk + P.C;
  for (int c0 = 0; c0 < D; c0 += DH) {
    float dk[DH], dv[DH];
#pragma unroll
    for (int c = 0; c < DH; ++c) dk[c] = dv[c] = 0.f;
    for (int i0 = 0; i0 < P.N; i0 += kTT) {
      __syncthreads();
      for (int e = threadIdx.x; e < kTT * D; e += kBT) {
        const int i = i0 + e / D, c = e % D;
        qt[e] = i < P.N ? qsrc[size_t(i) * ld + c] : __float2half(0.f);
        dt[e] = i < P.N ? dsrc[size_t(i) * P.C + c] : __float2half(0.f);
      }
      if (threadIdx.x < kTT) {
        const int i = i0 + threadIdx.x;
        float dl = 0.f;
        if (i < P.N)
          for (int c = 0; c < D; ++c) dl += __half2float(dsrc[size_t(i) * P.C + c]) * __half2float(osrc[size_t(i) * P.C + c]);
        st[threadIdx.x * 3] = i < P.N ? stats[size_t(i) * 2] : 0.f;
        st[threadIdx.x * 3 + 1] = i < P.N ? stats[size_t(i) * 2 + 1] : 0.f;
        st[threadIdx.x * 3 + 2] = dl;
      }
      __syncthreads();
      const int in_ = min(kTT, P.N - i0);
      for (int i = 0; i < in_; ++i) {
        float s = 0.f, dp = 0.f;
#pragma unroll 8
        for (int c = 0; c < D; ++c) {
          s += __half2float(qt[i * D + c]) * __half2float(kT[c * kBT + threadIdx.x]);
          dp += __half2float(dt[i * D + c]) * __half2float(vT[c * kBT + threadIdx.x]);
        }
        const float p = exp2f(s * P.scale_log2 - st[i * 3]) * st[i * 3 + 1];
        float pd = p;
        if (P.p_drop > 0.f) {
          const bool keep = attn_keep(P.seed + (P.seed_off ? __ldg(P.seed_off) : 0u), dir, bh, i0 + i, j, P.p_drop);
          pd = keep ? p * keep_scale : 0.f;
          dp = keep ? dp * keep_scale : 0.f;
        }
        const float ds = p * (dp - st[i * 3 + 2]) * P.scale;
#pragma unroll
        for (int c = 0; c < DH; ++c) {
          dk[c] += ds * __half2float(qt[i * D + c0 + c]);
          dv[c] += pd * __half2float(dt[i * D + c0 + c]);
        }
      }
    }
    if (j < P.n_pad) {
#pragma unroll
      for (int c = 0; c < DH; c += 2) {
        *reinterpret_cast<__half2*>(dstk + c0 + c) = valid ? __floats2half2_rn(dk[c], dk[c + 1]) : __floats2half2_rn(0.f, 0.f);
        *reinterpret_cast<__half2*>(dstv + c0 + c) = valid ? __floats2half2_rn(dv[c], dv[c + 1]) : __floats2half2_rn(0.f, 0.f);
      }
    }
  }
}


// ---------------------------------------------------------------------------------------------------------------
// Register-resident variants for head dims <= 64 (the P3 / P4 levels, where the token count is largest): the thread's own
// row (q and dO, or k and v) lives in registers, the other side's rows are broadcast from shared memory 16 bytes at a time,
// so the inner loops are FMA-bound instead of shared-memory-load-bound (two LDS per FMA in the kernels above).
constexpr int kT2 = 64;    // rows of the other side staged per tile

template <int D>
__global__ void __launch_bounds__(kBT) attn_bwd_q_reg_kernel(const AttnBwdParams P) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ __half sm_h[];
  __half* kt = sm_h;                  // [kT2][D]
  __half* vt = kt + kT2 * D;          // [kT2][D]
  const int dir = blockIdx.z, bh = blockIdx.y, b = bh / P.heads, head = bh % P.heads;
  const int i = blockIdx.x * kBT + threadIdx.x;
  const int ld = 3 * P.C;
  const __half* qsrc = (dir == 0 ? P.qkv[1] : P.qkv[0]) + size_t(b) * P.n_pad * ld + head * D;
  const __half* ksrc = (dir == 0 ? P.qkv[0] : P.qkv[1]) + size_t(b) * P.n_pad * ld + P.C + head * D;
  const __half* vsrc = ksrc + P.C;
  const __half* osrc = (dir == 0 ? P.o[0] : P.o[1]) + size_t(b) * P.n_pad * P.C + head * D;
  const __half* dsrc = (dir == 0 ? P.dout[0] : P.dout[1]) + size_t(b) * P.n_pad * P.C + head * D;
  const bool valid = i < P.N;
  float q[D], d_o[D], dq[D];
  float delta = 0.f;
#pragma unroll
  for (int c8 = 0; c8 < D / 8; ++c8) {
    float a[8], g[8], o[8];
    const uint4 z4 = make_uint4(0, 0, 0, 0);
    unpack8(valid ? __ldg(reinterpret_cast<const uint4*>(qsrc + size_t(i) * ld) + c8) : z4, a);
    unpack8(valid ? __ldg(reinterpret_cast<const uint4*>(dsrc + size_t(i) * P.C) + c8) : z4, g);
    unpack8(valid ? __ldg(reinterpret_cast<const uint4*>(osrc + size_t(i) * P.C) + c8) : z4, o);
#pragma unroll
    for (int e = 0; e < 8; ++e) { q[c8 * 8 + e] = a[e] * P.scale_log2; d_o[c8 * 8 + e] = g[e]; dq[c8 * 8 + e] = 0.f; delta += g[e] * o[e]; }
  }
  // pass 1: row max and sum (q carries scale * log2(e): scores come out in log2 units)
  float m = -INFINITY, l = 0.f;
  for (int j0 = 0; j0 < P.N; j0 += kT2) {
    __syncthreads();
    for (int e = threadIdx.x; e < kT2 * (D / 8); e += kBT) {
      const int j = j0 + e / (D / 8), c8 = e % (D / 8);
      reinterpret_cast<uint4*>(kt)[e] = j < P.N ? __ldg(reinterpret_cast<const uint4*>(ksrc + size_t(j) * ld) + c8) : make_uint4(0, 0, 0, 0);
    }
    __syncthreads();
    const int jn = min(kT2, P.N - j0);
    for (int j = 0; j < jn; ++j) {
      float s = 0.f;
#pragma unroll
      for (int c8 = 0; c8 < D / 8; ++c8) {
        float kf[8];
        unpack8(reinterpret_cast<const uint4*>(kt + j * D)[c8], kf);
#pragma unroll
        for (int e = 0; e < 8; ++e) s = fmaf(q[c8 * 8 + e], kf[e], s);
      }
      const float mn = fmaxf(m, s);
      l = l * exp2f(m - mn) + exp2f(s - mn);
      m = mn;
    }
  }
  const float inv_l = 1.f / l;
  if (valid) {
    float* st = P.stats + ((size_t(dir) * P.B * P.heads + bh) * P.n_pad + i) * 2;
    st[0] = m; st[1] = inv_l;
  }
  // pass 2: dQ
  const float keep_scale = 1.f / (1.f - P.p_drop);
  const uint32_t seed = P.seed + (P.seed_off ? __ldg(P.seed_off) : 0u);
  for (int j0 = 0; j0 < P.N; j0 += kT2) {
    __syncthreads();
    for (int e = threadIdx.x; e < kT2 * (D / 8); e += kBT) {
      const int j = j0 + e / (D / 8), c8 = e % (D / 8);
      const bool in = j < P.N;
      reinterpret_cast<uint4*>(kt)[e] = in ? __ldg(reinterpret_cast<const uint4*>(ksrc + size_t(j) * ld) + c8) : make_uint4(0, 0, 0, 0);
      reinterpret_cast<uint4*>(vt)[e] = in ? __ldg(reinterpret_cast<const uint4*>(vsrc + size_t(j) * ld) + c8) : make_uint4(0, 0, 0, 0);
    }
    __syncthreads();
    const int jn = min(kT2, P.N - j0);
    for (int j = 0; j < jn; ++j) {
      float s = 0.f, dp = 0.f;
#pragma unroll
      for (int c8 = 0; c8 < D / 8; ++c8) {
        float kf[8], vf[8];
        unpack8(reinterpret_cast<const uint4*>(kt + j * D)[c8], kf);
        unpack8(reinterpret_cast<const uint4*>(vt + j * D)[c8], vf);
#pragma unroll
        for (int e = 0; e < 8; ++e) { s = fmaf(q[c8 * 8 + e], kf[e], s); dp = fmaf(d_o[c8 * 8 + e], vf[e], dp); }
      }
      const float p = exp2f(s - m) * inv_l;
      if (P.p_drop > 0.f) dp = attn_keep(seed, dir, bh, i, j0 + j, P.p_drop) ? dp * keep_scale : 0.f;
      const float ds = p * (dp - delta) * P.scale;
#pragma unroll
      for (int c8 = 0; c8 < D / 8; ++c8) {
        float kf[8];
        unpack8(reinterpret_cast<const uint4*>(kt + j * D)[c8], kf);
#pragma unroll
        for (int e = 0; e < 8; ++e) dq[c8 * 8 + e] = fmaf(ds, kf[e], dq[c8 * 8 + e]);
      }
    }
  }
  if (i < P.n_pad) {
    __half* dst = (dir == 0 ? P.dqkv[1] : P.dqkv[0]) + (size_t(b) * P.n_pad + i) * ld + head * D;
#pragma unroll
    for (int c = 0; c < D; c += 2) *reinterpret_cast<__half2*>(dst + c) = valid ? __floats2half2_rn(dq[c], dq[c + 1]) : __floats2half2_rn(0.f, 0.f);
  }
}

template <int D>
__global__ void __launch_bounds__(kBT) attn_bwd_kv_reg_kernel(const AttnBwdParams P) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ __half sm_h[];
  __half* qt = sm_h;                  // [kT2][D]
  __half* dt = qt + kT2 * D;          // [kT2][D]  dO
  float* st = reinterpret_cast<float*>(dt + kT2 * D);      // [kT2][3] = m, 1/l, delta
  const int dir = blockIdx.z, bh = blockIdx.y, b = bh / P.heads, head = bh % P.heads;
  const int j = blockIdx.x * kBT + threadIdx.x;
  const int ld = 3 * P.C;
  const __half* qsrc = (dir == 0 ? P.qkv[1] : P.qkv[0]) + size_t(b) * P.n_pad * ld + head * D;
  const __half* ksrc = (dir == 0 ? P.qkv[0] : P.qkv[1]) + size_t(b) * P.n_pad * ld + P.C + head * D;
  const __half* vsrc = ksrc + P.C;
  const __half* osrc = (dir == 0 ? P.o[0] : P.o[1]) + size_t(b) * P.n_pad * P.C + head * D;
  const __half* dsrc = (dir == 0 ? P.dout[0] : P.dout[1]) + size_t(b) * P.n_pad * P.C + head * D;
  const float* stats = P.stats + (size_t(dir) * P.B * P.heads + bh) * P.n_pad * 2;
  const bool valid = j < P.N;
  __half2 kh[D / 2], vh[D / 2];       // this key's k and v rows, packed (unpacked on use)
  float dk[D], dv[D];
#pragma unroll
  for (int c8 = 0; c8 < D / 8; ++c8) {
    const uint4 z4 = make_uint4(0, 0, 0, 0);
    const uint4 ku = valid ? __ldg(reinterpret_cast<const uint4*>(ksrc + size_t(j) * ld) + c8) : z4;
    const uint4 vu = valid ? __ldg(reinterpret_cast<const uint4*>(vsrc + size_t(j) * ld) + c8) : z4;
#pragma unroll
    for (int e = 0; e < 4; ++e) { kh[c8 * 4 + e] = reinterpret_cast<const __half2*>(&ku)[e]; vh[c8 * 4 + e] = reinterpret_cast<const __half2*>(&vu)[e]; }
#pragma unroll
    for (int e = 0; e < 8; ++e) dk[c8 * 8 + e] = dv[c8 * 8 + e] = 0.f;
  }
  const float keep_scale = 1.f / (1.f - P.p_drop);
  const uint32_t seed = P.seed + (P.seed_off ? __ldg(P.seed_off) : 0u);
  for (int i0 = 0; i0 < P.N; i0 += kT2) {
    __syncthreads();
    for (int e = threadIdx.x; e < kT2 * (D / 8); e += kBT) {
      const int i = i0 + e / (D / 8), c8 = e % (D / 8);
      const bool in = i < P.N;
      reinterpret_cast<uint4*>(qt)[e] = in ? __ldg(reinterpret_cast<const uint4*>(qsrc + size_t(i) * ld) + c8) : make_uint4(0, 0, 0, 0);
      reinterpret_cast<uint4*>(dt)[e] = in ? __ldg(reinterpret_cast<const uint4*>(dsrc + size_t(i) * P.C) + c8) : make_uint4(0, 0, 0, 0);
    }
    if (threadIdx.x < kT2) {
      const int i = i0 + threadIdx.x;
      float dl = 0.f;
      if (i < P.N)
        for (int c = 0; c < D; ++c) dl += __half2float(dsrc[size_t(i) * P.C + c]) * __half2float(osrc[size_t(i) * P.C + c]);
      st[threadIdx.x * 3] = i < P.N ? stats[size_t(i) * 2] : 0.f;
      st[threadIdx.x * 3 + 1] = i < P.N ? stats[size_t(i) * 2 + 1] : 0.f;
      st[threadIdx.x * 3 + 2] = dl;
    }
    __syncthreads();
    const int in_ = min(kT2, P.N - i0);
    for (int i = 0; i < in_; ++i) {
      float s = 0.f, dp = 0.f;
#pragma unroll
      for (int c8 = 0; c8 < D / 8; ++c8) {
        float qf[8], gf[8];
        unpack8(reinterpret_cast<const uint4*>(qt + i * D)[c8], qf);
        unpack8(reinterpret_cast<const uint4*>(dt + i * D)[c8], gf);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 k2 = __half22float2(kh[c8 * 4 + e]), v2 = __half22float2(vh[c8 * 4 + e]);
          s = fmaf(qf[2 * e], k2.x, s); s = fmaf(qf[2 * e + 1], k2.y, s);
          dp = fmaf(gf[2 * e], v2.x, dp); dp = fmaf(gf[2 * e + 1], v2.y, dp);
        }
      }
      const float p = exp2f(s * P.scale_log2 - st[i * 3]) * st[i * 3 + 1];
      float pd = p;
      if (P.p_drop > 0.f) {
        const bool keep = attn_keep(seed, dir, bh, i0 + i, j, P.p_drop);
        pd = keep ? p * keep_scale : 0.f;
        dp = keep ? dp * keep_scale : 0.f;
      }
      const float ds = p * (dp - st[i * 3 + 2]) * P.scale;
#pragma unroll
      for (int c8 = 0; c8 < D / 8; ++c8) {
        float qf[8], gf[8];
        unpack8(reinterpret_cast<const uint4*>(qt + i * D)[c8], qf);
        unpack8(reinterpret_cast<const uint4*>(dt + i * D)[c8], gf);
#pragma unroll
        for (int e = 0; e < 8; ++e) { dk[c8 * 8 + e] = fmaf(ds, qf[e], dk[c8 * 8 + e]); dv[c8 * 8 + e] = fmaf(pd, gf[e], dv[c8 * 8 + e]); }
      }
    }
  }
  if (j < P.n_pad) {
    __half* dstk = (dir == 0 ? P.dqkv[0] : P.dqkv[1]) + (size_t(b) * P.n_pad + j) * ld + P.C + head * D;
    __half* dstv = dstk + P.C;
#pragma unroll
    for (int c = 0; c < D; c += 2) {
      *reinterpret_cast<__half2*>(dstk + c) = valid ? __floats2half2_rn(dk[c], dk[c + 1]) : __floats2half2_rn(0.f, 0.f);
      *reinterpret_cast<__half2*>(dstv + c) = valid ? __floats2half2_rn(dv[c], dv[c + 1]) : __floats2half2_rn(0.f, 0.f);
    }
  }
}

template <int D>
static int launch_attn_bwd_reg(const AttnBwdParams& P, cudaStream_t st) {
  const size_t smq = size_t(2 * kT2 * D) * sizeof(__half);
  const size_t smk = smq + kT2 * 3 * sizeof(float);
  dim3 gridp(blocks_for(P.n_pad, kBT), P.B * P.heads, 2);     // also zeroes the pad rows of the gradient
  if (int rc = launch_k("cross_attention_bwd(q)", attn_bwd_q_reg_kernel<D>, gridp, dim3(kBT), smq, st, P)) return rc;
  if constexpr (D <= 32) {
    return launch_k("cross_attention_bwd(kv)", attn_bwd_kv_reg_kernel<D>, gridp, dim3(kBT), smk, st, P);
  } else {     // k, v, dk, dv of a 64-wide head do not fit the register file together: the shared-memory variant (64 channels per pass)
    const size_t smo = size_t(2 * D * kBT + 2 * kTT * D) * sizeof(__half) + kTT * 3 * sizeof(float);
    static bool configured[kMaxDevices] = {false};
    if (int rc = configure_smem(attn_bwd_kv_kernel<D>, (int)smo, configured, "cross_attention_bwd: cudaFuncSetAttribute")) return rc;
    return launch_k("cross_attention_bwd(kv)", attn_bwd_kv_kernel<D>, gridp, dim3(kBT), smo, st, P);
  }
}

template <int D>
static int launch_attn_bwd(const AttnBwdParams& P, cudaStream_t st) {
  const size_t smq = size_t(2 * D * kBT + 2 * kTT * D) * sizeof(__half);
  const size_t smk = smq + kTT * 3 * sizeof(float);
  static bool configured[kMaxDevices] = {false};
  if (int rc = configure_smem(attn_bwd_q_kernel<D>, (int)smq, configured, "cross_attention_bwd: cudaFuncSetAttribute")) return rc;
  static bool configured2[kMaxDevices] = {false};
  if (int rc = configure_smem(attn_bwd_kv_kernel<D>, (int)smk, configured2, "cross_attention_bwd: cudaFuncSetAttribute")) return rc;
  dim3 gridp(blocks_for(P.n_pad, kBT), P.B * P.heads, 2);     // also zero the pad rows of the gradient
  if (int rc = launch_k("cross_attention_bwd(q)", attn_bwd_q_kernel<D>, gridp, dim3(kBT), smq, st, P)) return rc;
  return launch_k("cross_attention_bwd(kv)", attn_bwd_kv_kernel<D>, gridp, dim3(kBT), smk, st, P);
}

}  // namespace icaf

using namespace icaf;

extern "C" size_t icaf_cross_attention_bwd_workspace_bytes(int B, int n_pad, int heads) {
  return size_t(2) * B * heads * n_pad * 2 * sizeof(float);
}

extern "C" int icaf_cross_attention_bwd(const void* qkv_vis, const void* qkv_ir, const void* out_vis, const void* out_ir, const void* dout_vis,
                                        const void* dout_ir, void* dqkv_vis, void* dqkv_ir, int B, int N, int n_pad, int C, int heads, float p_drop,
                                        uint32_t seed, void* workspace, size_t workspace_bytes, void* stream) {
  if (!qkv_vis || !qkv_ir || !out_vis || !out_ir || !dout_vis || !dout_ir || !dqkv_vis || !dqkv_ir || !workspace)
    return set_error(ICAF_ERR_BAD_ARG, "cross_attention_bwd: null pointer");
  if (B < 1 || N < 1 || n_pad < N || heads < 1 || C % heads || !(p_drop >= 0.f && p_drop < 1.f)) return set_error(ICAF_ERR_BAD_ARG, "cross_attention_bwd: bad shape");
  if (workspace_bytes < icaf_cross_attention_bwd_workspace_bytes(B, n_pad, heads)) return set_error(ICAF_ERR_BAD_ARG, "cross_attention_bwd: workspace too small");
  const int d = C / heads;
  AttnBwdParams P;
  P.qkv[0] = (const __half*)qkv_vis; P.qkv[1] = (const __half*)qkv_ir; P.o[0] = (const __half*)out_vis; P.o[1] = (const __half*)out_ir;
  P.dout[0] = (const __half*)dout_vis; P.dout[1] = (const __half*)dout_ir; P.dqkv[0] = (__half*)dqkv_vis; P.dqkv[1] = (__half*)dqkv_ir;
  P.stats = (float*)workspace; P.B = B; P.N = N; P.n_pad = n_pad; P.C = C; P.heads = heads;
  P.scale = 1.0f / sqrtf(float(d)); P.scale_log2 = 1.4426950408889634f * P.scale; P.p_drop = p_drop; P.seed = seed; P.seed_off = seed_offset_ptr();
  cudaStream_t st = (cudaStream_t)stream;
  switch (d) {
    case 8: return launch_attn_bwd_reg<8>(P, st);        // yolov5n's P3 block
    case 16: return launch_attn_bwd_reg<16>(P, st);
    case 32: return launch_attn_bwd_reg<32>(P, st);
    case 64: return launch_attn_bwd_reg<64>(P, st);
    case 128: return launch_attn_bwd<128>(P, st);
    default: return set_error(ICAF_ERR_UNSUPPORTED, "cross_attention_bwd: head dim must be 8/16/32/64/128");
  }
}
