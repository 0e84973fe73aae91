// Training-mode kernels of the hot path that are not GEMMs (forward and backward): BatchNorm with batch statistics + SiLU
// (Conv.forward, models/common.py:56-57), exact-erf GELU and dropout, the LayerNorm backward (its parameter gradients are
// two-stage channel reductions; the forward is in dmff.cu), and the small reductions behind scalar-parameter gradients.
// fp16 activations / gradients, fp32 statistics and parameter gradients.  Every reduction is two-stage with a fixed
// summation order (deterministic; the reference trains with torch.use_deterministic_algorithms, utils/general.py:53-54).
#include "icaf_internal.cuh"

namespace icaf {

constexpr int kRedChunks = 1024;      // upper bound of the row chunks of a two-stage reduction (sizes the workspace); the launch picks <= this many

__device__ __forceinline__ float sigmoidf_(float z) { return __fdividef(1.f, 1.f + __expf(-z)); }

// ---------------------------------------------------------------------------------------------------------------
// per-channel partial sums over row chunks: out[chunk][which][c], which = 0 / 1.
// MODE 0: (x, x^2)  [BatchNorm statistics]      MODE 1: (dz, dz * xhat) with dz = dy * silu'(x*a + b)  [BN + SiLU backward]
// MODE 2: (dy, dy * xhat_row) with per-ROW (mean, rstd)  [LayerNorm gamma / beta gradients]   MODE 3: (x * y, 0)  [dot products]
template <int MODE>
__global__ void __launch_bounds__(256) chan_partial_kernel(const __half* __restrict__ x, const __half* __restrict__ dy, const float* __restrict__ a,
                                                           const float* __restrict__ b, const float* __restrict__ mean, const float* __restrict__ invstd,
                                                           float* __restrict__ out, long long rows, int C, int act, int chunks) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[256][17];
  // the 256 threads cover (g channel groups) x (rpp rows) per pass: all of them stay busy for narrow maps too (C = 64 -> 8 x 32)
  const int C8 = C >> 3;
  const int g = min(C8 - int(blockIdx.x) * 32, 32);
  const int rpp = 256 / g;
  const int tid = threadIdx.x;
  const bool active = tid < g * rpp;
  const int cgl = tid % g, rl = tid / g;
  const int cg = blockIdx.x * 32 + cgl;
  const long long per = (rows + chunks - 1) / chunks;
  const long long r0 = blockIdx.y * per, r1 = min(r0 + per, rows);
  float s0[8], s1[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) s0[e] = s1[e] = 0.f;
  if (active) {
    float av[8], bv[8], mv[8], iv[8];
    if (MODE == 1) {                                        // a = gamma, b = beta on entry -> per-channel affine of the BN apply
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        mv[e] = mean[cg * 8 + e]; iv[e] = invstd[cg * 8 + e];
        av[e] = a[cg * 8 + e] * iv[e]; bv[e] = b[cg * 8 + e] - mv[e] * av[e];
      }
    }
    // two rows per trip: both rows' loads are issued before either is consumed (twice the bytes in flight per thread)
    for (long long r = r0 + rl; r < r1; r += 2 * rpp) {
      const long long rb = r + rpp;
      const bool two = rb < r1;
      float xv[2][8], dv[2][8];
      const uint4 xa = ldg16(x + r * C + cg * 8);
      const uint4 xb = two ? ldg16(x + rb * C + cg * 8) : make_uint4(0, 0, 0, 0);
      uint4 da = make_uint4(0, 0, 0, 0), db = make_uint4(0, 0, 0, 0);
      if (MODE != 0) {
        da = ldg16(dy + r * C + cg * 8);
        if (two) db = ldg16(dy + rb * C + cg * 8);
      }
      unpack8(xa, xv[0]); unpack8(xb, xv[1]); unpack8(da, dv[0]); unpack8(db, dv[1]);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (h == 1 && !two) break;
        float rm = 0.f, ri = 0.f;
        if (MODE == 2) { rm = mean[h ? rb : r]; ri = invstd[h ? rb : r]; }
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float xe = xv[h][e], de = dv[h][e];
          if (MODE == 0) { s0[e] += xe; s1[e] += xe * xe; }
          if (MODE == 1) {
            const float z = xe * av[e] + bv[e];
            float dz = de;
            if (act) { const float sg = sigmoidf_(z); dz *= sg * (1.f + z * (1.f - sg)); }
            s0[e] += dz; s1[e] += dz * (xe - mv[e]) * iv[e];
          }
          if (MODE == 2) { s0[e] += de; s1[e] += de * (xe - rm) * ri; }
          if (MODE == 3) { s0[e] += xe * de; }
        }
      }
    }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) { red[tid][e] = s0[e]; red[tid][8 + e] = s1[e]; }
  __syncthreads();
  if (tid < g) {                                            // fixed order over the rpp row lanes: deterministic
#pragma unroll
    for (int e = 0; e < 16; ++e) {
      float s = 0.f;
      for (int y = 0; y < rpp; ++y) s += red[y * g + tid][e];
      out[(size_t(blockIdx.y) * 2 + (e >> 3)) * C + cg * 8 + (e & 7)] = s;
    }
  }
}

// second stages: block (32 channels, 32 chunk lanes); lane y sums chunks y, y + 32, ...; the 32 lane sums are added in lane order
constexpr int kFinLanes = 32;
__device__ __forceinline__ void chunk_sums(const float* __restrict__ part, int C, int chunks, int c, float& s, float& q, float (*sm)[kFinLanes][33]) {
  float a = 0.f, b2 = 0.f;
  if (c < C) {
#pragma unroll 4
    for (int k = threadIdx.y; k < chunks; k += kFinLanes) { a += __ldg(part + (size_t(k) * 2) * C + c); b2 += __ldg(part + (size_t(k) * 2 + 1) * C + c); }
  }
  sm[0][threadIdx.y][threadIdx.x] = a; sm[1][threadIdx.y][threadIdx.x] = b2;
  __syncthreads();
  s = q = 0.f;
  if (threadIdx.y == 0)
    for (int y = 0; y < kFinLanes; ++y) { s += sm[0][y][threadIdx.x]; q += sm[1][y][threadIdx.x]; }
}

// BatchNorm statistics, second stage: mean, invstd, and the running statistics update (momentum, unbiased variance).
// DEV_COUNT: the row count is read as fp32 from device memory (`count`) in place of `rows` (the global count of a synchronised
// BatchNorm); a template argument, so that the one-call path compiles to exactly the code it had before the synchronised form
template <bool DEV_COUNT>
__global__ void __launch_bounds__(1024) bn_finalize_kernel(const float* __restrict__ part, float* __restrict__ mean, float* __restrict__ invstd, float* run_mean,
                                                          float* run_var, int C, long long rows, float eps, float momentum, int chunks,
                                                          const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ ab,
                                                          const float* __restrict__ count) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float sm[2][kFinLanes][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  float s, q;
  chunk_sums(part, C, chunks, c, s, q, sm);
  if (c >= C || threadIdx.y) return;
  const float n = DEV_COUNT ? __ldg(count) : float(rows);
  const float m = s / n;
  const float var = fmaxf(q / n - m * m, 0.f);
  mean[c] = m;
  const float is = rsqrtf(var + eps);
  invstd[c] = is;
  const float a = gamma[c] * is;
  ab[c] = a; ab[C + c] = beta[c] - m * a;                   // the apply pass: y = act(x * a + b)
  if (run_mean) {
    run_mean[c] = (1.f - momentum) * run_mean[c] + momentum * m;
    const float unbias = DEV_COUNT ? (n > 1.f ? n / (n - 1.f) : 1.f) : (rows > 1 ? float(rows) / float(rows - 1) : 1.f);
    run_var[c] = (1.f - momentum) * run_var[c] + momentum * var * unbias;
  }
}
// generic second stage: out[which][c] = (accumulate ? out : 0) + scale * sum_chunks part
// out0/out1: sums (scale, accumulate); raw0/raw1 (optional): the unscaled sums as well (BatchNorm backward needs both in one pass)
// DEV_COUNT: count_out (optional): count_out[0] = n_rows; count (optional): inv_m = 1 / count[0], read from device memory
template <bool DEV_COUNT>
__global__ void __launch_bounds__(1024) chan_final_kernel(const float* __restrict__ part, float* __restrict__ out0, float* __restrict__ out1, int C, float scale,
                                                          int accumulate, int chunks, float* __restrict__ raw0, float* __restrict__ raw1,
                                                          const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ mean,
                                                          const float* __restrict__ invstd, float inv_m, float* __restrict__ coef,
                                                          const float* __restrict__ count, float* __restrict__ count_out, float n_rows) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float sm[2][kFinLanes][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  float s, q;
  chunk_sums(part, C, chunks, c, s, q, sm);
  if (c >= C || threadIdx.y) return;
  if (DEV_COUNT && count_out && c == 0) count_out[0] = n_rows;
  if (raw0) raw0[c] = s;
  if (raw1) raw1[c] = q;
  if (coef) {      // BatchNorm backward apply pass: dx = a * (dz - k1 - (x - mean) * k2), z = x * a + b
    if (DEV_COUNT && count) inv_m = 1.f / __ldg(count);
    const float is = invstd[c], a = gamma[c] * is, m = mean[c];
    coef[c] = a; coef[C + c] = beta[c] - m * a; coef[2 * C + c] = m; coef[3 * C + c] = s * inv_m; coef[4 * C + c] = q * inv_m * is;
  }
  if (out0) out0[c] = (accumulate ? out0[c] : 0.f) + scale * s;
  if (out1) out1[c] = (accumulate ? out1[c] : 0.f) + scale * q;
}
// scalar second stage of MODE 3 partials: out[0] = (accumulate ? out[0] : 0) + scale * sum of everything
__global__ void scalar_final_kernel(const float* __restrict__ part, float* __restrict__ out, int C, float scale, int accumulate, int chunks) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[1024];
  float s = 0.f;
  const int total = chunks * C;                            // fixed thread -> element map: deterministic
#pragma unroll 4
  for (int i = threadIdx.x; i < total; i += 1024) s += __ldg(part + size_t(i / C) * 2 * C + (i % C));
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = 512; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[0] = (accumulate ? out[0] : 0.f) + scale * red[0];
}

// y = act(x * a[c] + b[c])   (BatchNorm apply + SiLU; a = gamma * invstd, b = beta - mean * a: `ab` = [2][C] from the finalize pass)
__global__ void __launch_bounds__(256) affine_act_kernel(const __half* __restrict__ x, const float* __restrict__ ab, __half* __restrict__ y, long long n8, int C8,
                                                         int act) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n8) return;
  const int cg = int(i % C8), C = C8 * 8;
  float v[8], a[8], b[8];
  unpack8(ldg16(x + i * 8), v);
  ld8f(ab + cg * 8, a);
  ld8f(ab + C + cg * 8, b);
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float z = fmaf(v[e], a[e], b[e]);
    v[e] = act ? z * sigmoidf_(z) : z;
  }
  reinterpret_cast<uint4*>(y)[i] = pack8(v);
}
// dx = a * (dz - k1 - (x - mean) * k2),  dz = dy * act'(z), z = x * a + b   (`coef` = [5][C]: a, b, mean, k1 = S1 / M, k2 = invstd * S2 / M)
__global__ void __launch_bounds__(256) bn_bwd_apply_kernel(const __half* __restrict__ x, const __half* __restrict__ dy, const float* __restrict__ coef,
                                                           __half* __restrict__ dx, long long n8, int C8, int act) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n8) return;
  const int cg = int(i % C8), C = C8 * 8;
  float xv[8], dv[8], a[8], b[8], m[8], k1[8], k2[8];
  unpack8(ldg16(x + i * 8), xv);
  unpack8(ldg16(dy + i * 8), dv);
  ld8f(coef + cg * 8, a); ld8f(coef + C + cg * 8, b); ld8f(coef + 2 * C + cg * 8, m); ld8f(coef + 3 * C + cg * 8, k1); ld8f(coef + 4 * C + cg * 8, k2);
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    float dz = dv[e];
    if (act) { const float z = fmaf(xv[e], a[e], b[e]); const float sg = sigmoidf_(z); dz *= sg * fmaf(z, 1.f - sg, 1.f); }
    xv[e] = a[e] * (dz - k1[e] - (xv[e] - m[e]) * k2[e]);
  }
  reinterpret_cast<uint4*>(dx)[i] = pack8(xv);
}

// ---------------------------------------------------------------------------------------------------------------
// element-wise: MODE 0 gelu(x) [erf], 1 dy * gelu'(x), 2 dropout (x * keep / (1 - p); the same call is its own backward on dy)
template <int MODE>
__global__ void eltwise_kernel(const __half* __restrict__ x, const __half* __restrict__ dy, __half* __restrict__ y, long long n8, float p, uint32_t seed,
                               const uint32_t* __restrict__ seed_off) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n8) return;
  float xv[8], dv[8];
  unpack8(ldg16(x + i * 8), xv);
  if (MODE == 1) unpack8(ldg16(dy + i * 8), dv);
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    if (MODE == 0) xv[e] = gelu_erf_f(xv[e]);
    if (MODE == 1) {
      const float v = xv[e];
      const float cdf = 0.5f * (1.f + erff(v * 0.70710678118654752f));
      xv[e] = dv[e] * (cdf + v * 0.3989422804014327f * __expf(-0.5f * v * v));
    }
    if (MODE == 2) {
      const long long idx = i * 8 + e;
      const uint32_t h = dropout_hash(uint32_t(idx), uint32_t(idx >> 32), seed + (seed_off ? __ldg(seed_off) : 0u));
      xv[e] = (float(h >> 8) * (1.f / 16777216.f) >= p) ? xv[e] / (1.f - p) : 0.f;
    }
  }
  reinterpret_cast<uint4*>(y)[i] = pack8(xv);
}

// LayerNorm backward, dx part (one warp per row, C <= 2048): dx = rstd * (g - mean(g) - xhat * mean(g * xhat)), g = dy * gamma
__global__ void ln_bwd_kernel(const __half* __restrict__ x, const __half* __restrict__ dy, const float* __restrict__ gamma, __half* __restrict__ dx,
                              float* __restrict__ row_mean, float* __restrict__ row_rstd, long long rows, int C, float eps) {
  pdl_launch_dependents();
  pdl_wait();
  const long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31, nch = C >> 3;
  float xv[8][8], gv[8][8], mean, rstd;
  ln_row_moments(x, row, C, eps, xv, mean, rstd);
  float sg = 0.f, sgx = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int ch = lane + 32 * j;
    if (ch < nch) {
      unpack8(ldg16(dy + row * C + ch * 8), gv[j]);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        gv[j][e] *= gamma[ch * 8 + e];
        xv[j][e] = (xv[j][e] - mean) * rstd;
        sg += gv[j][e]; sgx += gv[j][e] * xv[j][e];
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { sg += __shfl_xor_sync(0xffffffffu, sg, o); sgx += __shfl_xor_sync(0xffffffffu, sgx, o); }
  sg /= float(C); sgx /= float(C);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int ch = lane + 32 * j;
    if (ch < nch) {
      float o[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = rstd * (gv[j][e] - sg - xv[j][e] * sgx);
      *reinterpret_cast<uint4*>(dx + row * C + ch * 8) = pack8(o);
    }
  }
  if (lane == 0) { row_mean[row] = mean; row_rstd[row] = rstd; }
}

// row chunks of a two-stage channel reduction: about 8 blocks per SM over the whole grid, at least four passes of work per block
static inline int pick_chunks(long long rows, int C, int cap_chunks = kRedChunks) {
  const int C8 = C / 8, bx = (C8 + 31) / 32, g = C8 < 32 ? C8 : 32, rpp = 256 / g;
  long long want = 1184 / bx, cap = (rows + 4ll * rpp - 1) / (4ll * rpp);
  long long c = want < cap ? want : cap;
  if (c > cap_chunks) c = cap_chunks;
  return c < 1 ? 1 : int(c);
}

}  // namespace icaf

using namespace icaf;

// [kRedChunks][2][C] partial sums, then 8 C floats of per-channel coefficients for the apply passes
static inline size_t ws_floats(int C) { return size_t(kRedChunks) * 2 * (C > 0 ? C : 1) + 8 * size_t(C > 0 ? C : 1); }
extern "C" size_t icaf_train_workspace_bytes(int C) { return ws_floats(C) * sizeof(float); }

extern "C" int icaf_bn_act_fwd(const void* x, const float* gamma, const float* beta, float* run_mean, float* run_var, void* y, float* save_mean,
                               float* save_invstd, int64_t rows, int C, float eps, float momentum, int act, float* workspace, size_t workspace_bytes,
                               void* stream) {
  if (!x || !gamma || !beta || !y || !save_mean || !save_invstd || !workspace || rows < 1 || C < 8 || C % 8) return set_error(ICAF_ERR_BAD_ARG, "bn_act_fwd: bad argument");
  if (workspace_bytes < icaf_train_workspace_bytes(C)) return set_error(ICAF_ERR_BAD_ARG, "bn_act_fwd: workspace too small (icaf_train_workspace_bytes)");
  cudaStream_t st = (cudaStream_t)stream;
  const int chunks = pick_chunks(rows, C);
  if (int rc = launch_k("bn_act_fwd(stats)", chan_partial_kernel<0>, dim3(blocks_for(C / 8, 32), chunks), dim3(256), 0, st, (const __half*)x,
                        (const __half*)nullptr, (const float*)nullptr, (const float*)nullptr, (const float*)nullptr, (const float*)nullptr, workspace,
                        (long long)rows, C, 0, chunks)) return rc;
  if (int rc = launch_k("bn_act_fwd(finalize)", bn_finalize_kernel<false>, dim3(blocks_for(C, 32)), dim3(32, kFinLanes), 0, st, (const float*)workspace,
                        save_mean, save_invstd, run_mean, run_var, C, (long long)rows, eps, momentum, chunks, gamma, beta,
                        workspace + size_t(kRedChunks) * 2 * C, (const float*)nullptr)) return rc;
  const long long n8 = rows * (C / 8);
  return launch_k("bn_act_fwd", affine_act_kernel, dim3(blocks_for(n8, 256)), dim3(256), 0, st, (const __half*)x,
                  (const float*)(workspace + size_t(kRedChunks) * 2 * C), (__half*)y, n8, C / 8, act);
}

extern "C" int icaf_bn_act_bwd(const void* x, const void* dy, const float* gamma, const float* beta, const float* save_mean, const float* save_invstd,
                               void* dx, float* dgamma, float* dbeta, int64_t rows, int C, int act, float grad_scale, int accumulate, float* workspace,
                               size_t workspace_bytes, void* stream) {
  if (!x || !dy || !gamma || !beta || !save_mean || !save_invstd || !dx || !workspace || rows < 1 || C < 8 || C % 8) return set_error(ICAF_ERR_BAD_ARG, "bn_act_bwd: bad argument");
  if (workspace_bytes < icaf_train_workspace_bytes(C)) return set_error(ICAF_ERR_BAD_ARG, "bn_act_bwd: workspace too small (icaf_train_workspace_bytes)");
  cudaStream_t st = (cudaStream_t)stream;
  float* coef = workspace + size_t(kRedChunks) * 2 * C;     // [5][C] coefficients of the apply pass
  const int chunks = pick_chunks(rows, C);
  if (int rc = launch_k("bn_act_bwd(partial)", chan_partial_kernel<1>, dim3(blocks_for(C / 8, 32), chunks), dim3(256), 0, st, (const __half*)x,
                        (const __half*)dy, gamma, beta, save_mean, save_invstd, workspace, (long long)rows, C, act, chunks)) return rc;
  // one second stage: the apply pass's coefficients and the parameter gradients dbeta = S1, dgamma = S2 (scaled by grad_scale)
  if (int rc = launch_k("bn_act_bwd(sums)", chan_final_kernel<false>, dim3(blocks_for(C, 32)), dim3(32, kFinLanes), 0, st, (const float*)workspace, dbeta,
                        dgamma, C, grad_scale, accumulate, chunks, (float*)nullptr, (float*)nullptr, gamma, beta, save_mean, save_invstd,
                        1.0f / float(rows), coef, (const float*)nullptr, (float*)nullptr, 0.f)) return rc;
  const long long n8 = rows * (C / 8);
  return launch_k("bn_act_bwd", bn_bwd_apply_kernel, dim3(blocks_for(n8, 256)), dim3(256), 0, st, (const __half*)x, (const __half*)dy,
                  (const float*)coef, (__half*)dx, n8, C / 8, act);
}

// Synchronised BatchNorm: the two calls above, each split where its per-channel sums are complete.  The caller sums the
// exchange buffer over the ranks between the phases.  Phase 2 reads the buffer as a one-chunk partial-sum array, so the
// second stages are the ones above run over one chunk, with the row count read from the buffer.
extern "C" int icaf_bn_act_fwd_stats(const void* x, int64_t rows, int C, float* stats, float* workspace, size_t workspace_bytes, void* stream) {
  if (!x || !stats || !workspace || rows < 1 || C < 8 || C % 8) return set_error(ICAF_ERR_BAD_ARG, "bn_act_fwd_stats: bad argument");
  if (workspace_bytes < icaf_train_workspace_bytes(C)) return set_error(ICAF_ERR_BAD_ARG, "bn_act_fwd_stats: workspace too small (icaf_train_workspace_bytes)");
  cudaStream_t st = (cudaStream_t)stream;
  const int chunks = pick_chunks(rows, C);
  if (int rc = launch_k("bn_act_fwd_stats(partial)", chan_partial_kernel<0>, dim3(blocks_for(C / 8, 32), chunks), dim3(256), 0, st, (const __half*)x,
                        (const __half*)nullptr, (const float*)nullptr, (const float*)nullptr, (const float*)nullptr, (const float*)nullptr, workspace,
                        (long long)rows, C, 0, chunks)) return rc;
  return launch_k("bn_act_fwd_stats(sums)", chan_final_kernel<true>, dim3(blocks_for(C, 32)), dim3(32, kFinLanes), 0, st, (const float*)workspace,
                  (float*)nullptr, (float*)nullptr, C, 0.f, 0, chunks, stats, stats + C, (const float*)nullptr, (const float*)nullptr,
                  (const float*)nullptr, (const float*)nullptr, 0.f, (float*)nullptr, (const float*)nullptr, stats + 2 * C, float(rows));
}

extern "C" int icaf_bn_act_fwd_apply(const void* x, const float* gamma, const float* beta, float* run_mean, float* run_var, const float* stats, void* y,
                                     float* save_mean, float* save_invstd, int64_t rows, int C, float eps, float momentum, int act, float* workspace,
                                     size_t workspace_bytes, void* stream) {
  if (!x || !gamma || !beta || !stats || !y || !save_mean || !save_invstd || !workspace || rows < 1 || C < 8 || C % 8) return set_error(ICAF_ERR_BAD_ARG, "bn_act_fwd_apply: bad argument");
  if (workspace_bytes < icaf_train_workspace_bytes(C)) return set_error(ICAF_ERR_BAD_ARG, "bn_act_fwd_apply: workspace too small (icaf_train_workspace_bytes)");
  cudaStream_t st = (cudaStream_t)stream;
  float* ab = workspace + size_t(kRedChunks) * 2 * C;
  if (int rc = launch_k("bn_act_fwd_apply(finalize)", bn_finalize_kernel<true>, dim3(blocks_for(C, 32)), dim3(32, kFinLanes), 0, st, stats, save_mean,
                        save_invstd, run_mean, run_var, C, (long long)rows, eps, momentum, 1, gamma, beta, ab, stats + 2 * C)) return rc;
  const long long n8 = rows * (C / 8);
  return launch_k("bn_act_fwd_apply", affine_act_kernel, dim3(blocks_for(n8, 256)), dim3(256), 0, st, (const __half*)x, (const float*)ab, (__half*)y,
                  n8, C / 8, act);
}

extern "C" int icaf_bn_act_bwd_sums(const void* x, const void* dy, const float* gamma, const float* beta, const float* save_mean, const float* save_invstd,
                                    float* dgamma, float* dbeta, float* sums, int64_t rows, int C, int act, float grad_scale, int accumulate, float* workspace,
                                    size_t workspace_bytes, void* stream) {
  if (!x || !dy || !gamma || !beta || !save_mean || !save_invstd || !sums || !workspace || rows < 1 || C < 8 || C % 8) return set_error(ICAF_ERR_BAD_ARG, "bn_act_bwd_sums: bad argument");
  if (workspace_bytes < icaf_train_workspace_bytes(C)) return set_error(ICAF_ERR_BAD_ARG, "bn_act_bwd_sums: workspace too small (icaf_train_workspace_bytes)");
  cudaStream_t st = (cudaStream_t)stream;
  const int chunks = pick_chunks(rows, C);
  if (int rc = launch_k("bn_act_bwd_sums(partial)", chan_partial_kernel<1>, dim3(blocks_for(C / 8, 32), chunks), dim3(256), 0, st, (const __half*)x,
                        (const __half*)dy, gamma, beta, save_mean, save_invstd, workspace, (long long)rows, C, act, chunks)) return rc;
  return launch_k("bn_act_bwd_sums(sums)", chan_final_kernel<false>, dim3(blocks_for(C, 32)), dim3(32, kFinLanes), 0, st, (const float*)workspace, dbeta,
                  dgamma, C, grad_scale, accumulate, chunks, sums, sums + C, (const float*)nullptr, (const float*)nullptr, (const float*)nullptr,
                  (const float*)nullptr, 0.f, (float*)nullptr, (const float*)nullptr, (float*)nullptr, 0.f);
}

extern "C" int icaf_bn_act_bwd_apply(const void* x, const void* dy, const float* gamma, const float* beta, const float* save_mean, const float* save_invstd,
                                     const float* sums, const float* count, void* dx, int64_t rows, int C, int act, float* workspace, size_t workspace_bytes,
                                     void* stream) {
  if (!x || !dy || !gamma || !beta || !save_mean || !save_invstd || !sums || !count || !dx || !workspace || rows < 1 || C < 8 || C % 8) return set_error(ICAF_ERR_BAD_ARG, "bn_act_bwd_apply: bad argument");
  if (workspace_bytes < icaf_train_workspace_bytes(C)) return set_error(ICAF_ERR_BAD_ARG, "bn_act_bwd_apply: workspace too small (icaf_train_workspace_bytes)");
  cudaStream_t st = (cudaStream_t)stream;
  float* coef = workspace + size_t(kRedChunks) * 2 * C;
  if (int rc = launch_k("bn_act_bwd_apply(coef)", chan_final_kernel<true>, dim3(blocks_for(C, 32)), dim3(32, kFinLanes), 0, st, sums, (float*)nullptr,
                        (float*)nullptr, C, 0.f, 0, 1, (float*)nullptr, (float*)nullptr, gamma, beta, save_mean, save_invstd, 0.f, coef, count,
                        (float*)nullptr, 0.f)) return rc;
  const long long n8 = rows * (C / 8);
  return launch_k("bn_act_bwd_apply", bn_bwd_apply_kernel, dim3(blocks_for(n8, 256)), dim3(256), 0, st, (const __half*)x, (const __half*)dy,
                  (const float*)coef, (__half*)dx, n8, C / 8, act);
}

// mode 0: y = gelu(x); 1: y = dy * gelu'(x); 2: y = dropout(x; p, seed) (apply it to dy with the same seed for the backward)
extern "C" int icaf_eltwise(int mode, const void* x, const void* dy, void* y, int64_t n, float p, uint32_t seed, void* stream) {
  if (!x || !y || n < 0 || n % 8 || (mode == 1 && !dy) || mode < 0 || mode > 2 || (mode == 2 && !(p >= 0.f && p < 1.f))) return set_error(ICAF_ERR_BAD_ARG, "eltwise: bad argument");
  if (n == 0) return ICAF_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const long long n8 = n / 8;
  auto kernel = mode == 0 ? eltwise_kernel<0> : (mode == 1 ? eltwise_kernel<1> : eltwise_kernel<2>);
  return launch_k("eltwise", kernel, dim3(blocks_for(n8, 256)), dim3(256), 0, st, (const __half*)x, (const __half*)dy, (__half*)y, n8, p, seed,
                  seed_offset_ptr());
}

extern "C" int icaf_layernorm_bwd(const void* x, const void* dy, const float* gamma, void* dx, float* dgamma, float* dbeta, int64_t rows, int C, float eps,
                                  float grad_scale, int accumulate, float* workspace, size_t workspace_bytes, void* stream) {
  if (!x || !dy || !gamma || !dx || !workspace || rows < 1 || C % 8 || C > 2048) return set_error(ICAF_ERR_BAD_ARG, "layernorm_bwd: bad argument (C % 8, C <= 2048)");
  if (workspace_bytes < icaf_train_workspace_bytes(C) + 2 * size_t(rows) * sizeof(float)) return set_error(ICAF_ERR_BAD_ARG, "layernorm_bwd: workspace too small (icaf_train_workspace_bytes + 2 rows floats)");
  cudaStream_t st = (cudaStream_t)stream;
  float* rmean = workspace + ws_floats(C);
  float* rrstd = rmean + rows;
  if (int rc = launch_k("layernorm_bwd(dx)", ln_bwd_kernel, dim3(blocks_for(rows, 4)), dim3(128), 0, st, (const __half*)x, (const __half*)dy, gamma,
                        (__half*)dx, rmean, rrstd, (long long)rows, C, eps)) return rc;
  if (dgamma || dbeta) {
    const int chunks = pick_chunks(rows, C);
    if (int rc = launch_k("layernorm_bwd(partial)", chan_partial_kernel<2>, dim3(blocks_for(C / 8, 32), chunks), dim3(256), 0, st, (const __half*)x,
                          (const __half*)dy, (const float*)nullptr, (const float*)nullptr, (const float*)rmean, (const float*)rrstd, workspace,
                          (long long)rows, C, 0, chunks)) return rc;
    if (int rc = launch_k("layernorm_bwd(param grads)", chan_final_kernel<false>, dim3(blocks_for(C, 32)), dim3(32, kFinLanes), 0, st,
                          (const float*)workspace, dbeta, dgamma, C, grad_scale, accumulate, chunks, (float*)nullptr, (float*)nullptr,
                          (const float*)nullptr, (const float*)nullptr, (const float*)nullptr, (const float*)nullptr, 0.f, (float*)nullptr,
                          (const float*)nullptr, (float*)nullptr, 0.f)) return rc;
  }
  return ICAF_OK;
}

// out[0] = (accumulate ? out[0] : 0) + scale * <x, y> over (rows, C) fp16 matrices (gradients of the scalar gains)
extern "C" int icaf_dot(const void* x, const void* y, int64_t rows, int C, float* out, float scale, int accumulate, float* workspace, size_t workspace_bytes,
                        void* stream) {
  if (!x || !y || !out || !workspace || rows < 1 || C < 8 || C % 8) return set_error(ICAF_ERR_BAD_ARG, "dot: bad argument");
  if (workspace_bytes < icaf_train_workspace_bytes(C)) return set_error(ICAF_ERR_BAD_ARG, "dot: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const int chunks = pick_chunks(rows, C, 64);
  if (int rc = launch_k("dot(partial)", chan_partial_kernel<3>, dim3(blocks_for(C / 8, 32), chunks), dim3(256), 0, st, (const __half*)x,
                        (const __half*)y, (const float*)nullptr, (const float*)nullptr, (const float*)nullptr, (const float*)nullptr, workspace,
                        (long long)rows, C, 0, chunks)) return rc;
  return launch_k("dot", scalar_final_kernel, dim3(1), dim3(1024), 0, st, (const float*)workspace, out, C, scale, accumulate, chunks);
}
