// The optimiser step of train.py:347-352 on the device: GradScaler's unscale and inf check, nesterov SGD / Adam gated on
// the device-side inf flag, GradScaler's scale update and ModelEMA.update.  Nothing here reads back to the host, so the
// whole step can be captured into a CUDA graph behind the backward pass.
//
// Every kernel except the scale update walks a device table of icaf_optim_tensor entries (icaf_b200.h).  Each tensor is
// cut into ICAF_OPTIM_CHUNK-element chunks numbered across the table (entry.chunk0); a grid of at most 8 blocks per SM
// strides over the chunks of the launch's table range and finds each chunk's tensor by binary search.  A range may start
// anywhere in a table: its first entry's chunk0 is the base.
//
// Bit-exactness against torch: every intermediate is rounded to fp32 where torch's separate foreach ops round it (one
// register value here per stored tensor there), scalars are converted double -> float as ATen's opmath converts them, and
// ATen's `a + alpha * b` list functor, its addcmul / addcdiv (std::fma) and its lerp are written as the fused
// multiply-adds nvcc makes of them.
#include "icaf_internal.cuh"

namespace icaf {

static_assert(sizeof(icaf_optim_tensor) == 64, "table entries are 64 bytes");
constexpr int kOptThreads = 256;
constexpr int kOptIlp = ICAF_OPTIM_CHUNK / kOptThreads;
static_assert(kOptIlp * kOptThreads == ICAF_OPTIM_CHUNK, "a chunk is kOptIlp elements per thread");

// Entry of the table range [t, t + n) that holds global chunk c (the last entry whose chunk0 <= c).
__device__ __forceinline__ const icaf_optim_tensor& chunk_tensor(const icaf_optim_tensor* t, int n, long long c) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (t[mid].chunk0 <= c) lo = mid; else hi = mid - 1;
  }
  return t[lo];
}

// Calls body(entry, first element of this thread in the chunk, valid[kOptIlp]) for every chunk this block owns; element j
// of the thread is first + j * kOptThreads.
template <typename Body>
__device__ __forceinline__ void for_each_chunk(const icaf_optim_tensor* t, int n, long long n_chunks, Body body) {
  const long long base = t[0].chunk0;
  for (long long c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    const icaf_optim_tensor& e = chunk_tensor(t, n, base + c);
    const long long first = (base + c - e.chunk0) * ICAF_OPTIM_CHUNK + threadIdx.x;
    bool valid[kOptIlp];
#pragma unroll
    for (int j = 0; j < kOptIlp; ++j) valid[j] = first + (long long)j * kOptThreads < e.numel;
    body(e, first, valid);
  }
}

// GradScaler.unscale_ (torch._amp_foreach_non_finite_check_and_unscale_): g *= inv_scale with inv_scale formed in double
// as GradScaler forms it; any non-finite input element sets *found_inf = 1.
__global__ void __launch_bounds__(kOptThreads) amp_unscale_kernel(const icaf_optim_tensor* t, int n, long long n_chunks,
                                                                  const float* scale, float* found_inf) {
  pdl_launch_dependents();
  pdl_wait();
  const float inv = (float)(1.0 / (double)*scale);
  bool bad = false;
  for_each_chunk(t, n, n_chunks, [&](const icaf_optim_tensor& e, long long first, const bool (&valid)[kOptIlp]) {
    float* g = static_cast<float*>(e.g);
    float x[kOptIlp];
#pragma unroll
    for (int j = 0; j < kOptIlp; ++j) x[j] = valid[j] ? g[first + j * kOptThreads] : 0.f;
#pragma unroll
    for (int j = 0; j < kOptIlp; ++j) {
      if (!valid[j]) continue;
      bad |= !isfinite(x[j]);
      g[first + j * kOptThreads] = inv == 1.f ? x[j] : __fmul_rn(x[j], inv);
    }
  });
  if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) *found_inf = 1.f;
}

// torch.optim.SGD's _multi_tensor_sgd with nesterov=True, dampening=0, maximize=False:
//   d = g + wd p (wd != 0);  buf = buf m;  buf = buf + d;  d = d + m buf;  p = p + (-lr) d.
__global__ void __launch_bounds__(kOptThreads) sgd_step_kernel(const icaf_optim_tensor* t, int n, long long n_chunks,
                                                               const double* hyper, const float* found_inf) {
  pdl_launch_dependents();
  pdl_wait();
  if (*found_inf != 0.f) return;
  const double lr = hyper[0], momentum = hyper[1], weight_decay = hyper[2];
  const float neg_lr = (float)-lr, m = (float)momentum, wd = (float)weight_decay;
  const bool decay = weight_decay != 0.0, use_buf = momentum != 0.0;
  for_each_chunk(t, n, n_chunks, [&](const icaf_optim_tensor& e, long long first, const bool (&valid)[kOptIlp]) {
    float* p = static_cast<float*>(e.p);
    const float* g = static_cast<const float*>(e.g);
    float* buf = static_cast<float*>(e.m);
    float pv[kOptIlp], gv[kOptIlp], bv[kOptIlp];
#pragma unroll
    for (int j = 0; j < kOptIlp; ++j) {
      const long long i = first + j * kOptThreads;
      pv[j] = valid[j] ? p[i] : 0.f;
      gv[j] = valid[j] ? g[i] : 0.f;
      bv[j] = valid[j] && use_buf ? buf[i] : 0.f;
    }
#pragma unroll
    for (int j = 0; j < kOptIlp; ++j) {
      if (!valid[j]) continue;
      const long long i = first + j * kOptThreads;
      float d = decay ? __fmaf_rn(wd, pv[j], gv[j]) : gv[j];
      if (use_buf) {
        const float b = __fadd_rn(__fmul_rn(bv[j], m), d);
        d = __fmaf_rn(m, b, d);
        buf[i] = b;
      }
      p[i] = __fmaf_rn(neg_lr, d, pv[j]);
    }
  });
}

// torch.optim.Adam's _multi_tensor_adam, non-capturable branch (amsgrad=False, maximize=False, L2 weight decay), at step
// s = step + 1 of each tensor.  bias_corr holds torch's double bc1 = 1 - beta1**s and bc2_sqrt = (1 - beta2**s)**0.5 at row s.
__global__ void __launch_bounds__(kOptThreads) adam_step_kernel(const icaf_optim_tensor* t, int n, long long n_chunks,
                                                                const double* hyper, const double* bias_corr, int bc_steps,
                                                                const float* found_inf) {
  pdl_launch_dependents();
  pdl_wait();
  if (*found_inf != 0.f) return;
  const double lr = hyper[0], beta1 = hyper[1], weight_decay = hyper[2], beta2 = hyper[3], eps = hyper[4];
  const float w1 = (float)(1.0 - beta1), b2 = (float)beta2, a2 = (float)(1.0 - beta2), feps = (float)eps, wd = (float)weight_decay;
  const bool decay = weight_decay != 0.0, small = fabsf(w1) < 0.5f;
  for_each_chunk(t, n, n_chunks, [&](const icaf_optim_tensor& e, long long first, const bool (&valid)[kOptIlp]) {
    const int s = (int)*static_cast<const float*>(e.step) + 1;
    if (s >= bc_steps) return;                      // the host keeps the table ahead of every reachable step
    const float step_size = (float)((lr / bias_corr[2 * s]) * -1.0), bc2_sqrt = (float)bias_corr[2 * s + 1];
    float* p = static_cast<float*>(e.p);
    const float* g = static_cast<const float*>(e.g);
    float* m = static_cast<float*>(e.m);
    float* v = static_cast<float*>(e.v);
    float pv[kOptIlp], gv[kOptIlp], mv[kOptIlp], vv[kOptIlp];
#pragma unroll
    for (int j = 0; j < kOptIlp; ++j) {
      const long long i = first + j * kOptThreads;
      pv[j] = valid[j] ? p[i] : 0.f;
      gv[j] = valid[j] ? g[i] : 0.f;
      mv[j] = valid[j] ? m[i] : 0.f;
      vv[j] = valid[j] ? v[i] : 0.f;
    }
#pragma unroll
    for (int j = 0; j < kOptIlp; ++j) {
      if (!valid[j]) continue;
      const long long i = first + j * kOptThreads;
      const float gd = decay ? __fmaf_rn(wd, pv[j], gv[j]) : gv[j];
      const float diff = __fsub_rn(gd, mv[j]);           // ATen lerp(m, g, w1)
      const float mn = small ? __fmaf_rn(w1, diff, mv[j]) : __fmaf_rn(-diff, __fsub_rn(1.f, w1), gd);
      const float vn = __fmaf_rn(a2, __fmul_rn(gd, gd), __fmul_rn(vv[j], b2));
      const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(vn), bc2_sqrt), feps);
      p[i] = __fmaf_rn(step_size, __fdiv_rn(mn, denom), pv[j]);
      m[i] = mn;
      v[i] = vn;
    }
  });
}

// Adam's step count: += 1 per tensor when the step was taken (after adam_step_kernel has read the old counts).
__global__ void __launch_bounds__(kOptThreads) adam_count_kernel(const icaf_optim_tensor* t, int n, const float* found_inf) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || *found_inf != 0.f) return;
  float* step = static_cast<float*>(t[i].step);
  *step = __fadd_rn(*step, 1.f);
}

// torch._amp_update_scale_, then clear the flag for the next window.
__global__ void amp_update_scale_kernel(float* scale, int* growth_tracker, float* found_inf, double growth_factor,
                                        double backoff_factor, int growth_interval) {
  pdl_launch_dependents();
  pdl_wait();
  if (*found_inf != 0.f) {
    *scale = (float)((double)*scale * backoff_factor);
    *growth_tracker = 0;
  } else {
    const int successful = *growth_tracker + 1;
    if (successful == growth_interval) {
      const float grown = (float)((double)*scale * growth_factor);
      if (isfinite(grown)) *scale = grown;
      *growth_tracker = 0;
    } else {
      *growth_tracker = successful;
    }
  }
  *found_inf = 0.f;
}

// ModelEMA.update: v = v float(d), then v = v + float(1 - d) src (entry.p = the EMA tensor, entry.g = the model's).
__global__ void __launch_bounds__(kOptThreads) ema_update_kernel(const icaf_optim_tensor* t, int n, long long n_chunks,
                                                                 const double* decay) {
  pdl_launch_dependents();
  pdl_wait();
  const double d = *decay;
  const float fd = (float)d, fa = (float)(1.0 - d);
  for_each_chunk(t, n, n_chunks, [&](const icaf_optim_tensor& e, long long first, const bool (&valid)[kOptIlp]) {
    float* v = static_cast<float*>(e.p);
    const float* src = static_cast<const float*>(e.g);
    float vv[kOptIlp], sv[kOptIlp];
#pragma unroll
    for (int j = 0; j < kOptIlp; ++j) {
      const long long i = first + j * kOptThreads;
      vv[j] = valid[j] ? v[i] : 0.f;
      sv[j] = valid[j] ? src[i] : 0.f;
    }
#pragma unroll
    for (int j = 0; j < kOptIlp; ++j)
      if (valid[j]) v[first + j * kOptThreads] = __fmaf_rn(fa, sv[j], __fmul_rn(vv[j], fd));
  });
}

// Host-side checks shared by the table walkers; returns ICAF_OK or the error already set.
int check_table(const char* what, const void* table, size_t table_bytes, int n_tensors, long long n_chunks) {
  char msg[160];
  if (!table) { snprintf(msg, sizeof msg, "%s: null table", what); return set_error(ICAF_ERR_BAD_ARG, msg); }
  if (reinterpret_cast<uintptr_t>(table) & 15) { snprintf(msg, sizeof msg, "%s: table not 16-byte aligned", what); return set_error(ICAF_ERR_BAD_ARG, msg); }
  const size_t need = icaf_optim_table_bytes(n_tensors);
  if (!need || table_bytes < need || n_chunks < 0) {
    snprintf(msg, sizeof msg, "%s: the table of %zu bytes does not hold %d tensors (icaf_optim_table_bytes), or n_chunks < 0", what, table_bytes, n_tensors);
    return set_error(ICAF_ERR_BAD_ARG, msg);
  }
  return ICAF_OK;
}

unsigned optim_grid(long long n_chunks) {
  const long long cap = 8LL * sm_count_cached();
  return (unsigned)(n_chunks < cap ? n_chunks : cap);
}

}  // namespace icaf

using namespace icaf;

extern "C" size_t icaf_optim_table_bytes(int n_tensors) {
  if (n_tensors < 1) return 0;
  return (size_t)n_tensors * sizeof(icaf_optim_tensor);
}

extern "C" int icaf_amp_unscale(const void* table, size_t table_bytes, int n_tensors, int64_t n_chunks, const float* scale, float* found_inf,
                                void* stream) {
  if (int rc = check_table("amp_unscale", table, table_bytes, n_tensors, n_chunks)) return rc;
  if (!scale || !found_inf) return set_error(ICAF_ERR_BAD_ARG, "amp_unscale: null scale or found_inf");
  if (!n_chunks) return ICAF_OK;
  return launch_k("amp_unscale", amp_unscale_kernel, dim3(optim_grid(n_chunks)), dim3(kOptThreads), 0, (cudaStream_t)stream,
                  static_cast<const icaf_optim_tensor*>(table), n_tensors, (long long)n_chunks, scale, found_inf);
}

extern "C" int icaf_sgd_step(const void* table, size_t table_bytes, int n_tensors, int64_t n_chunks, const double* hyper, int group,
                             int n_groups, const float* found_inf, void* stream) {
  if (int rc = check_table("sgd_step", table, table_bytes, n_tensors, n_chunks)) return rc;
  if (!hyper || !found_inf) return set_error(ICAF_ERR_BAD_ARG, "sgd_step: null hyper or found_inf");
  if (n_groups < 1 || group < 0 || group >= n_groups) return set_error(ICAF_ERR_BAD_ARG, "sgd_step: group index outside [0, n_groups)");
  if (!n_chunks) return ICAF_OK;
  return launch_k("sgd_step", sgd_step_kernel, dim3(optim_grid(n_chunks)), dim3(kOptThreads), 0, (cudaStream_t)stream,
                  static_cast<const icaf_optim_tensor*>(table), n_tensors, (long long)n_chunks, hyper + (size_t)group * ICAF_OPTIM_HYPER,
                  found_inf);
}

extern "C" int icaf_adam_step(const void* table, size_t table_bytes, int n_tensors, int64_t n_chunks, const double* hyper, int group,
                              int n_groups, const double* bias_corr, int bc_steps, const float* found_inf, void* stream) {
  if (int rc = check_table("adam_step", table, table_bytes, n_tensors, n_chunks)) return rc;
  if (!hyper || !bias_corr || !found_inf) return set_error(ICAF_ERR_BAD_ARG, "adam_step: null hyper, bias_corr or found_inf");
  if (n_groups < 1 || group < 0 || group >= n_groups) return set_error(ICAF_ERR_BAD_ARG, "adam_step: group index outside [0, n_groups)");
  if (bc_steps < 2) return set_error(ICAF_ERR_BAD_ARG, "adam_step: the bias-correction table needs rows 0 and 1 at least");
  const cudaStream_t st = (cudaStream_t)stream;
  const icaf_optim_tensor* t = static_cast<const icaf_optim_tensor*>(table);
  if (n_chunks) {
    if (int rc = launch_k("adam_step", adam_step_kernel, dim3(optim_grid(n_chunks)), dim3(kOptThreads), 0, st, t, n_tensors,
                          (long long)n_chunks, hyper + (size_t)group * ICAF_OPTIM_HYPER, bias_corr + (size_t)group * bc_steps * 2,
                          bc_steps, found_inf))
      return rc;
  }
  return launch_k("adam_count", adam_count_kernel, dim3(blocks_for(n_tensors, kOptThreads)), dim3(kOptThreads), 0, st, t, n_tensors,
                  found_inf);
}

extern "C" int icaf_amp_update_scale(float* scale, int* growth_tracker, float* found_inf, double growth_factor, double backoff_factor,
                                     int growth_interval, void* stream) {
  if (!scale || !growth_tracker || !found_inf) return set_error(ICAF_ERR_BAD_ARG, "amp_update_scale: null pointer");
  if (growth_interval < 1 || !(growth_factor > 1.0) || !(backoff_factor < 1.0)) return set_error(ICAF_ERR_BAD_ARG, "amp_update_scale: needs growth_interval >= 1, growth_factor > 1, backoff_factor < 1");
  return launch_k("amp_update_scale", amp_update_scale_kernel, dim3(1), dim3(1), 0, (cudaStream_t)stream, scale, growth_tracker,
                  found_inf, growth_factor, backoff_factor, growth_interval);
}

extern "C" int icaf_ema_update(const void* table, size_t table_bytes, int n_tensors, int64_t n_chunks, const double* decay, void* stream) {
  if (int rc = check_table("ema_update", table, table_bytes, n_tensors, n_chunks)) return rc;
  if (!decay) return set_error(ICAF_ERR_BAD_ARG, "ema_update: null decay");
  if (!n_chunks) return ICAF_OK;
  return launch_k("ema_update", ema_update_kernel, dim3(optim_grid(n_chunks)), dim3(kOptThreads), 0, (cudaStream_t)stream,
                  static_cast<const icaf_optim_tensor*>(table), n_tensors, (long long)n_chunks, decay);
}
