// Confluence on the decoded predictions (reference: utils/confluence.py:50-193), the reference's alternative to NMS:
// boxes are clustered by a normalised Manhattan distance instead of IoU.  Two launches, no host round trip:
//   1. confluence_cluster_kernel, one block per (class c, image b): gathers class c's candidates in row order (for
//      nc == 1 the best-class branch; both branches give one candidate per (row, class) with obj > conf_thres and
//      cls_c * obj > conf_thres in fp32), then runs the selection loop in fp64 and flags the kept candidates.
//   2. confluence_compact_kernel, one block per image: writes the kept rows in ascending (row, class) order, which is the
//      reference's np.unique(keep) order over its row-major candidate list.
// Distances (confluence.py:140-162): for boxes a, b, each axis is normalised by the min and max of its four coordinates,
// p = |x1a'-x1b'| + |x2a'-x2b'| + |y1a'-y1b'| + |y2a'-y2b'| in fp64 on the exactly widened fp32 coordinates; p is exactly
// symmetric.  A degenerate axis (max == min) gives 0/0 = NaN, which compares false everywhere, as in numpy.
// Selection: value_i = min over live j != i with p_ij < 2 of p_ij / conf_i (0 when there is none); the first i with the
// smallest value is kept, and it and every live j with p_best,j < p_thres leave.  Division by a positive conf is monotone,
// so each live row keeps min p (and which j gave it) and divides once; a row is rescanned, by one warp, only when
// that j has left.
// Per-candidate state (37 bytes) sits in shared memory up to kCfSmemCap candidates per class, otherwise in the class's
// slice of the workspace: the same code on generic pointers.
#include <climits>
#include <type_traits>

#include "icaf_internal.cuh"

namespace icaf {

constexpr int kCfThreads = 256, kCfWarps = kCfThreads / 32;
constexpr int kCfCompactThreads = 512;
constexpr int kCfSmemCap = 6144;                  // 37 B each: 227 328 B of dynamic shared memory
constexpr int kCfBytesPer = 37;                   // rowmin f64, box float4, conf f32, row i32, partner i32, state u8
constexpr double kCfStart = 10000.0;              // confluence.py:133, the scan's starting minimum

struct CfParams {
  const void* z;
  int B, R, ld, nc, Rm, max_det;                  // ld: row width; Rm: R rounded up to 16, the capacity of a workspace slice
  float conf_thres;
  double p_thres;
  float* det; int* index; int* count;
  char* slices;                                   // B * nc slices of Rm candidates
  unsigned char* keep;                            // (B, R, nc): 1 where (row, class) was kept
};

struct CfStore {
  double* rowmin; float4* box; float* conf; int* row; int* part; unsigned char* state;   // state: 0 gone, 1 live, 2 kept
};
// capacity m (a multiple of 16): every array stays 16-byte aligned
__device__ __forceinline__ CfStore cf_carve(char* base, int m) {
  CfStore s;
  s.rowmin = (double*)base;
  s.box = (float4*)(base + (size_t)m * 8);
  s.conf = (float*)(base + (size_t)m * 24);
  s.row = (int*)(base + (size_t)m * 28);
  s.part = (int*)(base + (size_t)m * 32);
  s.state = (unsigned char*)(base + (size_t)m * 36);
  return s;
}

// input modes: 0 = fp16 predictions, 1 = fp32 predictions (confluence_process), 2 = fp32 detection rows (confluence)
template <int M> using CfT = std::conditional_t<M == 0, __half, float>;
__device__ __forceinline__ float cf_ld(const __half* p) { return __half2float(*p); }
__device__ __forceinline__ float cf_ld(const float* p) { return *p; }

// whether (row, class c) is a candidate, and its confidence: cls_c * obj in fp32 above conf_thres for predictions
// (confluence_process:61-91), the row's own conf where its cls equals c for detection rows (confluence:123)
template <int M>
__device__ __forceinline__ bool cf_cand(const CfT<M>* row, int c, float thr, float& conf) {
  if constexpr (M == 2) {
    conf = row[4];
    return row[5] == float(c);
  } else {
    const float obj = cf_ld(row + 4);
    conf = __fmul_rn(cf_ld(row + 5 + c), obj);
    return obj > thr && conf > thr;
  }
}
// xywh2xyxy of confluence.py:6-13 in fp32 (detection rows are xyxy already)
template <int M>
__device__ __forceinline__ float4 cf_box(const CfT<M>* row) {
  if constexpr (M == 2) return make_float4(row[0], row[1], row[2], row[3]);
  const float cx = cf_ld(row), cy = cf_ld(row + 1), hw = __fmul_rn(cf_ld(row + 2), 0.5f), hh = __fmul_rn(cf_ld(row + 3), 0.5f);
  return make_float4(__fsub_rn(cx, hw), __fsub_rn(cy, hh), __fadd_rn(cx, hw), __fadd_rn(cy, hh));
}

// a / d correctly rounded, for 0 <= a <= d and for a = value numerators: operands are sums of widened fp32 values, so no
// quotient, product or remainder below leaves fp64's normal range.  __ddiv_rn would call its out-of-range path, and the
// call saves live registers to the stack.  The Newton quotient is within one ulp; the exact fma remainders of it and of
// its neighbour on the remainder's side pick the nearer (ties to even).  d == 0 only when a == 0 here: 0/0 = NaN.
__device__ __forceinline__ double cf_div(double a, double d) {
  if (d == 0.0) return __longlong_as_double(0x7ff8000000000000ll);
  double y;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(d));
  double e = __fma_rn(-d, y, 1.0);
  y = __fma_rn(y, e, y);
  e = __fma_rn(-d, y, 1.0);
  y = __fma_rn(y, e, y);
  double q = __dmul_rn(a, y);
  const double r = __fma_rn(-d, q, a);
  q = __fma_rn(r, y, q);
  const double r1 = __fma_rn(-d, q, a);
  if (r1 != 0.0) {
    const double q2 = __longlong_as_double(__double_as_longlong(q) + (r1 > 0.0 ? 1 : -1));
    const double r2 = __fma_rn(-d, q2, a);
    if (fabs(r2) < fabs(r1) || (fabs(r2) == fabs(r1) && !(__double_as_longlong(q2) & 1))) q = q2;
  }
  return q;
}

// one axis: |a1' - b1'| and |a2' - b2'| after normalising by the min and max of the four coordinates
__device__ __forceinline__ void cf_axis(double a1, double a2, double b1, double b2, double& t1, double& t2) {
  const double mn = fmin(fmin(a1, a2), fmin(b1, b2)), mx = fmax(fmax(a1, a2), fmax(b1, b2));
  const double d = __dsub_rn(mx, mn);
  const double na1 = cf_div(__dsub_rn(a1, mn), d), na2 = cf_div(__dsub_rn(a2, mn), d);
  const double nb1 = cf_div(__dsub_rn(b1, mn), d), nb2 = cf_div(__dsub_rn(b2, mn), d);
  t1 = fabs(__dsub_rn(na1, nb1));
  t2 = fabs(__dsub_rn(na2, nb2));
}
__device__ __forceinline__ double cf_p(const float4& a, const float4& b) {
  double x1, x2, y1, y2;
  cf_axis(a.x, a.z, b.x, b.z, x1, x2);
  cf_axis(a.y, a.w, b.y, b.w, y1, y2);
  return __dadd_rn(__dadd_rn(__dadd_rn(x1, x2), y1), y2);
}

// one warp: min p over the live j != i with p < 2, and the first j that gives it (-1: none)
__device__ __forceinline__ void cf_scan_row(const CfStore& s, int n, int i, int lane) {
  const float4 bi = s.box[i];
  double best = 2.0;
  int part = -1;
  for (int j = lane; j < n; j += 32) {
    if (j == i || s.state[j] != 1) continue;
    const double p = cf_p(bi, s.box[j]);
    if (p < best) { best = p; part = j; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int op = __shfl_xor_sync(0xffffffffu, part, o);
    if (ob < best || (ob == best && op < part)) { best = ob; part = op; }
  }
  if (lane == 0) { s.rowmin[i] = best; s.part[i] = part; }
}

template <int M>
__global__ void __launch_bounds__(kCfThreads) confluence_cluster_kernel(const CfParams P) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ __align__(16) char cf_smem[];
  __shared__ int warp_n[kCfWarps];
  __shared__ double red_v[kCfWarps];
  __shared__ int red_i[kCfWarps];
  __shared__ int s_n, s_best;
  const int c = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const CfT<M>* z = (const CfT<M>*)P.z + (size_t)b * P.R * P.ld;
  unsigned char* keep = P.keep + (size_t)b * P.R * P.nc + c;

  // count this class's candidates (and clear its keep flags)
  int my = 0;
  for (int r = tid; r < P.R; r += kCfThreads) {
    float conf;
    my += cf_cand<M>(z + (size_t)r * P.ld, c, P.conf_thres, conf);
    keep[(size_t)r * P.nc] = 0;
  }
  my = __reduce_add_sync(0xffffffffu, my);
  if (lane == 0) warp_n[warp] = my;
  __syncthreads();
  if (tid == 0) {
    int n = 0;
    for (int w = 0; w < kCfWarps; ++w) n += warp_n[w];
    s_n = n;
  }
  __syncthreads();
  const int n = s_n;
  if (n == 0) return;
  const CfStore s = cf_carve(n <= kCfSmemCap ? cf_smem : P.slices + ((size_t)b * P.nc + c) * P.Rm * kCfBytesPer,
                             n <= kCfSmemCap ? min(P.Rm, kCfSmemCap) : P.Rm);

  // gather in row order: a block-wide compaction per chunk of kCfThreads rows
  int base = 0;
  for (int r0 = 0; r0 < P.R; r0 += kCfThreads) {
    const int r = r0 + tid;
    float conf;
    const bool cand = r < P.R && cf_cand<M>(z + (size_t)r * P.ld, c, P.conf_thres, conf);
    const unsigned ball = __ballot_sync(0xffffffffu, cand);
    __syncthreads();                                   // warp_n of the previous chunk has been read
    if (lane == 0) warp_n[warp] = __popc(ball);
    __syncthreads();
    int off = base, total = 0;
    for (int w = 0; w < kCfWarps; ++w) {
      if (w < warp) off += warp_n[w];
      total += warp_n[w];
    }
    if (cand) {
      const int k = off + __popc(ball & ((1u << lane) - 1u));
      s.box[k] = cf_box<M>(z + (size_t)r * P.ld);
      s.conf[k] = conf;
      s.row[k] = r;
      s.state[k] = 1;
    }
    base += total;
  }
  __syncthreads();
  for (int i = warp; i < n; i += kCfWarps) cf_scan_row(s, n, i, lane);
  __syncthreads();

  for (;;) {
    // arg-min of value over the live rows, the first index winning ties
    double v = kCfStart;
    int vi = INT_MAX;
    for (int i = tid; i < n; i += kCfThreads) {
      if (s.state[i] != 1) continue;
      const double val = s.part[i] < 0 ? 0.0 : cf_div(s.rowmin[i], (double)s.conf[i]);
      if (val < v) { v = val; vi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double ov = __shfl_xor_sync(0xffffffffu, v, o);
      const int oi = __shfl_xor_sync(0xffffffffu, vi, o);
      if (ov < v || (ov == v && oi < vi)) { v = ov; vi = oi; }
    }
    if (lane == 0) { red_v[warp] = v; red_i[warp] = vi; }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < kCfWarps; ++w)
        if (red_v[w] < v || (red_v[w] == v && red_i[w] < vi)) { v = red_v[w]; vi = red_i[w]; }
      s_best = vi;
    }
    __syncthreads();
    const int best = s_best;
    if (best == INT_MAX) break;                        // no live row left
    const float4 bb = s.box[best];
    for (int j = tid; j < n; j += kCfThreads)
      if (j != best && s.state[j] == 1 && cf_p(bb, s.box[j]) < P.p_thres) s.state[j] = 0;
    if (tid == 0) s.state[best] = 2;
    __syncthreads();
    for (int i = warp; i < n; i += kCfWarps) {           // warp-uniform test: the rows whose minimum's neighbour left
      const int pj = s.part[i];
      if (s.state[i] == 1 && pj >= 0 && s.state[pj] != 1) cf_scan_row(s, n, i, lane);
    }
    __syncthreads();
  }
  for (int i = tid; i < n; i += kCfThreads)
    if (s.state[i] == 2) keep[(size_t)s.row[i] * P.nc] = 1;
}

// one block per image: the kept (row, class) pairs in ascending order, the first max_det written, the true count kept
template <int M>
__global__ void __launch_bounds__(kCfCompactThreads) confluence_compact_kernel(const CfParams P) {
  pdl_launch_dependents();
  pdl_wait();
  constexpr int kWarps = kCfCompactThreads / 32;
  __shared__ int warp_n[kWarps];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const CfT<M>* z = (const CfT<M>*)P.z + (size_t)b * P.R * P.ld;
  const unsigned char* keep = P.keep + (size_t)b * P.R * P.nc;
  float* det = P.det + (size_t)b * P.max_det * 6;
  const int S = P.R * P.nc;
  int base = 0;
  for (int s0 = 0; s0 < S; s0 += kCfCompactThreads) {
    const int s = s0 + tid;
    const bool kept = s < S && keep[s];
    const unsigned ball = __ballot_sync(0xffffffffu, kept);
    __syncthreads();
    if (lane == 0) warp_n[warp] = __popc(ball);
    __syncthreads();
    int off = base, total = 0;
    for (int w = 0; w < kWarps; ++w) {
      if (w < warp) off += warp_n[w];
      total += warp_n[w];
    }
    const int k = off + __popc(ball & ((1u << lane) - 1u));
    if (kept && k < P.max_det) {
      const int r = s / P.nc, c = s - r * P.nc;
      const CfT<M>* row = z + (size_t)r * P.ld;
      const float4 bx = cf_box<M>(row);
      float conf;
      cf_cand<M>(row, c, P.conf_thres, conf);
      float* d = det + (size_t)k * 6;
      d[0] = bx.x; d[1] = bx.y; d[2] = bx.z; d[3] = bx.w; d[4] = conf; d[5] = float(c);
      if (P.index) P.index[(size_t)b * P.max_det + k] = r;
    }
    base += total;
  }
  if (tid == 0) P.count[b] = base;
}

}  // namespace icaf

using namespace icaf;

static size_t cf_slices_bytes(int B, int R, int no) {
  return (size_t)B * (no - 5) * (size_t)((R + 15) / 16 * 16) * kCfBytesPer;
}

extern "C" size_t icaf_confluence_workspace_bytes(int B, int R, int no) {
  if (B < 1 || R < 1 || no < 6 || (long long)R * (no - 5) > INT_MAX - 1024) return 0;
  return cf_slices_bytes(B, R, no) + (size_t)B * R * (no - 5);
}

template <int M>
static int cf_launch(const CfParams& P, cudaStream_t st) {
  static bool done[kMaxDevices];
  if (int rc = configure_smem(confluence_cluster_kernel<M>, kCfSmemCap * kCfBytesPer, done, "confluence: smem")) return rc;
  const int smem = min(P.Rm, kCfSmemCap) * kCfBytesPer;
  if (int rc = launch_k("confluence(cluster)", confluence_cluster_kernel<M>, dim3((unsigned)P.nc, (unsigned)P.B), dim3(kCfThreads),
                        (size_t)smem, st, P))
    return rc;
  return launch_k("confluence(compact)", confluence_compact_kernel<M>, dim3(P.B), dim3(kCfCompactThreads), 0, st, P);
}

extern "C" int icaf_confluence(const void* z, int dtype, int B, int R, int no, float conf_thres, double p_thres, float* det,
                               int* index, int max_det, int* count, void* workspace, size_t workspace_bytes, void* stream) {
  if (!z || !det || !count || !workspace) return set_error(ICAF_ERR_BAD_ARG, "confluence: null pointer");
  if (dtype < 0 || dtype > 2) return set_error(ICAF_ERR_BAD_ARG, "confluence: dtype must be 0 (fp16), 1 (fp32) or 2 (fp32 detection rows)");
  if (B < 1 || R < 1 || no < 6 || max_det < 1) return set_error(ICAF_ERR_BAD_ARG, "confluence: bad shape (B, R, max_det >= 1, no >= 6)");
  if (B > 65535 || (long long)R * (no - 5) > INT_MAX - 1024)
    return set_error(ICAF_ERR_UNSUPPORTED, "confluence: B <= 65535 and R * nc must fit in int");
  // value = p / conf with p < 2 stays below the reference's starting minimum of 10000 only while conf > 2e-4; below that
  // the reference can find no box to keep and raises
  if (dtype != 2 && !(conf_thres >= 2.5e-4f)) return set_error(ICAF_ERR_BAD_ARG, "confluence: conf_thres must be >= 2.5e-4");
  if (p_thres != p_thres) return set_error(ICAF_ERR_BAD_ARG, "confluence: p_thres is NaN");
  const size_t need = icaf_confluence_workspace_bytes(B, R, no);
  if (workspace_bytes < need || (reinterpret_cast<uintptr_t>(workspace) & 15))
    return set_error(ICAF_ERR_BAD_ARG, "confluence: workspace too small (icaf_confluence_workspace_bytes) or not 16-byte aligned");
  CfParams P = {};
  P.z = z; P.B = B; P.R = R; P.ld = dtype == 2 ? 6 : no; P.nc = no - 5; P.Rm = (R + 15) / 16 * 16; P.max_det = max_det;
  P.conf_thres = conf_thres; P.p_thres = p_thres; P.det = det; P.index = index; P.count = count;
  P.slices = (char*)workspace;
  P.keep = (unsigned char*)workspace + cf_slices_bytes(B, R, no);
  cudaStream_t st = (cudaStream_t)stream;
  return dtype == 0 ? cf_launch<0>(P, st) : dtype == 1 ? cf_launch<1>(P, st) : cf_launch<2>(P, st);
}
