// Detection output: the Detect decode of one level (sigmoid, grid / anchor transform, raw logits) and the batched
// non-maximum suppression on the decoded predictions (best-class and multi-label branches, with their workspace sizes).
#include <climits>

#include "icaf_internal.cuh"

namespace icaf {

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

}  // namespace icaf

using namespace icaf;

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
