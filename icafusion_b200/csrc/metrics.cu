// Validation metrics: per-image matching of the NMS detections to the labels (test.py:196-227), one launch per batch; the
// KAIST log-average miss rate (evaluation_script/evaluation_script.py), and the %g rounding of test.py's result lines.
#include <cub/device/device_radix_sort.cuh>

#include "icaf_internal.cuh"

namespace icaf {

// One CTA per image, kMatchThreads threads.  The image's predictions are taken in chunks of kMatchThreads rows (one row per
// thread).  For each chunk:
//   1. the block walks `targets` in tiles of kMatchThreads rows; a ballot compacts the tile's rows of this image into shared
//      memory in row order (scaled to native pixels on the way), and every thread keeps the first label of its prediction's
//      class with the largest box_iou.  Labels are visited in row order, so "first" is the reference's `.max(1)` index.
//   2. warp 0 runs the greedy assignment over the chunk in row (= confidence) order, 32 rows at a time: a row is assigned when
//      its best IoU is > iouv[0], it is the first row of its 32 with that label (__match_any_sync) and the label is not yet
//      detected by an earlier row (a flag per target row in the workspace, zeroed by the first chunk's walk).
// The reference loops over the label classes (test.py:209) and breaks once every label is detected (:226-227).  Classes
// partition both the labels and the predictions, and a prediction only ever looks at labels of its own class, so one pass over
// all rows in row order assigns exactly what the per-class loops do.  The break is a pure early exit: once all labels are
// detected, no later row can be assigned.  Hence neither is needed here.
// Arithmetic mirrors the reference's fp32 CPU ops one for one (`__f*_rn`: nothing is contracted).  scale_coords divides by
// `gain` (IEEE division, as the CPU reference does; torch on CUDA multiplies by 1/gain instead).
constexpr int kMatchThreads = 256, kMatchMaxIou = 32;
struct MatchParams {
  const float* det; const int* count; const float* targets; const float* ratio_pad; const float* iouv;
  unsigned char* correct; float* native; int* detected;
  int B, max_det, T, niou, single_cls;
  float height, width;
};
__device__ __forceinline__ float clamp_to(float v, float hi) { return fminf(fmaxf(v, 0.f), hi); }
// utils/general.py:386-407 scale_coords with ratio_pad: subtract the pad, divide by the gain, clip to the original image
__device__ __forceinline__ float4 scale_coords(float4 b, const float* rp) {
  const float h0 = rp[0], w0 = rp[1], gain = rp[2], padw = rp[3], padh = rp[4];
  b.x = clamp_to(__fdiv_rn(__fsub_rn(b.x, padw), gain), w0);
  b.y = clamp_to(__fdiv_rn(__fsub_rn(b.y, padh), gain), h0);
  b.z = clamp_to(__fdiv_rn(__fsub_rn(b.z, padw), gain), w0);
  b.w = clamp_to(__fdiv_rn(__fsub_rn(b.w, padh), gain), h0);
  return b;
}
// utils/general.py:455-477 box_iou for one pair
__device__ __forceinline__ float box_iou(const float4& a, const float4& b) {
  const float area1 = __fmul_rn(__fsub_rn(a.z, a.x), __fsub_rn(a.w, a.y));
  const float area2 = __fmul_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y));
  const float iw = fmaxf(__fsub_rn(fminf(a.z, b.z), fmaxf(a.x, b.x)), 0.f);
  const float ih = fmaxf(__fsub_rn(fminf(a.w, b.w), fmaxf(a.y, b.y)), 0.f);
  const float inter = __fmul_rn(iw, ih);
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(area1, area2), inter));
}
__global__ void __launch_bounds__(kMatchThreads) match_detections_kernel(const MatchParams P) {
  pdl_launch_dependents();
  pdl_wait();
  constexpr int kWarps = kMatchThreads / 32;
  __shared__ float4 s_box[kMatchThreads];      // one tile of this image's labels, native pixels
  __shared__ float s_cls[kMatchThreads];
  __shared__ int s_row[kMatchThreads];
  __shared__ int s_wcnt[kWarps];
  __shared__ float s_best[kMatchThreads];      // per prediction of the chunk: best IoU (NaN if any IoU was NaN) and its label row
  __shared__ int s_lab[kMatchThreads];
  __shared__ float s_iouv[kMatchMaxIou];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* rp = P.ratio_pad + (size_t)b * 5;
  const float* det = P.det + (size_t)b * P.max_det * 6;
  const int n = min(max(P.count[b], 0), P.max_det);
  if (tid < P.niou) s_iouv[tid] = P.iouv[tid];
  for (int i = n * P.niou + tid; i < P.max_det * P.niou; i += kMatchThreads)    // rows past the count
    P.correct[(size_t)b * P.max_det * P.niou + i] = 0;
  if (P.native)
    for (int i = n * 4 + tid; i < P.max_det * 4; i += kMatchThreads) P.native[(size_t)b * P.max_det * 4 + i] = 0.f;
  const float fb = float(b);
  for (int c0 = 0; c0 < n; c0 += kMatchThreads) {
    const int r = c0 + tid;
    float4 pb = make_float4(0.f, 0.f, 0.f, 0.f);
    float pcls = 0.f;
    if (r < n) {
      const float* d = det + (size_t)r * 6;
      pb = scale_coords(make_float4(d[0], d[1], d[2], d[3]), rp);
      pcls = P.single_cls ? 0.f : d[5];
      if (P.native) reinterpret_cast<float4*>(P.native)[(size_t)b * P.max_det + r] = pb;
    }
    float best = -1.f;
    int lab = -1;
    bool nan = false;
    for (int t0 = 0; t0 < P.T; t0 += kMatchThreads) {
      const int t = t0 + tid;
      const float* tg = P.targets + (size_t)t * 6;
      const bool mine = t < P.T && tg[0] == fb;
      const unsigned bal = __ballot_sync(0xffffffffu, mine);
      __syncthreads();                         // the previous tile is consumed
      if (lane == 0) s_wcnt[warp] = __popc(bal);
      __syncthreads();
      int slot = __popc(bal & ((1u << lane) - 1u)), nt = 0;
      for (int w = 0; w < kWarps; ++w) {
        if (w < warp) slot += s_wcnt[w];
        nt += s_wcnt[w];
      }
      if (mine) {
        const float x = __fmul_rn(tg[2], P.width), y = __fmul_rn(tg[3], P.height);     // test.py:136, to pixels
        const float w = __fmul_rn(tg[4], P.width), h = __fmul_rn(tg[5], P.height);
        const float hw = __fdiv_rn(w, 2.f), hh = __fdiv_rn(h, 2.f);                  // xywh2xyxy, general.py:332-339
        s_box[slot] = scale_coords(make_float4(__fsub_rn(x, hw), __fsub_rn(y, hh), __fadd_rn(x, hw), __fadd_rn(y, hh)), rp);
        s_cls[slot] = tg[1];
        s_row[slot] = t;
        if (c0 == 0) P.detected[t] = 0;
      }
      __syncthreads();
      if (r < n) {
        for (int k = 0; k < nt; ++k) {
          if (s_cls[k] != pcls) continue;
          const float v = box_iou(pb, s_box[k]);
          if (v != v) nan = true;              // torch's max propagates NaN: such a row is never assigned
          else if (v > best) { best = v; lab = s_row[k]; }
        }
      }
    }
    s_best[tid] = nan ? __int_as_float(0x7fffffff) : best;
    s_lab[tid] = lab;
    __syncthreads();
    if (warp == 0) {
      const int m = min(kMatchThreads, n - c0);
      for (int s0 = 0; s0 < m; s0 += 32) {
        const int i = s0 + lane;
        const float v = i < m ? s_best[i] : 0.f;
        const int L = i < m && v > s_iouv[0] ? s_lab[i] : -1;
        const unsigned peers = __match_any_sync(0xffffffffu, L);
        bool hit = L >= 0 && (peers & ((1u << lane) - 1u)) == 0 && !P.detected[L];
        __syncwarp();
        if (hit) P.detected[L] = 1;
        __syncwarp();
        if (i < m) {
          unsigned char* row = P.correct + ((size_t)b * P.max_det + c0 + i) * P.niou;
          for (int k = 0; k < P.niou; ++k) row[k] = hit && v > s_iouv[k];
        }
      }
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// KAIST log-average miss rate: KAISTPedEval.evaluate / accumulate (evaluation_script.py:83-386) for the nine evaluations of
// evaluate() (:546-629).  Arithmetic is float64 through __d*_rn (nothing contracted), in the reference's operation order.
constexpr int kMrSetups = 7, kMrEvals = 9, kMrThrs = 9, kMrMaxDet = 1000, kMrMatchThreads = 32 * kMrSetups;
constexpr int kMrScanThreads = 1024, kMrScanItems = 8;
// KAISTParams.setDetParams: HtRng, OccRng (as bit masks over occlusion 0..2), bndRng and fppiThrs
__constant__ double kMrHt[kMrSetups][2] = {{55, 1e10}, {115, 1e10}, {45, 115}, {1, 45}, {1, 1e10}, {1, 1e10}, {1, 1e10}};
__constant__ int kMrOcc[kMrSetups] = {3, 1, 1, 1, 1, 2, 4};
__constant__ double kMrFppi[kMrThrs] = {0.0100, 0.0178, 0.0316, 0.0562, 0.1000, 0.1778, 0.3162, 0.5623, 1.0000};
__constant__ int kMrSetupOf[kMrEvals] = {0, 0, 0, 1, 2, 3, 4, 5, 6};   // all, day, night, near .. heavy
constexpr unsigned long long kMrAbsent = ~0ull, kMrNanKey = ~0ull - 1;

// Ascending order of this key is numpy's stable argsort of -score (mergesort): -0 == +0, NaN after every number.
// Slots without a detection get kMrAbsent, so every detection sorts before every empty slot.
__device__ __forceinline__ unsigned long long mr_desc_key(double score) {
  double x = -score;
  if (x != x) return kMrNanKey;
  if (x == 0.0) x = 0.0;
  const unsigned long long b = (unsigned long long)__double_as_longlong(x);
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
// Python's min(a, b) / max(a, b): the first argument unless the second compares strictly smaller / larger
__device__ __forceinline__ double py_min(double a, double b) { return b < a ? b : a; }
__device__ __forceinline__ double py_max(double a, double b) { return b > a ? b : a; }
// KAISTPedEval.iou (:148-179) for one pair; 0 where the loop `continue`s.  crowd (an ignored gt): the union is the
// detection's area.
__device__ __forceinline__ double mr_iou(double dx, double dy, double dw, double dh, double gx, double gy, double gw, double gh,
                                         bool crowd) {
  const double gx2 = __dadd_rn(gx, gw), gy2 = __dadd_rn(gy, gh), garea = __dmul_rn(gw, gh);
  const double dx2 = __dadd_rn(dx, dw), dy2 = __dadd_rn(dy, dh), darea = __dmul_rn(dw, dh);
  const double uw = __dsub_rn(py_min(dx2, gx2), py_max(dx, gx));
  if (uw <= 0.0) return 0.0;
  const double uh = __dsub_rn(py_min(dy2, gy2), py_max(dy, gy));
  if (uh <= 0.0) return 0.0;
  const double t = __dmul_rn(uw, uh);
  return __ddiv_rn(t, crowd ? darea : __dsub_rn(__dadd_rn(darea, garea), t));
}

struct MrParams {
  const double* gt_box; const double* gt_height; const int* gt_occ; const int* gt_ignore; const long long* gt_id;
  const int* gt_offset; const double* rows; const int* span;
  int images, gts, day, nrows, max_per_image;
  double* ys; int* counts; double* curves;
  // workspace
  unsigned long long* key; int* val; int* slot_img; unsigned* flags; unsigned char* gt_state; int* npig; int* present;
};

// Zero the per-run state: every slot empty, the sort's values the slot indices.
__global__ void __launch_bounds__(256) kaist_mr_init_kernel(const MrParams P) {
  pdl_launch_dependents();
  pdl_wait();
  const int r = blockIdx.x * 256 + threadIdx.x;
  if (r < P.nrows) {
    P.key[r] = kMrAbsent;
    P.val[r] = r;
    P.flags[r] = 0;
    P.slot_img[r] = 0;
  }
  if (r < 2 * kMrSetups) P.npig[r] = 0;
  if (r == 0) *P.present = 0;
}

// One CTA per image, one warp per setup.  The CTA ranks the image's detections stably by -score (computeIoU's and
// evaluateImg's argsort); slot offset + i then holds the detection of rank i.  Warp s gives every gt of the image its setup-s
// ignore flag (_prepare, :59-71) and runs evaluateImg's greedy loop (:225-258) over the detections in rank order.  The IoU
// row of rank i is that of the detection of rank order[order[i]]: computeIoU has already sorted the rows and evaluateImg
// indexes them by dtind again.  Per detection, over the gts spread across the lanes (32 per chunk):
//   - the regular gts come first (gts are sorted ignored-last, stably): the unmatched one with the largest IoU >= 0.5 wins,
//     ties to the later gt (the loop's test is `<`).  A NaN IoU passes every later test, so with one the last unmatched
//     regular gt wins.
//   - otherwise the first ignored gt with !(IoA < 0.5); the loop breaks at the next ignored gt, and ignored gts stay free.
// flags[slot] bit 2s: the detection is kept in setup s (dtIgnore == 0); bit 2s+1: it is a true positive there (dtMatches,
// the gt's annotation id, is nonzero: a match on annotation id 0 counts as a false positive).
__global__ void __launch_bounds__(kMrMatchThreads) kaist_mr_match_kernel(const MrParams P) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ unsigned long long s_key[kMrMaxDet];
  __shared__ short s_order[kMrMaxDet];
  __shared__ unsigned s_flags[kMrMaxDet];
  const int img = blockIdx.x, tid = threadIdx.x, lane = tid & 31, s = tid >> 5;
  const int off = P.span[2 * img];
  int n = min(max(P.span[2 * img + 1], 0), P.max_per_image);
  if (off < 0 || off > P.nrows) n = 0;
  else n = min(n, P.nrows - off);
  const double* rows = P.rows + (size_t)max(off, 0) * 5;
  for (int i = tid; i < n; i += kMrMatchThreads) {
    s_key[i] = mr_desc_key(rows[(size_t)i * 5 + 4]);
    s_flags[i] = 0;
  }
  __syncthreads();
  for (int i = tid; i < n; i += kMrMatchThreads) {
    const unsigned long long k = s_key[i];
    int rank = 0;
    for (int j = 0; j < n; ++j) rank += s_key[j] < k || (s_key[j] == k && j < i);
    s_order[rank] = (short)i;
  }
  __syncthreads();
  // this warp's setup: ignore flags and the regular-gt count (npig counts images with detections only)
  const int g0 = P.gt_offset[img], G = P.gt_offset[img + 1] - g0;
  unsigned char* state = P.gt_state + (size_t)s * P.gts + g0;     // bit 0: ignored in setup s, bit 1: matched
  int regular = 0;
  for (int c0 = 0; c0 < G; c0 += 32) {
    const int g = c0 + lane;
    bool ig = false;
    if (g < G) {
      const double* b = P.gt_box + (size_t)(g0 + g) * 4;
      const double h = P.gt_height[g0 + g];
      const int occ = P.gt_occ[g0 + g];
      ig = P.gt_ignore[g0 + g] != 0 || h < kMrHt[s][0] || h > kMrHt[s][1] ||
           !(occ >= 0 && occ < 3 && ((kMrOcc[s] >> occ) & 1)) || b[0] < 5.0 || b[1] < 5.0 ||
           __dadd_rn(b[0], b[2]) > 635.0 || __dadd_rn(b[1], b[3]) > 507.0;
      state[g] = ig ? 1 : 0;
    }
    regular += __popc(__ballot_sync(0xffffffffu, g < G && !ig));
  }
  if (lane == 0 && n > 0 && regular > 0) atomicAdd(&P.npig[2 * s + (img >= P.day)], regular);
  __syncwarp();
  for (int i = 0; i < n; ++i) {
    const double* d = rows + (size_t)s_order[s_order[i]] * 5;
    const double dx = d[0], dy = d[1], dw = d[2], dh = d[3];
    double bv = -1.0;
    int bi = -1, last_reg = -1, first_ig = 0x7fffffff;
    bool nan_reg = false;
    for (int c0 = 0; c0 < G; c0 += 32) {
      const int g = c0 + lane;
      if (g >= G) break;
      const unsigned char st = state[g];
      if (st & 2) continue;                                      // a matched regular gt
      const double* b = P.gt_box + (size_t)(g0 + g) * 4;
      const double v = mr_iou(dx, dy, dw, dh, b[0], b[1], b[2], b[3], st & 1);
      if (!(st & 1)) {
        last_reg = g;
        if (v != v) nan_reg = true;
        else if (v >= 0.5 && v >= bv) { bv = v; bi = g; }
      } else if (!(v < 0.5) && first_ig == 0x7fffffff) {
        first_ig = g;
      }
    }
    int match;
    if (__any_sync(0xffffffffu, nan_reg)) {
      match = last_reg;
      for (int o = 16; o; o >>= 1) match = max(match, __shfl_xor_sync(0xffffffffu, match, o));
    } else {
      for (int o = 16; o; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > bv || (ov == bv && oi > bi)) { bv = ov; bi = oi; }
      }
      match = bi;
    }
    bool kept = true, tp = false;
    if (match >= 0) {
      tp = P.gt_id[g0 + match] != 0;
      if (lane == 0) state[match] = 3;                          // gtMatches = the detection's id (>= 1)
    } else {
      for (int o = 16; o; o >>= 1) first_ig = min(first_ig, __shfl_xor_sync(0xffffffffu, first_ig, o));
      kept = first_ig == 0x7fffffff;                            // matched to an ignored gt: dtIgnore = 1
    }
    if (lane == 0 && kept) atomicOr(&s_flags[i], (1u << (2 * s)) | ((unsigned)tp << (2 * s + 1)));
    __syncwarp();
  }
  __syncthreads();
  for (int i = tid; i < n; i += kMrMatchThreads) {
    P.key[off + i] = s_key[s_order[i]];
    P.flags[off + i] = s_flags[i];
    P.slot_img[off + i] = img;
  }
  if (tid == 0 && n > 0) atomicAdd(P.present, n);
}

struct MrTri { int kept, tp, fp; };
__device__ __forceinline__ MrTri operator+(MrTri a, MrTri b) { return {a.kept + b.kept, a.tp + b.tp, a.fp + b.fp}; }

// Exclusive block scan over kMrScanThreads threads; *total gets the block's sum.
__device__ MrTri mr_block_scan(MrTri v, MrTri* s_warp, MrTri* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  MrTri inc = v;
  for (int o = 1; o < 32; o <<= 1) {
    MrTri u{__shfl_up_sync(0xffffffffu, inc.kept, o), __shfl_up_sync(0xffffffffu, inc.tp, o),
            __shfl_up_sync(0xffffffffu, inc.fp, o)};
    if (lane >= o) inc = inc + u;
  }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    MrTri w = s_warp[lane], wi = w;
    for (int o = 1; o < 32; o <<= 1) {
      MrTri u{__shfl_up_sync(0xffffffffu, wi.kept, o), __shfl_up_sync(0xffffffffu, wi.tp, o),
              __shfl_up_sync(0xffffffffu, wi.fp, o)};
      if (lane >= o) wi = wi + u;
    }
    s_warp[lane] = MrTri{wi.kept - w.kept, wi.tp - w.tp, wi.fp - w.fp};
    if (lane == 31) *total = wi;
  }
  __syncthreads();
  const MrTri base = s_warp[warp];
  return MrTri{base.kept + inc.kept - v.kept, base.tp + inc.tp - v.tp, base.fp + inc.fp - v.fp};
}

// One CTA per evaluation: accumulate (:296-386) over the detections in global -score order (one stable sort serves all
// nine evaluations: the order does not depend on the setup, and restricting a stable order to a subset keeps it stable).
// The kept detections (dtIgnore == 0, image in the evaluation's range) give cumulative TP / FP; fppi = fp / I0 and
// recall = tp / npig.  searchsorted(fppi, thr, 'right') - 1 is the last kept detection before the (K+1)-th false positive,
// K the largest count with K / I0 <= thr; an index of -1 reads the LAST recall (Python indexing), and with no kept
// detection the IndexError leaves q at 0.  npig == 0 (or no image with a detection) leaves ys at -1.
__global__ void __launch_bounds__(kMrScanThreads) kaist_mr_accumulate_kernel(const MrParams P) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ MrTri s_warp[32];
  __shared__ MrTri s_total, s_carry;
  __shared__ long long s_K[kMrThrs];
  __shared__ int s_kb[kMrThrs], s_tb[kMrThrs];
  const int e = blockIdx.x, tid = threadIdx.x, s = kMrSetupOf[e];
  const int day = min(P.day, P.images);
  const int lo = e == 2 ? day : 0, hi = e == 1 ? day : P.images;
  const int I0 = hi - lo;
  const int npig = e == 1 ? P.npig[2 * s] : e == 2 ? P.npig[2 * s + 1] : P.npig[2 * s] + P.npig[2 * s + 1];
  double* ys = P.ys + e * kMrThrs;
  if (I0 <= 0 || npig == 0) {
    if (tid < kMrThrs) ys[tid] = -1.0;
    if (tid == 0) { P.counts[3 * e] = 0; P.counts[3 * e + 1] = 0; P.counts[3 * e + 2] = npig; }
    return;
  }
  const double dI0 = (double)I0, dnpig = (double)npig;
  if (tid < kMrThrs) {
    const double thr = kMrFppi[tid];
    long long K = (long long)floor(thr * dI0);
    while (__ddiv_rn((double)(K + 1), dI0) <= thr) ++K;
    while (K > 0 && __ddiv_rn((double)K, dI0) > thr) --K;
    s_K[tid] = K;
    s_kb[tid] = -1;
    s_tb[tid] = 0;
  }
  if (tid == 0) s_carry = MrTri{0, 0, 0};
  __syncthreads();
  const int present = *P.present;
  const unsigned kbit = 1u << (2 * s), tbit = 1u << (2 * s + 1);
  double* xx = P.curves ? P.curves + (size_t)e * 2 * P.nrows : nullptr;
  double* yy = xx ? xx + P.nrows : nullptr;
  for (int t0 = 0; t0 < present; t0 += kMrScanThreads * kMrScanItems) {
    const int j0 = t0 + tid * kMrScanItems;
    unsigned char code[kMrScanItems];                           // bit 0 kept, bit 1 tp
    MrTri mine{0, 0, 0};
#pragma unroll
    for (int k = 0; k < kMrScanItems; ++k) {
      code[k] = 0;
      const int j = j0 + k;
      if (j < present) {
        const int slot = P.val[j];
        const unsigned f = P.flags[slot];
        const int im = P.slot_img[slot];
        if ((f & kbit) && im >= lo && im < hi) code[k] = 1 | ((f & tbit) ? 2 : 0);
      }
      mine.kept += code[k] & 1;
      mine.tp += code[k] >> 1;
      mine.fp += (code[k] & 1) && !(code[k] >> 1);
    }
    MrTri run = mr_block_scan(mine, s_warp, &s_total) + s_carry;
#pragma unroll
    for (int k = 0; k < kMrScanItems; ++k) {
      if (!(code[k] & 1)) continue;
      const bool tp = code[k] >> 1;
      const int kb = run.kept, tb = run.tp;                     // before this detection
      run.kept += 1;
      run.tp += tp;
      run.fp += !tp;
      if (xx) {
        xx[kb] = __ddiv_rn((double)run.fp, dI0);
        yy[kb] = __dsub_rn(1.0, __ddiv_rn((double)run.tp, dnpig));
      }
      if (!tp)
        for (int r = 0; r < kMrThrs; ++r)
          if (run.fp == s_K[r] + 1) { s_kb[r] = kb; s_tb[r] = tb; }
    }
    __syncthreads();
    if (tid == 0) s_carry = s_carry + s_total;
    __syncthreads();
  }
  if (tid < kMrThrs) {
    const MrTri all = s_carry;
    double q = 0.0;
    if (all.kept > 0) {
      const bool found = s_kb[tid] >= 0;
      const int idx = (found ? s_kb[tid] : all.kept) - 1;
      q = __ddiv_rn((double)(idx < 0 || !found ? all.tp : s_tb[tid]), dnpig);
    }
    ys[tid] = q;
    if (tid == 0) { P.counts[3 * e] = all.kept; P.counts[3 * e + 1] = all.tp; P.counts[3 * e + 2] = npig; }
  }
}

// test.py's result line for one detection, `%g` of fp32 values read back by float(): 6 significant digits, as a double.
// k = 5 - floor(log10|v|), the decade found by exact comparisons; then rint(v * 10^k) / 10^k.  Exact for v == 0 and
// 1e-7 <= |v| < 1e6: there 0 <= k <= 12, a 24-bit significand times 10^k = 2^k 5^k (5^12 < 2^28) fits in 53 bits, rint
// rounds ties to even as printf does, and dividing by the exact power of ten is correctly rounded, as float() is.  That
// covers every score at conf_thres >= 1e-7 and every non-degenerate pixel coordinate; outside it the value is the nearest
// 6-digit decimal up to a rounding of the scaled product.
__constant__ double kPow10[23] = {1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8, 1e9, 1e10, 1e11, 1e12, 1e13, 1e14, 1e15, 1e16,
                                  1e17, 1e18, 1e19, 1e20, 1e21, 1e22};
__device__ __forceinline__ double round_g6(float v) {
  if (v == 0.f || !isfinite(v)) return (double)v;
  const double a = fabs((double)v);
  if (a >= 1e6 || a < 1e-7) {
    const int d = (int)floor(log10(a));
    const double p = pow(10.0, (double)abs(d - 5));
    return d >= 5 ? __dmul_rn(rint(__ddiv_rn((double)v, p)), p) : __ddiv_rn(rint(__dmul_rn((double)v, p)), p);
  }
  const double x = __dmul_rn(a, 1e12);                          // exact; 10^5 <= x < 10^18
  int e = 5;
  while (e < 17 && x >= kPow10[e + 1]) ++e;
  while (e > 5 && x < kPow10[e]) --e;
  const int k = 17 - e;                                         // 5 - (e - 12)
  return __ddiv_rn(rint(__dmul_rn((double)v, kPow10[k])), kPow10[k]);
}

// One thread per (image of the batch, detection): rows[(p * max_det + i) * 5 ..] = the rounded x1, y1, w, h, score of
// test.py's line (w = x2 - x1 in fp32, xyxy2xywh2), p = image[b]; span[p] = (p * max_det, count[b]).
__global__ void __launch_bounds__(256) kaist_round_kernel(const float* native, const float* det, const int* count,
                                                          const int* image, int B, int max_det, int images, double* rows,
                                                          int* span) {
  pdl_launch_dependents();
  pdl_wait();
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= B * max_det) return;
  const int b = t / max_det, i = t % max_det, p = image[b];
  if (p < 0 || p >= images) return;
  const int n = min(max(count[b], 0), max_det);
  if (i == 0) { span[2 * p] = p * max_det; span[2 * p + 1] = n; }
  if (i >= n) return;
  const float* nb = native + (size_t)t * 4;
  double* r = rows + ((size_t)p * max_det + i) * 5;
  r[0] = round_g6(nb[0]);
  r[1] = round_g6(nb[1]);
  r[2] = round_g6(__fsub_rn(nb[2], nb[0]));
  r[3] = round_g6(__fsub_rn(nb[3], nb[1]));
  r[4] = round_g6(det[(size_t)t * 6 + 4]);
}

// Workspace of icaf_kaist_mr, carved in this order (each piece 256-byte aligned).
struct MrLayout { size_t key_in, key_out, val_in, val_out, slot_img, flags, gt_state, npig, sort_tmp, sort_bytes, total; };
inline int mr_layout(int images, int gts, int nrows, MrLayout* L) {
  auto up = [](size_t x) { return (x + 255) & ~size_t(255); };
  const size_t n = (size_t)max(nrows, 1);
  size_t o = 0;
  L->key_in = o;  o += up(n * 8);
  L->key_out = o; o += up(n * 8);
  L->val_in = o;  o += up(n * 4);
  L->val_out = o; o += up(n * 4);
  L->slot_img = o; o += up(n * 4);
  L->flags = o;   o += up(n * 4);
  L->gt_state = o; o += up((size_t)kMrSetups * max(gts, 1));
  L->npig = o;    o += up((2 * kMrSetups + 1) * 4);
  L->sort_bytes = 0;
  cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, L->sort_bytes, (unsigned long long*)nullptr,
                                                  (unsigned long long*)nullptr, (int*)nullptr, (int*)nullptr, max(nrows, 1));
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    return set_cuda_error(e, "kaist_mr: sizing the radix sort's temporary storage");
  }
  L->sort_tmp = o; o += up(L->sort_bytes);
  L->total = o;
  (void)images;
  return ICAF_OK;
}

}  // namespace icaf

using namespace icaf;

extern "C" size_t icaf_match_detections_workspace_bytes(int T) {
  if (T < 0) return 0;
  return (size_t)T * sizeof(int);
}

extern "C" int icaf_match_detections(const float* det, const int* count, int B, int max_det, const float* targets, int T,
                                     const float* ratio_pad, int height, int width, const float* iouv, int niou, int single_cls,
                                     unsigned char* correct, float* native, void* workspace, size_t workspace_bytes,
                                     void* stream) {
  if (!det || !count || !ratio_pad || !iouv || !correct || (T > 0 && (!targets || !workspace)))
    return set_error(ICAF_ERR_BAD_ARG, "match_detections: null pointer");
  if (B < 1 || max_det < 1 || T < 0 || niou < 1 || niou > kMatchMaxIou || height < 1 || width < 1)
    return set_error(ICAF_ERR_BAD_ARG, "match_detections: bad shape (B, max_det >= 1, T >= 0, 1 <= niou <= 32, height, width >= 1)");
  if (workspace_bytes < icaf_match_detections_workspace_bytes(T) || (reinterpret_cast<uintptr_t>(workspace) & 3))
    return set_error(ICAF_ERR_BAD_ARG, "match_detections: workspace too small (icaf_match_detections_workspace_bytes) or not 4-byte aligned");
  if (native && (reinterpret_cast<uintptr_t>(native) & 15))
    return set_error(ICAF_ERR_BAD_ARG, "match_detections: native must be 16-byte aligned");
  MatchParams P;
  P.det = det; P.count = count; P.targets = targets; P.ratio_pad = ratio_pad; P.iouv = iouv;
  P.correct = correct; P.native = native; P.detected = (int*)workspace;
  P.B = B; P.max_det = max_det; P.T = T; P.niou = niou; P.single_cls = single_cls;
  P.height = float(height); P.width = float(width);
  return launch_k("match_detections", match_detections_kernel, dim3(B), dim3(kMatchThreads), 0, (cudaStream_t)stream, P);
}

extern "C" size_t icaf_kaist_mr_workspace_bytes(int images, int gts, int rows) {
  if (images < 1 || gts < 0 || rows < 0) return 0;
  MrLayout L;
  return mr_layout(images, gts, rows, &L) == ICAF_OK ? L.total : 0;
}

extern "C" int icaf_kaist_mr(const double* gt_box, const double* gt_height, const int* gt_occlusion, const int* gt_ignore,
                             const long long* gt_id, const int* gt_offset, int images, int gts, int day_images,
                             const double* dt_rows, const int* dt_span, int rows, int max_per_image, double* ys, int* counts,
                             double* curves, void* workspace, size_t workspace_bytes, void* stream) {
  if (!gt_offset || !dt_span || !ys || !counts || !workspace || (gts > 0 && (!gt_box || !gt_height || !gt_occlusion ||
      !gt_ignore || !gt_id)) || (rows > 0 && !dt_rows))
    return set_error(ICAF_ERR_BAD_ARG, "kaist_mr: null pointer");
  if (images < 1 || gts < 0 || rows < 0 || day_images < 0 || max_per_image < 0)
    return set_error(ICAF_ERR_BAD_ARG, "kaist_mr: bad shape (images >= 1; gts, rows, day_images, max_per_image >= 0)");
  if (max_per_image > kMrMaxDet)
    return set_error(ICAF_ERR_BAD_ARG, "kaist_mr: more than 1000 detections in one image (the reference's maxDets; its "
                                       "evaluateImg indexes past its IoU rows there)");
  if (reinterpret_cast<uintptr_t>(workspace) & 255)
    return set_error(ICAF_ERR_BAD_ARG, "kaist_mr: workspace must be 256-byte aligned");
  MrLayout L;
  if (int rc = mr_layout(images, gts, rows, &L)) return rc;
  if (workspace_bytes < L.total)
    return set_error(ICAF_ERR_BAD_ARG, "kaist_mr: workspace too small (icaf_kaist_mr_workspace_bytes)");
  char* w = (char*)workspace;
  MrParams P;
  P.gt_box = gt_box; P.gt_height = gt_height; P.gt_occ = gt_occlusion; P.gt_ignore = gt_ignore; P.gt_id = gt_id;
  P.gt_offset = gt_offset; P.rows = dt_rows; P.span = dt_span;
  P.images = images; P.gts = gts; P.day = day_images; P.nrows = rows; P.max_per_image = max_per_image;
  P.ys = ys; P.counts = counts; P.curves = curves;
  P.key = (unsigned long long*)(w + L.key_in); P.val = (int*)(w + L.val_in); P.slot_img = (int*)(w + L.slot_img);
  P.flags = (unsigned*)(w + L.flags); P.gt_state = (unsigned char*)(w + L.gt_state); P.npig = (int*)(w + L.npig);
  P.present = P.npig + 2 * kMrSetups;
  const cudaStream_t st = (cudaStream_t)stream;
  if (int rc = launch_k("kaist_mr_init", kaist_mr_init_kernel, dim3(blocks_for(max(rows, 2 * kMrSetups), 256)), dim3(256), 0,
                        st, P))
    return rc;
  if (int rc = launch_k("kaist_mr_match", kaist_mr_match_kernel, dim3(images), dim3(kMrMatchThreads), 0, st, P)) return rc;
  // after the sort, P.val holds the slots in ascending key order (stable: equal keys keep slot order)
  unsigned long long* key_out = (unsigned long long*)(w + L.key_out);
  int* val_out = (int*)(w + L.val_out);
  if (rows > 0) {
    size_t tmp = L.sort_bytes;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(w + L.sort_tmp, tmp, P.key, key_out, P.val, val_out, rows, 0, 64, st);
    if (e != cudaSuccess) return set_cuda_error(e, "kaist_mr: radix sort");
    P.val = val_out;
  }
  return launch_k("kaist_mr_accumulate", kaist_mr_accumulate_kernel, dim3(kMrEvals), dim3(kMrScanThreads), 0, st, P);
}

extern "C" int icaf_kaist_round_detections(const float* native, const float* det, const int* count, const int* image, int B,
                                           int max_det, int images, double* rows, int* span, void* stream) {
  if (!native || !det || !count || !image || !rows || !span)
    return set_error(ICAF_ERR_BAD_ARG, "kaist_round_detections: null pointer");
  if (B < 1 || max_det < 1 || images < 1 || (long long)images * max_det > 0x7fffffffLL)
    return set_error(ICAF_ERR_BAD_ARG, "kaist_round_detections: bad shape (B, max_det, images >= 1; images * max_det < 2^31)");
  return launch_k("kaist_round_detections", kaist_round_kernel, dim3(blocks_for((long long)B * max_det, 256)), dim3(256), 0,
                  (cudaStream_t)stream, native, det, count, image, B, max_det, images, rows, span);
}
