// Validation metrics: per-image matching of the NMS detections to the labels (test.py:196-227), one launch per batch.
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
