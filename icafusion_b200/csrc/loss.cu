// Detection loss, forward (utils/loss.py:325-463 ComputeLoss.__call__ + build_targets): target assignment, CIoU box loss,
// objectness BCE against IoU-valued targets, class BCE -- three launches, no host round trip -- and its backward in two.
// Deterministic, forward and backward: no floating point atomics.  Objectness targets meet in an integer atomicMax; every
// sum is reduced in a fixed order, including the backward's sum over the candidates that meet in one cell (ascending
// candidate index, see loss_obj_bwd_kernel).
// Both BCE terms are optionally wrapped in the focal loss of utils/loss.py:37-64 (hyp fl_gamma > 0, loss.py:341-344): the
// candidate and objectness kernels, forward and backward, take it as a template argument, so the plain BCE path compiles to
// the code it has without it.
//   1. loss_candidates_kernel: one thread per (level, target, anchor, offset) candidate of build_targets (:405-463):
//      anchor-ratio match, the four half-cell neighbour offsets, grid cell, CIoU of the decoded prediction against the
//      target box (general.py:410-447), its (1 - iou) and class-BCE terms, objectness target into tobj by atomicMax
//      (the reference sorts by IoU before its scatter so that the largest IoU wins a contested cell, :374-377).
//   2. loss_obj_kernel: BCEWithLogits(p[..., 4], tobj) with pos_weight, per-block partial sums over fixed chunks.
//   3. loss_finalize_kernel: means, level balance, gains -> (loss * batch, lbox, lobj, lcls, 0).
#include <cmath>
#include <cstring>

#include "icaf_internal.cuh"

namespace icaf {

constexpr int kLossMaxLevels = 5;
constexpr int kLossObjBlocks = 256;     // partial sums per level

struct LossParams {
  const void* p[kLossMaxLevels];
  int ny[kLossMaxLevels], nx[kLossMaxLevels];
  long long cell_off[kLossMaxLevels];   // offset of the level's tobj slab (floats)
  float anchors[kLossMaxLevels * 8 * 2];
  float balance[kLossMaxLevels];
  int p_fp32, nl, B, na, no, nt;
  float box, obj, cls, cls_pw, obj_pw, anchor_t, gr, cp, cn;
  int nhwc;                             // 0: p is (B, na, ny, nx, no) contiguous; > 0: pixel pitch of the head's own (B, ny, nx, na*no) map
  const float* targets;                 // (nt, 6): image, class, x, y, w, h (normalised)
  int* cand_count;                      // [nl] matched candidates per level (written by finalize, read by the backward)
  const float* gout;                    // backward: d / d(out[0]) (device scalar)
  int* cell_head;                       // backward: per cell of all levels, first candidate of its list (-1: none)
  int* cand_next;                       // backward: [nl][nt][na][5] next candidate in the same cell's list (-1: end)
  float* cand_grad;                     // backward: [nl][nt][na][5][no] each candidate's box and class gradient
  void* dp[kLossMaxLevels];             // backward: fp16 / fp32 gradient of p, same memory layout as p
  float* tobj;                          // all levels, (B, na, ny, nx) each
  float* cand_box; float* cand_cls; int* cand_valid;     // [nl][nt][na][5]
  float* obj_part;                      // [nl][kLossObjBlocks]
  float* out;                           // 5 floats
  float fl_gamma;                       // focal-loss gamma (only read by the kFocal instantiations)
};

__device__ __forceinline__ float loss_ld(const void* p, int fp32, long long i) {
  return fp32 ? reinterpret_cast<const float*>(p)[i] : __half2float(reinterpret_cast<const __half*>(p)[i]);
}
__device__ __forceinline__ float sigmoid_f(float v) { return 1.f / (1.f + expf(-v)); }
// BCEWithLogitsLoss element with pos_weight (torch semantics): (1 - y) x + (1 + (pw - 1) y) (log(1 + exp(-|x|)) + max(-x, 0))
__device__ __forceinline__ float bce_logits(float x, float y, float pw) {
  const float lw = 1.f + (pw - 1.f) * y;
  return (1.f - y) * x + lw * (log1pf(expf(-fabsf(x))) + fmaxf(-x, 0.f));
}

// FocalLoss(BCEWithLogitsLoss, gamma, alpha = 0.25), utils/loss.py:37-64, per element:
//   bce(x, y) * (y a + (1 - y)(1 - a)) * (1 - p_t)^gamma,   p_t = y sigmoid(x) + (1 - y)(1 - sigmoid(x)).
constexpr float kFocalAlpha = 0.25f;
template <bool kFocal>
__device__ __forceinline__ float bce_elem(float x, float y, float pw, float gamma) {
  float l = bce_logits(x, y, pw);
  if constexpr (kFocal) {
    const float s = sigmoid_f(x);
    const float pt = y * s + (1.f - y) * (1.f - s);
    l *= (y * kFocalAlpha + (1.f - y) * (1.f - kFocalAlpha)) * powf(1.f - pt, gamma);
  }
  return l;
}
// d bce_elem / dx.  Plain: (1 - y) - (1 + (pw - 1) y)(1 - sigmoid(x)).  Focal: the product rule over the three factors, with
// d(1 - p_t)/dx = (1 - 2y) s (1 - s) -- the derivative autograd takes through the reference's FocalLoss.forward.
template <bool kFocal>
__device__ __forceinline__ float bce_elem_grad(float x, float y, float pw, float gamma) {
  const float lw = 1.f + (pw - 1.f) * y;
  if constexpr (!kFocal) {
    return (1.f - y) - lw * (1.f - sigmoid_f(x));
  } else {
    const float s = sigmoid_f(x);
    const float q = 1.f - (y * s + (1.f - y) * (1.f - s));
    const float af = y * kFocalAlpha + (1.f - y) * (1.f - kFocalAlpha);
    const float dbce = (1.f - y) - lw * (1.f - s);
    const float dq = (1.f - 2.f * y) * s * (1.f - s);
    return af * (dbce * powf(q, gamma) + bce_logits(x, y, pw) * gamma * powf(q, gamma - 1.f) * dq);
  }
}

// Forward-mode value with the four partial derivatives w.r.t. the raw box logits: the backward pass evaluates the very same
// CIoU expression as the forward pass (ciou_t below), on this type instead of float.
struct Dual4 { float v; float d[4]; };
__device__ __forceinline__ Dual4 mk(float v) { Dual4 r; r.v = v; r.d[0] = r.d[1] = r.d[2] = r.d[3] = 0.f; return r; }
#define ICAF_D4(expr_v, expr_d) Dual4 r; r.v = (expr_v); _Pragma("unroll") for (int i = 0; i < 4; ++i) r.d[i] = (expr_d); return r;
__device__ __forceinline__ Dual4 operator+(const Dual4& a, const Dual4& b) { ICAF_D4(a.v + b.v, a.d[i] + b.d[i]) }
__device__ __forceinline__ Dual4 operator-(const Dual4& a, const Dual4& b) { ICAF_D4(a.v - b.v, a.d[i] - b.d[i]) }
__device__ __forceinline__ Dual4 operator*(const Dual4& a, const Dual4& b) { ICAF_D4(a.v * b.v, a.d[i] * b.v + a.v * b.d[i]) }
__device__ __forceinline__ Dual4 operator/(const Dual4& a, const Dual4& b) { const float q = a.v / b.v; ICAF_D4(q, (a.d[i] - q * b.d[i]) / b.v) }
__device__ __forceinline__ Dual4 operator+(const Dual4& a, float b) { ICAF_D4(a.v + b, a.d[i]) }
__device__ __forceinline__ Dual4 operator-(const Dual4& a, float b) { ICAF_D4(a.v - b, a.d[i]) }
__device__ __forceinline__ Dual4 operator-(float a, const Dual4& b) { ICAF_D4(a - b.v, -b.d[i]) }
__device__ __forceinline__ Dual4 operator*(const Dual4& a, float b) { ICAF_D4(a.v * b, a.d[i] * b) }
__device__ __forceinline__ Dual4 operator/(const Dual4& a, float b) { ICAF_D4(a.v / b, a.d[i] / b) }
__device__ __forceinline__ Dual4 tmax(const Dual4& a, const Dual4& b) { return a.v >= b.v ? a : b; }
__device__ __forceinline__ Dual4 tmin(const Dual4& a, const Dual4& b) { return a.v <= b.v ? a : b; }
__device__ __forceinline__ Dual4 tmax(const Dual4& a, float b) { return a.v > b ? a : mk(b); }     // clamp(0): zero gradient at and below the bound
__device__ __forceinline__ Dual4 tmin(const Dual4& a, float b) { return a.v <= b ? a : mk(b); }
__device__ __forceinline__ Dual4 tmax(float a, const Dual4& b) { return tmax(b, a); }
__device__ __forceinline__ Dual4 tatan(const Dual4& a) { const float k = 1.f / (1.f + a.v * a.v); ICAF_D4(atanf(a.v), a.d[i] * k) }
__device__ __forceinline__ float val(const Dual4& a) { return a.v; }
__device__ __forceinline__ float tmax(float a, float b) { return fmaxf(a, b); }
__device__ __forceinline__ float tmin(float a, float b) { return fminf(a, b); }
__device__ __forceinline__ float tatan(float a) { return atanf(a); }
__device__ __forceinline__ float val(float a) { return a; }

// CIoU of the decoded prediction (px, py, pw, ph) against the target box (tx, ty, gw, gh): general.py:418-447 (xywh form,
// eps = 1e-7).  alpha is a constant of the graph (torch.no_grad, general.py:444-445).
template <typename T>
__device__ __forceinline__ T ciou_t(const T& px, const T& py, const T& pw, const T& ph, float tx, float ty, float gw, float gh) {
  const float eps = 1e-7f;
  const T b1x1 = px - pw / 2.f, b1x2 = px + pw / 2.f, b1y1 = py - ph / 2.f, b1y2 = py + ph / 2.f;
  const float b2x1 = tx - gw / 2, b2x2 = tx + gw / 2, b2y1 = ty - gh / 2, b2y2 = ty + gh / 2;
  const T inter = tmax(tmin(b1x2, b2x2) - tmax(b1x1, b2x1), 0.f) * tmax(tmin(b1y2, b2y2) - tmax(b1y1, b2y1), 0.f);
  const T w1 = b1x2 - b1x1, h1 = b1y2 - b1y1 + eps;
  const float w2 = b2x2 - b2x1, h2 = b2y2 - b2y1 + eps;
  const T uni = w1 * h1 + (w2 * h2) - inter + eps;
  const T iou = inter / uni;
  const T cw = tmax(b1x2, b2x2) - tmin(b1x1, b2x1), ch = tmax(b1y2, b2y2) - tmin(b1y1, b2y1);
  const T c2 = cw * cw + ch * ch + eps;
  const T dx = (b2x1 + b2x2) - b1x1 - b1x2, dy = (b2y1 + b2y2) - b1y1 - b1y2;
  const T rho2 = (dx * dx + dy * dy) / 4.f;
  const T da = atanf(w2 / h2) - tatan(w1 / h1);
  const T v = da * da * (4.f / (3.14159265358979323846f * 3.14159265358979323846f));
  const float alpha = val(v) / (val(v) - val(iou) + (1.f + eps));
  return iou - (rho2 / c2 + v * alpha);
}

// One (level, target, anchor, offset) candidate of build_targets (loss.py:405-463).
struct Cand {
  int lvl, a, c, gi, gj;
  long long cell;        // index in (B, na, ny, nx) order (tobj, cell_head)
  long long pb;          // element offset of the cell's `no` values in p / dp
  float tx, ty, gw, gh, aw, ah;
};
__device__ __forceinline__ long long cell_offset(const LossParams& P, int lvl, int b, int a, int gj, int gi) {
  const int ny = P.ny[lvl], nx = P.nx[lvl];
  return P.nhwc ? (((long long)b * ny + gj) * nx + gi) * P.nhwc + a * P.no : ((((long long)b * P.na + a) * ny + gj) * nx + gi) * P.no;
}
__device__ __forceinline__ bool cand_setup(const LossParams& P, long long idx, Cand& K) {
  const long long per_level = (long long)P.nt * P.na * 5;
  const int lvl = int(idx / per_level);
  long long r = idx - lvl * per_level;
  const int t = int(r / (P.na * 5));
  r -= (long long)t * P.na * 5;
  const int a = int(r / 5), k = int(r - a * 5);
  const float* tg = P.targets + (long long)t * 6;
  const int nx = P.nx[lvl], ny = P.ny[lvl];
  const float gx = tg[2] * nx, gy = tg[3] * ny, gw = tg[4] * nx, gh = tg[5] * ny;     // :425-426 targets * gain
  const float aw = P.anchors[(lvl * P.na + a) * 2], ah = P.anchors[(lvl * P.na + a) * 2 + 1];
  const float rw = gw / aw, rh = gh / ah;                                           // :429-430 anchor-multiple match
  if (!(fmaxf(fmaxf(rw, 1.f / rw), fmaxf(rh, 1.f / rh)) < P.anchor_t)) return false;
  float ox = 0.f, oy = 0.f;                                                         // :434-441 neighbour cells
  const float g = 0.5f;
  if (k == 1) { if (!(fmodf(gx, 1.f) < g && gx > 1.f)) return false; ox = g; }
  else if (k == 2) { if (!(fmodf(gy, 1.f) < g && gy > 1.f)) return false; oy = g; }
  else if (k == 3) { const float ix = nx - gx; if (!(fmodf(ix, 1.f) < g && ix > 1.f)) return false; ox = -g; }
  else if (k == 4) { const float iy = ny - gy; if (!(fmodf(iy, 1.f) < g && iy > 1.f)) return false; oy = -g; }
  const int b = int(tg[0]);
  int gi = int(gx - ox), gj = int(gy - oy);                                         // .long() truncates
  gi = min(max(gi, 0), nx - 1); gj = min(max(gj, 0), ny - 1);                       // :455 clamp_ (in place: tbox sees it too)
  if (b < 0 || b >= P.B) return false;
  K.lvl = lvl; K.a = a; K.c = int(tg[1]); K.gi = gi; K.gj = gj;
  K.tx = gx - gi; K.ty = gy - gj; K.gw = gw; K.gh = gh; K.aw = aw; K.ah = ah;       // :456 target box in cell units
  K.cell = (((long long)b * P.na + a) * ny + gj) * nx + gi;
  K.pb = cell_offset(P, lvl, b, a, gj, gi);
  return true;
}

template <bool kFocal>
__global__ void loss_candidates_kernel(const LossParams P) {
  pdl_launch_dependents();
  pdl_wait();
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long per_level = (long long)P.nt * P.na * 5;
  if (idx >= per_level * P.nl) return;
  P.cand_valid[idx] = 0;
  Cand K;
  if (!cand_setup(P, idx, K)) return;
  // prediction at (b, a, gj, gi)                                                     :355-360
  const long long pb = K.pb;
  const void* pl = P.p[K.lvl];
  const float sx = sigmoid_f(loss_ld(pl, P.p_fp32, pb)), sy = sigmoid_f(loss_ld(pl, P.p_fp32, pb + 1));
  const float sw = sigmoid_f(loss_ld(pl, P.p_fp32, pb + 2)), sh = sigmoid_f(loss_ld(pl, P.p_fp32, pb + 3));
  const float px = sx * 2.f - 0.5f, py = sy * 2.f - 0.5f;
  const float pw = (sw * 2.f) * (sw * 2.f) * K.aw, ph = (sh * 2.f) * (sh * 2.f) * K.ah;
  const float ciou = ciou_t<float>(px, py, pw, ph, K.tx, K.ty, K.gw, K.gh);
  P.cand_box[idx] = 1.f - ciou;                                                     // :361
  float lc = 0.f;
  if (P.no - 5 > 1) {                                                               // :380-383
    for (int j = 0; j < P.no - 5; ++j)
      lc += bce_elem<kFocal>(loss_ld(pl, P.p_fp32, pb + 5 + j), (j == K.c) ? P.cp : P.cn, P.cls_pw, P.fl_gamma);
  }
  P.cand_cls[idx] = lc;
  P.cand_valid[idx] = 1;
  const float score = (1.f - P.gr) + P.gr * fmaxf(ciou, 0.f);                       // :364-377 (largest IoU wins a cell)
  atomicMax(reinterpret_cast<int*>(P.tobj + P.cell_off[K.lvl] + K.cell), __float_as_int(score));
}

// Backward, 1 of 2: box and class gradients of every matched candidate, written to the candidate's own row of cand_grad,
// and the candidate pushed onto its cell's list (several candidates can meet in one cell).  The integer atomicExch leaves
// the list in the order the pushes land; loss_obj_bwd_kernel sorts it before it sums.
template <bool kFocal>
__global__ void loss_candidates_bwd_kernel(const LossParams P) {
  pdl_launch_dependents();
  pdl_wait();
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long per_level = (long long)P.nt * P.na * 5;
  if (idx >= per_level * P.nl || !P.cand_valid[idx]) return;
  Cand K;
  if (!cand_setup(P, idx, K)) return;
  const int n = P.cand_count[K.lvl];
  if (n <= 0) return;
  const float g = P.gout[0] * float(P.B);                                           // out[0] = loss * bs
  const void* pl = P.p[K.lvl];
  float s[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) s[i] = sigmoid_f(loss_ld(pl, P.p_fp32, K.pb + i));
  Dual4 px = mk(s[0] * 2.f - 0.5f), py = mk(s[1] * 2.f - 0.5f), pw = mk((s[2] * 2.f) * (s[2] * 2.f) * K.aw), ph = mk((s[3] * 2.f) * (s[3] * 2.f) * K.ah);
  px.d[0] = 2.f * s[0] * (1.f - s[0]); py.d[1] = 2.f * s[1] * (1.f - s[1]);
  pw.d[2] = 8.f * s[2] * K.aw * s[2] * (1.f - s[2]); ph.d[3] = 8.f * s[3] * K.ah * s[3] * (1.f - s[3]);
  const Dual4 ciou = ciou_t<Dual4>(px, py, pw, ph, K.tx, K.ty, K.gw, K.gh);
  float* row = P.cand_grad + idx * P.no;
  const float kb = -g * P.box / float(n);                                           // d(1 - ciou).mean()
#pragma unroll
  for (int i = 0; i < 4; ++i) row[i] = kb * ciou.d[i];
  if (P.no - 5 > 1) {
    const float kc = g * P.cls / (float(n) * float(P.no - 5));
    for (int j = 0; j < P.no - 5; ++j) {
      const float x = loss_ld(pl, P.p_fp32, K.pb + 5 + j), y = (j == K.c) ? P.cp : P.cn;
      row[5 + j] = kc * bce_elem_grad<kFocal>(x, y, P.cls_pw, P.fl_gamma);
    }
  }
  P.cand_next[idx] = atomicExch(P.cell_head + P.cell_off[K.lvl] + K.cell, int(idx));
}

// Backward, 2 of 2: objectness gradient of every cell, plus the gradients of the candidates in the cell, written as dp.  The
// one thread that owns a cell first relinks the cell's list by ascending candidate index (insertion sort: a list holds the
// few candidates that meet in one cell), then sums each channel over the list in that order from 0 -- the same sum
// whatever order the pushes landed in.
template <bool kFocal>
__global__ void __launch_bounds__(256) loss_obj_bwd_kernel(const LossParams P) {
  pdl_launch_dependents();
  pdl_wait();
  const int lvl = blockIdx.y;
  const int ny = P.ny[lvl], nx = P.nx[lvl];
  const long long cells = (long long)P.B * P.na * ny * nx;
  const float g = P.gout[0] * float(P.B) * P.obj * P.balance[lvl] / float(cells);
  for (long long c = blockIdx.x * 256ll + threadIdx.x; c < cells; c += 256ll * gridDim.x) {
    const int gi = int(c % nx);
    long long t = c / nx;
    const int gj = int(t % ny); t /= ny;
    const int a = int(t % P.na), b = int(t / P.na);
    const long long pb = cell_offset(P, lvl, b, a, gj, gi);
    int head = -1;
    for (int i = P.cell_head[P.cell_off[lvl] + c]; i >= 0;) {
      const int nxt = P.cand_next[i];
      if (head < 0 || i < head) {
        P.cand_next[i] = head; head = i;
      } else {
        int q = head;
        while (P.cand_next[q] >= 0 && P.cand_next[q] < i) q = P.cand_next[q];
        P.cand_next[i] = P.cand_next[q]; P.cand_next[q] = i;
      }
      i = nxt;
    }
    const float x = loss_ld(P.p[lvl], P.p_fp32, pb + 4), y = P.tobj[P.cell_off[lvl] + c];
    for (int j = 0; j < P.no; ++j) {
      float v = 0.f;
      if (j == 4) v += g * bce_elem_grad<kFocal>(x, y, P.obj_pw, P.fl_gamma);
      else if (j < 4 || P.no - 5 > 1)
        for (int i = head; i >= 0; i = P.cand_next[i]) v += P.cand_grad[(long long)i * P.no + j];
      if (P.p_fp32) reinterpret_cast<float*>(P.dp[lvl])[pb + j] = v;
      else reinterpret_cast<__half*>(P.dp[lvl])[pb + j] = __float2half(v);
    }
  }
}

template <bool kFocal>
__global__ void __launch_bounds__(256) loss_obj_kernel(const LossParams P) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[256];
  const int lvl = blockIdx.y;
  const long long cells = (long long)P.B * P.na * P.ny[lvl] * P.nx[lvl];
  const long long per = (cells + kLossObjBlocks - 1) / kLossObjBlocks;
  const long long c0 = blockIdx.x * per, c1 = min(c0 + per, cells);
  const float* tobj = P.tobj + P.cell_off[lvl];
  float s = 0.f;
  const int ny = P.ny[lvl], nx = P.nx[lvl];
  for (long long c = c0 + threadIdx.x; c < c1; c += 256) {
    long long pb = c * P.no;
    if (P.nhwc) {
      const int gi = int(c % nx);
      long long t = c / nx;
      const int gj = int(t % ny); t /= ny;
      pb = cell_offset(P, lvl, int(t / P.na), int(t % P.na), gj, gi);
    }
    s += bce_elem<kFocal>(loss_ld(P.p[lvl], P.p_fp32, pb + 4), tobj[c], P.obj_pw, P.fl_gamma);
  }
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) P.obj_part[lvl * kLossObjBlocks + blockIdx.x] = red[0];
}

__global__ void __launch_bounds__(256) loss_finalize_kernel(const LossParams P) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float rb[256], rc[256];
  __shared__ int rn[256];
  float lbox = 0.f, lobj = 0.f, lcls = 0.f;
  const long long per_level = (long long)P.nt * P.na * 5;
  for (int lvl = 0; lvl < P.nl; ++lvl) {
    float sb = 0.f, sc = 0.f;
    int n = 0;
    for (long long i = threadIdx.x; i < per_level; i += 256) {
      const long long j = lvl * per_level + i;
      if (P.cand_valid[j]) { sb += P.cand_box[j]; sc += P.cand_cls[j]; ++n; }
    }
    rb[threadIdx.x] = sb; rc[threadIdx.x] = sc; rn[threadIdx.x] = n;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
      if (threadIdx.x < o) { rb[threadIdx.x] += rb[threadIdx.x + o]; rc[threadIdx.x] += rc[threadIdx.x + o]; rn[threadIdx.x] += rn[threadIdx.x + o]; }
      __syncthreads();
    }
    float so = 0.f;
    if (threadIdx.x == 0) {
      for (int i = 0; i < kLossObjBlocks; ++i) so += P.obj_part[lvl * kLossObjBlocks + i];
      const long long cells = (long long)P.B * P.na * P.ny[lvl] * P.nx[lvl];
      P.cand_count[lvl] = rn[0];
      if (rn[0] > 0) {
        lbox += rb[0] / float(rn[0]);                                              // (1 - iou).mean()
        if (P.no - 5 > 1) lcls += rc[0] / (float(rn[0]) * float(P.no - 5));        // BCEcls mean over n x nc
      }
      lobj += (so / float(cells)) * P.balance[lvl];                                // :389-390
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    lbox *= P.box; lobj *= P.obj; lcls *= P.cls;                                    // :396-398
    P.out[0] = (lbox + lobj + lcls) * float(P.B);                                   // loss * bs
    P.out[1] = lbox; P.out[2] = lobj; P.out[3] = lcls; P.out[4] = 0.f;              // lrk (ranking loss) is disabled upstream (:386)
  }
}

static size_t align256(size_t v) { return (v + 255) & ~size_t(255); }

}  // namespace icaf

using namespace icaf;

extern "C" size_t icaf_loss_workspace_bytes(int B, int na, int nt, const int* ny, const int* nx, int nl, int no_bwd) {
  if (B < 1 || na < 1 || nt < 0 || nl < 1 || nl > kLossMaxLevels || !ny || !nx || no_bwd < 0) return 0;
  size_t cells = 0;
  for (int i = 0; i < nl; ++i) cells += (size_t)B * na * ny[i] * nx[i];
  const size_t cand = (size_t)nl * (nt > 0 ? nt : 1) * na * 5;
  const size_t fwd = align256(cells * 4) + 3 * align256(cand * 4) + align256((size_t)nl * kLossObjBlocks * 4) + align256(kLossMaxLevels * 4);
  return no_bwd ? fwd + align256(cells * 4) + align256(cand * 4) + align256(cand * no_bwd * 4) : fwd;
}

// Argument checks and workspace partition shared by the forward and the backward entry.
static int loss_setup(const char* what, const void* const* p, int p_fp32, int p_ld, const int* ny, const int* nx, int nl, int B, int na, int no,
                      const float* targets, int nt, const float* anchors_host, const icaf_loss_hyp* hyp, void* workspace, size_t workspace_bytes,
                      bool bwd, LossParams& P, size_t& cells, size_t& cand) {
  if (!p || !ny || !nx || !anchors_host || !hyp || !workspace) return set_error(ICAF_ERR_BAD_ARG, "compute_loss: null pointer");
  if (nl < 1 || nl > kLossMaxLevels || B < 1 || na < 1 || na > 8 || no < 6 || nt < 0 || (nt > 0 && !targets))
    return set_error(ICAF_ERR_BAD_ARG, "compute_loss: bad shape (nl <= 5, na <= 8)");
  if (bwd && (long long)nl * nt * na * 5 > 0x7fffffffLL)
    return set_error(ICAF_ERR_BAD_ARG, "compute_loss_bwd: more than 2^31 - 1 candidates (nl * nt * na * 5)");
  if (p_ld != 0 && p_ld < na * no) return set_error(ICAF_ERR_BAD_ARG, "compute_loss: p_ld is 0 ((B,na,ny,nx,no) contiguous) or the pixel pitch of the (B,ny,nx,na*no) head map");
  if (workspace_bytes < icaf_loss_workspace_bytes(B, na, nt, ny, nx, nl, bwd ? no : 0) || (reinterpret_cast<uintptr_t>(workspace) & 255))
    return set_error(ICAF_ERR_BAD_ARG, "compute_loss: workspace too small (icaf_loss_workspace_bytes) or not 256-byte aligned");
  (void)what;
  memset(&P, 0, sizeof(P));
  cells = 0;
  for (int i = 0; i < nl; ++i) {
    if (!p[i] || ny[i] < 1 || nx[i] < 1) return set_error(ICAF_ERR_BAD_ARG, "compute_loss: bad level");
    P.p[i] = p[i]; P.ny[i] = ny[i]; P.nx[i] = nx[i]; P.cell_off[i] = (long long)cells;
    cells += (size_t)B * na * ny[i] * nx[i];
    P.balance[i] = hyp->balance[i];
  }
  for (int i = 0; i < nl * na * 2; ++i) P.anchors[i] = anchors_host[i];
  P.p_fp32 = p_fp32; P.nhwc = p_ld; P.nl = nl; P.B = B; P.na = na; P.no = no; P.nt = nt;
  P.box = hyp->box; P.obj = hyp->obj; P.cls = hyp->cls; P.cls_pw = hyp->cls_pw; P.obj_pw = hyp->obj_pw;
  P.anchor_t = hyp->anchor_t; P.gr = hyp->gr; P.cp = hyp->cp; P.cn = hyp->cn;
  P.fl_gamma = hyp->fl_gamma;                                                        // <= 0: plain BCE (loss.py:342 `if g > 0`)
  P.targets = targets;
  cand = (size_t)nl * (nt > 0 ? nt : 1) * na * 5;
  char* w = (char*)workspace;
  P.tobj = (float*)w; w += align256(cells * 4);
  P.cand_box = (float*)w; w += align256(cand * 4);
  P.cand_cls = (float*)w; w += align256(cand * 4);
  P.cand_valid = (int*)w; w += align256(cand * 4);
  P.obj_part = (float*)w; w += align256((size_t)nl * kLossObjBlocks * 4);
  P.cand_count = (int*)w; w += align256(kLossMaxLevels * 4);
  if (bwd) {
    P.cell_head = (int*)w; w += align256(cells * 4);
    P.cand_next = (int*)w; w += align256(cand * 4);
    P.cand_grad = (float*)w;
  }
  return ICAF_OK;
}

extern "C" int icaf_compute_loss_fwd(const void* const* p, int p_fp32, int p_ld, const int* ny, const int* nx, int nl, int B, int na, int no,
                                     const float* targets, int nt, const float* anchors_host, const icaf_loss_hyp* hyp, float* out,
                                     void* workspace, size_t workspace_bytes, void* stream) {
  if (!out) return set_error(ICAF_ERR_BAD_ARG, "compute_loss: null pointer");
  LossParams P;
  size_t cells, cand;
  if (int rc = loss_setup("compute_loss", p, p_fp32, p_ld, ny, nx, nl, B, na, no, targets, nt, anchors_host, hyp, workspace, workspace_bytes, false, P, cells, cand))
    return rc;
  P.out = out;
  const bool focal = P.fl_gamma > 0.f;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(P.tobj, 0, cells * 4, st);                        // tobj = zeros_like(pi[..., 0])   :351
  if (e == cudaSuccess) e = cudaMemsetAsync(P.cand_valid, 0, cand * 4, st);
  if (e != cudaSuccess) return set_cuda_error(e, "compute_loss: cudaMemsetAsync");
  if (nt > 0) {
    const long long total = (long long)nl * nt * na * 5;
    if (int rc = launch_k("compute_loss(candidates)", focal ? loss_candidates_kernel<true> : loss_candidates_kernel<false>,
                          dim3(blocks_for(total, 128)), dim3(128), 0, st, P)) return rc;
  }
  if (int rc = launch_k("compute_loss(objectness)", focal ? loss_obj_kernel<true> : loss_obj_kernel<false>, dim3(kLossObjBlocks, nl),
                        dim3(256), 0, st, P)) return rc;
  return launch_k("compute_loss(finalize)", loss_finalize_kernel, dim3(1), dim3(256), 0, st, P);
}

extern "C" int icaf_compute_loss_bwd(const void* const* p, int p_fp32, int p_ld, const int* ny, const int* nx, int nl, int B, int na, int no,
                                     const float* targets, int nt, const float* anchors_host, const icaf_loss_hyp* hyp, const float* grad_out,
                                     void* const* dp, void* workspace, size_t workspace_bytes, void* stream) {
  if (!grad_out || !dp) return set_error(ICAF_ERR_BAD_ARG, "compute_loss_bwd: null pointer");
  LossParams P;
  size_t cells, cand;
  if (int rc = loss_setup("compute_loss_bwd", p, p_fp32, p_ld, ny, nx, nl, B, na, no, targets, nt, anchors_host, hyp, workspace, workspace_bytes, true, P, cells, cand))
    return rc;
  for (int i = 0; i < nl; ++i) {
    if (!dp[i]) return set_error(ICAF_ERR_BAD_ARG, "compute_loss_bwd: null gradient pointer");
    P.dp[i] = dp[i];
  }
  P.gout = grad_out;
  const bool focal = P.fl_gamma > 0.f;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(P.cell_head, 0xff, cells * 4, st);                // every cell's list empty (-1)
  if (e != cudaSuccess) return set_cuda_error(e, "compute_loss_bwd: cudaMemsetAsync");
  if (nt > 0) {
    const long long total = (long long)nl * nt * na * 5;
    if (int rc = launch_k("compute_loss_bwd(candidates)", focal ? loss_candidates_bwd_kernel<true> : loss_candidates_bwd_kernel<false>,
                          dim3(blocks_for(total, 128)), dim3(128), 0, st, P)) return rc;
  }
  return launch_k("compute_loss_bwd(objectness)", focal ? loss_obj_bwd_kernel<true> : loss_obj_bwd_kernel<false>,
                  dim3(kLossObjBlocks, nl), dim3(256), 0, st, P);
}
