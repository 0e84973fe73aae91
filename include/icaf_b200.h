/*
 * icaf_b200 -- C ABI of the H100 (sm_90a) kernels for the ICAFusion hot path:
 * the two-stream CSPDarknet Conv+BN+SiLU backbone and the DMFF cross-attention fusion block.
 *
 * The reference (chanchanchan97/ICAFusion) is pure Python/PyTorch and has no FFI of its own; these
 * entry points are what a binding for its operator library (models/common.py) calls instead of the
 * PyTorch ops cited at each function.  INTEGRATION.md shows the ctypes stub.
 *
 * Conventions
 *   - Plain C types only.  Every pointer is a DEVICE pointer unless stated otherwise.
 *   - Activations are fp16 NHWC "views": a base pointer plus a pixel pitch `ld` in elements, so a
 *     kernel can read or write a channel slice of a wider (concatenated) buffer in place.
 *     (A torch tensor of logical shape (B,C,H,W) in channels_last memory format is exactly this.)
 *   - Token tensors are fp16 (B, Npad, C) with Npad = N rounded up to 8.
 *   - The caller owns all memory (inputs, outputs, workspaces); the library never allocates device
 *     memory, never synchronises, and enqueues all work on the `stream` argument (a cudaStream_t),
 *     so it composes with the PyTorch caching allocator, autograd hooks and CUDA-graph capture.
 *   - Return value: ICAF_OK or an error code; icaf_last_error() gives a thread-local message.
 */
#ifndef ICAF_B200_H
#define ICAF_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ICAF_OK 0
#define ICAF_ERR_BAD_ARG 1
#define ICAF_ERR_UNSUPPORTED 2
#define ICAF_ERR_CUDA 3

#define ICAF_ACT_NONE 0
#define ICAF_ACT_SILU 1 /* nn.SiLU, models/common.py:54 */
#define ICAF_ACT_GELU 2 /* nn.GELU (erf), models/common.py:706 */

#define ICAF_EPI_BIAS_ROW 1   /* bias indexed by output row (swap-AB linears) instead of channel   */
#define ICAF_EPI_ADD_RES 2    /* y = act(acc+bias) + res          (Bottleneck shortcut, common.py:194) */
#define ICAF_EPI_SCALED_RES 4 /* y = alpha*res + beta*(acc+bias)  (LearnableCoefficient pairs, common.py:747-750) */
/* LayerNorm folded into the linear layer that consumes it (common.py:660-668, 749-750 + 704-706): the caller packs
 * W' = W diag(gamma), bias' = bias + W beta, ln_colsum[n] = sum_k W'[n][k]; the kernel runs the GEMM on the RAW rows and
 * normalises in the epilogue, y = act( rstd_m * (acc - mean_m * ln_colsum[n]) + bias'[n] ), with (mean, rstd) of input row m
 * from `ln_stats`: ln_parts (sum, sum of squares) fp32 pairs per row, as an EMIT_STATS producer or icaf_row_stats wrote
 * them.  1x1 geometry only, no residual, activation none or GELU. */
#define ICAF_EPI_LN_FOLD 8
/* With SCALED_RES: also write, per output row, (sum, sum of squares) partials of the fp16-rounded outputs to `stats_out`:
 * float2 [M][ceil(Cout/32)] (partials of one row sum to the row's totals) -- the ln_stats of the next LN_FOLD layer. */
#define ICAF_EPI_EMIT_STATS 16

int icaf_version(void);
const char* icaf_last_error(void);
/* Kernels this library has enqueued so far in this process (monotonic; one C-ABI compute call may launch more than one
 * kernel, e.g. a convolution whose last wave is peeled off as a split-K tail).  bench.py reports its per-step delta. */
long long icaf_kernel_launches(void);
/* Number of SMs of the current device (grid sizing of callers' workspaces); <0 on error.  Not affected by the target below. */
int icaf_sm_count(void);
/* SM-count target of the planners (as cublasSetSmCountTarget), process-wide: n > 0 makes every launch plan for
 * min(n, SM count of the device) SMs -- conv tile width, split-K and persistent CTA count, the weight-gradient splits
 * (and so icaf_conv2d_wgrad_workspace_bytes), the fused Bottleneck's CTAs and the grid-stride walkers' grids -- as on a
 * part or MIG slice with that many SMs; n = 0 restores the device's count; n < 0 is ICAF_ERR_BAD_ARG.
 *   - The target is read when a call plans its launch: CUDA graphs captured earlier keep the plans they captured, and a
 *     workspace sized under one target must be sized again under another.
 *   - Lowering the count never makes a launch need more co-resident CTAs than the full count does: persistent grids are
 *     at most the target in size, and split-K clusters are scheduled by the hardware as a unit. */
int icaf_set_sm_count_target(int n);

/* ---------------------------------------------------------------------------------------------
 * Implicit-GEMM convolution / linear layer on the Hopper tensor cores (wgmma).
 *   y[b,oy,ox,n] = epi( sum_{ky,kx,c} x[b, oy*s-p+ky, ox*s-p+kx, c] * w[n][(ky*kw+kx)*Cin + c] + bias[n] )
 * Replaces: Conv.forward / Conv.fuseforward (models/common.py:56-60: nn.Conv2d -> BatchNorm2d -> SiLU,
 * BN folded as utils/torch_utils.py:182-202), nn.Linear calls of CrossAttention / MLP
 * (common.py:660-668,683-685,704-715; a linear is the 1x1 case with Hi=Wi=1 rows as pixels) and
 * Detect's nn.Conv2d (models/yolo_test.py:49).
 * `n_io` problems of identical geometry (e.g. the RGB and the IR stream) run in one launch.
 * ------------------------------------------------------------------------------------------- */
typedef struct {
  int B, Hi, Wi, Cin; /* input  NHWC; Cin multiple of 8, or exactly 4 (packed 3-channel image, even Wi) */
  int Ho, Wo, Cout;   /* output NHWC */
  int kh, kw, stride, pad;
  int k_pad;  /* row pitch of the packed filter matrix: multiple of 64, >= kh*kw*Cin (zero padded) */
  int w_rows; /* rows present in the packed filter matrix (>= Cout, zero padded) */
  int act;    /* ICAF_ACT_* */
  int epi;    /* ICAF_EPI_* flags */
} icaf_conv_geom;

typedef struct {
  const void* x;     int64_t x_ld;   /* fp16 input view                                   */
  const void* w;                     /* fp16 [w_rows][k_pad], K order (ky,kx,c)           */
  const float* bias;                 /* fp32 [Cout] (or [rows] with BIAS_ROW); may be NULL */
  const void* res;   int64_t res_ld; /* fp16 residual view (ADD_RES / SCALED_RES) or NULL  */
  void* y;           int64_t y_ld;   /* fp16 output view                                   */
  const float* alpha;                /* device scalars for SCALED_RES                      */
  const float* beta;
  const float* ln_stats;             /* LN_FOLD: fp32 pairs [M][ln_parts] (sum, sum of squares) of the input rows */
  const float* ln_colsum;            /* LN_FOLD: fp32 [w_rows]                              */
  int ln_parts;                      /* LN_FOLD: partials per row, 1..64                     */
  float ln_eps;                      /* LN_FOLD: LayerNorm epsilon                           */
  float* stats_out;                  /* EMIT_STATS: fp32 pairs [M][ceil(Cout/32)]            */
} icaf_conv_io;

int icaf_conv2d_fwd(const icaf_conv_geom* g, const icaf_conv_io* io, int n_io, void* stream);

/* The dispatcher's decision for one layer geometry, computed on the HOST only (no device, no stream, no pointers):
 * which kernel family runs it, with which tile shapes, grid and shared memory.  icaf_conv2d_fwd launches exactly the
 * plan this returns for (geometry, n_io, SM count of the current device or its lower icaf_set_sm_count_target); the same
 * invariant checks run in both, so a GPU-less test can walk every layer of a model through the dispatcher
 * (tests/test_abi_cpu.py).
 * pair_mode: accepted for ABI stability and ignored (sm_90a has no CTA-pair MMA). */
#define ICAF_KERNEL_TC 0      /* wgmma implicit GEMM, 128 x BN tiles (conv_gemm.cu): one tile per CTA with split-K
                                 clusters, or, for BN = 128 grids of more than one wave, `ctas` persistent CTAs       */
typedef struct {
  int kernel;                            /* ICAF_KERNEL_*                                                     */
  int bn;                                /* output-channel tile width (32/64/128)                             */
  int a_mode;                            /* activation staging: 0 cp.async gather, 1 2-D TMA, 2 4-D TMA       */
  int tile_w, tile_h, tiles_x, tiles_y;  /* 4-D TMA: output-pixel tile and tiles per image                    */
  int cblk;                              /* channels per TMA box                                              */
  int halo;                              /* always 0 (halo copies belong to CTA-pair kernels)                 */
  int stages, splits;                    /* smem ring depth; split-K factor (= cluster size of the tc kernel) */
  int grid_x, grid_y, grid_z, cluster;   /* tile grid (m tiles x splits, n tiles, problems); cluster size     */
  int smem_bytes;                        /* dynamic shared memory per CTA                                     */
  int work_items;                        /* output tiles the grid covers                                      */
  int ctas;                              /* CTAs the launch starts: the tile grid's product, or at most the
                                            SM count when persistent CTAs walk the tiles                      */
} icaf_conv_plan;
int icaf_conv2d_plan(const icaf_conv_geom* g, int n_io, int sm_count, int pair_mode, icaf_conv_plan* out);

/* Test-only CUDA-core reference of the same contract (slow, obviously-correct); used by tests to
 * localise tensor-core bugs on the device.  Not called by the product path. */
int icaf_conv2d_fwd_simt(const icaf_conv_geom* g, const icaf_conv_io* io, int n_io, void* stream);

/* Fused Bottleneck with shortcut and 64 channels throughout (models/common.py:184-194, BN folded):
 *   y = x + SiLU(conv3x3/p1(h) + b2),   h = SiLU(conv1x1(x) + b1)
 * in one launch that keeps h on chip; the result equals icaf_conv2d_fwd of cv1 followed by that of cv2 with ADD_RES.
 * `n_io` problems of identical geometry (B, H, W) per launch.  x and y are fp16 NHWC views of 64 channels (16-byte aligned,
 * pitches multiples of 8); y must not overlap any x.  w1 / w3: the packed filters of icaf_conv2d_fwd (fp16 [64][64] and
 * [64][576], K order (ky,kx,c)); b1 / b2: fp32 [64]. */
typedef struct {
  const void* x;     int64_t x_ld;
  const void* w1;    const float* b1;
  const void* w3;    const float* b2;
  void* y;           int64_t y_ld;
} icaf_bottleneck_io;
int icaf_bottleneck_fwd(int B, int H, int W, const icaf_bottleneck_io* io, int n_io, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Input staging: (B,3,H,W) planar image -> fp16 NHWC with C padded to 4 (r,g,b,0).
 * Replaces the `.half()` / `/255` staging of detect_twostream.py:70-80 / train.py:295-297.
 * src_dtype: 0 = fp16, 1 = fp32, 2 = uint8 (scaled by `scale`, e.g. 1/255).
 * ------------------------------------------------------------------------------------------- */
int icaf_pack_image(const void* src, int src_dtype, float scale, int B, int H, int W, void* dst, void* stream);

/* Letterbox + BGR->RGB + HWC->CHW for a batch of decoded frames, on the device.  Replaces utils/datasets.py:1404-1427
 * letterbox (cv2.resize INTER_LINEAR + cv2.copyMakeBorder) and the `img[:, :, ::-1].transpose(2, 0, 1)` of datasets.py:238.
 * src: uint8 (B, H0, W0, 3) BGR; dst: uint8 (B, 3, H, W) RGB planar; the resized (new_h, new_w) frame sits at (top, left),
 * the rest is pad_value (114).  xtab / ytab: device int32 [new_w][4] = {x0, x1, a0, a1} and [new_h][4] = {y0, y1, b0, b1},
 * cv2's fixed-point bilinear taps (x 2048) -- built on the host (icafusion_b200/datasets.py:resize_taps); may be NULL when
 * (new_h, new_w) == (H0, W0).  Bit-exact against the cv2 pipeline. */
int icaf_letterbox(const void* src, int B, int H0, int W0, void* dst, int H, int W, int top, int left, int new_h, int new_w,
                   const int* xtab, const int* ytab, int pad_value, void* stream);

/* Validation batch staging: LoadMultiModalImagesAndLabels.__getitem__ (utils/datasets.py:948-1024) with augment=False,
 * rect=True -- load_image_rgb_ir's resize (:1097-1125: a copy at r = 1, cv2.resize INTER_LINEAR at r > 1, INTER_AREA at
 * r < 1), letterbox to the batch shape (scaleup=False: a border only), BGR->RGB, HWC->CHW -- and collate_fn's stack of the
 * 6-channel images, for a batch, one launch, bit-exact against cv2.  Geometry and tables are the host's
 * (icafusion_b200/valdata.py). */
#define ICAF_VAL_COPY 0        /* (h, w) == (H0, W0)                                                                     */
#define ICAF_VAL_LINEAR 1      /* INTER_LINEAR: xtab / ytab = int4 {i0, i1, w0, w1} rows [w] / [h] as for icaf_letterbox */
#define ICAF_VAL_AREA_FAST 2   /* INTER_AREA, integer scales sx, sy: block sums; 2 x 2 rounds (s + 2) >> 2, else
                                  saturate_cast<uchar>(s * (1.f / (sx sy)))                                                */
#define ICAF_VAL_AREA 3        /* INTER_AREA, other scales: xtab / ytab = [dst] int2 {first tap word (from the table),
                                  count} + int2 {si, alpha float bits} taps in cv2's order (computeResizeAreaTab)          */
typedef struct {
  const void* rgb; const void* ir;  /* device uint8 (H0, W0, 3) BGR frames of this sample                              */
  int H0, W0;                       /* decoded size                                                                    */
  int h, w;                         /* load_image size (int(h0 r), int(w0 r))                                          */
  int top, left;                    /* its place in the (H, W) batch image; the rest is 114                            */
  int mode;                         /* ICAF_VAL_*                                                                      */
  int xtab, ytab;                   /* word offsets of the column / row tables in the table region (16-byte aligned)   */
  int sx, sy;                       /* ICAF_VAL_AREA_FAST scales                                                        */
  int reserved;
} icaf_val_sample;

/* Bytes of the parameter block for B samples with n_words table words.  Layout: icaf_val_sample [B] at 0, int32 tables
 * [n_words] at align16(B * sizeof(icaf_val_sample)).  0 for a bad argument. */
size_t icaf_val_stage_params_bytes(int B, int n_words);

/* params: device block laid out as above (16-byte aligned); out: uint8 (B, 6, H, W) -- RGB frame in channels 0-2, IR frame
 * in 3-5, each R, G, B.  W % 4 == 0 (batch shapes are stride multiples). */
int icaf_val_stage(const void* params, size_t params_bytes, int B, int H, int W, int n_words, void* out, void* stream);

/* Same staging, space-to-depth layout: dst is (B, H/2, W/2, 16) fp16 with channel (dy*2+dx)*4 + c (c = r,g,b,0).
 * A 6x6 / stride 2 / pad 2 stem convolution over the image (yolov5 "P1/2" row of the model YAML) is then exactly a
 * 3x3 / stride 1 / pad 1 convolution over this tensor (ky = 2*ty+dy, kx = 2*tx+dx), which runs on the TMA path. H, W even. */
int icaf_pack_image_s2d(const void* src, int src_dtype, float scale, int B, int H, int W, void* dst, void* stream);

/* SPPF's three chained MaxPool2d(5,1,2) (models/common.py:259-266): y1,y2,y3 written as channel
 * slices; x is (B,H,W,C) view. */
int icaf_sppf_pool(const void* x, int64_t x_ld, void* y1, void* y2, void* y3, int64_t y_ld, int B, int H, int W,
                   int C, void* stream);

/* nn.Upsample(None, 2, 'nearest') (yolov5l_Transfusion_kaist.yaml:48,53) into a channel slice. */
int icaf_upsample2x(const void* x, int64_t x_ld, void* y, int64_t y_ld, int B, int H, int W, int C, void* stream);

/* Pull a read-only region (packed filters) into L2 ahead of its consumers: after an L2 flush every layer would
 * otherwise pay a DRAM round trip for its first filter tile.  Touches no data; purely a cache hint. */
int icaf_prefetch_l2(const void* ptr, size_t bytes, void* stream);

/* Copy a channel slice (Concat, models/common.py:313-321, when producer-side slice writes are not possible). */
int icaf_copy_channels(const void* x, int64_t x_ld, void* y, int64_t y_ld, int64_t pixels, int C, void* stream);

/* ---------------------------------------------------------------------------------------------
 * DMFF block pieces (models/common.py:762-891).
 * ------------------------------------------------------------------------------------------- */
/* AdaptivePool2d avg+max (common.py:868-891) + LearnableWeights (:579-587) + flatten/permute + pos_emb (:817-823):
 *   tok[b, n, c] = w[0]*avgpool + w[1]*maxpool + pos[n, c];  rows n in [N, Npad) are zeroed.
 * Two modalities per launch (x0/x1 ...). `mix` = 4 device floats {w1_vis, w2_vis, w1_ir, w2_ir}.
 * stats_* (both or neither; C % 32 == 0): fp32 pairs [B*Npad][C/32] (sum, sum of squares) of every token row per 32
 * channels -- the ln_stats (ln_parts = C/32) of the LN_FOLD projection that consumes the tokens. */
int icaf_dmff_pool_tokens(const void* x_vis, const void* x_ir, int64_t x_ld, const void* pos_vis, const void* pos_ir,
                          const float* mix, void* tok_vis, void* tok_ir, float* stats_vis, float* stats_ir, int B, int H,
                          int W, int C, int nh, int nw, int n_pad, void* stream);

/* nn.LayerNorm over the last dim (eps 1e-5) of `rows` x C fp16 tokens; two independent problems per launch
 * (x1 may be NULL).  gamma/beta are fp32 [C].  Replaces common.py:660,665,749-750. */
int icaf_layernorm(const void* x0, const void* x1, const float* g0, const float* b0, const float* g1,
                   const float* b1, void* y0, void* y1, int64_t rows, int C, float eps, void* stream);

/* (sum, sum of squares) of every row of a (rows, C) fp16 matrix -> fp32 pairs [rows][1]: the `ln_stats` (ln_parts = 1) of
 * an LN_FOLD layer whose input no EMIT_STATS epilogue produced (first loop of a DMFF block, stand-alone calls).
 * Two problems per launch (x1 may be NULL). */
int icaf_row_stats(const void* x0, const void* x1, float* stats0, float* stats1, int64_t rows, int C, void* stream);

/* Bidirectional cross-attention core (common.py:670-684), flash style: no N x N score matrix in HBM.
 *   out_vis = softmax(q_ir k_vis^T / sqrt(d)) v_vis ;  out_ir = softmax(q_vis k_ir^T / sqrt(d)) v_ir
 * Two input forms:
 *   fused  (vt_vis == vt_ir == NULL): qk_* are fp16 (B, Npad, 3C) rows [q | k | v] exactly as ONE fused projection GEMM
 *          emits them; the V tiles feed the tensor core as MN-major operands, no transpose anywhere;
 *   split  : qk_* fp16 (B, Npad, 2C) rows [q | k], vt_* fp16 (C, B*Npad) value projection stored transposed.
 * out_*: fp16 (B, Npad, C) heads merged (the layout out_proj consumes).  Every tile is staged by TMA.
 * Head dim C / heads: a multiple of 8 in [8, 128], or 160; others return ICAF_ERR_UNSUPPORTED. */
int icaf_cross_attention(const void* qk_vis, const void* qk_ir, const void* vt_vis, const void* vt_ir, void* out_vis,
                         void* out_ir, int B, int N, int n_pad, int C, int heads, void* stream);

/* Test-only CUDA-core reference of icaf_cross_attention (same contract, head dims up to 128 only). */
int icaf_cross_attention_simt(const void* qk_vis, const void* qk_ir, const void* vt_vis, const void* vt_ir,
                              void* out_vis, void* out_ir, int B, int N, int n_pad, int C, int heads, void* stream);

/* Token map -> feature map tail (common.py:827-840): reshape (B,nh,nw,C), F.interpolate to (H,W)
 * (mode 0 = bilinear align_corners=False [eval], 1 = nearest [train]), add the stream's own features,
 * write both modalities into one (B,H,W,2C) buffer = the Concat that feeds conv1x1_out. */
int icaf_dmff_upsample_cat(const void* tok_vis, const void* tok_ir, int n_pad, const void* x_vis, const void* x_ir,
                           int64_t x_ld, void* y, int64_t y_ld, int B, int H, int W, int C, int nh, int nw, int mode,
                           void* stream);

/* Detect head decode (models/yolo_test.py:49-65) for one level.  `p` is the 1x1-conv output
 * (B,ny,nx,p_ld) fp16 with na*no valid channels.  Writes
 *   x_out  (B,na,ny,nx,no) fp16  raw,   z (B, total_rows, no) rows [row_off, row_off+na*ny*nx) decoded,
 *   logits (B, total_rows, no-5) same rows.  anchors: host array na*2 floats (pixels). */
int icaf_detect_decode(const void* p, int64_t p_ld, void* x_out, void* z, void* logits, int B, int ny, int nx, int na,
                       int no, int total_rows, int row_off, float stride, const float* anchors_host, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Batched non-maximum suppression on the decoded predictions, fully on the device.
 * Replaces utils/general.py:518-607 non_max_suppression (best-class branch: conf = obj * max cls, both > conf_thres,
 * class-offset boxes unless `agnostic`, torchvision.ops.nms greedy suppression at iou_thres, max_nms = 30000 candidates,
 * first max_det kept).  z: fp16 (B, R, no) as icaf_detect_decode writes it; arithmetic in fp32 like the reference on
 * z.float().  class_mask: bit k set = keep class k (0 = all classes; at most 64 classes with a mask).
 * det: fp32 (B, max_det, 6) rows [x1, y1, x2, y2, conf, cls] in confidence order; count: int32 (B) rows valid per image.
 * workspace: icaf_nms_workspace_bytes(B, R) bytes of device memory, 8-byte aligned (caller owned).
 * ------------------------------------------------------------------------------------------- */
size_t icaf_nms_workspace_bytes(int B, int R);
int icaf_nms(const void* z, int B, int R, int no, float conf_thres, float iou_thres, int agnostic, uint64_t class_mask,
             int max_det, float* det, int* count, void* workspace, size_t workspace_bytes, void* stream);

/* Multi-label branch of the same function (utils/general.py:566-568, what test.py:139 asks for): one candidate per
 * (row, class j) with obj > conf_thres and cls_j * obj > conf_thres (class_mask applies per pair), sorted by descending
 * confidence with ties in (row * nc + j) order, cut to the first max_nms = 30000, then the same suppression.  A box may be
 * kept once per class (once in all unless `agnostic`).  det rows [x1, y1, x2, y2, cls_j * obj, j].  Same arguments as
 * icaf_nms; workspace: icaf_nms_multi_label_workspace_bytes(B, R, no) bytes (16 per row and class), 8-byte aligned;
 * R * (no - 5) must fit in int.  Returns 0 from the size query for a bad shape. */
size_t icaf_nms_multi_label_workspace_bytes(int B, int R, int no);
int icaf_nms_multi_label(const void* z, int B, int R, int no, float conf_thres, float iou_thres, int agnostic,
                         uint64_t class_mask, int max_det, float* det, int* count, void* workspace, size_t workspace_bytes,
                         void* stream);

/* ---------------------------------------------------------------------------------------------
 * Confluence on the decoded predictions, fully on the device: the reference's alternative to NMS
 * (utils/confluence.py:50-193 confluence_process + confluence), clustering by normalised Manhattan distance.
 * z: (B, R, no) decoded predictions, dtype 0 = fp16 or 1 = fp32 (read as they are: fp32 input is never rounded to fp16).
 * Candidates: one per (row r, class j) with obj > conf_thres and cls_j * obj > conf_thres in fp32 (for nc == 1 this is the
 * reference's best-class branch, otherwise its multi_label branch); boxes by xywh2xyxy in fp32.  Per class, in row order,
 * in fp64 on the widened values: p_ab = sum over x1, x2, y1, y2 of |a' - b'| with each axis normalised by the min and
 * max of its four coordinates (a degenerate axis gives NaN, which neither counts nor removes); the first box with the
 * smallest min over p_ij < 2 of p_ij / conf_i (0 without such j) is kept, and it and every box with p < p_thres leave.
 * det: fp32 (B, max_det, 6) rows [x1, y1, x2, y2, conf, cls] in ascending (row, class) order -- the reference's
 * np.unique(keep) order; there is no max_det cut in the reference, so count: int32 (B) holds the TRUE number kept per
 * image, and when it exceeds max_det the rows past max_det were not written (rows at or past the count are untouched).
 * index: optional int32 (B, max_det), the row r of each written detection (NULL: not written).
 * dtype 2: z holds fp32 detection rows (B, R, 6) [x1, y1, x2, y2, conf, cls], the input of confluence(): a row belongs to
 * class j when its cls == j (j < no - 5), there is no threshold (conf_thres is ignored) and every conf must be >= 2.5e-4.
 * conf_thres must be >= 2.5e-4: below 2e-4 the reference's scan, which starts at 10000, can find no box and raises.
 * Up to 6144 candidates of one class are clustered in shared memory, more in the workspace (correct at any count, slower).
 * workspace: icaf_confluence_workspace_bytes(B, R, no) bytes of device memory, 16-byte aligned (37 bytes per row and class
 * plus 1); R * (no - 5) must fit in int, B <= 65535.  Returns 0 from the size query for a bad shape.
 * ------------------------------------------------------------------------------------------- */
size_t icaf_confluence_workspace_bytes(int B, int R, int no);
int icaf_confluence(const void* z, int dtype, int B, int R, int no, float conf_thres, double p_thres, float* det, int* index,
                    int max_det, int* count, void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Validation: match one batch's NMS detections to its labels (test.py:196-227), one launch, no host round trip.
 * det / count: what icaf_nms / icaf_nms_multi_label write, fp32 (B, max_det, 6) and int32 (B).
 * targets: fp32 (T, 6) rows [image, cls, x, y, w, h] normalised to the (height, width) batch, in any order; rows whose image
 * is not one of 0..B-1 are ignored.  ratio_pad: fp32 (B, 5) rows [h0, w0, gain, padw, padh] (the loader's shapes[i]).
 * iouv: device fp32 (niou), 1 <= niou <= 32.  single_cls: every prediction counts as class 0.
 * Per image: both box sets go through scale_coords (pad, IEEE division by gain, clip to h0 x w0); each prediction takes the
 * first label of its class with the largest IoU; in row order, a prediction with IoU > iouv[0] whose label is not yet taken
 * takes it, and correct[b, r, k] = IoU > iouv[k].  correct: uint8 (B, max_det, niou); rows at or past count[b] are zero.
 * native: optional fp32 (B, max_det, 4), 16-byte aligned: the scale_coords boxes of the predictions (zero past count[b]).
 * workspace: icaf_match_detections_workspace_bytes(T) bytes of device memory, 4-byte aligned (may be NULL when T == 0).
 * ------------------------------------------------------------------------------------------- */
size_t icaf_match_detections_workspace_bytes(int T);
int icaf_match_detections(const float* det, const int* count, int B, int max_det, const float* targets, int T,
                          const float* ratio_pad, int height, int width, const float* iouv, int niou, int single_cls,
                          unsigned char* correct, float* native, void* workspace, size_t workspace_bytes, void* stream);

/* ---- KAIST log-average miss rate (evaluation_script/evaluation_script.py: evaluate) -------------------------------------
 * The nine evaluations of evaluate() (all, day, night on setup 0 over all / the first day_images / the other images; near,
 * medium, far, none, partial, heavy on setups 1-6 over all images) in one call: per (setup, image) the reference's greedy
 * matching at IoU 0.5 (its quirks included: the score sort applied twice to the IoU rows, a match on annotation id 0 counts
 * as a false positive), then one stable sort of all detections by descending score and one accumulation per evaluation.
 * gts, in CSR per image (images in ascending id order; gt_offset: int (images + 1)), in annotation-file order within an
 * image: gt_box float64 (gts, 4) x, y, w, h; gt_height float64 (gts); gt_occlusion, gt_ignore (the file's flag) int (gts);
 * gt_id int64 (gts), the annotation ids.  Detections: dt_rows float64 (rows, 5) x, y, w, h, score; dt_span int (images, 2)
 * (offset, count) per image, rows in file order, spans disjoint and in image order; every count <= max_per_image <= 1000.
 * Out: ys float64 (9, 9), the recall at each fppi threshold (-1 where the reference leaves -1: no image with detections or
 * no regular gt among them); counts int (9, 3): kept detections (the curve's length), their true positives, npig;
 * curves (optional) float64 (9, 2, rows): fppi and 1 - recall over the kept detections.  No host synchronisation.
 * workspace: icaf_kaist_mr_workspace_bytes(images, gts, rows) bytes, 256-byte aligned (0 = bad sizes, or no CUDA device
 * to size the radix sort's storage on).
 * ------------------------------------------------------------------------------------------- */
size_t icaf_kaist_mr_workspace_bytes(int images, int gts, int rows);
int icaf_kaist_mr(const double* gt_box, const double* gt_height, const int* gt_occlusion, const int* gt_ignore,
                  const long long* gt_id, const int* gt_offset, int images, int gts, int day_images, const double* dt_rows,
                  const int* dt_span, int rows, int max_per_image, double* ys, int* counts, double* curves, void* workspace,
                  size_t workspace_bytes, void* stream);
/* test.py's result lines in memory: for image b of a batch (B, max_det) and p = image[b] (its dataset index, < images),
 * rows[p * max_det + i] = float64 of `%g` of the fp32 x1, y1, x2 - x1, y2 - y1 of native[b, i] and the score det[b, i, 4]
 * (what float() reads back from the line), and span[p] = (p * max_det, count[b]): the dense layout of icaf_kaist_mr.  Exact
 * for values 0 and 1e-7 <= |v| < 1e6. */
int icaf_kaist_round_detections(const float* native, const float* det, const int* count, const int* image, int B, int max_det,
                                int images, double* rows, int* span, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Per-image validation results in one compact, ordered buffer (csrc/metrics.cu), so that the batches of a validation split
 * over ranks can be exchanged and put back in the one-process order.
 *
 * icaf_val_pack walks a parameter block of n_batches icaf_val_batch entries (in local image order: entry k covers local
 * images local0 .. local0 + B - 1), followed, with ICAF_VAL_PACK_POS, by an int32 region of n_images KAIST annotation
 * positions (16-byte aligned).  It writes the int32 words of one exchange buffer:
 *   [0..3]                      {n_images, n_rows, row_words, total_words}
 *   [4 + 4 k ..]                per image k: {global image index, kept count, first row, position (-1 without POS)}
 *   [4 + 4 n_images + r * row_words ..]   row r: {conf, class (fp32 bits), correct (bit j = iouv[j]), x1, y1, x2, y2 (NATIVE)}
 * The rows of an image follow its detections' order; the first rows come from an exclusive scan over the counts in local
 * image order (no atomics).  Counts are clamped to [0, max_det].  No allocation, no host synchronisation.
 *
 * icaf_val_merge takes n_bufs such buffers, buffer b at word b * buf_words, and writes flat arrays in global image order:
 * correct uint8 (n_rows, niou), conf / pcls fp32 (n_rows), native fp32 (n_rows, 4) (NATIVE), counts int32 (n_images),
 * offsets int32 (n_images + 1).  With mr_rows / mr_span it also writes the icaf_kaist_round_detections layout of every image
 * that has a position p < mr_images: rows at p * mr_max_det, span[p] = (p * mr_max_det, count); mr_span must be zeroed.
 * status int32 [4] = {images missing from every buffer, images in more than one buffer, malformed entries (image or
 * position out of range, inconsistent headers), rows written}: the merge is valid only when status == {0, 0, 0, n_rows}.
 * ------------------------------------------------------------------------------------------- */
#define ICAF_VAL_PACK_NATIVE 1   /* rows carry the native (scale_coords) box                                          */
#define ICAF_VAL_PACK_POS 2      /* the parameter block holds the KAIST positions region; headers carry them          */
typedef struct {
  const float* det;              /* fp32 (B, max_det, 6): what icaf_nms writes                                         */
  const int* count;              /* int32 (B)                                                                          */
  const unsigned char* correct;  /* uint8 (B, max_det, niou): what icaf_match_detections writes                        */
  const float* native;           /* fp32 (B, max_det, 4), or null without ICAF_VAL_PACK_NATIVE                         */
  int64_t image0;                /* global image index of the batch's first image                                      */
  int B, max_det;
  int local0;                    /* the batch's first image in the buffer                                              */
  int reserved[3];               /* 64-byte entries                                                                    */
} icaf_val_batch;

/* Bytes of the parameter block (0 for bad sizes). */
size_t icaf_val_pack_params_bytes(int n_batches, int n_images, int flags);
/* Bytes of the exchange buffer for n_images images of at most max_det rows (0 for bad sizes or overflow). */
size_t icaf_val_pack_bytes(int n_images, int max_det, int flags);
int icaf_val_pack(const void* params, size_t params_bytes, int n_batches, int n_images, int niou, int flags, void* out,
                  size_t out_bytes, void* stream);
/* Workspace of icaf_val_merge (0 for bad sizes). */
size_t icaf_val_merge_workspace_bytes(int n_images);
int icaf_val_merge(const void* bufs, int n_bufs, int64_t buf_words, int n_images, int n_rows, int niou, int flags,
                   unsigned char* correct, float* conf, float* pcls, float* native, int* counts, int* offsets, int* status,
                   double* mr_rows, int* mr_span, int mr_images, int mr_max_det, void* workspace, size_t workspace_bytes,
                   void* stream);

/* ---------------------------------------------------------------------------------------------
 * Detection loss, forward only (the validation loss test.py:132-133 accumulates; the training backward is not built):
 * utils/loss.py:325-463 ComputeLoss.__call__ + build_targets -- anchor-ratio matching with the four half-cell neighbour
 * offsets, CIoU box loss, objectness BCE against IoU-valued targets (largest IoU wins a contested cell), class BCE.
 * p: nl device pointers to the Detect training outputs (B, na, ny[i], nx[i], no), fp16 (p_fp32 = 0) or fp32 (1); arithmetic
 * in fp32.  targets: device fp32 (nt, 6) rows [image, class, x, y, w, h] normalised to [0, 1].  anchors_host: nl*na*2 floats
 * in grid units (Detect.anchors).  out: 5 device floats [loss * batch, lbox, lobj, lcls, 0].  fl_gamma > 0 wraps both BCE
 * terms in FocalLoss(gamma, alpha = 0.25) (loss.py:37-64, 341-344), in the forward and the backward; <= 0 keeps plain BCE.
 * Deterministic: no floating-point atomics.  workspace: icaf_loss_workspace_bytes(...) bytes, 256-byte aligned.
 * ------------------------------------------------------------------------------------------- */
typedef struct {
  float box, obj, cls;   /* loss gains hyp['box'], hyp['obj'], hyp['cls'] (already scaled as train.py:226-228 does) */
  float cls_pw, obj_pw;  /* BCE positive weights                                                                   */
  float anchor_t;        /* anchor-multiple threshold                                                              */
  float fl_gamma;        /* focal-loss gamma; > 0 turns the focal loss on for the class and objectness BCE         */
  float gr;              /* model.gr: objectness target = (1 - gr) + gr * iou                                      */
  float cp, cn;          /* smoothed positive / negative class targets (smooth_BCE, loss.py:15-17)                 */
  float balance[5];      /* per-level objectness weights: {4, 1, 0.4} for three levels (loss.py:346)               */
} icaf_loss_hyp;
/* p_ld: 0 when p[i] is the reference's (B, na, ny, nx, no) contiguous tensor; otherwise the pixel pitch (elements) of the
 * head's own (B, ny, nx, na*no) NHWC map (the training path hands the 1x1 head convolution's output over without a permute).
 * no_bwd: 0 for a forward-only workspace, `no` when icaf_compute_loss_bwd will follow. */
size_t icaf_loss_workspace_bytes(int B, int na, int nt, const int* ny, const int* nx, int nl, int no_bwd);
int icaf_compute_loss_fwd(const void* const* p, int p_fp32, int p_ld, const int* ny, const int* nx, int nl, int B, int na, int no,
                          const float* targets, int nt, const float* anchors_host, const icaf_loss_hyp* hyp, float* out,
                          void* workspace, size_t workspace_bytes, void* stream);
/* Backward of the loss (train.py:344 starts here): dp[i] = grad_out[0] * d out[0] / d p[i], in the dtype and memory layout of
 * p[i] (every element of the (cells x no) slab is written; pad channels of an NHWC map with p_ld > na*no are left alone).
 * Same arguments as the forward call that filled `workspace` (sized with no_bwd = no); grad_out: device fp32 scalar (the
 * GradScaler factor arrives here).  The CIoU derivative is the forward expression evaluated on forward-mode duals; the
 * objectness target and CIoU's alpha are constants, as in the reference (loss.py:372, general.py:444).  Candidate gradients
 * meeting in one cell are summed in fp32 by ascending candidate index (level, target, anchor, offset), then rounded once:
 * bit-reproducible, no floating-point atomics. */
int icaf_compute_loss_bwd(const void* const* p, int p_fp32, int p_ld, const int* ny, const int* nx, int nl, int B, int na, int no,
                          const float* targets, int nt, const float* anchors_host, const icaf_loss_hyp* hyp, const float* grad_out,
                          void* const* dp, void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Training-step building blocks (train.py:344 backward of the hot path's nn.Conv2d / nn.Linear layers).  Operator level
 * only: the whole-model backward / optimiser / DDP loop is not built (DESIGN.md section 7).
 * ------------------------------------------------------------------------------------------- */
/* Weight gradient dW[n][c][ky][kx] (fp32, PyTorch layout) = (accumulate ? dW : 0) + scale * sum_pixels dy[.., n] * x[.. shifted .., c]
 * of the convolution / linear layer described by `g` (Cin 16, 32 or a multiple of 64; Cout % 8 == 0; stride 1 or 2).
 * x, dy: fp16 NHWC views (pixel pitch x_ld / dy_ld).  wgmma GEMM over pixels with both operands MN-major, split over
 * the pixel range, splits summed in a fixed order (deterministic).  scale: 1 / loss scale.  workspace: caller owned,
 * icaf_conv2d_wgrad_workspace_bytes(g) bytes, 16-byte aligned. */
size_t icaf_conv2d_wgrad_workspace_bytes(const icaf_conv_geom* g);
int icaf_conv2d_wgrad(const icaf_conv_geom* g, const void* x, int64_t x_ld, const void* dy, int64_t dy_ld, float* dw, float scale,
                      int accumulate, void* workspace, size_t workspace_bytes, void* stream);
/* y (B, H2, W2, C) = x (B, H, W, C) with a zero between every two pixels (y[b, 2i, 2j] = x[b, i, j]): the data gradient of a
 * stride-2 convolution is the stride-1 icaf_conv2d_fwd of this tensor with the flipped, transposed filter. */
int icaf_zero_stuff2(const void* x, void* y, int B, int H, int W, int C, int H2, int W2, void* stream);
/* out[c] (fp32) = (accumulate ? out[c] : 0) + scale * sum_rows x[r][c] of a dense fp16 (rows, C) matrix: bias gradients.
 * Deterministic two-stage sum; workspace: 64 * C floats. */
int icaf_colsum(const void* x, int64_t rows, int C, float* out, float scale, int accumulate, float* workspace, size_t workspace_bytes,
                void* stream);

/* Reduction scratch of the kernels below: icaf_train_workspace_bytes(C) bytes (fp32, 16-byte aligned), plus what each states. */
size_t icaf_train_workspace_bytes(int C);
/* BatchNorm2d with BATCH statistics + activation (Conv.forward in training mode, models/common.py:56-57; act: 0 none, 1 SiLU):
 * x, y: dense fp16 (rows, C) = NHWC maps; statistics in fp32 over the rows; run_mean / run_var (may be NULL) get the momentum
 * update with the unbiased variance like nn.BatchNorm2d; save_mean / save_invstd (fp32 [C]) feed the backward. */
int icaf_bn_act_fwd(const void* x, const float* gamma, const float* beta, float* run_mean, float* run_var, void* y, float* save_mean,
                    float* save_invstd, int64_t rows, int C, float eps, float momentum, int act, float* workspace, size_t workspace_bytes,
                    void* stream);
/* Its backward: dx (fp16) and dgamma / dbeta (fp32, (accumulate ? += : =) grad_scale * value; may be NULL).
 * workspace: icaf_train_workspace_bytes(C) (it includes the per-channel coefficient block of the apply pass). */
int icaf_bn_act_bwd(const void* x, const void* dy, const float* gamma, const float* beta, const float* save_mean, const float* save_invstd,
                    void* dx, float* dgamma, float* dbeta, int64_t rows, int C, int act, float grad_scale, int accumulate, float* workspace,
                    size_t workspace_bytes, void* stream);
/* The same two calls in two phases each, for a BatchNorm synchronised over ranks (torch.nn.SyncBatchNorm).  The caller sums
 * the exchange buffer over the ranks between the phases (all-reduce).  Fed phase 1's buffer unchanged, phase 2 gives what
 * icaf_bn_act_fwd / icaf_bn_act_bwd give, bit for bit, for rows <= 2^24.
 * Forward phase 1: stats (fp32 [2C + 1]) = (sum x [C], sum x^2 [C], rows).  The count travels as fp32: above 2^24 rows it is
 * rounded, a relative error of at most 6e-8, below the error of the fp32 sums themselves.
 * Forward phase 2: mean, invstd and the running-statistics update (unbiased with the summed count) from the summed stats, then
 * y as icaf_bn_act_fwd.  The count is read from device memory: ranks may hold different row counts and no host read is needed.
 * Backward phase 1: dgamma / dbeta of this rank's rows as icaf_bn_act_bwd (DDP averages them), and sums (fp32 [2C]) =
 * (sum dz, sum dz * xhat).  Backward phase 2: dx from the summed sums and the forward's summed count (count = stats + 2C).
 * rows: this rank's rows.  workspace: icaf_train_workspace_bytes(C) each. */
int icaf_bn_act_fwd_stats(const void* x, int64_t rows, int C, float* stats, float* workspace, size_t workspace_bytes, void* stream);
int icaf_bn_act_fwd_apply(const void* x, const float* gamma, const float* beta, float* run_mean, float* run_var, const float* stats, void* y,
                          float* save_mean, float* save_invstd, int64_t rows, int C, float eps, float momentum, int act, float* workspace,
                          size_t workspace_bytes, void* stream);
int icaf_bn_act_bwd_sums(const void* x, const void* dy, const float* gamma, const float* beta, const float* save_mean, const float* save_invstd,
                         float* dgamma, float* dbeta, float* sums, int64_t rows, int C, int act, float grad_scale, int accumulate, float* workspace,
                         size_t workspace_bytes, void* stream);
int icaf_bn_act_bwd_apply(const void* x, const void* dy, const float* gamma, const float* beta, const float* save_mean, const float* save_invstd,
                          const float* sums, const float* count, void* dx, int64_t rows, int C, int act, float* workspace, size_t workspace_bytes,
                          void* stream);
/* Element-wise over n fp16 values (n % 8 == 0): mode 0 y = GELU_erf(x) (common.py:706); 1 y = dy * GELU'(x);
 * 2 y = dropout(x, p) with a counter-based mask keyed by (element index, seed) -- calling it on dy with the same seed is the backward. */
int icaf_eltwise(int mode, const void* x, const void* dy, void* y, int64_t n, float p, uint32_t seed, void* stream);
/* nn.LayerNorm backward over dense fp16 (rows, C), C <= 2048: dx, dgamma, dbeta as above.
 * workspace: icaf_train_workspace_bytes(C) + 2 rows floats. */
int icaf_layernorm_bwd(const void* x, const void* dy, const float* gamma, void* dx, float* dgamma, float* dbeta, int64_t rows, int C, float eps,
                       float grad_scale, int accumulate, float* workspace, size_t workspace_bytes, void* stream);
/* out[0] = (accumulate ? out[0] : 0) + scale * <x, y> over dense fp16 (rows, C): gradients of LearnableCoefficient / LearnableWeights. */
int icaf_dot(const void* x, const void* y, int64_t rows, int C, float* out, float scale, int accumulate, float* workspace, size_t workspace_bytes,
             void* stream);
/* Backward of nn.Upsample(None, 2, 'nearest'): dx (B, H, W, C) = sums of the 2 x 2 blocks of dy (B, 2H, 2W, C). */
int icaf_upsample2x_bwd(const void* dy, void* dx, int B, int H, int W, int C, void* stream);
/* Backward of one MaxPool2d(5, 1, 2) of SPPF's chain (common.py:259-266): x is that pool's input, dy the gradient of its output
 * (dense fp16 NHWC, C % 8 == 0).  workspace: B*H*W*C bytes (one arg-max code per window and channel), 8-byte aligned. */
int icaf_maxpool5_bwd(const void* x, const void* dy, void* dx, int B, int H, int W, int C, void* workspace, size_t workspace_bytes, void* stream);

/* Backward of icaf_dmff_pool_tokens w.r.t. the two feature maps (dense fp16 (B,H,W,C) gradients): every pixel gathers, from
 * each pooling window that contains it, dtok * (w_avg / window + w_max * [pixel is the window's first maximum]).  The
 * gradients of the mixing weights and positional embeddings are plain reductions of dtok (icaf_dot / icaf_colsum). */
int icaf_dmff_pool_tokens_bwd(const void* x_vis, const void* x_ir, int64_t x_ld, const void* dtok_vis, const void* dtok_ir, const float* mix,
                              void* dx_vis, void* dx_ir, int B, int H, int W, int C, int nh, int nw, int n_pad, void* workspace,
                              size_t workspace_bytes, void* stream);   /* workspace: 2*B*nh*nw*C bytes (arg-max codes), 8-byte aligned */
/* Backward of icaf_dmff_upsample_cat (mode 1, nearest: the training-mode tail, common.py:828-829) w.r.t. the token streams:
 * dtok[b][n] = sum of dcat over the pixels token n was copied to (pad rows get 0).  dcat: (B,H,W,2C) with pixel pitch d_ld;
 * the gradients of the two residual inputs are its channel halves. */
int icaf_dmff_upsample_cat_bwd(const void* dcat, int64_t d_ld, void* dtok_vis, void* dtok_ir, int B, int H, int W, int C, int nh, int nw,
                               int n_pad, int mode, void* stream);
/* fp32 master filter (Cout,Cin,kh,kw) -> fp16 bank [rows][k_pad] of icaf_conv2d_fwd, K order (ky,kx,channel), channel count
 * padded to chan_pad, padding written as zero.  transpose_flip = 0: the forward filter (rows >= Cout, channels = Cin);
 * 1: the data-gradient filter W'[c][n][ky][kx] = W[n][c][kh-1-ky][kw-1-kx] (rows >= Cin, channels = Cout). */
int icaf_pack_weight(const float* w, int Cout, int Cin, int kh, int kw, int chan_pad, int rows, int k_pad, int transpose_flip, void* out,
                     void* stream);
/* Both banks of one filter in one launch: out_fwd [rows_f][kpad_f] (channels = Cin) and out_dgrad [rows_d][kpad_d] (channels = Cout
 * padded to chan_pad_d). */
int icaf_pack_weight_pair(const float* w, int Cout, int Cin, int kh, int kw, int rows_f, int kpad_f, void* out_fwd, int chan_pad_d, int rows_d,
                          int kpad_d, void* out_dgrad, void* stream);

/* Optional device-side counter (one uint32) added to every dropout seed by the kernels at run time (NULL switches it off).  A
 * captured CUDA graph of the training step keeps its host-side seeds; bumping this counter on the device between replays gives
 * every replay fresh dropout masks, and the forward / backward kernels of one step still regenerate identical masks. */
int icaf_set_seed_offset(const void* device_u32);

/* Training-mode forward of the fused form: like icaf_cross_attention(qkv_vis, qkv_ir, NULL, NULL, ...) plus dropout with
 * probability p_drop on the attention probabilities (common.py:677,680; counter-based mask keyed by `seed`, reproduced by the
 * backward below).  Head dims up to 128 only: 160 has no dropout kernel and no backward. */
int icaf_cross_attention_train(const void* qkv_vis, const void* qkv_ir, void* out_vis, void* out_ir, int B, int N, int n_pad, int C, int heads,
                               float p_drop, uint32_t seed, void* stream);

/* Backward of icaf_cross_attention in its fused form (qkv_* fp16 (B, Npad, 3C) rows [q | k | v]; out_* the forward outputs,
 * dout_* their gradients, fp16 (B, Npad, C)): dqkv_* (same layout as qkv_*; pad rows zeroed).  Probabilities are recomputed;
 * p_drop / seed reproduce the dropout mask of a training forward (0 = none).  CUDA-core kernels for the pooled-token regime.
 * workspace: icaf_cross_attention_bwd_workspace_bytes(B, n_pad, heads). */
size_t icaf_cross_attention_bwd_workspace_bytes(int B, int n_pad, int heads);
int icaf_cross_attention_bwd(const void* qkv_vis, const void* qkv_ir, const void* out_vis, const void* out_ir, const void* dout_vis,
                             const void* dout_ir, void* dqkv_vis, void* dqkv_ir, int B, int N, int n_pad, int C, int heads, float p_drop,
                             uint32_t seed, void* workspace, size_t workspace_bytes, void* stream);

/* out = a[0] * x (+ b[0] * y when y != NULL) over n fp16 elements (n % 8 == 0, 16-byte aligned); a, b device fp32 scalars.
 * LearnableCoefficient.forward / LearnableWeights.forward called stand-alone (models/common.py:569-587). */
int icaf_axpby(const void* x, const void* y, const float* a, const float* b, void* out, int64_t n, void* stream);

/* ---------------------------------------------------------------------------------------------
 * fp32 DMFF token streams (training).  Under the reference's autocast a one-element fp32 parameter (LearnableWeights,
 * LearnableCoefficient) times an fp16 tensor promotes to fp32, so its token streams are fp32 from the pooling to the
 * upsample-and-add, and so are their gradients; GEMM operands are fp16 (autocast's cast at every Linear).  These entry points
 * are the fp32-stream forms of the calls above: tokens and token gradients fp32, maps, map gradients, LayerNorm outputs and
 * branch outputs fp16.  Every reduction keeps the fixed order of its fp16 form (deterministic, no atomics). */
/* icaf_dmff_pool_tokens with fp32 pos_emb and fp32 tokens: tok = fp32(w1 * fp16(avg)) + fp32(w2 * max) + pos, each step
 * rounded (no FMA contraction), pad rows 0.  No row statistics. */
int icaf_dmff_pool_tokens_f32(const void* x_vis, const void* x_ir, int64_t x_ld, const float* pos_vis, const float* pos_ir, const float* mix,
                              float* tok_vis, float* tok_ir, int B, int H, int W, int C, int nh, int nw, int n_pad, void* stream);
/* icaf_dmff_pool_tokens_bwd with fp32 token gradients; the map gradients are fp16, accumulated in fp32 and rounded once. */
int icaf_dmff_pool_tokens_bwd_f32(const void* x_vis, const void* x_ir, int64_t x_ld, const float* dtok_vis, const float* dtok_ir, const float* mix,
                                  void* dx_vis, void* dx_ir, int B, int H, int W, int C, int nh, int nw, int n_pad, void* workspace,
                                  size_t workspace_bytes, void* stream);   /* workspace: 2*B*nh*nw*C bytes, 8-byte aligned */
/* icaf_dmff_upsample_cat in its training mode (nearest) over fp32 tokens: token + map added in fp32, rounded once to the fp16
 * concat buffer. */
int icaf_dmff_upsample_cat_f32(const float* tok_vis, const float* tok_ir, int n_pad, const void* x_vis, const void* x_ir, int64_t x_ld,
                               void* y, int64_t y_ld, int B, int H, int W, int C, int nh, int nw, void* stream);
/* icaf_dmff_upsample_cat_bwd (nearest) with fp32 token gradients. */
int icaf_dmff_upsample_cat_bwd_f32(const void* dcat, int64_t d_ld, float* dtok_vis, float* dtok_ir, int B, int H, int W, int C, int nh, int nw,
                                   int n_pad, void* stream);
/* icaf_layernorm over fp32 tokens; y fp16 (the fp32 LayerNorm rounded once, as the Linear after it casts it). */
int icaf_layernorm_f32(const float* x0, const float* x1, const float* g0, const float* b0, const float* g1, const float* b1, void* y0, void* y1,
                       int64_t rows, int C, float eps, void* stream);
/* icaf_layernorm_bwd with fp32 x and dx and fp16 dy.  workspace: icaf_train_workspace_bytes(C) + 2 rows floats. */
int icaf_layernorm_bwd_f32(const float* x, const void* dy, const float* gamma, float* dx, float* dgamma, float* dbeta, int64_t rows, int C,
                           float eps, float grad_scale, int accumulate, float* workspace, size_t workspace_bytes, void* stream);
/* out = a[0] * x (+ b[0] * y) with x fp32, y fp16 (or NULL), n % 8 == 0: two rounded products and a rounded sum, torch's fp32
 * `a * x + b * y` bit for bit.  out is fp16 (rounded once) when out_f16, else fp32. */
int icaf_axpby_f32(const float* x, const void* y, const float* a, const float* b, void* out, int out_f16, int64_t n, void* stream);
/* icaf_dot with x fp32 and y fp16 (y_f16) or fp32. */
int icaf_dot_f32(const float* x, const void* y, int y_f16, int64_t rows, int C, float* out, float scale, int accumulate, float* workspace,
                 size_t workspace_bytes, void* stream);
/* icaf_colsum of a dense fp32 (rows, C) matrix; workspace: 64 * C floats. */
int icaf_colsum_f32(const float* x, int64_t rows, int C, float* out, float scale, int accumulate, float* workspace, size_t workspace_bytes,
                    void* stream);

/* ---------------------------------------------------------------------------------------------
 * Training augmentation of RGB/IR pairs: LoadMultiModalImagesAndLabels.__getitem__ (utils/datasets.py:948-1024) with
 * augment=True -- mosaic (load_mosaic_RGB_IR :1208-1309, resize of load_image_rgb_ir :1097-1125), affine warp
 * (random_perspective_rgb_ir :1535-1630, perspective = 0), HSV jitter (augment_hsv :1129-1141), flipud / fliplr and
 * BGR->RGB + HWC->CHW -- for a batch, one launch, bit-exact against the cv2 pipeline.  The random draws, the warp tables
 * and the LUTs are the host's (icafusion_b200/augment.py); the canvas is never materialised: every output pixel is
 * evaluated through warp -> canvas tile -> cv2.resize taps of the decoded frame -> HSV LUTs.
 * ------------------------------------------------------------------------------------------- */
typedef struct {
  const void* rgb; const void* ir;  /* device uint8 (H0, W0, 3) BGR frames of this tile's image                       */
  int H0, W0;                       /* decoded size                                                                    */
  int h, w;                         /* load_image size (int(h0 r), int(w0 r)); == (H0, W0): no resize                  */
  int x1a, y1a, x2a, y2a;           /* canvas rectangle [x1a, x2a) x [y1a, y2a) ...                                     */
  int x1b, y1b;                     /* ... filled from the resized image starting at (x1b, y1b)                         */
  int xtab, ytab;                   /* first row (int4 units) of the cv2.resize taps in the taps region: [w] / [h] rows */
} icaf_aug_tile;

typedef struct {
  icaf_aug_tile tile[4];
  int ntiles;                       /* 1..4; a later tile covers an earlier one where they overlap (placement order)   */
  int canvas;                       /* side of the square canvas: 2s with the mosaic, s without                         */
  int warp;                         /* 1: output = warpAffine(canvas) via the sample's tables; 0: output = canvas      */
  int flipud, fliplr;
  int reserved;
  unsigned char lut[2][3][256];     /* augment_hsv LUTs: [rgb, ir][hue, sat, val]                                        */
} icaf_aug_sample;

/* Bytes of the parameter block for B samples at output size s with n_taps resize-tap rows.  Layout (16-byte aligned regions):
 *   icaf_aug_sample [B]                       at 0
 *   int32 warp [B][4][s]                      at align16(B * sizeof(icaf_aug_sample)): per sample adelta[x], bdelta[x]
 *                                             (cvRound(M'0 x 1024), cvRound(M'3 x 1024)) and X0[y], Y0[y]
 *                                             (cvRound((M'1 y + M'2) 1024) + 16, likewise) of the inverted matrix M'
 *   int32 taps [n_taps][4]                    after the warp tables: {i0, i1, w0, w1} rows as for icaf_letterbox
 * 0 for a bad argument. */
size_t icaf_augment_params_bytes(int B, int s, int n_taps);

/* params: device block laid out as above (16-byte aligned); rgb_out / ir_out: uint8 (B, 3, s, s) RGB planar. */
int icaf_augment(const void* params, size_t params_bytes, int B, int s, int n_taps, void* rgb_out, void* ir_out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * The optimiser step of train.py:347-352 on the device (csrc/optim.cu): GradScaler.unscale_ with the inf check, nesterov
 * SGD or Adam skipped on the device when the check fired, GradScaler.update and ModelEMA.update -- bit-identical to torch's
 * foreach implementations, with no read-back, so the step can be captured into a CUDA graph.  All tensors are dense fp32.
 * ------------------------------------------------------------------------------------------- */
#define ICAF_OPTIM_CHUNK 2048  /* elements per chunk of a tensor table                                               */
#define ICAF_OPTIM_HYPER 8     /* doubles per parameter group in `hyper`: {lr, momentum | beta1, weight_decay, beta2,
                                  eps, unused x 3}, read from the device at run time                                  */
typedef struct {
  void* p;         /* updated in place: the parameter (ema: the EMA model's entry)                                    */
  void* g;         /* the gradient (ema: the model's entry); unscale updates it in place                             */
  void* m;         /* SGD momentum_buffer / Adam exp_avg                                                              */
  void* v;         /* Adam exp_avg_sq                                                                                 */
  void* step;      /* Adam: the tensor's fp32 step count                                                             */
  int64_t numel;
  int64_t chunk0;  /* first chunk of this tensor: chunk0 of the previous entry + ceil(its numel / ICAF_OPTIM_CHUNK)    */
  int64_t reserved;  /* 64-byte entries: every entry of a table starts a 16-byte aligned sub-table                  */
} icaf_optim_tensor;

/* Bytes of a device table of n_tensors entries (0 for n_tensors < 1).  A launch walks the n_tensors entries at `table`,
 * which may start anywhere in a larger table, and the n_chunks chunks they cover. */
size_t icaf_optim_table_bytes(int n_tensors);
/* GradScaler.unscale_: g *= float(1.0 / double(*scale)) over every entry; *found_inf = 1 when any element is non-finite. */
int icaf_amp_unscale(const void* table, size_t table_bytes, int n_tensors, int64_t n_chunks, const float* scale, float* found_inf,
                     void* stream);
/* torch.optim.SGD(nesterov=True, dampening=0) over one parameter group, skipped when *found_inf != 0:
 * d = g + wd p (wd != 0); buf = buf m + d; d = d + m buf; p = p - lr d, with {lr, m, wd} = hyper[group]. */
int icaf_sgd_step(const void* table, size_t table_bytes, int n_tensors, int64_t n_chunks, const double* hyper, int group, int n_groups,
                  const float* found_inf, void* stream);
/* torch.optim.Adam (amsgrad=False, L2 weight decay) over one parameter group, skipped when *found_inf != 0.  At each tensor's
 * step s = *step + 1 it reads bias_corr[group][s] = {1 - beta1**s, (1 - beta2**s)**0.5} (doubles, rows 0 .. bc_steps - 1, as
 * torch computes them on the host), then adds 1 to every step count. */
int icaf_adam_step(const void* table, size_t table_bytes, int n_tensors, int64_t n_chunks, const double* hyper, int group, int n_groups,
                   const double* bias_corr, int bc_steps, const float* found_inf, void* stream);
/* torch._amp_update_scale_ on GradScaler's scale (fp32) and growth tracker (int32), then *found_inf = 0. */
int icaf_amp_update_scale(float* scale, int* growth_tracker, float* found_inf, double growth_factor, double backoff_factor,
                          int growth_interval, void* stream);
/* ModelEMA.update with d = *decay (device double): p = p float(d), then p = p + float(1 - d) g. */
int icaf_ema_update(const void* table, size_t table_bytes, int n_tensors, int64_t n_chunks, const double* decay, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ICAF_B200_H */
