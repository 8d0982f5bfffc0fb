/* yolov3_b200 — C ABI of the Hopper-native (sm_90a) YOLOv3 detection hot path.
 *
 * The reference (ultralytics/yolov3, pure Python) has no FFI: its seams for this path are Python call signatures
 * (SURVEY.md §8b).  This header is the drop-in boundary a binding for those seams attaches to; each entry point cites
 * the reference interface it replaces.  Conventions:
 *   - plain pointers and sizes only; all data pointers are DEVICE pointers owned by the caller (PyTorch);
 *   - every function returns Y3_OK (0) or a negative Y3_ERR_*; text via y3_last_error(); nothing throws;
 *   - nothing allocates device memory, nothing synchronises the stream (the only host sync is y3_model_create's
 *     one-off capability probe); all launches go to the caller's stream and are CUDA-graph capturable;
 *   - re-entrant: no global mutable state besides the last-error string (thread-local) and a mutex-guarded
 *     per-process driver-entry-point cache.  A y3_model is immutable after create.
 * Activation layout ("padded NHWC"): bf16 [n, h+2, w+2, ld] with a one-pixel all-zero halo; a tensor may be a channel
 * slice [coff, coff+c) of a wider buffer (zero-copy Concat, models/common.py:424-428).
 */
#ifndef YOLOV3_B200_H
#define YOLOV3_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define Y3_OK 0
#define Y3_ERR_BAD_ARG (-1)     /* shape/alignment/enum not supported by this path */
#define Y3_ERR_CUDA (-2)        /* a CUDA runtime/driver call failed (message in y3_last_error) */
#define Y3_ERR_UNSUPPORTED (-3) /* device is not sm_90 (no fallback path exists by design) */

#define Y3_ACT_NONE 0
#define Y3_ACT_SILU 1

typedef void* y3_stream_t; /* cudaStream_t */

int y3_version(void);
/* Copies the calling thread's last error text into buf (NUL-terminated); returns its length. */
int y3_last_error(char* buf, size_t n);
/* Y3_OK iff the current CUDA device is compute capability 9.0. */
int y3_device_check(void);
/* sizeof() of the ABI structs, for bindings to verify their mirror definitions:
 * 0 y3_conv_desc, 1 y3_first_desc, 2 y3_pool_desc, 3 y3_detect_level, 4 y3_decode_desc, 5 y3_op, 6 y3_nms_params,
 * 7 y3_loss_desc, 8 y3_bn_act_desc, 9 y3_bn_bwd_desc, 10 y3_wgrad_desc, 11 y3_pack_item, 12 y3_letterbox_desc,
 * 13 y3_amax_desc, 14 y3_resize_item, 15 y3_augment_desc, 16 y3_jpeg_geom, 17 y3_jpeg_info, 18 y3_jpeg_desc,
 * 19 y3_halo_item. */
int64_t y3_abi_sizeof(int32_t which);
/* Programmatic dependent launch between consecutive kernels of a stream (on by default; env Y3_PDL=0 or on=0 turns it off).
 * Results are identical either way — only the launch boundaries overlap.  Returns the previous setting.  A tuning switch with
 * no counterpart in the reference. */
int y3_set_pdl(int32_t on);

/* ---------------------------------------------------------------------------------------------------------------
 * Conv + folded-BN + SiLU (+ residual add, + nearest-2x upsample, + concat-offset store, or fp32 head store).
 * Replaces Conv.forward_fuse (models/common.py:77-81) after BaseModel.fuse (models/yolo.py:163-172), the shortcut add
 * of Bottleneck.forward (common.py:163-165), nn.Upsample+Concat (models/yolov3.yaml:43-44,51-52) and Detect.m[i]
 * (models/yolo.py:96-98).  wgmma implicit GEMM; c_in % 16 == 0, c_out_pad = c_out rounded up to the tile N.
 * ksize 1|3 with stride 1, or ksize 3 with stride 2 (h, w even); pad = ksize/2.
 */
typedef struct y3_conv_desc {
  int32_t n, h, w;       /* batch, UNPADDED input height/width */
  int32_t c_in, c_out;   /* logical channels */
  int32_t ksize, stride;
  int32_t act;           /* Y3_ACT_* */
  const void* in;        /* padded NHWC bf16 [n, h+2, w+2, in_ld]; the conv reads channels [in_coff, in_coff+c_in) */
  int32_t in_ld, in_coff;
  const void* weight;    /* bf16 [c_out_pad, ksize*ksize*c_in], k index = (kh*ksize+kw)*c_in + c, BN folded */
  const float* bias;     /* fp32 [c_out_pad] */
  void* out;             /* padded NHWC bf16 [n, ho*u+2, wo*u+2, out_ld], u = 1+upsample; written at [out_coff, +c_out) */
  int32_t out_ld, out_coff;
  const void* res;       /* optional residual (NULL = none): padded NHWC bf16 with the conv-output geometry */
  int32_t res_ld, res_coff;
  int32_t upsample;      /* 1: replicate every output pixel 2x2 into `out` */
  float* out_f32;        /* Detect heads (NULL = off): fp32 pixel-major [n*ho*wo, out_f32_ld] instead of `out`;
                            columns [0, c_out_pad) of every row are written (pad columns = 0) */
  int32_t out_f32_ld;    /* >= c_out_pad, multiple of 4 */
  int32_t* err;          /* optional device int32 error word written by the in-kernel watchdog */
  int32_t weight_layout; /* Y3_W_*: how `weight` is packed (0 = tap-major as documented above) */
  /* FP8 inference (all zero = bf16 as above).  An e4m3 tensor holds code q for the value q * s of its per-tensor scale s. */
  int32_t in_fmt;        /* Y3_FMT_*: format of `in` and of `weight` (e4m3: c_in % 32 == 0, in_ld % 16 == 0) */
  int32_t out_fmt;       /* Y3_FMT_*: format of `out` and of `res` (ignored with out_f32); e4m3: out_ld, out_coff,
                            res_ld, res_coff % 16 == 0 */
  const float* dq;       /* e4m3 input: fp32 [c_out_pad], dq[n] = s_in * s_w[n]; y = act(acc * dq[n] + bias[n]) */
  float res_scale;       /* e4m3 output with res: > 0, the residual adds res_scale * r (the residual's own scale) */
  float out_inv_scale;   /* e4m3 output: stores sat_e4m3(y * out_inv_scale) */
} y3_conv_desc;
#define Y3_FMT_BF16 0
#define Y3_FMT_E4M3 1   /* float8_e4m3fn: max 448, stored round-to-nearest-even with saturation */
int y3_conv_bn_act_fwd(const y3_conv_desc* d, y3_stream_t stream);
/* Input gradient of a STRIDE-2 3x3 conv (training; autograd of Conv.forward, models/common.py:71-75) as four parity-class
 * convolutions of the un-stuffed output gradient: `in` = dy, padded NHWC [n, h+2, w+2, in_ld] on the conv's OUTPUT grid (h, w =
 * output size), `weight` = the dgrad pack [c_in_pad rows = dx channels, 9 * c_dy] (taps flipped, y3_pack_dgrad_batched), `out` = dx, padded
 * [n, 2h+2, 2w+2, out_ld]; `res` (optional, dx geometry) is added — pass `out` itself to accumulate.  ksize = 3, stride = 1 and
 * act = Y3_ACT_NONE in the descriptor (it describes the transposed conv on dy's grid). */
int y3_conv_dgrad_s2(const y3_conv_desc* d, y3_stream_t stream);
/* Weight layouts.  Y3_W_XPAIR (stride-2 3x3 with c_in in {16,32}, in_ld == c_in, in_coff == 0): bf16
 * [c_out_pad, 3, 2, 2, c_in] with element (kh, sp, par, c) = W[kh][2*sp+par][c] and zeros for the phantom column
 * 2*sp+par == 3 — two horizontally adjacent taps form one 2*c_in-channel GEMM k-block, which turns the 64-byte rows of
 * the thin first stride-2 layer (models/yolov3.yaml:19) into full 128-byte TMA rows.  y3_conv_weight_layout returns the
 * layout the kernel prefers for a descriptor's geometry (weight/bias/out pointers are not inspected); packing the
 * weights that way and setting weight_layout is optional — Y3_W_TAPS always works. */
#define Y3_W_TAPS 0
#define Y3_W_XPAIR 1
int y3_conv_weight_layout(const y3_conv_desc* d);
/* The kernel variant y3_conv_bn_act_fwd would launch for a descriptor (host-only query: pointers are checked for
 * alignment but never dereferenced, no tensor map is encoded, no GPU needed): tile shape, halo reuse (one A box per
 * filter row), weights resident in shared memory, x-paired stride-2 weights, tile counts and grid.  For tests and for
 * reading the selection heuristics off a model. */
typedef struct y3_conv_plan_info {
  int32_t block_n, block_k, halo, resident_weights, xpair;
  int32_t m_tiles, n_tiles, k_blocks, grid;
} y3_conv_plan_info;
int y3_conv_plan(const y3_conv_desc* d, y3_conv_plan_info* out);
/* Tile N the kernel will use for c_out (weights/bias must be padded to a multiple of it). */
int y3_conv_cout_pad(int32_t c_out);

/* First layer: 3x3 stride-1 pad-1 conv on the NCHW image (c_in = 3), folded BN + SiLU, writing padded NHWC bf16.
 * Replaces Conv.forward_fuse for layer 0 together with the caller-side `im.float() / 255` (detect.py:187-191,
 * val.py:358-359) and the NCHW->NHWC/bf16 conversion.  c_out in {16, 32}.
 * weight: fp32 [27, c_out] (k = (c*3+kh)*3+kw), bias fp32 [c_out]. */
#define Y3_IN_F32 0
#define Y3_IN_U8 1
typedef struct y3_first_desc {
  const void* in;        /* [n, 3, h, w] fp32 or uint8 */
  int32_t in_dtype;      /* Y3_IN_* */
  float in_div;          /* > 0: pixel = value / in_div (255 for uint8 images); 0: use as is */
  int32_t n, h, w;
  const float* weight;
  const float* bias;
  int32_t c_out;
  void* out;             /* padded NHWC bf16 [n, h+2, w+2, out_ld] */
  int32_t out_ld, out_coff;
} y3_first_desc;
int y3_conv_first_fwd(const y3_first_desc* d, y3_stream_t stream);

/* Max-pool on padded NHWC bf16 (nn.MaxPool2d of yolov3-tiny.yaml; SPP pools, models/common.py:279,290).
 * Window of output (y,x) = input rows [y*stride+off, +k) x cols [x*stride+off, +k); out-of-image elements are ignored
 * (-inf padding) unless oob_zero, where they count as 0 (ZeroPad2d followed by MaxPool2d). */
typedef struct y3_pool_desc {
  const void* in;
  int32_t in_ld, in_coff;
  void* out;
  int32_t out_ld, out_coff;
  int32_t n, h, w, c;    /* input size (unpadded), channels (multiple of 8) */
  int32_t ho, wo;
  int32_t k, stride, off, oob_zero;
  int32_t fmt;           /* Y3_FMT_* of `in` and `out` (0 = bf16); the e4m3 pool is exact and keeps the input's scale;
                            e4m3: c, ld and coff % 16 == 0.  The training entry points below take bf16 only */
} y3_pool_desc;
int y3_maxpool_fwd(const y3_pool_desc* d, y3_stream_t stream);
/* Training mode (SPP, models/common.py:281-290, under autograd): the forward also records idx[n, ho, wo, c] (uint8) =
 * dy*k + dx of the first maximum in row-major window order — the element torch.nn.MaxPool2d back-propagates to — and the
 * backward gathers dIn[p] (+)= sum of dOut over the windows whose argmax is p (no atomics).  For y3_maxpool_bwd the
 * descriptor's `in` is dOut (geometry ho x wo), `out` is dIn (geometry h x w); oob_zero windows are not supported. */
int y3_maxpool_train_fwd(const y3_pool_desc* d, uint8_t* idx, y3_stream_t stream);
int y3_maxpool_bwd(const y3_pool_desc* d, const uint8_t* idx, int32_t accumulate, y3_stream_t stream);

/* FP8 calibration: amax = max(amax, max |x|) over the n*h*w interior pixels of a padded NHWC slice [coff, coff+c) of
 * format fmt (Y3_FMT_*), in stored units (e4m3: codes); c, ld and coff % 8 == 0 (bf16) or % 16 == 0 (e4m3).
 * Order-independent (an atomic max on the float bits): deterministic. */
int y3_amax_nhwc(const void* x, int32_t fmt, int32_t ld, int32_t coff, int32_t n, int32_t h, int32_t w, int32_t c,
                 float* amax, y3_stream_t stream);

/* Layout helpers (tests / feeding intermediate tensors): NCHW fp32 <-> padded NHWC bf16 channel slice. */
int y3_nchw_to_padded_nhwc(const float* src, int32_t n, int32_t c, int32_t h, int32_t w, void* dst, int32_t dst_ld,
                           int32_t dst_coff, y3_stream_t stream);
int y3_padded_nhwc_to_nchw(const void* src, int32_t src_ld, int32_t src_coff, int32_t n, int32_t c, int32_t h,
                           int32_t w, float* dst, y3_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Detect decode.  Replaces the eval branch of Detect.forward and _make_grid (models/yolo.py:100-123):
 * z[b, off_l + (a*ny + y)*nx + x, :] = (xy: (2*sig + grid - 0.5)*stride, wh: (2*sig)^2 * anchor_px, rest: sig).
 */
#define Y3_MAX_LEVELS 5
#define Y3_MAX_ANCHORS 6
typedef struct y3_detect_level {
  const float* raw;                 /* y3_detect_decode_fwd: fp32 [bs, na, ny, nx, no] logits (the reference's x[i]) */
  const float* head;                /* y3_detect_head_decode_fwd: head-conv output, fp32 [bs*ny*nx, head_ld],
                                       column a*no + k (y3_conv_desc.out_f32) */
  int32_t head_ld;
  float* raw_out;                   /* y3_detect_head_decode_fwd: optional fp32 [bs, na, ny, nx, no] (models/yolo.py:98) */
  int32_t ny, nx;
  float stride;                     /* Detect.stride[i] */
  float anchor_w[Y3_MAX_ANCHORS];   /* anchors[i] * stride[i], pixels (anchor_grid, models/yolo.py:122) */
  float anchor_h[Y3_MAX_ANCHORS];
} y3_detect_level;
int y3_detect_decode_fwd(const y3_detect_level* levels, int32_t nl, int32_t bs, int32_t na, int32_t no, float* z,
                         y3_stream_t stream);
typedef struct y3_decode_desc {
  y3_detect_level levels[Y3_MAX_LEVELS];
  int32_t nl, bs, na, no;
  float* z;                         /* [bs, sum_l na*ny*nx, no] or NULL (training: logits only) */
} y3_decode_desc;
/* Fused head transpose + decode used by the graph executor: one pass from the head convs' pixel-major fp32 output to
 * z and to the reference-layout logits.  no = nc + 5 may be 5..Y3_MAX_DECODE_NO (nc <= 1024, the NMS limit): rows of up
 * to 256 elements go through register-array kernels that walk 4 z rows per warp, wider rows through a kernel that walks
 * one z row per warp. */
#define Y3_MAX_DECODE_NO 1029
int y3_detect_head_decode_fwd(const y3_decode_desc* d, y3_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Batched NMS.  Replaces non_max_suppression (utils/general.py:630-750) incl. torchvision.ops.nms (:733) for nm=0;
 * autolabel priors (labels=, :689-695) are appended to `pred` by the caller as obj = 1 / one-hot rows.  Sync-free: results are padded device arrays plus per-image counts.
 *   pred      fp32 [bs, n_rows, 5+nc]  (xywh, obj, cls...)
 *   out       fp32 [bs, max_det, 6]    rows (x1,y1,x2,y2,conf,cls) sorted by conf desc, zero beyond out_count[b]
 *   out_src   int32 [bs, max_det, 2]   optional (pred row, class) of every kept detection
 *   out_count int32 [bs]
 *   overflow  int32 [bs]               optional; non-zero = candidates found (> cap): rerun with a larger capacity
 * The wall-clock time_limit break of the reference (:675,746-748) is intentionally not reproduced.
 */
typedef struct y3_nms_params {
  int32_t bs, n_rows, nc;
  float conf_thres, iou_thres;      /* must lie in [0,1] (the reference asserts, :658-659) */
  int32_t multi_label, agnostic;
  int32_t max_det;                  /* :734 */
  int32_t max_nms;                  /* 30000 (:674); <= 32768 */
  float max_wh;                     /* 7680 (:673) */
  int32_t cap;                      /* per-image candidate capacity, power of two >= 4096 */
  const int32_t* classes;           /* HOST array of class ids to keep (:717-718), or NULL */
  int32_t n_classes;
} y3_nms_params;
int32_t y3_nms_default_capacity(int32_t n_rows, int32_t nc, int32_t multi_label);
int64_t y3_nms_workspace_bytes(int32_t bs, int32_t cap);
int y3_nms_batched(const float* pred, const y3_nms_params* params, void* workspace, int64_t workspace_bytes, float* out,
                   int32_t* out_src, int32_t* out_count, int32_t* overflow, y3_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Pairwise IoU.  Replaces box_iou (ultralytics; re-exported utils/metrics.py:10, used val.py:176): xyxy boxes,
 * out[i*m + j] = inter / (area1 + area2 - inter + eps).  box1 [n,4], box2 [m,4] fp32, 16-byte aligned. */
int y3_box_iou(const float* box1, int32_t n, const float* box2, int32_t m, float eps, float* out, y3_stream_t stream);
/* scale_boxes + clip_boxes (utils/general.py:613-626; callers detect.py:218, val.py:381-385): in place on columns 0..3
 * (xyxy) of n rows of `row_stride` floats: v = clamp((v - pad) / gain, 0, max) with pad_x/max_x for x1,x2 and pad_y/max_y
 * for y1,y2; gain = 1, pad = 0 gives clip_boxes. */
int y3_scale_boxes(float* boxes, int64_t n, int32_t row_stride, float pad_x, float pad_y, float gain, float max_x,
                   float max_y, y3_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Training loss, forward + backward.  Replaces ComputeLoss.__call__ / build_targets (utils/loss.py:131-244) with
 * bbox_iou(CIoU) and BCEWithLogitsLoss(pos_weight), FocalLoss around both BCE terms when fl_gamma > 0
 * (loss.py:31-63, 117-119) and the autobalance update of the objectness balance (loss.py:171-175); gr = 1.
 *   p[l]     fp32 [bs, na, ny_l, nx_l, nc+5] raw logits (train-mode Detect output, models/yolo.py:110)
 *   grad[l]  same shape (or NULL): receives d(out[0])/dp[l] * grad_scale
 *   targets  fp32 [nt, 6] = (image, class, x, y, w, h) normalised (collate_fn, utils/dataloaders.py:825-830)
 *   out      fp32 [4] = ((lbox+lobj+lcls)*bs, lbox, lobj, lcls)   (loss.py:181)
 */
typedef struct y3_loss_desc {
  int32_t nl, bs, na, nc;
  const float* p[Y3_MAX_LEVELS];
  float* grad[Y3_MAX_LEVELS];
  int32_t ny[Y3_MAX_LEVELS], nx[Y3_MAX_LEVELS];
  float anchors[Y3_MAX_LEVELS][Y3_MAX_ANCHORS][2]; /* Detect.anchors, grid units */
  const float* targets;
  int32_t nt;
  float box, obj, cls;       /* hyp gains (already rescaled as train.py:326-329) */
  float cls_pw, obj_pw;      /* BCE pos_weight */
  float anchor_t;
  float cp, cn;              /* smooth_bce(label_smoothing) targets */
  float balance[Y3_MAX_LEVELS];  /* objectness balance (autobalance = 0) */
  float grad_scale;          /* upstream gradient of out[0] (1 for loss.backward()) */
  double fl_gamma;           /* focal loss gamma: 0 = plain BCE, else finite and > 0 */
  double fl_alpha;           /* focal loss alpha (0.25) */
  int32_t autobalance;       /* 1: the balance is read from bal_state, updated there and normalised by bal_state[ssi] */
  int32_t ssi;               /* index of the stride-16 level in bal_state */
  int32_t n_balance;         /* entries of bal_state (nl <= n_balance <= Y3_MAX_LEVELS) */
  double* bal_state;         /* device fp64 [n_balance], autobalance = 1 only; carries from call to call */
} y3_loss_desc;
int64_t y3_loss_workspace_bytes(const y3_loss_desc* d);
int y3_loss_fwd_bwd(const y3_loss_desc* d, void* workspace, int64_t workspace_bytes, float* out, y3_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Training-mode Conv block (models/common.py:71-75 with BatchNorm2d in train mode) and its backward.  The convolution
 * (forward; dgrad = convolution with the transposed, tap-flipped weights) is y3_conv_bn_act_fwd with zero bias and
 * Y3_ACT_NONE; these entry points are the bandwidth-bound parts around it.  All activations: padded NHWC bf16 slices.
 */
/* Two-stage, atomic-free (bit-reproducible) reductions: a first-stage kernel writes one partial row per block into a
 * caller-owned workspace [y3_bn_partial_blocks(n, h, w, c)][width], a fixed-order second stage adds the rows. */
int32_t y3_bn_partial_blocks(int32_t n, int32_t h, int32_t w, int32_t c);  /* c = 0: one unit per image row (head gradient) */
/* per-channel sum and sum of squares of the conv output y over its n*h*w interior pixels:
 * partial[blocks][2][c] = (sum | sumsq).  c: power of two in [8, 2048]. */
int y3_bn_stats(const void* y, int32_t ld, int32_t coff, int32_t c, int32_t n, int32_t h, int32_t w, float* partial,
                y3_stream_t stream);
/* out[j] (+)= sum_b partial[b][j] for j < width, rows added in index order (SyncBatchNorm: sums before the all-reduce) */
int y3_colreduce_f32(const float* partial, int32_t nblk, int32_t width, float* out, int32_t accumulate, y3_stream_t stream);
/* batch statistics (given as nblk partial rows [2][c]; nblk = 1: already reduced) -> scale = gamma*rstd, shift = beta -
 * mean*scale, saved mean/rstd; running stats updated in place with the unbiased variance when non-NULL (nn.BatchNorm2d
 * semantics).  count = pixels behind the sums (n*h*w, times the world size under SyncBatchNorm). */
int y3_bn_finalize(const float* partial, int32_t nblk, const float* gamma, const float* beta, int32_t c, float count,
                   float eps, float momentum, float* scale, float* shift, float* mean, float* rstd, float* running_mean,
                   float* running_var, y3_stream_t stream);
typedef struct y3_bn_act_desc {
  const void* y;   int32_t y_ld, y_coff;       /* conv output (pre-BN) */
  const void* res; int32_t res_ld, res_coff;   /* optional residual added after the activation (Bottleneck shortcut) */
  void* out;       int32_t out_ld, out_coff;   /* a = SiLU(y*scale+shift) (+res); [n, h*u+2, w*u+2, out_ld], u = 1+upsample */
  const float* scale; const float* shift;
  int32_t n, h, w, c, upsample;
} y3_bn_act_desc;
int y3_bn_act_fwd(const y3_bn_act_desc* d, y3_stream_t stream);
typedef struct y3_bn_bwd_desc {
  const void* y;  int32_t y_ld, y_coff;        /* saved conv output */
  const void* da; int32_t da_ld, da_coff;      /* gradient w.r.t. the block output (2x geometry when upsample) */
  void* dy;       int32_t dy_ld, dy_coff;      /* gradient w.r.t. the conv output (input of dgrad / wgrad) */
  const float* scale; const float* shift; const float* mean; const float* rstd;
  float* sums;       /* [2][c] = (sum dz | sum dz*xhat): phase 0/1 out, phase 2 in (the all-reduced sums) */
  float* partial;    /* workspace [y3_bn_partial_blocks(n, h, w, c)][2][c] of the reduction phase (phases 0, 1) */
  float* dbeta_acc;  /* optional [c]: += sum dz      (the bn.bias gradient, accumulated like autograd does) */
  float* dgamma_acc; /* optional [c]: += sum dz*xhat (the bn.weight gradient) */
  int32_t n, h, w, c, upsample;
  int32_t phase;   /* 0: sums then apply (single GPU); 1: sums only; 2: apply only — SyncBatchNorm (train.py:270-272) puts
                      an all-reduce of the two sums between 1 and 2 */
  float count;     /* pixels behind the sums used by the apply phase (all ranks); 0 = this rank's n*h*w */
} y3_bn_bwd_desc;
int y3_bn_act_bwd(const y3_bn_bwd_desc* d, y3_stream_t stream);
/* Weight packs of the training engine: the fp32 masters live in ONE flat buffer with every conv weight stored
 * [co][kh][kw][ci] (channels_last strides of the [co,ci,k,k] parameter == the forward pack's order), so
 *   y3_f32_to_bf16        converts the whole buffer once per step (forward packs are views of the copy), and
 *   y3_pack_dgrad_batched transposes every layer of a device-resident table into its dgrad pack in one launch. */
int y3_f32_to_bf16(const float* src, void* dst, int64_t n, y3_stream_t stream);
typedef struct y3_pack_item {
  int64_t src_off;   /* element offset of this layer's [co_rows][k*k][ci] weights inside the bf16 flat copy */
  void* dst;         /* dgrad pack, bf16 [ci_pad][k*k][dst_co] (rows >= ci stay zero) */
  int32_t co_rows;   /* rows present in the source (c_out, or the padded 256 of a Detect head) */
  int32_t ci, k;
  int32_t dst_co;    /* row pitch of the pack = c_out the dgrad conv reduces over */
  int32_t tile_begin;/* first 32x32 transpose tile of this layer: k*k * ceil(co_rows/32) * ceil(ci/32) tiles each, consecutive */
  int32_t reserved;
} y3_pack_item;
int y3_pack_dgrad_batched(const y3_pack_item* items_dev, int32_t n_items, const void* wbf, int32_t total_tiles,
                          y3_stream_t stream);
/* Detect-head gradient: g = dL/draw fp32 [n, na, ny, nx, no] (ComputeLoss output) -> dy bf16 padded NHWC channel a*no+o
 * (the head conv's output order; channels >= na*no zeroed) and partial[y3_bn_partial_blocks(n, ny, 0, 0)][W256] column sums
 * (bias gradient = y3_colreduce_f32 over them), W = dy_ld - dy_coff >= na*no, W256 = W rounded up to a multiple of 256
 * (256 for every head of at most 80 classes and 3 anchors). */
int y3_head_grad_pack(const float* g, int32_t n, int32_t na, int32_t ny, int32_t nx, int32_t no, void* dy, int32_t dy_ld,
                      int32_t dy_coff, float* partial, y3_stream_t stream);
/* dW[co, kh*k+kw, ci] += sum_p dy[p, co] * x[p + shift(kh,kw), ci] on the stride-1 padded grid [n, h+2, w+2], with the
 * wgmma kernel.  dw is fp32 [co, k*k, ci]: the channels_last strides of a [co, ci, k, k] tensor, i.e. the training engine's
 * flat gradient buffer (the gradient IS the parameter's .grad view, no permute); each (co, tap) row is contiguous in ci,
 * so the kernel adds with 8-byte vector reductions.  co, ci multiples of 8; dy and x 16-byte aligned, dw 8-byte aligned. */
typedef struct y3_wgrad_desc {
  const void* dy; int32_t dy_ld, dy_coff;
  const void* x;  int32_t x_ld, x_coff;
  float* dw;
  int32_t co, ci, ksize, n, h, w;
  int32_t accumulate;     /* 1: dw holds earlier contributions that must be kept (always reduce, never plain-store) */
  int32_t deterministic;  /* 1: no split over pixels — one CTA per dW tile, bit-reproducible, slower on the early layers */
  int32_t stride;         /* 0/1: dy on x's grid.  2: a stride-2 conv — dy is the conv's own [n, h/2+2, w/2+2, dy_ld]
                             output-grid gradient, x is read through its row/column parity view; 3x3 and even h, w only */
} y3_wgrad_desc;
int y3_conv_wgrad(const y3_wgrad_desc* d, y3_stream_t stream);
/* dst (+)= src over the interior pixels of two padded NHWC bf16 slices of equal [n,h,w,c] (gradient fan-in) */
int y3_add_nhwc(const void* src, int32_t src_ld, int32_t src_coff, void* dst, int32_t dst_ld, int32_t dst_coff, int32_t n,
                int32_t h, int32_t w, int32_t c, int32_t accumulate, y3_stream_t stream);
/* 3x3 pad-1 im2col of the [n,3,h,w] image (Y3_IN_F32 | Y3_IN_U8, optional /in_div) into 32 bf16 channels of a padded
 * NHWC buffer, column (c*3+kh)*3+kw; lets training run layer 0 as a 1x1 conv with the generic kernels */
int y3_im2col_first(const void* in, int32_t in_dtype, float in_div, int32_t n, int32_t h, int32_t w, void* out,
                    int32_t out_ld, int32_t out_coff, y3_stream_t stream);
/* y3_im2col_first of the [n,3,src_h,src_w] image rescaled to h x w: the multi-scale step of the reference's training loop,
 * imgs.float() / 255 then F.interpolate(imgs, (h, w), mode="bilinear", align_corners=False), fused into layer 0's im2col.
 * The arithmetic restates torch's CUDA upsample_bilinear2d with no scale factors given: scale = float(src) / dst, source
 * index max(scale * (d + 0.5) - 0.5, 0), the +1 neighbour only inside the image.  Y3_IN_U8 with in_div > 0 multiplies
 * each source byte by the fp32 reciprocal of in_div first, as torch's division by a CPU scalar does. */
int y3_im2col_first_resize(const void* in, int32_t in_dtype, float in_div, int32_t n, int32_t src_h, int32_t src_w,
                           int32_t h, int32_t w, void* out, int32_t out_ld, int32_t out_coff, y3_stream_t stream);
/* Zeroes, for every item of a device-resident table, the one-pixel halo of a bf16 padded NHWC buffer [n, h+2, w+2, ld] and
 * channels [c_lo, ld) of its interior (c_lo = ld: none).  Training engines of different batch shapes share one activation
 * arena; an engine that takes the arena over from another restores with this one launch the zeros its kernels read. */
typedef struct y3_halo_item {
  void* p;
  int32_t n, h, w, ld;
  int32_t c_lo;
  int32_t reserved;
} y3_halo_item;
int y3_zero_halo_batched(const y3_halo_item* items_dev, int32_t n_items, y3_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Image pre-processing on the device (SURVEY §8(f) row f1): letterbox (utils/augmentations.py:104-134: cv2.resize
 * INTER_LINEAR to new_w x new_h, then a constant border) fused with the HWC->CHW / BGR->RGB step of the loaders
 * (utils/dataloaders.py:308-310).  src: uint8 [src_h, src_w, 3] with row pitch src_pitch bytes (a decoded BGR frame);
 * dst: uint8 [out_h, out_w, 3] (out_chw = 0) or [3, out_h, out_w] (out_chw = 1), channel order reversed when swap_rb.
 * The resized image sits at (top, left); everything else is pad[] (given in SOURCE channel order, 114 in the reference).
 * The resize reproduces OpenCV's 8-bit INTER_LINEAR bit for bit (incl. its 2x-shrink INTER_AREA shortcut and the plain copy
 * when no resize is needed).  The geometry (new size, offsets) is the caller's: letterbox's scalar arithmetic stays on the host. */
typedef struct y3_letterbox_desc {
  const void* src; int32_t src_h, src_w, src_pitch;
  int32_t new_h, new_w, top, left;
  void* dst;       int32_t out_h, out_w;
  int32_t out_chw, swap_rb;
  uint8_t pad[4];
} y3_letterbox_desc;
int y3_letterbox_u8(const y3_letterbox_desc* d, y3_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Training augmentation on the device (LoadImagesAndLabels.__getitem__ with augment=True, utils/dataloaders.py:659-822;
 * utils/augmentations.py:57-73,137-216,270-275) — csrc/y3_augment.cu.  Caller-owned buffers, no allocation, no
 * synchronisation: both entry points are graph-capturable.  The descriptor arrays live in DEVICE memory.
 *
 * y3_resize_u8_batched: load_image's cv2.resize (INTER_LINEAR; dst = ceil(w0 r) x ceil(h0 r)) of every item in one launch,
 *   the rule of y3_letterbox_u8.  src / dst are uint8 HWC BGR [h, w, 3] with row pitches in bytes.  `items` is in DEVICE
 *   memory and `host_items` the same array in HOST memory, from which every item is validated (non-null src / dst, positive
 *   sizes, pitches of at least 3 w bytes; Y3_ERR_BAD_ARG before any launch otherwise) and the grid is sized.
 * y3_augment_u8: one output image per descriptor into out [n, 3, out_h, out_w] (uint8 CHW RGB: a TrainEngine input).  Per
 *   output pixel: the affine warp of cv2.warpAffine (INTER_LINEAR, border 114; inv = the inverted M as
 *   cv::invertAffineTransform computes it: A11, A12, b1, A21, A22, b2) of a VIRTUAL canvas — up to 4 placements of resized
 *   sources (canvas rectangle [x0, x1) x [y0, y1), canvas pixel (X, Y) = source pixel (X - off_x, Y - off_y)), 114 elsewhere
 *   (load_mosaic's img4 or letterbox's border, never materialised); with mixup, the same of canvas[1] blended as
 *   trunc(a r + b (1 - r)) in double; with hsv, cv2's BGR2HSV, the three LUTs and HSV2BGR (augment_hsv); then flipud /
 *   fliplr and the HWC BGR -> CHW RGB store.  A descriptor with dst == NULL writes out[i]; one with dst set writes its
 *   out_h x out_w image at dst instead, rows dst_pitch bytes and planes dst_plane bytes apart (a quadrant of a 2x2 tile,
 *   a scratch image; collate_fn4 of train.py --quad).
 * y3_upsample2x_u8: collate_fn4's F.interpolate(scale_factor=2, bilinear, align_corners=False) and the cast back to uint8,
 *   in its exact integer form: per axis, output 2k = (x[k-1] + 3 x[k]) / 4 and 2k+1 = (3 x[k] + x[k+1]) / 4 with the
 *   indices clamped to the image; the product of the two axes' quarter weights over 16, truncated.  src: n uint8 CHW
 *   [3, h, w] images, contiguous; image k is written to out[dst_index[k]] of out [*, 3, 2h, 2w].  dst_index is in DEVICE
 *   memory. */
typedef struct y3_resize_item {
  const void* src; int32_t src_h, src_w, src_pitch;
  void* dst;       int32_t dst_h, dst_w, dst_pitch;
} y3_resize_item;
int y3_resize_u8_batched(const y3_resize_item* items, const y3_resize_item* host_items, int32_t n_items,
                         y3_stream_t stream);

#define Y3_AUG_MAX_PLACE 4
typedef struct y3_aug_place {
  const void* src;              /* uint8 HWC BGR, row pitch `pitch` bytes */
  int32_t pitch;
  int32_t x0, y0, x1, y1;       /* canvas rectangle */
  int32_t off_x, off_y;         /* canvas - source coordinates */
} y3_aug_place;
typedef struct y3_aug_canvas {
  y3_aug_place place[Y3_AUG_MAX_PLACE];
  int32_t n_place;
  double inv[6];                /* A11, A12, b1, A21, A22, b2 */
} y3_aug_canvas;
typedef struct y3_augment_desc {
  y3_aug_canvas canvas[2];      /* canvas[1] is read only with mixup */
  int32_t mixup, hsv, flipud, fliplr;
  double mix_r;                 /* np.random.beta(32, 32) */
  uint8_t lut[3][256];          /* hue, saturation, value */
  void* dst;                    /* NULL: out[i] */
  int64_t dst_plane;            /* with dst: bytes between the R, G and B planes ... */
  int32_t dst_pitch, reserved;  /* ... and between rows */
} y3_augment_desc;
int y3_augment_u8(const y3_augment_desc* descs, int32_t n, int32_t out_h, int32_t out_w, void* out, y3_stream_t stream);
int y3_upsample2x_u8(const void* src, const int32_t* dst_index, int32_t n, int32_t h, int32_t w, void* out,
                     y3_stream_t stream);

/* Validation loader on the device (LoadImagesAndLabels.__getitem__ with augment=False, utils/dataloaders.py:676-686,
 * 699-756) — csrc/y3_augment.cu.  Both entry points read their item array from DEVICE memory (`items` / `descs`) and take
 * the same array in HOST memory (`host_items` / `host_descs`), from which they validate every item and size the grid.
 * Caller-owned buffers, no allocation, no synchronisation.
 *
 * y3_resize_area_u8_batched: load_image's cv2.resize(..., INTER_AREA) of every item in one launch, bit for bit: integer
 *   factors take the block mean ((a+b+c+d+2)>>2 at 2x2), other scales the area tables of cv::resize in float.  Only
 *   scales >= 1 in both axes (dst <= src) are built; an item that scales up is refused with Y3_ERR_BAD_ARG.
 * y3_letterbox_u8_batched: y3_letterbox_u8 for n descriptors in one launch (letterbox's INTER_LINEAR resize + border +
 *   layout), e.g. every image of a rect validation batch written straight into its [bs, 3, H, W] uint8 input. */
int y3_resize_area_u8_batched(const y3_resize_item* items, const y3_resize_item* host_items, int32_t n_items,
                              y3_stream_t stream);
int y3_letterbox_u8_batched(const y3_letterbox_desc* descs, const y3_letterbox_desc* host_descs, int32_t n,
                            y3_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Baseline JPEG decode on the device, bit for bit cv2.imread / cv2.imdecode(IMREAD_COLOR) (libjpeg-turbo with its defaults:
 * accurate integer IDCT, fancy upsampling; EXIF orientation applied) — csrc/y3_jpeg.cu, csrc/y3_jpeg.cuh.
 *
 * y3_jpeg_parse (HOST code, no CUDA call): reads the markers of one file.  info->eligible = 1 when the device decodes it:
 *   SOF0 / SOF1 with 8-bit samples, Huffman coded, one interleaved scan of every component, 1 component or 3 in YCbCr, luma
 *   sampling 1x1, 2x1, 2x2, 1x2 or 4x1 with chroma 1x1, any DRI / APPn / COM, EXIF orientation 1-8.  Anything else, and a
 *   truncated or malformed file, gives eligible = 0 (decode it on the host).  Fills the geometry, the table blob (laid out for
 *   the device) and up to seg_cap (start, length) pairs of the restart segments in UNSTUFFED bytes; geom.n_segs is set even
 *   when it exceeds seg_cap (call again with room).  Returns Y3_OK, or Y3_ERR_BAD_ARG on a null argument.
 * y3_jpeg_workspace_bytes: device scratch one image needs (unstuffed bytes, decoder state, coefficients, component planes).
 * y3_jpeg_decode_batched: decodes n images in four launches on `stream`, each into its dst (uint8 HWC BGR [height, width, 3]
 *   as oriented, row pitch dst_pitch).  descs in DEVICE memory, the same array in HOST memory (validation, grid size).  Each
 *   desc's ws must lie inside [workspace, workspace + ws_bytes).  err_flags (device int32 [n]) gets 1 for an image whose
 *   entropy-coded data is corrupt (invalid code, run past 63, data ending inside a segment, wrong block count): decode that
 *   image on the host.  No allocation, no synchronisation, graph-capturable. */
#define Y3_JPEG_TABLE_BYTES 6080
typedef struct y3_jpeg_geom {
  int32_t src_h, src_w;             /* as coded */
  int32_t height, width;            /* as returned: swapped by EXIF orientations 5-8 */
  int32_t orientation;              /* EXIF 1-8 */
  int32_t ncomp;                    /* 1 or 3 */
  int32_t hmax, vmax;               /* luma sampling factors (1, 1 for one component) */
  int32_t mcus_x, mcus_y, blocks_per_mcu, n_blocks;
  int32_t restart_interval;         /* MCUs per restart segment, 0: one segment */
  int32_t n_segs;
  int32_t data_len;                 /* entropy-coded bytes in the file, RST markers included */
  int32_t unstuffed_len;            /* the same without byte stuffing and markers */
  int32_t comp_dc[3], comp_ac[3];   /* Huffman table ids (0 / 1) per component */
} y3_jpeg_geom;
typedef struct y3_jpeg_info {
  int32_t eligible;
  int32_t reserved;
  int64_t data_off;                 /* offset of the entropy-coded data in the file */
  y3_jpeg_geom geom;
  uint8_t tables[Y3_JPEG_TABLE_BYTES]; /* quantisation (natural order, per component) and Huffman lookup tables */
} y3_jpeg_info;
typedef struct y3_jpeg_desc {
  y3_jpeg_geom geom;
  const void* data;                 /* geom.data_len entropy-coded bytes */
  const void* tables;               /* Y3_JPEG_TABLE_BYTES, 8-byte aligned */
  const void* segs;                 /* int32 [n_segs][2] */
  void* ws;                         /* y3_jpeg_workspace_bytes(&geom) bytes, 256-byte aligned */
  void* dst;
  int32_t dst_pitch;
  int32_t reserved;
} y3_jpeg_desc;
int y3_jpeg_parse(const uint8_t* buf, int64_t len, y3_jpeg_info* info, int32_t* segs, int32_t seg_cap);
int64_t y3_jpeg_workspace_bytes(const y3_jpeg_geom* geom);
int y3_jpeg_decode_batched(const y3_jpeg_desc* descs, const y3_jpeg_desc* host_descs, int32_t n, void* workspace,
                           int64_t ws_bytes, int32_t* err_flags, y3_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Test-time augmentation (Model._forward_augment, models/yolo.py:239-280).
 * y3_scale_img_f32: scale_img (ultralytics; yolo.py:246) — bilinear (align_corners = false) resample of fp32 [n,c,h,w] (read
 *   left-right flipped when flip_lr) to rh x rw inside an [n,c,oh,ow] output whose right / bottom remainder is pad_value (0.447).
 * y3_tta_merge: rows [row_begin, row_end) of one view's decoded z [bs, rows, no] go to rows [out_row_off, ...) of the merged
 *   output [bs, out_rows, no] with _descale_pred applied (xywh /= scale; x = img_w - x when the view was flipped): the
 *   _clip_augmented row selection and the torch.cat of the reference are the addressing of this copy. */
int y3_scale_img_f32(const float* in, int32_t n, int32_t c, int32_t h, int32_t w, int32_t rh, int32_t rw, int32_t oh, int32_t ow,
                     int32_t flip_lr, float pad_value, float* out, y3_stream_t stream);
int y3_tta_merge(const float* z, int32_t bs, int32_t rows, int32_t no, int32_t row_begin, int32_t row_end, float scale,
                 int32_t flip_lr, float img_w, float* out, int32_t out_rows, int32_t out_row_off, y3_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Validation matching (val.process_batch, val.py:147-188) for a whole batch and all IoU thresholds in one launch.
 * det: [bs, det_stride, 6] rows (x1,y1,x2,y2,conf,cls) in confidence order (the NMS output), det_count[bs] valid rows per image
 * (NULL: max_det each); labels: [nl, 6] rows (image, cls, x1,y1,x2,y2) in the same coordinate space as det; iouv: [niou]
 * thresholds (val.py:301: linspace(0.5, 0.95, 10)).  correct[bs, max_det, niou] (bytes 0/1):
 *   correct[d, t] = 1  <=>  detection d's best same-class label l (IoU >= iouv[t], highest IoU) exists and d is the
 *   lowest-index detection whose best label is l  — the result of the reference's sort / np.unique / np.unique sequence.
 * IoU = inter / (area_label + area_det - inter + eps), the reference box_iou's fp32 operation order (eps 1e-7).
 * At most 1024 labels per image are matched; overflow[bs] (optional) reports how many were ignored. */
int y3_val_match(const float* det, const int32_t* det_count, int32_t bs, int32_t max_det, int32_t det_stride,
                 const float* labels, int32_t nl, const float* iouv, int32_t niou, float eps, uint8_t* correct,
                 int32_t* overflow, y3_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Validation metrics (val.py:379-429, utils/metrics.py:22-178) — csrc/y3_metrics.cu.  Caller-owned buffers, no allocation,
 * no synchronisation: every entry point is graph-capturable.
 *
 * y3_val_prepare: one batch of the validation loop in native image space (val.py:394-403).
 *   det [bs, max_det, 6] + det_count[bs] (the nms_batched output); img_params [bs, 5] = (gain, pad_x, pad_y, h0, w0) of each
 *   image's ratio_pad / original shape; targets [nt, 6] = (image, cls, x, y, w, h) normalised, image index inside the batch;
 *   img_w, img_h = the letterboxed batch's width and height.
 *   det_native [bs, max_det, 6]: rows scaled by scale_boxes (y3_scale_boxes' arithmetic), class 0 when single_cls, zero rows
 *   past the count; labels_native [nt, 6] = (image, cls, xyxy): x (w, h, w, h), xywh2xyxy, scale_boxes.
 *   acc_conf / acc_cls [bs * max_det], acc_count [bs] = min(det_count, max_det), acc_tcls [nt] = int(cls): the accumulator's
 *   slices of this batch.  y3_val_match(det_native, acc_count, ..., labels_native) then writes the batch's correct rows.
 * y3_confusion_update: ConfusionMatrix(nc, conf_thres, iou_thres).process_batch(predn, labelsn) for every image of a batch
 *   that has labels (val.py:390,406), added to matrix [(nc+1), (nc+1)] (row = predicted class, column = true class, index nc =
 *   background) with integer atomics.  IoU as y3_val_match (eps 1e-7); a bit-equal IoU goes to the lower label / detection
 *   index.  At most 1024 labels per image.
 * y3_ap_per_class: ap_per_class(tp, conf, pred_cls, target_cls) (utils/metrics.py:22-91) over n_images * stride rows
 *   (conf, cls fp32, tp [rows, niou] bytes; row d of image i counts when d < counts[i], counts NULL = all) and n_labels label
 *   classes tcls.  Classes are integers in [0, nc), nc <= 1024; a prediction of another class value is ignored.  px [1000]
 *   and xap [101] are np.linspace(0, 1, 1000) / (0, 1, 101).  Outputs are indexed by class id (a class without labels has
 *   no meaning there): npred [nc + 1], nt [nc], info [2] = (max-F1 index, 1 if any tp byte is set), ap [nc, niou],
 *   curves [3, nc, 1000] = p, r, f1 (ap_per_class's p / r / f1 before the max-F1 selection), best [5, nc] = p, r, f1, tp, fp
 *   at the max-F1 index.  Confidence ties keep row order (stable), where the reference's argsort is unstable.
 *   Workspace: y3_ap_workspace_bytes(n_images * stride, nc, niou) bytes (-1: unsupported shape). */
int y3_val_prepare(const float* det, const int32_t* det_count, int32_t bs, int32_t max_det, const float* img_params,
                   int32_t single_cls, const float* targets, int32_t nt, float img_w, float img_h, float* det_native,
                   float* labels_native, float* acc_conf, float* acc_cls, int32_t* acc_count, int32_t* acc_tcls,
                   y3_stream_t stream);
int y3_confusion_update(const float* det, const int32_t* det_count, int32_t bs, int32_t max_det, const float* labels,
                        int32_t nl, int32_t nc, float conf_thres, float iou_thres, float eps, unsigned long long* matrix,
                        y3_stream_t stream);
int64_t y3_ap_workspace_bytes(int32_t n_rows, int32_t nc, int32_t niou);
int y3_ap_per_class(const float* conf, const float* cls, const uint8_t* tp, const int32_t* counts, int32_t n_images,
                    int32_t stride, int32_t niou, const int32_t* tcls, int32_t n_labels, int32_t nc, const double* px,
                    const double* xap, void* workspace, int64_t workspace_bytes, int32_t* npred, int32_t* nt, int32_t* info,
                    double* ap, double* curves, double* best, y3_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Optimizer step over ONE flat fp32 parameter buffer (train.py:411-421: clip_grad_norm_(10.0), SGD-nesterov, Adam or AdamW
 * with the three parameter groups of smart_optimizer utils/torch_utils.py:207-237, ModelEMA.update) — csrc/y3_optim.cu.
 * Layout contract: every parameter occupies a slot whose length is a multiple of 256 elements; group[i] is the group of
 * elements [256 i, 256 i + 256): 0 = weights with decay, 1 = BatchNorm weights, 2 = biases, >= 3 = not trained (buffers,
 * and frozen parameters: requires_grad False).
 * hp_dev: DEVICE float[11] = lr[3], weight_decay[3], momentum, nesterov, max_norm (0: no clipping), ema decay of this
 * update, gradient pre-scale (1/world_size after a SUM all-reduce) — read at run time, so the launches can sit in a CUDA
 * graph while the scheduler changes them.
 */
int32_t y3_sumsq_blocks(void);  /* floats of workspace y3_grad_sumsq needs */
/* out[0] = sum g[i]^2 (two-stage, fixed order: bit-reproducible); n % 4 == 0.  group (optional, then n % 256 == 0): only the
 * elements whose group is < 3 count */
int y3_grad_sumsq(const float* g, const uint8_t* group, int64_t n, float* partial, float* out, y3_stream_t stream);
/* p, m (momentum buffer, zero-initialised), ema (optional) updated in place from g; gsumsq (from y3_grad_sumsq) is read
 * only when hp_dev[8] > 0.  n = elements of p (and of ema); g and m are only touched where group < 3. */
int y3_sgd_step(float* p, const float* g, float* m, float* ema, const uint8_t* group, int64_t n, const float* hp_dev,
                const float* gsumsq, y3_stream_t stream);
/* Adam / AdamW (train.py --optimizer), torch.optim.Adam's foreach arithmetic: p, m / v (exp_avg / exp_avg_sq, zero-initialised,
 * n_train elements), ema (optional) updated in place from g.  slot[c] = parameter slot of chunk c (read where group < 3).
 * hp_dev: DEVICE float[24] = coupled weight decay[3] (Adam), decoupled decay factor 1 - lr*wd [3] (AdamW, 1: none),
 * -, -, max_norm, ema decay, gradient pre-scale (hp[8..10] as y3_sgd_step), -, 1 - beta1 [3], beta2 [3], 1 - beta2 [3],
 * eps [3]; tab_dev: DEVICE float[2 * slots] = per slot {-lr / (1 - beta1^t), sqrt(1 - beta2^t)} at the slot's own step t. */
int y3_adam_step(float* p, const float* g, float* m, float* v, float* ema, const uint8_t* group, const int32_t* slot, int64_t n,
                 const float* hp_dev, const float* tab_dev, const float* gsumsq, y3_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Whole-graph executor.  Replaces BaseModel._forward_once (models/yolo.py:135-147): the Python loop over nn.Modules
 * becomes an immutable list of prepared launches (TMA descriptors encoded once at create) replayed on one stream.
 * All buffers belong to the caller; y3_model_forward is CUDA-graph capturable.
 */
#define Y3_OP_CONV_FIRST 1
#define Y3_OP_CONV 2
#define Y3_OP_MAXPOOL 3
#define Y3_OP_DECODE 4
#define Y3_OP_AMAX 5     /* FP8 calibration: y3_amax_nhwc of one producer's output, right after the producer */
typedef struct y3_amax_desc {
  const void* x;
  int32_t fmt, ld, coff, n, h, w, c;
  float* amax;
} y3_amax_desc;
typedef struct y3_op {
  int32_t kind;          /* Y3_OP_*: selects which member below is read */
  y3_conv_desc conv;
  y3_first_desc first;
  y3_pool_desc pool;
  y3_decode_desc decode;
  y3_amax_desc amax;
} y3_op;
typedef struct y3_model y3_model;
int y3_model_create(const y3_op* ops, int32_t n_ops, y3_model** out);
/* input: optional override of the first op's image pointer (NULL = the pointer given at create). */
int y3_model_forward(const y3_model* m, const void* input, y3_stream_t stream);
int32_t y3_model_num_launches(const y3_model* m);
/* Profiling aid (synchronises; not capturable): average device time of every launch over `iters` passes, measured
 * with CUDA events on `stream`; ms_out is a HOST array of y3_model_num_launches() floats. */
int y3_model_forward_timed(const y3_model* m, const void* input, y3_stream_t stream, float* ms_out, int32_t iters);
void y3_model_destroy(y3_model* m);

/* ---------------------------------------------------------------------------------------------------------------
 * AutoAnchor (utils/autoanchor.py, train.py:316) — csrc/y3_anchor.cu.  wh / obs: DEVICE [n, 2] fp32 label widths and heights.
 *
 * y3_anchor_metric: r = wh / k, x = min(r, 1 / r) over both coordinates, best = max of x over the na anchors, NaN
 *   propagating as torch; in fp32 (k rounded to fp32: check_anchors' metric) or, fp64 != 0, in fp64 (print_results).
 *   counts (DEVICE uint64[2]) = #(best > thr), #(x > thr) over all n * na; sums (DEVICE double[3]) = sum x, sum best, sum of
 *   the x > thr.  thr = 1 / anchor_t, rounded to the metric's precision and compared there, as torch compares a tensor with
 *   a Python float.  k: DEVICE double[na, 2].
 */
int y3_anchor_metric(const float* wh, int64_t n, const double* k, int32_t na, double thr, int32_t fp64, uint64_t* counts,
                     double* sums, y3_stream_t stream);
/* y3_anchor_evolve: kmean_anchors' genetic evolution (autoanchor.py:150-162), the generations in order on the stream with no
 * host synchronisation.  k0: DEVICE double[na, 2] (the sorted start anchors); v: DEVICE double[gen, na, 2] the mutation
 * factors, drawn by the caller.  Each generation: kg = (k * v[g]).clip(min=2.0) in fp64, fg = mean(best * (best > thr)) over
 * kg rounded to fp32 (best > thr compared in fp32 against thr rounded to fp32), summed exactly and rounded to fp32 once, then divided by n in fp32; accepted when fg > f.
 * Outputs (DEVICE): k_out double[na, 2], fit float[gen + 1] (the start fitness, then each candidate's), accepted uint8[gen].
 * fp32(thr) in [2^-9, 1], n <= 2^31.  Workspace: y3_anchor_evolve_workspace_bytes() bytes, 16-byte aligned. */
int64_t y3_anchor_evolve_workspace_bytes(void);
int y3_anchor_evolve(const float* wh, int64_t n, int32_t na, double thr, const double* k0, const double* v, int32_t gen,
                     double* k_out, float* fit, uint8_t* accepted, void* ws, int64_t ws_bytes, y3_stream_t stream);
/* scipy.cluster.vq.kmeans(obs, k, iter=restarts) with every restart run at once, bit for bit.  y3_kmeans_init takes the
 * restarts' initial codes (DEVICE int64 init_idx[restarts, k], rows of obs: scipy's choice(n, k, replace=False) draws) and
 * resets the per-restart state; each y3_kmeans_pass then runs one iteration of scipy's _kmeans loop for every restart not yet
 * done: vq, the fp32 mean distortion (numpy's pairwise sum), update_cluster_means with its empty clusters dropped and the
 * |change| > thresh test, or, once that test fails, the final vq.  Call passes until every status[r] is 2 (done).
 * Per restart (DEVICE): book float[restarts, k, 2] (first ncode[r] codes valid), ncode, status (0 running, 1 final vq next,
 * 2 done), dist (final mean distortion), passes (vq passes run).  k <= 32, restarts <= 64.
 * Workspace: y3_kmeans_workspace_bytes(n, restarts) bytes (-1: unsupported), 256-byte aligned. */
int64_t y3_kmeans_workspace_bytes(int64_t n, int32_t restarts);
int y3_kmeans_init(const float* obs, int64_t n, int32_t restarts, int32_t k, const int64_t* init_idx, float* book,
                   int32_t* ncode, int32_t* status, float* dist, int32_t* passes, void* ws, int64_t ws_bytes,
                   y3_stream_t stream);
int y3_kmeans_pass(const float* obs, int64_t n, int32_t restarts, int32_t k, float thresh, float* book, int32_t* ncode,
                   int32_t* status, float* dist, int32_t* passes, void* ws, int64_t ws_bytes, y3_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* YOLOV3_B200_H */
