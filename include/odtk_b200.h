/*
 * odtk_b200.h -- C ABI of the H100-native RetinaNet inference hot path.
 *
 * Drop-in boundary for NVIDIA/retinanet-examples (ODTK).  Every entry point is
 * plain C: raw device pointers, sizes, a cudaStream_t passed as void*.  No torch,
 * no C++ types.  The reference interface each function replaces is cited.
 *
 * Conventions shared by all post-processing entry points (they mirror
 * odtk::cuda::*, which is also what the TensorRT plugins' enqueue() call,
 * csrc/plugins/DecodePlugin.h:152-161, NMSPlugin.h:131-138):
 *   - cub-style two-phase workspace: call with workspace == NULL or
 *     workspace_size == 0 to get the required bytes (>= 0); the real call
 *     returns 0 (csrc/cuda/decode.cu:53-72, nms.cu:87-105).  The return type is
 *     64-bit (the reference returns int, which overflows for large batches).
 *   - the caller owns every buffer; the library never allocates device memory
 *     in these calls and never synchronises the host with the stream
 *     (the reference blocks B*5+B times per forward, decode.cu:103, nms.cu:131).
 *   - errors: a negative ODTK_E_* code; nothing is thrown across the boundary.
 */
#ifndef ODTK_B200_H_
#define ODTK_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ODTK_OK 0
#define ODTK_E_INVALID (-1)     /* bad argument (null pointer, size <= 0, ...)      */
#define ODTK_E_WORKSPACE (-2)   /* workspace too small (reference: utils.h:55-57)    */
#define ODTK_E_UNSUPPORTED (-3) /* size outside what the sm_90a kernels handle     */
#define ODTK_E_CUDA (-4)        /* a CUDA runtime / driver call failed               */

typedef void *odtk_stream_t; /* cudaStream_t */

/* Limits of the sm_90a kernels (documented deviations from "any size"). */
#define ODTK_MAX_TOP_N 4096      /* decode: top_n                                   */
#define ODTK_MAX_NMS_COUNT 6144  /* nms: candidates per image                       */
#define ODTK_MAX_DETECTIONS 1024 /* nms: detections_per_im                          */

/* Library identification: returns a static string "odtk_b200 <version> sm_90a". */
const char *odtk_b200_version(void);

/* ---- decode -------------------------------------------------------------------
 * Replaces odtk::cuda::decode (csrc/cuda/decode.h:30-35, decode.cu:44-171) and
 * odtk::cuda::decode_rotate (decode_rotate.h:30-35, decode_rotate.cu:42-179).
 *   inputs  = { scores [B, A*C, H, W], deltas [B, A*4|6, H, W] }  fp32, contiguous
 *   outputs = { scores [B, top_n], boxes [B, top_n, 4|6], classes [B, top_n] } fp32
 * Semantics: keep scores > score_thresh; if more than top_n survive, keep the
 * top_n by (score desc, flat index asc) in that order, else keep flat-index order;
 * decode each against anchors[4*a..] with the +1 width convention and the
 * reference's clamps; zero the tails.  anchors is a HOST pointer (the reference
 * takes std::vector<float>&; num_anchor_floats == 4*A, or 0 for raw deltas).    */
long long odtk_decode(int batch, const void *const *inputs, void *const *outputs, size_t height,
                      size_t width, size_t scale, size_t num_anchors, size_t num_classes,
                      const float *anchors, size_t num_anchor_floats, float score_thresh, int top_n,
                      void *workspace, size_t workspace_size, odtk_stream_t stream);

long long odtk_decode_rotate(int batch, const void *const *inputs, void *const *outputs, size_t height,
                             size_t width, size_t scale, size_t num_anchors, size_t num_classes,
                             const float *anchors, size_t num_anchor_floats, float score_thresh,
                             int top_n, void *workspace, size_t workspace_size, odtk_stream_t stream);

/* Extended decode (H100-native addition): same maths, but the three outputs are
 * written at element offset out_offset of rows that are out_stride entries long,
 * so that the five pyramid levels land directly in the [B, 5*top_n] buffers the
 * reference builds with torch.cat (odtk/model.py:164).  nbox = 4 or 6.          */
long long odtk_decode_ex(int batch, const void *const *inputs, void *const *outputs, size_t height,
                         size_t width, size_t scale, size_t num_anchors, size_t num_classes,
                         const float *anchors, size_t num_anchor_floats, float score_thresh,
                         int top_n, int nbox, size_t out_stride, size_t out_offset, void *workspace,
                         size_t workspace_size, odtk_stream_t stream);

/* All pyramid levels of the whole batch in three launches (H100-native addition; the
 * reference calls decode once per level, odtk/model.py:153-161, and torch.cat's the
 * results, :164).  Level l writes columns [out_offset + l*top_n, +top_n) of the
 * [B, out_stride] outputs.  anchors in odtk_level_t is a HOST pointer (4*A floats). */
#define ODTK_MAX_LEVELS 8
typedef struct {
  const void *scores;  /* device [B, A*C, H, W] fp32 */
  const void *deltas;  /* device [B, A*nbox, H, W] fp32 */
  size_t height, width, scale;
  const float *anchors; /* host, 4*A floats (ignored when num_anchor_floats == 0) */
} odtk_level_t;

long long odtk_decode_levels(int batch, int num_levels, const odtk_level_t *levels, size_t num_anchors,
                             size_t num_classes, size_t num_anchor_floats, float score_thresh, int top_n,
                             int nbox, void *const *outputs, size_t out_stride, size_t out_offset,
                             void *workspace, size_t workspace_size, odtk_stream_t stream);

/* Fused class-head path (H100-native): the last class-head convolution appends its above-threshold
 * scores straight to the decode workspace (odtk_conv2d with out_mode ODTK_OUT_CANDIDATES and the level's
 * sink) instead of writing the dense [B, A*C, H, W] score map that odtk_decode_levels would stream
 * through again.  odtk_decode_fused_begin lays out `workspace` (query the size with workspace == NULL)
 * with candidate lists large enough for every score, zeroes the counters and fills sinks[num_levels]
 * (host array); after the convolutions have run on the same stream (or on streams ordered after it),
 * odtk_decode_fused_finish selects the top_n per level and decodes the boxes exactly like
 * odtk_decode_levels.  levels[].scores is ignored (may be NULL); deltas are read by _finish only. */
typedef struct {
  int *counts;          /* device [B]: candidates appended per image                 */
  uint32_t *hist;       /* device [B, hist_bins]: score-key histogram per image      */
  void *cand;           /* device [B, cap] (uint32 key, uint32 flat index) pairs     */
  long long cap;
  uint32_t key_thresh;
  int shift, hist_bins;
  float thresh;         /* a score is a candidate iff score > thresh                 */
} odtk_cand_sink_t;

long long odtk_decode_fused_begin(int batch, int num_levels, const odtk_level_t *levels, size_t num_anchors,
                                  size_t num_classes, float score_thresh, int top_n, odtk_cand_sink_t *sinks,
                                  void *workspace, size_t workspace_size, odtk_stream_t stream);
long long odtk_decode_fused_finish(int batch, int num_levels, const odtk_level_t *levels, size_t num_anchors,
                                   size_t num_classes, size_t num_anchor_floats, float score_thresh, int top_n,
                                   int nbox, void *const *outputs, size_t out_stride, size_t out_offset,
                                   void *workspace, size_t workspace_size, odtk_stream_t stream);

/* ---- nms ----------------------------------------------------------------------
 * Replaces odtk::cuda::nms (csrc/cuda/nms.h:28-31, nms.cu:82-160) and
 * odtk::cuda::nms_rotate (nms_iou.h:28-31, nms_iou.cu:260-322).
 *   inputs  = { scores [B, count], boxes [B, count, 4|6], classes [B, count] } fp32
 *   outputs = { scores [B, D], boxes [B, D, 4|6], classes [B, D] }            fp32
 * Semantics: drop scores <= 0, stable sort descending, greedy same-class
 * suppression when overlap > nms_thresh (+1 widths; rotated: polygon clipping
 * with the reference's quirks), emit the first min(D, n) entries of (kept...,
 * suppressed...) exactly as the reference's second sort leaves them.           */
long long odtk_nms(int batch, const void *const *inputs, void *const *outputs, size_t count,
                   int detections_per_im, float nms_thresh, void *workspace, size_t workspace_size,
                   odtk_stream_t stream);

long long odtk_nms_rotate(int batch, const void *const *inputs, void *const *outputs, size_t count,
                          int detections_per_im, float nms_thresh, void *workspace,
                          size_t workspace_size, odtk_stream_t stream);

/* Extended nms: nbox = 4|6; out_index (device int32 [B, D], may be NULL) receives
 * the input position of every emitted entry (-1 for empty slots) -- the "kept
 * indices" the parity tests compare bit-exactly.  fixed_angle != 0 rotates the
 * max box with its OWN sin/cos instead of the candidate's (reference quirk,
 * nms_iou.cu:188-192); 0 is bug-compatible.                                     */
long long odtk_nms_ex(int batch, const void *const *inputs, void *const *outputs, size_t count,
                      int detections_per_im, float nms_thresh, int nbox, int fixed_angle,
                      int32_t *out_index, void *workspace, size_t workspace_size,
                      odtk_stream_t stream);

/* nms + gather (H100-native).  As odtk_nms_ex, plus:
 *   packed (device [B, D, 2 + nbox] fp32, may be NULL): the detections as (score, box..., class) rows -- the layout that
 *     travels between ranks; outputs may then be NULL.
 *   gather (may be NULL): image-wise sharded inference (odtk/infer.py:98-102 all_gathers the per-rank results).  Here
 *     the NMS kernel itself stores each image's packed rows into EVERY rank's gather buffer through NVLink peer
 *     mappings and counts its arrival there; odtk_gather_wait (same stream, after the call) returns once all ranks'
 *     rows of the current step have landed in THIS rank's buffer.  No NCCL launch, nothing between the kernels: the
 *     whole step, collective included, is CUDA-graph capturable.
 *     packed[p]: rank p's gather buffer (peer-mapped device pointer; packed[rank] is the local one), two parity
 *     halves of [num_peers * B, D, 2 + nbox] fp32 (step k lands in half k & 1, so a rank that runs ahead never
 *     overwrites rows its neighbour is still reading); flags[p]: rank p's arrival counters, uint32[num_peers],
 *     zero-initialised once; epoch: LOCAL device uint32 step counter, zero-initialised, advanced by odtk_gather_wait. */
#define ODTK_MAX_PEERS 8
typedef struct {
  void *packed[ODTK_MAX_PEERS];
  unsigned *flags[ODTK_MAX_PEERS];
  unsigned *epoch;
  int num_peers, rank;
} odtk_gather_t;
long long odtk_nms_gather(int batch, const void *const *inputs, void *const *outputs, size_t count,
                          int detections_per_im, float nms_thresh, int nbox, int fixed_angle, int32_t *out_index,
                          void *packed, const odtk_gather_t *gather, void *workspace, size_t workspace_size,
                          odtk_stream_t stream);
int odtk_gather_wait(const odtk_gather_t *gather, int batch, odtk_stream_t stream);

/* ---- iou (rotated target assignment) ---------------------------
 * Replaces odtk::cuda::iou (csrc/cuda/nms_iou.h:33-35, nms_iou.cu:324-387), the kernel behind
 * odtk._C.iou (csrc/extensions.cpp:47-67,200).
 *   inputs  = { boxes [num_boxes, 4 corners, (x, y)], anchors [num_anchors, 4, 2] }  fp32
 *   outputs = { iou [num_anchors, num_boxes] }                                        fp32
 * Element [a, j]: anchor a (jittered by 0.001 where a coordinate equals the same corner of box j)
 * clipped against the edges of box j, intersection / (area_a + area_j - intersection), with the
 * reference's NaN rules.  Same signature as the reference entry point; returns 0 or ODTK_E_*.   */
int odtk_iou(const void *const *inputs, void *const *outputs, int num_boxes, int num_anchors,
             odtk_stream_t stream);

/* ---- convolution engine ----------------------------------------------------------
 * Replaces the nn.Conv2d (+ BatchNorm + ReLU + residual / FPN upsample-add) library
 * calls of the reference's Model.forward (odtk/model.py:57-68,130-135;
 * odtk/backbones/fpn.py:45-61; torchvision resnet blocks): the reference has no
 * convolution kernel of its own (cuDNN through PyTorch).  Activations are NHWC fp16,
 * weights [Cout, ksize*ksize*Cin] fp16 (tap-major, channel-minor), fp32 accumulation.
 * odtk_conv2d handles 1x1 and 3x3 (pad ksize/2) convolutions with Cin % 64 == 0 on the
 * tensor cores, stride 1 or stride 2 (even sizes: parity-split view; odd sizes: element-strided TMA
 * boxes), all im2col-free.  odtk_lower_conv (explicit receptive-field gather) remains for callers
 * with Cin % 64 != 0. */
#define ODTK_OUT_NHWC_F16 0          /* y: [N, H, W, ldy] fp16                          */
#define ODTK_OUT_NCHW_F32 1          /* y: [N, Cout, H, W] fp32 (box head output)       */
#define ODTK_OUT_NCHW_F32_SIGMOID 2  /* same, sigmoid applied (odtk/model.py:140)       */
#define ODTK_OUT_CANDIDATES 3        /* sigmoid applied, scores > thresh appended to `sink` (y unused) */
typedef struct {
  const void *x;        /* NHWC fp16 [n, h, width, cin]                                 */
  const void *w;        /* fp16 [cout, ksize*ksize*cin]                                 */
  const float *bias;    /* fp32 [cout] or NULL (conv bias or folded BatchNorm shift)    */
  const void *residual; /* NHWC fp16 [n, h, width, ldr] added before ReLU, or NULL      */
  const void *upsample; /* NHWC fp16 [n, h/2, width/2, cout] nearest-upsampled and added */
  void *y;
  int n, h, width, cin, cout, ksize, relu /* 0 none, 1 ReLU, 2 ReLU6 (NHWC fp16 output only) */, out_mode, ldy, ldr;
  int stride;           /* 0/1, or 2: stride-2 conv (pad ksize/2); y is [n, (h-1)/2+1, (width-1)/2+1, ...] */
  const void *bias_op;  /* optional: bias packed by odtk_conv_pack_bias ([cout, 64] fp16).  Accepted for ABI
                           compatibility and not read: the sm_90a kernel adds the fp32 bias in its epilogue */
  const odtk_cand_sink_t *sink; /* out_mode ODTK_OUT_CANDIDATES: where the candidates go (host struct)       */
  int groups;           /* 0 / 1 dense; > 1: grouped 3x3 (ResNeXt, odtk/backbones/fpn.py:85-91): cin == cout, a group never
                           straddles a 64-channel chunk, w is [cout, 9*64] with the group's weights at the columns of
                           its input channels inside the chunk (zeros elsewhere: block-diagonal)                   */
  /* Views into a larger NHWC buffer (3x3 only; 0 = dense): the pyramid ATLAS holds the five FPN levels of a batch stacked
   * vertically in ONE [n, rows, width, C] tensor (zero gap rows between levels, zero columns right of the narrower ones),
   * so that a head layer runs as one launch over all levels instead of five.                                           */
  int x_rows, x_width;  /* x is the top-left h x width rectangle of images that are x_rows x x_width pixels apart        */
  int y_rows, y_row_off, y_width; /* NHWC y: pixel (i, r, c) is written at ((i * y_rows + y_row_off + r) * y_width + c)   */
  const void *tile_tab; /* device int32 [tab_tiles][4] = (row0, col0, row_limit, col_limit) of every 8 x 16 pixel tile of one
                           image: x and y are then whole atlases [n, h, width, C]; only pixels below the limits are written */
  int tab_tiles;
} odtk_conv_t;
int odtk_conv2d(const odtk_conv_t *desc, odtk_stream_t stream);

/* INT8 convolution (H100-native; the reference's INT8 mode is a TensorRT engine built with its entropy calibrator):
 * s8 activations x s8 weights on the integer tensor cores, exact s32 accumulation, then per output channel c
 *     y = fmaf((float)acc, alpha[c], bias[c])      alpha[c] = s_in * s_w[c], computed by the caller in fp32
 * then ReLU if requested, then one output mode:
 *     ODTK_OUT_NHWC_S8          y: NHWC s8 [n, h, width, cout], clamp(rint(y * inv_out_scale), -127, 127)
 *     ODTK_OUT_NCHW_F32[_SIGMOID], ODTK_OUT_CANDIDATES   as for odtk_conv2d
 * Weights: s8 [cout, ksize*ksize*cin] (tap-major, channel-minor, symmetric per output channel); activations symmetric,
 * zero-point 0, so zero padding (and the atlas gap rows / columns) stays exact.  Stride 1, ksize 1 or 3, cin % 128 == 0;
 * anything else returns ODTK_E_UNSUPPORTED.  x_rows / x_width (3x3 only) and tile_tab / tab_tiles are the atlas views of
 * odtk_conv_t (with a tile table y is a whole atlas like x).                                                          */
#define ODTK_OUT_NHWC_S8 4
typedef struct {
  const void *x;        /* NHWC s8 [n, h, width, cin]                                   */
  const void *w;        /* s8 [cout, ksize*ksize*cin]                                   */
  const float *alpha;   /* fp32 [cout]: s_in * s_w[c]                                   */
  const float *bias;    /* fp32 [cout] or NULL                                          */
  void *y;
  int n, h, width, cin, cout, ksize, relu, out_mode;
  float inv_out_scale;  /* ODTK_OUT_NHWC_S8: 1 / s_out                                  */
  const odtk_cand_sink_t *sink;
  int x_rows, x_width;
  const void *tile_tab;
  int tab_tiles;
} odtk_conv_s8_t;
int odtk_conv2d_s8(const odtk_conv_s8_t *desc, odtk_stream_t stream);
/* INT8 convolution with the backbone / FPN features (H100-native; odtk_conv2d_s8 is this call with the extension zeroed):
 *   stride     0/1, or 2 (pad ksize/2; y is [n, (h-1)/2+1, (width-1)/2+1, cout]): the parity-split view on even sizes,
 *              element-strided boxes on odd sizes or an x view, as for odtk_conv2d.
 *   residual   NHWC s8 [n, oh, ow, cout] (the output geometry) or NULL;  t = fmaf((float)r, res_scale, t)
 *   upsample   NHWC s8 [n, h/2, width/2, cout] (stride 1, h and width even) or NULL;
 *              t = fmaf((float)u, up_scale, t) with u the addend at (row >> 1, column >> 1): FPN nearest-2x upsample-add
 *   y_rows, y_row_off, y_width   ODTK_OUT_NHWC_S8 output into a level view of an atlas, as in odtk_conv_t (3x3 only)
 * The addends follow fmaf(acc, alpha, bias) in this order, then ReLU and requantisation.  Addends and output views need
 * out_mode ODTK_OUT_NHWC_S8; views and tile tables take no addends; anything else returns ODTK_E_UNSUPPORTED.           */
typedef struct {
  odtk_conv_s8_t base;
  int stride;
  const void *residual;
  float res_scale;
  const void *upsample;
  float up_scale;
  int y_rows, y_row_off, y_width;
} odtk_conv_s8_ex_t;
int odtk_conv2d_s8_ex(const odtk_conv_s8_ex_t *desc, odtk_stream_t stream);
/* s8 twin of odtk_copy_rows_f16 with ReLU: y = max(x, 0) over n x rows runs of row_elems int8 (pitches in elements,
 * everything a multiple of 16, 16-byte aligned): the input of FPN pyramid7, ReLU(P6), from a level of the s8 atlas. */
int odtk_relu_copy_rows_s8(const void *x, void *y, int n, int rows, int row_elems, long long x_img_pitch,
                           long long x_row_pitch, long long y_img_pitch, long long y_row_pitch, odtk_stream_t stream);
/* Full-precision convolution (the reference's --full-precision, odtk/main.py:192-195, odtk/infer.py:54-58): fp32
 * activations, fp32 weights split on the host into two tf32-valued halves w_hi = rna_tf32(w), w_lo = rna_tf32(w - w_hi)
 * (low 13 bits zero, [cout, ksize*ksize*cin], tap-major / channel-minor).  The kernel splits the activations the same way
 * and accumulates a_hi*b_lo + a_lo*b_hi + a_hi*b_hi on the tf32 tensor cores into fp32 ("3xTF32"): the operand error per
 * product is about 3 * 2^-22 |a||b| instead of 2^-11 for one TF32 pass.  Then + bias, + residual, + upsample (fp32 adds),
 * ReLU, and one output mode:
 *     ODTK_OUT_NHWC_F32          y: NHWC fp32 [n, oh, ow, ldy] (or a level view of an fp32 atlas)
 *     ODTK_OUT_NCHW_F32[_SIGMOID], ODTK_OUT_CANDIDATES   as for odtk_conv2d
 * ksize 1 / 3 with cin % 32 == 0, stride 1 / 2 (pad ksize/2), the views and tile tables of odtk_conv_t; or ksize 7,
 * stride 2, cin 3: the ResNet stem (pad 3) over x = the NHWC4 fp32 image [n, h+6, width+8, 4] of odtk_pad_input_f32, with
 * w packed [cout, 224] as k = r*32 + s*4 + c (zero for s = 7 or c = 3); any h and width.  NHWC outputs need cout even.  Addends and output
 * views need ODTK_OUT_NHWC_F32; views and tile tables are 3x3 without addends; upsample needs stride 1 and even h, width.
 * Anything else returns ODTK_E_UNSUPPORTED.                                                                           */
#define ODTK_OUT_NHWC_F32 5
typedef struct {
  const void *x;        /* NHWC fp32 [n, h, width, cin] (stem: NHWC4 fp32 [n, h+6, width+8, 4])   */
  const void *w_hi;     /* fp32 [cout, ksize*ksize*cin], tf32-valued                             */
  const void *w_lo;     /* fp32, same shape: rna_tf32(w - w_hi)                                  */
  const float *bias;    /* fp32 [cout] or NULL                                                   */
  const void *residual; /* NHWC fp32 [n, oh, ow, ldr] or NULL                                   */
  const void *upsample; /* NHWC fp32 [n, h/2, width/2, cout] (nearest-2x, stride 1) or NULL     */
  void *y;
  int n, h, width, cin, cout, ksize, stride, relu /* 0 / 1 */, out_mode, ldy, ldr;
  const odtk_cand_sink_t *sink;
  int x_rows, x_width;
  int y_rows, y_row_off, y_width;
  const void *tile_tab;
  int tab_tiles;
} odtk_conv_f32_t;
int odtk_conv2d_f32(const odtk_conv_f32_t *desc, odtk_stream_t stream);

/* ---- training: backward of the 3x3 stride-1 head convolutions (H100-native; the reference runs them through cuDNN's
 * autograd, odtk/train.py:94-123).  All three calls work over the pyramid atlas of odtk_conv_t (or a dense NHWC tensor).
 *
 * Weight gradient: dw[co, ci, ky, kx] = sum over images and pixels p of g[p, co] * x[p + (ky - 1, kx - 1), ci] (zero
 * padding), db[co] = sum_p g[p, co]; fp32 results in the reference's parameter layouts ([cout, cin, 3, 3], [cout]).
 *   g   NHWC fp16 [n, h, width, cout_pad]: the gradient w.r.t. the convolution's output (before its ReLU), cout_pad a
 *       multiple of 64, zero outside the pixels of the levels and in the channels >= cout
 *   x   NHWC fp16 [n, h, width, cin]: the convolution's input, cin % 128 == 0
 *   tile_tab / tab_tiles   the atlas tile table of odtk_conv_t, or NULL: the 8 x 16 tiles of a dense h x width image
 * Deterministic: the K (pixel) dimension is split over the CTAs, fp32 partials are summed in a fixed order, so two calls
 * on the same inputs return the same bits.  workspace == NULL or workspace_size == 0 returns the bytes needed.       */
typedef struct {
  const void *g;
  const void *x;
  float *dw;            /* fp32 [cout, cin, 3, 3]                                                            */
  float *db;            /* fp32 [cout] or NULL                                                               */
  int n, h, width, cin, cout, cout_pad;
  const void *tile_tab;
  int tab_tiles;
} odtk_wgrad_t;
long long odtk_conv_wgrad(const odtk_wgrad_t *desc, void *workspace, size_t workspace_size, odtk_stream_t stream);

/* Weight gradient of one FPN convolution (1x1 stride 1, 3x3 stride 1 pad 1, or 3x3 stride 2 pad 1) whose output is ONE
 * level of the gradient atlas and whose input is a dense tensor:
 *   dw[co, ci, ky, kx] = sum over images and level pixels (r, c) of g[r, c, co] * x[s (r - g_row0) + ky - p, s c + kx - p, ci]
 * (zero padding), db[co] = the sum of g over the level's rows only; fp32 results in the reference's layouts ([cout, cin,
 * ksize, ksize], [cout]).
 *   g   NHWC fp16 atlas [n, g_rows, g_width, cout_pad]: cout_pad a multiple of 64; zero outside the level's pixels within
 *       the level's tiles and in the channels >= cout (the other levels' rows may hold anything)
 *   x   NHWC fp16 [n, x_h, x_width, cin], cin % 128 == 0; the level is (x_h - 1) / s + 1 rows from g_row0 by
 *       (x_width - 1) / s + 1 columns
 *   tile_tab / tab_tiles   the level's tiles of the atlas tile table of odtk_conv_t (a contiguous slice of it), or NULL:
 *       g is the convolution's dense output [n, (x_h - 1) / s + 1, (x_width - 1) / s + 1, cout_pad] (g_rows / g_width those
 *       sizes, g_row0 0; tab_tiles ignored).  1x1 stride 2 (a ResNet downsample) is accepted only so.
 *   row_scale   fp32 [cout] or NULL: dw[co] is multiplied by row_scale[co] (a BatchNorm-folded weight w * gamma / sqrt(var +
 *       eps) gives d/dw with row_scale = gamma / sqrt(var + eps)); db is not scaled
 * cin and cout up to 2048 (ResNet stages 3-4).  Any other (ksize, stride) returns ODTK_E_UNSUPPORTED.  Deterministic and
 * with the workspace query of odtk_conv_wgrad.                                                                        */
typedef struct {
  const void *g;
  const void *x;
  float *dw;            /* fp32 [cout, cin, ksize, ksize]                                                    */
  float *db;            /* fp32 [cout] or NULL                                                               */
  int n, g_rows, g_width, g_row0, cout_pad;
  int x_h, x_width, cin, cout;
  int ksize, stride;
  const void *tile_tab;
  int tab_tiles;
  const float *row_scale;
} odtk_wgrad_ex_t;
long long odtk_conv_wgrad_ex(const odtk_wgrad_ex_t *desc, void *workspace, size_t workspace_size, odtk_stream_t stream);

/* The FPN's top-down pathway backward and pyramid7's input gradient, on fp16 NHWC atlases [n, rows, width, c], c % 8 == 0,
 * levels given as (row0, h, w) at columns [0, w):
 *   odtk_pool_add_f16   dst level += the pool x pool window sums of the src level (pool 2: the backward of the nearest 2x
 *                       upsample-add, dP_l += sumpool2x2(dP_{l-1}); pool 1: a plain add), rounded once:
 *                       fp16_rn((float)dst + ((s00 + s01) + (s10 + s11))); source pixels past the src level count as 0.
 *                       src == dst is allowed when the two levels' rows are disjoint.
 *   odtk_dilate_f16     dst[dst_row0 + 2y, 2x] = src[src_row0 + y, x] for the src_h x src_w level; nothing else of dst is
 *                       written, so a zeroed dst keeps zeros at the odd positions
 *   odtk_dilate_ex_f16  the same into a destination of its own geometry [n, dst_rows, dst_width, c] with stride 1 or 2:
 *                       dst[dst_row0 + s y, s x] = src[src_row0 + y, x] (src [n, src_rows, src_width, c]; src != dst).
 *                       Stride 1 copies an atlas level into a dense tensor (the FPN's C4 / C5 input gradients); stride 2
 *                       scatters a dense gradient into a stride-2 layer's input geometry for the stride-1 dgrad.       */
int odtk_pool_add_f16(const void *src, void *dst, int n, int rows, int width, int c, int src_row0, int src_h, int src_w,
                      int dst_row0, int dst_h, int dst_w, int pool, odtk_stream_t stream);
int odtk_dilate_f16(const void *src, void *dst, int n, int rows, int width, int c, int src_row0, int src_h, int src_w,
                    int dst_row0, odtk_stream_t stream);
int odtk_dilate_ex_f16(const void *src, void *dst, int n, int c, int src_rows, int src_width, int src_row0, int src_h,
                       int src_w, int dst_rows, int dst_width, int dst_row0, int stride, odtk_stream_t stream);

/* Loss gradients -> fp16 gradient atlas: level l's fp32 NCHW gradient [batch, channels, height, width] times *scale (a
 * DEVICE fp32 scalar, NULL for 1: the upstream autograd factor, e.g. a GradScaler scale, read without a host sync) lands at rows [row0, row0 + height) x columns [0, width) of the NHWC
 * fp16 atlas [batch, rows, atlas_width, cout_pad], channels >= `channels` as zeros.  Nothing else of the atlas is written:
 * the caller zero-fills it once (gap rows and columns right of the narrow levels are the convolutions' padding).  fp16
 * overflow gives +-inf (round to nearest), never a saturated value, so that a GradScaler sees it and skips the step.    */
typedef struct {
  const float *grad;    /* device fp32 [batch, channels, height, width] */
  int height, width, row0;
} odtk_grad_level_t;
int odtk_grad_to_atlas(int batch, int num_levels, const odtk_grad_level_t *levels, int channels, const float *scale, void *atlas,
                       int rows, int atlas_width, int cout_pad, odtk_stream_t stream);

/* Input gradient of a 3x3 stride-1 convolution, masked by the ReLU derivative of its input: odtk_conv2d on `base` (x =
 * the output gradient g, w = the weights rotated by 180 degrees with cin / cout swapped, out_mode ODTK_OUT_NHWC_F16, no
 * bias, no ReLU; residual adds a second gradient, e.g. the other head tower's), then every output element whose `mask`
 * element is not > 0 becomes 0.  mask: NHWC fp16 [n, h, width, cout] (the layer input saved by the forward pass; the
 * tile table's geometry when base.tile_tab is set), or NULL for no mask.  fp16 overflow gives +-inf.
 * base.ksize 1: the same for a 1x1 convolution (w = the transposed weights [cout, cin]) over dense tensors, with a mask
 * and cout % 128 == 0 (the input channels of a layer whose weight gradient odtk_conv_wgrad_ex takes).  Stride-2 layers:
 * scatter g with odtk_dilate_ex_f16 into the input geometry, then the stride-1 call.                                  */
typedef struct {
  odtk_conv_t base;
  const void *mask;
} odtk_conv_dgrad_t;
int odtk_conv2d_dgrad(const odtk_conv_dgrad_t *desc, odtk_stream_t stream);
/* fp32 twins of the small layers around the convolutions (full-precision mode), same geometry as the fp16 calls:
 *   odtk_pad_input_f32          NHWC fp32 RGB [n, h, w, 3] -> zero-bordered NHWC4 fp32 [n, h+6, w+8, 4]
 *   odtk_preprocess_u8_f32      as odtk_preprocess_u8, the normalised fp32 values without the fp16 rounding
 *   odtk_preprocess_resize_u8_f32   (declared after odtk_preprocess_resize_u8) the same resize, y NHWC4 fp32
 *   odtk_maxpool3x3s2_f32      NHWC fp32, c % 4 == 0
 *   odtk_relu_copy_rows_f32     y = max(x, 0) over n x rows runs of row_elems floats (pitches in elements, multiples of
 *                               4, 16-byte aligned): pyramid7's input ReLU(P6) from a level of the fp32 atlas        */
int odtk_pad_input_f32(const void *x, void *y, int n, int h, int w, odtk_stream_t stream);
int odtk_preprocess_u8_f32(const void *x, void *y, int n, int h, int w, int hs, int ws, const float *mean,
                           const float *std, odtk_stream_t stream);
int odtk_maxpool3x3s2_f32(const void *x, void *y, int n, int h, int w, int c, odtk_stream_t stream);
int odtk_relu_copy_rows_f32(const void *x, void *y, int n, int rows, int row_elems, long long x_img_pitch,
                            long long x_row_pitch, long long y_img_pitch, long long y_row_pitch, odtk_stream_t stream);
/* y[i] = clamp(rint((float)x[i] * inv_scale), -127, 127): fp16 -> s8, n % 8 == 0, 16-byte aligned x, 8-byte aligned y. */
int odtk_quantize_f16_s8(const void *x, void *y, long long n, float inv_scale, odtk_stream_t stream);
/* Introspection (tests): the kernel variant the last odtk_conv2d / odtk_stem_conv call of the calling host thread
 * launched.  mode: 0 GEMM rows (1x1), 1 shifted box per tap (3x3, odd-size stride 2), 2 stem, 3 even-size stride 2;
 * bn: N tile (64, 128 or 256); grid: persistent CTAs; tma_store: 1 if the fp16 NHWC epilogue stores its tiles with TMA
 * from shared memory (odtk_set_tma_store).  cluster, npatch, tile_t, b_resident, bias_mma, res_mma and up_mma are always
 * 0 on sm_90a (kept for ABI stability).  res_mma: 1 residual tile as one I * R
 * product, 2 residual chunks through the pipeline stages (R_j * I64), 0 residual (if any) added in the epilogue.  */
typedef struct {
  int mode, cluster, bn, num_m_tiles, num_n_tiles, nstages, npatch, tile_t, b_resident, bias_mma, res_mma, tma_store;
  int th, tw, grid, up_mma;
} odtk_conv_plan_t;
int odtk_conv_last_plan(odtk_conv_plan_t *out);
/* Encoded tensor maps are cached per (base pointer, geometry); hit / miss counters of the process.         */
int odtk_conv_map_cache_stats(long long *hits, long long *misses);
/* Launch budget: the persistent kernels of this library launched by the calling process after this call use at most `sms`
 * CTAs (0 = the whole device).  Two streams with complementary budgets run side by side on disjoint SMs: the tensor-bound
 * head towers of one half batch next to the HBM-bound backbone layers of the other (Model.forward, pipelined mode).  A CUDA
 * graph keeps the grids it was captured with.                                                                          */
int odtk_set_sm_budget(int sms);
/* fp16 NHWC outputs of odtk_conv2d, odtk_stem_conv and odtk_bottleneck_tail: 1 (default) stores each tile with TMA from
 * shared memory, 0 with direct stores from the registers; both give the same bytes.  Process-wide, read at launch time
 * (a CUDA graph keeps what it captured); returns the previous setting.                                                  */
int odtk_set_tma_store(int on);

/* Buffers shared between the GPU processes of one node (CUDA IPC): odtk_peer_alloc = cudaMalloc + zero fill + a 64-byte
 * handle to send to the other ranks (any transport); odtk_peer_open maps a received handle into the CALLING process with
 * its own device current, NVLink / NVSwitch peer access enabled -- the pointer is then valid in kernels of that device
 * (the in-kernel detection gather, odtk_nms_gather); odtk_peer_close / odtk_peer_free undo them.                    */
int odtk_peer_alloc(size_t bytes, void **ptr, void *handle64);
int odtk_peer_open(const void *handle64, void **ptr);
int odtk_peer_close(void *ptr);
int odtk_peer_free(void *ptr);

/* Tail of a stride-1 ResNet bottleneck block in ONE kernel (torchvision Bottleneck.forward behind
 * odtk/backbones/resnet.py:24-39; the reference runs it as two cuDNN convolutions + an elementwise add):
 *     y = relu( conv1x1( relu( conv3x3(x, w2) + b2 ), w3 ) + b3 + residual )
 * The [n, h, width, c1] output of the 3x3 never leaves the SM: it is rounded to fp16 exactly as a separate 3x3 launch
 * stores it and becomes the shared-memory A operand of the 1x1.  c1 in {64, 128}; c2 % 128 == 0,
 * c2 <= 512; x: NHWC fp16 [n, h, width, c1]; w2: fp16 [c1, 9*c1] (tap-major, channel-minor); w3: fp16 [c2, c1];
 * b2 / b3: fp32 or NULL; residual, y: NHWC fp16 [n, h, width, c2]; relu: applied to y.                          */
typedef struct {
  const void *x, *w2, *w3, *residual;
  const float *b2, *b3;
  void *y;
  int n, h, width, c1, c2, relu;
  /* first block of layer1 (its identity is a 1x1 projection of the 64-channel block input, torchvision `downsample`): when
   * xproj != NULL the kernel computes identity = xproj [n, h, width, 64] x wproj [c2, 64]^T itself on the tensor core
   * (residual is ignored, b3 must already include the projection's bias); c1 must be 64.                          */
  const void *xproj, *wproj;
  /* GEMM3 (optional, c1 == 64, no projection): the NEXT block's conv1 -- z = relu(w_next [c_next, c2] x y + b_next), c_next in
   * {64, 128} -- computed from the block output while its chunks are still in shared memory; z: NHWC fp16
   * [n, h, width, c_next].  y is written as usual (it is the next block's identity).                               */
  const void *w_next;
  const float *b_next;
  void *z;
  int c_next;
} odtk_bneck_t;
int odtk_bottleneck_tail(const odtk_bneck_t *desc, odtk_stream_t stream);
/* bias [cout] fp32 -> out [cout, 64] fp16 = (hi, lo, 0, ...) with hi + lo == bias to 2^-22 relative.       */
int odtk_conv_pack_bias(const float *bias, void *out, int cout, odtk_stream_t stream);

/* Gather the receptive fields of a ksize x ksize / stride / pad convolution over NHWC
 * fp16 x into out[pixels, kpad] (tap-major, channel-minor, zero padded to kpad columns;
 * relu != 0 applies ReLU to the gathered values: FPN pyramid7 input, fpn.py:55).     */
int odtk_lower_conv(const void *x, void *out, int n, int h, int w, int c, int ksize, int stride, int pad,
                    int kpad, int relu, odtk_stream_t stream);
/* ResNet stem (7x7 stride-2 pad-3 conv of the RGB image) without im2col: odtk_pad_input
 * zero-pads NHWC3 fp16 [n,h,w,3] to NHWC4 [n,h+6,w+8,4]; odtk_stem_conv runs the tensor-core
 * kernel over an overlapping-window tensor map of that buffer.  w: fp16 [cout, 7*32] with
 * k = r*32 + s*4 + c (zero for s = 7, c = 3); y: NHWC fp16 [n, h/2, w/2, cout]; h, w even.   */
int odtk_pad_input(const void *x, void *y, int n, int h, int w, odtk_stream_t stream);
int odtk_stem_conv(const void *xp, const void *w, const float *bias, void *y, int n, int h, int width,
                   int cout, int relu, odtk_stream_t stream);
/* Stem + max-pool fused (H100-native): 7x7/2 convolution + bias (folded BatchNorm) + ReLU + 3x3/2 pad-1 max-pool in one
 * kernel; the [n, h/2, w/2, 64] stem activation is never written.  xp, w as for odtk_stem_conv; cout must be 64;
 * y: NHWC fp16 [n, (h/2 - 1)/2 + 1, (w/2 - 1)/2 + 1, 64].  Bit-identical to odtk_stem_conv followed by
 * odtk_maxpool3x3s2 (the same fp16 values are pooled).                                                        */
int odtk_stem_pool(const void *xp, const void *w, const float *bias, void *y, int n, int h, int width, int cout,
                   int relu, odtk_stream_t stream);
/* Depthwise 3x3 convolution, pad 1, stride 1 / 2, + bias + activation (act: 0 none, 1 ReLU, 2 ReLU6): the middle layer of
 * MobileNetV2's inverted residual blocks (torchvision InvertedResidual behind odtk/backbones/mobilenet.py:5-25).
 * x: NHWC fp16 [n, h, width, c], c % 8 == 0; w: fp16 [9, c] (tap-major); bias: fp32 [c] or NULL;
 * y: NHWC fp16 [n, (h-1)/stride+1, (width-1)/stride+1, c].                                                        */
int odtk_depthwise3x3(const void *x, const void *w, const float *bias, void *y, int n, int h, int width, int c,
                      int stride, int act, odtk_stream_t stream);
/* y = max(x, 0), fp16, n % 8 == 0, 16-byte aligned (input of FPN pyramid7: ReLU(P6), odtk/backbones/fpn.py:55). */
int odtk_relu_f16(const void *x, void *y, long long n, odtk_stream_t stream);
/* 3-D strided copy (+ ReLU when relu != 0) of n x rows runs of row_elems fp16 (pitches in elements, everything a multiple
 * of 8): moves a pyramid level between a dense tensor and its rectangle of the atlas (see odtk_conv_t).          */
int odtk_copy_rows_f16(const void *x, void *y, int n, int rows, int row_elems, long long x_img_pitch,
                       long long x_row_pitch, long long y_img_pitch, long long y_row_pitch, int relu, odtk_stream_t stream);
/* 3x3 stride-2 pad-1 max-pool, NHWC fp16 (torchvision resnet stem).                  */
int odtk_maxpool3x3s2(const void *x, void *y, int n, int h, int w, int c, odtk_stream_t stream);

/* ---- focal loss (training path) -------------------------------------------------------
 * Replaces FocalLoss.forward (odtk/loss.py:13-18) + the mask / sum of
 * Model._compute_loss (odtk/model.py:195-199) and its autograd backward, in ONE pass:
 *   loss_i = mask_i * alpha_t * (1 - p_t)^gamma * BCEwithLogits(x_i, t_i)
 *   *loss_sum = sum_i loss_i;  grad_i = grad_scale * d(loss_sum)/dx_i
 * Targets: dense fp32 one-hot `target` [n] (+ optional dense `mask` [n]), the reference's
 * layout; or `cls_index` int32 [n / (num_classes*hw), hw] with the class id per anchor
 * position (-1 background, -2 ignored => mask 0) for logits laid out [group, class, hw].
 * loss_elem (per-element loss, [n]) and grad ([n]) may be NULL.  Two-phase workspace.  */
long long odtk_focal_loss(const float *logits, const float *target, const float *mask, const int *cls_index,
                          long long n, int num_classes, int hw, float alpha, float gamma, float grad_scale,
                          float *loss_elem, float *loss_sum, float *grad, void *workspace,
                          size_t workspace_size, odtk_stream_t stream);

/* Smooth L1 (odtk/loss.py:27-31; box loss of Model._compute_loss, odtk/model.py:201-205), same fused
 * forward + backward + masked-sum form as odtk_focal_loss.                                           */
long long odtk_smooth_l1_loss(const float *pred, const float *target, const float *mask, long long n,
                              float beta, float grad_scale, float *loss_elem, float *loss_sum, float *grad,
                              void *workspace, size_t workspace_size, odtk_stream_t stream);

/* Model._compute_loss in ONE launch (odtk/model.py:186-210): over all pyramid levels, focal
 * loss of the class logits against class-index targets with the (depth >= 0) mask, smooth L1 of the box deltas with the
 * (depth > 0) mask, per-level foreground counts clamp(min=1) summed, both losses divided by that sum -- and, when the
 * grad pointers are given, the gradients of the two NORMALISED losses w.r.t. the head outputs.  Deterministic (integer
 * counts, fixed-order double sums).  out: device float[4] = {cls_loss, box_loss, fg_total, 0}.  Two-phase workspace.  */
typedef struct {
  const void *cls_logits;   /* [B, A*C, H, W] fp32 raw logits (the heads with exporting / training semantics: no sigmoid) */
  const void *box_pred;     /* [B, A*nbox, H, W] fp32                                                                    */
  const int *cls_index;     /* [B, A, H, W] int32: class, -1 background, -2 ignored (odtk_snap_to_anchors)               */
  const float *box_target;  /* [B, A, nbox, H, W] fp32                                                                   */
  float *cls_grad;          /* like cls_logits, or NULL                                                                  */
  float *box_grad;          /* like box_pred, or NULL                                                                    */
  int height, width;
} odtk_loss_level_t;
long long odtk_retina_loss(int batch, int num_levels, const odtk_loss_level_t *levels, int num_anchors, int num_classes,
                           int nbox, float alpha, float gamma, float beta, float *out, void *workspace,
                           size_t workspace_size, odtk_stream_t stream);

/* ---- anchor target assignment --------------------------------------------
 * Replaces snap_to_anchors (odtk/box.py:134-186) + box2delta (:67-78) as called per image and level by
 * Model._extract_targets (odtk/model.py:167-184), for the whole batch in one launch.
 *   targets [B, G, 5] fp32 device: x, y, w, h, class; rows with class <= -1 are padding (the reference
 *   filters them on the host, odtk/model.py:174).  anchors: HOST pointer, 4*A floats (generate_anchors).
 *   Grid position (y, x) of anchor a covers (x*stride, y*stride) + anchors[a].
 * Outputs (device, fp32 unless noted), in the reference's layouts:
 *   cls_target [B, A, C, H, W] dense one-hot, may be NULL;  box_target [B, A, 4, H, W];
 *   depth [B, A, 1, H, W]: -1 ignored (iou_bg <= IoU < iou_fg), 0 background, class + 1 foreground;
 *   cls_index [B, A, H, W] int32, may be NULL: class, -1 background, -2 ignored -- the class-index
 *   target layout odtk_focal_loss consumes (H100-native: the dense one-hot never has to exist).
 * An image without valid rows yields zeros everywhere (odtk/box.py:140-143) and cls_index -1.         */
int odtk_snap_to_anchors(const float *targets, int batch, int max_boxes, int height, int width, int stride,
                         const float *anchors, int num_anchors, int num_classes, float iou_bg, float iou_fg,
                         float *cls_target, float *box_target, float *depth, int *cls_index,
                         odtk_stream_t stream);

/* ---- input side of `odtk infer` ---------------------------------------
 * Replaces the per-image tensor maths of CocoDataset.__getitem__ (odtk/data.py:113-123): uint8 HWC
 * [n,h,w,3] -> /255 -> (x - mean)/std -> zero padding to [hs, ws] (a multiple of the model stride),
 * written straight into the zero-padded NHWC4 fp16 buffer [n, hs+6, ws+8, 4] that odtk_stem_conv
 * reads (no fp32 image, no separate pad).  mean / std: 3 host floats.                                 */
int odtk_preprocess_u8(const void *x, void *y, int n, int h, int w, int hs, int ws, const float *mean,
                       const float *std, odtk_stream_t stream);

/* One image of odtk_preprocess_resize_u8: its uint8 HWC RGB pixels (contiguous) start `offset` bytes into x, and
 * it is resized from src_h x src_w to dst_h x dst_w.                                                          */
typedef struct {
  long long offset;
  int src_h, src_w, dst_h, dst_w;
} odtk_resize_image_t;

/* The whole input side of `odtk infer` for images of any size (odtk/data.py:55-60, 113-123, collate_fn
 * :154-176): each image is resized with Pillow's 8-bit Image.BILINEAR resampling (triangle filter, support
 * widened by the downscale factor, weights in IEEE double normalised by their sum, 22-bit fixed point,
 * horizontal pass rounded to uint8 before the vertical one; bit-exact), normalised with the operations of
 * odtk_preprocess_u8 and written at the top left of one canvas of the fp16 NHWC4 stem buffer
 * [n, canvas_h+6, canvas_w+8, 4].  Everything outside an image's dst rectangle is 0.  One fused kernel, no
 * intermediate image.
 *   images      host table of the n images: validated here, never read by the kernel;
 *   images_dev  device copy of the same table, read by the kernel.  Under a CUDA graph the caller may
 *               rewrite it (and x) before each replay with other sizes that fit the canvas;
 *   x_bytes     bytes readable from x: every image must lie in [x, x + x_bytes).
 * Two-phase: y == NULL returns the bytes y must hold.  ODTK_E_INVALID: a size <= 0, a dst larger than the
 * canvas, an odd canvas side, an image outside [x, x + x_bytes).  mean / std: 3 host floats.
 * Axes shrunk by more than 7x take a slower path that recomputes the filter taps per pixel.                  */
long long odtk_preprocess_resize_u8(const void *x, size_t x_bytes, const odtk_resize_image_t *images,
                                    const odtk_resize_image_t *images_dev, int n, int canvas_h, int canvas_w, void *y,
                                    const float *mean, const float *std, odtk_stream_t stream);
/* The same resize into the fp32 NHWC4 stem buffer of the full-precision mode: the normalised fp32 values without the
 * fp16 rounding.  Same arguments and checks; y == NULL returns the (fp32) bytes.                                 */
long long odtk_preprocess_resize_u8_f32(const void *x, size_t x_bytes, const odtk_resize_image_t *images,
                                        const odtk_resize_image_t *images_dev, int n, int canvas_h, int canvas_w, void *y,
                                        const float *mean, const float *std, odtk_stream_t stream);

/* ---- baseline JPEG decode (the Image.open(path).convert("RGB") of odtk/data.py:50, on the GPU) ------------------
 * One image of odtk_decode_jpeg: a baseline sequential Huffman-coded 8-bit JPEG (SOF0 / SOF1), grayscale or YCbCr
 * with luma sampling 1x1 (4:4:4), 2x1 (4:2:2) or 2x2 (4:2:0) and 1x1 chroma.  Byte offsets are from the start of
 * the input buffer `in`; the sums (seg_base, blk_base, pix_base) run over the images in order.                  */
typedef struct {
  long long scan_offset;   /* entropy-coded data of the scan, RSTn markers included, EOI excluded              */
  long long blk_base;      /* first 8x8 block of the image in the workspace (all components, Y then Cb, Cr)    */
  long long pix_base;      /* sum of height x width of the images before this one                              */
  int scan_bytes, height, width;
  int ncomp;               /* 1 (grayscale) or 3 (YCbCr)                                                        */
  int hmax, vmax;          /* luma sampling factors; 1, 1 for grayscale                                         */
  int restart_interval;    /* MCUs per restart segment, 0 = no restart markers                                  */
  int nseg;                /* restart segments: ceil(MCUs / restart_interval), 1 without DRI                    */
  int seg_base;            /* first segment of the image in the batch                                           */
  int quant[3];            /* per component: offset of 64 uint16 quantisation steps, row-major, 16-byte aligned */
  int dc[3], ac[3];        /* per component: offsets of its odtk_jpeg_huff_t DC and AC tables, 16-byte aligned */
} odtk_jpeg_image_t;

/* One Huffman table (T.81 annex C canonical code) as the decoder reads it. */
typedef struct {
  unsigned short look[256]; /* next 8 bits -> (code length << 8) | symbol; 0 when the code is longer than 8 bits   */
  int maxcode[18];          /* largest code of each length 1..16, -1 when there is none; [17] = INT_MAX           */
  int valoff[18];           /* val index of a code of length l = code + valoff[l]                                  */
  unsigned char val[256];   /* the symbols in code order                                                           */
} odtk_jpeg_huff_t;

/* Status bits per image (int32 status[n]; 0 = decoded).                                                      */
#define ODTK_JPEG_BAD_CODE 1       /* a bit pattern that is no code of the Huffman table                        */
#define ODTK_JPEG_BAD_INDEX 2      /* a run of zeros past coefficient 63                                        */
#define ODTK_JPEG_TRUNCATED 4      /* a restart segment ran out of entropy-coded data                           */
#define ODTK_JPEG_BAD_RESTART 8    /* the scan does not hold nseg - 1 restart markers                            */

/* Decode n baseline JPEGs bit-exactly as libjpeg(-turbo) does by default (Huffman decode, dequantisation, the
 * JDCT_ISLOW integer IDCT with its range limit, "fancy" triangle-filter chroma upsampling, the fixed-point table
 * YCbCr -> RGB conversion) into uint8 HWC RGB images; grayscale is replicated to three channels.  Four kernels:
 * restart-marker scan (one block per image), entropy decode (one thread per image and restart segment), IDCT (one
 * thread per 8x8 block), upsampling + colour conversion (one thread per pixel).
 *   in, in_bytes   device buffer [odtk_jpeg_image_t[n] | ... tables ... | entropy-coded bytes]; the descriptor
 *                  table at offset 0 is what the kernels read;
 *   images         host copy of that descriptor table: validated here, never read by a kernel;
 *   outs, outs_dev host table / its device copy: image i is written at y + outs[i].offset, src_h x src_w must be
 *                  its height x width (dst_h / dst_w are not read);
 *   workspace      restart segment bounds, int16 coefficient blocks, uint8 component planes; the kernels place
 *                  these regions from the totals of the device descriptor table, not from this call's host table;
 *   status         int32 [n] device: ODTK_JPEG_* bits of each image.  A corrupt stream never faults: its decoder
 *                  stops, sets the bits and the other images are unaffected.
 * Sizes come from the device tables, so a CUDA graph may replay the call after the caller rewrote `in` and
 * outs_dev with another batch of n images that the host tables validated and whose totals fit the buffers (its
 * workspace need, from the size query, at most workspace_bytes), even when it has more blocks or restart segments
 * than the batch the graph was captured with.  An image of more than INT32_MAX pixels is ODTK_E_UNSUPPORTED.
 * Two-phase: workspace == NULL returns the workspace bytes.  ODTK_E_INVALID: a size <= 0, inconsistent sums, an
 * offset outside its buffer; ODTK_E_UNSUPPORTED: a component count or sampling factors outside the above;
 * ODTK_E_WORKSPACE: workspace_bytes too small.                                                                */
long long odtk_decode_jpeg(const void *in, size_t in_bytes, const odtk_jpeg_image_t *images, int n,
                           const odtk_resize_image_t *outs, const odtk_resize_image_t *outs_dev, void *workspace,
                           size_t workspace_bytes, void *y, size_t y_bytes, int *status, odtk_stream_t stream);

/* ---- training input: uint8 resize and augmentation (odtk/data.py:55-123 with training=True) ----------------------
 * The resize of odtk_preprocess_resize_u8 (same kernel, same Pillow-exact BILINEAR arithmetic) keeping Pillow's uint8
 * result: image i is written as dst_h x dst_w HWC RGB at y + out_off[i], nothing else is written.
 *   images / images_dev, x_bytes   as odtk_preprocess_resize_u8;
 *   out_off / out_off_dev          host / device int64 [n] output offsets: the host copy is validated, never read by the
 *                                  kernel; every image must lie in [y, y + y_bytes).
 * Two-phase: y == NULL returns the bytes of the images packed one after another.  ODTK_E_INVALID as
 * odtk_preprocess_resize_u8, or an output outside [y, y + y_bytes).                                                  */
long long odtk_resize_u8_packed(const void *x, size_t x_bytes, const odtk_resize_image_t *images,
                                const odtk_resize_image_t *images_dev, const long long *out_off,
                                const long long *out_off_dev, int n, void *y, size_t y_bytes, odtk_stream_t stream);

#define ODTK_AUGMENT_BRIGHTNESS 1
#define ODTK_AUGMENT_CONTRAST 2
#define ODTK_AUGMENT_HUE 4
#define ODTK_AUGMENT_SATURATION 8

/* One image of odtk_augment_u8. */
typedef struct {
  long long offset;        /* its resized uint8 HWC RGB pixels (h x w) start `offset` bytes into x               */
  int h, w;                /* resized size                                                                       */
  int rot;                 /* Image.rotate(90 * rot), counter-clockwise, 0..3                                     */
  int expand;              /* rotate(..., expand=True): 90 / 270 give a w x h transpose.  0: the size stays h x w  */
                           /* and a non-square image is resampled NEAREST about its centre with black fill        */
  int flip;                /* then Image.FLIP_LEFT_RIGHT                                                          */
  int flags;               /* ODTK_AUGMENT_* adjustments applied, always in the order of the bit values           */
  float brightness;        /* ImageEnhance factors, as the C float Image.blend takes them, >= 0                   */
  float contrast;
  float saturation;
  int hue_shift;           /* 0..255, added modulo 256 to H of the uint8 HSV round trip                           */
} odtk_augment_image_t;

/* The per-image augmentations of CocoDataset / RotatedCocoDataset.__getitem__ (odtk/data.py:64-123) on uint8 images,
 * bit-exact to Pillow and torchvision's PIL functional: rotation, horizontal flip, ImageEnhance.Brightness (blend with
 * black), ImageEnhance.Contrast (blend with the grey int(mean(L) + 0.5), L the fixed-point convert("L") of the image
 * after rotation, flip and brightness, rotation fill included), adjust_hue (convert("HSV"), H += hue_shift,
 * convert("RGB")), ImageEnhance.Color (blend with convert("L")), then the normalisation of odtk_preprocess_u8.  The
 * result is the collated batch y, fp32 [n, canvas_h, canvas_w, 3] (NCHW's channels_last), every pixel outside an
 * image's rotated size exactly 0.0.  Two kernels: L sums (only when an image has ODTK_AUGMENT_CONTRAST), then one
 * thread per canvas pixel.
 *   images / images_dev  host copy (validated, never read by a kernel) / device copy of the n descriptors;
 *   workspace            8 bytes per image (the L sums).
 * Two-phase: workspace == NULL returns the workspace bytes.  ODTK_E_INVALID: a size <= 0, a rotated size larger than
 * the canvas, an image outside [x, x + x_bytes), rot outside 0..3, unknown flags, a negative or NaN factor, a
 * hue_shift outside 0..255; ODTK_E_WORKSPACE: workspace_bytes too small.                                              */
long long odtk_augment_u8(const void *x, size_t x_bytes, const odtk_augment_image_t *images,
                          const odtk_augment_image_t *images_dev, int n, int canvas_h, int canvas_w, void *workspace,
                          size_t workspace_bytes, float *y, const float *mean, const float *std, odtk_stream_t stream);

/* ---- per-kernel timing (H100-native addition; the reference has only a wall-clock
 * Profiler without CUDA sync, odtk/utils.py:140-167) ------------------------------
 * When enabled, every launch of a tagged kernel is bracketed by CUDA events on the
 * launching stream.  Tags: 0 score filter, 1 select+decode, 2 nms, 3 conv, 4 loss / target
 * assignment, 5 pad / max-pool / lowering / preprocess.
 * odtk_prof_get synchronises the device and returns summed ms and launch count.  */
void odtk_prof_enable(int on);
void odtk_prof_reset(void);
int odtk_prof_get(int tag, double *total_ms, long long *launches);
/* per-launch durations (ms) of `tag`, launch order, the last `cap` launches; returns how many were written */
long long odtk_prof_get_list(int tag, float *ms, long long cap);

#ifdef __cplusplus
}
#endif
#endif /* ODTK_B200_H_ */
