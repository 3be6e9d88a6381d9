/*
 * oracle/odtk_oracle.c -- TEST INFRASTRUCTURE ONLY.
 *
 * A plain-C, single-threaded, IEEE-754 (no FMA contraction, no fast-math)
 * restatement of the post-processing half of the ODTK inference hot path.
 * It exists so that tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline leg can check / time the CUDA product path against it.
 * Nothing in the product package may import, link or call this file.
 *
 * Each function cites the reference file:line it follows.  Where the
 * reference's CUDA and CPU paths disagree the CUDA
 * semantics are followed with IEEE arithmetic and stable ordering.
 *
 * Pinning status: decode / nms are pinned by fixtures generated from the
 * reference's own Python (tests/golden/, made by oracle/gen_golden.py) and, on
 * the GPU box, by the reference's own .cu files built into oracle/_ref.
 * nms_rotate has no runnable CPU reference (odtk/box.py:408 NameError); it is
 * pinned only by oracle/_ref on the GPU box.
 *
 * Build: gcc -O2 -ffp-contract=off -fno-fast-math -shared -fPIC (oracle/Makefile)
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------------- */
/* key transform used by cub::DeviceRadixSort for float keys (descending,   */
/* stable): larger key == sorts earlier.  nms.cu:135-137, decode.cu:111-112  */
static inline uint32_t float_key(float f) {
  uint32_t b;
  memcpy(&b, &f, 4);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

typedef struct {
  uint32_t key;
  int32_t idx;
  int32_t pos; /* position in the compacted list: the stable tie-break */
} cand_t;

static int cand_cmp_desc(const void *a, const void *b) {
  const cand_t *x = (const cand_t *)a, *y = (const cand_t *)b;
  if (x->key != y->key) return x->key > y->key ? -1 : 1;
  return x->pos < y->pos ? -1 : (x->pos > y->pos ? 1 : 0);
}

/* ------------------------------------------------------------------------- */
/* decode / decode_rotate: csrc/cuda/decode.cu:86-168,                        */
/* csrc/cuda/decode_rotate.cu:83-176.  nbox = 4 (axis aligned) or 6 (rotated) */
/* Layouts: scores [B, A*C, H, W], deltas [B, A*nbox, H, W], fp32 contiguous. */
/* anchors: num_anchors_floats = 4*A floats or 0 (no anchors: raw deltas).   */
/* Outputs [B, top_n], [B, top_n, nbox], [B, top_n]; must be pre-zeroed like  */
/* torch::zeros does in csrc/extensions.cpp:83-85 (box tails stay untouched). */
int oracle_decode(int batch, const float *scores, const float *deltas,
                  int height, int width, int scale, int num_anchors,
                  int num_classes, const float *anchors, int num_anchor_floats,
                  float score_thresh, int top_n, int nbox, float *out_scores,
                  float *out_boxes, float *out_classes) {
  const int64_t n = (int64_t)num_anchors * num_classes * height * width;
  cand_t *cand = (cand_t *)malloc(sizeof(cand_t) * (size_t)(n > 0 ? n : 1));
  if (!cand) return -1;
  for (int b = 0; b < batch; b++) {
    const float *s = scores + (int64_t)b * n;
    const float *d = deltas + (int64_t)b * (n / num_classes) * nbox;
    float *os = out_scores + (int64_t)b * top_n;
    float *ob = out_boxes + (int64_t)b * top_n * nbox;
    float *oc = out_classes + (int64_t)b * top_n;
    /* decode.cu:96-104: strict '>' threshold, ascending flat index */
    int64_t cnt = 0;
    for (int64_t i = 0; i < n; i++) {
      if (s[i] > score_thresh) {
        cand[cnt].key = float_key(s[i]);
        cand[cnt].idx = (int32_t)i;
        cand[cnt].pos = (int32_t)cnt;
        cnt++;
      }
    }
    /* decode.cu:108-115: only when count > top_n, stable sort descending */
    if (cnt > top_n) {
      qsort(cand, (size_t)cnt, sizeof(cand_t), cand_cmp_desc);
      cnt = top_n;
    }
    for (int64_t k = 0; k < cnt; k++) {
      /* decode.cu:122-131 index math (int32) */
      int i = cand[k].idx;
      int x = i % width;
      int y = (i / width) % height;
      int a = (i / num_classes / height / width) % num_anchors;
      int cls = (i / height / width) % num_classes;
      float box[6];
      for (int c = 0; c < nbox; c++)
        box[c] = d[((int64_t)(a * nbox + c) * height + y) * width + x];
      if (num_anchor_floats > 0) {
        /* decode.cu:133-156 */
        float fx = (float)((int64_t)x * scale);
        float fy = (float)((int64_t)y * scale);
        const float *an = anchors + 4 * a; /* decode_rotate.cu:139: 4*a too */
        float x1 = fx + an[0];
        float y1 = fy + an[1];
        float x2 = fx + an[2];
        float y2 = fy + an[3];
        float w = x2 - x1 + 1.0f;
        float h = y2 - y1 + 1.0f;
        float pred_ctr_x = box[0] * w + x1 + 0.5f * w;
        float pred_ctr_y = box[1] * h + y1 + 0.5f * h;
        float pred_w = expf(box[2]) * w;
        float pred_h = expf(box[3]) * h;
        float bx1 = fmaxf(0.0f, pred_ctr_x - 0.5f * pred_w);
        float by1 = fmaxf(0.0f, pred_ctr_y - 0.5f * pred_h);
        float bx2 = fminf(pred_ctr_x + 0.5f * pred_w - 1.0f,
                          (float)((int64_t)width * scale) - 1.0f);
        float by2 = fminf(pred_ctr_y + 0.5f * pred_h - 1.0f,
                          (float)((int64_t)height * scale) - 1.0f);
        box[0] = bx1; box[1] = by1; box[2] = bx2; box[3] = by2;
        /* rotated: sin, cos pass through (decode_rotate.cu:152-163) */
      }
      os[k] = s[i];
      for (int c = 0; c < nbox; c++) ob[k * nbox + c] = box[c];
      oc[k] = (float)cls;
    }
    /* decode.cu:162-167: zero tails of scores / classes only */
    for (int64_t k = cnt; k < top_n; k++) { os[k] = 0.0f; oc[k] = 0.0f; }
  }
  free(cand);
  return 0;
}

/* ------------------------------------------------------------------------- */
/* Rotated-rectangle IoU exactly as csrc/cuda/nms_iou.cu:44-169,199-248.     */
typedef struct { float x, y; } f2;
typedef struct { float a, b, c; } line_t;

static inline line_t make_line(f2 v1, f2 v2) { /* nms_iou.cu:87 */
  line_t l;
  l.a = v2.y - v1.y;
  l.b = v1.x - v2.x;
  l.c = v2.x * v1.y - v2.y * v1.x; /* v2.cross(v1), nms_iou.cu:66-68 */
  return l;
}
static inline float line_call(line_t l, f2 v) { /* nms_iou.cu:89-91 */
  return l.a * v.x + l.b * v.y + l.c;
}
static inline f2 line_isect(line_t l, line_t o) { /* nms_iou.cu:93-96 */
  float w = l.a * o.b - l.b * o.a;
  f2 r;
  r.x = (l.b * o.c - l.c * o.b) / w;
  r.y = (l.c * o.a - l.a * o.c) / w;
  return r;
}

#define KPTS 8
/* nms_iou.cu:114-169.  NOTE: the reference can write past new_intersection[8]
 * when both pushes fire for >4 points; we stop at 8 (documented deviation on
 * inputs where the reference is undefined). */
static float intersection_area(const f2 *mrect, const f2 *mrect_shift, f2 *inter) {
  int count = 4;
  for (int i = 0; i < 4; i++) {
    f2 inter_shift[KPTS];
    float lv[KPTS], lvs[KPTS];
    memset(inter_shift, 0, sizeof inter_shift);
    memset(lv, 0, sizeof lv);
    for (int k = 0; k < count; k++) inter_shift[k] = inter[k];
    line_t l1 = make_line(mrect[i], mrect_shift[i]);
    for (int j = 0; j < count; j++) lv[j] = line_call(l1, inter[j]);
    for (int k = 0; k < KPTS; k++) lvs[k] = lv[k];
    { /* rotateLeft(count) on both */
      float t = lvs[0];
      for (int k = 0; k < count - 1; k++) lvs[k] = lvs[k + 1];
      lvs[count - 1] = t;
      f2 t2 = inter_shift[0];
      for (int k = 0; k < count - 1; k++) inter_shift[k] = inter_shift[k + 1];
      inter_shift[count - 1] = t2;
    }
    f2 nw[KPTS];
    memset(nw, 0, sizeof nw);
    int temp = count;
    count = 0;
    for (int j = 0; j < temp; j++) {
      if (lv[j] <= 0) {
        if (count < KPTS) nw[count] = inter[j];
        count++;
      }
      if ((lv[j] * lvs[j]) <= 0) {
        line_t l2 = make_line(inter[j], inter_shift[j]);
        if (count < KPTS) nw[count] = line_isect(l1, l2);
        count++;
      }
    }
    if (count > KPTS) count = KPTS;
    for (int k = 0; k < count; k++) inter[k] = nw[k];
  }
  f2 sh[KPTS];
  memset(sh, 0, sizeof sh);
  for (int k = 0; k < count; k++) sh[k] = inter[k];
  if (count > 0) {
    f2 t = sh[0];
    for (int k = 0; k < count - 1; k++) sh[k] = sh[k + 1];
    sh[count - 1] = t;
  }
  float area = 0.0f;
  if (count > 2)
    for (int k = 0; k < count; k++)
      area += inter[k].x * sh[k].y - inter[k].y * sh[k].x;
  return fabsf(area / 2.0f);
}

/* nms_iou.cu:182-248.  ib, mb: (x1,y1,x2,y2,sin,cos).  fixed_angle == 0
 * reproduces the reference quirk (the max box is rotated with the CANDIDATE's
 * sin/cos, nms_iou.cu:188-192); fixed_angle == 1 uses the max box's own. */
float oracle_rotated_overlap(const float *ib, const float *mb, int fixed_angle) {
  float is = ib[4], ic = ib[5];
  float ms = fixed_angle ? mb[4] : ib[4], mc = fixed_angle ? mb[5] : ib[5];
  f2 inter[KPTS], irect[4], irect_s[4], mrect[4], mrect_s[4];
  for (int k = 0; k < KPTS; k++) { inter[k].x = -1.0f; inter[k].y = -1.0f; }
  f2 icent = {(ib[0] + ib[2]) / 2.0f, (ib[1] + ib[3]) / 2.0f};
  f2 mcent = {(mb[0] + mb[2]) / 2.0f, (mb[1] + mb[3]) / 2.0f};
  f2 iboxc[4] = {{ib[0] - icent.x, ib[1] - icent.y}, {ib[2] - icent.x, ib[1] - icent.y},
                 {ib[2] - icent.x, ib[3] - icent.y}, {ib[0] - icent.x, ib[3] - icent.y}};
  f2 mboxc[4] = {{mb[0] - mcent.x, mb[1] - mcent.y}, {mb[2] - mcent.x, mb[1] - mcent.y},
                 {mb[2] - mcent.x, mb[3] - mcent.y}, {mb[0] - mcent.x, mb[3] - mcent.y}};
  for (int b = 0; b < 4; b++) {
    float ix = (iboxc[b].x * ic - iboxc[b].y * is) + icent.x;
    float iy = (iboxc[b].y * ic + iboxc[b].x * is) + icent.y;
    float mx = (mboxc[b].x * mc - mboxc[b].y * ms) + mcent.x;
    float my = (mboxc[b].y * mc + mboxc[b].x * ms) + mcent.y;
    float px = (ix == mx) ? 0.001f : 0.0f; /* nms_iou.cu:210-217 */
    float py = (iy == my) ? 0.001f : 0.0f;
    inter[b].x = ix + px; inter[b].y = iy + py;
    irect[b].x = ix; irect[b].y = iy;
    mrect[b].x = mx; mrect[b].y = my;
  }
  for (int b = 0; b < 4; b++) { irect_s[b] = irect[(b + 1) & 3]; mrect_s[b] = mrect[(b + 1) & 3]; }
  float ia = intersection_area(mrect, mrect_s, inter);
  float irect_area = 0.0f, mrect_area = 0.0f;
  for (int k = 0; k < 4; k++) {
    irect_area += irect[k].x * irect_s[k].y - irect[k].y * irect_s[k].x;
    mrect_area += mrect[k].x * mrect_s[k].y - mrect[k].y * mrect_s[k].x;
  }
  float ua = (fabsf(irect_area) + fabsf(mrect_area)) / 2.0f;
  float overlap;
  if (isnan(ia) && isnan(ua)) overlap = 1.0f;
  else if (isnan(ia)) overlap = 0.0f;
  else overlap = ia / (ua - ia);
  return overlap;
}

/* iou_cuda_kernel + its host entry point (nms_iou.cu:324-387).  The host function passes
 * (num_anchors, num_boxes, anchors, boxes) into kernel parameters named (numBoxes, numAnchors,
 * b_box_vals, a_box_vals) -- nms_iou.cu:385 -- so, in terms of the REAL boxes and anchors:
 * out[a * nb + j]: rect1 = anchor a (the polygon that is clipped, jittered where equal to the
 * same corner of box j, :341-349), rect2 = box j (the clip rectangle, :359).                   */
void oracle_iou(const float *boxes, const float *anchors, int nb, int na, float *out) {
  for (int a = 0; a < na; a++) {
    for (int j = 0; j < nb; j++) {
      f2 inter[KPTS], rect1[4], rect1_s[4], rect2[4], rect2_s[4];
      for (int k = 0; k < KPTS; k++) { inter[k].x = -1.0f; inter[k].y = -1.0f; }
      for (int b = 0; b < 4; b++) {
        f2 pa = {anchors[(a * 4 + b) * 2], anchors[(a * 4 + b) * 2 + 1]};
        f2 pb = {boxes[(j * 4 + b) * 2], boxes[(j * 4 + b) * 2 + 1]};
        float px = (pa.x == pb.x) ? 0.001f : 0.0f;
        float py = (pa.y == pb.y) ? 0.001f : 0.0f;
        inter[b].x = pa.x + px; inter[b].y = pa.y + py;
        rect1[b] = pa;
        rect2[b] = pb;
      }
      for (int b = 0; b < 4; b++) { rect1_s[b] = rect1[(b + 1) & 3]; rect2_s[b] = rect2[(b + 1) & 3]; }
      float ia = intersection_area(rect2, rect2_s, inter);
      float a1 = 0.0f, a2 = 0.0f;
      for (int k = 0; k < 4; k++) {
        a1 += rect1[k].x * rect1_s[k].y - rect1[k].y * rect1_s[k].x;
        a2 += rect2[k].x * rect2_s[k].y - rect2[k].y * rect2_s[k].x;
      }
      float ua = (fabsf(a1) + fabsf(a2)) / 2.0f;
      float v;
      if (isnan(ia) && isnan(ua)) v = 1.0f;
      else if (isnan(ia)) v = 0.0f;
      else v = ia / (ua - ia);
      out[(int64_t)a * nb + j] = v;
    }
  }
}

/* nms.cu:57-69 */
float oracle_aligned_overlap(const float *ib, const float *mb) {
  float x1 = fmaxf(ib[0], mb[0]);
  float y1 = fmaxf(ib[1], mb[1]);
  float x2 = fminf(ib[2], mb[2]);
  float y2 = fminf(ib[3], mb[3]);
  float w = fmaxf(0.0f, x2 - x1 + 1);
  float h = fmaxf(0.0f, y2 - y1 + 1);
  float iarea = (ib[2] - ib[0] + 1) * (ib[3] - ib[1] + 1);
  float marea = (mb[2] - mb[0] + 1) * (mb[3] - mb[1] + 1);
  float inter = w * h;
  return inter / (iarea + marea - inter);
}

/* ------------------------------------------------------------------------- */
/* nms / nms_rotate: csrc/cuda/nms.cu:115-157 + nms_kernel :44-80;            */
/* csrc/cuda/nms_iou.cu:283-319 + nms_rotate_kernel :171-258.                 */
/* Inputs [B,count], [B,count,nbox], [B,count]; outputs [B,D], [B,D,nbox],    */
/* [B,D] pre-zeroed (extensions.cpp:128-130).  out_index (may be NULL)        */
/* receives the input position of every emitted entry (-1 for empty slots):   */
/* this is the "kept indices" vector the parity bar is bit-exact on.          */
int oracle_nms(int batch, const float *scores, const float *boxes,
               const float *classes, int count, int detections_per_im,
               float nms_thresh, int nbox, int fixed_angle, float *out_scores,
               float *out_boxes, float *out_classes, int32_t *out_index) {
  cand_t *cand = (cand_t *)malloc(sizeof(cand_t) * (size_t)(count > 0 ? count : 1));
  float *sc = (float *)malloc(sizeof(float) * (size_t)(count > 0 ? count : 1));
  if (!cand || !sc) return -1;
  for (int b = 0; b < batch; b++) {
    const float *s = scores + (int64_t)b * count;
    const float *bx = boxes + (int64_t)b * count * nbox;
    const float *cl = classes + (int64_t)b * count;
    float *os = out_scores + (int64_t)b * detections_per_im;
    float *ob = out_boxes + (int64_t)b * detections_per_im * nbox;
    float *oc = out_classes + (int64_t)b * detections_per_im;
    int32_t *oi = out_index ? out_index + (int64_t)b * detections_per_im : 0;
    if (oi) for (int k = 0; k < detections_per_im; k++) oi[k] = -1;
    /* nms.cu:125-132: drop scores <= 0 */
    int n = 0;
    for (int i = 0; i < count; i++)
      if (s[i] > 0.0f) { cand[n].key = float_key(s[i]); cand[n].idx = i; cand[n].pos = n; n++; }
    /* nms.cu:135-137: stable sort descending */
    qsort(cand, (size_t)n, sizeof(cand_t), cand_cmp_desc);
    for (int i = 0; i < n; i++) sc[i] = s[cand[i].idx];
    /* nms_kernel (nms.cu:49-79): serial greedy, class-gated */
    for (int m = 0; m < n; m++) {
      if (!(sc[m] > 0.0f)) continue;
      int mi = cand[m].idx;
      int mcls = (int)cl[mi];
      for (int i = m + 1; i < n; i++) {
        int ii = cand[i].idx;
        int icls = (int)cl[ii];
        if (mcls != icls) continue;
        float ov = (nbox == 4)
                       ? oracle_aligned_overlap(bx + (int64_t)ii * 4, bx + (int64_t)mi * 4)
                       : oracle_rotated_overlap(bx + (int64_t)ii * 6, bx + (int64_t)mi * 6, fixed_angle);
        if (ov > nms_thresh) sc[i] = 0.0f;
      }
    }
    /* nms.cu:146-147: stable re-sort by updated score (kept first, then the
     * suppressed zeros, each group in its previous order) */
    for (int i = 0; i < n; i++) { cand[i].key = float_key(sc[i]); cand[i].pos = i; }
    /* keep sc aligned with cand through the sort by re-reading afterwards */
    cand_t *tmp = (cand_t *)malloc(sizeof(cand_t) * (size_t)(n > 0 ? n : 1));
    float *sc2 = (float *)malloc(sizeof(float) * (size_t)(n > 0 ? n : 1));
    if (!tmp || !sc2) return -1;
    memcpy(tmp, cand, sizeof(cand_t) * (size_t)n);
    qsort(tmp, (size_t)n, sizeof(cand_t), cand_cmp_desc);
    for (int i = 0; i < n; i++) sc2[i] = sc[tmp[i].pos];
    /* nms.cu:150-156: first min(D, n) entries; boxes/classes gathered even
     * for suppressed (score 0) entries */
    int nd = n < detections_per_im ? n : detections_per_im;
    for (int k = 0; k < nd; k++) {
      int src = tmp[k].idx;
      os[k] = sc2[k];
      for (int c = 0; c < nbox; c++) ob[k * nbox + c] = bx[(int64_t)src * nbox + c];
      oc[k] = cl[src];
      if (oi) oi[k] = src;
    }
    for (int k = nd; k < detections_per_im; k++) os[k] = 0.0f;
    free(tmp);
    free(sc2);
  }
  free(cand);
  free(sc);
  return 0;
}

/* ------------------------------------------------------------------------- */
/* Focal loss forward + analytic backward: odtk/loss.py:13-18 as used by      */
/* odtk/model.py:195-199.  target holds one-hot {0,1}; mask multiplies the   */
/* loss (depth >= 0).  Returns the masked SUM in double; grad = d sum / dx    */
/* times grad_scale.  Written in double for the maths, fp32 for the storage.  */
double oracle_focal_loss(const float *logits, const float *target, const float *mask,
                         int64_t n, float alpha, float gamma, float grad_scale,
                         float *loss_out, float *grad_out) {
  double total = 0.0;
  for (int64_t i = 0; i < n; i++) {
    double x = logits[i], t = target[i], m = mask ? mask[i] : 1.0;
    double p = 1.0 / (1.0 + exp(-x));
    double ce = fmax(x, 0.0) - x * t + log1p(exp(-fabs(x)));
    double a = t * alpha + (1.0 - t) * (1.0 - alpha);
    double pt = (t == 1.0) ? p : 1.0 - p;
    double w = pow(1.0 - pt, gamma);
    double l = a * w * ce;
    if (loss_out) loss_out[i] = (float)(m * l);
    total += m * l;
    if (grad_out) {
      /* d(1-pt)/dx = (t==1 ? -1 : +1) * p(1-p);  dce/dx = p - t */
      double dq = ((t == 1.0) ? -1.0 : 1.0) * p * (1.0 - p);
      double q = 1.0 - pt;
      double dw = (gamma == 0.0) ? 0.0 : gamma * pow(q, gamma - 1.0) * dq;
      grad_out[i] = (float)(m * a * (dw * ce + w * (p - t)) * grad_scale);
    }
  }
  return total;
}

/* ------------------------------------------------------------------------- */
/* Smooth L1 forward + analytic backward: odtk/loss.py:27-31.                  */
double oracle_smooth_l1(const float *pred, const float *target, const float *mask, int64_t n, float beta,
                        float grad_scale, float *loss_out, float *grad_out) {
  double total = 0.0;
  for (int64_t i = 0; i < n; i++) {
    double d = (double)pred[i] - (double)target[i], x = fabs(d), m = mask ? mask[i] : 1.0;
    double l = (x >= beta) ? x - 0.5 * beta : 0.5 * x * x / beta;
    if (loss_out) loss_out[i] = (float)(m * l);
    total += m * l;
    if (grad_out) grad_out[i] = (float)(m * grad_scale * ((x >= beta) ? (d > 0 ? 1.0 : (d < 0 ? -1.0 : 0.0)) : d / beta));
  }
  return total;
}

/* ------------------------------------------------------------------------- */
/* Input normalisation + stride padding: odtk/data.py:113-123 (float32 maths). */
/* x: uint8 [h, w, 3]; out: float32 [3, hs, ws] (CHW like the reference).      */
void oracle_preprocess_u8(const uint8_t *x, int h, int w, int hs, int ws, const float *mean, const float *std,
                          float *out) {
  for (int c = 0; c < 3; c++)
    for (int y = 0; y < hs; y++)
      for (int xx = 0; xx < ws; xx++) {
        float v = 0.0f;
        if (y < h && xx < w) v = ((float)x[((size_t)y * w + xx) * 3 + c] / 255.0f - mean[c]) / std[c];
        out[((size_t)c * hs + y) * ws + xx] = v;
      }
}
