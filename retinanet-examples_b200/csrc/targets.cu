// targets.cu -- anchor target assignment for sm_90a.
//
// Replaces snap_to_anchors (reference odtk/box.py:134-186) as called per image and per pyramid level by
// Model._extract_targets (odtk/model.py:167-184): the reference builds the [A*H*W, #gt] IoU matrix, the arg-max, the
// box deltas (box2delta, odtk/box.py:67-78), the depth map and a dense one-hot class tensor with ~25 torch kernels and
// a host-synchronising boolean filter per image.  Here: ONE launch per level for the whole batch, one thread per anchor
// position, ground-truth boxes of the image staged in shared memory, no host sync (padding rows -- class < 0 -- are
// skipped on the device, which is what `target[target[:, -1] > -1]` does on the host).
//
// Outputs, in the reference's layouts: cls_target [B, A, C, H, W] (dense one-hot, optional), box_target [B, A, 4, H, W],
// depth [B, A, 1, H, W] (-1 ignored, 0 background, class + 1 foreground), and -- H100-native -- cls_index [B, A, H, W]
// int32 (class, -1 background, -2 ignored): exactly what odtk_focal_loss consumes, so the dense one-hot never has to
// exist.  Parity: IoU and thresholds in fp32 with the reference's operation order (compiled without FMA contraction,
// IEEE division): depth / classes / arg-max bit-exact; box deltas differ only by logf vs torch.log (<= 1 ulp).
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/odtk_b200.h"
#include "prof.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kMaxAnchors = 32;
constexpr int kChunk = kThreads;   // ground-truth rows staged per pass (one per thread)

struct SnapParams {
  const float *targets;   // [B, G, 5]: x, y, w, h, class (class < 0: padding row)
  float anchors[4 * kMaxAnchors];
  int batch, max_boxes, height, width, stride, num_anchors, num_classes;
  float iou_bg, iou_fg;
  float *cls_target, *box_target, *depth;
  int *cls_index;
};

__global__ void __launch_bounds__(kThreads) snap_to_anchors_kernel(const __grid_constant__ SnapParams p) {
  __shared__ float4 s_box[kChunk];   // x1, y1, x2, y2 (inclusive corners)
  __shared__ float s_area[kChunk];
  __shared__ float s_cls[kChunk];
  __shared__ int s_n;
  __shared__ int s_wcnt[kThreads / 32];
  const int hw = p.height * p.width;
  const int per_img = p.num_anchors * hw;
  const int img = blockIdx.y;
  const int e = blockIdx.x * kThreads + threadIdx.x;   // (a, y, x) within the image
  const bool active = e < per_img;
  const int a = active ? e / hw : 0;
  const int pos = active ? e - a * hw : 0;
  const int y = pos / p.width, x = pos - y * p.width;
  // anchor box at this grid position (odtk/box.py:147-150): (x*stride, y*stride) + anchor corners
  const float gx = (float)(x * p.stride), gy = (float)(y * p.stride);
  const float ax1 = gx + p.anchors[4 * a + 0], ay1 = gy + p.anchors[4 * a + 1];
  const float ax2 = gx + p.anchors[4 * a + 2], ay2 = gy + p.anchors[4 * a + 3];
  const float a_area = (ax2 - ax1 + 1.0f) * (ay2 - ay1 + 1.0f);

  float best = -INFINITY;           // max over the image's boxes, first maximum wins (torch.max semantics)
  float4 bbox = make_float4(0.f, 0.f, 0.f, 0.f);
  float bcls = 0.f;
  bool any = false;
  const float *t = p.targets + (long long)img * p.max_boxes * 5;
  for (int g0 = 0; g0 < p.max_boxes; g0 += kChunk) {
    __syncthreads();
    // stage the valid rows of this chunk, compacted IN THEIR ORIGINAL ORDER (the first-maximum rule depends on it):
    // thread i owns row g0 + i; ballot + warp-count prefix gives every valid row its slot
    {
      const int g = g0 + (int)threadIdx.x;
      float bx = 0.f, by = 0.f, bw = 0.f, bh = 0.f, c = -1.0f;
      if (g < p.max_boxes) {
        c = t[g * 5 + 4];
        bx = t[g * 5 + 0]; by = t[g * 5 + 1]; bw = t[g * 5 + 2]; bh = t[g * 5 + 3];
      }
      const bool valid = c > -1.0f;                                     // odtk/model.py:174
      const unsigned m = __ballot_sync(0xffffffffu, valid);
      const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
      if (lane == 0) s_wcnt[wid] = __popc(m);
      __syncthreads();
      int off = 0;
      for (int w = 0; w < wid; w++) off += s_wcnt[w];
      if (valid) {
        const int slot = off + __popc(m & ((1u << lane) - 1u));
        const float x2 = bx + bw - 1.0f, y2 = by + bh - 1.0f;          // odtk/box.py:153
        s_box[slot] = make_float4(bx, by, x2, y2);
        s_area[slot] = (x2 - bx + 1.0f) * (y2 - by + 1.0f);             // :157
        s_cls[slot] = c;
      }
      if (threadIdx.x == 0) {
        int n = 0;
        for (int w = 0; w < kThreads / 32; w++) n += s_wcnt[w];
        s_n = n;
      }
    }
    __syncthreads();
    const int n = s_n;
    for (int j = 0; j < n; j++) {
      const float4 b = s_box[j];
      const float ix = fmaxf(fminf(ax2, b.z) - fmaxf(ax1, b.x) + 1.0f, 0.0f);   // :154-156
      const float iy = fmaxf(fminf(ay2, b.w) - fmaxf(ay1, b.y) + 1.0f, 0.0f);
      const float inter = ix * iy;
      const float ov = inter / (a_area + s_area[j] - inter);                     // :159
      if (!any || ov > best) { best = ov; bbox = b; bcls = s_cls[j]; any = true; }
    }
  }
  if (!active) return;

  const long long base = (long long)img * per_img;
  float dep = 0.0f, d0 = 0.f, d1 = 0.f, d2 = 0.f, d3 = 0.f;
  int cidx = -1;                      // no boxes at all: everything zero (odtk/box.py:140-143)
  int onehot = -1;
  if (any) {
    // box2delta (odtk/box.py:67-78)
    const float aw = ax2 - ax1 + 1.0f, ah = ay2 - ay1 + 1.0f;
    const float acx = ax1 + 0.5f * aw, acy = ay1 + 0.5f * ah;
    const float bw = bbox.z - bbox.x + 1.0f, bh = bbox.w - bbox.y + 1.0f;
    const float bcx = bbox.x + 0.5f * bw, bcy = bbox.y + 0.5f * bh;
    d0 = (bcx - acx) / aw;
    d1 = (bcy - acy) / ah;
    d2 = logf(bw / aw);
    d3 = logf(bh / ah);
    const int cls = (int)bcls;        // .long() truncation (:176)
    dep = -1.0f;                                                       // :167-169
    if (best < p.iou_bg) dep = 0.0f;
    if (best >= p.iou_fg) dep = bcls + 1.0f;
    onehot = (best < p.iou_bg) ? -1 : cls;                             // :178-179 (ignored anchors keep their one-hot)
    cidx = (best < p.iou_bg) ? -1 : (best >= p.iou_fg ? cls : -2);
  }
  p.depth[base + e] = dep;
  float *bt = p.box_target + ((long long)img * p.num_anchors + a) * 4 * hw + pos;
  bt[0] = d0; bt[hw] = d1; bt[2 * hw] = d2; bt[3 * hw] = d3;
  if (p.cls_index) p.cls_index[base + e] = cidx;
  if (p.cls_target) {
    float *ct = p.cls_target + ((long long)img * p.num_anchors + a) * p.num_classes * hw + pos;
    for (int c = 0; c < p.num_classes; c++) ct[(long long)c * hw] = (c == onehot) ? 1.0f : 0.0f;
  }
}

}  // namespace

extern "C" int odtk_snap_to_anchors(const float *targets, int batch, int max_boxes, int height, int width, int stride,
                                    const float *anchors, int num_anchors, int num_classes, float iou_bg, float iou_fg,
                                    float *cls_target, float *box_target, float *depth, int *cls_index,
                                    odtk_stream_t stream_) {
  if (!box_target || !depth || !anchors) return ODTK_E_INVALID;
  if (batch <= 0 || height <= 0 || width <= 0 || stride <= 0 || num_anchors <= 0 || num_classes <= 0 || max_boxes < 0)
    return ODTK_E_INVALID;
  if (max_boxes > 0 && !targets) return ODTK_E_INVALID;
  if (num_anchors > kMaxAnchors) return ODTK_E_UNSUPPORTED;
  if ((long long)num_anchors * height * width >= (1ll << 31)) return ODTK_E_UNSUPPORTED;
  SnapParams p;
  p.targets = targets;
  for (int i = 0; i < 4 * num_anchors; i++) p.anchors[i] = anchors[i];
  p.batch = batch; p.max_boxes = max_boxes; p.height = height; p.width = width; p.stride = stride;
  p.num_anchors = num_anchors; p.num_classes = num_classes; p.iou_bg = iou_bg; p.iou_fg = iou_fg;
  p.cls_target = cls_target; p.box_target = box_target; p.depth = depth; p.cls_index = cls_index;
  const int per_img = num_anchors * height * width;
  dim3 grid((unsigned)((per_img + kThreads - 1) / kThreads), (unsigned)batch);
  cudaStream_t stream = (cudaStream_t)stream_;
  {
    OdtkProfScope prof(ODTK_PROF_LOSS, stream);
    snap_to_anchors_kernel<<<grid, kThreads, 0, stream>>>(p);
  }
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}
