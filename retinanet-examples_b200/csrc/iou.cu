// iou.cu -- polygon IoU of rotated target boxes against rotated anchors for sm_90a.
//
// Replaces odtk::cuda::iou + iou_cuda_kernel (reference csrc/cuda/nms_iou.cu:324-387, declared nms_iou.h:33-35), the
// kernel behind odtk._C.iou (csrc/extensions.cpp:47-67) that snap_to_anchors_rotated (odtk/box.py:218) uses to match
// ground-truth boxes to anchors during rotated-box training.  Both inputs are lists of quadrilaterals, 4 corners x
// (x, y) fp32 each; the output is [num_anchors, num_boxes].
//
// Quirk kept (nms_iou.cu:385): the host entry point hands (num_anchors, num_boxes, anchors, boxes) to a kernel whose
// parameters are named (numBoxes, numAnchors, b_box_vals, a_box_vals).  Net effect, restated here directly: element
// [a, j] clips ANCHOR a (jittered by 0.001 where a coordinate coincides with the same corner of box j) against the
// four edges of BOX j.  One thread per (anchor, box) pair; the boxes (few: one image's ground truth) sit in shared
// memory, anchor loads are coalesced 32-byte rows.
#include "common.cuh"
#include "polygon.cuh"
#include "prof.cuh"

namespace {

constexpr int kBoxTile = 64;   // ground-truth quads staged per pass

__global__ void __launch_bounds__(256) iou_kernel(const float *__restrict__ boxes, const float *__restrict__ anchors,
                                                   float *__restrict__ out, int num_boxes, int num_anchors) {
  __shared__ float sbox[kBoxTile][8];
  for (int j0 = 0; j0 < num_boxes; j0 += kBoxTile) {
    const int nb = min(kBoxTile, num_boxes - j0);
    __syncthreads();
    for (int i = threadIdx.x; i < nb * 8; i += blockDim.x) sbox[i >> 3][i & 7] = boxes[(long long)j0 * 8 + i];
    __syncthreads();
    for (long long a = (long long)blockIdx.x * blockDim.x + threadIdx.x; a < num_anchors; a += (long long)gridDim.x * blockDim.x) {
      const float4 a0 = __ldg(reinterpret_cast<const float4 *>(anchors + a * 8));
      const float4 a1 = __ldg(reinterpret_cast<const float4 *>(anchors + a * 8) + 1);
      const f2 rect1[4] = {{a0.x, a0.y}, {a0.z, a0.w}, {a1.x, a1.y}, {a1.z, a1.w}};
      float area1 = 0.0f;
#pragma unroll
      for (int k = 0; k < 4; k++) area1 += rect1[k].x * rect1[(k + 1) & 3].y - rect1[k].y * rect1[(k + 1) & 3].x;
      for (int j = 0; j < nb; j++) {
        f2 rect2[4], inter[8];
        float area2 = 0.0f;
#pragma unroll
        for (int b = 0; b < 4; b++) { rect2[b].x = sbox[j][2 * b]; rect2[b].y = sbox[j][2 * b + 1]; }
#pragma unroll
        for (int b = 0; b < 4; b++) {
          inter[b].x = rect1[b].x + ((rect1[b].x == rect2[b].x) ? 0.001f : 0.0f);
          inter[b].y = rect1[b].y + ((rect1[b].y == rect2[b].y) ? 0.001f : 0.0f);
          inter[4 + b].x = -1.0f; inter[4 + b].y = -1.0f;
          area2 += rect2[b].x * rect2[(b + 1) & 3].y - rect2[b].y * rect2[(b + 1) & 3].x;
        }
        const float ia = intersection_area(rect2, inter);
        const float ua = (fabsf(area1) + fabsf(area2)) / 2.0f;
        float v;
        if (isnan(ia) && isnan(ua)) v = 1.0f;
        else if (isnan(ia)) v = 0.0f;
        else v = ia / (ua - ia);
        out[a * num_boxes + j0 + j] = v;
      }
    }
  }
}

}  // namespace

extern "C" int odtk_iou(const void *const *inputs, void *const *outputs, int num_boxes, int num_anchors,
                        odtk_stream_t stream_) {
  if (!inputs || !outputs || !inputs[0] || !inputs[1] || !outputs[0]) return ODTK_E_INVALID;
  if (num_boxes < 0 || num_anchors < 0) return ODTK_E_INVALID;
  if (num_boxes == 0 || num_anchors == 0) return ODTK_OK;
  if (((uintptr_t)inputs[1]) & 15) return ODTK_E_INVALID;   // anchors are read as 16-byte vectors
  cudaStream_t stream = (cudaStream_t)stream_;
  long long blocks = ((long long)num_anchors + 255) / 256;
  const long long cap = (long long)odtk_sm_count() * 8;
  if (blocks > cap) blocks = cap;
  {
    OdtkProfScope prof(ODTK_PROF_LOSS, stream);
    iou_kernel<<<(int)blocks, 256, 0, stream>>>((const float *)inputs[0], (const float *)inputs[1], (float *)outputs[0],
                                                num_boxes, num_anchors);
  }
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}
