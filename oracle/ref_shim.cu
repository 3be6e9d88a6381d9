// oracle/ref_shim.cu -- TEST INFRASTRUCTURE ONLY.
//
// extern "C" doors onto the reference's own CUDA entry points
// (odtk::cuda::decode / decode_rotate / nms / nms_rotate,
// /root/reference/csrc/cuda/{decode,decode_rotate,nms,nms_iou}.h).  The four
// reference .cu files are compiled, unmodified, from where they lie under
// /root/reference by oracle/Makefile into oracle/_ref/libodtk_ref.so; no
// reference source is copied into this repository.  The result is (a) the GPU
// oracle the -m gpu parity tests pin against and (b) the "reference csrc/cuda
// plugins recompiled for sm_90a" comparator of BASELINE.json configs[1]/[4].
#include <cuda_runtime.h>
#include <vector>
#include "decode.h"
#include "decode_rotate.h"
#include "nms.h"
#include "nms_iou.h"

extern "C" {

long long ref_decode(int batch, const void *scores, const void *deltas, void *out_scores,
                     void *out_boxes, void *out_classes, int height, int width, int scale,
                     int num_anchors, int num_classes, const float *anchors, int n_anchor_floats,
                     float thresh, int top_n, int rotated, void *workspace, long long workspace_size,
                     cudaStream_t stream) {
  std::vector<float> a(anchors, anchors + n_anchor_floats);
  const void *inputs[2] = {scores, deltas};
  void *outputs[3] = {out_scores, out_boxes, out_classes};
  try {
    if (rotated)
      return odtk::cuda::decode_rotate(batch, workspace ? inputs : nullptr, workspace ? outputs : nullptr,
                                       height, width, scale, num_anchors, num_classes, a, thresh, top_n,
                                       workspace, (size_t)workspace_size, stream);
    return odtk::cuda::decode(batch, workspace ? inputs : nullptr, workspace ? outputs : nullptr, height,
                              width, scale, num_anchors, num_classes, a, thresh, top_n, workspace,
                              (size_t)workspace_size, stream);
  } catch (...) { return -1; }
}

long long ref_nms(int batch, const void *scores, const void *boxes, const void *classes,
                  void *out_scores, void *out_boxes, void *out_classes, int count, int detections,
                  float thresh, int rotated, void *workspace, long long workspace_size,
                  cudaStream_t stream) {
  const void *inputs[3] = {scores, boxes, classes};
  void *outputs[3] = {out_scores, out_boxes, out_classes};
  try {
    if (rotated)
      return odtk::cuda::nms_rotate(batch, workspace ? inputs : nullptr, workspace ? outputs : nullptr,
                                    count, detections, thresh, workspace, (size_t)workspace_size, stream);
    return odtk::cuda::nms(batch, workspace ? inputs : nullptr, workspace ? outputs : nullptr, count,
                           detections, thresh, workspace, (size_t)workspace_size, stream);
  } catch (...) { return -1; }
}

// odtk::cuda::iou (nms_iou.h:33-35): boxes / anchors as corner lists [n, 4, 2], out [num_anchors, num_boxes]
long long ref_iou(const void *boxes, const void *anchors, void *out, int num_boxes, int num_anchors, cudaStream_t stream) {
  const void *inputs[2] = {boxes, anchors};
  void *outputs[1] = {out};
  try {
    return odtk::cuda::iou(inputs, outputs, num_boxes, num_anchors, stream);
  } catch (...) { return -1; }
}

}  // extern "C"
