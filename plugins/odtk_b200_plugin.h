// odtk_b200_plugin.h -- TensorRT-plugin-shaped wrappers over the C ABI of the H100 hot path (include/odtk_b200.h).
//
// The reference's TensorRT plugins are thin shells around odtk::cuda::decode / nms: their
// configurePlugin() reads the geometry off the input descriptors, getWorkspaceSize() is the size query of the same
// function, enqueue() is the call itself (csrc/plugins/DecodePlugin.h:141-161,177-191; DecodeRotatePlugin.h; NMSPlugin.h:120-138;
// NMSRotatePlugin.h).  The C ABI keeps exactly that contract (two-phase workspace, caller-owned buffers, stream
// argument, no host synchronisation), so a plugin backed by the sm_90a kernels is the same three methods over
// odtk_decode / odtk_decode_rotate / odtk_nms / odtk_nms_rotate.  The classes below are those three methods, with the
// TensorRT signatures, independent of the TensorRT base class: a maintainer derives
//     class DecodePlugin : public nvinfer1::IPluginV2DynamicExt, private odtk_b200::DecodeBackend { ... }
// and forwards configurePlugin / getWorkspaceSize / enqueue (INTEGRATION.md shows the diff); serialisation, cloning and
// the creator stay as they are.  Header-only; links against libodtk_b200.so.  Compile-checked without TensorRT by
// plugins/plugin_check.cpp (nvinfer_stub.h supplies the few descriptor types).
#pragma once
#ifdef ODTK_B200_HAVE_NVINFER
#include <NvInfer.h>
#include <cuda_runtime_api.h>
#else
#include "nvinfer_stub.h"
#endif

#include <vector>

#include "../include/odtk_b200.h"

namespace odtk_b200 {

// RetinaNetDecode / RetinaNetDecodeRotate: inputs {scores [B, A*C, H, W], deltas [B, A*4|6, H, W]} fp32 linear,
// outputs {scores [B, top_n], boxes [B, top_n * 4|6], classes [B, top_n]} (DecodePlugin.h:108-118).
class DecodeBackend {
 public:
  DecodeBackend(float score_thresh, int top_n, std::vector<float> anchors, int scale, bool rotated = false)
      : score_thresh_(score_thresh), top_n_(top_n), anchors_(std::move(anchors)), scale_(scale), rotated_(rotated) {}

  // DecodePlugin.h:177-191: geometry from the descriptors the builder hands over
  void configurePlugin(const nvinfer1::DynamicPluginTensorDesc *in, int nbInputs, const nvinfer1::DynamicPluginTensorDesc *,
                       int nbOutputs) noexcept {
    if (nbInputs != 2 || nbOutputs != 3) return;
    const nvinfer1::Dims &s = in[0].desc.dims, &b = in[1].desc.dims;
    height_ = (size_t)s.d[2];
    width_ = (size_t)s.d[3];
    num_anchors_ = (size_t)b.d[1] / (rotated_ ? 6 : 4);
    num_classes_ = num_anchors_ ? (size_t)s.d[1] / num_anchors_ : 0;
  }

  bool supportsFormatCombination(int pos, const nvinfer1::PluginTensorDesc *io, int nbInputs, int nbOutputs) const noexcept {
    return nbInputs == 2 && nbOutputs == 3 && pos < 5 && io[pos].type == nvinfer1::DataType::kFLOAT &&
           io[pos].format == nvinfer1::PluginFormat::kLINEAR;      // the fp32 NCHW entry point (DecodePlugin.h:128-135)
  }

  // DecodePlugin.h:141-150: the size query of the decode entry point, cached per batch size
  size_t getWorkspaceSize(const nvinfer1::PluginTensorDesc *inputs, int, const nvinfer1::PluginTensorDesc *, int) const noexcept {
    const int batch = (int)inputs->dims.d[0];
    if (cached_batch_ != batch) {
      const long long n = call(batch, nullptr, nullptr, nullptr, 0, nullptr);
      cached_size_ = n > 0 ? (size_t)n : 0;
      cached_batch_ = batch;
    }
    return cached_size_;
  }

  // DecodePlugin.h:152-161.  0 on success, non-zero otherwise (TensorRT's convention); never throws, never blocks the host.
  int enqueue(const nvinfer1::PluginTensorDesc *inputDesc, const nvinfer1::PluginTensorDesc *outputDesc, const void *const *inputs,
              void *const *outputs, void *workspace, cudaStream_t stream) noexcept {
    const size_t ws = getWorkspaceSize(inputDesc, 2, outputDesc, 3);
    return call((int)inputDesc->dims.d[0], inputs, outputs, workspace, ws, stream) == ODTK_OK ? 0 : 1;
  }

 private:
  long long call(int batch, const void *const *inputs, void *const *outputs, void *workspace, size_t ws, cudaStream_t stream) const noexcept {
    auto fn = rotated_ ? odtk_decode_rotate : odtk_decode;
    return fn(batch, inputs, outputs, height_, width_, (size_t)scale_, num_anchors_, num_classes_, anchors_.data(),
              anchors_.size(), score_thresh_, top_n_, workspace, ws, (odtk_stream_t)stream);
  }
  float score_thresh_;
  int top_n_;
  std::vector<float> anchors_;
  int scale_;
  bool rotated_;
  size_t height_ = 0, width_ = 0, num_anchors_ = 0, num_classes_ = 0;
  mutable int cached_batch_ = -1;
  mutable size_t cached_size_ = 0;
};

// RetinaNetNMS / RetinaNetNMSRotate: inputs {scores [B, N], boxes [B, N * 4|6], classes [B, N]},
// outputs {scores [B, D], boxes [B, D * 4|6], classes [B, D]} (NMSPlugin.h:88-98).
class NmsBackend {
 public:
  NmsBackend(float nms_thresh, int detections_per_im, bool rotated = false)
      : nms_thresh_(nms_thresh), detections_per_im_(detections_per_im), rotated_(rotated) {}

  void configurePlugin(const nvinfer1::DynamicPluginTensorDesc *in, int nbInputs, const nvinfer1::DynamicPluginTensorDesc *,
                       int nbOutputs) noexcept {
    if (nbInputs == 3 && nbOutputs == 3) count_ = (size_t)in[0].desc.dims.d[1];     // NMSPlugin.h:152-160
  }

  size_t getWorkspaceSize(const nvinfer1::PluginTensorDesc *inputs, int, const nvinfer1::PluginTensorDesc *, int) const noexcept {
    const long long n = call((int)inputs->dims.d[0], nullptr, nullptr, nullptr, 0, nullptr);   // NMSPlugin.h:120-129
    return n > 0 ? (size_t)n : 0;
  }

  int enqueue(const nvinfer1::PluginTensorDesc *inputDesc, const nvinfer1::PluginTensorDesc *outputDesc, const void *const *inputs,
              void *const *outputs, void *workspace, cudaStream_t stream) noexcept {                   // NMSPlugin.h:131-138
    const size_t ws = getWorkspaceSize(inputDesc, 3, outputDesc, 3);
    return call((int)inputDesc->dims.d[0], inputs, outputs, workspace, ws, stream) == ODTK_OK ? 0 : 1;
  }

 private:
  long long call(int batch, const void *const *inputs, void *const *outputs, void *workspace, size_t ws, cudaStream_t stream) const noexcept {
    auto fn = rotated_ ? odtk_nms_rotate : odtk_nms;
    return fn(batch, inputs, outputs, count_, detections_per_im_, nms_thresh_, workspace, ws, (odtk_stream_t)stream);
  }
  float nms_thresh_;
  int detections_per_im_;
  bool rotated_;
  size_t count_ = 0;
};

}  // namespace odtk_b200
