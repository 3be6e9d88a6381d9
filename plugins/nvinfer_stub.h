// nvinfer_stub.h -- the handful of TensorRT types odtk_b200_plugin.h touches, for compile-checking the plugin-shaped
// wrappers in an image without TensorRT (this one: `import tensorrt` / <NvInfer.h> are absent).
// NOT TensorRT: with the real SDK define ODTK_B200_HAVE_NVINFER and this file is never included.
#pragma once
#include <cstddef>
#include <cstdint>

typedef struct CUstream_st *cudaStream_t;

namespace nvinfer1 {
enum class DataType : int32_t { kFLOAT = 0, kHALF = 1 };
enum class PluginFormat : int32_t { kLINEAR = 0 };
struct Dims { int32_t nbDims; int64_t d[8]; };
struct PluginTensorDesc { Dims dims; DataType type; PluginFormat format; float scale; };
struct DynamicPluginTensorDesc { PluginTensorDesc desc; Dims min, max; };
}  // namespace nvinfer1
