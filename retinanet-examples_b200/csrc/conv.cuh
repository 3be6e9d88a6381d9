// conv.cuh -- kernel-side parameter block of conv_gemm_kernel (see conv.cu).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdint.h>

// Host helpers shared by the TMA kernels (conv.cu, bottleneck.cu, stem.cu).
// Encode a tiled tensor map (cached per base pointer, data type and geometry); false if the driver rejects it.  dims and
// box are in elements of `dtype` (fp16, or UINT8 for int8 bytes).
bool encode_map(CUtensorMap *m, const void *base, int rank, const uint64_t *dims, const uint64_t *strides_bytes,
                const uint32_t *box, CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B, const uint32_t *elem_strides = nullptr,
                CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_FLOAT16);
// The spatial patch (TW x TH <= 128 pixels) that wastes the fewest accumulator rows on an H x W image.
void choose_patch(int H, int W, int &TH, int &TW);

struct ConvParams {
  int mode;             // 0: rows of a [M, Cin] matrix (1x1 / lowered conv); 1: spatial patch, one shifted box per tap
                        // (3x3 pad 1, or stride 2 with element-strided boxes when s2); 2: 7x7 stride-2 stem over a
                        // zero-padded NHWC4 image (overlapping-window 5-D map); 3: stride 2 on even sizes (parity-split view)
  int N, H, W, Cin, Cout;
  int taps, kw, pad;    // 1 / 7 / 9 taps
  int TH, TW, tiles_h, tiles_w;   // modes 1-3: patch and patches per image
  int num_m_tiles, num_n_tiles, kblocks_per_tap;
  int kblocks2;         // mode 0: extra K blocks from a second operand pair (A2 [M, 64 * kblocks2], B2 [Cout, 64 * kblocks2])
  long long M;          // N*H*W
  const float *bias;    // [Cout] fp32 (folded BatchNorm shift / conv bias) or NULL
  const __half *residual;  // NHWC fp16, row stride ldr, or NULL
  const __half *upsample;  // NHWC fp16 [N, H/2, W/2, Cout] (FPN top-down path) or NULL
  void *out;
  int relu, out_mode, ldy, ldr, up_h, up_w;
  int row_bytes;        // bytes of one K block row in shared memory: 128 (SWIZZLE_128B) or 64 (SWIZZLE_64B, stem)
  int nstages;          // pipeline stages that fit: (128 + BN) * row_bytes each
  const int4 *tile_tab;   // mode 1 over a pyramid atlas: per tile of one image (h0, w0, first row / column not to write)
  int tab_tiles;          // tiles per image in tile_tab
  int oH, oR, oW;         // NHWC output placement: pixel (img, h, w) is written at ((img * oH + oR + h) * oW + w) * ldy
  int grouped;          // grouped conv: kblocks_per_tap == 1 and the A channel coordinate is the N tile's own chunk (n0)
  int s2;               // mode 1: input pixel = 2 * output pixel + tap offset (element-strided TMA boxes), else 0
  // out_mode ODTK_OUT_CANDIDATES: the decode workspace of this pyramid level (decode.cu)
  int *cand_counts;          // [N]
  unsigned *cand_hist;       // [N, cand_hist_bins]
  uint2 *cand;               // [N, cand_cap]
  long long cand_cap;
  unsigned cand_key_thresh;
  int cand_shift, cand_hist_bins;
  float cand_thresh, cand_pre;   // candidate iff sigmoid(x) > thresh; x <= cand_pre can never pass
  // s8 launches (odtk_conv2d_s8): y = fmaf((float)acc, alpha[c], bias[c]); ODTK_OUT_NHWC_S8 stores
  // clamp(rint(y * inv_out_scale), -127, 127)
  const float *alpha;
  float inv_out_scale;
  // s8 addends of ODTK_OUT_NHWC_S8 (odtk_conv2d_s8_ex), each one more fmaf before ReLU: residual [M, Cout] at the output
  // pixel, upsample [N, up_h, up_w, Cout] at (h >> 1, w >> 1); NULL when absent
  const int8_t *res8, *up8;
  float res_scale, up_scale;
  // fp32 addends of ODTK_OUT_NHWC_F32 (odtk_conv2d_f32): residual [M, ldr] at the output pixel, upsample
  // [N, up_h, up_w, Cout] at (h >> 1, w >> 1); NULL when absent
  const float *res32, *up32;
  // input-gradient instance (odtk_conv2d_dgrad): NHWC fp16 [M, Cout] at the output pixel; an output element whose mask
  // element is not > 0 becomes 0 (the ReLU derivative of the forward layer's input), or NULL
  const __half *mask;
  // fp16 forward, ODTK_OUT_NHWC_F16: 1 if the epilogue stores through the output tensor map (TMA from shared memory), and
  // res_tma 1 if the producer then loads the residual (mode 0) into the ring after each tile's K blocks
  int tma_store, res_tma;
};
