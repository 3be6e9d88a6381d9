// augment.cu -- the training augmentations of odtk/data.py (CocoDataset / RotatedCocoDataset.__getitem__, :64-123)
// on the resized uint8 images, bit-exact to Pillow: rotation by quarter turns, horizontal flip, ImageEnhance
// Brightness / Contrast / Color, torchvision's PIL adjust_hue, then the normalisation and the collate padding.
//
// Compiled with -fmad=false (csrc/Makefile): every float and double expression below is Pillow's C expression with the
// same types and the same operation order, and no multiply-add may be contracted.
#include <cuda_runtime.h>
#include <math.h>

#include <algorithm>

#include "common.cuh"
#include "prof.cuh"

namespace {

constexpr int AUG_TW = 32, AUG_TH = 8;

// Size of the image after the rotation: 90 / 270 with expand transpose it, everything else keeps h x w.
__host__ __device__ __forceinline__ void rotated_size(const odtk_augment_image_t &im, int &H, int &W) {
  const bool t = (im.rot & 1) && im.expand;
  H = t ? im.w : im.h;
  W = t ? im.h : im.w;
}

// Source pixel (row, col) of output pixel (r, c) of the rotated and flipped image of size H x W; false for the black fill
// of a non-square 90 / 270 rotation without expand.  That case is Pillow's affine transform with NEAREST about the centre
// (w / 2, h / 2): with the matrix Pillow rounds to (0, -1, 1, 0) or (0, 1, -1, 0), every coordinate is a multiple of 0.5
// and the sampled index is the floor of it, which is what the integer shifts below compute.  On a square image the
// same formulas give the transpose.
__device__ __forceinline__ bool source_pixel(const odtk_augment_image_t &im, int W, int r, int c, int &sr, int &sc) {
  const int h = im.h, w = im.w;
  if (im.flip) c = W - 1 - c;
  switch (im.rot) {
    case 0: sr = r; sc = c; return true;
    case 2: sr = h - 1 - r; sc = w - 1 - c; return true;
    case 1:
      if (im.expand) { sr = c; sc = w - 1 - r; return true; }
      sc = (w + h - 1 - 2 * r) >> 1;
      sr = (h - w + 1 + 2 * c) >> 1;
      break;
    default:
      if (im.expand) { sr = h - 1 - c; sc = r; return true; }
      sc = (w - h + 1 + 2 * r) >> 1;
      sr = (w + h - 1 - 2 * c) >> 1;
      break;
  }
  return sr >= 0 && sr < h && sc >= 0 && sc < w;
}

__device__ __forceinline__ void load_pixel(const unsigned char *src, const odtk_augment_image_t &im, int W, int r, int c,
                                           unsigned v[3]) {
  int sr, sc;
  if (source_pixel(im, W, r, c, sr, sc)) {
    const unsigned char *p = src + ((long long)sr * im.w + sc) * 3;
    v[0] = __ldg(p); v[1] = __ldg(p + 1); v[2] = __ldg(p + 2);
  } else {
    v[0] = v[1] = v[2] = 0u;
  }
}

// Pillow's ImagingBlend (Blend.c) on one channel: in1 + alpha * (in2 - in1) in float; truncated for alpha in [0, 1],
// clamped to [0, 255] then truncated otherwise.
__device__ __forceinline__ unsigned blend8(unsigned in1, unsigned in2, float alpha) {
  const float t = (float)(int)in1 + alpha * (float)((int)in2 - (int)in1);
  if (alpha >= 0.0f && alpha <= 1.0f) return (unsigned)(unsigned char)t;
  if (t <= 0.0f) return 0u;
  if (t >= 255.0f) return 255u;
  return (unsigned)(unsigned char)t;
}

// convert("L") of an RGB pixel (Convert.c, L24): ITU-R 601-2 luma in 16-bit fixed point, rounded.
__device__ __forceinline__ unsigned luma8(const unsigned v[3]) {
  return (v[0] * 19595u + v[1] * 38470u + v[2] * 7471u + 0x8000u) >> 16;
}

__device__ __forceinline__ int clip8(int v) { return v <= 0 ? 0 : (v >= 255 ? 255 : v); }

// convert("HSV") (Convert.c rgb2hsv_row), H shifted by `shift` modulo 256, convert("RGB") (hsv2rgb): Pillow's mix of
// float and double arithmetic, expression for expression.
__device__ __forceinline__ void hue_shift(unsigned v[3], int shift) {
  const int r = v[0], g = v[1], b = v[2];
  const int maxc = max(r, max(g, b)), minc = min(r, min(g, b));
  int uh = 0, us = 0;
  const int uv = maxc;
  if (minc != maxc) {
    const float cr = (float)(maxc - minc);
    const float s = cr / (float)maxc;
    const float rc = (float)(maxc - r) / cr, gc = (float)(maxc - g) / cr, bc = (float)(maxc - b) / cr;
    float h;
    if (r == maxc) h = bc - gc;
    else if (g == maxc) h = (float)(2.0 + (double)rc - (double)bc);
    else h = (float)(4.0 + (double)gc - (double)rc);
    h = (float)fmod((double)h / 6.0 + 1.0, 1.0);
    uh = clip8((int)((double)h * 255.0));
    us = clip8((int)((double)s * 255.0));
  }
  uh = (uh + shift) & 255;
  if (us == 0) {
    v[0] = v[1] = v[2] = (unsigned)uv;
    return;
  }
  const int i = (int)floor((double)(float)uh * 6.0 / 255.0);
  const float f = (float)((double)(float)uh * 6.0 / 255.0 - (double)(float)i);
  const float fs = (float)((double)(float)us / 255.0);
  const double fv = (double)(float)uv;
  const int p = clip8((int)round(fv * (1.0 - (double)fs)));
  const int q = clip8((int)round(fv * (1.0 - (double)(fs * f))));
  const int t = clip8((int)round(fv * (1.0 - (double)fs * (1.0 - (double)f))));
  switch (i % 6) {
    case 0: v[0] = uv; v[1] = t; v[2] = p; break;
    case 1: v[0] = q; v[1] = uv; v[2] = p; break;
    case 2: v[0] = p; v[1] = uv; v[2] = t; break;
    case 3: v[0] = p; v[1] = q; v[2] = uv; break;
    case 4: v[0] = t; v[1] = p; v[2] = uv; break;
    default: v[0] = uv; v[1] = p; v[2] = q; break;
  }
}

// Per image with ODTK_AUGMENT_CONTRAST: sum over the rotated image of convert("L") after rotation, flip and brightness
// (the fill pixels count, as zeros).  grid (blocks, n), 256 threads; integer sums, so the order does not matter.
__global__ void augment_stats_kernel(const unsigned char *__restrict__ x, const odtk_augment_image_t *__restrict__ tab,
                                     unsigned long long *__restrict__ sums) {
  const odtk_augment_image_t im = tab[blockIdx.y];
  if (!(im.flags & ODTK_AUGMENT_CONTRAST)) return;
  int H, W;
  rotated_size(im, H, W);
  const unsigned char *src = x + im.offset;
  const long long total = (long long)H * W;
  unsigned long long acc = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / W), c = (int)(i % W);
    unsigned v[3];
    load_pixel(src, im, W, r, c, v);
    if (im.flags & ODTK_AUGMENT_BRIGHTNESS)
      for (int k = 0; k < 3; k++) v[k] = blend8(0u, v[k], im.brightness);
    acc += luma8(v);
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0 && acc) atomicAdd(sums + blockIdx.y, acc);
}

// One thread per canvas pixel: grid (ceil(canvas_w / 32), ceil(canvas_h / 8), n), 32 x 8 threads.  Row-major threads
// write consecutive 12-byte pixels; 90 / 270 turns read a column of the source per warp (through L1 / L2).
__global__ void __launch_bounds__(AUG_TW *AUG_TH) augment_apply_kernel(
    const unsigned char *__restrict__ x, const odtk_augment_image_t *__restrict__ tab,
    const unsigned long long *__restrict__ sums, float *__restrict__ y, int CH, int CW, float m0, float m1, float m2,
    float s0, float s1, float s2) {
  const int n = blockIdx.z;
  const int c = blockIdx.x * AUG_TW + threadIdx.x % AUG_TW, r = blockIdx.y * AUG_TH + threadIdx.x / AUG_TW;
  if (r >= CH || c >= CW) return;
  float *o = y + (((long long)n * CH + r) * CW + c) * 3;
  const odtk_augment_image_t im = tab[n];
  int H, W;
  rotated_size(im, H, W);
  if (r >= H || c >= W) {
    o[0] = o[1] = o[2] = 0.0f;
    return;
  }
  unsigned v[3];
  load_pixel(x + im.offset, im, W, r, c, v);
  if (im.flags & ODTK_AUGMENT_BRIGHTNESS)
    for (int k = 0; k < 3; k++) v[k] = blend8(0u, v[k], im.brightness);
  if (im.flags & ODTK_AUGMENT_CONTRAST) {
    // ImageStat mean: the integer sum over the pixel count in double, then int(mean + 0.5)
    const unsigned grey = (unsigned)(int)((double)sums[n] / (double)((long long)H * W) + 0.5);
    for (int k = 0; k < 3; k++) v[k] = blend8(grey, v[k], im.contrast);
  }
  if (im.flags & ODTK_AUGMENT_HUE) hue_shift(v, im.hue_shift);
  if (im.flags & ODTK_AUGMENT_SATURATION) {
    const unsigned l = luma8(v);
    for (int k = 0; k < 3; k++) v[k] = blend8(l, v[k], im.saturation);
  }
  o[0] = normalize_u8(v[0], m0, s0);
  o[1] = normalize_u8(v[1], m1, s1);
  o[2] = normalize_u8(v[2], m2, s2);
}

}  // namespace

extern "C" long long odtk_augment_u8(const void *x, size_t x_bytes, const odtk_augment_image_t *images,
                                     const odtk_augment_image_t *images_dev, int n, int canvas_h, int canvas_w,
                                     void *workspace, size_t workspace_bytes, float *y, const float *mean,
                                     const float *std, odtk_stream_t stream_) {
  if (!images || n <= 0 || n > 65535 || canvas_h <= 0 || canvas_w <= 0) return ODTK_E_INVALID;
  const int known = ODTK_AUGMENT_BRIGHTNESS | ODTK_AUGMENT_CONTRAST | ODTK_AUGMENT_HUE | ODTK_AUGMENT_SATURATION;
  bool contrast = false;
  long long max_px = 0;
  for (int i = 0; i < n; i++) {
    const odtk_augment_image_t &im = images[i];
    int H, W;
    rotated_size(im, H, W);
    if (im.h <= 0 || im.w <= 0 || H > canvas_h || W > canvas_w) return ODTK_E_INVALID;
    if (im.offset < 0 || (unsigned long long)im.offset + (unsigned long long)im.h * im.w * 3 > x_bytes) return ODTK_E_INVALID;
    if (im.rot < 0 || im.rot > 3 || (im.flags & ~known) || im.hue_shift < 0 || im.hue_shift > 255) return ODTK_E_INVALID;
    if (!(im.brightness >= 0.0f) || !(im.contrast >= 0.0f) || !(im.saturation >= 0.0f)) return ODTK_E_INVALID;
    contrast |= (im.flags & ODTK_AUGMENT_CONTRAST) != 0;
    max_px = max(max_px, (long long)H * W);
  }
  const size_t need = odtk_align_up((size_t)n * sizeof(unsigned long long));
  if (!workspace) return (long long)need;
  if (workspace_bytes < need) return ODTK_E_WORKSPACE;
  if (!x || !images_dev || !y || !mean || !std) return ODTK_E_INVALID;
  cudaStream_t s = (cudaStream_t)stream_;
  OdtkProfScope prof(ODTK_PROF_LAYER, s);
  unsigned long long *sums = (unsigned long long *)workspace;
  if (contrast) {
    if (cudaMemsetAsync(sums, 0, (size_t)n * sizeof(unsigned long long), s) != cudaSuccess) return ODTK_E_CUDA;
    const int blocks = (int)std::min<long long>((max_px + 4095) / 4096, 256);
    augment_stats_kernel<<<dim3(blocks, n), 256, 0, s>>>((const unsigned char *)x, images_dev, sums);
  }
  const dim3 grid((canvas_w + AUG_TW - 1) / AUG_TW, (canvas_h + AUG_TH - 1) / AUG_TH, n);
  augment_apply_kernel<<<grid, AUG_TW * AUG_TH, 0, s>>>((const unsigned char *)x, images_dev, sums, y, canvas_h, canvas_w,
                                                         mean[0], mean[1], mean[2], std[0], std[1], std[2]);
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}
