// layers.cu -- the small memory-bound layers around the tensor-core convolution:
//   * lowering of strided / 7x7 convolutions to GEMM rows (gather of the receptive field into
//     a [pixels, taps*C] fp16 matrix; used for the ResNet stem, the three stride-2 3x3 and 1x1
//     convolutions of the backbone, and FPN pyramid6 / pyramid7 -- together < 5 % of the FLOPs);
//   * 3x3 stride-2 max-pool (torchvision resnet.py maxpool), NHWC fp16.
// Reference call sites: odtk/backbones/resnet.py:25-28, odtk/backbones/fpn.py:54-55.
#include <cuda_fp16.h>

#include <type_traits>

#include "common.cuh"
#include "prof.cuh"

namespace {

// C % 8 == 0: one thread moves 8 channels (16 B) of one tap of one output pixel.
__global__ void lower_vec8_kernel(const __half *__restrict__ x, __half *__restrict__ out, int N, int H, int W, int C,
                                  int OH, int OW, int ks, int stride, int pad, int kpad, int relu) {
  const int c8n = C >> 3;
  const long long total = (long long)N * OH * OW * ks * ks * c8n;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int c8 = (int)(i % c8n);
    long long r = i / c8n;
    int tap = (int)(r % (ks * ks));
    long long m = r / (ks * ks);
    int ow = (int)(m % OW);
    long long t = m / OW;
    int oh = (int)(t % OH);
    int n = (int)(t / OH);
    int ih = oh * stride + tap / ks - pad, iw = ow * stride + tap % ks - pad;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (ih >= 0 && ih < H && iw >= 0 && iw < W) {
      v = __ldg(reinterpret_cast<const uint4 *>(x + (((long long)n * H + ih) * W + iw) * C + c8 * 8));
      if (relu) {
        __half2 *h = reinterpret_cast<__half2 *>(&v);
        const __half2 z = __float2half2_rn(0.0f);
#pragma unroll
        for (int j = 0; j < 4; j++) h[j] = __hmax2(h[j], z);
      }
    }
    *reinterpret_cast<uint4 *>(out + m * kpad + (long long)tap * C + c8 * 8) = v;
  }
}

// generic small-C path (the RGB stem): one thread produces 8 consecutive K entries.
__global__ void lower_generic_kernel(const __half *__restrict__ x, __half *__restrict__ out, int N, int H, int W, int C,
                                     int OH, int OW, int ks, int stride, int pad, int kpad) {
  const int k8n = kpad >> 3;
  const int kreal = ks * ks * C;
  const long long total = (long long)N * OH * OW * k8n;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int k8 = (int)(i % k8n);
    long long m = i / k8n;
    int ow = (int)(m % OW);
    long long t = m / OW;
    int oh = (int)(t % OH);
    int n = (int)(t / OH);
    __align__(16) __half v[8];
#pragma unroll
    for (int j = 0; j < 8; j++) {
      int k = k8 * 8 + j;
      __half val = __float2half_rn(0.0f);
      if (k < kreal) {
        int tap = k / C, c = k - tap * C;
        int ih = oh * stride + tap / ks - pad, iw = ow * stride + tap % ks - pad;
        if (ih >= 0 && ih < H && iw >= 0 && iw < W) val = x[(((long long)n * H + ih) * W + iw) * C + c];
      }
      v[j] = val;
    }
    *reinterpret_cast<uint4 *>(out + m * kpad + k8 * 8) = *reinterpret_cast<uint4 *>(v);
  }
}

__global__ void maxpool3x3s2_kernel(const __half *__restrict__ x, __half *__restrict__ y, int N, int H, int W, int C,
                                    int OH, int OW) {
  const int c8n = C >> 3;
  const long long total = (long long)N * OH * OW * c8n;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int c8 = (int)(i % c8n);
    long long m = i / c8n;
    int ow = (int)(m % OW);
    long long t = m / OW;
    int oh = (int)(t % OH);
    int n = (int)(t / OH);
    __half2 best[4];
    const __half2 ninf = __float2half2_rn(-65504.0f);
#pragma unroll
    for (int j = 0; j < 4; j++) best[j] = ninf;
#pragma unroll
    for (int dy = 0; dy < 3; dy++) {
      int ih = oh * 2 + dy - 1;
      if (ih < 0 || ih >= H) continue;
#pragma unroll
      for (int dx = 0; dx < 3; dx++) {
        int iw = ow * 2 + dx - 1;
        if (iw < 0 || iw >= W) continue;
        uint4 v = __ldg(reinterpret_cast<const uint4 *>(x + (((long long)n * H + ih) * W + iw) * C + c8 * 8));
        const __half2 *h = reinterpret_cast<const __half2 *>(&v);
#pragma unroll
        for (int j = 0; j < 4; j++) best[j] = __hmax2(best[j], h[j]);
      }
    }
    *reinterpret_cast<uint4 *>(y + m * C + c8 * 8) = *reinterpret_cast<uint4 *>(best);
  }
}

// RGB NHWC3 fp16 -> zero-padded NHWC4 [n, h+6, w+8, 4]: 3 rows/columns of zeros before, 3/5 after
// (the stem's overlapping-window tensor map never leaves the buffer).  One 8-byte pixel per thread.
__global__ void pad_input_kernel(const __half *__restrict__ x, __half *__restrict__ y, int N, int H, int W) {
  const int HP = H + 6, WP = W + 8;
  const long long total = (long long)N * HP * WP;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int xp = (int)(i % WP);
    long long t = i / WP;
    int yp = (int)(t % HP);
    int n = (int)(t / HP);
    int ih = yp - 3, iw = xp - 3;
    uint2 v = make_uint2(0u, 0u);
    if (ih >= 0 && ih < H && iw >= 0 && iw < W) {
      const unsigned short *s = reinterpret_cast<const unsigned short *>(x) + (((long long)n * H + ih) * W + iw) * 3;
      v.x = (unsigned)s[0] | ((unsigned)s[1] << 16);
      v.y = (unsigned)s[2];
    }
    reinterpret_cast<uint2 *>(y)[i] = v;
  }
}

// Same, for W % 8 == 0 (input rows start 16-byte aligned): one block per padded row; the 6-byte pixels of the input row
// are staged through shared memory with coalesced 16-byte loads, the padded row leaves as coalesced 16-byte stores
// (two 8-byte pixels each) -- the per-pixel version above issues three 2-byte loads per pixel.
__global__ void pad_input_rows_kernel(const __half *__restrict__ x, __half *__restrict__ y, int N, int H, int W) {
  extern __shared__ uint4 srow[];                                 // W * 6 bytes of the input row
  const int HP = H + 6, WP = W + 8;
  const int n = blockIdx.x / HP, yp = blockIdx.x - n * HP, ih = yp - 3;
  uint4 *dst = reinterpret_cast<uint4 *>(y + ((long long)n * HP + yp) * WP * 4);
  const int pairs = WP / 2;
  if (ih < 0 || ih >= H) {
    for (int i = threadIdx.x; i < pairs; i += blockDim.x) dst[i] = make_uint4(0u, 0u, 0u, 0u);
    return;
  }
  const uint4 *src = reinterpret_cast<const uint4 *>(x + ((long long)n * H + ih) * W * 3);
  const int nv = W * 6 / 16;
  for (int i = threadIdx.x; i < nv; i += blockDim.x) srow[i] = __ldg(src + i);
  __syncthreads();
  const unsigned short *s = reinterpret_cast<const unsigned short *>(srow);
  for (int i = threadIdx.x; i < pairs; i += blockDim.x) {
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    const int iw0 = 2 * i - 3, iw1 = iw0 + 1;
    if (iw0 >= 0 && iw0 < W) { v.x = (unsigned)s[iw0 * 3] | ((unsigned)s[iw0 * 3 + 1] << 16); v.y = (unsigned)s[iw0 * 3 + 2]; }
    if (iw1 >= 0 && iw1 < W) { v.z = (unsigned)s[iw1 * 3] | ((unsigned)s[iw1 * 3 + 1] << 16); v.w = (unsigned)s[iw1 * 3 + 2]; }
    dst[i] = v;
  }
}

// One RGB pixel of it as the stem's 8-byte NHWC4 pixel: one fp16 rounding.
__device__ __forceinline__ uint2 normalize_rgb_u8(unsigned r8, unsigned g8, unsigned b8, float m0, float m1, float m2,
                                                  float s0, float s1, float s2) {
  float r = normalize_u8(r8, m0, s0), g = normalize_u8(g8, m1, s1), b = normalize_u8(b8, m2, s2);
  __half2 rg = __floats2half2_rn(r, g);
  __half2 bz = __floats2half2_rn(b, 0.0f);
  return make_uint2(*reinterpret_cast<unsigned *>(&rg), *reinterpret_cast<unsigned *>(&bz));
}

// The same pixel as the 16-byte fp32 NHWC4 pixel of the full-precision stem (no rounding after the fp32 arithmetic).
__device__ __forceinline__ float4 normalize_rgb_u8_f32(unsigned r8, unsigned g8, unsigned b8, float m0, float m1, float m2,
                                                       float s0, float s1, float s2) {
  return make_float4(normalize_u8(r8, m0, s0), normalize_u8(g8, m1, s1), normalize_u8(b8, m2, s2), 0.0f);
}

// Input side of odtk infer (reference odtk/data.py:113-123): uint8 HWC image -> /255 -> (x - mean) / std
// -> zero padding to a multiple of the model stride, fused with the stem's own zero padding and the
// RGB -> NHWC4 widening: one 8-byte store per padded pixel, the fp32 full-image pass disappears.
__global__ void preprocess_u8_kernel(const unsigned char *__restrict__ x, __half *__restrict__ y, int N, int H, int W,
                                     int HS, int WS, float m0, float m1, float m2, float s0, float s1, float s2) {
  const int HP = HS + 6, WP = WS + 8;
  const long long total = (long long)N * HP * WP;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int xp = (int)(i % WP);
    long long t = i / WP;
    int yp = (int)(t % HP);
    int n = (int)(t / HP);
    int ih = yp - 3, iw = xp - 3;
    uint2 v = make_uint2(0u, 0u);
    if (ih >= 0 && ih < H && iw >= 0 && iw < W) {
      const unsigned char *s = x + (((long long)n * H + ih) * W + iw) * 3;
      v = normalize_rgb_u8(s[0], s[1], s[2], m0, m1, m2, s0, s1, s2);
    }
    reinterpret_cast<uint2 *>(y)[i] = v;
  }
}

// ---- Pillow-exact bilinear resize (PIL Image.resize(..., BILINEAR) on 8-bit RGB, the resize of odtk/data.py:60) ----
// Separable triangle filter.  Per output position o of an axis (in -> out samples): scale = in / out, the support is
// max(scale, 1), the window is [int(center - support + 0.5), int(center + support + 0.5)) clamped to the input, each tap
// weighs triangle((i - center + 0.5) / max(scale, 1)), the weights are divided by their sum and turned into 22-bit fixed
// point (rounding half away from zero).  Every double operation is an explicit round-to-nearest intrinsic, so no FMA
// contraction can change a bit against the C original.  Pixels accumulate in int32 from 1 << 21, >> 22, clamp to
// [0, 255]; the horizontal result is rounded to uint8 before the vertical pass reads it.  An axis whose lengths match
// gets weights (1, 0): the identity, like the pass Pillow skips.
constexpr int RS_BITS = 22;
constexpr int RS_TW = 32, RS_TH = 64, RS_ROWS = 8;   // 32 x 64 output tile per block of 32 x 8 threads
constexpr int RS_KMAX = 16;            // taps per position kept in shared memory (axes shrunk up to 7x)

struct ResampleAxis {
  double center, ss, ww;
  int lo, count;
};

__device__ __forceinline__ double resample_scale(int in_size, int out_size) {
  return __ddiv_rn((double)in_size, (double)out_size);
}

__device__ __forceinline__ int resample_ksize(int in_size, int out_size) {
  const double s = resample_scale(in_size, out_size);
  return (int)ceil(s < 1.0 ? 1.0 : s) * 2 + 1;
}

__device__ __forceinline__ double resample_tap(const ResampleAxis &a, int j) {
  double t = __dmul_rn(__dadd_rn(__dadd_rn((double)(a.lo + j), -a.center), 0.5), a.ss);
  if (t < 0.0) t = -t;
  return t < 1.0 ? __dadd_rn(1.0, -t) : 0.0;
}

__device__ ResampleAxis resample_axis(int o, int in_size, int out_size) {
  ResampleAxis a;
  const double scale = resample_scale(in_size, out_size);
  const double support = scale < 1.0 ? 1.0 : scale;          // filter support 1 x max(scale, 1)
  a.center = __dadd_rn(0.0, __dmul_rn(__dadd_rn((double)o, 0.5), scale));
  a.ss = __ddiv_rn(1.0, support);
  a.lo = max(__double2int_rz(__dadd_rn(__dadd_rn(a.center, -support), 0.5)), 0);
  a.count = min(__double2int_rz(__dadd_rn(__dadd_rn(a.center, support), 0.5)), in_size) - a.lo;
  double ww = 0.0;
  for (int j = 0; j < a.count; j++) ww = __dadd_rn(ww, resample_tap(a, j));
  a.ww = ww;
  return a;
}

__device__ __forceinline__ int resample_weight(const ResampleAxis &a, int j) {
  double k = resample_tap(a, j);
  if (a.ww != 0.0) k = __ddiv_rn(k, a.ww);
  const double f = __dmul_rn(k, (double)(1 << RS_BITS));
  return k < 0.0 ? __double2int_rz(__dadd_rn(-0.5, f)) : __double2int_rz(__dadd_rn(0.5, f));
}

__device__ __forceinline__ unsigned resample_clip8(int acc) { return (unsigned)min(max(acc >> RS_BITS, 0), 255); }

// grid (ceil((canvas_w + 8) / 32), ceil((canvas_h + 6) / 64), n), 256 threads = 32 columns x 8 rows, each thread writes
// the 8-byte NHWC4 pixels of one column of the 32 x 64 tile, every 8th row.  A tile that meets the image first puts the
// fixed-point taps of its 32 columns and 64 rows into shared memory (one thread per column / row, in parallel), then every
// pixel sums taps x source bytes (sources come through L1).  The taps' double arithmetic is the latency every block waits
// for once, hence the tall tile.
__device__ __forceinline__ int resample_acc_init() { return 1 << (RS_BITS - 1); }

// F32: the full-precision stem buffer, 16-byte fp32 NHWC4 pixels (normalize_rgb_u8_f32) instead of 8-byte fp16 ones.
// U8: Pillow's uint8 result itself, HWC RGB packed per image at y + out_off[n] (dst_h x dst_w, no border, no canvas), for
// the training augmentations that run on it; HS / WS and the normalisation are not used, the tile origin is (0, 0).
template <bool F32, bool U8 = false>
__global__ void __launch_bounds__(RS_TW * RS_ROWS, 3) preprocess_resize_u8_kernel(
    const unsigned char *__restrict__ x, const odtk_resize_image_t *__restrict__ tab,
    typename std::conditional<U8, unsigned char, typename std::conditional<F32, float4, uint2>::type>::type *__restrict__ y,
    int HS, int WS, float m0, float m1, float m2, float s0, float s1, float s2, const long long *__restrict__ out_off = nullptr) {
  using Pix = typename std::conditional<F32, float4, uint2>::type;
  __shared__ int s_wx[RS_KMAX][RS_TW], s_wy[RS_TH][RS_KMAX];     // column taps tap-major: lanes read consecutive words
  __shared__ int s_lox[RS_TW], s_nx[RS_TW], s_loy[RS_TH], s_ny[RS_TH];
  // normalize_rgb_u8(v, v, v): channel c of a pixel is its value's channel c.  The U8 instance neither fills nor reads
  // it (nor HP / WP); it stays declared here so that the fp16 / fp32 instances keep their exact shared-memory layout.
  __shared__ Pix s_norm[256];
  const int HP = HS + 6, WP = WS + 8;
  const int n = blockIdx.z;
  const odtk_resize_image_t im = tab[n];
  const int tx = threadIdx.x % RS_TW, ty = threadIdx.x / RS_TW;
  constexpr int B = U8 ? 0 : 3;                                             // stem border
  const int x0 = blockIdx.x * RS_TW - B, y0 = blockIdx.y * RS_TH - B;     // tile origin in image coordinates
  const int ox = x0 + tx, xp = ox + 3;
  const bool meets = x0 + RS_TW > 0 && x0 < im.dst_w && y0 + RS_TH > 0 && y0 < im.dst_h;                       // block-uniform
  const bool tables = meets && resample_ksize(im.src_w, im.dst_w) <= RS_KMAX && resample_ksize(im.src_h, im.dst_h) <= RS_KMAX;
  if (meets && !U8) {
    for (int v = threadIdx.x; v < 256; v += RS_TW * RS_ROWS) {
      if constexpr (F32) s_norm[v] = normalize_rgb_u8_f32(v, v, v, m0, m1, m2, s0, s1, s2);
      else s_norm[v] = normalize_rgb_u8(v, v, v, m0, m1, m2, s0, s1, s2);
    }
    if (!tables) __syncthreads();
  }
  if (tables && threadIdx.x >= RS_TW + RS_TH) {
    // while the tap threads work, the other warps prefetch the tile's source window into L1 (every row then hits; without
    // it each of a thread's 8 rows waits for its own miss).  A float estimate widened by the filter support + 2, clamped
    // to the image: a hint only, the exact windows come from the taps.
    const float sy = (float)im.src_h / im.dst_h, sx = (float)im.src_w / im.dst_w;
    const float hy = fmaxf(sy, 1.0f) + 2.0f, hx = fmaxf(sx, 1.0f) + 2.0f;
    const int r0 = max((int)((float)max(y0, 0) * sy - hy), 0), r1 = min((int)((float)(y0 + RS_TH) * sy + hy) + 1, im.src_h);
    const int c0 = max((int)((float)max(x0, 0) * sx - hx), 0), c1 = min((int)((float)(x0 + RS_TW) * sx + hx) + 1, im.src_w);
    const unsigned char *src = x + im.offset;
    const long long pitch = (long long)im.src_w * 3;
    const uintptr_t b0 = (uintptr_t)(src + (long long)c0 * 3) & ~(uintptr_t)127;
    const int lines = (int)(((uintptr_t)(src + (long long)c1 * 3 - 1) - b0) / 128) + 1;
    for (int i = threadIdx.x - (RS_TW + RS_TH); i < (r1 - r0) * lines; i += RS_TW * RS_ROWS - (RS_TW + RS_TH)) {
      const int r = r0 + i / lines, l = i % lines;
      const unsigned char *p = src + (long long)r * pitch + (long long)c0 * 3;
      const unsigned char *q = reinterpret_cast<const unsigned char *>(b0 + (uintptr_t)l * 128) + (long long)r * pitch;
      asm volatile("prefetch.global.L1 [%0];" ::"l"(q > p ? q : p));
    }
  }
  if (tables) {
    if (threadIdx.x < RS_TW) {
      const int o = x0 + threadIdx.x;
      if (o >= 0 && o < im.dst_w) {
        const ResampleAxis a = resample_axis(o, im.src_w, im.dst_w);
        s_lox[threadIdx.x] = a.lo;
        s_nx[threadIdx.x] = a.count;
        for (int j = 0; j < a.count; j++) s_wx[j][threadIdx.x] = resample_weight(a, j);
      }
    } else if (threadIdx.x < RS_TW + RS_TH) {
      const int r = threadIdx.x - RS_TW, o = y0 + r;
      if (o >= 0 && o < im.dst_h) {
        const ResampleAxis a = resample_axis(o, im.src_h, im.dst_h);
        s_loy[r] = a.lo;
        s_ny[r] = a.count;
        for (int j = 0; j < a.count; j++) s_wy[r][j] = resample_weight(a, j);
      }
    }
    __syncthreads();
  }
  const unsigned char *src = x + im.offset;
  const long long pitch = (long long)im.src_w * 3;
  for (int r = ty; r < RS_TH; r += RS_ROWS) {
    const int oy = y0 + r, yp = oy + 3;
    if (U8 ? oy >= im.dst_h : yp >= HP) break;
    Pix v;
    if constexpr (F32) v = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    else v = make_uint2(0u, 0u);
    if (meets && ox >= 0 && ox < im.dst_w && oy >= 0 && oy < im.dst_h) {
      int acc[3] = {resample_acc_init(), resample_acc_init(), resample_acc_init()};
      if (tables) {
        const int lox = s_lox[tx], nx = s_nx[tx], loy = s_loy[r], ny = s_ny[r];
        for (int j = 0; j < ny; j++) {
          const unsigned char *row = src + (long long)(loy + j) * pitch + lox * 3;
          int h[3] = {resample_acc_init(), resample_acc_init(), resample_acc_init()};
          for (int i = 0; i < nx; i++) {
            const int k = s_wx[i][tx];
#pragma unroll
            for (int c = 0; c < 3; c++) h[c] += (int)__ldg(row + i * 3 + c) * k;
          }
          const int kv = s_wy[r][j];
#pragma unroll
          for (int c = 0; c < 3; c++) acc[c] += (int)resample_clip8(h[c]) * kv;
        }
      } else {
        // strong downscale: the windows do not fit the shared tables, every pixel evaluates its own taps
        const ResampleAxis ax = resample_axis(ox, im.src_w, im.dst_w), ay = resample_axis(oy, im.src_h, im.dst_h);
        for (int j = 0; j < ay.count; j++) {
          const unsigned char *row = src + (long long)(ay.lo + j) * pitch + ax.lo * 3;
          int h[3] = {resample_acc_init(), resample_acc_init(), resample_acc_init()};
          for (int i = 0; i < ax.count; i++) {
            const int k = resample_weight(ax, i);
#pragma unroll
            for (int c = 0; c < 3; c++) h[c] += (int)__ldg(row + i * 3 + c) * k;
          }
          const int kv = resample_weight(ay, j);
#pragma unroll
          for (int c = 0; c < 3; c++) acc[c] += (int)resample_clip8(h[c]) * kv;
        }
      }
      if constexpr (U8) {
        unsigned char *o = y + out_off[n] + ((long long)oy * im.dst_w + ox) * 3;
#pragma unroll
        for (int c = 0; c < 3; c++) o[c] = (unsigned char)resample_clip8(acc[c]);
        continue;
      }
      // the normalisation is per channel: take r from the red value's entry, g from the green one's, b from the blue one's
      if constexpr (F32)
        v = make_float4(s_norm[resample_clip8(acc[0])].x, s_norm[resample_clip8(acc[1])].y, s_norm[resample_clip8(acc[2])].z, 0.0f);
      else
        v = make_uint2(__byte_perm(s_norm[resample_clip8(acc[0])].x, s_norm[resample_clip8(acc[1])].x, 0x7610),
                       s_norm[resample_clip8(acc[2])].y);
    }
    if constexpr (!U8)
      if (xp < WP) y[((long long)n * HP + yp) * WP + xp] = v;
  }
}

// y = max(x, 0) on fp16, 8 elements per thread (FPN pyramid7 reads ReLU(P6), fpn.py:55, while P6 itself is an output)
__global__ void relu_f16_kernel(const uint4 *__restrict__ x, uint4 *__restrict__ y, long long n8) {
  const __half2 z = __float2half2_rn(0.0f);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    uint4 v = __ldg(x + i);
    __half2 *h = reinterpret_cast<__half2 *>(&v);
#pragma unroll
    for (int j = 0; j < 4; j++) h[j] = __hmax2(h[j], z);
    y[i] = v;
  }
}

// 3-D strided copy (+ optional ReLU) of fp16 rows, 16 bytes per thread: moves a pyramid level between a dense
// [n, rows, row_elems] tensor and its rectangle inside the atlas (pitches in elements).
__global__ void copy_rows_f16_kernel(const __half *__restrict__ x, __half *__restrict__ y, int n, int rows, int row8,
                                     long long x_img, long long x_row, long long y_img, long long y_row, int relu) {
  const long long total = (long long)n * rows * row8;
  const __half2 z = __float2half2_rn(0.0f);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % row8);
    const long long t = i / row8;
    const int r = (int)(t % rows), im = (int)(t / rows);
    uint4 v = __ldg(reinterpret_cast<const uint4 *>(x + im * x_img + r * x_row) + c);
    if (relu) {
      __half2 *h = reinterpret_cast<__half2 *>(&v);
#pragma unroll
      for (int j = 0; j < 4; j++) h[j] = __hmax2(h[j], z);
    }
    reinterpret_cast<uint4 *>(y + im * y_img + r * y_row)[c] = v;
  }
}

// fp16 -> s8 with one per-tensor scale (the INT8 heads' input atlas): q = clamp(rint(x * inv_scale), -127, 127), 8
// elements per thread (16-byte load, 8-byte store).  Zeros stay zeros, so the atlas gap rows remain exact padding.
__global__ void quantize_f16_s8_kernel(const uint4 *__restrict__ x, uint2 *__restrict__ y, long long n8, float inv_scale) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    const uint4 v = __ldg(x + i);
    const __half2 *h = reinterpret_cast<const __half2 *>(&v);
    uint32_t out[2] = {0u, 0u};
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const float2 f = __half22float2(h[j]);
      const int q0 = min(max(__float2int_rn(__fmul_rn(f.x, inv_scale)), -127), 127);
      const int q1 = min(max(__float2int_rn(__fmul_rn(f.y, inv_scale)), -127), 127);
      out[j >> 1] |= (((uint32_t)q0 & 0xffu) | (((uint32_t)q1 & 0xffu) << 8)) << (16 * (j & 1));
    }
    y[i] = make_uint2(out[0], out[1]);
  }
}

// 3-D strided copy of s8 rows with ReLU, 16 bytes per thread (pyramid7's input ReLU(P6) from the s8 atlas): max with 0
// on symmetric s8 values is exact
__global__ void relu_copy_rows_s8_kernel(const int8_t *__restrict__ x, int8_t *__restrict__ y, int n, int rows, int row16,
                                         long long x_img, long long x_row, long long y_img, long long y_row) {
  const long long total = (long long)n * rows * row16;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % row16);
    const long long t = i / row16;
    const int r = (int)(t % rows), im = (int)(t / rows);
    uint4 v = __ldg(reinterpret_cast<const uint4 *>(x + im * x_img + r * x_row) + c);
    v.x = __vmaxs4(v.x, 0u); v.y = __vmaxs4(v.y, 0u); v.z = __vmaxs4(v.z, 0u); v.w = __vmaxs4(v.w, 0u);
    reinterpret_cast<uint4 *>(y + im * y_img + r * y_row)[c] = v;
  }
}

// ---- fp32 twins (full-precision mode, odtk_conv2d_f32) ----
// RGB NHWC3 fp32 -> zero-padded NHWC4 fp32 [n, h+6, w+8, 4], the border of pad_input_kernel.  One 16-byte pixel per thread.
__global__ void pad_input_f32_kernel(const float *__restrict__ x, float4 *__restrict__ y, int N, int H, int W) {
  const int HP = H + 6, WP = W + 8;
  const long long total = (long long)N * HP * WP;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int xp = (int)(i % WP);
    long long t = i / WP;
    int yp = (int)(t % HP);
    int n = (int)(t / HP);
    int ih = yp - 3, iw = xp - 3;
    float4 v = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    if (ih >= 0 && ih < H && iw >= 0 && iw < W) {
      const float *s = x + (((long long)n * H + ih) * W + iw) * 3;
      v = make_float4(__ldg(s), __ldg(s + 1), __ldg(s + 2), 0.0f);
    }
    y[i] = v;
  }
}

// preprocess_u8_kernel into the fp32 NHWC4 stem buffer
__global__ void preprocess_u8_f32_kernel(const unsigned char *__restrict__ x, float4 *__restrict__ y, int N, int H, int W,
                                         int HS, int WS, float m0, float m1, float m2, float s0, float s1, float s2) {
  const int HP = HS + 6, WP = WS + 8;
  const long long total = (long long)N * HP * WP;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int xp = (int)(i % WP);
    long long t = i / WP;
    int yp = (int)(t % HP);
    int n = (int)(t / HP);
    int ih = yp - 3, iw = xp - 3;
    float4 v = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    if (ih >= 0 && ih < H && iw >= 0 && iw < W) {
      const unsigned char *s = x + (((long long)n * H + ih) * W + iw) * 3;
      v = normalize_rgb_u8_f32(s[0], s[1], s[2], m0, m1, m2, s0, s1, s2);
    }
    y[i] = v;
  }
}

// 3x3 stride-2 pad-1 max-pool on NHWC fp32, 4 channels (16 bytes) per thread
__global__ void maxpool3x3s2_f32_kernel(const float *__restrict__ x, float *__restrict__ y, int N, int H, int W, int C,
                                        int OH, int OW) {
  const int c4n = C >> 2;
  const long long total = (long long)N * OH * OW * c4n;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int c4 = (int)(i % c4n);
    long long m = i / c4n;
    int ow = (int)(m % OW);
    long long t = m / OW;
    int oh = (int)(t % OH);
    int n = (int)(t / OH);
    float4 best = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
#pragma unroll
    for (int dy = 0; dy < 3; dy++) {
      int ih = oh * 2 + dy - 1;
      if (ih < 0 || ih >= H) continue;
#pragma unroll
      for (int dx = 0; dx < 3; dx++) {
        int iw = ow * 2 + dx - 1;
        if (iw < 0 || iw >= W) continue;
        const float4 v = __ldg(reinterpret_cast<const float4 *>(x + (((long long)n * H + ih) * W + iw) * C) + c4);
        best.x = fmaxf(best.x, v.x); best.y = fmaxf(best.y, v.y); best.z = fmaxf(best.z, v.z); best.w = fmaxf(best.w, v.w);
      }
    }
    reinterpret_cast<float4 *>(y + m * C)[c4] = best;
  }
}

// 3-D strided copy of fp32 rows with ReLU, 16 bytes per thread (pyramid7's input ReLU(P6) from the fp32 atlas)
__global__ void relu_copy_rows_f32_kernel(const float *__restrict__ x, float *__restrict__ y, int n, int rows, int row4,
                                          long long x_img, long long x_row, long long y_img, long long y_row) {
  const long long total = (long long)n * rows * row4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % row4);
    const long long t = i / row4;
    const int r = (int)(t % rows), im = (int)(t / rows);
    float4 v = __ldg(reinterpret_cast<const float4 *>(x + im * x_img + r * x_row) + c);
    v.x = fmaxf(v.x, 0.0f); v.y = fmaxf(v.y, 0.0f); v.z = fmaxf(v.z, 0.0f); v.w = fmaxf(v.w, 0.0f);
    reinterpret_cast<float4 *>(y + im * y_img + r * y_row)[c] = v;
  }
}

inline int grid_for(long long total, int threads) {
  long long b = (total + threads - 1) / threads;
  long long cap = (long long)odtk_sm_count() * 16;
  return (int)(b < cap ? (b < 1 ? 1 : b) : cap);
}

}  // namespace

extern "C" int odtk_lower_conv(const void *x, void *out, int n, int h, int w, int c, int ksize, int stride, int pad,
                               int kpad, int relu, odtk_stream_t stream_) {
  if (!x || !out || n <= 0 || h <= 0 || w <= 0 || c <= 0 || ksize <= 0 || stride <= 0 || pad < 0) return ODTK_E_INVALID;
  if (kpad < ksize * ksize * c || (kpad % 8)) return ODTK_E_INVALID;
  cudaStream_t stream = (cudaStream_t)stream_;
  const int oh = (h + 2 * pad - ksize) / stride + 1, ow = (w + 2 * pad - ksize) / stride + 1;
  if (c % 8 == 0 && kpad != ksize * ksize * c) return ODTK_E_INVALID;
  if (c % 8 != 0 && relu) return ODTK_E_UNSUPPORTED;
  OdtkProfScope prof(ODTK_PROF_LAYER, stream);
  if (c % 8 == 0) {
    long long total = (long long)n * oh * ow * ksize * ksize * (c / 8);
    lower_vec8_kernel<<<grid_for(total, 256), 256, 0, stream>>>((const __half *)x, (__half *)out, n, h, w, c, oh, ow,
                                                                ksize, stride, pad, kpad, relu);
  } else {
    long long total = (long long)n * oh * ow * (kpad / 8);
    lower_generic_kernel<<<grid_for(total, 256), 256, 0, stream>>>((const __half *)x, (__half *)out, n, h, w, c, oh,
                                                                   ow, ksize, stride, pad, kpad);
  }
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

extern "C" int odtk_maxpool3x3s2(const void *x, void *y, int n, int h, int w, int c, odtk_stream_t stream_) {
  if (!x || !y || n <= 0 || h <= 0 || w <= 0 || c <= 0 || (c % 8)) return ODTK_E_INVALID;
  const int oh = (h + 2 - 3) / 2 + 1, ow = (w + 2 - 3) / 2 + 1;
  long long total = (long long)n * oh * ow * (c / 8);
  OdtkProfScope prof(ODTK_PROF_LAYER, (cudaStream_t)stream_);
  maxpool3x3s2_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream_>>>((const __half *)x, (__half *)y, n, h, w,
                                                                               c, oh, ow);
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

extern "C" int odtk_pad_input(const void *x, void *y, int n, int h, int w, odtk_stream_t stream_) {
  if (!x || !y || n <= 0 || h <= 0 || w <= 0) return ODTK_E_INVALID;
  long long total = (long long)n * (h + 6) * (w + 8);
  OdtkProfScope prof(ODTK_PROF_LAYER, (cudaStream_t)stream_);
  if (w % 8 == 0 && (((uintptr_t)x | (uintptr_t)y) & 15) == 0 && (size_t)w * 6 <= 48 * 1024 && (long long)n * (h + 6) < (1ll << 31))
    pad_input_rows_kernel<<<n * (h + 6), 256, (size_t)w * 6, (cudaStream_t)stream_>>>((const __half *)x, (__half *)y, n, h, w);
  else
    pad_input_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream_>>>((const __half *)x, (__half *)y, n, h, w);
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

extern "C" int odtk_preprocess_u8(const void *x, void *y, int n, int h, int w, int hs, int ws, const float *mean,
                                  const float *std, odtk_stream_t stream_) {
  if (!x || !y || !mean || !std || n <= 0 || h <= 0 || w <= 0 || hs < h || ws < w) return ODTK_E_INVALID;
  long long total = (long long)n * (hs + 6) * (ws + 8);
  OdtkProfScope prof(ODTK_PROF_LAYER, (cudaStream_t)stream_);
  preprocess_u8_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream_>>>(
      (const unsigned char *)x, (__half *)y, n, h, w, hs, ws, mean[0], mean[1], mean[2], std[0], std[1], std[2]);
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

namespace {
template <bool F32>
long long preprocess_resize(const void *x, size_t x_bytes, const odtk_resize_image_t *images, const odtk_resize_image_t *images_dev,
                            int n, int canvas_h, int canvas_w, void *y, const float *mean, const float *std, odtk_stream_t stream_) {
  if (!images || n <= 0 || n > 65535 || canvas_h <= 0 || canvas_w <= 0 || (canvas_h % 2) || (canvas_w % 2)) return ODTK_E_INVALID;
  for (int i = 0; i < n; i++) {
    const odtk_resize_image_t &im = images[i];
    if (im.src_h <= 0 || im.src_w <= 0 || im.dst_h <= 0 || im.dst_w <= 0) return ODTK_E_INVALID;
    if (im.dst_h > canvas_h || im.dst_w > canvas_w) return ODTK_E_INVALID;
    if (im.offset < 0 || (unsigned long long)im.offset + (unsigned long long)im.src_h * im.src_w * 3 > x_bytes) return ODTK_E_INVALID;
  }
  const long long bytes = (long long)n * (canvas_h + 6) * (canvas_w + 8) * (F32 ? 16 : 8);
  if (!y) return bytes;
  if (!x || !images_dev || !mean || !std) return ODTK_E_INVALID;
  const dim3 grid((canvas_w + 8 + RS_TW - 1) / RS_TW, (canvas_h + 6 + RS_TH - 1) / RS_TH, n);
  OdtkProfScope prof(ODTK_PROF_LAYER, (cudaStream_t)stream_);
  preprocess_resize_u8_kernel<F32><<<grid, RS_TW * RS_ROWS, 0, (cudaStream_t)stream_>>>(
      (const unsigned char *)x, images_dev, (typename std::conditional<F32, float4, uint2>::type *)y, canvas_h, canvas_w,
      mean[0], mean[1], mean[2], std[0], std[1], std[2]);
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}
}  // namespace

extern "C" long long odtk_preprocess_resize_u8(const void *x, size_t x_bytes, const odtk_resize_image_t *images,
                                               const odtk_resize_image_t *images_dev, int n, int canvas_h, int canvas_w,
                                               void *y, const float *mean, const float *std, odtk_stream_t stream_) {
  return preprocess_resize<false>(x, x_bytes, images, images_dev, n, canvas_h, canvas_w, y, mean, std, stream_);
}

extern "C" long long odtk_preprocess_resize_u8_f32(const void *x, size_t x_bytes, const odtk_resize_image_t *images,
                                                   const odtk_resize_image_t *images_dev, int n, int canvas_h, int canvas_w,
                                                   void *y, const float *mean, const float *std, odtk_stream_t stream_) {
  return preprocess_resize<true>(x, x_bytes, images, images_dev, n, canvas_h, canvas_w, y, mean, std, stream_);
}

extern "C" long long odtk_resize_u8_packed(const void *x, size_t x_bytes, const odtk_resize_image_t *images,
                                           const odtk_resize_image_t *images_dev, const long long *out_off,
                                           const long long *out_off_dev, int n, void *y, size_t y_bytes,
                                           odtk_stream_t stream_) {
  if (!images || !out_off || n <= 0 || n > 65535) return ODTK_E_INVALID;
  long long packed = 0;
  int max_h = 0, max_w = 0;
  for (int i = 0; i < n; i++) {
    const odtk_resize_image_t &im = images[i];
    if (im.src_h <= 0 || im.src_w <= 0 || im.dst_h <= 0 || im.dst_w <= 0) return ODTK_E_INVALID;
    if (im.offset < 0 || (unsigned long long)im.offset + (unsigned long long)im.src_h * im.src_w * 3 > x_bytes) return ODTK_E_INVALID;
    const long long out = (long long)im.dst_h * im.dst_w * 3;
    if (y && (out_off[i] < 0 || (unsigned long long)out_off[i] + (unsigned long long)out > y_bytes)) return ODTK_E_INVALID;
    packed += out;
    max_h = max(max_h, im.dst_h);
    max_w = max(max_w, im.dst_w);
  }
  if (!y) return packed;
  if (!x || !images_dev || !out_off_dev) return ODTK_E_INVALID;
  const dim3 grid((max_w + RS_TW - 1) / RS_TW, (max_h + RS_TH - 1) / RS_TH, n);
  OdtkProfScope prof(ODTK_PROF_LAYER, (cudaStream_t)stream_);
  preprocess_resize_u8_kernel<false, true><<<grid, RS_TW * RS_ROWS, 0, (cudaStream_t)stream_>>>(
      (const unsigned char *)x, images_dev, (unsigned char *)y, 0, 0, 0.f, 0.f, 0.f, 1.f, 1.f, 1.f, out_off_dev);
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

extern "C" int odtk_pad_input_f32(const void *x, void *y, int n, int h, int w, odtk_stream_t stream_) {
  if (!x || !y || n <= 0 || h <= 0 || w <= 0 || ((uintptr_t)y & 15)) return ODTK_E_INVALID;
  const long long total = (long long)n * (h + 6) * (w + 8);
  OdtkProfScope prof(ODTK_PROF_LAYER, (cudaStream_t)stream_);
  pad_input_f32_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream_>>>((const float *)x, (float4 *)y, n, h, w);
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

extern "C" int odtk_preprocess_u8_f32(const void *x, void *y, int n, int h, int w, int hs, int ws, const float *mean,
                                      const float *std, odtk_stream_t stream_) {
  if (!x || !y || !mean || !std || n <= 0 || h <= 0 || w <= 0 || hs < h || ws < w || ((uintptr_t)y & 15)) return ODTK_E_INVALID;
  const long long total = (long long)n * (hs + 6) * (ws + 8);
  OdtkProfScope prof(ODTK_PROF_LAYER, (cudaStream_t)stream_);
  preprocess_u8_f32_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream_>>>(
      (const unsigned char *)x, (float4 *)y, n, h, w, hs, ws, mean[0], mean[1], mean[2], std[0], std[1], std[2]);
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

extern "C" int odtk_maxpool3x3s2_f32(const void *x, void *y, int n, int h, int w, int c, odtk_stream_t stream_) {
  if (!x || !y || n <= 0 || h <= 0 || w <= 0 || c <= 0 || (c % 4) || (((uintptr_t)x | (uintptr_t)y) & 15)) return ODTK_E_INVALID;
  const int oh = (h - 1) / 2 + 1, ow = (w - 1) / 2 + 1;
  const long long total = (long long)n * oh * ow * (c / 4);
  OdtkProfScope prof(ODTK_PROF_LAYER, (cudaStream_t)stream_);
  maxpool3x3s2_f32_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream_>>>((const float *)x, (float *)y, n, h, w, c, oh, ow);
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

extern "C" int odtk_relu_copy_rows_f32(const void *x, void *y, int n, int rows, int row_elems, long long x_img_pitch,
                                       long long x_row_pitch, long long y_img_pitch, long long y_row_pitch, odtk_stream_t stream_) {
  if (!x || !y || n <= 0 || rows <= 0 || row_elems <= 0 || (row_elems % 4)) return ODTK_E_INVALID;
  if ((x_img_pitch | x_row_pitch | y_img_pitch | y_row_pitch) % 4 || (((uintptr_t)x | (uintptr_t)y) & 15)) return ODTK_E_INVALID;
  const long long total = (long long)n * rows * (row_elems / 4);
  OdtkProfScope prof(ODTK_PROF_LAYER, (cudaStream_t)stream_);
  relu_copy_rows_f32_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream_>>>((const float *)x, (float *)y, n, rows, row_elems / 4,
                                                                                     x_img_pitch, x_row_pitch, y_img_pitch, y_row_pitch);
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

// Depthwise 3x3 convolution (MobileNetV2's inverted residual blocks, torchvision mobilenetv2.py InvertedResidual behind
// odtk/backbones/mobilenet.py:5-25), pad 1, stride 1 / 2, + bias (folded BatchNorm) + ReLU6.  NHWC fp16, 8 channels per
// thread (16-byte loads), fp32 accumulation in tap order; w: [9][c] fp16.  No contraction over channels: HBM / L2-bound.
__global__ void depthwise3x3_kernel(const __half *__restrict__ x, const __half *__restrict__ w, const float *__restrict__ bias,
                                    __half *__restrict__ y, int n, int h, int wd, int c, int oh, int ow, int stride, int act) {
  const int c8 = c >> 3;
  const long long total = (long long)n * oh * ow * c8;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int cc = (int)(i % c8);
    long long pix = i / c8;
    const int ox = (int)(pix % ow);
    pix /= ow;
    const int oy = (int)(pix % oh), img = (int)(pix / oh);
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; j++) acc[j] = 0.0f;
#pragma unroll
    for (int r = 0; r < 3; r++) {
      const int iy = oy * stride + r - 1;
      if (iy < 0 || iy >= h) continue;
#pragma unroll
      for (int s = 0; s < 3; s++) {
        const int ix = ox * stride + s - 1;
        if (ix < 0 || ix >= wd) continue;
        const uint4 xv = __ldg(reinterpret_cast<const uint4 *>(x + (((long long)img * h + iy) * wd + ix) * c + cc * 8));
        const uint4 wv = __ldg(reinterpret_cast<const uint4 *>(w + (long long)(r * 3 + s) * c + cc * 8));
        const __half2 *xh = reinterpret_cast<const __half2 *>(&xv), *wh = reinterpret_cast<const __half2 *>(&wv);
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const float2 a = __half22float2(xh[j]), b = __half22float2(wh[j]);
          acc[2 * j] = fmaf(a.x, b.x, acc[2 * j]);
          acc[2 * j + 1] = fmaf(a.y, b.y, acc[2 * j + 1]);
        }
      }
    }
    uint4 o;
    __half2 *oh2 = reinterpret_cast<__half2 *>(&o);
#pragma unroll
    for (int j = 0; j < 4; j++) {
      float a = acc[2 * j] + (bias ? __ldg(bias + cc * 8 + 2 * j) : 0.0f), b = acc[2 * j + 1] + (bias ? __ldg(bias + cc * 8 + 2 * j + 1) : 0.0f);
      if (act) { a = fmaxf(a, 0.0f); b = fmaxf(b, 0.0f); }
      if (act == 2) { a = fminf(a, 6.0f); b = fminf(b, 6.0f); }
      oh2[j] = __floats2half2_rn(a, b);
    }
    *reinterpret_cast<uint4 *>(y + (((long long)img * oh + oy) * ow + ox) * c + cc * 8) = o;
  }
}

extern "C" int odtk_depthwise3x3(const void *x, const void *w, const float *bias, void *y, int n, int h, int width, int c,
                                 int stride, int act, odtk_stream_t stream_) {
  if (!x || !w || !y || n <= 0 || h <= 0 || width <= 0 || c <= 0 || (c % 8) || (stride != 1 && stride != 2) || act < 0 || act > 2)
    return ODTK_E_INVALID;
  if (((uintptr_t)x | (uintptr_t)w | (uintptr_t)y) & 15) return ODTK_E_INVALID;
  const int oh = (h - 1) / stride + 1, ow = (width - 1) / stride + 1;
  const long long total = (long long)n * oh * ow * (c / 8);
  OdtkProfScope prof(ODTK_PROF_LAYER, (cudaStream_t)stream_);
  depthwise3x3_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream_>>>((const __half *)x, (const __half *)w, bias, (__half *)y, n, h,
                                                                              width, c, oh, ow, stride, act);
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

extern "C" int odtk_relu_f16(const void *x, void *y, long long n, odtk_stream_t stream_) {
  if (!x || !y || n <= 0 || (n % 8) || (((uintptr_t)x | (uintptr_t)y) & 15)) return ODTK_E_INVALID;
  OdtkProfScope prof(ODTK_PROF_LAYER, (cudaStream_t)stream_);
  relu_f16_kernel<<<grid_for(n / 8, 256), 256, 0, (cudaStream_t)stream_>>>((const uint4 *)x, (uint4 *)y, n / 8);
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

extern "C" int odtk_quantize_f16_s8(const void *x, void *y, long long n, float inv_scale, odtk_stream_t stream_) {
  if (!x || !y || n <= 0 || (n % 8) || ((uintptr_t)x & 15) || ((uintptr_t)y & 7)) return ODTK_E_INVALID;
  OdtkProfScope prof(ODTK_PROF_LAYER, (cudaStream_t)stream_);
  quantize_f16_s8_kernel<<<grid_for(n / 8, 256), 256, 0, (cudaStream_t)stream_>>>((const uint4 *)x, (uint2 *)y, n / 8, inv_scale);
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

extern "C" int odtk_relu_copy_rows_s8(const void *x, void *y, int n, int rows, int row_elems, long long x_img_pitch,
                                      long long x_row_pitch, long long y_img_pitch, long long y_row_pitch, odtk_stream_t stream_) {
  if (!x || !y || n <= 0 || rows <= 0 || row_elems <= 0 || (row_elems % 16)) return ODTK_E_INVALID;
  if ((x_img_pitch | x_row_pitch | y_img_pitch | y_row_pitch) % 16 || (((uintptr_t)x | (uintptr_t)y) & 15)) return ODTK_E_INVALID;
  const long long total = (long long)n * rows * (row_elems / 16);
  OdtkProfScope prof(ODTK_PROF_LAYER, (cudaStream_t)stream_);
  relu_copy_rows_s8_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream_>>>((const int8_t *)x, (int8_t *)y, n, rows, row_elems / 16,
                                                                                    x_img_pitch, x_row_pitch, y_img_pitch, y_row_pitch);
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

extern "C" int odtk_copy_rows_f16(const void *x, void *y, int n, int rows, int row_elems, long long x_img_pitch,
                                  long long x_row_pitch, long long y_img_pitch, long long y_row_pitch, int relu,
                                  odtk_stream_t stream_) {
  if (!x || !y || n <= 0 || rows <= 0 || row_elems <= 0 || (row_elems % 8)) return ODTK_E_INVALID;
  if ((x_img_pitch | x_row_pitch | y_img_pitch | y_row_pitch) % 8 || (((uintptr_t)x | (uintptr_t)y) & 15)) return ODTK_E_INVALID;
  const long long total = (long long)n * rows * (row_elems / 8);
  OdtkProfScope prof(ODTK_PROF_LAYER, (cudaStream_t)stream_);
  copy_rows_f16_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream_>>>((const __half *)x, (__half *)y, n, rows, row_elems / 8,
                                                                               x_img_pitch, x_row_pitch, y_img_pitch, y_row_pitch, relu);
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}
