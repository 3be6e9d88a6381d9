// stem.cu -- ResNet stem fused on the Hopper tensor cores (sm_90a): 7x7 stride-2 pad-3 convolution + bias (folded
// BatchNorm) + ReLU + 3x3 stride-2 pad-1 max-pool in ONE kernel; the [n, h/2, w/2, 64] stem activation is never written.
//
// A CTA tile is 5 x 5 pooled pixels.  Their 3x3 windows cover an 11 x 11 patch of stem pixels (121 accumulator rows,
// starting one stem row / column before 2 * the pooled origin), computed like odtk_stem_conv computes them: the A
// operand of filter row r is the overlapping-window 5-D tensor map of the zero-padded NHWC4 image (K = 32 per row,
// SWIZZLE_64B), 7 K blocks per tile, wgmma m64n64k16 with fp32 accumulation.  The epilogue rounds bias + accumulator
// to fp16 and applies ReLU exactly as the convolution epilogue does, stages the 11 x 11 x 64 tile in shared memory and
// pools it; stem pixels outside the image (the patch's first row / column at the top / left edge, its end at the
// bottom / right) are left out of the maximum, which is max-pool padding.  Bit-identical to odtk_stem_conv followed by
// odtk_maxpool3x3s2.
//   warpgroup 0     TMA producer (one thread): image patch + weight block per filter row, through an mbarrier ring.
//   warpgroups 1-2  64 of the 121 patch rows each: wgmma, epilogue; then all 256 threads pool.
#include <cuda.h>
#include <cuda_fp16.h>
#include <string.h>

#include <mutex>

#include "common.cuh"
#include "conv.cuh"
#include "prof.cuh"
#include "tc_ptx.cuh"
#include "wgmma.cuh"

namespace {

constexpr int kThreads = 384;
constexpr int kPool = 5;                    // pooled pixels per tile side
constexpr int kSide = 2 * kPool + 1;        // stem pixels per patch side: 11
constexpr int kRows = kSide * kSide;        // 121 accumulator rows
constexpr int kCout = 64;
constexpr int kABytes = 128 * 64;           // A: up to 128 rows x 32 fp16 (64 B)
constexpr int kStageBytes = kABytes + kCout * 64;
constexpr int kStages = 8;
constexpr int kTileBytes = kRows * kCout * 2;   // staged fp16 stem tile, [121][64]
constexpr int kSmemBytes = 1024 + kStages * kStageBytes + kTileBytes + 2 * kStages * 8;

struct StemParams {
  int N, OH, OW, PH, PW, tiles_h, tiles_w, total_tiles, relu;
  const float *bias;
  __half *out;
};

__global__ void __launch_bounds__(kThreads, 1)
stem_pool_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ StemParams p) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char *smem = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  __half *stile = reinterpret_cast<__half *>(smem + kStages * kStageBytes);
  uint64_t *full = reinterpret_cast<uint64_t *>(smem + kStages * kStageBytes + kTileBytes);
  uint64_t *empty = full + kStages;
  const int wg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0), tid = threadIdx.x & 127;
  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  grid_dep_launch_dependents();
  grid_dep_wait();
  const int per_img = p.tiles_h * p.tiles_w;
  auto origin = [&](int tile, int &img, int &ph0, int &pw0) {
    img = tile / per_img;
    const int r = tile - img * per_img;
    ph0 = (r / p.tiles_w) * kPool;
    pw0 = (r % p.tiles_w) * kPool;
  };
  int stage = 0;
  uint32_t phase = 0;

  if (wg == 0) {
    if (tid != 0) return;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      int img, ph0, pw0;
      origin(tile, img, ph0, pw0);
      for (int r = 0; r < 7; r++) {
        mbar_wait(&empty[stage], phase ^ 1u);
        unsigned char *s = smem + stage * kStageBytes;
        mbar_arrive_expect_tx(&full[stage], (uint32_t)(kRows * 64 + kCout * 64));
        // stem pixels (2 ph0 - 1 .., 2 pw0 - 1 ..): coordinate -1 is outside the map and zero-filled (never pooled)
        tma_load_5d(s, &tmA, &full[stage], 0, 2 * pw0 - 1, r, 2 * ph0 - 1, img);
        tma_load_2d(s + kABytes, &tmB, &full[stage], r * 32, 0);
        if (++stage == kStages) { stage = 0; phase ^= 1u; }
      }
    }
    return;
  }

  const int cw = wg - 1, warp = tid >> 5, lane = tid & 31, q = lane & 3, t = threadIdx.x - 128;
  float acc[32];
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    int img, ph0, pw0;
    origin(tile, img, ph0, pw0);
    int prev = -1;
    for (int r = 0; r < 7; r++) {
      mbar_wait(&full[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * kStageBytes);
      const uint64_t da = wgmma_desc(sa + (uint32_t)(cw * 64 * 64), 64), db = wgmma_desc(sa + kABytes, 64);
      wgmma_fence();
      Wgmma<64>::mma(acc, da, db, r ? 1 : 0);
      Wgmma<64>::mma(acc, da + 2, db + 2, 1);
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
      prev = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1u; }
    }
    wgmma_wait<0>();
    if (lane == 0) mbar_arrive(&empty[prev]);
    asm volatile("bar.sync 1, 256;" ::: "memory");   // the previous tile's pooling has read the staged tile
#pragma unroll
    for (int i = 0; i < 2; i++) {
      const int row = cw * 64 + warp * 16 + (lane >> 2) + 8 * i;
      if (row >= kRows) continue;
#pragma unroll
      for (int j = 0; j < 8; j++) {
        const int col = 8 * j + 2 * q;
        const float b0 = p.bias ? __ldg(p.bias + col) : 0.0f, b1 = p.bias ? __ldg(p.bias + col + 1) : 0.0f;
        __half2 v = __floats2half2_rn(acc[4 * j + 2 * i] + b0, acc[4 * j + 2 * i + 1] + b1);
        if (p.relu) v = __hmax2(v, __float2half2_rn(0.0f));
        *reinterpret_cast<__half2 *>(stile + row * kCout + col) = v;
      }
    }
    asm volatile("bar.sync 1, 256;" ::: "memory");
    // ---- 3x3 / 2 max-pool over the staged tile: 25 pooled pixels x 8 groups of 8 channels ----
    const int sh0 = 2 * ph0 - 1, sw0 = 2 * pw0 - 1;
    for (int it = t; it < kPool * kPool * 8; it += 256) {
      const int pix = it >> 3, cg = (it & 7) * 8, py = pix / kPool, px = pix - py * kPool;
      const int oh = ph0 + py, ow = pw0 + px;
      if (oh >= p.PH || ow >= p.PW) continue;
      __half2 m[4];
      bool any = false;
#pragma unroll
      for (int dy = 0; dy < 3; dy++) {
        const int ly = 2 * py + dy, gy = sh0 + ly;
        if (gy < 0 || gy >= p.OH) continue;
#pragma unroll
        for (int dx = 0; dx < 3; dx++) {
          const int lx = 2 * px + dx, gx = sw0 + lx;
          if (gx < 0 || gx >= p.OW) continue;
          const uint4 v = *reinterpret_cast<const uint4 *>(stile + (ly * kSide + lx) * kCout + cg);
          const __half2 *h = reinterpret_cast<const __half2 *>(&v);
#pragma unroll
          for (int k = 0; k < 4; k++) m[k] = any ? __hmax2(m[k], h[k]) : h[k];
          any = true;
        }
      }
      *reinterpret_cast<uint4 *>(p.out + (((long long)img * p.PH + oh) * p.PW + ow) * kCout + cg) = *reinterpret_cast<uint4 *>(m);
    }
  }
}

}  // namespace

// xp: zero-padded NHWC4 fp16 image [n, h+6, width+8, 4] (odtk_pad_input / odtk_preprocess_u8); w: [64, 7*32] fp16 packed
// like odtk_stem_conv's; y: NHWC fp16 [n, (h/2 - 1)/2 + 1, (width/2 - 1)/2 + 1, 64].  h, width even; cout == 64.
extern "C" int odtk_stem_pool(const void *xp, const void *w, const float *bias, void *y, int n, int h, int width, int cout,
                              int relu, odtk_stream_t stream_) {
  if (!xp || !w || !y || n <= 0 || h <= 0 || width <= 0) return ODTK_E_INVALID;
  if ((h & 1) || (width & 1) || cout != kCout) return ODTK_E_UNSUPPORTED;
  if (((uintptr_t)xp | (uintptr_t)w | (uintptr_t)y) & 15) return ODTK_E_INVALID;
  cudaStream_t stream = (cudaStream_t)stream_;
  static std::mutex mu;
  static bool configured[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return ODTK_E_CUDA;
  {
    std::lock_guard<std::mutex> lk(mu);
    if (!configured[dev]) {
      if (cudaFuncSetAttribute(stem_pool_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes) != cudaSuccess)
        return ODTK_E_CUDA;
      configured[dev] = true;
    }
  }
  StemParams p;
  memset(&p, 0, sizeof p);
  p.N = n; p.OH = h / 2; p.OW = width / 2;
  p.PH = (p.OH - 1) / 2 + 1; p.PW = (p.OW - 1) / 2 + 1;
  p.tiles_h = (p.PH + kPool - 1) / kPool; p.tiles_w = (p.PW + kPool - 1) / kPool;
  const long long total = (long long)n * p.tiles_h * p.tiles_w;
  if (total >= (1ll << 31) || (long long)n * p.OH * p.OW >= (1ll << 31)) return ODTK_E_UNSUPPORTED;
  p.total_tiles = (int)total;
  p.bias = bias; p.out = (__half *)y; p.relu = relu;
  const int HP = h + 6, WP = width + 8;
  CUtensorMap tmA, tmB;
  {   // the overlapping-window map of odtk_stem_conv: {32 elements, OW (16 B), 7 filter rows, OH (two padded rows), N}
    uint64_t dims[5] = {32, (uint64_t)p.OW, 7, (uint64_t)p.OH, (uint64_t)n};
    uint64_t str[4] = {16, (uint64_t)WP * 8, (uint64_t)WP * 16, (uint64_t)HP * WP * 8};
    uint32_t box[5] = {32, (uint32_t)kSide, 1, (uint32_t)kSide, 1};
    if (!encode_map(&tmA, xp, 5, dims, str, box, CU_TENSOR_MAP_SWIZZLE_64B)) return ODTK_E_UNSUPPORTED;
  }
  {
    uint64_t dims[2] = {224, (uint64_t)cout};
    uint64_t str[1] = {224 * 2};
    uint32_t box[2] = {32, (uint32_t)cout};
    if (!encode_map(&tmB, w, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_64B)) return ODTK_E_CUDA;
  }
  const int sms = odtk_sm_count();
  const int grid = p.total_tiles < sms ? p.total_tiles : sms;
  {
    OdtkProfScope prof(ODTK_PROF_CONV, stream);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = kSmemBytes;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = odtk_pdl_on() ? 1 : 0;
    cudaLaunchKernelEx(&cfg, stem_pool_kernel, tmA, tmB, p);
  }
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}
