// wgrad.cu -- backward of the head, FPN and ResNet stage 3-4 convolutions (sm_90a): the weight-gradient GEMM over the
// gradient atlas or a dense gradient, the bias gradient, the packing of the loss gradients into the fp16 gradient atlas,
// the FPN's top-down pathway backward and the scatter of a gradient into a strided layer's input geometry.
// The input gradient runs on conv_gemm_kernel (odtk_conv2d_dgrad, conv.cu).
//
//   dW[co, tap, ci] = sum over images and pixels (r, c) of  G[r, c, co] * X[s * (r - g_row0) + ky - p, s * c + kx - p, ci]
//
// (tap = ky * k + kx, p = k / 2) is a GEMM with M = Cout, N = k^2 * Cin and K = pixels.  One CTA owns a 128 x 128
// (co, tap-ci) output tile and a contiguous range of G's 8 x 16 pixel tiles (K split over CTAs so that 36 output tiles
// still fill the SMs):
//   warpgroup 0     TMA producer: per tile, two 64-channel boxes of G and two of X (the box under the tile, shifted by the
//                   tap; stride 2 through element-strided boxes, elementStrides 2 in H and W, as conv.cu loads odd-size
//                   stride-2 activations).
//   warpgroups 1-2  64 output channels each: wgmma m64n128k16 with BOTH operands MN-major (pixels are K, the outer
//                   dimension of the NHWC boxes): 128B-swizzled MN-major descriptors + the transpose immediates.
// Each CTA writes its fp32 partial tile; one reduce kernel sums the partials in split order and writes the [Cout, Cin, k, k]
// parameter layout, so the result is bit-identical run to run.  The bias gradient is a fixed-order column sum of G's level.
// A backbone convolution runs BatchNorm-folded (w' = w * gamma / sqrt(var + eps) per output channel); the reduce kernel's
// optional per-row scale turns d/dw' into d/dw without another pass over dw.
//
// Both entry points run the same launch routine:
//   odtk_conv_wgrad     (head layers) 3x3 stride 1: G and X are whole atlases of one geometry (g_row0 0) and the tile table
//                       lists every level's tiles, or both are dense tensors; the atlas's zero gap rows / columns and the
//                       hardware zero fill are the padding, exactly as in the forward pass.
//   odtk_conv_wgrad_ex  (FPN and backbone layers) 1x1, 3x3 stride 1 or 3x3 stride 2: G is one level of the gradient atlas
//                       (the level's slice of the tile table, first row g_row0), X a dense tensor.  G is zero outside the
//                       level (gap rows, columns right of a narrow level), so the in-bounds X values under it contribute
//                       nothing; the hardware zero fill outside X is the padding.  Without a tile table G is the dense
//                       output itself (the dense 8 x 16 tiles, g_row0 0; the TMA zero fill past its edge), which also
//                       admits 1x1 stride 2 (the ResNet downsample).  Up to 2048 channels on either side.
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

constexpr int kWThreads = 384;
constexpr int kWStages = 3;
constexpr int kBox = 128 * 128;          // one TMA box: 8 x 16 pixels x 64 fp16 channels = 16 KB
constexpr int kWStageBytes = 4 * kBox;   // G: 2 boxes (128 output channels); X: 2 boxes (128 input channels of one tap)
constexpr int kWSmem = kWStages * kWStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
constexpr int kMaxSplits = 32;
constexpr int kBiasBlocks = 264;

struct WgradParams {
  const int4 *tile_tab;   // atlas tile table (h0, w0, row limit, column limit) or NULL
  int tab_tiles;          // tiles per image
  int tiles_w;            // dense mode: tiles per tile row
  int n_tiles, mn_tiles;  // N tiles (taps * cin / 128); M x N tiles
  int cin, cout_pad;
  int ktiles, splits;     // K tiles (images x tiles) and the CTAs each output tile is split over
  float *ws;              // fp32 partials [splits, cout_pad, taps * cin]
  int ksize, stride, g_row0;   // taps ksize^2; X pixel s * (r - g_row0) + tap - ksize / 2
};

__global__ void __launch_bounds__(kWThreads, 1)
wgrad_kernel(const __grid_constant__ CUtensorMap tmG, const __grid_constant__ CUtensorMap tmX,
             const __grid_constant__ WgradParams p) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char *smem = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t *full = reinterpret_cast<uint64_t *>(smem + kWStages * kWStageBytes);
  uint64_t *empty = full + kWStages;
  const int wg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0), tid = threadIdx.x & 127;
  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmG) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmX) : "memory");
    for (int s = 0; s < kWStages; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8 /* one per consumer warp */); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // splits outer: the CTAs resident at the same time read the same pixel range (L2 hits across output tiles)
  const int split = blockIdx.x / p.mn_tiles, tile = blockIdx.x - split * p.mn_tiles;
  const int m_tile = tile / p.n_tiles, n_tile = tile - m_tile * p.n_tiles;
  const int m0 = m_tile * 128, n0 = n_tile * 128;
  const int tap = n0 / p.cin, ci0 = n0 - tap * p.cin;   // cin % 128 == 0: an N tile never straddles two taps
  const int k_begin = (int)((long long)p.ktiles * split / p.splits);
  const int k_end = (int)((long long)p.ktiles * (split + 1) / p.splits);

  if (wg == 0) {
    // ===================================== TMA producer =====================================
    if (tid != 0) return;
    const int dy = tap / p.ksize - p.ksize / 2, dx = tap % p.ksize - p.ksize / 2;
    int stage = 0;
    uint32_t phase = 0;
    for (int kt = k_begin; kt < k_end; kt++) {
      const int img = kt / p.tab_tiles, r = kt - img * p.tab_tiles;
      int h0, w0;
      if (p.tile_tab) { const int4 e = __ldg(p.tile_tab + r); h0 = e.x; w0 = e.y; }
      else { h0 = (r / p.tiles_w) * 8; w0 = (r % p.tiles_w) * 16; }
      mbar_wait(&empty[stage], phase ^ 1u);
      unsigned char *s = smem + stage * kWStageBytes;
      mbar_arrive_expect_tx(&full[stage], (uint32_t)kWStageBytes);
      tma_load_4d(s, &tmG, &full[stage], m0, w0, h0, img);
      tma_load_4d(s + kBox, &tmG, &full[stage], m0 + 64, w0, h0, img);   // past cout_pad: zero-filled, never stored
      const int xw = p.stride * w0 + dx, xh = p.stride * (h0 - p.g_row0) + dy;
      tma_load_4d(s + 2 * kBox, &tmX, &full[stage], ci0, xw, xh, img);
      tma_load_4d(s + 3 * kBox, &tmX, &full[stage], ci0 + 64, xw, xh, img);
      if (++stage == kWStages) { stage = 0; phase ^= 1u; }
    }
    return;
  }

  // ===================================== MMA + epilogue ======================================
  const int cw = wg - 1, warp = tid >> 5, lane = tid & 31, q = lane & 3;
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; i++) acc[i] = 0.0f;
  int stage = 0, prev = -1;
  uint32_t phase = 0;
  for (int kt = k_begin; kt < k_end; kt++) {
    mbar_wait(&full[stage], phase);
    const uint32_t s = smem_u32(smem + stage * kWStageBytes);
    // A = this warpgroup's G box (64 channels = one MN atom); B = the two X boxes, 64 channels (one MN atom, LBO) apart;
    // 8 pixel rows per K group (SBO 1024), 16 pixels per MMA = 2048 bytes
    const uint64_t da = wgmma_desc_mn(s + (uint32_t)(cw * kBox), kBox, 1024);
    const uint64_t db = wgmma_desc_mn(s + 2u * kBox, kBox, 1024);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 8; k++) WgmmaT128::mma(acc, da + (uint64_t)(k * (2048 >> 4)), db + (uint64_t)(k * (2048 >> 4)), 1);
    wgmma_commit();
    wgmma_wait<1>();   // the previous tile's MMAs are done reading their stage
    if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
    prev = stage;
    if (++stage == kWStages) { stage = 0; phase ^= 1u; }
  }
  wgmma_wait<0>();

  // thread holds rows (output channels) r and r + 8, columns 8 j + 2 q (+1)
  const int N = p.ksize * p.ksize * p.cin;
  float *ws = p.ws + (size_t)split * p.cout_pad * N;
#pragma unroll
  for (int i = 0; i < 2; i++) {
    const int co = m0 + cw * 64 + warp * 16 + (lane >> 2) + 8 * i;
    if (co >= p.cout_pad) continue;
    float *row = ws + (size_t)co * N + n0 + 2 * q;
#pragma unroll
    for (int j = 0; j < 16; j++) *reinterpret_cast<float2 *>(row + 8 * j) = make_float2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
  }
}

// bias gradient, pass 1: block b sums rows [rows * b / B, rows * (b + 1) / B) of g [rows, cpad] in row order, one thread
// per channel pair
__global__ void bgrad_partial_kernel(const __half *g, long long rows, int cpad, float *part) {
  const long long r0 = rows * blockIdx.x / gridDim.x, r1 = rows * (blockIdx.x + 1) / gridDim.x;
  for (int c = 2 * threadIdx.x; c < cpad; c += 2 * blockDim.x) {
    float s0 = 0.0f, s1 = 0.0f;
    const __half *col = g + c;
#pragma unroll 8
    for (long long r = r0; r < r1; r++) {
      const float2 v = __half22float2(*reinterpret_cast<const __half2 *>(col + r * cpad));
      s0 += v.x;
      s1 += v.y;
    }
    part[(size_t)blockIdx.x * cpad + c] = s0;
    part[(size_t)blockIdx.x * cpad + c + 1] = s1;
  }
}

// bias gradient of one atlas level, pass 1: the level's pixels of all images in order (img, row, column), `slab` = rows x
// atlas width of them per image, images `pitch` elements apart (g points at the level's first row); block b sums pixels
// [px * b / B, px * (b + 1) / B), one thread per channel pair
__global__ void bgrad_level_partial_kernel(const __half *g, long long px, long long slab, long long pitch, int cpad,
                                           float *part) {
  const long long r0 = px * blockIdx.x / gridDim.x, r1 = px * (blockIdx.x + 1) / gridDim.x;
  for (int c = 2 * threadIdx.x; c < cpad; c += 2 * blockDim.x) {
    float s0 = 0.0f, s1 = 0.0f;
    const long long img = r0 / slab;
    long long rem = r0 - img * slab;
    const __half *col = g + img * pitch + c;
    for (long long r = r0; r < r1; r++) {
      const float2 v = __half22float2(*reinterpret_cast<const __half2 *>(col + rem * cpad));
      s0 += v.x;
      s1 += v.y;
      if (++rem == slab) { rem = 0; col += pitch; }
    }
    part[(size_t)blockIdx.x * cpad + c] = s0;
    part[(size_t)blockIdx.x * cpad + c + 1] = s1;
  }
}

// dw[co, ci, tap] = sum over splits (in order) of ws[split, co, tap * cin + ci] (kScale: times row_scale[co], one rounding
// after the sum); db[co] = sum over blocks of part[b, co].  row_scale comes last so that the unscaled instances keep their
// parameter offsets.
template <int kTaps, bool kScale>
__global__ void wgrad_reduce_kernel(const float *ws, int splits, int cout, int cout_pad, int cin, float *dw,
                                    const float *part, int nparts, float *db, const float *row_scale) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long N = (long long)kTaps * cin;
  if (i < (long long)cout * cin) {
    const int co = (int)(i / cin), ci = (int)(i - (long long)co * cin);
    for (int t = 0; t < kTaps; t++) {
      const float *src = ws + (long long)co * N + (long long)t * cin + ci;
      float s = 0.0f;
      for (int k = 0; k < splits; k++) s += src[(long long)k * cout_pad * N];
      if constexpr (kScale) s *= __ldg(row_scale + co);
      dw[i * kTaps + t] = s;
    }
  }
  if (db && i < cout) {
    float s = 0.0f;
    for (int b = 0; b < nparts; b++) s += part[(long long)b * cout_pad + i];
    db[i] = s;
  }
}

// loss gradients (fp32 NCHW per level) -> fp16 NHWC gradient atlas: 32 pixels x 32 channels per block through shared memory
// (coalesced reads along the pixels, coalesced writes along the channels)
struct GradLevels {
  const float *grad[ODTK_MAX_LEVELS];
  int h[ODTK_MAX_LEVELS], w[ODTK_MAX_LEVELS], row0[ODTK_MAX_LEVELS];
  int blk0[ODTK_MAX_LEVELS + 1];   // first 32-pixel block of each level
};

__global__ void grad_to_atlas_kernel(const __grid_constant__ GradLevels L, int nl, int channels, const float *scale_ptr, __half *atlas,
                                     int rows, int aw, int cpad) {
  __shared__ float tile[32][33];
  const float scale = scale_ptr ? __ldg(scale_ptr) : 1.0f;
  const int img = blockIdx.z, c0 = blockIdx.y * 32;
  int l = 0;
  while (l + 1 < nl && (int)blockIdx.x >= L.blk0[l + 1]) l++;
  const int wl = L.w[l], hw = L.h[l] * wl;
  const int p0 = ((int)blockIdx.x - L.blk0[l]) * 32;
  const float *g = L.grad[l] + (size_t)img * channels * hw;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const int c = c0 + threadIdx.y + 8 * k, px = p0 + threadIdx.x;
    float v = 0.0f;
    if (c < channels && px < hw) v = g[(size_t)c * hw + px] * scale;
    tile[threadIdx.y + 8 * k][threadIdx.x] = v;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const int px = p0 + threadIdx.y + 8 * k;
    if (px >= hw) continue;
    const int y = px / wl, x = px - y * wl;
    // round to nearest: overflow is +-inf, never the largest finite half
    atlas[(((size_t)img * rows + L.row0[l] + y) * aw + x) * cpad + c0 + threadIdx.x] = __float2half_rn(tile[threadIdx.x][threadIdx.y + 8 * k]);
  }
}

constexpr int kMaxDevices = 64;
bool g_wgrad_ready[kMaxDevices];
std::mutex g_wgrad_mu;

bool wgrad_device_ready() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return false;
  std::lock_guard<std::mutex> lk(g_wgrad_mu);
  if (g_wgrad_ready[dev]) return true;
  if (cudaFuncSetAttribute(wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kWSmem) != cudaSuccess) return false;
  g_wgrad_ready[dev] = true;
  return true;
}

// K split: the number of splits (<= kMaxSplits, <= K tiles) whose CTA count fills the last wave best; fewer on ties
int choose_splits(int mn_tiles, int ktiles, int sms) {
  int best = 1;
  double best_eff = -1.0;
  for (int s = 1; s <= kMaxSplits && s <= ktiles; s++) {
    const long long total = (long long)mn_tiles * s;
    const long long waves = (total + sms - 1) / sms;
    const double eff = (double)total / (double)(waves * sms);
    if (eff > best_eff + 1e-9) { best_eff = eff; best = s; }
  }
  return best;
}

// One weight-gradient launch of either entry point, its arguments checked: G [n, g_rows, g_width, cout_pad], X [n, x_h,
// x_width, cin], the tiles of G from tile_tab (tab_tiles per image) or, tile_tab NULL, the dense 8 x 16 tiles of the
// g_rows x g_width image (tab_tiles = their count).  workspace NULL or workspace_size 0: returns the bytes needed.
long long wgrad_run(const odtk_wgrad_ex_t &d, void *workspace, size_t workspace_size, odtk_stream_t stream_) {
  const long long ktiles = (long long)d.n * d.tab_tiles;
  const int taps = d.ksize * d.ksize;
  const int N = taps * d.cin;
  const int n_tiles = N / 128, m_tiles = (d.cout_pad + 127) / 128;
  const int mn_tiles = m_tiles * n_tiles;
  const int sms = odtk_sm_count();
  const int splits = choose_splits(mn_tiles, (int)ktiles, sms);
  const size_t ws_part = odtk_align_up((size_t)splits * d.cout_pad * N * sizeof(float));
  const size_t ws_bias = odtk_align_up((size_t)kBiasBlocks * d.cout_pad * sizeof(float));
  const size_t need = ws_part + ws_bias;
  if (!workspace || workspace_size == 0) return (long long)need;
  if (workspace_size < need) return ODTK_E_WORKSPACE;
  if (!wgrad_device_ready()) return ODTK_E_CUDA;
  cudaStream_t stream = (cudaStream_t)stream_;

  CUtensorMap tmG, tmX;
  {
    const uint64_t C = (uint64_t)d.cout_pad, W = (uint64_t)d.g_width, H = (uint64_t)d.g_rows;
    uint64_t dims[4] = {C, W, H, (uint64_t)d.n};
    uint64_t str[3] = {C * 2, W * C * 2, H * W * C * 2};
    uint32_t box[4] = {64, 16, 8, 1};
    if (!encode_map(&tmG, d.g, 4, dims, str, box)) return ODTK_E_CUDA;
  }
  {
    // stride 2: boxDim = 2 x the pixels, elementStrides 2 -- the TMA unit loads every second pixel of a 32 x 16 window
    const uint64_t C = (uint64_t)d.cin, W = (uint64_t)d.x_width, H = (uint64_t)d.x_h;
    const uint32_t s = (uint32_t)d.stride;
    uint64_t dims[4] = {C, W, H, (uint64_t)d.n};
    uint64_t str[3] = {C * 2, W * C * 2, H * W * C * 2};
    uint32_t box[4] = {64, 16 * s, 8 * s, 1};
    uint32_t estr[4] = {1, s, s, 1};
    if (!encode_map(&tmX, d.x, 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, estr)) return ODTK_E_CUDA;
  }
  WgradParams p;
  memset(&p, 0, sizeof p);
  p.tile_tab = (const int4 *)d.tile_tab;
  p.tab_tiles = d.tab_tiles;
  p.tiles_w = (d.g_width + 15) / 16;
  p.n_tiles = n_tiles;
  p.mn_tiles = mn_tiles;
  p.cin = d.cin;
  p.cout_pad = d.cout_pad;
  p.ktiles = (int)ktiles;
  p.splits = splits;
  p.ws = (float *)workspace;
  p.ksize = d.ksize;
  p.stride = d.stride;
  p.g_row0 = d.g_row0;
  float *part = (float *)((char *)workspace + ws_part);
  {
    OdtkProfScope prof(ODTK_PROF_CONV, stream);
    wgrad_kernel<<<mn_tiles * splits, kWThreads, kWSmem, stream>>>(tmG, tmX, p);
    const int lh = (d.x_h - 1) / d.stride + 1;   // the level's rows
    if (d.db && lh == d.g_rows)                  // G is one level: its rows of all images are contiguous
      bgrad_partial_kernel<<<kBiasBlocks, 128, 0, stream>>>((const __half *)d.g, (long long)d.n * lh * d.g_width,
                                                           d.cout_pad, part);
    else if (d.db)
      bgrad_level_partial_kernel<<<kBiasBlocks, 128, 0, stream>>>(
          (const __half *)d.g + (size_t)d.g_row0 * d.g_width * d.cout_pad, (long long)d.n * lh * d.g_width,
          (long long)lh * d.g_width, (long long)d.g_rows * d.g_width * d.cout_pad, d.cout_pad, part);
    const long long elems = (long long)d.cout * d.cin;
    const unsigned blocks = (unsigned)((elems + 255) / 256);
    auto reduce = taps == 1 ? (d.row_scale ? wgrad_reduce_kernel<1, true> : wgrad_reduce_kernel<1, false>)
                            : (d.row_scale ? wgrad_reduce_kernel<9, true> : wgrad_reduce_kernel<9, false>);
    reduce<<<blocks, 256, 0, stream>>>(p.ws, splits, d.cout, d.cout_pad, d.cin, d.dw, part, kBiasBlocks, d.db, d.row_scale);
  }
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

}  // namespace

extern "C" long long odtk_conv_wgrad(const odtk_wgrad_t *d, void *workspace, size_t workspace_size, odtk_stream_t stream_) {
  if (!d || !d->g || !d->x || !d->dw) return ODTK_E_INVALID;
  if (d->n <= 0 || d->h <= 0 || d->width <= 0 || d->cin <= 0 || d->cout <= 0 || d->cout_pad <= 0) return ODTK_E_INVALID;
  if (d->cout > d->cout_pad) return ODTK_E_INVALID;
  if (d->cin % 128 || d->cout_pad % 64) return ODTK_E_UNSUPPORTED;   // 128-wide N tiles inside one tap; 64-channel G boxes
  if ((long long)d->n * d->h * d->width >= (1ll << 31)) return ODTK_E_UNSUPPORTED;
  if (((uintptr_t)d->g | (uintptr_t)d->x) & 15) return ODTK_E_INVALID;
  if (d->tile_tab && d->tab_tiles <= 0) return ODTK_E_INVALID;
  const int tiles_w = (d->width + 15) / 16;
  const int per_img = d->tile_tab ? d->tab_tiles : ((d->h + 7) / 8) * tiles_w;
  if ((long long)d->n * per_img >= (1ll << 31)) return ODTK_E_UNSUPPORTED;
  odtk_wgrad_ex_t e;
  memset(&e, 0, sizeof e);
  e.g = d->g; e.x = d->x; e.dw = d->dw; e.db = d->db;
  e.n = d->n; e.g_rows = e.x_h = d->h; e.g_width = e.x_width = d->width;
  e.cin = d->cin; e.cout = d->cout; e.cout_pad = d->cout_pad;
  e.ksize = 3; e.stride = 1;
  e.tile_tab = d->tile_tab; e.tab_tiles = per_img;
  return wgrad_run(e, workspace, workspace_size, stream_);
}

extern "C" int odtk_grad_to_atlas(int batch, int num_levels, const odtk_grad_level_t *levels, int channels, const float *scale,
                                  void *atlas, int rows, int atlas_width, int cout_pad, odtk_stream_t stream_) {
  if (!levels || !atlas || batch <= 0 || num_levels <= 0 || channels <= 0 || rows <= 0 || atlas_width <= 0)
    return ODTK_E_INVALID;
  if (num_levels > ODTK_MAX_LEVELS || batch > 65535) return ODTK_E_UNSUPPORTED;
  if (cout_pad < channels || cout_pad % 32 || ((uintptr_t)scale & 3)) return ODTK_E_INVALID;
  GradLevels L;
  memset(&L, 0, sizeof L);
  long long blocks = 0;
  for (int l = 0; l < num_levels; l++) {
    const odtk_grad_level_t &v = levels[l];
    if (!v.grad || v.height <= 0 || v.width <= 0 || v.row0 < 0) return ODTK_E_INVALID;
    if (v.width > atlas_width || (long long)v.row0 + v.height > rows) return ODTK_E_INVALID;
    if ((long long)channels * v.height * v.width >= (1ll << 31)) return ODTK_E_UNSUPPORTED;
    L.grad[l] = v.grad; L.h[l] = v.height; L.w[l] = v.width; L.row0[l] = v.row0;
    L.blk0[l] = (int)blocks;
    blocks += ((long long)v.height * v.width + 31) / 32;
  }
  if (blocks >= (1ll << 31)) return ODTK_E_UNSUPPORTED;
  L.blk0[num_levels] = (int)blocks;
  cudaStream_t stream = (cudaStream_t)stream_;
  {
    OdtkProfScope prof(ODTK_PROF_LAYER, stream);
    grad_to_atlas_kernel<<<dim3((unsigned)blocks, (unsigned)(cout_pad / 32), (unsigned)batch), dim3(32, 8), 0, stream>>>(
        L, num_levels, channels, scale, (__half *)atlas, rows, atlas_width, cout_pad);
  }
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

extern "C" long long odtk_conv_wgrad_ex(const odtk_wgrad_ex_t *d, void *workspace, size_t workspace_size, odtk_stream_t stream_) {
  if (!d || !d->g || !d->x || !d->dw) return ODTK_E_INVALID;
  const bool dense = !d->tile_tab;   // G is the convolution's whole dense output
  // 1x1 stride 2 (the ResNet downsample) only over a dense G: no FPN layer has that shape
  const bool mode_ok = (d->ksize == 1 && d->stride == 1) || (d->ksize == 3 && (d->stride == 1 || d->stride == 2)) ||
                       (d->ksize == 1 && d->stride == 2 && dense);
  if (dense && d->g_row0 != 0) return ODTK_E_INVALID;
  if (!mode_ok) return ODTK_E_UNSUPPORTED;
  if (d->n <= 0 || d->g_rows <= 0 || d->g_width <= 0 || d->g_row0 < 0 || d->x_h <= 0 || d->x_width <= 0 || d->cin <= 0 ||
      d->cout <= 0 || d->cout_pad <= 0 || (!dense && d->tab_tiles <= 0))
    return ODTK_E_INVALID;
  if (d->cout > d->cout_pad) return ODTK_E_INVALID;
  if (d->cin % 128 || d->cout_pad % 64) return ODTK_E_UNSUPPORTED;   // 128-wide N tiles inside one tap; 64-channel G boxes
  // the level is the convolution's output: (x - 1) / s + 1 rows and columns from row g_row0 of the atlas (dense: all of G)
  const int lh = (d->x_h - 1) / d->stride + 1, lw = (d->x_width - 1) / d->stride + 1;
  if ((long long)d->g_row0 + lh > d->g_rows || lw > d->g_width) return ODTK_E_INVALID;
  if (dense && (lh != d->g_rows || lw != d->g_width)) return ODTK_E_INVALID;
  if ((long long)d->n * d->g_rows * d->g_width >= (1ll << 31) || (long long)d->n * d->x_h * d->x_width >= (1ll << 31))
    return ODTK_E_UNSUPPORTED;
  if ((((uintptr_t)d->g | (uintptr_t)d->x | (uintptr_t)d->tile_tab) & 15) || ((uintptr_t)d->row_scale & 3)) return ODTK_E_INVALID;
  odtk_wgrad_ex_t e = *d;
  if (dense) e.tab_tiles = ((lh + 7) / 8) * ((lw + 15) / 16);   // wgrad_run's dense 8 x 16 tiles
  const long long ktiles = (long long)e.n * e.tab_tiles;
  if (ktiles >= (1ll << 31)) return ODTK_E_UNSUPPORTED;
  return wgrad_run(e, workspace, workspace_size, stream_);
}

// ---- the FPN's top-down pathway and pyramid7's input gradient: two small HBM-bound kernels over fp16 NHWC atlases -------
namespace {

// dst level (row0, h, w) += the pool x pool sums of src (row0, h, w) in fp32, 8 channels per thread:
//   out = fp16_rn((float)dst + ((s00 + s01) + (s10 + s11)))   (pool 2; pool 1: fp16_rn((float)dst + s00))
// source pixels past the source level count as 0
__global__ void pool_add_kernel(const __half *src, __half *dst, int n, int rows, int width, int c8, int sr0, int sh, int sw,
                                int dr0, int dh, int dw, int pool) {
  const long long total = (long long)n * dh * dw * c8;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int ch = (int)(i % c8);
  long long t = i / c8;
  const int x = (int)(t % dw);
  t /= dw;
  const int y = (int)(t % dh);
  const int img = (int)(t / dh);
  const long long img0 = (long long)img * rows;
  float s[4][8];
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const int sy = pool * y + (k >> 1), sx = pool * x + (k & 1);
    const bool in = (k == 0 || pool == 2) && sy < sh && sx < sw;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (in) v = *reinterpret_cast<const uint4 *>(src + (((img0 + sr0 + sy) * width + sx) * c8 + ch) * 8);
    const __half2 *h2 = reinterpret_cast<const __half2 *>(&v);
#pragma unroll
    for (int j = 0; j < 4; j++) { const float2 f = __half22float2(h2[j]); s[k][2 * j] = f.x; s[k][2 * j + 1] = f.y; }
  }
  __half *o = dst + (((img0 + dr0 + y) * width + x) * c8 + ch) * 8;
  uint4 v = *reinterpret_cast<const uint4 *>(o);
  __half2 *h2 = reinterpret_cast<__half2 *>(&v);
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const float2 f = __half22float2(h2[j]);
    const float a = f.x + ((s[0][2 * j] + s[1][2 * j]) + (s[2][2 * j] + s[3][2 * j]));
    const float b = f.y + ((s[0][2 * j + 1] + s[1][2 * j + 1]) + (s[2][2 * j + 1] + s[3][2 * j + 1]));
    h2[j] = __floats2half2_rn(a, b);
  }
  *reinterpret_cast<uint4 *>(o) = v;
}

// dst[dr0 + s y, s x] = src[sr0 + y, x] over the h x w source level; nothing else of dst is written.  kGeom false: dst has
// the source's geometry and s = 2 (the FPN's P7 -> P6 scatter); true: dst is [n, d_rows, d_width, c] and s is 1 or 2 (an
// atlas level into a dense tensor, a dense gradient into the even positions of a strided layer's input).
template <bool kGeom>
__global__ void dilate_kernel(const __half *src, __half *dst, int n, int rows, int width, int c8, int sr0, int h, int w, int dr0,
                              int d_rows, int d_width, int s) {
  const long long total = (long long)n * h * w * c8;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int ch = (int)(i % c8);
  long long t = i / c8;
  const int x = (int)(t % w);
  t /= w;
  const int y = (int)(t % h);
  if constexpr (kGeom) {
    const long long img = t / h;
    *reinterpret_cast<uint4 *>(dst + (((img * d_rows + dr0 + s * y) * d_width + s * x) * c8 + ch) * 8) =
        *reinterpret_cast<const uint4 *>(src + (((img * rows + sr0 + y) * width + x) * c8 + ch) * 8);
  } else {
    const long long img0 = (t / h) * rows;
    *reinterpret_cast<uint4 *>(dst + (((img0 + dr0 + 2 * y) * width + 2 * x) * c8 + ch) * 8) =
        *reinterpret_cast<const uint4 *>(src + (((img0 + sr0 + y) * width + x) * c8 + ch) * 8);
  }
}

}  // namespace

extern "C" int odtk_pool_add_f16(const void *src, void *dst, int n, int rows, int width, int c, int src_row0, int src_h,
                                 int src_w, int dst_row0, int dst_h, int dst_w, int pool, odtk_stream_t stream_) {
  if (!src || !dst || n <= 0 || rows <= 0 || width <= 0 || c <= 0 || (c % 8)) return ODTK_E_INVALID;
  if (pool != 1 && pool != 2) return ODTK_E_UNSUPPORTED;
  if (src_row0 < 0 || src_h <= 0 || src_w <= 0 || dst_row0 < 0 || dst_h <= 0 || dst_w <= 0) return ODTK_E_INVALID;
  if ((long long)src_row0 + src_h > rows || src_w > width || (long long)dst_row0 + dst_h > rows || dst_w > width)
    return ODTK_E_INVALID;
  if (src == dst && src_row0 < dst_row0 + dst_h && dst_row0 < src_row0 + src_h) return ODTK_E_INVALID;   // in place: disjoint levels
  if (((uintptr_t)src | (uintptr_t)dst) & 15) return ODTK_E_INVALID;
  const long long total = (long long)n * dst_h * dst_w * (c / 8);
  if ((long long)n * rows * width * c >= (1ll << 40)) return ODTK_E_UNSUPPORTED;
  {
    OdtkProfScope prof(ODTK_PROF_LAYER, (cudaStream_t)stream_);
    pool_add_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(
        (const __half *)src, (__half *)dst, n, rows, width, c / 8, src_row0, src_h, src_w, dst_row0, dst_h, dst_w, pool);
  }
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

extern "C" int odtk_dilate_f16(const void *src, void *dst, int n, int rows, int width, int c, int src_row0, int src_h,
                               int src_w, int dst_row0, odtk_stream_t stream_) {
  if (!src || !dst || n <= 0 || rows <= 0 || width <= 0 || c <= 0 || (c % 8)) return ODTK_E_INVALID;
  if (src_row0 < 0 || src_h <= 0 || src_w <= 0 || dst_row0 < 0) return ODTK_E_INVALID;
  if ((long long)src_row0 + src_h > rows || src_w > width || 2ll * (src_w - 1) >= width ||
      (long long)dst_row0 + 2ll * (src_h - 1) >= rows)
    return ODTK_E_INVALID;
  if (((uintptr_t)src | (uintptr_t)dst) & 15) return ODTK_E_INVALID;
  const long long total = (long long)n * src_h * src_w * (c / 8);
  if ((long long)n * rows * width * c >= (1ll << 40)) return ODTK_E_UNSUPPORTED;
  {
    OdtkProfScope prof(ODTK_PROF_LAYER, (cudaStream_t)stream_);
    dilate_kernel<false><<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(
        (const __half *)src, (__half *)dst, n, rows, width, c / 8, src_row0, src_h, src_w, dst_row0, 0, 0, 2);
  }
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

extern "C" int odtk_dilate_ex_f16(const void *src, void *dst, int n, int c, int src_rows, int src_width, int src_row0,
                                  int src_h, int src_w, int dst_rows, int dst_width, int dst_row0, int stride,
                                  odtk_stream_t stream_) {
  if (!src || !dst || n <= 0 || c <= 0 || (c % 8) || src_rows <= 0 || src_width <= 0 || dst_rows <= 0 || dst_width <= 0)
    return ODTK_E_INVALID;
  if (stride != 1 && stride != 2) return ODTK_E_UNSUPPORTED;
  if (src_row0 < 0 || src_h <= 0 || src_w <= 0 || dst_row0 < 0) return ODTK_E_INVALID;
  if ((long long)src_row0 + src_h > src_rows || src_w > src_width || (long long)stride * (src_w - 1) >= dst_width ||
      (long long)dst_row0 + (long long)stride * (src_h - 1) >= dst_rows)
    return ODTK_E_INVALID;
  if (src == dst) return ODTK_E_INVALID;
  if (((uintptr_t)src | (uintptr_t)dst) & 15) return ODTK_E_INVALID;
  const long long total = (long long)n * src_h * src_w * (c / 8);
  if ((long long)n * src_rows * src_width * c >= (1ll << 40) || (long long)n * dst_rows * dst_width * c >= (1ll << 40))
    return ODTK_E_UNSUPPORTED;
  {
    OdtkProfScope prof(ODTK_PROF_LAYER, (cudaStream_t)stream_);
    dilate_kernel<true><<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(
        (const __half *)src, (__half *)dst, n, src_rows, src_width, c / 8, src_row0, src_h, src_w, dst_row0, dst_rows,
        dst_width, stride);
  }
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}
