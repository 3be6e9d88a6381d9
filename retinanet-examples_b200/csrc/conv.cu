// conv.cu -- im2col-free implicit-GEMM convolution on the Hopper tensor cores (sm_90a, wgmma).
//
// Replaces the cuDNN convolutions behind nn.Conv2d in the reference's Model.forward
// (odtk/model.py:57-68,130-135, odtk/backbones/fpn.py:45-61, torchvision resnet blocks): the
// reference ships no convolution kernel of its own.  One persistent, warp-specialised kernel:
//
//   D[pixels, Cout] = sum over 64-channel chunks and taps (r,s) of  A_tap[pixels, 64] * W[Cout, 64]^T
//
//   warpgroup 0     TMA producer (one thread issues): cp.async.bulk.tensor loads of the activation operand straight
//                   from the NHWC tensor (the hardware zero-fills out-of-bounds rows/columns == conv padding: no
//                   im2col, no border code) and of the weight blocks (2-D map over [Cout, taps*Cin]) into swizzled
//                   shared memory, guarded by full/empty mbarriers.
//   warpgroups 1-2  MMA + epilogue, 64 accumulator rows (output pixels) each: wgmma.mma_async m64nNk16 (N = BN = 64
//                   or 128), fp32 accumulation in registers; the stage is released as soon as the next K block's
//                   MMAs are in flight.  The epilogue works on the registers: + bias, + residual / FPN nearest-
//                   upsample, ReLU / ReLU6, fp16 NHWC store -- or, for the last convolution of a head, (sigmoid +)
//                   fp32 NCHW in the layout the reference's decode entry point expects -- or, class head on the
//                   inference path, sigmoid + threshold + candidate append straight into the decode workspace.
//
// A-operand modes (ConvParams::mode):
//   0  1x1: 2-D [pixels, Cin] map (plain GEMM rows); optionally followed by K blocks of a second operand pair
//      (the projected identity of a bottleneck block: y = mid * W3^T + xproj * Wproj^T).
//   1  3x3 stride 1: one SHIFTED 4-D box per tap over a TH x TW pixel patch; a tile table maps the tiles of a
//      pyramid atlas.  Stride 2 on odd sizes: element-strided boxes (s2).
//   3  stride-2 1x1 / 3x3 on even sizes: parity-split 5-D view {2C, W/2, 2, H/2, N}.
//   2  7x7 stride-2 stem: overlapping-window 5-D map of the zero-padded NHWC4 image, 64-byte swizzle.
// Only Cin % 64 != 0 callers (RGB stems other than the 7x7) are first lowered to GEMM rows by layers.cu and run as mode 0.
#include <cuda.h>
#include <cuda_fp16.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>
#include <unordered_map>

#include "common.cuh"
#include "conv.cuh"
#include "prof.cuh"
#include "tc_ptx.cuh"
#include "wgmma.cuh"

namespace {

constexpr int kThreads = 384;
constexpr int kMaxStages = 8;
constexpr int kPipeBytes = 192 * 1024;   // 6 stages at BN = 128 (32 KB each), 8 at BN = 64
constexpr int kSmemBytes = kPipeBytes + 1024 /*align slack*/ + 256 /*barriers*/;

struct Barriers {
  uint64_t full[kMaxStages];
  uint64_t empty[kMaxStages];
};
static_assert(sizeof(Barriers) <= 256, "barrier block too small");

// ---------------------------------------------------------------------------------- kernel
template <int BN>
__global__ void __launch_bounds__(kThreads, 1)
conv_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2,
                 const __grid_constant__ ConvParams p) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char *smem = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  Barriers *bars = reinterpret_cast<Barriers *>(smem + kPipeBytes);
  const int kStages = p.nstages, rb = p.row_bytes;
  const int stage_bytes = (128 + BN) * rb;
  const int wg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0), tid = threadIdx.x & 127;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    for (int s = 0; s < kStages; s++) { mbar_init(&bars->full[s], 1); mbar_init(&bars->empty[s], 8 /* one per consumer warp */); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  grid_dep_launch_dependents();   // the next kernel's CTAs may take the SMs this grid frees (they wait for our completion)
  grid_dep_wait();                // everything above ran under the previous kernel's tail; its outputs are visible from here

  const int total_tiles = p.num_m_tiles * p.num_n_tiles;
  const int per_img = p.tile_tab ? p.tab_tiles : p.tiles_h * p.tiles_w;
  const int kb_main = p.taps * p.kblocks_per_tap, kb_all = kb_main + p.kblocks2;
  // tile origin: N fastest, so that the CTAs running at the same time share their input rows (one DRAM read, L2 hits)
  auto tile_origin = [&](int tile, int &m_tile, int &n_tile, int &img, int &h0, int &w0, int &hlim, int &wlim) {
    m_tile = tile / p.num_n_tiles;
    n_tile = tile - m_tile * p.num_n_tiles;
    img = 0; h0 = 0; w0 = 0; hlim = p.H; wlim = p.W;
    if (p.mode != 0) {
      img = m_tile / per_img;
      const int r = m_tile - img * per_img;
      h0 = (r / p.tiles_w) * p.TH;
      w0 = (r % p.tiles_w) * p.TW;
      if (p.tile_tab) { const int4 e = __ldg(p.tile_tab + r); h0 = e.x; w0 = e.y; hlim = e.z; wlim = e.w; }
    }
  };

  if (wg == 0) {
    // ===================================== TMA producer =====================================
    if (tid != 0) return;
    const uint32_t a_bytes = (uint32_t)((p.mode == 0 ? 128 : p.TH * p.TW) * rb), b_bytes = (uint32_t)(BN * rb);
    const int kelems = rb >> 1;   // K elements per block: 64 (SW128) or 32 (SW64)
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      int m_tile, n_tile, img, h0, w0, hlim, wlim;
      tile_origin(tile, m_tile, n_tile, img, h0, w0, hlim, wlim);
      const int n0 = n_tile * BN;
      // K order: 64-channel chunk outer, tap inner
      for (int kb = 0; kb < p.kblocks_per_tap; kb++) {
        const int kch = p.grouped ? n0 : kb * 64;   // input-channel coordinate: grouped convs read their own chunk only
        for (int tap = 0; tap < p.taps; tap++) {
          const int dy = tap / p.kw - p.pad, dx = tap % p.kw - p.pad;
          mbar_wait(&bars->empty[stage], phase ^ 1u);
          unsigned char *sa = smem + stage * stage_bytes;
          unsigned char *sb = sa + 128 * rb;
          mbar_arrive_expect_tx(&bars->full[stage], a_bytes + b_bytes);
          if (p.mode == 1) {
            tma_load_4d(sa, &tmA, &bars->full[stage], kch, (w0 << p.s2) + dx, (h0 << p.s2) + dy, img);
          } else if (p.mode == 3) {
            // stride 2: input pixel 2*o + d = 2*(o + (d < 0 ? -1 : 0)) + parity, on the parity-split 5-D view
            const int pw = dx < 0 ? 1 : dx, ph = dy < 0 ? 1 : dy;
            tma_load_5d(sa, &tmA, &bars->full[stage], pw * p.Cin + kch, w0 + (dx < 0 ? -1 : 0), ph, h0 + (dy < 0 ? -1 : 0), img);
          } else if (p.mode == 0) {
            tma_load_2d(sa, &tmA, &bars->full[stage], kch, m_tile * 128);
          } else {
            tma_load_5d(sa, &tmA, &bars->full[stage], 0, w0, tap, h0, img);   // stem: filter row `tap`
          }
          tma_load_2d(sb, &tmB, &bars->full[stage], (tap * p.kblocks_per_tap + kb) * kelems, n0);
          if (++stage == kStages) { stage = 0; phase ^= 1u; }
        }
      }
      for (int j = 0; j < p.kblocks2; j++) {
        mbar_wait(&bars->empty[stage], phase ^ 1u);
        unsigned char *sa = smem + stage * stage_bytes;
        mbar_arrive_expect_tx(&bars->full[stage], (uint32_t)((128 + BN) * 128));
        tma_load_2d(sa, &tmA2, &bars->full[stage], j * 64, m_tile * 128);
        tma_load_2d(sa + 128 * 128, &tmB2, &bars->full[stage], j * 64, n0);
        if (++stage == kStages) { stage = 0; phase ^= 1u; }
      }
    }
    return;
  }

  // ===================================== MMA + epilogue ======================================
  const int cw = wg - 1, warp = tid >> 5, lane = tid & 31;
  const int q = lane & 3;
  const int hw = p.H * p.W, patch = p.TH * p.TW;
  float acc[BN / 2];
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    int m_tile, n_tile, img0, h0, w0, hlim, wlim;
    tile_origin(tile, m_tile, n_tile, img0, h0, w0, hlim, wlim);
    const int n0 = n_tile * BN;
    int prev = -1;
    for (int kb = 0; kb < kb_all; kb++) {
      mbar_wait(&bars->full[stage], phase);
      const int brb = kb < kb_main ? rb : 128;
      const uint32_t sa = smem_u32(smem + stage * stage_bytes);
      const uint64_t da = wgmma_desc(sa + (uint32_t)(cw * 64 * brb), brb), db = wgmma_desc(sa + (uint32_t)(128 * brb), brb);
      wgmma_fence();
      if (brb == 128) {
#pragma unroll
        for (int k = 0; k < 4; k++) Wgmma<BN>::mma(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (kb | k) ? 1 : 0);
      } else {
#pragma unroll
        for (int k = 0; k < 2; k++) Wgmma<BN>::mma(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (kb | k) ? 1 : 0);
      }
      wgmma_commit();
      // the previous K block's MMAs have finished reading their stage once at most one group is in flight
      wgmma_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(&bars->empty[prev]);
      prev = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1u; }
    }
    wgmma_wait<0>();
    if (prev >= 0 && lane == 0) mbar_arrive(&bars->empty[prev]);

    // ---- epilogue: thread holds rows r and r + 8, columns 8 j + 2 q (+1) ----
#pragma unroll
    for (int i = 0; i < 2; i++) {
      const int row = cw * 64 + warp * 16 + (lane >> 2) + 8 * i;
      bool valid;
      int img, h, w;
      long long m;   // dense pixel index (residual / mode-0 rows)
      if (p.mode != 0) {
        const int dh = row / p.TW, dw = row - dh * p.TW;
        img = img0; h = h0 + dh; w = w0 + dw;
        valid = row < patch && h < hlim && w < wlim;
        m = ((long long)img * p.H + h) * p.W + w;
      } else {
        m = (long long)m_tile * 128 + row;
        valid = m < p.M;
        img = (int)(m / hw);
        const int rem = (int)(m - (long long)img * hw);
        h = rem / p.W;
        w = rem - h * p.W;
      }
      if (p.out_mode == ODTK_OUT_NHWC_F16) {
        if (!valid) continue;
        const long long opix = p.mode != 0 ? ((long long)img * p.oH + p.oR + h) * p.oW + w : m;
        __half *o = reinterpret_cast<__half *>(p.out) + opix * p.ldy;
        const __half *res = p.residual ? p.residual + m * p.ldr : nullptr;
        const __half *up = p.upsample ? p.upsample + (((long long)img * p.up_h + (h >> 1)) * p.up_w + (w >> 1)) * p.Cout : nullptr;
#pragma unroll
        for (int j = 0; j < BN / 8; j++) {
          const int col = n0 + 8 * j + 2 * q;
          if (col >= p.Cout) continue;   // Cout % 16 == 0: both columns of the pair are in range or neither
          float v0 = acc[4 * j + 2 * i], v1 = acc[4 * j + 2 * i + 1];
          if (p.bias) { v0 += __ldg(p.bias + col); v1 += __ldg(p.bias + col + 1); }
          if (res) { const float2 r = __half22float2(*reinterpret_cast<const __half2 *>(res + col)); v0 += r.x; v1 += r.y; }
          if (up) { const float2 u = __half22float2(*reinterpret_cast<const __half2 *>(up + col)); v0 += u.x; v1 += u.y; }
          __half2 y = __floats2half2_rn(v0, v1);
          if (p.relu) {   // on the packed halves: max(round(x), 0) == round(max(x, 0))
            y = __hmax2(y, __float2half2_rn(0.0f));
            if (p.relu == 2) y = __hmin2(y, __float2half2_rn(6.0f));   // ReLU6: 6.0 is exact in fp16
          }
          *reinterpret_cast<__half2 *>(o + col) = y;
        }
      } else if (p.out_mode == ODTK_OUT_CANDIDATES) {
        // class-head final layer: only the scores above the threshold leave the SM, appended to the decode workspace as
        // (key, flat NCHW index) pairs + the key histogram, exactly what decode.cu's score_filter_kernel would have
        // produced from the dense map.  Pass 1 counts this row's hits (one slot reservation per thread and row), pass 2
        // writes them.
        if (!valid) continue;
        const int pix = h * p.W + w;
        auto score = [&](int j, int k, float &sc) -> bool {
          const int col = n0 + 8 * j + 2 * q + k;
          if (col >= p.Cout) return false;
          float x = acc[4 * j + 2 * i + k] + (p.bias ? __ldg(p.bias + col) : 0.0f);
          if (p.relu) x = fmaxf(x, 0.0f);
          if (!(x > p.cand_pre)) return false;
          sc = sigmoidf_accurate(x);
          return sc > p.cand_thresh;
        };
        int cnt = 0;
#pragma unroll
        for (int j = 0; j < BN / 8; j++)
#pragma unroll
          for (int k = 0; k < 2; k++) { float sc; if (score(j, k, sc)) cnt++; }
        if (!cnt) continue;
        int base = atomicAdd(p.cand_counts + img, cnt);
        uint2 *dst = p.cand + (long long)img * p.cand_cap;
        unsigned *hist = p.cand_hist + (long long)img * p.cand_hist_bins;
#pragma unroll
        for (int j = 0; j < BN / 8; j++)
#pragma unroll
          for (int k = 0; k < 2; k++) {
            float sc;
            if (!score(j, k, sc)) continue;
            const uint32_t key = odtk_float_key(sc);
            if ((long long)base < p.cand_cap) dst[base] = make_uint2(key, (uint32_t)((n0 + 8 * j + 2 * q + k) * hw + pix));
            base++;
            const uint32_t dd = (key - p.cand_key_thresh) >> p.cand_shift;
            atomicAdd(hist + (dd < (uint32_t)(p.cand_hist_bins - 1) ? dd : (uint32_t)(p.cand_hist_bins - 1)), 1u);
          }
      } else {
        // fp32 NCHW (+ sigmoid)
        if (!valid) continue;
        float *o = reinterpret_cast<float *>(p.out) + (long long)img * p.Cout * hw + (long long)h * p.W + w;
#pragma unroll
        for (int j = 0; j < BN / 8; j++)
#pragma unroll
          for (int k = 0; k < 2; k++) {
            const int col = n0 + 8 * j + 2 * q + k;
            if (col >= p.Cout) continue;
            float x = acc[4 * j + 2 * i + k] + (p.bias ? __ldg(p.bias + col) : 0.0f);
            if (p.relu) x = fmaxf(x, 0.0f);
            if (p.out_mode == ODTK_OUT_NCHW_F32_SIGMOID) x = sigmoidf_accurate(x);
            o[(long long)col * hw] = x;
          }
      }
    }
  }
}

// ---------------------------------------------------------------------------------- host
// ---------------------------------------------------------------------------------- host
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void *ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess)
      return nullptr;
    fn = (EncodeTiledFn)ptr;
  }
  return fn;
}

// Encoded descriptors are pure functions of (base, geometry): cache them, so that eager / batch-1 callers stop paying
// 3-7 driver encodes per convolution (a CUDA-graph replay never did).  Keyed by value; bounded; thread-safe.
struct MapKey {
  const void *base;
  int rank, swz;
  uint64_t dims[5], strides[4];
  uint32_t box[5], es[5];
  bool operator==(const MapKey &o) const { return memcmp(this, &o, sizeof(MapKey)) == 0; }
};
struct MapKeyHash {
  size_t operator()(const MapKey &k) const {
    const unsigned char *b = reinterpret_cast<const unsigned char *>(&k);
    uint64_t h = 1469598103934665603ull;
    for (size_t i = 0; i < sizeof(MapKey); i++) { h ^= b[i]; h *= 1099511628211ull; }
    return (size_t)h;
  }
};
std::mutex g_map_mu;
std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_map_cache;
long long g_map_hits = 0, g_map_misses = 0;

}  // namespace

bool encode_map(CUtensorMap *m, const void *base, int rank, const uint64_t *dims, const uint64_t *strides_bytes,
                const uint32_t *box, CUtensorMapSwizzle swz, const uint32_t *elem_strides) {
  MapKey key;
  memset(&key, 0, sizeof key);
  key.base = base; key.rank = rank; key.swz = (int)swz;
  for (int i = 0; i < rank; i++) { key.dims[i] = dims[i]; key.box[i] = box[i]; key.es[i] = elem_strides ? elem_strides[i] : 1; }
  for (int i = 0; i < rank - 1; i++) key.strides[i] = strides_bytes[i];
  {
    std::lock_guard<std::mutex> lk(g_map_mu);
    auto it = g_map_cache.find(key);
    if (it != g_map_cache.end()) { *m = it->second; g_map_hits++; return true; }
  }
  EncodeTiledFn fn = get_encode();
  if (!fn) return false;
  cuuint64_t gdim[5], gstr[5];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; i++) { gdim[i] = dims[i]; bx[i] = box[i]; es[i] = key.es[i]; }
  for (int i = 0; i < rank - 1; i++) gstr[i] = strides_bytes[i];
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void *>(base), gdim, gstr, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return false;
  std::lock_guard<std::mutex> lk(g_map_mu);
  if (g_map_cache.size() >= 8192) g_map_cache.clear();
  g_map_cache.emplace(key, *m);
  g_map_misses++;
  return true;
}

// pick the spatial patch (TW x TH <= 128 pixels) that wastes the fewest accumulator rows
void choose_patch(int H, int W, int &TH, int &TW) {
  double best = -1;
  TH = 1; TW = 1;
  for (int tw = 1; tw <= 128 && tw <= W; tw++) {
    int thmax = 128 / tw;
    if (thmax > H) thmax = H;
    for (int th = 1; th <= thmax; th++) {
      long long tiles = (long long)((W + tw - 1) / tw) * ((H + th - 1) / th);
      double eff = (double)H * W / ((double)tiles * 128.0);
      // prefer wide patches on ties (coalesced NCHW stores, fewer TMA rows)
      if (eff > best + 1e-9 || (eff > best - 1e-9 && tw > TW)) { best = eff; TH = th; TW = tw; }
    }
  }
}

namespace {

template <int BN>
void launch_bn(int grid, cudaStream_t stream, const CUtensorMap &tmA, const CUtensorMap &tmB, const CUtensorMap &tmA2,
               const CUtensorMap &tmB2, const ConvParams &p) {
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
  cudaLaunchKernelEx(&cfg, conv_gemm_kernel<BN>, tmA, tmB, tmA2, tmB2, p);
}

// Per-device state (one process may drive several GPUs): the > 48 KB dynamic-shared-memory opt-in of every kernel
// instance is a per-device function attribute.
constexpr int kMaxDevices = 64;
bool g_dev_ready[kMaxDevices];
std::mutex g_dev_mu;

bool device_ready() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return false;
  std::lock_guard<std::mutex> lk(g_dev_mu);
  if (g_dev_ready[dev]) return true;
  if (cudaFuncSetAttribute(conv_gemm_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes) != cudaSuccess ||
      cudaFuncSetAttribute(conv_gemm_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes) != cudaSuccess)
    return false;
  g_dev_ready[dev] = true;
  return true;
}

thread_local odtk_conv_plan_t g_last_plan;

void set_stages(ConvParams &p, int BN) {
  p.nstages = kPipeBytes / ((128 + BN) * p.row_bytes);
  if (p.nstages > kMaxStages) p.nstages = kMaxStages;
}

int launch(const ConvParams &p, int BN, const CUtensorMap &tmA, const CUtensorMap &tmB, const CUtensorMap &tmA2,
           const CUtensorMap &tmB2, cudaStream_t stream) {
  const int total = p.num_m_tiles * p.num_n_tiles;
  const int sms = odtk_sm_count();   // the launch budget (odtk_set_sm_budget) or the whole device
  const int grid = total < sms ? total : sms;
  g_last_plan = odtk_conv_plan_t{p.mode, 0, BN, p.num_m_tiles, p.num_n_tiles, p.nstages, 0, 0, 0, 0, 0, 0, p.TH, p.TW, grid, 0};
  {
    OdtkProfScope prof(ODTK_PROF_CONV, stream);
    if (BN == 64) launch_bn<64>(grid, stream, tmA, tmB, tmA2, tmB2, p);
    else          launch_bn<128>(grid, stream, tmA, tmB, tmA2, tmB2, p);
  }
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

// odtk_conv2d, plus (mode 0 only) a second operand pair added to the same accumulator: y = x * w^T + x2 * w2^T with
// x2 [M, c2in], w2 [cout, c2in] (the projected identity of a bottleneck block)
int conv_run(const odtk_conv_t *d, const void *x2, const void *w2, int c2in, cudaStream_t stream) {
  if (!d || !d->x || !d->w) return ODTK_E_INVALID;
  if (d->out_mode == ODTK_OUT_CANDIDATES ? !d->sink : !d->y) return ODTK_E_INVALID;
  if (d->n <= 0 || d->h <= 0 || d->width <= 0 || d->cin <= 0 || d->cout <= 0) return ODTK_E_INVALID;
  if (d->ksize != 1 && d->ksize != 3) return ODTK_E_UNSUPPORTED;
  if (d->cin % 64 != 0) return ODTK_E_UNSUPPORTED;  // 64-channel K blocks (128-byte swizzle rows)
  const int groups = d->groups > 1 ? d->groups : 1;
  if (groups > 1) {
    // grouped convolution (ResNeXt conv2): output block j of 64 channels depends only on input chunk j, as long as a
    // group never straddles a 64-channel chunk; `w` is then [cout, ksize*ksize*64], block-diagonal inside the chunk
    if (d->cin != d->cout || d->cin % groups || 64 % (d->cin / groups) || d->residual || d->upsample || d->ksize != 3 ||
        d->out_mode != ODTK_OUT_NHWC_F16)
      return ODTK_E_UNSUPPORTED;
  }
  if (d->out_mode < 0 || d->out_mode > 3) return ODTK_E_INVALID;
  if (d->relu == 2 && d->out_mode != ODTK_OUT_NHWC_F16) return ODTK_E_UNSUPPORTED;   // ReLU6 only on fp16 activations
  if (d->out_mode == ODTK_OUT_NHWC_F16 && (d->cout % 16)) return ODTK_E_UNSUPPORTED;
  if (d->out_mode != ODTK_OUT_NHWC_F16 && (d->residual || d->upsample)) return ODTK_E_UNSUPPORTED;
  if ((long long)d->n * d->h * d->width >= (1ll << 31)) return ODTK_E_UNSUPPORTED;
  if (((uintptr_t)d->x | (uintptr_t)d->w | (d->out_mode == ODTK_OUT_CANDIDATES ? 0 : (uintptr_t)d->y)) & 15) return ODTK_E_INVALID;
  if ((d->residual && ((uintptr_t)d->residual & 3)) || (d->upsample && ((uintptr_t)d->upsample & 3))) return ODTK_E_INVALID;
  if (!device_ready()) return ODTK_E_CUDA;
  const int sms = odtk_sm_count();
  ConvParams p;
  memset(&p, 0, sizeof p);
  p.N = d->n; p.H = d->h; p.W = d->width; p.Cin = d->cin; p.Cout = d->cout;
  p.kw = d->ksize; p.taps = d->ksize * d->ksize; p.pad = d->ksize / 2;
  p.kblocks_per_tap = groups > 1 ? 1 : d->cin / 64;
  p.grouped = groups > 1;
  p.row_bytes = 128;
  p.M = (long long)d->n * d->h * d->width;
  p.bias = d->bias;
  p.residual = (const __half *)d->residual;
  p.upsample = (const __half *)d->upsample;
  p.out = d->y;
  p.relu = d->relu;
  p.out_mode = d->out_mode;
  p.ldy = d->ldy > 0 ? d->ldy : d->cout;
  p.ldr = d->ldr > 0 ? d->ldr : d->cout;
  p.up_h = d->h / 2; p.up_w = d->width / 2;
  if (p.out_mode == ODTK_OUT_CANDIDATES) {
    const odtk_cand_sink_t *k = d->sink;
    if (!k->counts || !k->hist || !k->cand || k->hist_bins <= 0) return ODTK_E_INVALID;
    if ((long long)d->cout * d->h * d->width >= (1ll << 32)) return ODTK_E_UNSUPPORTED;
    p.cand_counts = k->counts; p.cand_hist = k->hist; p.cand = (uint2 *)k->cand; p.cand_cap = k->cap;
    p.cand_key_thresh = k->key_thresh; p.cand_shift = k->shift; p.cand_hist_bins = k->hist_bins;
    p.cand_thresh = k->thresh;
    // sigmoid(x) > thresh implies x > logit(thresh) - margin (the SFU sigmoid is accurate to 1e-6 relative)
    p.cand_pre = (k->thresh > 1e-4f && k->thresh < 0.999f) ? logf(k->thresh / (1.0f - k->thresh)) - 0.05f : -INFINITY;
  }
  if (p.out_mode == ODTK_OUT_NHWC_F16 && (p.ldy % 8)) return ODTK_E_INVALID;
  if ((p.residual && (p.ldr & 1)) || (d->upsample && ((d->h & 1) || (d->width & 1)))) return ODTK_E_INVALID;
  const int stride = d->stride > 1 ? d->stride : 1;
  if (stride != 1 && stride != 2) return ODTK_E_UNSUPPORTED;
  // strided views: the input / output may be a rectangle of a larger NHWC buffer (a level of the pyramid atlas)
  const uint64_t xH = d->x_rows > 0 ? (uint64_t)d->x_rows : (uint64_t)d->h, xW = d->x_width > 0 ? (uint64_t)d->x_width : (uint64_t)d->width;
  const bool x_view = xH != (uint64_t)d->h || xW != (uint64_t)d->width;
  const bool y_view = d->y_rows > 0 || d->y_width > 0 || d->y_row_off > 0;
  if ((x_view || y_view || d->tile_tab) && (d->ksize != 3 || d->residual || d->upsample)) return ODTK_E_UNSUPPORTED;
  if (y_view && d->out_mode != ODTK_OUT_NHWC_F16) return ODTK_E_UNSUPPORTED;
  if (d->tile_tab && (d->tab_tiles <= 0 || stride != 1 || x_view || y_view)) return ODTK_E_INVALID;
  if (x2 && (d->ksize != 1 || stride != 1 || c2in <= 0 || c2in % 64 || !w2 || (((uintptr_t)x2 | (uintptr_t)w2) & 15))) return ODTK_E_INVALID;

  CUtensorMap tmA;
  if (stride == 2 && ((d->h & 1) || (d->width & 1) || x_view)) {
    // stride-2 1x1 / 3x3 (pad ksize/2) on odd sizes, im2col-free: one box per tap whose W and H dimensions are
    // traversed with element stride 2 (boxDim = 2 * pixels, elementStrides = 2: the TMA unit loads every second
    // pixel); the box origin 2*o + d may be -1 or reach past the edge: zero-filled == padding.
    const int OH = (d->h - 1) / 2 + 1, OW = (d->width - 1) / 2 + 1;
    p.mode = 1;
    p.s2 = 1;
    p.H = OH; p.W = OW;
    p.M = (long long)d->n * OH * OW;
    p.up_h = OH / 2; p.up_w = OW / 2;
    choose_patch(OH, OW, p.TH, p.TW);
    if (2 * p.TW > 256 || 2 * p.TH > 256) return ODTK_E_UNSUPPORTED;
    p.tiles_h = (OH + p.TH - 1) / p.TH;
    p.tiles_w = (OW + p.TW - 1) / p.TW;
    p.num_m_tiles = d->n * p.tiles_h * p.tiles_w;
    const uint64_t C = (uint64_t)d->cin, W = (uint64_t)d->width, H = (uint64_t)d->h;
    uint64_t dims[4] = {C, W, H, (uint64_t)d->n};
    uint64_t str[3] = {C * 2, xW * C * 2, xH * xW * C * 2};
    uint32_t box[4] = {64, (uint32_t)(2 * p.TW), (uint32_t)(2 * p.TH), 1};
    uint32_t es[4] = {1, 2, 2, 1};
    if (!encode_map(&tmA, d->x, 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, es)) return ODTK_E_CUDA;
  } else if (stride == 2) {
    // stride-2 1x1 / 3x3 (pad ksize/2) on even-sized inputs: 5-D parity-split view of the NHWC tensor
    // {2C (column parity x channel), W/2, 2 (row parity), H/2, N}; out-of-range half-rows/columns
    // (the -1 of the top/left taps) are zero-filled by the TMA unit == padding.
    if (d->upsample) return ODTK_E_UNSUPPORTED;
    const int OH = d->h / 2, OW = d->width / 2;
    p.mode = 3;
    p.H = OH; p.W = OW;
    p.M = (long long)d->n * OH * OW;
    p.up_h = OH / 2; p.up_w = OW / 2;
    choose_patch(OH, OW, p.TH, p.TW);
    p.tiles_h = (OH + p.TH - 1) / p.TH;
    p.tiles_w = (OW + p.TW - 1) / p.TW;
    p.num_m_tiles = d->n * p.tiles_h * p.tiles_w;
    const uint64_t C = (uint64_t)d->cin, W = (uint64_t)d->width, H = (uint64_t)d->h;
    uint64_t dims[5] = {2 * C, W / 2, 2, H / 2, (uint64_t)d->n};
    uint64_t str[4] = {2 * C * 2, W * C * 2, 2 * W * C * 2, H * W * C * 2};
    uint32_t box[5] = {64, (uint32_t)p.TW, 1, (uint32_t)p.TH, 1};
    if (!encode_map(&tmA, d->x, 5, dims, str, box)) return ODTK_E_CUDA;
  } else if (d->ksize == 1) {
    p.mode = 0;
    p.num_m_tiles = (int)((p.M + 127) / 128);
    uint64_t dims[2] = {(uint64_t)d->cin, (uint64_t)p.M};
    uint64_t str[1] = {(uint64_t)d->cin * 2};
    uint32_t box[2] = {64, 128};
    if (!encode_map(&tmA, d->x, 2, dims, str, box)) return ODTK_E_CUDA;
  } else {
    p.mode = 1;
    if (d->tile_tab) {   // atlas tile tables list 8 x 16 pixel tiles
      p.TH = 8; p.TW = 16;
      p.tile_tab = (const int4 *)d->tile_tab; p.tab_tiles = d->tab_tiles;
    } else {
      choose_patch(d->h, d->width, p.TH, p.TW);
    }
    p.tiles_h = (d->h + p.TH - 1) / p.TH;
    p.tiles_w = (d->width + p.TW - 1) / p.TW;
    p.num_m_tiles = d->tile_tab ? d->n * d->tab_tiles : d->n * p.tiles_h * p.tiles_w;
    const uint64_t C = (uint64_t)d->cin, W = (uint64_t)d->width, H = (uint64_t)d->h;
    uint64_t dims[4] = {C, W, H, (uint64_t)d->n};
    uint64_t str[3] = {C * 2, xW * C * 2, xH * xW * C * 2};
    uint32_t box[4] = {64, (uint32_t)p.TW, (uint32_t)p.TH, 1};
    if (!encode_map(&tmA, d->x, 4, dims, str, box)) return ODTK_E_CUDA;
  }
  p.oH = d->y_rows > 0 ? d->y_rows : p.H;
  p.oR = d->y_row_off > 0 ? d->y_row_off : 0;
  p.oW = d->y_width > 0 ? d->y_width : p.W;
  if ((long long)d->n * p.oH * p.oW >= (1ll << 31) || p.oR + p.H > p.oH || p.W > p.oW) return ODTK_E_INVALID;
  // N tile: 64 or 128 output channels.  128 halves the A-operand traffic; 64 when Cout is narrow, for grouped convs (one
  // 64-channel chunk per tile), or when 128-wide tiles would leave SMs idle.
  int BN = (groups > 1 || d->cout <= 64) ? 64 : 128;
  if (BN == 128 && (long long)p.num_m_tiles * ((d->cout + 127) / 128) < sms) BN = 64;
  p.num_n_tiles = (d->cout + BN - 1) / BN;
  set_stages(p, BN);
  CUtensorMap tmB, tmA2, tmB2;
  const uint64_t K = (uint64_t)p.taps * (groups > 1 ? 64 : d->cin);
  {
    uint64_t dims[2] = {K, (uint64_t)d->cout};
    uint64_t str[1] = {K * 2};
    uint32_t box[2] = {64, (uint32_t)BN};
    if (!encode_map(&tmB, d->w, 2, dims, str, box)) return ODTK_E_CUDA;
  }
  tmA2 = tmA; tmB2 = tmB;
  if (x2) {
    p.kblocks2 = c2in / 64;
    uint64_t dims[2] = {(uint64_t)c2in, (uint64_t)p.M}, str[1] = {(uint64_t)c2in * 2};
    uint32_t box[2] = {64, 128};
    uint64_t dimsW[2] = {(uint64_t)c2in, (uint64_t)d->cout}, strW[1] = {(uint64_t)c2in * 2};
    uint32_t boxW[2] = {64, (uint32_t)BN};
    if (!encode_map(&tmA2, x2, 2, dims, str, box) || !encode_map(&tmB2, w2, 2, dimsW, strW, boxW)) return ODTK_E_CUDA;
  }
  return launch(p, BN, tmA, tmB, tmA2, tmB2, stream);
}

// bias operand: [cout, 64] fp16 with (hi, lo, 0, ...): hi + lo == bias to 2^-22 relative
__global__ void pack_bias_kernel(const float *bias, __half *out, int cout) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < cout * 64; i += gridDim.x * blockDim.x) {
    const int c = i >> 6, k = i & 63;
    float v = 0.0f;
    if (k < 2) {
      const float b = bias[c];
      const float hi = __half2float(__float2half_rn(b));
      v = (k == 0) ? hi : b - hi;
    }
    out[i] = __float2half_rn(v);
  }
}

}  // namespace

extern "C" int odtk_conv2d(const odtk_conv_t *d, odtk_stream_t stream_) {
  return conv_run(d, nullptr, nullptr, 0, (cudaStream_t)stream_);
}

// ResNet stem: 7x7 stride-2 pad-3 convolution of the RGB image, im2col-free.  `xp` is the image
// zero-padded to NHWC4 [n, h+6, w+8, 4] fp16 by odtk_pad_input.  For filter row r the A operand of
// output pixels (oh, ow..) is the 8-pixel x 4-channel window starting at padded pixel (2*oh + r, 2*ow):
// 64 contiguous bytes, consecutive output pixels 16 bytes apart -- an OVERLAPPING-window 5-D tensor map
// {32 elements, OW (16 B), 7 rows (one padded row), OH (two padded rows), N}.  K = 7 blocks of 32
// (SWIZZLE_64B), weights packed [cout, 7*32] with k = r*32 + s*4 + c (zero for s = 7 or c = 3).
extern "C" int odtk_stem_conv(const void *xp, const void *w, const float *bias, void *y, int n, int h, int width,
                              int cout, int relu, odtk_stream_t stream_) {
  if (!xp || !w || !y || n <= 0 || h <= 0 || width <= 0) return ODTK_E_INVALID;
  if ((h & 1) || (width & 1) || cout % 16 || cout > 128) return ODTK_E_UNSUPPORTED;
  if (((uintptr_t)xp | (uintptr_t)w | (uintptr_t)y) & 15) return ODTK_E_INVALID;
  cudaStream_t stream = (cudaStream_t)stream_;
  if (!device_ready()) return ODTK_E_CUDA;
  const int OH = h / 2, OW = width / 2, HP = h + 6, WP = width + 8;
  if ((long long)n * OH * OW >= (1ll << 31)) return ODTK_E_UNSUPPORTED;
  ConvParams p;
  memset(&p, 0, sizeof p);
  p.mode = 2;
  p.N = n; p.H = OH; p.W = OW; p.Cin = 4; p.Cout = cout;
  p.kw = 1; p.taps = 7; p.pad = 0; p.kblocks_per_tap = 1;
  p.row_bytes = 64;
  p.M = (long long)n * OH * OW;
  const int BN = cout <= 64 ? 64 : 128;
  p.num_n_tiles = 1;
  set_stages(p, BN);
  p.bias = bias; p.out = y; p.relu = relu; p.out_mode = ODTK_OUT_NHWC_F16; p.ldy = cout; p.ldr = cout;
  p.oH = OH; p.oR = 0; p.oW = OW;
  choose_patch(OH, OW, p.TH, p.TW);
  p.tiles_h = (OH + p.TH - 1) / p.TH;
  p.tiles_w = (OW + p.TW - 1) / p.TW;
  p.num_m_tiles = n * p.tiles_h * p.tiles_w;
  CUtensorMap tmA, tmB;
  {
    uint64_t dims[5] = {32, (uint64_t)OW, 7, (uint64_t)OH, (uint64_t)n};
    uint64_t str[4] = {16, (uint64_t)WP * 8, (uint64_t)WP * 16, (uint64_t)HP * WP * 8};
    uint32_t box[5] = {32, (uint32_t)p.TW, 1, (uint32_t)p.TH, 1};
    if (!encode_map(&tmA, xp, 5, dims, str, box, CU_TENSOR_MAP_SWIZZLE_64B)) return ODTK_E_UNSUPPORTED;
  }
  {
    uint64_t dims[2] = {224, (uint64_t)cout};
    uint64_t str[1] = {224 * 2};
    uint32_t box[2] = {32, (uint32_t)BN};
    if (!encode_map(&tmB, w, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_64B)) return ODTK_E_CUDA;
  }
  return launch(p, BN, tmA, tmB, tmA, tmB, stream);
}

// Pack a fp32 bias vector into the [cout, 64] fp16 (hi, lo) layout (see odtk_conv_t.bias_op).
extern "C" int odtk_conv_pack_bias(const float *bias, void *out, int cout, odtk_stream_t stream_) {
  if (!bias || !out || cout <= 0) return ODTK_E_INVALID;
  pack_bias_kernel<<<(cout * 64 + 255) / 256, 256, 0, (cudaStream_t)stream_>>>(bias, (__half *)out, cout);
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

// What the last odtk_conv2d / odtk_stem_conv call of THIS host thread launched (tests assert which kernel variant ran).
extern "C" int odtk_conv_last_plan(odtk_conv_plan_t *out) {
  if (!out) return ODTK_E_INVALID;
  *out = g_last_plan;
  return ODTK_OK;
}
extern "C" int odtk_conv_map_cache_stats(long long *hits, long long *misses) {
  std::lock_guard<std::mutex> lk(g_map_mu);
  if (hits) *hits = g_map_hits;
  if (misses) *misses = g_map_misses;
  return ODTK_OK;
}
