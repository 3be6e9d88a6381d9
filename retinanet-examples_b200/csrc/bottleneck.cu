// bottleneck.cu -- the tail of a stride-1 ResNet bottleneck block in ONE kernel on the Hopper tensor cores (sm_90a):
//
//     mid = relu(conv3x3(x, W2) + b2)                       GEMM1: 9 * C1/64 K blocks, A = shifted TMA boxes of x
//     y   = act(mid * W3^T + b3 + identity)                  GEMM2: per 128-channel output tile, A = mid from shared memory
//     z   = relu(y * Wn^T + bn)          (optional)          GEMM3: the next block's conv1, A = y from shared memory
//
// identity is the residual tensor, or -- first block of layer1 -- xproj * Wproj^T, one more K block of GEMM2's
// accumulator.  `mid` never leaves the SM: GEMM1's epilogue rounds it to fp16 (exactly what a separate 3x3 launch would
// store) and writes it into shared memory in the 128-byte-swizzled K-major layout of a wgmma A operand; GEMM2 reads it
// from there.  GEMM3 reads the fp16 block output the same way instead of re-loading it from HBM.
//
//   warpgroup 0     TMA producer (one thread): x boxes + W2 blocks, then W3 (+ xproj / Wproj) blocks per output tile,
//                   then Wn blocks, through one ring of full / empty mbarrier stages -- in the order the consumers use them.
//   warpgroups 1-2  64 pixels of the 128-pixel tile each: wgmma.mma_async, fp32 accumulators in registers, epilogues.
//                   Every A row a warpgroup reads from shared memory it wrote itself, so a 128-thread named barrier
//                   (plus fence.proxy.async: generic-proxy stores -> async-proxy wgmma reads) is the only hand-over.
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
constexpr int kStageBytes = 2 * 16384;   // A: 128 rows x 128 B; B: up to 128 rows x 128 B
constexpr int kMaxStages = 6;
constexpr int kSmemLimit = 227 * 1024;
constexpr int kChunk = 16384;            // one 64-channel chunk of a [128 pixels][C] operand in shared memory

struct BtParams {
  int N, H, W, C2, TH, TW, tiles_h, tiles_w, total_tiles, nstages, relu, proj;
  int mid_off, ysm_off;                  // byte offsets of the mid / block-output operands in shared memory
  const float *b2, *b3, *bn;
  const __half *residual;
  __half *y, *z;
};

struct Ring {
  int stage = 0;
  uint32_t phase = 0;
  int n;
  __device__ void next() { if (++stage == n) { stage = 0; phase ^= 1u; } }
};

__device__ __forceinline__ void named_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void sts32(uint32_t saddr, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(saddr), "r"(v) : "memory"); }
// (row, col) of a [128][64 k] 128B-swizzled K-major chunk: the 16-byte unit (col / 8) is XOR-ed with row % 8
__device__ __forceinline__ uint32_t swz_off(int row, int col) {
  return (uint32_t)(row * 128 + ((((col & 63) >> 3) ^ (row & 7)) << 4) + (col & 7) * 2);
}
__device__ __forceinline__ uint32_t h2u(__half2 h) { return *reinterpret_cast<uint32_t *>(&h); }

template <int N>
__device__ __forceinline__ void mma_block(float (&acc)[N / 2], uint64_t da, uint64_t db, bool first) {
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 4; k++) Wgmma<N>::mma(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (first && k == 0) ? 0 : 1);
  wgmma_commit();
}

template <int C1, int N3>
__global__ void __launch_bounds__(kThreads, 1)
bottleneck_tail_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW2,
                       const __grid_constant__ CUtensorMap tmW3, const __grid_constant__ CUtensorMap tmXp,
                       const __grid_constant__ CUtensorMap tmWp, const __grid_constant__ CUtensorMap tmWn,
                       const __grid_constant__ BtParams p) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char *smem = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t *full = reinterpret_cast<uint64_t *>(smem + p.ysm_off + (N3 ? (p.C2 / 64) * kChunk : 0));
  uint64_t *empty = full + kMaxStages;
  const int wg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0), tid = threadIdx.x & 127;
  if (threadIdx.x == 0) {
    for (int s = 0; s < p.nstages; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8 /* one per consumer warp */); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  grid_dep_launch_dependents();
  grid_dep_wait();
  constexpr int KC1 = C1 / 64;
  const int n2tiles = p.C2 / 128, per_img = p.tiles_h * p.tiles_w;
  auto origin = [&](int tile, int &img, int &h0, int &w0) {
    img = tile / per_img;
    const int r = tile - img * per_img;
    h0 = (r / p.tiles_w) * p.TH;
    w0 = (r % p.tiles_w) * p.TW;
  };

  if (wg == 0) {
    // ===================================== TMA producer =====================================
    if (tid != 0) return;
    Ring ring;
    ring.n = p.nstages;
    const uint32_t a_bytes = (uint32_t)(p.TH * p.TW * 128);
    auto slot = [&](uint32_t bytes) -> unsigned char * {
      mbar_wait(&empty[ring.stage], ring.phase ^ 1u);
      mbar_arrive_expect_tx(&full[ring.stage], bytes);
      return smem + ring.stage * kStageBytes;
    };
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      int img, h0, w0;
      origin(tile, img, h0, w0);
      for (int kb = 0; kb < KC1; kb++)
        for (int tap = 0; tap < 9; tap++) {
          unsigned char *s = slot(a_bytes + C1 * 128);
          tma_load_4d(s, &tmX, &full[ring.stage], kb * 64, w0 + tap % 3 - 1, h0 + tap / 3 - 1, img);
          tma_load_2d(s + 16384, &tmW2, &full[ring.stage], (tap * KC1 + kb) * 64, 0);
          ring.next();
        }
      for (int n2 = 0; n2 < n2tiles; n2++) {
        for (int kb = 0; kb < KC1; kb++) {
          unsigned char *s = slot(128 * 128);
          tma_load_2d(s + 16384, &tmW3, &full[ring.stage], kb * 64, n2 * 128);
          ring.next();
        }
        if (p.proj) {
          unsigned char *s = slot(a_bytes + 128 * 128);
          tma_load_4d(s, &tmXp, &full[ring.stage], 0, w0, h0, img);
          tma_load_2d(s + 16384, &tmWp, &full[ring.stage], 0, n2 * 128);
          ring.next();
        }
      }
      if (N3)
        for (int kb = 0; kb < p.C2 / 64; kb++) {
          unsigned char *s = slot(N3 * 128);
          tma_load_2d(s + 16384, &tmWn, &full[ring.stage], kb * 64, 0);
          ring.next();
        }
    }
    return;
  }

  // ===================================== MMA + epilogues ====================================
  const int cw = wg - 1, warp = tid >> 5, lane = tid & 31, q = lane & 3;
  const uint32_t mid_s = smem_u32(smem + p.mid_off), ysm_s = smem_u32(smem + p.ysm_off);
  const uint32_t rows = (uint32_t)(cw * 64 * 128);   // this warpgroup's 64 rows inside a [128][64] operand chunk
  Ring ring;
  ring.n = p.nstages;
  int prev = -1;
  // one K block: wait for its stage, issue its 4 MMAs, and release the PREVIOUS block's stage once at most this
  // block's MMAs are in flight
  auto consumed = [&]() {
    wgmma_wait<1>();
    if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
    prev = ring.stage;
    ring.next();
  };
  auto drain = [&]() {
    wgmma_wait<0>();
    if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
    prev = -1;
  };
  float acc1[C1 / 2];
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    int img, h0, w0;
    origin(tile, img, h0, w0);
    // ---- GEMM1: the 3x3 ----
    for (int kb = 0; kb < 9 * KC1; kb++) {
      mbar_wait(&full[ring.stage], ring.phase);
      const uint32_t sa = smem_u32(smem + ring.stage * kStageBytes);
      mma_block<C1>(acc1, wgmma_desc(sa + rows, 128), wgmma_desc(sa + 16384, 128), kb == 0);
      consumed();
    }
    drain();
    // pixel of each of this thread's two accumulator rows
    int prow[2];
    long long pix[2];
    bool valid[2];
#pragma unroll
    for (int i = 0; i < 2; i++) {
      prow[i] = cw * 64 + warp * 16 + (lane >> 2) + 8 * i;
      const int dh = prow[i] / p.TW, dw = prow[i] - dh * p.TW, h = h0 + dh, w = w0 + dw;
      valid[i] = prow[i] < p.TH * p.TW && h < p.H && w < p.W;
      pix[i] = ((long long)img * p.H + h) * p.W + w;
    }
    named_sync(1 + cw);   // the previous tile's GEMM2 / GEMM3 of every warp of this warpgroup read `mid` / `ysm`
    // ---- epilogue 1: mid = fp16(relu(acc1 + b2)) -> the A operand of GEMM2 ----
#pragma unroll
    for (int j = 0; j < C1 / 8; j++) {
      const int col = 8 * j + 2 * q;
      const float b0 = p.b2 ? __ldg(p.b2 + col) : 0.0f, b1 = p.b2 ? __ldg(p.b2 + col + 1) : 0.0f;
#pragma unroll
      for (int i = 0; i < 2; i++) {
        const __half2 v = __hmax2(__floats2half2_rn(acc1[4 * j + 2 * i] + b0, acc1[4 * j + 2 * i + 1] + b1), __float2half2_rn(0.0f));
        sts32(mid_s + (uint32_t)((col >> 6) * kChunk) + swz_off(prow[i], col), h2u(v));
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    named_sync(1 + cw);
    // ---- GEMM2 per 128-channel output tile, + identity, epilogue 2 ----
    for (int n2 = 0; n2 < n2tiles; n2++) {
      float acc2[64];
      for (int kb = 0; kb < KC1; kb++) {
        mbar_wait(&full[ring.stage], ring.phase);
        const uint32_t sa = smem_u32(smem + ring.stage * kStageBytes);
        mma_block<128>(acc2, wgmma_desc(mid_s + (uint32_t)(kb * kChunk) + rows, 128), wgmma_desc(sa + 16384, 128), kb == 0);
        consumed();
      }
      if (p.proj) {
        mbar_wait(&full[ring.stage], ring.phase);
        const uint32_t sa = smem_u32(smem + ring.stage * kStageBytes);
        mma_block<128>(acc2, wgmma_desc(sa + rows, 128), wgmma_desc(sa + 16384, 128), false);
        consumed();
      }
      drain();
#pragma unroll
      for (int j = 0; j < 16; j++) {
        const int col = n2 * 128 + 8 * j + 2 * q;
        const float b0 = p.b3 ? __ldg(p.b3 + col) : 0.0f, b1 = p.b3 ? __ldg(p.b3 + col + 1) : 0.0f;
#pragma unroll
        for (int i = 0; i < 2; i++) {
          float v0 = acc2[4 * j + 2 * i] + b0, v1 = acc2[4 * j + 2 * i + 1] + b1;
          if (!p.proj && valid[i]) {
            const float2 r = __half22float2(*reinterpret_cast<const __half2 *>(p.residual + pix[i] * p.C2 + col));
            v0 += r.x; v1 += r.y;
          }
          __half2 y = __floats2half2_rn(v0, v1);
          if (p.relu) y = __hmax2(y, __float2half2_rn(0.0f));
          if (valid[i]) *reinterpret_cast<__half2 *>(p.y + pix[i] * p.C2 + col) = y;
          if (N3) sts32(ysm_s + (uint32_t)((col >> 6) * kChunk) + swz_off(prow[i], col), h2u(y));
        }
      }
    }
    if constexpr (N3 > 0) {
      // ---- GEMM3: the next block's conv1 from the fp16 block output ----
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      named_sync(1 + cw);
      float acc3[N3 / 2];
      for (int kb = 0; kb < p.C2 / 64; kb++) {
        mbar_wait(&full[ring.stage], ring.phase);
        const uint32_t sa = smem_u32(smem + ring.stage * kStageBytes);
        mma_block<N3>(acc3, wgmma_desc(ysm_s + (uint32_t)(kb * kChunk) + rows, 128), wgmma_desc(sa + 16384, 128), kb == 0);
        consumed();
      }
      drain();
#pragma unroll
      for (int j = 0; j < N3 / 8; j++) {
        const int col = 8 * j + 2 * q;
        const float b0 = p.bn ? __ldg(p.bn + col) : 0.0f, b1 = p.bn ? __ldg(p.bn + col + 1) : 0.0f;
#pragma unroll
        for (int i = 0; i < 2; i++)
          if (valid[i])
            *reinterpret_cast<__half2 *>(p.z + pix[i] * N3 + col) =
                __hmax2(__floats2half2_rn(acc3[4 * j + 2 * i] + b0, acc3[4 * j + 2 * i + 1] + b1), __float2half2_rn(0.0f));
      }
    }
  }
}

template <int C1, int N3>
int launch(int grid, int smem_bytes, cudaStream_t stream, const CUtensorMap *tm, const BtParams &p) {
  static std::mutex mu;
  static bool ready[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return ODTK_E_CUDA;
  {
    std::lock_guard<std::mutex> lk(mu);
    if (!ready[dev]) {
      if (cudaFuncSetAttribute(bottleneck_tail_kernel<C1, N3>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit) != cudaSuccess)
        return ODTK_E_CUDA;
      ready[dev] = true;
    }
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = (size_t)smem_bytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = odtk_pdl_on() ? 1 : 0;
  {
    OdtkProfScope prof(ODTK_PROF_CONV, stream);
    cudaLaunchKernelEx(&cfg, bottleneck_tail_kernel<C1, N3>, tm[0], tm[1], tm[2], tm[3], tm[4], tm[5], p);
  }
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

}  // namespace

extern "C" int odtk_bottleneck_tail(const odtk_bneck_t *d, odtk_stream_t stream_) {
  if (!d || !d->x || !d->w2 || !d->w3 || !d->y) return ODTK_E_INVALID;
  const bool proj = d->xproj != nullptr;
  if (proj ? (!d->wproj || d->c1 != 64) : !d->residual) return ODTK_E_INVALID;
  const int n3 = d->w_next ? d->c_next : 0;
  if (n3 && (proj || d->c1 != 64 || !d->z || (n3 != 64 && n3 != 128) || (((uintptr_t)d->w_next | (uintptr_t)d->z) & 15))) return ODTK_E_UNSUPPORTED;
  if (d->n <= 0 || d->h <= 0 || d->width <= 0) return ODTK_E_INVALID;
  if ((d->c1 != 64 && d->c1 != 128) || d->c2 % 128 != 0 || d->c2 <= 0 || d->c2 > 512) return ODTK_E_UNSUPPORTED;
  if (((uintptr_t)d->x | (uintptr_t)d->w2 | (uintptr_t)d->w3 | (uintptr_t)d->residual | (uintptr_t)d->y | (uintptr_t)d->xproj | (uintptr_t)d->wproj) & 15) return ODTK_E_INVALID;
  if ((long long)d->n * d->h * d->width >= (1ll << 31)) return ODTK_E_UNSUPPORTED;
  BtParams p;
  memset(&p, 0, sizeof p);
  p.N = d->n; p.H = d->h; p.W = d->width; p.C2 = d->c2;
  choose_patch(d->h, d->width, p.TH, p.TW);
  p.tiles_h = (d->h + p.TH - 1) / p.TH;
  p.tiles_w = (d->width + p.TW - 1) / p.TW;
  const long long total = (long long)d->n * p.tiles_h * p.tiles_w;
  if (total >= (1ll << 31)) return ODTK_E_UNSUPPORTED;
  p.total_tiles = (int)total;
  p.relu = d->relu; p.proj = proj;
  p.b2 = d->b2; p.b3 = d->b3; p.bn = d->b_next;
  p.residual = (const __half *)d->residual; p.y = (__half *)d->y; p.z = (__half *)d->z;
  // shared memory: stages | mid [128][C1] | block output [128][C2] (GEMM3 only) | barriers
  const int mid_bytes = (d->c1 / 64) * kChunk, ysm_bytes = n3 ? (d->c2 / 64) * kChunk : 0;
  int nst = (kSmemLimit - 1024 - 256 - mid_bytes - ysm_bytes) / kStageBytes;
  if (nst > kMaxStages) nst = kMaxStages;
  if (nst < 2) return ODTK_E_UNSUPPORTED;
  p.nstages = nst;
  p.mid_off = nst * kStageBytes;
  p.ysm_off = p.mid_off + mid_bytes;
  const int smem_bytes = 1024 + p.ysm_off + ysm_bytes + 2 * kMaxStages * 8;
  const uint64_t C1 = (uint64_t)d->c1, C2 = (uint64_t)d->c2, H = (uint64_t)d->h, W = (uint64_t)d->width, N = (uint64_t)d->n;
  CUtensorMap tm[6];
  {
    uint64_t dims[4] = {C1, W, H, N}, str[3] = {C1 * 2, W * C1 * 2, H * W * C1 * 2};
    uint32_t box[4] = {64, (uint32_t)p.TW, (uint32_t)p.TH, 1};
    if (!encode_map(&tm[0], d->x, 4, dims, str, box)) return ODTK_E_CUDA;
  }
  {
    uint64_t dims[2] = {9 * C1, C1}, str[1] = {9 * C1 * 2};
    uint32_t box[2] = {64, (uint32_t)d->c1};
    if (!encode_map(&tm[1], d->w2, 2, dims, str, box)) return ODTK_E_CUDA;
  }
  {
    uint64_t dims[2] = {C1, C2}, str[1] = {C1 * 2};
    uint32_t box[2] = {64, 128};
    if (!encode_map(&tm[2], d->w3, 2, dims, str, box)) return ODTK_E_CUDA;
  }
  tm[3] = tm[0]; tm[4] = tm[2]; tm[5] = tm[2];
  if (proj) {   // identity = xproj [n, h, width, 64] x wproj [c2, 64]^T: one more K block per output tile
    uint64_t dims[4] = {64, W, H, N}, str[3] = {64 * 2, W * 64 * 2, H * W * 64 * 2};
    uint32_t box[4] = {64, (uint32_t)p.TW, (uint32_t)p.TH, 1};
    uint64_t dimsW[2] = {64, C2}, strW[1] = {64 * 2};
    uint32_t boxW[2] = {64, 128};
    if (!encode_map(&tm[3], d->xproj, 4, dims, str, box) || !encode_map(&tm[4], d->wproj, 2, dimsW, strW, boxW)) return ODTK_E_CUDA;
  }
  if (n3) {
    uint64_t dims[2] = {C2, (uint64_t)n3}, str[1] = {C2 * 2};
    uint32_t box[2] = {64, (uint32_t)n3};
    if (!encode_map(&tm[5], d->w_next, 2, dims, str, box)) return ODTK_E_CUDA;
  }
  const int sms = odtk_sm_count();
  const int grid = p.total_tiles < sms ? p.total_tiles : sms;
  cudaStream_t stream = (cudaStream_t)stream_;
  if (d->c1 == 128) return launch<128, 0>(grid, smem_bytes, stream, tm, p);
  if (n3 == 64) return launch<64, 64>(grid, smem_bytes, stream, tm, p);
  if (n3 == 128) return launch<64, 128>(grid, smem_bytes, stream, tm, p);
  return launch<64, 0>(grid, smem_bytes, stream, tm, p);
}
