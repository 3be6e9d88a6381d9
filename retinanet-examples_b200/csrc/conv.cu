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
//   warpgroups 1-2  MMA + epilogue, 64 accumulator rows (output pixels) each: wgmma.mma_async m64nNk16 (N = BN = 64,
//                   128 or, fp16 forward only, 256), fp32 accumulation in registers; the stage is released as soon as the next K block's
//                   MMAs are in flight.  The epilogue works on the registers: + bias, + residual / FPN nearest-
//                   upsample, ReLU / ReLU6, fp16 NHWC store (fp16: stmatrix into shared memory, then a TMA store per
//                   64 columns; a mode-0 residual arrives through the ring) -- or, for the last convolution of a head, (sigmoid +)
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
// INT8 (odtk_conv2d_s8 / _ex): the same kernel instantiated on s8 operands -- 128-channel K blocks, wgmma m64nNk32 with s32
// accumulators, a dequantising epilogue (+ s8 residual / upsample addends) -- in modes 0, 1 (incl. s2) and 3.
// FP32 (odtk_conv2d_f32): instantiated on fp32 operands with split-TF32 ("3xTF32") products -- 32-channel K blocks (one
// 128-byte swizzle row), weights as two tf32-valued halves (w_hi, w_lo) that both stream through every stage; each consumer
// warpgroup splits its own 64 A rows in shared memory (hi rounded in place, lo into a side buffer) and issues three wgmma
// m64nNk8 tf32 MMAs per k8 step, a_hi*b_lo + a_lo*b_hi + a_hi*b_hi, into fp32 accumulators; fp32 NHWC epilogue (+ fp32
// residual / upsample addends) -- in modes 0, 1 (incl. s2 and tile tables), 2 (stem over an NHWC4 fp32 image) and 3.
#include <cuda.h>
#include <cuda_fp16.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>
#include <type_traits>
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
// FP32 instances: after the stages, the A_lo side buffers, 2 per consumer warpgroup (64 rows x 128 B each, double-buffered:
// the previous K block's MMAs may still read one while the next block is split into the other)
constexpr int kLoBytes = 64 * 128;
constexpr int kSplitBytes = 2 * 2 * kLoBytes;
constexpr int kSmemBytesF32 = kPipeBytes + kSplitBytes + 1024 + 256;
static_assert(kSmemBytesF32 <= 227 * 1024, "fp32 instance exceeds the opt-in shared memory");
// fp16 forward instances: after the stages, the two staging chunks of the TMA-store epilogue, [128 rows][64 channels] fp16
// each in the 128-byte swizzle of a TMA box (one is filled while the bulk store of the other still reads it)
constexpr int kStoreChunk = 128 * 128;
constexpr int kSmemBytesF16 = kPipeBytes + 2 * kStoreChunk + 1024 + 256;
static_assert(kSmemBytesF16 <= 227 * 1024, "fp16 instance exceeds the opt-in shared memory");

// operand types of conv_gemm_kernel; kOpF16Mask: fp16 with the ReLU-derivative mask of the input gradient (odtk_conv2d_dgrad)
enum ConvOp { kOpF16 = 0, kOpS8 = 1, kOpTF32x3 = 2, kOpF16Mask = 3 };
constexpr int smem_bytes(int op) { return op == kOpTF32x3 ? kSmemBytesF32 : op == kOpF16 ? kSmemBytesF16 : kSmemBytes; }

// round to the nearest tf32 value, ties away from zero (low 13 bits cleared)
__device__ __forceinline__ float tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

struct Barriers {
  uint64_t full[kMaxStages];
  uint64_t empty[kMaxStages];
};
static_assert(sizeof(Barriers) <= 256, "barrier block too small");

// ---------------------------------------------------------------------------------- kernel
// OP kOpS8: int8 operands (odtk_conv2d_s8).  A K block is then one 128-byte swizzle row of 128 channels instead of 64, the
// MMAs are the integer m64nNk32 form with exact s32 accumulators, and the epilogue dequantises with fmaf(acc, alpha, bias).
// OP kOpTF32x3: fp32 operands (odtk_conv2d_f32).  A K block is one 128-byte row of 32 channels; a stage holds A, then
// B_hi and B_lo (tmB / tmB2); the MMAs are three m64nNk8 tf32 products per k8 step (see the file comment).
// tmY (fp16 forward with p.tma_store): the NHWC output, written by TMA stores from shared memory (host: out_map); tmR (with
// p.res_tma): the mode-0 residual [M, ldr], loaded by the producer into the ring after each tile's K blocks.  They come
// after p so that the other instances keep their parameter offsets.
template <int BN, int OP>
__global__ void __launch_bounds__(kThreads, 1)
conv_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2,
                 const __grid_constant__ ConvParams p, const __grid_constant__ CUtensorMap tmY,
                 const __grid_constant__ CUtensorMap tmR) {
  constexpr bool S8 = OP == kOpS8, F32 = OP == kOpTF32x3;
  // residual boxes ([128 rows][64 channels], 16 KB) per ring stage: stages hold 24, 32 or 48 KB at BN 64, 128, 256
  constexpr int kResPerStage = BN == 64 ? 1 : 2;
  constexpr int BR = F32 ? 2 * BN : BN;   // B rows per stage: fp32 carries w_hi and w_lo
  extern __shared__ unsigned char smem_raw[];
  unsigned char *smem = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  Barriers *bars = reinterpret_cast<Barriers *>(smem + kPipeBytes + (F32 ? kSplitBytes : OP == kOpF16 ? 2 * kStoreChunk : 0));
  const int kStages = p.nstages, rb = p.row_bytes;
  const int stage_bytes = (128 + BR) * rb;
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
    // BN 256: the 128 fp32 accumulators per consumer thread need more than the 168 registers of a 384-thread CTA; the
    // producer warpgroup hands its registers back (40 each) and the consumers take 232: 232 * 256 + 40 * 128 <= 64 K.
    if constexpr (BN == 256) asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (tid != 0) return;
    const uint32_t a_bytes = (uint32_t)((p.mode == 0 ? 128 : p.TH * p.TW) * rb), b_bytes = (uint32_t)(BR * rb);
    const int kelems = S8 ? rb : F32 ? rb >> 2 : rb >> 1;   // K elements per block: 64 (SW128) or 32 (SW64); s8: 128; fp32: 32
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      int m_tile, n_tile, img, h0, w0, hlim, wlim;
      tile_origin(tile, m_tile, n_tile, img, h0, w0, hlim, wlim);
      const int n0 = n_tile * BN;
      // K order: 64-channel (s8: 128-channel, fp32: 32-channel) chunk outer, tap inner
      for (int kb = 0; kb < p.kblocks_per_tap; kb++) {
        const int kch = p.grouped ? n0 : kb * (S8 ? 128 : F32 ? 32 : 64);   // input-channel coordinate: grouped convs read their own chunk only
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
          if constexpr (F32) tma_load_2d(sb + BN * rb, &tmB2, &bars->full[stage], (tap * p.kblocks_per_tap + kb) * kelems, n0);
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
      if constexpr (OP == kOpF16) {
        if (p.res_tma) {   // the tile's residual, while its MMAs still run; rows past M and columns past Cout read as 0
          for (int c = 0; c < BN / 64; c += kResPerStage) {
            mbar_wait(&bars->empty[stage], phase ^ 1u);
            unsigned char *sr = smem + stage * stage_bytes;
            mbar_arrive_expect_tx(&bars->full[stage], (uint32_t)(kResPerStage * kStoreChunk));
            for (int k = 0; k < kResPerStage; k++)
              tma_load_2d(sr + k * kStoreChunk, &tmR, &bars->full[stage], n0 + 64 * (c + k), m_tile * 128);
            if (++stage == kStages) { stage = 0; phase ^= 1u; }
          }
        }
      }
    }
    return;
  }

  // ===================================== MMA + epilogue ======================================
  if constexpr (BN == 256) asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  const int cw = wg - 1, warp = tid >> 5, lane = tid & 31;
  const int q = lane & 3;
  const int hw = p.H * p.W, patch = p.TH * p.TW;
  typename std::conditional<S8, int, float>::type acc[BN / 2];
  int stage = 0;
  uint32_t phase = 0;
  int sbuf = 0;   // TMA-store epilogue: the staging chunk the next 64 columns go to
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
      if constexpr (F32) {
        // split this warpgroup's 64 A rows: hi = rna_tf32(a) in place, lo = rna_tf32(a - hi) (a - hi is exact) into the side
        // buffer of this K block's parity.  Elementwise, so the swizzle does not matter: 16 bytes per thread and pass.
        unsigned char *a_own = smem + stage * stage_bytes + cw * 64 * 128;
        unsigned char *a_lo = smem + kPipeBytes + (2 * cw + (kb & 1)) * kLoBytes;
#pragma unroll
        for (int i = 0; i < kLoBytes / (128 * 16); i++) {
          const int off = (tid + 128 * i) * 16;
          float4 v = *reinterpret_cast<const float4 *>(a_own + off), lo;
          float *vv = reinterpret_cast<float *>(&v), *ll = reinterpret_cast<float *>(&lo);
#pragma unroll
          for (int e = 0; e < 4; e++) {
            const float hi = tf32_rna(vv[e]);
            ll[e] = tf32_rna(vv[e] - hi);
            vv[e] = hi;
          }
          *reinterpret_cast<float4 *>(a_own + off) = v;
          *reinterpret_cast<float4 *>(a_lo + off) = lo;
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> async-proxy wgmma reads
        asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory");
        const uint64_t dlo = wgmma_desc(smem_u32(a_lo), 128), dbl = db + (uint64_t)((BN * 128) >> 4);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; k++) {   // small terms first
          WgmmaTF32<BN>::mma(acc, da + (uint64_t)(2 * k), dbl + (uint64_t)(2 * k), (kb | k) ? 1 : 0);
          WgmmaTF32<BN>::mma(acc, dlo + (uint64_t)(2 * k), db + (uint64_t)(2 * k), 1);
          WgmmaTF32<BN>::mma(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), 1);
        }
      } else {
        wgmma_fence();
        if constexpr (S8) {
#pragma unroll
          for (int k = 0; k < 4; k++) WgmmaS8<BN>::mma(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (kb | k) ? 1 : 0);
        } else if (brb == 128) {
#pragma unroll
          for (int k = 0; k < 4; k++) Wgmma<BN>::mma(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (kb | k) ? 1 : 0);
        } else {
#pragma unroll
          for (int k = 0; k < 2; k++) Wgmma<BN>::mma(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (kb | k) ? 1 : 0);
        }
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
    // fp16: + bias goes into the accumulators first, all of the tile's bias loads ahead of any store.  Every global store
    // below may alias a later load as far as the compiler knows, so a load left behind a store waits for it.
    constexpr bool F16 = OP == kOpF16 || OP == kOpF16Mask;
    if constexpr (F16) {
      if (p.bias) {
#pragma unroll
        for (int j = 0; j < BN / 8; j++)
#pragma unroll
          for (int k = 0; k < 2; k++) {
            const int col = n0 + 8 * j + 2 * q + k;
            if (col >= p.Cout) continue;
            const float b = __ldg(p.bias + col);
            acc[4 * j + k] += b;
            acc[4 * j + 2 + k] += b;
          }
      }
    }
    // fp32 value of accumulator a in column col before the activation: + bias; s8: fmaf(acc, alpha, bias) (dequantise)
    auto head_val = [&](int a, int col) -> float {
      if constexpr (F16) {
        return acc[a];
      } else {
        const float b = p.bias ? __ldg(p.bias + col) : 0.0f;
        if constexpr (S8) return fmaf((float)acc[a], __ldg(p.alpha + col), b);
        else return acc[a] + b;
      }
    };
    if constexpr (OP == kOpF16) {
      // TMA-store epilogue, 64 columns at a time: both consumer warpgroups write the chunk's fp16 values into a staging
      // chunk with stmatrix (its fragment layout is the accumulator's), then one thread stores the chunk with one bulk
      // tensor store.  The map clips the box at the output's edges (rows past M, the image or the level, columns past
      // Cout), so only tile-table tiles that end inside the atlas's gaps keep the direct stores below.  A residual comes
      // through the ring (p.res_tma; the host sends launches whose residual cannot to the direct path) and is read with
      // ldmatrix in the same layout; the upsample addend is loaded into registers.
      if (p.tma_store && (!p.tile_tab || (h0 + p.TH <= hlim && w0 + p.TW <= wlim))) {
        const __half *up[2];
#pragma unroll
        for (int i = 0; i < 2; i++) {
          const int row = cw * 64 + warp * 16 + (lane >> 2) + 8 * i;
          int img = img0, h, w;
          bool valid;
          if (p.mode != 0) {
            const int dh = row / p.TW, dw = row - dh * p.TW;
            h = h0 + dh; w = w0 + dw;
            valid = row < patch && h < hlim && w < wlim;
          } else {
            const long long m = (long long)m_tile * 128 + row;
            valid = m < p.M;
            img = (int)(m / hw);
            const int rem = (int)(m - (long long)img * hw);
            h = rem / p.W;
            w = rem - h * p.W;
          }
          up[i] = p.upsample && valid ? p.upsample + (((long long)img * p.up_h + (h >> 1)) * p.up_w + (w >> 1)) * p.Cout : nullptr;
        }
        // ldmatrix / stmatrix row address of this lane: row lane % 8 of matrix lane / 8; matrices 1 and 3 are the rows + 8,
        // 2 and 3 the next 8 columns
        const int srow = cw * 64 + warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8, scol = (lane >> 4) * 8;
        const uint32_t stg = smem_u32(smem + kPipeBytes);
        // upsample addends of kJ column blocks (8 columns each) and both rows into registers ahead of their stmatrix: one
        // DRAM round trip per batch.  A whole chunk's batch spills at BN 256.
        constexpr int kJ = BN == 256 ? 4 : 8;
#pragma unroll
        for (int c = 0; c < BN / 64; c++) {
          const uint32_t buf = stg + (uint32_t)(sbuf * kStoreChunk);
          const uint32_t rbox = smem_u32(smem + stage * stage_bytes) + (uint32_t)((c % kResPerStage) * kStoreChunk);
          if (p.res_tma && c % kResPerStage == 0) mbar_wait(&bars->full[stage], phase);
#pragma unroll
          for (int jb = 0; jb < 8; jb += kJ) {
            __half2 uv[2][kJ];
#pragma unroll
            for (int jj = 0; jj < kJ; jj++) {
              const int col = n0 + 64 * c + 8 * (jb + jj) + 2 * q;
              if (col >= p.Cout) continue;   // Cout % 16 == 0: both columns of the pair are in range or neither
#pragma unroll
              for (int i = 0; i < 2; i++)
                if (up[i]) uv[i][jj] = *reinterpret_cast<const __half2 *>(up[i] + col);
            }
            if (jb == 0) {
              if (threadIdx.x == 128) bulk_wait_read<1>();   // the store issued two chunks ago has read this staging chunk
              asm volatile("bar.sync 3, 256;" ::: "memory");
            }
#pragma unroll
            for (int jj = 0; jj < kJ; jj += 2) {
              const uint32_t off = swz128_off(srow, 8 * (jb + jj) + scol);
              uint32_t r[4];
              if (p.res_tma) ldmatrix_x4(rbox + off, r[0], r[1], r[2], r[3]);
#pragma unroll
              for (int t = 0; t < 4; t++) {
                const int i = t & 1, jl = jj + (t >> 1), j = 8 * c + jb + jl;
                float v0 = acc[4 * j + 2 * i], v1 = acc[4 * j + 2 * i + 1];
                if (p.res_tma) { const float2 a = __half22float2(*reinterpret_cast<const __half2 *>(&r[t])); v0 += a.x; v1 += a.y; }
                if (up[i] && n0 + 8 * j + 2 * q < p.Cout) { const float2 a = __half22float2(uv[i][jl]); v0 += a.x; v1 += a.y; }
                __half2 y = __floats2half2_rn(v0, v1);
                if (p.relu) {   // on the packed halves: max(round(x), 0) == round(max(x, 0))
                  y = __hmax2(y, __float2half2_rn(0.0f));
                  if (p.relu == 2) y = __hmin2(y, __float2half2_rn(6.0f));   // ReLU6: 6.0 is exact in fp16
                }
                r[t] = *reinterpret_cast<const uint32_t *>(&y);
              }
              stmatrix_x4(buf + off, r[0], r[1], r[2], r[3]);
            }
          }
          if (p.res_tma && (c + 1) % kResPerStage == 0) {   // this warp has read the residual stage
            __syncwarp();
            if (lane == 0) mbar_arrive(&bars->empty[stage]);
            if (++stage == kStages) { stage = 0; phase ^= 1u; }
          }
          fence_proxy_async();
          asm volatile("bar.sync 3, 256;" ::: "memory");
          if (threadIdx.x == 128) {
            if (p.mode == 0) tma_store_2d(&tmY, buf, n0 + 64 * c, m_tile * 128);
            else tma_store_4d(&tmY, buf, n0 + 64 * c, w0, h0, img0);
            bulk_commit();
          }
          sbuf ^= 1;
        }
        continue;
      }
    }
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
      if constexpr (S8) {
        if (p.out_mode == ODTK_OUT_NHWC_S8) {
          // requantise for the next s8 layer: one fp32 multiply, round to nearest even, saturate to the symmetric range
          if (!valid) continue;
          const long long opix = p.mode != 0 ? ((long long)img * p.oH + p.oR + h) * p.oW + w : m;
          int8_t *o = reinterpret_cast<int8_t *>(p.out) + opix * p.ldy;
          const int8_t *res = p.res8 ? p.res8 + m * p.Cout : nullptr;
          const int8_t *up = p.up8 ? p.up8 + (((long long)img * p.up_h + (h >> 1)) * p.up_w + (w >> 1)) * p.Cout : nullptr;
#pragma unroll
          for (int j = 0; j < BN / 8; j++) {
            const int col = n0 + 8 * j + 2 * q;
            if (col >= p.Cout) continue;   // Cout % 16 == 0: both columns of the pair are in range or neither
            const char2 r = res ? *reinterpret_cast<const char2 *>(res + col) : make_char2(0, 0);
            const char2 u = up ? *reinterpret_cast<const char2 *>(up + col) : make_char2(0, 0);
            int qv[2];
#pragma unroll
            for (int k = 0; k < 2; k++) {
              float y = head_val(4 * j + 2 * i + k, col + k);
              // one correctly rounded fma per addend, in this order (DESIGN §2)
              if (res) y = fmaf((float)(k ? r.y : r.x), p.res_scale, y);
              if (up) y = fmaf((float)(k ? u.y : u.x), p.up_scale, y);
              if (p.relu) y = fmaxf(y, 0.0f);
              qv[k] = min(max(__float2int_rn(__fmul_rn(y, p.inv_out_scale)), -127), 127);
            }
            *reinterpret_cast<char2 *>(o + col) = make_char2((signed char)qv[0], (signed char)qv[1]);
          }
          continue;
        }
      }
      if constexpr (F32) {
        if (p.out_mode == ODTK_OUT_NHWC_F32) {
          // fp32 activations: + bias, + residual, + upsample (fp32 adds in this order), ReLU
          if (!valid) continue;
          const long long opix = p.mode != 0 ? ((long long)img * p.oH + p.oR + h) * p.oW + w : m;
          float *o = reinterpret_cast<float *>(p.out) + opix * p.ldy;
          const float *res = p.res32 ? p.res32 + m * p.ldr : nullptr;
          const float *up = p.up32 ? p.up32 + (((long long)img * p.up_h + (h >> 1)) * p.up_w + (w >> 1)) * p.Cout : nullptr;
#pragma unroll
          for (int j = 0; j < BN / 8; j++) {
            const int col = n0 + 8 * j + 2 * q;
            if (col >= p.Cout) continue;   // Cout even: both columns of the pair are in range or neither
            float v0 = acc[4 * j + 2 * i], v1 = acc[4 * j + 2 * i + 1];
            if (p.bias) { v0 += __ldg(p.bias + col); v1 += __ldg(p.bias + col + 1); }
            if (res) { const float2 r = *reinterpret_cast<const float2 *>(res + col); v0 += r.x; v1 += r.y; }
            if (up) { const float2 u = *reinterpret_cast<const float2 *>(up + col); v0 += u.x; v1 += u.y; }
            if (p.relu) { v0 = fmaxf(v0, 0.0f); v1 = fmaxf(v1, 0.0f); }
            *reinterpret_cast<float2 *>(o + col) = make_float2(v0, v1);
          }
          continue;
        }
      }
      if ((OP == kOpF16 || OP == kOpF16Mask) && p.out_mode == ODTK_OUT_NHWC_F16) {
        if (!valid) continue;
        const long long opix = p.mode != 0 ? ((long long)img * p.oH + p.oR + h) * p.oW + w : m;
        __half *o = reinterpret_cast<__half *>(p.out) + opix * p.ldy;
        const __half *res = p.residual ? p.residual + m * p.ldr : nullptr;
        const __half *up = p.upsample ? p.upsample + (((long long)img * p.up_h + (h >> 1)) * p.up_w + (w >> 1)) * p.Cout : nullptr;
        const __half *msk = nullptr;
        if constexpr (OP == kOpF16Mask) msk = p.mask ? p.mask + m * p.Cout : nullptr;
        // 64 columns at a time (32 at BN 256, next to the TMA-store epilogue): first every addend of the chunk into
        // registers, then the stores -- one DRAM round trip per chunk instead of one per column pair.  Wider chunks spill.
        constexpr int kJ = BN == 256 ? 4 : 8;
#pragma unroll
        for (int j0 = 0; j0 < BN / 8; j0 += kJ) {
          __half2 rv[kJ], uv[kJ], mv[kJ];
#pragma unroll
          for (int jj = 0; jj < kJ; jj++) {
            const int col = n0 + 8 * (j0 + jj) + 2 * q;
            if (col >= p.Cout) continue;   // Cout % 16 == 0: both columns of the pair are in range or neither
            if (res) rv[jj] = *reinterpret_cast<const __half2 *>(res + col);
            if (up) uv[jj] = *reinterpret_cast<const __half2 *>(up + col);
            if constexpr (OP == kOpF16Mask)
              if (msk) mv[jj] = *reinterpret_cast<const __half2 *>(msk + col);
          }
#pragma unroll
          for (int jj = 0; jj < kJ; jj++) {
            const int j = j0 + jj, col = n0 + 8 * j + 2 * q;
            if (col >= p.Cout) continue;
            float v0 = acc[4 * j + 2 * i], v1 = acc[4 * j + 2 * i + 1];
            if (res) { const float2 r = __half22float2(rv[jj]); v0 += r.x; v1 += r.y; }
            if (up) { const float2 u = __half22float2(uv[jj]); v0 += u.x; v1 += u.y; }
            if constexpr (OP == kOpF16Mask) {
              if (msk) {   // a select, not a product: an inf gradient where the input was <= 0 still becomes 0
                if (!(__low2float(mv[jj]) > 0.0f)) v0 = 0.0f;
                if (!(__high2float(mv[jj]) > 0.0f)) v1 = 0.0f;
              }
            }
            __half2 y = __floats2half2_rn(v0, v1);
            if (p.relu) {   // on the packed halves: max(round(x), 0) == round(max(x, 0))
              y = __hmax2(y, __float2half2_rn(0.0f));
              if (p.relu == 2) y = __hmin2(y, __float2half2_rn(6.0f));   // ReLU6: 6.0 is exact in fp16
            }
            *reinterpret_cast<__half2 *>(o + col) = y;
          }
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
          float x = head_val(4 * j + 2 * i + k, col);
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
            float x = head_val(4 * j + 2 * i + k, col);
            if (p.relu) x = fmaxf(x, 0.0f);
            if (p.out_mode == ODTK_OUT_NCHW_F32_SIGMOID) x = sigmoidf_accurate(x);
            o[(long long)col * hw] = x;
          }
      }
    }
  }
  // the bulk stores must have written the output before the grid completes (the next kernel's griddepcontrol.wait)
  if constexpr (OP == kOpF16)
    if (threadIdx.x == 128) bulk_wait_all<0>();
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
  int rank, swz, dtype;
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
                const uint32_t *box, CUtensorMapSwizzle swz, const uint32_t *elem_strides, CUtensorMapDataType dtype) {
  MapKey key;
  memset(&key, 0, sizeof key);
  key.base = base; key.rank = rank; key.swz = (int)swz; key.dtype = (int)dtype;
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
  CUresult r = fn(m, dtype, (cuuint32_t)rank, const_cast<void *>(base), gdim, gstr, bx, es,
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

template <int BN, int OP>
void launch_bn(int grid, cudaStream_t stream, const CUtensorMap &tmA, const CUtensorMap &tmB, const CUtensorMap &tmA2,
               const CUtensorMap &tmB2, const ConvParams &p, const CUtensorMap &tmY, const CUtensorMap &tmR) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = smem_bytes(OP);
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = odtk_pdl_on() ? 1 : 0;
  cudaLaunchKernelEx(&cfg, conv_gemm_kernel<BN, OP>, tmA, tmB, tmA2, tmB2, p, tmY, tmR);
}

// Every compile-time instance of conv_gemm_kernel: N tile, operand type, launcher and dynamic shared memory.
struct Instance {
  int bn, op;
  const void *fn;
  void (*launch)(int, cudaStream_t, const CUtensorMap &, const CUtensorMap &, const CUtensorMap &, const CUtensorMap &,
                 const ConvParams &, const CUtensorMap &, const CUtensorMap &);
  int smem;
};
template <int BN, int OP>
constexpr Instance instance() {
  return {BN, OP, (const void *)conv_gemm_kernel<BN, OP>, launch_bn<BN, OP>, smem_bytes(OP)};
}
const Instance kInstances[] = {instance<64, kOpF16>(),     instance<128, kOpF16>(),     instance<256, kOpF16>(),
                               instance<64, kOpS8>(),      instance<128, kOpS8>(),      instance<64, kOpTF32x3>(),
                               instance<128, kOpTF32x3>(), instance<64, kOpF16Mask>(),  instance<128, kOpF16Mask>()};

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
  for (const Instance &k : kInstances)
    if (cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, k.smem) != cudaSuccess) return false;
  g_dev_ready[dev] = true;
  return true;
}

thread_local odtk_conv_plan_t g_last_plan;

void set_stages(ConvParams &p, int BN, int op) {
  p.nstages = kPipeBytes / ((128 + (op == kOpTF32x3 ? 2 * BN : BN)) * p.row_bytes);
  if (p.nstages > kMaxStages) p.nstages = kMaxStages;
}

// BN 256 loads each A box once per 128 x 256 tile instead of once per 128-wide N tile (a 3x3 256 -> 256 layer moves 25 %
// fewer bytes from L2 into shared memory) and issues half the wgmma instructions.  The tiles are twice as long, so the
// last, partial wave costs twice as much: they must fill at least kWideWaves waves of the launch's SMs.  Measured per
// launch at batch 32 (DESIGN §6): 1x1, 3x3 and stride-2 layers of 15-61 waves ran 2-11 % faster at BN 256, a 3x3 of 2
// waves 3 % slower; the candidate epilogue of the class output layer (P3, 91 waves) ran 4 % slower and keeps BN 128.
constexpr int kWideWaves = 12;
bool wide_tiles_pay(const ConvParams &p, int cout) {
  return p.out_mode != ODTK_OUT_CANDIDATES &&
         (long long)p.num_m_tiles * ((cout + 255) / 256) >= (long long)kWideWaves * odtk_sm_count();
}

// Output map of the TMA-store epilogue (fp16 NHWC, row stride ldy, a multiple of 8 elements): mode 0 a 2-D map over the
// [M, ldy] rows in {64, 128} boxes; the spatial modes a 4-D map {Cout, W, H, N} whose origin is row oR of the output view
// and whose strides are those of the view, in {64, TW, TH, 1} boxes -- the box is clipped at the level's own W and H, so
// nothing outside the view's rectangle is written.
bool out_map(const ConvParams &p, CUtensorMap &tmY) {
  const uint64_t ldy = (uint64_t)p.ldy * 2;
  if (p.mode == 0) {
    uint64_t dims[2] = {(uint64_t)p.Cout, (uint64_t)p.M}, str[1] = {ldy};
    uint32_t box[2] = {64, 128};
    return encode_map(&tmY, p.out, 2, dims, str, box);
  }
  const unsigned char *base = reinterpret_cast<const unsigned char *>(p.out) + (uint64_t)p.oR * p.oW * ldy;
  uint64_t dims[4] = {(uint64_t)p.Cout, (uint64_t)p.W, (uint64_t)p.H, (uint64_t)p.N};
  uint64_t str[3] = {ldy, (uint64_t)p.oW * ldy, (uint64_t)p.oH * p.oW * ldy};
  uint32_t box[4] = {64, (uint32_t)p.TW, (uint32_t)p.TH, 1};
  return encode_map(&tmY, base, 4, dims, str, box);
}

int launch(ConvParams p, int BN, const CUtensorMap &tmA, const CUtensorMap &tmB, const CUtensorMap &tmA2,
           const CUtensorMap &tmB2, cudaStream_t stream, int op) {
  const int total = p.num_m_tiles * p.num_n_tiles;
  const int sms = odtk_sm_count();   // the launch budget (odtk_set_sm_budget) or the whole device
  const int grid = total < sms ? total : sms;
  CUtensorMap tmY = tmA, tmR = tmA;
  p.tma_store = op == kOpF16 && p.out_mode == ODTK_OUT_NHWC_F16 && g_odtk_tma_store;
  if (p.tma_store && p.residual) {
    // the residual goes through the ring as [M, ldr] rows in {64, 128} boxes: mode 0, 16-byte aligned rows; other
    // residual launches keep the direct epilogue
    p.res_tma = p.mode == 0 && !((uintptr_t)p.residual & 15) && p.ldr % 8 == 0;
    p.tma_store = p.res_tma;
    uint64_t dims[2] = {(uint64_t)p.Cout, (uint64_t)p.M}, str[1] = {(uint64_t)p.ldr * 2};
    uint32_t box[2] = {64, 128};
    if (p.res_tma && !encode_map(&tmR, p.residual, 2, dims, str, box)) return ODTK_E_CUDA;
  }
  if (p.tma_store && !out_map(p, tmY)) return ODTK_E_CUDA;
  g_last_plan = odtk_conv_plan_t{p.mode, 0, BN, p.num_m_tiles, p.num_n_tiles, p.nstages, 0, 0, 0, 0, 0, p.tma_store,
                                 p.TH, p.TW, grid, 0};
  for (const Instance &k : kInstances)
    if (k.bn == BN && k.op == op) {
      OdtkProfScope prof(ODTK_PROF_CONV, stream);
      k.launch(grid, stream, tmA, tmB, tmA2, tmB2, p, tmY, tmR);
      return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
    }
  return ODTK_E_UNSUPPORTED;
}

// out_mode ODTK_OUT_CANDIDATES: the decode workspace of the level the launch covers
int set_sink(ConvParams &p, const odtk_cand_sink_t *k, int cout, int h, int width) {
  if (!k->counts || !k->hist || !k->cand || k->hist_bins <= 0) return ODTK_E_INVALID;
  if ((long long)cout * h * width >= (1ll << 32)) return ODTK_E_UNSUPPORTED;
  p.cand_counts = k->counts; p.cand_hist = k->hist; p.cand = (uint2 *)k->cand; p.cand_cap = k->cap;
  p.cand_key_thresh = k->key_thresh; p.cand_shift = k->shift; p.cand_hist_bins = k->hist_bins;
  p.cand_thresh = k->thresh;
  // sigmoid(x) > thresh implies x > logit(thresh) - margin (the SFU sigmoid is accurate to 1e-6 relative)
  p.cand_pre = (k->thresh > 1e-4f && k->thresh < 0.999f) ? logf(k->thresh / (1.0f - k->thresh)) - 0.05f : -INFINITY;
  return ODTK_OK;
}

CUtensorMapDataType map_type(int es) {
  return es == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : es == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
}

// A operand of a 1x1 / 3x3, stride 1 / 2 launch: the mode, the output patch and tile grid, and the tensor map of x (the
// top-left h x width rectangle of images xH x xW pixels apart).  es: bytes per element, 2 (fp16), 1 (s8) or 4 (fp32); a K
// block is one 128-byte swizzle row of channels either way.
int a_operand(ConvParams &p, CUtensorMap &tmA, const void *x, int n, int h, int width, int cin, int ksize, int stride,
              uint64_t xH, uint64_t xW, bool x_view, const void *tile_tab, int tab_tiles, int es) {
  const CUtensorMapDataType dt = map_type(es);
  const uint32_t kc = 128 / es;   // channels per K block
  const uint64_t C = (uint64_t)cin, W = (uint64_t)width, H = (uint64_t)h;
  if (stride == 2 && ((h & 1) || (width & 1) || x_view)) {
    // stride-2 1x1 / 3x3 (pad ksize/2) on odd sizes, im2col-free: one box per tap whose W and H dimensions are
    // traversed with element stride 2 (boxDim = 2 * pixels, elementStrides = 2: the TMA unit loads every second
    // pixel); the box origin 2*o + d may be -1 or reach past the edge: zero-filled == padding.
    const int OH = (h - 1) / 2 + 1, OW = (width - 1) / 2 + 1;
    p.mode = 1;
    p.s2 = 1;
    p.H = OH; p.W = OW;
    p.M = (long long)n * OH * OW;
    p.up_h = OH / 2; p.up_w = OW / 2;
    choose_patch(OH, OW, p.TH, p.TW);
    if (2 * p.TW > 256 || 2 * p.TH > 256) return ODTK_E_UNSUPPORTED;
    p.tiles_h = (OH + p.TH - 1) / p.TH;
    p.tiles_w = (OW + p.TW - 1) / p.TW;
    p.num_m_tiles = n * p.tiles_h * p.tiles_w;
    uint64_t dims[4] = {C, W, H, (uint64_t)n};
    uint64_t str[3] = {C * es, xW * C * es, xH * xW * C * es};
    uint32_t box[4] = {kc, (uint32_t)(2 * p.TW), (uint32_t)(2 * p.TH), 1};
    uint32_t estr[4] = {1, 2, 2, 1};
    if (!encode_map(&tmA, x, 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, estr, dt)) return ODTK_E_CUDA;
  } else if (stride == 2) {
    // stride-2 1x1 / 3x3 (pad ksize/2) on even-sized inputs: 5-D parity-split view of the NHWC tensor
    // {2C (column parity x channel), W/2, 2 (row parity), H/2, N}; out-of-range half-rows/columns
    // (the -1 of the top/left taps) are zero-filled by the TMA unit == padding.
    const int OH = h / 2, OW = width / 2;
    p.mode = 3;
    p.H = OH; p.W = OW;
    p.M = (long long)n * OH * OW;
    p.up_h = OH / 2; p.up_w = OW / 2;
    choose_patch(OH, OW, p.TH, p.TW);
    p.tiles_h = (OH + p.TH - 1) / p.TH;
    p.tiles_w = (OW + p.TW - 1) / p.TW;
    p.num_m_tiles = n * p.tiles_h * p.tiles_w;
    uint64_t dims[5] = {2 * C, W / 2, 2, H / 2, (uint64_t)n};
    uint64_t str[4] = {2 * C * es, W * C * es, 2 * W * C * es, H * W * C * es};
    uint32_t box[5] = {kc, (uint32_t)p.TW, 1, (uint32_t)p.TH, 1};
    if (!encode_map(&tmA, x, 5, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, nullptr, dt)) return ODTK_E_CUDA;
  } else if (ksize == 1) {
    p.mode = 0;
    p.num_m_tiles = (int)((p.M + 127) / 128);
    uint64_t dims[2] = {C, (uint64_t)p.M};
    uint64_t str[1] = {C * es};
    uint32_t box[2] = {kc, 128};
    if (!encode_map(&tmA, x, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, nullptr, dt)) return ODTK_E_CUDA;
  } else {
    p.mode = 1;
    if (tile_tab) {   // atlas tile tables list 8 x 16 pixel tiles
      p.TH = 8; p.TW = 16;
      p.tile_tab = (const int4 *)tile_tab; p.tab_tiles = tab_tiles;
    } else {
      choose_patch(h, width, p.TH, p.TW);
    }
    p.tiles_h = (h + p.TH - 1) / p.TH;
    p.tiles_w = (width + p.TW - 1) / p.TW;
    p.num_m_tiles = tile_tab ? n * tab_tiles : n * p.tiles_h * p.tiles_w;
    uint64_t dims[4] = {C, W, H, (uint64_t)n};
    uint64_t str[3] = {C * es, xW * C * es, xH * xW * C * es};
    uint32_t box[4] = {kc, (uint32_t)p.TW, (uint32_t)p.TH, 1};
    if (!encode_map(&tmA, x, 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, nullptr, dt)) return ODTK_E_CUDA;
  }
  return ODTK_OK;
}

// A operand of the ResNet stem (mode 2): 7x7 stride-2 pad-3 over the image zero-padded to NHWC4 [n, h+6, width+8, 4], im2col-
// free.  For filter row r the A operand of output pixels (oh, ow..) is the 8-pixel x 4-channel window starting at padded
// pixel (2*oh + r, 2*ow): 32 elements, consecutive output pixels 8 elements apart -- an OVERLAPPING-window 5-D tensor map
// {32 elements, OW, 7 rows (one padded row), OH (two padded rows), N}.  One window row is one swizzle row: 64 bytes in
// fp16, 128 in fp32; K = 7 blocks of 32.
int stem_operand(ConvParams &p, CUtensorMap &tmA, const void *xp, int n, int h, int width, int es) {
  const int OH = (h - 1) / 2 + 1, OW = (width - 1) / 2 + 1;
  const uint64_t HP = (uint64_t)h + 6, WP = (uint64_t)width + 8;
  p.mode = 2;
  p.H = OH; p.W = OW; p.Cin = 4;
  p.kw = 1; p.taps = 7; p.pad = 0; p.kblocks_per_tap = 1;
  p.row_bytes = 32 * es;
  p.M = (long long)n * OH * OW;
  choose_patch(OH, OW, p.TH, p.TW);
  p.tiles_h = (OH + p.TH - 1) / p.TH;
  p.tiles_w = (OW + p.TW - 1) / p.TW;
  p.num_m_tiles = n * p.tiles_h * p.tiles_w;
  uint64_t dims[5] = {32, (uint64_t)OW, 7, (uint64_t)OH, (uint64_t)n};
  uint64_t str[4] = {8 * (uint64_t)es, WP * 4 * es, WP * 8 * es, HP * WP * 4 * es};
  uint32_t box[5] = {32, (uint32_t)p.TW, 1, (uint32_t)p.TH, 1};
  if (!encode_map(&tmA, xp, 5, dims, str, box, es == 4 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B, nullptr,
                  map_type(es)))
    return ODTK_E_UNSUPPORTED;
  return ODTK_OK;
}

// B operand: weights [cout, K] in boxes of one swizzle row (p.row_bytes) x BN output channels
bool b_operand(CUtensorMap &tmB, const void *w, uint64_t K, int cout, int BN, int row_bytes, int es) {
  uint64_t dims[2] = {K, (uint64_t)cout};
  uint64_t str[1] = {K * es};
  uint32_t box[2] = {(uint32_t)(row_bytes / es), (uint32_t)BN};
  return encode_map(&tmB, w, 2, dims, str, box, row_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                    nullptr, map_type(es));
}

// What differs between the operand types of the convolution entry points; a K block is one 128-byte row of 128 / es
// channels, so Cin must be a multiple of that.
struct OpSpec {
  int op;           // conv_gemm_kernel instance
  int es;           // bytes per activation / weight element
  int nhwc_mode;    // the NHWC output mode; the others are ODTK_OUT_NCHW_F32[_SIGMOID] and ODTK_OUT_CANDIDATES
  int nhwc_cout;    // Cout multiple of NHWC outputs
  int ldy_mult;     // output row stride multiple of NHWC outputs
  int addend_align; // byte alignment of the residual / upsample addends
  bool relu6;       // relu 2 (ReLU6, NHWC output only) allowed; otherwise relu is 0 or 1
};
constexpr OpSpec kSpecF16 = {kOpF16, 2, ODTK_OUT_NHWC_F16, 16, 8, 4, true};
constexpr OpSpec kSpecS8 = {kOpS8, 1, ODTK_OUT_NHWC_S8, 16, 1, 2, false};
constexpr OpSpec kSpecF32 = {kOpTF32x3, 4, ODTK_OUT_NHWC_F32, 2, 2, 8, false};

// The fields of odtk_conv_t, odtk_conv_s8_ex_t and odtk_conv_f32_t in one place, plus the fp16-only extras: a second
// operand pair (mode 0) added to the same accumulator, y = x * w^T + x2 * w2^T with x2 [M, c2in], w2 [cout, c2in] (the
// projected identity of a bottleneck block), and the input-gradient launch (odtk_conv2d_dgrad: the masked instance, 3x3 or
// dense 1x1; a tile-table launch may then take a residual, a whole atlas like y).
struct ConvArgs {
  const void *x, *w, *w_lo, *residual, *upsample, *x2, *w2, *mask, *tile_tab;
  const float *bias, *alpha;
  void *y;
  const odtk_cand_sink_t *sink;
  int n, h, width, cin, cout, ksize, stride, relu, out_mode, ldy, ldr, groups, c2in, tab_tiles;
  int x_rows, x_width, y_rows, y_row_off, y_width;
  float inv_out_scale, res_scale, up_scale;
  bool dgrad;
};

// One convolution on conv_gemm_kernel: 1x1 as GEMM rows (mode 0), 3x3 as shifted boxes (mode 1) over a dense tensor, a
// level view of the atlas or the whole atlas with its tile table, stride 2 on the parity-split view (mode 3, even sizes) or
// element-strided boxes (odd sizes, level views), and in fp32 the 7x7 stem (mode 2).  NHWC outputs may add a residual and /
// or a nearest-upsampled addend, and may land in a level view of an atlas.  Every argument is checked before any CUDA call.
int conv_run(const ConvArgs &a, const OpSpec &s, cudaStream_t stream) {
  if (!a.x || !a.w || (s.op == kOpS8 && !a.alpha) || (s.op == kOpTF32x3 && !a.w_lo)) return ODTK_E_INVALID;
  // dgrad: 3x3, or 1x1 (mode 0, dense) masked, into the input channels of a layer odtk_conv_wgrad_ex takes
  const bool dgrad_1x1 = a.ksize == 1 && a.mask && a.cout % 128 == 0 && !a.tile_tab;
  if (a.dgrad && ((a.ksize != 3 && !dgrad_1x1) || a.stride > 1 || a.out_mode != ODTK_OUT_NHWC_F16 || a.relu ||
                  a.groups > 1 || a.upsample || a.x_rows > 0 || a.x_width > 0 || a.y_rows > 0 || a.y_width > 0 ||
                  a.y_row_off > 0))
    return ODTK_E_UNSUPPORTED;
  if (a.mask && ((uintptr_t)a.mask & 3)) return ODTK_E_INVALID;
  if (a.out_mode == ODTK_OUT_CANDIDATES ? !a.sink : !a.y) return ODTK_E_INVALID;
  if (a.n <= 0 || a.h <= 0 || a.width <= 0 || a.cin <= 0 || a.cout <= 0) return ODTK_E_INVALID;
  if (a.out_mode != s.nhwc_mode && a.out_mode != ODTK_OUT_NCHW_F32 && a.out_mode != ODTK_OUT_NCHW_F32_SIGMOID &&
      a.out_mode != ODTK_OUT_CANDIDATES)
    return ODTK_E_INVALID;
  const int stride = a.stride > 1 ? a.stride : 1;
  const bool stem = s.op == kOpTF32x3 && a.ksize == 7;   // the fp32 ResNet stem over the NHWC4 image
  const int kc = 128 / s.es;                              // channels per K block
  if (stem ? (a.cin != 3 || stride != 2) : ((a.ksize != 1 && a.ksize != 3) || a.cin % kc)) return ODTK_E_UNSUPPORTED;
  const int groups = a.groups > 1 ? a.groups : 1;
  if (groups > 1) {
    // grouped convolution (ResNeXt conv2): output block j of 64 channels depends only on input chunk j, as long as a
    // group never straddles a 64-channel chunk; `w` is then [cout, ksize*ksize*64], block-diagonal inside the chunk
    if (a.cin != a.cout || a.cin % groups || 64 % (a.cin / groups) || a.residual || a.upsample || a.ksize != 3 ||
        a.out_mode != ODTK_OUT_NHWC_F16)
      return ODTK_E_UNSUPPORTED;
  }
  if (stride != 1 && stride != 2) return ODTK_E_UNSUPPORTED;
  if (s.relu6 ? (a.relu == 2 && a.out_mode != s.nhwc_mode) : (a.relu != 0 && a.relu != 1)) return ODTK_E_UNSUPPORTED;
  const bool nhwc = a.out_mode == s.nhwc_mode;
  if (nhwc && (a.cout % s.nhwc_cout)) return ODTK_E_UNSUPPORTED;
  if ((long long)a.n * a.h * a.width >= (1ll << 31)) return ODTK_E_UNSUPPORTED;
  if (((uintptr_t)a.x | (uintptr_t)a.w | (uintptr_t)a.w_lo | (a.out_mode == ODTK_OUT_CANDIDATES ? 0 : (uintptr_t)a.y)) & 15)
    return ODTK_E_INVALID;
  // strided views: the input / output may be a rectangle of a larger NHWC buffer (a level of the pyramid atlas)
  const uint64_t xH = a.x_rows > 0 ? (uint64_t)a.x_rows : (uint64_t)a.h, xW = a.x_width > 0 ? (uint64_t)a.x_width : (uint64_t)a.width;
  const bool x_view = xH != (uint64_t)a.h || xW != (uint64_t)a.width;
  const bool y_view = a.y_rows > 0 || a.y_width > 0 || a.y_row_off > 0;
  const bool addend = a.residual || a.upsample;
  // addends and output views need the NHWC output; views and tile tables are 3x3 without addends
  if ((addend || y_view) && !nhwc) return ODTK_E_UNSUPPORTED;
  if ((x_view || y_view || (a.tile_tab && !a.dgrad)) && (a.ksize != 3 || addend)) return ODTK_E_UNSUPPORTED;
  if ((stem && addend) || (a.upsample && stride != 1)) return ODTK_E_UNSUPPORTED;
  if (a.tile_tab && (a.tab_tiles <= 0 || x_view || y_view || stride != 1)) return ODTK_E_INVALID;
  if ((((uintptr_t)a.residual | (uintptr_t)a.upsample) & (s.addend_align - 1)) || (a.upsample && ((a.h & 1) || (a.width & 1))))
    return ODTK_E_INVALID;
  const int ldy = a.ldy > 0 ? a.ldy : a.cout, ldr = a.ldr > 0 ? a.ldr : a.cout;
  if ((nhwc && ldy % s.ldy_mult) || (a.residual && (ldr & 1))) return ODTK_E_INVALID;
  if (a.x2 && (a.ksize != 1 || stride != 1 || a.c2in <= 0 || a.c2in % 64 || !a.w2 || (((uintptr_t)a.x2 | (uintptr_t)a.w2) & 15)))
    return ODTK_E_INVALID;
  if (a.dgrad && ldy != a.cout) return ODTK_E_UNSUPPORTED;   // the mask is read with the output's row stride
  if (!device_ready()) return ODTK_E_CUDA;
  const int op = a.dgrad ? kOpF16Mask : s.op;
  ConvParams p;
  memset(&p, 0, sizeof p);
  p.N = a.n; p.H = a.h; p.W = a.width; p.Cin = a.cin; p.Cout = a.cout;
  p.kw = a.ksize; p.taps = a.ksize * a.ksize; p.pad = a.ksize / 2;
  p.kblocks_per_tap = groups > 1 ? 1 : a.cin / kc;
  p.grouped = groups > 1;
  p.row_bytes = 128;
  p.M = (long long)a.n * a.h * a.width;
  p.bias = a.bias;
  p.out = a.y;
  p.relu = a.relu;
  p.out_mode = a.out_mode;
  p.ldy = ldy;
  p.ldr = ldr;
  p.up_h = a.h / 2; p.up_w = a.width / 2;
  if (s.op == kOpS8) {
    p.alpha = a.alpha;
    p.inv_out_scale = a.inv_out_scale;
    p.res8 = (const int8_t *)a.residual; p.res_scale = a.res_scale;
    p.up8 = (const int8_t *)a.upsample; p.up_scale = a.up_scale;
  } else if (s.op == kOpTF32x3) {
    p.res32 = (const float *)a.residual;
    p.up32 = (const float *)a.upsample;
  } else {
    p.residual = (const __half *)a.residual;
    p.upsample = (const __half *)a.upsample;
    p.mask = (const __half *)a.mask;
  }
  if (p.out_mode == ODTK_OUT_CANDIDATES) {
    const int rc = set_sink(p, a.sink, a.cout, a.h, a.width);
    if (rc != ODTK_OK) return rc;
  }
  CUtensorMap tmA;
  const int rc = stem ? stem_operand(p, tmA, a.x, a.n, a.h, a.width, s.es)
                      : a_operand(p, tmA, a.x, a.n, a.h, a.width, a.cin, a.ksize, stride, xH, xW, x_view, a.tile_tab,
                                  a.tab_tiles, s.es);
  if (rc != ODTK_OK) return rc;
  p.oH = a.y_rows > 0 ? a.y_rows : p.H;
  p.oR = a.y_row_off > 0 ? a.y_row_off : 0;
  p.oW = a.y_width > 0 ? a.y_width : p.W;
  if ((long long)a.n * p.oH * p.oW >= (1ll << 31) || p.oR + p.H > p.oH || p.W > p.oW) return ODTK_E_INVALID;
  // N tile: 64, 128 or 256 output channels.  128 halves the A-operand traffic; 64 when Cout is narrow, for grouped convs
  // (one 64-channel chunk per tile), or when 128-wide tiles would leave SMs idle; 256 (fp16 forward) for the wide layers
  // with enough tiles (wide_tiles_pay).
  int BN = (groups > 1 || a.cout <= 64) ? 64 : 128;
  if (BN == 128 && (long long)p.num_m_tiles * ((a.cout + 127) / 128) < odtk_sm_count()) BN = 64;
  if (BN == 128 && op == kOpF16 && a.cout > 128 && wide_tiles_pay(p, a.cout)) BN = 256;
  p.num_n_tiles = (a.cout + BN - 1) / BN;
  set_stages(p, BN, op);
  CUtensorMap tmB, tmA2 = tmA, tmB2;
  const uint64_t K = stem ? 224 : (uint64_t)p.taps * (groups > 1 ? 64 : a.cin);
  if (!b_operand(tmB, a.w, K, a.cout, BN, p.row_bytes, s.es)) return ODTK_E_CUDA;
  tmB2 = tmB;
  if (a.w_lo && !b_operand(tmB2, a.w_lo, K, a.cout, BN, p.row_bytes, s.es)) return ODTK_E_CUDA;   // fp32: the low weight half
  if (a.x2) {
    p.kblocks2 = a.c2in / 64;
    uint64_t dims[2] = {(uint64_t)a.c2in, (uint64_t)p.M}, str[1] = {(uint64_t)a.c2in * 2};
    uint32_t box[2] = {64, 128};
    if (!encode_map(&tmA2, a.x2, 2, dims, str, box) || !b_operand(tmB2, a.w2, a.c2in, a.cout, BN, 128, 2)) return ODTK_E_CUDA;
  }
  return launch(p, BN, tmA, tmB, tmA2, tmB2, stream, op);
}

ConvArgs f16_args(const odtk_conv_t *d) {
  ConvArgs a;
  memset(&a, 0, sizeof a);
  a.x = d->x; a.w = d->w; a.bias = d->bias; a.residual = d->residual; a.upsample = d->upsample; a.y = d->y;
  a.n = d->n; a.h = d->h; a.width = d->width; a.cin = d->cin; a.cout = d->cout; a.ksize = d->ksize; a.relu = d->relu;
  a.out_mode = d->out_mode; a.ldy = d->ldy; a.ldr = d->ldr; a.stride = d->stride; a.sink = d->sink; a.groups = d->groups;
  a.x_rows = d->x_rows; a.x_width = d->x_width; a.y_rows = d->y_rows; a.y_row_off = d->y_row_off; a.y_width = d->y_width;
  a.tile_tab = d->tile_tab; a.tab_tiles = d->tab_tiles;
  return a;
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
  if (!d) return ODTK_E_INVALID;
  return conv_run(f16_args(d), kSpecF16, (cudaStream_t)stream_);
}

extern "C" int odtk_conv2d_dgrad(const odtk_conv_dgrad_t *d, odtk_stream_t stream_) {
  if (!d) return ODTK_E_INVALID;
  ConvArgs a = f16_args(&d->base);
  a.dgrad = true;
  a.mask = d->mask;
  return conv_run(a, kSpecF16, (cudaStream_t)stream_);
}

extern "C" int odtk_conv2d_s8_ex(const odtk_conv_s8_ex_t *e, odtk_stream_t stream_) {
  if (!e) return ODTK_E_INVALID;
  const odtk_conv_s8_t *d = &e->base;
  ConvArgs a;
  memset(&a, 0, sizeof a);
  a.x = d->x; a.w = d->w; a.alpha = d->alpha; a.bias = d->bias; a.y = d->y;
  a.n = d->n; a.h = d->h; a.width = d->width; a.cin = d->cin; a.cout = d->cout; a.ksize = d->ksize; a.relu = d->relu;
  a.out_mode = d->out_mode; a.inv_out_scale = d->inv_out_scale; a.sink = d->sink;
  a.x_rows = d->x_rows; a.x_width = d->x_width; a.tile_tab = d->tile_tab; a.tab_tiles = d->tab_tiles;
  a.stride = e->stride; a.residual = e->residual; a.res_scale = e->res_scale; a.upsample = e->upsample; a.up_scale = e->up_scale;
  a.y_rows = e->y_rows; a.y_row_off = e->y_row_off; a.y_width = e->y_width;
  return conv_run(a, kSpecS8, (cudaStream_t)stream_);
}

extern "C" int odtk_conv2d_s8(const odtk_conv_s8_t *d, odtk_stream_t stream_) {
  if (!d) return ODTK_E_INVALID;
  odtk_conv_s8_ex_t e;
  memset(&e, 0, sizeof e);
  e.base = *d;
  return odtk_conv2d_s8_ex(&e, stream_);
}

extern "C" int odtk_conv2d_f32(const odtk_conv_f32_t *d, odtk_stream_t stream_) {
  if (!d) return ODTK_E_INVALID;
  ConvArgs a;
  memset(&a, 0, sizeof a);
  a.x = d->x; a.w = d->w_hi; a.w_lo = d->w_lo; a.bias = d->bias; a.residual = d->residual; a.upsample = d->upsample; a.y = d->y;
  a.n = d->n; a.h = d->h; a.width = d->width; a.cin = d->cin; a.cout = d->cout; a.ksize = d->ksize; a.stride = d->stride;
  a.relu = d->relu; a.out_mode = d->out_mode; a.ldy = d->ldy; a.ldr = d->ldr; a.sink = d->sink;
  a.x_rows = d->x_rows; a.x_width = d->x_width; a.y_rows = d->y_rows; a.y_row_off = d->y_row_off; a.y_width = d->y_width;
  a.tile_tab = d->tile_tab; a.tab_tiles = d->tab_tiles;
  return conv_run(a, kSpecF32, (cudaStream_t)stream_);
}

// ResNet stem in fp16: 7x7 stride-2 pad-3 convolution of the RGB image zero-padded to NHWC4 [n, h+6, w+8, 4] fp16 by
// odtk_pad_input (stem_operand), weights packed [cout, 7*32] with k = r*32 + s*4 + c (zero for s = 7 or c = 3).  Even h and
// width; one N tile (cout <= 128).
extern "C" int odtk_stem_conv(const void *xp, const void *w, const float *bias, void *y, int n, int h, int width,
                              int cout, int relu, odtk_stream_t stream_) {
  if (!xp || !w || !y || n <= 0 || h <= 0 || width <= 0) return ODTK_E_INVALID;
  if ((h & 1) || (width & 1) || cout % 16 || cout > 128) return ODTK_E_UNSUPPORTED;
  if (((uintptr_t)xp | (uintptr_t)w | (uintptr_t)y) & 15) return ODTK_E_INVALID;
  if (!device_ready()) return ODTK_E_CUDA;
  if ((long long)n * (h / 2) * (width / 2) >= (1ll << 31)) return ODTK_E_UNSUPPORTED;
  ConvParams p;
  memset(&p, 0, sizeof p);
  p.N = n; p.Cout = cout;
  CUtensorMap tmA, tmB;
  const int rc = stem_operand(p, tmA, xp, n, h, width, 2);
  if (rc != ODTK_OK) return rc;
  const int BN = cout <= 64 ? 64 : 128;
  p.num_n_tiles = 1;
  set_stages(p, BN, kOpF16);
  p.bias = bias; p.out = y; p.relu = relu; p.out_mode = ODTK_OUT_NHWC_F16; p.ldy = cout; p.ldr = cout;
  p.oH = p.H; p.oR = 0; p.oW = p.W;
  if (!b_operand(tmB, w, 224, cout, BN, p.row_bytes, 2)) return ODTK_E_CUDA;
  return launch(p, BN, tmA, tmB, tmA, tmB, (cudaStream_t)stream_, kOpF16);
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
