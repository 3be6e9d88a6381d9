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

// operand types of conv_gemm_kernel; kOpF16Mask: fp16 with the ReLU-derivative mask of the input gradient (odtk_conv2d_dgrad)
enum ConvOp { kOpF16 = 0, kOpS8 = 1, kOpTF32x3 = 2, kOpF16Mask = 3 };

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
template <int BN, int OP>
__global__ void __launch_bounds__(kThreads, 1)
conv_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2,
                 const __grid_constant__ ConvParams p) {
  constexpr bool S8 = OP == kOpS8, F32 = OP == kOpTF32x3;
  constexpr int BR = F32 ? 2 * BN : BN;   // B rows per stage: fp32 carries w_hi and w_lo
  extern __shared__ unsigned char smem_raw[];
  unsigned char *smem = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  Barriers *bars = reinterpret_cast<Barriers *>(smem + kPipeBytes + (F32 ? kSplitBytes : 0));
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
    }
    return;
  }

  // ===================================== MMA + epilogue ======================================
  const int cw = wg - 1, warp = tid >> 5, lane = tid & 31;
  const int q = lane & 3;
  const int hw = p.H * p.W, patch = p.TH * p.TW;
  typename std::conditional<S8, int, float>::type acc[BN / 2];
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
    // fp32 value of accumulator a in column col before the activation: + bias; s8: fmaf(acc, alpha, bias) (dequantise)
    auto head_val = [&](int a, int col) -> float {
      const float b = p.bias ? __ldg(p.bias + col) : 0.0f;
      if constexpr (S8) return fmaf((float)acc[a], __ldg(p.alpha + col), b);
      else return acc[a] + b;
    };
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
#pragma unroll
        for (int j = 0; j < BN / 8; j++) {
          const int col = n0 + 8 * j + 2 * q;
          if (col >= p.Cout) continue;   // Cout % 16 == 0: both columns of the pair are in range or neither
          float v0 = acc[4 * j + 2 * i], v1 = acc[4 * j + 2 * i + 1];
          if (p.bias) { v0 += __ldg(p.bias + col); v1 += __ldg(p.bias + col + 1); }
          if (res) { const float2 r = __half22float2(*reinterpret_cast<const __half2 *>(res + col)); v0 += r.x; v1 += r.y; }
          if (up) { const float2 u = __half22float2(*reinterpret_cast<const __half2 *>(up + col)); v0 += u.x; v1 += u.y; }
          if constexpr (OP == kOpF16Mask) {
            if (msk) {   // a select, not a product: an inf gradient where the input was <= 0 still becomes 0
              const __half2 mm = *reinterpret_cast<const __half2 *>(msk + col);
              if (!(__low2float(mm) > 0.0f)) v0 = 0.0f;
              if (!(__high2float(mm) > 0.0f)) v1 = 0.0f;
            }
          }
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
               const CUtensorMap &tmB2, const ConvParams &p) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = OP == kOpTF32x3 ? kSmemBytesF32 : kSmemBytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = odtk_pdl_on() ? 1 : 0;
  cudaLaunchKernelEx(&cfg, conv_gemm_kernel<BN, OP>, tmA, tmB, tmA2, tmB2, p);
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
  if (cudaFuncSetAttribute(conv_gemm_kernel<64, kOpF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes) != cudaSuccess ||
      cudaFuncSetAttribute(conv_gemm_kernel<128, kOpF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes) != cudaSuccess ||
      cudaFuncSetAttribute(conv_gemm_kernel<64, kOpS8>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes) != cudaSuccess ||
      cudaFuncSetAttribute(conv_gemm_kernel<128, kOpS8>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes) != cudaSuccess ||
      cudaFuncSetAttribute(conv_gemm_kernel<64, kOpTF32x3>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytesF32) != cudaSuccess ||
      cudaFuncSetAttribute(conv_gemm_kernel<128, kOpTF32x3>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytesF32) != cudaSuccess ||
      cudaFuncSetAttribute(conv_gemm_kernel<64, kOpF16Mask>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes) != cudaSuccess ||
      cudaFuncSetAttribute(conv_gemm_kernel<128, kOpF16Mask>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes) != cudaSuccess)
    return false;
  g_dev_ready[dev] = true;
  return true;
}

thread_local odtk_conv_plan_t g_last_plan;

void set_stages(ConvParams &p, int BN, int op = kOpF16) {
  p.nstages = kPipeBytes / ((128 + (op == kOpTF32x3 ? 2 * BN : BN)) * p.row_bytes);
  if (p.nstages > kMaxStages) p.nstages = kMaxStages;
}

int launch(const ConvParams &p, int BN, const CUtensorMap &tmA, const CUtensorMap &tmB, const CUtensorMap &tmA2,
           const CUtensorMap &tmB2, cudaStream_t stream, int op = kOpF16) {
  const int total = p.num_m_tiles * p.num_n_tiles;
  const int sms = odtk_sm_count();   // the launch budget (odtk_set_sm_budget) or the whole device
  const int grid = total < sms ? total : sms;
  g_last_plan = odtk_conv_plan_t{p.mode, 0, BN, p.num_m_tiles, p.num_n_tiles, p.nstages, 0, 0, 0, 0, 0, 0, p.TH, p.TW, grid, 0};
  {
    OdtkProfScope prof(ODTK_PROF_CONV, stream);
    if (op == kOpS8) {
      if (BN == 64) launch_bn<64, kOpS8>(grid, stream, tmA, tmB, tmA2, tmB2, p);
      else          launch_bn<128, kOpS8>(grid, stream, tmA, tmB, tmA2, tmB2, p);
    } else if (op == kOpTF32x3) {
      if (BN == 64) launch_bn<64, kOpTF32x3>(grid, stream, tmA, tmB, tmA2, tmB2, p);
      else          launch_bn<128, kOpTF32x3>(grid, stream, tmA, tmB, tmA2, tmB2, p);
    } else if (op == kOpF16Mask) {
      if (BN == 64) launch_bn<64, kOpF16Mask>(grid, stream, tmA, tmB, tmA2, tmB2, p);
      else          launch_bn<128, kOpF16Mask>(grid, stream, tmA, tmB, tmA2, tmB2, p);
    } else {
      if (BN == 64) launch_bn<64, kOpF16>(grid, stream, tmA, tmB, tmA2, tmB2, p);
      else          launch_bn<128, kOpF16>(grid, stream, tmA, tmB, tmA2, tmB2, p);
    }
  }
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
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

// A operand of a 1x1 / 3x3, stride 1 / 2 launch: the mode, the output patch and tile grid, and the tensor map of x (the
// top-left h x width rectangle of images xH x xW pixels apart).  es: bytes per element, 2 (fp16), 1 (s8) or 4 (fp32); a K
// block is one 128-byte swizzle row of channels either way.  Shared by odtk_conv2d, odtk_conv2d_s8_ex and odtk_conv2d_f32.
int a_operand(ConvParams &p, CUtensorMap &tmA, const void *x, int n, int h, int width, int cin, int ksize, int stride,
              uint64_t xH, uint64_t xW, bool x_view, const void *tile_tab, int tab_tiles, bool upsample, int es) {
  const CUtensorMapDataType dt = es == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                : es == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
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
    if (upsample) return ODTK_E_UNSUPPORTED;
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

// odtk_conv2d, plus (mode 0 only) a second operand pair added to the same accumulator: y = x * w^T + x2 * w2^T with
// x2 [M, c2in], w2 [cout, c2in] (the projected identity of a bottleneck block).  dgrad: odtk_conv2d_dgrad (the masked
// instance; a tile-table launch may then take a residual, a whole atlas like y).
int conv_run(const odtk_conv_t *d, const void *x2, const void *w2, int c2in, cudaStream_t stream, bool dgrad = false,
             const void *mask = nullptr) {
  if (!d || !d->x || !d->w) return ODTK_E_INVALID;
  if (dgrad && (d->ksize != 3 || d->stride > 1 || d->out_mode != ODTK_OUT_NHWC_F16 || d->relu || d->groups > 1 || d->upsample ||
                d->x_rows > 0 || d->x_width > 0 || d->y_rows > 0 || d->y_width > 0 || d->y_row_off > 0))
    return ODTK_E_UNSUPPORTED;
  if (mask && ((uintptr_t)mask & 3)) return ODTK_E_INVALID;
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
    const int rc = set_sink(p, d->sink, d->cout, d->h, d->width);
    if (rc != ODTK_OK) return rc;
  }
  if (p.out_mode == ODTK_OUT_NHWC_F16 && (p.ldy % 8)) return ODTK_E_INVALID;
  if ((p.residual && (p.ldr & 1)) || (d->upsample && ((d->h & 1) || (d->width & 1)))) return ODTK_E_INVALID;
  const int stride = d->stride > 1 ? d->stride : 1;
  if (stride != 1 && stride != 2) return ODTK_E_UNSUPPORTED;
  // strided views: the input / output may be a rectangle of a larger NHWC buffer (a level of the pyramid atlas)
  const uint64_t xH = d->x_rows > 0 ? (uint64_t)d->x_rows : (uint64_t)d->h, xW = d->x_width > 0 ? (uint64_t)d->x_width : (uint64_t)d->width;
  const bool x_view = xH != (uint64_t)d->h || xW != (uint64_t)d->width;
  const bool y_view = d->y_rows > 0 || d->y_width > 0 || d->y_row_off > 0;
  if ((x_view || y_view || (d->tile_tab && !dgrad)) && (d->ksize != 3 || d->residual || d->upsample)) return ODTK_E_UNSUPPORTED;
  if (y_view && d->out_mode != ODTK_OUT_NHWC_F16) return ODTK_E_UNSUPPORTED;
  if (d->tile_tab && (d->tab_tiles <= 0 || stride != 1 || x_view || y_view)) return ODTK_E_INVALID;
  if (x2 && (d->ksize != 1 || stride != 1 || c2in <= 0 || c2in % 64 || !w2 || (((uintptr_t)x2 | (uintptr_t)w2) & 15))) return ODTK_E_INVALID;
  if (dgrad && p.ldy != d->cout) return ODTK_E_UNSUPPORTED;   // the mask is read with the output's row stride
  p.mask = (const __half *)mask;

  CUtensorMap tmA;
  const int rc = a_operand(p, tmA, d->x, d->n, d->h, d->width, d->cin, d->ksize, stride, xH, xW, x_view, d->tile_tab,
                           d->tab_tiles, d->upsample != nullptr, 2);
  if (rc != ODTK_OK) return rc;
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
  return launch(p, BN, tmA, tmB, tmA2, tmB2, stream, dgrad ? kOpF16Mask : kOpF16);
}

// odtk_conv2d_s8_ex: the same kernel on s8 operands, with the geometry of odtk_conv2d: 1x1 as GEMM rows (mode 0), 3x3 as
// shifted boxes (mode 1) over a dense tensor, a level view of the atlas or the whole atlas with its tile table, stride 2 on
// the parity-split view (mode 3, even sizes) or element-strided boxes (odd sizes, level views).  NHWC s8 outputs may add a
// residual and / or a nearest-upsampled addend, and may land in a level view of an atlas.
int conv_run_s8(const odtk_conv_s8_ex_t *e, cudaStream_t stream) {
  if (!e) return ODTK_E_INVALID;
  const odtk_conv_s8_t *d = &e->base;
  if (!d->x || !d->w || !d->alpha) return ODTK_E_INVALID;
  if (d->out_mode == ODTK_OUT_CANDIDATES ? !d->sink : !d->y) return ODTK_E_INVALID;
  if (d->n <= 0 || d->h <= 0 || d->width <= 0 || d->cin <= 0 || d->cout <= 0) return ODTK_E_INVALID;
  if (d->out_mode != ODTK_OUT_NHWC_S8 && d->out_mode != ODTK_OUT_NCHW_F32 && d->out_mode != ODTK_OUT_NCHW_F32_SIGMOID &&
      d->out_mode != ODTK_OUT_CANDIDATES)
    return ODTK_E_INVALID;
  if ((d->ksize != 1 && d->ksize != 3) || d->cin % 128) return ODTK_E_UNSUPPORTED;   // 128-channel K blocks
  if (d->relu != 0 && d->relu != 1) return ODTK_E_UNSUPPORTED;
  if (d->out_mode == ODTK_OUT_NHWC_S8 && (d->cout % 16)) return ODTK_E_UNSUPPORTED;
  if ((long long)d->n * d->h * d->width >= (1ll << 31)) return ODTK_E_UNSUPPORTED;
  if (((uintptr_t)d->x | (uintptr_t)d->w | (d->out_mode == ODTK_OUT_CANDIDATES ? 0 : (uintptr_t)d->y)) & 15) return ODTK_E_INVALID;
  const int stride = e->stride > 1 ? e->stride : 1;
  if (stride != 1 && stride != 2) return ODTK_E_UNSUPPORTED;
  const uint64_t xH = d->x_rows > 0 ? (uint64_t)d->x_rows : (uint64_t)d->h, xW = d->x_width > 0 ? (uint64_t)d->x_width : (uint64_t)d->width;
  const bool x_view = xH != (uint64_t)d->h || xW != (uint64_t)d->width;
  const bool y_view = e->y_rows > 0 || e->y_width > 0 || e->y_row_off > 0;
  const bool addend = e->residual || e->upsample;
  // addends and output views: NHWC s8 only; views and tile tables: 3x3 without addends (as odtk_conv2d)
  if ((addend || y_view) && d->out_mode != ODTK_OUT_NHWC_S8) return ODTK_E_UNSUPPORTED;
  if ((x_view || y_view || d->tile_tab) && (d->ksize != 3 || addend)) return ODTK_E_UNSUPPORTED;
  if (e->upsample && stride != 1) return ODTK_E_UNSUPPORTED;
  if (d->tile_tab && (d->tab_tiles <= 0 || x_view || y_view || stride != 1)) return ODTK_E_INVALID;
  if ((((uintptr_t)e->residual | (uintptr_t)e->upsample) & 1) || (e->upsample && ((d->h & 1) || (d->width & 1)))) return ODTK_E_INVALID;
  if (!device_ready()) return ODTK_E_CUDA;
  const int sms = odtk_sm_count();
  ConvParams p;
  memset(&p, 0, sizeof p);
  p.N = d->n; p.H = d->h; p.W = d->width; p.Cin = d->cin; p.Cout = d->cout;
  p.kw = d->ksize; p.taps = d->ksize * d->ksize; p.pad = d->ksize / 2;
  p.kblocks_per_tap = d->cin / 128;
  p.row_bytes = 128;
  p.M = (long long)d->n * d->h * d->width;
  p.alpha = d->alpha;
  p.bias = d->bias;
  p.out = d->y;
  p.relu = d->relu;
  p.out_mode = d->out_mode;
  p.ldy = d->cout;
  p.ldr = d->cout;
  p.inv_out_scale = d->inv_out_scale;
  p.res8 = (const int8_t *)e->residual; p.res_scale = e->res_scale;
  p.up8 = (const int8_t *)e->upsample; p.up_scale = e->up_scale;
  p.up_h = d->h / 2; p.up_w = d->width / 2;
  if (p.out_mode == ODTK_OUT_CANDIDATES) {
    const int rc = set_sink(p, d->sink, d->cout, d->h, d->width);
    if (rc != ODTK_OK) return rc;
  }
  CUtensorMap tmA, tmB;
  const int rc = a_operand(p, tmA, d->x, d->n, d->h, d->width, d->cin, d->ksize, stride, xH, xW, x_view, d->tile_tab,
                           d->tab_tiles, e->upsample != nullptr, 1);
  if (rc != ODTK_OK) return rc;
  p.oH = e->y_rows > 0 ? e->y_rows : p.H;
  p.oR = e->y_row_off > 0 ? e->y_row_off : 0;
  p.oW = e->y_width > 0 ? e->y_width : p.W;
  if ((long long)d->n * p.oH * p.oW >= (1ll << 31) || p.oR + p.H > p.oH || p.W > p.oW) return ODTK_E_INVALID;
  // N tile as for odtk_conv2d
  int BN = d->cout <= 64 ? 64 : 128;
  if (BN == 128 && (long long)p.num_m_tiles * ((d->cout + 127) / 128) < sms) BN = 64;
  p.num_n_tiles = (d->cout + BN - 1) / BN;
  set_stages(p, BN);
  {
    const uint64_t K = (uint64_t)p.taps * d->cin;
    uint64_t dims[2] = {K, (uint64_t)d->cout};
    uint64_t str[1] = {K};
    uint32_t box[2] = {128, (uint32_t)BN};
    if (!encode_map(&tmB, d->w, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, nullptr, CU_TENSOR_MAP_DATA_TYPE_UINT8)) return ODTK_E_CUDA;
  }
  return launch(p, BN, tmA, tmB, tmA, tmB, stream, kOpS8);
}

// odtk_conv2d_f32: the kernel on fp32 operands (split TF32).  1x1 / 3x3 with the geometry of odtk_conv2d (dense, atlas views,
// tile tables, stride 2 on either view), plus ksize 7 / stride 2 / cin 3: the ResNet stem over the NHWC4 fp32 image
// [n, h+6, width+8, 4] (mode 2, any h and width).  NHWC fp32 outputs may add an fp32 residual and / or upsample addend and
// may land in a level view of an fp32 atlas.
int conv_run_f32(const odtk_conv_f32_t *d, cudaStream_t stream) {
  if (!d || !d->x || !d->w_hi || !d->w_lo) return ODTK_E_INVALID;
  if (d->out_mode == ODTK_OUT_CANDIDATES ? !d->sink : !d->y) return ODTK_E_INVALID;
  if (d->n <= 0 || d->h <= 0 || d->width <= 0 || d->cin <= 0 || d->cout <= 0) return ODTK_E_INVALID;
  if (d->out_mode != ODTK_OUT_NHWC_F32 && d->out_mode != ODTK_OUT_NCHW_F32 && d->out_mode != ODTK_OUT_NCHW_F32_SIGMOID &&
      d->out_mode != ODTK_OUT_CANDIDATES)
    return ODTK_E_INVALID;
  const int stride = d->stride > 1 ? d->stride : 1;
  const bool stem = d->ksize == 7;
  if (stem ? (d->cin != 3 || stride != 2) : ((d->ksize != 1 && d->ksize != 3) || d->cin % 32)) return ODTK_E_UNSUPPORTED;
  if (stride != 1 && stride != 2) return ODTK_E_UNSUPPORTED;
  if (d->relu != 0 && d->relu != 1) return ODTK_E_UNSUPPORTED;
  if (d->out_mode == ODTK_OUT_NHWC_F32 && (d->cout % 2)) return ODTK_E_UNSUPPORTED;   // float2 stores
  if ((long long)d->n * d->h * d->width >= (1ll << 31)) return ODTK_E_UNSUPPORTED;
  if (((uintptr_t)d->x | (uintptr_t)d->w_hi | (uintptr_t)d->w_lo | (d->out_mode == ODTK_OUT_CANDIDATES ? 0 : (uintptr_t)d->y)) & 15)
    return ODTK_E_INVALID;
  const uint64_t xH = d->x_rows > 0 ? (uint64_t)d->x_rows : (uint64_t)d->h, xW = d->x_width > 0 ? (uint64_t)d->x_width : (uint64_t)d->width;
  const bool x_view = xH != (uint64_t)d->h || xW != (uint64_t)d->width;
  const bool y_view = d->y_rows > 0 || d->y_width > 0 || d->y_row_off > 0;
  const bool addend = d->residual || d->upsample;
  // as odtk_conv2d_s8_ex: addends and output views need NHWC fp32, views and tile tables are 3x3 without addends
  if ((addend || y_view) && d->out_mode != ODTK_OUT_NHWC_F32) return ODTK_E_UNSUPPORTED;
  if ((x_view || y_view || d->tile_tab) && (d->ksize != 3 || addend)) return ODTK_E_UNSUPPORTED;
  if (stem && addend) return ODTK_E_UNSUPPORTED;
  if (d->upsample && stride != 1) return ODTK_E_UNSUPPORTED;
  if (d->tile_tab && (d->tab_tiles <= 0 || x_view || y_view || stride != 1)) return ODTK_E_INVALID;
  if ((((uintptr_t)d->residual | (uintptr_t)d->upsample) & 7) || (d->upsample && ((d->h & 1) || (d->width & 1)))) return ODTK_E_INVALID;
  if (!device_ready()) return ODTK_E_CUDA;
  const int sms = odtk_sm_count();
  ConvParams p;
  memset(&p, 0, sizeof p);
  p.N = d->n; p.H = d->h; p.W = d->width; p.Cin = d->cin; p.Cout = d->cout;
  p.row_bytes = 128;
  p.M = (long long)d->n * d->h * d->width;
  p.bias = d->bias;
  p.out = d->y;
  p.relu = d->relu;
  p.out_mode = d->out_mode;
  p.ldy = d->ldy > 0 ? d->ldy : d->cout;
  p.ldr = d->ldr > 0 ? d->ldr : d->cout;
  p.res32 = (const float *)d->residual;
  p.up32 = (const float *)d->upsample;
  p.up_h = d->h / 2; p.up_w = d->width / 2;
  if ((p.out_mode == ODTK_OUT_NHWC_F32 && (p.ldy & 1)) || (p.res32 && (p.ldr & 1))) return ODTK_E_INVALID;   // float2 accesses
  if (p.out_mode == ODTK_OUT_CANDIDATES) {
    const int rc = set_sink(p, d->sink, d->cout, d->h, d->width);
    if (rc != ODTK_OK) return rc;
  }
  CUtensorMap tmA, tmB, tmB2;
  uint64_t K;
  if (stem) {
    // NHWC4 window rows as in odtk_stem_conv, in fp32: 8 pixels x 4 channels = 32 floats = one 128-byte swizzle row
    const int OH = (d->h - 1) / 2 + 1, OW = (d->width - 1) / 2 + 1;
    const uint64_t HP = (uint64_t)d->h + 6, WP = (uint64_t)d->width + 8;
    p.mode = 2;
    p.H = OH; p.W = OW; p.Cin = 4;
    p.kw = 1; p.taps = 7; p.pad = 0; p.kblocks_per_tap = 1;
    p.M = (long long)d->n * OH * OW;
    choose_patch(OH, OW, p.TH, p.TW);
    p.tiles_h = (OH + p.TH - 1) / p.TH;
    p.tiles_w = (OW + p.TW - 1) / p.TW;
    p.num_m_tiles = d->n * p.tiles_h * p.tiles_w;
    uint64_t dims[5] = {32, (uint64_t)OW, 7, (uint64_t)OH, (uint64_t)d->n};
    uint64_t str[4] = {32, WP * 16, WP * 32, HP * WP * 16};
    uint32_t box[5] = {32, (uint32_t)p.TW, 1, (uint32_t)p.TH, 1};
    if (!encode_map(&tmA, d->x, 5, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, nullptr, CU_TENSOR_MAP_DATA_TYPE_FLOAT32))
      return ODTK_E_UNSUPPORTED;
    K = 224;
  } else {
    p.kw = d->ksize; p.taps = d->ksize * d->ksize; p.pad = d->ksize / 2;
    p.kblocks_per_tap = d->cin / 32;
    const int rc = a_operand(p, tmA, d->x, d->n, d->h, d->width, d->cin, d->ksize, stride, xH, xW, x_view, d->tile_tab,
                             d->tab_tiles, d->upsample != nullptr, 4);
    if (rc != ODTK_OK) return rc;
    K = (uint64_t)p.taps * d->cin;
  }
  p.oH = d->y_rows > 0 ? d->y_rows : p.H;
  p.oR = d->y_row_off > 0 ? d->y_row_off : 0;
  p.oW = d->y_width > 0 ? d->y_width : p.W;
  if ((long long)d->n * p.oH * p.oW >= (1ll << 31) || p.oR + p.H > p.oH || p.W > p.oW) return ODTK_E_INVALID;
  // N tile as for odtk_conv2d
  int BN = d->cout <= 64 ? 64 : 128;
  if (BN == 128 && (long long)p.num_m_tiles * ((d->cout + 127) / 128) < sms) BN = 64;
  p.num_n_tiles = (d->cout + BN - 1) / BN;
  set_stages(p, BN, kOpTF32x3);
  {
    uint64_t dims[2] = {K, (uint64_t)d->cout};
    uint64_t str[1] = {K * 4};
    uint32_t box[2] = {32, (uint32_t)BN};
    if (!encode_map(&tmB, d->w_hi, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, nullptr, CU_TENSOR_MAP_DATA_TYPE_FLOAT32) ||
        !encode_map(&tmB2, d->w_lo, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, nullptr, CU_TENSOR_MAP_DATA_TYPE_FLOAT32))
      return ODTK_E_CUDA;
  }
  return launch(p, BN, tmA, tmB, tmA, tmB2, stream, kOpTF32x3);
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

extern "C" int odtk_conv2d_dgrad(const odtk_conv_dgrad_t *d, odtk_stream_t stream_) {
  if (!d) return ODTK_E_INVALID;
  return conv_run(&d->base, nullptr, nullptr, 0, (cudaStream_t)stream_, true, d->mask);
}

extern "C" int odtk_conv2d_s8(const odtk_conv_s8_t *d, odtk_stream_t stream_) {
  if (!d) return ODTK_E_INVALID;
  odtk_conv_s8_ex_t e;
  memset(&e, 0, sizeof e);
  e.base = *d;
  return conv_run_s8(&e, (cudaStream_t)stream_);
}

extern "C" int odtk_conv2d_s8_ex(const odtk_conv_s8_ex_t *e, odtk_stream_t stream_) {
  return conv_run_s8(e, (cudaStream_t)stream_);
}

extern "C" int odtk_conv2d_f32(const odtk_conv_f32_t *d, odtk_stream_t stream_) {
  return conv_run_f32(d, (cudaStream_t)stream_);
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
