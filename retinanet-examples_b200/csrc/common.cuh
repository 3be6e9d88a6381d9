// common.cuh -- small device/host helpers shared by the sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/odtk_b200.h"

#define ODTK_ALIGN 256  // every workspace sub-buffer is 256-B aligned (reference: utils.h:28)

static inline size_t odtk_align_up(size_t x) { return (x + ODTK_ALIGN - 1) / ODTK_ALIGN * ODTK_ALIGN; }

// SM budget of the calling host thread's launches (0 = the whole device): persistent kernels size their grids from
// odtk_sm_count(), so two streams given complementary budgets run their kernels side by side on disjoint SMs
// (odtk_set_sm_budget, include/odtk_b200.h).  Defined in version.cu.
extern int g_odtk_sm_budget;
// 1 (default): the fp16 NHWC epilogues store their tiles with TMA from shared memory; 0: direct stores from the registers
// (odtk_set_tma_store).  Defined in version.cu.
extern int g_odtk_tma_store;

// SM count of the CURRENT device (cached per device ordinal; grids are sized from it, never from a constant)
static inline int odtk_sm_count_device() {
  static int cache[64];
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (dev >= 0 && dev < 64 && cache[dev] > 0) return cache[dev];
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) return 132;
  if (dev >= 0 && dev < 64) cache[dev] = n;
  return n;
}
// ODTK_PDL=0 turns programmatic dependent launch off (A/B); default on
static inline bool odtk_pdl_on() {
  static int on = -1;
  if (on < 0) { const char *e = getenv("ODTK_PDL"); on = e ? atoi(e) : 1; }
  return on != 0;
}
static inline int odtk_sm_count() {
  const int n = odtk_sm_count_device();
  return (g_odtk_sm_budget > 0 && g_odtk_sm_budget < n) ? g_odtk_sm_budget : n;
}

// Monotone float -> uint32 key; larger key == larger float.  This is the transform
// cub::DeviceRadixSort applies to float keys, so "descending, stable" in the
// reference (decode.cu:111, nms.cu:135) == descending on (key, ~position).
__host__ __device__ __forceinline__ uint32_t odtk_float_key(float f) {
#ifdef __CUDA_ARCH__
  uint32_t b = __float_as_uint(f);
#else
  uint32_t b;
  memcpy(&b, &f, 4);
#endif
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float odtk_key_float(uint32_t k) {
  uint32_t b = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  return __uint_as_float(b);
}

__device__ __forceinline__ float4 odtk_ld_stream_f4(const float4 *p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ float odtk_ld_stream_f1(const float *p) {
  float r;
  asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(r) : "l"(p));
  return r;
}

// In-place bitonic sort, DESCENDING, of P (power of two) 64-bit keys in shared memory by
// the whole CTA.  Keys are unique (composite of value and position) so the unstable
// network reproduces the reference's stable radix order exactly.
__device__ __forceinline__ void odtk_bitonic_desc_u64(unsigned long long *s, int P) {
  const int T = blockDim.x, t = threadIdx.x;
  for (int k = 2; k <= P; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = t; i < (P >> 1); i += T) {
        int lo = ((i & ~(j - 1)) << 1) | (i & (j - 1));
        int hi = lo | j;
        bool desc = ((lo & k) == 0);
        unsigned long long a = s[lo], b = s[hi];
        if ((a < b) == desc) { s[lo] = b; s[hi] = a; }
      }
      __syncthreads();
    }
  }
}

#define ODTK_HIST_BINS 2048
// Histogram suffix scan by the whole CTA: highest bin b* with sum_{bin >= b*} >= top_n, and
// that sum.  hist has ODTK_HIST_BINS entries in shared memory; requires sum(hist) >= top_n.
// scratch: s_w[32], s_res[2].
__device__ __forceinline__ void odtk_find_bstar(const uint32_t *shist, int top_n, int *s_w, int *s_res,
                                           int &bstar, int &nsel) {
  const int T = blockDim.x, t = threadIdx.x, lane = t & 31, warp = t >> 5, nwarp = T >> 5;
  const int per = ODTK_HIST_BINS / T;  // bins per thread, descending order
  int own = 0;
  for (int q = 0; q < per; q++) own += (int)shist[ODTK_HIST_BINS - 1 - (t * per + q)];
  int incl = own;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) s_w[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int w = lane < nwarp ? s_w[lane] : 0, wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int v = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi += v;
    }
    s_w[lane] = wi - w;  // exclusive
  }
  __syncthreads();
  incl += s_w[warp];
  int acc = incl - own;
  if (acc < top_n && incl >= top_n) {
    for (int q = 0; q < per; q++) {
      int b = ODTK_HIST_BINS - 1 - (t * per + q);
      acc += (int)shist[b];
      if (acc >= top_n) { s_res[0] = b; s_res[1] = acc; break; }
    }
  }
  __syncthreads();
  bstar = s_res[0];
  nsel = s_res[1];
}

// One channel of odtk's input normalisation (reference odtk/data.py:118-121), same operation order as the reference:
// float(u8) / 255, then - mean, then / std, fp32.  Shared by the preprocess kernels (layers.cu) and the training
// augmentation (augment.cu).
__device__ __forceinline__ float normalize_u8(unsigned v, float m, float s) { return ((float)v / 255.0f - m) / s; }

__host__ __device__ __forceinline__ int odtk_next_pow2(int x) {
  int p = 32;
  while (p < x) p <<= 1;
  return p;
}
