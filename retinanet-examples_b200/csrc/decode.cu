// decode.cu -- score filter + exact top-n + anchor box decode for sm_90a.
//
// Replaces odtk::cuda::decode / decode_rotate (reference csrc/cuda/decode.cu:44-171,
// decode_rotate.cu:42-179), which run, PER IMAGE and PER LEVEL with a host sync in between,
// thrust::transform -> cub::DeviceSelect -> D2H count -> gather -> cub radix sort ->
// thrust::transform.  Here ALL pyramid levels of the whole batch are three launches and no
// host sync (the per-level reference entry points are the one-level special case):
//
//   K1 score_filter_kernel   HBM-bound streaming pass over every [B, A*C*H*W] fp32 score map
//                            (128-bit L1-bypassing loads, register double-buffered so >= 4
//                            are always in flight per lane).  Survivors (score > thresh,
//                            ~0.5 %) are staged per warp in shared memory and flushed with
//                            ONE global atomic per >= 32 of them into a per-(level,image)
//                            candidate list (score key, flat index); a 2048-bin histogram of
//                            the score keys is accumulated on the side.
//   K2 gather_top_kernel     many CTAs per (level,image): the histogram gives the bin b* that
//                            holds the top_n-th score; candidates in bins >= b* (about top_n
//                            of them) are compacted into a short list (block-aggregated
//                            atomics, batched loads).
//   K3 select_decode_kernel  one CTA per (level,image): bitonic network on the unique
//                            composite key (score key, ~flat index) == the reference's stable
//                            order; every kept index is decoded in fp32, IEEE, no FMA
//                            contraction, same operation order as decode.cu:133-156, and
//                            written straight into the concatenated [B, L*top_n] outputs.
//
// Exactness never depends on the data: if a candidate list overflows, or a histogram bin holds
// more ties than the sort capacity, K3 falls back to an 8-pass radix select on the composite
// key (slow, exact).  Compile with -fmad=false (see Makefile).
#include <stdlib.h>

#include <memory>

#include "common.cuh"
#include "prof.cuh"

namespace {

constexpr int kHistBins = ODTK_HIST_BINS;
constexpr int kSortCap = ODTK_MAX_TOP_N;  // 4096 keys of 8 B = 32 KB shared
constexpr int kMaxAnchors = 32;           // anchor tables travel as kernel parameters
constexpr int kMaxLevels = ODTK_MAX_LEVELS;
constexpr int kFilterThreads = 256;
constexpr int kWarpsPerBlock = kFilterThreads / 32;
constexpr int kTile = 512;                 // elements per warp per iteration (4 x float4 x 32)
constexpr int kStage = 32 + kTile;         // per-warp staging entries
constexpr int kGatherSlices = 16;
constexpr int kGatherThreads = 256;

struct LevelDesc {
  const float *scores;  // [B, n]
  const float *deltas;  // [B, A*NBOX*H*W]
  long long n;          // A*C*H*W
  long long cand_off;   // first candidate entry of this level (entries), cap entries per image
  long long cap;
  int height, width, scale, out_offset;
  int blk_begin, blk_per_img;  // filter-kernel block range of this level
  int vec;                     // 128-bit loads allowed
  int pad;
};

struct DecodeParams {
  LevelDesc lv[kMaxLevels];
  float anchors[kMaxLevels][4 * kMaxAnchors];
  int num_levels, batch, num_anchors, num_classes, has_anchors, top_n, shift;
  float thresh;
  uint32_t key_thresh;
  int *counts;                 // [L*B]
  uint32_t *hist;              // [L*B, kHistBins]
  uint2 *cand;                 // per level: [B, cap_l]  (x = score key, y = flat index)
  int *selcount;               // [L*B]
  unsigned long long *sel;     // [L*B, kSortCap] composites gathered by K2
  float *out_scores, *out_boxes, *out_classes;
  long long out_stride;
};

__device__ __forceinline__ int hist_bin(uint32_t key, uint32_t key_thresh, int shift) {
  uint32_t d = (key - key_thresh) >> shift;
  return d < (uint32_t)(kHistBins - 1) ? (int)d : (kHistBins - 1);
}

// ------------------------------------------------------------------------------------
// K1: streaming filter.  grid = sum over levels of B * blk_per_img, block = 256.  V = 16-byte vectors per lane per
// tile (4: one 2 KB tile per warp in flight behind the one being filtered; 8: 4 KB -- more bytes in flight per SM).
template <int V>
__global__ void __launch_bounds__(kFilterThreads) score_filter_kernel(const __grid_constant__ DecodeParams p) {
  constexpr int kTileV = V * 128;            // elements per warp per iteration
  __shared__ uint2 stage[kWarpsPerBlock][kStage];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int level = 0;
#pragma unroll 1
  for (int l = 1; l < p.num_levels; l++)
    if ((int)blockIdx.x >= p.lv[l].blk_begin) level = l;
  const LevelDesc &L = p.lv[level];
  const int rel = (int)blockIdx.x - L.blk_begin;
  const int img = rel / L.blk_per_img, blk = rel - img * L.blk_per_img;
  const int slot = level * p.batch + img;
  const long long n = L.n;
  const float thresh = p.thresh;
  const float *s = L.scores + (long long)img * n;
  uint2 *cand = p.cand + L.cand_off + (long long)img * L.cap;
  const long long cap = L.cap;
  uint32_t *hist = p.hist + (long long)slot * kHistBins;
  uint2 *st = stage[warp];
  const unsigned lt_mask = (1u << lane) - 1u;
  int nstaged = 0;  // warp-uniform

  auto flush = [&]() {
    if (nstaged > 0) {
      __syncwarp();
      int base = 0;
      if (lane == 0) base = atomicAdd(p.counts + slot, nstaged);
      base = __shfl_sync(0xffffffffu, base, 0);
      for (int j = lane; j < nstaged; j += 32) {
        uint2 c = st[j];
        long long dst = (long long)base + j;
        if (dst < cap) cand[dst] = c;
        atomicAdd(hist + hist_bin(c.x, p.key_thresh, p.shift), 1u);
      }
      __syncwarp();
      nstaged = 0;
    }
  };
  auto push = [&](bool pass, float v, long long idx) {
    unsigned m = __ballot_sync(0xffffffffu, pass);
    if (m) {
      if (pass) st[nstaged + __popc(m & lt_mask)] = make_uint2(odtk_float_key(v), (uint32_t)idx);
      nstaged += __popc(m);
    }
  };

  const long long ntiles = (n + kTileV - 1) / kTileV;
  const long long wstride = (long long)L.blk_per_img * kWarpsPerBlock;
  long long t = (long long)blk * kWarpsPerBlock + warp;
  if (L.vec) {
    auto load_tile = [&](long long tt, float4 (&v)[V]) {
#pragma unroll
      for (int j = 0; j < V; j++) {
        long long e = tt * kTileV + (long long)(j * 32 + lane) * 4;
        // out-of-range lanes get `thresh`: thresh > thresh is false, so they never pass
        v[j] = (e < n) ? odtk_ld_stream_f4(reinterpret_cast<const float4 *>(s + e))
                       : make_float4(thresh, thresh, thresh, thresh);
      }
    };
    float4 cur[V], nxt[V];
    if (t < ntiles) load_tile(t, cur);
    for (; t < ntiles; t += wstride) {
      const bool more = (t + wstride) < ntiles;
      if (more) load_tile(t + wstride, nxt);
#pragma unroll
      for (int j = 0; j < V; j++) {
        long long e = t * kTileV + (long long)(j * 32 + lane) * 4;
        push(cur[j].x > thresh, cur[j].x, e + 0);
        push(cur[j].y > thresh, cur[j].y, e + 1);
        push(cur[j].z > thresh, cur[j].z, e + 2);
        push(cur[j].w > thresh, cur[j].w, e + 3);
        if ((j & 3) == 3 && nstaged >= 32) flush();      // the staging buffer holds 32 + 512 entries
      }
      if (more) {
#pragma unroll
        for (int j = 0; j < V; j++) cur[j] = nxt[j];
      }
    }
  } else {
    for (; t < ntiles; t += wstride) {
      const long long e0 = t * kTileV;
      float v[16];
      for (int h = 0; h < V / 4; h++) {
#pragma unroll
        for (int j = 0; j < 16; j++) {
          long long e = e0 + h * 512 + j * 32 + lane;
          v[j] = (e < n) ? odtk_ld_stream_f1(s + e) : thresh;
        }
#pragma unroll
        for (int j = 0; j < 16; j++) push(v[j] > thresh, v[j], e0 + h * 512 + j * 32 + lane);
        if (nstaged >= 32) flush();
      }
    }
  }
  flush();
}

// K1, bulk-copy variant: same filter, but the scores travel HBM -> shared memory as cp.async.bulk chunks through a ring
// of mbarrier-guarded stages (thread 0 keeps kBulkStages - 1 chunks in flight), so the bytes in flight per SM are set by
// the ring (6 x 8 KB per CTA), not by how many registers the compiler can spare for prefetched vectors.
constexpr int kBulkElems = 2048;                    // floats per chunk: 8 KB = 256 threads x 2 float4
constexpr int kBulkStages = 6;
__global__ void __launch_bounds__(kFilterThreads) score_filter_bulk_kernel(const __grid_constant__ DecodeParams p) {
  extern __shared__ __align__(128) unsigned char bulk_dyn[];       // the ring: kBulkStages x 8 KB (dynamic: static + ring > 48 KB)
  float (*ring)[kBulkElems] = reinterpret_cast<float (*)[kBulkElems]>(bulk_dyn);
  __shared__ uint2 stage[kWarpsPerBlock][kStage];
  __shared__ __align__(8) unsigned long long full[kBulkStages], empty[kBulkStages];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int level = 0;
#pragma unroll 1
  for (int l = 1; l < p.num_levels; l++)
    if ((int)blockIdx.x >= p.lv[l].blk_begin) level = l;
  const LevelDesc &L = p.lv[level];
  const int rel = (int)blockIdx.x - L.blk_begin;
  const int img = rel / L.blk_per_img, blk = rel - img * L.blk_per_img;
  const int slot = level * p.batch + img;
  const long long n = L.n;
  const float thresh = p.thresh;
  const float *s = L.scores + (long long)img * n;
  uint2 *cand = p.cand + L.cand_off + (long long)img * L.cap;
  const long long cap = L.cap;
  uint32_t *hist = p.hist + (long long)slot * kHistBins;
  uint2 *st = stage[warp];
  const unsigned lt_mask = (1u << lane) - 1u;
  int nstaged = 0;  // warp-uniform

  auto sa = [](const void *ptr) { return (uint32_t)__cvta_generic_to_shared(ptr); };
  if (threadIdx.x == 0) {
    for (int i = 0; i < kBulkStages; i++) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(sa(&full[i])), "r"(1));
      asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(sa(&empty[i])), "r"(kWarpsPerBlock));
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  auto wait = [&](unsigned long long *bar, uint32_t parity) {
    uint32_t done;
    do {
      asm volatile("{\n\t.reg .pred q;\n\tmbarrier.try_wait.parity.shared::cta.b64 q, [%1], %2;\n\tselp.u32 %0, 1, 0, q;\n\t}"
                   : "=r"(done) : "r"(sa(bar)), "r"(parity) : "memory");
    } while (!done);
  };
  auto flush = [&]() {
    if (nstaged > 0) {
      __syncwarp();
      int base = 0;
      if (lane == 0) base = atomicAdd(p.counts + slot, nstaged);
      base = __shfl_sync(0xffffffffu, base, 0);
      for (int j = lane; j < nstaged; j += 32) {
        uint2 c = st[j];
        long long dst = (long long)base + j;
        if (dst < cap) cand[dst] = c;
        atomicAdd(hist + hist_bin(c.x, p.key_thresh, p.shift), 1u);
      }
      __syncwarp();
      nstaged = 0;
    }
  };
  auto push = [&](bool pass, float v, long long idx) {
    unsigned m = __ballot_sync(0xffffffffu, pass);
    if (m) {
      if (pass) st[nstaged + __popc(m & lt_mask)] = make_uint2(odtk_float_key(v), (uint32_t)idx);
      nstaged += __popc(m);
    }
  };

  // chunks of this (level, image) owned by this block: blk, blk + blk_per_img, ...
  const long long nchunks = (n + kBulkElems - 1) / kBulkElems;
  const long long mine = blk < nchunks ? (nchunks - blk + L.blk_per_img - 1) / L.blk_per_img : 0;
  auto issue = [&](long long k) {        // thread 0: start the copy of this block's k-th chunk into stage k % kBulkStages
    const int sidx = (int)(k % kBulkStages);
    const long long e0 = ((long long)blk + k * L.blk_per_img) * kBulkElems;
    const long long left = n - e0;
    const uint32_t bytes = (uint32_t)((left >= kBulkElems ? kBulkElems : (left & ~3ll)) * 4);   // whole 16-byte units only
    if (k >= kBulkStages) wait(&empty[sidx], (uint32_t)(((k / kBulkStages) - 1) & 1));
    if (bytes) {
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(sa(&full[sidx])), "r"(bytes) : "memory");
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                   ::"r"(sa(&ring[sidx][0])), "l"(s + e0), "r"(bytes), "r"(sa(&full[sidx])) : "memory");
    } else {
      asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(sa(&full[sidx])) : "memory");
    }
  };
  if (threadIdx.x == 0)
    for (long long k = 0; k < mine && k < kBulkStages - 1; k++) issue(k);
  for (long long k = 0; k < mine; k++) {
    const int sidx = (int)(k % kBulkStages);
    if (threadIdx.x == 0 && k + kBulkStages - 1 < mine) issue(k + kBulkStages - 1);
    wait(&full[sidx], (uint32_t)((k / kBulkStages) & 1));
    const long long e0 = ((long long)blk + k * L.blk_per_img) * kBulkElems;
    const long long left = n - e0;
    const long long vec_elems = left >= kBulkElems ? kBulkElems : (left & ~3ll);
    float4 v[2];
#pragma unroll
    for (int j = 0; j < 2; j++) {
      const int off = (j * kFilterThreads + threadIdx.x) * 4;
      if (off < vec_elems) v[j] = *reinterpret_cast<const float4 *>(&ring[sidx][off]);
      else {   // tail of the level (fewer than 4 floats past the bulk copy) and the lanes beyond it
        v[j].x = (off + 0 < left) ? odtk_ld_stream_f1(s + e0 + off + 0) : thresh;
        v[j].y = (off + 1 < left) ? odtk_ld_stream_f1(s + e0 + off + 1) : thresh;
        v[j].z = (off + 2 < left) ? odtk_ld_stream_f1(s + e0 + off + 2) : thresh;
        v[j].w = (off + 3 < left) ? odtk_ld_stream_f1(s + e0 + off + 3) : thresh;
      }
    }
    __syncwarp();
    if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(sa(&empty[sidx])) : "memory");   // stage read
#pragma unroll
    for (int j = 0; j < 2; j++) {
      const long long e = e0 + (long long)(j * kFilterThreads + threadIdx.x) * 4;
      push(v[j].x > thresh, v[j].x, e + 0);
      push(v[j].y > thresh, v[j].y, e + 1);
      push(v[j].z > thresh, v[j].z, e + 2);
      push(v[j].w > thresh, v[j].w, e + 3);
    }
    if (nstaged >= 32) flush();
  }
  flush();
}

// K2: grid = (kGatherSlices, L*B), block = 256.
__global__ void __launch_bounds__(kGatherThreads) gather_top_kernel(const __grid_constant__ DecodeParams p) {
  __shared__ uint32_t shist[kHistBins];
  __shared__ int s_w[32];
  __shared__ int s_res[2];
  __shared__ int s_base;
  const int slot = blockIdx.y, level = slot / p.batch, img = slot - level * p.batch;
  const LevelDesc &L = p.lv[level];
  const int total = p.counts[slot];
  if (total <= p.top_n || (long long)total > L.cap) return;  // index mode / overflow: K3 handles it
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const uint32_t *hist = p.hist + (long long)slot * kHistBins;
  for (int i = t; i < kHistBins; i += kGatherThreads) shist[i] = hist[i];
  __syncthreads();
  int bstar, nsel;
  odtk_find_bstar(shist, p.top_n, s_w, s_res, bstar, nsel);
  if (nsel > kSortCap) return;  // tie bin too large: K3 runs the exact radix select
  const uint2 *cand = p.cand + L.cand_off + (long long)img * L.cap;
  unsigned long long *sel = p.sel + (long long)slot * kSortCap;
  const int per_slice = (total + kGatherSlices - 1) / kGatherSlices;
  const int j0 = blockIdx.x * per_slice;
  const int j1 = min(total, j0 + per_slice);
  constexpr int U = 8;
  for (int jb = j0; jb < j1; jb += kGatherThreads * U) {
    uint2 c[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      int j = jb + u * kGatherThreads + t;
      c[u] = (j < j1) ? cand[j] : make_uint2(0u, 0u);
    }
    bool hit[U];
    int mine = 0;
#pragma unroll
    for (int u = 0; u < U; u++) {
      int j = jb + u * kGatherThreads + t;
      hit[u] = (j < j1) && hist_bin(c[u].x, p.key_thresh, p.shift) >= bstar;
      mine += hit[u];
    }
    // block-aggregated reservation: warp scan -> one global atomic per CTA per batch
    int incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    __syncthreads();
    if (lane == 31) s_w[warp] = incl;
    __syncthreads();
    if (t == 0) {
      int acc = 0;
      for (int w = 0; w < kGatherThreads / 32; w++) { int v = s_w[w]; s_w[w] = acc; acc += v; }
      s_base = acc ? atomicAdd(p.selcount + slot, acc) : 0;
    }
    __syncthreads();
    int pos = s_base + s_w[warp] + incl - mine;
#pragma unroll
    for (int u = 0; u < U; u++)
      if (hit[u]) { sel[pos++] = ((unsigned long long)c[u].x << 32) | (uint32_t)(~c[u].y); }
  }
}

// ------------------------------------------------------------------------------------
// Block-wide radix select (8 passes x 8 bits, MSB first) of the `need`-th largest unique
// 64-bit composite among the items produced by src(j) for j in [0, total).  Returns the
// smallest composite that belongs to the top `need`.  Exact for any input; only used when
// the fast path cannot be (candidate overflow / a tie bin larger than kSortCap).
template <class Src>
__device__ unsigned long long radix_select_kth(Src src, long long total, int need, uint32_t *sh256,
                                               int *sh_misc) {
  unsigned long long prefix = 0;
  for (int pass = 7; pass >= 0; pass--) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) sh256[i] = 0;
    __syncthreads();
    const int sh = pass * 8;
    for (long long j = threadIdx.x; j < total; j += blockDim.x) {
      unsigned long long c;
      if (src(j, c)) {
        bool match = (pass == 7) ? true : ((c >> (sh + 8)) == prefix);
        if (match) atomicAdd(&sh256[(c >> sh) & 255], 1u);
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int acc = 0, d = 255;
      for (; d > 0; d--) {
        if (acc + (int)sh256[d] >= need) break;
        acc += (int)sh256[d];
      }
      sh_misc[0] = d;
      sh_misc[1] = need - acc;  // how many are still needed inside digit d
      sh_misc[2] = (int)sh256[d];
    }
    __syncthreads();
    prefix = (prefix << 8) | (unsigned long long)sh_misc[0];
    need = sh_misc[1];
    const int in_bucket = sh_misc[2];
    __syncthreads();
    if (in_bucket == need) return prefix << sh;  // the whole bucket is selected
  }
  return prefix;
}

// K3: grid = L*B, block = 1024.
template <int NBOX>
__global__ void __launch_bounds__(1024) select_decode_kernel(const __grid_constant__ DecodeParams p) {
  __shared__ unsigned long long skey[kSortCap];
  __shared__ uint32_t shist[kHistBins];
  __shared__ int s_w[32];
  __shared__ int s_misc[8];
  const int t = threadIdx.x;
  const int slot = blockIdx.x, level = slot / p.batch, img = slot - level * p.batch;
  const LevelDesc &L = p.lv[level];
  const long long total = p.counts[slot];
  const uint2 *cand = p.cand + L.cand_off + (long long)img * L.cap;
  const float *dense = L.scores + (long long)img * L.n;

  // composite in SCORE mode: (score key << 32) | ~index      -> score desc, index asc
  // composite in INDEX mode: (~index << 32) | score key       -> index asc
  const bool index_mode = total <= (long long)p.top_n;
  int nsel = 0;
  if (t == 0) s_misc[3] = 0;
  __syncthreads();

  if (index_mode) {
    nsel = (int)total;  // total <= top_n <= cap
    for (int j = t; j < nsel; j += blockDim.x) {
      uint2 c = cand[j];
      skey[j] = ((unsigned long long)(~c.y) << 32) | c.x;
    }
  } else {
    bool slow = total > L.cap;
    if (!slow) {
      const uint32_t *hist = p.hist + (long long)slot * kHistBins;
      for (int i = t; i < kHistBins; i += blockDim.x) shist[i] = hist[i];
      __syncthreads();
      int bstar;
      odtk_find_bstar(shist, p.top_n, s_w, s_misc, bstar, nsel);
      if (nsel > kSortCap) slow = true;
    }
    if (!slow) {
      // K2 gathered exactly the candidates of bins >= b*
      const unsigned long long *sel = p.sel + (long long)slot * kSortCap;
      for (int j = t; j < nsel; j += blockDim.x) skey[j] = sel[j];
    } else {
      unsigned long long kth;
      const float thresh = p.thresh;
      __syncthreads();
      if (total > L.cap) {  // candidate list overflowed: go back to the dense scores
        auto src = [=](long long j, unsigned long long &c) {
          float v = dense[j];
          if (!(v > thresh)) return false;
          c = ((unsigned long long)odtk_float_key(v) << 32) | (uint32_t)(~(uint32_t)j);
          return true;
        };
        kth = radix_select_kth(src, L.n, p.top_n, shist, s_misc);
        for (long long j = t; j < L.n; j += blockDim.x) {
          unsigned long long c;
          if (src(j, c) && c >= kth) skey[atomicAdd(&s_misc[3], 1)] = c;
        }
      } else {
        auto src = [=](long long j, unsigned long long &c) {
          uint2 v = cand[j];
          c = ((unsigned long long)v.x << 32) | (uint32_t)(~v.y);
          return true;
        };
        kth = radix_select_kth(src, total, p.top_n, shist, s_misc);
        for (long long j = t; j < total; j += blockDim.x) {
          unsigned long long c;
          if (src(j, c) && c >= kth) skey[atomicAdd(&s_misc[3], 1)] = c;
        }
      }
      __syncthreads();
      nsel = s_misc[3];  // == top_n
    }
  }

  // order the selected keys
  const int P = odtk_next_pow2(nsel);
  for (int j = nsel + t; j < P; j += blockDim.x) skey[j] = 0ull;
  __syncthreads();
  odtk_bitonic_desc_u64(skey, P);

  // decode: reference decode.cu:119-159 / decode_rotate.cu:115-166
  const int n_out = nsel < p.top_n ? nsel : p.top_n;
  const int H = L.height, W = L.width, A = p.num_anchors, C = p.num_classes;
  const float *d = L.deltas + (long long)img * ((long long)A * NBOX * H * W);
  const long long obase = (long long)img * p.out_stride + L.out_offset;
  float *os = p.out_scores + obase;
  float *ob = p.out_boxes + obase * NBOX;
  float *oc = p.out_classes + obase;
  const float *anchors = p.anchors[level];
  for (int k = t; k < p.top_n; k += blockDim.x) {
    if (k < n_out) {
      unsigned long long c = skey[k];
      uint32_t key = index_mode ? (uint32_t)c : (uint32_t)(c >> 32);
      int i = (int)(index_mode ? ~(uint32_t)(c >> 32) : ~(uint32_t)c);
      int x = i % W;
      int y = (i / W) % H;
      int a = (i / C / H / W) % A;
      int cls = (i / H / W) % C;
      float box[NBOX];
#pragma unroll
      for (int q = 0; q < NBOX; q++) box[q] = d[((long long)(a * NBOX + q) * H + y) * W + x];
      if (p.has_anchors) {
        float fx = (float)((long long)x * L.scale);
        float fy = (float)((long long)y * L.scale);
        const float *an = anchors + 4 * a;
        float x1 = fx + an[0];
        float y1 = fy + an[1];
        float x2 = fx + an[2];
        float y2 = fy + an[3];
        float w = x2 - x1 + 1.0f;
        float h = y2 - y1 + 1.0f;
        float pred_ctr_x = box[0] * w + x1 + 0.5f * w;
        float pred_ctr_y = box[1] * h + y1 + 0.5f * h;
        float pred_w = expf(box[2]) * w;
        float pred_h = expf(box[3]) * h;
        box[0] = fmaxf(0.0f, pred_ctr_x - 0.5f * pred_w);
        box[1] = fmaxf(0.0f, pred_ctr_y - 0.5f * pred_h);
        box[2] = fminf(pred_ctr_x + 0.5f * pred_w - 1.0f, (float)((long long)W * L.scale) - 1.0f);
        box[3] = fminf(pred_ctr_y + 0.5f * pred_h - 1.0f, (float)((long long)H * L.scale) - 1.0f);
      }
      os[k] = odtk_key_float(key);
#pragma unroll
      for (int q = 0; q < NBOX; q++) ob[(long long)k * NBOX + q] = box[q];
      oc[k] = (float)cls;
    } else {
      os[k] = 0.0f;
#pragma unroll
      for (int q = 0; q < NBOX; q++) ob[(long long)k * NBOX + q] = 0.0f;
      oc[k] = 0.0f;
    }
  }
}

// workspace layout: counts | selcount | hist | sel | cand(level 0) | cand(level 1) ...
struct DecodeWs {
  size_t counts_off, selcount_off, hist_off, zero_bytes, sel_off, cand_off, total;
};

long long level_cap(long long n, int top_n) {
  long long cap = n < (1ll << 20) ? n : (1ll << 20);
  return cap < top_n ? top_n : cap;
}

int choose_shift(uint32_t key_thresh) {
  uint32_t hi = odtk_float_key(1.0f);
  if (hi <= key_thresh) hi = key_thresh + 1;
  unsigned long long span = (unsigned long long)hi - key_thresh + 1;
  int s = 0;
  while ((span >> s) >= (unsigned long long)kHistBins) s++;
  return s;
}

}  // namespace

// mode 0: filter + gather + select (the drop-in path).  mode 1 ("begin"): lay out a workspace whose candidate
// lists can hold EVERY score (no overflow possible), zero the counters and describe the per-level sinks -- the
// class-head convolution's epilogue appends the candidates itself (conv.cu, ODTK_OUT_CANDIDATES).
// mode 2 ("finish"): gather + select + decode on those lists.
static long long decode_levels_impl(int mode, odtk_cand_sink_t *sinks, int batch, int num_levels,
                                    const odtk_level_t *levels, size_t num_anchors, size_t num_classes,
                                    size_t num_anchor_floats, float score_thresh, int top_n, int nbox,
                                    void *const *outputs, size_t out_stride, size_t out_offset, void *workspace,
                                    size_t workspace_size, odtk_stream_t stream_) {
  if (batch <= 0 || num_levels <= 0 || !levels || num_anchors == 0 || num_classes == 0 || top_n <= 0)
    return ODTK_E_INVALID;
  if (nbox != 4 && nbox != 6) return ODTK_E_INVALID;
  if (num_levels > kMaxLevels || top_n > ODTK_MAX_TOP_N || num_anchors > (size_t)kMaxAnchors)
    return ODTK_E_UNSUPPORTED;
  if (num_anchor_floats != 0 && num_anchor_floats != 4 * num_anchors) return ODTK_E_INVALID;
  // large (level descriptors + anchor tables): heap-allocated per call, so concurrent callers on different host
  // threads / streams never share staging state (the kernels take it by value at launch)
  std::unique_ptr<DecodeParams> staging(new DecodeParams);
  DecodeParams &p = *staging;
  const int slots = num_levels * batch;
  long long cand_entries = 0, total_n = 0;
  for (int l = 0; l < num_levels; l++) {
    if (levels[l].height == 0 || levels[l].width == 0) return ODTK_E_INVALID;
    long long n = (long long)num_anchors * num_classes * levels[l].height * levels[l].width;
    if (n >= (1ll << 31)) return ODTK_E_UNSUPPORTED;  // flat index is int32 (decode.cu:122)
    p.lv[l].n = n;
    p.lv[l].cap = (mode == 0) ? level_cap(n, top_n) : (n > top_n ? n : top_n);
    p.lv[l].cand_off = cand_entries;
    cand_entries += p.lv[l].cap * batch;
    total_n += n;
  }
  DecodeWs ws;
  ws.counts_off = 0;
  ws.selcount_off = odtk_align_up((size_t)slots * sizeof(int));
  ws.hist_off = ws.selcount_off + odtk_align_up((size_t)slots * sizeof(int));
  ws.zero_bytes = ws.hist_off + odtk_align_up((size_t)slots * kHistBins * sizeof(uint32_t));
  ws.sel_off = ws.zero_bytes;
  ws.cand_off = ws.sel_off + odtk_align_up((size_t)slots * kSortCap * sizeof(unsigned long long));
  ws.total = ws.cand_off + odtk_align_up((size_t)cand_entries * sizeof(uint2));
  if (!workspace || !workspace_size) return (long long)ws.total;
  if (workspace_size < ws.total) return ODTK_E_WORKSPACE;
  if (mode != 1) {
    if (!outputs || !outputs[0] || !outputs[1] || !outputs[2]) return ODTK_E_INVALID;
    if (out_stride < out_offset + (size_t)top_n * num_levels) return ODTK_E_INVALID;
  }
  cudaStream_t stream = (cudaStream_t)stream_;
  char *base = (char *)workspace;

  // filter grid: one wave of resident CTAs (55 registers x 256 threads -> 4 per SM) x the device's SM count,
  // split between levels by bytes.  ODTK_FILTER_CTAS_PER_SM overrides (tuning knob).
  static int ctas_per_sm = 0;
  if (!ctas_per_sm) {
    const char *e = getenv("ODTK_FILTER_CTAS_PER_SM");
    ctas_per_sm = e ? atoi(e) : 12;  // CTAs per SM of the streaming score filter
    if (ctas_per_sm < 1) ctas_per_sm = 12;
  }
  static int filter_vec = 0;
  if (!filter_vec) { const char *e = getenv("ODTK_FILTER_VEC"); filter_vec = (e && atoi(e) == 8) ? 8 : 4; }   // float4 loads (8-wide: 100 registers, half the resident warps)
  static int filter_bulk = -1;
  if (filter_bulk < 0) { const char *e = getenv("ODTK_FILTER_BULK"); filter_bulk = e ? atoi(e) : 0; }
  bool bulk_ok = filter_bulk != 0;
  for (int l = 0; l < num_levels && mode == 0; l++)     // bulk copies need 16-byte aligned rows of every image
    if ((((uintptr_t)levels[l].scores) & 15) || (((long long)num_anchors * num_classes * levels[l].height * levels[l].width) & 3)) bulk_ok = false;
  const long long budget = (long long)odtk_sm_count() * (bulk_ok ? (filter_bulk > 1 ? filter_bulk : 3) : ctas_per_sm);
  int blk = 0;
  for (int l = 0; l < num_levels; l++) {
    LevelDesc &L = p.lv[l];
    if ((mode == 0 && !levels[l].scores) || (mode != 1 && !levels[l].deltas)) return ODTK_E_INVALID;
    if (num_anchor_floats && !levels[l].anchors) return ODTK_E_INVALID;
    L.scores = (const float *)levels[l].scores;
    L.deltas = (const float *)levels[l].deltas;
    L.height = (int)levels[l].height;
    L.width = (int)levels[l].width;
    L.scale = (int)levels[l].scale;
    L.out_offset = (int)(out_offset + (size_t)l * top_n);
    long long ntiles = bulk_ok ? (L.n + kBulkElems - 1) / kBulkElems : (L.n + filter_vec * 128 - 1) / (filter_vec * 128);
    long long want = (budget * L.n + total_n * batch - 1) / (total_n * batch);
    long long maxb = bulk_ok ? ntiles : (ntiles + kWarpsPerBlock - 1) / kWarpsPerBlock;
    if (want > maxb) want = maxb;
    if (want < 1) want = 1;
    L.blk_per_img = (int)want;
    L.blk_begin = blk;
    blk += L.blk_per_img * batch;
    L.vec = (L.n % 4 == 0) && (((uintptr_t)L.scores) % 16 == 0);
    L.pad = 0;
    for (size_t i = 0; i < 4 * (size_t)kMaxAnchors; i++)
      p.anchors[l][i] = i < num_anchor_floats ? levels[l].anchors[i] : 0.0f;
  }
  p.num_levels = num_levels;
  p.batch = batch;
  p.num_anchors = (int)num_anchors;
  p.num_classes = (int)num_classes;
  p.has_anchors = num_anchor_floats != 0;
  p.top_n = top_n;
  p.thresh = score_thresh;
  p.key_thresh = odtk_float_key(score_thresh);
  p.shift = choose_shift(p.key_thresh);
  p.counts = (int *)(base + ws.counts_off);
  p.selcount = (int *)(base + ws.selcount_off);
  p.hist = (uint32_t *)(base + ws.hist_off);
  p.sel = (unsigned long long *)(base + ws.sel_off);
  p.cand = (uint2 *)(base + ws.cand_off);
  p.out_scores = mode != 1 ? (float *)outputs[0] : nullptr;
  p.out_boxes = mode != 1 ? (float *)outputs[1] : nullptr;
  p.out_classes = mode != 1 ? (float *)outputs[2] : nullptr;
  p.out_stride = (long long)out_stride;

  if (mode != 2 && cudaMemsetAsync(base, 0, ws.zero_bytes, stream) != cudaSuccess) return ODTK_E_CUDA;
  if (mode == 1) {
    if (!sinks) return ODTK_E_INVALID;
    for (int l = 0; l < num_levels; l++) {
      sinks[l].counts = p.counts + (size_t)l * batch;
      sinks[l].hist = p.hist + (size_t)l * batch * kHistBins;
      sinks[l].cand = p.cand + p.lv[l].cand_off;
      sinks[l].cap = p.lv[l].cap;
      sinks[l].key_thresh = p.key_thresh;
      sinks[l].shift = p.shift;
      sinks[l].thresh = score_thresh;
      sinks[l].hist_bins = kHistBins;
    }
    return ODTK_OK;
  }
  if (mode == 0) {
    OdtkProfScope prof(ODTK_PROF_FILTER, stream);
    if (bulk_ok) {
      static bool configured[64] = {};
      int dev = 0;
      cudaGetDevice(&dev);
      const int ring_bytes = kBulkStages * kBulkElems * (int)sizeof(float);
      if (dev < 0 || dev >= 64 || !configured[dev]) {
        if (cudaFuncSetAttribute(score_filter_bulk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ring_bytes) != cudaSuccess) return ODTK_E_CUDA;
        if (dev >= 0 && dev < 64) configured[dev] = true;
      }
      score_filter_bulk_kernel<<<blk, kFilterThreads, ring_bytes, stream>>>(p);
    }
    else if (filter_vec == 8) score_filter_kernel<8><<<blk, kFilterThreads, 0, stream>>>(p);
    else                      score_filter_kernel<4><<<blk, kFilterThreads, 0, stream>>>(p);
  }
  {
    OdtkProfScope prof(ODTK_PROF_SELECT, stream);
    gather_top_kernel<<<dim3(kGatherSlices, slots), kGatherThreads, 0, stream>>>(p);
    if (nbox == 4) select_decode_kernel<4><<<slots, 1024, 0, stream>>>(p);
    else           select_decode_kernel<6><<<slots, 1024, 0, stream>>>(p);
  }
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

extern "C" long long odtk_decode_levels(int batch, int num_levels, const odtk_level_t *levels,
                                        size_t num_anchors, size_t num_classes, size_t num_anchor_floats,
                                        float score_thresh, int top_n, int nbox, void *const *outputs,
                                        size_t out_stride, size_t out_offset, void *workspace,
                                        size_t workspace_size, odtk_stream_t stream) {
  return decode_levels_impl(0, nullptr, batch, num_levels, levels, num_anchors, num_classes, num_anchor_floats,
                            score_thresh, top_n, nbox, outputs, out_stride, out_offset, workspace, workspace_size, stream);
}

extern "C" long long odtk_decode_fused_begin(int batch, int num_levels, const odtk_level_t *levels, size_t num_anchors,
                                             size_t num_classes, float score_thresh, int top_n, odtk_cand_sink_t *sinks,
                                             void *workspace, size_t workspace_size, odtk_stream_t stream) {
  return decode_levels_impl(1, sinks, batch, num_levels, levels, num_anchors, num_classes, 0, score_thresh, top_n, 4,
                            nullptr, 0, 0, workspace, workspace_size, stream);
}

extern "C" long long odtk_decode_fused_finish(int batch, int num_levels, const odtk_level_t *levels, size_t num_anchors,
                                              size_t num_classes, size_t num_anchor_floats, float score_thresh,
                                              int top_n, int nbox, void *const *outputs, size_t out_stride,
                                              size_t out_offset, void *workspace, size_t workspace_size,
                                              odtk_stream_t stream) {
  return decode_levels_impl(2, nullptr, batch, num_levels, levels, num_anchors, num_classes, num_anchor_floats,
                            score_thresh, top_n, nbox, outputs, out_stride, out_offset, workspace, workspace_size, stream);
}

extern "C" long long odtk_decode_ex(int batch, const void *const *inputs, void *const *outputs,
                                    size_t height, size_t width, size_t scale, size_t num_anchors,
                                    size_t num_classes, const float *anchors, size_t num_anchor_floats,
                                    float score_thresh, int top_n, int nbox, size_t out_stride,
                                    size_t out_offset, void *workspace, size_t workspace_size,
                                    odtk_stream_t stream) {
  odtk_level_t lv;
  const bool query = !workspace || !workspace_size;
  if (!query && (!inputs || !inputs[0] || !inputs[1])) return ODTK_E_INVALID;
  lv.scores = query ? nullptr : inputs[0];
  lv.deltas = query ? nullptr : inputs[1];
  lv.height = height;
  lv.width = width;
  lv.scale = scale;
  lv.anchors = anchors;
  return odtk_decode_levels(batch, 1, &lv, num_anchors, num_classes, num_anchor_floats, score_thresh, top_n,
                            nbox, outputs, out_stride, out_offset, workspace, workspace_size, stream);
}

extern "C" long long odtk_decode(int batch, const void *const *inputs, void *const *outputs, size_t height,
                                 size_t width, size_t scale, size_t num_anchors, size_t num_classes,
                                 const float *anchors, size_t num_anchor_floats, float score_thresh,
                                 int top_n, void *workspace, size_t workspace_size, odtk_stream_t stream) {
  return odtk_decode_ex(batch, inputs, outputs, height, width, scale, num_anchors, num_classes, anchors,
                        num_anchor_floats, score_thresh, top_n, 4, (size_t)top_n, 0, workspace,
                        workspace_size, stream);
}

extern "C" long long odtk_decode_rotate(int batch, const void *const *inputs, void *const *outputs,
                                        size_t height, size_t width, size_t scale, size_t num_anchors,
                                        size_t num_classes, const float *anchors, size_t num_anchor_floats,
                                        float score_thresh, int top_n, void *workspace,
                                        size_t workspace_size, odtk_stream_t stream) {
  return odtk_decode_ex(batch, inputs, outputs, height, width, scale, num_anchors, num_classes, anchors,
                        num_anchor_floats, score_thresh, top_n, 6, (size_t)top_n, 0, workspace,
                        workspace_size, stream);
}
