// nms.cu -- batched per-image greedy NMS (axis-aligned and rotated) for sm_90a.
//
// Replaces odtk::cuda::nms + nms_kernel (reference csrc/cuda/nms.cu:44-160) and
// odtk::cuda::nms_rotate + nms_rotate_kernel (csrc/cuda/nms_iou.cu:114-322).  The
// reference handles ONE image at a time: cub select -> host sync -> gather -> 32-bit radix
// sort -> a single 1024-thread block that walks ALL n candidates serially with a
// __syncthreads each -> second radix sort -> gathers.  Here the whole batch is one launch,
// one CTA per image, nothing leaves shared memory:
//
//   1. unique composite keys (score key << 13 | ~position) for scores > 0, one block-wide
//      cub radix sort (45 bits) == the reference's stable descending device radix sort;
//   2. the ranks are resolved in chunks of 128: every candidate of the chunk is tested against the
//      keepers of earlier chunks, the same-class / overlap relation inside the chunk is evaluated
//      for all pairs at once into a 128 x 128 bit matrix (class gate first, IEEE division, +1
//      widths), and one warp resolves the chunk sequentially with bit operations only.  The walk
//      stops at detections_per_im keepers -- exact, because the output is the first D entries of
//      (kept..., suppressed...) and later candidates never change earlier decisions; with the BASELINE workload one chunk is enough;
//   3. if fewer than D were kept the tail is the first suppressed candidates in rank order
//      with score 0 and their boxes/classes, exactly what the reference's second sort
//      leaves there (nms.cu:146-156).
//
// Arithmetic: fp32, IEEE division, no FMA contraction (-fmad=false): the PyTorch path is
// the parity target, not the reference's --use_fast_math build.
#include <limits.h>
#include <string.h>

#include <cub/block/block_radix_sort.cuh>

#include "common.cuh"
#include "polygon.cuh"
#include "prof.cuh"

namespace {

constexpr int kThreads = 1024;
constexpr int kMaxCount = ODTK_MAX_NMS_COUNT;  // 6144
constexpr int kMaxRanks = kMaxCount / kThreads;  // ranks per thread
constexpr int kMaxDet = ODTK_MAX_DETECTIONS;

struct NmsParams {
  const float *scores, *boxes, *classes;  // [B,count], [B,count,NBOX], [B,count]
  float *out_scores, *out_boxes, *out_classes;   // may be NULL when only the packed form is wanted
  int32_t *out_index;  // may be NULL
  int count, detections;
  float thresh;
  int fixed_angle;
  // packed detections [B, D, 2 + NBOX] = (score, box..., class): the local copy and -- image-wise sharded inference,
  // odtk/infer.py:98-102 -- the same rows pushed straight into every peer GPU's gather buffer over NVLink
  float *packed_local;                 // [B, D, 2 + NBOX] or NULL
  float *peer_packed[ODTK_MAX_PEERS];  // peer p's gather buffer: 2 parity halves of [W * B, D, 2 + NBOX]
  unsigned *peer_flags[ODTK_MAX_PEERS];   // peer p's arrival counters [W]: += 1 per image of this rank
  const unsigned *epoch;               // local step counter (device): selects the parity half
  int num_peers, rank, batch;
};

constexpr int kPosBits = 13;  // count <= 6144 < 2^13
constexpr int kChunk = 128;   // ranks resolved per round
constexpr int kPrefixMin = 512;   // prefix mode: resolve at least this many top-scoring candidates first ...
constexpr int kPrefixCap = 2048;  // ... and at most this many (bitonic sort in shared memory)
#ifndef ODTK_NMS_RADIX_BITS
#define ODTK_NMS_RADIX_BITS 4
#endif
typedef cub::BlockRadixSort<unsigned long long, kThreads, kMaxRanks, cub::NullType, ODTK_NMS_RADIX_BITS> BlockSort;

// Shared memory: the radix-sort scratch is dead once the ranks sit in registers, so the
// per-window and keeper arrays alias it.
template <int NBOX>
struct NmsSmem {
  struct Data {
    float cbox[kChunk][NBOX];     // current chunk of 128 ranks
    int ccls[kChunk];
    int cidx[kChunk];
    int prevsup[kChunk];          // suppressed by a keeper of an earlier chunk
    unsigned mask[kChunk][kChunk / 32];   // bit j of row i: j < i would suppress i if it survives
    float kbox[kMaxDet][NBOX];    // keepers so far
    int kcls[kMaxDet];
    int kidx[kMaxDet];
    int tidx[kMaxDet];            // suppressed candidates in rank order (output tail)
  };
  union U {
    typename BlockSort::TempStorage sort;
    Data d;
  };
  struct All {
    U u;
    unsigned long long sel[kPrefixCap];   // prefix mode: composites of the candidates above the selection threshold
    uint32_t hist[ODTK_HIST_BINS];        // prefix mode: histogram of the score keys' top bits
  };
};

template <int NBOX>
__global__ void __launch_bounds__(kThreads) nms_batched_kernel(NmsParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  typename NmsSmem<NBOX>::All &all = *reinterpret_cast<typename NmsSmem<NBOX>::All *>(smem_raw);
  typename NmsSmem<NBOX>::U &sm = all.u;
  __shared__ int s_kept, s_ntail;
  __shared__ int s_n, s_nsel;
  __shared__ int s_w[32], s_res[2];

  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int img = blockIdx.x;
  const int count = p.count, D = p.detections;
  const float *sc = p.scores + (long long)img * count;
  const float *bx = p.boxes + (long long)img * count * NBOX;
  const float *cl = p.classes + (long long)img * count;

  // ---- 1. keys (nms.cu:125-137) -------------------------------------------------------------
  // composite = (score key << 13) | ~position: unique, so ANY descending sort of the composites reproduces cub's stable
  // descending order of the reference.
  if (t == 0) { s_n = 0; s_nsel = 0; }
  for (int i = t; i < ODTK_HIST_BINS; i += kThreads) all.hist[i] = 0u;
  __syncthreads();
  unsigned long long keys[kMaxRanks];
  int nvalid = 0;
#pragma unroll
  for (int k = 0; k < kMaxRanks; k++) {
    int i = t * kMaxRanks + k;  // blocked arrangement in, striped out
    unsigned long long c = 0ull;
    if (i < count) {
      float v = sc[i];
      if (v > 0.0f) {
        const uint32_t key = odtk_float_key(v);
        c = ((unsigned long long)key << kPosBits) | (unsigned)((~(unsigned)i) & ((1u << kPosBits) - 1u));
        atomicAdd(&all.hist[(key >> 20) & (ODTK_HIST_BINS - 1)], 1u);   // positive floats: sign bit set, 11 bits below it
        nvalid++;
      }
    }
    keys[k] = c;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) nvalid += __shfl_xor_sync(0xffffffffu, nvalid, o);
  if (lane == 0 && nvalid) atomicAdd(&s_n, nvalid);
  __syncthreads();
  const int n = s_n;
  const int nd = n < D ? n : D;

  // ---- 2. order.  Prefix mode: the output needs only the first D keepers, and the greedy walk never looks back, so it
  // is enough to order the top-scoring candidates: a histogram threshold selects between kPrefixMin and kPrefixCap of
  // them, a bitonic sort in shared memory orders those, and only if the walk exhausts them without reaching D keepers
  // (pathological overlap) the full block radix sort of all candidates runs.  Results are identical either way.
  int nsel = n;
  bool prefix = false;
  if (n > kPrefixMin) {
    int bstar, cnt;
    odtk_find_bstar(all.hist, kPrefixMin, s_w, s_res, bstar, cnt);
    if (cnt <= kPrefixCap) {
      prefix = true;
#pragma unroll
      for (int k = 0; k < kMaxRanks; k++) {
        const unsigned long long c = keys[k];
        if (c != 0ull && (int)((uint32_t)(c >> (kPosBits + 20)) & (ODTK_HIST_BINS - 1)) >= bstar) all.sel[atomicAdd(&s_nsel, 1)] = c;
      }
      __syncthreads();
      nsel = s_nsel;                     // == cnt
      const int P = odtk_next_pow2(nsel);
      for (int i = nsel + t; i < P; i += kThreads) all.sel[i] = 0ull;
      __syncthreads();
      odtk_bitonic_desc_u64(all.sel, P);
    }
  } else if (n > 0) {
    prefix = true;                       // few candidates: order all of them in shared memory
#pragma unroll
    for (int k = 0; k < kMaxRanks; k++)
      if (keys[k] != 0ull) all.sel[atomicAdd(&s_nsel, 1)] = keys[k];
    __syncthreads();
    const int P = odtk_next_pow2(n);
    for (int i = n + t; i < P; i += kThreads) all.sel[i] = 0ull;
    __syncthreads();
    odtk_bitonic_desc_u64(all.sel, P);
  }

  int kept = 0, ntail = 0;
#pragma unroll 1
  for (int attempt = 0; attempt < 2; attempt++) {
    if (attempt == 1) {
      if (!prefix || kept >= D || nsel >= n) break;        // the prefix was enough (always, on real detector outputs)
      prefix = false;
      nsel = n;
    }
    if (!prefix && n > 0) {
      __syncthreads();
      BlockSort(sm.sort).SortDescendingBlockedToStriped(keys, 0, 32 + kPosBits);   // thread t holds ranks t + k*1024
      __syncthreads();                   // sort scratch is dead from here on
    }

    // ---- greedy NMS in chunks of 128 ranks (nms_kernel, nms.cu:49-79) ---------------------
    // Per chunk: (A) every candidate is tested against the keepers of earlier chunks, (B) the
    // same-class / overlap relation INSIDE the chunk is evaluated for all pairs at once into a
    // 128 x 128 bit matrix, (C) one warp resolves the chunk sequentially with bit operations only
    // (candidate i survives iff no earlier SURVIVOR of the chunk has its bit set in row i).  All
    // floating-point work is parallel; the serial part is ~30 cycles per candidate and stops at D
    // keepers -- the reference's kernel runs one block-wide barrier per candidate instead.
    kept = 0; ntail = 0;
    const int nchunk = (nsel + kChunk - 1) / kChunk;
    if (t == 0) { s_kept = 0; s_ntail = 0; }
    __syncthreads();
#pragma unroll 1
    for (int c = 0; c < nchunk && kept < D; c++) {
      const int r0 = c * kChunk, cn = min(kChunk, nsel - r0);
      {
        unsigned long long key = 0ull;
        bool mine = false;
        if (prefix) {
          mine = t < cn;
          if (mine) key = all.sel[r0 + t];
        } else {
          // the chunk's ranks live in threads (r0 + i) % 1024, register slot (r0 + i) / 1024
          const int i = t - (r0 % kThreads);
          mine = i >= 0 && i < cn;
          const int slot = r0 / kThreads;
#pragma unroll
          for (int k = 0; k < kMaxRanks; k++)
            if (k == slot) key = keys[k];
        }
        if (mine) {
          const int i = prefix ? t : t - (r0 % kThreads);
          const int idx = (int)((~(unsigned)key) & ((1u << kPosBits) - 1u));
          if (NBOX == 4) {
            *reinterpret_cast<float4 *>(sm.d.cbox[i]) = *reinterpret_cast<const float4 *>(bx + (long long)idx * 4);
          } else {
#pragma unroll
            for (int q = 0; q < NBOX; q += 2)
              *reinterpret_cast<float2 *>(&sm.d.cbox[i][q]) = *reinterpret_cast<const float2 *>(bx + (long long)idx * NBOX + q);
          }
          sm.d.ccls[i] = (int)cl[idx];  // float -> int cast as nms.cu:55-56
          sm.d.cidx[i] = idx;
        }
        if (t < kChunk) {
          sm.d.prevsup[t] = 0;
#pragma unroll
          for (int w = 0; w < kChunk / 32; w++) sm.d.mask[t][w] = 0u;
        }
      }
      __syncthreads();
      // (A) against keepers of earlier chunks: pairs (i, q), i < cn, q < kept
      for (int pidx = t; pidx < cn * kept; pidx += kThreads) {
        const int i = pidx % cn, q = pidx / cn;
        if (sm.d.kcls[q] == sm.d.ccls[i]) {
          float ov = (NBOX == 4) ? aligned_overlap(sm.d.cbox[i], sm.d.kbox[q])
                                 : rotated_overlap(sm.d.cbox[i], sm.d.kbox[q], p.fixed_angle);
          if (ov > p.thresh) sm.d.prevsup[i] = 1;
        }
      }
      // (B) inside the chunk: pairs (i, j) with j < i; thread -> (i, 16 consecutive j)
      for (int pidx = t; pidx < cn * (kChunk / 16); pidx += kThreads) {
        const int i = pidx % cn, jg = pidx / cn;
        unsigned bits = 0u;
        const int icls = sm.d.ccls[i];
#pragma unroll 4
        for (int jj = 0; jj < 16; jj++) {
          const int j = jg * 16 + jj;
          if (j < i && sm.d.ccls[j] == icls) {
            float ov = (NBOX == 4) ? aligned_overlap(sm.d.cbox[i], sm.d.cbox[j])
                                   : rotated_overlap(sm.d.cbox[i], sm.d.cbox[j], p.fixed_angle);
            if (ov > p.thresh) bits |= 1u << jj;
          }
        }
        if (bits) atomicOr(&sm.d.mask[i][jg >> 1], bits << ((jg & 1) * 16));
      }
      __syncthreads();
      // (C) sequential resolution by one warp: lane w (< 4) owns survivor word w of the chunk
      if (warp == 0) {
        unsigned surv = 0u;
        int k2 = kept, nt2 = ntail;
        for (int i = 0; i < cn && k2 < D; i++) {
          const unsigned hit = (lane < kChunk / 32) ? (sm.d.mask[i][lane] & surv) : 0u;
          const bool dead = sm.d.prevsup[i] || __any_sync(0xffffffffu, hit != 0u);
          if (!dead) {
            if (lane == (i >> 5)) surv |= 1u << (i & 31);
            if (lane < NBOX) sm.d.kbox[k2][lane] = sm.d.cbox[i][lane];
            if (lane == 0) { sm.d.kcls[k2] = sm.d.ccls[i]; sm.d.kidx[k2] = sm.d.cidx[i]; }
            k2++;
          } else {
            if (lane == 0 && nt2 < D) sm.d.tidx[nt2] = sm.d.cidx[i];
            nt2++;
          }
        }
        if (lane == 0) { s_kept = k2; s_ntail = nt2; }
      }
      __syncthreads();
      kept = s_kept;
      ntail = s_ntail;
    }
    __syncthreads();
  }

  // ---- 3. outputs (nms.cu:150-156): kept..., then suppressed (score 0) up to min(D, n) ----
  float *os = p.out_scores ? p.out_scores + (long long)img * D : nullptr;
  float *ob = p.out_boxes ? p.out_boxes + (long long)img * D * NBOX : nullptr;
  float *oc = p.out_classes ? p.out_classes + (long long)img * D : nullptr;
  int32_t *oi = p.out_index ? p.out_index + (long long)img * D : nullptr;
  constexpr int PK = 2 + NBOX;
  float *pk = p.packed_local ? p.packed_local + (long long)img * D * PK : nullptr;
  const long long half = (long long)p.num_peers * p.batch * D * PK;      // floats per parity half of a gather buffer
  const long long prow = ((p.num_peers > 0 && p.epoch) ? (long long)(*p.epoch & 1u) * half : 0) + ((long long)p.rank * p.batch + img) * D * PK;
  for (int j = t; j < D; j += kThreads) {
    float v[PK];
    int i = -1;
    if (j < nd) {
      i = (j < kept) ? sm.d.kidx[j] : sm.d.tidx[j - kept];
      v[0] = (j < kept) ? sc[i] : 0.0f;
#pragma unroll
      for (int q = 0; q < NBOX; q++) v[1 + q] = bx[(long long)i * NBOX + q];
      v[PK - 1] = cl[i];
    } else {
#pragma unroll
      for (int q = 0; q < PK; q++) v[q] = 0.0f;
    }
    if (os) os[j] = v[0];
    if (ob) {
#pragma unroll
      for (int q = 0; q < NBOX; q++) ob[j * NBOX + q] = v[1 + q];
    }
    if (oc) oc[j] = v[PK - 1];
    if (oi) oi[j] = i;
    if (pk) {
#pragma unroll
      for (int q = 0; q < PK; q++) pk[j * PK + q] = v[q];
    }
    for (int pr = 0; pr < p.num_peers; pr++) {       // peer-mapped stores: the all-gather happens here, row by row
      float *dst = p.peer_packed[pr] + prow + (long long)j * PK;
#pragma unroll
      for (int q = 0; q < PK; q++) dst[q] = v[q];
    }
  }
  if (p.num_peers > 0) {
    __threadfence_system();                          // every thread's peer stores are visible system-wide ...
    __syncthreads();
    if (t < p.num_peers) atomicAdd_system(p.peer_flags[t] + p.rank, 1u);   // ... before the arrival is counted
  }
}

// Completes the in-kernel all-gather on the receiving side: waits until every rank has delivered all its images of the
// current step into this GPU's gather buffer, then advances the local step counter.  One warp.
__global__ void gather_wait_kernel(const volatile unsigned *flags, unsigned *epoch, int num_peers, int batch) {
  const unsigned target = (*epoch + 1u) * (unsigned)batch;
  if ((int)threadIdx.x < num_peers) {
    while ((int)(flags[threadIdx.x] - target) < 0) __nanosleep(64);
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) *epoch = *epoch + 1u;
}

template <int NBOX>
long long launch_nms(const NmsParams &p, int batch, cudaStream_t stream) {
  const size_t smem = sizeof(typename NmsSmem<NBOX>::All);
  // the > 48 KB dynamic shared memory opt-in is a per-device function attribute: once per (template instance, device)
  static bool configured[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return ODTK_E_CUDA;
  if (dev < 0 || dev >= 64 || !configured[dev]) {
    if (cudaFuncSetAttribute(nms_batched_kernel<NBOX>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)smem) != cudaSuccess)
      return ODTK_E_CUDA;
    if (dev >= 0 && dev < 64) configured[dev] = true;
  }
  {
    OdtkProfScope prof(ODTK_PROF_NMS, stream);
    nms_batched_kernel<NBOX><<<batch, kThreads, smem, stream>>>(p);
  }
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

}  // namespace

extern "C" long long odtk_nms_ex(int batch, const void *const *inputs, void *const *outputs, size_t count,
                                 int detections_per_im, float nms_thresh, int nbox, int fixed_angle,
                                 int32_t *out_index, void *workspace, size_t workspace_size,
                                 odtk_stream_t stream) {
  if (batch <= 0 || count == 0 || detections_per_im <= 0) return ODTK_E_INVALID;
  if (nbox != 4 && nbox != 6) return ODTK_E_INVALID;
  if (count > (size_t)kMaxCount || detections_per_im > kMaxDet) return ODTK_E_UNSUPPORTED;
  // Everything lives in shared memory; a token workspace keeps the two-phase convention.
  if (!workspace || !workspace_size) return ODTK_ALIGN;
  if (workspace_size < ODTK_ALIGN) return ODTK_E_WORKSPACE;
  return odtk_nms_gather(batch, inputs, outputs, count, detections_per_im, nms_thresh, nbox, fixed_angle, out_index,
                         nullptr, nullptr, workspace, workspace_size, stream);
}

extern "C" long long odtk_nms_gather(int batch, const void *const *inputs, void *const *outputs, size_t count,
                                     int detections_per_im, float nms_thresh, int nbox, int fixed_angle,
                                     int32_t *out_index, void *packed, const odtk_gather_t *gather, void *workspace,
                                     size_t workspace_size, odtk_stream_t stream) {
  if (batch <= 0 || count == 0 || detections_per_im <= 0) return ODTK_E_INVALID;
  if (nbox != 4 && nbox != 6) return ODTK_E_INVALID;
  if (count > (size_t)kMaxCount || detections_per_im > kMaxDet) return ODTK_E_UNSUPPORTED;
  if (!workspace || !workspace_size) return ODTK_ALIGN;
  if (workspace_size < ODTK_ALIGN) return ODTK_E_WORKSPACE;
  if (!inputs || !inputs[0] || !inputs[1] || !inputs[2]) return ODTK_E_INVALID;
  const bool have_out = outputs && outputs[0] && outputs[1] && outputs[2];
  if (!have_out && !packed && !(gather && gather->num_peers > 0)) return ODTK_E_INVALID;
  if (outputs && !have_out && (outputs[0] || outputs[1] || outputs[2])) return ODTK_E_INVALID;   // all three or none
  if (((uintptr_t)inputs[1]) % (nbox == 4 ? 16 : 8)) return ODTK_E_INVALID;  // vector loads of the boxes
  NmsParams p;
  memset(&p, 0, sizeof p);
  p.scores = (const float *)inputs[0];
  p.boxes = (const float *)inputs[1];
  p.classes = (const float *)inputs[2];
  if (have_out) { p.out_scores = (float *)outputs[0]; p.out_boxes = (float *)outputs[1]; p.out_classes = (float *)outputs[2]; }
  p.out_index = out_index;
  p.count = (int)count;
  p.detections = detections_per_im;
  p.thresh = nms_thresh;
  p.fixed_angle = fixed_angle;
  p.packed_local = (float *)packed;
  p.batch = batch;
  if (gather && gather->num_peers > 0) {
    if (gather->num_peers > ODTK_MAX_PEERS || gather->rank < 0 || gather->rank >= gather->num_peers || !gather->epoch)
      return ODTK_E_INVALID;
    for (int i = 0; i < gather->num_peers; i++) {
      if (!gather->packed[i] || !gather->flags[i]) return ODTK_E_INVALID;
      p.peer_packed[i] = (float *)gather->packed[i];
      p.peer_flags[i] = gather->flags[i];
    }
    p.num_peers = gather->num_peers;
    p.rank = gather->rank;
    p.epoch = gather->epoch;
  }
  return nbox == 4 ? launch_nms<4>(p, batch, (cudaStream_t)stream) : launch_nms<6>(p, batch, (cudaStream_t)stream);
}

extern "C" int odtk_gather_wait(const odtk_gather_t *gather, int batch, odtk_stream_t stream) {
  if (!gather || gather->num_peers <= 0 || gather->num_peers > ODTK_MAX_PEERS || batch <= 0 || !gather->epoch) return ODTK_E_INVALID;
  if (gather->rank < 0 || gather->rank >= gather->num_peers || !gather->flags[gather->rank]) return ODTK_E_INVALID;
  gather_wait_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(gather->flags[gather->rank], gather->epoch, gather->num_peers, batch);
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

extern "C" long long odtk_nms(int batch, const void *const *inputs, void *const *outputs, size_t count,
                              int detections_per_im, float nms_thresh, void *workspace,
                              size_t workspace_size, odtk_stream_t stream) {
  return odtk_nms_ex(batch, inputs, outputs, count, detections_per_im, nms_thresh, 4, 0, nullptr, workspace,
                     workspace_size, stream);
}

extern "C" long long odtk_nms_rotate(int batch, const void *const *inputs, void *const *outputs, size_t count,
                                     int detections_per_im, float nms_thresh, void *workspace,
                                     size_t workspace_size, odtk_stream_t stream) {
  return odtk_nms_ex(batch, inputs, outputs, count, detections_per_im, nms_thresh, 6, 0, nullptr, workspace,
                     workspace_size, stream);
}
