// loss.cu -- fused focal loss forward + backward for sm_90a (HBM-bound, one pass).
//
// Replaces FocalLoss.forward (reference odtk/loss.py:13-18) as used by Model._compute_loss
// (odtk/model.py:195-199): sigmoid, BCE-with-logits, alpha_t, p_t, the modulating factor, the
// (depth >= 0) mask, the sum, and -- in the same pass -- the gradient of that sum w.r.t. the
// logits, which the reference obtains by autograd through ~8 elementwise kernels, each a full
// pass over [B, A, C, H, W] fp32 (15.36 M elements per image at 3x800x1280).
//
// Targets come either dense (fp32 one-hot, the reference's layout) or as class indices
// [B*A, H*W] (class id, -1 = background, -2 = ignored), which removes the one-hot read
// altogether.  fp32 maths; 128-bit loads/stores; block partial sums in double, summed in a
// fixed order by a second tiny kernel, so the result is deterministic.
#include <cuda_fp16.h>
#include <string.h>

#include <cooperative_groups.h>

#include "common.cuh"
#include "prof.cuh"

namespace cg = cooperative_groups;

namespace {

constexpr int kThreads = 256;

struct LossParams {
  const float *logits;
  const float *target;   // dense one-hot or NULL
  const float *mask;     // dense mask or NULL
  const int *cls_index;  // [groups, hw] or NULL
  long long n;
  int num_classes, hw;   // indexed mode: element e -> group e / (C*hw), class (e / hw) % C, pos e % hw
  float alpha, gamma, grad_scale;
  float *loss_elem;      // or NULL
  float *grad;           // or NULL
  double *partials;      // [gridDim.x]
};

__device__ __forceinline__ void focal_one(float x, float t, float m, const LossParams &p, float &loss, float &grad) {
  const float e = expf(-fabsf(x));
  const float inv = 1.0f / (1.0f + e);
  const float pr = x >= 0.0f ? inv : e * inv;          // sigmoid(x)
  const float ce = fmaxf(x, 0.0f) - x * t + log1pf(e);   // BCE with logits
  const float a = t * p.alpha + (1.0f - t) * (1.0f - p.alpha);
  const bool pos = (t == 1.0f);
  const float q = pos ? 1.0f - pr : pr;                  // 1 - p_t
  float w, dwq;                                          // q^gamma, gamma * q^(gamma-1)
  if (p.gamma == 2.0f) { w = q * q; dwq = 2.0f * q; }
  else { w = powf(q, p.gamma); dwq = (p.gamma == 0.0f) ? 0.0f : p.gamma * powf(q, p.gamma - 1.0f); }
  loss = m * a * w * ce;
  const float dq = (pos ? -1.0f : 1.0f) * pr * (1.0f - pr);
  grad = m * a * (dwq * dq * ce + w * (pr - t)) * p.grad_scale;
}

__global__ void __launch_bounds__(kThreads) focal_loss_kernel(LossParams p) {
  __shared__ double s_part[kThreads / 32];
  double acc = 0.0;
  const long long nvec = p.n >> 2;
  const bool aligned = (((uintptr_t)p.logits | (uintptr_t)p.target | (uintptr_t)p.mask | (uintptr_t)p.cls_index |
                         (uintptr_t)p.loss_elem | (uintptr_t)p.grad) & 15) == 0;
  const bool vec_ok = aligned && ((p.n & 3) == 0) && (p.cls_index == nullptr || (p.hw & 3) == 0);   // else: scalar loop
  if (vec_ok) {
    for (long long v = (long long)blockIdx.x * kThreads + threadIdx.x; v < nvec; v += (long long)gridDim.x * kThreads) {
      const long long e0 = v << 2;
      float4 x4 = odtk_ld_stream_f4(reinterpret_cast<const float4 *>(p.logits) + v);
      float x[4] = {x4.x, x4.y, x4.z, x4.w}, t[4], m[4] = {1.f, 1.f, 1.f, 1.f};
      if (p.cls_index) {
        const long long chw = (long long)p.num_classes * p.hw;
        const long long g = e0 / chw;
        const long long r = e0 - g * chw;
        const int c = (int)(r / p.hw), pos = (int)(r - (long long)c * p.hw);
        int4 ci = *reinterpret_cast<const int4 *>(p.cls_index + g * p.hw + pos);
        int idx[4] = {ci.x, ci.y, ci.z, ci.w};
#pragma unroll
        for (int j = 0; j < 4; j++) { t[j] = (idx[j] == c) ? 1.0f : 0.0f; m[j] = (idx[j] == -2) ? 0.0f : 1.0f; }
      } else {
        float4 t4 = odtk_ld_stream_f4(reinterpret_cast<const float4 *>(p.target) + v);
        t[0] = t4.x; t[1] = t4.y; t[2] = t4.z; t[3] = t4.w;
        if (p.mask) {
          float4 m4 = odtk_ld_stream_f4(reinterpret_cast<const float4 *>(p.mask) + v);
          m[0] = m4.x; m[1] = m4.y; m[2] = m4.z; m[3] = m4.w;
        }
      }
      float l[4], g4[4];
#pragma unroll
      for (int j = 0; j < 4; j++) { focal_one(x[j], t[j], m[j], p, l[j], g4[j]); acc += (double)l[j]; }
      if (p.loss_elem) reinterpret_cast<float4 *>(p.loss_elem)[v] = make_float4(l[0], l[1], l[2], l[3]);
      if (p.grad) reinterpret_cast<float4 *>(p.grad)[v] = make_float4(g4[0], g4[1], g4[2], g4[3]);
    }
  } else {
    for (long long e = (long long)blockIdx.x * kThreads + threadIdx.x; e < p.n; e += (long long)gridDim.x * kThreads) {
      float x = p.logits[e], t, m = 1.0f;
      if (p.cls_index) {
        const long long chw = (long long)p.num_classes * p.hw;
        const long long g = e / chw;
        const long long r = e - g * chw;
        const int c = (int)(r / p.hw), pos = (int)(r - (long long)c * p.hw);
        const int idx = p.cls_index[g * p.hw + pos];
        t = (idx == c) ? 1.0f : 0.0f;
        m = (idx == -2) ? 0.0f : 1.0f;
      } else {
        t = p.target[e];
        if (p.mask) m = p.mask[e];
      }
      float l, g;
      focal_one(x, t, m, p, l, g);
      acc += (double)l;
      if (p.loss_elem) p.loss_elem[e] = l;
      if (p.grad) p.grad[e] = g;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < kThreads / 32; w++) s += s_part[w];
    p.partials[blockIdx.x] = s;
  }
}

// Smooth L1 (reference odtk/loss.py:27-31): x = |pred - target|; x >= beta ? x - beta/2 : x^2 / (2 beta);
// masked sum + gradient in the same pass (box regression loss of Model._compute_loss, model.py:201-205).
__global__ void __launch_bounds__(kThreads) smooth_l1_kernel(const float *pred, const float *target, const float *mask,
                                                             long long n, float beta, float grad_scale,
                                                             float *loss_elem, float *grad, double *partials) {
  __shared__ double s_part[kThreads / 32];
  double acc = 0.0;
  for (long long e = (long long)blockIdx.x * kThreads + threadIdx.x; e < n; e += (long long)gridDim.x * kThreads) {
    const float d = pred[e] - target[e], x = fabsf(d), m = mask ? mask[e] : 1.0f;
    const bool lin = x >= beta;
    const float l = m * (lin ? x - 0.5f * beta : 0.5f * x * x / beta);
    acc += (double)l;
    if (loss_elem) loss_elem[e] = l;
    if (grad) grad[e] = m * grad_scale * (lin ? (d > 0.0f ? 1.0f : (d < 0.0f ? -1.0f : 0.0f)) : d / beta);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < kThreads / 32; w++) s += s_part[w];
    partials[blockIdx.x] = s;
  }
}

__global__ void focal_loss_finish_kernel(const double *partials, int n, float *out) {
  double s = 0.0;
  for (int i = 0; i < n; i++) s += partials[i];  // fixed order: deterministic
  *out = (float)s;
}

// ---- Model._compute_loss in ONE launch (reference odtk/model.py:186-210) -----------------------------------------------
// All pyramid levels: focal loss of the class logits against the class-index targets with the (depth >= 0) mask, smooth
// L1 of the box deltas with the (depth > 0) mask, the per-level foreground counts clamp(min=1), their sum, and both
// losses divided by it -- plus, optionally, the gradients of the two normalised losses w.r.t. the head outputs.
// Cooperative launch: (A) count foreground positions per level (integer atomics: deterministic), grid barrier,
// (B) stream the heads once, block partial sums in double, grid barrier, (C) block 0 adds the partials in index order.
struct RetinaLevel {
  const float *cls_logits, *box_pred, *box_target;
  const int *cls_index;
  float *cls_grad, *box_grad;
  int hw;
  long long npos;        // B * A * hw
};
struct RetinaParams {
  RetinaLevel lv[ODTK_MAX_LEVELS];
  int num_levels, num_classes, nbox;
  float alpha, gamma, beta;
  int *counts;           // [ODTK_MAX_LEVELS], zeroed before the launch
  double *partials;      // [2 * gridDim.x]
  float *out;            // [4]: cls_loss, box_loss, fg_total, 0
};

__device__ __forceinline__ double block_sum(double acc, double *s_part) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = acc;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < kThreads / 32; w++) s += s_part[w];
  return s;
}

__global__ void __launch_bounds__(kThreads) retina_loss_kernel(RetinaParams p) {
  __shared__ double s_part[kThreads / 32];
  cg::grid_group grid = cg::this_grid();
  const long long tid = (long long)blockIdx.x * kThreads + threadIdx.x, nthr = (long long)gridDim.x * kThreads;
  // (A) foreground positions per level: (depth > 0).sum() == #(cls_index >= 0)
  for (int l = 0; l < p.num_levels; l++) {
    int cnt = 0;
    for (long long i = tid; i < p.lv[l].npos; i += nthr) cnt += (p.lv[l].cls_index[i] >= 0) ? 1 : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(p.counts + l, cnt);
  }
  grid.sync();
  float fg_total = 0.0f;
  for (int l = 0; l < p.num_levels; l++) fg_total += (float)max(p.counts[l], 1);   // .float().clamp(min=1), then the sum
  const float inv = 1.0f / fg_total;
  LossParams fp;
  fp.alpha = p.alpha; fp.gamma = p.gamma; fp.grad_scale = inv;
  // (B) one pass over the heads
  double acc_c = 0.0, acc_b = 0.0;
  for (int l = 0; l < p.num_levels; l++) {
    const RetinaLevel &L = p.lv[l];
    const int hw = L.hw, C = p.num_classes;
    const long long chw = (long long)C * hw, n = L.npos * C;
    const bool vec = (hw & 3) == 0 && (((uintptr_t)L.cls_logits | (uintptr_t)L.cls_index | (uintptr_t)L.cls_grad) & 15) == 0;
    if (vec) {
      for (long long v = tid; v < (n >> 2); v += nthr) {
        const long long e0 = v << 2, g = e0 / chw, r = e0 - g * chw;
        const int c = (int)(r / hw), pos = (int)(r - (long long)c * hw);
        const float4 x4 = odtk_ld_stream_f4(reinterpret_cast<const float4 *>(L.cls_logits) + v);
        const int4 ci = *reinterpret_cast<const int4 *>(L.cls_index + g * hw + pos);
        const float x[4] = {x4.x, x4.y, x4.z, x4.w};
        const int idx[4] = {ci.x, ci.y, ci.z, ci.w};
        float gr[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
          float lo;
          focal_one(x[j], idx[j] == c ? 1.0f : 0.0f, idx[j] == -2 ? 0.0f : 1.0f, fp, lo, gr[j]);
          acc_c += (double)lo;
        }
        if (L.cls_grad) reinterpret_cast<float4 *>(L.cls_grad)[v] = make_float4(gr[0], gr[1], gr[2], gr[3]);
      }
    } else {
      for (long long e = tid; e < n; e += nthr) {
        const long long g = e / chw, r = e - g * chw;
        const int c = (int)(r / hw), pos = (int)(r - (long long)c * hw);
        const int idx = L.cls_index[g * hw + pos];
        float lo, gr;
        focal_one(L.cls_logits[e], idx == c ? 1.0f : 0.0f, idx == -2 ? 0.0f : 1.0f, fp, lo, gr);
        acc_c += (double)lo;
        if (L.cls_grad) L.cls_grad[e] = gr;
      }
    }
    const long long nb = L.npos * p.nbox, bhw = (long long)p.nbox * hw;
    for (long long e = tid; e < nb; e += nthr) {
      const long long g = e / bhw, r = e - g * bhw;
      const int pos = (int)(r % hw);
      const float m = (L.cls_index[g * hw + pos] >= 0) ? 1.0f : 0.0f;
      const float d = L.box_pred[e] - L.box_target[e], x = fabsf(d);
      const bool lin = x >= p.beta;
      acc_b += (double)(m * (lin ? x - 0.5f * p.beta : 0.5f * x * x / p.beta));
      if (L.box_grad) L.box_grad[e] = m * inv * (lin ? (d > 0.0f ? 1.0f : (d < 0.0f ? -1.0f : 0.0f)) : d / p.beta);
    }
  }
  const double sc = block_sum(acc_c, s_part);
  const double sb = block_sum(acc_b, s_part);
  if (threadIdx.x == 0) { p.partials[blockIdx.x] = sc; p.partials[gridDim.x + blockIdx.x] = sb; }
  grid.sync();
  // (C) fixed-order final sums, normalised
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    double c = 0.0, b = 0.0;
    for (unsigned i = 0; i < gridDim.x; i++) { c += p.partials[i]; b += p.partials[gridDim.x + i]; }
    p.out[0] = (float)(c / (double)fg_total);
    p.out[1] = (float)(b / (double)fg_total);
    p.out[2] = fg_total;
    p.out[3] = 0.0f;
  }
}

int loss_grid(long long n) {
  long long b = (n / 4 + kThreads - 1) / kThreads / 4;
  if (b < 1) b = 1;
  if (b > odtk_sm_count() * 8) b = odtk_sm_count() * 8;
  return (int)b;
}

}  // namespace

extern "C" long long odtk_focal_loss(const float *logits, const float *target, const float *mask,
                                     const int *cls_index, long long n, int num_classes, int hw, float alpha,
                                     float gamma, float grad_scale, float *loss_elem, float *loss_sum, float *grad,
                                     void *workspace, size_t workspace_size, odtk_stream_t stream_) {
  if (n <= 0) return ODTK_E_INVALID;
  const int grid = loss_grid(n);
  const size_t need = odtk_align_up((size_t)grid * sizeof(double));
  if (!workspace || !workspace_size) return (long long)need;
  if (workspace_size < need) return ODTK_E_WORKSPACE;
  if (!logits || !loss_sum || (!target && !cls_index)) return ODTK_E_INVALID;
  if (cls_index && (num_classes <= 0 || hw <= 0 || n % ((long long)num_classes * hw))) return ODTK_E_INVALID;
  cudaStream_t stream = (cudaStream_t)stream_;
  LossParams p;
  p.logits = logits; p.target = target; p.mask = mask; p.cls_index = cls_index;
  p.n = n; p.num_classes = num_classes; p.hw = hw;
  p.alpha = alpha; p.gamma = gamma; p.grad_scale = grad_scale;
  p.loss_elem = loss_elem; p.grad = grad; p.partials = (double *)workspace;
  {
    OdtkProfScope prof(ODTK_PROF_LOSS, stream);
    focal_loss_kernel<<<grid, kThreads, 0, stream>>>(p);
  }
  focal_loss_finish_kernel<<<1, 1, 0, stream>>>(p.partials, grid, loss_sum);
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

extern "C" long long odtk_smooth_l1_loss(const float *pred, const float *target, const float *mask, long long n,
                                         float beta, float grad_scale, float *loss_elem, float *loss_sum, float *grad,
                                         void *workspace, size_t workspace_size, odtk_stream_t stream_) {
  if (n <= 0 || !(beta > 0.0f)) return ODTK_E_INVALID;
  const int grid = loss_grid(n);
  const size_t need = odtk_align_up((size_t)grid * sizeof(double));
  if (!workspace || !workspace_size) return (long long)need;
  if (workspace_size < need) return ODTK_E_WORKSPACE;
  if (!pred || !target || !loss_sum) return ODTK_E_INVALID;
  cudaStream_t stream = (cudaStream_t)stream_;
  {
    OdtkProfScope prof(ODTK_PROF_LOSS, stream);
    smooth_l1_kernel<<<grid, kThreads, 0, stream>>>(pred, target, mask, n, beta, grad_scale, loss_elem, grad,
                                                    (double *)workspace);
  }
  focal_loss_finish_kernel<<<1, 1, 0, stream>>>((const double *)workspace, grid, loss_sum);
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}

extern "C" long long odtk_retina_loss(int batch, int num_levels, const odtk_loss_level_t *levels, int num_anchors,
                                      int num_classes, int nbox, float alpha, float gamma, float beta, float *out,
                                      void *workspace, size_t workspace_size, odtk_stream_t stream_) {
  if (batch <= 0 || num_levels <= 0 || num_levels > ODTK_MAX_LEVELS || !levels || num_anchors <= 0 || num_classes <= 0)
    return ODTK_E_INVALID;
  if ((nbox != 4 && nbox != 6) || !(beta > 0.0f)) return ODTK_E_INVALID;
  int dev = 0, per_sm = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return ODTK_E_CUDA;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, retina_loss_kernel, kThreads, 0) != cudaSuccess || per_sm < 1)
    return ODTK_E_CUDA;
  if (per_sm > 4) per_sm = 4;
  const int grid = odtk_sm_count() * per_sm;               // co-resident by construction (cooperative launch checks it)
  const size_t counts_bytes = odtk_align_up(ODTK_MAX_LEVELS * sizeof(int));
  const size_t need = counts_bytes + odtk_align_up((size_t)2 * grid * sizeof(double));
  if (!workspace || !workspace_size) return (long long)need;
  if (workspace_size < need) return ODTK_E_WORKSPACE;
  if (!out) return ODTK_E_INVALID;
  RetinaParams p;
  memset(&p, 0, sizeof p);
  for (int l = 0; l < num_levels; l++) {
    const odtk_loss_level_t &s = levels[l];
    if (!s.cls_logits || !s.box_pred || !s.cls_index || !s.box_target || s.height <= 0 || s.width <= 0) return ODTK_E_INVALID;
    p.lv[l].cls_logits = (const float *)s.cls_logits; p.lv[l].box_pred = (const float *)s.box_pred;
    p.lv[l].cls_index = s.cls_index; p.lv[l].box_target = s.box_target;
    p.lv[l].cls_grad = s.cls_grad; p.lv[l].box_grad = s.box_grad;
    p.lv[l].hw = s.height * s.width;
    p.lv[l].npos = (long long)batch * num_anchors * s.height * s.width;
  }
  p.num_levels = num_levels; p.num_classes = num_classes; p.nbox = nbox;
  p.alpha = alpha; p.gamma = gamma; p.beta = beta;
  p.counts = (int *)workspace;
  p.partials = (double *)((char *)workspace + counts_bytes);
  p.out = out;
  cudaStream_t stream = (cudaStream_t)stream_;
  if (cudaMemsetAsync(p.counts, 0, ODTK_MAX_LEVELS * sizeof(int), stream) != cudaSuccess) return ODTK_E_CUDA;
  void *args[1] = {&p};
  {
    OdtkProfScope prof(ODTK_PROF_LOSS, stream);
    if (cudaLaunchCooperativeKernel((const void *)retina_loss_kernel, dim3(grid), dim3(kThreads), args, 0, stream) != cudaSuccess)
      return ODTK_E_CUDA;
  }
  return cudaGetLastError() == cudaSuccess ? ODTK_OK : ODTK_E_CUDA;
}
