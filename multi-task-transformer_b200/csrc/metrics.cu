// Evaluation meters on the device: the statistics of the reference's PerformanceMeter (TP/evaluation/*.py,
// IP/evaluation/*.py) accumulated into a caller-owned state buffer, with no host synchronisation. Each update is ONE
// enqueue-only launch on the caller's stream, so a validation loop (TP/utils/test_utils.py:29-39) can be captured in a
// CUDA graph together with predict(). get_score's formulas run on the host over one copy of the state (evaluate.py).
//
// State layout (8-byte words; mtt_meter_state_bytes):
//   CONFUSION  int64 M[(n+1)*(n+1)], M[g*(n+1)+p]: valid pixels with gt bin g and prediction bin p. Bins 0..n-1 are the
//              classes, bin n is "any other value" (a label that is neither a class nor ignore, a prediction outside
//              0..n-1), so tp/fp/fn of the reference's `==` comparisons follow exactly (eval_semseg.py:76-81).
//   SALIENCY   int64 tp[T], pp[T], ap[T] (eval_sal.py:50-60), T = n thresholds.
//   NORMALS    double sum_deg, int64 count; then the fixed-order reduction scratch.
//   DEPTH      int64 n_valid, double sum (g-p)^2, (log g - log p)^2, |g-p|/g, (g-p)^2/g; then the scratch.
//   EDGE       double sum of the per-pixel balanced BCE, int64 count; then the scratch.
// Integer counters are added with 64-bit integer atomics (exact, so order-free). Float sums are accumulated in fp64
// per CTA, written to per-CTA slots, and the last CTA to finish (ticket counter) adds the slots in block order: the
// result is bitwise reproducible for a given shape, and the ticket is back at 0 when the launch ends.
#include <math.h>

#include "glue.cuh"
#include "host_common.h"
#include "loss_terms.cuh"

namespace mtt {

constexpr int kMeterThreads = 256;
constexpr int kMeterMaxBlocks = 512;
constexpr int kMeterMaxClasses = 64;     // confusion histogram capacity: (64 + 1)^2 uint32 = 16.5 KB of shared memory
constexpr int kMeterMaxThresholds = 32;
constexpr int kMeterMaxSums = 4;

// float kinds: [header words][ticket][kMeterMaxBlocks * nsums partial doubles]
constexpr int kNormalsHeader = 2, kDepthHeader = 5, kEdgeHeader = 2;

// Adds this CTA's NS fp64 sums to sums[0..NS) in a fixed order: every CTA parks its values in its slots; the last CTA
// to arrive adds the slots of blocks 0, 1, 2, ... in turn and resets the ticket.
template <int NS>
__device__ void fixed_order_add(const double (&v)[NS], double* __restrict__ sums, unsigned int* ticket,
                                double* __restrict__ partial) {
  __shared__ bool last;
  if (threadIdx.x == 0) {
    for (int k = 0; k < NS; ++k) partial[(size_t)k * kMeterMaxBlocks + blockIdx.x] = v[k];
    __threadfence();
    last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  if (threadIdx.x < NS) {
    __threadfence();
    const double* p = partial + (size_t)threadIdx.x * kMeterMaxBlocks;
    double a = 0.0;
    for (unsigned int b = 0; b < gridDim.x; ++b) a += __ldcg(p + b);
    sums[threadIdx.x] += a;
  }
  if (threadIdx.x == 0) *ticket = 0u;
}

// ---- confusion counts (SemsegMeter eval_semseg.py:70-81, HumanPartsMeter eval_human_parts.py:33-42) -----------------
// The label's gt bin: a class 0..n-1 or n ("any other value"); fp32 maps (the transforms' [B,1,H,W]) and int64 maps
// (the Cityscapes-3D loader's [B,H,W]) compare with ignore the way torch compares them with the Python number.
__device__ __forceinline__ bool label_ignored(float g, float ignore) { return g == ignore; }
__device__ __forceinline__ bool label_ignored(long long g, float ignore) { return (double)g == (double)ignore; }
__device__ __forceinline__ int label_bin(float g, int n) { return (g >= 0.f && g < (float)n && g == floorf(g)) ? (int)g : n; }
__device__ __forceinline__ int label_bin(long long g, int n) { return (g >= 0 && g < n) ? (int)g : n; }

template <typename Label>
__global__ void __launch_bounds__(kMeterThreads)
confusion_kernel(const long long* __restrict__ pred, const Label* __restrict__ label, long long npix, int n,
                 float ignore, unsigned long long* __restrict__ M) {
  extern __shared__ unsigned int hist[];
  const int nb = n + 1, bins = nb * nb;
  for (int i = threadIdx.x; i < bins; i += blockDim.x) hist[i] = 0u;
  __syncthreads();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (long long)gridDim.x * blockDim.x) {
    const Label g = label[i];
    if (label_ignored(g, ignore)) continue;
    const long long p = pred[i];
    const int gb = label_bin(g, n);
    const int pb = (p >= 0 && p < n) ? (int)p : n;
    atomicAdd(&hist[gb * nb + pb], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < bins; i += blockDim.x)
    if (hist[i]) atomicAdd(&M[i], (unsigned long long)hist[i]);
}

// ---- saliency (SaliencyMeter eval_sal.py:21-60): prob = sigmoid(pred / 255), f_pred = prob >= thr, target long ----
__global__ void __launch_bounds__(kMeterThreads)
saliency_kernel(const float* __restrict__ pred, const float* __restrict__ label, long long npix,
                const float* __restrict__ thr, int T, float ignore, unsigned long long* __restrict__ st) {
  __shared__ unsigned long long sh[kMeterThreads];
  __shared__ float th[kMeterMaxThresholds];
  if (threadIdx.x < T) th[threadIdx.x] = thr[threadIdx.x];
  __syncthreads();
  unsigned int pp[kMeterMaxThresholds];
  long long tp[kMeterMaxThresholds];
  long long ap = 0;
#pragma unroll
  for (int k = 0; k < kMeterMaxThresholds; ++k) pp[k] = 0u, tp[k] = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (long long)gridDim.x * blockDim.x) {
    const float y = label[i];
    if (y == ignore) continue;
    const long long t = (long long)y;
    const float prob = 1.f / (1.f + expf(-(pred[i] / 255.f)));
    ap += t;
#pragma unroll
    for (int k = 0; k < kMeterMaxThresholds; ++k) {
      if (k < T && prob >= th[k]) {
        pp[k] += 1u;
        tp[k] += t;
      }
    }
  }
  unsigned long long* tp_g = st;
  unsigned long long* pp_g = st + T;
  unsigned long long* ap_g = st + 2 * T;
#pragma unroll
  for (int k = 0; k < kMeterMaxThresholds; ++k) {
    if (k < T) {   // T is uniform: every thread takes the same branches through the block sums
      const unsigned long long a = block_sum((unsigned long long)tp[k], sh);
      const unsigned long long b = block_sum((unsigned long long)pp[k], sh);
      if (threadIdx.x == 0) {
        atomicAdd(&tp_g[k], a);
        atomicAdd(&pp_g[k], b);
      }
    }
  }
  const unsigned long long a = block_sum((unsigned long long)ap, sh);
  if (threadIdx.x == 0)
    for (int k = 0; k < T; ++k) atomicAdd(&ap_g[k], a);
}

// ---- normals (NormalsMeter eval_normals.py:19-45) ------------------------------------------------------------------
// normalize_tensor: x / ||x||, and 0 where the norm is 0
__device__ __forceinline__ void normalize3(float& a, float& b, float& c) {
  const float nrm = sqrtf(a * a + b * b + c * c);
  if (nrm == 0.f) {
    a = b = c = 0.f;
  } else {
    a = a / nrm, b = b / nrm, c = c / nrm;
  }
}

__global__ void __launch_bounds__(kMeterThreads)
normals_kernel(const float* __restrict__ pred_nhwc, const float* __restrict__ label, long long npix, long long HW,
               float ignore, unsigned long long* __restrict__ st) {
  __shared__ double sh[kMeterThreads];
  __shared__ unsigned long long shu[kMeterThreads];
  double acc = 0.0;
  unsigned long long cnt = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / HW, q = i % HW;
    const float* l = label + b * 3 * HW + q;
    float g0 = l[0], g1 = l[HW], g2 = l[2 * HW];
    if (g0 == ignore || g1 == ignore || g2 == ignore) continue;
    const float* x = pred_nhwc + i * 3;
    float p0 = 2.f * x[0] / 255.f - 1.f, p1 = 2.f * x[1] / 255.f - 1.f, p2 = 2.f * x[2] / 255.f - 1.f;  // :36
    normalize3(p0, p1, p2);
    normalize3(g0, g1, g2);
    const float d0 = p0 - g0, d1 = p1 - g1, d2 = p2 - g2, s0 = p0 + g0, s1 = p1 + g1, s2 = p2 + g2;
    const float rad = 2.f * atan2f(sqrtf(d0 * d0 + d1 * d1 + d2 * d2), sqrtf(s0 * s0 + s1 * s1 + s2 * s2));
    acc += (double)(rad * (float)(180.0 / M_PI));
    cnt += 1;
  }
  const double v[1] = {block_sum(acc, sh)};
  cnt = block_sum(cnt, shu);
  if (threadIdx.x == 0) atomicAdd(&st[1], cnt);
  fixed_order_add<1>(v, reinterpret_cast<double*>(st), reinterpret_cast<unsigned int*>(st + kNormalsHeader),
                     reinterpret_cast<double*>(st + kNormalsHeader + 1));
}

// ---- depth (DepthMeter TP eval_depth.py:30-54 range mask; IP eval_depth.py DepthMeter ignore mask) ------------------
__global__ void __launch_bounds__(kMeterThreads)
depth_kernel(const float* __restrict__ pred, const float* __restrict__ label, long long npix, int use_range, float lo,
             float hi, float ignore, unsigned long long* __restrict__ st) {
  __shared__ double sh[kMeterThreads];
  __shared__ unsigned long long shu[kMeterThreads];
  double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
  unsigned long long cnt = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (long long)gridDim.x * blockDim.x) {
    float g = label[i];
    const bool ok = use_range ? (g < hi && g > lo) : (g != ignore);
    if (!ok) continue;
    float p = pred[i];
    g = g <= 0.f ? 1e-9f : g;          // :41-42, without writing the clamp back into the caller's tensors
    p = p <= 0.f ? 1e-9f : p;
    const float d = g - p, dl = logf(g) - logf(p);
    s0 += (double)(d * d);
    s1 += (double)(dl * dl);
    s2 += (double)(fabsf(d) / g);
    s3 += (double)(d * d / g);
    cnt += 1;
  }
  const double v[4] = {block_sum(s0, sh), block_sum(s1, sh), block_sum(s2, sh), block_sum(s3, sh)};
  cnt = block_sum(cnt, shu);
  if (threadIdx.x == 0) atomicAdd(&st[0], cnt);
  fixed_order_add<4>(v, reinterpret_cast<double*>(st + 1), reinterpret_cast<unsigned int*>(st + kDepthHeader),
                     reinterpret_cast<double*>(st + kDepthHeader + 1));
}

// ---- edge (EdgeMeter eval_edge.py:21-31): the balanced BCE of pred / 255 over valid pixels, weighted by their count;
// summed over pixels, sum = sum over updates of loss * numel --------------------------------------------------------
__global__ void __launch_bounds__(kMeterThreads)
edge_kernel(const float* __restrict__ pred, const float* __restrict__ label, long long npix, float pos_weight,
            float ignore, unsigned long long* __restrict__ st) {
  __shared__ double sh[kMeterThreads];
  __shared__ unsigned long long shu[kMeterThreads];
  double acc = 0.0;
  unsigned long long cnt = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (long long)gridDim.x * blockDim.x) {
    const float y = label[i];
    if (y == ignore) continue;
    acc += (double)balanced_bce_term(pred[i] / 255.f, y, pos_weight);
    cnt += 1;
  }
  const double v[1] = {block_sum(acc, sh)};
  cnt = block_sum(cnt, shu);
  if (threadIdx.x == 0) atomicAdd(&st[1], cnt);
  fixed_order_add<1>(v, reinterpret_cast<double*>(st), reinterpret_cast<unsigned int*>(st + kEdgeHeader),
                     reinterpret_cast<double*>(st + kEdgeHeader + 1));
}

static int meter_blocks(long long npix, int per_thread) {
  const long long per_block = (long long)kMeterThreads * per_thread;
  const long long b = (npix + per_block - 1) / per_block;
  return (int)(b < 1 ? 1 : (b > kMeterMaxBlocks ? kMeterMaxBlocks : b));
}

static long long meter_words(int kind, int n) {
  switch (kind) {
    case MTT_METER_CONFUSION: return (n >= 1 && n <= kMeterMaxClasses) ? (long long)(n + 1) * (n + 1) : -1;
    case MTT_METER_SALIENCY: return (n >= 1 && n <= kMeterMaxThresholds) ? 3LL * n : -1;
    case MTT_METER_NORMALS: return kNormalsHeader + 1 + kMeterMaxBlocks;
    case MTT_METER_DEPTH: return kDepthHeader + 1 + 4LL * kMeterMaxBlocks;
    case MTT_METER_EDGE: return kEdgeHeader + 1 + kMeterMaxBlocks;
    default: return -1;
  }
}

static int meter_args(const char* what, const void* pred, const void* label, const void* state, int B, int H, int W) {
  if (!pred || !label || !state || B <= 0 || H <= 0 || W <= 0)
    return set_error(MTT_ERR_BAD_SHAPE, "%s: bad arguments (B=%d %dx%d)", what, B, H, W);
  if (reinterpret_cast<uintptr_t>(state) & 7) return set_error(MTT_ERR_MISALIGNED, "%s: state must be 8-byte aligned", what);
  return MTT_OK;
}

}  // namespace mtt

using namespace mtt;
#define STREAM static_cast<cudaStream_t>(stream)
#define STATE static_cast<unsigned long long*>(state)

extern "C" {

size_t mtt_meter_state_bytes(int32_t kind, int32_t n) {
  const long long w = meter_words(kind, n);
  if (w < 0) {
    set_error(MTT_ERR_BAD_SHAPE, "mtt_meter_state_bytes: unknown kind %d or bad size %d (classes <= %d, thresholds <= %d)",
              kind, n, kMeterMaxClasses, kMeterMaxThresholds);
    return 0;
  }
  return (size_t)w * 8;
}

int mtt_meter_reset(void* state, int32_t kind, int32_t n, mtt_stream_t stream) {
  const long long w = meter_words(kind, n);
  if (w < 0)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_meter_reset: unknown kind %d or bad size %d (classes <= %d, thresholds <= %d)",
                     kind, n, kMeterMaxClasses, kMeterMaxThresholds);
  if (!state) return set_error(MTT_ERR_BAD_SHAPE, "mtt_meter_reset: null state");
  const cudaError_t e = cudaMemsetAsync(state, 0, (size_t)w * 8, STREAM);
  if (e != cudaSuccess) return set_error(MTT_ERR_LAUNCH, "mtt_meter_reset: %s", cudaGetErrorString(e));
  return MTT_OK;
}

}  // extern "C"

namespace mtt {

template <typename Label>
int confusion_update(const char* what, const int64_t* pred, const Label* label, int32_t B, int32_t H, int32_t W,
                     int32_t n_classes, float ignore_index, void* state, mtt_stream_t stream) {
  int rc = meter_args(what, pred, label, state, B, H, W);
  if (rc) return rc;
  if (n_classes < 1 || n_classes > kMeterMaxClasses)
    return set_error(MTT_ERR_BAD_SHAPE, "%s: %d classes (histogram capacity %d)", what, n_classes, kMeterMaxClasses);
  const long long npix = (long long)B * H * W;
  const size_t smem = (size_t)(n_classes + 1) * (n_classes + 1) * sizeof(unsigned int);
  confusion_kernel<Label><<<meter_blocks(npix, 16), kMeterThreads, smem, STREAM>>>(
      reinterpret_cast<const long long*>(pred), label, npix, n_classes, ignore_index, STATE);
  return check_launch(what);
}

}  // namespace mtt

extern "C" {

int mtt_meter_confusion_update(const int64_t* pred, const float* label, int32_t B, int32_t H, int32_t W,
                               int32_t n_classes, float ignore_index, void* state, mtt_stream_t stream) {
  return confusion_update("mtt_meter_confusion_update", pred, label, B, H, W, n_classes, ignore_index, state, stream);
}

int mtt_meter_confusion_update_i64(const int64_t* pred, const int64_t* label, int32_t B, int32_t H, int32_t W,
                                   int32_t n_classes, float ignore_index, void* state, mtt_stream_t stream) {
  return confusion_update("mtt_meter_confusion_update_i64", pred, reinterpret_cast<const long long*>(label), B, H, W,
                          n_classes, ignore_index, state, stream);
}

int mtt_meter_saliency_update(const float* pred, const float* label, int32_t B, int32_t H, int32_t W,
                              const float* thresholds, int32_t n_thresholds, float ignore_index, void* state,
                              mtt_stream_t stream) {
  int rc = meter_args("mtt_meter_saliency_update", pred, label, state, B, H, W);
  if (rc) return rc;
  if (!thresholds || n_thresholds < 1 || n_thresholds > kMeterMaxThresholds)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_meter_saliency_update: %d thresholds (at most %d)", n_thresholds,
                     kMeterMaxThresholds);
  const long long npix = (long long)B * H * W;
  saliency_kernel<<<meter_blocks(npix, 16), kMeterThreads, 0, STREAM>>>(pred, label, npix, thresholds, n_thresholds,
                                                                         ignore_index, STATE);
  return check_launch("mtt_meter_saliency_update");
}

int mtt_meter_normals_update(const float* pred_nhwc, const float* label, int32_t B, int32_t H, int32_t W,
                             float ignore_index, void* state, mtt_stream_t stream) {
  int rc = meter_args("mtt_meter_normals_update", pred_nhwc, label, state, B, H, W);
  if (rc) return rc;
  const long long HW = (long long)H * W, npix = B * HW;
  normals_kernel<<<meter_blocks(npix, 4), kMeterThreads, 0, STREAM>>>(pred_nhwc, label, npix, HW, ignore_index, STATE);
  return check_launch("mtt_meter_normals_update");
}

int mtt_meter_depth_update(const float* pred, const float* label, int32_t B, int32_t H, int32_t W, int32_t use_range,
                           float min_depth, float max_depth, float ignore_index, void* state, mtt_stream_t stream) {
  int rc = meter_args("mtt_meter_depth_update", pred, label, state, B, H, W);
  if (rc) return rc;
  const long long npix = (long long)B * H * W;
  depth_kernel<<<meter_blocks(npix, 4), kMeterThreads, 0, STREAM>>>(pred, label, npix, use_range ? 1 : 0, min_depth,
                                                                     max_depth, ignore_index, STATE);
  return check_launch("mtt_meter_depth_update");
}

int mtt_meter_edge_update(const float* pred, const float* label, int32_t B, int32_t H, int32_t W, float pos_weight,
                          float ignore_index, void* state, mtt_stream_t stream) {
  int rc = meter_args("mtt_meter_edge_update", pred, label, state, B, H, W);
  if (rc) return rc;
  if (!(pos_weight >= 0.f && pos_weight < 1.f))
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_meter_edge_update: pos_weight %g outside [0, 1)", (double)pos_weight);
  const long long npix = (long long)B * H * W;
  edge_kernel<<<meter_blocks(npix, 4), kMeterThreads, 0, STREAM>>>(pred, label, npix, pos_weight, ignore_index, STATE);
  return check_launch("mtt_meter_edge_update");
}

}  // extern "C"
