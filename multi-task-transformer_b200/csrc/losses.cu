// Training-loss reductions and their gradients with respect to the predictions, on the device (SURVEY.md section 8f
// N3 "loss reductions"; the scalar N1's backward starts from). Reference: TP/losses/loss_functions.py
//   CrossEntropyLoss (ignore regions, optional binary class balancing)   :15-55   semseg, human_parts, sal
//   BalancedBinaryCrossEntropyLoss (fixed pos_weight or HED-style)       :57-87   edge
//   L1Loss (optional L2 normalisation of the prediction, ignore regions) :144-176 normals, depth
// Predictions are NCHW fp32 (the model's output layout), labels fp32 [B,Cl,H,W] as the reference's datasets give them.
//
// Every loss is two or three enqueue-only kernels and NO host synchronisation: (1) label statistics (valid count,
// negative count) into a small device state, (2) per-block partial sums of the weighted per-pixel loss, reduced in a
// FIXED order by one thread block (bitwise reproducible), which also writes the scalar loss; the gradient kernel reads
// the same state. state layout (double[8]): 0 n_valid, 1 n_neg (sum of 1 - y over valid), 2 loss sum, 3 loss value.
#include <math.h>

#include "glue.cuh"
#include "host_common.h"
#include "loss_terms.cuh"

namespace mtt {

constexpr int kLossThreads = 256;
constexpr int kLossMaxBlocks = 1024;

// ---- (1) label statistics: n_valid and sum(1 - y) over valid entries; `all_channels`: a pixel is valid when every
// channel of the label differs from ignore (L1Loss :163), counted once per pixel.
__global__ void __launch_bounds__(kLossThreads)
label_stats_kernel(const float* __restrict__ label, long long npix, int Cl, long long HW, float ignore, int all_channels,
                   double* __restrict__ partial) {
  __shared__ double sh[kLossThreads];
  double nv = 0, nn = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / HW, p = i % HW;
    bool ok = true;
    float y0 = 0.f;
    if (all_channels) {
      for (int c = 0; c < Cl; ++c) ok = ok && (label[(b * Cl + c) * HW + p] != ignore);
    } else {
      y0 = label[b * Cl * HW + p];
      ok = y0 != ignore;
    }
    if (ok) {
      nv += 1.0;
      nn += 1.0 - (double)y0;
    }
  }
  nv = block_sum(nv, sh);
  nn = block_sum(nn, sh);
  if (threadIdx.x == 0) {
    partial[2 * blockIdx.x] = nv;
    partial[2 * blockIdx.x + 1] = nn;
  }
}

__global__ void __launch_bounds__(kLossThreads)
reduce_stats_kernel(const double* __restrict__ partial, int nblocks, double* __restrict__ state) {
  __shared__ double sh[kLossThreads];
  double a = 0, b = 0;
  for (int i = threadIdx.x; i < nblocks; i += blockDim.x) {
    a += partial[2 * i];
    b += partial[2 * i + 1];
  }
  a = block_sum(a, sh);
  b = block_sum(b, sh);
  if (threadIdx.x == 0) {
    state[0] = a;
    state[1] = b;
  }
}

// mode 0: loss = sum / max(n_valid, 1) (CrossEntropyLoss :53-55, L1Loss :171); mode 1: sum / n_valid, 0 when nothing is
// valid or (hed) no positive pixel exists (BalancedBinaryCrossEntropyLoss :70-72, reduction='mean' over the kept entries)
__global__ void __launch_bounds__(kLossThreads)
reduce_loss_kernel(const double* __restrict__ partial, int nblocks, double* __restrict__ state, int mode, int hed,
                   float* __restrict__ loss_out) {
  __shared__ double sh[kLossThreads];
  double a = 0;
  for (int i = threadIdx.x; i < nblocks; i += blockDim.x) a += partial[i];
  a = block_sum(a, sh);
  if (threadIdx.x == 0) {
    const double nv = state[0];
    double v;
    if (mode == 0) v = a / (nv > 1.0 ? nv : 1.0);
    else v = (nv <= 0.0 || (hed && state[1] == nv)) ? 0.0 : a / nv;
    state[2] = a;
    state[3] = v;
    *loss_out = (float)v;
  }
}

// ---- cross entropy -------------------------------------------------------------------------------------------------
// One thread per pixel: log-softmax over C channels (stride HW), target from the label, optional binary balancing
// weights (1 - w_pos, w_pos) with w_pos = n_neg / n_valid (:32-41). GRAD: dpred = (softmax - onehot) * w[y] * gscale /
// max(n_valid, 1), zero at ignored pixels.
template <bool GRAD>
__global__ void __launch_bounds__(kLossThreads)
ce_kernel(const float* __restrict__ pred, const float* __restrict__ label, long long npix, int C, long long HW,
          float ignore, int balanced, const double* __restrict__ state, double* __restrict__ partial,
          float* __restrict__ dpred, const float* __restrict__ gscale) {
  __shared__ double sh[kLossThreads];
  double acc = 0;
  const double nv = state[0];
  const float w_pos = balanced ? (float)(state[1] / (nv > 0 ? nv : 1.0)) : 1.f;
  const float gs = GRAD ? (*gscale) / (float)(nv > 1.0 ? nv : 1.0) : 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / HW, p = i % HW;
    const float* x = pred + b * C * HW + p;
    const float yl = label[b * HW + p];
    const bool keep = yl != ignore;
    if (!keep) {
      if (GRAD)
        for (int c = 0; c < C; ++c) dpred[b * C * HW + (long long)c * HW + p] = 0.f;
      continue;
    }
    int y = (int)yl;
    y = y < 0 ? 0 : (y > C - 1 ? C - 1 : y);
    float mx = -INFINITY;
    for (int c = 0; c < C; ++c) mx = fmaxf(mx, x[(long long)c * HW]);
    float se = 0.f;
    for (int c = 0; c < C; ++c) se += expf(x[(long long)c * HW] - mx);
    const float lse = mx + logf(se);
    const float w = balanced ? (y == 1 ? w_pos : 1.f - w_pos) : 1.f;
    if (!GRAD) {
      acc += (double)(w * (lse - x[(long long)y * HW]));
    } else {
      for (int c = 0; c < C; ++c) {
        const float sm = expf(x[(long long)c * HW] - lse);
        dpred[b * C * HW + (long long)c * HW + p] = (sm - (c == y ? 1.f : 0.f)) * w * gs;
      }
    }
  }
  if (!GRAD) {
    acc = block_sum(acc, sh);
    if (threadIdx.x == 0) partial[blockIdx.x] = acc;
  }
}

// ---- balanced binary cross entropy ------------------------------------------------------------------------------------
// per = w y softplus(-x) + (1 - w)(1 - y) softplus(x) (balanced_bce_term), mean over kept entries; w = pos_weight, or
// (hed) n_neg / n_valid.

template <bool GRAD>
__global__ void __launch_bounds__(kLossThreads)
bce_kernel(const float* __restrict__ pred, const float* __restrict__ label, long long n, float ignore, float pos_weight,
           int hed, const double* __restrict__ state, double* __restrict__ partial, float* __restrict__ dpred,
           const float* __restrict__ gscale) {
  __shared__ double sh[kLossThreads];
  double acc = 0;
  const double nv = state[0];
  const float w = hed ? (float)(state[1] / (nv > 0 ? nv : 1.0)) : pos_weight;
  const bool dead = nv <= 0.0 || (hed && state[1] == nv);   // the reference returns 0 (no gradient)
  const float gs = GRAD ? (dead ? 0.f : (*gscale) / (float)nv) : 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float y = label[i], x = pred[i];
    const bool keep = y != ignore;
    if (!GRAD) {
      if (keep) acc += (double)balanced_bce_term(x, y, w);
    } else {
      const float s = 1.f / (1.f + expf(-x));
      dpred[i] = keep ? (-(w * y) * (1.f - s) + (1.f - w) * (1.f - y) * s) * gs : 0.f;
    }
  }
  if (!GRAD) {
    acc = block_sum(acc, sh);
    if (threadIdx.x == 0) partial[blockIdx.x] = acc;
  }
}

// ---- L1 (optionally on the L2-normalised prediction) ------------------------------------------------------------------
// One thread per pixel; valid when every label channel differs from ignore (or always). loss = sum_c |n_c - l_c| over
// valid pixels / max(n_valid_pixels, 1); n = x / max(||x||, 1e-12) when normalising (F.normalize).
template <bool GRAD>
__global__ void __launch_bounds__(kLossThreads)
l1_kernel(const float* __restrict__ pred, const float* __restrict__ label, long long npix, int C, long long HW,
          float ignore, int use_ignore, int normalize, const double* __restrict__ state, double* __restrict__ partial,
          float* __restrict__ dpred, const float* __restrict__ gscale) {
  __shared__ double sh[kLossThreads];
  double acc = 0;
  const double nv = state[0];
  const float gs = GRAD ? (*gscale) / (float)(nv > 1.0 ? nv : 1.0) : 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / HW, p = i % HW;
    const float* x = pred + b * C * HW + p;
    const float* l = label + b * C * HW + p;
    bool keep = true;
    if (use_ignore)
      for (int c = 0; c < C; ++c) keep = keep && (l[(long long)c * HW] != ignore);
    if (!keep) {
      if (GRAD)
        for (int c = 0; c < C; ++c) dpred[b * C * HW + (long long)c * HW + p] = 0.f;
      continue;
    }
    float r = 1.f;
    if (normalize) {
      float ss = 0.f;
      for (int c = 0; c < C; ++c) ss += x[(long long)c * HW] * x[(long long)c * HW];
      r = fmaxf(sqrtf(ss), 1e-12f);
    }
    if (!GRAD) {
      float s = 0.f;
      for (int c = 0; c < C; ++c) s += fabsf(x[(long long)c * HW] / r - l[(long long)c * HW]);
      acc += (double)s;
    } else {
      // g_c = sign(n_c - l_c); d/dx = (g - n (n . g)) / r under normalisation, g otherwise
      float ng = 0.f;
      if (normalize)
        for (int c = 0; c < C; ++c) {
          const float nc = x[(long long)c * HW] / r, d = nc - l[(long long)c * HW];
          ng += nc * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f));
        }
      for (int c = 0; c < C; ++c) {
        const float nc = x[(long long)c * HW] / r, d = nc - l[(long long)c * HW];
        const float g = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);
        dpred[b * C * HW + (long long)c * HW + p] = (normalize ? (g - nc * ng) / r : g) * gs;
      }
    }
  }
  if (!GRAD) {
    acc = block_sum(acc, sh);
    if (threadIdx.x == 0) partial[blockIdx.x] = acc;
  }
}

static int loss_blocks(long long n) {
  long long b = (n + kLossThreads - 1) / kLossThreads;
  return (int)(b < 1 ? 1 : (b > kLossMaxBlocks ? kLossMaxBlocks : b));
}

}  // namespace mtt

using namespace mtt;
#define STREAM static_cast<cudaStream_t>(stream)

extern "C" {

size_t mtt_loss_workspace_bytes(void) { return (8 + 2 * kLossMaxBlocks) * sizeof(double); }

static int loss_args(const char* what, const void* pred, const void* label, const void* ws, int B, int C, int H, int W) {
  if (!pred || !label || !ws || B <= 0 || C <= 0 || H <= 0 || W <= 0)
    return set_error(MTT_ERR_BAD_SHAPE, "%s: bad arguments (B=%d C=%d %dx%d)", what, B, C, H, W);
  if (reinterpret_cast<uintptr_t>(ws) & 7) return set_error(MTT_ERR_MISALIGNED, "%s: workspace must be 8-byte aligned", what);
  return MTT_OK;
}

int mtt_loss_cross_entropy(const float* pred, const float* label, int32_t B, int32_t C, int32_t H, int32_t W,
                           float ignore_index, int32_t balanced, float* loss_out, void* workspace,
                           mtt_stream_t stream) {
  int rc = loss_args("mtt_loss_cross_entropy", pred, label, workspace, B, C, H, W);
  if (rc) return rc;
  if (!loss_out || (balanced && C != 2))
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_loss_cross_entropy: balanced weighting is binary (C=%d)", C);
  double* state = static_cast<double*>(workspace);
  double* partial = state + 8;
  const long long HW = (long long)H * W, npix = (long long)B * HW;
  const int nb = loss_blocks(npix);
  label_stats_kernel<<<nb, kLossThreads, 0, STREAM>>>(label, npix, 1, HW, ignore_index, 0, partial);
  reduce_stats_kernel<<<1, kLossThreads, 0, STREAM>>>(partial, nb, state);
  ce_kernel<false><<<nb, kLossThreads, 0, STREAM>>>(pred, label, npix, C, HW, ignore_index, balanced, state, partial,
                                                    nullptr, nullptr);
  reduce_loss_kernel<<<1, kLossThreads, 0, STREAM>>>(partial, nb, state, 0, 0, loss_out);
  return check_launch("mtt_loss_cross_entropy");
}

int mtt_loss_cross_entropy_grad(const float* pred, const float* label, int32_t B, int32_t C, int32_t H, int32_t W,
                                float ignore_index, int32_t balanced, const float* grad_scale, float* dpred,
                                const void* workspace, mtt_stream_t stream) {
  int rc = loss_args("mtt_loss_cross_entropy_grad", pred, label, workspace, B, C, H, W);
  if (rc) return rc;
  if (!grad_scale || !dpred) return set_error(MTT_ERR_BAD_SHAPE, "mtt_loss_cross_entropy_grad: null output");
  const long long HW = (long long)H * W, npix = (long long)B * HW;
  ce_kernel<true><<<loss_blocks(npix), kLossThreads, 0, STREAM>>>(
      pred, label, npix, C, HW, ignore_index, balanced, static_cast<const double*>(workspace), nullptr, dpred, grad_scale);
  return check_launch("mtt_loss_cross_entropy_grad");
}

int mtt_loss_balanced_bce(const float* pred, const float* label, int64_t n, float ignore_index, float pos_weight,
                          int32_t hed, float* loss_out, void* workspace, mtt_stream_t stream) {
  if (!pred || !label || !loss_out || !workspace || n <= 0)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_loss_balanced_bce: bad arguments");
  double* state = static_cast<double*>(workspace);
  double* partial = state + 8;
  const int nb = loss_blocks(n);
  label_stats_kernel<<<nb, kLossThreads, 0, STREAM>>>(label, n, 1, n, ignore_index, 0, partial);
  reduce_stats_kernel<<<1, kLossThreads, 0, STREAM>>>(partial, nb, state);
  bce_kernel<false><<<nb, kLossThreads, 0, STREAM>>>(pred, label, n, ignore_index, pos_weight, hed, state, partial, nullptr,
                                                     nullptr);
  reduce_loss_kernel<<<1, kLossThreads, 0, STREAM>>>(partial, nb, state, 1, hed, loss_out);
  return check_launch("mtt_loss_balanced_bce");
}

int mtt_loss_balanced_bce_grad(const float* pred, const float* label, int64_t n, float ignore_index, float pos_weight,
                               int32_t hed, const float* grad_scale, float* dpred, const void* workspace,
                               mtt_stream_t stream) {
  if (!pred || !label || !grad_scale || !dpred || !workspace || n <= 0)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_loss_balanced_bce_grad: bad arguments");
  bce_kernel<true><<<loss_blocks(n), kLossThreads, 0, STREAM>>>(pred, label, n, ignore_index, pos_weight, hed,
                                                                static_cast<const double*>(workspace), nullptr, dpred,
                                                                grad_scale);
  return check_launch("mtt_loss_balanced_bce_grad");
}

int mtt_loss_l1(const float* pred, const float* label, int32_t B, int32_t C, int32_t H, int32_t W, float ignore_index,
                int32_t use_ignore, int32_t normalize, float* loss_out, void* workspace, mtt_stream_t stream) {
  int rc = loss_args("mtt_loss_l1", pred, label, workspace, B, C, H, W);
  if (rc) return rc;
  if (!loss_out) return set_error(MTT_ERR_BAD_SHAPE, "mtt_loss_l1: null output");
  double* state = static_cast<double*>(workspace);
  double* partial = state + 8;
  const long long HW = (long long)H * W, npix = (long long)B * HW;
  const int nb = loss_blocks(npix);
  // without ignore regions every pixel is valid: an impossible ignore value keeps the same kernels
  const float ign = use_ignore ? ignore_index : nanf("");  // NaN != y for every y: all pixels valid
  label_stats_kernel<<<nb, kLossThreads, 0, STREAM>>>(label, npix, C, HW, ign, 1, partial);
  reduce_stats_kernel<<<1, kLossThreads, 0, STREAM>>>(partial, nb, state);
  l1_kernel<false><<<nb, kLossThreads, 0, STREAM>>>(pred, label, npix, C, HW, ignore_index, use_ignore, normalize, state,
                                                    partial, nullptr, nullptr);
  reduce_loss_kernel<<<1, kLossThreads, 0, STREAM>>>(partial, nb, state, 0, 0, loss_out);
  return check_launch("mtt_loss_l1");
}

int mtt_loss_l1_grad(const float* pred, const float* label, int32_t B, int32_t C, int32_t H, int32_t W,
                     float ignore_index, int32_t use_ignore, int32_t normalize, const float* grad_scale, float* dpred,
                     const void* workspace, mtt_stream_t stream) {
  int rc = loss_args("mtt_loss_l1_grad", pred, label, workspace, B, C, H, W);
  if (rc) return rc;
  if (!grad_scale || !dpred) return set_error(MTT_ERR_BAD_SHAPE, "mtt_loss_l1_grad: null output");
  const long long HW = (long long)H * W, npix = (long long)B * HW;
  l1_kernel<true><<<loss_blocks(npix), kLossThreads, 0, STREAM>>>(pred, label, npix, C, HW, ignore_index, use_ignore,
                                                                  normalize, static_cast<const double*>(workspace),
                                                                  nullptr, dpred, grad_scale);
  return check_launch("mtt_loss_l1_grad");
}

}  // extern "C"
