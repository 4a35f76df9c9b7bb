// Per-element loss terms shared by the training losses (losses.cu) and the evaluation meters (metrics.cu), so that a
// meter reporting a loss computes it with the same device code as the criterion.
#pragma once
#include <math.h>

namespace mtt {

__device__ __forceinline__ float softplusf(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }

// BalancedBinaryCrossEntropyLoss's per-element loss (TP/losses/loss_functions.py:57-87): binary cross entropy with
// logits and pos_weight = w / (1 - w), divided by 1 / (1 - w).
__device__ __forceinline__ float balanced_bce_term(float x, float y, float w) {
  return w * y * softplusf(-x) + (1.f - w) * (1.f - y) * softplusf(x);
}

}  // namespace mtt
