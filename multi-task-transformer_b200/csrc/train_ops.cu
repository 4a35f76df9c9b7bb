// Backward-pass and train-mode kernels of the TaskPrompter training step (SURVEY.md 8f N1; the loop being served is
// TaskPrompter/utils/train_utils.py:34-51). All HBM-bound: column reductions (bias / BatchNorm / LayerNorm parameter
// gradients), row-wise LayerNorm and softmax backward, the train-mode BatchNorm (batch statistics), the adjoints of the
// bilinear resize and of the spatial / channel gating, plane transposes that turn the K-major wgmma GEMM (mtt_gemm)
// into its dgrad / wgrad forms, and the fused Adam + clip step. Contractions stay on mtt_gemm / mtt_gemm_grouped.
#include "glue.cuh"
#include "host_common.h"
#include "postproc.cuh"

namespace mtt {

namespace {

__device__ __forceinline__ float act_fwd(float z, int act) {
  if (act == MTT_ACT_GELU) return gelu_erf(z);
  if (act == MTT_ACT_RELU) return fmaxf(z, 0.f);
  return z;
}
// d act(z) / dz; exact-erf GELU: Phi(z) + z * phi(z)
__device__ __forceinline__ float act_grad(float z, int act) {
  if (act == MTT_ACT_GELU) {
    const float cdf = 0.5f * (1.0f + erff(z * 0.70710678118654752440f));
    const float pdf = 0.39894228040143267794f * __expf(-0.5f * z * z);
    return cdf + z * pdf;
  }
  if (act == MTT_ACT_RELU) return z > 0.f ? 1.f : 0.f;
  return 1.f;
}

// ---- column reductions ----------------------------------------------------------------------------------------------
// out1[c] += sum_r v1(r, c), out2[c] += sum_r v2(r, c): block = 32 columns x 8 row lanes, grid.y row chunks, one atomicAdd
// per (block, column); sums in Acc (float, or double for the BatchNorm statistics). The caller zeroes the outputs unless it
// accumulates.
struct SumOp {          // bias gradients: v1 = x; logical row r = (g, i), i < in_group, at row g*src_group + src_offset + i
  const float* x; long long ld; long long in_group, src_group, src_offset;
  __device__ void operator()(long long r, int c, float& a, float& b) const {
    const long long pr = in_group > 0 ? map_row(r, in_group, src_group, src_offset) : r;   // no groups: src_offset unused
    a = x[pr * ld + c];
    b = 0.f;
  }
};
struct StatsOp {        // BatchNorm batch statistics in double: v1 = x, v2 = x^2 (exact: a float's square fits a double)
  const float* x; long long ld;
  __device__ void operator()(long long r, int c, double& a, double& b) const {
    a = (double)x[r * ld + c];
    b = a * a;
  }
};
struct BnBwdOp {        // v1 = dz, v2 = dz * xhat with dz = dy * act'(z), z = xhat * gamma + beta
  const float* x; long long ldx; const float* dy; long long lddy;
  const float* mean_rstd; const float* gamma; const float* beta; int cols; int act;
  __device__ void operator()(long long r, int c, float& a, float& b) const {
    const float xh = (x[r * ldx + c] - mean_rstd[c]) * mean_rstd[cols + c];
    const float dz = dy[r * lddy + c] * act_grad(xh * gamma[c] + beta[c], act);
    a = dz;
    b = dz * xh;
  }
};
struct LnBwdOp {        // v1 = dy (dbeta), v2 = dy * xhat (dgamma); per-row statistics from the row kernel
  const float* x; long long ldx; const float* dy; long long lddy; const float* stats;
  __device__ void operator()(long long r, int c, float& a, float& b) const {
    a = dy[r * lddy + c];
    b = a * (x[r * ldx + c] - stats[2 * r]) * stats[2 * r + 1];
  }
};

template <class Op, class Acc>
__global__ void __launch_bounds__(256)
colreduce_kernel(Op op, long long rows, int cols, Acc* __restrict__ out1, Acc* __restrict__ out2) {
  __shared__ Acc s1[8][33], s2[8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + tx;
  Acc a1 = 0, a2 = 0;
  if (c < cols) {
    for (long long r = (long long)blockIdx.y * 8 + ty; r < rows; r += (long long)gridDim.y * 8) {
      Acc u, v;
      op(r, c, u, v);
      a1 += u;
      a2 += v;
    }
  }
  s1[ty][tx] = a1;
  s2[ty][tx] = a2;
  __syncthreads();
  if (ty == 0 && c < cols) {
#pragma unroll
    for (int k = 1; k < 8; ++k) {
      a1 += s1[k][tx];
      a2 += s2[k][tx];
    }
    atomicAdd(out1 + c, a1);
    if (out2) atomicAdd(out2 + c, a2);
  }
}

template <class Op, class Acc>
int launch_colreduce(Op op, long long rows, int cols, Acc* out1, Acc* out2, cudaStream_t st, const char* what) {
  const int cb = (cols + 31) / 32;
  long long rb = (rows + 63) / 64;                       // >= 8 rows per row lane
  const long long cap = (long long)sm_count() * 8 / cb + 1;
  if (rb > cap) rb = cap;
  if (rb < 1) rb = 1;
  colreduce_kernel<Op, Acc><<<dim3(cb, (unsigned)rb), 256, 0, st>>>(op, rows, cols, out1, out2);
  return check_launch(what);
}

// ---- LayerNorm backward, one warp per row -----------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
ln_bwd_rows_kernel(const float* __restrict__ x, long long ldx, const float* __restrict__ dy, long long lddy,
                   const float* __restrict__ gamma, float eps, long long rows, int cols, float* __restrict__ dx,
                   long long lddx, int accumulate, float* __restrict__ stats) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const float* xr = x + row * ldx;
  const float* gr = dy + row * lddy;
  float s = 0.f;
  for (int c = lane; c < cols; c += 32) s += xr[c];
  const float mean = warp_sum(s) / (float)cols;
  float ss = 0.f;
  for (int c = lane; c < cols; c += 32) {
    const float a = xr[c] - mean;
    ss += a * a;
  }
  const float rstd = 1.0f / sqrtf(warp_sum(ss) / (float)cols + eps);
  float m1 = 0.f, m2 = 0.f;
  for (int c = lane; c < cols; c += 32) {
    const float g = gr[c] * gamma[c];
    m1 += g;
    m2 += g * (xr[c] - mean) * rstd;
  }
  m1 = warp_sum(m1) / (float)cols;
  m2 = warp_sum(m2) / (float)cols;
  float* o = dx + row * lddx;
  for (int c = lane; c < cols; c += 32) {
    const float xh = (xr[c] - mean) * rstd;
    float v = rstd * (gr[c] * gamma[c] - m1 - xh * m2);
    if (accumulate) v += o[c];
    o[c] = v;
  }
  if (lane == 0 && stats) {
    stats[2 * row] = mean;
    stats[2 * row + 1] = rstd;
  }
}

// ---- elementwise ------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
act_split_kernel(const float* __restrict__ pre, long long ld, long long rows, int cols, int act,
                 __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, long long ldo) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  for (int c = lane; c < cols; c += 32) store_split({hi, lo, ldo}, row, c, act_fwd(pre[row * ld + c], act));
}

__global__ void __launch_bounds__(256)
act_bwd_kernel(const float* __restrict__ pre, long long ld, const float* dy, long long lddy, long long rows,
               int cols, int act, float* dx, long long lddx) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  for (int c = lane; c < cols; c += 32) dx[row * lddx + c] = dy[row * lddy + c] * act_grad(pre[row * ld + c], act);
}

// dst[r, :] = (base ? base[r, :] : 0) + (scale ? scale[r] : 1) * src[r, :]   (residual add with per-sample DropPath scale)
__global__ void __launch_bounds__(256)
axpy_rows_kernel(const float* __restrict__ base, long long ldb, const float* __restrict__ src, long long lds,
                 const float* __restrict__ scale, long long rows, int cols, float* __restrict__ dst, long long ldd) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const float s = scale ? scale[row] : 1.f;
  for (int c = lane; c < cols; c += 32) {
    float v = s * src[row * lds + c];
    if (base) v += base[row * ldb + c];
    dst[row * ldd + c] = v;
  }
}

// ---- bf16 plane transpose [B][R][C] -> [B][C][ld_out >= R] -------------------------------------------------------------
// 64 x 64 tiles, bf16x2 loads along C and bf16x2 stores along R (128-byte rows both ways); blockIdx.z = (plane, image).
__global__ void __launch_bounds__(256)
transpose_planes_kernel(const __nv_bfloat16* __restrict__ in_hi, const __nv_bfloat16* __restrict__ in_lo, long long ld_in,
                        long long in_batch, int R, int C, __nv_bfloat16* __restrict__ out_hi,
                        __nv_bfloat16* __restrict__ out_lo, long long ld_out, long long out_batch, int B) {
  __shared__ unsigned short tile[64][66];
  const int plane = blockIdx.z / B, b = blockIdx.z % B;
  const unsigned short* ib = reinterpret_cast<const unsigned short*>(plane ? in_lo : in_hi) + (long long)b * in_batch;
  unsigned short* ob = reinterpret_cast<unsigned short*>(plane ? out_lo : out_hi) + (long long)b * out_batch;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r0 = blockIdx.y * 64, c0 = blockIdx.x * 64;
  const bool vec_in = ((ld_in & 1) == 0) && ((reinterpret_cast<uintptr_t>(ib) & 3) == 0);
  const bool vec_out = ((ld_out & 1) == 0) && ((reinterpret_cast<uintptr_t>(ob) & 3) == 0);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int r = r0 + warp * 8 + k, c = c0 + 2 * lane;
    unsigned short v0 = 0, v1 = 0;
    if (r < R && c < C) {
      const unsigned short* p = ib + (long long)r * ld_in + c;
      if (vec_in && c + 1 < C) {
        const uint32_t u = *reinterpret_cast<const uint32_t*>(p);
        v0 = (unsigned short)(u & 0xFFFF);
        v1 = (unsigned short)(u >> 16);
      } else {
        v0 = p[0];
        if (c + 1 < C) v1 = p[1];
      }
    }
    tile[warp * 8 + k][2 * lane] = v0;
    tile[warp * 8 + k][2 * lane + 1] = v1;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int c = c0 + warp * 8 + k, r = r0 + 2 * lane;
    if (c >= C || r >= R) continue;
    const unsigned short v0 = tile[2 * lane][warp * 8 + k], v1 = tile[2 * lane + 1][warp * 8 + k];
    unsigned short* p = ob + (long long)c * ld_out + r;
    if (vec_out && r + 1 < R) {
      *reinterpret_cast<uint32_t*>(p) = (uint32_t)v0 | ((uint32_t)v1 << 16);
    } else {
      p[0] = v0;
      if (r + 1 < R) p[1] = v1;
    }
  }
}

// ---- train-mode BatchNorm ----------------------------------------------------------------------------------------------
// The variance is sum x^2 / n - mean^2 formed in double: the cancellation costs ~1e-16 (mean/std)^2 of it, where the same
// subtraction over fp32 sums lost ~1e-6 (mean/std)^2 (1e-3 of the variance at mean/std = 30).
__global__ void bn_finalize_kernel(const double* __restrict__ sums, double count, int cols, float eps, float momentum,
                                   float* __restrict__ mean_rstd, float* __restrict__ running_mean,
                                   float* __restrict__ running_var) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  const double mean = sums[c] / count;
  double var = sums[cols + c] / count - mean * mean;     // biased (normalisation)
  if (var < 0.0) var = 0.0;
  mean_rstd[c] = (float)mean;
  mean_rstd[cols + c] = (float)(1.0 / sqrt(var + (double)eps));
  if (running_mean) {                                     // nn.BatchNorm2d: running_var takes the UNBIASED estimate
    const double unb = count > 1.0 ? var * count / (count - 1.0) : var;
    running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * (float)mean;
    running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unb;
  }
}

__global__ void __launch_bounds__(256)
bn_act_kernel(const float* __restrict__ x, long long ldx, long long rows, int cols, const float* __restrict__ mean_rstd,
              const float* __restrict__ gamma, const float* __restrict__ beta, int act, float* __restrict__ out_f32,
              long long ldo, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, long long ldbf) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  for (int c = lane; c < cols; c += 32) {
    const float xh = (x[row * ldx + c] - mean_rstd[c]) * mean_rstd[cols + c];
    const float y = act_fwd(xh * gamma[c] + beta[c], act);
    if (out_f32) out_f32[row * ldo + c] = y;
    if (hi) store_split({hi, lo, ldbf}, row, c, y);
  }
}

// dx = gamma * rstd * (dz - s1/count - xhat * s2/count), dz recomputed from (x, dy)
__global__ void __launch_bounds__(256)
bn_bwd_apply_kernel(const float* __restrict__ x, long long ldx, const float* __restrict__ dy, long long lddy,
                    long long rows, int cols, const float* __restrict__ mean_rstd, const float* __restrict__ gamma,
                    const float* __restrict__ beta, int act, const float* __restrict__ sums, float count,
                    float* __restrict__ dx, long long lddx) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  for (int c = lane; c < cols; c += 32) {
    const float rstd = mean_rstd[cols + c];
    const float xh = (x[row * ldx + c] - mean_rstd[c]) * rstd;
    const float dz = dy[row * lddy + c] * act_grad(xh * gamma[c] + beta[c], act);
    dx[row * lddx + c] = gamma[c] * rstd * (dz - sums[c] / count - xh * sums[cols + c] / count);
  }
}

// ---- attention backward: softmax ---------------------------------------------------------------------------------------
// P = softmax(scale * S) recomputed from the raw scores S, dS = scale * P * (dP - sum_j P dP) + d_raw on the first T rows (the
// prompt rows whose raw q.k are an output of the block, taskprompter.py:204). One block per (64 query rows, batch*head):
// phase 1 = row maximum and sum in ONE pass (warp per row; sum_j P dP comes precomputed as delta = rowdot(dO, O), the
// identity sum_j P_ij (dO_i . v_j) = dO_i . O_i), phase 2 = 64 x 64 tiles: dS is written row-major (the A operand of dQ = dS k)
// and, through a shared-memory transpose, P^T and dS^T key-major (the A operands of dV = P^T dO and dK = dS^T q) -- all as
// split planes; nothing of size N^2 is written in fp32.
__global__ void __launch_bounds__(256)
attn_softmax_bwd_kernel(const float* __restrict__ S, const float* __restrict__ dP, const float* __restrict__ delta,
                        long long ld, int N, float scale, const float* __restrict__ d_raw, int T,
                        __nv_bfloat16* __restrict__ ds_hi,
                        __nv_bfloat16* __restrict__ ds_lo, __nv_bfloat16* __restrict__ pt_hi, __nv_bfloat16* __restrict__ pt_lo,
                        __nv_bfloat16* __restrict__ dst_hi, __nv_bfloat16* __restrict__ dst_lo, long long ldbf) {
  __shared__ float stat[64][3];
  __shared__ float tp[64][65], td[64][65];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long bh = blockIdx.y;
  const int q0 = blockIdx.x * 64;
  const float* Sb = S + bh * N * ld;
  const float* Gb = dP + bh * N * ld;
  for (int k = 0; k < 8; ++k) {
    const int q = q0 + warp * 8 + k;
    if (q >= N) break;
    const float* s = Sb + (long long)q * ld;
    // one pass over the row: running maximum and rescaled sum per lane, merged across the warp
    float m = -INFINITY, l = 0.f;
    for (int j = lane; j < N; j += 32) {
      const float v = s[j] * scale;
      if (v > m) {
        l = l * __expf(m - v) + 1.f;
        m = v;
      } else {
        l += __expf(v - m);
      }
    }
    const float mw = warp_max(m);
    l = warp_sum(l * __expf(m - mw));
    if (lane == 0) {
      stat[warp * 8 + k][0] = mw;
      stat[warp * 8 + k][1] = 1.f / l;
      stat[warp * 8 + k][2] = delta[bh * N + q];
    }
  }
  __syncthreads();
  for (int k0 = 0; k0 < N; k0 += 64) {
    const int kk = k0 + 2 * lane;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int ql = warp * 8 + k, q = q0 + ql;
      float p0 = 0.f, p1 = 0.f, d0 = 0.f, d1 = 0.f;
      if (q < N && kk < N) {
        const float m = stat[ql][0], inv = stat[ql][1], dot = stat[ql][2];
        const bool two = kk + 1 < N;
        const float2 sv = two ? *reinterpret_cast<const float2*>(Sb + (long long)q * ld + kk)
                              : make_float2(Sb[(long long)q * ld + kk], 0.f);
        const float2 gv = two ? *reinterpret_cast<const float2*>(Gb + (long long)q * ld + kk)
                              : make_float2(Gb[(long long)q * ld + kk], 0.f);
        p0 = __expf(sv.x * scale - m) * inv;
        d0 = scale * p0 * (gv.x - dot);
        if (two) {
          p1 = __expf(sv.y * scale - m) * inv;
          d1 = scale * p1 * (gv.y - dot);
        }
        if (d_raw && q < T) {
          const float* dr = d_raw + (bh * T + q) * (long long)N + kk;
          d0 += dr[0];
          if (two) d1 += dr[1];
        }
        store_split2({ds_hi, ds_lo, ldbf}, bh * N + q, kk, d0, d1, two, false);
      }
      tp[ql][2 * lane] = p0;
      tp[ql][2 * lane + 1] = p1;
      td[ql][2 * lane] = d0;
      td[ql][2 * lane + 1] = d1;
    }
    __syncthreads();
    if (pt_hi) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int kl = warp * 8 + k, key = k0 + kl;
        const int q = q0 + 2 * lane;
        if (key >= N || q >= N) continue;
        const bool two = q + 1 < N;
        store_split2({pt_hi, pt_lo, ldbf}, bh * N + key, q, tp[2 * lane][kl], tp[2 * lane + 1][kl], two, false);
        store_split2({dst_hi, dst_lo, ldbf}, bh * N + key, q, td[2 * lane][kl], td[2 * lane + 1][kl], two, false);
      }
    }
    __syncthreads();
  }
}

// delta[(b*H + h)*N + i] = sum_d dO[b*N + i, h*dh + d] * O[b*N + i, h*dh + d]; O given as split planes. One warp per token row.
__global__ void __launch_bounds__(256)
attn_delta_kernel(const float* __restrict__ dO, long long lddo, const __nv_bfloat16* __restrict__ o_hi,
                  const __nv_bfloat16* __restrict__ o_lo, long long ldo, int B, int N, int H, int dh,
                  float* __restrict__ delta) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= (long long)B * N) return;
  const int lane = threadIdx.x & 31;
  const int b = (int)(row / N), i = (int)(row % N);
  for (int h = 0; h < H; ++h) {
    float acc = 0.f;
    for (int d = lane; d < dh; d += 32) {
      const long long c = (long long)h * dh + d;
      float o = __bfloat162float(o_hi[row * ldo + c]);
      if (o_lo) o += __bfloat162float(o_lo[row * ldo + c]);
      acc += dO[row * lddo + c] * o;
    }
    acc = warp_sum(acc);
    if (lane == 0) delta[((long long)b * H + h) * N + i] = acc;
  }
}

// ---- adjoint of the bilinear resize (align_corners = False, bilin_coord) -----------------------------------------------
// dy NHWC [B,H2,W2,C] (nchw = 0: one warp per output pixel, lanes over channels) or NCHW [B,C,H2,W2] (nchw = 1: one
// thread per output pixel, loop over channels); dx NHWC [B,h,w,C] accumulated with atomics (zeroed by the caller).
__global__ void __launch_bounds__(256)
bilinear_bwd_kernel(const float* __restrict__ dy, long long lddy, int nchw, int B, int h, int w, int C, int H2, int W2,
                    float sy, float sx, float* __restrict__ dx, long long lddx) {
  const long long total = (long long)B * H2 * W2;
  const long long gpix = nchw ? (long long)blockIdx.x * blockDim.x + threadIdx.x
                              : (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (gpix >= total) return;
  const int x = (int)(gpix % W2), y = (int)((gpix / W2) % H2), b = (int)(gpix / ((long long)W2 * H2));
  int y0, y1, x0, x1;
  float ly, lx;
  bilin_coord(y, sy, h, y0, y1, ly);
  bilin_coord(x, sx, w, x0, x1, lx);
  const float hy = 1.f - ly, hx = 1.f - lx;
  float* ob = dx + (long long)b * h * w * lddx;
  float* p00 = ob + ((long long)y0 * w + x0) * lddx;
  float* p01 = ob + ((long long)y0 * w + x1) * lddx;
  float* p10 = ob + ((long long)y1 * w + x0) * lddx;
  float* p11 = ob + ((long long)y1 * w + x1) * lddx;
  if (nchw) {
    const long long plane = (long long)H2 * W2;
    const float* src = dy + (long long)b * C * plane + (long long)y * W2 + x;
    for (int c = 0; c < C; ++c) {
      const float g = src[c * plane];
      atomicAdd(p00 + c, hy * hx * g);
      atomicAdd(p01 + c, hy * lx * g);
      atomicAdd(p10 + c, ly * hx * g);
      atomicAdd(p11 + c, ly * lx * g);
    }
  } else {
    const int lane = threadIdx.x & 31;
    const float* src = dy + gpix * lddy;
    for (int c = lane; c < C; c += 32) {
      const float g = src[c];
      atomicAdd(p00 + c, hy * hx * g);
      atomicAdd(p01 + c, hy * lx * g);
      atomicAdd(p10 + c, ly * hx * g);
      atomicAdd(p11 + c, ly * lx * g);
    }
  }
}

// ---- adjoint of the spatial / channel gating (mtt_gate_split) -----------------------------------------------------------
// Ys = X (1 + g_s), Yc = X (1 + g_c): dX += dYs (1 + g_s) + dYc (1 + g_c);
// d prompt_logits[b, head, t, T + pix] += sum_{c in head} dYs X;  d chan_logits[b, t, c, window] += sum_{pix in window} dYc X.
// One warp per (b, pixel) for dX and the spatial logits; the channel logits are a column reduction over the pixels of a
// window (gate_chan_bwd_kernel: one block per (column block, image, window), single writer, no atomics).
__global__ void __launch_bounds__(256)
gate_bwd_kernel(const float* __restrict__ x, long long ldx, long long x_group_rows, long long x_row_offset,
                const float* __restrict__ plog, const float* __restrict__ clog, int task, int B, int T, int N, int H,
                int C, int gh, int gw, int nh, int nw, const float* __restrict__ dys, const float* __restrict__ dyc,
                long long lddy, float* __restrict__ dx, long long lddx, float* __restrict__ d_plog) {
  const long long P = (long long)gh * gw;
  const long long gp = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (gp >= (long long)B * P) return;
  const int lane = threadIdx.x & 31;
  const int b = (int)(gp / P), pix = (int)(gp % P);
  const int win = chan_window(pix, gh, gw, nh, nw);
  const int dh = C / H;
  const long long xrow = (long long)b * x_group_rows + x_row_offset + pix;
  const float* xr = x + xrow * ldx;
  float* dxr = dx + xrow * lddx;
  const float* gs = dys + gp * lddy;
  const float* gc = dyc + gp * lddy;
  const float* cl = clog + (((long long)b * T + task) * C) * (nh * nw) + win;
  for (int hd = 0; hd < H; ++hd) {
    const long long li = (((long long)b * H + hd) * T + task) * N + T + pix;
    const float g = plog[li];
    float acc = 0.f;
    for (int c = hd * dh + lane; c < (hd + 1) * dh; c += 32) {
      const float xv = xr[c];
      const float a = gs[c], e = gc[c];
      acc += a * xv;
      dxr[c] += a * (1.f + g) + e * (1.f + cl[(long long)c * (nh * nw)]);
    }
    acc = warp_sum(acc);
    if (lane == 0) d_plog[li] += acc;
  }
}

__global__ void __launch_bounds__(256)
gate_chan_bwd_kernel(const float* __restrict__ x, long long ldx, long long x_group_rows, long long x_row_offset, int task,
                     int T, int C, int gh, int gw, int nh, int nw, const float* __restrict__ dyc, long long lddy,
                     float* __restrict__ d_clog) {
  __shared__ float sh[8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + tx;
  const int nwin = nh * nw, b = blockIdx.y / nwin, win = blockIdx.y % nwin;
  const int wh = gh / nh, ww = gw / nw, wy = win / nw, wx = win % nw;
  float acc = 0.f;
  if (c < C) {
    for (int k = ty; k < wh * ww; k += 8) {
      const int pix = (wy * wh + k / ww) * gw + wx * ww + k % ww;
      const long long xrow = (long long)b * x_group_rows + x_row_offset + pix;
      acc += dyc[((long long)b * gh * gw + pix) * lddy + c] * x[xrow * ldx + c];
    }
  }
  sh[ty][tx] = acc;
  __syncthreads();
  if (ty == 0 && c < C) {
#pragma unroll
    for (int k = 1; k < 8; ++k) acc += sh[k][tx];
    d_clog[(((long long)b * T + task) * C + c) * nwin + win] += acc;
  }
}

// ---- adjoint of the raw channel logits (mtt_chan_logits) ----------------------------------------------------------------
// Rc[b,t,c,win] = sum_{pix in win} cp[b,t,pix] xn[b,pix,c]:
// dcp[b,t,pix] = sum_c dRc[b,t,c,win(pix)] xn[b,pix,c];  dxn[b,pix,c] += sum_t dRc[b,t,c,win(pix)] cp[b,t,pix].
// xn is given as split planes of the joint stream (patch rows start at row T of every image). One warp per (b, pixel).
__global__ void __launch_bounds__(256)
chan_logits_bwd_kernel(const float* __restrict__ d_rc, const float* __restrict__ cp, const __nv_bfloat16* __restrict__ xn_hi,
                       const __nv_bfloat16* __restrict__ xn_lo, long long ldx, int B, int N, int T, int C, int gh, int gw,
                       int nh, int nw, float* __restrict__ dcp, float* __restrict__ dxn, long long lddx) {
  const long long P = (long long)gh * gw;
  const long long gp = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (gp >= (long long)B * P) return;
  const int lane = threadIdx.x & 31;
  const int b = (int)(gp / P), pix = (int)(gp % P);
  const int win = chan_window(pix, gh, gw, nh, nw);
  const int nwin = nh * nw;
  const long long row = (long long)b * N + T + pix;
  for (int t = 0; t < T; ++t) {
    const float* dr = d_rc + (((long long)b * T + t) * C) * nwin + win;
    const float cpv = cp[((long long)b * T + t) * P + pix];
    float acc = 0.f;
    for (int c = lane; c < C; c += 32) {
      float xv = __bfloat162float(xn_hi[row * ldx + c]);
      if (xn_lo) xv += __bfloat162float(xn_lo[row * ldx + c]);
      const float g = dr[(long long)c * nwin];
      acc += g * xv;
      dxn[row * lddx + c] += g * cpv;
    }
    acc = warp_sum(acc);
    if (lane == 0) dcp[((long long)b * T + t) * P + pix] = acc;
  }
}

// ---- cross-task reweighting backward (mtt_ctr_weights / mtt_ctr_mix) ---------------------------------------------------
// dw[b, t, j] = sum_{m in image b, c} dnew[t][m, c] * F[j][m, c]: grid (T*T, B, chunks), block reduction + atomicAdd.
__global__ void __launch_bounds__(256)
ctr_dw_kernel(const float* __restrict__ dnew, const float* __restrict__ F, int T, long long M, int C, long long ld,
              int rows_per_batch, float* __restrict__ dw) {
  const int t = blockIdx.x / T, j = blockIdx.x % T, b = blockIdx.y;
  const float* a = dnew + ((long long)t * M + (long long)b * rows_per_batch) * ld;
  const float* f = F + ((long long)j * M + (long long)b * rows_per_batch) * ld;
  float acc = 0.f;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long r = (long long)blockIdx.z * 8 + warp; r < rows_per_batch; r += (long long)gridDim.z * 8)
    for (int c = lane; c < C; c += 32) acc += a[r * ld + c] * f[r * ld + c];
  acc = warp_sum(acc);
  __shared__ float sh[8];
  if (lane == 0) sh[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int k = 0; k < 8; ++k) s += sh[k];
    atomicAdd(dw + ((long long)b * T + t) * T + j, s);
  }
}

// The two 1x1 convs around a GELU that make w from the prompt-prompt affinities (taskprompter.py:478-482), backward:
// w[b,t,j] = W2_t . gelu(W0_t . a + b0_t) + b2_t with a[h] = R[b,h,t,j]. One thread per (b, t, j); parameter gradients by
// atomics (tiny: T*H*H values).
__global__ void ctr_weights_bwd_kernel(const float* __restrict__ plog, int B, int H, int T, int N,
                                       const float* __restrict__ w0, const float* __restrict__ b0,
                                       const float* __restrict__ w2, const float* __restrict__ dw,
                                       float* __restrict__ d_plog, float* __restrict__ dw0, float* __restrict__ db0,
                                       float* __restrict__ dw2, float* __restrict__ db2) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * T * T) return;
  const int j = idx % T, t = (idx / T) % T, b = idx / (T * T);
  const float g = dw[idx];
  atomicAdd(db2 + t, g);
  for (int h = 0; h < H; ++h) {
    float z = b0[t * H + h];
    for (int k = 0; k < H; ++k) z += w0[((long long)t * H + h) * H + k] * plog[(((long long)b * H + k) * T + t) * N + j];
    atomicAdd(dw2 + t * H + h, g * act_fwd(z, MTT_ACT_GELU));
    const float dz = g * w2[t * H + h] * act_grad(z, MTT_ACT_GELU);
    atomicAdd(db0 + t * H + h, dz);
    for (int k = 0; k < H; ++k) {
      const long long li = (((long long)b * H + k) * T + t) * N + j;
      atomicAdd(dw0 + ((long long)t * H + h) * H + k, dz * plog[li]);
      atomicAdd(d_plog + li, dz * w0[((long long)t * H + h) * H + k]);
    }
  }
}

// ---- weight-gradient operands of the convolutions ----------------------------------------------------------------------
// 3x3 (pad 1) im2col, transposed and split: out[(c*9 + ky*3 + kx), p] = x[b, y+ky-1, x+kx-1, c] (0 outside), p = pixel
// index over [B,H,W]; rows in nn.Conv2d's weight order so that dW = dY^T . out^T is [Cout, Cin*9] = weight.view(Cout,-1).
// One block = 64 consecutive pixels x 32 channels, all nine taps: per tap the shifted [64 x 32] slab goes through a
// shared-memory tile (loads coalesced along channels, neighbouring taps hit L1 / L2) and leaves as 128-byte rows of 64
// pixels (one bf16x2 per lane), instead of one 32 x 32 tile of ONE tap per block with 2-byte stores, which wrote the
// 825 MB operand of a 350-channel 128 x 128 map at batch 4 at a small fraction of the plain fill rate.
__global__ void __launch_bounds__(256)
im2col3x3_t_kernel(const float* __restrict__ x, long long ldx, int B, int H, int W, int C, __nv_bfloat16* __restrict__ hi,
                   __nv_bfloat16* __restrict__ lo, long long ldo, int vec_out) {
  __shared__ float tile[64][33];
  const long long Ptot = (long long)B * H * W;
  const long long p0 = (long long)blockIdx.x * 64;
  const int c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  // the eight pixels this thread loads (rows ty*8 .. ty*8+7 of the tile), channel c0 + tx
  int px[8], py[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const long long p = p0 + ty * 8 + k;
    if (p < Ptot) {
      px[k] = (int)(p % W);
      py[k] = (int)((p / W) % H);
    } else {
      px[k] = py[k] = -1000000;   // never in bounds
    }
  }
  const bool c_ok = c0 + tx < C;
  const float* xc = x + c0 + tx;
  for (int tap = 0; tap < 9; ++tap) {
    const int dy = tap / 3 - 1, dx = tap % 3 - 1;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int sy = py[k] + dy, sx = px[k] + dx;
      float v = 0.f;
      if (c_ok && sy >= 0 && sy < H && sx >= 0 && sx < W) v = xc[(p0 + ty * 8 + k + (long long)dy * W + dx) * ldx];
      tile[ty * 8 + k][tx] = v;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = c0 + ty * 4 + k;
      const long long p = p0 + 2 * tx;
      if (c < C && p < Ptot) {
        uint32_t hh, ll;
        split_pack2(tile[2 * tx][ty * 4 + k], tile[2 * tx + 1][ty * 4 + k], hh, ll);
        const long long o = ((long long)c * 9 + tap) * ldo + p;
        if (vec_out && p + 1 < Ptot) {
          *reinterpret_cast<uint32_t*>(hi + o) = hh;
          if (lo) *reinterpret_cast<uint32_t*>(lo + o) = ll;
        } else {
          hi[o] = __ushort_as_bfloat16((unsigned short)(hh & 0xFFFF));
          if (lo) lo[o] = __ushort_as_bfloat16((unsigned short)(ll & 0xFFFF));
          if (p + 1 < Ptot) {
            hi[o + 1] = __ushort_as_bfloat16((unsigned short)(hh >> 16));
            if (lo) lo[o + 1] = __ushort_as_bfloat16((unsigned short)(ll >> 16));
          }
        }
      }
    }
    __syncthreads();
  }
}

// Patch-embedding im2col, transposed: out[(c, ky, kx), (b, py, px)] = img[b, c, py*patch + ky, px*patch + kx].
__global__ void __launch_bounds__(256)
im2col_patch_t_kernel(const float* __restrict__ img, int B, int Cin, int H, int W, int patch,
                      __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, long long ldo) {
  const int gh = H / patch, gw = W / patch;
  const long long cols = (long long)B * gh * gw;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)Cin * patch * patch * cols;
  if (idx >= total) return;
  const long long col = idx % cols;
  const int row = (int)(idx / cols);
  const int kx = row % patch, ky = (row / patch) % patch, c = row / (patch * patch);
  const int px = (int)(col % gw), py = (int)((col / gw) % gh), b = (int)(col / ((long long)gw * gh));
  const float v = img[(((long long)b * Cin + c) * H + py * patch + ky) * W + px * patch + kx];
  store_split({hi, lo, ldo}, row, col, v);
}

// ---- optimiser ----------------------------------------------------------------------------------------------------------
// sum of squares of a flat buffer into *out (atomic; the caller zeroes it)
__global__ void __launch_bounds__(256) sumsq_kernel(const float* __restrict__ g, long long n, float* __restrict__ out) {
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    acc += g[i] * g[i];
  acc = warp_sum(acc);
  __shared__ float sh[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) sh[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int k = 0; k < 8; ++k) s += sh[k];
    atomicAdd(out, s);
  }
}

// torch.optim.Adam (L2 weight decay added to the gradient, bias correction) behind clip_grad_norm_ (max_norm / (norm + 1e-6),
// clamped to 1): p, g, m, v flat fp32 arenas; gnorm_sq = sum of squared gradients (device scalar) or NULL = no clipping.
__global__ void __launch_bounds__(256)
adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, long long n,
            float lr, float beta1, float beta2, float omb1, float omb2, float eps, float wd, float bc1, float bc2,
            const float* __restrict__ gnorm_sq, float max_norm, float grad_scale) {
  float clip = grad_scale;
  if (gnorm_sq) {
    const float nrm = sqrtf(*gnorm_sq) * grad_scale;
    const float c = max_norm / (nrm + 1e-6f);
    clip *= c < 1.f ? c : 1.f;
  }
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float gi = g[i] * clip + wd * p[i];
    const float mi = beta1 * m[i] + omb1 * gi;
    const float vi = beta2 * v[i] + omb2 * gi * gi;
    m[i] = mi;
    v[i] = vi;
    p[i] -= lr / bc1 * mi / (sqrtf(vi) / sqrtf(bc2) + eps);
  }
}

inline unsigned row_blocks(long long rows) { return (unsigned)((rows + 7) / 8); }

}  // namespace

}  // namespace mtt

using namespace mtt;
#define ST static_cast<cudaStream_t>(stream)

extern "C" int mtt_colsum(const float* x, int64_t ldx, int64_t rows, int32_t cols, int64_t in_group, int64_t src_group,
                          int64_t src_offset, float* out, int32_t accumulate, mtt_stream_t stream) {
  if (!x || !out || rows <= 0 || cols <= 0) return set_error(MTT_ERR_BAD_SHAPE, "mtt_colsum: bad arguments");
  if (!accumulate) cudaMemsetAsync(out, 0, sizeof(float) * cols, ST);
  return launch_colreduce(SumOp{x, ldx, in_group, src_group, src_offset}, rows, cols, out, (float*)nullptr, ST,
                          "mtt_colsum");
}

extern "C" int mtt_layernorm_bwd(const float* x, int64_t ldx, const float* dy, int64_t lddy, const float* gamma, float eps,
                                 int64_t rows, int32_t cols, float* dx, int64_t lddx, int32_t accumulate_dx, float* dgamma,
                                 float* dbeta, float* stats_ws, mtt_stream_t stream) {
  if (!x || !dy || !gamma || !dx || !stats_ws || rows <= 0 || cols <= 0)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_layernorm_bwd: bad arguments");
  ln_bwd_rows_kernel<<<row_blocks(rows), 256, 0, ST>>>(x, ldx, dy, lddy, gamma, eps, rows, cols, dx, lddx, accumulate_dx,
                                                       stats_ws);
  int rc = check_launch("mtt_layernorm_bwd(rows)");
  if (rc || !dgamma) return rc;
  return launch_colreduce(LnBwdOp{x, ldx, dy, lddy, stats_ws}, rows, cols, dbeta, dgamma, ST, "mtt_layernorm_bwd(cols)");
}

extern "C" int mtt_act_split(const float* pre, int64_t ld, int64_t rows, int32_t cols, int32_t act, void* out_hi,
                             void* out_lo, int64_t ldo, mtt_stream_t stream) {
  if (!pre || !out_hi || rows <= 0 || cols <= 0) return set_error(MTT_ERR_BAD_SHAPE, "mtt_act_split: bad arguments");
  act_split_kernel<<<row_blocks(rows), 256, 0, ST>>>(pre, ld, rows, cols, act, static_cast<__nv_bfloat16*>(out_hi),
                                                     static_cast<__nv_bfloat16*>(out_lo), ldo);
  return check_launch("mtt_act_split");
}

extern "C" int mtt_act_bwd(const float* pre, int64_t ld, const float* dy, int64_t lddy, int64_t rows, int32_t cols,
                           int32_t act, float* dx, int64_t lddx, mtt_stream_t stream) {
  if (!pre || !dy || !dx || rows <= 0 || cols <= 0) return set_error(MTT_ERR_BAD_SHAPE, "mtt_act_bwd: bad arguments");
  act_bwd_kernel<<<row_blocks(rows), 256, 0, ST>>>(pre, ld, dy, lddy, rows, cols, act, dx, lddx);
  return check_launch("mtt_act_bwd");
}

extern "C" int mtt_axpy_rows(const float* base, int64_t ldb, const float* src, int64_t lds, const float* row_scale,
                             int64_t rows, int32_t cols, float* dst, int64_t ldd, mtt_stream_t stream) {
  if (!src || !dst || rows <= 0 || cols <= 0) return set_error(MTT_ERR_BAD_SHAPE, "mtt_axpy_rows: bad arguments");
  axpy_rows_kernel<<<row_blocks(rows), 256, 0, ST>>>(base, ldb, src, lds, row_scale, rows, cols, dst, ldd);
  return check_launch("mtt_axpy_rows");
}

extern "C" int mtt_transpose_planes(const void* in_hi, const void* in_lo, int64_t ld_in, int64_t in_batch_rows, int32_t B,
                                    int32_t R, int32_t C, void* out_hi, void* out_lo, int64_t ld_out,
                                    int64_t out_batch_stride, mtt_stream_t stream) {
  if (!in_hi || !out_hi || B <= 0 || R <= 0 || C <= 0 || ld_out < R)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_transpose_planes: bad arguments");
  const int planes = (in_lo && out_lo) ? 2 : 1;
  const dim3 grid((C + 63) / 64, (R + 63) / 64, B * planes);
  const long long ib = in_batch_rows * ld_in, ob = out_batch_stride > 0 ? out_batch_stride : (long long)C * ld_out;
  transpose_planes_kernel<<<grid, 256, 0, ST>>>(static_cast<const __nv_bfloat16*>(in_hi),
                                               static_cast<const __nv_bfloat16*>(in_lo), ld_in, ib, R, C,
                                               static_cast<__nv_bfloat16*>(out_hi), static_cast<__nv_bfloat16*>(out_lo),
                                               ld_out, ob, B);
  return check_launch("mtt_transpose_planes");
}

extern "C" int mtt_bn_stats(const float* x, int64_t ldx, int64_t rows, int32_t cols, double* sums, mtt_stream_t stream) {
  if (!x || !sums || rows <= 0 || cols <= 0) return set_error(MTT_ERR_BAD_SHAPE, "mtt_bn_stats: bad arguments");
  cudaMemsetAsync(sums, 0, sizeof(double) * 2 * cols, ST);
  return launch_colreduce(StatsOp{x, ldx}, rows, cols, sums, sums + cols, ST, "mtt_bn_stats");
}

extern "C" int mtt_bn_finalize(const double* sums, double count, int32_t cols, float eps, float momentum,
                               float* mean_rstd, float* running_mean, float* running_var, mtt_stream_t stream) {
  if (!sums || !mean_rstd || cols <= 0 || count <= 0.0) return set_error(MTT_ERR_BAD_SHAPE, "mtt_bn_finalize: bad arguments");
  bn_finalize_kernel<<<(cols + 127) / 128, 128, 0, ST>>>(sums, count, cols, eps, momentum, mean_rstd, running_mean,
                                                         running_var);
  return check_launch("mtt_bn_finalize");
}

extern "C" int mtt_bn_act(const float* x, int64_t ldx, int64_t rows, int32_t cols, const float* mean_rstd,
                          const float* gamma, const float* beta, int32_t act, float* out_f32, int64_t ldo, void* out_hi,
                          void* out_lo, int64_t ldbf, mtt_stream_t stream) {
  if (!x || !mean_rstd || !gamma || !beta || (!out_f32 && !out_hi) || rows <= 0 || cols <= 0)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_bn_act: bad arguments");
  bn_act_kernel<<<row_blocks(rows), 256, 0, ST>>>(x, ldx, rows, cols, mean_rstd, gamma, beta, act, out_f32, ldo,
                                                  static_cast<__nv_bfloat16*>(out_hi), static_cast<__nv_bfloat16*>(out_lo),
                                                  ldbf);
  return check_launch("mtt_bn_act");
}

extern "C" int mtt_bn_bwd_reduce(const float* x, int64_t ldx, const float* dy, int64_t lddy, int64_t rows, int32_t cols,
                                 const float* mean_rstd, const float* gamma, const float* beta, int32_t act, float* sums,
                                 mtt_stream_t stream) {
  if (!x || !dy || !mean_rstd || !gamma || !beta || !sums || rows <= 0 || cols <= 0)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_bn_bwd_reduce: bad arguments");
  cudaMemsetAsync(sums, 0, sizeof(float) * 2 * cols, ST);
  return launch_colreduce(BnBwdOp{x, ldx, dy, lddy, mean_rstd, gamma, beta, cols, act}, rows, cols, sums, sums + cols, ST,
                          "mtt_bn_bwd_reduce");
}

extern "C" int mtt_bn_bwd_apply(const float* x, int64_t ldx, const float* dy, int64_t lddy, int64_t rows, int32_t cols,
                                const float* mean_rstd, const float* gamma, const float* beta, int32_t act,
                                const float* sums, float count, float* dx, int64_t lddx, mtt_stream_t stream) {
  if (!x || !dy || !mean_rstd || !gamma || !beta || !sums || !dx || rows <= 0 || cols <= 0 || count <= 0.f)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_bn_bwd_apply: bad arguments");
  bn_bwd_apply_kernel<<<row_blocks(rows), 256, 0, ST>>>(x, ldx, dy, lddy, rows, cols, mean_rstd, gamma, beta, act, sums,
                                                        count, dx, lddx);
  return check_launch("mtt_bn_bwd_apply");
}

extern "C" int mtt_attn_delta(const float* dO, int64_t lddo, const void* o_hi, const void* o_lo, int64_t ldo, int32_t B,
                              int32_t N, int32_t H, int32_t head_dim, float* delta, mtt_stream_t stream) {
  if (!dO || !o_hi || !delta || B <= 0 || N <= 0 || H <= 0 || head_dim <= 0)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_attn_delta: bad arguments");
  attn_delta_kernel<<<row_blocks((long long)B * N), 256, 0, ST>>>(dO, lddo, static_cast<const __nv_bfloat16*>(o_hi),
                                                                static_cast<const __nv_bfloat16*>(o_lo), ldo, B, N, H,
                                                                head_dim, delta);
  return check_launch("mtt_attn_delta");
}

extern "C" int mtt_attn_softmax_bwd(const float* S, const float* dP, const float* delta, int64_t ld, int32_t BH, int32_t N,
                                    float scale, const float* d_raw, int32_t T, void* ds_hi, void* ds_lo, void* pt_hi,
                                    void* pt_lo, void* dst_hi, void* dst_lo, int64_t ldbf, mtt_stream_t stream) {
  if (!S || !dP || !delta || !ds_hi || BH <= 0 || N <= 0 || ld < N || ldbf < N || ld % 2 || ldbf % 2 || (pt_hi && !dst_hi))
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_attn_softmax_bwd: bad arguments");
  if ((reinterpret_cast<uintptr_t>(S) & 7) || (reinterpret_cast<uintptr_t>(dP) & 7))
    return set_error(MTT_ERR_MISALIGNED, "mtt_attn_softmax_bwd: S / dP must be 8-byte aligned");
  attn_softmax_bwd_kernel<<<dim3((N + 63) / 64, BH), 256, 0, ST>>>(
      S, dP, delta, ld, N, scale, d_raw, T, static_cast<__nv_bfloat16*>(ds_hi), static_cast<__nv_bfloat16*>(ds_lo),
      static_cast<__nv_bfloat16*>(pt_hi), static_cast<__nv_bfloat16*>(pt_lo), static_cast<__nv_bfloat16*>(dst_hi),
      static_cast<__nv_bfloat16*>(dst_lo), ldbf);
  return check_launch("mtt_attn_softmax_bwd");
}

extern "C" int mtt_bilinear_bwd(const float* dy, int64_t lddy, int32_t nchw, int32_t B, int32_t h, int32_t w, int32_t C,
                                int32_t H2, int32_t W2, float* dx, int64_t lddx, int32_t accumulate, mtt_stream_t stream) {
  if (!dy || !dx || B <= 0 || h <= 0 || w <= 0 || C <= 0 || H2 <= 0 || W2 <= 0)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_bilinear_bwd: bad arguments");
  if (!accumulate) cudaMemset2DAsync(dx, sizeof(float) * lddx, 0, sizeof(float) * C, (size_t)B * h * w, ST);
  const long long total = (long long)B * H2 * W2;
  const unsigned blocks = nchw ? (unsigned)((total + 255) / 256) : row_blocks(total);
  bilinear_bwd_kernel<<<blocks, 256, 0, ST>>>(dy, lddy, nchw, B, h, w, C, H2, W2, (float)h / H2, (float)w / W2, dx, lddx);
  return check_launch("mtt_bilinear_bwd");
}

extern "C" int mtt_gate_bwd(const float* x, int64_t ldx, int64_t x_group_rows, int64_t x_row_offset,
                            const float* prompt_logits, const float* chan_logits, int32_t task, int32_t B, int32_t T,
                            int32_t N, int32_t H, int32_t C, int32_t gh, int32_t gw, int32_t nh, int32_t nw,
                            const float* dys, const float* dyc, int64_t lddy, float* dx, int64_t lddx,
                            float* d_prompt_logits, float* d_chan_logits, mtt_stream_t stream) {
  if (!x || !prompt_logits || !chan_logits || !dys || !dyc || !dx || !d_prompt_logits || !d_chan_logits || B <= 0 ||
      C % H || gh % nh || gw % nw)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_gate_bwd: bad arguments");
  gate_bwd_kernel<<<row_blocks((long long)B * gh * gw), 256, 0, ST>>>(x, ldx, x_group_rows, x_row_offset, prompt_logits,
                                                                    chan_logits, task, B, T, N, H, C, gh, gw, nh, nw, dys,
                                                                    dyc, lddy, dx, lddx, d_prompt_logits);
  gate_chan_bwd_kernel<<<dim3((C + 31) / 32, B * nh * nw), 256, 0, ST>>>(x, ldx, x_group_rows, x_row_offset, task, T, C, gh,
                                                                        gw, nh, nw, dyc, lddy, d_chan_logits);
  return check_launch("mtt_gate_bwd");
}

extern "C" int mtt_chan_logits_bwd(const float* d_rc, const float* cp, const void* xn_hi, const void* xn_lo, int64_t ldx,
                                   int32_t B, int32_t N, int32_t T, int32_t C, int32_t gh, int32_t gw, int32_t nh,
                                   int32_t nw, float* dcp, float* dxn, int64_t lddx, mtt_stream_t stream) {
  if (!d_rc || !cp || !xn_hi || !dcp || !dxn || B <= 0 || gh % nh || gw % nw)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_chan_logits_bwd: bad arguments");
  chan_logits_bwd_kernel<<<row_blocks((long long)B * gh * gw), 256, 0, ST>>>(
      d_rc, cp, static_cast<const __nv_bfloat16*>(xn_hi), static_cast<const __nv_bfloat16*>(xn_lo), ldx, B, N, T, C, gh, gw,
      nh, nw, dcp, dxn, lddx);
  return check_launch("mtt_chan_logits_bwd");
}

extern "C" int mtt_ctr_bwd(const float* dnew, const float* F, int32_t T, int64_t M, int32_t C, int64_t ld,
                           int32_t rows_per_batch, const float* prompt_logits, int32_t B, int32_t H, int32_t N,
                           const float* w0, const float* b0, const float* w2, float* dw_ws, float* d_prompt_logits,
                           float* dw0, float* db0, float* dw2, float* db2, mtt_stream_t stream) {
  if (!dnew || !F || !prompt_logits || !w0 || !b0 || !w2 || !dw_ws || !d_prompt_logits || !dw0 || !db0 || !dw2 || !db2 ||
      T <= 0 || B <= 0 || M != (int64_t)B * rows_per_batch)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_ctr_bwd: bad arguments");
  cudaMemsetAsync(dw_ws, 0, sizeof(float) * B * T * T, ST);
  int chunks = (rows_per_batch + 63) / 64;
  if (chunks > 32) chunks = 32;
  ctr_dw_kernel<<<dim3(T * T, B, chunks), 256, 0, ST>>>(dnew, F, T, M, C, ld, rows_per_batch, dw_ws);
  ctr_weights_bwd_kernel<<<(B * T * T + 63) / 64, 64, 0, ST>>>(prompt_logits, B, H, T, N, w0, b0, w2, dw_ws,
                                                               d_prompt_logits, dw0, db0, dw2, db2);
  return check_launch("mtt_ctr_bwd");
}

extern "C" int mtt_im2col3x3_t(const float* x, int64_t ldx, int32_t B, int32_t H, int32_t W, int32_t C, void* out_hi,
                               void* out_lo, int64_t ldo, mtt_stream_t stream) {
  const long long P = (long long)B * H * W;
  if (!x || !out_hi || P <= 0 || C <= 0 || ldo < P) return set_error(MTT_ERR_BAD_SHAPE, "mtt_im2col3x3_t: bad arguments");
  const int cb = (C + 31) / 32;
  const int vec_out = (ldo % 2 == 0) && (reinterpret_cast<uintptr_t>(out_hi) % 4 == 0) &&
                      (!out_lo || reinterpret_cast<uintptr_t>(out_lo) % 4 == 0);
  im2col3x3_t_kernel<<<dim3((unsigned)((P + 63) / 64), cb), 256, 0, ST>>>(
      x, ldx, B, H, W, C, static_cast<__nv_bfloat16*>(out_hi), static_cast<__nv_bfloat16*>(out_lo), ldo, vec_out);
  return check_launch("mtt_im2col3x3_t");
}

extern "C" int mtt_im2col_patch_t(const float* img, int32_t B, int32_t Cin, int32_t H, int32_t W, int32_t patch,
                                  void* out_hi, void* out_lo, int64_t ldo, mtt_stream_t stream) {
  if (!img || !out_hi || B <= 0 || H % patch || W % patch)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_im2col_patch_t: bad arguments");
  const long long total = (long long)Cin * patch * patch * B * (H / patch) * (W / patch);
  im2col_patch_t_kernel<<<(unsigned)((total + 255) / 256), 256, 0, ST>>>(
      img, B, Cin, H, W, patch, static_cast<__nv_bfloat16*>(out_hi), static_cast<__nv_bfloat16*>(out_lo), ldo);
  return check_launch("mtt_im2col_patch_t");
}

extern "C" int mtt_sumsq(const float* g, int64_t n, float* out, int32_t accumulate, mtt_stream_t stream) {
  if (!g || !out || n <= 0) return set_error(MTT_ERR_BAD_SHAPE, "mtt_sumsq: bad arguments");
  if (!accumulate) cudaMemsetAsync(out, 0, sizeof(float), ST);
  long long blocks = (n + 255) / 256;
  const long long cap = (long long)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  sumsq_kernel<<<(unsigned)blocks, 256, 0, ST>>>(g, n, out);
  return check_launch("mtt_sumsq");
}

extern "C" int mtt_adam_step(float* p, const float* g, float* m, float* v, int64_t n, float lr, double beta1, double beta2,
                             float eps, float weight_decay, int32_t step, const float* gnorm_sq, float max_norm,
                             float grad_scale, mtt_stream_t stream) {
  if (!p || !g || !m || !v || n <= 0 || step <= 0) return set_error(MTT_ERR_BAD_SHAPE, "mtt_adam_step: bad arguments");
  long long blocks = (n + 255) / 256;
  const long long cap = (long long)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  // 1 - beta and the bias corrections from the double betas: 1 - (float)0.999 is 1.3e-5 off 0.001, and so is
  // 1 - 0.999f^step, which would scale v's increment and the step by that much against torch.optim.Adam
  const float bc1 = (float)(1.0 - pow(beta1, (double)step)), bc2 = (float)(1.0 - pow(beta2, (double)step));
  adam_kernel<<<(unsigned)blocks, 256, 0, ST>>>(p, g, m, v, n, lr, (float)beta1, (float)beta2, (float)(1.0 - beta1),
                                                (float)(1.0 - beta2), eps, weight_decay, bc1, bc2, gnorm_sq, max_norm,
                                                grad_scale);
  return check_launch("mtt_adam_step");
}
