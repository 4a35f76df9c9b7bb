// InvPT decoder kernels (reference: InvPT/models/transformers/invpt.py, transformer_decoder.py).
// The decoder's GEMMs / 3x3 convolutions run on gemm_tc.cu; this file holds the HBM / latency-bound
// pieces between them: row gathers, segmented (joint-channel) LayerNorm, depthwise-conv and
// average-pool token reductions, zero-insertion for the transposed convolution, and the small-KV
// cross-task attention with cross-scale score fusion.
#include <math.h>

#include "glue.cuh"
#include "host_common.h"

namespace mtt {

// ------------------------------------------------------------------------------------------------
// fp32 rows (gathered) -> split planes (dense).  e.g. x[:, 1:] of the ViT stream (vit.py:345-346).
__global__ void __launch_bounds__(256)
split_rows_kernel(const float* __restrict__ in, long long ld_in, long long in_group, long long src_group,
                  long long src_off, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                  long long ld_out, long long rows, int cols) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const float* src = in + map_row(row, in_group, src_group, src_off) * ld_in;
  for (int c = lane * 2; c < cols; c += 64) {
    const bool two = c + 1 < cols;
    store_split2({hi, lo, ld_out}, row, c, src[c], two ? src[c + 1] : 0.f, two && !(ld_out & 1), two);
  }
}

// ------------------------------------------------------------------------------------------------
// Segmented LayerNorm: a logical row is S segments of `cols` channels living in S physical rows
// (segment s at map_row(r) + s*seg_stride); statistics over all S*cols values, gamma/beta [S*cols].
// S = 1 with a row gather is the ViT's final norm on x[:, 1:]; S = T is InvPT's joint-channel
// LayerNorm over all tasks' tokens (invpt.py:524-526).  Segment s of logical row r is written to
// output row s*out_seg_stride + r.
__global__ void __launch_bounds__(256)
layernorm_seg_kernel(const float* __restrict__ in, long long ld_in, long long in_group, long long src_group,
                     long long src_off, long long seg_stride, int S, const float* __restrict__ gamma,
                     const float* __restrict__ beta, float eps, float* __restrict__ out_f32, long long ld_f32,
                     __nv_bfloat16* __restrict__ out_hi, __nv_bfloat16* __restrict__ out_lo, long long ld_bf,
                     long long out_seg_stride, long long rows, int cols) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const float* base = in + map_row(row, in_group, src_group, src_off) * ld_in;
  const float n = (float)S * (float)cols;
  float s = 0.f;
  for (int k = 0; k < S; ++k) {
    const float* src = base + (long long)k * seg_stride * ld_in;
    for (int c = lane; c < cols; c += 32) s += src[c];
  }
  const float mean = warp_sum(s) / n;
  float ss = 0.f;
  for (int k = 0; k < S; ++k) {
    const float* src = base + (long long)k * seg_stride * ld_in;
    for (int c = lane; c < cols; c += 32) {
      const float a = src[c] - mean;
      ss += a * a;
    }
  }
  const float rstd = 1.0f / sqrtf(warp_sum(ss) / n + eps);
  for (int k = 0; k < S; ++k) {
    const float* src = base + (long long)k * seg_stride * ld_in;
    const long long orow = (long long)k * out_seg_stride + row;
    for (int c = lane; c < cols; c += 32) {
      const float y = (src[c] - mean) * rstd * gamma[k * cols + c] + beta[k * cols + c];
      if (out_f32) out_f32[orow * ld_f32 + c] = y;
      if (out_hi) store_split({out_hi, out_lo, ld_bf}, orow, c, y);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Zero insertion (stride-2 up-sampling with zeros) so that ConvTranspose2d(k3, s2, p1, op1)
// (transformer_decoder.py:63) becomes a plain 3x3 convolution with the flipped kernel.
__global__ void __launch_bounds__(256)
zero_insert_kernel(const float* __restrict__ in, long long ld_in, long long src_group, long long src_off,
                   int h, int w, int C, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                   long long ld_out) {
  const long long opix = blockIdx.x;  // (b * 2h + Y) * 2w + X
  const int X = (int)(opix % (2 * w)), Y = (int)((opix / (2 * w)) % (2 * h));
  const int b = (int)(opix / ((long long)4 * w * h));
  const bool src_ok = !(X & 1) && !(Y & 1);
  const float* src = in + ((long long)b * src_group + src_off + (long long)(Y >> 1) * w + (X >> 1)) * ld_in;
  for (int c = threadIdx.x * 2; c < C; c += blockDim.x * 2) {
    uint32_t hh = 0, ll = 0;
    if (src_ok) split_pack2(src[c], src[c + 1], hh, ll);
    *reinterpret_cast<uint32_t*>(hi + opix * ld_out + c) = hh;
    if (lo) *reinterpret_cast<uint32_t*>(lo + opix * ld_out + c) = ll;
  }
}

// ------------------------------------------------------------------------------------------------
// Per-task depthwise 3x3 stride-2 conv (+ folded eval BatchNorm) producing the Q tokens
// (invpt.py:125-137,171-173).  in: fp32 joint tokens [B, T*h*w, C]; out: split joint [B, T*(h/2)(w/2), C].
__global__ void __launch_bounds__(256)
dwconv_s2_kernel(const float* __restrict__ in, long long ld_in, int T, int h, int w, int C,
                 const float* __restrict__ wgt /*[T,C,9]*/, const float* __restrict__ bias /*[T,C]*/,
                 __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, long long ld_out) {
  const int oh = h / 2, ow = w / 2;
  const long long orow = blockIdx.x;  // ((b*T + k) * oh + oy) * ow + ox
  const int ox = (int)(orow % ow), oy = (int)((orow / ow) % oh);
  const long long bk = orow / ((long long)ow * oh);
  const int k = (int)(bk % T);
  const float* base = in + bk * (long long)h * w * ld_in;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float acc = bias[k * C + c];
    const float* wc = wgt + ((long long)k * C + c) * 9;
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int iy = oy * 2 - 1 + ky;
      if (iy < 0 || iy >= h) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int ix = ox * 2 - 1 + kx;
        if (ix < 0 || ix >= w) continue;
        acc = fmaf(wc[ky * 3 + kx], base[((long long)iy * w + ix) * ld_in + c], acc);
      }
    }
    store_split({hi, lo, ld_out}, orow, c, acc);
  }
}

// Per-task average pooling, kernel = stride = s, ceil_mode, no padding (invpt.py:139-147).
__global__ void __launch_bounds__(256)
avgpool_kernel(const float* __restrict__ in, long long ld_in, int h, int w, int C, int s, int oh, int ow,
               __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, long long ld_out) {
  const long long orow = blockIdx.x;  // (bk * oh + oy) * ow + ox
  const int ox = (int)(orow % ow), oy = (int)((orow / ow) % oh);
  const long long bk = orow / ((long long)ow * oh);
  const float* base = in + bk * (long long)h * w * ld_in;
  const int y0 = oy * s, x0 = ox * s;
  const int y1 = min(y0 + s, h), x1 = min(x0 + s, w);
  const float inv = 1.0f / (float)((y1 - y0) * (x1 - x0));
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float acc = 0.f;
    for (int y = y0; y < y1; ++y)
      for (int x = x0; x < x1; ++x) acc += base[((long long)y * w + x) * ld_in + c];
    store_split({hi, lo, ld_out}, orow, c, acc * inv);
  }
}

// ------------------------------------------------------------------------------------------------
// InvPT cross-task attention (invpt.py:204-236), 2 heads, Tk keys shared by all tasks. The two contractions run on
// the wgmma GEMM as grouped launches over (batch, head) -- S = Q_h K_h^T and O_h = P_h V_h -- and this kernel is
// what sits between them, one warp per (batch, query):
//   s[h]     = raw[h] * C^-1/2                               (raw = q_h . k_h from the first GEMM)
//   prev_up  = bilinear x2 (per task, over the query grid) of the previous stage's fused score
//   f[o]     = Wf[o,0] s[0] + Wf[o,1] s[1] + Wf[o,2] prev_up[0] + Wf[o,3] prev_up[1] + bf[o]     (fuse_attn, :116,:229)
//   score_out = f (pre-softmax, consumed by the next stage, :230);  P = softmax(f) as split rows [(b*2+h)*Lq + l, Tk]
__device__ __forceinline__ void up2_coord(int d, int in_size, int& i0, int& i1, float& l1) {
  float s = 0.5f * (d + 0.5f) - 0.5f;
  if (s < 0.f) s = 0.f;
  i0 = (int)s;
  if (i0 > in_size - 1) i0 = in_size - 1;
  i1 = i0 + (i0 < in_size - 1 ? 1 : 0);
  l1 = s - (float)i0;
}

constexpr int kFuseMaxPerLane = 16;   // Tk <= 512 keys

__global__ void __launch_bounds__(256)
invpt_fuse_softmax_kernel(const float* __restrict__ raw, int B, int Lq, int Tk, float scale, const float* __restrict__ prev,
                          int T, int qh, int qw, const float* __restrict__ wf, const float* __restrict__ bf,
                          float* __restrict__ score_out, __nv_bfloat16* __restrict__ p_hi, __nv_bfloat16* __restrict__ p_lo,
                          long long ldp) {
  const long long wid = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);   // b * Lq + l
  if (wid >= (long long)B * Lq) return;
  const int lane = threadIdx.x & 31;
  const int b = (int)(wid / Lq), l = (int)(wid % Lq);
  const float* r0 = raw + (((long long)b * 2 + 0) * Lq + l) * Tk;
  const float* r1 = raw + (((long long)b * 2 + 1) * Lq + l) * Tk;
  float f0[kFuseMaxPerLane], f1[kFuseMaxPerLane];
  int y0 = 0, y1 = 0, x0 = 0, x1 = 0, task = 0, sh = 0, sw = 0;
  float ly = 0.f, lx = 0.f;
  if (prev) {
    sh = qh / 2;
    sw = qw / 2;
    task = l / (qh * qw);
    const int r = l % (qh * qw);
    up2_coord(r / qw, sh, y0, y1, ly);
    up2_coord(r % qw, sw, x0, x1, lx);
  }
  float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
  for (int k = 0; k < kFuseMaxPerLane; ++k) {
    const int t = lane + 32 * k;
    f0[k] = f1[k] = -INFINITY;
    if (t < Tk) {
      float s0 = r0[t] * scale, s1 = r1[t] * scale;
      if (prev) {
        float pu[2];
#pragma unroll
        for (int hd = 0; hd < 2; ++hd) {
          const float* pb = prev + (((long long)b * 2 + hd) * ((long long)T * sh * sw) + (long long)task * sh * sw) * Tk + t;
          const float p00 = pb[(long long)(y0 * sw + x0) * Tk], p01 = pb[(long long)(y0 * sw + x1) * Tk];
          const float p10 = pb[(long long)(y1 * sw + x0) * Tk], p11 = pb[(long long)(y1 * sw + x1) * Tk];
          pu[hd] = (1.f - ly) * ((1.f - lx) * p00 + lx * p01) + ly * ((1.f - lx) * p10 + lx * p11);
        }
        const float a0 = wf[0] * s0 + wf[1] * s1 + wf[2] * pu[0] + wf[3] * pu[1] + bf[0];
        const float a1 = wf[4] * s0 + wf[5] * s1 + wf[6] * pu[0] + wf[7] * pu[1] + bf[1];
        s0 = a0;
        s1 = a1;
      }
      f0[k] = s0;
      f1[k] = s1;
      if (score_out) {
        score_out[(((long long)b * 2 + 0) * Lq + l) * Tk + t] = s0;
        score_out[(((long long)b * 2 + 1) * Lq + l) * Tk + t] = s1;
      }
      m0 = fmaxf(m0, s0);
      m1 = fmaxf(m1, s1);
    }
  }
  m0 = warp_max(m0);
  m1 = warp_max(m1);
  float z0 = 0.f, z1 = 0.f;
#pragma unroll
  for (int k = 0; k < kFuseMaxPerLane; ++k) {
    if (lane + 32 * k < Tk) {
      f0[k] = expf(f0[k] - m0);
      f1[k] = expf(f1[k] - m1);
      z0 += f0[k];
      z1 += f1[k];
    }
  }
  const float i0 = 1.0f / warp_sum(z0), i1 = 1.0f / warp_sum(z1);
  __nv_bfloat16* h0 = p_hi + (((long long)b * 2 + 0) * Lq + l) * ldp;
  __nv_bfloat16* h1 = p_hi + (((long long)b * 2 + 1) * Lq + l) * ldp;
#pragma unroll
  for (int k = 0; k < kFuseMaxPerLane; ++k) {
    const int t = lane + 32 * k;
    if (t < Tk) {
      __nv_bfloat16 hh, ll;
      split_bf16(f0[k] * i0, hh, ll);
      h0[t] = hh;
      if (p_lo) p_lo[(h0 - p_hi) + t] = ll;
      split_bf16(f1[k] * i1, hh, ll);
      h1[t] = hh;
      if (p_lo) p_lo[(h1 - p_hi) + t] = ll;
    }
  }
}

}  // namespace mtt

using namespace mtt;
#define STREAM static_cast<cudaStream_t>(stream)

extern "C" int mtt_split_rows(const float* in, int64_t ld_in, int64_t in_group, int64_t src_group,
                              int64_t src_offset, void* out_hi, void* out_lo, int64_t ld_out, int64_t rows,
                              int32_t cols, mtt_stream_t stream) {
  if (!in || !out_hi || rows <= 0 || cols <= 0 || ld_out < cols)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_split_rows: bad arguments");
  split_rows_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, STREAM>>>(
      in, ld_in, in_group, src_group, src_offset, static_cast<__nv_bfloat16*>(out_hi),
      static_cast<__nv_bfloat16*>(out_lo), ld_out, rows, cols);
  return check_launch("mtt_split_rows");
}

extern "C" int mtt_layernorm_seg(const float* in, int64_t ld_in, int64_t in_group, int64_t src_group,
                                 int64_t src_offset, int64_t seg_stride, int32_t S, const float* gamma,
                                 const float* beta, float eps, float* out_f32, int64_t ld_f32, void* out_hi,
                                 void* out_lo, int64_t ld_bf, int64_t out_seg_stride, int64_t rows,
                                 int32_t cols, mtt_stream_t stream) {
  if (!in || !gamma || !beta || rows <= 0 || cols <= 0 || S <= 0 || (!out_f32 && !out_hi))
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_layernorm_seg: bad arguments");
  layernorm_seg_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, STREAM>>>(
      in, ld_in, in_group, src_group, src_offset, seg_stride, S, gamma, beta, eps, out_f32, ld_f32,
      static_cast<__nv_bfloat16*>(out_hi), static_cast<__nv_bfloat16*>(out_lo), ld_bf, out_seg_stride, rows,
      cols);
  return check_launch("mtt_layernorm_seg");
}

extern "C" int mtt_zero_insert(const float* in, int64_t ld_in, int64_t src_group, int64_t src_offset,
                               int32_t B, int32_t h, int32_t w, int32_t C, void* out_hi, void* out_lo,
                               int64_t ld_out, mtt_stream_t stream) {
  if (!in || !out_hi || B <= 0 || h <= 0 || w <= 0 || C <= 0 || (C & 1) || (ld_out & 1))
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_zero_insert: bad arguments");
  zero_insert_kernel<<<(unsigned)((long long)B * 4 * h * w), 256, 0, STREAM>>>(
      in, ld_in, src_group, src_offset, h, w, C, static_cast<__nv_bfloat16*>(out_hi),
      static_cast<__nv_bfloat16*>(out_lo), ld_out);
  return check_launch("mtt_zero_insert");
}

extern "C" int mtt_dwconv3x3_s2(const float* in, int64_t ld_in, int32_t B, int32_t T, int32_t h, int32_t w,
                                int32_t C, const float* weight, const float* bias, void* out_hi,
                                void* out_lo, int64_t ld_out, mtt_stream_t stream) {
  if (!in || !weight || !bias || !out_hi || B <= 0 || T <= 0 || h < 2 || w < 2 || (h & 1) || (w & 1))
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_dwconv3x3_s2: bad arguments (h=%d w=%d must be even)", h, w);
  const long long rows = (long long)B * T * (h / 2) * (w / 2);
  const int threads = C >= 256 ? 256 : (C >= 128 ? 128 : 64);
  dwconv_s2_kernel<<<(unsigned)rows, threads, 0, STREAM>>>(in, ld_in, T, h, w, C, weight, bias,
                                                          static_cast<__nv_bfloat16*>(out_hi),
                                                          static_cast<__nv_bfloat16*>(out_lo), ld_out);
  return check_launch("mtt_dwconv3x3_s2");
}

extern "C" int mtt_avgpool(const float* in, int64_t ld_in, int32_t BT, int32_t h, int32_t w, int32_t C,
                           int32_t s, void* out_hi, void* out_lo, int64_t ld_out, mtt_stream_t stream) {
  if (!in || !out_hi || BT <= 0 || h <= 0 || w <= 0 || s <= 0)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_avgpool: bad arguments");
  const int oh = (h + s - 1) / s, ow = (w + s - 1) / s;
  const int threads = C >= 256 ? 256 : (C >= 128 ? 128 : 64);
  avgpool_kernel<<<(unsigned)((long long)BT * oh * ow), threads, 0, STREAM>>>(
      in, ld_in, h, w, C, s, oh, ow, static_cast<__nv_bfloat16*>(out_hi),
      static_cast<__nv_bfloat16*>(out_lo), ld_out);
  return check_launch("mtt_avgpool");
}

extern "C" int mtt_invpt_fuse_softmax(const float* raw, int32_t B, int32_t Lq, int32_t Tk, float scale,
                                      const float* prev_score, int32_t T, int32_t qh, int32_t qw, const float* fuse_w,
                                      const float* fuse_b, float* score_out, void* p_hi, void* p_lo, int64_t ldp,
                                      mtt_stream_t stream) {
  if (!raw || !p_hi || B <= 0 || Lq <= 0 || Tk <= 0 || Tk > 32 * kFuseMaxPerLane || ldp < Tk)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_invpt_fuse_softmax: bad arguments (Tk=%d, at most %d)", Tk, 32 * kFuseMaxPerLane);
  if (prev_score && (T <= 0 || qh <= 0 || qw <= 0 || (qh & 1) || (qw & 1) || T * qh * qw != Lq || !fuse_w || !fuse_b))
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_invpt_fuse_softmax: bad fusion geometry");
  const long long rows = (long long)B * Lq;
  invpt_fuse_softmax_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, STREAM>>>(
      raw, B, Lq, Tk, scale, prev_score, T, qh, qw, fuse_w, fuse_b, score_out, static_cast<__nv_bfloat16*>(p_hi),
      static_cast<__nv_bfloat16*>(p_lo), ldp);
  return check_launch("mtt_invpt_fuse_softmax");
}
