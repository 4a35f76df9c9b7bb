// Row-wise HBM-bound kernels: fp32 -> split-bf16 cast and LayerNorm with split output.
// One warp per row, float4 loads, warp-shuffle reductions.
#include "glue.cuh"
#include "host_common.h"

namespace mtt {

__global__ void __launch_bounds__(256)
split_kernel(const float* __restrict__ in, long long ld_in, __nv_bfloat16* __restrict__ hi,
             __nv_bfloat16* __restrict__ lo, long long ld_out, long long rows, int cols, int cols_pad) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const float* src = in + row * ld_in;
  __nv_bfloat16* dh = hi + row * ld_out;
  __nv_bfloat16* dl = lo ? lo + row * ld_out : nullptr;
  for (int c = lane; c < cols_pad; c += 32) {
    const float x = c < cols ? src[c] : 0.f;
    __nv_bfloat16 h, l;
    split_bf16(x, h, l);
    dh[c] = h;
    if (dl) dl[c] = l;
  }
}

// LayerNorm, biased variance, two-pass statistics like ATen's CPU/CUDA kernels
// (reference: nn.LayerNorm at TP/models/transformers/taskprompter.py:262,266,329).
__global__ void __launch_bounds__(256)
layernorm_kernel(const float* __restrict__ in, long long ld_in, const float* __restrict__ gamma,
                 const float* __restrict__ beta, float eps, float* __restrict__ out_f32,
                 long long ld_f32, __nv_bfloat16* __restrict__ out_hi, __nv_bfloat16* __restrict__ out_lo,
                 long long ld_bf, long long rows, int cols) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const float* src = in + row * ld_in;
  const bool vec = ((cols & 3) == 0) && ((ld_in & 3) == 0) &&
                   ((reinterpret_cast<uintptr_t>(in) & 15) == 0);
  float s = 0.f;
  if (vec) {
    const float4* s4 = reinterpret_cast<const float4*>(src);
    for (int c = lane; c < cols / 4; c += 32) {
      const float4 v = s4[c];
      s += (v.x + v.y) + (v.z + v.w);
    }
  } else {
    for (int c = lane; c < cols; c += 32) s += src[c];
  }
  const float mean = warp_sum(s) / (float)cols;
  float ss = 0.f;
  if (vec) {
    const float4* s4 = reinterpret_cast<const float4*>(src);
    for (int c = lane; c < cols / 4; c += 32) {
      const float4 v = s4[c];
      const float a = v.x - mean, b = v.y - mean, cc = v.z - mean, d = v.w - mean;
      ss += (a * a + b * b) + (cc * cc + d * d);
    }
  } else {
    for (int c = lane; c < cols; c += 32) {
      const float a = src[c] - mean;
      ss += a * a;
    }
  }
  const float var = warp_sum(ss) / (float)cols;
  const float rstd = 1.0f / sqrtf(var + eps);
  for (int c = lane * 2; c < cols; c += 64) {
    const bool two = c + 1 < cols;
    const float y0 = (src[c] - mean) * rstd * gamma[c] + beta[c];
    const float y1 = two ? (src[c + 1] - mean) * rstd * gamma[c + 1] + beta[c + 1] : 0.f;
    if (out_f32) {
      out_f32[row * ld_f32 + c] = y0;
      if (two) out_f32[row * ld_f32 + c + 1] = y1;
    }
    if (out_hi) {
      if (two && ((ld_bf & 1) == 0)) {
        uint32_t h, l;
        split_pack2(y0, y1, h, l);
        *reinterpret_cast<uint32_t*>(out_hi + row * ld_bf + c) = h;
        if (out_lo) *reinterpret_cast<uint32_t*>(out_lo + row * ld_bf + c) = l;
      } else {
        __nv_bfloat16 h, l;
        split_bf16(y0, h, l);
        out_hi[row * ld_bf + c] = h;
        if (out_lo) out_lo[row * ld_bf + c] = l;
        if (two) {
          split_bf16(y1, h, l);
          out_hi[row * ld_bf + c + 1] = h;
          if (out_lo) out_lo[row * ld_bf + c + 1] = l;
        }
      }
    }
  }
}


// Fast path: the whole row lives in registers (cols % 128 == 0, cols <= 1024): one global read,
// 8-byte vector stores of the split planes.
template <int NV>  // float4 per lane
__global__ void __launch_bounds__(256)
layernorm_reg_kernel(const float* __restrict__ in, long long ld_in, const float* __restrict__ gamma,
                     const float* __restrict__ beta, float eps, float* __restrict__ out_f32, long long ld_f32,
                     __nv_bfloat16* __restrict__ out_hi, __nv_bfloat16* __restrict__ out_lo, long long ld_bf,
                     long long rows) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  constexpr int cols = NV * 128;
  const float4* s4 = reinterpret_cast<const float4*>(in + row * ld_in);
  float4 v[NV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    v[i] = s4[lane + i * 32];
    s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  }
  const float mean = warp_sum(s) / (float)cols;
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    ss += (a * a + b * b) + (c * c + d * d);
  }
  const float rstd = 1.0f / sqrtf(warp_sum(ss) / (float)cols + eps);
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  const float4* b4 = reinterpret_cast<const float4*>(beta);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c4 = lane + i * 32;
    const float4 g = __ldg(g4 + c4), bb = __ldg(b4 + c4);
    float4 y;
    y.x = (v[i].x - mean) * rstd * g.x + bb.x;
    y.y = (v[i].y - mean) * rstd * g.y + bb.y;
    y.z = (v[i].z - mean) * rstd * g.z + bb.z;
    y.w = (v[i].w - mean) * rstd * g.w + bb.w;
    if (out_f32) *reinterpret_cast<float4*>(out_f32 + row * ld_f32 + c4 * 4) = y;
    if (out_hi) {
      uint2 h, l;
      split_pack2(y.x, y.y, h.x, l.x);
      split_pack2(y.z, y.w, h.y, l.y);
      *reinterpret_cast<uint2*>(out_hi + row * ld_bf + c4 * 4) = h;
      if (out_lo) *reinterpret_cast<uint2*>(out_lo + row * ld_bf + c4 * 4) = l;
    }
  }
}

__global__ void __launch_bounds__(256)
sum_partials_kernel(const float* __restrict__ part, int S, long long M, int N, long long ld, const float* __restrict__ bias,
                    float* __restrict__ out, long long ldo) {
  const long long n = M * N;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const long long m = e / N;
    const int c = (int)(e % N);
    float acc = bias ? bias[c] : 0.f;
    for (int s = 0; s < S; ++s) acc += part[((long long)s * M + m) * ld + c];
    out[m * ldo + c] = acc;
  }
}

}  // namespace mtt

extern "C" int mtt_sum_partials(const float* partial, int32_t S, int64_t M, int32_t N, int64_t ld, const float* bias,
                                float* out, int64_t ldo, mtt_stream_t stream) {
  using namespace mtt;
  if (!partial || !out || S <= 0 || M <= 0 || N <= 0 || ld < N || ldo < N)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_sum_partials: bad arguments");
  const long long n = M * N;
  const int blocks = (int)((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096);
  sum_partials_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(partial, S, M, N, ld, bias, out, ldo);
  return check_launch("mtt_sum_partials");
}

extern "C" int mtt_split_f32(const float* in, int64_t ld_in, void* out_hi, void* out_lo,
                             int64_t ld_out, int64_t rows, int32_t cols, int32_t cols_pad,
                             mtt_stream_t stream) {
  using namespace mtt;
  if (!in || !out_hi || rows <= 0 || cols <= 0 || cols_pad < cols || ld_out < cols_pad)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_split_f32: bad arguments (rows=%lld cols=%d pad=%d)",
                     (long long)rows, cols, cols_pad);
  const int wpb = 8;
  const long long blocks = (rows + wpb - 1) / wpb;
  split_kernel<<<(unsigned)blocks, wpb * 32, 0, static_cast<cudaStream_t>(stream)>>>(
      in, ld_in, static_cast<__nv_bfloat16*>(out_hi), static_cast<__nv_bfloat16*>(out_lo), ld_out, rows,
      cols, cols_pad);
  return check_launch("mtt_split_f32");
}

extern "C" int mtt_layernorm(const float* in, int64_t ld_in, const float* gamma, const float* beta,
                             float eps, float* out_f32, int64_t ld_f32, void* out_hi, void* out_lo,
                             int64_t ld_bf, int64_t rows, int32_t cols, mtt_stream_t stream) {
  using namespace mtt;
  if (!in || !gamma || !beta || rows <= 0 || cols <= 0 || (!out_f32 && !out_hi))
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_layernorm: bad arguments (rows=%lld cols=%d)",
                     (long long)rows, cols);
  const int wpb = 8;
  const long long blocks = (rows + wpb - 1) / wpb;
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  const bool fast = cols % 128 == 0 && cols <= 1024 && ld_in % 4 == 0 && al16(in) && al16(gamma) && al16(beta) &&
                    (!out_f32 || (ld_f32 % 4 == 0 && al16(out_f32))) &&
                    (!out_hi || (ld_bf % 4 == 0 && (reinterpret_cast<uintptr_t>(out_hi) & 7) == 0 &&
                                 (!out_lo || (reinterpret_cast<uintptr_t>(out_lo) & 7) == 0)));
  if (fast) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    __nv_bfloat16* oh = static_cast<__nv_bfloat16*>(out_hi);
    __nv_bfloat16* ol = static_cast<__nv_bfloat16*>(out_lo);
#define MTT_LN_CASE(NV)                                                                                  \
  case NV:                                                                                               \
    layernorm_reg_kernel<NV><<<(unsigned)blocks, wpb * 32, 0, st>>>(in, ld_in, gamma, beta, eps, out_f32, \
                                                                   ld_f32, oh, ol, ld_bf, rows);         \
    break;
    switch (cols / 128) {
      MTT_LN_CASE(1) MTT_LN_CASE(2) MTT_LN_CASE(3) MTT_LN_CASE(4) MTT_LN_CASE(5) MTT_LN_CASE(6) MTT_LN_CASE(7)
      MTT_LN_CASE(8)
    }
#undef MTT_LN_CASE
    return check_launch("mtt_layernorm");
  }
  layernorm_kernel<<<(unsigned)blocks, wpb * 32, 0, static_cast<cudaStream_t>(stream)>>>(
      in, ld_in, gamma, beta, eps, out_f32, ld_f32, static_cast<__nv_bfloat16*>(out_hi),
      static_cast<__nv_bfloat16*>(out_lo), ld_bf, rows, cols);
  return check_launch("mtt_layernorm");
}
