// The named operators of the transformer block and of the task decoder (SURVEY.md section 8b): each entry point
// enqueues the launch sequence that replaces one eager-op group of the reference, with every intermediate living in
// a caller-provided workspace (mtt_workspace_bytes). Plus the parameter pre-packing entry points (BatchNorm folding,
// tap-major conv layout, split-bf16 cast) and the NCHW <-> NHWC layout kernels the nn.Module-level forwards use.
//
//   mtt_ln_qkv            TP taskprompter.py:272 (norm1) + :199 (cat) + :201 (qkv)         LayerNorm -> GEMM
//   mtt_proj_residual     :212 (proj) + :273,:276 (residual)                               GEMM, residual epilogue
//   mtt_ln_mlp_residual   :274,:277 (norm2, Mlp fc1 + GELU + fc2, residual)                LayerNorm -> GEMM+GELU -> GEMM+residual
//   mtt_gated_conv1x1     :436-447, :452-468, :471 (spatial + channel gating, two 1x1)     gate kernel -> 2 GEMMs into the cat buffer
//   mtt_conv3x3_bn_act    :362 / :691-695 (3x3 + BN + act, optional fused 1x1 head)        implicit-GEMM conv (-> GEMM)
#include "glue.cuh"
#include "host_common.h"

namespace mtt {

// ---------------------------------------------------------------- weight packing kernels
// One thread per packed element of out [N, taps * cin_pad]: element (n, tap, c) <- scale[n] * w(n, c, tap), where
// w is a Conv2d weight [N, Cin, kh, kw] or (transposed != 0) a ConvTranspose2d weight [Cin, N, kh, kw] read with
// the spatially flipped tap (the equivalent forward convolution). c >= Cin is zero padding.
__global__ void __launch_bounds__(256)
pack_conv_kernel(const float* __restrict__ w, const float* __restrict__ scale, int N, int Cin, int taps,
                 int cin_pad, int transposed, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                 long long ld) {
  const long long total = (long long)N * taps * cin_pad;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cin_pad);
    const int tap = (int)((i / cin_pad) % taps);
    const int n = (int)(i / ((long long)cin_pad * taps));
    float v = 0.f;
    if (c < Cin) {
      v = transposed ? w[((long long)c * N + n) * taps + (taps - 1 - tap)] : w[((long long)n * Cin + c) * taps + tap];
      if (scale) v *= scale[n];
    }
    store_split({hi, lo, ld}, n, (long long)tap * cin_pad + c, v);
  }
}

// eval-mode BatchNorm folding: scale[n] = gamma / sqrt(var + eps); bias_out[n] = (bias - mean) * scale + beta
__global__ void bn_fold_kernel(const float* __restrict__ bias, const float* __restrict__ gamma,
                               const float* __restrict__ beta, const float* __restrict__ mean,
                               const float* __restrict__ var, float eps, int N, float* __restrict__ scale,
                               float* __restrict__ bias_out) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const float b0 = bias ? bias[n] : 0.f;
  if (gamma) {
    const float s = gamma[n] / sqrtf(var[n] + eps);
    scale[n] = s;
    bias_out[n] = (b0 - mean[n]) * s + beta[n];
  } else {
    scale[n] = 1.f;
    bias_out[n] = b0;
  }
}

// ---------------------------------------------------------------- layout kernels (module-boundary forwards)
// NCHW fp32 [B, C, H*W] -> NHWC split [B*H*W, ld]: 32x32 smem transpose tiles, coalesced on both sides.
__global__ void __launch_bounds__(1024)
nchw_to_nhwc_split_kernel(const float* __restrict__ in, int C, int HW, __nv_bfloat16* __restrict__ hi,
                          __nv_bfloat16* __restrict__ lo, long long ld) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const float* src = in + (long long)b * C * HW;
  if (c0 + ty < C && p0 + tx < HW) tile[ty][tx] = src[(long long)(c0 + ty) * HW + p0 + tx];
  __syncthreads();
  const int p = p0 + ty, c = c0 + tx;
  if (p < HW && c < C) {
    store_split({hi, lo, ld}, (long long)b * HW + p, c, tile[tx][ty]);
  }
}

// NHWC fp32 rows [B*HW, ld] -> NCHW fp32 [B, C, HW]
__global__ void __launch_bounds__(1024)
nhwc_to_nchw_kernel(const float* __restrict__ in, long long ld, int C, int HW, float* __restrict__ out) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
  if (p0 + ty < HW && c0 + tx < C) tile[ty][tx] = in[((long long)b * HW + p0 + ty) * ld + c0 + tx];
  __syncthreads();
  if (c0 + ty < C && p0 + tx < HW) out[((long long)b * C + c0 + ty) * HW + p0 + tx] = tile[tx][ty];
}

static size_t planes_bytes(int nsplit, long long rows, long long ld) {
  return (size_t)nsplit * (size_t)rows * (size_t)ld * 2;
}
static long long pad8(long long x) { return (x + 7) / 8 * 8; }
static size_t align256(size_t x) { return (x + 255) / 256 * 256; }

}  // namespace mtt

using namespace mtt;
#define STREAM static_cast<cudaStream_t>(stream)

extern "C" {

int mtt_pack_weight(const float* w, int64_t ld_w, int32_t N, int32_t K, int32_t nsplit, void* out_hi, void* out_lo,
                    int64_t ld_out, mtt_stream_t stream) {
  if (nsplit != 1 && nsplit != 2) return set_error(MTT_ERR_BAD_SHAPE, "mtt_pack_weight: nsplit=%d", nsplit);
  return mtt_split_f32(w, ld_w, out_hi, nsplit == 2 ? out_lo : nullptr, ld_out, N, K, (int32_t)pad8(K), stream);
}

int mtt_pack_conv_weight(const float* w, const float* bias, const float* bn_gamma, const float* bn_beta,
                         const float* bn_mean, const float* bn_var, float bn_eps, int32_t N, int32_t Cin,
                         int32_t ksize, int32_t transposed, int32_t nsplit, void* out_hi, void* out_lo, int64_t ld_out,
                         float* bias_out, float* scale_ws, mtt_stream_t stream) {
  if (!w || !out_hi || !bias_out || !scale_ws || N <= 0 || Cin <= 0 || ksize < 1 || ksize > 3 ||
      (nsplit != 1 && nsplit != 2) || (nsplit == 2 && !out_lo))
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_pack_conv_weight: bad arguments (N=%d Cin=%d k=%d)", N, Cin, ksize);
  if (bn_gamma && (!bn_beta || !bn_mean || !bn_var))
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_pack_conv_weight: incomplete BatchNorm statistics");
  const int taps = ksize * ksize;
  const int cin_pad = (Cin + 63) / 64 * 64;
  if (ld_out < (int64_t)taps * cin_pad)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_pack_conv_weight: ld_out=%lld < %d", (long long)ld_out, taps * cin_pad);
  bn_fold_kernel<<<(N + 127) / 128, 128, 0, STREAM>>>(bias, bn_gamma, bn_beta, bn_mean, bn_var, bn_eps, N, scale_ws,
                                                      bias_out);
  int rc = check_launch("mtt_pack_conv_weight(fold)");
  if (rc) return rc;
  const long long total = (long long)N * taps * cin_pad;
  const int blocks = (int)((total + 255) / 256 < 4096 ? (total + 255) / 256 : 4096);
  pack_conv_kernel<<<blocks, 256, 0, STREAM>>>(w, scale_ws, N, Cin, taps, cin_pad, transposed,
                                               static_cast<__nv_bfloat16*>(out_hi),
                                               nsplit == 2 ? static_cast<__nv_bfloat16*>(out_lo) : nullptr, ld_out);
  return check_launch("mtt_pack_conv_weight");
}

int mtt_nchw_to_nhwc_split(const float* in, int32_t B, int32_t C, int32_t H, int32_t W, void* out_hi, void* out_lo,
                           int64_t ld_out, mtt_stream_t stream) {
  if (!in || !out_hi || B <= 0 || C <= 0 || H <= 0 || W <= 0 || ld_out < C)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_nchw_to_nhwc_split: bad arguments");
  dim3 grid((H * W + 31) / 32, (C + 31) / 32, B);
  nchw_to_nhwc_split_kernel<<<grid, dim3(32, 32), 0, STREAM>>>(in, C, H * W, static_cast<__nv_bfloat16*>(out_hi),
                                                              static_cast<__nv_bfloat16*>(out_lo), ld_out);
  return check_launch("mtt_nchw_to_nhwc_split");
}

int mtt_nhwc_to_nchw(const float* in, int64_t ld_in, int32_t B, int32_t C, int32_t H, int32_t W, float* out,
                     mtt_stream_t stream) {
  if (!in || !out || B <= 0 || C <= 0 || H <= 0 || W <= 0 || ld_in < C)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_nhwc_to_nchw: bad arguments");
  dim3 grid((H * W + 31) / 32, (C + 31) / 32, B);
  nhwc_to_nchw_kernel<<<grid, dim3(32, 32), 0, STREAM>>>(in, ld_in, C, H * W, out);
  return check_launch("mtt_nhwc_to_nchw");
}

// ------------------------------------------------------------------------------------------------ workspace sizes
size_t mtt_workspace_bytes(int32_t op, const mtt_shape* s) {
  if (!s) return 0;
  const int ns = s->nsplit == 1 ? 1 : 2;
  switch (op) {
    case MTT_OP_LN_QKV:  // LN1 output, split [ns][rows][pad8(C)], then the GEMM's stream-K workspace
      return align256(planes_bytes(ns, s->rows, pad8(s->C))) + align256(mtt_gemm_streamk_bytes());
    case MTT_OP_LN_MLP_RESIDUAL:  // LN2 output + hidden activations, then the stream-K workspace of fc1 / fc2
      return align256(planes_bytes(ns, s->rows, pad8(s->C))) + align256(planes_bytes(ns, s->rows, pad8(s->hidden))) +
             align256(mtt_gemm_streamk_bytes());
    case MTT_OP_GATED_CONV1X1:  // two gated copies of the patch map per task: [task][spatial | channel][plane][rows][ld]
      return (size_t)(s->T > 0 ? s->T : 1) * 2 * align256(planes_bytes(ns, s->rows, pad8(s->C)));
    case MTT_OP_CONV3X3_BN_ACT:  // hidden map between the 3x3 and a fused 1x1 head
      return align256(planes_bytes(ns, s->rows, pad8(s->hidden)));
    case MTT_OP_ATTN_FWD:
    case MTT_OP_PROJ_RESIDUAL:
    case MTT_OP_CHAN_PROMPT_LOGITS:
    case MTT_OP_BILINEAR_UP:
    case MTT_OP_INVPT_ATTN:
    case MTT_OP_LAYERNORM:
      return 0;  // single-kernel operators: no intermediate
    default:
      return 0;
  }
}

static int need_ws(const char* what, void* ws, size_t have, size_t want) {
  if (want && (!ws || have < want))
    return set_error(MTT_ERR_BAD_SHAPE, "%s: workspace %zu bytes < required %zu (mtt_workspace_bytes)", what, have,
                     want);
  if (want && (reinterpret_cast<uintptr_t>(ws) & 255))
    return set_error(MTT_ERR_MISALIGNED, "%s: workspace must be 256-byte aligned", what);
  return MTT_OK;
}

static void fill_b(mtt_gemm_desc& g, const mtt_weight* w) {
  g.b_hi = w->hi;
  g.b_lo = w->lo;
  g.ldb = w->ld;
}

int mtt_ln_qkv(const float* x, int64_t ldx, const float* gamma, const float* beta, float eps, const mtt_weight* wqkv,
               const float* bias, void* qkv_hi, void* qkv_lo, int64_t ldq, const mtt_shape* s, void* ws,
               size_t ws_bytes, mtt_stream_t stream) {
  if (!x || !wqkv || !qkv_hi || !s || s->rows <= 0 || s->C <= 0)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_ln_qkv: bad arguments");
  int rc = need_ws("mtt_ln_qkv", ws, ws_bytes, mtt_workspace_bytes(MTT_OP_LN_QKV, s));
  if (rc) return rc;
  const int ns = s->nsplit == 1 ? 1 : 2;
  const long long ldn = pad8(s->C);
  __nv_bfloat16* xn_hi = static_cast<__nv_bfloat16*>(ws);
  __nv_bfloat16* xn_lo = ns == 2 ? xn_hi + (long long)s->rows * ldn : nullptr;
  if ((rc = mtt_layernorm(x, ldx, gamma, beta, eps, nullptr, 0, xn_hi, xn_lo, ldn, s->rows, s->C, stream))) return rc;
  mtt_gemm_desc g = {};
  g.a_hi = xn_hi;
  g.a_lo = xn_lo;
  g.lda = ldn;
  fill_b(g, wqkv);
  g.M = s->rows;
  g.N = 3 * s->C;
  g.K = s->C;
  g.nsplit = ns;
  g.bias = bias;
  g.out_hi = qkv_hi;
  g.out_lo = qkv_lo;
  g.ldo_bf = ldq;
  g.sk_ws = static_cast<uint8_t*>(ws) + align256(planes_bytes(ns, s->rows, ldn));
  g.sk_ws_bytes = (int64_t)mtt_gemm_streamk_bytes();
  return mtt_gemm(&g, stream);
}

int mtt_proj_residual(const void* a_hi, const void* a_lo, int64_t lda, const mtt_weight* wproj, const float* bias,
                      float* x, int64_t ldx, const mtt_shape* s, mtt_stream_t stream) {
  if (!a_hi || !wproj || !x || !s) return set_error(MTT_ERR_BAD_SHAPE, "mtt_proj_residual: bad arguments");
  mtt_gemm_desc g = {};
  g.a_hi = a_hi;
  g.a_lo = a_lo;
  g.lda = lda;
  fill_b(g, wproj);
  g.M = s->rows;
  g.N = s->C;
  g.K = s->C;
  g.nsplit = s->nsplit == 1 ? 1 : 2;
  g.bias = bias;
  g.residual = x;
  g.ldr = ldx;
  g.out_f32 = x;
  g.ldo_f32 = ldx;
  return mtt_gemm(&g, stream);
}

int mtt_ln_mlp_residual(float* x, int64_t ldx, const float* gamma, const float* beta, float eps, const mtt_weight* w1,
                        const float* b1, const mtt_weight* w2, const float* b2, const mtt_shape* s, void* ws,
                        size_t ws_bytes, mtt_stream_t stream) {
  if (!x || !w1 || !w2 || !s || s->rows <= 0 || s->C <= 0 || s->hidden <= 0)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_ln_mlp_residual: bad arguments");
  int rc = need_ws("mtt_ln_mlp_residual", ws, ws_bytes, mtt_workspace_bytes(MTT_OP_LN_MLP_RESIDUAL, s));
  if (rc) return rc;
  const int ns = s->nsplit == 1 ? 1 : 2;
  const long long ldn = pad8(s->C), ldh = pad8(s->hidden);
  uint8_t* base = static_cast<uint8_t*>(ws);
  __nv_bfloat16* xn_hi = reinterpret_cast<__nv_bfloat16*>(base);
  __nv_bfloat16* xn_lo = ns == 2 ? xn_hi + (long long)s->rows * ldn : nullptr;
  __nv_bfloat16* h_hi = reinterpret_cast<__nv_bfloat16*>(base + align256(planes_bytes(ns, s->rows, ldn)));
  __nv_bfloat16* h_lo = ns == 2 ? h_hi + (long long)s->rows * ldh : nullptr;
  if ((rc = mtt_layernorm(x, ldx, gamma, beta, eps, nullptr, 0, xn_hi, xn_lo, ldn, s->rows, s->C, stream))) return rc;
  mtt_gemm_desc g = {};
  g.a_hi = xn_hi;
  g.a_lo = xn_lo;
  g.lda = ldn;
  fill_b(g, w1);
  g.M = s->rows;
  g.N = s->hidden;
  g.K = s->C;
  g.nsplit = ns;
  g.bias = b1;
  g.act = MTT_ACT_GELU;
  g.out_hi = h_hi;
  g.out_lo = h_lo;
  g.ldo_bf = ldh;
  void* sk_ws = base + align256(planes_bytes(ns, s->rows, ldn)) + align256(planes_bytes(ns, s->rows, ldh));
  g.sk_ws = sk_ws;
  g.sk_ws_bytes = (int64_t)mtt_gemm_streamk_bytes();
  if ((rc = mtt_gemm(&g, stream))) return rc;
  mtt_gemm_desc g2 = {};
  g2.a_hi = h_hi;
  g2.a_lo = h_lo;
  g2.lda = ldh;
  fill_b(g2, w2);
  g2.M = s->rows;
  g2.N = s->C;
  g2.K = s->hidden;
  g2.nsplit = ns;
  g2.bias = b2;
  g2.residual = x;
  g2.ldr = ldx;
  g2.out_f32 = x;
  g2.ldo_f32 = ldx;
  g2.sk_ws = sk_ws;   // fc2 follows fc1 on the same stream: the flags are zero again when it starts
  g2.sk_ws_bytes = (int64_t)mtt_gemm_streamk_bytes();
  return mtt_gemm(&g2, stream);
}

int mtt_gated_conv1x1(const float* x, int64_t ldx, int64_t x_group_rows, int64_t x_row_offset,
                      const float* prompt_logits, const float* chan_logits, int32_t ntasks, const mtt_gated_task* tasks,
                      int32_t gh, int32_t gw, int32_t nh, int32_t nw, int32_t e, int64_t ld_cat, int32_t chan_col,
                      const mtt_shape* s, void* ws, size_t ws_bytes, mtt_stream_t stream) {
  if (!x || !tasks || !s || ntasks <= 0 || ntasks > s->T || s->B <= 0 || gh <= 0 || gw <= 0 || e <= 0)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_gated_conv1x1: bad arguments");
  mtt_shape sh = *s;
  sh.rows = s->B * gh * gw;
  sh.T = ntasks;
  int rc = need_ws("mtt_gated_conv1x1", ws, ws_bytes, mtt_workspace_bytes(MTT_OP_GATED_CONV1X1, &sh));
  if (rc) return rc;
  const int ns = s->nsplit == 1 ? 1 : 2;
  const long long ldy = pad8(s->C), rows = sh.rows;
  const size_t pb = align256(planes_bytes(ns, rows, ldy));
  const long long task_stride = (long long)(2 * pb / 2);  // elements between consecutive tasks' planes
  uint8_t* base = static_cast<uint8_t*>(ws);
  auto ys_hi = [&](int k) { return reinterpret_cast<__nv_bfloat16*>(base + (size_t)k * 2 * pb); };
  auto yc_hi = [&](int k) { return reinterpret_cast<__nv_bfloat16*>(base + (size_t)k * 2 * pb + pb); };
  if ((rc = mtt_gate_split(x, ldx, x_group_rows, x_row_offset, prompt_logits, chan_logits, 0, ntasks, s->B, s->T, s->N,
                           s->H, s->C, gh, gw, nh, nw, ys_hi(0), ns == 2 ? ys_hi(0) + rows * ldy : nullptr, yc_hi(0),
                           ns == 2 ? yc_hi(0) + rows * ldy : nullptr, ldy, task_stride, stream)))
    return rc;
  constexpr int kChunk = 6;  // 12 problems per grouped launch
  for (int k0 = 0; k0 < ntasks; k0 += kChunk) {
    const int nk = ntasks - k0 < kChunk ? ntasks - k0 : kChunk;
    mtt_gemm_desc g[2 * kChunk];
    for (int k = 0; k < nk; ++k) {
      const mtt_gated_task& t = tasks[k0 + k];
      for (int which = 0; which < 2; ++which) {
        mtt_gemm_desc& d = g[2 * k + which];
        d = mtt_gemm_desc{};
        __nv_bfloat16* a = which ? yc_hi(k0 + k) : ys_hi(k0 + k);
        d.a_hi = a;
        d.a_lo = ns == 2 ? a + rows * ldy : nullptr;
        d.lda = ldy;
        fill_b(d, which ? &t.w_chan : &t.w_spa);
        d.M = (int32_t)rows;
        d.N = e;
        d.K = s->C;
        d.nsplit = ns;
        d.bias = which ? t.b_chan : t.b_spa;
        const long long col = which ? chan_col : 0;
        d.out_hi = static_cast<__nv_bfloat16*>(t.cat_hi) + col;
        d.out_lo = t.cat_lo ? static_cast<__nv_bfloat16*>(t.cat_lo) + col : nullptr;
        d.ldo_bf = ld_cat;
      }
    }
    if ((rc = mtt_gemm_grouped(g, 2 * nk, stream))) return rc;
  }
  return MTT_OK;
}

int mtt_conv3x3_bn_act(const void* a_hi, const void* a_lo, int64_t lda, int32_t B, int32_t H, int32_t W, int32_t Cin,
                       int32_t dil, const mtt_weight* w3, const float* b3, int32_t Cout, int32_t act, void* mid_hi,
                       void* mid_lo, int64_t ld_mid, const mtt_weight* w_head, const float* b_head, int32_t n_out,
                       float* out_f32, int64_t ldo, int32_t nsplit, void* ws, size_t ws_bytes, mtt_stream_t stream) {
  if (!a_hi || !w3 || B <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_conv3x3_bn_act: bad arguments");
  const int ns = nsplit == 1 ? 1 : 2;
  const long long rows = (long long)B * H * W;
  __nv_bfloat16* m_hi = static_cast<__nv_bfloat16*>(mid_hi);
  __nv_bfloat16* m_lo = static_cast<__nv_bfloat16*>(mid_lo);
  long long ldm = ld_mid;
  if (!m_hi) {  // the hidden map lives in the workspace (only legal with a fused head)
    if (!w_head) return set_error(MTT_ERR_BAD_SHAPE, "mtt_conv3x3_bn_act: neither an output map nor a fused head");
    mtt_shape sh = {};
    sh.rows = (int32_t)rows;
    sh.hidden = Cout;
    sh.nsplit = ns;
    int rc = need_ws("mtt_conv3x3_bn_act", ws, ws_bytes, mtt_workspace_bytes(MTT_OP_CONV3X3_BN_ACT, &sh));
    if (rc) return rc;
    ldm = pad8(Cout);
    m_hi = static_cast<__nv_bfloat16*>(ws);
    m_lo = ns == 2 ? m_hi + rows * ldm : nullptr;
  }
  mtt_gemm_desc g = {};
  g.a_hi = a_hi;
  g.a_lo = a_lo;
  g.lda = lda;
  fill_b(g, w3);
  g.M = (int32_t)rows;
  g.N = Cout;
  g.K = Cin;
  g.nsplit = ns;
  g.mode = 1;
  g.B = B;
  g.H = H;
  g.W = W;
  g.ksize = 3;
  g.dil = dil < 1 ? 1 : dil;
  g.bias = b3;
  g.act = act;
  g.out_hi = m_hi;
  g.out_lo = m_lo;
  g.ldo_bf = ldm;
  int rc = mtt_gemm(&g, stream);
  if (rc || !w_head) return rc;
  if (!out_f32 || n_out <= 0) return set_error(MTT_ERR_BAD_SHAPE, "mtt_conv3x3_bn_act: fused head without output");
  mtt_gemm_desc h = {};
  h.a_hi = m_hi;
  h.a_lo = m_lo;
  h.lda = ldm;
  fill_b(h, w_head);
  h.M = (int32_t)rows;
  h.N = n_out;
  h.K = Cout;
  h.nsplit = ns;
  h.bias = b_head;
  h.out_f32 = out_f32;
  h.ldo_f32 = ldo;
  return mtt_gemm(&h, stream);
}

}  // extern "C"
