// HBM-bound kernels around the GEMMs: patch im2col, prompt broadcast, the windowed channel-prompt
// logits (token_trans / token_trans1 themselves run on the wgmma GEMM with gathered A rows), spatial/channel gating, cross-task reweighting and
// bilinear resampling.  All are coalesced along the channel (innermost NHWC / token-major) axis,
// float4 / bf16x2 vectorised where the layout allows, with grids sized by the data (>= several
// waves of 132 SMs at the benchmark shapes).
#include <stdlib.h>

#include "glue.cuh"
#include "host_common.h"
#include "postproc.cuh"

namespace mtt {

// ------------------------------------------------------------------------------------------------
// im2col for the stride-16 patch embedding (timm PatchEmbed: Conv2d(k = s = patch)); column order
// (c, ky, kx) matches conv.weight.reshape(C_out, -1).   reference: taskprompter.py:393
__global__ void __launch_bounds__(256)
im2col_patch_kernel(const float* __restrict__ img, int Cin, int H, int W, int patch, int gw, int P,
                    __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, long long ld) {
  const long long row = blockIdx.x;  // b * P + p
  const int b = (int)(row / P), pidx = (int)(row % P);
  const int py = pidx / gw, px = pidx % gw;
  const int K = Cin * patch * patch;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const int c = k / (patch * patch);
    const int r = k % (patch * patch);
    const int ky = r / patch, kx = r % patch;
    const float v = img[(((long long)b * Cin + c) * H + py * patch + ky) * W + px * patch + kx];
    store_split({hi, lo, ld}, row, k, v);
  }
}

// dst[(b*group + t) * ld + c] = src[t*C + c]     reference: taskprompter.py:397
__global__ void broadcast_rows_kernel(const float* __restrict__ src, float* __restrict__ dst, int B, int T,
                                      int C, long long group, long long ld) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)B * T * C;
  if (i >= total) return;
  const int c = (int)(i % C);
  const int t = (int)((i / C) % T);
  const int b = (int)(i / ((long long)C * T));
  dst[((long long)b * group + t) * ld + c] = src[(long long)t * C + c];
}

// ------------------------------------------------------------------------------------------------
// Raw channel logits  Rc[b,t,c,i,j] = sum_{pixel in window (i,j)} cp[b,t,pixel] * xn[b,pixel,c]
// reference: taskprompter.py:236-240,246 (the softmax.V after it is dead code and not reproduced).
constexpr int kMaxTasks = 8;
// block = 32 channels x 32 pixel groups; grid = (C/32, windows, B): the pixel reduction is split over
// the 32 groups and finished through shared memory, so the grid fills the chip even with one window.
__global__ void __launch_bounds__(1024)
chan_logits_kernel(const float* __restrict__ cp, const __nv_bfloat16* __restrict__ xh,
                   const __nv_bfloat16* __restrict__ xl, long long ldx, int N, int T, int C, int gh, int gw,
                   int nh, int nw, float* __restrict__ out) {
  extern __shared__ float scp[];  // [T][wh*ww] then [T][32][33] partials
  const int b = blockIdx.z, win = blockIdx.y;
  const int wi = win / nw, wj = win % nw;
  const int wh = gh / nh, ww = gw / nw, wp = wh * ww;
  const int P = gh * gw;
  float* red = scp + T * wp;
  const int tid = threadIdx.y * 32 + threadIdx.x;
  for (int i = tid; i < T * wp; i += 1024) {
    const int t = i / wp, q = i % wp;
    const int pix = (wi * wh + q / ww) * gw + wj * ww + q % ww;
    scp[i] = cp[((long long)b * T + t) * P + pix];
  }
  __syncthreads();
  const int c = blockIdx.x * 32 + threadIdx.x;
  float acc[kMaxTasks];
#pragma unroll
  for (int t = 0; t < kMaxTasks; ++t) acc[t] = 0.f;
  if (c < C) {
    for (int q = threadIdx.y; q < wp; q += 32) {
      const int pix = (wi * wh + q / ww) * gw + wj * ww + q % ww;
      const long long row = (long long)b * N + T + pix;
      float x = __bfloat162float(xh[row * ldx + c]);
      if (xl) x += __bfloat162float(xl[row * ldx + c]);
#pragma unroll
      for (int t = 0; t < kMaxTasks; ++t)
        if (t < T) acc[t] = fmaf(scp[t * wp + q], x, acc[t]);
    }
  }
#pragma unroll
  for (int t = 0; t < kMaxTasks; ++t)
    if (t < T) red[(t * 32 + threadIdx.y) * 33 + threadIdx.x] = acc[t];
  __syncthreads();
  if (threadIdx.y < T && c < C) {
    const int t = threadIdx.y;
    float s = 0.f;
    for (int g = 0; g < 32; ++g) s += red[(t * 32 + g) * 33 + threadIdx.x];
    out[((((long long)b * T + t) * C + c) * nh + wi) * nw + wj] = s;
  }
}

// ------------------------------------------------------------------------------------------------
// Spatial and channel gating (taskprompter.py:436-446 and :452-467), both in one pass over X:
//   Ys[b,pix,c] = X[b,pix,c] * (1 + R[b, c / dh, t, T + pix])
//   Yc[b,pix,c] = X[b,pix,c] * (1 + Rc[b, t, c, window(pix)])
// written as split-bf16 A operands of the two 1x1 decode convolutions.
// One block per patch row (b, pix), one thread per 8 consecutive channels: X is read ONCE (two float4) and gated for
// `nt` consecutive tasks; every plane is written with 16-byte stores. Task k's planes start k * task_stride elements
// after task t0's (the workspace layout of mtt_gated_conv1x1).
__global__ void __launch_bounds__(128)
gate_split_kernel(const float* __restrict__ x, long long ldx, long long x_group, long long x_off,
                  const float* __restrict__ logits, const float* __restrict__ rc, int t0, int nt, int T, int N, int H,
                  int dh, int C, int gh, int gw, int nh, int nw, __nv_bfloat16* __restrict__ ys_hi,
                  __nv_bfloat16* __restrict__ ys_lo, __nv_bfloat16* __restrict__ yc_hi,
                  __nv_bfloat16* __restrict__ yc_lo, long long ldy, long long task_stride) {
  const int P = gh * gw;
  const long long row = blockIdx.x;  // b * P + pix
  const int b = (int)(row / P), pix = (int)(row % P);
  const int nwin = nh * nw;
  const int win = chan_window(pix, gh, gw, nh, nw);
  const float* xr = x + ((long long)b * x_group + x_off + pix) * ldx;
  for (int c = threadIdx.x * 8; c < C; c += blockDim.x * 8) {
    const float4 xa = *reinterpret_cast<const float4*>(xr + c), xb = *reinterpret_cast<const float4*>(xr + c + 4);
    const float xv[8] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
    for (int k = 0; k < nt; ++k) {
      const int t = t0 + k;
      // spatial gate: one scalar per (head, pixel); the 8 channels of this thread lie in one head (dh % 8 == 0)
      const float g = logits[(((long long)b * H + c / dh) * T + t) * N + T + pix];
      const float* rcr = rc + (((long long)b * T + t) * C + c) * nwin + win;  // + i * nwin
      float gc[8];
      if (nwin == 1) {
        const float4 ra = *reinterpret_cast<const float4*>(rcr), rb = *reinterpret_cast<const float4*>(rcr + 4);
        gc[0] = ra.x; gc[1] = ra.y; gc[2] = ra.z; gc[3] = ra.w; gc[4] = rb.x; gc[5] = rb.y; gc[6] = rb.z; gc[7] = rb.w;
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) gc[i] = rcr[(long long)i * nwin];
      }
      uint4 sh, sl, ch, cl;
      split_pack2(xv[0] * (1.f + g), xv[1] * (1.f + g), sh.x, sl.x);
      split_pack2(xv[2] * (1.f + g), xv[3] * (1.f + g), sh.y, sl.y);
      split_pack2(xv[4] * (1.f + g), xv[5] * (1.f + g), sh.z, sl.z);
      split_pack2(xv[6] * (1.f + g), xv[7] * (1.f + g), sh.w, sl.w);
      split_pack2(xv[0] * (1.f + gc[0]), xv[1] * (1.f + gc[1]), ch.x, cl.x);
      split_pack2(xv[2] * (1.f + gc[2]), xv[3] * (1.f + gc[3]), ch.y, cl.y);
      split_pack2(xv[4] * (1.f + gc[4]), xv[5] * (1.f + gc[5]), ch.z, cl.z);
      split_pack2(xv[6] * (1.f + gc[6]), xv[7] * (1.f + gc[7]), ch.w, cl.w);
      const long long o = (long long)k * task_stride + row * ldy + c;
      *reinterpret_cast<uint4*>(ys_hi + o) = sh;
      if (ys_lo) *reinterpret_cast<uint4*>(ys_lo + o) = sl;
      *reinterpret_cast<uint4*>(yc_hi + o) = ch;
      if (yc_lo) *reinterpret_cast<uint4*>(yc_lo + o) = cl;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Cross-task reweighting weights (taskprompter.py:481-483):
//   w[b,t,j] = W2_t . gelu(W0_t . R[b, :, t, j] + b0_t) + b2_t       (two 1x1 convs over the head axis)
__global__ void ctr_weights_kernel(const float* __restrict__ logits, int B, int H, int T, int N,
                                   const float* __restrict__ w0, const float* __restrict__ b0,
                                   const float* __restrict__ w2, const float* __restrict__ b2,
                                   float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * T * T) return;
  const int j = i % T, t = (i / T) % T, b = i / (T * T);
  float acc = b2[t];
  for (int o = 0; o < H; ++o) {
    float hsum = b0[t * H + o];
    for (int h = 0; h < H; ++h)
      hsum = fmaf(w0[((long long)t * H + o) * H + h], logits[(((long long)b * H + h) * T + t) * N + j], hsum);
    acc = fmaf(w2[t * H + o], gelu_erf(hsum), acc);
  }
  out[i] = acc;
}

// acc[t][m, :] (+)= sum_j w[b(m), t, j] * F[j][m, :]     (taskprompter.py:484 + level sum :411)
__global__ void __launch_bounds__(256)
ctr_mix_kernel(const float* __restrict__ F, const float* __restrict__ w, float* __restrict__ acc, int T,
               long long M, int C, long long ld, int rows_per_batch, int accumulate) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // over M * C/4
  const int c4 = C >> 2;
  if (i >= M * c4) return;
  const long long m = i / c4;
  const int c = (int)(i % c4) * 4;
  const int b = (int)(m / rows_per_batch);
  float4 f[kMaxTasks];
#pragma unroll
  for (int j = 0; j < kMaxTasks; ++j)
    if (j < T) f[j] = *reinterpret_cast<const float4*>(F + ((long long)j * M + m) * ld + c);
#pragma unroll
  for (int t = 0; t < kMaxTasks; ++t) {
    if (t >= T) break;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = 0; j < kMaxTasks; ++j) {
      if (j >= T) break;
      const float wv = w[((long long)b * T + t) * T + j];
      s.x = fmaf(wv, f[j].x, s.x);
      s.y = fmaf(wv, f[j].y, s.y);
      s.z = fmaf(wv, f[j].z, s.z);
      s.w = fmaf(wv, f[j].w, s.w);
    }
    float4* dst = reinterpret_cast<float4*>(acc + ((long long)t * M + m) * ld + c);
    if (accumulate) {
      const float4 o = *dst;
      s.x += o.x; s.y += o.y; s.z += o.z; s.w += o.w;
    }
    *dst = s;
  }
}

// ------------------------------------------------------------------------------------------------
// Bilinear resize, align_corners = False (bilin_coord, postproc.cuh).  NHWC fp32 in; NHWC (fp32 and/or split) or
// NCHW out.

// One warp per (run of up to kBilinRun consecutive output pixels of one output row, chunk of 64 * NCH channels). A lane
// owns NCH channel pairs (c, c + 64, ...) and walks the run keeping the four corner values of each pair in registers:
// when the left source column advances by one the old right column becomes the new left one, so an x4 up-sampling
// (taskprompter.py:420: 32x32 -> 128x128, 350 channels) reads ~0.75 source values per output value from L2 instead of 4.
// The run walk with one pair per lane is issue-bound (about 120 instructions per lane per pixel, most of them 64-bit
// index arithmetic and the output-form / odd-channel branches) -- hence the FAST instantiation for the decoder's form
// (about 50 instructions per pixel), output pointers that advance by a stride, and two pairs per lane behind one
// coordinate computation.
// The interpolation expression and its order are those of the one-pixel form: bit-identical results.
constexpr int kBilinRun = 16;   // longest run; short rows / small maps get shorter runs so that the launch still fills the SMs
static int bilin_run_len(long long rows, int W2, int chunks) {
  int run = kBilinRun;
  while (run > 1 && rows * ((W2 + run - 1) / run) * chunks < (long long)sm_count() * 48) run >>= 1;
  return run;
}
// two channel pairs per lane on wide maps: one coordinate computation feeds both
static int bilin_pairs_per_lane(int C) { return C > 64 ? 2 : 1; }

template <int NCH, bool VEC, bool FAST>   // FAST: even C, both split planes, no fp32 output (the decoder's hot form)
__global__ void __launch_bounds__(256)
bilinear_nhwc_kernel(const float* __restrict__ in, long long ld_in, long long in_brows, long long in_off, int B,
                     int h, int w, int C, int H2, int W2, float sy, float sx, float* __restrict__ out_f32,
                     long long ld_f32, __nv_bfloat16* __restrict__ out_hi, __nv_bfloat16* __restrict__ out_lo,
                     long long ld_bf, long long out_brows, long long out_off, int accumulate, int run_len,
                     int runs_per_row, int chunks) {
  long long wid = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (wid >= (long long)B * H2 * runs_per_row * chunks) return;
  const int lane = threadIdx.x & 31;
  const int chunk = (int)(wid % chunks);
  wid /= chunks;
  const int run = (int)(wid % runs_per_row);
  wid /= runs_per_row;
  const int y = (int)(wid % H2), b = (int)(wid / H2);
  const int c = chunk * (64 * NCH) + lane * 2;   // this lane's pairs start at c + 64 j
  if (c >= C) return;
  bool ok[NCH], two[NCH];
#pragma unroll
  for (int j = 0; j < NCH; ++j) {
    ok[j] = c + 64 * j < C;
    two[j] = FAST || c + 64 * j + 1 < C;
  }
  int y0, y1;
  float ly;
  bilin_coord(y, sy, h, y0, y1, ly);
  const float hy = 1.f - ly;
  const float* ib = in + ((long long)b * in_brows + in_off) * ld_in + c;
  const float* row0 = ib + (long long)y0 * w * ld_in;
  const float* row1 = ib + (long long)y1 * w * ld_in;
  float2 t0[NCH], t1[NCH], b0[NCH], b1[NCH];   // top / bottom source rows at the cached columns cx0, cx1
#pragma unroll
  for (int j = 0; j < NCH; ++j) t0[j] = t1[j] = b0[j] = b1[j] = make_float2(0.f, 0.f);
  auto load_col = [&](int xx, float2 (&tt)[NCH], float2 (&bb)[NCH]) {
    const float* q0 = row0 + (long long)xx * ld_in;
    const float* q1 = row1 + (long long)xx * ld_in;
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
      if (!ok[j]) continue;
      if (VEC && two[j]) {
        tt[j] = *reinterpret_cast<const float2*>(q0 + 64 * j);
        bb[j] = *reinterpret_cast<const float2*>(q1 + 64 * j);
      } else {
        tt[j] = make_float2(q0[64 * j], two[j] ? q0[64 * j + 1] : 0.f);
        bb[j] = make_float2(q1[64 * j], two[j] ? q1[64 * j + 1] : 0.f);
      }
    }
  };
  int cx0 = -1, cx1 = -1;
  const int xbeg = run * run_len;
  const int xend = xbeg + run_len < W2 ? xbeg + run_len : W2;
  const long long opix0 = (long long)b * out_brows + out_off + (long long)y * W2 + xbeg;
  float* of = (!FAST && out_f32) ? out_f32 + opix0 * ld_f32 + c : nullptr;
  __nv_bfloat16* ohi = (FAST || out_hi) ? out_hi + opix0 * ld_bf + c : nullptr;
  __nv_bfloat16* olo = (FAST || (out_hi && out_lo)) ? out_lo + opix0 * ld_bf + c : nullptr;
  for (int x = xbeg; x < xend; ++x) {
    int x0, x1;
    float lx;
    bilin_coord(x, sx, w, x0, x1, lx);
    if (x0 != cx0 || x1 != cx1) {
      if (x0 == cx1) {
#pragma unroll
        for (int j = 0; j < NCH; ++j) {
          t0[j] = t1[j];
          b0[j] = b1[j];
        }
      } else if (x0 != cx0) {
        load_col(x0, t0, b0);
      }
      if (x1 == x0) {
#pragma unroll
        for (int j = 0; j < NCH; ++j) {
          t1[j] = t0[j];
          b1[j] = b0[j];
        }
      } else {
        load_col(x1, t1, b1);
      }
      cx0 = x0;
      cx1 = x1;
    }
    const float hx = 1.f - lx;
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
      if (!ok[j]) continue;
      float v0 = hy * (hx * t0[j].x + lx * t1[j].x) + ly * (hx * b0[j].x + lx * b1[j].x);
      float v1 = two[j] ? hy * (hx * t0[j].y + lx * t1[j].y) + ly * (hx * b0[j].y + lx * b1[j].y) : 0.f;
      if (!FAST && of) {
        float* o = of + 64 * j;
        if (accumulate) {
          v0 += o[0];
          if (two[j]) v1 += o[1];
        }
        o[0] = v0;
        if (two[j]) o[1] = v1;
      }
      if (FAST) {
        uint32_t hh, ll;
        split_pack2(v0, v1, hh, ll);
        *reinterpret_cast<uint32_t*>(ohi + 64 * j) = hh;
        *reinterpret_cast<uint32_t*>(olo + 64 * j) = ll;
      } else if (ohi) {
        uint32_t hh, ll;
        split_pack2(v0, v1, hh, ll);
        if (two[j]) {
          *reinterpret_cast<uint32_t*>(ohi + 64 * j) = hh;
          if (olo) *reinterpret_cast<uint32_t*>(olo + 64 * j) = ll;
        } else {
          ohi[64 * j] = __ushort_as_bfloat16((unsigned short)(hh & 0xFFFF));
          if (olo) olo[64 * j] = __ushort_as_bfloat16((unsigned short)(ll & 0xFFFF));
        }
      }
    }
    if (!FAST && of) of += ld_f32;
    if (FAST || ohi) ohi += ld_bf;
    if (FAST || olo) olo += ld_bf;
  }
}

// NHWC fp32 [B,h,w,C] -> NCHW fp32 [B,C,H2,W2]; one thread per output pixel, loop over channels.
__global__ void __launch_bounds__(256)
bilinear_to_nchw_kernel(const float* __restrict__ in, long long ld_in, long long in_brows, long long in_off, int B,
                        int h, int w, int C, int H2, int W2, float sy, float sx, float* __restrict__ out) {
  const long long opix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (opix >= (long long)B * H2 * W2) return;
  const int x = (int)(opix % W2), y = (int)((opix / W2) % H2), b = (int)(opix / ((long long)W2 * H2));
  int y0, y1, x0, x1;
  float ly, lx;
  bilin_coord(y, sy, h, y0, y1, ly);
  bilin_coord(x, sx, w, x0, x1, lx);
  const float* ib = in + ((long long)b * in_brows + in_off) * ld_in;
  const float* p00 = ib + ((long long)y0 * w + x0) * ld_in;
  const float* p01 = ib + ((long long)y0 * w + x1) * ld_in;
  const float* p10 = ib + ((long long)y1 * w + x0) * ld_in;
  const float* p11 = ib + ((long long)y1 * w + x1) * ld_in;
  const float hy = 1.f - ly, hx = 1.f - lx;
  for (int c = 0; c < C; ++c) {
    const float v = hy * (hx * p00[c] + lx * p01[c]) + ly * (hx * p10[c] + lx * p11[c]);
    out[(((long long)b * C + c) * H2 + y) * W2 + x] = v;
  }
}

// Sum of up to three bilinearly resized NHWC sources, written once as a split tensor: InvPT's multi-scale
// aggregation (invpt.py:528-539 accumulates the three stages' per-task maps at 8h x 8w) without the three
// read-modify-write passes over the full-resolution fp32 map.  One warp per output pixel.
struct BilinSrc {
  const float* p;
  long long ld, batch_rows, row_off;
  int h, w;
};
// Same run walk as bilinear_nhwc_kernel: a warp owns a run of consecutive output pixels of one row for a chunk of
// 64 * NCH channels, a lane NCH channel pairs, and each source's four corner values per pair stay in registers (round 2
// read 12 corner rows per output pixel from L2: 173 us per launch at InvPT cfg3). Per output value the sources are added
// in the same order with the same expression.
template <int NSRC, int NCH, bool VEC>
__global__ void __launch_bounds__(256)
bilinear_sum3_kernel(BilinSrc s0, BilinSrc s1, BilinSrc s2, int B, int C, int H2, int W2,
                     __nv_bfloat16* __restrict__ out_hi, __nv_bfloat16* __restrict__ out_lo, long long ld_bf,
                     int run_len, int runs_per_row, int chunks) {
  long long wid = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (wid >= (long long)B * H2 * runs_per_row * chunks) return;
  const int lane = threadIdx.x & 31;
  const int chunk = (int)(wid % chunks);
  wid /= chunks;
  const int run = (int)(wid % runs_per_row);
  wid /= runs_per_row;
  const int y = (int)(wid % H2), b = (int)(wid / H2);
  const int c = chunk * (64 * NCH) + lane * 2;   // C is even: a lane always owns full channel pairs c + 64 j
  if (c >= C) return;
  bool ok[NCH];
#pragma unroll
  for (int j = 0; j < NCH; ++j) ok[j] = c + 64 * j < C;
  const BilinSrc* ss[3] = {&s0, &s1, &s2};
  const float* row0[NSRC];
  const float* row1[NSRC];
  float hy[NSRC], ly[NSRC], sx[NSRC];
  long long ld[NSRC];
  int w[NSRC], cx0[NSRC], cx1[NSRC];
  float2 t0[NSRC][NCH], t1[NSRC][NCH], b0[NSRC][NCH], b1[NSRC][NCH];
#pragma unroll
  for (int i = 0; i < NSRC; ++i) {
    const BilinSrc& s = *ss[i];
    int y0, y1;
    bilin_coord(y, (float)s.h / (float)H2, s.h, y0, y1, ly[i]);
    hy[i] = 1.f - ly[i];
    sx[i] = (float)s.w / (float)W2;
    ld[i] = s.ld;
    w[i] = s.w;
    const float* ib = s.p + ((long long)b * s.batch_rows + s.row_off) * s.ld + c;
    row0[i] = ib + (long long)y0 * s.w * s.ld;
    row1[i] = ib + (long long)y1 * s.w * s.ld;
    cx0[i] = cx1[i] = -1;
#pragma unroll
    for (int j = 0; j < NCH; ++j) t0[i][j] = t1[i][j] = b0[i][j] = b1[i][j] = make_float2(0.f, 0.f);
  }
  auto load_col = [&](const float* q0, const float* q1, float2 (&tt)[NCH], float2 (&bb)[NCH]) {
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
      if (!ok[j]) continue;
      if (VEC) {
        tt[j] = *reinterpret_cast<const float2*>(q0 + 64 * j);
        bb[j] = *reinterpret_cast<const float2*>(q1 + 64 * j);
      } else {
        tt[j] = make_float2(q0[64 * j], q0[64 * j + 1]);
        bb[j] = make_float2(q1[64 * j], q1[64 * j + 1]);
      }
    }
  };
  const int xbeg = run * run_len;
  const int xend = xbeg + run_len < W2 ? xbeg + run_len : W2;
  const long long opix0 = ((long long)b * H2 + y) * W2 + xbeg;
  __nv_bfloat16* ohi = out_hi + opix0 * ld_bf + c;
  __nv_bfloat16* olo = out_lo ? out_lo + opix0 * ld_bf + c : nullptr;
  for (int x = xbeg; x < xend; ++x) {
    float v0[NCH], v1[NCH];
#pragma unroll
    for (int j = 0; j < NCH; ++j) v0[j] = v1[j] = 0.f;
#pragma unroll
    for (int i = 0; i < NSRC; ++i) {
      int x0, x1;
      float lx;
      bilin_coord(x, sx[i], w[i], x0, x1, lx);
      if (x0 != cx0[i] || x1 != cx1[i]) {
        if (x0 == cx1[i]) {
#pragma unroll
          for (int j = 0; j < NCH; ++j) {
            t0[i][j] = t1[i][j];
            b0[i][j] = b1[i][j];
          }
        } else if (x0 != cx0[i]) {
          load_col(row0[i] + (long long)x0 * ld[i], row1[i] + (long long)x0 * ld[i], t0[i], b0[i]);
        }
        if (x1 == x0) {
#pragma unroll
          for (int j = 0; j < NCH; ++j) {
            t1[i][j] = t0[i][j];
            b1[i][j] = b0[i][j];
          }
        } else {
          load_col(row0[i] + (long long)x1 * ld[i], row1[i] + (long long)x1 * ld[i], t1[i], b1[i]);
        }
        cx0[i] = x0;
        cx1[i] = x1;
      }
      const float hx = 1.f - lx;
#pragma unroll
      for (int j = 0; j < NCH; ++j) {
        v0[j] += hy[i] * (hx * t0[i][j].x + lx * t1[i][j].x) + ly[i] * (hx * b0[i][j].x + lx * b1[i][j].x);
        v1[j] += hy[i] * (hx * t0[i][j].y + lx * t1[i][j].y) + ly[i] * (hx * b0[i][j].y + lx * b1[i][j].y);
      }
    }
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
      if (!ok[j]) continue;
      uint32_t hh, ll;
      split_pack2(v0[j], v1[j], hh, ll);
      *reinterpret_cast<uint32_t*>(ohi + 64 * j) = hh;
      if (olo) *reinterpret_cast<uint32_t*>(olo + 64 * j) = ll;
    }
    ohi += ld_bf;
    if (olo) olo += ld_bf;
  }
}

// Bilinear resize to the output size fused with the reference's prediction post-processing
// (get_output_pixel, postproc.cuh): the full-resolution fp32 logits are never written. Kind 0 writes int64 [B,H2,W2],
// kinds 1, 2 and 4 fp32 [B,H2,W2] (depth: [B,H2,W2,1]), kind 3 fp32 [B,H2,W2,3].
__global__ void __launch_bounds__(256)
bilinear_postproc_kernel(const float* __restrict__ in, long long ld_in, int B, int h, int w, int C, int H2, int W2,
                         float sy, float sx, int kind, long long* __restrict__ out_i64, float* __restrict__ out_f32) {
  const long long opix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (opix >= (long long)B * H2 * W2) return;
  const int x = (int)(opix % W2), y = (int)((opix / W2) % H2), b = (int)(opix / ((long long)W2 * H2));
  int y0, y1, x0, x1;
  float ly, lx;
  bilin_coord(y, sy, h, y0, y1, ly);
  bilin_coord(x, sx, w, x0, x1, lx);
  const float* ib = in + (long long)b * h * w * ld_in;
  const float* p00 = ib + ((long long)y0 * w + x0) * ld_in;
  const float* p01 = ib + ((long long)y0 * w + x1) * ld_in;
  const float* p10 = ib + ((long long)y1 * w + x0) * ld_in;
  const float* p11 = ib + ((long long)y1 * w + x1) * ld_in;
  const float hy = 1.f - ly, hx = 1.f - lx;
  auto val = [&](int c) { return hy * (hx * p00[c] + lx * p01[c]) + ly * (hx * p10[c] + lx * p11[c]); };
  struct Sink {
    long long* i64;
    float* f32;
    long long opix;
    __device__ void cls(int c) { i64[opix] = c; }
    __device__ void f1(float v) { f32[opix] = v; }
    __device__ void ch(int c, float v) { f32[opix * 3 + c] = v; }
  } sink{out_i64, out_f32, opix};
  get_output_pixel(kind, C, val, sink);
}

}  // namespace mtt

using namespace mtt;
#define STREAM static_cast<cudaStream_t>(stream)

extern "C" int mtt_im2col_patch(const float* img, int32_t B, int32_t Cin, int32_t H, int32_t W,
                                int32_t patch, void* out_hi, void* out_lo, int64_t ld_out,
                                mtt_stream_t stream) {
  if (!img || !out_hi || B <= 0 || Cin <= 0 || patch <= 0 || H % patch || W % patch ||
      ld_out < (int64_t)Cin * patch * patch)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_im2col_patch: bad arguments");
  const int gw = W / patch, P = (H / patch) * gw;
  im2col_patch_kernel<<<B * P, 256, 0, STREAM>>>(img, Cin, H, W, patch, gw, P,
                                                static_cast<__nv_bfloat16*>(out_hi),
                                                static_cast<__nv_bfloat16*>(out_lo), ld_out);
  return check_launch("mtt_im2col_patch");
}

extern "C" int mtt_broadcast_rows(const float* src, float* dst, int32_t B, int32_t T, int32_t C,
                                  int64_t group_rows, int64_t ld, mtt_stream_t stream) {
  if (!src || !dst || B <= 0 || T <= 0 || C <= 0)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_broadcast_rows: bad arguments");
  const long long total = (long long)B * T * C;
  broadcast_rows_kernel<<<(unsigned)((total + 255) / 256), 256, 0, STREAM>>>(src, dst, B, T, C, group_rows,
                                                                            ld);
  return check_launch("mtt_broadcast_rows");
}

extern "C" int mtt_chan_logits(const float* cp, const void* xn_hi, const void* xn_lo, int64_t ldx,
                               int32_t B, int32_t N, int32_t T, int32_t C, int32_t gh, int32_t gw,
                               int32_t nh, int32_t nw, float* out, mtt_stream_t stream) {
  if (!cp || !xn_hi || !out || T <= 0 || T > kMaxTasks || nh <= 0 || nw <= 0 || gh % nh || gw % nw ||
      N != T + gh * gw)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_chan_logits: bad arguments (T=%d grid %dx%d windows %dx%d)",
                     T, gh, gw, nh, nw);
  const int wp = (gh / nh) * (gw / nw);
  const size_t smem = ((size_t)T * wp + (size_t)T * 32 * 33) * sizeof(float);
  if (smem > 200 * 1024) return set_error(MTT_ERR_BAD_SHAPE, "mtt_chan_logits: window too large");
  static bool attr[kMaxDevices] = {};  // per device
  const int dev_ = current_device();
  if (!attr[dev_]) {
    cudaFuncSetAttribute(chan_logits_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    attr[dev_] = true;
  }
  dim3 grid((C + 31) / 32, nh * nw, B);
  chan_logits_kernel<<<grid, dim3(32, 32), smem, STREAM>>>(cp, static_cast<const __nv_bfloat16*>(xn_hi),
                                                 static_cast<const __nv_bfloat16*>(xn_lo), ldx, N, T, C, gh,
                                                 gw, nh, nw, out);
  return check_launch("mtt_chan_logits");
}

extern "C" int mtt_gate_split(const float* x, int64_t ldx, int64_t x_group_rows, int64_t x_row_offset,
                              const float* prompt_logits, const float* chan_logits, int32_t task, int32_t ntasks,
                              int32_t B, int32_t T, int32_t N, int32_t H, int32_t C, int32_t gh, int32_t gw,
                              int32_t nh, int32_t nw, void* ys_hi, void* ys_lo, void* yc_hi, void* yc_lo, int64_t ldy,
                              int64_t task_stride, mtt_stream_t stream) {
  if (!x || !prompt_logits || !chan_logits || !ys_hi || !yc_hi || C % 8 || ldy % 8 || ldx % 4 || C % H || (C / H) % 8 ||
      task < 0 || ntasks < 1 || task + ntasks > T || gh % nh || gw % nw || task_stride % 8)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_gate_split: bad arguments (C=%d H=%d tasks [%d,%d) of %d)", C, H, task,
                     task + ntasks, T);
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  if (!al16(x) || !al16(ys_hi) || !al16(yc_hi) || (ys_lo && !al16(ys_lo)) || (yc_lo && !al16(yc_lo)) ||
      (nh * nw == 1 && !al16(chan_logits)))
    return set_error(MTT_ERR_MISALIGNED, "mtt_gate_split: pointers must be 16-byte aligned");
  gate_split_kernel<<<B * gh * gw, 128, 0, STREAM>>>(
      x, ldx, x_group_rows, x_row_offset, prompt_logits, chan_logits, task, ntasks, T, N, H, C / H, C, gh, gw, nh,
      nw, static_cast<__nv_bfloat16*>(ys_hi), static_cast<__nv_bfloat16*>(ys_lo),
      static_cast<__nv_bfloat16*>(yc_hi), static_cast<__nv_bfloat16*>(yc_lo), ldy, task_stride);
  return check_launch("mtt_gate_split");
}

extern "C" int mtt_ctr_weights(const float* prompt_logits, int32_t B, int32_t H, int32_t T, int32_t N,
                               const float* w0, const float* b0, const float* w2, const float* b2,
                               float* out, mtt_stream_t stream) {
  if (!prompt_logits || !w0 || !b0 || !w2 || !b2 || !out || T <= 0)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_ctr_weights: bad arguments");
  const int total = B * T * T;
  ctr_weights_kernel<<<(total + 127) / 128, 128, 0, STREAM>>>(prompt_logits, B, H, T, N, w0, b0, w2, b2,
                                                             out);
  return check_launch("mtt_ctr_weights");
}

extern "C" int mtt_ctr_mix(const float* F, const float* w, float* acc, int32_t T, int64_t M, int32_t C,
                           int64_t ld, int32_t rows_per_batch, int32_t accumulate, mtt_stream_t stream) {
  if (!F || !w || !acc || T <= 0 || T > kMaxTasks || C % 4 || ld % 4 || rows_per_batch <= 0)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_ctr_mix: bad arguments (T=%d C=%d ld=%lld)", T, C,
                     (long long)ld);
  const long long total = M * (C / 4);
  ctr_mix_kernel<<<(unsigned)((total + 255) / 256), 256, 0, STREAM>>>(F, w, acc, T, M, C, ld,
                                                                     rows_per_batch, accumulate);
  return check_launch("mtt_ctr_mix");
}

extern "C" int mtt_bilinear(const float* in, int64_t ld_in, int32_t B, int32_t h, int32_t w, int32_t C,
                            int32_t H2, int32_t W2, float* out_f32, int64_t ld_f32, void* out_hi,
                            void* out_lo, int64_t ld_bf, float* out_nchw, int32_t accumulate,
                            int64_t in_batch_rows, int64_t in_row_offset, int64_t out_batch_rows,
                            int64_t out_row_offset, mtt_stream_t stream) {
  if (!in || B <= 0 || h <= 0 || w <= 0 || C <= 0 || H2 <= 0 || W2 <= 0 ||
      (!out_f32 && !out_hi && !out_nchw))
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_bilinear: bad arguments");
  const float sy = (float)h / (float)H2, sx = (float)w / (float)W2;
  const long long opix = (long long)B * H2 * W2;
  if (in_batch_rows <= 0) in_batch_rows = (long long)h * w;
  if (out_batch_rows <= 0) out_batch_rows = (long long)H2 * W2;
  if (out_nchw) {
    bilinear_to_nchw_kernel<<<(unsigned)((opix + 255) / 256), 256, 0, STREAM>>>(
        in, ld_in, in_batch_rows, in_row_offset, B, h, w, C, H2, W2, sy, sx, out_nchw);
    int rc = check_launch("mtt_bilinear(nchw)");
    if (rc) return rc;
  }
  if (out_f32 || out_hi) {
    if (out_hi && (ld_bf % 2))
      return set_error(MTT_ERR_MISALIGNED, "mtt_bilinear: ld_bf must be even");
    static int force_nch = -1;   // MTT_BILINEAR_PAIRS: 1 / 2 / 4 channel pairs per lane (tuning aid); 0 = by channel count
    if (force_nch < 0) {
      const char* e = getenv("MTT_BILINEAR_PAIRS");
      force_nch = e ? atoi(e) : 0;
    }
    const int nch = (force_nch == 1 || force_nch == 2 || force_nch == 4) ? force_nch : bilin_pairs_per_lane(C);
    const int chunks = (C + 64 * nch - 1) / (64 * nch);
    const int run_len = bilin_run_len((long long)B * H2, W2, chunks);
    const int runs = (W2 + run_len - 1) / run_len;
    const long long warps = (long long)B * H2 * runs * chunks;
    const unsigned blocks = (unsigned)((warps + 7) / 8);
    const bool vec = (ld_in % 2 == 0) && (reinterpret_cast<uintptr_t>(in) % 8 == 0);
    const bool fast = vec && (C % 2 == 0) && out_hi && out_lo && !out_f32;
#define MTT_BILIN(NCH, V, F)                                                                                             \
  bilinear_nhwc_kernel<NCH, V, F><<<blocks, 256, 0, STREAM>>>(                                                            \
      in, ld_in, in_batch_rows, in_row_offset, B, h, w, C, H2, W2, sy, sx, out_f32, ld_f32,                               \
      static_cast<__nv_bfloat16*>(out_hi), static_cast<__nv_bfloat16*>(out_lo), ld_bf, out_batch_rows, out_row_offset,   \
      accumulate, run_len, runs, chunks)
#define MTT_BILIN_N(NCH) do { if (fast) MTT_BILIN(NCH, true, true); else if (vec) MTT_BILIN(NCH, true, false); \
                              else MTT_BILIN(NCH, false, false); } while (0)
    if (nch == 4) MTT_BILIN_N(4); else if (nch == 2) MTT_BILIN_N(2); else MTT_BILIN_N(1);
#undef MTT_BILIN_N
#undef MTT_BILIN
    return check_launch("mtt_bilinear(nhwc)");
  }
  return MTT_OK;
}

extern "C" int mtt_bilinear_postproc(const float* in, int64_t ld_in, int32_t B, int32_t h, int32_t w, int32_t C,
                                     int32_t H2, int32_t W2, int32_t kind, int64_t* out_i64, float* out_f32,
                                     mtt_stream_t stream) {
  const int need_c[5] = {1, 1, 2, 3, 1};
  if (!in || B <= 0 || h <= 0 || w <= 0 || H2 <= 0 || W2 <= 0 || kind < 0 || kind > 4 || C < need_c[kind] ||
      (kind == 0 ? !out_i64 : !out_f32))
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_bilinear_postproc: bad arguments (kind=%d C=%d)", kind, C);
  const float sy = (float)h / (float)H2, sx = (float)w / (float)W2;
  const long long opix = (long long)B * H2 * W2;
  bilinear_postproc_kernel<<<(unsigned)((opix + 255) / 256), 256, 0, STREAM>>>(
      in, ld_in, B, h, w, C, H2, W2, sy, sx, kind, reinterpret_cast<long long*>(out_i64), out_f32);
  return check_launch("mtt_bilinear_postproc");
}

extern "C" int mtt_bilinear_sum3(const mtt_bilinear_src* srcs, int32_t nsrc, int32_t B, int32_t C, int32_t H2,
                                 int32_t W2, void* out_hi, void* out_lo, int64_t ld_bf, mtt_stream_t stream) {
  if (!srcs || nsrc < 1 || nsrc > 3 || B <= 0 || C <= 0 || (C & 1) || (ld_bf & 1) || !out_hi)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_bilinear_sum3: bad arguments (nsrc=%d C=%d)", nsrc, C);
  BilinSrc s[3] = {};
  for (int i = 0; i < nsrc; ++i) {
    if (!srcs[i].in || srcs[i].h <= 0 || srcs[i].w <= 0)
      return set_error(MTT_ERR_BAD_SHAPE, "mtt_bilinear_sum3: bad source %d", i);
    s[i].p = srcs[i].in;
    s[i].ld = srcs[i].ld_in;
    s[i].h = srcs[i].h;
    s[i].w = srcs[i].w;
    s[i].batch_rows = srcs[i].batch_rows > 0 ? srcs[i].batch_rows : (long long)srcs[i].h * srcs[i].w;
    s[i].row_off = srcs[i].row_offset;
  }
  bool vec = true;
  for (int i = 0; i < nsrc; ++i) vec = vec && (s[i].ld % 2 == 0) && (reinterpret_cast<uintptr_t>(s[i].p) % 8 == 0);
  const int nch = C > 64 ? 2 : 1;
  const int chunks = (C + 64 * nch - 1) / (64 * nch);
  const int run_len = bilin_run_len((long long)B * H2, W2, chunks);
  const int runs = (W2 + run_len - 1) / run_len;
  const long long warps = (long long)B * H2 * runs * chunks;
  const unsigned blocks = (unsigned)((warps + 7) / 8);
  auto hi = static_cast<__nv_bfloat16*>(out_hi);
  auto lo = static_cast<__nv_bfloat16*>(out_lo);
#define MTT_SUM3(NS, NC, V) \
  bilinear_sum3_kernel<NS, NC, V><<<blocks, 256, 0, STREAM>>>(s[0], s[1], s[2], B, C, H2, W2, hi, lo, ld_bf, run_len, runs, chunks)
#define MTT_SUM3_V(NS, NC) do { if (vec) MTT_SUM3(NS, NC, true); else MTT_SUM3(NS, NC, false); } while (0)
  if (nch == 2) {
    if (nsrc == 1) MTT_SUM3_V(1, 2); else if (nsrc == 2) MTT_SUM3_V(2, 2); else MTT_SUM3_V(3, 2);
  } else {
    if (nsrc == 1) MTT_SUM3_V(1, 1); else if (nsrc == 2) MTT_SUM3_V(2, 1); else MTT_SUM3_V(3, 1);
  }
#undef MTT_SUM3_V
#undef MTT_SUM3
  return check_launch("mtt_bilinear_sum3");
}
