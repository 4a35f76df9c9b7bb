// Kernels of the Swin-backbone TaskPrompter (SURVEY.md section 8f N2; reference
// TP/models/transformers/taskprompter_swin.py, cited as TP:line). Everything dense (qkv / proj / MLP / chan_kv /
// PatchMerging reduction / decoder convs) runs on mtt_gemm; these are the window bookkeeping, the window attention with
// prompts, relative-position bias and shift mask, the channel attention and the small PatchMerging helpers.
//
// Joint window stream: for image b and window w (row-major over the padded, cyclically shifted map) the rows
// [(b * nW + w) * (T + ws^2), +T) are the T (normalised) task prompts and the next ws^2 rows the window's tokens in
// row-major order (TP:177-181 puts the prompts FIRST in every window).
#include <math.h>

#include "glue.cuh"
#include "host_common.h"

namespace mtt {

struct WinGeom {
  int B, H, W, Hp, Wp, ws, shift, nWx, nW, wl, T, C;
};

// source pixel (b-relative index y * W + x) of token i of window w, or -1 for zero padding (TP:326-337: pad AFTER the
// norm, then roll by -shift: rolled (y', x') reads padded (y' + shift, x' + shift) mod (Hp, Wp))
__device__ __forceinline__ int win_source(const WinGeom& g, int w, int i) {
  const int y = (w / g.nWx) * g.ws + i / g.ws, x = (w % g.nWx) * g.ws + i % g.ws;
  int sy = y + g.shift, sx = x + g.shift;
  if (sy >= g.Hp) sy -= g.Hp;
  if (sx >= g.Wp) sx -= g.Wp;
  return (sy < g.H && sx < g.W) ? sy * g.W + sx : -1;
}

// ---- window partition + prompt replication: fp32 rows -> split rows of the joint window stream -----------------------
__global__ void __launch_bounds__(256)
swin_gather_kernel(const float* __restrict__ xn, long long ldx, const float* __restrict__ pn, long long ldp, WinGeom g,
                   __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, long long ld) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int per = g.T + g.wl;
  if (row >= (long long)g.B * g.nW * per) return;
  const int lane = threadIdx.x & 31;
  const int tok = (int)(row % per), w = (int)((row / per) % g.nW), b = (int)(row / ((long long)per * g.nW));
  const float* src = nullptr;
  if (tok < g.T) {
    src = pn + ((long long)b * g.T + tok) * ldp;
  } else {
    const int s = win_source(g, w, tok - g.T);
    if (s >= 0) src = xn + ((long long)b * g.H * g.W + s) * ldx;
  }
  __nv_bfloat16* dh = hi + row * ld;
  __nv_bfloat16* dl = lo ? lo + row * ld : nullptr;
  for (int c = lane * 2; c < g.C; c += 64) {
    const float a = src ? src[c] : 0.f, bq = (src && c + 1 < g.C) ? src[c + 1] : 0.f;
    uint32_t h, l;
    split_pack2(a, bq, h, l);
    if (c + 1 < g.C) {
      *reinterpret_cast<uint32_t*>(dh + c) = h;
      if (dl) *reinterpret_cast<uint32_t*>(dl + c) = l;
    } else {
      dh[c] = __ushort_as_bfloat16((unsigned short)(h & 0xFFFF));
      if (dl) dl[c] = __ushort_as_bfloat16((unsigned short)(l & 0xFFFF));
    }
  }
}

// ---- window attention (TP:183-206) ------------------------------------------------------------------------------------
// One CTA per (window, head); thread i owns query row i of the N = T + ws^2 tokens and runs an online softmax over the
// keys. K and V of the window are staged in shared memory as fp32 and read as float4 broadcasts (every thread reads the
// same key). The relative-position bias and the shift mask apply to patch x patch entries only (TP:196, :201) and are
// read through their TRANSPOSES so that consecutive threads read consecutive addresses. Prompt rows export their raw
// q . k (TP:189). Measured on Swin-B 1024x2048 (24 launches per forward): float2 reads 250 us per launch; two query
// rows per thread (half the shared-memory reads, 168 registers, 96 threads) was SLOWER (forward 23.6 -> 25.1 ms).
template <int DH>
__global__ void __launch_bounds__(192)
swin_attn_kernel(const __nv_bfloat16* __restrict__ q_hi, const __nv_bfloat16* __restrict__ q_lo, long long ldq, int C,
                 int heads, int T, int L, int nW, float scale, const float* __restrict__ biasT,
                 const float* __restrict__ maskT, __nv_bfloat16* __restrict__ o_hi, __nv_bfloat16* __restrict__ o_lo,
                 long long ldo, float* __restrict__ raw) {
  extern __shared__ __align__(16) float sm[];
  const int N = T + L;
  float* sK = sm;               // [N][DH]
  float* sV = sm + N * DH;      // [N][DH]
  const int bw = blockIdx.x, h = blockIdx.y;
  const long long row0 = (long long)bw * N;
  auto ld_f = [&](long long r, int col) {
    float v = __bfloat162float(q_hi[r * ldq + col]);
    if (q_lo) v += __bfloat162float(q_lo[r * ldq + col]);
    return v;
  };
  for (int i = threadIdx.x; i < N * DH; i += blockDim.x) {
    const int r = i / DH, d = i % DH;
    sK[i] = ld_f(row0 + r, C + h * DH + d);
    sV[i] = ld_f(row0 + r, 2 * C + h * DH + d);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    // q and the output accumulator as packed fp32 pairs (FFMA2); the accumulator is rescaled only when the running
    // maximum moves
    float2 q[DH / 2], o[DH / 2];
#pragma unroll
    for (int d = 0; d < DH / 2; ++d) {
      q[d] = make_float2(ld_f(row0 + i, h * DH + 2 * d), ld_f(row0 + i, h * DH + 2 * d + 1));
      o[d] = make_float2(0.f, 0.f);
    }
    float m = -INFINITY, l = 0.f;
    const bool patch_q = i >= T;
    const float* bcol = patch_q ? biasT + ((long long)h * L) * L + (i - T) : nullptr;                  // + (j - T) * L
    const float* mcol = (patch_q && maskT) ? maskT + ((long long)(bw % nW) * L) * L + (i - T) : nullptr;
    float* rrow = (!patch_q && raw) ? raw + (((long long)bw * heads + h) * T + i) * L : nullptr;
    for (int j = 0; j < N; ++j) {
      const float4* kj = reinterpret_cast<const float4*>(sK + j * DH);
      float2 acc = make_float2(0.f, 0.f);
#pragma unroll
      for (int d = 0; d < DH / 4; ++d) {
        const float4 k4 = kj[d];
        acc = ffma2(q[2 * d], make_float2(k4.x, k4.y), acc);
        acc = ffma2(q[2 * d + 1], make_float2(k4.z, k4.w), acc);
      }
      float s = acc.x + acc.y;
      if (rrow && j >= T) rrow[j - T] = s;
      s *= scale;
      if (patch_q && j >= T) {
        s += bcol[(long long)(j - T) * L];
        if (mcol) s += mcol[(long long)(j - T) * L];
      }
      if (s > m) {                                   // new running maximum: rescale what has been accumulated
        const float a = __expf(m - s);
        l *= a;
#pragma unroll
        for (int d = 0; d < DH / 2; ++d) o[d] = make_float2(o[d].x * a, o[d].y * a);
        m = s;
      }
      const float p = __expf(s - m);
      l += p;
      const float2 p2 = make_float2(p, p);
      const float4* vj = reinterpret_cast<const float4*>(sV + j * DH);
#pragma unroll
      for (int d = 0; d < DH / 4; ++d) {
        const float4 v4 = vj[d];
        o[2 * d] = ffma2(p2, make_float2(v4.x, v4.y), o[2 * d]);
        o[2 * d + 1] = ffma2(p2, make_float2(v4.z, v4.w), o[2 * d + 1]);
      }
    }
    const float inv = 1.f / l;
    __nv_bfloat16* dh = o_hi + (row0 + i) * ldo + h * DH;
    __nv_bfloat16* dl = o_lo ? o_lo + (row0 + i) * ldo + h * DH : nullptr;
#pragma unroll
    for (int d = 0; d < DH / 2; ++d) {
      uint32_t hh, ll;
      split_pack2(o[d].x * inv, o[d].y * inv, hh, ll);
      *reinterpret_cast<uint32_t*>(dh + 2 * d) = hh;
      if (dl) *reinterpret_cast<uint32_t*>(dl + 2 * d) = ll;
    }
  }
}

// ---- window reverse + un-shift + crop: xa, x += xa; prompt-row logits onto the map (TP:343-360, :399) ----------------
__global__ void __launch_bounds__(256)
swin_scatter_kernel(const float* __restrict__ o, long long ldo, WinGeom g, float* __restrict__ xa, long long ldxa,
                    float* __restrict__ x, long long ldx) {
  const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);   // (b, w, i)
  if (r >= (long long)g.B * g.nW * g.wl) return;
  const int lane = threadIdx.x & 31;
  const int i = (int)(r % g.wl), w = (int)((r / g.wl) % g.nW), b = (int)(r / ((long long)g.wl * g.nW));
  const int s = win_source(g, w, i);
  if (s < 0) return;
  const float* src = o + (((long long)b * g.nW + w) * (g.T + g.wl) + g.T + i) * ldo;
  const long long pix = (long long)b * g.H * g.W + s;
  for (int c = lane; c < g.C; c += 32) {
    const float v = src[c];
    xa[pix * ldxa + c] = v;
    x[pix * ldx + c] += v;
  }
}

// p[b, t, :] += mean over the windows of the prompt rows of the attention output (TP:210). Grid (B*T, C / 64): 64
// channels x 4 window groups per block, fixed-order reduction in shared memory.
__global__ void __launch_bounds__(256)
swin_prompt_mean_kernel(const float* __restrict__ o, long long ldo, WinGeom g, float* __restrict__ p, long long ldp) {
  __shared__ float part[4][64];
  const int bt = blockIdx.x, b = bt / g.T, t = bt % g.T;
  const int cl = threadIdx.x & 63, grp = threadIdx.x >> 6;
  const int c = blockIdx.y * 64 + cl;
  float acc = 0.f;
  if (c < g.C)
    for (int w = grp; w < g.nW; w += 4) acc += o[(((long long)b * g.nW + w) * (g.T + g.wl) + t) * ldo + c];
  part[grp][cl] = acc;
  __syncthreads();
  if (grp == 0 && c < g.C)
    p[(long long)bt * ldp + c] += (part[0][cl] + part[1][cl] + part[2][cl] + part[3][cl]) / (float)g.nW;
}

// raw [B*nW, heads, T, wl] -> logits [B, heads, T, T + H*W] at column T + pixel
__global__ void __launch_bounds__(256)
swin_logits_kernel(const float* __restrict__ raw, WinGeom g, int heads, float* __restrict__ logits) {
  const long long n = (long long)g.B * g.nW * heads * g.T * g.wl;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(e % g.wl);
    const int t = (int)((e / g.wl) % g.T);
    const int h = (int)((e / ((long long)g.wl * g.T)) % heads);
    const long long bw = e / ((long long)g.wl * g.T * heads);
    const int w = (int)(bw % g.nW), b = (int)(bw / g.nW);
    const int s = win_source(g, w, i);
    if (s >= 0) logits[(((long long)b * heads + h) * g.T + t) * (g.T + g.H * g.W) + g.T + s] = raw[e];
  }
}

// ---- [B, L, C] fp32 -> split [B*C, ld >= L] (the A operand of chan_kv, TP:379; dY^T / P^T / dS^T of the training step) --
// Tile = 64 rows (L) x 32 columns (C): 128-byte row reads, and every output row (one column of the input) is written as 64
// consecutive bf16 = 128 bytes (one bf16x2 per lane).
__global__ void __launch_bounds__(256)
transpose_split_kernel(const float* __restrict__ in, long long ld_in, int L, int C, __nv_bfloat16* __restrict__ hi,
                       __nv_bfloat16* __restrict__ lo, long long ld) {
  __shared__ float tile[64][33];
  const int b = blockIdx.z;
  const int l0 = blockIdx.x * 64, c0 = blockIdx.y * 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* src = in + (long long)b * L * ld_in;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int l = l0 + warp * 8 + k, c = c0 + lane;
    tile[warp * 8 + k][lane] = (l < L && c < C) ? src[(long long)l * ld_in + c] : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int c = c0 + warp * 4 + k;
    const int l = l0 + 2 * lane;
    if (c >= C || l >= L) continue;
    store_split2({hi, lo, ld}, (long long)b * C + c, l, tile[2 * lane][warp * 4 + k], tile[2 * lane + 1][warp * 4 + k],
                 l + 1 < L, false);
  }
}

// ---- channel attention (TP:383-396) ------------------------------------------------------------------------------------
// Grid (b, window g of the sqrt(ce) x sqrt(ce) embedding grid, task t) x chunks of 32 embedding columns. Every block
// computes the logits of its prompt against all C channels (warp per channel, lanes over the window's embedding
// entries: coalesced), the softmax statistics, and then ITS 32 output columns (8 channel groups x 32 columns, reduced in
// shared memory in a fixed order). Block y == 0 also writes raw_chan. kv [B*C, 2 ce] fp32 (k | v), q [B*T, ce]; the ce
// axis is (nh, wh, nw, ww).
__global__ void __launch_bounds__(256)
swin_chan_attn_kernel(const float* __restrict__ q, long long ldq, const float* __restrict__ kv, long long ldkv, int T, int C,
                      int ce, int nh, int nw, float scale, float* __restrict__ co, long long ldco,
                      __nv_bfloat16* __restrict__ cs_hi, __nv_bfloat16* __restrict__ cs_lo, long long ldcs,
                      float* __restrict__ rc) {
  extern __shared__ float sm[];
  const int r = (int)(sqrtf((float)ce) + 0.5f);
  const int wh = r / nh, ww = r / nw, we = wh * ww;
  float* sq = sm;            // [we]
  float* sp = sm + we;       // [C]
  __shared__ float red[256];
  const int t = blockIdx.x % T, g = (blockIdx.x / T) % (nh * nw), b = blockIdx.x / (T * nh * nw);
  const int ga = g / nw, gb = g % nw;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  auto eidx = [&](int e) { return ((ga * wh + e / ww) * nw + gb) * ww + e % ww; };
  for (int e = threadIdx.x; e < we; e += blockDim.x) sq[e] = q[((long long)b * T + t) * ldq + eidx(e)];
  __syncthreads();
  for (int c = warp; c < C; c += 8) {                      // logits: warp per channel
    const float* kr = kv + ((long long)b * C + c) * ldkv;
    float s = 0.f;
    for (int e = lane; e < we; e += 32) s = fmaf(sq[e], kr[eidx(e)], s);
    s = warp_sum(s);
    if (lane == 0) {
      if (blockIdx.y == 0) rc[(((long long)b * T + t) * C + c) * (nh * nw) + g] = s;   // raw_chan [B,T,C,nh,nw] (TP:391)
      sp[c] = s * scale;
    }
  }
  __syncthreads();
  float mx = -INFINITY;
  for (int c = threadIdx.x; c < C; c += blockDim.x) mx = fmaxf(mx, sp[c]);
  red[threadIdx.x] = mx;
  __syncthreads();
  for (int s = blockDim.x >> 1; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] = fmaxf(red[threadIdx.x], red[threadIdx.x + s]);
    __syncthreads();
  }
  mx = red[0];
  __syncthreads();
  float sum = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float p = __expf(sp[c] - mx);
    sp[c] = p;
    sum += p;
  }
  red[threadIdx.x] = sum;
  __syncthreads();
  for (int s = blockDim.x >> 1; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  const float inv = 1.f / red[0];
  __syncthreads();
  // outputs: this block's 32 embedding columns, 8 channel groups
  const int e = blockIdx.y * 32 + lane;
  float acc = 0.f;
  int col = 0;
  if (e < we) {
    col = eidx(e);
    for (int c = warp; c < C; c += 8) acc = fmaf(sp[c], kv[((long long)b * C + c) * ldkv + ce + col], acc);
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  if (warp == 0 && e < we) {
    float tot = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) tot += red[k * 32 + lane];
    tot *= inv;
    const long long orow = (long long)b * T + t;
    co[orow * ldco + col] = tot;
    store_split({cs_hi, cs_lo, ldcs}, orow, col, tot);
  }
}

// ---- PatchMerging helpers (TP:441-447, :458-466) ------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
swin_merge_kernel(const float* __restrict__ x, long long ldx, int B, int H, int W, int C, float* __restrict__ out,
                  long long ldo) {
  const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);   // (b, y2, x2, quadrant)
  const int H2 = H / 2, W2 = W / 2;
  if (r >= (long long)B * H2 * W2 * 4) return;
  const int lane = threadIdx.x & 31;
  const int qd = (int)(r & 3);
  const long long pix = r >> 2;
  const int x2 = (int)(pix % W2), y2 = (int)((pix / W2) % H2), b = (int)(pix / ((long long)W2 * H2));
  const int dy = qd & 1, dx = qd >> 1;                   // order (0,0), (1,0), (0,1), (1,1) (TP:441-444)
  const float* src = x + (((long long)b * H + 2 * y2 + dy) * W + 2 * x2 + dx) * ldx;
  float* dst = out + pix * ldo + (long long)qd * C;
  for (int c = lane; c < C; c += 32) dst[c] = src[c];
}

// stride-2 3x3 convolution (pad 1) over small channel counts on maps stored with a row prefix:
// in[b, ci, in_off + y * W + x] (channel stride in_stride) -> out[b, co, out_off + y2 * W2 + x2]
__global__ void __launch_bounds__(256)
conv3x3_s2_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias, int B, int Cin,
                  int Cout, int H, int W, long long in_stride, int in_off, long long out_stride, int out_off,
                  float* __restrict__ out) {
  const int H2 = H / 2, W2 = W / 2;
  const long long n = (long long)B * Cout * H2 * W2;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const int x2 = (int)(e % W2), y2 = (int)((e / W2) % H2);
    const int co = (int)((e / ((long long)W2 * H2)) % Cout), b = (int)(e / ((long long)W2 * H2 * Cout));
    float acc = bias ? bias[co] : 0.f;
    for (int ci = 0; ci < Cin; ++ci) {
      const float* ip = in + ((long long)b * Cin + ci) * in_stride + in_off;
      const float* wp = w + ((long long)co * Cin + ci) * 9;
#pragma unroll
      for (int ky = 0; ky < 3; ++ky) {
        const int y = 2 * y2 + ky - 1;
        if (y < 0 || y >= H) continue;
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          const int x = 2 * x2 + kx - 1;
          if (x < 0 || x >= W) continue;
          acc = fmaf(wp[ky * 3 + kx], ip[(long long)y * W + x], acc);
        }
      }
    }
    out[((long long)b * Cout + co) * out_stride + out_off + (long long)y2 * W2 + x2] = acc;
  }
}

// out[bt, o, w] = sum_c Wt[o, c] * rc[bt, c, w] (process_chan_attn over the channel axis of raw_chan, TP:463-466)
__global__ void __launch_bounds__(256)
chan_up_kernel(const float* __restrict__ rc, const float* __restrict__ w, int BT, int C, int Cout, int nwin,
               float* __restrict__ out) {
  const long long n = (long long)BT * Cout * nwin;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const int wn = (int)(e % nwin), o = (int)((e / nwin) % Cout);
    const long long bt = e / ((long long)nwin * Cout);
    const float* r = rc + bt * C * nwin + wn;
    const float* wr = w + (long long)o * C;
    float acc = 0.f;
    for (int c = 0; c < C; ++c) acc = fmaf(wr[c], r[(long long)c * nwin], acc);
    out[e] = acc;
  }
}

// ---- prompt-row logit maps between the gating layout and the reference's raw_spa_attn ----------------------------------
// logits [rows, T + L] holds map r at columns [T, T + L); maps [rows, L] is the reference's [B, heads, T, H, W]. One block
// row per map, consecutive threads on consecutive columns of both sides: coalesced reads and writes. to_maps = 0 writes
// the logits' map columns only (their first T columns are not part of the map and stay as they are).
__global__ void __launch_bounds__(256)
swin_logit_maps_kernel(const float* __restrict__ src, float* __restrict__ dst, int T, int L, int to_maps) {
  const long long r = blockIdx.y;
  const long long ld_src = to_maps ? T + L : L, ld_dst = to_maps ? L : T + L;
  const int off_src = to_maps ? T : 0, off_dst = to_maps ? 0 : T;
  const float* s = src + r * ld_src + off_src;
  float* d = dst + r * ld_dst + off_dst;
  for (int l = blockIdx.x * blockDim.x + threadIdx.x; l < L; l += gridDim.x * blockDim.x) d[l] = s[l];
}

static int make_geom(WinGeom& g, int B, int H, int W, int C, int T, int ws, int shift) {
  if (B <= 0 || H <= 0 || W <= 0 || C <= 0 || T < 0 || ws <= 0 || shift < 0 || shift >= ws)
    return set_error(MTT_ERR_BAD_SHAPE, "swin: bad window geometry (B=%d %dx%d C=%d T=%d ws=%d shift=%d)", B, H, W, C, T, ws,
                     shift);
  g.B = B;
  g.H = H;
  g.W = W;
  g.C = C;
  g.T = T;
  g.ws = ws;
  g.shift = shift;
  g.Hp = H + (ws - H % ws) % ws;
  g.Wp = W + (ws - W % ws) % ws;
  g.nWx = g.Wp / ws;
  g.nW = (g.Hp / ws) * g.nWx;
  g.wl = ws * ws;
  return MTT_OK;
}

}  // namespace mtt

using namespace mtt;
#define STREAM static_cast<cudaStream_t>(stream)

extern "C" {

int mtt_swin_window_gather(const float* xn, int64_t ldx, const float* pn, int64_t ldp, int32_t B, int32_t H, int32_t W,
                           int32_t C, int32_t T, int32_t ws, int32_t shift, void* out_hi, void* out_lo, int64_t ld_out,
                           mtt_stream_t stream) {
  WinGeom g;
  int rc = make_geom(g, B, H, W, C, T, ws, shift);
  if (rc) return rc;
  if (!xn || (T > 0 && !pn) || !out_hi || ld_out < C || (ld_out & 1))
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_swin_window_gather: bad arguments");
  const long long rows = (long long)B * g.nW * (T + g.wl);
  swin_gather_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, STREAM>>>(xn, ldx, pn, ldp, g, static_cast<__nv_bfloat16*>(out_hi),
                                                                    static_cast<__nv_bfloat16*>(out_lo), ld_out);
  return check_launch("mtt_swin_window_gather");
}

int mtt_swin_window_attention(const void* qkv_hi, const void* qkv_lo, int64_t ldq, int32_t BW, int32_t nW, int32_t T,
                              int32_t L, int32_t heads, int32_t head_dim, float scale, const float* biasT,
                              const float* maskT, void* out_hi, void* out_lo, int64_t ldo, float* raw,
                              mtt_stream_t stream) {
  if (!qkv_hi || !out_hi || !biasT || BW <= 0 || nW <= 0 || BW % nW || T < 0 || L <= 0 || heads <= 0 || (ldo & 1))
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_swin_window_attention: bad arguments");
  const int N = T + L, C = heads * head_dim;
  const size_t smem = (size_t)2 * N * head_dim * sizeof(float);
  if (smem > 200 * 1024) return set_error(MTT_ERR_BAD_SHAPE, "mtt_swin_window_attention: window too large (N=%d)", N);
  const __nv_bfloat16* qh = static_cast<const __nv_bfloat16*>(qkv_hi);
  const __nv_bfloat16* ql = static_cast<const __nv_bfloat16*>(qkv_lo);
  __nv_bfloat16* oh = static_cast<__nv_bfloat16*>(out_hi);
  __nv_bfloat16* ol = static_cast<__nv_bfloat16*>(out_lo);
  const int threads = N <= 64 ? 64 : (N <= 128 ? 128 : 192);
  dim3 grid(BW, heads);
#define MTT_SWIN_ATTN(DH)                                                                                        \
  case DH: {                                                                                                     \
    static bool attr[kMaxDevices] = {};                                                                          \
    const int dev_ = current_device();                                                                           \
    if (!attr[dev_]) {                                                                                           \
      cudaFuncSetAttribute(swin_attn_kernel<DH>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);       \
      attr[dev_] = true;                                                                                         \
    }                                                                                                            \
    swin_attn_kernel<DH><<<grid, threads, smem, STREAM>>>(qh, ql, ldq, C, heads, T, L, nW, scale, biasT, maskT, oh, ol, \
                                                          ldo, raw);                                             \
  } break;
  switch (head_dim) {
    MTT_SWIN_ATTN(8)
    MTT_SWIN_ATTN(16)
    MTT_SWIN_ATTN(32)
    MTT_SWIN_ATTN(64)
    default:
      return set_error(MTT_ERR_BAD_SHAPE, "mtt_swin_window_attention: head_dim=%d (8, 16, 32 or 64)", head_dim);
  }
#undef MTT_SWIN_ATTN
  return check_launch("mtt_swin_window_attention");
}

int mtt_swin_window_scatter(const float* o, int64_t ldo, const float* raw, int32_t B, int32_t H, int32_t W, int32_t C,
                            int32_t T, int32_t ws, int32_t shift, int32_t heads, int32_t update_prompts, float* xa,
                            int64_t ldxa, float* x, int64_t ldx, float* prompts, int64_t ldp, float* logits,
                            mtt_stream_t stream) {
  WinGeom g;
  int rc = make_geom(g, B, H, W, C, T, ws, shift);
  if (rc) return rc;
  if (!o || !xa || !x || (T > 0 && (!raw || !logits)) || (update_prompts && !prompts))
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_swin_window_scatter: bad arguments");
  const long long rows = (long long)B * g.nW * g.wl;
  swin_scatter_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, STREAM>>>(o, ldo, g, xa, ldxa, x, ldx);
  if ((rc = check_launch("mtt_swin_window_scatter(map)"))) return rc;
  if (update_prompts && T > 0) {
    swin_prompt_mean_kernel<<<dim3(B * T, (C + 63) / 64), 256, 0, STREAM>>>(o, ldo, g, prompts, ldp);
    if ((rc = check_launch("mtt_swin_window_scatter(prompts)"))) return rc;
  }
  if (T > 0) {
    const long long n = (long long)B * g.nW * heads * T * g.wl;
    const int blocks = (int)((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096);
    swin_logits_kernel<<<blocks, 256, 0, STREAM>>>(raw, g, heads, logits);
    if ((rc = check_launch("mtt_swin_window_scatter(logits)"))) return rc;
  }
  return MTT_OK;
}

int mtt_transpose_split(const float* in, int64_t ld_in, int32_t B, int32_t L, int32_t C, void* out_hi, void* out_lo,
                        int64_t ld_out, mtt_stream_t stream) {
  if (!in || !out_hi || B <= 0 || L <= 0 || C <= 0 || ld_out < L)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_transpose_split: bad arguments");
  if (ld_out % 2 || (reinterpret_cast<uintptr_t>(out_hi) & 3) || (reinterpret_cast<uintptr_t>(out_lo) & 3))
    return set_error(MTT_ERR_MISALIGNED, "mtt_transpose_split: output planes must be 4-byte aligned with an even ld");
  dim3 grid((L + 63) / 64, (C + 31) / 32, B);
  transpose_split_kernel<<<grid, 256, 0, STREAM>>>(in, ld_in, L, C, static_cast<__nv_bfloat16*>(out_hi),
                                                  static_cast<__nv_bfloat16*>(out_lo), ld_out);
  return check_launch("mtt_transpose_split");
}

int mtt_swin_chan_attention(const float* q, int64_t ldq, const float* kv, int64_t ldkv, int32_t B, int32_t T, int32_t C,
                            int32_t ce, int32_t nh, int32_t nw, float* chan_out, int64_t ldco, void* cs_hi, void* cs_lo,
                            int64_t ldcs, float* raw_chan, mtt_stream_t stream) {
  const int r = (int)(sqrt((double)ce) + 0.5);
  if (!q || !kv || !chan_out || !cs_hi || !raw_chan || B <= 0 || T <= 0 || C <= 0 || r * r != ce || nh <= 0 || nw <= 0 ||
      r % nh || r % nw)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_swin_chan_attention: bad arguments (ce=%d nh=%d nw=%d)", ce, nh, nw);
  const size_t smem = ((size_t)(r / nh) * (r / nw) + C) * sizeof(float);
  if (smem > 48 * 1024) return set_error(MTT_ERR_BAD_SHAPE, "mtt_swin_chan_attention: C=%d too large", C);
  const int we = (r / nh) * (r / nw);
  swin_chan_attn_kernel<<<dim3(B * nh * nw * T, (we + 31) / 32), 256, smem, STREAM>>>(
      q, ldq, kv, ldkv, T, C, ce, nh, nw, 1.0f / sqrtf((float)ce), chan_out, ldco, static_cast<__nv_bfloat16*>(cs_hi),
      static_cast<__nv_bfloat16*>(cs_lo), ldcs, raw_chan);
  return check_launch("mtt_swin_chan_attention");
}

int mtt_swin_merge_gather(const float* x, int64_t ldx, int32_t B, int32_t H, int32_t W, int32_t C, float* out, int64_t ldo,
                          mtt_stream_t stream) {
  if (!x || !out || B <= 0 || H <= 0 || W <= 0 || (H & 1) || (W & 1) || C <= 0 || ldo < 4 * C)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_swin_merge_gather: bad arguments (H=%d W=%d must be even)", H, W);
  const long long rows = (long long)B * (H / 2) * (W / 2) * 4;
  swin_merge_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, STREAM>>>(x, ldx, B, H, W, C, out, ldo);
  return check_launch("mtt_swin_merge_gather");
}

int mtt_conv3x3_s2_maps(const float* in, const float* w, const float* bias, int32_t B, int32_t Cin, int32_t Cout, int32_t H,
                        int32_t W, int64_t in_stride, int32_t in_offset, int64_t out_stride, int32_t out_offset, float* out,
                        mtt_stream_t stream) {
  if (!in || !w || !out || B <= 0 || Cin <= 0 || Cout <= 0 || H <= 0 || W <= 0 || (H & 1) || (W & 1))
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_conv3x3_s2_maps: bad arguments");
  const long long n = (long long)B * Cout * (H / 2) * (W / 2);
  const int blocks = (int)((n + 255) / 256 < 8192 ? (n + 255) / 256 : 8192);
  conv3x3_s2_kernel<<<blocks, 256, 0, STREAM>>>(in, w, bias, B, Cin, Cout, H, W, in_stride, in_offset, out_stride,
                                                out_offset, out);
  return check_launch("mtt_conv3x3_s2_maps");
}

int mtt_swin_chan_up(const float* raw_chan, const float* w, int32_t BT, int32_t C, int32_t Cout, int32_t nwin, float* out,
                     mtt_stream_t stream) {
  if (!raw_chan || !w || !out || BT <= 0 || C <= 0 || Cout <= 0 || nwin <= 0)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_swin_chan_up: bad arguments");
  const long long n = (long long)BT * Cout * nwin;
  chan_up_kernel<<<(unsigned)((n + 255) / 256), 256, 0, STREAM>>>(raw_chan, w, BT, C, Cout, nwin, out);
  return check_launch("mtt_swin_chan_up");
}

int mtt_swin_logit_maps(const float* src, float* dst, int32_t rows, int32_t T, int32_t L, int32_t to_maps,
                        mtt_stream_t stream) {
  if (!src || !dst || rows <= 0 || rows > 65535 || T < 0 || L <= 0)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_swin_logit_maps: bad arguments (rows=%d T=%d L=%d)", rows, T, L);
  const int bx = (L + 255) / 256 < 64 ? (L + 255) / 256 : 64;
  swin_logit_maps_kernel<<<dim3(bx, rows), 256, 0, STREAM>>>(src, dst, T, L, to_maps ? 1 : 0);
  return check_launch("mtt_swin_logit_maps");
}

}  // extern "C"
