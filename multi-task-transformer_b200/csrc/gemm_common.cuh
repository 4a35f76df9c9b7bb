// Shared by the wgmma GEMM / implicit-conv kernels (gemm_tc.cu) and their host side (gemm_host.cu):
// tile constants, the kernel parameter block, the A-tile TMA issue and the fused epilogue.
#pragma once
#include "host_common.h"
#include "ptx.cuh"

namespace mtt {

constexpr int BM = 128;  // rows of A (output pixels / tokens) per CTA
constexpr int BK = 64;   // K per pipeline stage: one 128-byte swizzle row of bf16
constexpr int kEpiWarps = 8;                        // two consumer warpgroups (MMA + epilogue), 64 rows each
constexpr int kGemmThreads = 128 + kEpiWarps * 32;  // warpgroup 0: TMA producer (one warp issues)
constexpr uint32_t kTileBytes = BM * BK * 2;  // 128 x 64 bf16 = 16 KB

struct GemmParams {
  int M, N;
  int num_kb, taps, ksize, dil, mode;
  int NB, H, W, TW, TH, tiles_x, tiles_y;
  int tiles_m;  // number of 128-row sub-tiles
  int tiles_n;  // number of N tiles (of the kernel's BN)
  int cin_pad;
  int k_last_steps;  // 16-wide MMA k-steps holding data in the last k-block of a tap (1..4); the rest is zero padding
  uint32_t a_box_bytes;
  const float* bias;
  int act;
  const float* residual;
  long long ldr;
  int res_row_mod;
  float* out_f32;
  long long ldo_f32;
  __nv_bfloat16* out_hi;
  __nv_bfloat16* out_lo;
  long long ldo_bf;
  int in_group, out_group, out_offset;
  int out_row_stride;  // >= 1: stride of the in-group row index (see mtt_gemm_desc)
  int vec_ok;  // every epilogue pointer is 16-byte aligned, ldr and ldo_f32 % 4 == 0, ldo_bf % 8 == 0
  int a_groups_per_tile;  // >0: A rows are gathered in groups through a rank-3 tensor map
  int debug;              // profiling aid (env MTT_GEMM_DEBUG): bit0 = skip TMA loads, bit1 = skip the epilogue,
                          // bit2 = run the epilogue without its global stores
  // stream-K tail of the 128 x 256 kernel: the first sk_tiles tiles are split along K over ALL CTAs
  int sk_tiles;           // 0: every tile is computed by one CTA
  float* sk_part;         // [CTA][128 rows][256 columns] fp32 partial accumulators
  unsigned int* sk_flags; // [CTA][consumer warp]: 1 = that warp's slice of the partial is published
};

// Stream-K workspace for `units` CTAs: flags first (zero before the first launch and left zero by every launch), then
// one 128 x 256 fp32 partial tile per CTA.
constexpr size_t kSkFlagBytes = 16384;  // up to 512 CTAs x 8 warps x 4 bytes
constexpr size_t sk_workspace_bytes(int units) { return kSkFlagBytes + (size_t)units * BM * 256 * 4; }

// Grouped launch (mtt_gemm_grouped): up to kMaxGroup problems of IDENTICAL geometry (M, N, K, mode, conv shape, nsplit,
// activation, row regrouping) that differ only in their operand / bias / residual / output pointers run as ONE
// persistent launch; tile index = problem * tiles_per_problem + tile. The per-task decoder chains of TaskPrompter
// (5 tasks x {spatial, channel} 1x1 convs, fea_fuse) are single-wave launches (96 tiles on 132 SMs) on their own.
constexpr int kMaxGroup = 32;
struct GroupProblem {
  const float* bias;
  const float* residual;
  float* out_f32;
  __nv_bfloat16* out_hi;
  __nv_bfloat16* out_lo;
};
struct GemmGroup {
  int count;              // 0: not grouped (the kernel uses its four direct tensor-map parameters)
  int tiles_per_problem;
  GroupProblem prob[kMaxGroup];
};
struct GemmGroupMaps {
  CUtensorMap m[kMaxGroup][4];  // A hi, A lo, B hi, B lo per problem
};

// Host: validates the descriptor, fills GemmParams (tiles_n left to the caller) and encodes the four
// tensor maps; the B map's box has `b_box_rows` rows of N.
int gemm_prepare(const mtt_gemm_desc* d, int b_box_rows, GemmParams& p, CUtensorMap maps[4]);

// ---- A tile (128 rows x 64 K) of sub-tile `ms`, k-block kb, filter tap (dy, dx) -----------------
template <int NSPLIT>
__device__ __forceinline__ void load_a_tile(const GemmParams& p, const CUtensorMap* tmA_hi,
                                            const CUtensorMap* tmA_lo, uint8_t* sa, uint64_t* bar, int ms,
                                            int kb, int dy, int dx) {
  auto ld2 = [&](void* dst, const CUtensorMap* m, int c0, int c1) { tma_load_2d(dst, m, bar, c0, c1); };
  auto ld3 = [&](void* dst, const CUtensorMap* m, int c0, int c1, int c2) { tma_load_3d(dst, m, bar, c0, c1, c2); };
  auto ld4 = [&](void* dst, const CUtensorMap* m, int c0, int c1, int c2, int c3) {
    tma_load_4d(dst, m, bar, c0, c1, c2, c3);
  };
  if (p.mode == 0 && p.a_groups_per_tile > 0) {
    ld3(sa, tmA_hi, kb * BK, 0, ms * p.a_groups_per_tile);
    if (NSPLIT == 2) ld3(sa + kTileBytes, tmA_lo, kb * BK, 0, ms * p.a_groups_per_tile);
  } else if (p.mode == 0) {
    ld2(sa, tmA_hi, kb * BK, ms * BM);
    if (NSPLIT == 2) ld2(sa + kTileBytes, tmA_lo, kb * BK, ms * BM);
  } else {
    const int per_img = p.tiles_x * p.tiles_y;
    const int cb = ms / per_img;
    const int r = ms - cb * per_img;
    const int cy = (r / p.tiles_x) * p.TH + dy;
    const int cx = (r % p.tiles_x) * p.TW + dx;
    ld4(sa, tmA_hi, kb * BK, cx, cy, cb);
    if (NSPLIT == 2) ld4(sa + kTileBytes, tmA_lo, kb * BK, cx, cy, cb);
  }
}

// ---- where does row `row` of sub-tile `ms` go? --------------------------------------------------
struct RowInfo {
  long long mo;  // output row (after regrouping)
  long long mr;  // residual row
  bool ok;
};
__device__ __forceinline__ RowInfo row_info(const GemmParams& p, int ms, int row) {
  RowInfo r;
  long long m;
  if (p.mode == 0) {
    m = (long long)ms * BM + row;
    r.ok = m < p.M;
    if (p.a_groups_per_tile > 0) r.ok = r.ok && ms < p.tiles_m;
  } else {
    const int per_img = p.tiles_x * p.tiles_y;
    const int cb = ms / per_img;
    const int t = ms - cb * per_img;
    const int y = (t / p.tiles_x) * p.TH + row / p.TW;
    const int x = (t % p.tiles_x) * p.TW + row % p.TW;
    r.ok = (cb < p.NB) && (row < p.TW * p.TH) && (y < p.H) && (x < p.W);
    m = ((long long)cb * p.H + y) * p.W + x;
  }
  r.mo = m;
  if (p.in_group > 0) r.mo = (m / p.in_group) * p.out_group + p.out_offset + (m % p.in_group) * p.out_row_stride;
  r.mr = (p.res_row_mod > 0) ? (m % p.res_row_mod) : r.mo;
  return r;
}

// ---- fused epilogue: bias, activation, residual, fp32 and split-bf16 stores of four adjacent columns n .. n + 3 of one
// row. The variant is fixed at compile time: ACT (mtt_act) and OUT (which outputs the descriptor has); bias and
// residual stay warp-uniform runtime flags. The kernel reads the bias (epilogue_bias4) once per chunk and the residual
// from shared memory before it calls epilogue_store4, which only computes and stores. `full`: all four columns lie
// inside N and the vector accesses are aligned (vec_ok: 16-byte fp32 and 8-byte bf16 groups, since n % 4 == 0);
// otherwise the columns inside N are written one by one.
enum { kOutF32 = 1, kOutSplit = 2, kOutBoth = 3 };

__device__ __forceinline__ float4 epilogue_bias4(const GemmParams& p, int n, bool full) {  // zero where absent or >= N
  float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
  if (!p.bias) return b;
  if (full) return __ldg(reinterpret_cast<const float4*>(p.bias + n));
  if (n < p.N) b.x = __ldg(p.bias + n);
  if (n + 1 < p.N) b.y = __ldg(p.bias + n + 1);
  if (n + 2 < p.N) b.z = __ldg(p.bias + n + 2);
  if (n + 3 < p.N) b.w = __ldg(p.bias + n + 3);
  return b;
}
// one element: bias add, activation, residual add, in that order (the adds only where the descriptor has the operand)
template <int ACT>
__device__ __forceinline__ float epilogue_op(float v, float b, float r, bool bias, bool res) {
  if (bias) v += b;
  if (ACT == MTT_ACT_GELU) v = gelu_erf(v);
  if (ACT == MTT_ACT_RELU) v = fmaxf(v, 0.f);
  if (res) v += r;
  return v;
}
// v: the four accumulator values, b / r: their bias and residual; of / ob: element offsets of column n of the output
// row in out_f32 / out_hi and out_lo
template <int ACT, int OUT>
__device__ __forceinline__ void epilogue_store4(const GemmParams& p, float4 v, float4 b, float4 r, long long of,
                                                long long ob, int n, bool full) {
  const bool bias = p.bias != nullptr, res = p.residual != nullptr;
  v.x = epilogue_op<ACT>(v.x, b.x, r.x, bias, res);
  v.y = epilogue_op<ACT>(v.y, b.y, r.y, bias, res);
  v.z = epilogue_op<ACT>(v.z, b.z, r.z, bias, res);
  v.w = epilogue_op<ACT>(v.w, b.w, r.w, bias, res);
  if (p.debug & 4) {  // profiling aid: the arithmetic runs, the global stores do not
    asm volatile("" ::"f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w));
    return;
  }
  if (full) {
    if (OUT & kOutF32) *reinterpret_cast<float4*>(p.out_f32 + of) = v;
    if (OUT & kOutSplit) {
      uint2 h, l;
      split_pack2(v.x, v.y, h.x, l.x);
      split_pack2(v.z, v.w, h.y, l.y);
      *reinterpret_cast<uint2*>(p.out_hi + ob) = h;
      if (p.out_lo) *reinterpret_cast<uint2*>(p.out_lo + ob) = l;
    }
    return;
  }
  const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (n + k >= p.N) break;
    if (OUT & kOutF32) p.out_f32[of + k] = e[k];
    if (OUT & kOutSplit) {
      __nv_bfloat16 h, l;
      split_bf16(e[k], h, l);
      p.out_hi[ob + k] = h;
      if (p.out_lo) p.out_lo[ob + k] = l;
    }
  }
}

// Entry points of the kernels (defined in gemm_tc.cu); bn = 128 or 256 columns per tile
int launch_gemm_tiles(const mtt_gemm_desc* d, int bn, cudaStream_t stream);
int launch_gemm_tiles_grouped(const mtt_gemm_desc* d, int count, int bn, cudaStream_t stream);
void set_gemm_streamk(int mode);
int streamk_tiles(int tiles, int k_iters, int pairs);
int streamk_schedule_host(int tiles, int k_iters, int pairs, int pair, int* out, int max_pieces);

}  // namespace mtt
