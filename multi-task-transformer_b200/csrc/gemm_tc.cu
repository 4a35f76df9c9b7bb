// Persistent, warp-specialised wgmma GEMM / implicit-GEMM convolution for sm_90a.
//
//   D[m, n] = act( sum_k A[m, k] * Bw[n, k] + bias[n] ) + residual[m, n]
//
// Operands are split-bf16 planes (hi, lo).  With NSPLIT = 2 every 64xBNx16 product is issued as
// three wgmma (hi*hi + hi*lo + lo*hi) accumulating in fp32 registers, which carries ~16 mantissa
// bits per operand -- the reference computes these contractions in fp32 (cuBLAS / cuDNN eager,
// TP/models/transformers/taskprompter.py:201,212,274,362,691) and single-pass bf16/tf32 does not
// meet its 1e-3 parity bar (SURVEY.md H1).  NSPLIT = 1 is plain bf16.
//
// Tiles are 128 x BN (BN = 128, or 256 for wide problems).  Roles (384 threads): warpgroup 0 = TMA producer (one
// warp issues, the warpgroup hands its registers to the consumers), warpgroups 1 and 2 = consumers, each owning 64
// rows of the tile: they wait for a stage, issue the wgmma chain on it, release the stage and, after the last k-block
// of a tile, run the fused epilogue through a per-warp shared-memory buffer.  One barrier ring (smem full / empty)
// and a static persistent tile schedule; the producer runs ahead into the next tile while the epilogue drains.
//
// Convolution (mode 1) is the same kernel: the A tile of 128 output pixels is a TH x TW patch of one
// NHWC image and each filter tap is a shifted rank-4 TMA box; TMA's out-of-bounds zero fill is the
// zero padding.  The K loop runs over taps x channel blocks.
#include <stdlib.h>

#include <type_traits>

#include "gemm_common.cuh"

namespace mtt {

constexpr int kEpiCols = 32;  // columns per staged epilogue chunk: 8 lanes per row, four rows per pass

template <int NSPLIT, int BN>
struct GemmCfg {
  static constexpr int kNsplit = NSPLIT, kBN = BN;
  static constexpr uint32_t kBTileBytes = BN * BK * 2;
  static constexpr uint32_t kStageBytes = NSPLIT * (kTileBytes + kBTileBytes);
  static constexpr int kStages = (200 * 1024) / kStageBytes;  // 3 / 6 stages (BN 128), 2 / 4 (BN 256)
  // stages | 256 B of mbarriers | per consumer warp, a 16 x kEpiCols fp32 accumulator chunk and the residual of that
  // chunk | per consumer warp, the residual-row table (+ 1 KB for alignment)
  static constexpr uint32_t kEpiBufBytes = kEpiWarps * 2 * 16 * kEpiCols * 4;
  static constexpr uint32_t kRowMapBytes = kEpiWarps * 16 * 8;  // per consumer warp, the residual rows of its 16 rows
  static constexpr uint32_t kSmemBytes = kStages * kStageBytes + 256 + kEpiBufBytes + kRowMapBytes + 1024;
  static_assert(kSmemBytes <= 227 * 1024, "exceeds the per-block shared memory of sm_90");
  // A planes whose fragments the consumers hold in registers for a stage (8 registers per k16 step and plane) and feed
  // to RS-form wgmma. Beside the 128 x 256 tile's acc[128] + part[64] only A_hi fits without spilling; its A_lo
  // (one wgmma per k16 step and half) stays in the shared-memory (SS) form.
  static constexpr int kRegPlanes = BN == 128 ? NSPLIT : 1;
};

// ---- stream-K tail (SK = true, single-problem kernel with 256-wide tiles) ------------------------------------------------
// With T tiles on P CTAs the plain persistent schedule runs ceil(T / P) rounds. Here the R = T mod P tiles that would
// form the ragged last round (tile indices [0, R)) are split along K instead: their R * k_iters k-blocks are dealt out
// evenly, CTA p taking the contiguous range [p W / P, (p + 1) W / P) of W = R * k_iters, which touches at most two tiles.
// The remaining T - R tiles run one CTA per tile as before (tile R + p + j P). Every CTA does its stream-K range FIRST.
//   * a range piece that starts inside a tile (k0 > 0) is a CONTRIBUTION: the consumer warps dump the raw fp32
//     accumulator to this CTA's slot of p.sk_part and publish it per warp (release store to p.sk_flags);
//   * the piece that holds a tile's first k-block OWNS the tile: its consumer warps wait for the warps of the following
//     CTAs whose ranges end the tile (a contribution is always a CTA's first piece, so it never waits on anything),
//     add their partials in CTA order (a fixed order: results are reproducible run to run) and run the fused epilogue.
//     The owner resets each flag it consumed, so the flag array is all-zero again when the launch retires.
// All CTAs are co-resident (grid <= number of SMs, one CTA per SM), so the owner's spin cannot starve a contributor.
// (The schedule code names its units "pairs" for the host test hook; on this kernel a unit is one CTA.)
struct SkSched {
  int n_sk;                  // 0..2 stream-K pieces of this unit
  int tile0, k0_0, k1_0;     // first piece (may start inside its tile)
  int k1_1;                  // second piece: tile0 + 1, k-blocks [0, k1_1)
  int dp_first, dp_step;     // whole tiles: dp_first + j * dp_step < num_tiles
  int n_seg;
  long long W;               // total stream-K k-blocks
};
template <bool SK>
__host__ __device__ __forceinline__ SkSched sk_schedule(const GemmParams& p, int pair, int num_pairs, int num_tiles, int k_iters) {
  SkSched s;
  s.n_sk = 0;
  s.tile0 = s.k0_0 = s.k1_0 = s.k1_1 = 0;
  s.W = 0;
  s.dp_first = pair;
  s.dp_step = num_pairs;
  if (SK && p.sk_tiles > 0) {
    s.W = (long long)p.sk_tiles * k_iters;
    const long long b = (long long)pair * s.W / num_pairs, e = (long long)(pair + 1) * s.W / num_pairs;
    if (e > b) {
      const int t0 = (int)(b / k_iters);
      const long long t0_end = (long long)(t0 + 1) * k_iters;
      s.tile0 = t0;
      s.k0_0 = (int)(b - (long long)t0 * k_iters);
      s.k1_0 = (int)((e < t0_end ? e : t0_end) - (long long)t0 * k_iters);
      s.n_sk = 1;
      if (e > t0_end) {
        s.k1_1 = (int)(e - t0_end);
        s.n_sk = 2;
      }
    }
    s.dp_first = p.sk_tiles + pair;
  }
  const int left = num_tiles - s.dp_first;
  s.n_seg = s.n_sk + (left > 0 ? (left + s.dp_step - 1) / s.dp_step : 0);
  return s;
}
// piece `si` of a unit's schedule: tile index and k-block range [k0, k1)
__host__ __device__ __forceinline__ void sk_piece(const SkSched& s, int si, int k_iters, int& tile, int& k0, int& k1) {
  if (si < s.n_sk) {
    tile = s.tile0 + si;
    k0 = si == 0 ? s.k0_0 : 0;
    k1 = si == 0 ? s.k1_0 : s.k1_1;
  } else {
    tile = s.dp_first + (si - s.n_sk) * s.dp_step;
    k0 = 0;
    k1 = k_iters;
  }
}
__device__ __forceinline__ void sk_flag_publish(unsigned int* f) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(f), "r"(1u) : "memory");
}
__device__ __forceinline__ unsigned int sk_flag_peek(const unsigned int* f) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(f) : "memory");
  return v;
}

// ---- stages of the kernel body -------------------------------------------------------------------------------------
// gemm_tc_body (below) is the driver; each stage is a function of its own. Warp 0 runs produce(); each consumer warp
// runs, per piece of its schedule: res_prefetch (the residual of the epilogue's first chunk), mma_piece (the piece's
// k-blocks into acc), then sk_contribute (a stream-K contribution ends there) or sk_collect (a stream-K owner adds the
// other CTAs' partials) and epilogue_piece.

constexpr uint32_t kTurnBar = 1;  // named barriers 1, 2: the consumer warpgroups' turns

// tile -> (problem, m-tile, n-tile); tpp = tiles per problem
struct PieceCoords {
  int g, mt, nt;
};
template <bool GROUPED>
__device__ __forceinline__ PieceCoords piece_coords(const GemmParams& p, int tpp, int tile) {
  const int g = GROUPED ? tile / tpp : 0;
  const int tl = GROUPED ? tile - g * tpp : tile;
  return PieceCoords{g, tl % p.tiles_m, tl / p.tiles_m};
}

// The TMA producer loop (warp 0, one elected lane issues): every k-block of every piece into the stage ring.
template <int NSPLIT, int BN, bool GROUPED>
__device__ __forceinline__ void produce(const CUtensorMap (*maps)[4], const GemmParams& p, const SkSched& sched,
                                        int tpp, int k_iters, uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar) {
  using Cfg = GemmCfg<NSPLIT, BN>;
  int stage = 0;
  uint32_t phase = 0;
  const uint32_t stage_tx = NSPLIT * (p.a_box_bytes + Cfg::kBTileBytes);
  for (int si = 0; si < sched.n_seg; ++si) {
    int tile, kbeg, kend;
    sk_piece(sched, si, k_iters, tile, kbeg, kend);
    const PieceCoords pc = piece_coords<GROUPED>(p, tpp, tile);
    const CUtensorMap* tmA_hi = &maps[pc.g][0];
    const CUtensorMap* tmA_lo = &maps[pc.g][1];
    const CUtensorMap* tmB_hi = &maps[pc.g][2];
    const CUtensorMap* tmB_lo = &maps[pc.g][3];
    for (int ki = kbeg; ki < kend; ++ki) {
      const int tap = ki / p.num_kb, kb = ki - tap * p.num_kb;
      const int dy = (tap / p.ksize - p.ksize / 2) * p.dil;
      const int dx = (tap % p.ksize - p.ksize / 2) * p.dil;
      mbar_wait(&empty_bar[stage], phase ^ 1);
      uint8_t* sa = smem + stage * Cfg::kStageBytes;
      uint8_t* sb = sa + NSPLIT * kTileBytes;
      if (elect_one()) {
        if (p.debug & 1) {  // profiling aid: no loads
          mbar_arrive(&full_bar[stage]);
        } else {
          mbar_arrive_expect_tx(&full_bar[stage], stage_tx);
          load_a_tile<NSPLIT>(p, tmA_hi, tmA_lo, sa, &full_bar[stage], pc.mt, kb, dy, dx);
          const int kcoord = tap * p.cin_pad + kb * BK;
          tma_load_2d(sb, tmB_hi, &full_bar[stage], kcoord, pc.nt * BN);
          if (NSPLIT == 2) tma_load_2d(sb + Cfg::kBTileBytes, tmB_lo, &full_bar[stage], kcoord, pc.nt * BN);
        }
      }
      __syncwarp();
      if (++stage == Cfg::kStages) {
        stage = 0;
        phase ^= 1;
      }
    }
  }
}

// What a consumer thread computes once from its warp and lane.
struct ConsumerWarp {
  int lane;
  int cw;          // consumer warpgroup: rows [64 cw, 64 cw + 64) of the tile
  int ew;          // consumer warp 0..7 (stream-K flag slot)
  int row0, col0;  // this thread's rows: row0 and row0 + 8, and columns col0 + 8 i + {0, 1}
  int wrow0;       // the warp's first row in the tile
  uint32_t a_off;  // byte offset of the warpgroup's 64 A rows in a stage's A plane
  uint32_t a_frag_off;
  int a_chunk, a_xor;
  uint32_t ebuf, rbuf, rmap;
};
template <typename Cfg>
__device__ __forceinline__ ConsumerWarp consumer_warp(uint8_t* smem, int warp, int lane) {
  ConsumerWarp c;
  c.lane = lane;
  c.cw = (warp - 4) >> 2;
  c.ew = warp - 4;
  c.row0 = c.cw * 64 + (warp & 3) * 16 + (lane >> 2);
  c.col0 = 2 * (lane & 3);
  c.a_off = (uint32_t)c.cw * 64 * 128;
  // ldmatrix source of this lane in the warpgroup's 64 A rows: row (lane % 8) + 8 ((lane / 8) % 2) of the warp's 16,
  // 16-byte chunk 2 ks + lane / 16 of the 128-byte row, stored at chunk ^ (row % 8) by the 128-byte swizzle
  const int lrow = (warp & 3) * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
  c.a_frag_off = c.a_off + (uint32_t)lrow * 128;
  c.a_chunk = lane >> 4;
  c.a_xor = lane & 7;
  c.wrow0 = c.cw * 64 + (warp & 3) * 16;
  // the warp's epilogue buffers, as shared addresses: ebuf, a 16 x kEpiCols fp32 chunk of the accumulator
  c.ebuf = smem_u32(smem + Cfg::kStages * Cfg::kStageBytes + 256) + c.ew * (2 * 16 * kEpiCols * 4);
  c.rbuf = c.ebuf + 16 * kEpiCols * 4;  // the residual of the chunk in ebuf
  // the residual row of each of the warp's 16 rows (8 bytes each, -1: the row is not written), set when a piece
  // starts; kept in shared memory, since the registers beside the 128 x 256 tile's accumulator are few
  c.rmap = smem_u32(smem + Cfg::kStages * Cfg::kStageBytes + 256 + Cfg::kEpiBufBytes) + c.ew * 16 * 8;
  return c;
}

// Copies the residual of rows [8 half, 8 half + 8) of the warp's 16, columns [n0, n0 + kEpiCols), to rbuf as one
// cp.async group. Lane l copies columns 4 (l % 8) .. 4 (l % 8) + 3 of rows 8 half + l / 8 and 8 half + l / 8 + 4;
// what lies outside the problem is zero-filled.
__device__ __forceinline__ void res_issue(const GemmParams& p, const ConsumerWarp& c, const float* res, int n0,
                                          int half) {
  const int n = n0 + 4 * (c.lane & 7);
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int r = 8 * half + (c.lane >> 3) + 4 * k;
    const long long m = ld_shared_s64(c.rmap + 8 * r);
    const uint32_t dst = c.rbuf + (r * kEpiCols + 4 * (c.lane & 7)) * 4;
    const float* src = res + (m >= 0 ? m * p.ldr + n : 0);
    if (p.vec_ok) {  // residual and ldr 16-byte aligned, n % 4 == 0
      const int cols = m >= 0 ? min(max(p.N - n, 0), 4) : 0;
      cp_async_cg16(dst, cols ? src : res, 4 * cols);
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const bool in = m >= 0 && n + e < p.N;
        cp_async_ca4(dst + 4 * e, in ? src + e : res, in ? 4 : 0);
      }
    }
  }
  cp_async_commit();
}

// The residual of the epilogue's first chunk: the copy has the whole mainloop to land, and is issued while acc holds
// nothing (rbuf is free: the previous piece's epilogue has read it). Also sets the warp's residual-row table.
template <int BN>
__device__ __forceinline__ void res_prefetch(const GemmParams& p, const ConsumerWarp& c, const float* res, int mt,
                                             int nt) {
  if (c.lane < 16) {
    const RowInfo ri = row_info(p, mt, c.wrow0 + c.lane);
    st_shared_s64(c.rmap + 8 * c.lane, ri.ok ? ri.mr : -1);
  }
  __syncwarp();
  res_issue(p, c, res, nt * BN, 0);
  res_issue(p, c, res, nt * BN, 1);
}

// Ordered consumer warpgroups: the two warpgroups take turns issuing their wgmma chains (one chain = one stage x
// one 128-column half), so that while one waits for its chain and folds it into acc, the other's chain keeps the
// tensor pipe busy. Named barrier kTurnBar + w opens warpgroup w's turn; each side arrives at the other's barrier
// after issuing. Warpgroup 1 opens the first turn, warpgroup 0 consumes the last opening after its loop.
__device__ __forceinline__ void wait_turn(int cw) {  // barrier ids are immediates; cw is uniform per warpgroup
  if (cw == 0) bar_sync<kTurnBar, 256>(); else bar_sync<kTurnBar + 1, 256>();
}
__device__ __forceinline__ void pass_turn(int cw) {
  if (cw == 0) bar_arrive<kTurnBar + 1, 256>(); else bar_arrive<kTurnBar, 256>();
}

// The k-blocks [kbeg, kend) of one piece, summed into acc (zeroed first). part and afr belong to the caller, so their
// registers stay the same across pieces.
template <int NSPLIT, int BN>
__device__ __forceinline__ void mma_piece(const GemmParams& p, const ConsumerWarp& c, uint8_t* smem, uint64_t* full_bar,
                                          uint64_t* empty_bar, int kbeg, int kend, int& stage, uint32_t& phase,
                                          float (&acc)[BN / 2], float (&part)[64],
                                          uint32_t (&afr)[BK / 16][GemmCfg<NSPLIT, BN>::kRegPlanes][4]) {
  using Cfg = GemmCfg<NSPLIT, BN>;
  constexpr int kRegPlanes = Cfg::kRegPlanes;
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  int kb = kbeg % p.num_kb;
  for (int ki = kbeg; ki < kend; ++ki) {
    const int nks = (++kb == p.num_kb) ? p.k_last_steps : BK / 16;  // zero-padded tail of K: no MMAs
    if (kb == p.num_kb) kb = 0;
    mbar_wait(&full_bar[stage], phase);
    const uint32_t sa = smem_u32(smem + stage * Cfg::kStageBytes);
    const uint32_t a_lo = sa + kTileBytes + c.a_off;
    const uint32_t b_hi = sa + NSPLIT * kTileBytes, b_lo = b_hi + Cfg::kBTileBytes;
    {  // each A fragment in registers is read from shared memory once per stage, not once per wgmma using it
      const uint32_t fa = sa + c.a_frag_off;
#pragma unroll
      for (int ks = 0; ks < BK / 16; ++ks) {
        const uint32_t sw = (uint32_t)(((2 * ks + c.a_chunk) ^ c.a_xor) << 4);
#pragma unroll
        for (int s = 0; s < kRegPlanes; ++s) ldmatrix_x4(afr[ks][s], fa + s * kTileBytes + sw);
      }
    }
    // The tensor core adds products into its accumulator with truncation, so a long chain of wgmma on one
    // accumulator drifts towards zero (a one-sided error that grows with K). Each stage's products are therefore
    // summed in a fresh accumulator and added to the tile's sum with a round-to-nearest FADD.
#pragma unroll
    for (int hn = 0; hn < BN / 128; ++hn) {
      const uint32_t bo = (uint32_t)hn * 128 * 128;  // 128 weight rows of 128 bytes
      wait_turn(c.cw);
      wgmma_fence_regs(part);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < BK / 16; ++ks) {
        if (ks >= nks) break;
        const uint64_t bdh = gmma_desc_sw128(b_hi + bo + ks * 32);
        wgmma_rs_n128<0>(part, afr[ks][0], bdh, ks > 0 ? 1 : 0);
        if (NSPLIT == 2) {
          wgmma_rs_n128<0>(part, afr[ks][0], gmma_desc_sw128(b_lo + bo + ks * 32), 1);
          if (kRegPlanes == 2)
            wgmma_rs_n128<0>(part, afr[ks][1], bdh, 1);
          else
            wgmma_ss_n128<0>(part, gmma_desc_sw128(a_lo + ks * 32), bdh, 1);
        }
      }
      wgmma_commit();
      pass_turn(c.cw);
      wgmma_wait<0>();
      wgmma_fence_regs(part);
#pragma unroll
      for (int ks = 0; ks < BK / 16; ++ks)
#pragma unroll
        for (int s = 0; s < kRegPlanes; ++s) wgmma_fence_regs(afr[ks][s]);
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[hn * 64 + i] += part[i];
    }
    __syncwarp();
    if (c.lane == 0) mbar_arrive(&empty_bar[stage]);  // this warp no longer reads the stage
    if (++stage == Cfg::kStages) {
      stage = 0;
      phase ^= 1;
    }
  }
}

// Stream-K contribution (a piece that starts inside its tile): dump the raw accumulator to this CTA's slot of sk_part
// and publish it for this warp.
template <int BN>
__device__ __forceinline__ void sk_contribute(const GemmParams& p, const ConsumerWarp& c, const float (&acc)[BN / 2]) {
  float* part = p.sk_part + (size_t)blockIdx.x * BM * 256;
#pragma unroll
  for (int i = 0; i < BN / 8; ++i) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
      *reinterpret_cast<float2*>(part + (size_t)(c.row0 + 8 * h) * 256 + 8 * i + c.col0) =
          make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
  }
  __threadfence();
  __syncwarp();
  if (c.lane == 0) sk_flag_publish(p.sk_flags + blockIdx.x * kEpiWarps + c.ew);
}

// Stream-K owner of `tile` (its piece holds the first k-block but not the last): wait for each following CTA whose
// range ends in the tile, add its partial to acc in CTA order, and hand its flag back as zero.
template <int BN>
__device__ __forceinline__ void sk_collect(const GemmParams& p, const ConsumerWarp& c, const SkSched& sched, int tile,
                                           int k_iters, float (&acc)[BN / 2]) {
  const long long tile_kend = (long long)(tile + 1) * k_iters;
  for (int pp = blockIdx.x + 1; pp < (int)gridDim.x && (long long)pp * sched.W / gridDim.x < tile_kend; ++pp) {
    unsigned int* flag = p.sk_flags + pp * kEpiWarps + c.ew;
    if (c.lane == 0) {
      while (sk_flag_peek(flag) == 0) {
      }
    }
    __syncwarp();
    __threadfence();
    const float* part = p.sk_part + (size_t)pp * BM * 256;
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float2 a = __ldcg(reinterpret_cast<const float2*>(part + (size_t)(c.row0 + 8 * h) * 256 + 8 * i + c.col0));
        acc[4 * i + 2 * h] += a.x;
        acc[4 * i + 2 * h + 1] += a.y;
      }
    }
    __syncwarp();
    if (c.lane == 0) *reinterpret_cast<volatile unsigned int*>(flag) = 0u;  // hand the flag back as zero
  }
}

// Grouped launch: problem g's pointers over the shared geometry.
__device__ __forceinline__ GemmParams problem_params(const GemmParams& p, const GemmGroup* grp, int g) {
  GemmParams pg = p;
  const GroupProblem& gp = grp->prob[g];
  pg.bias = gp.bias;
  pg.residual = gp.residual;
  pg.out_f32 = gp.out_f32;
  pg.out_hi = gp.out_hi;
  pg.out_lo = gp.out_lo;
  return pg;
}

// The fused epilogue of one piece, straight from the accumulator fragment. p: the kernel's parameters (geometry);
// pq: the problem's pointers (p itself for a single problem). The warp's 16 x BN slice goes out in 16 x kEpiCols chunks
// through its shared-memory buffer, with no global load on the per-row path:
//   * lane l writes rows 4 q + l / 8 (q = 0..3) of every chunk, columns 4 (l % 8) .. 4 (l % 8) + 3. The element
//     offsets of the warp's 16 output rows in out_f32 and in out_hi / out_lo are computed once per piece from the
//     row map (row_info), lane l holding those of row l % 16; a pass reads its row's with a shuffle and adds its
//     column (four rows of offsets per lane would not fit beside the 128 x 256 tile's accumulator). The residual
//     rows are in rmap;
//   * the bias of the lane's four columns is read once per chunk, while the fragment is written to ebuf;
//   * the chunk's residual is in rbuf (cp.async: the first chunk's was issued when the piece started, each half
//     of a later chunk's while the same half of the chunk before it is stored). res_issue makes lane l copy the
//     residual of the same rows and columns it stores.
// The fragment is written with unrolled 8-byte shared stores (acc needs compile-time indices, hence the branch
// per chunk in the rolled chunk loop), then 4 passes store four rows each, 8 lanes per row, four columns per
// lane: one contiguous 128-byte fp32 segment (64 bytes per bf16 plane) per row. Unrolling the whole epilogue
// over the fragment made it tens of thousands of instructions long and bound by instruction fetch. Columns are
// XOR-swizzled by row in 8-column groups, so both sides of ebuf are free of bank conflicts: a half-warp of the
// fragment stores covers rows 4 k .. 4 k + 3 and 8 columns of each, a quarter-warp of the 16-byte pass reads one
// row.
// The residual may be the output itself (x += f(x)): a chunk's residual is in shared memory before any store of
// that chunk, and the copy of chunk c + 1 overlaps only the stores of chunk c, whose columns are disjoint from it.
template <int BN, int ACT, int OUT>
__device__ __forceinline__ void epilogue_piece(const GemmParams& p, const GemmParams& pq, const ConsumerWarp& cs,
                                               const float (&acc)[BN / 2], int mt, int nt) {
  const int lane = cs.lane;
  const int lr = lane >> 3, c4 = 4 * (lane & 7);  // this lane's rows (4 q + lr) and first column in a chunk
  long long of_map, ob_map;  // row lane % 16 of the warp: element offsets of its column 0 in out_f32 / out_hi, out_lo
  int rows_ok = 0;           // bit q: row 4 q + lr is written
  {
    const RowInfo ri = row_info(p, mt, cs.wrow0 + (lane & 15));
    of_map = ri.mo * pq.ldo_f32;
    ob_map = ri.mo * pq.ldo_bf;
#pragma unroll
    for (int q = 0; q < 4; ++q) rows_ok |= (__shfl_sync(0xffffffffu, (int)ri.ok, 4 * q + lr) & 1) << q;
  }
  // fragment stores: row (lane / 4) + 8 h, columns 8 j + col0 + {0, 1} at 8-column group j ^ (row % 4)
  const uint32_t e_wr = cs.ebuf + ((lane >> 2) * kEpiCols + cs.col0) * 4, e_sw = ((lane >> 2) & 3) * 32;
  // pass reads: row 4 q + lr (row % 4 == lr), columns c4 .. c4 + 3 at their swizzled place
  const uint32_t e_rd = cs.ebuf + (lr * kEpiCols + (c4 ^ (lr << 3))) * 4;
  const uint32_t r_rd = cs.rbuf + (lr * kEpiCols + c4) * 4;
  constexpr int kChunks = BN / kEpiCols;
#pragma unroll 1
  for (int c = 0; c < kChunks; ++c) {
    const int n0 = nt * BN + c * kEpiCols, n = n0 + c4;
    const bool full = pq.vec_ok && n + 4 <= pq.N;
    const float4 b = epilogue_bias4(pq, n, full);
#pragma unroll
    for (int cc = 0; cc < kChunks; ++cc) {
      if (cc != c) continue;
#pragma unroll
      for (int j = 0; j < kEpiCols / 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int i = cc * (kEpiCols / 8) + j;
          st_shared_v2(e_wr + h * 8 * kEpiCols * 4 + ((j * 32) ^ e_sw), acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
        }
    }
    // rows [8 half, 8 half + 8) of the chunk: passes q = 2 half, 2 half + 1
    auto store_rows = [&](int half) {
#pragma unroll 1
      for (int q = 2 * half; q < 2 * half + 2; ++q) {
        const float4 v = ld_shared_v4(e_rd + q * 4 * kEpiCols * 4);
        const float4 rv = pq.residual ? ld_shared_v4(r_rd + q * 4 * kEpiCols * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
        const long long of = (OUT & kOutF32) ? __shfl_sync(0xffffffffu, of_map, 4 * q + lr) + n : 0;
        const long long ob = (OUT & kOutSplit) ? __shfl_sync(0xffffffffu, ob_map, 4 * q + lr) + n : 0;
        if (rows_ok & (1 << q)) epilogue_store4<ACT, OUT>(pq, v, b, rv, of, ob, n, full);
      }
    };
    // The residual arrives in two groups per chunk, rows 0-7 and rows 8-15; each half of rbuf is refilled with the
    // next chunk's rows as soon as this chunk's passes over it are done.
    if (pq.residual) cp_async_wait<1>();
    __syncwarp();
    store_rows(0);
    if (pq.residual) {
      __syncwarp();
      if (c + 1 < kChunks) {
        res_issue(p, cs, pq.residual, n0 + kEpiCols, 0);
        cp_async_wait<1>();
      } else {
        cp_async_wait<0>();
      }
      __syncwarp();
    }
    store_rows(1);
    __syncwarp();  // ebuf and rbuf are free for the next chunk
    if (pq.residual && c + 1 < kChunks) res_issue(p, cs, pq.residual, n0 + kEpiCols, 1);
  }
}

// The kernel body, shared by the single-problem kernel (GROUPED = false: `maps` holds one set of four tensor maps)
// and the grouped one (GROUPED = true: one set per problem, tile -> (problem, tile) through grp). ACT and OUT fix the
// epilogue variant (epilogue_store4).
template <int NSPLIT, int BN, bool GROUPED, bool SK, int ACT, int OUT>
__device__ __forceinline__ void gemm_tc_body(const CUtensorMap (*maps)[4], const GemmParams& p, const GemmGroup* grp) {
  static_assert(!SK || (BN == 256 && !GROUPED), "stream-K: single-problem kernel with 256-wide tiles only");
  using Cfg = GemmCfg<NSPLIT, BN>;
  constexpr int ST = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + ST * Cfg::kStageBytes);
  uint64_t* empty_bar = full_bar + ST;

  const int warp = threadIdx.x >> 5;
  const int tpp = p.tiles_m * p.tiles_n;  // tiles per problem
  const int num_tiles = GROUPED ? tpp * grp->count : tpp;
  const int k_iters = p.taps * p.num_kb;
  const SkSched sched = sk_schedule<SK>(p, blockIdx.x, gridDim.x, num_tiles, k_iters);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&maps[0][0]);
    tma_prefetch_desc(&maps[0][2]);
    if (NSPLIT == 2) {
      tma_prefetch_desc(&maps[0][1]);
      tma_prefetch_desc(&maps[0][3]);
    }
    for (int s = 0; s < ST; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kEpiWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {  // TMA producer: warp 0 issues, the warpgroup hands its registers to the consumers
    setmaxnreg_dec<40>();
    if (warp == 0) produce<NSPLIT, BN, GROUPED>(maps, p, sched, tpp, k_iters, smem, full_bar, empty_bar);
  } else {  // consumers: MMA + epilogue
    setmaxnreg_inc<232>();
    const ConsumerWarp c = consumer_warp<Cfg>(smem, warp, threadIdx.x & 31);
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];  // the tile's fp32 sum, in the m64nBN fragment layout (= the 128-column halves side by side)
    float part[64];     // one stage's products for one 128-column half
    uint32_t afr[BK / 16][Cfg::kRegPlanes][4];  // the stage's A fragments per k16 step (RS-form wgmma)
    if (c.cw == 1) pass_turn(c.cw);
    for (int si = 0; si < sched.n_seg; ++si) {
      int tile, kbeg, kend;
      sk_piece(sched, si, k_iters, tile, kbeg, kend);
      const PieceCoords pc = piece_coords<GROUPED>(p, tpp, tile);
      const float* res = GROUPED ? grp->prob[pc.g].residual : p.residual;
      if (res && !(SK && kbeg > 0) && !(p.debug & 2))  // a stream-K contribution has no epilogue
        res_prefetch<BN>(p, c, res, pc.mt, pc.nt);
      mma_piece<NSPLIT, BN>(p, c, smem, full_bar, empty_bar, kbeg, kend, stage, phase, acc, part, afr);
      const bool sk_contrib = SK && kbeg > 0;
      const bool sk_owner = SK && kbeg == 0 && kend < k_iters;
      if (SK && sk_contrib) {
        sk_contribute<BN>(p, c, acc);
        continue;
      }
      if (SK && sk_owner) sk_collect<BN>(p, c, sched, tile, k_iters, acc);
      if (p.debug & 2) continue;
      if constexpr (GROUPED)
        epilogue_piece<BN, ACT, OUT>(p, problem_params(p, grp, pc.g), c, acc, pc.mt, pc.nt);
      else
        epilogue_piece<BN, ACT, OUT>(p, p, c, acc, pc.mt, pc.nt);  // single problem: read the kernel parameters
    }
    if (c.cw == 0) wait_turn(c.cw);  // warpgroup 1's last opening: both barriers end their last phase
  }
}

struct GemmMaps1 {
  CUtensorMap m[1][4];
};

template <int NSPLIT, int BN, bool SK, int ACT, int OUT>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tc_kernel(const __grid_constant__ GemmMaps1 maps, const GemmParams p) {
  gemm_tc_body<NSPLIT, BN, false, SK, ACT, OUT>(maps.m, p, nullptr);
}

template <int NSPLIT, int BN, int ACT, int OUT>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tc_grouped_kernel(const __grid_constant__ GemmGroupMaps maps, const __grid_constant__ GemmGroup grp,
                       const GemmParams p) {
  gemm_tc_body<NSPLIT, BN, true, false, ACT, OUT>(maps.m, p, &grp);
}

// Launches `kernel` on `grid` CTAs with Cfg's shared memory, after its dynamic shared-memory opt-in, which is per
// device and per kernel instantiation (`done`: that instantiation's flags).
template <typename Cfg, typename Kernel, typename... Args>
static int launch_kernel(Kernel kernel, bool (&done)[kMaxDevices], const char* what, int grid, cudaStream_t stream,
                         const Args&... args) {
  const int dev_ = current_device();
  if (!done[dev_]) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) return set_error(MTT_ERR_LAUNCH, "%s: cudaFuncSetAttribute: %s", what, cudaGetErrorString(e));
    done[dev_] = true;
  }
  kernel<<<grid, kGemmThreads, Cfg::kSmemBytes, stream>>>(args...);
  return check_launch(what);
}

// The epilogue variant of a descriptor, as compile-time constants: its activation (gemm_prepare admits none, GELU and
// ReLU) and which outputs it has (at least one). f(EpiKind<ACT, OUT>{}) launches that variant's kernel.
template <int ACT_, int OUT_>
struct EpiKind {
  static constexpr int ACT = ACT_, OUT = OUT_;
};
template <int ACT, typename F>
static int with_epilogue_out(const GemmParams& p, F&& f) {
  if (!p.out_hi) return f(EpiKind<ACT, kOutF32>{});
  if (!p.out_f32) return f(EpiKind<ACT, kOutSplit>{});
  return f(EpiKind<ACT, kOutBoth>{});
}
template <typename F>
static int with_epilogue(const GemmParams& p, F&& f) {
  switch (p.act) {
    case MTT_ACT_NONE: return with_epilogue_out<MTT_ACT_NONE>(p, f);
    case MTT_ACT_GELU: return with_epilogue_out<MTT_ACT_GELU>(p, f);
    case MTT_ACT_RELU: return with_epilogue_out<MTT_ACT_RELU>(p, f);
  }
  return set_error(MTT_ERR_BAD_SHAPE, "mtt_gemm: no kernel for act=%d", p.act);
}

// The tile shape of a launch, split count (1, 2) and width (128, 256), as compile-time constants:
// f(GemmCfg<NSPLIT, BN>{}) launches that shape's kernel.
template <typename F>
static int with_tile(int nsplit, int bn, F&& f) {
  if (bn == 256) return nsplit == 2 ? f(GemmCfg<2, 256>{}) : f(GemmCfg<1, 256>{});
  return nsplit == 2 ? f(GemmCfg<2, 128>{}) : f(GemmCfg<1, 128>{});
}

// One launch on `grid` CTAs of the kernel for tile shape (nsplit, bn) and p's epilogue: with GemmMaps1 the
// single-problem kernel, split along K when p.sk_tiles > 0 (256-wide tiles only); with GemmGroupMaps the grouped kernel
// over grp's problems.
template <typename Maps>
static int launch_gemm(const Maps& maps, const GemmGroup* grp, const GemmParams& p, int nsplit, int bn, int grid,
                       cudaStream_t stream) {
  constexpr bool kGrouped = std::is_same<Maps, GemmGroupMaps>::value;
  const bool sk = p.sk_tiles > 0;
  const char* what = kGrouped ? "mtt_gemm_grouped" : sk ? "mtt_gemm(stream-K)" : "mtt_gemm";
  return with_tile(nsplit, bn, [&](auto cfg) {
    using Cfg = decltype(cfg);
    return with_epilogue(p, [&](auto e) {
      constexpr int NSPLIT = Cfg::kNsplit, BN = Cfg::kBN, ACT = decltype(e)::ACT, OUT = decltype(e)::OUT;
      static bool done[2][kMaxDevices] = {};  // the opt-ins of this shape's and epilogue's kernels; [1]: stream-K
      if constexpr (kGrouped) {
        return launch_kernel<Cfg>(gemm_tc_grouped_kernel<NSPLIT, BN, ACT, OUT>, done[0], what, grid, stream, maps, *grp,
                                  p);
      } else {
        if constexpr (BN == 256)
          if (sk)
            return launch_kernel<Cfg>(gemm_tc_kernel<NSPLIT, BN, true, ACT, OUT>, done[1], what, grid, stream, maps, p);
        return launch_kernel<Cfg>(gemm_tc_kernel<NSPLIT, BN, false, ACT, OUT>, done[0], what, grid, stream, maps, p);
      }
    });
  });
}

int launch_gemm_tiles_grouped(const mtt_gemm_desc* d, int count, int bn, cudaStream_t stream) {
  GemmParams p;
  GemmGroupMaps gm;
  GemmGroup grp;
  grp.count = count;
  for (int g = 0; g < count; ++g) {
    GemmParams pg;
    int rc = gemm_prepare(&d[g], bn, pg, gm.m[g]);
    if (rc) return rc;
    pg.tiles_n = (d[g].N + bn - 1) / bn;
    if (g == 0) {
      p = pg;
    } else {  // the epilogue's vector width is shared
      p.vec_ok = p.vec_ok && pg.vec_ok;
    }
    grp.prob[g] = GroupProblem{pg.bias, pg.residual, pg.out_f32, pg.out_hi, pg.out_lo};
  }
  grp.tiles_per_problem = p.tiles_m * p.tiles_n;
  const int tiles = grp.tiles_per_problem * grp.count;
  return launch_gemm(gm, &grp, p, d[0].nsplit, bn, tiles < sm_count() ? tiles : sm_count(), stream);
}

static int g_streamk = -1;  // -1: read MTT_GEMM_STREAMK once. 0 = off, 1 = automatic (default), 2 = whenever legal
void set_gemm_streamk(int mode) { g_streamk = mode < 0 ? 0 : (mode > 2 ? 2 : mode); }

// How many tiles of a `tiles`-tile, k_iters-deep problem go to the stream-K schedule on `pairs` units (CTAs here;
// 0 = none). Legal: a ragged last round whose split leaves every unit >= 4 k-blocks (the owner's wait assumes no unit is
// empty). Automatic: only a SINGLE partial round (tiles < units) that leaves >= 1/2 of the units idle and is >= 32
// k-blocks deep -- the policy kept from the first implementation of the schedule; it has not been re-tuned per shape.
int streamk_tiles(int tiles, int k_iters, int pairs) {
  if (g_streamk < 0) {
    const char* e = getenv("MTT_GEMM_STREAMK");
    set_gemm_streamk(e ? atoi(e) : 1);
  }
  if (!g_streamk || pairs < 2 || pairs * 2 * kEpiWarps * 4 > (int)kSkFlagBytes) return 0;
  const int r = tiles % pairs;
  if (r == 0 || (pairs - r) * 16 < pairs || (long long)r * k_iters / pairs < 4) return 0;
  if (g_streamk == 1 && (tiles >= pairs || (pairs - r) * 2 < pairs || k_iters < 32)) return 0;
  return r;
}

// Test hook (mtt_debug_streamk_schedule): the pieces unit `pair` of `pairs` runs, from the same code the kernel uses.
int streamk_schedule_host(int tiles, int k_iters, int pairs, int pair, int* out, int max_pieces) {
  GemmParams p = {};
  p.sk_tiles = streamk_tiles(tiles, k_iters, pairs);
  const int num_pairs = p.sk_tiles > 0 ? pairs : (tiles < pairs ? tiles : pairs);
  if (pair >= num_pairs) return 0;
  const SkSched s = sk_schedule<true>(p, pair, num_pairs, tiles, k_iters);
  int n = 0;
  for (int si = 0; si < s.n_seg && n < max_pieces; ++si, ++n) sk_piece(s, si, k_iters, out[3 * n], out[3 * n + 1], out[3 * n + 2]);
  return s.n_seg;
}

int launch_gemm_tiles(const mtt_gemm_desc* d, int bn, cudaStream_t stream) {
  GemmParams p;
  GemmMaps1 gm;
  int rc = gemm_prepare(d, bn, p, gm.m[0]);
  if (rc) return rc;
  p.tiles_n = (d->N + bn - 1) / bn;
  const int tiles = p.tiles_m * p.tiles_n;
  const int units = sm_count();
  if (bn == 256 && d->sk_ws) {
    // the caller lent a stream-K workspace (mtt_gemm_streamk_bytes): split the ragged last round of tiles along K
    const int r = streamk_tiles(tiles, p.taps * p.num_kb, units);
    if (r > 0) {
      if ((size_t)d->sk_ws_bytes < sk_workspace_bytes(units) || (reinterpret_cast<uintptr_t>(d->sk_ws) & 255))
        return set_error(MTT_ERR_BAD_SHAPE, "mtt_gemm: sk_ws of %lld bytes (256-byte aligned) < required %zu "
                         "(mtt_gemm_streamk_bytes)", (long long)d->sk_ws_bytes, sk_workspace_bytes(units));
      p.sk_tiles = r;
      p.sk_flags = static_cast<unsigned int*>(d->sk_ws);
      p.sk_part = reinterpret_cast<float*>(static_cast<uint8_t*>(d->sk_ws) + kSkFlagBytes);
    }
  }
  const int grid = p.sk_tiles > 0 ? units : (tiles < units ? tiles : units);
  return launch_gemm(gm, nullptr, p, d->nsplit, bn, grid, stream);
}

}  // namespace mtt
