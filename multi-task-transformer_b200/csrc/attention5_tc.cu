// Fused multi-head attention, the kernel of mtt_attention (contract in attention_tc.cu:
// TP/models/transformers/taskprompter.py:204-210, prompt-row raw logits :436-437,:482; IP vit.py:189-193).
//
// Warp-specialised wgmma kernel for sm_90a.  Each CTA (512 threads, one CTA per SM) owns one (batch, head,
// 192-query tile) item:
//   * warpgroup 0 = TMA producer (warp 0 issues; the warpgroup gives its registers to the consumers with setmaxnreg):
//     the item's query tile once, then 64-key K and V blocks through three-stage rings;
//   * warpgroups 1-3 = consumers, 64 query rows each.  A consumer warpgroup whose rows all lie past N exits at once;
//     the K / V release barriers count only the warpgroups with rows inside the sequence.  Per key block: S = Q K^T
//     as an SS-form wgmma (m64n64k16, Q and K from shared memory), an online softmax on the accumulator fragment (a
//     row lives in the four lanes of a quad: max / sum exchange by two shuffles), then P V as an RS-form wgmma that takes P straight
//     from registers -- the S accumulator fragment of 16 keys is, element for element, the A fragment of one k16 step --
//     added to the rescaled O in fp32 (not accumulated inside the tensor core, which truncates);
//   * split-bf16 parity mode (NSPLIT = 2): every product is hi*hi + hi*lo + lo*hi, P included (split on the fly);
//   * O stays in registers for the whole item and is normalised and stored (hi / lo planes) at the end.
#include <math.h>

#include "host_common.h"
#include "ptx.cuh"

namespace mtt {

// Three consumer warpgroups at 160 registers (parity mode needs O, the block's PV accumulator and the split P
// fragments live at once: 96 registers before addressing) and a 24-register producer warpgroup fill the register file:
// 128 * 24 + 384 * 160 = 64512 of 65536.
constexpr int kA5ConsumerWGs = 3;
constexpr int kA5Rows = 64 * kA5ConsumerWGs;             // query rows per item
constexpr int kA5Threads = 128 + 128 * kA5ConsumerWGs;   // producer warpgroup + consumers
constexpr uint32_t kA5QTile = kA5Rows * 64 * 2;          // one plane of the query tile (24 KB)
constexpr uint32_t kA5KVTile = 64 * 64 * 2;              // one plane of a 64-key K or V block (8 KB)
constexpr int kA5Stages = 3;

struct Attn5Params {
  int B, N, H, T;
  float scale_log2;  // scale * log2(e)
  __nv_bfloat16* out_hi;
  __nv_bfloat16* out_lo;
  float* prompt_logits;
};

template <int NSPLIT>
__global__ void __launch_bounds__(kA5Threads, 1)
attention5_kernel(const __grid_constant__ CUtensorMap tmq_hi, const __grid_constant__ CUtensorMap tmq_lo,
                  const __grid_constant__ CUtensorMap tmk_hi, const __grid_constant__ CUtensorMap tmk_lo,
                  const Attn5Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sQ = smem;                                 // [NSPLIT][16 KB]
  uint8_t* sK = sQ + NSPLIT * kA5QTile;               // [kA5Stages][NSPLIT][8 KB]
  uint8_t* sV = sK + kA5Stages * NSPLIT * kA5KVTile;  // [kA5Stages][NSPLIT][8 KB]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + kA5Stages * NSPLIT * kA5KVTile);
  uint64_t* q_full = bars;
  uint64_t* k_full = bars + 1;
  uint64_t* k_empty = k_full + kA5Stages;
  uint64_t* v_full = k_empty + kA5Stages;
  uint64_t* v_empty = v_full + kA5Stages;

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  const int C = p.H * 64;
  const int nkv = (p.N + 63) / 64;
  // query-tile-major order: the last tile of every (batch, head), the one with rows past N, is dispatched last
  const int qt = blockIdx.x / (p.B * p.H);
  const int h = blockIdx.x % p.H;
  const int b = (blockIdx.x / p.H) % p.B;
  const int n_act = min(kA5ConsumerWGs, (p.N - qt * kA5Rows + 63) / 64);  // consumer warpgroups with rows < N

  if (tid == 0) {
    tma_prefetch_desc(&tmq_hi);
    tma_prefetch_desc(&tmk_hi);
    if (NSPLIT == 2) {
      tma_prefetch_desc(&tmq_lo);
      tma_prefetch_desc(&tmk_lo);
    }
    mbar_init(q_full, 1);
    for (int s = 0; s < kA5Stages; ++s) {
      mbar_init(&k_full[s], 1);
      mbar_init(&k_empty[s], 4 * n_act);  // one arrival per active consumer warp
      mbar_init(&v_full[s], 1);
      mbar_init(&v_empty[s], 4 * n_act);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ------------------------------------------------------------------ TMA producer (warp 0, elected lane issues)
    setmaxnreg_dec<24>();
    if (warp != 0) return;
    if (elect_one()) {
      mbar_arrive_expect_tx(q_full, NSPLIT * kA5QTile);
      tma_load_3d(sQ, &tmq_hi, q_full, h * 64, qt * kA5Rows, b);
      if (NSPLIT == 2) tma_load_3d(sQ + kA5QTile, &tmq_lo, q_full, h * 64, qt * kA5Rows, b);
    }
    __syncwarp();
    for (int j = 0; j < nkv; ++j) {
      const int s = j % kA5Stages;
      const uint32_t ph = (j / kA5Stages) & 1;
      mbar_wait(&k_empty[s], ph ^ 1);
      if (elect_one()) {
        uint8_t* dk = sK + s * NSPLIT * kA5KVTile;
        mbar_arrive_expect_tx(&k_full[s], NSPLIT * kA5KVTile);
        tma_load_3d(dk, &tmk_hi, &k_full[s], C + h * 64, j * 64, b);
        if (NSPLIT == 2) tma_load_3d(dk + kA5KVTile, &tmk_lo, &k_full[s], C + h * 64, j * 64, b);
      }
      __syncwarp();
      mbar_wait(&v_empty[s], ph ^ 1);
      if (elect_one()) {
        uint8_t* dv = sV + s * NSPLIT * kA5KVTile;
        mbar_arrive_expect_tx(&v_full[s], NSPLIT * kA5KVTile);
        tma_load_3d(dv, &tmk_hi, &v_full[s], 2 * C + h * 64, j * 64, b);
        if (NSPLIT == 2) tma_load_3d(dv + kA5KVTile, &tmk_lo, &v_full[s], 2 * C + h * 64, j * 64, b);
      }
      __syncwarp();
    }
    return;
  }

  // -------------------------------------------------------------------- consumers
  setmaxnreg_inc<160>();
  const int cw = (warp >> 2) - 1;                             // rows [64 cw, 64 cw + 64) of the query tile
  if (cw >= n_act) return;                                    // all rows past N: no MMA, not counted by the barriers
  const int rloc = cw * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's rows: rloc and rloc + 8
  const int col0 = 2 * (lane & 3);                            // ... and columns col0 + 8 i + {0, 1}
  const uint32_t q_hi = smem_u32(sQ) + (uint32_t)cw * 64 * 128;
  const uint32_t q_lo = q_hi + kA5QTile;
  const float sl2 = p.scale_log2;

  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY};  // running maximum of the scaled logits (log2 domain), per row
  float l_run[2] = {0.f, 0.f};              // this thread's share of the row sums

  mbar_wait(q_full, 0);
  for (int j = 0; j < nkv; ++j) {
    const int s = j % kA5Stages;
    const uint32_t ph = (j / kA5Stages) & 1;
    const int kn = min(64, p.N - j * 64);

    // ---- S = Q K^T (64 rows x 64 keys per warpgroup)
    float sc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) sc[i] = 0.f;
    mbar_wait(&k_full[s], ph);
    const uint32_t k_hi = smem_u32(sK + s * NSPLIT * kA5KVTile), k_lo = k_hi + kA5KVTile;
    wgmma_fence_regs(sc);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const uint64_t qdh = gmma_desc_sw128(q_hi + ks * 32), kdh = gmma_desc_sw128(k_hi + ks * 32);
      wgmma_ss_n64<0>(sc, qdh, kdh, 1);
      if (NSPLIT == 2) {
        wgmma_ss_n64<0>(sc, qdh, gmma_desc_sw128(k_lo + ks * 32), 1);
        wgmma_ss_n64<0>(sc, gmma_desc_sw128(q_lo + ks * 32), kdh, 1);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&k_empty[s]);

    // ---- the raw logits of the prompt rows
    if (p.prompt_logits) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int q_row = qt * kA5Rows + rloc + 8 * hh;
        if (q_row < p.T) {
          float* ex = p.prompt_logits + (((long long)b * p.H + h) * p.T + q_row) * p.N + j * 64;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int c = 8 * i + col0;
            if (c < kn) ex[c] = sc[4 * i + 2 * hh];
            if (c + 1 < kn) ex[c + 1] = sc[4 * i + 2 * hh + 1];
          }
        }
      }
    }

    // ---- online softmax on the fragment: P = exp2(S c - m), O and l rescaled when m moves
    float alpha[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          if (8 * i + col0 + e >= kn) sc[4 * i + 2 * hh + e] = -INFINITY;  // keys past N (TMA zero fill)
          mx = fmaxf(mx, sc[4 * i + 2 * hh + e]);
        }
      }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[hh], mx * sl2);
      alpha[hh] = ex2_approx(m_run[hh] - m_new);  // 0 on the first block (m_run = -inf)
      m_run[hh] = m_new;
      float sum = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float pv = ex2_approx(fmaf(sc[4 * i + 2 * hh + e], sl2, -m_new));
          sc[4 * i + 2 * hh + e] = pv;
          sum += pv;
        }
      }
      l_run[hh] = l_run[hh] * alpha[hh] + sum;
    }

    // ---- O = alpha O + P V: the fragment of keys [16 kk, 16 kk + 16) is the A operand of k-step kk. The block's PV
    // is summed in a fresh accumulator and added to O with round-to-nearest FMAs: the tensor core adds into its
    // accumulator with truncation, which over many key blocks would bias O towards zero. A ragged last block runs all
    // four k-steps (P is 0 past N, V zero-filled): a divergent exit inside the chain makes ptxas serialise its MMAs.
    uint32_t ph_[4][4], pl_[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int i = 2 * kk + (r >> 1), hh = r & 1;
        if (NSPLIT == 2) split_pack2(sc[4 * i + 2 * hh], sc[4 * i + 2 * hh + 1], ph_[kk][r], pl_[kk][r]);
        else ph_[kk][r] = pack_bf16x2(sc[4 * i + 2 * hh], sc[4 * i + 2 * hh + 1]);
      }
    }
    mbar_wait(&v_full[s], ph);
    const uint32_t v_hi = smem_u32(sV + s * NSPLIT * kA5KVTile), v_lo = v_hi + kA5KVTile;
    float pvb[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) pvb[i] = 0.f;
    wgmma_fence_regs(pvb);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const uint64_t vdh = gmma_desc_sw128(v_hi + kk * 2048);  // V rows are keys: MN-major B operand
      wgmma_rs_n64<1>(pvb, ph_[kk], vdh, kk > 0 ? 1 : 0);
      if (NSPLIT == 2) {
        wgmma_rs_n64<1>(pvb, ph_[kk], gmma_desc_sw128(v_lo + kk * 2048), 1);
        wgmma_rs_n64<1>(pvb, pl_[kk], vdh, 1);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(pvb);
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int r = 0; r < 4; ++r) o[4 * i + r] = fmaf(o[4 * i + r], alpha[r >> 1], pvb[4 * i + r]);
    __syncwarp();
    if (lane == 0) mbar_arrive(&v_empty[s]);
  }

  // ---- epilogue: O / l, split, store the rows inside the sequence
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float l = l_run[hh];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = 1.0f / l;
    const int q_row = qt * kA5Rows + rloc + 8 * hh;
    if (q_row >= p.N) continue;
    const long long off = ((long long)b * p.N + q_row) * C + h * 64 + col0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      uint32_t hv, lv;
      split_pack2(o[4 * i + 2 * hh] * inv, o[4 * i + 2 * hh + 1] * inv, hv, lv);
      *reinterpret_cast<uint32_t*>(p.out_hi + off + 8 * i) = hv;
      if (NSPLIT == 2 || p.out_lo) *reinterpret_cast<uint32_t*>(p.out_lo + off + 8 * i) = lv;
    }
  }
}

template <int NSPLIT>
static int launch_attn5(const CUtensorMap* maps, const Attn5Params& p, cudaStream_t stream) {
  constexpr uint32_t smem = NSPLIT * kA5QTile + 2 * kA5Stages * NSPLIT * kA5KVTile + 1024 + 256;
  static bool attr_set[kMaxDevices] = {};  // the opt-in is per device (and per kernel instantiation)
  const int dev_ = current_device();
  if (!attr_set[dev_]) {
    cudaError_t e = cudaFuncSetAttribute(attention5_kernel<NSPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess)
      return set_error(MTT_ERR_LAUNCH, "attention: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    attr_set[dev_] = true;
  }
  const int total = ((p.N + kA5Rows - 1) / kA5Rows) * p.H * p.B;
  attention5_kernel<NSPLIT><<<total, kA5Threads, smem, stream>>>(maps[0], maps[1], maps[2], maps[3], p);
  return check_launch("mtt_attention");
}

int launch_attention5(const mtt_attn_desc* d, cudaStream_t stream) {
  const int C = d->H * 64;
  CUtensorMap maps[4];   // q hi/lo (kA5Rows-row box), k|v hi/lo (64-row box)
  const uint64_t dims[3] = {(uint64_t)3 * C, (uint64_t)d->N, (uint64_t)d->B};
  const uint64_t str[2] = {(uint64_t)3 * C * 2, (uint64_t)d->N * 3 * C * 2};
  const uint32_t qbox[3] = {64, kA5Rows, 1};
  const uint32_t kbox[3] = {64, 64, 1};
  int rc;
  if ((rc = make_tmap_bf16(&maps[0], d->qkv_hi, 3, dims, str, qbox))) return rc;
  if ((rc = make_tmap_bf16(&maps[2], d->qkv_hi, 3, dims, str, kbox))) return rc;
  if (d->nsplit == 2) {
    if ((rc = make_tmap_bf16(&maps[1], d->qkv_lo, 3, dims, str, qbox))) return rc;
    if ((rc = make_tmap_bf16(&maps[3], d->qkv_lo, 3, dims, str, kbox))) return rc;
  } else {
    maps[1] = maps[0];
    maps[3] = maps[2];
  }
  Attn5Params p;
  p.B = d->B;
  p.N = d->N;
  p.H = d->H;
  p.T = d->prompt_logits ? d->T : 0;
  p.scale_log2 = d->scale * 1.4426950408889634f;
  p.out_hi = static_cast<__nv_bfloat16*>(d->out_hi);
  p.out_lo = static_cast<__nv_bfloat16*>(d->out_lo);
  p.prompt_logits = d->prompt_logits;
  return d->nsplit == 2 ? launch_attn5<2>(maps, p, stream) : launch_attn5<1>(maps, p, stream);
}

}  // namespace mtt
