// Host side of mtt_gemm: descriptor validation, tensor-map encoding, kernel-variant selection.
#include <stdlib.h>

#include "gemm_common.cuh"

namespace mtt {

// Pick the TH x TW (<= 128 pixel) output patch that wastes the fewest MMA rows.
static void pick_conv_tile(int H, int W, int* TW, int* TH) {
  double best = -1;
  int btw = 1, bth = 1;
  for (int tw = 1; tw <= 128 && tw <= W; ++tw) {
    int th = 128 / tw;
    if (th > H) th = H;
    if (th < 1) continue;
    const long long tiles = (long long)((W + tw - 1) / tw) * ((H + th - 1) / th);
    const double eff = (double)H * W / ((double)tiles * 128.0);
    if (eff > best + 1e-9 || (eff > best - 1e-9 && tw > btw)) {
      best = eff;
      btw = tw;
      bth = th;
    }
  }
  *TW = btw;
  *TH = bth;
}

// The tensor maps of one split-bf16 operand: the hi plane's in maps[0], the lo plane's in maps[1] (nsplit 1 has no lo
// plane; maps[1] repeats maps[0]).
static int make_split_maps(const void* hi, const void* lo, int nsplit, int rank, const uint64_t* dims,
                           const uint64_t* strides, const uint32_t* box, CUtensorMap* maps) {
  int rc = make_tmap_bf16(&maps[0], hi, rank, dims, strides, box);
  if (rc) return rc;
  if (nsplit == 2) return make_tmap_bf16(&maps[1], lo, rank, dims, strides, box);
  maps[1] = maps[0];
  return MTT_OK;
}

int gemm_prepare(const mtt_gemm_desc* d, int b_box_rows, GemmParams& p, CUtensorMap maps[4]) {
  if (!d) return set_error(MTT_ERR_BAD_SHAPE, "mtt_gemm: null descriptor");
  if (d->M <= 0 || d->N <= 0 || d->K <= 0)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_gemm: M=%d N=%d K=%d must be positive", d->M, d->N, d->K);
  if (d->nsplit != 1 && d->nsplit != 2)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_gemm: nsplit=%d (1 or 2)", d->nsplit);
  if (!d->a_hi || !d->b_hi || (d->nsplit == 2 && (!d->a_lo || !d->b_lo)))
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_gemm: missing operand plane");
  if (!d->out_f32 && !d->out_hi) return set_error(MTT_ERR_BAD_SHAPE, "mtt_gemm: no output");
  if (d->act != MTT_ACT_NONE && d->act != MTT_ACT_GELU && d->act != MTT_ACT_RELU)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_gemm: act=%d (0 none, 1 GELU, 2 ReLU)", d->act);
  if (d->lda % 8 || d->ldb % 8)
    return set_error(MTT_ERR_MISALIGNED, "mtt_gemm: lda=%lld ldb=%lld must be multiples of 8",
                     (long long)d->lda, (long long)d->ldb);

  p = GemmParams{};
  {
    static int dbg = -1;
    if (dbg < 0) {
      const char* e = getenv("MTT_GEMM_DEBUG");
      dbg = e ? atoi(e) : 0;
    }
    p.debug = dbg;
  }
  p.M = d->M;
  p.N = d->N;
  p.mode = d->mode;
  p.num_kb = (d->K + BK - 1) / BK;
  p.k_last_steps = (d->K - (p.num_kb - 1) * BK + 15) / 16;  // columns past K are TMA zero fill: skip their MMAs
  p.tiles_n = 0;
  p.bias = d->bias;
  p.act = d->act;
  p.residual = d->residual;
  p.ldr = d->ldr;
  p.res_row_mod = d->res_row_mod;
  p.out_f32 = d->out_f32;
  p.ldo_f32 = d->ldo_f32;
  p.out_hi = static_cast<__nv_bfloat16*>(d->out_hi);
  p.out_lo = static_cast<__nv_bfloat16*>(d->out_lo);  // written whenever given: nsplit = 1 leaves no stale lo plane
  p.ldo_bf = d->ldo_bf;
  p.in_group = d->in_group;
  p.out_group = d->out_group;
  p.out_offset = d->out_offset;
  p.out_row_stride = d->out_row_stride > 1 ? d->out_row_stride : 1;
  if (p.out_hi && d->nsplit == 2 && !p.out_lo)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_gemm: out_lo missing for nsplit=2");

  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  p.vec_ok = 1;
  if (d->bias && !al16(d->bias)) p.vec_ok = 0;
  if (d->residual && (!al16(d->residual) || d->ldr % 4)) p.vec_ok = 0;
  if (d->out_f32 && (!al16(d->out_f32) || d->ldo_f32 % 4)) p.vec_ok = 0;
  if (d->out_hi && (!al16(d->out_hi) || d->ldo_bf % 8 || (p.out_lo && !al16(p.out_lo)))) p.vec_ok = 0;

  int rc;
  const int ksq = (d->mode == 1) ? d->ksize * d->ksize : 1;
  if (d->mode == 0 && d->a_group_rows > 0) {
    // gathered A: logical row r = (g, i) lives at physical row g * a_group_stride + i, i < a_group_rows
    const int g = d->a_group_rows;
    if (g > BM || d->M % g || d->a_group_stride < g)
      return set_error(MTT_ERR_BAD_SHAPE, "mtt_gemm: a_group_rows=%d must divide M=%d and be <= %d", g, d->M, BM);
    const int ngroups = d->M / g;
    const int gpt = BM / g;  // groups per tile
    if (ngroups > gpt && BM % g)
      return set_error(MTT_ERR_BAD_SHAPE, "mtt_gemm: %d groups of %d rows need %d %% %d == 0", ngroups, g, BM, g);
    p.taps = 1;
    p.ksize = 1;
    p.dil = 1;
    p.cin_pad = 0;
    p.a_groups_per_tile = ngroups < gpt ? ngroups : gpt;
    p.tiles_m = (ngroups + p.a_groups_per_tile - 1) / p.a_groups_per_tile;
    if (p.tiles_m > 1 && p.a_groups_per_tile * g != BM)
      return set_error(MTT_ERR_BAD_SHAPE, "mtt_gemm: gathered A tiles must be full");
    p.a_box_bytes = (uint32_t)(p.a_groups_per_tile * g) * BK * 2;
    const uint64_t dims[3] = {(uint64_t)d->K, (uint64_t)g, (uint64_t)ngroups};
    const uint64_t str[2] = {(uint64_t)d->lda * 2, (uint64_t)d->a_group_stride * d->lda * 2};
    const uint32_t box[3] = {BK, (uint32_t)g, (uint32_t)p.a_groups_per_tile};
    if ((rc = make_split_maps(d->a_hi, d->a_lo, d->nsplit, 3, dims, str, box, &maps[0]))) return rc;
  } else if (d->mode == 0) {
    p.taps = 1;
    p.ksize = 1;
    p.dil = 1;
    p.cin_pad = 0;
    p.tiles_m = (d->M + BM - 1) / BM;
    p.a_box_bytes = kTileBytes;
    const uint64_t dims[2] = {(uint64_t)d->K, (uint64_t)d->M};
    const uint64_t str[1] = {(uint64_t)d->lda * 2};
    const uint32_t box[2] = {BK, BM};
    if ((rc = make_split_maps(d->a_hi, d->a_lo, d->nsplit, 2, dims, str, box, &maps[0]))) return rc;
  } else if (d->mode == 1) {
    if (d->B <= 0 || d->H <= 0 || d->W <= 0 || (long long)d->B * d->H * d->W != d->M)
      return set_error(MTT_ERR_BAD_SHAPE, "mtt_gemm(conv): B*H*W = %d*%d*%d != M = %d", d->B, d->H,
                       d->W, d->M);
    if (d->ksize != 1 && d->ksize != 3)
      return set_error(MTT_ERR_BAD_SHAPE, "mtt_gemm(conv): ksize=%d (1 or 3)", d->ksize);
    if (d->dil < 1) return set_error(MTT_ERR_BAD_SHAPE, "mtt_gemm(conv): dil=%d", d->dil);
    p.taps = ksq;
    p.ksize = d->ksize;
    p.dil = d->dil;
    p.cin_pad = p.num_kb * BK;
    p.NB = d->B;
    p.H = d->H;
    p.W = d->W;
    pick_conv_tile(d->H, d->W, &p.TW, &p.TH);
    p.tiles_x = (d->W + p.TW - 1) / p.TW;
    p.tiles_y = (d->H + p.TH - 1) / p.TH;
    p.tiles_m = d->B * p.tiles_x * p.tiles_y;
    p.a_box_bytes = (uint32_t)(p.TW * p.TH) * BK * 2;
    const uint64_t dims[4] = {(uint64_t)d->K, (uint64_t)d->W, (uint64_t)d->H, (uint64_t)d->B};
    const uint64_t str[3] = {(uint64_t)d->lda * 2, (uint64_t)d->W * d->lda * 2,
                             (uint64_t)d->H * d->W * d->lda * 2};
    const uint32_t box[4] = {BK, (uint32_t)p.TW, (uint32_t)p.TH, 1};
    if ((rc = make_split_maps(d->a_hi, d->a_lo, d->nsplit, 4, dims, str, box, &maps[0]))) return rc;
  } else {
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_gemm: mode=%d", d->mode);
  }
  {
    const uint64_t ktot = (d->mode == 1) ? (uint64_t)ksq * p.cin_pad : (uint64_t)d->K;
    if ((uint64_t)d->ldb < ktot)
      return set_error(MTT_ERR_BAD_SHAPE, "mtt_gemm: ldb=%lld < packed K=%llu", (long long)d->ldb,
                       (unsigned long long)ktot);
    const uint64_t dims[2] = {ktot, (uint64_t)d->N};
    const uint64_t str[1] = {(uint64_t)d->ldb * 2};
    const uint32_t box[2] = {BK, (uint32_t)b_box_rows};
    if ((rc = make_split_maps(d->b_hi, d->b_lo, d->nsplit, 2, dims, str, box, &maps[2]))) return rc;
  }
  return MTT_OK;
}

// -1: read MTT_GEMM_VARIANT once; 0 auto, 1 = 128x128 tiles, 2 = 128x256 tiles (stream-K capable), 3 = 128x128 tiles
// (the number once named a CTA-pair tile shape; it is kept so that existing settings still select a valid kernel)
static int g_variant = -1;

// Columns per tile (128 or 256) for `count` problems of d's geometry. g_variant decides for every launch when it is
// not 0; MTT_GEMM_GROUPED_VARIANT (0 auto, 1, 2) is an A/B knob for grouped launches (count > 1) only. Otherwise the
// choice is made by tile counts, not per-shape timings.
static int tile_width(const mtt_gemm_desc* d, int count) {
  static int grouped = -1;
  if (g_variant < 0) {
    const char* e = getenv("MTT_GEMM_VARIANT");
    g_variant = e ? atoi(e) : 0;
  }
  if (grouped < 0) {
    const char* e = getenv("MTT_GEMM_GROUPED_VARIANT");
    grouped = e ? atoi(e) : 0;
  }
  int v = g_variant;
  if (v == 0 && count > 1) v = grouped;
  if (v == 0) {
    const int n256 = (d->N + 255) / 256 * 256;
    const long long wide_tiles = (long long)count * ((d->M + 127) / 128) * (n256 / 256);
    if (count > 1) {
      // Grouping can fill the SMs with 128 x 256 tiles where one problem alone could not: with >= one wave of wide
      // tiles and N close to a multiple of 256 they take the wide kernel. Gathered-A problems and tiny M stay on
      // 128 x 128.
      v = (d->a_group_rows == 0 && d->M >= 512 && d->N >= 256 && (n256 - d->N) * 8 <= n256 && wide_tiles >= sm_count())
              ? 2 : 1;
    } else if (d->mode == 1) {
      // The 128 x 256 tile reads half the B bytes per output of the 128 x 128 tile and gives each consumer warpgroup a
      // 64 x 256 wgmma; it needs enough tiles to fill the SMs and little waste in the last N tile. Narrow or ragged N
      // (decoder widths 300 / 350), short K and skinny M stay on 128 x 128.
      const long long k_eff = (long long)d->K * d->ksize * d->ksize;
      v = (k_eff >= 2048 && wide_tiles >= sm_count() && d->N > 256 && (n256 - d->N) * 8 <= n256) ? 2 : 1;
    } else {
      const bool wide = d->N >= 512 && (n256 - d->N) * 8 <= n256;
      v = (wide && d->M > 128 && (d->N >= 2048 || d->K >= 2048)) ? 2 : 1;
    }
  }
  return v == 2 ? 256 : 128;
}

}  // namespace mtt

extern "C" void mtt_set_gemm_variant(int v) { mtt::g_variant = v; }
extern "C" void mtt_set_gemm_streamk(int mode) { mtt::set_gemm_streamk(mode); }
extern "C" int mtt_debug_streamk_schedule(int32_t tiles, int32_t k_iters, int32_t pairs, int32_t pair, int32_t* pieces,
                                          int32_t max_pieces) {
  return mtt::streamk_schedule_host(tiles, k_iters, pairs, pair, pieces, max_pieces);
}
extern "C" size_t mtt_gemm_streamk_bytes(void) {
  const int n = mtt::sm_count();
  return mtt::sk_workspace_bytes(n > 0 ? n : 132);
}

extern "C" int mtt_gemm(const mtt_gemm_desc* d, mtt_stream_t stream_) {
  using namespace mtt;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!d) return set_error(MTT_ERR_BAD_SHAPE, "mtt_gemm: null descriptor");
  const int bn = tile_width(d, 1);
  const int taps = d->mode == 1 ? d->ksize * d->ksize : 1;
  ProfileScope prof(stream, 0, 2.0 * d->M * d->N * d->K * taps, d->M, d->N, d->K * taps);
  return launch_gemm_tiles(d, bn, stream);
}

extern "C" int mtt_gemm_grouped(const mtt_gemm_desc* d, int32_t count, mtt_stream_t stream_) {
  using namespace mtt;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!d || count <= 0) return set_error(MTT_ERR_BAD_SHAPE, "mtt_gemm_grouped: no problems");
  if (count == 1) return mtt_gemm(d, stream_);
  if (count > kMaxGroup) return set_error(MTT_ERR_BAD_SHAPE, "mtt_gemm_grouped: %d problems > %d", count, kMaxGroup);
  const mtt_gemm_desc& a = d[0];
  for (int g = 1; g < count; ++g) {
    const mtt_gemm_desc& b = d[g];
    const bool same = a.M == b.M && a.N == b.N && a.K == b.K && a.nsplit == b.nsplit && a.mode == b.mode && a.B == b.B &&
                      a.H == b.H && a.W == b.W && a.ksize == b.ksize && a.dil == b.dil && a.act == b.act &&
                      a.lda == b.lda && a.ldb == b.ldb && a.ldr == b.ldr && a.res_row_mod == b.res_row_mod &&
                      a.ldo_f32 == b.ldo_f32 && a.ldo_bf == b.ldo_bf && a.in_group == b.in_group &&
                      a.out_group == b.out_group && a.out_offset == b.out_offset && a.out_row_stride == b.out_row_stride &&
                      a.a_group_rows == b.a_group_rows && a.a_group_stride == b.a_group_stride &&
                      (a.bias == nullptr) == (b.bias == nullptr) && (a.residual == nullptr) == (b.residual == nullptr) &&
                      (a.out_f32 == nullptr) == (b.out_f32 == nullptr) && (a.out_hi == nullptr) == (b.out_hi == nullptr);
    if (!same)
      return set_error(MTT_ERR_BAD_SHAPE, "mtt_gemm_grouped: problem %d differs from problem 0 in more than its pointers", g);
  }
  double fl = 0;
  for (int g = 0; g < count; ++g) fl += 2.0 * d[g].M * d[g].N * d[g].K * (d[g].mode == 1 ? d[g].ksize * d[g].ksize : 1);
  ProfileScope prof(stream, 0, fl, a.M * count, a.N, a.K * (a.mode == 1 ? a.ksize * a.ksize : 1));
  return launch_gemm_tiles_grouped(d, count, tile_width(d, count), stream);
}
