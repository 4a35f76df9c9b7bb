// The reference's Cityscapes-3D training / evaluation targets (TP/data/cityscapes3d.py) over a batch of equally sized
// raw maps, in one launch:
//   disparity -> depth      (:150-160)  (d - 1) / 256 for d > 1, -1 for d <= 1, then 0 where the RAW label id is 10
//   encode_segmap           (:235-241)  void ids -> 255, the 19 valid ids -> 0..18, every other id unchanged
//   PIL NEAREST resize      (:206-221)  both maps to dd_label_map_size (H, W); (H, W) == (h, w) is the identity
// All three are pointwise, so they commute with nearest sampling: encoding / converting the sampled source pixel gives
// what the reference's encode -> float -> resize -> int order gives.
//
// PIL's NEAREST rule (Pillow 12.2, ImagingScaleAffine; restated and checked exhaustively in oracle/cityscapes_ref.py):
// with s = n_src / n_dst in double, the source coordinate of output index d is the running sum
// c_0 = s * 0.5, c_{d+1} = c_d + s (each addition rounded), and the index is trunc(c_d). The accumulated rounding
// differs from floor((d + 0.5) * s), e.g. 2 -> 7 picks source 0 at d = 3. Each block builds the x and y index tables
// in shared memory: when s is a short dyadic fraction every partial sum is exact and equals (d + 0.5) * s, so all
// threads fill the table at once (1024 -> 512 is s = 2); otherwise one thread per axis runs the reference's serial sum.
//
// Traffic: algorithmically 15 bytes per output pixel -- 1 B label id (read once; the sky test reuses it), 2 B
// disparity, 8 B int64 semseg, 4 B fp32 depth -- 31.5 MB for B = 4 at 512 x 1024. Each thread produces 4 adjacent
// pixels of a row and stores them with 16-byte vector stores (two for semseg, one for depth) when W % 4 == 0.
#include "host_common.h"

namespace mtt {

constexpr int kCsThreads = 256;
constexpr int kCsVec = 4;
constexpr int kCsIgnore = 255;

// encode_segmap's table: ids 0..33 of the void and valid lists, every other id maps to itself
__host__ __device__ constexpr int cs_encode(int id) {
  switch (id) {
    case 7: return 0;   case 8: return 1;   case 11: return 2;  case 12: return 3;  case 13: return 4;
    case 17: return 5;  case 19: return 6;  case 20: return 7;  case 21: return 8;  case 22: return 9;
    case 23: return 10; case 24: return 11; case 25: return 12; case 26: return 13; case 27: return 14;
    case 28: return 15; case 31: return 16; case 32: return 17; case 33: return 18;
    case 0: case 1: case 2: case 3: case 4: case 5: case 6: case 9: case 10: case 14: case 15: case 16: case 18:
    case 29: case 30: return kCsIgnore;
    default: return id;
  }
}

struct CsAxis {
  double step;   // n_src / n_dst
  int n_src, n_dst;
  int exact;     // the partial sums are exact: index = trunc((d + 0.5) * step)
};

// Fills tab[0..n_dst) with PIL's NEAREST source indices (see the header comment).
__device__ __forceinline__ void cs_axis_table(const CsAxis& a, int* tab, int lane_thread) {
  if (a.exact) {
    for (int d = threadIdx.x; d < a.n_dst; d += blockDim.x)
      tab[d] = min((int)__dmul_rn((double)d + 0.5, a.step), a.n_src - 1);
  } else if (threadIdx.x == lane_thread) {
    double c = __dmul_rn(a.step, 0.5);
    for (int d = 0; d < a.n_dst; ++d) {
      tab[d] = min((int)c, a.n_src - 1);   // PIL stops at n_src (never reached at these sizes); the clamp is a guard
      c = __dadd_rn(c, a.step);
    }
  }
}

struct CsPixel {
  long long sem;
  float depth;
};

__device__ __forceinline__ CsPixel cs_pixel(int id, const uint16_t* disp_row, int sx, const uint8_t* lut) {
  CsPixel p;
  p.sem = lut[id];
  p.depth = 0.f;
  if (disp_row) {
    const int d = disp_row[sx];
    // (d - 1) / 256 in fp32 (exact) and -1 where the disparity is invalid, then 0 where the RAW label id is 10. The
    // reference rewrites one array in place (:153 then :156), so d == 1 becomes 0 first and then -1 as well. It calls
    // the last mask the sky (`sky_mask = lbl == 10`, :159-160), but Cityscapes id 10 is "rail track" and sky is 23.
    // Both are reproduced as the reference has them, so the targets and depth scores match the reference's.
    p.depth = d > 1 ? __fdiv_rn(__fsub_rn((float)d, 1.f), 256.f) : -1.f;
    if (id == 10) p.depth = 0.f;
  }
  return p;
}

template <bool kVec>
__global__ void __launch_bounds__(kCsThreads)
cityscapes_targets_kernel(const uint8_t* __restrict__ ids, const uint16_t* __restrict__ disp, int B, int h, int w,
                          int H, int W, CsAxis ay, CsAxis ax, long long* __restrict__ semseg,
                          float* __restrict__ depth) {
  extern __shared__ int cs_smem[];
  int* xs = cs_smem;
  int* ys = cs_smem + W;
  uint8_t* lut = reinterpret_cast<uint8_t*>(cs_smem + W + H);
  for (int i = threadIdx.x; i < 256; i += blockDim.x) lut[i] = (uint8_t)cs_encode(i);
  cs_axis_table(ax, xs, 0);
  cs_axis_table(ay, ys, 32);
  __syncthreads();

  const int per_row = kVec ? W / kCsVec : W;
  const long long items = (long long)B * H * per_row;
  for (long long it = (long long)blockIdx.x * blockDim.x + threadIdx.x; it < items;
       it += (long long)gridDim.x * blockDim.x) {
    const long long row = it / per_row;            // b * H + y
    const int x0 = (int)(it - row * per_row) * (kVec ? kCsVec : 1);
    const int b = (int)(row / H), y = (int)(row - (long long)b * H);
    const long long src_row = (long long)b * h + ys[y];
    const uint8_t* id_row = ids + src_row * w;
    const uint16_t* disp_row = depth ? disp + src_row * w : nullptr;
    const long long o = row * W + x0;
    if constexpr (kVec) {
      CsPixel px[kCsVec];
#pragma unroll
      for (int j = 0; j < kCsVec; ++j) {
        const int sx = xs[x0 + j];
        px[j] = cs_pixel(id_row[sx], disp_row, sx, lut);
      }
      if (semseg) {
        longlong2* s2 = reinterpret_cast<longlong2*>(semseg + o);
        s2[0] = make_longlong2(px[0].sem, px[1].sem);
        s2[1] = make_longlong2(px[2].sem, px[3].sem);
      }
      if (depth) *reinterpret_cast<float4*>(depth + o) = make_float4(px[0].depth, px[1].depth, px[2].depth, px[3].depth);
    } else {
      const int sx = xs[x0];
      const CsPixel p = cs_pixel(id_row[sx], disp_row, sx, lut);
      if (semseg) semseg[o] = p.sem;
      if (depth) depth[o] = p.depth;
    }
  }
}

CsAxis cs_axis(int n_src, int n_dst) {
  CsAxis a;
  a.step = (double)n_src / (double)n_dst;
  a.n_src = n_src;
  a.n_dst = n_dst;
  // step = m / 2^30 with (2 n_dst + 1) m < 2^53: every c_d = (2d + 1) m / 2^31 is a double, so the serial sum is exact
  const double m = ldexp(a.step, 30);
  a.exact = m == floor(m) && (2.0 * n_dst + 1.0) * m < 9007199254740992.0;
  return a;
}

}  // namespace mtt

extern "C" int mtt_cityscapes_targets(const uint8_t* label_ids, const uint16_t* disparity, int32_t B, int32_t h,
                                      int32_t w, int32_t H, int32_t W, int64_t* semseg, float* depth,
                                      mtt_stream_t stream) {
  using namespace mtt;
  if (!label_ids || (!semseg && !depth) || (depth && !disparity) || B <= 0 || h <= 0 || w <= 0 || H <= 0 || W <= 0)
    return set_error(MTT_ERR_BAD_SHAPE,
                     "mtt_cityscapes_targets: bad arguments (B=%d h=%d w=%d H=%d W=%d; label ids and at least one "
                     "output are required, depth needs the disparity)", B, h, w, H, W);
  const size_t smem = (size_t)(H + W) * sizeof(int) + 256;
  if (smem > 48 * 1024)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_cityscapes_targets: %d x %d output needs %zu bytes of index tables (at "
                     "most 48 KB)", H, W, smem);
  const bool vec = W % kCsVec == 0 && (reinterpret_cast<uintptr_t>(semseg) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(depth) & 15) == 0;
  const long long items = (long long)B * H * (vec ? W / kCsVec : W);
  const long long want = (items + kCsThreads - 1) / kCsThreads;
  const unsigned grid = (unsigned)(want < 8LL * sm_count() ? want : 8LL * sm_count());
  const CsAxis ay = cs_axis(h, H), ax = cs_axis(w, W);
  auto* sem = reinterpret_cast<long long*>(semseg);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (vec)
    cityscapes_targets_kernel<true><<<grid, kCsThreads, smem, st>>>(label_ids, disparity, B, h, w, H, W, ay, ax, sem,
                                                                     depth);
  else
    cityscapes_targets_kernel<false><<<grid, kCsThreads, smem, st>>>(label_ids, disparity, B, h, w, H, W, ay, ax, sem,
                                                                      depth);
  return check_launch("mtt_cityscapes_targets");
}
