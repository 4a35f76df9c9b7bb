// Device helpers shared by the HBM-bound glue kernels around the GEMMs: warp and block reductions, the grouped-row map,
// the channel-prompt window of a patch pixel, and the split-bf16 plane stores. A forward kernel and its adjoint take
// their index formulas from here (the bilinear coordinate: bilin_coord, postproc.cuh), so the two cannot drift apart.
#pragma once
#include "ptx.cuh"

namespace mtt {

// ---------------------------------------------------------------- reductions
// xor butterfly: every lane ends with the warp's total, summed in the same order on every lane
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Sum over the block in a fixed tree order (bitwise reproducible); sh holds blockDim.x elements, blockDim.x is a power
// of two, and every thread of the block calls it.
template <class T>
__device__ __forceinline__ T block_sum(T v, T* sh) {
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int s = blockDim.x >> 1; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  const T r = sh[0];
  __syncthreads();
  return r;
}

// ---------------------------------------------------------------- indexing
// physical row of logical row r of a grouped buffer: (r / in_group) * src_group + src_off + r % in_group
// (in_group = 0: no grouping, r + src_off)
__device__ __forceinline__ long long map_row(long long r, long long in_group, long long src_group, long long src_off) {
  return in_group > 0 ? (r / in_group) * src_group + src_off + r % in_group : r + src_off;
}

// channel-prompt window (row-major over the nh x nw grid of windows) of pixel pix of a gh x gw patch grid
__device__ __forceinline__ int chan_window(int pix, int gh, int gw, int nh, int nw) {
  const int py = pix / gw, px = pix % gw;
  return (py / (gh / nh)) * nw + px / (gw / nw);
}

// ---------------------------------------------------------------- split-bf16 stores
// An output in split-bf16 form: x ~= hi + lo (split_bf16). lo == nullptr writes the hi plane only.
struct SplitPlanes {
  __nv_bfloat16* hi;
  __nv_bfloat16* lo;
  long long ld;
};

// x -> element (row, col)
__device__ __forceinline__ void store_split(const SplitPlanes& p, long long row, long long col, float x) {
  __nv_bfloat16 h, l;
  split_bf16(x, h, l);
  p.hi[row * p.ld + col] = h;
  if (p.lo) p.lo[row * p.ld + col] = l;
}

// (x0, x1) -> elements (row, col), (row, col + 1): one bf16x2 store per plane when `vec` (the caller's test that the
// pair is whole and 4-byte aligned), otherwise two-byte stores of col and, when `two`, of col + 1 (two = false where
// `vec` fails only for a lone last element).
__device__ __forceinline__ void store_split2(const SplitPlanes& p, long long row, long long col, float x0, float x1,
                                             bool vec, bool two) {
  uint32_t h, l;
  split_pack2(x0, x1, h, l);
  const long long o = row * p.ld + col;
  if (vec) {
    *reinterpret_cast<uint32_t*>(p.hi + o) = h;
    if (p.lo) *reinterpret_cast<uint32_t*>(p.lo + o) = l;
  } else {
    p.hi[o] = __ushort_as_bfloat16((unsigned short)(h & 0xFFFF));
    if (p.lo) p.lo[o] = __ushort_as_bfloat16((unsigned short)(l & 0xFFFF));
    if (two) {
      p.hi[o + 1] = __ushort_as_bfloat16((unsigned short)(h >> 16));
      if (p.lo) p.lo[o + 1] = __ushort_as_bfloat16((unsigned short)(l >> 16));
    }
  }
}

}  // namespace mtt
