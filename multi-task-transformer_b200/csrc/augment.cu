// The reference's PASCAL-Context / NYUD train and validation transform chains (TP/utils/common_config.py:96-121,
// TP/data/transforms.py) over a ragged batch of raw samples, in three launches whatever the batch size and task count:
//   augment_select_kernel  one block per (sample, crop candidate): the cat_max_ratio test of RandomCrop (:195-205) as a
//                          shared-memory label histogram gathered through the nearest-neighbour map (no scaled copy is
//                          made), and whether the candidate's human_parts crop is all 0 / 255 (AddIgnoreRegions :291-295)
//   augment_image_kernel   RandomScaling's bilinear resize (:56-57), crop, flip (:224-230), PhotoMetricDistortion
//                          (:376-407), Normalize (:246-251), PadImage (:102-130), HWC -> CHW (:265-273)
//   augment_labels_kernel  every label map: nearest resize, depth / scale (:61-63), crop, flip (normals x negated), pad,
//                          AddIgnoreRegions (:279-299), CHW
// The image and label kernels pick the crop candidate from the select kernel's flags (the first of 0..9 that passes,
// else the 11th, as the reference's loop ends), so the choice never leaves the device.
//
// Bit-exactness: the float arithmetic follows the reference operation by operation with explicit rounding intrinsics
// (no FMA contraction except where cv2 itself fuses, no FTZ), and the cv2 rules are the ones oracle/augment_ref.py
// restates and tests/test_augment.py checks against cv2 itself.
#include "host_common.h"

namespace mtt {

constexpr int kSelThreads = 512;

struct Norm3f {
  float mean[3];
  float std[3];
};

struct AugTasks {
  int32_t n;
  int32_t kind[MTT_AUG_MAX_TASKS];
  float* out[MTT_AUG_MAX_TASKS];
};

__device__ __forceinline__ void linear_coord(int d, double step, int n, int& i0, int& i1, float& t) {
  // cv2 INTER_LINEAR (float32, as the IPP path computes it): coordinate in double, fraction rounded to float
  const double f = __dadd_rn(__dmul_rn((double)d + 0.5, step), -0.5);
  double fl = floor(f);
  int i = (int)fl;
  double fr = f - fl;
  if (i < 0) { i = 0; fr = 0.0; }
  if (i >= n - 1) { i = n - 1; fr = 0.0; }
  i0 = i;
  i1 = min(i + 1, n - 1);
  t = (float)fr;
}

__device__ __forceinline__ int nearest_src(int d, double f, int n) {
  return min((int)floor(__dmul_rn((double)d, f)), n - 1);   // cv2 INTER_NEAREST
}

// Scaled-map coordinate (sy, sx) -> raw coordinate of the nearest-neighbour map.
__device__ __forceinline__ void nn_src(const mtt_augment_sample& s, int sy, int sx, int& ry, int& rx) {
  const bool same = s.sh == s.h && s.sw == s.w;   // cv2.resize copies when the size does not change
  ry = same ? sy : nearest_src(sy, s.nn_y, s.h);
  rx = same ? sx : nearest_src(sx, s.nn_x, s.w);
}

__device__ __forceinline__ int chosen_candidate(const mtt_augment_sample& s, const int32_t* flags, int b) {
  if (s.ncand == 0) return -1;
  for (int k = 0; k < MTT_AUG_CANDIDATES - 1; ++k)
    if (flags[b * MTT_AUG_CANDIDATES + k] & 1) return k;
  return MTT_AUG_CANDIDATES - 1;
}

// Output pixel (y, x) -> scaled-map pixel, or false in the padding; col / width: the pixel's column in the cropped,
// flipped image and that image's width (PhotoMetricDistortion's rows).
__device__ __forceinline__ bool out_to_scaled(const mtt_augment_sample& s, int k, int CH, int CW, int H, int W, int y,
                                              int x, int& sy, int& sx, int& col, int& width) {
  int oy = 0, ox = 0, ch = s.sh, cw = s.sw;
  if (k >= 0) {
    oy = s.cand[k][0];
    ox = s.cand[k][1];
    ch = min(CH, s.sh - oy);   // numpy slicing truncates
    cw = min(CW, s.sw - ox);
  }
  const int py = y - (H - ch) / 2, px = x - (W - cw) / 2;   // PadImage centres at (dh // 2, dw // 2)
  if (py < 0 || py >= ch || px < 0 || px >= cw) return false;
  sy = oy + py;
  sx = ox + (s.flip ? cw - 1 - px : px);
  col = px;
  width = cw;
  return true;
}

__global__ void __launch_bounds__(kSelThreads)
augment_select_kernel(const mtt_augment_sample* __restrict__ smp, const float* __restrict__ data, int semseg_task,
                      int parts_task, int CH, int CW, int32_t* __restrict__ flags) {
  __shared__ int hist[256];
  const int b = blockIdx.x, k = blockIdx.y;
  const mtt_augment_sample& s = smp[b];
  if (s.ncand == 0 && k > 0) return;   // no crop: one block checks the whole map
  for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
  __syncthreads();
  int y0 = 0, x0 = 0, ch = s.sh, cw = s.sw;
  if (s.ncand > 0) {
    y0 = s.cand[k][0];
    x0 = s.cand[k][1];
    ch = min(CH, s.sh - y0);
    cw = min(CW, s.sw - x0);
  }
  const bool want_hist = semseg_task >= 0 && s.ncand > 0 && k < MTT_AUG_CANDIDATES - 1;
  const float* seg = want_hist ? data + s.off[1 + semseg_task] : nullptr;
  const float* parts = parts_task >= 0 ? data + s.off[1 + parts_task] : nullptr;
  int parts_ok = 1;
  const int n = ch * cw;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    int ry, rx;
    nn_src(s, y0 + i / cw, x0 + i % cw, ry, rx);
    const long long src = (long long)ry * s.w + rx;
    if (seg) {
      const float v = seg[src];
      if (v >= 0.f && v < 255.f) atomicAdd(&hist[(int)v], 1);   // labels are integers; 255 is excluded (:202)
    }
    if (parts) {
      const float v = parts[src];
      parts_ok &= (v == 0.f || v == 255.f);
    }
  }
  parts_ok = __syncthreads_and(parts_ok);
  int nlab = 0, mx = 0, sum = 0;
  if (want_hist) {
    for (int i = threadIdx.x; i < 255; i += blockDim.x) {
      const int c = hist[i];
      nlab += c > 0;
      mx = max(mx, c);
      sum += c;
    }
  }
  // block reductions of the histogram statistics: labels present, largest count, total
  __shared__ int red[3][kSelThreads / 32];
  if (want_hist) {
    for (int o = 16; o > 0; o >>= 1) {
      nlab += __shfl_xor_sync(0xffffffffu, nlab, o);
      mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      sum += __shfl_xor_sync(0xffffffffu, sum, o);
    }
    if ((threadIdx.x & 31) == 0) {
      red[0][threadIdx.x >> 5] = nlab;
      red[1][threadIdx.x >> 5] = mx;
      red[2][threadIdx.x >> 5] = sum;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int pass = 0;
    if (want_hist) {
      int L = 0, M = 0, S = 0;
      for (int w = 0; w < kSelThreads / 32; ++w) {
        L += red[0][w];
        M = max(M, red[1][w]);
        S += red[2][w];
      }
      pass = L > 1 && 4ll * M < 3ll * S;   // max / sum < 0.75, exactly (:203)
    }
    flags[b * MTT_AUG_CANDIDATES + k] = pass | (parts_ok << 1);
  }
}

// ---- cv2 uint8 colour conversions (COLOR_RGB2HSV / COLOR_HSV2RGB, H in 0..179) --------------------------------------
__device__ __forceinline__ int div_table(int num, int i) { return i == 0 ? 0 : __double2int_rn((double)num / (double)i); }

__device__ __forceinline__ void rgb2hsv(int r, int g, int b, int& h, int& s, int& v) {
  v = max(max(b, g), r);
  const int diff = v - min(min(b, g), r);
  s = (diff * div_table(255 << 12, v) + (1 << 11)) >> 12;
  int hh = v == r ? g - b : (v == g ? b - r + 2 * diff : r - g + 4 * diff);
  const int hdiv = diff == 0 ? 0 : __double2int_rn((double)(180 << 12) / (6.0 * diff));
  hh = (hh * hdiv + (1 << 11)) >> 12;
  h = hh < 0 ? hh + 180 : hh;
}

// cv2 truncates x * 255 in the vector loop over the first floor(width / 32) * 32 pixels of a row and rounds (half to
// even) in the scalar tail (oracle/augment_ref.py).
__device__ __forceinline__ int to_u8(float x, bool vec) {
  const float y = __fmul_rn(x, 255.f);
  return min(max(vec ? (int)y : __float2int_rn(y), 0), 255);
}

__device__ __forceinline__ void hsv2rgb(int H, int S, int V, bool vec, int& r, int& g, int& b) {
  const float inv255 = 1.0f / 255.0f;
  const float s = __fmul_rn((float)S, inv255), v = __fmul_rn((float)V, inv255);
  if (s == 0.f) {
    r = g = b = to_u8(v, vec);
    return;
  }
  float h = __fmul_rn((float)H, 6.0f / 180.0f);
  int sector = (int)floorf(h);
  h = __fsub_rn(h, (float)sector);
  if ((unsigned)sector >= 6u) {
    sector = 0;
    h = 0.f;
  }
  float tab[4];
  tab[0] = v;
  tab[1] = __fmul_rn(v, __fsub_rn(1.f, s));
  tab[2] = __fmul_rn(v, __fmaf_rn(-s, h, 1.f));
  tab[3] = __fmul_rn(v, __fmaf_rn(-s, __fsub_rn(1.f, h), 1.f));
  const int sec[6][3] = {{1, 3, 0}, {1, 0, 2}, {3, 0, 1}, {0, 2, 1}, {0, 1, 3}, {2, 1, 0}};   // (b, g, r)
  b = to_u8(tab[sec[sector][0]], vec);
  g = to_u8(tab[sec[sector][1]], vec);
  r = to_u8(tab[sec[sector][2]], vec);
}

// PhotoMetricDistortion.convert (:334-338): clip(float32(x) * alpha + beta, 0, 255) truncated to uint8
__device__ __forceinline__ int convert(int x, float alpha, float beta) {
  const float f = __fadd_rn(__fmul_rn((float)x, alpha), beta);
  return (int)fminf(fmaxf(f, 0.f), 255.f);
}

__device__ __forceinline__ void photometric(const mtt_augment_sample& s, bool vec, int c[3]) {
  if (s.bright_on)
    for (int i = 0; i < 3; ++i) c[i] = convert(c[i], 1.f, s.beta);
  if (s.f_mode && s.contrast_on)
    for (int i = 0; i < 3; ++i) c[i] = convert(c[i], s.alpha, 0.f);
  if (s.sat_on) {
    int h, sat, v;
    rgb2hsv(c[0], c[1], c[2], h, sat, v);
    hsv2rgb(h, convert(sat, s.sat_alpha, 0.f), v, vec, c[0], c[1], c[2]);
  }
  if (s.hue_on) {
    int h, sat, v;
    rgb2hsv(c[0], c[1], c[2], h, sat, v);
    hsv2rgb(((h + s.hue_delta) % 180 + 180) % 180, sat, v, vec, c[0], c[1], c[2]);
  }
  if (!s.f_mode && s.contrast_on)
    for (int i = 0; i < 3; ++i) c[i] = convert(c[i], s.alpha, 0.f);
}

__device__ __forceinline__ float normalize(float x, float m, float sd) {
  return __fdiv_rn(__fsub_rn(__fdiv_rn(x, 255.0f), m), sd);
}

__global__ void __launch_bounds__(256)
augment_image_kernel(const mtt_augment_sample* __restrict__ smp, const float* __restrict__ data,
                     const int32_t* __restrict__ flags, int B, int H, int W, int CH, int CW, int train, Norm3f nm,
                     float* __restrict__ out, int32_t* __restrict__ chosen) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)B * H * W) return;
  const int x = (int)(idx % W), y = (int)((idx / W) % H), b = (int)(idx / ((long long)W * H));
  const mtt_augment_sample& s = smp[b];
  const int k = train ? chosen_candidate(s, flags, b) : -1;
  if (x == 0 && y == 0) chosen[b] = k;
  float* o = out + (long long)b * 3 * H * W + (long long)y * W + x;
  const long long plane = (long long)H * W;
  int sy, sx, col, width;
  if (!out_to_scaled(s, k, CH, CW, H, W, y, x, sy, sx, col, width)) {
    o[0] = o[plane] = o[2 * plane] = 0.f;   // PadImage fills the (normalised) image with 0
    return;
  }
  const float* img = data + s.off[0];
  float v[3];
  if (s.sh == s.h && s.sw == s.w) {
    for (int c = 0; c < 3; ++c) v[c] = img[((long long)sy * s.w + sx) * 3 + c];
  } else {
    int y0, y1, x0, x1;
    float ty, tx;
    linear_coord(sy, s.lin_y, s.h, y0, y1, ty);
    linear_coord(sx, s.lin_x, s.w, x0, x1, tx);
    for (int c = 0; c < 3; ++c) {
      const float a0 = img[((long long)y0 * s.w + x0) * 3 + c], a1 = img[((long long)y0 * s.w + x1) * 3 + c];
      const float b0 = img[((long long)y1 * s.w + x0) * 3 + c], b1 = img[((long long)y1 * s.w + x1) * 3 + c];
      const float r0 = __fmaf_rn(__fsub_rn(a1, a0), tx, a0);
      const float r1 = __fmaf_rn(__fsub_rn(b1, b0), tx, b0);
      v[c] = __fmaf_rn(__fsub_rn(r1, r0), ty, r0);
    }
  }
  if (train) {
    int u[3];
    for (int c = 0; c < 3; ++c) u[c] = (int)v[c];   // astype(np.uint8) truncates (:385)
    photometric(s, col < width / 32 * 32, u);
    for (int c = 0; c < 3; ++c) v[c] = (float)u[c];
  }
  for (int c = 0; c < 3; ++c) o[c * plane] = normalize(v[c], nm.mean[c], nm.std[c]);
}

__device__ __forceinline__ float label_fill(int kind) {
  return (kind == MTT_AUG_NORMALS || kind == MTT_AUG_DEPTH) ? 0.f : 255.f;   // PadImage.fill_index (:94-100)
}

__global__ void __launch_bounds__(256)
augment_labels_kernel(const mtt_augment_sample* __restrict__ smp, const float* __restrict__ data,
                      const int32_t* __restrict__ flags, int B, int H, int W, int CH, int CW, int train, AugTasks tk) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)B * H * W) return;
  const int x = (int)(idx % W), y = (int)((idx / W) % H), b = (int)(idx / ((long long)W * H));
  const mtt_augment_sample& s = smp[b];
  const int k = train ? chosen_candidate(s, flags, b) : -1;
  const int fk = k < 0 ? 0 : k;
  const long long plane = (long long)H * W, pix = (long long)y * W + x;
  int sy = 0, sx = 0, ry = 0, rx = 0, col, width;
  const bool inside = out_to_scaled(s, k, CH, CW, H, W, y, x, sy, sx, col, width);
  if (inside) nn_src(s, sy, sx, ry, rx);
  const long long src = (long long)ry * s.w + rx;
  for (int t = 0; t < tk.n; ++t) {
    const int kind = tk.kind[t];
    const int C = kind == MTT_AUG_NORMALS ? 3 : 1;
    float* o = tk.out[t] + (long long)b * C * plane + pix;
    const float* in = data + s.off[1 + t];
    float v[3];
    for (int c = 0; c < C; ++c) v[c] = inside ? in[src * C + c] : label_fill(kind);
    if (inside && kind == MTT_AUG_DEPTH && s.scaled) v[0] = __fdiv_rn(v[0], s.depth_scale);
    if (inside && kind == MTT_AUG_NORMALS && s.flip) v[0] = -v[0];
    if (kind == MTT_AUG_NORMALS) {
      const float n2 = __fadd_rn(__fadd_rn(__fmul_rn(v[0], v[0]), __fmul_rn(v[1], v[1])), __fmul_rn(v[2], v[2]));
      if (__fsqrt_rn(n2) == 0.f) v[0] = v[1] = v[2] = 255.f;
    } else if (kind == MTT_AUG_HUMAN_PARTS) {
      if (flags[b * MTT_AUG_CANDIDATES + fk] & 2) v[0] = 255.f;
    } else if (kind == MTT_AUG_DEPTH) {
      if (v[0] == 0.f) v[0] = -1.f;
    }
    for (int c = 0; c < C; ++c) o[c * plane] = v[c];
  }
}

}  // namespace mtt

extern "C" size_t mtt_augment_workspace_bytes(int32_t B) {
  return B > 0 ? (size_t)B * (MTT_AUG_CANDIDATES + 1) * sizeof(int32_t) : 0;
}

extern "C" int mtt_augment(const mtt_augment_desc* d, mtt_stream_t stream) {
  using namespace mtt;
  if (!d || !d->samples || !d->data || !d->image_out || !d->workspace || d->B <= 0 || d->H <= 0 || d->W <= 0 ||
      d->ntasks < 0 || d->ntasks > MTT_AUG_MAX_TASKS || (d->train && (d->crop_h <= 0 || d->crop_w <= 0)))
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_augment: bad arguments (B=%d H=%d W=%d ntasks=%d crop=%dx%d)",
                     d ? d->B : 0, d ? d->H : 0, d ? d->W : 0, d ? d->ntasks : 0, d ? d->crop_h : 0,
                     d ? d->crop_w : 0);
  if (d->train && (d->H != d->crop_h || d->W != d->crop_w))
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_augment: train output %dx%d != crop %dx%d", d->H, d->W, d->crop_h,
                     d->crop_w);
  if (d->workspace_bytes < mtt_augment_workspace_bytes(d->B))
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_augment: workspace of %zu bytes < %zu", d->workspace_bytes,
                     mtt_augment_workspace_bytes(d->B));
  AugTasks tk;
  tk.n = d->ntasks;
  int semseg = -1, parts = -1;
  for (int t = 0; t < d->ntasks; ++t) {
    const int kind = d->task_kind[t];
    if (kind < MTT_AUG_SEMSEG || kind > MTT_AUG_DEPTH || !d->task_out[t])
      return set_error(MTT_ERR_BAD_SHAPE, "mtt_augment: task %d has kind %d / output %p", t, kind, d->task_out[t]);
    for (int u = 0; u < t; ++u)
      if (d->task_kind[u] == kind) return set_error(MTT_ERR_BAD_SHAPE, "mtt_augment: task kind %d given twice", kind);
    if (kind == MTT_AUG_SEMSEG) semseg = t;
    if (kind == MTT_AUG_HUMAN_PARTS) parts = t;
    tk.kind[t] = kind;
    tk.out[t] = d->task_out[t];
  }
  if (d->train && semseg < 0)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_augment: the train chain's RandomCrop needs a semseg task");
  Norm3f nm;
  for (int c = 0; c < 3; ++c) {
    nm.mean[c] = d->mean[c];
    nm.std[c] = d->std[c];
    if (!(d->std[c] > 0.f)) return set_error(MTT_ERR_BAD_SHAPE, "mtt_augment: std[%d] = %g", c, d->std[c]);
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int32_t* flags = static_cast<int32_t*>(d->workspace);
  int32_t* chosen = flags + (size_t)d->B * MTT_AUG_CANDIDATES;
  const mtt_augment_sample* smp = static_cast<const mtt_augment_sample*>(d->samples);
  if (d->train || parts >= 0) {
    // validation: ncand == 0 in every record, so one block per sample checks human_parts over the whole map
    augment_select_kernel<<<dim3(d->B, d->train ? MTT_AUG_CANDIDATES : 1), kSelThreads, 0, st>>>(
        smp, d->data, d->train ? semseg : -1, parts, d->crop_h, d->crop_w, flags);
    if (int rc = check_launch("mtt_augment(select)")) return rc;
  }
  const long long total = (long long)d->B * d->H * d->W;
  const unsigned grid = (unsigned)((total + 255) / 256);
  augment_image_kernel<<<grid, 256, 0, st>>>(smp, d->data, flags, d->B, d->H, d->W, d->crop_h, d->crop_w, d->train,
                                             nm, d->image_out, chosen);
  if (int rc = check_launch("mtt_augment(image)")) return rc;
  if (d->ntasks > 0) {
    augment_labels_kernel<<<grid, 256, 0, st>>>(smp, d->data, flags, d->B, d->H, d->W, d->crop_h, d->crop_w, d->train,
                                                tk);
    if (int rc = check_launch("mtt_augment(labels)")) return rc;
  }
  return 0;
}
