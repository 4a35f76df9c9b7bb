// Predictions -> uint8 images (include/mtt_b200.h, mtt_render): the reference's prediction export
// (save_model_pred_for_one_task, TP/evaluation/evaluate_utils.py:69-151, IP/evaluation/evaluate_utils.py:69-105) and
// inference visualisation (vis_pred_for_one_task, TP/utils/visualization_utils.py:80-199), for every (task, image) pair
// of a call in two launches:
//   render_prepass_kernel  per (task, image): min / max of the JET depth over the crop, through the same resize and
//                          get_output arithmetic as the main pass, combined across blocks with 32-bit atomics on an
//                          order-preserving encoding (exact: min / max do not depend on order); and whether any label
//                          value differs from ignore_index (evaluate_utils.py:120 skip rule)
//   render_kernel          one thread per output pixel: source value (resize + get_output_pixel, or a get_output map),
//                          crop, encode (truncate / class id / palette / normals / JET), uint8 store
// Every value is computed independently of the launch geometry, so the output is bitwise reproducible.
#include "host_common.h"
#include "postproc.cuh"

namespace mtt {

constexpr int kRenderThreads = 256;
constexpr int kPrepassItems = 8;   // values per pre-pass thread

// cv2.applyColorMap(np.arange(256, dtype=np.uint8), cv2.COLORMAP_JET), BGR (cv2 data, generated with cv2 4.13)
static const uint8_t kJetBGR[256 * 3] = {
    128,0,0, 132,0,0, 136,0,0, 140,0,0, 144,0,0, 148,0,0, 152,0,0, 156,0,0,
    160,0,0, 164,0,0, 168,0,0, 172,0,0, 176,0,0, 180,0,0, 184,0,0, 188,0,0,
    192,0,0, 196,0,0, 200,0,0, 204,0,0, 208,0,0, 212,0,0, 216,0,0, 220,0,0,
    224,0,0, 228,0,0, 232,0,0, 236,0,0, 240,0,0, 244,0,0, 248,0,0, 252,0,0,
    255,0,0, 255,4,0, 255,8,0, 255,12,0, 255,16,0, 255,20,0, 255,24,0, 255,28,0,
    255,32,0, 255,36,0, 255,40,0, 255,44,0, 255,48,0, 255,52,0, 255,56,0, 255,60,0,
    255,64,0, 255,68,0, 255,72,0, 255,76,0, 255,80,0, 255,84,0, 255,88,0, 255,92,0,
    255,96,0, 255,100,0, 255,104,0, 255,108,0, 255,112,0, 255,116,0, 255,120,0, 255,124,0,
    255,128,0, 255,132,0, 255,136,0, 255,140,0, 255,144,0, 255,148,0, 255,152,0, 255,156,0,
    255,160,0, 255,164,0, 255,168,0, 255,172,0, 255,176,0, 255,180,0, 255,184,0, 255,188,0,
    255,192,0, 255,196,0, 255,200,0, 255,204,0, 255,208,0, 255,212,0, 255,216,0, 255,220,0,
    255,224,0, 255,228,0, 255,232,0, 255,236,0, 255,240,0, 255,244,0, 255,248,0, 255,252,0,
    254,255,2, 250,255,6, 246,255,10, 242,255,14, 238,255,18, 234,255,22, 230,255,26, 226,255,30,
    222,255,34, 218,255,38, 214,255,42, 210,255,46, 206,255,50, 202,255,54, 198,255,58, 194,255,62,
    190,255,66, 186,255,70, 182,255,74, 178,255,78, 174,255,82, 170,255,86, 166,255,90, 162,255,94,
    158,255,98, 154,255,102, 150,255,106, 146,255,110, 142,255,114, 138,255,118, 134,255,122, 130,255,126,
    126,255,130, 122,255,134, 118,255,138, 114,255,142, 110,255,146, 106,255,150, 102,255,154, 98,255,158,
    94,255,162, 90,255,166, 86,255,170, 82,255,174, 78,255,178, 74,255,182, 70,255,186, 66,255,190,
    62,255,194, 58,255,198, 54,255,202, 50,255,206, 46,255,210, 42,255,214, 38,255,218, 34,255,222,
    30,255,226, 26,255,230, 22,255,234, 18,255,238, 14,255,242, 10,255,246, 6,255,250, 1,255,254,
    0,252,255, 0,248,255, 0,244,255, 0,240,255, 0,236,255, 0,232,255, 0,228,255, 0,224,255,
    0,220,255, 0,216,255, 0,212,255, 0,208,255, 0,204,255, 0,200,255, 0,196,255, 0,192,255,
    0,188,255, 0,184,255, 0,180,255, 0,176,255, 0,172,255, 0,168,255, 0,164,255, 0,160,255,
    0,156,255, 0,152,255, 0,148,255, 0,144,255, 0,140,255, 0,136,255, 0,132,255, 0,128,255,
    0,124,255, 0,120,255, 0,116,255, 0,112,255, 0,108,255, 0,104,255, 0,100,255, 0,96,255,
    0,92,255, 0,88,255, 0,84,255, 0,80,255, 0,76,255, 0,72,255, 0,68,255, 0,64,255,
    0,60,255, 0,56,255, 0,52,255, 0,48,255, 0,44,255, 0,40,255, 0,36,255, 0,32,255,
    0,28,255, 0,24,255, 0,20,255, 0,16,255, 0,12,255, 0,8,255, 0,4,255, 0,0,255,
    0,0,252, 0,0,248, 0,0,244, 0,0,240, 0,0,236, 0,0,232, 0,0,228, 0,0,224,
    0,0,220, 0,0,216, 0,0,212, 0,0,208, 0,0,204, 0,0,200, 0,0,196, 0,0,192,
    0,0,188, 0,0,184, 0,0,180, 0,0,176, 0,0,172, 0,0,168, 0,0,164, 0,0,160,
    0,0,156, 0,0,152, 0,0,148, 0,0,144, 0,0,140, 0,0,136, 0,0,132, 0,0,128,};

struct RenderTask {
  const void* src;
  int32_t src_kind, C, h, w, post, enc, table_len, first;   // first: index of the task's first record
  const uint8_t* table;
  uint8_t* out;
  const float* label;
  long long label_numel;
  float ignore;
  int32_t* flags;
};

struct RenderRec {
  int32_t y0, x0, h, w;   // crop
  int32_t oh, ow;         // size of the map the crop is taken from (the resize target of LOGITS)
  long long off;
};

struct RenderParams {
  int32_t ntasks, nrec;
  RenderTask t[MTT_RENDER_MAX_TASKS];
  RenderRec r[MTT_RENDER_MAX_IMAGES];
};
static_assert(sizeof(RenderParams) <= 4000, "mtt_render: kernel parameters must fit the 4 KB limit");

__device__ __forceinline__ int rec_task(const RenderParams& p, int rec) {
  int t = 0;
  while (t + 1 < p.ntasks && p.t[t + 1].first <= rec) ++t;
  return t;
}

// Order-preserving float <-> uint32 encoding: a < b  <=>  enc(a) < enc(b) (NaN-free values).
__device__ __forceinline__ uint32_t enc_f(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float dec_f(uint32_t e) {
  return __uint_as_float((e & 0x80000000u) ? (e & 0x7fffffffu) : ~e);
}

// numpy's float32 -> uint8 cast on x86-64 (cvttss2si, then the low byte): NaN and |v| >= 2^31 give INT32_MIN -> 0.
__device__ __forceinline__ uint32_t np_u8(float v) {
  const int i = (v > -2147483648.f && v < 2147483648.f) ? (int)v : (int)0x80000000;
  return (uint32_t)i & 0xffu;
}

struct PixelValue {
  int cls;
  float f[3];
};

// get_output_pixel's sink
struct ValueSink {
  PixelValue* v;
  __device__ void cls(int c) { v->cls = c; }
  __device__ void f1(float x) { v->f[0] = x; }
  __device__ void ch(int c, float x) { v->f[c] = x; }
};

// The get_output-domain value at (y, x) of the out_h x out_w map of image b.
__device__ __forceinline__ PixelValue source_value(const RenderTask& t, const RenderRec& r, int b, int y, int x) {
  PixelValue v;
  v.cls = 0;
  v.f[0] = v.f[1] = v.f[2] = 0.f;
  if (t.src_kind == MTT_RENDER_SRC_LOGITS) {
    // F.interpolate(bilinear, align_corners=False) on NCHW, in mtt_bilinear_postproc's arithmetic
    int y0, y1, x0, x1;
    float ly, lx;
    bilin_coord(y, (float)t.h / (float)r.oh, t.h, y0, y1, ly);
    bilin_coord(x, (float)t.w / (float)r.ow, t.w, x0, x1, lx);
    const long long plane = (long long)t.h * t.w;
    const float* ib = static_cast<const float*>(t.src) + (long long)b * t.C * plane;
    const float* p00 = ib + (long long)y0 * t.w + x0;
    const float* p01 = ib + (long long)y0 * t.w + x1;
    const float* p10 = ib + (long long)y1 * t.w + x0;
    const float* p11 = ib + (long long)y1 * t.w + x1;
    const float hy = 1.f - ly, hx = 1.f - lx;
    auto val = [&](int c) {
      const long long o = c * plane;
      return hy * (hx * p00[o] + lx * p01[o]) + ly * (hx * p10[o] + lx * p11[o]);
    };
    ValueSink sink{&v};
    get_output_pixel(t.post, t.C, val, sink);
  } else if (t.src_kind == MTT_RENDER_SRC_CLASS) {
    v.cls = (int)static_cast<const long long*>(t.src)[((long long)b * t.h + y) * t.w + x];
  } else {
    const float* s = static_cast<const float*>(t.src) + (((long long)b * t.h + y) * t.w + x) * t.C;
    for (int c = 0; c < t.C && c < 3; ++c) v.f[c] = s[c];
  }
  return v;
}

__device__ __forceinline__ bool class_source(const RenderTask& t) {
  return t.src_kind == MTT_RENDER_SRC_CLASS || (t.src_kind == MTT_RENDER_SRC_LOGITS && t.post == 0);
}

__global__ void __launch_bounds__(kRenderThreads)
render_prepass_kernel(const __grid_constant__ RenderParams p, uint32_t* __restrict__ ws) {
  const int rec = blockIdx.y;
  const RenderTask& t = p.t[rec_task(p, rec)];
  const RenderRec& r = p.r[rec];
  const int b = rec - t.first;
  const long long base = (long long)blockIdx.x * kRenderThreads * kPrepassItems;
  __shared__ uint32_t red[3];
  if (threadIdx.x < 3) red[threadIdx.x] = 0u;
  __syncthreads();
  if (t.enc == MTT_RENDER_JET) {
    const long long n = (long long)r.h * r.w;
    uint32_t nmn = 0u, mx = 0u;   // ~enc(min), enc(max); 0 = empty for both
    for (int k = 0; k < kPrepassItems; ++k) {
      const long long i = base + (long long)k * kRenderThreads + threadIdx.x;
      if (i >= n) break;
      const PixelValue v = source_value(t, r, b, r.y0 + (int)(i / r.w), r.x0 + (int)(i % r.w));
      const uint32_t e = enc_f(v.f[0]);
      nmn = max(nmn, ~e);
      mx = max(mx, e);
    }
    for (int o = 16; o > 0; o >>= 1) {
      nmn = max(nmn, __shfl_xor_sync(0xffffffffu, nmn, o));
      mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    if ((threadIdx.x & 31) == 0) {
      atomicMax(&red[0], nmn);
      atomicMax(&red[1], mx);
    }
  }
  if (t.label) {
    const float* lab = t.label + (long long)b * t.label_numel;
    uint32_t any = 0u;
    for (int k = 0; k < kPrepassItems; ++k) {
      const long long i = base + (long long)k * kRenderThreads + threadIdx.x;
      if (i >= t.label_numel) break;
      any |= lab[i] != t.ignore;
    }
    any = __any_sync(0xffffffffu, any) ? 1u : 0u;
    if ((threadIdx.x & 31) == 0 && any) atomicOr(&red[2], 1u);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t* w = ws + (size_t)rec * 3;
    if (red[0]) atomicMax(&w[0], red[0]);
    if (red[1]) atomicMax(&w[1], red[1]);
    if (red[2]) atomicOr(&w[2], 1u);
  }
}

__global__ void __launch_bounds__(kRenderThreads)
render_kernel(const __grid_constant__ RenderParams p, const uint32_t* __restrict__ ws) {
  const int rec = blockIdx.y;
  const RenderTask& t = p.t[rec_task(p, rec)];
  const RenderRec& r = p.r[rec];
  const int b = rec - t.first;
  const long long i = (long long)blockIdx.x * kRenderThreads + threadIdx.x;
  if (i == 0 && t.flags) t.flags[b] = (t.label && t.label_numel > 0 && ws[(size_t)rec * 3 + 2] == 0u) ? 1 : 0;
  if (i >= (long long)r.h * r.w) return;
  const int y = (int)(i / r.w), x = (int)(i % r.w);
  const PixelValue v = source_value(t, r, b, r.y0 + y, r.x0 + x);
  uint8_t* o = t.out + r.off;
  if (t.enc == MTT_RENDER_U8) {
    o[i] = (uint8_t)(class_source(t) ? ((uint32_t)v.cls & 0xffu) : np_u8(v.f[0]));
  } else if (t.enc == MTT_RENDER_CLASS) {
    int c = v.cls;
    if (t.table && c >= 0 && c < 256) c = t.table[c];   // get_cityscapes_class (TP/utils/utils.py:17-24)
    o[i] = (uint8_t)((uint32_t)c & 0xffu);
  } else if (t.enc == MTT_RENDER_PALETTE_BGR) {
    const int c = v.cls;
    const bool ok = c >= 0 && c < t.table_len;
    o[i * 3 + 0] = ok ? t.table[c * 3 + 2] : 0;
    o[i * 3 + 1] = ok ? t.table[c * 3 + 1] : 0;
    o[i * 3 + 2] = ok ? t.table[c * 3 + 0] : 0;
  } else if (t.enc == MTT_RENDER_NORMALS_BGR) {
    o[i * 3 + 0] = (uint8_t)np_u8(v.f[2]);
    o[i * 3 + 1] = (uint8_t)np_u8(v.f[1]);
    o[i * 3 + 2] = (uint8_t)np_u8(v.f[0]);
  } else {
    // visualization_utils.py:175-177 in numpy's float32: (arr - arr.min()) / (arr.max() - arr.min()) * 255
    const float mn = dec_f(~ws[(size_t)rec * 3 + 0]), mx = dec_f(ws[(size_t)rec * 3 + 1]);
    const uint32_t k = np_u8(__fmul_rn(__fdiv_rn(__fsub_rn(v.f[0], mn), __fsub_rn(mx, mn)), 255.f));
    o[i * 3 + 0] = t.table[k * 3 + 0];
    o[i * 3 + 1] = t.table[k * 3 + 1];
    o[i * 3 + 2] = t.table[k * 3 + 2];
  }
}

}  // namespace mtt

extern "C" const uint8_t* mtt_render_jet_bgr(void) { return mtt::kJetBGR; }

extern "C" size_t mtt_render_workspace_bytes(int32_t n_tasks, int32_t B) {
  return (n_tasks > 0 && B > 0) ? (size_t)n_tasks * B * 3 * sizeof(uint32_t) : 0;
}

extern "C" int mtt_render(const mtt_render_desc* d, int32_t n, void* workspace, mtt_stream_t stream) {
  using namespace mtt;
  if (!d || n <= 0 || n > MTT_RENDER_MAX_TASKS || !workspace)
    return set_error(MTT_ERR_BAD_SHAPE, "mtt_render: bad arguments (n=%d, workspace %p)", n, workspace);
  if (reinterpret_cast<uintptr_t>(workspace) % 4)
    return set_error(MTT_ERR_MISALIGNED, "mtt_render: workspace must be 4-byte aligned");
  RenderParams p;   // built on the host, passed by value
  p.ntasks = n;
  p.nrec = 0;
  bool prepass = false;
  long long max_pix = 0, max_pre = 0;
  const int need_c[5] = {1, 1, 2, 3, 1};
  for (int k = 0; k < n; ++k) {
    const mtt_render_desc& s = d[k];
    RenderTask& t = p.t[k];
    if (s.src_kind < MTT_RENDER_SRC_LOGITS || s.src_kind > MTT_RENDER_SRC_MAP || s.encode < MTT_RENDER_U8 ||
        s.encode > MTT_RENDER_JET)
      return set_error(MTT_ERR_BAD_SHAPE, "mtt_render: task %d has source kind %d / encoding %d", k, s.src_kind,
                       s.encode);
    if (!s.src || !s.out || !s.crop || !s.offset || s.B <= 0 || s.C <= 0 || s.h <= 0 || s.w <= 0 || s.out_h <= 0 ||
        s.out_w <= 0 || s.out_bytes < 0)
      return set_error(MTT_ERR_BAD_SHAPE, "mtt_render: task %d: bad geometry or null pointer (B=%d C=%d %dx%d -> %dx%d)",
                       k, s.B, s.C, s.h, s.w, s.out_h, s.out_w);
    const bool logits = s.src_kind == MTT_RENDER_SRC_LOGITS;
    if (logits && (s.postproc < 0 || s.postproc > 4 || s.C < need_c[s.postproc]))
      return set_error(MTT_ERR_BAD_SHAPE, "mtt_render: task %d: get_output kind %d cannot take %d channels", k,
                       s.postproc, s.C);
    if (!logits && (s.out_h != s.h || s.out_w != s.w))
      return set_error(MTT_ERR_BAD_SHAPE, "mtt_render: task %d: a get_output map is not resized (%dx%d -> %dx%d)", k,
                       s.h, s.w, s.out_h, s.out_w);
    if (s.src_kind == MTT_RENDER_SRC_MAP && s.C != 1 && s.C != 3)
      return set_error(MTT_ERR_BAD_SHAPE, "mtt_render: task %d: a float map has 1 or 3 channels, not %d", k, s.C);
    const bool cls = s.src_kind == MTT_RENDER_SRC_CLASS || (logits && s.postproc == 0);
    const bool three = (logits && s.postproc == 3) || (s.src_kind == MTT_RENDER_SRC_MAP && s.C == 3);
    bool ok = true;
    int ch = 1;
    switch (s.encode) {
      case MTT_RENDER_U8: ok = !three; break;
      case MTT_RENDER_CLASS: ok = cls && (!s.table || s.table_len >= 256); break;
      case MTT_RENDER_PALETTE_BGR: ok = cls && s.table && s.table_len >= s.C; ch = 3; break;
      case MTT_RENDER_NORMALS_BGR: ok = three; ch = 3; break;
      default: ok = !cls && !three && s.table && s.table_len >= 256; ch = 3; break;
    }
    if (!ok)
      return set_error(MTT_ERR_BAD_SHAPE,
                       "mtt_render: task %d: encoding %d cannot take this source (kind %d, get_output %d, C=%d) or "
                       "its table (%d entries)", k, s.encode, s.src_kind, s.postproc, s.C, s.table_len);
    if (s.label && (!s.flags || s.label_numel < 0))
      return set_error(MTT_ERR_BAD_SHAPE, "mtt_render: task %d: a label needs a flags output", k);
    if (p.nrec + s.B > MTT_RENDER_MAX_IMAGES)
      return set_error(MTT_ERR_BAD_SHAPE, "mtt_render: more than %d (task, image) pairs", MTT_RENDER_MAX_IMAGES);
    t.src = s.src;
    t.src_kind = s.src_kind;
    t.C = s.C;
    t.h = s.h;
    t.w = s.w;
    t.post = logits ? s.postproc : -1;
    t.enc = s.encode;
    t.table = s.table;
    t.table_len = s.table ? s.table_len : 0;
    t.first = p.nrec;
    t.out = s.out;
    t.label = s.label;
    t.label_numel = s.label ? s.label_numel : 0;
    t.ignore = s.ignore_index;
    t.flags = s.flags;
    if (s.out_size && !logits)
      return set_error(MTT_ERR_BAD_SHAPE, "mtt_render: task %d: per-image sizes need a LOGITS source", k);
    for (int b = 0; b < s.B; ++b) {
      const int32_t* c = s.crop + 4 * b;
      const int oh = s.out_size ? s.out_size[2 * b] : s.out_h, ow = s.out_size ? s.out_size[2 * b + 1] : s.out_w;
      if (oh <= 0 || ow <= 0 || c[0] < 0 || c[1] < 0 || c[2] <= 0 || c[3] <= 0 || c[0] + c[2] > oh || c[1] + c[3] > ow)
        return set_error(MTT_ERR_BAD_SHAPE, "mtt_render: task %d image %d: crop (%d, %d, %d, %d) outside the %dx%d map",
                         k, b, c[0], c[1], c[2], c[3], oh, ow);
      const long long bytes = (long long)c[2] * c[3] * ch;
      if (s.offset[b] < 0 || s.offset[b] + bytes > s.out_bytes)
        return set_error(MTT_ERR_BAD_SHAPE, "mtt_render: task %d image %d: %lld bytes at offset %lld exceed %lld", k,
                         b, bytes, (long long)s.offset[b], (long long)s.out_bytes);
      RenderRec& r = p.r[p.nrec++];
      r.y0 = c[0];
      r.x0 = c[1];
      r.h = c[2];
      r.w = c[3];
      r.oh = oh;
      r.ow = ow;
      r.off = s.offset[b];
      max_pix = max(max_pix, (long long)c[2] * c[3]);
      if (s.encode == MTT_RENDER_JET) max_pre = max(max_pre, (long long)c[2] * c[3]);
      if (s.label) max_pre = max(max_pre, (long long)s.label_numel);
    }
    prepass = prepass || s.encode == MTT_RENDER_JET || s.label;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint32_t* ws = static_cast<uint32_t*>(workspace);
  if (prepass) {
    if (cudaMemsetAsync(ws, 0, (size_t)p.nrec * 3 * sizeof(uint32_t), st) != cudaSuccess)
      return set_error(MTT_ERR_LAUNCH, "mtt_render: workspace memset failed");
    if (max_pre > 0) {
      const long long per = (long long)kRenderThreads * kPrepassItems;
      render_prepass_kernel<<<dim3((unsigned)((max_pre + per - 1) / per), p.nrec), kRenderThreads, 0, st>>>(p, ws);
      if (int rc = check_launch("mtt_render(prepass)")) return rc;
    }
  }
  render_kernel<<<dim3((unsigned)((max_pix + kRenderThreads - 1) / kRenderThreads), p.nrec), kRenderThreads, 0, st>>>(
      p, ws);
  return check_launch("mtt_render");
}
