// Per-pixel pieces of the final resize and of the reference's get_output post-processing (TP/utils/utils.py:27-63),
// shared by mtt_bilinear_postproc (prompting.cu) and mtt_render (export.cu) so both compute the same bits.
#pragma once
#include <math.h>

namespace mtt {

// Bilinear resize, align_corners = False (ATen upsample_bilinear2d semantics; reference calls at
// taskprompter.py:420, taskprompter_wrapper.py:35): output coordinate d -> source rows / columns i0, i1 and the weight
// l1 of i1.
__device__ __forceinline__ void bilin_coord(int d, float scale, int in_size, int& i0, int& i1, float& l1) {
  float s = scale * (d + 0.5f) - 0.5f;
  if (s < 0.f) s = 0.f;
  i0 = (int)s;
  if (i0 > in_size - 1) i0 = in_size - 1;
  i1 = i0 + (i0 < in_size - 1 ? 1 : 0);
  l1 = s - (float)i0;
}

// get_output of one pixel from its C channel values val(c) (already resized), handed to the sink as
//   kind 0: argmax over channels -> out.cls(c)              (semseg, human_parts; first maximum wins, like torch.max)
//   kind 1: 255 * sigmoid(x)     -> out.f1(v)               (edge)
//   kind 2: 255 * softmax(x)[1]  -> out.f1(v)               (sal, 2 channels)
//   kind 3: (x/||x|| + 1)*255/2  -> out.ch(c, v), c = 0..2  (normals; F.normalize eps 1e-12)
//   kind 4: max(x, 0)            -> out.f1(v)               (depth)
template <class Val, class Sink>
__device__ __forceinline__ void get_output_pixel(int kind, int C, Val val, Sink& out) {
  if (kind == 0) {
    float best = val(0);
    int bi = 0;
    for (int c = 1; c < C; ++c) {
      const float v = val(c);
      if (v > best) {
        best = v;
        bi = c;
      }
    }
    out.cls(bi);
  } else if (kind == 1) {
    out.f1(255.f * (1.f / (1.f + expf(-val(0)))));
  } else if (kind == 2) {
    const float a = val(0), c1 = val(1);
    const float m = fmaxf(a, c1);
    const float e0 = expf(a - m), e1 = expf(c1 - m);
    out.f1(e1 / (e0 + e1) * 255.f);
  } else if (kind == 3) {
    const float a = val(0), c1 = val(1), c2 = val(2);
    const float n = fmaxf(sqrtf(a * a + c1 * c1 + c2 * c2), 1e-12f);
    out.ch(0, (a / n + 1.f) * 255.f / 2.f);
    out.ch(1, (c1 / n + 1.f) * 255.f / 2.f);
    out.ch(2, (c2 / n + 1.f) * 255.f / 2.f);
  } else {
    out.f1(fmaxf(val(0), 0.f));
  }
}

}  // namespace mtt
