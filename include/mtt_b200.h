/*
 * mtt_b200.h -- C ABI of libmtt_sm90.so: the sm_90a kernels behind the TaskPrompter / InvPT
 * forward hot path (reference: prismformore/Multi-Task-Transformer).
 *
 * The reference has no FFI of its own: its hot path is PyTorch eager ops called from nn.Module
 * forwards. Each entry point below replaces the eager-op sequence named in its comment
 * (file:line relative to the reference root; TP = TaskPrompter/, IP = InvPT/). The Python host
 * (multi-task-transformer_b200/) binds these with ctypes; INTEGRATION.md shows the binding a
 * reference maintainer would add.
 *
 * Conventions
 *  - Plain C: pointers are DEVICE pointers owned by the caller; the library never allocates,
 *    frees or synchronises; every call only enqueues work on `stream` (a cudaStream_t).
 *  - Return value: 0 = OK, negative = mtt_status; text via mtt_last_error() (thread local).
 *  - "split" tensors: an fp32 value x is carried as two bf16 planes, hi = bf16(x) and
 *    lo = bf16(x - hi), with identical layout. nsplit = 2 uses both planes (3 tensor-core MMAs per
 *    product: hi*hi + hi*lo + lo*hi, ~2^-17 relative error, the parity mode); nsplit = 1 uses only
 *    the hi plane (plain bf16, the speed mode). lo pointers may be NULL when nsplit = 1; an output lo
 *    plane that is given anyway (mtt_gemm, mtt_attention) is written as bf16(x - hi) in either mode.
 *  - All leading dimensions are in ELEMENTS.
 */
#ifndef MTT_B200_H_
#define MTT_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* mtt_stream_t; /* cudaStream_t */

enum mtt_status {
  MTT_OK = 0,
  MTT_ERR_BAD_SHAPE = -1,
  MTT_ERR_UNSUPPORTED_ARCH = -2,
  MTT_ERR_MISALIGNED = -3,
  MTT_ERR_LAUNCH = -4,
  MTT_ERR_DRIVER = -5
};

enum mtt_act { MTT_ACT_NONE = 0, MTT_ACT_GELU = 1, MTT_ACT_RELU = 2 };

/* ---- library ---------------------------------------------------------------------------- */
int mtt_version(void);
const char* mtt_last_error(void);
/* 0 iff the current device is compute capability 9.0 (H100); the kernels are sm_90a only. */
int mtt_device_check(void);
/* number of kernel launches issued by this library on the calling thread since the last reset */
int64_t mtt_launch_count(void);
void mtt_launch_count_reset(void);

/* Per-launch timing of the tensor-core kernels (bench.py's roofline block): between begin and end every mtt_gemm
 * (kind 0) and mtt_attention (kind 1) launch -- including those issued inside the composite operators -- is bracketed
 * by CUDA events on its stream and recorded with its algorithmic FLOPs (2*M*N*K*taps; attention 4*B*H*N*N*64).
 * mtt_profile_end synchronises the device, fills up to max_recs records and returns the total count in *n_recs.
 * Not usable during stream capture. */
typedef struct {
  int32_t kind, M, N, K;
  float ms;
  double flops;
} mtt_profile_rec;
int mtt_profile_begin(void);
int mtt_profile_end(mtt_profile_rec* out, int32_t max_recs, int32_t* n_recs);

/* ---- fp32 -> split bf16 planes ------------------------------------------------------------
 * Used for weight pre-packing and for inputs produced outside the library.
 * rows x cols fp32 (ld_in) -> hi/lo bf16 (ld_out); columns [cols, cols_pad) are written as zero. */
int mtt_split_f32(const float* in, int64_t ld_in, void* out_hi, void* out_lo, int64_t ld_out,
                  int64_t rows, int32_t cols, int32_t cols_pad, mtt_stream_t stream);

/* ---- LayerNorm over the last dim ---------------------------------------------------------
 * Replaces nn.LayerNorm calls: TP/models/transformers/taskprompter.py:272,274,277,413;
 * IP/models/transformers/vit.py:212-213,349; IP/models/transformers/invpt.py:298,307,526.
 * in [rows, cols] fp32 -> out_f32 (optional) and/or split bf16 (optional). */
int mtt_layernorm(const float* in, int64_t ld_in, const float* gamma, const float* beta, float eps,
                  float* out_f32, int64_t ld_f32, void* out_hi, void* out_lo, int64_t ld_bf,
                  int64_t rows, int32_t cols, mtt_stream_t stream);

/* ---- GEMM / implicit-GEMM convolution on wgmma -----------------------------------------
 * D[m, n] = act( sum_k A[m, k] * Bw[n, k] + bias[n] ) + residual[m, n]
 * mode 0 (linear): A is [M, lda] row-major. Replaces nn.Linear / 1x1 Conv2d:
 *   TP taskprompter.py:201 (qkv), :212 (proj), timm Mlp fc1/fc2 (:274,:277), :447,:468 (1x1
 *   decode convs), :362 (fea_fuse 1x1), :695 (linear_pred); IP vit.py:186,192, invpt.py:200-202.
 * mode 1 (conv): A is an NHWC activation [B, H, W, lda]; ksize x ksize taps, stride 1, dilation
 *   dil, zero padding dil*(ksize-1)/2. Bw is [N, ksize*ksize*cin_pad] with cin_pad = K rounded up
 *   to 64 (tap-major, zero padded). M = B*H*W. Replaces nn.Conv2d 3x3 (+ folded eval BatchNorm):
 *   TP taskprompter.py:362 (fea_fuse 3x3), :691 (ConvHead.mt_proj); IP transformer_decoder.py:113,
 *   invpt.py:33-38 (dilated), :493 (mt_proj).
 * Output rows can be regrouped: r_out = (r / in_group) * out_group + out_offset + r % in_group
 * (in_group = 0: identity); used to scatter patch rows into the joint [prompts; patches] stream. */
typedef struct {
  const void* a_hi;
  const void* a_lo;
  int64_t lda;
  const void* b_hi;
  const void* b_lo;
  int64_t ldb;
  int32_t M, N, K;
  int32_t nsplit;
  int32_t mode;
  int32_t B, H, W, ksize, dil;
  const float* bias;
  int32_t act;
  const float* residual;
  int64_t ldr;
  int32_t res_row_mod; /* >0: residual row = r % res_row_mod (row-broadcast, e.g. pos_embed) */
  float* out_f32;
  int64_t ldo_f32;
  void* out_hi;
  void* out_lo;
  int64_t ldo_bf;
  int32_t in_group, out_group, out_offset;
  /* mode 0 only. a_group_rows > 0: A's logical row r = (g, i) lives at physical row
   * g * a_group_stride + i (i < a_group_rows <= 128, a_group_rows | M): gathers e.g. the T prompt rows
   * of every image out of the joint [B*N, C] stream for token_trans (TP taskprompter.py:219). */
  int32_t a_group_rows;
  int64_t a_group_stride;
  /* >1: the in-group row index is multiplied by this stride, r_out = (r / in_group) * out_group + out_offset +
   * (r % in_group) * out_row_stride -- with in_group = W, out_group = 4W, stride 2, offset 2W*dy + dx the rows of an
   * [B,H,W] map land on the (dy,dx) phase of the [B,2H,2W] map: ConvTranspose2d(k2,s2) as four GEMMs
   * (TP taskprompter.py:704, DEConvHead). 0 / 1 = dense. */
  int32_t out_row_stride;
  /* Optional stream-K workspace (NULL = off), mtt_gemm_streamk_bytes() bytes, 256-byte aligned, zero-filled ONCE before
   * its first use (every launch leaves its flag words zero again) and not shared by launches that may run
   * concurrently. With it, a problem that mtt_gemm puts on the 128x256-tile kernel may split the tiles of its ragged
   * last round along K over all SMs instead of leaving most of them idle (policy: mtt_set_gemm_streamk; e.g. fc2
   * at batch 1: 36 tiles of 64 k-blocks on 132 SMs, or the weight-gradient GEMM of proj in the training step);
   * the partial sums are added in a fixed order, so results are reproducible. */
  void* sk_ws;
  int64_t sk_ws_bytes;
} mtt_gemm_desc;

int mtt_gemm(const mtt_gemm_desc* d, mtt_stream_t stream);
/* `count` (<= 32) problems that differ ONLY in their pointers (operands, bias, residual, outputs) as one persistent
 * launch: the T per-task 1x1 / 3x3 convs of a decoder level (TP taskprompter.py:447,:468,:362 for every task) are 96
 * tiles each -- less than one wave of 132 SMs -- and run as T x 96 tiles here. Same function as `count` mtt_gemm calls. */
int mtt_gemm_grouped(const mtt_gemm_desc* d, int32_t count, mtt_stream_t stream);
/* out[m, n] = bias[n] + sum_s partial[s][m, n] (fixed order: bitwise reproducible): the reduction step of a split-K GEMM
 * whose K chunks ran as the problems of one mtt_gemm_grouped launch (skinny M with a very long K: the Swin TaskPrompter's
 * chan_kv, Linear(H*W -> 2*ce) over 128 .. 1024 channel rows, TP taskprompter_swin.py:379). partial fp32 [S, M, ld]. */
int mtt_sum_partials(const float* partial, int32_t S, int64_t M, int32_t N, int64_t ld, const float* bias, float* out,
                     int64_t ldo, mtt_stream_t stream);
/* Kernel variant used by mtt_gemm: 0 = automatic (default; also env MTT_GEMM_VARIANT), 1 = 128x128
 * tiles, 2 = 128x256 tiles (the kernel with the stream-K schedule), 3 = 128x128 tiles (accepted for older settings).
 * All variants compute the same function; this is a tuning / testing knob. */
void mtt_set_gemm_variant(int variant);
/* Bytes of the stream-K workspace mtt_gemm_desc.sk_ws needs on the current device (flags + one fp32 128x256 partial
 * tile per SM, ~17 MB on an H100 with 132 SMs); mtt_workspace_bytes already includes it for the operators that use it. */
size_t mtt_gemm_streamk_bytes(void);
/* Stream-K policy (also env MTT_GEMM_STREAMK): 0 = off (sk_ws is ignored), 1 = automatic (default: problems of a
 * single partial round -- fewer tiles than SMs, >= 1/2 of the SMs idle, >= 32 k-blocks deep -- where the split
 * pays for its partial sums), 2 = whenever the split is legal. Tuning / testing knob: all settings compute the same
 * function. */
void mtt_set_gemm_streamk(int mode);
/* Test hook (no GPU needed): the work list of unit `pair` of `pairs` (one CTA per unit, one CTA per SM) for a problem
 * of `tiles` 128x256 tiles that are `k_iters` k-blocks deep, computed by the code the kernel runs. pieces receives up to
 * max_pieces triples (tile, first k-block, end k-block); returns the number of pieces of that unit. A piece that does
 * not start at k-block 0 is a stream-K contribution to the unit that holds the tile's first k-block. */
int mtt_debug_streamk_schedule(int32_t tiles, int32_t k_iters, int32_t pairs, int32_t pair, int32_t* pieces,
                               int32_t max_pieces);

/* ---- fused multi-head attention over the joint [prompts; patches] sequence ----------------
 * Replaces TP taskprompter.py:204-210 (raw = q k^T, softmax(raw*scale), attn @ v) and IP
 * vit.py:189-193, without materialising the [B,H,N,N] maps. qkv is the split output of the qkv
 * GEMM, [B*N, 3*H*64] with column order (q|k|v, head, 64) exactly as taskprompter.py:201 reshapes
 * it. out is [B*N, H*64] split. If prompt_logits != NULL the raw, UN-scaled logits of query rows
 * [0, T) are written as fp32 [B, H, T, N] (the only part of `raw_spa_attn` the reference consumes:
 * taskprompter.py:436-437, :482). head_dim must be 64. */
typedef struct {
  const void* qkv_hi;
  const void* qkv_lo;
  void* out_hi;
  void* out_lo;
  float* prompt_logits;
  int32_t B, N, H, T;
  int32_t nsplit;
  float scale;
} mtt_attn_desc;

int mtt_attention(const mtt_attn_desc* d, mtt_stream_t stream);
/* Kept for callers of earlier versions: there is one attention kernel (a TMA warp and two wgmma consumer warpgroups,
 * S and O in registers), so every value selects it. */
void mtt_set_attention_variant(int variant);
/* Kept for callers of earlier versions: the attention kernel records no clock trace, so the buffer is never written. */
void mtt_set_attention_trace(void* device_buf);

/* ---- patch embedding im2col ---------------------------------------------------------------
 * timm PatchEmbed (Conv2d k = s = patch) as a GEMM: img NCHW fp32 -> split [B*P, Cin*patch*patch],
 * column order (c, ky, kx) = conv.weight.reshape(C_out, -1). Replaces TP taskprompter.py:393,
 * IP vit.py:333. */
int mtt_im2col_patch(const float* img, int32_t B, int32_t Cin, int32_t H, int32_t W, int32_t patch,
                     void* out_hi, void* out_lo, int64_t ld_out, mtt_stream_t stream);

/* dst[(b*group_rows + t)*ld + c] = src[t*C + c]: task prompts / cls token into the joint stream
 * (TP taskprompter.py:397, IP vit.py:334-336). */
int mtt_broadcast_rows(const float* src, float* dst, int32_t B, int32_t T, int32_t C,
                       int64_t group_rows, int64_t ld, mtt_stream_t stream);

/* Raw channel logits Rc[b,t,c,i,j] = sum_{pixel in window (i,j)} cp[b,t,pixel] * xn[b,pixel,c]
 * (TP taskprompter.py:236-240,246). cp fp32 [B,T,P]; xn = split LN1 output of the joint stream
 * [B*N, ldx] (patch rows start at T); out fp32 [B,T,C,nh,nw]. */
int mtt_chan_logits(const float* cp, const void* xn_hi, const void* xn_lo, int64_t ldx, int32_t B,
                    int32_t N, int32_t T, int32_t C, int32_t gh, int32_t gw, int32_t nh, int32_t nw,
                    float* out, mtt_stream_t stream);

/* Spatial + channel gating of the patch feature map for `ntasks` consecutive tasks starting at `task`, X read once
 * (TP taskprompter.py:436-446, :452-467): Ys_t = X*(1 + R[b, c/dh, t, T+pix]), Yc_t = X*(1 + Rc[b,t,c,window(pix)]),
 * written as split [B*P, ldy] operands of the 1x1 decode convs; task t's planes start (t - task) * task_stride
 * ELEMENTS after the given pointers. X row (b, pix) is at x + (b*x_group_rows + x_row_offset + pix)*ldx.
 * C and the head dim must be multiples of 8. */
int mtt_gate_split(const float* x, int64_t ldx, int64_t x_group_rows, int64_t x_row_offset,
                   const float* prompt_logits, const float* chan_logits, int32_t task, int32_t ntasks, int32_t B,
                   int32_t T, int32_t N, int32_t H, int32_t C, int32_t gh, int32_t gw, int32_t nh,
                   int32_t nw, void* ys_hi, void* ys_lo, void* yc_hi, void* yc_lo, int64_t ldy, int64_t task_stride,
                   mtt_stream_t stream);

/* Cross-task reweighting (TP taskprompter.py:478-485).
 * mtt_ctr_weights: w[b,t,j] = W2_t . gelu(W0_t . R[b,:,t,j] + b0_t) + b2_t with W0 [T,H,H], b0 [T,H],
 *   W2 [T,H], b2 [T] (ctr_attn_conv.{il}.{task}.{0,2}); out fp32 [B,T,T].
 * mtt_ctr_mix: acc[t][m,:] (+)= sum_j w[b(m),t,j] * F[j][m,:]; F, acc fp32 [T, M, ld]. */
int mtt_ctr_weights(const float* prompt_logits, int32_t B, int32_t H, int32_t T, int32_t N,
                    const float* w0, const float* b0, const float* w2, const float* b2, float* out,
                    mtt_stream_t stream);
int mtt_ctr_mix(const float* F, const float* w, float* acc, int32_t T, int64_t M, int32_t C, int64_t ld,
                int32_t rows_per_batch, int32_t accumulate, mtt_stream_t stream);

/* Bilinear resize, align_corners=False (F.interpolate at TP taskprompter.py:420,
 * taskprompter_wrapper.py:35; IP transformer_net.py:35). in NHWC fp32 [B,h,w,C] (ld_in); outputs:
 * NHWC fp32 (optionally accumulated into) and/or NHWC split, and/or NCHW fp32 [B,C,H2,W2].
 * Image b starts at row b*in_batch_rows + in_row_offset of `in` (0 batch rows = dense h*w), and at row
 * b*out_batch_rows + out_row_offset of the NHWC outputs: lets per-task slices of InvPT's joint
 * [B, T*h*w, C] token buffers be resampled in place (IP invpt.py:299-305, :537). */
int mtt_bilinear(const float* in, int64_t ld_in, int32_t B, int32_t h, int32_t w, int32_t C, int32_t H2,
                 int32_t W2, float* out_f32, int64_t ld_f32, void* out_hi, void* out_lo, int64_t ld_bf,
                 float* out_nchw, int32_t accumulate, int64_t in_batch_rows, int64_t in_row_offset,
                 int64_t out_batch_rows, int64_t out_row_offset, mtt_stream_t stream);

/* Bilinear resize to the output size FUSED with the reference's prediction post-processing
 * (`get_output`, TP/utils/utils.py:27-63 -- the step right after the hot path, SURVEY.md section 8f N3), so the
 * full-resolution fp32 logits are never materialised. in: NHWC fp32 [B,h,w,C] (ld_in).
 * kind 0 argmax -> int64 [B,H2,W2] (semseg, human_parts); 1 255*sigmoid -> fp32 [B,H2,W2] (edge);
 * 2 255*softmax[...,1] -> fp32 [B,H2,W2] (sal); 3 (normalize+1)*255/2 -> fp32 [B,H2,W2,3] (normals);
 * 4 clamp(min=0) -> fp32 [B,H2,W2,1] (depth). */
int mtt_bilinear_postproc(const float* in, int64_t ld_in, int32_t B, int32_t h, int32_t w, int32_t C,
                          int32_t H2, int32_t W2, int32_t kind, int64_t* out_i64, float* out_f32,
                          mtt_stream_t stream);

/* Inference-time image pre-processing of the reference in one kernel -- the step in FRONT of the hot path
 * (SURVEY.md section 8f N3): TP/inference.py:127-133 (cv2.imread, float32, BGR2RGB), :93-115 get_infer_transforms =
 * Normalize (data/transforms.py:236-251: x/255, -mean, /std) -> DirectResize (inference.py:66-81: cv2.resize
 * INTER_LINEAR) -> ToTensor (transforms.py:265-273). img: uint8 [B,h,w,3] on the device, channel order BGR if
 * bgr != 0 (cv2.imread) else RGB; mean3 / std3: HOST pointers to three floats (RGB order); out: fp32 NCHW
 * [B,3,H,W], ready for mtt_im2col_patch. */
int mtt_preprocess_image(const uint8_t* img, int32_t B, int32_t h, int32_t w, int32_t bgr, const float* mean3,
                         const float* std3, float* out, int32_t H, int32_t W, mtt_stream_t stream);

/* Training-time augmentation of the reference (TP/utils/common_config.py:96-121, TP/data/transforms.py) over a ragged
 * batch of raw samples, in at most three launches. train != 0: RandomScaling(0.5, 2) -> RandomCrop(crop,
 * cat_max_ratio 0.75) -> RandomHorizontalFlip -> PhotoMetricDistortion -> Normalize -> PadImage(crop) ->
 * AddIgnoreRegions -> ToTensor, with every random draw given in the sample records; train == 0: the validation chain
 * Normalize -> PadImage -> AddIgnoreRegions -> ToTensor (records carry scale 1 and no crop; H x W is the padded size,
 * max(raw, test size), equal for every sample).
 * `samples` (device) holds B mtt_augment_sample records; `data` (device) the raw float32 HWC arrays they point into:
 * image [h,w,3] with integer values 0..255, label maps [h,w,1] (semseg, human_parts, sal, edge, depth) or [h,w,3]
 * (normals); semseg holds integer labels (255 = ignore). Outputs: image_out fp32 [B,3,H,W], task_out[t] fp32
 * [B,C,H,W]. workspace: mtt_augment_workspace_bytes(B) bytes (4-byte aligned): per (sample, candidate) flags
 * (bit 0 cat_max_ratio test passed, bit 1 human_parts crop is all 0 / 255), then the chosen candidate per sample
 * (int32, -1 = no crop). Bit-exact against the reference on the labels and on every stage after the uint8 cast of the
 * image; the cv2 rules restated are listed in oracle/augment_ref.py. */
#define MTT_AUG_MAX_TASKS 7
#define MTT_AUG_CANDIDATES 11
enum mtt_aug_task {
  MTT_AUG_SEMSEG = 0, MTT_AUG_HUMAN_PARTS = 1, MTT_AUG_SAL = 2, MTT_AUG_EDGE = 3, MTT_AUG_NORMALS = 4, MTT_AUG_DEPTH = 5
};
typedef struct {
  int64_t off[1 + MTT_AUG_MAX_TASKS]; /* float offsets into data: the image, then task t's map */
  double lin_y, lin_x;                /* h / sh, w / sw: the INTER_LINEAR source step */
  double nn_y, nn_x;                  /* 1 / (sh / h), 1 / (sw / w): the INTER_NEAREST source step */
  int32_t h, w, sh, sw;               /* raw and scaled size (scaled = raw when scale == 1) */
  int32_t scaled;                     /* scale != 1: depth is divided by depth_scale = float32(scale) */
  float depth_scale;
  int32_t ncand;                      /* 0: the scaled size equals the crop size (no crop), else MTT_AUG_CANDIDATES */
  int32_t cand[MTT_AUG_CANDIDATES][2]; /* crop offsets (y, x) */
  int32_t flip;
  int32_t bright_on, f_mode, contrast_on, sat_on, hue_on;
  float beta, alpha, sat_alpha;
  int32_t hue_delta;
} mtt_augment_sample;
typedef struct {
  const void* samples;
  const float* data;
  int32_t B, H, W;
  int32_t train;
  int32_t crop_h, crop_w; /* train: the crop size (= H, W) */
  int32_t ntasks;
  int32_t task_kind[MTT_AUG_MAX_TASKS]; /* mtt_aug_task, each at most once; train needs semseg */
  float* task_out[MTT_AUG_MAX_TASKS];
  float* image_out;
  float mean[3], std[3];
  void* workspace;
  size_t workspace_bytes;
} mtt_augment_desc;
size_t mtt_augment_workspace_bytes(int32_t B);
int mtt_augment(const mtt_augment_desc* d, mtt_stream_t stream);

/* Cityscapes-3D targets (TP/data/cityscapes3d.py:150-160 disparity, :235-241 encode_segmap, :206-228 PIL NEAREST
 * resize to dd_label_map_size) over a batch of equally sized raw maps, in one launch. label_ids: uint8 [B,h,w] (the
 * gtFine labelIds PNGs); disparity: uint16 [B,h,w] (the disparity PNGs), needed when depth is requested. Outputs at
 * H x W (H x W == h x w: no resize): semseg int64 [B,H,W] -- void ids -> 255, the 19 valid ids -> 0..18, other ids
 * unchanged; depth fp32 [B,1,H,W] -- (d - 1) / 256 for d > 1, -1 for d <= 1 (the reference's in-place steps also turn
 * d == 1 into -1), 0 where the raw label id is 10 (as the reference masks it). Either output may be NULL, not both. Source pixels follow Pillow's NEAREST rule, restated in
 * oracle/cityscapes_ref.py. */
int mtt_cityscapes_targets(const uint8_t* label_ids, const uint16_t* disparity, int32_t B, int32_t h, int32_t w,
                           int32_t H, int32_t W, int64_t* semseg, float* depth, mtt_stream_t stream);

/* Predictions -> uint8 images, for the reference's prediction export (save_model_pred_for_one_task,
 * TP/evaluation/evaluate_utils.py:69-151, IP/evaluation/evaluate_utils.py:69-105) and inference visualisation
 * (vis_pred_for_one_task, TP/utils/visualization_utils.py:80-199). One descriptor per task; all (task, image) pairs of
 * a call are rendered by one pre-pass launch (JET min / max, all-ignore label flags) and one main launch:
 *   source   LOGITS fp32 [B,C,h,w] (the wrapper's output), bilinearly resized to out_h x out_w (F.interpolate,
 *            align_corners=False; no resize when equal) and post-processed with get_output kind `postproc` (0 argmax,
 *            1 edge, 2 sal, 3 normals, 4 depth: the per-pixel code of mtt_bilinear_postproc); or a get_output map as
 *            predict() returns it, not resized: CLASS int64 [B,h,w], MAP fp32 [B,h,w,C] with C = 1 or 3;
 *   crop     per image (y0, x0, h, w) inside the out_h x out_w map, or inside out_size[i] when given (LOGITS: a
 *            resize target per image); host arrays, read at enqueue;
 *   encode   U8: astype(np.uint8) of a scalar map; CLASS: the class id as uint8, through `table` (256 ids, optional);
 *            PALETTE_BGR: RGB palette[class] stored B, G, R; NORMALS_BGR: the three channels truncated, stored B, G, R;
 *            JET: (v - min) / (max - min) * 255 in float32 over the image's crop, truncated, then the BGR `table`.
 *            Truncation is numpy's float32 -> uint8 cast on x86-64: the low byte of the int32 truncation, where NaN
 *            and out-of-range values give INT32_MIN; so a constant map (max == min, 0 / 0 = NaN) is JET index 0.
 *   store    uint8 at out + offset[i] (host array of byte offsets), [h,w] or HWC [h,w,3].
 * `label` (optional, device fp32 [B,label_numel]) sets flags[i] (device int32 [B]) to 1 when every value of image i's
 * label equals ignore_index (the reference's `len(label.unique()) == 1 and label.unique() == ignore` skip rule).
 * Tables are device data. workspace: mtt_render_workspace_bytes(n, max B) bytes, 4-byte aligned; the call zeroes it
 * with cudaMemsetAsync. At most MTT_RENDER_MAX_TASKS descriptors and MTT_RENDER_MAX_IMAGES (task, image) pairs per
 * call. Rejected: unknown kinds, a get_output kind the channel count cannot take, an encoding the source cannot take,
 * a palette shorter than the class count C, a crop outside the map, an offset outside out_bytes. */
#define MTT_RENDER_MAX_TASKS 8
#define MTT_RENDER_MAX_IMAGES 96
enum mtt_render_src { MTT_RENDER_SRC_LOGITS = 0, MTT_RENDER_SRC_CLASS = 1, MTT_RENDER_SRC_MAP = 2 };
enum mtt_render_encode {
  MTT_RENDER_U8 = 0, MTT_RENDER_CLASS = 1, MTT_RENDER_PALETTE_BGR = 2, MTT_RENDER_NORMALS_BGR = 3, MTT_RENDER_JET = 4
};
typedef struct {
  int32_t src_kind;       /* mtt_render_src */
  const void* src;        /* device */
  int32_t B, C, h, w;     /* source geometry; C: logit channels, MAP channels, or the class count of a CLASS map */
  int32_t out_h, out_w;   /* LOGITS: resize target; CLASS / MAP: h, w */
  int32_t postproc;       /* LOGITS: get_output kind 0..4; ignored otherwise */
  int32_t encode;         /* mtt_render_encode */
  const uint8_t* table;   /* device: palette [table_len][3] RGB, class-id table [table_len >= 256], JET [256][3] BGR */
  int32_t table_len;
  const int32_t* crop;    /* host [B][4]: y0, x0, h, w */
  const int64_t* offset;  /* host [B]: byte offset of each image in out */
  const int32_t* out_size; /* host [B][2], optional (LOGITS): per-image resize target instead of out_h x out_w */
  uint8_t* out;           /* device */
  int64_t out_bytes;
  const float* label;     /* device, optional */
  int64_t label_numel;    /* per image */
  float ignore_index;
  int32_t* flags;         /* device int32 [B]; required with label */
} mtt_render_desc;
size_t mtt_render_workspace_bytes(int32_t n_tasks, int32_t B);
int mtt_render(const mtt_render_desc* d, int32_t n, void* workspace, mtt_stream_t stream);
/* cv2.applyColorMap(np.arange(256, dtype=np.uint8), cv2.COLORMAP_JET): 256 BGR triples (host memory). */
const uint8_t* mtt_render_jet_bgr(void);

/* Sum of up to three bilinearly resized NHWC fp32 sources written once as a split tensor [B*H2*W2, ld_bf]:
 * InvPT's multi-scale aggregation of the three stages' per-task maps (IP invpt.py:528-539), in the
 * reference's accumulation order, without read-modify-write passes over the full-resolution map. */
typedef struct {
  const float* in;
  int64_t ld_in;
  int32_t h, w;
  int64_t batch_rows; /* rows between images of `in` (0: h*w) */
  int64_t row_offset; /* first row of image 0 */
} mtt_bilinear_src;
int mtt_bilinear_sum3(const mtt_bilinear_src* srcs, int32_t nsrc, int32_t B, int32_t C, int32_t H2, int32_t W2,
                      void* out_hi, void* out_lo, int64_t ld_bf, mtt_stream_t stream);

/* ---- InvPT decoder (IP/models/transformers/invpt.py, transformer_decoder.py) ---------------- */
/* fp32 rows gathered at (r / in_group) * src_group + src_offset + r % in_group -> dense split rows.
 * Replaces x[:, 1:] token selection + layout copies (IP vit.py:345-346, transformer_decoder.py:77). */
int mtt_split_rows(const float* in, int64_t ld_in, int64_t in_group, int64_t src_group, int64_t src_offset,
                   void* out_hi, void* out_lo, int64_t ld_out, int64_t rows, int32_t cols,
                   mtt_stream_t stream);

/* LayerNorm over S segments of `cols` channels (segment s of logical row r lives S*... at physical row
 * map(r) + s*seg_stride); gamma/beta [S*cols]; segment s is written to output row s*out_seg_stride + r.
 * S = 1: gathered LayerNorm (IP vit.py:348-349). S = T: the joint-channel LayerNorm over all tasks'
 * tokens, norm_mts (IP invpt.py:524-526). */
int mtt_layernorm_seg(const float* in, int64_t ld_in, int64_t in_group, int64_t src_group,
                      int64_t src_offset, int64_t seg_stride, int32_t S, const float* gamma,
                      const float* beta, float eps, float* out_f32, int64_t ld_f32, void* out_hi,
                      void* out_lo, int64_t ld_bf, int64_t out_seg_stride, int64_t rows, int32_t cols,
                      mtt_stream_t stream);

/* Stride-2 zero insertion [B,h,w,C] fp32 -> split [B,2h,2w,C]: ConvTranspose2d(k3,s2,p1,op1) then runs
 * as a 3x3 convolution with the flipped kernel on mtt_gemm (IP transformer_decoder.py:63). */
int mtt_zero_insert(const float* in, int64_t ld_in, int64_t src_group, int64_t src_offset, int32_t B,
                    int32_t h, int32_t w, int32_t C, void* out_hi, void* out_lo, int64_t ld_out,
                    mtt_stream_t stream);

/* Per-task depthwise 3x3 stride-2 conv with folded eval BatchNorm -> Q tokens (IP invpt.py:125-137).
 * in fp32 joint tokens [B, T*h*w, C]; weight [T,C,9], bias [T,C]; out split [B, T*(h/2)(w/2), C]. */
int mtt_dwconv3x3_s2(const float* in, int64_t ld_in, int32_t B, int32_t T, int32_t h, int32_t w, int32_t C,
                     const float* weight, const float* bias, void* out_hi, void* out_lo, int64_t ld_out,
                     mtt_stream_t stream);

/* Per-task average pooling kernel = stride = s, ceil_mode (IP invpt.py:139-147): in fp32 [BT, h*w, C]
 * -> split [BT, ceil(h/s)*ceil(w/s), C]. */
int mtt_avgpool(const float* in, int64_t ld_in, int32_t BT, int32_t h, int32_t w, int32_t C, int32_t s,
                void* out_hi, void* out_lo, int64_t ld_out, mtt_stream_t stream);

/* InvPT cross-task attention with cross-scale score fusion (IP invpt.py:204-236), 2 heads: the two contractions
 * (S = Q_h K_h^T, O_h = P_h V_h) are grouped mtt_gemm launches over (batch, head); this is the step between them.
 * raw fp32 [B,2,Lq,Tk] = un-scaled q_h . k_h; scale = C^-1/2. prev_score (optional) fp32 [B,2,T*(qh/2)*(qw/2),Tk] is
 * bilinearly up-sampled x2 per task over the query grid and mixed with the current scores by the 1x1 conv fuse_w [2,4],
 * fuse_b [2] (fuse_attn, :116,:229). score_out (optional, may alias raw) receives the fused pre-softmax scores (:230);
 * P = softmax over the Tk keys is written as split rows [(b*2 + h)*Lq + l, ldp]: the A operand of the second GEMM. */
int mtt_invpt_fuse_softmax(const float* raw, int32_t B, int32_t Lq, int32_t Tk, float scale, const float* prev_score,
                           int32_t T, int32_t qh, int32_t qw, const float* fuse_w, const float* fuse_b, float* score_out,
                           void* p_hi, void* p_lo, int64_t ldp, mtt_stream_t stream);

/* ---- the named operators of SURVEY.md section 8(b) -----------------------------------------------------------
 * Each replaces one eager-op group of the reference block / decoder with a fixed launch sequence; intermediates
 * live in the caller's workspace (size from mtt_workspace_bytes, 256-byte aligned), so nothing is allocated and
 * the whole forward stays capturable in one CUDA graph. A workspace is zero-filled ONCE by the caller when it is
 * allocated (the LayerNorm-fronted operators keep their GEMMs' stream-K flag words in it: mtt_gemm_desc.sk_ws) and
 * must not be shared by calls that can run concurrently on different streams.
 *
 * DEVIATIONS from the entry-point list SURVEY.md 8(b) sketched (all deliberate, same ownership / error / stream
 * rules): (1) attn_fwd, chan_prompt_logits, bilinear_up, invpt_attn, layernorm are the single-kernel entries above
 * (mtt_attention, mtt_chan_logits, mtt_bilinear, mtt_invpt_fuse_softmax between two mtt_gemm_grouped launches,
 * mtt_layernorm) under their own names;
 * (2) shapes travel in mtt_shape and weights in mtt_weight (pre-packed planes) instead of a flat argument list;
 * (3) LayerNorm is a kernel of the sequence, not a prologue inside the GEMM: the normalised rows are written once as
 * split planes (8.4 us per 16.8 MB at cfg4) and read back from L2 by the TMA producer. */
enum mtt_op {
  MTT_OP_LN_QKV = 1, MTT_OP_ATTN_FWD = 2, MTT_OP_PROJ_RESIDUAL = 3, MTT_OP_LN_MLP_RESIDUAL = 4,
  MTT_OP_CHAN_PROMPT_LOGITS = 5, MTT_OP_GATED_CONV1X1 = 6, MTT_OP_CONV3X3_BN_ACT = 7, MTT_OP_BILINEAR_UP = 8,
  MTT_OP_INVPT_ATTN = 9, MTT_OP_LAYERNORM = 10
};
typedef struct {
  int32_t rows;   /* token rows of the joint stream (B*N), or output pixels (B*H*W) for the conv operators */
  int32_t C;      /* model width */
  int32_t hidden; /* Mlp hidden width / conv output channels */
  int32_t nsplit; /* 2 = parity mode (both planes), 1 = speed mode */
  int32_t B, N, H, T; /* batch, tokens per image, heads, prompt rows */
} mtt_shape;
typedef struct {
  const void* hi; /* packed planes produced by mtt_pack_weight / mtt_pack_conv_weight (caller-owned) */
  const void* lo;
  int64_t ld;
} mtt_weight;

size_t mtt_workspace_bytes(int32_t op, const mtt_shape* shape);

/* qkv = LN(x) . Wqkv^T + b: TP taskprompter.py:272 (norm1 on prompts and patches), :199, :201. x fp32 [rows, C];
 * workspace receives LN(x) as split planes [nsplit][rows][pad8(C)] (the channel-prompt path reads it from there). */
int mtt_ln_qkv(const float* x, int64_t ldx, const float* gamma, const float* beta, float eps, const mtt_weight* wqkv,
               const float* bias, void* qkv_hi, void* qkv_lo, int64_t ldq, const mtt_shape* shape, void* workspace,
               size_t ws_bytes, mtt_stream_t stream);
/* x += attn_out . Wproj^T + b: TP taskprompter.py:212 + the residual adds of :273 / :276 (in place on x). */
int mtt_proj_residual(const void* a_hi, const void* a_lo, int64_t lda, const mtt_weight* wproj, const float* bias,
                      float* x, int64_t ldx, const mtt_shape* shape, mtt_stream_t stream);
/* x += fc2(gelu(fc1(LN(x)))): TP taskprompter.py:274 / :277 (timm Mlp, exact-erf GELU), in place on x. */
int mtt_ln_mlp_residual(float* x, int64_t ldx, const float* gamma, const float* beta, float eps, const mtt_weight* w1,
                        const float* b1, const mtt_weight* w2, const float* b2, const mtt_shape* shape,
                        void* workspace, size_t ws_bytes, mtt_stream_t stream);
/* Spatial and channel gating of the patch map for ALL `ntasks` tasks of a level + their 2*ntasks 1x1 decode convs,
 * each task's pair written side by side into its `cat` operand of fea_fuse (TP taskprompter.py:436-447, :452-468,
 * :471): columns [0, e) = spatial branch, [chan_col, chan_col + e) = channel branch. One gating launch (X read once)
 * and one grouped GEMM launch of 2*ntasks problems (chunks of 6 tasks). x / prompt_logits / chan_logits as in
 * mtt_gate_split; workspace: mtt_workspace_bytes(MTT_OP_GATED_CONV1X1) with shape.rows = B*gh*gw, shape.T = ntasks. */
typedef struct {
  mtt_weight w_spa;
  const float* b_spa;
  mtt_weight w_chan;
  const float* b_chan;
  void* cat_hi;
  void* cat_lo;
} mtt_gated_task;
int mtt_gated_conv1x1(const float* x, int64_t ldx, int64_t x_group_rows, int64_t x_row_offset,
                      const float* prompt_logits, const float* chan_logits, int32_t ntasks, const mtt_gated_task* tasks,
                      int32_t gh, int32_t gw, int32_t nh, int32_t nw, int32_t e, int64_t ld_cat, int32_t chan_col,
                      const mtt_shape* shape, void* workspace, size_t ws_bytes, mtt_stream_t stream);
/* 3x3 conv (stride 1, dilation dil, zero padding) with folded eval BatchNorm + activation on an NHWC split map, and
 * optionally the 1x1 prediction head right behind it (TP taskprompter.py:362 fea_fuse[1..3]; :691-695 ConvHead;
 * IP transformer_decoder.py:113, invpt.py:33-38, :493). mid_* = the activation map (NULL with a fused head: it then
 * lives in the workspace); w_head NULL = no head. */
int mtt_conv3x3_bn_act(const void* a_hi, const void* a_lo, int64_t lda, int32_t B, int32_t H, int32_t W, int32_t Cin,
                       int32_t dil, const mtt_weight* w3, const float* b3, int32_t Cout, int32_t act, void* mid_hi,
                       void* mid_lo, int64_t ld_mid, const mtt_weight* w_head, const float* b_head, int32_t n_out,
                       float* out_f32, int64_t ldo, int32_t nsplit, void* workspace, size_t ws_bytes,
                       mtt_stream_t stream);

/* ---- parameter pre-packing (once per parameter version; outputs are caller-owned tensors) ---------------------
 * mtt_pack_weight: nn.Linear / 1x1 conv weight fp32 [N, K] -> split planes [N, ld_out], K zero-padded to 8.
 * mtt_pack_conv_weight: Conv2d weight [N, Cin, k, k] (transposed = 0) or ConvTranspose2d weight [Cin, N, k, k]
 *   (transposed = 1: stored as the spatially flipped kernel of the equivalent convolution over the zero-inserted
 *   map) -> tap-major planes [N, k*k*cin_pad], cin_pad = Cin rounded up to 64, with an eval-mode BatchNorm folded in
 *   (bn_gamma NULL = none): w' = w * gamma / sqrt(var + eps), bias_out = (bias - mean) * gamma / sqrt(var + eps) +
 *   beta. scale_ws: N floats of scratch. */
int mtt_pack_weight(const float* w, int64_t ld_w, int32_t N, int32_t K, int32_t nsplit, void* out_hi, void* out_lo,
                    int64_t ld_out, mtt_stream_t stream);
int mtt_pack_conv_weight(const float* w, const float* bias, const float* bn_gamma, const float* bn_beta,
                         const float* bn_mean, const float* bn_var, float bn_eps, int32_t N, int32_t Cin,
                         int32_t ksize, int32_t transposed, int32_t nsplit, void* out_hi, void* out_lo, int64_t ld_out,
                         float* bias_out, float* scale_ws, mtt_stream_t stream);

/* ---- training losses and their gradients w.r.t. the predictions (SURVEY.md 8f N3) -------------------------------
 * TP/losses/loss_functions.py: CrossEntropyLoss :15-55 (ignore regions; balanced = binary class balancing :32-41),
 * BalancedBinaryCrossEntropyLoss :57-87 (fixed pos_weight, or hed != 0: HED-style weight from the labels), L1Loss
 * :144-176 (normalize = L2-normalise the prediction first; a pixel is valid when EVERY label channel differs from
 * ignore_index). pred NCHW fp32 [B,C,H,W] (the model's outputs), label fp32 ([B,1,H,W] for cross entropy / BCE,
 * [B,C,H,W] for L1). loss_out: one float ON THE DEVICE (reduction 'mean' exactly as the reference divides). No host
 * synchronisation; reductions run in a fixed order (bitwise reproducible). workspace: mtt_loss_workspace_bytes()
 * bytes, 8-byte aligned; the *_grad calls read the statistics the forward call left there and write
 * dpred = (*grad_scale) * d loss / d pred (grad_scale: one float on the device, the upstream gradient). */
size_t mtt_loss_workspace_bytes(void);
int mtt_loss_cross_entropy(const float* pred, const float* label, int32_t B, int32_t C, int32_t H, int32_t W,
                           float ignore_index, int32_t balanced, float* loss_out, void* workspace, mtt_stream_t stream);
int mtt_loss_cross_entropy_grad(const float* pred, const float* label, int32_t B, int32_t C, int32_t H, int32_t W,
                                float ignore_index, int32_t balanced, const float* grad_scale, float* dpred,
                                const void* workspace, mtt_stream_t stream);
int mtt_loss_balanced_bce(const float* pred, const float* label, int64_t n, float ignore_index, float pos_weight,
                          int32_t hed, float* loss_out, void* workspace, mtt_stream_t stream);
int mtt_loss_balanced_bce_grad(const float* pred, const float* label, int64_t n, float ignore_index, float pos_weight,
                               int32_t hed, const float* grad_scale, float* dpred, const void* workspace,
                               mtt_stream_t stream);
int mtt_loss_l1(const float* pred, const float* label, int32_t B, int32_t C, int32_t H, int32_t W, float ignore_index,
                int32_t use_ignore, int32_t normalize, float* loss_out, void* workspace, mtt_stream_t stream);
int mtt_loss_l1_grad(const float* pred, const float* label, int32_t B, int32_t C, int32_t H, int32_t W,
                     float ignore_index, int32_t use_ignore, int32_t normalize, const float* grad_scale, float* dpred,
                     const void* workspace, mtt_stream_t stream);

/* ---- evaluation meters (the reference's PerformanceMeter, TP/evaluation/evaluate_utils.py:13-66) ------------------
 * Each *_update enqueues ONE kernel that adds a batch's statistics into `state`, a caller-owned device buffer of
 * mtt_meter_state_bytes(kind, n) bytes (8-byte aligned; n = classes for CONFUSION, thresholds for SALIENCY, ignored
 * otherwise); mtt_meter_reset zeroes it with a cudaMemsetAsync on `stream`. Nothing is allocated or synchronised, so
 * updates can be captured in a CUDA graph; the score formulas run on the host over one copy of the state (layouts in
 * csrc/metrics.cu). Integer counters are int64; float sums are fp64, reduced in a fixed order (bitwise reproducible).
 * Inputs are predict()'s outputs (= the reference's get_output, TP/utils/utils.py:27-63) and the labels as the
 * reference's loader yields them: fp32 [B,C,H,W], ignore_index marking ignored pixels.
 *   CONFUSION  pred int64 [B,H,W] class map, label [B,1,H,W]; SemsegMeter eval_semseg.py:70-81 and HumanPartsMeter
 *              eval_human_parts.py:33-42 (n_classes <= 64).
 *   SALIENCY   pred fp32 [B,H,W] (255 * probability), label [B,1,H,W]; SaliencyMeter eval_sal.py:21-60:
 *              prob = sigmoid(pred / 255), counts per threshold (device array of n_thresholds <= 32 floats).
 *   NORMALS    pred fp32 [B,H,W,3] ((n + 1) * 255 / 2), label [B,3,H,W]; NormalsMeter eval_normals.py:33-45.
 *   DEPTH      pred fp32 with B*H*W elements, label [B,1,H,W]; valid = min_depth < gt < max_depth when use_range
 *              (TP eval_depth.py:36), gt != ignore_index otherwise (IP eval_depth.py DepthMeter). Values <= 0 count as
 *              1e-9 (:41-42); unlike the reference, the inputs are not modified.
 *   EDGE       pred fp32 [B,H,W] (255 * sigmoid), label [B,1,H,W]; EdgeMeter eval_edge.py:21-31 with a fixed
 *              pos_weight in [0, 1). */
enum mtt_meter_kind {
  MTT_METER_CONFUSION = 0,
  MTT_METER_SALIENCY = 1,
  MTT_METER_NORMALS = 2,
  MTT_METER_DEPTH = 3,
  MTT_METER_EDGE = 4
};
/* 0 (with the error text set) for an unknown kind or a size over the capacity */
size_t mtt_meter_state_bytes(int32_t kind, int32_t n);
int mtt_meter_reset(void* state, int32_t kind, int32_t n, mtt_stream_t stream);
int mtt_meter_confusion_update(const int64_t* pred, const float* label, int32_t B, int32_t H, int32_t W,
                               int32_t n_classes, float ignore_index, void* state, mtt_stream_t stream);
/* The same update with int64 labels [B,H,W] (the Cityscapes-3D loader's semseg, TP/data/cityscapes3d.py:227). */
int mtt_meter_confusion_update_i64(const int64_t* pred, const int64_t* label, int32_t B, int32_t H, int32_t W,
                                   int32_t n_classes, float ignore_index, void* state, mtt_stream_t stream);
int mtt_meter_saliency_update(const float* pred, const float* label, int32_t B, int32_t H, int32_t W,
                              const float* thresholds, int32_t n_thresholds, float ignore_index, void* state,
                              mtt_stream_t stream);
int mtt_meter_normals_update(const float* pred_nhwc, const float* label, int32_t B, int32_t H, int32_t W,
                             float ignore_index, void* state, mtt_stream_t stream);
int mtt_meter_depth_update(const float* pred, const float* label, int32_t B, int32_t H, int32_t W, int32_t use_range,
                           float min_depth, float max_depth, float ignore_index, void* state, mtt_stream_t stream);
int mtt_meter_edge_update(const float* pred, const float* label, int32_t B, int32_t H, int32_t W, float pos_weight,
                          float ignore_index, void* state, mtt_stream_t stream);

/* ---- BEV IoU of rotated boxes and NMS (SURVEY.md 8f N4) ---------------------------------------------------------
 * Replaces the reference's native extension TP/detection_toolbox/iou3d (iou3d_kernel.cu:253-439, iou3d.cpp:51-202).
 * Boxes are [x1, y1, x2, y2, ry] fp32 rows on the device. mtt_boxes_bev_pairwise: out[a, b] = overlap area (mode 0,
 * boxes_overlap_bev_gpu) or rotated IoU (mode 1, boxes_iou_bev_gpu). mtt_nms_bev: boxes must already be sorted by
 * descending score (iou3d_utils.py:38-42 does that before the call); keep[0 .. *num_keep) = indices of the survivors in
 * order, greedy suppression of every later box with IoU > thresh (rotated != 0: nms_gpu, else nms_normal_gpu). The
 * sweep runs on the device: keep (int64) and num_keep (int32) are DEVICE pointers, nothing is copied to the host or
 * allocated; workspace = mtt_nms_workspace_bytes(n) bytes, 8-byte aligned. */
int mtt_boxes_bev_pairwise(const float* boxes_a, int32_t num_a, const float* boxes_b, int32_t num_b, int32_t mode,
                           float* out, mtt_stream_t stream);
size_t mtt_nms_workspace_bytes(int32_t n);
int mtt_nms_bev(const float* boxes, int32_t n, float thresh, int32_t rotated, int64_t* keep, int32_t* num_keep,
                void* workspace, size_t ws_bytes, mtt_stream_t stream);

/* ---- Swin-backbone TaskPrompter (SURVEY.md 8f N2; TP = TaskPrompter/models/transformers/taskprompter_swin.py) --------
 * The joint window stream has, for image b and window w (row-major over the zero-padded, cyclically shifted map),
 * T prompt rows followed by ws*ws token rows: rows [(b*nW + w)*(T + ws*ws), ...). Geometry is always given as the
 * un-padded map (H, W), the window size ws and the cyclic shift (0 <= shift < ws); padding to multiples of ws is implied.
 *
 * mtt_swin_window_gather: LN1 outputs xn [B*H*W, C] and pn [B*T, C] (fp32) -> split joint window stream (TP:326-340,
 *   :177-181; padding rows are zero).
 * mtt_swin_window_attention: per (window, head) softmax((q k^T) * scale + B) v over the T + L tokens of a window, B =
 *   relative-position bias (+ shift mask of window w % nW) on the patch x patch entries only (TP:183-206). qkv = split
 *   output of the qkv GEMM on the joint stream, columns (q|k|v, head, head_dim). biasT [heads, L, L] and maskT
 *   [nW, L, L] (NULL = no shift) are stored TRANSPOSED ([.., key, query]). raw [BW, heads, T, L] receives the un-scaled
 *   q.k of the prompt rows against the window's tokens (TP:189). head_dim in {8, 16, 32, 64}.
 * mtt_swin_window_scatter: o = proj output on the joint stream (fp32) -> xa [B*H*W, C] (window reverse, un-shift,
 *   crop; TP:343-360), x += xa (TP:399), prompts += mean over windows of the prompt rows (TP:210; skipped when
 *   update_prompts = 0), and raw -> logits [B, heads, T, T + H*W] at column T + pixel: the layout mtt_gate_split reads.
 * mtt_transpose_split: [B, L, C] fp32 -> split [B*C, ld_out >= L]: the A operand of chan_kv (TP:379).
 * mtt_swin_chan_attention: q [B*T, ce], kv [B*C, 2*ce] (k | v) fp32 -> raw_chan [B,T,C,nh,nw] = un-scaled logits between
 *   each prompt and each CHANNEL inside every window of the sqrt(ce) x sqrt(ce) embedding grid, and chan_out [B*T, ce]
 *   (fp32 + split) = softmax(raw * ce^-1/2) v (TP:383-396).
 * mtt_swin_merge_gather: [B,H,W,C] -> [B*(H/2)*(W/2), 4C], quadrant order (0,0), (1,0), (0,1), (1,1) (TP:441-447).
 * mtt_conv3x3_s2_maps: stride-2 3x3 conv (pad 1) over maps stored as in[b, ci, in_offset + y*W + x] with channel stride
 *   in_stride (PatchMerging.spa_attn_ds on the logit maps, TP:458-460). w [Cout, Cin, 3, 3].
 * mtt_swin_chan_up: out[bt, o, win] = sum_c w[o, c] raw_chan[bt, c, win] (process_chan_attn, TP:463-466).
 * mtt_swin_logit_maps: the prompt-row logit maps between the gating layout logits [rows, T + L] (map r at columns
 *   [T, T + L)) and the reference's raw_spa_attn [B, heads, T, H, W] = maps [rows, L], rows = B*heads*T <= 65535.
 *   to_maps != 0: src = logits, dst = maps; to_maps = 0: src = maps, dst = logits (its columns < T are not written).
 *   The sub-module forwards' layout change (SwinTransformerBlock / PatchMerging, TP:352-365, :453-460). */
int mtt_swin_window_gather(const float* xn, int64_t ldx, const float* pn, int64_t ldp, int32_t B, int32_t H, int32_t W,
                           int32_t C, int32_t T, int32_t ws, int32_t shift, void* out_hi, void* out_lo, int64_t ld_out,
                           mtt_stream_t stream);
int mtt_swin_window_attention(const void* qkv_hi, const void* qkv_lo, int64_t ldq, int32_t BW, int32_t nW, int32_t T,
                              int32_t L, int32_t heads, int32_t head_dim, float scale, const float* biasT,
                              const float* maskT, void* out_hi, void* out_lo, int64_t ldo, float* raw,
                              mtt_stream_t stream);
int mtt_swin_window_scatter(const float* o, int64_t ldo, const float* raw, int32_t B, int32_t H, int32_t W, int32_t C,
                            int32_t T, int32_t ws, int32_t shift, int32_t heads, int32_t update_prompts, float* xa,
                            int64_t ldxa, float* x, int64_t ldx, float* prompts, int64_t ldp, float* logits,
                            mtt_stream_t stream);
int mtt_transpose_split(const float* in, int64_t ld_in, int32_t B, int32_t L, int32_t C, void* out_hi, void* out_lo,
                        int64_t ld_out, mtt_stream_t stream);
int mtt_swin_chan_attention(const float* q, int64_t ldq, const float* kv, int64_t ldkv, int32_t B, int32_t T, int32_t C,
                            int32_t ce, int32_t nh, int32_t nw, float* chan_out, int64_t ldco, void* cs_hi, void* cs_lo,
                            int64_t ldcs, float* raw_chan, mtt_stream_t stream);
int mtt_swin_merge_gather(const float* x, int64_t ldx, int32_t B, int32_t H, int32_t W, int32_t C, float* out, int64_t ldo,
                          mtt_stream_t stream);
int mtt_conv3x3_s2_maps(const float* in, const float* w, const float* bias, int32_t B, int32_t Cin, int32_t Cout, int32_t H,
                        int32_t W, int64_t in_stride, int32_t in_offset, int64_t out_stride, int32_t out_offset, float* out,
                        mtt_stream_t stream);
int mtt_swin_chan_up(const float* raw_chan, const float* w, int32_t BT, int32_t C, int32_t Cout, int32_t nwin, float* out,
                     mtt_stream_t stream);
int mtt_swin_logit_maps(const float* src, float* dst, int32_t rows, int32_t T, int32_t L, int32_t to_maps,
                        mtt_stream_t stream);

/* ---- layout changes at the nn.Module boundaries (ConvHead.forward takes / returns NCHW like the reference) ---- */
int mtt_nchw_to_nhwc_split(const float* in, int32_t B, int32_t C, int32_t H, int32_t W, void* out_hi, void* out_lo,
                           int64_t ld_out, mtt_stream_t stream);
int mtt_nhwc_to_nchw(const float* in, int64_t ld_in, int32_t B, int32_t C, int32_t H, int32_t W, float* out,
                     mtt_stream_t stream);

/* ---- training step: backward-pass and train-mode kernels (SURVEY.md 8f N1) ------------------------------------------
 * The loop served is TaskPrompter/utils/train_utils.py:34-51 (forward, criterion, backward, clip_grad_norm_, Adam step)
 * under main.py:92-94 (SyncBatchNorm + DDP). Contractions of the backward pass run on mtt_gemm / mtt_gemm_grouped: for
 * Y = A W^T, dA = dY (W^T)^T and dW = dY^T (A^T)^T are K-major GEMMs once the operands are transposed
 * (mtt_transpose_split for fp32 -> split, mtt_transpose_planes for split -> split). Everything here is fp32, row-major,
 * [rows, cols] with a leading dimension in elements.
 *
 * mtt_colsum: out[c] (+)= sum_r x[row(r), c] (bias gradients; pos_embed / task_prompts gradients over the batch); with
 *   in_group > 0 logical row r = (g, i), i < in_group, is physical row g*src_group + src_offset + i (as mtt_split_rows).
 * mtt_layernorm_bwd: dx (+)= LN'(x) dy; dgamma[c] += sum_r dy xhat, dbeta[c] += sum_r dy (accumulated: zero them once per
 *   step); stats_ws: 2*rows floats of scratch. (nn.LayerNorm eps 1e-6, TP taskprompter.py:262,266,329.)
 * mtt_act_split / mtt_act_bwd: act(pre) -> split planes (the A operand of the next GEMM); dx = dy * act'(pre) (dx may be dy).
 * mtt_axpy_rows: dst[r,:] = base[r,:] + row_scale[r] * src[r,:] (base / row_scale may be NULL): residual adds under
 *   DropPath (TP taskprompter.py:273-277; timm 0.5.4 drop_path: per-sample mask / keep_prob) and their adjoints.
 * mtt_transpose_planes: bf16 planes [B][R][C] (image b at row b*in_batch_rows) -> image b's [C, R] block at element offset
 *   b*out_batch_stride of the output (0 = C*ld_out: blocks stacked by rows; R: side by side along the columns); exact.
 * mtt_bn_stats / mtt_bn_finalize / mtt_bn_act: train-mode BatchNorm2d over NHWC rows: sums = (sum x, sum x^2) per channel
 *   [2*cols] accumulated in DOUBLE (all-reduce them across ranks for SyncBatchNorm, main.py:92), mean_rstd [2*cols] from
 *   sums / count with the variance sum x^2 / count - mean^2 formed in double (in fp32 that subtraction loses ~1e-6
 *   (mean/std)^2 of the variance, in double ~1e-16 (mean/std)^2) and the running statistics updated like nn.BatchNorm2d
 *   (momentum, unbiased running_var), then y = act(xhat*gamma + beta) as fp32 and / or split planes. mtt_bn_bwd_reduce: sums = (sum dz, sum dz*xhat), dz = dy * act'(z) (= dbeta, dgamma; all-reduce
 *   for SyncBatchNorm); mtt_bn_bwd_apply: dx = gamma*rstd*(dz - sums[0]/count - xhat*sums[1]/count).
 * mtt_attn_softmax_bwd: per (batch*head) rows of raw scores S [BH, N, ld] and dP [BH, N, ld] (fp32, read only):
 *   P = softmax(scale*S) recomputed, dS = scale*P*(dP - delta) with delta [BH, N] = sum_j P dP = rowdot(dO, O) from
 *   mtt_attn_delta (dO fp32 [B*N, H*head_dim], O = the forward's split output) (+ d_raw [BH, T, N] on the first T rows: the gradient of
 *   the exported prompt logits, TP taskprompter.py:204). Outputs, all split planes with row stride ldbf: dS row-major
 *   [BH*N queries, N] and (optional, NULL to skip) P^T and dS^T key-major [BH*N keys, N queries] -- the A operands of
 *   dQ = dS k, dV = P^T dO and dK = dS^T q.
 * mtt_bilinear_bwd: adjoint of mtt_bilinear (align_corners = False): dy NHWC (nchw = 0) or NCHW [B,C,H2,W2] (nchw = 1,
 *   lddy unused) -> dx NHWC [B,h,w,C] (+)=.
 * mtt_gate_bwd: adjoint of mtt_gate_split for one task: dx (+)=, d_prompt_logits [B,H,T,N] (+)= at column T + pixel,
 *   d_chan_logits [B,T,C,nh,nw] (+)=; dys / dyc fp32 [B*gh*gw, lddy].
 * mtt_chan_logits_bwd: adjoint of mtt_chan_logits: dcp [B,T,P] (=) and dxn (+)= on the patch rows of the joint stream.
 * mtt_ctr_bwd: adjoint of mtt_ctr_weights + the weights' use in mtt_ctr_mix: dnew, F fp32 [T, M, ld]; d_prompt_logits
 *   (+)= on the prompt-prompt columns; dw0 [T,H,H], db0 [T,H], dw2 [T,H], db2 [T] (+)=. dw_ws: B*T*T floats. (The feature
 *   gradients dF[j] = sum_t w[b,t,j] dnew[t] are mtt_ctr_mix with the transposed weights.)
 * mtt_im2col3x3_t / mtt_im2col_patch_t: the transposed, split im2col operands of the convolution weight gradients:
 *   rows (c, ky, kx) in nn.Conv2d.weight order, columns = output pixels (ldo >= B*H*W).
 * mtt_sumsq + mtt_adam_step: clip_grad_norm_(max_norm, 2) and torch.optim.Adam on flat fp32 arenas (p, g, m, v of n
 *   elements): g is scaled by grad_scale (1 / world size after a sum all-reduce) and by min(1, max_norm / (norm + 1e-6))
 *   when gnorm_sq (device scalar, sum of squared gradients BEFORE grad_scale) is given; weight decay is Adam's L2 form.
 *   beta1 / beta2 are double (as torch.optim.Adam keeps them): 1 - beta and the bias corrections are formed from them. */
int mtt_colsum(const float* x, int64_t ldx, int64_t rows, int32_t cols, int64_t in_group, int64_t src_group, int64_t src_offset,
               float* out, int32_t accumulate, mtt_stream_t stream);
int mtt_layernorm_bwd(const float* x, int64_t ldx, const float* dy, int64_t lddy, const float* gamma, float eps, int64_t rows,
                      int32_t cols, float* dx, int64_t lddx, int32_t accumulate_dx, float* dgamma, float* dbeta,
                      float* stats_ws, mtt_stream_t stream);
int mtt_act_split(const float* pre, int64_t ld, int64_t rows, int32_t cols, int32_t act, void* out_hi, void* out_lo,
                  int64_t ldo, mtt_stream_t stream);
int mtt_act_bwd(const float* pre, int64_t ld, const float* dy, int64_t lddy, int64_t rows, int32_t cols, int32_t act,
                float* dx, int64_t lddx, mtt_stream_t stream);
int mtt_axpy_rows(const float* base, int64_t ldb, const float* src, int64_t lds, const float* row_scale, int64_t rows,
                  int32_t cols, float* dst, int64_t ldd, mtt_stream_t stream);
int mtt_transpose_planes(const void* in_hi, const void* in_lo, int64_t ld_in, int64_t in_batch_rows, int32_t B, int32_t R,
                         int32_t C, void* out_hi, void* out_lo, int64_t ld_out, int64_t out_batch_stride,
                         mtt_stream_t stream);
int mtt_bn_stats(const float* x, int64_t ldx, int64_t rows, int32_t cols, double* sums, mtt_stream_t stream);
int mtt_bn_finalize(const double* sums, double count, int32_t cols, float eps, float momentum, float* mean_rstd,
                    float* running_mean, float* running_var, mtt_stream_t stream);
int mtt_bn_act(const float* x, int64_t ldx, int64_t rows, int32_t cols, const float* mean_rstd, const float* gamma,
               const float* beta, int32_t act, float* out_f32, int64_t ldo, void* out_hi, void* out_lo, int64_t ldbf,
               mtt_stream_t stream);
int mtt_bn_bwd_reduce(const float* x, int64_t ldx, const float* dy, int64_t lddy, int64_t rows, int32_t cols,
                      const float* mean_rstd, const float* gamma, const float* beta, int32_t act, float* sums,
                      mtt_stream_t stream);
int mtt_bn_bwd_apply(const float* x, int64_t ldx, const float* dy, int64_t lddy, int64_t rows, int32_t cols,
                     const float* mean_rstd, const float* gamma, const float* beta, int32_t act, const float* sums,
                     float count, float* dx, int64_t lddx, mtt_stream_t stream);
int mtt_attn_delta(const float* dO, int64_t lddo, const void* o_hi, const void* o_lo, int64_t ldo, int32_t B, int32_t N,
                   int32_t H, int32_t head_dim, float* delta, mtt_stream_t stream);
int mtt_attn_softmax_bwd(const float* S, const float* dP, const float* delta, int64_t ld, int32_t BH, int32_t N, float scale,
                         const float* d_raw, int32_t T, void* ds_hi, void* ds_lo, void* pt_hi, void* pt_lo, void* dst_hi,
                         void* dst_lo, int64_t ldbf, mtt_stream_t stream);
int mtt_bilinear_bwd(const float* dy, int64_t lddy, int32_t nchw, int32_t B, int32_t h, int32_t w, int32_t C, int32_t H2,
                     int32_t W2, float* dx, int64_t lddx, int32_t accumulate, mtt_stream_t stream);
int mtt_gate_bwd(const float* x, int64_t ldx, int64_t x_group_rows, int64_t x_row_offset, const float* prompt_logits,
                 const float* chan_logits, int32_t task, int32_t B, int32_t T, int32_t N, int32_t H, int32_t C, int32_t gh,
                 int32_t gw, int32_t nh, int32_t nw, const float* dys, const float* dyc, int64_t lddy, float* dx,
                 int64_t lddx, float* d_prompt_logits, float* d_chan_logits, mtt_stream_t stream);
int mtt_chan_logits_bwd(const float* d_rc, const float* cp, const void* xn_hi, const void* xn_lo, int64_t ldx, int32_t B,
                        int32_t N, int32_t T, int32_t C, int32_t gh, int32_t gw, int32_t nh, int32_t nw, float* dcp,
                        float* dxn, int64_t lddx, mtt_stream_t stream);
int mtt_ctr_bwd(const float* dnew, const float* F, int32_t T, int64_t M, int32_t C, int64_t ld, int32_t rows_per_batch,
                const float* prompt_logits, int32_t B, int32_t H, int32_t N, const float* w0, const float* b0,
                const float* w2, float* dw_ws, float* d_prompt_logits, float* dw0, float* db0, float* dw2, float* db2,
                mtt_stream_t stream);
int mtt_im2col3x3_t(const float* x, int64_t ldx, int32_t B, int32_t H, int32_t W, int32_t C, void* out_hi, void* out_lo,
                    int64_t ldo, mtt_stream_t stream);
int mtt_im2col_patch_t(const float* img, int32_t B, int32_t Cin, int32_t H, int32_t W, int32_t patch, void* out_hi,
                       void* out_lo, int64_t ldo, mtt_stream_t stream);
int mtt_sumsq(const float* g, int64_t n, float* out, int32_t accumulate, mtt_stream_t stream);
int mtt_adam_step(float* p, const float* g, float* m, float* v, int64_t n, float lr, double beta1, double beta2, float eps,
                  float weight_decay, int32_t step, const float* gnorm_sq, float max_norm, float grad_scale,
                  mtt_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* MTT_B200_H_ */
