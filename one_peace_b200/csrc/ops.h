// Internal C++ declarations of the non-GEMM kernels' host launchers.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace opb {

int attention_fwd(const void* qkv, const float* bias, const uint8_t* key_pad, void* out, float* lse, float* ln_stats,
                  int B, int S, int H, int s_pad, long bias_bstride, cudaStream_t stream);
int attention_lut_fwd(const void* qkv, const float* lut, int lut_len, const int* code_row, const int* code_col,
                      const uint8_t* key_pad, void* out, float* lse, float* ln_stats, int B, int S, int H, int seg_split,
                      cudaStream_t stream);
// LUT form of the relative-position bias: bias[h][i][j] = lut[h][code_row[i] - code_col[j]] (see kernels.RelPosBias), zero
// between the two modality segments [0, seg_split) / [seg_split, S) of a concatenated sequence when seg_split > 0.
struct LutBias {
  const float* lut = nullptr;
  int lut_len = 0;
  const int* code_row = nullptr;
  const int* code_col = nullptr;
  int seg_split = 0;
};
// Short-sequence forward (csrc/attention_wgmma.cu): wgmma, one (sample, head) per work unit with the whole key row in
// registers.  attention_fwd / attention_lut_fwd dispatch to it for S <= kAttnShortMaxS when the LUT row (if any) fits its
// shared-memory slot; arguments as launch_fwd in attention.cu.
constexpr int kAttnShortMaxS = 224;
constexpr int kAttnShortMaxLut = 4096;
int attention_fwd_short(const void* qkv, const float* bias, const uint8_t* key_pad, void* out, float* lse, float* ln_stats,
                        int B, int S, int H, int s_pad, long bias_bstride, const LutBias& lb, cudaStream_t stream);
int relpos_lut_build(const float* table, const int* idx, float* lut, int L, int H, cudaStream_t stream);
// Decomposed relative-position terms of the detection backbone (csrc/relpos_decomp.cu, attention.cu): rel_h fp32
// [B, H, S, kh], rel_w [B, H, S, kw]; key_y / key_x int32 [S] the key grid coordinates, kh * kw == S.
struct DecompRel {
  const float* rel_h = nullptr;
  const float* rel_w = nullptr;
  const int* key_y = nullptr;
  const int* key_x = nullptr;
  int kh = 0, kw = 0;
};
constexpr int kDecompMaxK = 256;     // grid side limit of both kernels (shared-memory staging of the tables and rows)
int attention_decomp_fwd(const void* qkv, const float* lut, int lut_len, const int* code_row, const int* code_col,
                         const DecompRel& dr, void* out, float* lse, float* ln_stats, int B, int S, int H,
                         cudaStream_t stream);
int relpos_decomp_proj(const void* qkv, const float* rel_pos_h, const float* rel_pos_w, const int* pos_y, const int* pos_x,
                       float q_unscale, float* rel_h, float* rel_w, int B, int S, int H, int kh, int kw, cudaStream_t stream);
// Temporal attention of the video backbone (csrc/attention_temporal.cu): softmax over the T frames of each (clip, token, head)
// in the frame-major rows of qkv [Bv * T * N, 3 * H * 64]; out, ln_stats as attention_fwd.
constexpr int kTemporalMinT = 2;
constexpr int kTemporalMaxT = 32;
int attention_temporal_fwd(const void* qkv, void* out, float* ln_stats, int Bv, int T, int N, int H, cudaStream_t stream);
// its adjoint: dqkv [Bv * T * N, 3 * H * 64] from qkv, the forward output and its gradient (dq multiplied by q_scale)
int attention_temporal_bwd(const void* qkv, const void* out, const void* d_out, void* dqkv, int Bv, int T, int N, int H,
                           float q_scale, cudaStream_t stream);
// Multi-scale deformable attention (csrc/ms_deform_attn.cu), D = 32 channels per head; level_hw [L, 2] (H_l, W_l) and
// level_start [L] are host arrays, passed to the kernel by value.
constexpr int kMsdaMaxL = 4;
constexpr int kMsdaMaxP = 8;
int ms_deform_attn_fwd(const void* value, const float* proj, const float* ref, void* out, int N, int S_in, int Lq, int H,
                       int D, int L, int P, int L_ref, const int* level_hw, const int* level_start, cudaStream_t stream);
int ms_deform_attn_bwd(const void* value, const float* proj, const float* ref, const void* d_out, float* d_value,
                       float* d_proj, int N, int S_in, int Lq, int H, int D, int L, int P, int L_ref, const int* level_hw,
                       const int* level_start, cudaStream_t stream);
// Segmentation backbone (csrc/seg.cu): ConvFFN's per-level depthwise 3x3 conv + bias + GELU over token rows, and one
// output map (residual sum, bilinear ViT term, optional pixel-shuffled transposed conv, folded BatchNorm) to fp32 NCHW.
constexpr int kSegMaxL = 4;
int seg_dwconv_gelu(const void* x, const float* w, const float* bias, void* y, int B, int C, int n_levels,
                    const int* level_hw, cudaStream_t stream);
int seg_out_map(const float* c, long c_sample_rows, long c_row0, const float* x, long x_sample_rows, long x_row0, int gw,
                const float* extra, const float* scale, const float* shift, float* out, int B, int C, int Hl, int Wl,
                cudaStream_t stream);
int ln_stats_finalize(const float* partial, int parts, int rows, int dim, float eps, float* mu, float* rstd,
                      cudaStream_t stream);

struct LnRemap {
  int row_period = 0, row_valid = 0, out_period = 0, out_row_shift = 0;
  int group_in = 0, group_out = 0;
  int accumulate = 0;
  int raw = 0;
  float* mu_out = nullptr;
  float* rstd_out = nullptr;
};
int layernorm(const void* in, int in_dtype, long ld_in, void* out, int out_dtype, long ld_out, const float* gamma,
              const float* beta, int rows, int dim, float eps, int gelu, int merge_grid_w, const LnRemap& rm,
              cudaStream_t stream);
int pack_group_halo(const float* x, long ldx, void* out, int B, int T, int x_period, int x_row_shift, int out_period,
                    int halo, int dim, int group_in, int group_out, cudaStream_t stream);

int text_embed(const int64_t* tokens, const void* table, int table_dtype, const float* pos, const float* cls,
               float* x, uint8_t* pad_mask, int B, int T, int D, int pad_idx, cudaStream_t stream);
int image_patchify4(const void* img, int img_dtype, void* out, int B, int R, cudaStream_t stream);
int cls_row_init(const float* cls, const float* pos0, float* x, long batch_stride, int B, int D, cudaStream_t stream);
int relpos_bias_build(const float* table, const int64_t* bucket, float* bias, int S, int s_pad, int H,
                      long ld_bucket, cudaStream_t stream);
int audio_frame10(const void* wav, int wav_dtype, void* out, int B, long n_samples, long pitch, cudaStream_t stream);
int l2_normalize_rows(const float* x, long ldx, float* y, void* y_bf16, int rows, int D, cudaStream_t stream);
int zero_padded_rows(float* x, const uint8_t* pad_mask, int rows, int D, cudaStream_t stream);

int transpose_bf16(const void* in, long ld_in, void* out, int rows, int cols, cudaStream_t stream);
int split_bf16x3(const float* const* xs, void* const* outs, const int64_t* rows, const int* sides, int count, int d,
                 cudaStream_t stream);
int infonce_lse_gemm(const void* a_local, const void* b_all, const float* scale, int b, int n, int d, int target_offset, float* ws,
                     int n_valid, cudaStream_t stream);
int infonce_merge_reduce(const float* ws_a, const float* ws_b, int b, int n, int n_valid, float eps, int target_offset, float* lse_a,
                         float* lse_b, float* loss_ab, int* am_ab, float* out3, unsigned int* ticket, cudaStream_t stream);
long infonce_ws_floats(int b, int n);
int infonce_grad(const void* a_local, const void* b_all, const float* scale, const float* row_lse, int b, int n, int d,
                 int k_logits, int target_offset, float eps, void* g_ws, float* ws_gz, float* grad_a, int n_valid, float coef,
                 cudaStream_t stream);
int infonce_dscale(const float* ws_a, const float* ws_b, int b, int n, float* out, cudaStream_t stream);

// One entry per parameter tensor (device-resident table, 64 bytes; mirrored by ctypes in optim/adam_fused.py)
struct AdamTensor {
  void* p;         // parameter (fp32 or bf16)
  const void* g;   // gradient (fp32 or bf16)
  float* m;        // exp_avg
  float* v;        // exp_avg_sq
  float* master;   // optional fp32 master copy (nullptr: up-cast p)
  long numel;
  int group;
  int p_dtype;     // 0 fp32, 1 bf16
  int g_dtype;
  int pad_;
};
constexpr int kAdamMaxGroups = 128;
struct AdamGroups {
  float lr[kAdamMaxGroups];         // lr * lr_scale of the group (base_optimizer.py:8-13)
  float wd[kAdamMaxGroups];
  float bias_corr[kAdamMaxGroups];  // sqrt(1 - b2^t) / (1 - b1^t)
  float beta1, beta2, eps;
};
int adam_multi_step(const void* tensors, const int* chunk_tensor, const long* chunk_off, int n_chunks,
                    const AdamGroups& groups, const float* grad_scale, cudaStream_t stream);
int grad_norm_clip(const void* tensors, const int* chunk_tensor, const long* chunk_off, int n_chunks, float* partial,
                   float multiply_factor, float max_norm, float* out2, cudaStream_t stream);

// Adan (optim/adan.py:146-223): one entry per parameter tensor (device-resident table, 80 bytes; mirrored in optim/adan.py)
struct AdanTensor {
  void* p;         // parameter (fp32 or bf16)
  const void* g;   // gradient (fp32 or bf16)
  float* m;        // exp_avg
  float* n;        // exp_avg_diff
  float* v;        // exp_avg_sq
  float* pre;      // pre_grad (the previous step's scaled gradient)
  float* master;   // optional fp32 master copy (nullptr: up-cast p)
  long numel;
  int group;
  int p_dtype;     // 0 fp32, 1 bf16
  int g_dtype;
  int first;       // 1: the parameter's first step (adan.py:197-198): diff = 0, pre is written and never read
};
constexpr int kAdanMaxGroups = 128;
struct AdanGroups {
  float lr[kAdanMaxGroups];
  float wd[kAdanMaxGroups];
  float bc1[kAdanMaxGroups];        // 1 - b1^t with the group's step t
  float bc2[kAdanMaxGroups];        // 1 - b2^t
  float sqrt_bc3[kAdanMaxGroups];   // sqrt(1 - b3^t)
  int no_prox[kAdanMaxGroups];
  float beta1, beta2, beta3, eps;
};
int adan_multi_step(const void* tensors, const int* chunk_tensor, const long* chunk_off, int n_chunks,
                    const AdanGroups& groups, const float* grad_scale, cudaStream_t stream);

// ---- backward pass (backward.cu, attention_bwd.cu) ----
long bwd_ws_floats(int dim);
int layernorm_bwd(const void* x, int x_dtype, long ldx, const void* dy, int dy_dtype, long ld_dy, const float* gamma,
                  const float* beta, void* dx, int dx_dtype, long ld_dx, int accumulate, int rows, int dim, float eps,
                  int gelu, int dy_merge_w, float* ws, float* dgamma, float* dbeta, cudaStream_t stream);
int geglu_fwd(const void* gl, void* u, long rows, int F, cudaStream_t stream);
int geglu_bwd(const void* gl, const void* du, void* dgl, long rows, int F, cudaStream_t stream);
int gelu_fwd(const void* z, void* y, long rows, int F, cudaStream_t stream);
int gelu_bwd(const void* z, const void* dy, void* dz, long rows, int F, cudaStream_t stream);
int scale_resid_fwd(const float* x, const void* o, const float* gamma, const float* row_scale, float* out, long rows,
                    int n, cudaStream_t stream);
int scale_resid_bwd(const float* dx, const void* o, const float* gamma, const float* row_scale, void* d_o, float* ws,
                    float* dgamma, float* dbias, int rows, int n, int in_period, int in_valid, int in_shift,
                    cudaStream_t stream);
int batch_sum_f32(const float* in, long ld, float* out, int B, long n, int accumulate, cudaStream_t stream);
int l2_normalize_bwd(const float* x, long ldx, const float* dy, long ld_dy, float* dx, void* dx_bf16, int rows, int D,
                     cudaStream_t stream);
int window_gather(const void* in, void* out, int B, int t_in, int t_out, int stride, int kw, int pad, int groups, int cg,
                  cudaStream_t stream);
int window_scatter(const void* dwin, void* dx, int B, int t_in, int t_out, int stride, int kw, int pad, int groups, int cg,
                   cudaStream_t stream);
int text_embed_bwd(const float* dx, const int64_t* tokens, float* dtable, float* dpos, float* dcls, int B, int T, int D,
                   int pad_idx, cudaStream_t stream);
int colsum_bf16(const void* y, long ldy, float* ws, float* out, int rows, int n, cudaStream_t stream);
int attn_delta(const void* d_o, const void* o, float* delta, int B, int S, int H, cudaStream_t stream);
int relpos_bias_bwd(const float* dbias, const int64_t* bucket, float* dtable, int S, int s_pad, int H, long ld_bucket,
                    cudaStream_t stream);
// bias_t / dbias_t (optional, S <= 224, only when bias and dbias are null): the batch-shared bias and its gradient as TRANSPOSED
// tables (relpos_bias_transpose / relpos_dbias_fold).
int attention_bwd(const void* qkv, const void* out, const void* d_out, const float* bias, const uint8_t* key_pad,
                  const float* lse, float* delta, void* dqkv, float* dbias, int B, int S, int H, int s_pad,
                  float q_scale, long bias_bstride, cudaStream_t stream, const void* bias_t = nullptr,
                  float* dbias_t = nullptr);
int relpos_bias_transpose(const float* bias, void* bias_t, int S, int s_pad, int H, cudaStream_t stream);
int relpos_dbias_fold(const float* dbias_t, float* dbias, int S, int s_pad, int H, cudaStream_t stream);
int relpos_dbias_center(float* dbias, int S, int s_pad, int H, cudaStream_t stream);

// ---- pretraining path: row gathers, sample-dependent / block-diagonal dense relative-position bias (gather.cu) ----
int row_gather(const void* src, int src_dtype, long ld_src, const int64_t* idx, const float* fill, const float* add,
               long add_period, void* out, int out_dtype, long ld_out, long rows, int dim, cudaStream_t stream);
int row_scatter_add(const void* dout, int dout_dtype, long ld_dout, const int64_t* idx, float* dsrc, long ld_dsrc, long rows,
                    int dim, cudaStream_t stream);
int relpos_bias_block(const float* table, const int64_t* bucket, long ld_bucket, const int64_t* ids, long ids_ld, int Bb,
                      int n, int lo, float* bias, int S, int s_pad, int H, cudaStream_t stream);
int relpos_bias_block_bwd(const float* dbias, const int64_t* bucket, long ld_bucket, const int64_t* ids, long ids_ld, int Bb,
                          int n, int lo, float* dtable, int S, int s_pad, int H, cudaStream_t stream);

// ---- parameter preprocessing for the fused-LayerNorm GEMM chain (pack.cu) ----
int ln_fold(const void* W, int w_dtype, long ldw, const float* g, const float* beta, const float* bias_in, int N, int K,
            int interleave, void* out_w, long ldo, float* colsum, float* bias_out, cudaStream_t stream);

// ---- retrieval evaluation (recall.cu) ----
int topk10_rows(const float* sim, long ld, int* idx, float* val, int R, int C, cudaStream_t stream);
int recall_hits(const int* idx, const int64_t* cand_ids, const int64_t* row_ids, int R, int* hits3, cudaStream_t stream);

// csrc/classify.cu: attention pooling of the classification head and the classification criteria
int attn_pool_fwd(const void* kv, const float* q, const uint8_t* key_pad, void* out, float* lse, int B, int T, int d,
                  cudaStream_t stream);
int attn_pool_bwd(const void* kv, const float* q, const uint8_t* key_pad, const float* lse, const void* dout, void* dkv,
                  float* dq_ws, float* dq, int B, int T, int d, cudaStream_t stream);
int classify_loss(const float* logits, long ld, int rows, int n_valid, int mode, const int64_t* labels, const float* targets,
                  long ld_t, float eps, int num_choices, float* row_loss, float* dlogits, float* row_correct, float* out2,
                  unsigned int* ticket, cudaStream_t stream);

// csrc/grounding.cu: the box loss of refcoco_criterion and the hit counter of IouAcc
int refcoco_loss(const float* logits, long ld, const float* targets, int B, int nsentences, float* out, int* valid, float* giou,
                 float* dlogits, cudaStream_t stream);
int iou_acc(const float* hyps, long ld_h, const float* refs, long ld_r, int n, int* hits, int* row_hit, cudaStream_t stream);

// csrc/metrics.cu: the argmax hit counter of Accuracy, the sigmoid packing of MAP and the per-class average precision
int argmax_hits(const void* logits, int dtype, long ld, long cs, int n, int C, const void* targets, int tmode, long ldt,
                int64_t* hyp, float* score, cudaStream_t stream);
int sum_f64(const float* x, long n, double* out, cudaStream_t stream);
int sigmoid_pack(const void* logits, int dtype, long ld, long cs, const float* targets, long ldt, int n, int C, float* probs,
                 uint8_t* labels, long row_offset, int* flags, cudaStream_t stream);
long average_precision_ws_bytes(int N, int C);
int average_precision(const float* probs, const uint8_t* labels, int N, int C, void* ws, long ws_bytes, double* ap,
                      double* mean, int64_t* npos, cudaStream_t stream);

// csrc/vit_head.cu: the pooled head of OnePeaceViT (mean over the patch rows + fc_norm) and its adjoint
long token_mean_ln_ws_floats(int B, int S, int d);
int token_mean_ln_fwd(const float* x, long ld, int B, int S, int d, const float* gamma, const float* beta, float eps, float* ws,
                      long ws_floats, float* m, void* y, float* mean, float* rstd, cudaStream_t stream);
int token_mean_ln_bwd(const float* dy, const float* m, const float* mean, const float* rstd, const float* gamma, int B, int S,
                      int d, float* dgamma, float* dbeta, float* ws, float* dx, long ld_dx, cudaStream_t stream);

}  // namespace opb
