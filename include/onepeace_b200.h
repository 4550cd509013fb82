/*
 * onepeace_b200.h — C ABI of libonepeace_b200.so (hand-written sm_90a kernels for the ONE-PEACE
 * encoder / contrastive / optimizer hot path).
 *
 * Conventions (SURVEY.md §8b "What a C-ABI replacement exports"):
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer unless stated otherwise;
 *   - no ownership transfer: the caller (PyTorch) allocates inputs, outputs and workspaces;
 *   - kernels are enqueued on `stream` (a cudaStream_t passed as void*); calls are asynchronous;
 *   - return value: OPB_OK (0) or an OPB_ERR_* code; opb_status_string() names it.  The Python host
 *     raises RuntimeError on non-zero, matching the reference's "Python exceptions only" convention;
 *   - re-entrant; no global state except cached driver entry points and per-kernel attributes.
 *
 * Each entry point cites the reference code (under /root/reference/one_peace/) it replaces.
 */
#ifndef ONEPEACE_B200_H_
#define ONEPEACE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OPB_OK 0
#define OPB_ERR_INVALID 1      /* bad shape / alignment / null pointer */
#define OPB_ERR_CUDA 2         /* CUDA runtime / driver error at launch */
#define OPB_ERR_UNSUPPORTED 3  /* shape outside what the kernels were built for */

/* dtype tags */
#define OPB_F32 0
#define OPB_BF16 1

/* GEMM epilogues */
#define OPB_EPI_STORE_BF16 0
#define OPB_EPI_GEGLU_BF16 1
#define OPB_EPI_RESID_F32 2
#define OPB_EPI_STORE_F32 3
#define OPB_EPI_GELU_BF16 4

/* ABI version / status names: the host raises RuntimeError on any non-zero status — the reference's error convention is
 * Python exceptions only (e.g. transformer_encoder.py:136-137, multihead_attention.py:55-57; SURVEY.md 8b). */
int opb_abi_version(void);
const char* opb_status_string(int status);

/*
 * C = epilogue(A[M,K] . B[N,K]^T), bf16 operands (row pitches lda/ldb in elements), fp32 accumulate in
 * registers via wgmma, TMA-fed.  Replaces the nn.Linear / F.linear calls of
 *   models/transformer/multihead_attention.py:103-105,124 (q/k/v/out projections),
 *   models/transformer/transformer_layer.py:54-67,149-157 (GeGLU wi_0/wi_1, fc2),
 *   models/one_peace/one_peace_retrieval.py:114-117 (*_proj),
 * and, on patchified inputs, the stride==kernel convolutions of models/adapter/image.py:66-75 and the
 * Conv1d stacks of models/adapter/audio.py:46-80,254-311.
 *   epi = OPB_EPI_STORE_BF16 : out_bf16 = (acc + bias[n]) * colscale[n]
 *         OPB_EPI_GELU_BF16  : out_bf16 = gelu((acc + bias[n]) * colscale[n])
 *         OPB_EPI_GEGLU_BF16 : out_bf16[:, t*128+j] = gelu(acc[:, t*256+j]) * acc[:, t*256+128+j]   (N/2 cols)
 *         OPB_EPI_RESID_F32  : out_f32 = resid + gamma[n] * (acc + bias[n])   (transformer_layer.py:70-88)
 *         OPB_EPI_STORE_F32  : out_f32 = acc + bias[n]
 * bias/colscale/gamma/resid may be NULL.  Row remapping: if out_group > 0,
 *   out_row = (m / out_group) * out_group_stride + (m % out_group) + out_row_offset;
 * if resid_period > 0 the residual row is (m % resid_period) + resid_row_offset (broadcast table),
 * otherwise it is out_row.  If out_group_valid > 0, rows with (m % out_group) >= out_group_valid are computed but
 * not stored (allocation slack rows of the audio frame buffers).  cta_group: 0, 1 or 2 (accepted for compatibility; every GEMM runs 128x256 tiles).
 * resid may overlap the output only as the in-place update (resid == out, ldr == ldo, resid_period == 0) and must not
 * overlap the bf16 copy of opb_gemm_bf16_ex; any other overlap returns OPB_ERR_INVALID before anything is launched.
 */
int opb_gemm_bf16(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K, int epi, void* out,
                  int64_t ldo, const float* bias, const float* colscale, const float* gamma, const float* resid,
                  int64_t ldr, int out_group, int out_group_stride, int out_row_offset, int out_group_valid,
                  int resid_period, int resid_row_offset, int cta_group, void* stream);

/*
 * Grouped Conv1d over channel-last activations as one grouped sliding-window wgmma GEMM (the positional conv
 * stack of models/adapter/audio.py:57-80: Conv1d(1536,1536,k=19,pad=9,groups=16)):
 *   out[r, g*n_per_group + n] = epi( bias + sum_{j<taps} sum_{c<c_pad} X[r + j, g, c] * W[g*n_per_group + n, j*c_pad + c] )
 * X bf16 [rows + taps - 1, groups, c_pad] (c_pad % 64 == 0; the caller supplies the zero halo / channel padding),
 * W bf16 [groups*n_per_group, taps*c_pad], out bf16 or fp32 [rows, groups*n_per_group] per `epi`
 * (OPB_EPI_STORE_BF16 / GELU_BF16 / STORE_F32 / RESID_F32 with the same optional vectors as opb_gemm_bf16).
 */
int opb_grouped_conv1d_bf16(const void* X, const void* W, int rows, int groups, int c_pad, int taps, int n_per_group,
                            int epi, void* out, int64_t ldo, const float* bias, void* stream);

/*
 * Fused self-attention: out = softmax_fp32(q k^T + bias[h] (+ -inf on padded keys)) v.
 * Replaces models/transformer/multihead_attention.py:107-115 together with the (B,H,S,S) bias
 * materialisation of models/transformer/transformer_encoder.py:144-162.
 *   qkv  bf16 [B*S, 3*H*64] (q | k | v, q already scaled), out bf16 [B*S, H*64]
 *   bias fp32 [H, S, s_pad] or NULL (s_pad even, >= S);  key_pad uint8 [B, S] (1 = pad) or NULL
 *   bias_batch_stride  0: one table shared by the batch; > 0: element stride between per-sample tables [B, H, S, s_pad]
 *        (the preserve_ids gathers of the pretraining student passes make the bias sample-dependent,
 *        models/adapter/text.py:92-101, image.py:188-204)
 *   lse  fp32 [B, H, S] or NULL (log-sum-exp per query row, kept for the backward pass)
 *   ln_stats fp32 [H, B*S, 2] or NULL: per-(head, row) partial (sum, sum of squares) of the output row, from which
 *        opb_ln_stats_finalize derives the statistics of the inner LayerNorm (multihead_attention.py:122-123) that
 *        the out_proj GEMM then applies in its epilogue
 */
int opb_attention_fwd(const void* qkv, const float* bias, const uint8_t* key_pad, void* out, float* lse,
                      float* ln_stats, int B, int S, int H, int s_pad, int64_t bias_batch_stride, void* stream);

/*
 * Self-attention with the LUT-form bias (vision, text).  Same kernel and math as opb_attention_fwd; the relative-
 * position bias is given in LUT form:  bias[h][i][j] = lut[h][code_row[i] - code_col[j]]  (lut fp32 [H, lut_len],
 * code_row / code_col int32 [S]; built by the adapters from rel_pos_table + rp_bucket — every ONE-PEACE bucket scheme is
 * a function of a per-position code difference plus three CLS ids, adapter/text.py:18-29,62-68, image.py:19-34).
 * lse / ln_stats as in opb_attention_fwd (either may be NULL).
 * seg_split > 0: the sequence is a concatenation of two modalities ('vl' / 'al', transformer_encoder.py:116-137) with
 * rows [0, seg_split) and [seg_split, S); the bias is block-diagonal (zero between modalities, :148-158).
 * lut_max fp32 [H] = max_l lut[h][l] (for seg_split > 0: max(that, 0)): the kernel shifts the soft-max by the upper bound
 * max_j q.k_j + lut_max[h] of the biased row maximum, so the row maximum is found without touching the bias.
 * Any S and lut_len: the kernel reads the LUT from global memory.  The adapters choose this form for S <= 384 and
 * opb_attention_fwd with the dense table above that.
 */
int opb_attention_tc_fwd(const void* qkv, const float* lut, const float* lut_max, int lut_len, const int32_t* code_row,
                         const int32_t* code_col, const uint8_t* key_pad, void* out, float* lse, float* ln_stats, int B,
                         int S, int H, int seg_split, void* stream);

/* lut[h][l] = table[idx[l]][h]  (table fp32 [num_buckets, H], idx int32 [L], lut fp32 [H, L]): the rel_pos_table lookup of
 * adapter/text.py:84-91 / image.py:164-171 restricted to the distinct (code_row - code_col) values. */
int opb_relpos_lut_build(const float* table, const int32_t* idx, float* lut, int L, int H, void* stream);

/*
 * Decomposed relative position of the detection backbone (one_peace_vision/det/models/onepeace.py:204-207, detectron2's
 * add_decomposed_rel_pos), on a kh x kw grid of S = kh * kw tokens per sequence, head_dim 64.
 *   opb_relpos_decomp_proj : rel_h fp32 [B, H, S, kh], rel_w fp32 [B, H, S, kw] with
 *       rel_h[b][h][i][ky] = q . rel_pos_h[pos_y[i] - ky + kh - 1],  rel_w[b][h][i][kx] = q . rel_pos_w[pos_x[i] - kx + kw - 1]
 *     where q = q_unscale * qkv[b * S + i, h * 64 : h * 64 + 64] (the bf16 q columns carry head_dim^-0.5; the reference
 *     uses the unscaled q, so q_unscale = 8).  rel_pos_h fp32 [2 kh - 1, 64], rel_pos_w fp32 [2 kw - 1, 64]; pos_y / pos_x
 *     int32 [S] the grid position of each row (any row order).  fp32 products, summed over the 64 channels in order.
 *   opb_attention_decomp_fwd : opb_attention_tc_fwd's LUT-form attention (no key padding, no seg_split) with
 *     rel_h[b][h][i][key_y[j]] + rel_w[b][h][i][key_x[j]] added to logit (i, j) after the LUT bias; key_y / key_x int32
 *     [S] the key grid coordinates.  out / lse / ln_stats as in opb_attention_fwd (lse and ln_stats may be NULL).
 * Both need kh * kw == S and 1 <= kh, kw <= 256.  A row position or key coordinate outside the grid yields NaN in the
 * terms or logits it touches (never an out-of-bounds read).
 */
int opb_relpos_decomp_proj(const void* qkv, const float* rel_pos_h, const float* rel_pos_w, const int32_t* pos_y,
                           const int32_t* pos_x, float q_unscale, float* rel_h, float* rel_w, int B, int S, int H, int kh,
                           int kw, void* stream);
int opb_attention_decomp_fwd(const void* qkv, const float* lut, int lut_len, const int32_t* code_row,
                             const int32_t* code_col, const float* rel_h, const float* rel_w, const int32_t* key_y,
                             const int32_t* key_x, int kh, int kw, void* out, float* lse, float* ln_stats, int B, int S,
                             int H, void* stream);

/*
 * Temporal attention of the video backbone (one_peace_vision/video/mmaction_custom/models/backbones/onepeace.py:331-337 with
 * num_tadapter = 1: rearrange 'n (b t) d -> t (b n) d', self_attn, rearrange back).  It replaces the reference's two
 * rearranges and its bmm / softmax / bmm over Bv * N sequences of T frames.
 *   qkv : bf16 [Bv * T * N, 3 * H * 64], frame-major rows (row (b * T + t) * N + n), q pre-scaled by head_dim^-0.5.
 *   out : bf16 [Bv * T * N, H * 64], the same rows: out[(b, t, n), h] = softmax_t'(q_t . k_t') v_t' over the T frames of
 *         (b, n), no bias, no padding.
 *   ln_stats : fp32 [H, Bv * T * N, 2], opb_attention_fwd's per-(head, row) (sum, sum of squares) records of the fp32 output
 *         values, for ln_partial = (ln_stats, H, H * 64, eps) of the out_proj GEMM.
 * Needs 2 <= T <= 32, Bv, N, H >= 1, non-null 16-byte aligned qkv / out and an 8-byte aligned ln_stats; anything else
 * returns OPB_ERR_INVALID before a launch.
 */
int opb_attention_temporal_fwd(const void* qkv, void* out, float* ln_stats, int Bv, int T, int N, int H, void* stream);

/*
 * Adjoint of opb_attention_temporal_fwd.  qkv is the forward's operand, out its output and d_out the gradient of out, all in
 * the same frame-major rows and read in place at a stride of N rows.  Writes every element of dqkv bf16
 * [Bv * T * N, 3 * H * 64] = [dq | dk | dv], dq multiplied by q_scale (the gradient of the un-scaled projection, as
 * opb_attention_bwd).  P is recomputed with the forward's arithmetic, so no log-sum-exp is needed.  No atomics: repeated
 * launches are bit-identical.  Needs 2 <= T <= 32, Bv, N, H >= 1 and non-null 16-byte aligned pointers; anything else
 * returns OPB_ERR_INVALID before a launch.
 */
int opb_attention_temporal_bwd(const void* qkv, const void* out, const void* d_out, void* dqkv, int Bv, int T, int N, int H,
                               float q_scale, void* stream);

/*
 * Multi-scale deformable attention core (one_peace_vision/seg/ops, MSDeformAttn) with D = 32 channels per head, fused with
 * the soft-max over each head's L * P logits and the sampling locations loc = ref + off / (W_l, H_l).
 *   value : bf16 [N * S_in, H * 32], the value_proj output; level l of sample n owns rows n * S_in + start_l + y * W_l + x.
 *   proj  : fp32 [N * Lq, 3 * H * L * P] = [offsets (h, l, p, xy) | logits (h, l * P + p)], the reference's orders.
 *   ref   : fp32 [N * Lq, L_ref, 2] reference points (x, y), L_ref = 1 (shared by every level) or L.
 *   level_hw [L, 2] = (H_l, W_l) and level_start [L]: HOST int32 arrays, passed to the kernel by value (no device copy).
 *   out   : bf16 [N * Lq, H * 32] = sum over (l, p) of softmax(logits)_lp * bilinear(value_l, loc * (W_l, H_l) - 0.5), taps
 *           outside the level read as zero (grid_sample, align_corners = False, padding_mode = zeros); fp32 accumulation.
 * No atomics, one write per output element: repeated launches are bit-identical.  Needs D == 32, 1 <= L <= 4, 1 <= P <= 8,
 * L_ref in {1, L}, N, S_in, Lq, H >= 1, every level inside S_in and non-null 16-byte aligned device pointers; anything else
 * returns OPB_ERR_INVALID before a launch.
 */
int opb_ms_deform_attn_fwd(const void* value, const float* proj, const float* ref, void* out, int N, int S_in, int Lq, int H,
                           int D, int L, int P, int L_ref, const int32_t* level_hw, const int32_t* level_start, void* stream);

/*
 * Adjoint of opb_ms_deform_attn_fwd for d_out bf16 [N * Lq, H * 32], with the forward's arguments.
 *   d_value : fp32 [N * S_in, H * 32], ACCUMULATED (the caller zeroes it): a_lp * tap weight * d_out, scattered with fp32
 *             vector atomics, so repeats differ in the last bits.
 *   d_proj  : fp32 [N * Lq, 3 * H * L * P], every element written: the offset gradients d_loc / (W_l, H_l) (taps outside
 *             the level contribute nothing) and the logit gradients a * (dA - sum a dA).  No atomics: bit-identical repeats.
 * No gradient of the reference points.  Argument checks as the forward.
 */
int opb_ms_deform_attn_bwd(const void* value, const float* proj, const float* ref, const void* d_out, float* d_value,
                           float* d_proj, int N, int S_in, int Lq, int H, int D, int L, int P, int L_ref,
                           const int32_t* level_hw, const int32_t* level_start, void* stream);

/*
 * Segmentation backbone (one_peace_vision/seg, OnePeaceAdapter).
 *   opb_seg_dwconv_gelu : ConvFFN's depthwise conv (adapter_modules.py:69-84) + bias + exact GELU over token rows.
 *     x, y bf16 [B * T, C], T = sum_l H_l W_l; each sample's rows hold the n_levels levels back to back, level l a row-major
 *     H_l x W_l grid (level_hw [n_levels, 2] = (H_l, W_l), a HOST int32 array passed by value).  Each level is convolved on
 *     its own grid with zero padding at its border:  y = gelu_erf(sum_{ky, kx} x[tap] * w[ky * 3 + kx, c] + bias[c]), fp32
 *     products summed in tap order.  w fp32 [9, C] (the conv weight [C, 1, 3, 3] rearranged tap-major), bias fp32 [C].
 *     No atomics: repeats are bit-identical.  Needs B >= 1, C % 8 == 0, 1 <= n_levels <= 4, positive level sides and
 *     non-null 16-byte aligned pointers, else OPB_ERR_INVALID before a launch.
 *   opb_seg_out_map : one output map of onepeace_adapter.py:114-134, fp32 NCHW out [B, C, Hl, Wl]:
 *       out[b, c, y, x] = scale[c] * (extra[b, y, x, c] + c_l[b, y, x, c] + up[b, c, y, x]) + shift[c]
 *     c_l : fp32 rows, pixel (y, x) of sample b at row b * c_sample_rows + c_row0 + y * Wl + x, C wide.
 *     up  : the bilinear resize (align_corners = False, scale gw / Hl and gw / Wl) of the gw x gw grid of fp32 rows
 *           b * x_sample_rows + x_row0 + i * gw + j of x.
 *     extra : NULL, or fp32 [B * (Hl / 2) * (Wl / 2), 4 * C], the transposed conv (k = s = 2) as one GEMM with columns
 *           (dy, dx, c): pixel (y, x) reads row (b, y / 2, x / 2), column ((y % 2) * 2 + x % 2) * C + c.
 *     scale / shift fp32 [C]: the eval BatchNorm folded.  C % 32 == 0, rows inside their samples, even Hl and Wl with
 *     extra, else OPB_ERR_INVALID before a launch.
 */
int opb_seg_dwconv_gelu(const void* x, const float* w, const float* bias, void* y, int B, int C, int n_levels,
                        const int32_t* level_hw, void* stream);
int opb_seg_out_map(const float* c, int64_t c_sample_rows, int64_t c_row0, const float* x, int64_t x_sample_rows,
                    int64_t x_row0, int gw, const float* extra, const float* scale, const float* shift, float* out, int B,
                    int C, int Hl, int Wl, void* stream);

/*
 * GEMM with the full epilogue description (superset of opb_gemm_bf16).  Adds the fused-LayerNorm form
 *   LN(x) W^T + b  =  rstd[m] * (acc - mu[m] * colsum[n]) + bias'[n]
 * where A holds the UN-normalised rows (bf16), B = W * diag(ln_weight) (bf16), colsum[n] = sum_k B[n,k],
 * bias'[n] = sum_k ln_bias[k] W[n,k] + b[n]; and the side outputs that feed the NEXT LayerNorm: stats_out
 * [ceil(N/256) (RESID) or 2*N/256 (GEGLU: one record per 64 output columns), M, 2] partial (sum, sum of squares)
 * of the stored values, and out_bf16 (a bf16
 * copy of the fp32 output of OPB_EPI_RESID_F32).  This replaces the four LayerNorm passes per encoder layer of
 * models/transformer/transformer_layer.py:185,202 / multihead_attention.py:122-123 / transformer_layer.py:154.
 */
typedef struct opb_gemm_args {
  const void* A; int64_t lda;
  const void* B; int64_t ldb;
  int32_t M, N, K, epi;
  void* out; int64_t ldo;
  const float* bias; const float* colscale; const float* gamma; const float* resid; int64_t ldr;
  int32_t out_group, out_group_stride, out_row_offset, out_group_valid, resid_period, resid_row_offset;
  const float* ln_mu; const float* ln_rstd; const float* ln_colsum;
  float* stats_out;
  void* out_bf16; int64_t ldo_bf16;
  int32_t cta_group; int32_t reserved;
  /* optional fp32 scratch of >= 256 * N * 4 bytes: lets OPB_EPI_RESID_F32 GEMMs schedule the partially filled last
   * row of tiles as split-K pieces (removes a whole wave when (M / 256) * ceil(N / 256) just fits the SM pairs) */
  void* workspace; int64_t workspace_bytes;
  /* alternative to ln_mu / ln_rstd: partial (sum, sum of squares) records [ln_parts, M, 2] of the A rows written by the
   * producing kernel; each epilogue thread reduces its row's records itself (no opb_ln_stats_finalize launch) */
  const float* ln_partial; int32_t ln_parts; int32_t ln_dim; float ln_eps; int32_t reserved2;
} opb_gemm_args;
/* opb_gemm_bf16 plus the fused-LayerNorm / statistics / bf16-copy options: one call = LayerNorm + Linear (+ GeGLU |
 * + LayerScale + residual) of transformer_layer.py:185-224 / multihead_attention.py:103-107,122-124. */
int opb_gemm_bf16_ex(const opb_gemm_args* args, void* stream);

/*
 * Row statistics + cast: out_bf16[r,:] = bf16(x[r,:]) (UN-normalised), mu[r] = mean, rstd[r] = 1/sqrt(var + eps).
 * Prepares the first encoder layer's input for the fused-LayerNorm GEMMs (later layers get the same three tensors
 * from the preceding GEMM's epilogue): the statistics half of self_attn_layer_norm, transformer_layer.py:185,
 * components.py:23-26.
 */
int opb_row_stats_cast(const float* x, int64_t ld_in, void* out_bf16, int64_t ld_out, float* mu, float* rstd,
                       int rows, int dim, float eps, void* stream);

/* mu[r], rstd[r] from `parts` partial (sum, sumsq) records per row (layout [parts, rows, 2]); deterministic order.
 * Statistics of the FFN LayerNorm over the 6144-wide GeGLU output (transformer_layer.py:154) and of the inner attention
 * LayerNorm (multihead_attention.py:122-123) when they are not reduced inside the consumer GEMM. */
int opb_ln_stats_finalize(const float* partial, int parts, int rows, int dim, float eps, float* mu, float* rstd,
                          void* stream);

/*
 * Row LayerNorm (torch.nn.LayerNorm semantics; models/components.py:23-26) with optional exact GELU and
 * optional 2x2 pixel-merge scatter (models/adapter/image.py:37-47 LayerNorm2D + the following stride-2
 * conv's patch gather).  in/out dtype tags: OPB_F32 / OPB_BF16; gamma/beta fp32 or both NULL.
 * Sequence remap (row_period > 0): input row = b*row_period + t, rows with t >= row_valid are skipped, output row =
 * b*out_period + t + out_row_shift.  Channel-group padding (group_in > 0): output column = (c / group_in) * group_out
 * + c % group_in.  accumulate (fp32 output only): out += y.  These serve the audio adapter's halo / CLS layouts
 * (models/adapter/audio.py:57-80,194-197).
 */
int opb_layernorm(const void* in, int in_dtype, int64_t ld_in, void* out, int out_dtype, int64_t ld_out,
                  const float* gamma, const float* beta, int rows, int dim, float eps, int gelu, int merge_grid_w,
                  int row_period, int row_valid, int out_period, int out_row_shift, int group_in, int group_out,
                  int accumulate, void* stream);

/*
 * fp32 feature rows -> bf16 grouped / channel-padded / halo'd operand of opb_grouped_conv1d_bf16 (the zero padding of
 * Conv1d(padding = k // 2, groups = 16) in adapter/audio.py:57-80):
 * out[b, halo + t, g, :group_in] = x[b*x_period + x_row_shift + t, g*group_in:(g+1)*group_in] (padding columns zero).
 */
int opb_pack_group_halo(const float* x, int64_t ldx, void* out, int B, int T, int x_period, int x_row_shift,
                        int out_period, int halo, int dim, int group_in, int group_out, void* stream);

/*
 * Text adapter front end: x[b,0,:] = cls + pos[0]; x[b,1+t,:] = embed[tok[b,t]] + pos[1+t]; rows of padded
 * tokens are zeroed and flagged in pad_mask.  Replaces models/adapter/text.py:125-129,144-146,153 and the
 * pad zeroing of models/transformer/transformer_encoder.py:139-142.
 *   tokens int64 [B,T]; table [V,D] (table_dtype OPB_F32/OPB_BF16); pos fp32 [>=T+1, D]; cls fp32 [D]
 *   x fp32 [B, T+1, D]; pad_mask uint8 [B, T+1]
 */
int opb_text_embed(const int64_t* tokens, const void* table, int table_dtype, const float* pos, const float* cls,
                   float* x, uint8_t* pad_mask, int B, int T, int D, int pad_idx, void* stream);

/*
 * im2col of the 4x4 / stride-4 stem convolution (models/adapter/image.py:67):
 * out[(b,oy,ox), (c,ky,kx)] = img[b,c,4oy+ky,4ox+kx], bf16 [B*(R/4)^2, 48]; img [B,3,R,R] fp32 or bf16.
 */
int opb_image_patchify4(const void* img, int img_dtype, void* out, int B, int R, void* stream);

/* x[b, 0, :] = cls + pos0 for every batch element (image.py:239-240,253; audio.py:195-197). */
int opb_cls_row_init(const float* cls, const float* pos0, float* x, int64_t batch_stride, int B, int D,
                     void* stream);

/*
 * Relative-position bias for one forward: bias[h,i,j] = table[bucket[i*ld_bucket + j], h], i,j < S, written as
 * fp32 [H, S, s_pad] (zero padded columns).  Replaces get_rel_pos_bias (text.py:84-91, image.py:164-171,
 * audio.py:124-131) and the per-batch expansion in transformer_encoder.py:144-158.
 */
int opb_relpos_bias_build(const float* table, const int64_t* bucket, float* bias, int S, int s_pad, int H,
                          int64_t ld_bucket, void* stream);

/*
 * im2col of the first wav2vec conv (k=10, s=5, C_in=1; models/adapter/audio.py:270-284):
 * out[(b,t), j] = wav[b, 5t+j] (j<10), zero padded to 16 columns, bf16 [B*pitch, 16]; wav [B, n_samples].
 */
int opb_audio_frame10(const void* wav, int wav_dtype, void* out, int B, int64_t n_samples, int64_t pitch,
                      void* stream);

/* y = x / max(||x||_2, 1e-12) per row (one_peace_retrieval.py:116); y fp32 [rows,D], optional bf16 copy. */
int opb_l2_normalize_rows(const float* x, int64_t ldx, float* y, void* y_bf16, int rows, int D, void* stream);

/* x[row,:] = 0 where pad_mask[row] (transformer_encoder.py:139-142). */
int opb_zero_padded_rows(float* x, const uint8_t* pad_mask, int rows, int D, void* stream);

/* bf16 [rows, cols] (row pitch ld_in) -> [cols, rows]: lays the gathered embeddings out K-major for the gradient GEMM of
 * criterions/image_text_retrieval_loss.py:95-96 (autograd of `logits @ logits_all.t()`), and every dW = dY^T X operand of
 * the encoder backward. */
int opb_transpose_bf16(const void* in, int64_t ld_in, void* out, int rows, int cols, void* stream);

/*
 * fp32 [rows, d] -> bf16 [rows, 3d] split x = hi + lo: side 0 -> [hi|hi|lo] (local operand), side 1 -> [hi|lo|hi]
 * (gathered operand).  One K = 3d GEMM then gives hi.hi + hi.lo + lo.hi, i.e. logits accurate to ~2^-16 — the similarity
 * matrices of criterions/image_text_retrieval_loss.py:95-96 and metrics/recall.py:33 are fp32 products in the reference.
 * 1 <= count <= 4 tensors of the same d in one launch; xs / outs / rows / sides: HOST arrays of count.
 */
int opb_split_bf16x3(const float* const* xs, void* const* outs, const int64_t* rows, const int* sides, int count, int d,
                     void* stream);

/*
 * Cross-modal InfoNCE (criterions/image_text_retrieval_loss.py:91-112, :16-26; pretrain twin
 * image_text_pretrain_loss.py:164-185).  One direction: a_local bf16 [b,k] (this rank's rows), b_all bf16 [n,k] (all ranks'
 * rows of the other modality in rank-major order, detached); k = d for plain bf16 operands or 3d for the
 * opb_split_bf16x3 layout; scale = device scalar exp(clamp(logit_scale)).
 * Targets: row i -> column i + target_offset (target_offset = rank * b).
 * n_valid (0 = n): number of real classes when b_all was zero-padded to n % 8 == 0 rows; columns >= n_valid are ignored
 * (-inf logits, zero gradient).  coef (0 = 1 / (2 b)): weight of a row's loss in the gradient.  These two serve the
 * single-direction DCL loss (image_text_pretrain_loss.py:187-208: masked student rows vs the local batch's teacher rows,
 * mean over rows -> coef = 1 / b), which is the same tiled similarity + log-softmax as one InfoNCE direction.
 *   opb_infonce_ws_floats     size (floats) of the partial workspace `ws` of one direction
 *   opb_infonce_lse_gemm      the LSE_PARTIAL GEMM of one direction: per-tile row partials into ws
 *   opb_infonce_merge_reduce  merges one or both directions' partials (ws_b = row_lse_b = NULL: one direction; dirs = 1 or 2)
 *                             into row_lse [b] per direction (needed by opb_infonce_grad) and writes out3 = {sum of the
 *                             dirs * b row losses / (dirs * b), #correct a->b, #correct b->a (0 for one direction)} in one
 *                             launch: the last block to finish performs the fixed-order reduction.  loss_ab fp32 [dirs * b]
 *                             (label-smoothed NLL per row) and argmax_ab int32 [dirs * b] hold direction a's rows, then b's;
 *                             ticket = one uint32 that must be zero on entry and is left at zero.
 *   opb_infonce_grad          grad_a fp32 [b,d] = d(loss)/d(a_local) (local rows only; no gradient to b_all, :30-38);
 *                             b_all is read in place as the MN-major operand of the G . B_all product (no transposed copy);
 *                             g_ws bf16 [b,n] scratch; ws_gz [ceil(n/256), b]
 *   opb_infonce_dscale        out[0] = d(loss)/d(logit_scale) from the two directions' ws_gz
 */
int64_t opb_infonce_ws_floats(int b, int n);
int opb_infonce_lse_gemm(const void* a_local, const void* b_all, const float* scale, int b, int n, int d, int target_offset,
                         float* ws, int n_valid, void* stream);
int opb_infonce_merge_reduce(const float* ws_a, const float* ws_b, int b, int n, int n_valid, float label_smoothing,
                             int target_offset, float* row_lse_a, float* row_lse_b, float* loss_ab, int* argmax_ab, float* out3,
                             uint32_t* ticket, void* stream);
int opb_infonce_grad(const void* a_local, const void* b_all, const float* scale, const float* row_lse, int b, int n, int d,
                     int k_logits, int target_offset, float label_smoothing, void* g_ws, float* ws_gz, float* grad_a,
                     int n_valid, float coef, void* stream);
int opb_infonce_dscale(const float* ws_gz_a, const float* ws_gz_b, int b, int n, float* out, void* stream);

/*
 * Fused multi-tensor Adam (optim/adam.py:173-253 python form; optional fp32 master as optim/adam_fused.py:45-50)
 * and global grad-norm + clip coefficient (optim/fp16_optimizer_memory_efficent.py:96-116, bf16 branch).
 *   tensors       device array of n_tensors records {void* p; const void* g; float* m; float* v; float* master;
 *                 int64 numel; int32 group, p_dtype, g_dtype, pad}  (64 bytes each)
 *   chunk_tensor / chunk_off   device arrays [n_chunks]: tensor index and element offset of every 8192-element chunk
 *   lr, wd, bias_corr          HOST arrays [n_groups <= 128]: lr*lr_scale, weight decay, sqrt(1-b2^t)/(1-b1^t)
 *   grad_scale    device scalar multiplied into every gradient (NULL = 1): out2[1] of opb_grad_norm_clip
 * opb_grad_norm_clip: out2[0] = multiply_factor * ||g||_2, out2[1] = multiply_factor * min(1, max_norm/(norm+1e-6))
 * (max_norm <= 0: no clipping; a NaN norm gives a NaN out2[1]); `partial` is an [n_chunks] fp32 scratch.  Deterministic
 * reduction order.
 */
int opb_adam_chunk_elems(void);
int opb_adam_multi_step(const void* tensors, const int32_t* chunk_tensor, const int64_t* chunk_off, int n_chunks,
                        const float* lr, const float* wd, const float* bias_corr, int n_groups, float beta1,
                        float beta2, float eps, const float* grad_scale, void* stream);
int opb_grad_norm_clip(const void* tensors, const int32_t* chunk_tensor, const int64_t* chunk_off, int n_chunks,
                       float* partial, float multiply_factor, float max_norm, float* out2, void* stream);

/*
 * Fused multi-tensor Adan step (optim/adan.py:146-223, registered as `adan` at :53; one launch per step, same
 * 8192-element chunk table as opb_adam_multi_step).  Per element, fp32, each operation rounded on its own:
 *   g = grad * grad_scale;  diff = g - pre_grad (0 on a parameter's first step, :197-198);  u = g + b2 diff (:205)
 *   m = b1 m + (1-b1) g;  n = b2 n + (1-b2) diff;  v = b3 v + (1-b3) u^2                              (:206-208)
 *   upd = (m / bc1 + (b2 n) / bc2) / (sqrt(v) / sqrt_bc3 + eps)                                       (:210-211)
 *   no_prox = 0: p = (p - lr upd) / (1 + lr wd);  no_prox = 1: p = p (1 - lr wd) - lr upd            (:213-218)
 *   pre_grad = g                                                                                       (:220)
 *   tensors       device array of records {void* p; const void* g; float* m (exp_avg); float* n (exp_avg_diff);
 *                 float* v (exp_avg_sq); float* pre_grad; float* master; int64 numel; int32 group, p_dtype, g_dtype,
 *                 first}  (80 bytes each; dtype 0 fp32, 1 bf16; master NULL = up-cast p; first = 1: diff = 0 and
 *                 pre_grad is only written, it may hold anything)
 *   lr, wd, no_prox, bc1 (1 - b1^t), bc2 (1 - b2^t), sqrt_bc3 (sqrt(1 - b3^t))   HOST arrays [n_groups <= 128], t the
 *                 group's step count (:160-169)
 *   grad_scale    device scalar multiplied into every gradient (NULL = 1); pre_grad stores the scaled gradient
 * Null pointers give OPB_ERR_INVALID and a group count outside 1..128 OPB_ERR_UNSUPPORTED, before any CUDA call.
 */
int opb_adan_multi_step(const void* tensors, const int32_t* chunk_tensor, const int64_t* chunk_off, int n_chunks,
                        const float* lr, const float* wd, const int32_t* no_prox, const float* bc1, const float* bc2,
                        const float* sqrt_bc3, int n_groups, float beta1, float beta2, float beta3, float eps,
                        const float* grad_scale, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Backward pass of the encoder layer (autograd of models/transformer/transformer_layer.py:165-228 and
 * multihead_attention.py:103-126; the reference relies on torch autograd, these are the hand-written adjoints).
 * Column-reduction entry points take `ws`: fp32 scratch of opb_bwd_ws_floats(dim) floats.
 * ------------------------------------------------------------------------------------------------------------------ */
int64_t opb_bwd_ws_floats(int dim);

/* LayerNorm backward (components.py:23-26): y = LN(x) * gamma + beta, or y = gelu(LN(x) * gamma + beta) when gelu != 0
 * (adapter/image.py:66-75).  dx = assign or (accumulate != 0, fp32 only) add;  dgamma / dbeta fp32 [dim] or NULL.
 * dy_merge_w > 0: dy is the gradient of the NEXT conv's 2x2 pixel-merged operand [rows / 4, 4 * dim] (the forward's
 * opb_layernorm merge_grid_w scatter) and is gathered accordingly.
 * Dtype tags OPB_F32 / OPB_BF16; dim % 4 == 0, dim <= 6144. */
int opb_layernorm_bwd(const void* x, int x_dtype, int64_t ldx, const void* dy, int dy_dtype, int64_t ld_dy,
                      const float* gamma, const float* beta, void* dx, int dx_dtype, int64_t ld_dx, int accumulate,
                      int rows, int dim, float eps, int gelu, int dy_merge_w, float* ws, float* dgamma, float* dbeta,
                      void* stream);

/* GeGLU on the un-fused projection gl = [g | l] bf16 [rows, 2F] (transformer_layer.py:54-67): u = gelu_erf(g) * l and
 * its adjoint dgl = [du * l * gelu'(g) | du * gelu(g)]. */
int opb_geglu_fwd(const void* gl, void* u, int64_t rows, int F, void* stream);
int opb_geglu_bwd(const void* gl, const void* du, void* dgl, int64_t rows, int F, void* stream);

/* Exact-erf GELU on the video adapters' bf16 pre-activations z [rows, F] (onepeace.py:29-39): y = gelu_erf(z), and its
 * adjoint dz = dy * gelu'(z).  F % 8 == 0, 16-byte aligned non-null pointers, else OPB_ERR_INVALID. */
int opb_gelu_fwd(const void* z, void* y, int64_t rows, int F, void* stream);
int opb_gelu_bwd(const void* z, const void* dy, void* dz, int64_t rows, int F, void* stream);

/* LayerScale + drop-path residual (transformer_layer.py:70-88): out = x + row_scale[r] * gamma[n] * o  (o bf16; gamma /
 * row_scale may be NULL = 1) and its adjoint: d_o = bf16(row_scale * gamma * dx), dgamma = sum_r row_scale * dx * o,
 * dbias = sum_r row_scale * gamma * dx in fp32, before the bf16 rounding of d_o (the bias gradient of the Linear that
 * produced o; opb_colsum_bf16 instead sums the rounded values it is given). */
int opb_scale_resid_fwd(const float* x, const void* o, const float* gamma, const float* row_scale, float* out,
                        int64_t rows, int n, void* stream);
int opb_scale_resid_bwd(const float* dx, const void* o, const float* gamma, const float* row_scale, void* d_o, float* ws,
                        float* dgamma, float* dbias, int rows, int n, int in_period, int in_valid, int in_shift,
                        void* stream);   /* in_valid > 0: output row r reads dx row (r / in_valid) * in_period + in_shift + r % in_valid */

/* out[n] = sum over rows of y bf16 [rows, n]: bias gradients of the nn.Linear layers (components.py:29-35; q / v / out_proj,
 * multihead_attention.py:40-43). */
int opb_colsum_bf16(const void* y, int64_t ldy, float* ws, float* out, int rows, int n, void* stream);

/* Attention backward (multihead_attention.py:107-115): from qkv (q scaled), the forward output `out`, its gradient
 * `d_out` and the forward's log-sum-exp, writes dqkv bf16 [B*S, 3*H*64] (dq already multiplied by q_scale, i.e. the
 * gradient of the un-scaled projection) and adds the relative-position-bias gradient into dbias fp32 [H,S,s_pad]
 * (or NULL).  delta: fp32 scratch [B,H,S].  bias_batch_stride as in opb_attention_fwd (bias and dbias then hold one
 * table per sample). */
int opb_attention_bwd(const void* qkv, const void* out, const void* d_out, const float* bias, const uint8_t* key_pad,
                      const float* lse, float* delta, void* dqkv, float* dbias, int B, int S, int H, int s_pad,
                      float q_scale, int64_t bias_batch_stride, void* stream);

/* Same product, S <= 224 only (csrc/attention_bwd.cu), with the batch-shared relative-position bias and
 * its gradient held as TRANSPOSED tables so that a thread's (key, query-pair) words sit at fixed offsets:
 *   bias_t   H x 256 x 112 half2 words: bias[h][q][key] * log2(e) at [h][key][q / 2], zero for key >= S or q >= S
 *            (opb_relpos_bias_transpose builds it from the dense table of adapter/text.py:84-91, image.py:164-171);
 *   dbias_t  H x 256 x 224 fp32, accumulated with atomic adds over all layers that share the table, folded back into
 *            the dense (H,S,s_pad) gradient once per stack by opb_relpos_dbias_fold.  Either may be NULL (no bias / no
 *            bias gradient).  Returns OPB_ERR_UNSUPPORTED for S > 224. */
int opb_attention_bwd_t(const void* qkv, const void* out, const void* d_out, const void* bias_t, const uint8_t* key_pad,
                        const float* lse, float* delta, void* dqkv, float* dbias_t, int B, int S, int H, float q_scale,
                        void* stream);
int opb_relpos_bias_transpose(const float* bias, void* bias_t, int S, int s_pad, int H, void* stream);
int opb_relpos_dbias_fold(const float* dbias_t, float* dbias, int S, int s_pad, int H, void* stream);
/* dbias[h][i][:S] -= mean_j dbias[h][i][j]: projects the accumulated bias gradient of a single-modality stack onto the zero-row-sum
 * subspace the exact gradient lives in (softmax is invariant to per-row logit shifts, multihead_attention.py:107-115), removing
 * the row-coherent offset that delta = sum(dO * O) from the bf16-rounded forward output leaves (csrc/attention_bwd_tc.cu). */
int opb_relpos_dbias_center(float* dbias, int S, int s_pad, int H, void* stream);

/* out[c] (+)= sum_b in[b * ld + c]: gradients of batch-broadcast parameters (cls_embedding / pos_embed expanded over the
 * batch, adapter/image.py:239-253, audio.py:194-197). */
int opb_batch_sum_f32(const float* in, int64_t ld, float* out, int B, int64_t n, int accumulate, void* stream);

/* Adjoint of opb_l2_normalize_rows (F.normalize, one_peace_retrieval.py:116): dx = (dy - y (y.dy)) / |x|; fp32 and / or
 * bf16 output (the bf16 copy feeds the projection's dW / dX GEMMs). */
int opb_l2_normalize_bwd(const float* x, int64_t ldx, const float* dy, int64_t ld_dy, float* dx, void* dx_bf16, int rows,
                         int D, void* stream);

/* Adjoint of opb_text_embed (adapter/text.py:125-129,144-146): scatter-adds dx [B,T+1,D] into the fp32 gradients of
 * embed_tokens.weight [V,D], embed_positions.weight [>=T+1,D] and cls_embedding [D]; padded tokens get none. */
int opb_text_embed_bwd(const float* dx, const int64_t* tokens, float* dtable, float* dpos, float* dcls, int B, int T,
                       int D, int pad_idx, void* stream);

/* Channel-last 1-D convolution windows for the audio adapter's TRAINING path (adapter/audio.py:57-80 conv positions:
 * k = 19, pad 9, 16 groups; :254-311 feature extractor: k in {3, 2}, stride 2).  The inference path feeds the GEMM with
 * overlapping TMA views; training materialises the window matrix because dW = dY^T . windows needs it K-major.
 *   opb_window_gather : out[g][(b,t)][j*cg + c] = in[b, t*stride + j - pad, g*cg + c]  (0 outside the clip)
 *                       in bf16 [B*t_in, groups*cg] -> out bf16 [groups][B*t_out][kw*cg]
 *   opb_window_scatter: its adjoint (col2im), dx bf16 [B*t_in, groups*cg], gather form (deterministic)  */
int opb_window_gather(const void* in, void* out, int B, int t_in, int t_out, int stride, int kw, int pad, int groups,
                      int cg, void* stream);
int opb_window_scatter(const void* dwin, void* dx, int B, int t_in, int t_out, int stride, int kw, int pad, int groups,
                       int cg, void* stream);

/* dtable[bucket[i,j], h] += dbias[h,i,j]  (adjoint of opb_relpos_bias_build; adapter/text.py:84-91, image.py:164-171) */
int opb_relpos_bias_bwd(const float* dbias, const int64_t* bucket, float* dtable, int S, int s_pad, int H,
                        int64_t ld_bucket, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Retrieval evaluation (one_peace/metrics/recall.py:22-78; SURVEY.md 8f "next" row 3).
 *   opb_topk10_rows : idx int32 [R,10] (and val fp32 [R,10] unless NULL) = the 10 largest entries of every row of
 *                     sim fp32 [R,C] (row pitch ld), descending; ties -> smaller column first  (scores.topk(k=10), :39,:50)
 *   opb_recall_hits : hits[0..2] += number of rows whose own id (row_ids[r]) appears among the candidate ids of its first
 *                     1 / 5 / 10 ranked columns  (:41, :52); hits int32[3], caller zeroes it
 * ------------------------------------------------------------------------------------------------------------------ */
int opb_topk10_rows(const float* sim, int64_t ld, int32_t* idx, float* val, int R, int C, void* stream);
int opb_recall_hits(const int32_t* idx, const int64_t* cand_ids, const int64_t* row_ids, int R, int32_t* hits,
                    void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Pretraining path (SURVEY.md 8f rows 1-2): preserve_ids gathers, mask-token canvas, sample-dependent / block-diagonal
 * dense relative-position bias.
 *   opb_row_gather      : out[r, :dim] = (idx[r] >= 0 ? src[idx[r], :dim] : (fill ? fill[:dim] : 0)) + (add ?
 *                         add[r % add_period, :dim] : 0)   (dtype tags OPB_F32 / OPB_BF16; dim % 4 == 0; fill / add fp32; `add`
 *                         is the positional table of `x = adapter_embedding + pos_embed`, text.py:157).  Replaces adapter_embedding.gather / pos_embed.gather of
 *                         models/adapter/text.py:92-95 (image.py:188-192, audio.py:126-128), the decoder canvas
 *                         `mask_token.repeat(...)[left_preserve_indices] = preserve_embed[...]` (text.py:135-142) and the
 *                         masked-row / non-padded-row selections of compute_dcl_loss (image_text_pretrain_loss.py:190-202).
 *   opb_row_scatter_add : dsrc[idx[r], :] += dout[r, :] for idx[r] >= 0 (fp32 accumulation): its adjoint.
 *   opb_relpos_bias_block : bias[bb, h, lo+i, lo+j] = table[bucket[p_i, p_j], h] for i, j < n, with p_i = ids[bb, i]
 *                         (negative -> n - 1, the reference's masked_fill of padded slots, text.py:148) or p_i = i when ids
 *                         is NULL (then Bb = 1).  bias fp32 [Bb, H, S, s_pad], caller zeroes it: one call per modality places
 *                         that modality's block on the diagonal (transformer_encoder.py:148-158) and, with ids, performs the
 *                         two-axis bias gather of gather_features (text.py:96-101).
 *   opb_relpos_bias_block_bwd : dtable[bucket[p_i, p_j], h] += dbias[bb, h, lo+i, lo+j].
 * ------------------------------------------------------------------------------------------------------------------ */
int opb_row_gather(const void* src, int src_dtype, int64_t ld_src, const int64_t* idx, const float* fill, const float* add,
                   int64_t add_period, void* out, int out_dtype, int64_t ld_out, int64_t rows, int dim, void* stream);
int opb_row_scatter_add(const void* dout, int dout_dtype, int64_t ld_dout, const int64_t* idx, float* dsrc, int64_t ld_dsrc,
                        int64_t rows, int dim, void* stream);
int opb_relpos_bias_block(const float* table, const int64_t* bucket, int64_t ld_bucket, const int64_t* ids, int64_t ids_ld,
                          int Bb, int n, int lo, float* bias, int S, int s_pad, int H, void* stream);
int opb_relpos_bias_block_bwd(const float* dbias, const int64_t* bucket, int64_t ld_bucket, const int64_t* ids,
                              int64_t ids_ld, int Bb, int n, int lo, float* dtable, int S, int s_pad, int H, void* stream);

/*
 * GEMM with MN-major operands: out[M, N] = A B^T (+ bias[n]) where A is given as [K, M] row-major when a_mn != 0 (else the usual
 * [M, K]) and B as [K, N] row-major when b_mn != 0 (else [N, K]).  Contractions over the ROWS of activation matrices without a
 * transposed copy: every dW = dY^T X of the backward pass (torch autograd of the nn.Linear layers of
 * transformer_layer.py / multihead_attention.py) is opb_gemm_bf16_t(dY, ldy, 1, X, ldx, 1, N_out, K_in, rows, ...); the
 * InfoNCE gradient G . B_all (image_text_retrieval_loss.py:95-96) uses b_mn = 1.  epilogue: OPB_EPI_STORE_BF16 / _F32.
 */
int opb_gemm_bf16_t(const void* A, int64_t lda, int a_mn, const void* B, int64_t ldb, int b_mn, int M, int N, int K, int epilogue,
                    void* out, int64_t ldo, const float* bias, int cta_group, void* stream);

/*
 * Fold a LayerNorm into the nn.Linear that follows it (the fused-LN GEMM chain; reference: the four LayerNorm -> Linear pairs
 * of models/transformer/transformer_layer.py:185-219 and multihead_attention.py:103-124):
 *   out_w[row(n), k] = bf16(W[n,k] * ln_weight[k]),  colsum[row(n)] = sum_k out_w[row(n), k],
 *   bias_out[row(n)] = sum_k W[n,k] * ln_bias[k] + bias_in[n]
 * W fp32 / bf16 [N, K] (dtype tag, row pitch ldw); ln_weight / ln_bias / bias_in fp32 or NULL (1 / 0 / 0).
 * interleave 0: row(n) = n; 1 / 2: the wi_0 / wi_1 half of the GeGLU tile interleave, row(n) = (n / 128) * 256 [+ 128] + n % 128.
 */
int opb_ln_fold(const void* W, int w_dtype, int64_t ldw, const float* ln_weight, const float* ln_bias, const float* bias_in,
                int N, int K, int interleave, void* out_w, int64_t ldo, float* colsum, float* bias_out, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Classification head of one_peace_classify.
 *   opb_attn_pool_fwd : MultiheadAttentionPooling (models/one_peace/one_peace_base.py:146-173) after its k/v projection: per
 *                       sample b and head h, s_j = q[h] . k[b,j,h] (q NOT scaled), p = softmax_j(s) in fp32 over the keys with
 *                       key_pad[b,j] == 0, out[b, h*64:(h+1)*64] = bf16(sum_j p_j v[b,j,h]), lse[b*H + h] = log sum_j e^s_j.
 *                       kv bf16 [B, T, 2d] (k in columns [0, d), v in [d, 2d)), q fp32 [H, 64], key_pad uint8 [B, T] or NULL,
 *                       out bf16 [B, d], lse fp32 [B, H]; H = d / 64, any T >= 1.  Padded key rows are never read.  A sample
 *                       whose keys are all padded gets out = 0 and lse = -inf (the reference produces NaN there).
 *   opb_attn_pool_bwd : its adjoint for dout bf16 [B, d]: dkv bf16 [B, T, 2d] with dk[b,j,h] = p_j (dout[b,h] . v_j - delta) q[h],
 *                       dv[b,j,h] = p_j dout[b,h]; padded key rows are written as exact zeros.  dq fp32 [H, 64] = sum_b sum_j
 *                       ds_j k_j through the per-(b, h) partials dq_ws fp32 [B, H, 64] (caller-allocated scratch) summed over b in
 *                       order: no atomics, repeat launches are bit-identical.
 * ------------------------------------------------------------------------------------------------------------------ */
int opb_attn_pool_fwd(const void* kv, const float* q, const uint8_t* key_pad, void* out, float* lse, int B, int T, int d,
                      void* stream);
int opb_attn_pool_bwd(const void* kv, const float* q, const uint8_t* key_pad, const float* lse, const void* dout, void* dkv,
                      float* dq_ws, float* dq, int B, int T, int d, void* stream);

/*
 * Classification criteria (criterions/classify_loss.py:48-64 and criterions/hinge_loss.py:41-53), forward and the gradient of a
 * unit upstream gradient in one launch.  logits fp32 [rows, ld], of which the first n_valid columns are classes (the rest is
 * the padding of the classifier GEMM to N % 8 == 0 and is never read).  mode:
 *   0  hard labels int64 [rows]: cross_entropy(label_smoothing = eps); n_correct = (argmax == label), first index on ties; a
 *      label outside [0, n_valid) contributes nothing (ignore_index);
 *   1  soft targets fp32 [rows, ld_t]: -(targets * log_softmax).sum(); n_correct = (softmax * targets).sum(); eps unused;
 *   2  multi-label targets fp32 [rows, ld_t]: binary_cross_entropy_with_logits; n_correct = targets[argmax];
 *   3  hinge over groups of num_choices rows (n_valid == 1, labels int64 [rows / num_choices]): sum_c max(0, 1 + z_c - z_label),
 *      the positive's own term included; n_correct = (argmax == label).
 * Writes row_loss / row_correct fp32 [rows] ([rows / num_choices] for mode 3), dlogits fp32 [rows, ld] (zero in the padding
 * columns) and out2 = {sum of row_loss, sum of row_correct}, summed in a fixed order by the last CTA to finish.  ticket: one
 * zero-initialised uint32, left at zero.
 */
int opb_classify_loss(const float* logits, int64_t ld, int rows, int n_valid, int mode, const int64_t* labels,
                      const float* targets, int64_t ld_t, float eps, int num_choices, float* row_loss, float* dlogits,
                      float* row_correct, float* out2, unsigned int* ticket, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Visual grounding (refcoco_criterion and IouAcc).
 *   opb_refcoco_loss : criterions/refcoco_loss.py:36-46 and its gradient with respect to the logits, in fp32, in one launch.
 *                      p = sigmoid(logits[r, 0:4]) against targets fp32 [B, 4] (x0, y0, x1, y1, contiguous):
 *                        L1 = sum_{r,j} |p - t| / nsentences, gradient sign(p - t) / nsentences (0 at a tie);
 *                        valid[r] = p0 < p2 && p1 < p3 (strict; selects rows, no gradient through it);
 *                        giou[r] = torchvision.ops.generalized_box_iou of (p_r, t_r), written for every row;
 *                        loss = L1 + sum over valid rows of (1 - giou) / n_valid; NaN when n_valid == 0 (the reference's
 *                        mean of an empty tensor), while the gradient stays finite: the L1 part only.
 *                      The GIoU gradient follows torch's autograd: max / min give half the gradient to each side at a tie,
 *                      clamp(min=0) passes it where its argument is >= 0, and the targets get none.
 *                      logits fp32 [B, ld], ld >= 4 (columns [4, ld) are not read); out fp32 [3] = {loss, L1 part, n_valid};
 *                      valid int32 [B]; giou fp32 [B]; dlogits fp32 [B, ld] = d loss / d logits with columns [4, ld) set to
 *                      0.  One CTA, fixed-order sums: repeated launches are bit-identical.  Status 1 for B <= 0, ld < 4,
 *                      nsentences <= 0 or a null pointer, before anything is launched.
 *   opb_iou_acc      : metrics/iou_acc.py:20-32: hits[0] += number of rows r < n with iou >= 0.5 and w_i > 0 and h_i > 0, where
 *                      the intersection takes the max / min corners and iou = area_i / (area_p + area_t - area_i), every
 *                      operation in the reference's order and rounded on its own (no FMA contraction), so the count equals
 *                      the reference's fp32 count exactly.  hyps / refs fp32 [n, >= 4] at row pitches ld_h / ld_r; hits one
 *                      int32 the caller zeroes once and reads when it wants the total (nothing synchronises); row_hit int32
 *                      [n] or NULL receives the per-row flag.  Status 1 for n <= 0, a pitch < 4 or a null hyps / refs / hits.
 * ------------------------------------------------------------------------------------------------------------------ */
int opb_refcoco_loss(const float* logits, int64_t ld, const float* targets, int B, int nsentences, float* out, int* valid,
                     float* giou, float* dlogits, void* stream);
int opb_iou_acc(const float* hyps, int64_t ld_h, const float* refs, int64_t ld_r, int n, int* hits, int* row_hit, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Classification evaluation (Accuracy and MAP).
 *   opb_argmax_hits   : metrics/accuracy.py:20-25: hyp[r] = torch.argmax(logits[r, 0:C]) as int64 (the first maximal
 *                       index; a NaN is the maximum, so the first NaN wins; bf16 compares after its exact up-cast) and
 *                       score[r] fp32 = the row's hit: tmode 0 int64 labels [n] -> 1 / 0 for hyp == label; tmode 1 fp32
 *                       labels [n] -> 1 / 0 for float(hyp) == label (torch.eq's promotion); tmode 2 soft scores fp32
 *                       [n, ldt] -> targets[r, hyp] exactly.  logits fp32 (dtype OPB_F32) or bf16 (OPB_BF16) at element
 *                       (r, j) = logits[r * ld + j * cs], so padded rows and column-strided views are read in place.
 *                       One warp per row for C > 8, one thread per row for C <= 8.  Status 1 for n <= 0, C outside
 *                       [1, 4096], ld or cs < 1, an unknown dtype / tmode, ldt < C with tmode 2, or a null pointer.
 *   opb_sum_f64       : out[0] = sum of x fp32 [n] in fp64 in a fixed order (one CTA): bit-identical on every run.
 *                       Status 1 for n <= 0 or a null pointer.
 *   opb_sigmoid_pack  : metrics/map.py:20-23 and the torch.sigmoid of :34: for r < n, j < C, with o = (row_offset + r) * C + j,
 *                       probs[o] = 1 / (1 + expf(-x)) in IEEE fp32 (torch.sigmoid's CUDA fp32 result bit for bit; bf16 is
 *                       up-cast first) and labels[o] = uint8(targets[r * ldt + j] == 1).  flags int32 [2] (the caller
 *                       zeroes it once): flags[0] += number of targets outside {0, 1}, flags[1] += number of NaN
 *                       probabilities.  Status 1 for n <= 0, C outside [1, 4096], ld or cs < 1, ldt < C, row_offset < 0,
 *                       an unknown dtype or a null pointer.
 *   opb_average_precision : sklearn.metrics.average_precision_score(labels, probs, average=None) and the np.mean of
 *                       metrics/map.py:43.  probs fp32 [N, C] in [0, 1] (values outside are clamped into it), labels uint8
 *                       [N, C] (non-zero = positive), 1 <= N < 2^24, 1 <= C <= 4096, N * C < 2^31.  Per class: sort by
 *                       probability, descending; group equal probabilities; ap[c] = sum over groups g of
 *                       pos_g * TP_g / (TP_g + FP_g) / P_c with TP / FP counted through g, 0 when P_c = 0.  Counts are exact
 *                       integers, each group's term is formed in fp64 and the terms are summed in a fixed order; mean[0] is
 *                       the fp64 mean of ap in class order; npos int64 [C] = P_c.  Device-wide LSD radix sort of
 *                       class-major 64-bit keys in the workspace of opb_average_precision_ws_bytes(N, C) bytes (-1 for a
 *                       shape outside the range above).  Status 1 for a shape outside that range, a smaller workspace or a
 *                       null pointer.
 * ------------------------------------------------------------------------------------------------------------------ */
int opb_argmax_hits(const void* logits, int dtype, int64_t ld, int64_t cs, int n, int C, const void* targets, int tmode,
                    int64_t ldt, int64_t* hyp, float* score, void* stream);
int opb_sum_f64(const float* x, int64_t n, double* out, void* stream);
int opb_sigmoid_pack(const void* logits, int dtype, int64_t ld, int64_t cs, const float* targets, int64_t ldt, int n, int C,
                     float* probs, uint8_t* labels, int64_t row_offset, int* flags, void* stream);
int64_t opb_average_precision_ws_bytes(int N, int C);
int opb_average_precision(const float* probs, const uint8_t* labels, int N, int C, void* ws, int64_t ws_bytes, double* ap,
                          double* mean, int64_t* npos, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Pooled head of OnePeaceViT (one_peace_vision/classification/models_vit.py:431-434, global_pool=True).
 *   opb_token_mean_ln_ws_floats : floats of the forward's workspace for (B, S, d); -1 for a shape the kernels refuse.
 *   opb_token_mean_ln_fwd : m[b] = mean of x[b, 1:S, :] over the S - 1 patch rows (the CLS row 0 is excluded; the sum is
 *                           divided by S - 1), then fc_norm: y[b] = bf16((m[b] - mean[b]) * rstd[b] * gamma + beta) with
 *                           mean[b] / rstd[b] = the LayerNorm statistics of m[b] over d (biased variance, rstd =
 *                           1 / sqrt(var + eps)).  x fp32, row (b, s) at x + (b * S + s) * ld; m fp32 [B, d] (kept for the
 *                           backward), y bf16 [B, d] (the A operand of the head GEMM), mean / rstd fp32 [B].  The row sum is
 *                           split across CTAs per (sample, 256-column slice, row range) into ws and merged in split order by
 *                           one CTA per sample: the split count depends on the shape only, there are no atomics, and repeated
 *                           launches are bit-identical.
 *   opb_token_mean_ln_bwd : its adjoint for dy = d loss / d y fp32 [B, d]: dgamma / dbeta fp32 [d] summed over b in order;
 *                           dx fp32 (row (b, s) at dx + (b * S + s) * ld_dx) = the LayerNorm adjoint of row b divided by
 *                           S - 1 in every patch row s >= 1 and exact zeros in the CLS row s = 0.  Every row of dx is
 *                           written exactly once, so it needs no zeroing.  ws: fp32 [B, d] scratch.
 * Both need 1 <= B <= 65535, S >= 2, d >= 4 with d % 4 == 0, a row pitch >= d with pitch % 4 == 0, x / dx / ws 16-byte
 * aligned, eps >= 0 and a large enough workspace; anything else (or a null pointer) returns status 1 before any launch.
 * ------------------------------------------------------------------------------------------------------------------ */
int64_t opb_token_mean_ln_ws_floats(int B, int S, int d);
int opb_token_mean_ln_fwd(const float* x, int64_t ld, int B, int S, int d, const float* gamma, const float* beta, float eps,
                          float* ws, int64_t ws_floats, float* m, void* y, float* mean, float* rstd, void* stream);
int opb_token_mean_ln_bwd(const float* dy, const float* m, const float* mean, const float* rstd, const float* gamma, int B,
                          int S, int d, float* dgamma, float* dbeta, float* ws, float* dx, int64_t ld_dx, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ONEPEACE_B200_H_ */
