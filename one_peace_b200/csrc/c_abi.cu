// extern "C" boundary of libonepeace_b200.so — see include/onepeace_b200.h for the contract.
#include "../../include/onepeace_b200.h"

#include "common.cuh"
#include "gemm.h"
#include "ops.h"

#include <stdlib.h>

extern "C" {

int opb_abi_version(void) { return 3; }

const char* opb_status_string(int status) {
  switch (status) {
    case OPB_OK: return "ok";
    case OPB_ERR_INVALID: return "invalid argument (shape / alignment / null pointer)";
    case OPB_ERR_CUDA: return "CUDA error at launch";
    case OPB_ERR_UNSUPPORTED: return "unsupported shape";
    default: return "unknown status";
  }
}

int opb_gemm_bf16(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K, int epi, void* out,
                  int64_t ldo, const float* bias, const float* colscale, const float* gamma, const float* resid,
                  int64_t ldr, int out_group, int out_group_stride, int out_row_offset, int out_group_valid,
                  int resid_period, int resid_row_offset, int cta_group, void* stream) {
  if (A == nullptr || B == nullptr || out == nullptr) return OPB_ERR_INVALID;
  opb::GemmEpilogue ep;
  ep.out = out;
  ep.ldo = ldo;
  ep.bias = bias;
  ep.colscale = colscale;
  ep.gamma = gamma;
  ep.resid = resid;
  ep.ldr = ldr;
  ep.out_group = out_group;
  ep.out_group_stride = out_group_stride;
  ep.out_row_offset = out_row_offset;
  ep.out_group_valid = out_group_valid;
  ep.resid_period = resid_period;
  ep.resid_row_offset = resid_row_offset;
  return opb::gemm_bf16(A, static_cast<int>(lda), B, static_cast<int>(ldb), M, N, K, epi, ep, cta_group,
                        static_cast<cudaStream_t>(stream));
}

int opb_attention_fwd(const void* qkv, const float* bias, const uint8_t* key_pad, void* out, float* lse,
                      float* ln_stats, int B, int S, int H, int s_pad, int64_t bias_batch_stride, void* stream) {
  if (qkv == nullptr || out == nullptr || bias_batch_stride < 0) return OPB_ERR_INVALID;
  return opb::attention_fwd(qkv, bias, key_pad, out, lse, ln_stats, B, S, H, s_pad, bias_batch_stride,
                            static_cast<cudaStream_t>(stream));
}

int opb_attention_tc_fwd(const void* qkv, const float* lut, const float* lut_max, int lut_len, const int32_t* code_row,
                         const int32_t* code_col, const uint8_t* key_pad, void* out, float* lse, float* ln_stats, int B,
                         int S, int H, int seg_split, void* stream) {
  if (!qkv || !lut || !lut_max || !code_row || !code_col || !out) return OPB_ERR_INVALID;
  return opb::attention_lut_fwd(qkv, lut, lut_len, code_row, code_col, key_pad, out, lse, ln_stats, B, S, H, seg_split,
                                static_cast<cudaStream_t>(stream));
}

int opb_attention_temporal_fwd(const void* qkv, void* out, float* ln_stats, int Bv, int T, int N, int H, void* stream) {
  return opb::attention_temporal_fwd(qkv, out, ln_stats, Bv, T, N, H, static_cast<cudaStream_t>(stream));
}

int opb_attention_temporal_bwd(const void* qkv, const void* out, const void* d_out, void* dqkv, int Bv, int T, int N, int H,
                               float q_scale, void* stream) {
  return opb::attention_temporal_bwd(qkv, out, d_out, dqkv, Bv, T, N, H, q_scale, static_cast<cudaStream_t>(stream));
}

int opb_ms_deform_attn_fwd(const void* value, const float* proj, const float* ref, void* out, int N, int S_in, int Lq, int H,
                           int D, int L, int P, int L_ref, const int32_t* level_hw, const int32_t* level_start, void* stream) {
  return opb::ms_deform_attn_fwd(value, proj, ref, out, N, S_in, Lq, H, D, L, P, L_ref, level_hw, level_start,
                                 static_cast<cudaStream_t>(stream));
}

int opb_ms_deform_attn_bwd(const void* value, const float* proj, const float* ref, const void* d_out, float* d_value,
                           float* d_proj, int N, int S_in, int Lq, int H, int D, int L, int P, int L_ref,
                           const int32_t* level_hw, const int32_t* level_start, void* stream) {
  return opb::ms_deform_attn_bwd(value, proj, ref, d_out, d_value, d_proj, N, S_in, Lq, H, D, L, P, L_ref, level_hw,
                                 level_start, static_cast<cudaStream_t>(stream));
}

int opb_relpos_lut_build(const float* table, const int32_t* idx, float* lut, int L, int H, void* stream) {
  if (!table || !idx || !lut) return OPB_ERR_INVALID;
  return opb::relpos_lut_build(table, idx, lut, L, H, static_cast<cudaStream_t>(stream));
}

int opb_relpos_decomp_proj(const void* qkv, const float* rel_pos_h, const float* rel_pos_w, const int32_t* pos_y,
                           const int32_t* pos_x, float q_unscale, float* rel_h, float* rel_w, int B, int S, int H, int kh,
                           int kw, void* stream) {
  if (!qkv || !rel_pos_h || !rel_pos_w || !pos_y || !pos_x || !rel_h || !rel_w) return OPB_ERR_INVALID;
  return opb::relpos_decomp_proj(qkv, rel_pos_h, rel_pos_w, pos_y, pos_x, q_unscale, rel_h, rel_w, B, S, H, kh, kw,
                                 static_cast<cudaStream_t>(stream));
}

int opb_attention_decomp_fwd(const void* qkv, const float* lut, int lut_len, const int32_t* code_row,
                             const int32_t* code_col, const float* rel_h, const float* rel_w, const int32_t* key_y,
                             const int32_t* key_x, int kh, int kw, void* out, float* lse, float* ln_stats, int B, int S,
                             int H, void* stream) {
  if (!qkv || !lut || !code_row || !code_col || !rel_h || !rel_w || !key_y || !key_x || !out) return OPB_ERR_INVALID;
  opb::DecompRel dr;
  dr.rel_h = rel_h; dr.rel_w = rel_w; dr.key_y = key_y; dr.key_x = key_x; dr.kh = kh; dr.kw = kw;
  return opb::attention_decomp_fwd(qkv, lut, lut_len, code_row, code_col, dr, out, lse, ln_stats, B, S, H,
                                   static_cast<cudaStream_t>(stream));
}

int opb_gemm_bf16_ex(const opb_gemm_args* a, void* stream) {
  if (a == nullptr || a->A == nullptr || a->B == nullptr || a->out == nullptr) return OPB_ERR_INVALID;
  if ((a->ln_mu == nullptr) != (a->ln_rstd == nullptr)) return OPB_ERR_INVALID;
  if (a->ln_mu != nullptr && a->ln_partial != nullptr) return OPB_ERR_INVALID;
  if ((a->ln_colsum != nullptr) != (a->ln_mu != nullptr || a->ln_partial != nullptr)) return OPB_ERR_INVALID;
  if (a->ln_partial != nullptr && (a->ln_parts <= 0 || a->ln_dim <= 0)) return OPB_ERR_INVALID;
  opb::GemmEpilogue ep;
  ep.out = a->out; ep.ldo = a->ldo;
  ep.bias = a->bias; ep.colscale = a->colscale; ep.gamma = a->gamma; ep.resid = a->resid; ep.ldr = a->ldr;
  ep.out_group = a->out_group; ep.out_group_stride = a->out_group_stride; ep.out_row_offset = a->out_row_offset;
  ep.out_group_valid = a->out_group_valid; ep.resid_period = a->resid_period; ep.resid_row_offset = a->resid_row_offset;
  ep.ln_mu = a->ln_mu; ep.ln_rstd = a->ln_rstd; ep.ln_colsum = a->ln_colsum;
  ep.stats_out = a->stats_out; ep.out_bf16 = a->out_bf16; ep.ldo_bf16 = a->ldo_bf16;
  ep.workspace = a->workspace; ep.workspace_bytes = a->workspace_bytes;
  ep.ln_partial = a->ln_partial; ep.ln_parts = a->ln_parts; ep.ln_dim = a->ln_dim; ep.ln_eps = a->ln_eps;
  return opb::gemm_bf16(a->A, static_cast<int>(a->lda), a->B, static_cast<int>(a->ldb), a->M, a->N, a->K, a->epi, ep,
                        a->cta_group, static_cast<cudaStream_t>(stream));
}

int opb_row_stats_cast(const float* x, int64_t ld_in, void* out_bf16, int64_t ld_out, float* mu, float* rstd,
                       int rows, int dim, float eps, void* stream) {
  if (!x || !out_bf16 || !mu || !rstd) return OPB_ERR_INVALID;
  opb::LnRemap rm;
  rm.raw = 1; rm.mu_out = mu; rm.rstd_out = rstd;
  return opb::layernorm(x, 0, ld_in, out_bf16, 1, ld_out, nullptr, nullptr, rows, dim, eps, 0, 0, rm,
                        static_cast<cudaStream_t>(stream));
}

int opb_ln_stats_finalize(const float* partial, int parts, int rows, int dim, float eps, float* mu, float* rstd,
                          void* stream) {
  if (!partial || !mu || !rstd) return OPB_ERR_INVALID;
  return opb::ln_stats_finalize(partial, parts, rows, dim, eps, mu, rstd, static_cast<cudaStream_t>(stream));
}

int opb_layernorm(const void* in, int in_dtype, int64_t ld_in, void* out, int out_dtype, int64_t ld_out,
                  const float* gamma, const float* beta, int rows, int dim, float eps, int gelu, int merge_grid_w,
                  int row_period, int row_valid, int out_period, int out_row_shift, int group_in, int group_out,
                  int accumulate, void* stream) {
  if (in == nullptr || out == nullptr) return OPB_ERR_INVALID;
  opb::LnRemap rm;
  rm.row_period = row_period; rm.row_valid = row_valid; rm.out_period = out_period; rm.out_row_shift = out_row_shift;
  rm.group_in = group_in; rm.group_out = group_out; rm.accumulate = accumulate;
  return opb::layernorm(in, in_dtype, ld_in, out, out_dtype, ld_out, gamma, beta, rows, dim, eps, gelu,
                        merge_grid_w, rm, static_cast<cudaStream_t>(stream));
}

int opb_grouped_conv1d_bf16(const void* X, const void* W, int rows, int groups, int c_pad, int taps, int n_per_group,
                            int epi, void* out, int64_t ldo, const float* bias, void* stream) {
  if (!X || !W || !out) return OPB_ERR_INVALID;
  opb::GemmEpilogue ep;
  ep.out = out;
  ep.ldo = ldo;
  ep.bias = bias;
  return opb::gemm_bf16_grouped_window(X, W, rows, groups, c_pad, taps, n_per_group, epi, ep,
                                       static_cast<cudaStream_t>(stream));
}

int opb_pack_group_halo(const float* x, int64_t ldx, void* out, int B, int T, int x_period, int x_row_shift,
                        int out_period, int halo, int dim, int group_in, int group_out, void* stream) {
  if (!x || !out) return OPB_ERR_INVALID;
  return opb::pack_group_halo(x, ldx, out, B, T, x_period, x_row_shift, out_period, halo, dim, group_in, group_out,
                              static_cast<cudaStream_t>(stream));
}

int opb_text_embed(const int64_t* tokens, const void* table, int table_dtype, const float* pos, const float* cls,
                   float* x, uint8_t* pad_mask, int B, int T, int D, int pad_idx, void* stream) {
  if (!tokens || !table || !pos || !cls || !x || !pad_mask) return OPB_ERR_INVALID;
  return opb::text_embed(tokens, table, table_dtype, pos, cls, x, pad_mask, B, T, D, pad_idx,
                         static_cast<cudaStream_t>(stream));
}

int opb_image_patchify4(const void* img, int img_dtype, void* out, int B, int R, void* stream) {
  if (!img || !out) return OPB_ERR_INVALID;
  return opb::image_patchify4(img, img_dtype, out, B, R, static_cast<cudaStream_t>(stream));
}

int opb_cls_row_init(const float* cls, const float* pos0, float* x, int64_t batch_stride, int B, int D,
                     void* stream) {
  if (!cls || !pos0 || !x) return OPB_ERR_INVALID;
  return opb::cls_row_init(cls, pos0, x, batch_stride, B, D, static_cast<cudaStream_t>(stream));
}

int opb_relpos_bias_build(const float* table, const int64_t* bucket, float* bias, int S, int s_pad, int H,
                          int64_t ld_bucket, void* stream) {
  if (!table || !bucket || !bias) return OPB_ERR_INVALID;
  return opb::relpos_bias_build(table, bucket, bias, S, s_pad, H, ld_bucket, static_cast<cudaStream_t>(stream));
}

int opb_audio_frame10(const void* wav, int wav_dtype, void* out, int B, int64_t n_samples, int64_t pitch,
                      void* stream) {
  if (!wav || !out) return OPB_ERR_INVALID;
  return opb::audio_frame10(wav, wav_dtype, out, B, n_samples, pitch, static_cast<cudaStream_t>(stream));
}

int opb_l2_normalize_rows(const float* x, int64_t ldx, float* y, void* y_bf16, int rows, int D, void* stream) {
  if (!x || !y) return OPB_ERR_INVALID;
  return opb::l2_normalize_rows(x, ldx, y, y_bf16, rows, D, static_cast<cudaStream_t>(stream));
}

int opb_zero_padded_rows(float* x, const uint8_t* pad_mask, int rows, int D, void* stream) {
  if (!x || !pad_mask) return OPB_ERR_INVALID;
  return opb::zero_padded_rows(x, pad_mask, rows, D, static_cast<cudaStream_t>(stream));
}

int opb_transpose_bf16(const void* in, int64_t ld_in, void* out, int rows, int cols, void* stream) {
  if (!in || !out) return OPB_ERR_INVALID;
  return opb::transpose_bf16(in, ld_in, out, rows, cols, static_cast<cudaStream_t>(stream));
}

int opb_split_bf16x3(const float* const* xs, void* const* outs, const int64_t* rows, const int* sides, int count, int d,
                     void* stream) {
  if (!xs || !outs || !rows || !sides) return OPB_ERR_INVALID;
  return opb::split_bf16x3(xs, outs, rows, sides, count, d, static_cast<cudaStream_t>(stream));
}

int64_t opb_infonce_ws_floats(int b, int n) { return opb::infonce_ws_floats(b, n); }

int opb_infonce_lse_gemm(const void* a_local, const void* b_all, const float* scale, int b, int n, int d, int target_offset,
                         float* ws, int n_valid, void* stream) {
  if (!a_local || !b_all || !scale || !ws) return OPB_ERR_INVALID;
  return opb::infonce_lse_gemm(a_local, b_all, scale, b, n, d, target_offset, ws, n_valid, static_cast<cudaStream_t>(stream));
}

int opb_infonce_merge_reduce(const float* ws_a, const float* ws_b, int b, int n, int n_valid, float label_smoothing,
                             int target_offset, float* row_lse_a, float* row_lse_b, float* loss_ab, int* argmax_ab, float* out3,
                             uint32_t* ticket, void* stream) {
  if (!ws_a || !row_lse_a || !loss_ab || !argmax_ab || !out3 || !ticket) return OPB_ERR_INVALID;
  return opb::infonce_merge_reduce(ws_a, ws_b, b, n, n_valid, label_smoothing, target_offset, row_lse_a, row_lse_b, loss_ab,
                                   argmax_ab, out3, ticket, static_cast<cudaStream_t>(stream));
}

int opb_infonce_grad(const void* a_local, const void* b_all, const float* scale, const float* row_lse, int b, int n, int d,
                     int k_logits, int target_offset, float label_smoothing, void* g_ws, float* ws_gz, float* grad_a,
                     int n_valid, float coef, void* stream) {
  if (!a_local || !b_all || !scale || !row_lse || !g_ws || !ws_gz || !grad_a) return OPB_ERR_INVALID;
  return opb::infonce_grad(a_local, b_all, scale, row_lse, b, n, d, k_logits, target_offset, label_smoothing,
                           g_ws, ws_gz, grad_a, n_valid, coef, static_cast<cudaStream_t>(stream));
}

int opb_infonce_dscale(const float* ws_gz_a, const float* ws_gz_b, int b, int n, float* out, void* stream) {
  if (!ws_gz_a || !ws_gz_b || !out || b <= 0 || n <= 0) return OPB_ERR_INVALID;
  return opb::infonce_dscale(ws_gz_a, ws_gz_b, b, n, out, static_cast<cudaStream_t>(stream));
}

int opb_adam_chunk_elems(void) { return 8192; }

int opb_adam_multi_step(const void* tensors, const int32_t* chunk_tensor, const int64_t* chunk_off, int n_chunks,
                        const float* lr, const float* wd, const float* bias_corr, int n_groups, float beta1,
                        float beta2, float eps, const float* grad_scale, void* stream) {
  if (!tensors || !chunk_tensor || !chunk_off || !lr || !wd || !bias_corr) return OPB_ERR_INVALID;
  if (n_groups <= 0 || n_groups > opb::kAdamMaxGroups) return OPB_ERR_UNSUPPORTED;
  opb::AdamGroups g;
  for (int i = 0; i < n_groups; ++i) { g.lr[i] = lr[i]; g.wd[i] = wd[i]; g.bias_corr[i] = bias_corr[i]; }
  g.beta1 = beta1; g.beta2 = beta2; g.eps = eps;
  return opb::adam_multi_step(tensors, chunk_tensor, reinterpret_cast<const long*>(chunk_off), n_chunks, g, grad_scale,
                              static_cast<cudaStream_t>(stream));
}

int opb_adan_multi_step(const void* tensors, const int32_t* chunk_tensor, const int64_t* chunk_off, int n_chunks,
                        const float* lr, const float* wd, const int32_t* no_prox, const float* bc1, const float* bc2,
                        const float* sqrt_bc3, int n_groups, float beta1, float beta2, float beta3, float eps,
                        const float* grad_scale, void* stream) {
  if (!tensors || !chunk_tensor || !chunk_off || !lr || !wd || !no_prox || !bc1 || !bc2 || !sqrt_bc3) return OPB_ERR_INVALID;
  if (n_groups <= 0 || n_groups > opb::kAdanMaxGroups) return OPB_ERR_UNSUPPORTED;
  opb::AdanGroups g;
  for (int i = 0; i < n_groups; ++i) {
    g.lr[i] = lr[i]; g.wd[i] = wd[i]; g.no_prox[i] = no_prox[i];
    g.bc1[i] = bc1[i]; g.bc2[i] = bc2[i]; g.sqrt_bc3[i] = sqrt_bc3[i];
  }
  g.beta1 = beta1; g.beta2 = beta2; g.beta3 = beta3; g.eps = eps;
  return opb::adan_multi_step(tensors, chunk_tensor, reinterpret_cast<const long*>(chunk_off), n_chunks, g, grad_scale,
                              static_cast<cudaStream_t>(stream));
}

int opb_grad_norm_clip(const void* tensors, const int32_t* chunk_tensor, const int64_t* chunk_off, int n_chunks,
                       float* partial, float multiply_factor, float max_norm, float* out2, void* stream) {
  if (!tensors || !chunk_tensor || !chunk_off || !partial || !out2) return OPB_ERR_INVALID;
  return opb::grad_norm_clip(tensors, chunk_tensor, reinterpret_cast<const long*>(chunk_off), n_chunks, partial,
                             multiply_factor, max_norm, out2, static_cast<cudaStream_t>(stream));
}

int64_t opb_bwd_ws_floats(int dim) { return opb::bwd_ws_floats(dim); }

int opb_layernorm_bwd(const void* x, int x_dtype, int64_t ldx, const void* dy, int dy_dtype, int64_t ld_dy,
                      const float* gamma, const float* beta, void* dx, int dx_dtype, int64_t ld_dx, int accumulate,
                      int rows, int dim, float eps, int gelu, int dy_merge_w, float* ws, float* dgamma, float* dbeta,
                      void* stream) {
  if (!x || !dy || !dx) return OPB_ERR_INVALID;
  return opb::layernorm_bwd(x, x_dtype, ldx, dy, dy_dtype, ld_dy, gamma, beta, dx, dx_dtype, ld_dx, accumulate, rows, dim,
                            eps, gelu, dy_merge_w, ws, dgamma, dbeta, static_cast<cudaStream_t>(stream));
}

int opb_geglu_fwd(const void* gl, void* u, int64_t rows, int F, void* stream) {
  if (!gl || !u) return OPB_ERR_INVALID;
  return opb::geglu_fwd(gl, u, rows, F, static_cast<cudaStream_t>(stream));
}

int opb_geglu_bwd(const void* gl, const void* du, void* dgl, int64_t rows, int F, void* stream) {
  if (!gl || !du || !dgl) return OPB_ERR_INVALID;
  return opb::geglu_bwd(gl, du, dgl, rows, F, static_cast<cudaStream_t>(stream));
}

int opb_gelu_fwd(const void* z, void* y, int64_t rows, int F, void* stream) {
  if (!z || !y) return OPB_ERR_INVALID;
  return opb::gelu_fwd(z, y, rows, F, static_cast<cudaStream_t>(stream));
}

int opb_gelu_bwd(const void* z, const void* dy, void* dz, int64_t rows, int F, void* stream) {
  if (!z || !dy || !dz) return OPB_ERR_INVALID;
  return opb::gelu_bwd(z, dy, dz, rows, F, static_cast<cudaStream_t>(stream));
}

int opb_scale_resid_fwd(const float* x, const void* o, const float* gamma, const float* row_scale, float* out,
                        int64_t rows, int n, void* stream) {
  if (!x || !o || !out) return OPB_ERR_INVALID;
  return opb::scale_resid_fwd(x, o, gamma, row_scale, out, rows, n, static_cast<cudaStream_t>(stream));
}

int opb_scale_resid_bwd(const float* dx, const void* o, const float* gamma, const float* row_scale, void* d_o, float* ws,
                        float* dgamma, float* dbias, int rows, int n, int in_period, int in_valid, int in_shift,
                        void* stream) {
  if (!dx || !d_o) return OPB_ERR_INVALID;
  return opb::scale_resid_bwd(dx, o, gamma, row_scale, d_o, ws, dgamma, dbias, rows, n, in_period, in_valid, in_shift,
                              static_cast<cudaStream_t>(stream));
}

int opb_batch_sum_f32(const float* in, int64_t ld, float* out, int B, int64_t n, int accumulate, void* stream) {
  if (!in || !out) return OPB_ERR_INVALID;
  return opb::batch_sum_f32(in, ld, out, B, n, accumulate, static_cast<cudaStream_t>(stream));
}

int opb_l2_normalize_bwd(const float* x, int64_t ldx, const float* dy, int64_t ld_dy, float* dx, void* dx_bf16, int rows,
                         int D, void* stream) {
  if (!x || !dy) return OPB_ERR_INVALID;
  return opb::l2_normalize_bwd(x, ldx, dy, ld_dy, dx, dx_bf16, rows, D, static_cast<cudaStream_t>(stream));
}

int opb_window_gather(const void* in, void* out, int B, int t_in, int t_out, int stride, int kw, int pad, int groups,
                      int cg, void* stream) {
  if (!in || !out) return OPB_ERR_INVALID;
  return opb::window_gather(in, out, B, t_in, t_out, stride, kw, pad, groups, cg, static_cast<cudaStream_t>(stream));
}

int opb_window_scatter(const void* dwin, void* dx, int B, int t_in, int t_out, int stride, int kw, int pad, int groups,
                       int cg, void* stream) {
  if (!dwin || !dx) return OPB_ERR_INVALID;
  return opb::window_scatter(dwin, dx, B, t_in, t_out, stride, kw, pad, groups, cg, static_cast<cudaStream_t>(stream));
}

int opb_text_embed_bwd(const float* dx, const int64_t* tokens, float* dtable, float* dpos, float* dcls, int B, int T,
                       int D, int pad_idx, void* stream) {
  if (!dx || !tokens || !dtable || !dpos || !dcls) return OPB_ERR_INVALID;
  return opb::text_embed_bwd(dx, tokens, dtable, dpos, dcls, B, T, D, pad_idx, static_cast<cudaStream_t>(stream));
}

int opb_colsum_bf16(const void* y, int64_t ldy, float* ws, float* out, int rows, int n, void* stream) {
  if (!y || !out) return OPB_ERR_INVALID;
  return opb::colsum_bf16(y, ldy, ws, out, rows, n, static_cast<cudaStream_t>(stream));
}

int opb_attention_bwd(const void* qkv, const void* out, const void* d_out, const float* bias, const uint8_t* key_pad,
                      const float* lse, float* delta, void* dqkv, float* dbias, int B, int S, int H, int s_pad,
                      float q_scale, int64_t bias_batch_stride, void* stream) {
  if (!qkv || !out || !d_out || !dqkv || bias_batch_stride < 0) return OPB_ERR_INVALID;
  return opb::attention_bwd(qkv, out, d_out, bias, key_pad, lse, delta, dqkv, dbias, B, S, H, s_pad, q_scale,
                            bias_batch_stride, static_cast<cudaStream_t>(stream));
}

int opb_attention_bwd_t(const void* qkv, const void* out, const void* d_out, const void* bias_t, const uint8_t* key_pad,
                        const float* lse, float* delta, void* dqkv, float* dbias_t, int B, int S, int H, float q_scale,
                        void* stream) {
  if (!qkv || !out || !d_out || !dqkv || !lse || !delta || B <= 0 || S <= 0 || H <= 0) return OPB_ERR_INVALID;
  if (S > 224) return OPB_ERR_UNSUPPORTED;
  return opb::attention_bwd(qkv, out, d_out, nullptr, key_pad, lse, delta, dqkv, nullptr, B, S, H, 0, q_scale, 0,
                            static_cast<cudaStream_t>(stream), bias_t, dbias_t);
}

int opb_relpos_bias_transpose(const float* bias, void* bias_t, int S, int s_pad, int H, void* stream) {
  if (!bias || !bias_t) return OPB_ERR_INVALID;
  return opb::relpos_bias_transpose(bias, bias_t, S, s_pad, H, static_cast<cudaStream_t>(stream));
}

int opb_relpos_dbias_fold(const float* dbias_t, float* dbias, int S, int s_pad, int H, void* stream) {
  if (!dbias_t || !dbias) return OPB_ERR_INVALID;
  return opb::relpos_dbias_fold(dbias_t, dbias, S, s_pad, H, static_cast<cudaStream_t>(stream));
}

int opb_relpos_dbias_center(float* dbias, int S, int s_pad, int H, void* stream) {
  if (!dbias) return OPB_ERR_INVALID;
  return opb::relpos_dbias_center(dbias, S, s_pad, H, static_cast<cudaStream_t>(stream));
}

int opb_relpos_bias_bwd(const float* dbias, const int64_t* bucket, float* dtable, int S, int s_pad, int H,
                        int64_t ld_bucket, void* stream) {
  if (!dbias || !bucket || !dtable) return OPB_ERR_INVALID;
  return opb::relpos_bias_bwd(dbias, bucket, dtable, S, s_pad, H, ld_bucket, static_cast<cudaStream_t>(stream));
}

int opb_topk10_rows(const float* sim, int64_t ld, int32_t* idx, float* val, int R, int C, void* stream) {
  if (!sim || !idx) return OPB_ERR_INVALID;
  return opb::topk10_rows(sim, ld, idx, val, R, C, static_cast<cudaStream_t>(stream));
}

int opb_recall_hits(const int32_t* idx, const int64_t* cand_ids, const int64_t* row_ids, int R, int32_t* hits,
                    void* stream) {
  if (!idx || !cand_ids || !row_ids || !hits) return OPB_ERR_INVALID;
  return opb::recall_hits(idx, cand_ids, row_ids, R, hits, static_cast<cudaStream_t>(stream));
}

int opb_row_gather(const void* src, int src_dtype, int64_t ld_src, const int64_t* idx, const float* fill, const float* add,
                   int64_t add_period, void* out, int out_dtype, int64_t ld_out, int64_t rows, int dim, void* stream) {
  if (!src || !idx || !out) return OPB_ERR_INVALID;
  return opb::row_gather(src, src_dtype, ld_src, idx, fill, add, add_period, out, out_dtype, ld_out, rows, dim,
                         static_cast<cudaStream_t>(stream));
}

int opb_row_scatter_add(const void* dout, int dout_dtype, int64_t ld_dout, const int64_t* idx, float* dsrc, int64_t ld_dsrc,
                        int64_t rows, int dim, void* stream) {
  if (!dout || !idx || !dsrc) return OPB_ERR_INVALID;
  return opb::row_scatter_add(dout, dout_dtype, ld_dout, idx, dsrc, ld_dsrc, rows, dim, static_cast<cudaStream_t>(stream));
}

int opb_relpos_bias_block(const float* table, const int64_t* bucket, int64_t ld_bucket, const int64_t* ids, int64_t ids_ld,
                          int Bb, int n, int lo, float* bias, int S, int s_pad, int H, void* stream) {
  if (!table || !bucket || !bias) return OPB_ERR_INVALID;
  return opb::relpos_bias_block(table, bucket, ld_bucket, ids, ids_ld, Bb, n, lo, bias, S, s_pad, H,
                                static_cast<cudaStream_t>(stream));
}

int opb_relpos_bias_block_bwd(const float* dbias, const int64_t* bucket, int64_t ld_bucket, const int64_t* ids,
                              int64_t ids_ld, int Bb, int n, int lo, float* dtable, int S, int s_pad, int H, void* stream) {
  if (!dbias || !bucket || !dtable) return OPB_ERR_INVALID;
  return opb::relpos_bias_block_bwd(dbias, bucket, ld_bucket, ids, ids_ld, Bb, n, lo, dtable, S, s_pad, H,
                                    static_cast<cudaStream_t>(stream));
}

int opb_gemm_bf16_t(const void* A, int64_t lda, int a_mn, const void* B, int64_t ldb, int b_mn, int M, int N, int K, int epilogue,
                    void* out, int64_t ldo, const float* bias, int cta_group, void* stream) {
  if (!A || !B || !out) return OPB_ERR_INVALID;
  opb::GemmEpilogue ep;
  ep.out = out;
  ep.ldo = ldo;
  ep.bias = bias;
  return opb::gemm_bf16_t(A, static_cast<int>(lda), a_mn, B, static_cast<int>(ldb), b_mn, M, N, K, epilogue, ep, cta_group,
                          static_cast<cudaStream_t>(stream));
}

int opb_ln_fold(const void* W, int w_dtype, int64_t ldw, const float* ln_weight, const float* ln_bias, const float* bias_in,
                int N, int K, int interleave, void* out_w, int64_t ldo, float* colsum, float* bias_out, void* stream) {
  if (!W || !out_w || !colsum || !bias_out) return OPB_ERR_INVALID;
  return opb::ln_fold(W, w_dtype, ldw, ln_weight, ln_bias, bias_in, N, K, interleave, out_w, ldo, colsum, bias_out,
                      static_cast<cudaStream_t>(stream));
}

int opb_attn_pool_fwd(const void* kv, const float* q, const uint8_t* key_pad, void* out, float* lse, int B, int T, int d,
                      void* stream) {
  if (!kv || !q || !out || !lse) return OPB_ERR_INVALID;
  return opb::attn_pool_fwd(kv, q, key_pad, out, lse, B, T, d, static_cast<cudaStream_t>(stream));
}

int opb_attn_pool_bwd(const void* kv, const float* q, const uint8_t* key_pad, const float* lse, const void* dout, void* dkv,
                      float* dq_ws, float* dq, int B, int T, int d, void* stream) {
  if (!kv || !q || !lse || !dout || !dkv || !dq_ws || !dq) return OPB_ERR_INVALID;
  return opb::attn_pool_bwd(kv, q, key_pad, lse, dout, dkv, dq_ws, dq, B, T, d, static_cast<cudaStream_t>(stream));
}

int opb_classify_loss(const float* logits, int64_t ld, int rows, int n_valid, int mode, const int64_t* labels,
                      const float* targets, int64_t ld_t, float eps, int num_choices, float* row_loss, float* dlogits,
                      float* row_correct, float* out2, unsigned int* ticket, void* stream) {
  if (!logits || !row_loss || !dlogits || !row_correct || !out2 || !ticket) return OPB_ERR_INVALID;
  return opb::classify_loss(logits, ld, rows, n_valid, mode, labels, targets, ld_t, eps, num_choices, row_loss, dlogits,
                            row_correct, out2, ticket, static_cast<cudaStream_t>(stream));
}

int opb_refcoco_loss(const float* logits, int64_t ld, const float* targets, int B, int nsentences, float* out, int* valid,
                     float* giou, float* dlogits, void* stream) {
  if (!logits || !targets || !out || !valid || !giou || !dlogits) return OPB_ERR_INVALID;
  return opb::refcoco_loss(logits, ld, targets, B, nsentences, out, valid, giou, dlogits, static_cast<cudaStream_t>(stream));
}

int opb_iou_acc(const float* hyps, int64_t ld_h, const float* refs, int64_t ld_r, int n, int* hits, int* row_hit, void* stream) {
  if (!hyps || !refs || !hits) return OPB_ERR_INVALID;
  return opb::iou_acc(hyps, ld_h, refs, ld_r, n, hits, row_hit, static_cast<cudaStream_t>(stream));
}

int opb_argmax_hits(const void* logits, int dtype, int64_t ld, int64_t cs, int n, int C, const void* targets, int tmode,
                    int64_t ldt, int64_t* hyp, float* score, void* stream) {
  if (!logits || !targets || !hyp || !score) return OPB_ERR_INVALID;
  return opb::argmax_hits(logits, dtype, ld, cs, n, C, targets, tmode, ldt, hyp, score, static_cast<cudaStream_t>(stream));
}

int opb_sum_f64(const float* x, int64_t n, double* out, void* stream) {
  if (!x || !out) return OPB_ERR_INVALID;
  return opb::sum_f64(x, n, out, static_cast<cudaStream_t>(stream));
}

int opb_sigmoid_pack(const void* logits, int dtype, int64_t ld, int64_t cs, const float* targets, int64_t ldt, int n, int C,
                     float* probs, uint8_t* labels, int64_t row_offset, int* flags, void* stream) {
  if (!logits || !targets || !probs || !labels || !flags) return OPB_ERR_INVALID;
  return opb::sigmoid_pack(logits, dtype, ld, cs, targets, ldt, n, C, probs, labels, row_offset, flags,
                           static_cast<cudaStream_t>(stream));
}

int64_t opb_average_precision_ws_bytes(int N, int C) { return opb::average_precision_ws_bytes(N, C); }

int opb_average_precision(const float* probs, const uint8_t* labels, int N, int C, void* ws, int64_t ws_bytes, double* ap,
                          double* mean, int64_t* npos, void* stream) {
  if (!probs || !labels || !ws || !ap || !mean || !npos) return OPB_ERR_INVALID;
  return opb::average_precision(probs, labels, N, C, ws, ws_bytes, ap, mean, npos, static_cast<cudaStream_t>(stream));
}

int64_t opb_token_mean_ln_ws_floats(int B, int S, int d) { return opb::token_mean_ln_ws_floats(B, S, d); }

int opb_token_mean_ln_fwd(const float* x, int64_t ld, int B, int S, int d, const float* gamma, const float* beta, float eps,
                          float* ws, int64_t ws_floats, float* m, void* y, float* mean, float* rstd, void* stream) {
  if (!x || !gamma || !beta || !ws || !m || !y || !mean || !rstd) return OPB_ERR_INVALID;
  return opb::token_mean_ln_fwd(x, ld, B, S, d, gamma, beta, eps, ws, ws_floats, m, y, mean, rstd,
                                static_cast<cudaStream_t>(stream));
}

int opb_token_mean_ln_bwd(const float* dy, const float* m, const float* mean, const float* rstd, const float* gamma, int B,
                          int S, int d, float* dgamma, float* dbeta, float* ws, float* dx, int64_t ld_dx, void* stream) {
  if (!dy || !m || !mean || !rstd || !gamma || !dgamma || !dbeta || !ws || !dx) return OPB_ERR_INVALID;
  return opb::token_mean_ln_bwd(dy, m, mean, rstd, gamma, B, S, d, dgamma, dbeta, ws, dx, ld_dx,
                                static_cast<cudaStream_t>(stream));
}

}  // extern "C"
