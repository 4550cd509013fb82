// Internal (C++) interface of the wgmma GEMM; the C-ABI wrappers live in c_abi.cu.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace opb {

enum GemmEpi : int {
  EPI_STORE_BF16 = 0,  // out_bf16 = (acc + bias) * colscale
  EPI_GEGLU_BF16 = 1,  // out_bf16[:, t*128 + j] = gelu(acc[:, j]) * acc[:, 128 + j]   (N/2 output columns)
  EPI_RESID_F32 = 2,   // out_f32 = resid + gamma * (acc + bias)
  EPI_STORE_F32 = 3,   // out_f32 = acc + bias
  EPI_GELU_BF16 = 4,   // out_bf16 = gelu((acc + bias) * colscale)
  // contrastive head (criterions/image_text_retrieval_loss.py:91-112), z = scale * acc:
  EPI_LSE_PARTIAL = 5,   // per (row, 256-col tile): running max / sum-exp / sum z / arg-max / target logit -> ws
  EPI_SOFTMAX_GRAD = 6,  // out_bf16 = coef*scale * (exp(z - lse[row]) - (1-eps-eps_i)[col==target] - eps_i); sum_j g*z -> ws
};

struct GemmEpilogue {
  void* out = nullptr;             // bf16 or fp32, see GemmEpi
  long ldo = 0;                    // output row pitch, elements
  const float* bias = nullptr;     // [N] or null
  const float* colscale = nullptr; // [N] or null
  const float* gamma = nullptr;    // [N] or null (EPI_RESID_F32)
  // fp32 residual or null (EPI_RESID_F32).  It may overlap the outputs only as the in-place update: resid == out, ldr == ldo
  // and resid_period == 0 (anything else is refused, see resid_aliasing_ok in gemm_wgmma.cu)
  const float* resid = nullptr;
  long ldr = 0;                    // residual row pitch
  // optional row remapping: out_row = (m / out_group) * out_group_stride + (m % out_group) + out_row_offset
  int out_group = 0;
  int out_group_stride = 0;
  int out_row_offset = 0;
  int out_group_valid = 0;         // if > 0: rows with (m % out_group) >= out_group_valid are not stored
  // optional broadcast residual: resid_row = (m % resid_period) + resid_row_offset
  int resid_period = 0;
  int resid_row_offset = 0;
  // Fused LayerNorm of the A operand (A holds the UN-normalised rows in bf16, B holds W * diag(ln_weight)):
  //   LN(x) W^T + b = rstd[m] * (acc - mu[m] * colsum[n]) + bias'[n],  colsum[n] = sum_k B[n,k],
  //   bias'[n] = sum_k ln_bias[k] W[n,k] + b[n]  (passed through `bias`)
  const float* ln_mu = nullptr;      // [M]
  const float* ln_rstd = nullptr;    // [M]
  const float* ln_colsum = nullptr;  // [N]
  // alternative to ln_mu / ln_rstd: the producer's partial (sum, sum of squares) records [ln_parts, M, 2]; each
  // epilogue thread reduces the records of its row itself (index order -> deterministic), which removes the separate
  // ln_stats_finalize launch for small part counts (6 for the residual GEMMs, 24 for attention)
  const float* ln_partial = nullptr;
  int ln_parts = 0;
  int ln_dim = 0;
  float ln_eps = 1e-5f;
  // side outputs for the NEXT LayerNorm (EPI_RESID_F32 / EPI_GEGLU_BF16): per (n-tile, row) partial (sum, sum of
  // squares) of the stored values, and (EPI_RESID_F32) a bf16 copy of the output that feeds the next GEMM
  float* stats_out = nullptr;        // [n_tiles, M, 2]
  void* out_bf16 = nullptr;
  long ldo_bf16 = 0;
  // optional fp32 scratch (one [M rounded up to 128, N] slab per piece) enabling the small-M split-K schedule of the
  // EPI_RESID_F32 / EPI_STORE_BF16 GEMMs (M <= 256)
  void* workspace = nullptr;
  long workspace_bytes = 0;
  // contrastive-head epilogues
  const float* scale_ptr = nullptr;  // device scalar: exp(clamp(logit_scale))
  const float* row_lse = nullptr;    // [M] log-sum-exp per row (EPI_SOFTMAX_GRAD)
  float* ws = nullptr;               // EPI_LSE_PARTIAL: [n_tiles, M, 8];  EPI_SOFTMAX_GRAD: [n_tiles, M]
  int target_offset = 0;             // target column of row m is m + target_offset (rank * local batch)
  float eps = 0.f;                   // label smoothing
  float eps_i = 0.f;                 // eps / (N - 1)
  float coef = 1.f;                  // 1 / (2 b)
  int n_valid = 0;                   // > 0: only columns < n_valid are classes (B rows beyond it are zero padding up to N % 8 == 0)
};

// C = epilogue(A[M,K] . B[N,K]^T); A, B bf16 row-major with pitches lda, ldb (elements).
// cta_group: 0, 1 or 2, accepted for compatibility and unused (every tile is 128 x 256).  Returns an OPB_* status.
int gemm_bf16(const void* A, int lda, const void* B, int ldb, int M, int N, int K, int epi, const GemmEpilogue& ep,
              int cta_group, cudaStream_t stream);

// Same with MN-major operands: a_mn != 0 -> A is given as [K, M] row-major (C = A^T-stored^T ...), b_mn != 0 -> B as [K, N]
// row-major.  dW = dY^T X is gemm_bf16_t(dY, ldy, 1, X, ldx, 1, N_out, K_in, rows, ...): no transposed copies.
int gemm_bf16_t(const void* A, int lda, int a_mn, const void* B, int ldb, int b_mn, int M, int N, int K, int epi,
                const GemmEpilogue& ep, int cta_group, cudaStream_t stream);

// Grouped "sliding window" GEMM = grouped Conv1d over channel-last activations:
//   out[r, g*n_per_group + n] = epilogue( sum_{j < taps} sum_{c < c_pad} X[(r + j), g, c] * W[g*n_per_group + n, j*c_pad + c] )
// X is bf16 [rows + taps - 1, groups, c_pad] (c_pad a multiple of 64), W is bf16 [groups*n_per_group, taps*c_pad].
// TMA map of a batch of bf16 row-major matrices (csrc/attention_wgmma.cu): dims {cols, rows, batches}, pitches ld and
// batch_stride (elements), box = 64 cols x box_rows x 1 with the 128-byte swizzle.
int make_tmap_bf16_batched(CUtensorMap* out, const void* ptr, uint64_t cols, uint64_t rows, uint64_t ld, uint64_t batches,
                           uint64_t batch_stride, uint32_t box_rows);

int gemm_bf16_grouped_window(const void* X, const void* W, int rows, int groups, int c_pad, int taps, int n_per_group,
                             int epi, const GemmEpilogue& ep, cudaStream_t stream);

}  // namespace opb
