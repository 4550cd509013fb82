// Fused self-attention for the modality-shared encoder (reference: multihead_attention.py:103-115,
// transformer_encoder.py:144-162):
//     P = softmax_fp32( q k^T + relpos_bias[h] (+ -inf on padded keys) ),  o = P v
// q is already scaled (the QKV GEMM epilogue applies head_dim^-0.5 after the bias, as the reference
// does).  The (B,H,S,S) bias tensor the reference materialises is never built: the kernel reads the
// batch-shared (H,S,S_pad) fp32 table (1.9-3.7 MB, L2 resident) and the (B,S) key-padding mask.
//
// Layout: qkv is the QKV-GEMM output [B*S, 3*H*64] bf16 (q | k | v); out is [B*S, H*64] bf16.
// One CTA = one (head, 64-query chunk, batch element); 4 warps x 16 query rows; keys streamed in blocks of 64
// through double-buffered shared memory (cp.async); online softmax in fp32; scores and P.V on mma.sync.m16n8k16
// bf16 tensor cores (sequence lengths here are 17..750, i.e. 1.6 % of the layer FLOPs — see SURVEY.md 7, "hard
// parts").  Each thread reads the bias of its two query rows straight from the fp32 table (L2 resident) or gathers
// it from the LUT.  Warps whose 16 query rows are all >= S and key n-tiles / k-steps that are all >= S are skipped
// (S = 197 = 3*64 + 5 leaves mostly-empty edge tiles).
//
// Sequences of at most kAttnShortMaxS tokens run on the wgmma kernel of attention_wgmma.cu instead (see launch_fwd).
#include "common.cuh"
#include "ops.h"

namespace opb {

constexpr int kHd = 64;          // head dim (all ONE-PEACE configs: 1536/24 = 256/4 = 64)
constexpr int kQTile = 64;       // query rows per CTA
constexpr int kKTile = 64;       // keys per smem stage
constexpr int kRowPad = 72;      // smem row pitch in bf16 (144 B) -> conflict-free ldmatrix

OPB_DEVICE void cp_async16(void* dst, const void* src, bool valid) {
  uint32_t d = smem_u32(dst);
  int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(src), "r"(sz) : "memory");
}
OPB_DEVICE void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
OPB_DEVICE void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

OPB_DEVICE void ldmatrix_x4(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p)));
}
OPB_DEVICE void ldmatrix_x4_trans(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p)));
}
OPB_DEVICE void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

struct AttnSmem {
  __nv_bfloat16 q[kQTile][kRowPad];
  __nv_bfloat16 k[2][kKTile][kRowPad];
  __nv_bfloat16 v[2][kKTile][kRowPad];
};
static_assert(sizeof(AttnSmem) <= 48 * 1024, "launched without an opt-in for more dynamic shared memory");

OPB_DEVICE float lut_bias(const LutBias& lb, const float* lut_h, int crow, int qrow, int key, int S) {
  if (qrow >= S || key >= S || (lb.seg_split > 0 && ((qrow < lb.seg_split) != (key < lb.seg_split)))) return 0.f;
  return lut_h[crow - lb.code_col[key]];
}

__global__ void __launch_bounds__(128, 4)
attention_fwd_kernel(const __nv_bfloat16* __restrict__ qkv, const float* __restrict__ bias,
                     const uint8_t* __restrict__ key_pad, __nv_bfloat16* __restrict__ out, float* __restrict__ lse,
                     float* __restrict__ ln_stats, int B, int S, int H, int s_pad, long bias_bstride,
                     const LutBias lb) {
  extern __shared__ __align__(16) uint8_t attn_smem_raw[];
  AttnSmem& sm = *reinterpret_cast<AttnSmem*>(attn_smem_raw);

  const int q_chunks = (S + kQTile - 1) / kQTile;
  const int chunk = blockIdx.x % q_chunks;
  const int h = (blockIdx.x / q_chunks) % H;
  const int b = blockIdx.x / (q_chunks * H);
  const int D = H * kHd;
  const long row_pitch = 3L * D;
  const int q0 = chunk * kQTile;
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int num_kblocks = (S + kKTile - 1) / kKTile;
  const bool warp_active = (q0 + warp * 16) < S;       // warp-uniform: all 16 rows of this warp are padding otherwise

  const int qrow_lo = q0 + warp * 16 + g;   // this thread's two query rows
  const int qrow_hi = qrow_lo + 8;
  // bias_bstride != 0: one (H,S,s_pad) table per batch element (preserve_ids gathers, adapter/text.py:92-101)
  const float* bias_lo = bias ? bias + b * bias_bstride + (static_cast<long>(h) * S + (qrow_lo < S ? qrow_lo : 0)) * s_pad : nullptr;
  const float* bias_hi = bias ? bias + b * bias_bstride + (static_cast<long>(h) * S + (qrow_hi < S ? qrow_hi : 0)) * s_pad : nullptr;

  const float* lut_h = lb.lut != nullptr ? lb.lut + static_cast<long>(h) * lb.lut_len : nullptr;
  const int crow_lo = lut_h != nullptr ? lb.code_row[qrow_lo < S ? qrow_lo : 0] : 0;
  const int crow_hi = lut_h != nullptr ? lb.code_row[qrow_hi < S ? qrow_hi : 0] : 0;

  const __nv_bfloat16* qbase = qkv + (static_cast<long>(b) * S) * row_pitch + h * kHd;
  const __nv_bfloat16* kbase = qbase + D;
  const __nv_bfloat16* vbase = qbase + 2 * D;

  // --- async loads: Q tile, then K/V block 0 ---
  for (int i = tid; i < kQTile * 8; i += 128) {
    const int r = i >> 3, c = (i & 7) * 8;
    const bool ok = (q0 + r) < S;
    cp_async16(&sm.q[r][c], qbase + static_cast<long>(ok ? q0 + r : 0) * row_pitch + c, ok);
  }
  auto load_kv = [&](int kb, int buf) {
    const int k0 = kb * kKTile;
    for (int i = tid; i < kKTile * 8; i += 128) {
      const int r = i >> 3, c = (i & 7) * 8;
      const bool ok = (k0 + r) < S;
      const long off = static_cast<long>(ok ? k0 + r : 0) * row_pitch + c;
      cp_async16(&sm.k[buf][r][c], kbase + off, ok);
      cp_async16(&sm.v[buf][r][c], vbase + off, ok);
    }
  };
  load_kv(0, 0);
  cp_async_commit();

  uint32_t qf[4][4];
  float o[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
  float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;
  const uint8_t* kp = key_pad ? key_pad + static_cast<long>(b) * S : nullptr;

  for (int kb = 0; kb < num_kblocks; ++kb) {
    const int buf = kb & 1;
    if (kb + 1 < num_kblocks) load_kv(kb + 1, buf ^ 1);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();

    if (warp_active) {
      if (kb == 0) {
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          const int r = warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
          const int c = ks * 16 + (lane >> 4) * 8;
          ldmatrix_x4(qf[ks], &sm.q[r][c]);
        }
      }
      const int k0 = kb * kKTile;
      const int keys_here = min(kKTile, S - k0);
      const int nt_valid = (keys_here + 7) >> 3;      // key n-tiles (8 keys) with at least one real key
      const int kk_valid = (keys_here + 15) >> 4;     // P.V k-steps (16 keys) with at least one real key

      // ---- scores: 16 x 64 per warp ----
      float s[8][4];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
        if (nt < nt_valid) {
          uint32_t kf0[4], kf1[4];
          const int r = nt * 8 + (lane & 7);
          const int c = (lane >> 3) * 8;
          ldmatrix_x4(kf0, &sm.k[buf][r][c]);        // d 0..31
          ldmatrix_x4(kf1, &sm.k[buf][r][c + 32]);   // d 32..63
          mma16816(s[nt], qf[0], kf0[0], kf0[1]);
          mma16816(s[nt], qf[1], kf0[2], kf0[3]);
          mma16816(s[nt], qf[2], kf1[0], kf1[1]);
          mma16816(s[nt], qf[3], kf1[2], kf1[3]);
        }
      }

      // ---- bias, masks ----
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int key = k0 + nt * 8 + 2 * t;
        float b00 = 0.f, b01 = 0.f, b10 = 0.f, b11 = 0.f;
        if (bias != nullptr && key < S) {   // s_pad is even and >= S, so key + 1 is readable
          const float2 x = *reinterpret_cast<const float2*>(bias_lo + key);
          const float2 y = *reinterpret_cast<const float2*>(bias_hi + key);
          b00 = x.x; b01 = x.y; b10 = y.x; b11 = y.y;
        } else if (lut_h != nullptr && key < S) {
          b00 = lut_bias(lb, lut_h, crow_lo, qrow_lo, key, S); b01 = lut_bias(lb, lut_h, crow_lo, qrow_lo, key + 1, S);
          b10 = lut_bias(lb, lut_h, crow_hi, qrow_hi, key, S); b11 = lut_bias(lb, lut_h, crow_hi, qrow_hi, key + 1, S);
        }
        const bool dead0 = (key >= S) || (kp != nullptr && kp[key] != 0);
        const bool dead1 = (key + 1 >= S) || (kp != nullptr && kp[key + 1] != 0);
        s[nt][0] = dead0 ? -INFINITY : s[nt][0] + b00;
        s[nt][1] = dead1 ? -INFINITY : s[nt][1] + b01;
        s[nt][2] = dead0 ? -INFINITY : s[nt][2] + b10;
        s[nt][3] = dead1 ? -INFINITY : s[nt][3] + b11;
      }

      // ---- online softmax (rows g and g+8 of this warp's 16) ----
      float mx_lo = -INFINITY, mx_hi = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        mx_lo = fmaxf(mx_lo, fmaxf(s[nt][0], s[nt][1]));
        mx_hi = fmaxf(mx_hi, fmaxf(s[nt][2], s[nt][3]));
      }
      mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 1));
      mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 2));
      mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 1));
      mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 2));
      const float mn_lo = fmaxf(m_lo, mx_lo), mn_hi = fmaxf(m_hi, mx_hi);
      const float base_lo = (mn_lo == -INFINITY) ? 0.f : mn_lo;
      const float base_hi = (mn_hi == -INFINITY) ? 0.f : mn_hi;
      const float corr_lo = __expf(m_lo - base_lo), corr_hi = __expf(m_hi - base_hi);
      m_lo = mn_lo; m_hi = mn_hi;
      float sum_lo = 0.f, sum_hi = 0.f;
      uint32_t pf[8][2];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const float p0 = __expf(s[nt][0] - base_lo), p1 = __expf(s[nt][1] - base_lo);
        const float p2 = __expf(s[nt][2] - base_hi), p3 = __expf(s[nt][3] - base_hi);
        sum_lo += p0 + p1;
        sum_hi += p2 + p3;
        pf[nt][0] = pack_bf16x2(p0, p1);
        pf[nt][1] = pack_bf16x2(p2, p3);
      }
      l_lo = l_lo * corr_lo + sum_lo;
      l_hi = l_hi * corr_hi + sum_hi;
#pragma unroll
      for (int nd = 0; nd < 8; ++nd) {
        o[nd][0] *= corr_lo; o[nd][1] *= corr_lo;
        o[nd][2] *= corr_hi; o[nd][3] *= corr_hi;
      }

      // ---- O += P . V ----
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        if (kk < kk_valid) {
          uint32_t a[4] = {pf[2 * kk][0], pf[2 * kk][1], pf[2 * kk + 1][0], pf[2 * kk + 1][1]};
#pragma unroll
          for (int ndp = 0; ndp < 4; ++ndp) {
            uint32_t vf[4];
            const int r = kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
            const int c = ndp * 16 + (lane >> 4) * 8;
            ldmatrix_x4_trans(vf, &sm.v[buf][r][c]);
            mma16816(o[2 * ndp], a, vf[0], vf[1]);
            mma16816(o[2 * ndp + 1], a, vf[2], vf[3]);
          }
        }
      }
    }
    __syncthreads();   // everyone done with buf (and, on the last block, with q) before it is refilled
  }
  cp_async_wait<0>();

  // ---- finalize ----
  if (warp_active) {
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1);
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
    const float inv_lo = l_lo > 0.f ? 1.f / l_lo : 0.f;
    const float inv_hi = l_hi > 0.f ? 1.f / l_hi : 0.f;
    if (ln_stats != nullptr) {
      // per-(head, row) partial (sum, sum of squares) of the output row: the inner LayerNorm over all heads
      // (multihead_attention.py:122-123) is finished inside the out_proj GEMM epilogue
      float s_lo = 0.f, q_lo = 0.f, s_hi = 0.f, q_hi = 0.f;
#pragma unroll
      for (int nd = 0; nd < 8; ++nd) {
        const float a0 = o[nd][0] * inv_lo, a1 = o[nd][1] * inv_lo, a2 = o[nd][2] * inv_hi, a3 = o[nd][3] * inv_hi;
        s_lo += a0 + a1; q_lo += a0 * a0 + a1 * a1;
        s_hi += a2 + a3; q_hi += a2 * a2 + a3 * a3;
      }
      s_lo += __shfl_xor_sync(0xffffffffu, s_lo, 1); s_lo += __shfl_xor_sync(0xffffffffu, s_lo, 2);
      q_lo += __shfl_xor_sync(0xffffffffu, q_lo, 1); q_lo += __shfl_xor_sync(0xffffffffu, q_lo, 2);
      s_hi += __shfl_xor_sync(0xffffffffu, s_hi, 1); s_hi += __shfl_xor_sync(0xffffffffu, s_hi, 2);
      q_hi += __shfl_xor_sync(0xffffffffu, q_hi, 1); q_hi += __shfl_xor_sync(0xffffffffu, q_hi, 2);
      const long rows_total = static_cast<long>(B) * S;
      if (t == 0 && qrow_lo < S)
        *reinterpret_cast<float2*>(ln_stats + (h * rows_total + static_cast<long>(b) * S + qrow_lo) * 2) = make_float2(s_lo, q_lo);
      if (t == 0 && qrow_hi < S)
        *reinterpret_cast<float2*>(ln_stats + (h * rows_total + static_cast<long>(b) * S + qrow_hi) * 2) = make_float2(s_hi, q_hi);
    }
    if (qrow_lo < S) {
      __nv_bfloat16* op = out + (static_cast<long>(b) * S + qrow_lo) * D + h * kHd + 2 * t;
#pragma unroll
      for (int nd = 0; nd < 8; ++nd)
        *reinterpret_cast<uint32_t*>(op + nd * 8) = pack_bf16x2(o[nd][0] * inv_lo, o[nd][1] * inv_lo);
      if (lse != nullptr && t == 0) lse[(static_cast<long>(b) * H + h) * S + qrow_lo] = m_lo + __logf(l_lo);
    }
    if (qrow_hi < S) {
      __nv_bfloat16* op = out + (static_cast<long>(b) * S + qrow_hi) * D + h * kHd + 2 * t;
#pragma unroll
      for (int nd = 0; nd < 8; ++nd)
        *reinterpret_cast<uint32_t*>(op + nd * 8) = pack_bf16x2(o[nd][2] * inv_hi, o[nd][3] * inv_hi);
      if (lse != nullptr && t == 0) lse[(static_cast<long>(b) * H + h) * S + qrow_hi] = m_hi + __logf(l_hi);
    }
  }
}

static int launch_fwd(const void* qkv, const float* bias, const uint8_t* key_pad, void* out, float* lse, float* ln_stats,
                      int B, int S, int H, int s_pad, long bias_bstride, const LutBias& lb, cudaStream_t stream) {
  if (B <= 0 || S <= 0 || H <= 0) return OPB_ERR_INVALID;
  if (bias != nullptr && (s_pad < S || (s_pad & 3))) return OPB_ERR_INVALID;
  if (S <= kAttnShortMaxS && lb.lut_len <= kAttnShortMaxLut)
    return attention_fwd_short(qkv, bias, key_pad, out, lse, ln_stats, B, S, H, s_pad, bias_bstride, lb, stream);
  const int q_chunks = (S + kQTile - 1) / kQTile;
  const long grid = static_cast<long>(H) * q_chunks * B;
  attention_fwd_kernel<<<static_cast<unsigned>(grid), 128, sizeof(AttnSmem), stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(qkv), bias, key_pad, reinterpret_cast<__nv_bfloat16*>(out), lse, ln_stats,
      B, S, H, s_pad, bias_bstride, lb);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

int attention_fwd(const void* qkv, const float* bias, const uint8_t* key_pad, void* out, float* lse, float* ln_stats,
                  int B, int S, int H, int s_pad, long bias_bstride, cudaStream_t stream) {
  return launch_fwd(qkv, bias, key_pad, out, lse, ln_stats, B, S, H, s_pad, bias_bstride, LutBias(), stream);
}

// Same kernel with the LUT form of the bias (no (H, S, S_pad) table is read).  `lut_max` (a per-head upper bound of the
// bias) is part of the C ABI but not needed by the online soft-max.
int attention_lut_fwd(const void* qkv, const float* lut, int lut_len, const int* code_row, const int* code_col,
                      const uint8_t* key_pad, void* out, float* lse, float* ln_stats, int B, int S, int H, int seg_split,
                      cudaStream_t stream) {
  if (B <= 0 || S <= 0 || H <= 0 || lut_len <= 0 || seg_split < 0 || seg_split >= S) return OPB_ERR_INVALID;
  LutBias lb;
  lb.lut = lut; lb.lut_len = lut_len; lb.code_row = code_row; lb.code_col = code_col; lb.seg_split = seg_split;
  return launch_fwd(qkv, nullptr, key_pad, out, lse, ln_stats, B, S, H, 0, 0, lb, stream);
}

// lut[h][l] = table[idx[l]][h]
__global__ void relpos_lut_kernel(const float* __restrict__ table, const int* __restrict__ idx, float* __restrict__ lut,
                                  int L, int H) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= L) return;
  const long bk = idx[l];
  for (int h = 0; h < H; ++h) lut[static_cast<long>(h) * L + l] = table[bk * H + h];
}

int relpos_lut_build(const float* table, const int* idx, float* lut, int L, int H, cudaStream_t stream) {
  if (L <= 0 || H <= 0) return OPB_ERR_INVALID;
  relpos_lut_kernel<<<(L + 255) / 256, 256, 0, stream>>>(table, idx, lut, L, H);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

}  // namespace opb
