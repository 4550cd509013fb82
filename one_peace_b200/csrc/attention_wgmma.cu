// Attention forward for sequences of at most kAttnShortMaxS = 224 tokens, on wgmma.  Same contract as attention_fwd_kernel
// in attention.cu (every bias form, key padding, optional lse / ln_stats), with a structure that fits short rows:
//   * work unit = (sample b, head h).  A persistent grid of one CTA per SM walks the units with a fixed stride, so K and V
//     are read from global memory once per unit instead of once per 64-query chunk;
//   * warpgroup 0 (registers lowered with setmaxnreg): one thread loads the unit's Q, K and V by TMA in 64-column x 32-row
//     boxes of qkv viewed as [B][S][3 * D] (rows >= S zero-filled, nothing of the next sample is read); warps 1-3 copy
//     the head's LUT row and the sample's key-padding row into shared memory, so every score's bias is a shared-memory
//     gather.  The whole unit is double-buffered behind full / empty mbarriers: unit n + 1 loads while unit n computes;
//   * warpgroups 1 and 2 split the unit's 64-row query tiles.  S = Q K^T runs on wgmma.m64n32k16 (Q and K K-major from
//     shared memory, keys in chunks of 32), so a row of up to 224 scores stays whole in registers (112 per thread) and the
//     soft-max needs no online rescale.  P is rounded to bf16 A fragments in registers and O = P V runs on
//     wgmma.m64n64k16 with V as the MN-major B operand.
// The accumulator fragment holds rows g, g + 8 and columns 2t, 2t + 1 of every 8-column group, as mma.sync.m16n8 does, so
// bias, masking (by select: dense tables hold NaN in their pad columns), soft-max and the finalisation are those of
// attention.cu.  Output rows >= S are never stored: in [B * S, D] they belong to the next sample.
#include "common.cuh"
#include "gemm.h"
#include "ops.h"

namespace opb {
namespace {

constexpr int kHd = 64;
constexpr int kThreads = 384;
constexpr int kStagerThreads = 96;                 // warps 1-3 of warpgroup 0
constexpr int kBoxRows = 32;                       // TMA box: 64 columns (128 B) x 32 rows
constexpr int kBoxBytes = kBoxRows * 128;
constexpr int kKeyChunks = kAttnShortMaxS / 32;    // 32-key wgmma chunks of the longest row

// One unit's buffer (all offsets 1024-aligned where the 128-byte swizzle needs it)
constexpr int kOffQ = 0;                                        // 4 query tiles of 64 rows x 128 B
constexpr int kOffK = kOffQ + 4 * 64 * 128;                     // keys: up to 224 rows x 128 B
constexpr int kOffV = kOffK + kAttnShortMaxS * 128;
constexpr int kOffLut = kOffV + kAttnShortMaxS * 128;           // fp32 LUT row of head h
constexpr int kOffPad = kOffLut + kAttnShortMaxLut * 4;         // key_pad row of sample b
constexpr int kBufBytes = (kOffPad + kAttnShortMaxS + 1023) / 1024 * 1024;
constexpr int kOffCodes = 2 * kBufBytes;                        // code_row[224], code_col[224]: once per CTA
constexpr int kOffBars = kOffCodes + 2 * kAttnShortMaxS * 4;
constexpr int kSmemBytes = kOffBars + 64 + 1024;                // + barriers + alignment slack
static_assert(kSmemBytes <= 227 * 1024, "one CTA per SM");

enum BiasForm : int { kNoBias = 0, kDense = 1, kLut = 2, kLutSeg = 3 };   // kLutSeg: two-segment LUT

struct ShortArgs {
  const float* bias;          // dense (H, S, s_pad) table, per sample bias_bstride apart
  long bias_bstride;
  int s_pad;
  LutBias lb;
  const uint8_t* key_pad;     // [B, S] or null
  __nv_bfloat16* out;         // [B * S, D]
  float* lse;                 // [B, H, S] or null
  float* ln_stats;            // [H, B * S, 2] or null
  int B, S, H;
};

// D[64 x 32] (+)= A[64 x 16] . B[32 x 16]^T, A and B K-major in shared memory
OPB_DEVICE void wgmma_m64n32k16_ss(float (&d)[16], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d));
}

// D[64 x 64] (+)= A[64 x 16] . B[16 x 64], A bf16 fragments in registers, B MN-major in shared memory
OPB_DEVICE void wgmma_m64n64k16_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(scale_d));
}

// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma window
template <int N>
OPB_DEVICE void fence_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

OPB_DEVICE float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
OPB_DEVICE float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// Dense form: this thread's bias of 32-key chunk c, rows lo / hi (s_pad is even and >= S, so key + 1 is readable).
OPB_DEVICE void load_bias_chunk(float2 (&dst)[4][2], const float* bias_lo, const float* bias_hi, int c, int t, int S) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int key = (4 * c + j) * 8 + 2 * t;
    dst[j][0] = key < S ? *reinterpret_cast<const float2*>(bias_lo + key) : make_float2(0.f, 0.f);
    dst[j][1] = key < S ? *reinterpret_cast<const float2*>(bias_hi + key) : make_float2(0.f, 0.f);
  }
}

// One 64-row query tile `qt` of unit (b, h) on one consumer warpgroup; `buf` holds the unit's operands.
template <int kForm, int kChunks>
OPB_DEVICE void attend_tile(const ShortArgs& a, const uint8_t* buf, const int* code_row_s, const int* code_col_s, int b,
                            int h, int qt) {
  const int S = a.S, D = a.H * kHd;
  const int warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int row_lo = qt * 64 + warp * 16 + g, row_hi = row_lo + 8;   // this thread's two query rows
  const int rl = row_lo < S ? row_lo : 0, rh = row_hi < S ? row_hi : 0;   // rows >= S compute row 0's bias (never stored)
  // A warp whose 16 query rows are all >= S (3 of the 4 in the last tile at S = 197) only takes part in the wgmmas.
  const bool warp_live = qt * 64 + warp * 16 < S;

  // Dense form: the bias of two 32-key chunks is in flight at a time, the first two while Q K^T runs.  A __syncwarp per
  // chunk (its memory ordering) keeps ptxas from hoisting every load, which costs 2 x 112 registers and spills.
  const float* bias_lo = nullptr;
  const float* bias_hi = nullptr;
  float2 pre[2][4][2];
  if (kForm == kDense && warp_live) {
    bias_lo = a.bias + b * a.bias_bstride + (static_cast<long>(h) * S + rl) * a.s_pad;
    bias_hi = a.bias + b * a.bias_bstride + (static_cast<long>(h) * S + rh) * a.s_pad;
    load_bias_chunk(pre[0], bias_lo, bias_hi, 0, t, S);
    if (kChunks > 1) load_bias_chunk(pre[1], bias_lo, bias_hi, 1, t, S);
  }

  // ---- scores: 64 x (32 * kChunks) ----
  float s[kChunks][16];
  const uint32_t q_addr = smem_u32(buf + kOffQ) + qt * 8192;
  const uint32_t k_addr = smem_u32(buf + kOffK);
  wgmma_fence();
#pragma unroll
  for (int c = 0; c < kChunks; ++c) {
#pragma unroll
    for (int k = 0; k < 4; ++k)
      wgmma_m64n32k16_ss(s[c], wgmma_desc_sw128(q_addr + 32 * k, 8192), wgmma_desc_sw128(k_addr + c * 4096 + 32 * k, 8192),
                         k > 0 ? 1u : 0u);
  }
  wgmma_commit();
  wgmma_wait<0>();
#pragma unroll
  for (int c = 0; c < kChunks; ++c) fence_regs(s[c]);

  // ---- bias, masks, row maxima, soft-max ----
  float mx_lo = -INFINITY, mx_hi = -INFINITY, sum_lo = 0.f, sum_hi = 0.f;
  uint32_t pf[4 * kChunks][2];
  if (warp_live) {
    const uint8_t* kp = a.key_pad != nullptr ? buf + kOffPad : nullptr;
    const float* lut_s = reinterpret_cast<const float*>(buf + kOffLut);
    const int crow_lo = kForm >= kLut ? code_row_s[rl] : 0;
    const int crow_hi = kForm >= kLut ? code_row_s[rh] : 0;
    const int seg = a.lb.seg_split;
    const bool first_lo = rl < seg, first_hi = rh < seg;
#pragma unroll
    for (int nt = 0; nt < 4 * kChunks; ++nt) {
      const int c = nt >> 2, e = (nt & 3) * 4;
      const int key = nt * 8 + 2 * t;
      float b00 = 0.f, b01 = 0.f, b10 = 0.f, b11 = 0.f;
      if (kForm == kDense) {
        if ((nt & 3) == 0) __syncwarp();
        const float2 x = pre[c & 1][nt & 3][0], y = pre[c & 1][nt & 3][1];
        b00 = x.x; b01 = x.y; b10 = y.x; b11 = y.y;
        if ((nt & 3) == 3 && c + 2 < kChunks) load_bias_chunk(pre[c & 1], bias_lo, bias_hi, c + 2, t, S);
      } else if (kForm == kLut) {
        // code_col_s holds code_col[S - 1] past S, so every gather stays inside the LUT row (keys >= S are masked below)
        const int2 cc = *reinterpret_cast<const int2*>(code_col_s + key);
        b00 = lut_s[crow_lo - cc.x]; b01 = lut_s[crow_lo - cc.y];
        b10 = lut_s[crow_hi - cc.x]; b11 = lut_s[crow_hi - cc.y];
      } else if (kForm == kLutSeg) {
        // zero across the two segments, where the code difference may leave the LUT row: gather entry 0 there instead
        const int2 cc = *reinterpret_cast<const int2*>(code_col_s + key);
        const bool kf0 = key < seg, kf1 = key + 1 < seg;
        const bool s00 = first_lo == kf0, s01 = first_lo == kf1, s10 = first_hi == kf0, s11 = first_hi == kf1;
        b00 = lut_s[s00 ? crow_lo - cc.x : 0]; b01 = lut_s[s01 ? crow_lo - cc.y : 0];
        b10 = lut_s[s10 ? crow_hi - cc.x : 0]; b11 = lut_s[s11 ? crow_hi - cc.y : 0];
        b00 = s00 ? b00 : 0.f; b01 = s01 ? b01 : 0.f;
        b10 = s10 ? b10 : 0.f; b11 = s11 ? b11 : 0.f;
      }
      bool dead0 = key >= S, dead1 = key + 1 >= S;
      if (kp != nullptr) {
        const uint32_t pair = *reinterpret_cast<const uint16_t*>(kp + key);
        dead0 = dead0 || (pair & 0xffu) != 0;
        dead1 = dead1 || (pair >> 8) != 0;
      }
      s[c][e + 0] = dead0 ? -INFINITY : s[c][e + 0] + b00;
      s[c][e + 1] = dead1 ? -INFINITY : s[c][e + 1] + b01;
      s[c][e + 2] = dead0 ? -INFINITY : s[c][e + 2] + b10;
      s[c][e + 3] = dead1 ? -INFINITY : s[c][e + 3] + b11;
      mx_lo = fmaxf(mx_lo, fmaxf(s[c][e + 0], s[c][e + 1]));
      mx_hi = fmaxf(mx_hi, fmaxf(s[c][e + 2], s[c][e + 3]));
    }
    mx_lo = quad_max(mx_lo);
    mx_hi = quad_max(mx_hi);

    // the denominator sums the unrounded fp32 p, P.V takes p rounded to bf16
    const float base_lo = (mx_lo == -INFINITY) ? 0.f : mx_lo;
    const float base_hi = (mx_hi == -INFINITY) ? 0.f : mx_hi;
#pragma unroll
    for (int nt = 0; nt < 4 * kChunks; ++nt) {
      const int c = nt >> 2, e = (nt & 3) * 4;
      const float p0 = __expf(s[c][e + 0] - base_lo), p1 = __expf(s[c][e + 1] - base_lo);
      const float p2 = __expf(s[c][e + 2] - base_hi), p3 = __expf(s[c][e + 3] - base_hi);
      sum_lo += p0 + p1;
      sum_hi += p2 + p3;
      pf[nt][0] = pack_bf16x2(p0, p1);
      pf[nt][1] = pack_bf16x2(p2, p3);
    }
  } else {
#pragma unroll
    for (int nt = 0; nt < 4 * kChunks; ++nt) pf[nt][0] = pf[nt][1] = 0u;
  }

  // ---- O = P . V (key steps of 16; keys >= S have p = 0 and zero-filled V rows, so they add exact zeros) ----
  float o[32];
  const uint32_t v_addr = smem_u32(buf + kOffV);
#pragma unroll
  for (int nt = 0; nt < 4 * kChunks; ++nt) asm volatile("" : "+r"(pf[nt][0]), "+r"(pf[nt][1])::"memory");
  fence_regs(o);
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < 2 * kChunks; ++kk) {
    const uint32_t af[4] = {pf[2 * kk][0], pf[2 * kk][1], pf[2 * kk + 1][0], pf[2 * kk + 1][1]};
    wgmma_m64n64k16_rs(o, af, wgmma_desc_sw128(v_addr + kk * 2048, 8192), kk > 0 ? 1u : 0u);
  }
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(o);

  // ---- finalise ----
  const float l_lo = quad_sum(sum_lo), l_hi = quad_sum(sum_hi);
  const float inv_lo = l_lo > 0.f ? 1.f / l_lo : 0.f;
  const float inv_hi = l_hi > 0.f ? 1.f / l_hi : 0.f;
  const long rows_total = static_cast<long>(a.B) * S;
  if (a.ln_stats != nullptr) {
    // per-(head, row) partial (sum, sum of squares) of the output row: the inner LayerNorm over all heads
    // (multihead_attention.py:122-123) is finished inside the out_proj GEMM epilogue
    float s_lo = 0.f, q_lo = 0.f, s_hi = 0.f, q_hi = 0.f;
#pragma unroll
    for (int nd = 0; nd < 8; ++nd) {
      const float a0 = o[4 * nd] * inv_lo, a1 = o[4 * nd + 1] * inv_lo;
      const float a2 = o[4 * nd + 2] * inv_hi, a3 = o[4 * nd + 3] * inv_hi;
      s_lo += a0 + a1; q_lo += a0 * a0 + a1 * a1;
      s_hi += a2 + a3; q_hi += a2 * a2 + a3 * a3;
    }
    s_lo = quad_sum(s_lo); q_lo = quad_sum(q_lo);
    s_hi = quad_sum(s_hi); q_hi = quad_sum(q_hi);
    if (t == 0 && row_lo < S)
      *reinterpret_cast<float2*>(a.ln_stats + (h * rows_total + static_cast<long>(b) * S + row_lo) * 2) = make_float2(s_lo, q_lo);
    if (t == 0 && row_hi < S)
      *reinterpret_cast<float2*>(a.ln_stats + (h * rows_total + static_cast<long>(b) * S + row_hi) * 2) = make_float2(s_hi, q_hi);
  }
  if (row_lo < S) {
    __nv_bfloat16* op = a.out + (static_cast<long>(b) * S + row_lo) * D + h * kHd + 2 * t;
#pragma unroll
    for (int nd = 0; nd < 8; ++nd)
      *reinterpret_cast<uint32_t*>(op + nd * 8) = pack_bf16x2(o[4 * nd] * inv_lo, o[4 * nd + 1] * inv_lo);
    if (a.lse != nullptr && t == 0) a.lse[(static_cast<long>(b) * a.H + h) * S + row_lo] = mx_lo + __logf(l_lo);
  }
  if (row_hi < S) {
    __nv_bfloat16* op = a.out + (static_cast<long>(b) * S + row_hi) * D + h * kHd + 2 * t;
#pragma unroll
    for (int nd = 0; nd < 8; ++nd)
      *reinterpret_cast<uint32_t*>(op + nd * 8) = pack_bf16x2(o[4 * nd + 2] * inv_hi, o[4 * nd + 3] * inv_hi);
    if (a.lse != nullptr && t == 0) a.lse[(static_cast<long>(b) * a.H + h) * S + row_hi] = mx_hi + __logf(l_hi);
  }
}

// Persistent: CTA i runs units i, i + gridDim.x, ... (unit = b * H + h); the j-th unit of a CTA uses buffer j & 1 and
// phase (j >> 1) & 1 of that buffer's barriers.
template <int kForm, int kChunks>
__global__ void __launch_bounds__(kThreads, 1)
attention_short_kernel(const __grid_constant__ CUtensorMap tm_qkv, const ShortArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  int* code_row_s = reinterpret_cast<int*>(smem + kOffCodes);
  int* code_col_s = code_row_s + kAttnShortMaxS;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kOffBars);   // [2] Q/K/V landed and the small operands staged
  uint64_t* empty = full + 2;                                     // [2] both consumer warpgroups are done with the buffer

  const int S = a.S, H = a.H, D = H * kHd;
  const int units = a.B * H;
  const int n_qt = (S + 63) / 64;   // query tiles; the kChunks = ceil(S / 32) key chunks are also the TMA boxes per operand
  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_qkv);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&full[i], 1 + kStagerThreads);
      mbar_init(&empty[i], 8);   // lane 0 of each of the 8 consumer warps
    }
    fence_barrier_init();
  }
  if (kForm >= kLut) {
    for (int i = threadIdx.x; i < kAttnShortMaxS; i += kThreads) {
      if (i < S) code_row_s[i] = a.lb.code_row[i];
      code_col_s[i] = a.lb.code_col[i < S ? i : S - 1];
    }
  }
  __syncthreads();

  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      // ===================== TMA producer =====================
      uint32_t j = 0;
      for (int unit = blockIdx.x; unit < units; unit += gridDim.x, ++j) {
        const int b = unit / H, h = unit - b * H;
        uint8_t* buf = smem + (j & 1) * kBufBytes;
        mbar_wait_quiet(&empty[j & 1], ((j >> 1) & 1) ^ 1);
        // box rows past S are zero-filled and counted; Q rows past 32 * kChunks of the last tile are not loaded (their
        // scores only reach rows >= S, which are never stored)
        mbar_arrive_expect_tx(&full[j & 1], 3 * kChunks * kBoxBytes);
        for (int i = 0; i < kChunks; ++i) {
          tma_load_3d(&tm_qkv, &full[j & 1], buf + kOffQ + i * kBoxBytes, h * kHd, i * kBoxRows, b);
          tma_load_3d(&tm_qkv, &full[j & 1], buf + kOffK + i * kBoxBytes, D + h * kHd, i * kBoxRows, b);
          tma_load_3d(&tm_qkv, &full[j & 1], buf + kOffV + i * kBoxBytes, 2 * D + h * kHd, i * kBoxRows, b);
        }
      }
    } else if (threadIdx.x >= 32) {
      // ===================== LUT row / key-padding stager (warps 1-3) =====================
      const int t = threadIdx.x - 32;
      uint32_t j = 0;
      for (int unit = blockIdx.x; unit < units; unit += gridDim.x, ++j) {
        const int b = unit / H, h = unit - b * H;
        uint8_t* buf = smem + (j & 1) * kBufBytes;
        mbar_wait_quiet(&empty[j & 1], ((j >> 1) & 1) ^ 1);
        if (kForm >= kLut) {
          const float* src = a.lb.lut + static_cast<long>(h) * a.lb.lut_len;
          float* dst = reinterpret_cast<float*>(buf + kOffLut);
          for (int i = t; i < a.lb.lut_len; i += kStagerThreads) dst[i] = src[i];
        }
        if (a.key_pad != nullptr) {
          const uint8_t* src = a.key_pad + static_cast<long>(b) * S;
          for (int i = t; i < S; i += kStagerThreads) buf[kOffPad + i] = src[i];
        }
        mbar_arrive(&full[j & 1]);
      }
    }
  } else {
    // ===================== consumers =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int cw = wg - 1;
    uint32_t j = 0;
    for (int unit = blockIdx.x; unit < units; unit += gridDim.x, ++j) {
      const int b = unit / H, h = unit - b * H;
      const uint8_t* buf = smem + (j & 1) * kBufBytes;
      mbar_wait_quiet(&full[j & 1], (j >> 1) & 1);
      for (int qt = cw; qt < n_qt; qt += 2) attend_tile<kForm, kChunks>(a, buf, code_row_s, code_col_s, b, h, qt);
      __syncwarp();
      if ((threadIdx.x & 31) == 0) mbar_arrive(&empty[j & 1]);
    }
  }
}

template <int kForm, int kChunks>
int launch_short(const CUtensorMap& tm, const ShortArgs& a, cudaStream_t stream) {
  auto kern = attention_short_kernel<kForm, kChunks>;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes) != cudaSuccess)
      return OPB_ERR_CUDA;
    attr_set = true;
  }
  const int units = a.B * a.H;
  const int grid = units < sm_count() ? units : sm_count();
  kern<<<grid, kThreads, kSmemBytes, stream>>>(tm, a);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

// wgmma's N is an immediate: one instantiation per 32-key chunk count
template <int kForm>
int launch_form(const CUtensorMap& tm, const ShortArgs& a, cudaStream_t stream) {
  static_assert(kKeyChunks == 7, "one case per chunk count");
  switch ((a.S + 31) / 32) {
    case 1: return launch_short<kForm, 1>(tm, a, stream);
    case 2: return launch_short<kForm, 2>(tm, a, stream);
    case 3: return launch_short<kForm, 3>(tm, a, stream);
    case 4: return launch_short<kForm, 4>(tm, a, stream);
    case 5: return launch_short<kForm, 5>(tm, a, stream);
    case 6: return launch_short<kForm, 6>(tm, a, stream);
    case 7: return launch_short<kForm, 7>(tm, a, stream);
    default: return OPB_ERR_INVALID;
  }
}

}  // namespace

int attention_fwd_short(const void* qkv, const float* bias, const uint8_t* key_pad, void* out, float* lse, float* ln_stats,
                        int B, int S, int H, int s_pad, long bias_bstride, const LutBias& lb, cudaStream_t stream) {
  if (B <= 0 || S <= 0 || H <= 0 || S > kAttnShortMaxS || lb.lut_len > kAttnShortMaxLut) return OPB_ERR_INVALID;
  const uint64_t D = static_cast<uint64_t>(H) * kHd;
  CUtensorMap tm;
  const int rc = make_tmap_bf16_batched(&tm, qkv, 3 * D, S, 3 * D, B, S * 3 * D, kBoxRows);
  if (rc != OPB_OK) return rc;
  ShortArgs a;
  a.bias = bias; a.bias_bstride = bias_bstride; a.s_pad = s_pad; a.lb = lb;
  a.key_pad = key_pad;
  a.out = reinterpret_cast<__nv_bfloat16*>(out); a.lse = lse; a.ln_stats = ln_stats;
  a.B = B; a.S = S; a.H = H;
  if (bias != nullptr) return launch_form<kDense>(tm, a, stream);
  if (lb.lut != nullptr) return lb.seg_split > 0 ? launch_form<kLutSeg>(tm, a, stream) : launch_form<kLut>(tm, a, stream);
  return launch_form<kNoBias>(tm, a, stream);
}

}  // namespace opb
