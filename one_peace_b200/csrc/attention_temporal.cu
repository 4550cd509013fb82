// Temporal attention of the video backbone (one_peace_vision/video/mmaction_custom/models/backbones/onepeace.py:331-337,
// num_tadapter = 1): for every clip b, token n and head h, softmax over the T frames of q_t . k_t', then P . V.  No bias,
// no padding, q already scaled by the QKV epilogue.
//
// Layout: qkv is the QKV-GEMM output [Bv * T * N, 3 * H * 64] bf16 in frame-major rows, row (b * T + t) * N + n; the T
// rows of one (b, n) are N rows apart and are read in place at that stride (no gather of the QKV tensor, no permutation
// back).  out [Bv * T * N, H * 64] bf16 uses the same rows.  ln_stats fp32 [H, M, 2] (M = Bv * T * N) holds each (head,
// row) (sum, sum of squares) of the fp32 output values before their bf16 rounding: opb_attention_fwd's records, which the
// out_proj GEMM reduces for the inner LayerNorm.
//
// One warp per (b, n, h): the warp stages its T (<= kTp) q / k / v rows in its own slice of shared memory with 16-byte
// cp.async (rows >= T zero-filled), computes the scores on mma.sync.m16n8k16 (one or two 16-row m-tiles), masks keys >= T,
// takes the softmax in fp32 registers and P . V on the same tensor cores.  The arithmetic per query row is the one of
// attention.cu's kernel for a single key block: the same max, __expf, fp32 row sum and bf16 P.
#include "common.cuh"
#include "ops.h"

namespace opb {
namespace {

constexpr int kHd = 64;
constexpr int kPitch = 72;       // smem row pitch in bf16 (144 B): conflict-free ldmatrix

OPB_DEVICE void cp_async16_zfill(void* dst, const void* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
OPB_DEVICE void ldsm_x4(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
OPB_DEVICE void ldsm_x4_trans(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
OPB_DEVICE void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <int kTp>
struct TemporalSmem {
  __nv_bfloat16 q[kTp][kPitch];
  __nv_bfloat16 k[kTp][kPitch];
  __nv_bfloat16 v[kTp][kPitch];
};

}  // namespace

// kTp = 16 (T <= 16, 4 warps per CTA) or 32 (T <= 32, 2 warps per CTA): 27.6 KB of static shared memory either way
template <int kTp>
__global__ void __launch_bounds__(32 * (64 / kTp))
attention_temporal_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ out, float* __restrict__ ln_stats,
                          int Bv, int T, int N, int H) {
  constexpr int kWarps = 64 / kTp;
  __shared__ __align__(16) TemporalSmem<kTp> smem[kWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long unit = static_cast<long>(blockIdx.x) * kWarps + warp;
  if (unit >= static_cast<long>(Bv) * N * H) return;      // warp-uniform; no CTA-wide barrier follows
  const int h = static_cast<int>(unit % H);
  const long bn = unit / H;
  const int n = static_cast<int>(bn % N);
  const long b = bn / N;
  const int D = H * kHd;
  const long pitch = 3L * D;
  const long M = static_cast<long>(Bv) * T * N;
  const long row0 = b * T * N + n;                         // frame t of this (b, n) is row row0 + t * N
  const __nv_bfloat16* base = qkv + row0 * pitch + h * kHd;
  TemporalSmem<kTp>& s = smem[warp];

  for (int i = lane; i < kTp * 8; i += 32) {
    const int r = i >> 3, c = (i & 7) * 8;
    const bool ok = r < T;
    const __nv_bfloat16* src = base + static_cast<long>(ok ? r : 0) * N * pitch + c;
    cp_async16_zfill(&s.q[r][c], src, ok);
    cp_async16_zfill(&s.k[r][c], src + D, ok);
    cp_async16_zfill(&s.v[r][c], src + 2 * D, ok);
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncwarp();

  const int g = lane >> 2, t4 = lane & 3;
#pragma unroll
  for (int mt = 0; mt < kTp / 16; ++mt) {
    if (mt * 16 >= T) break;
    uint32_t qf[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)
      ldsm_x4(qf[ks], &s.q[mt * 16 + (lane & 7) + ((lane >> 3) & 1) * 8][ks * 16 + (lane >> 4) * 8]);

    float sc[kTp / 8][4];
#pragma unroll
    for (int nt = 0; nt < kTp / 8; ++nt) {
      sc[nt][0] = sc[nt][1] = sc[nt][2] = sc[nt][3] = 0.f;
      uint32_t kf0[4], kf1[4];
      const int r = nt * 8 + (lane & 7), c = (lane >> 3) * 8;
      ldsm_x4(kf0, &s.k[r][c]);
      ldsm_x4(kf1, &s.k[r][c + 32]);
      mma_bf16_16816(sc[nt], qf[0], kf0[0], kf0[1]);
      mma_bf16_16816(sc[nt], qf[1], kf0[2], kf0[3]);
      mma_bf16_16816(sc[nt], qf[2], kf1[0], kf1[1]);
      mma_bf16_16816(sc[nt], qf[3], kf1[2], kf1[3]);
    }

    float mx_lo = -INFINITY, mx_hi = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < kTp / 8; ++nt) {
      const int key = nt * 8 + 2 * t4;
      if (key >= T) { sc[nt][0] = -INFINITY; sc[nt][2] = -INFINITY; }
      if (key + 1 >= T) { sc[nt][1] = -INFINITY; sc[nt][3] = -INFINITY; }
      mx_lo = fmaxf(mx_lo, fmaxf(sc[nt][0], sc[nt][1]));
      mx_hi = fmaxf(mx_hi, fmaxf(sc[nt][2], sc[nt][3]));
    }
    mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 1));
    mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 2));
    mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 1));
    mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 2));   // key 0 is real: both maxima are finite

    float l_lo = 0.f, l_hi = 0.f;
    uint32_t pf[kTp / 8][2];
#pragma unroll
    for (int nt = 0; nt < kTp / 8; ++nt) {
      const float p0 = __expf(sc[nt][0] - mx_lo), p1 = __expf(sc[nt][1] - mx_lo);
      const float p2 = __expf(sc[nt][2] - mx_hi), p3 = __expf(sc[nt][3] - mx_hi);
      l_lo += p0 + p1;
      l_hi += p2 + p3;
      pf[nt][0] = pack_bf16x2(p0, p1);
      pf[nt][1] = pack_bf16x2(p2, p3);
    }

    float o[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
#pragma unroll
    for (int kk = 0; kk < kTp / 16; ++kk) {
      const uint32_t a[4] = {pf[2 * kk][0], pf[2 * kk][1], pf[2 * kk + 1][0], pf[2 * kk + 1][1]};
#pragma unroll
      for (int ndp = 0; ndp < 4; ++ndp) {
        uint32_t vf[4];
        ldsm_x4_trans(vf, &s.v[kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8][ndp * 16 + (lane >> 4) * 8]);
        mma_bf16_16816(o[2 * ndp], a, vf[0], vf[1]);
        mma_bf16_16816(o[2 * ndp + 1], a, vf[2], vf[3]);
      }
    }

    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1);
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
    const float inv_lo = 1.f / l_lo, inv_hi = 1.f / l_hi;
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

    const int t_lo = mt * 16 + g, t_hi = t_lo + 8;
    if (t_lo < T) {
      const long row = row0 + static_cast<long>(t_lo) * N;
      if (t4 == 0) *reinterpret_cast<float2*>(ln_stats + (h * M + row) * 2) = make_float2(s_lo, q_lo);
      __nv_bfloat16* op = out + row * D + h * kHd + 2 * t4;
#pragma unroll
      for (int nd = 0; nd < 8; ++nd)
        *reinterpret_cast<uint32_t*>(op + nd * 8) = pack_bf16x2(o[nd][0] * inv_lo, o[nd][1] * inv_lo);
    }
    if (t_hi < T) {
      const long row = row0 + static_cast<long>(t_hi) * N;
      if (t4 == 0) *reinterpret_cast<float2*>(ln_stats + (h * M + row) * 2) = make_float2(s_hi, q_hi);
      __nv_bfloat16* op = out + row * D + h * kHd + 2 * t4;
#pragma unroll
      for (int nd = 0; nd < 8; ++nd)
        *reinterpret_cast<uint32_t*>(op + nd * 8) = pack_bf16x2(o[nd][2] * inv_hi, o[nd][3] * inv_hi);
    }
  }
}

namespace {

template <int kTp>
int launch_temporal(const void* qkv, void* out, float* ln_stats, int Bv, int T, int N, int H, cudaStream_t stream) {
  constexpr int kWarps = 64 / kTp;
  const long units = static_cast<long>(Bv) * N * H;
  const long grid = (units + kWarps - 1) / kWarps;
  if (grid > 0x7fffffffL) return OPB_ERR_INVALID;
  attention_temporal_kernel<kTp><<<static_cast<unsigned>(grid), 32 * kWarps, 0, stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(qkv), reinterpret_cast<__nv_bfloat16*>(out), ln_stats, Bv, T, N, H);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

}  // namespace

int attention_temporal_fwd(const void* qkv, void* out, float* ln_stats, int Bv, int T, int N, int H, cudaStream_t stream) {
  if (qkv == nullptr || out == nullptr || ln_stats == nullptr) return OPB_ERR_INVALID;
  if (Bv <= 0 || N <= 0 || H <= 0 || T < kTemporalMinT || T > kTemporalMaxT) return OPB_ERR_INVALID;
  if ((reinterpret_cast<uintptr_t>(qkv) & 15) || (reinterpret_cast<uintptr_t>(out) & 15) ||
      (reinterpret_cast<uintptr_t>(ln_stats) & 7))
    return OPB_ERR_INVALID;
  return T <= 16 ? launch_temporal<16>(qkv, out, ln_stats, Bv, T, N, H, stream)
                 : launch_temporal<32>(qkv, out, ln_stats, Bv, T, N, H, stream);
}

// ---------------------------------------------------------------------------------------------------------------------
// Backward.  One warp per (b, n, h), the forward's unit: the warp stages q, k, v and dO of its T rows (zero-filled to kTp),
// recomputes the scores and P with the forward's arithmetic (max, __expf, fp32 row sum; P = p / l, no log-sum-exp is
// saved), then per 16-query m-tile
//   dP = dO V^T,  delta = rowsum(dO o O) (O read from `out`),  dS = P o (dP - delta),  dQ = q_scale * dS K,
// keeping P and dS as bf16 in shared memory, and per 16-key m-tile dV = P^T dO and dK = dS^T Q from their transposes
// (ldmatrix.trans).  All products run on mma.sync.m16n8k16 with fp32 accumulation.  Each warp writes its own rows of its
// head's three column blocks and nothing else: no atomics, so repeated launches are bit-identical.
namespace {

template <int kTp>
struct TemporalBwdSmem {
  __nv_bfloat16 q[kTp][kPitch];
  __nv_bfloat16 k[kTp][kPitch];
  __nv_bfloat16 v[kTp][kPitch];
  __nv_bfloat16 dout[kTp][kPitch];
  __nv_bfloat16 p[kTp][kTp + 8];        // P[query][key]
  __nv_bfloat16 ds[kTp][kTp + 8];       // dS[query][key]
};

// A fragment (rows m0.., k0..) of X^T where X [k][m] is row-major in shared memory
template <int kLd>
OPB_DEVICE void ldsm_a_transposed(uint32_t (&r)[4], const __nv_bfloat16 (*x)[kLd], int m0, int k0, int lane) {
  const int j = lane >> 3;
  ldsm_x4_trans(r, &x[k0 + (j >> 1) * 8 + (lane & 7)][m0 + (j & 1) * 8]);
}

// B fragments of the k16 x n16 block (k0.., n0..) of Y [k][n] row-major in shared memory: {b0, b1} of n-tile n0 and of n0 + 8
OPB_DEVICE void ldsm_b_kn(uint32_t (&r)[4], const __nv_bfloat16 (*y)[kPitch], int k0, int n0, int lane) {
  ldsm_x4_trans(r, &y[k0 + (lane & 7) + ((lane >> 3) & 1) * 8][n0 + (lane >> 4) * 8]);
}

// acc[nt] (16 x 8 tiles over the kTp columns) = A B^T with A the 16 x 64 rows a0.. of `a`, B^T the kTp x 64 rows of `b`
template <int kTp>
OPB_DEVICE void rows_times_rows_t(float (&acc)[kTp / 8][4], const __nv_bfloat16 (*a)[kPitch], const __nv_bfloat16 (*b)[kPitch],
                                  int a0, int lane) {
  uint32_t af[4][4];
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) ldsm_x4(af[ks], &a[a0 + (lane & 7) + ((lane >> 3) & 1) * 8][ks * 16 + (lane >> 4) * 8]);
#pragma unroll
  for (int nt = 0; nt < kTp / 8; ++nt) {
    acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
    uint32_t b0[4], b1[4];
    const int r = nt * 8 + (lane & 7), c = (lane >> 3) * 8;
    ldsm_x4(b0, &b[r][c]);
    ldsm_x4(b1, &b[r][c + 32]);
    mma_bf16_16816(acc[nt], af[0], b0[0], b0[1]);
    mma_bf16_16816(acc[nt], af[1], b0[2], b0[3]);
    mma_bf16_16816(acc[nt], af[2], b1[0], b1[1]);
    mma_bf16_16816(acc[nt], af[3], b1[2], b1[3]);
  }
}

// 16 rows x 64 columns of fp32 accumulators -> bf16 at dst rows r_lo = row0 + t_lo * N and r_hi (rows >= T skipped)
OPB_DEVICE void store_rows(__nv_bfloat16* dst, long pitch, long row0, long N, int t_lo, int T, const float (&acc)[8][4],
                           float scale, int t4) {
  if (t_lo < T) {
    __nv_bfloat16* o = dst + (row0 + static_cast<long>(t_lo) * N) * pitch + 2 * t4;
#pragma unroll
    for (int nd = 0; nd < 8; ++nd) *reinterpret_cast<uint32_t*>(o + nd * 8) = pack_bf16x2(acc[nd][0] * scale, acc[nd][1] * scale);
  }
  if (t_lo + 8 < T) {
    __nv_bfloat16* o = dst + (row0 + static_cast<long>(t_lo + 8) * N) * pitch + 2 * t4;
#pragma unroll
    for (int nd = 0; nd < 8; ++nd) *reinterpret_cast<uint32_t*>(o + nd * 8) = pack_bf16x2(acc[nd][2] * scale, acc[nd][3] * scale);
  }
}

// delta of query row t: sum over the 64 columns of dO o O; each lane of a quad sums 16 columns
OPB_DEVICE float row_delta(const __nv_bfloat16* drow, const __nv_bfloat16* orow, bool valid, int t4) {
  float acc = 0.f;
  if (valid) {
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const uint4 dv = *reinterpret_cast<const uint4*>(drow + t4 * 16 + half * 8);
      const uint4 ov = *reinterpret_cast<const uint4*>(orow + t4 * 16 + half * 8);
      const uint32_t dw[4] = {dv.x, dv.y, dv.z, dv.w}, ow[4] = {ov.x, ov.y, ov.z, ov.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 a = unpack_bf16x2(dw[e]), b = unpack_bf16x2(ow[e]);
        acc = fmaf(a.x, b.x, acc);
        acc = fmaf(a.y, b.y, acc);
      }
    }
  }
  acc += __shfl_xor_sync(0xffffffffu, acc, 1);
  acc += __shfl_xor_sync(0xffffffffu, acc, 2);
  return acc;
}

}  // namespace

// kTp = 16 (T <= 16, 4 warps per CTA, 10.5 KB each: 42 KB) or 32 (T <= 32, 2 warps per CTA, 23 KB each: 46 KB) of
// static shared memory
template <int kTp>
__global__ void __launch_bounds__(32 * (64 / kTp))
attention_temporal_bwd_kernel(const __nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ out,
                              const __nv_bfloat16* __restrict__ d_out, __nv_bfloat16* __restrict__ dqkv, int Bv, int T,
                              int N, int H, float q_scale) {
  constexpr int kWarps = 64 / kTp;
  __shared__ __align__(16) TemporalBwdSmem<kTp> smem[kWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long unit = static_cast<long>(blockIdx.x) * kWarps + warp;
  if (unit >= static_cast<long>(Bv) * N * H) return;      // warp-uniform; no CTA-wide barrier follows
  const int h = static_cast<int>(unit % H);
  const long bn = unit / H;
  const int n = static_cast<int>(bn % N);
  const long b = bn / N;
  const int D = H * kHd;
  const long pitch = 3L * D;
  const long row0 = b * T * N + n;                         // frame t of this (b, n) is row row0 + t * N
  const __nv_bfloat16* base = qkv + row0 * pitch + h * kHd;
  const __nv_bfloat16* dbase = d_out + row0 * D + h * kHd;
  TemporalBwdSmem<kTp>& s = smem[warp];

  for (int i = lane; i < kTp * 8; i += 32) {
    const int r = i >> 3, c = (i & 7) * 8;
    const bool ok = r < T;
    const long rr = static_cast<long>(ok ? r : 0) * N;
    const __nv_bfloat16* src = base + rr * pitch + c;
    cp_async16_zfill(&s.q[r][c], src, ok);
    cp_async16_zfill(&s.k[r][c], src + D, ok);
    cp_async16_zfill(&s.v[r][c], src + 2 * D, ok);
    cp_async16_zfill(&s.dout[r][c], dbase + rr * D + c, ok);
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncwarp();

  const int g = lane >> 2, t4 = lane & 3;
#pragma unroll
  for (int mt = 0; mt < kTp / 16; ++mt) {
    const int t_lo = mt * 16 + g, t_hi = t_lo + 8;
    // P, recomputed exactly as the forward computes it
    float sc[kTp / 8][4];
    rows_times_rows_t<kTp>(sc, s.q, s.k, mt * 16, lane);
    float mx_lo = -INFINITY, mx_hi = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < kTp / 8; ++nt) {
      const int key = nt * 8 + 2 * t4;
      if (key >= T) { sc[nt][0] = -INFINITY; sc[nt][2] = -INFINITY; }
      if (key + 1 >= T) { sc[nt][1] = -INFINITY; sc[nt][3] = -INFINITY; }
      mx_lo = fmaxf(mx_lo, fmaxf(sc[nt][0], sc[nt][1]));
      mx_hi = fmaxf(mx_hi, fmaxf(sc[nt][2], sc[nt][3]));
    }
    mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 1));
    mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 2));
    mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 1));
    mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 2));   // key 0 is real: both maxima are finite
    float l_lo = 0.f, l_hi = 0.f;
#pragma unroll
    for (int nt = 0; nt < kTp / 8; ++nt) {
      sc[nt][0] = __expf(sc[nt][0] - mx_lo); sc[nt][1] = __expf(sc[nt][1] - mx_lo);
      sc[nt][2] = __expf(sc[nt][2] - mx_hi); sc[nt][3] = __expf(sc[nt][3] - mx_hi);
      l_lo += sc[nt][0] + sc[nt][1];
      l_hi += sc[nt][2] + sc[nt][3];
    }
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1);
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
    // query rows >= T (zero q) are given P = 0, so that they add nothing to dV and dK
    const float inv_lo = t_lo < T ? 1.f / l_lo : 0.f, inv_hi = t_hi < T ? 1.f / l_hi : 0.f;

    float dp[kTp / 8][4];
    rows_times_rows_t<kTp>(dp, s.dout, s.v, mt * 16, lane);
    const __nv_bfloat16* orow = out + h * kHd;
    const float dl_lo = row_delta(&s.dout[t_lo][0], orow + (row0 + static_cast<long>(t_lo < T ? t_lo : 0) * N) * D,
                                  t_lo < T, t4);
    const float dl_hi = row_delta(&s.dout[t_hi][0], orow + (row0 + static_cast<long>(t_hi < T ? t_hi : 0) * N) * D,
                                  t_hi < T, t4);

    uint32_t dsf[kTp / 8][2];
#pragma unroll
    for (int nt = 0; nt < kTp / 8; ++nt) {
      const float p0 = sc[nt][0] * inv_lo, p1 = sc[nt][1] * inv_lo, p2 = sc[nt][2] * inv_hi, p3 = sc[nt][3] * inv_hi;
      const int c = nt * 8 + 2 * t4;
      *reinterpret_cast<uint32_t*>(&s.p[t_lo][c]) = pack_bf16x2(p0, p1);
      *reinterpret_cast<uint32_t*>(&s.p[t_hi][c]) = pack_bf16x2(p2, p3);
      dsf[nt][0] = pack_bf16x2(p0 * (dp[nt][0] - dl_lo), p1 * (dp[nt][1] - dl_lo));
      dsf[nt][1] = pack_bf16x2(p2 * (dp[nt][2] - dl_hi), p3 * (dp[nt][3] - dl_hi));
      *reinterpret_cast<uint32_t*>(&s.ds[t_lo][c]) = dsf[nt][0];
      *reinterpret_cast<uint32_t*>(&s.ds[t_hi][c]) = dsf[nt][1];
    }

    // dQ = q_scale * dS K over the kTp keys
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f; }
#pragma unroll
    for (int kk = 0; kk < kTp / 16; ++kk) {
      const uint32_t a[4] = {dsf[2 * kk][0], dsf[2 * kk][1], dsf[2 * kk + 1][0], dsf[2 * kk + 1][1]};
#pragma unroll
      for (int ndp = 0; ndp < 4; ++ndp) {
        uint32_t kf[4];
        ldsm_b_kn(kf, s.k, kk * 16, ndp * 16, lane);
        mma_bf16_16816(acc[2 * ndp], a, kf[0], kf[1]);
        mma_bf16_16816(acc[2 * ndp + 1], a, kf[2], kf[3]);
      }
    }
    store_rows(dqkv + h * kHd, pitch, row0, N, t_lo, T, acc, q_scale, t4);
  }
  __syncwarp();

  // dV = P^T dO and dK = dS^T Q, 16 keys at a time, contracting over the kTp queries
#pragma unroll
  for (int kt = 0; kt < kTp / 16; ++kt) {
    float dv[8][4], dk[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f;
      dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = 0.f;
    }
#pragma unroll
    for (int kq = 0; kq < kTp / 16; ++kq) {
      uint32_t pa[4], da[4];
      ldsm_a_transposed<kTp + 8>(pa, s.p, kt * 16, kq * 16, lane);
      ldsm_a_transposed<kTp + 8>(da, s.ds, kt * 16, kq * 16, lane);
#pragma unroll
      for (int ndp = 0; ndp < 4; ++ndp) {
        uint32_t of[4], qf[4];
        ldsm_b_kn(of, s.dout, kq * 16, ndp * 16, lane);
        ldsm_b_kn(qf, s.q, kq * 16, ndp * 16, lane);
        mma_bf16_16816(dv[2 * ndp], pa, of[0], of[1]);
        mma_bf16_16816(dv[2 * ndp + 1], pa, of[2], of[3]);
        mma_bf16_16816(dk[2 * ndp], da, qf[0], qf[1]);
        mma_bf16_16816(dk[2 * ndp + 1], da, qf[2], qf[3]);
      }
    }
    store_rows(dqkv + D + h * kHd, pitch, row0, N, kt * 16 + g, T, dk, 1.f, t4);
    store_rows(dqkv + 2 * D + h * kHd, pitch, row0, N, kt * 16 + g, T, dv, 1.f, t4);
  }
}

namespace {

template <int kTp>
int launch_temporal_bwd(const void* qkv, const void* out, const void* d_out, void* dqkv, int Bv, int T, int N, int H,
                        float q_scale, cudaStream_t stream) {
  constexpr int kWarps = 64 / kTp;
  const long units = static_cast<long>(Bv) * N * H;
  const long grid = (units + kWarps - 1) / kWarps;
  if (grid > 0x7fffffffL) return OPB_ERR_INVALID;
  attention_temporal_bwd_kernel<kTp><<<static_cast<unsigned>(grid), 32 * kWarps, 0, stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(qkv), reinterpret_cast<const __nv_bfloat16*>(out),
      reinterpret_cast<const __nv_bfloat16*>(d_out), reinterpret_cast<__nv_bfloat16*>(dqkv), Bv, T, N, H, q_scale);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

}  // namespace

int attention_temporal_bwd(const void* qkv, const void* out, const void* d_out, void* dqkv, int Bv, int T, int N, int H,
                           float q_scale, cudaStream_t stream) {
  if (qkv == nullptr || out == nullptr || d_out == nullptr || dqkv == nullptr) return OPB_ERR_INVALID;
  if (Bv <= 0 || N <= 0 || H <= 0 || T < kTemporalMinT || T > kTemporalMaxT) return OPB_ERR_INVALID;
  if ((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(d_out) |
       reinterpret_cast<uintptr_t>(dqkv)) & 15)
    return OPB_ERR_INVALID;
  return T <= 16 ? launch_temporal_bwd<16>(qkv, out, d_out, dqkv, Bv, T, N, H, q_scale, stream)
                 : launch_temporal_bwd<32>(qkv, out, d_out, dqkv, Bv, T, N, H, q_scale, stream);
}

}  // namespace opb
