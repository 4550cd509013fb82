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

}  // namespace opb
