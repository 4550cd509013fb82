// Decomposed relative-position terms of the detection backbone's attention (detectron2 add_decomposed_rel_pos, called at
// one_peace_vision/det/models/onepeace.py:206-207):
//     rel_h[b][h][i][ky] = q_i . rel_pos_h[pos_y[i] - ky + kh - 1],   rel_w[b][h][i][kx] = q_i . rel_pos_w[pos_x[i] - kx + kw - 1]
// with q_i the UNSCALED q row of head h: q_unscale * (the bf16 q columns of the QKV GEMM output, which carry head_dim^-0.5).
//
// For every row the kh terms read a contiguous window of kh consecutive table rows, so the kernel computes the full
// product P[i][r] = q_i . table[r] for all 2k - 1 table rows (fp32 FMAs, c = 0..63 in order) and scatters each P[i][r]
// to ky = pos[i] + k - 1 - r when that lies in [0, k).  One CTA = (128 rows, (b, h), table): the q tile and the table
// are staged transposed in shared memory; a thread owns 8 rows x 2 table rows of each 32-row table chunk.  A position
// outside [0, k) writes NaN into that row's terms instead of reading out of bounds.
#include "common.cuh"
#include "ops.h"

namespace opb {

namespace {
constexpr int kRows = 128;          // sequence rows per CTA
constexpr int kQPitch = kRows + 4;  // Qt[c][row]
constexpr int kChunk = 32;          // table rows per pass (16 threads x 2)
}

__global__ void __launch_bounds__(256)
relpos_decomp_proj_kernel(const __nv_bfloat16* __restrict__ qkv, const float* __restrict__ rel_pos_h,
                          const float* __restrict__ rel_pos_w, const int* __restrict__ pos_y,
                          const int* __restrict__ pos_x, float q_unscale, float* __restrict__ rel_h,
                          float* __restrict__ rel_w, int B, int S, int H, int kh, int kw) {
  extern __shared__ __align__(16) float proj_smem[];
  const bool is_w = blockIdx.z == 1;
  const float* __restrict__ table = is_w ? rel_pos_w : rel_pos_h;
  const int* __restrict__ pos = is_w ? pos_x : pos_y;
  float* __restrict__ dst = is_w ? rel_w : rel_h;
  const int k = is_w ? kw : kh;
  const int nr = 2 * k - 1;
  const int nr_pad = (nr + kChunk - 1) / kChunk * kChunk;
  float* Qt = proj_smem;                 // [64][kQPitch]
  float* Tt = proj_smem + 64 * kQPitch;  // [64][nr_pad]
  const int bh = blockIdx.y, b = bh / H, h = bh % H;
  const int i0 = blockIdx.x * kRows;
  const int tid = threadIdx.x;
  const long ld = 3L * H * 64;

  for (int e = tid; e < kRows * 8; e += 256) {       // 8 bf16 of one q row per step
    const int r = e >> 3, c = (e & 7) * 8;
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (i0 + r < S) {
      const uint4 u = *reinterpret_cast<const uint4*>(qkv + (static_cast<long>(b) * S + i0 + r) * ld + h * 64 + c);
      const __nv_bfloat16* x = reinterpret_cast<const __nv_bfloat16*>(&u);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = __bfloat162float(x[j]) * q_unscale;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) Qt[(c + j) * kQPitch + r] = v[j];
  }
  for (int e = tid; e < nr_pad * 64; e += 256) {
    const int r = e >> 6, c = e & 63;
    Tt[c * nr_pad + r] = r < nr ? table[r * 64 + c] : 0.f;
  }
  __syncthreads();

  const int cg = tid & 15, rg = tid >> 4;           // table rows c0 + 2 cg + {0, 1}; sequence rows 8 rg + {0..7}
  int p[8];
#pragma unroll
  for (int a = 0; a < 8; ++a) {
    const int i = i0 + rg * 8 + a;
    p[a] = i < S ? pos[i] : 0;
  }
  for (int c0 = 0; c0 < nr; c0 += kChunk) {
    float acc[8][2];
#pragma unroll
    for (int a = 0; a < 8; ++a) acc[a][0] = acc[a][1] = 0.f;
#pragma unroll 8
    for (int c = 0; c < 64; ++c) {
      const float4 qa = *reinterpret_cast<const float4*>(&Qt[c * kQPitch + rg * 8]);
      const float4 qb = *reinterpret_cast<const float4*>(&Qt[c * kQPitch + rg * 8 + 4]);
      const float2 tb = *reinterpret_cast<const float2*>(&Tt[c * nr_pad + c0 + 2 * cg]);
      const float q[8] = {qa.x, qa.y, qa.z, qa.w, qb.x, qb.y, qb.z, qb.w};
#pragma unroll
      for (int a = 0; a < 8; ++a) {
        acc[a][0] = fmaf(q[a], tb.x, acc[a][0]);
        acc[a][1] = fmaf(q[a], tb.y, acc[a][1]);
      }
    }
#pragma unroll
    for (int a = 0; a < 8; ++a) {
      const int i = i0 + rg * 8 + a;
      if (i >= S) continue;
      float* row = dst + (static_cast<long>(bh) * S + i) * k;
      const bool ok = static_cast<unsigned>(p[a]) < static_cast<unsigned>(k);
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int r = c0 + 2 * cg + j;
        if (!ok) {
          if (r < k) row[r] = NAN;
        } else {
          const int ky = p[a] + k - 1 - r;
          if (r < nr && ky >= 0 && ky < k) row[ky] = acc[a][j];
        }
      }
    }
  }
}

int relpos_decomp_proj(const void* qkv, const float* rel_pos_h, const float* rel_pos_w, const int* pos_y, const int* pos_x,
                       float q_unscale, float* rel_h, float* rel_w, int B, int S, int H, int kh, int kw, cudaStream_t stream) {
  if (B <= 0 || S <= 0 || H <= 0 || kh <= 0 || kw <= 0 || kh > kDecompMaxK || kw > kDecompMaxK) return OPB_ERR_INVALID;
  if (static_cast<long>(kh) * kw != S || static_cast<long>(B) * H > 65535) return OPB_ERR_INVALID;
  if (!(q_unscale == q_unscale) || q_unscale == INFINITY || q_unscale == -INFINITY) return OPB_ERR_INVALID;
  const int nr_pad = (2 * (kh > kw ? kh : kw) - 1 + kChunk - 1) / kChunk * kChunk;
  const size_t smem = sizeof(float) * 64 * (kQPitch + nr_pad);
  static size_t smem_set = 0;
  if (smem > smem_set) {
    if (cudaFuncSetAttribute(relpos_decomp_proj_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             static_cast<int>(smem)) != cudaSuccess)
      return OPB_ERR_CUDA;
    smem_set = smem;
  }
  const dim3 grid((S + kRows - 1) / kRows, B * H, 2);
  relpos_decomp_proj_kernel<<<grid, 256, smem, stream>>>(reinterpret_cast<const __nv_bfloat16*>(qkv), rel_pos_h, rel_pos_w,
                                                         pos_y, pos_x, q_unscale, rel_h, rel_w, B, S, H, kh, kw);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

}  // namespace opb
