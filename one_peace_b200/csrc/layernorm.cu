// Row LayerNorm kernels (eps inside the sqrt, biased variance — torch.nn.LayerNorm semantics, which is
// what one_peace/models/components.py:23-26 builds).  HBM-bound: one pass, the row lives in registers,
// two-step mean / centred variance in fp32, 16-byte vector loads/stores, one warp per row.
//
//   in : fp32 (residual stream) or bf16 (GEMM / attention outputs), row pitch ld_in
//   out: bf16 (feeds the next wgmma GEMM as its K-major A operand) or fp32
//   optional affine (gamma/beta may be null: the audio conv-pos LN is non-affine, audio.py:71),
//   optional exact-erf GELU after the norm (hMLP stem and wav2vec-style conv blocks: LN -> GELU),
//   optional 2x2 pixel-merge scatter of the output row, which lays the result out as the A operand
//   of the next stride-2 patch conv (image.py:66-75) so that conv is a plain GEMM.
#include "common.cuh"
#include "ops.h"

namespace opb {

struct LnArgs {
  const void* in;
  void* out;
  const float* gamma;
  const float* beta;
  long ld_in;       // elements
  long ld_out;      // elements
  int rows;
  int dim;
  float eps;
  int gelu;
  // pixel-merge scatter (0 = off): input rows are (b, y, x) over a grid_w x grid_w map
  int merge_grid_w;
  // sequence remap (0 = off): input row = b * row_period + t; rows with t >= row_valid are skipped;
  // output row = b * out_period + t + out_row_shift   (halo / CLS offsets of the audio adapter buffers)
  int row_period, row_valid, out_period, out_row_shift;
  // channel-group padding (0 = off): output column = (c / group_in) * group_out + c % group_in
  int group_in, group_out;
  int accumulate;   // fp32 output only: out += y
  // statistics-only mode: write the UN-normalised row (cast to TOut) plus mean / rstd, for the fused-LN GEMMs
  int raw;
  float* mu_out;
  float* rstd_out;
};

template <typename T>
OPB_DEVICE void load8(const T* p, float (&v)[8]);
template <>
OPB_DEVICE void load8<float>(const float* p, float (&v)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p);
  const float4 b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
template <>
OPB_DEVICE void load8<__nv_bfloat16>(const __nv_bfloat16* p, float (&v)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  float2 f;
  f = unpack_bf16x2(u.x); v[0] = f.x; v[1] = f.y;
  f = unpack_bf16x2(u.y); v[2] = f.x; v[3] = f.y;
  f = unpack_bf16x2(u.z); v[4] = f.x; v[5] = f.y;
  f = unpack_bf16x2(u.w); v[6] = f.x; v[7] = f.y;
}
template <typename T>
OPB_DEVICE void store8(T* p, const float (&v)[8]);
template <>
OPB_DEVICE void store8<float>(float* p, const float (&v)[8]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
}
template <>
OPB_DEVICE void store8<__nv_bfloat16>(__nv_bfloat16* p, const float (&v)[8]) {
  uint4 u;
  u.x = pack_bf16x2(v[0], v[1]);
  u.y = pack_bf16x2(v[2], v[3]);
  u.z = pack_bf16x2(v[4], v[5]);
  u.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(p) = u;
}

// One WARP per row: the whole row is fetched with all of the lane's 16-byte loads in flight at once (VPL vectors
// of 8 elements per lane), reduced with shuffles only (no shared memory, no block barriers), normalised from
// registers and written once.  4 rows per 128-thread CTA.  (The first version used one CTA per row with a single
// outstanding load per thread and reached only ~3.5 TB/s; a row of 1536 fp32 is 6 KB, so ~50 KB must be in flight
// per SM to cover HBM latency.)
template <typename TIn, typename TOut, int VPL>
__global__ void __launch_bounds__(128) layernorm_kernel(const LnArgs a) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (row >= a.rows) return;
  if (a.row_period > 0 && (row % a.row_period) >= a.row_valid) return;   // warp-uniform
  const TIn* in = reinterpret_cast<const TIn*>(a.in) + static_cast<long>(row) * a.ld_in;
  const int nvec = a.dim >> 3;

  // raw loads first (kept packed), then convert
  constexpr bool kInF32 = sizeof(TIn) == 4;
  uint4 raw[VPL * (kInF32 ? 2 : 1)];
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int v = i * 32 + lane;
    if (v < nvec) {
      if constexpr (kInF32) {
        raw[2 * i] = *reinterpret_cast<const uint4*>(in + v * 8);
        raw[2 * i + 1] = *reinterpret_cast<const uint4*>(in + v * 8 + 4);
      } else {
        raw[i] = *reinterpret_cast<const uint4*>(in + v * 8);
      }
    }
  }
  auto unpack = [&](int i, float (&x)[8]) {
    if constexpr (kInF32) {
      x[0] = __uint_as_float(raw[2 * i].x); x[1] = __uint_as_float(raw[2 * i].y);
      x[2] = __uint_as_float(raw[2 * i].z); x[3] = __uint_as_float(raw[2 * i].w);
      x[4] = __uint_as_float(raw[2 * i + 1].x); x[5] = __uint_as_float(raw[2 * i + 1].y);
      x[6] = __uint_as_float(raw[2 * i + 1].z); x[7] = __uint_as_float(raw[2 * i + 1].w);
    } else {
      float2 f;
      f = unpack_bf16x2(raw[i].x); x[0] = f.x; x[1] = f.y;
      f = unpack_bf16x2(raw[i].y); x[2] = f.x; x[3] = f.y;
      f = unpack_bf16x2(raw[i].z); x[4] = f.x; x[5] = f.y;
      f = unpack_bf16x2(raw[i].w); x[6] = f.x; x[7] = f.y;
    }
  };
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    if (i * 32 + lane < nvec) {
      float x[8];
      unpack(i, x);
#pragma unroll
      for (int e = 0; e < 8; ++e) sum += x[e];
    }
  }
  const float mean = warp_sum(sum) / a.dim;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    if (i * 32 + lane < nvec) {
      float x[8];
      unpack(i, x);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float d = x[e] - mean;
        sq += d * d;
      }
    }
  }
  const float var = warp_sum(sq) / a.dim;
  const float rstd = rsqrtf(var + a.eps);

  if (a.raw) {
    if (lane == 0) { a.mu_out[row] = mean; a.rstd_out[row] = rstd; }
    TOut* o = reinterpret_cast<TOut*>(a.out) + static_cast<long>(row) * a.ld_out;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int c = (i * 32 + lane) * 8;
      if (c < a.dim) {
        float y[8];
        unpack(i, y);
        store8<TOut>(o + c, y);
      }
    }
    return;
  }
  long orow = row;
  long ocol0 = 0;
  if (a.merge_grid_w > 0) {
    const int w = a.merge_grid_w;
    const int xx = row % w;
    const int yy = (row / w) % w;
    const int bb = row / (w * w);
    orow = (static_cast<long>(bb) * (w / 2) + yy / 2) * (w / 2) + xx / 2;
    ocol0 = static_cast<long>((yy & 1) * 2 + (xx & 1)) * a.dim;
  }
  if (a.row_period > 0) orow = static_cast<long>(row / a.row_period) * a.out_period + (row % a.row_period) + a.out_row_shift;
  TOut* out = reinterpret_cast<TOut*>(a.out) + orow * a.ld_out + ocol0;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int c = (i * 32 + lane) * 8;
    if (c < a.dim) {
      float y[8];
      unpack(i, y);
#pragma unroll
      for (int e = 0; e < 8; ++e) y[e] = (y[e] - mean) * rstd;
      if (a.gamma != nullptr) {
        float gm[8], bt[8];
        load8<float>(a.gamma + c, gm);
        load8<float>(a.beta + c, bt);
#pragma unroll
        for (int e = 0; e < 8; ++e) y[e] = y[e] * gm[e] + bt[e];
      }
      if (a.gelu) {
#pragma unroll
        for (int e = 0; e < 8; ++e) y[e] = gelu_erf(y[e]);
      }
      const int oc = a.group_in > 0 ? (c / a.group_in) * a.group_out + (c % a.group_in) : c;
      if constexpr (sizeof(TOut) == 4) {
        if (a.accumulate) {
          float prev[8];
          load8<float>(reinterpret_cast<const float*>(out) + oc, prev);
#pragma unroll
          for (int e = 0; e < 8; ++e) y[e] += prev[e];
        }
      }
      store8<TOut>(out + oc, y);
    }
  }
}

template <typename TIn, typename TOut>
static int launch_ln(const LnArgs& a, cudaStream_t stream) {
  const int need = (a.dim / 8 + 31) / 32;      // vectors per lane
  const unsigned grid = (a.rows + 3) / 4;
#define OPB_LN(V) layernorm_kernel<TIn, TOut, V><<<grid, 128, 0, stream>>>(a)
  if (need <= 1) OPB_LN(1);
  else if (need <= 2) OPB_LN(2);
  else if (need <= 4) OPB_LN(4);
  else if (need <= 6) OPB_LN(6);
  else if (need <= 8) OPB_LN(8);
  else if (need <= 12) OPB_LN(12);             // fp32 rows up to 3072: the classifier of a head_scale_ratio 2 head at d 1536
  else if (sizeof(TIn) == 2 && need <= 24) OPB_LN(24);
  else return OPB_ERR_UNSUPPORTED;            // rows wider than 6144 (bf16) / 3072 (fp32) are not on this path
#undef OPB_LN
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

// Reduces the per-(part, row) partial (sum, sum of squares) written by the producing GEMM / attention epilogues to
// the row mean and 1/sqrt(var + eps) the consuming GEMM epilogue applies (fused LayerNorm, see gemm.h).  Parts are
// summed in index order (deterministic).  var = E[x^2] - mean^2 in fp32, clamped at 0.
__global__ void ln_stats_finalize_kernel(const float* __restrict__ partial, int parts, int rows, int dim, float eps,
                                         float* __restrict__ mu, float* __restrict__ rstd) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  float s = 0.f, q = 0.f;
  for (int p = 0; p < parts; ++p) {
    const float2 v = *reinterpret_cast<const float2*>(partial + (static_cast<long>(p) * rows + r) * 2);
    s += v.x;
    q += v.y;
  }
  const float mean = s / dim;
  const float var = fmaxf(q / dim - mean * mean, 0.f);
  mu[r] = mean;
  rstd[r] = rsqrtf(var + eps);
}

int ln_stats_finalize(const float* partial, int parts, int rows, int dim, float eps, float* mu, float* rstd,
                      cudaStream_t stream) {
  if (parts <= 0 || rows <= 0 || dim <= 0) return OPB_ERR_INVALID;
  ln_stats_finalize_kernel<<<(rows + 255) / 256, 256, 0, stream>>>(partial, parts, rows, dim, eps, mu, rstd);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

// in_dtype / out_dtype: 0 = fp32, 1 = bf16
int layernorm(const void* in, int in_dtype, long ld_in, void* out, int out_dtype, long ld_out, const float* gamma,
              const float* beta, int rows, int dim, float eps, int gelu, int merge_grid_w, const LnRemap& rm,
              cudaStream_t stream) {
  if (rows <= 0 || dim <= 0 || dim % 8 != 0 || ld_in % 8 != 0 || ld_out % 8 != 0) return OPB_ERR_INVALID;
  if ((gamma == nullptr) != (beta == nullptr)) return OPB_ERR_INVALID;
  if (merge_grid_w < 0 || (merge_grid_w & 1)) return OPB_ERR_INVALID;
  if (rm.group_in > 0 && (rm.group_in % 8 != 0 || rm.group_out % 8 != 0 || rm.group_out < rm.group_in)) return OPB_ERR_INVALID;
  if (rm.accumulate && out_dtype != 0) return OPB_ERR_INVALID;
  if (rm.row_period > 0 && merge_grid_w > 0) return OPB_ERR_INVALID;
  LnArgs a{in, out, gamma, beta, ld_in, ld_out, rows, dim, eps, gelu, merge_grid_w, rm.row_period, rm.row_valid,
           rm.out_period, rm.out_row_shift, rm.group_in, rm.group_out, rm.accumulate, rm.raw, rm.mu_out, rm.rstd_out};
  if (rm.raw && (rm.mu_out == nullptr || rm.rstd_out == nullptr)) return OPB_ERR_INVALID;
  if (in_dtype == 0 && out_dtype == 1) return launch_ln<float, __nv_bfloat16>(a, stream);
  if (in_dtype == 1 && out_dtype == 1) return launch_ln<__nv_bfloat16, __nv_bfloat16>(a, stream);
  if (in_dtype == 0 && out_dtype == 0) return launch_ln<float, float>(a, stream);
  if (in_dtype == 1 && out_dtype == 0) return launch_ln<__nv_bfloat16, float>(a, stream);
  return OPB_ERR_INVALID;
}

}  // namespace opb
