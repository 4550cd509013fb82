// Pooled classification head of OnePeaceViT (one_peace_vision/classification/models_vit.py:431-434, global_pool=True):
//     m    = x[:, 1:, :].mean(dim=1)                 mean over the S - 1 patch rows; the CLS row is excluded
//     y    = fc_norm(m)                              LayerNorm over d with the module's eps, affine
// and its adjoint, which broadcasts d m / (S - 1) into every patch row of dx and writes exact zeros into the CLS row.
//
// The forward reads B * S * d fp32 values (400 MB at B = 64, S = 1025, d = 1536) and is HBM-bound.  It runs as
//   token_mean_partial_kernel : grid (column slice, row split, sample); each CTA sums its rows of a 256-column slice with
//                               four row lanes of 16-byte loads, merges the lanes in lane order and stores one partial row;
//   token_mean_ln_kernel      : one CTA per sample sums the partial rows in split order, divides by S - 1 and applies the
//                               LayerNorm (two-pass variance, fixed-order CTA sums).
// The backward runs as
//   token_mean_ln_bwd_kernel  : CTAs [0, B) form one sample's LayerNorm adjoint scaled by 1 / (S - 1); CTAs [B, B + d/256)
//                               sum dgamma / dbeta over the samples in sample order;
//   token_broadcast_kernel    : grid (column slice, row split, sample); every row of dx is written exactly once.
// No atomics anywhere: every sum runs in an order fixed by the shape, so repeated launches are bit-identical.
#include "common.cuh"
#include "ops.h"

namespace opb {

namespace {

constexpr int kVec = 64;                       // float4 columns per CTA slice (256 columns)
constexpr int kLanes = 4;                      // row lanes per CTA
constexpr int kThreads = kVec * kLanes;        // 256
constexpr int kMinRowsPerSplit = 16;           // four rows per lane at least
constexpr int kTargetCtas = 2048;              // ~2 waves of 8 resident 256-thread CTAs on each of 132 SMs
constexpr int kLnThreads = 256;

int col_slices(int d) { return (d / 4 + kVec - 1) / kVec; }

// row splits of the S - 1 patch rows; a function of the shape only, so the summation order is too
int row_splits(int B, int S, int d) {
  const int rows = S - 1;
  const int want = (kTargetCtas + B * col_slices(d) - 1) / (B * col_slices(d));
  const int cap = (rows + kMinRowsPerSplit - 1) / kMinRowsPerSplit;
  return want < 1 ? 1 : (want > cap ? cap : want);
}

OPB_DEVICE float4 add4(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }

// fixed-order sum over a 256-thread CTA (butterfly within each warp, then the warp totals in warp order)
OPB_DEVICE float cta_sum(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int w = 0; w < kLnThreads / 32; ++w) s += red[w];
  return s;
}

__global__ void __launch_bounds__(kThreads)
token_mean_partial_kernel(const float* __restrict__ x, long ld, int S, int d, int rows_per_split, float* __restrict__ partial) {
  __shared__ float4 red[kLanes][kVec];
  const int b = blockIdx.z, split = blockIdx.y;
  const int v = threadIdx.x % kVec, lane = threadIdx.x / kVec;
  const int c = (blockIdx.x * kVec + v) * 4;
  const int r0 = 1 + split * rows_per_split;
  const int r1 = min(S, r0 + rows_per_split);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c < d) {
    const float* base = x + static_cast<long>(b) * S * ld + c;
    int r = r0 + lane;
    // four independent 16-byte loads in flight per thread; added in row order, as the one-row tail is
    for (; r + 3 * kLanes < r1; r += 4 * kLanes) {
      const float4 a0 = __ldcs(reinterpret_cast<const float4*>(base + static_cast<long>(r) * ld));
      const float4 a1 = __ldcs(reinterpret_cast<const float4*>(base + static_cast<long>(r + kLanes) * ld));
      const float4 a2 = __ldcs(reinterpret_cast<const float4*>(base + static_cast<long>(r + 2 * kLanes) * ld));
      const float4 a3 = __ldcs(reinterpret_cast<const float4*>(base + static_cast<long>(r + 3 * kLanes) * ld));
      acc = add4(add4(add4(add4(acc, a0), a1), a2), a3);
    }
    for (; r < r1; r += kLanes) acc = add4(acc, __ldcs(reinterpret_cast<const float4*>(base + static_cast<long>(r) * ld)));
  }
  red[lane][v] = acc;
  __syncthreads();
  if (lane == 0 && c < d) {
    float4 s = red[0][v];
#pragma unroll
    for (int l = 1; l < kLanes; ++l) s = add4(s, red[l][v]);
    *reinterpret_cast<float4*>(partial + (static_cast<long>(split) * gridDim.z + b) * d + c) = s;
  }
}

__global__ void __launch_bounds__(kLnThreads)
token_mean_ln_kernel(const float* __restrict__ partial, int nsplit, int B, int S, int d, const float* __restrict__ gamma,
                     const float* __restrict__ beta, float eps, float* __restrict__ m, __nv_bfloat16* __restrict__ y,
                     float* __restrict__ mean, float* __restrict__ rstd) {
  __shared__ float red[kLnThreads / 32];
  const int b = blockIdx.x;
  const float n = static_cast<float>(S - 1);
  float* mb = m + static_cast<long>(b) * d;
  float s1 = 0.f;
  for (int c = threadIdx.x; c < d; c += kLnThreads) {
    float s = 0.f;
    for (int j = 0; j < nsplit; ++j) s += partial[(static_cast<long>(j) * B + b) * d + c];
    const float mv = __fdiv_rn(s, n);
    mb[c] = mv;
    s1 += mv;
  }
  const float mu = cta_sum(s1, red) / static_cast<float>(d);
  float s2 = 0.f;
  for (int c = threadIdx.x; c < d; c += kLnThreads) {
    const float t = mb[c] - mu;
    s2 += t * t;
  }
  const float rs = rsqrtf(cta_sum(s2, red) / static_cast<float>(d) + eps);
  for (int c = threadIdx.x; c < d; c += kLnThreads)
    y[static_cast<long>(b) * d + c] = __float2bfloat16_rn((mb[c] - mu) * rs * gamma[c] + beta[c]);
  if (threadIdx.x == 0) {
    mean[b] = mu;
    rstd[b] = rs;
  }
}

__global__ void __launch_bounds__(kLnThreads)
token_mean_ln_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ m, const float* __restrict__ mean,
                         const float* __restrict__ rstd, const float* __restrict__ gamma, int B, int S, int d,
                         float* __restrict__ dgamma, float* __restrict__ dbeta, float* __restrict__ g) {
  __shared__ float red[kLnThreads / 32];
  if (blockIdx.x >= B) {                              // dgamma / dbeta of one column per thread, samples in order
    const int c = (blockIdx.x - B) * kLnThreads + threadIdx.x;
    if (c >= d) return;
    float sg = 0.f, sb = 0.f;
    for (int b = 0; b < B; ++b) {
      const long o = static_cast<long>(b) * d + c;
      sg += dy[o] * ((m[o] - mean[b]) * rstd[b]);
      sb += dy[o];
    }
    dgamma[c] = sg;
    dbeta[c] = sb;
    return;
  }
  const int b = blockIdx.x;
  const float mu = mean[b], rs = rstd[b];
  const float* mb = m + static_cast<long>(b) * d;
  const float* db = dy + static_cast<long>(b) * d;
  float a1 = 0.f, a2 = 0.f;
  for (int c = threadIdx.x; c < d; c += kLnThreads) {
    const float gx = db[c] * gamma[c];
    a1 += gx;
    a2 += gx * ((mb[c] - mu) * rs);
  }
  const float inv_d = 1.f / static_cast<float>(d);
  const float mean_g = cta_sum(a1, red) * inv_d;
  const float mean_gx = cta_sum(a2, red) * inv_d;
  const float n = static_cast<float>(S - 1);
  for (int c = threadIdx.x; c < d; c += kLnThreads) {
    const float xh = (mb[c] - mu) * rs;
    const float dm = rs * (db[c] * gamma[c] - mean_g - xh * mean_gx);
    g[static_cast<long>(b) * d + c] = __fdiv_rn(dm, n);
  }
}

__global__ void __launch_bounds__(kThreads)
token_broadcast_kernel(const float* __restrict__ g, int S, int d, int rows_per_split, float* __restrict__ dx, long ld) {
  const int b = blockIdx.z, split = blockIdx.y;
  const int v = threadIdx.x % kVec, lane = threadIdx.x / kVec;
  const int c = (blockIdx.x * kVec + v) * 4;
  if (c >= d) return;
  const float4 val = *reinterpret_cast<const float4*>(g + static_cast<long>(b) * d + c);
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  float* base = dx + static_cast<long>(b) * S * ld + c;
  const int r1 = min(S, (split + 1) * rows_per_split);
  for (int r = split * rows_per_split + lane; r < r1; r += kLanes)
    __stcs(reinterpret_cast<float4*>(base + static_cast<long>(r) * ld), r == 0 ? zero : val);
}

bool shape_ok(int B, int S, int d) { return B >= 1 && B <= 65535 && S >= 2 && d >= 4 && d % 4 == 0; }
bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace

long token_mean_ln_ws_floats(int B, int S, int d) {
  if (!shape_ok(B, S, d)) return -1;
  return static_cast<long>(row_splits(B, S, d)) * B * d;
}

int token_mean_ln_fwd(const float* x, long ld, int B, int S, int d, const float* gamma, const float* beta, float eps, float* ws,
                      long ws_floats, float* m, void* y, float* mean, float* rstd, cudaStream_t stream) {
  if (!shape_ok(B, S, d) || ld < d || ld % 4 != 0 || !aligned16(x) || !aligned16(ws) || !(eps >= 0.f)) return OPB_ERR_INVALID;
  const int nsplit = row_splits(B, S, d);
  if (ws_floats < static_cast<long>(nsplit) * B * d) return OPB_ERR_INVALID;
  const int rows_per_split = (S - 1 + nsplit - 1) / nsplit;
  token_mean_partial_kernel<<<dim3(col_slices(d), nsplit, B), kThreads, 0, stream>>>(x, ld, S, d, rows_per_split, ws);
  token_mean_ln_kernel<<<B, kLnThreads, 0, stream>>>(ws, nsplit, B, S, d, gamma, beta, eps, m,
                                                     static_cast<__nv_bfloat16*>(y), mean, rstd);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

int token_mean_ln_bwd(const float* dy, const float* m, const float* mean, const float* rstd, const float* gamma, int B, int S,
                      int d, float* dgamma, float* dbeta, float* ws, float* dx, long ld_dx, cudaStream_t stream) {
  if (!shape_ok(B, S, d) || ld_dx < d || ld_dx % 4 != 0 || !aligned16(dx) || !aligned16(ws)) return OPB_ERR_INVALID;
  // the broadcast covers all S rows (the CLS row gets the zeros), split like the forward's patch rows
  const int nsplit = row_splits(B, S + 1, d);
  const int rows_per_split = (S + nsplit - 1) / nsplit;
  token_mean_ln_bwd_kernel<<<B + (d + kLnThreads - 1) / kLnThreads, kLnThreads, 0, stream>>>(dy, m, mean, rstd, gamma, B, S, d,
                                                                                            dgamma, dbeta, ws);
  token_broadcast_kernel<<<dim3(col_slices(d), nsplit, B), kThreads, 0, stream>>>(ws, S, d, rows_per_split, dx, ld_dx);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

}  // namespace opb
