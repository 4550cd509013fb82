// Row-wise / column-reduction kernels of the encoder BACKWARD pass (reference: autograd through
// transformer_layer.py:165-228, multihead_attention.py:103-126, components.py:23-44):
//   layernorm_bwd     dx, dgamma, dbeta of  y = LN(x) * gamma + beta  (optionally y = gelu(LN(x)...), the hMLP stem)
//   geglu_fwd/bwd     u = gelu_erf(g) * l  on the un-fused [M, 2F] projection (transformer_layer.py:54-67)
//   gelu_fwd/bwd      y = gelu_erf(z) on the video adapters' [M, F] pre-activations (onepeace.py:29-39) and dz = dy gelu'(z)
//   scale_resid_fwd   x_out = x + row_scale * gamma * o           (LayerScale + drop-path residual, :70-88)
//   scale_resid_bwd   do = row_scale * gamma * dx, dgamma = sum_rows row_scale * dx * o, dbias = sum_rows do
//   colsum            bias gradients: sum over rows of a bf16 [M, n] matrix
//   attn_delta        delta[b,h,s] = sum_d dO * O  (softmax backward row term)
//   relpos_bias_bwd   dtable[bucket[i,j], h] += dbias[h,i,j]      (adapter/text.py:84-91, image.py:164-171)
// All are HBM-bound: one CTA walks rows grid-stride, every thread owns fixed 4-column groups, so the column
// reductions (dgamma / dbeta / dbias) accumulate in registers over the CTA's rows and are finished by a second tiny
// kernel over the per-CTA partials (deterministic: fixed row -> CTA assignment, fixed summation order).
#include "common.cuh"
#include "ops.h"

namespace opb {

namespace {

constexpr int kBwdThreads = 256;
constexpr int kMaxGroups = 6;          // 4-column groups per thread: dim <= 6 * 256 * 4 = 6144
constexpr int kBwdMaxBlocks = 132 * 8;

OPB_DEVICE float gelu_grad(float z) {
  // d/dz [ z * Phi(z) ] = Phi(z) + z * phi(z)
  const float cdf = 0.5f * (1.f + fast_erf(z * 0.70710678118654752f));
  const float pdf = 0.3989422804014327f * __expf(-0.5f * z * z);
  return cdf + z * pdf;
}

template <typename T>
OPB_DEVICE float4 load4(const T* p) {
  if constexpr (sizeof(T) == 4) {
    return *reinterpret_cast<const float4*>(p);
  } else {
    const uint2 v = *reinterpret_cast<const uint2*>(p);
    const float2 lo = unpack_bf16x2(v.x), hi = unpack_bf16x2(v.y);
    return make_float4(lo.x, lo.y, hi.x, hi.y);
  }
}
template <typename T>
OPB_DEVICE void store4(T* p, float4 v) {
  if constexpr (sizeof(T) == 4) {
    *reinterpret_cast<float4*>(p) = v;
  } else {
    uint2 o;
    o.x = pack_bf16x2(v.x, v.y);
    o.y = pack_bf16x2(v.z, v.w);
    *reinterpret_cast<uint2*>(p) = o;
  }
}

// sums two values over the CTA; every thread gets both totals
template <int THREADS>
OPB_DEVICE float2 block_sum2(float a, float b, float2* red) {
  a = warp_sum(a);
  b = warp_sum(b);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();                       // previous use of `red` finished
  if (lane == 0) red[warp] = make_float2(a, b);
  __syncthreads();
  float2 t = make_float2(0.f, 0.f);
#pragma unroll
  for (int w = 0; w < THREADS / 32; ++w) { t.x += red[w].x; t.y += red[w].y; }
  return t;
}

// sums four values over the CTA with ONE barrier pair; every thread gets all totals
template <int THREADS>
OPB_DEVICE float4 block_sum4(float a, float b, float c, float d, float4* red) {
  a = warp_sum(a); b = warp_sum(b); c = warp_sum(c); d = warp_sum(d);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();                       // previous use of `red` finished
  if (lane == 0) red[warp] = make_float4(a, b, c, d);
  __syncthreads();
  float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int w = 0; w < THREADS / 32; ++w) { const float4 r = red[w]; t.x += r.x; t.y += r.y; t.z += r.z; t.w += r.w; }
  return t;
}

// ---------------------------------------------------------------------------------------------------------------
// One CTA per row (grid-stride); THREADS x GROUPS float4 column groups cover `dim`.  gamma / beta are re-read per row
// (L1 hits) instead of living in registers: the kernel is HBM-bound and needs the occupancy (first version: 170
// registers, one 256-thread CTA per SM, 8x off the HBM roofline).
template <typename TX, typename TDY, typename TDX, int THREADS, int GROUPS>
__global__ void __launch_bounds__(THREADS, (THREADS * GROUPS >= 1536) ? 2 : 4)
layernorm_bwd_kernel(const TX* __restrict__ x, long ldx, const TDY* __restrict__ dy, long ld_dy,
                     const float* __restrict__ gamma, const float* __restrict__ beta, TDX* __restrict__ dx, long ld_dx,
                     int accumulate, float* __restrict__ partial, int rows, int dim, float eps, int gelu,
                     int dy_merge_w) {
  __shared__ float2 red[THREADS / 32];
  __shared__ float4 red4[THREADS / 32];
  const int ngroups = dim >> 2;
  float4 dg[GROUPS], db[GROUPS];
#pragma unroll
  for (int k = 0; k < GROUPS; ++k) dg[k] = db[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  const float inv_dim = 1.f / dim;
  // Software pipeline over the CTA's rows: the loads of row r + gridDim (and the old dx of row r when accumulating) are
  // issued before the three block reductions of row r, so HBM latency hides behind them (round 1 issued them after:
  // 0.46 of the HBM peak).
  auto load_row = [&](int row, float4 (&xr)[GROUPS], float4 (&gr)[GROUPS], float& shift) {
    shift = load4(x + row * ldx).x;          // x[row][0]: the shift of the single-pass statistics, fetched with the row (broadcast)
    // the forward's 2x2 pixel-merge scatter (layernorm.cu, adapter/image.py:37-47): row (b, y, x) of the w x w grid
    // went to row (b, y/2, x/2), column block (y%2)*2 + x%2 of the next conv's operand
    const TDY* dyr = dy + row * ld_dy;
    if (dy_merge_w > 0) {
      const int w = dy_merge_w;
      const int xx = row % w, yy = (row / w) % w, bb = row / (w * w);
      dyr = dy + ((static_cast<long>(bb) * (w / 2) + yy / 2) * (w / 2) + xx / 2) * ld_dy + ((yy & 1) * 2 + (xx & 1)) * dim;
    }
#pragma unroll
    for (int k = 0; k < GROUPS; ++k) {
      const int g = threadIdx.x + k * THREADS;
      if (g < ngroups) {
        xr[k] = load4(x + row * ldx + 4 * g);
        gr[k] = load4(dyr + 4 * g);
      } else {
        xr[k] = gr[k] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
  };
  constexpr bool kPrefetch = THREADS == 128;   // dim <= 1536 variants only: the wider ones have no registers to spare (and 12-24 KB rows)
  float4 xn[kPrefetch ? GROUPS : 1], gn[kPrefetch ? GROUPS : 1];
  float kn = 0.f;
  if constexpr (kPrefetch) {
    if (blockIdx.x < rows) load_row(blockIdx.x, xn, gn, kn);
  }
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    float4 xv[GROUPS], gv[GROUPS], oldv[GROUPS];
    float s1 = 0.f, ksh = 0.f;
    if constexpr (kPrefetch) {
#pragma unroll
      for (int k = 0; k < GROUPS; ++k) { xv[k] = xn[k]; gv[k] = gn[k]; }
      ksh = kn;
      if (row + static_cast<int>(gridDim.x) < rows) load_row(row + gridDim.x, xn, gn, kn);
    } else {
      load_row(row, xv, gv, ksh);
    }
    if (accumulate) {
#pragma unroll
      for (int k = 0; k < GROUPS; ++k) {
        const int g = threadIdx.x + k * THREADS;
        oldv[k] = g < ngroups ? load4(dx + row * ld_dx + 4 * g) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    if (!gelu) {
      // Plain LayerNorm adjoint with ONE block reduction per row instead of three (round 2: the FFN LayerNorm rows, 6144 wide,
      // ran at 0.68 of the HBM peak, the CTA idling in three barrier pairs per row).  With the shift K = x[row][0]:
      //   mean = K + S1/n, var = S2/n - (S1/n)^2            S1 = sum (x-K), S2 = sum (x-K)^2   (shifted: no cancellation)
      //   sum dy g = B1,   sum dy g xhat = rstd (B2 - (S1/n) B1)                                 B2 = sum dy g (x-K)
      float a1 = 0.f, a2 = 0.f, b1 = 0.f, b2 = 0.f;
#pragma unroll
      for (int k = 0; k < GROUPS; ++k) {
        const int g = threadIdx.x + k * THREADS;
        if (g < ngroups) {
          const float4 gm = gamma != nullptr ? __ldg(reinterpret_cast<const float4*>(gamma + 4 * g)) : make_float4(1.f, 1.f, 1.f, 1.f);
          xv[k].x -= ksh; xv[k].y -= ksh; xv[k].z -= ksh; xv[k].w -= ksh;
          a1 += xv[k].x + xv[k].y + xv[k].z + xv[k].w;
          a2 += xv[k].x * xv[k].x + xv[k].y * xv[k].y + xv[k].z * xv[k].z + xv[k].w * xv[k].w;
          const float4 gy = make_float4(gv[k].x * gm.x, gv[k].y * gm.y, gv[k].z * gm.z, gv[k].w * gm.w);
          b1 += gy.x + gy.y + gy.z + gy.w;
          b2 += gy.x * xv[k].x + gy.y * xv[k].y + gy.z * xv[k].z + gy.w * xv[k].w;
        }
      }
      const float4 t = block_sum4<THREADS>(a1, a2, b1, b2, red4);
      const float ms = t.x * inv_dim;                                  // mean - K
      const float rstd = rsqrtf(fmaxf(t.y * inv_dim - ms * ms, 0.f) + eps);
      const float m1 = t.z * inv_dim, m2 = rstd * (t.w - ms * t.z) * inv_dim;
#pragma unroll
      for (int k = 0; k < GROUPS; ++k) {
        const int g = threadIdx.x + k * THREADS;
        if (g < ngroups) {
          const float4 gm = gamma != nullptr ? __ldg(reinterpret_cast<const float4*>(gamma + 4 * g)) : make_float4(1.f, 1.f, 1.f, 1.f);
          const float4 xh = make_float4((xv[k].x - ms) * rstd, (xv[k].y - ms) * rstd, (xv[k].z - ms) * rstd, (xv[k].w - ms) * rstd);
          dg[k].x += gv[k].x * xh.x; dg[k].y += gv[k].y * xh.y; dg[k].z += gv[k].z * xh.z; dg[k].w += gv[k].w * xh.w;
          db[k].x += gv[k].x; db[k].y += gv[k].y; db[k].z += gv[k].z; db[k].w += gv[k].w;
          float4 o;
          o.x = rstd * (gv[k].x * gm.x - m1 - xh.x * m2);
          o.y = rstd * (gv[k].y * gm.y - m1 - xh.y * m2);
          o.z = rstd * (gv[k].z * gm.z - m1 - xh.z * m2);
          o.w = rstd * (gv[k].w * gm.w - m1 - xh.w * m2);
          if (accumulate) { o.x += oldv[k].x; o.y += oldv[k].y; o.z += oldv[k].z; o.w += oldv[k].w; }
          store4(dx + row * ld_dx + 4 * g, o);
        }
      }
      continue;
    }
#pragma unroll
    for (int k = 0; k < GROUPS; ++k) s1 += xv[k].x + xv[k].y + xv[k].z + xv[k].w;
    const float mean = block_sum2<THREADS>(s1, 0.f, red).x * inv_dim;
    float s2 = 0.f;
#pragma unroll
    for (int k = 0; k < GROUPS; ++k) {
      const int g = threadIdx.x + k * THREADS;
      if (g < ngroups) {
        xv[k].x -= mean; xv[k].y -= mean; xv[k].z -= mean; xv[k].w -= mean;
        s2 += xv[k].x * xv[k].x + xv[k].y * xv[k].y + xv[k].z * xv[k].z + xv[k].w * xv[k].w;
      }
    }
    const float rstd = rsqrtf(block_sum2<THREADS>(s2, 0.f, red).x * inv_dim + eps);
    float c1 = 0.f, c2 = 0.f;
#pragma unroll
    for (int k = 0; k < GROUPS; ++k) {
      const int g = threadIdx.x + k * THREADS;
      if (g < ngroups) {
        const float4 gm = gamma != nullptr ? __ldg(reinterpret_cast<const float4*>(gamma + 4 * g)) : make_float4(1.f, 1.f, 1.f, 1.f);
        xv[k].x *= rstd; xv[k].y *= rstd; xv[k].z *= rstd; xv[k].w *= rstd;       // x-hat
        if (gelu) {
          const float4 bt = beta != nullptr ? __ldg(reinterpret_cast<const float4*>(beta + 4 * g)) : make_float4(0.f, 0.f, 0.f, 0.f);
          gv[k].x *= gelu_grad(fmaf(xv[k].x, gm.x, bt.x));
          gv[k].y *= gelu_grad(fmaf(xv[k].y, gm.y, bt.y));
          gv[k].z *= gelu_grad(fmaf(xv[k].z, gm.z, bt.z));
          gv[k].w *= gelu_grad(fmaf(xv[k].w, gm.w, bt.w));
        }
        dg[k].x += gv[k].x * xv[k].x; dg[k].y += gv[k].y * xv[k].y; dg[k].z += gv[k].z * xv[k].z; dg[k].w += gv[k].w * xv[k].w;
        db[k].x += gv[k].x; db[k].y += gv[k].y; db[k].z += gv[k].z; db[k].w += gv[k].w;
        gv[k].x *= gm.x; gv[k].y *= gm.y; gv[k].z *= gm.z; gv[k].w *= gm.w;   // dy * gamma
        c1 += gv[k].x + gv[k].y + gv[k].z + gv[k].w;
        c2 += gv[k].x * xv[k].x + gv[k].y * xv[k].y + gv[k].z * xv[k].z + gv[k].w * xv[k].w;
      }
    }
    const float2 c = block_sum2<THREADS>(c1, c2, red);
    const float m1 = c.x * inv_dim, m2 = c.y * inv_dim;
#pragma unroll
    for (int k = 0; k < GROUPS; ++k) {
      const int g = threadIdx.x + k * THREADS;
      if (g < ngroups) {
        float4 o;
        o.x = rstd * (gv[k].x - m1 - xv[k].x * m2);
        o.y = rstd * (gv[k].y - m1 - xv[k].y * m2);
        o.z = rstd * (gv[k].z - m1 - xv[k].z * m2);
        o.w = rstd * (gv[k].w - m1 - xv[k].w * m2);
        TDX* p = dx + row * ld_dx + 4 * g;
        if (accumulate) { o.x += oldv[k].x; o.y += oldv[k].y; o.z += oldv[k].z; o.w += oldv[k].w; }
        store4(p, o);
      }
    }
  }
  if (partial != nullptr) {
    float* pg = partial + static_cast<long>(blockIdx.x) * 2 * dim;
#pragma unroll
    for (int k = 0; k < GROUPS; ++k) {
      const int g = threadIdx.x + k * THREADS;
      if (g < ngroups) {
        *reinterpret_cast<float4*>(pg + 4 * g) = dg[k];
        *reinterpret_cast<float4*>(pg + dim + 4 * g) = db[k];
      }
    }
  }
}

// out_v[c] = sum_p partial[p * stride + v * n + c]   (c < n; v = blockIdx.y selects one of up to two vectors that share the
// partial records, e.g. dgamma | dbeta).  CTA = 32 columns x 32 part-lanes: the `parts` (up to 1184) records of a column are
// summed by 32 threads in a fixed interleaved order with four independent loads in flight, then combined in a fixed order
// (deterministic).  The 8-lane, one-vector-per-launch version took 11 us per call, 1053 calls = 4 % of a training step.
__global__ void __launch_bounds__(1024)
partial_reduce_kernel(const float* __restrict__ partial, int parts, long stride, float* __restrict__ out0,
                      float* __restrict__ out1, int n) {
  __shared__ float red[32][33];
  const int cx = threadIdx.x & 31, py = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cx;
  float* out = blockIdx.y == 0 ? out0 : out1;
  if (out == nullptr) return;                      // uniform per CTA
  const float* src = partial + static_cast<long>(blockIdx.y) * n + c;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  if (c < n) {
    int p = py;
    for (; p + 96 < parts; p += 128) {
      s0 += src[p * stride]; s1 += src[(p + 32) * stride]; s2 += src[(p + 64) * stride]; s3 += src[(p + 96) * stride];
    }
    for (; p < parts; p += 32) s0 += src[p * stride];
  }
  red[py][cx] = (s0 + s1) + (s2 + s3);
  __syncthreads();
  if (py == 0 && c < n) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 32; ++k) t += red[k][cx];
    out[c] = t;
  }
}

int grid_for_rows(int rows) { return rows < kBwdMaxBlocks ? rows : kBwdMaxBlocks; }

// out0 <- vector 0 of the records, out1 <- vector 1 (n floats further); either may be null
int reduce_partials(const float* partial, int parts, long stride, float* out0, float* out1, int n, cudaStream_t stream) {
  if (out0 == nullptr && out1 == nullptr) return OPB_OK;
  partial_reduce_kernel<<<dim3((n + 31) / 32, out1 != nullptr ? 2 : 1), 1024, 0, stream>>>(partial, parts, stride, out0, out1, n);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

// ---------------------------------------------------------------------------------------------------------------
// 16-byte accesses (8 bf16 per thread), column group fixed per thread, rows walked with a grid stride in y — no 64-bit index
// division in the loop, two rows in flight per thread (the 8-byte / div-per-iteration version ran at 0.71 of the HBM peak).
OPB_DEVICE void unpack8(const uint4 v, float (&f)[8]) {
  const float2 a = unpack_bf16x2(v.x), b = unpack_bf16x2(v.y), c = unpack_bf16x2(v.z), d = unpack_bf16x2(v.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
OPB_DEVICE uint4 pack8(const float (&f)[8]) {
  return make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
}

__global__ void __launch_bounds__(256)
geglu_fwd_kernel(const __nv_bfloat16* __restrict__ gl, __nv_bfloat16* __restrict__ u, long rows, int F) {
  const int c = (blockIdx.x * 256 + threadIdx.x) * 8;
  if (c >= F) return;
  for (long r = blockIdx.y; r < rows; r += 2L * gridDim.y) {
    const long r2 = r + gridDim.y;
    const bool two = r2 < rows;
    const uint4 g0 = *reinterpret_cast<const uint4*>(gl + r * 2 * F + c), l0 = *reinterpret_cast<const uint4*>(gl + r * 2 * F + F + c);
    uint4 g1 = g0, l1 = l0;
    if (two) { g1 = *reinterpret_cast<const uint4*>(gl + r2 * 2 * F + c); l1 = *reinterpret_cast<const uint4*>(gl + r2 * 2 * F + F + c); }
    float g[8], l[8], o[8];
    unpack8(g0, g); unpack8(l0, l);
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = gelu_erf(g[e]) * l[e];
    *reinterpret_cast<uint4*>(u + r * F + c) = pack8(o);
    if (two) {
      unpack8(g1, g); unpack8(l1, l);
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = gelu_erf(g[e]) * l[e];
      *reinterpret_cast<uint4*>(u + r2 * F + c) = pack8(o);
    }
  }
}

__global__ void __launch_bounds__(256)
geglu_bwd_kernel(const __nv_bfloat16* __restrict__ gl, const __nv_bfloat16* __restrict__ du, __nv_bfloat16* __restrict__ dgl,
                 long rows, int F) {
  const int c = (blockIdx.x * 256 + threadIdx.x) * 8;
  if (c >= F) return;
  for (long r = blockIdx.y; r < rows; r += gridDim.y) {
    const uint4 gv = *reinterpret_cast<const uint4*>(gl + r * 2 * F + c), lv = *reinterpret_cast<const uint4*>(gl + r * 2 * F + F + c);
    const uint4 dv = *reinterpret_cast<const uint4*>(du + r * F + c);
    float g[8], l[8], d[8], og[8], ol[8];
    unpack8(gv, g); unpack8(lv, l); unpack8(dv, d);
#pragma unroll
    for (int e = 0; e < 8; ++e) { og[e] = d[e] * l[e] * gelu_grad(g[e]); ol[e] = d[e] * gelu_erf(g[e]); }
    *reinterpret_cast<uint4*>(dgl + r * 2 * F + c) = pack8(og);
    *reinterpret_cast<uint4*>(dgl + r * 2 * F + F + c) = pack8(ol);
  }
}

__global__ void __launch_bounds__(256)
gelu_fwd_kernel(const __nv_bfloat16* __restrict__ z, __nv_bfloat16* __restrict__ y, long n8) {
  for (long i = static_cast<long>(blockIdx.x) * 256 + threadIdx.x; i < n8; i += static_cast<long>(gridDim.x) * 256) {
    float f[8];
    unpack8(reinterpret_cast<const uint4*>(z)[i], f);
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] = gelu_erf(f[e]);
    reinterpret_cast<uint4*>(y)[i] = pack8(f);
  }
}

__global__ void __launch_bounds__(256)
gelu_bwd_kernel(const __nv_bfloat16* __restrict__ z, const __nv_bfloat16* __restrict__ dy, __nv_bfloat16* __restrict__ dz,
                long n8) {
  for (long i = static_cast<long>(blockIdx.x) * 256 + threadIdx.x; i < n8; i += static_cast<long>(gridDim.x) * 256) {
    float f[8], d[8];
    unpack8(reinterpret_cast<const uint4*>(z)[i], f);
    unpack8(reinterpret_cast<const uint4*>(dy)[i], d);
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] = d[e] * gelu_grad(f[e]);
    reinterpret_cast<uint4*>(dz)[i] = pack8(f);
  }
}

// ---------------------------------------------------------------------------------------------------------------
__global__ void scale_resid_fwd_kernel(const float* __restrict__ x, const __nv_bfloat16* __restrict__ o,
                                       const float* __restrict__ gamma, const float* __restrict__ row_scale,
                                       float* __restrict__ out, long rows, int n) {
  const long total = rows * (n / 4);
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const long r = i / (n / 4);
    const int c = static_cast<int>(i % (n / 4)) * 4;
    const float rs = row_scale != nullptr ? row_scale[r] : 1.f;
    const float4 g = gamma != nullptr ? *reinterpret_cast<const float4*>(gamma + c) : make_float4(1.f, 1.f, 1.f, 1.f);
    const float4 xv = *reinterpret_cast<const float4*>(x + r * n + c);
    const float4 ov = load4(o + r * n + c);
    *reinterpret_cast<float4*>(out + r * n + c) =
        make_float4(fmaf(rs * g.x, ov.x, xv.x), fmaf(rs * g.y, ov.y, xv.y), fmaf(rs * g.z, ov.z, xv.z), fmaf(rs * g.w, ov.w, xv.w));
  }
}

// partial layout: [block][2][n] = (dgamma, dbias)
__global__ void __launch_bounds__(kBwdThreads)
scale_resid_bwd_kernel(const float* __restrict__ dx, const __nv_bfloat16* __restrict__ o, const float* __restrict__ gamma,
                       const float* __restrict__ row_scale, __nv_bfloat16* __restrict__ d_o, float* __restrict__ partial,
                       int rows, int n, int in_period, int in_valid, int in_shift) {
  const int ngroups = n >> 2;
  float4 dg[kMaxGroups], db[kMaxGroups], gm[kMaxGroups];
#pragma unroll
  for (int k = 0; k < kMaxGroups; ++k) {
    dg[k] = db[k] = make_float4(0.f, 0.f, 0.f, 0.f);
    const int g = threadIdx.x + k * kBwdThreads;
    gm[k] = (g < ngroups && gamma != nullptr) ? *reinterpret_cast<const float4*>(gamma + 4 * g) : make_float4(1.f, 1.f, 1.f, 1.f);
  }
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    const float rs = row_scale != nullptr ? row_scale[row] : 1.f;
    // optional gather of the input rows: output row r reads dx row (r / in_valid) * in_period + in_shift + r % in_valid
    // (the token rows behind the CLS slot of every batch element)
    const long irow = in_valid > 0 ? static_cast<long>(row / in_valid) * in_period + in_shift + row % in_valid : row;
#pragma unroll
    for (int k = 0; k < kMaxGroups; ++k) {
      const int g = threadIdx.x + k * kBwdThreads;
      if (g < ngroups) {
        float4 d = *reinterpret_cast<const float4*>(dx + irow * n + 4 * g);
        d.x *= rs; d.y *= rs; d.z *= rs; d.w *= rs;
        if (o != nullptr) {
          const float4 ov = load4(o + static_cast<long>(row) * n + 4 * g);
          dg[k].x += d.x * ov.x; dg[k].y += d.y * ov.y; dg[k].z += d.z * ov.z; dg[k].w += d.w * ov.w;
        }
        d.x *= gm[k].x; d.y *= gm[k].y; d.z *= gm[k].z; d.w *= gm[k].w;
        // d_o is rounded to bf16 for the dW GEMM; the bias gradient sums the unrounded fp32 d (colsum, which serves
        // passes that only have d_o, sums the rounded values instead)
        uint2 pk;
        pk.x = pack_bf16x2(d.x, d.y);
        pk.y = pack_bf16x2(d.z, d.w);
        *reinterpret_cast<uint2*>(d_o + static_cast<long>(row) * n + 4 * g) = pk;
        db[k].x += d.x; db[k].y += d.y; db[k].z += d.z; db[k].w += d.w;
      }
    }
  }
  float* pg = partial + static_cast<long>(blockIdx.x) * 2 * n;
#pragma unroll
  for (int k = 0; k < kMaxGroups; ++k) {
    const int g = threadIdx.x + k * kBwdThreads;
    if (g < ngroups) {
      *reinterpret_cast<float4*>(pg + 4 * g) = dg[k];
      *reinterpret_cast<float4*>(pg + n + 4 * g) = db[k];
    }
  }
}

__global__ void __launch_bounds__(kBwdThreads)
colsum_kernel(const __nv_bfloat16* __restrict__ y, long ldy, float* __restrict__ partial, int rows, int n) {
  const int ngroups = n >> 2;
  float4 acc[kMaxGroups];
#pragma unroll
  for (int k = 0; k < kMaxGroups; ++k) acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
#pragma unroll
    for (int k = 0; k < kMaxGroups; ++k) {
      const int g = threadIdx.x + k * kBwdThreads;
      if (g < ngroups) {
        const float4 v = load4(y + row * ldy + 4 * g);
        acc[k].x += v.x; acc[k].y += v.y; acc[k].z += v.z; acc[k].w += v.w;
      }
    }
  }
  float* pg = partial + static_cast<long>(blockIdx.x) * n;
#pragma unroll
  for (int k = 0; k < kMaxGroups; ++k) {
    const int g = threadIdx.x + k * kBwdThreads;
    if (g < ngroups) *reinterpret_cast<float4*>(pg + 4 * g) = acc[k];
  }
}

// one warp per row: delta[(b*H + h)*S + s] = sum_d dO[row, h*64 + d] * O[row, h*64 + d]
__global__ void attn_delta_kernel(const __nv_bfloat16* __restrict__ d_o, const __nv_bfloat16* __restrict__ o,
                                  float* __restrict__ delta, int B, int S, int H) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B * S) return;
  const int b = warp / S, s = warp % S;
  const long base = static_cast<long>(warp) * H * 64;
  for (int h = 0; h < H; ++h) {
    const uint32_t a = *reinterpret_cast<const uint32_t*>(d_o + base + h * 64 + 2 * lane);
    const uint32_t c = *reinterpret_cast<const uint32_t*>(o + base + h * 64 + 2 * lane);
    const float2 af = unpack_bf16x2(a), cf = unpack_bf16x2(c);
    const float t = warp_sum(af.x * cf.x + af.y * cf.y);
    if (lane == 0) delta[(static_cast<long>(b) * H + h) * S + s] = t;
  }
}

__global__ void relpos_bias_bwd_kernel(const float* __restrict__ dbias, const int64_t* __restrict__ bucket,
                                       float* __restrict__ dtable, int S, int s_pad, int H, long ld_bucket) {
  const int i = blockIdx.x;
  for (int idx = threadIdx.x; idx < S * H; idx += blockDim.x) {
    const int h = idx / S, j = idx % S;
    const long bk = bucket[i * ld_bucket + j];
    atomicAdd(dtable + bk * H + h, dbias[(static_cast<long>(h) * S + i) * s_pad + j]);
  }
}

// out[c] (+)= sum_b in[b * ld + c]
__global__ void batch_sum_kernel(const float* __restrict__ in, long ld, float* __restrict__ out, int B, long n, int accumulate) {
  const long c = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  if (c >= n) return;
  float s = 0.f;
  for (int b = 0; b < B; ++b) s += in[b * ld + c];
  out[c] = accumulate ? out[c] + s : s;
}

// y = x / max(|x|, 1e-12) (F.normalize): dx = (dy - y (y . dy)) / |x|;  one warp per row
__global__ void l2_normalize_bwd_kernel(const float* __restrict__ x, long ldx, const float* __restrict__ dy, long ld_dy,
                                        float* __restrict__ dx, __nv_bfloat16* __restrict__ dx_bf16, int rows, int D) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* xr = x + row * ldx;
  const float* gr = dy + row * ld_dy;
  float ss = 0.f, dot = 0.f;
  for (int c = lane; c < D; c += 32) { ss += xr[c] * xr[c]; dot += xr[c] * gr[c]; }
  ss = warp_sum(ss);
  dot = warp_sum(dot);
  const float nrm = fmaxf(sqrtf(ss), 1e-12f);
  const float inv = 1.f / nrm;
  const float k = dot * inv * inv * inv;       // (y . dy) / |x| * (1 / |x|) with y = x / |x|
  for (int c = lane; c < D; c += 32) {
    const float v = gr[c] * inv - xr[c] * k;
    if (dx != nullptr) dx[static_cast<long>(row) * D + c] = v;
    if (dx_bf16 != nullptr) dx_bf16[static_cast<long>(row) * D + c] = __float2bfloat16(v);
  }
}

// adjoint of text_embed (adapters.cu; adapter/text.py:125-129,144-146): one CTA per (b, s) row of dx [B, T+1, D]
__global__ void text_embed_bwd_kernel(const float* __restrict__ dx, const int64_t* __restrict__ tokens,
                                      float* __restrict__ dtable, float* __restrict__ dpos, float* __restrict__ dcls,
                                      int B, int T, int D, int pad_idx) {
  const int row = blockIdx.x;
  const int S = T + 1;
  const int b = row / S, s = row % S;
  const float* g = dx + static_cast<long>(row) * D;
  if (s == 0) {
    for (int c = threadIdx.x; c < D; c += blockDim.x) {
      atomicAdd(dcls + c, g[c]);
      atomicAdd(dpos + c, g[c]);
    }
    return;
  }
  const long tok = tokens[static_cast<long>(b) * T + (s - 1)];
  if (tok == pad_idx) return;                 // padded rows were zeroed in the forward: no gradient
  float* dt = dtable + tok * D;
  float* dp = dpos + static_cast<long>(s) * D;
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    atomicAdd(dt + c, g[c]);
    atomicAdd(dp + c, g[c]);
  }
}

// im2col of a channel-last 1-D convolution (audio adapter, adapter/audio.py:57-80,254-311), grouped:
//   out[g][(b, t)][j * cg + c] = in[b, t * stride + j - pad, g * cg + c]   (zero outside [0, t_in))
// in: bf16 [B * t_in, groups * cg]; out: bf16 [groups][B * t_out][kw * cg].  8 channels (16 bytes) per thread.
__global__ void window_gather_kernel(const __nv_bfloat16* __restrict__ in, __nv_bfloat16* __restrict__ out, int B, int t_in,
                                     int t_out, int stride, int kw, int pad, int groups, int cg) {
  const int vpr = cg / 8;                                   // vectors per (row, tap)
  const long per_group = static_cast<long>(B) * t_out * kw * vpr;
  const long total = per_group * groups;
  const int C = groups * cg;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(i / per_group);
    long r = i % per_group;
    const int v = static_cast<int>(r % vpr); r /= vpr;
    const int j = static_cast<int>(r % kw); r /= kw;
    const int t = static_cast<int>(r % t_out);
    const int b = static_cast<int>(r / t_out);
    const int s = t * stride + j - pad;
    uint4 d = make_uint4(0u, 0u, 0u, 0u);
    if (s >= 0 && s < t_in) d = *reinterpret_cast<const uint4*>(in + (static_cast<long>(b) * t_in + s) * C + g * cg + 8 * v);
    *reinterpret_cast<uint4*>(out + ((static_cast<long>(g) * B * t_out + static_cast<long>(b) * t_out + t) * kw + j) * cg + 8 * v) = d;
  }
}

// col2im (adjoint of window_gather): dx[b, s, g * cg + c] = sum over (t, j) with t * stride + j - pad == s of
// dwin[g][(b, t)][j * cg + c];  fp32 accumulation, bf16 output.  Gather form: no atomics, deterministic.
__global__ void window_scatter_kernel(const __nv_bfloat16* __restrict__ dwin, __nv_bfloat16* __restrict__ dx, int B, int t_in,
                                      int t_out, int stride, int kw, int pad, int groups, int cg) {
  const int vpr = cg / 8;
  const int C = groups * cg;
  const long total = static_cast<long>(B) * t_in * groups * vpr;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long>(gridDim.x) * blockDim.x) {
    long r = i;
    const int v = static_cast<int>(r % vpr); r /= vpr;
    const int g = static_cast<int>(r % groups); r /= groups;
    const int s = static_cast<int>(r % t_in);
    const int b = static_cast<int>(r / t_in);
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int j = 0; j < kw; ++j) {
      const int num = s + pad - j;
      if (num < 0 || num % stride != 0) continue;
      const int t = num / stride;
      if (t >= t_out) continue;
      const uint4 d = *reinterpret_cast<const uint4*>(
          dwin + ((static_cast<long>(g) * B * t_out + static_cast<long>(b) * t_out + t) * kw + j) * cg + 8 * v);
      const float2 a0 = unpack_bf16x2(d.x), a1 = unpack_bf16x2(d.y), a2 = unpack_bf16x2(d.z), a3 = unpack_bf16x2(d.w);
      acc[0] += a0.x; acc[1] += a0.y; acc[2] += a1.x; acc[3] += a1.y; acc[4] += a2.x; acc[5] += a2.y; acc[6] += a3.x; acc[7] += a3.y;
    }
    uint4 o;
    o.x = pack_bf16x2(acc[0], acc[1]); o.y = pack_bf16x2(acc[2], acc[3]);
    o.z = pack_bf16x2(acc[4], acc[5]); o.w = pack_bf16x2(acc[6], acc[7]);
    *reinterpret_cast<uint4*>(dx + (static_cast<long>(b) * t_in + s) * C + g * cg + 8 * v) = o;
  }
}

}  // namespace

// ws: at least layernorm_bwd_ws_floats(dim) floats
long bwd_ws_floats(int dim) { return static_cast<long>(kBwdMaxBlocks) * 2 * dim; }

int layernorm_bwd(const void* x, int x_dtype, long ldx, const void* dy, int dy_dtype, long ld_dy, const float* gamma,
                  const float* beta, void* dx, int dx_dtype, long ld_dx, int accumulate, int rows, int dim, float eps,
                  int gelu, int dy_merge_w, float* ws, float* dgamma, float* dbeta, cudaStream_t stream) {
  if (rows <= 0 || dim <= 0 || (dim & 3) || dim > kMaxGroups * kBwdThreads * 4) return OPB_ERR_INVALID;
  if (dy_merge_w < 0 || (dy_merge_w & 1) || (dy_merge_w > 0 && rows % (dy_merge_w * dy_merge_w) != 0)) return OPB_ERR_INVALID;
  if ((ldx & 3) || (ld_dy & 3) || (ld_dx & 3)) return OPB_ERR_INVALID;
  if (accumulate && dx_dtype != 0) return OPB_ERR_INVALID;
  const bool want_param_grads = (dgamma != nullptr || dbeta != nullptr);
  if (want_param_grads && ws == nullptr) return OPB_ERR_INVALID;
  float* partial = want_param_grads ? ws : nullptr;
  // (threads, float4 groups per thread): 128 x 1 (dim <= 512), 128 x 3 (<= 1536), 256 x 3 (<= 3072), 256 x 6 (<= 6144)
  const int cfg = dim <= 512 ? 0 : (dim <= 1536 ? 1 : (dim <= 3072 ? 2 : 3));
  const int per_sm = cfg <= 1 ? 8 : (cfg == 2 ? 4 : 2);
  int grid = 132 * per_sm;
  if (grid > rows) grid = rows;
#define OPB_LNB_CFG(TX, TDY, TDX, TH, GR)                                                                             \
  layernorm_bwd_kernel<TX, TDY, TDX, TH, GR><<<grid, TH, 0, stream>>>(                                                \
      reinterpret_cast<const TX*>(x), ldx, reinterpret_cast<const TDY*>(dy), ld_dy, gamma, beta,                      \
      reinterpret_cast<TDX*>(dx), ld_dx, accumulate, partial, rows, dim, eps, gelu, dy_merge_w)
#define OPB_LNB(TX, TDY, TDX)                                                                                         \
  do {                                                                                                                \
    if (cfg == 0) OPB_LNB_CFG(TX, TDY, TDX, 128, 1);                                                                  \
    else if (cfg == 1) OPB_LNB_CFG(TX, TDY, TDX, 128, 3);                                                             \
    else if (cfg == 2) OPB_LNB_CFG(TX, TDY, TDX, 256, 3);                                                             \
    else OPB_LNB_CFG(TX, TDY, TDX, 256, 6);                                                                           \
  } while (0)
  const int key = (x_dtype != 0) * 4 + (dy_dtype != 0) * 2 + (dx_dtype != 0);
  switch (key) {
    case 0: OPB_LNB(float, float, float); break;
    case 1: OPB_LNB(float, float, __nv_bfloat16); break;
    case 2: OPB_LNB(float, __nv_bfloat16, float); break;
    case 3: OPB_LNB(float, __nv_bfloat16, __nv_bfloat16); break;
    case 4: OPB_LNB(__nv_bfloat16, float, float); break;
    case 5: OPB_LNB(__nv_bfloat16, float, __nv_bfloat16); break;
    case 6: OPB_LNB(__nv_bfloat16, __nv_bfloat16, float); break;
    default: OPB_LNB(__nv_bfloat16, __nv_bfloat16, __nv_bfloat16); break;
  }
#undef OPB_LNB_CFG
#undef OPB_LNB
  if (cudaGetLastError() != cudaSuccess) return OPB_ERR_CUDA;
  return reduce_partials(ws, grid, 2L * dim, dgamma, dbeta, dim, stream);
}

static int elementwise_grid(long total) {
  long g = (total + 255) / 256;
  if (g > 132L * 16) g = 132L * 16;
  return static_cast<int>(g < 1 ? 1 : g);
}

int geglu_fwd(const void* gl, void* u, long rows, int F, cudaStream_t stream) {
  if (rows <= 0 || F <= 0 || (F & 7) || (reinterpret_cast<uintptr_t>(gl) & 15) || (reinterpret_cast<uintptr_t>(u) & 15)) return OPB_ERR_INVALID;
  const unsigned gx = static_cast<unsigned>((F / 8 + 255) / 256);
  const unsigned gy = static_cast<unsigned>(rows < 132L * 16 / gx ? rows : 132L * 16 / gx);
  geglu_fwd_kernel<<<dim3(gx, gy > 0 ? gy : 1), 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(gl),
                                                                 reinterpret_cast<__nv_bfloat16*>(u), rows, F);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

int geglu_bwd(const void* gl, const void* du, void* dgl, long rows, int F, cudaStream_t stream) {
  if (rows <= 0 || F <= 0 || (F & 7) || (reinterpret_cast<uintptr_t>(gl) & 15) || (reinterpret_cast<uintptr_t>(du) & 15) ||
      (reinterpret_cast<uintptr_t>(dgl) & 15))
    return OPB_ERR_INVALID;
  const unsigned gx = static_cast<unsigned>((F / 8 + 255) / 256);
  const unsigned gy = static_cast<unsigned>(rows < 132L * 16 / gx ? rows : 132L * 16 / gx);
  geglu_bwd_kernel<<<dim3(gx, gy > 0 ? gy : 1), 256, 0, stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(gl), reinterpret_cast<const __nv_bfloat16*>(du),
      reinterpret_cast<__nv_bfloat16*>(dgl), rows, F);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

int gelu_fwd(const void* z, void* y, long rows, int F, cudaStream_t stream) {
  if (rows <= 0 || F <= 0 || (F & 7) || ((reinterpret_cast<uintptr_t>(z) | reinterpret_cast<uintptr_t>(y)) & 15))
    return OPB_ERR_INVALID;
  const long n8 = rows * (F / 8);
  gelu_fwd_kernel<<<elementwise_grid(n8), 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(z),
                                                             reinterpret_cast<__nv_bfloat16*>(y), n8);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

int gelu_bwd(const void* z, const void* dy, void* dz, long rows, int F, cudaStream_t stream) {
  if (rows <= 0 || F <= 0 || (F & 7) ||
      ((reinterpret_cast<uintptr_t>(z) | reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(dz)) & 15))
    return OPB_ERR_INVALID;
  const long n8 = rows * (F / 8);
  gelu_bwd_kernel<<<elementwise_grid(n8), 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(z),
                                                             reinterpret_cast<const __nv_bfloat16*>(dy),
                                                             reinterpret_cast<__nv_bfloat16*>(dz), n8);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

int scale_resid_fwd(const float* x, const void* o, const float* gamma, const float* row_scale, float* out, long rows,
                    int n, cudaStream_t stream) {
  if (rows <= 0 || n <= 0 || (n & 3)) return OPB_ERR_INVALID;
  scale_resid_fwd_kernel<<<elementwise_grid(rows * (n / 4)), 256, 0, stream>>>(
      x, reinterpret_cast<const __nv_bfloat16*>(o), gamma, row_scale, out, rows, n);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

int scale_resid_bwd(const float* dx, const void* o, const float* gamma, const float* row_scale, void* d_o, float* ws,
                    float* dgamma, float* dbias, int rows, int n, int in_period, int in_valid, int in_shift,
                    cudaStream_t stream) {
  if (rows <= 0 || n <= 0 || (n & 3) || n > kMaxGroups * kBwdThreads * 4 || ws == nullptr) return OPB_ERR_INVALID;
  if (dgamma != nullptr && o == nullptr) return OPB_ERR_INVALID;
  const int grid = grid_for_rows(rows);
  scale_resid_bwd_kernel<<<grid, kBwdThreads, 0, stream>>>(dx, reinterpret_cast<const __nv_bfloat16*>(o), gamma, row_scale,
                                                           reinterpret_cast<__nv_bfloat16*>(d_o), ws, rows, n, in_period,
                                                           in_valid, in_shift);
  if (cudaGetLastError() != cudaSuccess) return OPB_ERR_CUDA;
  return reduce_partials(ws, grid, 2L * n, dgamma, dbias, n, stream);
}

int colsum_bf16(const void* y, long ldy, float* ws, float* out, int rows, int n, cudaStream_t stream) {
  if (rows <= 0 || n <= 0 || (n & 3) || (ldy & 3) || n > kMaxGroups * kBwdThreads * 4 || ws == nullptr) return OPB_ERR_INVALID;
  const int grid = grid_for_rows(rows);
  colsum_kernel<<<grid, kBwdThreads, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(y), ldy, ws, rows, n);
  if (cudaGetLastError() != cudaSuccess) return OPB_ERR_CUDA;
  return reduce_partials(ws, grid, n, out, nullptr, n, stream);
}

int attn_delta(const void* d_o, const void* o, float* delta, int B, int S, int H, cudaStream_t stream) {
  if (B <= 0 || S <= 0 || H <= 0) return OPB_ERR_INVALID;
  const long warps = static_cast<long>(B) * S;
  attn_delta_kernel<<<static_cast<unsigned>((warps * 32 + 255) / 256), 256, 0, stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(d_o), reinterpret_cast<const __nv_bfloat16*>(o), delta, B, S, H);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

int relpos_bias_bwd(const float* dbias, const int64_t* bucket, float* dtable, int S, int s_pad, int H, long ld_bucket,
                    cudaStream_t stream) {
  if (S <= 0 || s_pad < S || H <= 0) return OPB_ERR_INVALID;
  relpos_bias_bwd_kernel<<<S, 256, 0, stream>>>(dbias, bucket, dtable, S, s_pad, H, ld_bucket);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

int batch_sum_f32(const float* in, long ld, float* out, int B, long n, int accumulate, cudaStream_t stream) {
  if (B <= 0 || n <= 0) return OPB_ERR_INVALID;
  batch_sum_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(in, ld, out, B, n, accumulate);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

int l2_normalize_bwd(const float* x, long ldx, const float* dy, long ld_dy, float* dx, void* dx_bf16, int rows, int D,
                     cudaStream_t stream) {
  if (rows <= 0 || D <= 0 || (dx == nullptr && dx_bf16 == nullptr)) return OPB_ERR_INVALID;
  l2_normalize_bwd_kernel<<<(rows * 32 + 255) / 256, 256, 0, stream>>>(x, ldx, dy, ld_dy, dx,
                                                                       reinterpret_cast<__nv_bfloat16*>(dx_bf16), rows, D);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

int text_embed_bwd(const float* dx, const int64_t* tokens, float* dtable, float* dpos, float* dcls, int B, int T, int D,
                   int pad_idx, cudaStream_t stream) {
  if (B <= 0 || T <= 0 || D <= 0) return OPB_ERR_INVALID;
  text_embed_bwd_kernel<<<B * (T + 1), 256, 0, stream>>>(dx, tokens, dtable, dpos, dcls, B, T, D, pad_idx);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

static int window_check(int B, int t_in, int t_out, int stride, int kw, int pad, int groups, int cg) {
  if (B <= 0 || t_in <= 0 || t_out <= 0 || stride <= 0 || kw <= 0 || pad < 0 || groups <= 0 || cg <= 0 || (cg & 7)) return OPB_ERR_INVALID;
  if (static_cast<long>(t_out - 1) * stride + kw - 1 - pad > static_cast<long>(t_in) - 1 + pad) return OPB_ERR_INVALID;   // windows stay inside the padded input
  return OPB_OK;
}

int window_gather(const void* in, void* out, int B, int t_in, int t_out, int stride, int kw, int pad, int groups, int cg,
                  cudaStream_t stream) {
  const int rc = window_check(B, t_in, t_out, stride, kw, pad, groups, cg);
  if (rc != OPB_OK) return rc;
  const long total = static_cast<long>(B) * t_out * kw * (cg / 8) * groups;
  window_gather_kernel<<<elementwise_grid(total), 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(in),
                                                                  reinterpret_cast<__nv_bfloat16*>(out), B, t_in, t_out, stride,
                                                                  kw, pad, groups, cg);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

int window_scatter(const void* dwin, void* dx, int B, int t_in, int t_out, int stride, int kw, int pad, int groups, int cg,
                   cudaStream_t stream) {
  const int rc = window_check(B, t_in, t_out, stride, kw, pad, groups, cg);
  if (rc != OPB_OK) return rc;
  const long total = static_cast<long>(B) * t_in * groups * (cg / 8);
  window_scatter_kernel<<<elementwise_grid(total), 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(dwin),
                                                                   reinterpret_cast<__nv_bfloat16*>(dx), B, t_in, t_out, stride,
                                                                   kw, pad, groups, cg);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

}  // namespace opb
