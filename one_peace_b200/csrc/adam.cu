// Fused multi-tensor Adam step + global grad-norm / clip (optim/adam.py:173-253 python form — the defined
// oracle, SURVEY.md §8c; wrapper semantics of optim/fp16_optimizer_memory_efficent.py:96-130).
//
//   per element, fp32:   g  = grad * grad_scale                 (deferred multiply_grads * clip coefficient)
//                        m  = b1 m + (1-b1) g ;  v = b2 v + (1-b2) g^2
//                        p -= lr wd p                           (decoupled decay, :243-246)
//                        p -= lr sqrt(1-b2^t)/(1-b1^t) * m / (sqrt(v) + eps)      (eps on the un-corrected sqrt(v))
//   p is read from the fp32 master copy when one is given (adam_fused.py keeps p_data_fp32), else up-cast from the
//   bf16 parameter (adam.py:197-199) — and written back to both.
//
// HBM-bound: one pass, 16-byte vector accesses, one CTA per 8192-element chunk of one tensor; the chunk table
// lives in device memory and is built once per parameter set.  Traffic with a master copy: read g(2) + p32/m/v (12),
// write p32/m/v (12) + p16 (2) = 28 B / parameter.
//
// The grad norm is a two-stage reduction with a fixed order (per-chunk partials, then one block sums them in
// index order in fp64), so identical gradients give bit-identical norms on every rank — the trainer's cross-rank
// consistency check (trainer.py:1245-1282) relies on that.
#include "common.cuh"
#include "ops.h"

namespace opb {

constexpr int kChunk = 8192;
constexpr int kAdamThreads = 256;

template <typename T>
OPB_DEVICE void ld4(const T* p, float (&v)[4]);
template <>
OPB_DEVICE void ld4<float>(const float* p, float (&v)[4]) {
  const float4 a = *reinterpret_cast<const float4*>(p);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
}
template <>
OPB_DEVICE void ld4<__nv_bfloat16>(const __nv_bfloat16* p, float (&v)[4]) {
  const uint2 u = *reinterpret_cast<const uint2*>(p);
  const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
}
template <typename T>
OPB_DEVICE void st4(T* p, const float (&v)[4]);
template <>
OPB_DEVICE void st4<float>(float* p, const float (&v)[4]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
template <>
OPB_DEVICE void st4<__nv_bfloat16>(__nv_bfloat16* p, const float (&v)[4]) {
  uint2 u;
  u.x = pack_bf16x2(v[0], v[1]);
  u.y = pack_bf16x2(v[2], v[3]);
  *reinterpret_cast<uint2*>(p) = u;
}

template <typename T>
OPB_DEVICE float ld1(const T* p, long i);
template <>
OPB_DEVICE float ld1<float>(const float* p, long i) { return p[i]; }
template <>
OPB_DEVICE float ld1<__nv_bfloat16>(const __nv_bfloat16* p, long i) { return __bfloat162float(p[i]); }
template <typename T>
OPB_DEVICE void st1(T* p, long i, float v);
template <>
OPB_DEVICE void st1<float>(float* p, long i, float v) { p[i] = v; }
template <>
OPB_DEVICE void st1<__nv_bfloat16>(__nv_bfloat16* p, long i, float v) { p[i] = __float2bfloat16(v); }

OPB_DEVICE void adam_math(float& p, float g, float& m, float& v, float b1, float b2, float eps, float lr_wd,
                          float step_size) {
  m = __fadd_rn(__fmul_rn(m, b1), __fmul_rn(g, 1.f - b1));
  v = __fadd_rn(__fmul_rn(v, b2), __fmul_rn(__fmul_rn(1.f - b2, g), g));   // addcmul_: value * t1 * t2
  const float denom = __fadd_rn(sqrtf(v), eps);
  if (lr_wd != 0.f) p = __fadd_rn(p, __fmul_rn(p, -lr_wd));
  p = __fadd_rn(p, __fmul_rn(-step_size, __fdiv_rn(m, denom)));
}

template <typename TP, typename TG>
__device__ void adam_chunk(const AdamTensor& t, long off, long n, float gscale, float b1, float b2, float eps,
                           float lr_wd, float step_size) {
  TP* p = reinterpret_cast<TP*>(t.p) + off;
  const TG* g = reinterpret_cast<const TG*>(t.g) + off;
  float* m = t.m + off;
  float* v = t.v + off;
  float* master = t.master ? t.master + off : nullptr;
  const bool vec_ok = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                        reinterpret_cast<uintptr_t>(v) | reinterpret_cast<uintptr_t>(master)) & 15) == 0;
  if (vec_ok) {
    const long n4 = n & ~3L;
    for (long i = threadIdx.x * 4L; i < n4; i += kAdamThreads * 4L) {
      float pv[4], gv[4], mv[4], vv[4];
      if (master) ld4<float>(master + i, pv); else ld4<TP>(p + i, pv);
      ld4<TG>(g + i, gv);
      ld4<float>(m + i, mv);
      ld4<float>(v + i, vv);
#pragma unroll
      for (int e = 0; e < 4; ++e) adam_math(pv[e], gv[e] * gscale, mv[e], vv[e], b1, b2, eps, lr_wd, step_size);
      st4<float>(m + i, mv);
      st4<float>(v + i, vv);
      if (master) st4<float>(master + i, pv);
      st4<TP>(p + i, pv);
    }
    for (long i = n4 + threadIdx.x; i < n; i += kAdamThreads) {
      float pv = master ? master[i] : ld1<TP>(p, i);
      float mv = m[i], vv = v[i];
      adam_math(pv, ld1<TG>(g, i) * gscale, mv, vv, b1, b2, eps, lr_wd, step_size);
      m[i] = mv; v[i] = vv;
      if (master) master[i] = pv;
      st1<TP>(p, i, pv);
    }
  } else {
    for (long i = threadIdx.x; i < n; i += kAdamThreads) {
      float pv = master ? master[i] : ld1<TP>(p, i);
      float mv = m[i], vv = v[i];
      adam_math(pv, ld1<TG>(g, i) * gscale, mv, vv, b1, b2, eps, lr_wd, step_size);
      m[i] = mv; v[i] = vv;
      if (master) master[i] = pv;
      st1<TP>(p, i, pv);
    }
  }
}

__global__ void __launch_bounds__(kAdamThreads)
adam_multi_kernel(const AdamTensor* __restrict__ tensors, const int* __restrict__ chunk_tensor,
                  const long* __restrict__ chunk_off, const AdamGroups groups, const float* __restrict__ grad_scale) {
  const int c = blockIdx.x;
  const AdamTensor t = tensors[chunk_tensor[c]];
  const long off = chunk_off[c];
  long n = t.numel - off;
  if (n > kChunk) n = kChunk;
  const float gscale = grad_scale ? *grad_scale : 1.f;
  const int gi = t.group;
  const float lr = groups.lr[gi];
  const float lr_wd = groups.wd[gi] * lr;
  const float step_size = lr * groups.bias_corr[gi];
  const float b1 = groups.beta1, b2 = groups.beta2, eps = groups.eps;
  if (t.p_dtype == 0 && t.g_dtype == 0) adam_chunk<float, float>(t, off, n, gscale, b1, b2, eps, lr_wd, step_size);
  else if (t.p_dtype == 1 && t.g_dtype == 1) adam_chunk<__nv_bfloat16, __nv_bfloat16>(t, off, n, gscale, b1, b2, eps, lr_wd, step_size);
  else if (t.p_dtype == 1 && t.g_dtype == 0) adam_chunk<__nv_bfloat16, float>(t, off, n, gscale, b1, b2, eps, lr_wd, step_size);
  else adam_chunk<float, __nv_bfloat16>(t, off, n, gscale, b1, b2, eps, lr_wd, step_size);
}

int adam_multi_step(const void* tensors, const int* chunk_tensor, const long* chunk_off, int n_chunks,
                    const AdamGroups& groups, const float* grad_scale, cudaStream_t stream) {
  if (n_chunks <= 0) return OPB_ERR_INVALID;
  adam_multi_kernel<<<n_chunks, kAdamThreads, 0, stream>>>(reinterpret_cast<const AdamTensor*>(tensors), chunk_tensor,
                                                           chunk_off, groups, grad_scale);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

// ---- Adan (optim/adan.py:146-223), same chunk table and launch shape as Adam ----
//   per element, fp32:   g = grad * grad_scale ;  diff = g - (first ? g : pre) ;  u = g + b2 diff
//                        m = b1 m + (1-b1) g ;  n = b2 n + (1-b2) diff ;  v = b3 v + (1-b3) u^2
//                        upd = (m / bc1 + (b2 n) / bc2) / (sqrt(v) / sqrt(bc3) + eps)
//                        proximal (no_prox = 0):  p = (p - lr upd) / (1 + lr wd)      (:216-218)
//                        no_prox = 1:             p = p (1 - lr wd) - lr upd          (:213-215)
//                        pre = g                                                       (:220, the scaled gradient)
// Each operation is rounded on its own, in the reference's order.  Traffic: read g + p + m/n/v/pre (16), write
// m/n/v/pre (16) + p: 38 B / parameter with bf16 p and g, 44 B with fp32 p and g or with a master copy.
struct AdanCoef {
  float b1, b2, b3, c1, c2, c3, eps, lr, decay, bc1, bc2, sbc3;
  bool no_prox;
};

OPB_DEVICE void adan_math(float& p, float g, float& pre, float& m, float& n, float& v, bool first, const AdanCoef& c) {
  // first step: pre_grad = g (:197-198), so diff = g - g: 0, or NaN for a non-finite g, as in the reference
  const float diff = __fsub_rn(g, first ? g : pre);
  const float u = __fadd_rn(g, __fmul_rn(c.b2, diff));
  m = __fadd_rn(__fmul_rn(m, c.b1), __fmul_rn(g, c.c1));
  n = __fadd_rn(__fmul_rn(n, c.b2), __fmul_rn(diff, c.c2));
  v = __fadd_rn(__fmul_rn(v, c.b3), __fmul_rn(__fmul_rn(c.c3, u), u));   // addcmul_: value * t1 * t2
  const float denom = __fadd_rn(__fdiv_rn(sqrtf(v), c.sbc3), c.eps);
  const float upd = __fdiv_rn(__fadd_rn(__fdiv_rn(m, c.bc1), __fdiv_rn(__fmul_rn(c.b2, n), c.bc2)), denom);
  if (c.no_prox) p = __fadd_rn(__fmul_rn(p, c.decay), __fmul_rn(-c.lr, upd));
  else p = __fdiv_rn(__fadd_rn(p, __fmul_rn(-c.lr, upd)), c.decay);
  pre = g;
}

template <typename TP, typename TG>
__device__ void adan_chunk(const AdanTensor& t, long off, long cnt, float gscale, const AdanCoef& c) {
  TP* p = reinterpret_cast<TP*>(t.p) + off;
  const TG* g = reinterpret_cast<const TG*>(t.g) + off;
  float* m = t.m + off;
  float* n = t.n + off;
  float* v = t.v + off;
  float* pre = t.pre + off;
  float* master = t.master ? t.master + off : nullptr;
  const bool first = t.first != 0;
  const bool vec_ok = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                        reinterpret_cast<uintptr_t>(n) | reinterpret_cast<uintptr_t>(v) | reinterpret_cast<uintptr_t>(pre) |
                        reinterpret_cast<uintptr_t>(master)) & 15) == 0;
  long i0 = threadIdx.x;
  if (vec_ok) {
    const long n4 = cnt & ~3L;
    for (long i = threadIdx.x * 4L; i < n4; i += kAdamThreads * 4L) {
      float pv[4], gv[4], mv[4], nv[4], vv[4], qv[4] = {0.f, 0.f, 0.f, 0.f};
      if (master) ld4<float>(master + i, pv); else ld4<TP>(p + i, pv);
      ld4<TG>(g + i, gv);
      ld4<float>(m + i, mv);
      ld4<float>(n + i, nv);
      ld4<float>(v + i, vv);
      if (!first) ld4<float>(pre + i, qv);
#pragma unroll
      for (int e = 0; e < 4; ++e) adan_math(pv[e], __fmul_rn(gv[e], gscale), qv[e], mv[e], nv[e], vv[e], first, c);
      st4<float>(m + i, mv);
      st4<float>(n + i, nv);
      st4<float>(v + i, vv);
      st4<float>(pre + i, qv);
      if (master) st4<float>(master + i, pv);
      st4<TP>(p + i, pv);
    }
    i0 = n4 + threadIdx.x;
  }
  for (long i = i0; i < cnt; i += kAdamThreads) {
    float pv = master ? master[i] : ld1<TP>(p, i);
    float qv = first ? 0.f : pre[i];
    float mv = m[i], nv = n[i], vv = v[i];
    adan_math(pv, __fmul_rn(ld1<TG>(g, i), gscale), qv, mv, nv, vv, first, c);
    m[i] = mv; n[i] = nv; v[i] = vv; pre[i] = qv;
    if (master) master[i] = pv;
    st1<TP>(p, i, pv);
  }
}

__global__ void __launch_bounds__(kAdamThreads)
adan_multi_kernel(const AdanTensor* __restrict__ tensors, const int* __restrict__ chunk_tensor,
                  const long* __restrict__ chunk_off, const AdanGroups groups, const float* __restrict__ grad_scale) {
  const int ci = blockIdx.x;
  const AdanTensor t = tensors[chunk_tensor[ci]];
  const long off = chunk_off[ci];
  long cnt = t.numel - off;
  if (cnt > kChunk) cnt = kChunk;
  const float gscale = grad_scale ? *grad_scale : 1.f;
  const int gi = t.group;
  AdanCoef c;
  c.b1 = groups.beta1; c.b2 = groups.beta2; c.b3 = groups.beta3; c.eps = groups.eps;
  c.c1 = 1.f - c.b1; c.c2 = 1.f - c.b2; c.c3 = 1.f - c.b3;
  c.lr = groups.lr[gi];
  c.no_prox = groups.no_prox[gi] != 0;
  const float lr_wd = __fmul_rn(c.lr, groups.wd[gi]);
  c.decay = c.no_prox ? __fsub_rn(1.f, lr_wd) : __fadd_rn(1.f, lr_wd);
  c.bc1 = groups.bc1[gi]; c.bc2 = groups.bc2[gi]; c.sbc3 = groups.sqrt_bc3[gi];
  if (t.p_dtype == 0 && t.g_dtype == 0) adan_chunk<float, float>(t, off, cnt, gscale, c);
  else if (t.p_dtype == 1 && t.g_dtype == 1) adan_chunk<__nv_bfloat16, __nv_bfloat16>(t, off, cnt, gscale, c);
  else if (t.p_dtype == 1 && t.g_dtype == 0) adan_chunk<__nv_bfloat16, float>(t, off, cnt, gscale, c);
  else adan_chunk<float, __nv_bfloat16>(t, off, cnt, gscale, c);
}

int adan_multi_step(const void* tensors, const int* chunk_tensor, const long* chunk_off, int n_chunks,
                    const AdanGroups& groups, const float* grad_scale, cudaStream_t stream) {
  if (n_chunks <= 0) return OPB_ERR_INVALID;
  adan_multi_kernel<<<n_chunks, kAdamThreads, 0, stream>>>(reinterpret_cast<const AdanTensor*>(tensors), chunk_tensor,
                                                           chunk_off, groups, grad_scale);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

// ---- grad norm: stage 1 = per-CTA sum of squares, stage 2 = ordered fp64 sum + clip coefficient ----
// CTA b owns chunks b, b + grid, b + 2 grid, ... (fixed assignment); every thread adds ITS elements of those chunks in that
// order into one register and the CTA reduces once at the end (fixed tree), so identical gradients give bit-identical norms
// on every rank and run (the trainer's cross-rank check, trainer.py:1245-1282).  Round-2 rework after the bench's hbm_kernels
// line showed 0.48-0.54 of the HBM peak: the per-chunk version paid a three-deep dependent metadata chain (chunk -> tensor ->
// pointer) and two block barriers for every 16 KB; now the next chunk's metadata is fetched before the current chunk's data
// loads are issued and nothing synchronises inside the loop.
struct SumsqMeta {
  const void* g; long n; int dtype;
};
OPB_DEVICE SumsqMeta sumsq_meta(const AdamTensor* __restrict__ tensors, const int* __restrict__ chunk_tensor,
                                const long* __restrict__ chunk_off, int c) {
  const AdamTensor* t = tensors + chunk_tensor[c];
  const long off = chunk_off[c];
  SumsqMeta m;
  m.dtype = t->g_dtype;
  long n = t->numel - off;
  m.n = n > kChunk ? kChunk : n;
  m.g = m.dtype == 0 ? static_cast<const void*>(reinterpret_cast<const float*>(t->g) + off)
                     : static_cast<const void*>(reinterpret_cast<const __nv_bfloat16*>(t->g) + off);
  return m;
}

__global__ void __launch_bounds__(kAdamThreads)
grad_sumsq_kernel(const AdamTensor* __restrict__ tensors, const int* __restrict__ chunk_tensor,
                  const long* __restrict__ chunk_off, float* __restrict__ partial, int n_chunks) {
  __shared__ float red[kAdamThreads / 32];
  float acc = 0.f;
  int c = blockIdx.x;
  SumsqMeta cur = {nullptr, 0, 0};
  if (c < n_chunks) cur = sumsq_meta(tensors, chunk_tensor, chunk_off, c);
  while (c < n_chunks) {
    const int cn = c + gridDim.x;
    SumsqMeta nxt = {nullptr, 0, 0};
    if (cn < n_chunks) nxt = sumsq_meta(tensors, chunk_tensor, chunk_off, cn);
    const long n = cur.n;
    if (cur.dtype == 0) {
      const float* g = reinterpret_cast<const float*>(cur.g);
      if ((reinterpret_cast<uintptr_t>(g) & 15) == 0 && n == kChunk) {
        float4 v[kChunk / (kAdamThreads * 4)];
#pragma unroll
        for (int k = 0; k < kChunk / (kAdamThreads * 4); ++k) v[k] = reinterpret_cast<const float4*>(g)[k * kAdamThreads + threadIdx.x];
#pragma unroll
        for (int k = 0; k < kChunk / (kAdamThreads * 4); ++k) acc += v[k].x * v[k].x + v[k].y * v[k].y + v[k].z * v[k].z + v[k].w * v[k].w;
      } else {
        for (long i = threadIdx.x; i < n; i += kAdamThreads) acc += g[i] * g[i];
      }
    } else {
      const __nv_bfloat16* g = reinterpret_cast<const __nv_bfloat16*>(cur.g);
      if ((reinterpret_cast<uintptr_t>(g) & 15) == 0 && n == kChunk) {
        uint4 v[kChunk / (kAdamThreads * 8)];
#pragma unroll
        for (int k = 0; k < kChunk / (kAdamThreads * 8); ++k) v[k] = reinterpret_cast<const uint4*>(g)[k * kAdamThreads + threadIdx.x];
#pragma unroll
        for (int k = 0; k < kChunk / (kAdamThreads * 8); ++k) {
          const float2 a = unpack_bf16x2(v[k].x), b = unpack_bf16x2(v[k].y), c2 = unpack_bf16x2(v[k].z), d = unpack_bf16x2(v[k].w);
          acc += a.x * a.x + a.y * a.y + b.x * b.x + b.y * b.y + c2.x * c2.x + c2.y * c2.y + d.x * d.x + d.y * d.y;
        }
      } else {
        for (long i = threadIdx.x; i < n; i += kAdamThreads) {
          const float x = __bfloat162float(g[i]);
          acc += x * x;
        }
      }
    }
    cur = nxt;
    c = cn;
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int w = 0; w < kAdamThreads / 32; ++w) s += red[w];
    partial[blockIdx.x] = s;
  }
}

// out[0] = multiply_factor * ||g||_2 ; out[1] = grad_scale = multiply_factor * clamp(max_norm / (norm + 1e-6), max=1)
__global__ void grad_norm_finalize_kernel(const float* __restrict__ partial, int n, float multiply_factor,
                                          float max_norm, float* __restrict__ out) {
  __shared__ double red[32];
  // fixed assignment of partials to threads and fixed tree order -> run-to-run and rank-to-rank deterministic
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) acc += static_cast<double>(partial[i]);
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < (blockDim.x >> 5); ++w) s += red[w];
    const float norm = multiply_factor * static_cast<float>(sqrt(s));
    float coef = 1.f;
    if (max_norm > 0.f) {
      // clamp(max=1) that keeps a NaN norm (fminf would drop it): a NaN gradient must poison the step, as in the reference
      const float r = max_norm / (norm + 1e-6f);
      coef = r >= 1.f ? 1.f : r;
    }
    out[0] = norm;
    out[1] = multiply_factor * coef;
  }
}

int grad_norm_clip(const void* tensors, const int* chunk_tensor, const long* chunk_off, int n_chunks, float* partial,
                   float multiply_factor, float max_norm, float* out2, cudaStream_t stream) {
  if (n_chunks <= 0) return OPB_ERR_INVALID;
  const int grid = n_chunks < 132 * 8 ? n_chunks : 132 * 8;
  grad_sumsq_kernel<<<grid, kAdamThreads, 0, stream>>>(reinterpret_cast<const AdamTensor*>(tensors), chunk_tensor, chunk_off,
                                                       partial, n_chunks);
  grad_norm_finalize_kernel<<<1, 1024, 0, stream>>>(partial, grid, multiply_factor, max_norm, out2);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

}  // namespace opb
