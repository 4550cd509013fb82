// Classification head of one_peace_classify (models/one_peace/one_peace_base.py:132-235, criterions/classify_loss.py,
// criterions/hinge_loss.py): the attention pooling of MultiheadAttentionPooling and the classification criteria.
//
// Attention pooling, per (sample b, head h) with a learned, UNSCALED query q_h (one_peace_base.py:146-173):
//     s_j = q_h . k_jh,  p = softmax_j(s) over the unpadded keys (fp32),  out_bh = sum_j p_j v_jh,  lse_bh = log sum_j e^s_j
// kv bf16 [B, T, 2d] holds k then v of every key row (one GEMM writes both).  One CTA per (h, b): 8 warps, each warp takes 4 keys
// at a time with 8 lanes per key (lane c of a group owns head elements 8c..8c+7, one 16-byte vector of k and of v), and runs an
// online soft-max; the 32 key groups are merged in a fixed order at the end, so results do not depend on scheduling.  Padded
// keys are never loaded.
// Backward: delta = sum_j p_j (dout . v_j) in a first sweep, then dk_j = p_j (dout . v_j - delta) q, dv_j = p_j dout; padded
// key rows of dkv are written as zeros.  dq = sum_b sum_j ds_j k_j goes through per-(b, h) partials and a fixed-order sum over b.
#include "common.cuh"
#include "ops.h"

namespace opb {

constexpr int kPoolThreads = 256;
constexpr int kPoolGroups = kPoolThreads / 8;       // 32 key groups of 8 lanes
constexpr int kPoolUnroll = 4;                      // keys in flight per lane

OPB_DEVICE float group8_sum(float v, unsigned mask) {
  v += __shfl_xor_sync(mask, v, 1);
  v += __shfl_xor_sync(mask, v, 2);
  v += __shfl_xor_sync(mask, v, 4);
  return v;
}

OPB_DEVICE void unpack8(const uint4& u, float* f) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}

OPB_DEVICE uint4 pack8(const float* f) {
  uint4 u;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return u;
}

// (m, l, acc) <- merge of two online soft-max states (every lane merges in a fixed pattern: results are run-to-run identical)
OPB_DEVICE void merge_state(float& m, float& l, float* acc, float m2, float l2, const float* acc2) {
  const float mn = fmaxf(m, m2);
  const float a = m == -INFINITY ? 0.f : expf(m - mn);
  const float b = m2 == -INFINITY ? 0.f : expf(m2 - mn);
  l = l * a + l2 * b;
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = acc[i] * a + acc2[i] * b;
  m = mn;
}

__global__ void __launch_bounds__(kPoolThreads)
attn_pool_fwd_kernel(const __nv_bfloat16* __restrict__ kv, const float* __restrict__ q, const uint8_t* __restrict__ key_pad,
                     __nv_bfloat16* __restrict__ out, float* __restrict__ lse, int T, int H) {
  const int h = blockIdx.x, b = blockIdx.y, d = H * 64;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int grp = threadIdx.x >> 3, c = lane & 7;
  const unsigned gmask = 0xffu << (lane & 24);
  float qv[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) qv[i] = q[h * 64 + c * 8 + i];
  const __nv_bfloat16* base = kv + static_cast<long>(b) * T * 2 * d + h * 64 + c * 8;
  const uint8_t* pad = key_pad != nullptr ? key_pad + static_cast<long>(b) * T : nullptr;
  float m = -INFINITY, l = 0.f, acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  for (int j0 = grp; j0 < T; j0 += kPoolGroups * kPoolUnroll) {
    uint4 kr[kPoolUnroll], vr[kPoolUnroll];
    bool ok[kPoolUnroll];
#pragma unroll
    for (int u = 0; u < kPoolUnroll; ++u) {
      const int j = j0 + u * kPoolGroups;
      ok[u] = j < T && (pad == nullptr || pad[j] == 0);
      kr[u] = vr[u] = make_uint4(0u, 0u, 0u, 0u);
      if (ok[u]) {
        const __nv_bfloat16* r = base + static_cast<long>(j) * 2 * d;
        kr[u] = *reinterpret_cast<const uint4*>(r);
        vr[u] = *reinterpret_cast<const uint4*>(r + d);
      }
    }
#pragma unroll
    for (int u = 0; u < kPoolUnroll; ++u) {
      if (!ok[u]) continue;                       // uniform over the 8 lanes of a key group
      float kf[8], vf[8];
      unpack8(kr[u], kf);
      unpack8(vr[u], vf);
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) s = fmaf(qv[i], kf[i], s);
      s = group8_sum(s, gmask);
      const float mn = fmaxf(m, s);
      const float a = expf(m - mn), p = expf(s - mn);
      l = l * a + p;
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fmaf(p, vf[i], acc[i] * a);
      m = mn;
    }
  }
  // the 4 key groups of a warp (lanes c, c+8, c+16, c+24), then the 8 warps in order
#pragma unroll
  for (int off = 8; off <= 16; off <<= 1) {
    float acc2[8];
    const float m2 = __shfl_xor_sync(0xffffffffu, m, off), l2 = __shfl_xor_sync(0xffffffffu, l, off);
#pragma unroll
    for (int i = 0; i < 8; ++i) acc2[i] = __shfl_xor_sync(0xffffffffu, acc[i], off);
    merge_state(m, l, acc, m2, l2, acc2);
  }
  __shared__ float sm_m[8][8], sm_l[8][8], sm_acc[8][8][8];
  if (lane < 8) {
    sm_m[warp][c] = m;
    sm_l[warp][c] = l;
#pragma unroll
    for (int i = 0; i < 8; ++i) sm_acc[warp][c][i] = acc[i];
  }
  __syncthreads();
  if (threadIdx.x < 8) {
    m = sm_m[0][c];
    l = sm_l[0][c];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = sm_acc[0][c][i];
    for (int w = 1; w < 8; ++w) merge_state(m, l, acc, sm_m[w][c], sm_l[w][c], sm_acc[w][c]);
    float o[8];
    const float inv = l > 0.f ? 1.f / l : 0.f;      // every key padded: out = 0, lse = -inf
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i] = acc[i] * inv;
    *reinterpret_cast<uint4*>(out + static_cast<long>(b) * d + h * 64 + c * 8) = pack8(o);
    if (c == 0) lse[b * H + h] = l > 0.f ? m + logf(l) : -INFINITY;
  }
}

// fixed-order sum of one value per thread over the CTA; every thread gets the result
OPB_DEVICE float cta_sum(float v, float* red) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
  for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) t += red[w];
  return t;
}

__global__ void __launch_bounds__(kPoolThreads)
attn_pool_bwd_kernel(const __nv_bfloat16* __restrict__ kv, const float* __restrict__ q, const uint8_t* __restrict__ key_pad,
                     const float* __restrict__ lse, const __nv_bfloat16* __restrict__ dout, __nv_bfloat16* __restrict__ dkv,
                     float* __restrict__ dq_part, int T, int H) {
  const int h = blockIdx.x, b = blockIdx.y, d = H * 64;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int grp = threadIdx.x >> 3, c = lane & 7;
  const unsigned gmask = 0xffu << (lane & 24);
  __shared__ float red[kPoolThreads / 32];
  __shared__ float sm_dq[8][64];
  float qv[8], dov[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) qv[i] = q[h * 64 + c * 8 + i];
  unpack8(*reinterpret_cast<const uint4*>(dout + static_cast<long>(b) * d + h * 64 + c * 8), dov);
  const float L = lse[b * H + h];
  const bool none = L == -INFINITY;                 // every key padded: all gradients are zero
  const long row0 = static_cast<long>(b) * T;
  const __nv_bfloat16* base = kv + row0 * 2 * d + h * 64 + c * 8;
  __nv_bfloat16* dbase = dkv + row0 * 2 * d + h * 64 + c * 8;
  const uint8_t* pad = key_pad != nullptr ? key_pad + row0 : nullptr;
  // sweep 1: delta = sum_j p_j (dout . v_j)
  float delta = 0.f;
  if (!none) {
    for (int j0 = grp; j0 < T; j0 += kPoolGroups * kPoolUnroll) {
      uint4 kr[kPoolUnroll], vr[kPoolUnroll];
      bool ok[kPoolUnroll];
#pragma unroll
      for (int u = 0; u < kPoolUnroll; ++u) {
        const int j = j0 + u * kPoolGroups;
        ok[u] = j < T && (pad == nullptr || pad[j] == 0);
        kr[u] = vr[u] = make_uint4(0u, 0u, 0u, 0u);
        if (ok[u]) {
          const __nv_bfloat16* r = base + static_cast<long>(j) * 2 * d;
          kr[u] = *reinterpret_cast<const uint4*>(r);
          vr[u] = *reinterpret_cast<const uint4*>(r + d);
        }
      }
#pragma unroll
      for (int u = 0; u < kPoolUnroll; ++u) {
        if (!ok[u]) continue;
        float kf[8], vf[8];
        unpack8(kr[u], kf);
        unpack8(vr[u], vf);
        float s = 0.f, dp = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) { s = fmaf(qv[i], kf[i], s); dp = fmaf(dov[i], vf[i], dp); }
        s = group8_sum(s, gmask);
        dp = group8_sum(dp, gmask);
        delta = fmaf(expf(s - L), dp, delta);
      }
    }
  }
  // every lane of a key group holds the same partial: count it once (lane c == 0)
  delta = cta_sum(c == 0 ? delta : 0.f, red);
  // sweep 2: dk, dv (zeros on padded rows) and the dq partial
  float dqa[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) dqa[i] = 0.f;
  const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
  for (int j0 = grp; j0 < T; j0 += kPoolGroups * kPoolUnroll) {
    uint4 kr[kPoolUnroll], vr[kPoolUnroll];
    bool ok[kPoolUnroll];
#pragma unroll
    for (int u = 0; u < kPoolUnroll; ++u) {
      const int j = j0 + u * kPoolGroups;
      ok[u] = !none && j < T && (pad == nullptr || pad[j] == 0);
      kr[u] = vr[u] = zero;
      if (ok[u]) {
        const __nv_bfloat16* r = base + static_cast<long>(j) * 2 * d;
        kr[u] = *reinterpret_cast<const uint4*>(r);
        vr[u] = *reinterpret_cast<const uint4*>(r + d);
      }
    }
#pragma unroll
    for (int u = 0; u < kPoolUnroll; ++u) {
      const int j = j0 + u * kPoolGroups;
      if (j >= T) continue;
      __nv_bfloat16* w = dbase + static_cast<long>(j) * 2 * d;
      if (!ok[u]) {
        *reinterpret_cast<uint4*>(w) = zero;
        *reinterpret_cast<uint4*>(w + d) = zero;
        continue;
      }
      float kf[8], vf[8];
      unpack8(kr[u], kf);
      unpack8(vr[u], vf);
      float s = 0.f, dp = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) { s = fmaf(qv[i], kf[i], s); dp = fmaf(dov[i], vf[i], dp); }
      s = group8_sum(s, gmask);
      dp = group8_sum(dp, gmask);
      const float p = expf(s - L);
      const float ds = p * (dp - delta);
      float dk[8], dv[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        dk[i] = ds * qv[i];
        dv[i] = p * dov[i];
        dqa[i] = fmaf(ds, kf[i], dqa[i]);
      }
      *reinterpret_cast<uint4*>(w) = pack8(dk);
      *reinterpret_cast<uint4*>(w + d) = pack8(dv);
    }
  }
  // dq partial of this (b, h): the 4 key groups of a warp, then the 8 warps in order
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    dqa[i] += __shfl_xor_sync(0xffffffffu, dqa[i], 8);
    dqa[i] += __shfl_xor_sync(0xffffffffu, dqa[i], 16);
  }
  if (lane < 8) {
#pragma unroll
    for (int i = 0; i < 8; ++i) sm_dq[warp][c * 8 + i] = dqa[i];
  }
  __syncthreads();
  if (threadIdx.x < 64) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += sm_dq[w][threadIdx.x];
    dq_part[(static_cast<long>(b) * H + h) * 64 + threadIdx.x] = t;
  }
}

// dq[h*64 + e] = sum_b dq_part[b, h, e], b in order
__global__ void attn_pool_dq_kernel(const float* __restrict__ dq_part, float* __restrict__ dq, int B, int n) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  float t = 0.f;
  for (int b = 0; b < B; ++b) t += dq_part[static_cast<long>(b) * n + e];
  dq[e] = t;
}

// ---------------------------------------------------------------------------------------------------------------------------
// classification criteria.  One CTA per logits row (per group of num_choices rows for the hinge form).
// ---------------------------------------------------------------------------------------------------------------------------
constexpr int kLossThreads = 256;

// (max, first index of the max) over the CTA; every thread gets the result
OPB_DEVICE void cta_argmax(float& v, int& idx, float* rv, int* ri) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const float v2 = __shfl_xor_sync(0xffffffffu, v, off);
    const int i2 = __shfl_xor_sync(0xffffffffu, idx, off);
    if (v2 > v || (v2 == v && i2 < idx)) { v = v2; idx = i2; }
  }
  const int warp = threadIdx.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) { rv[warp] = v; ri[warp] = idx; }
  __syncthreads();
  v = rv[0];
  idx = ri[0];
  for (int w = 1; w < kLossThreads / 32; ++w)
    if (rv[w] > v || (rv[w] == v && ri[w] < idx)) { v = rv[w]; idx = ri[w]; }
}

__global__ void __launch_bounds__(kLossThreads)
classify_loss_kernel(const float* __restrict__ logits, long ld, int rows, int n_valid, int mode, const int64_t* __restrict__ labels,
                     const float* __restrict__ targets, long ld_t, float eps, int num_choices, float* __restrict__ row_loss,
                     float* __restrict__ dlogits, float* __restrict__ row_correct, float* __restrict__ out2,
                     unsigned int* __restrict__ ticket) {
  __shared__ float red[kLossThreads / 32];
  __shared__ int redi[kLossThreads / 32];
  __shared__ bool last;
  const int r = blockIdx.x;
  float loss = 0.f, correct = 0.f;
  if (mode == 3) {
    // hinge_loss.py:44-51: logits [G * nc, 1] viewed as [G, nc]; loss = sum_c max(0, 1 + z_c - z_t) (the positive's own term
    // contributes its constant 1; the configured margin is not used by the reference)
    const long r0 = static_cast<long>(r) * num_choices;
    const long t = labels[r];
    const bool valid = t >= 0 && t < num_choices;
    const float zt = valid ? logits[(r0 + t) * ld] : 0.f;
    if (threadIdx.x == 0 && valid) {
      float best = logits[r0 * ld];
      int bi = 0;
      for (int c = 0; c < num_choices; ++c) {
        const float z = logits[(r0 + c) * ld];
        const float h = 1.f + z - zt;
        if (h > 0.f) loss += h;
        if (z > best) { best = z; bi = c; }
      }
      correct = bi == t ? 1.f : 0.f;
    }
    for (long e = threadIdx.x; e < num_choices * ld; e += blockDim.x) {
      const int c = static_cast<int>(e / ld), col = static_cast<int>(e % ld);
      float g = 0.f;
      if (valid && col == 0) {
        const float z = logits[(r0 + c) * ld];
        g = (1.f + z - zt > 0.f) ? 1.f : 0.f;
        if (c == t) {
          float n_act = 0.f;
          for (int cc = 0; cc < num_choices; ++cc) n_act += (1.f + logits[(r0 + cc) * ld] - zt > 0.f) ? 1.f : 0.f;
          g -= n_act;
        }
      }
      dlogits[r0 * ld + e] = g;
    }
  } else {
    const float* z = logits + static_cast<long>(r) * ld;
    float* dz = dlogits + static_cast<long>(r) * ld;
    float mx = -INFINITY;
    int am = 0x7fffffff;
    for (int cc = threadIdx.x; cc < n_valid; cc += blockDim.x)
      if (z[cc] > mx) { mx = z[cc]; am = cc; }
    cta_argmax(mx, am, red, redi);
    if (mode == 2) {
      // multi-label: binary_cross_entropy_with_logits, n_correct = targets[argmax]
      const float* tr = targets + static_cast<long>(r) * ld_t;
      float part = 0.f;
      for (int cc = threadIdx.x; cc < n_valid; cc += blockDim.x) {
        const float x = z[cc], t = tr[cc];
        part += fmaxf(x, 0.f) - x * t + log1pf(expf(-fabsf(x)));
        dz[cc] = 1.f / (1.f + expf(-x)) - t;
      }
      loss = cta_sum(part, red);
      correct = tr[am];
    } else {
      float se = 0.f;
      for (int cc = threadIdx.x; cc < n_valid; cc += blockDim.x) se += expf(z[cc] - mx);
      const float lse = mx + logf(cta_sum(se, red));
      if (mode == 1) {
        // soft targets: -(targets * log_softmax).sum(), n_correct = (softmax * targets).sum(); eps is not applied
        const float* tr = targets + static_cast<long>(r) * ld_t;
        float pl = 0.f, pt = 0.f, pc = 0.f;
        for (int cc = threadIdx.x; cc < n_valid; cc += blockDim.x) {
          const float t = tr[cc];
          pl += t * (lse - z[cc]);
          pt += t;
          pc += expf(z[cc] - lse) * t;
        }
        loss = cta_sum(pl, red);
        const float tsum = cta_sum(pt, red);
        correct = cta_sum(pc, red);
        for (int cc = threadIdx.x; cc < n_valid; cc += blockDim.x) dz[cc] = tsum * expf(z[cc] - lse) - tr[cc];
      } else {
        // hard labels: cross_entropy(label_smoothing=eps); a label outside [0, n_valid) (ignore_index) contributes nothing
        const long t = labels[r];
        const bool valid = t >= 0 && t < n_valid;
        float zs = 0.f;
        for (int cc = threadIdx.x; cc < n_valid; cc += blockDim.x) zs += z[cc];
        zs = cta_sum(zs, red);
        if (valid) {
          loss = (1.f - eps) * (lse - z[t]) + eps * (lse - zs / n_valid);
          correct = am == t ? 1.f : 0.f;
        }
        const float u = eps / n_valid;
        for (int cc = threadIdx.x; cc < n_valid; cc += blockDim.x)
          dz[cc] = valid ? expf(z[cc] - lse) - (cc == t ? 1.f - eps : 0.f) - u : 0.f;
      }
    }
    for (long cc = n_valid + threadIdx.x; cc < ld; cc += blockDim.x) dz[cc] = 0.f;
  }
  if (threadIdx.x == 0) {
    row_loss[r] = loss;
    row_correct[r] = correct;
  }
  // the last CTA to finish sums every row in a fixed order and resets the ticket
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  float la = 0.f, ca = 0.f;
  for (int i = threadIdx.x; i < rows; i += blockDim.x) { la += __ldcg(row_loss + i); ca += __ldcg(row_correct + i); }
  la = cta_sum(la, red);
  ca = cta_sum(ca, red);
  if (threadIdx.x == 0) {
    out2[0] = la;
    out2[1] = ca;
    *ticket = 0u;
  }
}

int attn_pool_fwd(const void* kv, const float* q, const uint8_t* key_pad, void* out, float* lse, int B, int T, int d,
                  cudaStream_t stream) {
  if (B <= 0 || T <= 0 || d <= 0 || d % 64 != 0) return OPB_ERR_INVALID;
  if (B > 65535) return OPB_ERR_UNSUPPORTED;
  const int H = d / 64;
  attn_pool_fwd_kernel<<<dim3(H, B), kPoolThreads, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(kv), q, key_pad,
                                                                reinterpret_cast<__nv_bfloat16*>(out), lse, T, H);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

int attn_pool_bwd(const void* kv, const float* q, const uint8_t* key_pad, const float* lse, const void* dout, void* dkv,
                  float* dq_ws, float* dq, int B, int T, int d, cudaStream_t stream) {
  if (B <= 0 || T <= 0 || d <= 0 || d % 64 != 0) return OPB_ERR_INVALID;
  if (B > 65535) return OPB_ERR_UNSUPPORTED;
  const int H = d / 64;
  attn_pool_bwd_kernel<<<dim3(H, B), kPoolThreads, 0, stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(kv), q, key_pad, lse, reinterpret_cast<const __nv_bfloat16*>(dout),
      reinterpret_cast<__nv_bfloat16*>(dkv), dq_ws, T, H);
  if (cudaGetLastError() != cudaSuccess) return OPB_ERR_CUDA;
  attn_pool_dq_kernel<<<(d + 255) / 256, 256, 0, stream>>>(dq_ws, dq, B, d);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

int classify_loss(const float* logits, long ld, int rows, int n_valid, int mode, const int64_t* labels, const float* targets,
                  long ld_t, float eps, int num_choices, float* row_loss, float* dlogits, float* row_correct, float* out2,
                  unsigned int* ticket, cudaStream_t stream) {
  if (rows <= 0 || n_valid <= 0 || ld < n_valid || mode < 0 || mode > 3) return OPB_ERR_INVALID;
  if ((mode == 0 || mode == 3) && labels == nullptr) return OPB_ERR_INVALID;
  if ((mode == 1 || mode == 2) && (targets == nullptr || ld_t < n_valid)) return OPB_ERR_INVALID;
  int grid = rows;
  if (mode == 3) {
    if (n_valid != 1 || num_choices <= 0 || rows % num_choices != 0) return OPB_ERR_INVALID;
    grid = rows / num_choices;
  }
  classify_loss_kernel<<<grid, kLossThreads, 0, stream>>>(logits, ld, grid, n_valid, mode, labels, targets, ld_t, eps, num_choices,
                                                           row_loss, dlogits, row_correct, out2, ticket);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

}  // namespace opb
