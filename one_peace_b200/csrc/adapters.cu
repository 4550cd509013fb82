// Modality-adapter kernels that are not GEMMs: coalesced, 16-byte-vectorised HBM kernels.
//   text_embed          adapter/text.py:125-129,144-146,153 + transformer_encoder.py:139-142 (pad rows zeroed)
//   image_patchify4     im2col for the 4x4/stride-4 stem conv (adapter/image.py:67) -> bf16 A operand
//   cls_row_init        x[b,0,:] = cls + pos[0]   (image.py:239-240,253 / audio.py:195-197)
//   relpos_bias_build   table[bucket[:S,:S]] -> (H,S,S_pad) fp32 (text.py:84-91, image.py:164-171), built
//                       ONCE per forward for the whole batch instead of the reference's (B,H,S,S)
//   audio_frame10       im2col for the first wav2vec conv (k=10, s=5, C_in=1; audio.py:276) -> bf16 [rows,16]
//   l2_normalize_rows   F.normalize(dim=1) (one_peace_retrieval.py:116)
#include "common.cuh"
#include "ops.h"

namespace opb {

template <typename TTab>
__global__ void text_embed_kernel(const int64_t* __restrict__ tokens, const TTab* __restrict__ table,
                                  const float* __restrict__ pos, const float* __restrict__ cls,
                                  float* __restrict__ x, uint8_t* __restrict__ pad_mask, int B, int T, int D,
                                  int pad_idx) {
  const int row = blockIdx.x;          // over B * (T + 1)
  const int S = T + 1;
  const int b = row / S, s = row % S;
  float* xo = x + static_cast<long>(row) * D;
  const float* pp = pos + static_cast<long>(s) * D;
  bool is_pad = false;
  long tok = 0;
  if (s > 0) {
    tok = tokens[static_cast<long>(b) * T + (s - 1)];
    is_pad = (tok == pad_idx);
  }
  if (threadIdx.x == 0) pad_mask[row] = is_pad ? 1 : 0;
  for (int c = threadIdx.x * 4; c < D; c += blockDim.x * 4) {
    float4 o;
    if (is_pad) {
      o = make_float4(0.f, 0.f, 0.f, 0.f);
    } else {
      const float4 p4 = *reinterpret_cast<const float4*>(pp + c);
      float e0, e1, e2, e3;
      if (s == 0) {
        const float4 c4 = *reinterpret_cast<const float4*>(cls + c);
        e0 = c4.x; e1 = c4.y; e2 = c4.z; e3 = c4.w;
      } else if constexpr (sizeof(TTab) == 4) {
        const float4 t4 = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(table) + tok * D + c);
        e0 = t4.x; e1 = t4.y; e2 = t4.z; e3 = t4.w;
      } else {
        const uint2 u = *reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(table) + tok * D + c);
        const float2 a = unpack_bf16x2(u.x), bq = unpack_bf16x2(u.y);
        e0 = a.x; e1 = a.y; e2 = bq.x; e3 = bq.y;
      }
      o = make_float4(e0 + p4.x, e1 + p4.y, e2 + p4.z, e3 + p4.w);
    }
    *reinterpret_cast<float4*>(xo + c) = o;
  }
}

int text_embed(const int64_t* tokens, const void* table, int table_dtype, const float* pos, const float* cls,
               float* x, uint8_t* pad_mask, int B, int T, int D, int pad_idx, cudaStream_t stream) {
  if (B <= 0 || T <= 0 || D % 4 != 0) return OPB_ERR_INVALID;
  const int rows = B * (T + 1);
  int threads = D / 4;
  threads = threads > 256 ? 256 : ((threads + 31) / 32) * 32;
  if (table_dtype == 0)
    text_embed_kernel<float><<<rows, threads, 0, stream>>>(tokens, reinterpret_cast<const float*>(table), pos, cls,
                                                           x, pad_mask, B, T, D, pad_idx);
  else
    text_embed_kernel<__nv_bfloat16><<<rows, threads, 0, stream>>>(
        tokens, reinterpret_cast<const __nv_bfloat16*>(table), pos, cls, x, pad_mask, B, T, D, pad_idx);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

// out[(b, oy, ox), (c, ky, kx)] = img[b, c, 4*oy + ky, 4*ox + kx]; one thread = one (row, c) = 16 values
template <typename TImg>
__global__ void image_patchify4_kernel(const TImg* __restrict__ img, __nv_bfloat16* __restrict__ out, int B, int R) {
  const int G = R / 4;
  const long total = static_cast<long>(B) * G * G * 3;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long>(gridDim.x) * blockDim.x) {
    // consecutive threads -> consecutive ox (coalesced 16-byte reads along an image row)
    const int ox = i % G;
    const int c = (i / G) % 3;
    const int oy = (i / (3L * G)) % G;
    const int b = i / (3L * G * G);
    const TImg* src = img + ((static_cast<long>(b) * 3 + c) * R + 4 * oy) * R + 4 * ox;
    uint32_t packed[8];
#pragma unroll
    for (int ky = 0; ky < 4; ++ky) {
      float v0, v1, v2, v3;
      if constexpr (sizeof(TImg) == 4) {
        const float4 f = *reinterpret_cast<const float4*>(src + static_cast<long>(ky) * R);
        v0 = f.x; v1 = f.y; v2 = f.z; v3 = f.w;
      } else {
        const uint2 u = *reinterpret_cast<const uint2*>(src + static_cast<long>(ky) * R);
        const float2 a = unpack_bf16x2(u.x), bq = unpack_bf16x2(u.y);
        v0 = a.x; v1 = a.y; v2 = bq.x; v3 = bq.y;
      }
      packed[2 * ky] = pack_bf16x2(v0, v1);
      packed[2 * ky + 1] = pack_bf16x2(v2, v3);
    }
    __nv_bfloat16* dst = out + ((static_cast<long>(b) * G + oy) * G + ox) * 48 + c * 16;
    *reinterpret_cast<uint4*>(dst) = make_uint4(packed[0], packed[1], packed[2], packed[3]);
    *reinterpret_cast<uint4*>(dst + 8) = make_uint4(packed[4], packed[5], packed[6], packed[7]);
  }
}

int image_patchify4(const void* img, int img_dtype, void* out, int B, int R, cudaStream_t stream) {
  if (B <= 0 || R <= 0 || R % 16 != 0) return OPB_ERR_INVALID;
  const long total = static_cast<long>(B) * (R / 4) * (R / 4) * 3;
  const int threads = 256;
  long blocks = (total + threads - 1) / threads;
  if (blocks > 132L * 32) blocks = 132L * 32;
  if (img_dtype == 0)
    image_patchify4_kernel<float><<<static_cast<unsigned>(blocks), threads, 0, stream>>>(
        reinterpret_cast<const float*>(img), reinterpret_cast<__nv_bfloat16*>(out), B, R);
  else
    image_patchify4_kernel<__nv_bfloat16><<<static_cast<unsigned>(blocks), threads, 0, stream>>>(
        reinterpret_cast<const __nv_bfloat16*>(img), reinterpret_cast<__nv_bfloat16*>(out), B, R);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

__global__ void cls_row_init_kernel(const float* __restrict__ cls, const float* __restrict__ pos0,
                                    float* __restrict__ x, long batch_stride, int D) {
  float* xo = x + blockIdx.x * batch_stride;
  for (int c = threadIdx.x * 4; c < D; c += blockDim.x * 4) {
    const float4 a = *reinterpret_cast<const float4*>(cls + c);
    const float4 p = *reinterpret_cast<const float4*>(pos0 + c);
    *reinterpret_cast<float4*>(xo + c) = make_float4(a.x + p.x, a.y + p.y, a.z + p.z, a.w + p.w);
  }
}

int cls_row_init(const float* cls, const float* pos0, float* x, long batch_stride, int B, int D,
                 cudaStream_t stream) {
  if (B <= 0 || D % 4 != 0) return OPB_ERR_INVALID;
  cls_row_init_kernel<<<B, 128, 0, stream>>>(cls, pos0, x, batch_stride, D);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

// bias[h, i, j] = table[bucket[i * ld_bucket + j], h]  for i, j < S;  columns S..s_pad-1 are zero
__global__ void relpos_bias_kernel(const float* __restrict__ table, const int64_t* __restrict__ bucket,
                                   float* __restrict__ bias, int S, int s_pad, int H, long ld_bucket) {
  const int i = blockIdx.x;
  for (int j = threadIdx.x; j < s_pad; j += blockDim.x) {
    const bool ok = j < S;
    const long bk = ok ? bucket[static_cast<long>(i) * ld_bucket + j] : 0;
    for (int h = 0; h < H; ++h)
      bias[(static_cast<long>(h) * S + i) * s_pad + j] = ok ? table[bk * H + h] : 0.f;
  }
}

int relpos_bias_build(const float* table, const int64_t* bucket, float* bias, int S, int s_pad, int H,
                      long ld_bucket, cudaStream_t stream) {
  if (S <= 0 || s_pad < S || H <= 0) return OPB_ERR_INVALID;
  relpos_bias_kernel<<<S, 128, 0, stream>>>(table, bucket, bias, S, s_pad, H, ld_bucket);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

// out[(b, t), j] = wav[b, 5 t + j] for j < 10 and 5 t + j < n_samples, zero elsewhere (j in 10..15, samples past the clip
// end), for every t < pitch: the slack rows t >= frames hold the clip's partial last frames, which only the slack rows of
// later layers read.
template <typename TWav>
__global__ void audio_frame10_kernel(const TWav* __restrict__ wav, __nv_bfloat16* __restrict__ out, int B,
                                     long n_samples, long pitch) {
  const long total = static_cast<long>(B) * pitch;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long>(gridDim.x) * blockDim.x) {
    const long t = i % pitch;
    const long b = i / pitch;
    const TWav* src = wav + b * n_samples;
    float v[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const long idx = 5 * t + j;
      float f = 0.f;
      if (j < 10 && idx < n_samples) {
        if constexpr (sizeof(TWav) == 4) f = src[idx];
        else f = __bfloat162float(src[idx]);
      }
      v[j] = f;
    }
    uint4 o0, o1;
    o0.x = pack_bf16x2(v[0], v[1]); o0.y = pack_bf16x2(v[2], v[3]);
    o0.z = pack_bf16x2(v[4], v[5]); o0.w = pack_bf16x2(v[6], v[7]);
    o1.x = pack_bf16x2(v[8], v[9]); o1.y = pack_bf16x2(v[10], v[11]);
    o1.z = pack_bf16x2(v[12], v[13]); o1.w = pack_bf16x2(v[14], v[15]);
    uint4* dst = reinterpret_cast<uint4*>(out + i * 16);
    dst[0] = o0;
    dst[1] = o1;
  }
}

int audio_frame10(const void* wav, int wav_dtype, void* out, int B, long n_samples, long pitch,
                  cudaStream_t stream) {
  if (B <= 0 || n_samples < 10 || pitch <= 0) return OPB_ERR_INVALID;
  const long total = static_cast<long>(B) * pitch;
  long blocks = (total + 255) / 256;
  if (blocks > 132L * 16) blocks = 132L * 16;
  if (wav_dtype == 0)
    audio_frame10_kernel<float><<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
        reinterpret_cast<const float*>(wav), reinterpret_cast<__nv_bfloat16*>(out), B, n_samples, pitch);
  else
    audio_frame10_kernel<__nv_bfloat16><<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
        reinterpret_cast<const __nv_bfloat16*>(wav), reinterpret_cast<__nv_bfloat16*>(out), B, n_samples, pitch);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

// y = x / max(||x||_2, 1e-12) per row; fp32 in, fp32 out and (optionally) a bf16 copy for the InfoNCE GEMM
__global__ void l2_normalize_kernel(const float* __restrict__ x, long ldx, float* __restrict__ y,
                                    __nv_bfloat16* __restrict__ y16, int D) {
  __shared__ float red[8];
  const float* xi = x + blockIdx.x * ldx;
  float ss = 0.f;
  for (int c = threadIdx.x; c < D; c += blockDim.x) ss += xi[c] * xi[c];
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
  for (int i = 0; i < (blockDim.x + 31) / 32; ++i) tot += red[i];
  const float inv = 1.f / fmaxf(sqrtf(tot), 1e-12f);
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    const float v = xi[c] * inv;
    y[static_cast<long>(blockIdx.x) * D + c] = v;
    if (y16 != nullptr) y16[static_cast<long>(blockIdx.x) * D + c] = __float2bfloat16(v);
  }
}

int l2_normalize_rows(const float* x, long ldx, float* y, void* y_bf16, int rows, int D, cudaStream_t stream) {
  if (rows <= 0 || D <= 0) return OPB_ERR_INVALID;
  l2_normalize_kernel<<<rows, 256, 0, stream>>>(x, ldx, y, reinterpret_cast<__nv_bfloat16*>(y_bf16), D);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

// Lays an fp32 feature sequence out as the bf16 operand of the grouped positional conv (audio.py:57-80):
// out[b, halo + t, g, :group_in] = x[b*x_period + x_row_shift + t, g*group_in : (g+1)*group_in], zero elsewhere
// in the written rows' padding columns; halo rows are left untouched (the buffer is zero-initialised once).
__global__ void pack_group_halo_kernel(const float* __restrict__ x, long ldx, __nv_bfloat16* __restrict__ out, int T,
                                       int x_period, int x_row_shift, int out_period, int halo, int dim,
                                       int group_in, int group_out) {
  const int b = blockIdx.x / T, t = blockIdx.x % T;
  const float* xi = x + (static_cast<long>(b) * x_period + x_row_shift + t) * ldx;
  const int groups = dim / group_in;
  __nv_bfloat16* o = out + (static_cast<long>(b) * out_period + halo + t) * groups * group_out;
  for (int c = threadIdx.x * 8; c < groups * group_out; c += blockDim.x * 8) {
    const int g = c / group_out, ci = c % group_out;
    uint4 u = make_uint4(0, 0, 0, 0);
    if (ci < group_in) {
      const float4 a = *reinterpret_cast<const float4*>(xi + g * group_in + ci);
      const float4 bq = *reinterpret_cast<const float4*>(xi + g * group_in + ci + 4);
      u.x = pack_bf16x2(a.x, a.y); u.y = pack_bf16x2(a.z, a.w);
      u.z = pack_bf16x2(bq.x, bq.y); u.w = pack_bf16x2(bq.z, bq.w);
    }
    *reinterpret_cast<uint4*>(o + c) = u;
  }
}

int pack_group_halo(const float* x, long ldx, void* out, int B, int T, int x_period, int x_row_shift, int out_period,
                    int halo, int dim, int group_in, int group_out, cudaStream_t stream) {
  if (B <= 0 || T <= 0 || group_in % 8 != 0 || group_out % 8 != 0 || dim % group_in != 0 || group_out < group_in)
    return OPB_ERR_INVALID;
  pack_group_halo_kernel<<<B * T, 256, 0, stream>>>(x, ldx, reinterpret_cast<__nv_bfloat16*>(out), T, x_period,
                                                    x_row_shift, out_period, halo, dim, group_in, group_out);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

// x[row, :] = 0 where pad_mask[row] != 0   (transformer_encoder.py:139-142)
__global__ void zero_padded_rows_kernel(float* __restrict__ x, const uint8_t* __restrict__ pad, int D) {
  if (pad[blockIdx.x] == 0) return;
  float* xo = x + static_cast<long>(blockIdx.x) * D;
  for (int c = threadIdx.x * 4; c < D; c += blockDim.x * 4)
    *reinterpret_cast<float4*>(xo + c) = make_float4(0.f, 0.f, 0.f, 0.f);
}

int zero_padded_rows(float* x, const uint8_t* pad_mask, int rows, int D, cudaStream_t stream) {
  if (rows <= 0 || D % 4 != 0) return OPB_ERR_INVALID;
  zero_padded_rows_kernel<<<rows, 128, 0, stream>>>(x, pad_mask, D);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

}  // namespace opb
