// Multi-scale deformable attention (one_peace_vision/seg/ops, MSDeformAttn) for D = 32 channels per head, forward and
// adjoint, with the soft-max and the sampling-location arithmetic the reference module does in torch fused in.
//
// Layout: value bf16 [N * S_in, H * 32] (the value_proj output; level l of sample n owns rows n * S_in + start_l + y * W_l
// + x); proj fp32 [N * Lq, 3 * H * L * P] = [offsets (h, l, p, xy) | logits (h, l * P + p)]; ref fp32 [N * Lq, L_ref, 2]
// (x, y) in [0, 1], L_ref = 1 broadcast over the levels; out bf16 [N * Lq, H * 32].
//
// One warp per (sample, query, head).  Lane j < L * P sets up point j: its soft-max weight a_j (fp32, over all L * P
// logits of the head), loc = ref + off / (W_l, H_l) and the pixel coordinate loc * W_l - 0.5 (align_corners = False).
// Eight groups of four lanes then take the points in turn; lane (g, c) reads 8 channels (16 bytes) of each of the four
// bilinear taps, so one tap row of a head (64 bytes) is one coalesced group load.  Taps outside the level read as zero.
// Each group sums its points in order and the eight group sums are added by a fixed shuffle tree: there are no atomics in
// the forward and repeated launches are bit-identical.
//
// The adjoint recomputes the same taps.  d_value gets a_j * w_tap * d_out scattered with fp32 float4 atomics (its repeats
// differ in the last bits).  The per-point sums over the 32 channels (dA_j and the two derivatives of the sample with
// respect to its pixel coordinates) are reduced inside the group by a fixed shuffle order, so d_proj has no atomics and is
// bit-identical across repeats.
#include "common.cuh"
#include "ops.h"

namespace opb {

// Level shapes and start rows, a kernel parameter: __grid_constant__ lets the kernels index it in parameter space.
struct MsdaLevels {
  int h[kMsdaMaxL];
  int w[kMsdaMaxL];
  int start[kMsdaMaxL];
};

namespace {

constexpr int kD = 32;
constexpr int kWarpsPerCta = 8;

OPB_DEVICE void load8(float (&v)[8], const __nv_bfloat16* p) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const __nv_bfloat162* b = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = __bfloat1622float2(b[i]);
    v[2 * i] = f.x;
    v[2 * i + 1] = f.y;
  }
}

// Point set-up of lane j < L * P of head h in query row `row`: the soft-max weight and the pixel coordinates (x, y).
struct Point {
  float a, x, y;
};
OPB_DEVICE Point point_setup(const float* __restrict__ proj, const float* __restrict__ ref, long row, int h, int H, int L,
                             int P, int L_ref, const MsdaLevels& lv, int lane) {
  const int LP = L * P;
  const float* pr = proj + row * (3L * H * LP);
  float logit = -INFINITY, x = 0.f, y = 0.f;
  if (lane < LP) {
    const int l = lane / P;
    const float2 off = make_float2(pr[2 * (h * LP + lane)], pr[2 * (h * LP + lane) + 1]);   // rows are 4-byte aligned
    logit = pr[2 * H * LP + h * LP + lane];
    const float2 rp = *reinterpret_cast<const float2*>(ref + 2 * (row * L_ref + (L_ref == 1 ? 0 : l)));
    const float W = static_cast<float>(lv.w[l]), Hh = static_cast<float>(lv.h[l]);
    // the reference's order: loc = ref + off / normaliser (torch), then loc * W - 0.5 (ms_deform_im2col_cuda.cuh)
    x = __fsub_rn(__fmul_rn(__fadd_rn(rp.x, __fdiv_rn(off.x, W)), W), 0.5f);
    y = __fsub_rn(__fmul_rn(__fadd_rn(rp.y, __fdiv_rn(off.y, Hh)), Hh), 0.5f);
  }
  const float m = warp_max(logit);
  const float e = lane < LP ? expf(logit - m) : 0.f;
  const float s = warp_sum(e);
  return {e / s, x, y};
}

// The four taps of a sample at pixel coordinates (x, y) inside (-1, W) x (-1, H): corner weights and row offsets
// (-1 for a tap outside the level).
struct Taps {
  float w[4];
  int r[4];
  float lx, ly, hx, hy;
};
OPB_DEVICE Taps taps(float x, float y, int Hl, int Wl) {
  Taps t;
  const int y0 = static_cast<int>(floorf(y)), x0 = static_cast<int>(floorf(x));
  const int y1 = y0 + 1, x1 = x0 + 1;
  t.ly = y - static_cast<float>(y0);
  t.lx = x - static_cast<float>(x0);
  t.hy = 1.f - t.ly;
  t.hx = 1.f - t.lx;
  t.w[0] = t.hy * t.hx;
  t.w[1] = t.hy * t.lx;
  t.w[2] = t.ly * t.hx;
  t.w[3] = t.ly * t.lx;
  t.r[0] = (y0 >= 0 && x0 >= 0) ? y0 * Wl + x0 : -1;
  t.r[1] = (y0 >= 0 && x1 <= Wl - 1) ? y0 * Wl + x1 : -1;
  t.r[2] = (y1 <= Hl - 1 && x0 >= 0) ? y1 * Wl + x0 : -1;
  t.r[3] = (y1 <= Hl - 1 && x1 <= Wl - 1) ? y1 * Wl + x1 : -1;
  return t;
}

OPB_DEVICE bool inside(float x, float y, int Hl, int Wl) {
  return y > -1.f && x > -1.f && y < static_cast<float>(Hl) && x < static_cast<float>(Wl);
}

}  // namespace

__global__ void __launch_bounds__(32 * kWarpsPerCta)
ms_deform_attn_fwd_kernel(const __nv_bfloat16* __restrict__ value, const float* __restrict__ proj, const float* __restrict__ ref,
                          __nv_bfloat16* __restrict__ out, long units, int S_in, int Lq, int H, int L, int P, int L_ref,
                          const __grid_constant__ MsdaLevels lv) {
  const int lane = threadIdx.x & 31;
  const long unit = static_cast<long>(blockIdx.x) * kWarpsPerCta + (threadIdx.x >> 5);
  if (unit >= units) return;                                 // warp-uniform; no CTA-wide barrier follows
  const int h = static_cast<int>(unit % H);
  const long row = unit / H;
  const long n = row / Lq;
  const int LP = L * P;
  const long HD = static_cast<long>(H) * kD;
  const Point pt = point_setup(proj, ref, row, h, H, L, P, L_ref, lv, lane);
  const int g = lane >> 2, c8 = (lane & 3) * 8;
  const __nv_bfloat16* vbase = value + n * S_in * HD + h * kD + c8;
  float acc[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) acc[c] = 0.f;
  for (int j0 = 0; j0 < LP; j0 += 8) {
    const int j = j0 + g;
    const float a = __shfl_sync(0xffffffffu, pt.a, j & 31);
    const float x = __shfl_sync(0xffffffffu, pt.x, j & 31);
    const float y = __shfl_sync(0xffffffffu, pt.y, j & 31);
    if (j >= LP) continue;
    const int l = j / P, Hl = lv.h[l], Wl = lv.w[l];
    if (!inside(x, y, Hl, Wl)) continue;
    const Taps t = taps(x, y, Hl, Wl);
    const __nv_bfloat16* lbase = vbase + lv.start[l] * HD;
    float v[4][8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (t.r[k] >= 0) {
        load8(v[k], lbase + t.r[k] * HD);
      } else {
#pragma unroll
        for (int c = 0; c < 8; ++c) v[k][c] = 0.f;
      }
    }
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const float s = t.w[0] * v[0][c] + t.w[1] * v[1][c] + t.w[2] * v[2][c] + t.w[3] * v[3][c];
      acc[c] += a * s;
    }
  }
#pragma unroll
  for (int o = 4; o < 32; o <<= 1) {
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], o);
  }
  if (g == 0) {
    uint4 u;
    __nv_bfloat162* b = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) b[i] = __floats2bfloat162_rn(acc[2 * i], acc[2 * i + 1]);
    *reinterpret_cast<uint4*>(out + row * HD + h * kD + c8) = u;
  }
}

__global__ void __launch_bounds__(32 * kWarpsPerCta)
ms_deform_attn_bwd_kernel(const __nv_bfloat16* __restrict__ value, const float* __restrict__ proj, const float* __restrict__ ref,
                          const __nv_bfloat16* __restrict__ d_out, float* __restrict__ d_value, float* __restrict__ d_proj,
                          long units, int S_in, int Lq, int H, int L, int P, int L_ref,
                          const __grid_constant__ MsdaLevels lv) {
  const int lane = threadIdx.x & 31;
  const long unit = static_cast<long>(blockIdx.x) * kWarpsPerCta + (threadIdx.x >> 5);
  if (unit >= units) return;
  const int h = static_cast<int>(unit % H);
  const long row = unit / H;
  const long n = row / Lq;
  const int LP = L * P;
  const long HD = static_cast<long>(H) * kD;
  const Point pt = point_setup(proj, ref, row, h, H, L, P, L_ref, lv, lane);
  const int g = lane >> 2, c8 = (lane & 3) * 8;
  const long vofs = n * S_in * HD + h * kD + c8;
  float dout[8];
  load8(dout, d_out + row * HD + h * kD + c8);
  float dA = 0.f, dX = 0.f, dY = 0.f;                       // lane j's point: sums over the 32 channels
  for (int j0 = 0; j0 < LP; j0 += 8) {
    const int j = j0 + g;
    const float a = __shfl_sync(0xffffffffu, pt.a, j & 31);
    const float x = __shfl_sync(0xffffffffu, pt.x, j & 31);
    const float y = __shfl_sync(0xffffffffu, pt.y, j & 31);
    float gA = 0.f, gX = 0.f, gY = 0.f;
    if (j < LP) {
      const int l = j / P, Hl = lv.h[l], Wl = lv.w[l];
      if (inside(x, y, Hl, Wl)) {
        const Taps t = taps(x, y, Hl, Wl);
        const long lofs = vofs + lv.start[l] * HD;
        float v[4][8];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          if (t.r[k] >= 0) {
            load8(v[k], value + lofs + t.r[k] * HD);
          } else {
#pragma unroll
            for (int c = 0; c < 8; ++c) v[k][c] = 0.f;
          }
        }
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const float s = t.w[0] * v[0][c] + t.w[1] * v[1][c] + t.w[2] * v[2][c] + t.w[3] * v[3][c];
          gA += dout[c] * s;
          gX += dout[c] * (t.hy * (v[1][c] - v[0][c]) + t.ly * (v[3][c] - v[2][c]));
          gY += dout[c] * (t.hx * (v[2][c] - v[0][c]) + t.lx * (v[3][c] - v[1][c]));
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          if (t.r[k] < 0) continue;
          const float s = a * t.w[k];
          float4* dst = reinterpret_cast<float4*>(d_value + lofs + t.r[k] * HD);
          atomicAdd(dst, make_float4(s * dout[0], s * dout[1], s * dout[2], s * dout[3]));
          atomicAdd(dst + 1, make_float4(s * dout[4], s * dout[5], s * dout[6], s * dout[7]));
        }
      }
    }
#pragma unroll
    for (int o = 1; o < 4; o <<= 1) {
      gA += __shfl_xor_sync(0xffffffffu, gA, o);
      gX += __shfl_xor_sync(0xffffffffu, gX, o);
      gY += __shfl_xor_sync(0xffffffffu, gY, o);
    }
    // lane j0 + i takes the sums of group i
    const int src = (lane & 7) * 4;
    gA = __shfl_sync(0xffffffffu, gA, src);
    gX = __shfl_sync(0xffffffffu, gX, src);
    gY = __shfl_sync(0xffffffffu, gY, src);
    if ((lane >> 3) == (j0 >> 3)) {
      dA = gA;
      dX = gX;
      dY = gY;
    }
  }
  const float sad = warp_sum(lane < LP ? pt.a * dA : 0.f);
  if (lane < LP) {
    const int l = lane / P;
    const float W = static_cast<float>(lv.w[l]), Hh = static_cast<float>(lv.h[l]);
    float* dp = d_proj + row * (3L * H * LP);
    // d_loc = (W, H) * a * d sample / d pixel coordinate, then d_off = d_loc / (W, H)
    const float dlx = W * (pt.a * dX), dly = Hh * (pt.a * dY);
    dp[2 * (h * LP + lane)] = dlx / W;
    dp[2 * (h * LP + lane) + 1] = dly / Hh;
    dp[2 * H * LP + h * LP + lane] = pt.a * (dA - sad);
  }
}

namespace {

bool aligned16(const void* p) { return p != nullptr && (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

int check_args(int N, int S_in, int Lq, int H, int D, int L, int P, int L_ref, const int* level_hw, const int* level_start,
               MsdaLevels* lv, long* units) {
  if (N <= 0 || S_in <= 0 || Lq <= 0 || H <= 0 || D != kD) return OPB_ERR_INVALID;
  if (L < 1 || L > kMsdaMaxL || P < 1 || P > kMsdaMaxP || (L_ref != 1 && L_ref != L)) return OPB_ERR_INVALID;
  if (level_hw == nullptr || level_start == nullptr) return OPB_ERR_INVALID;
  *lv = MsdaLevels{};
  for (int l = 0; l < L; ++l) {
    const int hl = level_hw[2 * l], wl = level_hw[2 * l + 1], st = level_start[l];
    if (hl <= 0 || wl <= 0 || st < 0 || static_cast<long>(st) + static_cast<long>(hl) * wl > S_in) return OPB_ERR_INVALID;
    lv->h[l] = hl;
    lv->w[l] = wl;
    lv->start[l] = st;
  }
  *units = static_cast<long>(N) * Lq * H;
  if ((*units + kWarpsPerCta - 1) / kWarpsPerCta > 0x7fffffffL) return OPB_ERR_INVALID;
  return OPB_OK;
}

}  // namespace

int ms_deform_attn_fwd(const void* value, const float* proj, const float* ref, void* out, int N, int S_in, int Lq, int H,
                       int D, int L, int P, int L_ref, const int* level_hw, const int* level_start, cudaStream_t stream) {
  if (!aligned16(value) || !aligned16(proj) || !aligned16(ref) || !aligned16(out)) return OPB_ERR_INVALID;
  MsdaLevels lv;
  long units = 0;
  const int st = check_args(N, S_in, Lq, H, D, L, P, L_ref, level_hw, level_start, &lv, &units);
  if (st != OPB_OK) return st;
  const unsigned grid = static_cast<unsigned>((units + kWarpsPerCta - 1) / kWarpsPerCta);
  ms_deform_attn_fwd_kernel<<<grid, 32 * kWarpsPerCta, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(value), proj, ref, static_cast<__nv_bfloat16*>(out), units, S_in, Lq, H, L, P, L_ref,
      lv);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

int ms_deform_attn_bwd(const void* value, const float* proj, const float* ref, const void* d_out, float* d_value,
                       float* d_proj, int N, int S_in, int Lq, int H, int D, int L, int P, int L_ref, const int* level_hw,
                       const int* level_start, cudaStream_t stream) {
  if (!aligned16(value) || !aligned16(proj) || !aligned16(ref) || !aligned16(d_out) || !aligned16(d_value) ||
      !aligned16(d_proj))
    return OPB_ERR_INVALID;
  MsdaLevels lv;
  long units = 0;
  const int st = check_args(N, S_in, Lq, H, D, L, P, L_ref, level_hw, level_start, &lv, &units);
  if (st != OPB_OK) return st;
  const unsigned grid = static_cast<unsigned>((units + kWarpsPerCta - 1) / kWarpsPerCta);
  ms_deform_attn_bwd_kernel<<<grid, 32 * kWarpsPerCta, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(value), proj, ref, static_cast<const __nv_bfloat16*>(d_out), d_value, d_proj, units,
      S_in, Lq, H, L, P, L_ref, lv);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

}  // namespace opb
