// Semantic segmentation backbone (one_peace_vision/seg, OnePeaceAdapter): the two steps no other kernel of the project does.
//
// opb_seg_dwconv_gelu: ConvFFN's depthwise 3x3 conv + bias + exact GELU (adapter_modules.py:47-84) over the token rows of
// c, where each sample's rows hold up to four levels back to back, each a row-major H_l x W_l grid.  Each level is
// convolved on its own grid with zero padding at its border.  One thread per (token, 8 channels): nine 16-byte tap loads,
// fp32 products summed in tap order (ky, kx row-major), then the bias, then gelu_erf.  One write per output element.
//
// opb_seg_out_map: one output map of onepeace_adapter.py:114-134,
//   f[b, c, y, x] = scale[c] * (extra + c_l[b, y W + x, c] + up(x_l)[b, c, y, x]) + shift[c]
// where extra = convT(c2) read with the pixel-shuffle index (level 1 only), up the bilinear resize (align_corners = False)
// of the ViT's gw x gw patch grid, and (scale, shift) the folded eval BatchNorm.  A CTA takes 32 consecutive pixels of one
// sample and 32 channels: it reads the token-major inputs along channels, transposes through shared memory and writes
// 32 consecutive pixels of each channel (128-byte lines) of the channel-major map.
#include "common.cuh"
#include "ops.h"

namespace opb {

struct SegLevels {
  int h[kSegMaxL];
  int w[kSegMaxL];
  int start[kSegMaxL];
  int n_levels;
  int tokens;  // rows per sample
};

namespace {

constexpr int kDwThreads = 256;

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

// x, y bf16 [B * tokens, C]; w fp32 [9, C] (tap ky * 3 + kx); bias fp32 [C].
__global__ void __launch_bounds__(kDwThreads) seg_dwconv_gelu_kernel(const __nv_bfloat16* __restrict__ x,
                                                                     const float* __restrict__ w,
                                                                     const float* __restrict__ bias,
                                                                     __nv_bfloat16* __restrict__ y, long units, int C,
                                                                     const __grid_constant__ SegLevels lv) {
  const long u = static_cast<long>(blockIdx.x) * kDwThreads + threadIdx.x;
  if (u >= units) return;
  const int cg = C / 8;
  const int c0 = static_cast<int>(u % cg) * 8;
  const long row = u / cg;
  const int t = static_cast<int>(row % lv.tokens);
  const long base = row - t;  // first row of the sample
  int l = 0;
  while (l + 1 < lv.n_levels && t >= lv.start[l + 1]) ++l;
  const int p = t - lv.start[l], W = lv.w[l], H = lv.h[l];
  const int py = p / W, px = p % W;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
#pragma unroll
  for (int ky = 0; ky < 3; ++ky) {
    const int yy = py + ky - 1;
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const int xx = px + kx - 1;
      if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;
      float v[8];
      load8(v, x + (base + lv.start[l] + static_cast<long>(yy) * W + xx) * C + c0);
      const float4 w0 = *reinterpret_cast<const float4*>(w + (ky * 3 + kx) * C + c0);
      const float4 w1 = *reinterpret_cast<const float4*>(w + (ky * 3 + kx) * C + c0 + 4);
      acc[0] = fmaf(v[0], w0.x, acc[0]);
      acc[1] = fmaf(v[1], w0.y, acc[1]);
      acc[2] = fmaf(v[2], w0.z, acc[2]);
      acc[3] = fmaf(v[3], w0.w, acc[3]);
      acc[4] = fmaf(v[4], w1.x, acc[4]);
      acc[5] = fmaf(v[5], w1.y, acc[5]);
      acc[6] = fmaf(v[6], w1.z, acc[6]);
      acc[7] = fmaf(v[7], w1.w, acc[7]);
    }
  }
  const float4 b0 = *reinterpret_cast<const float4*>(bias + c0);
  const float4 b1 = *reinterpret_cast<const float4*>(bias + c0 + 4);
  const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
  uint4 o;
  uint32_t* op = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
  for (int i = 0; i < 4; ++i) op[i] = pack_bf16x2(gelu_erf(acc[2 * i] + bb[2 * i]), gelu_erf(acc[2 * i + 1] + bb[2 * i + 1]));
  *reinterpret_cast<uint4*>(y + row * C + c0) = o;
}

constexpr int kMapTile = 32;
constexpr int kMapRows = 8;

// Source index of output coordinate `o` of a bilinear resize from n_in to n_out samples (align_corners = False):
// torch's area_pixel_compute_source_index with scale n_in / n_out, clamped at 0.
OPB_DEVICE void lin_src(int o, int n_in, int n_out, int& i0, int& i1, float& f) {
  const float s = fmaxf((static_cast<float>(o) + 0.5f) * (static_cast<float>(n_in) / static_cast<float>(n_out)) - 0.5f, 0.f);
  i0 = min(static_cast<int>(s), n_in - 1);
  i1 = min(i0 + 1, n_in - 1);
  f = s - static_cast<float>(i0);
}

__global__ void __launch_bounds__(kMapTile * kMapRows) seg_out_map_kernel(
    const float* __restrict__ c, long c_sample_rows, long c_row0, const float* __restrict__ xv, long x_sample_rows,
    long x_row0, int gw, const float* __restrict__ extra, const float* __restrict__ scale, const float* __restrict__ shift,
    float* __restrict__ out, int C, int Hl, int Wl) {
  __shared__ float tile[kMapTile][kMapTile + 1];
  const int HW = Hl * Wl;
  const int p0 = blockIdx.x * kMapTile, c0 = blockIdx.y * kMapTile, b = blockIdx.z;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int ch = c0 + tx;
  const float sc = scale[ch], sh = shift[ch];
  for (int i = ty; i < kMapTile; i += kMapRows) {
    const int p = p0 + i;
    if (p >= HW) break;
    const int py = p / Wl, px = p % Wl;
    float v = c[(b * c_sample_rows + c_row0 + p) * static_cast<long>(C) + ch];
    if (extra != nullptr) {  // convT(c2): [(b, y / 2, x / 2), (dy, dx, c)]
      const long r = (static_cast<long>(b) * (Hl / 2) + py / 2) * (Wl / 2) + px / 2;
      v = extra[r * 4 * C + ((py & 1) * 2 + (px & 1)) * C + ch] + v;
    }
    int y0, y1, x0, x1;
    float fy, fx;
    lin_src(py, gw, Hl, y0, y1, fy);
    lin_src(px, gw, Wl, x0, x1, fx);
    const float* xb = xv + (b * x_sample_rows + x_row0) * static_cast<long>(C) + ch;
    const float a00 = xb[(static_cast<long>(y0) * gw + x0) * C], a01 = xb[(static_cast<long>(y0) * gw + x1) * C];
    const float a10 = xb[(static_cast<long>(y1) * gw + x0) * C], a11 = xb[(static_cast<long>(y1) * gw + x1) * C];
    const float up = (1.f - fy) * ((1.f - fx) * a00 + fx * a01) + fy * ((1.f - fx) * a10 + fx * a11);
    tile[i][tx] = fmaf(v + up, sc, sh);
  }
  __syncthreads();
  const int p = p0 + tx;
  if (p >= HW) return;
  for (int j = ty; j < kMapTile; j += kMapRows)
    out[(static_cast<long>(b) * C + c0 + j) * HW + p] = tile[tx][j];
}

bool aligned16(const void* p) { return p != nullptr && (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

int seg_dwconv_gelu(const void* x, const float* w, const float* bias, void* y, int B, int C, int n_levels,
                    const int* level_hw, cudaStream_t stream) {
  if (!aligned16(x) || !aligned16(w) || !aligned16(bias) || !aligned16(y) || level_hw == nullptr) return OPB_ERR_INVALID;
  if (B <= 0 || C <= 0 || C % 8 != 0 || n_levels < 1 || n_levels > kSegMaxL) return OPB_ERR_INVALID;
  SegLevels lv{};
  long tokens = 0;
  for (int l = 0; l < n_levels; ++l) {
    const int h = level_hw[2 * l], wl = level_hw[2 * l + 1];
    if (h <= 0 || wl <= 0) return OPB_ERR_INVALID;
    lv.h[l] = h;
    lv.w[l] = wl;
    lv.start[l] = static_cast<int>(tokens);
    tokens += static_cast<long>(h) * wl;
    if (tokens > 0x7fffffffL) return OPB_ERR_INVALID;
  }
  lv.n_levels = n_levels;
  lv.tokens = static_cast<int>(tokens);
  const long units = static_cast<long>(B) * tokens * (C / 8);
  const long grid = (units + kDwThreads - 1) / kDwThreads;
  if (grid > 0x7fffffffL) return OPB_ERR_INVALID;
  seg_dwconv_gelu_kernel<<<static_cast<unsigned>(grid), kDwThreads, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(x), w, bias, static_cast<__nv_bfloat16*>(y), units, C, lv);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

int seg_out_map(const float* c, long c_sample_rows, long c_row0, const float* x, long x_sample_rows, long x_row0, int gw,
                const float* extra, const float* scale, const float* shift, float* out, int B, int C, int Hl, int Wl,
                cudaStream_t stream) {
  if (c == nullptr || x == nullptr || scale == nullptr || shift == nullptr || out == nullptr) return OPB_ERR_INVALID;
  if (B <= 0 || C <= 0 || C % kMapTile != 0 || Hl <= 0 || Wl <= 0 || gw <= 0) return OPB_ERR_INVALID;
  if (c_sample_rows < c_row0 + static_cast<long>(Hl) * Wl || c_row0 < 0) return OPB_ERR_INVALID;
  if (x_sample_rows < x_row0 + static_cast<long>(gw) * gw || x_row0 < 0) return OPB_ERR_INVALID;
  if (extra != nullptr && ((Hl & 1) || (Wl & 1))) return OPB_ERR_INVALID;
  const long tiles = (static_cast<long>(Hl) * Wl + kMapTile - 1) / kMapTile;
  if (tiles > 0x7fffffffL || B > 65535 || C / kMapTile > 65535) return OPB_ERR_INVALID;
  const dim3 grid(static_cast<unsigned>(tiles), C / kMapTile, B);
  seg_out_map_kernel<<<grid, dim3(kMapTile, kMapRows), 0, stream>>>(c, c_sample_rows, c_row0, x, x_sample_rows, x_row0, gw,
                                                                    extra, scale, shift, out, C, Hl, Wl);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

}  // namespace opb
