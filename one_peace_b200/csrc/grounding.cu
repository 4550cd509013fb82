// Visual grounding (criterions/refcoco_loss.py:36-46, metrics/iou_acc.py:20-32): the L1 + GIoU box loss of refcoco_criterion
// with its gradient, and the IoU >= 0.5 hit counter of IouAcc.
//
// Box loss, per row r of p = sigmoid(logits[r, 0:4]) against the target box t = targets[r] (x0, y0, x1, y1):
//     L1     = sum_{r,j} |p_rj - t_rj| / nsentences                      (F.l1_loss(reduction='sum') / nsentences)
//     valid  = p0 < p2 and p1 < p3 (strict; selects rows, carries no gradient)
//     GIoU   = torchvision.ops.generalized_box_iou(p, t) per row: inter = prod clamp(min(p_hi, t_hi) - max(p_lo, t_lo), 0),
//              union = area_p + area_t - inter, C = prod clamp(max(p_hi, t_hi) - min(p_lo, t_lo), 0),
//              giou = inter / union - (C - union) / C
//     loss   = L1 + mean over valid rows of (1 - giou)   (NaN when no row is valid, as the reference's mean of an empty tensor)
// The gradient follows torch's autograd of that expression: max / min split the gradient in half at a tie, clamp(min=0) passes
// it where its argument is >= 0, the target gets none, and a valid row's GIoU gradient is divided by n_valid.  An invalid row
// (or every row when n_valid == 0) gets the L1 gradient sign(p - t) / nsentences only.
// One CTA loops over the rows twice (the GIoU gradient needs n_valid first); every sum runs in a fixed order, so repeated
// launches are bit-identical.
#include "common.cuh"
#include "ops.h"

namespace opb {

namespace {

constexpr int kBoxThreads = 256;

// d max(a, b) / d a as torch's maximum backward (half at a tie); d min(a, b) / d a likewise
OPB_DEVICE float dmax_a(float a, float b) { return a > b ? 1.f : (a == b ? 0.5f : 0.f); }
OPB_DEVICE float dmin_a(float a, float b) { return a < b ? 1.f : (a == b ? 0.5f : 0.f); }

struct BoxRow {
  float p[4];
  float l1;        // sum_j |p_j - t_j|
  bool valid;
  float giou;
};

OPB_DEVICE BoxRow box_row(const float* z, const float* t) {
  BoxRow r;
#pragma unroll
  for (int j = 0; j < 4; ++j) r.p[j] = 1.f / (1.f + expf(-z[j]));
  r.l1 = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) r.l1 += fabsf(r.p[j] - t[j]);
  r.valid = r.p[0] < r.p[2] && r.p[1] < r.p[3];
  const float* p = r.p;
  const float a1 = (p[2] - p[0]) * (p[3] - p[1]), a2 = (t[2] - t[0]) * (t[3] - t[1]);
  const float w = fmaxf(fminf(p[2], t[2]) - fmaxf(p[0], t[0]), 0.f);
  const float h = fmaxf(fminf(p[3], t[3]) - fmaxf(p[1], t[1]), 0.f);
  const float inter = w * h;
  const float uni = a1 + a2 - inter;
  const float wc = fmaxf(fmaxf(p[2], t[2]) - fminf(p[0], t[0]), 0.f);
  const float hc = fmaxf(fmaxf(p[3], t[3]) - fminf(p[1], t[1]), 0.f);
  const float c = wc * hc;
  r.giou = inter / uni - (c - uni) / c;
  return r;
}

// d giou / d p of one row (torchvision's formulas, differentiated as torch's autograd does)
OPB_DEVICE void giou_grad(const float* p, const float* t, float* g) {
  const float a1 = (p[2] - p[0]) * (p[3] - p[1]), a2 = (t[2] - t[0]) * (t[3] - t[1]);
  const float wr = fminf(p[2], t[2]) - fmaxf(p[0], t[0]), hr = fminf(p[3], t[3]) - fmaxf(p[1], t[1]);
  const float w = fmaxf(wr, 0.f), h = fmaxf(hr, 0.f);
  const float inter = w * h;
  const float uni = a1 + a2 - inter;
  const float wcr = fmaxf(p[2], t[2]) - fminf(p[0], t[0]), hcr = fmaxf(p[3], t[3]) - fminf(p[1], t[1]);
  const float wc = fmaxf(wcr, 0.f), hc = fmaxf(hcr, 0.f);
  const float c = wc * hc;
  // giou = inter / union - (C - union) / C
  const float d_uni = -inter / (uni * uni) + 1.f / c;
  const float d_inter = 1.f / uni - d_uni;           // union = a1 + a2 - inter
  const float d_c = -uni / (c * c);
  // area of p: (p2 - p0) (p3 - p1)
  g[0] = -d_uni * (p[3] - p[1]);
  g[2] = d_uni * (p[3] - p[1]);
  g[1] = -d_uni * (p[2] - p[0]);
  g[3] = d_uni * (p[2] - p[0]);
  // intersection: clamp passes where its argument is >= 0
  const float dw = wr >= 0.f ? d_inter * h : 0.f, dh = hr >= 0.f ? d_inter * w : 0.f;
  g[2] += dw * dmin_a(p[2], t[2]);
  g[0] -= dw * dmax_a(p[0], t[0]);
  g[3] += dh * dmin_a(p[3], t[3]);
  g[1] -= dh * dmax_a(p[1], t[1]);
  // enclosing box
  const float dwc = wcr >= 0.f ? d_c * hc : 0.f, dhc = hcr >= 0.f ? d_c * wc : 0.f;
  g[2] += dwc * dmax_a(p[2], t[2]);
  g[0] -= dwc * dmin_a(p[0], t[0]);
  g[3] += dhc * dmax_a(p[3], t[3]);
  g[1] -= dhc * dmin_a(p[1], t[1]);
}

OPB_DEVICE float sign0(float x) { return x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f); }

// fixed-order sum over the CTA; every thread gets the result
OPB_DEVICE float box_cta_sum(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
  for (int w = 0; w < kBoxThreads / 32; ++w) s += red[w];
  return s;
}

__global__ void __launch_bounds__(kBoxThreads)
refcoco_loss_kernel(const float* __restrict__ logits, long ld, const float* __restrict__ targets, int B, float nsent,
                    float* __restrict__ out, int* __restrict__ valid, float* __restrict__ giou, float* __restrict__ dlogits) {
  __shared__ float red[kBoxThreads / 32];
  float l1 = 0.f, gsum = 0.f, nv = 0.f;
  for (int r = threadIdx.x; r < B; r += kBoxThreads) {
    const BoxRow b = box_row(logits + static_cast<long>(r) * ld, targets + static_cast<long>(r) * 4);
    l1 += b.l1;
    if (b.valid) {
      gsum += 1.f - b.giou;
      nv += 1.f;
    }
    valid[r] = b.valid ? 1 : 0;
    giou[r] = b.giou;
  }
  l1 = box_cta_sum(l1, red);
  gsum = box_cta_sum(gsum, red);
  nv = box_cta_sum(nv, red);                          // exact: integers below 2^24
  const float inv_ns = 1.f / nsent;
  for (int r = threadIdx.x; r < B; r += kBoxThreads) {
    const float* z = logits + static_cast<long>(r) * ld;
    const float* t = targets + static_cast<long>(r) * 4;
    const BoxRow b = box_row(z, t);
    float g[4] = {0.f, 0.f, 0.f, 0.f};
    if (b.valid) giou_grad(b.p, t, g);
    float* dz = dlogits + static_cast<long>(r) * ld;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float dp = sign0(b.p[j] - t[j]) * inv_ns;
      if (b.valid) dp += -g[j] / nv;
      dz[j] = dp * (1.f - b.p[j]) * b.p[j];
    }
    for (long j = 4; j < ld; ++j) dz[j] = 0.f;
  }
  if (threadIdx.x == 0) {
    const float l1_part = l1 / nsent;
    out[0] = l1_part + (nv > 0.f ? gsum / nv : __int_as_float(0x7fc00000));
    out[1] = l1_part;
    out[2] = nv;
  }
}

// iou_acc.py:20-32 in its own operation order, every step rounded separately (no FMA contraction)
__global__ void iou_acc_kernel(const float* __restrict__ hyps, long ld_h, const float* __restrict__ refs, long ld_r, int n,
                               int* __restrict__ hits, int* __restrict__ row_hit) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  bool hit = false;
  if (r < n) {
    const float* h = hyps + static_cast<long>(r) * ld_h;
    const float* f = refs + static_cast<long>(r) * ld_r;
    const float i0 = h[0] < f[0] ? f[0] : h[0], i1 = h[1] < f[1] ? f[1] : h[1];
    const float i2 = h[2] < f[2] ? h[2] : f[2], i3 = h[3] < f[3] ? h[3] : f[3];
    const float area_p = __fmul_rn(__fsub_rn(h[2], h[0]), __fsub_rn(h[3], h[1]));
    const float area_t = __fmul_rn(__fsub_rn(f[2], f[0]), __fsub_rn(f[3], f[1]));
    const float iw = __fsub_rn(i2, i0), ih = __fsub_rn(i3, i1);
    const float area_i = __fmul_rn(iw, ih);
    const float iou = __fdiv_rn(area_i, __fsub_rn(__fadd_rn(area_p, area_t), area_i));
    hit = iou >= 0.5f && iw > 0.f && ih > 0.f;
    if (row_hit != nullptr) row_hit[r] = hit ? 1 : 0;
  }
  const unsigned m = __ballot_sync(0xffffffffu, hit);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(hits, __popc(m));
}

}  // namespace

int refcoco_loss(const float* logits, long ld, const float* targets, int B, int nsentences, float* out, int* valid, float* giou,
                 float* dlogits, cudaStream_t stream) {
  if (B <= 0 || ld < 4 || nsentences <= 0) return OPB_ERR_INVALID;
  refcoco_loss_kernel<<<1, kBoxThreads, 0, stream>>>(logits, ld, targets, B, static_cast<float>(nsentences), out, valid, giou,
                                                     dlogits);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

int iou_acc(const float* hyps, long ld_h, const float* refs, long ld_r, int n, int* hits, int* row_hit, cudaStream_t stream) {
  if (n <= 0 || ld_h < 4 || ld_r < 4) return OPB_ERR_INVALID;
  iou_acc_kernel<<<(n + 255) / 256, 256, 0, stream>>>(hyps, ld_h, refs, ld_r, n, hits, row_hit);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

}  // namespace opb
