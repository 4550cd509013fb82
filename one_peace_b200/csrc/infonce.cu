// Cross-modal InfoNCE head (criterions/image_text_retrieval_loss.py:91-112; pretrain twin
// image_text_pretrain_loss.py:164-185).  For one direction with local rows A (b x d), gathered rows
// B_all (n x d, n = world * b, detached) and s = exp(clamp(logit_scale)):
//     Z = s * A B_all^T,  loss_i = (1-eps-eps_i) (lse_i - z_{i,t_i}) + eps_i (n lse_i - sum_j z_ij),  t_i = i + rank*b
//     dL/dA = (s / 2b) G B_all,  G_ij = softmax(Z)_ij - (1-eps-eps_i) [j == t_i] - eps_i      (local rows only,
//     no gradient to B_all: the gathers are detached, :30-38)
// The b x n logits are never materialised in fp32: the wgmma GEMM epilogues reduce each 128x256 tile to
// per-row partials (forward) or write the bf16 gradient factor G directly (backward), and a second GEMM
// contracts G with B_all.  This file holds the small merge / reduction kernels and the host sequencing.
#include "common.cuh"
#include "gemm.h"
#include "ops.h"

namespace opb {

// d(loss)/d(logit_scale) = coef * sum_ij G_ij z_ij over both directions (ws_a / ws_b: [n_tiles, b] partials)
__global__ void infonce_dscale_kernel(const float* __restrict__ ws_a, const float* __restrict__ ws_b, long count,
                                      float coef, float* __restrict__ out) {
  __shared__ float red[32];
  float acc = 0.f;
  for (long i = threadIdx.x; i < count; i += blockDim.x) acc += ws_a[i] + ws_b[i];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < (blockDim.x >> 5); ++w) t += red[w];
    out[0] = t * coef;
  }
}

// bf16 [rows, cols] -> [cols, rows] through a padded smem tile (coalesced both ways)
__global__ void transpose_bf16_kernel(const __nv_bfloat16* __restrict__ in, long ld_in,
                                      __nv_bfloat16* __restrict__ out, int rows, int cols) {
  __shared__ __nv_bfloat16 tile[64][66];
  const int r0 = blockIdx.y * 64, c0 = blockIdx.x * 64;
  for (int i = threadIdx.y; i < 64; i += blockDim.y) {
    const int r = r0 + i;
    for (int j = threadIdx.x; j < 64; j += blockDim.x) {
      const int c = c0 + j;
      tile[i][j] = (r < rows && c < cols) ? in[static_cast<long>(r) * ld_in + c] : __float2bfloat16(0.f);
    }
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 64; i += blockDim.y) {
    const int c = c0 + i;
    for (int j = threadIdx.x; j < 64; j += blockDim.x) {
      const int r = r0 + j;
      if (r < rows && c < cols) out[static_cast<long>(c) * rows + r] = tile[j][i];
    }
  }
}

// 16-byte version (rows, cols, ld_in multiples of 8; 16-byte aligned bases): 64 x 64 tile, every global access is a
// full 16-byte vector (the 2-byte version above moves 64 B per warp instruction and ran at ~1.5 TB/s; the backward
// pass transposes ~0.75 GB per layer for its dW GEMM operands).
__global__ void __launch_bounds__(256)
transpose_bf16_vec_kernel(const __nv_bfloat16* __restrict__ in, long ld_in, __nv_bfloat16* __restrict__ out, int rows,
                          int cols) {
  __shared__ __align__(16) __nv_bfloat16 tile[64][72];      // [col][row], 144-byte pitch
  const int r0 = blockIdx.y * 64, c0 = blockIdx.x * 64;
#pragma unroll
  for (int it = 0; it < 2; ++it) {
    const int v = threadIdx.x + it * 256;                   // 512 vectors: 64 rows x 8 vectors
    const int r = v >> 3, cv = (v & 7) * 8;
    uint4 d = make_uint4(0u, 0u, 0u, 0u);
    if (r0 + r < rows && c0 + cv < cols) d = *reinterpret_cast<const uint4*>(in + static_cast<long>(r0 + r) * ld_in + c0 + cv);
    const __nv_bfloat16* e = reinterpret_cast<const __nv_bfloat16*>(&d);
#pragma unroll
    for (int j = 0; j < 8; ++j) tile[cv + j][r] = e[j];
  }
  __syncthreads();
#pragma unroll
  for (int it = 0; it < 2; ++it) {
    const int v = threadIdx.x + it * 256;
    const int c = v >> 3, rv = (v & 7) * 8;
    if (c0 + c < cols && r0 + rv < rows)
      *reinterpret_cast<uint4*>(out + static_cast<long>(c0 + c) * rows + r0 + rv) = *reinterpret_cast<const uint4*>(&tile[c][rv]);
  }
}

int transpose_bf16(const void* in, long ld_in, void* out, int rows, int cols, cudaStream_t stream) {
  if (rows <= 0 || cols <= 0 || ld_in < cols) return OPB_ERR_INVALID;
  if ((rows & 7) == 0 && (cols & 7) == 0 && (ld_in & 7) == 0 && (reinterpret_cast<uintptr_t>(in) & 15) == 0 &&
      (reinterpret_cast<uintptr_t>(out) & 15) == 0) {
    dim3 vgrid((cols + 63) / 64, (rows + 63) / 64);
    transpose_bf16_vec_kernel<<<vgrid, 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(in), ld_in,
                                                         reinterpret_cast<__nv_bfloat16*>(out), rows, cols);
    return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
  }
  dim3 grid((cols + 63) / 64, (rows + 63) / 64), block(32, 8);
  transpose_bf16_kernel<<<grid, block, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(in), ld_in,
                                                    reinterpret_cast<__nv_bfloat16*>(out), rows, cols);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

// fp32 [rows, d] -> bf16 [rows, 3d]: x = hi + lo with hi = bf16(x), lo = bf16(x - hi).
// side 0 (the local operand): [hi | hi | lo];  side 1 (the gathered operand): [hi | lo | hi], so that one K = 3d
// wgmma GEMM yields hi.hi + hi.lo + lo.hi — the logits to ~2^-16 relative instead of bf16's 2^-9, which is what
// keeps the loss within 1e-3 of the fp32 oracle at small d / large logit_scale.
// Up to four tensors in ONE launch (the operands of one InfoNCE step: a_local, b_local side 0; a_all, b_all side 1):
// blockIdx.y selects the tensor.
struct SplitArgs {
  const float* x[4];
  __nv_bfloat16* out[4];
  long total[4];
  int side[4];
};
__global__ void split_bf16x3_kernel(const SplitArgs sp, int d) {
  const int t = blockIdx.y;
  const float* __restrict__ x = sp.x[t];
  __nv_bfloat16* __restrict__ out = sp.out[t];
  const long total = sp.total[t];
  const int side = sp.side[t];
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long>(gridDim.x) * blockDim.x) {
    const long r = i / d;
    const int c = i % d;
    const float v = x[i];
    const __nv_bfloat16 hi = __float2bfloat16(v);
    const __nv_bfloat16 lo = __float2bfloat16(v - __bfloat162float(hi));
    __nv_bfloat16* o = out + r * 3L * d + c;
    o[0] = hi;
    o[d] = side == 0 ? hi : lo;
    o[2L * d] = side == 0 ? lo : hi;
  }
}

int split_bf16x3(const float* const* xs, void* const* outs, const int64_t* rows, const int* sides, int count, int d,
                 cudaStream_t stream) {
  if (count < 1 || count > 4 || d <= 0) return OPB_ERR_INVALID;
  SplitArgs sp;
  long mx = 0;
  for (int t = 0; t < count; ++t) {
    if (xs[t] == nullptr || outs[t] == nullptr || rows[t] <= 0 || (sides[t] != 0 && sides[t] != 1)) return OPB_ERR_INVALID;
    sp.x[t] = xs[t]; sp.out[t] = reinterpret_cast<__nv_bfloat16*>(outs[t]); sp.total[t] = rows[t] * d; sp.side[t] = sides[t];
    if (sp.total[t] > mx) mx = sp.total[t];
  }
  long blocks = (mx + 255) / 256;
  if (blocks > 132L * 16 / count) blocks = 132L * 16 / count;      // at most 16 blocks per SM over all tensors
  split_bf16x3_kernel<<<dim3(static_cast<unsigned>(blocks), count), 256, 0, stream>>>(sp, d);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

// merge of one or both directions' per-tile partials + the step's scalar outputs in one launch.  blockIdx.y = direction
// (gridDim.y = 1 or 2); every block merges 128 rows and takes a ticket; the LAST block to finish sums all gridDim.y * b row
// losses / hit flags in a fixed order (the result does not depend on which block that is) and resets the ticket counter for
// the next call.
__global__ void __launch_bounds__(128)
infonce_merge_reduce_kernel(const float* __restrict__ ws_a, const float* __restrict__ ws_b, int n_tiles, int b, int n, float eps,
                            int target_offset, float* __restrict__ lse_a, float* __restrict__ lse_b, float* __restrict__ loss_ab,
                            int* __restrict__ am_ab, float* __restrict__ out3, unsigned int* __restrict__ ticket) {
  __shared__ float red[3][4];
  __shared__ bool last;
  const int dirs = gridDim.y;
  const int dir = blockIdx.y;
  const float* __restrict__ ws = dir == 0 ? ws_a : ws_b;
  float* __restrict__ row_lse = dir == 0 ? lse_a : lse_b;
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row < b) {
    float m = -INFINITY;
    for (int t = 0; t < n_tiles; ++t) m = fmaxf(m, ws[(static_cast<long>(t) * b + row) * 8]);
    float s = 0.f, zsum = 0.f, best = -INFINITY, ztgt = 0.f;
    int best_idx = 0;
    for (int t = 0; t < n_tiles; ++t) {
      const float* w = ws + (static_cast<long>(t) * b + row) * 8;
      const float4 p0 = *reinterpret_cast<const float4*>(w);
      const float4 p1 = *reinterpret_cast<const float4*>(w + 4);
      s += p0.y * __expf(p0.x - m);
      zsum += p0.z;
      if (p0.w > best) { best = p0.w; best_idx = __float_as_int(p1.x); }   // strict >: first maximum wins (torch.argmax)
      if (p1.z != 0.f) ztgt = p1.y;
    }
    const float lse = m + logf(s);
    const float nll = lse - ztgt;
    float loss = nll;
    if (eps != 0.f) {
      const float eps_i = eps / (n - 1);
      loss = (1.f - eps - eps_i) * nll + eps_i * (n * lse - zsum);
    }
    row_lse[row] = lse;
    loss_ab[dir * b + row] = loss;
    am_ab[dir * b + row] = best_idx;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(ticket, 1u) == gridDim.x * gridDim.y - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  float la = 0.f, ca = 0.f, cb = 0.f;
  for (int i = threadIdx.x; i < b; i += blockDim.x) {
    float l = __ldcg(loss_ab + i);
    ca += (__ldcg(am_ab + i) == i + target_offset) ? 1.f : 0.f;
    if (dirs == 2) {
      l += __ldcg(loss_ab + b + i);
      cb += (__ldcg(am_ab + b + i) == i + target_offset) ? 1.f : 0.f;
    }
    la += l;
  }
  la = warp_sum(la); ca = warp_sum(ca); cb = warp_sum(cb);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { red[0][warp] = la; red[1][warp] = ca; red[2][warp] = cb; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float t0 = 0.f, t1 = 0.f, t2 = 0.f;
    for (int w = 0; w < 4; ++w) { t0 += red[0][w]; t1 += red[1][w]; t2 += red[2][w]; }
    out3[0] = t0 / (static_cast<float>(dirs) * b);
    out3[1] = t1;
    out3[2] = t2;
    *ticket = 0u;
  }
}

static int n_tiles_of(int n) { return (n + 255) / 256; }

long infonce_ws_floats(int b, int n) { return static_cast<long>(n_tiles_of(n)) * b * 8; }

// LSE_PARTIAL GEMM of one direction (the merge runs later, for every direction at once: infonce_merge_reduce)
int infonce_lse_gemm(const void* a_local, const void* b_all, const float* scale, int b, int n, int d, int target_offset, float* ws,
                     int n_valid, cudaStream_t stream) {
  if (b <= 0 || n <= 0 || d <= 0 || d % 8 != 0 || n % 8 != 0 || n_valid < 0 || n_valid > n) return OPB_ERR_INVALID;
  GemmEpilogue ep;
  ep.out = ws;            // unused by this epilogue but must be non-null for the generic checks
  ep.scale_ptr = scale;
  ep.ws = ws;
  ep.target_offset = target_offset;
  ep.n_valid = n_valid;
  return gemm_bf16(a_local, d, b_all, d, b, n, d, EPI_LSE_PARTIAL, ep, 0, stream);
}

// ws_b == lse_b == nullptr: one direction.  scratch: loss_ab fp32 [dirs b], am_ab int32 [dirs b], ticket: one zero-initialised
// uint32 (left at zero)
int infonce_merge_reduce(const float* ws_a, const float* ws_b, int b, int n, int n_valid, float eps, int target_offset, float* lse_a,
                         float* lse_b, float* loss_ab, int* am_ab, float* out3, unsigned int* ticket, cudaStream_t stream) {
  if (b <= 0 || n <= 0 || n_valid < 0 || n_valid > n || (ws_b == nullptr) != (lse_b == nullptr)) return OPB_ERR_INVALID;
  const int n_cls = n_valid > 0 ? n_valid : n;
  const int dirs = ws_b != nullptr ? 2 : 1;
  infonce_merge_reduce_kernel<<<dim3((b + 127) / 128, dirs), 128, 0, stream>>>(ws_a, ws_b, n_tiles_of(n), b, n_cls, eps, target_offset,
                                                                                lse_a, lse_b, loss_ab, am_ab, out3, ticket);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

// backward for one direction: grad_a fp32 [b, d] = (s / 2b) G B_all ; ws_gz [n_tiles, b] row partials of sum G z
int infonce_grad(const void* a_local, const void* b_all, const float* scale, const float* row_lse, int b, int n, int d,
                 int k_logits, int target_offset, float eps, void* g_ws, float* ws_gz, float* grad_a, int n_valid, float coef,
                 cudaStream_t stream) {
  if (b <= 0 || n <= 0 || d <= 0 || d % 8 != 0 || n % 8 != 0 || k_logits % 8 != 0 || n_valid < 0 || n_valid > n)
    return OPB_ERR_INVALID;
  const int n_cls = n_valid > 0 ? n_valid : n;
  GemmEpilogue ep;
  ep.out = g_ws;
  ep.ldo = n;
  ep.scale_ptr = scale;
  ep.row_lse = row_lse;
  ep.ws = ws_gz;
  ep.target_offset = target_offset;
  ep.eps = eps;
  ep.n_valid = n_valid;
  ep.eps_i = (eps != 0.f) ? eps / (n_cls - 1) : 0.f;
  ep.coef = coef > 0.f ? coef : 1.f / (2.f * b);
  int rc = gemm_bf16(a_local, k_logits, b_all, k_logits, b, n, k_logits, EPI_SOFTMAX_GRAD, ep, 0, stream);
  if (rc != OPB_OK) return rc;
  GemmEpilogue e2;
  e2.out = grad_a;
  e2.ldo = d;
  // grad_a = G . B_all: a contraction over the n gathered rows.  B_all ([n, k_logits], its first d columns = the bf16 "hi" part)
  // is the MN-major B operand as it stands, so no transposed copy is needed.
  return gemm_bf16_t(g_ws, n, 0, b_all, k_logits, 1, b, d, n, EPI_STORE_F32, e2, 0, stream);
}

int infonce_dscale(const float* ws_a, const float* ws_b, int b, int n, float* out, cudaStream_t stream) {
  infonce_dscale_kernel<<<1, 1024, 0, stream>>>(ws_a, ws_b, static_cast<long>(n_tiles_of(n)) * b, 1.f / (2.f * b),
                                               out);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

}  // namespace opb
