// Classification evaluation (metrics/accuracy.py:20-25, metrics/map.py:20-43): the argmax hit counter of Accuracy, the
// sigmoid + label packing of MAP, and scikit-learn's average precision per class with its mean.
//
// Argmax: torch.argmax's order.  A NaN is the maximum (the first NaN wins), equal values go to the lower index, bf16 is
// compared after its exact up-cast.  One warp per row for C > 8 (lane-strided, then a butterfly over that total order),
// one thread per row for C <= 8.
//
// Sigmoid: 1 / (1 + expf(-x)) in IEEE fp32, which is torch.sigmoid's CUDA fp32 formula; the library is built without
// fast-math, so expf and the division are the full-precision ones and the probabilities are torch's bit for bit.
//
// Average precision (sklearn.metrics.average_precision_score, average=None), per class c over its N samples:
//     sort by probability, descending; group equal probabilities; with TP_g / FP_g counted through group g,
//     AP_c = sum_g pos_g * TP_g / (TP_g + FP_g) / P_c        (0 when P_c = 0, as scikit-learn 1.9 returns)
// Every element becomes one 64-bit key: class << 31 | (0x3F800000 - bits(p)) << 1 | label, so ascending keys run class by
// class, probability descending inside a class, and a group is a run of equal key >> 1.  An LSD radix sort (8 bits per pass:
// per-tile histograms, a scan per digit, a stable scatter) orders the keys; one CTA per class then walks its N sorted keys
// with integer prefix sums (plain for TP, segmented at group starts for pos_g).  Each group's term is formed in fp64 at the
// group's last element and the terms are summed in a fixed order, so repeated launches are bit-identical.
#include <climits>

#include "common.cuh"
#include "ops.h"

namespace opb {

namespace {

constexpr int kMaxClasses = 4096;

OPB_DEVICE float to_f32(float x) { return x; }
OPB_DEVICE float to_f32(__nv_bfloat16 x) { return __bfloat162float(x); }

// torch.argmax's comparison (ATen's GreaterOrNan): does (v, i) beat (bv, bi)?
OPB_DEVICE bool argmax_better(float v, int i, float bv, int bi) {
  const bool vn = v != v, bn = bv != bv;
  if (vn || bn) return vn && (!bn || i < bi);
  return v > bv || (v == bv && i < bi);
}

// tmode 0: int64 labels (hyp == t); 1: fp32 labels compared as torch.eq does (the int64 hypothesis promoted to fp32);
// 2: soft scores fp32 [n, ldt], the score is targets[r, hyp]
OPB_DEVICE float row_score(int hyp, const void* targets, int tmode, long ldt, long r) {
  if (tmode == 0) return static_cast<const int64_t*>(targets)[r] == static_cast<int64_t>(hyp) ? 1.f : 0.f;
  if (tmode == 1) return static_cast<const float*>(targets)[r] == static_cast<float>(hyp) ? 1.f : 0.f;
  return static_cast<const float*>(targets)[r * ldt + hyp];
}

template <typename T>
__global__ void __launch_bounds__(256)
argmax_warp_kernel(const T* __restrict__ x, long ld, long cs, int n, int C, const void* __restrict__ targets, int tmode,
                   long ldt, int64_t* __restrict__ hyp, float* __restrict__ score) {
  const long r = static_cast<long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (r >= n) return;                                  // warp-uniform
  const int lane = threadIdx.x & 31;
  const T* row = x + r * ld;
  float bv = __int_as_float(0xff800000);               // -inf with index INT_MAX loses to every real element
  int bi = INT_MAX;
  for (int j = lane; j < C; j += 32) {
    const float v = to_f32(row[static_cast<long>(j) * cs]);
    if (argmax_better(v, j, bv, bi)) {
      bv = v;
      bi = j;
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (argmax_better(ov, oi, bv, bi)) {
      bv = ov;
      bi = oi;
    }
  }
  if (lane == 0) {
    hyp[r] = bi;
    score[r] = row_score(bi, targets, tmode, ldt, r);
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
argmax_thread_kernel(const T* __restrict__ x, long ld, long cs, int n, int C, const void* __restrict__ targets, int tmode,
                     long ldt, int64_t* __restrict__ hyp, float* __restrict__ score) {
  const long r = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const T* row = x + r * ld;
  float bv = to_f32(row[0]);
  int bi = 0;
  for (int j = 1; j < C; ++j) {
    const float v = to_f32(row[static_cast<long>(j) * cs]);
    if (argmax_better(v, j, bv, bi)) {
      bv = v;
      bi = j;
    }
  }
  hyp[r] = bi;
  score[r] = row_score(bi, targets, tmode, ldt, r);
}

constexpr int kSumThreads = 1024;

// fixed order: each thread sums its stride sequentially, then lane 0 of a butterfly per warp, then warp 0 over the warps
__global__ void __launch_bounds__(kSumThreads) sum_f64_kernel(const float* __restrict__ x, long n, double* __restrict__ out) {
  __shared__ double red[kSumThreads / 32];
  double s = 0.0;
  for (long i = threadIdx.x; i < n; i += kSumThreads) s += static_cast<double>(x[i]);
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = red[threadIdx.x];
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) out[0] = s;
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
sigmoid_pack_kernel(const T* __restrict__ x, long ld, long cs, const float* __restrict__ t, long ldt, int n, int C,
                    float* __restrict__ probs, uint8_t* __restrict__ labels, long row_offset, int* __restrict__ flags) {
  const long idx = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  bool bad_t = false, bad_p = false;
  if (idx < static_cast<long>(n) * C) {
    const long r = idx / C;
    const long j = idx - r * C;
    const float z = to_f32(x[r * ld + j * cs]);
    const float p = 1.0f / (1.0f + expf(-z));
    const float y = t[r * ldt + j];
    bad_t = !(y == 0.f || y == 1.f);
    bad_p = p != p;
    const long o = (row_offset + r) * C + j;
    probs[o] = p;
    labels[o] = y == 1.f ? 1 : 0;
  }
  const unsigned mt = __ballot_sync(0xffffffffu, bad_t), mp = __ballot_sync(0xffffffffu, bad_p);
  if ((threadIdx.x & 31) == 0) {
    if (mt) atomicAdd(flags, __popc(mt));
    if (mp) atomicAdd(flags + 1, __popc(mp));
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// average precision
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kSortThreads = 256, kSortItems = 16, kTile = kSortThreads * kSortItems;
constexpr int kSortWarps = kSortThreads / 32;
constexpr int kScanThreads = 1024, kWalkThreads = 1024;
constexpr int kMaxPasses = 8;
constexpr uint32_t kOneBits = 0x3F800000u;           // bits of 1.0f: every probability in [0, 1] lies at or below it

__global__ void ap_keys_kernel(const float* __restrict__ probs, const uint8_t* __restrict__ labels, int N, int C,
                               uint64_t* __restrict__ keys) {
  const long idx = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<long>(N) * C) return;
  const long r = idx / C;
  const long c = idx - r * C;
  uint32_t b = __float_as_uint(probs[idx]);
  if (b > kOneBits) b = (b >> 31) ? 0u : kOneBits;   // outside [0, 1] (or NaN): clamped, so the key stays in its class
  keys[c * N + r] = (static_cast<uint64_t>(c) << 31) | (static_cast<uint64_t>(kOneBits - b) << 1) | (labels[idx] ? 1u : 0u);
}

// hist[d * tiles + tile] = number of keys of the tile whose digit is d; totals[d] += the same (integer atomics: exact)
__global__ void __launch_bounds__(kSortThreads)
radix_hist_kernel(const uint64_t* __restrict__ keys, long M, int shift, int tiles, uint32_t* __restrict__ hist,
                  uint32_t* __restrict__ totals) {
  __shared__ uint32_t h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  const long base = static_cast<long>(blockIdx.x) * kTile;
#pragma unroll 4
  for (int k = 0; k < kSortItems; ++k) {
    const long i = base + k * kSortThreads + threadIdx.x;
    if (i < M) atomicAdd(&h[(keys[i] >> shift) & 255u], 1u);
  }
  __syncthreads();
  const uint32_t v = h[threadIdx.x];
  hist[static_cast<long>(threadIdx.x) * tiles + blockIdx.x] = v;
  if (v) atomicAdd(&totals[threadIdx.x], v);
}

// one CTA per digit d: hist[d, :] <- sum_{e < d} totals[e] + exclusive prefix over the tiles of hist[d, :]
__global__ void __launch_bounds__(kScanThreads)
radix_scan_kernel(uint32_t* __restrict__ hist, int tiles, const uint32_t* __restrict__ totals) {
  __shared__ uint32_t warp_tot[kScanThreads / 32];
  __shared__ uint32_t s_base;
  const int d = blockIdx.x, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    uint32_t b = 0;
    for (int e = 0; e < d; ++e) b += totals[e];
    s_base = b;
  }
  __syncthreads();
  uint32_t carry = s_base;
  uint32_t* row = hist + static_cast<long>(d) * tiles;
  for (int c0 = 0; c0 < tiles; c0 += kScanThreads) {
    const int i = c0 + threadIdx.x;
    const uint32_t v = i < tiles ? row[i] : 0u;
    uint32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t u = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += u;
    }
    if (lane == 31) warp_tot[w] = x;
    __syncthreads();
    if (w == 0) {
      uint32_t y = warp_tot[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t u = __shfl_up_sync(0xffffffffu, y, o);
        if (lane >= o) y += u;
      }
      warp_tot[lane] = y;
    }
    __syncthreads();
    if (i < tiles) row[i] = carry + (w ? warp_tot[w - 1] : 0u) + x - v;
    carry += warp_tot[kScanThreads / 32 - 1];
    __syncthreads();
  }
}

// stable scatter: the keys of a tile go out in position order (round, warp, lane) behind the tile's offset for their digit
__global__ void __launch_bounds__(kSortThreads)
radix_scatter_kernel(const uint64_t* __restrict__ in, uint64_t* __restrict__ out, long M, int shift, int tiles,
                     const uint32_t* __restrict__ hist) {
  __shared__ uint32_t offs[256];
  __shared__ uint32_t wcnt[kSortWarps][256];
  __shared__ uint32_t woff[kSortWarps][256];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  offs[t] = hist[static_cast<long>(t) * tiles + blockIdx.x];
#pragma unroll
  for (int w = 0; w < kSortWarps; ++w) wcnt[w][t] = 0;
  __syncthreads();
  const uint32_t lt = (1u << lane) - 1u;
  const long base = static_cast<long>(blockIdx.x) * kTile;
  for (int k = 0; k < kSortItems; ++k) {
    const long i = base + k * kSortThreads + t;
    if (base + k * kSortThreads >= M) break;           // block-uniform
    const bool ok = i < M;
    const uint64_t key = ok ? in[i] : 0ull;
    const uint32_t d = ok ? static_cast<uint32_t>((key >> shift) & 255u) : 0xffffffffu;
    const uint32_t peers = __match_any_sync(0xffffffffu, d);
    const uint32_t rank = __popc(peers & lt);
    if (ok && rank == 0) wcnt[warp][d] = __popc(peers);
    __syncthreads();
    uint32_t run = offs[t];
#pragma unroll
    for (int w = 0; w < kSortWarps; ++w) {
      const uint32_t c = wcnt[w][t];
      woff[w][t] = run;
      wcnt[w][t] = 0;
      run += c;
    }
    offs[t] = run;
    __syncthreads();
    if (ok) out[woff[warp][d] + rank] = key;
  }
}

// block-wide inclusive scan of (cum, seg, flag): cum a plain sum, seg a sum that restarts where flag is set
struct SegScan {
  int cum, seg, f;
};

OPB_DEVICE SegScan combine(SegScan l, SegScan r) {
  SegScan o;
  o.cum = l.cum + r.cum;
  o.seg = r.f ? r.seg : l.seg + r.seg;
  o.f = l.f | r.f;
  return o;
}

OPB_DEVICE SegScan warp_segscan(SegScan x, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    SegScan u;
    u.cum = __shfl_up_sync(0xffffffffu, x.cum, o);
    u.seg = __shfl_up_sync(0xffffffffu, x.seg, o);
    u.f = __shfl_up_sync(0xffffffffu, x.f, o);
    if (lane >= o) x = combine(u, x);
  }
  return x;
}

OPB_DEVICE uint32_t group_of(uint64_t key) { return static_cast<uint32_t>(key >> 1) & 0x3fffffffu; }

// one CTA per class over its N sorted keys; ap[c] = sum_g pos_g * TP_g / (TP_g + FP_g) / P, npos[c] = P
__global__ void __launch_bounds__(kWalkThreads)
ap_walk_kernel(const uint64_t* __restrict__ keys, int N, double* __restrict__ ap, int64_t* __restrict__ npos) {
  __shared__ SegScan s_agg[kWalkThreads / 32];
  __shared__ double s_red[kWalkThreads / 32];
  __shared__ int s_carry[2];
  const int c = blockIdx.x, t = threadIdx.x, lane = t & 31, w = t >> 5;
  const uint64_t* k = keys + static_cast<long>(c) * N;
  int carry_cum = 0, carry_seg = 0;
  double acc = 0.0;
  for (int c0 = 0; c0 < N; c0 += kWalkThreads) {
    const int i = c0 + t;
    const bool ok = i < N;
    SegScan x = {0, 0, 0};
    bool end = false;
    if (ok) {
      const uint64_t key = k[i];
      const uint32_t g = group_of(key);
      x.cum = x.seg = static_cast<int>(key & 1u);
      x.f = (i == 0 || group_of(k[i - 1]) != g) ? 1 : 0;
      end = i == N - 1 || group_of(k[i + 1]) != g;
    }
    x = warp_segscan(x, lane);
    if (lane == 31) s_agg[w] = x;
    __syncthreads();
    if (w == 0) s_agg[lane] = warp_segscan(s_agg[lane], lane);
    __syncthreads();
    if (w) x = combine(s_agg[w - 1], x);
    x = combine(SegScan{carry_cum, carry_seg, 0}, x);
    double term = 0.0;
    if (ok && end) term = static_cast<double>(x.seg) * (static_cast<double>(x.cum) / static_cast<double>(i + 1));
#pragma unroll
    for (int o = 16; o; o >>= 1) term += __shfl_xor_sync(0xffffffffu, term, o);
    if (lane == 0) s_red[w] = term;
    if (i == min(c0 + kWalkThreads, N) - 1) {
      s_carry[0] = x.cum;
      s_carry[1] = x.seg;
    }
    __syncthreads();
    if (w == 0) {
      double s = s_red[lane];
#pragma unroll
      for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      acc += s;                                        // lane 0's value is the one kept
    }
    carry_cum = s_carry[0];
    carry_seg = s_carry[1];
    __syncthreads();
  }
  if (t == 0) {
    ap[c] = carry_cum > 0 ? acc / static_cast<double>(carry_cum) : 0.0;
    npos[c] = carry_cum;
  }
}

// the mean over classes, summed in class order
__global__ void ap_mean_kernel(const double* __restrict__ ap, int C, double* __restrict__ mean) {
  if (threadIdx.x != 0) return;
  double s = 0.0;
  for (int c = 0; c < C; ++c) s += ap[c];
  mean[0] = s / static_cast<double>(C);
}

struct ApWorkspace {
  uint64_t* keys[2];
  uint32_t* hist;
  uint32_t* totals;
  long bytes;
};

long align256(long b) { return (b + 255) / 256 * 256; }

int ap_passes(int C) {
  int cbits = 0;
  while ((1 << cbits) < C) ++cbits;
  return (31 + cbits + 7) / 8;
}

ApWorkspace ap_workspace(int N, int C, void* base) {
  const long M = static_cast<long>(N) * C;
  const long tiles = (M + kTile - 1) / kTile;
  char* p = static_cast<char*>(base);
  ApWorkspace ws;
  long off = 0;
  ws.keys[0] = reinterpret_cast<uint64_t*>(p + off);
  off += align256(M * 8);
  ws.keys[1] = reinterpret_cast<uint64_t*>(p + off);
  off += align256(M * 8);
  ws.hist = reinterpret_cast<uint32_t*>(p + off);
  off += align256(256 * tiles * 4);
  ws.totals = reinterpret_cast<uint32_t*>(p + off);
  off += align256(256 * kMaxPasses * 4);
  ws.bytes = off;
  return ws;
}

bool ap_shape_ok(int N, int C) {
  return N >= 1 && N < (1 << 24) && C >= 1 && C <= kMaxClasses && static_cast<long>(N) * C <= INT_MAX;
}

}  // namespace

int argmax_hits(const void* logits, int dtype, long ld, long cs, int n, int C, const void* targets, int tmode, long ldt,
                int64_t* hyp, float* score, cudaStream_t stream) {
  if (n <= 0 || C < 1 || C > kMaxClasses || ld < 1 || cs < 1 || (dtype != 0 && dtype != 1) || tmode < 0 || tmode > 2 ||
      (tmode == 2 && ldt < C))
    return OPB_ERR_INVALID;
  if (C <= 8) {
    const int grid = (n + 255) / 256;
    if (dtype == 0)
      argmax_thread_kernel<<<grid, 256, 0, stream>>>(static_cast<const float*>(logits), ld, cs, n, C, targets, tmode, ldt, hyp,
                                                     score);
    else
      argmax_thread_kernel<<<grid, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(logits), ld, cs, n, C, targets, tmode,
                                                     ldt, hyp, score);
  } else {
    const int grid = (n + 7) / 8;
    if (dtype == 0)
      argmax_warp_kernel<<<grid, 256, 0, stream>>>(static_cast<const float*>(logits), ld, cs, n, C, targets, tmode, ldt, hyp,
                                                   score);
    else
      argmax_warp_kernel<<<grid, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(logits), ld, cs, n, C, targets, tmode, ldt,
                                                   hyp, score);
  }
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

int sum_f64(const float* x, long n, double* out, cudaStream_t stream) {
  if (n <= 0) return OPB_ERR_INVALID;
  sum_f64_kernel<<<1, kSumThreads, 0, stream>>>(x, n, out);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

int sigmoid_pack(const void* logits, int dtype, long ld, long cs, const float* targets, long ldt, int n, int C, float* probs,
                 uint8_t* labels, long row_offset, int* flags, cudaStream_t stream) {
  if (n <= 0 || C < 1 || C > kMaxClasses || ld < 1 || cs < 1 || ldt < C || row_offset < 0 || (dtype != 0 && dtype != 1))
    return OPB_ERR_INVALID;
  const long total = static_cast<long>(n) * C;
  const unsigned grid = static_cast<unsigned>((total + 255) / 256);
  if (dtype == 0)
    sigmoid_pack_kernel<<<grid, 256, 0, stream>>>(static_cast<const float*>(logits), ld, cs, targets, ldt, n, C, probs, labels,
                                                  row_offset, flags);
  else
    sigmoid_pack_kernel<<<grid, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(logits), ld, cs, targets, ldt, n, C, probs,
                                                  labels, row_offset, flags);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

long average_precision_ws_bytes(int N, int C) {
  if (!ap_shape_ok(N, C)) return -1;
  return ap_workspace(N, C, nullptr).bytes;
}

int average_precision(const float* probs, const uint8_t* labels, int N, int C, void* ws, long ws_bytes, double* ap,
                      double* mean, int64_t* npos, cudaStream_t stream) {
  if (!ap_shape_ok(N, C)) return OPB_ERR_INVALID;
  const ApWorkspace w = ap_workspace(N, C, ws);
  if (ws_bytes < w.bytes) return OPB_ERR_INVALID;
  const long M = static_cast<long>(N) * C;
  const int tiles = static_cast<int>((M + kTile - 1) / kTile);
  if (cudaMemsetAsync(w.totals, 0, 256 * kMaxPasses * sizeof(uint32_t), stream) != cudaSuccess) return OPB_ERR_CUDA;
  ap_keys_kernel<<<static_cast<unsigned>((M + 255) / 256), 256, 0, stream>>>(probs, labels, N, C, w.keys[0]);
  const int passes = ap_passes(C);
  for (int p = 0; p < passes; ++p) {
    const uint64_t* in = w.keys[p & 1];
    uint64_t* out = w.keys[(p + 1) & 1];
    uint32_t* totals = w.totals + 256 * p;
    radix_hist_kernel<<<tiles, kSortThreads, 0, stream>>>(in, M, 8 * p, tiles, w.hist, totals);
    radix_scan_kernel<<<256, kScanThreads, 0, stream>>>(w.hist, tiles, totals);
    radix_scatter_kernel<<<tiles, kSortThreads, 0, stream>>>(in, out, M, 8 * p, tiles, w.hist);
  }
  ap_walk_kernel<<<C, kWalkThreads, 0, stream>>>(w.keys[passes & 1], N, ap, npos);
  ap_mean_kernel<<<1, 32, 0, stream>>>(ap, C, mean);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

}  // namespace opb
