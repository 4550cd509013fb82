// Retrieval evaluation (reference: one_peace/metrics/recall.py:22-78): top-k of every row of the similarity matrix and
// Recall@{1,5,10} counters.
//   topk_rows    one warp per row of sim fp32 [R, C]: the 10 largest entries of the row under a total order, in
//                descending order.  Values rank in IEEE order with -0.0 equal to +0.0, every NaN above +inf (as
//                torch.topk ranks NaN) and -inf like any other value; equal values rank by the smaller column.  That is a
//                stable descending sort of the row.  Slots past C get column -1 and value -inf.
//                Every lane keeps a sorted private top-10 of its strided columns in registers as packed 64-bit keys
//                (order key << 32 | ~column, so one unsigned compare ranks value and column), then 10 rounds of a
//                warp-wide max merge the 32 lists.  An empty slot is the key 0, whose column field ~0xffffffff no column
//                has; every entry is larger.  Values are read back from sim, so they keep their bits.  One pass over
//                sim: 5000 x 25010 fp32 in 0.47 ms on an H100 80GB HBM3 at 700 W (scripts/bench_topk10.py).
//   recall_hits  hits[0..2] += [cand_ids[idx[r, p]] == row_ids[r] for some p < 1 / 5 / 10]  (recall.py:39-41,50-52)
#include "common.cuh"
#include "ops.h"

namespace opb {

namespace {

constexpr int kTopK = 10;
constexpr int kBatch = 16;                    // loads in flight per lane (5000 x 25010 on an H100: 16 beats 8 and 4)

// order-preserving unsigned key of an fp32 value: negative values bit-flipped, positive ones with the sign bit set; both
// zeros map to the key of +0.0 and every NaN to the largest key
OPB_DEVICE uint32_t order_key(float x) {
  const uint32_t u = __float_as_uint(x);
  const uint32_t k = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return x != x ? 0xffffffffu : (x == 0.f ? 0x80000000u : k);
}

// the value of an order key (+0.0 for both zeros); NaN for the key of NaN and for 0, the empty slot
OPB_DEVICE float key_value(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

__global__ void topk_rows_kernel(const float* __restrict__ sim, long ld, int* __restrict__ idx, float* __restrict__ val,
                                 int R, int C) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= R) return;
  const float* s = sim + row * ld;
  unsigned long long t[kTopK];
#pragma unroll
  for (int i = 0; i < kTopK; ++i) t[i] = 0ull;
  uint32_t floor_key = 0;                     // order key of t[kTopK - 1] (0: empty)
  float floor_val = key_value(0);             // its value; NaN when the slot is empty or holds a NaN
  // A lane visits its columns in increasing order, so an entry whose key equals the last one's has the larger column and
  // ranks below it: only a strictly larger key enters the list.  !(x <= floor_val) is true for every such x (and for
  // more when floor_val is NaN), so the common case costs one float compare.
  auto consider = [&](float x, int c) {
    if (x <= floor_val) return;
    const uint32_t k = order_key(x);
    if (k > floor_key) {
      t[kTopK - 1] = (static_cast<unsigned long long>(k) << 32) | static_cast<uint32_t>(~c);
#pragma unroll
      for (int i = kTopK - 1; i > 0; --i) {
        if (t[i] > t[i - 1]) {
          const unsigned long long tt = t[i]; t[i] = t[i - 1]; t[i - 1] = tt;
        }
      }
      floor_key = static_cast<uint32_t>(t[kTopK - 1] >> 32);
      floor_val = key_value(floor_key);
    }
  };
  int c = lane;
  for (; c + 32 * (kBatch - 1) < C; c += 32 * kBatch) {     // kBatch loads in flight per lane
    float xb[kBatch];
#pragma unroll
    for (int u = 0; u < kBatch; ++u) xb[u] = s[c + 32 * u];
#pragma unroll
    for (int u = 0; u < kBatch; ++u) consider(xb[u], c + 32 * u);
  }
  for (; c < C; c += 32) consider(s[c], c);
  int mine = -1;                              // lane k keeps the column of round k
  for (int k = 0; k < kTopK; ++k) {
    unsigned long long b = t[0];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long ob = __shfl_xor_sync(0xffffffffu, b, o);
      b = ob > b ? ob : b;
    }
    if (lane == k && b != 0ull) mine = static_cast<int>(~static_cast<uint32_t>(b));
    if (t[0] == b && b != 0ull) {             // the winning lane pops its head (keys are unique per column)
#pragma unroll
      for (int i = 0; i < kTopK - 1; ++i) t[i] = t[i + 1];
      t[kTopK - 1] = 0ull;
    }
  }
  if (lane < kTopK) {
    idx[static_cast<long>(row) * kTopK + lane] = mine;
    if (val != nullptr) val[static_cast<long>(row) * kTopK + lane] = mine < 0 ? -INFINITY : s[mine];
  }
}

__global__ void recall_hits_kernel(const int* __restrict__ idx, const int64_t* __restrict__ cand_ids,
                                   const int64_t* __restrict__ row_ids, int R, int* __restrict__ hits) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  int first = kTopK;
  if (r < R) {
    const int64_t want = row_ids[r];
    for (int p = kTopK - 1; p >= 0; --p) {
      const int c = idx[static_cast<long>(r) * kTopK + p];
      if (c >= 0 && cand_ids[c] == want) first = p;
    }
  }
  const unsigned m1 = __ballot_sync(0xffffffffu, first < 1), m5 = __ballot_sync(0xffffffffu, first < 5),
                 m10 = __ballot_sync(0xffffffffu, first < 10);
  if ((threadIdx.x & 31) == 0) {
    if (m1) atomicAdd(hits + 0, __popc(m1));
    if (m5) atomicAdd(hits + 1, __popc(m5));
    if (m10) atomicAdd(hits + 2, __popc(m10));
  }
}

}  // namespace

int topk10_rows(const float* sim, long ld, int* idx, float* val, int R, int C, cudaStream_t stream) {
  if (R <= 0 || C <= 0 || ld < C) return OPB_ERR_INVALID;
  topk_rows_kernel<<<static_cast<unsigned>((static_cast<long>(R) * 32 + 255) / 256), 256, 0, stream>>>(sim, ld, idx, val, R, C);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

int recall_hits(const int* idx, const int64_t* cand_ids, const int64_t* row_ids, int R, int* hits3, cudaStream_t stream) {
  if (R <= 0) return OPB_ERR_INVALID;
  recall_hits_kernel<<<(R + 255) / 256, 256, 0, stream>>>(idx, cand_ids, row_ids, R, hits3);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

}  // namespace opb
