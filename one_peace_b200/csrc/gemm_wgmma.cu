// Warp-specialised bf16 GEMM for sm_90a (Hopper):  C[M,N] = epilogue( A[M,K] . B[N,K]^T )
//
//   * operands are bf16, K-major (activations [rows, K], nn.Linear weights [out, in]) or MN-major (given as [K, rows]: the
//     weight gradient dW = dY^T X and the InfoNCE gradient), staged into shared memory by TMA with the 128-byte swizzle,
//     BLOCK_K = 64, four pipeline stages (4 x 48 KB; three in the kernels that stage their output tile, see below);
//   * persistent: one CTA per SM walks 128 x 256 output tiles (grouped in bands of row panels, see kBandM) with the stage ring
//     running on across tiles, so the next tile's loads overlap the current tile's epilogue.  Three warpgroups: in warpgroup 0
//     one thread issues the TMA loads and warps 1-3 stage the next tile's epilogue operands (LayerNorm row statistics, column
//     vectors) in shared memory (register budget lowered with setmaxnreg); warpgroups 1 and 2 own 64 rows each and issue
//     wgmma.m64n256k16 (fp32 accumulators in registers, 128 per thread);
//   * the fused epilogue runs on the accumulator fragments.  A thread holds two rows (r, r + 8) x 2 adjacent columns of every
//     8-column group, so per-row reductions (LayerNorm statistics, soft-max partials) are finished with two shuffles inside a
//     quad.  gemm_bf16_kernel stores the results straight to global memory.  gemm_bf16_tma_out_kernel (the bf16 epilogues on
//     a plain row-major output) writes them with stmatrix into a per-warpgroup shared-memory copy of its 64 output rows and
//     one thread hands that to TMA bulk stores, so the stores drain while the warpgroup runs the next tile's mainloop.
//     gemm_bf16_resid_tma_kernel (the residual epilogue on plain aligned operands) has the producer load the fp32 residual
//     into the stage ring after the tile's k-blocks, 64 columns per stage, and stores each chunk's fp32 result and bf16
//     copy from that stage with TMA (see epilogue_resid_ring).
//
// Fused epilogues (what the reference runs as separate ATen kernels, SURVEY.md 2.5 K1'/K3/K4):
//   EPI_STORE_BF16 : out_bf16 = (acc + bias[n]) * colscale[n]        (q/k/v projection, q pre-scaled;
//                                                                     multihead_attention.py:103-107)
//   EPI_GEGLU_BF16 : out_bf16[:, t*128+j] = gelu(acc[:, j]) * acc[:, 128+j] on a W0/W1-interleaved
//                    weight (transformer_layer.py:54-67) — the 2*ffn wide intermediate never hits HBM
//   EPI_RESID_F32  : out_f32 = resid + gamma[n] * (acc + bias[n])    (out_proj / fc2 + LayerScale +
//                                                                     residual, transformer_layer.py:70-88)
//   EPI_STORE_F32  : out_f32 = acc + bias[n]
//   EPI_GELU_BF16, EPI_LSE_PARTIAL, EPI_SOFTMAX_GRAD: see gemm.h
#include "common.cuh"
#include "gemm.h"

#include <mutex>

namespace opb {

constexpr int kBlockM = 128;   // rows of A per CTA (two consumer warpgroups x 64)
constexpr int kBlockN = 256;   // output columns per tile = wgmma N
constexpr int kBlockK = 64;    // 64 bf16 = 128 bytes = one swizzle row
constexpr int kStages = 4;          // gemm_bf16_kernel
constexpr int kStagesTmaOut = 3;    // gemm_bf16_tma_out_kernel: the output staging area takes the fourth stage's room
constexpr int kABytes = kBlockM * kBlockK * 2;   // 16 KB
constexpr int kBBytes = kBlockN * kBlockK * 2;   // 32 KB
constexpr int kStageBytes = kABytes + kBBytes;
constexpr int kThreads = 384;
// Tiles run in bands of kBandM row panels, row panel fastest inside a band: the CTAs resident at one time cover a few A
// panels and a run of weight panels, so each weight panel is read from HBM about once per band instead of once per row panel.
// On an H100 bands of 8 and 16 time the same; bands of 1 (row-major tile order) make the GeGLU GEMM about 6 % slower.
constexpr int kBandM = 8;
// Column groups of the residual fragment loaded ahead of their stores in the EPI_RESID_F32 epilogue (see epilogue()): 16
// float2 = 32 registers fit next to the 128 accumulators without spills, a whole fragment row of 32 does not.
constexpr int kResidBatch = 16;

// Epilogue operands of one tile, staged in shared memory by the spare warps of the producer warpgroup while the consumers
// run the mainloop (two buffers: tile i + 1 is staged while tile i's epilogue reads).
struct EpiOperands {
  float2 row[kBlockM];   // fused-LayerNorm (mu, rstd) of the tile's rows
  float colsum[kBlockN], bias[kBlockN], gamma[kBlockN], colscale[kBlockN];   // the tile's slices of the column vectors
};
constexpr int kStagerThreads = 96;   // warps 1-3 of warpgroup 0
// Output staging of gemm_bf16_tma_out_kernel, right after the stage ring: per consumer warpgroup its 64 rows x 256 bf16
// columns as four 64 x 64 boxes (8 KB, 128-byte swizzle), the box layout of the output tensor map.
constexpr int kOutBoxBytes = 64 * 128;
constexpr int kOutStageBytes = 4 * kOutBoxBytes;
// stage ring (+ output staging) + barriers + epilogue operands + alignment slack
constexpr int smem_bytes(int stages, bool tma_out) {
  return stages * kStageBytes + (tma_out ? 2 * kOutStageBytes : 0) + 1024 + 2 * sizeof(EpiOperands) + 1024;
}
constexpr int kSmemBytes = smem_bytes(kStages, false);
constexpr int kSmemBytesTmaOut = smem_bytes(kStagesTmaOut, true);
static_assert(kSmemBytesTmaOut <= 227 * 1024, "output staging does not fit next to the stage ring");
// Residual chunks of gemm_bf16_resid_tma_kernel: a stage holds 64 columns of the tile's 128 rows, the fp32 residual (then
// result) as two 32-column boxes of 16 KB and the bf16 copy as one 64-column box after them, all with the 128-byte swizzle.
// A consumer warpgroup's 64 rows are the second half of each box (8 KB in).
constexpr int kChunks = kBlockN / 64;
constexpr int kResidBoxBytes = kBlockM * 128;
constexpr int kChunkBf16Offset = 2 * kResidBoxBytes;
static_assert(kChunkBf16Offset + kBlockM * 128 == kStageBytes, "a residual chunk fills one stage");

struct GemmGeom {
  int M, N, K;          // per group: rows, output columns, reduction length (= taps * kb_inner * 64 when windowed)
  int kb_inner;         // k-blocks per tap (inner A coordinate wraps every kb_inner blocks); K-blocks total = taps * kb_inner
  int num_k_blocks;
  int groups;           // independent problems sharing A rows (grouped conv); 1 otherwise
  int a_group_c0;       // inner A coordinate offset per group
  int b_group_rows;     // B row offset per group (= N)
  // MN-major operands: the operand is given as [K rows, MN cols] row-major.  TMA stages [64 k-rows][64 MN elements = 128 B]
  // boxes, one per 64-wide MN chunk, 8 KB apart, and the wgmma descriptors select the transposed (MN-major) layout.
  int a_mn;
  int b_mn;
  // Small-M split-K (gemm_bf16): the K range is cut into pieces of kb_per_piece k-blocks (0 = off); work unit (piece, tile) stores its
  // raw fp32 accumulators into slab `piece` of split_ws ([pieces][m_pad][N]) and gemm_split_epilogue_kernel adds the slabs in
  // piece order (deterministic) and applies the epilogue.
  int kb_per_piece;
  int m_pad;
  float* split_ws;
};

// ----------------------------------------------------------------------------------------------
// wgmma helpers (descriptor, fence / commit / wait: common.cuh)
// ----------------------------------------------------------------------------------------------
// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma window
OPB_DEVICE void fence_acc(float (&d)[128]) {
#pragma unroll
  for (int i = 0; i < 128; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 256] (+)= A[64 x 16] . B[256 x 16]^T, bf16 -> fp32; TA / TB = 1: operand stored MN-major
template <int TA, int TB>
OPB_DEVICE void wgmma_m64n256k16(float (&d)[128], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
      "}, %128, %129, p, 1, 1, %131, %132;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d), "n"(TA), "n"(TB));
}

// ----------------------------------------------------------------------------------------------
// kernel
// ----------------------------------------------------------------------------------------------
// Row statistics for the fused-LayerNorm epilogue: either precomputed (mu, rstd) or reduced here from partial records, in
// record order.  The variance E[x^2] - mu^2 is rounded explicitly: once (kFusedVar: the GeGLU and residual epilogues) or after
// the product and the difference each (the others).  That is how earlier versions of this kernel evaluated it, so results
// stay bit-identical, and they no longer depend on how the compiler contracts the expression where it is inlined.
template <bool kFusedVar = false>
OPB_DEVICE void load_ln_stats(const GemmEpilogue& ep, int row, int M, float& mu, float& rs) {
  mu = 0.f; rs = 1.f;
  const int rc = row < M ? row : M - 1;
  if (ep.ln_partial != nullptr) {
    float s1 = 0.f, s2 = 0.f;
#pragma unroll 8
    for (int p = 0; p < ep.ln_parts; ++p) {
      const float2 v = *reinterpret_cast<const float2*>(ep.ln_partial + (static_cast<long>(p) * M + rc) * 2);
      s1 += v.x; s2 += v.y;
    }
    mu = s1 / ep.ln_dim;
    const float ex2 = s2 / ep.ln_dim;
    const float var = kFusedVar ? fmaf(-mu, mu, ex2) : __fsub_rn(ex2, __fmul_rn(mu, mu));
    rs = rsqrtf(fmaxf(var, 0.f) + ep.ln_eps);
  } else if (ep.ln_mu != nullptr) {
    mu = ep.ln_mu[rc];
    rs = ep.ln_rstd[rc];
  }
}

OPB_DEVICE float2 ldf2(const float* p) { return *reinterpret_cast<const float2*>(p); }
OPB_DEVICE float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// One tile's k-blocks.  `it0` counts the k-blocks this CTA consumed for earlier tiles: the stage ring and its phases run on
// across tiles, so the producer fills the next tile's stages while the current tile's epilogue runs.
template <int TA, int TB, int S>
OPB_DEVICE void mainloop(float (&d)[128], uint8_t* smem, uint64_t* full, uint64_t* empty, int num_k_blocks, int cw,
                         uint32_t it0) {
  // descriptor advance per 16-deep wgmma: 32 B inside the swizzle row (K-major) or two 8-row k groups = 2048 B (MN-major)
  constexpr uint32_t step_a = TA ? 2048 : 32, step_b = TB ? 2048 : 32;
  const bool signal = (threadIdx.x & 31) == 0;
  for (int kb = 0; kb < num_k_blocks; ++kb) {
    const uint32_t it = it0 + kb;
    const uint32_t s = it % S;
    mbar_wait_quiet(&full[s], (it / S) & 1);
    const uint32_t sa = smem_u32(smem + s * kStageBytes) + cw * 8192;   // this warpgroup's 64 rows (K-major) / M chunk (MN-major)
    const uint32_t sb = smem_u32(smem + s * kStageBytes + kABytes);
    fence_acc(d);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBlockK / 16; ++k)
      wgmma_m64n256k16<TA, TB>(d, wgmma_desc_sw128(sa + k * step_a, 8192), wgmma_desc_sw128(sb + k * step_b, 8192),
                               (kb > 0 || k > 0) ? 1u : 0u);
    wgmma_commit();
    fence_acc(d);
    if (kb > 0) {             // the previous stage's wgmmas are done: hand its buffers back to the producer
      wgmma_wait<1>();
      fence_acc(d);
      __syncwarp();
      if (signal) mbar_arrive(&empty[(it - 1) % S]);
    }
  }
  wgmma_wait<0>();
  fence_acc(d);
  __syncwarp();
  if (signal) mbar_arrive(&empty[(it0 + num_k_blocks - 1) % S]);
}

// Output staging (gemm_bf16_tma_out_kernel).  The bf16 pairs v[0 .. kGroups) of fragment row h, one per 8-column group, go
// into the warpgroup's staging area with one stmatrix.x4 per 4 groups: matrix i is the 8 x 8 block of rows (warp, h) and
// column group 4 q + i, lane l gives the address of row l & 7 of matrix l >> 3.  With the 128-byte swizzle the 8 rows of a
// matrix hit 8 different 16-byte bank groups, so the stores are conflict-free.  Called after the loop that computes v: an
// aligned (convergent) instruction inside it would keep the compiler from specialising that loop on the epilogue's flags.
template <int kGroups>
OPB_DEVICE void stage_out_row(uint32_t stage, int h, const uint32_t (&v)[kGroups]) {
  const int lane = threadIdx.x & 31;
  const int row = ((threadIdx.x & 127) >> 5) * 16 + 8 * h + (lane & 7);
#pragma unroll
  for (int q = 0; q < kGroups / 4; ++q) {
    const int cg = 4 * q + (lane >> 3);
    const uint32_t addr = stage + (cg >> 3) * kOutBoxBytes + sw128_off(row, cg & 7);
    asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v[4 * q]),
                 "r"(v[4 * q + 1]), "r"(v[4 * q + 2]), "r"(v[4 * q + 3]));
  }
}

OPB_DEVICE void warpgroup_bar_sync(int cw) {
  if (cw == 0) asm volatile("bar.sync 1, 128;" ::: "memory");
  else asm volatile("bar.sync 2, 128;" ::: "memory");
}

// Before the staging area is written again: the previous tile's bulk stores have finished reading it.  Only the thread that
// issued them can wait for them; the named barrier (one per consumer warpgroup, id 1 + cw) passes that on to its warps.
OPB_DEVICE void acquire_out_stage(int cw) {
  if ((threadIdx.x & 127) == 0) bulk_wait_read<0>();
  warpgroup_bar_sync(cw);
}

// After the epilogue has staged the tile: make the shared-memory writes visible to the async proxy, meet at the warpgroup's
// barrier, and let one thread store the boxes of rows row0 .. row0 + 63 that hold output, as one bulk group.  Rows >= rows
// and columns >= cols of a box are clipped by the tensor map; boxes wholly outside are not issued.
OPB_DEVICE void store_out_tile(const CUtensorMap& tm_out, uint8_t* stage, int row0, int col0, int rows, int cols, int boxes,
                               int cw) {
  fence_proxy_async();
  warpgroup_bar_sync(cw);
  if ((threadIdx.x & 127) == 0) {
    if (row0 < rows) {
      for (int b = 0; b < boxes; ++b)
        if (col0 + 64 * b < cols) tma_store_2d(&tm_out, stage + b * kOutBoxBytes, col0 + 64 * b, row0);
    }
    bulk_commit();
  }
}

// the epilogues that take their operands from EpiOperands (the contrastive-head ones read none of them)
constexpr bool epi_staged(int epi) { return epi != EPI_LSE_PARTIAL && epi != EPI_SOFTMAX_GRAD; }

// Stager side: fill `st` for tile (m_blk, n_blk, grp), thread `t` of kStagerThreads.
template <int EPI>
OPB_DEVICE void stage_epi_operands(EpiOperands* st, const GemmEpilogue& ep, const GemmGeom& geo, int m_blk, int n_blk, int grp,
                                   int t) {
  if (ep.ln_partial != nullptr || ep.ln_mu != nullptr) {
    for (int r = t; r < kBlockM; r += kStagerThreads) {
      float mu, rs;
      load_ln_stats<EPI == EPI_GEGLU_BF16 || EPI == EPI_RESID_F32>(ep, m_blk * kBlockM + r, geo.M, mu, rs);
      st->row[r] = make_float2(mu, rs);
    }
  }
  for (int c = t; c < kBlockN; c += kStagerThreads) {
    const int tc = n_blk * kBlockN + c;
    const bool ok = tc < geo.N;
    const int col = grp * geo.N + tc;
    st->colsum[c] = ok && ep.ln_colsum != nullptr ? ep.ln_colsum[col] : 0.f;
    st->bias[c] = ok && ep.bias != nullptr ? ep.bias[col] : 0.f;
    st->gamma[c] = ok && ep.gamma != nullptr ? ep.gamma[col] : 0.f;
    st->colscale[c] = ok && ep.colscale != nullptr ? ep.colscale[col] : 0.f;
  }
}

// kTmaOut: the bf16 results go to the warpgroup's output staging area at shared address `out_stage` (all 64 rows and every
// column of the tile; store_out_tile clips them) instead of global memory.  The values and their order are the same.
template <int EPI, bool kTmaOut>
OPB_DEVICE void epilogue(const float (&d)[128], const GemmEpilogue& ep, const GemmGeom& geo, const EpiOperands* st,
                         uint32_t out_stage, int m_blk, int n_blk, int grp, int cw) {
  const int M = geo.M, N = geo.N;
  const int t = threadIdx.x & 127;
  const int lane = t & 31;
  const int quad = lane & 3;
  const int rloc = cw * 64 + (t >> 5) * 16 + (lane >> 2);   // row inside the tile (fragment row r)
  const int rbase = m_blk * kBlockM + rloc;
  const int col0 = n_blk * kBlockN;   // first column of the tile inside the group
  const int gcol0 = grp * N;          // first global output column of the group
#pragma unroll
  for (int h = 0; h < 2; ++h) {       // fragment rows r and r + 8
    const int row = rbase + 8 * h;
    bool row_ok = row < M;
    if (ep.out_group > 0 && ep.out_group_valid > 0 && (row % ep.out_group) >= ep.out_group_valid) row_ok = false;
    // output / residual row mapping (lets adapters scatter rows behind a CLS slot and broadcast a positional table over the batch)
    long out_row = row;
    if (ep.out_group > 0) out_row = static_cast<long>(row / ep.out_group) * ep.out_group_stride + (row % ep.out_group) + ep.out_row_offset;
    long res_row = out_row;
    if (ep.resid_period > 0) res_row = (row % ep.resid_period) + ep.resid_row_offset;

    if constexpr (EPI == EPI_LSE_PARTIAL) {
      // z = scale * acc: per (row, 256-column tile) running max / sum-exp / sum z / arg-max / target logit
      const float scale = *ep.scale_ptr;
      const int tgt = row + ep.target_offset;
      const int nv = ep.n_valid > 0 ? ep.n_valid : N;
      float m = -INFINITY;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int col = col0 + 8 * j + 2 * quad;
        if (col < nv) m = fmaxf(m, scale * d[4 * j + 2 * h]);
        if (col + 1 < nv) m = fmaxf(m, scale * d[4 * j + 2 * h + 1]);
      }
      float ssum = 0.f, zsum = 0.f, best = -INFINITY, ztgt = 0.f;
      int best_idx = 0, has_tgt = 0;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = col0 + 8 * j + 2 * quad + e;
          if (col < nv) {
            const float z = scale * d[4 * j + 2 * h + e];
            ssum += __expf(z - m);
            zsum += z;
            if (z > best) { best = z; best_idx = col; }
            if (col == tgt) { ztgt = z; has_tgt = 1; }
          }
        }
      }
#pragma unroll
      for (int o = 1; o <= 2; o <<= 1) {
        const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, ssum, o);
        const float zs2 = __shfl_xor_sync(0xffffffffu, zsum, o), b2 = __shfl_xor_sync(0xffffffffu, best, o);
        const int i2 = __shfl_xor_sync(0xffffffffu, best_idx, o), h2 = __shfl_xor_sync(0xffffffffu, has_tgt, o);
        const float zt2 = __shfl_xor_sync(0xffffffffu, ztgt, o);
        const float mn = fmaxf(m, m2);
        ssum = (m > -INFINITY ? ssum * __expf(m - mn) : 0.f) + (m2 > -INFINITY ? s2 * __expf(m2 - mn) : 0.f);
        m = mn;
        zsum += zs2;
        if (b2 > best || (b2 == best && i2 < best_idx)) { best = b2; best_idx = i2; }
        if (h2) { ztgt = zt2; has_tgt = 1; }
      }
      if (row_ok && quad == 0) {
        float* w = ep.ws + (static_cast<long>(n_blk) * M + row) * 8;
        *reinterpret_cast<float4*>(w) = make_float4(m, ssum, zsum, best);
        *reinterpret_cast<float4*>(w + 4) = make_float4(__int_as_float(best_idx), ztgt, has_tgt ? 1.f : 0.f, 0.f);
      }
    } else if constexpr (EPI == EPI_SOFTMAX_GRAD) {
      const float scale = *ep.scale_ptr;
      const float gscale = scale * ep.coef;
      const int tgt = row + ep.target_offset;
      const float lse = row_ok ? ep.row_lse[row] : 0.f;
      const float hit = 1.f - ep.eps - ep.eps_i;
      const int nv = ep.n_valid > 0 ? ep.n_valid : N;
      float gz = 0.f;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int col = col0 + 8 * j + 2 * quad;
        if (!row_ok || col >= N) continue;
        float gq[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float z = scale * d[4 * j + 2 * h + e];
          float g = __expf(z - lse) - ep.eps_i;
          if (col + e == tgt) g -= hit;
          if (col + e >= nv) g = 0.f;
          gz += g * z;
          gq[e] = g * gscale;
        }
        *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(ep.out) + out_row * ep.ldo + col) = pack_bf16x2(gq[0], gq[1]);
      }
      gz = quad_sum(gz);
      if (row_ok && quad == 0) ep.ws[static_cast<long>(n_blk) * M + row] = gz;
    } else {
      const float2 mr = (ep.ln_partial != nullptr || ep.ln_mu != nullptr) ? st->row[rloc + 8 * h] : make_float2(0.f, 1.f);
      const float mu = mr.x, rs = mr.y;
      const bool has_ln = ep.ln_colsum != nullptr;
      float st_sum = 0.f, st_sq = 0.f;   // partial statistics of the stored values (next LayerNorm)
      if constexpr (EPI == EPI_GEGLU_BF16) {
        __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(ep.out) + out_row * ep.ldo + n_blk * (kBlockN / 2);
        uint32_t packed[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int tc = 8 * j + 2 * quad;    // gate column inside the tile; its linear partner is tc + 128
          float g0 = d[4 * j + 2 * h], g1 = d[4 * j + 2 * h + 1];
          float l0 = d[4 * (j + 16) + 2 * h], l1 = d[4 * (j + 16) + 2 * h + 1];
          if (has_ln) {
            const float2 cg = ldf2(st->colsum + tc), cl = ldf2(st->colsum + tc + kBlockN / 2);
            g0 = rs * (g0 - mu * cg.x); g1 = rs * (g1 - mu * cg.y);
            l0 = rs * (l0 - mu * cl.x); l1 = rs * (l1 - mu * cl.y);
          }
          if (ep.bias != nullptr) {
            const float2 bg = ldf2(st->bias + tc), bl = ldf2(st->bias + tc + kBlockN / 2);
            g0 += bg.x; g1 += bg.y; l0 += bl.x; l1 += bl.y;
          }
          const float u0 = gelu_erf(g0) * l0, u1 = gelu_erf(g1) * l1;
          st_sum += u0 + u1;
          st_sq += u0 * u0 + u1 * u1;
          if constexpr (kTmaOut) packed[j] = pack_bf16x2(u0, u1);
          else if (row_ok) *reinterpret_cast<uint32_t*>(out + tc) = pack_bf16x2(u0, u1);
        }
        if constexpr (kTmaOut) stage_out_row(out_stage, h, packed);
        st_sum = quad_sum(st_sum);
        st_sq = quad_sum(st_sq);
        if (row_ok && quad == 0 && ep.stats_out != nullptr) {   // [2 * n_tiles, M] records, the second of a tile is zero
          *reinterpret_cast<float2*>(ep.stats_out + (static_cast<long>(n_blk * 2) * M + row) * 2) = make_float2(st_sum, st_sq);
          *reinterpret_cast<float2*>(ep.stats_out + (static_cast<long>(n_blk * 2 + 1) * M + row) * 2) = make_float2(0.f, 0.f);
        }
      } else {
        // EPI_RESID_F32: the thread's residual fragment of this row is read in batches of kResidBatch column groups, each
        // batch loaded before any of its stores.  `out` and `resid` may alias (the stack updates the residual stream in
        // place), so the compiler cannot hoist a load above an earlier store: loaded inside the column loop, every column
        // group would wait for its own global round trip.  Loading ahead is safe because an element of `resid` that is also
        // an output element is the one this thread writes from the same fragment slot (gemm_bf16 refuses any other overlap).
        uint32_t packed[32];
#pragma unroll
        for (int jb = 0; jb < 32; jb += kResidBatch) {
          float2 res[kResidBatch];
          if constexpr (EPI == EPI_RESID_F32) {
            if (ep.resid != nullptr && row_ok) {
              const float* rp = ep.resid + res_row * ep.ldr + gcol0;
#pragma unroll
              for (int jj = 0; jj < kResidBatch; ++jj) {
                const int tc = col0 + 8 * (jb + jj) + 2 * quad;
                if (tc < N) res[jj] = ldf2(rp + tc);
              }
            }
          }
#pragma unroll
          for (int jj = 0; jj < kResidBatch; ++jj) {
            const int j = jb + jj;
            const int lc = 8 * j + 2 * quad;           // column inside the tile
            const int tc = col0 + lc;                  // column inside the group
            if (!kTmaOut && tc >= N) continue;         // (staged: columns >= N hold zeros and are clipped)
            const int col = gcol0 + tc;
            float x0 = d[4 * j + 2 * h], x1 = d[4 * j + 2 * h + 1];
            if (has_ln) {
              const float2 c = ldf2(st->colsum + lc);
              x0 = rs * (x0 - mu * c.x); x1 = rs * (x1 - mu * c.y);
            }
            if (ep.bias != nullptr) {
              const float2 b = ldf2(st->bias + lc);
              x0 += b.x; x1 += b.y;
            }
            if constexpr (EPI == EPI_STORE_BF16 || EPI == EPI_GELU_BF16) {
              if (ep.colscale != nullptr) {
                const float2 s = ldf2(st->colscale + lc);
                x0 *= s.x; x1 *= s.y;
              }
              if constexpr (EPI == EPI_GELU_BF16) { x0 = gelu_erf(x0); x1 = gelu_erf(x1); }
              if constexpr (kTmaOut) {
                packed[j] = pack_bf16x2(x0, x1);
              } else {
                if (row_ok) *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(ep.out) + out_row * ep.ldo + col) = pack_bf16x2(x0, x1);
              }
            } else {
              if constexpr (EPI == EPI_RESID_F32) {
                if (ep.gamma != nullptr) {
                  const float2 g = ldf2(st->gamma + lc);
                  x0 *= g.x; x1 *= g.y;
                }
                if (ep.resid != nullptr && row_ok) {
                  x0 += res[jj].x; x1 += res[jj].y;
                }
                st_sum += x0 + x1;
                st_sq += x0 * x0 + x1 * x1;
                if (row_ok && ep.out_bf16 != nullptr)
                  *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(ep.out_bf16) + out_row * ep.ldo_bf16 + col) = pack_bf16x2(x0, x1);
              }
              if (row_ok) *reinterpret_cast<float2*>(reinterpret_cast<float*>(ep.out) + out_row * ep.ldo + col) = make_float2(x0, x1);
            }
          }
        }
        if constexpr (kTmaOut) stage_out_row(out_stage, h, packed);
        if constexpr (EPI == EPI_RESID_F32) {
          st_sum = quad_sum(st_sum);
          st_sq = quad_sum(st_sq);
          if (row_ok && quad == 0 && ep.stats_out != nullptr)
            *reinterpret_cast<float2*>(ep.stats_out + (static_cast<long>(n_blk) * M + row) * 2) = make_float2(st_sum, st_sq);
        }
      }
    }
  }
}

// EPI_RESID_F32 through the stage ring (gemm_bf16_resid_tma_kernel).  The producer follows the tile's k-blocks with kChunks
// ring entries, entry it + c holding the residual of tile columns 64 c .. 64 c + 63 (rows >= M and columns >= N zero-filled).
// For each chunk the warpgroup computes its 64 rows with the operations of epilogue<EPI_RESID_F32>, in the same order (st_sum
// / st_sq run over the columns left to right across the chunks), writes the fp32 result over the residual it read and the
// bf16 copy next to it, and one thread stores both with TMA as one bulk group (rows >= M and columns >= N clipped).  A
// chunk's stage goes back to the producer once the stores of both warpgroups have read it: chunk c - 1 after chunk c's stores
// are issued, the last chunk before the warpgroup leaves.  That is required, not only early: the next tile's first k-blocks
// land in these stages, so a stage still held when the consumers wait on the next tile's `full` barriers would never fill.
template <int S>
OPB_DEVICE void epilogue_resid_ring(const float (&d)[128], const GemmEpilogue& ep, const GemmGeom& geo, const EpiOperands* st,
                                    uint8_t* smem, uint64_t* full, uint64_t* empty, const CUtensorMap& tm_out,
                                    const CUtensorMap& tm_out_bf16, uint32_t it, int m_blk, int n_blk, int cw) {
  const int M = geo.M, N = geo.N;
  const int t = threadIdx.x & 127;
  const int lane = t & 31;
  const int quad = lane & 3;
  const int rloc = cw * 64 + (t >> 5) * 16 + (lane >> 2);   // row inside the tile and the chunk's boxes (fragment row r)
  const int rbase = m_blk * kBlockM + rloc;
  const int row0 = m_blk * kBlockM + cw * 64;                // first row of the warpgroup's stores
  const bool has_ln = ep.ln_colsum != nullptr;
  const bool has_rows = ep.ln_partial != nullptr || ep.ln_mu != nullptr;
  float st_sum[2] = {0.f, 0.f}, st_sq[2] = {0.f, 0.f};   // partial statistics of the stored values (next LayerNorm)
#pragma unroll
  for (int c = 0; c < kChunks; ++c) {
    const uint32_t s = (it + c) % S;
    mbar_wait_quiet(&full[s], ((it + c) / S) & 1);
    uint8_t* stage = smem + s * kStageBytes;
#pragma unroll
    for (int h = 0; h < 2; ++h) {       // fragment rows r and r + 8
      const int r = rloc + 8 * h;
      const bool row_ok = rbase + 8 * h < M;
      const float2 mr = has_rows ? st->row[r] : make_float2(0.f, 1.f);
      const float mu = mr.x, rs = mr.y;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int j = 8 * c + jj;                  // column group of the fragment
        const int lc = 8 * j + 2 * quad;           // column inside the tile
        float2* f = reinterpret_cast<float2*>(stage + (jj >> 2) * kResidBoxBytes + sw128_off(r, 2 * (jj & 3) + (quad >> 1)) +
                                              8 * (quad & 1));
        float x0 = d[4 * j + 2 * h], x1 = d[4 * j + 2 * h + 1];
        if (has_ln) {
          const float2 cs = ldf2(st->colsum + lc);
          x0 = rs * (x0 - mu * cs.x); x1 = rs * (x1 - mu * cs.y);
        }
        if (ep.bias != nullptr) {
          const float2 b = ldf2(st->bias + lc);
          x0 += b.x; x1 += b.y;
        }
        if (ep.gamma != nullptr) {
          const float2 g = ldf2(st->gamma + lc);
          x0 *= g.x; x1 *= g.y;
        }
        if (row_ok) {
          const float2 res = *f;
          x0 += res.x; x1 += res.y;
        }
        st_sum[h] += x0 + x1;
        st_sq[h] += x0 * x0 + x1 * x1;
        *f = make_float2(x0, x1);
        *reinterpret_cast<uint32_t*>(stage + kChunkBf16Offset + sw128_off(r, jj) + 4 * quad) = pack_bf16x2(x0, x1);
      }
    }
    fence_proxy_async();
    warpgroup_bar_sync(cw);
    if (t == 0) {
      const int col = n_blk * kBlockN + 64 * c;
      if (row0 < M) {
        for (int b = 0; b < 2; ++b)
          if (col + 32 * b < N) tma_store_2d(&tm_out, stage + b * kResidBoxBytes + cw * 64 * 128, col + 32 * b, row0);
        if (ep.out_bf16 != nullptr && col < N) tma_store_2d(&tm_out_bf16, stage + kChunkBf16Offset + cw * 64 * 128, col, row0);
      }
      bulk_commit();
      if (c > 0) {                     // the stores of chunk c - 1 have read their stage
        bulk_wait_read<1>();
        mbar_arrive_count(&empty[(it + c - 1) % S], 4);
      }
      if (c == kChunks - 1) {
        bulk_wait_read<0>();
        mbar_arrive_count(&empty[s], 4);
      }
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = rbase + 8 * h;
    const float s1 = quad_sum(st_sum[h]), s2 = quad_sum(st_sq[h]);
    if (row < M && quad == 0 && ep.stats_out != nullptr)
      *reinterpret_cast<float2*>(ep.stats_out + (static_cast<long>(n_blk) * M + row) * 2) = make_float2(s1, s2);
  }
}

// Work unit -> tile.  Units are split-K piece-major (a single piece unless split-K), then group-major; inside a group the
// tiles run in bands of kBandM row panels, row panel fastest.
struct TileCoord {
  int piece, grp, m_blk, n_blk;
};
OPB_DEVICE TileCoord tile_coord(int unit, int num_m_tiles, int num_n_tiles, int groups) {
  const int per_group = num_m_tiles * num_n_tiles;
  TileCoord c;
  c.piece = unit / (per_group * groups);
  const int tile = unit - c.piece * per_group * groups;
  c.grp = tile / per_group;
  const int tin = tile - c.grp * per_group;
  const int band = tin / (kBandM * num_n_tiles);
  const int m0 = band * kBandM;
  const int band_rows = min(kBandM, num_m_tiles - m0);
  const int r = tin - m0 * num_n_tiles;
  c.m_blk = m0 + r % band_rows;
  c.n_blk = r / band_rows;
  return c;
}

// How a kernel's epilogue results leave the SM: stored from registers (gemm_bf16_kernel), staged bf16 tile and TMA stores
// (gemm_bf16_tma_out_kernel), or the residual epilogue's chunks through the stage ring (gemm_bf16_resid_tma_kernel).
enum class OutPath { kDirect, kTmaBf16, kResidRing };

// Persistent: the grid holds as many CTAs as can be resident and CTA b runs units b, b + gridDim.x, ...  Barrier set-up and
// descriptor prefetch happen once per CTA.  The body of the three kernels: S pipeline stages; kTmaBf16 stages the bf16 output
// tile in shared memory and stores it with TMA through tm_out; kResidRing loads the residual through tm_res into the stage
// ring and stores through tm_out (fp32) and tm_out_bf16 (see epilogue_resid_ring).  Maps a path does not use are null.
template <int EPI, int S, OutPath kPath>
OPB_DEVICE void gemm_body(const CUtensorMap& tm_a, const CUtensorMap& tm_b, const CUtensorMap* tm_out, const CUtensorMap* tm_res,
                          const CUtensorMap* tm_out_bf16, const GemmEpilogue& ep, const GemmGeom& geo) {
  constexpr bool kTmaOut = kPath == OutPath::kTmaBf16;
  constexpr bool kRing = kPath == OutPath::kResidRing;
  // no static shared memory: the dynamic window starts at the 1024-aligned base the 128-byte swizzle needs (checked)
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw;
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* out_stage = smem + S * kStageBytes;   // [2 consumer warpgroups][kOutStageBytes] (kTmaOut)
  uint8_t* bars = out_stage + (kTmaOut ? 2 * kOutStageBytes : 0);
  uint64_t* full = reinterpret_cast<uint64_t*>(bars);
  uint64_t* empty = full + S;
  uint64_t* epi_full = empty + S;         // [2] operands of the buffer's tile are staged
  uint64_t* epi_empty = epi_full + 2;     // [2] the buffer's epilogue is done reading
  EpiOperands* epi_ops = reinterpret_cast<EpiOperands*>(bars + 1024);

  const int wg = threadIdx.x >> 7;
  const int num_m_tiles = (geo.M + kBlockM - 1) / kBlockM;
  const int num_n_tiles = (geo.N + kBlockN - 1) / kBlockN;
  const int pieces = geo.kb_per_piece > 0 ? (geo.num_k_blocks + geo.kb_per_piece - 1) / geo.kb_per_piece : 1;
  const int units = num_m_tiles * num_n_tiles * geo.groups * pieces;
  // split-K pieces store raw accumulators and need no epilogue operands
  const bool staged = epi_staged(EPI) && (kTmaOut || kRing || geo.kb_per_piece == 0);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_a);
    tma_prefetch_desc(&tm_b);
    if constexpr (kTmaOut || kRing) tma_prefetch_desc(tm_out);
    if constexpr (kRing) {
      tma_prefetch_desc(tm_res);
      if (ep.out_bf16 != nullptr) tma_prefetch_desc(tm_out_bf16);
    }
    for (int i = 0; i < S; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8);   // lane 0 of each of the 8 consumer warps
    }
    for (int i = 0; i < 2; ++i) {
      mbar_init(&epi_full[i], kStagerThreads);
      mbar_init(&epi_empty[i], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      // ===================== TMA producer =====================
      uint32_t it = 0;   // k-blocks issued by this CTA: stage it % S, phase (it / S) & 1
      for (int unit = blockIdx.x; unit < units; unit += gridDim.x) {
        const TileCoord tc = tile_coord(unit, num_m_tiles, num_n_tiles, geo.groups);
        const int kb0 = geo.kb_per_piece > 0 ? tc.piece * geo.kb_per_piece : 0;
        const int kb1 = geo.kb_per_piece > 0 ? min(geo.num_k_blocks, kb0 + geo.kb_per_piece) : geo.num_k_blocks;
        const int a_row = tc.m_blk * kBlockM;
        const int b_row = tc.grp * geo.b_group_rows + tc.n_blk * kBlockN;
        const int a_c0 = tc.grp * geo.a_group_c0;
        int kin = kb0 % geo.kb_inner, tap = kb0 / geo.kb_inner;
        for (int kb = kb0; kb < kb1; ++kb, ++it) {
          const uint32_t s = it % S;
          mbar_wait_quiet(&empty[s], ((it / S) & 1) ^ 1);
          uint8_t* sa = smem + s * kStageBytes;
          uint8_t* sb = sa + kABytes;
          mbar_arrive_expect_tx(&full[s], kStageBytes);     // out-of-bounds box elements are zero-filled and counted
          if (geo.a_mn) {
#pragma unroll
            for (int i = 0; i < kBlockM / 64; ++i) tma_load_2d(&tm_a, &full[s], sa + i * 8192, a_row + 64 * i, kb * kBlockK);
          } else {
            tma_load_3d(&tm_a, &full[s], sa, a_c0 + kin * kBlockK, tap, a_row);
          }
          if (geo.b_mn) {
#pragma unroll
            for (int i = 0; i < kBlockN / 64; ++i) tma_load_2d(&tm_b, &full[s], sb + i * 8192, b_row + 64 * i, kb * kBlockK);
          } else {
            tma_load_2d(&tm_b, &full[s], sb, kb * kBlockK, b_row);
          }
          if (++kin == geo.kb_inner) { kin = 0; ++tap; }
        }
        if constexpr (kRing) {
          // the tile's residual, kChunks ring entries of 64 columns (see epilogue_resid_ring)
          for (int c = 0; c < kChunks; ++c, ++it) {
            const uint32_t s = it % S;
            mbar_wait_quiet(&empty[s], ((it / S) & 1) ^ 1);
            uint8_t* sr = smem + s * kStageBytes;
            mbar_arrive_expect_tx(&full[s], 2 * kResidBoxBytes);
            for (int b = 0; b < 2; ++b)
              tma_load_2d(tm_res, &full[s], sr + b * kResidBoxBytes, tc.n_blk * kBlockN + 64 * c + 32 * b, a_row);
          }
        }
      }
    } else if (threadIdx.x >= 32 && staged) {
      // ===================== epilogue-operand stager (warps 1-3) =====================
      uint32_t j = 0;   // tiles staged: buffer j & 1, phase (j >> 1) & 1
      for (int unit = blockIdx.x; unit < units; unit += gridDim.x, ++j) {
        const TileCoord tc = tile_coord(unit, num_m_tiles, num_n_tiles, geo.groups);
        mbar_wait_quiet(&epi_empty[j & 1], ((j >> 1) & 1) ^ 1);
        stage_epi_operands<EPI>(&epi_ops[j & 1], ep, geo, tc.m_blk, tc.n_blk, tc.grp, threadIdx.x - 32);
        mbar_arrive(&epi_full[j & 1]);
      }
    }
  } else {
    // ===================== consumers: wgmma + epilogue =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int cw = wg - 1;
    uint8_t* my_stage = out_stage + cw * kOutStageBytes;
    float d[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) d[i] = 0.f;
    uint32_t it = 0, j = 0;
    for (int unit = blockIdx.x; unit < units; unit += gridDim.x, ++j) {
      const TileCoord tc = tile_coord(unit, num_m_tiles, num_n_tiles, geo.groups);
      const int kb0 = geo.kb_per_piece > 0 ? tc.piece * geo.kb_per_piece : 0;
      const int kb1 = geo.kb_per_piece > 0 ? min(geo.num_k_blocks, kb0 + geo.kb_per_piece) : geo.num_k_blocks;
      if (geo.a_mn) {
        if (geo.b_mn) mainloop<1, 1, S>(d, smem, full, empty, kb1 - kb0, cw, it);
        else mainloop<1, 0, S>(d, smem, full, empty, kb1 - kb0, cw, it);
      } else {
        if (geo.b_mn) mainloop<0, 1, S>(d, smem, full, empty, kb1 - kb0, cw, it);
        else mainloop<0, 0, S>(d, smem, full, empty, kb1 - kb0, cw, it);
      }
      it += kb1 - kb0;
      if (kPath == OutPath::kDirect && geo.kb_per_piece > 0) {   // (the TMA-store kernels never run split-K)
        // split-K piece: raw partial accumulators of all m_pad rows into this piece's slab (plain stores, no atomics)
        const int t = threadIdx.x & 127, lane = t & 31;
        const int r0 = tc.m_blk * kBlockM + cw * 64 + (t >> 5) * 16 + (lane >> 2);
        float* w = geo.split_ws + static_cast<long>(tc.piece) * geo.m_pad * geo.N;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int c = 0; c < 32; ++c) {
            const int col = tc.n_blk * kBlockN + 8 * c + 2 * (lane & 3);
            if (col < geo.N)
              *reinterpret_cast<float2*>(w + static_cast<long>(r0 + 8 * h) * geo.N + col) = make_float2(d[4 * c + 2 * h], d[4 * c + 2 * h + 1]);
          }
        }
      } else if (staged) {
        mbar_wait_quiet(&epi_full[j & 1], (j >> 1) & 1);
        if constexpr (kTmaOut) acquire_out_stage(cw);
        if constexpr (kRing) {
          epilogue_resid_ring<S>(d, ep, geo, &epi_ops[j & 1], smem, full, empty, *tm_out, *tm_out_bf16, it, tc.m_blk, tc.n_blk, cw);
          it += kChunks;
        } else {
          epilogue<EPI, kTmaOut>(d, ep, geo, &epi_ops[j & 1], smem_u32(my_stage), tc.m_blk, tc.n_blk, tc.grp, cw);
        }
        __syncwarp();
        if ((threadIdx.x & 31) == 0) mbar_arrive(&epi_empty[j & 1]);
        if constexpr (kTmaOut) {
          // GeGLU writes kBlockN / 2 columns per tile: two boxes
          constexpr int cols_per_tile = EPI == EPI_GEGLU_BF16 ? kBlockN / 2 : kBlockN;
          store_out_tile(*tm_out, my_stage, tc.m_blk * kBlockM + cw * 64, tc.n_blk * cols_per_tile, geo.M,
                         EPI == EPI_GEGLU_BF16 ? geo.N / 2 : geo.N, cols_per_tile / 64, cw);
        }
      } else {
        epilogue<EPI, false>(d, ep, geo, nullptr, 0, tc.m_blk, tc.n_blk, tc.grp, cw);
      }
    }
    // the staging area must outlive the last bulk stores
    if constexpr (kTmaOut || kRing) {
      if ((threadIdx.x & 127) == 0) bulk_wait_all<0>();
    }
  }
}

template <int EPI>
__global__ void __launch_bounds__(kThreads, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b, const GemmEpilogue ep,
                 const GemmGeom geo) {
  gemm_body<EPI, kStages, OutPath::kDirect>(tm_a, tm_b, nullptr, nullptr, nullptr, ep, geo);
}

// The bf16 epilogues with the output tile staged in shared memory and stored by TMA through tm_out (rows M, columns N, or
// N / 2 for GeGLU; box 64 x 64, 128-byte swizzle).  Taken only for a single group, no split-K and no row remapping (see
// tma_out_applies).
template <int EPI>
__global__ void __launch_bounds__(kThreads, 1)
gemm_bf16_tma_out_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b,
                         const __grid_constant__ CUtensorMap tm_out, const GemmEpilogue ep, const GemmGeom geo) {
  static_assert(EPI == EPI_STORE_BF16 || EPI == EPI_GELU_BF16 || EPI == EPI_GEGLU_BF16, "bf16 epilogues only");
  gemm_body<EPI, kStagesTmaOut, OutPath::kTmaBf16>(tm_a, tm_b, &tm_out, nullptr, nullptr, ep, geo);
}

// EPI_RESID_F32 with the residual loaded into the stage ring by TMA through tm_res (fp32 [M, N], box 32 x 128) and the results
// stored by TMA through tm_out (fp32 [M, N], box 32 x 64) and tm_out_bf16 (bf16 [M, N], box 64 x 64; unused without
// out_bf16), all with the 128-byte swizzle.  Four stages and no shared memory beyond gemm_bf16_kernel's.  Taken only for a
// single group, no split-K, no row remapping or residual period, and 16-byte aligned operands (see resid_ring_applies).
template <int EPI>
__global__ void __launch_bounds__(kThreads, 1)
gemm_bf16_resid_tma_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b,
                           const __grid_constant__ CUtensorMap tm_res, const __grid_constant__ CUtensorMap tm_out,
                           const __grid_constant__ CUtensorMap tm_out_bf16, const GemmEpilogue ep, const GemmGeom geo) {
  static_assert(EPI == EPI_RESID_F32, "the residual epilogue only");
  gemm_body<EPI, kStages, OutPath::kResidRing>(tm_a, tm_b, &tm_out, &tm_res, &tm_out_bf16, ep, geo);
}

// Epilogue of the small-M split-K schedule: x = sum of the piece slabs (fixed order), then the EPI_RESID_F32 epilogue
// (resid + gamma * (rstd * (acc - mu * colsum) + bias), bf16 copy, per-256-column LayerNorm statistics) or the EPI_STORE_BF16 one
// ((rstd * (acc - mu * colsum) + bias) * colscale).  One CTA (256 threads) per (row, 256-column tile).
__global__ void __launch_bounds__(256)
gemm_split_epilogue_kernel(const GemmEpilogue ep, const GemmGeom geo, int pieces, int epi) {
  __shared__ float red[2][8];
  const int M = geo.M, N = geo.N;
  const int row = blockIdx.x;
  float mu, rs;
  if (ep.ln_partial != nullptr) {
    // the whole CTA works on one row: reduce its partial records cooperatively
    float s1 = 0.f, s2 = 0.f;
    for (int p = threadIdx.x; p < ep.ln_parts; p += blockDim.x) {
      const float2 v = *reinterpret_cast<const float2*>(ep.ln_partial + (static_cast<long>(p) * M + row) * 2);
      s1 += v.x; s2 += v.y;
    }
    s1 = warp_sum(s1); s2 = warp_sum(s2);
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = s1; red[1][threadIdx.x >> 5] = s2; }
    __syncthreads();
    s1 = s2 = 0.f;
    for (int i = 0; i < 8; ++i) { s1 += red[0][i]; s2 += red[1][i]; }
    mu = s1 / ep.ln_dim;
    rs = rsqrtf(fmaxf(s2 / ep.ln_dim - mu * mu, 0.f) + ep.ln_eps);
  } else {
    load_ln_stats(ep, row, M, mu, rs);
  }
  const int t = blockIdx.y;
  const int col = t * kBlockN + threadIdx.x;
  const long slab = static_cast<long>(geo.m_pad) * N;
  float x = 0.f;
  if (col < N) {
    const float* w = geo.split_ws + static_cast<long>(row) * N + col;
    for (int p = 0; p < pieces; ++p) x += w[p * slab];
    if (ep.ln_colsum) x = rs * (x - mu * ep.ln_colsum[col]);
    if (ep.bias) x += ep.bias[col];
    if (epi == EPI_STORE_BF16) {
      if (ep.colscale) x *= ep.colscale[col];
      reinterpret_cast<__nv_bfloat16*>(ep.out)[static_cast<long>(row) * ep.ldo + col] = __float2bfloat16(x);
    } else {
      if (ep.gamma) x *= ep.gamma[col];
      if (ep.resid) x += ep.resid[static_cast<long>(row) * ep.ldr + col];
      reinterpret_cast<float*>(ep.out)[static_cast<long>(row) * ep.ldo + col] = x;
      if (ep.out_bf16) reinterpret_cast<__nv_bfloat16*>(ep.out_bf16)[static_cast<long>(row) * ep.ldo_bf16 + col] = __float2bfloat16(x);
    }
  }
  if (ep.stats_out != nullptr) {
    const float s1 = warp_sum(x), s2 = warp_sum(x * x);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = s1; red[1][threadIdx.x >> 5] = s2; }
    __syncthreads();
    if (threadIdx.x == 0) {
      float a = 0.f, b = 0.f;
      for (int i = 0; i < 8; ++i) { a += red[0][i]; b += red[1][i]; }
      *reinterpret_cast<float2*>(ep.stats_out + (static_cast<long>(t) * M + row) * 2) = make_float2(a, b);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess) {
      fn = reinterpret_cast<PFN_encodeTiled>(p);
    }
  });
  return fn;
}

// 2D bf16 row-major [rows, cols] with row pitch ld (elements); box = 64 cols x box_rows, 128B swizzle.
int make_tmap_bf16_2d(CUtensorMap* out, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld,
                      uint32_t box_rows) {
  PFN_encodeTiled enc = get_encode_fn();
  if (enc == nullptr) return OPB_ERR_CUDA;
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0 || (ld * 2) % 16 != 0) return OPB_ERR_INVALID;
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {ld * 2};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(kBlockK), box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), gdim, gstride, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? OPB_OK : OPB_ERR_CUDA;
}

// 2D fp32 row-major [rows, cols] with row pitch ld (elements); box = 32 cols (128 bytes) x box_rows, 128B swizzle.
static int make_tmap_f32_2d(CUtensorMap* out, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
  PFN_encodeTiled enc = get_encode_fn();
  if (enc == nullptr) return OPB_ERR_CUDA;
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0 || (ld * 4) % 16 != 0) return OPB_ERR_INVALID;
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {ld * 4};
  cuuint32_t box[2] = {32, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(ptr), gdim, gstride, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? OPB_OK : OPB_ERR_CUDA;
}

// 3D view of the A operand: dims {k_inner, taps, rows}; element (c, j, r) lives at ptr + r*row_stride + j*tap_stride + c.
// A plain [rows, K] matrix is the taps == 1 case.  box = 64 x 1 x box_rows, 128B swizzle (same smem image as 2D).
int make_tmap_bf16_3d(CUtensorMap* out, const void* ptr, uint64_t k_inner, uint64_t taps, uint64_t tap_stride,
                      uint64_t rows, uint64_t row_stride, uint32_t box_rows) {
  PFN_encodeTiled enc = get_encode_fn();
  if (enc == nullptr) return OPB_ERR_CUDA;
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0 || (tap_stride * 2) % 16 != 0 || (row_stride * 2) % 16 != 0)
    return OPB_ERR_INVALID;
  cuuint64_t gdim[3] = {k_inner, taps, rows};
  cuuint64_t gstride[2] = {tap_stride * 2, row_stride * 2};
  cuuint32_t box[3] = {static_cast<cuuint32_t>(kBlockK), 1, box_rows};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), gdim, gstride, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? OPB_OK : OPB_ERR_CUDA;
}

// 3D view of a batch of row-major matrices: dims {cols, rows, batches}; element (c, r, b) lives at
// ptr + b*batch_stride + r*ld + c.  box = 64 cols x box_rows x 1, 128B swizzle; rows >= `rows` of a box are zero-filled,
// so a box never reads into the next matrix of the batch.
int make_tmap_bf16_batched(CUtensorMap* out, const void* ptr, uint64_t cols, uint64_t rows, uint64_t ld, uint64_t batches,
                           uint64_t batch_stride, uint32_t box_rows) {
  PFN_encodeTiled enc = get_encode_fn();
  if (enc == nullptr) return OPB_ERR_CUDA;
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0 || (ld * 2) % 16 != 0 || (batch_stride * 2) % 16 != 0)
    return OPB_ERR_INVALID;
  cuuint64_t gdim[3] = {cols, rows, batches};
  cuuint64_t gstride[2] = {ld * 2, batch_stride * 2};
  cuuint32_t box[3] = {static_cast<cuuint32_t>(kBlockK), box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), gdim, gstride, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? OPB_OK : OPB_ERR_CUDA;
}

// The kernel of path kPath.  `to` holds its tensor maps: none (kDirect), the bf16 output (kTmaBf16), or the residual, the
// fp32 output and the bf16 copy (kResidRing).
template <int EPI, OutPath kPath>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap* to, const GemmEpilogue& ep,
                       const GemmGeom& geo, cudaStream_t stream) {
  constexpr bool kTmaOut = kPath == OutPath::kTmaBf16;
  constexpr int smem = kTmaOut ? kSmemBytesTmaOut : kSmemBytes;
  const void* kern;
  if constexpr (kTmaOut) kern = reinterpret_cast<const void*>(gemm_bf16_tma_out_kernel<EPI>);
  else if constexpr (kPath == OutPath::kResidRing) kern = reinterpret_cast<const void*>(gemm_bf16_resid_tma_kernel<EPI>);
  else kern = reinterpret_cast<const void*>(gemm_bf16_kernel<EPI>);
  static int resident = 0;   // CTAs resident at once over the whole GPU
  if (resident == 0) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
      return OPB_ERR_CUDA;
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kThreads, smem) != cudaSuccess || per_sm < 1)
      return OPB_ERR_CUDA;
    resident = per_sm * sm_count();
  }
  const int pieces = geo.kb_per_piece > 0 ? (geo.num_k_blocks + geo.kb_per_piece - 1) / geo.kb_per_piece : 1;
  const long units = static_cast<long>((geo.M + kBlockM - 1) / kBlockM) * ((geo.N + kBlockN - 1) / kBlockN) * geo.groups * pieces;
  const unsigned grid = static_cast<unsigned>(units < resident ? units : resident);
  if constexpr (kTmaOut) gemm_bf16_tma_out_kernel<EPI><<<grid, kThreads, smem, stream>>>(ta, tb, to[0], ep, geo);
  else if constexpr (kPath == OutPath::kResidRing)
    gemm_bf16_resid_tma_kernel<EPI><<<grid, kThreads, smem, stream>>>(ta, tb, to[0], to[1], to[2], ep, geo);
  else gemm_bf16_kernel<EPI><<<grid, kThreads, smem, stream>>>(ta, tb, ep, geo);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

// `to` != nullptr: the tensor maps of the TMA-store kernels (the bf16 output for the bf16 epilogues, see tma_out_applies;
// the residual, fp32 output and bf16 copy for EPI_RESID_F32, see resid_ring_applies)
static int dispatch_gemm(int epi, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap* to, const GemmEpilogue& ep,
                         const GemmGeom& geo, cudaStream_t stream) {
  constexpr OutPath D = OutPath::kDirect, T = OutPath::kTmaBf16;
  if (to != nullptr) {
    switch (epi) {
      case EPI_STORE_BF16: return launch_gemm<EPI_STORE_BF16, T>(ta, tb, to, ep, geo, stream);
      case EPI_GELU_BF16: return launch_gemm<EPI_GELU_BF16, T>(ta, tb, to, ep, geo, stream);
      case EPI_GEGLU_BF16: return launch_gemm<EPI_GEGLU_BF16, T>(ta, tb, to, ep, geo, stream);
      case EPI_RESID_F32: return launch_gemm<EPI_RESID_F32, OutPath::kResidRing>(ta, tb, to, ep, geo, stream);
      default: return OPB_ERR_INVALID;
    }
  }
  switch (epi) {
    case EPI_STORE_BF16: return launch_gemm<EPI_STORE_BF16, D>(ta, tb, nullptr, ep, geo, stream);
    case EPI_GELU_BF16: return launch_gemm<EPI_GELU_BF16, D>(ta, tb, nullptr, ep, geo, stream);
    case EPI_GEGLU_BF16: return launch_gemm<EPI_GEGLU_BF16, D>(ta, tb, nullptr, ep, geo, stream);
    case EPI_RESID_F32: return launch_gemm<EPI_RESID_F32, D>(ta, tb, nullptr, ep, geo, stream);
    case EPI_STORE_F32: return launch_gemm<EPI_STORE_F32, D>(ta, tb, nullptr, ep, geo, stream);
    case EPI_LSE_PARTIAL: return launch_gemm<EPI_LSE_PARTIAL, D>(ta, tb, nullptr, ep, geo, stream);
    case EPI_SOFTMAX_GRAD: return launch_gemm<EPI_SOFTMAX_GRAD, D>(ta, tb, nullptr, ep, geo, stream);
    default: return OPB_ERR_INVALID;
  }
}

// The bf16 epilogues store through shared memory and TMA (gemm_bf16_tma_out_kernel) when the output is one plain row-major
// bf16 matrix a tensor map can describe: no split-K (its pieces store fp32 slabs), one group (the 256 columns of a grouped-
// window tile would run into the next group's columns), no row remapping, a 16-byte aligned base and row pitch, and a pitch no
// smaller than the row.  Every other call keeps the direct-store kernel.
static bool tma_out_applies(int epi, const GemmEpilogue& ep, const GemmGeom& geo, long out_cols) {
  return (epi == EPI_STORE_BF16 || epi == EPI_GELU_BF16 || epi == EPI_GEGLU_BF16) && geo.kb_per_piece == 0 && geo.groups == 1 &&
         ep.out_group == 0 && (reinterpret_cast<uintptr_t>(ep.out) & 15) == 0 && (ep.ldo * 2) % 16 == 0 && ep.ldo >= out_cols;
}

// EPI_RESID_F32 loads its residual into the stage ring and stores its results with TMA (gemm_bf16_resid_tma_kernel) when the
// residual, the fp32 output and the bf16 copy (if any) are each one plain row-major [M, N] matrix a tensor map can describe:
// no split-K, one group, no row remapping, no residual period, 16-byte aligned bases and row pitches, pitches no smaller than
// the row.  Every other call (the small-M split-K path, the adapters' remapped rows, misaligned operands) keeps
// gemm_bf16_kernel.  Updating the residual in place (resid == out) is safe: a chunk is loaded whole before any of it is
// stored, and tiles are disjoint.
static bool resid_ring_applies(int epi, const GemmEpilogue& ep, const GemmGeom& geo) {
  auto plain = [&](const void* p, long ld, int esz) {
    return (reinterpret_cast<uintptr_t>(p) & 15) == 0 && (ld * esz) % 16 == 0 && ld >= geo.N;
  };
  return epi == EPI_RESID_F32 && geo.kb_per_piece == 0 && geo.groups == 1 && ep.out_group == 0 && ep.resid_period == 0 &&
         ep.resid != nullptr && plain(ep.resid, ep.ldr, 4) && plain(ep.out, ep.ldo, 4) &&
         (ep.out_bf16 == nullptr || plain(ep.out_bf16, ep.ldo_bf16, 2));
}

// Bytes [begin, end) spanned by rows lo..hi of a row-major matrix with pitch ld and `cols` columns of `esz` bytes.
struct ByteSpan {
  const char* begin;
  const char* end;
};
static ByteSpan row_span(const void* p, long lo, long hi, long ld, long cols, int esz) {
  const char* c = static_cast<const char*>(p);
  return {c + lo * ld * esz, c + (hi * ld + cols) * esz};
}
static bool spans_meet(const ByteSpan& a, const ByteSpan& b) { return a.begin < b.end && b.begin < a.end; }

// The EPI_RESID_F32 epilogue loads a batch of residual values before it stores the outputs of that batch (see epilogue()).
// That is only correct if no output store lands on a residual element that is read for another output element: `resid`
// either lies apart from both outputs, or it is the fp32 output itself with the same pitch and row mapping (the in-place
// update of the residual stream).
static bool resid_aliasing_ok(const GemmEpilogue& ep, int M, long cols) {
  if (ep.resid == nullptr) return true;
  // output rows of rows 0..M-1: the mapping is linear in the group index and the row inside the group, so its extremes are
  // at the corners of that grid
  auto out_row = [&](long m) {
    return ep.out_group > 0 ? (m / ep.out_group) * ep.out_group_stride + m % ep.out_group + ep.out_row_offset : m;
  };
  const long g = ep.out_group > 0 ? ep.out_group : M, last = M - 1, q = last / g;
  const long corners[5] = {0, (g < M ? g : M) - 1, q * g, last, q > 0 ? q * g - 1 : 0};
  long lo = out_row(0), hi = lo;
  for (long m : corners) {
    lo = out_row(m) < lo ? out_row(m) : lo;
    hi = out_row(m) > hi ? out_row(m) : hi;
  }
  long rlo = lo, rhi = hi;
  if (ep.resid_period > 0) {
    rlo = ep.resid_row_offset;
    rhi = rlo + (ep.resid_period < M ? ep.resid_period : M) - 1;
  }
  const ByteSpan res = row_span(ep.resid, rlo, rhi, ep.ldr, cols, 4);
  if (ep.out_bf16 != nullptr && spans_meet(res, row_span(ep.out_bf16, lo, hi, ep.ldo_bf16, cols, 2))) return false;
  if (!spans_meet(res, row_span(ep.out, lo, hi, ep.ldo, cols, 4))) return true;
  return ep.resid == ep.out && ep.ldr == ep.ldo && ep.resid_period == 0;
}

static GemmGeom plain_geom(int M, int N, int K) {
  GemmGeom geo;
  geo.M = M; geo.N = N; geo.K = K;
  geo.num_k_blocks = (K + kBlockK - 1) / kBlockK;
  geo.kb_inner = geo.num_k_blocks;      // one "tap": the inner coordinate never wraps
  geo.groups = 1;
  geo.a_group_c0 = 0;
  geo.b_group_rows = 0;
  geo.a_mn = geo.b_mn = 0;
  geo.kb_per_piece = 0;
  geo.m_pad = 0;
  geo.split_ws = nullptr;
  return geo;
}

int gemm_bf16(const void* A, int lda, const void* B, int ldb, int M, int N, int K, int epi, const GemmEpilogue& ep,
              int cta_group, cudaStream_t stream) {
  if (M <= 0 || N <= 0 || K <= 0) return OPB_ERR_INVALID;
  if (K % 8 != 0 || N % 8 != 0 || lda % 8 != 0 || ldb % 8 != 0) return OPB_ERR_INVALID;
  if (epi == EPI_GEGLU_BF16 && N % kBlockN != 0) return OPB_ERR_INVALID;
  if (cta_group < 0 || cta_group > 2) return OPB_ERR_INVALID;
  if (epi == EPI_RESID_F32 && !resid_aliasing_ok(ep, M, N)) return OPB_ERR_INVALID;
  GemmGeom geo = plain_geom(M, N, K);
  // Small-M split-K (a handful of texts through the 4B stack): M <= 256 gives N / 256 x 1-2 tiles, so a few CTAs would stream
  // the whole weight while the other SMs idle.  With a workspace, the fp32-residual and the plain bf16-store GEMMs instead split
  // their K range over the idle SMs and finish in gemm_split_epilogue_kernel.
  const int m_tiles = (M + kBlockM - 1) / kBlockM, n_tiles = (N + kBlockN - 1) / kBlockN;
  const bool split_ok = (epi == EPI_RESID_F32 || (epi == EPI_STORE_BF16 && ep.stats_out == nullptr)) && ep.workspace != nullptr &&
                        ep.out_group == 0 && ep.resid_period == 0 && M <= 2 * kBlockM && geo.num_k_blocks >= 8;
  int pieces = 1;
  if (split_ok) {
    const long slab_bytes = static_cast<long>(m_tiles) * kBlockM * N * 4;
    pieces = sm_count() / (m_tiles * n_tiles);
    if (pieces > geo.num_k_blocks / 2) pieces = geo.num_k_blocks / 2;
    if (pieces > ep.workspace_bytes / slab_bytes) pieces = static_cast<int>(ep.workspace_bytes / slab_bytes);
    if (pieces >= 2) {
      geo.kb_per_piece = (geo.num_k_blocks + pieces - 1) / pieces;
      pieces = (geo.num_k_blocks + geo.kb_per_piece - 1) / geo.kb_per_piece;
      geo.m_pad = m_tiles * kBlockM;
      geo.split_ws = reinterpret_cast<float*>(ep.workspace);
    }
  }
  CUtensorMap ta, tb;
  int rc = make_tmap_bf16_3d(&ta, A, K, 1, lda, M, lda, kBlockM);
  if (rc != OPB_OK) return rc;
  rc = make_tmap_bf16_2d(&tb, B, N, K, ldb, kBlockN);
  if (rc != OPB_OK) return rc;
  const long out_cols = epi == EPI_GEGLU_BF16 ? N / 2 : N;
  CUtensorMap to[3];
  const bool tma_out = tma_out_applies(epi, ep, geo, out_cols);
  const bool ring = resid_ring_applies(epi, ep, geo);
  if (tma_out && (rc = make_tmap_bf16_2d(&to[0], ep.out, M, out_cols, ep.ldo, 64)) != OPB_OK) return rc;
  if (ring) {
    if ((rc = make_tmap_f32_2d(&to[0], ep.resid, M, N, ep.ldr, kBlockM)) != OPB_OK) return rc;
    if ((rc = make_tmap_f32_2d(&to[1], ep.out, M, N, ep.ldo, 64)) != OPB_OK) return rc;
    to[2] = to[1];   // (not read without a bf16 copy)
    if (ep.out_bf16 != nullptr && (rc = make_tmap_bf16_2d(&to[2], ep.out_bf16, M, N, ep.ldo_bf16, 64)) != OPB_OK) return rc;
  }
  rc = dispatch_gemm(epi, ta, tb, tma_out || ring ? to : nullptr, ep, geo, stream);
  if (rc != OPB_OK || geo.kb_per_piece == 0) return rc;
  gemm_split_epilogue_kernel<<<dim3(M, n_tiles), 256, 0, stream>>>(ep, geo, pieces, epi);
  return cudaGetLastError() == cudaSuccess ? OPB_OK : OPB_ERR_CUDA;
}

// C[M, N] = epilogue(A . B^T) with either operand given MN-major (see GemmGeom::a_mn): A as [K, M] row-major (pitch lda), B as
// [K, N] row-major (pitch ldb).  K may be any length (TMA zero-fills past the last row); STORE epilogues only.
int gemm_bf16_t(const void* A, int lda, int a_mn, const void* B, int ldb, int b_mn, int M, int N, int K, int epi,
                const GemmEpilogue& ep, int cta_group, cudaStream_t stream) {
  if (M <= 0 || N <= 0 || K <= 0 || lda % 8 != 0 || ldb % 8 != 0 || N % 8 != 0) return OPB_ERR_INVALID;
  if (epi != EPI_STORE_BF16 && epi != EPI_STORE_F32) return OPB_ERR_INVALID;
  if ((!a_mn && K % 8 != 0) || (!b_mn && K % 8 != 0) || (a_mn && M % 8 != 0)) return OPB_ERR_INVALID;
  if (cta_group < 0 || cta_group > 2) return OPB_ERR_INVALID;
  GemmGeom geo = plain_geom(M, N, K);
  geo.a_mn = a_mn ? 1 : 0;
  geo.b_mn = b_mn ? 1 : 0;
  CUtensorMap ta, tb;
  int rc = a_mn ? make_tmap_bf16_2d(&ta, A, K, M, lda, 64) : make_tmap_bf16_3d(&ta, A, K, 1, lda, M, lda, kBlockM);
  if (rc != OPB_OK) return rc;
  rc = b_mn ? make_tmap_bf16_2d(&tb, B, K, N, ldb, 64) : make_tmap_bf16_2d(&tb, B, N, K, ldb, kBlockN);
  if (rc != OPB_OK) return rc;
  CUtensorMap to;
  const bool tma_out = tma_out_applies(epi, ep, geo, N);
  if (tma_out && (rc = make_tmap_bf16_2d(&to, ep.out, M, N, ep.ldo, 64)) != OPB_OK) return rc;
  return dispatch_gemm(epi, ta, tb, tma_out ? &to : nullptr, ep, geo, stream);
}

int gemm_bf16_grouped_window(const void* X, const void* W, int rows, int groups, int c_pad, int taps, int n_per_group,
                             int epi, const GemmEpilogue& ep, cudaStream_t stream) {
  if (rows <= 0 || groups <= 0 || taps <= 0 || n_per_group <= 0) return OPB_ERR_INVALID;
  if (c_pad % kBlockK != 0 || n_per_group % 8 != 0 || n_per_group > kBlockN) return OPB_ERR_INVALID;
  if (epi == EPI_GEGLU_BF16 || epi == EPI_LSE_PARTIAL || epi == EPI_SOFTMAX_GRAD) return OPB_ERR_INVALID;
  if (epi == EPI_RESID_F32 && !resid_aliasing_ok(ep, rows, static_cast<long>(groups) * n_per_group)) return OPB_ERR_INVALID;
  GemmGeom geo = plain_geom(rows, n_per_group, taps * c_pad);
  geo.kb_inner = c_pad / kBlockK;
  geo.num_k_blocks = taps * geo.kb_inner;
  geo.groups = groups;
  geo.a_group_c0 = c_pad;
  geo.b_group_rows = n_per_group;
  const long row_stride = static_cast<long>(groups) * c_pad;
  CUtensorMap ta, tb;
  // dims {groups*c_pad, taps, rows}: tap j of output row r reads input row r + j (tap stride == row stride)
  int rc = make_tmap_bf16_3d(&ta, X, row_stride, taps, row_stride, rows, row_stride, kBlockM);
  if (rc != OPB_OK) return rc;
  rc = make_tmap_bf16_2d(&tb, W, static_cast<uint64_t>(groups) * n_per_group, geo.K, geo.K, kBlockN);
  if (rc != OPB_OK) return rc;
  return dispatch_gemm(epi, ta, tb, nullptr, ep, geo, stream);
}

}  // namespace opb
