// Generic bf16 wgmma GEMM for sm_90a:  D[M,N] (+)= A[M,K] * B[N,K]^T, fp32 accumulation in registers.
//
// One CTA computes one 128 x BLOCK_N output tile (optionally one K-split of it).  Warp roles:
//   warpgroups 0-1 : consumers, 64 accumulator rows each (wgmma m64nNk16, one K block in flight while the next is issued)
//   warp 8 : TMA producer (one elected lane)   global -> 128B-swizzled shared memory ring
//   After the main loop the consumers stage the fp32 tile in the (then idle) operand ring and run the fused
//   bias / GELU / GELU' / residual / fp32-atomic (split-K) tail on it, one accumulator row per thread.  Two CTAs share an SM
//   (shared memory and registers are sized for it), so one CTA's epilogue runs under the other's main loop.
// Operands may be K-major (reduction dim contiguous) or MN-major (reduction dim strided; used by the
// weight-gradient GEMMs), selected per operand.  All the "view" tricks of the WavLM path (strided
// Conv1d as an overlapping-row view, grouped pos_conv taps, per-batch tiles) are expressed on the host
// as <=4-D TMA tensor maps plus a small integer matrix that maps tile indices to TMA coordinates.
// Row GEMMs (K-major, bf16 out) with N >= 256 run the persistent 128 x 256 gemm_ws_kernel further down instead, and weight
// gradients with K >= 256 its stream-K sibling gemm_ws_wgrad_kernel.
#pragma once
#include "ptx.cuh"
#include "ws_epilogue.cuh"

namespace b200 {

struct EpiTensor {
  void* p;
  long long bs;  // batch stride (elements)
  long long ld;  // row stride (elements)
};

enum : int {
  EPI_GELU = 1,      // out = gelu(acc + bias); if out2.p: out2 = acc + bias (pre-activation)
  EPI_DGELU = 2,     // acc *= gelu'(aux)
  EPI_OUT_F32 = 4,   // out is fp32
  EPI_ATOMIC = 8,    // fp32 atomicAdd into out (split-K / accumulation)
  EPI_COLSUM = 16,   // atomically accumulate column sums of the final value into colsum[col] (bias grads)
  EPI_ACCUM = 32,    // fp32 out += value, non-atomic (single writer per element: split-K disabled)
  EPI_GELU_STORE_GRAD = 64,  // with EPI_GELU: out2 receives gelu'(acc + bias) instead of the pre-activation
  EPI_AUX_IS_GRAD = 128,     // with EPI_DGELU: aux already holds gelu'(.) (written by an EPI_GELU_STORE_GRAD forward): acc *= aux
};

// variables the coordinate matrices multiply: {1, m0, mb, n_tile, k0, kbatch, kb, sub}
constexpr int kCoordVars = 8;

struct GemmParams {
  int m_rows;            // valid rows per batch
  int m_tiles_per_batch; // ceil over m_tile_stride
  int m_tile_stride;     // rows between consecutive M tiles (128 normally)
  int m_tile_valid;      // max valid rows per tile (128 normally; Cg for grouped wgrad)
  int m_tiles;           // M tiles over all batches (persistent kernel)
  int n_total;           // valid output columns
  int n_out_stride;      // output column stride per N tile
  int n_tile_valid;      // max valid columns per tile
  int k_blocks;          // total number of 64-wide K blocks
  int k_blocks_per_batch;  // >0: K iterates (batch, row-block); 0: plain
  int k_blocks_per_split;
  int ca[4][kCoordVars];
  int cb[4][kCoordVars];
  int flags;
  const float* bias;     // [n] fp32 or null
  float* colsum;         // [n] fp32 or null (EPI_COLSUM)
  EpiTensor out, out2, aux, res1, res2;
  // ragged batches (null = every row counts).  m_valid[b]: rows of batch b that hold real frames -- an M tile that starts at or
  // beyond it is not computed, its output rows are written as zeros.  k_valid[b] (weight gradients, K iterates over (batch, row
  // block)): row blocks that start at or beyond it are not loaded / multiplied (their gradient rows are zero by construction:
  // nothing downstream of a padded frame reaches the loss).
  const int* m_valid;
  const int* k_valid;
};

template <int BLOCK_N>
struct GemmCfg {
  static constexpr int kStages = (BLOCK_N <= 64) ? 4 : 3;
  static constexpr int kABytes = 128 * 128;          // 128 rows x 64 bf16
  static constexpr int kBBytes = BLOCK_N * 128;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kAccPitch = BLOCK_N + 8;      // fp32 staging row (floats): conflict-free fragment stores
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024;
  static constexpr int kThreads = 288;
  static_assert(128 * kAccPitch * 4 <= kStages * kStageBytes, "accumulator staging must fit in the operand ring");
  static_assert(2 * (kSmemBytes + 1024) <= 233472, "two CTAs per SM");
};

__device__ __forceinline__ int coord_dot(const int* row, const int* v) {
  int s = 0;
#pragma unroll
  for (int i = 0; i < kCoordVars; ++i) s += row[i] * v[i];
  return s;
}

// Per-thread row pointers of the epilogue tensors (computed once per tile: the epilogue is issue-bound -- one warp per
// scheduler -- so every instruction removed from the per-element path is wall-clock time).
struct EpiRow {
  __nv_bfloat16* out_bf;
  float* out_f32;
  __nv_bfloat16* out2;
  const __nv_bfloat16* aux;
  const __nv_bfloat16* res1;
  const __nv_bfloat16* res2;
};
__device__ __forceinline__ EpiRow make_epi_row(const GemmParams& p, int mb, long long row) {
  EpiRow e;
  e.out_bf = static_cast<__nv_bfloat16*>(p.out.p) + mb * p.out.bs + row * p.out.ld;
  e.out_f32 = static_cast<float*>(p.out.p) + mb * p.out.bs + row * p.out.ld;
  e.out2 = p.out2.p ? static_cast<__nv_bfloat16*>(p.out2.p) + mb * p.out2.bs + row * p.out2.ld : nullptr;
  e.aux = p.aux.p ? static_cast<const __nv_bfloat16*>(p.aux.p) + mb * p.aux.bs + row * p.aux.ld : nullptr;
  e.res1 = p.res1.p ? static_cast<const __nv_bfloat16*>(p.res1.p) + mb * p.res1.bs + row * p.res1.ld : nullptr;
  e.res2 = p.res2.p ? static_cast<const __nv_bfloat16*>(p.res2.p) + mb * p.res2.bs + row * p.res2.ld : nullptr;
  return e;
}
__device__ __forceinline__ void add_bf16x8(float* a8, const __nv_bfloat16* src) {
  const uint4 w = *reinterpret_cast<const uint4*>(src);
  const uint32_t wu[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 f = unpack_bf16x2(wu[j]);
    a8[2 * j] += f.x;
    a8[2 * j + 1] += f.y;
  }
}
__device__ __forceinline__ uint4 pack_bf16x8(const float* a8) {
  uint4 w;
  w.x = pack_bf16x2(a8[0], a8[1]); w.y = pack_bf16x2(a8[2], a8[3]);
  w.z = pack_bf16x2(a8[4], a8[5]); w.w = pack_bf16x2(a8[6], a8[7]);
  return w;
}

// One 32-column chunk of the fused epilogue for this thread's accumulator row (src = the chunk in the fp32 staging tile).
__device__ __forceinline__ void epilogue_chunk32(const GemmParams& p, const EpiRow& e, const float* src, int c0, int n_valid,
                                                 int col_base, bool row_ok, int lane) {
  const int flags = p.flags;
  float acc[32];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 v = reinterpret_cast<const float4*>(src)[j];
    acc[4 * j] = v.x; acc[4 * j + 1] = v.y; acc[4 * j + 2] = v.z; acc[4 * j + 3] = v.w;
  }
  const bool full = (c0 + 32 <= n_valid);  // warp-uniform
  if (p.bias != nullptr) {
    const float* bp = p.bias + col_base + c0;
    if (full) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 b4 = __ldg(reinterpret_cast<const float4*>(bp) + j);
        acc[4 * j] += b4.x; acc[4 * j + 1] += b4.y; acc[4 * j + 2] += b4.z; acc[4 * j + 3] += b4.w;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (c0 + j < n_valid) acc[j] += __ldg(bp + j);
    }
  }
  if (row_ok) {
    const int col0 = col_base + c0;
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      if (!full && (c0 + g * 8 >= n_valid)) break;
      const int col = col0 + g * 8;
      float* a8 = acc + g * 8;
      if (flags & EPI_GELU) {
        if (flags & EPI_GELU_STORE_GRAD) {
          float g8[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) a8[j] = gelu_with_grad_f(a8[j], g8[j]);
          if (e.out2 != nullptr) *reinterpret_cast<uint4*>(e.out2 + col) = pack_bf16x8(g8);
        } else {
          if (e.out2 != nullptr) *reinterpret_cast<uint4*>(e.out2 + col) = pack_bf16x8(a8);
#pragma unroll
          for (int j = 0; j < 8; ++j) a8[j] = gelu_f(a8[j]);
        }
      }
      if (flags & EPI_DGELU) {
        const uint4 w = *reinterpret_cast<const uint4*>(e.aux + col);
        const uint32_t wu[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = unpack_bf16x2(wu[j]);
          a8[2 * j] *= (flags & EPI_AUX_IS_GRAD) ? f.x : gelu_grad_f(f.x);
          a8[2 * j + 1] *= (flags & EPI_AUX_IS_GRAD) ? f.y : gelu_grad_f(f.y);
        }
      }
      if (e.res1 != nullptr) add_bf16x8(a8, e.res1 + col);
      if (e.res2 != nullptr) add_bf16x8(a8, e.res2 + col);
      if (flags & EPI_OUT_F32) {
        float* o = e.out_f32 + col;
        if (flags & EPI_ATOMIC) {
          // 128-bit vector reductions (REDG.E.ADD.F32x4): the split-K epilogue is bound by LSU issue, not bytes
          red_add_f32x4(o, a8[0], a8[1], a8[2], a8[3]);
          red_add_f32x4(o + 4, a8[4], a8[5], a8[6], a8[7]);
        } else if (flags & EPI_ACCUM) {
          float4 o0 = *reinterpret_cast<float4*>(o), o1 = *reinterpret_cast<float4*>(o + 4);
          o0.x += a8[0]; o0.y += a8[1]; o0.z += a8[2]; o0.w += a8[3];
          o1.x += a8[4]; o1.y += a8[5]; o1.z += a8[6]; o1.w += a8[7];
          *reinterpret_cast<float4*>(o) = o0;
          *reinterpret_cast<float4*>(o + 4) = o1;
        } else {
          *reinterpret_cast<float4*>(o) = make_float4(a8[0], a8[1], a8[2], a8[3]);
          *reinterpret_cast<float4*>(o + 4) = make_float4(a8[4], a8[5], a8[6], a8[7]);
        }
      } else {
        *reinterpret_cast<uint4*>(e.out_bf + col) = pack_bf16x8(a8);
      }
    }
  }
  if (flags & EPI_COLSUM) {
    // column sums of the stored values over this warp's 32 rows: transpose-reduce, then one atomic per column
    float cv[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      float t = row_ok ? acc[j] : 0.0f;
      if (!(flags & EPI_OUT_F32)) t = __bfloat162float(__float2bfloat16_rn(t));
      cv[j] = t;
    }
    const float csum = warp_colsum32(cv, lane);
    if ((c0 + lane) < n_valid) atomicAdd(p.colsum + col_base + c0 + lane, csum);
  }
}


template <int N, bool TA, bool TB>
__device__ __forceinline__ void wgmma_tile(float* acc, uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (N == 64) wgmma_m64n64k16<TA ? 1 : 0, TB ? 1 : 0>(acc, da, db, scale_d);
  else wgmma_m64n128k16<TA ? 1 : 0, TB ? 1 : 0>(acc, da, db, scale_d);
}

// Consumer tail shared by the GEMM kernels: the two consumer warpgroups (threads 0..255) stage their fp32 accumulators in
// shared memory (rows [64 c, 64 c + 64) of a 128 x BLOCK_N tile) and run the fused epilogue on it.  Warp ew = 0..7 owns rows
// 32 (ew & 3) .. + 31 (one per lane) and the column half ew >> 2.  Every consumer MMA must have completed before the call
// (the staging tile overlaps the operand ring).
template <int BLOCK_N>
__device__ __forceinline__ void gemm_consumer_tail(const GemmParams& p, const float* acc, float* acc_s, int mb, int m0,
                                                   int col_base, int n_valid, int m_valid) {
  constexpr int kPitch = BLOCK_N + 8;
  const int ew = threadIdx.x >> 5, lane = threadIdx.x & 31;
  named_bar_sync(1, 256);
  acc_to_smem<BLOCK_N>(acc, acc_s, kPitch, 64 * (ew >> 2));
  named_bar_sync(1, 256);
  const int r = (ew & 3) * 32 + lane;
  const EpiRow erow = make_epi_row(p, mb, static_cast<long long>(m0) + r);
#pragma unroll 1
  for (int c0 = (ew >> 2) * (BLOCK_N / 2); c0 < ((ew >> 2) + 1) * (BLOCK_N / 2); c0 += 32) {
    if (c0 >= n_valid) break;  // warp-uniform
    epilogue_chunk32(p, erow, acc_s + r * kPitch + c0, c0, n_valid, col_base, r < m_valid, lane);
  }
}

// Output rows of an M tile that holds only padded frames (ragged batch): zeros, so that padded frames stay FINITE (a NaN in a
// padded key row would survive the -inf mask as NaN * 0 in the probabilities x V product).  bf16 outputs only.
__device__ __forceinline__ void zero_dead_tile(const GemmParams& p, int mb, int m0, int col_base, int n_valid) {
  const int rows = min(p.m_tile_valid, p.m_rows - m0), c8 = n_valid / 8;
  for (int i = threadIdx.x; i < rows * c8; i += blockDim.x) {
    const long long row = static_cast<long long>(m0) + i / c8;
    const int col = col_base + (i % c8) * 8;
    *reinterpret_cast<uint4*>(static_cast<__nv_bfloat16*>(p.out.p) + mb * p.out.bs + row * p.out.ld + col) = make_uint4(0u, 0u, 0u, 0u);
    if (p.out2.p != nullptr)
      *reinterpret_cast<uint4*>(static_cast<__nv_bfloat16*>(p.out2.p) + mb * p.out2.bs + row * p.out2.ld + col) = make_uint4(0u, 0u, 0u, 0u);
  }
}

template <int BLOCK_N, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(288, 2) gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA,
                                                           const __grid_constant__ CUtensorMap tmB,
                                                           const __grid_constant__ GemmParams p) {
  pdl_launch_dependents();
  using Cfg = GemmCfg<BLOCK_N>;
  constexpr int kStages = Cfg::kStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int n_tile = blockIdx.x;
  const int mb = blockIdx.y / p.m_tiles_per_batch;
  const int m0 = (blockIdx.y % p.m_tiles_per_batch) * p.m_tile_stride;
  const int kb_begin = blockIdx.z * p.k_blocks_per_split;
  const int kb_end = min(kb_begin + p.k_blocks_per_split, p.k_blocks);
  if (kb_begin >= kb_end) return;  // uniform per CTA
  const int col_base = n_tile * p.n_out_stride;
  const int n_valid = min(p.n_tile_valid, p.n_total - col_base);

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // 1024-aligned, still a __shared__ pointer (LDS/STS, not generic)
  __shared__ uint64_t full_bar[kStages];
  __shared__ uint64_t empty_bar[kStages];

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
#pragma unroll
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);  // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();  // prologue overlapped the previous kernel's tail; global memory is touched only from here on

  if (p.m_valid != nullptr && m0 >= p.m_valid[mb]) {
    zero_dead_tile(p, mb, m0, col_base, n_valid);
    return;
  }
  // ragged weight gradients: a 64-row K block at or beyond its batch's valid rows is neither loaded nor multiplied
  auto kb_live = [&](int kb) {
    if (p.k_valid == nullptr) return true;
    const int kbatch = kb / p.k_blocks_per_batch;
    return (kb - kbatch * p.k_blocks_per_batch) * 64 < p.k_valid[kbatch];
  };

  if (warp == 8) {
    if (lane == 0) {
      // ------------------------------------------------------------ TMA producer
      int v[kCoordVars];
      v[0] = 1; v[1] = m0; v[2] = mb; v[3] = n_tile;
      int it = 0;
      for (int kb = kb_begin; kb < kb_end; ++kb) {
        if (!kb_live(kb)) continue;
        const int s = it % kStages;
        const uint32_t ph = (it / kStages) & 1;
        ++it;
        mbar_wait(&empty_bar[s], ph ^ 1);
        if (p.k_blocks_per_batch > 0) {
          v[5] = kb / p.k_blocks_per_batch;
          v[4] = (kb % p.k_blocks_per_batch) * 64;
        } else {
          v[5] = 0;
          v[4] = kb * 64;
        }
        v[6] = kb;
        uint8_t* sa = smem + s * Cfg::kStageBytes;
        uint8_t* sb = sa + Cfg::kABytes;
        mbar_expect_tx(&full_bar[s], Cfg::kStageBytes);
        if constexpr (!A_MN) {
          v[7] = 0;
          tma_load_4d(sa, &tmA, &full_bar[s], coord_dot(p.ca[0], v), coord_dot(p.ca[1], v), coord_dot(p.ca[2], v),
                      coord_dot(p.ca[3], v));
        } else {
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            v[7] = 64 * i;
            tma_load_4d(sa + i * 8192, &tmA, &full_bar[s], coord_dot(p.ca[0], v), coord_dot(p.ca[1], v),
                        coord_dot(p.ca[2], v), coord_dot(p.ca[3], v));
          }
        }
        if constexpr (!B_MN) {
          v[7] = 0;
          tma_load_4d(sb, &tmB, &full_bar[s], coord_dot(p.cb[0], v), coord_dot(p.cb[1], v), coord_dot(p.cb[2], v),
                      coord_dot(p.cb[3], v));
        } else {
#pragma unroll
          for (int i = 0; i < BLOCK_N / 64; ++i) {
            v[7] = 64 * i;
            tma_load_4d(sb + i * 8192, &tmB, &full_bar[s], coord_dot(p.cb[0], v), coord_dot(p.cb[1], v),
                        coord_dot(p.cb[2], v), coord_dot(p.cb[3], v));
          }
        }
      }
    }
  } else {
    // -------------------------------------------------------------- consumers: warpgroup c owns rows 64 c .. 64 c + 63
    const int c = warp >> 2;
    float acc[BLOCK_N / 2];  // written by the first MMA (scale_d = 0)
    int it = 0;
    for (int kb = kb_begin; kb < kb_end; ++kb) {
      if (!kb_live(kb)) continue;
      const int s = it % kStages;
      mbar_wait(&full_bar[s], (it / kStages) & 1);
      // rows 64 c.. of A: 64 rows x 128 B (K-major) or the second 64-row MN block (MN-major) -- 8 KB either way
      const uint32_t sa = smem_u32(smem + s * Cfg::kStageBytes) + c * 8192;
      const uint32_t sb = smem_u32(smem + s * Cfg::kStageBytes + Cfg::kABytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint64_t da = A_MN ? make_smem_desc_sw128(sa + k * 2048, 8192, 1024) : make_smem_desc_sw128(sa + k * 32, 16, 1024);
        const uint64_t db = B_MN ? make_smem_desc_sw128(sb + k * 2048, 8192, 1024) : make_smem_desc_sw128(sb + k * 32, 16, 1024);
        wgmma_tile<BLOCK_N, A_MN, B_MN>(acc, da, db, (it > 0 || k > 0) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<1>();  // the previous K block's MMAs have retired: its stage goes back to the producer
      if (it > 0 && lane == 0) mbar_arrive(&empty_bar[(it - 1) % kStages]);
      ++it;
    }
    wgmma_wait<0>();
    if (it == 0) {  // no live K block (ragged weight gradient): the split contributes zeros
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
    }
    gemm_consumer_tail<BLOCK_N>(p, acc, reinterpret_cast<float*>(smem), mb, m0, col_base, n_valid,
                                min(p.m_tile_valid, p.m_rows - m0));
  }
}

// ------------------------------------------------------------------------------- persistent 128 x 256 row GEMM
// D[M, N] = A[M, K] * B[N, K]^T with K-major operands and a bf16 output (b200s_gemm_rows: the layer, conv and projection GEMMs).
// One CTA per SM walks the 128 x 256 output tiles with N fastest inside a 128-row band, so the CTAs resident at any time share
// their A bands in L2 and A is read from HBM about once.  Warp roles:
//   warpgroup 0    : TMA producer (one elected lane); it hands its registers to the consumers
//   warpgroups 1-2 : consumers, 64 rows of the tile each (wgmma m64n256k16, 128 fp32 accumulators per thread)
// The producer runs ahead into the next tile while the consumers run the epilogue, so the operand ring is never epilogue staging:
// each consumer warpgroup moves 64 accumulator columns at a time into its own 16 KB buffer and applies the fused epilogue
// (epilogue_chunk32's semantics, bf16 output) row-wise, 16 lanes per 64-column row segment, so every global load and store of a
// warp covers two whole 128-byte lines.
// The epilogue's bf16 inputs (GELU' aux, residuals) are fetched with per-thread asynchronous copies into a per-warpgroup buffer
// one 64-column chunk ahead -- chunk 0 while the tile's main loop runs -- so their latency is never paid row by row.
struct WsCfg {
  static constexpr int kStages = 3;
  static constexpr int kABytes = 128 * 128;  // 128 rows x 64 bf16
  static constexpr int kBBytes = 256 * 128;  // 256 rows x 64 bf16
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kEpiBytes = 64 * 64 * 4;  // one consumer warpgroup's 64 x 64 fp32 staging chunk
  static constexpr int kPfBytes = 3 * 8 * 128 * 8;  // one consumer warpgroup's prefetched inputs: {aux, res1, res2} x 8 rows x 128 threads x 4 bf16
  static constexpr int kSmemBytes = kStages * kStageBytes + 2 * kEpiBytes + 2 * kPfBytes + 1024;
  static constexpr int kThreads = 384;
  static_assert(kSmemBytes + 1024 <= 232448, "one CTA per SM");
};

__global__ void __launch_bounds__(384, 1) gemm_ws_kernel(const __grid_constant__ CUtensorMap tmA,
                                                         const __grid_constant__ CUtensorMap tmB,
                                                         const __grid_constant__ GemmParams p) {
  pdl_launch_dependents();
  using Cfg = WsCfg;
  constexpr int kStages = Cfg::kStages;
  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;
  const int n_tiles = (p.n_total + 255) / 256;
  const int num_tiles = p.m_tiles * n_tiles;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  __shared__ uint64_t full_bar[kStages];
  __shared__ uint64_t empty_bar[kStages];

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
#pragma unroll
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);  // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();

  if (wg == 0) {
    // ------------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int mt = tile / n_tiles, n_tile = tile - mt * n_tiles;
        const int mb = mt / p.m_tiles_per_batch, m0 = (mt - mb * p.m_tiles_per_batch) * 128;
        for (int kb = 0; kb < p.k_blocks; ++kb, ++it) {
          const int s = it % kStages;
          mbar_wait(&empty_bar[s], ((it / kStages) & 1) ^ 1);
          uint8_t* sa = smem + s * Cfg::kStageBytes;
          mbar_expect_tx(&full_bar[s], Cfg::kStageBytes);
          tma_load_4d(sa, &tmA, &full_bar[s], kb * 64, m0, mb, 0);
          tma_load_4d(sa + Cfg::kABytes, &tmB, &full_bar[s], kb * 64, n_tile * 256, 0, 0);
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------- consumers: warpgroup c owns rows 64 c .. 64 c + 63
  setmaxnreg_inc<232>();
  const int c = wg - 1;
  const int t = threadIdx.x & 127, w = t >> 5;
  float* stage = reinterpret_cast<float*>(smem + kStages * Cfg::kStageBytes + c * Cfg::kEpiBytes);
  uint2* pf = reinterpret_cast<uint2*>(smem + kStages * Cfg::kStageBytes + 2 * Cfg::kEpiBytes + c * Cfg::kPfBytes);
  const int cq = ws_lane_col(lane);  // epilogue: this lane's 4 columns of a 64-column chunk
  const EpiTensor* const pf_src[3] = {&p.aux, &p.res1, &p.res2};
  float acc[128];                  // written by each tile's first MMA (scale_d = 0)
  int it = 0;
  for (int tile = blockIdx.x; tile < p.m_tiles * n_tiles; tile += gridDim.x) {
    const int mt = tile / n_tiles, n_tile = tile - mt * n_tiles;
    const int mb = mt / p.m_tiles_per_batch, m0 = (mt - mb * p.m_tiles_per_batch) * 128;
    const int col_base = n_tile * 256;
    const int n_valid = min(256, p.n_total - col_base);
    const int rows_here = min(128, p.m_rows - m0) - 64 * c;  // valid rows of this warpgroup's half (may be <= 0)
    // the 4 columns x 8 rows of chunk j's epilogue inputs that this thread reads are copied into its own slots pf[(q, i), t]
    auto prefetch = [&](int j) {
      const int cl = 64 * j + cq;
      if (cl < n_valid) {
#pragma unroll
        for (int q = 0; q < 3; ++q) {
          const EpiTensor& e = *pf_src[q];
          if (e.p == nullptr) continue;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int r = ws_chunk_row(w, i, lane);
            if (r < rows_here)
              cp_async_8(pf + (q * 8 + i) * 128 + t, static_cast<const __nv_bfloat16*>(e.p) + mb * e.bs +
                                                         (static_cast<long long>(m0) + 64 * c + r) * e.ld + col_base + cl);
          }
        }
      }
      cp_async_commit();
    };
    prefetch(0);
    for (int kb = 0; kb < p.k_blocks; ++kb, ++it) {
      const int s = it % kStages;
      mbar_wait(&full_bar[s], (it / kStages) & 1);
      const uint32_t sa = smem_u32(smem + s * Cfg::kStageBytes) + c * 8192;  // rows 64 c .. of A: 64 rows x 128 B
      const uint32_t sb = smem_u32(smem + s * Cfg::kStageBytes + Cfg::kABytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_m64n256k16<0, 0>(acc, make_smem_desc_sw128(sa + k * 32, 16, 1024), make_smem_desc_sw128(sb + k * 32, 16, 1024),
                               (kb > 0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();  // the previous K block's MMAs have retired: its stage goes back to the producer
      if (kb > 0 && lane == 0) mbar_arrive(&empty_bar[(it - 1) % kStages]);
    }
    wgmma_wait<0>();
    if (lane == 0) mbar_arrive(&empty_bar[(it - 1) % kStages]);

    // ---- epilogue, 64 columns at a time (ws_stage_chunk)
    const int flags = p.flags;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (64 * j >= n_valid) break;  // warpgroup-uniform
      named_bar_sync(1 + c, 128);    // the previous chunk has been read out of the staging buffer
      ws_stage_chunk(acc, stage, j, w, lane);
      const int cl = 64 * j + cq;
      const bool col_ok = cl < n_valid;
      const int col = col_base + cl;
      named_bar_sync(1 + c, 128);
      float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f);
      if (p.bias != nullptr && col_ok) b4 = __ldg(reinterpret_cast<const float4*>(p.bias + col));
      float cs[4] = {0.f, 0.f, 0.f, 0.f};
      cp_async_wait_all();  // this thread's inputs of chunk j have landed
#pragma unroll 4
      for (int i = 0; i < 8; ++i) {
        const int r = ws_chunk_row(w, i, lane);
        const float4 v4 = ws_load_row(stage, r, cq);
        if (!col_ok || r >= rows_here) continue;
        float v[4] = {v4.x + b4.x, v4.y + b4.y, v4.z + b4.z, v4.w + b4.w};
        const long long row = static_cast<long long>(m0) + 64 * c + r;
        if (flags & EPI_GELU) {
          __nv_bfloat16* o2 =
              p.out2.p ? static_cast<__nv_bfloat16*>(p.out2.p) + mb * p.out2.bs + row * p.out2.ld + col : nullptr;
          if (flags & EPI_GELU_STORE_GRAD) {
            float g[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) v[k] = gelu_with_grad_f(v[k], g[k]);
            if (o2 != nullptr) *reinterpret_cast<uint2*>(o2) = pack_bf16x4(g);
          } else {
            if (o2 != nullptr) *reinterpret_cast<uint2*>(o2) = pack_bf16x4(v);
#pragma unroll
            for (int k = 0; k < 4; ++k) v[k] = gelu_f(v[k]);
          }
        }
        if (flags & EPI_DGELU) {
          const uint2 a = pf[(0 * 8 + i) * 128 + t];
          const float2 f0 = unpack_bf16x2(a.x), f1 = unpack_bf16x2(a.y);
          const float f[4] = {f0.x, f0.y, f1.x, f1.y};
#pragma unroll
          for (int k = 0; k < 4; ++k) v[k] *= (flags & EPI_AUX_IS_GRAD) ? f[k] : gelu_grad_f(f[k]);
        }
        if (p.res1.p != nullptr) add_bf16x4(v, pf[(1 * 8 + i) * 128 + t]);
        if (p.res2.p != nullptr) add_bf16x4(v, pf[(2 * 8 + i) * 128 + t]);
        *reinterpret_cast<uint2*>(static_cast<__nv_bfloat16*>(p.out.p) + mb * p.out.bs + row * p.out.ld + col) = pack_bf16x4(v);
        if (flags & EPI_COLSUM) {
#pragma unroll
          for (int k = 0; k < 4; ++k) cs[k] += __bfloat162float(__float2bfloat16_rn(v[k]));
        }
      }
      if (j < 3) prefetch(j + 1);  // this thread's slots have been read
      if (flags & EPI_COLSUM) {
        // column sums of the stored values over this warpgroup's 64 rows: lane pairs, then the 4 warps through the staging
        // buffer, then one atomic per column
#pragma unroll
        for (int k = 0; k < 4; ++k) cs[k] += __shfl_xor_sync(0xffffffffu, cs[k], 16);
        named_bar_sync(1 + c, 128);  // the chunk has been read: the buffer is free
        if (lane < 16) *reinterpret_cast<float4*>(stage + w * 64 + cq) = make_float4(cs[0], cs[1], cs[2], cs[3]);
        named_bar_sync(1 + c, 128);
        if (t < 64 && 64 * j + t < n_valid)
          atomicAdd(p.colsum + col_base + 64 * j + t, stage[t] + stage[64 + t] + stage[128 + t] + stage[192 + t]);
      }
    }
  }
}

// ------------------------------------------------------------------------ persistent 128 x 256 stream-K weight gradient
// dW[N, K] += sum over token rows of Y[row, n] X[row, k] (b200s_gemm_wgrad with K >= 256; p.m_rows = N, p.n_total = K).  Both
// operands are MN-major and the reduction runs over K blocks = (batch, 64-row block).  Warp roles, ring and staging buffers are
// gemm_ws_kernel's; a stage holds A as two 64 x 64 boxes (128 rows of dW x 64 tokens) and B as four (256 columns x 64 tokens).
// Stream-K: the (tile, live K block) iteration space, tile-major, is cut into gridDim.x equal contiguous ranges.  A CTA accumulates
// each piece of a tile in its range in registers and adds it to dW with vector fp32 reductions, row-coalesced through the staging
// buffer, so there is no fix-up pass and no tile-count quantisation.
// Walk order: the K blocks of tile t are visited rotated by rot(t) = t * Kl - (start of the range holding the tile's first block),
// Kl = live K blocks.  At step s of its range a CTA then reads K block s + d * L (mod Kl), L = range length, d = which piece of
// its tile it is working on.  The CTAs running together form a few fronts, each reading the same 64 token rows of Y and X at the
// same time, and the fronts cover disjoint K blocks over the run, so Y and X are read from HBM about once.  (Unrotated, each CTA
// would read token rows of its own, and the operands would come from HBM up to once per tile.)
// Ragged batches: only live K blocks (below k_valid) are in the iteration space, so the ranges stay equal in work.
__device__ __forceinline__ int wgrad_live_blocks(const GemmParams& p, int b) {
  return p.k_valid == nullptr ? p.k_blocks_per_batch : min(p.k_blocks_per_batch, (max(__ldg(p.k_valid + b), 0) + 63) / 64);
}

__global__ void __launch_bounds__(384, 1) gemm_ws_wgrad_kernel(const __grid_constant__ CUtensorMap tmA,
                                                               const __grid_constant__ CUtensorMap tmB,
                                                               const __grid_constant__ GemmParams p) {
  pdl_launch_dependents();
  using Cfg = WsCfg;
  constexpr int kStages = Cfg::kStages;
  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;
  const int n_tiles = (p.n_total + 255) / 256;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  __shared__ uint64_t full_bar[kStages];
  __shared__ uint64_t empty_bar[kStages];

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
#pragma unroll
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);  // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();

  const int batches = p.k_blocks / p.k_blocks_per_batch;
  int kl = 0;
  for (int b = 0; b < batches; ++b) kl += wgrad_live_blocks(p, b);
  const long long total = static_cast<long long>(p.m_tiles) * n_tiles * kl;
  const long long g_begin = blockIdx.x * total / gridDim.x, g_end = (blockIdx.x + 1) * total / gridDim.x;
  // the pieces of this CTA's range: tile t, its K blocks j0 .. j1 - 1 in walk order
  auto piece = [&](long long g, int& t, int& j0, int& j1) {
    t = static_cast<int>(g / kl);
    j0 = static_cast<int>(g - static_cast<long long>(t) * kl);
    j1 = static_cast<int>(min(static_cast<long long>(kl), j0 + (g_end - g)));
  };

  if (wg == 0) {
    // ------------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int it = 0;
      for (long long g = g_begin; g < g_end;) {
        int t, j0, j1;
        piece(g, t, j0, j1);
        g += j1 - j0;
        const int mt = t / n_tiles, n_tile = t - mt * n_tiles;
        const long long x = static_cast<long long>(t) * kl;
        const long long i0 = ((x + 1) * gridDim.x + total - 1) / total - 1;  // the range holding block 0 of tile t
        int l = j0 + static_cast<int>((x - i0 * total / gridDim.x) % kl);  // rotated live block index
        if (l >= kl) l -= kl;
        int kbatch = 0;
        while (l >= wgrad_live_blocks(p, kbatch)) l -= wgrad_live_blocks(p, kbatch++);
        for (int j = j0; j < j1; ++j, ++it) {
          const int s = it % kStages;
          mbar_wait(&empty_bar[s], ((it / kStages) & 1) ^ 1);
          uint8_t* sa = smem + s * Cfg::kStageBytes;
          uint8_t* sb = sa + Cfg::kABytes;
          mbar_expect_tx(&full_bar[s], Cfg::kStageBytes);
#pragma unroll
          for (int i = 0; i < 2; ++i) tma_load_4d(sa + i * 8192, &tmA, &full_bar[s], mt * 128 + 64 * i, l * 64, kbatch, 0);
#pragma unroll
          for (int i = 0; i < 4; ++i) tma_load_4d(sb + i * 8192, &tmB, &full_bar[s], n_tile * 256 + 64 * i, l * 64, kbatch, 0);
          if (++l == wgrad_live_blocks(p, kbatch)) {  // next live block, wrapping around the batches
            l = 0;
            do {
              if (++kbatch == batches) kbatch = 0;
            } while (wgrad_live_blocks(p, kbatch) == 0);
          }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------- consumers: warpgroup c owns rows 64 c .. 64 c + 63 of a tile
  setmaxnreg_inc<232>();
  const int c = wg - 1;
  const int w = (threadIdx.x & 127) >> 5;
  float* stage = reinterpret_cast<float*>(smem + kStages * Cfg::kStageBytes + c * Cfg::kEpiBytes);
  const int cq = ws_lane_col(lane);
  float acc[128];  // written by each piece's first MMA (scale_d = 0)
  int it = 0;
  for (long long g = g_begin; g < g_end;) {
    int t, j0, j1;
    piece(g, t, j0, j1);
    g += j1 - j0;
    for (int j = 0; j < j1 - j0; ++j, ++it) {
      const int s = it % kStages;
      mbar_wait(&full_bar[s], (it / kStages) & 1);
      const uint32_t sa = smem_u32(smem + s * Cfg::kStageBytes) + c * 8192;  // this warpgroup's 64 rows of dW x 64 tokens
      const uint32_t sb = smem_u32(smem + s * Cfg::kStageBytes + Cfg::kABytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_m64n256k16<1, 1>(acc, make_smem_desc_sw128(sa + k * 2048, 8192, 1024),
                               make_smem_desc_sw128(sb + k * 2048, 8192, 1024), (j > 0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();  // the previous K block's MMAs have retired: its stage goes back to the producer
      if (j > 0 && lane == 0) mbar_arrive(&empty_bar[(it - 1) % kStages]);
    }
    wgmma_wait<0>();
    if (lane == 0) mbar_arrive(&empty_bar[(it - 1) % kStages]);

    // ---- dW += the piece, 64 columns at a time (ws_stage_chunk), 16 lanes per 64-column row segment
    const int mt = t / n_tiles, n_tile = t - mt * n_tiles;
    const int m0 = mt * 128, col_base = n_tile * 256;
    const int n_valid = min(256, p.n_total - col_base);
    const int rows_here = min(128, p.m_rows - m0) - 64 * c;  // valid rows of this warpgroup's half (may be <= 0)
    float* out = static_cast<float*>(p.out.p) + (static_cast<long long>(m0) + 64 * c) * p.out.ld + col_base;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (64 * j >= n_valid) break;  // warpgroup-uniform
      named_bar_sync(1 + c, 128);    // the previous chunk has been read out of the staging buffer
      ws_stage_chunk(acc, stage, j, w, lane);
      named_bar_sync(1 + c, 128);
      const int cl = 64 * j + cq;
      if (cl < n_valid) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int r = ws_chunk_row(w, i, lane);
          if (r < rows_here) {
            const float4 v = ws_load_row(stage, r, cq);
            red_add_f32x4(out + r * p.out.ld + cl, v.x, v.y, v.z, v.w);
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------- pos_conv, windowed
// Grouped Conv1d(k = taps, padding = taps/2) as an implicit GEMM whose A operand is loaded ONCE per tile: the 128 frames of a
// tile need input rows m0 .. m0+127+taps-1 of the zero-padded activation, and tap j multiplies rows m0+j .. m0+j+127 -- the same
// shared-memory tile, shifted by j rows.  One 256-row TMA box brings the window in; every tap is four wgmma per consumer
// warpgroup whose A descriptor starts j rows (j * 128 bytes) into the tile.  Only the per-tap weight tile (8 KB) streams through
// the TMA ring, so the kernel reads ~1/3 of the bytes of the box-per-tap formulation.
// grid (groups * KB, m_tiles * batches); block 288 (two consumer warpgroups, TMA warp); fused tail = epilogue_chunk32.
// KB = 64-channel blocks of a group's padded width (Cgp = 64 KB): with KB = 2 (65..128 channels per group) the window and every
// tap's weight tile are two 64-channel K blocks, and CTA (g, h) computes the group's output channels 64 h .. 64 h + 63 (the
// epilogue keeps the valid ones; input channels past the group multiply zero weights).
template <int KB>
struct PosconvCfg {
  static constexpr int kStages = KB == 1 ? 6 : 4;
  static constexpr int kABytes = KB * 256 * 128;  // KB blocks of 256 rows x 64 bf16
  static constexpr int kBBytes = KB * 64 * 128;   // 64 output channels x 64 KB input channels of one tap
  static constexpr int kSmemBytes = kABytes + kStages * kBBytes + 1024;
  static constexpr int kThreads = 288;
};

template <int KB>
__global__ void __launch_bounds__(288, 2) posconv_window_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                const __grid_constant__ CUtensorMap tmB,
                                                                const __grid_constant__ GemmParams p, int taps, int cg) {
  pdl_launch_dependents();
  using Cfg = PosconvCfg<KB>;
  constexpr int kStages = Cfg::kStages;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int g = blockIdx.x / KB, h = blockIdx.x % KB;
  const int mb = blockIdx.y / p.m_tiles_per_batch;
  const int m0 = (blockIdx.y % p.m_tiles_per_batch) * 128;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sA = smem;
  uint8_t* sB = smem + Cfg::kABytes;
  __shared__ uint64_t a_full, full_bar[kStages], empty_bar[kStages];

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    mbar_init(&a_full, 1);
#pragma unroll
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();

  if (warp == 8) {
    if (lane == 0) {
      mbar_expect_tx(&a_full, Cfg::kABytes);
#pragma unroll
      for (int kb = 0; kb < KB; ++kb)  // rows m0 .. m0+255 of this group's channels (zero-filled past the end)
        tma_load_4d(sA + kb * 32768, &tmA, &a_full, g * cg + 64 * kb, m0, mb, 0);
      for (int j = 0; j < taps; ++j) {
        const int s = j % kStages;
        mbar_wait(&empty_bar[s], ((j / kStages) & 1) ^ 1);
        mbar_expect_tx(&full_bar[s], Cfg::kBBytes);
#pragma unroll
        for (int kb = 0; kb < KB; ++kb)
          tma_load_4d(sB + s * Cfg::kBBytes + kb * 8192, &tmB, &full_bar[s], (j * KB + kb) * 64, (g * KB + h) * 64, 0, 0);
      }
    }
  } else {
    const int c = warp >> 2;
    float acc[32];  // written by the first tap's MMAs (scale_d = 0)
    mbar_wait(&a_full, 0);
    for (int j = 0; j < taps; ++j) {
      const int s = j % kStages;
      mbar_wait(&full_bar[s], (j / kStages) & 1);
      const uint32_t sa = smem_u32(sA) + (64 * c + j) * 128;  // this warpgroup's 64 rows of the window, shifted by j rows
      const uint32_t sb = smem_u32(sB + s * Cfg::kBBytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4 * KB; ++k)
        wgmma_tile<64, false, false>(acc, make_smem_desc_sw128(sa + (k >> 2) * 32768 + (k & 3) * 32, 16, 1024),
                                     make_smem_desc_sw128(sb + (k >> 2) * 8192 + (k & 3) * 32, 16, 1024),
                                     (j > 0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();
      if (j > 0 && lane == 0) mbar_arrive(&empty_bar[(j - 1) % kStages]);
    }
    wgmma_wait<0>();
    gemm_consumer_tail<64>(p, acc, reinterpret_cast<float*>(smem), mb, m0, g * cg + 64 * h, min(64, cg - 64 * h),
                           min(128, p.m_rows - m0));
  }
}

}  // namespace b200
