// Shared pieces of the gated-relative-position-bias attention kernels (forward, dK/dV backward, dQ backward).
//
// Math (MultiheadAttention fast path, WavLM/modules.py:457-564; SURVEY.md S7-S9):
//   logit[b,h,i,j] = scale * q_i . k_j + gate[b,h,i] * tab[h, j - i + T - 1]      (-inf where key j is padded)
//   P = softmax_j(logit),  O = P V
// The [B*H,T,T] bias of the reference is never materialised: it is Toeplitz, so a (query tile, key tile) pair reads only 255
// consecutive entries of the per-head table.  Each kernel stages that window per tile in shared memory (the forward one key tile
// ahead, the backward 128 new entries per query tile) and adds gate_i * tab[j-i] inside the softmax loop, so shared memory is
// constant in T: 88,352 bytes for the forward, 176,128 for the backward.
// Layout: q/k/v are column slices of the fused projection output qkv[B, T, 3D] (head h of q at columns h*HD.., k at
// D + h*HD.., v at 2D + h*HD..); no head-major reshuffle exists.  Every attention operand (qkv, dO and the fp32 dQ accumulator)
// is read or reduced through a head-shaped TMA map [B, T, slots, HD] whose innermost dimension is exactly one head, addressed
// by (column in the head, head slot, row, batch): slot h, H + h or 2H + h of qkv for q, k or v, slot h of dO and dQ.  A box
// never reaches into a neighbouring head: columns beyond HD are zero-filled on loads and clipped on reductions.
// Head width HD is 64, 80 or 120 (a template parameter of the kernels; HeadTile below).  A [rows][HD] tile in shared memory is
// one or two 64-column SWIZZLE_128B blocks ([rows][128 B] each) and, at HD = 80, a 16-column SWIZZLE_32B block ([rows][32 B])
// behind them: a 160-byte row is wider than the 128-byte swizzle span, so the head's columns 64..79 come from a second map
// with a 16-column box.  At HD = 120 the second 64-column box reads columns 64..127 of the head, and TMA fills 120..127 with
// zeros.  K = HD products are k16 steps over the 128-byte blocks (at HD = 120 the last one over the zero tail) plus, at 80,
// one on the 32-byte block; N = HD products are one n64 or n128 wgmma (MN-major B, dead columns 120..127 zero) plus, at 80, an
// n16 one on the same A operand.  Every store writes exactly the head's HD columns.
#pragma once
#include "common.h"
#include "dropout.cuh"
#include "ptx.cuh"

#include <type_traits>

namespace b200 {

constexpr int kAttnTile = 128;  // queries per CTA tile == keys per tile
constexpr float kLog2e = 1.4426950408889634f;

// the shared-memory tile and the MMA shapes of head width HD
template <int HD>
struct HeadTile {
  static_assert(HD == 64 || HD == 80 || HD == 120, "head width 64, 80 or 120");
  static constexpr bool kBias = HD == 64;                       // the relative-position bias is built at this width only
  static constexpr int kBlocks = HD == 120 ? 2 : 1;             // 64-column SWIZZLE_128B blocks
  static constexpr bool kTail = HD == 80;                       // and a 16-column SWIZZLE_32B block behind them
  static constexpr int kCols = 64 * kBlocks + (kTail ? 16 : 0);  // bf16 columns of a tile row: 64, 80 or 128
  static constexpr int kKSteps = 4 * kBlocks;                   // k16 steps of a K = HD product on the 128-byte blocks
  static constexpr int kN = 64 * kBlocks;                       // N of the main wgmma of an N = HD product (+ n16 on the tail)
  static constexpr int kAcc = kN / 2;                           // its fp32 accumulator registers per thread
};

template <int N, int TA, int TB>
__device__ __forceinline__ void wgmma_ss(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  static_assert(N == 16 || N == 64 || N == 128, "n16, n64 or n128");
  if constexpr (N == 128) wgmma_m64n128k16<TA, TB>(d, desc_a, desc_b, scale_d);
  else if constexpr (N == 64) wgmma_m64n64k16<TA, TB>(d, desc_a, desc_b, scale_d);
  else wgmma_m64n16k16<TA, TB>(d, desc_a, desc_b, scale_d);
}
template <int N>
__device__ __forceinline__ void wgmma_rs(float* d, const uint32_t* a, uint64_t desc_b, uint32_t scale_d) {
  static_assert(N == 16 || N == 64 || N == 128, "n16, n64 or n128");
  if constexpr (N == 128) wgmma_m64n128k16_rs<1>(d, a, desc_b, scale_d);
  else if constexpr (N == 64) wgmma_m64n64k16_rs<1>(d, a, desc_b, scale_d);
  else wgmma_m64n16k16_rs<1>(d, a, desc_b, scale_d);
}

// A 64-row x HD fp32 accumulator of one warpgroup in the wgmma fragment layout (ptx.cuh): this thread holds rows r0 and r0 + 8
// (fragment row rr = 0, 1) at columns 8 g + 2 (lane & 3) + {0, 1}.
template <int HD>
struct HeadAcc {
  using HT = HeadTile<HD>;
  float v[HT::kAcc];  // columns 0..63 (0..127 at HD = 120, of which 120..127 are dead)
  float tail[8];      // columns 64..79 (HD = 80 only)

  __device__ __forceinline__ void zero() {
#pragma unroll
    for (int i = 0; i < HT::kAcc; ++i) v[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) tail[i] = 0.f;
  }
  __device__ __forceinline__ void scale_row(int rr, float f) {
#pragma unroll
    for (int g = 0; g < HT::kAcc / 4; ++g) {
      v[4 * g + 2 * rr] *= f;
      v[4 * g + 2 * rr + 1] *= f;
    }
    if (HT::kTail) {
#pragma unroll
      for (int g = 0; g < 2; ++g) {
        tail[4 * g + 2 * rr] *= f;
        tail[4 * g + 2 * rr + 1] *= f;
      }
    }
  }
  // bf16 pairs of fragment row rr times s into the HD columns of a row; dst points at the row's column 2 (lane & 3)
  __device__ __forceinline__ void store_row(__nv_bfloat16* dst, int rr, float s) const {
#pragma unroll
    for (int g = 0; g < HT::kAcc / 4; ++g)
      if (8 * g < HD) *reinterpret_cast<uint32_t*>(dst + 8 * g) = pack_bf16x2(v[4 * g + 2 * rr] * s, v[4 * g + 2 * rr + 1] * s);
    if (HT::kTail) {
#pragma unroll
      for (int g = 0; g < 2; ++g)
        *reinterpret_cast<uint32_t*>(dst + 64 + 8 * g) = pack_bf16x2(tail[4 * g + 2 * rr] * s, tail[4 * g + 2 * rr + 1] * s);
    }
  }
};

// one [ROWS][HD] bf16 tile of head slot `slot`, rows row0 .., batch b into `dst` in the layout above, as boxes of BOX_ROWS
// rows: m64 is the 64-column SWIZZLE_128B map, m16 the 16-column SWIZZLE_32B map (read only at HD = 80)
template <int HD, int ROWS, int BOX_ROWS>
__device__ __forceinline__ void tma_load_head(uint8_t* dst, const CUtensorMap* m64, const CUtensorMap* m16, uint64_t* bar,
                                              int slot, int row0, int b) {
  using HT = HeadTile<HD>;
#pragma unroll
  for (int r = 0; r < ROWS; r += BOX_ROWS) {
#pragma unroll
    for (int blk = 0; blk < HT::kBlocks; ++blk) tma_load_4d(dst + blk * ROWS * 128 + r * 128, m64, bar, 64 * blk, slot, row0 + r, b);
    if (HT::kTail) tma_load_4d(dst + HT::kBlocks * ROWS * 128 + r * 32, m16, bar, 64 * HT::kBlocks, slot, row0 + r, b);
  }
}

// acc = A B^T over the head width (a K = HD product: S = Q K^T, S^T = K Q^T, dP^T = V dO^T).  A = rows a_row0 .. a_row0 + 63
// of a [128][HD] tile, `a` the address of row a_row0 in the tile's first block (kept by the caller across its loop: computed
// here, the address costs the backward registers); B = an [N][HD] tile.  Both K-major.  The caller fences and commits.
template <int HD, int N>
__device__ __forceinline__ void mma_k_head(float* acc, uint32_t a, int a_row0, uint32_t b_tile) {
  using HT = HeadTile<HD>;
#pragma unroll
  for (int k = 0; k < HT::kKSteps; ++k)
    wgmma_ss<N, 0, 0>(acc, make_smem_desc_sw128(a + (k >> 2) * (kAttnTile * 128) + (k & 3) * 32, 16, 1024),
                      make_smem_desc_sw128(b_tile + (k >> 2) * (N * 128) + (k & 3) * 32, 16, 1024), k > 0 ? 1u : 0u);
  if (HT::kTail)  // the 32-byte block behind the 128-byte one (row a_row0 at 32 a_row0 instead of 128 a_row0)
    wgmma_ss<N, 0, 0>(acc, make_smem_desc_sw32(a + kAttnTile * 128 - a_row0 * 96), make_smem_desc_sw32(b_tile + N * 128), 1u);
}

// B operand of k16 step k of an N = HD product: rows 16 k .. of a [K][HD] tile, read MN-major
template <int HD, int K>
__device__ __forceinline__ uint64_t head_desc_mn(uint32_t b_tile, int k) {  // (the block stride is not read at n64)
  return make_smem_desc_sw128(b_tile + k * 2048, HeadTile<HD>::kBlocks == 2 ? K * 128 : 8192, 1024);
}
template <int K>
__device__ __forceinline__ uint64_t tail_desc_mn(uint32_t b_tile, int k) {
  return make_smem_desc_sw32(b_tile + K * 128 + k * 512);
}

// c (+)= A B over the head width (an N = HD product) with A in registers (O += P V, dV += P^T dO): A = K / 16 k-slices of bf16
// fragments (4 words each), B = a [K][HD] tile.  accumulate = false overwrites c.  The caller fences and commits.
template <int HD, int K>
__device__ __forceinline__ void mma_n_head(HeadAcc<HD>& c, const uint32_t* a, uint32_t b_tile, bool accumulate) {
  using HT = HeadTile<HD>;
#pragma unroll
  for (int k = 0; k < K / 16; ++k) {
    const uint32_t sd = (accumulate || k > 0) ? 1u : 0u;
    wgmma_rs<HT::kN>(c.v, a + 4 * k, head_desc_mn<HD, K>(b_tile, k), sd);
    if (HT::kTail) wgmma_rs<16>(c.tail, a + 4 * k, tail_desc_mn<K>(b_tile, k), sd);
  }
}
// the same with A = rows a_row0 .. a_row0 + 63 of a [K / 64 blocks][128][64] bf16 SWIZZLE_128B tile in shared memory, K-major
// (dK += dS^T Q)
template <int HD, int K>
__device__ __forceinline__ void mma_n_head(HeadAcc<HD>& c, uint32_t a_tile, int a_row0, uint32_t b_tile, bool accumulate) {
  using HT = HeadTile<HD>;
#pragma unroll
  for (int k = 0; k < K / 16; ++k) {
    const uint32_t sd = (accumulate || k > 0) ? 1u : 0u;
    const uint64_t da = make_smem_desc_sw128(a_tile + (k >> 2) * (kAttnTile * 128) + a_row0 * 128 + (k & 3) * 32, 16, 1024);
    wgmma_ss<HT::kN, 0, 1>(c.v, da, head_desc_mn<HD, K>(b_tile, k), sd);
    if (HT::kTail) wgmma_ss<16, 0, 1>(c.tail, da, tail_desc_mn<K>(b_tile, k), sd);
  }
}

struct AttnParams {
  int T, H, B, D;          // D = H * head width
  int n_tiles;             // ceil(T / 128)
  float scale;             // head_dim^-0.5
  const float* gate;       // [B,H,T] or null (=1)
  const float* tab;        // [H, 2T-1] or null (no relative position bias)
  const uint8_t* key_pad;  // [B,T] or null
  __nv_bfloat16* out;      // [B,T,D]
  float* lse;              // [B,H,T], log2 domain
  // backward
  const __nv_bfloat16* dout;  // [B,T,D]
  const float* delta;         // [B,H,T] rowsum(dO * O)
  __nv_bfloat16* dqkv;        // [B,T,3D]
  float* dgate;               // [B,H,T]
  float* dtab;                // [H, 2T-1] (atomic accumulation)
  // dropout on the probabilities (attention_dropout, WavLM/modules.py:551): keep bits of query rows 32w..32w+31 against key
  // j live in word drop_mask[((b*H + h) * 4*n_tiles + w) * 128*n_tiles + j] (bit i & 31 = query i), written by the forward
  // kernel from the counter-based hash of dropout.cuh and re-read by the backward kernel; kept probabilities scale by drop_rp
  uint32_t* drop_mask;
  uint32_t drop_k0, drop_k1, drop_thr_hi;
  float drop_rp;              // 1 / (1 - p)
};

// words of the attention dropout bit mask for a [B,H,T,T] probability tensor
static inline long long attn_drop_mask_words(int B, int H, int T) {
  const long long n = (T + kAttnTile - 1) / kAttnTile;
  return static_cast<long long>(B) * H * (4 * n) * (kAttnTile * n);
}

// ---- host side

// [B, T, cols] bf16 or fp32 seen as [B, T, cols / hd heads, hd]: box = box_cols columns of one head x box_rows rows (gemm.cu)
int make_head_tmap(CUtensorMap* out, const void* ptr, CUtensorMapDataType dtype, int T, int B, int cols, int hd, int box_cols,
                   int box_rows, CUtensorMapSwizzle swizzle);

// the maps of one bf16 operand [B, T, cols]: m64 with the 64-column SWIZZLE_128B box and, at head width 80, m16 with the
// 16-column SWIZZLE_32B box (elsewhere m16 is a copy of m64 that the kernels do not read)
static inline int make_operand_tmaps(CUtensorMap* m64, CUtensorMap* m16, const void* ptr, int T, int B, int cols, int hd,
                                     int box_rows) {
  if (make_head_tmap(m64, ptr, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, T, B, cols, hd, 64, box_rows, CU_TENSOR_MAP_SWIZZLE_128B))
    return -3;
  if (hd != 80) {
    *m16 = *m64;
    return 0;
  }
  return make_head_tmap(m16, ptr, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, T, B, cols, hd, 16, box_rows, CU_TENSOR_MAP_SWIZZLE_32B) ? -3 : 0;
}

// argument checks shared by the attention entry points `op`: the head widths the kernels are built for, and the bias at 64 only
static inline int attn_check_head(const char* op, int head_dim, bool bias) {
  B200_CHECK_ARG(head_dim == 64 || head_dim == 80 || head_dim == 120, "%s: head_dim=%d is not supported (64, 80 or 120)", op,
                 head_dim);
  B200_CHECK_ARG(head_dim == 64 || !bias, "%s: the relative-position bias needs head_dim 64 (got %d)", op, head_dim);
  return 0;
}

// f(HD, BIAS, DROP) with the kernel instantiation's parameters as std::integral_constant, for a (head_dim, bias, dropout) that
// passed attn_check_head
template <class F>
static int attn_dispatch(int head_dim, bool bias, bool drop, F&& f) {
  auto with_drop = [&](auto hd, auto has_bias) { return drop ? f(hd, has_bias, std::true_type{}) : f(hd, has_bias, std::false_type{}); };
  if (head_dim == 120) return with_drop(std::integral_constant<int, 120>{}, std::false_type{});
  if (head_dim == 80) return with_drop(std::integral_constant<int, 80>{}, std::false_type{});
  return bias ? with_drop(std::integral_constant<int, 64>{}, std::true_type{})
              : with_drop(std::integral_constant<int, 64>{}, std::false_type{});
}

}  // namespace b200
