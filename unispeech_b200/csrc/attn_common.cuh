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
// D + h*HD.., v at 2D + h*HD..), read by TMA with a strided 3-D tensor map; no head-major reshuffle exists.
// Head width HD is 64, 80 or 120 (a template parameter of the kernels).  A [rows][HD] tile is one 64-column SWIZZLE_128B block
// ([rows][128 B]) and, at HD = 80, a 16-column SWIZZLE_32B block ([rows][32 B]) right behind it: a 160-byte row is wider than
// the 128-byte swizzle span, and the two boxes load exactly the head's columns.  K = 80 products are four k16 steps on the
// first block and one on the second; N = 80 products are an n64 and an n16 wgmma on the same A operand.
// At HD = 120 the tensor map's innermost dimension is exactly one head (120 columns, then the 3H or H head slots, rows,
// batch), and a [rows][120] tile is two 64-column SWIZZLE_128B blocks: columns 120..127 of the second box lie outside the
// head, so TMA fills them with zeros and no column of a neighbouring head is read.  K = 120 products are eight k16 steps (the
// last one over the zero tail); N = 120 products are one n128 wgmma with MN-major B operands whose dead columns 120..127
// are zero, and every store writes exactly the head's 120 columns.
#pragma once
#include "dropout.cuh"
#include "ptx.cuh"

namespace b200 {

constexpr int kAttnTile = 128;  // queries per CTA tile == keys per tile
constexpr float kLog2e = 1.4426950408889634f;

// bf16 columns of a tile row in shared memory: the head width, or 128 at HD = 120 (two 64-column blocks, zero tail)
template <int HD>
constexpr int attn_tile_cols() { return HD == 120 ? 128 : HD; }

// one [ROWS][HD] bf16 tile of a [B, T, cols] tensor (columns c0 .., rows row0 ..) into `dst` in the layout above, as boxes of
// BOX_ROWS rows: m64 holds the 64-column SWIZZLE_128B map, m16 the 16-column SWIZZLE_32B map (read only at HD = 80).  At
// HD = 120, m64 is the head-shaped map (coordinates: column in the head, head slot c0 / 120, row, batch) and m16 is not read.
template <int HD, int ROWS, int BOX_ROWS>
__device__ __forceinline__ void tma_load_head(uint8_t* dst, const CUtensorMap* m64, const CUtensorMap* m16, uint64_t* bar,
                                              int c0, int row0, int b) {
#pragma unroll
  for (int r = 0; r < ROWS; r += BOX_ROWS) {
    if (HD == 120) {
      tma_load_4d(dst + r * 128, m64, bar, 0, c0 / HD, row0 + r, b);
      tma_load_4d(dst + ROWS * 128 + r * 128, m64, bar, 64, c0 / HD, row0 + r, b);
    } else {
      tma_load_4d(dst + r * 128, m64, bar, c0, row0 + r, b, 0);
      if (HD == 80) tma_load_4d(dst + ROWS * 128 + r * 32, m16, bar, c0 + 64, row0 + r, b, 0);
    }
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

}  // namespace b200
