// Shared pieces of the gated-relative-position-bias attention kernels (forward, dK/dV backward, dQ backward).
//
// Math (MultiheadAttention fast path, WavLM/modules.py:457-564; SURVEY.md S7-S9):
//   logit[b,h,i,j] = scale * q_i . k_j + gate[b,h,i] * tab[h, j - i + T - 1]      (-inf where key j is padded)
//   P = softmax_j(logit),  O = P V
// The [B*H,T,T] bias of the reference is never materialised: it is Toeplitz, so a (query tile, key tile) pair reads only 255
// consecutive entries of the per-head table.  Each kernel stages that window per tile in shared memory (the forward one key tile
// ahead, the backward 128 new entries per query tile) and adds gate_i * tab[j-i] inside the softmax loop, so shared memory is
// constant in T: 88,352 bytes for the forward, 176,128 for the backward.
// Layout: q/k/v are column slices of the fused projection output qkv[B, T, 3D] (head h of q at columns h*64.., k at
// D + h*64.., v at 2D + h*64..), read by TMA with a strided 3-D tensor map; no head-major reshuffle exists.
#pragma once
#include "dropout.cuh"
#include "ptx.cuh"

namespace b200 {

constexpr int kAttnTile = 128;  // queries per CTA tile == keys per tile
constexpr int kHeadDim = 64;
constexpr float kLog2e = 1.4426950408889634f;

struct AttnParams {
  int T, H, B, D;          // D = H * 64
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

// write 8 consecutive bf16 of row r, 16-byte chunk index `chunk` (0..15 over 128 columns) into a K-major SWIZZLE_128B tile
// made of two [128 rows][64 cols] blocks (the layout of a K-major wgmma operand, and -- read as
// MN-major -- for the transposed use).
__device__ __forceinline__ void store_sw128_chunk(uint8_t* tile, int r, int chunk, uint4 v) {
  const int kb = chunk >> 3;       // which 64-column block
  const int c = chunk & 7;         // 16-byte chunk inside the 128-byte row
  uint8_t* p = tile + kb * 16384 + r * 128 + ((c ^ (r & 7)) << 4);
  *reinterpret_cast<uint4*>(p) = v;
}

}  // namespace b200
