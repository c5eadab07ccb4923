// Flash-style attention forward with the WavLM gated relative-position bias, wgmma + TMA (sm_90a).
//
// One CTA = 128 query rows of one (batch, head): two consumer warpgroups and one producer warp (288 threads).
//   producer warp: lane 0 loads Q once and K / V key tiles into two-stage rings with TMA; the warp fills the per-key-tile bias /
//     key-mask stage (double-buffered, one tile ahead)
//   consumer warpgroup c = 0, 1: rows 64 c .. 64 c + 63.  Per key tile n (128 keys):
//     S_n  = Q_c K_n^T        wgmma m64n128k16 into 64 fp32 registers (accumulator fragment layout, see ptx.cuh)
//     p    = exp2(S*scale*log2e + gate_i*log2e*tab[j-i] + keymask - m_i)      on the fragments, ONE pass
//     P_n  -> bf16 pairs in registers, the A operand of
//     O   += P_n V_n          wgmma m64n64k16 register-A form (V_n read MN-major from the TMA tile), O in registers
// S and P are never live at once (the softmax turns S into P in place), which keeps a consumer inside the 168 registers that
// 288 threads allow; a producer warpgroup with setmaxnreg does not raise that ceiling (ptxas still allocates 168).
// The two consumers ping-pong through two named barriers: a warpgroup issues S_n, hands the turn to the other warpgroup and runs
// its softmax while the other's MMAs execute.  Neither the scores nor P go through shared memory.
// The softmax is invariant to the reference m_i subtracted in the exponent, so m_i is fixed by the first tile that has a finite
// score for the row (a max over the quad of threads that hold the row) and never refreshed: the accumulator needs no per-tile
// rescale (fp32 sums / accumulators absorb factors up to 2^80).  If a later score outgrows the reference by more than that,
// the warpgroup re-bases: it rescales its row sums and accumulator rows, recomputes S and then the tile -- a correctness path
// that real inputs do not take.  Each thread sums its 32 columns of a row; the quad's partial sums are added once, at the end.
// Padding: key tiles that are fully padded at the END of the utterance are skipped (the loop runs over n_eff tiles), and a CTA
// whose 128 query rows are all padded only writes zeros -- padded frames never influence valid ones (keys are masked) and the
// reference's values there are unspecified garbage, so the ragged batch does not pay for its padding.
// Bias and key mask are staged per key tile, so shared memory does not grow with T: the bias of (row r, key k0 + c) is
// window[c - r + 127] with window[k] = tab[h, k0 + k + T - 1 - (q0 + 127)].  A thread reads it for column pairs (c, c + 1),
// c even; the window is kept as TWO copies shifted by one element, so that each pair is one aligned 8-byte load whatever the
// parity of r.  Next to it: the tile's 128-float additive key mask and its flag (0 no masked key, 1 some, 2 all).  The stage
// of tile n lives in buffer n & 1 and is refilled with tile n + 2 once tile n's V has been released.  The table is at most a
// few MB and stays in L2.
// Dropout: the keep bits of a column pair are one hash word; a warp holds 16 consecutive query rows, i.e. one 16-bit half of
// each mask word, which it assembles from ballots and stores as u16 (no cross-warp merge).
// Head width HD = 64, 80 or 120: tiles, maps and MMA shapes per width are in attn_common.cuh (HeadTile).  A tile is 16, 20 or
// 32 KB and O is 32, 40 or 64 fp32 registers per thread (at 120 columns 120..127 are zero and never stored).
// Shared memory: 5 tiles of Q / K / V rings (81920 B at HD 64, 102400 B at 80, 163840 B at 120) + 2 x 2704 B of stages
// + 1024 B alignment = 88352 B (HD 64), 108832 B (HD 80) or 170272 B (HD 120) for every T.
#include "../../include/unispeech_b200.h"
#include "attn_common.cuh"
#include "common.h"
#include <type_traits>

namespace b200 {

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// bits 0, 4, 8, ..., 28 of x -> bits 0..7
__device__ __forceinline__ uint32_t gather_every4th_bit(uint32_t x) {
  x &= 0x11111111u;
  x = (x | (x >> 3)) & 0x03030303u;
  x = (x | (x >> 6)) & 0x000F000Fu;
  return (x | (x >> 12)) & 0xFFu;
}

constexpr int kFwdThreads = 288;                // two consumer warpgroups + one producer warp
// floats of ONE bias-window copy: 256 entries + 16, so that the two copies sit 16 banks apart (a warp's 8-byte loads touch 14
// consecutive floats of each copy: no bank conflict)
constexpr int kTabStride = 2 * kAttnTile + 16;
constexpr int kMaskOff = 2 * kTabStride;        // the key mask, then the flag
constexpr int kStageFloats = kMaskOff + kAttnTile + 4;
// shared-memory map of head width HD: Q tile (rows of consumer c at 8192 c, and 2048 c in the 32-byte block), 2-stage K and V
// rings, then the two per-key-tile stages (bias copies, key mask, flag)
template <int HD>
struct FwdMap {
  static constexpr int kTile = kAttnTile * HeadTile<HD>::kCols * 2;  // one [128][HD] bf16 tile
  static constexpr int kQ = 0, kK = kTile, kV = 3 * kTile, kStage = 5 * kTile;
  static constexpr int kSmem = kStage + 2 * kStageFloats * 4 + 1024;  // (+ 1024 for the alignment of the base)
};
constexpr float kRebase = 1.2089258e24f;        // 2^80: a tile whose row sum reaches this is re-based on its own maximum

template <int HD, bool HAS_BIAS, bool DROP>
__global__ void __launch_bounds__(kFwdThreads, 1) attn_fwd_kernel(const __grid_constant__ CUtensorMap tm,
                                                                 const __grid_constant__ CUtensorMap tm16,
                                                                 const __grid_constant__ AttnParams p) {
  using HT = HeadTile<HD>;
  static_assert(HT::kBias || !HAS_BIAS, "the relative-position bias at this head width");
  using M = FwdMap<HD>;
  pdl_grid_sync();
  const int tid = threadIdx.x, wg = tid >> 7, lane = tid & 31;
  const int q0 = blockIdx.x * kAttnTile, h = blockIdx.y, b = blockIdx.z;
  const int T = p.T, D = p.D, N = p.n_tiles;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // 1024-aligned, still a __shared__ pointer (LDS/STS, not generic)
  uint8_t* sQ = smem + M::kQ;
  float* stage = reinterpret_cast<float*>(smem + M::kStage);

  __shared__ uint64_t q_full, k_full[2], k_empty[2], v_full[2], v_empty[2], stage_full[2];

  // ---- key padding: the number of key tiles that hold any valid key, and whether any of this CTA's 128 query rows is live.
  // ONE pass over the utterance's pad bytes (every thread takes a few), shared-memory counters, one barrier: the prologue pays a
  // single global-load latency instead of one per key tile.
  __shared__ int n_eff_s, live_s;
  if (tid == 0) { n_eff_s = p.key_pad != nullptr ? 1 : N; live_s = 0; }
  __syncthreads();
  if (p.key_pad != nullptr) {
    int last_valid = -1;
    bool live = false;
    for (int j = tid; j < T; j += kFwdThreads) {
      if (p.key_pad[static_cast<long long>(b) * T + j] == 0) {
        last_valid = j;                                        // increasing j: the last hit is the largest
        if (j >= q0 && j < q0 + kAttnTile) live = true;
      }
    }
    if (last_valid >= 0) atomicMax(&n_eff_s, last_valid / kAttnTile + 1);
    if (live) live_s = 1;
  }
  __syncthreads();
  const int n_eff = n_eff_s;
  // ---- a CTA whose query rows are all padded (or beyond T) has nothing to compute
  if (p.key_pad != nullptr && live_s == 0) {
    if (tid < kAttnTile && q0 + tid < T) {
      uint4* dst = reinterpret_cast<uint4*>(p.out + (static_cast<long long>(b) * T + q0 + tid) * D + h * HD);
#pragma unroll
      for (int g = 0; g < HD / 8; ++g) dst[g] = make_uint4(0u, 0u, 0u, 0u);
      if (p.lse != nullptr) p.lse[(static_cast<long long>(b) * p.H + h) * T + q0 + tid] = INFINITY;
    }
    return;
  }

  auto load_k = [&](int n) {
    const int s = n & 1;
    mbar_expect_tx(&k_full[s], M::kTile);
    tma_load_head<HD, kAttnTile, kAttnTile>(smem + M::kK + s * M::kTile, &tm, &tm16, &k_full[s], p.H + h, n * kAttnTile, b);
  };
  auto load_v = [&](int n) {
    const int s = n & 1;
    mbar_expect_tx(&v_full[s], M::kTile);
    tma_load_head<HD, kAttnTile, kAttnTile>(smem + M::kV + s * M::kTile, &tm, &tm16, &v_full[s], 2 * p.H + h, n * kAttnTile, b);
  };
  if (tid == 0) {
    // the TMA thread initialises the barriers and puts Q and the first two K / V tiles in flight right away (the other warps
    // see the barriers after the __syncthreads below)
    tma_prefetch_desc(&tm);
    if (HT::kTail) tma_prefetch_desc(&tm16);
    mbar_init(&q_full, 1);
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      mbar_init(&k_full[s], 1);
      mbar_init(&v_full[s], 1);
      mbar_init(&k_empty[s], 8);      // one arrival per consumer warp once its softmax is done with S
      mbar_init(&v_empty[s], 8);      // ... once its PV MMAs have retired (its softmax has read the stage, too)
      mbar_init(&stage_full[s], 32);  // one arrival per lane of the stage warp once its part of the stage is stored
    }
    fence_mbar_init();
    mbar_expect_tx(&q_full, M::kTile);
    tma_load_head<HD, kAttnTile, kAttnTile>(sQ, &tm, &tm16, &q_full, h, q0, b);
    for (int n = 0; n < 2 && n < n_eff; ++n) {
      load_k(n);
      load_v(n);
    }
  }
  __syncthreads();

  if (tid >= 2 * 128) {
    // ------------------------------------------------------------------ producer warp
    // lane 0 loads K / V tile n into slot n & 1 once tile n - 2 has released it; the warp fills the stage of tile n: lane l
    // loads window entries l + 32 t (257 are needed: 256 for copy 0, shifted by one for copy 1) and builds the key mask of
    // keys k0 + 4 l .. k0 + 4 l + 3
    for (int n = 0; n < n_eff; ++n) {
      const int s = n & 1;
      if (n >= 2) {
        const uint32_t ph = ((n >> 1) - 1) & 1;
        mbar_wait(&k_empty[s], ph);
        if (lane == 0) load_k(n);
        mbar_wait(&v_empty[s], ph);
        if (lane == 0) load_v(n);
      }
      float* stg = stage + s * kStageFloats;
      const int k0 = n * kAttnTile;
      if (HAS_BIAS) {
        const int base = k0 + (T - 1) - (q0 + kAttnTile - 1);
        const float* tab_h = p.tab + static_cast<long long>(h) * (2 * T - 1);
        float v[9];
#pragma unroll
        for (int t = 0; t < 9; ++t) {
          const int i = lane + 32 * t, gi = base + i;
          v[t] = (i <= 2 * kAttnTile && gi >= 0 && gi < 2 * T - 1) ? tab_h[gi] : 0.f;
        }
#pragma unroll
        for (int t = 0; t < 9; ++t) {
          const int i = lane + 32 * t;
          if (i < 2 * kAttnTile) stg[i] = v[t];
          if (i >= 1 && i <= 2 * kAttnTile) stg[kTabStride + i - 1] = v[t];
        }
      }
      float kb[4];
      int cnt = 0;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int j = k0 + 4 * lane + e;
        const bool masked = (j >= T) || (p.key_pad != nullptr && p.key_pad[static_cast<long long>(b) * T + j] != 0);
        kb[e] = masked ? -INFINITY : 0.f;
        cnt += masked ? 1 : 0;
      }
      reinterpret_cast<float4*>(stg + kMaskOff)[lane] = make_float4(kb[0], kb[1], kb[2], kb[3]);
      cnt = __reduce_add_sync(0xffffffffu, cnt);
      if (lane == 0) reinterpret_cast<int*>(stg)[kMaskOff + kAttnTile] = (cnt == 0) ? 0 : (cnt == kAttnTile ? 2 : 1);
      mbar_arrive(&stage_full[s]);
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroup c: rows 64 c .. 64 c + 63
  const int c = wg, w = (tid >> 5) & 3, quad = lane & 3;
  const int r0 = 64 * c + 16 * w + (lane >> 2);  // this thread's rows of the tile: r0 and r0 + 8 (fragment rows, ptx.cuh)
  float gl[2] = {0.f, 0.f};
  if (HAS_BIAS) {
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int row = q0 + r0 + 8 * rr;
      const float g = (p.gate != nullptr && row < T) ? p.gate[(static_cast<long long>(b) * p.H + h) * T + row] : 1.0f;
      gl[rr] = g * kLog2e;
    }
  }
  const float sc = p.scale * kLog2e;
  // the bias pair of (row r0, columns 8 j + 2 quad + {0, 1}) is window[e], window[e + 1] with e = 8 j + 2 quad + 127 - r0: in
  // copy 0 at e if e is even, in copy 1 (window shifted by one) at e - 1 if it is odd.  Row r0 + 8 reads 8 floats lower.
  const int toff = kAttnTile - 1 - r0;
  const int tab_off = (toff & 1) * kTabStride + (toff & ~1) + 2 * quad;
  // dropout on the probabilities: per-row hash keys, and this warp's half of the mask words of its 16 rows
  uint32_t rk0[2] = {0u, 0u}, rk1[2] = {0u, 0u};
  uint16_t* mask16 = nullptr;
  if (DROP) {
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const uint32_t rowid = static_cast<uint32_t>(b * p.H + h) * static_cast<uint32_t>(T) + static_cast<uint32_t>(q0 + r0 + 8 * rr);
      rk0[rr] = drop_row_k0(p.drop_k0, rowid);
      rk1[rr] = drop_row_k1(p.drop_k1, rowid);
    }
    const int row16 = q0 + 64 * c + 16 * w;  // bits row16 & 31 .. + 15 of the words: the low or the high half
    mask16 = reinterpret_cast<uint16_t*>(p.drop_mask + (static_cast<long long>(b * p.H + h) * (4 * N) + (row16 >> 5)) *
                                                           (N * kAttnTile)) + ((row16 >> 4) & 1);
  }

  HeadAcc<HD> o;  // O rows r0, r0 + 8
  o.zero();
  float m_ref[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const uint32_t aQ = smem_u32(sQ) + 8192 * c;  // this consumer's 64 rows of Q

  // ping-pong: consumer c issues its S MMAs after syncing on barrier 1 + c, then arrives on the other's barrier 2 - c, so
  // that one warpgroup's softmax runs while the other's MMAs hold the tensor pipe
  if (c == 1) named_bar_arrive(1, 2 * 128);
  mbar_wait(&q_full, 0);
#pragma unroll 1
  for (int n = 0; n < n_eff; ++n) {
    const int s = n & 1, k0 = n * kAttnTile;
    float acc[64];    // S: acc[i] is row r0 + 8 ((i >> 1) & 1), column 8 (i >> 2) + 2 quad + (i & 1)
    uint32_t pk[32];  // P: bf16 pairs in the register-A layout (pk[i / 2] = columns of acc[i], acc[i + 1])
    mbar_wait(&k_full[s], (n >> 1) & 1);
    named_bar_sync(1 + c, 2 * 128);
    const uint32_t bK = smem_u32(smem + M::kK + s * M::kTile);
    auto qk = [&]() {  // S = Q K_n^T
      wgmma_fence();
      mma_k_head<HD, kAttnTile>(acc, aQ, 64 * c, bK);
      wgmma_commit();
    };
    qk();
    if (c == 0 || n + 1 < n_eff) named_bar_arrive(2 - c, 2 * 128);  // every sync on either barrier has its arrival
    wgmma_wait<0>();

    mbar_wait(&stage_full[s], (n >> 1) & 1);
    const float* stg = stage + s * kStageFloats;
    const float* tabp = stg + tab_off;
    const float* kbias = stg + kMaskOff + 2 * quad;
    const bool msk = reinterpret_cast<const int*>(stg)[kMaskOff + kAttnTile] != 0;

    auto tile_max = [&](float* mx) {  // row maxima of the exponent argument over this tile (bias and key mask included)
      mx[0] = mx[1] = -INFINITY;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        float2 kb = make_float2(0.f, 0.f);
        if (msk) kb = *reinterpret_cast<const float2*>(kbias + 8 * j);
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          float x0 = acc[4 * j + 2 * rr] * sc, x1 = acc[4 * j + 2 * rr + 1] * sc;
          if (HAS_BIAS) {
            const float2 tb = *reinterpret_cast<const float2*>(tabp - 8 * rr + 8 * j);
            x0 = fmaf(gl[rr], tb.x, x0); x1 = fmaf(gl[rr], tb.y, x1);
          }
          if (msk) { x0 += kb.x; x1 += kb.y; }
          mx[rr] = fmaxf(mx[rr], fmaxf(x0, x1));
        }
      }
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        mx[rr] = fmaxf(mx[rr], __shfl_xor_sync(0xffffffffu, mx[rr], 1));
        mx[rr] = fmaxf(mx[rr], __shfl_xor_sync(0xffffffffu, mx[rr], 2));
      }
    };
    // rows that have not seen a finite score yet take this tile's maximum as their reference (first tile, or only masked
    // keys so far); they hold l = 0 and an all-zero accumulator, so nothing has to be rescaled
    if (__any_sync(0xffffffffu, m_ref[0] == -INFINITY || m_ref[1] == -INFINITY)) {
      float mx[2];
      tile_max(mx);
#pragma unroll
      for (int rr = 0; rr < 2; ++rr)
        if (m_ref[rr] == -INFINITY) m_ref[rr] = mx[rr];
    }
    // one pass over the tile: probabilities (relative to m_ref) -> bf16 pairs in pk; lsum = this thread's part of the row sums.
    // MSK is a compile-time flag so that the common tiles (no padded key) carry no mask arithmetic at all.
    auto softmax_tile = [&](auto MSK, float* lsum) {
      constexpr bool kMsk = decltype(MSK)::value;
      float neg_ref[2], part[2][2];
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        neg_ref[rr] = (m_ref[rr] == -INFINITY) ? 0.f : -m_ref[rr];
        part[rr][0] = part[rr][1] = 0.f;
      }
      uint32_t sel[2] = {0u, 0u};  // dropout: ballots (rows r0 - r0 % 8 + 0..7, + 8) of the key column this lane stores
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        float2 kb = make_float2(0.f, 0.f);
        if (kMsk) kb = *reinterpret_cast<const float2*>(kbias + 8 * j);
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const int i = 4 * j + 2 * rr;
          float x0 = fmaf(acc[i], sc, neg_ref[rr]), x1 = fmaf(acc[i + 1], sc, neg_ref[rr]);
          if (HAS_BIAS) {
            const float2 tb = *reinterpret_cast<const float2*>(tabp - 8 * rr + 8 * j);
            x0 = fmaf(gl[rr], tb.x, x0); x1 = fmaf(gl[rr], tb.y, x1);
          }
          if (kMsk) { x0 += kb.x; x1 += kb.y; }
          float e0 = fast_exp2(x0), e1 = fast_exp2(x1);
          part[rr][0] += e0;  // the normaliser is taken before dropout
          part[rr][1] += e1;
          if (DROP) {
            const uint32_t hb = drop_bits(rk0[rr], rk1[rr], static_cast<uint32_t>(k0 + 8 * j + 2 * quad) >> 1);
            const bool keep0 = drop_keep_lo(hb, p.drop_thr_hi), keep1 = drop_keep_hi(hb, p.drop_thr_hi);
            e0 = keep0 ? e0 : 0.f;
            e1 = keep1 ? e1 : 0.f;
            // bit 4 g + q of a ballot: row (lane group) g, column 8 j + 2 q (+ 1).  Lane L stores key column
            // 8 (4 (j >> 2) + (L >> 3)) + (L & 7), so it keeps the ballots of its column's j and parity.
            const uint32_t bal0 = __ballot_sync(0xffffffffu, keep0), bal1 = __ballot_sync(0xffffffffu, keep1);
            if ((lane >> 3) == (j & 3)) sel[rr] = (lane & 1) ? bal1 : bal0;
          }
          pk[i >> 1] = pack_bf16x2(e0, e1);
        }
        if (DROP && (j & 3) == 3) {
          const int q = (lane & 7) >> 1;
          const uint32_t bits = gather_every4th_bit(sel[0] >> q) | (gather_every4th_bit(sel[1] >> q) << 8);
          mask16[2 * (k0 + 8 * ((j & ~3) + (lane >> 3)) + (lane & 7))] = static_cast<uint16_t>(bits);
        }
      }
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) lsum[rr] = part[rr][0] + part[rr][1];
    };
    float lsum[2];
#pragma unroll 1
    while (true) {
      if (msk) softmax_tile(std::true_type{}, lsum);
      else softmax_tile(std::false_type{}, lsum);
      // warpgroup-wide decision (barrier 3 + c): the re-base issues wgmma, which all four warps must execute
      if (!named_bar_any(3 + c, 128, !(lsum[0] < kRebase) || !(lsum[1] < kRebase))) break;
      // ---- re-base (rare): a score outgrew the reference by 2^80.  Move the warpgroup's rows to the tile maximum (rows whose
      // maximum is not above their reference keep it exactly): rescale the row sums and the accumulator rows, then recompute
      // the tile.
      qk();  // the softmax consumed S in place: recompute it (K_n is released only after the softmax)
      wgmma_wait<0>();
      float mx[2];
      tile_max(mx);
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const float m_new = fmaxf(m_ref[rr], mx[rr]);
        const float factor = (m_ref[rr] == -INFINITY) ? 0.f : fast_exp2(m_ref[rr] - m_new);
        l_run[rr] *= factor;
        m_ref[rr] = m_new;
        o.scale_row(rr, factor);
      }
    }
    if (lane == 0) mbar_arrive(&k_empty[s]);
    l_run[0] += lsum[0];
    l_run[1] += lsum[1];

    // ---- O += P V_n: P as the register A operand
    mbar_wait(&v_full[s], (n >> 1) & 1);
    const uint32_t bV = smem_u32(smem + M::kV + s * M::kTile);
    wgmma_fence();
    mma_n_head<HD, kAttnTile>(o, pk, bV, true);
    wgmma_commit();
    wgmma_wait<0>();
    if (lane == 0) mbar_arrive(&v_empty[s]);
  }

  // O / l straight from the fragments: bf16 pairs of the rows r0, r0 + 8
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    float l = l_run[rr];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int row = q0 + r0 + 8 * rr;
    if (row < T) {
      if (p.lse != nullptr && quad == 0)
        p.lse[(static_cast<long long>(b) * p.H + h) * T + row] = (l > 0.f) ? (m_ref[rr] + log2f(l)) : INFINITY;
      const float inv = l > 0.f ? (DROP ? p.drop_rp : 1.0f) / l : 0.f;
      o.store_row(p.out + (static_cast<long long>(b) * T + row) * D + h * HD + 2 * quad, rr, inv);
    }
  }
}

}  // namespace b200

using namespace b200;

extern "C" {

// out[b,t,h*HD+d] = softmax_j(scale q.k + gate*tab[j-i], key padding) v     (WavLM/modules.py:540-563 replaced)
// qkv: bf16 [B,T,3D] fused projection output; gate: fp32 [B,H,T] or NULL; tab: fp32 [H,2T-1] or NULL (no bias);
// key_pad: uint8 [B,T] or NULL; out: bf16 [B,T,D]; lse: fp32 [B,H,T] (log2-domain log-sum-exp, saved for backward).
// head_dim HD: 64, or 80 / 120 without the bias.  Rows of `out` at padded query frames are unspecified-but-finite (zeros where a
// whole 128-row block is padded).
int b200s_attn_fwd_dropout(const void* qkv, const float* gate, const float* tab, const uint8_t* key_pad, void* out, float* lse,
                           int B, int T, int H, float scale, float drop_p, uint32_t key0, uint32_t key1, uint32_t* drop_mask,
                           int head_dim, b200s_stream stream) {
  B200_CHECK_ARG(qkv && out, "attn_fwd: null pointer");
  if (const int rc = attn_check_head("attn_fwd", head_dim, tab != nullptr)) return rc;
  B200_CHECK_ARG(drop_p >= 0.f && drop_p < 1.f, "attn_fwd: dropout p=%f out of range [0,1)", static_cast<double>(drop_p));
  B200_CHECK_ARG(drop_p == 0.f || drop_mask != nullptr, "attn_fwd: dropout needs the mask buffer (b200s_attn_dropout_mask_words)");
  B200_CHECK_ARG(static_cast<long long>(B) * H * T < (1LL << 32), "attn_fwd: B*H*T exceeds the 32-bit dropout row counter");
  const int D = H * head_dim;
  CUtensorMap tm, tm16;
  AttnParams p;
  memset(&p, 0, sizeof(p));
  p.T = T; p.H = H; p.B = B; p.D = D;
  p.n_tiles = ceil_div(T, kAttnTile);
  B200_CHECK_ARG(T >= 1, "attn_fwd: T=%d out of range", T);
  if (make_operand_tmaps(&tm, &tm16, qkv, T, B, 3 * D, head_dim, kAttnTile)) return -3;
  p.scale = scale;
  p.gate = gate; p.tab = tab; p.key_pad = key_pad;
  p.out = static_cast<__nv_bfloat16*>(out);
  p.lse = lse;
  const bool drop = drop_p > 0.f;
  p.drop_mask = drop_mask;
  p.drop_k0 = key0; p.drop_k1 = key1;
  p.drop_thr_hi = drop_threshold16(drop_p) << 16;
  p.drop_rp = 1.0f / (1.0f - drop_p);
  dim3 grid(ceil_div(T, kAttnTile), H, B);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  return attn_dispatch(head_dim, tab != nullptr, drop, [&](auto hd, auto bias, auto dp) {
    const auto kern = attn_fwd_kernel<hd, bias, dp>;
    constexpr int smem = FwdMap<hd>::kSmem;
    B200_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    B200_CHECK_CUDA(launch_pdl(kern, grid, dim3(kFwdThreads), smem, st, tm, tm16, p));
    B200_CHECK_LAUNCH();
    return 0;
  });
}

int b200s_attn_fwd(const void* qkv, const float* gate, const float* tab, const uint8_t* key_pad, void* out, float* lse,
                   int B, int T, int H, float scale, int head_dim, b200s_stream stream) {
  return b200s_attn_fwd_dropout(qkv, gate, tab, key_pad, out, lse, B, T, H, scale, 0.f, 0u, 0u, nullptr, head_dim, stream);
}

long long b200s_attn_dropout_mask_words(int B, int T, int H) { return attn_drop_mask_words(B, H, T); }

}  // extern "C"
