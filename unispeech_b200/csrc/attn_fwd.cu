// Flash-style attention forward with the WavLM gated relative-position bias, wgmma + TMA (sm_90a).
//
// One CTA = 128 query rows of one (batch, head): one warpgroup (128 threads) that issues the tensor-core work AND owns one query
// row per thread for the softmax, plus one TMA producer warp.  Per key tile n (128 keys):
//   S_n  = Q K_n^T           wgmma m64n128k16 (two 64-row halves) -> fp32 staging tile in shared memory, one row per thread
//   p    = exp2(S*scale*log2e + gate_i*log2e*tab[j-i] + keymask - m_i)      ONE pass over the scores
//   P_n -> shared memory in the K-major SWIZZLE_128B operand layout (bf16)
//   O   += P_n V_n           wgmma m64n64k16 (V_n read MN-major from the TMA tile), fp32 accumulator in registers (fragments)
// Thread r owns query row r of the staged scores: the row reference / sum of the softmax are thread-local.  The accumulator rows
// are spread over the fragments; a per-row factor in shared memory (1 unless the row was re-based) carries a re-base to them.
// The softmax is invariant to the reference m_i subtracted in the exponent, so m_i is fixed by the first tile that has a finite
// score for the row and never refreshed: the accumulator needs no per-tile rescale (fp32 sums / accumulators absorb factors up to
// 2^80).  If a later score outgrows the reference by more than that, the warp re-bases: it rescales its row sums (and, through
// the per-row factor, the accumulator rows) and recomputes the tile -- a correctness path that real inputs do not take.
// K_{n+1} is loaded while the softmax of tile n runs (K and V have separate barriers).
// Padding: key tiles that are fully padded at the END of the utterance are skipped (the loop runs over n_eff tiles), and a CTA
// whose 128 query rows are all padded only writes zeros -- padded frames never influence valid ones (keys are masked) and the
// reference's values there are unspecified garbage, so the ragged batch does not pay for its padding.
// Bias and key mask are staged per key tile, so shared memory does not grow with T: key tile n reads the 255 consecutive bias
// entries slice[k0 .. k0 + 254] (slice[k] = tab[h, k + T - 1 - (q0 + 127)]), kept as FOUR copies shifted by 0..3 elements so
// that the 32 consecutive entries a thread needs per 32-column chunk are 8 aligned 128-bit loads instead of 32 scalar ones,
// next to the tile's 128-float additive key mask and its flag.  The TMA warp, idle between its K / V issues, fills that stage
// one tile ahead (tile n in buffer n & 1) and arrives on the buffer's mbarrier; the stage of tile n - 2 is free once the
// v_empty arrival of that tile has been seen.  The table is at most a few MB and stays in L2.
// Shared memory: 149504 B of Q / K / V / P / scores + 2 x 4752 B of stages + 1024 B alignment = 160032 B for every T.
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
// 32 x 32 bit-matrix transpose across a warp: on entry bit j of lane l's word is element (l, j); on return bit l of lane j's
// word is that element.  Five butterfly stages (one shuffle + three logic ops each) replace 32 ballots.
__device__ __forceinline__ uint32_t warp_bit_transpose(uint32_t x, int lane) {
#pragma unroll
  for (int s = 16; s >= 1; s >>= 1) {
    const uint32_t m = (s == 16) ? 0x0000FFFFu : (s == 8) ? 0x00FF00FFu : (s == 4) ? 0x0F0F0F0Fu : (s == 2) ? 0x33333333u : 0x55555555u;
    const uint32_t y = __shfl_xor_sync(0xffffffffu, x, s);
    x = (lane & s) ? ((x & ~m) | ((y >> s) & m)) : ((x & m) | ((y << s) & ~m));
  }
  return x;
}
__device__ __forceinline__ void mbar_arrive_rel(uint64_t* bar) {
  asm volatile("mbarrier.arrive.release.cta.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

constexpr int kFwdQ = 0;                        // 16 KB
constexpr int kFwdK = 16384;                    // 16 KB
constexpr int kFwdV = 32768;                    // 16 KB
constexpr int kFwdP = 49152;                    // 32 KB: [2 key blocks][128 rows][64 keys] bf16
constexpr int kSPitch = kAttnTile + 4;          // fp32 score row (floats)
constexpr int kFwdS = 81920;                    // fp32 scores [128][kSPitch]
constexpr int kFwdStage = kFwdS + kAttnTile * kSPitch * 4;  // 149504: two per-key-tile stages (bias copies, key mask)
constexpr int kFwdThreads = 160;                // one warpgroup + TMA warp
constexpr int kTabCopies = 4;
// floats of ONE bias-table copy: 256 window entries + 8 so that consecutive copies start 8 banks apart (conflict-free 128-bit
// loads across the quarter warp, whose lanes alternate between the four copies)
constexpr int kTabStride = 2 * kAttnTile + 8;
constexpr int kStageFloats = kTabCopies * kTabStride + kAttnTile + 4;   // copies, key mask, flag (+3 floats of padding)
constexpr int kFwdSmem = kFwdStage + 2 * kStageFloats * 4 + 1024;       // 160032 (+ 1024 for the alignment of the base)
constexpr float kRebase = 1.2089258e24f;        // 2^80: a tile whose row sum reaches this is re-based on its own maximum

__device__ __forceinline__ void lds_row32(const float* src, uint32_t* r) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 v = reinterpret_cast<const float4*>(src)[i];
    r[4 * i] = __float_as_uint(v.x); r[4 * i + 1] = __float_as_uint(v.y);
    r[4 * i + 2] = __float_as_uint(v.z); r[4 * i + 3] = __float_as_uint(v.w);
  }
}

template <bool HAS_BIAS, bool DROP>
__global__ void __launch_bounds__(kFwdThreads, 1) attn_fwd_kernel(const __grid_constant__ CUtensorMap tm,
                                                                 const __grid_constant__ AttnParams p) {
  pdl_grid_sync();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int q0 = blockIdx.x * kAttnTile, h = blockIdx.y, b = blockIdx.z;
  const int T = p.T, D = p.D, N = p.n_tiles;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // 1024-aligned, still a __shared__ pointer (LDS/STS, not generic)
  uint8_t* sQ = smem + kFwdQ;
  uint8_t* sK = smem + kFwdK;
  uint8_t* sV = smem + kFwdV;
  uint8_t* sP = smem + kFwdP;
  float* s_f = reinterpret_cast<float*>(smem + kFwdS);
  // stage of key tile n in buffer n & 1: [4][kTabStride] bias copies (copy c holds window[i + c], window[i] = slice[k0 + i]),
  // then the tile's 128-float additive key mask, then its flag (0 no masked key, 1 some, 2 all)
  float* stage = reinterpret_cast<float*>(smem + kFwdStage);

  __shared__ uint64_t q_full, k_full, k_empty, v_full, v_empty, stage_full[2];
  __shared__ float row_scale[kAttnTile];  // per query row: re-base factor of the current tile, then 1 / row sum for the epilogue

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
      uint4* dst = reinterpret_cast<uint4*>(p.out + (static_cast<long long>(b) * T + q0 + tid) * D + h * kHeadDim);
#pragma unroll
      for (int g = 0; g < 8; ++g) dst[g] = make_uint4(0u, 0u, 0u, 0u);
      if (p.lse != nullptr) p.lse[(static_cast<long long>(b) * p.H + h) * T + q0 + tid] = INFINITY;
    }
    return;
  }

  if (warp == 4 && lane == 0) {
    // the TMA thread initialises the barriers itself and puts Q and the first K / V tiles in flight right away (the other
    // warps see the barriers after the __syncthreads below)
    tma_prefetch_desc(&tm);
    mbar_init(&q_full, 1);
    mbar_init(&k_full, 1);
    mbar_init(&v_full, 1);
    mbar_init(&k_empty, 4);   // one arrival per warp of the warpgroup once its S MMAs have retired
    mbar_init(&v_empty, 4);   // ... once its PV MMAs have retired
    mbar_init(&stage_full[0], 32);   // one arrival per lane of the TMA warp once its part of the stage is stored
    mbar_init(&stage_full[1], 32);
    fence_mbar_init();
    mbar_expect_tx(&q_full, 16384);
    tma_load_4d(sQ, &tm, &q_full, h * kHeadDim, q0, b, 0);
    mbar_expect_tx(&k_full, 16384);
    tma_load_4d(sK, &tm, &k_full, D + h * kHeadDim, 0, b, 0);
    mbar_expect_tx(&v_full, 16384);
    tma_load_4d(sV, &tm, &v_full, 2 * D + h * kHeadDim, 0, b, 0);
  }
  __syncthreads();

  if (warp == 4) {
    // ------------------------------------------------------------------ TMA producer warp
    // stage of key tile n: lane l loads window entries l + 32 t (259 are needed: 255 read + the 3 of the widest shift) and
    // stores each into the copies that hold it, and builds the key mask of keys k0 + 4 l .. k0 + 4 l + 3
    auto fill_stage = [&](int n) {
      float* stg = stage + (n & 1) * kStageFloats;
      const int k0 = n * kAttnTile;
      if (HAS_BIAS) {
        const int base = k0 + (T - 1) - (q0 + kAttnTile - 1);
        const float* tab_h = p.tab + static_cast<long long>(h) * (2 * T - 1);
        float v[9];
#pragma unroll
        for (int t = 0; t < 9; ++t) {
          const int i = lane + 32 * t, gi = base + i;
          v[t] = (i < 2 * kAttnTile + kTabCopies - 1 && gi >= 0 && gi < 2 * T - 1) ? tab_h[gi] : 0.f;
        }
#pragma unroll
        for (int t = 0; t < 9; ++t)
#pragma unroll
          for (int c = 0; c < kTabCopies; ++c) {
            const int k = lane + 32 * t - c;
            if (k >= 0 && k < 2 * kAttnTile) stg[c * kTabStride + k] = v[t];
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
      reinterpret_cast<float4*>(stg + kTabCopies * kTabStride)[lane] = make_float4(kb[0], kb[1], kb[2], kb[3]);
      cnt = __reduce_add_sync(0xffffffffu, cnt);
      if (lane == 0) reinterpret_cast<int*>(stg)[kTabCopies * kTabStride + kAttnTile] = (cnt == 0) ? 0 : (cnt == kAttnTile ? 2 : 1);
      mbar_arrive(&stage_full[n & 1]);
    };
    fill_stage(0);
    if (n_eff > 1) fill_stage(1);
    for (int n = 1; n < n_eff; ++n) {  // (Q and tile 0 were issued in the prologue)
      const uint32_t ph = (n - 1) & 1;
      mbar_wait(&k_empty, ph);
      if (lane == 0) {
        mbar_expect_tx(&k_full, 16384);
        tma_load_4d(sK, &tm, &k_full, D + h * kHeadDim, n * kAttnTile, b, 0);
      }
      mbar_wait(&v_empty, ph);
      if (lane == 0) {
        mbar_expect_tx(&v_full, 16384);
        tma_load_4d(sV, &tm, &v_full, 2 * D + h * kHeadDim, n * kAttnTile, b, 0);
      }
      // tile n - 1 has retired its PV MMAs, so its stage (buffer (n + 1) & 1) has been read: fill it with tile n + 1
      if (n + 1 < n_eff) fill_stage(n + 1);
    }
  } else {
    // ------------------------------------------------------------------ the warpgroup: MMAs + softmax, thread = query row
    const int r = tid;
    const bool row_valid = (q0 + r) < T;
    const float* s_row = s_f + r * kSPitch;
    const int fr = 16 * (warp & 3) + (lane >> 2);   // first fragment row of this thread in each 64-row half (the other is fr + 8)
    float o_acc[2][32];                             // O rows [64 hm, 64 hm + 64) x 64 columns, wgmma fragment layout

    float gl = 0.f;
    if (HAS_BIAS) {
      const float g = (p.gate != nullptr && row_valid) ? p.gate[(static_cast<long long>(b) * p.H + h) * T + q0 + r] : 1.0f;
      gl = g * kLog2e;
    }
    const float sc = p.scale * kLog2e;
    // this row's part of a tile's bias window: entry (key k0 + j) = window[j + 127 - r]; copy a = (127 - r) & 3 is the one in
    // which that part starts on a 16-byte boundary
    const int toff = kAttnTile - 1 - r;
    const int tab_off = (toff & 3) * kTabStride + (toff & ~3);
    // dropout on the probabilities: per-row hash keys, and where this warp's 32 rows keep their bits (one word per key column)
    uint32_t rk0 = 0, rk1 = 0;
    uint32_t* mask_row = nullptr;
    if (DROP) {
      const uint32_t rowid = static_cast<uint32_t>(b * p.H + h) * static_cast<uint32_t>(T) + static_cast<uint32_t>(q0 + r);
      rk0 = drop_row_k0(p.drop_k0, rowid);
      rk1 = drop_row_k1(p.drop_k1, rowid);
      mask_row = p.drop_mask + (static_cast<long long>(b * p.H + h) * (4 * N) + ((q0 + r) >> 5)) * (N * kAttnTile);
    }

    float m_ref = -INFINITY, l_run = 0.f;
    mbar_wait(&q_full, 0);

    for (int n = 0; n < n_eff; ++n) {
      const int k0 = n * kAttnTile;
      // ---- S = Q K_n^T (two 64-row halves) -> fp32 staging tile
      mbar_wait(&k_full, n & 1);
#pragma unroll 1
      for (int hm = 0; hm < 2; ++hm) {
        float acc[64];
        const uint32_t a = smem_u32(sQ) + hm * 8192, bb = smem_u32(sK);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_m64n128k16<0, 0>(acc, make_smem_desc_sw128(a + k * 32, 16, 1024), make_smem_desc_sw128(bb + k * 32, 16, 1024),
                                 k > 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        acc_to_smem<128>(acc, s_f, kSPitch, 64 * hm);
      }
      if (lane == 0) mbar_arrive(&k_empty);  // this warp's S MMAs have retired: K may be refilled
      named_bar_sync(1, kAttnTile);           // the whole score tile is staged
      mbar_wait(&stage_full[n & 1], (n >> 1) & 1);
      const float* stg = stage + (n & 1) * kStageFloats;
      const float4* tab4 = reinterpret_cast<const float4*>(stg + tab_off);
      const float* kbias = stg + kTabCopies * kTabStride;
      const bool msk = reinterpret_cast<const int*>(stg)[kTabCopies * kTabStride + kAttnTile] != 0;

      auto tile_max = [&]() {  // row maximum of the exponent argument over this tile (bias and key mask included)
        float mx = -INFINITY;
#pragma unroll 1
        for (int c0 = 0; c0 < kAttnTile; c0 += 32) {
          uint32_t su[32];
          lds_row32(s_row + c0, su);
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            float4 tb = make_float4(0.f, 0.f, 0.f, 0.f);
            if (HAS_BIAS) tb = tab4[c0 / 4 + q];
            float x0 = __uint_as_float(su[4 * q]) * sc, x1 = __uint_as_float(su[4 * q + 1]) * sc;
            float x2 = __uint_as_float(su[4 * q + 2]) * sc, x3 = __uint_as_float(su[4 * q + 3]) * sc;
            if (HAS_BIAS) {
              x0 = fmaf(gl, tb.x, x0); x1 = fmaf(gl, tb.y, x1); x2 = fmaf(gl, tb.z, x2); x3 = fmaf(gl, tb.w, x3);
            }
            if (msk) {
              const float4 kb = *reinterpret_cast<const float4*>(kbias + c0 + 4 * q);
              x0 += kb.x; x1 += kb.y; x2 += kb.z; x3 += kb.w;
            }
            mx = fmaxf(fmaxf(mx, fmaxf(x0, x1)), fmaxf(x2, x3));
          }
        }
        return mx;
      };

      // rows that have not seen a finite score yet take this tile's maximum as their reference (first tile, or only masked
      // keys so far); they hold l = 0 and an all-zero accumulator, so nothing has to be rescaled
      if (__any_sync(0xffffffffu, m_ref == -INFINITY)) {
        const float mx = tile_max();
        if (m_ref == -INFINITY) m_ref = mx;
      }
      // one pass over the tile: probabilities (relative to m_ref) -> bf16 P tile in shared memory; returns the row sum.
      // MSK is a compile-time flag so that the common tiles (no padded key) carry no mask arithmetic at all.
      auto softmax_tile = [&](auto MSK) -> float {
        constexpr bool kMsk = decltype(MSK)::value;
        const float neg_ref = (m_ref == -INFINITY) ? 0.f : -m_ref;
        float part0 = 0.f, part1 = 0.f, part2 = 0.f, part3 = 0.f;
#pragma unroll 1
        for (int cc = 0; cc < 4; ++cc) {
          const int c0 = cc * 32;
          uint32_t su[32];
          lds_row32(s_row + c0, su);
          float pv[32];
          uint32_t rowbits = 0, hbits = 0;
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            float4 tb = make_float4(0.f, 0.f, 0.f, 0.f), kb = make_float4(0.f, 0.f, 0.f, 0.f);
            if (HAS_BIAS) tb = tab4[c0 / 4 + q];
            if (kMsk) kb = *reinterpret_cast<const float4*>(kbias + c0 + 4 * q);
            const float tbv[4] = {tb.x, tb.y, tb.z, tb.w};
            const float kbv[4] = {kb.x, kb.y, kb.z, kb.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const int j = 4 * q + e;
              float x = fmaf(__uint_as_float(su[j]), sc, neg_ref);
              if (HAS_BIAS) x = fmaf(gl, tbv[e], x);
              if (kMsk) x += kbv[e];
              const float ex = fast_exp2(x);
              // four independent partial sums: the normaliser (taken before dropout) is not one 128-long dependent chain
              if (e == 0) part0 += ex; else if (e == 1) part1 += ex; else if (e == 2) part2 += ex; else part3 += ex;
              if (DROP) {
                if ((j & 1) == 0) hbits = drop_bits(rk0, rk1, static_cast<uint32_t>(k0 + c0 + j) >> 1);
                const bool keep = (j & 1) ? drop_keep_hi(hbits, p.drop_thr_hi) : drop_keep_lo(hbits, p.drop_thr_hi);
                if (keep) rowbits |= (1u << j);  // this row's decisions for the 32 key columns
                pv[j] = keep ? ex : 0.f;
              } else {
                pv[j] = ex;
              }
            }
          }
          if (DROP) {
            // the backward walks key-major: store, per key column, one word whose bit l is the decision of query row l of this warp
            const uint32_t mword = warp_bit_transpose(rowbits, lane);
            mask_row[k0 + c0 + lane] = mword;
          }
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            uint4 w;
            w.x = pack_bf16x2(pv[g * 8 + 0], pv[g * 8 + 1]);
            w.y = pack_bf16x2(pv[g * 8 + 2], pv[g * 8 + 3]);
            w.z = pack_bf16x2(pv[g * 8 + 4], pv[g * 8 + 5]);
            w.w = pack_bf16x2(pv[g * 8 + 6], pv[g * 8 + 7]);
            store_sw128_chunk(sP, r, (c0 >> 3) + g, w);
          }
        }
        return (part0 + part1) + (part2 + part3);
      };
      float lsum, fac = 1.0f;
#pragma unroll 1
      while (true) {
        lsum = msk ? softmax_tile(std::true_type{}) : softmax_tile(std::false_type{});
        if (!__any_sync(0xffffffffu, !(lsum < kRebase))) break;
        // ---- re-base (rare): a score outgrew the reference by 2^80.  Move this warp's rows to the tile maximum: rescale the row
        // sums now and the accumulator rows before the next PV product (row_scale), then recompute the tile.
        const float m_new = fmaxf(m_ref, tile_max());
        const float factor = (m_ref == -INFINITY) ? 0.f : fast_exp2(m_ref - m_new);
        fac *= factor;
        l_run *= factor;
        m_ref = m_new;
      }
      l_run += lsum;
      row_scale[r] = fac;

      // ---- O += P V_n (two 64-row halves, accumulators in registers)
      fence_proxy_async_smem();  // generic-proxy smem writes (P) -> visible to the tensor core (async proxy)
      named_bar_sync(1, kAttnTile);
      if (n > 0) {  // re-based rows (factor 1 everywhere else: exact)
#pragma unroll
        for (int hm = 0; hm < 2; ++hm) {
          const float f0 = row_scale[64 * hm + fr], f1 = row_scale[64 * hm + fr + 8];
#pragma unroll
          for (int i = 0; i < 32; ++i) o_acc[hm][i] *= ((i >> 1) & 1) ? f1 : f0;
        }
      }
      mbar_wait(&v_full, n & 1);
      const uint32_t bv = smem_u32(sV);
      wgmma_fence();
#pragma unroll
      for (int hm = 0; hm < 2; ++hm) {
        const uint32_t a = smem_u32(sP) + hm * 8192;
#pragma unroll
        for (int k = 0; k < 8; ++k)
          wgmma_m64n64k16<0, 1>(o_acc[hm], make_smem_desc_sw128(a + (k >> 2) * 16384 + (k & 3) * 32, 16, 1024),
                                make_smem_desc_sw128(bv + k * 2048, 8192, 1024), (n > 0 || k > 0) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      if (lane == 0) mbar_arrive(&v_empty);
      named_bar_sync(1, kAttnTile);  // every MMA of the tile has retired: the score / P tiles and row_scale may be overwritten
    }

    row_scale[r] = l_run > 0.f ? (DROP ? p.drop_rp : 1.0f) / l_run : 0.f;
    if (row_valid && p.lse != nullptr)
      p.lse[(static_cast<long long>(b) * p.H + h) * T + q0 + r] = (l_run > 0.f) ? (m_ref + log2f(l_run)) : INFINITY;
    named_bar_sync(1, kAttnTile);
    // O / l straight from the fragments: bf16 pairs of the thread's rows fr, fr + 8 of each half
#pragma unroll
    for (int hm = 0; hm < 2; ++hm) {
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int row = 64 * hm + fr + 8 * rr;
        if (q0 + row < T) {
          const float inv = row_scale[row];
          __nv_bfloat16* dst = p.out + (static_cast<long long>(b) * T + q0 + row) * D + h * kHeadDim + 2 * (lane & 3);
#pragma unroll
          for (int g = 0; g < 8; ++g)
            *reinterpret_cast<uint32_t*>(dst + 8 * g) =
                pack_bf16x2(o_acc[hm][4 * g + 2 * rr] * inv, o_acc[hm][4 * g + 2 * rr + 1] * inv);
        }
      }
    }
  }
}

int make_qkv_tmap(CUtensorMap* out, const void* qkv, int T, int B, int D3, int box_rows);

}  // namespace b200

using namespace b200;

extern "C" {

// out[b,t,h*64+d] = softmax_j(scale q.k + gate*tab[j-i], key padding) v     (WavLM/modules.py:540-563 replaced)
// qkv: bf16 [B,T,3D] fused projection output; gate: fp32 [B,H,T] or NULL; tab: fp32 [H,2T-1] or NULL (no bias);
// key_pad: uint8 [B,T] or NULL; out: bf16 [B,T,D]; lse: fp32 [B,H,T] (log2-domain log-sum-exp, saved for backward).
// Rows of `out` at padded query frames are unspecified-but-finite (zeros where a whole 128-row block is padded).
int b200s_attn_fwd_dropout(const void* qkv, const float* gate, const float* tab, const uint8_t* key_pad, void* out, float* lse,
                           int B, int T, int H, float scale, float drop_p, uint32_t key0, uint32_t key1, uint32_t* drop_mask,
                           b200s_stream stream) {
  B200_CHECK_ARG(qkv && out, "attn_fwd: null pointer");
  B200_CHECK_ARG(drop_p >= 0.f && drop_p < 1.f, "attn_fwd: dropout p=%f out of range [0,1)", static_cast<double>(drop_p));
  B200_CHECK_ARG(drop_p == 0.f || drop_mask != nullptr, "attn_fwd: dropout needs the mask buffer (b200s_attn_dropout_mask_words)");
  B200_CHECK_ARG(static_cast<long long>(B) * H * T < (1LL << 32), "attn_fwd: B*H*T exceeds the 32-bit dropout row counter");
  const int D = H * kHeadDim;
  CUtensorMap tm;
  AttnParams p;
  memset(&p, 0, sizeof(p));
  p.T = T; p.H = H; p.B = B; p.D = D;
  p.n_tiles = ceil_div(T, kAttnTile);
  B200_CHECK_ARG(T >= 1, "attn_fwd: T=%d out of range", T);
  const int smem = kFwdSmem;
  if (make_qkv_tmap(&tm, qkv, T, B, 3 * D, kAttnTile)) return -3;
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
  void (*kern)(const CUtensorMap, const AttnParams) =
      tab != nullptr ? (drop ? attn_fwd_kernel<true, true> : attn_fwd_kernel<true, false>)
                     : (drop ? attn_fwd_kernel<false, true> : attn_fwd_kernel<false, false>);
  B200_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  B200_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(kFwdThreads), smem, st, tm, p));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_attn_fwd(const void* qkv, const float* gate, const float* tab, const uint8_t* key_pad, void* out, float* lse,
                   int B, int T, int H, float scale, b200s_stream stream) {
  return b200s_attn_fwd_dropout(qkv, gate, tab, key_pad, out, lse, B, T, H, scale, 0.f, 0u, 0u, nullptr, stream);
}

long long b200s_attn_dropout_mask_words(int B, int T, int H) { return attn_drop_mask_words(B, H, T); }

}  // extern "C"
