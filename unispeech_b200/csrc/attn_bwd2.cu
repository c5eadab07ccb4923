// Fused attention backward with the gated relative-position bias (autograd of WavLM/modules.py:521-563): ONE tensor-core
// kernel produces dQ, dK, dV, d gate and d tab, so the probabilities are recomputed once.  wgmma + TMA (sm_90a).
//
// CTA = 128 keys of one (batch, head); it walks over the 128-row query tiles with two warpgroups (WG w = 0, 1).  The scores
// are computed transposed: WG w owns key rows 64 w .. 64 w + 63 against all 128 queries of the
// tile, which are also the rows of its dK / dV accumulators (registers, across the whole loop).  Per query tile:
//   S^T = K_w Q^T, dP^T = V_w dO^T          wgmma m64n128k16, two commit groups
//   P^T = exp2(S^T*scale*log2e + gate_i*log2e*tab[j-i] + keymask_j - lse_i)      on the S^T fragments while dP^T is still
//                                           on the tensor pipe;  dS^T = P^T o (dP^T - Delta_i) * scale  after it lands
//   dV += P^T dO                            A = P^T as bf16 register fragments (wgmma RS form), B = dO MN-major: P never goes
//                                           through shared memory
//   dS^T -> shared memory (bf16 [2 query blocks][128 keys][64 queries], SWIZZLE_128B); gate*dS/scale -> a bf16 [128][130]
//   staging tile; d gate_i = sum_j dS_ij tab[j-i]: a column sum of the fragments (shuffles + one shared slot per warp),
//   one global atomic per query and tile
//   (all 256 threads) barrier, then
//   dK += dS^T Q                            A = this WG's rows of the dS^T tile (K-major), B = Q MN-major
//   dQ_i = dS K                             this WG's 64 queries: A = dS^T tile read MN-major, B = K MN-major
//   d tab[d] = sum_i gate_i dS_{i,i+d}      diagonal sums of the staged tile while the dV / dK / dQ MMAs run, into two
//                                           128-float shared blocks (see below) flushed with atomics
//   dQ (fp32) -> the WG's half of the staging tile (it aliases the WG's own gate*dS rows), then one thread adds it into
//   the fp32 [B,T,D] buffer with TMA bulk-tensor reductions (the box clips at T); the buffer is rewritten only after the
//   reduction has read it
// Thread 0 loads K / V once and refills a 2-stage ring of Q / dO tiles with TMA as soon as both warpgroups are done with a
// stage; the per-query lse, Delta*scale and gate terms of the next tile are loaded into registers while the tile's dK / dQ
// MMAs run and stored to their stage at its end.
// Registers: the S^T and dP^T fragments and the dK / dV accumulators alone take 192 per thread, and ptxas uses 248-255 (CUDA
// 12.9).  Hence:
// - No producer warpgroup.  With one (384 threads, setmaxnreg.dec<40> / setmaxnreg.inc<232>) an earlier revision of this
//   kernel, which also took dS^T as a register operand, compiled with 364-424 bytes of spills per variant, against 0-60 for
//   the same code at 256 threads.
// - dK reads dS^T from shared memory, not registers: 32 more registers live through the dS^T pass spilled.
// - Query tiles do not overlap: issuing tile qi+1's S^T / dP^T (128 registers) before tile qi's dK / dQ group retires does
//   not fit, and the two warpgroups run in step (the dS^T tile and the staging tile are shared by both).  Overlap is within a
//   tile: exp2 with the dP^T chain, and the diagonal sums, the d gate flush and the next tile's loads with dV / dK / dQ.
// - The bias variant without dropout keeps 4 bytes of spill (a loop-invariant value stored before the query loop and
//   reloaded once per query tile); the other three variants have none.
// Bias window: inside a tile the bias of (key row kr, query column c) is tab[h, m - 128 + k0 - 128 qi + T - 1] with the window
// coordinate m = kr - c + 128 in [1, 255], kept in a 256-float shared window at a fixed place (every read is base + immediate,
// which the register budget needs).  The window of tile qi + 1 is the window of tile qi shifted by 128, so once tile qi's reads
// are behind its middle barrier, threads 0..127 move the lower half up and copy the one new entry each into the lower half
// (cp.async: no register is carried across the MMAs).  Shared memory is 176,128 bytes for every T.
// d tab: two 128-float accumulator blocks, lower (m < 128: the wrapped diagonal tasks) and upper (m >= 128).  The upper block of
// tile qi gets no contribution from a later tile, so after tile qi it is flushed to global memory, the lower block moves up
// (it continues as the upper block of tile qi + 1) and the lower block is cleared.  At most NQ * 128 + 128 global atomics per CTA.
// Dropout: the keep bit of (query i, key j) is bit i & 31 of word drop_mask[block(i), j], written by the forward kernel.
// Padding: a CTA whose 128 keys are all padded writes zero dK / dV rows and exits; query tiles that are fully padded at the end
// of the utterance are not visited (their probabilities are zero: the forward leaves lse = +inf there).
// Head widths 80 and 120 (no bias; tiles, maps and MMA shapes per width in attn_common.cuh): dK / dV take 80 or 128
// accumulator registers instead of 64, which the 128-query tiling above cannot afford, so the query tile is 64 rows: S^T / dP^T
// are m64n64 (32 registers each) and the dS^T tile is one [128 keys][64 queries] block.  The dropout mask words are the same
// (a tile covers two 32-query blocks instead of four).  dQ = dS K is decomposed per width, each dQ element reduced through
// the head-shaped fp32 map ([64 queries][32 columns] SWIZZLE_128B boxes, and at 80 a [64][16] unswizzled one):
// - 64: warpgroup w computes queries 64 w .. 64 w + 63 of the tile over all 128 keys, once per key tile;
// - 80: each warpgroup computes its 64 keys' share of the tile's 64 x 80 dQ (the reductions add the two shares);
// - 120: warpgroup w computes columns 64 w .. 64 w + 63 of the tile's 64 x 120 dQ over all 128 keys, once per key tile; the
//   box at column 96 clips at 120.
#include "../../include/unispeech_b200.h"
#include "attn_common.cuh"
#include "common.h"

#include <algorithm>

namespace b200 {

namespace {

__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

constexpr int kWStride = 130;      // bf16 per staged row of the gate*dS tile (65 words: conflict-free diagonal reads)
constexpr int kFThreads = 256;     // two warpgroups

// shared-memory map of head width HD (bytes from the 1024-aligned base); at HD = 64:
//   K 0, V 16384 (16 KB tiles); Q 32768, dO 65536 (2 stages x 16 KB); dS^T 98304 ([2 query blocks][128 keys][64 queries] bf16,
//   32 KB); at 131072 the gate*dS staging for the diagonal sums ([128 keys][kWStride] bf16, 33280 B), aliased by the dQ
//   staging of WG 0 at kFW and of WG 1 at kFW + kFDQ1 (16 KB each: two [64 queries][32] fp32 SWIZZLE_128B boxes, inside each
//   WG's own staged rows); per stage lse, Delta*scale, gate*log2e, gate/scale [4][128] fp32 at 164864; d gate partial column
//   sums [8 warps][128] fp32 at 168960; 174080 bytes with the alignment slack (+ 2 KB static: bias window and d tab blocks).
// At HD = 80: 20 KB K / V tiles, 10 KB Q / dO stages (64 queries), one 16 KB dS^T block, and 20 KB of dQ staging per WG
// (two [64][32] SWIZZLE_128B boxes and one [64][16] fp32 box): 148480 bytes.  At HD = 120: 32 KB K / V tiles, 16 KB Q / dO
// stages, one 16 KB dS^T block and 16 KB of dQ staging per WG: 189440 bytes.  All are the same for every T.
template <int HD>
struct BwdMap {
  static constexpr int kQT = HD == 64 ? kAttnTile : 64;  // queries per tile
  static constexpr int kKV = kAttnTile * HeadTile<HD>::kCols * 2;  // one K or V tile
  static constexpr int kQS = kQT * HeadTile<HD>::kCols * 2;        // one Q or dO stage
  static constexpr int kFK = 0, kFV = kKV, kFQ = 2 * kKV, kFDO = kFQ + 2 * kQS, kFDS = kFDO + 2 * kQS;
  static constexpr int kFW = kFDS + kAttnTile * kQT * 2;
  static constexpr int kFDQ1 = HD == 64 ? 17408 : HD == 80 ? 64 * HD * 4 : 16384;
  static constexpr int kFWBytes = kFDQ1 + (HD == 80 ? 64 * HD * 4 : 16384);
  static constexpr int kFScal = kFW + kFWBytes;
  static constexpr int kFDg = kFScal + 2 * 4 * 512;
  static constexpr int kFSmem = kFDg + 8 * 512 + 1024;
};
static_assert(BwdMap<64>::kFDS == 98304 && BwdMap<64>::kFScal == 164864 && BwdMap<64>::kFSmem == 174080, "HD 64 map");
static_assert(BwdMap<80>::kFSmem == 148480 && BwdMap<120>::kFSmem == 189440, "HD 80 / 120 maps");

}  // namespace

template <int HD, bool HAS_BIAS, bool DROP>
__global__ void __launch_bounds__(kFThreads, 1) attn_bwd_fused_kernel(const __grid_constant__ CUtensorMap tm_qkv,
                                                                      const __grid_constant__ CUtensorMap tm_do,
                                                                      const __grid_constant__ CUtensorMap tm_dq,
                                                                      const __grid_constant__ CUtensorMap tm_qkv16,
                                                                      const __grid_constant__ CUtensorMap tm_do16,
                                                                      const __grid_constant__ CUtensorMap tm_dq16,
                                                                      const __grid_constant__ AttnParams p) {
  using HT = HeadTile<HD>;
  static_assert(HT::kBias || !HAS_BIAS, "the relative-position bias at this head width");
  using M = BwdMap<HD>;
  constexpr int QT = M::kQT, kFDS = M::kFDS, kFW = M::kFW, kFDQ1 = M::kFDQ1;
  pdl_grid_sync();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int k0 = blockIdx.x * kAttnTile, h = blockIdx.y, b = blockIdx.z;
  const int T = p.T, D = p.D, N = p.n_tiles;
  const long long bh = static_cast<long long>(b) * p.H + h;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // 1024-aligned, still a __shared__ pointer (LDS/STS, not generic)
  uint8_t* sK = smem + M::kFK;
  uint8_t* sV = smem + M::kFV;
  uint8_t* sQ = smem + M::kFQ;
  uint8_t* sDO = smem + M::kFDO;
  uint8_t* sDS = smem + kFDS;
  float* scal = reinterpret_cast<float*>(smem + M::kFScal);
  float* dgp = reinterpret_cast<float*>(smem + M::kFDg);
  // static, not in the dynamic map: addressed by immediates, which keeps the bias variants within their register budget
  __shared__ __align__(16) float win_s[2 * kAttnTile];    // bias window of the current query tile, by m
  __shared__ float dtab_acc[2 * kAttnTile];                // d tab blocks: lower (m < 128), upper

  __shared__ uint64_t kv_full, qdo_full[2];
  __shared__ uint32_t key_mask_s[4];  // bit j of word j>>5: key k0 + j is padded / beyond T

  // ---- padding: which of this CTA's keys are masked, and how many query tiles hold a valid query.  ONE pass over the
  // utterance's pad bytes (every thread takes a few), one block-wide reduction: the prologue pays a single global-load latency.
  __shared__ int nq_s;
  if (tid == 0) nq_s = 1;
  int NQ = QT == kAttnTile ? N : (T + QT - 1) / QT;  // query tiles to visit
  {
    bool masked = false;
    if (tid < kAttnTile) {
      const int j = k0 + tid;
      masked = (j >= T) || (p.key_pad != nullptr && p.key_pad[static_cast<long long>(b) * T + j] != 0);
      const uint32_t bal = __ballot_sync(0xffffffffu, masked);
      if (lane == 0) key_mask_s[warp] = bal;
    }
    int last_live = -1;
    if (p.key_pad != nullptr) {
      for (int i = tid; i < T; i += kFThreads)
        if (p.key_pad[static_cast<long long>(b) * T + i] == 0) last_live = i;   // increasing i: the last hit is the largest
    }
    const int n_masked = __syncthreads_count(masked);
    if (n_masked == kAttnTile) {
      // nothing attends to these keys: dK = dV = 0
      if (tid < kAttnTile && k0 + tid < T) {
        __nv_bfloat16* dst = p.dqkv + (static_cast<long long>(b) * T + k0 + tid) * (3 * D) + D + h * HD;
#pragma unroll
        for (int g = 0; g < HD / 8; ++g) {
          *reinterpret_cast<uint4*>(dst + g * 8) = make_uint4(0u, 0u, 0u, 0u);
          *reinterpret_cast<uint4*>(dst + D + g * 8) = make_uint4(0u, 0u, 0u, 0u);
        }
      }
      return;
    }
    if (p.key_pad != nullptr) {
      if (last_live >= 0) atomicMax(&nq_s, last_live / QT + 1);
      __syncthreads();
      NQ = nq_s;
    }
  }

  if (tid == 0) {
    // thread 0 initialises the barriers itself and puts K, V and the first Q / dO tiles in flight right away: they
    // land while the rest of the CTA is still filling the tables (the other warps see the barriers after the __syncthreads below)
    tma_prefetch_desc(&tm_qkv);
    tma_prefetch_desc(&tm_do);
    tma_prefetch_desc(&tm_dq);
    if (HT::kTail) {
      tma_prefetch_desc(&tm_qkv16);
      tma_prefetch_desc(&tm_do16);
      tma_prefetch_desc(&tm_dq16);
    }
    mbar_init(&kv_full, 1);
    for (int i = 0; i < 2; ++i) mbar_init(&qdo_full[i], 1);
    fence_mbar_init();
    mbar_expect_tx(&kv_full, 2 * M::kKV);
    tma_load_head<HD, kAttnTile, QT>(sK, &tm_qkv, &tm_qkv16, &kv_full, p.H + h, k0, b);
    tma_load_head<HD, kAttnTile, QT>(sV, &tm_qkv, &tm_qkv16, &kv_full, 2 * p.H + h, k0, b);
    for (int qi = 0; qi < 2 && qi < NQ; ++qi) {
      mbar_expect_tx(&qdo_full[qi], 2 * M::kQS);
      tma_load_head<HD, QT, QT>(sQ + qi * M::kQS, &tm_qkv, &tm_qkv16, &qdo_full[qi], h, qi * QT, b);
      tma_load_head<HD, QT, QT>(sDO + qi * M::kQS, &tm_do, &tm_do16, &qdo_full[qi], h, qi * QT, b);
    }
  }

  // global index of window entry m of query tile qi: tab[h, m + win_base - 128 qi] (0 outside [0, 2T - 1))
  const int win_base = k0 - kAttnTile + (T - 1);
  if (HAS_BIAS) {  // tile 0's window, one entry per thread; cleared d tab blocks
    const int gi = tid + win_base;
    win_s[tid] = (gi >= 0 && gi < 2 * T - 1) ? p.tab[static_cast<long long>(h) * (2 * T - 1) + gi] : 0.f;
    dtab_acc[tid] = 0.f;
  }
  // per-query terms of a query tile, two per thread: threads 0..127 lse and Delta*scale, threads 128..255 gate*log2e and
  // gate/scale of query tid & 127 (lse = +inf marks out-of-range queries: p = exp2(-inf) = 0)
  const float inv_scale = 1.0f / p.scale;
  auto load_terms = [&](int qi, float& t0, float& t1) {
    const int i = qi * QT + (tid & 127);
    t0 = tid < kAttnTile ? INFINITY : 0.f;
    t1 = 0.f;
    if (i < T) {
      if (tid < kAttnTile) {
        t0 = p.lse[bh * T + i];
        t1 = p.delta[bh * T + i] * p.scale;
      } else if (HAS_BIAS) {
        const float gate = (p.gate != nullptr) ? p.gate[bh * T + i] : 1.0f;
        t0 = gate * kLog2e;
        t1 = gate * inv_scale;
      }
    }
  };
  auto store_terms = [&](int qi, float t0, float t1) {
    float* ts = scal + (qi & 1) * 4 * kAttnTile + (tid >> 7) * 2 * kAttnTile + (tid & 127);
    ts[0] = t0;
    ts[kAttnTile] = t1;
  };
  {
    float t0, t1;
    load_terms(0, t0, t1);
    store_terms(0, t0, t1);
  }
  __syncthreads();

  {
    const int w = warp >> 2;                 // warpgroup: key rows 64 w .. 64 w + 63
    const int wq = warp & 3;
    const int kr = 64 * w + 16 * wq + (lane >> 2);   // first of this thread's two fragment key rows (the other is kr + 8)
    const int fc = 2 * (lane & 3);                    // column of fragment element 0 inside each 8-column group
    const float sc = p.scale * kLog2e;
    bool row_masked[2];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) row_masked[rr] = ((key_mask_s[(kr + 8 * rr) >> 5] >> ((kr + 8 * rr) & 31)) & 1u) != 0u;
    const bool flusher = (tid & 127) == 0;   // issues this WG's dQ reductions
    uint8_t* dq_stage = smem + kFW + w * kFDQ1;
    const uint32_t ak = smem_u32(sK) + w * 8192, av = smem_u32(sV) + w * 8192;  // this WG's 64 rows of K, V
    uint32_t* wtile = reinterpret_cast<uint32_t*>(smem + kFW);
    const uint32_t* kw_row = p.drop_mask + bh * (4 * N) * (N * kAttnTile) + k0 + kr;  // dropout words of key row kr, block 0

    HeadAcc<HD> dv_acc, dk_acc;  // written by the first tile's MMAs (scale_d = 0)

    // diagonal sums of the staged gate*dS tile of query tile qi.  Task (e, s): elements (key (ii + e) & 127, query ii) for
    // ii = 16 s .. 16 s + 15: diagonal key - query = e (not wrapped, ii + e < 128) or e - 128 (wrapped).  The wrap point is a
    // per-task constant, so every load is base + immediate.  The two diagonals are summed separately: the wrapped sum taken as
    // (all - not wrapped) would carry an error of EPS32 times the other diagonal's sum, which can be larger than its own.
    auto diag_task = [&](int qi, int e, int s) {
      const int w0 = kAttnTile - e - 16 * s;  // queries ii = 16 s + c with c >= w0 are on the wrapped diagonal
      const uint32_t base_nw = smem_u32(wtile) + static_cast<uint32_t>(((16 * s + e) * kWStride + 16 * s) * 2);
      const uint32_t base_w = base_nw - static_cast<uint32_t>(kAttnTile * kWStride * 2);
      float acc_w = 0.f, acc_nw = 0.f;
#pragma unroll
      for (int c = 0; c < 16; ++c) {
        const bool wrapped = c >= w0;
        uint32_t v16;
        asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v16) : "r"((wrapped ? base_w : base_nw) + c * (kWStride + 1) * 2));
        const float v = __uint_as_float(v16 << 16);
        if (wrapped) acc_w += v;
        else acc_nw += v;
      }
      if (w0 > 0) atomicAdd(&dtab_acc[kAttnTile + e], acc_nw);   // upper block (m = e + 128)
      if (w0 < 16) atomicAdd(&dtab_acc[e], acc_w);               // lower block (m = e)
    };

    mbar_wait(&kv_full, 0);
    for (int qi = 0; qi < NQ; ++qi) {
      const int st = qi & 1;
      mbar_wait(&qdo_full[st], (qi >> 1) & 1);
      const uint32_t bq = smem_u32(sQ + st * M::kQS), bdo = smem_u32(sDO + st * M::kQS);
      float s_acc[QT / 2], d_acc[QT / 2];
      // S^T = K_w Q^T and dP^T = V_w dO^T over the head width
      wgmma_fence();
      mma_k_head<HD, QT>(s_acc, ak, 64 * w, bq);
      wgmma_commit();
      mma_k_head<HD, QT>(d_acc, av, 64 * w, bdo);
      wgmma_commit();
      // dropout keep words of this thread's two key rows for the tile's 32-query blocks
      uint32_t kw[2][QT / 32];
      if (DROP) {
#pragma unroll
        for (int rr = 0; rr < 2; ++rr)
#pragma unroll
          for (int blk = 0; blk < QT / 32; ++blk)
            kw[rr][blk] = kw_row[(qi * (QT / 32) + blk) * (N * kAttnTile) + 8 * rr];  // < 512 N^2: int below T = 262,016
      }
      // the previous tile's dQ reduction has read this WG's staging buffer before the buffer is written again
      if (qi > 0) {
        if (flusher) bulk_wait_read0();
        named_bar_sync(2 + w, 128);
      }
      const float* ts = scal + st * 4 * kAttnTile;   // lse, Delta*scale, gate*log2e, gate/scale of the tile's queries
      const int tb0 = kr + kAttnTile;   // win_s index of (key row kr, query 0)

      // P^T on the S^T fragments while the dP^T chain runs (fp32, in place)
      wgmma_wait<1>();
#pragma unroll
      for (int g = 0; g < QT / 8; ++g) {
        const float2 lse = *reinterpret_cast<const float2*>(ts + 8 * g + fc);
        float2 gl = make_float2(0.f, 0.f);
        if (HAS_BIAS) gl = *reinterpret_cast<const float2*>(ts + 2 * kAttnTile + 8 * g + fc);
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int idx = 4 * g + 2 * rr + e;
            float x = fmaf(s_acc[idx], sc, -(e ? lse.y : lse.x));
            if (HAS_BIAS) x = fmaf(e ? gl.y : gl.x, win_s[tb0 + 8 * rr - (8 * g + fc + e)], x);
            const float pr = ex2f(x);
            s_acc[idx] = row_masked[rr] ? 0.f : pr;
          }
        }
      }

      // dS^T after dP^T lands; bf16 operands for dV / dK, the dS^T tile and the staging tile; d gate column partials
      wgmma_wait<0>();
      uint32_t p16[QT / 4];
#pragma unroll
      for (int hq = 0; hq < QT / 64; ++hq) {   // query halves: 16 d gate partials live at a time
      float dg[16];
#pragma unroll
      for (int g = 8 * hq; g < 8 * hq + 8; ++g) {
        const float2 dsc = *reinterpret_cast<const float2*>(ts + kAttnTile + 8 * g + fc);
        float2 gos = make_float2(0.f, 0.f);
        if (HAS_BIAS) gos = *reinterpret_cast<const float2*>(ts + 3 * kAttnTile + 8 * g + fc);
        dg[2 * g - 16 * hq] = 0.f;
        dg[2 * g + 1 - 16 * hq] = 0.f;
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const int r = kr + 8 * rr;
          float pd2[2], ds2[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int idx = 4 * g + 2 * rr + e;
            const float pr = s_acc[idx];
            float dpv = d_acc[idx];
            bool keep = true;
            if (DROP) {  // O = (P o M) V / (1-p):  dP = M o (dO V^T) / (1-p);  dV takes the dropped probabilities (scaled at the end)
              keep = ((kw[rr][g >> 2] >> ((8 * g + fc + e) & 31)) & 1u) != 0u;
              dpv = keep ? dpv * p.drop_rp : 0.f;
            }
            const float ds = pr * fmaf(dpv, p.scale, -(e ? dsc.y : dsc.x));  // dS * scale
            pd2[e] = keep ? pr : 0.f;
            ds2[e] = ds;
            if (HAS_BIAS) dg[2 * g + e - 16 * hq] = fmaf(ds, win_s[tb0 + 8 * rr - (8 * g + fc + e)], dg[2 * g + e - 16 * hq]);
          }
          p16[2 * g + rr] = pack_bf16x2(pd2[0], pd2[1]);
          // dS^T tile: query block g >> 3, row = key, 16-byte chunk g & 7 (SWIZZLE_128B)
          *reinterpret_cast<uint32_t*>(sDS + (g >> 3) * 16384 + r * 128 + (((g & 7) ^ (r & 7)) << 4) + fc * 2) =
              pack_bf16x2(ds2[0], ds2[1]);
          if (HAS_BIAS) wtile[r * (kWStride / 2) + 4 * g + (fc >> 1)] = pack_bf16x2((gos.x) * ds2[0], (gos.y) * ds2[1]);
        }
      }
      if (HAS_BIAS && p.dgate != nullptr) {
        // column sums over the warp's 16 key rows (reduce-scatter over lane bits 2..4): lane l keeps columns
        // 64 hq + 8 (l >> 2) + fc + e, e = 0, 1
        float a[8], c4[4], c2[2];
        {
          const bool up = (lane & 16) != 0;
#pragma unroll
          for (int i = 0; i < 8; ++i) a[i] = (up ? dg[i + 8] : dg[i]) + __shfl_xor_sync(0xffffffffu, up ? dg[i] : dg[i + 8], 16);
        }
        {
          const bool up = (lane & 8) != 0;
#pragma unroll
          for (int i = 0; i < 4; ++i) c4[i] = (up ? a[i + 4] : a[i]) + __shfl_xor_sync(0xffffffffu, up ? a[i] : a[i + 4], 8);
        }
        {
          const bool up = (lane & 4) != 0;
#pragma unroll
          for (int i = 0; i < 2; ++i) c2[i] = (up ? c4[i + 2] : c4[i]) + __shfl_xor_sync(0xffffffffu, up ? c4[i] : c4[i + 2], 4);
        }
        *reinterpret_cast<float2*>(dgp + warp * kAttnTile + 64 * hq + 8 * (lane >> 2) + fc) = make_float2(c2[0], c2[1]);
      }
      }

      // ---- dV += P^T dO (this WG's 64 keys; A = P^T from registers)
      wgmma_fence();
      mma_n_head<HD, QT>(dv_acc, p16, bdo, qi > 0);  // K = the tile's queries
      wgmma_commit();
      fence_proxy_async_smem();  // generic-proxy smem writes -> visible to the tensor core (async proxy)
      named_bar_sync(1, kFThreads);

      // ---- dK += dS^T Q (this WG's 64 keys; A = its rows of the dS^T tile, K-major).  From shared memory rather than registers:
      // 32 more live registers through the dS^T pass would spill.
      mma_n_head<HD, QT>(dk_acc, smem_u32(sDS), 64 * w, bq, qi > 0);
      // ---- dQ = dS K.  HD 64: this WG's 64 queries, K = 128 keys.  HD 80: the tile's 64 queries, K = this WG's 64 keys (the two
      // WGs' shares are added by the reductions).  HD 120: the tile's 64 queries x this WG's 64 columns, K = 128 keys.  A = the
      // dS^T tile read MN-major, 16 keys per step.
      float dq[32], dq16[8];
      constexpr int kDqSteps = QT == kAttnTile || HD == 120 ? 8 : 4;
      const uint32_t dq_a = smem_u32(sDS) + (QT == kAttnTile ? w * 16384 : HD == 120 ? 0 : w * 8192);
      const uint32_t dq_b = smem_u32(sK) + (QT == kAttnTile ? 0 : HD == 120 ? w * 16384 : w * 8192);
#pragma unroll
      for (int k = 0; k < kDqSteps; ++k) {
        const uint64_t da = make_smem_desc_sw128(dq_a + k * 2048, 16384, 1024);
        wgmma_m64n64k16<1, 1>(dq, da, make_smem_desc_sw128(dq_b + k * 2048, 8192, 1024), k > 0 ? 1u : 0u);
        if (HD == 80)
          wgmma_m64n16k16<1, 1>(dq16, da, make_smem_desc_sw32(smem_u32(sK) + kAttnTile * 128 + w * 2048 + k * 512), k > 0 ? 1u : 0u);
      }
      wgmma_commit();
      // the next tile's per-query terms: loaded while the MMAs run, stored once this tile's have been read (not earlier: live
      // across the exp2 pass they would push that pass over the register budget)
      float nt0, nt1;
      if (qi + 1 < NQ) {
        load_terms(qi + 1, nt0, nt1);
        if (HAS_BIAS && tid < kAttnTile) {
          // the window of tile qi + 1 (this tile's reads are behind the barrier above): the lower half moves up, the new
          // entry m = tid comes straight from global memory
          win_s[kAttnTile + tid] = win_s[tid];
          const int gi = tid + win_base - (qi + 1) * kAttnTile;
          const bool ok = gi >= 0;   // gi < 2T - 1 holds
          cp_async_4_zfill(win_s + tid, p.tab + static_cast<long long>(h) * (2 * T - 1) + (ok ? gi : 0), ok);
          cp_async_commit();
        }
      }
      if (HAS_BIAS) {  // the diagonal sums and the d gate flush while the MMAs run
#pragma unroll 1
        for (int s = tid >> 7; s < 8; s += 2) diag_task(qi, tid & 127, s);
        if (p.dgate != nullptr && tid < kAttnTile) {
          const int i = qi * kAttnTile + tid;
          float v = 0.f;
#pragma unroll
          for (int wp = 0; wp < 8; ++wp) v += dgp[wp * kAttnTile + tid];
          if (i < T) atomicAdd(p.dgate + bh * T + i, v * inv_scale);
        }
      }
      wgmma_wait<0>();
      if (qi + 1 < NQ) {
        store_terms(qi + 1, nt0, nt1);
        if (HAS_BIAS && tid < kAttnTile) cp_async_wait_all();
      }
      named_bar_sync(1, kFThreads);  // the Q / dO stage, the staging, dS^T and d gate tiles of this query tile are consumed
      if (tid == 0 && qi + 2 < NQ) {
        mbar_expect_tx(&qdo_full[st], 2 * M::kQS);
        tma_load_head<HD, QT, QT>(sQ + st * M::kQS, &tm_qkv, &tm_qkv16, &qdo_full[st], h, (qi + 2) * QT, b);
        tma_load_head<HD, QT, QT>(sDO + st * M::kQS, &tm_do, &tm_do16, &qdo_full[st], h, (qi + 2) * QT, b);
      }

      // dQ rows of this WG -> the staging boxes ([64 queries][32 fp32], SWIZZLE_128B, and at HD = 80 [64][16] fp32 behind
      // them; the staged dS already carries the softmax scale) -> TMA reductions into dq_acc[b, q, h*HD + col]
      {
        const int r0 = 16 * wq + (lane >> 2);
#pragma unroll
        for (int g = 0; g < 8; ++g)
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            const int r = r0 + 8 * rr, col = 8 * g + fc;
            *reinterpret_cast<float2*>(dq_stage + (col >> 5) * 8192 + r * 128 + ((((col & 31) >> 2) ^ (r & 7)) << 4) + (col & 3) * 4) =
                make_float2(dq[4 * g + 2 * rr], dq[4 * g + 2 * rr + 1]);
          }
        if (HD == 80) {
#pragma unroll
          for (int g = 0; g < 2; ++g)
#pragma unroll
            for (int rr = 0; rr < 2; ++rr)
              *reinterpret_cast<float2*>(dq_stage + 16384 + (r0 + 8 * rr) * 64 + (8 * g + fc) * 4) =
                  make_float2(dq16[4 * g + 2 * rr], dq16[4 * g + 2 * rr + 1]);
        }
      }
      fence_proxy_async_smem();
      named_bar_sync(2 + w, 128);
      const int dq_row = QT == kAttnTile ? qi * kAttnTile + 64 * w : qi * QT;
      if (flusher && dq_row < T) {
        const int dq_col = HD == 120 ? 64 * w : 0;
        tma_reduce_add_4d(&tm_dq, smem_u32(dq_stage), dq_col, h, dq_row, b);
        tma_reduce_add_4d(&tm_dq, smem_u32(dq_stage) + 8192, dq_col + 32, h, dq_row, b);
        if (HD == 80) tma_reduce_add_4d(&tm_dq16, smem_u32(dq_stage) + 16384, 64, h, dq_row, b);
        bulk_commit();
      }
      if (HAS_BIAS && tid >= kAttnTile) {
        // this tile's upper d tab block is complete (its diagonal sums are behind the closing barrier): flush it, move the lower
        // block up and clear it, before tile qi + 1's diagonal sums start after that tile's middle barrier
        const int e = tid - kAttnTile;
        const int gi = e + win_base + kAttnTile - qi * kAttnTile;
        const float v = dtab_acc[kAttnTile + e];
        dtab_acc[kAttnTile + e] = dtab_acc[e];
        dtab_acc[e] = 0.f;
        if (p.dtab != nullptr && gi < 2 * T - 1 && v != 0.f) atomicAdd(p.dtab + static_cast<long long>(h) * (2 * T - 1) + gi, v);
      }
    }
    if (flusher) bulk_wait0();
    // ---- dK / dV rows of this WG (keys k0 + 64 w ..): bf16 pairs straight from the fragments
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int key = k0 + kr + 8 * rr;
      if (key < T) {
        __nv_bfloat16* dst = p.dqkv + (static_cast<long long>(b) * T + key) * (3 * D) + h * HD + fc;
        dv_acc.store_row(dst + 2 * D, rr, DROP ? p.drop_rp : 1.0f);  // dV = (P o M)^T dO / (1-p)
        dk_acc.store_row(dst + D, rr, 1.0f);
      }
    }
  }

  if (HAS_BIAS && p.dtab != nullptr && tid >= kAttnTile) {
    // the last tile's lower d tab block, which this thread moved to the upper block at the end of the loop -> global (the
    // relative-position table is shared by all layers: atomics)
    const int gi = (tid - kAttnTile) + win_base - (NQ - 1) * kAttnTile;
    const float v = dtab_acc[tid];
    if (gi >= 0 && gi < 2 * T - 1 && v != 0.f) atomicAdd(p.dtab + static_cast<long long>(h) * (2 * T - 1) + gi, v);
  }
}

// Delta_i = sum_d dO_id O_id (fp32 [B,H,T]); also clears d gate, which the fused kernel accumulates with atomics.
template <int HD>
__global__ void __launch_bounds__(256) attn_delta2_kernel(const __nv_bfloat16* __restrict__ o,
                                                          const __nv_bfloat16* __restrict__ dout, int B, int T, int H,
                                                          float* __restrict__ delta, float* __restrict__ dgate) {
  pdl_grid_sync();
  const int lane = threadIdx.x & 31;
  const long long row = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (row >= static_cast<long long>(B) * T) return;
  const int D = H * HD;
  const long long b = row / T, t = row % T;
  for (int h = 0; h < H; ++h) {
    float part = 0.f;
#pragma unroll
    for (int c = 2 * lane; c < HD; c += 64) {  // column pairs: one per lane, and at HD 80 a second one for lanes 0..7
      const float2 a = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(o + row * D + h * HD + c));
      const float2 g = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(dout + row * D + h * HD + c));
      part += a.x * g.x + a.y * g.y;
    }
    const float s = warp_sum(part);
    if (lane == 0) {
      delta[(b * H + h) * T + t] = s;
      if (dgate != nullptr) dgate[(b * H + h) * T + t] = 0.f;
    }
  }
}

// dq_acc (fp32 [B*T, D]) -> bf16 into the q columns of dqkv [B*T, 3D]; the accumulator is cleared for the next layer.
__global__ void __launch_bounds__(256) attn_dq_convert_kernel(float* __restrict__ dq_acc, __nv_bfloat16* __restrict__ dqkv,
                                                              long long rows, int D) {
  pdl_grid_sync();
  const int vec_per_row = D / 8;
  const long long n = rows * vec_per_row;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = i / vec_per_row;
    const int c = static_cast<int>(i % vec_per_row) * 8;
    float4* src = reinterpret_cast<float4*>(dq_acc + row * D + c);
    const float4 a = src[0], bq = src[1];
    uint4 w;
    w.x = pack_bf16x2(a.x, a.y); w.y = pack_bf16x2(a.z, a.w);
    w.z = pack_bf16x2(bq.x, bq.y); w.w = pack_bf16x2(bq.z, bq.w);
    *reinterpret_cast<uint4*>(dqkv + row * 3 * D + c) = w;
    src[0] = make_float4(0.f, 0.f, 0.f, 0.f);
    src[1] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// Delta pre-kernel, the fused kernel and the dQ conversion on one stream (see the entry points below for the contract).
static int attn_bwd_launch(const void* qkv, const void* out, const void* dout, const float* gate, const float* tab,
                           const uint8_t* key_pad, const float* lse, float* delta, float* dq_acc, void* dqkv, float* dgate,
                           float* dtab, int B, int T, int H, float scale, float drop_p, const uint32_t* drop_mask,
                           int head_dim, cudaStream_t st) {
  const int D = H * head_dim;
  const long long rows = static_cast<long long>(B) * T;
  CUtensorMap tm_qkv, tm_do, tm_dq, tm_qkv16, tm_do16, tm_dq16;
  const int box_rows = head_dim == 64 ? kAttnTile : BwdMap<80>::kQT;
  if (make_operand_tmaps(&tm_qkv, &tm_qkv16, qkv, T, B, 3 * D, head_dim, box_rows)) return -3;
  if (make_operand_tmaps(&tm_do, &tm_do16, dout, T, B, D, head_dim, box_rows)) return -3;
  // dQ reductions: [64 queries][32 columns] boxes (one 128-byte swizzle row), and at width 80 [64][16] unswizzled
  if (make_head_tmap(&tm_dq, dq_acc, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, T, B, D, head_dim, 32, 64, CU_TENSOR_MAP_SWIZZLE_128B))
    return -3;
  tm_dq16 = tm_dq;
  if (head_dim == 80 &&
      make_head_tmap(&tm_dq16, dq_acc, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, T, B, D, head_dim, 16, 64, CU_TENSOR_MAP_SWIZZLE_NONE))
    return -3;
  AttnParams p;
  memset(&p, 0, sizeof(p));
  p.T = T; p.H = H; p.B = B; p.D = D;
  p.n_tiles = ceil_div(T, kAttnTile);
  p.scale = scale;
  p.gate = gate; p.tab = tab; p.key_pad = key_pad;
  p.lse = const_cast<float*>(lse);
  p.dout = static_cast<const __nv_bfloat16*>(dout);
  p.delta = delta;
  p.dqkv = static_cast<__nv_bfloat16*>(dqkv);
  p.dgate = dgate;
  p.dtab = dtab;
  const bool drop = drop_p > 0.f;
  p.drop_mask = const_cast<uint32_t*>(drop_mask);
  p.drop_rp = 1.0f / (1.0f - drop_p);
  const int rc = attn_dispatch(head_dim, tab != nullptr, drop, [&](auto hd, auto bias, auto dp) {
    B200_CHECK_CUDA(launch_pdl(attn_delta2_kernel<hd>, dim3(static_cast<unsigned>(ceil_div_ll(rows * 32, 256))), dim3(256), 0,
                               st, static_cast<const __nv_bfloat16*>(out), static_cast<const __nv_bfloat16*>(dout), B, T, H,
                               delta, tab != nullptr ? dgate : nullptr));
    B200_CHECK_LAUNCH();
    const auto kern = attn_bwd_fused_kernel<hd, bias, dp>;
    constexpr int smem = BwdMap<hd>::kFSmem;
    B200_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    B200_CHECK_CUDA(launch_pdl(kern, dim3(p.n_tiles, H, B), dim3(kFThreads), smem, st, tm_qkv, tm_do, tm_dq, tm_qkv16, tm_do16,
                               tm_dq16, p));
    B200_CHECK_LAUNCH();
    return 0;
  });
  if (rc) return rc;
  const long long nvec = rows * (D / 8);
  const int blocks = static_cast<int>(std::min<long long>(ceil_div_ll(nvec, 256), static_cast<long long>(sm_count()) * 16));
  B200_CHECK_CUDA(launch_pdl(attn_dq_convert_kernel, dim3(blocks), dim3(256), 0, st, dq_acc, static_cast<__nv_bfloat16*>(dqkv), rows, D));
  B200_CHECK_LAUNCH();
  return 0;
}

}  // namespace b200

using namespace b200;

extern "C" {

// Backward of b200s_attn_fwd.  out/dout: bf16 [B,T,D]; lse from the forward; delta: fp32 [B,H,T] workspace;
// dqkv: bf16 [B,T,3D] (fully written for valid rows); dgate: fp32 [B,H,T] (written); dtab: fp32 [H,2T-1] (ACCUMULATED with
// atomics -- the caller zeroes it once per step, the table is shared by all layers).  gate/tab/dgate/dtab NULL = no bias.
// The fp32 dQ reduction buffer is allocated on the stream for the call (b200s_attn_bwd_fused takes it from the caller).
int b200s_attn_bwd(const void* qkv, const void* out, const void* dout, const float* gate, const float* tab,
                   const uint8_t* key_pad, const float* lse, float* delta, void* dqkv, float* dgate, float* dtab, int B,
                   int T, int H, float scale, int head_dim, b200s_stream stream) {
  B200_CHECK_ARG(qkv && out && dout && lse && delta && dqkv, "attn_bwd: null pointer");
  if (const int rc = attn_check_head("attn_bwd", head_dim, tab != nullptr)) return rc;
  B200_CHECK_ARG(T >= 1, "attn_bwd: T=%d out of range", T);
  B200_CHECK_ARG(!tab || (dgate && dtab), "attn_bwd: bias given but dgate/dtab missing");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t bytes = sizeof(float) * static_cast<size_t>(B) * T * H * head_dim;
  void* dq_acc = nullptr;
  B200_CHECK_CUDA(cudaMallocAsync(&dq_acc, bytes, st));
  B200_CHECK_CUDA(cudaMemsetAsync(dq_acc, 0, bytes, st));
  const int rc = attn_bwd_launch(qkv, out, dout, gate, tab, key_pad, lse, delta, static_cast<float*>(dq_acc), dqkv, dgate, dtab, B,
                                 T, H, scale, 0.f, nullptr, head_dim, st);
  B200_CHECK_CUDA(cudaFreeAsync(dq_acc, st));
  return rc;
}

// Fused backward of b200s_attn_fwd.  Same contract as b200s_attn_bwd plus dq_acc: fp32 [B,T,D] workspace that must be ZERO
// on entry and is zero again on return (the q gradient is reduced there across key tiles before it is rounded to bf16).
int b200s_attn_bwd_fused_dropout(const void* qkv, const void* out, const void* dout, const float* gate, const float* tab,
                                 const uint8_t* key_pad, const float* lse, float* delta, float* dq_acc, void* dqkv,
                                 float* dgate, float* dtab, int B, int T, int H, float scale, float drop_p,
                                 const uint32_t* drop_mask, int head_dim, b200s_stream stream) {
  B200_CHECK_ARG(qkv && out && dout && lse && delta && dqkv && dq_acc, "attn_bwd_fused: null pointer");
  if (const int rc = attn_check_head("attn_bwd_fused", head_dim, tab != nullptr)) return rc;
  B200_CHECK_ARG(drop_p >= 0.f && drop_p < 1.f, "attn_bwd_fused: dropout p=%f out of range [0,1)", static_cast<double>(drop_p));
  B200_CHECK_ARG(drop_p == 0.f || drop_mask != nullptr, "attn_bwd_fused: dropout needs the mask written by b200s_attn_fwd_dropout");
  B200_CHECK_ARG(T >= 1, "attn_bwd_fused: T=%d out of range", T);
  B200_CHECK_ARG(!tab || (dgate && dtab), "attn_bwd_fused: bias given but dgate/dtab missing");
  return attn_bwd_launch(qkv, out, dout, gate, tab, key_pad, lse, delta, dq_acc, dqkv, dgate, dtab, B, T, H, scale, drop_p,
                         drop_mask, head_dim, static_cast<cudaStream_t>(stream));
}

int b200s_attn_bwd_fused(const void* qkv, const void* out, const void* dout, const float* gate, const float* tab,
                         const uint8_t* key_pad, const float* lse, float* delta, float* dq_acc, void* dqkv, float* dgate,
                         float* dtab, int B, int T, int H, float scale, int head_dim, b200s_stream stream) {
  return b200s_attn_bwd_fused_dropout(qkv, out, dout, gate, tab, key_pad, lse, delta, dq_acc, dqkv, dgate, dtab, B, T, H, scale,
                                      0.f, nullptr, head_dim, stream);
}

}  // extern "C"
