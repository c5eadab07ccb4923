// K-means over bf16 encoder features: the label stage of HuBERT-style pre-training (the recipe's learn_kmeans.py /
// dump_km_label.py), without a [N, K] distance matrix and without floating-point atomics.
//
//   assign    labels[n] = argmin_k (|c_k|^2 - 2 x_n . c_k), ties to the lowest k; score[n] = that minimum
//             A wgmma GEMM X . C^T with the arg-min fused into the accumulator fragments.  One persistent CTA walks 128-row
//             bands; for each band it walks every 256-wide centroid tile (K <= 1024: at most 4), keeping each row's running best
//             in registers.  Warp roles are gemm_ws_kernel's: a TMA producer warpgroup, two consumer warpgroups (m64n256k16).
//   update    counts[k], sums[k, :] = sum of the rows labelled k, inertia = sum over labelled rows of |x|^2 + score (fp64)
//             A stable counting sort of row ids by label (per-warp chunk histograms, a scan, a per-warp scatter with
//             __match_any_sync ranks), then fixed 2048-row pieces of each label's segment summed in a fixed order, then the
//             pieces of each label combined in a fixed order.  A label holding half of all rows is thousands of pieces that run in
//             parallel.  Integer atomics only: two calls give bit-identical results.
//   centers   centre = sum / count (an empty cluster keeps its previous centre, scipy.cluster.vq.kmeans2's rule), the bf16
//             copy the assignment multiplies, and |c|^2 of that bf16 copy, so the score is consistent with the operands.
//   k-means++ (Arthur & Vassilvitskii 2007): first centre uniform, each next one drawn with probability D(x)^2 (fp64 prefix sums,
//             the counter-based hash of dropout.cuh keyed by the seed), D(x) <- min(D(x), |x - c_new|^2) in fp32.
#include <math.h>

#include <algorithm>
#include <mutex>

#include "../../include/unispeech_b200.h"
#include "common.h"
#include "dropout.cuh"
#include "ptx.cuh"

namespace b200 {

int make_rows_tmap(CUtensorMap* out, const void* ptr, long long cols, long long rows, long long batches, long long row_stride,
                   long long batch_stride, int box_rows);

namespace {

constexpr int kMaxK = B200S_KMEANS_MAX_K;
constexpr int kTileN = 256;      // centroid tile of the assignment (centres are padded to a multiple of it)
constexpr int kChunk = 4096;     // rows per warp in the counting sort
constexpr int kPiece = 2048;     // sorted rows per partial sum
constexpr int kColsPerCta = 256; // columns per CTA of the partial sums (32 lanes x 8 bf16)

struct AssignCfg {
  static constexpr int kStages = 4;
  static constexpr int kABytes = 128 * 128;  // 128 rows x 64 bf16
  static constexpr int kBBytes = 256 * 128;  // 256 centres x 64 bf16
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kSmemBytes = kStages * kStageBytes + kMaxK * 4 + 1024;
  static constexpr int kThreads = 384;
  static_assert(kSmemBytes + 1024 <= 232448, "one CTA per SM");
};

struct AssignParams {
  int rows;             // rows per batch
  int bands_per_batch;  // ceil(rows / 128)
  int bands;            // bands over all batches
  int k;                // clusters
  int n_tiles;          // centroid tiles (Kp / 256)
  int k_blocks;         // D / 64
  const int* valid;     // [batches] valid rows, or null
  const float* cnorm;   // [Kp]
  int* labels;          // [batches, rows]
  float* score;         // [batches, rows] or null
  const int* prev;      // [batches, rows] or null
  int* changed;         // int32 counter or null
};

__device__ __forceinline__ bool band_live(const AssignParams& p, int band, int& mb, int& m0, int& vrows) {
  mb = band / p.bands_per_batch;
  m0 = (band - mb * p.bands_per_batch) * 128;
  vrows = p.valid == nullptr ? p.rows : min(max(__ldg(p.valid + mb), 0), p.rows);
  return m0 < vrows;
}

__global__ void __launch_bounds__(384, 1) kmeans_assign_kernel(const __grid_constant__ CUtensorMap tmX,
                                                               const __grid_constant__ CUtensorMap tmC,
                                                               const __grid_constant__ AssignParams p) {
  pdl_launch_dependents();
  using Cfg = AssignCfg;
  constexpr int kStages = Cfg::kStages;
  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  float* cn_s = reinterpret_cast<float*>(smem + kStages * Cfg::kStageBytes);
  __shared__ uint64_t full_bar[kStages];
  __shared__ uint64_t empty_bar[kStages];

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmX);
    tma_prefetch_desc(&tmC);
#pragma unroll
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);  // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  pdl_wait();
  // |c|^2 of every centroid column; padded columns are +inf and never win (inf - 2 * 0 = inf is not < anything)
  for (int i = threadIdx.x; i < p.n_tiles * kTileN; i += blockDim.x) cn_s[i] = i < p.k ? p.cnorm[i] : INFINITY;
  __syncthreads();

  if (wg == 0) {
    // ------------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int it = 0;
      for (int band = blockIdx.x; band < p.bands; band += gridDim.x) {
        int mb, m0, vrows;
        if (!band_live(p, band, mb, m0, vrows)) continue;
        for (int nt = 0; nt < p.n_tiles; ++nt) {
          for (int kb = 0; kb < p.k_blocks; ++kb, ++it) {
            const int s = it % kStages;
            mbar_wait(&empty_bar[s], ((it / kStages) & 1) ^ 1);
            uint8_t* sa = smem + s * Cfg::kStageBytes;
            mbar_expect_tx(&full_bar[s], Cfg::kStageBytes);
            tma_load_4d(sa, &tmX, &full_bar[s], kb * 64, m0, mb, 0);
            tma_load_4d(sa + Cfg::kABytes, &tmC, &full_bar[s], kb * 64, nt * kTileN, 0, 0);
          }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------- consumers: warpgroup c owns rows 64 c .. 64 c + 63 of a band
  setmaxnreg_inc<232>();
  const int c = wg - 1;
  const int t = threadIdx.x & 127, w = t >> 5, q = lane & 3;
  float acc[128];  // written by each tile's first MMA (scale_d = 0)
  int it = 0;
  for (int band = blockIdx.x; band < p.bands; band += gridDim.x) {
    int mb, m0, vrows;
    const long long lab0 = static_cast<long long>(band / p.bands_per_batch) * p.rows;
    if (!band_live(p, band, mb, m0, vrows)) {
      if (t < 64 && m0 + 64 * c + t < p.rows) p.labels[lab0 + m0 + 64 * c + t] = -1;
      continue;
    }
    // this thread's rows (accumulator fragment): 16 w + lane / 4 and 8 below it
    float best[2] = {INFINITY, INFINITY};
    int bidx[2] = {0, 0};
    for (int nt = 0; nt < p.n_tiles; ++nt) {
      for (int kb = 0; kb < p.k_blocks; ++kb, ++it) {
        const int s = it % kStages;
        mbar_wait(&full_bar[s], (it / kStages) & 1);
        const uint32_t sa = smem_u32(smem + s * Cfg::kStageBytes) + c * 8192;  // rows 64 c .. of the band: 64 rows x 128 B
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
      // running arg-min: d[4 j + 2 h + e] is row 8 h (+ base), column 8 j + 2 q + e -- visited in increasing column order, so
      // the strict comparison keeps the lowest index among equal scores
      const float* cn = cn_s + nt * kTileN + 2 * q;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const float2 cc = *reinterpret_cast<const float2*>(cn + 8 * j);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float s0 = fmaf(-2.f, acc[4 * j + 2 * h], cc.x);
          const float s1 = fmaf(-2.f, acc[4 * j + 2 * h + 1], cc.y);
          if (s0 < best[h]) { best[h] = s0; bidx[h] = nt * kTileN + 8 * j + 2 * q; }
          if (s1 < best[h]) { best[h] = s1; bidx[h] = nt * kTileN + 8 * j + 2 * q + 1; }
        }
      }
    }
    // the four lanes of a quad hold interleaved columns of the same two rows
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float ob = __shfl_xor_sync(0xffffffffu, best[h], o);
        const int oi = __shfl_xor_sync(0xffffffffu, bidx[h], o);
        if (ob < best[h] || (ob == best[h] && oi < bidx[h])) { best[h] = ob; bidx[h] = oi; }
      }
    }
    int changed = 0;
    if (q == 0) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = m0 + 64 * c + 16 * w + (lane >> 2) + 8 * h;
        if (r >= p.rows) continue;
        const long long i = lab0 + r;
        if (r < vrows) {
          p.labels[i] = bidx[h];
          if (p.score != nullptr) p.score[i] = best[h];
          if (p.prev != nullptr) changed += p.prev[i] != bidx[h];
        } else {
          p.labels[i] = -1;
        }
      }
    }
    if (p.changed != nullptr) {
      changed = __reduce_add_sync(0xffffffffu, changed);
      if (lane == 0 && changed > 0) atomicAdd(p.changed, changed);
    }
  }
}

// ---------------------------------------------------------------------------------------------------- block scans
// Exclusive scan over the block (blockDim.x a multiple of 32, <= 1024); *total = the sum over the block.  tmp: 32 slots.
template <typename T>
__device__ __forceinline__ T block_excl_scan(T v, T* tmp, T* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  T incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T n = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += n;
  }
  __syncthreads();  // tmp may still be read by a previous call
  if (lane == 31) tmp[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    T s = lane < nw ? tmp[lane] : T(0);
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const T n = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += n;
    }
    if (lane < nw) tmp[lane] = s;
  }
  __syncthreads();
  *total = tmp[nw - 1];
  return (warp > 0 ? tmp[warp - 1] : T(0)) + incl - v;
}

// ------------------------------------------------------------------------------------------ update: counting sort
// hist[k * nchunks + chunk] = rows of the chunk (kChunk rows, one warp) labelled k.  Labels outside [0, K) are skipped.
__global__ void __launch_bounds__(256) kmeans_hist_kernel(const int* __restrict__ labels, int n, int K, int nchunks,
                                                          int* __restrict__ hist) {
  pdl_grid_sync();
  extern __shared__ int cnt_s[];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int chunk = blockIdx.x * 8 + w;
  if (chunk >= nchunks) return;
  int* cnt = cnt_s + w * K;
  for (int k = lane; k < K; k += 32) cnt[k] = 0;
  __syncwarp();
  const int end = min(n, (chunk + 1) * kChunk);
  for (int r = chunk * kChunk + lane; r < end; r += 32) {
    const int lab = labels[r];
    if (lab >= 0 && lab < K) atomicAdd(cnt + lab, 1);
  }
  __syncwarp();
  for (int k = lane; k < K; k += 32) hist[static_cast<long long>(k) * nchunks + chunk] = cnt[k];
}

// One CTA per label: exclusive scan of its chunk counts in place; counts[k] = the label's rows.
__global__ void __launch_bounds__(1024) kmeans_scan_chunks_kernel(int* __restrict__ hist, int nchunks, int* __restrict__ counts) {
  pdl_grid_sync();
  __shared__ int tmp[32];
  int* h = hist + static_cast<long long>(blockIdx.x) * nchunks;
  int carry = 0;
  for (int i0 = 0; i0 < nchunks; i0 += blockDim.x) {
    const int i = i0 + threadIdx.x;
    const int v = i < nchunks ? h[i] : 0;
    int tot;
    const int ex = block_excl_scan(v, tmp, &tot);
    if (i < nchunks) h[i] = carry + ex;
    carry += tot;
  }
  if (threadIdx.x == 0) counts[blockIdx.x] = carry;
}

// One CTA: off[k] = first sorted position of label k, pstart[k] = its first piece (off[K], pstart[K] = totals).
__global__ void __launch_bounds__(1024) kmeans_offsets_kernel(const int* __restrict__ counts, int K, int* __restrict__ off,
                                                              int* __restrict__ pstart) {
  pdl_grid_sync();
  __shared__ int tmp[32];
  const int k = threadIdx.x;
  const int cnt = k < K ? counts[k] : 0;
  int tot, ptot;
  const int o = block_excl_scan(cnt, tmp, &tot);
  const int po = block_excl_scan((cnt + kPiece - 1) / kPiece, tmp, &ptot);
  if (k < K) {
    off[k] = o;
    pstart[k] = po;
  }
  if (k == 0) {
    off[K] = tot;
    pstart[K] = ptot;
  }
}

// Each warp walks its chunk again, 32 rows at a time in row order: the rank of a row among the lanes holding the same label is
// the number of lower lanes in its __match_any_sync group, so perm lists every label's rows in increasing row order.
__global__ void __launch_bounds__(256) kmeans_scatter_kernel(const int* __restrict__ labels, int n, int K, int nchunks,
                                                             const int* __restrict__ hist, const int* __restrict__ off,
                                                             int* __restrict__ perm) {
  pdl_grid_sync();
  extern __shared__ int base_s[];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int chunk = blockIdx.x * 8 + w;
  if (chunk >= nchunks) return;
  int* base = base_s + w * K;
  for (int k = lane; k < K; k += 32) base[k] = off[k] + hist[static_cast<long long>(k) * nchunks + chunk];
  __syncwarp();
  const int end = min(n, (chunk + 1) * kChunk);
  const unsigned lt = (1u << lane) - 1u;
  for (int r0 = chunk * kChunk; r0 < end; r0 += 32) {
    const int r = r0 + lane;
    int lab = r < end ? labels[r] : -1;
    if (lab >= K) lab = -1;
    const unsigned m = __match_any_sync(0xffffffffu, lab);
    if (lab >= 0) perm[base[lab] + __popc(m & lt)] = r;
    __syncwarp();
    if (lab >= 0 && (m & lt) == 0) base[lab] += __popc(m);
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------ update: fixed-order sums
// grid (max pieces, ceil(D / 256)), 8 warps: piece j of label k covers sorted positions off[k] + kPiece (j - pstart[k]) ..;
// lane l of every warp owns columns 256 y + 8 l .. + 7, warp w the rows w, w + 8, ... of the piece, in order.  The 8 warps are
// then added in order.  ipart[j * ny + y] = sum |x|^2 over the piece's rows and this CTA's columns (+ the scores when y = 0).
__global__ void __launch_bounds__(256) kmeans_piece_kernel(const __nv_bfloat16* __restrict__ x, long long x_rs, int D,
                                                           const int* __restrict__ perm, const float* __restrict__ score,
                                                           const int* __restrict__ off, const int* __restrict__ pstart, int K,
                                                           float* __restrict__ part, double* __restrict__ ipart) {
  pdl_grid_sync();
  __shared__ float red[8][kColsPerCta];
  __shared__ double wsum[8];
  const int j = blockIdx.x, y = blockIdx.y, ny = gridDim.y;
  if (j >= pstart[K]) return;  // uniform per CTA
  int lo = 0, hi = K - 1;      // the largest k with pstart[k] <= j (an empty label shares its pstart with the next label)
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (pstart[mid] <= j) lo = mid; else hi = mid - 1;
  }
  const int k = lo;
  const int begin = off[k] + (j - pstart[k]) * kPiece, end = min(begin + kPiece, off[k + 1]);
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int col = y * kColsPerCta + 8 * lane;
  const bool active = col < D;
  float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float ss = 0.f;
  double sc = 0.0;
  constexpr int kU = 4;  // rows in flight per warp
  for (int i0 = begin + w; i0 < end; i0 += 8 * kU) {
    int rid[kU];
    uint4 v[kU];
#pragma unroll
    for (int u = 0; u < kU; ++u) rid[u] = i0 + 8 * u < end ? perm[i0 + 8 * u] : -1;
#pragma unroll
    for (int u = 0; u < kU; ++u)
      v[u] = (rid[u] >= 0 && active) ? __ldg(reinterpret_cast<const uint4*>(x + rid[u] * x_rs + col)) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const uint32_t wu[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = unpack_bf16x2(wu[e]);
        a[2 * e] += f.x;
        a[2 * e + 1] += f.y;
        ss = fmaf(f.x, f.x, ss);
        ss = fmaf(f.y, f.y, ss);
      }
      if (y == 0 && lane == 0 && rid[u] >= 0) sc += static_cast<double>(score[rid[u]]);
    }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) red[w][8 * lane + e] = a[e];
  const float wss = warp_sum(ss);
  if (lane == 0) wsum[w] = static_cast<double>(wss) + sc;
  __syncthreads();
  const int tcol = y * kColsPerCta + threadIdx.x;
  if (tcol < D) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += red[i][threadIdx.x];
    part[static_cast<long long>(j) * D + tcol] = s;
  }
  if (threadIdx.x == 0) {
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += wsum[i];
    ipart[static_cast<long long>(j) * ny + y] = s;
  }
}

// grid (K, ceil(D / 256)), 8 warps: warp w adds pieces pstart[k] + w, + 8, ... (fp64), then the 8 warps in order.  CTA (0, 0)
// also adds every ipart entry in a fixed order into *inertia.
__global__ void __launch_bounds__(256) kmeans_combine_kernel(const float* __restrict__ part, const double* __restrict__ ipart,
                                                             const int* __restrict__ pstart, int K, int D, float* __restrict__ sums,
                                                             double* __restrict__ inertia) {
  pdl_grid_sync();
  __shared__ double red[8][kColsPerCta];
  __shared__ double tmp[32];
  const int k = blockIdx.x, y = blockIdx.y;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int col = y * kColsPerCta + 8 * lane;
  double a[8] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  if (col < D) {
    for (int j = pstart[k] + w; j < pstart[k + 1]; j += 8) {
      const float4* src = reinterpret_cast<const float4*>(part + static_cast<long long>(j) * D + col);
      const float4 v0 = src[0], v1 = src[1];
      a[0] += v0.x; a[1] += v0.y; a[2] += v0.z; a[3] += v0.w;
      a[4] += v1.x; a[5] += v1.y; a[6] += v1.z; a[7] += v1.w;
    }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) red[w][8 * lane + e] = a[e];
  __syncthreads();
  const int tcol = y * kColsPerCta + threadIdx.x;
  if (tcol < D) {
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += red[i][threadIdx.x];
    sums[static_cast<long long>(k) * D + tcol] = static_cast<float>(s);
  }
  if (k == 0 && y == 0) {
    const long long n = static_cast<long long>(pstart[K]) * gridDim.y;
    double s = 0.0;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) s += ipart[i];
    double tot;
    const double ex = block_excl_scan(s, tmp, &tot);  // (a fixed-order block sum)
    (void)ex;
    if (threadIdx.x == 0) *inertia = tot;
  }
}

// ------------------------------------------------------------------------------------------ centres
// One CTA per padded centre row: centers[k] = sums[k] / counts[k] when counts[k] > 0 (sums / counts null: unchanged); the bf16
// copy; cnorm[k] = |bf16 copy|^2 (fp32, fixed-order reduction).  Rows k >= K of the bf16 copy are zeros.
__global__ void __launch_bounds__(256) kmeans_centers_kernel(const float* __restrict__ sums, const int* __restrict__ counts, int K,
                                                             int D, float* __restrict__ centers, __nv_bfloat16* __restrict__ cbf,
                                                             float* __restrict__ cnorm) {
  pdl_grid_sync();
  __shared__ float tmp[32];
  const int k = blockIdx.x;
  __nv_bfloat16* dst = cbf + static_cast<long long>(k) * D;
  if (k >= K) {
    for (int d = threadIdx.x; d < D; d += blockDim.x) dst[d] = __float2bfloat16_rn(0.f);
    if (threadIdx.x == 0) cnorm[k] = 0.f;
    return;
  }
  const int cnt = counts != nullptr ? counts[k] : 0;
  const float inv = cnt > 0 ? 1.0f / static_cast<float>(cnt) : 0.f;
  float* cf = centers + static_cast<long long>(k) * D;
  float ss = 0.f;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float v = cf[d];
    if (sums != nullptr && cnt > 0) {
      v = sums[static_cast<long long>(k) * D + d] * inv;
      cf[d] = v;
    }
    const __nv_bfloat16 b = __float2bfloat16_rn(v);
    dst[d] = b;
    const float f = __bfloat162float(b);
    ss = fmaf(f, f, ss);
  }
  float tot;
  block_excl_scan(ss, tmp, &tot);
  if (threadIdx.x == 0) cnorm[k] = tot;
}

// ------------------------------------------------------------------------------------------ k-means++
__device__ __forceinline__ double u01_53(uint32_t k0, uint32_t k1, uint32_t ctr) {
  const uint32_t a = drop_bits(k0, k1, 2u * ctr) >> 5, b = drop_bits(k0, k1, 2u * ctr + 1u) >> 6;
  return (static_cast<double>(a) * 67108864.0 + static_cast<double>(b)) * (1.0 / 9007199254740992.0);  // [0, 1)
}

// One CTA of 1024 threads.  j < K: draws centre j (j = 0 uniform, else with probability d2[i] / sum d2 through fp64 prefix sums
// over fixed per-thread ranges) and writes its fp32 copy to centers[j].  *total = sum d2 (fp64) of the current state.
__global__ void __launch_bounds__(1024) kmeanspp_draw_kernel(const float* __restrict__ d2, int n, int j, int K, uint32_t k0,
                                                             uint32_t k1, const __nv_bfloat16* __restrict__ x, long long x_rs, int D,
                                                             float* __restrict__ centers, double* __restrict__ total) {
  pdl_grid_sync();
  __shared__ double tmp[32];
  __shared__ int sel;
  const int t = threadIdx.x;
  const int per = (n + blockDim.x - 1) / blockDim.x;
  const int i0 = min(n, t * per), i1 = min(n, i0 + per);
  if (t == 0) sel = -1;
  double tot = 0.0;
  if (j > 0) {
    double s = 0.0;
    for (int i = i0; i < i1; ++i) s += d2[i];
    const double base = block_excl_scan(s, tmp, &tot);
    if (total != nullptr && t == 0) *total = tot;
    if (j >= K) return;
    if (tot > 0.0) {
      const double u = u01_53(k0, k1, static_cast<uint32_t>(j)) * tot;
      // the range holding u; the last non-empty range also takes u >= its end (rounding of the prefix sums)
      if (s > 0.0 && u >= base && (u < base + s || base + s >= tot)) {
        double acc = base;
        int pick = -1;
        for (int i = i0; i < i1; ++i) {
          if (d2[i] > 0.f) pick = i;
          acc += d2[i];
          if (u < acc && d2[i] > 0.f) break;
        }
        sel = pick;
      }
    }
  }
  __syncthreads();
  if (sel < 0 && t == 0) sel = min(n - 1, static_cast<int>(u01_53(k0, k1, static_cast<uint32_t>(j)) * n));  // j = 0, or sum d2 = 0
  __syncthreads();
  const __nv_bfloat16* src = x + static_cast<long long>(sel) * x_rs;
  for (int d = t; d < D; d += blockDim.x) centers[static_cast<long long>(j) * D + d] = __bfloat162float(src[d]);
}

// One warp per row: d2[i] = min(d2[i], |x_i - c|^2) (first: d2[i] = |x_i - c|^2), fp32 from the bf16 row and the centre.
__global__ void __launch_bounds__(256) kmeanspp_dist_kernel(const __nv_bfloat16* __restrict__ x, long long x_rs, int n, int D,
                                                            const float* __restrict__ c, float* __restrict__ d2, int first) {
  pdl_grid_sync();
  const int lane = threadIdx.x & 31;
  const long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (i >= n) return;
  const __nv_bfloat16* row = x + i * x_rs;
  float s = 0.f;
  for (int d = 8 * lane; d < D; d += 256) {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(row + d));
    const float4 c0 = __ldg(reinterpret_cast<const float4*>(c + d)), c1 = __ldg(reinterpret_cast<const float4*>(c + d + 4));
    const float cv[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
    const uint32_t wu[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = unpack_bf16x2(wu[e]);
      const float a = f.x - cv[2 * e], b = f.y - cv[2 * e + 1];
      s = fmaf(a, a, s);
      s = fmaf(b, b, s);
    }
  }
  s = warp_sum(s);
  if (lane == 0) d2[i] = first ? s : fminf(d2[i], s);
}

struct UpdateWs {
  int* hist;
  int* off;
  int* pstart;
  int* perm;
  float* part;
  double* ipart;
  long long bytes;
};

// workspace of b200s_kmeans_update: chunk histograms, offsets, the sorted row ids and the partial sums (base 0: sizes only)
UpdateWs update_ws(uintptr_t base, long long n, int K, int D) {
  const long long nchunks = (n + kChunk - 1) / kChunk, pieces = (n + kPiece - 1) / kPiece + K, ny = (D + kColsPerCta - 1) / kColsPerCta;
  auto al = [](long long b) { return (b + 255) / 256 * 256; };
  long long o = 0;
  auto take = [&](long long bytes) {
    const uintptr_t p = base + static_cast<uintptr_t>(o);
    o += al(bytes);
    return p;
  };
  UpdateWs w;
  w.hist = reinterpret_cast<int*>(take(4LL * K * nchunks));
  w.off = reinterpret_cast<int*>(take(4LL * (K + 1)));
  w.pstart = reinterpret_cast<int*>(take(4LL * (K + 1)));
  w.perm = reinterpret_cast<int*>(take(4LL * n));
  w.part = reinterpret_cast<float*>(take(4LL * pieces * D));
  w.ipart = reinterpret_cast<double*>(take(8LL * pieces * ny));
  w.bytes = o;
  return w;
}

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

int b200s_kmeans_assign(const void* x, long long x_bs, long long x_rs, int rows, int batches, int D, const int* valid,
                        const void* centers, const float* cnorm, int K, int* labels, float* score, const int* prev_labels,
                        int* changed, b200s_stream stream) {
  B200_CHECK_ARG(x && centers && cnorm && labels, "kmeans_assign: null pointer");
  B200_CHECK_ARG(rows > 0 && batches > 0, "kmeans_assign: bad sizes (rows=%d, batches=%d)", rows, batches);
  B200_CHECK_ARG(K >= 1 && K <= kMaxK, "kmeans_assign: K=%d outside [1, %d]", K, kMaxK);
  B200_CHECK_ARG(D > 0 && D % 64 == 0, "kmeans_assign: D=%d must be a positive multiple of 64 (zero-pad the features)", D);
  B200_CHECK_ARG((prev_labels == nullptr) == (changed == nullptr), "kmeans_assign: prev_labels and changed go together");
  CUtensorMap tx, tc;
  const int n_tiles = ceil_div(K, kTileN);
  if (const int rc = make_rows_tmap(&tx, x, D, rows, batches, x_rs, x_bs, 128)) return rc;
  if (const int rc = make_rows_tmap(&tc, centers, D, static_cast<long long>(n_tiles) * kTileN, 1, D, 0, kTileN)) return rc;
  AssignParams p;
  p.rows = rows;
  p.bands_per_batch = ceil_div(rows, 128);
  B200_CHECK_ARG(static_cast<long long>(p.bands_per_batch) * batches < (1LL << 31), "kmeans_assign: too many rows");
  p.bands = p.bands_per_batch * batches;
  p.k = K;
  p.n_tiles = n_tiles;
  p.k_blocks = D / 64;
  p.valid = valid;
  p.cnorm = cnorm;
  p.labels = labels;
  p.score = score;
  p.prev = prev_labels;
  p.changed = changed;
  static std::once_flag once;
  static cudaError_t attr_err = cudaSuccess;
  std::call_once(once, [] {
    attr_err = cudaFuncSetAttribute(kmeans_assign_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AssignCfg::kSmemBytes);
  });
  B200_CHECK_CUDA(attr_err);
  B200_CHECK_CUDA(launch_pdl(kmeans_assign_kernel, dim3(std::min(p.bands, sm_count())), dim3(AssignCfg::kThreads),
                             AssignCfg::kSmemBytes, static_cast<cudaStream_t>(stream), tx, tc, p));
  B200_CHECK_LAUNCH();
  return 0;
}

long long b200s_kmeans_update_workspace(long long n, int K, int D) {
  if (n <= 0 || K < 1 || K > kMaxK || D <= 0) return -1;
  return update_ws(0, n, K, D).bytes;
}

int b200s_kmeans_update(const void* x, long long x_rs, int n, int D, const int* labels, const float* score, int K, void* workspace,
                        long long workspace_bytes, int* counts, float* sums, double* inertia, b200s_stream stream) {
  B200_CHECK_ARG(x && labels && score && workspace && counts && sums && inertia, "kmeans_update: null pointer");
  B200_CHECK_ARG(n > 0, "kmeans_update: n=%d must be positive", n);
  B200_CHECK_ARG(K >= 1 && K <= kMaxK, "kmeans_update: K=%d outside [1, %d]", K, kMaxK);
  B200_CHECK_ARG(D > 0 && D % 64 == 0, "kmeans_update: D=%d must be a positive multiple of 64", D);
  B200_CHECK_ARG(x_rs >= D && x_rs % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0,
                 "kmeans_update: rows must be 16-byte aligned (row stride %lld)", x_rs);
  const UpdateWs w = update_ws(reinterpret_cast<uintptr_t>(workspace), n, K, D);
  B200_CHECK_ARG(workspace_bytes >= w.bytes, "kmeans_update: workspace of %lld bytes, need %lld", workspace_bytes, w.bytes);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int nchunks = ceil_div(n, kChunk), ny = ceil_div(D, kColsPerCta);
  const int max_pieces = ceil_div(n, kPiece) + K;
  const __nv_bfloat16* xb = static_cast<const __nv_bfloat16*>(x);
  B200_CHECK_CUDA(launch_pdl(kmeans_hist_kernel, dim3(ceil_div(nchunks, 8)), dim3(256), 8 * K * sizeof(int), st, labels, n, K,
                             nchunks, w.hist));
  B200_CHECK_LAUNCH();
  B200_CHECK_CUDA(launch_pdl(kmeans_scan_chunks_kernel, dim3(K), dim3(1024), 0, st, w.hist, nchunks, counts));
  B200_CHECK_LAUNCH();
  B200_CHECK_CUDA(launch_pdl(kmeans_offsets_kernel, dim3(1), dim3(1024), 0, st, static_cast<const int*>(counts), K, w.off,
                             w.pstart));
  B200_CHECK_LAUNCH();
  B200_CHECK_CUDA(launch_pdl(kmeans_scatter_kernel, dim3(ceil_div(nchunks, 8)), dim3(256), 8 * K * sizeof(int), st, labels, n, K,
                             nchunks, static_cast<const int*>(w.hist), static_cast<const int*>(w.off), w.perm));
  B200_CHECK_LAUNCH();
  B200_CHECK_CUDA(launch_pdl(kmeans_piece_kernel, dim3(max_pieces, ny), dim3(256), 0, st, xb, x_rs, D,
                             static_cast<const int*>(w.perm), score, static_cast<const int*>(w.off),
                             static_cast<const int*>(w.pstart), K, w.part, w.ipart));
  B200_CHECK_LAUNCH();
  B200_CHECK_CUDA(launch_pdl(kmeans_combine_kernel, dim3(K, ny), dim3(256), 0, st, static_cast<const float*>(w.part),
                             static_cast<const double*>(w.ipart), static_cast<const int*>(w.pstart), K, D, sums, inertia));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_kmeans_centers(const float* sums, const int* counts, int K, int D, float* centers, void* centers_bf16, float* cnorm,
                         b200s_stream stream) {
  B200_CHECK_ARG(centers && centers_bf16 && cnorm, "kmeans_centers: null pointer");
  B200_CHECK_ARG((sums == nullptr) == (counts == nullptr), "kmeans_centers: sums and counts go together");
  B200_CHECK_ARG(K >= 1 && K <= kMaxK, "kmeans_centers: K=%d outside [1, %d]", K, kMaxK);
  B200_CHECK_ARG(D > 0 && D % 64 == 0, "kmeans_centers: D=%d must be a positive multiple of 64", D);
  B200_CHECK_CUDA(launch_pdl(kmeans_centers_kernel, dim3(ceil_div(K, kTileN) * kTileN), dim3(256), 0,
                             static_cast<cudaStream_t>(stream), sums, counts, K, D, centers,
                             static_cast<__nv_bfloat16*>(centers_bf16), cnorm));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_kmeanspp_init(const void* x, long long x_rs, int n, int D, int K, uint32_t seed0, uint32_t seed1, float* d2,
                        float* centers, double* inertia, b200s_stream stream) {
  B200_CHECK_ARG(x && d2 && centers, "kmeanspp_init: null pointer");
  B200_CHECK_ARG(n > 0, "kmeanspp_init: n=%d must be positive", n);
  B200_CHECK_ARG(K >= 1 && K <= kMaxK, "kmeanspp_init: K=%d outside [1, %d]", K, kMaxK);
  B200_CHECK_ARG(D > 0 && D % 64 == 0, "kmeanspp_init: D=%d must be a positive multiple of 64", D);
  B200_CHECK_ARG(x_rs >= D && x_rs % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0,
                 "kmeanspp_init: rows must be 16-byte aligned (row stride %lld)", x_rs);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const __nv_bfloat16* xb = static_cast<const __nv_bfloat16*>(x);
  const uint32_t k0 = fmix32(seed0 ^ 0x6B6D6561u), k1 = fmix32(seed1 + 0x2B2B2B2Bu);
  const unsigned dist_blocks = static_cast<unsigned>(ceil_div_ll(static_cast<long long>(n) * 32, 256));
  for (int j = 0; j <= K; ++j) {
    if (j < K || inertia != nullptr) {
      B200_CHECK_CUDA(launch_pdl(kmeanspp_draw_kernel, dim3(1), dim3(1024), 0, st, static_cast<const float*>(d2), n, j, K, k0, k1,
                                 xb, x_rs, D, centers, j == K ? inertia : nullptr));
      B200_CHECK_LAUNCH();
    }
    if (j < K) {
      B200_CHECK_CUDA(launch_pdl(kmeanspp_dist_kernel, dim3(dist_blocks), dim3(256), 0, st, xb, x_rs, n, D,
                                 static_cast<const float*>(centers + static_cast<long long>(j) * D), d2, j == 0 ? 1 : 0));
      B200_CHECK_LAUNCH();
    }
  }
  return 0;
}

}  // extern "C"
