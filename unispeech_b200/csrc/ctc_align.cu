// CTC forced alignment: the most probable CTC path of a known transcript through the bf16 logits of the fine-tuning wrappers'
// `proj` head (the Viterbi form of the trellis of ctc.cu, max in place of log-sum-exp, plus backpointers), with the tie rule of
// torchaudio.functional.forced_align so that paths and frame scores agree with it bit for bit.
//
//   viterbi kernel    one CTA per utterance.  Thread i owns the P consecutive positions [P i, P i + P) of the extended label
//                     sequence l' = (blank, l_1, blank, ..., l_S, blank) and keeps their alpha in registers; the s-1 / s-2
//                     neighbours of its first two positions come from lane i-1 by shuffle, or, for lane 0, from the previous
//                     warp's last two values in shared memory (double-buffered by frame parity): ONE barrier per frame.  The
//                     emissions (one blank and P/2 label logits per frame) and lse are loaded into registers kPre frames ahead of
//                     use.  P is chosen from Smax at launch (2, 4, 8, 16 or 32, at most 512 threads).  Every frame writes the
//                     2-bit choices of all positions as whole 32-bit words (16 positions per word; lanes sharing a word OR their
//                     bits together with shuffles first).  At the end it writes score[b] and, as a hand-off to the backtrack,
//                     the end position into labels[b, T_b - 1] (-1 when the utterance is infeasible).
//   backtrack kernel  one warp per utterance.  Per chunk of 32 frames each lane fetches the five backpointer words that can
//                     hold its frame's position (the path moves down at most 2 positions a frame) into shared memory, lane 0
//                     walks the 32 frames through shared memory only, and the lanes write labels and frame scores.  One
//                     dependent global latency per 32 frames.
//
// Tie rule (torchaudio's, checked against it in tests/test_ctc_align_cpu.py): skip if skip > advance && skip > stay, else
// advance if advance > stay && advance > skip, else stay -- strict comparisons, so ties go to stay, and advance == skip > stay
// takes stay.  The end is position L-1 if alpha(L-1) > alpha(L-2), else L-2.
#include <limits.h>
#include <math.h>

#include "../../include/unispeech_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace b200 {

namespace {

constexpr int kMaxV = 1024;
constexpr int kMaxThreads = 512;
constexpr int kMaxWarps = kMaxThreads / 32;
constexpr int kChunk = 32;   // backtrack frames per fetch
constexpr int kWin = 5;      // backpointer words fetched per frame: positions [pos - 62, pos] of a 32-frame chunk

__device__ __forceinline__ float bf(const __nv_bfloat16* p) { return __bfloat162float(*p); }

// The blank's logit and the 2 HP label logits of one frame (raw bf16 bits, two to a register; the odd half of the last register
// is a spare read of a valid class when P = 2).
template <int HP>
__device__ __forceinline__ void load_row(const __nv_bfloat16* row, int blank, const uint32_t (&lab)[HP], float& qb,
                                         uint32_t (&ql)[HP]) {
  const unsigned short* r = reinterpret_cast<const unsigned short*>(row);
  qb = bf(row + blank);
#pragma unroll
  for (int h = 0; h < HP; ++h) ql[h] = static_cast<uint32_t>(r[lab[h] & 0xffffu]) | (static_cast<uint32_t>(r[lab[h] >> 16]) << 16);
}

__device__ __forceinline__ int words_per_frame(int Smax) { return (2 * Smax + 1 + 15) >> 4; }

template <int P>
__global__ void __launch_bounds__(kMaxThreads) ctc_align_viterbi_kernel(
    const __nv_bfloat16* __restrict__ x, long long fs, long long bs, const float* __restrict__ lse,
    const int* __restrict__ input_len, const int* __restrict__ targets, int Smax, const int* __restrict__ target_len, int T,
    int V, int blank, uint32_t* __restrict__ bp, int* __restrict__ labels, float* __restrict__ score) {
  constexpr int H = P / 2;                  // label positions per thread (odd j), the even ones are blanks
  constexpr int HP = (H + 1) / 2;           // registers holding them (and their prefetched logits) two to a register
  constexpr int kPre = P >= 16 ? 2 : 4;     // register prefetch distance in frames
  constexpr int G = P < 16 ? 16 / P : 1;    // lanes sharing one backpointer word
  constexpr int NW = P < 16 ? 1 : P / 16;   // backpointer words per thread
  __shared__ float nb[2][kMaxWarps][2];     // [parity][warp][last, second to last] alpha of each warp's last lane
  __shared__ int bad, reps;
  __shared__ float fin[2];
  pdl_grid_sync();
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int s0 = tid * P, W = words_per_frame(Smax);
  const int len = min(max(input_len[b], 0), T);
  const int tl_raw = target_len[b], tl = min(max(tl_raw, 0), Smax), L = 2 * tl + 1;
  if (tid == 0) {
    bad = (tl_raw < 0 || tl_raw > Smax) ? 1 : 0;
    reps = 0;
  }
  __syncthreads();
  const int* tg = targets + static_cast<long long>(b) * Smax;
  uint32_t lab[HP];                // the thread's labels, two 16-bit class ids per register
  uint32_t skip = 0, valid = 0;    // bit j: position s0 + j skips / lies inside [0, L)
  int nrep = 0, nbad = 0;
#pragma unroll
  for (int h = 0; h < HP; ++h) lab[h] = static_cast<uint32_t>(blank) * 0x10001u;
#pragma unroll
  for (int h = 0; h < H; ++h) {
    const int k = (s0 >> 1) + h;  // label index of position s0 + 2h + 1
    if (k < tl) {
      const int c = tg[k];
      nbad += (c < 0 || c >= V || c == blank) ? 1 : 0;
      const uint32_t cc = (c < 0 || c >= V) ? blank : c;
      lab[h >> 1] = (h & 1) ? ((lab[h >> 1] & 0xffffu) | (cc << 16)) : ((lab[h >> 1] & 0xffff0000u) | cc);
      if (k > 0) {
        const int p = tg[k - 1];
        if (p == c) ++nrep;
        else skip |= 1u << (2 * h + 1);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < P; ++j)
    if (s0 + j < L) valid |= 1u << j;
  if (nbad) bad = 1;
  if (nrep) atomicAdd(&reps, nrep);  // integer: order does not matter
  __syncthreads();
  const bool infeasible = bad || len < tl + reps;
  if (infeasible) {
    if (tid == 0) {
      score[b] = -INFINITY;
      if (len > 0) labels[static_cast<long long>(b) * T + len - 1] = -1;
    }
    return;
  }
  if (len == 0) {  // S = 0 on no frames: the empty path
    if (tid == 0) score[b] = 0.f;
    return;
  }

  const __nv_bfloat16* x_b = x + b * bs;
  const float* lse_b = lse + static_cast<long long>(b) * T;
  uint32_t* bp_b = bp + static_cast<long long>(b) * T * W;
  float a[P];
#pragma unroll
  for (int j = 0; j < P; ++j) a[j] = -INFINITY;
  if (tid == 0) a[0] = 0.f;  // "alpha_{-1}": all mass before position 0, so frame 0 needs no special case
  if (lane == 31) {
    nb[0][warp][0] = a[P - 1];
    nb[0][warp][1] = a[P - 2];
  }
  const bool any = s0 < L;  // a thread wholly past L only keeps -inf and writes its backpointer words
  float q_lse[kPre], q_b[kPre];
  uint32_t q_l[kPre][HP];  // raw bf16 logits of the labels, two to a register
#pragma unroll
  for (int f = 0; f < kPre; ++f) {
    q_lse[f] = 0.f;
    q_b[f] = 0.f;
#pragma unroll
    for (int h = 0; h < HP; ++h) q_l[f][h] = 0u;
    if (f < len) {
      q_lse[f] = lse_b[f];
      if (any) load_row<HP>(x_b + f * fs, blank, lab, q_b[f], q_l[f]);
    }
  }
  __syncthreads();
  int cur = 0;
  for (int t0 = 0; t0 < len; t0 += kPre) {
#pragma unroll
    for (int f = 0; f < kPre; ++f) {
      const int t = t0 + f;
      if (t >= len) break;
      const float lse_t = q_lse[f];
      const float e_b = q_b[f] - lse_t;
      float e_l[H];
#pragma unroll
      for (int h = 0; h < H; ++h)
        e_l[h] = __uint_as_float((h & 1) ? (q_l[f][h >> 1] & 0xffff0000u) : (q_l[f][h >> 1] << 16)) - lse_t;
      if (t + kPre < len) {
        q_lse[f] = lse_b[t + kPre];
        if (any) load_row<HP>(x_b + (t + kPre) * fs, blank, lab, q_b[f], q_l[f]);
      }
      // neighbours below s0: lane - 1, or the previous warp's last lane through shared memory
      float p1 = __shfl_up_sync(0xffffffffu, a[P - 1], 1), p2 = __shfl_up_sync(0xffffffffu, a[P - 2], 1);
      if (lane == 0) {
        p1 = warp > 0 ? nb[cur][warp - 1][0] : -INFINITY;
        p2 = warp > 0 ? nb[cur][warp - 1][1] : -INFINITY;
      }
      uint32_t code[NW];
#pragma unroll
      for (int w = 0; w < NW; ++w) code[w] = 0;
      float n[P];
#pragma unroll
      for (int j = 0; j < P; ++j) {
        const float x0 = a[j];
        const float x1 = j >= 1 ? a[j - 1] : p1;
        const float x2 = (skip >> j & 1) ? (j >= 2 ? a[j - 2] : (j == 1 ? p1 : p2)) : -INFINITY;
        float v;
        uint32_t c;
        if (x2 > x1 && x2 > x0) {
          v = x2;
          c = 2;
        } else if (x1 > x0 && x1 > x2) {
          v = x1;
          c = 1;
        } else {
          v = x0;
          c = 0;
        }
        v += (j & 1) ? e_l[j >> 1] : e_b;
        n[j] = (valid >> j & 1) ? v : -INFINITY;
        code[j >> 4] |= c << (2 * ((s0 + j) & 15));
      }
#pragma unroll
      for (int j = 0; j < P; ++j) a[j] = n[j];
      if (lane == 31) {
        nb[cur ^ 1][warp][0] = a[P - 1];
        nb[cur ^ 1][warp][1] = a[P - 2];
      }
      if constexpr (G > 1) {
#pragma unroll
        for (int o = 1; o < G; o <<= 1) code[0] |= __shfl_xor_sync(0xffffffffu, code[0], o);
      }
      uint32_t* row_bp = bp_b + static_cast<long long>(t) * W;
      const int w0 = s0 >> 4;
      if (G == 1 || (tid & (G - 1)) == 0) {
#pragma unroll
        for (int w = 0; w < NW; ++w)
          if (w0 + w < W) row_bp[w0 + w] = code[w];
      }
      __syncthreads();
      cur ^= 1;
    }
  }
  // end position: L-1 if alpha(L-1) > alpha(L-2), else L-2 (position 0 when S = 0)
#pragma unroll
  for (int j = 0; j < P; ++j) {
    if (s0 + j == L - 1) fin[0] = a[j];
    if (s0 + j == L - 2) fin[1] = a[j];
  }
  __syncthreads();
  if (tid == 0) {
    const bool last_blank = L == 1 || fin[0] > fin[1];
    score[b] = last_blank ? fin[0] : fin[1];
    labels[static_cast<long long>(b) * T + len - 1] = last_blank ? L - 1 : L - 2;
  }
}

// One warp per utterance, launched after the Viterbi kernel on the same stream.
__global__ void __launch_bounds__(32) ctc_align_backtrack_kernel(
    const __nv_bfloat16* __restrict__ x, long long fs, long long bs, const float* __restrict__ lse,
    const int* __restrict__ input_len, const int* __restrict__ targets, int Smax, int T, int blank,
    const uint32_t* __restrict__ bp, int* __restrict__ labels, float* __restrict__ frame_scores) {
  __shared__ uint32_t sw[kChunk][kWin];
  __shared__ int spos[kChunk];
  pdl_grid_sync();
  const int b = blockIdx.x, lane = threadIdx.x, W = words_per_frame(Smax);
  const int len = min(max(input_len[b], 0), T);
  int* lab_b = labels + static_cast<long long>(b) * T;
  float* fs_b = frame_scores + static_cast<long long>(b) * T;
  for (int t = len + lane; t < T; t += 32) {  // padded frames
    lab_b[t] = -1;
    fs_b[t] = 0.f;
  }
  if (len == 0) return;
  int pos = lab_b[len - 1];  // hand-off from the Viterbi kernel: the end position, -1 = infeasible
  __syncwarp();
  if (pos < 0) {
    for (int t = lane; t < len; t += 32) {
      lab_b[t] = -1;
      fs_b[t] = 0.f;
    }
    return;
  }
  const int* tg = targets + static_cast<long long>(b) * Smax;
  const __nv_bfloat16* x_b = x + b * bs;
  const float* lse_b = lse + static_cast<long long>(b) * T;
  const uint32_t* bp_b = bp + static_cast<long long>(b) * T * W;
  for (int hi = len - 1; hi >= 0; hi -= kChunk) {
    const int wlo = max((pos >> 4) - (kWin - 1), 0);
    const int t = hi - lane;
    if (t >= 0) {
#pragma unroll
      for (int k = 0; k < kWin; ++k) sw[lane][k] = (wlo + k < W) ? bp_b[static_cast<long long>(t) * W + wlo + k] : 0u;
    }
    __syncwarp();
    if (lane == 0) {
      for (int i = 0; i < kChunk && hi - i >= 0; ++i) {
        spos[i] = pos;
        pos -= (sw[i][(pos >> 4) - wlo] >> (2 * (pos & 15))) & 3u;
      }
    }
    __syncwarp();
    pos = __shfl_sync(0xffffffffu, pos, 0);
    if (t >= 0) {
      const int p = spos[lane];
      const int c = (p & 1) ? tg[p >> 1] : blank;
      lab_b[t] = c;
      fs_b[t] = bf(x_b + t * fs + c) - lse_b[t];
    }
    __syncwarp();
  }
}

template <int P>
cudaError_t launch_viterbi(int B, cudaStream_t st, const __nv_bfloat16* x, long long fs, long long bs, const float* lse,
                           const int* input_len, const int* targets, int Smax, const int* target_len, int T, int V, int blank,
                           uint32_t* bp, int* labels, float* score) {
  const int threads = ceil_div(ceil_div(2 * Smax + 1, P), 32) * 32;
  return launch_pdl(ctc_align_viterbi_kernel<P>, dim3(B), dim3(threads), 0, st, x, fs, bs, lse, input_len, targets, Smax,
                    target_len, T, V, blank, bp, labels, score);
}

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

long long b200s_ctc_align_workspace_bytes(int B, int T, int Smax) {
  if (B < 1 || T < 1 || Smax < 0 || Smax > B200S_CTC_ALIGN_MAX_TARGET) return -1;
  return static_cast<long long>(B) * T * ((2LL * Smax + 1 + 15) / 16) * 4;
}

int b200s_ctc_align(const void* logits, long long frame_stride, long long batch_stride, const float* lse, const int* input_len,
                    const int* targets, int Smax, const int* target_len, int B, int T, int V, int blank, void* workspace,
                    long long workspace_bytes, int* labels, float* frame_scores, float* score, b200s_stream stream) {
  B200_CHECK_ARG(logits && lse && input_len && target_len && workspace && labels && frame_scores && score,
                 "ctc_align: null pointer");
  B200_CHECK_ARG(B > 0 && T > 0, "ctc_align: need B > 0 and T > 0 (B=%d T=%d)", B, T);
  B200_CHECK_ARG(V >= 1 && V <= kMaxV, "ctc_align: V=%d outside [1, %d]", V, kMaxV);
  B200_CHECK_ARG(blank >= 0 && blank < V, "ctc_align: blank=%d outside [0, V=%d)", blank, V);
  B200_CHECK_ARG(Smax >= 0 && Smax <= B200S_CTC_ALIGN_MAX_TARGET, "ctc_align: Smax=%d outside [0, %d]", Smax,
                 B200S_CTC_ALIGN_MAX_TARGET);
  B200_CHECK_ARG(targets || Smax == 0, "ctc_align: null targets");
  const long long need = b200s_ctc_align_workspace_bytes(B, T, Smax);
  B200_CHECK_ARG(workspace_bytes >= need, "ctc_align: workspace of %lld bytes, need %lld", workspace_bytes, need);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const auto* x = static_cast<const __nv_bfloat16*>(logits);
  auto* bp = static_cast<uint32_t*>(workspace);
  const int Lmax = 2 * Smax + 1;
  cudaError_t e;
  if (Lmax <= 2 * kMaxThreads)
    e = launch_viterbi<2>(B, st, x, frame_stride, batch_stride, lse, input_len, targets, Smax, target_len, T, V, blank, bp,
                          labels, score);
  else if (Lmax <= 4 * kMaxThreads)
    e = launch_viterbi<4>(B, st, x, frame_stride, batch_stride, lse, input_len, targets, Smax, target_len, T, V, blank, bp,
                          labels, score);
  else if (Lmax <= 8 * kMaxThreads)
    e = launch_viterbi<8>(B, st, x, frame_stride, batch_stride, lse, input_len, targets, Smax, target_len, T, V, blank, bp,
                          labels, score);
  else if (Lmax <= 16 * kMaxThreads)
    e = launch_viterbi<16>(B, st, x, frame_stride, batch_stride, lse, input_len, targets, Smax, target_len, T, V, blank, bp,
                           labels, score);
  else
    e = launch_viterbi<32>(B, st, x, frame_stride, batch_stride, lse, input_len, targets, Smax, target_len, T, V, blank, bp,
                           labels, score);
  B200_CHECK_CUDA(e);
  B200_CHECK_LAUNCH();
  B200_CHECK_CUDA(launch_pdl(ctc_align_backtrack_kernel, dim3(B), dim3(32), 0, st, x, frame_stride, batch_stride, lse, input_len,
                             targets, Smax, T, blank, static_cast<const uint32_t*>(bp), labels, frame_scores));
  B200_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"
