// Device helpers shared by the CTC beam-search kernels (csrc/ctc_decode.cu: lexicon-free, csrc/ctc_decode_lex.cu: lexicon-
// constrained): the rolling hash, lae, the (score, hash) keys and their block radix select, and the n-gram LM lookups.
#pragma once

#include <math.h>

#include "../../include/unispeech_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace b200 {

// Backtrack of a beam search (csrc/ctc_decode.cu): one warp per (utterance, n-best entry) over the backpointers `bp`
// ((parent slot | (appended class + 1) << 8) per (b, t, slot)); lengths[b, n] holds the final slot on entry (-1 for none) and
// the hypothesis length on exit.  Launched with PDL on `st` after the search kernel that wrote bp and lengths.
cudaError_t ctc_decode_backtrack_launch(const int* input_len, int B, int T, int beam, int nbest, const uint32_t* bp,
                                        int* tokens, int* lengths, cudaStream_t st);

namespace {

constexpr int kMaxV = 1024;
constexpr int kMaxBeam = B200S_CTC_DECODE_MAX_BEAM;
constexpr int kCtx = B200S_CTC_LM_MAX_ORDER - 1;  // words of LM context a beam keeps
constexpr int kThreads = 256;
constexpr float kLn10 = 2.302585092994046f;

__device__ __forceinline__ uint64_t splitmix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
// The one rolling hash: prefixes (class ids), partial words (class ids), spellings (class ids) and n-grams (word ids), each
// from 0 for the empty sequence.
__device__ __forceinline__ uint64_t hash_step(uint64_t h, int x) { return splitmix64(h ^ static_cast<uint64_t>(x + 1)); }

// log(exp(a) + exp(b)) in fp32; exactly symmetric, -inf when both are
__device__ __forceinline__ float lae(float a, float b) {
  const float m = fmaxf(a, b);
  if (m == -INFINITY) return -INFINITY;
  return m + log1pf(expf(-fabsf(a - b)));
}

// Order-preserving map of an fp32 score to uint32 (larger score, larger key).
__device__ __forceinline__ uint32_t ord(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

struct Key {     // (s, h) compared lexicographically, larger is better
  uint32_t s;
  uint64_t h;
};

__device__ __forceinline__ uint32_t digit(const Key& k, int d) {
  return d < 32 ? (k.s >> (24 - d)) & 255u : static_cast<uint32_t>(k.h >> (88 - d)) & 255u;
}
// top d bits of k == / >= those of p (p's lower bits are zero)
__device__ __forceinline__ bool top_eq(const Key& k, const Key& p, int d) {
  if (d == 0) return true;
  if (d <= 32) return ((k.s ^ p.s) >> (32 - d)) == 0;
  if (k.s != p.s) return false;
  return d == 96 ? k.h == p.h : ((k.h ^ p.h) >> (96 - d)) == 0;
}
__device__ __forceinline__ bool top_ge(const Key& k, const Key& p, int d) {
  if (d == 0) return true;
  if (d <= 32) return (k.s >> (32 - d)) >= (p.s >> (32 - d));
  if (k.s != p.s) return k.s > p.s;
  return d == 96 ? k.h >= p.h : (k.h >> (96 - d)) >= (p.h >> (96 - d));
}
__device__ __forceinline__ bool better(const Key& a, const Key& b) { return a.s != b.s ? a.s > b.s : a.h > b.h; }

struct Entry {  // a selected key and the index of its candidate
  Key k;
  int q;
};

struct Select {  // result of select_top: keys whose top d bits are >= those of p are the chosen ones
  Key p;
  int d, r, done;
  int hist[256];
};

// Block-wide radix select (8-bit digits, most significant first) of the `need` best of n keys; key(q, with_hash, k) returns
// false for an entry that takes no part.  The hash half of a key is only asked for once the score digits do not separate.
template <class F>
__device__ void select_top(int n, int need, F key, Select& sel) {
  const int tid = threadIdx.x, lane = tid & 31;
  if (tid == 0) {
    sel.p = Key{0u, 0ull};
    sel.d = 0;
    sel.r = need;
    sel.done = 0;
  }
  for (int d = 0; d < 96; d += 8) {
    for (int i = tid; i < 256; i += kThreads) sel.hist[i] = 0;
    __syncthreads();
    const Key p = sel.p;
    for (int q = tid; q < n; q += kThreads) {
      Key k;
      if (key(q, d >= 32, k) && top_eq(k, p, d)) atomicAdd(&sel.hist[digit(k, d)], 1);  // integer: order does not matter
    }
    __syncthreads();
    if (tid < 32) {
      // lane l owns bins 255 - 8 l .. 248 - 8 l (descending)
      int c[8], s = 0;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        c[i] = sel.hist[255 - 8 * lane - i];
        s += c[i];
      }
      int incl = s;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      const int total = __shfl_sync(0xffffffffu, incl, 31), r = sel.r;
      if (d == 0 && total <= r) {
        if (lane == 0) sel.done = 1;  // everything is chosen (d stays 0)
      } else {
        const int excl = incl - s;
        if (excl < r && r <= incl) {  // exactly one lane
          int above = excl, bin = 0, cnt = 0;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            if (cnt == 0 && above + c[i] >= r) {
              bin = 255 - 8 * lane - i;
              cnt = c[i];
            } else if (cnt == 0) {
              above += c[i];
            }
          }
          Key np = sel.p;
          if (d < 32) np.s |= static_cast<uint32_t>(bin) << (24 - d);
          else np.h |= static_cast<uint64_t>(bin) << (88 - d);
          sel.p = np;
          sel.d = d + 8;
          sel.r = r - above;
          if (cnt == r - above || d + 8 == 96) sel.done = 1;
        }
      }
    }
    __syncthreads();
    if (sel.done) break;
  }
}

struct Lm {
  const unsigned long long* ng_keys;
  const uint2* ng_vals;  // (log10 p, log10 backoff) as fp32 bits
  unsigned long long ng_mask;
  const unsigned long long* sp_keys;
  const uint2* sp_vals;  // (word id, 0)
  unsigned long long sp_mask;
  int order, bos, eos, unk, has_unk;
  float weight, word_score, unk_score;
};

__device__ __forceinline__ int probe(const unsigned long long* keys, unsigned long long mask, uint64_t key) {
  if (key == 0) return -1;
  for (unsigned long long s = key & mask;; s = (s + 1) & mask) {
    const unsigned long long k = keys[s];
    if (k == key) return static_cast<int>(s);
    if (k == 0) return -1;
  }
}

// ln P(w | ctx[0..m)) by ARPA backoff: the longest n-gram (ctx suffix, w) that exists gives log10 p; each longer context that
// did not match adds its log10 backoff (0 when it is not an n-gram).  Summed in fp32 from the longest context down, then p,
// then scaled by ln 10.
__device__ float ln_prob(const Lm& lm, const int* ctx, int m, int w) {
  float acc = 0.f;
  for (int L = m; L >= 0; --L) {
    uint64_t k = 0;
    for (int i = m - L; i < m; ++i) k = hash_step(k, ctx[i]);
    const uint64_t kc = k;
    k = hash_step(k, w);
    const int s = probe(lm.ng_keys, lm.ng_mask, k);
    if (s >= 0) {
      acc = __fadd_rn(acc, __uint_as_float(lm.ng_vals[s].x));
      break;
    }
    if (L >= 1) {
      const int sc = probe(lm.ng_keys, lm.ng_mask, kc);
      if (sc >= 0) acc = __fadd_rn(acc, __uint_as_float(lm.ng_vals[sc].y));
    }
  }
  return __fmul_rn(acc, kLn10);
}

// Append word w to a context that keeps the last order - 1 words.
__device__ __forceinline__ void push_word(int* ctx, int& m, int w, int order) {
  if (order <= 1) return;
  if (m < order - 1) {
    ctx[m++] = w;
    return;
  }
#pragma unroll
  for (int i = 0; i + 1 < kCtx; ++i)
    if (i + 1 < m) ctx[i] = ctx[i + 1];
  ctx[m - 1] = w;
}

}  // namespace

}  // namespace b200
