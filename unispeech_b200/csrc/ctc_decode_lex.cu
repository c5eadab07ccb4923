// Lexicon-constrained CTC prefix beam search: the search of csrc/ctc_decode.cu with every partial word held to a path of a word
// trie (flashlight's LexiconDecoder), optional word n-gram LM scoring at word boundaries, and the LM look-ahead of each trie node
// ("max smearing") in the ranking score.  The semantics are written down in include/unispeech_b200.h
// (b200s_ctc_decode_lexicon) and restated in numpy by oracle/lexicon_oracle.py, which is their definition.
//
//   search kernel       one CTA per utterance, beams in shared memory double-buffered by frame; a beam carries its trie node in
//                       place of the partial word's hash.  Per frame: lp of the frame into shared memory; the top beam_token
//                       non-blank classes T_K (block radix select on (lp, -class)) as a bitmask and as a list in class order;
//                       one thread per beam loads its node's child mask into shared memory (with the running popcount that
//                       numbers the children) and ANDs it with T_K, plus the boundary bit where the node may end a word; the
//                       stay of every beam, with the extension of its parent that reaches the same prefix merged in and that
//                       extension's bit cleared; then a block radix select of the beam best over the stays and the (beam,
//                       T_K position) pairs whose bit is set, by (score desc, prefix hash asc), and a rank count.
//   backtrack           ctc_decode.cu's backtrack kernel (ctc_decode_backtrack_launch): the backpointers have its format.
//
// Trie (built on the host, unispeech_b200/lexicon.py): nodes in BFS order with the children of a node contiguous in class order;
// per node a child bitmask over the classes (W = ceil(V / 32) words), the index of its first child (a child is first_child +
// the number of mask bits below its class), the word it ends (-1 none, -2 a word the LM does not know, else its LM word id) and
// its look-ahead score.  Nothing is hashed, so nothing can collide.
//
// No candidate pruning.  ctc_decode.cu extends each beam only by the first min(beam_token, beam + 2) classes of T_K, because
// each of those positions holds a candidate at least as good as any later one.  That argument fails here twice: the lexicon
// removes classes per beam (the first positions may hold no candidate of this beam at all), and the look-ahead reorders the
// extensions of one parent (a class of lower lp can lead to a node of a much better smear).  So every allowed (beam, T_K
// position) pair takes part, and beam_token is what bounds the work: at most beam * (beam_token + 1) <= 128 * 1024
// candidates per frame.  They are enumerated by index, never stored, so no limit beyond those of b200s_ctc_decode applies.
#include "ctc_decode_common.cuh"

namespace b200 {

namespace {

constexpr int kMaxW = kMaxV / 32;

struct LexBeams {
  unsigned long long h[kMaxBeam], ph[kMaxBeam];  // prefix, prefix without its last class
  float pb[kMaxBeam], pnb[kMaxBeam], lm[kMaxBeam];
  int node[kMaxBeam], last[kMaxBeam], nctx[kMaxBeam];
  int ctx[kCtx][kMaxBeam];
};

struct Trie {
  const uint32_t* mask;   // [nodes, W]
  const int* first;       // [nodes]
  const int* word;        // [nodes]
  const float* smear;     // [nodes], or null: no look-ahead
  int W;
};

// LM part of ending the word `end` (a trie node's word: -2 a word the LM does not know, else its LM word id) after context
// ctx[0..m); *wid = the word id it pushes.  Without an LM only word_score.
__device__ float lex_word_term(const Lm& lm, int end, const int* ctx, int m, int* wid) {
  const bool oov = end < 0;
  *wid = oov ? lm.unk : end;
  if (lm.order == 0) return lm.word_score;
  float t = 0.f;
  if (!oov || lm.has_unk) t = __fmul_rn(lm.weight, ln_prob(lm, ctx, m, *wid));
  t = __fadd_rn(t, lm.word_score);
  if (oov) t = __fadd_rn(t, lm.unk_score);
  return t;
}

// the LM part of a ranking score: lm + lm_weight * smear(node), in that fp32 order
__device__ __forceinline__ float rank_lm(const Lm& lm, float l, float smear) { return __fadd_rn(l, __fmul_rn(lm.weight, smear)); }

__global__ void __launch_bounds__(kThreads, 1) ctc_decode_lexicon_kernel(
    const __nv_bfloat16* __restrict__ x, long long fs, long long bs, const float* __restrict__ lse,
    const int* __restrict__ input_len, int T, int V, int blank, int beam, int nbest, int beam_token, int boundary, Lm lm,
    Trie trie, uint32_t* __restrict__ bp, int* __restrict__ lengths, float* __restrict__ scores) {
  __shared__ LexBeams bm[2];
  __shared__ float lps[kMaxV];
  __shared__ short tk[kMaxV];           // T_K in class order
  __shared__ uint32_t inset[kMaxW];     // T_K membership
  __shared__ int ipre[kMaxW];           // T_K members in the words below
  __shared__ float base[kMaxBeam], sscore[kMaxBeam], spb[kMaxBeam], spnb[kMaxBeam], bdelta[kMaxBeam];
  __shared__ int bwid[kMaxBeam];
  __shared__ Entry list[kMaxBeam];
  __shared__ int nlist, nvalid;
  __shared__ Select sel;
  // per beam, W words each: the node's child mask, the candidate bits (children and the boundary, in T_K, not merged into a
  // stay), and the number of children in the words below
  extern __shared__ uint32_t dyn[];
  const int W = trie.W;
  uint32_t* cmask = dyn;
  uint32_t* cbit = dyn + beam * W;
  unsigned short* cpre = reinterpret_cast<unsigned short*>(dyn + 2 * beam * W);
  pdl_grid_sync();
  const int b = blockIdx.x, tid = threadIdx.x;
  const int len = min(max(input_len[b], 0), T);
  const bool use_lm = lm.order > 0;
  const int K = beam_token;
  const bool all_in = K >= V - 1;
  const __nv_bfloat16* x_b = x + b * bs;
  const float* lse_b = lse + static_cast<long long>(b) * T;
  uint32_t* bp_b = bp + static_cast<long long>(b) * T * beam;
  if (tid == 0) {
    bm[0].h[0] = bm[0].ph[0] = 0ull;
    bm[0].pb[0] = 0.f;
    bm[0].pnb[0] = -INFINITY;
    bm[0].lm[0] = 0.f;
    bm[0].node[0] = 0;
    bm[0].last[0] = -1;
    bm[0].nctx[0] = 0;
    if (use_lm && lm.order > 1) {
      bm[0].ctx[0][0] = lm.bos;
      bm[0].nctx[0] = 1;
    }
  }
  int nb = 1;
  auto tok_key = [&](int c, bool, Key& k) {
    if (c == blank) return false;
    k = Key{ord(lps[c]), ~static_cast<uint64_t>(c)};
    return true;
  };
  auto smear_of = [&](int node) { return trie.smear != nullptr ? trie.smear[node] : 0.f; };
  // the child of beam j's node by class c (a bit of its child mask)
  auto child_of = [&](int j, int node, int c) {
    const int w = c >> 5;
    return trie.first[node] + cpre[j * W + w] + __popc(cmask[j * W + w] & ((1u << (c & 31)) - 1u));
  };
  for (int t = 0; t < len; ++t) {
    const LexBeams& cb = bm[t & 1];
    LexBeams& nx = bm[(t & 1) ^ 1];
    const float lse_t = lse_b[t];
    const __nv_bfloat16* row = x_b + t * fs;
    for (int c = tid; c < V; c += kThreads) lps[c] = __bfloat162float(row[c]) - lse_t;
    for (int i = tid; i < kMaxW; i += kThreads) {
      uint32_t m = 0u;
      if (all_in) {
        const int lo = 32 * i;
        m = lo + 32 <= V ? 0xffffffffu : (lo < V ? (1u << (V - lo)) - 1u : 0u);
        if ((blank >> 5) == i) m &= ~(1u << (blank & 31));
      }
      inset[i] = m;
    }
    if (tid == 0) nlist = 0;
    __syncthreads();
    // ---- T_K: membership, then the list in class order
    if (!all_in) {
      select_top(V, K, tok_key, sel);
      const Key p = sel.p;
      const int d = sel.d;
      for (int c = tid; c < V; c += kThreads) {
        Key k;
        if (tok_key(c, true, k) && top_ge(k, p, d)) atomicOr(&inset[c >> 5], 1u << (c & 31));
      }
      __syncthreads();
    }
    if (tid < 32) {
      const int cnt = tid < W ? __popc(inset[tid]) : 0;
      int incl = cnt;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (tid >= o) incl += v;
      }
      ipre[tid] = incl - cnt;
    }
    // ---- per beam: the node's child mask and candidate bits; the LM term of ending its word
    if (tid < nb) {
      const int j = tid, node = cb.node[j];
      const int end = node != 0 ? trie.word[node] : -1;
      const bool bok = node == 0 || end != -1;  // the boundary may follow: an empty word, or a word's end
      int run = 0;
      for (int w = 0; w < W; ++w) {
        const uint32_t m = trie.mask[static_cast<long long>(node) * W + w];
        uint32_t bits = m;
        if (bok && (boundary >> 5) == w) bits |= 1u << (boundary & 31);
        cmask[j * W + w] = m;
        cbit[j * W + w] = bits & inset[w];
        cpre[j * W + w] = static_cast<unsigned short>(run);
        run += __popc(m);
      }
      float bd = 0.f;
      int wid = -1;
      if (node != 0 && end != -1 && ((inset[boundary >> 5] >> (boundary & 31)) & 1u)) {
        int ctx[kCtx > 0 ? kCtx : 1];
#pragma unroll
        for (int u = 0; u < kCtx; ++u) ctx[u] = cb.ctx[u][j];
        bd = lex_word_term(lm, end, ctx, cb.nctx[j], &wid);
      }
      bdelta[j] = bd;
      bwid[j] = wid;
    }
    __syncthreads();
    for (int c = tid; c < V; c += kThreads) {
      const uint32_t m = inset[c >> 5];
      if ((m >> (c & 31)) & 1u) tk[ipre[c >> 5] + __popc(m & ((1u << (c & 31)) - 1u))] = static_cast<short>(c);
    }
    // ---- stays (blank, repeat) with the merged extension of their parent
    if (tid < nb) {
      const int i = tid, li = cb.last[i];
      const float a = lae(cb.pb[i], cb.pnb[i]);
      base[i] = a;
      spb[i] = a + lps[blank];
      float pnb = li >= 0 ? cb.pnb[i] + lps[li] : -INFINITY;
      if (li >= 0) {
        const unsigned long long ph = cb.ph[i];
        int j = -1;
        for (int u = 0; u < nb && j < 0; ++u)
          if (cb.h[u] == ph && u != i) j = u;
        // only this thread touches bit li of beam j: prefix(j) + li is beam i's prefix
        const uint32_t bit = 1u << (li & 31);
        if (j >= 0 && (cbit[j * W + (li >> 5)] & bit)) {
          const float e = (li == cb.last[j] ? cb.pb[j] : lae(cb.pb[j], cb.pnb[j])) + lps[li];
          pnb = lae(pnb, e);
          atomicAnd(&cbit[j * W + (li >> 5)], ~bit);
        }
      }
      spnb[i] = pnb;
      sscore[i] = __fadd_rn(lae(spb[i], pnb), rank_lm(lm, cb.lm[i], smear_of(cb.node[i])));
    }
    __syncthreads();
    // ---- candidates: q < nb the stay of beam q, else parent (q - nb) / K extended by the class at T_K position (q - nb) % K
    auto cand = [&](int q, bool with_hash, Key& k) {
      if (q < nb) {
        k = Key{ord(sscore[q]), with_hash ? ~static_cast<uint64_t>(cb.h[q]) : 0ull};
        return true;
      }
      const int e = q - nb, j = e / K, c = tk[e - j * K];
      if (!((cbit[j * W + (c >> 5)] >> (c & 31)) & 1u)) return false;
      const float ac = (c == cb.last[j] ? cb.pb[j] : base[j]) + lps[c];
      float r;
      if (c == boundary) {
        r = rank_lm(lm, cb.node[j] != 0 ? __fadd_rn(cb.lm[j], bdelta[j]) : cb.lm[j], 0.f);
      } else {
        const int node = cb.node[j];
        r = rank_lm(lm, cb.lm[j], smear_of(child_of(j, node, c)));
      }
      k = Key{ord(__fadd_rn(ac, r)), with_hash ? ~static_cast<uint64_t>(hash_step(cb.h[j], c)) : 0ull};
      return true;
    };
    const int n = nb + nb * K;
    select_top(n, beam, cand, sel);
    {
      const Key p = sel.p;
      const int d = sel.d;
      for (int q = tid; q < n; q += kThreads) {
        Key k;
        if (cand(q, true, k) && top_ge(k, p, d)) {
          const int i = atomicAdd(&nlist, 1);
          if (i < beam) list[i] = Entry{k, q};
        }
      }
    }
    __syncthreads();
    const int nn = min(nlist, beam);
    if (tid < nn) {
      const Entry e = list[tid];
      int r = 0;
      for (int i = 0; i < nn; ++i) r += better(list[i].k, e.k) ? 1 : 0;
      const int q = e.q;
      int j, c;
      if (q < nb) {
        j = q;
        c = -1;
        nx.h[r] = cb.h[j];
        nx.ph[r] = cb.ph[j];
        nx.pb[r] = spb[j];
        nx.pnb[r] = spnb[j];
        nx.lm[r] = cb.lm[j];
        nx.node[r] = cb.node[j];
        nx.last[r] = cb.last[j];
        nx.nctx[r] = cb.nctx[j];
#pragma unroll
        for (int u = 0; u < kCtx; ++u) nx.ctx[u][r] = cb.ctx[u][j];
      } else {
        const int ee = q - nb;
        j = ee / K;
        c = tk[ee - j * K];
        nx.h[r] = ~e.k.h;
        nx.ph[r] = cb.h[j];
        nx.pb[r] = -INFINITY;
        nx.pnb[r] = (c == cb.last[j] ? cb.pb[j] : base[j]) + lps[c];
        nx.last[r] = c;
        int ctx[kCtx > 0 ? kCtx : 1], m = cb.nctx[j];
#pragma unroll
        for (int u = 0; u < kCtx; ++u) ctx[u] = cb.ctx[u][j];
        float l = cb.lm[j];
        int node = 0;
        if (c == boundary) {
          if (cb.node[j] != 0) {
            l = __fadd_rn(l, bdelta[j]);
            if (use_lm) push_word(ctx, m, bwid[j], lm.order);
          }
        } else {
          node = child_of(j, cb.node[j], c);
        }
        nx.node[r] = node;
        nx.lm[r] = l;
        nx.nctx[r] = m;
#pragma unroll
        for (int u = 0; u < kCtx; ++u) nx.ctx[u][r] = ctx[u];
      }
      bp_b[static_cast<long long>(t) * beam + r] = static_cast<uint32_t>(j) | (static_cast<uint32_t>(c + 1) << 8);
    }
    nb = nn;
    __syncthreads();
  }
  // ---- end of utterance: the open word (a hypothesis inside a word that is not a lexicon word is dropped) and </s>, then the
  // n-best of the survivors by (score desc, hash asc)
  const LexBeams& fb = bm[len & 1];
  if (tid == 0) nvalid = 0;
  __syncthreads();
  if (tid < nb) {
    const int node = fb.node[tid];
    const int end = node != 0 ? trie.word[node] : -1;
    const bool valid = node == 0 || end != -1;
    float s = -INFINITY;
    if (valid) {
      float l = fb.lm[tid];
      int ctx[kCtx > 0 ? kCtx : 1], m = fb.nctx[tid];
#pragma unroll
      for (int u = 0; u < kCtx; ++u) ctx[u] = fb.ctx[u][tid];
      if (node != 0) {
        int wid;
        l = __fadd_rn(l, lex_word_term(lm, end, ctx, m, &wid));
        if (use_lm) push_word(ctx, m, wid, lm.order);
      }
      if (use_lm) l = __fadd_rn(l, __fmul_rn(lm.weight, ln_prob(lm, ctx, m, lm.eos)));
      s = lae(fb.pb[tid], fb.pnb[tid]) + l;
      atomicAdd(&nvalid, 1);
    }
    sscore[tid] = s;
    bwid[tid] = valid ? 1 : 0;
  }
  __syncthreads();
  if (tid < nb && bwid[tid]) {
    const Key e{ord(sscore[tid]), ~static_cast<uint64_t>(fb.h[tid])};
    int r = 0;
    for (int i = 0; i < nb; ++i)
      r += (bwid[i] && better(Key{ord(sscore[i]), ~static_cast<uint64_t>(fb.h[i])}, e)) ? 1 : 0;
    if (r < nbest) {
      scores[b * nbest + r] = sscore[tid];
      lengths[b * nbest + r] = tid;  // hand-off to the backtrack: the final slot
    }
  }
  if (tid < nbest && tid >= nvalid) {
    scores[b * nbest + tid] = -INFINITY;
    lengths[b * nbest + tid] = -1;
  }
}

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

long long b200s_ctc_trie_bytes(long long nodes, int V) {
  if (nodes < 1 || V < 2 || V > kMaxV) return -1;
  return nodes * (4LL * ((V + 31) / 32) + 12);
}

int b200s_ctc_decode_lexicon(const void* logits, long long frame_stride, long long batch_stride, const float* lse,
                             const int* input_len, int B, int T, int V, int blank, int beam, int nbest, int beam_token,
                             int word_boundary, const void* lm_keys, const void* lm_vals, long long lm_capacity, int order, int bos,
                             int eos, int unk, int has_unk, float lm_weight, float word_score, float unk_score,
                             const uint32_t* trie_mask, const int* trie_first_child, const int* trie_word,
                             const float* trie_smear, long long trie_nodes, void* workspace, long long workspace_bytes,
                             int* tokens, int* lengths, float* scores, b200s_stream stream) {
  B200_CHECK_ARG(logits && lse && input_len && workspace && tokens && lengths && scores, "ctc_decode_lexicon: null pointer");
  B200_CHECK_ARG(B > 0 && T > 0, "ctc_decode_lexicon: need B > 0 and T > 0 (B=%d T=%d)", B, T);
  B200_CHECK_ARG(V >= 2 && V <= kMaxV, "ctc_decode_lexicon: V=%d outside [2, %d]", V, kMaxV);
  B200_CHECK_ARG(blank >= 0 && blank < V, "ctc_decode_lexicon: blank=%d outside [0, V=%d)", blank, V);
  B200_CHECK_ARG(beam >= 1 && beam <= kMaxBeam, "ctc_decode_lexicon: beam=%d outside [1, %d]", beam, kMaxBeam);
  B200_CHECK_ARG(nbest >= 1 && nbest <= beam, "ctc_decode_lexicon: nbest=%d outside [1, beam=%d]", nbest, beam);
  B200_CHECK_ARG(beam_token >= 1 && beam_token <= V - 1, "ctc_decode_lexicon: beam_token=%d outside [1, V-1=%d]", beam_token,
                 V - 1);
  B200_CHECK_ARG(word_boundary >= 0 && word_boundary < V && word_boundary != blank,
                 "ctc_decode_lexicon: word_boundary=%d must be a class in [0, V=%d) other than blank=%d", word_boundary, V, blank);
  B200_CHECK_ARG(trie_mask && trie_first_child && trie_word, "ctc_decode_lexicon: null trie array");
  B200_CHECK_ARG(trie_nodes >= 1 && trie_nodes <= B200S_CTC_TRIE_MAX_NODES, "ctc_decode_lexicon: %lld trie nodes outside [1, %d]",
                 trie_nodes, B200S_CTC_TRIE_MAX_NODES);
  Lm lm{};
  lm.weight = lm_weight;
  lm.word_score = word_score;
  lm.unk_score = unk_score;
  if (order > 0) {
    B200_CHECK_ARG(order <= B200S_CTC_LM_MAX_ORDER, "ctc_decode_lexicon: LM order %d outside [1, %d]", order,
                   B200S_CTC_LM_MAX_ORDER);
    B200_CHECK_ARG(lm_keys && lm_vals, "ctc_decode_lexicon: null LM table");
    B200_CHECK_ARG(lm_capacity > 0 && (lm_capacity & (lm_capacity - 1)) == 0,
                   "ctc_decode_lexicon: LM table capacity %lld must be a power of two", lm_capacity);
    lm.ng_keys = static_cast<const unsigned long long*>(lm_keys);
    lm.ng_vals = static_cast<const uint2*>(lm_vals);
    lm.ng_mask = static_cast<unsigned long long>(lm_capacity) - 1;
    lm.order = order;
    lm.bos = bos;
    lm.eos = eos;
    lm.unk = unk;
    lm.has_unk = has_unk ? 1 : 0;
  } else {
    B200_CHECK_ARG(order == 0, "ctc_decode_lexicon: LM order %d outside [1, %d]", order, B200S_CTC_LM_MAX_ORDER);
  }
  const long long need = b200s_ctc_decode_workspace_bytes(B, T, beam);
  B200_CHECK_ARG(workspace_bytes >= need, "ctc_decode_lexicon: workspace of %lld bytes, need %lld", workspace_bytes, need);
  const int W = (V + 31) / 32;
  const size_t smem = static_cast<size_t>(beam) * W * 10;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  B200_CHECK_CUDA(cudaFuncSetAttribute(ctc_decode_lexicon_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(kMaxBeam * kMaxW * 10)));
  auto* bp = static_cast<uint32_t*>(workspace);
  const Trie trie{trie_mask, trie_first_child, trie_word, trie_smear, W};
  B200_CHECK_CUDA(launch_pdl(ctc_decode_lexicon_kernel, dim3(B), dim3(kThreads), smem, st,
                             static_cast<const __nv_bfloat16*>(logits), frame_stride, batch_stride, lse, input_len, T, V, blank,
                             beam, nbest, beam_token, word_boundary, lm, trie, bp, lengths, scores));
  B200_CHECK_LAUNCH();
  B200_CHECK_CUDA(ctc_decode_backtrack_launch(input_len, B, T, beam, nbest, bp, tokens, lengths, st));
  B200_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"
