// CTC prefix beam search (Hannun et al. 2014) over the bf16 logits of the fine-tuning wrappers' `proj` head, with optional
// word-level n-gram LM scoring at word boundaries (lexicon-free: any spelling is a word; spellings the LM knows get their n-gram
// probability, the others score as <unk>).  The semantics are written down in include/unispeech_b200.h and restated in numpy by
// oracle/decode_oracle.py, which is their definition.
//
//   table build kernel  one thread per entry: hashes an int sequence (an n-gram's word ids, or a word's class-id spelling) with
//                       the same rolling hash the search uses, and inserts (key, two 32-bit values) into an open-addressing
//                       table by atomicCAS with linear probing.  A key that is already present is a 64-bit collision (the host
//                       rejects duplicate n-grams and spellings first) and is reported in *status, never resolved.
//   search kernel       one CTA per utterance, beams in shared memory double-buffered by frame.  Per frame: lp of the frame into
//                       shared memory; the top beam_token non-blank classes (membership) and the first M = min(beam_token,
//                       beam + 2) of them sorted, by a block radix select on (lp, -class); per beam the stay candidate (blank
//                       and repeat) with the extension of its parent that reaches the same prefix merged in (found by hash);
//                       the LM term of a boundary extension (spelling lookup, n-gram lookups with backoff); then a block radix
//                       select of the beam best of the candidates by (score desc, prefix hash asc) and a rank count among the
//                       selected.  Each new beam's (parent slot, appended class or -1) goes to the workspace.
//   backtrack kernel    one warp per (utterance, n-best entry): fetches the backpointers of 32 frames at a time into shared
//                       memory, lane 0 walks them, the lanes write the classes from the end of the row; the row is then moved
//                       to its front.
//
// Candidate pruning: an extension of parent j by the class at sorted position k >= M cannot reach the beam -- each of the first
// M positions holds a candidate at least as good (an extension, or the stay it was merged into), except the parent's last class
// (lower: its extension starts from pb) and the word boundary (its LM term can move it either way).  So each parent is extended
// by the first M sorted classes plus the boundary class when it is in the top beam_token; this equals the full candidate set
// except where exact score ties straddle the beam cutoff.
#include "ctc_decode_common.cuh"

namespace b200 {

namespace {

constexpr int kMaxCols = kMaxBeam + 3;           // per-parent extension columns: M <= beam + 2 sorted classes + the boundary
constexpr int kColWords = (kMaxCols + 31) / 32;
constexpr int kChunk = 32;                       // backtrack frames per fetch

// LM term of ending the partial word with spelling hash wh after context ctx[0..m); *wid = the word id it pushes.
__device__ float word_term(const Lm& lm, uint64_t wh, const int* ctx, int m, int* wid) {
  const int s = probe(lm.sp_keys, lm.sp_mask, wh);
  const bool oov = s < 0;
  *wid = oov ? lm.unk : static_cast<int>(lm.sp_vals[s].x);
  float t = 0.f;
  if (!oov || lm.has_unk) t = __fmul_rn(lm.weight, ln_prob(lm, ctx, m, *wid));
  t = __fadd_rn(t, lm.word_score);
  if (oov) t = __fadd_rn(t, lm.unk_score);
  return t;
}

struct Beams {
  unsigned long long h[kMaxBeam], ph[kMaxBeam], w[kMaxBeam];  // prefix, prefix without its last class, partial word
  float pb[kMaxBeam], pnb[kMaxBeam], lm[kMaxBeam];
  int last[kMaxBeam], nctx[kMaxBeam];
  int ctx[kCtx][kMaxBeam];
};

__global__ void __launch_bounds__(kThreads) ctc_decode_search_kernel(
    const __nv_bfloat16* __restrict__ x, long long fs, long long bs, const float* __restrict__ lse,
    const int* __restrict__ input_len, int T, int V, int blank, int beam, int nbest, int beam_token, int boundary, Lm lm,
    uint32_t* __restrict__ bp, int* __restrict__ lengths, float* __restrict__ scores) {
  __shared__ Beams bm[2];
  __shared__ float lps[kMaxV];
  __shared__ short tokpos[kMaxV];       // column of a class in this frame's sorted list, kMaxCols if it is not there
  __shared__ uint32_t inset[kMaxV / 32];  // top beam_token membership (used when beam_token < V - 1)
  __shared__ int sorted[kMaxCols];
  __shared__ float base[kMaxBeam], sscore[kMaxBeam], spb[kMaxBeam], spnb[kMaxBeam], bdelta[kMaxBeam];
  __shared__ int bwid[kMaxBeam];
  __shared__ uint32_t merged[kMaxBeam][kColWords];
  __shared__ Entry list[kMaxCols];
  __shared__ int nlist, bcol;
  __shared__ Select sel;
  pdl_grid_sync();
  const int b = blockIdx.x, tid = threadIdx.x;
  const int len = min(max(input_len[b], 0), T);
  const bool use_lm = lm.order > 0;
  const int K = beam_token, M = min(beam_token, beam + 2), ncol = M + 1;
  const bool all_in = K >= V - 1;
  const __nv_bfloat16* x_b = x + b * bs;
  const float* lse_b = lse + static_cast<long long>(b) * T;
  uint32_t* bp_b = bp + static_cast<long long>(b) * T * beam;
  if (tid == 0) {
    bm[0].h[0] = bm[0].ph[0] = bm[0].w[0] = 0ull;
    bm[0].pb[0] = 0.f;
    bm[0].pnb[0] = -INFINITY;
    bm[0].lm[0] = 0.f;
    bm[0].last[0] = -1;
    bm[0].nctx[0] = 0;
    if (use_lm && lm.order > 1) {
      bm[0].ctx[0][0] = lm.bos;
      bm[0].nctx[0] = 1;
    }
  }
  int nb = 1;
  auto in_top = [&](int c) { return c != blank && (all_in || ((inset[c >> 5] >> (c & 31)) & 1u)); };
  auto tok_key = [&](int c, bool, Key& k) {
    if (c == blank) return false;
    k = Key{ord(lps[c]), ~static_cast<uint64_t>(c)};
    return true;
  };
  for (int t = 0; t < len; ++t) {
    const Beams& cb = bm[t & 1];
    Beams& nx = bm[(t & 1) ^ 1];
    const float lse_t = lse_b[t];
    const __nv_bfloat16* row = x_b + t * fs;
    for (int c = tid; c < V; c += kThreads) {
      lps[c] = __bfloat162float(row[c]) - lse_t;
      tokpos[c] = kMaxCols;
    }
    for (int i = tid; i < kMaxBeam * kColWords; i += kThreads) (&merged[0][0])[i] = 0u;
    for (int i = tid; i < kMaxV / 32; i += kThreads) inset[i] = 0u;
    if (tid == 0) nlist = 0;
    __syncthreads();
    // ---- the frame's classes: top-K membership, the first M sorted
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
    select_top(V, M, tok_key, sel);
    {
      const Key p = sel.p;
      const int d = sel.d;
      for (int c = tid; c < V; c += kThreads) {
        Key k;
        if (tok_key(c, true, k) && top_ge(k, p, d)) {
          const int i = atomicAdd(&nlist, 1);
          if (i < M) list[i] = Entry{k, c};
        }
      }
    }
    __syncthreads();
    if (tid < M) {
      const Entry e = list[tid];
      int r = 0;
      for (int i = 0; i < M; ++i) r += better(list[i].k, e.k) ? 1 : 0;
      sorted[r] = e.q;
      tokpos[e.q] = static_cast<short>(r);
    }
    __syncthreads();
    if (tid == 0) {
      bcol = use_lm && in_top(boundary) && tokpos[boundary] == kMaxCols;
      if (bcol) tokpos[boundary] = static_cast<short>(M);
      nlist = 0;
    }
    __syncthreads();
    // ---- stays (blank, repeat) with the merged extension of their parent; the boundary LM term of every parent
    if (tid < nb) {
      const int i = tid, li = cb.last[i];
      const float a = lae(cb.pb[i], cb.pnb[i]);
      base[i] = a;
      spb[i] = a + lps[blank];
      float pnb = li >= 0 ? cb.pnb[i] + lps[li] : -INFINITY;
      if (li >= 0 && in_top(li)) {
        const unsigned long long ph = cb.ph[i];
        int j = -1;
        for (int u = 0; u < nb && j < 0; ++u)
          if (cb.h[u] == ph && u != i) j = u;
        if (j >= 0) {
          const float e = (li == cb.last[j] ? cb.pb[j] : lae(cb.pb[j], cb.pnb[j])) + lps[li];
          pnb = lae(pnb, e);
          const int col = tokpos[li];
          if (col < ncol) atomicOr(&merged[j][col >> 5], 1u << (col & 31));
        }
      }
      spnb[i] = pnb;
      sscore[i] = lae(spb[i], pnb) + cb.lm[i];
      float bd = 0.f;
      int wid = -1;
      if (use_lm && cb.w[i] != 0ull && in_top(boundary)) {
        int ctx[kCtx > 0 ? kCtx : 1];
#pragma unroll
        for (int u = 0; u < kCtx; ++u) ctx[u] = cb.ctx[u][i];
        bd = word_term(lm, cb.w[i], ctx, cb.nctx[i], &wid);
      }
      bdelta[i] = bd;
      bwid[i] = wid;
    }
    __syncthreads();
    // ---- candidates: q < nb the stay of beam q, else parent (q - nb) / ncol extended by column (q - nb) % ncol
    auto cand = [&](int q, bool with_hash, Key& k) {
      if (q < nb) {
        k = Key{ord(sscore[q]), with_hash ? ~static_cast<uint64_t>(cb.h[q]) : 0ull};
        return true;
      }
      const int e = q - nb, j = e / ncol, col = e - j * ncol;
      if (col == M && !bcol) return false;
      if ((merged[j][col >> 5] >> (col & 31)) & 1u) return false;
      const int c = col < M ? sorted[col] : boundary;
      const float ac = (c == cb.last[j] ? cb.pb[j] : base[j]) + lps[c];
      const float l = (use_lm && c == boundary) ? __fadd_rn(cb.lm[j], bdelta[j]) : cb.lm[j];
      k = Key{ord(ac + l), with_hash ? ~static_cast<uint64_t>(hash_step(cb.h[j], c)) : 0ull};
      return true;
    };
    const int n = nb + nb * ncol;
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
        nx.w[r] = cb.w[j];
        nx.pb[r] = spb[j];
        nx.pnb[r] = spnb[j];
        nx.lm[r] = cb.lm[j];
        nx.last[r] = cb.last[j];
        nx.nctx[r] = cb.nctx[j];
#pragma unroll
        for (int u = 0; u < kCtx; ++u) nx.ctx[u][r] = cb.ctx[u][j];
      } else {
        const int ee = q - nb, col = ee % ncol;
        j = ee / ncol;
        c = col < M ? sorted[col] : boundary;
        nx.h[r] = ~e.k.h;
        nx.ph[r] = cb.h[j];
        nx.pb[r] = -INFINITY;
        nx.pnb[r] = (c == cb.last[j] ? cb.pb[j] : base[j]) + lps[c];
        nx.last[r] = c;
        int ctx[kCtx > 0 ? kCtx : 1], m = cb.nctx[j];
#pragma unroll
        for (int u = 0; u < kCtx; ++u) ctx[u] = cb.ctx[u][j];
        float l = cb.lm[j];
        unsigned long long w = 0ull;
        if (use_lm && c == boundary) {
          if (cb.w[j] != 0ull) {
            l = __fadd_rn(l, bdelta[j]);
            push_word(ctx, m, bwid[j], lm.order);
          }
        } else {
          w = hash_step(cb.w[j], c);
        }
        nx.w[r] = w;
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
  // ---- end of utterance: the partial word and </s>, then the n-best by (score desc, hash asc)
  const Beams& fb = bm[len & 1];
  if (tid < nb) {
    float l = fb.lm[tid];
    if (use_lm) {
      int ctx[kCtx > 0 ? kCtx : 1], m = fb.nctx[tid];
#pragma unroll
      for (int u = 0; u < kCtx; ++u) ctx[u] = fb.ctx[u][tid];
      if (fb.w[tid] != 0ull) {
        int wid;
        l = __fadd_rn(l, word_term(lm, fb.w[tid], ctx, m, &wid));
        push_word(ctx, m, wid, lm.order);
      }
      l = __fadd_rn(l, __fmul_rn(lm.weight, ln_prob(lm, ctx, m, lm.eos)));
    }
    sscore[tid] = lae(fb.pb[tid], fb.pnb[tid]) + l;
  }
  __syncthreads();
  if (tid < nb) {
    const Key e{ord(sscore[tid]), ~static_cast<uint64_t>(fb.h[tid])};
    int r = 0;
    for (int i = 0; i < nb; ++i) r += better(Key{ord(sscore[i]), ~static_cast<uint64_t>(fb.h[i])}, e) ? 1 : 0;
    if (r < nbest) {
      scores[b * nbest + r] = sscore[tid];
      lengths[b * nbest + r] = tid;  // hand-off to the backtrack: the final slot
    }
  } else if (tid < nbest) {
    scores[b * nbest + tid] = -INFINITY;
    lengths[b * nbest + tid] = -1;
  }
}

// One warp per (utterance, n-best entry), launched after the search kernel on the same stream.
__global__ void __launch_bounds__(32) ctc_decode_backtrack_kernel(const int* __restrict__ input_len, int T, int beam, int nbest,
                                                                  const uint32_t* __restrict__ bp, int* __restrict__ tokens,
                                                                  int* __restrict__ lengths) {
  __shared__ uint32_t sw[kChunk][kMaxBeam];
  __shared__ int stok[kChunk];
  pdl_grid_sync();
  const int b = blockIdx.x, n = blockIdx.y, lane = threadIdx.x;
  const int len = min(max(input_len[b], 0), T);
  int* row = tokens + (static_cast<long long>(b) * nbest + n) * T;
  int slot = lengths[b * nbest + n];
  __syncwarp();
  const uint32_t* bp_b = bp + static_cast<long long>(b) * T * beam;
  int pos = T;  // tokens are written backwards from the end of the row
  if (slot >= 0) {
    for (int hi = len - 1; hi >= 0; hi -= kChunk) {
      for (int f = 0; f < kChunk && hi - f >= 0; ++f)
        for (int s = lane; s < beam; s += 32) sw[f][s] = bp_b[static_cast<long long>(hi - f) * beam + s];
      __syncwarp();
      if (lane == 0) {
        for (int f = 0; f < kChunk; ++f) {
          if (hi - f < 0) {
            stok[f] = -1;
            continue;
          }
          const uint32_t e = sw[f][slot];
          stok[f] = static_cast<int>(e >> 8) - 1;
          slot = static_cast<int>(e & 255u);
        }
      }
      __syncwarp();
      const int tk = stok[lane];
      const unsigned m = __ballot_sync(0xffffffffu, tk >= 0);
      if (tk >= 0) row[pos - 1 - __popc(m & ((1u << lane) - 1u))] = tk;
      pos -= __popc(m);
      __syncwarp();
    }
  }
  const int cnt = T - pos;
  for (int i0 = 0; i0 < cnt; i0 += 32) {  // move [pos, T) to [0, cnt): every source chunk is read before it can be overwritten
    const int i = i0 + lane;
    const int v = i < cnt ? row[pos + i] : 0;
    __syncwarp();
    if (i < cnt) row[i] = v;
    __syncwarp();
  }
  for (int i = cnt + lane; i < T; i += 32) row[i] = -1;
  if (lane == 0) lengths[b * nbest + n] = cnt;
}

__global__ void ctc_lm_table_build_kernel(const int* __restrict__ seqs, int n, int width, const uint32_t* __restrict__ v0,
                                          const uint32_t* __restrict__ v1, unsigned long long* __restrict__ keys,
                                          uint2* __restrict__ vals, long long capacity, int* __restrict__ status) {
  pdl_grid_sync();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t k = 0;
  for (int j = 0; j < width; ++j) {
    const int id = seqs[static_cast<long long>(i) * width + j];
    if (id < 0) break;
    k = hash_step(k, id);
  }
  if (k == 0) {  // 0 marks an empty slot
    atomicOr(status, 1);
    return;
  }
  const unsigned long long mask = static_cast<unsigned long long>(capacity) - 1;
  unsigned long long s = k & mask;
  for (long long p = 0; p < capacity; ++p, s = (s + 1) & mask) {
    const unsigned long long prev = atomicCAS(keys + s, 0ull, k);
    if (prev == 0ull) {
      vals[s] = make_uint2(v0[i], v1 ? v1[i] : 0u);
      return;
    }
    if (prev == k) {
      atomicOr(status, 1);
      return;
    }
  }
  atomicOr(status, 2);
}

}  // namespace

cudaError_t ctc_decode_backtrack_launch(const int* input_len, int B, int T, int beam, int nbest, const uint32_t* bp,
                                        int* tokens, int* lengths, cudaStream_t st) {
  return launch_pdl(ctc_decode_backtrack_kernel, dim3(B, nbest), dim3(32), 0, st, input_len, T, beam, nbest, bp, tokens, lengths);
}

}  // namespace b200

using namespace b200;

extern "C" {

long long b200s_ctc_decode_workspace_bytes(int B, int T, int beam) {
  if (B < 1 || T < 1 || beam < 1 || beam > kMaxBeam) return -1;
  return static_cast<long long>(B) * T * beam * 4;
}

int b200s_ctc_lm_table_build(const int* seqs, int n, int width, const uint32_t* v0, const uint32_t* v1, void* keys, void* vals,
                             long long capacity, int* status, b200s_stream stream) {
  B200_CHECK_ARG(seqs && v0 && keys && vals && status, "ctc_lm_table_build: null pointer");
  B200_CHECK_ARG(n >= 1 && width >= 1, "ctc_lm_table_build: need n >= 1 and width >= 1 (n=%d width=%d)", n, width);
  B200_CHECK_ARG(capacity > n && (capacity & (capacity - 1)) == 0,
                 "ctc_lm_table_build: capacity %lld must be a power of two above n=%d", capacity, n);
  B200_CHECK_CUDA(launch_pdl(ctc_lm_table_build_kernel, dim3(ceil_div(n, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream),
                             seqs, n, width, v0, v1, static_cast<unsigned long long*>(keys), static_cast<uint2*>(vals), capacity,
                             status));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_ctc_decode(const void* logits, long long frame_stride, long long batch_stride, const float* lse, const int* input_len,
                     int B, int T, int V, int blank, int beam, int nbest, int beam_token, int word_boundary, const void* lm_keys,
                     const void* lm_vals, long long lm_capacity, const void* spell_keys, const void* spell_vals,
                     long long spell_capacity, int order, int bos, int eos, int unk, int has_unk, float lm_weight, float word_score,
                     float unk_score, void* workspace, long long workspace_bytes, int* tokens, int* lengths, float* scores,
                     b200s_stream stream) {
  B200_CHECK_ARG(logits && lse && input_len && workspace && tokens && lengths && scores, "ctc_decode: null pointer");
  B200_CHECK_ARG(B > 0 && T > 0, "ctc_decode: need B > 0 and T > 0 (B=%d T=%d)", B, T);
  B200_CHECK_ARG(V >= 2 && V <= kMaxV, "ctc_decode: V=%d outside [2, %d]", V, kMaxV);
  B200_CHECK_ARG(blank >= 0 && blank < V, "ctc_decode: blank=%d outside [0, V=%d)", blank, V);
  B200_CHECK_ARG(beam >= 1 && beam <= kMaxBeam, "ctc_decode: beam=%d outside [1, %d]", beam, kMaxBeam);
  B200_CHECK_ARG(nbest >= 1 && nbest <= beam, "ctc_decode: nbest=%d outside [1, beam=%d]", nbest, beam);
  B200_CHECK_ARG(beam_token >= 1 && beam_token <= V - 1, "ctc_decode: beam_token=%d outside [1, V-1=%d]", beam_token, V - 1);
  Lm lm{};
  if (order > 0) {
    B200_CHECK_ARG(order <= B200S_CTC_LM_MAX_ORDER, "ctc_decode: LM order %d outside [1, %d]", order, B200S_CTC_LM_MAX_ORDER);
    B200_CHECK_ARG(lm_keys && lm_vals && spell_keys && spell_vals, "ctc_decode: null LM table");
    B200_CHECK_ARG(lm_capacity > 0 && (lm_capacity & (lm_capacity - 1)) == 0 && spell_capacity > 0 &&
                       (spell_capacity & (spell_capacity - 1)) == 0,
                   "ctc_decode: LM table capacities must be powers of two (%lld, %lld)", lm_capacity, spell_capacity);
    B200_CHECK_ARG(word_boundary >= 0 && word_boundary < V && word_boundary != blank,
                   "ctc_decode: word_boundary=%d must be a class in [0, V=%d) other than blank=%d", word_boundary, V, blank);
    lm = Lm{static_cast<const unsigned long long*>(lm_keys), static_cast<const uint2*>(lm_vals),
            static_cast<unsigned long long>(lm_capacity) - 1, static_cast<const unsigned long long*>(spell_keys),
            static_cast<const uint2*>(spell_vals), static_cast<unsigned long long>(spell_capacity) - 1, order, bos, eos, unk,
            has_unk ? 1 : 0, lm_weight, word_score, unk_score};
  } else {
    B200_CHECK_ARG(order == 0, "ctc_decode: LM order %d outside [1, %d]", order, B200S_CTC_LM_MAX_ORDER);
  }
  const long long need = b200s_ctc_decode_workspace_bytes(B, T, beam);
  B200_CHECK_ARG(workspace_bytes >= need, "ctc_decode: workspace of %lld bytes, need %lld", workspace_bytes, need);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  auto* bp = static_cast<uint32_t*>(workspace);
  B200_CHECK_CUDA(launch_pdl(ctc_decode_search_kernel, dim3(B), dim3(kThreads), 0, st, static_cast<const __nv_bfloat16*>(logits),
                             frame_stride, batch_stride, lse, input_len, T, V, blank, beam, nbest, beam_token,
                             order > 0 ? word_boundary : -1, lm, bp, lengths, scores));
  B200_CHECK_LAUNCH();
  B200_CHECK_CUDA(launch_pdl(ctc_decode_backtrack_kernel, dim3(B, nbest), dim3(32), 0, st, input_len, T, beam, nbest,
                             static_cast<const uint32_t*>(bp), tokens, lengths));
  B200_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"
