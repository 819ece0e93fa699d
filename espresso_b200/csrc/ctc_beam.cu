// espresso_b200 -- CTC prefix beam search (frame-synchronous, fp32 log space) with optional LSTM-LM or n-gram LM
// shallow fusion.
//
// Replaces the decoding half of espresso/tools/ctc_decoder.py:18-188 (beam_size, lm_weight, word_score; the reference
// reaches it through flashlight's LexiconFreeDecoder + KenLM).  Three kernels:
//   frames   : one pass over every (b, t) logit row: fp32 log-normaliser, lp[blank] and the top-K allowed tokens
//              (blank / pad / eos / unk excluded) ranked by (logit desc, token id asc).  The logits are read once.
//   search   : one CTA per sentence over frames [t0, t1): stay / extend / merge / prune / select in shared memory.
//              Without an LM one launch covers every frame; with an LM the host launches it once per frame and
//              advances the LM rows in between (new_order / grown / fed).
//   finalize : + lm_weight * log P_LM(eos | y), sort, backtrack the parent table into padded outputs.
// The search and finalize kernels are instantiated per LM mode (kRows: LSTM-LM rows or none; kNgram: an ARPA n-gram
// scored inside the kernel, lexicon-free; kLexicon: the n-gram through a lexicon trie); the modes share the stay /
// extend / merge / prune / select code.  With an n-gram one search launch covers every frame, as without an LM.
//
// Search semantics (oracle/ctc_beam.py states the same in float64):
//   state per slot: prefix y, pb / pnb (log-prob of ending in blank / non-blank), lm (accumulated lm_weight *
//   log P_LM + word_score per token); score = logaddexp(pb, pnb) + lm.  Start: one empty prefix, pb = 0.
//   stay      pb' = lae(pb, pnb) + lp[blank];  pnb' = pnb + lp[last(y)] (y non-empty)
//   extend v  ext = (v == last(y) ? pb : lae(pb, pnb)) + lp[v]; y+v gets pnb = ext, pb = -inf,
//             lm += lm_weight * log P_LM(v | y) + word_score
//   merge     y+v already live as h'  ->  pnb'(h') = lae(pnb'(h'), ext), the candidate is dropped.  Prefixes are
//             identified by a 64-bit rolling hash + length + last token (no token strings on the device).
//   prune     candidates below best - beam_threshold are dropped; the best `beam` remain, ordered by (score desc,
//             candidate index asc), candidate index = h * (K + 1) + j (j = 0 stay, j = 1..K extensions in rank order).
//             New slot k holds the k-th candidate; slots without a candidate are dead (score -inf).
//
// n-gram modes (include/espresso_b200.h: EspNgram, EspLexicon; oracle/ngram.py states them in float64).  LM scores
// are log10 (KenLM's unit, which flashlight's KenLM wrapper passes on unscaled -- that comes from flashlight's source,
// not in the reference tree), the acoustic term stays in natural log.  Each slot also holds an n-gram state.
//   kNgram    extend v: lm += lm_weight * log10 P(v | y) + word_score; finalize: + lm_weight * log10 P(</s> | y).
//   kLexicon  a slot also holds a trie node and a look-ahead term; score = lae(pb, pnb) + lm + lookahead.  Extending a
//             slot at node n with token v needs a child c of n labelled v (no out-of-lexicon path: unk_weight = -inf).
//             Per (slot, token rank) the candidates are: the in-word continuation when c has children (lookahead =
//             lm_weight * smear(c)), then each word w ending at c by ascending word id (back to the root, lm +=
//             lm_weight * log10 P(w | words) + word_score, lookahead = 0).  Candidate index = h * (1 + K * W1) + j,
//             j = 0 stay, j = 1 + rank * W1 + q (W1 = 1 + max words at one node, q = 0 in-word, q >= 1 words).
//             A hypothesis is its tokens and its word segmentation: a completed word folds a marker into the prefix
//             hash, and merging also compares the trie node.  Finalize keeps root slots only, + lm_weight *
//             log10 P(</s> | words).
//             Deliberate differences from flashlight's LexiconDecoder: prefix-identical candidates are log-added (as
//             above) where flashlight keeps the max (log_add = false); smear(root) = 0, so a word's net LM term is
//             exactly lm_weight * log10 P(w | h) (a constant per-word offset in flashlight's smearing acts as a shift of
//             word_score); the reference's silence (sil_weight = 0) never enters, as the search never proposes eos.
#include "common.cuh"
#include "espresso_b200.h"
#include <math.h>

namespace {

constexpr float kNegInf = -INFINITY;
constexpr int kT = 256;            // threads per CTA, all three kernels
constexpr int kMaxBeam = 128;      // beam_size and beam_size_token limit
constexpr int kMaxV = 65535;       // token ids fit the 16-bit tie-break field of the frame keys
constexpr int kHashSlots = 256;    // open-addressing table over the live prefixes (load <= 1/2)
enum LmMode { kRows = 0, kNgram = 1, kLexicon = 2 };

__device__ __forceinline__ float lae(float a, float b) {
  const float m = fmaxf(a, b);
  if (m == kNegInf) return kNegInf;
  return m + log1pf(expf(-fabsf(a - b)));
}

// order-preserving float -> uint32 (larger float => larger key); -0 is folded into +0 by the caller
__device__ __forceinline__ uint32_t fkey(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ uint32_t bkey(uint16_t b) {
  if (b == 0x8000u) b = 0;  // -0 ties with +0
  return (b & 0x8000u) ? (uint32_t)(~b & 0xFFFFu) : (uint32_t)(b | 0x8000u);
}

// ---- n-gram probe (include/espresso_b200.h: EspNgram) -------------------------------------------------------------
__device__ __forceinline__ int ng_order_of(const EspNgram& g, int e) {
  int o = 1;
  while (o < g.order && e >= g.order_off[o]) ++o;
  return o;
}
// log10 P(w | state s); *next = the state after w
__device__ __forceinline__ float ngram_probe(const EspNgram& g, int s, int w, int* next) {
  float acc = 0.f;
  while (s >= 0) {
    const int hi = g.child_hi[s];
    int lo = g.child_lo[s], h2 = hi;
    while (lo < h2) {
      const int mid = (lo + h2) >> 1;
      if (g.word[mid] < w) lo = mid + 1; else h2 = mid;
    }
    if (lo < hi && g.word[lo] == w) {
      *next = ng_order_of(g, lo) < g.order ? lo : g.suffix[lo];
      return acc + g.prob[lo];
    }
    acc += g.backoff[s];
    s = g.suffix[s];
  }
  *next = g.order > 1 ? w : -1;
  return acc + g.prob[w];
}
// child of trie node n labelled v, or -1
__device__ __forceinline__ int trie_child(const EspLexicon& x, int n, int v) {
  int lo = x.child_off[n], hi = x.child_off[n + 1];
  const int end = hi;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (x.child_tok[mid] < v) lo = mid + 1; else hi = mid;
  }
  return (lo < end && x.child_tok[lo] == v) ? x.child_node[lo] : -1;
}

__global__ void __launch_bounds__(kT)
ngram_score_kernel(const __grid_constant__ EspNgram g, int n, const int* __restrict__ states, const int* __restrict__ words,
                   float* __restrict__ out_logp, int* __restrict__ out_next) {
  esp_pdl();
  for (int i = blockIdx.x * kT + threadIdx.x; i < n; i += gridDim.x * kT) {
    int nx;
    out_logp[i] = ngram_probe(g, states[i], words[i], &nx);
    out_next[i] = nx;
  }
}

// ---- block helpers (blockDim.x == kT) ------------------------------------------------------------------------
__device__ __forceinline__ int blk_isum(int c, int* ired) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) ired[threadIdx.x >> 5] = c;
  __syncthreads();
  int r = 0;
#pragma unroll
  for (int w = 0; w < kT / 32; ++w) r += ired[w];
  __syncthreads();
  return r;
}

// k-th largest key (1-based) among the items i < n for which key_of(i, &key) is true: returns tau with
// count(key > tau) < k <= count(key >= tau).  MSB-first radix select, 4 passes of 8 bits; k must be in [1, count].
struct RadixScratch {
  uint32_t hist[256];
  uint32_t wsum[kT / 32];
  uint32_t prefix, k;
};
template <class F>
__device__ __forceinline__ uint32_t radix_kth(int n, uint32_t k, F key_of, RadixScratch& rs) {
  uint32_t prefix = 0, mask = 0;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
#pragma unroll 1
  for (int shift = 24; shift >= 0; shift -= 8) {
    rs.hist[tid] = 0;
    __syncthreads();
    for (int i = tid; i < n; i += kT) {
      uint32_t key;
      if (key_of(i, key) && (key & mask) == prefix) atomicAdd(&rs.hist[(key >> shift) & 255u], 1u);
    }
    __syncthreads();
    // descending digits: thread j owns digit 255 - j; inclusive prefix sum over threads
    const uint32_t c = rs.hist[255 - tid];
    uint32_t incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += y;
    }
    if (lane == 31) rs.wsum[warp] = incl;
    __syncthreads();
    for (int w = 0; w < warp; ++w) incl += rs.wsum[w];
    if (incl >= k && incl - c < k) {  // exactly one thread
      rs.prefix = prefix | ((uint32_t)(255 - tid) << shift);
      rs.k = k - (incl - c);
    }
    __syncthreads();
    prefix = rs.prefix;
    k = rs.k;
    mask |= 0xFFu << shift;
    __syncthreads();
  }
  return prefix;
}

// ---- frames ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kT)
ctc_beam_frames_kernel(const bf16* __restrict__ logits, long stride_b, long stride_t, int V, int t_max,
                       const int* __restrict__ in_lens, int K, int blank, int pad, int eos, int unk,
                       float* __restrict__ lse_out, float* __restrict__ lpb_out, int* __restrict__ tok_out,
                       float* __restrict__ lp_out) {
  esp_pdl();
  extern __shared__ __align__(16) uint16_t row_sh[];  // the row's raw bf16 bits
  __shared__ float red[32];
  __shared__ int ired[32];
  __shared__ RadixScratch rs;
  __shared__ uint32_t sel[kMaxBeam];
  __shared__ int nsel;
  const int b = blockIdx.y, t = blockIdx.x;
  if (t >= in_lens[b]) return;
  const bf16* row = logits + (long)b * stride_b + (long)t * stride_t;
  const uint16_t* rowu = reinterpret_cast<const uint16_t*>(row);
  float mx = kNegInf;
  const int nvec = ((reinterpret_cast<uintptr_t>(row) & 15) == 0) ? V / 8 : 0;
  for (int vi = threadIdx.x; vi < nvec; vi += kT) {
    const uint4 q = __ldg(reinterpret_cast<const uint4*>(row) + vi);
    *reinterpret_cast<uint4*>(row_sh + vi * 8) = q;
    float a, c;
    unpack_bf16x2(q.x, a, c); mx = fmaxf(mx, fmaxf(a, c));
    unpack_bf16x2(q.y, a, c); mx = fmaxf(mx, fmaxf(a, c));
    unpack_bf16x2(q.z, a, c); mx = fmaxf(mx, fmaxf(a, c));
    unpack_bf16x2(q.w, a, c); mx = fmaxf(mx, fmaxf(a, c));
  }
  for (int v = nvec * 8 + threadIdx.x; v < V; v += kT) {
    const uint16_t u = rowu[v];
    row_sh[v] = u;
    mx = fmaxf(mx, __uint_as_float((uint32_t)u << 16));
  }
  mx = block_max<kT>(mx, red);  // its barriers also publish row_sh
  float s = 0.f;
  if (mx != kNegInf)
    for (int v = threadIdx.x; v < V; v += kT) s += expf(__uint_as_float((uint32_t)row_sh[v] << 16) - mx);
  s = block_sum<kT>(s, red);
  const float lse = mx + logf(s);
  const long r = (long)b * t_max + t;
  if (threadIdx.x == 0) {
    lse_out[r] = lse;
    lpb_out[r] = __uint_as_float((uint32_t)row_sh[blank] << 16) - lse;
    nsel = 0;
  }
  // key = (ordered logit << 16) | (0xFFFF - v): unique, larger = better; excluded tokens have key 0
  auto key_of = [=](int v, uint32_t& key) {
    key = (v == blank || v == pad || v == eos || v == unk) ? 0u : ((bkey(row_sh[v]) << 16) | (uint32_t)(0xFFFF - v));
    return key != 0u;
  };
  int n_ok = 0;
  for (int v = threadIdx.x; v < V; v += kT) { uint32_t k; n_ok += key_of(v, k); }
  n_ok = blk_isum(n_ok, ired);
  const int keff = K < n_ok ? K : n_ok;
  if (keff > 0) {
    const uint32_t tau = radix_kth(V, (uint32_t)keff, key_of, rs);
    for (int v = threadIdx.x; v < V; v += kT) {
      uint32_t k;
      if (key_of(v, k) && k >= tau) sel[atomicAdd(&nsel, 1)] = k;
    }
    __syncthreads();
  }
  for (int i = threadIdx.x; i < K; i += kT) {
    int tok = -1;
    float lp = kNegInf;
    if (i < keff) {
      const uint32_t k = sel[i];
      int rank = 0;
      for (int j = 0; j < keff; ++j) rank += sel[j] > k;
      tok = 0xFFFF - (int)(k & 0xFFFFu);
      lp = __uint_as_float((uint32_t)row_sh[tok] << 16) - lse;
      tok_out[r * K + rank] = tok;
      lp_out[r * K + rank] = lp;
    } else {
      tok_out[r * K + i] = tok;
      lp_out[r * K + i] = lp;
    }
  }
}

// ---- search ---------------------------------------------------------------------------------------------------
struct SearchArgs {
  const bf16* logits;
  long stride_b, stride_t;
  int V, t_max;
  const int* in_lens;
  const float* lse;
  const float* lpb;
  const int* top_tok;
  const float* top_lp;
  int K, beam;
  float threshold;
  int t0, t1;
  const void* lm;
  int lm_f32;
  long ld_lm;
  int lm_blank;  // >= 0: the LM vocabulary lacks the blank at this index (LM column = v - (v > lm_blank))
  float lm_weight, word_score;
  int eos;
  int* new_order;
  int* grown;
  int* fed;
  // workspace
  float* pb;
  float* pnb;
  float* lmacc;
  int* last;
  int* len;
  unsigned long long* hash;
  int* par;    // [t_max, B * beam] source slot
  int* ptok;   // [t_max, B * beam] token appended at t, -1 for a stay
  // n-gram modes
  EspNgram ng;
  EspLexicon lex;
  const int* tok_word;  // kNgram: CTC token -> n-gram word id
  int W1;               // candidates per (slot, token rank): 1 + max words ending at one trie node (1 without a lexicon)
  int* node;
  int* lmst;
  float* la;
};

__device__ __forceinline__ int lm_col(int v, int lm_blank) { return (lm_blank >= 0 && v > lm_blank) ? v - 1 : v; }
__device__ __forceinline__ float lm_val(const void* lm, int f32, long off) {
  return f32 ? ((const float*)lm)[off] : bf2f(((const bf16*)lm)[off]);
}

// log-sum-exp of the LM row of every live slot, one warp per row
__device__ __forceinline__ void lm_row_lse(const SearchArgs& a, long rb, const float* sc, float* lse_lm, int Vlm) {
  const int lane = threadIdx.x & 31;
  for (int h = threadIdx.x >> 5; h < a.beam; h += kT / 32) {
    if (sc[h] == kNegInf) { if (lane == 0) lse_lm[h] = 0.f; continue; }
    const long off = (rb + h) * a.ld_lm;
    float m = kNegInf, s = 0.f;
    for (int v = lane; v < Vlm; v += 32) {
      const float x = lm_val(a.lm, a.lm_f32, off + v);
      if (x == kNegInf) continue;
      if (x > m) { s = s * expf(m - x) + 1.f; m = x; } else { s += expf(x - m); }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, m, o), os = __shfl_xor_sync(0xffffffffu, s, o);
      const float nm = fmaxf(m, om);
      s = (nm == kNegInf) ? 0.f : s * expf(m - nm) + os * expf(om - nm);
      m = nm;
    }
    if (lane == 0) lse_lm[h] = m + logf(s);
  }
}

struct SearchSmem {
  float pb[kMaxBeam], pnb[kMaxBeam], lm[kMaxBeam], sc[kMaxBeam], lse_lm[kMaxBeam];
  float spb[kMaxBeam], spnb[kMaxBeam], merge_in[kMaxBeam];
  float npb[kMaxBeam], npnb[kMaxBeam], nlm[kMaxBeam];
  unsigned long long hash[kMaxBeam], nhash[kMaxBeam];
  int last[kMaxBeam], len[kMaxBeam], nlast[kMaxBeam], nlen[kMaxBeam];
  int sel[kMaxBeam], slot_c[kMaxBeam];
  int node[kMaxBeam], st[kMaxBeam], nnode[kMaxBeam], nst[kMaxBeam];
  float la[kMaxBeam], nla[kMaxBeam];
  int ttok[kMaxBeam];
  float tlp[kMaxBeam];
  int tab[kHashSlots];
  RadixScratch rs;
  float red[32];
  int ired[32];
  int nsel;
  float lpb;
};

__device__ __forceinline__ float ext_lp(const SearchSmem& S, int h, int v, float lpv) {
  return ((S.len[h] > 0 && v == S.last[h]) ? S.pb[h] : lae(S.pb[h], S.pnb[h])) + lpv;
}
__device__ __forceinline__ float ext_lm(const SearchArgs& a, const SearchSmem& S, long rb, int h, int v) {
  float l = S.lm[h] + a.word_score;
  if (a.lm) l += a.lm_weight * (lm_val(a.lm, a.lm_f32, (rb + h) * a.ld_lm + lm_col(v, a.lm_blank)) - S.lse_lm[h]);
  return l;
}

// an n-gram-mode extension of slot h by token v: its lm, lookahead, trie node, n-gram state and prefix hash
struct Ext {
  float lm, la;
  int node, st;
  unsigned long long hash;
};
__device__ __forceinline__ void ngram_ext(const SearchArgs& a, const SearchSmem& S, int h, int v, Ext& o) {
  o.hash = esp_hash_u64(S.hash[h], (unsigned long long)v);
  const float lp = ngram_probe(a.ng, S.st[h], a.tok_word[v], &o.st);
  o.lm = (S.lm[h] + a.word_score) + a.lm_weight * lp;
  o.la = 0.f;
  o.node = 0;
}
// through the lexicon: candidate q of the move to trie child c (q = 0 in-word, q >= 1 the (q-1)-th word ending at c);
// false when there is no such candidate
__device__ __forceinline__ bool lex_ext(const SearchArgs& a, const SearchSmem& S, int h, int v, int c, int q, Ext& o) {
  o.hash = esp_hash_u64(S.hash[h], (unsigned long long)v);
  if (q == 0) {  // inside the word
    if (a.lex.child_off[c + 1] == a.lex.child_off[c]) return false;
    o.lm = S.lm[h];
    o.la = a.lm_weight * a.lex.smear[c];
    o.node = c;
    o.st = S.st[h];
    return true;
  }
  const int wi = a.lex.word_off[c] + q - 1;
  if (wi >= a.lex.word_off[c + 1]) return false;
  const int w = a.lex.words[wi];
  const float lp = ngram_probe(a.ng, S.st[h], a.lex.word_lm[w], &o.st);
  o.lm = (S.lm[h] + a.word_score) + a.lm_weight * lp;
  o.la = 0.f;
  o.node = 0;
  o.hash = esp_hash_u64(o.hash, (1ull << 32) | (unsigned long long)w);  // the word boundary is part of the identity
  return true;
}

// merge target of an extension: the live slot with the same prefix hash, last token, length and trie node, or -1
__device__ __forceinline__ int find_live(const SearchSmem& S, const Ext& o, int v, int len) {
  for (int p = (int)(o.hash & (kHashSlots - 1));; p = (p + 1) & (kHashSlots - 1)) {
    const int x = S.tab[p];
    if (x < 0) return -1;
    if (S.hash[x] == o.hash && S.last[x] == v && S.len[x] == len && S.node[x] == o.node) return x;
  }
}

template <int MODE>
__global__ void __launch_bounds__(kT, 1)
ctc_beam_search_kernel(SearchArgs a, int Vlm) {
  esp_pdl();
  extern __shared__ float cs[];  // candidate scores [beam * (1 + K * W1)]
  __shared__ SearchSmem S;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int beam = a.beam, K = a.K, W1 = MODE == kLexicon ? a.W1 : 1;
  const int K1 = 1 + a.K * W1, n = a.beam * K1;
  const int n_items = a.beam * (a.K + 1);  // (slot, j): j = 0 stay, j >= 1 the token of rank j - 1
  const long rb = (long)b * beam;
  const int T = a.in_lens[b];
  if (tid < beam) {
    if (a.t0 == 0) {  // one empty prefix, every other slot dead
      S.pb[tid] = tid == 0 ? 0.f : kNegInf;
      S.pnb[tid] = kNegInf;
      S.lm[tid] = 0.f;
      S.last[tid] = -1;
      S.len[tid] = 0;
      S.hash[tid] = 0ull;
      if constexpr (MODE != kRows) {
        S.node[tid] = 0;
        S.st[tid] = a.ng.start;
        S.la[tid] = 0.f;
      }
    } else {
      S.pb[tid] = a.pb[rb + tid];
      S.pnb[tid] = a.pnb[rb + tid];
      S.lm[tid] = a.lmacc[rb + tid];
      S.last[tid] = a.last[rb + tid];
      S.len[tid] = a.len[rb + tid];
      S.hash[tid] = a.hash[rb + tid];
      if constexpr (MODE != kRows) {
        S.node[tid] = a.node[rb + tid];
        S.st[tid] = a.lmst[rb + tid];
        S.la[tid] = a.la[rb + tid];
      }
    }
    if (a.new_order) {  // frames past the sentence's end leave every row where it is
      a.new_order[rb + tid] = (int)(rb + tid);
      a.grown[rb + tid] = 0;
      a.fed[rb + tid] = lm_col(a.eos, a.lm_blank);
    }
  }
  __syncthreads();
  const int tend = a.t1 < T ? a.t1 : T;
#pragma unroll 1
  for (int t = a.t0; t < tend; ++t) {
    const long fr = (long)b * a.t_max + t;
    const float lse_t = a.lse[fr];
    const bf16* row = a.logits + (long)b * a.stride_b + (long)t * a.stride_t;
    for (int i = tid; i < K; i += kT) {
      S.ttok[i] = a.top_tok[fr * K + i];
      S.tlp[i] = a.top_lp[fr * K + i];
    }
    for (int i = tid; i < kHashSlots; i += kT) S.tab[i] = -1;
    if (tid < beam) {
      S.sc[tid] = lae(S.pb[tid], S.pnb[tid]) + S.lm[tid];
      if constexpr (MODE == kLexicon) S.sc[tid] += S.la[tid];
      S.merge_in[tid] = kNegInf;
    }
    if (tid == 0) S.lpb = a.lpb[fr];
    __syncthreads();
    if (tid < beam && S.sc[tid] != kNegInf) {  // index the live prefixes by hash
      int p = (int)(S.hash[tid] & (kHashSlots - 1));
      while (atomicCAS(&S.tab[p], -1, tid) != -1) p = (p + 1) & (kHashSlots - 1);
    }
    if (MODE == kRows && a.lm) lm_row_lse(a, rb, S.sc, S.lse_lm, Vlm);
    __syncthreads();
    // 1. stays (j = 0) and extensions (j >= 1); an extension that re-creates a live prefix merges into its stay
    for (int c = tid; c < n_items; c += kT) {
      const int h = c / (K + 1), j = c - h * (K + 1);
      if constexpr (MODE == kLexicon) {  // one item writes the W1 candidates of its (slot, token rank)
        const bool live_h = S.sc[h] != kNegInf;
        if (j == 0) {
          if (live_h) {
            S.spb[h] = lae(S.pb[h], S.pnb[h]) + S.lpb;
            S.spnb[h] = S.len[h] > 0 ? S.pnb[h] + (bf2f(row[S.last[h]]) - lse_t) : kNegInf;
          }
          continue;
        }
        const int r = j - 1, v = S.ttok[r];
        const int ch = (live_h && v >= 0) ? trie_child(a.lex, S.node[h], v) : -1;
        const float e = ch >= 0 ? ext_lp(S, h, v, S.tlp[r]) : kNegInf;
        float* out = cs + h * K1 + 1 + r * W1;
        for (int q = 0; q < W1; ++q) {
          float score = kNegInf;
          Ext o;
          if (ch >= 0 && lex_ext(a, S, h, v, ch, q, o)) {
            const int hit = find_live(S, o, v, S.len[h] + 1);
            if (hit >= 0) S.merge_in[hit] = e;  // one parent (prefix and segmentation), so one writer
            else
              score = (e + o.lm) + o.la;
          }
          out[q] = score + 0.f;
        }
        continue;
      }
      float score = kNegInf;
      if (S.sc[h] != kNegInf) {
        if (j == 0) {
          S.spb[h] = lae(S.pb[h], S.pnb[h]) + S.lpb;
          S.spnb[h] = S.len[h] > 0 ? S.pnb[h] + (bf2f(row[S.last[h]]) - lse_t) : kNegInf;
        } else if constexpr (MODE == kNgram) {
          const int v = S.ttok[j - 1];
          if (v >= 0) {
            Ext o;
            ngram_ext(a, S, h, v, o);
            const float e = ext_lp(S, h, v, S.tlp[j - 1]);
            const int hit = find_live(S, o, v, S.len[h] + 1);
            if (hit >= 0) S.merge_in[hit] = e;  // y+v has exactly one parent prefix y, so one writer
            else
              score = e + o.lm;
          }
        } else {
          const int v = S.ttok[j - 1];
          if (v >= 0) {
            const float e = ext_lp(S, h, v, S.tlp[j - 1]);
            const unsigned long long hv = esp_hash_u64(S.hash[h], (unsigned long long)v);
            int hit = -1;
            for (int p = (int)(hv & (kHashSlots - 1));; p = (p + 1) & (kHashSlots - 1)) {
              const int q = S.tab[p];
              if (q < 0) break;
              if (S.hash[q] == hv && S.last[q] == v && S.len[q] == S.len[h] + 1) { hit = q; break; }
            }
            if (hit >= 0) S.merge_in[hit] = e;  // y+v has exactly one parent prefix y, so one writer
            else
              score = e + ext_lm(a, S, rb, h, v);
          }
        }
      }
      if (j != 0) cs[c] = score + 0.f;  // + 0 folds -0 into +0 for the ordered keys
    }
    __syncthreads();
    if (tid < beam) {
      float sc = kNegInf;
      if (S.sc[tid] != kNegInf) {
        S.spnb[tid] = lae(S.spnb[tid], S.merge_in[tid]);
        sc = lae(S.spb[tid], S.spnb[tid]) + S.lm[tid];
        if constexpr (MODE == kLexicon) sc += S.la[tid];
      }
      cs[tid * K1] = sc + 0.f;
    }
    __syncthreads();
    // 2. prune: threshold, then the best `beam` by (score desc, index asc)
    float best = kNegInf;
    #pragma unroll 1
    for (int c = tid; c < n; c += kT) best = fmaxf(best, cs[c]);
    best = block_max<kT>(best, S.red);
    const float floor_ = best - a.threshold;
    int live = 0;
    #pragma unroll 1
    for (int c = tid; c < n; c += kT) {
      float v = cs[c];
      if (v != v || v < floor_) { v = kNegInf; cs[c] = v; }
      live += v != kNegInf;
    }
    live = blk_isum(live, S.ired);
    const int kk = live < beam ? live : beam;
    if (tid == 0) S.nsel = 0;
    if (kk > 0) {
      const uint32_t tau = radix_kth(n, (uint32_t)kk, [=](int c, uint32_t& key) {
        key = fkey(cs[c]);
        return cs[c] != kNegInf;
      }, S.rs);
      int m = 0;
      #pragma unroll 1
      for (int c = tid; c < n; c += kT) m += cs[c] != kNegInf && fkey(cs[c]) > tau;
      const int n_gt = blk_isum(m, S.ired);
      const int need = kk - n_gt;  // >= 1: ties at tau are taken by ascending candidate index
      const uint32_t inv = radix_kth(n, (uint32_t)need, [=](int c, uint32_t& key) {
        key = ~(uint32_t)c;
        return cs[c] != kNegInf && fkey(cs[c]) == tau;
      }, S.rs);
      const int cmax = (int)~inv;
      #pragma unroll 1
      for (int c = tid; c < n; c += kT) {
        const float v = cs[c];
        if (v == kNegInf) continue;
        const uint32_t k = fkey(v);
        if (k > tau || (k == tau && c <= cmax)) S.sel[atomicAdd(&S.nsel, 1)] = c;
      }
      __syncthreads();
      if (tid < kk) {
        const int c = S.sel[tid];
        const float v = cs[c];
        int rank = 0;
        for (int i = 0; i < kk; ++i) {
          const int c2 = S.sel[i];
          const float v2 = cs[c2];
          rank += (v2 > v) || (v2 == v && c2 < c);
        }
        S.slot_c[rank] = c;
      }
      __syncthreads();
    }
    // 3. the new hypotheses
    const bool last_frame = t + 1 == tend;
    if (tid < beam) {
      const int k = tid;
      int src = k, tok = -1;
      if (k < kk) {
        const int c = S.slot_c[k];
        const int h = c / K1, j = c - h * K1;
        src = h;
        if (j == 0) {
          S.npb[k] = S.spb[h]; S.npnb[k] = S.spnb[h]; S.nlm[k] = S.lm[h];
          S.nlast[k] = S.last[h]; S.nlen[k] = S.len[h]; S.nhash[k] = S.hash[h];
          if constexpr (MODE != kRows) { S.nnode[k] = S.node[h]; S.nst[k] = S.st[h]; S.nla[k] = S.la[h]; }
        } else if constexpr (MODE != kRows) {
          const int r = (j - 1) / W1, q = (j - 1) - r * W1;
          const int v = S.ttok[r];
          Ext o;
          if constexpr (MODE == kLexicon)
            lex_ext(a, S, h, v, trie_child(a.lex, S.node[h], v), q, o);  // a kept candidate exists
          else
            ngram_ext(a, S, h, v, o);
          tok = v;
          S.npb[k] = kNegInf; S.npnb[k] = ext_lp(S, h, v, S.tlp[r]); S.nlm[k] = o.lm;
          S.nlast[k] = v; S.nlen[k] = S.len[h] + 1; S.nhash[k] = o.hash;
          S.nnode[k] = o.node; S.nst[k] = o.st; S.nla[k] = o.la;
        } else {
          const int v = S.ttok[j - 1];
          tok = v;
          S.npb[k] = kNegInf; S.npnb[k] = ext_lp(S, h, v, S.tlp[j - 1]); S.nlm[k] = ext_lm(a, S, rb, h, v);
          S.nlast[k] = v; S.nlen[k] = S.len[h] + 1; S.nhash[k] = esp_hash_u64(S.hash[h], (unsigned long long)v);
        }
      } else {
        S.npb[k] = kNegInf; S.npnb[k] = kNegInf; S.nlm[k] = 0.f;
        S.nlast[k] = -1; S.nlen[k] = 0; S.nhash[k] = 0ull;
        if constexpr (MODE != kRows) { S.nnode[k] = 0; S.nst[k] = a.ng.start; S.nla[k] = 0.f; }
      }
      a.par[(long)t * gridDim.x * beam + rb + k] = src;
      a.ptok[(long)t * gridDim.x * beam + rb + k] = tok;
      if (last_frame && a.new_order) {
        a.new_order[rb + k] = (int)(rb + src);
        a.grown[rb + k] = tok >= 0;
        a.fed[rb + k] = lm_col(tok >= 0 ? tok : a.eos, a.lm_blank);
      }
    }
    __syncthreads();
    if (tid < beam) {
      S.pb[tid] = S.npb[tid]; S.pnb[tid] = S.npnb[tid]; S.lm[tid] = S.nlm[tid];
      S.last[tid] = S.nlast[tid]; S.len[tid] = S.nlen[tid]; S.hash[tid] = S.nhash[tid];
      if constexpr (MODE != kRows) { S.node[tid] = S.nnode[tid]; S.st[tid] = S.nst[tid]; S.la[tid] = S.nla[tid]; }
    }
    __syncthreads();
  }
  if (tid < beam) {
    a.pb[rb + tid] = S.pb[tid];
    a.pnb[rb + tid] = S.pnb[tid];
    a.lmacc[rb + tid] = S.lm[tid];
    a.last[rb + tid] = S.last[tid];
    a.len[rb + tid] = S.len[tid];
    a.hash[rb + tid] = S.hash[tid];
    if constexpr (MODE != kRows) {
      a.node[rb + tid] = S.node[tid];
      a.lmst[rb + tid] = S.st[tid];
      a.la[rb + tid] = S.la[tid];
    }
  }
}

// ---- finalize -------------------------------------------------------------------------------------------------
template <int MODE>
__global__ void __launch_bounds__(kT)
ctc_beam_finalize_kernel(SearchArgs a, int Vlm, int nbest, int pad, int* __restrict__ out_tok, int* __restrict__ out_len,
                         float* __restrict__ out_score, int* __restrict__ out_frames) {
  esp_pdl();
  __shared__ float sc[kMaxBeam], lse_lm[kMaxBeam];
  __shared__ int order[kMaxBeam];
  const int b = blockIdx.x, tid = threadIdx.x, beam = a.beam;
  const long rb = (long)b * beam;
  const int T = a.in_lens[b] < a.t_max ? a.in_lens[b] : a.t_max;
  if constexpr (MODE == kRows) {
    if (tid < beam) sc[tid] = lae(a.pb[rb + tid], a.pnb[rb + tid]) + a.lmacc[rb + tid];
    __syncthreads();
    if (a.lm) lm_row_lse(a, rb, sc, lse_lm, Vlm);
    __syncthreads();
    if (tid < beam && a.lm && sc[tid] != kNegInf)
      sc[tid] += a.lm_weight * (lm_val(a.lm, a.lm_f32, (rb + tid) * a.ld_lm + lm_col(a.eos, a.lm_blank)) - lse_lm[tid]);
  } else if (tid < beam) {
    float s = lae(a.pb[rb + tid], a.pnb[rb + tid]) + a.lmacc[rb + tid];
    if (MODE == kLexicon) s = a.node[rb + tid] == 0 ? s + a.la[rb + tid] : kNegInf;  // no hypothesis ends inside a word
    if (s != kNegInf) {
      int nx;
      s += a.lm_weight * ngram_probe(a.ng, a.lmst[rb + tid], a.ng.eos, &nx);
    }
    sc[tid] = s;
  }
  __syncthreads();
  if (tid < beam) {
    const float v = sc[tid];
    int rank = 0;
    for (int i = 0; i < beam; ++i) rank += (sc[i] > v) || (sc[i] == v && i < tid);
    order[rank] = tid;
  }
  __syncthreads();
  // one thread per returned hypothesis walks the parent table back from the sentence's last frame
  if (tid < nbest) {
    const long o = (long)b * nbest + tid;
    int* ot = out_tok + o * a.t_max;
    int* of = out_frames ? out_frames + o * a.t_max : nullptr;
    int L = 0;
    float s = kNegInf;
    if (tid < beam) {
      const int k0 = order[tid];
      s = sc[k0];
      if (s != kNegInf) {
        L = a.len[rb + k0];
        int k = k0, p = L;
        for (int t = T - 1; t >= 0 && p > 0; --t) {
          const long e = (long)t * gridDim.x * beam + rb + k;
          const int tok = a.ptok[e];
          if (tok >= 0) {
            --p;
            ot[p] = tok;
            if (of) of[p] = t;
          }
          k = a.par[e];
        }
      }
    }
    for (int p = L; p < a.t_max; ++p) {
      ot[p] = pad;
      if (of) of[p] = -1;
    }
    out_len[o] = L;
    out_score[o] = s;
  }
}

struct Ws {
  float *pb, *pnb, *lm;
  int *last, *len;
  unsigned long long* hash;
  int *par, *ptok;
  int *node, *lmst;  // n-gram modes only, after the rest
  float* la;
};
inline Ws carve(void* ws, long B, long t_max, long beam) {
  char* p = (char*)ws;
  const long N = B * beam;
  Ws w;
  w.hash = (unsigned long long*)p; p += align256(N * 8);
  w.pb = (float*)p; p += align256(N * 4);
  w.pnb = (float*)p; p += align256(N * 4);
  w.lm = (float*)p; p += align256(N * 4);
  w.last = (int*)p; p += align256(N * 4);
  w.len = (int*)p; p += align256(N * 4);
  w.par = (int*)p; p += align256(t_max * N * 4);
  w.ptok = (int*)p; p += align256(t_max * N * 4);
  w.node = (int*)p; p += align256(N * 4);
  w.lmst = (int*)p; p += align256(N * 4);
  w.la = (float*)p;
  return w;
}

}  // namespace

extern "C" int64_t esp_ctc_beam_workspace_bytes(int32_t B, int32_t t_max, int32_t beam) {
  const long N = (long)B * beam;
  return align256(N * 8) + 5 * align256(N * 4) + 2 * align256((long)t_max * N * 4);
}

extern "C" int esp_ctc_beam_frames(const void* logits, int64_t stride_b, int64_t stride_t, int32_t V, int32_t B,
                                   int32_t t_max, const int32_t* in_lens, int32_t K, int32_t blank, int32_t pad,
                                   int32_t eos, int32_t unk, float* lse, float* lp_blank, int32_t* top_tok,
                                   float* top_lp, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(B >= 0 && t_max >= 0 && V > 0, "bad CTC beam shape");
  ESP_CHECK(V <= kMaxV, "vocabulary too large for the CTC beam search (V=%d > %d)", V, kMaxV);
  ESP_CHECK(K >= 1 && K <= kMaxBeam, "beam_size_token %d out of range [1, %d]", K, kMaxBeam);
  ESP_CHECK(blank >= 0 && blank < V, "blank index out of range");
  if (B == 0 || t_max == 0) return 0;
  ESP_CHECK(logits && in_lens && lse && lp_blank && top_tok && top_lp, "null pointer passed to esp_ctc_beam_frames");
  const size_t smem = ((size_t)V * 2 + 15) / 16 * 16;
  ESP_SMEM_OPTIN(ctc_beam_frames_kernel, smem);
  ESP_CUDA(esp_launch(ctc_beam_frames_kernel, dim3(t_max, B), kT, smem, st, (const bf16*)logits, (long)stride_b, (long)stride_t,
                      V, t_max, in_lens, K, blank, pad, eos, unk, lse, lp_blank, top_tok, top_lp));
  return 0;
}

static int beam_args(SearchArgs& a, const void* logits, int64_t stride_b, int64_t stride_t, int32_t V, int32_t B,
                     int32_t t_max, const int32_t* in_lens, int32_t K, int32_t beam, const void* lm, int32_t lm_f32,
                     int64_t ld_lm, int32_t V_lm, int32_t lm_blank, float lm_weight, int32_t eos, void* workspace) {
  ESP_CHECK(beam >= 1 && beam <= kMaxBeam, "beam_size %d out of range [1, %d]", beam, kMaxBeam);
  ESP_CHECK(K >= 1 && K <= kMaxBeam, "beam_size_token %d out of range [1, %d]", K, kMaxBeam);
  ESP_CHECK(B >= 0 && t_max >= 0 && V > 0 && V <= kMaxV, "bad CTC beam shape");
  ESP_CHECK(workspace && in_lens, "null pointer passed to the CTC beam search");
  ESP_CHECK(!lm || (V_lm > 0 && ld_lm >= V_lm && eos >= 0 && eos < V), "bad LM rows for the CTC beam search");
  ESP_CHECK(!lm || V_lm == V - (lm_blank >= 0 ? 1 : 0), "LM vocabulary (%d) does not match the CTC vocabulary (%d)", V_lm, V);
  a = SearchArgs();
  a.logits = (const bf16*)logits; a.stride_b = stride_b; a.stride_t = stride_t; a.V = V; a.t_max = t_max;
  a.in_lens = in_lens; a.K = K; a.beam = beam;
  a.lm = lm; a.lm_f32 = lm_f32; a.ld_lm = ld_lm; a.lm_blank = lm_blank; a.lm_weight = lm_weight; a.eos = eos;
  Ws w = carve(workspace, B, t_max, beam);
  a.pb = w.pb; a.pnb = w.pnb; a.lmacc = w.lm; a.last = w.last; a.len = w.len; a.hash = w.hash; a.par = w.par; a.ptok = w.ptok;
  return 0;
}

extern "C" int esp_ctc_beam_search(const void* logits, int64_t stride_b, int64_t stride_t, int32_t V, int32_t B,
                                   int32_t t_max, const int32_t* in_lens, const float* lse, const float* lp_blank,
                                   const int32_t* top_tok, const float* top_lp, int32_t K, int32_t beam,
                                   float beam_threshold, int32_t t0, int32_t t1, const void* lm, int32_t lm_f32,
                                   int64_t ld_lm, int32_t V_lm, int32_t lm_blank, float lm_weight, float word_score,
                                   int32_t eos, int32_t* new_order, int32_t* grown, int32_t* fed, void* workspace,
                                   void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  SearchArgs a;
  if (beam_args(a, logits, stride_b, stride_t, V, B, t_max, in_lens, K, beam, lm, lm_f32, ld_lm, V_lm, lm_blank, lm_weight,
                eos, workspace))
    return -1;
  ESP_CHECK(t0 >= 0 && t0 <= t1 && t1 <= t_max, "frame range [%d, %d) out of [0, %d]", t0, t1, t_max);
  ESP_CHECK(!new_order == !grown && !new_order == !fed, "new_order, grown and fed go together");
  ESP_CHECK(!(beam_threshold < 0.f), "beam_threshold must be >= 0");
  if (B == 0) return 0;
  ESP_CHECK(t0 == t1 || (lse && lp_blank && top_tok && top_lp && logits), "null pointer passed to esp_ctc_beam_search");
  a.lse = lse; a.lpb = lp_blank; a.top_tok = top_tok; a.top_lp = top_lp; a.threshold = beam_threshold;
  a.t0 = t0; a.t1 = t1; a.word_score = word_score; a.new_order = new_order; a.grown = grown; a.fed = fed;
  const size_t smem = (size_t)beam * (K + 1) * sizeof(float);
  ESP_SMEM_OPTIN(ctc_beam_search_kernel<kRows>, smem);
  ESP_CUDA(esp_launch(ctc_beam_search_kernel<kRows>, dim3(B), kT, smem, st, a, (int)V_lm));
  return 0;
}

extern "C" int esp_ctc_beam_finalize(int32_t B, int32_t t_max, const int32_t* in_lens, int32_t V, int32_t beam,
                                     int32_t nbest, const void* lm, int32_t lm_f32, int64_t ld_lm, int32_t V_lm,
                                     int32_t lm_blank, float lm_weight, int32_t eos, int32_t pad, void* workspace,
                                     int32_t* out_tokens, int32_t* out_len, float* out_scores, int32_t* out_frames,
                                     void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  SearchArgs a;
  if (beam_args(a, nullptr, 0, 0, V, B, t_max, in_lens, 1, beam, lm, lm_f32, ld_lm, V_lm, lm_blank, lm_weight, eos,
                workspace))
    return -1;
  ESP_CHECK(nbest >= 1 && nbest <= kMaxBeam, "nbest %d out of range [1, %d]", nbest, kMaxBeam);
  if (B == 0) return 0;
  ESP_CHECK(out_tokens && out_len && out_scores, "null pointer passed to esp_ctc_beam_finalize");
  ESP_CUDA(esp_launch(ctc_beam_finalize_kernel<kRows>, dim3(B), kT, 0, st, a, (int)V_lm, nbest, pad, out_tokens, out_len, out_scores,
                      out_frames));
  return 0;
}

// ---- n-gram entry points ----------------------------------------------------------------------------------------
extern "C" int esp_ngram_score(const EspNgram* lm, int32_t n, const int32_t* states, const int32_t* words, float* out_logp,
                               int32_t* out_next, void* stream) {
  ESP_CHECK(lm && n >= 0, "esp_ngram_score: bad arguments");
  if (n == 0) return 0;
  ESP_CHECK(states && words && out_logp && out_next && lm->word, "null pointer passed to esp_ngram_score");
  ESP_CUDA(esp_launch(ngram_score_kernel, dim3(grid_for(n, kT)), kT, 0, (cudaStream_t)stream, *lm, (int)n, states, words,
                      out_logp, out_next));
  return 0;
}

extern "C" int64_t esp_ctc_ngram_workspace_bytes(int32_t B, int32_t t_max, int32_t beam) {
  return esp_ctc_beam_workspace_bytes(B, t_max, beam) + 3 * align256((long)B * beam * 4);
}

// shared memory of the n-gram search: candidate scores + the static SearchSmem, within the H100's 227 KB per block
static int ngram_smem(int beam, int K, const EspLexicon* lex, size_t& smem, int& W1) {
  W1 = lex ? 1 + lex->max_words : 1;
  smem = (size_t)beam * (1 + (size_t)K * W1) * sizeof(float);
  const size_t limit = 227 * 1024 - sizeof(SearchSmem);
  ESP_CHECK(smem <= limit,
            "the n-gram CTC search does not fit in shared memory: beam %d x (1 + beam_size_token %d x (1 + %d words at "
            "one lexicon node)) candidates need %zu bytes, at most %zu fit; lower the beam or beam_size_token",
            beam, K, W1 - 1, smem, limit);
  return 0;
}

static int ngram_args(SearchArgs& a, const EspNgram* lm, const int32_t* tok_word, const EspLexicon* lex, float lm_weight,
                      float word_score, int32_t B, int32_t t_max, int32_t beam, void* workspace) {
  ESP_CHECK(lm && lm->word && lm->order >= 1 && lm->order <= 6, "bad n-gram tables passed to the CTC search");
  ESP_CHECK(!lex || (lex->child_off && lex->word_off && lex->word_lm && lex->smear && lex->num_nodes >= 1 &&
                     lex->max_words >= 0), "bad lexicon trie passed to the CTC search");
  a.ng = *lm;
  if (lex) a.lex = *lex;
  a.tok_word = tok_word;
  a.W1 = lex ? 1 + lex->max_words : 1;
  a.lm = nullptr;
  a.lm_weight = lm_weight;
  a.word_score = word_score;
  Ws w = carve(workspace, B, t_max, beam);
  a.node = w.node; a.lmst = w.lmst; a.la = w.la;
  return 0;
}

extern "C" int esp_ctc_ngram_search(const void* logits, int64_t stride_b, int64_t stride_t, int32_t V, int32_t B,
                                    int32_t t_max, const int32_t* in_lens, const float* lse, const float* lp_blank,
                                    const int32_t* top_tok, const float* top_lp, int32_t K, int32_t beam,
                                    float beam_threshold, const EspNgram* lm, const int32_t* tok_word, int32_t n_tok_word,
                                    const EspLexicon* lex, float lm_weight, float word_score, void* workspace,
                                    void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  SearchArgs a;
  if (beam_args(a, logits, stride_b, stride_t, V, B, t_max, in_lens, K, beam, nullptr, 0, 0, 0, -1, lm_weight, 0, workspace))
    return -1;
  if (ngram_args(a, lm, tok_word, lex, lm_weight, word_score, B, t_max, beam, workspace)) return -1;
  ESP_CHECK(lex || tok_word, "the lexicon-free n-gram search needs tok_word");
  ESP_CHECK(lex || n_tok_word >= V, "tok_word maps %d tokens, the CTC vocabulary has %d: the model's output is wider than the "
            "dictionary the n-gram words were mapped from", n_tok_word, V);
  ESP_CHECK(!(beam_threshold < 0.f), "beam_threshold must be >= 0");
  size_t smem;
  int W1;
  if (ngram_smem(beam, K, lex, smem, W1)) return -1;
  if (B == 0) return 0;
  ESP_CHECK(t_max == 0 || (lse && lp_blank && top_tok && top_lp && logits), "null pointer passed to esp_ctc_ngram_search");
  a.lse = lse; a.lpb = lp_blank; a.top_tok = top_tok; a.top_lp = top_lp; a.threshold = beam_threshold;
  a.t0 = 0; a.t1 = t_max;
  if (lex) {
    ESP_SMEM_OPTIN(ctc_beam_search_kernel<kLexicon>, smem);
    ESP_CUDA(esp_launch(ctc_beam_search_kernel<kLexicon>, dim3(B), kT, smem, st, a, 0));
  } else {
    ESP_SMEM_OPTIN(ctc_beam_search_kernel<kNgram>, smem);
    ESP_CUDA(esp_launch(ctc_beam_search_kernel<kNgram>, dim3(B), kT, smem, st, a, 0));
  }
  return 0;
}

extern "C" int esp_ctc_ngram_finalize(int32_t B, int32_t t_max, const int32_t* in_lens, int32_t V, int32_t beam,
                                      int32_t nbest, const EspNgram* lm, const EspLexicon* lex, float lm_weight,
                                      int32_t pad, void* workspace, int32_t* out_tokens, int32_t* out_len,
                                      float* out_scores, int32_t* out_frames, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  SearchArgs a;
  if (beam_args(a, nullptr, 0, 0, V, B, t_max, in_lens, 1, beam, nullptr, 0, 0, 0, -1, lm_weight, 0, workspace)) return -1;
  if (ngram_args(a, lm, nullptr, lex, lm_weight, 0.f, B, t_max, beam, workspace)) return -1;
  ESP_CHECK(nbest >= 1 && nbest <= kMaxBeam, "nbest %d out of range [1, %d]", nbest, kMaxBeam);
  if (B == 0) return 0;
  ESP_CHECK(out_tokens && out_len && out_scores, "null pointer passed to esp_ctc_ngram_finalize");
  if (lex)
    ESP_CUDA(esp_launch(ctc_beam_finalize_kernel<kLexicon>, dim3(B), kT, 0, st, a, 0, nbest, pad, out_tokens, out_len,
                        out_scores, out_frames));
  else
    ESP_CUDA(esp_launch(ctc_beam_finalize_kernel<kNgram>, dim3(B), kT, 0, st, a, 0, nbest, pad, out_tokens, out_len,
                        out_scores, out_frames));
  return 0;
}
