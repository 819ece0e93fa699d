// espresso_b200 -- transducer adaptive-expansion beam search, the whole batch at once (the search steps of
// espresso/tools/transducer_beam_search_decoder.py:270-601 and transducer_utils.py select_k_expansions).
//
// The host loop (espresso_b200/tools/transducer_beam_search_decoder.py: BatchedAdaptiveExpansionSearch) runs the
// prediction network, the LM and the joint GEMMs; these kernels do everything between them on the device tables of
// EspRnntBeam (include/espresso_b200.h):
//   lprobs       one CTA per row: fp32 log_softmax(logits / temperature), LM fusion over the non-blank symbols
//                renormalised to the transducer's non-blank mass, eos folded into blank, + the row's score; the row's
//                top k and its raw blank log-prob.
//   prefix_merge one CTA per utterance: length sort (longest first) and the pairs (j, i), i a prefix of j at most
//                alpha tokens shorter, with the ring rows and tokens of each path step.
//   merge_scores one CTA per utterance: each pair's path score log-added into j, pairs in the listed order.
//   select       one CTA per utterance: one expansion round (prune by gamma, keep the best k, set blanks aside, extend
//                the prefix pool for the others), or the frame's final combination into the best `beam` rows.
//   finalize     one CTA per utterance: scores / (len - 1), sort, backtrack the pool.
//
// Order rule: wherever the host search's order is unspecified (torch.topk / argsort ties, -inf rows, nemit = 0
// divisions), everything here ranks by (key desc, candidate index asc).  Candidate indices follow the order in which
// the host forms candidates: a round's proposals are row * k + rank over the rows in their current order, the final
// combination lists the set-aside entries (in the order they were set aside) before the live rows, the length sort
// and the final sort index the rows.  A NaN key ranks after every number.
//
// Prefix identity: a pool node holds (parent, token, length, esp_hash_u64(parent hash, token)); i is a prefix of j
// iff len_i < len_j and j's ancestor at depth len_i has i's hash -- the rule csrc/ctc_beam.cu merges prefixes by.
#include "common.cuh"
#include "espresso_b200.h"
#include <math.h>

namespace {

constexpr float kNegInf = -INFINITY;
constexpr int kT = 256;
constexpr int kMaxK = 32;                    // beam + beta
constexpr int kMaxCand = kMaxK * kMaxK;      // proposals of one utterance in one round
constexpr int kMaxBeam = 16;
constexpr int kMaxAlpha = 8;
constexpr int kMaxSteps = kMaxBeam * (kMaxBeam - 1) / 2 * kMaxAlpha;

__device__ __forceinline__ float lae(float a, float b) {
  const float m = fmaxf(a, b);
  if (m == kNegInf) return kNegInf;
  return m + log1pf(expf(-fabsf(a - b)));
}

// (key desc, index asc); NaN after every number
__device__ __forceinline__ bool better(float ka, int ia, float kb, int ib) {
  const bool na = ka != ka, nb = kb != kb;
  if (na || nb) return nb && (!na || ia < ib);
  return ka > kb || (ka == kb && ia < ib);
}

// rank of item c among the `n` items with ok[i]: how many beat it
__device__ __forceinline__ int rank_of(int c, int n, const float* key, const bool* ok) {
  int r = 0;
  for (int i = 0; i < n; ++i) r += (ok[i] && better(key[i], i, key[c], c));
  return r;
}

__device__ __forceinline__ float load_x(const void* p, long i, bool f32) {
  return f32 ? static_cast<const float*>(p)[i] : bf2f(static_cast<const bf16*>(p)[i]);
}

// log-softmax normaliser of x[0..n) (fp32 in shared memory)
__device__ float block_lse(const float* x, int n, float* red) {
  float mx = kNegInf;
  for (int v = threadIdx.x; v < n; v += kT) mx = fmaxf(mx, x[v]);
  mx = block_max<kT>(mx, red);
  float s = 0.f;
  if (mx != kNegInf)
    for (int v = threadIdx.x; v < n; v += kT) s += expf(x[v] - mx);
  s = block_sum<kT>(s, red);
  return mx + logf(s);
}

// The transducer row lp[0..V) (normalised) and, with an LM, its normalised row lm[0..V_lm): the LM's log-prob of each
// non-blank v and the fusion's renormalisation term log sum exp(lp_nb) - log sum exp(lp_nb + w * lm_nb).
__device__ __forceinline__ float lm_of(const float* lm, int v, int blank, bool no_blank_in_lm) {
  return lm[no_blank_in_lm && v > blank ? v - 1 : v];
}
__device__ float fusion_scale(const float* lp, const float* lm, int V, int blank, float w, bool nbl, float* red) {
  float s1 = 0.f, s2 = 0.f;
  for (int v = threadIdx.x; v < V; v += kT) {
    if (v == blank) continue;
    s1 += expf(lp[v]);
    s2 += expf(lp[v] + w * lm_of(lm, v, blank, nbl));
  }
  s1 = block_sum<kT>(s1, red);
  s2 = block_sum<kT>(s2, red);
  return logf(s1) - logf(s2);
}

// ---- lprobs ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kT)
rnnt_beam_lprobs_kernel(const void* __restrict__ logits, long ld, int V, const float* __restrict__ scores, int k, int blank,
                        float inv_temp, int eos, int fold_eos, const void* __restrict__ lm_logits, long ld_lm, int lm_f32,
                        float lm_weight, int nbl, float* __restrict__ val, int* __restrict__ tok, float* __restrict__ lpb) {
  esp_pdl();
  extern __shared__ float sh[];
  float* lp = sh;
  float* lm = sh + V;
  __shared__ float red[32];
  __shared__ float wv[kT / 32];
  __shared__ int wi[kT / 32];
  const long r = blockIdx.x;
  const bf16* row = static_cast<const bf16*>(logits) + r * ld;
  for (int v = threadIdx.x; v < V; v += kT) lp[v] = bf2f(row[v]) * inv_temp;
  __syncthreads();
  const float lse = block_lse(lp, V, red);
  for (int v = threadIdx.x; v < V; v += kT) lp[v] -= lse;
  __syncthreads();
  if (threadIdx.x == 0) lpb[r] = lp[blank];
  if (lm_logits != nullptr) {
    const int V_lm = V - nbl;
    for (int v = threadIdx.x; v < V_lm; v += kT) lm[v] = load_x(lm_logits, r * ld_lm + v, lm_f32);
    __syncthreads();
    const float lse_lm = block_lse(lm, V_lm, red);
    for (int v = threadIdx.x; v < V_lm; v += kT) lm[v] -= lse_lm;
    __syncthreads();
    const float scale = fusion_scale(lp, lm, V, blank, lm_weight, nbl, red);
    for (int v = threadIdx.x; v < V; v += kT)
      if (v != blank) lp[v] += lm_weight * lm_of(lm, v, blank, nbl) + scale;
    __syncthreads();
  }
  if (fold_eos && threadIdx.x == 0) {
    lp[blank] = lae(lp[blank], lp[eos]);
    lp[eos] = kNegInf;
  }
  __syncthreads();
  const float sc = scores[r];
  for (int v = threadIdx.x; v < V; v += kT) lp[v] += sc;
  __syncthreads();
  // top k by repeated block arg-max; a taken entry is marked NaN (a NaN row entry would rank last anyway)
  for (int q = 0; q < k; ++q) {
    float bv = kNegInf;
    int bi = 0x7fffffff;
    for (int v = threadIdx.x; v < V; v += kT) {
      const float x = lp[v];
      if (x == x && better(x, v, bv, bi)) bv = x, bi = v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (better(ov, oi, bv, bi)) bv = ov, bi = oi;
    }
    if ((threadIdx.x & 31) == 0) wv[threadIdx.x >> 5] = bv, wi[threadIdx.x >> 5] = bi;
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < kT / 32; ++w)
        if (better(wv[w], wi[w], bv, bi)) bv = wv[w], bi = wi[w];
      if (bi >= V) bi = 0, bv = kNegInf;  // only when k exceeds the row's numbers (never for k <= V)
      val[r * k + q] = bv;
      tok[r * k + q] = bi;
      lp[bi] = __int_as_float(0x7fc00000);
    }
    __syncthreads();
  }
}

// ---- prefix merge -----------------------------------------------------------------------------------------------------
__device__ __forceinline__ int ancestor(const EspRnntBeam& s, int b, int node, int up) {
  for (; up > 0; --up) node = s.p_parent[(long)b * s.P + node];
  return node;
}

__global__ void __launch_bounds__(32)
rnnt_beam_prefix_merge_kernel(const __grid_constant__ EspRnntBeam s, int t) {
  esp_pdl();
  const int b = blockIdx.x, K = s.K, base = b * K;
  if (threadIdx.x != 0) return;  // at most beam rows: the pair search is serial
  const int n = s.nrow[b];
  const bool active = t < s.nframes[b];
  s.nlive[b] = active ? n : 0;
  s.na[b] = 0;
  s.m_npair[b] = 0;
  if (!active) {
    for (int p = 0; p < K; ++p) s.srow[base + p] = s.fsrc[base + p] = base + p;
    return;
  }
  float sc[kMaxK];
  int ne[kMaxK], ln[kMaxK], nd[kMaxK], ord[kMaxK];
  for (int p = 0; p < n; ++p) sc[p] = s.score[base + p], ne[p] = s.nemit[base + p], ln[p] = s.len[base + p], nd[p] = s.node[base + p];
  for (int p = 0; p < n; ++p) {  // length sort, longest first, ties by row
    int r = 0;
    for (int q = 0; q < n; ++q) r += ln[q] > ln[p] || (ln[q] == ln[p] && q < p);
    ord[r] = p;
  }
  for (int p = 0; p < K; ++p) {
    const int o = p < n ? ord[p] : p;
    s.srow[base + p] = base + o;
    if (p < n) s.score[base + p] = sc[o], s.nemit[base + p] = ne[o], s.len[base + p] = ln[o], s.node[base + p] = nd[o];
  }
  const long pb = (long)b * s.P;
  int npair = 0, nstep = 0;
  for (int pj = 0; pj + 1 < n; ++pj)
    for (int pi = pj + 1; pi < n; ++pi) {
      const int li = ln[ord[pi]], lj = ln[ord[pj]];
      if (!(li < lj && lj <= li + s.alpha)) continue;
      const int nj = nd[ord[pj]], ni = nd[ord[pi]];
      if (s.p_hash[pb + ancestor(s, b, nj, lj - li)] != s.p_hash[pb + ni]) continue;
      int* pr = s.m_pair + ((long)b * s.Pm + npair) * 4;
      pr[0] = pj, pr[1] = pi, pr[2] = b * s.S + nstep, pr[3] = lj - li;
      for (int pos = li - 1; pos < lj - 1; ++pos) {
        const int src = pos == li - 1 ? pi : pj, age = pos == li - 1 ? 0 : lj - 1 - pos;
        s.m_ring[b * s.S + nstep] = age * s.ring_stride + base + ord[src];
        s.m_tok[b * s.S + nstep] = s.p_tok[pb + ancestor(s, b, nj, lj - pos - 2)];
        ++nstep;
      }
      ++npair;
    }
  s.m_npair[b] = npair;
}

__global__ void __launch_bounds__(kT)
rnnt_beam_merge_scores_kernel(const void* __restrict__ logits, long ld, int V, const __grid_constant__ EspRnntBeam s,
                              float inv_temp, int blank, const void* __restrict__ lm_logits, long ld_lm, int lm_f32,
                              float lm_weight, int nbl) {
  esp_pdl();
  extern __shared__ float sh[];
  float* lp = sh;
  float* lm = sh + V;
  __shared__ float red[32];
  __shared__ float contrib[kMaxSteps];
  const int b = blockIdx.x, K = s.K, np = s.m_npair[b];
  if (np == 0) return;
  const int* last = s.m_pair + ((long)b * s.Pm + np - 1) * 4;
  const int s0 = b * s.S, s1 = last[2] + last[3];
  for (int st = s0; st < s1; ++st) {
    const bf16* row = static_cast<const bf16*>(logits) + (long)st * ld;
    for (int v = threadIdx.x; v < V; v += kT) lp[v] = bf2f(row[v]) * inv_temp;
    __syncthreads();
    const float lse = block_lse(lp, V, red);
    for (int v = threadIdx.x; v < V; v += kT) lp[v] -= lse;
    __syncthreads();
    const int tk = s.m_tok[st];
    float c = lp[tk];
    if (lm_logits != nullptr) {
      const int V_lm = V - nbl;
      for (int v = threadIdx.x; v < V_lm; v += kT) lm[v] = load_x(lm_logits, (long)st * ld_lm + v, lm_f32);
      __syncthreads();
      const float lse_lm = block_lse(lm, V_lm, red);
      for (int v = threadIdx.x; v < V_lm; v += kT) lm[v] -= lse_lm;
      __syncthreads();
      const float scale = fusion_scale(lp, lm, V, blank, lm_weight, nbl, red);
      c = c + lm_weight * lm_of(lm, tk, blank, nbl) + scale;
    }
    if (threadIdx.x == 0) contrib[st - s0] = c;
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  for (int q = 0; q < np; ++q) {
    const int* pr = s.m_pair + ((long)b * s.Pm + q) * 4;
    float acc = s.score[b * K + pr[1]];
    for (int st = pr[2]; st < pr[2] + pr[3]; ++st) acc += contrib[st - s0];
    s.score[b * K + pr[0]] = lae(s.score[b * K + pr[0]], acc);
  }
}

// ---- select -------------------------------------------------------------------------------------------------------------
struct Cand {
  float score;
  int nemit, len, node, src;
};

// the best `beam` of the set-aside entries (and, when final, the live rows charged their blank) become the rows
__device__ void combine(const EspRnntBeam& s, int b, int rnd, int beam, int normalize, const float* lpb, bool final,
                        Cand* c, float* key, bool* ok, int* sel) {
  const int K = s.K, A = s.A, BK = s.B * s.K;
  const int na = s.na[b], nl = final ? s.nlive[b] : 0, n = na + nl;
  for (int q = threadIdx.x; q < n; q += kT) {
    Cand x;
    if (q < na) {
      const long a = (long)b * A + q;
      x = Cand{s.a_score[a], s.a_nemit[a], s.a_len[a], s.a_node[a], s.a_src[a]};
    } else {
      const int r = b * K + q - na;
      x = Cand{s.score[r] + lpb[r], s.nemit[r] + 1, s.len[r], s.node[r], (rnd + 1) * BK + r};
    }
    c[q] = x;
    key[q] = normalize ? x.score / (float)x.nemit : x.score;
    ok[q] = true;
  }
  __syncthreads();
  for (int q = threadIdx.x; q < n; q += kT) {
    const int r = rank_of(q, n, key, ok);
    if (r < beam) sel[r] = q;
  }
  __syncthreads();
  const int m = n < beam ? n : beam;
  for (int p = threadIdx.x; p < m; p += kT) {
    const Cand x = c[sel[p]];
    const int r = b * K + p;
    s.score[r] = x.score, s.nemit[r] = x.nemit, s.len[r] = x.len, s.node[r] = x.node, s.fsrc[r] = x.src;
  }
  if (threadIdx.x == 0) s.nrow[b] = m, s.nlive[b] = 0;
}

__global__ void __launch_bounds__(kT)
rnnt_beam_select_kernel(const float* __restrict__ val, const int* __restrict__ tok, int k, const float* __restrict__ lpb,
                        const __grid_constant__ EspRnntBeam s, int rnd, int beam, int blank, float gamma, int normalize,
                        int final) {
  esp_pdl();
  __shared__ Cand c[kMaxCand];
  __shared__ float key[kMaxCand];
  __shared__ bool ok[kMaxCand];
  __shared__ int sel[kMaxCand];
  __shared__ int rnemit[kMaxK], rlen[kMaxK], rnode[kMaxK], rsrow[kMaxK];
  const int b = blockIdx.x, K = s.K, BK = s.B * s.K;
  const int n = s.nlive[b];
  if (n == 0) return;
  if (final) {
    combine(s, b, rnd, beam, normalize, lpb, true, c, key, ok, sel);
    return;
  }
  const int nc = n * k;
  int nonblank = 0;
  for (int q = threadIdx.x; q < nc; q += kT) nonblank |= tok[(long)(b * K + q / k) * k + q % k] != blank;
  const bool all_blank = !__syncthreads_or(nonblank);
  for (int r = threadIdx.x; r < n; r += kT) {
    rnemit[r] = s.nemit[b * K + r], rlen[r] = s.len[b * K + r], rnode[r] = s.node[b * K + r], rsrow[r] = s.srow[b * K + r];
  }
  __syncthreads();
  for (int q = threadIdx.x; q < nc; q += kT) {
    const int r = q / k;
    const long i = (long)(b * K + r) * k + q % k;
    const float v = val[i];
    const int ne = rnemit[r] + (all_blank ? 0 : 1);
    ok[q] = gamma < 0.f || v >= val[(long)(b * K + r) * k] - gamma;
    key[q] = normalize ? v / (float)ne : v;
  }
  __syncthreads();
  for (int q = threadIdx.x; q < nc; q += kT) {
    if (!ok[q]) continue;
    const int r = rank_of(q, nc, key, ok);
    if (r < k) sel[r] = q;
  }
  __syncthreads();
  if (threadIdx.x == 0) {  // at most k survivors: set aside or extend, in rank order
    int kept = 0;
    for (int q = 0; q < nc; ++q) kept += ok[q];
    const int m_all = kept < k ? kept : k;
    int m = 0, na = s.na[b], npool = s.npool[b];
    const long pb = (long)b * s.P;
    for (int p = 0; p < m_all; ++p) {
      const int q = sel[p], r = q / k;
      const long i = (long)(b * K + r) * k + q % k;
      const float v = val[i];
      const int x = tok[i], ne = rnemit[r] + (all_blank ? 0 : 1);
      if (x == blank) {
        const long a = (long)b * s.A + na++;
        s.a_score[a] = v, s.a_nemit[a] = ne, s.a_len[a] = rlen[r], s.a_node[a] = rnode[r], s.a_src[a] = rnd * BK + rsrow[r];
      } else {
        const int row = b * K + m++;
        const int nd = npool++;
        s.p_parent[pb + nd] = rnode[r];
        s.p_tok[pb + nd] = x;
        s.p_len[pb + nd] = s.p_len[pb + rnode[r]] + 1;
        s.p_hash[pb + nd] = esp_hash_u64(s.p_hash[pb + rnode[r]], (unsigned long long)x);
        s.score[row] = v, s.nemit[row] = ne, s.len[row] = rlen[r] + 1, s.node[row] = nd;
        s.parent[row] = rsrow[r], s.prev[row] = x, s.srow[row] = row;
      }
    }
    s.na[b] = na;
    s.npool[b] = npool;
    s.nlive[b] = m;
  }
  __syncthreads();
  if (s.nlive[b] == 0) combine(s, b, rnd, beam, normalize, lpb, false, c, key, ok, sel);
}

// ---- finalize -----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32)
rnnt_beam_finalize_kernel(const __grid_constant__ EspRnntBeam s, int L, int pad, long long* __restrict__ tokens,
                          float* __restrict__ scores, int* __restrict__ lens) {
  esp_pdl();
  const int b = blockIdx.x, K = s.K;
  if (threadIdx.x != 0) return;
  const int n = s.nrow[b];
  float norm[kMaxK];
  for (int p = 0; p < n; ++p) norm[p] = s.score[b * K + p] / (float)(s.len[b * K + p] - 1);
  for (int p = 0; p < K; ++p) {
    long long* out = tokens + ((long)b * K + p) * L;
    for (int d = 0; d < L; ++d) out[d] = pad;
    scores[b * K + p] = kNegInf;
    lens[b * K + p] = 0;
  }
  for (int p = 0; p < n; ++p) {
    int r = 0;
    for (int q = 0; q < n; ++q) r += better(norm[q], q, norm[p], p);
    const int ln = s.len[b * K + p] - 1;
    scores[b * K + r] = norm[p];
    lens[b * K + r] = ln;
    long long* out = tokens + ((long)b * K + r) * L;
    int node = s.node[b * K + p];
    for (int d = ln - 1; d >= 0; --d) {
      if (d < L) out[d] = s.p_tok[(long)b * s.P + node];
      node = s.p_parent[(long)b * s.P + node];
    }
  }
}

size_t row_smem(int V, const void* lm_logits, int nbl) { return sizeof(float) * ((size_t)V + (lm_logits ? V - nbl : 0)); }

}  // namespace

extern "C" int esp_rnnt_beam_lprobs(const void* logits, int64_t ld, int32_t V, int32_t n, const float* scores, int32_t k,
                                    int32_t blank, float temperature, int32_t eos, int32_t fold_eos, const void* lm_logits,
                                    int64_t ld_lm, int32_t lm_f32, float lm_weight, int32_t no_blank_in_lm, float* val,
                                    int32_t* tok, float* lpb, void* stream) {
  ESP_CHECK(k >= 1 && k <= V, "rnnt_beam_lprobs: k must be in [1, V]");
  ESP_CHECK(blank >= 0 && blank < V && (!fold_eos || (eos >= 0 && eos < V)), "rnnt_beam_lprobs: blank / eos out of range");
  ESP_CHECK(temperature > 0.f, "rnnt_beam_lprobs: temperature must be positive");
  if (n == 0) return 0;
  const size_t smem = row_smem(V, lm_logits, no_blank_in_lm);
  ESP_CHECK(smem <= 200 * 1024, "rnnt_beam_lprobs: vocabulary too large for one CTA's shared memory");
  ESP_SMEM_OPTIN(rnnt_beam_lprobs_kernel, smem);
  ESP_CUDA(esp_launch(rnnt_beam_lprobs_kernel, n, kT, smem, (cudaStream_t)stream, logits, (long)ld, V, scores, k, blank,
                      1.f / temperature, eos, fold_eos, lm_logits, (long)ld_lm, lm_f32, lm_weight, no_blank_in_lm, val, tok, lpb));
  return 0;
}

static int check_state(const EspRnntBeam* s) {
  ESP_CHECK(s->K >= 1 && s->K <= kMaxK, "rnnt_beam: beam + beta must be in [1, %d]", kMaxK);
  ESP_CHECK(s->Pm <= kMaxBeam * (kMaxBeam - 1) / 2, "rnnt_beam: beam must be at most %d", kMaxBeam);
  ESP_CHECK(s->alpha >= 1 && s->alpha <= kMaxAlpha, "rnnt_beam: prefix_alpha must be in [1, %d]", kMaxAlpha);
  ESP_CHECK(s->A + s->K <= kMaxCand, "rnnt_beam: (expansions per frame + 1) x (beam + beta) must be at most %d", kMaxCand);
  return 0;
}

extern "C" int esp_rnnt_beam_prefix_merge(const EspRnntBeam* s, int32_t t, void* stream) {
  if (check_state(s)) return 1;
  ESP_CUDA(esp_launch(rnnt_beam_prefix_merge_kernel, s->B, 32, 0, (cudaStream_t)stream, *s, t));
  return 0;
}

extern "C" int esp_rnnt_beam_merge_scores(const void* logits, int64_t ld, int32_t V, const EspRnntBeam* s, float temperature,
                                          int32_t blank, const void* lm_logits, int64_t ld_lm, int32_t lm_f32, float lm_weight,
                                          int32_t no_blank_in_lm, void* stream) {
  if (check_state(s)) return 1;
  const size_t smem = row_smem(V, lm_logits, no_blank_in_lm);
  ESP_CHECK(smem <= 200 * 1024, "rnnt_beam_merge_scores: vocabulary too large for one CTA's shared memory");
  ESP_SMEM_OPTIN(rnnt_beam_merge_scores_kernel, smem);
  ESP_CUDA(esp_launch(rnnt_beam_merge_scores_kernel, s->B, kT, smem, (cudaStream_t)stream, logits, (long)ld, V, *s,
                      1.f / temperature, blank, lm_logits, (long)ld_lm, lm_f32, lm_weight, no_blank_in_lm));
  return 0;
}

extern "C" int esp_rnnt_beam_select(const float* val, const int32_t* tok, int32_t k, const float* lpb, const EspRnntBeam* s,
                                    int32_t rnd, int32_t beam, int32_t blank, float gamma, int32_t normalize, int32_t final,
                                    void* stream) {
  if (check_state(s)) return 1;
  ESP_CHECK(final || k == s->K, "rnnt_beam_select: k must be the state's K");
  ESP_CHECK(beam >= 1 && beam <= s->K, "rnnt_beam_select: beam must be in [1, K]");
  ESP_CUDA(esp_launch(rnnt_beam_select_kernel, s->B, kT, 0, (cudaStream_t)stream, val, tok, k, lpb, *s, rnd, beam, blank,
                      gamma, normalize, final));
  return 0;
}

extern "C" int esp_rnnt_beam_finalize(const EspRnntBeam* s, int32_t L, int32_t pad, int64_t* tokens, float* scores,
                                      int32_t* lens, void* stream) {
  if (check_state(s)) return 1;
  ESP_CUDA(esp_launch(rnnt_beam_finalize_kernel, s->B, 32, 0, (cudaStream_t)stream, *s, L, pad, (long long*)tokens, scores,
                      lens));
  return 0;
}
