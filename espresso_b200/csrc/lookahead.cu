// espresso_b200 -- word-level language-model fusion kernels for beam search.
//
// Look-ahead word LM (espresso/models/tensorized_lookahead_language_model.py:84-262; Hori et al., arXiv:1808.02608
// Eqn. 15): a word LM scores SUBWORD hypotheses through a lexical prefix tree.  Every hypothesis keeps a tree node and
// the inclusive cumulative sum of the word distribution P(w | history); the probability of continuing with subword s is
//     [cum(hi(child_s)) - cum(lo(child_s))] / [cum(hi(node)) - cum(lo(node))]
// because the words below a node are contiguous in the (lexically sorted) word dictionary.
//
// The reference stores the tree as a dense [nodes, max_children] int64 table and runs ~40 small tensor ops per search
// step.  Here the tree is CSR (children sorted by subword id) and one search step is three launches:
//   lookahead_words_kernel   reorder nodes by the beam permutation, pick the word each hypothesis has just completed
//   wordlm_cumsum_kernel     softmax + inclusive scan of the word-LM logits (only rows that crossed a word boundary,
//                            the others gather their parent's row), one CTA per hypothesis
//   lookahead_step_kernel    tree transition + the whole subword log-probability row, staged in shared memory
// HBM-bound: 4 Vw bytes read + 4 Vw written per hypothesis for the scan, 4 Vs written for the output row.
#include <math.h>

#include "common.cuh"
#include "espresso_b200.h"

namespace {

constexpr int kScanThreads = 1024;

// ---- (1) nodes after beam reordering + the word fed to the word LM --------------------------------------------------
__global__ void lookahead_words_kernel(const int* __restrict__ nodes_in, const int* __restrict__ new_order,
                                       const int* __restrict__ node_word, int word_unk, int N, int* __restrict__ nodes_out,
                                       int* __restrict__ words) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const int node = nodes_in[new_order ? new_order[n] : n];
  nodes_out[n] = node;
  const int w = node_word[node];
  words[n] = w < 0 ? word_unk : w;  // non-terminal or out-of-tree: <unk> (:129-130)
}

// ---- (2) cum[n, :] = cumsum(softmax(logits[n, :Vw]))  or  cum_in[new_order[n], :] ----------------------------------
template <typename T>
__device__ __forceinline__ float ldf(const T* p, long i);
template <>
__device__ __forceinline__ float ldf<float>(const float* p, long i) { return p[i]; }
template <>
__device__ __forceinline__ float ldf<bf16>(const bf16* p, long i) { return bf2f(p[i]); }

template <typename T>
__global__ void __launch_bounds__(kScanThreads)
wordlm_cumsum_kernel(const T* __restrict__ logits, long ld, int Vw, const int* __restrict__ prev_tokens, long tok_stride,
                     int space_idx, int first, const float* __restrict__ cum_in, const int* __restrict__ new_order,
                     float* __restrict__ cum_out, float* __restrict__ eos_logprob, int word_eos, int log_mode) {
  const int n = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float* out = cum_out + (long)n * Vw;
  const bool fresh = first || prev_tokens[(long)n * tok_stride] == space_idx;
  if (!fresh) {
    // no word boundary: the distribution of the parent hypothesis carries over (reorder_incremental_state :264-272)
    const float* src = cum_in + (long)(new_order ? new_order[n] : n) * Vw;
    for (int i = tid; i < Vw; i += kScanThreads) out[i] = src[i];
    if (tid == 0) eos_logprob[n] = 0.f;  // never read for such rows
    return;
  }
  const T* x = logits + (long)n * ld;
  __shared__ float s_f[32];
  __shared__ double s_d[32];
  __shared__ double s_carry;
  // max
  float m = -INFINITY;
  for (int i = tid; i < Vw; i += kScanThreads) m = fmaxf(m, ldf(x, i));
  m = warp_max(m);
  if (lane == 0) s_f[warp] = m;
  __syncthreads();
  m = s_f[lane];
  m = warp_max(m);
  __syncthreads();
  // normaliser (double: Vw can be ~10^5 and the differences below cancel)
  double z = 0.0;
  for (int i = tid; i < Vw; i += kScanThreads) z += (double)__expf(ldf(x, i) - m);
  z = warp_sum_d(z);
  if (lane == 0) s_d[warp] = z;
  __syncthreads();
  z = s_d[lane];
  z = warp_sum_d(z);
  __syncthreads();
  const double inv_z = 1.0 / z;
  const float log_z = (float)log(z);
  if (tid == 0) {
    s_carry = 0.0;
    eos_logprob[n] = (ldf(x, word_eos) - m) - log_z;
  }
  if (log_mode) {  // multi-level LM: the row holds log-probabilities, no scan
    for (int i = tid; i < Vw; i += kScanThreads) out[i] = (ldf(x, i) - m) - log_z;
    return;
  }
  __syncthreads();
  // tiled inclusive scan, carry in double
  for (int base = 0; base < Vw; base += kScanThreads) {
    const int i = base + tid;
    double v = i < Vw ? (double)__expf(ldf(x, i) - m) : 0.0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double t = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += t;
    }
    if (lane == 31) s_d[warp] = v;
    __syncthreads();
    if (warp == 0) {
      double t = s_d[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const double u = __shfl_up_sync(0xffffffffu, t, o);
        if (lane >= o) t += u;
      }
      s_d[lane] = t;  // inclusive totals of warps 0..lane
    }
    __syncthreads();
    const double carry = s_carry + (warp > 0 ? s_d[warp - 1] : 0.0);
    if (i < Vw) out[i] = (float)((carry + v) * inv_z);
    __syncthreads();
    if (tid == kScanThreads - 1) s_carry = carry + v;
    __syncthreads();
  }
}

// ---- (3) tree transition + subword log-probabilities ----------------------------------------------------------------
struct TreeView {
  const int* child_off;   // [n_nodes + 1]
  const int* child_tok;   // [n_edges] subword id, ascending inside a node
  const int* child_node;  // [n_edges]
  const int* node_word;   // [n_nodes] word id or -1
  const int* node_lo;     // [n_nodes] first word id - 1
  const int* node_hi;     // [n_nodes] last word id
};

__global__ void __launch_bounds__(256)
lookahead_step_kernel(const int* __restrict__ prev_tokens, long tok_stride, int first, const int* __restrict__ nodes_in,
                      int* __restrict__ nodes_out, const float* __restrict__ cum, int Vw, const float* __restrict__ eos_logprob,
                      TreeView tr, int space_idx, int eos_idx, int pad_idx, int word_unk, float oov_penalty, int open_vocab,
                      float zero, float* __restrict__ out, long ld_out, int Vs) {
  extern __shared__ float row[];  // [Vs] probabilities
  __shared__ int s_node;
  const int n = blockIdx.x;
  const int tid = threadIdx.x;
  const int prev = prev_tokens[(long)n * tok_stride];
  const bool after_space = !first && prev == space_idx;
  const float* cs = cum + (long)n * Vw;
  // -- transition (:150-164): <space> -> root (1); a child labelled `prev` -> that child; otherwise out of the tree (0)
  if (tid == 0) s_node = first ? 1 : (after_space ? 1 : 0);
  __syncthreads();
  if (!first && !after_space) {
    const int cur = nodes_in[n];
    const int e0 = tr.child_off[cur], e1 = tr.child_off[cur + 1];  // node 0 has no edges
    for (int e = e0 + tid; e < e1; e += blockDim.x)
      if (tr.child_tok[e] == prev) s_node = tr.child_node[e];  // at most one match
    __syncthreads();
  }
  const int node = s_node;
  if (tid == 0) nodes_out[n] = node;
  // -- base value of the row (:173-197)
  float base;
  if (!open_vocab) base = zero;
  else if (node == 0) base = 1.f;                                            // case 4: free run outside the lexicon
  else base = oov_penalty * (cs[word_unk] - cs[word_unk - 1]);               // case 3
  for (int i = tid; i < Vs; i += blockDim.x) row[i] = base;
  __syncthreads();
  if (open_vocab && node != 0 && tid == 0) {
    if (after_space || prev == eos_idx) row[space_idx] = zero;  // no empty words
    if (!after_space) row[eos_idx] = zero;                      // sentences end after a <space>
  }
  // -- mass below this node (:199-209)
  float sum_p = 1.f;
  if (node > 1) sum_p = cs[tr.node_hi[node]] - cs[tr.node_lo[node]];
  const bool dead = sum_p < zero;
  __syncthreads();
  // -- case 2: children (:211-233)
  {
    const int e0 = tr.child_off[node], e1 = tr.child_off[node + 1];
    for (int e = e0 + tid; e < e1; e += blockDim.x) {
      const int c = tr.child_node[e];
      const float p = dead ? zero : (cs[tr.node_hi[c]] - cs[tr.node_lo[c]]) / sum_p;
      row[tr.child_tok[e]] = p;
    }
  }
  __syncthreads();
  if (tid == 0) {
    row[pad_idx] = zero;
    // -- case 1: the node ends a word -> <space> carries the word probability (:236-255)
    const int w = tr.node_word[node];
    if (w >= 0) row[space_idx] = dead ? zero : (cs[w] - cs[w - 1]) / sum_p;
  }
  __syncthreads();
  float* o = out + (long)n * ld_out;
  for (int i = tid; i < Vs; i += blockDim.x) {
    float v = __logf(fmaxf(row[i], zero));
    if (after_space && i == eos_idx) v = eos_logprob[n];  // word-level </s> (:260-263)
    o[i] = v;
  }
  for (int i = Vs + tid; i < ld_out; i += blockDim.x) o[i] = -INFINITY;  // row padding never wins
}


// ---- multi-level (subword + word) LM: espresso/models/external_language_model.py:385-555 ---------------------------
// The subword LM scores every step; when a hypothesis completes a word (emits <space>) the word LM's log-probability of
// that word REPLACES what the subword LM has accumulated inside the word (cumlp), and an out-of-lexicon word gets the
// word LM's <unk> score plus a penalty.  One CTA per hypothesis: tree transition, bookkeeping of cumlp from the previous
// step's (reordered) output row, log-softmax of the subword LM's logits scaled by its weight, and the <space> / </s>
// corrections, written as the fp32 row the search consumes and the next step reads back.
template <typename T>
__global__ void __launch_bounds__(256)
multilevel_step_kernel(const int* __restrict__ prev_tokens, long tok_stride, int first, const int* __restrict__ nodes_in,
                       int* __restrict__ nodes_out, const int* __restrict__ new_order, const float* __restrict__ wlp, int Vw,
                       const T* __restrict__ sub, long ld_sub, int sub_is_logits, float sub_weight,
                       const float* __restrict__ out_prev, const float* __restrict__ cumlp_in, float* __restrict__ cumlp_out,
                       TreeView tr, int space_idx, int eos_idx, int word_unk, int word_eos, float log_oov_penalty,
                       int open_vocab, float logzero, float* __restrict__ out, long ld_out, int Vs) {
  __shared__ int s_node;
  __shared__ float s_red[8];
  const int n = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int prev = prev_tokens[(long)n * tok_stride];
  const bool after_space = !first && prev == space_idx;
  const int src = new_order ? new_order[n] : n;
  // -- transition (:437-455); nodes_in is already reordered (lookahead_words_kernel)
  if (tid == 0) s_node = (first || after_space) ? 1 : 0;
  __syncthreads();
  if (!first && !after_space) {
    const int cur = nodes_in[n];
    const int e0 = tr.child_off[cur], e1 = tr.child_off[cur + 1];
    for (int e = e0 + tid; e < e1; e += blockDim.x)
      if (tr.child_tok[e] == prev) s_node = tr.child_node[e];
    __syncthreads();
  }
  const int node = s_node;
  const bool is_child = !first && !after_space && node != 0;
  // -- log-probability the subword LM has spent inside the current word (:456-470)
  float cum = 0.f;
  if (!first) {
    const bool add = open_vocab ? !after_space : is_child;
    if (add) cum = cumlp_in[src] + out_prev[(long)src * ld_out + prev];
  }
  // -- subword LM row: weight * log_softmax (or weight * given log-probs)
  const T* x = sub + (long)n * ld_sub;
  float shift = 0.f;
  if (sub_is_logits) {
    float m = -INFINITY;
    for (int i = tid; i < Vs; i += blockDim.x) m = fmaxf(m, ldf(x, i));
    m = warp_max(m);
    if (lane == 0) s_red[warp] = m;
    __syncthreads();
    m = warp_max(lane < 8 ? s_red[lane] : -INFINITY);
    __syncthreads();
    float z = 0.f;
    for (int i = tid; i < Vs; i += blockDim.x) z += __expf(ldf(x, i) - m);
    z = warp_sum(z);
    if (lane == 0) s_red[warp] = z;
    __syncthreads();
    z = warp_sum(lane < 8 ? s_red[lane] : 0.f);
    shift = m + __logf(z);
  }
  const bool oov_row = !open_vocab && !first && !after_space && !is_child;  // closed vocabulary: dead hypothesis (:483-485)
  // -- <space> and </s> corrections (:497-533)
  const int w = tr.node_word[node];
  const float* wl = wlp + (long)n * Vw;
  float v_space = wl[w >= 0 ? w : word_unk] + (w >= 0 ? -cum : log_oov_penalty);
  if (after_space || prev == eos_idx) v_space = logzero;
  float* o = out + (long)n * ld_out;
  for (int i = tid; i < Vs; i += blockDim.x) {
    float v = oov_row ? logzero : (ldf(x, i) - shift) * sub_weight;
    if (i == space_idx) v = v_space;
    if (i == eos_idx) v = after_space ? v + wl[word_eos] : logzero;
    o[i] = v;
  }
  for (int i = Vs + tid; i < ld_out; i += blockDim.x) o[i] = -INFINITY;
  if (tid == 0) {
    nodes_out[n] = node;
    cumlp_out[n] = cum;
  }
}

}  // namespace

extern "C" int esp_lookahead_words(const int32_t* nodes_in, const int32_t* new_order, const int32_t* node_word,
                                   int32_t word_unk, int32_t N, int32_t* nodes_out, int32_t* words, void* stream) {
  ESP_CHECK(nodes_in && node_word && nodes_out && words, "bad arguments to esp_lookahead_words");
  if (N == 0) return 0;
  ESP_CUDA(esp_launch_plain(lookahead_words_kernel, (N + 127) / 128, 128, 0, (cudaStream_t)stream, nodes_in, new_order, node_word,
                            word_unk, N, nodes_out, words));
  return 0;
}

extern "C" int esp_wordlm_cumsum(const void* logits, int32_t logits_f32, int64_t ld, int32_t N, int32_t Vw,
                                 const int32_t* prev_tokens, int64_t tok_stride, int32_t space_idx, int32_t first,
                                 const float* cum_in, const int32_t* new_order, float* cum_out, float* eos_logprob,
                                 int32_t word_eos, int32_t log_mode, void* stream) {
  ESP_CHECK(logits && cum_out && eos_logprob && Vw > 1 && word_eos >= 0 && word_eos < Vw, "bad arguments to esp_wordlm_cumsum");
  ESP_CHECK(first || (prev_tokens && cum_in && cum_in != cum_out), "esp_wordlm_cumsum: later steps need prev_tokens and a "
            "separate cum_in (rows are gathered across hypotheses)");
  if (N == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (logits_f32)
    ESP_CUDA(esp_launch_plain(wordlm_cumsum_kernel<float>, N, kScanThreads, 0, st, (const float*)logits, ld, Vw, prev_tokens,
                              tok_stride, space_idx, first, cum_in, new_order, cum_out, eos_logprob, word_eos, log_mode));
  else
    ESP_CUDA(esp_launch_plain(wordlm_cumsum_kernel<bf16>, N, kScanThreads, 0, st, (const bf16*)logits, ld, Vw, prev_tokens,
                              tok_stride, space_idx, first, cum_in, new_order, cum_out, eos_logprob, word_eos, log_mode));
  return 0;
}

extern "C" int esp_lookahead_step(const int32_t* prev_tokens, int64_t tok_stride, int32_t N, int32_t first,
                                  const int32_t* nodes_in, int32_t* nodes_out, const float* cum, int32_t Vw,
                                  const float* eos_logprob, const int32_t* child_off, const int32_t* child_tok,
                                  const int32_t* child_node, const int32_t* node_word, const int32_t* node_lo,
                                  const int32_t* node_hi, int32_t space_idx, int32_t eos_idx, int32_t pad_idx, int32_t word_unk,
                                  float oov_penalty, int32_t open_vocab, float zero, float* out, int64_t ld_out, int32_t Vs,
                                  void* stream) {
  ESP_CHECK(prev_tokens && nodes_in && nodes_out && cum && eos_logprob && child_off && child_tok && child_node && node_word &&
                node_lo && node_hi && out,
            "bad arguments to esp_lookahead_step");
  ESP_CHECK(Vs > 0 && ld_out >= Vs && space_idx >= 0 && space_idx < Vs && eos_idx >= 0 && eos_idx < Vs && pad_idx >= 0 &&
                pad_idx < Vs && word_unk >= 1 && word_unk < Vw,
            "esp_lookahead_step: symbol indices out of range");
  ESP_CHECK((size_t)Vs * sizeof(float) <= 200 * 1024, "esp_lookahead_step: subword vocabulary of %d does not fit in shared memory", Vs);
  if (N == 0) return 0;
  const size_t smem = (size_t)Vs * sizeof(float);
  ESP_SMEM_OPTIN(lookahead_step_kernel, smem);
  TreeView tr{child_off, child_tok, child_node, node_word, node_lo, node_hi};
  ESP_CUDA(esp_launch_plain(lookahead_step_kernel, N, 256, smem, (cudaStream_t)stream, prev_tokens, tok_stride, first, nodes_in,
                            nodes_out, cum, Vw, eos_logprob, tr, space_idx, eos_idx, pad_idx, word_unk, oov_penalty, open_vocab,
                            zero, out, ld_out, Vs));
  return 0;
}

extern "C" int esp_multilevel_step(const int32_t* prev_tokens, int64_t tok_stride, int32_t N, int32_t first, const int32_t* nodes_in,
                                   int32_t* nodes_out, const int32_t* new_order, const float* wordlm_logprobs, int32_t Vw,
                                   const void* sub, int32_t sub_f32, int64_t ld_sub, int32_t sub_is_logits, float sub_weight,
                                   const float* out_prev, const float* cumlp_in, float* cumlp_out, const int32_t* child_off,
                                   const int32_t* child_tok, const int32_t* child_node, const int32_t* node_word,
                                   int32_t space_idx, int32_t eos_idx, int32_t word_unk, int32_t word_eos, float log_oov_penalty,
                                   int32_t open_vocab, float logzero, float* out, int64_t ld_out, int32_t Vs, void* stream) {
  ESP_CHECK(prev_tokens && nodes_in && nodes_out && wordlm_logprobs && sub && cumlp_out && child_off && child_tok && child_node &&
                node_word && out,
            "bad arguments to esp_multilevel_step");
  ESP_CHECK(first || (out_prev && cumlp_in && out_prev != out && cumlp_in != cumlp_out),
            "esp_multilevel_step: later steps read the previous step's rows of OTHER hypotheses (separate buffers needed)");
  ESP_CHECK(Vs > 0 && ld_out >= Vs && space_idx >= 0 && space_idx < Vs && eos_idx >= 0 && eos_idx < Vs && word_unk >= 0 &&
                word_unk < Vw && word_eos >= 0 && word_eos < Vw,
            "esp_multilevel_step: symbol indices out of range");
  if (N == 0) return 0;
  TreeView tr{child_off, child_tok, child_node, node_word, nullptr, nullptr};
  cudaStream_t st = (cudaStream_t)stream;
  if (sub_f32)
    ESP_CUDA(esp_launch_plain(multilevel_step_kernel<float>, N, 256, 0, st, prev_tokens, tok_stride, first, nodes_in, nodes_out,
                              new_order, wordlm_logprobs, Vw, (const float*)sub, ld_sub, sub_is_logits, sub_weight, out_prev,
                              cumlp_in, cumlp_out, tr, space_idx, eos_idx, word_unk, word_eos, log_oov_penalty, open_vocab,
                              logzero, out, ld_out, Vs));
  else
    ESP_CUDA(esp_launch_plain(multilevel_step_kernel<bf16>, N, 256, 0, st, prev_tokens, tok_stride, first, nodes_in, nodes_out,
                              new_order, wordlm_logprobs, Vw, (const bf16*)sub, ld_sub, sub_is_logits, sub_weight, out_prev,
                              cumlp_in, cumlp_out, tr, space_idx, eos_idx, word_unk, word_eos, log_oov_penalty, open_vocab,
                              logzero, out, ld_out, Vs));
  return 0;
}
