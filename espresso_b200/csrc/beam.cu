// espresso_b200 -- batched beam search step kernels (fairseq/sequence_generator.py:355-609, fairseq/search.py:103-144).
//
//   beam_merge    (:385-427) fp32 log-softmax of the decoder logits (/temperature) [+ lm_weight * log-softmax of the
//                 LM logits], NaN -> -inf, pad = -inf, unk -= penalty, max-len => only eos, eos_factor gate,
//                 min-len => no eos, + cumulative hypothesis score.  One pass writes the fp32 candidate table.
//   beam_topk     (search.py:117-144) top min(2*beam, nb*V-1) over the sentence's nb*V candidates, ordered by
//                 (score descending, flat index ascending) -- a deterministic refinement of torch.topk.
//   beam_bookkeep (:460-609 + finalize_hypos :657-766) eos candidates among the first `beam` are finalised
//                 (tokens, length-normalised score, positional scores) into per-sentence slots; the first
//                 `beam` non-eos candidates become the next hypotheses (tokens / cumulative scores re-gathered
//                 into the other half of a ping-pong buffer) and `new_order` tells the model how to reorder its
//                 incremental state.  Finished sentences stay in the batch (static shapes; results unchanged).
//                 beam_bookkeep_attn also copies each finalised hypothesis's encoder-attention columns (:690,739-748).
//   gather_rows   (multihead_attention.py:964-989 reorder_incremental_state) dst[i] = src[idx[i]].
// The ~40 tiny launches and 3-4 host syncs per step of the reference become 3 launches + one flag read.
#include "common.cuh"
#include "espresso_b200.h"
#include <math.h>

namespace {

constexpr float kNegInf = -INFINITY;
constexpr int kT = 256;

__device__ __forceinline__ float ldx(const void* p, int is_f32, long i) {
  return is_f32 ? ((const float*)p)[i] : bf2f(((const bf16*)p)[i]);
}
__device__ __forceinline__ float row_lse(const void* x, int f32, long off, int V, float inv_temp, float* red) {
  float mx = kNegInf;
  for (int v = threadIdx.x; v < V; v += kT) mx = fmaxf(mx, ldx(x, f32, off + v) * inv_temp);
  mx = block_max<kT>(mx, red);
  float s = 0.f;
  for (int v = threadIdx.x; v < V; v += kT) s += expf(ldx(x, f32, off + v) * inv_temp - mx);
  s = block_sum<kT>(s, red);
  return mx + logf(s);
}

__global__ void __launch_bounds__(kT)
beam_merge_kernel(const void* __restrict__ x, int x_f32, long ldx_, int x_is_logits, float inv_temp,
                  const void* __restrict__ lm, int lm_f32, long ldlm, int lm_is_logits, float lm_weight, int V,
                  const float* __restrict__ prev, int pad, int unk, float unk_penalty, int eos, int force_eos,
                  int use_eos_factor, float eos_factor, int ban_eos, float* __restrict__ out) {
  __shared__ float red[32];
  const long n = blockIdx.x;
  const long xo = n * ldx_, lo = n * ldlm;
  float lse = 0.f, lse_lm = 0.f;
  if (x_is_logits) lse = row_lse(x, x_f32, xo, V, inv_temp, red);
  if (lm && lm_is_logits) lse_lm = row_lse(lm, lm_f32, lo, V, 1.f, red);
  float* o = out + n * V;
  float mx = kNegInf;
  for (int v = threadIdx.x; v < V; v += kT) {
    float lp = x_is_logits ? ldx(x, x_f32, xo + v) * inv_temp - lse : ldx(x, x_f32, xo + v);
    if (lm) lp += lm_weight * (ldx(lm, lm_f32, lo + v) - lse_lm);
    if (lp != lp) lp = kNegInf;          // lprobs[lprobs != lprobs] = -inf
    if (v == pad) lp = kNegInf;          // never select pad
    if (v == unk) lp -= unk_penalty;
    if (force_eos && v != eos) lp = kNegInf;
    o[v] = lp;
    mx = fmaxf(mx, lp);
  }
  mx = block_max<kT>(mx, red);  // also orders the writes above before the eos fix-ups below
  if (threadIdx.x == 0) {
    float e = o[eos];
    if (!force_eos && use_eos_factor && e < eos_factor * mx) e = kNegInf;  // :404-410
    if (ban_eos) e = kNegInf;                                             // :422-424
    o[eos] = e;
  }
  __syncthreads();
  if (prev) {
    const float p = prev[n];
    for (int v = threadIdx.x; v < V; v += kT) o[v] += p;  // search.py:124-126
  }
}

// lexicographic "better": larger value first, then smaller index
__device__ __forceinline__ bool better(float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); }

__global__ void __launch_bounds__(kT)
beam_topk_kernel(const float* __restrict__ cand, long sent_stride, int n_cand, int K, int V, float* __restrict__ out_s,
                 int* __restrict__ out_tok, int* __restrict__ out_beam) {
  __shared__ float sv[kT / 32];
  __shared__ int si[kT / 32];
  __shared__ float lastv_s;
  __shared__ int lasti_s;
  const float* c = cand + (long)blockIdx.x * sent_stride;
  if (threadIdx.x == 0) { lastv_s = INFINITY; lasti_s = -1; }
  __syncthreads();
  for (int r = 0; r < K; ++r) {
    const float lv = lastv_s;
    const int li = lasti_s;
    float bv = kNegInf;
    int bi = 0x7fffffff;
    for (int i = threadIdx.x; i < n_cand; i += kT) {
      const float v = c[i];
      const bool after = (v < lv) || (v == lv && i > li);  // strictly after the previous pick in the total order
      if (after && better(v, i, bv, bi)) { bv = v; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = bv; si[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < kT / 32; ++w)
        if (better(sv[w], si[w], bv, bi)) { bv = sv[w]; bi = si[w]; }
      if (bi == 0x7fffffff) { bv = kNegInf; bi = 0; }  // fewer than K candidates: cannot happen for K <= n_cand
      lastv_s = bv;
      lasti_s = bi;
      out_s[(long)blockIdx.x * K + r] = bv;
      out_tok[(long)blockIdx.x * K + r] = bi % V;
      out_beam[(long)blockIdx.x * K + r] = bi / V;
    }
    __syncthreads();
  }
}

// Small K (2 x beam <= 16, i.e. every recipe's beam): ONE pass over the candidates.  Each thread keeps the KMAX best of its
// strided slice in registers (sorted, static indices), then the block runs K rounds of "every thread offers the head of its
// list, block arg-best, the winner advances" -- exact, same total order (value desc, index asc) as the K-pass kernel.
template <int KMAX>
__global__ void __launch_bounds__(kT)
beam_topk_small_kernel(const float* __restrict__ cand, long sent_stride, int n_cand, int K, int V, float* __restrict__ out_s,
                       int* __restrict__ out_tok, int* __restrict__ out_beam) {
  __shared__ float sv[kT / 32];
  __shared__ int si[kT / 32];
  __shared__ int s_win;
  const float* c = cand + (long)blockIdx.x * sent_stride;
  float lv[KMAX];
  int li[KMAX];
#pragma unroll
  for (int k = 0; k < KMAX; ++k) { lv[k] = kNegInf; li[k] = 0x7fffffff; }
  for (int i = threadIdx.x; i < n_cand; i += kT) {
    const float v = c[i];
    if (better(v, i, lv[KMAX - 1], li[KMAX - 1])) {
      lv[KMAX - 1] = v;
      li[KMAX - 1] = i;
#pragma unroll
      for (int k = KMAX - 1; k > 0; --k) {
        if (better(lv[k], li[k], lv[k - 1], li[k - 1])) {
          const float tv = lv[k]; lv[k] = lv[k - 1]; lv[k - 1] = tv;
          const int ti = li[k]; li[k] = li[k - 1]; li[k - 1] = ti;
        }
      }
    }
  }
  for (int r = 0; r < K; ++r) {
    float bv = lv[0];
    int bi = li[0];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = bv; si[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < kT / 32; ++w)
        if (better(sv[w], si[w], bv, bi)) { bv = sv[w]; bi = si[w]; }
      if (bi == 0x7fffffff) { bv = kNegInf; bi = 0; }
      s_win = bi;
      out_s[(long)blockIdx.x * K + r] = bv;
      out_tok[(long)blockIdx.x * K + r] = bi % V;
      out_beam[(long)blockIdx.x * K + r] = bi / V;
    }
    __syncthreads();
    if (li[0] == s_win) {  // the winner pops its head (indices are unique, so exactly one thread does)
#pragma unroll
      for (int k = 0; k < KMAX - 1; ++k) { lv[k] = lv[k + 1]; li[k] = li[k + 1]; }
      lv[KMAX - 1] = kNegInf;
      li[KMAX - 1] = 0x7fffffff;
    }
    __syncthreads();
  }
}

struct BK {
  int step, max_len, beam, K, eos, pad, L;  // L = row length of tokens (max_len + 2) ; scores rows have L - 1
  int normalize;
  float len_penalty;
};

// Encoder-attention history of the search (ATTN instance only): att [T_max, N, Tk] fp32, row (t, r) written by the
// decoder at step t for cache row r; anc [T_max, N] = the ancestry table of the current step (csrc/decode_attn.cu);
// fin_attn [bsz, beam, L - 1, Tk] receives row t = att[t][anc[t][row]] of every finalised hypothesis (step-major, so
// both the gather and the store are contiguous Tk-float rows; the host transposes to the reference's [Tk, len]).
struct BKAttn {
  const float* att;
  const int* anc;
  float* fin_attn;
  int N, Tk;
};

template <bool ATTN>
__global__ void __launch_bounds__(32)
beam_bookkeep_kernel(BK p, const float* __restrict__ cs, const int* __restrict__ ct, const int* __restrict__ cb,
                     const int* __restrict__ tok_in, int* __restrict__ tok_out, const float* __restrict__ sc_in,
                     float* __restrict__ sc_out, unsigned char* __restrict__ ignore, unsigned char* __restrict__ finished,
                     int* __restrict__ nfin, int* __restrict__ fin_tok, int* __restrict__ fin_len,
                     float* __restrict__ fin_score, float* __restrict__ fin_pos, int* __restrict__ new_order,
                     int* __restrict__ n_unfinished, BKAttn a) {
  const int s = blockIdx.x, lane = threadIdx.x;
  const int beam = p.beam, K = p.K, step = p.step, L = p.L;
  const long rb = (long)s * beam;
  __shared__ int src_c[64];  // candidate chosen for each new hypothesis slot
  __shared__ int done;
  if (finished[s]) {  // keep the rows alive but inert
    for (int k = 0; k < beam; ++k) {
      for (int j = lane; j < L; j += 32) tok_out[(rb + k) * L + j] = tok_in[(rb + k) * L + j];
      for (int j = lane; j < L - 1; j += 32) sc_out[(rb + k) * (L - 1) + j] = sc_in[(rb + k) * (L - 1) + j];
      if (lane == 0) new_order[rb + k] = (int)(rb + k);
    }
    return;
  }
  const float* S = cs + (long)s * K;
  const int* Tk = ct + (long)s * K;
  const int* Bm = cb + (long)s * K;
  // ---- 1. finalise eos candidates among the first `beam` (in candidate order), :467-495 + finalize_hypos
  int had_eos = 0;
  const int nb = beam < K ? beam : K;
  for (int c = 0; c < nb; ++c) {
    const bool is_eos = (Tk[c] == p.eos) && (S[c] != kNegInf) && !ignore[rb + c];
    if (!is_eos) continue;
    had_eos = 1;
    const int slot = nfin[s];
    if (slot < beam) {  // len(finalized[sent]) < beam_size
      const long row = rb + Bm[c];
      int* ft = fin_tok + ((long)s * beam + slot) * (L - 1);
      float* fp = fin_pos + ((long)s * beam + slot) * (L - 1);
      for (int j = lane; j < step; j += 32) ft[j] = tok_in[row * L + 1 + j];  // tokens[1 : step+1]
      for (int j = lane; j <= step; j += 32) {
        const float cur = (j == step) ? S[c] : sc_in[row * (L - 1) + j];
        const float prv = (j == 0) ? 0.f : sc_in[row * (L - 1) + j - 1];
        fp[j] = cur - prv;  // pos_scores[:, 1:] -= pos_scores[:, :-1]
      }
      if constexpr (ATTN) {  // attn.index_select(0, bbsz_idx)[:, :, 1:step + 2] of the reference (:690), one row per step
        const float* __restrict__ att = a.att;
        const int* __restrict__ anc = a.anc;
        float* __restrict__ fa = a.fin_attn + ((long)s * beam + slot) * (L - 1) * a.Tk;
        for (int t = 0; t <= step; ++t) {
          const float* src = att + ((long)t * a.N + anc[(long)t * a.N + row]) * a.Tk;
          for (int j = lane; j < a.Tk; j += 32) fa[(long)t * a.Tk + j] = src[j];
        }
      }
      if (lane == 0) {
        ft[step] = p.eos;
        fin_len[(long)s * beam + slot] = step + 1;
        fin_score[(long)s * beam + slot] = p.normalize ? S[c] / powf((float)(step + 1), p.len_penalty) : S[c];
        nfin[s] = slot + 1;
      }
      __syncwarp();
    }
  }
  __syncwarp();
  if (lane == 0) {
    done = 0;
    if (had_eos && (nfin[s] == beam || step == p.max_len)) {  // is_finished, only for sentences seen this step
      finished[s] = 1;
      done = 1;
      atomicSub(n_unfinished, 1);
    }
  }
  __syncwarp();
  if (done || step >= p.max_len) {
    for (int k = 0; k < beam; ++k) {
      for (int j = lane; j < L; j += 32) tok_out[(rb + k) * L + j] = tok_in[(rb + k) * L + j];
      for (int j = lane; j < L - 1; j += 32) sc_out[(rb + k) * (L - 1) + j] = sc_in[(rb + k) * (L - 1) + j];
      if (lane == 0) new_order[rb + k] = (int)(rb + k);
    }
    return;
  }
  // ---- 2. choose the next hypotheses: the first `beam` candidates that are neither eos nor ignored, in order;
  //         if there are fewer, masked candidates follow in order and are flagged in `ignore` (:551-575)
  if (lane == 0) {
    int n = 0;
    for (int pass = 0; pass < 2 && n < beam; ++pass) {
      for (int c = 0; c < K && n < beam; ++c) {
        const bool raw_eos = (Tk[c] == p.eos) && (S[c] != kNegInf);
        const bool masked = (c < beam) ? (raw_eos || ignore[rb + c]) : raw_eos;
        if ((pass == 0) != masked) src_c[n++] = c | (masked ? 0x10000 : 0);
      }
    }
    for (; n < beam; ++n) src_c[n] = 0 | 0x10000;
  }
  __syncwarp();
  // read the old ignore flags before overwriting: they were only needed above
  for (int k = 0; k < beam; ++k) {
    const int c = src_c[k] & 0xFFFF;
    const long old = rb + Bm[c];
    for (int j = lane; j <= step; j += 32) tok_out[(rb + k) * L + j] = tok_in[old * L + j];
    for (int j = lane; j < step; j += 32) sc_out[(rb + k) * (L - 1) + j] = sc_in[old * (L - 1) + j];
    if (lane == 0) {
      tok_out[(rb + k) * L + step + 1] = Tk[c];
      sc_out[(rb + k) * (L - 1) + step] = S[c];
      new_order[rb + k] = (int)old;
    }
    for (int j = step + 2 + lane; j < L; j += 32) tok_out[(rb + k) * L + j] = p.pad;
  }
  __syncwarp();
  if (lane == 0)
    for (int k = 0; k < beam; ++k) ignore[rb + k] = (src_c[k] & 0x10000) ? 1 : 0;
}

__global__ void __launch_bounds__(256)
gather_rows_kernel(const uint4* __restrict__ src, const int* __restrict__ idx, long row_vec, long n_rows,
                   uint4* __restrict__ dst) {
  const long total = n_rows * row_vec;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long r = i / row_vec, c = i % row_vec;
    dst[i] = src[(long)idx[r] * row_vec + c];
  }
}

}  // namespace

extern "C" int esp_beam_merge(const void* x, int32_t x_f32, int64_t ld_x, int32_t x_is_logits, float temperature,
                              const void* lm, int32_t lm_f32, int64_t ld_lm, int32_t lm_is_logits, float lm_weight,
                              int32_t N, int32_t V, const float* prev_scores, int32_t pad, int32_t unk, float unk_penalty,
                              int32_t eos, int32_t force_eos, int32_t use_eos_factor, float eos_factor, int32_t ban_eos,
                              float* out, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(x && out && V > 0 && temperature > 0.f, "bad arguments to esp_beam_merge");
  if (N == 0) return 0;
  ESP_CUDA(esp_launch_plain(beam_merge_kernel, N, kT, 0, st, x, x_f32, ld_x, x_is_logits, 1.f / temperature, lm, lm_f32, ld_lm,
                            lm_is_logits, lm_weight, V, prev_scores, pad, unk, unk_penalty, eos, force_eos, use_eos_factor,
                            eos_factor, ban_eos, out));
  return 0;
}

extern "C" int esp_beam_topk(const float* cand, int64_t sent_stride, int32_t bsz, int32_t n_cand, int32_t K, int32_t V,
                             float* out_scores, int32_t* out_tokens, int32_t* out_beams, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(K >= 1 && K <= n_cand, "top-k size %d out of range (n_cand=%d)", K, n_cand);
  if (bsz == 0) return 0;
  if (K <= 16)
    ESP_CUDA(esp_launch_plain(beam_topk_small_kernel<16>, bsz, kT, 0, st, cand, sent_stride, n_cand, K, V, out_scores, out_tokens,
                              out_beams));
  else
    ESP_CUDA(esp_launch_plain(beam_topk_kernel, bsz, kT, 0, st, cand, sent_stride, n_cand, K, V, out_scores, out_tokens,
                              out_beams));
  return 0;
}

extern "C" int esp_beam_bookkeep(int32_t step, int32_t max_len, int32_t bsz, int32_t beam, int32_t K, int32_t eos, int32_t pad,
                                 int32_t normalize, float len_penalty, const float* cand_scores, const int32_t* cand_tokens,
                                 const int32_t* cand_beams, const int32_t* tokens_in, int32_t* tokens_out,
                                 const float* scores_in, float* scores_out, uint8_t* ignore, uint8_t* finished,
                                 int32_t* nfin, int32_t* fin_tokens, int32_t* fin_len, float* fin_score, float* fin_pos,
                                 int32_t* new_order, int32_t* n_unfinished, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(beam >= 1 && beam <= 64 && K >= 1, "beam size must be in [1, 64]");
  if (bsz == 0) return 0;
  BK p;
  p.step = step; p.max_len = max_len; p.beam = beam; p.K = K; p.eos = eos; p.pad = pad; p.L = max_len + 2;
  p.normalize = normalize; p.len_penalty = len_penalty;
  ESP_CUDA(esp_launch_plain(beam_bookkeep_kernel<false>, bsz, 32, 0, st, p, cand_scores, cand_tokens, cand_beams, tokens_in,
                            tokens_out, scores_in, scores_out, ignore, finished, nfin, fin_tokens, fin_len, fin_score, fin_pos,
                            new_order, n_unfinished, BKAttn{}));
  return 0;
}

extern "C" int esp_beam_bookkeep_attn(int32_t step, int32_t max_len, int32_t bsz, int32_t beam, int32_t K, int32_t eos,
                                      int32_t pad, int32_t normalize, float len_penalty, const float* cand_scores,
                                      const int32_t* cand_tokens, const int32_t* cand_beams, const int32_t* tokens_in,
                                      int32_t* tokens_out, const float* scores_in, float* scores_out, uint8_t* ignore,
                                      uint8_t* finished, int32_t* nfin, int32_t* fin_tokens, int32_t* fin_len, float* fin_score,
                                      float* fin_pos, int32_t* new_order, int32_t* n_unfinished, const float* att,
                                      const int32_t* anc, int32_t Tk, float* fin_attn, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(beam >= 1 && beam <= 64 && K >= 1, "beam size must be in [1, 64]");
  ESP_CHECK(att && anc && fin_attn && Tk >= 1, "esp_beam_bookkeep_attn: attention history, ancestry table and fin_attn needed");
  if (bsz == 0) return 0;
  BK p;
  p.step = step; p.max_len = max_len; p.beam = beam; p.K = K; p.eos = eos; p.pad = pad; p.L = max_len + 2;
  p.normalize = normalize; p.len_penalty = len_penalty;
  BKAttn a;
  a.att = att; a.anc = anc; a.fin_attn = fin_attn; a.N = bsz * beam; a.Tk = Tk;
  ESP_CUDA(esp_launch_plain(beam_bookkeep_kernel<true>, bsz, 32, 0, st, p, cand_scores, cand_tokens, cand_beams, tokens_in,
                            tokens_out, scores_in, scores_out, ignore, finished, nfin, fin_tokens, fin_len, fin_score, fin_pos,
                            new_order, n_unfinished, a));
  return 0;
}

extern "C" int esp_gather_rows(const void* src, const int32_t* idx, int64_t row_bytes, int64_t n_rows, void* dst, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(row_bytes % 16 == 0, "gather_rows: rows must be multiples of 16 bytes");
  ESP_CHECK((((uintptr_t)src | (uintptr_t)dst) & 15) == 0, "gather_rows: buffers must be 16-byte aligned");
  if (n_rows == 0 || row_bytes == 0) return 0;
  const long total = n_rows * (row_bytes / 16);
  ESP_CUDA(esp_launch_plain(gather_rows_kernel, grid_for(total, 256), 256, 0, st, (const uint4*)src, idx, row_bytes / 16, n_rows,
                            (uint4*)dst));
  return 0;
}
