// espresso_b200 -- the optional parts of the beam search step: fairseq's search-option set beyond plain BeamSearch.
//
//   block_ngrams    (fairseq/ngram_repeat_block.py, called at sequence_generator.py:448-449) -inf for every token that
//                   would complete an n-gram already present in the hypothesis: the last n-1 tokens (columns
//                   step-n+2 .. step of the token buffer, column 0 = the start symbol) are compared with every earlier
//                   window tokens[i .. i+n-2], i < step-n+2, and tokens[i+n-1] is banned where they match.
//   prefix          (sequence_generator.py:414-424 -> _prefix_tokens :623-657) rows whose prefix token at `step` is
//                   not pad keep only that token; a sentence whose prefix token is eos gets its first beam's tokens,
//                   scores and candidate row copied into every beam.
//   diverse_groups  (search.py:551-618 DiverseBeamSearch) beams g::G form group g; group g > 0 adds
//                   -strength * (number of times each token was chosen by earlier groups at this step), then a
//                   BeamSearch step inside the group; candidates come out interleaved by group.
//   sibling_topk    (search.py:745-810 DiverseSiblingsSearch, step > 0) per-hypothesis top k, minus rank * rate, then
//                   top k over the sentence's beam * k pool.
//   sample          (search.py:621-742 Sampling) one draw per candidate from p = exp(lprobs) of its row (step 0: beam
//                   draws from each sentence's first row), restricted to the top-k or top-p set, by an inverse-CDF draw
//                   on the counter RNG of common.cuh.
// Every top-k here orders candidates by (score descending, flat index ascending), as esp_beam_topk does.
#include "common.cuh"
#include "espresso_b200.h"
#include <math.h>

namespace {

constexpr float kNegInf = -INFINITY;
constexpr int kT = 256;

__device__ __forceinline__ bool better(float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); }

// One CTA per hypothesis row; thread i compares window i with the row's last n-1 tokens.
__global__ void __launch_bounds__(128)
block_ngrams_kernel(const int* __restrict__ tokens, long ld_tok, int step, int n, float* __restrict__ lp, long ld_lp, int V) {
  const int* t = tokens + (long)blockIdx.x * ld_tok;
  const int tail = step - n + 2;  // first column of the last n-1 tokens = number of earlier windows
  for (int i = threadIdx.x; i < tail; i += blockDim.x) {
    bool same = true;
    for (int k = 0; k < n - 1 && same; ++k) same = t[i + k] == t[tail + k];
    const int ban = t[i + n - 1];
    if (same && ban >= 0 && ban < V) lp[(long)blockIdx.x * ld_lp + ban] = kNegInf;
  }
}

// One CTA per sentence.
__global__ void __launch_bounds__(kT)
prefix_kernel(const int* __restrict__ prefix, long ld_prefix, int beam, int step, int pad, int eos, float* __restrict__ cand,
              int V, int* __restrict__ tokens, int L, float* __restrict__ scores) {
  const int s = blockIdx.x;
  const int pt = prefix[(long)s * ld_prefix + step];
  if (pt == pad || pt < 0 || pt >= V) return;
  const long r0 = (long)s * beam;
  const bool rep = pt == eos;  // replicate_first_beam: every beam becomes a copy of beam 0
  const float keep0 = cand[r0 * V + pt];
  for (long i = threadIdx.x; i < (long)beam * V; i += kT) {
    const int b = (int)(i / V), v = (int)(i - (long)b * V);
    float* c = cand + (r0 + b) * V + v;
    if (v != pt) *c = kNegInf;
    else if (rep && b > 0) *c = keep0;
  }
  if (!rep) return;
  for (long i = threadIdx.x; i < (long)(beam - 1) * L; i += kT) {
    const long b = 1 + i / L, j = i % L;
    tokens[(r0 + b) * L + j] = tokens[r0 * L + j];
  }
  for (long i = threadIdx.x; i < (long)(beam - 1) * (L - 1); i += kT) {
    const long b = 1 + i / (L - 1), j = i % (L - 1);
    scores[(r0 + b) * (L - 1) + j] = scores[r0 * (L - 1) + j];
  }
}

// One CTA per sentence; `cnt` (dynamic shared memory, V floats) counts the tokens chosen by earlier groups.  The group's
// candidate value is (lprob + (-strength) * count) + cumulative score, in the reference's order of fp32 operations.
__global__ void __launch_bounds__(kT)
diverse_groups_kernel(const float* __restrict__ lp, const float* __restrict__ prev, int beam, int V, int G, int Kg, float neg_strength,
                      float* __restrict__ out_s, int* __restrict__ out_t, int* __restrict__ out_b) {
  extern __shared__ float cnt[];
  __shared__ float sv[kT / 32];
  __shared__ int si[kT / 32];
  __shared__ float lastv_s;
  __shared__ int lasti_s;
  __shared__ int picked[64];
  const int s = blockIdx.x, bg = beam / G, K = Kg * G;
  const int n_cand = prev ? bg * V : V;  // step 0: the group's first beam only
  for (int v = threadIdx.x; v < V; v += kT) cnt[v] = 0.f;
  for (int g = 0; g < G; ++g) {
    if (threadIdx.x == 0) { lastv_s = INFINITY; lasti_s = -1; }
    __syncthreads();
    for (int r = 0; r < Kg; ++r) {
      const float lv = lastv_s;
      const int li = lasti_s;
      float bv = kNegInf;
      int bi = 0x7fffffff;
      for (int i = threadIdx.x; i < n_cand; i += kT) {
        const int j = i / V, v = i - j * V;
        const long row = (long)s * beam + g + (long)j * G;
        float x = lp[row * V + v];
        if (g > 0) x = __fadd_rn(x, __fmul_rn(neg_strength, cnt[v]));
        if (prev) x = __fadd_rn(x, prev[row]);
        const bool after = (x < lv) || (x == lv && i > li);
        if (after && better(x, i, bv, bi)) { bv = x; bi = i; }
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
        if (bi == 0x7fffffff) { bv = kNegInf; bi = 0; }  // cannot happen: Kg < n_cand
        lastv_s = bv;
        lasti_s = bi;
        const long o = (long)s * K + (long)r * G + g;  // torch.stack(..., dim=2).view(bsz, -1)
        out_s[o] = bv;
        out_t[o] = bi % V;
        out_b[o] = (bi / V) * G + g;
        picked[r] = bi % V;
      }
      __syncthreads();
    }
    if (threadIdx.x == 0)  // diversity_buf.scatter_add_ after the whole group
      for (int r = 0; r < Kg; ++r) cnt[picked[r]] += 1.f;
    __syncthreads();
  }
}

__global__ void sibling_penalty_kernel(float* __restrict__ s, long n, int k, float rate) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
    s[i] = __fsub_rn(s[i], __fmul_rn((float)(i % k + 1), rate));  // s_list[i].sub_(arange(1, k + 1) * rate)
}

// out_t holds each winner's rank inside its hypothesis's list; replace it by that entry's token
__global__ void sibling_remap_kernel(const int* __restrict__ work_t, const int* __restrict__ out_b, int beam, int k, long n,
                                     int* __restrict__ out_t) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const long s = i / k;
    out_t[i] = work_t[(s * beam + out_b[i]) * k + out_t[i]];
  }
}

// ---- sampling -----------------------------------------------------------------------------------------------------
// Probabilities are ranked by (p descending, token ascending).  Masses are fixed point, W = floor(p * 2^40) (an exact
// scaling of the fp32 p), so every sum is exact and independent of the summation order.  Top-p keeps the tokens whose
// preceding mass in that order is < floor(topp * 2^40) (the reference's "cumsum < p, plus one more token"); top-k keeps
// the tokens with fewer than k tokens before them.  The draw takes T = floor(h * sum(W) / 2^64) for a 64-bit hash h of
// (seed, step, row, draw) and picks the token whose cumulative kept mass, in token order, first exceeds T.
constexpr int kS = 256;
constexpr float kFix = 1099511627776.f;  // 2^40

// exclusive prefix of v over the CTA's threads; `total` = the sum over all of them.  sh: kS / 32 entries.
__device__ __forceinline__ unsigned long long block_scan_u64(unsigned long long v, unsigned long long* sh,
                                                             unsigned long long& total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  unsigned long long x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) sh[w] = x;
  __syncthreads();
  unsigned long long off = 0, tot = 0;
#pragma unroll
  for (int i = 0; i < kS / 32; ++i) {
    if (i < w) off += sh[i];
    tot += sh[i];
  }
  __syncthreads();
  total = tot;
  return off + x - v;
}

// One CTA per output candidate o = s * beam + j.
__global__ void __launch_bounds__(kS)
sample_kernel(const float* __restrict__ lp, const float* __restrict__ prev, int beam, int V, int topk, float topp,
              const unsigned long long* __restrict__ seed_ptr, int step, float* __restrict__ out_s, int* __restrict__ out_t,
              int* __restrict__ out_b) {
  extern __shared__ float p[];
  __shared__ unsigned long long sh[kS / 32];
  __shared__ int s_pick;
  const int o = blockIdx.x, s = o / beam, j = o - s * beam;
  const long row = prev ? (long)o : (long)s * beam;  // step 0: every draw comes from the sentence's first row
  for (int v = threadIdx.x; v < V; v += kS) p[v] = expf(lp[row * V + v]);
  if (threadIdx.x == 0) s_pick = -1;
  __syncthreads();
  const int C = (V + kS - 1) / kS, v0 = min(V, (int)threadIdx.x * C), v1 = min(V, v0 + C);
  const bool by_mass = topp > 0.f, trunc = by_mass || (topk > 0 && topk < V);
  const unsigned long long limit = by_mass ? __float2ull_rz(topp * kFix) : (unsigned long long)topk;
  auto mass = [&](float x) -> unsigned long long { return by_mass ? __float2ull_rz(x * kFix) : 1ull; };
  // smallest u with (mass of the tokens whose p has bit pattern > u) < limit: the p of the last kept token
  unsigned lo = 0, hi = 0x7f800000u;
  unsigned long long tot;
  while (trunc && lo < hi) {
    const unsigned mid = lo + (hi - lo) / 2;
    unsigned long long g = 0;
    for (int v = v0; v < v1; ++v)
      if (__float_as_uint(p[v]) > mid) g += mass(p[v]);
    block_scan_u64(g, sh, tot);
    if (tot < limit) hi = mid;
    else lo = mid + 1;
  }
  const unsigned ustar = lo;
  unsigned long long above = 0, tie = 0;
  if (trunc) {
    unsigned long long g = 0;
    for (int v = v0; v < v1; ++v) {
      const unsigned b = __float_as_uint(p[v]);
      if (b > ustar) g += mass(p[v]);
      else if (b == ustar) tie += mass(p[v]);
    }
    block_scan_u64(g, sh, above);
  }
  // tokens whose p equals the last kept p are kept in token order while the mass before them is < limit
  const unsigned long long tie0 = above + block_scan_u64(tie, sh, tot);
  unsigned long long run = tie0, w = 0;
  for (int v = v0; v < v1; ++v) {
    const unsigned b = __float_as_uint(p[v]);
    const bool keep = !trunc || b > ustar || (b == ustar && run < limit);
    if (trunc && b == ustar) run += mass(p[v]);
    if (keep) w += __float2ull_rz(p[v] * kFix);
  }
  unsigned long long wtot;
  const unsigned long long w0 = block_scan_u64(w, sh, wtot);
  const unsigned long long h = esp_hash_u64(esp_hash_u64(*seed_ptr, (unsigned long long)step),
                                            ((unsigned long long)row << 16) | (unsigned long long)(prev ? 0 : j));
  const unsigned long long T = __umul64hi(h, wtot);
  if (wtot > 0 && T >= w0 && T < w0 + w) {
    unsigned long long cum = w0;
    run = tie0;
    for (int v = v0; v < v1; ++v) {
      const unsigned b = __float_as_uint(p[v]);
      const bool keep = !trunc || b > ustar || (b == ustar && run < limit);
      if (trunc && b == ustar) run += mass(p[v]);
      if (!keep) continue;
      cum += __float2ull_rz(p[v] * kFix);
      if (T < cum) { s_pick = v; break; }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const int k = s_pick < 0 ? 0 : s_pick;  // no mass at all (every token -inf): a -inf candidate
    float sc = s_pick < 0 ? kNegInf : logf(p[k]);
    if (prev) sc = __fadd_rn(sc, prev[o]);
    out_s[o] = sc;
    out_t[o] = k;
    out_b[o] = prev ? j : 0;
  }
}

}  // namespace

extern "C" int esp_beam_sample(const float* lprobs, const float* prev_scores, int32_t bsz, int32_t beam, int32_t V, int32_t topk,
                               float topp, const uint64_t* seed, int32_t step, float* out_scores, int32_t* out_tokens,
                               int32_t* out_beams, void* stream) {
  ESP_CHECK(lprobs && seed && out_scores && out_tokens && out_beams && beam >= 1 && beam < 65536 && V > 0 && step >= 0,
            "bad arguments to esp_beam_sample");
  ESP_CHECK(!(topp > 0.f) || topp <= 1.f, "esp_beam_sample: top-p %g outside (0, 1]", (double)topp);
  const size_t smem = (size_t)V * sizeof(float);
  ESP_CHECK(smem <= 200 * 1024, "esp_beam_sample: vocabulary of %d does not fit in shared memory", V);
  if (bsz == 0) return 0;
  ESP_SMEM_OPTIN(sample_kernel, smem);
  ESP_CUDA(esp_launch_plain(sample_kernel, bsz * beam, kS, smem, (cudaStream_t)stream, lprobs, prev_scores, beam, V, topk, topp,
                            (const unsigned long long*)seed, step, out_scores, out_tokens, out_beams));
  return 0;
}

extern "C" int esp_beam_block_ngrams(const int32_t* tokens, int64_t ld_tokens, int32_t N, int32_t step, int32_t n, float* lprobs,
                                     int64_t ld_lprobs, int32_t V, void* stream) {
  ESP_CHECK(tokens && lprobs && n >= 1 && step >= 0 && V > 0, "bad arguments to esp_beam_block_ngrams (n=%d, step=%d)", n, step);
  ESP_CHECK(ld_tokens >= step + 1, "esp_beam_block_ngrams: token rows (%lld) shorter than step + 1", (long long)ld_tokens);
  if (N == 0 || step - n + 2 <= 0) return 0;  // no earlier window yet
  ESP_CUDA(esp_launch_plain(block_ngrams_kernel, N, 128, 0, (cudaStream_t)stream, tokens, (long)ld_tokens, step, n, lprobs,
                            (long)ld_lprobs, V));
  return 0;
}

extern "C" int esp_beam_prefix(const int32_t* prefix, int64_t ld_prefix, int32_t bsz, int32_t beam, int32_t step, int32_t pad,
                               int32_t eos, float* cand, int32_t V, int32_t* tokens, int32_t L, float* scores, void* stream) {
  ESP_CHECK(prefix && cand && tokens && scores && beam >= 1 && V > 0 && L >= 2, "bad arguments to esp_beam_prefix");
  ESP_CHECK(step >= 0 && step < ld_prefix && step < L - 1, "esp_beam_prefix: step %d outside the prefix", step);
  if (bsz == 0) return 0;
  ESP_CUDA(esp_launch_plain(prefix_kernel, bsz, kT, 0, (cudaStream_t)stream, prefix, (long)ld_prefix, beam, step, pad, eos, cand, V,
                            tokens, L, scores));
  return 0;
}

extern "C" int esp_beam_diverse_groups(const float* lprobs, const float* prev_scores, int32_t bsz, int32_t beam, int32_t V,
                                       int32_t groups, int32_t Kg, float strength, float* out_scores, int32_t* out_tokens,
                                       int32_t* out_beams, void* stream) {
  ESP_CHECK(lprobs && out_scores && out_tokens && out_beams && V > 0, "bad arguments to esp_beam_diverse_groups");
  ESP_CHECK(groups >= 1 && beam % groups == 0, "DiverseBeamSearch requires --beam to be divisible by the number of groups");
  const int n_cand = prev_scores ? beam / groups * V : V;
  ESP_CHECK(Kg >= 1 && Kg <= 64 && Kg < n_cand, "esp_beam_diverse_groups: %d candidates per group out of range", Kg);
  const size_t smem = (size_t)V * sizeof(float);
  ESP_CHECK(smem <= 200 * 1024, "esp_beam_diverse_groups: vocabulary of %d does not fit the token counts in shared memory", V);
  if (bsz == 0) return 0;
  ESP_SMEM_OPTIN(diverse_groups_kernel, smem);
  ESP_CUDA(esp_launch_plain(diverse_groups_kernel, bsz, kT, smem, (cudaStream_t)stream, lprobs, prev_scores, beam, V, groups, Kg,
                            -strength, out_scores, out_tokens, out_beams));
  return 0;
}

extern "C" int esp_beam_sibling_topk(const float* cand, int32_t bsz, int32_t beam, int32_t V, int32_t k, float rate, float* work_s,
                                     int32_t* work_t, int32_t* work_b, float* out_scores, int32_t* out_tokens, int32_t* out_beams,
                                     void* stream) {
  ESP_CHECK(cand && work_s && work_t && work_b && out_scores && out_tokens && out_beams && beam >= 1,
            "bad arguments to esp_beam_sibling_topk");
  ESP_CHECK(k >= 1 && k <= V, "esp_beam_sibling_topk: k = %d exceeds the vocabulary (%d)", k, V);
  if (bsz == 0) return 0;
  const long N = (long)bsz * beam;
  if (esp_beam_topk(cand, V, (int32_t)N, V, k, V, work_s, work_t, work_b, stream) != 0) return -1;
  ESP_CUDA(esp_launch_plain(sibling_penalty_kernel, grid_for(N * k, 256), 256, 0, (cudaStream_t)stream, work_s, N * k, k, rate));
  // the pool of sentence s is work_s[s * beam * k ...]: "tokens" of this top-k are ranks, its "beams" are hypotheses
  if (esp_beam_topk(work_s, (int64_t)beam * k, bsz, beam * k, k, k, out_scores, out_tokens, out_beams, stream) != 0) return -1;
  ESP_CUDA(esp_launch_plain(sibling_remap_kernel, grid_for((long)bsz * k, 256), 256, 0, (cudaStream_t)stream, work_t, out_beams,
                            beam, k, (long)bsz * k, out_tokens));
  return 0;
}
