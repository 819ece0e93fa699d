// espresso_b200 -- label-smoothed cross-entropy fused with the fp32 log-softmax, forward + backward.
//
// Replaces espresso/criterions/label_smoothed_cross_entropy_v2.py:49-120,216-240:
//   lprobs = log_softmax(logits.float());  nll = -lprobs[target]
//   uniform : loss = (1 - eps - eps_i) * nll + eps_i * (-sum_v lprobs[v]),  eps_i = eps / (V - 1)
//   unigram : loss = (1 - eps) * nll + eps * (-sum_v u[v] lprobs[v])        (u = smoothed unigram distribution)
//   temporal: loss = (1 - eps) * nll + eps * (-sum_v m[v] lprobs[v]),  m = the neighbouring targets at distance
//             +-1 / +-2 with weights 5 : 2, normalised, <pad> neighbours dropped (arXiv 1612.02695)
// rows with target == pad give 0.  In every case loss = a * nll + sum_v w_v * (-lprobs[v]) and the autograd is
//   dloss/dlogits = softmax * (a + sum_v w_v) - a * onehot(target) - w.
// One CTA per target token: the logits row is read once (cached in registers), the gradient row is written
// once; the [B*U, V] fp32 log-prob tensor is never materialised.  Algorithmic bytes: 4*V per token.
// Also: embedding lookup (x = E[tok]*scale + pos) and its scatter-add backward
//   (fairseq/models/transformer/transformer_decoder.py:254-300), and a row-wise argmax used by the greedy
//   CTC decoder (espresso/tools/ctc_decoder.py:163-188).
#include "common.cuh"
#include "espresso_b200.h"
#include <math.h>

namespace {

constexpr int kThreads = 256;
constexpr int kCache = 4;  // uint4 per thread -> rows up to 8192 entries stay in registers

// smoothing weights of one row: w_v = base (uniform) + wu * unigram[v] + the (at most 4) temporal neighbours
struct SmoothW {
  float base, wu;
  const float* unigram;
  int nb[4];
  float nw[4];
  __device__ __forceinline__ float at(int v) const {
    float w = base;
    if (unigram) w += wu * __ldg(unigram + v);
#pragma unroll
    for (int k = 0; k < 4; ++k) w += (v == nb[k]) ? nw[k] : 0.f;
    return w;
  }
};

__global__ void __launch_bounds__(kThreads)
lsce_kernel(const bf16* __restrict__ logits, long ld, int V, const int* __restrict__ targets, int pad_idx, float eps,
            int smoothing, const float* __restrict__ unigram, int U, float grad_scale, float* __restrict__ loss,
            float* __restrict__ nll, bf16* __restrict__ grad) {
  __shared__ float red[32];
  const long r = blockIdx.x;
  const bf16* row = logits + r * ld;
  const int tgt = targets[r];
  const int ld_pad = (int)((ld < (long)((V + 7) / 8 * 8)) ? ld : (V + 7) / 8 * 8);
  if (tgt == pad_idx) {  // ignore_index: zero loss, zero gradient
    if (threadIdx.x == 0) { loss[r] = 0.f; nll[r] = 0.f; }
    if (grad) {
      bf16* g = grad + r * ld;
      for (int v = threadIdx.x; v < ld_pad; v += kThreads) g[v] = f2bf(0.f);
    }
    return;
  }
  // ---- smoothing weights of this row
  SmoothW sw;
  sw.base = 0.f; sw.wu = 0.f; sw.unigram = nullptr;
#pragma unroll
  for (int k = 0; k < 4; ++k) { sw.nb[k] = -1; sw.nw[k] = 0.f; }
  float a_nll;  // weight of the nll term
  if (smoothing == 0) {
    sw.base = eps / (float)(V - 1);
    a_nll = 1.f - eps - sw.base;
  } else if (smoothing == 1) {
    sw.unigram = unigram;
    sw.wu = eps;
    a_nll = 1.f - eps;
  } else {
    // temporal: rows are [B, U]; neighbours inside the same sentence, <pad> neighbours carry no mass
    a_nll = 1.f - eps;
    const int t = (int)(r % U);
    const int off[4] = {-2, -1, 1, 2};
    const float cnt[4] = {2.f, 5.f, 5.f, 2.f};
    float tot = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int tt = t + off[k];
      if (tt >= 0 && tt < U) {
        const int id = targets[r + off[k]];
        if (id != pad_idx) { sw.nb[k] = id; sw.nw[k] = cnt[k]; tot += cnt[k]; }
      }
    }
    const float inv = tot > 0.f ? eps / tot : 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) sw.nw[k] *= inv;
  }
  const int nvec = V / 8;  // rows are 16-byte aligned (ld % 8 == 0)
  float x[kCache][8];
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < kCache; ++i) {
    const int vi = threadIdx.x + i * kThreads;
    if (vi < nvec) {
      const uint4 q = *reinterpret_cast<const uint4*>(row + vi * 8);
      unpack_bf16x2(q.x, x[i][0], x[i][1]);
      unpack_bf16x2(q.y, x[i][2], x[i][3]);
      unpack_bf16x2(q.z, x[i][4], x[i][5]);
      unpack_bf16x2(q.w, x[i][6], x[i][7]);
#pragma unroll
      for (int j = 0; j < 8; ++j) mx = fmaxf(mx, x[i][j]);
    }
  }
  for (int v = kCache * kThreads * 8 + threadIdx.x; v < nvec * 8; v += kThreads) mx = fmaxf(mx, bf2f(row[v]));
  for (int v = nvec * 8 + threadIdx.x; v < V; v += kThreads) mx = fmaxf(mx, bf2f(row[v]));
  mx = block_max<kThreads>(mx, red);
  // se = sum exp(x - mx); swx = sum_v w_v x_v; sws = sum_v w_v   (dense part: uniform constant or unigram vector)
  float se = 0.f, swx = 0.f, sws = 0.f;
  auto acc = [&](int v, float a) {
    se += expf(a - mx);
    const float w = sw.base + (sw.unigram ? sw.wu * __ldg(sw.unigram + v) : 0.f);
    swx += w * a;
    sws += w;
  };
#pragma unroll
  for (int i = 0; i < kCache; ++i) {
    const int vi = threadIdx.x + i * kThreads;
    if (vi < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) acc(vi * 8 + j, x[i][j]);
    }
  }
  for (int v = kCache * kThreads * 8 + threadIdx.x; v < nvec * 8; v += kThreads) acc(v, bf2f(row[v]));
  for (int v = nvec * 8 + threadIdx.x; v < V; v += kThreads) acc(v, bf2f(row[v]));
  se = block_sum<kThreads>(se, red);
  swx = block_sum<kThreads>(swx, red);
  sws = block_sum<kThreads>(sws, red);
#pragma unroll
  for (int k = 0; k < 4; ++k) {  // sparse (temporal) part
    if (sw.nb[k] >= 0) {
      swx += sw.nw[k] * bf2f(row[sw.nb[k]]);
      sws += sw.nw[k];
    }
  }
  const float lse = mx + logf(se);
  if (threadIdx.x == 0) {
    const float n = lse - bf2f(row[tgt]);
    nll[r] = n;
    loss[r] = a_nll * n + (sws * lse - swx);  // sum_v w_v * (lse - x_v)
  }
  if (!grad) return;
  bf16* g = grad + r * ld;
  const float coef = a_nll + sws;  // = 1 for uniform smoothing and for normalised unigram / temporal weights
  auto gval = [&](int v, float a) { return (coef * expf(a - lse) - (v == tgt ? a_nll : 0.f) - sw.at(v)) * grad_scale; };
#pragma unroll
  for (int i = 0; i < kCache; ++i) {
    const int vi = threadIdx.x + i * kThreads;
    if (vi < nvec) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = gval(vi * 8 + j, x[i][j]);
      uint4 q;
      q.x = pack_bf16x2(o[0], o[1]);
      q.y = pack_bf16x2(o[2], o[3]);
      q.z = pack_bf16x2(o[4], o[5]);
      q.w = pack_bf16x2(o[6], o[7]);
      *reinterpret_cast<uint4*>(g + vi * 8) = q;
    }
  }
  for (int v = kCache * kThreads * 8 + threadIdx.x; v < nvec * 8; v += kThreads) g[v] = f2bf(gval(v, bf2f(row[v])));
  for (int v = nvec * 8 + threadIdx.x; v < ld_pad; v += kThreads) g[v] = f2bf(v < V ? gval(v, bf2f(row[v])) : 0.f);
}

// x[r, :] = E[tok[r], :] * scale + pos[r % U, :]   (pos optional), optional dropout
__global__ void __launch_bounds__(256)
embed_fwd_kernel(const int* __restrict__ tok, const bf16* __restrict__ E, const bf16* __restrict__ pos, int U, int d,
                 float scale, long R, int pad_idx, bf16* __restrict__ x, float drop_p, uint32_t thresh,
                 unsigned long long seed0, const unsigned long long* __restrict__ seed_ptr) {
  const unsigned long long seed = seed0 + (seed_ptr ? *seed_ptr : 0ull);
  const long nvec = R * (d >> 3);
  const float ds = drop_p > 0.f ? 65536.f / (65536.f - (float)thresh) : 1.f;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long)gridDim.x * blockDim.x) {
    const long r = i / (d >> 3);
    const int c = (int)(i % (d >> 3)) * 8;
    const int t = tok[r];
    float e[8], p[8], o[8];
    const uint4 q = *reinterpret_cast<const uint4*>(E + (long)t * d + c);
    unpack_bf16x2(q.x, e[0], e[1]);
    unpack_bf16x2(q.y, e[2], e[3]);
    unpack_bf16x2(q.z, e[4], e[5]);
    unpack_bf16x2(q.w, e[6], e[7]);
#pragma unroll
    for (int j = 0; j < 8; ++j) p[j] = 0.f;
    if (pos && t != pad_idx) {  // sinusoidal positions: pad tokens get the zero (padding_idx) row
      const uint4 pq = *reinterpret_cast<const uint4*>(pos + (long)(r % U) * d + c);
      unpack_bf16x2(pq.x, p[0], p[1]);
      unpack_bf16x2(pq.y, p[2], p[3]);
      unpack_bf16x2(pq.z, p[4], p[5]);
      unpack_bf16x2(pq.w, p[6], p[7]);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o[j] = bf2f(f2bf(e[j] * scale)) + p[j];  // embed_scale * embed_tokens(x) is a bf16 tensor in the reference
      if (drop_p > 0.f) o[j] = esp_dropout_keep(seed, (unsigned long long)r * d + c + j, thresh) ? o[j] * ds : 0.f;
    }
    uint4 w;
    w.x = pack_bf16x2(o[0], o[1]);
    w.y = pack_bf16x2(o[2], o[3]);
    w.z = pack_bf16x2(o[4], o[5]);
    w.w = pack_bf16x2(o[6], o[7]);
    *reinterpret_cast<uint4*>(x + r * d + c) = w;
  }
}

// dE[tok[r], :] += scale * dropmask(dx[r, :]).  Each term is the fp32 product fp32(dx * fp32(dropscale * scale)); the
// reference's autograd rounds scale * dx to bf16 (the dtype of the scaled embedding) before the embedding backward adds
// it.  Keeping the fp32 product is deliberate: it drops one bf16 rounding per term and changes no expected value.
__global__ void __launch_bounds__(256)
embed_bwd_kernel(const int* __restrict__ tok, const bf16* __restrict__ dx, int d, float scale, long R, int pad_idx,
                 float* __restrict__ dE, float drop_p, uint32_t thresh, unsigned long long seed0,
                 const unsigned long long* __restrict__ seed_ptr) {
  const unsigned long long seed = seed0 + (seed_ptr ? *seed_ptr : 0ull);
  const long n = R * d;
  const float ds = (drop_p > 0.f ? 65536.f / (65536.f - (float)thresh) : 1.f) * scale;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const long r = i / d;
    const int c = (int)(i % d);
    const int t = tok[r];
    if (t == pad_idx) continue;  // nn.Embedding(padding_idx): the pad row receives no gradient
    float g = bf2f(dx[i]);
    if (drop_p > 0.f && !esp_dropout_keep(seed, (unsigned long long)i, thresh)) continue;
    atomicAdd(&dE[(long)t * d + c], g * ds);
  }
}

// (a, ia) ranks before (b, ib) in torch.argmax's order: NaN above every number, then the larger value, then the
// smaller index (the first NaN and the first of equal maxima win)
__device__ __forceinline__ bool argmax_before(float a, int ia, float b, int ib) {
  const bool an = a != a, bn = b != b;
  if (an || bn) return an && (!bn || ia < ib);
  return a > b || (a == b && ia < ib);
}

// argmax over the first V entries of each row, as torch.argmax: the first index wins ties, and a row holding NaN (a
// diverged model, a bf16 overflow) returns its first NaN, so the result is always in [0, V)
__global__ void __launch_bounds__(128)
argmax_rows_kernel(const bf16* __restrict__ x, long ld, int V, long R, int* __restrict__ out) {
  const long r = blockIdx.x;
  if (r >= R) return;
  const bf16* row = x + r * ld;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int v = threadIdx.x; v < V; v += blockDim.x) {
    const float a = bf2f(row[v]);
    if (argmax_before(a, v, best, bi)) { best = a; bi = v; }
  }
  __shared__ float sb[128];
  __shared__ int si[128];
  sb[threadIdx.x] = best;
  si[threadIdx.x] = bi;
  __syncthreads();
  for (int s = 64; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      const float ob = sb[threadIdx.x + s];
      const int oi = si[threadIdx.x + s];
      if (argmax_before(ob, oi, sb[threadIdx.x], si[threadIdx.x])) { sb[threadIdx.x] = ob; si[threadIdx.x] = oi; }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) out[r] = si[0];
}

}  // namespace

extern "C" int esp_lsce_loss(const void* logits, int64_t ld, int32_t V, int64_t R, const int32_t* targets, int32_t pad_idx,
                             float eps, int32_t smoothing_type, const float* unigram, int32_t U, float grad_scale,
                             float* loss, float* nll, void* grad, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(V > 1 && ld >= V && ld % 8 == 0, "LS-CE needs V > 1 and a row stride that is a multiple of 8 (ld=%ld, V=%d)", (long)ld, V);
  ESP_CHECK(logits && targets && loss && nll, "null pointer passed to esp_lsce_loss");
  // rows are read and the gradient written with 16-byte vector accesses
  ESP_CHECK((((uintptr_t)logits | (uintptr_t)grad) & 15) == 0, "esp_lsce_loss needs 16-byte aligned logits and grad");
  ESP_CHECK(smoothing_type >= 0 && smoothing_type <= 2, "smoothing_type: 0 uniform, 1 unigram, 2 temporal");
  ESP_CHECK(smoothing_type != 1 || unigram != nullptr, "unigram smoothing needs the unigram distribution (fp32 [V])");
  ESP_CHECK(smoothing_type != 2 || (U > 0 && R % U == 0), "temporal smoothing needs rows = B * U (U=%d, R=%ld)", U, (long)R);
  if (R == 0) return 0;
  ESP_CUDA(esp_launch_plain(lsce_kernel, (unsigned)R, kThreads, 0, st, (const bf16*)logits, ld, V, targets, pad_idx, eps,
                            smoothing_type, smoothing_type == 1 ? unigram : nullptr, U > 0 ? U : 1, grad_scale, loss, nll,
                            (bf16*)grad));
  return 0;
}

extern "C" int esp_embed_fwd(const int32_t* tokens, const void* E, const void* pos, int32_t U, int32_t d, float scale,
                             int64_t R, int32_t pad_idx, void* x, float drop_p, uint64_t seed, const uint64_t* seed_ptr,
                             void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(d % 8 == 0, "embedding width must be a multiple of 8");
  // E, pos and x are read and written with 16-byte vector accesses
  ESP_CHECK((((uintptr_t)E | (uintptr_t)pos | (uintptr_t)x) & 15) == 0, "esp_embed_fwd needs 16-byte aligned E, pos and x");
  if (R == 0) return 0;
  ESP_CUDA(esp_launch_plain(embed_fwd_kernel, grid_for(R * (d / 8), 256), 256, 0, st, tokens, (const bf16*)E, (const bf16*)pos, U,
                            d, scale, R, pad_idx, (bf16*)x, drop_p, esp_dropout_thresh(drop_p), seed,
                            (const unsigned long long*)seed_ptr));
  return 0;
}

extern "C" int esp_embed_bwd(const int32_t* tokens, const void* dx, int32_t d, float scale, int64_t R, int32_t pad_idx,
                             float* dE, float drop_p, uint64_t seed, const uint64_t* seed_ptr, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (R == 0) return 0;
  ESP_CUDA(esp_launch_plain(embed_bwd_kernel, grid_for(R * d, 256), 256, 0, st, tokens, (const bf16*)dx, d, scale, R, pad_idx, dE,
                            drop_p, esp_dropout_thresh(drop_p), seed, (const unsigned long long*)seed_ptr));
  return 0;
}

extern "C" int esp_argmax_rows(const void* x, int64_t ld, int32_t V, int64_t R, int32_t* out, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(V >= 1 && ld >= V, "argmax_rows needs V >= 1 and a row stride of at least V (ld=%ld, V=%d)", (long)ld, V);
  if (R == 0) return 0;
  ESP_CUDA(esp_launch_plain(argmax_rows_kernel, (unsigned)R, 128, 0, st, (const bf16*)x, ld, V, R, out));
  return 0;
}
