// espresso_b200 -- single-query attention kernels for incremental (beam search) decoding.
//
// Replaces the incremental branch of fairseq/modules/multihead_attention.py:639-760,878-897 (self-attention over
// the cached prefix, encoder attention over per-sentence "beamable" K/V :661-669) and the O(t) index_select of
// every cached tensor per step (`reorder_incremental_state`, :964-989):
//   * K/V of step t are written once at cache[t, row, :] by the projection GEMM and never moved;
//   * beam reordering only re-gathers the int32 ancestry table anc[t][n] = cache row holding hypothesis n's
//     key/value at time t (esp_decode_update_ancestry), which the attention kernel follows.
// Prefix decoding (a CTC prefix beam search fused with a Transformer LM, whose hypotheses grow on different frames
// and by different amounts) keeps the cache by FRAME SLOT instead: kv [S, N, 2d], slot s written at frame s - 1 for
// every row (slot 0 = the eos context), and per hypothesis a path table cells[i][n] = flat cell slot * N + row of its
// i-th key, i < len[n] (esp_decode_update_paths).  Every slot is fresh, so a write never overwrites a cell that another
// hypothesis still reads -- the collision a per-position cache meets when rows have different lengths.
// One warp per (hypothesis, head): phase 1 lanes <- keys (scores, fp32 softmax), phase 2 lanes <- head dims.
#include "common.cuh"
#include "espresso_b200.h"
#include <math.h>

namespace {

constexpr int kMaxKeys = 1280;  // encoder frames after 4x subsampling (36 s -> 900) / decoder steps

// q [N, d]; the K/V of cell c are kv + c * 2d (+d for V).
// PATHS = false: T = step+1 keys; key t of hypothesis n is cell t*N + idx[t*N+n] (idx = the ancestry table).
// PATHS = true:  T = lens[n] keys (0 writes zeros); key t of hypothesis n is cell idx[t*N+n] (idx = the path table).
template <bool PATHS>
__global__ void __launch_bounds__(128)
decode_self_attn_kernel(const bf16* __restrict__ q, const bf16* __restrict__ kv, const int* __restrict__ idx,
                        const int* __restrict__ lens, int N, int H, int hd, int T, float scale, bf16* __restrict__ out) {
  extern __shared__ float sm[];  // [warps][T] probabilities
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gw = blockIdx.x * (blockDim.x >> 5) + warp;
  if (gw >= N * H) return;
  const int n = gw / H, h = gw % H;
  if constexpr (PATHS) T = lens[n];
  auto cell = [&](int t) -> long {
    const int i = idx[(long)t * N + n];
    return PATHS ? (long)i : (long)t * N + i;
  };
  const int d = H * hd;
  float* p = sm + warp * kMaxKeys;
  const bf16* qp = q + (long)n * d + h * hd;
  float mx = -INFINITY;
  for (int t = lane; t < T; t += 32) {
    const bf16* kp = kv + cell(t) * 2 * d + h * hd;
    float s = 0.f;
    for (int c = 0; c < hd; c += 2) {
      const __nv_bfloat162 a = *reinterpret_cast<const __nv_bfloat162*>(qp + c);
      const __nv_bfloat162 b = *reinterpret_cast<const __nv_bfloat162*>(kp + c);
      s += __low2float(a) * __low2float(b) + __high2float(a) * __high2float(b);
    }
    s *= scale;
    p[t] = s;
    mx = fmaxf(mx, s);
  }
  mx = warp_max(mx);
  float sum = 0.f;
  for (int t = lane; t < T; t += 32) {
    const float e = __expf(p[t] - mx);
    p[t] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  __syncwarp();
  const float inv = 1.f / sum;
  for (int c = lane * 2; c < hd; c += 64) {
    float a0 = 0.f, a1 = 0.f;
    for (int t = 0; t < T; ++t) {
      const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(kv + cell(t) * 2 * d + d + h * hd + c);
      const float w = bf2f(f2bf(p[t] * inv));  // attention weights are cast to the model dtype before P.V
      a0 += w * __low2float(v);
      a1 += w * __high2float(v);
    }
    *reinterpret_cast<__nv_bfloat162*>(out + (long)n * d + h * hd + c) = __floats2bfloat162_rn(a0, a1);
  }
}

// q [N, d]; encoder K/V per SENTENCE: kv [bsz, Tk, 2d] (k | v); sentence of hypothesis n = n / beam.
// WEIGHTS: one CTA per hypothesis, warp h = head h (same per-warp code, so the context is bit-identical to the plain
// launch); after P.V the CTA writes the fp32 head-mean of the softmax probabilities, summed in head order 0..H-1, to
// weights[n, 0:Tk] (padded keys exactly 0) -- the reference's need_weights path, multihead_attention.py:864,913-915.
template <bool WEIGHTS>
__global__ void __launch_bounds__(WEIGHTS ? 1024 : 128)
decode_cross_attn_kernel(const bf16* __restrict__ q, const bf16* __restrict__ kv, const int* __restrict__ lens, int N, int beam,
                         int H, int hd, int Tk, float scale, bf16* __restrict__ out, float* __restrict__ weights) {
  extern __shared__ float sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gw = blockIdx.x * (blockDim.x >> 5) + warp;
  if (gw >= N * H) return;
  const int n = gw / H, h = gw % H;
  const int d = H * hd;
  const int sent = n / beam;
  const int T = lens ? min(lens[sent], Tk) : Tk;  // encoder_padding_mask -> -inf
  float* p = sm + warp * kMaxKeys;
  const bf16* qp = q + (long)n * d + h * hd;
  const bf16* base = kv + (long)sent * Tk * 2 * d;
  float mx = -INFINITY;
  for (int t = lane; t < T; t += 32) {
    const bf16* kp = base + (long)t * 2 * d + h * hd;
    float s = 0.f;
    for (int c = 0; c < hd; c += 2) {
      const __nv_bfloat162 a = *reinterpret_cast<const __nv_bfloat162*>(qp + c);
      const __nv_bfloat162 b = *reinterpret_cast<const __nv_bfloat162*>(kp + c);
      s += __low2float(a) * __low2float(b) + __high2float(a) * __high2float(b);
    }
    s *= scale;
    p[t] = s;
    mx = fmaxf(mx, s);
  }
  mx = warp_max(mx);
  float sum = 0.f;
  for (int t = lane; t < T; t += 32) {
    const float e = __expf(p[t] - mx);
    p[t] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  __syncwarp();
  const float inv = 1.f / sum;
  for (int c = lane * 2; c < hd; c += 64) {
    float a0 = 0.f, a1 = 0.f;
    for (int t = 0; t < T; ++t) {
      const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(base + (long)t * 2 * d + d + h * hd + c);
      const float w = bf2f(f2bf(p[t] * inv));
      a0 += w * __low2float(v);
      a1 += w * __high2float(v);
    }
    *reinterpret_cast<__nv_bfloat162*>(out + (long)n * d + h * hd + c) = __floats2bfloat162_rn(a0, a1);
  }
  if constexpr (WEIGHTS) {
    for (int t = lane; t < T; t += 32) p[t] *= inv;  // fp32 probabilities of head h
    __syncthreads();
    const float inv_h = 1.f / (float)H;
    float* wr = weights + (long)n * Tk;
    for (int t = threadIdx.x; t < Tk; t += blockDim.x) {
      float acc = 0.f;
      if (t < T)
        for (int hh = 0; hh < H; ++hh) acc += sm[hh * kMaxKeys + t];
      wr[t] = acc * inv_h;
    }
  }
}

// anc_out[t][n] = anc_in[t][new_order[n]] for t < step ; anc_out[step][n] = n
__global__ void __launch_bounds__(256)
update_ancestry_kernel(const int* __restrict__ anc_in, int* __restrict__ anc_out, const int* __restrict__ new_order, int N, int step) {
  const long total = (long)(step + 1) * N;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int t = (int)(i / N), n = (int)(i % N);
    anc_out[i] = (t == step) ? n : anc_in[(long)t * N + (new_order ? new_order[n] : n)];
  }
}

// With p = new_order[n]: cells_out[i][n] = cells_in[i][p] for i < len_in[p]; cells_out[len_in[p]][n] = slot*N + n when
// grown[n]; len_out[n] = len_in[p] + grown[n]; pos_out[n] = len_in[p].  len_in <= slot, so i <= slot covers every path.
__global__ void __launch_bounds__(256)
update_paths_kernel(const int* __restrict__ cells_in, const int* __restrict__ len_in, int* __restrict__ cells_out,
                    int* __restrict__ len_out, int* __restrict__ pos_out, const int* __restrict__ new_order,
                    const int* __restrict__ grown, int N, int slot) {
  const long total = (long)(slot + 1) * N;
  for (long k = (long)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (long)gridDim.x * blockDim.x) {
    const int i = (int)(k / N), n = (int)(k % N);
    const int p = new_order[n], L = len_in[p], g = grown[n] != 0;
    if (i < L)
      cells_out[k] = cells_in[(long)i * N + p];
    else if (i == L && g)
      cells_out[k] = slot * N + n;
    if (i == 0) {
      len_out[n] = L + g;
      if (pos_out) pos_out[n] = L;
    }
  }
}

}  // namespace

extern "C" int esp_decode_self_attn(const void* q, const void* kv_cache, const int32_t* anc, int32_t N, int32_t H, int32_t hd,
                                    int32_t T, float scale, void* out, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(T >= 1 && T <= kMaxKeys && hd % 2 == 0, "decode self-attention: bad shape (T=%d)", T);
  if (N == 0) return 0;
  const int warps = 4;
  const size_t smem = (size_t)warps * kMaxKeys * sizeof(float);
  ESP_CUDA(esp_launch_plain(decode_self_attn_kernel<false>, (N * H + warps - 1) / warps, warps * 32, smem, st, (const bf16*)q,
                            (const bf16*)kv_cache, anc, nullptr, N, H, hd, T, scale, (bf16*)out));
  return 0;
}

extern "C" int esp_decode_self_attn_paths(const void* q, const void* kv_cache, const int32_t* cells, const int32_t* len,
                                          int32_t slots, int32_t N, int32_t H, int32_t hd, float scale, void* out, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(slots >= 1 && slots <= kMaxKeys && hd % 2 == 0, "decode self-attention over paths: bad shape (slots=%d)", slots);
  if (N == 0) return 0;
  const int warps = 4;
  const size_t smem = (size_t)warps * kMaxKeys * sizeof(float);
  ESP_CUDA(esp_launch_plain(decode_self_attn_kernel<true>, (N * H + warps - 1) / warps, warps * 32, smem, st, (const bf16*)q,
                            (const bf16*)kv_cache, cells, len, N, H, hd, 0, scale, (bf16*)out));
  return 0;
}

extern "C" int esp_decode_cross_attn(const void* q, const void* kv, const int32_t* lens, int32_t N, int32_t beam, int32_t H,
                                     int32_t hd, int32_t Tk, float scale, void* out, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(Tk >= 1 && Tk <= kMaxKeys && hd % 2 == 0 && beam >= 1, "decode cross-attention: bad shape (Tk=%d)", Tk);
  if (N == 0) return 0;
  const int warps = 4;
  const size_t smem = (size_t)warps * kMaxKeys * sizeof(float);
  ESP_CUDA(esp_launch_plain(decode_cross_attn_kernel<false>, (N * H + warps - 1) / warps, warps * 32, smem, st, (const bf16*)q,
                            (const bf16*)kv, lens, N, beam, H, hd, Tk, scale, (bf16*)out, nullptr));
  return 0;
}

extern "C" int esp_decode_cross_attn_weights(const void* q, const void* kv, const int32_t* lens, int32_t N, int32_t beam, int32_t H,
                                             int32_t hd, int32_t Tk, float scale, void* out, float* weights, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(Tk >= 1 && Tk <= kMaxKeys && hd % 2 == 0 && beam >= 1, "decode cross-attention: bad shape (Tk=%d)", Tk);
  ESP_CHECK(H >= 1 && H <= 32 && weights, "decode cross-attention weights: need 1 <= H <= 32 and a weights buffer (H=%d)", H);
  if (N == 0) return 0;
  const size_t smem = (size_t)H * kMaxKeys * sizeof(float);  // up to 160 KB at H = 32
  ESP_SMEM_OPTIN(decode_cross_attn_kernel<true>, smem);
  ESP_CUDA(esp_launch_plain(decode_cross_attn_kernel<true>, N, H * 32, smem, st, (const bf16*)q, (const bf16*)kv, lens, N, beam,
                            H, hd, Tk, scale, (bf16*)out, weights));
  return 0;
}

extern "C" int esp_decode_update_ancestry(const int32_t* anc_in, int32_t* anc_out, const int32_t* new_order, int32_t N,
                                          int32_t step, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (N == 0) return 0;
  const long total = (long)(step + 1) * N;
  ESP_CUDA(esp_launch_plain(update_ancestry_kernel, (unsigned)((total + 255) / 256), 256, 0, st, anc_in, anc_out, new_order, N,
                            step));
  return 0;
}

extern "C" int esp_decode_update_paths(const int32_t* cells_in, const int32_t* len_in, int32_t* cells_out, int32_t* len_out,
                                       int32_t* pos_out, const int32_t* new_order, const int32_t* grown, int32_t slot, int32_t N,
                                       void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(slot >= 0 && cells_in != cells_out && len_in != len_out && new_order && grown,
            "decode_update_paths: need slot >= 0, separate in / out tables, new_order and grown (slot=%d)", slot);
  if (N == 0) return 0;
  const long total = (long)(slot + 1) * N;
  ESP_CUDA(esp_launch_plain(update_paths_kernel, (unsigned)((total + 255) / 256), 256, 0, st, cells_in, len_in, cells_out, len_out,
                            pos_out, new_order, grown, N, slot));
  return 0;
}
