// espresso_b200 -- CTC loss forward + backward fused with the fp32 log-softmax.
//
// Replaces (espresso/criterions/ctc_loss.py:59-103):
//   lprobs = model.get_normalized_probs(net_output, log_probs=True)   # fp32 [T',B,V] materialised
//   F.ctc_loss(lprobs, targets, in_lens, tgt_lens, blank, reduction="sum", zero_infinity)
// and its autograd backward through log_softmax.  The fp32 [T',B,V] log-prob tensor and its fp32
// gradient are never written: three kernels touch HBM with
//   prep : read logits once            -> row log-sum-exp + emissions gathered at the 2U+1 extended labels
//   scan : alpha (warp 0) and beta (warp 1) recursions per utterance, states in registers,
//          neighbour states by warp shuffle (no block barriers on the serial path)
//   grad : read logits again, write d(loss)/d(logits) = softmax - occupancy   (bf16)
// => algorithmic bytes 6*V per encoder frame (SURVEY.md §8d).
#include "common.cuh"
#include "espresso_b200.h"
#include <math.h>

namespace {

constexpr float kNegInf = -INFINITY;

__device__ __forceinline__ float lse2(float a, float b) {
  const float m = fmaxf(a, b);
  if (m == kNegInf) return kNegInf;
  return m + logf(__expf(a - m) + __expf(b - m));
}
// branch-free 3-term logsumexp for the scan's serial chain (c = -inf when the skip transition is not allowed);
// ex2/lg2.approx: ~1e-7 relative per step, far inside the loss tolerance
__device__ __forceinline__ float lse3_fast(float a, float b, float c) {
  const float hi = fmaxf(a, b), lo = fminf(a, b);
  const float m = fmaxf(hi, c), mid = fminf(hi, c);  // the largest term contributes exactly 1
  const float mm = (m == kNegInf) ? 0.f : m;
  const float r = mm + __logf(1.f + __expf(mid - mm) + __expf(lo - mm));
  return (m == kNegInf) ? kNegInf : r;
}

// ---- prep: row LSE + emissions at extended labels ------------------------------------------------
constexpr int kPrepThreads = 256;
constexpr int kPrepCache = 4;  // uint4 (8 bf16) per thread cached in registers: V <= 256*4*8 = 8192

__global__ void __launch_bounds__(kPrepThreads)
ctc_prep_kernel(const bf16* __restrict__ logits, long stride_b, long stride_t, int V, int t_max,
                const int* __restrict__ in_lens, const int* __restrict__ targets, int u_max,
                const int* __restrict__ tgt_lens, int blank, float* __restrict__ lse_out,
                float* __restrict__ lp_ext, int s_max) {
  esp_pdl();
  __shared__ float red[32];
  const int b = blockIdx.y, t = blockIdx.x;
  if (t >= in_lens[b]) return;
  const bf16* row = logits + (long)b * stride_b + (long)t * stride_t;
  const bool vec_ok = ((((uintptr_t)row) & 15) == 0);
  const int nvec = vec_ok ? V / 8 : 0;
  uint4 cache[kPrepCache];
  float mx = kNegInf;
#pragma unroll
  for (int i = 0; i < kPrepCache; ++i) {
    const int vi = threadIdx.x + i * kPrepThreads;
    if (vi < nvec) {
      cache[i] = *reinterpret_cast<const uint4*>(row + vi * 8);
      float a, c;
      unpack_bf16x2(cache[i].x, a, c); mx = fmaxf(mx, fmaxf(a, c));
      unpack_bf16x2(cache[i].y, a, c); mx = fmaxf(mx, fmaxf(a, c));
      unpack_bf16x2(cache[i].z, a, c); mx = fmaxf(mx, fmaxf(a, c));
      unpack_bf16x2(cache[i].w, a, c); mx = fmaxf(mx, fmaxf(a, c));
    }
  }
  for (int vi = threadIdx.x + kPrepCache * kPrepThreads; vi < nvec; vi += kPrepThreads) {
    const uint4 q = *reinterpret_cast<const uint4*>(row + vi * 8);
    float a, c;
    unpack_bf16x2(q.x, a, c); mx = fmaxf(mx, fmaxf(a, c));
    unpack_bf16x2(q.y, a, c); mx = fmaxf(mx, fmaxf(a, c));
    unpack_bf16x2(q.z, a, c); mx = fmaxf(mx, fmaxf(a, c));
    unpack_bf16x2(q.w, a, c); mx = fmaxf(mx, fmaxf(a, c));
  }
  for (int v = nvec * 8 + threadIdx.x; v < V; v += kPrepThreads) mx = fmaxf(mx, bf2f(row[v]));
  mx = block_max<kPrepThreads>(mx, red);
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < kPrepCache; ++i) {
    const int vi = threadIdx.x + i * kPrepThreads;
    if (vi < nvec) {
      float a, c;
      unpack_bf16x2(cache[i].x, a, c); sum += __expf(a - mx) + __expf(c - mx);
      unpack_bf16x2(cache[i].y, a, c); sum += __expf(a - mx) + __expf(c - mx);
      unpack_bf16x2(cache[i].z, a, c); sum += __expf(a - mx) + __expf(c - mx);
      unpack_bf16x2(cache[i].w, a, c); sum += __expf(a - mx) + __expf(c - mx);
    }
  }
  for (int vi = threadIdx.x + kPrepCache * kPrepThreads; vi < nvec; vi += kPrepThreads) {
    const uint4 q = *reinterpret_cast<const uint4*>(row + vi * 8);
    float a, c;
    unpack_bf16x2(q.x, a, c); sum += __expf(a - mx) + __expf(c - mx);
    unpack_bf16x2(q.y, a, c); sum += __expf(a - mx) + __expf(c - mx);
    unpack_bf16x2(q.z, a, c); sum += __expf(a - mx) + __expf(c - mx);
    unpack_bf16x2(q.w, a, c); sum += __expf(a - mx) + __expf(c - mx);
  }
  for (int v = nvec * 8 + threadIdx.x; v < V; v += kPrepThreads) sum += __expf(bf2f(row[v]) - mx);
  sum = block_sum<kPrepThreads>(sum, red);
  const float lse = mx + logf(sum);
  if (threadIdx.x == 0) lse_out[(long)b * t_max + t] = lse;
  const int U = tgt_lens[b];
  const int S = 2 * U + 1;
  float* dst = lp_ext + ((long)b * t_max + t) * s_max;
  for (int s = threadIdx.x; s < S; s += kPrepThreads) {
    const int lab = (s & 1) ? targets[(long)b * u_max + (s >> 1)] : blank;
    dst[s] = bf2f(row[lab]) - lse;
  }
}

// ---- scan: alpha / beta recursions -----------------------------------------------------------------
// One CTA per utterance; threads [0, G) run alpha (t ascending), threads [G, 2G) run beta (t descending), C
// consecutive states per thread (C = 1 up to 512 extended states).  A time step of one direction is: publish the
// current column to shared memory (double-buffered by step parity), one named barrier over the G threads of that
// direction, read the two neighbours, one 3-term logsumexp.  The serial chain per step is therefore ~one barrier +
// one logsumexp regardless of the target length; emission rows are prefetched kScanDepth steps ahead.
constexpr int kScanDepth = 4;

__device__ __forceinline__ void group_barrier(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

template <int C>
__global__ void __launch_bounds__(1024)
ctc_scan_kernel(const float* __restrict__ lp_ext, float* __restrict__ alpha, float* __restrict__ beta,
                int t_max, int s_max, const int* __restrict__ in_lens, const int* __restrict__ targets,
                int u_max, const int* __restrict__ tgt_lens, int blank, float* __restrict__ nll, int G) {
  esp_pdl();
  extern __shared__ float scan_sh[];  // [2 directions][2 parities][G*C + 4]
  const int b = blockIdx.x;
  const int dir = threadIdx.x >= G;  // 0 alpha, 1 beta
  const int tid = threadIdx.x - dir * G;
  const int T = in_lens[b];
  const int U = tgt_lens[b];
  const int S = 2 * U + 1;
  if (T <= 0) {
    if (threadIdx.x == 0) nll[b] = (U == 0) ? 0.f : INFINITY;
    return;
  }
  const int W = G * C + 4;  // column buffer: 2 pad cells (-inf) on each side
  float* buf0 = scan_sh + dir * 2 * W;
  float* buf1 = buf0 + W;
  if (tid < 2) {
    buf0[tid] = kNegInf; buf0[W - 1 - tid] = kNegInf;
    buf1[tid] = kNegInf; buf1[W - 1 - tid] = kNegInf;
  }
  const long base = (long)b * t_max * s_max;
  const int s0 = tid * C;
  const float* lp = lp_ext + base;
  // which states may take the s-2 (alpha) / s+2 (beta) skip transition
  bool skip[C], live[C];
#pragma unroll
  for (int i = 0; i < C; ++i) {
    const int s = s0 + i;
    live[i] = s < S;
    skip[i] = false;
    if ((s & 1) && s < S) {
      const int u = s >> 1;
      if (dir == 0) {
        if (u >= 1) skip[i] = targets[(long)b * u_max + u] != targets[(long)b * u_max + u - 1];
      } else {
        if (u + 1 < U) skip[i] = targets[(long)b * u_max + u] != targets[(long)b * u_max + u + 1];
      }
    }
  }
  float cur[C], pre[kScanDepth][C];
  float* out = (dir == 0 ? alpha : beta) + base;
  const int tstart = dir == 0 ? 0 : T - 1;
  const int tstep = dir == 0 ? 1 : -1;
  // t = tstart: initial column
#pragma unroll
  for (int i = 0; i < C; ++i) {
    const int s = s0 + i;
    const bool init = dir == 0 ? (s < 2) : (s >= S - 2);
    cur[i] = (live[i] && init) ? lp[(long)tstart * s_max + s] : kNegInf;
    if (live[i]) out[(long)tstart * s_max + s] = cur[i];
  }
#pragma unroll
  for (int d = 0; d < kScanDepth; ++d) {
    const int t = tstart + tstep * (1 + d);
#pragma unroll
    for (int i = 0; i < C; ++i) pre[d][i] = (live[i] && t >= 0 && t < T) ? lp[(long)t * s_max + s0 + i] : 0.f;
  }
  int par = 0;
  for (int n0 = 1; n0 < T; n0 += kScanDepth) {
#pragma unroll
    for (int d = 0; d < kScanDepth; ++d) {
      const int n = n0 + d;  // step count from the start; CTA-uniform
      if (n < T) {
        const int t = tstart + tstep * n;
        float em[C];
#pragma unroll
        for (int i = 0; i < C; ++i) em[i] = pre[d][i];
        const int tn = t + tstep * kScanDepth;
        if (n + kScanDepth < T) {
#pragma unroll
          for (int i = 0; i < C; ++i)
            if (live[i]) pre[d][i] = lp[(long)tn * s_max + s0 + i];
        }
        float* bufp = par ? buf1 : buf0;
#pragma unroll
        for (int i = 0; i < C; ++i) bufp[2 + s0 + i] = cur[i];
        group_barrier(1 + dir, G);
        float nw[C];
#pragma unroll
        for (int i = 0; i < C; ++i) {
          // alpha: neighbours s-1, s-2 ; beta: s+1, s+2 (pad cells hold -inf)
          const int q = 2 + s0 + i;
          const float n1 = dir == 0 ? bufp[q - 1] : bufp[q + 1];
          const float n2 = dir == 0 ? bufp[q - 2] : bufp[q + 2];
          const float acc = lse3_fast(cur[i], n1, skip[i] ? n2 : kNegInf);
          nw[i] = live[i] ? acc + em[i] : kNegInf;
        }
#pragma unroll
        for (int i = 0; i < C; ++i) {
          cur[i] = nw[i];
          if (live[i]) out[(long)t * s_max + s0 + i] = cur[i];
        }
        par ^= 1;
      }
    }
  }
  if (dir == 0) {
    // nll = -logsumexp(alpha_{T-1}(S-1), alpha_{T-1}(S-2))
    float* bufp = par ? buf1 : buf0;
#pragma unroll
    for (int i = 0; i < C; ++i) bufp[2 + s0 + i] = cur[i];
    group_barrier(1, G);
    if (tid == 0) nll[b] = -lse2(bufp[2 + S - 1], S >= 2 ? bufp[2 + S - 2] : kNegInf);
  }
}

// ---- grad: softmax - occupancy ------------------------------------------------------------------
constexpr int kGradThreads = 256;

__global__ void __launch_bounds__(kGradThreads)
ctc_grad_kernel(const bf16* __restrict__ logits, long stride_b, long stride_t, int V, int ld_pad, int t_max,
                const int* __restrict__ in_lens, const int* __restrict__ targets, int u_max,
                const int* __restrict__ tgt_lens, int blank, int zero_infinity, float grad_scale,
                const float* __restrict__ lse_in, const float* __restrict__ lp_ext,
                const float* __restrict__ alpha, const float* __restrict__ beta, const float* __restrict__ nll,
                int s_max, bf16* __restrict__ grad) {
  esp_pdl();
  extern __shared__ float occ[];
  const int b = blockIdx.y, t = blockIdx.x;
  bf16* grow = grad + (long)b * stride_b + (long)t * stride_t;
  const float loss = nll[b];
  const bool dead = (t >= in_lens[b]) || isinf(loss) || isnan(loss);
  if (dead) {
    for (int v = threadIdx.x; v < ld_pad; v += kGradThreads) grow[v] = f2bf(0.f);
    return;
  }
  for (int v = threadIdx.x; v < V; v += kGradThreads) occ[v] = 0.f;
  __syncthreads();
  const int S = 2 * tgt_lens[b] + 1;
  const long off = ((long)b * t_max + t) * s_max;
  for (int s = threadIdx.x; s < S; s += kGradThreads) {
    const float lab_lp = lp_ext[off + s];
    const float ab = alpha[off + s] + beta[off + s];
    if (ab != kNegInf) {
      const int lab = (s & 1) ? targets[(long)b * u_max + (s >> 1)] : blank;
      atomicAdd(&occ[lab], __expf(ab - lab_lp + loss));
    }
  }
  __syncthreads();
  const bf16* row = logits + (long)b * stride_b + (long)t * stride_t;
  const float lse = lse_in[(long)b * t_max + t];
  const bool vec_ok = (ld_pad % 8 == 0) && (((stride_b | stride_t) & 7) == 0) &&
                      ((reinterpret_cast<uintptr_t>(logits) | reinterpret_cast<uintptr_t>(grad)) & 15) == 0;
  if (vec_ok) {
    // 16-byte path: 8 vocabulary entries per thread and iteration
    for (int v0 = threadIdx.x * 8; v0 < ld_pad; v0 += kGradThreads * 8) {
      const uint4 q = *reinterpret_cast<const uint4*>(row + v0);
      float x[8];
      unpack_bf16x2(q.x, x[0], x[1]);
      unpack_bf16x2(q.y, x[2], x[3]);
      unpack_bf16x2(q.z, x[4], x[5]);
      unpack_bf16x2(q.w, x[6], x[7]);
#pragma unroll
      for (int j = 0; j < 8; ++j) x[j] = (v0 + j < V) ? (__expf(x[j] - lse) - occ[v0 + j]) * grad_scale : 0.f;
      uint4 o;
      o.x = pack_bf16x2(x[0], x[1]);
      o.y = pack_bf16x2(x[2], x[3]);
      o.z = pack_bf16x2(x[4], x[5]);
      o.w = pack_bf16x2(x[6], x[7]);
      *reinterpret_cast<uint4*>(grow + v0) = o;
    }
    return;
  }
  for (int v = threadIdx.x; v < ld_pad; v += kGradThreads) {
    float g = 0.f;
    if (v < V) g = (__expf(bf2f(row[v]) - lse) - occ[v]) * grad_scale;
    grow[v] = f2bf(g);
  }
}

__global__ void ctc_finalize_kernel(const float* __restrict__ nll, int B, int zero_infinity, float* __restrict__ loss) {
  esp_pdl();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float l = nll[b];
  if (zero_infinity && (isinf(l) || isnan(l))) l = 0.f;
  loss[b] = l;
}

}  // namespace

extern "C" int64_t esp_ctc_workspace_bytes(int32_t B, int32_t t_max, int32_t u_max) {
  const long s_max = (2L * u_max + 1 + 3) / 4 * 4;  // rows padded to 16 bytes for vector access
  const long cells = (long)B * t_max * s_max;
  return align256((long)B * t_max * 4) + 3 * align256(cells * 4) + align256((long)B * 4);
}

extern "C" int esp_ctc_loss(const void* logits, int64_t stride_b, int64_t stride_t, int32_t V, int32_t B,
                            int32_t t_max, const int32_t* in_lens, const int32_t* targets, int32_t u_max,
                            const int32_t* tgt_lens, int32_t blank, int32_t zero_infinity, float grad_scale,
                            float* loss, void* grad, void* workspace, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(B >= 0 && t_max >= 0 && u_max >= 0 && V > 0, "bad CTC shape");
  if (B == 0) return 0;
  ESP_CHECK(logits && in_lens && tgt_lens && loss && workspace, "null pointer passed to esp_ctc_loss");
  ESP_CHECK(u_max == 0 || targets != nullptr, "targets is null");
  ESP_CHECK(blank >= 0 && blank < V, "blank index out of range");
  const int s_max = (2 * u_max + 1 + 3) / 4 * 4;  // rows padded to 16 bytes for vector access
  ESP_CHECK(s_max <= 32 * 32, "CTC target too long for the register scan (u_max=%d > 511)", u_max);
  char* ws = (char*)workspace;
  float* lse = (float*)ws; ws += align256((long)B * t_max * 4);
  const long cells = (long)B * t_max * s_max;
  float* lp_ext = (float*)ws; ws += align256(cells * 4);
  float* alpha = (float*)ws; ws += align256(cells * 4);
  float* beta = (float*)ws; ws += align256(cells * 4);
  float* nll = (float*)ws;
  if (t_max > 0)
    ESP_CUDA(esp_launch(ctc_prep_kernel, dim3(t_max, B), kPrepThreads, 0, st, (const bf16*)logits, stride_b, stride_t, V, t_max,
                        in_lens, targets, u_max, tgt_lens, blank, lse, lp_ext, s_max));
  {
    const int C = s_max > 512 ? 2 : 1;
    int G = ((s_max + C - 1) / C + 31) / 32 * 32;
    if (G > 512) G = 512;
    const size_t smem = (size_t)4 * (G * C + 4) * sizeof(float);
    if (C == 1)
      ESP_CUDA(esp_launch(ctc_scan_kernel<1>, B, 2 * G, smem, st, lp_ext, alpha, beta, t_max, s_max, in_lens, targets, u_max,
                          tgt_lens, blank, nll, G));
    else
      ESP_CUDA(esp_launch(ctc_scan_kernel<2>, B, 2 * G, smem, st, lp_ext, alpha, beta, t_max, s_max, in_lens, targets, u_max,
                          tgt_lens, blank, nll, G));
  }
  ESP_CUDA(esp_launch(ctc_finalize_kernel, (B + 127) / 128, 128, 0, st, nll, B, zero_infinity, loss));
  if (grad && t_max > 0) {
    // padded row width: rows are written up to the next multiple of 8 when the row stride leaves room
    long min_stride = stride_t < stride_b ? stride_t : stride_b;
    int ld_pad = V;
    if (B == 1 && t_max > 1) min_stride = stride_t;
    if (t_max == 1 && B > 1) min_stride = stride_b;
    const int v8 = (V + 7) / 8 * 8;
    if (min_stride >= v8) ld_pad = v8;
    ESP_CHECK((size_t)V * 4 <= 200 * 1024, "vocabulary too large for the CTC gradient kernel");
    ESP_SMEM_OPTIN(ctc_grad_kernel, (size_t)V * 4);
    ESP_CUDA(esp_launch(ctc_grad_kernel, dim3(t_max, B), kGradThreads, V * 4, st, (const bf16*)logits, stride_b, stride_t, V,
                        ld_pad, t_max, in_lens, targets, u_max, tgt_lens, blank, zero_infinity, grad_scale, lse, lp_ext, alpha,
                        beta, nll, s_max, (bf16*)grad));
  }
  return 0;
}
