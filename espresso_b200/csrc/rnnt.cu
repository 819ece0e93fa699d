// espresso_b200 -- RNN-T (transducer) loss fused with the log-softmax, and the joint network's broadcast stage.
//
// Replaces espresso/criterions/transducer_loss.py:130-140  torchaudio.functional.rnnt_loss(logits [B,T,U+1,V],
// targets, T-lens, U-lens, blank, clamp=-1, fused_log_softmax=True, reduction="sum") and its backward, and
// espresso/models/transformer/speech_transformer_transducer_base.py:279-299  joint():
//   relu(LN(W_e enc)[:, :, None, :] + LN(W_d dec)[:, None, :, :]).
// Loss kernels:
//   prep : one CTA per lattice cell (b,t,u): row log-sum-exp over V, emits lp_blank and lp_label (2 floats/cell);
//          logits are read once                                                            (2*V bytes / cell)
//   scan : alpha and beta over the (T,U) lattice by anti-diagonal wavefronts, one CTA per utterance and direction,
//          previous diagonal kept in shared memory (log-domain)
//   grad : d(loss)/d(logits)[v] = softmax_v * exp(alpha+beta-ll) - [v=blank] exp(alpha+beta(t+1,u)+lp_blank-ll)
//                                                               - [v=y_u+1] exp(alpha+beta(t,u+1)+lp_label-ll)
//          logits read again, gradient written once                                         (4*V bytes / cell)
// => 6*V bytes per lattice cell (SURVEY.md §8d); the fp32 [B,T,U+1,V] log-prob tensor is never materialised.
#include "common.cuh"
#include "espresso_b200.h"
#include <math.h>

namespace {

constexpr float kNegInf = -INFINITY;
constexpr int kT = 256;

__device__ __forceinline__ float lae(float a, float b) {
  const float m = fmaxf(a, b);
  if (m == kNegInf) return kNegInf;
  return m + logf(expf(a - m) + expf(b - m));
}

// grid (U1, T, B)
__global__ void __launch_bounds__(kT)
rnnt_prep_kernel(const bf16* __restrict__ logits, long ld, int V, int T, int U1, const int* __restrict__ t_lens,
                 const int* __restrict__ u_lens, const int* __restrict__ targets, int u_max, int blank,
                 float* __restrict__ lse_out, float* __restrict__ lpb, float* __restrict__ lpl) {
  __shared__ float red[32];
  const int u = blockIdx.x, t = blockIdx.y, b = blockIdx.z;
  if (t >= t_lens[b] || u > u_lens[b]) return;
  const long cell = ((long)b * T + t) * U1 + u;
  const bf16* row = logits + cell * ld;
  const int nvec = V / 8;
  float mx = kNegInf;
  for (int vi = threadIdx.x; vi < nvec; vi += kT) {
    const uint4 q = *reinterpret_cast<const uint4*>(row + vi * 8);
    float a, c;
    unpack_bf16x2(q.x, a, c); mx = fmaxf(mx, fmaxf(a, c));
    unpack_bf16x2(q.y, a, c); mx = fmaxf(mx, fmaxf(a, c));
    unpack_bf16x2(q.z, a, c); mx = fmaxf(mx, fmaxf(a, c));
    unpack_bf16x2(q.w, a, c); mx = fmaxf(mx, fmaxf(a, c));
  }
  for (int v = nvec * 8 + threadIdx.x; v < V; v += kT) mx = fmaxf(mx, bf2f(row[v]));
  mx = block_max<kT>(mx, red);
  float s = 0.f;
  for (int vi = threadIdx.x; vi < nvec; vi += kT) {
    const uint4 q = *reinterpret_cast<const uint4*>(row + vi * 8);
    float a, c;
    unpack_bf16x2(q.x, a, c); s += expf(a - mx) + expf(c - mx);
    unpack_bf16x2(q.y, a, c); s += expf(a - mx) + expf(c - mx);
    unpack_bf16x2(q.z, a, c); s += expf(a - mx) + expf(c - mx);
    unpack_bf16x2(q.w, a, c); s += expf(a - mx) + expf(c - mx);
  }
  for (int v = nvec * 8 + threadIdx.x; v < V; v += kT) s += expf(bf2f(row[v]) - mx);
  s = block_sum<kT>(s, red);
  if (threadIdx.x == 0) {
    const float lse = mx + logf(s);
    lse_out[cell] = lse;
    lpb[cell] = bf2f(row[blank]) - lse;
    lpl[cell] = (u < u_lens[b]) ? bf2f(row[targets[(long)b * u_max + u]]) - lse : kNegInf;
  }
}

// grid (B, 2): y = 0 alpha, y = 1 beta.  Anti-diagonal wavefront; thread <-> u.
__global__ void __launch_bounds__(kT)
rnnt_scan_kernel(const float* __restrict__ lpb, const float* __restrict__ lpl, int T, int U1, const int* __restrict__ t_lens,
                 const int* __restrict__ u_lens, float* __restrict__ alpha, float* __restrict__ beta, float* __restrict__ ll) {
  extern __shared__ float sm[];  // [2][U1] previous / current diagonal
  const int b = blockIdx.x;
  const int Tb = t_lens[b], Ub = u_lens[b] + 1;  // lattice is Tb x Ub
  const long base = (long)b * T * U1;
  if (Tb <= 0) {
    if (blockIdx.y == 0 && threadIdx.x == 0) ll[b] = kNegInf;
    return;
  }
  float* prev = sm;
  float* cur = sm + U1;
  const int ndiag = Tb + Ub - 1;
  if (blockIdx.y == 0) {
    for (int dg = 0; dg < ndiag; ++dg) {
      for (int u = threadIdx.x; u < Ub; u += kT) {
        const int t = dg - u;
        if (t < 0 || t >= Tb) continue;
        float a;
        if (t == 0 && u == 0) a = 0.f;
        else {
          const float up = (t > 0) ? prev[u] + lpb[base + (long)(t - 1) * U1 + u] : kNegInf;        // from (t-1,u) by blank
          const float left = (u > 0) ? prev[u - 1] + lpl[base + (long)t * U1 + u - 1] : kNegInf;    // from (t,u-1) by label
          a = lae(up, left);
        }
        cur[u] = a;
        alpha[base + (long)t * U1 + u] = a;
      }
      __syncthreads();
      float* tmp = prev; prev = cur; cur = tmp;
    }
    if (threadIdx.x == 0) ll[b] = alpha[base + (long)(Tb - 1) * U1 + Ub - 1] + lpb[base + (long)(Tb - 1) * U1 + Ub - 1];
  } else {
    for (int dg = ndiag - 1; dg >= 0; --dg) {
      for (int u = threadIdx.x; u < Ub; u += kT) {
        const int t = dg - u;
        if (t < 0 || t >= Tb) continue;
        float v;
        if (t == Tb - 1 && u == Ub - 1) v = lpb[base + (long)t * U1 + u];
        else {
          const float down = (t + 1 < Tb) ? prev[u] + lpb[base + (long)t * U1 + u] : kNegInf;       // to (t+1,u)
          const float right = (u + 1 < Ub) ? prev[u + 1] + lpl[base + (long)t * U1 + u] : kNegInf;  // to (t,u+1)
          v = lae(down, right);
        }
        cur[u] = v;
        beta[base + (long)t * U1 + u] = v;
      }
      __syncthreads();
      float* tmp = prev; prev = cur; cur = tmp;
    }
  }
}

// grid (U1, T, B)
__global__ void __launch_bounds__(kT)
rnnt_grad_kernel(const bf16* __restrict__ logits, long ld, int V, int T, int U1, const int* __restrict__ t_lens,
                 const int* __restrict__ u_lens, const int* __restrict__ targets, int u_max, int blank,
                 const float* __restrict__ lse_in, const float* __restrict__ lpb, const float* __restrict__ lpl,
                 const float* __restrict__ alpha, const float* __restrict__ beta, const float* __restrict__ ll,
                 float grad_scale, bf16* __restrict__ grad) {
  const int u = blockIdx.x, t = blockIdx.y, b = blockIdx.z;
  const long cell = ((long)b * T + t) * U1 + u;
  bf16* g = grad + cell * ld;
  const int ldp = (int)(ld < (long)((V + 7) / 8 * 8) ? ld : (V + 7) / 8 * 8);
  const int Tb = t_lens[b], Ub = u_lens[b];
  const float L = ll[b];
  if (t >= Tb || u > Ub || !(L > kNegInf) || L != L) {
    for (int v = threadIdx.x; v < ldp; v += kT) g[v] = f2bf(0.f);
    return;
  }
  const long base = (long)b * T * U1;
  const float a = alpha[cell], be = beta[cell];
  const float occ = expf(a + be - L);                                  // sum over both outgoing arcs
  const float nb = (t + 1 < Tb) ? beta[base + (long)(t + 1) * U1 + u] : ((u == Ub) ? 0.f : kNegInf);
  const float gb = expf(a + nb + lpb[cell] - L);                       // blank arc
  const float gl = (u < Ub) ? expf(a + beta[base + (long)t * U1 + u + 1] + lpl[cell] - L) : 0.f;  // label arc
  const int lab = (u < Ub) ? targets[(long)b * u_max + u] : -1;
  const float lse = lse_in[cell];
  const bf16* row = logits + cell * ld;
  for (int v = threadIdx.x; v < ldp; v += kT) {
    float gv = 0.f;
    if (v < V) {
      gv = expf(bf2f(row[v]) - lse) * occ;
      if (v == blank) gv -= gb;
      if (v == lab) gv -= gl;
      gv *= grad_scale;
    }
    g[v] = f2bf(gv);
  }
}

__global__ void rnnt_finalize_kernel(const float* __restrict__ ll, int B, float* __restrict__ loss) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) loss[b] = -ll[b];
}

// F[b,t,u,:] = relu(e[b,t,:] + d[b,u,:])
__global__ void __launch_bounds__(256)
joint_fwd_kernel(const bf16* __restrict__ e, const bf16* __restrict__ d, int B, int T, int U1, int J, bf16* __restrict__ f) {
  const long nvec = (long)B * T * U1 * (J >> 3);
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % (J >> 3)) * 8;
    const long cell = i / (J >> 3);
    const int u = (int)(cell % U1);
    const long bt = cell / U1;
    const int b = (int)(bt / T);
    const uint4 qa = *reinterpret_cast<const uint4*>(e + bt * J + c);
    const uint4 qb = *reinterpret_cast<const uint4*>(d + ((long)b * U1 + u) * J + c);
    float x[8], y[8];
    unpack_bf16x2(qa.x, x[0], x[1]); unpack_bf16x2(qa.y, x[2], x[3]); unpack_bf16x2(qa.z, x[4], x[5]); unpack_bf16x2(qa.w, x[6], x[7]);
    unpack_bf16x2(qb.x, y[0], y[1]); unpack_bf16x2(qb.y, y[2], y[3]); unpack_bf16x2(qb.z, y[4], y[5]); unpack_bf16x2(qb.w, y[6], y[7]);
    uint4 o;
    o.x = pack_bf16x2(fmaxf(x[0] + y[0], 0.f), fmaxf(x[1] + y[1], 0.f));
    o.y = pack_bf16x2(fmaxf(x[2] + y[2], 0.f), fmaxf(x[3] + y[3], 0.f));
    o.z = pack_bf16x2(fmaxf(x[4] + y[4], 0.f), fmaxf(x[5] + y[5], 0.f));
    o.w = pack_bf16x2(fmaxf(x[6] + y[6], 0.f), fmaxf(x[7] + y[7], 0.f));
    *reinterpret_cast<uint4*>(f + i * 8) = o;
  }
}

// de[b,t,:] = sum_u dF*(F>0) ; dd[b,u,:] += sum_t dF*(F>0)  (dd fp32 via atomics, de written directly)
// grid (T, B), block = J/8 x 8... one thread per 8 channels, loops over u.
__global__ void __launch_bounds__(256)
joint_bwd_kernel(const bf16* __restrict__ df, const bf16* __restrict__ f, int B, int T, int U1, int J, bf16* __restrict__ de,
                 float* __restrict__ dd) {
  const int t = blockIdx.x, b = blockIdx.y;
  const long bt = (long)b * T + t;
  for (int cv = threadIdx.x; cv < (J >> 3); cv += blockDim.x) {
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int u = 0; u < U1; ++u) {
      const long off = (bt * U1 + u) * J + cv * 8;
      const uint4 qg = *reinterpret_cast<const uint4*>(df + off);
      const uint4 qf = *reinterpret_cast<const uint4*>(f + off);
      float g[8], x[8];
      unpack_bf16x2(qg.x, g[0], g[1]); unpack_bf16x2(qg.y, g[2], g[3]); unpack_bf16x2(qg.z, g[4], g[5]); unpack_bf16x2(qg.w, g[6], g[7]);
      unpack_bf16x2(qf.x, x[0], x[1]); unpack_bf16x2(qf.y, x[2], x[3]); unpack_bf16x2(qf.z, x[4], x[5]); unpack_bf16x2(qf.w, x[6], x[7]);
      float* ddp = dd + ((long)b * U1 + u) * J + cv * 8;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float v = x[j] > 0.f ? g[j] : 0.f;
        acc[j] += v;
        if (v != 0.f) atomicAdd(ddp + j, v);
      }
    }
    uint4 o;
    o.x = pack_bf16x2(acc[0], acc[1]);
    o.y = pack_bf16x2(acc[2], acc[3]);
    o.z = pack_bf16x2(acc[4], acc[5]);
    o.w = pack_bf16x2(acc[6], acc[7]);
    *reinterpret_cast<uint4*>(de + bt * J + cv * 8) = o;
  }
}

}  // namespace

extern "C" int64_t esp_rnnt_workspace_bytes(int32_t B, int32_t T, int32_t U1) {
  const long cells = (long)B * T * U1;
  return 5 * align256(cells * 4) + align256((long)B * 4);
}

extern "C" int esp_rnnt_loss(const void* logits, int64_t ld, int32_t V, int32_t B, int32_t T, int32_t U1, const int32_t* t_lens,
                             const int32_t* u_lens, const int32_t* targets, int32_t u_max, int32_t blank, float grad_scale,
                             float* loss, void* grad, void* workspace, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(B >= 0 && T >= 1 && U1 >= 1 && V > 1 && ld >= V && ld % 8 == 0, "bad RNN-T shape");
  ESP_CHECK(logits && t_lens && u_lens && loss && workspace, "null pointer passed to esp_rnnt_loss");
  ESP_CHECK(((uintptr_t)logits & 15) == 0, "esp_rnnt_loss needs 16-byte aligned logits (rows are read as 16-byte vectors)");
  ESP_CHECK(U1 * 2 * 4 <= 48 * 1024, "RNN-T target too long for the wavefront scan");
  if (B == 0) return 0;
  const long cells = (long)B * T * U1;
  char* ws = (char*)workspace;
  float* lse = (float*)ws; ws += align256(cells * 4);
  float* lpb = (float*)ws; ws += align256(cells * 4);
  float* lpl = (float*)ws; ws += align256(cells * 4);
  float* alpha = (float*)ws; ws += align256(cells * 4);
  float* beta = (float*)ws; ws += align256(cells * 4);
  float* ll = (float*)ws;
  dim3 grid(U1, T, B);
  ESP_CUDA(esp_launch_plain(rnnt_prep_kernel, grid, kT, 0, st, (const bf16*)logits, ld, V, T, U1, t_lens, u_lens, targets, u_max,
                            blank, lse, lpb, lpl));
  ESP_CUDA(esp_launch_plain(rnnt_scan_kernel, dim3(B, 2), kT, 2 * U1 * sizeof(float), st, lpb, lpl, T, U1, t_lens, u_lens, alpha,
                            beta, ll));
  ESP_CUDA(esp_launch_plain(rnnt_finalize_kernel, (B + 127) / 128, 128, 0, st, ll, B, loss));
  if (grad) {
    ESP_CUDA(esp_launch_plain(rnnt_grad_kernel, grid, kT, 0, st, (const bf16*)logits, ld, V, T, U1, t_lens, u_lens, targets,
                              u_max, blank, lse, lpb, lpl, alpha, beta, ll, grad_scale, (bf16*)grad));
  }
  return 0;
}

extern "C" int esp_joint_fwd(const void* enc, const void* dec, int32_t B, int32_t T, int32_t U1, int32_t J, void* out, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(J % 8 == 0, "joint dim must be a multiple of 8");
  // enc, dec and out are read and written with 16-byte vector accesses
  ESP_CHECK((((uintptr_t)enc | (uintptr_t)dec | (uintptr_t)out) & 15) == 0, "esp_joint_fwd needs 16-byte aligned enc, dec and out");
  const long nvec = (long)B * T * U1 * (J / 8);
  if (nvec == 0) return 0;
  ESP_CUDA(esp_launch_plain(joint_fwd_kernel, grid_for(nvec, 256, 16), 256, 0, st, (const bf16*)enc, (const bf16*)dec, B, T, U1,
                            J, (bf16*)out));
  return 0;
}

extern "C" int esp_joint_bwd(const void* df, const void* f, int32_t B, int32_t T, int32_t U1, int32_t J, void* denc, float* ddec,
                             void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(J % 8 == 0, "joint dim must be a multiple of 8");
  ESP_CHECK(B <= 65535, "esp_joint_bwd launches one CTA row per utterance: B must be at most 65535 (B=%d)", B);
  // df, f and denc are read and written with 16-byte vector accesses
  ESP_CHECK((((uintptr_t)df | (uintptr_t)f | (uintptr_t)denc) & 15) == 0, "esp_joint_bwd needs 16-byte aligned df, f and denc");
  if ((long)B * T * U1 == 0) return 0;
  ESP_CUDA(esp_launch_plain(joint_bwd_kernel, dim3(T, B), (J / 8) < 256 ? ((J / 8 + 31) / 32 * 32) : 256, 0, st, (const bf16*)df,
                            (const bf16*)f, B, T, U1, J, (bf16*)denc, ddec));
  return 0;
}
