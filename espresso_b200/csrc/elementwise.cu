// espresso_b200 -- HBM-bound kernels of the Conformer/Transformer block, forward and backward.
//
//   LayerNorm                fairseq/modules/layer_norm.py (torch.nn.LayerNorm), used at
//                            fairseq/modules/conformer_layer.py:79-81,134-136 and
//                            espresso/modules/conformer_with_relative_positional_embedding_encoder_layer.py:118,143
//   GLU + depthwise conv k   fairseq/modules/conformer_layer.py:88-93   (+ BatchNorm batch statistics)
//   BatchNorm1d + SiLU       fairseq/modules/conformer_layer.py:95-96   (batch stats incl. padded frames)
//   rel-pos softmax          fairseq/modules/multihead_attention.py:841-867 (key-padding -inf, fp32 softmax, dropout)
//   (q+u)*s, (q+v)*s         fairseq/modules/multihead_attention.py:679-688
//   dropout                  torch.nn.Dropout call sites of the modules above (stateless counter RNG)
//   column sums              bias / pos_bias gradients
// All tensors are batch-major [B, T, C] bf16 with fp32 statistics; every kernel reads each input
// element once and writes each output element once (vectorised 16-byte accesses).
#include "common.cuh"
#include "espresso_b200.h"
#include <math.h>

namespace {

__device__ __forceinline__ void load8(const bf16* p, float (&v)[8]) {
  const uint4 q = *reinterpret_cast<const uint4*>(p);
  unpack_bf16x2(q.x, v[0], v[1]);
  unpack_bf16x2(q.y, v[2], v[3]);
  unpack_bf16x2(q.z, v[4], v[5]);
  unpack_bf16x2(q.w, v[6], v[7]);
}
__device__ __forceinline__ void unpack8(const uint4& q, float (&v)[8]) {
  unpack_bf16x2(q.x, v[0], v[1]);
  unpack_bf16x2(q.y, v[2], v[3]);
  unpack_bf16x2(q.z, v[4], v[5]);
  unpack_bf16x2(q.w, v[6], v[7]);
}
// 8 consecutive floats (32-byte aligned offsets: channel groups of 8)
__device__ __forceinline__ void loadf8(const float* p, float (&v)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
  v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void store8(bf16* p, const float (&v)[8]) {
  uint4 q;
  q.x = pack_bf16x2(v[0], v[1]);
  q.y = pack_bf16x2(v[2], v[3]);
  q.z = pack_bf16x2(v[4], v[5]);
  q.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(p) = q;
}

// Column reductions (esp_colsum: the pos_bias_u / pos_bias_v gradients) finish in two levels so that neither same-sector atomic
// contention nor a long serial tail is on the critical path: every CTA adds its per-column partial sums to one of
// kRedSlots scratch rows (fire-and-forget RED, contention / kRedSlots), the LAST CTA to finish (ticket counter) sums
// the kRedSlots rows, accumulates into the destination and re-zeroes the scratch.  Scratch is module-static device
// memory: kernels of one stream serialise, and the library is driven from one stream per device.
constexpr int kRedSlots = 8;
constexpr int kRedMaxCols = 4096;
__device__ float g_red_slots[2][kRedSlots][kRedMaxCols];
__device__ unsigned int g_red_ticket[1 + kRedMaxCols / 256];

// ================================================================================================
// LayerNorm: one warp per row, row cached in registers (d <= 2048, d % 8 == 0)
// ================================================================================================
constexpr int kLnMaxVec = 8;  // uint4 per lane (template parameter NV <= kLnMaxVec)

template <int NV>
__global__ void __launch_bounds__(256)
ln_fwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ gamma, const bf16* __restrict__ beta, float eps,
              long R, int d, bf16* __restrict__ y, float* __restrict__ mean_out, float* __restrict__ rstd_out,
              const int* __restrict__ lens, int T, float drop_p, uint32_t drop_thresh, unsigned long long seed0,
              const unsigned long long* __restrict__ seed_ptr) {
  esp_pdl();
  const unsigned long long seed = seed0 + (seed_ptr ? *seed_ptr : 0ull);
  const int lane = threadIdx.x & 31;
  const long warp0 = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long nwarps = (long)gridDim.x * (blockDim.x >> 5);
  const int nvec = d >> 3;
  const float drop_scale = drop_p > 0.f ? 65536.f / (65536.f - (float)drop_thresh) : 1.f;
  for (long r = warp0; r < R; r += nwarps) {
    const bf16* xr = x + r * d;
    float v[NV][8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) {
        load8(xr + vi * 8, v[i]);
#pragma unroll
        for (int j = 0; j < 8; ++j) s += v[i][j];
      }
    }
    const float mean = warp_sum(s) / (float)d;
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float c = v[i][j] - mean;
          ss += c * c;
        }
      }
    }
    const float rstd = rsqrtf(warp_sum(ss) / (float)d + eps);
    if (lane == 0) {
      if (mean_out) mean_out[r] = mean;
      if (rstd_out) rstd_out[r] = rstd;
    }
    // optional: zero padded rows (t >= len_b) -- speech_transformer_encoder.py:354-357
    bool zero_row = false;
    if (lens) {
      const int b = (int)(r / T), t = (int)(r % T);
      zero_row = t >= lens[b];
    }
    bf16* yr = y + r * d;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) {
        float g[8], bb[8], o[8];
        load8(gamma + vi * 8, g);
        load8(beta + vi * 8, bb);
        bool keep[8];
        if (drop_p > 0.f) esp_keep8(seed, (unsigned long long)r * d + vi * 8, drop_thresh, keep);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float t = (v[i][j] - mean) * rstd * g[j] + bb[j];
          if (drop_p > 0.f) t = keep[j] ? t * drop_scale : 0.f;
          o[j] = zero_row ? 0.f : t;
        }
        store8(yr + vi * 8, o);
      }
    }
  }
}

// dx = rstd * (g*dy - mean(g*dy) - xhat*mean(g*dy*xhat)) [+ dres];  dgamma += dy*xhat; dbeta += dy
template <int NV>
__global__ void __launch_bounds__(256, NV <= 2 ? 2 : 1)
ln_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x, const float* __restrict__ mean_in,
              const float* __restrict__ rstd_in, const bf16* __restrict__ gamma, const bf16* __restrict__ dres, long R,
              int d, bf16* __restrict__ dx, float* __restrict__ dgamma, float* __restrict__ dbeta,
              const int* __restrict__ lens, int T, float drop_p, uint32_t drop_thresh, unsigned long long seed0,
              const unsigned long long* __restrict__ seed_ptr, bf16* __restrict__ dx2, float scale2, uint32_t thresh2,
              unsigned long long seed2_0) {
  esp_pdl();
  const unsigned long long seed = seed0 + (seed_ptr ? *seed_ptr : 0ull);
  const unsigned long long seed2 = seed2_0 + (seed_ptr ? *seed_ptr : 0ull);
  // dx2 = dropout(dx) * scale2 on the SAME counter stream as esp_dropout (index r*d + c): the masked gradient the next
  // module's backward starts with, produced here instead of by a separate pass over dx
  const float ds2 = thresh2 > 0 ? scale2 * 65536.f / (65536.f - (float)thresh2) : scale2;
  extern __shared__ float sm_red[];  // [warps][2][NV * 256]: per-warp partial column sums, transposed
  const int lane = threadIdx.x & 31;
  const int nw = blockDim.x >> 5;
  const long warp0 = (long)blockIdx.x * nw + (threadIdx.x >> 5);
  const long nwarps = (long)gridDim.x * nw;
  const int nvec = d >> 3;
  const float drop_scale = drop_p > 0.f ? 65536.f / (65536.f - (float)drop_thresh) : 1.f;
  float ag[NV][8], ab[NV][8];
#pragma unroll
  for (int i = 0; i < NV; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) ag[i][j] = ab[i][j] = 0.f;
  uint4 gq[NV];  // gamma stays in registers (packed) for every row of this warp
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int vi = lane + i * 32;
    gq[i] = vi < nvec ? *reinterpret_cast<const uint4*>(gamma + vi * 8) : make_uint4(0, 0, 0, 0);
  }
  for (long r = warp0; r < R; r += nwarps) {
    bool zero_row = false;
    if (lens) {
      const int b = (int)(r / T), t = (int)(r % T);
      zero_row = t >= lens[b];
    }
    // All global loads of the row are issued up front and stay PACKED in registers (bf16 pairs); both passes unpack
    // them again, which is cheaper than keeping 2 x NV x 8 floats alive (register pressure decides the occupancy of
    // this latency-bound kernel).
    uint4 dq[NV], xq[NV], rq[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) {
        dq[i] = *reinterpret_cast<const uint4*>(dy + r * d + vi * 8);
        xq[i] = *reinterpret_cast<const uint4*>(x + r * d + vi * 8);
        if (dres) rq[i] = *reinterpret_cast<const uint4*>(dres + r * d + vi * 8);
      }
    }
    const float mean = mean_in[r], rstd = rstd_in[r];
    const float dsc = (drop_p > 0.f) ? drop_scale : 1.f;
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) {
        if (zero_row) {
          dq[i] = make_uint4(0, 0, 0, 0);
        } else if (drop_p > 0.f) {
          // dropped elements are zeroed in the packed copy; the 1/(1-p) scale is applied on unpack
          bool keep[8];
          esp_keep8(seed, (unsigned long long)r * d + vi * 8, drop_thresh, keep);
          dq[i].x &= (keep[0] ? 0x0000FFFFu : 0u) | (keep[1] ? 0xFFFF0000u : 0u);
          dq[i].y &= (keep[2] ? 0x0000FFFFu : 0u) | (keep[3] ? 0xFFFF0000u : 0u);
          dq[i].z &= (keep[4] ? 0x0000FFFFu : 0u) | (keep[5] ? 0xFFFF0000u : 0u);
          dq[i].w &= (keep[6] ? 0x0000FFFFu : 0u) | (keep[7] ? 0xFFFF0000u : 0u);
        }
        float a[8], xv[8], g[8];
        unpack8(dq[i], a);
        unpack8(xq[i], xv);
        unpack8(gq[i], g);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float dyv = a[j] * dsc;
          const float h = (xv[j] - mean) * rstd;
          const float gd = dyv * g[j];
          ag[i][j] += dyv * h;
          ab[i][j] += dyv;
          s1 += gd;
          s2 += gd * h;
        }
      }
    }
    s1 = warp_sum(s1) / (float)d;
    s2 = warp_sum(s2) / (float)d;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) {
        float a[8], xv[8], g[8], o[8], rr[8];
        unpack8(dq[i], a);
        unpack8(xq[i], xv);
        unpack8(gq[i], g);
        if (dres) unpack8(rq[i], rr);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float h = (xv[j] - mean) * rstd;
          o[j] = rstd * (a[j] * dsc * g[j] - s1 - h * s2);
          if (dres) o[j] += rr[j];
        }
        store8(dx + r * d + vi * 8, o);
        if (dx2) {
          bool keep2[8];
          if (thresh2 > 0) esp_keep8(seed2, (unsigned long long)r * d + vi * 8, thresh2, keep2);
          float o2[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) o2[j] = (thresh2 > 0 && !keep2[j]) ? 0.f : bf2f(f2bf(o[j])) * ds2;  // dropout of the bf16 dx
          store8(dx2 + r * d + vi * 8, o2);
        }
      }
    }
  }
  // Block reduce of the per-column partial sums WITHOUT shared-memory atomics (64 conflicting atomics per thread were the
  // tail of this kernel): every warp parks its partials transposed ([value index][lane] -> conflict-free), then each
  // thread adds the 8 warps' values of 4 (gamma) + 4 (beta) columns and sends them to the cross-CTA slots.
  if (dgamma == nullptr && dbeta == nullptr) return;
  {
    const int warp = threadIdx.x >> 5;
    float* mine = sm_red + (size_t)warp * (2 * NV * 256);
#pragma unroll
    for (int i = 0; i < NV; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        mine[(i * 8 + j) * 32 + lane] = ag[i][j];
        mine[NV * 256 + (i * 8 + j) * 32 + lane] = ab[i][j];
      }
  }
  __syncthreads();
  // Thread g owns 4 consecutive columns of one destination: 16-byte vector reductions at L2 straight into the (fp32,
  // accumulating) parameter gradients -- fire and forget: no scratch slots, no ticket, no serial fold by a last CTA.
  const bool vec_ok = ((reinterpret_cast<uintptr_t>(dgamma) | reinterpret_cast<uintptr_t>(dbeta)) & 15) == 0;
  for (int g = threadIdx.x; g < 2 * NV * 64; g += blockDim.x) {
    const int ln = g & 31, r = g >> 5;
    const int jh = (r & 1) * 4, i = (r >> 1) % NV, which = (r >> 1) / NV;
    float a[4] = {0.f, 0.f, 0.f, 0.f};
    for (int w = 0; w < nw; ++w) {
      const float* src = sm_red + (size_t)w * (2 * NV * 256) + which * (NV * 256) + (i * 8 + jh) * 32 + ln;
#pragma unroll
      for (int t = 0; t < 4; ++t) a[t] += src[t * 32];
    }
    float* dst = which == 0 ? dgamma : dbeta;
    const int col = (ln + 32 * i) * 8 + jh;
    if (dst == nullptr || col >= d) continue;
    if (vec_ok) {
      red_add_v4(dst + col, a[0], a[1], a[2], a[3]);
    } else {
#pragma unroll
      for (int t = 0; t < 4; ++t) atomicAdd(dst + col + t, a[t]);
    }
  }
}

// ================================================================================================
// generic elementwise / reductions over [R, N] bf16 (N % 8 == 0, row stride ld)
// ================================================================================================
// out[n] += scale * sum_r x[r, n]     (fp32; per-CTA partials, last CTA of each column block finishes)
// grid (column blocks of 256 columns, row splits); block = 32 column-vectors x 8 row lanes
__global__ void __launch_bounds__(256)
colsum_kernel(const bf16* __restrict__ x, long R, int N, long ld, float scale, float* __restrict__ out) {
  esp_pdl();
  const int cv = blockIdx.x * 32 + (threadIdx.x & 31);
  const int rl = threadIdx.x >> 5;
  __shared__ float red[8][32][8];
  __shared__ int s_last;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (cv * 8 < N) {
    const long stride = (long)gridDim.y * 8;
    long r = (long)blockIdx.y * 8 + rl;
    for (; r + 3 * stride < R; r += 4 * stride) {  // 4 independent loads in flight per thread
      float v0[8], v1[8], v2[8], v3[8];
      load8(x + r * ld + cv * 8, v0);
      load8(x + (r + stride) * ld + cv * 8, v1);
      load8(x + (r + 2 * stride) * ld + cv * 8, v2);
      load8(x + (r + 3 * stride) * ld + cv * 8, v3);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += (v0[j] + v1[j]) + (v2[j] + v3[j]);
    }
    for (; r < R; r += stride) {
      float v[8];
      load8(x + r * ld + cv * 8, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += v[j];
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[rl][threadIdx.x & 31][j] = acc[j];
  __syncthreads();
  if (rl == 0) {
    const int slot = blockIdx.y % kRedSlots;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float sacc = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) sacc += red[k][threadIdx.x & 31][j];
      const int col = cv * 8 + j;
      if (col < N) atomicAdd(&g_red_slots[0][slot][col], sacc);
    }
  }
  // one ticket per column block: its last row-split CTA finishes the block's 256 columns
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(&g_red_ticket[1 + blockIdx.x], 1u) == gridDim.y - 1);
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c < N) {
    float a0 = 0.f;
#pragma unroll
    for (int k = 0; k < kRedSlots; ++k) a0 += __ldcg(&g_red_slots[0][k][c]);
#pragma unroll
    for (int k = 0; k < kRedSlots; ++k) __stcg(&g_red_slots[0][k][c], 0.f);
    out[c] += a0 * scale;
  }
  if (threadIdx.x == 0) g_red_ticket[1 + blockIdx.x] = 0u;
}

// y = dropout(x) * scale  (same counter RNG as the GEMM epilogue: index = r*N + n)
__global__ void __launch_bounds__(256)
dropout_kernel(const bf16* __restrict__ x, long R, int N, long ldx, long ldy, float scale, float drop_p,
               uint32_t thresh, unsigned long long seed0, const unsigned long long* __restrict__ seed_ptr,
               bf16* __restrict__ y) {
  esp_pdl();
  const unsigned long long seed = seed0 + (seed_ptr ? *seed_ptr : 0ull);
  const long nvec = R * (N >> 3);
  const float ds = drop_p > 0.f ? scale * 65536.f / (65536.f - (float)thresh) : scale;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long)gridDim.x * blockDim.x) {
    long r;
    unsigned cvi;
    esp_divmod(i, (unsigned)(N >> 3), r, cvi);
    const int c = (int)cvi * 8;
    float v[8];
    load8(x + r * ldx + c, v);
    bool keep[8];
    if (drop_p > 0.f) esp_keep8(seed, (unsigned long long)r * N + c, thresh, keep);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = (drop_p > 0.f && !keep[j]) ? 0.f : v[j] * ds;
    store8(y + r * ldy + c, v);
  }
}

// zero rows t >= lens[b] of x [B, T, N]
__global__ void __launch_bounds__(256)
mask_rows_kernel(bf16* __restrict__ x, const int* __restrict__ lens, int B, int T, int N) {
  esp_pdl();
  const long nvec = (long)B * T * (N >> 3);
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long)gridDim.x * blockDim.x) {
    long r;
    unsigned cvi;
    esp_divmod(i, (unsigned)(N >> 3), r, cvi);
    const int b = (int)((unsigned)r / (unsigned)T), t = (int)((unsigned)r % (unsigned)T);  // B*T < 2^31
    if (t >= lens[b]) *reinterpret_cast<uint4*>(x + i * 8) = make_uint4(0, 0, 0, 0);
  }
}

// q_u = (q + u) * s ; q_v = (q + v) * s          (multihead_attention.py:679-688)
__global__ void __launch_bounds__(256)
qprep_fwd_kernel(const bf16* __restrict__ q, long ldq, const bf16* __restrict__ u, const bf16* __restrict__ v, float s,
                 long R, int d, bf16* __restrict__ qu, bf16* __restrict__ qv) {
  esp_pdl();
  const long nvec = R * (d >> 3);
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long)gridDim.x * blockDim.x) {
    long r;
    unsigned cvi;
    esp_divmod(i, (unsigned)(d >> 3), r, cvi);
    const int c = (int)cvi * 8;
    float a[8], bu[8], bv[8], o1[8], o2[8];
    load8(q + r * ldq + c, a);
    load8(u + c, bu);
    load8(v + c, bv);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      // the reference rounds (q + bias) to bf16 before scaling; mirror that
      o1[j] = bf2f(f2bf(a[j] + bu[j])) * s;
      o2[j] = bf2f(f2bf(a[j] + bv[j])) * s;
    }
    store8(qu + r * d + c, o1);
    store8(qv + r * d + c, o2);
  }
}
// dq = s * (dqu + dqv)  -> written with row stride ld_out
__global__ void __launch_bounds__(256)
qprep_bwd_kernel(const bf16* __restrict__ dqu, const bf16* __restrict__ dqv, float s, long R, int d,
                 bf16* __restrict__ dq, long ld_out) {
  esp_pdl();
  const long nvec = R * (d >> 3);
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long)gridDim.x * blockDim.x) {
    long r;
    unsigned cvi;
    esp_divmod(i, (unsigned)(d >> 3), r, cvi);
    const int c = (int)cvi * 8;
    float a[8], b[8], o[8];
    load8(dqu + r * d + c, a);
    load8(dqv + r * d + c, b);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = s * (a[j] + b[j]);
    store8(dq + r * ld_out + c, o);
  }
}

// ================================================================================================
// attention softmax over keys with key-padding mask; one warp per (head, batch, query) row
// scores layout [H, B, T, ld] bf16.  T <= 32*kSmMax.
// ================================================================================================
constexpr int kSmMaxT = 1280;  // keys per row (36 s of audio after 4x subsampling = 900)

// Each lane owns NI groups of 8 consecutive keys: j = (i*32 + lane)*8 + e.  Dropout indices are row*ld + j
// (ld % 8 == 0, so every group is hash-aligned).
// kRelax: relaxed attention (multihead_attention.py:869-872) -- p_out keeps the plain softmax P (the backward needs it) and
// pd_out = dropout(bf16(bf16(keep_w * P) + add_w)) with keep_w = 1 - w and add_w = w / T over ALL T keys (padded ones
// included, as the reference divides by src_len); columns [T, ld) stay zero.
template <int NI, bool kRelax>
__global__ void __launch_bounds__(256)
attn_softmax_fwd_kernel(const bf16* __restrict__ s_in, int H, int B, int Tq, int T, int ld, const int* __restrict__ lens,
                        int causal, bf16* __restrict__ p_out, bf16* __restrict__ pd_out, float drop_p, uint32_t thresh,
                        unsigned long long seed0, const unsigned long long* __restrict__ seed_ptr, float keep_w, float add_w) {
  esp_pdl();
  // rows = H*B*Tq queries, T keys per row; causal: key j is visible to query i iff j <= i (future_mask, -inf)
  const unsigned long long seed = seed0 + (seed_ptr ? *seed_ptr : 0ull);
  const int lane = threadIdx.x & 31;
  const long row = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long rows = (long)H * B * Tq;
  if (row >= rows) return;
  const int b = (int)((row / Tq) % B);
  int klen = lens ? min(lens[b], T) : T;
  if (causal) klen = min(klen, (int)(row % Tq) + 1);
  const bf16* sr = s_in + row * ld;
  float v[NI][8];
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < NI; ++i) {
    const int j = (i * 32 + lane) * 8;
    if (j < ld) load8(sr + j, v[i]);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      v[i][e] = (j + e < klen) ? v[i][e] : -INFINITY;  // key_padding_mask -> -inf (:848-854)
      mx = fmaxf(mx, v[i][e]);
    }
  }
  mx = warp_max(mx);
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < NI; ++i)
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      v[i][e] = (v[i][e] == -INFINITY) ? 0.f : __expf(v[i][e] - mx);
      sum += v[i][e];
    }
  sum = warp_sum(sum);
  const float inv = sum > 0.f ? 1.f / sum : 0.f;  // no visible key (lens[b] == 0): P = 0, not 0 * inf = NaN
  const float ds = drop_p > 0.f ? 65536.f / (65536.f - (float)thresh) : 1.f;
#pragma unroll
  for (int i = 0; i < NI; ++i) {
    const int j = (i * 32 + lane) * 8;
    if (j < ld) {
      // softmax in fp32, result cast to the model dtype (fairseq/utils.py:514-525 + .type_as)
      float o[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = bf2f(f2bf(v[i][e] * inv));
      store8(p_out + row * ld + j, o);
      if constexpr (kRelax) {
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] = j + e < T ? bf2f(f2bf(bf2f(f2bf(keep_w * o[e])) + add_w)) : 0.f;
      }
      if (pd_out && drop_p > 0.f) {
        bool k[8];
        esp_keep8(seed, (unsigned long long)row * ld + j, thresh, k);
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] = k[e] ? o[e] * ds : 0.f;
      }
      if (pd_out) store8(pd_out + row * ld + j, o);
    }
  }
}

// dS = P * (dP - sum_j dP*P), dP = dropmask * dPd / (1-p);  also scatters dS into the skewed
// relative-position layout dBD[row, (T-1) - i + j]  (zeros elsewhere).
template <int NI>
__global__ void __launch_bounds__(256)
attn_softmax_bwd_kernel(const bf16* __restrict__ p_in, const bf16* __restrict__ dpd, int H, int B, int Tq, int T, int ld,
                        bf16* __restrict__ ds_out, bf16* __restrict__ dbd_out, int ldp, float drop_p,
                        uint32_t thresh, unsigned long long seed0, const unsigned long long* __restrict__ seed_ptr) {
  esp_pdl();
  const unsigned long long seed = seed0 + (seed_ptr ? *seed_ptr : 0ull);
  const int lane = threadIdx.x & 31;
  const long row = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long rows = (long)H * B * Tq;
  if (row >= rows) return;
  const int qi = (int)(row % Tq);
  const float dscale = drop_p > 0.f ? 65536.f / (65536.f - (float)thresh) : 1.f;
  float pv[NI][8], dv[NI][8];
  float dot = 0.f;
#pragma unroll
  for (int i = 0; i < NI; ++i) {
    const int j = (i * 32 + lane) * 8;
#pragma unroll
    for (int e = 0; e < 8; ++e) pv[i][e] = dv[i][e] = 0.f;
    if (j < ld) {
      load8(p_in + row * ld + j, pv[i]);
      load8(dpd + row * ld + j, dv[i]);
      bool k[8];
      if (drop_p > 0.f) esp_keep8(seed, (unsigned long long)row * ld + j, thresh, k);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        if (j + e >= T) { pv[i][e] = 0.f; dv[i][e] = 0.f; }
        else if (drop_p > 0.f) dv[i][e] = k[e] ? dv[i][e] * dscale : 0.f;
        dot += dv[i][e] * pv[i][e];
      }
    }
  }
  dot = warp_sum(dot);
  bf16* dbd = dbd_out ? dbd_out + row * ldp : nullptr;
  const int lo = (T - 1) - qi;  // dBD column of key j = 0
  if (dbd) {
    // zero the parts of the skewed row that no (i, j) maps to
    for (int r = lane; r < ldp; r += 32)
      if (r < lo || r >= lo + T) dbd[r] = f2bf(0.f);
  }
#pragma unroll
  for (int i = 0; i < NI; ++i) {
    const int j = (i * 32 + lane) * 8;
    if (j < ld) {
      float o[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = pv[i][e] * (dv[i][e] - dot);
      store8(ds_out + row * ld + j, o);
      if (dbd) {
#pragma unroll
        for (int e = 0; e < 8; ++e)
          if (j + e < T) dbd[lo + j + e] = f2bf(o[e]);
      }
    }
  }
}

// ================================================================================================
// Conformer convolution module body: GLU -> depthwise conv (k odd, 'same' zero padding over the
// padded batch length T) -> BatchNorm1d statistics.   conformer_layer.py:88-95
//   g [B, T, 2C] bf16 ; w [C, k] bf16 ; y [B, T, C] bf16 ; stats double [2, C] (sum, sum of squares)
// CTA tile: 64 time steps x 64 channels.
// ================================================================================================
constexpr int kDwT = 64, kDwC = 64, kDwMaxK = 31;

// Thread mapping: 64 channels x 4 time groups; a thread produces kDwPerThr = 16 CONSECUTIVE outputs of one
// channel with a register sliding window, so each staged input is read from shared memory once per thread
// (46 loads for 16 x 31 FMAs) instead of once per tap.
constexpr int kDwPerThr = kDwT / 4;

__global__ void __launch_bounds__(256)
glu_dwconv_fwd_kernel(const bf16* __restrict__ g, const bf16* __restrict__ w, int B, int T, int Cn, int ksz,
                      bf16* __restrict__ y, double* __restrict__ stats) {
  esp_pdl();
  __shared__ float tile[kDwT + kDwMaxK - 1][kDwC + 1];
  __shared__ float red[2][4][kDwC];
  const int b = blockIdx.z, t0 = blockIdx.x * kDwT, c0 = blockIdx.y * kDwC;
  const int half = ksz >> 1;
  const int cl = threadIdx.x & 63, tg = threadIdx.x >> 6;
  // taps of the tile's 64 channels: one coalesced pass into shared memory, then 31 conflict-free reads per thread
  __shared__ float wsm[kDwC * kDwMaxK];
  for (int i = threadIdx.x; i < kDwC * ksz; i += blockDim.x) wsm[i] = bf2f(w[(long)c0 * ksz + i]);
  // staging with 16-byte loads: one task = 8 channels of one row
  for (int i = threadIdx.x; i < (kDwT + ksz - 1) * (kDwC / 8); i += blockDim.x) {
    const int r = i >> 3, cv = (i & 7) * 8;
    const int t = t0 + r - half;
    float v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (t >= 0 && t < T) {
      const bf16* row = g + ((long)b * T + t) * 2 * Cn + c0 + cv;
      float a[8], gate[8];
      load8(row, a);
      load8(row + Cn, gate);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = bf2f(f2bf(a[j] * sigmoidf_(gate[j])));  // GLU output is bf16 in the reference
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) tile[r][cv + j] = v[j];
  }
  __syncthreads();
  float wr[kDwMaxK];
#pragma unroll
  for (int k = 0; k < kDwMaxK; ++k) wr[k] = k < ksz ? wsm[cl * ksz + k] : 0.f;
  const int tb = tg * kDwPerThr;  // first local output of this thread
  float acc[kDwPerThr];
#pragma unroll
  for (int i = 0; i < kDwPerThr; ++i) acc[i] = 0.f;
  // input row r = tb + i + k contributes to output i with tap k
#pragma unroll
  for (int r = 0; r < kDwPerThr + kDwMaxK - 1; ++r) {
    if (r < kDwPerThr + ksz - 1) {
      const float xv = tile[tb + r][cl];
#pragma unroll
      for (int i = 0; i < kDwPerThr; ++i) {
        const int k = r - i;
        if (k >= 0 && k < kDwMaxK) acc[i] = fmaf(xv, wr[k], acc[i]);
      }
    }
  }
  float s1 = 0.f, s2 = 0.f;
  __syncthreads();  // every thread has consumed its inputs: the tile is reused to collect the outputs
#pragma unroll
  for (int i = 0; i < kDwPerThr; ++i) {
    const int t = t0 + tb + i;
    const float of = bf2f(f2bf(acc[i]));
    tile[tb + i][cl] = of;
    if (t < T) {
      s1 += of;
      s2 += of * of;
    }
  }
  red[0][tg][cl] = s1;
  red[1][tg][cl] = s2;
  __syncthreads();
  // 16-byte stores: one task = 8 channels of one row (instead of sixteen 2-byte stores per thread)
  for (int i = threadIdx.x; i < kDwT * (kDwC / 8); i += blockDim.x) {
    const int r = i >> 3, cv = (i & 7) * 8;
    const int t = t0 + r;
    if (t >= T) continue;
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = tile[r][cv + j];
    store8(y + ((long)b * T + t) * Cn + c0 + cv, o);
  }
  if (stats && tg == 0) {
    const float a = red[0][0][cl] + red[0][1][cl] + red[0][2][cl] + red[0][3][cl];
    const float q = red[1][0][cl] + red[1][1][cl] + red[1][2][cl] + red[1][3][cl];
    atomicAdd(&stats[c0 + cl], (double)a);
    atomicAdd(&stats[Cn + c0 + cl], (double)q);
  }
}

// backward of GLU + depthwise conv:
//   dglu[t,c] = sum_k w[c,k] * dy[t - k + half, c]
//   dw[c,k]  += sum_t dy[t,c] * glu[t + k - half, c]
//   dg[:, :C] = dglu * sigmoid(gate) ; dg[:, C:] = dglu * a * sigmoid(gate) * (1 - sigmoid(gate))
__global__ void __launch_bounds__(256)
glu_dwconv_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ g, const bf16* __restrict__ w, int B,
                      int T, int Cn, int ksz, bf16* __restrict__ dg, float* __restrict__ dw) {
  esp_pdl();
  extern __shared__ __align__(16) uint8_t dw_smem[];
  typedef float TileT[kDwC + 1];
  TileT* dyt = reinterpret_cast<TileT*>(dw_smem);                       // dy at t0-half .. t0+63+half
  TileT* glt = dyt + (kDwT + kDwMaxK - 1);                              // glu at the same times
  typedef float RedT[kDwMaxK][kDwC];
  RedT* dwred = reinterpret_cast<RedT*>(glt + (kDwT + kDwMaxK - 1));    // [4][k][channel]: conflict-free
  const int b = blockIdx.z, t0 = blockIdx.x * kDwT, c0 = blockIdx.y * kDwC;
  const int half = ksz >> 1;
  const int cl = threadIdx.x & 63, tg = threadIdx.x >> 6;
  __shared__ float wsm[kDwC * kDwMaxK];
  for (int i = threadIdx.x; i < kDwC * ksz; i += blockDim.x) wsm[i] = bf2f(w[(long)c0 * ksz + i]);
  for (int i = threadIdx.x; i < (kDwT + ksz - 1) * (kDwC / 8); i += blockDim.x) {
    const int r = i >> 3, cv = (i & 7) * 8;
    const int t = t0 + r - half;
    float dv[8] = {0, 0, 0, 0, 0, 0, 0, 0}, gl[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (t >= 0 && t < T) {
      load8(dy + ((long)b * T + t) * Cn + c0 + cv, dv);
      const bf16* row = g + ((long)b * T + t) * 2 * Cn + c0 + cv;
      float a[8], gate[8];
      load8(row, a);
      load8(row + Cn, gate);
#pragma unroll
      for (int j = 0; j < 8; ++j) gl[j] = bf2f(f2bf(a[j] * sigmoidf_(gate[j])));
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      dyt[r][cv + j] = dv[j];
      glt[r][cv + j] = gl[j];
    }
  }
  __syncthreads();
  const int tb = tg * kDwPerThr;
  // ---- input gradient: dglu[i] = sum_k w[k] * dy[t - k + half].  With the taps flipped (wf[k'] = w[ksz-1-k'])
  // this is the forward correlation dglu[i] = sum_k' wf[k'] * dyt[tb + i + k'] (2*half = ksz-1): static indexing.
  {
    float wf[kDwMaxK];
#pragma unroll
    for (int k = 0; k < kDwMaxK; ++k) wf[k] = k < ksz ? wsm[cl * ksz + (ksz - 1 - k)] : 0.f;
    float acc[kDwPerThr];
#pragma unroll
    for (int i = 0; i < kDwPerThr; ++i) acc[i] = 0.f;
#pragma unroll
    for (int r = 0; r < kDwPerThr + kDwMaxK - 1; ++r) {
      if (r < kDwPerThr + ksz - 1) {
        const float dv = dyt[tb + r][cl];
#pragma unroll
        for (int i = 0; i < kDwPerThr; ++i) {
          const int k = r - i;
          if (k >= 0 && k < kDwMaxK) acc[i] = fmaf(dv, wf[k], acc[i]);
        }
      }
    }
    // park dglu in shared memory (the dwred area is free until the weight-gradient pass) ...
    float (*dgl)[kDwC + 1] = reinterpret_cast<float (*)[kDwC + 1]>(dwred);
#pragma unroll
    for (int i = 0; i < kDwPerThr; ++i) dgl[tb + i][cl] = acc[i];
  }
  __syncthreads();
  // ... and write both halves of dg with 16-byte vectors: one task = 8 channels of one row (a and the gate are re-read
  // with 16-byte loads; the scalar 2-byte loads / stores of this epilogue were the bulk of the kernel's memory instructions)
  {
    float (*dgl)[kDwC + 1] = reinterpret_cast<float (*)[kDwC + 1]>(dwred);
    for (int i = threadIdx.x; i < kDwT * (kDwC / 8); i += blockDim.x) {
      const int r = i >> 3, cv = (i & 7) * 8;
      const int t = t0 + r;
      if (t >= T) continue;
      const bf16* row = g + ((long)b * T + t) * 2 * Cn + c0 + cv;
      float a[8], gate[8], o1[8], o2[8];
      load8(row, a);
      load8(row + Cn, gate);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float sg = sigmoidf_(gate[j]);
        const float d = dgl[r][cv + j];
        o1[j] = d * sg;
        o2[j] = d * a[j] * sg * (1.f - sg);
      }
      bf16* orow = dg + ((long)b * T + t) * 2 * Cn + c0 + cv;
      store8(orow, o1);
      store8(orow + Cn, o2);
    }
  }
  __syncthreads();
  // ---- weight gradient: dw[k] += sum_i dy[tb+i] * glu[tb + i + k - half] = dyt[tb+i+half] * glt[tb+i+k]
  {
    float acc[kDwMaxK];
#pragma unroll
    for (int k = 0; k < kDwMaxK; ++k) acc[k] = 0.f;
    float dreg[kDwPerThr];
#pragma unroll
    for (int i = 0; i < kDwPerThr; ++i) dreg[i] = (t0 + tb + i < T) ? dyt[tb + i + half][cl] : 0.f;
#pragma unroll
    for (int r = 0; r < kDwPerThr + kDwMaxK - 1; ++r) {
      if (r < kDwPerThr + ksz - 1) {
        const float gv = glt[tb + r][cl];
#pragma unroll
        for (int i = 0; i < kDwPerThr; ++i) {
          const int k = r - i;
          if (k >= 0 && k < kDwMaxK) acc[k] = fmaf(dreg[i], gv, acc[k]);
        }
      }
    }
#pragma unroll
    for (int k = 0; k < kDwMaxK; ++k) dwred[tg][k][cl] = acc[k];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kDwC * ksz; i += blockDim.x) {
    const int k = i / kDwC, c = i % kDwC;
    const float sacc = dwred[0][k][c] + dwred[1][k][c] + dwred[2][k][c] + dwred[3][k][c];
    atomicAdd(&dw[(long)(c0 + c) * ksz + k], sacc);
  }
}

// mean/rstd per channel from the double (sum, sumsq) accumulators (training) or the running stats
// (eval); also the running-stat update  rm = (1-m) rm + m mean ; rv = (1-m) rv + m * unbiased var
__global__ void bn_finalize_kernel(const double* __restrict__ stats, long R, int Cn, float eps, float momentum,
                                   float* __restrict__ run_mean, float* __restrict__ run_var, int training,
                                   float* __restrict__ mr) {
  esp_pdl();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= Cn) return;
  if (training) {
    const double m = stats[c] / (double)R;
    double var = stats[Cn + c] / (double)R - m * m;
    if (var < 0) var = 0;
    mr[c] = (float)m;
    mr[Cn + c] = rsqrtf((float)var + eps);
    if (run_mean && run_var) {
      const double unb = R > 1 ? var * (double)R / (double)(R - 1) : var;
      run_mean[c] = (1.f - momentum) * run_mean[c] + momentum * (float)m;
      run_var[c] = (1.f - momentum) * run_var[c] + momentum * (float)unb;
    }
  } else {
    mr[c] = run_mean[c];
    mr[Cn + c] = rsqrtf(run_var[c] + eps);
  }
}

// Activation after BatchNorm: 1 = SiLU (Conformer conv module), 2 = ReLU (conv front end).
__device__ __forceinline__ float bn_act(float bn, int act) { return act == 1 ? siluf_(bn) : fmaxf(bn, 0.f); }
__device__ __forceinline__ float bn_act_grad(float bn, int act) { return act == 1 ? silu_gradf_(bn) : (bn > 0.f ? 1.f : 0.f); }

// Thread mapping for per-channel reductions over x [R, C] (C/8 divides 256): a thread walks 16-byte vectors
// with a stride that is a multiple of C/8, so it always sees the same 8 channels and accumulates in
// registers; one shared-memory pass + one double atomic per channel per CTA finishes the job.
// stats[c] += sum_r x[r,c] ; stats[C + c] += sum_r x[r,c]^2
__global__ void __launch_bounds__(256)
bn_stats_kernel(const bf16* __restrict__ x, const bf16* __restrict__ pre_bias, long R, int Cn,
                double* __restrict__ stats) {
  esp_pdl();
  __shared__ float red[2][256][8];
  const int cv = Cn >> 3;
  const long nvec = R * cv;
  float a1[8] = {0, 0, 0, 0, 0, 0, 0, 0}, a2[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  float pb[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  // grid stride is a multiple of cv => the channel group of this thread is fixed
  if (pre_bias) load8(pre_bias + (int)(((long)blockIdx.x * 256 + threadIdx.x) % cv) * 8, pb);
  for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < nvec; i += (long)gridDim.x * 256) {
    float v[8];
    load8(x + i * 8, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (pre_bias) v[j] = bf2f(f2bf(v[j] + pb[j]));  // the tensor being normalised is bf16(x + bias)
      a1[j] += v[j];
      a2[j] += v[j] * v[j];
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    red[0][threadIdx.x][j] = a1[j];
    red[1][threadIdx.x][j] = a2[j];
  }
  __syncthreads();
  if (threadIdx.x < cv) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float s1 = 0.f, s2 = 0.f;
      for (int k = threadIdx.x; k < 256; k += cv) {
        s1 += red[0][k][j];
        s2 += red[1][k][j];
      }
      atomicAdd(&stats[threadIdx.x * 8 + j], (double)s1);
      atomicAdd(&stats[Cn + threadIdx.x * 8 + j], (double)s2);
    }
  }
}

// z = act(bn(y))
__global__ void __launch_bounds__(256)
bn_act_fwd_kernel(const bf16* __restrict__ y, const bf16* __restrict__ pre_bias, long R, int Cn, const float* __restrict__ mr,
                  const bf16* __restrict__ gamma, const bf16* __restrict__ beta, int act, bf16* __restrict__ z) {
  esp_pdl();
  const long nvec = R * (Cn >> 3);
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long)gridDim.x * blockDim.x) {
    long rq_;
    unsigned cvi;
    esp_divmod(i, (unsigned)(Cn >> 3), rq_, cvi);
    const int c = (int)cvi * 8;
    float v[8], gm[8], bt[8], mu[8], rs[8];
    load8(y + i * 8, v);
    load8(gamma + c, gm);
    load8(beta + c, bt);
    loadf8(mr + c, mu);
    loadf8(mr + Cn + c, rs);
    if (pre_bias) {
      float pb[8];
      load8(pre_bias + c, pb);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = bf2f(f2bf(v[j] + pb[j]));
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float bn = bf2f(f2bf((v[j] - mu[j]) * rs[j] * gm[j] + bt[j]));  // BN output is bf16
      v[j] = bn_act(bn, act);
    }
    store8(z + i * 8, v);
  }
}

// pass 1 of BN+act backward: s1[c] = sum dbn, s2[c] = sum dbn * xhat   (dbn = dz * act'(bn))
__global__ void __launch_bounds__(256)
bn_act_bwd_reduce_kernel(const bf16* __restrict__ dz, const bf16* __restrict__ y, const bf16* __restrict__ pre_bias, long R, int Cn,
                         const float* __restrict__ mr, const bf16* __restrict__ gamma,
                         const bf16* __restrict__ beta, int act, double* __restrict__ sums) {
  esp_pdl();
  __shared__ float red[2][256][8];
  const int cv = Cn >> 3;
  const long nvec = R * cv;
  float a1[8] = {0, 0, 0, 0, 0, 0, 0, 0}, a2[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  // grid stride is a multiple of cv => the channel group of this thread is fixed
  const int c = (int)(((long)blockIdx.x * 256 + threadIdx.x) % cv) * 8;
  float gm[8], bt[8], mean[8], rstd[8];
  load8(gamma + c, gm);
  load8(beta + c, bt);
  loadf8(mr + c, mean);
  loadf8(mr + Cn + c, rstd);
  float pb[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (pre_bias) load8(pre_bias + c, pb);
  const long stride = (long)gridDim.x * 256;
  long i = (long)blockIdx.x * 256 + threadIdx.x;
  auto accumulate = [&](const uint4& dq, const uint4& vq) {
    float d[8], v[8];
    unpack8(dq, d);
    unpack8(vq, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (pre_bias) v[j] = bf2f(f2bf(v[j] + pb[j]));
      const float xh = (v[j] - mean[j]) * rstd[j];
      const float bn = bf2f(f2bf(xh * gm[j] + bt[j]));
      const float dbn = d[j] * bn_act_grad(bn, act);
      a1[j] += dbn;
      a2[j] += dbn * xh;
    }
  };
  for (; i + 3 * stride < nvec; i += 4 * stride) {  // 8 independent 16-byte loads in flight per thread
    uint4 dq[4], vq[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      dq[u] = *reinterpret_cast<const uint4*>(dz + (i + u * stride) * 8);
      vq[u] = *reinterpret_cast<const uint4*>(y + (i + u * stride) * 8);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) accumulate(dq[u], vq[u]);
  }
  for (; i < nvec; i += stride)
    accumulate(*reinterpret_cast<const uint4*>(dz + i * 8), *reinterpret_cast<const uint4*>(y + i * 8));
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    red[0][threadIdx.x][j] = a1[j];
    red[1][threadIdx.x][j] = a2[j];
  }
  __syncthreads();
  if (threadIdx.x < cv) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float s1 = 0.f, s2 = 0.f;
      for (int k = threadIdx.x; k < 256; k += cv) {
        s1 += red[0][k][j];
        s2 += red[1][k][j];
      }
      atomicAdd(&sums[threadIdx.x * 8 + j], (double)s1);
      atomicAdd(&sums[Cn + threadIdx.x * 8 + j], (double)s2);
    }
  }
}

// pass 2: dy = gamma * rstd * (dbn - s1/n - xhat * s2/n)
__global__ void __launch_bounds__(256)
bn_act_bwd_apply_kernel(const bf16* __restrict__ dz, const bf16* __restrict__ y, const bf16* __restrict__ pre_bias, long R, int Cn,
                        const float* __restrict__ mr, const float* __restrict__ coef,
                        const bf16* __restrict__ gamma, const bf16* __restrict__ beta, int act, bf16* __restrict__ dy) {
  esp_pdl();
  const long nvec = R * (Cn >> 3);
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long)gridDim.x * blockDim.x) {
    long rq_;
    unsigned cvi;
    esp_divmod(i, (unsigned)(Cn >> 3), rq_, cvi);
    const int c = (int)cvi * 8;
    float d[8], v[8], gm[8], bt[8], o[8], mu[8], rs[8], m1[8], m2[8];
    load8(dz + i * 8, d);
    load8(y + i * 8, v);
    load8(gamma + c, gm);
    load8(beta + c, bt);
    loadf8(mr + c, mu);
    loadf8(mr + Cn + c, rs);
    loadf8(coef + c, m1);
    loadf8(coef + Cn + c, m2);
    if (pre_bias) {
      float pb[8];
      load8(pre_bias + c, pb);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = bf2f(f2bf(v[j] + pb[j]));
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float xh = (v[j] - mu[j]) * rs[j];
      const float bn = bf2f(f2bf(xh * gm[j] + bt[j]));
      const float dbn = d[j] * bn_act_grad(bn, act);
      o[j] = gm[j] * rs[j] * (dbn - m1[j] - xh * m2[j]);
    }
    store8(dy + i * 8, o);
  }
}
// dgamma += s2 ; dbeta += s1 ; and the float means m1 = s1/n, m2 = s2/n used by the apply pass, written to `coef`: 2C
// floats that follow the 2C double sums in the caller's 3C-double workspace
__global__ void bn_param_grad_kernel(double* __restrict__ sums, long R, int Cn, float* __restrict__ dgamma,
                                     float* __restrict__ dbeta, float* __restrict__ coef) {
  esp_pdl();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= Cn) return;
  const double s1 = sums[c], s2 = sums[Cn + c];
  if (dgamma) atomicAdd(&dgamma[c], (float)s2);
  if (dbeta) atomicAdd(&dbeta[c], (float)s1);
  coef[c] = (float)(s1 / (double)R);
  coef[Cn + c] = (float)(s2 / (double)R);
}

}  // namespace

// =================================================================================================
// C ABI
// =================================================================================================
#define ESP_ST cudaStream_t st = (cudaStream_t)stream

extern "C" int esp_layer_norm_fwd(const void* x, const void* gamma, const void* beta, float eps, int64_t R, int32_t d,
                                  void* y, float* mean, float* rstd, const int32_t* lens, int32_t T, float drop_p,
                                  uint64_t seed, const uint64_t* seed_ptr, void* stream) {
  ESP_ST;
  ESP_CHECK(d % 8 == 0 && d <= 256 * kLnMaxVec, "LayerNorm width %d unsupported (need d%%8==0, d<=2048)", d);
  ESP_CHECK(lens == nullptr || (T >= 1 && R % T == 0), "LayerNorm with lens needs rows [B, T]: T >= 1 dividing R (T=%d)", T);
  if (R == 0) return 0;
#define ESP_LN_FWD(NV)                                                                                                      \
  ESP_CUDA(esp_launch(ln_fwd_kernel<NV>, grid_for(R, 8), 256, 0, st, (const bf16*)x, (const bf16*)gamma, (const bf16*)beta, eps, \
                      R, d, (bf16*)y, mean, rstd, lens, T, drop_p, esp_dropout_thresh(drop_p), seed,                             \
                      (const unsigned long long*)seed_ptr))
  if (d <= 512) ESP_LN_FWD(2);
  else if (d <= 1024) ESP_LN_FWD(4);
  else ESP_LN_FWD(8);
#undef ESP_LN_FWD
  return 0;
}

extern "C" int esp_layer_norm_bwd2(const void* dy, const void* x, const float* mean, const float* rstd, const void* gamma,
                                   const void* dres, int64_t R, int32_t d, void* dx, float* dgamma, float* dbeta,
                                   const int32_t* lens, int32_t T, float drop_p, uint64_t seed, const uint64_t* seed_ptr,
                                   void* dx2, float drop_p2, uint64_t seed2, float scale2, void* stream) {
  ESP_ST;
  ESP_CHECK(d % 8 == 0 && d <= 256 * kLnMaxVec, "LayerNorm width %d unsupported", d);
  ESP_CHECK(lens == nullptr || (T >= 1 && R % T == 0), "LayerNorm with lens needs rows [B, T]: T >= 1 dividing R (T=%d)", T);
  if (R == 0) return 0;
  ESP_CHECK(d <= kRedMaxCols, "LayerNorm backward: at most %d columns", kRedMaxCols);
#define ESP_LN_BWD(NV)                                                                                                     \
  {                                                                                                                        \
    ESP_SMEM_OPTIN(ln_bwd_kernel<NV>, 8 * 2 * NV * 256 * sizeof(float));                                                   \
    ESP_CUDA(esp_launch(ln_bwd_kernel<NV>, grid_for(R, 8, 2), 256, 8 * 2 * NV * 256 * sizeof(float), st, (const bf16*)dy,  \
                        (const bf16*)x, mean, rstd, (const bf16*)gamma, (const bf16*)dres, R, d, (bf16*)dx, dgamma, dbeta, \
                        lens, T, drop_p, esp_dropout_thresh(drop_p), seed, (const unsigned long long*)seed_ptr, (bf16*)dx2, \
                        scale2, dx2 ? esp_dropout_thresh(drop_p2) : 0u, (unsigned long long)seed2));                      \
  }
  if (d <= 512) ESP_LN_BWD(2)
  else if (d <= 1024) ESP_LN_BWD(4)
  else ESP_LN_BWD(8)
#undef ESP_LN_BWD
  return 0;
}

extern "C" int esp_layer_norm_bwd(const void* dy, const void* x, const float* mean, const float* rstd, const void* gamma,
                                  const void* dres, int64_t R, int32_t d, void* dx, float* dgamma, float* dbeta,
                                  const int32_t* lens, int32_t T, float drop_p, uint64_t seed, const uint64_t* seed_ptr,
                                  void* stream) {
  return esp_layer_norm_bwd2(dy, x, mean, rstd, gamma, dres, R, d, dx, dgamma, dbeta, lens, T, drop_p, seed, seed_ptr, nullptr, 0.f, 0,
                             1.f, stream);
}

extern "C" int esp_colsum(const void* x, int64_t R, int32_t N, int64_t ld, float scale, float* out, void* stream) {
  ESP_ST;
  ESP_CHECK(N % 8 == 0 && ld % 8 == 0, "colsum needs N and ld multiples of 8");
  if (R == 0 || N == 0) return 0;
  for (int c0 = 0; c0 < N; c0 += kRedMaxCols) {  // wide matrices (vocabulary-sized) go in column panels
    const int n = (N - c0 < kRedMaxCols) ? (N - c0) : kRedMaxCols;
    const unsigned gx = (n / 8 + 31) / 32;
    long gy = (2L * esp_num_sms() + gx - 1) / gx;  // ~2 CTAs per SM in total
    const long max_gy = (R + 31) / 32;              // at least 4 rows per row lane
    if (gy > max_gy) gy = max_gy;
    if (gy < 1) gy = 1;
    dim3 grid(gx, (unsigned)gy);
    ESP_CUDA(esp_launch(colsum_kernel, grid, 256, 0, st, (const bf16*)x + c0, R, n, ld, scale, out + c0));
  }
  return 0;
}

extern "C" int esp_dropout(const void* x, int64_t R, int32_t N, int64_t ldx, int64_t ldy, float scale, float drop_p,
                           uint64_t seed, const uint64_t* seed_ptr, void* y, void* stream) {
  ESP_ST;
  ESP_CHECK(N % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0, "dropout needs N/ld multiples of 8");
  if (R == 0 || N == 0) return 0;
  ESP_CUDA(esp_launch(dropout_kernel, grid_for(R * (N / 8), 256), 256, 0, st, (const bf16*)x, R, N, ldx, ldy, scale, drop_p,
                      esp_dropout_thresh(drop_p), seed, (const unsigned long long*)seed_ptr, (bf16*)y));
  return 0;
}

extern "C" int esp_mask_rows(void* x, const int32_t* lens, int32_t B, int32_t T, int32_t N, void* stream) {
  ESP_ST;
  ESP_CHECK(N % 8 == 0, "mask_rows needs N %% 8 == 0");
  if ((long)B * T * N == 0) return 0;
  ESP_CUDA(esp_launch(mask_rows_kernel, grid_for((long)B * T * (N / 8), 256), 256, 0, st, (bf16*)x, lens, B, T, N));
  return 0;
}

extern "C" int esp_qprep_fwd(const void* q, int64_t ldq, const void* u, const void* v, float scale, int64_t R, int32_t d,
                             void* qu, void* qv, void* stream) {
  ESP_ST;
  ESP_CHECK(d % 8 == 0 && ldq % 8 == 0, "qprep needs d/ld multiples of 8");
  if (R == 0) return 0;
  ESP_CUDA(esp_launch(qprep_fwd_kernel, grid_for(R * (d / 8), 256), 256, 0, st, (const bf16*)q, ldq, (const bf16*)u,
                      (const bf16*)v, scale, R, d, (bf16*)qu, (bf16*)qv));
  return 0;
}

extern "C" int esp_qprep_bwd(const void* dqu, const void* dqv, float scale, int64_t R, int32_t d, void* dq, int64_t ld_out,
                             void* stream) {
  ESP_ST;
  ESP_CHECK(d % 8 == 0 && ld_out % 8 == 0, "qprep needs d/ld multiples of 8");
  if (R == 0) return 0;
  ESP_CUDA(esp_launch(qprep_bwd_kernel, grid_for(R * (d / 8), 256), 256, 0, st, (const bf16*)dqu, (const bf16*)dqv, scale, R, d,
                      (bf16*)dq, ld_out));
  return 0;
}

extern "C" int esp_attn_softmax_fwd(const void* scores, int32_t H, int32_t B, int32_t Tq, int32_t T, int32_t ld,
                                    const int32_t* lens, int32_t causal, void* p, void* p_drop, float drop_p, uint64_t seed,
                                    const uint64_t* seed_ptr, void* stream) {
  ESP_ST;
  ESP_CHECK(!causal || Tq == T, "causal attention needs Tq == Tk");
  ESP_CHECK(T <= kSmMaxT, "attention length %d exceeds the register softmax limit %d", T, kSmMaxT);
  ESP_CHECK(ld >= T && ld <= kSmMaxT && ld % 8 == 0, "bad score row stride %d", ld);
  ESP_CHECK(drop_p <= 0.f || p_drop != nullptr, "dropout requested but p_drop is null");
  const long rows = (long)H * B * Tq;
  if (rows == 0) return 0;
  const unsigned grid = (unsigned)((rows + 7) / 8);
  bf16* pd = drop_p > 0.f ? (bf16*)p_drop : nullptr;
#define ESP_SMF(NI)                                                                                                      \
  ESP_CUDA(esp_launch(attn_softmax_fwd_kernel<NI, false>, grid, 256, 0, st, (const bf16*)scores, H, B, Tq, T, ld, lens,   \
                      causal, (bf16*)p, pd, drop_p, esp_dropout_thresh(drop_p), seed, (const unsigned long long*)seed_ptr, \
                      1.f, 0.f))
  if (ld <= 256) ESP_SMF(1);
  else if (ld <= 512) ESP_SMF(2);
  else if (ld <= 768) ESP_SMF(3);
  else if (ld <= 1024) ESP_SMF(4);
  else ESP_SMF(5);
#undef ESP_SMF
  return 0;
}

extern "C" int esp_attn_softmax_relaxed_fwd(const void* scores, int32_t H, int32_t B, int32_t Tq, int32_t T, int32_t ld,
                                            const int32_t* lens, void* p, void* p_drop, double relax_w, float drop_p,
                                            uint64_t seed, const uint64_t* seed_ptr, void* stream) {
  ESP_ST;
  ESP_CHECK(T > 0 && T <= kSmMaxT, "attention length %d outside the register softmax range (1..%d)", T, kSmMaxT);
  ESP_CHECK(ld >= T && ld <= kSmMaxT && ld % 8 == 0, "bad score row stride %d", ld);
  ESP_CHECK(relax_w > 0.0 && relax_w <= 1.0, "relaxed attention weight must be in (0, 1] (got %g)", relax_w);
  ESP_CHECK(p && p_drop, "relaxed attention writes both p and p_drop");
  const long rows = (long)H * B * Tq;
  if (rows == 0) return 0;
  const unsigned grid = (unsigned)((rows + 7) / 8);
  // the reference's Python scalars (1 - w, w / src_len) are doubles, applied as fp32 by the bf16 tensor ops
  const float keep_w = (float)(1.0 - relax_w), add_w = (float)(relax_w / T);
#define ESP_SMF(NI)                                                                                                      \
  ESP_CUDA(esp_launch(attn_softmax_fwd_kernel<NI, true>, grid, 256, 0, st, (const bf16*)scores, H, B, Tq, T, ld, lens, 0, \
                      (bf16*)p, (bf16*)p_drop, drop_p, esp_dropout_thresh(drop_p), seed,                                  \
                      (const unsigned long long*)seed_ptr, keep_w, add_w))
  if (ld <= 256) ESP_SMF(1);
  else if (ld <= 512) ESP_SMF(2);
  else if (ld <= 768) ESP_SMF(3);
  else if (ld <= 1024) ESP_SMF(4);
  else ESP_SMF(5);
#undef ESP_SMF
  return 0;
}

extern "C" int esp_attn_softmax_bwd(const void* p, const void* dp_drop, int32_t H, int32_t B, int32_t Tq, int32_t T,
                                    int32_t ld, void* ds, void* dbd, int32_t ldp, float drop_p, uint64_t seed,
                                    const uint64_t* seed_ptr, void* stream) {
  ESP_ST;
  ESP_CHECK(T <= kSmMaxT && ld >= T && ld <= kSmMaxT && ld % 8 == 0, "bad attention softmax-bwd shape");
  ESP_CHECK(dbd == nullptr || (ldp >= 2 * T - 1 && Tq == T), "dBD needs Tq == Tk and ldp >= 2T-1");
  const long rows = (long)H * B * Tq;
  if (rows == 0) return 0;
  const unsigned grid = (unsigned)((rows + 7) / 8);
#define ESP_SMB(NI)                                                                                                      \
  ESP_CUDA(esp_launch(attn_softmax_bwd_kernel<NI>, grid, 256, 0, st, (const bf16*)p, (const bf16*)dp_drop, H, B, Tq, T, ld, \
                      (bf16*)ds, (bf16*)dbd, ldp, drop_p, esp_dropout_thresh(drop_p), seed,                              \
                      (const unsigned long long*)seed_ptr))
  if (ld <= 256) ESP_SMB(1);
  else if (ld <= 512) ESP_SMB(2);
  else if (ld <= 768) ESP_SMB(3);
  else if (ld <= 1024) ESP_SMB(4);
  else ESP_SMB(5);
#undef ESP_SMB
  return 0;
}

extern "C" int esp_glu_dwconv_fwd(const void* g, const void* w, int32_t B, int32_t T, int32_t C, int32_t ksz, void* y,
                                  double* stats, void* stream) {
  ESP_ST;
  ESP_CHECK(C % kDwC == 0, "depthwise conv channels must be a multiple of %d", kDwC);
  ESP_CHECK((ksz & 1) && ksz <= kDwMaxK, "depthwise kernel size must be odd and <= %d", kDwMaxK);
  if ((long)B * T == 0) return 0;
  dim3 grid((T + kDwT - 1) / kDwT, C / kDwC, B);
  ESP_CUDA(esp_launch(glu_dwconv_fwd_kernel, grid, 256, 0, st, (const bf16*)g, (const bf16*)w, B, T, C, ksz, (bf16*)y, stats));
  return 0;
}

extern "C" int esp_glu_dwconv_bwd(const void* dy, const void* g, const void* w, int32_t B, int32_t T, int32_t C, int32_t ksz,
                                  void* dg, float* dw, void* stream) {
  ESP_ST;
  ESP_CHECK(C % kDwC == 0 && (ksz & 1) && ksz <= kDwMaxK, "unsupported depthwise conv shape");
  if ((long)B * T == 0) return 0;
  dim3 grid((T + kDwT - 1) / kDwT, C / kDwC, B);
  constexpr size_t kSmem = sizeof(float) * (2 * (kDwT + kDwMaxK - 1) * (kDwC + 1) + 4 * kDwMaxK * kDwC);
  ESP_SMEM_OPTIN(glu_dwconv_bwd_kernel, kSmem);
  ESP_CUDA(esp_launch(glu_dwconv_bwd_kernel, grid, 256, kSmem, st, (const bf16*)dy, (const bf16*)g, (const bf16*)w, B, T, C, ksz,
                      (bf16*)dg, dw));
  return 0;
}

extern "C" int esp_bn_finalize(const double* stats, int64_t R, int32_t C, float eps, float momentum, float* run_mean,
                               float* run_var, int32_t training, float* mr, void* stream) {
  ESP_ST;
  ESP_CHECK(mr != nullptr, "bn_finalize: null output");
  ESP_CHECK(training ? stats != nullptr : (run_mean && run_var), "bn_finalize: missing statistics");
  ESP_CHECK(!training || R >= 1, "bn_finalize: batch statistics of %lld rows", (long long)R);
  ESP_CUDA(esp_launch(bn_finalize_kernel, (C + 127) / 128, 128, 0, st, stats, R, C, eps, momentum, run_mean, run_var, training,
                      mr));
  return 0;
}

// The BatchNorm reductions keep each thread on one channel group: 256-thread CTAs with C/8 dividing 256.  Every CTA ends
// with one double atomic per channel, so their grids stay at 2 CTAs per SM.
extern "C" int esp_bn_stats(const void* x, const void* pre_bias, int64_t R, int32_t C, double* stats, void* stream) {
  ESP_ST;
  ESP_CHECK(C % 8 == 0 && 256 % (C / 8) == 0, "bn_stats: C/8 must divide 256 (got C=%d)", C);
  if (R == 0) return 0;
  ESP_CUDA(esp_launch(bn_stats_kernel, grid_for(R * (C / 8), 256, 2), 256, 0, st, (const bf16*)x, (const bf16*)pre_bias, R, C,
                      stats));
  return 0;
}

extern "C" int esp_bn_act_fwd(const void* y, const void* pre_bias, int64_t R, int32_t C, const float* mr, const void* gamma,
                              const void* beta, int32_t act, void* z, void* stream) {
  ESP_ST;
  ESP_CHECK(C % 8 == 0, "BatchNorm channels must be a multiple of 8");
  ESP_CHECK(act == 1 || act == 2, "bn_act: act must be 1 (SiLU) or 2 (ReLU)");
  if (R == 0) return 0;
  ESP_CUDA(esp_launch(bn_act_fwd_kernel, grid_for(R * (C / 8), 256), 256, 0, st, (const bf16*)y, (const bf16*)pre_bias, R, C, mr,
                      (const bf16*)gamma, (const bf16*)beta, act, (bf16*)z));
  return 0;
}

extern "C" int esp_bn_act_bwd(const void* dz, const void* y, const void* pre_bias, int64_t R, int32_t C, const float* mr,
                              const void* gamma, const void* beta, int32_t act, double* sums, void* dy, float* dgamma,
                              float* dbeta, void* stream) {
  ESP_ST;
  ESP_CHECK(C % 8 == 0 && 256 % (C / 8) == 0, "bn_act_bwd: C/8 must divide 256 (got C=%d)", C);
  ESP_CHECK(act == 1 || act == 2, "bn_act: act must be 1 (SiLU) or 2 (ReLU)");
  if (R == 0) return 0;
  ESP_CUDA(cudaMemsetAsync(sums, 0, 2 * C * sizeof(double), st));
  ESP_CUDA(esp_launch(bn_act_bwd_reduce_kernel, grid_for(R * (C / 8), 256, 2), 256, 0, st, (const bf16*)dz, (const bf16*)y,
                      (const bf16*)pre_bias, R, C, mr, (const bf16*)gamma, (const bf16*)beta, act, sums));
  // the 2C float coefficients live after the 2C double sums: the workspace is 3C doubles (include/espresso_b200.h)
  float* coef = reinterpret_cast<float*>(sums + 2 * C);
  ESP_CUDA(esp_launch(bn_param_grad_kernel, (C + 127) / 128, 128, 0, st, sums, R, C, dgamma, dbeta, coef));
  ESP_CUDA(esp_launch(bn_act_bwd_apply_kernel, grid_for(R * (C / 8), 256), 256, 0, st, (const bf16*)dz, (const bf16*)y,
                      (const bf16*)pre_bias, R, C, mr, coef, (const bf16*)gamma, (const bf16*)beta, act, (bf16*)dy));
  return 0;
}

// ================================================================================================
// First convolution of the conv front end: ONE input channel (the fbank "image" [B, T, F]) -> Cout.
// espresso/modules/speech_convolutions.py:78-102 with in_channels = 1: a 3x3 convolution whose reduction is 9 long -- not
// GEMM-shaped work.  It is HBM-bound on its OUTPUT (Cout x more bytes than the input): each thread produces 8 channels of
// one output position from 9 cached input samples and writes one 16-byte vector; the gradient of the 9 x Cout taps reads
// dy once (16-byte vectors) and reduces registers -> shared memory -> one atomic per tap, channel and CTA.
// The following convolutions (64 / 128 input channels) are implicit GEMMs on the wgmma kernel (gemm_tcgen05.cu).
// ================================================================================================
namespace {

// x [B, T, F] bf16, w [Cout, 3, 3] bf16, y [B, To, Fo, Cout] bf16.
// The grid stride is a multiple of Cout/8, so a thread keeps the same 8 output channels: their 72 taps live in registers.
// One trip produces kC1Pos ADJACENT output positions along F from one 3 x ((kC1Pos - 1) * SF + 3) window of input samples
// (4.5 cached 2-byte loads + 72 FMAs + one 16-byte store per output vector); 32-bit position arithmetic.
constexpr int kC1Pos = 4;
template <int SF>
__global__ void __launch_bounds__(256)
conv1_fwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w, bf16* __restrict__ y, int B, int T, int F, int Cout,
                 int st, int To, int Fo) {
  esp_pdl();
  constexpr int W = (kC1Pos - 1) * SF + 3;
  const int cv = Cout >> 3;
  const int Fo4 = (Fo + kC1Pos - 1) / kC1Pos;
  const long total = (long)B * To * Fo4 * cv;
  const long i0 = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int c8 = (int)(i0 % cv) * 8;
  float wr[9][8];
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int k = 0; k < 9; ++k) wr[k][j] = bf2f(w[(c8 + j) * 9 + k]);
  const unsigned npos = (unsigned)(total / cv), pstep = (unsigned)(((long)gridDim.x * blockDim.x) / cv);
  for (unsigned pos = (unsigned)(i0 / cv); pos < npos; pos += pstep) {
    const unsigned bt = pos / (unsigned)Fo4;
    const int f4 = (int)(pos - bt * (unsigned)Fo4) * kC1Pos;
    const int b = (int)(bt / (unsigned)To), to = (int)(bt - (unsigned)b * (unsigned)To);
    float xw[3][W];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int t = to * st + r - 1;
      const bf16* xr = x + ((long)b * T + t) * F;
#pragma unroll
      for (int c = 0; c < W; ++c) {
        const int f = f4 * SF + c - 1;
        xw[r][c] = (t >= 0 && t < T && f >= 0 && f < F) ? bf2f(xr[f]) : 0.f;
      }
    }
    bf16* yrow = y + (((long)b * To + to) * Fo + f4) * Cout + c8;
#pragma unroll
    for (int u = 0; u < kC1Pos; ++u) {
      if (f4 + u >= Fo) break;
      float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[j] = fmaf(xw[r][u * SF + c], wr[r * 3 + c][j], acc[j]);
      store8(yrow + (long)u * Cout, acc);
    }
  }
}

// dw[co, tap] += sum_{b, to, fo} dy[b, to, fo, co] * x[b, to*st + r - 1, fo*sf + c - 1]
// Same thread mapping (fixed 8 channels per thread, 72 register accumulators).  One trip covers kC1Pos ADJACENT output
// positions along F: their dy vectors are loaded first (kC1Pos 16-byte loads in flight per thread) and they share one
// 3 x ((kC1Pos - 1) * SF + 3) window of input samples.
template <int SF>
__global__ void __launch_bounds__(256, 2)
conv1_wgrad_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x, float* __restrict__ dw, int B, int T, int F,
                   int Cout, int st, int To, int Fo) {
  esp_pdl();
  extern __shared__ float c1red[];  // [72 values][256 threads]: conflict-free
  constexpr int W = (kC1Pos - 1) * SF + 3;
  const int cv = Cout >> 3;
  const int Fo4 = (Fo + kC1Pos - 1) / kC1Pos;
  const long total = (long)B * To * Fo4 * cv;
  float acc[9][8];
#pragma unroll
  for (int k = 0; k < 9; ++k)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[k][j] = 0.f;
  const int c8 = (int)(((long)blockIdx.x * blockDim.x + threadIdx.x) % cv) * 8;
  const unsigned npos = (unsigned)(total / cv), pstep = (unsigned)(((long)gridDim.x * blockDim.x) / cv);
  for (unsigned pos = (unsigned)(((long)blockIdx.x * blockDim.x + threadIdx.x) / cv); pos < npos; pos += pstep) {
    const unsigned bt = pos / (unsigned)Fo4;
    const int f4 = (int)(pos - bt * (unsigned)Fo4) * kC1Pos;
    const int b = (int)(bt / (unsigned)To), to = (int)(bt - (unsigned)b * (unsigned)To);
    uint4 dq[kC1Pos];
    const bf16* drow = dy + (((long)b * To + to) * Fo + f4) * Cout + c8;
#pragma unroll
    for (int u = 0; u < kC1Pos; ++u)
      dq[u] = (f4 + u < Fo) ? *reinterpret_cast<const uint4*>(drow + (long)u * Cout) : make_uint4(0, 0, 0, 0);
    float xw[3][W];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int t = to * st + r - 1;
      const bf16* xr = x + ((long)b * T + t) * F;
#pragma unroll
      for (int c = 0; c < W; ++c) {
        const int f = f4 * SF + c - 1;
        xw[r][c] = (t >= 0 && t < T && f >= 0 && f < F) ? bf2f(xr[f]) : 0.f;
      }
    }
#pragma unroll
    for (int u = 0; u < kC1Pos; ++u) {
      float d[8];
      unpack8(dq[u], d);
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[r * 3 + c][j] = fmaf(d[j], xw[r][u * SF + c], acc[r * 3 + c][j]);
    }
  }
#pragma unroll
  for (int k = 0; k < 9; ++k)
#pragma unroll
    for (int j = 0; j < 8; ++j) c1red[(k * 8 + j) * 256 + threadIdx.x] = acc[k][j];
  __syncthreads();
  // threads with the same (threadIdx.x % cv) hold the same channels: fold them, then one atomic per (channel, tap)
  for (int o = threadIdx.x; o < 72 * cv; o += blockDim.x) {
    const int g = o % cv, kj = o / cv;  // kj = tap * 8 + j
    float sacc = 0.f;
    for (int th = g; th < 256; th += cv) sacc += c1red[kj * 256 + th];
    atomicAdd(dw + (g * 8 + (kj & 7)) * 9 + (kj >> 3), sacc);
  }
}

}  // namespace

extern "C" int esp_conv3x3_c1_fwd(const void* x, const void* w, void* y, int32_t B, int32_t T, int32_t F, int32_t Cout,
                                  int32_t st, int32_t sf, void* stream) {
  cudaStream_t st_ = (cudaStream_t)stream;
  ESP_CHECK(Cout % 8 == 0 && 256 % (Cout / 8) == 0, "conv3x3 (1 input channel): Cout/8 must divide 256 (got %d)", Cout);
  ESP_CHECK(st >= 1 && (sf == 1 || sf == 2), "conv3x3 (1 input channel): frequency stride 1 or 2 (got %d)", sf);
  const int To = (T + st - 1) / st, Fo = (F + sf - 1) / sf;
  const long total = (long)B * To * ((Fo + kC1Pos - 1) / kC1Pos) * (Cout / 8);
  if (total == 0) return 0;
  const int grid = grid_for(total, 256);
  if (sf == 1)
    ESP_CUDA(esp_launch(conv1_fwd_kernel<1>, grid, 256, 0, st_, (const bf16*)x, (const bf16*)w, (bf16*)y, B, T, F, Cout, st, To,
                        Fo));
  else
    ESP_CUDA(esp_launch(conv1_fwd_kernel<2>, grid, 256, 0, st_, (const bf16*)x, (const bf16*)w, (bf16*)y, B, T, F, Cout, st, To,
                        Fo));
  return 0;
}

extern "C" int esp_conv3x3_c1_wgrad(const void* dy, const void* x, float* dw, int32_t B, int32_t T, int32_t F, int32_t Cout,
                                    int32_t st, int32_t sf, void* stream) {
  cudaStream_t st_ = (cudaStream_t)stream;
  ESP_CHECK(Cout % 8 == 0 && 256 % (Cout / 8) == 0, "conv3x3 (1 input channel) wgrad: Cout/8 must divide 256 (got %d)", Cout);
  ESP_CHECK(st >= 1 && (sf == 1 || sf == 2), "conv3x3 (1 input channel) wgrad: time stride >= 1 and frequency stride 1 or 2 (got %d, %d)",
            st, sf);
  const int To = (T + st - 1) / st, Fo = (F + sf - 1) / sf;
  const long total = (long)B * To * ((Fo + kC1Pos - 1) / kC1Pos) * (Cout / 8);
  if (total == 0) return 0;
  const int smem = 72 * 256 * (int)sizeof(float);
  const int grid = grid_for(total, 256, 2);  // one wave of resident CTAs: each ends with 9 x Cout atomics
  if (sf == 1) {
    ESP_SMEM_OPTIN(conv1_wgrad_kernel<1>, smem);
    ESP_CUDA(esp_launch(conv1_wgrad_kernel<1>, grid, 256, smem, st_, (const bf16*)dy, (const bf16*)x, dw, B, T, F, Cout, st, To,
                        Fo));
  } else {
    ESP_SMEM_OPTIN(conv1_wgrad_kernel<2>, smem);
    ESP_CUDA(esp_launch(conv1_wgrad_kernel<2>, grid, 256, smem, st_, (const bf16*)dy, (const bf16*)x, dw, B, T, F, Cout, st, To,
                        Fo));
  }
  return 0;
}
