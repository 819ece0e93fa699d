// espresso_b200 -- fused relative-position self-attention forward for sm_90a (H100).
//
//   ctx[b, i, h] = sum_j dropout( softmax_j( qu_i . k_j + qv_i . p_{(T-1)-i+j}  (+ key-padding mask) ) )[i, j] v_j
//
// Reference (rel-pos branch of fairseq/modules/multihead_attention.py): scores AC = q_u k^T (:788), BD = q_v pos^T over
// the 2T-1 relative positions (:815-823), the Transformer-XL skew BD[i, j] <- BD_full[i, (T-1)-i+j] (:824-830), key-padding
// mask -> -inf (:841-859), fp32 softmax cast back to the model dtype (:864-867), dropout, P v (:897).  The reference (and
// the round-1 build) round-trips BD_full, the scores, the probabilities and the dropped probabilities through HBM; here
// the scores and the relative-position logits never leave the SM:
//
//   * one CTA per (128-query tile, head, utterance); key tiles of 128 are streamed with TMA (SWIZZLE_128B) through a
//     2-stage ring (K, V) and a 3-slot ring of 128-row relative-position blocks; one warp issues the loads;
//   * two warpgroups own 64 query rows each.  Per key tile a warpgroup computes with wgmma (accumulators in registers)
//     W = Qv [Pblk_lo; Pblk_hi]^T -- the 255 relative positions this (query tile, key tile) pair can see -- and stages it
//     in shared memory as bf16 (as the reference keeps BD), then S = Qu K^T.  The skew is a column re-index of the
//     staged rows: BD[r, c] = W[r, 127 - r + c].  A row's W values are written and read by the same four lanes, so the
//     staging needs no barrier beyond the warp;
//   * two passes over the key tiles: pass 1 accumulates the row maximum and the normaliser online, pass 2 recomputes the
//     logits, forms the NORMALISED probabilities in registers, writes them (bf16) for the backward pass, applies the
//     counter-RNG dropout (same stream as esp_attn_softmax_fwd/bwd) and accumulates O += P V with the dropped
//     probabilities as the register A operand of wgmma.  Normalising before P V removes the online-softmax rescale of O.
//
// Outputs: ctx [B*T, d] bf16; when `p_out` is given (training) the probabilities P [H,B,T,ld] and, with dropout, the
// dropped probabilities Pd -- exactly what esp_attn_softmax_fwd produced, so the existing backward kernels are unchanged.
#include "common.cuh"
#include "espresso_b200.h"
#include "sm90.cuh"
#include <cuda.h>
#include <stdlib.h>

namespace {

using namespace sm90;

constexpr int kTile = 128;      // query rows per CTA = key columns per step
constexpr int kHd = 64;         // head dim (one SWIZZLE_128B row of bf16)
constexpr int kThreads = 288;   // warps 0-7: two MMA / softmax warpgroups (64 query rows each), warp 8: TMA
constexpr int kTileBytes = kTile * kHd * 2;  // 16 KB
constexpr int kWLd = 264;                    // W staging row: 256 bf16 + 8 pad (conflict-free fragment stores)
constexpr int kOffQu = 0;
constexpr int kOffQv = kOffQu + kTileBytes;
constexpr int kOffK = kOffQv + kTileBytes;         // 2 stages
constexpr int kOffV = kOffK + 2 * kTileBytes;      // 2 stages
constexpr int kOffP = kOffV + 2 * kTileBytes;      // 3 relative-position blocks
constexpr int kOffW = kOffP + 3 * kTileBytes;      // W staging, 128 rows x kWLd bf16
constexpr int kOffBar = kOffW + kTile * kWLd * 2;
constexpr int kSmemBytes = kOffBar + 128 + 1024;   // barriers, alignment slack

struct Params {
  int B, T, H, d, ld;       // ld: row stride of the probability tensors (multiple of 8, >= T)
  int pos_hstride;          // head stride (elements) inside a projected-position row: hd, or 0 (table shared by heads)
  const int* lens;          // valid keys per utterance or nullptr
  const int* key_lo;        // optional per-query-row visible key range [key_lo[i], key_hi[i]) (streaming / context masks)
  const int* key_hi;
  bf16* ctx;                // [B*T, d]
  bf16* p_out;              // [H, B, T, ld] or nullptr
  bf16* pd_out;             // [H, B, T, ld] or nullptr (no dropout)
  float drop_p;
  uint32_t thresh;
  unsigned long long seed;
  const unsigned long long* seed_ptr;
};

__global__ void __launch_bounds__(kThreads, 1)
attn_fused_fwd_kernel(const __grid_constant__ CUtensorMap tmQu, const __grid_constant__ CUtensorMap tmQv,
                      const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                      const __grid_constant__ CUtensorMap tmP, const Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const uint32_t sb = smem_u32(smem);
  const uint32_t bar0 = sb + kOffBar;
  // mbarriers: Q | K + positions loaded, stage 0,1 | V loaded, stage 0,1 | K stage read, 0,1 | V stage read, 0,1
  const uint32_t barQ = bar0, barK0 = bar0 + 8, barV0 = bar0 + 24, barKR0 = bar0 + 40, barVR0 = bar0 + 56;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int T = p.T;
  const int i0 = qt * kTile;
  const int nkt = (T + kTile - 1) / kTile;  // key tiles
  const int total = 2 * nkt;                // pass 1 (statistics) + pass 2 (probabilities, P V)
  const int wbase = (T - 1) - i0 - (kTile - 1);  // relative position seen by (row 127, key 0); block a = wbase + 128 a

  esp_pdl_trigger();
  if (threadIdx.x == 256) {
    mbar_init(barQ, 1);
    for (int s = 0; s < 2; ++s) {
      mbar_init(barK0 + 8 * s, 1);
      mbar_init(barV0 + 8 * s, 1);
      mbar_init(barKR0 + 8 * s, 8);  // one arrive per MMA warp
      mbar_init(barVR0 + 8 * s, 8);
    }
    fence_mbar_init();
    prefetch_tmap(&tmQu);
    prefetch_tmap(&tmK);
    prefetch_tmap(&tmP);
  }
  __syncthreads();
  esp_pdl_wait();

  if (warp == 8) {
    // ============================== TMA loads (one thread) ======================================================
    if (lane == 0) {
      const int pcol = h * p.pos_hstride;
      // K tile + relative-position blocks of iteration `it`.  Block a lives in ring slot a % 3; within a pass tile jt needs
      // blocks jt (loaded by the previous iteration) and jt + 1.
      auto load_k = [&](int it) {
        const int jt = it % nkt, st = it & 1;
        const bool first = jt == 0;
        const uint32_t bar = barK0 + 8 * st;
        mbar_expect_tx(bar, (uint32_t)kTileBytes * (first ? 3 : 2));
        tma_load_4d(sb + kOffK + st * kTileBytes, &tmK, bar, h * kHd, jt * kTile, b, 0);
        if (first) tma_load_4d(sb + kOffP + (jt % 3) * kTileBytes, &tmP, bar, pcol, wbase + jt * kTile, 0, 0);
        tma_load_4d(sb + kOffP + ((jt + 1) % 3) * kTileBytes, &tmP, bar, pcol, wbase + (jt + 1) * kTile, 0, 0);
      };
      // iteration `it` has read its K stage and relative-position blocks (stage barrier it & 1, use it >> 1)
      auto wait_k_read = [&](int it) { mbar_wait(barKR0 + 8 * (it & 1), (it >> 1) & 1); };
      mbar_expect_tx(barQ, 2 * kTileBytes);
      tma_load_4d(sb + kOffQu, &tmQu, barQ, h * kHd, i0, b, 0);
      tma_load_4d(sb + kOffQv, &tmQv, barQ, h * kHd, i0, b, 0);
      load_k(0);
      for (int it = 0; it < total; ++it) {
        if (it + 1 < total) {
          // K stage (it+1)&1 and ring slot (jt+2)%3 were last read by iteration it-1.  Across the pass boundary the ring
          // restarts at block 0 and would overwrite blocks THIS iteration reads: wait for it instead.
          if ((it + 1) % nkt == 0) wait_k_read(it);
          else if (it >= 1) wait_k_read(it - 1);
          load_k(it + 1);
        }
        if (it >= nkt) {
          // V tile of this pass-2 tile; its stage was last read by P V(jt-2)
          const int jt = it - nkt;
          if (jt >= 2) mbar_wait(barVR0 + 8 * (jt & 1), ((jt - 2) >> 1) & 1);
          const uint32_t bar = barV0 + 8 * (jt & 1);
          mbar_expect_tx(bar, kTileBytes);
          tma_load_4d(sb + kOffV + (jt & 1) * kTileBytes, &tmV, bar, h * kHd, jt * kTile, b, 0);
        }
      }
    }
  } else {
    // ============================== MMA + softmax warpgroups =====================================================
    const int wg = warp >> 2;
    const int t = threadIdx.x & 127;
    // accumulator fragment rows of this thread (tile-local): fr and fr + 8; columns 8 j + fc, + 1 for j = 0..15
    const int fr = wg * 64 + (t >> 5) * 16 + ((t & 31) >> 2), fc = 2 * (t & 3);
    const unsigned long long seed = p.seed + (p.seed_ptr ? *p.seed_ptr : 0ull);
    const float dscale = p.drop_p > 0.f ? 65536.f / (65536.f - (float)p.thresh) : 1.f;
    const float kLog2e = 1.4426950408889634f;
    const int klen = p.lens ? min(p.lens[b], T) : T;
    int kmin[2] = {0, 0}, kmax[2] = {T, T};
    long prow[2];
    bool row_ok[2];
#pragma unroll
    for (int x = 0; x < 2; ++x) {
      const int qi = i0 + fr + 8 * x;
      row_ok[x] = qi < T;
      prow[x] = ((long)h * p.B + b) * T + qi;  // row of the probability tensors
      if (p.key_lo) {  // chunk-streaming / limited-context attention: a contiguous key range per query row
        const int qr = min(qi, T - 1);
        kmin[x] = p.key_lo[qr];
        kmax[x] = p.key_hi[qr];
      }
    }
    bf16* const wst = reinterpret_cast<bf16*>(smem + kOffW);
    const uint32_t sqv = sb + kOffQv + wg * (64 * 128), squ = sb + kOffQu + wg * (64 * 128);
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f}, inv_l[2] = {0.f, 0.f};
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    mbar_wait(barQ, 0);

    for (int it = 0; it < total; ++it) {
      const int jt = it % nkt, st = it & 1;
      const bool pass2 = it >= nkt;
      mbar_wait(barK0 + 8 * st, (it >> 1) & 1);
      const uint32_t sk = sb + kOffK + st * kTileBytes;
      float acc[64];
      // ---- W = Qv [P_jt; P_jt+1]^T, one 128-column half at a time, staged as bf16 rows of 256 relative positions ----
#pragma unroll 1
      for (int half = 0; half < 2; ++half) {
        const uint32_t pblk = sb + kOffP + ((jt + half) % 3) * kTileBytes;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kHd / 16; ++k)
          wgmma_ss_n128<0, 0>(acc, make_sdesc(sqv + k * 32, 16, 1024), make_sdesc(pblk + k * 32, 16, 1024), k);
        wgmma_commit();
        wgmma_wait<0>();
        fence_acc(acc);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int c = half * 128 + 8 * j + fc;
          *reinterpret_cast<uint32_t*>(wst + fr * kWLd + c) = pack_bf16x2(acc[4 * j], acc[4 * j + 1]);
          *reinterpret_cast<uint32_t*>(wst + (fr + 8) * kWLd + c) = pack_bf16x2(acc[4 * j + 2], acc[4 * j + 3]);
        }
      }
      // ---- S = Qu K^T ----
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kHd / 16; ++k)
        wgmma_ss_n128<0, 0>(acc, make_sdesc(squ + k * 32, 16, 1024), make_sdesc(sk + k * 32, 16, 1024), k);
      wgmma_commit();
      wgmma_wait<0>();
      fence_acc(acc);
      // the K stage and the position blocks are consumed: the loader may refill them
      __syncwarp();
      if (lane == 0) mbar_arrive(barKR0 + 8 * st);
      // ---- logits s = S + W[r, 127 - r + c], masked beyond the utterance's keys (in place in acc) ----
      float tmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int x = 0; x < 2; ++x)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int r = fr + 8 * x, c = 8 * j + fc + e;
            const int key = jt * kTile + c;
            float a = acc[4 * j + 2 * x + e] + bf2f(wst[r * kWLd + (kTile - 1) - r + c]);
            if (p.key_lo && (key < kmin[x] || key >= kmax[x])) {
              // hidden keys: the reference ADDS bf16(-1e4) to its bf16 scores (transformer_layer.py:189-192,
              // multihead_attention.py:835-839) -- finite, so a row whose visible keys are all padding still
              // normalises over the hidden ones
              a = __bfloat162float(__float2bfloat16_rn(a - 9984.f));
            }
            a = key < klen ? a : -INFINITY;  // key padding: -inf (:841-859)
            acc[4 * j + 2 * x + e] = a;
            tmax[x] = fmaxf(tmax[x], a);
          }
      if (!pass2) {
        // ---- pass 1: online maximum and normaliser; the four lanes of a quad share a row ----
#pragma unroll
        for (int x = 0; x < 2; ++x) {
          tmax[x] = fmaxf(tmax[x], __shfl_xor_sync(0xffffffffu, tmax[x], 1));
          tmax[x] = fmaxf(tmax[x], __shfl_xor_sync(0xffffffffu, tmax[x], 2));
          const float m_new = fmaxf(m_run[x], tmax[x]);
          float sum = 0.f;
          if (m_new > -INFINITY) {
            const float mb = m_new * kLog2e;
#pragma unroll
            for (int j = 0; j < 16; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e) sum += exp2f(fmaf(acc[4 * j + 2 * x + e], kLog2e, -mb));  // exp2(-inf) = 0
          }
          sum += __shfl_xor_sync(0xffffffffu, sum, 1);
          sum += __shfl_xor_sync(0xffffffffu, sum, 2);
          if (m_new > -INFINITY) {
            l_run[x] = (m_run[x] > -INFINITY ? l_run[x] * exp2f((m_run[x] - m_new) * kLog2e) : 0.f) + sum;
            m_run[x] = m_new;
          }
          if (it == nkt - 1) inv_l[x] = l_run[x] > 0.f ? 1.f / l_run[x] : 0.f;
        }
      } else {
        // ---- pass 2: normalised probabilities, dropout, register A operand of P V ----
        const int tj = it - nkt;
        uint32_t afrag[32];
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
          for (int x = 0; x < 2; ++x) {
            const float mb = m_run[x] * kLog2e;
            float pr[2], pd[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float pv = exp2f(fmaf(acc[4 * j + 2 * x + e], kLog2e, -mb)) * inv_l[x];
              pr[e] = bf2f(f2bf(pv));  // softmax in fp32, cast to the model dtype (fairseq/utils.py:514-525 + .type_as)
              pd[e] = pr[e];
            }
            const int key = jt * kTile + 8 * j + fc;
            const unsigned long long idx = (unsigned long long)prow[x] * p.ld + key;
            if (p.drop_p > 0.f) {
              // idx is even and prow * ld a multiple of 8: both elements are lanes of the same 4-element hash group
              const unsigned long long hsh = esp_hash_u64(seed, idx >> 2);
#pragma unroll
              for (int e = 0; e < 2; ++e)
                pd[e] = ((uint32_t)(hsh >> (16 * ((idx & 3) + e))) & 0xFFFFu) >= p.thresh ? pd[e] * dscale : 0.f;
            }
            const uint32_t wpr = pack_bf16x2(pr[0], pr[1]), wpd = pack_bf16x2(pd[0], pd[1]);
            afrag[2 * j + x] = wpd;
            if (row_ok[x] && key < p.ld) {
              if (p.p_out) *reinterpret_cast<uint32_t*>(p.p_out + prow[x] * p.ld + key) = wpr;
              if (p.pd_out) *reinterpret_cast<uint32_t*>(p.pd_out + prow[x] * p.ld + key) = wpd;
            }
          }
        mbar_wait(barV0 + 8 * (tj & 1), (tj >> 1) & 1);
        const uint32_t sv = sb + kOffV + (tj & 1) * kTileBytes;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kTile / 16; ++k) {
          // A fragment of keys 16k .. 16k+15: accumulator column groups 2k and 2k+1, rows fr and fr + 8
          const uint32_t a4[4] = {afrag[4 * k], afrag[4 * k + 1], afrag[4 * k + 2], afrag[4 * k + 3]};
          wgmma_rs_n64<1>(o, a4, make_sdesc(sv + k * 2048, kTileBytes, 1024), 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        fence_acc(o);
        __syncwarp();
        if (lane == 0) mbar_arrive(barVR0 + 8 * (tj & 1));
      }
    }
    // ---- epilogue: O (already normalised) -> ctx ----
#pragma unroll
    for (int x = 0; x < 2; ++x) {
      if (!row_ok[x]) continue;
      bf16* dst = p.ctx + ((long)b * T + i0 + fr + 8 * x) * p.d + h * kHd + fc;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack_bf16x2(o[4 * j + 2 * x], o[4 * j + 2 * x + 1]);
    }
  }
}

}  // namespace

int esp_make_tmap_bf16(CUtensorMap* tm, const void* base, long inner, long rows, long ld, int nb1, long s1, int nb2,
                       long s2, int box_rows);  // gemm_tcgen05.cu

extern "C" int esp_attn_fused_fwd(const void* qu, const void* qv, int64_t ldq, const void* k, const void* v, int64_t ldkv,
                                  const void* pos, int64_t ldpos, int32_t pos_hstride, int32_t B, int32_t T, int32_t H,
                                  int32_t head_dim, const int32_t* lens, const int32_t* key_lo, const int32_t* key_hi,
                                  void* ctx, int64_t ldctx, void* p_out, void* pd_out, int32_t ldp, float drop_p,
                                  uint64_t seed, const uint64_t* seed_ptr, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(head_dim == kHd, "fused attention is built for head_dim 64 (got %d)", head_dim);
  ESP_CHECK(B >= 0 && T >= 0 && H > 0, "bad attention shape");
  if (B == 0 || T == 0) return 0;
  ESP_CHECK(qu && qv && k && v && pos && ctx, "null pointer passed to esp_attn_fused_fwd");
  ESP_CHECK(p_out == nullptr || (ldp >= T && ldp % 8 == 0), "probability row stride must be a multiple of 8 and >= T");
  ESP_CHECK(drop_p <= 0.f || p_out == nullptr || pd_out != nullptr, "dropout with saved probabilities needs pd_out");
  ESP_CHECK(ldctx == (int64_t)H * kHd, "ctx must be [B*T, H*64] contiguous");
  ESP_CHECK(B <= 65535 && H <= 65535, "grid limits");
  CUtensorMap tqu, tqv, tk, tv, tp;
  int rc;
  if ((rc = esp_make_tmap_bf16(&tqu, qu, (long)H * kHd, T, ldq, B, (long)T * ldq, 1, 0, kTile))) return rc;
  if ((rc = esp_make_tmap_bf16(&tqv, qv, (long)H * kHd, T, ldq, B, (long)T * ldq, 1, 0, kTile))) return rc;
  if ((rc = esp_make_tmap_bf16(&tk, k, (long)H * kHd, T, ldkv, B, (long)T * ldkv, 1, 0, kTile))) return rc;
  if ((rc = esp_make_tmap_bf16(&tv, v, (long)H * kHd, T, ldkv, B, (long)T * ldkv, 1, 0, kTile))) return rc;
  const long pos_cols = pos_hstride ? (long)H * kHd : kHd;
  if ((rc = esp_make_tmap_bf16(&tp, pos, pos_cols, 2L * T - 1, ldpos, 1, 0, 1, 0, kTile))) return rc;
  Params pr;
  pr.B = B; pr.T = T; pr.H = H; pr.d = (int)ldctx; pr.ld = ldp; pr.pos_hstride = pos_hstride;
  ESP_CHECK((key_lo == nullptr) == (key_hi == nullptr), "key_lo and key_hi must be given together");
  pr.key_lo = key_lo; pr.key_hi = key_hi;
  pr.lens = lens; pr.ctx = (bf16*)ctx; pr.p_out = (bf16*)p_out; pr.pd_out = drop_p > 0.f ? (bf16*)pd_out : nullptr;
  pr.drop_p = drop_p; pr.thresh = esp_dropout_thresh(drop_p); pr.seed = seed;
  pr.seed_ptr = (const unsigned long long*)seed_ptr;
  ESP_SMEM_OPTIN(attn_fused_fwd_kernel, kSmemBytes);
  dim3 grid((T + kTile - 1) / kTile, H, B);
  ESP_CUDA(esp_launch(attn_fused_fwd_kernel, grid, kThreads, kSmemBytes, st, tqu, tqv, tk, tv, tp, pr));
  return 0;
}
