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
//   * one CTA per (128-query tile, head, utterance), three warpgroups.  Warpgroup 0 is the producer: one thread streams
//     the key tiles (K, V: 2-stage rings) and the 128-row relative-position blocks (2-slot ring) with TMA (SWIZZLE_128B).
//     Warpgroups 1-2 own 64 query rows each and do all the math.  setmaxnreg moves registers from the producer (24 per
//     thread; its code uses R0-R11) to the math warpgroups (240).  ptxas (CUDA 12.9) still keeps the math body within
//     R0-R165 of the launch's 168, but only with this split does it report 0 spill bytes (at 232: 60 B; without
//     setmaxnreg: 92 B).  The W staging is addressed in the shared window (LDS / STS), not through generic pointers;
//   * W_a = Qv Pblk_a^T is the 128 relative positions of position block a (wgmma m64n128k16, fp32 accumulators) as this
//     query tile sees them.  Key tile jt needs blocks jt and jt + 1: the 255 relative positions of the (query tile, key
//     tile) pair.  Each block's W half is computed ONCE per pass and staged as bf16 (as the reference keeps BD) in a
//     256-column row buffer: [W_jt | W_jt+1]; after tile jt the right half is moved to the left and W_jt+2 is stored on
//     the right.  The skew is a column re-index of the staged rows: BD[r, c] = W[r, 127 - r + c].  A row's W values are
//     written, moved and read by the same four lanes, so the staging needs no barrier beyond the warp;
//   * per key tile the wgmma groups are W_jt+1, S_jt and (pass 2) P V_jt.  P V_jt is retired at the next tile, together
//     with W_jt+2, so it runs behind the W move and the next tile's MMA issue; its register A fragments stay live until
//     then.  Keeping W_jt+2 in flight through the softmax as well needs a second 64-float accumulator, which at 168
//     registers made ptxas serialise every wgmma;
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
constexpr int kThreads = 384;   // warpgroup 0: TMA producer; warpgroups 1-2: MMA / softmax (64 query rows each)
constexpr int kProducerRegs = 24, kConsumerRegs = 240;  // 128 * 24 + 256 * 240 <= 64K registers
constexpr int kTileBytes = kTile * kHd * 2;  // 16 KB
constexpr int kWLd = 264;                    // W staging row: 256 bf16 + 8 pad (conflict-free fragment stores)
constexpr int kOffQu = 0;
constexpr int kOffQv = kOffQu + kTileBytes;
constexpr int kOffK = kOffQv + kTileBytes;         // 2 stages
constexpr int kOffV = kOffK + 2 * kTileBytes;      // 2 stages
constexpr int kOffP = kOffV + 2 * kTileBytes;      // 2 relative-position blocks
constexpr int kOffW = kOffP + 2 * kTileBytes;      // W staging, 128 rows x kWLd bf16
// the instance without positions (kPos = false) has no position ring and no W staging: its barriers follow the V ring
template <bool kPos>
constexpr int kOffBar = kPos ? kOffW + kTile * kWLd * 2 : kOffP;
template <bool kPos>
constexpr int kSmemBytes = kOffBar<kPos> + 128 + 1024;   // barriers, alignment slack

// Profiling build only (-DESP_ATTN_FWD_PHASES, made by profiles/attn_fwd_ab.py --phases): thread 0 of each math
// warpgroup adds the SM clocks spent in each phase of the key-tile loop to g_attn_fwd_phase_clk.
enum { kPhW, kPhStageW, kPhS, kPhLogits, kPhStats, kPhProbs, kPhPV, kPhMoveW, kPhases };
#ifdef ESP_ATTN_FWD_PHASES
__device__ unsigned long long g_attn_fwd_phase_clk[kPhases];
#define ESP_PHASE(i)                                    \
  if (t == 0) {                                         \
    const long long c_ = clock64();                     \
    ph_clk[i] += c_ - ph_t;                             \
    ph_t = c_;                                          \
  }
#else
#define ESP_PHASE(i)
#endif

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

// kPos = false: plain scaled dot-product attention, s = q k^T (q already scaled).  No position block is loaded, no W
// group issued, staged or moved, and no skew read; tmQv and tmP are not used.  Everything else -- the two passes, the
// saved P / Pd, the dropout stream, the key-padding and key-range rules -- is the same code as the kPos instance.
template <bool kPos>
__global__ void __launch_bounds__(kThreads, 1)
attn_fused_fwd_kernel(const __grid_constant__ CUtensorMap tmQu, const __grid_constant__ CUtensorMap tmQv,
                      const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                      const __grid_constant__ CUtensorMap tmP, const Params p) {
  extern __shared__ uint8_t smem_raw[];
  // offset from smem_raw (not an integer round trip), so the compiler keeps the shared address space: LDS / STS
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t sb = smem_u32(smem);
  const uint32_t bar0 = sb + kOffBar<kPos>;
  // mbarriers, stages / slots 0,1 each: Q | K loaded | V loaded | position block loaded | K read | V read | block read
  const uint32_t barQ = bar0, barK0 = bar0 + 8, barV0 = bar0 + 24, barP0 = bar0 + 40, barKR0 = bar0 + 56,
                 barVR0 = bar0 + 72, barPR0 = bar0 + 88;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int T = p.T;
  const int i0 = qt * kTile;
  const int nkt = (T + kTile - 1) / kTile;  // key tiles; a pass reads position blocks 0 .. nkt
  const int wbase = (T - 1) - i0 - (kTile - 1);  // relative position seen by (row 127, key 0); block a = wbase + 128 a

  esp_pdl_trigger();
  if (threadIdx.x == 0) {
    mbar_init(barQ, 1);
    for (int s = 0; s < 2; ++s) {
      mbar_init(barK0 + 8 * s, 1);
      mbar_init(barV0 + 8 * s, 1);
      mbar_init(barP0 + 8 * s, 1);
      mbar_init(barKR0 + 8 * s, 8);  // one arrive per MMA warp
      mbar_init(barVR0 + 8 * s, 8);
      mbar_init(barPR0 + 8 * s, 8);
    }
    fence_mbar_init();
    prefetch_tmap(&tmQu);
    prefetch_tmap(&tmK);
    if constexpr (kPos) prefetch_tmap(&tmP);
  }
  __syncthreads();
  esp_pdl_wait();

  if (warp < 4) {
    // ============================== TMA loads (one thread) ======================================================
    setmaxnreg_dec<kProducerRegs>();
    if (threadIdx.x == 0) {
      const int pcol = h * p.pos_hstride;
      // Issue order = the order in which the consumers first wait: per pass blocks 0, 1, then per key tile K_jt,
      // block jt + 2, V_jt (pass 2).  Each ring slot is refilled once the consumers released its previous content.
      int pseq = 0;
      auto load_pos = [&](int a) {
        const int s = pseq & 1;
        if (pseq >= 2) mbar_wait(barPR0 + 8 * s, ((pseq >> 1) - 1) & 1);
        mbar_expect_tx(barP0 + 8 * s, kTileBytes);
        tma_load_4d(sb + kOffP + s * kTileBytes, &tmP, barP0 + 8 * s, pcol, wbase + a * kTile, 0, 0);
        ++pseq;
      };
      mbar_expect_tx(barQ, (kPos ? 2 : 1) * kTileBytes);
      tma_load_4d(sb + kOffQu, &tmQu, barQ, h * kHd, i0, b, 0);
      if constexpr (kPos) tma_load_4d(sb + kOffQv, &tmQv, barQ, h * kHd, i0, b, 0);
      for (int pass = 0; pass < 2; ++pass) {
        if constexpr (kPos) {
          load_pos(0);
          load_pos(1);
        }
        for (int jt = 0; jt < nkt; ++jt) {
          const int it = pass * nkt + jt, st = it & 1;
          if (it >= 2) mbar_wait(barKR0 + 8 * st, ((it >> 1) - 1) & 1);
          mbar_expect_tx(barK0 + 8 * st, kTileBytes);
          tma_load_4d(sb + kOffK + st * kTileBytes, &tmK, barK0 + 8 * st, h * kHd, jt * kTile, b, 0);
          if (kPos && jt + 2 <= nkt) load_pos(jt + 2);
          if (pass == 1) {
            if (jt >= 2) mbar_wait(barVR0 + 8 * (jt & 1), ((jt >> 1) - 1) & 1);
            mbar_expect_tx(barV0 + 8 * (jt & 1), kTileBytes);
            tma_load_4d(sb + kOffV + (jt & 1) * kTileBytes, &tmV, barV0 + 8 * (jt & 1), h * kHd, jt * kTile, b, 0);
          }
        }
      }
    }
  } else {
    // ============================== MMA + softmax warpgroups =====================================================
    setmaxnreg_inc<kConsumerRegs>();
    const int wg = (warp >> 2) - 1;
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
    // Dropout: one hash covers a 4-element group, i.e. the keys of a lane pair (t & 3 = 0,1 or 2,3) in one row.  Lane t
    // hashes row x = t & 1 and hands its partner the 32-bit half the partner's two keys use.
    const unsigned long long hrow = (unsigned long long)((t & 1) ? prow[1] : prow[0]) * p.ld;
    bf16* const wst = reinterpret_cast<bf16*>(smem + kOffW);
    const uint32_t sqv = sb + kOffQv + wg * (64 * 128), squ = sb + kOffQu + wg * (64 * 128);
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f}, inv_l[2] = {0.f, 0.f};
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    float accW[64], accS[64];
    uint32_t afrag[32];
    int pseq = 0;  // position blocks consumed (ring slot pseq & 1)

    auto issue_w = [&]() {  // W of the next position block into accW (one wgmma group)
      const int s = pseq & 1;
      mbar_wait(barP0 + 8 * s, (pseq >> 1) & 1);
      const uint32_t pblk = sb + kOffP + s * kTileBytes;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kHd / 16; ++k)
        wgmma_ss_n128<0, 0>(accW, make_sdesc(sqv + k * 32, 16, 1024), make_sdesc(pblk + k * 32, 16, 1024), k);
      wgmma_commit();
    };
    auto release = [&](uint32_t bar) {
      __syncwarp();
      if (lane == 0) mbar_arrive(bar);
    };
    // the retired W group in accW -> bf16 columns [col, col + 128) of the staging rows; its position block is free.
    // The warp barrier in release() orders these stores after the quad's earlier reads of the same columns.
    auto stage_w = [&](int col) {
      fence_acc(accW);
      release(barPR0 + 8 * (pseq & 1));
      ++pseq;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int c = col + 8 * j + fc;
        *reinterpret_cast<uint32_t*>(wst + fr * kWLd + c) = pack_bf16x2(accW[4 * j], accW[4 * j + 1]);
        *reinterpret_cast<uint32_t*>(wst + (fr + 8) * kWLd + c) = pack_bf16x2(accW[4 * j + 2], accW[4 * j + 3]);
      }
      __syncwarp();
    };

    mbar_wait(barQ, 0);
#ifdef ESP_ATTN_FWD_PHASES
    long long ph_clk[kPhases] = {}, ph_t = clock64();
#endif
    for (int pass = 0; pass < 2; ++pass) {
      const bool pass2 = pass == 1;
      if constexpr (kPos) {
        // W of block 0 -> left half
        issue_w();
        wgmma_wait<0>();
        ESP_PHASE(kPhW);
        stage_w(0);
        ESP_PHASE(kPhStageW);
      }
      for (int jt = 0; jt < nkt; ++jt) {
        const int it = pass * nkt + jt, st = it & 1;
        if constexpr (kPos) {
          // ---- W_jt+1 -> right half ----
          issue_w();
          wgmma_wait<0>();
          ESP_PHASE(kPhW);
          if (pass2 && jt > 0) {
            fence_acc(o);
            release(barVR0 + 8 * ((jt - 1) & 1));
          }
          stage_w(kTile);
          ESP_PHASE(kPhStageW);
        }
        // ---- S = Qu K^T ----
        mbar_wait(barK0 + 8 * st, (it >> 1) & 1);
        const uint32_t sk = sb + kOffK + st * kTileBytes;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kHd / 16; ++k)
          wgmma_ss_n128<0, 0>(accS, make_sdesc(squ + k * 32, 16, 1024), make_sdesc(sk + k * 32, 16, 1024), k);
        wgmma_commit();
        wgmma_wait<0>();
        fence_acc(accS);
        release(barKR0 + 8 * st);  // the K stage is consumed: the loader may refill it
        ESP_PHASE(kPhS);
        // ---- logits s = S + W[r, 127 - r + c], masked beyond the utterance's keys (in place in accS) ----
        float tmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
          for (int x = 0; x < 2; ++x)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int r = fr + 8 * x, c = 8 * j + fc + e;
              const int key = jt * kTile + c;
              float a = accS[4 * j + 2 * x + e];
              if constexpr (kPos) a += bf2f(wst[r * kWLd + (kTile - 1) - r + c]);
              if (p.key_lo && (key < kmin[x] || key >= kmax[x])) {
                // hidden keys: the reference ADDS bf16(-1e4) to its bf16 scores (transformer_layer.py:189-192,
                // multihead_attention.py:835-839) -- finite, so a row whose visible keys are all padding still
                // normalises over the hidden ones
                a = __bfloat162float(__float2bfloat16_rn(a - 9984.f));
              }
              a = key < klen ? a : -INFINITY;  // key padding: -inf (:841-859)
              accS[4 * j + 2 * x + e] = a;
              tmax[x] = fmaxf(tmax[x], a);
            }
        ESP_PHASE(kPhLogits);
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
                for (int e = 0; e < 2; ++e) sum += exp2f(fmaf(accS[4 * j + 2 * x + e], kLog2e, -mb));  // exp2(-inf) = 0
            }
            sum += __shfl_xor_sync(0xffffffffu, sum, 1);
            sum += __shfl_xor_sync(0xffffffffu, sum, 2);
            if (m_new > -INFINITY) {
              l_run[x] = (m_run[x] > -INFINITY ? l_run[x] * exp2f((m_run[x] - m_new) * kLog2e) : 0.f) + sum;
              m_run[x] = m_new;
            }
            if (jt == nkt - 1) {
              inv_l[x] = l_run[x] > 0.f ? 1.f / l_run[x] : 0.f;
              // no visible key (lens[b] == 0): pass 2 then forms exp2(-inf) * 0 = 0, not exp2(-inf + inf) = NaN
              if (m_run[x] == -INFINITY) m_run[x] = 0.f;
            }
          }
          ESP_PHASE(kPhStats);
        } else {
          // ---- pass 2: normalised probabilities, dropout, register A operand of P V ----
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const int key = jt * kTile + 8 * j + fc;
            uint32_t hw[2] = {0u, 0u};  // 16-bit keep lanes of this thread's two keys, rows fr and fr + 8
            if (p.drop_p > 0.f) {
              // idx = prow * ld + key is even and prow * ld a multiple of 8: the lane pair's keys form one hash group
              const unsigned long long hsh = esp_hash_u64(seed, (hrow + key) >> 2);
              const uint32_t lo = (uint32_t)hsh, hi = (uint32_t)(hsh >> 32);
              const uint32_t own = (t & 1) ? hi : lo, other = __shfl_xor_sync(0xffffffffu, (t & 1) ? lo : hi, 1);
              hw[0] = (t & 1) ? other : own;
              hw[1] = (t & 1) ? own : other;
            }
#pragma unroll
            for (int x = 0; x < 2; ++x) {
              const float mb = m_run[x] * kLog2e;
              float pr[2], pd[2];
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const float pv = exp2f(fmaf(accS[4 * j + 2 * x + e], kLog2e, -mb)) * inv_l[x];
                pr[e] = bf2f(f2bf(pv));  // softmax in fp32, cast to the model dtype (fairseq/utils.py:514-525 + .type_as)
                pd[e] = pr[e];
              }
              if (p.drop_p > 0.f) {
#pragma unroll
                for (int e = 0; e < 2; ++e) pd[e] = ((hw[x] >> (16 * e)) & 0xFFFFu) >= p.thresh ? pd[e] * dscale : 0.f;
              }
              const uint32_t wpr = pack_bf16x2(pr[0], pr[1]), wpd = pack_bf16x2(pd[0], pd[1]);
              afrag[2 * j + x] = wpd;
              if (row_ok[x] && key < p.ld) {
                if (p.p_out) *reinterpret_cast<uint32_t*>(p.p_out + prow[x] * p.ld + key) = wpr;
                if (p.pd_out) *reinterpret_cast<uint32_t*>(p.pd_out + prow[x] * p.ld + key) = wpd;
              }
            }
          }
          ESP_PHASE(kPhProbs);
          mbar_wait(barV0 + 8 * (jt & 1), (jt >> 1) & 1);
          const uint32_t sv = sb + kOffV + (jt & 1) * kTileBytes;
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < kTile / 16; ++k) {
            // A fragment of keys 16k .. 16k+15: accumulator column groups 2k and 2k+1, rows fr and fr + 8
            const uint32_t a4[4] = {afrag[4 * k], afrag[4 * k + 1], afrag[4 * k + 2], afrag[4 * k + 3]};
            wgmma_rs_n64<1>(o, a4, make_sdesc(sv + k * 2048, kTileBytes, 1024), 1u);
          }
          wgmma_commit();
          if constexpr (!kPos) {
            // no W group to hide it behind: retire P V_jt here.  Keeping it in flight into the next tile's S group
            // (A fragments live) makes ptxas spill 52-56 bytes at 168 registers.
            wgmma_wait<0>();
            fence_acc(o);
            release(barVR0 + 8 * (jt & 1));
          }
          ESP_PHASE(kPhPV);
        }
        if (kPos && jt + 1 < nkt) {
          // ---- W_jt+1 moves to the left half: each lane of the quad moves 32 columns of the quad's two rows ----
          __syncwarp();
#pragma unroll
          for (int x = 0; x < 2; ++x) {
            uint4* row = reinterpret_cast<uint4*>(wst + (fr + 8 * x) * kWLd);
#pragma unroll
            for (int k = 0; k < 4; ++k) row[4 * (t & 3) + k] = row[16 + 4 * (t & 3) + k];
          }
        }
        ESP_PHASE(kPhMoveW);
      }
    }
    wgmma_wait<0>();
    fence_acc(o);
#ifdef ESP_ATTN_FWD_PHASES
    if (t == 0)
      for (int i = 0; i < kPhases; ++i) atomicAdd(&g_attn_fwd_phase_clk[i], (unsigned long long)ph_clk[i]);
#endif
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

#ifdef ESP_ATTN_FWD_PHASES
// SM clocks per phase summed since the last call (kPhW .. kPhMoveW), then reset
extern "C" int esp_attn_fwd_phase_clk(unsigned long long* out) {
  ESP_CUDA(cudaMemcpyFromSymbol(out, g_attn_fwd_phase_clk, sizeof(unsigned long long) * kPhases));
  static const unsigned long long zero[kPhases] = {};
  ESP_CUDA(cudaMemcpyToSymbol(g_attn_fwd_phase_clk, zero, sizeof(zero)));
  return 0;
}
#endif

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
  // pos == NULL selects plain scaled dot-product attention (no relative positions; qv is then not read)
  const bool has_pos = pos != nullptr;
  ESP_CHECK(qu && (qv || !has_pos) && k && v && ctx, "null pointer passed to esp_attn_fused_fwd");
  // the key tiles cover columns [0, 128 ceil(T/128)) of a probability row: a wider row would keep unwritten columns
  ESP_CHECK(p_out == nullptr || (ldp >= T && ldp % 8 == 0 && ldp <= (T + kTile - 1) / kTile * kTile),
            "probability row stride must be a multiple of 8 in [T, 128 ceil(T/128)] (T=%d, ldp=%d)", T, ldp);
  ESP_CHECK(drop_p <= 0.f || p_out == nullptr || pd_out != nullptr, "dropout with saved probabilities needs pd_out");
  ESP_CHECK(ldctx == (int64_t)H * kHd, "ctx must be [B*T, H*64] contiguous");
  ESP_CHECK(B <= 65535 && H <= 65535, "grid limits");
  CUtensorMap tqu, tqv, tk, tv, tp;
  int rc;
  if ((rc = esp_make_tmap_bf16(&tqu, qu, (long)H * kHd, T, ldq, B, (long)T * ldq, 1, 0, kTile))) return rc;
  if ((rc = esp_make_tmap_bf16(&tk, k, (long)H * kHd, T, ldkv, B, (long)T * ldkv, 1, 0, kTile))) return rc;
  if ((rc = esp_make_tmap_bf16(&tv, v, (long)H * kHd, T, ldkv, B, (long)T * ldkv, 1, 0, kTile))) return rc;
  if (has_pos) {
    if ((rc = esp_make_tmap_bf16(&tqv, qv, (long)H * kHd, T, ldq, B, (long)T * ldq, 1, 0, kTile))) return rc;
    const long pos_cols = pos_hstride ? (long)H * kHd : kHd;
    if ((rc = esp_make_tmap_bf16(&tp, pos, pos_cols, 2L * T - 1, ldpos, 1, 0, 1, 0, kTile))) return rc;
  } else {
    tqv = tp = tqu;  // unused by the instance without positions
    pos_hstride = 0;
  }  Params pr;
  pr.B = B; pr.T = T; pr.H = H; pr.d = (int)ldctx; pr.ld = ldp; pr.pos_hstride = pos_hstride;
  ESP_CHECK((key_lo == nullptr) == (key_hi == nullptr), "key_lo and key_hi must be given together");
  pr.key_lo = key_lo; pr.key_hi = key_hi;
  pr.lens = lens; pr.ctx = (bf16*)ctx; pr.p_out = (bf16*)p_out; pr.pd_out = drop_p > 0.f ? (bf16*)pd_out : nullptr;
  pr.drop_p = drop_p; pr.thresh = esp_dropout_thresh(drop_p); pr.seed = seed;
  pr.seed_ptr = (const unsigned long long*)seed_ptr;
  dim3 grid((T + kTile - 1) / kTile, H, B);
  if (has_pos) {
    ESP_SMEM_OPTIN(attn_fused_fwd_kernel<true>, kSmemBytes<true>);
    ESP_CUDA(esp_launch(attn_fused_fwd_kernel<true>, grid, kThreads, kSmemBytes<true>, st, tqu, tqv, tk, tv, tp, pr));
  } else {
    ESP_SMEM_OPTIN(attn_fused_fwd_kernel<false>, kSmemBytes<false>);
    ESP_CUDA(esp_launch(attn_fused_fwd_kernel<false>, grid, kThreads, kSmemBytes<false>, st, tqu, tqv, tk, tv, tp, pr));
  }
  return 0;
}
