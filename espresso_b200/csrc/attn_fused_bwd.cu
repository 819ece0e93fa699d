// espresso_b200 -- fused relative-position self-attention BACKWARD (score side) for sm_90a (H100).
//
// Backward of  ctx = dropout(softmax(qu k^T + skew(qv pos^T))) v   (fairseq/modules/multihead_attention.py:788-897) given
// dctx and the probabilities saved by esp_attn_fused_fwd.  One CTA per (128-key tile, head, utterance) walks the query
// tiles and keeps everything between the saved probabilities and the four results on chip:
//
//   dPd = dctx_i v_j^T                      wgmma, registers (each warpgroup 64 query rows x 128 keys)
//   dS  = P . (mask/keep . dPd - D_i)       same threads;  D_i = sum_e dctx[i,e] ctx[i,e]  (= sum_j P dP)
//   dV_j += Pd^T dctx_i ,  dK_j += dS^T qu_i   wgmma (each warpgroup 64 keys), accumulators stay in registers over the
//                                           whole query loop
//
// and writes dS [H,B,T,ld] once; for relative-position attention attn_skew_kernel then writes its skewed copy dBD[., i, (T-1)-i+j] (zeros elsewhere;
// inverse of the Transformer-XL shift, :824-830) for the three remaining GEMMs (dq_u = dS k, dq_v = dBD pos,
// dpos = dBD^T q_v).  Plain scaled dot-product attention (dbd == NULL) needs only dq = s dS k and skips that launch,
// and with it the skew kernel's 1024-frame row limit.  It replaces four launches of the unfused chain (the dPd GEMM, esp_attn_softmax_bwd, the dV and dK
// GEMMs) and the HBM round trips of dPd (write + read), P_drop and two reads of dS.
//
// Operand tiles are TMA boxes (SWIZZLE_128B) of 64 columns x 128 rows.  The probability tile [128 queries x 128 keys]
// (two 64-key chunks) is at the same time
//   * the MN-major A operand of an M = keys, K = queries product (dV, dK: the transposes are free), and
//   * the place where the dS threads overwrite P with dS (same rows, same 16-byte units).
#include "common.cuh"
#include "espresso_b200.h"
#include "sm90.cuh"
#include <cuda.h>
#include <stdlib.h>

namespace {

using namespace sm90;

constexpr int kTile = 128;
constexpr int kHd = 64;
constexpr int kThreads = 288;  // warps 0-7: two MMA / dS warpgroups, warp 8: TMA
constexpr int kTileBytes = kTile * kHd * 2;  // 16 KB: one 64-column x 128-row box
constexpr int kOffV = 0;
constexpr int kOffStage = kTileBytes;
constexpr int kStDO = 0, kStQu = kTileBytes, kStP = 2 * kTileBytes, kStX = 4 * kTileBytes;
constexpr int kStageBytes = 6 * kTileBytes;  // dctx_i, qu_i, P (2 chunks), P_drop (2 chunks)
constexpr int kOffBar = kOffStage + 2 * kStageBytes;
constexpr int kSmemBytes = kOffBar + 256 + 1024;

struct Params {
  int B, T, H, ld;
  const float* D;            // [H, B, T] row dots
  bf16* ds_out;              // [H, B, T, ld]
  bf16* dk_out;              // [B*T, ld_out] (head h at column h*64)
  bf16* dv_out;
  long ld_out;
  float drop_p;
  uint32_t thresh;
  unsigned long long seed;
  const unsigned long long* seed_ptr;
};

// D[h, b, t] = sum_e dctx[b*T+t, h*64+e] * ctx[b*T+t, h*64+e]: one warp per row of [B*T, H*64], 8 lanes per head
__global__ void __launch_bounds__(256)
attn_rowdot_kernel(const bf16* __restrict__ a, const bf16* __restrict__ c, long R, int T, int H, long ld,
                   float* __restrict__ D) {
  esp_pdl();
  const int lane = threadIdx.x & 31;
  const long row = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= R) return;
  const int b = (int)(row / T), t = (int)(row % T), B = (int)(R / T);
  for (int h0 = 0; h0 < H; h0 += 4) {  // 32 lanes x 8 elements = 4 heads per trip
    const int h = h0 + (lane >> 3);
    float s = 0.f;
    if (h < H) {
      const uint4 qa = *reinterpret_cast<const uint4*>(a + row * ld + h0 * kHd + lane * 8);
      const uint4 qc = *reinterpret_cast<const uint4*>(c + row * ld + h0 * kHd + lane * 8);
      float x0, x1, y0, y1;
      unpack_bf16x2(qa.x, x0, x1); unpack_bf16x2(qc.x, y0, y1); s += x0 * y0 + x1 * y1;
      unpack_bf16x2(qa.y, x0, x1); unpack_bf16x2(qc.y, y0, y1); s += x0 * y0 + x1 * y1;
      unpack_bf16x2(qa.z, x0, x1); unpack_bf16x2(qc.z, y0, y1); s += x0 * y0 + x1 * y1;
      unpack_bf16x2(qa.w, x0, x1); unpack_bf16x2(qc.w, y0, y1); s += x0 * y0 + x1 * y1;
    }
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    s += __shfl_xor_sync(0xffffffffu, s, 4);
    if ((lane & 7) == 0 && h < H) D[((long)h * B + b) * T + t] = s;
  }
}

// dBD[row, (T-1) - i + j] = dS[row, j], zeros elsewhere (inverse of the Transformer-XL shift, :824-830): one warp per row
// (h, b, i).  The row is staged in shared memory with 16-byte loads; every destination-aligned group of 8 columns is then the
// tail of one source unit and the head of the next (the split point eo = ((T-1)-i) mod 8 is the same for the whole row), so a
// lane builds a group from two 16-byte shared-memory loads and a funnel shift and writes it with one aligned 16-byte store.
// Plenty of resident warps hide the latencies -- which the fused kernel above, with its eight dS warps per SM, cannot.
constexpr int kSkewWarps = 8;
constexpr int kSkewMaxUnits = 130;  // T <= 1024: 128 source units + one zero unit on either side
__global__ void __launch_bounds__(kSkewWarps * 32)
attn_skew_kernel(const bf16* __restrict__ ds, bf16* __restrict__ dbd, long rows, int T, int ld, int ldp) {
  esp_pdl();
  __shared__ uint4 stage[kSkewWarps][kSkewMaxUnits];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const long row = (long)blockIdx.x * kSkewWarps + w;
  if (row >= rows) return;
  const int i = (int)(row % T);
  const int nu = (T + 7) >> 3;  // source units that hold keys (ld >= 8 nu; columns T..8nu-1 of dS are zero)
  uint4* st = stage[w];
  const uint4* src = reinterpret_cast<const uint4*>(ds + row * (long)ld);
  // staged units: index 0 = zeros, 1..nu = the row, nu+1 = zeros
  for (int u = lane; u < nu + 2; u += 32) st[u] = (u >= 1 && u <= nu) ? src[u - 1] : make_uint4(0, 0, 0, 0);
  __syncwarp();
  const int cs = (T - 1) - i;      // destination column of key 0
  const int a = cs & ~7, eo = cs & 7;
  const int ga = a >> 3;           // destination group that holds key 0
  uint4* dst = reinterpret_cast<uint4*>(dbd + row * (long)ldp);
  const int ngroups = ldp >> 3;
  for (int gd = lane; gd < ngroups; gd += 32) {
    const int g = gd - ga;  // group index inside the window: source units g - 1 (tail) and g (head)
    uint4 o = make_uint4(0, 0, 0, 0);
    if (g >= 0 && g <= nu) {
      const uint4 u0 = st[g], u1 = st[g + 1];  // staged index = unit + 1
      const uint32_t x[8] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z, u1.w};
      switch (8 - eo) {  // first element of the group inside the 16-element pair (warp-uniform)
        case 8: o = u1; break;
        case 7: o = make_uint4(__funnelshift_r(x[3], x[4], 16), __funnelshift_r(x[4], x[5], 16), __funnelshift_r(x[5], x[6], 16), __funnelshift_r(x[6], x[7], 16)); break;
        case 6: o = make_uint4(x[3], x[4], x[5], x[6]); break;
        case 5: o = make_uint4(__funnelshift_r(x[2], x[3], 16), __funnelshift_r(x[3], x[4], 16), __funnelshift_r(x[4], x[5], 16), __funnelshift_r(x[5], x[6], 16)); break;
        case 4: o = make_uint4(x[2], x[3], x[4], x[5]); break;
        case 3: o = make_uint4(__funnelshift_r(x[1], x[2], 16), __funnelshift_r(x[2], x[3], 16), __funnelshift_r(x[3], x[4], 16), __funnelshift_r(x[4], x[5], 16)); break;
        case 2: o = make_uint4(x[1], x[2], x[3], x[4]); break;
        default: o = make_uint4(__funnelshift_r(x[0], x[1], 16), __funnelshift_r(x[1], x[2], 16), __funnelshift_r(x[2], x[3], 16), __funnelshift_r(x[3], x[4], 16)); break;
      }
    }
    dst[gd] = o;
  }
}

__global__ void __launch_bounds__(kThreads, 1)
attn_fused_bwd_kernel(const __grid_constant__ CUtensorMap tmDO, const __grid_constant__ CUtensorMap tmQu,
                      const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmP,
                      const __grid_constant__ CUtensorMap tmPd, const Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const uint32_t sb = smem_u32(smem);
  const uint32_t bar0 = sb + kOffBar;
  // mbarriers: V | stage loaded x2 | stage consumed by the MMAs x2
  const uint32_t barV = bar0, barL = bar0 + 8, barFree = bar0 + 24;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int jt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int T = p.T;
  const int j0 = jt * kTile;
  const int nqt = (T + kTile - 1) / kTile;  // query tiles

  esp_pdl_trigger();
  if (threadIdx.x == 256) {
    mbar_init(barV, 1);
    for (int s = 0; s < 2; ++s) {
      mbar_init(barL + 8 * s, 1);
      mbar_init(barFree + 8 * s, 8);  // one arrive per MMA warp
    }
    fence_mbar_init();
    prefetch_tmap(&tmDO);
    prefetch_tmap(&tmP);
    prefetch_tmap(&tmPd);
  }
  __syncthreads();
  esp_pdl_wait();

  if (warp == 8) {
    // ============================== TMA loads (one thread) ======================================================
    if (lane == 0) {
      auto load_stage = [&](int i) {
        const int s = i & 1;
        const uint32_t bar = barL + 8 * s, st = sb + kOffStage + s * kStageBytes;
        mbar_expect_tx(bar, (uint32_t)kStageBytes);
        tma_load_4d(st + kStDO, &tmDO, bar, h * kHd, i * kTile, b, 0);
        tma_load_4d(st + kStQu, &tmQu, bar, h * kHd, i * kTile, b, 0);
        tma_load_4d(st + kStP, &tmP, bar, j0, i * kTile, b, h);
        tma_load_4d(st + kStP + kTileBytes, &tmP, bar, j0 + 64, i * kTile, b, h);
        tma_load_4d(st + kStX, &tmPd, bar, j0, i * kTile, b, h);
        tma_load_4d(st + kStX + kTileBytes, &tmPd, bar, j0 + 64, i * kTile, b, h);
      };
      mbar_expect_tx(barV, kTileBytes);
      tma_load_4d(sb + kOffV, &tmV, barV, h * kHd, j0, b, 0);
      load_stage(0);
      if (nqt > 1) load_stage(1);
      for (int i = 0; i + 2 < nqt; ++i) {
        mbar_wait(barFree + 8 * (i & 1), (i >> 1) & 1);  // query tile i is done with its stage
        load_stage(i + 2);
      }
    }
  } else {
    // ============================== MMA + dS warpgroups ==========================================================
    const int wg = warp >> 2;
    const int t = threadIdx.x & 127;
    // accumulator fragment: rows fr, fr + 8 of the warpgroup's 64 (query rows for dPd, key rows for dV / dK);
    // columns 8 j + fc, + 1
    const int fr = (t >> 5) * 16 + ((t & 31) >> 2), fc = 2 * (t & 3);
    const unsigned long long seed = p.seed + (p.seed_ptr ? *p.seed_ptr : 0ull);
    const float dscale = p.drop_p > 0.f ? 65536.f / (65536.f - (float)p.thresh) : 1.f;
    const long hb = (long)h * p.B + b;
    float dv[32], dk[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) dv[i] = dk[i] = 0.f;
    mbar_wait(barV, 0);

    for (int i = 0; i < nqt; ++i) {
      const int s = i & 1;
      const uint32_t st = sb + kOffStage + s * kStageBytes;
      uint8_t* const stg = smem + kOffStage + s * kStageBytes;
      mbar_wait(barL + 8 * s, (i >> 1) & 1);
      // ---- dPd = dctx_i v_j^T for this warpgroup's 64 query rows ----
      float acc[64];
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kHd / 16; ++k)
        wgmma_ss_n128<0, 0>(acc, make_sdesc(st + kStDO + wg * (64 * 128) + k * 32, 16, 1024),
                            make_sdesc(sb + kOffV + k * 32, 16, 1024), k);
      wgmma_commit();
      wgmma_wait<0>();
      fence_acc(acc);
      // ---- dS = P (keep . dPd . scale - D), written over P in the operand tile and to ds_out ----
#pragma unroll
      for (int x = 0; x < 2; ++x) {
        const int r = wg * 64 + fr + 8 * x;  // query row inside the tile
        const int qi = i * kTile + r;
        const bool row_ok = qi < T;
        const long prow = hb * T + qi;
        const float Dv = row_ok ? p.D[prow] : 0.f;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int c = 8 * j + fc;  // key inside the tile
          uint32_t* pp = reinterpret_cast<uint32_t*>(stg + kStP + (c >> 6) * kTileBytes + r * 128 +
                                                     (((((c & 63) >> 3) ^ (r & 7))) << 4) + (c & 7) * 2);
          float p0, p1;
          unpack_bf16x2(*pp, p0, p1);
          float d0 = acc[4 * j + 2 * x], d1 = acc[4 * j + 2 * x + 1];
          const int key = j0 + c;
          if (p.drop_p > 0.f) {
            // the index is even and prow * ld a multiple of 8: both elements are lanes of the same 4-element hash group
            const unsigned long long idx = (unsigned long long)prow * p.ld + key;
            const unsigned long long hsh = esp_hash_u64(seed, idx >> 2);
            d0 = ((uint32_t)(hsh >> (16 * (idx & 3))) & 0xFFFFu) >= p.thresh ? d0 * dscale : 0.f;
            d1 = ((uint32_t)(hsh >> (16 * ((idx & 3) + 1))) & 0xFFFFu) >= p.thresh ? d1 * dscale : 0.f;
          }
          const uint32_t w = pack_bf16x2(p0 * (d0 - Dv), p1 * (d1 - Dv));
          *pp = w;
          if (row_ok && key < p.ld) *reinterpret_cast<uint32_t*>(p.ds_out + prow * p.ld + key) = w;
        }
      }
      // every dS of the tile is in shared memory (both warpgroups) and visible to the tensor cores
      fence_proxy_async_smem();
      named_sync(1, 256);
      // ---- dV_j += Pd^T dctx_i ; dK_j += dS^T qu_i : M = this warpgroup's 64 keys, K = the tile's 128 queries ----
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kTile / 16; ++k)
        wgmma_ss_n64<1, 1>(dv, make_sdesc(st + kStX + wg * kTileBytes + k * 2048, kTileBytes, 1024),
                           make_sdesc(st + kStDO + k * 2048, kTileBytes, 1024), 1u);
#pragma unroll
      for (int k = 0; k < kTile / 16; ++k)
        wgmma_ss_n64<1, 1>(dk, make_sdesc(st + kStP + wg * kTileBytes + k * 2048, kTileBytes, 1024),
                           make_sdesc(st + kStQu + k * 2048, kTileBytes, 1024), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      fence_acc(dv);
      fence_acc(dk);
      __syncwarp();
      if (lane == 0) mbar_arrive(barFree + 8 * s);
    }
    // ---- epilogue: dV_j, dK_j -> bf16 rows of the fused dqkv buffer ----
#pragma unroll
    for (int x = 0; x < 2; ++x) {
      const int kj = j0 + wg * 64 + fr + 8 * x;
      if (kj >= T) continue;
      bf16* dvp = p.dv_out + ((long)b * T + kj) * p.ld_out + h * kHd + fc;
      bf16* dkp = p.dk_out + ((long)b * T + kj) * p.ld_out + h * kHd + fc;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        *reinterpret_cast<uint32_t*>(dvp + 8 * j) = pack_bf16x2(dv[4 * j + 2 * x], dv[4 * j + 2 * x + 1]);
        *reinterpret_cast<uint32_t*>(dkp + 8 * j) = pack_bf16x2(dk[4 * j + 2 * x], dk[4 * j + 2 * x + 1]);
      }
    }
  }
}

}  // namespace

int esp_make_tmap_bf16(CUtensorMap* tm, const void* base, long inner, long rows, long ld, int nb1, long s1, int nb2,
                       long s2, int box_rows);  // gemm_tcgen05.cu

extern "C" int esp_attn_fused_bwd(const void* dctx, const void* ctx, int64_t ldctx, const void* qu, int64_t ldq, const void* v,
                                  int64_t ldkv, const void* p, const void* pd, int32_t ldp_probs, int32_t B, int32_t T,
                                  int32_t H, int32_t head_dim, float drop_p, uint64_t seed, const uint64_t* seed_ptr,
                                  float* rowdot_ws, void* ds, void* dbd, int32_t ldbd, void* dk, void* dv, int64_t ld_out,
                                  void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(head_dim == kHd, "fused attention backward is built for head_dim 64 (got %d)", head_dim);
  ESP_CHECK(B >= 0 && T >= 0 && H > 0, "bad attention shape");
  if (B == 0 || T == 0) return 0;
  ESP_CHECK(dctx && ctx && qu && v && p && pd && rowdot_ws && ds && dk && dv, "null pointer passed to esp_attn_fused_bwd");
  ESP_CHECK(ldp_probs >= T && ldp_probs % 8 == 0 && ldp_probs <= (T + kTile - 1) / kTile * kTile,
            "probability row stride must be a multiple of 8 in [T, 128 ceil(T/128)] (T=%d, ldp=%d)", T, ldp_probs);
  ESP_CHECK(dbd == nullptr || (ldbd >= 2 * T - 1 && ldbd % 8 == 0), "dBD row stride must be a multiple of 8 and >= 2T-1");
  ESP_CHECK(ldctx % 8 == 0 && ldq % 8 == 0 && ldkv % 8 == 0 && ld_out % 8 == 0, "row strides must be multiples of 8");
  ESP_CHECK(((uintptr_t)dk & 15) == 0 && ((uintptr_t)dv & 15) == 0, "dk / dv must be 16-byte aligned");
  ESP_CHECK(B <= 65535 && H <= 65535, "grid limits");
  ESP_CHECK(dbd == nullptr || T <= 8 * (kSkewMaxUnits - 2), "relative-position attention backward: at most %d frames",
            8 * (kSkewMaxUnits - 2));
  const long R = (long)B * T;
  ESP_CUDA(esp_launch(attn_rowdot_kernel, (unsigned)((R + 7) / 8), 256, 0, st, (const bf16*)dctx, (const bf16*)ctx, R, T, H,
                      (long)ldctx, rowdot_ws));
  CUtensorMap tdo, tqu, tv, tp, tpd;
  int rc;
  if ((rc = esp_make_tmap_bf16(&tdo, dctx, (long)H * kHd, T, ldctx, B, (long)T * ldctx, 1, 0, kTile))) return rc;
  if ((rc = esp_make_tmap_bf16(&tqu, qu, (long)H * kHd, T, ldq, B, (long)T * ldq, 1, 0, kTile))) return rc;
  if ((rc = esp_make_tmap_bf16(&tv, v, (long)H * kHd, T, ldkv, B, (long)T * ldkv, 1, 0, kTile))) return rc;
  if ((rc = esp_make_tmap_bf16(&tp, p, ldp_probs, T, ldp_probs, B, (long)T * ldp_probs, H, (long)B * T * ldp_probs, kTile))) return rc;
  if ((rc = esp_make_tmap_bf16(&tpd, pd, ldp_probs, T, ldp_probs, B, (long)T * ldp_probs, H, (long)B * T * ldp_probs, kTile))) return rc;
  Params pr;
  pr.B = B; pr.T = T; pr.H = H; pr.ld = ldp_probs;
  pr.D = rowdot_ws; pr.ds_out = (bf16*)ds; pr.dk_out = (bf16*)dk; pr.dv_out = (bf16*)dv;
  pr.ld_out = ld_out;
  pr.drop_p = drop_p; pr.thresh = esp_dropout_thresh(drop_p); pr.seed = seed;
  pr.seed_ptr = (const unsigned long long*)seed_ptr;
  ESP_SMEM_OPTIN(attn_fused_bwd_kernel, kSmemBytes);
  dim3 grid((T + kTile - 1) / kTile, H, B);
  ESP_CUDA(esp_launch(attn_fused_bwd_kernel, grid, kThreads, kSmemBytes, st, tdo, tqu, tv, tp, tpd, pr));
  if (dbd == nullptr) return 0;
  const long rows = (long)H * B * T;
  ESP_CUDA(esp_launch(attn_skew_kernel, (unsigned)((rows + kSkewWarps - 1) / kSkewWarps), kSkewWarps * 32, 0, st, (const bf16*)ds,
                      (bf16*)dbd, rows, T, (int)ldp_probs, (int)ldbd));
  return 0;
}
