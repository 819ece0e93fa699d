// espresso_b200 -- persistent warp-specialised bf16 GEMM for sm_90a (H100).
//
//   C[b][M,N] = epilogue( op(A[b])[M,K] * op(B[b])[N,K]^T )        fp32 accumulate in registers
//
// * operands staged by TMA (cp.async.bulk.tensor, SWIZZLE_128B) into a multi-stage smem ring,
// * two consumer warpgroups, each issuing wgmma.mma_async (m64 x BN x k16) for its 64 rows of the 128-row tile,
// * the epilogue stages the accumulator through shared memory so that every thread owns 16 consecutive columns of one
//   row at a time, and fuses bias / activation (+grad) / dropout / scaled residual / relative-position skew, writing
//   bf16 or fp32 straight to HBM.  Two more warpgroups run it, one per 64-row half of the tile (two threads per row),
//   while the consumers already run the next tile's MMAs.
//
// This one kernel replaces every dense contraction on the Espresso hot path:
//   Linear layers                fairseq/modules/conformer_layer.py:134-146 (FFN), :79-101 (pw convs)
//   q/k/v/out/pos projections    fairseq/modules/multihead_attention.py:650-653,799-814,899-907
//   QK^T, (q+v)P^T, PV           fairseq/modules/multihead_attention.py:788,815-823,897
//   fc0 / fc_out                 espresso/models/transformer/speech_transformer_encoder.py:341-343,
//                                .../speech_transformer_encoder_model.py:207-208
// and their dgrad / wgrad counterparts (operand majors are template flags: K-major or MN-major
// smem descriptors, so no transposes are ever materialised).
#include "common.cuh"
#include "espresso_b200.h"
#include "sm90.cuh"
#include <cuda.h>

namespace {

using namespace sm90;

constexpr int BM = 128;
constexpr int BK = 64;  // 64 bf16 = 128 bytes = one SWIZZLE_128B row
// columns per step of the fused epilogue: at 16, every role fits the 96 registers a 640-thread launch leaves it (at 32
// the epilogue spills its loop state, and giving it more registers through setmaxnreg made the training step slower)
constexpr int kEpiW = 16;
// Warpgroup 0: warp 0 TMA, warps 2-3 bias-gradient row sums; warpgroups 1-2: MMA; warpgroups 3-4: epilogue.  640 threads
// leave every role 96 registers (65 536 / 640, rounded down to a multiple of 8): enough for the 64-register accumulator
// of a 128-wide tile and the mainloop around it, and for the epilogue's 16-column steps.
constexpr int kThreads = 640;

struct EpiParams {
  void* C;
  bf16* C2;
  const bf16* bias;
  const bf16* aux;
  const void* R;
  long ldc, ld_aux, ldr;
  long sC1, sC2, sAux1, sAux2, sR1, sR2;
  int c_f32, r_f32, act, drop_mode, skew_r, atomic;
  float alpha, beta, drop_scale;
  uint32_t drop_thresh;
  unsigned long long seed;
  const unsigned long long* seed_ptr;
};

// 3x3 convolutions of the conv front end as implicit GEMMs on this kernel (espresso/modules/speech_convolutions.py:78-102).
// Activations are channels-last [B, T, F, C]; a tile of im2col rows is a (bt x bf) box of output positions, and the A
// tile of one filter tap is that box of the INPUT shifted by the tap (and strided by the convolution stride through the
// tensor map's element strides) -- one TMA box load, zero padding = TMA out-of-bounds fill.  Nothing is materialised.
//   mode 1 (fprop / dgrad): A = implicit im2col (K-major), K block kb = (tap, 64-channel block); output rows are
//           scattered back to positions (strided for the parity classes of a stride-2 dgrad);
//   mode 2 (wgrad): the reduction runs over POSITIONS (K block = one 64-position box); A = dY^T, B = the shifted input
//           box of the tap that owns the N chunk, both MN-major; the epilogue is the ordinary fp32 accumulate.
struct ConvGeom {
  int mode;
  int bf_log2, bt;        // box of positions: bf = 1 << bf_log2 along F, bt along T  (bt * bf = 128 in mode 1, 64 in mode 2)
  int tiles_t, tiles_f;   // boxes per utterance
  int st, sf;             // box start in the tensor behind the shifted loads = box index * (bt * st, bf * sf) + offset[tap]
  int cblocks;            // mode 1: 64-channel K blocks per tap
  int cin;                // mode 2: channels per tap along N
  int OT, OF, ost, osf, opt, opf;  // mode 1 output mapping: (t, f) -> (t * ost + opt, f * osf + opf), valid below (OT, OF)
  signed char offt[9], offf[9], btap[9];  // per tap: offsets of the shifted box; tap coordinate in the (ci, tap, co) weight view
};

struct KParams {
  int M, N, K, nb1, nb2, ksplit;
  ConvGeom cv;
  float* rowsum_a;     // optional: rowsum_a[m] += rowsum_scale * sum_k A[m, k] (bias gradient of a weight-gradient GEMM)
  float rowsum_scale;
  int a_b1, a_b2, b_b1, b_b2;  // 0 => operand is broadcast along that batch dim
  EpiParams ep;
};

// Profiling build only (-DESP_GEMM_PHASES, made by profiles/gemm_phases.py): thread 0 of each MMA and epilogue warpgroup
// adds the SM clocks of its role's phases to g_gemm_phase_clk (kPhEpiTiles counts the tiles, or tile halves, served).
enum { kPhMmaAccWait, kPhMmaLoop, kPhEpiBusy, kPhEpiLoop, kPhEpiTiles, kPhases };
#ifdef ESP_GEMM_PHASES
__device__ unsigned long long g_gemm_phase_clk[kPhases];
struct PhaseClk {
  long long c[kPhases] = {};
  __device__ __forceinline__ long long now() const { return clock64(); }
  __device__ __forceinline__ void add(int i, long long v) { c[i] += v; }
  __device__ __forceinline__ void flush(bool leader) const {
    if (leader)
      for (int i = 0; i < kPhases; ++i) atomicAdd(&g_gemm_phase_clk[i], (unsigned long long)c[i]);
  }
};
#else
struct PhaseClk {
  __device__ __forceinline__ long long now() const { return 0; }
  __device__ __forceinline__ void add(int, long long) {}
  __device__ __forceinline__ void flush(bool) const {}
};
#endif

// sigmoid through the single-MUFU tanh approximation (|err| ~ 5e-4: below bf16 output resolution)
__device__ __forceinline__ float fast_sigmoid(float x) {
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.5f * x));
  return fmaf(0.5f, t, 0.5f);
}
__device__ __forceinline__ void load8f(const bf16* p, float* v) {
  const uint4 q = __ldg(reinterpret_cast<const uint4*>(p));
  unpack_bf16x2(q.x, v[0], v[1]);
  unpack_bf16x2(q.y, v[2], v[3]);
  unpack_bf16x2(q.z, v[4], v[5]);
  unpack_bf16x2(q.w, v[6], v[7]);
}
// W consecutive bf16 (vectorised when 16-byte aligned and fully in range)
template <int W>
__device__ __forceinline__ void load_bf16(const bf16* p, int valid, float* v) {
  if (valid >= W && ((reinterpret_cast<uintptr_t>(p) & 15) == 0)) {
#pragma unroll
    for (int j = 0; j < W; j += 8) load8f(p + j, v + j);
  } else {
#pragma unroll
    for (int j = 0; j < W; ++j) v[j] = j < valid ? bf2f(p[j]) : 0.f;
  }
}
// A row-per-thread epilogue writes each 32-byte L2 sector with two back-to-back 16-byte stores of the same thread.
template <int W>
__device__ __forceinline__ void store_bf16(bf16* p, int valid, const float* v) {
  if (valid >= W && ((reinterpret_cast<uintptr_t>(p) & 15) == 0)) {
#pragma unroll
    for (int j = 0; j < W; j += 8) {
      uint4 o;
      o.x = pack_bf16x2(v[j], v[j + 1]);
      o.y = pack_bf16x2(v[j + 2], v[j + 3]);
      o.z = pack_bf16x2(v[j + 4], v[j + 5]);
      o.w = pack_bf16x2(v[j + 6], v[j + 7]);
      *reinterpret_cast<uint4*>(p + j) = o;
    }
  } else {
    for (int j = 0; j < W; ++j)
      if (j < valid) p[j] = f2bf(v[j]);
  }
}
// dropout over W consecutive logical indices starting at idx0: one hash per 4 elements when aligned
template <int W>
__device__ __forceinline__ void dropout_chunk(float* v, unsigned long long seed, unsigned long long idx0, uint32_t thresh,
                                              float scale) {
  if ((idx0 & 3ull) == 0) {
#pragma unroll
    for (int g4 = 0; g4 < W / 4; ++g4) {
      const unsigned long long h = esp_hash_u64(seed, (idx0 >> 2) + g4);
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const uint32_t lane16 = (uint32_t)(h >> (16 * t)) & 0xFFFFu;
        v[g4 * 4 + t] = lane16 >= thresh ? v[g4 * 4 + t] * scale : 0.f;
      }
    }
  } else {
#pragma unroll
    for (int j = 0; j < W; ++j) v[j] = esp_dropout_keep(seed, idx0 + j, thresh) ? v[j] * scale : 0.f;
  }
}

// The fused epilogue of W consecutive accumulator columns n0 .. n0+W-1 of output row m (v: the accumulator values).
template <int W>
__device__ __forceinline__ void epilogue_chunk(const KParams& p, const EpiParams& e, float* v, int m, int n0, long c_off,
                                               long aux_off, long r_off, unsigned long long rng_row,
                                               unsigned long long seed) {
  const int valid = p.N - n0;  // >= 1; >= W for a full chunk
  if (e.atomic) {
    // split-K / gradient accumulation: C (fp32) += alpha * acc, vector reductions at L2
    float* cp = (float*)e.C + c_off + n0;
    if (valid >= W && ((reinterpret_cast<uintptr_t>(cp) & 15) == 0)) {
#pragma unroll
      for (int j = 0; j < W; j += 4)
        red_add_v4(cp + j, v[j] * e.alpha, v[j + 1] * e.alpha, v[j + 2] * e.alpha, v[j + 3] * e.alpha);
    } else {
      for (int j = 0; j < W; ++j)
        if (j < valid) atomicAdd(cp + j, v[j] * e.alpha);
    }
    return;
  }
  if (e.bias) {
    float bv[W];
    load_bf16<W>(e.bias + n0, valid, bv);
#pragma unroll
    for (int j = 0; j < W; ++j) v[j] += bv[j];
  }
  if (e.C2) store_bf16<W>(e.C2 + c_off + n0, valid, v);
  if (e.drop_mode == 2) dropout_chunk<W>(v, seed, rng_row + n0, e.drop_thresh, e.drop_scale);
  if (e.act == ESP_ACT_SILU) {
#pragma unroll
    for (int j = 0; j < W; ++j) v[j] *= fast_sigmoid(v[j]);
  } else if (e.act == ESP_ACT_RELU) {
#pragma unroll
    for (int j = 0; j < W; ++j) v[j] = fmaxf(v[j], 0.f);
  } else if (e.act == ESP_ACT_SILU_BWD) {
    float u[W];
    load_bf16<W>(e.aux + aux_off + n0, valid, u);
#pragma unroll
    for (int j = 0; j < W; ++j) {
      const float sg = fast_sigmoid(u[j]);
      v[j] *= sg * fmaf(u[j], 1.f - sg, 1.f);
    }
  } else if (e.act == ESP_ACT_RELU_BWD) {
    float u[W];
    load_bf16<W>(e.aux + aux_off + n0, valid, u);
#pragma unroll
    for (int j = 0; j < W; ++j) v[j] = u[j] > 0.f ? v[j] : 0.f;
  }
  if (e.drop_mode == 1) dropout_chunk<W>(v, seed, rng_row + n0, e.drop_thresh, e.drop_scale);
  if (e.alpha != 1.f) {
#pragma unroll
    for (int j = 0; j < W; ++j) v[j] *= e.alpha;
  }
  if (e.R) {
    if (e.skew_r) {
      // Transformer-XL skew fused into the score GEMM: R is BD_full[row m, (skew_r-1)-m+n]
      // (fairseq/modules/multihead_attention.py:824-830 as_strided trick).  W consecutive but arbitrarily aligned
      // bf16 -> W / 2 + 1 aligned words, re-aligned with a funnel shift when the first element sits in the upper half of its word.
      const bf16* rr = (const bf16*)e.R + r_off + (e.skew_r - 1 - m) + n0;
      if (valid >= W) {
        const bool odd = (reinterpret_cast<uintptr_t>(rr) & 2) != 0;
        const uint32_t* wp = reinterpret_cast<const uint32_t*>(rr - (odd ? 1 : 0));
        uint32_t sk[W / 2 + 1];
#pragma unroll
        for (int j = 0; j < W / 2 + 1; ++j) sk[j] = __ldg(wp + j);
#pragma unroll
        for (int j = 0; j < W / 2; ++j) {
          const uint32_t w = odd ? __funnelshift_r(sk[j], sk[j + 1], 16) : sk[j];
          float lo, hi;
          unpack_bf16x2(w, lo, hi);
          v[2 * j] += e.beta * lo;
          v[2 * j + 1] += e.beta * hi;
        }
      } else {
#pragma unroll
        for (int j = 0; j < W; ++j)
          if (j < valid) v[j] += e.beta * bf2f(rr[j]);
      }
    } else if (e.r_f32) {
      const float* rr = (const float*)e.R + r_off + n0;
#pragma unroll
      for (int j = 0; j < W; ++j)
        if (j < valid) v[j] += e.beta * rr[j];
    } else {
      float rv[W];
      load_bf16<W>((const bf16*)e.R + r_off + n0, valid, rv);
#pragma unroll
      for (int j = 0; j < W; ++j) v[j] = fmaf(e.beta, rv[j], v[j]);
    }
  }
  if (e.c_f32) {
    float* cp = (float*)e.C + c_off + n0;
    if (valid >= W && ((reinterpret_cast<uintptr_t>(cp) & 15) == 0)) {
#pragma unroll
      for (int j = 0; j < W; j += 4) *reinterpret_cast<float4*>(cp + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
    } else {
      for (int j = 0; j < W; ++j)
        if (j < valid) cp[j] = v[j];
    }
  } else {
    store_bf16<W>((bf16*)e.C + c_off + n0, valid, v);
  }
}

// The fused epilogue of one column half (BN / 2 columns) of row ml (0..127) of tile (mt, nt, batch bt): src is the
// half's staged fp32 accumulator, chunk c at src + kEpiW c, holding output columns n_base + kEpiW c ...
template <int BN, int MC>
__device__ __forceinline__ void epilogue_row(const KParams& p, const EpiParams& e, unsigned long long seed,
                                             const float* src, int ml, int mt, int bt, int n_base) {
  const int b1 = bt % p.nb1, b2 = bt / p.nb1;
  const int m = mt * BM + ml;
  bool row_ok = m < p.M;
  long c_off = (long)b1 * e.sC1 + (long)b2 * e.sC2 + (long)m * e.ldc;
  if (MC == 1 && p.cv.mode == 1) {
    // row of an im2col tile -> its output position (channels-last activation; strided for dgrad parity classes)
    const ConvGeom& g = p.cv;
    const int tf = mt % g.tiles_f, tt = (mt / g.tiles_f) % g.tiles_t, cb = mt / (g.tiles_f * g.tiles_t);
    const int ot = (tt * g.bt + (ml >> g.bf_log2)) * g.ost + g.opt;
    const int of = ((tf << g.bf_log2) + (ml & ((1 << g.bf_log2) - 1))) * g.osf + g.opf;
    row_ok = ot < g.OT && of < g.OF;
    c_off = (((long)cb * g.OT + ot) * g.OF + of) * e.ldc;
  }
  if (!row_ok) return;
  const long aux_off = (long)b1 * e.sAux1 + (long)b2 * e.sAux2 + (long)m * e.ld_aux;
  const long r_off = (long)b1 * e.sR1 + (long)b2 * e.sR2 + (long)m * e.ldr;
  const unsigned long long rng_row = ((unsigned long long)bt * p.M + m) * (unsigned long long)p.N;
#pragma unroll 1
  for (int c = 0; c < BN / 2 / kEpiW; ++c) {
    const int n0 = n_base + c * kEpiW;
    if (n0 >= p.N) break;
    float v[kEpiW];
#pragma unroll
    for (int j = 0; j < kEpiW; j += 4) {
      const float4 q = *reinterpret_cast<const float4*>(src + c * kEpiW + j);
      v[j] = q.x; v[j + 1] = q.y; v[j + 2] = q.z; v[j + 3] = q.w;
    }
    epilogue_chunk<kEpiW>(p, e, v, m, n0, c_off, aux_off, r_off, rng_row, seed);
  }
}

template <int BN>
struct SmemLayout {
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = BN == 128 ? 4 : 6;
  // accumulator staging of the epilogue: the whole 128 x BN fp32 tile (the 64 rows of each consumer warpgroup one after
  // the other), rows padded by 4 floats so that 16-byte reads of 8 consecutive rows at one column hit distinct banks
  static constexpr int kEpiLd = BN + 4;
  static constexpr int kEpiOffset = kStages * kStageBytes;
  static constexpr int kBarOffset = kEpiOffset + 2 * 64 * kEpiLd * 4;
  static constexpr int kTotal = kBarOffset + 256 + 1024;  // + alignment slack
};

template <int BN, int TA, int TB>
__device__ __forceinline__ void mma_k16(float (&d)[BN / 2], uint64_t da, uint64_t db, uint32_t accumulate) {
  if constexpr (BN == 64) wgmma_ss_n64<TA, TB>(d, da, db, accumulate);
  else wgmma_ss_n128<TA, TB>(d, da, db, accumulate);
}

// MC = 2: the kernel runs as 2-CTA clusters along M.  The two CTAs of a cluster work on M-adjacent tiles of the same
// (N tile, batch, K split), so they need the SAME B tile: each loads half of it and multicasts it to both, which cuts
// the L2->SM operand traffic per CTA from (128 + BN) to (128 + BN/2) rows per k-block.  A ring slot is refilled only
// when the consumers of BOTH CTAs have released it (each consumer warp arrives on its own and on the peer's barrier).
//
// Epilogue warpgroups, one handoff per 64-row half h: consumer warpgroup h stages its half of a finished tile's
// accumulator and arrives on acc_full[h], then goes on with the next tile's k-blocks; epilogue warpgroup h (warpgroup
// 3 + h) waits on acc_full[h], runs the epilogue of those rows from the staging buffer and arrives on acc_empty[h], which
// consumer warpgroup h waits for before it stages its half of the next tile.  The two halves never wait for each other.
template <int BN, bool A_K, bool B_K, int MC>
__global__ void __launch_bounds__(kThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const KParams p) {
  constexpr int CL = MC;  // cluster size
  using L = SmemLayout<BN>;
  constexpr int S = L::kStages;
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B tiles need 1024-byte alignment.
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t bar_base = smem_base + L::kBarOffset;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (S + s); };
  auto acc_full = [&](int h) { return bar_base + 8u * (2 * S + h); };
  auto acc_empty = [&](int h) { return bar_base + 8u * (2 * S + 2 + h); };

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  // With MC = 2 a work item is a PAIR of M tiles: "tiles_m" counts pairs and this CTA owns tile 2*pair + rank
  // (a missing odd tile is all out-of-bounds rows: TMA zero-fills, the epilogue's row guard drops it).
  const int crank = MC > 1 ? (int)cluster_ctarank() : 0;
  const int tiles_m = ((p.M + BM - 1) / BM + CL - 1) / CL;
  const int tiles_n = (p.N + BN - 1) / BN;
  const int nbatch = p.nb1 * p.nb2;
  const int num_kb_all = (p.K + BK - 1) / BK;
  const int kb_per = (num_kb_all + p.ksplit - 1) / p.ksplit;
  const int total_tiles = tiles_m * tiles_n * nbatch * p.ksplit;  // work items = output tiles (pairs) x K splits
  const int work0 = blockIdx.x / CL, work_stride = gridDim.x / CL;
  const bool rowsum = !A_K && p.rowsum_a != nullptr;

  esp_pdl_trigger();  // the next kernel may be scheduled behind this grid's CTAs (it waits for our completion itself)
  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(full_bar(s), 1);
      // one arrive per consumer warp of every CTA of the cluster (+2: the two row-sum warps also read the A tile)
      mbar_init(empty_bar(s), 8 * CL + (rowsum ? 2 : 0));
    }
    for (int h = 0; h < 2; ++h) {
      mbar_init(acc_full(h), 128);   // every thread of consumer warpgroup h, after its accumulator stores
      mbar_init(acc_empty(h), 128);  // every thread of epilogue warpgroup h, after its staging reads
    }
    fence_mbar_init();
  }
  __syncthreads();
  if (MC > 1) cluster_sync_all();  // peer barriers are initialised before any multicast / remote arrive
  // barrier init and descriptor prefetch above overlap the previous kernel's tail; nothing before this point touches
  // global memory written by earlier kernels
  esp_pdl_wait();

  if (warp < 4) {
    if (warp == 0) {
      // ================================ TMA producer =====================================
      if (lane == 0) {
        uint32_t it = 0;
        for (int work = work0; work < total_tiles; work += work_stride) {
          const int ks = work % p.ksplit;
          const int tile = work / p.ksplit;
          const int kb0 = ks * kb_per;
          const int kb1 = min(num_kb_all, kb0 + kb_per);
          if (kb0 >= kb1) continue;  // empty K split (all roles skip it identically)
          const int mt = (tile % tiles_m) * CL + crank;
          const int rest = tile / tiles_m;
          const int nt = rest % tiles_n;
          const int bt = rest / tiles_n;
          const int b1 = bt % p.nb1, b2 = bt / p.nb1;
          for (int kb = kb0; kb < kb1; ++kb, ++it) {
            const int s = it % S;
            const uint32_t ph = (it / S) & 1;
            mbar_wait(empty_bar(s), ph ^ 1);
            const uint32_t sa = smem_base + s * L::kStageBytes;
            const uint32_t sb = sa + L::kABytes;
            mbar_expect_tx(full_bar(s), L::kStageBytes);
            if (MC == 1 && p.cv.mode == 1) {
              // implicit im2col: the tile's box of positions, shifted by this K block's tap
              const ConvGeom& g = p.cv;
              const int tf = mt % g.tiles_f, tt = (mt / g.tiles_f) % g.tiles_t, cb = mt / (g.tiles_f * g.tiles_t);
              const int tap = kb / g.cblocks, c0 = (kb - tap * g.cblocks) * 64;
              tma_load_4d(sa, &tmA, full_bar(s), c0, (tf << g.bf_log2) * g.sf + g.offf[tap], tt * g.bt * g.st + g.offt[tap], cb);
              if (B_K) {
                tma_load_4d(sb, &tmB, full_bar(s), kb * BK, nt * BN, 0, 0);  // weights [Cout, (tap, ci)]
              } else {
#pragma unroll
                for (int j = 0; j < BN / 64; ++j)  // weights viewed (ci, tap, co): rows = 64 output channels of this tap
                  tma_load_4d(sb + j * (BK * 128), &tmB, full_bar(s), nt * BN + 64 * j, g.btap[tap], c0, 0);
              }
              continue;
            }
            if (MC == 1 && p.cv.mode == 2) {
              // weight gradient: K block = one box of 64 positions; A = dY^T, B = the input box shifted by the chunk's tap
              const ConvGeom& g = p.cv;
              const int tf = kb % g.tiles_f, tt = (kb / g.tiles_f) % g.tiles_t, cb = kb / (g.tiles_f * g.tiles_t);
#pragma unroll
              for (int j = 0; j < BM / 64; ++j)
                tma_load_4d(sa + j * (BK * 128), &tmA, full_bar(s), mt * BM + 64 * j, tf << g.bf_log2, tt * g.bt, cb);
#pragma unroll
              for (int j = 0; j < BN / 64; ++j) {
                const int n = nt * BN + 64 * j;
                if (n < p.N) {
                  const int tap = n / g.cin, c0 = n - tap * g.cin;
                  tma_load_4d(sb + j * (BK * 128), &tmB, full_bar(s), c0, (tf << g.bf_log2) * g.sf + g.offf[tap],
                              tt * g.bt * g.st + g.offt[tap], cb);
                } else {  // chunk beyond the last tap: an all-out-of-bounds box (zero fill; the bytes still arrive)
                  tma_load_4d(sb + j * (BK * 128), &tmB, full_bar(s), g.cin, 0, 0, cb);
                }
              }
              continue;
            }
            if (A_K) {
              tma_load_4d(sa, &tmA, full_bar(s), kb * BK, mt * BM, b1 * p.a_b1, b2 * p.a_b2);
            } else {
#pragma unroll
              for (int j = 0; j < BM / 64; ++j)
                tma_load_4d(sa + j * (BK * 128), &tmA, full_bar(s), mt * BM + 64 * j, kb * BK,
                            b1 * p.a_b1, b2 * p.a_b2);
            }
            if (MC == 1) {
              if (B_K) {
                tma_load_4d(sb, &tmB, full_bar(s), kb * BK, nt * BN, b1 * p.b_b1, b2 * p.b_b2);
              } else {
#pragma unroll
                for (int j = 0; j < BN / 64; ++j)
                  tma_load_4d(sb + j * (BK * 128), &tmB, full_bar(s), nt * BN + 64 * j, kb * BK,
                              b1 * p.b_b1, b2 * p.b_b2);
              }
            } else {
              // this CTA fetches half `crank` of the B tile for both CTAs (the tensor map's box is BN/2 rows when
              // B is K-major; MN-major tiles are made of 64-wide chunks, half of them each)
              if (B_K) {
                tma_load_4d_mc(sb + crank * (BN / 2) * 128, &tmB, full_bar(s), kb * BK, nt * BN + crank * (BN / 2),
                               b1 * p.b_b1, b2 * p.b_b2, (uint16_t)0x3);
              } else {
#pragma unroll
                for (int j = 0; j < BN / 128; ++j) {
                  const int jj = crank * (BN / 128) + j;
                  tma_load_4d_mc(sb + jj * (BK * 128), &tmB, full_bar(s), nt * BN + 64 * jj, kb * BK, b1 * p.b_b1,
                                 b2 * p.b_b2, (uint16_t)0x3);
                }
              }
            }
          }
        }
      }
    } else if (rowsum && (warp == 2 || warp == 3)) {
      // ================================ bias gradient ======================================
      // Weight-gradient GEMMs (A = dy^T, MN-major): the row sums of A over the whole reduction are the bias gradient of the
      // same layer.  Two warps of the producer warpgroup read every A tile from shared memory (the data the tensor cores
      // consume anyway) and accumulate it -- the separate column-sum pass over dy disappears.
      // A tile layout (MN-major, SWIZZLE_128B): BM/64 boxes of [BK k-rows][64 m]; row k of a box is 128 bytes, its 16-byte
      // unit u (8 consecutive m) lives at unit u ^ (k & 7).  Lane l owns unit (l & 15) of the 16 units of a k-row pair.
      const int u = lane & 15;
      const uint32_t unit_base = (uint32_t)(u >> 3) * (BK * 128);
      const int u7 = u & 7;
      const int parts = tiles_n >= 4 ? 4 : (tiles_n >= 2 ? 2 : 1);  // CTAs per M tile that share the summing
      const int rows_per = 32 / parts;                              // k rows per warp, CTA and k-block
      uint32_t it = 0;
      for (int work = work0; work < total_tiles; work += work_stride) {
        const int ks = work % p.ksplit;
        const int tile = work / p.ksplit;
        const int kb0 = ks * kb_per;
        const int kb1 = min(num_kb_all, kb0 + kb_per);
        if (kb0 >= kb1) continue;
        const int mt = (tile % tiles_m) * CL + crank;
        const int nt = (tile / tiles_m) % tiles_n;
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        for (int kb = kb0; kb < kb1; ++kb, ++it) {
          const int s = it % S;
          mbar_wait(full_bar(s), (it / S) & 1);
          if (nt < parts) {
            // The CTAs that share this M tile (one per N tile) split the k rows of every tile between them, so each of the
            // two warps reads 16 / parts row pairs per k-block (every CTA still takes part in the barrier protocol).
            const uint8_t* ta_ = smem + s * L::kStageBytes + unit_base;
            const int kbase = (warp - 2) * 32 + nt * rows_per + (lane >> 4);
            uint4 q4[8];
#pragma unroll 1
            for (int i0 = 0; i0 < rows_per / 2; i0 += 8) {
#pragma unroll
              for (int i = 0; i < 8; ++i) {  // 8 independent 16-byte loads in flight
                const int k = kbase + 2 * (i0 + i);
                q4[i] = (i0 + i < rows_per / 2) ? *reinterpret_cast<const uint4*>(ta_ + k * 128 + ((u7 ^ (k & 7)) << 4))
                                                : make_uint4(0, 0, 0, 0);
              }
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                // bf16 -> fp32 is a shift / mask of the packed word
                acc[0] += __uint_as_float(q4[i].x << 16); acc[1] += __uint_as_float(q4[i].x & 0xFFFF0000u);
                acc[2] += __uint_as_float(q4[i].y << 16); acc[3] += __uint_as_float(q4[i].y & 0xFFFF0000u);
                acc[4] += __uint_as_float(q4[i].z << 16); acc[5] += __uint_as_float(q4[i].z & 0xFFFF0000u);
                acc[6] += __uint_as_float(q4[i].w << 16); acc[7] += __uint_as_float(q4[i].w & 0xFFFF0000u);
              }
            }
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(empty_bar(s));
        }
        if (nt < parts) {
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[e] += __shfl_xor_sync(0xffffffffu, acc[e], 16);
          if (lane < 16) {
            const int m0 = mt * BM + u * 8;
#pragma unroll
            for (int e = 0; e < 8; ++e)
              if (m0 + e < p.M) atomicAdd(p.rowsum_a + m0 + e, acc[e] * p.rowsum_scale);
          }
        }
      }
    }
  } else if (warp < 12) {
    // ================================ MMA ================================================
    const int wg = (warp >> 2) - 1;       // consumer warpgroup: rows 64 wg .. 64 wg + 63 of the tile
    const int t = threadIdx.x - 128 * (wg + 1);
    float* const stg = reinterpret_cast<float*>(smem + L::kEpiOffset) + wg * 64 * L::kEpiLd;
    float acc[BN / 2];
    uint32_t it = 0, staged = 0;
    PhaseClk ph;
    const long long loop0 = ph.now();
    for (int work = work0; work < total_tiles; work += work_stride) {
      const int ks = work % p.ksplit;
      const int tile = work / p.ksplit;
      const int kb0 = ks * kb_per;
      const int kb1 = min(num_kb_all, kb0 + kb_per);
      if (kb0 >= kb1) continue;
      const int mt = (tile % tiles_m) * CL + crank;
      const int rest = tile / tiles_m;
      const int nt = rest % tiles_n;
      const int bt = rest / tiles_n;

      // ---- mainloop: one wgmma group per k-block, at most two in flight; a slot is released once its group retired
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb, ++it) {
        const int s = it % S;
        mbar_wait(full_bar(s), (it / S) & 1);
        const uint32_t sa = smem_base + s * L::kStageBytes + wg * (64 * 128);  // K-major: 64 rows; MN-major: chunk wg
        const uint32_t sb = smem_base + s * L::kStageBytes + L::kABytes;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          const uint64_t da = A_K ? make_sdesc(sa + k * 32, 16, 1024) : make_sdesc(sa + k * 2048, BK * 128, 1024);
          const uint64_t db = B_K ? make_sdesc(sb + k * 32, 16, 1024) : make_sdesc(sb + k * 2048, BK * 128, 1024);
          mma_k16<BN, A_K ? 0 : 1, B_K ? 0 : 1>(acc, da, db, (kb != kb0 || k != 0) ? 1u : 0u);
        }
        wgmma_commit();
        if (prev >= 0) {
          wgmma_wait<1>();
          if (lane == 0) {
            mbar_arrive(empty_bar(prev));
            if (MC > 1) mbar_arrive_cluster(empty_bar(prev), (uint32_t)(crank ^ 1));
          }
        }
        prev = s;
      }
      wgmma_wait<0>();
      fence_acc(acc);
      if (lane == 0) {
        mbar_arrive(empty_bar(prev));
        if (MC > 1) mbar_arrive_cluster(empty_bar(prev), (uint32_t)(crank ^ 1));
      }

      // ---- stage the accumulator: thread t holds rows fr, fr + 8 of the warpgroup's 64, two columns of every 8
      const int fr = (t >> 5) * 16 + ((t & 31) >> 2), fc = 2 * (t & 3);
      const long long w0 = ph.now();
      mbar_wait(acc_empty(wg), (staged & 1) ^ 1);  // epilogue warpgroup wg has read this half of the previous tile
      ph.add(kPhMmaAccWait, ph.now() - w0);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        *reinterpret_cast<float2*>(stg + fr * L::kEpiLd + 8 * j + fc) = make_float2(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<float2*>(stg + (fr + 8) * L::kEpiLd + 8 * j + fc) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      }
      mbar_arrive(acc_full(wg));
      ++staged;
    }
    ph.add(kPhMmaLoop, ph.now() - loop0);
    ph.flush(t == 0);
  } else {
    // ================================ epilogue warpgroups ==================================
    // Epilogue warpgroup h serves the 64 rows that MMA warpgroup h stages, two threads per row: lane l of warp w takes
    // row 16 w + (l & 15) of the half and column half l >> 4.  The 8 lanes of a quarter-warp then read 8 distinct rows
    // at the padded row pitch, free of bank conflicts (two lanes of one row would sit BN / 2 = 0 mod 32 banks apart).
    const int h = (warp - 12) >> 2;
    const int ml = 64 * h + 16 * (warp & 3) + (lane & 15);
    const int ch = lane >> 4;
    const EpiParams& e = p.ep;
    const unsigned long long seed = e.seed + (e.seed_ptr ? *e.seed_ptr : 0ull);
    const float* const src = reinterpret_cast<const float*>(smem + L::kEpiOffset) + ml * L::kEpiLd + ch * (BN / 2);
    uint32_t staged = 0;
    PhaseClk ph;
    const long long loop0 = ph.now();
    for (int work = work0; work < total_tiles; work += work_stride) {
      const int ks = work % p.ksplit;
      const int tile = work / p.ksplit;
      const int kb0 = ks * kb_per;
      const int kb1 = min(num_kb_all, kb0 + kb_per);
      if (kb0 >= kb1) continue;
      const int mt = (tile % tiles_m) * CL + crank;
      const int rest = tile / tiles_m;
      const int nt = rest % tiles_n;
      const int bt = rest / tiles_n;
      mbar_wait(acc_full(h), staged & 1);
      const long long b0 = ph.now();
      epilogue_row<BN, MC>(p, e, seed, src, ml, mt, bt, nt * BN + ch * (BN / 2));
      mbar_arrive(acc_empty(h));
      ph.add(kPhEpiBusy, ph.now() - b0);
      ph.add(kPhEpiTiles, 1);
      ++staged;
    }
    ph.add(kPhEpiLoop, ph.now() - loop0);
    ph.flush((threadIdx.x & 127) == 0);
  }

  __syncthreads();
  if (MC > 1) cluster_sync_all();  // no CTA exits while its peer may still signal or write into its shared memory
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (PFN_encodeTiled)p;
  }
  return fn;
}

// 4-D bf16 SWIZZLE_128B tensor map: dims innermost first, byte strides of dims 1-3, box[0] = 64 elements (one
// SWIZZLE_128B row).  Element strides > 1 make the box skip positions (strided convolution: boxDim = elements spanned,
// the engine writes ceil(boxDim / stride) of them densely).
int make_tmap_box(CUtensorMap* tm, const void* base, const cuuint64_t dims[4], const cuuint64_t strides_b[3],
                  const cuuint32_t box[4], const cuuint32_t estr[4]) {
  PFN_encodeTiled enc = get_encode();
  ESP_CHECK(enc != nullptr, "cuTensorMapEncodeTiled entry point unavailable");
  // cuTensorMapEncodeTiled is a DRIVER call: the calling thread needs a current context.  PyTorch's
  // autograd engine runs backward on its own threads where only the runtime device is set, so bind the
  // primary context once per thread (cudaFree(0) is the canonical no-op that does it).
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) {
    ESP_CUDA(cudaFree(0));
    ctx_bound = true;
  }
  ESP_CHECK(((uintptr_t)base & 15) == 0, "TMA operand base must be 16-byte aligned");
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides_b, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  ESP_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d): dims %llu %llu %llu %llu box %u %u %u %u", (int)r,
            (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2], (unsigned long long)dims[3],
            box[0], box[1], box[2], box[3]);
  return 0;
}

// co-resident 2-CTA clusters of a kernel variant (clusters sit inside one GPC: with odd SM counts per GPC fewer than
// SMs/2 pairs fit at once -- ask the runtime instead of assuming)
template <typename K>
int cluster_slots(K kfn, int smem_bytes, int threads) {
  int slots = esp_num_sms() / 2;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(esp_num_sms() / 2 * 2);
  cfg.blockDim = dim3(threads);
  cfg.dynamicSmemBytes = smem_bytes;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, kfn, &cfg) == cudaSuccess && n > 0 && n < slots) slots = n;
  (void)cudaGetLastError();
  return slots;
}

template <int BN, bool A_K, bool B_K, int MC>
int launch(const CUtensorMap& ta, const CUtensorMap& tb, const KParams& kp, cudaStream_t st) {
  using L = SmemLayout<BN>;
  auto kfn = gemm_wgmma_kernel<BN, A_K, B_K, MC>;
  ESP_SMEM_OPTIN(kfn, L::kTotal);
  const int tiles_m = (((kp.M + BM - 1) / BM) + MC - 1) / MC;
  const int work = tiles_m * ((kp.N + BN - 1) / BN) * kp.nb1 * kp.nb2 * kp.ksplit;
  static int slots = 0;  // persistent grid = what is co-resident
  if (slots == 0) slots = MC > 1 ? cluster_slots(kfn, L::kTotal, kThreads) : esp_num_sms();
  int grid = (work < slots ? work : slots) * MC;
  if (grid < 1) return 0;
  ESP_CUDA(esp_launch_cluster(kfn, grid, kThreads, L::kTotal, st, MC, ta, tb, kp));
  return 0;
}

template <int BN, int MC>
int dispatch_major(bool ak, bool bk, const CUtensorMap& ta, const CUtensorMap& tb, const KParams& kp, cudaStream_t st) {
  if (ak && bk) return launch<BN, true, true, MC>(ta, tb, kp, st);
  if (ak && !bk) return launch<BN, true, false, MC>(ta, tb, kp, st);
  if (!ak && bk) return launch<BN, false, true, MC>(ta, tb, kp, st);
  return launch<BN, false, false, MC>(ta, tb, kp, st);
}

}  // namespace

#ifdef ESP_GEMM_PHASES
// SM clocks per phase (kPhMmaAccWait .. kPhEpiTiles) summed since the last call, then reset
extern "C" int esp_gemm_phase_clk(unsigned long long* out) {
  ESP_CUDA(cudaMemcpyFromSymbol(out, g_gemm_phase_clk, sizeof(unsigned long long) * kPhases));
  static const unsigned long long zero[kPhases] = {};
  ESP_CUDA(cudaMemcpyToSymbol(g_gemm_phase_clk, zero, sizeof(zero)));
  return 0;
}
#endif

int esp_make_tmap_bf16(CUtensorMap* tm, const void* base, long inner, long rows, long ld, int nb1, long s1, int nb2,
                       long s2, int box_rows) {
  ESP_CHECK((ld % 8) == 0, "GEMM operand leading dimension (%ld) must be a multiple of 8 elements", ld);
  // Broadcast / singleton batch dims get size 1 (coordinate forced to 0 by the kernel) and a
  // dummy legal stride.
  long dummy = ((rows * ld + 7) / 8) * 8;
  if (nb1 <= 1 || s1 == 0) { nb1 = 1; s1 = dummy; }
  if (nb2 <= 1 || s2 == 0) { nb2 = 1; s2 = dummy * (nb1 > 1 ? nb1 : 1); }
  ESP_CHECK((s1 % 8) == 0 && (s2 % 8) == 0, "GEMM batch strides must be multiples of 8 elements");
  const cuuint64_t dims[4] = {(cuuint64_t)inner, (cuuint64_t)rows, (cuuint64_t)nb1, (cuuint64_t)nb2};
  const cuuint64_t strides[3] = {(cuuint64_t)ld * 2, (cuuint64_t)s1 * 2, (cuuint64_t)s2 * 2};
  const cuuint32_t box[4] = {64, (cuuint32_t)box_rows, 1, 1};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  return make_tmap_box(tm, base, dims, strides, box, estr);
}

extern "C" int esp_gemm_bf16(const EspGemm* g, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(g != nullptr, "null gemm descriptor");
  ESP_CHECK(g->M >= 0 && g->N >= 0 && g->K > 0, "bad GEMM shape %ld x %ld x %ld", (long)g->M, (long)g->N,
            (long)g->K);
  ESP_CHECK(g->tile_n == 0 || g->tile_n == 64 || g->tile_n == 128, "GEMM tile_n must be 0 (auto), 64 or 128 (got %d)",
            (int)g->tile_n);
  if (g->M == 0 || g->N == 0) return 0;
  const int nb1 = g->nb1 > 0 ? g->nb1 : 1, nb2 = g->nb2 > 0 ? g->nb2 : 1;
  CUtensorMap ta, tb;
  const bool ak = g->a_kmajor != 0, bk = g->b_kmajor != 0;
  // tile width: wide tiles have the best operand-bytes per flop (a 128 x BN tile reads (128+BN)*64*2 B from L2 per
  // 128*BN*64*2 flop); narrow ones only when N is small or the machine would be badly under-filled.
  const int sms = esp_num_sms();
  const long tm = (g->M + BM - 1) / BM;
  auto tiles_for = [&](int w) { return tm * ((g->N + w - 1) / w) * (long)nb1 * nb2; };
  int bn;
  int ksplit = 1;
  int mode = 1;  // 1: single CTA, 2: 2-CTA cluster sharing the B tile (multicast)
  const int num_kb = (int)((g->K + BK - 1) / BK);
  // utilisation of `slots` persistent workers by `items` equal work items
  auto eff = [](long items, long slots) {
    const long waves = (items + slots - 1) / slots;
    return (double)items / (double)(waves * slots);
  };
  if (g->accumulate) {
    // gradient GEMMs: long reduction (K = rows of the batch), small output -> split K across CTAs and
    // accumulate with vector reductions; keep >= 4 k-blocks per split.
    bn = g->N > 64 ? 128 : 64;
    const long t = tiles_for(bn);
    const int max_split = num_kb / 4 > 0 ? num_kb / 4 : 1;
    double best = -1.0;
    for (int ks = 1; ks <= max_split && (long)(ks - 1) * t < sms; ++ks) {
      const double e = eff(t * ks, sms) - 0.01 * ks;  // prefer fewer splits at equal utilisation (less red traffic)
      if (e > best) { best = e; ksplit = ks; }
    }
  } else {
    if (g->N <= 64) bn = 64;
    else if (g->N <= 128 && tiles_for(128) * 10 < (long)sms * 6 && tiles_for(64) < sms) bn = 64;
    else bn = 128;
  }
  if (g->tile_n) bn = g->tile_n;
  // 2-CTA multicast pairs along M: worth it when the pairing wastes (almost) no tile
  if (bn == 128 && (tm % 2 == 0 || tm >= 16)) mode = 2;
  int rc;
  if (ak) rc = esp_make_tmap_bf16(&ta, g->A, g->K, g->M, g->lda, nb1, g->sA1, nb2, g->sA2, BM);
  else    rc = esp_make_tmap_bf16(&ta, g->A, g->M, g->K, g->lda, nb1, g->sA1, nb2, g->sA2, BK);
  if (rc) return rc;
  if (bk) rc = esp_make_tmap_bf16(&tb, g->B, g->K, g->N, g->ldb, nb1, g->sB1, nb2, g->sB2, bn / mode);
  else    rc = esp_make_tmap_bf16(&tb, g->B, g->N, g->K, g->ldb, nb1, g->sB1, nb2, g->sB2, BK);
  if (rc) return rc;

  KParams kp;
  kp.cv.mode = 0;
  kp.rowsum_a = g->rowsum_a;
  kp.rowsum_scale = g->rowsum_scale;
  if (g->rowsum_a) {
    ESP_CHECK(!ak && g->accumulate && nb1 == 1 && nb2 == 1, "rowsum_a needs an MN-major A operand, accumulate = 1, no batch dims");
  }
  kp.M = (int)g->M; kp.N = (int)g->N; kp.K = (int)g->K; kp.nb1 = nb1; kp.nb2 = nb2; kp.ksplit = ksplit;
  kp.a_b1 = (nb1 > 1 && g->sA1 != 0) ? 1 : 0;
  kp.a_b2 = (nb2 > 1 && g->sA2 != 0) ? 1 : 0;
  kp.b_b1 = (nb1 > 1 && g->sB1 != 0) ? 1 : 0;
  kp.b_b2 = (nb2 > 1 && g->sB2 != 0) ? 1 : 0;
  EpiParams& e = kp.ep;
  e.C = g->C; e.C2 = (bf16*)g->C2; e.bias = (const bf16*)g->bias; e.aux = (const bf16*)g->aux; e.R = g->R;
  e.ldc = g->ldc; e.ld_aux = g->ld_aux; e.ldr = g->ldr;
  e.sC1 = g->sC1; e.sC2 = g->sC2; e.sAux1 = g->sAux1; e.sAux2 = g->sAux2; e.sR1 = g->sR1; e.sR2 = g->sR2;
  e.c_f32 = g->c_f32; e.r_f32 = g->r_f32; e.act = g->act; e.skew_r = g->skew_r; e.atomic = g->accumulate ? 1 : 0;
  e.drop_mode = (g->drop_p > 0.f) ? g->drop_mode : 0;
  e.alpha = g->alpha; e.beta = g->beta;
  e.drop_thresh = esp_dropout_thresh(g->drop_p);
  e.drop_scale = esp_dropout_scale(g->drop_p);
  e.seed = g->seed;
  e.seed_ptr = (const unsigned long long*)g->seed_ptr;
  ESP_CHECK(g->C != nullptr, "GEMM output pointer is null");
  ESP_CHECK(!g->accumulate || g->c_f32, "accumulate (atomic) output must be fp32");
  ESP_CHECK(!(e.act >= ESP_ACT_RELU_BWD) || e.aux != nullptr, "activation-gradient epilogue needs aux");
  if (bn == 64) return dispatch_major<64, 1>(ak, bk, ta, tb, kp, st);
  return mode == 2 ? dispatch_major<128, 2>(ak, bk, ta, tb, kp, st) : dispatch_major<128, 1>(ak, bk, ta, tb, kp, st);
}

// ------------------------------------------------------------------------------------------
// 3x3 convolutions of the conv front end (implicit GEMMs, ConvGeom above)
// ------------------------------------------------------------------------------------------
namespace {

// tensor map over a channels-last activation [B, T, F, C] (dims innermost first: C, F, T, B), boxes of box_f x box_t
// positions strided by (sf, st)
int act_tmap(CUtensorMap* tm, const void* base, int B, int T, int F, int C, int box_f, int box_t, int sf, int st) {
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)F, (cuuint64_t)T, (cuuint64_t)B};
  const cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)F * C * 2, (cuuint64_t)T * F * C * 2};
  const cuuint32_t box[4] = {64, (cuuint32_t)(box_f * sf), (cuuint32_t)(box_t * st), 1};
  const cuuint32_t estr[4] = {1, (cuuint32_t)sf, (cuuint32_t)st, 1};
  return make_tmap_box(tm, base, dims, strides, box, estr);
}

// box of `n` positions: as wide along F as divides it evenly (power of two, at most 16), the rest along T
void pick_box(int n, int Fpos, int* bf_log2, int* bt) {
  int l = 0;
  while (l < 4 && (1 << (l + 1)) <= n && Fpos % (1 << (l + 1)) == 0) ++l;
  *bf_log2 = l;
  *bt = n >> l;
}

void zero_epi(KParams& kp) {
  EpiParams& e = kp.ep;
  e.C = nullptr; e.C2 = nullptr; e.bias = nullptr; e.aux = nullptr; e.R = nullptr;
  e.ldc = e.ld_aux = e.ldr = 0;
  e.sC1 = e.sC2 = e.sAux1 = e.sAux2 = e.sR1 = e.sR2 = 0;
  e.c_f32 = e.r_f32 = e.act = e.drop_mode = e.skew_r = e.atomic = 0;
  e.alpha = 1.f; e.beta = 0.f; e.drop_scale = 1.f; e.drop_thresh = 0; e.seed = 0; e.seed_ptr = nullptr;
  kp.rowsum_a = nullptr; kp.rowsum_scale = 0.f;
  kp.nb1 = kp.nb2 = 1; kp.ksplit = 1; kp.a_b1 = kp.a_b2 = kp.b_b1 = kp.b_b2 = 0;
}

int conv_check(int B, int T, int F, int Cin, int Cout, int st, int sf) {
  ESP_CHECK(B > 0 && T > 0 && F > 0, "conv3x3: empty input");
  ESP_CHECK(Cin % 64 == 0 && Cout % 64 == 0, "conv3x3 (tensor-core path): channel counts must be multiples of 64 (got %d -> %d)", Cin, Cout);
  ESP_CHECK((st == 1 || st == 2) && (sf == 1 || sf == 2), "conv3x3: strides 1 or 2 (got %d x %d)", st, sf);
  return 0;
}

}  // namespace

// y[b, to, fo, :] = sum_{r,s,ci} x[b, to*st + r - 1, fo*sf + s - 1, ci] * w[:, r, s, ci]      (zero padding 1, no bias)
// x [B, T, F, Cin], w [Cout, 3, 3, Cin], y [B, ceil(T/st), ceil(F/sf), Cout], all bf16 channels-last.
extern "C" int esp_conv3x3_fwd(const void* x, const void* w, void* y, int32_t B, int32_t T, int32_t F, int32_t Cin,
                               int32_t Cout, int32_t st, int32_t sf, void* stream) {
  cudaStream_t s_ = (cudaStream_t)stream;
  if (int rc = conv_check(B, T, F, Cin, Cout, st, sf)) return rc;
  const int To = (T + st - 1) / st, Fo = (F + sf - 1) / sf;
  KParams kp;
  zero_epi(kp);
  ConvGeom& g = kp.cv;
  g.mode = 1;
  pick_box(128, Fo, &g.bf_log2, &g.bt);
  const int bf = 1 << g.bf_log2;
  g.tiles_t = (To + g.bt - 1) / g.bt;
  g.tiles_f = (Fo + bf - 1) / bf;
  g.st = st; g.sf = sf; g.cblocks = Cin / 64; g.cin = Cin;
  g.OT = To; g.OF = Fo; g.ost = g.osf = 1; g.opt = g.opf = 0;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      g.offt[r * 3 + c] = (signed char)(r - 1);
      g.offf[r * 3 + c] = (signed char)(c - 1);
      g.btap[r * 3 + c] = (signed char)(r * 3 + c);
    }
  const int bn = Cout % 128 == 0 ? 128 : 64;
  CUtensorMap ta, tb;
  if (int rc = act_tmap(&ta, x, B, T, F, Cin, bf, g.bt, sf, st)) return rc;
  if (int rc = esp_make_tmap_bf16(&tb, w, 9L * Cin, Cout, 9L * Cin, 1, 0, 1, 0, bn)) return rc;
  kp.M = B * g.tiles_t * g.tiles_f * BM; kp.N = Cout; kp.K = 9 * Cin;
  kp.ep.C = y; kp.ep.ldc = Cout;
  return bn == 128 ? launch<128, true, true, 1>(ta, tb, kp, s_) : launch<64, true, true, 1>(ta, tb, kp, s_);
}

// dx[b, t, f, :] = sum over the taps (r, s) and output positions with to*st + r - 1 == t, fo*sf + s - 1 == f of
//                  dy[b, to, fo, :] . w[:, r, s, :]
// One launch per parity class (t mod st, f mod sf): inside a class every position sees the same taps, so the class is a
// small un-strided convolution of dy whose outputs are written st x sf apart.
extern "C" int esp_conv3x3_dgrad(const void* dy, const void* w, void* dx, int32_t B, int32_t T, int32_t F, int32_t Cin,
                                 int32_t Cout, int32_t st, int32_t sf, void* stream) {
  cudaStream_t s_ = (cudaStream_t)stream;
  if (int rc = conv_check(B, T, F, Cin, Cout, st, sf)) return rc;
  const int To = (T + st - 1) / st, Fo = (F + sf - 1) / sf;
  const int bn = Cin % 128 == 0 ? 128 : 64;
  CUtensorMap tb;
  {
    // weights [Cout][tap][Cin] viewed (ci, tap, co): a K block = 64 output channels of one tap, MN-major rows of 64 ci
    const cuuint64_t dims[4] = {(cuuint64_t)Cin, 9, (cuuint64_t)Cout, 1};
    const cuuint64_t strides[3] = {(cuuint64_t)Cin * 2, (cuuint64_t)9 * Cin * 2, (cuuint64_t)9 * Cin * Cout * 2};
    const cuuint32_t box[4] = {64, 1, 64, 1};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    if (int rc = make_tmap_box(&tb, w, dims, strides, box, estr)) return rc;
  }
  for (int pt = 0; pt < st; ++pt)
    for (int pf = 0; pf < sf; ++pf) {
      const int U = (T - pt + st - 1) / st, V = (F - pf + sf - 1) / sf;  // positions of this class
      if (U <= 0 || V <= 0) continue;
      KParams kp;
      zero_epi(kp);
      ConvGeom& g = kp.cv;
      g.mode = 1;
      pick_box(128, V, &g.bf_log2, &g.bt);
      const int bf = 1 << g.bf_log2;
      g.tiles_t = (U + g.bt - 1) / g.bt;
      g.tiles_f = (V + bf - 1) / bf;
      g.st = g.sf = 1; g.cblocks = Cout / 64; g.cin = Cin;
      g.OT = T; g.OF = F; g.ost = st; g.osf = sf; g.opt = pt; g.opf = pf;
      int nt = 0;
      for (int r = 0; r < 3; ++r) {
        if ((pt + 1 - r) % st != 0) continue;  // t = to*st + r - 1  =>  to = (t + 1 - r) / st = u + (pt + 1 - r) / st
        for (int c = 0; c < 3; ++c) {
          if ((pf + 1 - c) % sf != 0) continue;
          g.offt[nt] = (signed char)((pt + 1 - r) / st);
          g.offf[nt] = (signed char)((pf + 1 - c) / sf);
          g.btap[nt] = (signed char)(r * 3 + c);
          ++nt;
        }
      }
      ESP_CHECK(nt > 0, "conv3x3 dgrad: parity class without taps");
      CUtensorMap ta;
      if (int rc = act_tmap(&ta, dy, B, To, Fo, Cout, bf, g.bt, 1, 1)) return rc;
      kp.M = B * g.tiles_t * g.tiles_f * BM; kp.N = Cin; kp.K = nt * Cout;
      kp.ep.C = dx; kp.ep.ldc = Cin;
      const int rc = bn == 128 ? launch<128, true, false, 1>(ta, tb, kp, s_) : launch<64, true, false, 1>(ta, tb, kp, s_);
      if (rc) return rc;
    }
  return 0;
}

// dw[co, r, s, ci] += sum_{b, to, fo} dy[b, to, fo, co] * x[b, to*st + r - 1, fo*sf + s - 1, ci]      (fp32 accumulate)
extern "C" int esp_conv3x3_wgrad(const void* dy, const void* x, float* dw, int32_t B, int32_t T, int32_t F, int32_t Cin,
                                 int32_t Cout, int32_t st, int32_t sf, void* stream) {
  cudaStream_t s_ = (cudaStream_t)stream;
  if (int rc = conv_check(B, T, F, Cin, Cout, st, sf)) return rc;
  const int To = (T + st - 1) / st, Fo = (F + sf - 1) / sf;
  KParams kp;
  zero_epi(kp);
  ConvGeom& g = kp.cv;
  g.mode = 2;
  pick_box(64, Fo, &g.bf_log2, &g.bt);
  const int bf = 1 << g.bf_log2;
  g.tiles_t = (To + g.bt - 1) / g.bt;
  g.tiles_f = (Fo + bf - 1) / bf;
  g.st = st; g.sf = sf; g.cblocks = Cin / 64; g.cin = Cin;
  g.OT = To; g.OF = Fo; g.ost = g.osf = 1; g.opt = g.opf = 0;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      g.offt[r * 3 + c] = (signed char)(r - 1);
      g.offf[r * 3 + c] = (signed char)(c - 1);
      g.btap[r * 3 + c] = (signed char)(r * 3 + c);
    }
  CUtensorMap ta, tb;
  if (int rc = act_tmap(&ta, dy, B, To, Fo, Cout, bf, g.bt, 1, 1)) return rc;
  if (int rc = act_tmap(&tb, x, B, T, F, Cin, bf, g.bt, sf, st)) return rc;
  const long kblocks = (long)B * g.tiles_t * g.tiles_f;
  kp.M = Cout; kp.N = 9 * Cin; kp.K = (int)(kblocks * BK);
  ESP_CHECK(kblocks * BK < (1L << 31), "conv3x3 wgrad: too many positions");
  const int tiles = ((Cout + BM - 1) / BM) * ((9 * Cin + 127) / 128);
  int ks = esp_num_sms() / tiles;  // fill the machine; every split keeps a long reduction (>= 8 position boxes)
  if (ks > kblocks / 8) ks = (int)(kblocks / 8);
  if (ks < 1) ks = 1;
  kp.ksplit = ks;
  kp.ep.C = dw; kp.ep.ldc = 9 * Cin; kp.ep.c_f32 = 1; kp.ep.atomic = 1;
  return launch<128, false, false, 1>(ta, tb, kp, s_);
}
