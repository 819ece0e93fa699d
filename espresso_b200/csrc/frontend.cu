// espresso_b200 -- fused on-device front end (one launch per batch):
//   framing (25 ms / 10 ms, snip_edges) -> DC removal -> pre-emphasis 0.97 -> Povey window ->
//   zero-pad 400->512 -> real FFT -> power -> 80 triangular mel bins -> log(max(eps,.)) ->
//   global CMVN -> adaptive SpecAugment (host-drawn mask descriptors, fill = utterance mean).
//
// Reference path being replaced (CPU, per utterance, in DataLoader workers):
//   espresso/data/feat_text_dataset.py:128-161
//   espresso/tools/utils.py:426-454 -> torchaudio/compliance/kaldi.py:154-218,436-512,514-646
//   fairseq/data/audio/feature_transforms/global_cmvn.py:26-29
//   espresso/data/feature_transforms/adaptive_specaugment.py:77-136
//
// Data movement: every waveform sample is read from HBM exactly once with 16-byte loads (a CTA stages the samples of
// 64 consecutive frames in shared memory, so the 2.5x frame overlap is served on-chip); each
// output element is written once (+ once more inside SpecAugment masks, painted by a second grid-wide kernel once the
// utterance means are known).  Algorithmic bytes per
// audio-second: 16000*4 (fp32 wave) + 100*80*2 (bf16 feats) = 80 000 B.
#include "common.cuh"
#include "espresso_b200.h"
#include <math.h>
#include <mutex>

namespace {

constexpr int kFrameLen = 400;
constexpr int kShift = 160;
constexpr int kBins = 80;
constexpr int kFramesPerCta = 64;  // per-CTA table staging (8 KB) amortised over 64 frames; 42 KB of samples
constexpr int kWarps = 8;
constexpr int kSamplesPerCta = (kFramesPerCta - 1) * kShift + kFrameLen;  // 5360
constexpr int kMaxMelW = 640;  // total non-zero triangular weights (actual ~ 510)

struct Tables {
  float window[kFrameLen];
  float tw256[256];  // (cos, -sin)(2*pi*k/256), k < 128
  float tw512[512];  // (cos, -sin)(2*pi*k/512), k < 256
  int mel_start[kBins];
  int mel_len[kBins];
  int mel_off[kBins];
  float mel_w[kMaxMelW];
};

__device__ Tables g_tables;

void build_tables(Tables& t) {
  const double PI = 3.14159265358979323846;
  for (int i = 0; i < kFrameLen; ++i) {
    // torch.hann_window(400, periodic=False).pow(0.85)   (kaldi.py:98-100)
    float h = (float)(0.5 - 0.5 * cos(2.0 * PI * i / (kFrameLen - 1)));
    t.window[i] = powf(h, 0.85f);
  }
  for (int k = 0; k < 128; ++k) {
    t.tw256[2 * k] = (float)cos(2.0 * PI * k / 256.0);
    t.tw256[2 * k + 1] = (float)(-sin(2.0 * PI * k / 256.0));
  }
  for (int k = 0; k < 256; ++k) {
    t.tw512[2 * k] = (float)cos(2.0 * PI * k / 512.0);
    t.tw512[2 * k + 1] = (float)(-sin(2.0 * PI * k / 512.0));
  }
  // get_mel_banks(80, 512, 16000, 20, 0 -> nyquist)   (kaldi.py:436-512); computed in fp32 like the
  // reference's tensor arithmetic.
  auto mel = [](float f) { return 1127.0f * logf(1.0f + f / 700.0f); };
  const float low = mel(20.f), high = mel(8000.f);
  const float delta = (high - low) / (kBins + 1);
  int off = 0;
  for (int b = 0; b < kBins; ++b) {
    const float left = low + b * delta, center = low + (b + 1.0f) * delta, right = low + (b + 2.0f) * delta;
    int start = -1, len = 0;
    for (int k = 0; k < 256; ++k) {
      const float mk = mel(31.25f * k);
      const float up = (mk - left) / (center - left);
      const float down = (right - mk) / (right - center);
      const float w = fmaxf(0.f, fminf(up, down));
      if (w > 0.f) {
        if (start < 0) start = k;
        len = k - start + 1;
      }
    }
    if (start < 0) { start = 0; len = 0; }
    t.mel_start[b] = start;
    t.mel_len[b] = len;
    t.mel_off[b] = off;
    for (int k = start; k < start + len; ++k) {
      const float mk = mel(31.25f * k);
      const float up = (mk - left) / (center - left);
      const float down = (right - mk) / (right - center);
      if (off < kMaxMelW) t.mel_w[off] = fmaxf(0.f, fminf(up, down));
      ++off;
    }
  }
}

struct Smem {
  alignas(16) float samples[kSamplesPerCta];
  Tables t;
  float re[kWarps][256];
  float im[kWarps][256];
  float pw[kWarps][256];
  double red[kWarps];
};

template <typename WaveT>
__device__ __forceinline__ float load_sample(const WaveT* p);
template <>
__device__ __forceinline__ float load_sample<float>(const float* p) { return *p; }
template <>
__device__ __forceinline__ float load_sample<int16_t>(const int16_t* p) { return (float)(*p); }

template <typename WaveT>
__global__ void __launch_bounds__(kWarps * 32)
frontend_kernel(const WaveT* __restrict__ wave, long wave_ld, const int* __restrict__ n_samples,
                const float* __restrict__ cmvn_mean, const float* __restrict__ cmvn_std,
                const int* __restrict__ freq_masks, int n_freq_masks, const int* __restrict__ time_masks,
                int max_time_masks, void* __restrict__ out, int out_f32, int t_max, int* __restrict__ out_lens,
                double* __restrict__ ws_sum, unsigned int* __restrict__ ws_cnt) {
  esp_pdl();
  extern __shared__ __align__(16) uint8_t smem_raw[];
  Smem& sm = *reinterpret_cast<Smem*>(smem_raw);
  const int b = blockIdx.y;
  const int chunk = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = n_samples[b];
  const int m = n >= kFrameLen ? 1 + (n - kFrameLen) / kShift : 0;  // utils.py:457-486 (snip_edges)
  const int f_begin = chunk * kFramesPerCta;
  if (chunk == 0 && threadIdx.x == 0 && out_lens) out_lens[b] = m;

  // ---- stage tables + this CTA's samples ------------------------------------------------------
  {
    const float* src = reinterpret_cast<const float*>(&g_tables);
    float* dst = reinterpret_cast<float*>(&sm.t);
    for (int i = threadIdx.x; i < (int)(sizeof(Tables) / 4); i += blockDim.x) dst[i] = src[i];
    const long s0 = (long)f_begin * kShift;
    const WaveT* wrow = wave + (long)b * wave_ld;
    // fp32 waveforms: 16-byte vector loads (s0 is a multiple of 4 samples) whenever the row is 16-byte aligned
    bool vec = false;
    if (sizeof(WaveT) == 4) vec = ((reinterpret_cast<uintptr_t>(wrow) & 15) == 0);
    if (vec) {
      const float4* w4 = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(wrow) + s0);
      float4* d4 = reinterpret_cast<float4*>(sm.samples);
      for (int i = threadIdx.x; i < kSamplesPerCta / 4; i += blockDim.x) {
        const long s = s0 + 4 * i;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (s + 3 < n) {
          v = __ldg(w4 + i);
        } else {
          const float* wf = reinterpret_cast<const float*>(wrow);
          if (s < n) v.x = wf[s];
          if (s + 1 < n) v.y = wf[s + 1];
          if (s + 2 < n) v.z = wf[s + 2];
        }
        d4[i] = v;
      }
    } else {
      for (int i = threadIdx.x; i < kSamplesPerCta; i += blockDim.x) {
        const long s = s0 + i;
        sm.samples[i] = (s < n) ? load_sample<WaveT>(wrow + s) : 0.f;
      }
    }
  }
  __syncthreads();

  float* re = sm.re[warp];
  float* im = sm.im[warp];
  float* pw = sm.pw[warp];
  double local_sum = 0.0;

  for (int fi = warp; fi < kFramesPerCta; fi += kWarps) {
    const int f = f_begin + fi;
    if (f >= t_max) break;
    const long orow = ((long)b * t_max + f) * kBins;
    if (f >= m) {  // right padding: collate_frames pads with 0.0
      for (int j = lane; j < kBins; j += 32) {
        if (out_f32) ((float*)out)[orow + j] = 0.f;
        else ((bf16*)out)[orow + j] = f2bf(0.f);
      }
      continue;
    }
    const float* x = sm.samples + fi * kShift;
    // remove_dc_offset (kaldi.py:183-186)
    float s = 0.f;
    for (int j = lane; j < kFrameLen; j += 32) s += x[j];
    const float mean = warp_sum(s) / (float)kFrameLen;
    // pre-emphasis with replicate pad (kaldi.py:193-198), window (kaldi.py:201-204), zero pad to 512,
    // packed as a 256-point complex sequence z[n] = y[2n] + i*y[2n+1] in bit-reversed order.
    for (int j = lane; j < 512; j += 32) {
      float y = 0.f;
      if (j < kFrameLen) {
        const float v = x[j] - mean;
        const float pv = x[j > 0 ? j - 1 : 0] - mean;
        y = (v - 0.97f * pv) * sm.t.window[j];
      }
      const int nidx = __brev((unsigned)(j >> 1)) >> 24;
      if (j & 1) im[nidx] = y;
      else re[nidx] = y;
    }
    __syncwarp();
    // 256-point radix-2 DIT FFT in shared memory, one warp per frame.
#pragma unroll
    for (int st = 0; st < 8; ++st) {
      const int half = 1 << st;
      for (int bf = lane; bf < 128; bf += 32) {
        const int grp = bf >> st;
        const int pos = bf & (half - 1);
        const int i0 = (grp << (st + 1)) + pos;
        const int i1 = i0 + half;
        const int tk = pos << (7 - st);
        const float wr = sm.t.tw256[2 * tk], wi = sm.t.tw256[2 * tk + 1];
        const float ar = re[i1], ai = im[i1];
        const float tr = wr * ar - wi * ai;
        const float ti = wr * ai + wi * ar;
        const float ur = re[i0], ui = im[i0];
        re[i0] = ur + tr;
        im[i0] = ui + ti;
        re[i1] = ur - tr;
        im[i1] = ui - ti;
      }
      __syncwarp();
    }
    // split the packed transform into the real-input spectrum; power (kaldi.py:616-618).
    for (int k = lane; k < 256; k += 32) {
      const int kn = (256 - k) & 255;
      const float a = re[k], bb = im[k], c = re[kn], d = im[kn];
      const float er = 0.5f * (a + c), ei = 0.5f * (bb - d);
      const float orr = 0.5f * (bb + d), oi = -0.5f * (a - c);
      const float wr = sm.t.tw512[2 * k], wi = sm.t.tw512[2 * k + 1];
      const float xr = er + wr * orr - wi * oi;
      const float xi = ei + wr * oi + wi * orr;
      pw[k] = xr * xr + xi * xi;
    }
    __syncwarp();
    // mel filterbank (sparse triangles), log, CMVN (kaldi.py:621-633; global_cmvn.py:26-29)
    for (int j = lane; j < kBins; j += 32) {
      const int st0 = sm.t.mel_start[j], len = sm.t.mel_len[j];
      const float* w = sm.t.mel_w + sm.t.mel_off[j];
      float e = 0.f;
      for (int k = 0; k < len; ++k) e = fmaf(pw[st0 + k], w[k], e);
      float v = logf(fmaxf(e, 1.1920928955078125e-07f));
      if (cmvn_mean) v = (v - cmvn_mean[j]) / cmvn_std[j];
      local_sum += (double)v;
      if (out_f32) ((float*)out)[orow + j] = v;
      else ((bf16*)out)[orow + j] = f2bf(v);
    }
    __syncwarp();
  }

  // ---- SpecAugment needs the utterance mean (fill value): accumulate it; specaug_paint_kernel (same stream, next
  //      launch) paints the masks with every CTA of the grid in parallel ----------------------------------------
  const bool have_masks = (freq_masks && n_freq_masks > 0) || (time_masks && max_time_masks > 0);
  if (!have_masks || m == 0) return;  // uniform per CTA (depends on b only)
  local_sum = warp_sum_d(local_sum);
  if (lane == 0) sm.red[warp] = local_sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    double tot = 0.0;
    for (int w = 0; w < kWarps; ++w) tot += sm.red[w];
    atomicAdd(&ws_sum[b], tot);
  }
}

// Adaptive SpecAugment masks (espresso/data/feature_transforms/adaptive_specaugment.py:111-134): every CTA owns 32 frames
// of one utterance and overwrites the elements that fall inside ANY of the utterance's frequency / time masks with the
// utterance mean -- the features themselves are not read.  The last CTA of an utterance (ticket) clears the workspace.
constexpr int kMaxMasks = 64;
__global__ void __launch_bounds__(256)
specaug_paint_kernel(const int* __restrict__ n_samples, const int* __restrict__ freq_masks, int n_freq_masks,
                     const int* __restrict__ time_masks, int max_time_masks, void* __restrict__ out, int out_f32, int t_max,
                     double* __restrict__ ws_sum, unsigned int* __restrict__ ws_cnt) {
  esp_pdl();
  __shared__ int s_f0[kMaxMasks], s_f1[kMaxMasks], s_t0[kMaxMasks], s_t1[kMaxMasks];
  __shared__ int s_nf, s_nt;
  const int b = blockIdx.y;
  const int n = n_samples[b];
  const int m = n >= kFrameLen ? 1 + (n - kFrameLen) / kShift : 0;
  if (m == 0) return;
  if (threadIdx.x == 0) {
    int nf = 0, nt = 0;
    for (int i = 0; i < n_freq_masks && nf < kMaxMasks; ++i) {
      const int f0 = freq_masks[((long)b * n_freq_masks + i) * 2], fw = freq_masks[((long)b * n_freq_masks + i) * 2 + 1];
      if (fw > 0) { s_f0[nf] = f0; s_f1[nf] = min(f0 + fw, kBins); ++nf; }
    }
    for (int i = 0; i < max_time_masks && nt < kMaxMasks; ++i) {
      const int t0 = time_masks[((long)b * max_time_masks + i) * 2], tw = time_masks[((long)b * max_time_masks + i) * 2 + 1];
      if (tw > 0) { s_t0[nt] = t0; s_t1[nt] = min(t0 + tw, m); ++nt; }
    }
    s_nf = nf;
    s_nt = nt;
  }
  __syncthreads();
  const float fill = (float)(ws_sum[b] / ((double)m * (double)kBins));
  const bf16 fill_bf = f2bf(fill);
  const int f_begin = blockIdx.x * kFramesPerCta;
  // per-row / per-column flags first (64 + 80 small loops), then every element tests two flags instead of every mask
  __shared__ unsigned char s_trow[kFramesPerCta], s_fcol[kBins];
  for (int i = threadIdx.x; i < kFramesPerCta + kBins; i += blockDim.x) {
    if (i < kFramesPerCta) {
      const int t = f_begin + i;
      bool hit = false;
      for (int k = 0; k < s_nt; ++k) hit |= (t >= s_t0[k]) & (t < s_t1[k]);
      s_trow[i] = hit && t < m;
    } else {
      const int j = i - kFramesPerCta;
      bool hit = false;
      for (int k = 0; k < s_nf; ++k) hit |= (j >= s_f0[k]) & (j < s_f1[k]);
      s_fcol[j] = hit;
    }
  }
  __syncthreads();
  for (int e = threadIdx.x; e < kFramesPerCta * kBins; e += blockDim.x) {
    const int r = e / kBins, j = e % kBins;
    const int t = f_begin + r;
    if (t >= m) break;  // e is monotone in t
    if (s_trow[r] | s_fcol[j]) {
      const long o = ((long)b * t_max + t) * kBins + j;
      if (out_f32) ((float*)out)[o] = fill;
      else ((bf16*)out)[o] = fill_bf;
    }
  }
  __syncthreads();  // every thread has read ws_sum[b]
  if (threadIdx.x == 0) {  // leave the workspace clean for the next launch
    __threadfence();
    const unsigned ticket = atomicAdd(&ws_cnt[b], 1u);
    if (ticket == gridDim.x - 1) {
      ws_sum[b] = 0.0;
      ws_cnt[b] = 0u;
    }
  }
}

std::once_flag g_once;
cudaError_t g_table_err = cudaSuccess;

}  // namespace

extern "C" int64_t esp_frontend_workspace_bytes(int32_t B) { return (int64_t)B * 16; }

extern "C" int esp_frontend_fbank(const void* wave, int32_t wave_i16, int64_t wave_ld, const int32_t* n_samples,
                                  int32_t B, const float* cmvn_mean, const float* cmvn_std,
                                  const int32_t* freq_masks, int32_t n_freq_masks, const int32_t* time_masks,
                                  int32_t max_time_masks, void* out, int32_t out_f32, int32_t t_max,
                                  int32_t* out_lens, void* workspace, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(B >= 0 && t_max >= 0, "bad front-end shape");
  if (B == 0 || t_max == 0) return 0;
  ESP_CHECK(wave && n_samples && out && workspace, "null pointer passed to esp_frontend_fbank");
  ESP_CHECK((cmvn_mean == nullptr) == (cmvn_std == nullptr), "cmvn_mean and cmvn_std must be given together");
  std::call_once(g_once, [] {
    Tables* t = new Tables();
    build_tables(*t);
    g_table_err = cudaMemcpyToSymbol(g_tables, t, sizeof(Tables));
    delete t;
  });
  ESP_CUDA(g_table_err);
  double* ws_sum = (double*)workspace;
  unsigned int* ws_cnt = (unsigned int*)((char*)workspace + (size_t)B * 8);
  dim3 grid((t_max + kFramesPerCta - 1) / kFramesPerCta, B);
  const size_t smem = sizeof(Smem);
  if (wave_i16) {
    ESP_SMEM_OPTIN(frontend_kernel<int16_t>, smem);
    ESP_CUDA(esp_launch(frontend_kernel<int16_t>, grid, kWarps * 32, smem, st, (const int16_t*)wave, wave_ld, n_samples,
                        cmvn_mean, cmvn_std, freq_masks, n_freq_masks, time_masks, max_time_masks, out, out_f32, t_max, out_lens,
                        ws_sum, ws_cnt));
  } else {
    ESP_SMEM_OPTIN(frontend_kernel<float>, smem);
    ESP_CUDA(esp_launch(frontend_kernel<float>, grid, kWarps * 32, smem, st, (const float*)wave, wave_ld, n_samples, cmvn_mean,
                        cmvn_std, freq_masks, n_freq_masks, time_masks, max_time_masks, out, out_f32, t_max, out_lens, ws_sum,
                        ws_cnt));
  }
  const bool have_masks = (freq_masks && n_freq_masks > 0) || (time_masks && max_time_masks > 0);
  if (have_masks) {
    ESP_CHECK(n_freq_masks <= kMaxMasks && max_time_masks <= kMaxMasks, "at most %d masks of each kind per utterance", kMaxMasks);
    ESP_CUDA(esp_launch(specaug_paint_kernel, grid, 256, 0, st, n_samples, freq_masks, n_freq_masks, time_masks, max_time_masks,
                        out, out_f32, t_max, ws_sum, ws_cnt));
  }
  return 0;
}
