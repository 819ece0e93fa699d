// espresso_b200 -- adaptive SpecAugment on right-padded features [B, T, F]: time warp -> frequency masks -> time masks,
// with the host-drawn descriptors and the utterance mean BEFORE the warp as the fill value.
//
// Reference path being replaced (CPU, per utterance, in DataLoader workers):
//   espresso/data/feat_text_dataset.py:128-161 (feature transforms for Kaldi features and waveforms alike)
//   espresso/data/feature_transforms/adaptive_specaugment.py:77-136 (the warp is cv2.resize(..., INTER_LINEAR))
//
// The warp resizes the time axis of frames [0, w0) to w0 + w rows and of [w0, m) to m - w0 - w rows; the frequency axis
// keeps its size, so OpenCV's horizontal pass is a copy.  The OpenCV wheels hand a float32 INTER_LINEAR resize to Intel
// IPP, whose rule, for an output row r of a segment of S source rows resized to D rows, is:
//   f = (r + 0.5) * (1 / ((double)D / S)) - 0.5;  sy = floor(f);  fy = (float)(f - sy);
//   sy < 0 -> (sy, fy) = (0, 0);  sy >= S - 1 -> (sy, fy) = (S - 1, 0);
//   out[r] = fmaf(in[sy + 1] - in[sy], fy, in[sy])   (fy = 0 copies the row).
// oracle/specaug.py states the same rule and tests/golden/specaug_timewarp.npz pins it against cv2 itself.
//
// Two launches, both on a grid of (32-frame chunks, utterances):
//   specaug_warp_kernel writes every output element once: the warped (or copied) value for frames < m, zero beyond.
//     With masks it also stores the double sum of its chunk's INPUT frames in workspace[b][chunk].
//   specaug_mask_kernel adds an utterance's chunk sums in a fixed order (no atomics: the same bits on every run) and
//     overwrites its chunk's masked elements with the mean.
// Bytes: input read once (plus the rows a warp re-reads from cache), output written once, masked elements twice.
#include "common.cuh"
#include "espresso_b200.h"

namespace {

constexpr int kRows = 32;  // frames per CTA
constexpr int kThreads = 256;
constexpr int kMaxMasks = 64;

template <typename T>
__device__ __forceinline__ float ld_f(const T* p);
template <>
__device__ __forceinline__ float ld_f<float>(const float* p) { return __ldg(p); }
template <>
__device__ __forceinline__ float ld_f<bf16>(const bf16* p) { return bf2f(*p); }

template <typename T>
__device__ __forceinline__ void st_f(T* p, float v);
template <>
__device__ __forceinline__ void st_f<float>(float* p, float v) { *p = v; }
template <>
__device__ __forceinline__ void st_f<bf16>(bf16* p, float v) { *p = f2bf(v); }

// frames of utterance b: lens[b] clamped to [0, T]
__device__ __forceinline__ int frames_of(const int* lens, int b, int T) { return min(max(lens[b], 0), T); }

template <typename InT, typename OutT>
__global__ void __launch_bounds__(kThreads)
specaug_warp_kernel(const InT* __restrict__ x, OutT* __restrict__ y, int T, int F, const int* __restrict__ lens,
                    const int* __restrict__ time_warp, double* __restrict__ ws) {
  esp_pdl();
  __shared__ int s_src0[kRows], s_src1[kRows];
  __shared__ float s_fy[kRows];
  __shared__ double s_red[kThreads / 32];
  const int b = blockIdx.y;
  const int t_begin = blockIdx.x * kRows;
  const int rows = min(kRows, T - t_begin);
  const int m = frames_of(lens, b, T);
  if (threadIdx.x < rows) {
    const int t = t_begin + threadIdx.x;
    int s0 = t, s1 = t;
    float fy = 0.f;
    const int w0 = time_warp ? time_warp[2 * b] : 0, w = time_warp ? time_warp[2 * b + 1] : 0;
    // (w0, 0) is the identity; a pair that does not split the utterance into two non-empty parts is ignored
    if (w != 0 && w0 > 0 && w0 < m && w0 + w > 0 && w0 + w < m && t < m) {
      const bool upper = t < w0 + w;
      const int base = upper ? 0 : w0;
      const int S = upper ? w0 : m - w0;
      const int D = upper ? w0 + w : m - w0 - w;
      const int r = upper ? t : t - (w0 + w);
      const double scale = 1.0 / ((double)D / (double)S);
      const double f = (r + 0.5) * scale - 0.5;
      int sy = (int)floor(f);
      fy = (float)(f - sy);
      if (sy < 0) sy = 0, fy = 0.f;
      if (sy >= S - 1) sy = S - 1, fy = 0.f;
      s0 = base + sy;
      s1 = base + min(sy + 1, S - 1);
    }
    s_src0[threadIdx.x] = s0;
    s_src1[threadIdx.x] = s1;
    s_fy[threadIdx.x] = fy;
  }
  __syncthreads();
  const InT* xb = x + (long)b * T * F;
  OutT* yc = y + ((long)b * T + t_begin) * F;
  const int n = rows * F;
  for (int e = threadIdx.x; e < n; e += kThreads) {
    const int r = e / F, f = e - r * F;
    float v = 0.f;  // frames >= m: zero, as collate pads them
    if (t_begin + r < m) {
      v = ld_f(xb + (long)s_src0[r] * F + f);
      const float fy = s_fy[r];
      if (fy != 0.f) v = __fmaf_rn(__fsub_rn(ld_f(xb + (long)s_src1[r] * F + f), v), fy, v);
    }
    st_f(yc + e, v);
  }
  if (!ws) return;
  // the fill value is the mean of the input: this chunk's share, over its frames < m
  const InT* xc = xb + (long)t_begin * F;
  const int valid = max(0, min(rows, m - t_begin)) * F;
  double s = 0.0;
  for (int e = threadIdx.x; e < valid; e += kThreads) s += (double)ld_f(xc + e);
  s = warp_sum_d(s);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double tot = 0.0;
    for (int i = 0; i < kThreads / 32; ++i) tot += s_red[i];
    ws[(long)b * gridDim.x + blockIdx.x] = tot;
  }
}

template <typename OutT>
__global__ void __launch_bounds__(kThreads)
specaug_mask_kernel(OutT* __restrict__ y, int T, int F, const int* __restrict__ lens, const int* __restrict__ freq_masks,
                    int n_freq_masks, const int* __restrict__ time_masks, int max_time_masks,
                    const double* __restrict__ ws) {
  esp_pdl();
  __shared__ int s_f0[kMaxMasks], s_f1[kMaxMasks];
  __shared__ int s_nf;
  __shared__ unsigned char s_trow[kRows];
  __shared__ float s_fill;
  const int b = blockIdx.y;
  const int t_begin = blockIdx.x * kRows;
  const int m = frames_of(lens, b, T);
  if (t_begin >= m) return;  // uniform per CTA
  const int rows = min(kRows, m - t_begin);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 0) {  // the utterance sum, in the same order in every CTA and on every run
    double s = 0.0;
    for (int c = lane; c < (int)gridDim.x; c += 32) s += ws[(long)b * gridDim.x + c];
    s = warp_sum_d(s);
    if (lane == 0) s_fill = (float)(s / ((double)m * (double)F));
  } else if (warp == 1) {
    if (lane < rows) {
      const int t = t_begin + lane;
      bool hit = false;
      for (int i = 0; i < max_time_masks; ++i) {
        const int t0 = time_masks[((long)b * max_time_masks + i) * 2], tw = time_masks[((long)b * max_time_masks + i) * 2 + 1];
        hit |= tw > 0 && t >= t0 && t < t0 + tw;
      }
      s_trow[lane] = hit;
    }
  } else if (threadIdx.x == 64) {
    int nf = 0;
    for (int i = 0; i < n_freq_masks; ++i) {
      const int f0 = freq_masks[((long)b * n_freq_masks + i) * 2], fw = freq_masks[((long)b * n_freq_masks + i) * 2 + 1];
      if (fw > 0) s_f0[nf] = f0, s_f1[nf] = min(f0 + fw, F), ++nf;
    }
    s_nf = nf;
  }
  __syncthreads();
  const float fill = s_fill;
  OutT* yc = y + ((long)b * T + t_begin) * F;
  for (int e = threadIdx.x; e < rows * F; e += kThreads) {
    const int r = e / F, f = e - r * F;
    bool hit = s_trow[r];
    for (int k = 0; k < s_nf; ++k) hit |= f >= s_f0[k] && f < s_f1[k];
    if (hit) st_f(yc + e, fill);
  }
}

template <typename InT, typename OutT>
cudaError_t launch_warp(dim3 grid, cudaStream_t st, const void* in, void* out, int T, int F, const int* lens,
                        const int* time_warp, double* ws) {
  return esp_launch(specaug_warp_kernel<InT, OutT>, grid, kThreads, 0, st, (const InT*)in, (OutT*)out, T, F, lens,
                    time_warp, ws);
}

}  // namespace

extern "C" int64_t esp_specaug_workspace_bytes(int32_t B, int32_t T) {
  return (int64_t)B * ((T + kRows - 1) / kRows) * (int64_t)sizeof(double);
}

extern "C" int esp_specaug_features(const void* in, int32_t in_f32, void* out, int32_t out_f32, int32_t B, int32_t T,
                                    int32_t F, const int32_t* lens, const int32_t* time_warp, const int32_t* freq_masks,
                                    int32_t n_freq_masks, const int32_t* time_masks, int32_t max_time_masks,
                                    void* workspace, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(B >= 0 && T >= 0 && F >= 1, "bad SpecAugment shape B=%d T=%d F=%d", B, T, F);
  ESP_CHECK(n_freq_masks >= 0 && max_time_masks >= 0, "negative mask count");
  if (B == 0 || T == 0) return 0;
  ESP_CHECK(in && out && lens, "null pointer passed to esp_specaug_features");
  ESP_CHECK(in != out, "esp_specaug_features writes out of place: in and out must not alias");
  const bool have_masks = (freq_masks && n_freq_masks > 0) || (time_masks && max_time_masks > 0);
  if (have_masks) {
    ESP_CHECK(workspace, "esp_specaug_features needs a workspace of esp_specaug_workspace_bytes(B, T) with masks");
    ESP_CHECK(n_freq_masks <= kMaxMasks && max_time_masks <= kMaxMasks, "at most %d masks of each kind per utterance",
              kMaxMasks);
  }
  if (!freq_masks) n_freq_masks = 0;
  if (!time_masks) max_time_masks = 0;
  double* ws = have_masks ? (double*)workspace : nullptr;
  const dim3 grid((T + kRows - 1) / kRows, B);
  auto warp = in_f32 ? (out_f32 ? launch_warp<float, float> : launch_warp<float, bf16>)
                     : (out_f32 ? launch_warp<bf16, float> : launch_warp<bf16, bf16>);
  ESP_CUDA(warp(grid, st, in, out, T, F, lens, time_warp, ws));
  if (have_masks) {
    if (out_f32)
      ESP_CUDA(esp_launch(specaug_mask_kernel<float>, grid, kThreads, 0, st, (float*)out, T, F, lens, freq_masks,
                          n_freq_masks, time_masks, max_time_masks, (const double*)ws));
    else
      ESP_CUDA(esp_launch(specaug_mask_kernel<bf16>, grid, kThreads, 0, st, (bf16*)out, T, F, lens, freq_masks,
                          n_freq_masks, time_masks, max_time_masks, (const double*)ws));
  }
  return 0;
}
