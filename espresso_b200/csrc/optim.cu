// espresso_b200 -- optimizer step of the data-parallel update, on flat buffers.
//
// Replaces, for `--bf16` training (fairseq/trainer.py:903-953):
//   FP16Optimizer._sync_fp16_grads_to_fp32 / multiply_grads / clip_grad_norm / step / _sync_fp32_params_to_fp16
//     fairseq/optim/fp16_optimizer.py:109-168,  fairseq/utils.py:347-397 (clip_grad_norm_)
//   Adam.step  fairseq/optim/adam.py:150-239 (decoupled weight decay, bias correction, eps outside sqrt)
// Gradients live in ONE flat fp32 buffer (the wgrad GEMMs and reduction kernels write into it directly,
// and the NCCL all-reduce runs on it in place -- no flatten/unflatten copies as in
// fairseq/distributed/legacy_distributed_data_parallel.py:127-163).  The global sample_size arrives in the
// buffer's tail through the same all-reduce, so the normalisation 1/sample_size (trainer.py:918-923) and
// the clip coefficient are computed on the device: the whole update needs no host synchronisation.
#include "common.cuh"
#include "espresso_b200.h"

namespace {

__global__ void __launch_bounds__(256)
sumsq_kernel(const float* __restrict__ g, long n, float* __restrict__ out) {
  esp_pdl();
  float s = 0.f;
  const long n4 = n >> 2;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
    const float4 v = g4[i];
    s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  for (long i = (n4 << 2) + (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
    s += g[i] * g[i];
  __shared__ float red[8];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float r = threadIdx.x < 8 ? red[threadIdx.x] : 0.f;
    r = warp_sum(r);
    if (threadIdx.x == 0) atomicAdd(out, r);
  }
}

// one fused pass: normalise + clip + Adam + bf16 write-back
__global__ void __launch_bounds__(256)
adam_kernel(float* __restrict__ p32, float* __restrict__ m, float* __restrict__ v, const float* __restrict__ g,
            bf16* __restrict__ p16, long n, float lr, float beta1, float beta2, float eps, float weight_decay,
            float step, const float* __restrict__ sumsq, const float* __restrict__ denom_ptr,
            float denom_const, float clip_norm, float* __restrict__ gnorm_out, const float* __restrict__ hyper) {
  esp_pdl();
  if (hyper) {  // schedule values live in device memory so a captured graph replays with fresh ones
    lr = hyper[0];
    step = hyper[1];
  }
  const float bias1 = 1.f - powf(beta1, step);
  const float bias2 = 1.f - powf(beta2, step);
  const float denom = denom_ptr ? *denom_ptr : denom_const;
  const float gscale = denom > 0.f ? 1.f / denom : 0.f;                 // multiply_grads(world/sample_size) after the
                                                                        // pre-divided sum == 1/sum(sample_size)
  const float gnorm = sqrtf(*sumsq) * gscale;                           // utils.clip_grad_norm_ on the scaled grads
  float coef = 1.f;
  if (clip_norm > 0.f) coef = fminf(1.f, clip_norm / (gnorm + 1e-6f));  // fairseq/utils.py:392-395
  if (gnorm_out && blockIdx.x == 0 && threadIdx.x == 0) *gnorm_out = gnorm;
  const float gs = gscale * coef;
  const float step_size = lr * sqrtf(bias2) / bias1;                    // adam.py:213-216
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const float gi = g[i] * gs;
    float p = p32[i];
    const float mi = beta1 * m[i] + (1.f - beta1) * gi;
    const float vi = beta2 * v[i] + (1.f - beta2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    if (weight_decay != 0.f) p -= weight_decay * lr * p;                 // adam.py:218-221
    p -= step_size * mi / (sqrtf(vi) + eps);
    p32[i] = p;
    p16[i] = f2bf(p);
  }
}

__global__ void __launch_bounds__(256)
cast_f32_to_bf16_kernel(const float* __restrict__ x, long n, bf16* __restrict__ y) {
  esp_pdl();
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) y[i] = f2bf(x[i]);
}
__global__ void __launch_bounds__(256)
cast_bf16_to_f32_kernel(const bf16* __restrict__ x, long n, float* __restrict__ y) {
  esp_pdl();
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) y[i] = bf2f(x[i]);
}

}  // namespace

extern "C" int esp_sumsq_f32(const float* g, int64_t n, float* out, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(((uintptr_t)g & 15) == 0, "sumsq input must be 16-byte aligned");
  ESP_CUDA(cudaMemsetAsync(out, 0, sizeof(float), st));
  if (n > 0) {
    ESP_CUDA(esp_launch(sumsq_kernel, grid_for(n / 4 + 1, 1024), 256, 0, st, g, n, out));
  }
  return 0;
}

extern "C" int esp_adam_step(float* p32, float* m, float* v, const float* g, void* p16, int64_t n, float lr, float beta1,
                             float beta2, float eps, float weight_decay, int32_t step, const float* sumsq,
                             const float* denom_dev, float denom_const, float clip_norm, float* gnorm_out,
                             const float* hyper_dev, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ESP_CHECK(step >= 1 || hyper_dev != nullptr, "Adam step count must start at 1");
  ESP_CHECK(sumsq != nullptr, "Adam needs the squared gradient norm (esp_sumsq_f32)");
  if (n == 0) return 0;
  ESP_CUDA(esp_launch(adam_kernel, grid_for(n, 1024), 256, 0, st, p32, m, v, g, (bf16*)p16, n, lr, beta1, beta2, eps,
                      weight_decay, (float)step, sumsq, denom_dev, denom_const, clip_norm, gnorm_out, hyper_dev));
  return 0;
}

extern "C" int esp_cast_f32_bf16(const float* x, int64_t n, void* y, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) return 0;
  ESP_CUDA(esp_launch(cast_f32_to_bf16_kernel, grid_for(n, 1024), 256, 0, st, x, n, (bf16*)y));
  return 0;
}
extern "C" int esp_cast_bf16_f32(const void* x, int64_t n, float* y, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) return 0;
  ESP_CUDA(esp_launch(cast_bf16_to_f32_kernel, grid_for(n, 1024), 256, 0, st, (const bf16*)x, n, y));
  return 0;
}
