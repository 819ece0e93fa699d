// espresso_b200 -- shared device/host helpers for the sm_90a kernels.
#pragma once
#include <utility>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>

typedef __nv_bfloat16 bf16;

// ---- error plumbing for the C ABI (no exceptions cross the boundary) -------------------------
void esp_set_error(const char* fmt, ...);
#define ESP_CHECK(cond, ...)                 \
  do {                                       \
    if (!(cond)) {                           \
      esp_set_error(__VA_ARGS__);            \
      return -1;                             \
    }                                        \
  } while (0)
#define ESP_CUDA(expr)                                                              \
  do {                                                                              \
    cudaError_t _e = (expr);                                                        \
    if (_e != cudaSuccess) {                                                        \
      esp_set_error("%s:%d CUDA error: %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
      return -2;                                                                    \
    }                                                                               \
  } while (0)

// Raises `kernel`'s dynamic shared-memory limit to `bytes` (needed above 48 KB).  The attribute is per function and per
// process, so each call site keeps the largest size it has set and calls the runtime only when that grows.
#define ESP_SMEM_OPTIN(kernel, bytes)                                                                \
  do {                                                                                               \
    static size_t _optin = 0;                                                                        \
    const size_t _b = (bytes);                                                                       \
    if (_b > _optin) {                                                                               \
      ESP_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)_b));  \
      _optin = _b;                                                                                   \
    }                                                                                                \
  } while (0)

int esp_num_sms();
void esp_count_launch(int n);  // capi.cu: the counter behind esp_launch_count()

// 1-D grid for a grid-stride loop: one CTA per `per_block` items, at most `max_waves` CTAs per SM
inline int grid_for(long work_items, int per_block, int max_waves = 8) {
  long g = (work_items + per_block - 1) / per_block;
  long cap = (long)esp_num_sms() * max_waves;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

// workspace carving: every sub-buffer starts on a 256-byte boundary
inline long align256(long x) { return (x + 255) / 256 * 256; }

// ---- small device helpers --------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// max / sum over a block of NT threads (blockDim.x == NT); `red` holds NT/32 floats.  Every thread gets the result, and
// the trailing barrier lets the caller reuse `red` straight away.
template <int NT>
__device__ __forceinline__ float block_max(float v, float* red) {
  v = warp_max(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = (threadIdx.x & 31) < (NT >> 5) ? red[threadIdx.x & 31] : -INFINITY;
  r = warp_max(r);
  __syncthreads();
  return r;
}
template <int NT>
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = (threadIdx.x & 31) < (NT >> 5) ? red[threadIdx.x & 31] : 0.f;
  r = warp_sum(r);
  __syncthreads();
  return r;
}

__device__ __forceinline__ float bf2f(bf16 v) { return __bfloat162float(v); }
__device__ __forceinline__ bf16 f2bf(float v) { return __float2bfloat16_rn(v); }

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ void unpack_bf16x2(uint32_t p, float& lo, float& hi) {
  __nv_bfloat162 t = *reinterpret_cast<__nv_bfloat162*>(&p);
  lo = __low2float(t);
  hi = __high2float(t);
}

// ex2.approx + rcp.approx: ~2 ulp, far below the bf16 rounding of every consumer (1 + inf -> rcp = 0 is the right limit)
__device__ __forceinline__ float sigmoidf_(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }
__device__ __forceinline__ float siluf_(float x) { return x * sigmoidf_(x); }
// d/dx [x*sigmoid(x)]
__device__ __forceinline__ float silu_gradf_(float x) {
  float s = sigmoidf_(x);
  return s * (1.f + x * (1.f - s));
}

// ---- kernel launches and programmatic dependent launch (PDL) ------------------------------------------
// Every hot-path kernel starts with esp_pdl(): it lets the NEXT kernel of the stream be scheduled as soon as this
// grid's CTAs have all started (its CTAs then sit in griddepcontrol.wait), and blocks this kernel until every
// kernel before it has completed and flushed.  With esp_launch() (below) setting the programmatic-serialisation
// attribute, launch latency and kernel prologues overlap the tail of the previous kernel -- in eager streams and in
// captured CUDA graphs alike.  Without the attribute both instructions are no-ops.
#ifdef __CUDACC__
__device__ __forceinline__ void esp_pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void esp_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void esp_pdl() {
  esp_pdl_trigger();
  esp_pdl_wait();
}

bool esp_pdl_enabled();  // capi.cu: ESP_PDL=0 in the environment disables the launch attribute

// Every kernel is launched here, and every call site is ESP_CUDA(esp_launch...(...)).  The launch leaves no error
// pending (cudaGetLastError), is counted for esp_launch_count() only when it was accepted, and returns the error.
// `cluster_x` > 1 launches thread-block clusters of that many CTAs along x (grid.x must be a multiple of it); `pdl`
// sets the programmatic-serialisation attribute.
template <typename... KArgs, typename... Args>
inline cudaError_t esp_launch_ex(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                 int cluster_x, bool pdl, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (cluster_x > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster_x;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  if (pdl && esp_pdl_enabled()) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
  const cudaError_t pending = cudaGetLastError();
  if (e == cudaSuccess) e = pending;
  if (e == cudaSuccess) esp_count_launch(1);
  return e;
}
// kernels that begin with esp_pdl()
template <typename... KArgs, typename... Args>
inline cudaError_t esp_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  return esp_launch_ex(kernel, grid, block, smem, st, 1, true, std::forward<Args>(args)...);
}
template <typename... KArgs, typename... Args>
inline cudaError_t esp_launch_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                      int cluster_x, Args&&... args) {
  return esp_launch_ex(kernel, grid, block, smem, st, cluster_x, true, std::forward<Args>(args)...);
}
// kernels without esp_pdl(): no launch attribute
template <typename... KArgs, typename... Args>
inline cudaError_t esp_launch_plain(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                    Args&&... args) {
  return esp_launch_ex(kernel, grid, block, smem, st, 1, false, std::forward<Args>(args)...);
}
#endif

#ifdef __CUDACC__
// fire-and-forget fp32 vector reduction at L2 (one request for 4 consecutive floats; p must be 16-byte aligned)
__device__ __forceinline__ void red_add_v4(float* p, float a, float b, float c, float d) {
  asm volatile("red.global.v4.f32.add [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
#endif

// ---- counter-based RNG for dropout ---------------------------------------------------------------
// Stateless: the backward pass regenerates the identical mask from (seed, logical element index), so
// dropout masks are never stored in HBM.  One 64-bit hash (splitmix64 finaliser keyed by the seed) yields
// FOUR 16-bit lanes = the keep decisions of elements 4g..4g+3, so a kernel that walks 4 (or 32)
// consecutive elements pays one hash per 4 elements.  p is quantised to 1/65536 and the rescale uses the
// quantised keep probability, so E[dropout(x)] = x exactly.
__host__ __device__ __forceinline__ unsigned long long esp_hash_u64(unsigned long long seed, unsigned long long g) {
  unsigned long long z = g + seed * 0x9E3779B97F4A7C15ull + 0xD1B54A32D192ED03ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
// keep-decision of element idx: its 16-bit lane of the group hash must be >= thresh (= round(p * 65536))
__host__ __device__ __forceinline__ bool esp_dropout_keep(unsigned long long seed, unsigned long long idx, uint32_t thresh) {
  const unsigned long long h = esp_hash_u64(seed, idx >> 2);
  return (uint32_t)((h >> (16 * (idx & 3))) & 0xFFFFull) >= thresh;
}
#ifdef __CUDACC__
// keep decisions of 8 consecutive elements whose first logical index idx0 is a multiple of 8: two hashes, not eight
__device__ __forceinline__ void esp_keep8(unsigned long long seed, unsigned long long idx0, uint32_t thresh, bool (&k)[8]) {
  const unsigned long long h0 = esp_hash_u64(seed, idx0 >> 2), h1 = esp_hash_u64(seed, (idx0 >> 2) + 1);
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    k[t] = ((uint32_t)(h0 >> (16 * t)) & 0xFFFFu) >= thresh;
    k[4 + t] = ((uint32_t)(h1 >> (16 * t)) & 0xFFFFu) >= thresh;
  }
}
// i = q * n + r for a grid-stride index: 32-bit division whenever the index fits (64-bit division is ~100 instructions)
__device__ __forceinline__ void esp_divmod(long i, unsigned n, long& q, unsigned& r) {
  if ((unsigned long long)i >> 32) {
    q = i / (long)n;
    r = (unsigned)(i - q * (long)n);
  } else {
    const unsigned iq = (unsigned)i / n;
    q = iq;
    r = (unsigned)i - iq * n;
  }
}
#endif
static inline uint32_t esp_dropout_thresh(float p) {
  double t = (double)p * 65536.0 + 0.5;
  if (t < 0) t = 0;
  if (t > 65535.0) t = 65535.0;
  return (uint32_t)t;
}
// 1 / (quantised keep probability)
static inline float esp_dropout_scale(float p) {
  if (!(p > 0.f)) return 1.f;
  return (float)(65536.0 / (65536.0 - (double)esp_dropout_thresh(p)));
}
