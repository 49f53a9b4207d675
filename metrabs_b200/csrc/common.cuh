// Shared helpers for the metrabs_b200 CUDA sources (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <map>
#include <mutex>
#include <type_traits>
#include <utility>

namespace mtb {

enum Act : int { ACT_NONE = 0, ACT_SILU = 1, ACT_RELU = 2, ACT_HSWISH = 3, ACT_SIGMOID = 4, ACT_HSIGMOID = 5 };

template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(std::forward<Args>(args))...);
}

// streaming multiprocessors of the current device (grid sizes of the persistent / grid-stride kernels)
inline int num_sms() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
    n = 132;
  return n;
}

// Raises `kernel`'s dynamic shared-memory limit on the current device to `bytes`, unless an earlier call already raised it
// that far there.  The limit belongs to the device's context: a process with handles on two devices needs it on both.
inline cudaError_t smem_opt_in(const void* kernel, int bytes) {
  static std::mutex mu;
  static std::map<std::pair<int, const void*>, int> raised;  // (device, kernel) -> limit set
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lock(mu);
  int& limit = raised[{dev, kernel}];
  if (limit >= bytes) return cudaSuccess;
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess) limit = bytes;
  return e;
}

// launch_k for kernels that may take more than 48 KB of dynamic shared memory; nullptr on success, else the CUDA error
template <typename... KArgs, typename... Args>
inline const char* launch_smem(void (*kernel)(KArgs...), dim3 grid, dim3 block, int smem, cudaStream_t st, Args&&... args) {
  cudaError_t e = smem_opt_in((const void*)kernel, smem);
  if (e == cudaSuccess) {
    launch_k(kernel, grid, block, (size_t)smem, st, std::forward<Args>(args)...);
    e = cudaGetLastError();
  }
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

// Calls f(std::integral_constant<int, V>{}) for the V of Vs equal to v and returns its result, or `none` when v is not listed.
// Each call site lists the values it launches with, so only those kernel instances are compiled.
template <int... Vs, typename R, typename F>
inline R with_const(int v, R none, F&& f) {
  R r = none;
  (void)((v == Vs && (r = f(std::integral_constant<int, Vs>{}), true)) || ...);
  return r;
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + __expf(-x)); }

__device__ __forceinline__ float apply_act(float x, int act) {
  switch (act) {
    case ACT_SILU: return x * sigmoidf_(x);
    case ACT_RELU: return fmaxf(x, 0.0f);
    case ACT_HSWISH: return x * fminf(fmaxf(x + 3.0f, 0.0f), 6.0f) * (1.0f / 6.0f);
    case ACT_SIGMOID: return sigmoidf_(x);
    case ACT_HSIGMOID: return fminf(fmaxf(x + 3.0f, 0.0f), 6.0f) * (1.0f / 6.0f);
    default: return x;
  }
}

// compile-time activation (exact expf forms: used by the fp32 parity kernels).  A runtime switch inside per-element code
// gets if-converted into every branch, so kernels dispatch ONCE per thread with act_dispatch and run a templated body.
template <int ACT>
__device__ __forceinline__ float act_t(float x) {
  if constexpr (ACT == ACT_SILU) return x * sigmoidf_(x);
  else if constexpr (ACT == ACT_RELU) return fmaxf(x, 0.0f);
  else if constexpr (ACT == ACT_HSWISH) return x * fminf(fmaxf(x + 3.0f, 0.0f), 6.0f) * (1.0f / 6.0f);
  else if constexpr (ACT == ACT_SIGMOID) return sigmoidf_(x);
  else if constexpr (ACT == ACT_HSIGMOID) return fminf(fmaxf(x + 3.0f, 0.0f), 6.0f) * (1.0f / 6.0f);
  else return x;
}
template <int V>
struct IntTag {
  static constexpr int value = V;
};
template <typename F>
__device__ __forceinline__ void act_dispatch(int act, F&& f) {
  switch (act) {
    case ACT_SILU: f(IntTag<ACT_SILU>{}); break;
    case ACT_RELU: f(IntTag<ACT_RELU>{}); break;
    case ACT_HSWISH: f(IntTag<ACT_HSWISH>{}); break;
    case ACT_SIGMOID: f(IntTag<ACT_SIGMOID>{}); break;
    case ACT_HSIGMOID: f(IntTag<ACT_HSIGMOID>{}); break;
    default: f(IntTag<ACT_NONE>{}); break;
  }
}

// ---- 4-wide vector load/store for fp32, bf16 and fp16 activation storage -------------------------------------
template <typename T>
__device__ __forceinline__ float4 load4(const T* p);
template <>
__device__ __forceinline__ float4 load4<float>(const float* p) {
  return *reinterpret_cast<const float4*>(p);
}
template <>
__device__ __forceinline__ float4 load4<__nv_bfloat16>(const __nv_bfloat16* p) {
  uint2 u = *reinterpret_cast<const uint2*>(p);
  __nv_bfloat162 a = *reinterpret_cast<__nv_bfloat162*>(&u.x);
  __nv_bfloat162 b = *reinterpret_cast<__nv_bfloat162*>(&u.y);
  float2 fa = __bfloat1622float2(a), fb = __bfloat1622float2(b);
  return make_float4(fa.x, fa.y, fb.x, fb.y);
}
template <>
__device__ __forceinline__ float4 load4<__half>(const __half* p) {
  uint2 u = *reinterpret_cast<const uint2*>(p);
  float2 fa = __half22float2(*reinterpret_cast<__half2*>(&u.x)), fb = __half22float2(*reinterpret_cast<__half2*>(&u.y));
  return make_float4(fa.x, fa.y, fb.x, fb.y);
}
template <typename T>
__device__ __forceinline__ void store4(T* p, float4 v);
template <>
__device__ __forceinline__ void store4<float>(float* p, float4 v) {
  *reinterpret_cast<float4*>(p) = v;
}
template <>
__device__ __forceinline__ void store4<__half>(__half* p, float4 v) {
  __half2 a = __floats2half2_rn(v.x, v.y);
  __half2 b = __floats2half2_rn(v.z, v.w);
  uint2 u;
  u.x = *reinterpret_cast<uint32_t*>(&a);
  u.y = *reinterpret_cast<uint32_t*>(&b);
  *reinterpret_cast<uint2*>(p) = u;
}
template <>
__device__ __forceinline__ void store4<__nv_bfloat16>(__nv_bfloat16* p, float4 v) {
  __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y);
  __nv_bfloat162 b = __floats2bfloat162_rn(v.z, v.w);
  uint2 u;
  u.x = *reinterpret_cast<uint32_t*>(&a);
  u.y = *reinterpret_cast<uint32_t*>(&b);
  *reinterpret_cast<uint2*>(p) = u;
}
template <typename T>
__device__ __forceinline__ float load1(const T* p);
template <>
__device__ __forceinline__ float load1<float>(const float* p) { return *p; }
template <>
__device__ __forceinline__ float load1<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }
template <>
__device__ __forceinline__ float load1<__half>(const __half* p) { return __half2float(*p); }
template <typename T>
__device__ __forceinline__ void store1(T* p, float v);
template <>
__device__ __forceinline__ void store1<float>(float* p, float v) { *p = v; }
template <>
__device__ __forceinline__ void store1<__nv_bfloat16>(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }
template <>
__device__ __forceinline__ void store1<__half>(__half* p, float v) { *p = __float2half_rn(v); }

// ---- 16-bit activation storage (bf16 or fp16): packed pairs, rounded to nearest even (fp16 overflow gives inf) -----------
template <typename T>
struct Pair16;
template <>
struct Pair16<__nv_bfloat16> {
  typedef __nv_bfloat162 type;
  static __device__ __forceinline__ type pack(float a, float b) { return __floats2bfloat162_rn(a, b); }
  static __device__ __forceinline__ float2 unpack(type v) { return __bfloat1622float2(v); }
};
template <>
struct Pair16<__half> {
  typedef __half2 type;
  static __device__ __forceinline__ type pack(float a, float b) { return __floats2half2_rn(a, b); }
  static __device__ __forceinline__ float2 unpack(type v) { return __half22float2(v); }
};
template <typename T>
constexpr bool is_f16 = std::is_same<T, __half>::value;

// SiLU of the fp16 kernels: x * rcp(1 + 2^(-x log2 e)) with ex2.approx and rcp.approx, ~2 fp32 ulps of error.  Cost: two MUFU
// ops and three FP32 ops per element, against one MUFU op and two FP32 ops for the bf16 kernels' h + h * tanh.approx(h)
// (h = x / 2), whose ~2^-11 relative error is below a bf16 ulp but a whole fp16 ulp (and far more relative to the small
// outputs of negative x).  The .ftz forms skip the denormal fix-ups __expf / __fdividef add: a flushed 2^(-x log2 e) (x > 87)
// gives x, a flushed reciprocal (x < -87) gives -0, both what the exact value rounds to in fp16.
__device__ __forceinline__ float silu_f16out(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  return x * r;
}

// fp32 pairs: kernels written against two-wide arithmetic (f2_fma / f2_mul / f2_add).  Each half is the scalar IEEE
// fma / mul / add with round-to-nearest (__fmaf_rn etc. are never contracted or reassociated), so a kernel using them is
// bit-identical to its scalar formulation.
typedef float2 f32x2;
__device__ __forceinline__ f32x2 f2_pack(float lo, float hi) { return make_float2(lo, hi); }
__device__ __forceinline__ void f2_unpack(f32x2 v, float& lo, float& hi) { lo = v.x; hi = v.y; }
__device__ __forceinline__ f32x2 f2_fma(f32x2 a, f32x2 b, f32x2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ f32x2 f2_mul(f32x2 a, f32x2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ f32x2 f2_add(f32x2 a, f32x2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace mtb
