// CUDA-core (fp32 FMA) convolution kernels over NHWC activations: the fp32 parity mode of the backbone
// (MTB_PRECISION_FP32) and the fallback for layers that are not GEMM-shaped (stem with Cin=3, depthwise).
// Reference semantics: explicit zero pad then VALID conv (backbones/efficientnet.py:1127-1161), BN folded into
// weight+bias at load time, activation and residual add fused in the epilogue.
#pragma once
#include "common.cuh"

namespace mtb {

// The kernels take it as `const __grid_constant__ ConvParams p` and read it in place: their lambdas take p by reference,
// and without the qualifier ptxas's register allocation follows the struct's size.
struct ConvParams {
  const void* in;        // [B,Hin,Win,Cin]
  const void* res;       // optional residual [B,Hout,Wout,Cout]
  void* out;             // [B,Hout,Wout,Cout]
  const float* w;        // [R*S*Cin][Cout]  (k = (r*S+s)*Cin + c)
  const float* bias;     // [Cout]
  const float* a_scale;  // optional per-(b,cin) multiplier of the input (squeeze-excitation), [B][Cin]
  int res_first = 0;              // 1: add the residual BEFORE the activation (ResNet), 0: after (EfficientNet)
  int ksplit = 1;                 // > 1: blockIdx.z owns a K slice and writes its raw partial sums to out + z*M*Cout (fp32)
  int a_splits = 1;               // > 1: the input is a stack of partial slices (the pooled means the depthwise kernels
  size_t a_split_stride = 0;      //   leave for SE fc1); they are summed on load in a fixed order: deterministic
  int B, Hin, Win, Cin, Hout, Wout, Cout, R, S, stride, dil, pad_t, pad_l, act;
};

// ----------------------------------------------------------------------------------------------------------
// implicit-GEMM conv: M = B*Hout*Wout pixels, N = Cout, K = R*S*Cin.  Requires Cin % 4 == 0, Cout % 4 == 0.
// ----------------------------------------------------------------------------------------------------------
template <int BM, int BN, int TM, int TN, typename TIn, typename TOut>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
conv_igemm_kernel(const __grid_constant__ ConvParams p) {
  constexpr int BK = 16;
  constexpr int NT = (BM / TM) * (BN / TN);
  constexpr int A_LD = (BM * BK / 4) / NT;  // float4 loads of A per thread per tile
  constexpr int B_LD = (BK * BN / 4) / NT;
  static_assert(A_LD >= 1 && B_LD >= 1, "tile too small for the thread count");
  constexpr int GM = TM / 4, GN = TN / 4;            // 4-wide groups per thread
  constexpr int GSM = (BM / TM) * 4, GSN = (BN / TN) * 4;  // group strides

  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];

  const int tid = threadIdx.x;
  const int M = p.B * p.Hout * p.Wout;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const TIn* __restrict__ in = reinterpret_cast<const TIn*>(p.in);

  // per-thread A rows
  int a_row[A_LD], a_kq[A_LD], a_ih0[A_LD], a_iw0[A_LD], a_b[A_LD];
  bool a_ok[A_LD];
#pragma unroll
  for (int i = 0; i < A_LD; ++i) {
    int idx = tid + i * NT;
    a_row[i] = idx >> 2;
    a_kq[i] = idx & 3;
    int m = m0 + a_row[i];
    a_ok[i] = m < M;
    int mm = a_ok[i] ? m : 0;
    int b = mm / (p.Hout * p.Wout);
    int r = mm - b * p.Hout * p.Wout;
    int oh = r / p.Wout, ow = r - oh * p.Wout;
    a_b[i] = b;
    a_ih0[i] = oh * p.stride - p.pad_t;
    a_iw0[i] = ow * p.stride - p.pad_l;
  }
  int b_krow[B_LD], b_n[B_LD];
#pragma unroll
  for (int i = 0; i < B_LD; ++i) {
    int idx = tid + i * NT;
    b_krow[i] = idx / (BN / 4);
    b_n[i] = (idx % (BN / 4)) * 4;
  }

  const int cchunks = (p.Cin + BK - 1) / BK;
  const int T_all = p.R * p.S * cchunks;
  const int t_begin = (int)((long long)T_all * blockIdx.z / p.ksplit);
  const int T = (int)((long long)T_all * (blockIdx.z + 1) / p.ksplit);

  float4 ra[A_LD], rb[B_LD];
  auto load_tile = [&](int t) {
    int tap = t / cchunks;
    int c0 = (t - tap * cchunks) * BK;
    int r = tap / p.S, s = tap - r * p.S;
#pragma unroll
    for (int i = 0; i < A_LD; ++i) {
      int ih = a_ih0[i] + r * p.dil, iw = a_iw0[i] + s * p.dil;
      int c = c0 + a_kq[i] * 4;
      bool ok = a_ok[i] && ih >= 0 && ih < p.Hin && iw >= 0 && iw < p.Win && c < p.Cin;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (ok) {
        const TIn* ap = in + ((size_t)(a_b[i] * p.Hin + ih) * p.Win + iw) * p.Cin + c;
        v = load4<TIn>(ap);
#pragma unroll 1  // at most 8 slices; unrolled, the 64x64 fp32 instance (SE fc1) spills
        for (int z = 1; z < p.a_splits; ++z) {
          float4 u = load4<TIn>(ap + (size_t)z * p.a_split_stride);
          v.x += u.x; v.y += u.y; v.z += u.z; v.w += u.w;
        }
        if (p.a_scale) {
          float4 sc = *reinterpret_cast<const float4*>(p.a_scale + (size_t)a_b[i] * p.Cin + c);
          v.x *= sc.x; v.y *= sc.y; v.z *= sc.z; v.w *= sc.w;
        }
      }
      ra[i] = v;
    }
#pragma unroll
    for (int i = 0; i < B_LD; ++i) {
      int c = c0 + b_krow[i];
      int n = n0 + b_n[i];
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (c < p.Cin && n < p.Cout) v = *reinterpret_cast<const float4*>(p.w + (size_t)(tap * p.Cin + c) * p.Cout + n);
      rb[i] = v;
    }
  };
  auto store_tile = [&]() {
#pragma unroll
    for (int i = 0; i < A_LD; ++i) {
      int k = a_kq[i] * 4;
      As[k + 0][a_row[i]] = ra[i].x;
      As[k + 1][a_row[i]] = ra[i].y;
      As[k + 2][a_row[i]] = ra[i].z;
      As[k + 3][a_row[i]] = ra[i].w;
    }
#pragma unroll
    for (int i = 0; i < B_LD; ++i) *reinterpret_cast<float4*>(&Bs[b_krow[i]][b_n[i]]) = rb[i];
  };

  const int ty = tid / (BN / TN), tx = tid % (BN / TN);
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  if (t_begin < T) {
    load_tile(t_begin);
    store_tile();
  }
  __syncthreads();
  for (int t = t_begin; t < T; ++t) {
    if (t + 1 < T) load_tile(t + 1);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[TM], b[TN];
#pragma unroll
      for (int g = 0; g < GM; ++g) {
        float4 v = *reinterpret_cast<const float4*>(&As[kk][ty * 4 + g * GSM]);
        a[g * 4 + 0] = v.x; a[g * 4 + 1] = v.y; a[g * 4 + 2] = v.z; a[g * 4 + 3] = v.w;
      }
#pragma unroll
      for (int g = 0; g < GN; ++g) {
        float4 v = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4 + g * GSN]);
        b[g * 4 + 0] = v.x; b[g * 4 + 1] = v.y; b[g * 4 + 2] = v.z; b[g * 4 + 3] = v.w;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
    if (t + 1 < T) {
      store_tile();
      __syncthreads();
    }
  }

  // epilogue: bias + activation (+ residual); the activation is dispatched once, outside the per-element code
  TOut* __restrict__ out = reinterpret_cast<TOut*>(p.out);
  const TOut* __restrict__ res = reinterpret_cast<const TOut*>(p.res);
  if (p.ksplit > 1) {  // raw partial sums of this K slice; the consumer sums the slices and applies bias/activation
    if constexpr (sizeof(TOut) == 4) {
#pragma unroll
      for (int gi = 0; gi < GM; ++gi)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          int m = m0 + ty * 4 + gi * GSM + i;
          if (m >= M) continue;
#pragma unroll
          for (int gj = 0; gj < GN; ++gj) {
            int n = n0 + tx * 4 + gj * GSN;
            if (n >= p.Cout) continue;
            float* o = reinterpret_cast<float*>(out) + ((size_t)blockIdx.z * M + m) * p.Cout + n;
            *reinterpret_cast<float4*>(o) = make_float4(acc[gi * 4 + i][gj * 4 + 0], acc[gi * 4 + i][gj * 4 + 1],
                                                        acc[gi * 4 + i][gj * 4 + 2], acc[gi * 4 + i][gj * 4 + 3]);
          }
        }
    }
    return;
  }
  act_dispatch(p.act, [&](auto tag) {
    constexpr int ACT = decltype(tag)::value;
#pragma unroll
    for (int gi = 0; gi < GM; ++gi)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        int m = m0 + ty * 4 + gi * GSM + i;
        if (m >= M) continue;
#pragma unroll
        for (int gj = 0; gj < GN; ++gj) {
          int n = n0 + tx * 4 + gj * GSN;
          if (n >= p.Cout) continue;
          float4 bv = *reinterpret_cast<const float4*>(p.bias + n);
          float4 v = make_float4(acc[gi * 4 + i][gj * 4 + 0] + bv.x, acc[gi * 4 + i][gj * 4 + 1] + bv.y,
                                 acc[gi * 4 + i][gj * 4 + 2] + bv.z, acc[gi * 4 + i][gj * 4 + 3] + bv.w);
          size_t o = (size_t)m * p.Cout + n;
          float4 rv = make_float4(0.f, 0.f, 0.f, 0.f);
          if (res) rv = load4<TOut>(res + o);
          if (p.res_first) { v.x += rv.x; v.y += rv.y; v.z += rv.z; v.w += rv.w; }
          v.x = act_t<ACT>(v.x); v.y = act_t<ACT>(v.y); v.z = act_t<ACT>(v.z); v.w = act_t<ACT>(v.w);
          if (!p.res_first) { v.x += rv.x; v.y += rv.y; v.z += rv.z; v.w += rv.w; }
          store4<TOut>(out + o, v);
        }
      }
  });
}

// ----------------------------------------------------------------------------------------------------------
// depthwise conv, NHWC, one thread per (pixel, 4 channels).  w: [R*S][C], C % 4 == 0.
// ----------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) dwconv_kernel(const __grid_constant__ ConvParams p) {
  const T* __restrict__ in = reinterpret_cast<const T*>(p.in);
  T* __restrict__ out = reinterpret_cast<T*>(p.out);
  const int C4 = p.Cout >> 2;
  const size_t total = (size_t)p.B * p.Hout * p.Wout * C4;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    int c = (int)(idx % C4) * 4;
    size_t pix = idx / C4;
    int ow = (int)(pix % p.Wout);
    size_t t = pix / p.Wout;
    int oh = (int)(t % p.Hout);
    int b = (int)(t / p.Hout);
    float4 acc = *reinterpret_cast<const float4*>(p.bias + c);
    for (int r = 0; r < p.R; ++r) {
      int ih = oh * p.stride - p.pad_t + r * p.dil;
      if (ih < 0 || ih >= p.Hin) continue;
      for (int s = 0; s < p.S; ++s) {
        int iw = ow * p.stride - p.pad_l + s * p.dil;
        if (iw < 0 || iw >= p.Win) continue;
        float4 v = load4<T>(in + ((size_t)(b * p.Hin + ih) * p.Win + iw) * p.Cin + c);
        float4 wv = *reinterpret_cast<const float4*>(p.w + (size_t)(r * p.S + s) * p.Cout + c);
        acc.x = fmaf(v.x, wv.x, acc.x);
        acc.y = fmaf(v.y, wv.y, acc.y);
        acc.z = fmaf(v.z, wv.z, acc.z);
        acc.w = fmaf(v.w, wv.w, acc.w);
      }
    }
    act_dispatch(p.act, [&](auto tag) {
      constexpr int ACT = decltype(tag)::value;
      acc.x = act_t<ACT>(acc.x); acc.y = act_t<ACT>(acc.y); acc.z = act_t<ACT>(acc.z); acc.w = act_t<ACT>(acc.w);
    });
    store4<T>(out + pix * p.Cout + c, acc);
  }
}

// ----------------------------------------------------------------------------------------------------------
// depthwise 3x3 (+ stride 2) + bias + activation + squeeze-excitation pooling, bf16 or fp16 NHWC, 8 channels x 4 output
// pixels per thread: every input column vector is loaded once per row and reused by the outputs it feeds
// (18 / 27 16-byte loads per 4 outputs instead of 36), and the per-channel sums of the SE squeeze are reduced in the
// block and stored (already divided by Hout*Wout) as partial slice pooled[blockIdx.y][b][c]; the consumer (fc1) sums the
// <= 8 slices in a fixed order (deterministic, no atomics), so the pooling pass never re-reads the tensor.
// grid (ceil(C/256), min(ceil(strips/8), 8), B), block (32, 8).
// ----------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float fast_tanh(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// compile-time activation; SiLU with one MUFU op for bf16 outputs, silu_f16out (two) for fp16 outputs
template <int ACT, typename T = __nv_bfloat16>
__device__ __forceinline__ float fast_act(float x) {
  if constexpr (ACT == ACT_SILU && is_f16<T>) {
    return silu_f16out(x);
  } else if constexpr (ACT == ACT_SILU) {
    float h = 0.5f * x;
    return fmaf(h, fast_tanh(h), h);
  } else if constexpr (ACT == ACT_RELU) {
    return fmaxf(x, 0.0f);
  } else if constexpr (ACT == ACT_HSWISH) {
    return x * __saturatef(fmaf(x, 1.0f / 6.0f, 0.5f));
  } else {
    return x;
  }
}

// one packed word of two 16-bit elements -> fp32 pair.  bf16 widens with a 16-bit shift / mask (one ALU op per element);
// fp16 needs a real conversion (HADD2.F32 / F2F per pair).
template <typename T>
__device__ __forceinline__ f32x2 unpack2_16b(unsigned w) {
  if constexpr (is_f16<T>) {
    return __half22float2(*reinterpret_cast<const __half2*>(&w));
  } else {
    return f2_pack(__uint_as_float(w << 16), __uint_as_float(w & 0xffff0000u));
  }
}

template <typename T, int STRIDE, int ACT, int OW = 4>
__global__ void __launch_bounds__(256, OW == 2 ? 3 : 2) dwconv3x3_pool_16b_kernel(const __grid_constant__ ConvParams p, float* __restrict__ pooled) {
  // OW outputs per thread along W; T: element type (__nv_bfloat16 or __half)
  constexpr int NCOL = (OW - 1) * STRIDE + 3;    // input columns feeding them
  const T* __restrict__ in = reinterpret_cast<const T*>(p.in);
  T* __restrict__ out = reinterpret_cast<T*>(p.out);
  const int C = p.Cout;
  const int cv = blockIdx.x * 32 + threadIdx.x;  // channel vector (8 channels)
  const int c = cv * 8;
  const int strips_w = (p.Wout + OW - 1) / OW;
  const int b = blockIdx.z;
  const int cstride = C >> 3;                    // uint4 per pixel
  float psum[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) psum[k] = 0.f;
  float bias[8];
  if (c < C) {
    float4 b0 = *reinterpret_cast<const float4*>(p.bias + c), b1 = *reinterpret_cast<const float4*>(p.bias + c + 4);
    bias[0] = b0.x; bias[1] = b0.y; bias[2] = b0.z; bias[3] = b0.w;
    bias[4] = b1.x; bias[5] = b1.y; bias[6] = b1.z; bias[7] = b1.w;
  }
  for (int strip = blockIdx.y * 8 + threadIdx.y; c < C && strip < strips_w * p.Hout; strip += gridDim.y * 8) {
    const int oh = strip / strips_w;
    const int ow0 = (strip - oh * strips_w) * OW;
    const int iw0 = ow0 * STRIDE - p.pad_l;
    unsigned colmask = 0;
#pragma unroll
    for (int x = 0; x < NCOL; ++x)
      if (iw0 + x >= 0 && iw0 + x < p.Win) colmask |= 1u << x;
    float acc[OW][8];
#pragma unroll
    for (int i = 0; i < OW; ++i)
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[i][k] = bias[k];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int ih = oh * STRIDE - p.pad_t + r;
      if (ih < 0 || ih >= p.Hin) continue;  // warp-uniform (a warp shares its strip)
      // 16-byte vectors of the NCOL input columns of this row (all loads issued before any use)
      const uint4* rowp = reinterpret_cast<const uint4*>(in + ((size_t)(b * p.Hin + ih) * p.Win) * C + c) + (ptrdiff_t)iw0 * cstride;
      uint4 raw[NCOL];
#pragma unroll
      for (int x = 0; x < NCOL; ++x) raw[x] = (colmask >> x) & 1u ? __ldg(rowp + (ptrdiff_t)x * cstride) : make_uint4(0u, 0u, 0u, 0u);
      float w[3][8];
#pragma unroll
      for (int s_ = 0; s_ < 3; ++s_) {
        const float* wp = p.w + (size_t)(r * 3 + s_) * C + c;
        float4 w0 = __ldg(reinterpret_cast<const float4*>(wp)), w1 = __ldg(reinterpret_cast<const float4*>(wp + 4));
        w[s_][0] = w0.x; w[s_][1] = w0.y; w[s_][2] = w0.z; w[s_][3] = w0.w;
        w[s_][4] = w1.x; w[s_][5] = w1.y; w[s_][6] = w1.z; w[s_][7] = w1.w;
      }
#pragma unroll
      for (int x = 0; x < NCOL; ++x) {
        const unsigned wd[4] = {raw[x].x, raw[x].y, raw[x].z, raw[x].w};
        float v[8];
#pragma unroll
        for (int k = 0; k < 4; ++k) f2_unpack(unpack2_16b<T>(wd[k]), v[2 * k], v[2 * k + 1]);
#pragma unroll
        for (int i = 0; i < OW; ++i) {
          const int s_ = x - i * STRIDE;  // compile-time after unrolling
          if (s_ >= 0 && s_ < 3) {
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[i][k] = fmaf(v[k], w[s_][k], acc[i][k]);
          }
        }
      }
    }
    T* orow = out + ((size_t)(b * p.Hout + oh) * p.Wout + ow0) * C + c;
#pragma unroll
    for (int i = 0; i < OW; ++i) {
      if (ow0 + i >= p.Wout) continue;
      uint4 ov;
      typename Pair16<T>::type* o2 = reinterpret_cast<typename Pair16<T>::type*>(&ov);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float a0 = fast_act<ACT, T>(acc[i][2 * k]), a1 = fast_act<ACT, T>(acc[i][2 * k + 1]);
        o2[k] = Pair16<T>::pack(a0, a1);
        psum[2 * k] += a0;
        psum[2 * k + 1] += a1;
      }
      *reinterpret_cast<uint4*>(orow + (size_t)i * C) = ov;
    }
  }
  if (pooled) {
    __shared__ float red[8][32][9];
#pragma unroll
    for (int k = 0; k < 8; ++k) red[threadIdx.y][threadIdx.x][k] = psum[k];
    __syncthreads();
    if (threadIdx.y == 0 && c < C) {
      const float inv = 1.0f / (float)(p.Hout * p.Wout);
      float t[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        t[k] = 0.f;
#pragma unroll
        for (int y = 0; y < 8; ++y) t[k] += red[y][threadIdx.x][k];
        t[k] *= inv;
      }
      float* dst = pooled + ((size_t)blockIdx.y * gridDim.z + b) * C + c;
      *reinterpret_cast<float4*>(dst) = make_float4(t[0], t[1], t[2], t[3]);
      *reinterpret_cast<float4*>(dst + 4) = make_float4(t[4], t[5], t[6], t[7]);
    }
  }
}

// fp32-storage twin of the strip kernel above for the 3xTF32 parity mode: 4 channels (one 16-byte vector) x OW output pixels
// per thread, exact activation (expf SiLU), the same block-reduced partial pooling slices.  grid (ceil(C/128), slices, B).
template <int STRIDE, int ACT, int OW = 4>
__global__ void __launch_bounds__(256, 3) dwconv3x3_pool_f32_kernel(const __grid_constant__ ConvParams p, float* __restrict__ pooled) {
  constexpr int NCOL = (OW - 1) * STRIDE + 3;
  const float* __restrict__ in = reinterpret_cast<const float*>(p.in);
  float* __restrict__ out = reinterpret_cast<float*>(p.out);
  const int C = p.Cout;
  const int c = (blockIdx.x * 32 + threadIdx.x) * 4;
  const int strips_w = (p.Wout + OW - 1) / OW;
  const int b = blockIdx.z;
  const int cstride = C >> 2;  // float4 per pixel
  float psum[4] = {0.f, 0.f, 0.f, 0.f};
  float4 bias4 = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c < C) bias4 = *reinterpret_cast<const float4*>(p.bias + c);
  for (int strip = blockIdx.y * 8 + threadIdx.y; c < C && strip < strips_w * p.Hout; strip += gridDim.y * 8) {
    const int oh = strip / strips_w;
    const int ow0 = (strip - oh * strips_w) * OW;
    const int iw0 = ow0 * STRIDE - p.pad_l;
    unsigned colmask = 0;
#pragma unroll
    for (int x = 0; x < NCOL; ++x)
      if (iw0 + x >= 0 && iw0 + x < p.Win) colmask |= 1u << x;
    float4 acc[OW];
#pragma unroll
    for (int i = 0; i < OW; ++i) acc[i] = bias4;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int ih = oh * STRIDE - p.pad_t + r;
      if (ih < 0 || ih >= p.Hin) continue;  // warp-uniform (a warp shares its strip)
      const float4* rowp = reinterpret_cast<const float4*>(in + ((size_t)(b * p.Hin + ih) * p.Win) * C + c) + (ptrdiff_t)iw0 * cstride;
      float4 raw[NCOL];
#pragma unroll
      for (int x = 0; x < NCOL; ++x) raw[x] = (colmask >> x) & 1u ? __ldg(rowp + (ptrdiff_t)x * cstride) : make_float4(0.f, 0.f, 0.f, 0.f);
      float4 w[3];
#pragma unroll
      for (int s_ = 0; s_ < 3; ++s_) w[s_] = __ldg(reinterpret_cast<const float4*>(p.w + (size_t)(r * 3 + s_) * C + c));
#pragma unroll
      for (int x = 0; x < NCOL; ++x) {
#pragma unroll
        for (int i = 0; i < OW; ++i) {
          const int s_ = x - i * STRIDE;  // compile-time after unrolling
          if (s_ >= 0 && s_ < 3) {
            acc[i].x = fmaf(raw[x].x, w[s_].x, acc[i].x);
            acc[i].y = fmaf(raw[x].y, w[s_].y, acc[i].y);
            acc[i].z = fmaf(raw[x].z, w[s_].z, acc[i].z);
            acc[i].w = fmaf(raw[x].w, w[s_].w, acc[i].w);
          }
        }
      }
    }
    float* orow = out + ((size_t)(b * p.Hout + oh) * p.Wout + ow0) * C + c;
#pragma unroll
    for (int i = 0; i < OW; ++i) {
      if (ow0 + i >= p.Wout) continue;
      float4 o = make_float4(act_t<ACT>(acc[i].x), act_t<ACT>(acc[i].y), act_t<ACT>(acc[i].z), act_t<ACT>(acc[i].w));
      psum[0] += o.x; psum[1] += o.y; psum[2] += o.z; psum[3] += o.w;
      *reinterpret_cast<float4*>(orow + (size_t)i * C) = o;
    }
  }
  if (pooled) {
    __shared__ float red[8][32][5];
#pragma unroll
    for (int k = 0; k < 4; ++k) red[threadIdx.y][threadIdx.x][k] = psum[k];
    __syncthreads();
    if (threadIdx.y == 0 && c < C) {
      const float inv = 1.0f / (float)(p.Hout * p.Wout);
      float t[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        t[k] = 0.f;
#pragma unroll
        for (int y = 0; y < 8; ++y) t[k] += red[y][threadIdx.x][k];
        t[k] *= inv;
      }
      *reinterpret_cast<float4*>(pooled + ((size_t)blockIdx.y * gridDim.z + b) * C + c) = make_float4(t[0], t[1], t[2], t[3]);
    }
  }
}

// ----------------------------------------------------------------------------------------------------------
// depthwise 5x5 (stride 1 or 2) + bias + activation, bf16 or fp16 NHWC, C % 8 == 0: the per-thread layout of
// dwconv3x3_pool_16b_kernel (8 channels x OW output pixels, 16-byte loads), so each of the (OW-1)*STRIDE + 5 input column vectors of a
// row is loaded once and feeds every output that uses it (40 / 55 loads per 4 outputs instead of 100).  The arithmetic is
// dwconv_kernel's, operation for operation: each accumulator starts at the bias, the taps are added with fmaf in row-major
// order (r outer, s inner), taps outside the map are skipped, the activation is the exact act_t and the result is rounded
// to nearest even; the outputs are bit-identical to dwconv_kernel's on the same inputs.
// POOL = false: no pooling (the SE squeeze stays a separate pool_mean_kernel pass).  One grid-stride loop over (crop, output
// row, strip, channel vector), channel vectors fastest: narrow layers (72, 96, 120 channels) fill whole warps.
// grid grid_for(items, 256), block 256; `pooled` is unused.
// POOL = true: also the SE squeeze of the outputs AS STORED (rounded to T), as the partial slices pooled[blockIdx.y][b][c]
// already divided by Hout*Wout, like dwconv3x3_pool_16b_kernel; fc1 sums the slices in a fixed order (deterministic, no
// atomics).  grid (channel chunks, slices, B); a block is blockDim.x / cb groups of cb = ceil(C/8 / gridDim.x) channel
// vectors, group g of slice y walks the strips y*groups + g, += gridDim.y*groups of crop blockIdx.z.  `pooled` may be null.
// ----------------------------------------------------------------------------------------------------------
template <typename T, int STRIDE, int ACT, int OW = 4, bool POOL = false>
__global__ void __launch_bounds__(256) dwconv5x5_16b_kernel(const __grid_constant__ ConvParams p, float* __restrict__ pooled) {
  constexpr int NCOL = (OW - 1) * STRIDE + 5;  // input columns feeding OW outputs
  const T* __restrict__ in = reinterpret_cast<const T*>(p.in);
  T* __restrict__ out = reinterpret_cast<T*>(p.out);
  const int C = p.Cout;
  const int cstride = C >> 3;  // uint4 per pixel
  const int strips_w = (p.Wout + OW - 1) / OW;
  // POOL: thread (g, cv) of the block is channel vector cv of group g, and its loop index is a strip (oh * strips_w + ow0 / OW)
  // of crop blockIdx.z.  The if-constexpr forms below leave the POOL = false kernel exactly as it was before pooling existed.
  struct PoolThread { int cb, groups, g, cv; float psum[8]; };
  struct NoPool {};
  std::conditional_t<POOL, PoolThread, NoPool> pt;
  if constexpr (POOL) {
    pt.cb = (cstride + gridDim.x - 1) / gridDim.x;
    pt.groups = blockDim.x / pt.cb;
    pt.g = threadIdx.x / pt.cb;
    pt.cv = blockIdx.x * pt.cb + threadIdx.x % pt.cb;
#pragma unroll
    for (int k = 0; k < 8; ++k) pt.psum[k] = 0.f;
  }
  const size_t total = [&] {
    if constexpr (POOL) return pt.g < pt.groups && pt.cv < cstride ? (size_t)strips_w * p.Hout : (size_t)0;
    else return (size_t)p.B * p.Hout * strips_w * cstride;
  }();
  const size_t first = [&] {
    if constexpr (POOL) return (size_t)blockIdx.y * pt.groups + pt.g;
    else return (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  }();
  const size_t step = [&] {
    if constexpr (POOL) return (size_t)gridDim.y * pt.groups;
    else return (size_t)gridDim.x * blockDim.x;
  }();
  for (size_t idx = first; idx < total; idx += step) {
    int c, ow0, oh, b;
    if constexpr (POOL) {
      c = pt.cv * 8;
      oh = (int)(idx / strips_w);
      ow0 = (int)(idx - (size_t)oh * strips_w) * OW;
      b = blockIdx.z;
    } else {
      c = (int)(idx % cstride) * 8;
      size_t t = idx / cstride;
      ow0 = (int)(t % strips_w) * OW;
      t /= strips_w;
      oh = (int)(t % p.Hout);
      b = (int)(t / p.Hout);
    }
    const int iw0 = ow0 * STRIDE - p.pad_l;
    unsigned colmask = 0;
#pragma unroll
    for (int x = 0; x < NCOL; ++x)
      if (iw0 + x >= 0 && iw0 + x < p.Win) colmask |= 1u << x;
    float acc[OW][8];
    {
      const float4 b0 = *reinterpret_cast<const float4*>(p.bias + c), b1 = *reinterpret_cast<const float4*>(p.bias + c + 4);
      const float bias[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < OW; ++i)
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[i][k] = bias[k];
    }
#pragma unroll
    for (int r = 0; r < 5; ++r) {
      const int ih = oh * STRIDE - p.pad_t + r;
      if (ih < 0 || ih >= p.Hin) continue;
      const uint4* rowp = reinterpret_cast<const uint4*>(in + ((size_t)(b * p.Hin + ih) * p.Win) * C + c) + (ptrdiff_t)iw0 * cstride;
      uint4 raw[NCOL];
#pragma unroll
      for (int x = 0; x < NCOL; ++x) raw[x] = (colmask >> x) & 1u ? __ldg(rowp + (ptrdiff_t)x * cstride) : make_uint4(0u, 0u, 0u, 0u);
      float w[5][8];
#pragma unroll
      for (int s_ = 0; s_ < 5; ++s_) {
        const float* wp = p.w + (size_t)(r * 5 + s_) * C + c;
        const float4 w0 = __ldg(reinterpret_cast<const float4*>(wp)), w1 = __ldg(reinterpret_cast<const float4*>(wp + 4));
        w[s_][0] = w0.x; w[s_][1] = w0.y; w[s_][2] = w0.z; w[s_][3] = w0.w;
        w[s_][4] = w1.x; w[s_][5] = w1.y; w[s_][6] = w1.z; w[s_][7] = w1.w;
      }
      // ascending x visits each output's taps in ascending s; a column outside the map is skipped, not added as zero
#pragma unroll
      for (int x = 0; x < NCOL; ++x) {
        if (!((colmask >> x) & 1u)) continue;
        const unsigned wd[4] = {raw[x].x, raw[x].y, raw[x].z, raw[x].w};
        float v[8];
#pragma unroll
        for (int k = 0; k < 4; ++k) f2_unpack(unpack2_16b<T>(wd[k]), v[2 * k], v[2 * k + 1]);
#pragma unroll
        for (int i = 0; i < OW; ++i) {
          const int s_ = x - i * STRIDE;  // compile-time after unrolling
          if (s_ >= 0 && s_ < 5) {
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[i][k] = fmaf(v[k], w[s_][k], acc[i][k]);
          }
        }
      }
    }
    T* orow = out + ((size_t)(b * p.Hout + oh) * p.Wout + ow0) * C + c;
#pragma unroll
    for (int i = 0; i < OW; ++i) {
      if (ow0 + i >= p.Wout) continue;
      uint4 ov;
      typename Pair16<T>::type* o2 = reinterpret_cast<typename Pair16<T>::type*>(&ov);
#pragma unroll
      for (int k = 0; k < 4; ++k) o2[k] = Pair16<T>::pack(act_t<ACT>(acc[i][2 * k]), act_t<ACT>(acc[i][2 * k + 1]));
      *reinterpret_cast<uint4*>(orow + (size_t)i * C) = ov;
      if constexpr (POOL) {  // the values as stored
        const unsigned wd[4] = {ov.x, ov.y, ov.z, ov.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          float v0, v1;
          f2_unpack(unpack2_16b<T>(wd[k]), v0, v1);
          pt.psum[2 * k] += v0;
          pt.psum[2 * k + 1] += v1;
        }
      }
    }
  }
  if constexpr (POOL) {
    if (pooled) {
      __shared__ float red[256][9];
#pragma unroll
      for (int k = 0; k < 8; ++k) red[threadIdx.x][k] = pt.psum[k];
      __syncthreads();
      if (pt.g == 0 && pt.cv < cstride) {
        const float inv = 1.0f / (float)(p.Hout * p.Wout);
        float t[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          t[k] = 0.f;
          for (int y = 0; y < pt.groups; ++y) t[k] += red[y * pt.cb + threadIdx.x][k];
          t[k] *= inv;
        }
        float* dst = pooled + ((size_t)blockIdx.y * gridDim.z + blockIdx.z) * C + pt.cv * 8;
        *reinterpret_cast<float4*>(dst) = make_float4(t[0], t[1], t[2], t[3]);
        *reinterpret_cast<float4*>(dst + 4) = make_float4(t[4], t[5], t[6], t[7]);
      }
    }
  }
}

// ----------------------------------------------------------------------------------------------------------
// stem: direct conv for tiny Cin (3) reading the caller's NCHW fp32 crops, with the per-channel input affine
// (PreprocLayer x*2-1, backbones/efficientnet.py:1185) applied to in-bounds pixels only (pad happens AFTER
// preprocessing in the reference), writing NHWC.  w: [R*S*Cin][Cout], one thread per (pixel, 4 out channels).
// ----------------------------------------------------------------------------------------------------------
struct StemParams {
  const float* in;  // [B,Cin,Hin,Win]
  void* out;        // [B,Hout,Wout,Cout]
  const float* w;
  const float* bias;
  float pre_scale[4], pre_shift[4];
  int B, Hin, Win, Cin, Hout, Wout, Cout, R, S, stride, pad_t, pad_l, act;
};

template <typename TOut>
__global__ void __launch_bounds__(256) stem_conv_kernel(StemParams p) {
  extern __shared__ float sw[];  // weights [R*S*Cin][Cout] + bias [Cout]
  const int K = p.R * p.S * p.Cin;
  for (int i = threadIdx.x; i < K * p.Cout; i += blockDim.x) sw[i] = p.w[i];
  float* sb = sw + K * p.Cout;
  for (int i = threadIdx.x; i < p.Cout; i += blockDim.x) sb[i] = p.bias[i];
  __syncthreads();
  TOut* __restrict__ out = reinterpret_cast<TOut*>(p.out);
  const int C4 = p.Cout >> 2;
  const size_t total = (size_t)p.B * p.Hout * p.Wout * C4;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    int c = (int)(idx % C4) * 4;
    size_t pix = idx / C4;
    int ow = (int)(pix % p.Wout);
    size_t t = pix / p.Wout;
    int oh = (int)(t % p.Hout);
    int b = (int)(t / p.Hout);
    float4 acc = *reinterpret_cast<const float4*>(sb + c);
    for (int r = 0; r < p.R; ++r) {
      int ih = oh * p.stride - p.pad_t + r;
      if (ih < 0 || ih >= p.Hin) continue;
      for (int s = 0; s < p.S; ++s) {
        int iw = ow * p.stride - p.pad_l + s;
        if (iw < 0 || iw >= p.Win) continue;
        for (int ci = 0; ci < p.Cin; ++ci) {
          float v = __ldg(p.in + ((size_t)(b * p.Cin + ci) * p.Hin + ih) * p.Win + iw) * p.pre_scale[ci] + p.pre_shift[ci];
          float4 wv = *reinterpret_cast<const float4*>(sw + (size_t)((r * p.S + s) * p.Cin + ci) * p.Cout + c);
          acc.x = fmaf(v, wv.x, acc.x);
          acc.y = fmaf(v, wv.y, acc.y);
          acc.z = fmaf(v, wv.z, acc.z);
          acc.w = fmaf(v, wv.w, acc.w);
        }
      }
    }
    act_dispatch(p.act, [&](auto tag) {
      constexpr int ACT = decltype(tag)::value;
      acc.x = act_t<ACT>(acc.x); acc.y = act_t<ACT>(acc.y); acc.z = act_t<ACT>(acc.z); acc.w = act_t<ACT>(acc.w);
    });
    store4<TOut>(out + pix * p.Cout + c, acc);
  }
}

// ----------------------------------------------------------------------------------------------------------
// stem, second form: one thread per (pixel, CPT output channels) - the R*S*Cin input taps are loaded ONCE per pixel
// (the first form re-loads them in each of its Cout/4 threads) and every weight float4 is a shared-memory broadcast.
// ----------------------------------------------------------------------------------------------------------
template <typename TOut, int CPT>
__global__ void __launch_bounds__(128) stem_conv_wide_kernel(StemParams p) {
  extern __shared__ float sw[];  // weights [R*S*Cin][Cout] + bias [Cout]
  const int K = p.R * p.S * p.Cin;
  for (int i = threadIdx.x; i < K * p.Cout; i += blockDim.x) sw[i] = p.w[i];
  float* sb = sw + K * p.Cout;
  for (int i = threadIdx.x; i < p.Cout; i += blockDim.x) sb[i] = p.bias[i];
  __syncthreads();
  TOut* __restrict__ out = reinterpret_cast<TOut*>(p.out);
  const int groups = p.Cout / CPT;
  const size_t total = (size_t)p.B * p.Hout * p.Wout * groups;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int c0 = (int)(idx % groups) * CPT;
    size_t pix = idx / groups;
    int ow = (int)(pix % p.Wout);
    size_t t = pix / p.Wout;
    int oh = (int)(t % p.Hout);
    int b = (int)(t / p.Hout);
    float acc[CPT];
#pragma unroll
    for (int j = 0; j < CPT; ++j) acc[j] = sb[c0 + j];
    for (int r = 0; r < p.R; ++r) {
      int ih = oh * p.stride - p.pad_t + r;
      if (ih < 0 || ih >= p.Hin) continue;
      for (int s = 0; s < p.S; ++s) {
        int iw = ow * p.stride - p.pad_l + s;
        if (iw < 0 || iw >= p.Win) continue;
        for (int ci = 0; ci < p.Cin; ++ci) {
          float v = __ldg(p.in + ((size_t)(b * p.Cin + ci) * p.Hin + ih) * p.Win + iw) * p.pre_scale[ci] + p.pre_shift[ci];
          const float* wrow = sw + (size_t)((r * p.S + s) * p.Cin + ci) * p.Cout + c0;
#pragma unroll
          for (int j = 0; j < CPT; j += 4) {
            float4 wv = *reinterpret_cast<const float4*>(wrow + j);
            acc[j + 0] = fmaf(v, wv.x, acc[j + 0]);
            acc[j + 1] = fmaf(v, wv.y, acc[j + 1]);
            acc[j + 2] = fmaf(v, wv.z, acc[j + 2]);
            acc[j + 3] = fmaf(v, wv.w, acc[j + 3]);
          }
        }
      }
    }
    act_dispatch(p.act, [&](auto tag) {
      constexpr int ACT = decltype(tag)::value;
#pragma unroll
      for (int j = 0; j < CPT; ++j) acc[j] = act_t<ACT>(acc[j]);
    });
#pragma unroll
    for (int j = 0; j < CPT; j += 4)
      store4<TOut>(out + pix * p.Cout + c0 + j, make_float4(acc[j], acc[j + 1], acc[j + 2], acc[j + 3]));
  }
}

// ----------------------------------------------------------------------------------------------------------
// stem, third form: the EfficientNet stem itself (3x3, stride 2, 3 input channels, all CPT = Cout output channels per thread),
// fully unrolled; two output channels per FFMA2 (same IEEE fma per channel and the same tap order as the forms above: the
// results are bit-identical), every weight float4 a shared-memory broadcast.  stem_conv_wide_kernel ran this layer at 13
// TFLOP/s (7.4x its HBM floor): runtime tap loops, 64-bit address arithmetic per tap and one scalar FMA per weight.
// ----------------------------------------------------------------------------------------------------------
template <typename TOut, int CPT>
__global__ void __launch_bounds__(128) stem3x3s2_kernel(StemParams p) {
  extern __shared__ float sw[];  // weights [27][Cout] + bias [Cout]
  for (int i = threadIdx.x; i < 27 * CPT; i += blockDim.x) sw[i] = p.w[i];
  float* sb = sw + 27 * CPT;
  for (int i = threadIdx.x; i < CPT; i += blockDim.x) sb[i] = p.bias[i];
  __syncthreads();
  TOut* __restrict__ out = reinterpret_cast<TOut*>(p.out);
  const size_t total = (size_t)p.B * p.Hout * p.Wout;
  const size_t plane = (size_t)p.Hin * p.Win;
  for (size_t pix = (size_t)blockIdx.x * blockDim.x + threadIdx.x; pix < total; pix += (size_t)gridDim.x * blockDim.x) {
    const int ow = (int)(pix % p.Wout);
    const size_t t = pix / p.Wout;
    const int oh = (int)(t % p.Hout);
    const int b = (int)(t / p.Hout);
    f32x2 acc[CPT / 2];
#pragma unroll
    for (int j = 0; j < CPT / 2; ++j) acc[j] = f2_pack(sb[2 * j], sb[2 * j + 1]);
    const float* img = p.in + (size_t)b * 3 * plane;
    const int ih0 = oh * 2 - p.pad_t, iw0 = ow * 2 - p.pad_l;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int ih = ih0 + r;
      const bool rok = ih >= 0 && ih < p.Hin;
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int iw = iw0 + s;
        if (rok && iw >= 0 && iw < p.Win) {  // an out-of-image tap contributes nothing (the reference pads AFTER x*2-1)
          const float* px = img + (size_t)ih * p.Win + iw;
#pragma unroll
          for (int ci = 0; ci < 3; ++ci) {
            const float v = __ldg(px + ci * plane) * p.pre_scale[ci] + p.pre_shift[ci];
            const f32x2 vv = f2_pack(v, v);
            const float4* wrow = reinterpret_cast<const float4*>(sw + ((r * 3 + s) * 3 + ci) * CPT);
#pragma unroll
            for (int j = 0; j < CPT / 4; ++j) {
              const float4 wv = wrow[j];
              acc[2 * j] = f2_fma(vv, f2_pack(wv.x, wv.y), acc[2 * j]);
              acc[2 * j + 1] = f2_fma(vv, f2_pack(wv.z, wv.w), acc[2 * j + 1]);
            }
          }
        }
      }
    }
    float o[CPT];
#pragma unroll
    for (int j = 0; j < CPT / 2; ++j) f2_unpack(acc[j], o[2 * j], o[2 * j + 1]);
    act_dispatch(p.act, [&](auto tag) {
      constexpr int ACT = decltype(tag)::value;
#pragma unroll
      for (int j = 0; j < CPT; ++j) o[j] = act_t<ACT>(o[j]);
    });
#pragma unroll
    for (int j = 0; j < CPT; j += 4) store4<TOut>(out + pix * CPT + j, make_float4(o[j], o[j + 1], o[j + 2], o[j + 3]));
  }
}

// ----------------------------------------------------------------------------------------------------------
// global average pool over the spatial axes (squeeze of squeeze-excitation): in [B,P,C] -> mean [B,C] fp32.
// grid (ceil(C/128), B), block (32, 8).
// ----------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) pool_mean_kernel(const T* __restrict__ in, float* __restrict__ out, int P, int C) {
  __shared__ float4 red[8][32];
  const int c = (blockIdx.x * 32 + threadIdx.x) * 4;
  const int b = blockIdx.y;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c < C) {
    const T* base = in + (size_t)b * P * C + c;
    for (int px = threadIdx.y; px < P; px += 8) {
      float4 v = load4<T>(base + (size_t)px * C);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
  }
  red[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    float4 s = red[0][threadIdx.x];
#pragma unroll
    for (int i = 1; i < 8; ++i) {
      float4 v = red[i][threadIdx.x];
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    float inv = 1.0f / (float)P;
    *reinterpret_cast<float4*>(out + (size_t)b * C + c) = make_float4(s.x * inv, s.y * inv, s.z * inv, s.w * inv);
  }
}

// sums the split-K partial slices of a squeeze-excitation fc1 ([ksplit][B][C] raw sums), adds the bias and applies the
// activation: hidden[b][c] = act(sum_z partial[z][b][c] + bias[c]).  Fixed summation order (deterministic).
__global__ void __launch_bounds__(256) se_reduce_kernel(const float* __restrict__ partial, const float* __restrict__ bias,
                                                        float* __restrict__ out, int n, int C, int ksplit, int act) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float v = 0.f;
  for (int z = 0; z < ksplit; ++z) v += partial[(size_t)z * n + i];
  out[i] = apply_act(v + bias[i % C], act);
}

// max pool (ResNet stem, metrabs_tf/backbones/resnet.py:187-193), NHWC.  The reference pads with ZeroPadding2D and
// pools VALID, so an out-of-bounds tap contributes the value 0 to the max.
template <typename T>
__global__ void __launch_bounds__(256) maxpool_kernel(const __grid_constant__ ConvParams p) {
  const T* __restrict__ in = reinterpret_cast<const T*>(p.in);
  T* __restrict__ out = reinterpret_cast<T*>(p.out);
  const int C4 = p.Cout >> 2;
  const size_t total = (size_t)p.B * p.Hout * p.Wout * C4;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    int c = (int)(idx % C4) * 4;
    size_t pix = idx / C4;
    int ow = (int)(pix % p.Wout);
    size_t t = pix / p.Wout;
    int oh = (int)(t % p.Hout);
    int b = (int)(t / p.Hout);
    float4 acc = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    for (int r = 0; r < p.R; ++r) {
      int ih = oh * p.stride - p.pad_t + r;
      for (int s = 0; s < p.S; ++s) {
        int iw = ow * p.stride - p.pad_l + s;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (ih >= 0 && ih < p.Hin && iw >= 0 && iw < p.Win)
          v = load4<T>(in + ((size_t)(b * p.Hin + ih) * p.Win + iw) * p.Cin + c);
        acc.x = fmaxf(acc.x, v.x); acc.y = fmaxf(acc.y, v.y); acc.z = fmaxf(acc.z, v.z); acc.w = fmaxf(acc.w, v.w);
      }
    }
    store4<T>(out + pix * p.Cout + c, acc);
  }
}

// ---------------------------------------------------------------------------------------------- launchers
template <typename TIn, typename TOut>
inline cudaError_t launch_conv_igemm(const ConvParams& p, cudaStream_t st) {
  const int M = p.B * p.Hout * p.Wout;
  if (p.Cout > 64 && M >= 128 * (size_t)num_sms()) {
    dim3 grid((M + 127) / 128, (p.Cout + 127) / 128);
    launch_k(conv_igemm_kernel<128, 128, 8, 8, TIn, TOut>, dim3(grid), dim3(256), 0, st, p);
  } else if (M >= 128 * (size_t)num_sms()) {
    dim3 grid((M + 127) / 128, (p.Cout + 63) / 64);
    launch_k(conv_igemm_kernel<128, 64, 8, 4, TIn, TOut>, dim3(grid), dim3(256), 0, st, p);
  } else {
    dim3 grid((M + 63) / 64, (p.Cout + 63) / 64, p.ksplit);
    launch_k(conv_igemm_kernel<64, 64, 4, 4, TIn, TOut>, dim3(grid), dim3(256), 0, st, p);
  }
  return cudaGetLastError();
}

inline int grid_for(size_t total, int block) {
  size_t g = (total + block - 1) / block;
  size_t cap = (size_t)num_sms() * 16;
  return (int)(g < cap ? (g ? g : 1) : cap);
}

}  // namespace mtb
