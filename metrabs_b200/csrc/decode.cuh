// Soft-argmax decode and absolute reconstruction kernels.
//   ptu.soft_argmax / decode_heatmap / linspace   (/root/reference/metrabs_pytorch/ptu.py:47-92)
//   heatmap_to_image / heatmap_to_metric           (models/util.py:6-33)
//   reconstruct_absolute & helpers                 (ptu3d.py:9-33, 52-121)
#pragma once
#include "common.cuh"

namespace mtb {

// Online-softmax state of one (b, joint) row: running max m, S = sum e, and the e-weighted INDEX sums.
struct SoftState {
  float m, s, sx, sy, sz;
};

__device__ __forceinline__ void soft_init(SoftState& a) {
  a.m = -INFINITY; a.s = 0.f; a.sx = 0.f; a.sy = 0.f; a.sz = 0.f;
}
__device__ __forceinline__ void soft_merge(SoftState& a, const SoftState& b) {
  float m = fmaxf(a.m, b.m);
  if (m == -INFINITY) return;
  float fa = exp2f((a.m - m) * 1.4426950408889634f), fb = exp2f((b.m - m) * 1.4426950408889634f);
  a.s = a.s * fa + b.s * fb;
  a.sx = a.sx * fa + b.sx * fb;
  a.sy = a.sy * fa + b.sy * fb;
  a.sz = a.sz * fa + b.sz * fb;
  a.m = m;
}
__device__ __forceinline__ SoftState soft_shfl_xor(const SoftState& a, int o) {
  SoftState b;
  b.m = __shfl_xor_sync(0xffffffffu, a.m, o);
  b.s = __shfl_xor_sync(0xffffffffu, a.s, o);
  b.sx = __shfl_xor_sync(0xffffffffu, a.sx, o);
  b.sy = __shfl_xor_sync(0xffffffffu, a.sy, o);
  b.sz = __shfl_xor_sync(0xffffffffu, a.sz, o);
  return b;
}
// linspace(0,1,n)[i] expectation: sum(e*i)/sum(e)/(n-1); n == 1 -> 0.5  (ptu.py:83-84)
__device__ __forceinline__ float soft_coord(float weighted_index_sum, float s, int n) {
  return n > 1 ? weighted_index_sum / s / (float)(n - 1) : 0.5f;
}
// the same expectation with tf.linspace(0, 1, n), which is [0] for n == 1 (tfu.py:230): the TF-only Metro and Model25D heads
__device__ __forceinline__ float soft_coord_tf(float weighted_index_sum, float s, int n) {
  return n > 1 ? weighted_index_sum / s / (float)(n - 1) : 0.f;
}

// ----------------------------------------------------------------------------------------------------------
// Standalone soft-argmax over the REFERENCE layout: logits [B,D,J,H,W] (D >= 1) -> out [B,J,3] = (x,y,z), or,
// with two_d != 0, logits [B,J,H,W] -> out [B,J,2].  One CTA per (b,j) row: D segments of H*W contiguous
// elements.  Single pass over HBM (algorithmic bytes = the logits once), 128-bit loads when W % 4 == 0.
// ----------------------------------------------------------------------------------------------------------
// 16-byte vector of logits -> floats (4 fp32 or 8 bf16)
template <typename T>
struct Vec16;
template <>
struct Vec16<float> {
  static constexpr int N = 4;
  static __device__ __forceinline__ void load(const float* p, float* v) {
    float4 q = __ldg(reinterpret_cast<const float4*>(p));
    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
  }
};
template <>
struct Vec16<__nv_bfloat16> {
  static constexpr int N = 8;
  static __device__ __forceinline__ void load(const __nv_bfloat16* p, float* v) {
    uint4 q = __ldg(reinterpret_cast<const uint4*>(p));
    const unsigned w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      v[2 * i] = __uint_as_float(w[i] << 16);
      v[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
  }
};

template <>
struct Vec16<__half> {
  static constexpr int N = 8;
  static __device__ __forceinline__ void load(const __half* p, float* v) {
    uint4 q = __ldg(reinterpret_cast<const uint4*>(p));
    const unsigned w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
      v[2 * i] = f.x;
      v[2 * i + 1] = f.y;
    }
  }
};

// fp32 pairs for the 16-bit-logit soft-argmax (8 elements per 16-byte load); each operation is the scalar IEEE fma / mul / add
// per half, so results do not depend on how the compiler schedules the pair
typedef float2 sa_f2;
__device__ __forceinline__ sa_f2 sa_pack(float lo, float hi) { return make_float2(lo, hi); }
__device__ __forceinline__ void sa_unpack(sa_f2 v, float& lo, float& hi) { lo = v.x; hi = v.y; }
__device__ __forceinline__ sa_f2 sa_fma(sa_f2 a, sa_f2 b, sa_f2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ sa_f2 sa_mul(sa_f2 a, sa_f2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ sa_f2 sa_add(sa_f2 a, sa_f2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }

__device__ __forceinline__ float ex2_fast(float x) {  // one MUFU op; inputs here are <= 0
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// VEC = elements per load: 16 bytes' worth (4 fp32 / 8 bf16) when W % VEC == 0 and the base is 16-byte aligned, else 1.
// UNROLL independent 16-byte loads are in flight per thread before any is consumed.  The first version of this kernel
// spent ~32 lane-instructions per element (ncu: issue slots 73 % busy at 51 % of HBM peak: integer divisions per vector,
// int->float converts and the slow-path exp2f per element); this one spends ~9: power-of-two index math when H*W and W
// are powers of two (POW2), exp2 as one FFMA + one MUFU (the shared factor 2^(-m*log2e) cancels in sum(e*x)/sum(e), so
// its rounding is irrelevant), and the x-weights as compile-time constants plus one FMA per vector.
template <typename T, int VEC, bool POW2>
__global__ void __launch_bounds__(256) softargmax_bdjhw_kernel(const T* __restrict__ logits, float* __restrict__ out,
                                                               int J, int D, int H, int W, int two_d, int hw_shift,
                                                               int w_shift) {
  constexpr int UNROLL = 4;
  const int row = blockIdx.x;  // b*J + j
  const int b = row / J, j = row - b * J;
  const int HW = H * W;
  const int n = D * HW;
  constexpr float L2E = 1.4426950408889634f;
  float m = -INFINITY, mL = -INFINITY, s_ = 0.f, sx = 0.f, sy = 0.f, sz = 0.f;
  const int step = blockDim.x * VEC;
  const T* base = logits + ((size_t)b * D * J + j) * HW;
  const size_t dstride = (size_t)J * HW;
  for (int e0 = threadIdx.x * VEC; e0 < n; e0 += step * UNROLL) {
    float v[UNROLL][VEC];
    int dd[UNROLL], yy[UNROLL], xx[UNROLL];
    bool ok[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const int e = e0 + u * step;
      ok[u] = e < n;
      const int ee = ok[u] ? e : 0;
      int d, rem, y;
      if (POW2) {
        d = ee >> hw_shift;
        rem = ee & (HW - 1);
        y = rem >> w_shift;
        xx[u] = rem & (W - 1);
      } else {
        d = ee / HW;
        rem = ee - d * HW;
        y = rem / W;
        xx[u] = rem - y * W;
      }
      dd[u] = d; yy[u] = y;
      const T* ptr = base + (size_t)d * dstride + rem;
      if (ok[u]) {
        if constexpr (VEC == 1) v[u][0] = load1<T>(ptr);
        else Vec16<T>::load(ptr, v[u]);
      } else {
#pragma unroll
        for (int i = 0; i < VEC; ++i) v[u][i] = -INFINITY;  // exp2(-inf) = 0: contributes nothing
      }
    }
    float vm = v[0][0];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u)
#pragma unroll
      for (int i = 0; i < VEC; ++i) vm = fmaxf(vm, v[u][i]);
    if (vm > m) {
      const float mL_new = vm * L2E;
      const float f = ex2_fast(mL - mL_new);  // same rounded offsets as the elements use; first time exp2(-inf) = 0
      s_ *= f; sx *= f; sy *= f; sz *= f;
      m = vm;
      mL = mL_new;
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      float es = 0.f, ex = 0.f;
      if constexpr (VEC == 8) {
        // 16-bit logits: scale / sum / index-weighted sum on packed fp32 pairs (4 FFMA2 + 3 FADD2 + FMUL2 + 3 FFMA2 per 8 elements)
        const sa_f2 l2 = sa_pack(L2E, L2E), nm = sa_pack(-mL, -mL);
        sa_f2 e2[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          float a, b;
          sa_unpack(sa_fma(sa_pack(v[u][2 * i], v[u][2 * i + 1]), l2, nm), a, b);
          e2[i] = sa_pack(ex2_fast(a), ex2_fast(b));
        }
        float lo, hi;
        sa_unpack(sa_add(sa_add(e2[0], e2[1]), sa_add(e2[2], e2[3])), lo, hi);
        es = lo + hi;
        sa_f2 xw = sa_mul(e2[0], sa_pack(0.f, 1.f));
        xw = sa_fma(e2[1], sa_pack(2.f, 3.f), xw);
        xw = sa_fma(e2[2], sa_pack(4.f, 5.f), xw);
        xw = sa_fma(e2[3], sa_pack(6.f, 7.f), xw);
        sa_unpack(xw, lo, hi);
        ex = lo + hi;
      } else {
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
          const float ee = ex2_fast(fmaf(v[u][i], L2E, -mL));
          es += ee;
          if (i > 0) ex = fmaf(ee, (float)i, ex);
        }
      }
      s_ += es;
      sx += fmaf(es, (float)xx[u], ex);
      sy = fmaf(es, (float)yy[u], sy);
      sz = fmaf(es, (float)dd[u], sz);
    }
  }
  SoftState st;
  st.m = m; st.s = s_; st.sx = sx; st.sy = sy; st.sz = sz;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    SoftState other = soft_shfl_xor(st, o);
    soft_merge(st, other);
  }
  __shared__ SoftState red[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) red[warp] = st;
  __syncthreads();
  if (threadIdx.x == 0) {
    SoftState a = red[0];
    for (int i = 1; i < (int)(blockDim.x >> 5); ++i) soft_merge(a, red[i]);
    if (two_d) {
      out[(size_t)row * 2 + 0] = soft_coord(a.sx, a.s, W);
      out[(size_t)row * 2 + 1] = soft_coord(a.sy, a.s, H);
    } else {
      out[(size_t)row * 3 + 0] = soft_coord(a.sx, a.s, W);
      out[(size_t)row * 3 + 1] = soft_coord(a.sy, a.s, H);
      out[(size_t)row * 3 + 2] = soft_coord(a.sz, a.s, D);
    }
  }
}

// ----------------------------------------------------------------------------------------------------------
// Soft-argmax over the library-internal NHWC logits [B, P=H*W, N=J*(1+D)], channel n = J + d*J + j (n < J: 2D).
// One CTA per crop; thread (cx, py): channel lane cx, pixel slice py; per-channel states merged in smem, then
// the D depth slices of each joint are merged.  Outputs are the [0,1] heatmap coordinates; `scale` applies
// heatmap_to_image / heatmap_to_metric (models/util.py) when non-null.
// HEAD3D: the head of the TF-only Metro / Model25D classes (metrabs_tf/models/metro.py:34-44, twofive.py:46-56): no 2D
// block, N = D*J with channel n = d*J + j, tf.linspace's n == 1 rule, and the 3D scale (met_*) applied to x and y; out2d,
// when non-null, receives the same x and y.
// ----------------------------------------------------------------------------------------------------------
struct DecodeScale {
  float img_mul, img_add;  // coords2d px = c * img_mul + img_add          (heatmap_to_image)
  float met_mul, met_add;  // xy_mm = (c * img_mul + img_add) * box/S  =>  c * met_mul + met_add (Model25D: = img_*)
  float z_mul;             // z_mm = c * box_size_mm
  int apply;
};

template <typename T, bool HEAD3D = false>
__global__ void __launch_bounds__(512) softargmax_bhwn_kernel(const T* __restrict__ logits, float* __restrict__ out2d,
                                                              float* __restrict__ out3d, int J, int D, int H, int W,
                                                              int ld, DecodeScale sc) {
  extern __shared__ float sm[];  // [N][4] per-channel (m, s, sx, sy) + [PY][128][4] merge scratch
  const int N = HEAD3D ? J * D : J * (1 + D);
  const int P = H * W;
  const int b = blockIdx.x;
  const int cx = threadIdx.x & 127, py = threadIdx.x >> 7;  // 128 x 4
  constexpr int PY = 4;
  constexpr float L2E = 1.4426950408889634f;
  float4* chan = reinterpret_cast<float4*>(sm);
  float4* scratch = chan + N;
  const T* base = logits + (size_t)b * P * ld;  // ld >= N: row stride (head channels padded to 4)
  for (int n0 = 0; n0 < N; n0 += 128) {
    int n = n0 + cx;
    float m = -INFINITY, s = 0.f, sx = 0.f, sy = 0.f;
    if (n < N) {
      for (int p = py; p < P; p += PY) {
        float v = load1<T>(base + (size_t)p * ld + n);
        int y = p / W, x = p - y * W;
        if (v > m) {
          float f = exp2f((m - v) * L2E);
          s *= f; sx *= f; sy *= f;
          m = v;
        }
        float e = exp2f((v - m) * L2E);
        s += e;
        sx = fmaf(e, (float)x, sx);
        sy = fmaf(e, (float)y, sy);
      }
    }
    scratch[py * 128 + cx] = make_float4(m, s, sx, sy);
    __syncthreads();
    if (py == 0 && n < N) {
      SoftState a;
      a.m = m; a.s = s; a.sx = sx; a.sy = sy; a.sz = 0.f;
      for (int q = 1; q < PY; ++q) {
        float4 o = scratch[q * 128 + cx];
        SoftState bb;
        bb.m = o.x; bb.s = o.y; bb.sx = o.z; bb.sy = o.w; bb.sz = 0.f;
        soft_merge(a, bb);
      }
      chan[n] = make_float4(a.m, a.s, a.sx, a.sy);
    }
    __syncthreads();
  }
  for (int j = threadIdx.x; j < J; j += blockDim.x) {
    if constexpr (HEAD3D) {
      SoftState a;
      soft_init(a);
      for (int d = 0; d < D; ++d) {
        float4 c = chan[d * J + j];
        SoftState bb;
        bb.m = c.x; bb.s = c.y; bb.sx = c.z; bb.sy = c.w; bb.sz = c.y * (float)d;
        soft_merge(a, bb);
      }
      const float x = fmaf(soft_coord_tf(a.sx, a.s, W), sc.met_mul, sc.met_add);
      const float y = fmaf(soft_coord_tf(a.sy, a.s, H), sc.met_mul, sc.met_add);
      const float z = soft_coord_tf(a.sz, a.s, D) * sc.z_mul;
      out3d[((size_t)b * J + j) * 3 + 0] = x;
      out3d[((size_t)b * J + j) * 3 + 1] = y;
      out3d[((size_t)b * J + j) * 3 + 2] = z;
      if (out2d) {
        out2d[((size_t)b * J + j) * 2 + 0] = x;
        out2d[((size_t)b * J + j) * 2 + 1] = y;
      }
      continue;
    }
    if (out2d) {
      float4 c = chan[j];
      float x = soft_coord(c.z, c.y, W), y = soft_coord(c.w, c.y, H);
      if (sc.apply) {
        x = fmaf(x, sc.img_mul, sc.img_add);
        y = fmaf(y, sc.img_mul, sc.img_add);
      }
      out2d[((size_t)b * J + j) * 2 + 0] = x;
      out2d[((size_t)b * J + j) * 2 + 1] = y;
    }
    if (out3d && D > 0) {
      SoftState a;
      soft_init(a);
      for (int d = 0; d < D; ++d) {
        float4 c = chan[J + d * J + j];
        SoftState bb;
        bb.m = c.x; bb.s = c.y; bb.sx = c.z; bb.sy = c.w; bb.sz = c.y * (float)d;
        soft_merge(a, bb);
      }
      float x = soft_coord(a.sx, a.s, W), y = soft_coord(a.sy, a.s, H), z = soft_coord(a.sz, a.s, D);
      if (sc.apply) {
        x = fmaf(x, sc.met_mul, sc.met_add);
        y = fmaf(y, sc.met_mul, sc.met_add);
        z = z * sc.z_mul;
      }
      out3d[((size_t)b * J + j) * 3 + 0] = x;
      out3d[((size_t)b * J + j) * 3 + 1] = y;
      out3d[((size_t)b * J + j) * 3 + 2] = z;
    }
  }
}

// ----------------------------------------------------------------------------------------------------------
// reconstruct_absolute (ptu3d.py:9-33).  Two launches because reconstruct_ref_fullpersp normalises with
// BATCH-GLOBAL RMS scalars (ptu3d.py:71-74):
//   pass 1 (grid B): K^-1, normalized 2D, per-crop sums of n2d^2 and (n2d*z_rel - xy_rel)^2 -> partial[B][2] (fp64)
//   pass 2 (grid B): every CTA reduces partial[] in a fixed order (deterministic), then one warp per crop builds
//   the 3x3 weighted ridge normal equations in fp64, solves, un-scales, back-projects and mixes.
// ----------------------------------------------------------------------------------------------------------
struct ReconParams {
  const float* c2d;   // [B,J,2]
  const float* c3d;   // [B,J,3]
  const float* K;     // [B,3,3]
  float* out;         // [B,J,3]
  double* partial;    // [B][2]
  float* n2d;         // [B,J,2] scratch
  int B, J;
  float fov_lower, fov_upper, mix;
  int use_mix;
};

__device__ __forceinline__ void inv3x3(const float* k, float* inv) {
  // fp64 closed form of torch.linalg.inv for a 3x3 (ptu3d.py:12)
  double a = k[0], b = k[1], c = k[2], d = k[3], e = k[4], f = k[5], g = k[6], h = k[7], i = k[8];
  double A = e * i - f * h, Bc = -(d * i - f * g), C = d * h - e * g;
  double det = a * A + b * Bc + c * C;
  double r = 1.0 / det;
  inv[0] = (float)(A * r);  inv[1] = (float)(-(b * i - c * h) * r); inv[2] = (float)((b * f - c * e) * r);
  inv[3] = (float)(Bc * r); inv[4] = (float)((a * i - c * g) * r);  inv[5] = (float)(-(a * f - c * d) * r);
  inv[6] = (float)(C * r);  inv[7] = (float)(-(a * h - b * g) * r); inv[8] = (float)((a * e - b * d) * r);
}

__global__ void __launch_bounds__(128) recon_pass1_kernel(ReconParams p) {
  const int b = blockIdx.x;
  __shared__ float kinv[9];
  __shared__ double red[4][2];
  if (threadIdx.x == 0) inv3x3(p.K + (size_t)b * 9, kinv);
  __syncthreads();
  double s2d = 0.0, sb = 0.0;
  for (int j = threadIdx.x; j < p.J; j += blockDim.x) {
    float x = p.c2d[((size_t)b * p.J + j) * 2 + 0], y = p.c2d[((size_t)b * p.J + j) * 2 + 1];
    // (to_homogeneous(c2d) @ Kinv^T)[..., :2]  (ptu3d.py:13)
    float nx = x * kinv[0] + y * kinv[1] + kinv[2];
    float ny = x * kinv[3] + y * kinv[4] + kinv[5];
    p.n2d[((size_t)b * p.J + j) * 2 + 0] = nx;
    p.n2d[((size_t)b * p.J + j) * 2 + 1] = ny;
    float rx = p.c3d[((size_t)b * p.J + j) * 3 + 0], ry = p.c3d[((size_t)b * p.J + j) * 3 + 1],
          rz = p.c3d[((size_t)b * p.J + j) * 3 + 2];
    float bx = nx * rz - rx, by = ny * rz - ry;  // rel_backproj (ptu3d.py:89)
    s2d += (double)nx * nx + (double)ny * ny;
    sb += (double)bx * bx + (double)by * by;
  }
  s2d = warp_sum(s2d);
  sb = warp_sum(sb);
  if ((threadIdx.x & 31) == 0) {
    red[threadIdx.x >> 5][0] = s2d;
    red[threadIdx.x >> 5][1] = sb;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0, c = 0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { a += red[i][0]; c += red[i][1]; }
    p.partial[(size_t)b * 2 + 0] = a;
    p.partial[(size_t)b * 2 + 1] = c;
  }
}

__global__ void __launch_bounds__(128) recon_pass2_kernel(ReconParams p) {
  const int b = blockIdx.x;
  __shared__ double red[4][9 + 3];
  __shared__ double tot[2];
  __shared__ float ref[3];
  // batch-global sums, fixed order
  double a = 0, c = 0;
  for (int i = threadIdx.x; i < p.B; i += blockDim.x) { a += p.partial[(size_t)i * 2]; c += p.partial[(size_t)i * 2 + 1]; }
  a = warp_sum(a);
  c = warp_sum(c);
  if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5][0] = a; red[threadIdx.x >> 5][1] = c; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double x = 0, y = 0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { x += red[i][0]; y += red[i][1]; }
    tot[0] = x; tot[1] = y;
  }
  __syncthreads();
  const double cnt = (double)p.B * p.J * 2;
  const float scale2d = (float)sqrt(tot[0] / cnt);  // rms_normalize (ptu3d.py:71-74)
  const float scaleb = (float)sqrt(tot[1] / cnt);
  // normal equations of the weighted system: rows [1,0,-x~; 0,1,-y~] * w, rhs b~ * w, plus 0.1*I ridge rows
  double n[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) n[i] = 0.0;
  for (int j = threadIdx.x; j < p.J; j += blockDim.x) {
    size_t o = (size_t)b * p.J + j;
    float px = p.c2d[o * 2], py = p.c2d[o * 2 + 1];
    bool infov = px >= p.fov_lower && px <= p.fov_upper && py >= p.fov_lower && py <= p.fov_upper;
    float nx = p.n2d[o * 2], ny = p.n2d[o * 2 + 1];
    float rx = p.c3d[o * 3], ry = p.c3d[o * 3 + 1], rz = p.c3d[o * 3 + 2];
    float w = (infov ? 1.0f : 0.0f) + 1e-4f;
    double w2 = (double)w * w;
    double xt = (double)(nx / scale2d), yt = (double)(ny / scale2d);
    double bx = (double)((nx * rz - rx) / scaleb), by = (double)((ny * rz - ry) / scaleb);
    // A^T W^2 A (symmetric: 00 01 02 11 12 22) and A^T W^2 b
    n[0] += w2;            // (0,0)
    n[2] += -w2 * xt;      // (0,2)
    n[4] += w2;            // (1,1)
    n[5] += -w2 * yt;      // (1,2)
    n[8] += w2 * (xt * xt + yt * yt);  // (2,2)
    n[9] += w2 * bx;
    n[10] += w2 * by;
    n[11] += -w2 * (xt * bx + yt * by);
  }
#pragma unroll
  for (int i = 0; i < 12; ++i) n[i] = warp_sum(n[i]);
  __syncthreads();
  if ((threadIdx.x & 31) == 0)
    for (int i = 0; i < 12; ++i) red[threadIdx.x >> 5][i] = n[i];
  __syncthreads();
  if (threadIdx.x == 0) {
    double s[12];
    for (int i = 0; i < 12; ++i) {
      s[i] = 0;
      for (int q = 0; q < (int)(blockDim.x >> 5); ++q) s[i] += red[q][i];
    }
    const double lam = 1e-2;  // (sqrt(1e-2))^2, ptu3d.py:96-98
    double a00 = s[0] + lam, a02 = s[2], a11 = s[4] + lam, a12 = s[5], a22 = s[8] + lam;
    double b0 = s[9], b1 = s[10], b2 = s[11];
    // a01 = 0.  Eliminate r0, r1:  r0 = (b0 - a02 r2)/a00, r1 = (b1 - a12 r2)/a11
    double den = a22 - a02 * a02 / a00 - a12 * a12 / a11;
    double r2 = (b2 - a02 * b0 / a00 - a12 * b1 / a11) / den;
    double r0 = (b0 - a02 * r2) / a00, r1 = (b1 - a12 * r2) / a11;
    ref[0] = (float)r0 * scaleb;                  // ptu3d.py:103-104
    ref[1] = (float)r1 * scaleb;
    ref[2] = (float)r2 * (scaleb / scale2d);
  }
  __syncthreads();
  for (int j = threadIdx.x; j < p.J; j += blockDim.x) {
    size_t o = (size_t)b * p.J + j;
    float px = p.c2d[o * 2], py = p.c2d[o * 2 + 1];
    bool infov = px >= p.fov_lower && px <= p.fov_upper && py >= p.fov_lower && py <= p.fov_upper;
    float nx = p.n2d[o * 2], ny = p.n2d[o * 2 + 1];
    float rx = p.c3d[o * 3], ry = p.c3d[o * 3 + 1], rz = p.c3d[o * 3 + 2];
    float a3x = rx + ref[0], a3y = ry + ref[1], a3z = rz + ref[2];
    float zz = rz + ref[2];
    float a2x = nx * zz, a2y = ny * zz, a2z = zz;  // back_project (ptu3d.py:108-110)
    if (p.use_mix) {
      a2x = p.mix * a3x + (1.f - p.mix) * a2x;
      a2y = p.mix * a3y + (1.f - p.mix) * a2y;
      a2z = p.mix * a3z + (1.f - p.mix) * a2z;
    }
    p.out[o * 3 + 0] = infov ? a2x : a3x;
    p.out[o * 3 + 1] = infov ? a2y : a3y;
    p.out[o * 3 + 2] = infov ? a2z : a3z;
  }
}

// ----------------------------------------------------------------------------------------------------------
// reconstruct_absolute_by_bone_lengths (metrabs_tf/tfu3d.py:219-269), the absolute step of Model25D: coords25d [B,J,3] =
// (x px, y px, z mm) -> camera-space joints [B,J,3].  Per crop b, with n2d = ([x, y, 1] K^-1^T)[:2], z_rel = z - mean_j z
// (or z - z[J-1]), x_j = [n2d_j, 1] and per bone e = (i, j):  a = x_i - x_j, bv = x_i z_rel_i - x_j z_rel_j, c = |a|^2,
// d = 2 a.bv, e = |bv|^2, w = (in_fov_i && in_fov_j) + 1e-8, the residual r_e(z) = (sqrt(z^2 c + z d + e) - L_e) w.
// tensorflow_graphics' Levenberg-Marquardt minimises sum_b sum_e r^2 over the z of the WHOLE batch from 1500 / projected
// size: its Jacobian [B*E, B] is block-diagonal, so each step is per crop z -= sum_e J r / (sum_e J^2 + lam), and the step
// is taken for every crop iff the batch objective decreases, else lam *= 10 (lam starts at 1e-20; 10 iterations).  The
// accept decision couples the crops, so one CTA runs the whole solve: a warp per crop (crops strided over the warps), the
// per-crop sums as fixed warp butterflies, the batch sums over crops in ascending order per thread and then over threads in
// a fixed tree.  No atomics: the result is bit-identical from run to run.
// ----------------------------------------------------------------------------------------------------------
struct BoneSolveParams {
  const float* c25;   // [B,J,3]
  const float* K;     // [B,3,3]
  const int2* edges;  // [E] joint pairs
  const float* len;   // [E] ideal bone lengths, mm
  float* out;         // [B,J,3]
  float4* coef;       // [B][E] scratch: (c, d, e, w) per bone
  float* z;           // [B] scratch: the accepted z_ref
  float* z_new;       // [B] scratch: the candidate of this iteration
  float* obj;         // [B] scratch: per-crop objective of the candidate (before the loop: of the initial guess)
  int B, J, E;
  float fov_lower, fov_upper;
  int mean_relative;
};
constexpr int BONE_THREADS = 512;
constexpr int BONE_ITERS = 10;

// K^-1 and the centre of z (mean over the joints, or the last joint) of crop b; identical in every lane of the warp
__device__ __forceinline__ void bone_crop_setup(const BoneSolveParams& p, int b, int lane, float* kinv, float& zc) {
  inv3x3(p.K + (size_t)b * 9, kinv);
  const float* c = p.c25 + (size_t)b * p.J * 3;
  if (p.mean_relative) {
    float s = 0.f;
    for (int j = lane; j < p.J; j += 32) s += c[j * 3 + 2];
    zc = warp_sum(s) / (float)p.J;
  } else {
    zc = c[(p.J - 1) * 3 + 2];
  }
}

__device__ __forceinline__ float bone_residual(float4 q, float L, float z) {
  return (sqrtf(z * z * q.x + z * q.y + q.z) - L) * q.w;
}

// sum of v[0..n) in ascending order per thread, then a fixed tree over the CTA (every thread gets the total)
__device__ __forceinline__ float bone_block_sum(const float* v, int n, float* red) {
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += BONE_THREADS) s += v[i];
  s = warp_sum(s);
  __syncthreads();  // red[] is reused by consecutive calls
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  float t = 0.f;
  for (int w = 0; w < BONE_THREADS / 32; ++w) t += red[w];
  return t;
}

__global__ void __launch_bounds__(BONE_THREADS) bone_solve_kernel(BoneSolveParams p) {
  __shared__ float red[BONE_THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int n_warps = BONE_THREADS / 32;
  // pass 1: bone coefficients, initial guess and its objective
  for (int b = warp; b < p.B; b += n_warps) {
    float kinv[9], zc;
    bone_crop_setup(p, b, lane, kinv, zc);
    const float* c = p.c25 + (size_t)b * p.J * 3;
    float lox = INFINITY, hix = -INFINITY, loy = INFINITY, hiy = -INFINITY;
    for (int j = lane; j < p.J; j += 32) {
      const float x = c[j * 3], y = c[j * 3 + 1];
      const float nx = x * kinv[0] + y * kinv[1] + kinv[2], ny = x * kinv[3] + y * kinv[4] + kinv[5];
      lox = fminf(lox, nx); hix = fmaxf(hix, nx);
      loy = fminf(loy, ny); hiy = fmaxf(hiy, ny);
    }
    lox = -warp_max(-lox); loy = -warp_max(-loy);
    hix = warp_max(hix); hiy = warp_max(hiy);
    const float guess = 1500.f / fmaxf(hix - lox, hiy - loy);
    float r2 = 0.f;
    for (int e = lane; e < p.E; e += 32) {
      const int2 ij = p.edges[e];
      float n[2][2], zr[2];
      bool fov[2];
      for (int k = 0; k < 2; ++k) {
        const float* q = c + (k == 0 ? ij.x : ij.y) * 3;
        n[k][0] = q[0] * kinv[0] + q[1] * kinv[1] + kinv[2];
        n[k][1] = q[0] * kinv[3] + q[1] * kinv[4] + kinv[5];
        zr[k] = q[2] - zc;
        fov[k] = q[0] >= p.fov_lower && q[0] <= p.fov_upper && q[1] >= p.fov_lower && q[1] <= p.fov_upper;
      }
      const float ax = n[0][0] - n[1][0], ay = n[0][1] - n[1][1];  // the homogeneous components cancel
      const float bx = n[0][0] * zr[0] - n[1][0] * zr[1], by = n[0][1] * zr[0] - n[1][1] * zr[1], bz = zr[0] - zr[1];
      const float4 q = make_float4(ax * ax + ay * ay, 2.f * (ax * bx + ay * by), bx * bx + by * by + bz * bz,
                                   (fov[0] && fov[1] ? 1.f : 0.f) + 1e-8f);
      p.coef[(size_t)b * p.E + e] = q;
      const float r = bone_residual(q, p.len[e], guess);
      r2 += r * r;
    }
    r2 = warp_sum(r2);
    if (lane == 0) {
      p.z[b] = guess;
      p.obj[b] = r2;
    }
  }
  __syncthreads();
  float total = bone_block_sum(p.obj, p.B, red);
  float lam = 1e-20f;
  for (int it = 0; it < BONE_ITERS; ++it) {
    for (int b = warp; b < p.B; b += n_warps) {
      const float z = p.z[b];
      const float4* q = p.coef + (size_t)b * p.E;
      float jr = 0.f, jj = 0.f;
      for (int e = lane; e < p.E; e += 32) {
        const float4 c = q[e];
        const float s = sqrtf(z * z * c.x + z * c.y + c.z);
        const float r = (s - p.len[e]) * c.w;
        const float jac = c.w * (2.f * z * c.x + c.y) / (2.f * s);
        jr += jac * r;
        jj += jac * jac;
      }
      const float zn = z - warp_sum(jr) / (warp_sum(jj) + lam);
      float r2 = 0.f;
      for (int e = lane; e < p.E; e += 32) {
        const float r = bone_residual(q[e], p.len[e], zn);
        r2 += r * r;
      }
      r2 = warp_sum(r2);
      if (lane == 0) {
        p.z_new[b] = zn;
        p.obj[b] = r2;
      }
    }
    __syncthreads();
    const float total_new = bone_block_sum(p.obj, p.B, red);
    if (total_new < total) {  // the same decision in every thread
      total = total_new;
      for (int b = threadIdx.x; b < p.B; b += BONE_THREADS) p.z[b] = p.z_new[b];
    } else {
      lam *= 10.f;
    }
    __syncthreads();
  }
  // back_project (tfu3d.py:200-201): [n2d, 1] * (z_rel + z_ref)
  for (int b = warp; b < p.B; b += n_warps) {
    float kinv[9], zc;
    bone_crop_setup(p, b, lane, kinv, zc);
    const float zref = p.z[b];
    const float* c = p.c25 + (size_t)b * p.J * 3;
    float* o = p.out + (size_t)b * p.J * 3;
    for (int j = lane; j < p.J; j += 32) {
      const float x = c[j * 3], y = c[j * 3 + 1];
      const float nx = x * kinv[0] + y * kinv[1] + kinv[2], ny = x * kinv[3] + y * kinv[4] + kinv[5];
      const float zz = (c[j * 3 + 2] - zc) + zref;
      o[j * 3 + 0] = nx * zz;
      o[j * 3 + 1] = ny * zz;
      o[j * 3 + 2] = zz;
    }
  }
}

// tfu3d.linear_combine_points (metrabs_tf/tfu3d.py:48-49): out[b,J',c] = sum_l pts[b,l,c] * w[l,J'].  Grid (B, ceil(n_out/128)),
// 128 threads; the CTA stages its crop's [L,3] points in shared memory (dynamic, L*3 floats), each thread owns one output point
// and accumulates in fp32 with l ascending, reading w[l*n_out + j] coalesced across the warp.
__global__ void __launch_bounds__(128) combine_points_kernel(const float* __restrict__ pts, const float* __restrict__ w,
                                                             float* __restrict__ out, int L, int n_out) {
  extern __shared__ float sp[];
  const int b = blockIdx.x;
  const float* src = pts + (size_t)b * L * 3;
  for (int i = threadIdx.x; i < L * 3; i += blockDim.x) sp[i] = src[i];
  __syncthreads();
  const int j = blockIdx.y * blockDim.x + threadIdx.x;
  if (j >= n_out) return;
  float x = 0.f, y = 0.f, z = 0.f;
  for (int l = 0; l < L; ++l) {
    const float wl = __ldg(w + (size_t)l * n_out + j);
    x = fmaf(sp[l * 3 + 0], wl, x);
    y = fmaf(sp[l * 3 + 1], wl, y);
    z = fmaf(sp[l * 3 + 2], wl, z);
  }
  float* o = out + ((size_t)b * n_out + j) * 3;
  o[0] = x;
  o[1] = y;
  o[2] = z;
}

}  // namespace mtb
