// 3xTF32 tensor-core path (sm_90a): the PARITY mode on wgmma.  fp32 NHWC activations and fp32 weights are staged by TMA
// exactly as they sit in HBM; each consumer warpgroup rewrites ITS 64 rows of every landed A tile in shared memory as
//     x_hi = tf32(x)  (round to nearest, low 13 mantissa bits zero)      x_lo = x - x_hi  (exact in fp32)
// (the weights arrive split: hi and lo planes prepared on the host) and issues, per K step of 8, three wgmma kind tf32
// products:
//     P += A_hi * B_hi          S += A_lo * B_hi          S += A_hi * B_lo
// into TWO kinds of register accumulators.  Why two: the tensor core's fp32 accumulate TRUNCATES (round toward zero), so a
// long accumulation chain carries a bias that grows linearly with K - one accumulator for everything lands above the 1e-3
// bar on EfficientNetV2-S features.  The cure is the one of Ootomo & Yokota (2022, "Recovering single precision accuracy
// from Tensor Cores"): accumulate OUTSIDE the tensor core.  The main term runs in short chains of T32_CHAIN k-blocks into a
// partial accumulator P that is added to the fp32 accumulator with round-to-nearest FADDs; the correction terms are 2^-11 of
// the main term, so their truncation error is negligible and they keep one accumulator S for the whole tile.
//
//   mode 0   1x1 stride-1 conv == GEMM  D[pixels, Cout] = A[pixels, Cin] * W[Cout, Cin]^T (2D TMA); the squeeze-excitation
//            scale of an MBConv projection (backbones/efficientnet.py:110-173, `scale * x`) is applied to the A tile before
//            the split: the separate scaling pass of the bf16 mode does not exist here
//   mode 1   RxS conv (stride 1/2, dilation) as implicit GEMM: per tap the A tile is a shifted [8 x 16] pixel box of the
//            NHWC input fetched by a 4D TMA; out-of-bounds = the reference's explicit zero padding (efficientnet.py:1127-1161)
//   epilogue registers -> + folded-BN bias, exact activation, + residual, fp32 NHWC store.
//
// Tiles: M = 128 pixels x N = BN <= 64 channels.  Shared-memory stage: [A raw/hi 128 rows | B hi BN rows | A lo | B lo],
// rows of 128 bytes (32 fp32, 128B swizzle).  The lo tile mirrors the raw tile byte for byte, so the split never needs to
// undo the TMA swizzle.
#pragma once
#include "tc_gemm.cuh"

namespace mtb {

constexpr int T32_RB = 128;       // bytes per operand row (32 fp32)
constexpr int T32_BK = T32_RB / 4;
constexpr int T32_CHAIN = 2;      // k-blocks (8 MMAs of the main term) per partial chain

template <int BN>
struct T32Ring {
  static constexpr int lo_off = (TC_BM + BN) * T32_RB;
  static constexpr int stage_bytes = 2 * lo_off;
  static constexpr int stages = 4;
  static constexpr int smem_bytes = stages * stage_bytes + 1024 /*align slack*/ + 256 /*barriers*/;
};

struct Tc32Params {
  const float* res;
  const float* bias;
  float* out;
  const float* a_scale;  // mode 0: squeeze-excitation scale [B][Cin] applied to A before the split (nullptr: none)
  int a_scale_P;         // pixels per crop
  int mode;              // 0 flat 1x1 stride 1; 1 spatial tiles (4D TMA per tap)
  int Hin, Win;
  int M;                 // mode 0: rows
  int Cout, Cin;
  int kchunks, taps;
  int Hout, Wout, tiles_w, tiles_h, pad_t, pad_l, S, stride, dil;
};

// hi = x rounded to tf32 (nearest, ties away: integer add on the bit pattern, carries into the exponent correctly),
// lo = x - hi (exact: hi and x agree in sign/exponent up to one binade, the difference has <= 13 significant bits)
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  hi = __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u);
  lo = x - hi;
}

// explicit shared-window 16-byte accesses (a generic pointer into dynamic shared memory compiles to LD.E / ST.E)
__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, const float4& v) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
// SiLU for the parity epilogue: x * 1/(1 + 2^(-x log2 e)) on the MUFU units (ex2.approx, rcp.approx: ~2 ulp each); the
// CUDA-core fp32 mode's expf + IEEE division costs ~3x the instructions and sat on the accumulator warps' critical path
template <int ACT>
__device__ __forceinline__ float t32_act(float x) {
  if constexpr (ACT == ACT_SILU) {
    float e, r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
    return x * r;
  } else {
    return act_t<ACT>(x);
  }
}

// Splits the 16-byte chunks first, first + step, ... (< end) of the A tile of one stage: raw fp32 -> hi in place + lo in the
// mirror tile; with `sc` the squeeze-excitation scale s[crop(row)][k..k+3] is applied first (mode 0).  The TMA swizzle puts
// logical chunk j ^ swz(r) at physical position j of row r (128B swizzle: swz = r & 7; 64B swizzle: swz = (r >> 1) & 3).
template <int RB>
__device__ __forceinline__ void t32_split_a(uint32_t base, uint32_t lo_off, int first, int end, int step, const float* __restrict__ sc,
                                            int m_row0, int M, int P, int Cin, int k0) {
  constexpr int CPR = RB / 16;
  if (sc != nullptr) {
    int last_key = -1;
    float4 s4 = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 2
    for (int i = first; i < end; i += step) {
      float4 v = lds128(base + i * 16);
      const int r = i / CPR, j = i - r * CPR;
      const int swz = RB == 128 ? (r & 7) : ((r >> 1) & 3);
      const int k = k0 + ((j ^ swz) << 2);
      const int m = m_row0 + r;
      if (m < M && k < Cin) {
        const int crop = m / P;
        const int key = crop * 8 + swz;
        if (key != last_key) {  // the scale vector is re-read only when the crop (or the swizzled K offset) changes
          s4 = __ldg(reinterpret_cast<const float4*>(sc + (size_t)crop * Cin + k));
          last_key = key;
        }
        v.x *= s4.x; v.y *= s4.y; v.z *= s4.z; v.w *= s4.w;
      }
      float4 h, l;
      split_tf32(v.x, h.x, l.x);
      split_tf32(v.y, h.y, l.y);
      split_tf32(v.z, h.z, l.z);
      split_tf32(v.w, h.w, l.w);
      sts128(base + i * 16, h);
      sts128(base + lo_off + i * 16, l);
    }
  } else {
#pragma unroll 4
    for (int i = first; i < end; i += step) {
      const float4 v = lds128(base + i * 16);
      float4 h, l;
      split_tf32(v.x, h.x, l.x);
      split_tf32(v.y, h.y, l.y);
      split_tf32(v.z, h.z, l.z);
      split_tf32(v.w, h.w, l.w);
      sts128(base + i * 16, h);
      sts128(base + lo_off + i * 16, l);
    }
  }
}

template <int ACT, int RES, int BN>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc32_conv_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const Tc32Params p) {
  using Ring = T32Ring<BN>;
  constexpr int STAGES = Ring::stages;
  constexpr int NR = BN / 2;  // accumulator registers per thread
  extern __shared__ uint8_t tc_smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)tc_smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* full = (uint64_t*)(smem + STAGES * Ring::stage_bytes);
  uint64_t* empty = full + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == TC_CONSUMER_WARPS * 32) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], TC_CONSUMER_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int m_blk = blockIdx.x, n_blk = blockIdx.y;
  const int num_kb = p.taps * p.kchunks;
  if (warp == TC_CONSUMER_WARPS) {
    // ===== TMA producer: A raw, weights hi plane (rows [0, Cout)) and lo plane (rows [Cout, 2 Cout)) =====
    if (lane == 0) {
      for (int kb = 0; kb < num_kb; ++kb) {
        const int s = kb % STAGES;
        mbar_wait(&empty[s], ((kb / STAGES) & 1) ^ 1);
        uint8_t* sa = smem + s * Ring::stage_bytes;
        const int tap = kb / p.kchunks, kc = kb - tap * p.kchunks;
        mbar_expect_tx(&full[s], (TC_BM + 2 * BN) * T32_RB);
        tma_load_a_tile<T32_BK>(sa, &tmA, &full[s], p, m_blk, kb);
        tma_load_2d(sa + TC_BM * T32_RB, &tmB, &full[s], tap * p.Cin + kc * T32_BK, n_blk * BN);
        tma_load_2d(sa + Ring::lo_off + TC_BM * T32_RB, &tmB, &full[s], tap * p.Cin + kc * T32_BK, p.Cout + n_blk * BN);
      }
    }
    return;
  }
  // ===== consumers: warpgroup wg splits and multiplies tile rows [64 wg, +64) =====
  const int wg = warp >> 2, tid = threadIdx.x & 127;
  constexpr int CPR = T32_RB / 16;  // 16-byte chunks per row
  float acc[NR], pacc[NR], sacc[NR];
#pragma unroll
  for (int i = 0; i < NR; ++i) acc[i] = pacc[i] = sacc[i] = 0.f;
  int pos = 0;
  for (int kb = 0; kb < num_kb; ++kb) {
    const int s = kb % STAGES;
    mbar_wait(&full[s], (kb / STAGES) & 1);
    const uint32_t base = smem_u32(smem + s * Ring::stage_bytes);
    const int kc = kb % p.kchunks;
    t32_split_a<T32_RB>(base, (uint32_t)Ring::lo_off, wg * 64 * CPR + tid, (wg + 1) * 64 * CPR, 128, p.a_scale, m_blk * TC_BM, p.M,
                        p.a_scale_P, p.Cin, kc * T32_BK);
    fence_proxy_async();  // generic-proxy writes -> visible to the tensor core (async proxy)
    wg_sync(wg);
    const uint32_t a_hi = base + wg * 64 * T32_RB, b_hi = base + TC_BM * T32_RB;
    const uint32_t a_lo = a_hi + Ring::lo_off, b_lo = b_hi + Ring::lo_off;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < T32_RB / 32; ++k) {
      wgmma_tf32<BN>(sacc, gmma_desc<T32_RB>(a_lo + 32 * k), gmma_desc<T32_RB>(b_hi + 32 * k), (uint32_t)(kb | k));
      wgmma_tf32<BN>(sacc, gmma_desc<T32_RB>(a_hi + 32 * k), gmma_desc<T32_RB>(b_lo + 32 * k), 1u);
      wgmma_tf32<BN>(pacc, gmma_desc<T32_RB>(a_hi + 32 * k), gmma_desc<T32_RB>(b_hi + 32 * k), (uint32_t)(pos | k));
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs<NR>(pacc);
    wgmma_fence_regs<NR>(sacc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);
    if (pos == T32_CHAIN - 1 || kb == num_kb - 1) {
#pragma unroll
      for (int i = 0; i < NR; ++i) acc[i] += pacc[i];
      pos = 0;
    } else {
      ++pos;
    }
  }
#pragma unroll
  for (int i = 0; i < NR; ++i) acc[i] += sacc[i];

  // ===== epilogue: thread rows r0 = 64 wg + 16 (warp & 3) + lane / 4 and r0 + 8, columns 8 j + 2 (lane % 4) + {0, 1} =====
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  // The bias pairs and both rows' residual pairs are loaded in one batch before the first store: loaded between the stores,
  // which might alias them, each load waited out its latency before the next one was issued.
  const int c0 = n_blk * BN + 2 * (lane & 3);
  float2 bv[BN / 8], rv2[RES != 0 ? 2 : 1][BN / 8];
  size_t off[2];
  bool row_ok[2];
#pragma unroll
  for (int j = 0; j < BN / 8; ++j)
    if (c0 + 8 * j < p.Cout) bv[j] = __ldg(reinterpret_cast<const float2*>(p.bias + c0 + 8 * j));
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    row_ok[h] = tile_row_offset(p.mode, m_blk, r0 + 8 * h, p.M, p.Cout, p.tiles_w, p.tiles_h, p.Hout, p.Wout, off[h]);
    if constexpr (RES != 0) {
      if (row_ok[h]) {
#pragma unroll
        for (int j = 0; j < BN / 8; ++j)
          if (c0 + 8 * j < p.Cout) rv2[h][j] = *reinterpret_cast<const float2*>(p.res + off[h] + c0 + 8 * j);
      }
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (!row_ok[h]) continue;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int c = c0 + 8 * j;
      if (c >= p.Cout) break;  // Cout % 4 == 0: column c + 1 is valid with c
      float o0 = acc[4 * j + 2 * h] + bv[j].x, o1 = acc[4 * j + 2 * h + 1] + bv[j].y;
      if constexpr (RES != 0) {
        const float2 rv = rv2[h][j];
        if constexpr (RES == 2) {
          o0 = t32_act<ACT>(o0 + rv.x);
          o1 = t32_act<ACT>(o1 + rv.y);
        } else {
          o0 = t32_act<ACT>(o0) + rv.x;
          o1 = t32_act<ACT>(o1) + rv.y;
        }
      } else {
        o0 = t32_act<ACT>(o0);
        o1 = t32_act<ACT>(o1);
      }
      *reinterpret_cast<float2*>(p.out + off[h] + c) = make_float2(o0, o1);
    }
  }
}

// ------------------------------------------------------------------------------------------------ host side
struct Tc32Weights {
  bool ready = false;
  float* d_w = nullptr;     // fp32 [2][Cout][taps*Cin] K-major (BN folded): hi plane, lo plane
  float* d_bias = nullptr;  // [Cout]
  int Cout = 0, Cin = 0, taps = 1, S = 1;
  mutable TmapCache maps;   // (input, weights)
};

// wk: fp32 [K = taps*Cin][Cout] (BN folded) -> two K-major planes [2][Cout][K]: hi = tf32(w) (round to nearest, as
// split_tf32 on the device) and lo = w - hi (exact in fp32)
inline const char* tc32_prepare_weights(Tc32Weights& w, const float* wk, const float* bias, int K, int cout, int R, int S, int cin,
                                        std::vector<void*>& allocs) {
  std::vector<float> t((size_t)2 * K * cout);
  for (int k = 0; k < K; ++k)
    for (int n = 0; n < cout; ++n) {
      const float x = wk[(size_t)k * cout + n];
      uint32_t u;
      memcpy(&u, &x, 4);
      u = (u + 0x1000u) & 0xffffe000u;
      float hi;
      memcpy(&hi, &u, 4);
      t[(size_t)n * K + k] = hi;
      t[(size_t)cout * K + (size_t)n * K + k] = x - hi;
    }
  const char* e = upload_dev(allocs, (void**)&w.d_w, t.data(), t.size() * 4);
  if (!e) e = upload_dev(allocs, (void**)&w.d_bias, bias, (size_t)cout * 4);
  if (e) return e;
  w.Cout = cout; w.Cin = cin; w.taps = R * S; w.S = S;
  w.ready = true;
  return nullptr;
}

// the 3xTF32 kernel takes what the bf16 tensor-core kernel takes, with fp32 alignment rules (16-byte TMA strides / stores)
inline bool tc32_eligible(bool is_conv, bool depthwise, bool small_io, int k, int stride, int cin, int cout) {
  if (!is_conv || depthwise || small_io) return false;
  if (cin % 4 != 0 || cout % 4 != 0) return false;
  return (stride == 1 || stride == 2) && (k == 1 || k == 3);
}

inline const char* tc32_conv_launch(const Tc32Weights& w, const ConvParams& p, bool res_first, cudaStream_t st) {
  Tc32Params q;
  q.res = (const float*)p.res; q.bias = w.d_bias; q.out = (float*)p.out;
  q.mode = (p.R == 1 && p.stride == 1) ? 0 : 1;
  q.a_scale = q.mode == 0 ? p.a_scale : nullptr;
  if (p.a_scale && q.mode != 0) return "squeeze-excitation scale on a spatial conv is not supported by the 3xTF32 kernel";
  q.a_scale_P = p.Hin * p.Win;
  q.Hin = p.Hin; q.Win = p.Win;
  q.Cout = p.Cout; q.Cin = p.Cin;
  q.taps = w.taps; q.S = w.S; q.stride = p.stride; q.dil = p.dil;
  q.Hout = p.Hout; q.Wout = p.Wout; q.pad_t = p.pad_t; q.pad_l = p.pad_l;
  q.tiles_w = (p.Wout + TC_TILE_W - 1) / TC_TILE_W;
  q.tiles_h = (p.Hout + TC_TILE_H - 1) / TC_TILE_H;
  q.M = p.B * p.Hout * p.Wout;
  q.kchunks = (p.Cin + T32_BK - 1) / T32_BK;
  const int m_tiles = q.mode == 0 ? (q.M + TC_BM - 1) / TC_BM : p.B * q.tiles_w * q.tiles_h;
  const int bn = p.Cout <= 32 ? 32 : 64;
  const CUtensorMap* m = nullptr;  // input, weights
  const char* e = w.maps.get(&m, [&](CUtensorMap* c) {
    const CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_128B;  // T32_BK fp32 = 128-byte rows
    const char* r = q.mode == 0 ? make_tmap_2d<float>(&c[0], p.in, q.M, p.Cin, TC_BM, T32_BK, sw)
                                : make_tmap_nhwc<float>(&c[0], p.in, p.B, p.Hin, p.Win, p.Cin, T32_BK, TC_TILE_W, TC_TILE_H, 1, p.stride, sw);
    return r ? r : make_tmap_2d<float>(&c[1], w.d_w, (uint64_t)2 * p.Cout, (uint64_t)w.taps * p.Cin, bn, T32_BK, sw);
  }, p.in, w.d_w, p.B, p.Hin, p.Win, p.Cin, p.Hout, p.Wout, p.Cout, w.taps, p.stride, bn);
  if (e) return e;
  const dim3 grid(m_tiles, (p.Cout + bn - 1) / bn);
  const int res_mode = p.res ? (res_first ? 2 : 1) : 0;
  return with_const<ACT_NONE, ACT_SILU, ACT_RELU, ACT_HSWISH>(p.act, "unsupported activation in the 3xTF32 epilogue", [&](auto act) {
    return with_const<0, 1, 2>(res_mode, "unsupported residual mode", [&](auto res) {
      return with_const<32, 64>(bn, "unsupported N tile", [&](auto bn_) {
        return launch_smem(tc32_conv_kernel<act, res, bn_>, grid, dim3(TC_THREADS), T32Ring<bn_>::smem_bytes, st, m[0], m[1], q);
      });
    });
  });
}

}  // namespace mtb
