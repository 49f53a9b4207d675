// Fused FusedMBConv block (backbones/efficientnet.py:176-234, expand_ratio != 1, stride 1):
//
//     y = x + BN2(conv1x1( SiLU(BN1(conv3x3(x))) ))            x: [B,H,W,Cin] bf16 or fp16 NHWC, expanded width Cexp = 4*Cin
//
// as ONE kernel: the 128-pixel x Cexp expanded tile never leaves the SM.  Per output tile (16 x 8 pixels, as mode 1 of
// tc_conv_kernel) and per chunk of 128 expanded channels:
//   GEMM-1  (3x3 expand, implicit GEMM)   acc1[128 x 128] = shifted input boxes x W1[chunk rows]^T
//   epilogue-1  acc1 -> + folded-BN bias -> SiLU -> bf16 / fp16 -> shared memory in the 128B-swizzled K-major operand layout:
//           it IS the A operand of GEMM-2 (channels >= Cexp are written as zeros)
//   GEMM-2  (1x1 projection)  acc2[128 x Cout] += A2 x W2[:, chunk]^T, the W2 slice travelling through the same TMA ring
// and after the last chunk epilogue-2: acc2 -> + bias -> + residual x -> 16-bit store.  Each consumer warpgroup owns 64 rows
// of the tile in both GEMMs, so the A2 hand-over needs only a warpgroup barrier.  The MMA sequence of every output element
// (tap-major K of GEMM-1, chunk-major K of GEMM-2, K = 16 per wgmma) and every rounding are those of the two-launch path
// (tc_conv_kernel twice, with the same activation form per element type), less the GEMM-1 steps that would only add exact
// zeros, so the fused block reproduces it.
//
// Persistent: one CTA per SM walks tiles t = blockIdx.x, blockIdx.x + gridDim.x, ...  The input of a tile is read once, as
// three column-shifted 16 x 10-pixel boxes per 64-channel k-chunk (tma_load_tap_boxes), kept resident across the tile's
// expanded-channel chunks; tap (r, s) of GEMM-1 is box s from pixel row r on.  The ring carries only weights: 16 KB stages
// holding a W1 block [128 expanded channels x 64] or one 64-channel half of the W2 slice [Cout x 64].  The producer streams
// the k-blocks of the CTA's whole tile sequence, and loads the next tile's boxes as soon as the last GEMM-1 of the current
// tile has read them, under its last epilogue-1, GEMM-2 and epilogue-2.
#pragma once
#include "tc_gemm.cuh"

namespace mtb {

constexpr int FMB_NC = 128;                                         // expanded channels per chunk (N of GEMM-1, K of GEMM-2)
constexpr int FMB_BOX_H = TC_TILE_H + 2;                            // the tile's 8 input rows and the row above and below
constexpr int FMB_BOX_BYTES = TC_TILE_W * FMB_BOX_H * TC_BK * 2;    // 20 KB (a multiple of 1024: every box is swizzle-aligned)
constexpr int FMB_W_BYTES = FMB_NC * TC_BK * 2;                     // ring stage: W1 block 16 KB, or W2 half BN2 x 128 B <= 16 KB
constexpr int FMB_A2_BYTES = TC_BM * FMB_NC * 2;  // two 16 KB swizzle tiles (expanded channels 0-63, 64-127 of the chunk)

// Shared memory per BN2 (= tc_pick_bn(Cout), Cout = Cin): [3 x kchunks boxes | ring | A2 | barriers].  Cin <= 64 is one
// 64-channel k-chunk (BN2 <= 64): 60 KB of boxes + 8 x 16 KB ring + 32 KB = 221 KB; Cin 72 to 96 is two (BN2 = 128): 120 KB
// of boxes + 4 x 16 KB + 32 KB = 216 KB.
template <int BN2>
struct FmbSmem {
  static constexpr int kchunks = BN2 == 128 ? 2 : 1;
  static constexpr int stages = BN2 == 128 ? 4 : 8;
  static constexpr int ring_off = 3 * kchunks * FMB_BOX_BYTES;
  static constexpr int a2_off = ring_off + stages * FMB_W_BYTES;
  static constexpr int bar_off = a2_off + FMB_A2_BYTES;
  static constexpr int smem_bytes = bar_off + 256 + 1024 /*align slack*/;
};

struct FmbParams {
  TcConvParams g;           // geometry of the 3x3 expand conv (mode 1); g.res = x (residual), g.out = block output, g.m_tiles tiles
  const float* bias1;       // [Cexp]
  int Cexp, nch, has_res;
};

// one committed group of GEMM-1: the first NK k16 steps of k-block kb (A tile at shared address a, W1 block at b)
template <typename T, int NK>
__device__ __forceinline__ void fmb_gemm1_kblock(float* acc1, uint32_t a, uint32_t b, int kb) {
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < NK; ++k) wgmma_16b<T, FMB_NC>(acc1, gmma_desc<128>(a + 32 * k), gmma_desc<128>(b + 32 * k), (uint32_t)(kb | k));
  wgmma_commit();
}

template <typename T, int BN2>
__global__ void __launch_bounds__(TC_THREADS, 1)
fmb_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW1, const __grid_constant__ CUtensorMap tmW2,
           const FmbParams p) {
  using L = FmbSmem<BN2>;
  constexpr int STAGES = L::stages, KCH = L::kchunks, NUM_KB = 9 * KCH;
  extern __shared__ uint8_t tc_smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)tc_smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* full = (uint64_t*)(smem + L::bar_off);
  uint64_t* empty = full + STAGES;
  uint64_t* box_full = empty + STAGES;
  uint64_t* box_empty = box_full + 1;
  const TcConvParams& g = p.g;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == TC_CONSUMER_WARPS * 32) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmW1);
    tma_prefetch_desc(&tmW2);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], TC_CONSUMER_WARPS);
    }
    mbar_init(box_full, 1);
    mbar_init(box_empty, TC_CONSUMER_WARPS);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == TC_CONSUMER_WARPS) {
    // ===== TMA producer: per tile the input boxes, then per chunk NUM_KB W1 blocks and the two W2 halves =====
    if (lane == 0) {
      int it = 0, n = 0;
      for (int t = blockIdx.x; t < g.m_tiles; t += gridDim.x, ++n) {
        mbar_wait(box_empty, (n & 1) ^ 1);
        mbar_expect_tx(box_full, 3 * KCH * FMB_BOX_BYTES);
#pragma unroll
        for (int kc = 0; kc < KCH; ++kc) tma_load_tap_boxes(smem + 3 * kc * FMB_BOX_BYTES, FMB_BOX_BYTES, &tmA, box_full, g, t, kc);
        for (int c = 0; c < p.nch; ++c) {
          for (int kb = 0; kb < NUM_KB + 2; ++kb, ++it) {
            const int s = it % STAGES;
            mbar_wait(&empty[s], ((it / STAGES) & 1) ^ 1);
            uint8_t* st = smem + L::ring_off + s * FMB_W_BYTES;
            if (kb < NUM_KB) {
              const int tap = kb / KCH, kc = kb - tap * KCH;
              mbar_expect_tx(&full[s], FMB_W_BYTES);
              tma_load_2d(st, &tmW1, &full[s], tap * g.Cin + kc * TC_BK, c * FMB_NC);
            } else {
              mbar_expect_tx(&full[s], BN2 * TC_BK * 2);
              tma_load_2d(st, &tmW2, &full[s], c * FMB_NC + (kb - NUM_KB) * TC_BK, 0);
            }
          }
        }
      }
    }
    return;
  }
  const int wg = warp >> 2;
  const uint32_t boxes = smem_u32(smem) + wg * 64 * 128, ring = smem_u32(smem + L::ring_off), a2 = smem_u32(smem + L::a2_off);
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // fragment rows r0, r0 + 8; columns 8 j + 2 (lane % 4) + {0, 1}
  typedef typename Pair16<T>::type T2;
  const T* __restrict__ res = (const T*)g.res;
  T* __restrict__ out = (T*)g.out;
  // k16 steps of the last k-chunk that hold input channels: KL_HI at Cin 24-32, 56-64 and 88-96 (BN2 = 32, 64, 128), one
  // fewer at Cin 16, 40-48 and 72-80.  The steps after them would multiply TMA zero fill only and add exact zeros, so they
  // are not issued (as tc_conv3x3s1_kernel issues K = CK per tap).
  constexpr int KL_HI = BN2 == 64 ? 4 : 2;
  const bool kl_hi = g.Cin - TC_BK * (KCH - 1) > 16 * (KL_HI - 1);
  int it = 0, n = 0;
  for (int t = blockIdx.x; t < g.m_tiles; t += gridDim.x, ++n) {
    float acc2[BN2 / 2];
#pragma unroll
    for (int i = 0; i < BN2 / 2; ++i) acc2[i] = 0.f;
    mbar_wait(box_full, n & 1);
    for (int c = 0; c < p.nch; ++c) {
      // ---- GEMM-1 ----
      float acc1[FMB_NC / 2];
#pragma unroll
      for (int i = 0; i < FMB_NC / 2; ++i) acc1[i] = 0.f;
      int prev = -1;
      for (int tap = 0; tap < 9; ++tap) {
        const int r = tap / 3, sx = tap - 3 * r;
#pragma unroll
        for (int kc = 0; kc < KCH; ++kc, ++it) {
          const int kb = tap * KCH + kc, s = it % STAGES;
          mbar_wait(&full[s], (it / STAGES) & 1);
          const uint32_t a = boxes + (uint32_t)(3 * kc + sx) * FMB_BOX_BYTES + (uint32_t)r * (TC_TILE_W * 128);
          const uint32_t b = ring + s * FMB_W_BYTES;
          if (kc + 1 < KCH) fmb_gemm1_kblock<T, TC_BK / 16>(acc1, a, b, kb);
          else if (kl_hi) fmb_gemm1_kblock<T, KL_HI>(acc1, a, b, kb);  // one uniform branch, in the last k-chunk only
          else fmb_gemm1_kblock<T, KL_HI - 1>(acc1, a, b, kb);
          wgmma_wait<1>();
          __syncwarp();
          if (prev >= 0) {
            if (lane == 0) mbar_arrive(&empty[prev]);
          } else if (c > 0 && lane == 0) {  // the previous chunk's GEMM-2 has retired: release its two W2 stages
            mbar_arrive(&empty[(it - 2) % STAGES]);
            mbar_arrive(&empty[(it - 1) % STAGES]);
          }
          prev = s;
        }
      }
      // ---- epilogue-1: + bias, SiLU, 16-bit -> A2 (this warpgroup's rows; 16-byte chunk j of row r at j ^ (r & 7)) ----
      // Column blocks of JB1 groups, the first block's bias pairs loaded while the last k-block's MMAs run.  A2 is written
      // with .shared stores: a generic store might alias global memory, and no load could be issued ahead of it.  At
      // BN2 = 128 both accumulators hold 128 of the 168 registers, and a first block of 4 or more groups spills.
      constexpr int JB1 = BN2 == 128 ? 2 : FMB_NC / 8;
#pragma unroll
      for (int j0 = 0; j0 < FMB_NC / 8; j0 += JB1) {
        float2 bv[JB1];
#pragma unroll
        for (int jj = 0; jj < JB1; ++jj) {  // Cexp % 16 == 0: col + 1 is valid with col
          const int col = c * FMB_NC + 8 * (j0 + jj) + 2 * (lane & 3);
          bv[jj] = col < p.Cexp ? __ldg(reinterpret_cast<const float2*>(p.bias1 + col)) : make_float2(0.f, 0.f);
        }
        if (j0 == 0) {
          wgmma_wait<0>();
          wgmma_fence_regs<FMB_NC / 2>(acc1);
          __syncwarp();
          if (lane == 0) {
            mbar_arrive(&empty[prev]);
            if (c == p.nch - 1) mbar_arrive(box_empty);  // the tile's last read of its input boxes
          }
        }
#pragma unroll
        for (int jj = 0; jj < JB1; ++jj) {
          const int j = j0 + jj, cc = 8 * j + 2 * (lane & 3);  // column within the chunk
          const bool live = c * FMB_NC + cc < p.Cexp;
          const uint32_t sub = (uint32_t)(cc >> 6) * (TC_BM * 128), kc = (uint32_t)(cc & 63);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = r0 + 8 * h;
            const uint32_t v = pair16_bits<T>(
                Pair16<T>::pack(tc_act<ACT_SILU, T>(acc1[4 * j + 2 * h] + bv[jj].x), tc_act<ACT_SILU, T>(acc1[4 * j + 2 * h + 1] + bv[jj].y)));
            const uint32_t off = sub + (uint32_t)r * 128 + ((((kc >> 3) ^ (uint32_t)(r & 7))) << 4) + (kc & 7) * 2;
            // zeros past Cexp by a select: a branch per column pair kept ptxas from overlapping the columns' SiLU chains
            st_shared_b32(a2 + off, live ? v : 0u);
          }
        }
      }
      fence_proxy_async();  // generic-proxy writes -> visible to the tensor core (async proxy)
      wg_sync(wg);
      // ---- GEMM-2: acc2 += A2 x W2[:, chunk]^T, the two 64-channel halves of the W2 slice in consecutive stages ----
      // Not waited for here: the next chunk's first GEMM-1 k-block is issued behind it, and its wgmma.wait_group 1 retires
      // this group (groups retire in order) before the stages are released and before epilogue-1 rewrites A2.  The last
      // chunk's group is waited for under epilogue-2's first loads.
      {
        const int s0 = it % STAGES, s1 = (it + 1) % STAGES;
        mbar_wait(&full[s0], (it / STAGES) & 1);
        mbar_wait(&full[s1], ((it + 1) / STAGES) & 1);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < FMB_NC / 16; ++k) {
          const uint32_t sub = (uint32_t)(k >> 2), ko = (uint32_t)(k & 3) * 32;
          const uint32_t b = ring + (sub ? s1 : s0) * FMB_W_BYTES;
          wgmma_16b<T, BN2>(acc2, gmma_desc<128>(a2 + sub * (TC_BM * 128) + wg * 64 * 128 + ko), gmma_desc<128>(b + ko), (uint32_t)(c | k));
        }
        wgmma_commit();
        it += 2;
      }
    }
    // ---- epilogue-2: + bias, + residual x, 16-bit store ----
    // All of the thread's bias and residual pairs are loaded in one batch while the last chunk's GEMM-2 runs: issued one by
    // one between the stores, which might alias them, each waited out its L2 latency with the MMAs of both warpgroups idle.
    // Every batch element is set on every path: an element left unset where its load is skipped stays live around the
    // whole tile loop, next to both accumulators, and at BN2 = 128 that spilled.
    const int c0 = 2 * (lane & 3);
    float2 bv[BN2 / 8];
    T2 rv[2][BN2 / 8];
    size_t off[2];
    bool row_ok[2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
      row_ok[h] = tile_row_offset(1, t, r0 + 8 * h, g.M, g.Cout, g.tiles_w, g.tiles_h, g.Hout, g.Wout, off[h]);
#pragma unroll
    for (int j = 0; j < BN2 / 8; ++j) {
      const int cidx = c0 + 8 * j;
      bv[j] = cidx < g.Cout ? __ldg(reinterpret_cast<const float2*>(g.bias + cidx)) : make_float2(0.f, 0.f);
#pragma unroll
      for (int h = 0; h < 2; ++h)
        rv[h][j] = p.has_res && row_ok[h] && cidx < g.Cout ? *reinterpret_cast<const T2*>(res + off[h] + cidx) : Pair16<T>::pack(0.f, 0.f);
    }
    wgmma_wait<0>();
    wgmma_fence_regs<BN2 / 2>(acc2);
    __syncwarp();
    if (lane == 0) {
      mbar_arrive(&empty[(it - 2) % STAGES]);
      mbar_arrive(&empty[(it - 1) % STAGES]);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!row_ok[h]) continue;
#pragma unroll
      for (int j = 0; j < BN2 / 8; ++j) {
        const int cidx = c0 + 8 * j;
        if (cidx >= g.Cout) break;
        float o0 = acc2[4 * j + 2 * h] + bv[j].x, o1 = acc2[4 * j + 2 * h + 1] + bv[j].y;
        if (p.has_res) {
          const float2 f = Pair16<T>::unpack(rv[h][j]);
          o0 += f.x;
          o1 += f.y;
        }
        *reinterpret_cast<T2*>(out + off[h] + cidx) = Pair16<T>::pack(o0, o1);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ host side
struct FmbWeights {
  bool ready = false;
  const TcWeights* w1 = nullptr;  // the expand conv's 16-bit K-major weights [Cexp][9*Cin] + bias
  const TcWeights* w2 = nullptr;  // the projection's [Cout][Cexp] + bias
  int Cin = 0, Cexp = 0, Cout = 0, bn2 = 0;
  mutable TmapCache maps;         // (block input in 16 x 10-pixel boxes for tma_load_tap_boxes, W1, W2)
};

// shapes the fused kernel covers: 3x3 stride-1 expand (SiLU) + 1x1 projection, Cin = Cout (identity-shaped block).
// Cin = Cout a multiple of 8 but not of 16 (24, 40, 56, 72, 88; EfficientNetV2-B2 / -B3 run 40 and 56) takes the same path as
// the multiples of 16, with nothing left over per 16-wide k step that is not already zeros:
//  - every row stride is a multiple of 16 bytes, as the TMA requires: input pixels 2 Cin (80, 112 B), W1 rows 18 Cin, W2 rows
//    2 Cexp = 8 Cin;
//  - the boxes' channels Cin..63 of a 64-channel k-chunk are TMA zero fill, and they meet the columns tap * Cin + Cin.. of the
//    tap's W1 k-block (the next tap's first columns, or zero fill past 9 Cin): the products are zeros, the same ones
//    tc_conv_kernel multiplies on its own 3x3 launch, whose k-blocks start at the same tap * Cin + kc * 64;
//  - Cexp = 4 Cin is a multiple of 32, so a partial last expand chunk (Cexp 160, 224) ends on a 16-wide k step of GEMM-2:
//    A2 holds zeros from Cexp on and the W2 columns past Cexp are zero fill, so GEMM-2 adds zero products after the
//    projection's own k-blocks (as at Cexp 192), and every bias1 pair col, col + 1 lies below Cexp or both past it;
//  - BN2 = tc_pick_bn(Cout) = 64 at Cout 40, 56 (32 at 24, 128 at 72, 88), with one k-chunk exactly when Cin <= 64; W2 rows
//    Cout..BN2-1 are zero fill, and epilogue-2 stops at the first column pair >= Cout, each pair (bias, residual, output)
//    4-byte aligned because Cout and the pair's column are even.
inline bool fmb_shape_ok(int cin, int cexp, int cout) {
  return cin % 8 == 0 && cin >= 16 && cin <= 96 && cout == cin && cexp % 16 == 0 && cexp >= 32 && cexp <= 512;
}

inline void fmb_prepare(FmbWeights& f, const TcWeights& w1, const TcWeights& w2) {
  f.ready = false;
  if (!fmb_shape_ok(w1.Cin, w1.Cout, w2.Cout) || w2.Cin != w1.Cout || w1.taps != 9) return;
  f.w1 = &w1; f.w2 = &w2;
  f.Cin = w1.Cin; f.Cexp = w1.Cout; f.Cout = w2.Cout;
  f.bn2 = tc_pick_bn(f.Cout);
  f.ready = true;
}

template <typename T>
inline const char* fmb_launch(const FmbWeights& f, const void* in, void* out, int B, int H, int W, int pad_t, int pad_l, bool has_res,
                              cudaStream_t st) {
  if (!f.ready) return "fused FusedMBConv block not prepared";
  FmbParams q;
  TcConvParams& g = q.g;
  g.res = in; g.bias = f.w2->d_bias; g.out = out;
  g.mode = 1;
  g.Hin = H; g.Win = W; g.Hout = H; g.Wout = W;
  g.Cin = f.Cin; g.Cout = f.Cout;
  g.taps = 9; g.S = 3; g.stride = 1; g.dil = 1; g.pad_t = pad_t; g.pad_l = pad_l;
  g.kchunks = (f.Cin + TC_BK - 1) / TC_BK;
  g.tiles_w = (W + TC_TILE_W - 1) / TC_TILE_W;
  g.tiles_h = (H + TC_TILE_H - 1) / TC_TILE_H;
  g.M = B * H * W;
  q.bias1 = f.w1->d_bias;
  q.Cexp = f.Cexp;
  q.nch = (f.Cexp + FMB_NC - 1) / FMB_NC;
  q.has_res = has_res ? 1 : 0;
  const CUtensorMap* m = nullptr;  // block input, W1, W2
  const char* e = f.maps.get(&m, [&](CUtensorMap* c) {
    const CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_128B;
    const char* r = make_tmap_nhwc<T>(&c[0], in, B, H, W, f.Cin, TC_BK, TC_TILE_W, FMB_BOX_H, 1, 1, sw);
    if (!r) r = make_tmap_2d<T>(&c[1], f.w1->d_w, f.Cexp, (uint64_t)9 * f.Cin, FMB_NC, TC_BK, sw);
    return r ? r : make_tmap_2d<T>(&c[2], f.w2->d_w, f.Cout, f.Cexp, f.bn2, TC_BK, sw);
  }, in, f.w1->d_w, f.w2->d_w, B, H, W, f.Cin, f.Cexp, f.Cout, f.bn2);
  if (e) return e;
  g.m_tiles = B * g.tiles_w * g.tiles_h;
  const int grid = std::min(g.m_tiles, num_sms());  // persistent: one CTA per SM
  return with_const<32, 64, 128>(f.bn2, "unsupported N tile", [&](auto bn2) {
    if (q.g.kchunks != FmbSmem<bn2>::kchunks) return "fmb_kernel: k-chunks do not match the output width";
    return launch_smem(fmb_kernel<T, bn2>, dim3(grid), dim3(TC_THREADS), FmbSmem<bn2>::smem_bytes, st, m[0], m[1], m[2], q);
  });
}

}  // namespace mtb
